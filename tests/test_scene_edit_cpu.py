"""The scene edits (trb_scene_update_keyframes / _device / _color_keys / _materials) without a GPU: the exports, the ctypes declarations
against the Rust ones in INTEGRATION.md, a plain-C caller's statuses, and the Scene wrappers' checks, which raise before anything
reaches the library."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_scene_update_keyframes", "trb_scene_update_keyframes_device", "trb_scene_update_color_keys", "trb_scene_update_materials"]


def test_new_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for name in NEW:
        assert hasattr(trb, name) and name in F.TRB_SYMBOLS, name
        m = re.search(r"fn %s\((.*?)\)\s*->\s*c_int;" % name, doc, re.S)
        assert m, name
        rust = [p.split(":", 1)[1].strip() for p in m.group(1).split(",") if p.strip()]
        ct = getattr(trb, name).argtypes
        assert len(ct) == len(rust), name
        for i, (r, c) in enumerate(zip(rust, ct)):
            if r.startswith("*"):
                assert c is C.c_void_p or issubclass(c, C._Pointer), (name, i, r, c)
            else:
                assert c is {"u32": C.c_uint32, "c_int": C.c_int}[r], (name, i, r, c)
        assert "`%s(" % name in doc, "no table row for " + name


def test_dtypes_match_the_structures_and_the_rust_declarations():
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for dt, st, rust, size in ((F.KEYFRAME_DTYPE, F.Keyframe, "TrbKeyframe", 40), (F.COLOR_KEY_DTYPE, F.ColorKey, "TrbColorKey", 20),
                               (F.MATERIAL_DTYPE, F.Material, "TrbMaterial", 56)):
        assert dt.itemsize == C.sizeof(st) == size
        assert [n for n, _ in st._fields_] == list(dt.names)
        assert re.search(r"pub struct %s \{" % rust, doc), rust
        assert re.search(r"// trb_\w+: .*, %d bytes\npub struct %s " % (size, rust), doc), rust


def test_plain_c_caller_gets_the_argument_statuses(tmp_path):
    exe = str(tmp_path / "scene_edit_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "scene_edit_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    status = {l.split()[1]: int(l.split()[2]) for l in out if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {"trb_scene_update_keyframes:null_scene": F.TRB_INVALID_ARG, "trb_scene_update_keyframes_device:null_scene": F.TRB_INVALID_ARG,
                      "trb_scene_update_color_keys:null_scene": F.TRB_INVALID_ARG, "trb_scene_update_materials:null_scene": F.TRB_INVALID_ARG,
                      "trb_scene_update_materials:null_scene_empty": F.TRB_INVALID_ARG}


def test_null_scene_needs_no_device(trb):
    kf = np.zeros(1, F.KEYFRAME_DTYPE)
    assert trb.trb_scene_update_keyframes(None, 0, 1, F.ptr(kf)) == F.TRB_INVALID_ARG
    assert trb.trb_scene_update_keyframes_device(None, 0, 1, F.ptr(kf), None) == F.TRB_INVALID_ARG
    assert trb.trb_scene_update_color_keys(None, 0, 0, None) == F.TRB_INVALID_ARG
    assert trb.trb_scene_update_materials(None, 0xffffffff, 2, None) == F.TRB_INVALID_ARG


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError("reached the library: " + name)


def _unopened_scene():
    """a Scene over a real description whose library handle fails on any use: the checks must raise first"""
    s = api.Scene.__new__(api.Scene)
    s._desc, s._lib, s._h = SB.scene_instances(3, 1).finish(), _NoLibrary(), None
    return s


def test_scene_instances_is_the_cornell_box_with_k_static_spheres():
    d = SB.scene_instances(5, 2).finish()
    # five walls and the light (two levels each but the light), then one static level per sphere, then the camera
    assert d.n_instances == 6 + 5 and d.n_keyframes == 5 * 2 + 1 + 5 + 1
    spheres = [d.instances[i] for i in range(6, 11)]
    assert all(s.shape == F.SHAPE_SPHERE and s.kind == F.INST_RECEIVER and s.n_splines == 1 for s in spheres)
    assert all(d.splines[s.spline_first].n_ctrl == 1 for s in spheres)
    a, b = SB.scene_instances(5, 2).finish(), SB.scene_instances(5, 3).finish()
    assert [tuple(a.keyframes[i].translation) for i in range(11, 16)] == [tuple(d.keyframes[i].translation) for i in range(11, 16)]
    assert [tuple(a.keyframes[i].translation) for i in range(11, 16)] != [tuple(b.keyframes[i].translation) for i in range(11, 16)]


@pytest.mark.parametrize("call", [
    lambda s: s.update_keyframes(0, np.zeros(2, np.float32)),                 # wrong dtype
    lambda s: s.update_keyframes(0, np.zeros((2, 1), F.KEYFRAME_DTYPE)),      # not 1-d
    lambda s: s.update_keyframes(14, np.zeros(2, F.KEYFRAME_DTYPE)),          # past the end (15 keyframes)
    lambda s: s.update_keyframes(-1, np.zeros(1, F.KEYFRAME_DTYPE)),
    lambda s: s.update_keyframes_device(10, 10, 1),
    lambda s: s.update_keyframes_device(0, -1, 1),
    lambda s: s.update_color_keys(0, np.zeros(1, F.KEYFRAME_DTYPE)),
    lambda s: s.update_color_keys(1, np.zeros(1, F.COLOR_KEY_DTYPE)),         # one colour key
    lambda s: s.update_materials(0, np.zeros(1, F.COLOR_KEY_DTYPE)),
    lambda s: s.update_materials(3, np.zeros(2, F.MATERIAL_DTYPE)),           # four materials
], ids=["kf_dtype", "kf_ndim", "kf_range", "kf_negative", "kf_device_range", "kf_device_count", "ck_dtype", "ck_range", "mat_dtype",
        "mat_range"])
def test_wrappers_reject_wrong_arrays_before_the_library(call):
    s = _unopened_scene()
    assert (s._desc.n_keyframes, s._desc.n_color_keys, s._desc.n_materials) == (15, 1, 4)
    with pytest.raises(ValueError):
        call(s)
