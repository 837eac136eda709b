"""trb_scene_update_mesh without a GPU: the exports, the ctypes declarations against the Rust ones in INTEGRATION.md, a plain-C caller's
statuses, and Scene.update_mesh's shape checks, which raise before anything reaches the library."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_scene_update_mesh", "trb_scene_update_mesh_device"]


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


def test_plain_c_caller_gets_the_argument_statuses(tmp_path):
    exe = str(tmp_path / "mesh_update_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "mesh_update_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    status = {l.split()[1]: int(l.split()[2]) for l in out if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {"trb_scene_update_mesh:null_scene": F.TRB_INVALID_ARG, "trb_scene_update_mesh:null_all": F.TRB_INVALID_ARG,
                      "trb_scene_update_mesh_device:null_scene": F.TRB_INVALID_ARG, "trb_scene_update_mesh_device:null_all": F.TRB_INVALID_ARG}


def test_null_scene_needs_no_device(trb):
    v = np.zeros(9, np.float32)
    assert trb.trb_scene_update_mesh(None, 0, F.ptr(v), None, None) == F.TRB_INVALID_ARG
    assert trb.trb_scene_update_mesh_device(None, 0, None, None, None, None) == F.TRB_INVALID_ARG


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError("reached the library: " + name)


def _unopened_scene():
    """a Scene over a real description whose library handle fails on any use: the checks must raise first"""
    b = SB.SceneBuilder(8, 8, 1)
    mats = SB.cornell_walls(b)
    SB.cornell_light(b, mats["white"])
    m = b.add_mesh(*SB.heightfield_mesh(4, 1))
    b.receiver(F.SHAPE_MESH, mats["white"], [SB.trs()], mesh=m)
    b.add_camera([SB.trs(t=(0, 12, -60))])
    s = api.Scene.__new__(api.Scene)
    s._desc, s._lib, s._h = b.finish(), _NoLibrary(), None
    return s


@pytest.mark.parametrize("kw", [dict(positions=np.zeros((15, 3))), dict(positions=np.zeros((16, 2))), dict(normals=np.zeros((16, 4))),
                                dict(texcoords=np.zeros((16, 3))), dict(texcoords=np.zeros(33)), dict(positions=np.zeros((16, 3)), normals=np.zeros(47))])
def test_update_mesh_rejects_wrong_shapes_before_the_library(kw):
    s = _unopened_scene()
    assert s._desc.meshes[0].n_verts == 16
    with pytest.raises(ValueError):
        s.update_mesh(0, **kw)


def test_update_mesh_rejects_a_mesh_index_out_of_range_before_the_library():
    s = _unopened_scene()
    for k in (1, -1):
        with pytest.raises(ValueError):
            s.update_mesh(k, positions=np.zeros((16, 3)))
        with pytest.raises(ValueError):
            s.update_mesh_device(k, 1)
    s._h = None
    assert s.close() is None  # a handle that was never opened is not destroyed
