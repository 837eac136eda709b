"""trb_scene_replace_objects without a GPU: the export and its ctypes declaration against the Rust one in INTEGRATION.md, the layout of
trb_scene_objects as a plain-C caller sees it against the ctypes mirror, the null-argument statuses, and the builder helpers:
SceneBuilder.objects() is the object section of finish(), and remove_instance leaves the builder that never added the instance."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, scenebuild as SB

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SECTION = ["cameras", "instances", "splines", "keyframes", "knots", "color_keys", "fov_floats"]


def test_symbol_is_exported_and_bound_like_the_rust_declaration(trb):
    name = "trb_scene_replace_objects"
    assert hasattr(trb, name) and name in F.TRB_SYMBOLS
    assert getattr(trb, name).argtypes == [C.c_void_p, C.POINTER(F.SceneObjects)]
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    assert re.search(r"fn %s\(scene: \*mut c_void, objects: \*const TrbSceneObjects\)\s*->\s*c_int;" % name, doc)
    assert "`%s(" % name in doc, "no table row"
    m = re.search(r"pub struct TrbSceneObjects \{(.*?)\}", doc, re.S)
    assert m and re.findall(r"(\w+)\s*:", m.group(1)) == [f for f, _ in F.SceneObjects._fields_]
    assert re.search(r"// trb_scene_objects: .*, %d bytes\npub struct TrbSceneObjects " % C.sizeof(F.SceneObjects), doc)


def test_plain_c_caller_sees_the_ctypes_layout_and_the_null_statuses(tmp_path):
    exe = str(tmp_path / "scene_objects_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "scene_objects_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = [l.split() for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()]
    assert ["sizeof", "trb_scene_objects", str(C.sizeof(F.SceneObjects))] in out
    assert [(l[1], int(l[2])) for l in out if l[0] == "offset"] == [(f, getattr(F.SceneObjects, f).offset) for f, _ in F.SceneObjects._fields_]
    status = {l[1]: int(l[2]) for l in out if l[0] == "status"}
    assert status == {"null_scene": F.TRB_INVALID_ARG, "null_both": F.TRB_INVALID_ARG, "TRB_INVALID_ARG": F.TRB_INVALID_ARG}
    # the section's fields are the description's, name for name and type for type
    desc = dict(F.SceneDesc._fields_)
    assert all(desc[f] is t for f, t in F.SceneObjects._fields_)


def test_null_scene_or_null_objects_needs_no_device(trb):
    o = SB.scene_instances(2, 1).objects()
    assert trb.trb_scene_replace_objects(None, C.byref(o)) == F.TRB_INVALID_ARG
    assert trb.trb_last_error() == b"null scene"
    assert trb.trb_scene_replace_objects(None, None) == F.TRB_INVALID_ARG


def section(d):
    """the seven arrays of a SceneDesc or SceneObjects as bytes"""
    out = {}
    for name in SECTION:
        n, p = getattr(d, "n_" + name), getattr(d, name)
        out[name] = (n, C.string_at(p, n * C.sizeof(p._type_)) if n else b"")
    return out


def test_objects_is_the_object_section_of_finish():
    for b in (SB.scene_animated(32, 32, 2, animated_fov=True), SB.scene_materials_zoo(32, 32, 2), SB.scene_instances(7, 3)):
        assert section(b.objects()) == section(b.finish())


def zoo_with(extra, skip=()):
    """scene_materials_zoo's objects plus the `extra` ones, built from scratch without the additions named in `skip`"""
    b = SB.scene_materials_zoo(32, 32, 2)
    spin = SB.Anim([SB.trs(q=SB.quat_axis_angle((0, 1, 0), a)) for a in (0, 90, 170, 250)], degree=2)
    adds = {
        "keyed": lambda: b.receiver(F.SHAPE_SPHERE, 3, [spin, SB.trs(t=(0, 4, 0), s=3.0)], p0=1.0),
        "light": lambda: b.area_light(F.SHAPE_DISK, 0, [SB.trs(t=(1, 20, 2))], [((1.0, 0.6, 0.3, 30), 0.0), ((0.3, 1.0, 0.4, 60), 0.4)], p0=2.0),
        "point": lambda: b.point_light([SB.Anim([SB.trs(t=(-10, 15, -12)), SB.trs(t=(10, 18, -10))], degree=1)], (1, 1, 1, 50)),
        "sphere": lambda: b.receiver(F.SHAPE_SPHERE, 4, [SB.trs(t=(2, 2, 2))], p0=0.5),
    }
    index = {}
    for name in extra:
        if name not in skip:
            index[name] = adds[name]()
    b.add_camera([SB.Anim([SB.trs(t=(-3, 12, -60)), SB.trs(t=(4, 12, -60))], degree=1)], fov=[28.0, 34.0, 30.0], fov_degree=2, active_at=2)
    return b, index


@pytest.mark.parametrize("victim", ["keyed", "light", "point", "sphere"])
def test_remove_instance_compacts_to_the_builder_that_never_added_it(victim):
    extra = ["keyed", "light", "point", "sphere"]
    b, index = zoo_with(extra)
    removed = b.remove_instance(index[victim])
    assert removed[0] == {"keyed": F.INST_RECEIVER, "light": F.INST_EMITTER_AREA, "point": F.INST_EMITTER_POINT, "sphere": F.INST_RECEIVER}[victim]
    scratch, _ = zoo_with(extra, skip=(victim,))
    assert section(b.objects()) == section(scratch.objects())
    for name in ("instances", "splines", "keyframes", "knots", "color_keys", "cameras", "fov_floats"):
        assert getattr(b, name) == getattr(scratch, name), name


def test_remove_every_added_instance_in_any_order_restores_the_scene():
    extra = ["keyed", "light", "point", "sphere"]
    base, _ = zoo_with([])
    rng = np.random.default_rng(4)
    for _ in range(4):
        b, index = zoo_with(extra)
        for name in rng.permutation(extra):
            i = index[name]
            b.remove_instance(i)
            index = {k: v - (v > i) for k, v in index.items()}
        assert section(b.objects()) == section(base.objects())
