"""trb_scene_replace_meshes without a GPU: the exports and their ctypes declarations against the Rust ones in INTEGRATION.md, the layout
of trb_scene_meshes as a plain-C caller sees it against the ctypes mirror, the null-argument statuses, and the builder helpers:
meshes_section() is the mesh list of finish() with `keep` naming the meshes the scene already has, set_mesh makes a mesh new, and
remove_mesh leaves the builder that never added the mesh. (A `keep` entry out of range or repeated needs a scene, so a device: the
GPU tests check those statuses.)"""
import ctypes as C
import os
import re
import subprocess

import pytest

from tray_rust_b200 import _ffi as F, scenebuild as SB

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARGS = r"scene: \*mut c_void, meshes: \*const TrbSceneMeshes, objects: \*const TrbSceneObjects"
FUNCS = {"trb_scene_replace_meshes": ARGS, "trb_scene_replace_meshes_device": ARGS + r",\s*cuda_stream: \*mut c_void"}


def test_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for name, args in FUNCS.items():
        assert hasattr(trb, name) and name in F.TRB_SYMBOLS
        assert re.search(r"fn %s\(%s\)\s*->\s*c_int;" % (name, args), doc), name
        assert "`%s(" % name in doc, "no table row for " + name
    assert trb.trb_scene_replace_meshes.argtypes == [C.c_void_p, C.POINTER(F.SceneMeshes), C.POINTER(F.SceneObjects)]
    assert trb.trb_scene_replace_meshes_device.argtypes == [C.c_void_p, C.POINTER(F.SceneMeshes), C.POINTER(F.SceneObjects), C.c_void_p]
    m = re.search(r"// trb_scene_meshes: .*, %d bytes\npub struct TrbSceneMeshes \{(.*?)\}" % C.sizeof(F.SceneMeshes), doc, re.S)
    assert m and re.findall(r"(\w+)\s*:", m.group(1)) == [f for f, _ in F.SceneMeshes._fields_]
    m = re.search(r"// trb_mesh: .*, %d bytes\npub struct TrbMesh \{(.*?)\}" % C.sizeof(F.Mesh), doc, re.S)
    assert m and re.findall(r"(\w+)\s*:", m.group(1)) == [f for f, _ in F.Mesh._fields_]
    assert re.search(r"const TRB_MESH_NEW: u32 = 0x%x;" % F.MESH_NEW, doc, re.I)


def test_plain_c_caller_sees_the_ctypes_layout_and_the_null_statuses(tmp_path):
    exe = str(tmp_path / "mesh_replace_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "mesh_replace_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = [l.split() for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()]
    assert ["sizeof", "trb_scene_meshes", str(C.sizeof(F.SceneMeshes))] in out
    assert [(l[1], int(l[2])) for l in out if l[0] == "offset"] == [(f, getattr(F.SceneMeshes, f).offset) for f, _ in F.SceneMeshes._fields_]
    assert ["const", "TRB_MESH_NEW", str(F.MESH_NEW)] in out
    status = {l[1]: int(l[2]) for l in out if l[0] == "status"}
    assert status == {"null_scene": F.TRB_INVALID_ARG, "null_scene_device": F.TRB_INVALID_ARG, "null_both": F.TRB_INVALID_ARG,
                      "TRB_INVALID_ARG": F.TRB_INVALID_ARG}
    # the section's mesh array is the description's
    assert dict(F.SceneDesc._fields_)["meshes"] is dict(F.SceneMeshes._fields_)["meshes"]


def test_null_scene_or_null_section_needs_no_device(trb):
    b = SB.scene_instances(2, 1, mesh=True)
    b.finish()
    s, o = b.meshes_section(), b.objects()
    for f in (trb.trb_scene_replace_meshes, lambda *a: trb.trb_scene_replace_meshes_device(*a, None)):
        assert f(None, C.byref(s), C.byref(o)) == F.TRB_INVALID_ARG
        assert trb.trb_last_error() == b"null scene"
        assert f(None, None, None) == F.TRB_INVALID_ARG


def meshes_of(d):
    """a SceneDesc's or SceneMeshes' mesh list as (n_verts, n_tris, the four arrays' bytes)"""
    out = []
    for i in range(d.n_meshes):
        m = d.meshes[i]
        out.append((m.n_verts, m.n_tris) + tuple(C.string_at(p, k * 4) for p, k in
                                                 ((m.positions, 3 * m.n_verts), (m.normals, 3 * m.n_verts), (m.texcoords, 2 * m.n_verts),
                                                  (m.indices, 3 * m.n_tris))))
    return out


def test_section_is_the_mesh_list_of_finish_and_keeps_what_the_scene_has():
    b = SB.scene_materials_zoo(32, 32, 2)
    b.add_mesh(*SB.icosphere_mesh(1))
    d = b.finish()
    s = b.meshes_section()
    assert meshes_of(s) == meshes_of(d) and list(s.keep[:s.n_meshes]) == [0, 1]
    b.set_mesh(0, *SB.icosphere_mesh(3))
    b.add_mesh(*SB.icosphere_mesh(0))
    s = b.meshes_section()
    assert list(s.keep[:s.n_meshes]) == [F.MESH_NEW, 1, F.MESH_NEW]
    assert s.meshes[0].n_tris == 1280 and s.meshes[2].n_tris == 20
    s = b.meshes_section()  # relative to the section just given
    assert list(s.keep[:s.n_meshes]) == [0, 1, 2]
    b.meshes[0], b.meshes[2] = b.meshes[2], b.meshes[0]
    s = b.meshes_section()
    assert list(s.keep[:s.n_meshes]) == [2, 1, 0]


def with_meshes(skip=None):
    """scene_materials_zoo (its icosphere is mesh 0) with three more meshes and an instance of each, built from scratch without mesh
    `skip` and its instance"""
    b = SB.scene_materials_zoo(32, 32, 2)
    for k, subdiv in enumerate((0, 1, 2)):
        if k + 1 == skip:
            continue
        m = b.add_mesh(*SB.icosphere_mesh(subdiv, 1.0 + k, 0.1, k))
        b.receiver(F.SHAPE_MESH, 2, [SB.trs(t=(k, 5, 3))], mesh=m)
    return b


@pytest.mark.parametrize("victim", [1, 2, 3])
def test_remove_mesh_renumbers_to_the_builder_that_never_added_it(victim):
    b = with_meshes()
    with pytest.raises(ValueError, match="used by instances"):
        b.remove_mesh(victim)
    user = [k for k, it in enumerate(b.instances) if it[1] == F.SHAPE_MESH and it[4] == victim]
    b.remove_instance(user[0])
    removed = b.remove_mesh(victim)
    assert len(removed[3]) == 20 * 4 ** (victim - 1)
    scratch = with_meshes(skip=victim)
    assert b.instances == scratch.instances
    assert meshes_of(b.finish()) == meshes_of(scratch.finish())
    assert meshes_of(b.meshes_section()) == meshes_of(scratch.meshes_section())
