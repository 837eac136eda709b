"""trb_scene_replace_settings and trb_scene_replace_materials without a GPU: the exports and their ctypes declarations against the Rust
ones in INTEGRATION.md, the layouts of trb_scene_materials, trb_film and trb_integrator as a plain-C caller sees them against the ctypes
mirrors, the null-argument statuses, and the builder helpers: materials_section() is the material section of finish(), and
remove_material, remove_texture and remove_merl_table leave the builder that never added the entry."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, scenebuild as SB

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAT_ARGS = r"scene: \*mut c_void, materials: \*const TrbSceneMaterials, objects: \*const TrbSceneObjects"
FUNCS = {"trb_scene_replace_settings": r"scene: \*mut c_void, film: \*const TrbFilm, integrator: \*const TrbIntegrator",
         "trb_scene_replace_materials": MAT_ARGS, "trb_scene_replace_materials_device": MAT_ARGS + r",\s*cuda_stream: \*mut c_void"}


def rust_fields(doc, c_name, rust_name, size):
    m = re.search(r"// %s: .*, %d bytes\npub struct %s \{(.*?)\}" % (c_name, size, rust_name), doc, re.S)
    assert m, rust_name
    return [f if f != "ty" else "type" for f in re.findall(r"(\w+)\s*:", m.group(1))]


def test_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for name, args in FUNCS.items():
        assert hasattr(trb, name) and name in F.TRB_SYMBOLS
        assert re.search(r"fn %s\(%s\)\s*->\s*c_int;" % (name, args), doc), name
        assert "`%s(" % name in doc, "no table row for " + name
    assert trb.trb_scene_replace_settings.argtypes == [C.c_void_p, C.POINTER(F.Film), C.POINTER(F.Integrator)]
    assert trb.trb_scene_replace_materials.argtypes == [C.c_void_p, C.POINTER(F.SceneMaterials), C.POINTER(F.SceneObjects)]
    assert trb.trb_scene_replace_materials_device.argtypes == [C.c_void_p, C.POINTER(F.SceneMaterials), C.POINTER(F.SceneObjects), C.c_void_p]
    for c_name, rust_name, cls in (("trb_scene_materials", "TrbSceneMaterials", F.SceneMaterials), ("trb_film", "TrbFilm", F.Film),
                                   ("trb_integrator", "TrbIntegrator", F.Integrator), ("trb_texture", "TrbTexture", F.Texture),
                                   ("trb_image", "TrbImage", F.Image)):
        assert rust_fields(doc, c_name, rust_name, C.sizeof(cls)) == [f for f, _ in cls._fields_], rust_name


def test_plain_c_caller_sees_the_ctypes_layout_and_the_null_statuses(tmp_path):
    exe = str(tmp_path / "scene_settings_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "scene_settings_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = [l.split() for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()]
    for name, cls in (("trb_scene_materials", F.SceneMaterials), ("trb_film", F.Film), ("trb_integrator", F.Integrator)):
        assert ["sizeof", name, str(C.sizeof(cls))] in out
    assert [(l[1], int(l[2])) for l in out if l[0] == "offset"] == [(f, getattr(F.SceneMaterials, f).offset) for f, _ in F.SceneMaterials._fields_]
    status = {l[1]: int(l[2]) for l in out if l[0] == "status"}
    assert status == {"settings_null_scene": F.TRB_INVALID_ARG, "settings_all_null": F.TRB_INVALID_ARG, "materials_null_scene": F.TRB_INVALID_ARG,
                      "materials_null_scene_device": F.TRB_INVALID_ARG, "materials_null_both": F.TRB_INVALID_ARG, "TRB_INVALID_ARG": F.TRB_INVALID_ARG}
    # the section's fields are the description's
    desc = dict(F.SceneDesc._fields_)
    assert all(desc[f] is t for f, t in F.SceneMaterials._fields_)


def test_null_scene_or_null_section_needs_no_device(trb):
    b = SB.scene_materials_zoo(32, 32, 2)
    d = b.finish()
    s, o = b.materials_section(), b.objects()
    assert trb.trb_scene_replace_settings(None, C.byref(d.film), C.byref(d.integrator)) == F.TRB_INVALID_ARG
    assert trb.trb_last_error() == b"null scene"
    assert trb.trb_scene_replace_settings(None, None, None) == F.TRB_INVALID_ARG
    for f in (trb.trb_scene_replace_materials, lambda *a: trb.trb_scene_replace_materials_device(*a, None)):
        assert f(None, C.byref(s), C.byref(o)) == F.TRB_INVALID_ARG
        assert trb.trb_last_error() == b"null scene"
        assert f(None, None, None) == F.TRB_INVALID_ARG


def section_of(d):
    """a SceneDesc's or SceneMaterials' material section as plain values: material records, MERL tables, textures, images with texels"""
    mats = [bytes(d.materials[i]) for i in range(d.n_materials)]
    merl = [C.string_at(d.merl_tables[i], F.MERL_TABLE_FLOATS * 4) for i in range(d.n_merl)]
    tex = [(d.textures[i].first_image, d.textures[i].n_images) for i in range(d.n_textures)]
    img = [(d.images[i].width, d.images[i].height, d.images[i].time, C.string_at(d.images[i].rgba8, 4 * d.images[i].width * d.images[i].height))
           for i in range(d.n_images)]
    return mats, merl, tex, img


def frames(seed, n, size=4):
    rng = np.random.default_rng(seed)
    return [(rng.integers(0, 256, (size, size + k, 4), dtype=np.uint8), 0.25 * k) for k in range(n)]


MERL_USER = {0: 1, 1: 3}  # table -> the material (of the five below) that uses it
TEX_USER = {0: 0, 1: 4, 2: 2}  # texture -> the material that is bound to it


def with_entries(skip_material=None, skip_texture=None, skip_merl=None):
    """scene_materials_zoo with three textures (one animated), two MERL tables and five materials using them, each on a sphere, built
    from scratch without the entries named: a skipped texture leaves its material unbound, a skipped table goes with its material"""
    b = SB.scene_materials_zoo(32, 32, 2)
    tex = {k: b.add_texture(frames(k, n)) for k, n in enumerate((1, 3, 1)) if k != skip_texture}
    merl = {k: b.add_merl_table(SB.synthetic_merl_table(seed=k + 1) * (k + 1)) for k in range(2) if k != skip_merl}
    specs = [(F.MAT_MATTE, dict(tex_c0=tex.get(0, 0))), (F.MAT_MERL, dict(merl=merl.get(0))), (F.MAT_PLASTIC, dict(tex_c1=tex.get(2, 0))),
             (F.MAT_MERL, dict(merl=merl.get(1))), (F.MAT_GLASS, dict(tex_eta=tex.get(1, 0)))]
    for k, (mtype, kw) in enumerate(specs):
        if k == skip_material or (skip_merl is not None and k == MERL_USER[skip_merl]):
            continue
        m = b.add_material(mtype, (0.5, 0.4, 0.3), (0.6, 0.6, 0.6), roughness=0.2, eta=1.4, **kw)
        b.receiver(F.SHAPE_SPHERE, m, [SB.trs(t=(k, 5, 3))], p0=1.0)
    return b


def user_of(b, k):
    """the index of the five materials' k-th in b, and the instance that uses it"""
    m = len(b.materials) - 5 + k
    return m, [i for i, it in enumerate(b.instances) if it[0] != F.INST_EMITTER_POINT and it[5] == m][0]


def test_section_is_the_material_section_of_finish():
    b = with_entries()
    assert section_of(b.materials_section()) == section_of(b.finish())
    assert len(section_of(b.finish())[3]) == 5


@pytest.mark.parametrize("victim", [0, 1, 2])
def test_remove_texture_renumbers_to_the_builder_that_never_added_it(victim):
    b = with_entries()
    with pytest.raises(ValueError, match="used by materials"):
        b.remove_texture(victim)
    m, _ = user_of(b, TEX_USER[victim])
    b.materials[m] = b.materials[m][:6] + ((0, 0, 0, 0),)
    removed = b.remove_texture(victim)
    assert len(removed) == (1, 3, 1)[victim]
    scratch = with_entries(skip_texture=victim)
    assert b.materials == scratch.materials and b.textures == scratch.textures
    assert section_of(b.materials_section()) == section_of(scratch.materials_section())


@pytest.mark.parametrize("victim", [0, 1])
def test_remove_merl_table_renumbers_to_the_builder_that_never_added_it(victim):
    b = with_entries()
    with pytest.raises(ValueError, match="used by materials"):
        b.remove_merl_table(victim)
    m, inst = user_of(b, MERL_USER[victim])
    b.remove_instance(inst)
    b.remove_material(m)
    b.remove_merl_table(victim)
    scratch = with_entries(skip_merl=victim)
    assert b.instances == scratch.instances and b.materials == scratch.materials
    assert section_of(b.materials_section()) == section_of(scratch.materials_section())


@pytest.mark.parametrize("victim", [0, 2, 4])
def test_remove_material_renumbers_to_the_builder_that_never_added_it(victim):
    b = with_entries()
    m, inst = user_of(b, victim)
    with pytest.raises(ValueError, match="used by instances"):
        b.remove_material(m)
    b.remove_instance(inst)
    b.remove_material(m)
    scratch = with_entries(skip_material=victim)
    assert b.instances == scratch.instances and b.materials == scratch.materials
    assert section_of(b.materials_section()) == section_of(scratch.materials_section())
