"""AOV renders without a GPU: the struct layout, the exports, the ctypes declarations against the Rust ones in INTEGRATION.md, a plain-C
caller's statuses, Scene.render_aov's shape checks (which raise before anything reaches the library), decode_nearest, and the oracle's
AOV records (oracle_aov) against known answers: a matte wall's albedo, normal and analytic depth, the float32 Fresnel formulas of
metal, plastic, clear and tinted glass restated step by step in numpy, a textured matte's bilinear texture sample, and misses."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_aov import pyaov as A
from test_mesh_update_cpu import _unopened_scene

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_render_aov", "trb_render_aov_device", "trb_render_samples_aov"]
f32 = np.float32


def test_aov_sample_layout_matches_the_header_and_the_rust_declaration(tmp_path):
    out = _run_abi(tmp_path)
    sizes = {l.split()[0]: int(l.split()[2]) for l in out if " sizeof " in l}
    offs = {l.split()[0]: int(l.split()[1]) for l in out if l.split()[0].count(".") == 1 and not l.startswith("status")}
    assert sizes == {"trb_aov_sample": 32, "trb_aov_film": 24}
    assert F.AOV_SAMPLE_DTYPE.itemsize == 32 and C.sizeof(F.AovFilm) == 24
    for name in F.AOV_SAMPLE_DTYPE.names:
        assert F.AOV_SAMPLE_DTYPE.fields[name][1] == offs["trb_aov_sample." + name], name
    for name, _ in F.AovFilm._fields_:
        assert getattr(F.AovFilm, name).offset == offs["trb_aov_film." + name], name
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for rust, fields in (("TrbAovSample", list(F.AOV_SAMPLE_DTYPE.names)), ("TrbAovFilm", [n for n, _ in F.AovFilm._fields_])):
        m = re.search(r"pub struct %s \{(.*?)\}" % rust, doc, re.S)
        assert m, rust
        assert re.findall(r"(\w+)\s*:", m.group(1)) == fields, rust


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
                assert c is {"u32": C.c_uint32, "usize": C.c_size_t, "c_int": C.c_int}[r], (name, i, r, c)
        assert "`%s(" % name in doc, "no table row for " + name


def _run_abi(tmp_path):
    exe = str(tmp_path / "aov_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "aov_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_plain_c_caller_gets_the_argument_statuses(tmp_path):
    status = {l.split()[1]: int(l.split()[2]) for l in _run_abi(tmp_path) if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {k: F.TRB_INVALID_ARG for k in ("trb_render_aov:null_scene", "trb_render_aov:null_cfg", "trb_render_aov_device:null_scene",
                                                     "trb_render_samples_aov:null_scene", "trb_render_samples_aov:null_buffers")}


def test_null_scene_needs_no_device(trb):
    cfg = api._cfg()
    film = np.zeros(4, np.float32)
    aov = F.AovFilm(None, None, None)
    assert trb.trb_render_aov(None, C.byref(cfg), F.ptr(film), C.byref(aov), None) == F.TRB_INVALID_ARG
    assert trb.trb_render_aov_device(None, C.byref(cfg), F.ptr(film), C.byref(aov), None, None) == F.TRB_INVALID_ARG
    assert trb.trb_render_samples_aov(None, C.byref(cfg), 0, None, None, None) == F.TRB_INVALID_ARG


@pytest.mark.parametrize("kw", [dict(film=np.zeros((8, 8, 3), np.float32)), dict(film=np.zeros((8, 8, 4), np.float64)),
                                dict(albedo=np.zeros((8, 8, 4), np.float64)), dict(normal=np.zeros((8, 4, 4), np.float32)),
                                dict(nearest=np.zeros((8, 8), np.uint32)), dict(nearest=np.zeros((8, 8, 1), np.uint64)),
                                dict(albedo=np.zeros((8, 8, 8), np.float32)[:, :, :4])])
def test_render_aov_rejects_wrong_shapes_before_the_library(kw):
    s = _unopened_scene()
    s.width, s.height = s._desc.film.width, s._desc.film.height  # what Scene.__init__ reads from the library
    assert (s.width, s.height) == (8, 8)
    with pytest.raises(ValueError):
        s.render_aov(**kw)
    s._h = None


def test_decode_nearest_splits_depth_and_instance():
    depth = np.array([1.5, np.inf, 0.0, 1e-30], np.float32)
    inst = np.array([7, F.MISS, 0, 123456], np.uint32)
    key = (depth.view(np.uint32).astype(np.uint64) << np.uint64(32)) | inst.astype(np.uint64)
    d, i = api.decode_nearest(key.reshape(2, 2))
    assert d.dtype == np.float32 and i.dtype == np.uint32 and d.shape == (2, 2)
    assert np.array_equal(d.reshape(-1).view(np.uint32), depth.view(np.uint32)) and np.array_equal(i.reshape(-1), inst)
    assert int(key[1]) == 0x7f800000ffffffff  # an all-miss pixel


# ---- the oracle's AOV records against known answers ---------------------------------------------------------------------------
def wall_scene(mtype=F.MAT_MATTE, c0=(0.2, 0.4, 0.6), c1=(0, 0, 0), roughness=0.0, eta=1.0, tex_c0=0, image=None, facing=True):
    """a 16x16 camera at z = -10 looking down +z at a 1000 x 1000 rectangle in the plane z = 0 (normal +z); facing=False turns the
    camera around, so every ray misses"""
    b = SB.SceneBuilder(16, 16, 2)
    if image is not None:
        tex_c0 = b.add_texture(image)
    m = b.add_material(mtype, c0=c0, c1=c1, roughness=roughness, eta=eta, tex_c0=tex_c0)
    b.receiver(F.SHAPE_RECT, m, [SB.trs()], p0=1000.0, p1=1000.0)
    b.point_light([SB.trs(t=(0, 0, -5))], (1, 1, 1, 10))
    b.add_camera([SB.trs(t=(0, 0, -10), q=(0, 0, 0, 1) if facing else SB.quat_axis_angle((0, 1, 0), 180))], fov=30.0)
    s = A.AovOracleScene(b.finish())
    s.update_frame(0, 0.0, 0.0)
    return s


def _albedo(mtype, **kw):
    s = wall_scene(mtype, **kw)
    _, aov, _ = s.render_samples_aov()
    assert (aov["inst"] == 0).all()
    return aov["albedo"]


def test_matte_wall_gives_its_colour_the_wall_normal_and_the_analytic_depth():
    s = wall_scene()
    samples, aov, st = s.render_samples_aov()
    want, _ = s.render_samples()
    assert samples.tobytes() == want.tobytes() and st.camera_samples == len(aov) == 16 * 16 * 2
    assert (aov["inst"] == 0).all()
    assert np.array_equal(aov["albedo"], np.tile(np.array([0.2, 0.4, 0.6], f32), (len(aov), 1)))
    assert np.array_equal(aov["n"], np.tile(np.array([0, 0, 1], f32), (len(aov), 1)))
    rays, _ = s.camera_rays()
    d = rays["d"].astype(np.float64)
    assert np.allclose(aov["depth"], 10.0 * np.linalg.norm(d, axis=1) / d[:, 2], rtol=1e-5, atol=0)  # plane z = 0 from z = -10


def _conductor(eta, k):  # fresnel.rs:19-28 at cos 1, float32, left to right
    eta, k, c, one = np.array(eta, f32), np.array(k, f32), f32(1.0), f32(1.0)
    a = (eta * eta + k * k) * c * c
    r_par = (a - eta * c * f32(2.0) + one) / (a + eta * c * f32(2.0) + one)
    b = eta * eta + k * k
    cc = c * c
    r_perp = (b - eta * c * f32(2.0) + cc) / (b + eta * c * f32(2.0) + cc)
    return (r_par + r_perp) * f32(0.5)


def _dielectric(eta):  # fresnel.rs:48-66 at cos 1 from outside (eta_i = 1): sin_t = 0, cos_t = 1
    ei, et, ci = f32(1.0), f32(eta), f32(1.0)
    sin_t = ei / et * np.sqrt(max(f32(0.0), f32(1.0) - ci * ci), dtype=f32)
    ct = np.sqrt(max(f32(0.0), f32(1.0) - sin_t * sin_t), dtype=f32)
    r_par = (et * ci - ei * ct) / (et * ci + ei * ct)
    r_perp = (ei * ci - et * ct) / (ei * ci + et * ct)
    return f32(0.5) * (r_par * r_par + r_perp * r_perp)


@pytest.mark.parametrize("mtype", [F.MAT_METAL, F.MAT_SPECULAR_METAL])
def test_metal_albedo_is_the_conductor_fresnel_at_normal_incidence(mtype):
    eta, k = (0.2, 0.9, 1.1), (3.9, 2.4, 2.2)
    got = _albedo(mtype, c0=eta, c1=k, roughness=0.1)
    want = np.clip(f32(0.0) + f32(1.0) * _conductor(eta, k), 0, 1).astype(f32)
    assert np.array_equal(got, np.tile(want, (len(got), 1)))


def test_plastic_albedo_is_diffuse_plus_gloss_times_the_dielectric_fresnel_of_1_5():
    d, g = np.array((0.3, 0.5, 0.1), f32), np.array((0.9, 0.8, 0.7), f32)
    got = _albedo(F.MAT_PLASTIC, c0=d, c1=g, roughness=0.2)
    want = np.clip((f32(0.0) + d) + g * _dielectric(1.5), 0, 1).astype(f32)
    assert np.array_equal(got, np.tile(want, (len(got), 1)))
    got = _albedo(F.MAT_PLASTIC, c0=(0, 0, 0), c1=g, roughness=0.2)  # a black diffuse colour: no Lambertian lobe
    assert np.array_equal(got, np.tile(np.clip(f32(0.0) + g * _dielectric(1.5), 0, 1).astype(f32), (len(got), 1)))


@pytest.mark.parametrize("mtype", [F.MAT_GLASS, F.MAT_ROUGH_GLASS])
@pytest.mark.parametrize("reflect,transmit,eta", [((1, 1, 1), (1, 1, 1), 1.5), ((0.9, 0.6, 0.3), (0.2, 0.7, 1.0), 1.33), ((0, 0, 0), (0.5, 0.5, 0.9), 2.4)])
def test_glass_albedo_is_reflect_times_f_plus_transmit_times_one_minus_f(mtype, reflect, transmit, eta):
    r, t = np.array(reflect, f32), np.array(transmit, f32)
    got = _albedo(mtype, c0=r, c1=t, eta=eta, roughness=0.3)
    fr = _dielectric(eta)
    acc = np.zeros(3, f32)
    if r.any():
        acc = acc + r * fr
    if t.any():
        acc = acc + t * (f32(1.0) - fr)
    assert np.array_equal(got, np.tile(np.clip(acc, 0, 1).astype(f32), (len(got), 1)))


def test_textured_matte_gives_the_bilinear_texture_sample_at_the_hit():
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (2, 3, 4), dtype=np.uint8)  # 3 wide, 2 high
    s = wall_scene(image=img)
    _, aov, _ = s.render_samples_aov()
    rays, _ = s.camera_rays()
    q = np.zeros(len(rays), F.QUERY_RAY_DTYPE)
    q["o"], q["d"], q["min_t"], q["max_t"] = rays["o"], rays["d"], rays["min_t"], rays["max_t"]
    rec, _ = s.intersect_records(q)
    assert (rec["inst"] == 0).all()
    h, w = img.shape[:2]

    def texel(x, y):  # Image::get_color: clamped to the last texel, c / 255
        return img[np.minimum(y, h - 1), np.minimum(x, w - 1), :3].astype(f32) / f32(255.0)

    x, y = rec["u"] * f32(w), rec["v"] * f32(h)
    x0, y0 = x.astype(np.uint32), y.astype(np.uint32)
    sx, sy = (x - x0.astype(f32))[:, None], (y - y0.astype(f32))[:, None]
    one = f32(1.0)
    want = (texel(x0, y0) * (one - sx) * (one - sy) + texel(x0 + 1, y0) * sx * (one - sy) + texel(x0, y0 + 1) * (one - sx) * sy
            + texel(x0 + 1, y0 + 1) * sx * sy)
    assert np.array_equal(aov["albedo"], np.clip(f32(0.0) + want, 0, 1).astype(f32))


def test_misses_give_the_miss_record():
    s = wall_scene(facing=False)
    _, aov, _ = s.render_samples_aov()
    assert (aov["inst"] == F.MISS).all() and np.isposinf(aov["depth"]).all()
    assert not aov["albedo"].any() and not aov["n"].any()
