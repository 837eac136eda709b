"""The ray queries without a GPU: the trb_query_ray / trb_intersection layout (plain C, ctypes, numpy and the Rust declarations in
INTEGRATION.md), the exports and the argument checks that need no device, and the oracle's orc_intersect_records / orc_occluded
against orc_intersect and against closed forms."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, scenebuild as SB
from oracle import pyoracle as O
from oracle_queries import pyqueries as Q
from test_textures import checker, textured_floor

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_intersect_records", "trb_intersect_records_device", "trb_occluded", "trb_occluded_device"]
STRUCTS = {"trb_query_ray": (F.QueryRay, F.QUERY_RAY_DTYPE, "TrbQueryRay"), "trb_intersection": (F.Intersection, F.INTERSECTION_DTYPE, "TrbIntersection")}


# ---- ray sets shared with tests/test_queries_gpu.py ---------------------------------------------------------------------------
def query_rays(rays, time):
    """QUERY_RAY_DTYPE records from RAY_DTYPE rays and a time (scalar or per ray)."""
    q = np.zeros(len(rays), F.QUERY_RAY_DTYPE)
    for k in ("o", "d", "min_t", "max_t"):
        q[k] = rays[k]
    q["time"] = time
    return q


def random_rays(n, seed, lo, hi, t0, t1):
    """Incoherent rays: origins uniform in the box [lo, hi], directions uniform on the sphere, times uniform in [t0, t1]."""
    rng = np.random.default_rng(seed)
    q = np.zeros(n, F.QUERY_RAY_DTYPE)
    q["o"] = rng.uniform(lo, hi, size=(n, 3))
    d = rng.normal(size=(n, 3))
    q["d"] = d / np.linalg.norm(d, axis=1, keepdims=True)
    q["max_t"] = np.inf
    q["time"] = rng.uniform(t0, t1, size=n)
    return q


def edge_rays(time):
    """test_edge_cases' awkward rays: zero, NaN, denormal and huge directions, a max_t shorter than any hit."""
    q = np.zeros(6, F.QUERY_RAY_DTYPE)
    q["o"] = [0, 12, -60]
    q["d"] = [[0, 0, 1], [0, 0, -1], [0, 0, 0], [np.nan, 0, 1], [0, 1e-30, 1], [1e30, 0, 1]]
    q["max_t"] = [np.inf, np.inf, np.inf, np.inf, np.inf, 1e-3]
    q["time"] = time
    return q


def at_hit_rays(q, rec):
    """For every ray that hits: max_t exactly at the hit, min_t exactly at the hit, and max_t one ulp short of it."""
    h = q[rec["inst"] != F.MISS].copy()
    t = rec["t"][rec["inst"] != F.MISS]
    a, b, c = h.copy(), h.copy(), h.copy()
    a["max_t"] = t
    b["min_t"] = t
    c["max_t"] = np.nextafter(t, np.float32(0))
    return np.concatenate([a, b, c])


# ---- layout, exports, argument checks ---------------------------------------------------------------------------------------
def _c_layout(tmp_path):
    exe = str(tmp_path / "query_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "query_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_plain_c_layout_matches_ctypes_numpy_and_the_rust_declarations(tmp_path):
    lines = _c_layout(tmp_path)
    sizes = {l.split()[0]: int(l.split()[2]) for l in lines if " sizeof " in l}
    offsets = {}
    for l in lines:
        a, *b = l.split()
        if "." in a and len(b) == 1:
            offsets.setdefault(a.split(".")[0], []).append((a.split(".")[1], int(b[0])))
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    width = {"u32": 4, "f32": 4}
    for cname, (ct, dt, rust) in STRUCTS.items():
        assert C.sizeof(ct) == sizes[cname] == dt.itemsize, cname
        assert [(f, getattr(ct, f).offset) for f, _ in ct._fields_] == offsets[cname], cname
        assert [(f, dt.fields[f][1]) for f in dt.names] == offsets[cname], cname
        m = re.search(r"pub struct %s \{(.*?)\}" % rust, doc, re.S)
        assert m, rust
        fields = re.findall(r"(\w+)\s*:\s*(\[(\w+);\s*(\d+)\]|\w+)", m.group(1))
        off = 0
        for (name, whole, elem, count), (cf, co) in zip(fields, offsets[cname]):
            assert name == cf and off == co, (rust, name)
            off += width[elem] * int(count) if elem else width[whole]
        assert len(fields) == len(offsets[cname]) and off == sizes[cname], rust


def test_plain_c_caller_gets_invalid_arg_for_null_arguments(tmp_path):
    status = {l.split()[1]: int(l.split()[2]) for l in _c_layout(tmp_path) if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {n: F.TRB_INVALID_ARG for n in NEW}


def test_new_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    rust_to_ctypes = {"*mut c_void": (C.c_void_p,), "usize": (C.c_size_t,), "u32": (C.c_uint32,), "*const TrbQueryRay": (C.c_void_p,),
                      "*mut TrbIntersection": (C.c_void_p,), "*mut u8": (C.c_void_p,), "*mut TrbStats": (C.POINTER(F.Stats), C.c_void_p)}
    for name in NEW:
        assert hasattr(trb, name) and name in F.TRB_SYMBOLS, name
        m = re.search(r"fn %s\((.*?)\)\s*->\s*c_int;" % name, doc, re.S)
        assert m, name
        rust = [p.split(":", 1)[1].strip() for p in m.group(1).split(",") if p.strip()]
        ct = getattr(trb, name).argtypes
        assert len(ct) == len(rust), name
        for i, (r, c) in enumerate(zip(rust, ct)):
            assert c in rust_to_ctypes[r], (name, i, r, c)
        assert "`%s(" % name in doc, "no table row for " + name


def test_argument_checks_need_no_device(trb):
    ray = np.zeros(1, F.QUERY_RAY_DTYPE)
    rec = np.zeros(1, F.INTERSECTION_DTYPE)
    occ = np.zeros(1, np.uint8)
    fake = C.c_void_p(1)  # never dereferenced: every call below fails its argument checks first
    calls = [
        lambda: trb.trb_intersect_records(None, 1, F.ptr(ray), F.ptr(rec), 0, None),
        lambda: trb.trb_intersect_records(fake, 1, None, F.ptr(rec), 0, None),
        lambda: trb.trb_intersect_records(fake, 1, F.ptr(ray), None, 0, None),
        lambda: trb.trb_intersect_records(fake, 1, F.ptr(ray), F.ptr(rec), F.RENDER_REFERENCE_SHADOW, None),  # occlusion only
        lambda: trb.trb_intersect_records_device(fake, 1, None, F.ptr(rec), 0, None, None),
        lambda: trb.trb_intersect_records_device(fake, 1, F.ptr(ray), F.ptr(rec), F.RENDER_MEGAKERNEL, None, None),
        lambda: trb.trb_occluded(None, 1, F.ptr(ray), F.ptr(occ), 0, None),
        lambda: trb.trb_occluded(fake, 1, F.ptr(ray), None, 0, None),
        lambda: trb.trb_occluded(fake, 1, F.ptr(ray), F.ptr(occ), F.RENDER_TIME_TRACE, None),
        lambda: trb.trb_occluded_device(fake, 1, None, F.ptr(occ), 0, None, None),
        lambda: trb.trb_occluded_device(fake, 1, F.ptr(ray.view(np.uint8)[4:]), F.ptr(occ), 0, None, None),  # not 16-byte aligned
    ]
    for k, call in enumerate(calls):
        assert call() == F.TRB_INVALID_ARG, k


# ---- the oracle ------------------------------------------------------------------------------------------------------------
def _scene(desc, frame=0, start=0.0, end=0.0):
    o = Q.QueryOracleScene(desc)
    o.update_frame(frame, start, end)
    return o


@pytest.mark.parametrize("name", ["zoo", "smallpt", "keyframed"])
def test_records_at_shutter_open_equal_orc_intersect(name):
    if name == "keyframed":
        o = _scene(SB.scene_animated(16, 16, 2).finish(), 1, 0.25, 0.5)
        t0 = 0.25
    else:
        o = _scene((SB.scene_materials_zoo(16, 16, 2, SB.synthetic_merl_table()) if name == "zoo" else SB.scene_smallpt_like(16, 16, 2)).finish())
        t0 = 0.0
    rays, _ = o.camera_rays(seed=3)
    q = np.concatenate([query_rays(rays, t0), random_rays(4096, 5, (-14, 1, -10), (14, 23, 18), t0, t0), edge_rays(t0)])
    rec, st = o.intersect_records(q)
    ref = np.zeros(len(q), F.RAY_DTYPE)
    for k in ("o", "d", "min_t", "max_t"):
        ref[k] = q[k]
    hits, hst = o.intersect(ref)
    assert rec["t"].tobytes() == hits["t"].tobytes()
    assert (rec["inst"] == hits["inst"]).all() and (rec["prim"] == hits["prim"]).all()
    assert (st.node_tests, st.tri_tests, st.inst_tests) == (hst.node_tests, hst.tri_tests, hst.inst_tests)
    assert st.rays_primary == len(q) and st.rays_shadow == 0
    hit = rec["inst"] != F.MISS
    assert 100 < hit.sum() < len(q)
    assert (rec["time"][hit] == np.float32(t0)).all() and not rec[~hit]["p"].any() and (rec["material"][~hit] == 0).all()
    # a record's material is its instance's
    mats = np.array([o._desc.instances[i].material for i in range(o._desc.n_instances)])
    assert (rec["material"][hit] == mats[rec["inst"][hit]]).all()


def _unit_sphere():
    b = SB.SceneBuilder(8, 8, 1)
    m = b.add_material(F.MAT_MATTE, (0.5, 0.5, 0.5), roughness=0.0)
    b.receiver(F.SHAPE_SPHERE, m, [SB.trs()], p0=1.0)
    b.point_light([SB.trs(t=(0, 10, 0))], (1, 1, 1, 1))
    b.add_camera([SB.trs(t=(0, 0, -10))])
    return b.finish()


def test_unit_sphere_hit_along_an_axis_is_that_axis():
    o = _scene(_unit_sphere())
    axes = np.concatenate([np.eye(3), -np.eye(3)]).astype(np.float32)
    q = np.zeros(6, F.QUERY_RAY_DTYPE)
    q["o"] = axes * 5.0
    q["d"] = 0.0 - axes  # +0.0 off-axis components: with -0.0, 1/d = -inf and the reference's box test (sign by d < 0) misses
    q["max_t"] = np.inf
    q["time"] = 0.75
    rec, _ = o.intersect_records(q)
    assert (rec["inst"] == 0).all() and (rec["t"] == 4.0).all() and (rec["time"] == np.float32(0.75)).all()
    for k in ("p", "n", "ng"):
        assert np.array_equal(rec[k], axes), k
    # with_normal (sphere.rs:80): n == ng; dp_du is tangent
    assert np.allclose(np.einsum("ij,ij->i", rec["dp_du"], rec["n"]), 0.0, atol=1e-5)


def test_rectangle_normal_is_the_cross_product_and_uv_is_the_floor_parameterisation():
    img = checker(5, 7, 1)
    o = _scene(textured_floor(img).finish())
    rays, _ = o.camera_rays(seed=4)
    rec, _ = o.intersect_records(query_rays(rays, 0.0))
    assert (rec["inst"] == 0).all()
    p = rays["o"].astype(np.float64) + rays["d"].astype(np.float64) * rec["t"][:, None].astype(np.float64)
    assert np.allclose(rec["p"], p, atol=1e-4)
    # DifferentialGeometry::new (differential_geometry.rs:35): n = normalize(cross(dp_du, dp_dv)); the floor faces +y
    c = np.cross(rec["dp_du"].astype(np.float64), rec["dp_dv"].astype(np.float64))
    assert np.allclose(rec["n"], c / np.linalg.norm(c, axis=1, keepdims=True), atol=1e-6)
    assert np.allclose(rec["n"], [0, 1, 0], atol=1e-6) and np.allclose(rec["ng"], [0, 1, 0], atol=1e-6)
    # rectangle.rs:54-55 in object space; rotate_x(-90) maps object (x, y, 0) to world (x, 0, -y) (test_textures)
    assert np.allclose(rec["u"], (p[:, 0] + 4.0) / 8.0, atol=1e-5)
    assert np.allclose(rec["v"], (-p[:, 2] + 3.0) / 6.0, atol=1e-5)


@pytest.mark.parametrize("name", ["zoo", "keyframed"])
def test_orc_occluded_is_record_is_a_hit(name):
    if name == "keyframed":
        o = _scene(SB.scene_animated(16, 16, 2).finish(), 1, 0.25, 0.5)
        t0, t1 = 0.25, 0.375
    else:
        o = _scene(SB.scene_materials_zoo(16, 16, 2, SB.synthetic_merl_table()).finish())
        t0, t1 = 0.0, 0.0
    q = random_rays(4096, 9, (-14, 1, -10), (14, 23, 18), t0, t1)
    q["max_t"] = np.random.default_rng(2).uniform(0.5, 30.0, size=len(q))
    q = np.concatenate([q, edge_rays(t0)])
    rec, st = o.intersect_records(q)
    occ, ost = o.occluded(q)
    assert (occ == (rec["inst"] != F.MISS)).all() and 0 < occ.sum() < len(q)
    # the closest-hit walk of light/mod.rs:30-37 performs exactly Scene::intersect's tests
    assert (ost.node_tests, ost.tri_tests, ost.inst_tests) == (st.node_tests, st.tri_tests, st.inst_tests)
    assert ost.rays_shadow == len(q) and ost.rays_primary == 0
