"""trb_illumination without a GPU: the trb_illum_ray layout (plain C, ctypes, numpy and the Rust declaration in INTEGRATION.md),
the exports and the argument checks that need no device, and the oracle's orc_illumination against orc_render_samples and a
closed form."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, scenebuild as SB
from oracle_queries import pyqueries as Q

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_illumination", "trb_illumination_device"]


# ---- ray sets shared with tests/test_illumination_gpu.py ----------------------------------------------------------------------
def camera_samples(o, **kw):
    """The camera rays of a render's selection as ILLUM_RAY_DTYPE rays keyed like the render's samples (key = pixel, sample = si).
    Every ray's time is the shutter-open 0: the scenes these are used with render at a [0, 0] shutter."""
    rays, _ = o.camera_rays(**kw)
    blocks = o.block_list(kw.get("block_start", 0), kw.get("block_count", 0)).astype(np.int64)
    cnt = len(rays) // (64 * len(blocks))
    i = np.arange(len(rays))
    item, pix = i // (64 * cnt), (i // cnt) % 64
    q = np.zeros(len(rays), F.ILLUM_RAY_DTYPE)
    for k in ("o", "d", "min_t", "max_t"):
        q[k] = rays[k]
    q["key"] = (blocks[item, 1] * 8 + pix // 8) * o.width + blocks[item, 0] * 8 + pix % 8
    q["sample"] = kw.get("sample_first", 0) + i % cnt
    return q


def illum_rays(q, key0=0, sample0=0):
    """ILLUM_RAY_DTYPE rays from QUERY_RAY_DTYPE rays: consecutive keys from key0, and first sample sample0."""
    r = np.zeros(len(q), F.ILLUM_RAY_DTYPE)
    for k in ("o", "d", "min_t", "max_t", "time"):
        r[k] = q[k]
    r["key"] = key0 + np.arange(len(q), dtype=np.uint32)
    r["sample"] = sample0
    return r


# ---- layout, exports, argument checks ---------------------------------------------------------------------------------------
def _c_run(tmp_path):
    exe = str(tmp_path / "illumination_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "illumination_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_plain_c_layout_matches_ctypes_numpy_and_the_rust_declaration(tmp_path):
    lines = _c_run(tmp_path)
    size = [int(l.split()[2]) for l in lines if l.startswith("trb_illum_ray sizeof ")][0]
    offsets = [(l.split()[0].split(".")[1], int(l.split()[1])) for l in lines if l.startswith("trb_illum_ray.")]
    assert C.sizeof(F.IllumRay) == size == F.ILLUM_RAY_DTYPE.itemsize == 48
    assert [(f, getattr(F.IllumRay, f).offset) for f, _ in F.IllumRay._fields_] == offsets
    assert [(f, F.ILLUM_RAY_DTYPE.fields[f][1]) for f in F.ILLUM_RAY_DTYPE.names] == offsets
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    m = re.search(r"pub struct TrbIllumRay \{(.*?)\}", doc, re.S)
    assert m
    fields = re.findall(r"(\w+)\s*:\s*(\[(\w+);\s*(\d+)\]|\w+)", m.group(1))
    off = 0
    for (name, whole, elem, count), (cf, co) in zip(fields, offsets):
        assert name == cf and off == co, name
        off += 4 * int(count) if elem else 4
    assert len(fields) == len(offsets) and off == size


def test_plain_c_caller_gets_invalid_arg_for_null_arguments_and_spp_0(tmp_path):
    status = {l.split()[1]: int(l.split()[2]) for l in _c_run(tmp_path) if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {n: F.TRB_INVALID_ARG for n in NEW + ["trb_illumination_spp0"]}


def test_new_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    rust_to_ctypes = {"*mut c_void": (C.c_void_p,), "usize": (C.c_size_t,), "u32": (C.c_uint32,), "*const TrbIllumRay": (C.c_void_p,),
                      "*mut f32": (C.c_void_p,), "*mut TrbStats": (C.POINTER(F.Stats), C.c_void_p)}
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
    ray = np.zeros(1, F.ILLUM_RAY_DTYPE)
    rgb = np.zeros(4, np.float32)
    fake = C.c_void_p(1)  # never dereferenced: every call below fails its argument checks first
    calls = [
        lambda: trb.trb_illumination(None, 1, F.ptr(ray), 1, 1, F.ptr(rgb), 0, None),
        lambda: trb.trb_illumination(fake, 1, None, 1, 1, F.ptr(rgb), 0, None),
        lambda: trb.trb_illumination(fake, 1, F.ptr(ray), 1, 1, None, 0, None),
        lambda: trb.trb_illumination(fake, 1, F.ptr(ray), 0, 1, F.ptr(rgb), 0, None),        # spp == 0
        lambda: trb.trb_illumination(fake, 1, F.ptr(ray), 65537, 1, F.ptr(rgb), 0, None),    # spp > 65536
        lambda: trb.trb_illumination(fake, 1, F.ptr(ray), 1, 1, F.ptr(rgb), F.RENDER_MEGAKERNEL, None),
        lambda: trb.trb_illumination(fake, 1, F.ptr(ray), 1, 1, F.ptr(rgb), F.RENDER_TIME_TRACE, None),
        lambda: trb.trb_illumination(fake, 1, F.ptr(ray), 1, 1, F.ptr(rgb), 64, None),
        lambda: trb.trb_illumination_device(fake, 1, None, 1, 1, F.ptr(rgb), 0, None, None),
        lambda: trb.trb_illumination_device(fake, 1, F.ptr(ray), 1, 1, None, 0, None, None),
        lambda: trb.trb_illumination_device(fake, 1, F.ptr(ray), 0, 1, F.ptr(rgb), 0, None, None),
        lambda: trb.trb_illumination_device(fake, 1, F.ptr(ray.view(np.uint8)[4:]), 1, 1, F.ptr(rgb), 0, None, None),  # rays not 16-byte aligned
        lambda: trb.trb_illumination_device(fake, 1, F.ptr(ray), 1, 1, F.ptr(rgb.view(np.uint8)[2:]), 0, None, None),  # rgb not 4-byte aligned
        lambda: trb.trb_illumination_device(fake, 1, F.ptr(ray), 1, 1, F.ptr(rgb), F.RENDER_MEGAKERNEL, None, None),
    ]
    for k, call in enumerate(calls):
        assert call() == F.TRB_INVALID_ARG, k


# ---- the oracle ------------------------------------------------------------------------------------------------------------
def _scene(desc, frame=0, start=0.0, end=0.0):
    o = Q.QueryOracleScene(desc)
    o.update_frame(frame, start, end)
    return o


@pytest.mark.parametrize("name", ["zoo", "smallpt"])
def test_clamped_camera_rays_equal_orc_render_samples(name):
    """the oracle-side twin of the GPU's 'same as the render' check: key = pixel, sample = si, spp 1, clamp"""
    desc = (SB.scene_materials_zoo(16, 16, 4, SB.synthetic_merl_table()) if name == "zoo" else SB.scene_smallpt_like(16, 16, 4)).finish()
    o = _scene(desc)
    q = camera_samples(o, seed=7)
    samples, sst = o.render_samples(seed=7)
    st = F.Stats()
    rgb = o.illumination(q, spp=1, seed=7, clamp=True, stats=st)
    want = np.stack([samples["r"], samples["g"], samples["b"]], axis=1)
    assert rgb.tobytes() == want.tobytes()
    for k in ("camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation", "node_tests", "tri_tests", "inst_tests"):
        assert getattr(st, k) == getattr(sst, k), k
    assert (rgb > 0).any()
    # unclamped radiance can exceed 1; the clamped mean cannot
    assert rgb.max() <= 1.0 and o.illumination(q, spp=1, seed=7).max() >= rgb.max()


def _unit_sphere(integrator):
    b = SB.SceneBuilder(8, 8, 1)
    m = b.add_material(F.MAT_MATTE, (0.5, 0.5, 0.5), roughness=0.0)
    b.receiver(F.SHAPE_SPHERE, m, [SB.trs()], p0=1.0)
    b.point_light([SB.trs(t=(0, 10, 0))], (1, 1, 1, 1))
    b.add_camera([SB.trs(t=(0, 0, -10))])
    b.integrator = (integrator, 0, 0)
    return b.finish()


def test_normals_debug_on_a_sphere_hit_along_an_axis_is_n_plus_one_over_two():
    o = _scene(_unit_sphere(F.INTEGRATOR_NORMALS_DEBUG))
    axes = np.concatenate([np.eye(3), -np.eye(3)]).astype(np.float32)
    q = np.zeros(6, F.ILLUM_RAY_DTYPE)
    q["o"] = axes * 5.0
    q["d"] = 0.0 - axes  # +0.0 off-axis components (see test_queries_cpu.test_unit_sphere_hit_along_an_axis_is_that_axis)
    q["max_t"] = np.inf
    rgb = o.illumination(q, spp=3)
    assert np.array_equal(rgb, (axes + 1.0) / 2.0)
    q["d"] = -q["d"]  # pointing away: a miss is black
    assert not o.illumination(q).any()
