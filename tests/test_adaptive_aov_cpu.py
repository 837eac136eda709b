"""AOVs of Adaptive renders without a GPU: the new entry points' exports and plain-C statuses, the Adaptive AOV oracle
(oracle_adaptive_aov) against orc_render_samples_adaptive and against known answers on a matte wall, and trb_tray --adaptive's
refusals, which come before any scene is created."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_adaptive.pyadaptive import AdaptiveOracleScene
from oracle_adaptive_aov.pyadaptiveaov import AdaptiveAovOracleScene

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_render_adaptive_aov", "trb_render_adaptive_aov_device", "trb_render_samples_adaptive_aov"]
KEYS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation", "node_tests", "tri_tests", "inst_tests"]
f32 = np.float32


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
                assert c is {"u32": C.c_uint32, "usize": C.c_size_t}[r], (name, i, r, c)
        assert "`%s(" % name in doc, "no table row for " + name
        assert name + "(" in open(os.path.join(REPO, "include", "trb.h")).read(), name


def test_plain_c_caller_gets_the_argument_statuses(tmp_path):
    exe = str(tmp_path / "adaptive_aov_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "adaptive_aov_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    status = {l.split()[1]: int(l.split()[2]) for l in out if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {k: F.TRB_INVALID_ARG for k in (
        "trb_render_adaptive_aov:null_scene", "trb_render_adaptive_aov:null_adaptive", "trb_render_adaptive_aov:null_aov",
        "trb_render_adaptive_aov_device:null_scene", "trb_render_samples_adaptive_aov:null_scene", "trb_render_samples_adaptive_aov:null_buffers")}


def test_render_adaptive_aov_rejects_wrong_shapes_before_the_library():
    s = api.Scene.__new__(api.Scene)  # never opened: the checks run before the library is called
    s.width, s.height = 8, 8
    for kw in (dict(film=np.zeros((8, 8, 3), np.float32)), dict(albedo=np.zeros((8, 8, 4), np.float64)),
               dict(nearest=np.zeros((8, 8), np.uint32))):
        with pytest.raises(ValueError):
            s.render_adaptive_aov(2, 8, **kw)


# ---- the oracle --------------------------------------------------------------------------------------------------------------
def _counters(st):
    return [getattr(st, k) for k in KEYS]


def _taken(spp_of_slot_pixel, mpp):
    """(n,) bool: which records of the (block, pixel, slot) layout a pixel took, from its per-record sample count"""
    return np.tile(np.arange(mpp), len(spp_of_slot_pixel)) < np.repeat(spp_of_slot_pixel, mpp)


def _pixel_counts(o, spp, block_start=0, block_count=0, **_):
    """pixel_spp in the (block, pixel) order of the parity layout"""
    xy = o.block_list(block_start, block_count).astype(np.int64)
    k = np.arange(64)
    return spp[xy[:, 1:2] * 8 + k[None, :] // 8, xy[:, 0:1] * 8 + k[None, :] % 8].reshape(-1)


def test_oracle_returns_the_adaptive_oracles_samples_counts_and_stats_and_zero_untaken_slots():
    desc = SB.scene_materials_zoo(32, 32, 1, SB.synthetic_merl_table()).finish()
    o, a = AdaptiveOracleScene(desc), AdaptiveAovOracleScene(desc)
    o.update_frame(0, 0.0, 0.0); a.update_frame(0, 0.0, 0.0)
    for mn, mx, kw in ((2, 16, dict(seed=3)), (4, 32, dict(seed=7, block_start=3, block_count=9))):
        want, wspp, wst = o.render_samples_adaptive(mn, mx, **kw)
        got, aov, spp, st = a.render_samples_adaptive_aov(mn, mx, **kw)
        assert got.tobytes() == want.tobytes() and spp.tobytes() == wspp.tobytes() and _counters(st) == _counters(wst)
        assert len(aov) == len(got)
        mpp = a.adaptive_schedule(mn, mx)[3]
        taken = _taken(_pixel_counts(a, spp, **kw), mpp)
        assert taken.sum() == st.camera_samples and (spp > pow2(mn)).any(), "the zoo should make some pixels refine"
        assert not aov[~taken].view(np.uint8).any(), "slots a pixel did not take are zero"
        hit = aov["inst"][taken] != F.MISS
        assert hit.any() and (aov["depth"][taken][~hit] == np.inf).all()
        assert np.allclose(np.linalg.norm(aov["n"][taken][hit], axis=1), 1.0, atol=1e-5)


def pow2(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def wall_scene(c0=(0.2, 0.4, 0.6)):
    """a 16x16 camera at z = -10 looking down +z at a 1000 x 1000 matte rectangle in the plane z = 0 (normal +z)"""
    b = SB.SceneBuilder(16, 16, 2)
    m = b.add_material(F.MAT_MATTE, c0=c0)
    b.receiver(F.SHAPE_RECT, m, [SB.trs()], p0=1000.0, p1=1000.0)
    b.point_light([SB.trs(t=(0, 0, -5))], (1, 1, 1, 10))
    b.add_camera([SB.trs(t=(0, 0, -10), q=(0, 0, 0, 1))], fov=30.0)
    s = AdaptiveAovOracleScene(b.finish())
    s.update_frame(0, 0.0, 0.0)
    return s


def _depth_at(s, x, y):
    """the wall's distance along the camera ray through film position (x, y): the camera's square 30-degree view, so the ray through
    (x, y) is (u t, v t, 1) with u, v in [-1, 1] over the film and t = tan(15 deg); checked against the oracle's own LD camera rays"""
    t = np.tan(np.radians(15.0))
    u, v = (2.0 * np.asarray(x, np.float64) / s.width - 1.0) * t, (2.0 * np.asarray(y, np.float64) / s.height - 1.0) * t
    return 10.0 * np.sqrt(1.0 + u * u + v * v)


def test_matte_wall_slots_give_its_colour_normal_instance_and_the_analytic_depth():
    s = wall_scene()
    rays, xy = s.camera_rays()  # the analytic depth's camera model, checked on LowDiscrepancy's rays
    d = rays["d"].astype(np.float64)
    assert np.allclose(_depth_at(s, xy[:, 0], xy[:, 1]), 10.0 * np.linalg.norm(d, axis=1) / d[:, 2], rtol=1e-6, atol=0)
    for mn, mx in ((1, 8), (4, 64)):
        samples, aov, spp, st = s.render_samples_adaptive_aov(mn, mx, seed=5)
        taken = _taken(_pixel_counts(s, spp), s.adaptive_schedule(mn, mx)[3])
        rec, smp = aov[taken], samples[taken]
        assert len(rec) == st.camera_samples and (spp >= pow2(mn)).all()
        assert (rec["inst"] == 0).all()
        assert np.array_equal(rec["albedo"], np.tile(np.array([0.2, 0.4, 0.6], f32), (len(rec), 1)))
        assert np.array_equal(rec["n"], np.tile(np.array([0, 0, 1], f32), (len(rec), 1)))
        assert np.allclose(rec["depth"], _depth_at(s, smp["x"], smp["y"]), rtol=1e-5, atol=0)


# ---- trb_tray --adaptive ------------------------------------------------------------------------------------------------------
def _refused(args, needle):
    m = H.Proc([H.TRAY] + args)
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and needle in err, (args, err)
    return err


def test_tray_adaptive_refusals_come_before_the_scene(tmp_path):
    H.build_programs()
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    for args, needle in ((["--adaptive", "2", "16", "--spp", "4"], "--adaptive excludes --spp"),
                         (["--adaptive", "2", "16", "--denoise"], "--adaptive excludes --denoise"),
                         (["--adaptive", "2", "16", "--denoise-temporal"], "--adaptive excludes --denoise"),
                         (["--adaptive", "2", "16", "--denoise-temporal", "--temporal-gradients"], "--adaptive excludes --denoise"),
                         (["--adaptive", "16", "2"], "--adaptive 16 2"),
                         (["--master", "127.0.0.1:1", "--adaptive", "2", "16"], "--adaptive is not available with --master")):
        err = _refused([missing] + args, needle)
        assert "no_such_scene" not in err, err
    _refused(["--worker", "--adaptive", "2", "16"], "--adaptive is not available with --worker")
    m = H.Proc([H.TRAY, missing, "--adaptive", "2"])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 2 and "--adaptive needs two non-negative integers" in err


def test_tray_adaptive_refuses_a_non_path_integrator_before_creating_the_scene(tmp_path):
    H.build_programs()
    scene = json.load(open(H.CORNELL))
    scene["integrator"] = {"type": "whitted", "min_depth": 4}
    scene["objects"] = [o for o in scene["objects"] if o.get("geometry", {}).get("type") != "mesh"]
    path = tmp_path / "whitted.json"
    path.write_text(json.dumps(scene))
    # exits 1 with the refusal, on a machine with or without a GPU (creating the scene without one would exit 3)
    _refused([str(path), "--adaptive", "2", "16", "-o", str(tmp_path / "frames")], "--adaptive needs the path integrator")
    _refused([str(path), "--adaptive", "2", "16", "--denoise-moments", "-o", str(tmp_path / "frames")], "needs the path integrator")
