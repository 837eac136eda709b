"""Motion vectors without a GPU: the exports against INTEGRATION.md's Rust declarations, a plain-C caller's statuses and record size,
decode_motion, and the motion oracle (oracle_motion) on known answers (a static scene, dt = 0 on a keyframed one, a camera sliding
along its x axis in front of a fronto-parallel plane, a surface that ends up behind the camera) and against a float64 numpy
restatement of include/trb.h "Motion vectors" on the keyframed scene with and without an animated fov."""
import math
import os
import re
import subprocess

import numpy as np
import pytest
from scipy.interpolate import BSpline

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle import pyoracle as O
from oracle_motion import pymotion as PM

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_render_aov_motion", "trb_render_aov_motion_device", "trb_render_adaptive_aov_motion", "trb_render_adaptive_aov_motion_device",
       "trb_render_samples_aov_motion"]


def test_new_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for name in NEW:
        assert hasattr(trb, name) and name in F.TRB_SYMBOLS, name
        m = re.search(r"fn %s\((.*?)\)\s*->\s*c_int;" % name, doc, re.S)
        assert m, name
        rust = [p.split(":", 1)[1].strip() for p in m.group(1).split(",") if p.strip()]
        assert len(getattr(trb, name).argtypes) == len(rust), name
        assert "`%s(" % name in doc, "no table row for " + name
    assert F.MOTION_SAMPLE_DTYPE.itemsize == 16


def test_plain_c_caller_gets_the_argument_statuses(tmp_path):
    exe = str(tmp_path / "motion_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "motion_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    assert "size trb_motion_sample 16" in out
    st = {l.split()[1]: int(l.split()[2]) for l in out if l.startswith("status ")}
    inv = st.pop("TRB_INVALID_ARG")
    st.pop("TRB_OK")
    assert len(st) == 5 and all(v == inv for v in st.values()), st


def test_decode_motion_divides_by_the_weight_and_leaves_nan_elsewhere():
    m = np.array([[[2.0, -1.0, 0.5, 1.0], [1.0, 1.0, 0.0, 1.0]], [[0.0, 0.0, -0.25, 0.5], [3.0, 6.0, 3.0, 3.0]]], np.float32)
    d = api.decode_motion(m)
    assert d.shape == (2, 2, 2) and d.dtype == np.float32
    assert np.array_equal(d[0, 0], [4.0, -2.0]) and np.array_equal(d[1, 1], [1.0, 2.0])
    assert np.isnan(d[0, 1]).all() and np.isnan(d[1, 0]).all()


def plane_scene(cam, rect=400.0, w=32, h=24, frames=4, fov=40.0):
    """a matte rectangle in the plane z = 0 facing a camera that looks along +z (shutter 0: every ray at the frame's start)"""
    b = SB.SceneBuilder(w, h, 2, 2, 4)
    b.film.update(frames=frames, start_frame=0, end_frame=frames - 1, scene_time=1.0)
    m = b.add_material(F.MAT_MATTE, (0.7, 0.7, 0.7), roughness=0.0)
    b.receiver(F.SHAPE_RECT, m, [SB.trs()], p0=rect, p1=rect)
    b.point_light([SB.trs(t=(0, 0, -5))], (1, 1, 1, 10))
    b.add_camera(cam, fov=fov, shutter_size=0.0)
    return b


def _hits(o, **kw):
    rays, _ = o.camera_rays(**kw)
    return o.intersect(rays)[0]["inst"] != F.MISS


def test_a_static_scene_gives_zero_motion_valid_at_hits_and_invalid_at_misses():
    o = PM.MotionOracleScene(plane_scene([SB.trs(t=(0, 0, -10))], rect=4.0).finish())
    o.update_frame(1, 0.25, 0.5)
    kw = dict(seed=3, spp=4)
    rec = o.motion_samples(dt=-0.25, **kw)
    hit = _hits(o, **kw)
    assert hit.any() and not hit.all()
    assert np.array_equal(rec["valid"], hit.astype(np.float32))
    assert (rec["dx"] == 0).all() and (rec["dy"] == 0).all() and (rec["reserved"] == 0).all()
    assert not np.signbit(rec["dx"]).any() and not np.signbit(rec["dy"]).any()


@pytest.mark.parametrize("animated_fov", [False, True])
def test_dt_zero_gives_exact_zeros_on_a_keyframed_scene(animated_fov):
    o = PM.MotionOracleScene(SB.scene_animated(32, 32, 4, animated_fov=animated_fov).finish())
    o.update_frame(1, 0.25, 0.5)
    rec = o.motion_samples(dt=0.0, seed=5)
    assert rec["valid"].sum() > 0.5 * len(rec)
    assert (rec["dx"] == 0).all() and (rec["dy"] == 0).all()
    moving = o.motion_samples(seed=5)  # one frame back: the camera and the instances moved
    assert np.abs(moving["dx"]).max() > 0.1


def test_a_camera_sliding_along_x_gives_the_analytic_shift():
    w, h, fov, d, z = 32, 24, 40.0, 2.0, 10.0
    o = PM.MotionOracleScene(plane_scene([SB.Anim([SB.trs(t=(0, 0, -z)), SB.trs(t=(d, 0, -z))], degree=1)], w=w, h=h, fov=fov).finish())
    o.update_frame(1, 0.25, 0.5)  # camera x(t) = d t; t = 0.25, t + dt = 0
    rec = o.motion_samples(dt=-0.25, seed=9, spp=2)
    assert (rec["valid"] == 1).all()
    # the camera moved by dx_cam = x(t + dt) - x(t) = -0.25 d: a fixed point moves by -dx_cam in camera x, and the screen window spans
    # +-1 on the shorter axis over min(w, h) / 2 pixels; raster x grows with camera x
    want = 0.25 * d * (min(w, h) / 2.0) / (z * math.tan(math.radians(fov) / 2.0))
    np.testing.assert_allclose(rec["dx"], want, rtol=1e-4)
    assert (rec["dy"] == 0).all()
    fwd = o.motion_samples(dt=0.25, seed=9, spp=2)  # forward flow: the opposite shift
    np.testing.assert_allclose(fwd["dx"], -want, rtol=1e-4)


def test_a_surface_behind_the_camera_is_invalid():
    # camera z(t) = 10 - 40 t looking along +z at the plane z = 0: at t = 0.5 the plane is 10 ahead, at t = 0 it is 10 behind
    o = PM.MotionOracleScene(plane_scene([SB.Anim([SB.trs(t=(0, 0, 10)), SB.trs(t=(0, 0, -30))], degree=1)]).finish())
    o.update_frame(2, 0.5, 0.75)
    back = o.motion_samples(dt=-0.5, seed=2, spp=2)
    assert (back["valid"] == 0).all() and (back["dx"] == 0).all() and (back["dy"] == 0).all()
    near = o.motion_samples(dt=-0.125, seed=2, spp=2)
    assert (near["valid"] == 1).all()


# ---- float64 restatement ------------------------------------------------------------------------------------------------------------
def _tan(b, cam, tau_fov):
    """tan(fov / 2) in float64 of camera tuple `cam` with its fov spline sampled at tau_fov (clamped to the knot domain)"""
    if not cam[6]:
        return math.tan(math.radians(cam[2]) / 2.0)
    deg, n, cf, kn, kf = cam[5], cam[6], cam[7], cam[8], cam[9]
    ctrl, knots = np.array(b.fov_floats[cf:cf + n], np.float64), np.sort(np.array(b.fov_floats[kf:kf + kn], np.float64))
    t = min(max(tau_fov, knots[deg]), knots[-1 - deg])
    return math.tan(math.radians(float(BSpline(knots, ctrl, deg)(t))) / 2.0)


def restated(make, frame, dt, **kw):
    """steps 1-5 in float64 over the oracle's camera rays and intersection records; the transforms at any time are read from a twin
    scene with one more instance that carries the camera's transform stack"""
    b = make()
    desc = b.finish()
    o = PM.MotionOracleScene(desc)
    o.update_frame(*frame)
    rays, _ = o.camera_rays(**kw)
    t = np.float32(frame[1])  # shutter 0: every ray's time is the frame's start
    q = np.zeros(len(rays), F.QUERY_RAY_DTYPE)
    q["o"], q["d"], q["min_t"], q["max_t"], q["time"] = rays["o"], rays["d"], rays["min_t"], rays["max_t"], t
    rec, _ = o.intersect_records(q)
    twin = make()
    cam = twin.cameras[0]
    twin.instances.append((F.INST_RECEIVER, F.SHAPE_SPHERE, 1.0, 0.0, 0, 0, cam[0], cam[1], 0, 0))
    probe = O.OracleScene(twin.finish())

    def xf(i, tau):
        probe.update_frame(0, float(tau), float(tau))
        m, inv = probe.transform(i)
        return np.asarray(m, np.float64), np.asarray(inv, np.float64)

    t_then = np.float32(t + np.float32(dt))
    mid = np.float32((np.float32(frame[1]) + np.float32(frame[2])) / np.float32(2.0))
    tan0, tan1 = _tan(b, cam, float(mid)), _tan(b, cam, float(np.float32(mid + np.float32(dt))))
    c0, c1 = xf(len(b.instances), t)[1], xf(len(b.instances), t_then)[1]
    w, h = float(desc.film.width), float(desc.film.height)
    a = w / h
    x0, x1, y0, y1 = (-a, a, -1.0, 1.0) if a > 1 else (-1.0, 1.0, -1.0 / a, 1.0 / a)

    def raster(cinv, tan_fov, p):
        qc = p @ cinv.T
        X, Y = qc[:, 0] / (qc[:, 2] * tan_fov), qc[:, 1] / (qc[:, 2] * tan_fov)
        return (X - x0) / (x1 - x0) * w, (Y - y1) / (y0 - y1) * h, qc[:, 2] > 0

    out = np.zeros((len(rec), 3))
    for inst in np.unique(rec["inst"][rec["inst"] != F.MISS]):
        sel = rec["inst"] == inst
        m0, i0 = xf(int(inst), t)
        m1, _ = xf(int(inst), t_then)
        p = np.concatenate([rec["p"][sel].astype(np.float64), np.ones((sel.sum(), 1))], axis=1)
        po = p @ i0.T
        rx0, ry0, v0 = raster(c0, tan0, po @ m0.T)
        rx1, ry1, v1 = raster(c1, tan1, po @ m1.T)
        v = v0 & v1
        out[sel] = np.stack([np.where(v, rx1 - rx0, 0.0), np.where(v, ry1 - ry0, 0.0), v.astype(np.float64)], axis=1)
    return o, out


@pytest.mark.parametrize("animated_fov", [False, True])
def test_the_oracle_equals_a_float64_restatement_on_the_keyframed_scene(animated_fov):
    def make():
        b = SB.scene_animated(32, 32, 4, animated_fov=animated_fov)
        b.cameras[0] = b.cameras[0][:3] + (0.0,) + b.cameras[0][4:]  # shutter 0: the ray times are known
        return b

    for frame in ((1, 0.25, 0.5), (2, 0.5, 0.75)):
        o, want = restated(make, frame, -0.25, seed=11, spp=4)
        got = o.motion_samples(dt=-0.25, seed=11, spp=4)
        assert np.array_equal(got["valid"], want[:, 2].astype(np.float32))
        assert got["valid"].sum() > 0.5 * len(got) and np.abs(want[:, 0]).max() > 0.1
        # float32 arithmetic on raster positions below 64: a few ulps of 64 each, and the difference of two of them
        np.testing.assert_allclose(got["dx"], want[:, 0], rtol=0, atol=2e-3)
        np.testing.assert_allclose(got["dy"], want[:, 1], rtol=0, atol=2e-3)
