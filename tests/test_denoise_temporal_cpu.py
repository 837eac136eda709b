"""The temporal denoiser without a GPU: the struct layouts against ctypes and the Rust declarations in INTEGRATION.md, the exports, a
plain-C caller's statuses, the parameter refusals, trb_tray --denoise-temporal's argument refusals, and the oracle (oracle_temporal)
against a float64 numpy restatement of include/trb.h "Temporal denoising" steps 1-4 and 6 over synthetic frames, and against known
answers."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F
from oracle_denoise import pydenoise as D
from oracle_temporal import pytemporal as T
from test_denoise_cpu import EPS_A, _lum, synthetic

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_denoise_history_create", "trb_denoise_history_destroy", "trb_denoise_history_reset", "trb_denoise_temporal",
       "trb_denoise_temporal_device"]


def _run_abi(tmp_path):
    exe = str(tmp_path / "denoise_temporal_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"),
                    os.path.join(REPO, "tests", "c", "denoise_temporal_abi.c"), "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_structs_match_the_header_ctypes_and_the_rust_declarations(tmp_path):
    out = _run_abi(tmp_path)
    sizes = {l.split()[0]: int(l.split()[2]) for l in out if " sizeof " in l}
    offs = {l.split()[0]: int(l.split()[1]) for l in out if l.split()[0].count(".") == 1 and not l.startswith("status")}
    assert sizes == {"trb_denoise_temporal_params": 32, "trb_denoise_temporal_output": 24}
    assert C.sizeof(F.DenoiseTemporalParams) == 32 and C.sizeof(F.DenoiseTemporalOutput) == 24
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for cls, cname, rust in ((F.DenoiseTemporalParams, "trb_denoise_temporal_params", "TrbDenoiseTemporalParams"),
                             (F.DenoiseTemporalOutput, "trb_denoise_temporal_output", "TrbDenoiseTemporalOutput")):
        for name, _ in cls._fields_:
            assert getattr(cls, name).offset == offs[cname + "." + name], name
        m = re.search(r"pub struct %s \{(.*?)\}" % rust, doc, re.S)
        assert m, rust
        assert re.findall(r"(\w+)\s*:", m.group(1)) == [n for n, _ in cls._fields_], rust


def test_new_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for name in NEW:
        assert hasattr(trb, name) and name in F.TRB_SYMBOLS, name
        m = re.search(r"fn %s\((.*?)\)\s*->\s*c_int;" % name, doc, re.S)
        assert m, name
        rust = [p.split(":", 1)[1].strip() for p in m.group(1).split(",") if p.strip()]
        assert len(getattr(trb, name).argtypes) == len(rust), name
        assert "`%s(" % name in doc, "no table row for " + name


def test_plain_c_caller_gets_the_argument_statuses(tmp_path):
    st = {l.split()[1]: int(l.split()[2]) for l in _run_abi(tmp_path) if l.startswith("status ")}
    inv, ok = st.pop("TRB_INVALID_ARG"), st.pop("TRB_OK")
    assert st.pop("trb_denoise_history_destroy:null") == ok
    assert all(v == inv for v in st.values()), st


def _params(**kw):
    from tray_rust_b200.api import _temporal_params
    return _temporal_params(kw)


@pytest.mark.parametrize("bad", [dict(max_history=0), dict(max_history=256), dict(depth_tolerance=0.0), dict(depth_tolerance=-1.0),
                                 dict(depth_tolerance=float("inf")), dict(depth_tolerance=float("nan")), dict(normal_threshold=1.5),
                                 dict(normal_threshold=-1.01), dict(normal_threshold=float("nan")), dict(iterations=11),
                                 dict(normal_power=3), dict(sigma_luminance=0.0)])
def test_every_parameter_refusal_is_checked_before_the_scene(trb, bad):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    d_in = F.DenoiseInput(*([film.ctypes.data] * 4), near.ctypes.data)
    out = F.DenoiseTemporalOutput(film.ctypes.data, None, None)
    prm = _params(**bad)
    for fn in (lambda: trb.trb_denoise_temporal(None, None, C.byref(d_in), C.byref(prm), C.byref(out)),
               lambda: trb.trb_denoise_temporal_device(None, None, C.byref(d_in), C.byref(prm), C.byref(out), None)):
        assert fn() == F.TRB_INVALID_ARG
        assert b"temporal" in trb.trb_last_error() or b"denoise" in trb.trb_last_error()
    with pytest.raises(ValueError):  # the oracle refuses them too
        T.denoise_temporal_frame(_static_frame(4, 4)[0], T.History(), *synthetic(np.random.default_rng(0), 4, 4, False), **bad)


def test_unknown_parameters_are_refused_by_the_binding():
    with pytest.raises(TypeError):
        _params(history=3)


# ---- trb_tray --denoise-temporal --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def programs():
    H.build_programs()


@pytest.mark.parametrize("args,needle", [(["--master", "127.0.0.1:1"], "not available with --master"),
                                         (["--worker"], "not available with --worker"),
                                         (["--spp", "1"], "at least 2 samples"),
                                         (["--denoise"], "exclude each other")])
def test_tray_denoise_temporal_argument_refusals(programs, tmp_path, args, needle):
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    m = H.Proc([H.TRAY] + ([] if args == ["--worker"] else [missing]) + args + ["--denoise-temporal", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and needle in err and "no_such_scene" not in err, err
    assert not (tmp_path / "x.png").exists()


# ---- the oracle against a float64 restatement -------------------------------------------------------------------------------------

W_, H_ = 24, 16
ASPECT = W_ / H_
X0, X1, Y0, Y1 = -ASPECT, ASPECT, -1.0, 1.0


def _px_to_cam(w, h):
    """A raster -> camera matrix with camera_ray's screen window: (x, y) -> (X, Y, 1)"""
    a = np.float32(w) / np.float32(h)
    x0, x1, y0, y1 = (-a, a, -1.0, 1.0) if a > 1 else (-1.0, 1.0, -1.0 / a, 1.0 / a)
    return np.array([[(x1 - x0) / w, 0, 0, x0], [0, -(y1 - y0) / h, 0, y1], [0, 0, 0, 1], [0, 0, 0, 1]], np.float32)


def _rot_y(deg):
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    return np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]])


def _translate(x, y, z):
    m = np.eye(4)
    m[:3, 3] = (x, y, z)
    return m


def _frame(w, h, cam, mats, tan=0.5):
    cam = np.asarray(cam, np.float32)
    mats = np.asarray(mats, np.float32)
    invs = np.linalg.inv(mats.astype(np.float64)).astype(np.float32)
    return T.make_frame(_px_to_cam(w, h), cam, np.linalg.inv(cam.astype(np.float64)).astype(np.float32), tan, invs, mats), (cam, mats, invs)


def _static_frame(w, h):
    return _frame(w, h, np.eye(4), [np.eye(4)] * 3)


def _xf(m, p):
    r = m[:3, :3] @ p + m[:3, 3]
    wv = m[3, :3] @ p + m[3, 3]
    return r / wv if abs(wv - 1.0) < 1.1920929e-7 else r


class NpHistory:
    """include/trb.h "Temporal denoising" steps 1-4 and 6 in float64, pixel by pixel (the a-trous step is the spatial oracle's)"""

    def __init__(self):
        self.prev = None

    def step(self, frame_mats, tan, A, B, aovs, max_history=8, depth_tolerance=0.05, normal_threshold=0.9):
        cam, mats, invs = (m.astype(np.float64) for m in frame_mats)
        h, w = A.shape[:2]
        A64, B64 = A.astype(np.float64), B.astype(np.float64)
        alb, nrm = aovs["albedo_w"].astype(np.float64), aovs["normal_w"].astype(np.float64)
        z_all = (aovs["nearest"] >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
        ids = (aovs["nearest"] & np.uint64(0xffffffff)).astype(np.int64)
        p2c = _px_to_cam(w, h).astype(np.float64)
        out = np.full((h, w, 3), np.nan)
        motion = np.full((h, w, 2), np.nan)
        hl = np.zeros((h, w), np.int64)
        store = {}
        cam_inv = np.linalg.inv(cam)
        with np.errstate(all="ignore"):
            for y in range(h):
                for x in range(w):
                    a, b = A64[y, x], B64[y, x]
                    Wt = a[3] + b[3]
                    if Wt <= 0:
                        continue
                    c = (a[:3] + b[:3]) / Wt
                    albedo = alb[y, x, :3] / alb[y, x, 3]
                    d = np.where(albedo > EPS_A, albedo, EPS_A)
                    e, ea, eb = c / d, a[:3] / a[3] / d, b[:3] / b[3] / d
                    v = (_lum(ea) - _lum(eb)) ** 2 * 0.25
                    m = nrm[y, x, :3] / nrm[y, x, 3]
                    len2 = (m * m).sum()
                    z = z_all[y, x]
                    if not (np.isfinite(c).all() and np.isfinite(albedo).all() and np.isfinite(m).all() and np.isfinite(len2)
                            and np.isfinite(e).all() and np.isfinite(v) and not np.isnan(z) and z != -np.inf):
                        continue
                    n = m / np.sqrt(len2) if len2 != 0 else np.zeros(3)
                    has_n = len2 != 0
                    i = ids[y, x]
                    S, sa, sb, len_prev = 0.0, np.zeros(3), np.zeros(3), 0
                    P = self.prev
                    if P is not None and i < P["n"] and i < len(mats) and np.isfinite(z):
                        pc = _xf(p2c, np.array([x + 0.5, y + 0.5, 0.0]))
                        dd = np.array([tan, tan, 1.0]) * pc
                        dd = dd / np.linalg.norm(dd)
                        o, dr = cam[:3, 3], cam[:3, :3] @ dd
                        q = _xf(P["cam_inv"], _xf(P["mats"][i], _xf(invs[i], o + z * dr)))
                        if q[2] > 0:
                            X, Y = q[0] / (q[2] * P["tan"]), q[1] / (q[2] * P["tan"])
                            a_ = w / h
                            x0, x1, y0, y1 = (-a_, a_, -1.0, 1.0) if a_ > 1 else (-1.0, 1.0, -1.0 / a_, 1.0 / a_)
                            r = np.array([(X - x0) / (x1 - x0) * w, (Y - y1) / (y0 - y1) * h])
                            motion[y, x] = r - (x + 0.5, y + 0.5)
                            ql = np.linalg.norm(q)
                            cc = r - 0.5
                            f = np.floor(cc)
                            fr = cc - f
                            for ox, oy in ((0, 0), (1, 0), (0, 1), (1, 1)):
                                tx, ty = int(f[0]) + ox, int(f[1]) + oy
                                wt = (fr[0] if ox else 1 - fr[0]) * (fr[1] if oy else 1 - fr[1])
                                if not (0 <= tx < w and 0 <= ty < h) or (ty, tx) not in P["store"]:
                                    continue
                                s = P["store"][(ty, tx)]
                                if s["i"] != i or not abs(s["z"] - ql) <= depth_tolerance * ql:
                                    continue
                                t_n = (s["n"] != 0).any()
                                if t_n != has_n or (has_n and not (s["n"] @ n >= normal_threshold)):
                                    continue
                                S += wt
                                sa += wt * s["ha"]
                                sb += wt * s["hb"]
                                if wt > 0:
                                    len_prev = max(len_prev, s["len"])
                    npr = min(len_prev + 1, max_history) if S > 0 else 1
                    if npr > 1:
                        al = 1.0 / npr
                        Ha, Hb = sa / S, sb / S
                        e = al * e + (1 - al) * (Ha + Hb) * 0.5
                        ea, eb = al * ea + (1 - al) * Ha, al * eb + (1 - al) * Hb
                    out[y, x] = e * d
                    hl[y, x] = npr
                    if np.isfinite(z):
                        store[(y, x)] = dict(ha=ea, hb=eb, n=n, z=z, i=i, len=npr)
        self.prev = dict(cam_inv=cam_inv, tan=tan, n=len(mats), mats=mats, store=store)
        return out, motion, hl


def _scene_inputs(rng, h, w, ids, depth=None):
    A, B, aovs = synthetic(rng, h, w, specials=True)
    if depth is not None:
        z = (aovs["nearest"] >> np.uint64(32)).astype(np.uint32).view(np.float32)
        keep = ~np.isfinite(z) | np.isnan(z)
        z = np.where(keep, z, depth).astype(np.float32)
        aovs["nearest"] = z.view(np.uint32).astype(np.uint64) << np.uint64(32)
    aovs["nearest"] = aovs["nearest"] | ids.astype(np.uint64)
    nrm = aovs["normal_w"]  # one surface orientation in every frame, so that the normal test passes where nothing flipped
    keep = np.isfinite(nrm).all(-1) & (nrm[..., :3] != 0).any(-1)
    nrm[keep, :3] = np.array([0.0, 0.0, -1.0], np.float32) * nrm[keep, 3:]
    return A, B, aovs


def _compare(got, want, oracle_motion, np_motion, oracle_hl, np_hl):
    out, mo, hl = got, oracle_motion, oracle_hl
    valid = np.isfinite(want).all(-1)
    scale = np.abs(want[valid]).max()
    np.testing.assert_allclose(out[..., :3][valid], want[valid], rtol=1e-3, atol=1e-3 * scale)
    assert np.array_equal(np.isnan(mo), np.isnan(np_motion))
    m = ~np.isnan(np_motion)
    np.testing.assert_allclose(mo[m], np_motion[m], rtol=1e-3, atol=1e-3)
    assert np.array_equal(hl, np_hl)


def test_oracle_equals_the_float64_restatement_over_moving_frames():
    """Camera and instances move between three frames; taps fall outside the image, on other instances, at other depths and
    normals; instance 3 is past the snapshot's count; instance 2 moves behind the previous camera (q.z <= 0)"""
    rng = np.random.default_rng(11)
    h, w = H_, W_
    ids = np.broadcast_to((np.arange(w)[None, :] // 8) % 3, (h, w)).copy()  # three vertical bands
    ids[rng.random((h, w)) < 0.05] = 3
    mats = [np.eye(4), _translate(0.3, 0.1, 0.0), _translate(0, 0, 0)]
    hist, oh = NpHistory(), T.History()
    tan = 0.5
    cams = [_translate(0, 0, -10.0), _translate(0.4, -0.2, -10.0) @ _rot_y(2.0), _translate(0.9, -0.1, -9.5) @ _rot_y(3.5)]
    insts = [mats, [_translate(0.1, 0, 0), _translate(0.5, 0.1, 0.2), _translate(0, 0, 0)],
             [_translate(0.2, 0.05, 0), _translate(0.6, 0.2, 0.3), _translate(0, 0, 30.0)]]
    depth = (10.0 + rng.uniform(-0.05, 0.05, (h, w))).astype(np.float32)
    rejected = 0
    for k in range(3):
        f, raw = _frame(w, h, cams[k], insts[k], tan)
        A, B, aovs = _scene_inputs(rng, h, w, ids if k < 2 else np.where(rng.random((h, w)) < 0.2, (ids + 1) % 3, ids), depth)
        if k == 2:  # depth and normal rejections
            z = (aovs["nearest"] >> np.uint64(32)).astype(np.uint32).view(np.float32).copy()
            far = rng.random((h, w)) < 0.15
            z[far & np.isfinite(z)] *= 1.5
            aovs["nearest"] = (z.view(np.uint32).astype(np.uint64) << np.uint64(32)) | (aovs["nearest"] & np.uint64(0xffffffff))
            flip = rng.random((h, w)) < 0.15
            aovs["normal_w"][flip, :3] *= -1
        got = T.denoise_temporal_frame(f, oh, A, B, aovs, iterations=0)
        want = hist.step(raw, tan, A, B, aovs)
        _compare(got[0], want[0], got[1], want[1], got[2], want[2])
        if k:
            rejected += int(((want[2] == 1) & ~np.isnan(want[1][..., 0])).sum())
            assert (want[2] > 1).sum() > 0.15 * h * w  # history kept where the specials leave pixels filtered
    assert rejected > 10


def test_with_history_length_1_the_oracle_is_the_spatial_oracle_bit_for_bit():
    rng = np.random.default_rng(3)
    f, _ = _static_frame(W_, H_)
    hist = T.History()
    for k in range(3):
        A, B, aovs = synthetic(rng, H_, W_)
        for params in (dict(max_history=1), dict(max_history=1, iterations=2, normal_power=8)):
            got, motion, hl = T.denoise_temporal_frame(f, hist, A, B, aovs, **params)
            spatial = {k2: v for k2, v in params.items() if k2 != "max_history"}
            assert got.tobytes() == D.denoise(A, B, aovs, **spatial).tobytes()
            assert set(np.unique(hl)) <= {0, 1}
    hist.reset()  # and the first call after a reset, with the default max_history
    A, B, aovs = synthetic(rng, H_, W_)
    assert T.denoise_temporal_frame(f, hist, A, B, aovs)[0].tobytes() == D.denoise(A, B, aovs).tobytes()


def test_identical_static_frames_count_1_2_and_clamp_at_max_history():
    rng = np.random.default_rng(4)
    w, h = W_, H_
    f, _ = _frame(w, h, _translate(0, 0, -10.0), [np.eye(4)] * 2)
    A, B, aovs = synthetic(rng, h, w, specials=False)
    z = np.full((h, w), 10.0, np.float32)
    z[:, :3] = np.inf  # misses never accumulate
    aovs["nearest"] = (z.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(1)
    hist = T.History()
    for k in range(7):
        _, motion, hl = T.denoise_temporal_frame(f, hist, A, B, aovs, max_history=5)
        assert (hl[:, 3:] == min(k + 1, 5)).all(), (k, np.unique(hl[:, 3:]))
        assert (hl[:, :3] == 1).all() and np.isnan(motion[:, :3]).all()
        if k:
            assert np.abs(motion[:, 3:]).max() < 1e-3


def test_a_camera_translation_gives_the_analytic_motion():
    """A fronto-parallel plane at depth 10 seen by a camera moved by t along x: every point moves by -t / (10 tan) screen units, that
    is -t / (10 tan) * w / (X1 - X0) pixels"""
    rng = np.random.default_rng(5)
    w, h, tan, t = W_, H_, 0.5, 0.37
    A, B, aovs = synthetic(rng, h, w, specials=False)
    hist = T.History()
    for k, cam in enumerate((_translate(0, 0, 0), _translate(t, 0, 0))):
        f, _ = _frame(w, h, cam, [np.eye(4)], tan)
        # depth along each pixel's ray to the plane z = 10 of the first camera
        xs, ys = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
        X = (xs / w) * (X1 - X0) + X0
        Y = Y1 - (ys / h) * (Y1 - Y0)
        z = (10.0 * np.sqrt((tan * X) ** 2 + (tan * Y) ** 2 + 1.0)).astype(np.float32)
        aovs["nearest"] = z.view(np.uint32).astype(np.uint64) << np.uint64(32)
        _, motion, hl = T.denoise_temporal_frame(f, hist, A, B, aovs)
    want = t / (10.0 * tan) * w / (X1 - X0)  # the camera moved right, the previous image of a point lies to its right
    assert np.abs(motion[..., 0] - want).max() < 1e-3, (motion[..., 0].min(), motion[..., 0].max(), want)
    assert np.abs(motion[..., 1]).max() < 1e-3
