"""The variance temporal denoiser without a GPU: the exports against INTEGRATION.md's Rust declarations and table rows, a plain-C
caller's statuses, the parameter and null-argument refusals, the Python argument checks, trb_tray --denoise-variance-temporal's
argument refusals, and the oracle (oracle_variance_temporal) over synthetic films and histories: n' = 1 and max_history 1 are
orc_denoise_variance bit for bit (misses, W <= 0, one effective sample, NaN and +-inf, every border), lambda 1 is too, the blend equals
a float64 numpy restatement of include/trb.h "Variance temporal denoising" as n' climbs to max_history and is shortened by lambda,
and on a static sequence with a given v_f per frame V follows the closed form of its recursion."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F
from oracle_gradient import pygradient as G
from oracle_variance import pyvariance as V
from oracle_variance_temporal import pyvariancetemporal as VT
from test_denoise_cpu import synthetic
from test_denoise_moments_cpu import H_, W_, _static_sequence
from test_denoise_temporal_cpu import _px_to_cam, _translate
from test_denoise_variance_cpu import _lum_film

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_denoise_variance_temporal", "trb_denoise_variance_temporal_device", "trb_denoise_variance_temporal_gradient",
       "trb_denoise_variance_temporal_gradient_device"]
GW, GH = (W_ + 2) // 3, (H_ + 2) // 3
TAN = 0.5


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
    exe = str(tmp_path / "denoise_variance_temporal_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"),
                    os.path.join(REPO, "tests", "c", "denoise_variance_temporal_abi.c"), "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe],
                   check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    st = {l.split()[1]: int(l.split()[2]) for l in out if l.startswith("status ")}
    inv = st.pop("TRB_INVALID_ARG")
    st.pop("TRB_OK")
    assert len(st) == 23 and all(v == inv for v in st.values()), st


def _inputs():
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    return film, near, F.DenoiseFrame(*([film.ctypes.data] * 3), near.ctypes.data)


@pytest.mark.parametrize("bad", [dict(max_history=0), dict(max_history=256), dict(depth_tolerance=float("nan")), dict(depth_tolerance=0.0),
                                 dict(normal_threshold=1.5), dict(iterations=11), dict(normal_power=3), dict(sigma_luminance=0.0),
                                 dict(sigma_depth=float("inf"))])
def test_every_parameter_refusal_is_checked_before_the_scene(trb, bad):
    from tray_rust_b200.api import _gradient_params, _temporal_params
    film, near, d_in = _inputs()
    prm, gprm = _temporal_params(bad), _gradient_params(bad)
    out = F.DenoiseMomentsOutput(film.ctypes.data, None, None, None)
    gout = F.DenoiseMomentsGradientOutput(film.ctypes.data, None, None, None, None)
    lum = film.ctypes.data
    for fn in (lambda: trb.trb_denoise_variance_temporal(None, None, C.byref(d_in), lum, C.byref(prm), C.byref(out)),
               lambda: trb.trb_denoise_variance_temporal_device(None, None, C.byref(d_in), lum, C.byref(prm), C.byref(out), None),
               lambda: trb.trb_denoise_variance_temporal_gradient(None, None, C.byref(d_in), lum, C.byref(gprm), 1, C.byref(gout)),
               lambda: trb.trb_denoise_variance_temporal_gradient_device(None, None, C.byref(d_in), lum, C.byref(gprm), 1, C.byref(gout), None)):
        assert fn() == F.TRB_INVALID_ARG
        assert b"denoise" in trb.trb_last_error()
    colour, _, aovs = synthetic(np.random.default_rng(0), 4, 4, False)
    aovs["lum_w"] = np.ones((4, 4, 4), np.float32)
    with pytest.raises(ValueError):  # the oracle refuses them too
        VT.denoise_variance_temporal_lambda_frame(_frame(4, 4), VT.History(), colour, aovs, np.zeros(4, np.float32), **bad)


@pytest.mark.parametrize("gradient_iterations", [7, 2 ** 31])
def test_gradient_iterations_above_6_are_refused_before_the_scene(trb, gradient_iterations):
    from tray_rust_b200.api import _gradient_params
    film, near, d_in = _inputs()
    gprm = _gradient_params(dict(gradient_iterations=gradient_iterations))
    gout = F.DenoiseMomentsGradientOutput(film.ctypes.data, None, None, None, None)
    assert trb.trb_denoise_variance_temporal_gradient(None, None, C.byref(d_in), film.ctypes.data, C.byref(gprm), 1, C.byref(gout)) == F.TRB_INVALID_ARG
    assert b"iterations" in trb.trb_last_error()


def test_null_members_are_refused(trb):
    film, near, d_in = _inputs()
    out = F.DenoiseMomentsOutput(film.ctypes.data, None, None, None)
    gout = F.DenoiseMomentsGradientOutput(film.ctypes.data, None, None, None, None)
    for k in range(4):
        ptrs = [film.ctypes.data] * 3 + [near.ctypes.data]
        ptrs[k] = None
        bad = F.DenoiseFrame(*ptrs)
        assert trb.trb_denoise_variance_temporal(None, None, C.byref(bad), film.ctypes.data, None, C.byref(out)) == F.TRB_INVALID_ARG
        assert trb.trb_denoise_variance_temporal_gradient(None, None, C.byref(bad), film.ctypes.data, None, 1, C.byref(gout)) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_variance_temporal(None, None, C.byref(d_in), None, None, C.byref(out)) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_variance_temporal_device(None, None, C.byref(d_in), None, None, C.byref(out), None) == F.TRB_INVALID_ARG
    no_rgbw = F.DenoiseMomentsOutput(None, None, None, None)
    assert trb.trb_denoise_variance_temporal(None, None, C.byref(d_in), film.ctypes.data, None, C.byref(no_rgbw)) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_variance_temporal(None, None, C.byref(d_in), film.ctypes.data, None, None) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_variance_temporal(None, None, None, film.ctypes.data, None, C.byref(out)) == F.TRB_INVALID_ARG


def _api_scene():
    from tray_rust_b200 import api
    s = object.__new__(api.Scene)
    s.__dict__.update(height=4, width=6, _h=None, _lib=None)
    return s


def _good_aovs():
    return {"albedo_w": np.zeros((4, 6, 4), np.float32), "normal_w": np.zeros((4, 6, 4), np.float32), "nearest": np.zeros((4, 6), np.uint64),
            "lum_w": np.zeros((4, 6, 4), np.float32)}


@pytest.mark.parametrize("gradient", [False, True])
@pytest.mark.parametrize("which,bad", [("colour", np.zeros((4, 6, 4), np.float64)), ("lum_w", None), ("lum_w", np.zeros((4, 6, 3), np.float32)),
                                       ("nearest", np.zeros((4, 6), np.uint32)), ("out", np.zeros((4, 6, 3), np.float32)),
                                       ("variance", np.zeros((4, 6), np.float64)), ("history_length", np.zeros((4, 6), np.int32)),
                                       ("motion", np.zeros((4, 6, 2), np.float64))])
def test_python_argument_checks(gradient, which, bad):
    from tray_rust_b200 import api
    colour, aovs, kw = np.zeros((4, 6, 4), np.float32), _good_aovs(), {}
    if which == "colour":
        colour = bad
    elif which in aovs:
        aovs[which] = bad
    else:
        kw[which] = bad
    with pytest.raises(ValueError, match=which):
        if gradient:
            api.Scene.denoise_variance_temporal_gradient(_api_scene(), None, colour, aovs, 1, **kw)
        else:
            api.Scene.denoise_variance_temporal(_api_scene(), None, colour, aovs, **kw)


def test_python_lambda_check_and_unknown_parameters():
    from tray_rust_b200 import api
    with pytest.raises(ValueError, match="lambda"):
        api.Scene.denoise_variance_temporal_gradient(_api_scene(), None, np.zeros((4, 6, 4), np.float32), _good_aovs(), 1,
                                                     lam=np.zeros((6, 4), np.float32))
    with pytest.raises(TypeError):
        api.Scene.denoise_variance_temporal(_api_scene(), None, np.zeros((4, 6, 4), np.float32), _good_aovs(), gradient_iterations=3)
    with pytest.raises(TypeError):
        api.Scene.denoise_variance_temporal_gradient_device(_api_scene(), None, 0, 0, 0, 0, 0, 1, 0, lambda_=0)


def test_render_denoised_variance_temporal_refuses_spp_with_the_adaptive_sampler():
    from tray_rust_b200 import api
    with pytest.raises(ValueError, match="spp"):
        api.Scene.render_denoised_variance_temporal(_api_scene(), None, spp=4, adaptive=(2, 8))


# ---- trb_tray --denoise-variance-temporal -------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def programs():
    H.build_programs()


@pytest.mark.parametrize("args,needle", [(["--master", "127.0.0.1:1"], "not available with --master"),
                                         (["--worker"], "not available with --worker"),
                                         (["--devices", "0,1"], "one GPU"),
                                         (["--denoise"], "choose one denoiser"),
                                         (["--denoise-temporal"], "choose one denoiser"),
                                         (["--denoise-temporal", "--temporal-gradients"], "choose one denoiser"),
                                         (["--denoise-moments"], "choose one denoiser"),
                                         (["--denoise-moments", "--moment-gradients"], "choose one denoiser"),
                                         (["--denoise-variance"], "choose one denoiser"),
                                         (["--spp", "1"], "at least 2 samples"),
                                         (["--adaptive", "1", "8"], "MIN of at least 2"),
                                         (["--variance-gradients", "--spp", "1"], "at least 2 samples"),
                                         (["--variance-gradients", "--devices", "0"], "one GPU")])
def test_tray_denoise_variance_temporal_argument_refusals(programs, tmp_path, args, needle):
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    m = H.Proc([H.TRAY] + ([] if args == ["--worker"] else [missing]) + args + ["--denoise-variance-temporal", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and needle in err and "no_such_scene" not in err, err
    assert not (tmp_path / "x.png").exists()


@pytest.mark.parametrize("args,needle", [([], "--variance-gradients needs --denoise-variance-temporal"),
                                         (["--denoise-variance"], "--variance-gradients needs --denoise-variance-temporal"),
                                         (["--denoise-moments"], "--variance-gradients needs --denoise-variance-temporal"),
                                         (["--master", "127.0.0.1:1"], "--variance-gradients is not available with --master"),
                                         (["--worker"], "--variance-gradients is not available with --worker")])
def test_tray_variance_gradients_argument_refusals(programs, tmp_path, args, needle):
    missing = str(tmp_path / "no_such_scene.json")
    m = H.Proc([H.TRAY] + ([] if "--worker" in args else [missing]) + args + ["--variance-gradients", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and needle in err and "no_such_scene" not in err, err
    assert not (tmp_path / "x.png").exists()


def test_tray_denoise_variance_temporal_refuses_non_path_integrators_and_1_spp_scenes_before_rendering(programs, tmp_path):
    import json
    text = open(H.CORNELL).read().replace('"models/', '"%s/models/' % os.path.dirname(H.CORNELL))
    scene = json.loads(text)
    cases = (("whitted", dict(scene, integrator={"type": "whitted", "min_depth": 0, "max_depth": 4}), "path integrator"),
             ("one_spp", dict(scene, film=dict(scene["film"], samples=1)), "at least 2 samples"))
    for name, desc, needle in cases:
        path = str(tmp_path / ("%s.json" % name))
        with open(path, "w") as f:
            json.dump(desc, f)
        m = H.Proc([H.TRAY, path, "--denoise-variance-temporal", "--spp", "0", "-o", str(tmp_path / "x.png")])
        try:
            rc, _, err = m.finish(timeout=60)
        finally:
            m.kill()
        assert rc == 1 and needle in err and "--denoise-variance-temporal" in err, (name, err)
        assert not (tmp_path / "x.png").exists()


def test_usage_names_the_flags(programs):
    out = subprocess.run([H.TRAY, "--help"], capture_output=True, text=True).stdout
    assert "--denoise-variance-temporal" in out and "--variance-gradients" in out


# ---- the oracle against orc_denoise_variance and a float64 restatement ---------------------------------------------------------------

def _frame(w, h, cam=None, n_instances=2):
    """A frame with camera cam (default: 10 units back) and identity instances"""
    cam = np.asarray(_translate(0.0, 0.0, -10.0) if cam is None else cam, np.float32)
    cam_inv = np.linalg.inv(cam.astype(np.float64)).astype(np.float32)
    eye = [np.eye(4, dtype=np.float32)] * n_instances
    return G.make_frame(_px_to_cam(w, h), cam, cam_inv, TAN, eye, eye)


def _same(x, y):
    return np.asarray(x).tobytes() == np.asarray(y).tobytes()


def _moving_inputs(seed, n_frames, h=H_, w=W_):
    """n_frames of synthetic films with lum_w films over two depth planes, with specials (W <= 0, NaN, inf, misses, one effective
    sample, a whole border row below two effective samples) drawn afresh every frame under a camera that does not move"""
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n_frames):
        a, _, aovs = synthetic(rng, h, w, True)
        aovs["nearest"] = (aovs["nearest"] & ~np.uint64(0xffffffff)) | np.uint64(1)
        miss = rng.random((h, w)) < 0.05
        aovs["nearest"][miss] = np.uint64(0x7f800000 << 32) | np.uint64(0xffffffff)
        aovs["lum_w"] = _lum_film(rng, a, True)
        rows.append((a, aovs))
    return rows


def _zero(w=W_, h=H_):
    return np.zeros(((w + 2) // 3) * ((h + 2) // 3), np.float32)


@pytest.mark.parametrize("shape", [(H_, W_), (13, 21), (40, 9)])
@pytest.mark.parametrize("params", [{}, dict(iterations=0), dict(iterations=3, normal_power=16, sigma_luminance=1.5, sigma_depth=0.25)])
def test_empty_history_and_max_history_1_are_orc_denoise_variance_bit_for_bit(shape, params):
    h, w = shape
    f = _frame(w, h)
    fresh_each, one = VT.History(), VT.History()
    for k, (a, aovs) in enumerate(_moving_inputs(3 + h, 3, h, w)):
        want, want_var = V.denoise_variance(a, aovs, variance=True, **params)
        fresh_each.reset()
        for hist, mh in ((fresh_each, 8), (one, 1)):
            rgbw, motion, hl, var, lam = VT.denoise_variance_temporal_lambda_frame(f, hist, a, aovs, _zero(w, h), max_history=mh, **params)
            assert _same(rgbw, want) and _same(var, want_var), (k, mh)
            valid = ~np.isnan(want_var)
            assert (hl[valid] == 1).all() and (hl[~valid] == 0).all()
            assert np.isnan(motion[~valid]).all() and (motion.view(np.uint32)[np.isnan(motion)] == 0x7fffffff).all()
        assert (~valid).any() and valid.any()


def test_lambda_one_is_orc_denoise_variance_every_frame():
    f, hist = _frame(W_, H_), VT.History()
    for k, (a, aovs) in enumerate(_moving_inputs(31, 4)):
        want, want_var = V.denoise_variance(a, aovs, variance=True)
        rgbw, _, hl, var, lam = VT.denoise_variance_temporal_lambda_frame(f, hist, a, aovs, _zero() + 1)
        assert _same(rgbw, want) and _same(var, want_var) and (lam == 1).all(), k
        assert hl.max() == 1


def test_lambda_is_read_from_the_pixel_stratum():
    rng = np.random.default_rng(8)
    a, aovs = _moving_inputs(8, 1)[0]
    lam_s = rng.random(GW * GH).astype(np.float32)
    lam = VT.denoise_variance_temporal_lambda_frame(_frame(W_, H_), VT.History(), a, aovs, lam_s)[4]
    assert _same(lam, lam_s.reshape(GH, GW).repeat(3, 0).repeat(3, 1)[:H_, :W_])


def _static_lum(rng, cols, n_eff=None):
    """A lum_w film per colour film: V1 = W, V2 = V1^2 / n_eff (drawn per pixel and frame unless given), moments around the pixel's
    demodulated luminance"""
    out = []
    for c in cols:
        h, w = c.shape[:2]
        V1 = c[..., 3].astype(np.float64)
        n = rng.uniform(2.0, 30.0, (h, w)) if n_eff is None else np.full((h, w), float(n_eff))
        m1 = rng.uniform(0, 3, (h, w))
        s2 = rng.uniform(0, 1, (h, w)) ** 2
        out.append(np.stack([m1 * V1, (s2 + m1 * m1) * V1, V1 * V1 / n, V1], -1).astype(np.float32))
    return out


def _np_v(lum):
    lw = lum.astype(np.float64)
    m1, m2 = lw[..., 0] / lw[..., 3], lw[..., 1] / lw[..., 3]
    return np.maximum(m2 - m1 * m1, 0.0) * lw[..., 2] / (lw[..., 3] ** 2 - lw[..., 2])


# one lambda per frame, the same in every stratum: n' climbs, is halved, resets to 1, climbs again
LAMS = [0.0, 0.0, 0.0, 0.0, 0.5, 0.0, 1.0, 0.3, 0.0, 0.0, 0.0, 0.0]


@pytest.mark.parametrize("max_history", [8, 3])
def test_oracle_equals_the_float64_restatement_of_the_blend(max_history):
    rng = np.random.default_rng(40 + max_history)
    cols, aovs = _static_sequence(rng, len(LAMS))
    lums = _static_lum(rng, cols)
    f, hist = _frame(W_, H_), VT.History()
    z = (aovs["nearest"] >> np.uint64(32)).astype(np.uint32).view(np.float32)
    e_bar = V_ = npr = None
    seen = []
    for k, (c, lum, lam) in enumerate(zip(cols, lums, LAMS)):
        got = VT.denoise_variance_temporal_lambda_frame(f, hist, c, dict(aovs, lum_w=lum), np.full(GW * GH, lam, np.float32),
                                                        max_history=max_history, iterations=0)
        # steps 2-3 in float64: a static camera reprojects every pixel onto itself (its neighbours' taps weigh ~1e-6)
        e = c[..., :3].astype(np.float64) / c[..., 3:].astype(np.float64)
        vf = _np_v(lum)
        if npr is None:
            npr = np.ones(vf.shape, np.int64)
            e_bar, V_ = e, vf
        else:
            kept = np.isfinite(z)  # a pixel at infinite depth keeps no history
            npr = np.where(kept, np.minimum(np.floor((1.0 - np.float32(lam)) * npr.astype(np.float64)).astype(np.int64) + 1, max_history), 1)
            al = 1.0 / npr
            keep = npr > 1
            e_bar = np.where(keep[..., None], al[..., None] * e + (1 - al[..., None]) * e_bar, e)
            V_ = np.where(keep, al * al * vf + (1 - al) ** 2 * V_, vf)
        rgbw, motion, hl, var, _ = got
        assert np.array_equal(hl, npr.astype(np.uint32)), k
        np.testing.assert_allclose(var, V_, rtol=2e-4, atol=1e-6 * V_.max(), err_msg="frame %d" % k)
        # iterations 0: the output is ē * d, and ē blends the colour c / d, so it is the blend of c
        np.testing.assert_allclose(rgbw[..., :3], e_bar, rtol=2e-4, atol=1e-5 * np.abs(e_bar).max(), err_msg="frame %d" % k)
        seen.append(int(npr.max()))
    if max_history == 8:
        assert seen == [1, 2, 3, 4, 3, 4, 1, 1, 2, 3, 4, 5]
    else:
        assert seen == [1, 2, 3, 3, 2, 3, 1, 1, 2, 3, 3, 3]  # n' crosses max_history and stays there


def test_static_sequence_variance_follows_the_closed_form_of_the_recursion():
    """With v_f = v in every frame, V_k = v / k while n' = k <= M, then V_{k+1} = V_k (1 - 1/M)^2 + v / M^2 towards v / (2M - 1)"""
    M, frames = 5, 14
    rng = np.random.default_rng(77)
    cols, aovs = _static_sequence(rng, frames)
    lum = _static_lum(rng, cols[:1], n_eff=8)[0]
    f, hist = _frame(W_, H_), VT.History()
    v = V.denoise_variance(cols[0], dict(aovs, lum_w=lum), variance=True)[1].astype(np.float64)  # v_f in float32, as the call computes it
    kept = np.isfinite((aovs["nearest"] >> np.uint64(32)).astype(np.uint32).view(np.float32))  # infinite depth keeps no history
    assert kept.mean() > 0.5
    want = v.copy()
    for k in range(1, frames + 1):
        _, _, hl, var, _ = VT.denoise_variance_temporal_lambda_frame(f, hist, cols[k - 1], dict(aovs, lum_w=lum), _zero(), max_history=M)
        if k <= M:
            want = v / k
        else:
            want = want * (1 - 1 / M) ** 2 + v / M ** 2
        assert (hl[kept] == min(k, M)).all() and (hl[~kept] == 1).all()
        # the neighbours' taps weigh ~1e-6 each and carry their own V
        np.testing.assert_allclose(var[kept], want[kept], rtol=1e-4, atol=1e-6 * v.max(), err_msg="frame %d" % k)
        assert _same(var[~kept], v[~kept].astype(np.float32))
    Vstar = v / (2 * M - 1)
    closed = Vstar + (v / M - Vstar) * (1 - 1 / M) ** (2 * (frames - M))
    np.testing.assert_allclose(var[kept], closed[kept], rtol=1e-4, atol=1e-6 * v.max())


def test_invalid_pixels_have_nan_variance_no_history_and_still_a_lambda():
    a, aovs = _moving_inputs(7, 1)[0]
    lam_s = np.full(GW * GH, 0.25, np.float32)
    out, motion, hl, var, lam = VT.denoise_variance_temporal_lambda_frame(_frame(W_, H_), VT.History(), a, aovs, lam_s)
    bad = ~np.isfinite(a).all(-1) | (a[..., 3] <= 0)
    assert bad.any() and np.all(np.isnan(var[bad])) and np.all(hl[bad] == 0)
    assert np.all(var.view(np.uint32)[np.isnan(var)] == 0x7fffffff)
    assert np.all(out[a[..., 3] <= 0] == 0) and (lam == 0.25).all()

