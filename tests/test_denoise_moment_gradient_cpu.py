"""The moment gradients without a GPU: the output struct's layout against ctypes and the Rust declarations in INTEGRATION.md, the
exports, a plain-C caller's statuses, the parameter refusals, the Python argument checks, trb_tray --moment-gradients's argument
refusals, and the oracle (oracle_moment_gradient) over synthetic frames: lambda 0 everywhere is the moment oracle bit for bit, lambda
1 its max_history 1 output, and the lambda-shortened blend equals a float64 numpy restatement of include/trb.h "Moment gradients" as
n' crosses TRB_DENOISE_MOMENTS_MIN_HISTORY both ways."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F
from oracle_gradient import pygradient as G
from oracle_moment_gradient import pymomentgradient as MG
from oracle_moments import pymoments as M
from test_denoise_cpu import _lum, synthetic
from test_denoise_moments_cpu import H_, W_, _np_variance, _static_sequence, _guides
from test_denoise_temporal_cpu import _px_to_cam, _translate

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_denoise_moments_gradient", "trb_denoise_moments_gradient_device"]
GW, GH = (W_ + 2) // 3, (H_ + 2) // 3
TAN = 0.5


def _run_abi(tmp_path):
    exe = str(tmp_path / "denoise_moment_gradient_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"),
                    os.path.join(REPO, "tests", "c", "denoise_moment_gradient_abi.c"), "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe],
                   check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_output_struct_matches_the_header_ctypes_and_the_rust_declaration(tmp_path):
    out = _run_abi(tmp_path)
    sizes = {l.split()[0]: int(l.split()[2]) for l in out if " sizeof " in l}
    offs = {l.split()[0]: int(l.split()[1]) for l in out if l.split()[0].count(".") == 1 and not l.startswith("status")}
    assert sizes == {"trb_denoise_moments_gradient_output": 40}
    assert C.sizeof(F.DenoiseMomentsGradientOutput) == 40
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    cname = "trb_denoise_moments_gradient_output"
    for name, _ in F.DenoiseMomentsGradientOutput._fields_:
        assert getattr(F.DenoiseMomentsGradientOutput, name).offset == offs[cname + "." + name.rstrip("_")], name
    m = re.search(r"pub struct TrbDenoiseMomentsGradientOutput \{(.*?)\}", doc, re.S)
    assert m
    assert re.findall(r"(\w+)\s*:", m.group(1)) == [n.rstrip("_") for n, _ in F.DenoiseMomentsGradientOutput._fields_]


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
    inv = st.pop("TRB_INVALID_ARG")
    st.pop("TRB_OK")
    assert len(st) == 10 and all(v == inv for v in st.values()), st


def _params(**kw):
    from tray_rust_b200.api import _gradient_params
    return _gradient_params(kw)


@pytest.mark.parametrize("bad", [dict(gradient_iterations=7), dict(gradient_iterations=2 ** 31), dict(max_history=0), dict(max_history=256),
                                 dict(depth_tolerance=float("nan")), dict(normal_threshold=1.5), dict(iterations=11),
                                 dict(normal_power=3), dict(sigma_luminance=0.0)])
def test_every_parameter_refusal_is_checked_before_the_scene(trb, bad):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    d_in = F.DenoiseFrame(*([film.ctypes.data] * 3), near.ctypes.data)
    out = F.DenoiseMomentsGradientOutput(film.ctypes.data, None, None, None, None)
    prm = _params(**bad)
    for fn in (lambda: trb.trb_denoise_moments_gradient(None, None, C.byref(d_in), C.byref(prm), 1, C.byref(out)),
               lambda: trb.trb_denoise_moments_gradient_device(None, None, C.byref(d_in), C.byref(prm), 1, C.byref(out), None)):
        assert fn() == F.TRB_INVALID_ARG
        assert b"temporal" in trb.trb_last_error() or b"denoise" in trb.trb_last_error()
    a, _, aovs = synthetic(np.random.default_rng(0), 4, 4, False)
    with pytest.raises(ValueError):  # the oracle refuses them too
        MG.denoise_moments_lambda_frame(_frames(4, 4, np.eye(4))[1], MG.History(), a, aovs, np.zeros(4, np.float32), **bad)


def test_null_members_are_refused(trb):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    out = F.DenoiseMomentsGradientOutput(film.ctypes.data, None, None, None, None)
    for k in range(4):
        ptrs = [film.ctypes.data] * 3 + [near.ctypes.data]
        ptrs[k] = None
        d_in = F.DenoiseFrame(*ptrs)
        assert trb.trb_denoise_moments_gradient(None, None, C.byref(d_in), None, 1, C.byref(out)) == F.TRB_INVALID_ARG
    d_in = F.DenoiseFrame(*([film.ctypes.data] * 3), near.ctypes.data)
    assert trb.trb_denoise_moments_gradient(None, None, C.byref(d_in), None, 1, C.byref(F.DenoiseMomentsGradientOutput())) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_moments_gradient(None, None, None, None, 1, C.byref(out)) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_moments_gradient(None, None, C.byref(d_in), None, 1, None) == F.TRB_INVALID_ARG


def _api_scene():
    from tray_rust_b200 import api
    s = object.__new__(api.Scene)
    s.__dict__.update(height=4, width=6, _h=None, _lib=None)
    return s


def _good_aovs():
    return {"albedo_w": np.zeros((4, 6, 4), np.float32), "normal_w": np.zeros((4, 6, 4), np.float32), "nearest": np.zeros((4, 6), np.uint64)}


@pytest.mark.parametrize("which,bad", [("colour", np.zeros((4, 6, 4), np.float64)), ("nearest", np.zeros((4, 6), np.uint32)),
                                       ("out", np.zeros((4, 6, 3), np.float32)), ("variance", np.zeros((4, 6), np.float64)),
                                       ("lambda", np.zeros((4, 6), np.float64)), ("lambda", np.zeros((6, 4), np.float32)),
                                       ("lambda", np.zeros((4, 12), np.float32)[:, ::2])])
def test_python_argument_checks(which, bad):
    from tray_rust_b200 import api
    colour, aovs, kw = np.zeros((4, 6, 4), np.float32), _good_aovs(), {}
    if which == "colour":
        colour = bad
    elif which in aovs:
        aovs[which] = bad
    else:
        kw["lam" if which == "lambda" else which] = bad
    with pytest.raises(ValueError, match=which):
        api.Scene.denoise_moments_gradient(_api_scene(), None, colour, aovs, 1, **kw)


def test_unknown_parameters_are_refused_by_the_binding():
    from tray_rust_b200 import api
    with pytest.raises(TypeError):
        _params(gradients=3)
    with pytest.raises(TypeError):
        api.Scene.denoise_moments_gradient(_api_scene(), None, np.zeros((4, 6, 4), np.float32), _good_aovs(), 1, history=3)
    with pytest.raises(TypeError):
        api.Scene.denoise_moments_gradient_device(_api_scene(), None, 0, 0, 0, 0, 1, 0, lambda_=0)


# ---- trb_tray --moment-gradients ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def programs():
    H.build_programs()


@pytest.mark.parametrize("args,needle", [([], "needs --denoise-moments"), (["--denoise-temporal"], "needs --denoise-moments"),
                                         (["--master", "127.0.0.1:1"], "--moment-gradients is not available with --master"),
                                         (["--denoise-moments", "--master", "127.0.0.1:1"], "not available with --master"),
                                         (["--worker"], "--moment-gradients is not available with --worker"),
                                         (["--denoise-moments", "--worker"], "not available with --worker")])
def test_tray_moment_gradients_argument_refusals(programs, tmp_path, args, needle):
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    m = H.Proc([H.TRAY] + ([] if "--worker" in args else [missing]) + args + ["--moment-gradients", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and needle in err and "no_such_scene" not in err, err
    assert not (tmp_path / "x.png").exists()


def test_usage_names_the_flag(programs):
    out = subprocess.run([H.TRAY, "--help"], capture_output=True, text=True).stdout
    assert "--moment-gradients" in out and "--denoise-moments only" in out


# ---- the oracle against the moment oracle and a float64 restatement -----------------------------------------------------------------

def _frames(w, h, cam, n_instances=2):
    """The same frame (camera cam, identity instances) as the moment oracle's and the gradient oracle's frame types"""
    cam = np.asarray(cam, np.float32)
    cam_inv = np.linalg.inv(cam.astype(np.float64)).astype(np.float32)
    eye = [np.eye(4, dtype=np.float32)] * n_instances
    return (M.make_frame(_px_to_cam(w, h), cam, cam_inv, TAN, eye, eye),
            G.make_frame(_px_to_cam(w, h), cam, cam_inv, TAN, eye, eye))


def _moving_inputs(seed, n_frames, specials=True):
    """n_frames of synthetic films over two depth planes with specials (W <= 0, NaN, inf, misses) drawn afresh every frame, under
    a camera that does not move: a pixel keeps its history while it stays valid, and loses it where a special falls"""
    rng = np.random.default_rng(seed)
    rows = []
    for k in range(n_frames):
        a, _, aovs = synthetic(rng, H_, W_, specials)
        aovs["nearest"] = (aovs["nearest"] & ~np.uint64(0xffffffff)) | np.uint64(1)
        miss = rng.random((H_, W_)) < 0.05
        aovs["nearest"][miss] = np.uint64(0x7f800000 << 32) | np.uint64(0xffffffff)
        rows.append((_frames(W_, H_, _translate(0.0, 0.0, -10.0)), a, aovs))
    return rows


def _same(x, y):
    return np.asarray(x).tobytes() == np.asarray(y).tobytes()


@pytest.mark.parametrize("params", [{}, dict(max_history=3, iterations=0), dict(sigma_luminance=1.0, normal_power=16)])
def test_lambda_zero_is_the_moment_oracle_bit_for_bit(params):
    mh, gh = M.History(), MG.History()
    zero = np.zeros(GW * GH, np.float32)
    for k, ((mf, gf), a, aovs) in enumerate(_moving_inputs(5, 6)):
        want = M.denoise_moments_frame(mf, mh, a, aovs, **params)
        got = MG.denoise_moments_lambda_frame(gf, gh, a, aovs, zero, **params)
        for name, x, y in zip(("rgbw", "motion", "history_length", "variance"), want, got[:4]):
            assert _same(x, y), (k, name)
        assert not got[4].any()
    assert want[2].max() == params.get("max_history", 6) and (want[2] == 0).any() and (want[2] == 1).any()


def test_lambda_one_is_the_moment_oracle_at_max_history_1():
    mh, gh = M.History(), MG.History()
    one = np.ones(GW * GH, np.float32)
    for k, ((mf, gf), a, aovs) in enumerate(_moving_inputs(6, 4)):
        want = M.denoise_moments_frame(mf, mh, a, aovs, max_history=1)
        got = MG.denoise_moments_lambda_frame(gf, gh, a, aovs, one)
        for name, x, y in zip(("rgbw", "motion", "history_length", "variance"), want, got[:4]):
            assert _same(x, y), (k, name)
        assert (got[4] == 1.0).all() and got[2].max() == 1


def test_lambda_is_read_from_the_pixel_stratum():
    rng = np.random.default_rng(8)
    (_, gf), a, aovs = _moving_inputs(8, 1)[0]
    lam_s = rng.random(GW * GH).astype(np.float32)
    lam = MG.denoise_moments_lambda_frame(gf, MG.History(), a, aovs, lam_s)[4]
    want = lam_s.reshape(GH, GW).repeat(3, 0).repeat(3, 1)[:H_, :W_]
    assert _same(lam, want)


# one lambda per frame (the same in every stratum, so a pixel and the taps it reprojects onto share n'): n' climbs to 4, drops to 3
# (the spatial estimate with its 4/3 boost), climbs back, resets to 1 and stays 1 for floor(0.7 * 1) = 0
LAMS = [0.0, 0.0, 0.0, 0.0, 0.5, 0.0, 1.0, 0.3, 0.0]


def _np_lambda_sequence(cols, aovs, lams, max_history=8):
    """Steps 1 and 3 in float64 on a static frame with n' = min(floor((1 - lambda) len_prev) + 1, max_history): (ē, mu1, mu2, n')"""
    d, n, z, g = _guides(aovs)
    out = []
    e_bar = mu1 = mu2 = None
    npr = None
    for k, (col, lam) in enumerate(zip(cols, lams)):
        c = col[..., :3].astype(np.float64) / col[..., 3:].astype(np.float64)
        e = c / d
        l = _lum(e)
        if npr is None:
            npr = np.ones(z.shape, np.int64)
        else:
            hist = np.isfinite(z)
            npr = np.where(hist, np.minimum(np.floor((1.0 - np.float32(lam)) * npr.astype(np.float64)).astype(np.int64) + 1, max_history), 1)
        if e_bar is None:
            e_bar, mu1, mu2 = e, l, l * l
        else:
            a = 1.0 / npr
            keep = npr > 1
            e_bar = np.where(keep[..., None], a[..., None] * e + (1 - a[..., None]) * e_bar, e)
            mu1 = np.where(keep, a * l + (1 - a) * mu1, l)
            mu2 = np.where(keep, a * l * l + (1 - a) * mu2, l * l)
        out.append((e_bar, mu1, mu2, npr))
    return out, (d, n, z, g)


@pytest.mark.parametrize("max_history", [8, 3])
def test_oracle_equals_the_float64_restatement_of_the_shortened_blend(max_history):
    cols, aovs = _static_sequence(np.random.default_rng(12), len(LAMS))
    gf = _frames(W_, H_, _translate(0, 0, -10.0))[1]
    hist = MG.History()
    got = [MG.denoise_moments_lambda_frame(gf, hist, c, aovs, np.full(GW * GH, lam, np.float32), max_history=max_history)
           for c, lam in zip(cols, LAMS)]
    want, (d, n, z, g) = _np_lambda_sequence(cols, aovs, LAMS, max_history)
    seen = []
    for k, ((rgbw, motion, hl, var, lam), (e_bar, mu1, mu2, npr)) in enumerate(zip(got, want)):
        assert np.array_equal(hl, npr.astype(np.uint32)), k
        v64 = _np_variance(e_bar, mu1, mu2, npr, n, z, g)
        np.testing.assert_allclose(var, v64, rtol=1e-3, atol=1e-5 * np.abs(mu2).max(), err_msg="frame %d" % k)
        seen.append(int(npr.max()))
    if max_history == 8:
        assert seen == [1, 2, 3, 4, 3, 4, 1, 1, 2]  # across MIN_HISTORY up, down and up again, then reset
    else:
        assert seen == [1, 2, 3, 3, 2, 3, 1, 1, 2]


def test_invalid_pixels_have_nan_variance_and_no_history_and_still_a_lambda():
    (_, gf), a, aovs = _moving_inputs(7, 1)[0]
    lam_s = np.full(GW * GH, 0.25, np.float32)
    out, motion, hl, var, lam = MG.denoise_moments_lambda_frame(gf, MG.History(), a, aovs, lam_s)
    bad = ~np.isfinite(a).all(-1) | (a[..., 3] <= 0)
    assert bad.any() and np.all(np.isnan(var[bad])) and np.all(hl[bad] == 0)
    assert np.all(var.view(np.uint32)[np.isnan(var)] == 0x7fffffff)
    assert np.all(out[a[..., 3] <= 0] == 0) and (lam == 0.25).all()
