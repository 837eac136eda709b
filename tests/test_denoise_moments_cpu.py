"""The moment denoiser without a GPU: the struct layouts against ctypes and the Rust declarations in INTEGRATION.md, the exports, a
plain-C caller's statuses, the parameter refusals, the Python argument checks, trb_tray --denoise-moments's argument refusals, and
the oracle (oracle_moments) against a float64 numpy restatement of include/trb.h "Moment denoising" steps 1, 3 and 4 over static
synthetic frames: a constant image has no variance, the 7x7 estimate with its 4 / n' boost below TRB_DENOISE_MOMENTS_MIN_HISTORY
frames, and the pixel's own moments from there on."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F
from oracle_moments import pymoments as M
from test_denoise_cpu import EPS_A, EPS_L, EPS_Z, _lum, synthetic
from test_denoise_temporal_cpu import _frame, _static_frame, _translate

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_denoise_moments", "trb_denoise_moments_device"]


def _run_abi(tmp_path):
    exe = str(tmp_path / "denoise_moments_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"),
                    os.path.join(REPO, "tests", "c", "denoise_moments_abi.c"), "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_structs_match_the_header_ctypes_and_the_rust_declarations(tmp_path):
    out = _run_abi(tmp_path)
    sizes = {l.split()[0]: int(l.split()[2]) for l in out if " sizeof " in l}
    offs = {l.split()[0]: int(l.split()[1]) for l in out if l.split()[0].count(".") == 1 and not l.startswith("status")}
    assert sizes == {"trb_denoise_frame": 32, "trb_denoise_moments_output": 32}
    assert C.sizeof(F.DenoiseFrame) == 32 and C.sizeof(F.DenoiseMomentsOutput) == 32
    consts = {l.split()[1]: int(l.split()[2]) for l in out if l.startswith("const ")}
    assert consts == {"TRB_DENOISE_MOMENTS_MIN_HISTORY": F.DENOISE_MOMENTS_MIN_HISTORY, "TRB_DENOISE_MOMENTS_RADIUS": F.DENOISE_MOMENTS_RADIUS}
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for cls, cname, rust in ((F.DenoiseFrame, "trb_denoise_frame", "TrbDenoiseFrame"),
                             (F.DenoiseMomentsOutput, "trb_denoise_moments_output", "TrbDenoiseMomentsOutput")):
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
    inv = st.pop("TRB_INVALID_ARG")
    st.pop("TRB_OK")
    assert st and all(v == inv for v in st.values()), st


def _params(**kw):
    from tray_rust_b200.api import _temporal_params
    return _temporal_params(kw)


@pytest.mark.parametrize("bad", [dict(max_history=0), dict(max_history=256), dict(depth_tolerance=0.0), dict(depth_tolerance=float("inf")),
                                 dict(normal_threshold=1.5), dict(normal_threshold=float("nan")), dict(iterations=11),
                                 dict(normal_power=3), dict(sigma_luminance=0.0), dict(sigma_depth=float("nan"))])
def test_every_parameter_refusal_is_checked_before_the_scene(trb, bad):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    d_in = F.DenoiseFrame(*([film.ctypes.data] * 3), near.ctypes.data)
    out = F.DenoiseMomentsOutput(film.ctypes.data, None, None, None)
    prm = _params(**bad)
    for fn in (lambda: trb.trb_denoise_moments(None, None, C.byref(d_in), C.byref(prm), C.byref(out)),
               lambda: trb.trb_denoise_moments_device(None, None, C.byref(d_in), C.byref(prm), C.byref(out), None)):
        assert fn() == F.TRB_INVALID_ARG
        assert b"temporal" in trb.trb_last_error() or b"denoise" in trb.trb_last_error()
    a, _, aovs = synthetic(np.random.default_rng(0), 4, 4, False)
    with pytest.raises(ValueError):  # the oracle refuses them too
        M.denoise_moments_frame(_static_frame(4, 4)[0], M.History(), a, aovs, **bad)


def test_null_members_are_refused(trb):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    out = F.DenoiseMomentsOutput(film.ctypes.data, None, None, None)
    for k in range(4):
        ptrs = [film.ctypes.data] * 3 + [near.ctypes.data]
        ptrs[k] = None
        d_in = F.DenoiseFrame(*ptrs)
        assert trb.trb_denoise_moments(None, None, C.byref(d_in), None, C.byref(out)) == F.TRB_INVALID_ARG
    d_in = F.DenoiseFrame(*([film.ctypes.data] * 3), near.ctypes.data)
    assert trb.trb_denoise_moments(None, None, C.byref(d_in), None, C.byref(F.DenoiseMomentsOutput())) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_moments(None, None, None, None, C.byref(out)) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_moments(None, None, C.byref(d_in), None, None) == F.TRB_INVALID_ARG


def _api_scene():
    from tray_rust_b200 import api
    s = object.__new__(api.Scene)
    s.__dict__.update(height=4, width=6, _h=None, _lib=None)
    return s


@pytest.mark.parametrize("which,bad", [("colour", np.zeros((4, 6, 4), np.float64)), ("colour", np.zeros((6, 4, 4), np.float32)),
                                       ("albedo_w", None), ("nearest", np.zeros((4, 6), np.uint32)),
                                       ("out", np.zeros((4, 6, 3), np.float32)), ("variance", np.zeros((4, 6), np.float64)),
                                       ("motion", np.zeros((4, 6, 2), np.float32)[:, ::-1]),
                                       ("history_length", np.zeros((4, 6), np.int32))])
def test_python_argument_checks(which, bad):
    from tray_rust_b200 import api
    s = _api_scene()
    colour = np.zeros((4, 6, 4), np.float32)
    aovs = {"albedo_w": np.zeros((4, 6, 4), np.float32), "normal_w": np.zeros((4, 6, 4), np.float32), "nearest": np.zeros((4, 6), np.uint64)}
    kw = {}
    if which == "colour":
        colour = bad
    elif which in aovs:
        aovs[which] = bad
    else:
        kw[which] = bad
    with pytest.raises(ValueError, match=which):
        api.Scene.denoise_moments(s, None, colour, aovs, **kw)
    good = {"albedo_w": np.zeros((4, 6, 4), np.float32), "normal_w": np.zeros((4, 6, 4), np.float32), "nearest": np.zeros((4, 6), np.uint64)}
    with pytest.raises(TypeError):
        api.Scene.denoise_moments(s, None, np.zeros((4, 6, 4), np.float32), good, history=3)


def test_render_denoised_moments_takes_the_whole_sample_range():
    from tray_rust_b200 import api
    for k in ("sample_first", "sample_count"):
        with pytest.raises(ValueError, match=k):
            api.Scene.render_denoised_moments(_api_scene(), None, spp=1, **{k: 0})


# ---- trb_tray --denoise-moments -----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def programs():
    H.build_programs()


@pytest.mark.parametrize("args,needle", [(["--master", "127.0.0.1:1"], "not available with --master"),
                                         (["--worker"], "not available with --worker"),
                                         (["--denoise"], "choose one denoiser"),
                                         (["--denoise-temporal"], "choose one denoiser"),
                                         (["--denoise-temporal", "--temporal-gradients"], "choose one denoiser"),
                                         (["--temporal-gradients"], "choose one denoiser")])
def test_tray_denoise_moments_argument_refusals(programs, tmp_path, args, needle):
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    m = H.Proc([H.TRAY] + ([] if args == ["--worker"] else [missing]) + args + ["--denoise-moments", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and needle in err and "no_such_scene" not in err, err
    assert not (tmp_path / "x.png").exists()


def test_tray_denoise_moments_refuses_non_path_integrators_before_rendering(programs, tmp_path):
    import json
    text = open(H.CORNELL).read().replace('"models/', '"%s/models/' % os.path.dirname(H.CORNELL))  # the copy lives elsewhere
    scene = json.loads(text)
    for name, integrator in (("whitted", {"type": "whitted", "min_depth": 0, "max_depth": 4}), ("normals", {"type": "normals_debug"})):
        path = str(tmp_path / ("%s.json" % name))
        with open(path, "w") as f:
            json.dump(dict(scene, integrator=integrator, film=dict(scene["film"], samples=1)), f)
        m = H.Proc([H.TRAY, path, "--denoise-moments", "-o", str(tmp_path / "x.png")])
        try:
            rc, _, err = m.finish(timeout=60)
        finally:
            m.kill()
        assert rc == 1 and "path integrator" in err, (name, err)
        assert not (tmp_path / "x.png").exists()


# ---- the oracle against a float64 restatement -------------------------------------------------------------------------------------

W_, H_ = 24, 16
DEF = dict(sigma_luminance=4.0, sigma_depth=1.0, normal_power=128)


def _guides(aovs):
    """Per pixel: the divisor d, the unit normal (0 if none), z and the depth gradient, in float64 (the contract's step 1)"""
    alb, nrm = aovs["albedo_w"].astype(np.float64), aovs["normal_w"].astype(np.float64)
    a = alb[..., :3] / alb[..., 3:]
    d = np.where(a > EPS_A, a, EPS_A)
    m = nrm[..., :3] / nrm[..., 3:]
    l2 = (m * m).sum(-1)
    n = np.where(l2[..., None] != 0, m / np.sqrt(np.where(l2 != 0, l2, 1))[..., None], 0.0)
    z = (aovs["nearest"] >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
    h, w = z.shape
    g = np.zeros((h, w, 2))
    for y in range(h):
        for x in range(w):
            if not np.isfinite(z[y, x]):
                continue
            for ax, (lo_ok, hi_ok, zlo, zhi) in enumerate(((x > 0, x + 1 < w, z[y, x - 1] if x > 0 else 0, z[y, x + 1] if x + 1 < w else 0),
                                                           (y > 0, y + 1 < h, z[y - 1, x] if y > 0 else 0, z[y + 1, x] if y + 1 < h else 0))):
                lo, hi = lo_ok and np.isfinite(zlo), hi_ok and np.isfinite(zhi)
                g[y, x, ax] = (zhi - zlo) * 0.5 if lo and hi else (zhi - z[y, x] if hi else (z[y, x] - zlo if lo else 0.0))
    return d, n, z, g


def _np_variance(e_bar, mu1, mu2, npr, n, z, g, sigma_luminance=4.0, sigma_depth=1.0, normal_power=128):
    """Step 4 in float64 for every pixel (all valid)"""
    h, w = z.shape
    v = np.zeros((h, w))
    L = _lum(e_bar)
    R = F.DENOISE_MOMENTS_RADIUS
    for y in range(h):
        for x in range(w):
            if npr[y, x] >= F.DENOISE_MOMENTS_MIN_HISTORY:
                v[y, x] = max(0.0, mu2[y, x] - mu1[y, x] ** 2)
                continue
            sw = s1 = s2 = 0.0
            p_nrm = n[y, x].any()
            for dy in range(-R, R + 1):
                for dx in range(-R, R + 1):
                    qx, qy = x + dx, y + dy
                    if not (0 <= qx < w and 0 <= qy < h):
                        continue
                    wl = np.exp(-abs(L[y, x] - L[qy, qx]) / (sigma_luminance + EPS_L))
                    q_nrm = n[qy, qx].any()
                    wn = (max(0.0, n[y, x] @ n[qy, qx]) ** normal_power) if p_nrm and q_nrm else float(p_nrm == q_nrm)
                    pi, qi = np.isinf(z[y, x]), np.isinf(z[qy, qx])
                    if pi or qi:
                        wz = float(pi and qi)
                    else:
                        wz = np.exp(-abs(z[y, x] - z[qy, qx]) / (sigma_depth * abs(g[y, x, 0] * dx + g[y, x, 1] * dy) + EPS_Z))
                    wt = wl * wn * wz
                    sw, s1, s2 = sw + wt, s1 + wt * mu1[qy, qx], s2 + wt * mu2[qy, qx]
            v[y, x] = max(0.0, s2 / sw - (s1 / sw) ** 2) * 4.0 / npr[y, x]
    return v


def _static_sequence(rng, n_frames, constant=False):
    """n_frames colour films over one set of AOVs (no specials: every pixel is valid in every frame)"""
    _, _, aovs = synthetic(rng, H_, W_, False)
    aovs["nearest"] = (aovs["nearest"] & ~np.uint64(0xffffffff)) | np.uint64(1)  # instance 1 of _oracle_sequence's frame
    # albedos away from the divisor's floor: a pixel reprojects onto itself up to rounding, so its neighbours' taps weigh ~1e-6, and
    # demodulated neighbours 1000 times brighter would show through that
    aovs["albedo_w"][..., :3] = rng.uniform(0.2, 1.0, (H_, W_, 3)) * aovs["albedo_w"][..., 3:]
    cols = []
    for _ in range(n_frames):
        c = rng.uniform(0, 3, (H_, W_, 3)) if not constant else np.full((H_, W_, 3), 0.7)
        wt = rng.uniform(0.5, 1.5, (H_, W_, 1))
        cols.append(np.concatenate([c * wt, wt], -1).astype(np.float32))
    return cols, aovs


def _np_sequence(cols, aovs, max_history=8):
    """Steps 1 and 3 in float64 on a static frame, where every finite-z pixel's history is itself: (ē, mu1, mu2, n') per frame"""
    d, n, z, g = _guides(aovs)
    out = []
    e_bar = mu1 = mu2 = None
    for k, col in enumerate(cols):
        c = col[..., :3].astype(np.float64) / col[..., 3:].astype(np.float64)
        e = c / d
        l = _lum(e)
        npr = np.where(np.isfinite(z), min(k + 1, max_history), 1)
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


def _oracle_sequence(cols, aovs, **params):
    frame = _frame(W_, H_, _translate(0, 0, -10.0), [np.eye(4)] * 2)[0]  # the camera 10 in front of the depth planes, never moving
    hist = M.History()
    return [M.denoise_moments_frame(frame, hist, c, aovs, **params) for c in cols]


def test_a_constant_image_has_no_variance():
    """Constant colour over a constant albedo: every pixel has the same demodulated luminance, so its variance is 0 up to rounding"""
    cols, aovs = _static_sequence(np.random.default_rng(3), 6, constant=True)
    aovs["albedo_w"][..., :3] = 0.5 * aovs["albedo_w"][..., 3:]
    l = 0.7 / 0.5
    for k, (_, _, hl, var) in enumerate(_oracle_sequence(cols, aovs)):
        assert np.all(var >= 0) and np.all(var <= 1e-5 * l * l), (k, var.max())  # a few float32 ulps of l^2, boosted


@pytest.mark.parametrize("max_history", [8, 3, 1])
def test_oracle_equals_the_float64_restatement(max_history):
    """The 7x7 estimate with its 4 / n' boost while n' < 4, and max(0, mu2 - mu1^2) from n' = 4 on; history lengths exact"""
    cols, aovs = _static_sequence(np.random.default_rng(11), 6)
    got = _oracle_sequence(cols, aovs, max_history=max_history)
    want, (d, n, z, g) = _np_sequence(cols, aovs, max_history)
    switched = False
    for k, ((rgbw, motion, hl, var), (e_bar, mu1, mu2, npr)) in enumerate(zip(got, want)):
        assert np.array_equal(hl, npr.astype(np.uint32)), k
        v64 = _np_variance(e_bar, mu1, mu2, npr, n, z, g)
        np.testing.assert_allclose(var, v64, rtol=1e-3, atol=1e-5 * np.abs(mu2).max(), err_msg="frame %d" % k)
        switched = switched or (npr >= F.DENOISE_MOMENTS_MIN_HISTORY).any()
        # the output with iterations 0 is ē * d
    assert switched == (max_history >= F.DENOISE_MOMENTS_MIN_HISTORY)
    e_bar = want[-1][0]
    out0 = _oracle_sequence(cols, aovs, max_history=max_history, iterations=0)[-1][0]
    np.testing.assert_allclose(out0[..., :3], e_bar * d, rtol=1e-4, atol=1e-6)
    assert np.all(out0[..., 3] == 1)


def test_the_boost_and_the_switch():
    """Over identical frames the spatial moments do not change, so the estimate scales by 4 / n' while n' < 4 (finite z); from
    n' = 4 on, the pixel's own moments, which do not vary, give (almost) zero"""
    cols, aovs = _static_sequence(np.random.default_rng(5), 1)
    got = _oracle_sequence(cols * 5, aovs)
    z = _guides(aovs)[2]
    finite = np.isfinite(z)
    v1 = got[0][3][finite]
    big = v1 > 1e-3
    assert big.sum() > finite.sum() // 2
    for k in (1, 2):
        np.testing.assert_allclose(got[k][3][finite][big] / v1[big], 1.0 / (k + 1), rtol=1e-3)
        assert np.all(got[k][2][finite] == k + 1)
    mu2 = _np_sequence(cols, aovs)[0][0][2]
    for k in (3, 4):
        assert np.all(got[k][3][finite] <= 1e-4 * (1 + mu2[finite])), k  # rounding of mu2 - mu1^2 only
        assert np.all(got[k][2][finite] == k + 1)


def test_invalid_pixels_have_nan_variance_and_no_history():
    rng = np.random.default_rng(7)
    a, _, aovs = synthetic(rng, H_, W_, True)
    out, motion, hl, var = _oracle_sequence([a], aovs)[0]
    bad = ~np.isfinite(a).all(-1) | (a[..., 3] <= 0)
    assert np.all(np.isnan(var[bad])) and np.all(hl[bad] == 0)
    assert np.all(var.view(np.uint32)[np.isnan(var)] == 0x7fffffff)
    assert np.all(out[a[..., 3] <= 0] == 0)
