"""The sample-variance denoiser without a GPU: the exports against INTEGRATION.md's Rust declarations, a plain-C caller's statuses,
the parameter and null-argument refusals, trb_tray --denoise-variance's argument refusals, the oracle's lum_w film against a numpy
restatement of RenderTarget::write over its own sample records, and orc_denoise_variance against a float64 numpy restatement of
include/trb.h "Sample variance" over synthetic films (misses, W <= 0, one effective sample, NaN and +-inf, every border) and on
known answers."""
import ctypes as C
import json
import os
import re
import subprocess
import zlib

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F, scenebuild as SB
from oracle_variance import pyvariance as V
from test_denoise_cpu import EPS_A, EPS_L, EPS_Z, H5, _flat, _lum, _shift, synthetic

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_render_aov_lum", "trb_render_aov_lum_device", "trb_render_adaptive_aov_lum", "trb_render_adaptive_aov_lum_device",
       "trb_denoise_variance", "trb_denoise_variance_device"]


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
    exe = str(tmp_path / "denoise_variance_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"),
                    os.path.join(REPO, "tests", "c", "denoise_variance_abi.c"), "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    st = {l.split()[1]: int(l.split()[2]) for l in out if l.startswith("status ")}
    inv = st.pop("TRB_INVALID_ARG")
    st.pop("TRB_OK")
    assert len(st) == 12 and all(v == inv for v in st.values()), st


def _params(**kw):
    from tray_rust_b200.api import _denoise_params
    return _denoise_params(kw)


@pytest.mark.parametrize("bad", [dict(iterations=11), dict(normal_power=3), dict(normal_power=2048), dict(sigma_luminance=0.0),
                                 dict(sigma_luminance=float("inf")), dict(sigma_depth=float("nan"))])
def test_every_parameter_refusal_is_checked_before_the_scene(trb, bad):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    d_in = F.DenoiseFrame(*([film.ctypes.data] * 3), near.ctypes.data)
    prm = _params(**bad)
    for fn in (lambda: trb.trb_denoise_variance(None, C.byref(d_in), film.ctypes.data, C.byref(prm), film.ctypes.data, None),
               lambda: trb.trb_denoise_variance_device(None, C.byref(d_in), film.ctypes.data, C.byref(prm), film.ctypes.data, None, None)):
        assert fn() == F.TRB_INVALID_ARG
        assert b"denoise" in trb.trb_last_error()
    colour, _, aovs = synthetic(np.random.default_rng(0), 4, 4, False)
    aovs["lum_w"] = np.ones((4, 4, 4), np.float32)
    with pytest.raises(ValueError):  # the oracle refuses them too
        V.denoise_variance(colour, aovs, **bad)


def test_null_members_are_refused(trb):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    for k in range(4):
        ptrs = [film.ctypes.data] * 3 + [near.ctypes.data]
        ptrs[k] = None
        d_in = F.DenoiseFrame(*ptrs)
        assert trb.trb_denoise_variance(None, C.byref(d_in), film.ctypes.data, None, film.ctypes.data, None) == F.TRB_INVALID_ARG
    d_in = F.DenoiseFrame(*([film.ctypes.data] * 3), near.ctypes.data)
    assert trb.trb_denoise_variance(None, C.byref(d_in), None, None, film.ctypes.data, None) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_variance(None, C.byref(d_in), film.ctypes.data, None, None, None) == F.TRB_INVALID_ARG
    assert trb.trb_denoise_variance(None, None, film.ctypes.data, None, film.ctypes.data, None) == F.TRB_INVALID_ARG


def _api_scene():
    from tray_rust_b200 import api
    s = object.__new__(api.Scene)
    s.__dict__.update(height=4, width=6, _h=None, _lib=None)
    return s


@pytest.mark.parametrize("which,bad", [("colour", np.zeros((4, 6, 4), np.float64)), ("lum_w", None), ("lum_w", np.zeros((4, 6, 3), np.float32)),
                                       ("nearest", np.zeros((4, 6), np.uint32)), ("out", np.zeros((4, 6, 3), np.float32)),
                                       ("variance", np.zeros((4, 6), np.float64))])
def test_python_argument_checks(which, bad):
    from tray_rust_b200 import api
    colour = np.zeros((4, 6, 4), np.float32)
    aovs = {"albedo_w": np.zeros((4, 6, 4), np.float32), "normal_w": np.zeros((4, 6, 4), np.float32), "nearest": np.zeros((4, 6), np.uint64),
            "lum_w": np.zeros((4, 6, 4), np.float32)}
    kw = {}
    if which == "colour":
        colour = bad
    elif which in aovs:
        aovs[which] = bad
    else:
        kw[which] = bad
    with pytest.raises(ValueError, match=which):
        api.Scene.denoise_variance(_api_scene(), colour, aovs, **kw)


def test_render_denoised_variance_refuses_spp_with_the_adaptive_sampler():
    from tray_rust_b200 import api
    with pytest.raises(ValueError, match="spp"):
        api.Scene.render_denoised_variance(_api_scene(), spp=4, adaptive=(2, 8))


# ---- trb_tray --denoise-variance ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def programs():
    H.build_programs()


@pytest.mark.parametrize("args,needle", [(["--master", "127.0.0.1:1"], "not available with --master"),
                                         (["--worker"], "not available with --worker"),
                                         (["--devices", "0,1"], "one GPU"),
                                         (["--denoise"], "choose one denoiser"),
                                         (["--denoise-temporal"], "choose one denoiser"),
                                         (["--denoise-moments"], "choose one denoiser"),
                                         (["--denoise-moments", "--moment-gradients"], "choose one denoiser"),
                                         (["--spp", "1"], "at least 2 samples"),
                                         (["--adaptive", "1", "8"], "MIN of at least 2")])
def test_tray_denoise_variance_argument_refusals(programs, tmp_path, args, needle):
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    m = H.Proc([H.TRAY] + ([] if args == ["--worker"] else [missing]) + args + ["--denoise-variance", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and needle in err and "no_such_scene" not in err, err
    assert not (tmp_path / "x.png").exists()


def test_tray_denoise_variance_spp_0_keeps_the_scenes_samples(programs, tmp_path):
    """--spp 0 means the scene's film.samples, as in every mode: not refused up front, then checked against the scene"""
    missing = str(tmp_path / "no_such_scene.json")
    m = H.Proc([H.TRAY, missing, "--spp", "0", "--denoise-variance", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and "no_such_scene" in err and "at least 2 samples" not in err, err
    scene = json.loads(open(H.CORNELL).read().replace('"models/', '"%s/models/' % os.path.dirname(H.CORNELL)))
    path = str(tmp_path / "one_spp.json")
    with open(path, "w") as f:
        json.dump(dict(scene, film=dict(scene["film"], samples=1)), f)
    m = H.Proc([H.TRAY, path, "--spp", "0", "--denoise-variance", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and "at least 2 samples" in err and "the scene has 1" in err, err
    assert not (tmp_path / "x.png").exists()


def test_tray_denoise_variance_refuses_non_path_integrators_and_1_spp_scenes_before_rendering(programs, tmp_path):
    text = open(H.CORNELL).read().replace('"models/', '"%s/models/' % os.path.dirname(H.CORNELL))  # the copy lives elsewhere
    scene = json.loads(text)
    cases = (("whitted", dict(scene, integrator={"type": "whitted", "min_depth": 0, "max_depth": 4}), "path integrator"),
             ("normals", dict(scene, integrator={"type": "normals_debug"}), "path integrator"),
             ("one_spp", dict(scene, film=dict(scene["film"], samples=1)), "at least 2 samples"))
    for name, desc, needle in cases:
        path = str(tmp_path / ("%s.json" % name))
        with open(path, "w") as f:
            json.dump(desc, f)
        m = H.Proc([H.TRAY, path, "--denoise-variance", "-o", str(tmp_path / "x.png")])
        try:
            rc, _, err = m.finish(timeout=60)
        finally:
            m.kill()
        assert rc == 1 and needle in err, (name, err)
        assert not (tmp_path / "x.png").exists()


# ---- the oracle's lum_w film against a numpy restatement ------------------------------------------------------------------------

def _np_lum_film(desc, table, samples, albedo, blocks, per_block):
    """RenderTarget::write's rules in numpy, float32 products, one offset of the footprint at a time over all samples: the filter
    table, the block's filter_pixel_width window, the 2x2 lock blocks, and (w l, w l^2, w^2, w)"""
    f = desc.film
    wd, ht = f.width, f.height
    fw, fh = np.float32(f.filter_w), np.float32(f.filter_h)
    inv_w, inv_h = np.float32(1) / fw, np.float32(1) / fh
    fpw_x, fpw_y = int(np.floor(fw / np.float32(0.5))), int(np.floor(fh / np.float32(0.5)))
    c = np.stack([samples["r"], samples["g"], samples["b"]], -1).astype(np.float32)
    d = np.where(albedo > np.float32(EPS_A), albedo, np.float32(EPS_A)).astype(np.float32)
    q = c / d
    l = (np.float32(0.2126) * q[:, 0] + np.float32(0.7152) * q[:, 1]) + np.float32(0.0722) * q[:, 2]
    sx, sy = samples["x"].astype(np.float32), samples["y"].astype(np.float32)
    bx = np.repeat(blocks[:, 0].astype(np.int64) * 8, per_block)
    by = np.repeat(blocks[:, 1].astype(np.int64) * 8, per_block)
    x_lo, x_hi = np.maximum(bx - fpw_x, 0), np.minimum(bx + 8 + fpw_x, wd - 1)
    y_lo, y_hi = np.maximum(by - fpw_y, 0), np.minimum(by + 8 + fpw_y, ht - 1)
    px, py = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)

    def takes(s, i, lo, hi, fpw):  # the 2x2 lock block of pixel i takes the sample
        b0 = (i >> 1) << 1
        w0, w1 = np.maximum(lo, b0), np.minimum(hi + 1, b0 + 2)
        return (s >= (w0 - fpw).astype(np.float32)) & (s < (w1 + fpw).astype(np.float32))

    film = np.zeros((ht * wd, 4), np.float64)
    r = max(fpw_x, fpw_y) + 2
    for dy in range(-r, r + 1):
        iy = py + dy
        fy = np.abs(iy.astype(np.float32) - (sy - np.float32(0.5))) * inv_h
        vy = (iy >= y_lo) & (iy <= y_hi) & ~(fy > fh) & takes(sy, iy, y_lo, y_hi, fpw_y)
        for dx in range(-r, r + 1):
            ix = px + dx
            fx = np.abs(ix.astype(np.float32) - (sx - np.float32(0.5))) * inv_w
            ok = vy & (ix >= x_lo) & (ix <= x_hi) & ~(fx > fw) & takes(sx, ix, x_lo, x_hi, fpw_x)
            fyi = np.minimum((fy * np.float32(16)).astype(np.uint32), 15)
            fxi = np.minimum((fx * np.float32(16)).astype(np.uint32), 15)
            w = table.reshape(-1)[fyi * 16 + fxi].astype(np.float32)
            vals = np.stack([w * l, w * (l * l), w * w, w], -1)
            np.add.at(film, (iy * wd + ix)[ok], vals[ok])
    return film.reshape(ht, wd, 4)


@pytest.mark.parametrize("filt", ["mitchell", "gaussian"])
def test_oracle_lum_film_equals_the_numpy_restatement(filt):
    desc = SB.scene_smallpt_like(32, 24, 4).finish()
    if filt == "gaussian":
        desc.film.filter_type, desc.film.filter_w, desc.film.filter_h, desc.film.filter_b = 1, 1.5, 1.5, 2.0
    o = V.VarianceOracleScene(desc)
    o.update_frame()
    samples, _ = o.render_samples(seed=5)
    blocks = o.block_list()
    per_block = len(samples) // len(blocks)
    rng = np.random.default_rng(2)
    aov = np.zeros(len(samples), F.AOV_SAMPLE_DTYPE)
    aov["albedo"] = rng.uniform(0, 1, (len(samples), 3)).astype(np.float32)
    aov["albedo"][rng.random(len(samples)) < 0.2] = 0  # misses and black albedo: the divisor's floor
    regions = np.repeat(blocks[:, 1] * (o.width // 8) + blocks[:, 0], per_block).astype(np.uint32)
    got = o.lum_film(samples, aov, regions)
    want = _np_lum_film(desc, o.filter_table(), samples, aov["albedo"], blocks, per_block)
    scale = np.abs(want).max(axis=(0, 1))
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-5 * scale.max())
    # the fourth channel is the colour film's W, and w^2 never negative
    colour = o.film_write(samples, regions)
    np.testing.assert_allclose(got[..., 3], colour[..., 3], rtol=1e-5, atol=1e-6)
    assert (got[..., 2] >= 0).all()
    if filt == "mitchell":
        assert (want[..., 2] > np.abs(want[..., 3]) ** 2 / per_block / 64).any()


# ---- orc_denoise_variance against a float64 restatement ---------------------------------------------------------------------------

def _lum_film(rng, colour, specials):
    """A lum_w film consistent with a plausible number of samples per pixel: V1 = the colour's W, V2 = V1^2 / n_eff, and moments
    around the pixel's demodulated luminance; with `specials`, one-sample pixels (V1^2 == V2), V1 <= 0, NaN and inf"""
    h, w = colour.shape[:2]
    V1 = colour[..., 3].astype(np.float64)
    n_eff = rng.uniform(1.5, 40, (h, w))
    V2 = V1 * V1 / n_eff
    m1 = rng.uniform(0, 3, (h, w))
    var = rng.uniform(0, 1, (h, w)) ** 3 * 2
    lum = np.stack([m1 * V1, (var + m1 * m1) * V1, V2, V1], -1).astype(np.float32)
    if specials:
        pick = lambda p: rng.random((h, w)) < p  # noqa: E731
        one = pick(0.05)
        lum[one, 2] = lum[one, 3] * lum[one, 3]
        lum[pick(0.03), 3] = 0
        lum[pick(0.02), 1] = np.nan
        lum[pick(0.02), 0] = np.inf
        lum[pick(0.02), 2] = np.inf
        lum[0, :, 2] = lum[0, :, 3] * lum[0, :, 3] * 2  # a whole border row below two effective samples
    return lum


def reference(colour, aovs, iterations=5, normal_power=128, sigma_luminance=4.0, sigma_depth=1.0):
    """include/trb.h "Sample variance" in float64, vectorised over the image, one tap offset at a time"""
    A = colour.astype(np.float64)
    alb, nrm, lw = (aovs[k].astype(np.float64) for k in ("albedo_w", "normal_w", "lum_w"))
    z = (aovs["nearest"] >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
    with np.errstate(all="ignore"):
        W = A[..., 3]
        empty = W <= 0
        c = A[..., :3] / W[..., None]
        albedo = alb[..., :3] / alb[..., 3:]
        d = np.where(albedo > EPS_A, albedo, EPS_A)
        e = c / d
        V1, V2 = lw[..., 3], lw[..., 2]
        m1, m2 = lw[..., 0] / V1, lw[..., 1] / V1
        s2 = m2 - m1 * m1
        l32 = aovs["lum_w"]  # the one-sample test is a float32 decision: V2 written as V1 * V1 is exactly that product there
        two = (l32[..., 3] > 0) & (l32[..., 3] * l32[..., 3] > l32[..., 2])
        v = np.where(two, np.where(s2 > 0, s2, 0.0) * V2 / (V1 * V1 - V2), np.nan)
        m = nrm[..., :3] / nrm[..., 3:]
        len2 = (m * m).sum(-1)
        fin = lambda x: np.isfinite(x).all(-1) if x.ndim == 3 else np.isfinite(x)  # noqa: E731
        valid = ~empty & fin(c) & fin(albedo) & fin(m) & fin(len2) & fin(e) & fin(v) & ~np.isnan(z) & (z != -np.inf)
        has_n = valid & (len2 != 0)
        n = np.where(has_n[..., None], m / np.sqrt(len2)[..., None], 0.0)
        zf = np.where(np.isfinite(z), z, np.nan)
        grads = []
        for dx, dy in ((1, 0), (0, 1)):
            lo, hi = _shift(zf, -dx, -dy, np.nan), _shift(zf, dx, dy, np.nan)
            g = np.where(np.isfinite(lo) & np.isfinite(hi), (hi - lo) * 0.5, np.where(np.isfinite(hi), hi - z, np.where(np.isfinite(lo), z - lo, 0.0)))
            grads.append(np.where(np.isfinite(z), g, 0.0))
        gx, gy = grads
        v0 = np.where(valid, v, np.nan)
        e = np.where(valid[..., None], e, 0.0)
        v = np.where(valid, v, 0.0)
        for it in range(iterations):
            s = 1 << it
            gs, gk = np.zeros_like(v), np.zeros_like(v)
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    k = (0.5 if dx == 0 else 0.25) * (0.5 if dy == 0 else 0.25)
                    vq = _shift(valid, dx, dy, False)
                    gk += k * vq
                    gs += k * np.where(vq, _shift(v, dx, dy, 0.0), 0.0)
            denom_l = sigma_luminance * np.sqrt(gs / gk) + EPS_L
            lp = _lum(e)
            se, sw, sv = np.zeros_like(e), np.zeros_like(v), np.zeros_like(v)
            for dy in range(-2, 3):
                for dx in range(-2, 3):
                    vq = _shift(valid, s * dx, s * dy, False)
                    eq, zq, nq = _shift(e, s * dx, s * dy, 0.0), _shift(z, s * dx, s * dy, 0.0), _shift(n, s * dx, s * dy, 0.0)
                    hq = _shift(has_n, s * dx, s * dy, False)
                    wl = np.exp(-np.abs(lp - _lum(eq)) / denom_l)
                    wn = np.where(has_n & hq, np.maximum(0.0, (n * nq).sum(-1)) ** normal_power, np.where(has_n == hq, 1.0, 0.0))
                    pi, qi = np.isinf(z), np.isinf(zq)
                    wz = np.where(pi | qi, np.where(pi & qi, 1.0, 0.0),
                                  np.exp(-np.abs(z - zq) / (sigma_depth * np.abs(gx * (s * dx) + gy * (s * dy)) + EPS_Z)))
                    w = np.where(vq, H5[dx + 2] * H5[dy + 2] * wl * wn * wz, 0.0)
                    se += w[..., None] * eq
                    sw += w
                    sv += w * w * np.where(vq, _shift(v, s * dx, s * dy, 0.0), 0.0)
            e = np.where(valid[..., None], se / sw[..., None], 0.0)
            v = np.where(valid, sv / (sw * sw), 0.0)
        out = np.zeros(A.shape)
        out[..., :3] = np.where(valid[..., None], e * d, np.where(empty[..., None], 0.0, c))
        out[..., 3] = np.where(empty, 0.0, 1.0)
    return out, v0, valid, empty


def _synthetic(rng, h, w, specials=True):
    A, _, aovs = synthetic(rng, h, w, specials)
    aovs["lum_w"] = _lum_film(rng, A, specials)
    return A, aovs


@pytest.mark.parametrize("shape", [(16, 16), (13, 21), (40, 9)])
@pytest.mark.parametrize("params", [dict(), dict(iterations=0), dict(iterations=1), dict(iterations=6, normal_power=16, sigma_luminance=1.5, sigma_depth=0.25),
                                    dict(iterations=3, normal_power=1024, sigma_luminance=30.0, sigma_depth=4.0)])
def test_oracle_equals_the_float64_restatement(shape, params):
    rng = np.random.default_rng(zlib.crc32(repr((shape, sorted(params.items()))).encode()))
    colour, aovs = _synthetic(rng, *shape)
    got, var = V.denoise_variance(colour, aovs, variance=True, **params)
    want, v0, valid, empty = reference(colour, aovs, **params)
    assert valid.sum() > 0.4 * valid.size and (~valid & ~empty).any() and empty.any()
    np.testing.assert_array_equal(np.isnan(var), ~valid)
    # m2 - m1^2 cancels in float32: each pixel's error is a few ulps of (|m2| + m1^2), scaled like v by V2 / (V1^2 - V2)
    lw = aovs["lum_w"].astype(np.float64)
    with np.errstate(all="ignore"):
        m1, m2 = lw[..., 0] / lw[..., 3], lw[..., 1] / lw[..., 3]
        cancel = (np.abs(m2) + m1 * m1) * lw[..., 2] / (lw[..., 3] ** 2 - lw[..., 2])
    err = np.abs(var[valid] - v0[valid])
    assert ((err == 0) | (err <= 1e-4 * np.abs(v0[valid]) + 1e-6 * cancel[valid])).all()  # infinite moments give v = 0 exactly
    assert np.array_equal(got[empty], np.zeros_like(got[empty]))
    copied = ~valid & ~empty
    np.testing.assert_allclose(got[copied], want[copied].astype(np.float32), rtol=1e-6, atol=0, equal_nan=True)
    scale = np.abs(want[valid]).max()
    np.testing.assert_allclose(got[valid], want[valid], rtol=1e-3, atol=1e-4 * scale)
    nan_bits = got.view(np.uint32)[np.isnan(got)]
    assert nan_bits.size and (nan_bits == 0x7fffffff).all()
    assert (var.view(np.uint32)[np.isnan(var)] == 0x7fffffff).all()


def test_at_most_one_effective_sample_is_copied_through():
    rng = np.random.default_rng(21)
    colour, aovs = _synthetic(rng, 12, 12, specials=False)
    lum = aovs["lum_w"]
    lum[3, 4, 2] = lum[3, 4, 3] * lum[3, 4, 3]  # V1^2 == V2: one sample
    lum[5, 6, 3] = 0.0
    lum[7, 8, 3] = -0.5
    got, var = V.denoise_variance(colour, aovs, variance=True)
    for y, x in ((3, 4), (5, 6), (7, 8)):
        assert np.isnan(var[y, x])
        np.testing.assert_array_equal(got[y, x, :3], colour[y, x, :3] / colour[y, x, 3])
        assert got[y, x, 3] == 1
    assert np.isfinite(var).sum() == var.size - 3


def _flat_lum(h, w, l, n=16, s2=0.0):
    """A lum_w film of n equal-weight samples per pixel with demodulated luminance mean l and variance s2"""
    lum = np.zeros((h, w, 4), np.float32)
    lum[..., 3] = n
    lum[..., 2] = n
    lum[..., 0] = n * np.asarray(l)
    lum[..., 1] = n * (s2 + np.asarray(l) ** 2)
    return lum


def test_a_constant_image_passes_unchanged():
    A, B, aovs = _flat(20, 28, (0.3, 0.6, 1.7))
    colour = A + B
    c = colour[..., :3] / colour[..., 3:]
    aovs["lum_w"] = _flat_lum(20, 28, _lum(c / 0.5), s2=0.3)
    for params in (dict(), dict(iterations=10), dict(normal_power=1, sigma_luminance=0.01)):
        out = V.denoise_variance(colour, aovs, **params)
        np.testing.assert_allclose(out[..., :3], c, rtol=2e-6, atol=0)
        assert (out[..., 3] == 1).all()


@pytest.mark.parametrize("iterations", [1, 5, 10])
def test_a_zero_variance_step_edge_stays_a_step(iterations):
    h, w = 16, 32
    colour = np.where(np.arange(w)[None, :, None] < 13, np.float32(0.2), np.float32(0.8)) * np.ones((h, w, 3), np.float32)
    A, B, aovs = _flat(h, w, colour)
    aovs["lum_w"] = _flat_lum(h, w, np.where(np.arange(w)[None, :] < 13, 0.4, 1.6) * np.ones((h, w)))
    out = V.denoise_variance(A + B, aovs, iterations=iterations)
    np.testing.assert_allclose(out[:, :13, :3], 0.2, rtol=1e-6, atol=0)
    np.testing.assert_allclose(out[:, 13:, :3], 0.8, rtol=1e-6, atol=0)


def test_zero_iterations_is_e_times_d():
    rng = np.random.default_rng(4)
    colour, aovs = _synthetic(rng, 16, 24, specials=False)
    out = V.denoise_variance(colour, aovs, iterations=0)
    c = colour[..., :3] / colour[..., 3:]
    a = aovs["albedo_w"][..., :3] / aovs["albedo_w"][..., 3:]
    d = np.where(a > np.float32(EPS_A), a, np.float32(EPS_A))
    np.testing.assert_array_equal(out[..., :3], (c / d) * d)
    assert (out[..., 3] == 1).all()
