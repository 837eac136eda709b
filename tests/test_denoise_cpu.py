"""The denoiser without a GPU: the struct layouts against ctypes and the Rust declarations in INTEGRATION.md, the exports, a plain-C
caller's statuses, every parameter refusal, Scene.denoise's shape checks, trb_tray --denoise's argument refusals, and the oracle
(oracle_denoise) against a float64 numpy restatement of DESIGN.md §4 "Denoising" on synthetic films and against known answers."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F
from oracle_denoise import pydenoise as D
from test_mesh_update_cpu import _unopened_scene

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_denoise", "trb_denoise_device"]
EPS_A, EPS_L, EPS_Z = 1e-3, 1e-6, 1e-2  # TRB_DENOISE_EPS_* of include/trb.h
H5 = np.array([1 / 16, 1 / 4, 3 / 8, 1 / 4, 1 / 16])


def _run_abi(tmp_path):
    exe = str(tmp_path / "denoise_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "denoise_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_structs_match_the_header_ctypes_and_the_rust_declarations(tmp_path):
    out = _run_abi(tmp_path)
    sizes = {l.split()[0]: int(l.split()[2]) for l in out if " sizeof " in l}
    offs = {l.split()[0]: int(l.split()[1]) for l in out if l.split()[0].count(".") == 1 and not l.startswith("status")}
    assert sizes == {"trb_denoise_input": 40, "trb_denoise_params": 16}
    assert C.sizeof(F.DenoiseInput) == 40 and C.sizeof(F.DenoiseParams) == 16
    for cls, cname in ((F.DenoiseInput, "trb_denoise_input"), (F.DenoiseParams, "trb_denoise_params")):
        for name, _ in cls._fields_:
            assert getattr(cls, name).offset == offs[cname + "." + name], name
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for rust, cls in (("TrbDenoiseInput", F.DenoiseInput), ("TrbDenoiseParams", F.DenoiseParams)):
        m = re.search(r"pub struct %s \{(.*?)\}" % rust, doc, re.S)
        assert m, rust
        assert re.findall(r"(\w+)\s*:", m.group(1)) == [n for n, _ in cls._fields_], rust
    header = open(os.path.join(REPO, "include", "trb.h")).read()
    for name, v in (("ALBEDO", EPS_A), ("LUMINANCE", EPS_L), ("DEPTH", EPS_Z)):
        assert float(re.search(r"#define TRB_DENOISE_EPS_%s ([0-9.e-]+)f" % name, header).group(1)) == v


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
            assert r.startswith("*") and (c is C.c_void_p or issubclass(c, C._Pointer)), (name, i, r, c)
        assert "`%s(" % name in doc, "no table row for " + name


def test_plain_c_caller_gets_the_argument_statuses(tmp_path):
    status = {l.split()[1]: int(l.split()[2]) for l in _run_abi(tmp_path) if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {k: F.TRB_INVALID_ARG for k in ("trb_denoise:null_scene", "trb_denoise:null_input", "trb_denoise:null_normal",
                                                     "trb_denoise:bad_params", "trb_denoise_device:null_scene", "trb_denoise_device:bad_params")}


BAD_PARAMS = [dict(iterations=11), dict(iterations=1000), dict(normal_power=0), dict(normal_power=3), dict(normal_power=2048),
              dict(normal_power=96), dict(sigma_luminance=0.0), dict(sigma_luminance=-1.0), dict(sigma_luminance=float("inf")),
              dict(sigma_luminance=float("nan")), dict(sigma_depth=0.0), dict(sigma_depth=-2.0), dict(sigma_depth=float("inf")),
              dict(sigma_depth=float("nan"))]


@pytest.mark.parametrize("bad", BAD_PARAMS)
def test_every_parameter_refusal_is_checked_before_the_scene(trb, bad):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    d_in = F.DenoiseInput(*(film.ctypes.data,) * 4, near.ctypes.data)
    prm = F.DenoiseParams(**dict(F.DENOISE_DEFAULTS, **bad))
    for call in (lambda: trb.trb_denoise(None, C.byref(d_in), C.byref(prm), F.ptr(film)),
                 lambda: trb.trb_denoise_device(None, C.byref(d_in), C.byref(prm), F.ptr(film), None)):
        assert call() == F.TRB_INVALID_ARG
        assert b"denoise" in trb.trb_last_error() and b"null" not in trb.trb_last_error()
    with pytest.raises(ValueError):  # the oracle refuses the same parameters
        D.denoise(np.ones((2, 2, 4), np.float32), np.ones((2, 2, 4), np.float32),
                  dict(albedo_w=np.ones((2, 2, 4), np.float32), normal_w=np.ones((2, 2, 4), np.float32), nearest=np.zeros((2, 2), np.uint64)), **bad)


@pytest.mark.parametrize("good", [dict(iterations=0), dict(iterations=10), dict(normal_power=1), dict(normal_power=1024),
                                  dict(sigma_luminance=1e-30), dict(sigma_depth=1e30)])
def test_edge_parameters_pass_the_checks(trb, good):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    d_in = F.DenoiseInput(*(film.ctypes.data,) * 4, near.ctypes.data)
    prm = F.DenoiseParams(**dict(F.DENOISE_DEFAULTS, **good))
    assert trb.trb_denoise(None, C.byref(d_in), C.byref(prm), F.ptr(film)) == F.TRB_INVALID_ARG
    assert b"null" in trb.trb_last_error()  # refused for the null scene, not for the parameters


def _aovs(h, w):
    return dict(albedo_w=np.zeros((h, w, 4), np.float32), normal_w=np.zeros((h, w, 4), np.float32), nearest=np.zeros((h, w), np.uint64))


@pytest.mark.parametrize("case", ["colour_a", "colour_b", "albedo_w", "normal_w", "nearest", "out", "float64", "missing"])
def test_scene_denoise_rejects_wrong_shapes_before_the_library(case):
    s = _unopened_scene()
    s.width, s.height = s._desc.film.width, s._desc.film.height
    a, b, aovs, out = np.zeros((8, 8, 4), np.float32), np.zeros((8, 8, 4), np.float32), _aovs(8, 8), None
    if case == "colour_a":
        a = np.zeros((8, 8, 3), np.float32)
    elif case == "colour_b":
        b = np.zeros((8, 8, 8), np.float32)[:, :, :4]
    elif case in ("albedo_w", "normal_w"):
        aovs[case] = np.zeros((8, 4, 4), np.float32)
    elif case == "nearest":
        aovs[case] = np.zeros((8, 8), np.uint32)
    elif case == "out":
        out = np.zeros((8, 8, 4), np.float64)
    elif case == "float64":
        a = np.zeros((8, 8, 4), np.float64)
    else:
        del aovs["normal_w"]
    with pytest.raises(ValueError):
        s.denoise(a, b, aovs, out=out)
    with pytest.raises(TypeError):
        s.denoise(np.zeros((8, 8, 4), np.float32), np.zeros((8, 8, 4), np.float32), _aovs(8, 8), sigma=1.0)
    s._h = None


def test_render_denoised_refuses_fewer_than_2_spp():
    s = _unopened_scene()
    s.width, s.height, s.spp = s._desc.film.width, s._desc.film.height, 1
    for spp in (0, 1):
        with pytest.raises(ValueError, match="at least 2 samples"):
            s.render_denoised(spp)
    s._h = None


# ---- trb_tray --denoise ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def programs():
    H.build_programs()


@pytest.mark.parametrize("args,needle", [(["--master", "127.0.0.1:1"], "not available with --master"),
                                         (["--worker"], "not available with --worker"),
                                         (["--spp", "1"], "at least 2 samples")])
def test_tray_denoise_argument_refusals(programs, tmp_path, args, needle):
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    m = H.Proc([H.TRAY] + ([] if args == ["--worker"] else [missing]) + args + ["--denoise", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and needle in err and "no_such_scene" not in err, err
    assert not (tmp_path / "x.png").exists()


def test_tray_denoise_refuses_a_1_spp_scene_and_non_path_integrators_before_rendering(programs, tmp_path):
    import json
    text = open(H.CORNELL).read().replace('"models/', '"%s/models/' % os.path.dirname(H.CORNELL))  # the copy lives elsewhere
    scene = json.loads(text)
    cases = [("spp1", dict(scene, film=dict(scene["film"], samples=1)), "at least 2 samples"),
             ("whitted", dict(scene, integrator={"type": "whitted", "min_depth": 0, "max_depth": 4}), "path integrator"),
             ("normals", dict(scene, integrator={"type": "normals_debug"}), "path integrator")]
    for name, desc, needle in cases:
        path = str(tmp_path / ("%s.json" % name))
        with open(path, "w") as f:
            json.dump(desc, f)
        d = H.load_desc(path)  # the copy loads, with the integrator and samples as written
        assert (d.contents.integrator.type != F.INTEGRATOR_PATH) == (name != "spp1") and (d.contents.film.samples == 1) == (name == "spp1")
        H.free_desc(d)
        m = H.Proc([H.TRAY, path, "--denoise", "-o", str(tmp_path / "x.png")])
        try:
            rc, _, err = m.finish(timeout=60)
        finally:
            m.kill()
        assert rc == 1 and needle in err, (name, err)
        assert not (tmp_path / "x.png").exists()


# ---- the oracle against a float64 restatement -----------------------------------------------------------------------------------

def _shift(a, dx, dy, fill):
    """b[y, x] = a[y + dy, x + dx], `fill` outside the image"""
    h, w = a.shape[:2]
    b = np.full_like(a, fill)
    ys, yd = (slice(dy, h), slice(0, h - dy)) if dy >= 0 else (slice(0, h + dy), slice(-dy, h))
    xs, xd = (slice(dx, w), slice(0, w - dx)) if dx >= 0 else (slice(0, w + dx), slice(-dx, w))
    if ys.stop > ys.start and xs.stop > xs.start:
        b[yd, xd] = a[ys, xs]
    return b


def _lum(e):
    return 0.2126 * e[..., 0] + 0.7152 * e[..., 1] + 0.0722 * e[..., 2]


def reference(A, B, aovs, iterations=5, normal_power=128, sigma_luminance=4.0, sigma_depth=1.0):
    """DESIGN.md §4 "Denoising" in float64, vectorised over the image, one tap offset at a time"""
    A, B = A.astype(np.float64), B.astype(np.float64)
    alb, nrm = aovs["albedo_w"].astype(np.float64), aovs["normal_w"].astype(np.float64)
    z = (aovs["nearest"] >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
    with np.errstate(all="ignore"):
        W = A[..., 3] + B[..., 3]
        empty = W <= 0
        c = (A[..., :3] + B[..., :3]) / W[..., None]
        albedo = alb[..., :3] / alb[..., 3:]
        d = np.where(albedo > EPS_A, albedo, EPS_A)
        e = c / d
        v = (_lum(A[..., :3] / A[..., 3:] / d) - _lum(B[..., :3] / B[..., 3:] / d)) ** 2 * 0.25
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
    return out, valid, empty


def synthetic(rng, h, w, specials=True):
    """Random half films of a plausible render: positive weights near 1, colours in [0, 4) with a few negative ones, two depth
    planes and misses, unit-ish normals; with `specials`, zero and negative weights, NaN / +-inf colours, albedos, normals and
    depths scattered over the image, borders included."""
    wa, wb = rng.uniform(0.5, 1.5, (h, w)).astype(np.float32), rng.uniform(0.5, 1.5, (h, w)).astype(np.float32)
    base = rng.uniform(0, 2, (h, w, 3))
    A = np.concatenate([(base + rng.uniform(-0.5, 2, (h, w, 3))) * wa[..., None], wa[..., None]], -1).astype(np.float32)
    B = np.concatenate([(base + rng.uniform(-0.5, 2, (h, w, 3))) * wb[..., None], wb[..., None]], -1).astype(np.float32)
    wsum = (wa + wb)[..., None]
    alb = np.concatenate([rng.uniform(0, 1, (h, w, 3)) * wsum, wsum], -1).astype(np.float32)
    alb[rng.random((h, w)) < 0.1, :3] = 0  # black albedo: the divisor's floor
    nr = rng.normal(size=(h, w, 3))
    nr[..., 2] = np.abs(nr[..., 2]) + 3
    nrm = np.concatenate([nr * wsum, wsum], -1).astype(np.float32)
    depth = np.where(np.arange(w)[None, :] < w // 2, 5.0 + 0.1 * np.arange(h)[:, None], 9.0 + 0.05 * np.arange(w)[None, :]).astype(np.float32)
    miss = rng.random((h, w)) < 0.1
    depth[miss] = np.inf
    nrm[miss, :3] = 0
    alb[miss, :3] = 0
    if specials:
        pick = lambda p: rng.random((h, w)) < p  # noqa: E731
        for arr, ch in ((A, 0), (B, 1), (alb, 2), (nrm, 0)):
            arr[pick(0.02), ch] = np.nan
            arr[pick(0.02), ch] = np.inf
            arr[pick(0.02), ch] = -np.inf
        zero = pick(0.05)
        zero[0, :3] = True
        zero[-1, -2:] = True
        zero[:, 0] &= pick(0.5)[:, 0]
        A[zero, 3] = 0
        B[zero, 3] = 0
        neg = pick(0.02)
        A[neg, 3] = -0.5
        B[neg, 3] = -0.25
        depth[pick(0.02)] = np.nan
        depth[pick(0.02)] = -np.inf
        A[pick(0.05), :3] *= -1  # negative colours
    near = (depth.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(3)
    return A, B, dict(albedo_w=alb, normal_w=nrm, nearest=near)


def assert_close_to_reference(got, want, valid, empty):
    """Float32 against float64: the exp and square-root arguments carry about 1e-6 of relative error, which the weights pass on
    scaled by their arguments (at most ~87 where dexp is not 0): 1e-3 of the local magnitude bounds it."""
    assert np.array_equal(got[empty], np.zeros_like(got[empty]))
    copied = ~valid & ~empty
    np.testing.assert_allclose(got[copied], want[copied].astype(np.float32), rtol=1e-6, atol=0, equal_nan=True)
    assert np.isfinite(got[valid]).all()
    scale = np.abs(want[valid]).max() if valid.any() else 1.0
    np.testing.assert_allclose(got[valid], want[valid], rtol=1e-3, atol=1e-4 * scale)


@pytest.mark.parametrize("shape", [(16, 16), (13, 21), (40, 9)])
@pytest.mark.parametrize("params", [dict(), dict(iterations=0), dict(iterations=1), dict(iterations=6, normal_power=16, sigma_luminance=1.5, sigma_depth=0.25),
                                    dict(iterations=3, normal_power=1024, sigma_luminance=30.0, sigma_depth=4.0)])
def test_oracle_equals_the_float64_restatement(shape, params):
    rng = np.random.default_rng(hash((shape, tuple(sorted(params.items())))) % 2**32)
    A, B, aovs = synthetic(rng, *shape)
    got = D.denoise(A, B, aovs, **params)
    want, valid, empty = reference(A, B, aovs, **params)
    assert valid.sum() > 0.5 * valid.size and (~valid & ~empty).any() and empty.any()
    assert_close_to_reference(got, want, valid, empty)
    assert np.isnan(got).any() and np.isinf(got).any()  # non-finite inputs are copied through


def test_oracle_equals_the_float64_restatement_without_specials():
    rng = np.random.default_rng(9)
    A, B, aovs = synthetic(rng, 24, 24, specials=False)
    for iterations in (1, 5, 10):
        got = D.denoise(A, B, aovs, iterations=iterations)
        want, valid, empty = reference(A, B, aovs, iterations=iterations)
        assert valid.all()
        assert_close_to_reference(got, want, valid, empty)


def _flat(h, w, colour, albedo=(0.5, 0.5, 0.5), depth=4.0, weight=(1.0, 1.0), noise=None):
    """two half films of `colour` (per pixel if an array) with the same guides everywhere: unit normal +z, constant depth"""
    col = np.broadcast_to(np.asarray(colour, np.float32), (h, w, 3))
    A = np.concatenate([col * np.float32(weight[0]), np.full((h, w, 1), weight[0], np.float32)], -1)
    B = np.concatenate([col * np.float32(weight[1]), np.full((h, w, 1), weight[1], np.float32)], -1)
    if noise is not None:
        A[..., :3] += noise.astype(np.float32)
        B[..., :3] -= noise.astype(np.float32)
    ws = np.float32(weight[0] + weight[1])
    alb = np.concatenate([np.broadcast_to(np.asarray(albedo, np.float32) * ws, (h, w, 3)), np.full((h, w, 1), ws, np.float32)], -1)
    nrm = np.concatenate([np.zeros((h, w, 2), np.float32), np.full((h, w, 2), ws, np.float32)], -1)
    near = np.full((h, w), (int(np.float32(depth).view(np.uint32)) << 32) | 1, np.uint64)
    return A, B, dict(albedo_w=np.ascontiguousarray(alb), normal_w=nrm, nearest=near)


def test_a_constant_image_is_unchanged():
    A, B, aovs = _flat(20, 28, (0.3, 0.6, 1.7), weight=(0.75, 1.25))
    c = (A[..., :3] + B[..., :3]) / (A[..., 3:] + B[..., 3:])
    for params in (dict(), dict(iterations=10), dict(normal_power=1, sigma_luminance=0.01)):
        out = D.denoise(A, B, aovs, **params)
        np.testing.assert_allclose(out[..., :3], c, rtol=2e-6, atol=0)
        assert (out[..., 3] == 1).all()


def test_zero_iterations_is_the_input_colour():
    rng = np.random.default_rng(4)
    A, B, aovs = synthetic(rng, 16, 24, specials=False)
    out = D.denoise(A, B, aovs, iterations=0)
    c = (A[..., :3] + B[..., :3]) / (A[..., 3:] + B[..., 3:])
    np.testing.assert_allclose(out[..., :3], c, rtol=2e-7, atol=0)
    assert (out[..., 3] == 1).all()


@pytest.mark.parametrize("shape", [(16, 16), (11, 23)])
def test_one_iteration_with_equal_guides_and_huge_sigma_is_the_b3_convolution(shape):
    h, w = shape
    rng = np.random.default_rng(7)
    colour = rng.uniform(0, 1, (h, w, 3))
    noise = rng.uniform(0.01, 0.02, (h, w, 3))  # a variance everywhere, so the luminance test's denominator is sigma * sqrt(g)
    A, B, aovs = _flat(h, w, colour, albedo=(1, 1, 1), noise=noise)
    out = D.denoise(A, B, aovs, iterations=1, normal_power=1, sigma_luminance=1e30)
    e = ((A[..., :3] + B[..., :3]) / (A[..., 3:] + B[..., 3:])).astype(np.float64)
    num, den = np.zeros_like(e), np.zeros((h, w))
    for dy in range(-2, 3):
        for dx in range(-2, 3):
            inside = _shift(np.ones((h, w), bool), dx, dy, False)
            num += H5[dx + 2] * H5[dy + 2] * _shift(e, dx, dy, 0.0)
            den += H5[dx + 2] * H5[dy + 2] * inside
    np.testing.assert_allclose(out[..., :3], num / den[..., None], rtol=1e-5, atol=0)


@pytest.mark.parametrize("iterations", [1, 5, 10])
def test_a_step_edge_with_zero_variance_stays_a_step(iterations):
    h, w = 16, 32
    colour = np.where(np.arange(w)[None, :, None] < 13, np.float32(0.2), np.float32(0.8)) * np.ones((h, w, 3), np.float32)
    A, B, aovs = _flat(h, w, colour)
    out = D.denoise(A, B, aovs, iterations=iterations)
    np.testing.assert_allclose(out[:, :13, :3], 0.2, rtol=1e-6, atol=0)
    np.testing.assert_allclose(out[:, 13:, :3], 0.8, rtol=1e-6, atol=0)
