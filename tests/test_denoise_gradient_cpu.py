"""The temporal gradients without a GPU: the struct layouts against ctypes and the Rust declarations in INTEGRATION.md, the exports, a
plain-C caller's statuses, the parameter refusals, trb_tray --temporal-gradients' argument refusals, and the oracle (oracle_gradient)
against a float64 numpy restatement of include/trb.h "Temporal gradients" steps 1-2 over synthetic records, and against the known
answers of step 3: no change gives lambda 0 and the plain temporal output, a full change lambda 1 and the spatial output."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F
from oracle_gradient import pygradient as G
from oracle_temporal import pytemporal as T
from test_denoise_temporal_cpu import _px_to_cam, _scene_inputs, _translate, _xf

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_denoise_temporal_gradient", "trb_denoise_temporal_gradient_device"]


def _run_abi(tmp_path):
    exe = str(tmp_path / "denoise_gradient_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"),
                    os.path.join(REPO, "tests", "c", "denoise_gradient_abi.c"), "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_structs_match_the_header_ctypes_and_the_rust_declarations(tmp_path):
    out = _run_abi(tmp_path)
    sizes = {l.split()[0]: int(l.split()[2]) for l in out if " sizeof " in l}
    offs = {l.split()[0]: int(l.split()[1]) for l in out if l.split()[0].count(".") == 1 and not l.startswith("status")}
    assert sizes == {"trb_denoise_gradient_params": 48, "trb_denoise_gradient_output": 32}
    assert C.sizeof(F.DenoiseGradientParams) == 48 and C.sizeof(F.DenoiseGradientOutput) == 32
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for cls, cname, rust in ((F.DenoiseGradientParams, "trb_denoise_gradient_params", "TrbDenoiseGradientParams"),
                             (F.DenoiseGradientOutput, "trb_denoise_gradient_output", "TrbDenoiseGradientOutput")):
        cfields = [n.rstrip("_") for n, _ in cls._fields_]  # ctypes' lambda_ is the header's lambda
        for (name, _), cf in zip(cls._fields_, cfields):
            assert getattr(cls, name).offset == offs[cname + "." + cf], name
        m = re.search(r"pub struct %s \{(.*?)\}" % rust, doc, re.S)
        assert m, rust
        assert re.findall(r"(\w+)\s*:", m.group(1)) == cfields, rust


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
    from tray_rust_b200.api import _gradient_params
    return _gradient_params(kw)


@pytest.mark.parametrize("bad", [dict(gradient_iterations=7), dict(gradient_iterations=2 ** 31), dict(max_history=0),
                                 dict(depth_tolerance=float("nan")), dict(normal_threshold=1.5), dict(iterations=11)])
def test_every_parameter_refusal_is_checked_before_the_scene(trb, bad):
    film = np.zeros(16, np.float32)
    near = np.zeros(4, np.uint64)
    d_in = F.DenoiseInput(*([film.ctypes.data] * 4), near.ctypes.data)
    out = F.DenoiseGradientOutput(film.ctypes.data, None, None, None)
    prm = _params(**bad)
    for fn in (lambda: trb.trb_denoise_temporal_gradient(None, None, C.byref(d_in), C.byref(prm), 1, C.byref(out)),
               lambda: trb.trb_denoise_temporal_gradient_device(None, None, C.byref(d_in), C.byref(prm), 1, C.byref(out), None)):
        assert fn() == F.TRB_INVALID_ARG
        assert b"temporal" in trb.trb_last_error() or b"denoise" in trb.trb_last_error()


def test_unknown_parameters_are_refused_by_the_binding():
    with pytest.raises(TypeError):
        _params(gradients=3)


# ---- trb_tray --temporal-gradients ------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def programs():
    H.build_programs()


@pytest.mark.parametrize("args,needle", [([], "needs --denoise-temporal"), (["--denoise"], "needs --denoise-temporal"),
                                         (["--denoise-temporal", "--master", "127.0.0.1:1"], "not available with --master"),
                                         (["--denoise-temporal", "--worker"], "not available with --worker"),
                                         (["--worker"], "not available with --worker")])
def test_tray_temporal_gradients_argument_refusals(programs, tmp_path, args, needle):
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    m = H.Proc([H.TRAY] + ([] if "--worker" in args else [missing]) + args + ["--temporal-gradients", "-o", str(tmp_path / "x.png")])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 1 and needle in err and "no_such_scene" not in err, err
    assert not (tmp_path / "x.png").exists()


def test_usage_names_the_flag(programs):
    out = subprocess.run([H.TRAY, "--help"], capture_output=True, text=True).stdout
    assert "--temporal-gradients" in out and "--denoise-temporal only" in out


# ---- the oracle against a float64 restatement -------------------------------------------------------------------------------------

W_, H_ = 24, 18
GW, GH = 8, 6
TAN = 0.5


def _frame(cam, mats, shutter_open=0.0):
    cam = np.asarray(cam, np.float32)
    mats = np.asarray(mats, np.float32)
    invs = np.linalg.inv(mats.astype(np.float64)).astype(np.float32)
    f = G.make_frame(_px_to_cam(W_, H_), cam, np.linalg.inv(cam.astype(np.float64)).astype(np.float32), TAN, invs, mats, shutter_open)
    return f, (cam, mats, invs)


def _ray(cam, x, y):
    """float64 unit camera-space direction through raster (x, y), and its world origin and direction"""
    a = W_ / H_
    X, Y = (x / W_) * 2 * a - a, 1.0 - (y / H_) * 2.0
    d = np.array([TAN * X, TAN * Y, 1.0])
    d /= np.linalg.norm(d)
    return cam[:3, 3].astype(np.float64), cam[:3, :3].astype(np.float64) @ d


def _records(rng, cam, mats, invs):
    """One record per stratum at a pixel centre of it, on instance k % 3 at a depth in [2, 6): a float64 p_w taken to object space"""
    rec = np.zeros(GW * GH, G.RECORD_DTYPE)
    pix = []
    for s in range(GW * GH):
        sx, sy = s % GW, s // GW
        px, py = 3 * sx + int(rng.integers(0, 3)), 3 * sy + int(rng.integers(0, 3))
        o, d = _ray(cam.astype(np.float64), px + 0.5, py + 0.5)
        depth = 2.0 + 4.0 * rng.random()
        i = s % 3
        pw = o + depth * d
        rec[s]["p_o"] = _xf(invs[i].astype(np.float64), pw)
        rec[s]["inst"] = i if rng.random() > 0.1 else 0xffffffff
        rec[s]["o"], rec[s]["d"], rec[s]["time"] = o, d, 0.25
        rec[s]["key"] = py * W_ + px
        rec[s]["lum"] = rng.random()
        pix.append((px, py))
    return rec, pix


def _np_project(rec, cam, mats, nearest, n_prev=3, depth_tolerance=0.05):
    """Step 1's projection and winners in float64: target stratum -> (dist, j)"""
    cam64 = cam.astype(np.float64)
    cam_inv = np.linalg.inv(cam64)
    a = W_ / H_
    win = {}
    for j, r in enumerate(rec):
        i = int(r["inst"])
        if i == 0xffffffff or i >= len(mats) or i >= n_prev:
            continue
        pw = _xf(mats[i].astype(np.float64), r["p_o"].astype(np.float64))
        q = _xf(cam_inv, pw)
        if not q[2] > 0:
            continue
        X, Y = q[0] / (q[2] * TAN), q[1] / (q[2] * TAN)
        rx, ry = (X + a) / (2 * a) * W_, (Y - 1.0) / -2.0 * H_
        if not (0 <= rx < W_ and 0 <= ry < H_):
            continue
        px, py = int(rx), int(ry)
        key = int(nearest[py, px])
        z = np.array([key >> 32], np.uint32).view(np.float32)[0]
        if key & 0xffffffff != i:
            continue
        dist = np.linalg.norm(pw - cam64[:3, 3])
        if not abs(z - dist) <= depth_tolerance * z:
            continue
        t = (py // 3) * GW + px // 3
        if t not in win or (dist, j) < win[t]:
            win[t] = (dist, j)
    return win


def _np_lambda(win, rec, l_cur, normal_w, nearest, normal_threshold=0.9, iterations=3):
    """Step 1's (delta, m, c) and step 2 in float64"""
    S = GW * GH
    d, m, c = np.zeros(S), np.zeros(S), np.zeros(S)
    for t, (_, j) in win.items():
        lc, lp = float(l_cur[t]), float(rec[j]["lum"])
        d[t], m[t], c[t] = lc - lp, max(lc, lp), 1.0
    n, ids = np.zeros((S, 3)), np.zeros(S, np.uint64)
    for t in range(S):
        x, y = min(3 * (t % GW) + 1, W_ - 1), min(3 * (t // GW) + 1, H_ - 1)
        v = normal_w[y, x, :3].astype(np.float64) / normal_w[y, x, 3]
        if np.isfinite(v).all() and (v != 0).any():
            n[t] = v / np.linalg.norm(v)
        ids[t] = nearest[y, x] & np.uint64(0xffffffff)
    h = [1 / 16, 1 / 4, 3 / 8, 1 / 4, 1 / 16]
    for k in range(iterations):
        s = 1 << k
        d2, m2, c2 = np.zeros(S), np.zeros(S), np.zeros(S)
        for t in range(S):
            x, y = t % GW, t // GW
            Wt = sd = sm = 0.0
            for dy in range(-2, 3):
                for dx in range(-2, 3):
                    qx, qy = x + s * dx, y + s * dy
                    if not (0 <= qx < GW and 0 <= qy < GH):
                        continue
                    q = qy * GW + qx
                    if c[q] <= 0:
                        continue
                    if q != t:
                        pn, qn = (n[t] != 0).any(), (n[q] != 0).any()
                        if ids[q] != ids[t] or pn != qn or (pn and not n[t] @ n[q] >= normal_threshold):
                            continue
                    w = h[dx + 2] * h[dy + 2]
                    Wt, sd, sm = Wt + w, sd + w * d[q], sm + w * m[q]
            if Wt > 0:
                d2[t], m2[t], c2[t] = sd / Wt, sm / Wt, 1.0
        d, m, c = d2, m2, c2
    return np.where((c > 0) & (m > 0), np.minimum(1.0, np.abs(d) / np.where(m > 0, m, 1)), 0.0)


def _scene(rng, cam, mats, rec, pix):
    """Current-frame inputs: each record's pixel holds its instance at its float64 distance, except some with another instance or a
    depth 50% off; every other pixel a random instance and depth"""
    ids = rng.integers(0, 3, (H_, W_))
    depth = (2.0 + 4.0 * rng.random((H_, W_))).astype(np.float32)
    A, B, aovs = _scene_inputs(rng, H_, W_, ids, depth)
    near = aovs["nearest"]
    for j, (px, py) in enumerate(pix):
        i = int(rec[j]["inst"])
        if i == 0xffffffff:
            continue
        pw = _xf(mats[i].astype(np.float64), rec[j]["p_o"].astype(np.float64))
        dist = np.linalg.norm(pw - cam[:3, 3].astype(np.float64))
        u = rng.random()
        ii, zz = (i, dist) if u < 0.7 else ((i + 1) % 3, dist) if u < 0.85 else (i, dist * 1.5)
        near[py, px] = (np.uint64(np.array([zz], np.float32).view(np.uint32)[0]) << np.uint64(32)) | np.uint64(ii)
    return A, B, aovs


@pytest.mark.parametrize("move", ["nothing", "instance", "camera"])
def test_oracle_projection_winners_and_lambda_equal_the_float64_restatement(move):
    rng = np.random.default_rng(5)
    cam0 = _translate(0.0, 0.0, -1.0)
    mats0 = [np.eye(4), _translate(0.3, 0.1, 0.0), _translate(-0.2, 0.0, 0.5)]
    f0, (cam0, mats0, invs0) = _frame(cam0, mats0)
    rec, pix = _records(rng, cam0, mats0, invs0)
    cam1, mats1 = cam0.astype(np.float64), [m.astype(np.float64) for m in mats0]
    if move == "instance":
        mats1[1] = _translate(0.3, 0.1, 0.0) @ _translate(0.02, -0.01, 0.0)
    elif move == "camera":
        cam1 = _translate(0.01, 0.0, -1.0)
    f1, (cam1, mats1, _) = _frame(cam1, mats1, shutter_open=0.5)
    A, B, aovs = _scene(rng, cam1, mats1, rec, pix)
    l_cur = rng.random(GW * GH).astype(np.float32)
    slot, rays, dm, lam = G.lambda_frame(W_, H_, f1, rec, 3, mats0, cam0, 0.0, l_cur, aovs["normal_w"], aovs["nearest"])
    win = _np_project(rec, cam1, mats1, aovs["nearest"])
    got = {t: int(s) & 0xffffffff for t, s in enumerate(slot) if s != np.uint64(0xffffffffffffffff)}
    assert len(win) > GW * GH // 3, len(win)
    assert got == {t: j for t, (_, j) in win.items()}
    for t, j in got.items():  # the rays: the recorded one only where camera and instance did not move; time shifted by the shutter
        r = rays[t]
        reuse = move == "nothing" or (move == "instance" and rec[j]["inst"] != 1)
        assert np.array_equal(r["o"], rec[j]["o"]) == reuse or not reuse and np.allclose(r["o"], rec[j]["o"])
        assert r["key"] == rec[j]["key"] and r["sample"] == 0 and r["time"] == np.float32(0.25) + np.float32(0.5)
        if reuse:
            assert r["d"].tobytes() == rec[j]["d"].tobytes()
        else:
            pw = _xf(mats1[rec[j]["inst"]].astype(np.float64), rec[j]["p_o"].astype(np.float64))
            want = (pw - cam1[:3, 3]) / np.linalg.norm(pw - cam1[:3, 3])
            np.testing.assert_allclose(r["d"], want, atol=1e-5)
    want = _np_lambda(win, rec, l_cur, aovs["normal_w"], aovs["nearest"])
    np.testing.assert_allclose(lam, want, rtol=1e-4, atol=1e-5)
    assert (lam > 0).sum() > 10


def test_lambda_of_every_iteration_count_equals_the_float64_restatement():
    rng = np.random.default_rng(8)
    f, (cam, mats, invs) = _frame(np.eye(4), [np.eye(4)] * 3)
    rec, pix = _records(rng, cam, mats, invs)
    A, B, aovs = _scene(rng, cam, mats, rec, pix)
    l_cur = rng.random(GW * GH).astype(np.float32)
    win = _np_project(rec, cam, mats, aovs["nearest"])
    for it in range(7):
        for thr in (0.9, -1.0):
            lam = G.lambda_frame(W_, H_, f, rec, 3, mats, cam, 0.0, l_cur, aovs["normal_w"], aovs["nearest"], normal_threshold=thr, iterations=it)[3]
            np.testing.assert_allclose(lam, _np_lambda(win, rec, l_cur, aovs["normal_w"], aovs["nearest"], thr, it), rtol=1e-4, atol=1e-5)


def _temporal_pair(lam_value):
    """Three frames of a static synthetic scene through the plain temporal oracle and the lambda oracle with a constant lambda"""
    rng = np.random.default_rng(3)
    ids = np.broadcast_to((np.arange(W_)[None, :] // 8) % 3, (H_, W_)).copy()
    tf = T.make_frame(_px_to_cam(W_, H_), np.eye(4), np.eye(4), TAN, [np.eye(4)] * 3, [np.eye(4)] * 3)
    gf = _frame(np.eye(4), [np.eye(4)] * 3)[0]
    th, gh = T.History(), G.History()
    rows = []
    for k in range(3):
        A, B, aovs = _scene_inputs(rng, H_, W_, ids, np.float32(3.0))
        plain = T.denoise_temporal_frame(tf, th, A, B, aovs, iterations=2)
        lam_s = np.full(GW * GH, lam_value, np.float32)
        grad = G.denoise_temporal_lambda_frame(gf, gh, A, B, aovs, lam_s, iterations=2)
        rows.append((plain, grad))
    return rows


def test_delta_zero_gives_lambda_zero_and_the_plain_temporal_output():
    rng = np.random.default_rng(9)
    f, (cam, mats, invs) = _frame(np.eye(4), [np.eye(4)] * 3)
    rec, pix = _records(rng, cam, mats, invs)
    A, B, aovs = _scene(rng, cam, mats, rec, pix)
    _, _, dm, lam = G.lambda_frame(W_, H_, f, rec, 3, mats, cam, 0.0, rec["lum"], aovs["normal_w"], aovs["nearest"])
    assert (dm[:, 2] > 0).sum() > 10 and not dm[:, 0].any() and not lam.any()
    for k, (plain, grad) in enumerate(_temporal_pair(0.0)):
        for x, y in zip(plain, grad[:3]):
            assert x.tobytes() == y.tobytes(), k
        assert not grad[3].any()
    assert plain[2].max() == 3


def test_m_equal_to_delta_gives_lambda_one_and_the_spatial_output():
    rng = np.random.default_rng(10)
    f, (cam, mats, invs) = _frame(np.eye(4), [np.eye(4)] * 3)
    rec, pix = _records(rng, cam, mats, invs)
    rec["lum"] = 0.0
    A, B, aovs = _scene(rng, cam, mats, rec, pix)
    l_cur = 0.25 + rng.random(GW * GH).astype(np.float32)
    slot, _, dm, lam = G.lambda_frame(W_, H_, f, rec, 3, mats, cam, 0.0, l_cur, aovs["normal_w"], aovs["nearest"], iterations=0)
    won = slot != np.uint64(0xffffffffffffffff)
    assert won.sum() > 10 and np.array_equal(dm[won, 0], dm[won, 1]) and (lam[won] == 1.0).all() and not lam[~won].any()
    for k, (_, grad) in enumerate(_temporal_pair(1.0)):
        assert grad[2].max() == 1 and (grad[3] == 1.0).all(), k
    # lambda 1 everywhere is the first call of a history, which is the spatial filter's output bit for bit
    tf = T.make_frame(_px_to_cam(W_, H_), np.eye(4), np.eye(4), TAN, [np.eye(4)] * 3, [np.eye(4)] * 3)
    rng = np.random.default_rng(3)
    ids = np.broadcast_to((np.arange(W_)[None, :] // 8) % 3, (H_, W_)).copy()
    gf = _frame(np.eye(4), [np.eye(4)] * 3)[0]
    gh, th = G.History(), T.History()
    for k in range(3):
        A, B, aovs = _scene_inputs(rng, H_, W_, ids, np.float32(3.0))
        grad = G.denoise_temporal_lambda_frame(gf, gh, A, B, aovs, np.ones(GW * GH, np.float32), iterations=2)
        th.reset()
        first = T.denoise_temporal_frame(tf, th, A, B, aovs, iterations=2)
        assert grad[0].tobytes() == first[0].tobytes() and grad[2].tobytes() == first[2].tobytes(), k
