"""The temporal denoiser on an H100 (k_dn_temporal, then k_dn_atrous once per iteration): every frame's output, motion and history
length equal the oracle's orc_denoise_temporal bit for bit over sequences of the keyframed scene (with and without an animated fov), C1,
the textured scene and the MERL zoo, split and fused shading, and over synthetic films with specials; the first call, a call after
reset, max_history 1 and the first call after replace_objects equal trb_denoise; motion matches float64 projections; the device form
on a side stream equals the host form; the error cases leave the history as it was; trb_tray --denoise-temporal writes what
Scene.render_denoised_temporal computes; and accumulating over frames lowers the error and the flicker."""
import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_temporal import pytemporal as T
from test_aov_gpu import partial_wall
from test_denoise_cpu import synthetic
from test_denoise_gpu import halves, rmse
from test_queries_gpu import json_desc
from test_textures import textured_zoo

pytestmark = pytest.mark.gpu


def frame_times(k):
    return (k, 0.25 * k, 0.25 * (k + 1))


def run_sequence(desc, frames, seed=3, split=None, spp=2, **params):
    """Render frames as halves (seed + frame), denoise them with the library and the oracle; assert the three outputs bit for bit"""
    g, o = api.Scene(desc), T.Scene(desc)
    if split is not None:
        g.set_option("shade.split", split)
    hist, oh = api.DenoiseHistory(g), T.History()
    lens = []
    for k in frames:
        g.update_frame(*frame_times(k))
        o.update_frame(*frame_times(k))
        a, b, aovs = halves(g, spp=spp, seed=seed + k, flags=F.RENDER_NO_UPDATE)
        got = g.denoise_temporal(hist, a, b, aovs, motion=True, history_length=True, **params)
        want = T.denoise_temporal(o, oh, a, b, aovs, **params)
        for x, y, name in zip(got, want, ("rgbw", "motion", "history_length")):
            assert x.tobytes() == y.tobytes(), (k, name, np.argwhere(x.view(np.uint32) != y.view(np.uint32))[:5])
        lens.append(got[2])
    g.close()
    return lens


SEQ = {
    "animated": lambda: SB.scene_animated(48, 32, 2).finish(),
    "animated_fov": lambda: SB.scene_animated(48, 32, 2, animated_fov=True).finish(),
    "c1": lambda: json_desc("c1_cornell_box.json", 48, 32, 2),
    "textured": lambda: textured_zoo(2, 32).finish(),
    "zoo": lambda: SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()).finish(),
}


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("name", sorted(SEQ))
def test_sequences_equal_the_oracle(name, split):
    lens = run_sequence(SEQ[name](), range(5), split=split)
    assert lens[-1].max() > 1  # history was reused


@pytest.mark.parametrize("params", [dict(max_history=1), dict(max_history=2), dict(max_history=255, iterations=2),
                                    dict(depth_tolerance=1e-6, normal_threshold=1.0), dict(depth_tolerance=1e3, normal_threshold=-1.0)])
def test_history_parameters_equal_the_oracle(params):
    lens = run_sequence(SEQ["animated"](), range(4), **params)
    assert max(int(x.max()) for x in lens) <= params.get("max_history", 8)


def test_synthetic_films_with_specials_equal_the_oracle():
    g = api.Scene(partial_wall().finish())
    o = T.Scene(partial_wall().finish())
    g.update_frame()
    o.update_frame()
    hist, oh = api.DenoiseHistory(g), T.History()
    rng = np.random.default_rng(21)
    for k in range(3):
        a, b, aovs = synthetic(rng, g.height, g.width)
        aovs["nearest"] = (aovs["nearest"] & ~np.uint64(0xffffffff)) | rng.integers(0, 3, (g.height, g.width)).astype(np.uint64)
        got = g.denoise_temporal(hist, a, b, aovs, motion=True, history_length=True, iterations=2)
        want = T.denoise_temporal(o, oh, a, b, aovs, iterations=2)
        for x, y in zip(got, want):
            assert x.tobytes() == y.tobytes(), k


def test_identity_with_the_spatial_denoiser():
    desc = SB.scene_animated(48, 32, 2)
    g = api.Scene(desc.finish())
    hist = api.DenoiseHistory(g)
    outs = []
    for k in range(3):
        g.update_frame(*frame_times(k))
        a, b, aovs = halves(g, seed=k, flags=F.RENDER_NO_UPDATE)
        spatial = g.denoise(a, b, aovs)
        got = g.denoise_temporal(hist, a, b, aovs)
        assert (got.tobytes() == spatial.tobytes()) == (k == 0), k  # the first call only
        assert g.denoise_temporal(api.DenoiseHistory(g), a, b, aovs, max_history=1).tobytes() == spatial.tobytes()
        outs.append((a, b, aovs, spatial))
    hist.reset()
    a, b, aovs, spatial = outs[-1]
    assert g.denoise_temporal(hist, a, b, aovs).tobytes() == spatial.tobytes()  # after reset
    g.denoise_temporal(hist, a, b, aovs)
    g.replace_objects(desc.objects())  # renumbers instances: the history is of another generation
    g.update_frame(*frame_times(2))
    assert g.denoise_temporal(hist, a, b, aovs).tobytes() == g.denoise(a, b, aovs).tobytes()
    assert g.denoise_temporal(hist, a, b, aovs).tobytes() != g.denoise(a, b, aovs).tobytes()


def _motion_f64(g, aovs, cam_t, prev_cam_t, shift, tan):
    """float64 motion for a camera translated from prev_cam_t to cam_t (no rotation) and a scene translated by `shift` since"""
    h, w = g.height, g.width
    z = (aovs["nearest"] >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
    a = w / h
    x0, x1, y0, y1 = (-a, a, -1.0, 1.0) if a > 1 else (-1.0, 1.0, -1.0 / a, 1.0 / a)
    xs, ys = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    X, Y = xs / w * (x1 - x0) + x0, y1 - ys / h * (y1 - y0)
    d = np.stack([tan * X, tan * Y, np.ones_like(X)], -1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    p = np.asarray(cam_t) + z[..., None] * d - np.asarray(shift)
    q = p - np.asarray(prev_cam_t)
    rx = (q[..., 0] / (q[..., 2] * tan) - x0) / (x1 - x0) * w
    ry = (q[..., 1] / (q[..., 2] * tan) - y1) / (y0 - y1) * h
    return np.stack([rx - xs, ry - ys], -1), np.isfinite(z)


@pytest.mark.parametrize("move", ["instance", "camera", "nothing"])
def test_motion_matches_float64_projections(move):
    b = partial_wall()
    b.integrator = (F.INTEGRATOR_PATH, 1, 2)
    g = api.Scene(b.finish())
    hist = api.DenoiseHistory(g)
    tan = float(np.tan(np.radians(15.0)))
    cam0 = np.array(b.keyframes[-1][0], np.float64)
    g.update_frame()
    a, bb, aovs = halves(g, seed=1, flags=F.RENDER_NO_UPDATE)
    g.denoise_temporal(hist, a, bb, aovs)
    shift, cam1 = np.zeros(3), cam0.copy()
    idx = 0 if move == "instance" else len(b.keyframes) - 1
    if move != "nothing":
        t, q, s = b.keyframes[idx]
        delta = np.array([0.3, -0.2, 0.0])
        b.keyframes[idx] = (tuple(float(x) for x in np.asarray(t) + delta), q, s)
        g.update_keyframes(idx, np.array([b.keyframes[idx]], F.KEYFRAME_DTYPE))
        if move == "instance":
            shift = delta
        else:
            cam1 = cam0 + delta
    g.update_frame()
    a, bb, aovs = halves(g, seed=2, flags=F.RENDER_NO_UPDATE)
    _, motion, hl = g.denoise_temporal(hist, a, bb, aovs, motion=True, history_length=True)
    want, hit = _motion_f64(g, aovs, cam1, cam0, shift, tan)
    assert hit.sum() > 50
    err = np.abs(motion[hit] - want[hit]).max()
    print(move, "max motion error %.2e px, max |motion| %.3f px" % (err, np.abs(want[hit]).max()))
    assert err < 1e-3
    assert np.isnan(motion[~hit]).all()
    if move == "nothing":
        assert np.abs(motion[hit]).max() < 1e-3 and (hl[hit] == 2).mean() > 0.9


def test_device_form_on_a_side_stream_equals_the_host_form():
    import torch
    desc = SB.scene_animated(48, 32, 2).finish()
    g = api.Scene(desc)
    hist_h, hist_d = api.DenoiseHistory(g), api.DenoiseHistory(g)
    st = torch.cuda.Stream()
    for k in range(4):
        g.update_frame(*frame_times(k))
        a, b, aovs = halves(g, seed=k, flags=F.RENDER_NO_UPDATE)
        want = g.denoise_temporal(hist_h, a, b, aovs, motion=True, history_length=True)
        t = [torch.from_numpy(x).cuda() for x in (a, b, aovs["albedo_w"], aovs["normal_w"], aovs["nearest"].view(np.int64))]
        out = torch.full_like(t[0], float("nan"))
        mo = torch.full((g.height, g.width, 2), float("nan"), device="cuda")
        hl = torch.full((g.height, g.width), 7, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            g.denoise_temporal_device(hist_d, *(x.data_ptr() for x in t), out.data_ptr(), mo.data_ptr(), hl.data_ptr(), stream=st.cuda_stream)
        st.synchronize()
        assert out.cpu().numpy().tobytes() == want[0].tobytes()
        assert mo.cpu().numpy().tobytes() == want[1].tobytes()
        assert hl.cpu().numpy().view(np.uint32).tobytes() == want[2].tobytes()


def test_error_cases_leave_the_history_as_it_was():
    b = partial_wall()
    g, other = api.Scene(b.finish()), api.Scene(b.finish())
    g.update_frame()
    other.update_frame()
    hist, twin = api.DenoiseHistory(g), api.DenoiseHistory(g)
    rng = np.random.default_rng(2)
    a, bb, aovs = synthetic(rng, g.height, g.width, specials=False)
    aovs["nearest"] &= ~np.uint64(0xffffffff)  # the wall, instance 0: the same frame twice accumulates
    for h in (hist, twin):
        g.denoise_temporal(h, a, bb, aovs)
    with pytest.raises(api.TrbError) as e:  # a history of another scene
        other.denoise_temporal(hist, a, bb, aovs)
    assert e.value.status == F.TRB_INVALID_ARG
    with pytest.raises(api.TrbError) as e:  # bad parameters
        g.denoise_temporal(hist, a, bb, aovs, max_history=0)
    assert e.value.status == F.TRB_INVALID_ARG
    with pytest.raises(api.TrbError):  # an output on top of an input
        g.denoise_temporal(hist, a, bb, aovs, out=a)
    x = g.denoise_temporal(hist, a, bb, aovs, motion=True, history_length=True)
    y = g.denoise_temporal(twin, a, bb, aovs, motion=True, history_length=True)
    assert all(p.tobytes() == q.tobytes() for p, q in zip(x, y))
    assert x[2].max() == 2
    b.film = dict(b.film, width=48, height=40)  # another film size: refused until reset
    g.replace_settings(b.film)
    g.update_frame()
    a3, b3, aovs3 = synthetic(rng, 40, 48, specials=False)
    with pytest.raises(api.TrbError) as e:
        g.denoise_temporal(hist, a3, b3, aovs3)
    assert e.value.status == F.TRB_INVALID_ARG and "film size" in str(e.value)
    hist.reset()
    assert g.denoise_temporal(hist, a3, b3, aovs3).tobytes() == g.denoise(a3, b3, aovs3).tobytes()


def test_tray_denoise_temporal_writes_what_render_denoised_temporal_computes(tmp_path):
    import os
    import sys
    H.build_programs()
    sys.path.insert(0, os.path.join(H.REPO, "tests", "golden"))
    import make_scenes
    merl = os.path.join(H.SCENES, "merl", "synthetic.binary")  # c5_tr15_like's measured material, generated where needed
    if not os.path.exists(merl):
        make_scenes.write_synthetic_merl(merl)
    out = tmp_path / "frames"
    p = H.Proc([H.TRAY, H.C5, "--denoise-temporal", "--spp", "2", "-o", str(out), "--seed", "7", "--start-frame", "0", "--end-frame", "2"])
    try:
        rc, _, err = p.finish(timeout=600)
    finally:
        p.kill()
    assert rc == 0, err
    d = H.load_desc(H.C5, 0, 0, 2)
    g = api.Scene(d.contents)
    hist = api.DenoiseHistory(g)
    for k in range(3):
        den, _, _, _ = g.render_denoised_temporal(hist, seed=7, current_frame=k)
        got = H.read_png(out / ("frame%05d.png" % k))
        diff = np.abs(got.astype(int) - g.to_srgb8(den).astype(int))
        assert diff.max() <= 1 and np.count_nonzero(diff) < 1e-3 * diff.size, (k, diff.max())
    g.close()


# ---- quality ----------------------------------------------------------------------------------------------------------------------

def test_quality_on_a_static_c1_sequence():
    g = api.Scene(json_desc("c1_cornell_box.json", 256, 256, 2))
    g.update_frame()
    ref, _ = g.render(spp=1024, seed=99, flags=F.RENDER_NO_UPDATE)
    hist = api.DenoiseHistory(g)
    temporal, spatial = [], []
    for k in range(16):
        a, b, aovs = halves(g, spp=2, seed=1 + k, flags=F.RENDER_NO_UPDATE)
        temporal.append(g.denoise_temporal(hist, a, b, aovs))
        spatial.append(g.denoise(a, b, aovs))
    flick = lambda xs: float(np.mean([np.abs(xs[k][..., :3] - xs[k - 1][..., :3]).mean() for k in range(8, 16)]))  # noqa: E731
    r = dict(rmse_t=rmse(temporal[-1], ref), rmse_s=rmse(spatial[-1], ref), flicker_t=flick(temporal), flicker_s=flick(spatial))
    print("c1 static 16 frames at 2 spp", r)
    assert r["rmse_t"] < r["rmse_s"], r
    assert r["flicker_t"] < r["flicker_s"], r


def keyframed_quality_rows():
    desc = SB.scene_animated(256, 256, 2).finish()
    g = api.Scene(desc)
    hist = api.DenoiseHistory(g)
    rows = []
    for k in range(4):
        g.update_frame(*frame_times(k))
        ref, aov_ref, _ = g.render_aov(spp=256, seed=99, albedo=False, normal=False, flags=F.RENDER_NO_UPDATE)
        inst = (aov_ref["nearest"] & np.uint64(0xffffffff)).astype(np.uint32)
        moving = np.isin(inst, [5, 6, 7])  # the flying sphere, the spinning mesh and the glass sphere (after the five walls)
        a, b, aovs = halves(g, spp=2, seed=1 + k, flags=F.RENDER_NO_UPDATE)
        t = g.denoise_temporal(hist, a, b, aovs)
        s = g.denoise(a, b, aovs)
        rows.append(dict(frame=k, t=rmse(t, ref), s=rmse(s, ref), t_moving=rmse(t, ref, moving), s_moving=rmse(s, ref, moving),
                         moving=float(moving.mean())))
    print("scene_animated 256x256 2 spp", rows)
    g.close()
    return rows


def test_quality_on_the_keyframed_scene_without_ghosting():
    for r in keyframed_quality_rows()[1:]:
        assert r["moving"] > 0 and r["t_moving"] <= 1.1 * r["s_moving"], r


# Measured on an H100: mean RMSE over frames 1-3 of 0.0284 temporal against 0.0185 spatial. The keyframed scene's area light moves and
# changes colour and its point light moves, so the shading of the static walls changes under their history, which lags behind it; the
# history has no test for a change of shading (SVGF's temporal gradients are not built).
@pytest.mark.xfail(strict=True, reason="the history lags behind the keyframed scene's changing lights: 0.0284 temporal against 0.0185 spatial")
def test_quality_on_the_keyframed_scene_is_lower_on_average():
    rows = keyframed_quality_rows()[1:]
    assert np.mean([r["t"] for r in rows]) < np.mean([r["s"] for r in rows]), rows
