"""The temporal gradients on an H100 (k_gr_project, k_gr_resolve, the re-shade illumination, k_gr_delta, k_gr_atrous, then
k_dn_temporal_grad and the a-trous iterations, then k_gr_record, the ray queries, the record illumination and k_gr_store): every
frame's output, motion, history length and lambda equal the oracle's orc_denoise_temporal_gradient bit for bit; with nothing changing
lambda is 0 and the output is trb_denoise_temporal's; a light dimmed between frames drops the history; on the keyframed scene the
gradient output beats the spatial filter; the device form on a side stream equals the host form; the error cases leave the history as
it was; and trb_tray --denoise-temporal --temporal-gradients writes what render_denoised_temporal(gradients=True) computes."""
import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_gradient import pygradient as G
from test_denoise_gpu import halves, rmse
from test_denoise_temporal_gpu import SEQ, frame_times
from test_queries_gpu import json_desc

pytestmark = pytest.mark.gpu


def run_sequence(desc, frames, seed=3, split=None, spp=2, **params):
    """Render frames as halves (seed + frame), denoise them with the library and the oracle; assert the four outputs bit for bit"""
    g, o = api.Scene(desc), G.Scene(desc)
    if split is not None:
        g.set_option("shade.split", split)
    hist, oh = api.DenoiseHistory(g), G.History()
    lams, lens = [], []
    for k in frames:
        g.update_frame(*frame_times(k))
        o.update_frame(*frame_times(k))
        a, b, aovs = halves(g, spp=spp, seed=seed + k, flags=F.RENDER_NO_UPDATE)
        got = g.denoise_temporal_gradient(hist, a, b, aovs, seed + k, motion=True, history_length=True, lam=True, **params)
        want = G.denoise_temporal_gradient(o, oh, a, b, aovs, seed + k, **params)
        for x, y, name in zip(got, want, ("rgbw", "motion", "history_length", "lambda")):
            assert x.tobytes() == y.tobytes(), (k, name, np.argwhere(x.view(np.uint32) != y.view(np.uint32))[:5])
        lens.append(got[2])
        lams.append(got[3])
    g.close()
    return lens, lams


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("name", sorted(SEQ))
def test_sequences_equal_the_oracle(name, split):
    lens, lams = run_sequence(SEQ[name](), range(5), split=split)
    assert lens[-1].max() > 1 and not lams[0].any()


@pytest.mark.parametrize("params", [dict(gradient_iterations=0), dict(gradient_iterations=6, max_history=3)])
def test_gradient_parameters_equal_the_oracle(params):
    lens, lams = run_sequence(SEQ["animated"](), range(3), **params)
    assert max(float(x.max()) for x in lams) > 0


@pytest.mark.parametrize("times", ["one_frame", "frame_times"])
def test_nothing_changing_gives_lambda_zero_and_the_plain_output(times):
    g = api.Scene(json_desc("c1_cornell_box.json", 48, 32, 2))
    hg, hp = api.DenoiseHistory(g), api.DenoiseHistory(g)
    if times == "one_frame":
        g.update_frame()
    for k in range(8):
        if times == "frame_times":
            g.update_frame(*frame_times(k))
        a, b, aovs = halves(g, spp=2, seed=1 + k, flags=F.RENDER_NO_UPDATE)
        got = g.denoise_temporal_gradient(hg, a, b, aovs, 1 + k, motion=True, history_length=True, lam=True)
        want = g.denoise_temporal(hp, a, b, aovs, motion=True, history_length=True)
        assert not got[3].any(), k
        for x, y in zip(got[:3], want):
            assert x.tobytes() == y.tobytes(), k
    assert got[2].max() == 8
    g.close()


def test_first_call_reset_plain_call_and_max_history_1():
    g = api.Scene(SB.scene_animated(48, 32, 2).finish())
    hg, hp = api.DenoiseHistory(g), api.DenoiseHistory(g)
    frames = []
    for k in range(3):
        g.update_frame(*frame_times(k))
        frames.append(halves(g, seed=k, flags=F.RENDER_NO_UPDATE))
        a, b, aovs = frames[-1]
        got = g.denoise_temporal_gradient(hg, a, b, aovs, k, lam=True)
        plain = g.denoise_temporal(hp, a, b, aovs)
        if k == 0:  # the first call has no gradients
            assert got[0].tobytes() == plain.tobytes() and not got[1].any()
        one = g.denoise_temporal_gradient(api.DenoiseHistory(g), a, b, aovs, k, max_history=1)
        assert one.tobytes() == g.denoise(a, b, aovs).tobytes()
    a, b, aovs = frames[-1]
    hg.reset()
    hp.reset()
    got = g.denoise_temporal_gradient(hg, a, b, aovs, 9, lam=True)
    assert got[0].tobytes() == g.denoise_temporal(hp, a, b, aovs).tobytes() and not got[1].any()  # after reset
    g.denoise_temporal(hg, a, b, aovs)  # a plain call invalidates the records
    g.denoise_temporal(hp, a, b, aovs)
    got = g.denoise_temporal_gradient(hg, a, b, aovs, 10, lam=True)
    assert got[0].tobytes() == g.denoise_temporal(hp, a, b, aovs).tobytes() and not got[1].any()
    g.close()


def test_a_dimmed_light_drops_the_history():
    desc = json_desc("c1_cornell_box.json", 128, 128, 2)
    key = np.array([(tuple(desc.color_keys[0].rgba), desc.color_keys[0].time)], F.COLOR_KEY_DTYPE)
    g = api.Scene(desc)
    g.update_frame()
    hg, hp = api.DenoiseHistory(g), api.DenoiseHistory(g)
    for k in range(6):
        a, b, aovs = halves(g, spp=2, seed=1 + k, flags=F.RENDER_NO_UPDATE)
        g.denoise_temporal_gradient(hg, a, b, aovs, 1 + k)
        g.denoise_temporal(hp, a, b, aovs)
    key["rgba"] *= np.float32(0.1)
    g.update_color_keys(0, key)
    g.update_frame()
    ref, _ = g.render(spp=1024, seed=99, flags=F.RENDER_NO_UPDATE)
    a, b, aovs = halves(g, spp=2, seed=50, flags=F.RENDER_NO_UPDATE)
    got, _, hl, lam = g.denoise_temporal_gradient(hg, a, b, aovs, 50, motion=True, history_length=True, lam=True)
    plain, hl_p = g.denoise_temporal(hp, a, b, aovs, history_length=True)
    had = hl_p > 1  # valid pixels with a history
    r = dict(short=float((hl[had] <= 2).mean()), plain_long=float((hl_p[had] > 2).mean()), lam_mean=float(lam[had].mean()),
             rmse_g=rmse(got, ref), rmse_p=rmse(plain, ref))
    print("c1 light x0.1", r)
    assert had.sum() > 1000
    assert r["short"] >= 0.9 and r["plain_long"] >= 0.9, r
    assert r["rmse_g"] < r["rmse_p"], r
    g.close()


def test_device_form_on_a_side_stream_equals_the_host_form():
    import torch
    desc = SB.scene_animated(48, 32, 2).finish()
    g = api.Scene(desc)
    hist_h, hist_d = api.DenoiseHistory(g), api.DenoiseHistory(g)
    st = torch.cuda.Stream()
    for k in range(4):
        g.update_frame(*frame_times(k))
        a, b, aovs = halves(g, seed=k, flags=F.RENDER_NO_UPDATE)
        want = g.denoise_temporal_gradient(hist_h, a, b, aovs, k, motion=True, history_length=True, lam=True)
        t = [torch.from_numpy(x).cuda() for x in (a, b, aovs["albedo_w"], aovs["normal_w"], aovs["nearest"].view(np.int64))]
        out = torch.full_like(t[0], float("nan"))
        mo = torch.full((g.height, g.width, 2), float("nan"), device="cuda")
        hl = torch.full((g.height, g.width), 7, dtype=torch.int32, device="cuda")
        lam = torch.full((g.height, g.width), float("nan"), device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            g.denoise_temporal_gradient_device(hist_d, *(x.data_ptr() for x in t), k, out.data_ptr(), mo.data_ptr(), hl.data_ptr(),
                                               lam.data_ptr(), stream=st.cuda_stream)
        st.synchronize()
        assert out.cpu().numpy().tobytes() == want[0].tobytes()
        assert mo.cpu().numpy().tobytes() == want[1].tobytes()
        assert hl.cpu().numpy().view(np.uint32).tobytes() == want[2].tobytes()
        assert lam.cpu().numpy().tobytes() == want[3].tobytes()
    g.close()


def test_error_cases_leave_the_history_as_it_was():
    g = api.Scene(SB.scene_animated(48, 32, 2).finish())
    other = api.Scene(SB.scene_animated(48, 32, 2).finish())
    other.update_frame()
    hist, twin = api.DenoiseHistory(g), api.DenoiseHistory(g)
    frames = []
    for k in range(2):
        g.update_frame(*frame_times(k))
        frames.append(halves(g, seed=k, flags=F.RENDER_NO_UPDATE))
        for h in (hist, twin):
            g.denoise_temporal_gradient(h, *frames[-1], k)
    g.update_frame(*frame_times(2))
    a, bb, aovs = halves(g, seed=2, flags=F.RENDER_NO_UPDATE)
    with pytest.raises(api.TrbError) as e:  # a history of another scene
        other.denoise_temporal_gradient(hist, a, bb, aovs, 2)
    assert e.value.status == F.TRB_INVALID_ARG
    for bad in (dict(gradient_iterations=7), dict(max_history=0)):
        with pytest.raises(api.TrbError) as e:
            g.denoise_temporal_gradient(hist, a, bb, aovs, 2, **bad)
        assert e.value.status == F.TRB_INVALID_ARG
    with pytest.raises(api.TrbError):  # an output on top of an input
        g.denoise_temporal_gradient(hist, a, bb, aovs, 2, out=a)
    x = g.denoise_temporal_gradient(hist, a, bb, aovs, 2, motion=True, history_length=True, lam=True)
    y = g.denoise_temporal_gradient(twin, a, bb, aovs, 2, motion=True, history_length=True, lam=True)
    assert all(p.tobytes() == q.tobytes() for p, q in zip(x, y))
    g.close()
    other.close()


def test_tray_temporal_gradients_writes_what_render_denoised_temporal_computes(tmp_path):
    import os
    import sys
    H.build_programs()
    sys.path.insert(0, os.path.join(H.REPO, "tests", "golden"))
    import make_scenes
    merl = os.path.join(H.SCENES, "merl", "synthetic.binary")
    if not os.path.exists(merl):
        make_scenes.write_synthetic_merl(merl)
    out = tmp_path / "frames"
    p = H.Proc([H.TRAY, H.C5, "--denoise-temporal", "--temporal-gradients", "--spp", "2", "-o", str(out), "--seed", "7",
                "--start-frame", "0", "--end-frame", "2"])
    try:
        rc, _, err = p.finish(timeout=600)
    finally:
        p.kill()
    assert rc == 0, err
    d = H.load_desc(H.C5, 0, 0, 2)
    g = api.Scene(d.contents)
    hist = api.DenoiseHistory(g)
    for k in range(3):
        den, _, _, _ = g.render_denoised_temporal(hist, seed=7, current_frame=k, gradients=True)
        got = H.read_png(out / ("frame%05d.png" % k))
        diff = np.abs(got.astype(int) - g.to_srgb8(den).astype(int))
        assert diff.max() <= 1 and np.count_nonzero(diff) < 1e-3 * diff.size, (k, diff.max())
    g.close()


# ---- quality ----------------------------------------------------------------------------------------------------------------------

def keyframed_quality_rows():
    """test_denoise_temporal_gpu.keyframed_quality_rows' setup with the gradient call beside the plain one"""
    desc = SB.scene_animated(256, 256, 2).finish()
    g = api.Scene(desc)
    hg, hp = api.DenoiseHistory(g), api.DenoiseHistory(g)
    rows = []
    for k in range(4):
        g.update_frame(*frame_times(k))
        ref, aov_ref, _ = g.render_aov(spp=256, seed=99, albedo=False, normal=False, flags=F.RENDER_NO_UPDATE)
        inst = (aov_ref["nearest"] & np.uint64(0xffffffff)).astype(np.uint32)
        moving = np.isin(inst, [5, 6, 7])
        a, b, aovs = halves(g, spp=2, seed=1 + k, flags=F.RENDER_NO_UPDATE)
        gr = g.denoise_temporal_gradient(hg, a, b, aovs, 1 + k)
        t = g.denoise_temporal(hp, a, b, aovs)
        s = g.denoise(a, b, aovs)
        rows.append(dict(frame=k, g=rmse(gr, ref), t=rmse(t, ref), s=rmse(s, ref), g_moving=rmse(gr, ref, moving),
                         s_moving=rmse(s, ref, moving)))
    print("scene_animated 256x256 2 spp", rows)
    g.close()
    return rows


def test_quality_on_the_keyframed_scene():
    rows = keyframed_quality_rows()[1:]
    assert np.mean([r["g"] for r in rows]) < np.mean([r["s"] for r in rows]), rows
    for r in rows:
        assert r["g_moving"] <= 1.1 * r["s_moving"], r


def test_quality_on_c1_with_an_orbiting_camera():
    desc = json_desc("c1_cornell_box.json", 256, 256, 2)
    g = api.Scene(desc)
    cam_idx = 0  # the camera's keyframe comes first
    base = desc.keyframes[cam_idx]
    t0 = np.array(base.translation, np.float64)
    hg, hp = api.DenoiseHistory(g), api.DenoiseHistory(g)
    for k in range(16):
        ang = np.radians(1.5 * k)
        t = t0 + np.array([60 * np.sin(ang), 0.0, 60 * (1 - np.cos(ang))])
        key = np.array([(tuple(t), tuple(base.rotation), tuple(base.scaling))], F.KEYFRAME_DTYPE)
        g.update_keyframes(cam_idx, key)
        g.update_frame()
        a, b, aovs = halves(g, spp=2, seed=1 + k, flags=F.RENDER_NO_UPDATE)
        gr = g.denoise_temporal_gradient(hg, a, b, aovs, 1 + k)
        pl = g.denoise_temporal(hp, a, b, aovs)
    s = g.denoise(a, b, aovs)
    ref, _ = g.render(spp=256, seed=99, flags=F.RENDER_NO_UPDATE)
    r = dict(g=rmse(gr, ref), t=rmse(pl, ref), s=rmse(s, ref))
    print("c1 camera arc 16 frames at 2 spp", r)
    assert r["g"] <= 1.1 * r["t"] and r["g"] < r["s"], r
    g.close()
