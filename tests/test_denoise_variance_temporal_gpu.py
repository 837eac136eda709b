"""The variance temporal denoiser on an H100 (k_dn_temporal_variance, or the gradient steps around k_dn_temporal_variance_grad, then
the a-trous iterations): every frame's output, motion, history length, variance and lambda equal the oracle's bit for bit over
LowDiscrepancy and Adaptive sequences, a static C1, C1 on a camera arc and the keyframed scene; the device form on a side stream
equals the host form; an empty history and max_history 1 are trb_denoise_variance; a gradient call on an unchanged scene is the plain
call; the history families; the error cases; the variance shrinks with the history as its recursion predicts; the quality against
the single-frame call; a dimmed light drops the history; trb_tray --denoise-variance-temporal writes what
render_denoised_variance_temporal computes."""
import numpy as np
import pytest
import torch

import cli_helpers as H
from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_variance_temporal import pyvariancetemporal as VT
from test_aov_gpu import partial_wall
from test_denoise_cpu import synthetic
from test_denoise_gpu import halves, rmse
from test_denoise_temporal_gpu import frame_times
from test_denoise_variance_cpu import _lum_film
from test_queries_gpu import json_desc

pytestmark = pytest.mark.gpu
OUTS = ("rgbw", "motion", "history_length", "variance", "lambda")


def render(g, seed, spp=2, adaptive=None):
    """One render of the current frame with the AOVs and the lum_w film: (film, aovs)"""
    if adaptive:
        film, aovs, _, _ = g.render_adaptive_aov(adaptive[0], adaptive[1], lum=True, seed=seed, flags=F.RENDER_NO_UPDATE)
    else:
        film, aovs, _ = g.render_aov(spp=spp, lum=True, seed=seed, flags=F.RENDER_NO_UPDATE)
    return film, aovs


def _arc_key(base, k):
    t = np.array(base.translation, np.float64)
    ang = np.radians(1.5 * k)
    t = t + np.array([60 * np.sin(ang), 0.0, 60 * (1 - np.cos(ang))])
    return np.array([(tuple(t), tuple(base.rotation), tuple(base.scaling))], F.KEYFRAME_DTYPE)


def run_sequence(desc, frames, seed=3, spp=2, adaptive=None, gradients=False, arc=False, **params):
    """Render frames once (seed + frame), denoise them with the library and the oracle; assert every output bit for bit. arc: the
    camera (keyframe 0) moves along an arc, set with update_keyframes on the library's scene and in a fresh oracle scene per frame."""
    g = api.Scene(desc)
    o = None if arc else VT.Scene(desc)
    hist, oh = api.DenoiseHistory(g), VT.History()
    base = desc.keyframes[0]
    base = type(base).from_buffer_copy(base)
    lens = []
    for k in frames:
        if arc:
            key = _arc_key(base, k)
            g.update_keyframes(0, key)
            kf = desc.keyframes[0]
            for i in range(3):
                kf.translation[i] = float(key["translation"][0][i])
            o = VT.Scene(desc)
            g.update_frame()
            o.update_frame()
        else:
            g.update_frame(*frame_times(k))
            o.update_frame(*frame_times(k))
        film, aovs = render(g, seed + k, spp, adaptive)
        if gradients:
            got = g.denoise_variance_temporal_gradient(hist, film, aovs, seed + k, motion=True, history_length=True, variance=True, lam=True,
                                                       **params)
            want = VT.denoise_variance_temporal_gradient(o, oh, film, aovs, seed + k, **params)
        else:
            got = g.denoise_variance_temporal(hist, film, aovs, motion=True, history_length=True, variance=True, **params)
            want = VT.denoise_variance_temporal(o, oh, film, aovs, **params)
        for x, y, name in zip(got, want, OUTS):
            assert x.tobytes() == y.tobytes(), (k, name, np.argwhere(x.view(np.uint32) != y.view(np.uint32))[:5])
        lens.append(got[2])
    g.close()
    return lens


CASES = {
    "c1_static": lambda: dict(desc=json_desc("c1_cornell_box.json", 48, 32, 2)),
    "c1_arc": lambda: dict(desc=json_desc("c1_cornell_box.json", 48, 32, 2), arc=True),
    "animated": lambda: dict(desc=SB.scene_animated(48, 32, 2).finish()),
    "animated_4spp": lambda: dict(desc=SB.scene_animated(48, 32, 4).finish(), spp=4, max_history=3, iterations=2),
    "adaptive_c1": lambda: dict(desc=json_desc("c1_cornell_box.json", 48, 32, 2), adaptive=(2, 8)),
    "adaptive_animated": lambda: dict(desc=SB.scene_animated(48, 32, 2).finish(), adaptive=(2, 8)),
    "gradient_animated": lambda: dict(desc=SB.scene_animated(48, 32, 2).finish(), gradients=True),
    "gradient_c1": lambda: dict(desc=json_desc("c1_cornell_box.json", 48, 32, 2), gradients=True, gradient_iterations=0),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_sequences_equal_the_oracle(name):
    kw = CASES[name]()
    lens = run_sequence(kw.pop("desc"), range(5), **kw)
    assert lens[-1].max() > 1


def test_device_form_on_a_side_stream_equals_the_host_form():
    g = api.Scene(SB.scene_animated(48, 32, 2).finish())
    hists = {gr: (api.DenoiseHistory(g), api.DenoiseHistory(g)) for gr in (False, True)}
    st = torch.cuda.Stream()
    for k in range(4):
        g.update_frame(*frame_times(k))
        film, aovs = render(g, k, adaptive=(2, 8) if k % 2 else None)
        t = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (film, aovs["albedo_w"], aovs["normal_w"], aovs["nearest"].view(np.int64),
                                                                          aovs["lum_w"])]
        for gr, (hh, hd) in hists.items():
            if gr:
                want = g.denoise_variance_temporal_gradient(hh, film, aovs, k, motion=True, history_length=True, variance=True, lam=True)
            else:
                want = g.denoise_variance_temporal(hh, film, aovs, motion=True, history_length=True, variance=True)
            out = torch.full_like(t[0], float("nan"))
            mo = torch.full((g.height, g.width, 2), float("nan"), device="cuda")
            hl = torch.full((g.height, g.width), 7, dtype=torch.int32, device="cuda")
            var = torch.full((g.height, g.width), -1.0, device="cuda")
            lam = torch.full((g.height, g.width), -1.0, device="cuda")
            torch.cuda.synchronize()
            with torch.cuda.stream(st):
                if gr:
                    g.denoise_variance_temporal_gradient_device(hd, *(x.data_ptr() for x in t), k, out.data_ptr(), mo.data_ptr(), hl.data_ptr(),
                                                                var.data_ptr(), lam.data_ptr(), stream=st.cuda_stream)
                else:
                    g.denoise_variance_temporal_device(hd, *(x.data_ptr() for x in t), out.data_ptr(), mo.data_ptr(), hl.data_ptr(),
                                                       var.data_ptr(), stream=st.cuda_stream)
            st.synchronize()
            got = [out.cpu().numpy(), mo.cpu().numpy(), hl.cpu().numpy().view(np.uint32), var.cpu().numpy(), lam.cpu().numpy()]
            for x, y, name in zip(got, want, OUTS):
                assert x.tobytes() == y.tobytes(), (k, gr, name)
    assert want[2].max() > 1
    with pytest.raises(api.TrbError) as e:  # misaligned lum_w
        g.denoise_variance_temporal_device(hd, *(x.data_ptr() for x in t[:4]), t[4].data_ptr() + 4, out.data_ptr())
    assert e.value.status == F.TRB_INVALID_ARG
    with pytest.raises(api.TrbError) as e:
        g.denoise_variance_temporal_gradient_device(hd, *(x.data_ptr() for x in t[:4]), t[4].data_ptr() + 8, 1, out.data_ptr())
    assert e.value.status == F.TRB_INVALID_ARG
    with pytest.raises(api.TrbError) as e:  # misaligned colour, variance
        g.denoise_variance_temporal_device(hd, t[0].data_ptr() + 4, *(x.data_ptr() for x in t[1:]), out.data_ptr())
    assert e.value.status == F.TRB_INVALID_ARG
    with pytest.raises(api.TrbError) as e:
        g.denoise_variance_temporal_device(hd, *(x.data_ptr() for x in t), out.data_ptr(), None, None, var.data_ptr() + 2)
    assert e.value.status == F.TRB_INVALID_ARG
    g.close()


def test_an_empty_history_and_max_history_1_are_trb_denoise_variance():
    g = api.Scene(SB.scene_animated(48, 32, 2).finish())
    hist = api.DenoiseHistory(g)
    for k in range(3):
        g.update_frame(*frame_times(k))
        for adaptive in (None, (2, 8)):
            film, aovs = render(g, 10 + k, adaptive=adaptive)
            want = g.denoise_variance(film, aovs, variance=True)
            fresh = g.denoise_variance_temporal(api.DenoiseHistory(g), film, aovs, variance=True)
            one = g.denoise_variance_temporal(hist, film, aovs, variance=True, history_length=True, max_history=1)
            assert fresh[0].tobytes() == want[0].tobytes() and fresh[1].tobytes() == want[1].tobytes(), k
            assert one[0].tobytes() == want[0].tobytes() and one[2].tobytes() == want[1].tobytes(), k
            assert one[1].max() == 1
            g.update_frame(*frame_times(k))  # the Adaptive render of the same frame next
    g.close()


@pytest.mark.parametrize("adaptive", [None, (2, 8)])
def test_a_gradient_call_on_an_unchanged_scene_is_the_plain_call(adaptive):
    g = api.Scene(json_desc("c1_cornell_box.json", 64, 48, 2))
    g.update_frame()
    hg, hp = api.DenoiseHistory(g), api.DenoiseHistory(g)
    for k in range(5):
        film, aovs = render(g, 1 + k, adaptive=adaptive)
        got = g.denoise_variance_temporal_gradient(hg, film, aovs, 1 + k, motion=True, history_length=True, variance=True, lam=True)
        want = g.denoise_variance_temporal(hp, film, aovs, motion=True, history_length=True, variance=True)
        assert not got[4].any(), k
        assert all(x.tobytes() == y.tobytes() for x, y in zip(got[:4], want)), k
    assert want[2].max() == 5
    g.close()


def test_history_families():
    """A moment call and a half-film call after a variance call find no history, a variance call after either finds none, and a
    gradient call after a plain variance call has lambda 0"""
    g = api.Scene(json_desc("c1_cornell_box.json", 48, 32, 2))
    g.update_frame()
    film, aovs = render(g, 1)
    a, b, aovs2 = halves(g, spp=2, seed=1, flags=F.RENDER_NO_UPDATE)

    def variance_pair(h):
        return (g.denoise_variance_temporal(h, film, aovs, history_length=True, variance=True),
                g.denoise_variance_temporal(api.DenoiseHistory(g), film, aovs, history_length=True, variance=True))

    h = api.DenoiseHistory(g)
    for _ in range(2):
        g.denoise_variance_temporal(h, film, aovs)
    m = g.denoise_moments(h, film, aovs, history_length=True)
    assert m[1].max() == 1 and m[0].tobytes() == g.denoise_moments(api.DenoiseHistory(g), film, aovs).tobytes()
    got, fresh = variance_pair(h)  # after a moment call
    assert got[1].max() == 1 and all(x.tobytes() == y.tobytes() for x, y in zip(got, fresh))
    g.denoise_variance_temporal(h, film, aovs)
    t = g.denoise_temporal(h, a, b, aovs2, history_length=True)
    assert t[1].max() == 1 and t[0].tobytes() == g.denoise_temporal(api.DenoiseHistory(g), a, b, aovs2).tobytes()
    got, fresh = variance_pair(h)  # after a half-film call
    assert got[1].max() == 1 and all(x.tobytes() == y.tobytes() for x, y in zip(got, fresh))
    # a gradient call after a plain variance call: records invalid, lambda 0, the history kept
    g.denoise_variance_temporal_gradient(h, film, aovs, 5)
    g.denoise_variance_temporal(h, film, aovs)
    gr = g.denoise_variance_temporal_gradient(h, film, aovs, 6, history_length=True, lam=True)
    assert not gr[2].any() and gr[1].max() == 4
    # a moment gradient call after a variance gradient call: another family, no history
    mg = g.denoise_moments_gradient(h, film, aovs, 7, history_length=True, lam=True)
    assert mg[1].max() == 1 and not mg[2].any()
    g.close()


def test_error_cases_leave_the_history_as_it_was():
    b = partial_wall()
    g, other = api.Scene(b.finish()), api.Scene(b.finish())
    g.update_frame()
    other.update_frame()
    hist, twin = api.DenoiseHistory(g), api.DenoiseHistory(g)
    rng = np.random.default_rng(2)
    a, _, aovs = synthetic(rng, g.height, g.width, specials=False)
    aovs["nearest"] &= ~np.uint64(0xffffffff)  # the wall, instance 0: the same frame twice accumulates
    aovs["lum_w"] = _lum_film(rng, a, False)
    for h in (hist, twin):
        g.denoise_variance_temporal(h, a, aovs)
    with pytest.raises(api.TrbError) as e:  # a history of another scene
        other.denoise_variance_temporal(hist, a, aovs)
    assert e.value.status == F.TRB_INVALID_ARG
    for bad in (dict(max_history=0), dict(depth_tolerance=-1.0), dict(iterations=11)):
        with pytest.raises(api.TrbError) as e:
            g.denoise_variance_temporal(hist, a, aovs, **bad)
        assert e.value.status == F.TRB_INVALID_ARG
    with pytest.raises(api.TrbError) as e:
        g.denoise_variance_temporal_gradient(hist, a, aovs, 2, gradient_iterations=7)
    assert e.value.status == F.TRB_INVALID_ARG
    with pytest.raises(api.TrbError):  # an output on top of an input
        g.denoise_variance_temporal(hist, a, aovs, out=a)
    with pytest.raises(api.TrbError):  # an output on top of lum_w
        g.denoise_variance_temporal(hist, a, aovs, out=aovs["lum_w"])
    with pytest.raises(api.TrbError) as e:  # lambda on top of lum_w
        g.denoise_variance_temporal_gradient(hist, a, aovs, 2, lam=aovs["lum_w"].reshape(-1)[: g.height * g.width].reshape(g.height, g.width))
    assert "lambda" in str(e.value)
    x = g.denoise_variance_temporal(hist, a, aovs, motion=True, history_length=True, variance=True)
    y = g.denoise_variance_temporal(twin, a, aovs, motion=True, history_length=True, variance=True)
    assert all(p.tobytes() == q.tobytes() for p, q in zip(x, y))
    assert x[2].max() == 2
    b.film = dict(b.film, width=48, height=40)  # another film size: refused until reset
    g.replace_settings(b.film)
    g.update_frame()
    a3, _, aovs3 = synthetic(rng, 40, 48, specials=False)
    aovs3["lum_w"] = _lum_film(rng, a3, False)
    with pytest.raises(api.TrbError) as e:
        g.denoise_variance_temporal(hist, a3, aovs3)
    assert e.value.status == F.TRB_INVALID_ARG and "film size" in str(e.value)
    hist.reset()
    assert g.denoise_variance_temporal(hist, a3, aovs3).tobytes() == g.denoise_variance_temporal(api.DenoiseHistory(g), a3, aovs3).tobytes()
    g.close()
    other.close()


# ---- semantics and quality on C1 ------------------------------------------------------------------------------------------------

def test_the_variance_shrinks_with_the_history_as_its_recursion_predicts():
    """16 frames of a static C1 at 2 spp, max_history 8: V averages 1/k to frame 8, then blends by 1/8, so V_16 / v_f is about
    sum_{j<9} (1/64) (7/8)^(2j) + (7/8)^18 / 8 = 0.074 for v_f the same every frame"""
    g = api.Scene(json_desc("c1_cornell_box.json", 256, 256, 2))
    g.update_frame()
    hist = api.DenoiseHistory(g)
    for k in range(16):
        film, aovs = render(g, 1 + k)
        _, hl, V = g.denoise_variance_temporal(hist, film, aovs, history_length=True, variance=True)
    _, v = g.denoise_variance(film, aovs, variance=True)
    both = np.isfinite(V) & np.isfinite(v) & (hl == 8)
    ratio = V[both].astype(np.float64).mean() / v[both].astype(np.float64).mean()
    print("c1 256x256 2 spp frame 16: mean V / mean v_f", ratio, "pixels", int(both.sum()))
    assert both.mean() > 0.5
    assert 0.05 <= ratio <= 0.11, ratio
    g.close()


def _clamped(x):
    return np.clip(x[..., :3] / np.maximum(x[..., 3:], 1e-12), 0, 1)


@pytest.mark.parametrize("adaptive", [None, (2, 8)])
def test_quality_against_the_single_frame_call(adaptive):
    g = api.Scene(json_desc("c1_cornell_box.json", 128, 128, 2))
    g.update_frame()
    ref, _ = g.render(spp=1024, seed=99, flags=F.RENDER_NO_UPDATE)
    hist = api.DenoiseHistory(g)
    t, s = [], []
    for k in range(16):
        film, aovs = render(g, 1 + k, adaptive=adaptive)
        t.append(_clamped(g.denoise_variance_temporal(hist, film, aovs)))
        s.append(_clamped(g.denoise_variance(film, aovs)))
    flick = lambda seq: float(np.mean([np.abs(seq[k] - seq[k - 1]).mean() for k in range(8, 16)]))  # noqa: E731
    r = dict(rmse_t=rmse(t[-1], ref), rmse_s=rmse(s[-1], ref), flicker_t=flick(t), flicker_s=flick(s))
    print("c1 128x128 static", adaptive or "2 spp", r)
    assert r["rmse_t"] < r["rmse_s"] and r["flicker_t"] < r["flicker_s"], r
    g.close()


def test_a_dimmed_light_drops_the_history():
    desc = json_desc("c1_cornell_box.json", 128, 128, 2)
    key = np.array([(tuple(desc.color_keys[0].rgba), desc.color_keys[0].time)], F.COLOR_KEY_DTYPE)
    g = api.Scene(desc)
    g.update_frame()
    hg, hp = api.DenoiseHistory(g), api.DenoiseHistory(g)
    for k in range(6):
        film, aovs = render(g, 1 + k)
        g.denoise_variance_temporal_gradient(hg, film, aovs, 1 + k)
        g.denoise_variance_temporal(hp, film, aovs)
    key["rgba"] *= np.float32(0.1)
    g.update_color_keys(0, key)
    g.update_frame()
    ref, _ = g.render(spp=1024, seed=99, flags=F.RENDER_NO_UPDATE)
    film, aovs = render(g, 50)
    got, hl, lam = g.denoise_variance_temporal_gradient(hg, film, aovs, 50, history_length=True, lam=True)
    plain, hl_p = g.denoise_variance_temporal(hp, film, aovs, history_length=True)
    had = hl_p > 1
    r = dict(short=float((hl[had] <= 2).mean()), lam_mean=float(lam[had].mean()), rmse_g=rmse(got, ref), rmse_p=rmse(plain, ref))
    print("c1 light x0.1 at 2 spp", r)
    assert had.sum() > 1000
    assert r["short"] >= 0.99, r
    assert r["rmse_g"] < 0.5 * r["rmse_p"], r
    g.close()


# ---- trb_tray ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("extra", [["--spp", "2"], ["--adaptive", "2", "8"], ["--spp", "2", "--variance-gradients"],
                                   ["--adaptive", "2", "8", "--variance-gradients"]])
def test_tray_denoise_variance_temporal_writes_what_render_denoised_variance_temporal_computes(tmp_path, extra):
    H.build_programs()
    out = tmp_path / "frames"
    p = H.Proc([H.TRAY, H.CORNELL, "--denoise-variance-temporal", "-o", str(out), "--seed", "7", "--start-frame", "0", "--end-frame", "2"]
               + extra)
    try:
        rc, _, err = p.finish(timeout=600)
    finally:
        p.kill()
    assert rc == 0, err
    adaptive = "--adaptive" in extra
    d = H.load_desc(H.CORNELL, 0, 0, 0 if adaptive else 2)
    g = api.Scene(d.contents)
    hist = api.DenoiseHistory(g)
    for k in range(3):
        den = g.render_denoised_variance_temporal(hist, spp=0 if adaptive else 2, adaptive=(2, 8) if adaptive else None, seed=7,
                                                  current_frame=k, gradients="--variance-gradients" in extra)[0]
        got = H.read_png(out / ("frame%05d.png" % k))
        diff = np.abs(got.astype(int) - g.to_srgb8(den).astype(int))
        assert diff.max() <= 1 and np.count_nonzero(diff) < 1e-3 * diff.size, (k, diff.max())
    g.close()
