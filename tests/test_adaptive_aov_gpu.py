"""AOVs of Adaptive renders on an H100 (k_wf_aov_ad between the round-0 trace and shade of every Adaptive pass, the colour film's
ADAPT kernel over the records, k_wf_nearest_ad, and k_ad_aov_slots for the parity layout): every taken slot's AOV record equals the
Adaptive AOV oracle's bit for bit, samples, pixel counts and counters equal render_samples_adaptive's, the films equal film writes of
the taken slots' records, the device form equals the host form, and render_denoised_adaptive is the moment denoiser over
render_adaptive_aov's outputs."""
import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_adaptive_aov.pyadaptiveaov import AdaptiveAovOracleScene
from test_adaptive_aov_cpu import _pixel_counts, _taken
from test_aov_gpu import FILM_TOL, SCENES, partial_wall
from test_denoise_gpu import rmse
from test_queries_gpu import json_desc

pytestmark = pytest.mark.gpu
COUNTERS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation", "node_tests", "tri_tests", "inst_tests"]
REF = F.RENDER_STATS | F.RENDER_REFERENCE_SHADOW  # the oracle's shadow rays, so its counters compare


def counters(st):
    return [getattr(st, k) for k in COUNTERS]


def scene(name):
    desc, frame = SCENES[name]()
    g = api.Scene(desc)
    g.update_frame(*frame)
    return g, desc, frame


def check_records(g, o, mn, mx, **kw):
    samples, aov, spp, st = g.render_samples_adaptive_aov(mn, mx, flags=REF, **kw)
    plain, pspp, pst = g.render_samples_adaptive(mn, mx, flags=REF, **kw)
    assert samples.tobytes() == plain.tobytes() and (spp == pspp).all() and counters(st) == counters(pst)
    osamples, oaov, ospp, ost = o.render_samples_adaptive_aov(mn, mx, **kw)
    assert (spp == ospp).all() and samples.tobytes() == osamples.tobytes() and counters(st) == counters(ost)
    assert aov.tobytes() == oaov.tobytes(), "AOV records differ in %d slots" % int((aov.view(np.uint8).reshape(-1, 32) !=
                                                                                   oaov.view(np.uint8).reshape(-1, 32)).any(1).sum())
    assert (aov["inst"] != F.MISS).any() and (spp > mn).any()


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_records_equal_the_oracle(name, split):
    g, desc, frame = scene(name)
    o = AdaptiveAovOracleScene(desc)
    o.update_frame(*frame)
    g.set_option("shade.split", split)
    check_records(g, o, 2, 16, seed=7)


def test_c4_wide_leaves_on_block_ranges():
    desc = SB.scene_c4(1_000_000, 256, 128, 2).finish()
    g, o = api.Scene(desc), AdaptiveAovOracleScene(desc)
    g.update_frame(); o.update_frame()
    g.set_option("trace.wide_leaf", 1)
    nb = g.n_blocks()
    for start, count in ((0, 64), (nb - 64, 64)):
        check_records(g, o, 2, 16, seed=3, block_start=start, block_count=count)


def regions_and_pixels(g, spp, mpp, **kw):
    """per record of the (block, pixel, slot) layout: the film region (by * width / 8 + bx) and the pixel (y * width + x)"""
    xy = g.block_list(kw.get("block_start", 0), kw.get("block_count", 0)).astype(np.int64)
    k = np.arange(64)
    region = np.repeat(xy[:, 1] * (g.width // 8) + xy[:, 0], 64 * mpp)
    pixel = ((xy[:, 1:2] * 8 + k // 8) * g.width + xy[:, 0:1] * 8 + k % 8).reshape(-1).repeat(mpp)
    return region, pixel


def expected_aovs(g, mn, mx, **kw):
    """film_write of the taken slots' records, and np.minimum.at of their nearest keys"""
    samples, aov, spp, _ = g.render_samples_adaptive_aov(mn, mx, **kw)
    mpp = api.adaptive_schedule(mn, mx)[3]
    taken = _taken(_pixel_counts(g, spp, **kw), mpp)
    region, pixel = regions_and_pixels(g, spp, mpp, **kw)
    films = {}
    for key, field in (("albedo_w", "albedo"), ("normal_w", "n")):
        s = samples[taken].copy()
        s["r"], s["g"], s["b"] = aov[field][taken, 0], aov[field][taken, 1], aov[field][taken, 2]
        films[key] = g.film_write(s, region[taken].astype(np.uint32))
    key = (aov["depth"].view(np.uint32).astype(np.uint64) << np.uint64(32)) | aov["inst"].astype(np.uint64)
    near = np.full(g.width * g.height, np.iinfo(np.uint64).max, np.uint64)
    np.minimum.at(near, pixel[taken], key[taken])
    films["nearest"] = near.reshape(g.height, g.width)
    return films, spp


@pytest.mark.parametrize("name", ["c1", "zoo", "keyframed_f1", "partial"])
def test_films_equal_film_writes_of_the_taken_records(name):
    g, _, _ = scene(name)
    kw = dict(seed=11, flags=F.RENDER_STATS | F.RENDER_NO_UPDATE)
    film, aovs, spp, st = g.render_adaptive_aov(2, 16, **kw)
    ref, rspp, rst = g.render_adaptive(2, 16, **kw)
    np.testing.assert_allclose(film, ref, **FILM_TOL)
    assert (spp == rspp).all() and counters(st) == counters(rst)
    want, wspp = expected_aovs(g, 2, 16, seed=11)
    assert (wspp == spp).all()
    for k in ("albedo_w", "normal_w"):
        np.testing.assert_allclose(aovs[k], want[k], **FILM_TOL)
        np.testing.assert_allclose(aovs[k][..., 3], film[..., 3], **FILM_TOL)
    assert np.array_equal(aovs["nearest"], want["nearest"])


def test_block_ranges_and_small_passes_change_only_the_addition_order():
    g = api.Scene(SB.scene_smallpt_like(128, 128, 16).finish())
    g.update_frame()
    kw = dict(seed=4, flags=F.RENDER_NO_UPDATE)
    full, aovs, spp, st = g.render_adaptive_aov(2, 32, **kw)
    assert (spp > 2).any()
    g.set_option("pass.paths", 64 * 32 * 3)  # a few blocks per pass
    again, aovs2, spp2, st2 = g.render_adaptive_aov(2, 32, **kw)
    g.set_option("pass.paths", 1 << 24)
    assert (spp == spp2).all() and counters(st)[:5] == counters(st2)[:5]
    nb = g.n_blocks()
    half, haovs, s0, _ = g.render_adaptive_aov(2, 32, block_start=0, block_count=nb // 2, **kw)
    _, _, s1, _ = g.render_adaptive_aov(2, 32, half, albedo=haovs["albedo_w"], normal=haovs["normal_w"], nearest=haovs["nearest"],
                                        block_start=nb // 2, block_count=nb - nb // 2, **kw)
    assert (s0 + s1 == spp).all()
    for f, a in ((again, aovs2), (half, haovs)):
        np.testing.assert_allclose(f, full, **FILM_TOL)
        for k in ("albedo_w", "normal_w"):
            np.testing.assert_allclose(a[k], aovs[k], **FILM_TOL)
        assert np.array_equal(a["nearest"], aovs["nearest"])


# ---- the device form ---------------------------------------------------------------------------------------------------------
class DeviceOut:
    """torch buffers of one device render: film, albedo_w, normal_w (h, w, 4) f32, nearest (h, w) all ones, pixel counts, stats"""

    def __init__(self, g, stream):
        import torch
        dev = "cuda:%d" % g.device
        self.film, self.albedo, self.normal = (torch.zeros((g.height, g.width, 4), dtype=torch.float32, device=dev) for _ in range(3))
        self.nearest = torch.full((g.height, g.width), -1, dtype=torch.int64, device=dev)
        self.spp = torch.zeros((g.height, g.width), dtype=torch.int32, device=dev)
        self.stats = torch.zeros(9, dtype=torch.int64, device=dev)
        stream.wait_stream(torch.cuda.current_stream(self.film.device))  # the buffers are filled on the current stream

    def render(self, g, mn, mx, stream, skip=(), **kw):
        p = {k: (None if k in skip else getattr(self, k).data_ptr()) for k in ("albedo", "normal", "nearest")}
        g.render_adaptive_aov_device(mn, mx, self.film.data_ptr(), p["albedo"], p["normal"], p["nearest"], self.spp.data_ptr(),
                                     self.stats.data_ptr(), stream.cuda_stream, **kw)

    def host(self):
        st = F.Stats.from_buffer_copy(self.stats.cpu().numpy().tobytes())
        aovs = {"albedo_w": self.albedo.cpu().numpy(), "normal_w": self.normal.cpu().numpy(), "nearest": self.nearest.cpu().numpy().view(np.uint64)}
        return self.film.cpu().numpy(), aovs, self.spp.cpu().numpy().view(np.uint32), st


def test_device_form_equals_the_host_form_returns_at_once_and_takes_null_outputs():
    import torch
    g, _, _ = scene("zoo")
    kw = dict(seed=9, flags=F.RENDER_STATS | F.RENDER_NO_UPDATE)
    film, aovs, spp, st = g.render_adaptive_aov(2, 16, **kw)
    s = torch.cuda.Stream()
    warm = DeviceOut(g, s)
    warm.render(g, 2, 16, s, **kw)  # first use may allocate (and so synchronise)
    s.synchronize()
    out = DeviceOut(g, s)
    with torch.cuda.stream(s):
        torch.cuda._sleep(2_000_000_000)  # about a second of GPU time ahead of the render
    out.render(g, 2, 16, s, **kw)
    assert not s.query(), "the call waited for its stream"
    s.synchronize()
    for d in (warm, out):
        dfilm, daovs, dspp, dst = d.host()
        np.testing.assert_allclose(dfilm, film, **FILM_TOL)
        assert (dspp == spp).all() and counters(dst) == counters(st)
        for k in ("albedo_w", "normal_w"):
            np.testing.assert_allclose(daovs[k], aovs[k], **FILM_TOL)
        assert np.array_equal(daovs["nearest"], aovs["nearest"])
    for skip in ("albedo", "normal", "nearest"):
        d = DeviceOut(g, s)
        d.render(g, 2, 16, s, skip=(skip,), **kw)
        s.synchronize()
        dfilm, daovs, dspp, _ = d.host()
        np.testing.assert_allclose(dfilm, film, **FILM_TOL)
        assert (dspp == spp).all()
        for k, name in (("albedo_w", "albedo"), ("normal_w", "normal")):
            if name == skip:
                assert not daovs[k].any()
            else:
                np.testing.assert_allclose(daovs[k], aovs[k], **FILM_TOL)
        assert np.array_equal(daovs["nearest"], np.full_like(aovs["nearest"], np.iinfo(np.uint64).max) if skip == "nearest" else aovs["nearest"])


def test_error_statuses():
    import torch
    g = api.Scene(SB.scene_materials_zoo(16, 16, 4).finish())
    g.update_frame()
    t = torch.zeros(16 * 16 * 4 + 4, dtype=torch.float32, device="cuda")
    n = torch.zeros(16 * 16 + 1, dtype=torch.int64, device="cuda")
    calls = (lambda **kw: g.render_adaptive_aov(2, 8, **kw), lambda **kw: g.render_samples_adaptive_aov(2, 8, **kw),
             lambda **kw: g.render_adaptive_aov_device(2, 8, t.data_ptr(), t.data_ptr(), None, n.data_ptr(), **kw))
    for call in calls:
        for kw, status in ((dict(spp=4), F.TRB_INVALID_ARG), (dict(sample_first=1), F.TRB_INVALID_ARG), (dict(sample_count=2), F.TRB_INVALID_ARG),
                           (dict(flags=F.RENDER_MEGAKERNEL), F.TRB_UNSUPPORTED)):
            with pytest.raises(api.TrbError) as e:
                call(**kw)
            assert e.value.status == status, kw
    with pytest.raises(api.TrbError) as e:
        g.render_adaptive_aov(8, 4)
    assert e.value.status == F.TRB_INVALID_ARG
    for bad in (dict(d_film=t.data_ptr() + 4), dict(d_albedo=t.data_ptr() + 4), dict(d_normal=t.data_ptr() + 8), dict(d_nearest=n.data_ptr() + 4)):
        args = dict(d_film=t.data_ptr(), d_albedo=None, d_normal=None, d_nearest=None)
        args.update(bad)
        with pytest.raises(api.TrbError) as e:
            g.render_adaptive_aov_device(2, 8, **args)
        assert e.value.status == F.TRB_INVALID_ARG, bad
    for integ in ((F.INTEGRATOR_WHITTED, 0, 4), (F.INTEGRATOR_NORMALS_DEBUG, 0, 0)):
        w = api.Scene(partial_wall(integ).finish())
        w.update_frame()
        for call in (lambda: w.render_adaptive_aov(2, 8), lambda: w.render_samples_adaptive_aov(2, 8),
                     lambda: w.render_adaptive_aov_device(2, 8, t.data_ptr())):
            with pytest.raises(api.TrbError) as e:
                call()
            assert e.value.status == F.TRB_UNSUPPORTED, integ
    torch.cuda.synchronize()


# ---- denoising ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gradients", [False, True])
def test_render_denoised_adaptive_is_the_moment_call_on_the_adaptive_outputs(gradients):
    g, _, _ = scene("c1")
    hist, twin = api.DenoiseHistory(g), api.DenoiseHistory(g)
    for k in range(3):
        den, film, aovs, spp, st = g.render_denoised_adaptive(hist, 2, 16, seed=5, current_frame=0, denoise=dict(iterations=3),
                                                              gradients=gradients, flags=F.RENDER_NO_UPDATE)
        assert int(spp.sum()) == st.camera_samples
        if gradients:
            want = g.denoise_moments_gradient(twin, film, aovs, 5, iterations=3)
        else:
            want = g.denoise_moments(twin, film, aovs, iterations=3)
        assert den.tobytes() == want.tobytes(), k


# Measured on an H100 80GB HBM3 (700 W): RMSE 0.0445 denoised against 0.1092 noisy, Adaptive (2, 32) on C1 at 256x256.
def test_single_image_quality_on_c1():
    g = api.Scene(json_desc("c1_cornell_box.json", 256, 256, 1))
    g.update_frame()
    ref, _ = g.render(spp=1024, seed=99, flags=F.RENDER_NO_UPDATE)
    den, film, _, spp, _ = g.render_denoised_adaptive(api.DenoiseHistory(g), 2, 32, seed=1, denoise={"max_history": 1}, flags=F.RENDER_NO_UPDATE)
    r = dict(denoised=rmse(den, ref), noisy=rmse(film, ref), mean_spp=float(spp.mean()))
    print("c1 256x256 Adaptive (2, 32)", r)
    assert r["denoised"] < r["noisy"], r


def test_history_over_four_static_frames():
    g = api.Scene(json_desc("c1_cornell_box.json", 64, 64, 1))
    g.update_frame()
    hist = api.DenoiseHistory(g)
    for k in range(4):
        (_, hl), _, _, _, _ = g.render_denoised_adaptive(hist, 2, 8, seed=1, current_frame=k, denoise={"history_length": True},
                                                         flags=F.RENDER_NO_UPDATE)
        assert hl.max() == k + 1, (k, hl.max())
    assert (hl == 4).mean() > 0.9


def test_tray_adaptive_denoise_moments_writes_what_render_denoised_adaptive_computes(tmp_path):
    H.build_programs()
    out = tmp_path / "frames"
    p = H.Proc([H.TRAY, H.CORNELL, "--adaptive", "2", "16", "--denoise-moments", "-o", str(out), "--seed", "7"])
    try:
        rc, _, err = p.finish(timeout=600)
    finally:
        p.kill()
    assert rc == 0, err
    d = H.load_desc(H.CORNELL)
    g = api.Scene(d.contents)
    den, _, _, _, _ = g.render_denoised_adaptive(api.DenoiseHistory(g), 2, 16, seed=7, current_frame=0)
    got = H.read_png(out / "frame00000.png")
    # the films are summed with float atomics, whose order can move a last bit and so, rarely, one 8-bit level
    diff = np.abs(got.astype(int) - g.to_srgb8(den).astype(int))
    assert diff.max() <= 1 and np.count_nonzero(diff) < 1e-3 * diff.size, diff.max()
    g.close()
