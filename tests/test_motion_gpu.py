"""Motion vectors on an H100 (k_wf_motion / k_wf_motion_ad next to k_wf_aov, then the colour film's kernel over the records): every
camera sample's record equals the motion oracle's bit for bit (C1, C2, the keyframed scene at frames 1 and 2 with and without an
animated fov, C4's million triangles with wide leaves); the colour film, AOV records, nearest, lum_w, pixel counts and counters are those of the
calls without motion; motion_w equals trb_film_write of the records (LowDiscrepancy and Adaptive); the device form on a side stream
equals the host form; the statuses; and decode_motion agrees with the temporal denoiser's reprojection on a camera arc."""
import numpy as np
import pytest
import torch

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_motion import pymotion as PM
from test_adaptive_aov_cpu import _pixel_counts, _taken
from test_adaptive_aov_gpu import regions_and_pixels
from test_aov_gpu import FILM_TOL
from test_denoise_gpu import halves
from test_queries_gpu import json_desc

pytestmark = pytest.mark.gpu
COUNTERS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation", "node_tests", "tri_tests", "inst_tests"]


def counters(st):
    return [getattr(st, k) for k in COUNTERS]


def _shutter0(b):
    b.cameras[0] = b.cameras[0][:3] + (0.0,) + b.cameras[0][4:]
    return b


PARITY = {
    "c1": lambda: (json_desc("c1_cornell_box.json", 32, 24, 2), (0, 0.0, 0.0), -0.25, {}),
    "c2": lambda: (json_desc("c2_smallpt.json", 32, 32, 2), (0, 0.0, 0.0), -0.25, {}),
    "animated_f1": lambda: (SB.scene_animated(32, 32, 4).finish(), (1, 0.25, 0.5), None, {}),
    "animated_f2": lambda: (SB.scene_animated(32, 32, 4).finish(), (2, 0.5, 0.75), None, {}),
    "animated_fov_f2": lambda: (SB.scene_animated(32, 32, 4, animated_fov=True).finish(), (2, 0.5, 0.75), None, {}),
    "animated_fov_f1_forward": lambda: (SB.scene_animated(32, 32, 4, animated_fov=True).finish(), (1, 0.25, 0.5), 0.25, {}),
    "c4_wide_leaf": lambda: (SB.scene_c4(1_000_000, 384, 216, 1).finish(), (0, 0.0, 0.0), -0.25, {"trace.wide_leaf": 1}),
}


@pytest.mark.parametrize("name", sorted(PARITY))
def test_records_equal_the_oracle_bit_for_bit_and_leave_the_aov_call_as_it_is(name):
    desc, frame, dt, options = PARITY[name]()
    g = api.Scene(desc)
    for k, v in options.items():
        g.set_option(k, v)
    g.update_frame(*frame)
    o = PM.MotionOracleScene(desc)
    o.update_frame(*frame)
    kw = dict(seed=7, flags=F.RENDER_STATS)
    motion = True if dt is None else dt
    s, a, m, st = g.render_samples_aov(motion=motion, **kw)
    s0, a0, st0 = g.render_samples_aov(**kw)
    assert s.tobytes() == s0.tobytes() and a.tobytes() == a0.tobytes() and counters(st) == counters(st0)
    want = o.motion_samples(dt=dt, **{k: v for k, v in kw.items() if k != "flags"})
    bad = np.argwhere(m.view(np.uint32).reshape(-1, 4) != want.view(np.uint32).reshape(-1, 4))
    assert m.tobytes() == want.tobytes(), (name, bad[:5], m[bad[:5, 0]], want[bad[:5, 0]])
    assert (m["valid"] == 1).sum() > 0.3 * len(m) and (m["reserved"] == 0).all()
    if name.startswith("animated"):
        assert np.abs(m["dx"]).max() > 0.1


@pytest.mark.parametrize("v2", [0, 1])
@pytest.mark.parametrize("name", ["c1", "animated_f1"])
def test_motion_film_equals_a_film_write_of_the_records_and_the_rest_is_unchanged(name, v2):
    desc, frame, dt, _ = PARITY[name]()
    g = api.Scene(desc)
    g.set_option("film.v2", v2)
    g.update_frame(*frame)
    motion = True if dt is None else dt
    kw = dict(seed=11, spp=4, flags=F.RENDER_STATS | F.RENDER_NO_UPDATE)
    film, aovs, st = g.render_aov(lum=True, motion=motion, **kw)
    ref, raovs, rst = g.render_aov(lum=True, **kw)
    np.testing.assert_allclose(film, ref, **FILM_TOL)
    for k in ("albedo_w", "normal_w", "lum_w"):
        np.testing.assert_allclose(aovs[k], raovs[k], **FILM_TOL)
    assert np.array_equal(aovs["nearest"], raovs["nearest"]) and counters(st) == counters(rst)
    # lum_w may be NULL
    film2, aovs2, st2 = g.render_aov(motion=motion, **kw)
    np.testing.assert_allclose(film2, ref, **FILM_TOL)
    np.testing.assert_allclose(aovs2["motion_w"], aovs["motion_w"], **FILM_TOL)
    assert "lum_w" not in aovs2 and counters(st2) == counters(rst)
    # the film of the records
    s, _, m, _ = g.render_samples_aov(motion=motion, seed=11, spp=4)
    s["r"], s["g"], s["b"] = m["valid"] * m["dx"], m["valid"] * m["dy"], m["valid"]
    want = g.film_write(s, g.sample_regions(seed=11, spp=4))
    np.testing.assert_allclose(aovs["motion_w"], want, rtol=1e-4, atol=1e-5 * max(1.0, float(np.abs(want).max())))
    np.testing.assert_allclose(aovs["motion_w"][..., 3], film[..., 3], **FILM_TOL)
    dm = api.decode_motion(aovs["motion_w"])
    assert dm.shape == (g.height, g.width, 2) and np.isfinite(dm).any()


def test_the_device_form_on_a_side_stream_equals_the_host_form():
    g = api.Scene(SB.scene_animated(64, 64, 8).finish())
    g.update_frame(1, 0.25, 0.5)
    h, w = g.height, g.width
    kw = dict(seed=4, flags=F.RENDER_NO_UPDATE)
    film, aovs, _ = g.render_aov(lum=True, motion=True, **kw)
    for with_lum in (True, False):
        d_film, d_alb, d_nrm, d_lum, d_mo = (torch.zeros((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(5))
        d_near = torch.full((h, w), -1, dtype=torch.int64, device="cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            g.render_aov_device(d_film.data_ptr(), d_alb.data_ptr(), d_nrm.data_ptr(), d_near.data_ptr(), stream=s.cuda_stream,
                                d_lum=d_lum.data_ptr() if with_lum else None, d_motion=d_mo.data_ptr(), **kw)
        s.synchronize()
        np.testing.assert_allclose(d_film.cpu().numpy(), film, **FILM_TOL)
        np.testing.assert_allclose(d_mo.cpu().numpy(), aovs["motion_w"], **FILM_TOL)
        assert np.array_equal(d_near.cpu().numpy().view(np.uint64), aovs["nearest"])
        if with_lum:
            np.testing.assert_allclose(d_lum.cpu().numpy(), aovs["lum_w"], **FILM_TOL)
        else:
            assert not d_lum.any()
    # the Adaptive device form against its host form
    film, aovs, spp, _ = g.render_adaptive_aov(2, 16, motion=True, **kw)
    d_film, d_mo = (torch.zeros((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(2))
    d_spp = torch.zeros((h, w), dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g.render_adaptive_aov_device(2, 16, d_film.data_ptr(), d_pixel_spp=d_spp.data_ptr(), stream=s.cuda_stream, d_motion=d_mo.data_ptr(), **kw)
    s.synchronize()
    np.testing.assert_allclose(d_film.cpu().numpy(), film, **FILM_TOL)
    np.testing.assert_allclose(d_mo.cpu().numpy(), aovs["motion_w"], **FILM_TOL)
    assert np.array_equal(d_spp.cpu().numpy().view(np.uint32), spp)


def test_adaptive_motion_film_equals_a_film_write_of_the_slots_it_took():
    b = _shutter0(SB.scene_animated(32, 32, 4))  # shutter 0: a slot's motion depends on its raster position only
    desc = b.finish()
    g = api.Scene(desc)
    g.update_frame(1, 0.25, 0.5)
    o = PM.MotionOracleScene(desc)
    o.update_frame(1, 0.25, 0.5)
    kw = dict(seed=5, flags=F.RENDER_STATS | F.RENDER_NO_UPDATE)
    film, aovs, spp, st = g.render_adaptive_aov(2, 16, lum=True, motion=True, **kw)
    ref, raovs, rspp, rst = g.render_adaptive_aov(2, 16, lum=True, **kw)
    np.testing.assert_allclose(film, ref, **FILM_TOL)
    for k in ("albedo_w", "normal_w", "lum_w"):
        np.testing.assert_allclose(aovs[k], raovs[k], **FILM_TOL)
    assert np.array_equal(spp, rspp) and np.array_equal(aovs["nearest"], raovs["nearest"]) and counters(st) == counters(rst)
    samples, _, sspp, _ = g.render_samples_adaptive_aov(2, 16, seed=5)
    assert np.array_equal(sspp, spp)
    mpp = api.adaptive_schedule(2, 16)[3]
    taken = _taken(_pixel_counts(g, spp, seed=5), mpp)
    region, _ = regions_and_pixels(g, spp, mpp, seed=5)
    s = samples[taken].copy()
    m = o.motion_at(s["x"], s["y"], 0.0)
    s["r"], s["g"], s["b"] = m["valid"] * m["dx"], m["valid"] * m["dy"], m["valid"]
    want = g.film_write(s, region[taken].astype(np.uint32))
    assert np.abs(m["dx"]).max() > 0.1
    np.testing.assert_allclose(aovs["motion_w"], want, rtol=1e-4, atol=1e-5 * max(1.0, float(np.abs(want).max())))


def test_statuses():
    g = api.Scene(SB.scene_animated(16, 16, 2).finish())
    g.update_frame(1, 0.25, 0.5)
    for bad in (float("nan"), float("inf"), -float("inf")):
        for call in (lambda: g.render_aov(motion=bad), lambda: g.render_adaptive_aov(2, 8, motion=bad),
                     lambda: g.render_samples_aov(motion=bad)):
            with pytest.raises(api.TrbError) as e:
                call()
            assert e.value.status == F.TRB_INVALID_ARG and "dt" in str(e.value)
    buf = torch.zeros(16 * 16 * 4 + 16, dtype=torch.float32, device="cuda")
    film = torch.zeros((16, 16, 4), dtype=torch.float32, device="cuda")
    for call in (lambda p: g.render_aov_device(film.data_ptr(), d_motion=p, flags=F.RENDER_NO_UPDATE),
                 lambda p: g.render_adaptive_aov_device(2, 8, film.data_ptr(), d_motion=p, flags=F.RENDER_NO_UPDATE)):
        with pytest.raises(api.TrbError) as e:
            call(buf.data_ptr() + 4)  # misaligned
        assert e.value.status == F.TRB_INVALID_ARG
    for call in (lambda: g.render_aov_device(film.data_ptr(), d_motion=buf.data_ptr(), motion_dt=float("nan"), flags=F.RENDER_NO_UPDATE),
                 lambda: g.render_adaptive_aov_device(2, 8, film.data_ptr(), d_motion=buf.data_ptr(), motion_dt=float("nan"), flags=F.RENDER_NO_UPDATE)):
        with pytest.raises(api.TrbError) as e:
            call()
        assert e.value.status == F.TRB_INVALID_ARG
    torch.cuda.synchronize()
    with pytest.raises(api.TrbError) as e:
        g.render_aov(motion=True, flags=F.RENDER_MEGAKERNEL)
    assert e.value.status == F.TRB_UNSUPPORTED
    for integ in (F.INTEGRATOR_WHITTED, F.INTEGRATOR_NORMALS_DEBUG):
        b = SB.scene_animated(16, 16, 2)
        b.integrator = (integ, 2, 6)
        w = api.Scene(b.finish())
        w.update_frame(1, 0.25, 0.5)
        for call in (lambda: w.render_aov(motion=True, flags=F.RENDER_NO_UPDATE), lambda: w.render_samples_aov(motion=True),
                     lambda: w.render_adaptive_aov(2, 8, motion=True, flags=F.RENDER_NO_UPDATE)):
            with pytest.raises(api.TrbError) as e:
                call()
            assert e.value.status == F.TRB_UNSUPPORTED


def camera_arc(frames=8):
    """a plastic square and a sphere in front of a camera on a keyframed arc (translation and a turn about y); shutter 0"""
    b = SB.SceneBuilder(96, 64, 4, 1, 2)
    b.film.update(frames=frames, start_frame=0, end_frame=frames - 1, scene_time=1.0)
    m = b.add_material(F.MAT_PLASTIC, c0=(0.2, 0.4, 0.6), c1=(0.5, 0.5, 0.5), roughness=0.1)
    b.receiver(F.SHAPE_RECT, m, [SB.trs(t=(0, 0, 2))], p0=14.0, p1=10.0)
    b.receiver(F.SHAPE_SPHERE, m, [SB.trs(t=(1.0, 0.5, -1.0))], p0=1.5)
    b.point_light([SB.trs(t=(0, 2, -6))], (1, 1, 1, 40))
    arc = SB.Anim([SB.trs(t=(-1.0, 0.0, -10.0), q=SB.quat_axis_angle((0, 1, 0), 4.0)), SB.trs(t=(0.0, 0.3, -10.3)),
                   SB.trs(t=(1.0, 0.5, -10.0), q=SB.quat_axis_angle((0, 1, 0), -4.0))], degree=2)
    b.add_camera([arc], fov=40.0, shutter_size=0.0)
    return b


def test_decode_motion_agrees_with_the_temporal_denoisers_reprojection_on_a_camera_arc():
    g = api.Scene(camera_arc().finish())
    step = g.frame_step()
    hist = api.DenoiseHistory(g)
    k = 3
    g.update_frame(k - 1, (k - 1) * step, k * step)
    a, b, aovs = halves(g, spp=4, seed=1, flags=F.RENDER_NO_UPDATE)
    g.denoise_temporal(hist, a, b, aovs)
    g.update_frame(k, k * step, (k + 1) * step)
    a, b, aovs = halves(g, spp=4, seed=2, flags=F.RENDER_NO_UPDATE)
    _, dn_motion, _ = g.denoise_temporal(hist, a, b, aovs, motion=True, history_length=True)
    _, maovs, _ = g.render_aov(motion=True, spp=16, seed=3, flags=F.RENDER_NO_UPDATE)
    mv = api.decode_motion(maovs["motion_w"])
    # pixels whose 5x5 neighbourhood (the Mitchell filter's reach of 2 px) is one instance, with both motions defined
    inst = api.decode_nearest(aovs["nearest"])[1].astype(np.int64)
    h, w = inst.shape
    pad = np.pad(inst, 2, constant_values=-1)
    one = np.ones((h, w), bool)
    spread = np.zeros((h, w))
    mpad = np.pad(dn_motion, ((2, 2), (2, 2), (0, 0)), constant_values=np.nan)
    for dy in range(5):
        for dx in range(5):
            one &= pad[dy:dy + h, dx:dx + w] == inst
            with np.errstate(invalid="ignore"):
                spread = np.fmax(spread, np.abs(mpad[dy:dy + h, dx:dx + w] - dn_motion).max(-1))
    sel = one & (inst != 0xffffffff) & np.isfinite(dn_motion).all(-1) & np.isfinite(mv).all(-1)
    assert sel.sum() > 0.3 * h * w
    # Both are previous minus current. motion_w is the filter-weighted mean of per-sample motions within 2 px of the pixel centre, the
    # denoiser's is one pixel-centre value at the pixel's nearest depth: they differ by at most the variation of the motion field over
    # that reach, weighted by the filter's sum |w| / sum w (below 1.5 for Mitchell-Netravali 1/3, 1/3), plus float32 rounding.
    tol = 1.5 * spread + 1e-3
    err = np.abs(mv - dn_motion).max(-1)
    print("motion vs denoiser: max |motion| %.3f px, max error %.4f px, max tolerance %.4f px, median error %.2e px"
          % (np.abs(dn_motion[sel]).max(), err[sel].max(), tol[sel].max(), np.median(err[sel])))
    assert np.abs(dn_motion[sel]).max() > 1.0
    assert (err[sel] <= tol[sel]).all()
