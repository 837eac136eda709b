"""The denoiser on an H100 (k_dn_prepare, then k_dn_atrous once per iteration): the output equals the oracle's orc_denoise bit for bit
on the same input arrays, rendered as two half-sample AOV renders of the AOV scenes (split and fused shading), of a block-range
render, of C4 at 1920x1080, and on synthetic films with NaN, +-inf, negative colours and zero weights; the host and device forms
agree; the scratch follows replace_settings; the denoised image is closer to a 1024-spp reference than the noisy one; trb_tray
--denoise writes what Scene.render_denoised computes."""
import os

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_denoise import pydenoise as D
from test_aov_gpu import SCENES, partial_wall
from test_denoise_cpu import synthetic
from test_queries_gpu import json_desc
from test_textures import textured_zoo

pytestmark = pytest.mark.gpu


def halves(g, spp=4, **kw):
    """samples [0, spp/2) and [spp/2, spp) into two films, the AOVs over both (what Scene.render_denoised renders)"""
    a, aovs, _ = g.render_aov(spp=spp, sample_first=0, sample_count=spp // 2, **kw)
    b, _, _ = g.render_aov(albedo=aovs["albedo_w"], normal=aovs["normal_w"], nearest=aovs["nearest"], spp=spp, sample_first=spp // 2,
                           sample_count=spp // 2, **kw)
    return a, b, aovs


def assert_bit_exact(g, a, b, aovs, **params):
    got = g.denoise(a, b, aovs, **params)
    want = D.denoise(a, b, aovs, **params)
    assert got.tobytes() == want.tobytes(), np.argwhere(got.view(np.uint32) != want.view(np.uint32))[:5]
    return got


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_aov_scenes_equal_the_oracle(name, split):
    desc, frame = SCENES[name]()
    g = api.Scene(desc)
    g.update_frame(*frame)
    g.set_option("shade.split", split)
    a, b, aovs = halves(g, seed=7, flags=F.RENDER_NO_UPDATE)
    out = assert_bit_exact(g, a, b, aovs)
    assert (out[..., 3] == 1).all() and np.isfinite(out).all()
    assert not np.array_equal(out[..., :3], ((a + b)[..., :3] / (a + b)[..., 3:]))  # the filter did something


@pytest.mark.parametrize("params", [dict(iterations=0), dict(iterations=1), dict(iterations=5), dict(iterations=10),
                                    dict(iterations=3, normal_power=1, sigma_luminance=0.5, sigma_depth=8.0),
                                    dict(iterations=4, normal_power=1024, sigma_luminance=40.0, sigma_depth=0.05)])
def test_c1_iterations_and_parameters_equal_the_oracle(params):
    g = api.Scene(json_desc("c1_cornell_box.json", 64, 48, 4))
    g.update_frame()
    a, b, aovs = halves(g, seed=3, flags=F.RENDER_NO_UPDATE)
    assert_bit_exact(g, a, b, aovs, **params)


def test_block_range_render_leaves_zero_pixels_and_equals_the_oracle():
    g = api.Scene(json_desc("c1_cornell_box.json", 64, 48, 4))
    g.update_frame()
    a, b, aovs = halves(g, seed=5, block_start=7, block_count=20, flags=F.RENDER_NO_UPDATE)
    empty = (a[..., 3] + b[..., 3]) <= 0
    assert empty.any() and (~empty).any()
    out = assert_bit_exact(g, a, b, aovs)
    assert not out[empty].any()


def test_c4_1080p_2spp_equals_the_oracle():
    g = api.Scene(SB.scene_c4(1_000_000, 1920, 1080, 2).finish())
    g.update_frame()
    a, b, aovs = halves(g, spp=2, seed=1, flags=F.RENDER_NO_UPDATE)
    assert_bit_exact(g, a, b, aovs)


@pytest.mark.parametrize("iterations", [0, 1, 5, 10])
def test_synthetic_films_with_specials_equal_the_oracle(iterations):
    g = api.Scene(partial_wall().finish())
    rng = np.random.default_rng(100 + iterations)
    a, b, aovs = synthetic(rng, g.height, g.width)
    out = assert_bit_exact(g, a, b, aovs, iterations=iterations, normal_power=32, sigma_luminance=2.0)
    assert np.isnan(out).any() and np.isinf(out).any() and (out[..., 3] == 0).any()


def test_device_form_on_a_torch_side_stream_equals_the_host_form():
    import torch
    desc, frame = SCENES["zoo"]()
    g = api.Scene(desc)
    g.update_frame(*frame)
    a, b, aovs = halves(g, seed=4, flags=F.RENDER_NO_UPDATE)
    for params in (dict(), dict(iterations=0), dict(iterations=2, normal_power=4)):
        want = g.denoise(a, b, aovs, **params)
        t = [torch.from_numpy(x).cuda() for x in (a, b, aovs["albedo_w"], aovs["normal_w"], aovs["nearest"].view(np.int64))]
        out = torch.full_like(t[0], float("nan"))
        torch.cuda.synchronize()
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            g.denoise_device(*(x.data_ptr() for x in t), out.data_ptr(), stream=st.cuda_stream, **params)
        st.synchronize()
        assert out.cpu().numpy().tobytes() == want.tobytes()


def test_device_form_statuses():
    import torch
    g = api.Scene(partial_wall().finish())
    g.update_frame()
    n = g.width * g.height * 4
    buf = torch.zeros(6 * n + 64, dtype=torch.float32, device="cuda")
    p = buf.data_ptr()
    films = [p + k * n * 4 for k in range(5)]  # a, b, albedo, normal, nearest (n floats are ample for width*height uint64)
    out = p + 5 * n * 4
    ok = films + [out]
    g.denoise_device(*ok)
    torch.cuda.synchronize()
    for k, off in ((0, 4), (2, 8), (4, 4), (5, 4)):
        args = list(ok)
        args[k] += off
        with pytest.raises(api.TrbError) as e:
            g.denoise_device(*args)
        assert e.value.status == F.TRB_INVALID_ARG
    for k in range(5):  # the output on top of any input
        args = list(ok)
        args[5] = films[k] + (16 if k else 0)
        with pytest.raises(api.TrbError) as e:
            g.denoise_device(*args)
        assert e.value.status == F.TRB_INVALID_ARG and "overlaps" in str(e.value)
    for k in range(5):
        args = list(ok)
        args[k] = None
        with pytest.raises(api.TrbError) as e:
            g.denoise_device(*args)
        assert e.value.status == F.TRB_INVALID_ARG
    torch.cuda.synchronize()


def test_scratch_follows_replace_settings_to_a_larger_and_a_smaller_film():
    b = partial_wall()
    g = api.Scene(b.finish())
    g.update_frame()
    rng = np.random.default_rng(8)
    a0, b0, aov0 = synthetic(rng, g.height, g.width)
    assert_bit_exact(g, a0, b0, aov0)  # the scratch exists at 32 x 32
    for w, h in ((96, 64), (16, 24)):
        b.film = dict(b.film, width=w, height=h)
        g.replace_settings(b.film)
        fresh = api.Scene(b.finish())
        a, bb, aovs = synthetic(rng, h, w)
        got = assert_bit_exact(g, a, bb, aovs)
        assert got.tobytes() == fresh.denoise(a, bb, aovs).tobytes()
        fresh.close()


# ---- quality ----------------------------------------------------------------------------------------------------------------------

def rmse(x, ref, mask=None):
    c = np.clip(x[..., :3] / np.maximum(x[..., 3:], 1e-12), 0, 1) if x.shape[-1] == 4 else x
    r = np.clip(ref[..., :3] / ref[..., 3:], 0, 1)
    d = (c - r) ** 2
    if mask is not None:
        d = d[mask]
    return float(np.sqrt(d.mean()))


@pytest.mark.parametrize("scene", ["c1_cornell_box.json", "c2_smallpt.json"])
def test_quality_on_c1_and_c2(scene):
    g = api.Scene(json_desc(scene, 256, 256, 4))
    g.update_frame()
    ref, _ = g.render(spp=1024, seed=99, flags=F.RENDER_NO_UPDATE)
    noisy16, _ = g.render(spp=16, seed=5, flags=F.RENDER_NO_UPDATE)
    den4, noisy4, _, _ = g.render_denoised(4, seed=5, flags=F.RENDER_NO_UPDATE)
    den64, _, _, _ = g.render_denoised(64, seed=5, flags=F.RENDER_NO_UPDATE)
    r = dict(den4=rmse(den4, ref), noisy4=rmse(noisy4, ref), noisy16=rmse(noisy16, ref), den64=rmse(den64, ref))
    print(scene, r)
    assert r["den4"] < r["noisy16"], r
    assert r["den64"] < r["den4"], r


def test_quality_at_albedo_edges_of_the_textured_scene():
    desc = textured_zoo(4, 128).finish()
    g = api.Scene(desc)
    g.update_frame(1, 0.5, 1.0)
    kw = dict(flags=F.RENDER_NO_UPDATE)
    ref, ref_aovs, _ = g.render_aov(spp=1024, seed=99, normal=False, nearest=False, **kw)
    albedo = ref_aovs["albedo_w"][..., :3] / np.maximum(ref_aovs["albedo_w"][..., 3:], 1e-12)
    jump = np.zeros(albedo.shape[:2], bool)
    for axis in (0, 1):
        d = np.abs(np.diff(albedo, axis=axis)).max(-1) > 0.1
        if axis == 0:
            jump[1:] |= d; jump[:-1] |= d
        else:
            jump[:, 1:] |= d; jump[:, :-1] |= d
    edge = jump.copy()  # within one pixel of an albedo edge
    edge[1:] |= jump[:-1]; edge[:-1] |= jump[1:]; edge[:, 1:] |= jump[:, :-1]; edge[:, :-1] |= jump[:, 1:]
    assert 0.02 < edge.mean() < 0.8
    den4, noisy4, _, _ = g.render_denoised(4, seed=5, **kw)
    r = dict(den4=rmse(den4, ref, edge), noisy4=rmse(noisy4, ref, edge))
    print("textured edges", r, float(edge.mean()))
    assert r["den4"] < r["noisy4"], r


# ---- trb_tray --denoise -----------------------------------------------------------------------------------------------------------

def test_tray_denoise_writes_what_render_denoised_computes(tmp_path):
    H.build_programs()
    png = tmp_path / "c1.png"
    p = H.Proc([H.TRAY, H.CORNELL, "--denoise", "-o", str(png), "--seed", "7"])
    try:
        rc, out, err = p.finish(timeout=600)
    finally:
        p.kill()
    assert rc == 0, err
    g = api.Scene(json_desc("c1_cornell_box.json", 0, 0, 0))
    den, _, _, _ = g.render_denoised(seed=7)
    want = g.to_srgb8(den)
    got = H.read_png(png)
    d = np.abs(got.astype(int) - want.astype(int))
    print("trb_tray --denoise vs render_denoised: max byte difference %d, %.2e of the bytes differ" % (d.max(), np.count_nonzero(d) / d.size))
    assert d.max() <= 1 and np.count_nonzero(d) < 1e-3 * d.size, (d.max(), np.count_nonzero(d) / d.size)
