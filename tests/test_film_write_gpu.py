"""trb_film_write on an H100: the sort by region and the per-block gather (k_film_keys, CUB's radix sort, k_film_starts,
k_film_gather) must leave the film orc_film_write leaves, bit for bit, and trb_render_samples written with it must be the film of a
one-thread reference render. trb_camera_rays_device must give trb_camera_rays' bits."""
import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_queries import pyqueries as Q
from test_film_write_cpu import random_samples
from test_illumination_cpu import camera_samples
from test_illumination_gpu import SCENES as ILLUM_SCENES, same_bits

pytestmark = pytest.mark.gpu

FILTERS = {  # name -> (type, w, h, b, c): fpw 4; fpw 6 / 5 with the lock-block filter rejecting; fpw 8
    "mitchell": (F.FILTER_MITCHELL_NETRAVALI, 2.0, 2.0, 1 / 3, 1 / 3),
    "gauss_wide": (F.FILTER_GAUSSIAN, 3.0, 2.5, 0.5, 0.0),
    "gauss_fpw8": (F.FILTER_GAUSSIAN, 4.0, 4.0, 0.5, 0.0),
}


def torch():
    import torch as t
    return t


def film_scene(w, h, filt):
    b = SB.scene_smallpt_like(w, h, 1)
    t, fw, fh, fb, fc = FILTERS[filt]
    b.film.update(filter_type=t, filter_w=fw, filter_h=fh, filter_b=fb, filter_c=fc)
    desc = b.finish()
    return api.Scene(desc), Q.QueryOracleScene(desc)


def awkward_samples(rng, w, h):
    """random positions up to 20 px beyond their region, pixel and block edges, x = px + 1, NaN and +-inf positions, negative /
    NaN / inf colours, out-of-range regions"""
    s, reg = random_samples(rng, 3000, w, h)
    nbx, nr = w // 8, (w // 8) * (h // 8)
    k = np.arange(len(s))
    px = (reg % nbx) * 8 + rng.integers(0, 8, len(s))
    one = k % 11 == 0
    s["x"][one] = (px[one] + 1).astype(np.float32)  # an LD position that rounded up to the next pixel (and sometimes block)
    s["x"][k % 97 == 1], s["y"][k % 89 == 2] = np.nan, np.nan
    s["x"][k % 101 == 3], s["y"][k % 103 == 4] = np.inf, -np.inf
    s["r"][k % 107 == 5], s["g"][k % 109 == 6], s["b"][k % 113 == 7] = np.nan, np.inf, -np.inf
    reg[k % 53 == 8] = nr + rng.integers(0, 1000, (k % 53 == 8).sum())
    reg[k % 59 == 9] = 0xFFFFFFFF
    return s, reg


def films(rng, w, h):
    z = np.zeros((h, w, 4), np.float32)
    r = rng.uniform(-2, 2, (h, w, 4)).astype(np.float32)
    nz = r.copy()
    nz[::2, 1::3] = -0.0
    return {"zero": z, "random": r, "negzero": nz}


@pytest.mark.parametrize("filt", sorted(FILTERS))
def test_matches_orc_film_write(filt):
    w, h = 40, 24  # not square, not multiples of 16
    g, o = film_scene(w, h, filt)
    rng = np.random.default_rng(sorted(FILTERS).index(filt) + 1)
    s, reg = awkward_samples(rng, w, h)
    for name, f0 in films(rng, w, h).items():
        want = o.film_write(s, reg, f0.copy())
        got = g.film_write(s, reg, f0.copy())
        assert same_bits(got, want), (filt, name)
        assert (np.signbit(got) == np.signbit(want))[~np.isnan(want)].all(), (filt, name)
        for n in (0, 1):
            assert same_bits(g.film_write(s[:n], reg[:n], f0.copy()), o.film_write(s[:n], reg[:n], f0.copy())), (filt, name, n)
    assert np.isnan(got).any() and (got != f0).any()


def test_every_sample_in_one_region():
    g, o = film_scene(40, 24, "gauss_wide")
    rng = np.random.default_rng(5)
    n = 1 << 16
    s = np.zeros(n, F.SAMPLE_DTYPE)
    s["x"], s["y"] = rng.uniform(2, 30, n).astype(np.float32), rng.uniform(0, 24, n).astype(np.float32)
    for k in ("r", "g", "b"):
        s[k] = rng.uniform(0, 1, n).astype(np.float32)
    reg = np.full(n, 6, np.uint32)  # block (1, 1)
    f0 = films(rng, 40, 24)["negzero"]
    assert g.film_write(s, reg, f0.copy()).tobytes() == o.film_write(s, reg, f0.copy()).tobytes()


@pytest.mark.parametrize("name", ["c1", "c2", "zoo", "textured", "keyframed"])
def test_render_samples_written_are_the_one_thread_reference_render(name):
    desc, frame = ILLUM_SCENES[name]()
    g, o = api.Scene(desc), Q.QueryOracleScene(desc)
    g.update_frame(*frame); o.update_frame(*frame)
    samples, _ = g.render_samples(seed=4)
    film = g.film_write(samples, g.sample_regions())
    ref, _ = o.render(seed=4, threads=1, flags=F.RENDER_NO_UPDATE)
    assert film.tobytes() == ref.tobytes(), name
    assert film[..., 3].any()


def test_c4_block_range_matches_the_render_film():
    g = api.Scene(SB.scene_c4(1_000_000, 1920, 1080, 8).finish())
    g.update_frame(0, 0.0, 0.0)
    kw = dict(block_start=9000, block_count=512, seed=3)
    samples, _ = g.render_samples(**kw)
    film = g.film_write(samples, g.sample_regions(**kw))
    ref, _ = g.render(flags=F.RENDER_NO_UPDATE, **kw)
    m = np.abs(ref[..., 3]) > 0.1  # the selected blocks and the fringe their filter reaches with some weight
    assert m.sum() > 512 * 64 and ((film != 0) == (ref != 0)).all()
    img_g, img_r = film[m][:, :3] / film[m][:, 3:], ref[m][:, :3] / ref[m][:, 3:]
    assert np.sqrt(np.mean((img_g - img_r) ** 2)) < 1e-5 and np.allclose(film, ref, rtol=1e-4, atol=1e-5)


def test_camera_rays_device_equals_the_host_form():
    T = torch()
    for name, kw in (("keyframed", {}), ("c1", dict(block_start=3, block_count=5, sample_first=1, sample_count=1))):
        desc, frame = ILLUM_SCENES[name]()
        g = api.Scene(desc)
        g.update_frame(*frame)
        rays, xy = g.camera_rays(seed=9, **kw)
        d_rays = T.zeros(len(rays) * 8, dtype=T.float32, device="cuda:0")
        d_xy = T.zeros(len(rays) * 2, dtype=T.float32, device="cuda:0")
        s = T.cuda.Stream()
        assert g.camera_rays_device(d_rays.data_ptr(), d_xy.data_ptr(), stream=s.cuda_stream, seed=9, **kw) == len(rays)
        s.synchronize()
        assert d_rays.cpu().numpy().tobytes() == rays.tobytes() and d_xy.cpu().numpy().tobytes() == xy.tobytes(), name


def test_device_pipeline_on_a_torch_stream_equals_the_host_pipeline():
    """camera_rays_device -> illumination_device (key = pixel, sample = si, spp 1, clamp) -> film_write_device, all on one stream"""
    T = torch()
    desc, frame = ILLUM_SCENES["zoo"]()
    g = api.Scene(desc)
    g.update_frame(*frame)
    samples, _ = g.render_samples(seed=6)
    want = g.film_write(samples, g.sample_regions())
    q = camera_samples(g, seed=6)  # the keys and sample indices (host constants); the rays come from the device below
    n = len(q)
    dev = T.device("cuda:0")
    s = T.cuda.Stream()
    s.wait_stream(T.cuda.current_stream())
    with T.cuda.stream(s):
        d_rays = T.zeros((n, 8), dtype=T.float32, device=dev)
        d_xy = T.zeros((n, 2), dtype=T.float32, device=dev)
        g.camera_rays_device(d_rays.data_ptr(), d_xy.data_ptr(), stream=s.cuda_stream, seed=6)
        illum = T.zeros((n, 12), dtype=T.float32, device=dev)
        illum[:, :8] = d_rays
        illum.view(T.int32)[:, 9] = T.from_numpy(q["key"].view(np.int32)).to(dev, non_blocking=True)
        illum.view(T.int32)[:, 10] = T.from_numpy(q["sample"].view(np.int32)).to(dev, non_blocking=True)
        d_rgb = T.zeros((n, 3), dtype=T.float32, device=dev)
        g.illumination_device(n, illum.data_ptr(), d_rgb.data_ptr(), spp=1, seed=6, clamp=True, stream=s.cuda_stream)
        d_s = T.cat([d_xy, d_rgb], dim=1).contiguous()
        d_reg = T.from_numpy(g.sample_regions().view(np.int32)).to(dev, non_blocking=True)
        d_film = T.zeros((g.height, g.width, 4), dtype=T.float32, device=dev)
        g.film_write_device(n, d_s.data_ptr(), d_reg.data_ptr(), d_film.data_ptr(), stream=s.cuda_stream)
    s.synchronize()
    g.check_error()
    assert d_film.cpu().numpy().tobytes() == want.tobytes()


def test_deterministic_at_1080p_host_and_device():
    T = torch()
    g = api.Scene(SB.scene_smallpt_like(1920, 1080, 1).finish())
    rng = np.random.default_rng(8)
    s, reg = random_samples(rng, 1 << 22, 1920, 1080, spread=6.0)
    a = g.film_write(s, reg)
    b = g.film_write(s, reg)
    dev = T.device("cuda:0")
    d_s = T.from_numpy(s.view(np.float32).reshape(-1, 5).copy()).to(dev)
    d_reg = T.from_numpy(reg.view(np.int32).copy()).to(dev)
    d_film = T.zeros((1080, 1920, 4), dtype=T.float32, device=dev)
    st = T.cuda.Stream()
    g.film_write_device(len(s), d_s.data_ptr(), d_reg.data_ptr(), d_film.data_ptr(), stream=st.cuda_stream)  # the scratch has grown
    st.wait_stream(T.cuda.current_stream())
    with T.cuda.stream(st):
        T.cuda._sleep(2_000_000_000)  # about a second of GPU time ahead of the write
    d_film2 = T.zeros_like(d_film)
    g.film_write_device(len(s), d_s.data_ptr(), d_reg.data_ptr(), d_film2.data_ptr(), stream=st.cuda_stream)
    assert not st.query(), "the call waited for its stream"
    st.synchronize()
    assert a.tobytes() == b.tobytes() == d_film.cpu().numpy().tobytes() == d_film2.cpu().numpy().tobytes()
    assert (a[..., 3] != 0).mean() > 0.99


def test_statuses():
    T = torch()
    desc, frame = ILLUM_SCENES["c1"]()
    fresh = api.Scene(desc)
    s, reg = random_samples(np.random.default_rng(1), 64, fresh.width, fresh.height)
    assert fresh.film_write(s, reg).any()  # no update_frame needed: the filter is fixed at creation
    assert not fresh.film_write(s[:0], reg[:0]).any()
    fresh.film_write_device(0, None, None, None)
    lib = F.load_trb()
    film = np.zeros((fresh.height, fresh.width, 4), np.float32)
    assert lib.trb_film_write(fresh._h, 1 << 32, F.ptr(s), F.ptr(reg), F.ptr(film)) == F.TRB_INVALID_ARG
    d = T.zeros(64 * 5 + 4, dtype=T.float32, device="cuda:0")
    r = T.zeros(64 + 4, dtype=T.int32, device="cuda:0")
    f = T.zeros(fresh.height * fresh.width * 4 + 4, dtype=T.float32, device="cuda:0")
    for args in ((d.data_ptr() + 2, r.data_ptr(), f.data_ptr()), (d.data_ptr(), r.data_ptr() + 1, f.data_ptr()),
                 (d.data_ptr(), r.data_ptr(), f.data_ptr() + 2)):
        with pytest.raises(api.TrbError) as e:
            fresh.film_write_device(64, *args)
        assert e.value.status == F.TRB_INVALID_ARG
    assert lib.trb_film_write_device(fresh._h, (1 << 32) + 64, d.data_ptr(), r.data_ptr(), f.data_ptr(), None) == F.TRB_INVALID_ARG
    with pytest.raises(api.TrbError) as e:
        fresh.camera_rays_device(d.data_ptr(), d.data_ptr())
    assert e.value.status == F.TRB_INVALID_ARG and "Update frame must be called before rendering" in str(e.value)
    fresh.update_frame(*frame)
    with pytest.raises(api.TrbError) as e:
        fresh.camera_rays_device(d.data_ptr() + 2, d.data_ptr(), block_count=1, sample_count=1)
    assert e.value.status == F.TRB_INVALID_ARG
