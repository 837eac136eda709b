"""trb_illumination on an H100: Integrator::illumination along caller rays runs on the render's wavefront kernels (k_illum_load,
k_wf_trace with PIPE bit 64 for round 0, the MODE 2 shade kernels, k_illum_reduce; k_simple_integrator<2> for Whitted and
NormalsDebug) and must equal the oracle's orc_illumination bit for bit — every output and every counter — and, for camera rays
keyed like the render's samples, trb_render_samples itself."""
import os

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_queries import pyqueries as Q
from test_illumination_cpu import camera_samples, illum_rays
from test_queries_cpu import at_hit_rays, edge_rays, query_rays, random_rays
from test_queries_gpu import json_desc
from test_textures import textured_zoo

pytestmark = pytest.mark.gpu
RAYS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation"]
TESTS = ["node_tests", "tri_tests", "inst_tests"]


def torch():
    import torch as t
    return t


def _integrator(b, integ):
    b.integrator = integ
    return b


# name -> (description, (frame, start, end)); the shutter interval is [start, start + shutter_size * (end - start)]
SCENES = {
    "c1": lambda: (json_desc("c1_cornell_box.json", 32, 24, 2), (0, 0.0, 0.0)),
    "c2": lambda: (json_desc("c2_smallpt.json", 32, 32, 2), (0, 0.0, 0.0)),
    "zoo": lambda: (SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()).finish(), (0, 0.0, 0.0)),
    "textured": lambda: (textured_zoo(2, 32).finish(), (1, 0.5, 1.0)),
    "keyframed": lambda: (SB.scene_animated(32, 32, 2, animated_fov=True).finish(), (1, 0.25, 0.5)),
    "whitted": lambda: (_integrator(SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()), (F.INTEGRATOR_WHITTED, 0, 4)).finish(), (0, 0.0, 0.0)),
    "normals": lambda: (_integrator(SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()), (F.INTEGRATOR_NORMALS_DEBUG, 0, 0)).finish(), (0, 0.0, 0.0)),
}


def both(desc, frame):
    g, o = api.Scene(desc), Q.QueryOracleScene(desc)
    g.update_frame(*frame); o.update_frame(*frame)
    return g, o


def shutter(frame):
    _, start, end = frame
    return start, start + 0.5 * (end - start)


def ray_set(o, frame, seed, n_random=2048):
    """camera rays at spread times, incoherent rays, unnormalised directions, the edge cases, min_t / max_t exactly at the hits"""
    t0, t1 = shutter(frame)
    rays, _ = o.camera_rays(seed=seed)
    rng = np.random.default_rng(seed)
    times = rng.uniform(t0, t1, size=len(rays)).astype(np.float32)
    rnd = random_rays(n_random, seed, (-14, 1, -10), (14, 23, 18), t0, t1)
    long_ = rnd[: n_random // 4].copy()
    long_["d"] *= rng.uniform(0.25, 4.0, size=(len(long_), 1)).astype(np.float32)  # not normalised: used as given
    q = np.concatenate([query_rays(rays, times), rnd, long_, edge_rays(t0)])
    rec, _ = o.intersect_records(q)
    hits = at_hit_rays(q, rec)
    q = np.concatenate([q, hits[rng.permutation(len(hits))[:512]]])
    return illum_rays(q, key0=seed * 7919, sample0=seed)


def counters(st, keys):
    return [getattr(st, k) for k in keys]


def same_bits(a, b):
    """Bit for bit, except that a NaN only has to be a NaN: x86 and the GPU make NaNs with different signs and payloads (the edge
    rays and unnormalised directions can make them)."""
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and (na == nb).all() and a[~na].tobytes() == b[~nb].tobytes()


@pytest.mark.parametrize("name", sorted(SCENES))
def test_matches_orc_illumination(name):
    desc, frame = SCENES[name]()
    g, o = both(desc, frame)
    q = ray_set(o, frame, 11)
    for spp in (1, 3, 16):
        qs = q if spp < 16 else q[::4]
        for clamp in (False, True):
            ost = F.Stats()
            want = o.illumination(qs, spp=spp, seed=5, clamp=clamp, stats=ost)
            rst, ast = F.Stats(), F.Stats()
            ref = g.illumination(qs, spp=spp, seed=5, clamp=clamp, stats=rst, reference=True)
            anyh = g.illumination(qs, spp=spp, seed=5, clamp=clamp, stats=ast)
            tag = (name, spp, clamp)
            assert same_bits(ref, want), tag
            assert same_bits(anyh, want), tag  # any-hit shadow rays: same booleans, same radiance
            assert counters(rst, RAYS + TESTS) == counters(ost, RAYS + TESTS), tag
            assert counters(ast, RAYS) == counters(ost, RAYS) and ast.node_tests <= rst.node_tests, tag
            assert ost.camera_samples == ost.rays_primary == len(qs) * spp, tag
            assert same_bits(g.illumination(qs, spp=spp, seed=5, clamp=clamp), want), tag  # the counter-free kernels
    assert (want > 0).any() and (want == 0).all(axis=1).any()
    if name not in ("normals", "whitted"):
        assert ost.rays_continuation > 0 and ost.rays_shadow > 0


@pytest.mark.parametrize("split", [0, 1])
def test_camera_rays_keyed_like_the_render_give_its_samples(split):
    """trb_camera_rays + key = pixel, sample = si, spp = 1, clamp == trb_render_samples' r, g, b (these scenes render at a [0, 0]
    shutter, so every camera ray's time is 0)"""
    cases = [("c1", {}), ("c2", {}), ("zoo", {})]
    for name, kw in cases + [("c4", dict(block_start=300, block_count=48))]:
        if name == "c4":
            g = api.Scene(SB.scene_c4(1_000_000, 256, 256, 4).finish())
            g.update_frame(0, 0.0, 0.0)
        else:
            desc, frame = SCENES[name]()
            g = api.Scene(desc)
            g.update_frame(*frame)
        g.set_option("shade.split", split)
        q = camera_samples(g, seed=3, **kw)
        samples, sst = g.render_samples(seed=3, **kw)
        st = F.Stats()
        rgb = g.illumination(q, spp=1, seed=3, clamp=True, stats=st, reference=True)
        want = np.stack([samples["r"], samples["g"], samples["b"]], axis=1)
        assert rgb.tobytes() == want.tobytes(), name
        assert counters(st, RAYS) == counters(sst, RAYS), name


def test_spp_k_is_the_float32_sum_of_k_single_sample_calls():
    desc, frame = SCENES["keyframed"]()
    g, o = both(desc, frame)
    q = ray_set(o, frame, 12)
    for clamp in (False, True):
        k = 5
        whole = g.illumination(q, spp=k, seed=9, clamp=clamp)
        acc = None
        for j in range(k):
            qj = q.copy()
            qj["sample"] = q["sample"] + j
            one = g.illumination(qj, spp=1, seed=9, clamp=clamp)
            acc = one if acc is None else (acc + one).astype(np.float32)
        assert same_bits(whole, (acc / np.float32(k)).astype(np.float32)), clamp


def test_many_small_passes_give_the_bytes_of_one_pass():
    for name in ("zoo", "keyframed", "whitted"):
        desc, frame = SCENES[name]()
        g, o = both(desc, frame)
        q = ray_set(o, frame, 14)
        st1, st2 = F.Stats(), F.Stats()
        one = g.illumination(q, spp=3, seed=2, stats=st1, reference=True)
        g.set_option("pass.paths", 1000)  # 1024 paths per pass: 341 rays of 3 samples
        assert len(q) * 3 > 8 * 1024
        many = g.illumination(q, spp=3, seed=2, stats=st2, reference=True)
        assert same_bits(many, one), name
        assert counters(st2, RAYS + TESTS) == counters(st1, RAYS + TESTS), name


def test_device_form_equals_the_host_form_and_does_not_wait():
    T = torch()
    desc, frame = SCENES["keyframed"]()
    g, o = both(desc, frame)
    q = ray_set(o, frame, 13)
    n = len(q)
    hst = F.Stats()
    host = g.illumination(q, spp=4, seed=8, clamp=True, stats=hst)
    dev = T.device("cuda:0")
    d_rays = T.from_numpy(q.view(np.uint8).copy()).to(dev)
    d_rgb = T.zeros(n * 3, dtype=T.float32, device=dev)
    d_st = T.zeros(9, dtype=T.int64, device=dev)
    s = T.cuda.Stream()
    s.wait_stream(T.cuda.current_stream())
    with T.cuda.stream(s):
        T.cuda._sleep(2_000_000_000)  # about a second of GPU time ahead of the queries
    g.illumination_device(n, d_rays.data_ptr(), d_rgb.data_ptr(), spp=4, seed=8, clamp=True, d_stats=d_st.data_ptr(), stream=s.cuda_stream, stats=True)
    assert not s.query(), "the call waited for its stream"
    s.synchronize()
    g.check_error()
    assert same_bits(d_rgb.cpu().numpy().reshape(n, 3), host)
    st = F.Stats.from_buffer_copy(d_st.cpu().numpy().tobytes())
    assert counters(st, RAYS + TESTS) == counters(hst, RAYS + TESTS)


def test_c4_incoherent_rays_match_the_oracle():
    desc = SB.scene_c4(1_000_000, 64, 64, 1).finish()
    g, o = both(desc, (0, 0.0, 0.0))
    q = illum_rays(random_rays(1 << 18, 21, (-14, 1, -10), (14, 23, 18), 0.0, 0.0))
    ost, gst = F.Stats(), F.Stats()
    want = o.illumination(q, spp=4, seed=3, stats=ost)
    got = g.illumination(q, spp=4, seed=3, stats=gst, reference=True)
    assert same_bits(got, want)
    assert counters(gst, RAYS + TESTS) == counters(ost, RAYS + TESTS)


def test_statuses():
    T = torch()
    desc, frame = SCENES["zoo"]()
    fresh = api.Scene(desc)
    q = illum_rays(random_rays(64, 1, (-1, 1, -1), (1, 2, 1), 0.0, 0.0))
    with pytest.raises(api.TrbError) as e:
        fresh.illumination(q)
    assert e.value.status == F.TRB_INVALID_ARG and "Update frame must be called before rendering" in str(e.value)
    fresh.update_frame(*frame)
    for kw in (dict(spp=0), dict(spp=65537)):
        with pytest.raises(api.TrbError) as e:
            fresh.illumination(q, **kw)
        assert e.value.status == F.TRB_INVALID_ARG, kw
    st = F.Stats()
    assert fresh.illumination(q[:0], stats=st).shape == (0, 3) and st.rays_primary == 0
    fresh.illumination_device(0, None, None)
    d = T.zeros(64 * 48 + 64, dtype=T.uint8, device="cuda:0")
    out = T.zeros(64 * 3 + 4, dtype=T.float32, device="cuda:0")
    for args in ((d.data_ptr() + 4, out.data_ptr()), (d.data_ptr(), out.data_ptr() + 2)):  # rays 16-byte, rgb 4-byte aligned
        with pytest.raises(api.TrbError) as e:
            fresh.illumination_device(1, *args)
        assert e.value.status == F.TRB_INVALID_ARG
    lib = F.load_trb()
    rgb = np.zeros((len(q), 3), np.float32)
    for flags in (F.RENDER_MEGAKERNEL, F.RENDER_TIME_TRACE, F.RENDER_NO_UPDATE, 64):
        assert lib.trb_illumination(fresh._h, len(q), F.ptr(q), 1, 1, F.ptr(rgb), flags, None) == F.TRB_INVALID_ARG, flags
    assert fresh.illumination(q[:2], spp=65536).shape == (2, 3)  # the largest accepted spp: a pass holds whole rays
