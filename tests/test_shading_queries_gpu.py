"""The shading queries on an H100: trb_bsdf_eval / trb_bsdf_sample (Material::bsdf with BSDF::eval, pdf and sample at a record),
trb_light_sample / trb_light_pdf (Light::sample_incident and Light::pdf), trb_emitted (Emitter::radiance) and trb_scene_lights run the
render's device functions and must equal the oracle bit for bit (a NaN only has to be a NaN). examples/query_path.py composes them into
the render's path tracer: its estimate must converge to trb_illumination's."""
import os
import sys

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api
from test_illumination_cpu import illum_rays
from test_illumination_gpu import SCENES as ILLUM_SCENES, both, same_bits, shutter
from test_queries_cpu import edge_rays, query_rays, random_rays

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
import query_path as QP  # noqa: E402

pytestmark = pytest.mark.gpu
SCENES = {k: ILLUM_SCENES[k] for k in ("c1", "c2", "zoo", "textured", "keyframed")}
ONE_MINUS_ULP = np.nextafter(np.float32(1), np.float32(0))


def torch():
    import torch as t
    return t


def same(a, b):
    """same_bits over every 4-byte word of two structured or float arrays"""
    return same_bits(np.ascontiguousarray(a).view(np.float32), np.ascontiguousarray(b).view(np.float32))


def _unit(v):
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def records(desc, o, frame, seed):
    """records of camera and incoherent rays from intersect_records, plus synthetic records for every material: random frames and
    points, zero or denormal dp_du, times spread beyond the shutter interval (animated textures), and out-of-range ones"""
    t0, t1 = shutter(frame)
    rng = np.random.default_rng(seed)
    rays, _ = o.camera_rays(seed=seed)
    q = np.concatenate([query_rays(rays, rng.uniform(t0, t1, len(rays)).astype(np.float32)),
                        random_rays(2048, seed, (-14, 1, -10), (14, 23, 18), t0, t1), edge_rays(t0)])
    rec, _ = o.intersect_records(q)
    hits = rec[rec["inst"] != F.MISS]
    n_mat = desc.n_materials
    syn = np.zeros(64 * n_mat, F.INTERSECTION_DTYPE)
    syn["material"] = np.arange(len(syn)) % n_mat
    syn["p"] = rng.uniform(-10, 20, (len(syn), 3))
    syn["n"] = _unit(rng.normal(size=(len(syn), 3)))
    syn["ng"] = syn["n"]
    syn["dp_du"] = rng.normal(size=(len(syn), 3)) * rng.uniform(0.01, 50, (len(syn), 1))
    syn["dp_du"][::9] = 0.0
    syn["dp_du"][1::9] = [1e-40, 0.0, 0.0]
    syn["u"], syn["v"] = rng.uniform(-0.2, 1.2, len(syn)), rng.uniform(-0.2, 1.2, len(syn))
    syn["time"] = rng.uniform(0.0, 1.5, len(syn))
    bad = np.zeros(3, F.INTERSECTION_DTYPE)
    bad["inst"], bad["material"], bad["n"], bad["dp_du"] = [F.MISS, 0, 0], [0, n_mat, 0xFFFFFFFF], (0, 0, 1), (1, 0, 0)
    return np.concatenate([hits, syn, bad]), len(bad)


def directions(rec, rng):
    """(wo, wi) pairs per record in several kinds: random, both hemispheres, grazing (shading-space z = +-0), exact mirror,
    unnormalised, zero and NaN vectors"""
    n = len(rec)
    nn = rec["n"] / np.maximum(np.linalg.norm(rec["n"], axis=1, keepdims=True), 1e-30)
    bt = rec["dp_du"] / np.maximum(np.linalg.norm(rec["dp_du"], axis=1, keepdims=True), 1e-30)
    tan = np.cross(nn, bt).astype(np.float32)
    wo = _unit(rng.normal(size=(n, 3)))
    wo = np.where((wo * nn).sum(1, keepdims=True) < 0, -wo, wo).astype(np.float32)  # mostly above the surface
    wo[::7] *= -1.0
    mirror = (2.0 * (wo * nn).sum(1, keepdims=True) * nn - wo).astype(np.float32)
    kinds = [_unit(rng.normal(size=(n, 3))), -wo, mirror, tan, -tan, mirror * np.float32(3.5), np.zeros((n, 3), np.float32),
             np.full((n, 3), np.nan, np.float32)]
    wos = [wo, wo, wo, wo, wo, wo * np.float32(0.25), wo, wo]
    wos[6] = np.where(np.arange(n)[:, None] % 2 == 0, wo, 0.0).astype(np.float32)  # a zero wo too
    return np.concatenate(wos), np.concatenate(kinds), len(kinds)


@pytest.mark.parametrize("name", sorted(SCENES))
def test_bsdf_queries_match_the_oracle(name):
    desc, frame = SCENES[name]()
    g, o = both(desc, frame)
    rng = np.random.default_rng(3)
    rec, n_bad = records(desc, o, frame, 5)
    wo, wi, k = directions(rec, rng)
    recs = np.tile(rec, k)
    n = len(recs)
    eq = np.zeros(n, F.BSDF_EVAL_QUERY_DTYPE)
    eq["wo"], eq["wi"], eq["bxdf"] = wo, wi, np.arange(n) % 32  # all 32 lobe sets
    want = o.bsdf_eval(recs, eq)
    got = g.bsdf_eval(recs, eq)
    assert same(got, want), name
    assert (want[:, :3] > 0).any() and (want[:, 3] > 0).any()
    sq = np.zeros(n, F.BSDF_SAMPLE_QUERY_DTYPE)
    sq["wo"], sq["bxdf"] = wo, (np.arange(n) * 7) % 32
    edges = np.array([0.0, ONE_MINUS_ULP, 1.0], np.float32)
    sq["u"] = np.where(rng.random((n, 2)) < 0.2, edges[rng.integers(0, 3, (n, 2))], rng.random((n, 2))).astype(np.float32)
    sq["u_comp"] = np.where(rng.random(n) < 0.3, edges[rng.integers(0, 3, n)], rng.random(n)).astype(np.float32)  # 1.0: the clamp
    want = o.bsdf_sample(recs, sq)
    assert same(g.bsdf_sample(recs, sq), want), name
    assert len(np.unique(want["sampled"])) >= 2 and (want["pdf"] > 0).any()
    # out of range (a miss, material == n_materials, material 0xffffffff): zeros
    bad = np.concatenate([np.arange(len(rec) - n_bad, len(rec)) + j * len(rec) for j in range(k)])
    assert not want[bad].view(np.uint8).any()
    assert not g.bsdf_eval(recs[bad], eq[bad]).any()


def light_points(g, o, desc, frame, rng, lights):
    """receiving points: hit points, and for every area light points inside, on and outside a sphere about its centre of radius
    p0 times its scale (the dist_sqr - r^2 < 1e-4 branch of sphere.rs for sphere lights)"""
    t0, t1 = shutter(frame)
    rays, _ = o.camera_rays(seed=2)
    rec, _ = o.intersect_records(query_rays(rays, rng.uniform(t0, t1, len(rays)).astype(np.float32)))
    pts = [rec["p"][rec["inst"] != F.MISS]]
    for li in lights:
        inst = desc.instances[int(li)]
        if inst.kind != F.INST_EMITTER_AREA:
            continue
        m, _ = g.transform(int(li))
        c, r = m[:3, 3], inst.p0 * np.linalg.norm(m[:3, 0])
        s = np.array([0.0, 0.5, 0.9999, 1.0, 1.00001, 1.001, 1.01, 2.0, 5.0], np.float32)
        dirs = _unit(rng.normal(size=(len(s), 3)))
        pts.append((c + r * s[:, None] * dirs).astype(np.float32))
    return np.concatenate(pts).astype(np.float32)


@pytest.mark.parametrize("name", sorted(SCENES))
def test_light_queries_match_the_oracle(name):
    desc, frame = SCENES[name]()
    g, o = both(desc, frame)
    rng = np.random.default_rng(7)
    lights = g.lights()
    assert np.array_equal(lights, o.lights()) and len(lights) == g.n_lights
    pts = light_points(g, o, desc, frame, rng, lights)
    t0, t1 = shutter(frame)
    n = len(pts) * len(lights)
    q = np.zeros(n + 4, F.LIGHT_QUERY_DTYPE)
    q["p"][:n] = np.tile(pts, (len(lights), 1))
    q["light"][:n] = np.repeat(lights, len(pts))
    q["time"] = rng.uniform(t0, t1, len(q))  # per-query times across the shutter interval (keyframed lights and emission)
    edges = np.array([0.0, ONE_MINUS_ULP, 1.0], np.float32)
    q["u"] = np.where(rng.random((len(q), 2)) < 0.2, edges[rng.integers(0, 3, (len(q), 2))], rng.random((len(q), 2))).astype(np.float32)
    receiver = next(i for i in range(desc.n_instances) if desc.instances[i].kind == F.INST_RECEIVER)
    q["light"][n:] = [receiver, desc.n_instances, F.MISS, desc.n_instances + 7]  # not lights: zeros
    want = o.light_sample(q)
    got = g.light_sample(q)
    assert same(got, want), name
    assert not want[n:].view(np.uint8).any() and (want["pdf"][:n] > 0).any()
    # the shadow rays go straight into trb_occluded and give the oracle's booleans
    sh = got["shadow"][:n]
    occ, _ = o.occluded(sh)
    gocc, _ = g.occluded(sh)
    assert np.array_equal(gocc, occ)
    # Light::pdf: sampled directions, random directions (mostly misses), and directions to each light's centre (a disk's hole)
    centres = np.stack([g.transform(int(li))[0][:3, 3] for li in q["light"][:n]])
    pq = np.zeros(3 * n + 4, F.LIGHT_PDF_QUERY_DTYPE)
    for j, w in enumerate([want["wi"][:n], _unit(rng.normal(size=(n, 3))), (centres - q["p"][:n]).astype(np.float32)]):
        pq["p"][j * n:(j + 1) * n], pq["wi"][j * n:(j + 1) * n] = q["p"][:n], w
        pq["light"][j * n:(j + 1) * n], pq["time"][j * n:(j + 1) * n] = q["light"][:n], q["time"][:n]
    pq["light"][3 * n:] = q["light"][n:]
    pq["wi"][3 * n:] = (0, 0, 1)
    wpdf = o.light_pdf(pq)
    assert same_bits(g.light_pdf(pq), wpdf), name
    assert (wpdf[3 * n:] == 0).all() and (wpdf > 0).any()


@pytest.mark.parametrize("name", sorted(SCENES))
def test_emitted_matches_the_oracle(name):
    desc, frame = SCENES[name]()
    g, o = both(desc, frame)
    rng = np.random.default_rng(9)
    t0, t1 = shutter(frame)
    ni = desc.n_instances
    insts = np.concatenate([np.arange(ni), [ni, F.MISS]]).astype(np.uint32)
    m = 64
    q = np.zeros(len(insts) * m, F.EMIT_QUERY_DTYPE)
    q["inst"] = np.repeat(insts, m)
    q["n"] = _unit(rng.normal(size=(len(q), 3)))
    w = rng.normal(size=(len(q), 3)).astype(np.float32)  # both signs of dot(w, n)
    w[::5] = 0.0
    w[1::5] = -q["n"][1::5]
    q["w"] = w
    q["time"] = rng.uniform(t0 - 0.25, t1 + 0.25, len(q))
    want = o.emitted(q)
    assert same_bits(g.emitted(q), want), name
    assert (want > 0).any() and not want[-2 * m:].any()


def test_bsdf_queries_and_emitted_need_no_frame_light_queries_do():
    desc, frame = SCENES["keyframed"]()
    fresh, (g, o) = api.Scene(desc), both(desc, frame)
    rec, _ = records(desc, o, frame, 4)
    rng = np.random.default_rng(1)
    wo, wi, _ = directions(rec, rng)
    eq = np.zeros(len(rec), F.BSDF_EVAL_QUERY_DTYPE)
    eq["wo"], eq["wi"], eq["bxdf"] = wo[:len(rec)], wi[:len(rec)], F.BXDF_ALL
    assert same(fresh.bsdf_eval(rec, eq), g.bsdf_eval(rec, eq))
    mq = np.zeros(256, F.EMIT_QUERY_DTYPE)
    mq["inst"] = np.arange(256) % desc.n_instances
    mq["w"], mq["n"], mq["time"] = (0, 0, 1), (0, 0, 1), np.linspace(0, 1, 256)
    assert same_bits(fresh.emitted(mq), g.emitted(mq)) and fresh.emitted(mq).any()
    for call in (lambda: fresh.light_sample(np.zeros(4, F.LIGHT_QUERY_DTYPE)), lambda: fresh.light_pdf(np.zeros(4, F.LIGHT_PDF_QUERY_DTYPE))):
        with pytest.raises(api.TrbError) as e:
            call()
        assert e.value.status == F.TRB_INVALID_ARG and "Update frame" in str(e.value)
    assert g.light_sample(np.zeros(0, F.LIGHT_QUERY_DTYPE)).shape == (0,)  # n == 0 is TRB_OK
    assert np.array_equal(fresh.lights(), o.lights())


def test_device_forms_give_the_host_bytes_and_do_not_wait():
    T = torch()
    desc, frame = SCENES["keyframed"]()
    g, o = both(desc, frame)
    rng = np.random.default_rng(2)
    rec, _ = records(desc, o, frame, 6)
    wo, wi, _ = directions(rec, rng)
    n = len(rec)
    eq = np.zeros(n, F.BSDF_EVAL_QUERY_DTYPE)
    eq["wo"], eq["wi"], eq["bxdf"] = wo[:n], wi[:n], np.arange(n) % 32
    sq = np.zeros(n, F.BSDF_SAMPLE_QUERY_DTYPE)
    sq["wo"], sq["bxdf"], sq["u"], sq["u_comp"] = wo[:n], F.BXDF_ALL, rng.random((n, 2)), rng.random(n)
    lq = np.zeros(n, F.LIGHT_QUERY_DTYPE)
    lq["p"], lq["light"], lq["u"], lq["time"] = rec["p"], g.lights()[np.arange(n) % g.n_lights], rng.random((n, 2)), rng.random(n)
    pq = np.zeros(n, F.LIGHT_PDF_QUERY_DTYPE)
    pq["p"], pq["light"], pq["wi"], pq["time"] = rec["p"], lq["light"], wi[:n], lq["time"]
    mq = np.zeros(n, F.EMIT_QUERY_DTYPE)
    mq["w"], mq["n"], mq["inst"], mq["time"] = wo[:n], rec["ng"], np.arange(n) % desc.n_instances, lq["time"]
    dev = T.device("cuda:0")
    up = lambda a: T.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(dev)  # noqa: E731
    d_rec = up(rec)
    outs = {k: T.zeros(n * size, dtype=T.uint8, device=dev) for k, size in (("eval", 16), ("sample", 32), ("light", 80), ("pdf", 4), ("emit", 12))}
    ins = {k: up(a) for k, a in (("eval", eq), ("sample", sq), ("light", lq), ("pdf", pq), ("emit", mq))}
    s = T.cuda.Stream()
    s.wait_stream(T.cuda.current_stream())
    with T.cuda.stream(s):
        T.cuda._sleep(2_000_000_000)  # about a second of GPU time ahead of the queries
    st = s.cuda_stream
    g.bsdf_eval_device(n, d_rec.data_ptr(), ins["eval"].data_ptr(), outs["eval"].data_ptr(), stream=st)
    g.bsdf_sample_device(n, d_rec.data_ptr(), ins["sample"].data_ptr(), outs["sample"].data_ptr(), stream=st)
    g.light_sample_device(n, ins["light"].data_ptr(), outs["light"].data_ptr(), stream=st)
    g.light_pdf_device(n, ins["pdf"].data_ptr(), outs["pdf"].data_ptr(), stream=st)
    g.emitted_device(n, ins["emit"].data_ptr(), outs["emit"].data_ptr(), stream=st)
    assert not s.query(), "a call waited for its stream"
    s.synchronize()
    got = {k: v.cpu().numpy() for k, v in outs.items()}
    assert got["eval"].tobytes() == g.bsdf_eval(rec, eq).tobytes()
    assert got["sample"].tobytes() == g.bsdf_sample(rec, sq).tobytes()
    assert got["light"].tobytes() == g.light_sample(lq).tobytes()
    assert got["pdf"].tobytes() == g.light_pdf(pq).tobytes()
    assert got["emit"].tobytes() == g.emitted(mq).tobytes()
    g.bsdf_eval_device(0, None, None, None)  # n == 0 is TRB_OK
    for call in (lambda: g.bsdf_eval_device(1, d_rec.data_ptr() + 4, ins["eval"].data_ptr(), outs["eval"].data_ptr()),
                 lambda: g.bsdf_eval_device(1, d_rec.data_ptr(), ins["eval"].data_ptr(), outs["eval"].data_ptr() + 4),
                 lambda: g.light_pdf_device(1, ins["pdf"].data_ptr(), outs["pdf"].data_ptr() + 2),
                 lambda: g.emitted_device(1, ins["emit"].data_ptr() + 8, outs["emit"].data_ptr())):
        with pytest.raises(api.TrbError) as e:
            call()
        assert e.value.status == F.TRB_INVALID_ARG


@pytest.mark.parametrize("name", ["c2", "zoo"])
def test_query_path_converges_to_trb_illumination(name):
    """examples/query_path.py's integrator (torch random numbers) against trb_illumination (its own sample streams) on the same camera
    rays: the image means agree within 3 sigma, and the RMSE against a 4096-spp trb_illumination image halves per 4x samples"""
    desc, frame = SCENES[name]()
    g = api.Scene(desc)
    g.update_frame(*frame)
    rays, _ = g.camera_rays(spp=1)
    q = illum_rays(query_rays(rays, np.zeros(len(rays), np.float32)), key0=0, sample0=0)
    ref = g.illumination(q, spp=4096, seed=77, clamp=True)
    errs = {}
    for spp in (16, 64, 256):
        a = QP.render_rays(g, rays, spp, 1000 + spp, desc.integrator.min_depth, desc.integrator.max_depth, clamp=True)
        b = g.illumination(q, spp=spp, seed=2000 + spp, clamp=True)
        diff = (a - b).reshape(-1, 3)
        sigma = diff.std(axis=0) / np.sqrt(len(diff))
        assert (np.abs(diff.mean(axis=0)) < 3 * sigma + 1e-4).all(), (name, spp, diff.mean(axis=0), sigma)
        errs[spp] = float(np.sqrt(np.mean((a - ref) ** 2)))
    r1, r2 = errs[16] / errs[64], errs[64] / errs[256]
    assert 1.5 < r1 < 2.7 and 1.5 < r2 < 2.7, (name, errs)
