"""Ray queries on an H100: trb_intersect_records and trb_occluded run the render's wavefront trace kernel (k_wf_trace, PIPE bit 64)
and must equal the oracle's Scene::intersect / OcclusionTester::occluded bit for bit — every record field, and the test counters
— on C1, C2, the material zoo, the textured scene, a keyframed scene with per-ray times and C4 (1 M triangles). At shutter-open
time they must also equal trb_intersect, whose one-thread-per-ray k_intersect is an independent device traversal."""
import ctypes as C
import os

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_queries import pyqueries as Q
from test_queries_cpu import at_hit_rays, edge_rays, query_rays, random_rays
from test_textures import textured_zoo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = ["node_tests", "tri_tests", "inst_tests"]


def torch():
    import torch as t
    return t


def json_desc(name, w, h, spp):
    lib = F.load_trb()
    d = C.POINTER(F.SceneDesc)()
    assert lib.trb_desc_load_json(os.path.join(HERE, "golden", "scenes", name).encode(), w, h, spp, C.byref(d)) == F.TRB_OK, lib.trb_last_error()
    return d.contents  # kept alive for the oracle (tiny)


# name -> (description, (frame, start, end)); the shutter interval is [start, start + shutter_size * (end - start)]
SCENES = {
    "c1": lambda: (json_desc("c1_cornell_box.json", 32, 24, 2), (0, 0.0, 0.0)),
    "c2": lambda: (json_desc("c2_smallpt.json", 32, 32, 2), (0, 0.0, 0.0)),
    "zoo": lambda: (SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()).finish(), (0, 0.0, 0.0)),
    "textured": lambda: (textured_zoo(2, 32).finish(), (1, 0.5, 1.0)),
    "keyframed": lambda: (SB.scene_animated(32, 32, 2, animated_fov=True).finish(), (1, 0.25, 0.5)),
}


def both(desc, frame):
    g, o = api.Scene(desc), Q.QueryOracleScene(desc)
    g.update_frame(*frame); o.update_frame(*frame)
    return g, o


def shutter(frame):
    _, start, end = frame
    return start, start + 0.5 * (end - start)


def ray_set(o, frame, seed):
    """camera rays at spread times, incoherent rays, the edge cases, and min_t / max_t exactly at the hits"""
    t0, t1 = shutter(frame)
    rays, _ = o.camera_rays(seed=seed)
    times = np.random.default_rng(seed).uniform(t0, t1, size=len(rays)).astype(np.float32)
    q = np.concatenate([query_rays(rays, times), random_rays(8192, seed, (-14, 1, -10), (14, 23, 18), t0, t1), edge_rays(t0)])
    rec, _ = o.intersect_records(q)
    return np.concatenate([q, at_hit_rays(q, rec)])


def counters_of(st):
    return [getattr(st, k) for k in TESTS]


@pytest.mark.parametrize("name", sorted(SCENES))
def test_records_and_occlusion_match_the_oracle(name):
    desc, frame = SCENES[name]()
    g, o = both(desc, frame)
    q = ray_set(o, frame, 11)
    orec, ost = o.intersect_records(q)
    grec, _ = g.intersect_records(q)
    grec_s, gst = g.intersect_records(q, stats=True)
    assert grec.tobytes() == orec.tobytes(), "fields differ: %s" % [f for f in F.INTERSECTION_DTYPE.names if grec[f].tobytes() != orec[f].tobytes()]
    assert grec_s.tobytes() == orec.tobytes()
    assert counters_of(gst) == counters_of(ost) and gst.rays_primary == len(q) and gst.rays_shadow == 0
    hit = orec["inst"] != F.MISS
    assert 0.1 < hit.mean() < 1.0
    # occlusion: the same booleans in both modes; the reference mode's counters are the oracle's, any-hit tests no more nodes
    oocc, oost = o.occluded(q)
    ref, rst = g.occluded(q, reference=True, stats=True)
    anyh, ast = g.occluded(q, stats=True)
    assert (oocc == hit).all() and (ref == oocc).all() and (anyh == oocc).all()
    assert counters_of(rst) == counters_of(oost) and rst.rays_shadow == len(q) and rst.rays_primary == 0
    assert ast.node_tests <= rst.node_tests and ast.rays_shadow == len(q)
    assert (g.occluded(q)[0] == oocc).all()


@pytest.mark.parametrize("exact_box", [0, 1])
def test_shutter_open_records_equal_trb_intersect(exact_box):
    """k_wf_trace (refill, phased micro-steps, box_hit_finite or the literal box test, RayHome) against k_intersect hit for hit"""
    for name in ("zoo", "keyframed", "c1"):
        desc, frame = SCENES[name]()
        g, o = both(desc, frame)
        g.set_option("trace.exact_box", exact_box)
        q = ray_set(o, frame, 12)
        q["time"] = shutter(frame)[0]  # trb_intersect traces at the frame's shutter-open time
        rays = np.zeros(len(q), F.RAY_DTYPE)
        for k in ("o", "d", "min_t", "max_t"):
            rays[k] = q[k]
        hits, hst = g.intersect(rays)
        rec, st = g.intersect_records(q, stats=True)
        assert rec["t"].tobytes() == hits["t"].tobytes(), name
        assert (rec["inst"] == hits["inst"]).all() and (rec["prim"] == hits["prim"]).all(), name
        assert counters_of(st) == counters_of(hst), name


def test_c4_incoherent_rays_match_the_oracle():
    desc = SB.scene_c4(1_000_000, 64, 64, 1).finish()
    g, o = both(desc, (0, 0.0, 0.0))
    q = random_rays(1 << 20, 21, (-14, 1, -10), (14, 23, 18), 0.0, 0.0)
    orec, ost = o.intersect_records(q)
    grec, gst = g.intersect_records(q, stats=True)
    assert grec.tobytes() == orec.tobytes()
    assert counters_of(gst) == counters_of(ost)
    occ, _ = g.occluded(q)
    assert (occ == (orec["inst"] != F.MISS)).all()


def test_device_variants_equal_the_host_variants_and_do_not_wait():
    T = torch()
    desc, frame = SCENES["keyframed"]()
    g, o = both(desc, frame)
    q = ray_set(o, frame, 13)
    n = len(q)
    hrec, hst = g.intersect_records(q, stats=True)
    hocc, host = g.occluded(q, stats=True)
    dev = T.device("cuda:0")
    d_rays = T.from_numpy(q.view(np.uint8).copy()).to(dev)
    d_rec = T.zeros(n * F.INTERSECTION_DTYPE.itemsize, dtype=T.uint8, device=dev)
    d_occ = T.zeros(n, dtype=T.uint8, device=dev)
    d_st = T.zeros(9, dtype=T.int64, device=dev)
    s = T.cuda.Stream()
    s.wait_stream(T.cuda.current_stream())
    with T.cuda.stream(s):
        T.cuda._sleep(2_000_000_000)  # about a second of GPU time ahead of the queries
    g.intersect_records_device(n, d_rays.data_ptr(), d_rec.data_ptr(), d_st.data_ptr(), s.cuda_stream, stats=True)
    g.occluded_device(n, d_rays.data_ptr(), d_occ.data_ptr(), d_st.data_ptr(), s.cuda_stream, stats=True)
    assert not s.query(), "the calls waited for their stream"
    s.synchronize()
    g.check_error()
    assert d_rec.cpu().numpy().tobytes() == hrec.tobytes()
    assert (d_occ.cpu().numpy().astype(bool) == hocc).all()
    st = F.Stats.from_buffer_copy(d_st.cpu().numpy().tobytes())
    assert counters_of(st) == [a + b for a, b in zip(counters_of(hst), counters_of(host))]
    assert st.rays_primary == n and st.rays_shadow == n


def test_many_small_passes_give_the_bytes_of_one_pass():
    desc, frame = SCENES["keyframed"]()
    g, o = both(desc, frame)
    q = ray_set(o, frame, 14)
    one, st1 = g.intersect_records(q, stats=True)
    occ1, _ = g.occluded(q, reference=True)
    g.set_option("pass.paths", 1000)  # rounded up to 1024 rays per pass
    assert len(q) > 4 * 1024
    many, st2 = g.intersect_records(q, stats=True)
    occ2, _ = g.occluded(q, reference=True)
    assert many.tobytes() == one.tobytes() and counters_of(st2) == counters_of(st1) and (occ2 == occ1).all()


def test_statuses():
    T = torch()
    desc, frame = SCENES["zoo"]()
    fresh = api.Scene(desc)
    q = random_rays(64, 1, (-1, 1, -1), (1, 2, 1), 0.0, 0.0)
    for call in (lambda: fresh.intersect_records(q), lambda: fresh.occluded(q)):
        with pytest.raises(api.TrbError) as e:
            call()
        assert e.value.status == F.TRB_INVALID_ARG and "Update frame must be called before rendering" in str(e.value)
    fresh.update_frame(*frame)
    rec, st = fresh.intersect_records(q[:0])
    assert len(rec) == 0 and st.rays_primary == 0
    assert len(fresh.occluded(q[:0])[0]) == 0
    fresh.intersect_records_device(0, None, None)
    fresh.occluded_device(0, None, None)
    d = T.zeros(64 * 96 + 16, dtype=T.uint8, device="cuda:0")
    with pytest.raises(api.TrbError) as e:
        fresh.intersect_records_device(1, d.data_ptr() + 4, d.data_ptr())  # rays not 16-byte aligned
    assert e.value.status == F.TRB_INVALID_ARG
