"""Wide mesh leaf references on an H100 (DESIGN.md §4 "Mesh leaf forms"): a mesh leaf reference without a count, whose leaf ends at
the triangle carrying the leaf mark, so that a mesh may hold up to 2^30 triangles instead of 2^25.

  * The option trace.wide_leaf 1 puts every scene on the wide form: radiance, counters and every query must equal the default
    (narrow) form and the oracle bit for bit, on the small scenes of the query tests, on C4, and through the megakernel.
  * A 35 M-triangle heightfield (more than 2^25 triangles, refused before the wide form) is created, its queries and sampled
    render ranges equal the oracle bit for bit, and the accepted hits include triangles stored at leaf slots >= 2^25.
  * On a wide scene the option-selected experimental trace variants return TRB_UNSUPPORTED.
"""
import resource
import time

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_queries import pyqueries as Q
from test_gpu_fullsize import check_ranges, one_call_frame
from test_illumination_gpu import SCENES, both, counters, ray_set as illum_ray_set, same_bits
from test_queries_cpu import random_rays
from test_queries_gpu import ray_set as query_ray_set

pytestmark = pytest.mark.gpu
TESTS = ["node_tests", "tri_tests", "inst_tests"]
RAYS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation"]


def wide_scene(desc, frame):
    w = api.Scene(desc)
    w.set_option("trace.wide_leaf", 1)
    w.update_frame(*frame)
    return w


def check_queries(w, o, q, iq, frame, g=None):
    """intersect_records, occluded (both modes) and illumination on w against the oracle; trb_intersect against g's if given"""
    orec, ost = o.intersect_records(q)
    wrec, wst = w.intersect_records(q, stats=True)
    assert wrec.tobytes() == orec.tobytes(), [f for f in F.INTERSECTION_DTYPE.names if wrec[f].tobytes() != orec[f].tobytes()]
    assert w.intersect_records(q)[0].tobytes() == orec.tobytes()
    assert counters(wst, TESTS) == counters(ost, TESTS)
    oocc, oost = o.occluded(q)
    ref, rst = w.occluded(q, reference=True, stats=True)
    anyh, ast = w.occluded(q, stats=True)
    assert (ref == oocc).all() and (anyh == oocc).all() and (w.occluded(q)[0] == oocc).all()
    assert counters(rst, TESTS) == counters(oost, TESTS) and ast.node_tests <= rst.node_tests
    if g is not None:
        rays = np.zeros(len(q), F.RAY_DTYPE)
        for k in ("o", "d", "min_t", "max_t"):
            rays[k] = q[k]
        (wh, whs), (gh, ghs) = w.intersect(rays), g.intersect(rays)
        assert wh.tobytes() == gh.tobytes() and counters(whs, TESTS) == counters(ghs, TESTS)
    if iq is not None:
        ost = F.Stats()
        want = o.illumination(iq, spp=3, seed=5, stats=ost)
        rst = F.Stats()
        assert same_bits(w.illumination(iq, spp=3, seed=5, stats=rst, reference=True), want)
        assert counters(rst, RAYS + TESTS) == counters(ost, RAYS + TESTS)
        assert same_bits(w.illumination(iq, spp=3, seed=5), want)


@pytest.mark.parametrize("name", sorted(SCENES))
def test_forced_wide_form_equals_the_default_form_and_the_oracle(name):
    desc, frame = SCENES[name]()
    g, o = both(desc, frame)
    w = wide_scene(desc, frame)
    check_ranges(w, o, [(0, 0)], 4, 7, frame=frame[0])                    # every block: radiance in both shadow modes, counters, film
    kw = dict(spp=4, seed=7, current_frame=frame[0], flags=F.RENDER_STATS | F.RENDER_REFERENCE_SHADOW)
    (ws, wst), (gs, gst) = w.render_samples(**kw), g.render_samples(**kw)
    assert ws.tobytes() == gs.tobytes() and counters(wst, RAYS + TESTS) == counters(gst, RAYS + TESTS)
    mk = dict(kw, flags=kw["flags"] | F.RENDER_MEGAKERNEL)
    (wm, wmst), (os_, ost) = w.render_samples(**mk), o.render_samples(**dict(kw, flags=0))
    assert wm.tobytes() == os_.tobytes() and counters(wmst, RAYS + TESTS) == counters(ost, RAYS + TESTS)
    w.update_frame(*frame)
    q = query_ray_set(o, frame, 11)
    t_open = frame[1]
    q_open = q.copy()
    q_open["time"] = t_open                                                # trb_intersect traces at shutter-open time
    check_queries(w, o, q, illum_ray_set(o, frame, 11), frame)
    check_queries(w, o, q_open, None, frame, g=g)


def test_wide_option_repacks_an_existing_scene_both_ways():
    desc, frame = SCENES["zoo"]()
    g, o = both(desc, frame)
    q = query_ray_set(o, frame, 3)
    want, _ = o.intersect_records(q)
    for form in (1, 0, 1, 0):
        g.set_option("trace.wide_leaf", form)
        assert g.intersect_records(q)[0].tobytes() == want.tobytes(), form
        assert g.render_samples(spp=2, seed=3)[0].tobytes() == o.render_samples(spp=2, seed=3)[0].tobytes(), form


def test_c4_forced_wide_sampled_ranges_match_the_oracle():
    desc = SB.scene_c4(1_000_000, 1920, 1080, 4096).finish()
    w, o = api.Scene(desc), Q.QueryOracleScene(desc)
    w.set_option("trace.wide_leaf", 1)
    w.update_frame(0, 0.0, 0.0); o.update_frame(0, 0.0, 0.0)
    nb = w.n_blocks()
    check_ranges(w, o, [(3000, 400), (nb // 2 - 200, 400), (nb - 600, 400)], 4, 1)
    q = random_rays(1 << 18, 21, (-14, 1, -10), (14, 23, 18), 0.0, 0.0)
    check_queries(w, o, q, None, (0, 0.0, 0.0))


def test_statuses_on_a_wide_scene():
    desc, frame = SCENES["zoo"]()
    w = wide_scene(desc, frame)
    w.render(spp=2, seed=1)
    for name, value in [("trace.quads", 1), ("trace.sched", 0)] + [("trace.pipe", p) for p in (0, 1, 33, 34, 35, 37)]:
        w.set_option(name, value)
        with pytest.raises(api.TrbError) as e:
            w.render(spp=2, seed=1)
        assert e.value.status == F.TRB_UNSUPPORTED and "trace.wide_leaf" in str(e.value), (name, value)
        w.set_option(name, {"trace.quads": 0, "trace.sched": 6, "trace.pipe": 36}[name])
    w.render(spp=2, seed=1)
    w.set_option("trace.wide_leaf", 0)                                  # a scene that fits the narrow form goes back to it
    w.set_option("trace.pipe", 0)
    w.render(spp=2, seed=1)


def test_heightfield_of_35m_triangles_matches_the_oracle():
    """A 4200 x 4200-vertex heightfield: 35 263 202 triangles, more than 2^25 (the narrow form's limit)."""
    t0 = time.perf_counter()
    desc = SB.scene_heightfield(4200, 1920, 1080, 4).finish()
    t1 = time.perf_counter()
    assert desc.meshes[0].n_tris == 2 * 4199 ** 2 > (1 << 25)
    import torch
    free0, _ = torch.cuda.mem_get_info(0)
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    g = api.Scene(desc)
    t2 = time.perf_counter()
    free1, _ = torch.cuda.mem_get_info(0)
    rss1 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    o = Q.QueryOracleScene(desc)
    t3 = time.perf_counter()
    print("heightfield: generate %.1f s, trb_scene_create %.1f s (device memory %.2f GB, peak host RSS %.2f -> %.2f GB), oracle build %.1f s"
          % (t1 - t0, t2 - t1, (free0 - free1) / 1e9, rss0 / 1e6, rss1 / 1e6, t3 - t2))
    frame = (0, 0.0, 0.0)
    g.update_frame(*frame); o.update_frame(*frame)
    # the scene is on the wide form whatever the option says: the experimental variants are refused
    g.set_option("trace.wide_leaf", 0)
    g.set_option("trace.pipe", 0)
    with pytest.raises(api.TrbError) as e:
        g.render(spp=1, seed=1, block_count=1)
    assert e.value.status == F.TRB_UNSUPPORTED
    g.set_option("trace.pipe", 36)
    # triangles at slots >= 2^25 of the build order, and rays from the camera to their centroids
    nodes, order = g.bvh(0)
    on, oo = o.bvh(0)
    assert nodes.tobytes() == on.tobytes() and np.array_equal(order, oo)
    slot_of = np.empty(len(order), np.int64)
    slot_of[order] = np.arange(len(order))
    mi = [i for i in range(desc.n_instances) if desc.instances[i].shape == F.SHAPE_MESH][0]
    far = order[(1 << 25):][np.random.default_rng(1).permutation(len(order) - (1 << 25))[:8192]]
    p = np.ctypeslib.as_array(desc.meshes[0].positions, shape=(desc.meshes[0].n_verts * 3,)).reshape(-1, 3)
    ix = np.ctypeslib.as_array(desc.meshes[0].indices, shape=(desc.meshes[0].n_tris * 3,)).reshape(-1, 3)
    aim = p[ix[far]].mean(axis=1)
    aimed = np.zeros(len(far), F.QUERY_RAY_DTYPE)
    aimed["o"] = (0.0, 12.0, -60.0)
    aimed["d"] = aim - np.array([0.0, 12.0, -60.0], np.float32)
    aimed["max_t"] = np.inf
    cam, _ = o.camera_rays(seed=3, spp=1)                                  # every pixel, every 7th kept: 296 229 camera rays
    cq = np.zeros(len(cam), F.QUERY_RAY_DTYPE)
    for k in ("o", "d", "min_t", "max_t"):
        cq[k] = cam[k]
    q = np.concatenate([cq[::7], random_rays(1 << 17, 5, (-14, 1, -10), (14, 23, 18), 0.0, 0.0), aimed])
    assert len(q) >= 1 << 18
    check_queries(g, o, q, None, frame)
    rec, _ = g.intersect_records(q)
    on_mesh = rec["inst"] == mi
    assert (slot_of[rec["prim"][on_mesh]] >= (1 << 25)).sum() > 1000, "no accepted hit at a leaf slot >= 2^25"
    nb = g.n_blocks()
    check_ranges(g, o, [(5000, 96), (nb // 2 - 48, 96), (nb - 2000, 96)], 2, 9)
    one_call_frame(g, 1, 9)
