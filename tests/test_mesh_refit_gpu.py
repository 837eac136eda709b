"""trb_scene_refit_mesh on an H100, against the oracle refit of the same scene (oracle_refit): every mesh tree (nodes and ordered_geom,
bit for bit but for the sign of a bound tied between -0 and +0), per-sample radiance and every counter in both shadow modes, intersection
records, occlusion in both modes and illumination on camera and incoherent rays with per-ray times, and the film to rounding. Covered:
a heightfield under a travelling wave over several steps, identical positions (everything as before the call and as a fresh scene), a
mesh under a static and a keyframed instance moved out of its old bounds with the frame on the device, on the host and not yet set,
normals and texcoords alongside on a textured mesh, the wide leaf form and toggling it after a refit, Whitted and NormalsDebug, Adaptive
per-pixel counts, refit(A) then refit(B), a refit then update_mesh, replace_meshes keeping a refit mesh, the device form from a torch
side stream with a render in flight, a one-device trb_group, every failure status, and the 35 M-triangle heightfield on the wide
leaf form against the numpy restatement and the oracle."""
import gc

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_refit import pyrefit as R
from test_mesh_refit_cpu import assert_tree_equal, restated_tree
from test_mesh_update_gpu import FRAME, SEED_A, SEED_B, assert_same, counters, fresh, heightfield, ray_sets, scene

pytestmark = pytest.mark.gpu
REF = F.RENDER_STATS | F.RENDER_REFERENCE_SHADOW


def wave(p, t, amp=1.5):
    """a travelling wave on a heightfield's heights: crests move along x with t, and reach above and below the built bounds"""
    q = p.copy()
    q[:, 1] += (amp * np.sin(0.7 * p[:, 0] - 2.0 * t) * np.cos(0.3 * p[:, 2] + t)).astype(np.float32)
    return q


def image(film):
    return film[..., :3] / np.maximum(film[..., 3:], 1e-6)


def both(desc, frame=FRAME, frame_device=1, set_frame=True):
    u = api.Scene(desc)
    u.set_option("frame.device", frame_device)
    o = R.RefitOracleScene(desc)
    if set_frame:
        u.update_frame(*frame)
        o.update_frame(*frame)
    return u, o


def refit(u, o, mesh, *arrays):
    u.refit_mesh(mesh, *arrays)
    o.refit_mesh(mesh, *arrays)


def assert_matches(u, o, frame=FRAME, spp=2, meshes=(0,), film=True, queries=True, n_random=8192):
    """U (the product after refits) against O (the oracle after the same refits) on everything a caller can observe"""
    for i in meshes:
        (un, uo), (on, oo) = u.bvh(i), o.bvh(i)
        assert uo.tobytes() == oo.tobytes(), i
        assert_tree_equal(un, on)
    (us, ust), (os_, ost) = u.render_samples(flags=REF, spp=spp, seed=3), o.render_samples(spp=spp, seed=3)
    assert us.tobytes() == os_.tobytes() and counters(ust) == counters(ost)
    ds, dst = u.render_samples(flags=F.RENDER_STATS, spp=spp, seed=3)  # any-hit shadow rays: the same radiance, fewer tests
    assert ds.tobytes() == os_.tobytes() and counters(dst)[:5] == counters(ost)[:5] and dst.node_tests <= ost.node_tests
    if queries:
        q, il = ray_sets(u, frame, n_random)
        (ur, ust), (orr, ost) = u.intersect_records(q, stats=True), o.intersect_records(q)
        assert ur.tobytes() == orr.tobytes() and counters(ust)[5:] == counters(ost)[5:]
        ref_occ = o.occluded(q)[0]
        for mode in (False, True):
            assert np.array_equal(u.occluded(q, reference=mode)[0], ref_occ)
        sa, sb = F.Stats(), F.Stats()
        assert u.illumination(il, spp=2, stats=sa, reference=True).tobytes() == o.illumination(il, spp=2, stats=sb).tobytes()
        assert counters(sa) == counters(sb)
    if film:  # the film render sets its own frame (Exec::render): the caller's frame is set again afterwards
        (uf, _), (of, _) = u.render(spp=spp, seed=7), o.render(spp=spp, seed=7)
        assert np.sqrt(np.mean((image(uf) - image(of)) ** 2)) < 1e-5
        u.update_frame(*frame)
        o.update_frame(*frame)


def test_travelling_wave_over_several_steps():
    ma = heightfield(SEED_A)
    u, o = both(scene(ma))
    built, _ = u.bvh(0)
    for step in range(1, 5):
        refit(u, o, 0, wave(ma[0], 0.4 * step))
        assert_matches(u, o, queries=step == 4, film=step == 4)
    assert not np.array_equal(u.bvh(0)[0]["bmax"], built["bmax"])
    assert u.bvh(0)[0]["bmax"][0, 1] > built["bmax"][0, 1]  # the crests rose above the built root


def test_identical_positions_change_nothing():
    ma = heightfield(SEED_A)
    u = fresh(scene(ma))
    tree, order = u.bvh(0)
    before = u.render_samples(flags=REF, spp=2, seed=3)
    u.refit_mesh(0, ma[0])
    (un, uo) = u.bvh(0)
    assert un.tobytes() == tree.tobytes() and uo.tobytes() == order.tobytes()
    after = u.render_samples(flags=REF, spp=2, seed=3)
    assert after[0].tobytes() == before[0].tobytes() and counters(after[1]) == counters(before[1])
    assert_same(u, fresh(scene(ma)))


@pytest.mark.parametrize("frame_device,set_frame", [(1, True), (0, True), (1, False)])
def test_shared_mesh_with_a_keyframed_instance_moved_out_of_its_bounds(frame_device, set_frame):
    frame = (0, 0.0, 1.0)
    ma, moved = heightfield(SEED_A, 128), heightfield(SEED_A, 128, shift=5.0)
    u, o = both(scene(ma, keyframed=True), frame, frame_device, set_frame)
    refit(u, o, 0, wave(moved[0], 0.3))
    if not set_frame:
        u.update_frame(*frame)
        o.update_frame(*frame)
    assert_matches(u, o, frame)
    q, _ = ray_sets(u, frame)
    rec = u.intersect_records(q)[0]
    hit_mesh = (rec["inst"] >= 6) & (rec["inst"] != 0xffffffff)  # instances 6 and 7: five walls and the light come first
    assert np.any(hit_mesh & (rec["p"][:, 1] > float(ma[0][:, 1].max()) + 0.5))  # hits above the old bounds


def test_normals_and_texcoords_alongside_on_a_textured_mesh():
    ma, mb = heightfield(SEED_A), heightfield(SEED_B)
    u, o = both(scene(ma, textured=True))
    uv = np.ascontiguousarray(ma[2][::-1])
    refit(u, o, 0, wave(ma[0], 1.0), mb[1], uv)
    assert_matches(u, o)
    refit(u, o, 0, None, ma[1], None)  # attributes alone: the tree stays
    assert_matches(u, o, queries=False)


def test_wide_leaf_form_and_toggling_it_after_a_refit():
    ma = heightfield(SEED_A)
    u, o = both(scene(ma))
    u.set_option("trace.wide_leaf", 1)
    refit(u, o, 0, wave(ma[0], 0.5))
    assert_matches(u, o, film=False)
    u.set_option("trace.wide_leaf", 0)  # re-packs every mesh from its host tree, which the refit left stale
    assert_matches(u, o, film=False, queries=False)
    refit(u, o, 0, wave(ma[0], 1.5))
    u.set_option("trace.wide_leaf", 1)
    assert_matches(u, o, film=False)


@pytest.mark.parametrize("integrator", [F.INTEGRATOR_WHITTED, F.INTEGRATOR_NORMALS_DEBUG])
def test_whitted_and_normals_debug(integrator):
    ma = heightfield(SEED_A, 128)
    u, o = both(scene(ma, integrator))
    refit(u, o, 0, wave(ma[0], 0.8))
    assert_matches(u, o, queries=False)
    q, _ = ray_sets(u)
    assert u.intersect_records(q)[0].tobytes() == o.intersect_records(q)[0].tobytes()


def test_adaptive_per_pixel_counts_after_a_refit():
    ma = heightfield(SEED_A, 128)
    desc = scene(ma)
    u = api.Scene(desc)
    a = R.AdaptiveRefitOracleScene(desc)
    u.update_frame(*FRAME)
    a.update_frame(*FRAME)
    p = wave(ma[0], 0.6)
    u.refit_mesh(0, p)
    a.refit_mesh(0, p)
    (uf, us, ust), (of, os_, ost) = u.render_adaptive(2, 16, seed=3), a.render_adaptive(2, 16, seed=3)
    assert np.array_equal(us, os_)
    assert np.sqrt(np.mean((image(uf) - image(of)) ** 2)) < 1e-5


def test_refit_a_then_b_equals_refit_b_alone():
    ma = heightfield(SEED_A)
    pa, pb = wave(ma[0], 0.3, 3.0), wave(ma[0], 2.1)
    u, v = fresh(scene(ma)), fresh(scene(ma))
    u.refit_mesh(0, pa)
    u.refit_mesh(0, pb)
    v.refit_mesh(0, pb)
    assert_same(u, v)


def test_refit_then_update_mesh_equals_a_fresh_scene():
    ma, mb = heightfield(SEED_A), heightfield(SEED_B)
    u = fresh(scene(ma))
    u.refit_mesh(0, wave(ma[0], 0.7))
    u.update_mesh(0, *mb[:3])
    assert_same(u, fresh(scene(mb)))
    u.refit_mesh(0, wave(mb[0], 0.2))  # a refit after the rebuild runs on the new topology
    o = R.RefitOracleScene(scene(mb))
    o.update_frame(*FRAME)
    o.refit_mesh(0, wave(mb[0], 0.2))
    assert_matches(u, o, film=False)


def test_replace_meshes_keeping_a_refit_mesh():
    ma, mb = heightfield(SEED_A, 128), SB.icosphere_mesh(3, radius=3.0)
    b = SB.SceneBuilder(48, 32, 4, 3, 6)
    mats = SB.cornell_walls(b)
    SB.cornell_light(b, mats["white"])
    m0 = b.add_mesh(*ma)
    m1 = b.add_mesh(mb[0] + np.float32([0, 10, 0]), *mb[1:])
    b.receiver(F.SHAPE_MESH, mats["white"], [SB.trs()], mesh=m0)
    b.receiver(F.SHAPE_MESH, mats["white"], [SB.trs()], mesh=m1)
    b.add_camera([SB.trs(t=(0, 12, -60))], fov=30.0)
    desc = b.finish()
    u, o = both(desc)
    p = wave(ma[0], 0.9)
    refit(u, o, 0, p)
    # keep both meshes in swapped order (the refit one moves with its records, boxes and stale host tree), instances renumbered
    b.meshes[0], b.meshes[1] = b.meshes[1], b.meshes[0]
    b.instances = [it[:4] + (1 - it[4],) + it[5:] if it[1] == F.SHAPE_MESH else it for it in b.instances]
    sec = b.meshes_section()
    assert list(sec.keep[:2]) == [1, 0]
    u.replace_meshes(sec, b.objects())
    u.update_frame(*FRAME)
    assert_tree_equal(u.bvh(1)[0], o.bvh(0)[0])
    assert u.bvh(1)[1].tobytes() == o.bvh(0)[1].tobytes() and u.bvh(0)[0].tobytes() == o.bvh(1)[0].tobytes()
    (us, ust), (os_, ost) = u.render_samples(flags=REF, spp=2, seed=3), o.render_samples(spp=2, seed=3)
    assert us.tobytes() == os_.tobytes() and counters(ust) == counters(ost)
    q, _ = ray_sets(u)
    assert u.intersect_records(q)[0]["t"].tobytes() == o.intersect_records(q)[0]["t"].tobytes()


def test_device_form_from_a_side_stream_equals_the_host_form_with_a_render_in_flight():
    import torch
    ma, mb = heightfield(SEED_A), heightfield(SEED_B)
    u, h = fresh(scene(ma)), fresh(scene(ma))
    p = wave(ma[0], 1.2)
    film = torch.zeros((u.height, u.width, 4), dtype=torch.float32, device="cuda")
    render_stream, s = torch.cuda.Stream(), torch.cuda.Stream()
    u.render_device(film.data_ptr(), stream=render_stream.cuda_stream, spp=4, seed=5)  # still running while the refit starts
    with torch.cuda.stream(s):
        dp, dn = (torch.from_numpy(np.ascontiguousarray(a)).to("cuda", non_blocking=False) * 1.0 for a in (p, mb[1]))
    u.refit_mesh_device(0, dp.data_ptr(), dn.data_ptr(), None, stream=s.cuda_stream)
    h.refit_mesh(0, p, mb[1])
    torch.cuda.synchronize()
    u.update_frame(*FRAME)  # the render set its own frame, which the refit re-ran
    assert_same(u, h, film=False)
    o = R.RefitOracleScene(scene(ma))
    o.update_frame(*FRAME)
    o.refit_mesh(0, p, mb[1])
    assert_matches(u, o, film=False, queries=False)


def test_one_device_group_refit_through_its_replica():
    ma = heightfield(SEED_A, 128)
    desc = scene(ma)
    g = api.Group(desc, [0])
    lib = F.load_trb()
    rep = lib.trb_group_scene(g._h, 0)
    assert rep
    p = np.ascontiguousarray(wave(ma[0], 0.4))
    assert lib.trb_scene_refit_mesh(rep, 0, F.ptr(p), None, None) == F.TRB_OK, lib.trb_last_error()
    o = R.RefitOracleScene(desc)
    o.refit_mesh(0, p)
    (gf, gst), (of, ost) = g.render(spp=2, seed=3), o.render(spp=2, seed=3)
    assert np.sqrt(np.mean((image(gf) - image(of)) ** 2)) < 1e-5
    assert (gst.camera_samples, gst.rays_primary, gst.rays_continuation) == (ost.camera_samples, ost.rays_primary, ost.rays_continuation)


def lit_mesh(mesh):
    """one mesh instance under the area light: two instances, few enough for the instance tree to take infinite bounds"""
    b = SB.SceneBuilder(48, 32, 4, 3, 6)
    mat = b.add_material(F.MAT_MATTE, (0.74, 0.74, 0.73), roughness=1.0)
    SB.cornell_light(b, mat)
    b.receiver(F.SHAPE_MESH, mat, [SB.trs()], mesh=b.add_mesh(*mesh))
    b.add_camera([SB.trs(t=(0, 12, -60))], fov=30.0)
    return b.finish()


def test_failure_statuses_and_positions_a_rebuild_refuses():
    ma = heightfield(SEED_A, 128)
    u, o = both(scene(ma))
    lib = F.load_trb()
    assert lib.trb_scene_refit_mesh(None, 0, F.ptr(ma[0]), None, None) == F.TRB_INVALID_ARG
    assert lib.trb_scene_refit_mesh(u._h, 1, F.ptr(ma[0]), None, None) == F.TRB_INVALID_ARG
    assert lib.trb_scene_refit_mesh_device(u._h, 7, None, None, None, None) == F.TRB_INVALID_ARG
    assert lib.trb_scene_refit_mesh(u._h, 0, None, None, None) == F.TRB_OK
    assert lib.trb_scene_refit_mesh_device(u._h, 0, None, None, None, None) == F.TRB_OK
    assert_matches(u, o, queries=False, film=False)
    # trace.quads reads DQuad records, which a refit mesh does not have
    refit(u, o, 0, wave(ma[0], 0.5))
    u.set_option("trace.quads", 1)
    with pytest.raises(api.TrbError) as e:
        u.render(spp=1)
    assert e.value.status == F.TRB_UNSUPPORTED
    u.set_option("trace.quads", 0)
    u.update_frame(*FRAME)
    assert_matches(u, o, film=False, queries=False)
    # infinite x on half the vertices (and NaN on a few): the SAH build refuses such a mesh (an empty split), the refit takes it
    bad = ma[0].copy()
    bad[: len(bad) // 2, 0] = np.inf
    bad[len(bad) // 2: len(bad) // 2 + 7] = np.nan
    with pytest.raises(api.TrbError) as e:
        api.Scene(lit_mesh((bad, ma[1], ma[2], ma[3])))
    assert "infinite coordinates" in str(e.value)
    v, w = both(lit_mesh(ma))
    with pytest.raises(api.TrbError):
        v.update_mesh(0, positions=bad)
    refit(v, w, 0, bad)
    assert_matches(v, w, film=False)
    # among more than four instances the frame's instance tree refuses infinite bounds (trb_scene_update_frame's rule): the mesh is
    # refit and the re-run frame returns that status (the oracle, whose instance tree would not end, is refit without a frame)
    u2 = fresh(scene(ma))
    o2 = R.RefitOracleScene(scene(ma))
    with pytest.raises(api.TrbError) as e:
        u2.refit_mesh(0, bad)
    assert e.value.status == F.TRB_INVALID_ARG and "instance tree cannot be built" in str(e.value)
    o2.refit_mesh(0, bad)
    assert_tree_equal(u2.bvh(0)[0], o2.bvh(0)[0])


def test_heightfield_35m_triangles_on_the_wide_form():
    grid = 4200
    desc = SB.scene_heightfield(grid, 64, 48, 2, seed=SEED_A).finish()
    u = fresh(desc)
    u.set_option("trace.wide_leaf", 1)
    built, order = u.bvh(0)
    mesh = desc.meshes[0]
    p0 = np.ctypeslib.as_array(mesh.positions, (mesh.n_verts * 3,)).reshape(-1, 3)
    idx = np.ctypeslib.as_array(mesh.indices, (mesh.n_tris * 3,)).reshape(-1, 3)
    p = wave(p0, 0.5)
    u.refit_mesh(0, p)
    got, got_order = u.bvh(0)
    assert got_order.tobytes() == order.tobytes()
    assert_tree_equal(got, restated_tree(built, order, p, idx))
    del got, got_order, built
    gc.collect()
    o = R.RefitOracleScene(desc)
    o.update_frame(*FRAME)
    o.refit_mesh(0, p)
    q, _ = ray_sets(u, n_random=1 << 18)
    q = q[: 1 << 18]
    (ur, ust), (orr, ost) = u.intersect_records(q, stats=True), o.intersect_records(q)
    assert ur.tobytes() == orr.tobytes() and counters(ust)[5:] == counters(ost)[5:]
    for start, count in ((0, 4), (8, 16), (40, 8)):
        (us, ust), (os_, ost) = (x.render_samples(spp=2, seed=3, block_start=start, block_count=count, **k)
                                 for x, k in ((u, dict(flags=REF)), (o, {})))
        assert us.tobytes() == os_.tobytes() and counters(ust) == counters(ost)

