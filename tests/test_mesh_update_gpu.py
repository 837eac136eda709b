"""trb_scene_update_mesh on an H100: after an update the scene must be indistinguishable, bit for bit, from trb_scene_create on the
description with the new arrays — the mesh tree (and the oracle's tree for that description), per-sample radiance and every counter
in both shadow modes, the film, and intersection records, occlusion and illumination on camera and incoherent rays. Covered: a
heightfield updated from one seed to another and back, identical arrays, normals or texcoords alone on a textured mesh, a mesh
under two instances (one keyframed) moved out of its old bounds with the frame built on the device and on the host, the wide leaf
form, the host-build fallback, device arrays on a torch side stream, Whitted and NormalsDebug, failures that leave the scene as it
was, the 35 M-triangle heightfield, and a one-device trb_group."""
import ctypes as C
import gc

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle import pyoracle as O
from oracle_queries import pyqueries as Q
from test_queries_cpu import query_rays, random_rays

pytestmark = pytest.mark.gpu
COUNTERS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation", "node_tests", "tri_tests", "inst_tests"]
GRID = 256
SEED_A, SEED_B = 0x4E16F1D, 0x1234567
FRAME = (0, 0.0, 0.0)


def heightfield(seed, grid=GRID, shift=0.0):
    p, n, t, i = SB.heightfield_mesh(grid, seed)
    p = p.copy()
    p[:, 1] += np.float32(shift)
    return p, n, t, i


def checker(k=16):
    y, x = np.mgrid[0:k, 0:k]
    px = np.zeros((k, k, 4), np.uint8)
    px[..., 0] = np.where((x + y) % 2, 230, 30)
    px[..., 1] = (x * 255 // (k - 1)).astype(np.uint8)
    px[..., 2] = (y * 255 // (k - 1)).astype(np.uint8)
    px[..., 3] = 255
    return px


def scene(mesh, integrator=F.INTEGRATOR_PATH, textured=False, keyframed=False, w=48, h=32, spp=4):
    """the Cornell walls and light around one mesh instance; keyframed adds a second, moving instance of the same mesh"""
    b = SB.SceneBuilder(w, h, spp, 3, 6)
    b.integrator = (integrator, 3, 6)
    mats = SB.cornell_walls(b)
    SB.cornell_light(b, mats["white"])
    m = b.add_mesh(*mesh)
    tex = b.add_texture(checker()) if textured else 0
    mat = b.add_material(F.MAT_MATTE, (0.74, 0.74, 0.73), roughness=1.0, tex_c0=tex)
    b.receiver(F.SHAPE_MESH, mat, [SB.trs()], mesh=m)
    if keyframed:
        anim = SB.Anim([(( -3, 0, 0), (0, 0, 0, 1), (0.5, 0.5, 0.5)), ((0, 2, 2), (0, 0, 0, 1), (0.5, 0.5, 0.5)),
                        ((3, 1, 0), (0, 0, 0, 1), (0.5, 0.5, 0.5)), ((4, -1, 1), (0, 0, 0, 1), (0.5, 0.5, 0.5))])
        b.receiver(F.SHAPE_MESH, mat, [anim], mesh=m)
    b.add_camera([SB.trs(t=(0, 12, -60))], fov=30.0)
    return b.finish()


def rmse(a, b):
    """films accumulate with float atomics, so two renders of one scene agree to rounding only"""
    return float(np.sqrt(np.mean((a.astype(np.float64) - b) ** 2)))


def counters(st):
    return [getattr(st, k) for k in COUNTERS]


def ray_sets(g, frame=FRAME, n_random=8192, seed=5):
    _, start, end = frame
    t1 = start + 0.5 * (end - start)
    cam, _ = g.camera_rays(spp=1, seed=seed)
    times = np.random.default_rng(seed).uniform(start, t1, size=len(cam)).astype(np.float32)
    q = np.concatenate([query_rays(cam, times), random_rays(n_random, seed, (-14, 1, -10), (14, 23, 18), start, t1)])
    il = np.zeros(len(q), F.ILLUM_RAY_DTYPE)
    for k in ("o", "d", "min_t", "max_t", "time"):
        il[k] = q[k]
    il["key"] = np.arange(len(q), dtype=np.uint32)
    return q, il


def assert_same(u, f, frame=FRAME, spp=2, n_meshes=1, film=True, queries=True):
    """U (updated) against F (fresh) on everything a caller can observe"""
    for i in range(n_meshes):
        (un, uo), (fn, fo) = u.bvh(i), f.bvh(i)
        assert un.tobytes() == fn.tobytes() and uo.tobytes() == fo.tobytes(), i
    for flags in (F.RENDER_STATS, F.RENDER_STATS | F.RENDER_REFERENCE_SHADOW):
        (us, ust), (fs, fst) = u.render_samples(flags=flags, spp=spp, seed=3), f.render_samples(flags=flags, spp=spp, seed=3)
        assert us.tobytes() == fs.tobytes(), flags
        assert counters(ust) == counters(fst), flags
    if film:
        (uf, _), (ff, _) = u.render(spp=spp, seed=7), f.render(spp=spp, seed=7)
        assert rmse(uf, ff) < 1e-5
    if queries:
        q, il = ray_sets(f, frame)
        (ur, ust), (fr, fst) = u.intersect_records(q, stats=True), f.intersect_records(q, stats=True)
        assert ur.tobytes() == fr.tobytes() and counters(ust) == counters(fst)
        for ref in (False, True):
            assert np.array_equal(u.occluded(q, reference=ref)[0], f.occluded(q, reference=ref)[0])
        sa, sb = F.Stats(), F.Stats()
        assert u.illumination(il, spp=2, stats=sa).tobytes() == f.illumination(il, spp=2, stats=sb).tobytes()
        assert counters(sa) == counters(sb)


def fresh(desc, frame=FRAME):
    f = api.Scene(desc)
    f.update_frame(*frame)
    return f


def test_heightfield_seed_a_to_b_and_back():
    ma, mb = heightfield(SEED_A), heightfield(SEED_B)
    da, db = scene(ma), scene(mb)
    u = api.Scene(da)
    u.update_frame(*FRAME)
    before = u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3)
    u.update_mesh(0, *mb[:3])
    f = fresh(db)
    assert_same(u, f)
    on, oo = O.OracleScene(db).bvh(0)
    un, uo = u.bvh(0)
    assert un.tobytes() == on.tobytes() and uo.tobytes() == oo.tobytes()
    q, _ = ray_sets(f)
    o = Q.QueryOracleScene(db)
    o.update_frame(*FRAME)
    assert u.intersect_records(q)[0].tobytes() == o.intersect_records(q)[0].tobytes()
    u.update_mesh(0, *ma[:3])
    assert_same(u, fresh(da))
    after = u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3)
    assert after[0].tobytes() == before[0].tobytes() and counters(after[1]) == counters(before[1])


def test_identical_arrays_change_nothing():
    ma = heightfield(SEED_A)
    u, f = fresh(scene(ma)), fresh(scene(ma))
    u.update_mesh(0, *ma[:3])
    assert_same(u, f)


def test_normals_then_texcoords_only_on_a_textured_mesh():
    ma, mb = heightfield(SEED_A), heightfield(SEED_B)
    u = fresh(scene(ma, textured=True))
    tree = u.bvh(0)
    u.update_mesh(0, normals=mb[1])
    assert u.bvh(0)[0].tobytes() == tree[0].tobytes()
    assert_same(u, fresh(scene((ma[0], mb[1], ma[2], ma[3]), textured=True)))
    uv = np.ascontiguousarray(ma[2][::-1])
    u.update_mesh(0, texcoords=uv)
    assert u.bvh(0)[0].tobytes() == tree[0].tobytes()
    assert_same(u, fresh(scene((ma[0], mb[1], uv, ma[3]), textured=True)))


@pytest.mark.parametrize("frame_device", [1, 0])
def test_shared_mesh_with_a_keyframed_instance_moved_out_of_its_bounds(frame_device):
    frame = (0, 0.0, 1.0)
    ma, moved = heightfield(SEED_A, 128), heightfield(SEED_A, 128, shift=5.0)
    u = api.Scene(scene(ma, keyframed=True))
    u.set_option("frame.device", frame_device)
    u.update_frame(*frame)
    u.update_mesh(0, positions=moved[0])
    f = api.Scene(scene(moved, keyframed=True))
    f.set_option("frame.device", frame_device)
    f.update_frame(*frame)
    assert_same(u, f, frame)
    # hits above the old bounds: the instance bounds and the TLAS were refreshed
    q, _ = ray_sets(f, frame)
    rec = u.intersect_records(q)[0]
    hit_mesh = (rec["inst"] >= 6) & (rec["inst"] != 0xffffffff)  # instances 6 and 7: five walls and the light come first
    assert np.any(hit_mesh & (rec["p"][:, 1] > float(ma[0][:, 1].max()) + 0.5))


def test_update_before_the_first_frame():
    frame = (0, 0.0, 1.0)
    ma, moved = heightfield(SEED_A, 128), heightfield(SEED_A, 128, shift=5.0)
    u = api.Scene(scene(ma, keyframed=True))
    u.update_mesh(0, positions=moved[0])
    u.update_frame(*frame)
    assert_same(u, fresh(scene(moved, keyframed=True), frame), frame)


def test_wide_leaf_form_and_toggling_it_after_an_update():
    ma, mb = heightfield(SEED_A), heightfield(SEED_B)
    u = api.Scene(scene(ma))
    u.set_option("trace.wide_leaf", 1)
    u.update_frame(*FRAME)
    u.update_mesh(0, *mb[:3])
    f = api.Scene(scene(mb))
    f.set_option("trace.wide_leaf", 1)
    f.update_frame(*FRAME)
    assert_same(u, f, film=False)
    u.set_option("trace.wide_leaf", 0)
    f.set_option("trace.wide_leaf", 0)
    assert_same(u, f, film=False)
    u.update_mesh(0, *ma[:3])
    u.set_option("trace.wide_leaf", 1)
    g = api.Scene(scene(ma))
    g.set_option("trace.wide_leaf", 1)
    g.update_frame(*FRAME)
    assert_same(u, g, film=False, queries=False)


def test_host_build_fallback_gives_the_device_bytes(monkeypatch):
    ma, mb = heightfield(SEED_A), heightfield(SEED_B)
    monkeypatch.setenv("TRB_BUILD_DEVICE", "0")
    h = fresh(scene(ma))
    monkeypatch.delenv("TRB_BUILD_DEVICE")
    h.update_mesh(0, *mb[:3])
    d = fresh(scene(ma))
    d.update_mesh(0, *mb[:3])
    assert_same(h, d, film=False)
    assert_same(h, fresh(scene(mb)), film=False, queries=False)


def test_device_arrays_on_a_side_stream_equal_the_host_form():
    import torch
    ma, mb = heightfield(SEED_A), heightfield(SEED_B)
    u, h = fresh(scene(ma)), fresh(scene(ma))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        dp, dn, dt = (torch.from_numpy(np.ascontiguousarray(a)).to("cuda", non_blocking=False) * 1.0 for a in mb[:3])
    u.update_mesh_device(0, dp.data_ptr(), dn.data_ptr(), dt.data_ptr(), stream=s.cuda_stream)
    h.update_mesh(0, *mb[:3])
    assert_same(u, h, film=False)


@pytest.mark.parametrize("integrator", [F.INTEGRATOR_WHITTED, F.INTEGRATOR_NORMALS_DEBUG])
def test_whitted_and_normals_debug(integrator):
    ma, mb = heightfield(SEED_A, 128), heightfield(SEED_B, 128)
    u = fresh(scene(ma, integrator))
    u.update_mesh(0, *mb[:3])
    f = fresh(scene(mb, integrator))
    (ua, ust), (fa, fst) = u.render(spp=2, seed=5), f.render(spp=2, seed=5)
    assert rmse(ua, fa) < 1e-5 and counters(ust) == counters(fst)
    assert u.bvh(0)[0].tobytes() == f.bvh(0)[0].tobytes()
    q, _ = ray_sets(f)
    assert u.intersect_records(q)[0].tobytes() == f.intersect_records(q)[0].tobytes()


def test_failures_leave_the_scene_as_it_was():
    ma = heightfield(SEED_A, 128)
    u = fresh(scene(ma))
    before = u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3)
    tree = u.bvh(0)
    bad = ma[0].copy()
    bad[: len(bad) // 2, 0] = np.inf  # the x centroids of half the triangles: one bucket, a split with an empty child
    with pytest.raises(api.TrbError) as e:
        u.update_mesh(0, positions=bad)
    assert e.value.status == F.TRB_INVALID_ARG and "infinite coordinates" in str(e.value)
    # trb_scene_create rejects the same description with the same status and message
    with pytest.raises(api.TrbError) as e2:
        api.Scene(scene((bad, ma[1], ma[2], ma[3])))
    assert e2.value.status == e.value.status and str(e2.value) == str(e.value)
    after = u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3)
    assert after[0].tobytes() == before[0].tobytes() and counters(after[1]) == counters(before[1])
    assert u.bvh(0)[0].tobytes() == tree[0].tobytes()
    lib = F.load_trb()
    assert lib.trb_scene_update_mesh(u._h, 1, F.ptr(ma[0]), None, None) == F.TRB_INVALID_ARG
    assert lib.trb_scene_update_mesh_device(u._h, 7, None, None, None, None) == F.TRB_INVALID_ARG
    assert lib.trb_scene_update_mesh(u._h, 0, None, None, None) == F.TRB_OK
    # trace.quads reads DQuad records, which an updated mesh does not have
    q = fresh(scene(ma))
    q.set_option("trace.quads", 1)
    q.render(spp=1)
    q.update_mesh(0, positions=ma[0])
    with pytest.raises(api.TrbError) as e3:
        q.render(spp=1)
    assert e3.value.status == F.TRB_UNSUPPORTED
    q.set_option("trace.quads", 0)
    assert_same(q, fresh(scene(ma)), film=False, queries=False)


@pytest.mark.parametrize("build_device", ["1", "0"])
def test_record_buffer_grows_from_a_collapsed_mesh_and_back(build_device, monkeypatch):
    """15 triangles collapsed onto one point are one leaf (no interior node, an empty record buffer); spread out they need interior
    records, so the update must replace the buffer with a larger one. Device build and the host fallback (TRB_BUILD_DEVICE=0)."""
    spread = SB.random_triangle_mesh(15, 9)
    collapsed = (np.zeros_like(spread[0]),) + spread[1:]
    monkeypatch.setenv("TRB_BUILD_DEVICE", build_device)
    u = fresh(scene(collapsed))
    root, _ = u.bvh(0)
    assert len(root) == 1 and root[0]["b"] & F.BVH_LEAF
    u.update_mesh(0, positions=spread[0])
    f = fresh(scene(spread))
    assert len(f.bvh(0)[0]) > 1
    assert_same(u, f, film=False)
    u.update_mesh(0, positions=collapsed[0])
    assert_same(u, fresh(scene(collapsed)), film=False)


def fits_narrow(nodes):
    leaf = (nodes["b"] & F.BVH_LEAF) != 0
    return not np.any(leaf & (((nodes["b"] & ~np.uint32(F.BVH_LEAF)) > 31) | (nodes["a"] >= (1 << 25))))


def test_leaf_form_changes_with_the_tree():
    """A mesh of 2^25 + 1 triangles: a 4097 x 4097 heightfield and one triangle far away. At -x the SAH build puts that triangle
    first and every leaf fits the narrow reference; at +x it becomes the last leaf, alone at slot 2^25, which only the wide
    reference addresses. Updating between the two switches the scene's leaf form both ways (the device packer's narrow-fit test,
    then every mesh re-packed), and each state must equal a fresh scene."""
    grid = 4097
    p, n, t, i = SB.heightfield_mesh(grid, SEED_A)
    tri = np.array([[0, 10, 0], [0, 11, 0], [0, 10, 1]], np.float32)
    idx = np.concatenate([i, np.arange(len(p), len(p) + 3, dtype=np.uint32)[None, :]])
    nrm = np.concatenate([n, np.tile(np.array([[1, 0, 0]], np.float32), (3, 1))])
    uv = np.concatenate([t, np.zeros((3, 2), np.float32)])
    pos = {side: np.concatenate([p, tri + np.float32([side * 1000.0, 0, 0])]) for side in (-1, 1)}
    del p, n, t, i
    assert len(idx) == (1 << 25) + 1

    def reference(side):
        f = fresh(scene((pos[side], nrm, uv, idx)))
        nodes, order = f.bvh(0)
        q, _ = ray_sets(f, n_random=1 << 16)
        out = (nodes.tobytes().__hash__(), order.tobytes().__hash__(), fits_narrow(nodes), q, f.intersect_records(q, stats=True),
               f.render_samples(flags=F.RENDER_STATS, spp=2, seed=3, block_start=4, block_count=8))
        f.close()
        return out

    def check(u, ref):
        nodes, order = u.bvh(0)
        assert (nodes.tobytes().__hash__(), order.tobytes().__hash__()) == ref[:2]
        r = u.intersect_records(ref[3], stats=True)
        assert r[0].tobytes() == ref[4][0].tobytes() and counters(r[1]) == counters(ref[4][1])
        s = u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3, block_start=4, block_count=8)
        assert s[0].tobytes() == ref[5][0].tobytes() and counters(s[1]) == counters(ref[5][1])

    narrow_ref, wide_ref = reference(-1), reference(1)
    gc.collect()
    assert narrow_ref[2] and not wide_ref[2]
    u = fresh(scene((pos[-1], nrm, uv, idx)))
    u.update_mesh(0, positions=pos[1])
    check(u, wide_ref)
    u.update_mesh(0, positions=pos[-1])
    check(u, narrow_ref)


def test_heightfield_35m_triangles():
    grid = 4200
    desc_b = SB.scene_heightfield(grid, 64, 48, 2, seed=SEED_B).finish()
    f = fresh(desc_b)
    fn, fo = f.bvh(0)
    digest = (fn.tobytes().__hash__(), fo.tobytes().__hash__())
    q, _ = ray_sets(f, n_random=1 << 18)
    q = q[: 1 << 18] if len(q) > (1 << 18) else q
    rec = f.intersect_records(q, stats=True)
    sam = f.render_samples(flags=F.RENDER_STATS, spp=2, seed=3, block_start=8, block_count=16)
    f.close()
    del f, fn, fo, desc_b
    gc.collect()
    mb = SB.heightfield_mesh(grid, SEED_B)
    u = fresh(SB.scene_heightfield(grid, 64, 48, 2, seed=SEED_A).finish())
    u.update_mesh(0, *mb[:3])
    del mb
    un, uo = u.bvh(0)
    assert (un.tobytes().__hash__(), uo.tobytes().__hash__()) == digest
    del un, uo
    r = u.intersect_records(q, stats=True)
    assert r[0].tobytes() == rec[0].tobytes() and counters(r[1]) == counters(rec[1])
    s = u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3, block_start=8, block_count=16)
    assert s[0].tobytes() == sam[0].tobytes() and counters(s[1]) == counters(sam[1])


def test_one_device_group_updated_through_its_replica():
    ma, mb = heightfield(SEED_A, 128), heightfield(SEED_B, 128)
    da, db = scene(ma), scene(mb)
    ga, gb = api.Group(da, [0]), api.Group(db, [0])
    lib = F.load_trb()
    rep = lib.trb_group_scene(ga._h, 0)
    assert rep
    pos = np.ascontiguousarray(mb[0])
    nrm, uv = np.ascontiguousarray(mb[1]), np.ascontiguousarray(mb[2])
    assert lib.trb_scene_update_mesh(rep, 0, F.ptr(pos), F.ptr(nrm), F.ptr(uv)) == F.TRB_OK, lib.trb_last_error()
    (fa, sa), (fb, sb) = ga.render(spp=2, seed=3), gb.render(spp=2, seed=3)
    assert rmse(fa, fb) < 1e-5 and counters(sa) == counters(sb)
