"""trb_scene_replace_meshes on an H100: after a replacement the scene U must be indistinguishable from F, trb_scene_create on the
builder's description (and update_frame with the same arguments), on everything test_scene_edit_gpu's assert_edited observes plus every
mesh tree. Covered: a mesh added with an instance and removed with it, an unused mesh added and removed without an object section,
frames built on the device, on the host and not at all, a mesh's topology changed (the record buffer grows and shrinks), meshes
permuted, a call that keeps every mesh and builds nothing, Whitted and NormalsDebug, trace.wide_leaf, the host-build fallback,
trace.quads on new meshes and after removing a mesh update_mesh rebuilt, a mesh of 2^25 + 1 triangles that switches the leaf form and
back, the device form from a side stream and its index check, every failure status, twenty random replacements among the other edits
with the Adaptive counts, device memory after 200 add / remove cycles, a render in flight on a side stream, and a one-device group."""
import ctypes as C
import gc

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from test_mesh_update_gpu import FRAME, SEED_A, counters, ray_sets, rmse
from test_scene_edit_gpu import ANIM_FRAME, MAT_MESH, MAT_SPHERE, assert_edited, base, mat
from test_scene_objects_gpu import FLY, MESH_INST, rebind, snapshot

pytestmark = pytest.mark.gpu


class Meshed:
    """scene U and the builder of its description: replace() hands U the builder's mesh list (and object section), fresh() creates F"""

    def __init__(self, b, frame=FRAME, frame_device=1, set_frame=True, options=()):
        self.b, self.frame, self.options = b, frame, (("frame.device", frame_device),) + tuple(options)
        self.u = self._scene(set_frame)

    def _scene(self, set_frame=True):
        s = api.Scene(self.b.finish())
        for name, value in self.options:
            s.set_option(name, value)
        if set_frame:
            s.update_frame(*self.frame)
        return s

    def replace(self, objects=True):
        self.u.replace_meshes(self.b.meshes_section(), self.b.objects() if objects else None)
        assert self.u._desc.n_meshes == len(self.b.meshes) and self.u.n_instances == len(self.b.instances)

    def fresh(self):
        return self._scene()

    def check(self, **kw):
        f = self.fresh()
        assert_edited(self.u, f, self.frame, **kw)
        self.u.update_frame(*self.frame)  # the film render set its own frame (Exec::render)


def trees(u):
    """the TLAS and every mesh tree, nodes and order, as bytes"""
    return [b"".join(a.tobytes() for a in u.bvh(i)) for i in range(-1, u._desc.n_meshes)]


def section(meshes, keep):
    """a trb_scene_meshes of the given arrays with an explicit keep list"""
    t = SB.SceneBuilder()
    t.meshes = list(meshes)
    s = t.meshes_section()
    for i, k in enumerate(keep):
        s.keep[i] = k
    return s


def ball(subdiv=2, seed=11):
    return SB.icosphere_mesh(subdiv, 1.3, 0.2, seed)


@pytest.mark.parametrize("how", ["device_frame", "host_frame", "before_first_frame"])
def test_meshes_added_and_removed_with_and_without_their_instances(how):
    b = base()
    e = Meshed(b, frame_device=0 if how == "host_frame" else 1, set_frame=how != "before_first_frame")
    before = snapshot(e.u) if how != "before_first_frame" else None
    unused = b.add_mesh(*ball(1, 3))  # an unused mesh, no object section
    e.replace(objects=False)
    if how == "before_first_frame":
        with pytest.raises(api.TrbError):  # no frame was set, so none was built
            e.u.render_samples(spp=1)
        e.u.update_frame(*e.frame)
        before = None
    e.check()
    m = b.add_mesh(*ball())  # a mesh and an instance of it in one call
    b.receiver(F.SHAPE_MESH, MAT_MESH, [SB.trs(t=(-4, 14, 0), q=SB.quat_axis_angle((0, 0, 1), 30), s=2)], mesh=m)
    e.replace()
    e.check()
    b.remove_instance(len(b.instances) - 1)  # removed with its instance
    b.remove_mesh(m)
    e.replace()
    e.check()
    b.remove_mesh(unused)
    e.replace(objects=False)
    e.check(film=False)
    if before is not None:
        assert snapshot(e.u) == before


def test_topology_changed_grows_and_shrinks_the_records():
    b = base()
    e = Meshed(b)
    for subdiv in (1, 3, 0):
        b.set_mesh(0, *SB.icosphere_mesh(subdiv, 1.0, 0.1, 7))
        e.replace(objects=False)
        assert len(e.u.bvh(0)[1]) == 20 * 4 ** subdiv
        e.check()


def test_meshes_permuted_and_a_call_that_keeps_every_mesh_builds_nothing():
    b = base()
    for k in range(2):
        m = b.add_mesh(*ball(k + 1, k))
        b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(-6 + 6 * k, 16, 3), s=2)], mesh=m)
    e = Meshed(b)
    perm = [2, 0, 1]  # new mesh i is old mesh perm[i]
    b.meshes = [b.meshes[j] for j in perm]
    for i, it in enumerate(b.instances):
        if it[1] == F.SHAPE_MESH:
            rebind(b, i, mesh=perm.index(it[4]))
    s = b.meshes_section()
    assert list(s.keep[:3]) == perm
    e.u.replace_meshes(s, b.objects())
    e.check()
    lib = F.load_trb()
    n0 = lib.trb_launch_count()
    e.u.replace_meshes(b.meshes_section(), None)
    replaced = lib.trb_launch_count() - n0
    n0 = lib.trb_launch_count()
    e.u.update_frame(*e.frame)
    assert replaced == lib.trb_launch_count() - n0
    e.check(film=False)


@pytest.mark.parametrize("integrator", [F.INTEGRATOR_WHITTED, F.INTEGRATOR_NORMALS_DEBUG])
def test_whitted_and_normals_debug(integrator):
    b = base(integrator)
    e = Meshed(b)
    m = b.add_mesh(*ball())
    b.receiver(F.SHAPE_MESH, MAT_MESH, [SB.Anim(FLY, degree=2)], mesh=m)
    b.remove_instance(MESH_INST)
    b.remove_mesh(0)
    e.replace()
    f = e.fresh()
    (ua, ust), (fa, fst) = e.u.render(spp=2, seed=5), f.render(spp=2, seed=5)
    assert rmse(ua, fa) < 1e-5 and counters(ust) == counters(fst)
    assert trees(e.u) == trees(f)
    q, _ = ray_sets(f)
    assert e.u.intersect_records(q)[0].tobytes() == f.intersect_records(q)[0].tobytes()


def test_wide_leaf_form():
    b = base()
    e = Meshed(b, options=(("trace.wide_leaf", 1),))
    m = b.add_mesh(*ball())
    b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(-4, 14, 0), s=2)], mesh=m)
    e.replace()
    e.check()


def test_host_build_fallback_gives_the_device_bytes(monkeypatch):
    b = base()
    monkeypatch.setenv("TRB_BUILD_DEVICE", "0")
    e = Meshed(b)
    monkeypatch.delenv("TRB_BUILD_DEVICE")
    m = b.add_mesh(*ball(3))
    b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(-4, 14, 0), s=2)], mesh=m)
    b.set_mesh(0, *SB.icosphere_mesh(1, 1.0, 0.1, 7))
    e.replace()
    e.check(film=False)


def test_trace_quads_on_new_meshes_and_after_removing_an_updated_mesh():
    b = base()
    m = b.add_mesh(*ball(1))
    b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(-4, 14, 0), s=2)], mesh=m)
    e = Meshed(b, options=(("trace.quads", 1),))
    n = b.add_mesh(*ball(3, 5))
    b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(4, 16, 2), s=2)], mesh=n)
    e.replace()
    assert snapshot(e.u) == snapshot(e.fresh())
    p, nn, t, i = b.meshes[m]
    e.u.update_mesh(m, p * np.float32(1.1))  # rebuilt without DQuad records: trace.quads refuses the scene
    with pytest.raises(api.TrbError) as ex:
        e.u.render(spp=1)
    assert ex.value.status == F.TRB_UNSUPPORTED
    b.remove_instance(len(b.instances) - 2)
    b.remove_mesh(m)
    e.replace()
    e.u.render(spp=1)
    e.u.update_frame(*e.frame)
    assert snapshot(e.u) == snapshot(e.fresh())


def test_a_mesh_of_2_25_plus_1_triangles_switches_the_leaf_form_and_back():
    """The mesh of test_mesh_update_gpu's leaf-form test with its lone triangle at +x, the last leaf alone at slot 2^25: only the wide
    reference addresses it, so adding it re-packs every mesh of the scene in the wide form and removing it re-packs them narrow."""
    p, n, t, i = SB.heightfield_mesh(4097, SEED_A)
    tri = np.array([[1000, 10, 0], [1000, 11, 0], [1000, 10, 1]], np.float32)
    big = (np.concatenate([p, tri]), np.concatenate([n, np.tile(np.array([[1, 0, 0]], np.float32), (3, 1))]),
           np.concatenate([t, np.zeros((3, 2), np.float32)]), np.concatenate([i, np.arange(len(p), len(p) + 3, dtype=np.uint32)[None, :]]))
    del p, n, t, i
    assert len(big[3]) == (1 << 25) + 1
    b = base()
    m = b.add_mesh(*big)
    b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(0, 2, 0), s=0.5)], mesh=m)
    f = api.Scene(b.finish())
    f.update_frame(*FRAME)
    digest = [hash(x) for x in trees(f)]
    q, _ = ray_sets(f, n_random=1 << 16)
    ref = (f.intersect_records(q, stats=True), f.render_samples(flags=F.RENDER_STATS, spp=2, seed=3, block_start=4, block_count=8))
    f.close()
    del f
    gc.collect()
    b.remove_instance(len(b.instances) - 1)
    b.remove_mesh(m)
    e = Meshed(b)
    small = snapshot(e.u)
    m = b.add_mesh(*big)
    b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(0, 2, 0), s=0.5)], mesh=m)
    e.replace()
    assert [hash(x) for x in trees(e.u)] == digest
    r = e.u.intersect_records(q, stats=True)
    assert r[0].tobytes() == ref[0][0].tobytes() and counters(r[1]) == counters(ref[0][1])
    s = e.u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3, block_start=4, block_count=8)
    assert s[0].tobytes() == ref[1][0].tobytes() and counters(s[1]) == counters(ref[1][1])
    b.remove_instance(len(b.instances) - 1)
    b.remove_mesh(m)
    e.replace()
    assert snapshot(e.u) == small
    e.check(film=False)


def device_section(meshes, keep, stream):
    """a trb_scene_meshes whose new meshes are torch tensors on the device, filled on `stream`; returns it with the tensors"""
    import torch
    s = section(meshes, keep)
    held = []
    with torch.cuda.stream(stream):
        for k, (p, n, t, i) in enumerate(meshes):
            if keep[k] != F.MESH_NEW:
                continue
            arrays = [torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).to("cuda", non_blocking=False) for a in (p, n, t, i)]
            held += arrays
            m = s.meshes[k]
            m.positions, m.normals, m.texcoords = (C.cast(a.data_ptr(), C.POINTER(F.f32)) for a in arrays[:3])
            m.indices = C.cast(arrays[3].data_ptr(), C.POINTER(F.u32))
    return s, held


def test_device_form_from_a_side_stream_and_its_index_check():
    import torch
    b = base()
    e = Meshed(b)
    before, tree = snapshot(e.u), trees(e.u)
    st = torch.cuda.Stream()
    for bad in (7, 44):  # a 15-triangle mesh: 45 indices, 11 vector loads and a one-index tail
        p, n, t, i = SB.random_triangle_mesh(15, 9)
        i = i.copy()
        i.reshape(-1)[bad] = len(p)
        s, held = device_section([b.meshes[0], (p, n, t, i)], [0, F.MESH_NEW], st)
        with pytest.raises(api.TrbError) as ex:
            e.u.replace_meshes_device(s, stream=st.cuda_stream)
        assert ex.value.status == F.TRB_INVALID_ARG and "mesh index out of range" in str(ex.value)
        assert snapshot(e.u) == before and trees(e.u) == tree
    m = b.add_mesh(*ball(3))
    b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(-4, 14, 0), s=2)], mesh=m)
    b.set_mesh(0, *SB.random_triangle_mesh(15, 9))
    s, held = device_section(b.meshes, [F.MESH_NEW, F.MESH_NEW], st)
    e.u.replace_meshes_device(s, b.objects(), stream=st.cuda_stream)
    e.check()


def two_meshes():
    """base() with a second mesh and an instance of it"""
    b = base()
    m = b.add_mesh(*ball())
    b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(-4, 14, 0), s=2)], mesh=m)
    return b, m


def test_failures_leave_the_scene_as_it_was():
    b, m = two_meshes()
    e = Meshed(b, (1, 0.0, 0.0))
    u, lib = e.u, F.load_trb()
    before, tree = snapshot(u), trees(u)

    def unchanged():
        assert snapshot(u) == before and trees(u) == tree and u._desc.n_meshes == 2 and u.n_instances == len(b.instances)

    def fails(sec, objects=None, status=F.TRB_INVALID_ARG, desc=None):
        with pytest.raises(api.TrbError) as ex:
            u.replace_meshes(sec, objects)
        assert ex.value.status == status
        if desc is not None:  # trb_scene_create refuses that description alike
            with pytest.raises(api.TrbError) as ex2:
                api.Scene(desc)
            assert ex2.value.status == status and str(ex.value) == str(ex2.value)
        unchanged()
        return str(ex.value)

    # test_mesh_update_gpu's input: the x centroids of half of 32 258 triangles infinite, one bucket, a split with an empty child at
    # the root (a mesh of more than 1024 triangles, which the builder splits level by level, where it detects the empty child)
    hf = SB.heightfield_mesh(128, SEED_A)
    inf = hf[0].copy()
    inf[: len(inf) // 2, 0] = np.inf
    bad, _ = two_meshes()
    bad.set_mesh(m, inf, *hf[1:])
    assert "infinite coordinates" in fails(section(bad.meshes, [0, F.MESH_NEW]), desc=bad.finish())
    past, _ = two_meshes()
    past.meshes.pop()  # the mesh instance points past the new list
    assert "mesh index out of range" in fails(section(b.meshes[:1], [0]), desc=past.finish())
    assert "kept mesh index out of range" in fails(section(b.meshes, [0, 2]))
    assert "kept twice" in fails(section(b.meshes, [0, 0]))
    late, _ = two_meshes()
    late.cameras[0] = late.cameras[0][:4] + (2,) + late.cameras[0][5:]
    assert "no camera is active" in fails(section(b.meshes, [0, 1]), late.objects())
    empty = section(b.meshes, [0, F.MESH_NEW])
    empty.meshes[1].n_tris = 0
    assert "empty mesh" in fails(empty)
    tiny = section(b.meshes, [0, F.MESH_NEW])
    tiny.meshes[1].normals = C.cast(None, C.POINTER(F.f32))
    assert "Normals" in fails(tiny)
    nokeep = section(b.meshes, [0, 1])
    nokeep.keep = C.cast(None, C.POINTER(F.u32))
    assert lib.trb_scene_replace_meshes(u._h, C.byref(nokeep), None) == F.TRB_INVALID_ARG
    nomeshes = section(b.meshes, [0, F.MESH_NEW])
    nomeshes.meshes = C.cast(None, C.POINTER(F.Mesh))
    assert lib.trb_scene_replace_meshes(u._h, C.byref(nomeshes), None) == F.TRB_INVALID_ARG
    assert lib.trb_scene_replace_meshes(u._h, None, None) == F.TRB_INVALID_ARG
    unchanged()
    e.replace()
    e.check()


def test_twenty_random_replacements_among_the_other_edits_then_adaptive_counts():
    b = base()
    b.receiver(F.SHAPE_SPHERE, MAT_SPHERE, [SB.Anim(FLY, degree=2)], p0=1.0)
    e = Meshed(b, ANIM_FRAME)
    rng = np.random.default_rng(22)
    for step in range(20):
        op = step % 4 if len(b.meshes) > 1 else 0
        if op == 0:  # a new mesh and an instance of it, keyframed or not
            m = b.add_mesh(*SB.icosphere_mesh(int(rng.integers(0, 3)), float(rng.uniform(0.5, 1.5)), 0.15, int(rng.integers(1 << 30))))
            xf = [SB.Anim([(tuple(np.add(t, rng.uniform(-2, 2, 3))), q, s) for t, q, s in FLY], degree=int(rng.integers(1, 4)))] \
                if rng.random() < 0.4 else [SB.trs(t=rng.uniform((-10, 2, -5), (10, 20, 15)), s=float(rng.uniform(0.5, 2.5)))]
            b.receiver(F.SHAPE_MESH, int(rng.choice([MAT_SPHERE, MAT_MESH])), xf, mesh=m)
        elif op == 1:  # a mesh other than the first removed with its instances
            m = int(rng.integers(1, len(b.meshes)))
            for i in reversed(range(len(b.instances))):
                if b.instances[i][1] == F.SHAPE_MESH and b.instances[i][4] == m:
                    b.remove_instance(i)
            b.remove_mesh(m)
        elif op == 2:  # a topology change
            m = int(rng.integers(0, len(b.meshes)))
            b.set_mesh(m, *SB.icosphere_mesh(int(rng.integers(0, 4)), 1.0, 0.1, int(rng.integers(1 << 30))))
        else:  # an instance bound to another mesh, and the list reversed
            i = MESH_INST
            rebind(b, i, mesh=int(rng.integers(0, len(b.meshes))))
            n = len(b.meshes)
            b.meshes.reverse()
            for k, it in enumerate(b.instances):
                if it[1] == F.SHAPE_MESH:
                    rebind(b, k, mesh=n - 1 - it[4])
        e.replace(objects=op != 2)
        if op == 0:  # and one of the edits that keep the structure, on the new section
            first = int(rng.integers(0, len(b.keyframes)))
            t, q, s = b.keyframes[first]
            b.keyframes[first] = (tuple(float(x + d) for x, d in zip(t, rng.uniform(-0.5, 0.5, 3))), q, s)
            e.u.update_keyframes(first, np.array([b.keyframes[first]], F.KEYFRAME_DTYPE))
        elif op == 1:
            b.materials[MAT_SPHERE] = mat(int(rng.integers(0, 6)), rng.uniform(0.1, 0.9, 3), rng.uniform(0.5, 3.0, 3), roughness=float(rng.uniform(0, 0.5)))
            e.u.update_materials(MAT_SPHERE, np.array([b.materials[MAT_SPHERE]], F.MATERIAL_DTYPE))
        if step in (4, 9, 14):
            e.check(film=False)
    f = e.fresh()
    assert_edited(e.u, f, ANIM_FRAME)
    (ua, us, ust), (fa, fs, fst) = e.u.render_adaptive(2, 16, seed=3), f.render_adaptive(2, 16, seed=3)
    assert us.tobytes() == fs.tobytes() and counters(ust) == counters(fst) and rmse(ua, fa) < 1e-5


def test_two_hundred_add_remove_cycles_do_not_grow_the_scene():
    import torch
    b = base()
    e = Meshed(b)
    added, removed = section([b.meshes[0], SB.icosphere_mesh(4)], [0, F.MESH_NEW]), section(b.meshes, [0])
    free = []
    for k in range(200):  # an add and a remove; each added mesh holds about 1 MB of buffers
        e.u.replace_meshes(added if k % 2 == 0 else removed)
        if k in (1, 199):
            torch.cuda.synchronize()
            free.append(torch.cuda.mem_get_info()[0])
    assert free[1] >= free[0] - (8 << 20), free
    e.check(film=False)


def test_render_in_flight_on_a_side_stream_finishes_on_the_old_meshes():
    import torch
    b = base()
    b.film.update(width=256, height=256)
    e = Meshed(b)
    ref, _ = e.fresh().render(spp=4, seed=7)
    s = torch.cuda.Stream()
    film = torch.zeros((256, 256, 4), dtype=torch.float32, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    e.u.render_device(film.data_ptr(), stream=s.cuda_stream, spp=4, seed=7)
    b.remove_instance(MESH_INST)  # frees every mesh buffer the passes in flight read
    b.remove_mesh(0)
    e.replace()
    s.synchronize()
    assert rmse(film.cpu().numpy(), ref) < 1e-5
    e.check()


def test_one_device_group_replaced_through_its_replica():
    b = base()
    ga = api.Group(b.finish(), [0])
    m = b.add_mesh(*ball())
    b.receiver(F.SHAPE_MESH, MAT_SPHERE, [SB.trs(t=(-4, 14, 0), s=2)], mesh=m)
    sec, objs = b.meshes_section(), b.objects()
    gb = api.Group(b.finish(), [0])
    lib = F.load_trb()
    rep = lib.trb_group_scene(ga._h, 0)
    assert rep
    assert lib.trb_scene_replace_meshes(rep, C.byref(sec), C.byref(objs)) == F.TRB_OK, lib.trb_last_error()
    (fa, sa), (fb, sb) = ga.render(spp=2, seed=3), gb.render(spp=2, seed=3)
    assert rmse(fa, fb) < 1e-5 and counters(sa) == counters(sb)
