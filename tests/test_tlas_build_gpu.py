"""The frame's instance tree built by the level builder on an H100 (DESIGN.md §4 "`update_frame` on the device"): the bytes of the
one-thread build (option frame.tlas_min forces either builder) on the shipped scene shapes, on instance-heavy scenes in sphere and mesh
form and on bounds in the zero planes, none of which is -0; the oracle's and the host path's tree at 100 000 instances; the edit calls on 20 000
instances against freshly created scenes; coincident instances and bounds no build would end on; and no device allocation per frame."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle_queries import pyqueries as Q
from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from test_mesh_update_gpu import counters
from test_queries_cpu import random_rays

pytestmark = pytest.mark.gpu
LEVEL, ONE_THREAD = 0, 1 << 40  # frame.tlas_min: the level builder for every scene / for none
SCENES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scenes")
FRAME = (0, 0.0, 0.0)


def observe(s, transforms=True):
    """what a caller sees of a frame: the tree, every instance's transform, per-sample radiance with the counters, hit records"""
    nodes, order = s.bvh(-1)
    out = [nodes.tobytes(), order.tobytes()]
    if transforms:
        out += [a.tobytes() for i in range(s.n_instances) for a in s.transform(i)]
    samples, st = s.render_samples(flags=F.RENDER_STATS, spp=1, seed=3)
    rec, rst = s.intersect_records(random_rays(1 << 14, 3, (-14, 1, -10), (14, 23, 18), 0.0, 0.0), stats=True)
    return out + [samples.tobytes(), counters(st), rec.tobytes(), counters(rst)]


def both_builders(desc, frame=FRAME, transforms=True):
    s = api.Scene(desc)
    seen = []
    for tlas_min in (LEVEL, ONE_THREAD):
        s.set_option("frame.tlas_min", tlas_min)
        s.update_frame(*frame)
        seen.append(observe(s, transforms))
    s.close()
    assert seen[0] == seen[1]
    nodes = np.frombuffer(seen[0][0], F.NODE_DTYPE)
    boxes = np.concatenate([nodes["bmin"], nodes["bmax"]], axis=1)
    # no bound is -0, which is why the level builder's zero rule and the one-thread kernel's cannot differ on instance bounds
    assert not np.any((boxes == 0) & np.signbit(boxes))
    return seen[0]


def zero_ties():
    """rectangles and disks in the planes x = 0, y = 0 and z = 0, facing both ways, some mirrored by a negative scale and some translated
    by -0: products that are -0 abound, and every bound that is zero must still come out +0 (DESIGN.md §4)"""
    b = SB.SceneBuilder(32, 32, 1, 2, 4)
    m = b.add_material(F.MAT_MATTE, (0.7, 0.7, 0.7), roughness=1.0)
    turns = [((0, 1, 0), 0), ((0, 1, 0), 180), ((0, 1, 0), 90), ((0, 1, 0), -90), ((1, 0, 0), 90), ((1, 0, 0), -90)]
    for k, (axis, deg) in enumerate(turns * 4):
        q = SB.quat_axis_angle(axis, deg)
        s = (-1.0, 1.0, 1.0) if k % 3 == 0 else ((1.0, -1.0, -1.0) if k % 5 == 0 else (1.0, 1.0, 1.0))
        if k % 2:
            b.receiver(F.SHAPE_RECT, m, [SB.trs(q=q, s=s)], p0=2.0 + k // 6, p1=2.0)
        else:
            b.receiver(F.SHAPE_DISK, m, [SB.trs(q=q, s=s)], p0=1.0 + k // 6, p1=0.0)
    for k in range(8):  # and rectangles that only touch a zero plane
        b.receiver(F.SHAPE_RECT, m, [SB.trs(t=(k - 4.0, -0.0, -0.0), s=(1, -1, -1) if k % 2 else (1, 1, 1))], p0=2.0, p1=2.0)
    for k in range(4):  # two-level stacks of mirrored, -0-translated levels
        b.receiver(F.SHAPE_RECT, m, [SB.trs(t=(-0.0, -0.0, -0.0), s=(-1, -1, -1)), SB.trs(t=(-0.0, 0, -0.0), q=SB.quat_axis_angle((0, 0, 1), 90 * k), s=(1, -1, -1))],
                   p0=2.0, p1=1.0 + k)
    b.area_light(F.SHAPE_SPHERE, m, [SB.trs(t=(3, 6, -3))], (1, 1, 1, 30), p0=1.0)
    b.add_camera([SB.trs(t=(2, 3, -20))], fov=40.0)
    return b


def test_shipped_scene_shapes_have_the_same_bytes_from_both_builders():
    for name in ("c1_cornell_box.json", "c2_smallpt.json"):
        lib, dp = F.load_trb(), C.POINTER(F.SceneDesc)()
        assert lib.trb_desc_load_json(os.path.join(SCENES, name).encode(), 48, 48, 1, C.byref(dp)) == F.TRB_OK, name
        try:
            both_builders(dp.contents)
        finally:
            lib.trb_desc_free(dp)
    both_builders(SB.scene_materials_zoo(48, 48, 1, SB.synthetic_merl_table()).finish())
    anim = SB.scene_animated(48, 48, 1, frames=6, scene_time=1.5).finish()
    assert both_builders(anim, (1, 0.25, 0.5)) != both_builders(anim, (4, 1.0, 1.25))


def test_bounds_in_the_zero_planes_are_plus_zero_and_equal_from_both_builders():
    seen = both_builders(zero_ties().finish())  # asserts that no bound is -0
    nodes = np.frombuffer(seen[0], F.NODE_DTYPE)
    assert np.count_nonzero(nodes["bmin"] == 0) and np.count_nonzero(nodes["bmax"] == 0)


def test_fewer_than_five_instances_through_the_level_builder():
    """a root that is a leaf (one node, no record) and roots that take the n < 5 sort"""
    for n in (1, 2, 3, 4):
        b = SB.SceneBuilder(32, 32, 1, 2, 4)
        m = b.add_material(F.MAT_MATTE, (0.7, 0.7, 0.7), roughness=1.0)
        b.area_light(F.SHAPE_SPHERE, m, [SB.trs(t=(0, 6, 0))], (1, 1, 1, 30), p0=1.0)
        for k in range(n - 1):
            b.receiver(F.SHAPE_SPHERE, m, [SB.trs(t=(3.0 * k - 3, 0, k))], p0=1.0)
        b.add_camera([SB.trs(t=(0, 2, -20))], fov=40.0)
        seen = both_builders(b.finish())
        assert n > 1 or len(np.frombuffer(seen[0], F.NODE_DTYPE)) == 1


@pytest.mark.parametrize("mesh", [False, True], ids=["spheres", "mesh_instances"])
def test_instance_counts_around_every_case_of_the_build(mesh):
    for k in (1, 2, 4, 5, 33, 1000, 3000, 20_000):
        both_builders(SB.scene_instances(k, 21 + k, 32, 32, 1, mesh=mesh).finish(), transforms=k <= 1000)


def test_hundred_thousand_instances_against_the_oracle_and_the_host_path():
    desc = SB.scene_instances(100_000, 5, 64, 64, 1).finish()
    o = Q.QueryOracleScene(desc)
    o.update_frame(*FRAME)
    on, oo = o.bvh(-1)
    g = api.Scene(desc)
    g.set_option("frame.tlas_min", LEVEL)
    trees = {}
    for dev in (1, 0):
        g.set_option("frame.device", dev)
        g.update_frame(*FRAME)
        trees[dev] = g.bvh(-1)
        assert trees[dev][0].tobytes() == on.tobytes() and np.array_equal(trees[dev][1], oo), dev
    g.set_option("frame.device", 1)
    gs, gst = g.render_samples(flags=F.RENDER_STATS, spp=1, seed=6)
    assert gs.tobytes() == o.render_samples(spp=1, seed=6)[0].tobytes()
    # the oracle walks shadow rays as the reference does: the counters are its own in that mode
    ref = F.RENDER_STATS | F.RENDER_REFERENCE_SHADOW
    (rs, rst), (os_, ost) = g.render_samples(flags=ref, spp=1, seed=6), o.render_samples(flags=ref, spp=1, seed=6)
    assert rs.tobytes() == os_.tobytes() and counters(rst) == counters(ost)
    q = random_rays(1 << 14, 3, (-14, 1, -10), (14, 23, 18), 0.0, 0.0)
    level = g.intersect_records(q, stats=True)
    assert np.count_nonzero(level[0]["inst"] >= 6) > 1000  # the spheres are hit
    orec, ost = o.intersect_records(q)
    assert level[0].tobytes() == orec.tobytes() and counters(level[1]) == counters(ost)
    g.set_option("frame.device", 0)  # the host-built tree answers the same
    host = g.intersect_records(q, stats=True)
    assert level[0].tobytes() == host[0].tobytes() and counters(level[1]) == counters(host[1])
    hs, hst = g.render_samples(flags=F.RENDER_STATS, spp=1, seed=6)
    assert hs.tobytes() == gs.tobytes() and counters(hst) == counters(gst)


def test_edit_calls_on_twenty_thousand_instances_match_fresh_scenes():
    import torch
    k, first = 20_000, 11  # five walls (two levels each) and the light come first
    b = SB.scene_instances(k, 9, 32, 32, 1)
    u = api.Scene(b.finish())
    u.set_option("frame.tlas_min", LEVEL)
    u.update_frame(*FRAME)

    def fresh():
        f = api.Scene(b.finish())
        f.set_option("frame.tlas_min", ONE_THREAD if len(b.instances) < 1000 else LEVEL)
        f.update_frame(*FRAME)
        seen = observe(f, transforms=len(b.instances) < 1000)
        f.close()
        return seen
    rng = np.random.default_rng(10)
    new = [SB.trs(t=rng.uniform((-13, 1, -8), (13, 22, 18)), s=0.3) for _ in range(k)]
    d = torch.from_numpy(np.array(new, F.KEYFRAME_DTYPE).view(np.float32).reshape(k, 10).copy()).cuda()
    u.update_keyframes_device(first, k, d.data_ptr())
    b.keyframes[first:first + k] = new
    assert observe(u, False) == fresh()
    for t in rng.uniform((-13, 1, -8), (13, 22, 18), size=(k, 3)):  # grown to 40 000
        b.receiver(F.SHAPE_SPHERE, 3, [SB.trs(t=t, s=0.3)], p0=1.0)
    u.replace_objects(b.objects())
    assert u.n_instances == 6 + 2 * k and observe(u, False) == fresh()
    small = SB.scene_instances(5, 9, 32, 32, 1)  # shrunk to 5 receivers: the same meshes (none) and materials
    b = small
    u.replace_objects(b.objects())
    assert u.n_instances == 11 and observe(u) == fresh()
    u.close()


def test_level_builder_first_run_on_a_shrunk_scene_then_grown_within_the_capacity():
    """the level builder's scratch is sized by the scene's instance capacity, not by the frame that first runs it"""
    b = SB.scene_instances(1000, 4, 32, 32, 1)
    u = api.Scene(b.finish())
    u.set_option("frame.tlas_min", ONE_THREAD)
    u.update_frame(*FRAME)  # capacity for 1006 instances, built by one thread
    u.replace_objects(SB.scene_instances(5, 4, 32, 32, 1).objects())
    u.set_option("frame.tlas_min", LEVEL)  # the level builder's first frame: 11 instances
    grown = SB.scene_instances(900, 6, 32, 32, 1)
    u.replace_objects(grown.objects())  # 906 instances, within the capacity
    f = api.Scene(grown.finish())
    f.set_option("frame.tlas_min", ONE_THREAD)
    f.update_frame(*FRAME)
    assert observe(u) == observe(f)
    u.check_error()


def test_coincident_instances_and_refused_bounds():
    b = SB.SceneBuilder(32, 32, 1, 2, 4)
    m = b.add_material(F.MAT_MATTE, (0.7, 0.7, 0.7), roughness=1.0)
    for _ in range(40):  # coincident centroids: split in place down to leaves of fewer than four, so every leaf fits its reference
        b.receiver(F.SHAPE_SPHERE, m, [SB.trs(t=(0, 1, 0))], p0=1.0)
    b.area_light(F.SHAPE_SPHERE, m, [SB.trs(t=(3, 6, -3))], (1, 1, 1, 30), p0=1.0)
    b.add_camera([SB.trs(t=(0, 1, -20))], fov=30.0)
    seen = both_builders(b.finish())
    leaves = np.frombuffer(seen[0], F.NODE_DTYPE)["b"]
    assert max(int(x) & 0x7fffffff for x in leaves if int(x) >> 31) < 4
    # one instance infinitely far away among more than four: neither the reference's build nor bvh_build_arrays would ever end on these
    # bounds, so both builders refuse them before any serial build starts (one thread: the kernel returns before building; level
    # builder: with 7 instances before the serial subtrees, with 207 after the first level)
    for k, tlas_min in ((0, ONE_THREAD), (0, LEVEL), (200, LEVEL)):
        b = SB.scene_instances(k, 1, 32, 32, 1)
        good = b.objects()
        b.receiver(F.SHAPE_SPHERE, 3, [SB.trs(t=(float("inf"), 0, 0))], p0=1.0)
        s = api.Scene(b.finish())
        s.set_option("frame.tlas_min", tlas_min)
        with pytest.raises(api.TrbError) as e:
            s.update_frame(*FRAME)
        assert e.value.status == F.TRB_INVALID_ARG and "instance tree" in str(e.value), (k, tlas_min)
        with pytest.raises(api.TrbError):
            s.render_samples(spp=1)  # no frame is ready
    k = 200
    s.replace_objects(good)
    s.update_frame(*FRAME)
    f = api.Scene(SB.scene_instances(k, 1, 32, 32, 1).finish())
    f.update_frame(*FRAME)
    assert observe(s) == observe(f)


def test_frames_do_not_allocate_device_memory():
    import torch
    s = api.Scene(SB.scene_instances(5000, 3, 32, 32, 1).finish())
    s.set_option("frame.tlas_min", LEVEL)
    s.update_frame(*FRAME)
    torch.cuda.synchronize()
    free = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        s.update_frame(*FRAME)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free
