"""trb_scene_replace_objects on an H100: after a replacement the scene U must be indistinguishable from F, trb_scene_create on the
description with the new object section (and update_frame with the same arguments), on everything test_scene_edit_gpu's assert_edited
observes: the TLAS and the instance transforms, per-sample radiance and every counter in both shadow modes, films, intersection
records, occlusion and illumination, the BSDF, light and emission queries and the light list. Covered: receivers, mesh instances,
area and point lights added and removed, instances bound to another material (fused and split shading, MERL), mesh, radius and kind,
static scenes that gain keyframed instances and lose them again, keyframed and second cameras, frames built on the device, on the
host and not at all, Whitted and NormalsDebug, the wide leaf form, twenty random replacements among the other edits with the Adaptive
sampler's counts, 10 -> 10 000 -> 10 instances, device memory after 200 replacements, a render in flight on a side stream, and
every failure status."""
import ctypes as C

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from test_mesh_update_gpu import FRAME, counters, ray_sets, rmse
from test_queries_cpu import random_rays
from test_scene_edit_gpu import ANIM_FRAME, MAT_MESH, MAT_SPHERE, assert_edited, base, mat

pytestmark = pytest.mark.gpu
LIGHT, SPHERE, MESH_INST = 5, 6, 7  # instances of base(): walls 0-4, light, sphere, mesh instance
FLY = [SB.trs(t=(-8, 4, 0)), SB.trs(t=(-2, 10, 4), s=1.5), SB.trs(t=(4, 6, 8)), SB.trs(t=(8, 12, 2), s=2.0)]


def stocked(integrator=F.INTEGRATOR_PATH):
    """base() with what a replacement can bind but not add: materials of four more kinds and a second mesh, all unused"""
    b = base(integrator)
    kinds = dict(plastic=b.add_material(F.MAT_PLASTIC, (0.8, 0.2, 0.2), (0.8, 0.8, 0.8), roughness=0.1),
                 glass=b.add_material(F.MAT_GLASS, (1, 1, 1), (1, 1, 1), eta=1.5),
                 metal=b.add_material(F.MAT_METAL, (0.155, 0.117, 0.138), (4.83, 3.12, 2.15), roughness=0.3),
                 merl=b.add_material(F.MAT_MERL, merl=b.add_merl_table(SB.synthetic_merl_table())))
    other = b.add_mesh(*SB.icosphere_mesh(1, 1.3, 0.2, 11))
    return b, kinds, other


def rebind(b, i, **fields):
    names = ["kind", "shape", "p0", "p1", "mesh", "material", "spline_first", "n_splines", "emission_first", "n_emission"]
    it = dict(zip(names, b.instances[i]))
    it.update(fields)
    b.instances[i] = tuple(it[k] for k in names)


class Replaced:
    """scene U and the builder of its description: replace() hands U the builder's object section, fresh() creates F from the builder"""

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

    def replace(self, b=None):
        """with b: another builder over the same meshes and materials takes over"""
        self.b = b or self.b
        self.u.replace_objects(self.b.objects())
        assert (self.u.n_instances, self.u._desc.n_keyframes) == (len(self.b.instances), len(self.b.keyframes))

    def fresh(self):
        return self._scene()

    def check(self, **kw):
        f = self.fresh()
        assert self.u.n_lights == f.n_lights and self.u.lights().tolist() == [i for i, it in enumerate(self.b.instances) if it[0] != F.INST_RECEIVER]
        assert_edited(self.u, f, self.frame, **kw)
        self.u.update_frame(*self.frame)  # the film render set its own frame (Exec::render)


def snapshot(u):
    s, st = u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3)
    return s.tobytes(), counters(st)


@pytest.mark.parametrize("how", ["device_frame", "host_frame", "before_first_frame"])
def test_a_sphere_and_a_second_mesh_instance_added_and_removed_again(how):
    b, kinds, _ = stocked()
    e = Replaced(b, frame_device=0 if how == "host_frame" else 1, set_frame=how != "before_first_frame")
    if how == "before_first_frame":
        i = b.receiver(F.SHAPE_SPHERE, MAT_SPHERE, [SB.trs(t=(0, 15, 5), s=2)], p0=1.0)
        e.replace()
        with pytest.raises(api.TrbError):  # no frame was set, so none was built
            e.u.render_samples(spp=1)
        e.u.update_frame(*e.frame)
        e.check()
        return
    before = snapshot(e.u)
    i = b.receiver(F.SHAPE_SPHERE, MAT_SPHERE, [SB.trs(t=(0, 15, 5), s=2)], p0=1.0)
    e.replace()
    assert snapshot(e.u) != before
    e.check()
    j = b.receiver(F.SHAPE_MESH, MAT_MESH, [SB.trs(t=(-4, 14, 0), q=SB.quat_axis_angle((0, 0, 1), 30), s=2)], mesh=0)
    e.replace()
    e.check()
    b.remove_instance(i)
    e.replace()
    e.check()
    b.remove_instance(j - 1)
    e.replace()
    e.check(film=False)
    assert snapshot(e.u) == before


def test_lights_added_and_the_original_one_removed():
    b, _, _ = stocked()
    e = Replaced(b)
    b.area_light(F.SHAPE_RECT, 0, [SB.trs(t=(-10, 23.8, 5), q=SB.quat_axis_angle((1, 0, 0), 90))], (0.4, 0.9, 1.0, 25), p0=4, p1=3)
    e.replace()
    assert e.u.n_lights == 2
    e.check()
    b.point_light([SB.trs(t=(8, 18, -10))], (1, 1, 1, 150))
    e.replace()
    assert e.u.lights().tolist() == [LIGHT, 8, 9]
    e.check()
    b.remove_instance(LIGHT)
    e.replace()
    assert e.u.lights().tolist() == [7, 8]
    e.check()


def test_instances_bound_to_other_materials_meshes_sizes_and_kinds():
    b, kinds, other = stocked()
    e = Replaced(b)  # all matte: the split kernels' matte instantiations
    rebind(b, SPHERE, material=kinds["glass"])  # two kinds
    e.replace()
    e.check()
    for i in range(len(b.instances)):  # one kind that is not matte: the fused kernel
        rebind(b, i, material=kinds["plastic"])
    e.replace()
    e.check()
    rebind(b, MESH_INST, material=kinds["merl"], mesh=other)  # a MERL material: split again; and the other mesh
    e.replace()
    e.check()
    for i in range(5):
        rebind(b, i, material=i % 3)
    rebind(b, SPHERE, p0=1.6, material=MAT_SPHERE)
    rebind(b, LIGHT, shape=F.SHAPE_DISK, p0=4.0, p1=1.0, material=0)
    e.replace()
    e.check()
    b.color_keys.append(((3.0, 9.0, 6.0, 1.0), 0.0))  # the sphere turns into an emitter
    rebind(b, SPHERE, kind=F.INST_EMITTER_AREA, emission_first=len(b.color_keys) - 1, n_emission=1)
    e.replace()
    assert e.u.lights().tolist() == [LIGHT, SPHERE]
    e.check()


def keyed(n_keyed=0, camera="static", emission=None, second_camera=False):
    """stocked() around n_keyed flying spheres, a static or keyframed camera, optionally keyframed emission and a camera from frame 2 on"""
    b, kinds, _ = stocked()
    if emission:  # the light, now the last object so far
        b.remove_instance(LIGHT)
        SB.cornell_light(b, 0, emission)
    for k in range(n_keyed):
        keys = [(tuple(x + 0.3 * k * s for x, s in zip(t, (1, -0.2, 0.5))), q, sc) for t, q, sc in FLY]
        b.receiver(F.SHAPE_SPHERE, kinds["plastic"] if k % 2 else MAT_SPHERE, [SB.Anim(keys, degree=2), SB.trs(s=0.6)], p0=1.0)
    if camera == "keyframed":
        b.cameras.clear()
        b.add_camera([SB.Anim([SB.trs(t=(-3, 12, -60)), SB.trs(t=(0, 13, -58), q=SB.quat_axis_angle((0, 1, 0), 3)), SB.trs(t=(4, 12, -60))], degree=2)],
                     fov=[28.0, 34.0, 30.0, 26.0], fov_degree=2)
    if second_camera:
        b.add_camera([SB.trs(t=(10, 14, -55), q=SB.quat_axis_angle((0, 1, 0), -9))], fov=35.0, active_at=2)
    return b


def test_static_scene_gains_keyframed_instances_camera_and_emission_and_loses_them():
    e = Replaced(keyed(), ANIM_FRAME)
    before = snapshot(e.u)
    e.replace(keyed(1))  # the keyframed kernel instantiations, and a per-path transform table
    e.check()
    e.replace(keyed(40, camera="keyframed"))
    e.check()
    e.replace(keyed(0, camera="keyframed"))  # no keyframed instance, but the camera still is
    e.check()
    e.replace(keyed(2, emission=[((1.0, 0.6, 0.3, 30), 0.0), ((0.3, 1.0, 0.4, 60), 0.4), ((0.4, 0.5, 1.0, 20), 0.9)]))
    e.check()
    e.replace(keyed())
    e.check(film=False)
    assert snapshot(e.u) == before


def test_second_camera_takes_over_at_its_frame():
    e = Replaced(keyed(), (0, 0.0, 0.25))
    e.replace(keyed(1, second_camera=True))
    f = e.fresh()
    rays = []
    for frame in range(4):
        for s in (e.u, f):
            s.update_frame(frame, 0.25 * frame, 0.25 * (frame + 1))
        rays.append(f.camera_rays(spp=1, seed=2)[0].tobytes())
        assert e.u.camera_rays(spp=1, seed=2)[0].tobytes() == rays[-1]
        assert snapshot(e.u) == snapshot(f), frame
    assert rays[1] != rays[2]
    # replaced while the second camera is the active one: selected anew, as on a new scene's first frame
    e.frame = (3, 0.75, 1.0)
    e.replace(keyed(2, second_camera=True))
    e.check()


@pytest.mark.parametrize("integrator", [F.INTEGRATOR_WHITTED, F.INTEGRATOR_NORMALS_DEBUG])
def test_whitted_and_normals_debug(integrator):
    b, kinds, other = stocked(integrator)
    e = Replaced(b)
    b.receiver(F.SHAPE_SPHERE, kinds["glass"], [SB.trs(t=(0, 15, 5), s=2)], p0=1.0)
    b.receiver(F.SHAPE_MESH, kinds["metal"], [SB.Anim(FLY, degree=2)], mesh=other)
    b.remove_instance(SPHERE)
    e.replace()
    f = e.fresh()
    (ua, ust), (fa, fst) = e.u.render(spp=2, seed=5), f.render(spp=2, seed=5)
    assert rmse(ua, fa) < 1e-5 and counters(ust) == counters(fst)
    assert e.u.bvh(-1)[0].tobytes() == f.bvh(-1)[0].tobytes()
    q, _ = ray_sets(f)
    assert e.u.intersect_records(q)[0].tobytes() == f.intersect_records(q)[0].tobytes()


def test_wide_leaf_form():
    b, kinds, other = stocked()
    e = Replaced(b, options=(("trace.wide_leaf", 1),))
    b.receiver(F.SHAPE_MESH, kinds["plastic"], [SB.trs(t=(-4, 14, 0), s=2)], mesh=other)
    b.remove_instance(SPHERE)
    e.replace()
    e.check()


def test_twenty_random_replacements_among_the_other_edits_then_adaptive_counts():
    b, kinds, other = stocked()
    b.receiver(F.SHAPE_SPHERE, kinds["plastic"], [SB.Anim(FLY, degree=2)], p0=1.0)
    e = Replaced(b, ANIM_FRAME)
    rng = np.random.default_rng(21)
    mats = [MAT_SPHERE, MAT_MESH] + list(kinds.values())
    for step in range(20):
        op = step % 4 if len(b.instances) > 8 else 0
        if op == 0:  # add
            xf = [SB.Anim([(tuple(np.add(t, rng.uniform(-2, 2, 3))), q, s) for t, q, s in FLY], degree=int(rng.integers(1, 4)))] \
                if rng.random() < 0.4 else [SB.trs(t=rng.uniform((-10, 2, -5), (10, 20, 15)), s=float(rng.uniform(0.5, 2.5)))]
            if rng.random() < 0.5:
                b.receiver(F.SHAPE_MESH, int(rng.choice(mats)), xf, mesh=int(rng.integers(0, 2)))
            elif rng.random() < 0.7:
                b.receiver(F.SHAPE_SPHERE, int(rng.choice(mats)), xf, p0=1.0)
            else:
                b.area_light(F.SHAPE_SPHERE, 0, xf, tuple(rng.uniform(1, 30, 3)), p0=0.5)
        elif op == 1:  # remove one of the objects after the walls and the first light
            b.remove_instance(int(rng.integers(LIGHT + 1, len(b.instances))))
        elif op == 2:  # rebind
            i = int(rng.integers(0, len(b.instances)))
            if b.instances[i][0] != F.INST_EMITTER_POINT:
                rebind(b, i, material=int(rng.choice(mats)))
            if b.instances[i][1] == F.SHAPE_MESH:
                rebind(b, i, mesh=int(rng.integers(0, 2)))
        e.replace()
        # and one of the edits that keep the structure, on the new section
        if op == 0:
            first = int(rng.integers(0, len(b.keyframes)))
            t, q, s = b.keyframes[first]
            b.keyframes[first] = (tuple(float(x + d) for x, d in zip(t, rng.uniform(-0.5, 0.5, 3))), q, s)
            e.u.update_keyframes(first, np.array([b.keyframes[first]], F.KEYFRAME_DTYPE))
        elif op == 1:
            first = int(rng.integers(0, len(b.color_keys)))
            b.color_keys[first] = (tuple(float(x) for x in rng.uniform(0.1, 40.0, 4)), b.color_keys[first][1])
            e.u.update_color_keys(first, np.array([b.color_keys[first]], F.COLOR_KEY_DTYPE))
        elif op == 2:
            b.materials[MAT_SPHERE] = mat(int(rng.integers(0, 6)), rng.uniform(0.1, 0.9, 3), rng.uniform(0.5, 3.0, 3), roughness=float(rng.uniform(0, 0.5)))
            e.u.update_materials(MAT_SPHERE, np.array([b.materials[MAT_SPHERE]], F.MATERIAL_DTYPE))
        else:
            p, n, t, i = b.meshes[other]
            p = (p * np.float32(rng.uniform(0.8, 1.25))).astype(np.float32)
            b.meshes[other] = (p, n, t, i)
            e.u.update_mesh(other, p)
        if step in (4, 9, 14):
            e.check(film=False)
    f = e.fresh()
    assert_edited(e.u, f, ANIM_FRAME)
    (ua, us, ust), (fa, fs, fst) = e.u.render_adaptive(2, 16, seed=3), f.render_adaptive(2, 16, seed=3)
    assert us.tobytes() == fs.tobytes() and counters(ust) == counters(fst) and rmse(ua, fa) < 1e-5


def test_ten_to_ten_thousand_instances_and_back():
    e = Replaced(SB.scene_instances(10, 9))
    before = snapshot(e.u)
    for k in (10_000, 10):
        e.replace(SB.scene_instances(k, 9))
        f = e.fresh()
        (un, uo), (fn, fo) = e.u.bvh(-1), f.bvh(-1)
        assert un.tobytes() == fn.tobytes() and uo.tobytes() == fo.tobytes()
        q = random_rays(1 << 16, 3, (-14, 1, -10), (14, 23, 18), 0.0, 0.0)
        (ur, ust), (fr, fst) = e.u.intersect_records(q, stats=True), f.intersect_records(q, stats=True)
        assert ur.tobytes() == fr.tobytes() and counters(ust) == counters(fst)
        assert k == 10 or np.count_nonzero(fr["inst"] >= 6) > 1000  # the spheres are hit
        assert snapshot(e.u) == snapshot(f)
    assert snapshot(e.u) == before


def test_two_hundred_replacements_do_not_grow_the_scene():
    import torch
    small, large = SB.scene_instances(1000, 9), SB.scene_instances(3000, 9)
    e = Replaced(small)
    sections = [large.objects(), small.objects()]
    free = []
    for k in range(201):  # ends on the section it began with; each replacement's buffers are several hundred KB
        e.u.replace_objects(sections[k % 2])
        if k in (0, 200):
            torch.cuda.synchronize()
            free.append(torch.cuda.mem_get_info()[0])
    # kept buffers would add up to more than 100 MB; the allowance is for whatever else uses the device meanwhile
    assert free[1] >= free[0] - (8 << 20), free
    e.b = large
    f = e.fresh()
    assert e.u.bvh(-1)[0].tobytes() == f.bvh(-1)[0].tobytes() and snapshot(e.u) == snapshot(f)


def test_render_in_flight_on_a_side_stream_finishes_on_the_old_objects():
    import torch
    b, kinds, _ = stocked()
    b.film.update(width=256, height=256)
    e = Replaced(b)
    ref, _ = e.fresh().render(spp=4, seed=7)
    s = torch.cuda.Stream()
    film = torch.zeros((256, 256, 4), dtype=torch.float32, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    e.u.render_device(film.data_ptr(), stream=s.cuda_stream, spp=4, seed=7)
    b.remove_instance(MESH_INST)  # frees and replaces every buffer the passes in flight read
    b.remove_instance(SPHERE)
    e.replace()
    s.synchronize()
    assert rmse(film.cpu().numpy(), ref) < 1e-5
    e.check()


def test_failures_leave_the_scene_as_it_was():
    b, kinds, other = stocked()
    e = Replaced(b, (1, 0.0, 0.0))
    u, lib = e.u, F.load_trb()
    before = snapshot(u)

    def fails(change, status=F.TRB_INVALID_ARG, created=True):
        """the section of stocked() after change(builder): replace_objects and, where the fault is the section's, Scene() fail alike"""
        bad, _, _ = stocked()
        change(bad)
        with pytest.raises(api.TrbError) as ex:
            u.replace_objects(bad.objects())
        assert ex.value.status == status
        if created:
            with pytest.raises(api.TrbError) as ex2:
                api.Scene(bad.finish())
            assert ex2.value.status == status and str(ex.value) == str(ex2.value)
        assert snapshot(u) == before and u.n_instances == 8
        return str(ex.value)

    def no_lights(x):
        x.remove_instance(LIGHT)

    def no_objects(x):
        x.instances.clear()

    def no_camera(x):
        x.cameras.clear()

    def knots(x, values, degree=2):
        x.receiver(F.SHAPE_SPHERE, 0, [SB.Anim(FLY, knots=values, degree=degree)], p0=1.0)

    assert "light" in fails(no_lights)
    assert "objects" in fails(no_objects)
    assert "camera" in fails(no_camera)
    fails(lambda x: rebind(x, SPHERE, kind=3))
    fails(lambda x: rebind(x, SPHERE, shape=5))
    assert "geometry" in fails(lambda x: rebind(x, SPHERE, shape=F.SHAPE_NONE))
    assert "not sampleable" in fails(lambda x: rebind(x, LIGHT, shape=F.SHAPE_MESH))
    assert "emission" in fails(lambda x: rebind(x, SPHERE, kind=F.INST_EMITTER_AREA))
    assert "emission" in fails(lambda x: rebind(x, LIGHT, emission_first=0xffffffff, n_emission=2))
    assert "spline range" in fails(lambda x: rebind(x, SPHERE, spline_first=0xffffffff, n_splines=2))
    assert "mesh index" in fails(lambda x: rebind(x, MESH_INST, mesh=2))
    assert "material index" in fails(lambda x: rebind(x, SPHERE, material=len(x.materials)))
    def short_knots(x):  # the flying sphere's spline is the builder's last
        knots(x, SB.clamped_knots(4, 2))
        d, n_ctrl, ctrl_first, n_knots, knot_first = x.splines[-1]
        x.splines[-1] = (d, n_ctrl, ctrl_first, n_knots - 1, knot_first)

    assert "knots.len()" in fails(short_knots)
    assert "NaN" in fails(lambda x: knots(x, [0, 0, 0, float("nan"), 1, 1, 1]))
    assert "Too few" in fails(lambda x: x.splines.__setitem__(-1, (3, 2, 0, 6, 0)))
    assert "control points" in fails(lambda x: x.splines.__setitem__(-1, (0, 1, len(x.keyframes), 2, 0)))
    assert "degree" in fails(lambda x: x.receiver(F.SHAPE_SPHERE, 0, [SB.Anim(FLY + FLY, degree=6)], p0=1.0), F.TRB_UNSUPPORTED)
    # a section that creates a scene, but has no camera for the frame that is set
    assert "no camera is active" in fails(lambda x: x.cameras.__setitem__(0, x.cameras[0][:4] + (2,) + x.cameras[0][5:]), created=False)
    # null arguments and arrays
    good = b.objects()
    assert lib.trb_scene_replace_objects(u._h, None) == F.TRB_INVALID_ARG
    for name, _ in F.SceneObjects._fields_[1::2]:
        if getattr(good, "n_" + name):
            o = F.SceneObjects.from_buffer_copy(good)
            setattr(o, name, C.cast(None, type(getattr(o, name))))
            assert lib.trb_scene_replace_objects(u._h, C.byref(o)) == F.TRB_INVALID_ARG, name
            assert b"null array" in lib.trb_last_error()
    assert snapshot(u) == before
    u.replace_objects(good)
    e.check()
