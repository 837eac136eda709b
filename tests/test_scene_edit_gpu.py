"""trb_scene_update_keyframes / _device / _color_keys / _materials on an H100: after an edit the scene U must be indistinguishable from
F, trb_scene_create on the edited description (and update_frame with the same arguments), on everything a caller can observe: the TLAS
and the instance transforms, per-sample radiance and every counter in both shadow modes, films, intersection records, occlusion and
illumination, the BSDF, light and emission queries and the light list. Covered: instances and the camera moved (frame built on the
device, on the host, and edits before the first frame), the distinct-spline tables split and merged, colour keys of area, point and
keyframed emitters, every material kind changed, Lambertian / Oren-Nayar, texture bindings, edits that switch the shading kernels,
Whitted and NormalsDebug, the device form on a torch side stream, twenty random edits in sequence with the Adaptive sampler's per-pixel
counts, 10 000 instances moved at once, every failure status, and a one-device trb_group."""
import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from test_mesh_update_gpu import FRAME, assert_same, checker, counters, ray_sets, rmse
from test_queries_cpu import random_rays

pytestmark = pytest.mark.gpu
ANIM_FRAME = (0, 0.0, 1.0)
# keyframes, materials and instances of base(): walls 0-9 (two levels each), light 10, sphere 11, mesh instance 12, camera 13
KF_SPHERE, KF_MESH, KF_CAMERA = 11, 12, 13
MAT_SPHERE, MAT_MESH = 3, 4


def base(integrator=F.INTEGRATOR_PATH, w=48, h=32, spp=4):
    """the Cornell walls and light around a static sphere and a static mesh instance, all matte; a texture bound to the mesh's colour"""
    b = SB.SceneBuilder(w, h, spp, 3, 6)
    b.integrator = (integrator, 3, 6)
    mats = SB.cornell_walls(b)
    SB.cornell_light(b, mats["white"])
    tex = b.add_texture(checker())
    sphere = b.add_material(F.MAT_MATTE, (0.7, 0.3, 0.2), roughness=1.0)
    mesh = b.add_material(F.MAT_MATTE, (0.74, 0.74, 0.73), roughness=1.0, tex_c0=tex)
    b.receiver(F.SHAPE_SPHERE, sphere, [SB.trs(t=(-5, 4, 4), s=3)], p0=1.0)
    m = b.add_mesh(*SB.icosphere_mesh(2, 1.0, 0.1, 7))
    b.receiver(F.SHAPE_MESH, mesh, [SB.trs(t=(5, 4, 2), s=3)], mesh=m)
    b.add_camera([SB.trs(t=(0, 12, -60))], fov=30.0)
    return b


def mat(mtype, c0=(0.5, 0.5, 0.5), c1=(0.5, 0.5, 0.5), roughness=0.0, eta=1.5, merl=0, tex=(0, 0, 0, 0)):
    """a material as SceneBuilder keeps it"""
    return (mtype, tuple(float(x) for x in c0), tuple(float(x) for x in c1), float(roughness), float(eta), merl, tuple(tex))


def unit(v):
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def assert_shading(u, f, frame, seed=11):
    """the five shading queries and the light list at hit records of F"""
    q, _ = ray_sets(f, frame, n_random=4096, seed=seed)
    rec = f.intersect_records(q)[0]
    rec = rec[rec["inst"] != F.MISS]
    n, rng = len(rec), np.random.default_rng(seed)
    ev = np.zeros(n, F.BSDF_EVAL_QUERY_DTYPE)
    ev["wo"], ev["wi"], ev["bxdf"] = unit(rng.normal(size=(n, 3))), unit(rng.normal(size=(n, 3))), F.BXDF_ALL
    assert u.bsdf_eval(rec, ev).tobytes() == f.bsdf_eval(rec, ev).tobytes()
    sq = np.zeros(n, F.BSDF_SAMPLE_QUERY_DTYPE)
    sq["wo"], sq["bxdf"], sq["u"], sq["u_comp"] = unit(rng.normal(size=(n, 3))), F.BXDF_ALL, rng.random((n, 2)), rng.random(n)
    assert u.bsdf_sample(rec, sq).tobytes() == f.bsdf_sample(rec, sq).tobytes()
    lights = f.lights()
    assert u.lights().tobytes() == lights.tobytes()
    lq = np.zeros(n, F.LIGHT_QUERY_DTYPE)
    lq["p"], lq["time"], lq["u"], lq["light"] = rec["p"], rec["time"], rng.random((n, 2)), rng.integers(0, len(lights), n)
    assert u.light_sample(lq).tobytes() == f.light_sample(lq).tobytes()
    pq = np.zeros(n, F.LIGHT_PDF_QUERY_DTYPE)
    pq["p"], pq["time"], pq["wi"], pq["light"] = rec["p"], rec["time"], unit(rng.normal(size=(n, 3))), lq["light"]
    assert u.light_pdf(pq).tobytes() == f.light_pdf(pq).tobytes()
    eq = np.zeros(n, F.EMIT_QUERY_DTYPE)
    eq["w"], eq["time"], eq["n"] = unit(rng.normal(size=(n, 3))), rec["time"], rec["n"]
    eq["inst"] = rng.choice(np.concatenate([lights, [0]]), n)
    assert u.emitted(eq).tobytes() == f.emitted(eq).tobytes()


def assert_edited(u, f, frame=FRAME, film=True, shading=True):
    assert_same(u, f, frame, n_meshes=u._desc.n_meshes, film=film)
    (un, uo), (fn, fo) = u.bvh(-1), f.bvh(-1)
    assert un.tobytes() == fn.tobytes() and uo.tobytes() == fo.tobytes()
    for i in range(u.n_instances):
        assert all(a.tobytes() == b.tobytes() for a, b in zip(u.transform(i), f.transform(i))), i
    if shading:
        assert_shading(u, f, frame)


class Edited:
    """scene U under edits, and the builder of its description, which gets the same edits: fresh() creates F from it"""

    def __init__(self, b, frame=FRAME, frame_device=1, set_frame=True):
        self.b, self.frame, self.frame_device = b, frame, frame_device
        self.u = api.Scene(b.finish())
        self.u.set_option("frame.device", frame_device)
        if set_frame:
            self.u.update_frame(*frame)

    def keyframes(self, first, items):
        self.b.keyframes[first:first + len(items)] = items
        self.u.update_keyframes(first, np.array(items, F.KEYFRAME_DTYPE))

    def color_keys(self, first, items):
        self.b.color_keys[first:first + len(items)] = items
        self.u.update_color_keys(first, np.array(items, F.COLOR_KEY_DTYPE))

    def materials(self, first, items):
        self.b.materials[first:first + len(items)] = items
        self.u.update_materials(first, np.array(items, F.MATERIAL_DTYPE))

    def fresh(self):
        f = api.Scene(self.b.finish())
        f.set_option("frame.device", self.frame_device)
        f.update_frame(*self.frame)
        return f

    def check(self, **kw):
        assert_edited(self.u, self.fresh(), self.frame, **kw)
        # the film render runs update_frame for its own frame (Exec::render): set this one again, which a keyframe edit re-runs
        self.u.update_frame(*self.frame)


@pytest.mark.parametrize("how", ["device_frame", "host_frame", "before_first_frame"])
def test_static_sphere_and_mesh_instance_moved_out_of_their_bounds(how):
    e = Edited(base(), frame_device=0 if how == "host_frame" else 1, set_frame=how != "before_first_frame")
    root = e.u.bvh(-1)[0][0].tobytes() if how != "before_first_frame" else None
    e.keyframes(KF_SPHERE, [SB.trs(t=(-6, 15, 10), s=2.5)])
    e.keyframes(KF_MESH, [SB.trs(t=(7, 17, 13), q=SB.quat_axis_angle((0, 1, 0), 40), s=2)])
    if how == "before_first_frame":
        e.u.update_frame(*e.frame)
    else:
        assert e.u.bvh(-1)[0][0].tobytes() != root  # the TLAS root box grew
    e.check()


def test_camera_moved_static_then_keyframed():
    e = Edited(base())
    e.keyframes(KF_CAMERA, [SB.trs(t=(3, 14, -50), q=SB.quat_axis_angle((0, 1, 0), 4))])
    e.check()
    a = Edited(SB.scene_animated(48, 32, 4), ANIM_FRAME)
    cam = a.b.cameras[0]
    ctrl = a.b.splines[cam[0]][2]
    a.keyframes(ctrl + 1, [SB.trs(t=(2, 15, -55), q=SB.quat_axis_angle((0, 1, 0), -6))])
    a.check()


def twins(second_keys):
    """base() and two spheres on keyframed splines: the first's keys, and second_keys"""
    keys = [SB.trs(t=(-8, 4, 0)), SB.trs(t=(-2, 10, 4)), SB.trs(t=(4, 6, 8)), SB.trs(t=(8, 12, 2))]
    b = base()
    b.receiver(F.SHAPE_SPHERE, MAT_SPHERE, [SB.Anim(keys, degree=2)], p0=1.0)
    b.receiver(F.SHAPE_SPHERE, MAT_MESH, [SB.Anim(second_keys or keys, degree=2)], p0=1.0)
    return b, keys, len(b.keyframes) - 4


def test_identical_keyframed_splines_stop_sharing_a_row_when_one_is_edited():
    b, keys, second = twins(None)
    e = Edited(b, ANIM_FRAME)
    e.keyframes(second + 2, [SB.trs(t=(2, 3, 12))])
    e.check()
    e.keyframes(second + 2, [keys[2]])  # equal again
    e.check()


def test_different_keyframed_splines_edited_to_become_identical():
    other = [SB.trs(t=(8, 4, 0)), SB.trs(t=(2, 10, 4)), SB.trs(t=(-4, 6, 8)), SB.trs(t=(-8, 12, 2))]
    b, keys, second = twins(other)
    e = Edited(b, ANIM_FRAME)
    e.keyframes(second, keys)
    e.check()


def test_colour_keys_of_area_point_and_keyframed_emitters():
    z = Edited(SB.scene_materials_zoo(48, 32, 4))
    assert len(z.b.color_keys) == 3  # the panel light, the point light, the disk light
    z.color_keys(0, [((2.0, 1.0, 0.5, 1.0), 0.0)])
    z.check()
    z.color_keys(1, [((90.0, 10.0, 40.0, 1.0), 0.0), ((5.0, 20.0, 10.0, 1.0), 0.0)])
    z.check()
    a = Edited(SB.scene_animated(48, 32, 4), ANIM_FRAME)
    disk = [k for k, inst in enumerate(a.b.instances) if inst[9] == 3][0]
    first = a.b.instances[disk][8]
    a.color_keys(first, [((0.2, 0.9, 0.1, 50.0), 0.1), ((0.9, 0.1, 0.9, 10.0), 0.5)])
    a.check()


def test_every_material_kind_changed_to_another_including_merl():
    z = Edited(SB.scene_materials_zoo(48, 32, 4, merl_table=SB.synthetic_merl_table()))
    new = []
    for m in z.b.materials:  # kind k becomes k + 1 (MERL becomes matte)
        k = (m[0] + 1) % 7
        new.append(mat(k, m[1] if k != F.MAT_MERL else (0, 0, 0), (0.6, 0.7, 0.8) if k in (F.MAT_PLASTIC, F.MAT_ROUGH_GLASS) else m[2],
                       roughness=0.25 if k != F.MAT_MATTE else 0.0, eta=1.33, merl=0))
    z.materials(0, new)
    z.check()


def test_lambertian_and_oren_nayar_and_texture_bindings():
    e = Edited(base())
    e.materials(MAT_SPHERE, [mat(F.MAT_MATTE, (0.7, 0.3, 0.2), roughness=0.0)])  # Oren-Nayar -> Lambertian
    e.materials(0, [mat(F.MAT_MATTE, SB.CORNELL_MATS["white"], roughness=25.0)])  # and the white walls rougher
    e.check()
    e.materials(MAT_SPHERE, [mat(F.MAT_MATTE, (0.7, 0.3, 0.2), roughness=10.0, tex=(1, 0, 0, 0))])  # a texture bound
    e.materials(MAT_MESH, [mat(F.MAT_MATTE, (0.74, 0.74, 0.73), roughness=1.0)])  # and one removed
    e.check()


def test_shading_kernels_switch_with_the_material_kinds():
    e = Edited(base())  # all matte: split kernels with the matte instantiations
    e.materials(MAT_SPHERE, [mat(F.MAT_PLASTIC, (0.8, 0.2, 0.2), (0.8, 0.8, 0.8), roughness=0.1)])  # mixed
    e.check()
    plastic = [mat(F.MAT_PLASTIC, (0.2 + 0.1 * i, 0.5, 0.5), (0.8, 0.8, 0.8), roughness=0.2) for i in range(5)]
    e.materials(0, plastic)  # one kind, not matte: the fused kernel
    e.check()
    e.materials(MAT_MESH, [mat(F.MAT_METAL, (0.155, 0.117, 0.138), (4.83, 3.12, 2.15), roughness=0.3)])  # mixed again
    e.check()


@pytest.mark.parametrize("integrator", [F.INTEGRATOR_WHITTED, F.INTEGRATOR_NORMALS_DEBUG])
def test_whitted_and_normals_debug(integrator):
    e = Edited(base(integrator))
    e.keyframes(KF_SPHERE, [SB.trs(t=(-6, 15, 10), s=2.5)])
    e.materials(MAT_MESH, [mat(F.MAT_GLASS, (1, 1, 1), (1, 1, 1), eta=1.5)])
    f = e.fresh()
    (ua, ust), (fa, fst) = e.u.render(spp=2, seed=5), f.render(spp=2, seed=5)
    assert rmse(ua, fa) < 1e-5 and counters(ust) == counters(fst)
    assert e.u.bvh(-1)[0].tobytes() == f.bvh(-1)[0].tobytes()
    q, _ = ray_sets(f)
    assert e.u.intersect_records(q)[0].tobytes() == f.intersect_records(q)[0].tobytes()


def test_device_keyframes_from_a_torch_side_stream():
    import torch
    e = Edited(base())
    new = [SB.trs(t=(-6, 15, 10), s=2.5), SB.trs(t=(7, 17, 13), q=SB.quat_axis_angle((0, 1, 0), 40), s=2)]
    host = np.array(new, F.KEYFRAME_DTYPE)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d = torch.from_numpy(host.view(np.float32).reshape(2, 10).copy()).to("cuda") * 1.0
    e.u.update_keyframes_device(KF_SPHERE, 2, d.data_ptr(), stream=s.cuda_stream)
    e.b.keyframes[KF_SPHERE:KF_SPHERE + 2] = new
    e.check()


def test_twenty_random_edits_in_sequence_then_adaptive_counts():
    b = SB.scene_animated(48, 32, 4)
    b.receiver(F.SHAPE_SPHERE, b.add_material(F.MAT_MERL, merl=b.add_merl_table(SB.synthetic_merl_table())), [SB.trs(t=(-6, 10, 10), s=2.5)],
               p0=1.0)
    e = Edited(b, ANIM_FRAME)
    rng = np.random.default_rng(20)
    n_kf, n_ck, n_mat = len(b.keyframes), len(b.color_keys), len(b.materials)
    for step in range(20):
        kind = step % 3
        if kind == 0:
            first = int(rng.integers(0, n_kf))
            cnt = int(rng.integers(1, min(4, n_kf - first) + 1))
            items = [(tuple(float(x) + float(d) for x, d in zip(k[0], rng.uniform(-0.5, 0.5, 3))), k[1], k[2])
                     for k in b.keyframes[first:first + cnt]]
            e.keyframes(first, items)
        elif kind == 1:
            first = int(rng.integers(0, n_ck))
            e.color_keys(first, [(tuple(float(x) for x in rng.uniform(0.1, 40.0, 4)), b.color_keys[first][1])])
        else:
            first = int(rng.integers(0, n_mat))
            k = int(rng.integers(0, 7))
            e.materials(first, [mat(k, rng.uniform(0.1, 0.9, 3), rng.uniform(0.5, 3.0, 3), roughness=float(rng.uniform(0, 0.5)),
                                    eta=float(rng.uniform(1.2, 1.8)), merl=0)])
    f = e.fresh()
    assert_edited(e.u, f, ANIM_FRAME)
    (ua, us, ust), (fa, fs, fst) = e.u.render_adaptive(2, 16, seed=3), f.render_adaptive(2, 16, seed=3)
    assert us.tobytes() == fs.tobytes() and counters(ust) == counters(fst) and rmse(ua, fa) < 1e-5


def test_ten_thousand_instances_moved_through_the_device_form():
    import torch
    k = 10_000
    b = SB.scene_instances(k, 9)
    e = Edited(b)
    first = 11  # five walls (two levels each) and the light come first
    rng = np.random.default_rng(10)
    new = [SB.trs(t=rng.uniform((-13, 1, -8), (13, 22, 18)), s=0.3) for _ in range(k)]
    d = torch.from_numpy(np.array(new, F.KEYFRAME_DTYPE).view(np.float32).reshape(k, 10).copy()).cuda()
    e.u.update_keyframes_device(first, k, d.data_ptr())
    b.keyframes[first:first + k] = new
    f = e.fresh()
    (un, uo), (fn, fo) = e.u.bvh(-1), f.bvh(-1)
    assert un.tobytes() == fn.tobytes() and uo.tobytes() == fo.tobytes()
    q = random_rays(1 << 16, 3, (-14, 1, -10), (14, 23, 18), 0.0, 0.0)
    (ur, ust), (fr, fst) = e.u.intersect_records(q, stats=True), f.intersect_records(q, stats=True)
    assert ur.tobytes() == fr.tobytes() and counters(ust) == counters(fst)
    assert np.count_nonzero(fr["inst"] >= 6) > 1000  # the spheres are hit
    us, fs = e.u.render_samples(flags=F.RENDER_STATS, spp=1, seed=3), f.render_samples(flags=F.RENDER_STATS, spp=1, seed=3)
    assert us[0].tobytes() == fs[0].tobytes() and counters(us[1]) == counters(fs[1])


def test_failures_leave_the_scene_as_it_was():
    import torch
    e = Edited(base())
    u, lib = e.u, F.load_trb()
    before = u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3)

    def unchanged():
        after = u.render_samples(flags=F.RENDER_STATS, spp=2, seed=3)
        assert after[0].tobytes() == before[0].tobytes() and counters(after[1]) == counters(before[1])

    kf = np.array([SB.trs(t=(1, 2, 3))] * 2, F.KEYFRAME_DTYPE)
    ck = np.array([((1.0, 1.0, 1.0, 1.0), 0.0)] * 2, F.COLOR_KEY_DTYPE)
    good = np.array([mat(F.MAT_GLASS)], F.MATERIAL_DTYPE)
    n_kf, n_ck, n_mat = len(e.b.keyframes), len(e.b.color_keys), len(e.b.materials)
    d = torch.zeros(32, dtype=torch.float32, device="cuda")
    for rc in (lib.trb_scene_update_keyframes(u._h, 0, 1, None), lib.trb_scene_update_keyframes(u._h, n_kf - 1, 2, F.ptr(kf)),
               lib.trb_scene_update_keyframes(u._h, 0xffffffff, 2, F.ptr(kf)), lib.trb_scene_update_keyframes(u._h, n_kf, 1, F.ptr(kf)),
               lib.trb_scene_update_keyframes_device(u._h, 0, 1, None, None), lib.trb_scene_update_keyframes_device(u._h, 0, 1, d.data_ptr() + 2, None),
               lib.trb_scene_update_keyframes_device(u._h, 0xfffffffe, 3, d.data_ptr(), None),
               lib.trb_scene_update_color_keys(u._h, 0, 1, None), lib.trb_scene_update_color_keys(u._h, n_ck, 1, F.ptr(ck)),
               lib.trb_scene_update_color_keys(u._h, 0xffffffff, 1, F.ptr(ck)),
               lib.trb_scene_update_materials(u._h, 0, 1, None), lib.trb_scene_update_materials(u._h, n_mat, 1, F.ptr(good)),
               lib.trb_scene_update_materials(u._h, 0xffffffff, 0xffffffff, F.ptr(good))):
        assert rc == F.TRB_INVALID_ARG, lib.trb_last_error()
        unchanged()
    for rc in (lib.trb_scene_update_keyframes(u._h, 0, 0, None), lib.trb_scene_update_keyframes_device(u._h, 0, 0, None, None),
               lib.trb_scene_update_color_keys(u._h, 0, 0, None), lib.trb_scene_update_materials(u._h, 0, 0, None)):
        assert rc == F.TRB_OK
    unchanged()
    # invalid materials: trb_scene_create's statuses and messages, and a valid entry before an invalid one is not written either
    for bad in (mat(7), mat(F.MAT_MERL, merl=0), mat(F.MAT_MATTE, tex=(0, 2, 0, 0))):
        with pytest.raises(api.TrbError) as ex:
            u.update_materials(MAT_SPHERE, np.array([mat(F.MAT_GLASS), bad], F.MATERIAL_DTYPE))
        b = base()
        b.materials[MAT_SPHERE + 1] = bad
        with pytest.raises(api.TrbError) as ex2:
            api.Scene(b.finish())
        assert ex.value.status == ex2.value.status == F.TRB_INVALID_ARG and str(ex.value) == str(ex2.value)
        unchanged()
    assert_edited(u, e.fresh(), film=False)


def test_one_device_group_edited_through_its_replica():
    b = base()
    ga = api.Group(b.finish(), [0])
    new = [SB.trs(t=(-6, 15, 10), s=2.5)]
    b.keyframes[KF_SPHERE] = new[0]
    b.materials[MAT_MESH] = mat(F.MAT_PLASTIC, (0.8, 0.2, 0.2), (0.8, 0.8, 0.8), roughness=0.1)
    b.color_keys[0] = ((30.0, 20.0, 10.0, 1.0), 0.0)
    gb = api.Group(b.finish(), [0])
    lib = F.load_trb()
    rep = lib.trb_group_scene(ga._h, 0)
    assert rep
    kf, m, ck = np.array(new, F.KEYFRAME_DTYPE), np.array([b.materials[MAT_MESH]], F.MATERIAL_DTYPE), np.array([b.color_keys[0]], F.COLOR_KEY_DTYPE)
    assert lib.trb_scene_update_keyframes(rep, KF_SPHERE, 1, F.ptr(kf)) == F.TRB_OK, lib.trb_last_error()
    assert lib.trb_scene_update_materials(rep, MAT_MESH, 1, F.ptr(m)) == F.TRB_OK, lib.trb_last_error()
    assert lib.trb_scene_update_color_keys(rep, 0, 1, F.ptr(ck)) == F.TRB_OK, lib.trb_last_error()
    (fa, sa), (fb, sb) = ga.render(spp=2, seed=3), gb.render(spp=2, seed=3)
    assert rmse(fa, fb) < 1e-5 and counters(sa) == counters(sb)
