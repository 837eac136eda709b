"""trb_scene_replace_materials on an H100: after a replacement the scene U must be indistinguishable from F, trb_scene_create on the
builder's description (and update_frame with the same arguments), on everything test_scene_edit_gpu's assert_edited observes. Covered:
a material added and bound through the object section, then removed; a scene without textures gaining one and losing it; an
AnimatedImage; a MERL table and material added and removed (the shading switches between the fused and split kernels); the device
form from torch tensors on a side stream; every failure status; a render in flight on a side stream; device memory over 100
replacements; and a one-device group."""
import ctypes as C

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from test_mesh_update_gpu import FRAME, checker, counters, rmse
from test_scene_edit_gpu import ANIM_FRAME, MAT_MESH, MAT_SPHERE, assert_edited, base
from test_scene_objects_gpu import rebind, snapshot

pytestmark = pytest.mark.gpu
SPHERE_INST = 6  # base(): five walls, the light, then the sphere and the mesh instance


class Shaded:
    """scene U and the builder of its description: replace() hands U the builder's material section (and object section), fresh()
    creates F"""

    def __init__(self, b, frame=FRAME):
        self.b, self.frame = b, frame
        self.u = api.Scene(b.finish())
        self.u.update_frame(*frame)

    def replace(self, objects=False):
        self.u.replace_materials(self.b.materials_section(), self.b.objects() if objects else None)
        assert self.u._desc.n_materials == len(self.b.materials) and self.u._desc.n_textures == len(self.b.textures)

    def fresh(self):
        f = api.Scene(self.b.finish())
        f.update_frame(*self.frame)
        return f

    def check(self, **kw):
        assert_edited(self.u, self.fresh(), self.frame, **kw)
        self.u.update_frame(*self.frame)


def untextured():
    """base() without its texture: the mesh's material bound to a constant"""
    b = base()
    b.materials[MAT_MESH] = b.materials[MAT_MESH][:6] + ((0, 0, 0, 0),)
    b.remove_texture(0)
    return b


def test_material_added_and_bound_through_the_object_section_then_removed():
    b = base()
    e = Shaded(b)
    m = b.add_material(F.MAT_PLASTIC, (0.2, 0.7, 0.3), (0.8, 0.8, 0.8), roughness=0.15)
    rebind(b, SPHERE_INST, material=m)
    e.replace(objects=True)
    e.check()
    rebind(b, SPHERE_INST, material=MAT_SPHERE)
    e.replace(objects=True)
    b.remove_material(m)
    e.replace()
    e.check()


def test_a_scene_without_textures_gains_one_and_loses_it():
    b = untextured()
    e = Shaded(b)
    e.check()
    t = b.add_texture(checker(8))
    b.materials[MAT_SPHERE] = b.materials[MAT_SPHERE][:6] + ((t, 0, 0, 0),)
    e.replace()
    e.check()
    b.materials[MAT_SPHERE] = b.materials[MAT_SPHERE][:6] + ((0, 0, 0, 0),)
    b.remove_texture(t - 1)
    e.replace()
    e.check()


def test_animated_image():
    b = SB.scene_animated(48, 32, 4)
    e = Shaded(b, ANIM_FRAME)
    rng = np.random.default_rng(3)
    t = b.add_texture([(rng.integers(0, 256, (8 + 4 * k, 8, 4), dtype=np.uint8), 0.3 * k) for k in range(3)])
    b.materials[0] = b.materials[0][:6] + ((t, 0, 0, 0),)  # the white walls, over the shutter interval of the frame
    e.replace()
    e.check()


def test_merl_table_and_material_added_and_removed_switch_the_shading_kernels():
    b = untextured()
    for k, it in enumerate(b.instances):  # one kind (matte) everywhere: the fused kernel
        assert it[0] == F.INST_EMITTER_POINT or b.materials[it[5]][0] == F.MAT_MATTE
    e = Shaded(b)
    t = b.add_merl_table(SB.synthetic_merl_table())
    m = b.add_material(F.MAT_MERL, merl=t)
    rebind(b, SPHERE_INST, material=m)
    e.replace(objects=True)  # MERL: the split kernels with material buckets
    e.check()
    rebind(b, SPHERE_INST, material=MAT_SPHERE)
    e.replace(objects=True)
    b.remove_material(m)
    b.remove_merl_table(t)
    e.replace()
    e.check()
    assert e.u._desc.n_merl == 0


def test_device_form_from_torch_tensors_on_a_side_stream():
    import torch
    b = base()
    b.receiver(F.SHAPE_SPHERE, b.add_material(F.MAT_MERL, merl=b.add_merl_table(SB.synthetic_merl_table())), [SB.trs(t=(-6, 10, 10), s=2.5)],
               p0=1.0)
    e = Shaded(b)
    rng = np.random.default_rng(9)
    t = b.add_texture([(rng.integers(0, 256, (32, 48, 4), dtype=np.uint8), 0.5 * k) for k in range(2)])
    b.materials[MAT_SPHERE] = b.materials[MAT_SPHERE][:6] + ((t, 0, 0, 0),)
    b.merl[0] = SB.synthetic_merl_table(seed=2) * 0.5
    host_images, host_merl = list(b.images), list(b.merl)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):  # every table and frame produced on the side stream, as a decoder or another render would
        b.images = [(torch.from_numpy(px).to("cuda") + 0, tm) for px, tm in host_images]
        b.merl = [torch.from_numpy(m).to("cuda") * 1.0 for m in host_merl]
    sec = b.materials_section()  # holds the tensors
    b.images, b.merl = host_images, host_merl
    e.u.replace_materials_device(sec, None, stream=s.cuda_stream)
    e.check()


def test_failures_leave_the_scene_as_it_was():
    b = base()
    e = Shaded(b)
    u, lib = e.u, F.load_trb()
    before = snapshot(u)

    def fails(sec, objects=None, status=F.TRB_INVALID_ARG, desc=None):
        with pytest.raises(api.TrbError) as ex:
            u.replace_materials(sec, objects)
        assert ex.value.status == status
        if desc is not None:  # trb_scene_create refuses that description alike
            with pytest.raises(api.TrbError) as ex2:
                api.Scene(desc)
            assert ex2.value.status == status and str(ex.value) == str(ex2.value)
        assert snapshot(u) == before and u._desc.n_materials == len(b.materials)
        return str(ex.value)

    def variant(edit):
        v = base()
        edit(v)
        return v

    cases = [
        (lambda v: v.materials.__setitem__(MAT_SPHERE, v.materials[MAT_SPHERE][:0] + (9,) + v.materials[MAT_SPHERE][1:]), "unrecognized material type"),
        (lambda v: v.materials.__setitem__(MAT_SPHERE, (F.MAT_MERL,) + v.materials[MAT_SPHERE][1:5] + (0,) + v.materials[MAT_SPHERE][6:]),
         "merl table index out of range"),
        (lambda v: v.materials.__setitem__(MAT_SPHERE, v.materials[MAT_SPHERE][:6] + ((2, 0, 0, 0),)), "texture index out of range"),
        (lambda v: v.textures.__setitem__(0, (0, 2)), "texture image range out of bounds"),
        (lambda v: v.images.__setitem__(0, (np.zeros((0, 4, 4), np.uint8), 0.0)), "empty image"),
        (lambda v: v.materials.pop(), "material index out of range"),
    ]
    for edit, msg in cases:
        v = variant(edit)
        assert msg in fails(v.materials_section(), desc=v.finish())
    big = variant(lambda v: None)
    sec = big.materials_section()
    sec.images[0].width, sec.images[0].height = 1 << 16, 1 << 16  # 2^32 texels: refused before any texel is read
    assert "2^32 texels" in fails(sec, status=F.TRB_UNSUPPORTED)
    late = variant(lambda v: None)
    late.cameras[0] = late.cameras[0][:4] + (2,) + late.cameras[0][5:]
    assert "no camera is active" in fails(b.materials_section(), late.objects())
    for field in ("materials", "textures", "images"):
        sec = b.materials_section()
        setattr(sec, field, None)
        assert "null array" in fails(sec)
    merl = variant(lambda v: v.add_merl_table(SB.synthetic_merl_table()))
    sec = merl.materials_section()
    sec.merl_tables[0] = None
    assert "null MERL table" in fails(sec)
    assert lib.trb_scene_replace_materials(u._h, None, None) == F.TRB_INVALID_ARG
    assert lib.trb_scene_replace_materials_device(u._h, None, None, None) == F.TRB_INVALID_ARG
    assert snapshot(u) == before
    e.replace()
    e.check()


def test_render_in_flight_on_a_side_stream_finishes_on_the_old_materials():
    import torch
    b = base(w=256, h=256)
    e = Shaded(b)
    ref, _ = e.fresh().render(spp=4, seed=7)
    s = torch.cuda.Stream()
    film = torch.zeros((256, 256, 4), dtype=torch.float32, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    e.u.render_device(film.data_ptr(), stream=s.cuda_stream, spp=4, seed=7)
    b.materials[MAT_SPHERE] = b.materials[MAT_SPHERE][:1] + ((0.1, 0.9, 0.1),) + b.materials[MAT_SPHERE][2:]
    b.add_texture(checker(64))
    e.replace()  # frees the material records and texels the passes in flight read
    s.synchronize()
    assert rmse(film.cpu().numpy(), ref) < 1e-5
    e.check()


def test_a_hundred_replacements_do_not_grow_the_scene():
    import torch
    b = base()
    e = Shaded(b)
    small = b.materials_section()
    b.add_texture(np.zeros((512, 512, 4), np.uint8))
    b.add_merl_table(SB.synthetic_merl_table())
    big = b.materials_section()  # 1 MB of texels and a 17.5 MB MERL table more
    free = []
    for k in range(100):
        e.u.replace_materials(big if k % 2 == 0 else small)
        if k in (1, 99):
            torch.cuda.synchronize()
            free.append(torch.cuda.mem_get_info()[0])
    assert free[1] >= free[0] - (8 << 20), free
    b.merl.pop()
    b.remove_texture(1)
    e.check(film=False)


def test_one_device_group_replaced_through_its_replica():
    b = base()
    ga = api.Group(b.finish(), [0])
    t = b.add_merl_table(SB.synthetic_merl_table())
    m = b.add_material(F.MAT_MERL, merl=t)
    rebind(b, SPHERE_INST, material=m)
    sec, objs = b.materials_section(), b.objects()
    gb = api.Group(b.finish(), [0])
    lib = F.load_trb()
    rep = lib.trb_group_scene(ga._h, 0)
    assert rep
    assert lib.trb_scene_replace_materials(rep, C.byref(sec), C.byref(objs)) == F.TRB_OK, lib.trb_last_error()
    (fa, sa), (fb, sb) = ga.render(spp=2, seed=3), gb.render(spp=2, seed=3)
    assert rmse(fa, fb) < 1e-5 and counters(sa) == counters(sb)
