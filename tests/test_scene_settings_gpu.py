"""trb_scene_replace_settings on an H100: after a replacement the scene U must be indistinguishable from F, trb_scene_create on the
builder's description (and update_frame with the same arguments), on everything test_scene_edit_gpu's assert_edited observes, plus the
film's size and spp, the filter table, the block list and sample regions, the camera rays and a film write. Covered: resolution
changes with frames built on the device, on the host and not at all; an Adaptive render on a grown film (the per-pixel state is sized
anew); Mitchell to Gaussian and a filter of 8 pixel widths; film.samples with spp 0; Path, Whitted and NormalsDebug with their depth
limits; every failure status; a render in flight on a side stream; device memory over 100 replacements; and a one-device group."""
import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api
from test_mesh_update_gpu import FRAME, counters, ray_sets, rmse
from test_scene_edit_gpu import assert_edited, base
from test_scene_objects_gpu import snapshot

pytestmark = pytest.mark.gpu


class Settled:
    """scene U and the builder of its description: replace() hands U the builder's film and integrator, fresh() creates F"""

    def __init__(self, b, frame=FRAME, frame_device=1, set_frame=True):
        self.b, self.frame, self.frame_device = b, frame, frame_device
        self.u = api.Scene(b.finish())
        self.u.set_option("frame.device", frame_device)
        if set_frame:
            self.u.update_frame(*frame)

    def replace(self, film=True, integrator=True):
        self.u.replace_settings(dict(self.b.film) if film else None, tuple(self.b.integrator) if integrator else None)
        assert (self.u.width, self.u.height) == (self.b.film["width"], self.b.film["height"])

    def fresh(self):
        f = api.Scene(self.b.finish())
        f.set_option("frame.device", self.frame_device)
        f.update_frame(*self.frame)
        return f

    def check(self, **kw):
        f = self.fresh()
        assert_edited(self.u, f, self.frame, **kw)
        assert_settings(self.u, f)
        self.u.update_frame(*self.frame)


def assert_settings(u, f):
    """what the film decides: size, rounded spp and block count, the filter table, the block list, the sample regions, the camera rays
    and a film write of the same samples"""
    assert (u.width, u.height, u.spp, u.total_blocks) == (f.width, f.height, f.spp, f.total_blocks)
    assert u.filter_table().tobytes() == f.filter_table().tobytes()
    assert u.block_list().tobytes() == f.block_list().tobytes()
    assert u.sample_regions(spp=2).tobytes() == f.sample_regions(spp=2).tobytes()
    (ur, ux), (fr, fx) = u.camera_rays(spp=2, seed=5), f.camera_rays(spp=2, seed=5)
    assert ur.tobytes() == fr.tobytes() and ux.tobytes() == fx.tobytes()
    s, _ = f.render_samples(spp=2, seed=5)
    regions = f.sample_regions(spp=2)
    assert u.film_write(s, regions).tobytes() == f.film_write(s, regions).tobytes()


@pytest.mark.parametrize("how", ["device_frame", "host_frame", "before_first_frame"])
def test_resolution_changes_and_back(how):
    b = base()
    e = Settled(b, frame_device=0 if how == "host_frame" else 1, set_frame=how != "before_first_frame")
    for w, h in ((64, 64), (16, 8), (48, 32)):
        b.film.update(width=w, height=h)
        e.replace(integrator=False)
        if how == "before_first_frame" and (w, h) == (64, 64):
            with pytest.raises(api.TrbError):  # no frame was set, so none was built
                e.u.render_samples(spp=1)
            e.u.update_frame(*e.frame)
        e.check()


def test_adaptive_on_a_grown_film_counts_like_a_fresh_scene():
    b = base(w=16, h=16)
    e = Settled(b)
    e.u.render_adaptive(2, 16, seed=3)  # the per-pixel state is allocated for 16 x 16
    b.film.update(width=64, height=48)
    e.replace(integrator=False)
    f = e.fresh()
    (ua, us, ust), (fa, fs, fst) = e.u.render_adaptive(2, 16, seed=3), f.render_adaptive(2, 16, seed=3)
    assert us.shape == (48, 64) and us.tobytes() == fs.tobytes() and counters(ust) == counters(fst) and rmse(ua, fa) < 1e-5
    b.film.update(width=16, height=8)
    e.replace(integrator=False)
    f = e.fresh()
    (ua, us, ust), (fa, fs, fst) = e.u.render_adaptive(2, 16, seed=4), f.render_adaptive(2, 16, seed=4)
    assert us.tobytes() == fs.tobytes() and counters(ust) == counters(fst) and rmse(ua, fa) < 1e-5


def test_mitchell_to_gaussian_and_a_filter_of_eight_pixel_widths():
    b = base()
    e = Settled(b)
    b.film.update(filter_type=F.FILTER_GAUSSIAN, filter_w=1.5, filter_h=1.5, filter_b=2.0)
    e.replace(integrator=False)
    e.check()
    b.film.update(filter_w=4.0, filter_h=3.25)  # fpw 8 by 6
    e.replace(integrator=False)
    e.check()
    b.film.update(filter_type=F.FILTER_MITCHELL_NETRAVALI, filter_w=2.0, filter_h=2.0, filter_b=1.0 / 3.0, filter_c=1.0 / 3.0)
    e.replace(integrator=False)
    e.check()


def test_film_samples_changed_and_rendered_with_spp_0():
    b = base()
    e = Settled(b)
    for samples in (8, 3, 1):
        b.film.update(samples=samples)
        e.replace(integrator=False)
        f = e.fresh()
        assert e.u.spp == f.spp == 1 << (samples - 1).bit_length()
        (ua, ust), (fa, fst) = e.u.render(spp=0, seed=5, flags=F.RENDER_STATS), f.render(spp=0, seed=5, flags=F.RENDER_STATS)
        assert rmse(ua, fa) < 1e-5 and counters(ust) == counters(fst)
        us, fs = e.u.render_samples(spp=0, seed=5), f.render_samples(spp=0, seed=5)
        assert us[0].tobytes() == fs[0].tobytes()


def assert_simple(u, f):
    """a Whitted or NormalsDebug scene: films, counters, the instance tree and hit records"""
    (ua, ust), (fa, fst) = u.render(spp=2, seed=5, flags=F.RENDER_STATS), f.render(spp=2, seed=5, flags=F.RENDER_STATS)
    assert rmse(ua, fa) < 1e-5 and counters(ust) == counters(fst)
    us, fs = u.render_samples(spp=2, seed=5), f.render_samples(spp=2, seed=5)
    assert us[0].tobytes() == fs[0].tobytes()
    assert u.bvh(-1)[0].tobytes() == f.bvh(-1)[0].tobytes()
    q, _ = ray_sets(f)
    assert u.intersect_records(q)[0].tobytes() == f.intersect_records(q)[0].tobytes()


def test_path_whitted_normals_debug_and_back_with_depth_limits():
    b = base()
    e = Settled(b)
    lib = F.load_trb()
    for integrator in ((F.INTEGRATOR_WHITTED, 0, 5), (F.INTEGRATOR_NORMALS_DEBUG, 0, 1), (F.INTEGRATOR_WHITTED, 0, 24), (F.INTEGRATOR_PATH, 2, 5)):
        b.integrator = integrator
        e.replace(film=False)
        f = e.fresh()
        if integrator[0] == F.INTEGRATOR_PATH:
            e.check()
            continue
        assert_simple(e.u, f)
        with pytest.raises(api.TrbError) as ex:  # the Adaptive sampler stays refused
            e.u.render_adaptive(2, 16)
        assert ex.value.status == F.TRB_UNSUPPORTED
        e.u.update_frame(*e.frame)
    before = snapshot(e.u)
    for integrator, status in (((F.INTEGRATOR_PATH, 2, 58), F.TRB_UNSUPPORTED), ((F.INTEGRATOR_WHITTED, 0, 25), F.TRB_UNSUPPORTED),
                               ((3, 2, 5), F.TRB_INVALID_ARG)):
        rc = lib.trb_scene_replace_settings(e.u._h, None, F.Integrator(*integrator))
        msg = lib.trb_last_error()
        bad = base()
        bad.integrator = integrator
        with pytest.raises(api.TrbError) as ex:
            api.Scene(bad.finish())
        assert rc == ex.value.status == status and str(ex.value).endswith(": " + msg.decode())
        assert snapshot(e.u) == before
    b.integrator = (F.INTEGRATOR_PATH, 3, 57)
    e.replace(film=False)
    e.check(film=False)


def test_failures_leave_the_scene_as_it_was():
    b = base()
    e = Settled(b)
    u, lib = e.u, F.load_trb()
    before, table = snapshot(u), u.filter_table().tobytes()
    for change, status in ((dict(width=44), F.TRB_INVALID_ARG), (dict(height=0), F.TRB_INVALID_ARG), (dict(frames=0), F.TRB_INVALID_ARG),
                           (dict(filter_w=0.0), F.TRB_INVALID_ARG), (dict(filter_h=-1.0), F.TRB_INVALID_ARG),
                           (dict(filter_w=4.5), F.TRB_UNSUPPORTED), (dict(filter_h=float("nan")), F.TRB_INVALID_ARG)):
        film = dict(b.film, **change)
        with pytest.raises(api.TrbError) as ex:
            u.replace_settings(film)
        bad = base()
        bad.film.update(change)
        with pytest.raises(api.TrbError) as ex2:
            api.Scene(bad.finish())
        assert ex.value.status == ex2.value.status == status and str(ex.value) == str(ex2.value), change
        assert snapshot(u) == before and u.filter_table().tobytes() == table and (u.width, u.height) == (48, 32)
    assert lib.trb_scene_replace_settings(None, None, None) == F.TRB_INVALID_ARG
    assert lib.trb_scene_replace_settings(u._h, None, None) == F.TRB_OK  # nothing replaced
    assert snapshot(u) == before
    e.check()


def test_render_in_flight_on_a_side_stream_finishes_on_the_old_film():
    import torch
    b = base(w=256, h=256)
    e = Settled(b)
    ref, _ = e.fresh().render(spp=4, seed=7)
    s = torch.cuda.Stream()
    film = torch.zeros((256, 256, 4), dtype=torch.float32, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    e.u.render_device(film.data_ptr(), stream=s.cuda_stream, spp=4, seed=7)
    b.film.update(width=64, height=32)
    e.replace(integrator=False)  # frees the film state and block list the passes in flight read
    s.synchronize()
    assert rmse(film.cpu().numpy(), ref) < 1e-5
    e.check()


def test_a_hundred_replacements_do_not_grow_the_scene():
    import torch
    b = base()
    e = Settled(b)
    big, small = dict(b.film, width=512, height=512), dict(b.film, width=48, height=32)
    free = []
    for k in range(100):  # each large film holds about 5 MB of device film and Adaptive state
        e.u.replace_settings(big if k % 2 == 0 else small)
        if k % 2 == 0:
            e.u.render_adaptive(1, 1, seed=k)
        if k in (1, 99):
            torch.cuda.synchronize()
            free.append(torch.cuda.mem_get_info()[0])
    assert free[1] >= free[0] - (8 << 20), free
    e.check(film=False)


def test_one_device_group_replaced_through_its_replica():
    b = base()
    ga = api.Group(b.finish(), [0])
    b.film.update(width=64, height=16, samples=8)
    b.integrator = (F.INTEGRATOR_PATH, 2, 5)
    gb = api.Group(b.finish(), [0])
    lib = F.load_trb()
    rep = lib.trb_group_scene(ga._h, 0)
    assert rep
    assert lib.trb_scene_replace_settings(rep, F.Film(**b.film), F.Integrator(*b.integrator)) == F.TRB_OK, lib.trb_last_error()
    ga.width, ga.height = 64, 16
    (fa, sa), (fb, sb) = ga.render(spp=2, seed=3), gb.render(spp=2, seed=3)
    assert fa.shape == fb.shape and rmse(fa, fb) < 1e-5 and counters(sa) == counters(sb)


@pytest.mark.skipif("__import__('torch').cuda.device_count() < 2")
def test_group_of_two_refuses_replicas_of_different_film_sizes():
    b = base()
    g = api.Group(b.finish(), [0, 1])
    lib = F.load_trb()
    film = F.Film(**dict(b.film, width=64))
    assert lib.trb_scene_replace_settings(lib.trb_group_scene(g._h, 1), film, None) == F.TRB_OK
    with pytest.raises(api.TrbError) as ex:
        g.render(spp=1)
    assert ex.value.status == F.TRB_INVALID_ARG and "different film sizes" in str(ex.value)
    assert lib.trb_scene_replace_settings(lib.trb_group_scene(g._h, 0), film, None) == F.TRB_OK
    g.width = 64
    g.render(spp=1)
