"""AOV renders on an H100 (k_wf_aov between the round-0 trace and shade; the colour film kernel over the records, and k_wf_nearest, after
the colour film): every camera sample's
AOV record equals the oracle's orc_render_samples_aov bit for bit (Cornell, smallpt, the material zoo with MERL, textures, a keyframed
scene at two frames, C4 with wide leaves; split and fused shading; after material replacement and a mesh refit), the colour render
is unchanged, normals, depths and instances agree with NormalsDebug and the ray queries, and the films agree with trb_film_write of the
records."""
import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_aov import pyaov as A
from test_queries_gpu import json_desc
from test_textures import textured_zoo

pytestmark = pytest.mark.gpu
FILM_TOL = dict(rtol=1e-4, atol=1e-5)
COUNTERS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation", "node_tests", "tri_tests", "inst_tests"]


def _integrator(b, integ):
    b.integrator = integ
    return b


def partial_wall(integrator=(F.INTEGRATOR_PATH, 4, 8)):
    """a 4 x 4 plastic square in front of the camera, which sees past its edges: hits and misses in one frame"""
    b = SB.SceneBuilder(32, 32, 2)
    b.integrator = integrator
    m = b.add_material(F.MAT_PLASTIC, c0=(0.2, 0.4, 0.6), c1=(0.5, 0.5, 0.5), roughness=0.1)
    b.receiver(F.SHAPE_RECT, m, [SB.trs(q=SB.quat_axis_angle((1, 1, 0), 20))], p0=4.0, p1=4.0)
    b.point_light([SB.trs(t=(0, 0, -5))], (1, 1, 1, 10))
    b.add_camera([SB.trs(t=(0, 0, -10))], fov=30.0)
    return b


SCENES = {
    "partial": lambda: (partial_wall().finish(), (0, 0.0, 0.0)),
    "c1": lambda: (json_desc("c1_cornell_box.json", 32, 24, 2), (0, 0.0, 0.0)),
    "c2": lambda: (json_desc("c2_smallpt.json", 32, 32, 2), (0, 0.0, 0.0)),
    "zoo": lambda: (SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()).finish(), (0, 0.0, 0.0)),
    "textured": lambda: (textured_zoo(2, 32).finish(), (1, 0.5, 1.0)),
    "keyframed_f1": lambda: (SB.scene_animated(32, 32, 2).finish(), (1, 0.25, 0.5)),
    "keyframed_f2": lambda: (SB.scene_animated(32, 32, 2).finish(), (2, 0.5, 0.75)),
}


def assert_records_equal(got, want):
    assert got.dtype == want.dtype == F.AOV_SAMPLE_DTYPE and len(got) == len(want)
    assert got.tobytes() == want.tobytes()


def stats_equal(a, b):
    return all(getattr(a, k) == getattr(b, k) for k in COUNTERS)


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_records_equal_the_oracle_and_the_render_is_unchanged(name, split):
    desc, frame = SCENES[name]()
    g, o = api.Scene(desc), A.AovOracleScene(desc)
    g.update_frame(*frame); o.update_frame(*frame)
    g.set_option("shade.split", split)
    samples, aov, st = g.render_samples_aov(seed=7, flags=F.RENDER_STATS)
    _, want, _ = o.render_samples_aov(seed=7)
    assert_records_equal(aov, want)
    plain, st0 = g.render_samples(seed=7, flags=F.RENDER_STATS)
    assert samples.tobytes() == plain.tobytes() and stats_equal(st, st0)
    assert (aov["inst"] != F.MISS).any()


def test_c4_wide_leaves():
    desc = SB.scene_c4(1_000_000, 64, 64, 2).finish()
    g, o = api.Scene(desc), A.AovOracleScene(desc)
    g.update_frame(); o.update_frame()
    g.set_option("trace.wide_leaf", 1)
    samples, aov, st = g.render_samples_aov(seed=3, flags=F.RENDER_STATS)
    assert_records_equal(aov, o.render_samples_aov(seed=3)[1])
    plain, st0 = g.render_samples(seed=3, flags=F.RENDER_STATS)
    assert samples.tobytes() == plain.tobytes() and stats_equal(st, st0)


@pytest.mark.parametrize("name", ["zoo", "partial"])
def test_normals_depths_and_instances_agree_with_normals_debug_and_the_ray_queries(name):
    desc, frame = SCENES[name]()
    g = api.Scene(desc)
    g.update_frame(*frame)
    _, aov, _ = g.render_samples_aov(seed=5)
    hit = aov["inst"] != F.MISS
    assert hit.any() and (name == "zoo" or (~hit).any())
    b = SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()) if name == "zoo" else partial_wall()
    nd = api.Scene(_integrator(b, (F.INTEGRATOR_NORMALS_DEBUG, 0, 0)).finish())
    nd.update_frame(*frame)
    col, _ = nd.render_samples(seed=5)
    want = np.clip((aov["n"] + np.float32(1.0)) / np.float32(2.0), 0, 1).astype(np.float32)
    got = np.stack([col["r"], col["g"], col["b"]], axis=1)
    assert np.array_equal(got[hit], want[hit]) and not got[~hit].any()  # NormalsDebug's miss is black
    rays, _ = g.camera_rays(seed=5)  # a static scene: the rays' time does not matter
    q = np.zeros(len(rays), F.QUERY_RAY_DTYPE)
    q["o"], q["d"], q["min_t"], q["max_t"] = rays["o"], rays["d"], rays["min_t"], rays["max_t"]
    rec, _ = g.intersect_records(q)
    assert np.array_equal(rec["inst"], aov["inst"])
    assert np.array_equal(rec["t"].view(np.uint32), aov["depth"].view(np.uint32))


def pixel_of_samples(g, **kw):
    """the pixel (y * width + x) every camera sample was taken for, in render_samples order"""
    xy = g.block_list(kw.get("block_start", 0), kw.get("block_count", 0)).astype(np.int64)
    n = len(g.sample_regions(**kw))
    per = n // (len(xy) * 64)
    k = np.arange(64)
    px = (xy[:, 0:1] * 8 + k % 8)[:, :, None].repeat(per, 2).reshape(-1)
    py = (xy[:, 1:2] * 8 + k // 8)[:, :, None].repeat(per, 2).reshape(-1)
    return py * g.width + px


def host_nearest(g, aov, **kw):
    key = (aov["depth"].view(np.uint32).astype(np.uint64) << np.uint64(32)) | aov["inst"].astype(np.uint64)
    out = np.full(g.width * g.height, np.iinfo(np.uint64).max, np.uint64)
    np.minimum.at(out, pixel_of_samples(g, **kw), key)
    return out.reshape(g.height, g.width)


@pytest.mark.parametrize("name", ["c1", "zoo", "keyframed_f1", "partial"])
def test_films_equal_film_writes_of_the_records_and_the_colour_render_is_unchanged(name):
    desc, frame = SCENES[name]()
    g = api.Scene(desc)
    g.update_frame(*frame)
    kw = dict(seed=11, flags=F.RENDER_STATS | F.RENDER_NO_UPDATE)
    film, aovs, st = g.render_aov(**kw)
    ref, st0 = g.render(**kw)
    np.testing.assert_allclose(film, ref, **FILM_TOL)
    assert stats_equal(st, st0)
    samples, aov, _ = g.render_samples_aov(seed=11)
    regions = g.sample_regions(seed=11)
    for key, field in (("albedo_w", "albedo"), ("normal_w", "n")):
        s = samples.copy()
        s["r"], s["g"], s["b"] = aov[field][:, 0], aov[field][:, 1], aov[field][:, 2]
        np.testing.assert_allclose(aovs[key], g.film_write(s, regions), **FILM_TOL)
        np.testing.assert_allclose(aovs[key][..., 3], film[..., 3], **FILM_TOL)
    assert np.array_equal(aovs["nearest"], host_nearest(g, aov, seed=11))


def test_nearest_composes_across_calls_and_passes():
    desc, frame = SCENES["partial"]()
    g = api.Scene(desc)
    g.update_frame(*frame)
    kw = dict(seed=2, spp=4, flags=F.RENDER_NO_UPDATE)
    _, aov, _ = g.render_samples_aov(**kw)
    want = host_nearest(g, aov, **kw)
    _, one, _ = g.render_aov(**kw)
    assert np.array_equal(one["nearest"], want)
    assert (want == np.uint64(0x7f800000ffffffff)).any() and (want != np.uint64(0x7f800000ffffffff)).any()  # all-miss pixels and hit pixels
    near = np.full((g.height, g.width), np.iinfo(np.uint64).max, np.uint64)
    film = np.zeros((g.height, g.width, 4), np.float32)
    for first in (0, 2):  # two calls by sample range into the same buffers
        g.render_aov(film, albedo=False, normal=False, nearest=near, sample_first=first, sample_count=2, **kw)
    assert np.array_equal(near, want)
    g.set_option("pass.paths", 1000)  # several passes per call
    _, many, _ = g.render_aov(**kw)
    assert np.array_equal(many["nearest"], want)
    np.testing.assert_allclose(many["albedo_w"], one["albedo_w"], **FILM_TOL)


def test_device_form_on_a_torch_stream_equals_the_host_form_and_each_output_may_be_null():
    import torch
    desc, frame = SCENES["zoo"]()
    g = api.Scene(desc)
    g.update_frame(*frame)
    kw = dict(seed=4, flags=F.RENDER_NO_UPDATE)
    film, aovs, _ = g.render_aov(**kw)
    h, w = g.height, g.width
    for keep in (("albedo_w", "normal_w", "nearest"), ("albedo_w",), ("normal_w",), ("nearest",), ()):
        d = dict(film=torch.zeros((h, w, 4), dtype=torch.float32, device="cuda"),
                 albedo_w=torch.zeros((h, w, 4), dtype=torch.float32, device="cuda"),
                 normal_w=torch.zeros((h, w, 4), dtype=torch.float32, device="cuda"),
                 nearest=torch.full((h, w), -1, dtype=torch.int64, device="cuda"))
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            g.render_aov_device(d["film"].data_ptr(), *(d[k].data_ptr() if k in keep else None for k in ("albedo_w", "normal_w", "nearest")),
                                stream=st.cuda_stream, **kw)
        st.synchronize()
        np.testing.assert_allclose(d["film"].cpu().numpy(), film, **FILM_TOL)
        for k in ("albedo_w", "normal_w"):
            got = d[k].cpu().numpy()
            if k in keep:
                np.testing.assert_allclose(got, aovs[k], **FILM_TOL)
            else:
                assert not got.any()
        near = d["nearest"].cpu().numpy().view(np.uint64)
        assert np.array_equal(near, aovs["nearest"] if "nearest" in keep else np.full((h, w), np.iinfo(np.uint64).max, np.uint64))


def test_records_follow_replace_materials_and_refit_mesh():
    b = SB.SceneBuilder(32, 32, 2)
    mats = SB.cornell_walls(b)
    SB.cornell_light(b, mats["white"])
    mb = SB.heightfield_mesh(8, 1)
    m = b.add_mesh(*mb)
    b.receiver(F.SHAPE_MESH, mats["white"], [SB.trs()], mesh=m)
    b.add_camera([SB.trs(t=(0, 12, -60))])
    g = api.Scene(b.finish())
    g.update_frame()
    g.render_samples_aov(seed=9)  # the AOV path state exists before the edits
    b.materials[mats["white"]] = (F.MAT_PLASTIC, (0.3, 0.6, 0.2), (0.8, 0.8, 0.8), 0.1, 1.0, 0, (0, 0, 0, 0))
    g.replace_materials(b.materials_section())
    p = mb[0].copy()
    p[:, 1] += np.float32(2.0) * np.sin(p[:, 0]).astype(np.float32)
    g.refit_mesh(m, p)
    o = A.AovOracleScene(b.finish())  # the new materials over the created mesh, then the same refit: the kept tree
    o.update_frame()
    o.refit_mesh(m, p)
    _, aov, _ = g.render_samples_aov(seed=9)
    assert_records_equal(aov, o.render_samples_aov(seed=9)[1])
    assert (aov["inst"] == len(b.instances) - 1).any()


def test_statuses():
    import torch
    desc, frame = SCENES["zoo"]()
    for integ in (F.INTEGRATOR_WHITTED, F.INTEGRATOR_NORMALS_DEBUG):
        s = api.Scene(_integrator(SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()), (integ, 0, 4)).finish())
        s.update_frame()
        for call in (lambda: s.render_aov(), lambda: s.render_samples_aov()):
            with pytest.raises(api.TrbError) as e:
                call()
            assert e.value.status == F.TRB_UNSUPPORTED
    g = api.Scene(desc)
    g.update_frame(*frame)
    for call in (lambda: g.render_aov(flags=F.RENDER_MEGAKERNEL), lambda: g.render_samples_aov(flags=F.RENDER_MEGAKERNEL)):
        with pytest.raises(api.TrbError) as e:
            call()
        assert e.value.status == F.TRB_UNSUPPORTED
    film = torch.zeros(g.height * g.width * 4 + 4, dtype=torch.float32, device="cuda")
    near = torch.zeros(g.height * g.width + 1, dtype=torch.int64, device="cuda")
    base, nb = film.data_ptr(), near.data_ptr()
    for args in ((base + 4, None, None, None), (base, base + 8, None, None), (base, None, base + 4, None), (base, None, None, nb + 4)):
        with pytest.raises(api.TrbError) as e:
            g.render_aov_device(*args)
        assert e.value.status == F.TRB_INVALID_ARG
    torch.cuda.synchronize()
