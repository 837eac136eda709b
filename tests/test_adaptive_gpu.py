"""The Adaptive sampler on the GPU (trb_render_adaptive / trb_render_samples_adaptive) against the oracle's literal
thread_work + Adaptive: per-sample records bit-exact, per-pixel sample counts and ray / test counters equal, film RMSE."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_adaptive.pyadaptive import AdaptiveOracleScene

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SCENES = os.path.join(HERE, "golden", "scenes")
sys.path.insert(0, HERE)
KEYS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation", "node_tests", "tri_tests", "inst_tests"]


def img(film):
    return film[..., :3] / np.maximum(film[..., 3:], 1e-6)


def film_close(gf, of):
    assert np.allclose(gf, of, rtol=2e-4, atol=2e-5 * max(1.0, float(np.abs(of).max())))
    solid = of[..., 3] > 0.25 * float(of[..., 3].max())
    assert float(np.sqrt(np.mean((img(gf)[solid] - img(of)[solid]) ** 2))) < 1e-5


def load_json(name, w, h, spp):
    lib = F.load_trb()
    d = C.POINTER(F.SceneDesc)()
    assert lib.trb_desc_load_json(os.path.join(SCENES, name).encode(), w, h, spp, C.byref(d)) == F.TRB_OK, lib.trb_last_error()
    return d, lib


def check_adaptive(g, o, mn, mx, seed, frame=0, block_start=0, block_count=0, film=True):
    """records + counts + counters (both shadow modes), film of the same selection; returns the GPU pixel counts."""
    kw = dict(seed=seed, current_frame=frame, block_start=block_start, block_count=block_count)
    gs, gspp, gst = g.render_samples_adaptive(mn, mx, flags=F.RENDER_STATS | F.RENDER_REFERENCE_SHADOW, **kw)
    os_, ospp, ost = o.render_samples_adaptive(mn, mx, **kw)
    assert (gspp == ospp).all(), "per-pixel sample counts differ: %d pixels" % int((gspp != ospp).sum())
    assert gs.tobytes() == os_.tobytes(), "per-sample records differ"
    assert [getattr(gst, k) for k in KEYS] == [getattr(ost, k) for k in KEYS]
    assert int(gspp.sum()) == gst.camera_samples
    gs2, gspp2, gst2 = g.render_samples_adaptive(mn, mx, **kw)  # product default: any-hit shadow rays
    assert gs2.tobytes() == os_.tobytes() and (gspp2 == ospp).all() and gst2.rays_total() == ost.rays_total()
    if film:
        gf, fspp, fst = g.render_adaptive(mn, mx, flags=F.RENDER_NO_UPDATE, **kw)
        of, _, _ = o.render_adaptive(mn, mx, flags=F.RENDER_NO_UPDATE, **kw)
        assert (fspp == ospp).all() and int(fspp.sum()) == fst.camera_samples
        film_close(gf, of)
    return gspp


def test_c1_reduced_vs_oracle():
    d, lib = load_json("c1_cornell_box.json", 96, 96, 16)
    try:
        g, o = api.Scene(d.contents), AdaptiveOracleScene(d.contents)
        g.update_frame(0, 0.0, 0.0); o.update_frame(0, 0.0, 0.0)
        spp = check_adaptive(g, o, 4, 64, 3)
        assert spp.min() >= 4 and spp.max() <= 68 and (spp > 4).any()
    finally:
        lib.trb_desc_free(d)


def test_c2_smallpt_glass_and_metal_vs_oracle():
    d, lib = load_json("c2_smallpt.json", 128, 128, 16)
    try:
        g, o = api.Scene(d.contents), AdaptiveOracleScene(d.contents)
        g.update_frame(0, 0.0, 0.0); o.update_frame(0, 0.0, 0.0)
        spp = check_adaptive(g, o, 2, 32, 5)
        assert (spp > 2).mean() > 0.05, "glass and metal should make many pixels refine"
    finally:
        lib.trb_desc_free(d)


def test_zoo_and_split_shading_vs_oracle():
    desc = SB.scene_materials_zoo(64, 64, 8, SB.synthetic_merl_table()).finish()
    g, o = api.Scene(desc), AdaptiveOracleScene(desc)
    g.update_frame(0, 0.0, 0.0); o.update_frame(0, 0.0, 0.0)
    check_adaptive(g, o, 1, 16, 9)
    g.set_option("shade.split", 0)  # the fused shade kernel reads the same offset
    check_adaptive(g, o, 1, 16, 9, film=False)


def test_keyframed_scene_vs_oracle():
    desc = SB.scene_animated(48, 48, 4, frames=4, scene_time=1.0, animated_fov=True).finish()
    g, o = api.Scene(desc), AdaptiveOracleScene(desc)
    step = 1.0 / 4
    for frame in (0, 2):
        g.update_frame(frame, frame * step, (frame + 1) * step); o.update_frame(frame, frame * step, (frame + 1) * step)
        check_adaptive(g, o, 2, 16, 13, frame=frame)


def test_textured_scene_vs_oracle():
    from test_textures import textured_zoo
    desc = textured_zoo(8, 48).finish()
    g, o = api.Scene(desc), AdaptiveOracleScene(desc)
    g.update_frame(0, 0.0, 0.0); o.update_frame(0, 0.0, 0.0)
    check_adaptive(g, o, 2, 16, 17)


def test_pass_split_and_block_ranges_change_only_addition_order():
    desc = SB.scene_smallpt_like(128, 128, 16).finish()
    g = api.Scene(desc)
    full, spp, st = g.render_adaptive(2, 32, seed=4)
    assert int(spp.sum()) == st.camera_samples
    g.set_option("pass.paths", 64 * 32 * 3)  # a few blocks per pass
    again, spp2, st2 = g.render_adaptive(2, 32, seed=4)
    g.set_option("pass.paths", 1 << 24)
    assert (spp == spp2).all() and [getattr(st, k) for k in KEYS[:5]] == [getattr(st2, k) for k in KEYS[:5]]
    assert np.allclose(full, again, rtol=2e-4, atol=2e-5)
    nb = g.n_blocks()
    halves, s0spp, s0 = g.render_adaptive(2, 32, seed=4, block_start=0, block_count=nb // 2)
    _, s1spp, s1 = g.render_adaptive(2, 32, halves, seed=4, block_start=nb // 2, block_count=nb - nb // 2, flags=F.RENDER_NO_UPDATE)
    assert (s0spp + s1spp == spp).all() and s0.rays_total() + s1.rays_total() == st.rays_total()
    assert np.allclose(full, halves, rtol=2e-4, atol=2e-5)


def test_c4_full_size_one_call_vs_oracle_on_block_ranges():
    desc = SB.scene_c4(1_000_000, 1920, 1080, 4096).finish()
    g, o = api.Scene(desc), AdaptiveOracleScene(desc)
    film, spp, st = g.render_adaptive(4, 16, seed=1)
    assert int(spp.sum()) == st.camera_samples and spp.min() >= 4 and spp.max() <= 16
    assert np.isfinite(film).all() and (film[8:-8, 8:-8, 3] > 0).all()
    o.update_frame(0, 0.0, 0.0)
    nb = g.n_blocks()
    for start, count in [(3000, 300), (nb // 2 - 150, 300), (nb - 400, 300)]:
        part = check_adaptive(g, o, 4, 16, 1, block_start=start, block_count=count, film=False)
        sel = part > 0
        assert (part[sel] == spp[sel]).all(), "a pixel's count does not depend on the selection"


def test_error_statuses():
    desc = SB.scene_materials_zoo(16, 16, 4).finish()
    g = api.Scene(desc)
    for kw, status in [(dict(spp=4), F.TRB_INVALID_ARG), (dict(sample_first=1), F.TRB_INVALID_ARG), (dict(sample_count=2), F.TRB_INVALID_ARG),
                       (dict(flags=F.RENDER_MEGAKERNEL), F.TRB_UNSUPPORTED)]:
        with pytest.raises(api.TrbError) as e:
            g.render_adaptive(2, 8, **kw)
        assert e.value.status == status, kw
    with pytest.raises(api.TrbError) as e:
        g.render_adaptive(8, 4)
    assert e.value.status == F.TRB_INVALID_ARG
    b = SB.scene_materials_zoo(16, 16, 4)
    b.integrator = (F.INTEGRATOR_WHITTED, 0, 4)
    w = api.Scene(b.finish())
    with pytest.raises(api.TrbError) as e:
        w.render_adaptive(2, 8)
    assert e.value.status == F.TRB_UNSUPPORTED
