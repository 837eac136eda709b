"""Small scenes under compute-sanitizer (memcheck / racecheck / initcheck): wavefront and megakernel, film and samples."""
import sys, os
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tray_rust_b200 import _ffi as F, api, scenebuild as SB
for name, b in (("zoo", SB.scene_materials_zoo(32, 32, 4, SB.synthetic_merl_table())), ("c4_5k", SB.scene_c4(5000, 64, 32, 4))):
    g = api.Scene(b.finish())
    g.update_frame(0, 0.0, 0.0)
    film, st = g.render(seed=3)                          # default film kernel (k_wf_film_v2: per-warp private tiles, lockstep RMW)
    g.set_option("film.v2", 0)
    film_a, _ = g.render(seed=3)                         # shared-memory-atomics film kernel
    g.set_option("film.v2", 1)
    g.set_option("pass.paths", 4096)                     # several internal passes per call
    film_p, _ = g.render(seed=3)
    g.set_option("pass.paths", 1 << 24)
    assert np.allclose(film, film_a, rtol=1e-4, atol=1e-5) and np.allclose(film, film_p, rtol=1e-4, atol=1e-5)
    s, _ = g.render_samples(seed=3, flags=F.RENDER_STATS)
    s2, _ = g.render_samples(seed=3, flags=F.RENDER_MEGAKERNEL)
    f2, _ = g.render(seed=3, flags=F.RENDER_MEGAKERNEL)
    rays, _ = g.camera_rays(seed=3)
    h, _ = g.intersect(rays)
    print(name, "ok", st.rays_total(), s.tobytes() == s2.tobytes(), float(np.abs(film - f2).max()), g.to_srgb8(film).mean())
    g.close()
# a filter whose reach exceeds filter_pixel_width (the 2x2 lock-block sample rule) through both film kernels
bw = SB.scene_smallpt_like(32, 32, 4)
bw.film.update(filter_type=F.FILTER_GAUSSIAN, filter_w=3.0, filter_h=2.5, filter_b=0.5, filter_c=0.0)
g = api.Scene(bw.finish())
fa, _ = g.render(seed=3)
g.set_option("film.v2", 0)
fb, _ = g.render(seed=3)
print("wide filter ok", bool(np.allclose(fa, fb, rtol=1e-4, atol=1e-5)))
g.close()
# image textures, split shade kernels, ray-queue sorting, the Whitted kernel
import importlib.util
spec = importlib.util.spec_from_file_location("tt", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "test_textures.py"))
tt = importlib.util.module_from_spec(spec); spec.loader.exec_module(tt)
g = api.Scene(tt.textured_zoo(4, 32).finish())
g.update_frame(1, 0.5, 1.0)
a, _ = g.render_samples(seed=3)
g.set_option("shade.split", 1); g.set_option("sort.mode", 1)
b2, _ = g.render_samples(seed=3)
film_t, _ = g.render(seed=3, flags=F.RENDER_NO_UPDATE)
print("textured / split / sorted ok", a.tobytes() == b2.tobytes(), float(film_t.sum()) > 0)
g.close()
bw2 = SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()); bw2.integrator = (F.INTEGRATOR_WHITTED, 0, 3)
g = api.Scene(bw2.finish())
fw, stw = g.render(seed=3)
print("whitted ok", stw.rays_total(), float(fw.sum()) > 0)
g.close()
# keyframed kernels (ANIM variants) and the optional DQuad records
g = api.Scene(SB.scene_animated(32, 32, 4).finish())
for fr in (0, 2):
    g.update_frame(fr, fr * 0.25, (fr + 1) * 0.25)
    film, st = g.render(seed=3, flags=F.RENDER_NO_UPDATE)
    s, _ = g.render_samples(seed=3, flags=F.RENDER_STATS)
    s2, _ = g.render_samples(seed=3, flags=F.RENDER_MEGAKERNEL)
    print("animated frame", fr, "ok", st.rays_total(), s.tobytes() == s2.tobytes())
g.close()
g = api.Scene(SB.scene_c4(5000, 64, 32, 4).finish())
g.update_frame(0, 0.0, 0.0)
g.set_option("trace.quads", 1)
a, _ = g.render_samples(seed=3)
g.set_option("trace.quads", 0)
b, _ = g.render_samples(seed=3)
print("quads ok", a.tobytes() == b.tobytes())
g.close()
# round-2 trace variants: forced literal box test, the round-1 kernel, the box self-test
import ctypes as C
g = api.Scene(SB.scene_c4(5000, 64, 32, 4).finish())
g.update_frame(0, 0.0, 0.0)
ref, _ = g.render_samples(seed=3)
g.set_option("trace.exact_box", 1); a, _ = g.render_samples(seed=3)
g.set_option("trace.exact_box", 0); g.set_option("trace.pipe", 0); b, _ = g.render_samples(seed=3)
out = (C.c_uint64 * 4)()
rc = F.load_trb().trb_selftest_box(1 << 16, 5, out)
print("trace variants ok", a.tobytes() == ref.tobytes(), b.tobytes() == ref.tobytes(), rc, [int(x) for x in out])
g.close()
# the Adaptive sampler: adaptive generate / decide / compaction kernels and the ADAPT film variants (both film kernels), several passes
g = api.Scene(SB.scene_smallpt_like(32, 32, 4).finish())
fa, spp, st = g.render_adaptive(1, 16, seed=3)
g.set_option("film.v2", 0); g.set_option("pass.paths", 64 * 16 * 2)
fb, spp2, _ = g.render_adaptive(1, 16, seed=3)
rec, spp3, _ = g.render_samples_adaptive(1, 16, seed=3)
print("adaptive ok", int(spp.sum()) == st.camera_samples, bool((spp == spp2).all() and (spp == spp3).all()), bool(np.allclose(fa, fb, rtol=1e-4, atol=1e-5)))
g.close()
# a mesh refit (k_refit_parents, k_refit_tris, k_refit_nodes) on both leaf forms, the host tree read back, then a render of it
hf = SB.heightfield_mesh(64, 7)
g = api.Scene(SB.scene_heightfield(64, 32, 32, 2).finish())
g.update_frame(0, 0.0, 0.0)
for wide in (0, 1):
    g.set_option("trace.wide_leaf", wide)
    p = hf[0].copy(); p[:, 1] += np.sin(p[:, 0] + wide).astype(np.float32)
    g.refit_mesh(0, p)
    nodes, _ = g.bvh(0)
    s, st = g.render_samples(seed=3, flags=F.RENDER_STATS)
    print("refit ok", wide, len(nodes), st.rays_total())
g.close()
# AOV renders (k_wf_aov, k_wf_film_aov): per-sample records and films, keyframed and static
for d in (SB.scene_animated(32, 32, 2).finish(), SB.scene_materials_zoo(32, 32, 2, SB.synthetic_merl_table()).finish()):
    g = api.Scene(d)
    g.update_frame(1, 0.25, 0.5)
    _, aov, _ = g.render_samples_aov(seed=3)
    _, aovs, _ = g.render_aov(seed=3, flags=F.RENDER_NO_UPDATE)
    print("aov ok", int((aov["inst"] != F.MISS).sum()), float(aovs["albedo_w"][..., 3].sum()))
    g.close()
# the denoiser (k_dn_prepare, k_dn_atrous): a block-range render leaves zero-weight pixels; every iteration count's step reaches the
# borders of a 40 x 24 image
g = api.Scene(SB.scene_c4(5000, 40, 24, 4).finish())
g.update_frame(0, 0.0, 0.0)
den, film, aovs, _ = g.render_denoised(4, seed=3, block_start=2, block_count=10)
for it in (0, 1, 10):
    d = g.denoise(film, film, aovs, iterations=it)
print("denoise ok", float(den[..., :3].sum()), int((den[..., 3] == 0).sum()))
g.close()
# the temporal denoiser (k_dn_temporal): three frames of the keyframed scene with motion and history lengths, taps reaching the borders,
# then a history reset
g = api.Scene(SB.scene_animated(40, 24, 2).finish())
hist = api.DenoiseHistory(g)
for k in range(3):
    den, film, aovs, _ = g.render_denoised_temporal(hist, 2, seed=3, current_frame=k)
    _, motion, hl = g.denoise_temporal(hist, film, film, aovs, motion=True, history_length=True, iterations=1)
hist.reset()
print("denoise temporal ok", float(den[..., :3].sum()), int(hl.max()), int(np.isnan(motion).sum()))
g.close()
# the temporal gradients (k_gr_*, k_dn_temporal_grad): four frames of the keyframed scene with every output, the records re-shaded
# from the second frame on, the last with no a-trous pass, then a reset
g = api.Scene(SB.scene_animated(40, 24, 2).finish())
hist = api.DenoiseHistory(g)
for k in range(4):
    den, film, aovs, _ = g.render_denoised_temporal(hist, 2, seed=3, current_frame=k, gradients=True)
_, motion, hl, lam = g.denoise_temporal_gradient(hist, film, film, aovs, 9, motion=True, history_length=True, lam=True, gradient_iterations=0)
hist.reset()
print("denoise gradient ok", float(den[..., :3].sum()), int(hl.max()), float(lam.max()))
g.close()
# the moment denoiser (k_dn_temporal_moments, k_dn_moments_variance): six 1-spp frames of the keyframed scene with every output, so
# both variance branches and the 7x7 taps at the borders run, the last with no a-trous pass, then a reset
g = api.Scene(SB.scene_animated(40, 24, 1).finish())
hist = api.DenoiseHistory(g)
for k in range(6):
    den, film, aovs, _ = g.render_denoised_moments(hist, 1, seed=3, current_frame=k)
_, motion, hl, var = g.denoise_moments(hist, film, aovs, motion=True, history_length=True, variance=True, iterations=0)
hist.reset()
print("denoise moments ok", float(den[..., :3].sum()), int(hl.max()), float(np.nanmax(var)))
g.close()
# the moment gradients (k_gr_*, k_dn_temporal_moments_grad): five 1-spp frames of the keyframed scene, the records re-shaded from the
# second frame on, the last with every output and no a-trous pass, then a reset
g = api.Scene(SB.scene_animated(40, 24, 1).finish())
hist = api.DenoiseHistory(g)
for k in range(5):
    den, film, aovs, _ = g.render_denoised_moments(hist, 1, seed=3, current_frame=k, gradients=True)
_, motion, hl, var, lam = g.denoise_moments_gradient(hist, film, aovs, 9, motion=True, history_length=True, variance=True, lam=True,
                                                     gradient_iterations=0)
hist.reset()
print("denoise moment gradient ok", float(den[..., :3].sum()), int(hl.max()), float(lam.max()))
g.close()
