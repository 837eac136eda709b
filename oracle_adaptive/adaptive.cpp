/* The parity oracle plus the reference's Adaptive sampler (src/sampler/adaptive.rs) driven by thread_work
 * (src/exec/multithreaded.rs:72-114) — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into
 * oracle/_build/liboracle_adaptive.so and loaded by oracle_adaptive/pyadaptive.py.
 *
 * This translation unit is the detmath oracle (oracle/oracle.cpp, included whole, so every orc_* entry point is here too) with
 * one difference: LowDiscrepancy's per-path sample arrays are filled at offset 0 (ld.rs:57,62), the Adaptive sampler's at
 * samples_taken (adaptive.rs:110,115). Entry b of a shuffled array is sample_02(perm(b) + offset, scramble); PathSamples
 * (orc_shade.h) computes perm(b) with dm_permute and nothing else there calls it, so the offset is added by wrapping
 * dm_permute for orc_shade.h only. It is 0 except while an Adaptive camera sample is being shaded, so the LowDiscrepancy entry
 * points of this library compute exactly what liboracle_det.so computes.
 */
#include <cstdint>
#include "../include/trb.h"
#include "../oracle/detmath.h"

static thread_local uint32_t t_ld_offset = 0; /* samples_taken of the Adaptive round being shaded on this thread */
static inline uint32_t dm_permute_with_ld_offset(uint32_t i, uint32_t l, uint32_t p) { return dm_permute(i, l, p) + t_ld_offset; }
#define dm_permute dm_permute_with_ld_offset
#include "../oracle/orc_shade.h"
#undef dm_permute
#include "../oracle/oracle.cpp"

/* ---- the Adaptive sampler (sampler/adaptive.rs) driven by thread_work (multithreaded.rs:72-114) ----------------------------
 * Literal: the pixel's whole sample list is kept and needs_supersampling walks all of it. RNG streams (DESIGN.md §2): round r of
 * a pixel draws its position / time scrambles and shuffle keys from (seed, pixel, DM_AD_PIXEL_STREAM0 - r, dim); the camera
 * sample in slot i (its index in the pixel's list) uses (seed, pixel, i, dim) like LowDiscrepancy's sample i. */
#define DM_AD_PIXEL_STREAM0 0xfffffffeU
static inline uint32_t usize_next_power_of_two(uint32_t v) { uint32_t p = 1; while (p < v) p <<= 1; return p; }
struct Adaptive {
    uint32_t min_spp, max_spp, step_size, samples_taken = 0, round = 0;
    float avg_luminance = 0.0f;
    /* Adaptive::new (adaptive.rs:34-49); false where the reference's `max_spp - min_spp` underflows (it panics) */
    bool init(uint32_t min_in, uint32_t max_in) {
        if (min_in > (1u << 24) || max_in > (1u << 24)) return false;
        min_spp = usize_next_power_of_two(min_in); max_spp = usize_next_power_of_two(max_in);
        if (max_spp < min_spp) return false;
        step_size = usize_next_power_of_two((max_spp - min_spp) / 5);
        return true;
    }
    /* get_samples (adaptive.rs:82-106): how many samples this round takes; samples_taken is increased first */
    uint32_t begin_round() {
        if (samples_taken == 0) { samples_taken += min_spp; return min_spp; }
        samples_taken += step_size;
        return step_size;
    }
    /* needs_supersampling (adaptive.rs:54-78) */
    bool needs_supersampling(const std::vector<ImageSample>& samples) {
        const float max_contrast = 0.5f;
        if (samples_taken == min_spp) {
            float ac = 0.0f;
            for (const ImageSample& s : samples) ac = ac + s.color.luminance();
            avg_luminance = ac / (float)samples.size();
        } else {
            const size_t prev_samples = samples.size() - step_size;
            float ac = avg_luminance;
            for (size_t i = prev_samples; i < samples.size(); ++i) ac = (samples[i].color.luminance() + (float)(i - 1) * ac) / (float)i;
            avg_luminance = ac;
        }
        for (const ImageSample& s : samples)
            if (fabsf(s.color.luminance() - avg_luminance) / avg_luminance > max_contrast) return true;
        return false;
    }
    /* report_results (adaptive.rs:127-141): true = the pixel is done */
    bool report_results(const std::vector<ImageSample>& samples) { return samples_taken >= max_spp || !needs_supersampling(samples); }
};
static uint32_t adaptive_max_per_pixel(const Adaptive& a) {
    const uint32_t k = (a.max_spp - a.min_spp + a.step_size - 1) / a.step_size;
    return a.min_spp + k * a.step_size;
}

/* mode 0: splat to film; 1: dump samples (max_per_pixel slots per pixel, unused ones zero) */
static int render_adaptive_impl(orc_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, int mode, float* film, trb_sample* out_samples,
                                size_t n_out, uint32_t* pixel_spp, trb_stats* stats, int threads) {
    if (s->active_camera < 0) { g_err = "update_frame must be called before rendering"; return TRB_INVALID_ARG; }
    if (cfg->spp || cfg->sample_first || cfg->sample_count) { g_err = "the Adaptive sampler owns the sample schedule"; return TRB_INVALID_ARG; }
    Adaptive proto;
    if (!proto.init(ad->min_spp, ad->max_spp)) { g_err = "max_spp < min_spp after rounding"; return TRB_INVALID_ARG; }
    if (s->shade.integrator != TRB_INTEGRATOR_PATH) { g_err = "the Adaptive sampler is built for the path integrator only"; return TRB_UNSUPPORTED; }
    const uint32_t mpp = adaptive_max_per_pixel(proto);
    auto blocks = s->block_list(cfg->block_start, cfg->block_count);
    if (mode == 1 && n_out != blocks.size() * 64 * (size_t)mpp) { g_err = "output size mismatch"; return TRB_INVALID_ARG; }
    const Camera& camera = s->cameras[s->active_camera];
    const uint32_t width = s->film.width;
    Counters total;
    auto t0 = std::chrono::steady_clock::now();
#ifdef _OPENMP
    const int nt = threads > 0 ? threads : omp_get_max_threads();
#else
    const int nt = 1;
#endif
    (void)nt;
#pragma omp parallel num_threads(nt)
    {
        Counters cnt;
        std::vector<ImageSample> block_samples, pixel_samples;
#pragma omp for schedule(dynamic, 1)
        for (long bi = 0; bi < (long)blocks.size(); ++bi) {
            uint32_t bx = blocks[bi].first * 8, by = blocks[bi].second * 8;
            block_samples.clear();
            for (uint32_t py = by; py < by + 8; ++py)
                for (uint32_t px = bx; px < bx + 8; ++px) {
                    const uint32_t pixel = py * width + px;
                    Adaptive sampler = proto;
                    pixel_samples.clear(); /* block_samples[pixel_samples..] of thread_work */
                    for (;;) {
                        const uint32_t n = sampler.begin_round();
                        const uint32_t offset = sampler.samples_taken, round = sampler.round++;
                        const uint32_t hs_pos0 = dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_POS0);
                        const uint32_t scr0 = dm_scramble(hs_pos0), scr1 = dm_scramble(dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_POS1));
                        const uint32_t kpos = dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_POS_PERM);
                        const uint32_t scrt = dm_scramble(dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_TIME));
                        const uint32_t ktime = dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_TIME_PERM);
                        for (uint32_t e = 0; e < n; ++e) {
                            const uint32_t slot = (uint32_t)pixel_samples.size();
                            /* get_samples: sample_2d(.., samples_taken) shuffled over n entries; get_samples_1d over max_spp entries */
                            const uint32_t ip = dm_permute(e, n, kpos) + offset;
                            const float sx = van_der_corput(ip, scr0) + (float)px;
                            const float sy = sobol(ip, scr1) + (float)py;
                            const float tm = van_der_corput(dm_permute(e, sampler.max_spp, ktime) + offset, scrt);
                            Ray ray = camera.generate_ray(sx, sy, tm);
                            cnt.camera_samples++;
                            Hit hit;
                            Col c(0.0f);
                            cnt.rays[0]++;
                            if (s->geom.intersect(ray, hit, cnt)) {
                                PathSamples ps{cfg->seed, pixel, slot, s->shade.max_depth + 1};
                                t_ld_offset = offset; /* the per-path arrays: sample_02(perm(b) + samples_taken) */
                                c = s->shade.illumination(ray, hit, ps, cnt).clamp(); /* multithreaded.rs:98-99 */
                                t_ld_offset = 0;
                            }
                            pixel_samples.push_back(ImageSample{sx, sy, c});
                            if (mode == 1) {
                                trb_sample& o = out_samples[((size_t)bi * 64 + (py - by) * 8 + (px - bx)) * mpp + slot];
                                o.x = sx; o.y = sy; o.r = c.r; o.g = c.g; o.b = c.b;
                            }
                        }
                        if (sampler.report_results(pixel_samples)) break;
                    }
                    if (pixel_spp) pixel_spp[pixel] = (uint32_t)pixel_samples.size();
                    block_samples.insert(block_samples.end(), pixel_samples.begin(), pixel_samples.end());
                }
            if (mode == 0) s->rt.write(block_samples, (int)bx, (int)by, (int)bx + 8, (int)by + 8, film, true);
        }
#pragma omp critical
        total.add(cnt);
    }
    auto t1 = std::chrono::steady_clock::now();
    if (stats) {
        memset(stats, 0, sizeof *stats);
        stats->camera_samples = total.camera_samples;
        stats->rays_primary = total.rays[0]; stats->rays_shadow = total.rays[1]; stats->rays_mis = total.rays[2]; stats->rays_continuation = total.rays[3];
        stats->node_tests = total.node_tests; stats->tri_tests = total.tri_tests; stats->inst_tests = total.inst_tests;
        stats->kernel_ms = std::chrono::duration<float, std::milli>(t1 - t0).count();
    }
    return TRB_OK;
}
extern "C" {
int orc_render_adaptive(orc_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* film_rgbw, uint32_t* pixel_spp, trb_stats* stats, int threads) {
    if (!(cfg->flags & TRB_RENDER_NO_UPDATE)) {
        float time_step = s->film.scene_time / (float)s->film.frames;
        s->update_frame(cfg->current_frame, (float)cfg->current_frame * time_step, ((float)cfg->current_frame + 1.0f) * time_step);
    }
    return render_adaptive_impl(s, cfg, ad, 0, film_rgbw, nullptr, 0, pixel_spp, stats, threads);
}
int orc_render_samples_adaptive(orc_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, size_t n, trb_sample* samples, uint32_t* pixel_spp,
                                trb_stats* stats, int threads) {
    return render_adaptive_impl(s, cfg, ad, 1, nullptr, samples, n, pixel_spp, stats, threads);
}
/* Adaptive::new's rounded schedule and the largest per-pixel sample count */
int orc_adaptive_schedule(const trb_adaptive* ad, uint32_t* out4) {
    Adaptive a;
    if (!a.init(ad->min_spp, ad->max_spp)) { g_err = "max_spp < min_spp after rounding"; return TRB_INVALID_ARG; }
    out4[0] = a.min_spp; out4[1] = a.max_spp; out4[2] = a.step_size; out4[3] = adaptive_max_per_pixel(a);
    return TRB_OK;
}

} // extern "C"
