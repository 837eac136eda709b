/* The parity oracle's AOV records — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into oracle/_build/liboracle_aov.so
 * and loaded by oracle_aov/pyaov.py.
 *
 * This translation unit is the mesh-refit oracle (oracle_refit/refit.cpp: the ray-query oracle plus orc_scene_refit_mesh, all
 * included whole and unchanged) plus
 *   orc_render_samples_aov  for every camera sample of the selection, in orc_render_samples' order, the AOV record of its primary hit
 *                           (DESIGN.md §4 "AOVs"): the camera ray of render_impl, Scene::intersect, then Material::bsdf at the hit's
 *                           DifferentialGeometry. depth = the ray's max_t after the walk (+inf on a miss), inst = the instance or
 *                           TRB_MISS, n = BSDF::n (bsdf.rs:38-44), albedo = the sum over the BSDF's lobes, in allocation order, of
 *                           colour x the lobe's own Fresnel at cos 1 (diffuse lobes: colour; transmission lobes: colour x (1 - F));
 *                           MERL: pi x BSDF::eval(n, n, all lobes); each channel clamped to [0, 1]; zero on a miss.
 *                           samples (may be NULL) and stats receive orc_render_samples' records and counters of the same selection.
 */
#include "../oracle_refit/refit.cpp"
#include "aov_albedo.h"

extern "C" {

int orc_render_samples_aov(orc_scene* s, const trb_render_cfg* cfg, size_t n, trb_sample* samples, trb_aov_sample* aov, trb_stats* stats) {
    if (s->active_camera < 0) { g_err = "update_frame must be called before rendering"; return TRB_INVALID_ARG; }
    const uint32_t spp = cfg->spp ? next_pow2(cfg->spp) : s->spp_pow2;
    const uint32_t s_first = cfg->sample_first, s_count = cfg->sample_count ? cfg->sample_count : spp - std::min(spp, s_first);
    if (s_first + s_count > spp) { g_err = "sample range exceeds spp"; return TRB_INVALID_ARG; }
    auto blocks = s->block_list(cfg->block_start, cfg->block_count);
    if (n != blocks.size() * 64 * (size_t)s_count) { g_err = "output size mismatch"; return TRB_INVALID_ARG; }
    int rc;
    if (samples && (rc = orc_render_samples(s, cfg, n, samples, stats, 0)) != TRB_OK) return rc;
    const Camera& camera = s->cameras[s->active_camera];
#pragma omp parallel for schedule(dynamic, 1)
    for (long bi = 0; bi < (long)blocks.size(); ++bi) {
        size_t o = (size_t)bi * 64 * s_count;
        for (uint32_t k = 0; k < 64; ++k) {
            const uint32_t px = blocks[bi].first * 8 + k % 8, py = blocks[bi].second * 8 + k / 8;
            const PixelStreams st = pixel_streams(cfg->seed, py * s->film.width + px);
            for (uint32_t si = s_first; si < s_first + s_count; ++si, ++o) { /* render_impl's camera sample */
                const uint32_t ip = dm_permute(si, spp, st.kpos);
                const float sx = van_der_corput(ip, st.scr0) + (float)px, sy = sobol(ip, st.scr1) + (float)py;
                Ray ray = camera.generate_ray(sx, sy, van_der_corput(dm_permute(si, spp, st.ktime), st.scrt));
                Counters cnt;
                Hit hit;
                trb_aov_sample& a = aov[o];
                memset(&a, 0, sizeof a);
                a.depth = INFINITY; a.inst = TRB_MISS;
                if (!s->geom.intersect(ray, hit, cnt)) continue;
                BSDF b;
                s->shade.materials[s->geom.instances[hit.inst].material].bsdf(hit.dg, b);
                const Col c = aov_albedo(b);
                a.albedo[0] = c.r; a.albedo[1] = c.g; a.albedo[2] = c.b;
                a.depth = ray.max_t;
                put3(a.n, b.n);
                a.inst = hit.inst;
            }
        }
    }
    return TRB_OK;
}

} // extern "C"
