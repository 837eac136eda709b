/* The Adaptive sampler's AOV records — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into
 * oracle/_build/liboracle_adaptive_aov.so and loaded by oracle_adaptive_aov/pyadaptiveaov.py.
 *
 * This translation unit is the Adaptive-sampler oracle (oracle_adaptive/adaptive.cpp, included whole and unchanged) plus
 *   orc_render_samples_adaptive_aov  orc_render_samples_adaptive's samples, pixel_spp and stats of the same arguments, and the AOV
 *                                    record (DESIGN.md §4 "AOVs", "Adaptive AOVs") of every slot the literal thread_work + Adaptive
 *                                    run took, in the same (block, pixel, slot) layout with max_per_pixel slots per pixel: the slot's
 *                                    camera ray (round r's streams, entry e, offset samples_taken, as render_adaptive_impl draws it),
 *                                    Scene::intersect, then Material::bsdf at the hit (oracle_aov/aov_albedo.h). Slots a pixel did not
 *                                    take are zero.
 */
#include "../oracle_adaptive/adaptive.cpp"
#include "../oracle_aov/aov_albedo.h"

extern "C" {

int orc_render_samples_adaptive_aov(orc_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, size_t n, trb_sample* samples, trb_aov_sample* aov,
                                    uint32_t* pixel_spp, trb_stats* stats, int threads) {
    std::vector<uint32_t> own;
    if (!pixel_spp) { own.assign((size_t)s->film.width * s->film.height, 0u); pixel_spp = own.data(); }
    const int rc = render_adaptive_impl(s, cfg, ad, 1, nullptr, samples, n, pixel_spp, stats, threads); /* checks every argument */
    if (rc != TRB_OK) return rc;
    Adaptive proto;
    proto.init(ad->min_spp, ad->max_spp);
    const uint32_t mpp = adaptive_max_per_pixel(proto), width = s->film.width;
    auto blocks = s->block_list(cfg->block_start, cfg->block_count);
    memset(aov, 0, n * sizeof(trb_aov_sample));
    const Camera& camera = s->cameras[s->active_camera];
#pragma omp parallel for schedule(dynamic, 1)
    for (long bi = 0; bi < (long)blocks.size(); ++bi)
        for (uint32_t k = 0; k < 64; ++k) {
            const uint32_t px = blocks[bi].first * 8 + k % 8, py = blocks[bi].second * 8 + k / 8, pixel = py * width + px;
            for (uint32_t slot = 0; slot < pixel_spp[pixel]; ++slot) {
                /* the round that took the slot: round 0 takes min_spp, every later round step_size; offset = samples_taken after it */
                const uint32_t round = slot < proto.min_spp ? 0u : 1u + (slot - proto.min_spp) / proto.step_size;
                const uint32_t e = round == 0 ? slot : (slot - proto.min_spp) % proto.step_size;
                const uint32_t count = round == 0 ? proto.min_spp : proto.step_size, offset = proto.min_spp + round * proto.step_size;
                const uint32_t scr0 = dm_scramble(dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_POS0));
                const uint32_t scr1 = dm_scramble(dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_POS1));
                const uint32_t kpos = dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_POS_PERM);
                const uint32_t scrt = dm_scramble(dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_TIME));
                const uint32_t ktime = dm_rng(cfg->seed, pixel, DM_AD_PIXEL_STREAM0 - round, DM_PX_TIME_PERM);
                const uint32_t ip = dm_permute(e, count, kpos) + offset;
                const float sx = van_der_corput(ip, scr0) + (float)px, sy = sobol(ip, scr1) + (float)py;
                Ray ray = camera.generate_ray(sx, sy, van_der_corput(dm_permute(e, proto.max_spp, ktime) + offset, scrt));
                trb_aov_sample& a = aov[((size_t)bi * 64 + k) * mpp + slot];
                a.depth = INFINITY; a.inst = TRB_MISS;
                Counters cnt;
                Hit hit;
                if (!s->geom.intersect(ray, hit, cnt)) continue;
                BSDF b;
                s->shade.materials[s->geom.instances[hit.inst].material].bsdf(hit.dg, b);
                const Col c = aov_albedo(b);
                a.albedo[0] = c.r; a.albedo[1] = c.g; a.albedo[2] = c.b;
                a.depth = ray.max_t;
                a.n[0] = b.n.x; a.n[1] = b.n.y; a.n[2] = b.n.z;
                a.inst = hit.inst;
            }
        }
    return TRB_OK;
}

} // extern "C"
