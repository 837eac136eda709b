/* The sample-variance oracle — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into oracle/_build/liboracle_variance.so
 * and loaded by oracle_variance/pyvariance.py.
 *
 * This translation unit is the ray-query oracle (oracle_queries/queries.cpp, which includes oracle/oracle.cpp) and the denoiser
 * oracle (oracle_denoise/denoise.cpp), both included whole and unchanged, plus the contract of include/trb.h "Sample variance"
 * (DESIGN.md §4):
 *   orc_lum_film          the lum_w film of caller samples: each sample's (x, y) and radiance (trb_sample, as orc_render_samples and
 *                         orc_render_samples_adaptive give them) with the albedo of its AOV record (trb_aov_sample, as
 *                         orc_render_samples_aov and orc_render_samples_adaptive_aov give them), written as orc_film_write writes
 *                         colours (RenderTarget::write once per region, in the block list's order) with (w l, w (l l), w w, w) in
 *                         place of (w c, w). A region index >= the block count skips the sample.
 *   orc_denoise_variance  trb_denoise_variance restated over host films: the pixel rules here, then denoise.cpp's a-trous filter.
 */
#include "../oracle_queries/queries.cpp"
#include "../oracle_denoise/denoise.cpp"

namespace {

struct LumSample { float x, y, l; };

/* RenderTarget::write (oracle.cpp's RenderTarget::write, render_target.rs:77-165) with the lum_w film's four products */
void lum_write(const RenderTarget& rt, const std::vector<LumSample>& samples, int rx0, int ry0, int rx1, int ry1, float* film) {
    const int ls = 2;
    const int x_range[2] = {std::max(rx0 - rt.fpw[0], 0), std::min(rx1 + rt.fpw[0], rt.width - 1)};
    const int y_range[2] = {std::max(ry0 - rt.fpw[1], 0), std::min(ry1 + rt.fpw[1], rt.height - 1)};
    if (x_range[1] - x_range[0] < 0 || y_range[1] - y_range[0] < 0) return;
    const int bxr[2] = {x_range[0] / ls, x_range[1] / ls}, byr[2] = {y_range[0] / ls, y_range[1] / ls};
    float filtered[4][4];
    for (int y = byr[0]; y <= byr[1]; ++y)
        for (int x = bxr[0]; x <= bxr[1]; ++x) {
            const int bxs = x * ls, bys = y * ls;
            const int xw[2] = {std::max(x_range[0], bxs), std::min(x_range[1] + 1, bxs + ls)};
            const int yw[2] = {std::max(y_range[0], bys), std::min(y_range[1] + 1, bys + ls)};
            for (int i = 0; i < 4; ++i) for (int k = 0; k < 4; ++k) filtered[i][k] = 0.0f;
            for (const LumSample& c : samples) {
                if (!(c.x >= (float)(xw[0] - rt.fpw[0]) && c.x < (float)(xw[1] + rt.fpw[0]) && c.y >= (float)(yw[0] - rt.fpw[1]) &&
                      c.y < (float)(yw[1] + rt.fpw[1])))
                    continue;
                const float img_x = c.x - 0.5f, img_y = c.y - 0.5f;
                for (int iy = yw[0]; iy < yw[1]; ++iy) {
                    const float fy = fabsf((float)iy - img_y) * rt.filter.inv_h;
                    if (fy > rt.filter.h) continue;
                    const uint32_t fy_idx = std::min(f2u(fy * 16.0f), 15u);
                    for (int ix = xw[0]; ix < xw[1]; ++ix) {
                        const float fx = fabsf((float)ix - img_x) * rt.filter.inv_w;
                        if (fx > rt.filter.w) continue;
                        const uint32_t fx_idx = std::min(f2u(fx * 16.0f), 15u);
                        const float w = rt.table[fy_idx * 16 + fx_idx];
                        const int px = (iy - bys) * ls + ix - bxs;
                        filtered[px][0] += w * c.l;
                        filtered[px][1] += w * (c.l * c.l);
                        filtered[px][2] += w * w;
                        filtered[px][3] += w;
                    }
                }
            }
            for (int iy = yw[0]; iy < yw[1]; ++iy)
                for (int ix = xw[0]; ix < xw[1]; ++ix) {
                    const int px = (iy - bys) * ls + ix - bxs;
                    float* dst = film + ((size_t)iy * rt.width + ix) * 4;
                    for (int k = 0; k < 4; ++k) dst[k] += filtered[px][k];
                }
        }
}

}  // namespace

extern "C" {

int orc_lum_film(orc_scene* s, size_t n, const trb_sample* samples, const trb_aov_sample* aov, const uint32_t* regions, float* lum_w) {
    if (!s || (n && (!samples || !aov || !regions)) || !lum_w) return TRB_INVALID_ARG;
    const uint32_t nbx = s->film.width / 8, nr = nbx * (s->film.height / 8);
    std::vector<std::vector<LumSample>> by_region(nr);
    for (size_t i = 0; i < n; ++i) {
        if (regions[i] >= nr) continue;
        const float c[3] = {samples[i].r, samples[i].g, samples[i].b};
        float d[3];
        for (int k = 0; k < 3; ++k) d[k] = aov[i].albedo[k] > TRB_DENOISE_EPS_ALBEDO ? aov[i].albedo[k] : TRB_DENOISE_EPS_ALBEDO;
        const float l = 0.2126f * (c[0] / d[0]) + 0.7152f * (c[1] / d[1]) + 0.0722f * (c[2] / d[2]);
        by_region[regions[i]].push_back(LumSample{samples[i].x, samples[i].y, l});
    }
    for (const auto& b : s->block_list(0, 0)) {
        const std::vector<LumSample>& v = by_region[b.second * nbx + b.first];
        if (v.empty()) continue;
        const int x0 = (int)b.first * 8, y0 = (int)b.second * 8;
        lum_write(s->rt, v, x0, y0, x0 + 8, y0 + 8, lum_w);
    }
    return TRB_OK;
}

int orc_denoise_variance(uint32_t width, uint32_t height, const trb_denoise_frame* in, const float* lum_w, const trb_denoise_params* params,
                         float* rgbw, float* variance) {
    trb_denoise_params p;
    int squarings;
    if (!denoise_params(params, p, squarings)) return TRB_INVALID_ARG;
    if (!in || !lum_w || !rgbw || !in->colour || !in->albedo_w || !in->normal_w || !in->nearest) return TRB_INVALID_ARG;
    const long W = width, H = height, N = W * H;
    const float qnan = dm_from_bits(0x7fffffffu);
    std::vector<Px> px(N);
    std::vector<float> e(N * 3, 0.0f), v(N, qnan);
    for (long y = 0; y < H; ++y)
        for (long x = 0; x < W; ++x) {
            const long i = y * W + x;
            Px& q = px[i];
            const float* A = in->colour + 4 * i;
            const float* al = in->albedo_w + 4 * i;
            const float* nw = in->normal_w + 4 * i;
            const float* lw = lum_w + 4 * i;
            if (A[3] <= 0.0f) { q.empty = true; continue; }
            /* 1: trb_denoise's guides over the single film */
            bool ok = true;
            float m[3];
            for (int k = 0; k < 3; ++k) {
                q.c[k] = A[k] / A[3];
                const float albedo = al[k] / al[3];
                ok = ok && fin(q.c[k]) && fin(albedo);
                q.d[k] = albedo > TRB_DENOISE_EPS_ALBEDO ? albedo : TRB_DENOISE_EPS_ALBEDO;
                e[3 * i + k] = q.c[k] / q.d[k];
                m[k] = nw[k] / nw[3];
                ok = ok && fin(m[k]) && fin(e[3 * i + k]);
            }
            /* 2: the variance of the pixel's weighted mean of l */
            const float V1 = lw[3], V2 = lw[2];
            float vi = qnan;
            if (V1 > 0.0f && V1 * V1 > V2) {
                const float m1 = lw[0] / V1, m2 = lw[1] / V1;
                const float s2 = m2 - m1 * m1;
                vi = (s2 > 0.0f ? s2 : 0.0f) * V2 / (V1 * V1 - V2);
            }
            const float len2 = m[0] * m[0] + m[1] * m[1] + m[2] * m[2];
            q.z = depth_of(in->nearest[i]);
            /* 3: copy-through */
            ok = ok && fin(len2) && fin(vi) && !std::isnan(q.z) && q.z != -INFINITY;
            if (!ok) continue;
            q.valid = true;
            v[i] = vi;
            if (len2 != 0.0f) {
                q.has_n = true;
                const float l = std::sqrt(len2);
                for (int k = 0; k < 3; ++k) q.n[k] = m[k] / l;
            }
            if (fin(q.z)) {
                q.gx = axis_gradient(q.z, x > 0, x > 0 ? depth_of(in->nearest[i - 1]) : 0.0f, x + 1 < W, x + 1 < W ? depth_of(in->nearest[i + 1]) : 0.0f);
                q.gy = axis_gradient(q.z, y > 0, y > 0 ? depth_of(in->nearest[i - W]) : 0.0f, y + 1 < H, y + 1 < H ? depth_of(in->nearest[i + W]) : 0.0f);
            }
        }
    if (variance)
        for (long i = 0; i < N; ++i) variance[i] = px[i].valid ? v[i] : qnan;
    /* 4: trb_denoise's iterations; the filter reads v only at valid pixels */
    denoise_filter(W, H, p, squarings, px, std::move(e), std::move(v), rgbw);
    return TRB_OK;
}

}  // extern "C"
