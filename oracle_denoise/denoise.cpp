/* The parity oracle's denoiser — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into oracle/_build/liboracle_denoise.so
 * and loaded by oracle_denoise/pydenoise.py.
 *
 *   orc_denoise  the filter of include/trb.h "Denoising" (DESIGN.md §4 "Denoising") restated pixel by pixel and tap by tap, in the
 *                header's order, float32 without contraction (-ffp-contract=off), with oracle/detmath.h's dm_expf for exp. It needs
 *                no scene: width and height are arguments. Statuses: TRB_INVALID_ARG for a null pointer or the parameters
 *                trb_denoise refuses.
 *
 * oracle_temporal/temporal.cpp includes this file whole for denoise_params, denoise_prepare and denoise_filter.
 *
 * Nothing here is shared with the library's kernels (tray_rust_b200/csrc/trb_denoise.cuh): the per-pixel state is a plain struct,
 * validity is a bool, and every iteration is a fresh pass over the image.
 */
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>
#include "../oracle/detmath.h"
#include "../include/trb.h"

namespace {

struct Px {
    bool empty = false;    // A.w + B.w <= 0: output zero
    bool valid = false;    // filtered, and a neighbour of others
    float c[3] = {0, 0, 0};
    float d[3] = {1, 1, 1};
    float n[3] = {0, 0, 0};
    bool has_n = false;
    float z = 0, gx = 0, gy = 0;
};

bool fin(float x) { return std::isfinite(x); }
float lum(const float* e) { return 0.2126f * e[0] + 0.7152f * e[1] + 0.0722f * e[2]; }
float depth_of(uint64_t key) { return dm_from_bits((uint32_t)(key >> 32)); }

float axis_gradient(float z, bool lo_in, float zlo, bool hi_in, float zhi) {
    const bool lo = lo_in && fin(zlo), hi = hi_in && fin(zhi);
    if (lo && hi) return (zhi - zlo) * 0.5f;
    if (hi) return zhi - z;
    if (lo) return z - zlo;
    return 0.0f;
}

/* The parameters (NULL: the defaults) into p and log2(normal_power); false where trb_denoise refuses them */
bool denoise_params(const trb_denoise_params* params, trb_denoise_params& p, int& squarings) {
    p = trb_denoise_params{5, 128, 4.0f, 1.0f};
    if (params) p = *params;
    if (p.iterations > 10) return false;
    squarings = -1;
    for (int k = 0; k <= 10; ++k)
        if (p.normal_power == (1u << k)) squarings = k;
    if (squarings < 0) return false;
    return p.sigma_luminance > 0.0f && fin(p.sigma_luminance) && p.sigma_depth > 0.0f && fin(p.sigma_depth);
}

/* The per-pixel rules before the first iteration: px, e (3 per pixel) and v; ea and eb (3 per pixel, may be NULL) receive the
 * demodulated halves e_a and e_b */
void denoise_prepare(long W, long H, const trb_denoise_input* in, std::vector<Px>& px, std::vector<float>& e, std::vector<float>& v,
                     std::vector<float>* ea_all, std::vector<float>* eb_all) {
    const long N = W * H;
    px.assign(N, Px());
    e.assign(N * 3, 0.0f); v.assign(N, 0.0f);
    if (ea_all) ea_all->assign(N * 3, 0.0f);
    if (eb_all) eb_all->assign(N * 3, 0.0f);
    for (long y = 0; y < H; ++y)
        for (long x = 0; x < W; ++x) {
            const long i = y * W + x;
            Px& q = px[i];
            const float* A = in->colour_a + 4 * i;
            const float* B = in->colour_b + 4 * i;
            const float* al = in->albedo_w + 4 * i;
            const float* nw = in->normal_w + 4 * i;
            const float wsum = A[3] + B[3];
            if (wsum <= 0.0f) { q.empty = true; continue; }
            bool ok = true;
            float ea[3], eb[3], m[3];
            for (int k = 0; k < 3; ++k) {
                q.c[k] = (A[k] + B[k]) / wsum;
                const float albedo = al[k] / al[3];
                ok = ok && fin(q.c[k]) && fin(albedo);
                q.d[k] = albedo > TRB_DENOISE_EPS_ALBEDO ? albedo : TRB_DENOISE_EPS_ALBEDO;
                e[3 * i + k] = q.c[k] / q.d[k];
                ea[k] = A[k] / A[3] / q.d[k];
                eb[k] = B[k] / B[3] / q.d[k];
                m[k] = nw[k] / nw[3];
                ok = ok && fin(m[k]) && fin(e[3 * i + k]);
                if (ea_all) (*ea_all)[3 * i + k] = ea[k];
                if (eb_all) (*eb_all)[3 * i + k] = eb[k];
            }
            const float dl = lum(ea) - lum(eb);
            v[i] = dl * dl * 0.25f;
            const float len2 = m[0] * m[0] + m[1] * m[1] + m[2] * m[2];
            q.z = depth_of(in->nearest[i]);
            ok = ok && fin(len2) && fin(v[i]) && !std::isnan(q.z) && q.z != -INFINITY;
            if (!ok) continue;
            q.valid = true;
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
}

/* The a-trous iterations from (e, v) and the output film */
void denoise_filter(long W, long H, const trb_denoise_params& p, int squarings, const std::vector<Px>& px, std::vector<float> e,
                    std::vector<float> v, float* out) {
    const long N = W * H;
    const float h[5] = {1.0f / 16.0f, 1.0f / 4.0f, 3.0f / 8.0f, 1.0f / 4.0f, 1.0f / 16.0f};
    const float k3[3] = {0.25f, 0.5f, 0.25f};
    std::vector<float> e2(N * 3), v2(N);
    for (uint32_t it = 0; it < p.iterations; ++it) {
        const long s = 1L << it;
#pragma omp parallel for schedule(static)
        for (long y = 0; y < H; ++y)
            for (long x = 0; x < W; ++x) {
                const long i = y * W + x;
                const Px& P = px[i];
                if (!P.valid) continue;
                float gs = 0.0f, gk = 0.0f;  // g3x3 of the variance
                for (long dy = -1; dy <= 1; ++dy)
                    for (long dx = -1; dx <= 1; ++dx) {
                        const long qx = x + dx, qy = y + dy;
                        if (qx < 0 || qx >= W || qy < 0 || qy >= H || !px[qy * W + qx].valid) continue;
                        const float k = k3[dx + 1] * k3[dy + 1];
                        gk = gk + k;
                        gs = gs + k * v[qy * W + qx];
                    }
                const float lp = lum(&e[3 * i]);
                const float sigma_l = p.sigma_luminance * std::sqrt(gs / gk) + TRB_DENOISE_EPS_LUMINANCE;
                float se[3] = {0, 0, 0}, sw = 0.0f, sv = 0.0f;
                for (long dy = -2; dy <= 2; ++dy)
                    for (long dx = -2; dx <= 2; ++dx) {
                        const long qx = x + s * dx, qy = y + s * dy;
                        if (qx < 0 || qx >= W || qy < 0 || qy >= H) continue;
                        const long j = qy * W + qx;
                        const Px& Q = px[j];
                        if (!Q.valid) continue;
                        const float w_l = dm_expf(-(std::fabs(lp - lum(&e[3 * j])) / sigma_l));
                        float w_n;
                        if (P.has_n && Q.has_n) {
                            const float dot = P.n[0] * Q.n[0] + P.n[1] * Q.n[1] + P.n[2] * Q.n[2];
                            w_n = dot > 0.0f ? dot : 0.0f;
                            for (int k = 0; k < squarings; ++k) w_n = w_n * w_n;
                        } else {
                            w_n = P.has_n == Q.has_n ? 1.0f : 0.0f;
                        }
                        float w_z;
                        const bool pi = std::isinf(P.z), qi = std::isinf(Q.z);
                        if (pi || qi) {
                            w_z = pi && qi ? 1.0f : 0.0f;
                        } else {
                            const float along = P.gx * (float)(s * dx) + P.gy * (float)(s * dy);
                            w_z = dm_expf(-(std::fabs(P.z - Q.z) / (p.sigma_depth * std::fabs(along) + TRB_DENOISE_EPS_DEPTH)));
                        }
                        const float w = h[dx + 2] * h[dy + 2] * w_l * w_n * w_z;
                        for (int k = 0; k < 3; ++k) se[k] = se[k] + w * e[3 * j + k];
                        sw = sw + w;
                        sv = sv + w * w * v[j];
                    }
                for (int k = 0; k < 3; ++k) e2[3 * i + k] = se[k] / sw;
                v2[i] = sv / (sw * sw);
            }
        e.swap(e2);
        v.swap(v2);
    }
    for (long i = 0; i < N; ++i) {
        const Px& P = px[i];
        float* o = out + 4 * i;
        if (P.empty) { o[0] = o[1] = o[2] = o[3] = 0.0f; continue; }
        for (int k = 0; k < 3; ++k) {
            o[k] = P.valid ? e[3 * i + k] * P.d[k] : P.c[k];
            if (std::isnan(o[k])) o[k] = dm_from_bits(0x7fffffffu);  // the one NaN the contract writes
        }
        o[3] = 1.0f;
    }
}

}  // namespace

extern "C" {

int orc_denoise(uint32_t width, uint32_t height, const trb_denoise_input* in, const trb_denoise_params* params, float* out) {
    trb_denoise_params p;
    int squarings;
    if (!denoise_params(params, p, squarings)) return TRB_INVALID_ARG;
    if (!in || !out || !in->colour_a || !in->colour_b || !in->albedo_w || !in->normal_w || !in->nearest) return TRB_INVALID_ARG;
    std::vector<Px> px;
    std::vector<float> e, v;
    denoise_prepare(width, height, in, px, e, v, nullptr, nullptr);
    denoise_filter(width, height, p, squarings, px, std::move(e), std::move(v), out);
    return TRB_OK;
}

}  // extern "C"
