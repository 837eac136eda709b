// trb_denoise.cuh — the denoiser of trb_denoise / trb_denoise_device (include/trb.h "Denoising", DESIGN.md §4 "Denoising"): SVGF's
// edge-avoiding a-trous filter over the demodulated colour of two half renders, guided by their albedo, normal and nearest-hit films.
// Three kernels: k_dn_prepare reads the inputs once into a guide record per pixel and the first (e, v) buffer; k_dn_atrous runs one
// iteration, ping-ponging two (e, v) buffers, and the last one remodulates into the output film; k_dn_temporal takes k_dn_prepare's place
// for trb_denoise_temporal*, blending each pixel's reprojected history into the first (e, v) buffer; k_dn_temporal_moments and
// k_dn_moments_variance take it for trb_denoise_moments* (k_dn_temporal_moments_grad for trb_denoise_moments_gradient*), one film with
// the variance from luminance moments; k_dn_variance_prepare takes it for trb_denoise_variance*, one film with the variance of
// its own samples (the lum_w film); k_dn_temporal_variance (k_dn_temporal_variance_grad) takes it for trb_denoise_variance_temporal*
// (the _gradient forms), that variance carried through the history. Float32 in the header's order, no atomics: every pixel's sums run in tap order, so the output is reproducible bit for bit (the oracle restates it in oracle_denoise/).
#pragma once
#include "trb_detmath.cuh"
#include "trb_kernels.cuh"
#include "../../include/trb.h"

namespace trb {

struct DnParams {
    int width, height;
    uint32_t iterations;
    uint32_t normal_squarings;   // log2(normal_power)
    float sigma_l, sigma_z;
};

// The scene's scratch for n pixels, 72 bytes each: guide (n, z) with z = NaN marking a pixel that is not filtered, the albedo divisor d,
// two (e, v) buffers, and the depth gradient
struct DnScratch {
    float4* guide;
    float4* divisor;
    float4* ev[2];
    float2* grad;
};
constexpr size_t DN_BYTES_PER_PIXEL = 4 * sizeof(float4) + sizeof(float2);

__device__ __forceinline__ bool dn_finite(float x) { return fabsf(x) < __int_as_float(0x7f800000); }
__device__ __forceinline__ float dn_lum(float r, float g, float b) { return 0.2126f * r + 0.7152f * g + 0.0722f * b; }
// every NaN the output holds is written as 0x7fffffff, whatever its inputs carried
__device__ __forceinline__ float4 dn_out(float r, float g, float b, float w) {
    const float qnan = __int_as_float(0x7fffffff);
    return make_float4(r == r ? r : qnan, g == g ? g : qnan, b == b ? b : qnan, w);
}
__device__ __forceinline__ float dn_depth(const unsigned long long* nearest, int i) { return __uint_as_float((uint32_t)(nearest[i] >> 32)); }

// one axis of the depth gradient: central, one-sided, or 0 (z finite)
__device__ __forceinline__ float dn_grad(float z, bool has_lo, float zlo, bool has_hi, float zhi) {
    has_lo = has_lo && dn_finite(zlo);
    has_hi = has_hi && dn_finite(zhi);
    if (has_lo && has_hi) return (zhi - zlo) * 0.5f;
    if (has_hi) return zhi - z;
    if (has_lo) return z - zlo;
    return 0.0f;
}

// trb_denoise's pixel from m on, once c, the albedo a, d, e and v are known (shared by k_dn_prepare and k_dn_variance_prepare): m, len2
// and z, the copy-through test, then the guide, gradient, divisor and first (e, v) records. Returns whether p is filtered. prm and sc
// are taken by value, as the kernels hold them.
__device__ __forceinline__ bool dn_prepare_px(const DnParams prm, int x, int y, int i, float c0, float c1, float c2, float a0, float a1, float a2,
                                              float d0, float d1, float d2, float e0, float e1, float e2, float v, float4 nw,
                                              const unsigned long long* __restrict__ nearest, DnScratch sc, float4* __restrict__ out) {
    const float m0 = nw.x / nw.w, m1 = nw.y / nw.w, m2 = nw.z / nw.w;
    const float len2 = m0 * m0 + m1 * m1 + m2 * m2;
    const float z = dn_depth(nearest, i);
    const bool ok = dn_finite(c0) && dn_finite(c1) && dn_finite(c2) && dn_finite(a0) && dn_finite(a1) && dn_finite(a2) && dn_finite(m0) &&
                    dn_finite(m1) && dn_finite(m2) && dn_finite(len2) && dn_finite(e0) && dn_finite(e1) && dn_finite(e2) && dn_finite(v) &&
                    z == z && z != __int_as_float(0xff800000);
    if (!ok) {
        out[i] = dn_out(c0, c1, c2, 1.0f);
        sc.guide[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0x7fc00000));
        return false;
    }
    float n0 = 0.0f, n1 = 0.0f, n2 = 0.0f;
    if (len2 != 0.0f) {
        const float l = sqrtf(len2);
        n0 = m0 / l; n1 = m1 / l; n2 = m2 / l;
    }
    float gx = 0.0f, gy = 0.0f;
    if (dn_finite(z)) {
        const bool l = x > 0, r = x + 1 < prm.width, u = y > 0, dn = y + 1 < prm.height;
        gx = dn_grad(z, l, l ? dn_depth(nearest, i - 1) : 0.0f, r, r ? dn_depth(nearest, i + 1) : 0.0f);
        gy = dn_grad(z, u, u ? dn_depth(nearest, i - prm.width) : 0.0f, dn, dn ? dn_depth(nearest, i + prm.width) : 0.0f);
    }
    sc.guide[i] = make_float4(n0, n1, n2, z);
    sc.grad[i] = make_float2(gx, gy);
    sc.divisor[i] = make_float4(d0, d1, d2, 0.0f);
    sc.ev[0][i] = make_float4(e0, e1, e2, v);
    if (prm.iterations == 0) out[i] = dn_out(e0 * d0, e1 * d1, e2 * d2, 1.0f);
    return true;
}

__global__ void __launch_bounds__(256) k_dn_prepare(const DnParams prm, const float4* __restrict__ ca, const float4* __restrict__ cb,
                                                    const float4* __restrict__ alb, const float4* __restrict__ nrm,
                                                    const unsigned long long* __restrict__ nearest, DnScratch sc, float4* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= prm.width || y >= prm.height) return;
    const int i = y * prm.width + x;
    const float4 A = ca[i], B = cb[i];
    const float W = A.w + B.w;
    if (W <= 0.0f) {
        out[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        sc.guide[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0x7fc00000));
        return;
    }
    const float c0 = (A.x + B.x) / W, c1 = (A.y + B.y) / W, c2 = (A.z + B.z) / W;
    const float4 al = alb[i], nw = nrm[i];
    const float a0 = al.x / al.w, a1 = al.y / al.w, a2 = al.z / al.w;
    const float d0 = a0 > TRB_DENOISE_EPS_ALBEDO ? a0 : TRB_DENOISE_EPS_ALBEDO, d1 = a1 > TRB_DENOISE_EPS_ALBEDO ? a1 : TRB_DENOISE_EPS_ALBEDO,
                d2 = a2 > TRB_DENOISE_EPS_ALBEDO ? a2 : TRB_DENOISE_EPS_ALBEDO;
    const float e0 = c0 / d0, e1 = c1 / d1, e2 = c2 / d2;
    const float la = dn_lum(A.x / A.w / d0, A.y / A.w / d1, A.z / A.w / d2), lb = dn_lum(B.x / B.w / d0, B.y / B.w / d1, B.z / B.w / d2);
    const float dl = la - lb;
    const float v = dl * dl * 0.25f;
    dn_prepare_px(prm, x, y, i, c0, c1, c2, a0, a1, a2, d0, d1, d2, e0, e1, e2, v, nw, nearest, sc, out);
}

// Step 2 of "Sample variance": the variance of the pixel's weighted mean of l from its lum_w record, NaN for at most one effective sample
__device__ __forceinline__ float dn_sample_variance(float4 lw) {
    const float V1 = lw.w, V2 = lw.z;
    if (!(V1 > 0.0f && V1 * V1 > V2)) return __int_as_float(0x7fffffff);
    const float m1 = lw.x / V1, m2 = lw.y / V1;
    const float s = m2 - m1 * m1;
    return (s > 0.0f ? s : 0.0f) * V2 / (V1 * V1 - V2);
}

// trb_denoise_variance's k_dn_prepare (include/trb.h "Sample variance"): one film, and v from the pixel's own samples in lum_w.
// Writes the same scratch, and var (may be null) receives v, NaN where the pixel is not filtered.
__global__ void __launch_bounds__(256) k_dn_variance_prepare(const DnParams prm, const float4* __restrict__ col, const float4* __restrict__ lum,
                                                             const float4* __restrict__ alb, const float4* __restrict__ nrm,
                                                             const unsigned long long* __restrict__ nearest, DnScratch sc, float4* __restrict__ out,
                                                             float* __restrict__ var) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= prm.width || y >= prm.height) return;
    const int i = y * prm.width + x;
    const float qnan = __int_as_float(0x7fffffff);
    const float4 A = col[i];
    const float W = A.w;
    if (W <= 0.0f) {
        out[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        sc.guide[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0x7fc00000));
        if (var) var[i] = qnan;
        return;
    }
    const float c0 = A.x / W, c1 = A.y / W, c2 = A.z / W;
    const float4 al = alb[i], nw = nrm[i], lw = lum[i];
    const float a0 = al.x / al.w, a1 = al.y / al.w, a2 = al.z / al.w;
    const float d0 = a0 > TRB_DENOISE_EPS_ALBEDO ? a0 : TRB_DENOISE_EPS_ALBEDO, d1 = a1 > TRB_DENOISE_EPS_ALBEDO ? a1 : TRB_DENOISE_EPS_ALBEDO,
                d2 = a2 > TRB_DENOISE_EPS_ALBEDO ? a2 : TRB_DENOISE_EPS_ALBEDO;
    const float e0 = c0 / d0, e1 = c1 / d1, e2 = c2 / d2;
    const float v = dn_sample_variance(lw);
    const bool filtered = dn_prepare_px(prm, x, y, i, c0, c1, c2, a0, a1, a2, d0, d1, d2, e0, e1, e2, v, nw, nearest, sc, out);
    if (var) var[i] = filtered ? v : qnan;
}

// One a-trous iteration at step s from ev_in to ev_out, or, the last one, remodulated into out (ev_out unused)
__global__ void __launch_bounds__(256) k_dn_atrous(const DnParams prm, int s, const float4* __restrict__ guide, const float2* __restrict__ grad,
                                                   const float4* __restrict__ divisor, const float4* __restrict__ ev_in,
                                                   float4* __restrict__ ev_out, float4* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= prm.width || y >= prm.height) return;
    const int W = prm.width, H = prm.height, i = y * W + x;
    const float4 gp = guide[i];
    if (gp.w != gp.w) return; // not filtered: k_dn_prepare wrote its output
    const float4 ep = ev_in[i];
    const float lp = dn_lum(ep.x, ep.y, ep.z);
    float gs = 0.0f, gk = 0.0f;
    for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
            const int qx = x + dx, qy = y + dy;
            if (qx < 0 || qx >= W || qy < 0 || qy >= H) continue;
            const int q = qy * W + qx;
            if (guide[q].w != guide[q].w) continue;
            const float k = (dx == 0 ? 0.5f : 0.25f) * (dy == 0 ? 0.5f : 0.25f);
            gk = gk + k;
            gs = gs + k * ev_in[q].w;
        }
    const float denom_l = prm.sigma_l * sqrtf(gs / gk) + TRB_DENOISE_EPS_LUMINANCE;
    const float2 g = grad[i];
    const bool p_inf = !dn_finite(gp.w), p_nrm = gp.x != 0.0f || gp.y != 0.0f || gp.z != 0.0f;
    const float h[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, sw = 0.0f, sv = 0.0f;
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy) {
        const int qy = y + s * dy;
        if (qy < 0 || qy >= H) continue;
#pragma unroll
        for (int dx = -2; dx <= 2; ++dx) {
            const int qx = x + s * dx;
            if (qx < 0 || qx >= W) continue;
            const int q = qy * W + qx;
            const float4 gq = guide[q];
            if (gq.w != gq.w) continue;
            const float4 eq = ev_in[q];
            const float wl = dexp(-(fabsf(lp - dn_lum(eq.x, eq.y, eq.z)) / denom_l));
            float wn;
            const bool q_nrm = gq.x != 0.0f || gq.y != 0.0f || gq.z != 0.0f;
            if (p_nrm != q_nrm) wn = 0.0f;
            else if (!p_nrm) wn = 1.0f;
            else {
                const float dot = gp.x * gq.x + gp.y * gq.y + gp.z * gq.z;
                wn = dot > 0.0f ? dot : 0.0f;
                for (uint32_t k = 0; k < prm.normal_squarings; ++k) wn = wn * wn;
            }
            float wz;
            const bool q_inf = !dn_finite(gq.w);
            if (p_inf != q_inf) wz = 0.0f;
            else if (p_inf) wz = 1.0f;
            else wz = dexp(-(fabsf(gp.w - gq.w) / (prm.sigma_z * fabsf(g.x * (float)(s * dx) + g.y * (float)(s * dy)) + TRB_DENOISE_EPS_DEPTH)));
            float w = h[dx + 2] * h[dy + 2];
            w = w * wl;
            w = w * wn;
            w = w * wz;
            s0 = s0 + w * eq.x; s1 = s1 + w * eq.y; s2 = s2 + w * eq.z;
            sw = sw + w;
            sv = sv + w * w * eq.w;
        }
    }
    const float e0 = s0 / sw, e1 = s1 / sw, e2 = s2 / sw;
    if (out) {
        const float4 d = divisor[i];
        out[i] = dn_out(e0 * d.x, e1 * d.y, e2 * d.z, 1.0f);
    } else {
        ev_out[i] = make_float4(e0, e1, e2, sv / (sw * sw));
    }
}

// ---- temporal denoising (trb_denoise_temporal*, include/trb.h "Temporal denoising") ---------------------------------------------
// The current frame's camera and the history's snapshot of the frame it was written at; has_prev = 0 for an empty history or one of
// another object generation
struct DnTemporal {
    float px_to_cam[16], cam_mat[16], scaling[3];
    uint32_t n_cur;
    float cam_inv_prev[16];
    float tan_prev, w_prev, h_prev, x0, x1, y0, y1; // the previous film's size and screen window (camera_setup's)
    uint32_t n_prev, has_prev;
    uint32_t max_history;
    float depth_tolerance, normal_threshold;
};

// One history set, 48 bytes per pixel: (H_a, z), (H_b, inst bits), (n, len bits); len == 0 is "none"
struct DnHistory {
    float4* a;
    float4* b;
    float4* n;
};
constexpr size_t DN_HISTORY_BYTES_PER_PIXEL = 3 * sizeof(float4);

// Steps 1-3 of "Temporal denoising" for pixel (x, y) with depth z, instance id and unit normal n (0 if none): the motion (NaN where
// none), S, the tap-weighted sums of the a and b records' first three channels (divided by S by the caller) and len_prev. Shared by
// the half-film kernels (a, b = H_a, H_b) and k_dn_temporal_moments (a = H, b = (M1, M2, 0)).
__device__ __forceinline__ void dn_reproject(const DnParams& prm, const DnTemporal& tp, int x, int y, float z, uint32_t id, float n0, float n1,
                                             float n2, const DInstance* __restrict__ inst, const float* __restrict__ mat_prev, const DnHistory& hin,
                                             float& mx, float& my, float& S, float& ha0, float& ha1, float& ha2, float& hb0, float& hb1,
                                             float& hb2, uint32_t& len_prev) {
    const float qnan = __int_as_float(0x7fffffff);
    mx = qnan; my = qnan; S = 0.0f; ha0 = 0.0f; ha1 = 0.0f; ha2 = 0.0f; hb0 = 0.0f; hb1 = 0.0f; hb2 = 0.0f;
    len_prev = 0;
    if (tp.has_prev && id < tp.n_prev && id < tp.n_cur && dn_finite(z)) {
        const f3 pc = xf_point(tp.px_to_cam, mk((float)x + 0.5f, (float)y + 0.5f, 0.0f));
        const f3 dir = xf_vector(tp.cam_mat, unit(mk(tp.scaling[0], tp.scaling[1], tp.scaling[2]) * pc));
        const f3 o = xf_point(tp.cam_mat, splat(0.0f));
        const f3 pw = mk(o.x + z * dir.x, o.y + z * dir.y, o.z + z * dir.z);
        const f3 q = xf_point(tp.cam_inv_prev, xf_point(mat_prev + 16 * (size_t)id, xf_point(inst[id].inv, pw)));
        if (q.z > 0.0f) {
            const float X = q.x / (q.z * tp.tan_prev), Y = q.y / (q.z * tp.tan_prev);
            const float rx = (X - tp.x0) / (tp.x1 - tp.x0) * tp.w_prev, ry = (Y - tp.y1) / (tp.y0 - tp.y1) * tp.h_prev;
            mx = rx - ((float)x + 0.5f); my = ry - ((float)y + 0.5f);
            const float ql = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z);
            const float cx = rx - 0.5f, cy = ry - 0.5f, fx = floorf(cx), fy = floorf(cy), ax = cx - fx, ay = cy - fy;
            const bool p_nrm = n0 != 0.0f || n1 != 0.0f || n2 != 0.0f;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float tx = fx + (float)(k & 1), ty = fy + (float)(k >> 1);
                const float w = ((k & 1) ? ax : 1.0f - ax) * ((k >> 1) ? ay : 1.0f - ay);
                if (!(tx >= 0.0f && tx <= tp.w_prev - 1.0f && ty >= 0.0f && ty <= tp.h_prev - 1.0f)) continue;
                const int j = (int)ty * prm.width + (int)tx;
                const float4 tn = hin.n[j];
                const uint32_t tlen = __float_as_uint(tn.w);
                if (tlen == 0u) continue;
                const float4 ta = hin.a[j], tb = hin.b[j];
                if (__float_as_uint(tb.w) != id) continue;
                if (!(fabsf(ta.w - ql) <= tp.depth_tolerance * ql)) continue;
                const bool t_nrm = tn.x != 0.0f || tn.y != 0.0f || tn.z != 0.0f;
                if (t_nrm != p_nrm) continue;
                if (p_nrm && !(tn.x * n0 + tn.y * n1 + tn.z * n2 >= tp.normal_threshold)) continue;
                S = S + w;
                ha0 = ha0 + w * ta.x; ha1 = ha1 + w * ta.y; ha2 = ha2 + w * ta.z;
                hb0 = hb0 + w * tb.x; hb1 = hb1 + w * tb.y; hb2 = hb2 + w * tb.z;
                if (w > 0.0f && tlen > len_prev) len_prev = tlen;
            }
        }
    }
}

// k_dn_prepare's reads and writes, plus the reprojected history blended into (ē, v) before the a-trous iterations (1 + N launches as
// for trb_denoise). mat_prev: the snapshot's object -> world matrices, 16 floats per instance; the current inverses are read from the
// frame's instance records.
// The body of k_dn_temporal (GRAD false) and k_dn_temporal_grad (GRAD true: step 4 shortens the history by the pixel's stratum's
// lambda, include/trb.h "Temporal gradients", and lam_out receives it). lam_s: S lambdas on the stratum grid of gw columns.
template <bool GRAD>
__device__ __forceinline__ void dn_temporal_px(const DnParams prm, const DnTemporal& tp, const float4* __restrict__ ca, const float4* __restrict__ cb,
                                               const float4* __restrict__ alb, const float4* __restrict__ nrm,
                                               const unsigned long long* __restrict__ nearest, DnScratch sc, float4* __restrict__ out,
                                               const DInstance* __restrict__ inst, const float* __restrict__ mat_prev, const DnHistory hin,
                                               const DnHistory hout, float2* __restrict__ motion, uint32_t* __restrict__ hlen,
                                               const float* __restrict__ lam_s, uint32_t gw, float* __restrict__ lam_out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= prm.width || y >= prm.height) return;
    const int i = y * prm.width + x;
    const float qnan = __int_as_float(0x7fffffff);
    float lam = 0.0f;
    if (GRAD) {
        lam = lam_s[(uint32_t)(y / 3) * gw + (uint32_t)(x / 3)];
        if (lam_out) lam_out[i] = lam;
    }
    const float4 A = ca[i], B = cb[i];
    const float W = A.w + B.w;
    if (W <= 0.0f) {
        out[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        sc.guide[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0x7fc00000));
        hout.n[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (motion) motion[i] = make_float2(qnan, qnan);
        if (hlen) hlen[i] = 0u;
        return;
    }
    const float c0 = (A.x + B.x) / W, c1 = (A.y + B.y) / W, c2 = (A.z + B.z) / W;
    const float4 al = alb[i], nw = nrm[i];
    const float a0 = al.x / al.w, a1 = al.y / al.w, a2 = al.z / al.w;
    const float d0 = a0 > TRB_DENOISE_EPS_ALBEDO ? a0 : TRB_DENOISE_EPS_ALBEDO, d1 = a1 > TRB_DENOISE_EPS_ALBEDO ? a1 : TRB_DENOISE_EPS_ALBEDO,
                d2 = a2 > TRB_DENOISE_EPS_ALBEDO ? a2 : TRB_DENOISE_EPS_ALBEDO;
    float e0 = c0 / d0, e1 = c1 / d1, e2 = c2 / d2;
    float ea0 = A.x / A.w / d0, ea1 = A.y / A.w / d1, ea2 = A.z / A.w / d2;
    float eb0 = B.x / B.w / d0, eb1 = B.y / B.w / d1, eb2 = B.z / B.w / d2;
    const float dl = dn_lum(ea0, ea1, ea2) - dn_lum(eb0, eb1, eb2);
    float v = dl * dl * 0.25f;
    const float m0 = nw.x / nw.w, m1 = nw.y / nw.w, m2 = nw.z / nw.w;
    const float len2 = m0 * m0 + m1 * m1 + m2 * m2;
    const unsigned long long key = nearest[i];
    const float z = __uint_as_float((uint32_t)(key >> 32));
    const bool ok = dn_finite(c0) && dn_finite(c1) && dn_finite(c2) && dn_finite(a0) && dn_finite(a1) && dn_finite(a2) && dn_finite(m0) &&
                    dn_finite(m1) && dn_finite(m2) && dn_finite(len2) && dn_finite(e0) && dn_finite(e1) && dn_finite(e2) && dn_finite(v) &&
                    z == z && z != __int_as_float(0xff800000);
    if (!ok) {
        out[i] = dn_out(c0, c1, c2, 1.0f);
        sc.guide[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0x7fc00000));
        hout.n[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (motion) motion[i] = make_float2(qnan, qnan);
        if (hlen) hlen[i] = 0u;
        return;
    }
    float n0 = 0.0f, n1 = 0.0f, n2 = 0.0f;
    if (len2 != 0.0f) {
        const float l = sqrtf(len2);
        n0 = m0 / l; n1 = m1 / l; n2 = m2 / l;
    }
    float gx = 0.0f, gy = 0.0f;
    if (dn_finite(z)) {
        const bool l = x > 0, r = x + 1 < prm.width, u = y > 0, dn = y + 1 < prm.height;
        gx = dn_grad(z, l, l ? dn_depth(nearest, i - 1) : 0.0f, r, r ? dn_depth(nearest, i + 1) : 0.0f);
        gy = dn_grad(z, u, u ? dn_depth(nearest, i - prm.width) : 0.0f, dn, dn ? dn_depth(nearest, i + prm.width) : 0.0f);
    }
    // 1-3: reconstruct, reproject into the snapshot's frame, gather the history taps
    const uint32_t id = (uint32_t)key;
    float mx, my, S, ha0, ha1, ha2, hb0, hb1, hb2;
    uint32_t len_prev;
    dn_reproject(prm, tp, x, y, z, id, n0, n1, n2, inst, mat_prev, hin, mx, my, S, ha0, ha1, ha2, hb0, hb1, hb2, len_prev);
    // 4: blend
    uint32_t np = 1;
    if (GRAD) {
        if (S > 0.0f) {
            const uint32_t len_adj = (uint32_t)floorf((1.0f - lam) * (float)len_prev);
            np = len_adj + 1 < tp.max_history ? len_adj + 1 : tp.max_history;
        }
    } else {
        if (S > 0.0f) np = len_prev + 1 < tp.max_history ? len_prev + 1 : tp.max_history;
    }
    if (np > 1) {
        ha0 = ha0 / S; ha1 = ha1 / S; ha2 = ha2 / S;
        hb0 = hb0 / S; hb1 = hb1 / S; hb2 = hb2 / S;
        const float alpha = 1.0f / (float)np, beta = 1.0f - alpha;
        e0 = alpha * e0 + beta * ((ha0 + hb0) * 0.5f);
        e1 = alpha * e1 + beta * ((ha1 + hb1) * 0.5f);
        e2 = alpha * e2 + beta * ((ha2 + hb2) * 0.5f);
        ea0 = alpha * ea0 + beta * ha0; ea1 = alpha * ea1 + beta * ha1; ea2 = alpha * ea2 + beta * ha2;
        eb0 = alpha * eb0 + beta * hb0; eb1 = alpha * eb1 + beta * hb1; eb2 = alpha * eb2 + beta * hb2;
        const float dt = dn_lum(ea0, ea1, ea2) - dn_lum(eb0, eb1, eb2);
        v = dt * dt * 0.25f;
    }
    // 5-6: the a-trous inputs as k_dn_prepare writes them, and the new history
    sc.guide[i] = make_float4(n0, n1, n2, z);
    sc.grad[i] = make_float2(gx, gy);
    sc.divisor[i] = make_float4(d0, d1, d2, 0.0f);
    sc.ev[0][i] = make_float4(e0, e1, e2, v);
    if (prm.iterations == 0) out[i] = dn_out(e0 * d0, e1 * d1, e2 * d2, 1.0f);
    if (dn_finite(z)) {
        hout.a[i] = make_float4(ea0, ea1, ea2, z);
        hout.b[i] = make_float4(eb0, eb1, eb2, __uint_as_float(id));
        hout.n[i] = make_float4(n0, n1, n2, __uint_as_float(np));
    } else {
        hout.n[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    if (motion) motion[i] = make_float2(mx == mx ? mx : qnan, my == my ? my : qnan);
    if (hlen) hlen[i] = np;
}

__global__ void __launch_bounds__(256) k_dn_temporal(const DnParams prm, const __grid_constant__ DnTemporal tp, const float4* __restrict__ ca,
                                                     const float4* __restrict__ cb, const float4* __restrict__ alb, const float4* __restrict__ nrm,
                                                     const unsigned long long* __restrict__ nearest, DnScratch sc, float4* __restrict__ out,
                                                     const DInstance* __restrict__ inst, const float* __restrict__ mat_prev, const DnHistory hin,
                                                     const DnHistory hout, float2* __restrict__ motion, uint32_t* __restrict__ hlen) {
    dn_temporal_px<false>(prm, tp, ca, cb, alb, nrm, nearest, sc, out, inst, mat_prev, hin, hout, motion, hlen, nullptr, 0u, nullptr);
}

__global__ void __launch_bounds__(256) k_dn_temporal_grad(const DnParams prm, const __grid_constant__ DnTemporal tp, const float4* __restrict__ ca,
                                                          const float4* __restrict__ cb, const float4* __restrict__ alb, const float4* __restrict__ nrm,
                                                          const unsigned long long* __restrict__ nearest, DnScratch sc, float4* __restrict__ out,
                                                          const DInstance* __restrict__ inst, const float* __restrict__ mat_prev, const DnHistory hin,
                                                          const DnHistory hout, float2* __restrict__ motion, uint32_t* __restrict__ hlen,
                                                          const float* __restrict__ lam_s, uint32_t gw, float* __restrict__ lam_out) {
    dn_temporal_px<true>(prm, tp, ca, cb, alb, nrm, nearest, sc, out, inst, mat_prev, hin, hout, motion, hlen, lam_s, gw, lam_out);
}

// ---- moment denoising (trb_denoise_moments*, include/trb.h "Moment denoising") ---------------------------------------------------
// One moment record per pixel, 16 bytes: (L(ē), mu1, mu2, n' bits), read by k_dn_moments_variance for the pixel and its 7x7 taps.
// Moment calls take the scene's scratch to DN_MOMENTS_BYTES_PER_PIXEL, the records after the 72 bytes of DnScratch (16-byte aligned).
constexpr size_t DN_MOMENTS_BYTES_PER_PIXEL = DN_BYTES_PER_PIXEL + sizeof(float4);

// Steps 1-3 and 6 of "Moment denoising": trb_denoise's pixel over one film, the history reprojected and gathered as in "Temporal
// denoising" (dn_reproject; a set's records are (ē, z), (mu1, mu2, 0, inst bits), (n, n' bits)) and the blend of the colour and the
// luminance moments. Writes the guide, gradient and divisor as k_dn_prepare does, ev[0] = (ē, 0) (k_dn_moments_variance fills in v),
// the moment record, the history, motion and history length.
// The body of k_dn_temporal_moments (GRAD false) and k_dn_temporal_moments_grad (GRAD true: step 3 shortens the history by the
// pixel's stratum's lambda, include/trb.h "Moment gradients", and lam_out receives it). lam_s: S lambdas on the stratum grid of gw
// columns. tp is taken by value: by reference, k_dn_temporal_moments compiled to other SASS than its body had as a kernel of its own.
template <bool GRAD>
__device__ __forceinline__ void dn_temporal_moments_px(const DnParams prm, const DnTemporal tp, const float4* __restrict__ col,
                                                       const float4* __restrict__ alb, const float4* __restrict__ nrm,
                                                       const unsigned long long* __restrict__ nearest, DnScratch sc, float4* __restrict__ mom,
                                                       float4* __restrict__ out, const DInstance* __restrict__ inst,
                                                       const float* __restrict__ mat_prev, const DnHistory hin, const DnHistory hout,
                                                       float2* __restrict__ motion, uint32_t* __restrict__ hlen, const float* __restrict__ lam_s,
                                                       uint32_t gw, float* __restrict__ lam_out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= prm.width || y >= prm.height) return;
    const int i = y * prm.width + x;
    const float qnan = __int_as_float(0x7fffffff);
    float lam = 0.0f;
    if (GRAD) {
        lam = lam_s[(uint32_t)(y / 3) * gw + (uint32_t)(x / 3)];
        if (lam_out) lam_out[i] = lam;
    }
    const float4 A = col[i];
    const float W = A.w;
    if (W <= 0.0f) {
        out[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        sc.guide[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0x7fc00000));
        hout.n[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (motion) motion[i] = make_float2(qnan, qnan);
        if (hlen) hlen[i] = 0u;
        return;
    }
    const float c0 = A.x / W, c1 = A.y / W, c2 = A.z / W;
    const float4 al = alb[i], nw = nrm[i];
    const float a0 = al.x / al.w, a1 = al.y / al.w, a2 = al.z / al.w;
    const float d0 = a0 > TRB_DENOISE_EPS_ALBEDO ? a0 : TRB_DENOISE_EPS_ALBEDO, d1 = a1 > TRB_DENOISE_EPS_ALBEDO ? a1 : TRB_DENOISE_EPS_ALBEDO,
                d2 = a2 > TRB_DENOISE_EPS_ALBEDO ? a2 : TRB_DENOISE_EPS_ALBEDO;
    float e0 = c0 / d0, e1 = c1 / d1, e2 = c2 / d2;
    const float m0 = nw.x / nw.w, m1 = nw.y / nw.w, m2 = nw.z / nw.w;
    const float len2 = m0 * m0 + m1 * m1 + m2 * m2;
    const unsigned long long key = nearest[i];
    const float z = __uint_as_float((uint32_t)(key >> 32));
    const bool ok = dn_finite(c0) && dn_finite(c1) && dn_finite(c2) && dn_finite(a0) && dn_finite(a1) && dn_finite(a2) && dn_finite(m0) &&
                    dn_finite(m1) && dn_finite(m2) && dn_finite(len2) && dn_finite(e0) && dn_finite(e1) && dn_finite(e2) && z == z &&
                    z != __int_as_float(0xff800000);
    if (!ok) {
        out[i] = dn_out(c0, c1, c2, 1.0f);
        sc.guide[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0x7fc00000));
        hout.n[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (motion) motion[i] = make_float2(qnan, qnan);
        if (hlen) hlen[i] = 0u;
        return;
    }
    float n0 = 0.0f, n1 = 0.0f, n2 = 0.0f;
    if (len2 != 0.0f) {
        const float l = sqrtf(len2);
        n0 = m0 / l; n1 = m1 / l; n2 = m2 / l;
    }
    float gx = 0.0f, gy = 0.0f;
    if (dn_finite(z)) {
        const bool l = x > 0, r = x + 1 < prm.width, u = y > 0, dn = y + 1 < prm.height;
        gx = dn_grad(z, l, l ? dn_depth(nearest, i - 1) : 0.0f, r, r ? dn_depth(nearest, i + 1) : 0.0f);
        gy = dn_grad(z, u, u ? dn_depth(nearest, i - prm.width) : 0.0f, dn, dn ? dn_depth(nearest, i + prm.width) : 0.0f);
    }
    const float l = dn_lum(e0, e1, e2);
    // 2: reconstruct, reproject, gather H' and the moments (hb0, hb1)
    const uint32_t id = (uint32_t)key;
    float mx, my, S, h0, h1, h2, M1, M2, M3;
    uint32_t len_prev;
    dn_reproject(prm, tp, x, y, z, id, n0, n1, n2, inst, mat_prev, hin, mx, my, S, h0, h1, h2, M1, M2, M3, len_prev);
    // 3: blend colour and moments with the same 1 / n'
    uint32_t np = 1;
    if (GRAD) {
        if (S > 0.0f) {
            const uint32_t len_adj = (uint32_t)floorf((1.0f - lam) * (float)len_prev);
            np = len_adj + 1 < tp.max_history ? len_adj + 1 : tp.max_history;
        }
    } else {
        if (S > 0.0f) np = len_prev + 1 < tp.max_history ? len_prev + 1 : tp.max_history;
    }
    float mu1 = l, mu2 = l * l;
    if (np > 1) {
        h0 = h0 / S; h1 = h1 / S; h2 = h2 / S;
        M1 = M1 / S; M2 = M2 / S;
        const float alpha = 1.0f / (float)np, beta = 1.0f - alpha;
        e0 = alpha * e0 + beta * h0; e1 = alpha * e1 + beta * h1; e2 = alpha * e2 + beta * h2;
        mu1 = alpha * l + beta * M1;
        mu2 = alpha * (l * l) + beta * M2;
    }
    sc.guide[i] = make_float4(n0, n1, n2, z);
    sc.grad[i] = make_float2(gx, gy);
    sc.divisor[i] = make_float4(d0, d1, d2, 0.0f);
    sc.ev[0][i] = make_float4(e0, e1, e2, 0.0f);
    mom[i] = make_float4(dn_lum(e0, e1, e2), mu1, mu2, __uint_as_float(np));
    if (prm.iterations == 0) out[i] = dn_out(e0 * d0, e1 * d1, e2 * d2, 1.0f);
    // 6: the new history
    if (dn_finite(z)) {
        hout.a[i] = make_float4(e0, e1, e2, z);
        hout.b[i] = make_float4(mu1, mu2, 0.0f, __uint_as_float(id));
        hout.n[i] = make_float4(n0, n1, n2, __uint_as_float(np));
    } else {
        hout.n[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    if (motion) motion[i] = make_float2(mx == mx ? mx : qnan, my == my ? my : qnan);
    if (hlen) hlen[i] = np;
}

__global__ void __launch_bounds__(256) k_dn_temporal_moments(const DnParams prm, const __grid_constant__ DnTemporal tp, const float4* __restrict__ col,
                                                             const float4* __restrict__ alb, const float4* __restrict__ nrm,
                                                             const unsigned long long* __restrict__ nearest, DnScratch sc, float4* __restrict__ mom,
                                                             float4* __restrict__ out, const DInstance* __restrict__ inst, const float* __restrict__ mat_prev,
                                                             const DnHistory hin, const DnHistory hout, float2* __restrict__ motion,
                                                             uint32_t* __restrict__ hlen) {
    dn_temporal_moments_px<false>(prm, tp, col, alb, nrm, nearest, sc, mom, out, inst, mat_prev, hin, hout, motion, hlen, nullptr, 0u, nullptr);
}

__global__ void __launch_bounds__(256) k_dn_temporal_moments_grad(const DnParams prm, const __grid_constant__ DnTemporal tp,
                                                                  const float4* __restrict__ col, const float4* __restrict__ alb,
                                                                  const float4* __restrict__ nrm, const unsigned long long* __restrict__ nearest,
                                                                  DnScratch sc, float4* __restrict__ mom, float4* __restrict__ out,
                                                                  const DInstance* __restrict__ inst, const float* __restrict__ mat_prev,
                                                                  const DnHistory hin, const DnHistory hout, float2* __restrict__ motion,
                                                                  uint32_t* __restrict__ hlen, const float* __restrict__ lam_s, uint32_t gw,
                                                                  float* __restrict__ lam_out) {
    dn_temporal_moments_px<true>(prm, tp, col, alb, nrm, nearest, sc, mom, out, inst, mat_prev, hin, hout, motion, hlen, lam_s, gw, lam_out);
}

// ---- variance temporal denoising (trb_denoise_variance_temporal*, include/trb.h "Variance temporal denoising") --------------------
// Steps 1-3 and 5: k_dn_variance_prepare's pixel, the history reprojected and gathered as in "Temporal denoising" (dn_reproject; a
// set's records are (ē, z), (V, 0, 0, inst bits), (n, n' bits)) and the blend ē = alpha e + beta H', V = alpha^2 v_f + beta^2 V'.
// Writes the scratch k_dn_prepare writes with ev[0] = (ē, V), the history, motion, history length and variance.
// The body of k_dn_temporal_variance (GRAD false) and k_dn_temporal_variance_grad (GRAD true: n' shortened by the pixel's stratum's
// lambda, and lam_out receives it). tp is taken by value, as in dn_temporal_moments_px.
template <bool GRAD>
__device__ __forceinline__ void dn_temporal_variance_px(const DnParams prm, const DnTemporal tp, const float4* __restrict__ col,
                                                        const float4* __restrict__ lum, const float4* __restrict__ alb,
                                                        const float4* __restrict__ nrm, const unsigned long long* __restrict__ nearest,
                                                        DnScratch sc, float4* __restrict__ out, const DInstance* __restrict__ inst,
                                                        const float* __restrict__ mat_prev, const DnHistory hin, const DnHistory hout,
                                                        float2* __restrict__ motion, uint32_t* __restrict__ hlen, float* __restrict__ var,
                                                        const float* __restrict__ lam_s, uint32_t gw, float* __restrict__ lam_out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= prm.width || y >= prm.height) return;
    const int i = y * prm.width + x;
    const float qnan = __int_as_float(0x7fffffff);
    float lam = 0.0f;
    if (GRAD) {
        lam = lam_s[(uint32_t)(y / 3) * gw + (uint32_t)(x / 3)];
        if (lam_out) lam_out[i] = lam;
    }
    const float4 A = col[i];
    const float W = A.w;
    if (W <= 0.0f) {
        out[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        sc.guide[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0x7fc00000));
        hout.n[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (motion) motion[i] = make_float2(qnan, qnan);
        if (hlen) hlen[i] = 0u;
        if (var) var[i] = qnan;
        return;
    }
    const float c0 = A.x / W, c1 = A.y / W, c2 = A.z / W;
    const float4 al = alb[i], nw = nrm[i], lw = lum[i];
    const float a0 = al.x / al.w, a1 = al.y / al.w, a2 = al.z / al.w;
    const float d0 = a0 > TRB_DENOISE_EPS_ALBEDO ? a0 : TRB_DENOISE_EPS_ALBEDO, d1 = a1 > TRB_DENOISE_EPS_ALBEDO ? a1 : TRB_DENOISE_EPS_ALBEDO,
                d2 = a2 > TRB_DENOISE_EPS_ALBEDO ? a2 : TRB_DENOISE_EPS_ALBEDO;
    float e0 = c0 / d0, e1 = c1 / d1, e2 = c2 / d2;
    const float v = dn_sample_variance(lw);
    const float m0 = nw.x / nw.w, m1 = nw.y / nw.w, m2 = nw.z / nw.w;
    const float len2 = m0 * m0 + m1 * m1 + m2 * m2;
    const unsigned long long key = nearest[i];
    const float z = __uint_as_float((uint32_t)(key >> 32));
    const bool ok = dn_finite(c0) && dn_finite(c1) && dn_finite(c2) && dn_finite(a0) && dn_finite(a1) && dn_finite(a2) && dn_finite(m0) &&
                    dn_finite(m1) && dn_finite(m2) && dn_finite(len2) && dn_finite(e0) && dn_finite(e1) && dn_finite(e2) && dn_finite(v) &&
                    z == z && z != __int_as_float(0xff800000);
    if (!ok) {
        out[i] = dn_out(c0, c1, c2, 1.0f);
        sc.guide[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(0x7fc00000));
        hout.n[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (motion) motion[i] = make_float2(qnan, qnan);
        if (hlen) hlen[i] = 0u;
        if (var) var[i] = qnan;
        return;
    }
    float n0 = 0.0f, n1 = 0.0f, n2 = 0.0f;
    if (len2 != 0.0f) {
        const float l = sqrtf(len2);
        n0 = m0 / l; n1 = m1 / l; n2 = m2 / l;
    }
    float gx = 0.0f, gy = 0.0f;
    if (dn_finite(z)) {
        const bool l = x > 0, r = x + 1 < prm.width, u = y > 0, dn = y + 1 < prm.height;
        gx = dn_grad(z, l, l ? dn_depth(nearest, i - 1) : 0.0f, r, r ? dn_depth(nearest, i + 1) : 0.0f);
        gy = dn_grad(z, u, u ? dn_depth(nearest, i - prm.width) : 0.0f, dn, dn ? dn_depth(nearest, i + prm.width) : 0.0f);
    }
    // 2: reconstruct, reproject, gather H' and V' (hv0)
    const uint32_t id = (uint32_t)key;
    float mx, my, S, h0, h1, h2, hv0, hv1, hv2;
    uint32_t len_prev;
    dn_reproject(prm, tp, x, y, z, id, n0, n1, n2, inst, mat_prev, hin, mx, my, S, h0, h1, h2, hv0, hv1, hv2, len_prev);
    // 3: blend the colour with 1 / n' and the variance with its square
    uint32_t np = 1;
    if (GRAD) {
        if (S > 0.0f) {
            const uint32_t len_adj = (uint32_t)floorf((1.0f - lam) * (float)len_prev);
            np = len_adj + 1 < tp.max_history ? len_adj + 1 : tp.max_history;
        }
    } else {
        if (S > 0.0f) np = len_prev + 1 < tp.max_history ? len_prev + 1 : tp.max_history;
    }
    float V = v;
    if (np > 1) {
        h0 = h0 / S; h1 = h1 / S; h2 = h2 / S;
        hv0 = hv0 / S;
        const float alpha = 1.0f / (float)np, beta = 1.0f - alpha;
        e0 = alpha * e0 + beta * h0; e1 = alpha * e1 + beta * h1; e2 = alpha * e2 + beta * h2;
        V = (alpha * alpha) * v + (beta * beta) * hv0;
    }
    sc.guide[i] = make_float4(n0, n1, n2, z);
    sc.grad[i] = make_float2(gx, gy);
    sc.divisor[i] = make_float4(d0, d1, d2, 0.0f);
    sc.ev[0][i] = make_float4(e0, e1, e2, V);
    if (prm.iterations == 0) out[i] = dn_out(e0 * d0, e1 * d1, e2 * d2, 1.0f);
    // 5: the new history
    if (dn_finite(z)) {
        hout.a[i] = make_float4(e0, e1, e2, z);
        hout.b[i] = make_float4(V, 0.0f, 0.0f, __uint_as_float(id));
        hout.n[i] = make_float4(n0, n1, n2, __uint_as_float(np));
    } else {
        hout.n[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    if (motion) motion[i] = make_float2(mx == mx ? mx : qnan, my == my ? my : qnan);
    if (hlen) hlen[i] = np;
    if (var) var[i] = V;
}

__global__ void __launch_bounds__(256) k_dn_temporal_variance(const DnParams prm, const __grid_constant__ DnTemporal tp, const float4* __restrict__ col,
                                                              const float4* __restrict__ lum, const float4* __restrict__ alb,
                                                              const float4* __restrict__ nrm, const unsigned long long* __restrict__ nearest,
                                                              DnScratch sc, float4* __restrict__ out, const DInstance* __restrict__ inst,
                                                              const float* __restrict__ mat_prev, const DnHistory hin, const DnHistory hout,
                                                              float2* __restrict__ motion, uint32_t* __restrict__ hlen, float* __restrict__ var) {
    dn_temporal_variance_px<false>(prm, tp, col, lum, alb, nrm, nearest, sc, out, inst, mat_prev, hin, hout, motion, hlen, var, nullptr, 0u, nullptr);
}

__global__ void __launch_bounds__(256) k_dn_temporal_variance_grad(const DnParams prm, const __grid_constant__ DnTemporal tp,
                                                                   const float4* __restrict__ col, const float4* __restrict__ lum,
                                                                   const float4* __restrict__ alb, const float4* __restrict__ nrm,
                                                                   const unsigned long long* __restrict__ nearest, DnScratch sc,
                                                                   float4* __restrict__ out, const DInstance* __restrict__ inst,
                                                                   const float* __restrict__ mat_prev, const DnHistory hin, const DnHistory hout,
                                                                   float2* __restrict__ motion, uint32_t* __restrict__ hlen, float* __restrict__ var,
                                                                   const float* __restrict__ lam_s, uint32_t gw, float* __restrict__ lam_out) {
    dn_temporal_variance_px<true>(prm, tp, col, lum, alb, nrm, nearest, sc, out, inst, mat_prev, hin, hout, motion, hlen, var, lam_s, gw, lam_out);
}

// Step 4 of "Moment denoising": each filtered pixel's variance, mu2 - mu1^2 from its own moments once n' >= MIN_HISTORY, else the
// 7x7 edge-stopped estimate over its neighbours' moments boosted by 4 / n'. Writes v into ev[0].w (and var, NaN where not filtered).
__global__ void __launch_bounds__(256) k_dn_moments_variance(const DnParams prm, const float4* __restrict__ guide, const float2* __restrict__ grad,
                                                             const float4* __restrict__ mom, float4* __restrict__ ev, float* __restrict__ var) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= prm.width || y >= prm.height) return;
    const int W = prm.width, H = prm.height, i = y * W + x;
    const float4 gp = guide[i];
    if (gp.w != gp.w) { // not filtered
        if (var) var[i] = __int_as_float(0x7fffffff);
        return;
    }
    const float4 mp = mom[i];
    const uint32_t np = __float_as_uint(mp.w);
    float v;
    if (np >= TRB_DENOISE_MOMENTS_MIN_HISTORY) {
        v = mp.z - mp.y * mp.y;
        v = v > 0.0f ? v : 0.0f;
    } else {
        const float2 g = grad[i];
        const bool p_inf = !dn_finite(gp.w), p_nrm = gp.x != 0.0f || gp.y != 0.0f || gp.z != 0.0f;
        const float denom_l = prm.sigma_l + TRB_DENOISE_EPS_LUMINANCE;
        float sw = 0.0f, s1 = 0.0f, s2 = 0.0f;
        for (int dy = -TRB_DENOISE_MOMENTS_RADIUS; dy <= TRB_DENOISE_MOMENTS_RADIUS; ++dy) {
            const int qy = y + dy;
            if (qy < 0 || qy >= H) continue;
            for (int dx = -TRB_DENOISE_MOMENTS_RADIUS; dx <= TRB_DENOISE_MOMENTS_RADIUS; ++dx) {
                const int qx = x + dx;
                if (qx < 0 || qx >= W) continue;
                const int q = qy * W + qx;
                const float4 gq = guide[q];
                if (gq.w != gq.w) continue;
                const float4 mq = mom[q];
                const float wl = dexp(-(fabsf(mp.x - mq.x) / denom_l));
                float wn;
                const bool q_nrm = gq.x != 0.0f || gq.y != 0.0f || gq.z != 0.0f;
                if (p_nrm != q_nrm) wn = 0.0f;
                else if (!p_nrm) wn = 1.0f;
                else {
                    const float dot = gp.x * gq.x + gp.y * gq.y + gp.z * gq.z;
                    wn = dot > 0.0f ? dot : 0.0f;
                    for (uint32_t k = 0; k < prm.normal_squarings; ++k) wn = wn * wn;
                }
                float wz;
                const bool q_inf = !dn_finite(gq.w);
                if (p_inf != q_inf) wz = 0.0f;
                else if (p_inf) wz = 1.0f;
                else wz = dexp(-(fabsf(gp.w - gq.w) / (prm.sigma_z * fabsf(g.x * (float)dx + g.y * (float)dy) + TRB_DENOISE_EPS_DEPTH)));
                float w = wl * wn;
                w = w * wz;
                sw = sw + w;
                s1 = s1 + w * mq.y;
                s2 = s2 + w * mq.z;
            }
        }
        const float m1 = s1 / sw, m2 = s2 / sw;
        v = m2 - m1 * m1;
        v = v > 0.0f ? v : 0.0f;
        v = v * (4.0f / (float)np);
    }
    reinterpret_cast<float*>(ev + i)[3] = v;
    if (var) var[i] = v;
}

// ---- temporal gradients (trb_denoise_temporal_gradient*, include/trb.h "Temporal gradients") --------------------------------------
// One gradient record per 3x3 stratum, 64 bytes: (p_o, inst bits) (o, time) (d, key bits) (L, 0, 0, 0); inst == TRB_MISS: none
struct GrRecords {
    float4* r;       // 4 float4 per stratum
};
constexpr uint32_t GR_STRATUM = 3;
constexpr uint32_t GR_PICK_STREAM = 0xfffffffeu;

// The current frame (camera at shutter-open, film size, stratum grid) and the snapshot the records were written at
struct GrFrame {
    float cam_mat[16], cam_inv[16];
    float tan_cur, x0, x1, y0, y1, w, h;
    uint32_t width, height, gw, gh;
    uint32_t n_cur, n_prev;
    uint32_t cam_same;      // the current cam_mat is bit-identical to the snapshot's
    float dt;               // shutter_open_cur - shutter_open_prev
    float depth_tolerance, normal_threshold;
};

__device__ __forceinline__ float gr_lum(float r, float g, float b) { return 0.2126f * r + 0.7152f * g + 0.0722f * b; }

// Step 1, forward projection: record j of the read set to the raster of the current frame; the winner of each target stratum is the
// smallest (float bits of the distance << 32 | j)
__global__ void __launch_bounds__(256) k_gr_project(const __grid_constant__ GrFrame f, const float4* __restrict__ rec,
                                                    const DInstance* __restrict__ inst, const unsigned long long* __restrict__ nearest,
                                                    unsigned long long* __restrict__ slot) {
    const uint32_t S = f.gw * f.gh;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < S; j += gridDim.x * blockDim.x) {
        const float4 r0 = rec[4 * (size_t)j];
        const uint32_t id = __float_as_uint(r0.w);
        if (id == TRB_MISS || id >= f.n_cur || id >= f.n_prev) continue;
        const f3 pw = xf_point(inst[id].mat, mk(r0.x, r0.y, r0.z));
        const f3 q = xf_point(f.cam_inv, pw);
        if (!(q.z > 0.0f)) continue;
        const float X = q.x / (q.z * f.tan_cur), Y = q.y / (q.z * f.tan_cur);
        const float rx = (X - f.x0) / (f.x1 - f.x0) * f.w, ry = (Y - f.y1) / (f.y0 - f.y1) * f.h;
        if (!(rx >= 0.0f && rx < f.w && ry >= 0.0f && ry < f.h)) continue;
        const uint32_t px = (uint32_t)rx, py = (uint32_t)ry;
        if (px >= f.width || py >= f.height) continue;
        const unsigned long long key = nearest[(size_t)py * f.width + px];
        if ((uint32_t)key != id) continue;
        const float z = __uint_as_float((uint32_t)(key >> 32));
        const f3 o = xf_point(f.cam_mat, splat(0.0f));
        const f3 v = mk(pw.x - o.x, pw.y - o.y, pw.z - o.z);
        const float dist = sqrtf(v.x * v.x + v.y * v.y + v.z * v.z);
        if (!(fabsf(z - dist) <= f.depth_tolerance * z)) continue;
        const uint32_t t = (py / GR_STRATUM) * f.gw + px / GR_STRATUM;
        atomicMin(slot + t, ((unsigned long long)__float_as_uint(dist) << 32) | j);
    }
}

// Step 1, the winner's illumination ray (the recorded one when camera and instance did not move, else from the camera to p_w'), and
// each stratum's guide for the reconstruction: its representative pixel's unit normal (0 if none) and instance
__global__ void __launch_bounds__(256) k_gr_resolve(const __grid_constant__ GrFrame f, const float4* __restrict__ rec, const DInstance* __restrict__ inst,
                                                    const float* __restrict__ mat_prev, const unsigned long long* __restrict__ slot,
                                                    const float4* __restrict__ nrm, const unsigned long long* __restrict__ nearest,
                                                    trb_illum_ray* __restrict__ rays, float4* __restrict__ guide) {
    const uint32_t S = f.gw * f.gh;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < S; t += gridDim.x * blockDim.x) {
        const uint32_t sx = t % f.gw, sy = t / f.gw;
        const uint32_t rx = min(sx * GR_STRATUM + 1, f.width - 1), ry = min(sy * GR_STRATUM + 1, f.height - 1);
        const size_t rp = (size_t)ry * f.width + rx;
        const float4 nw = nrm[rp];
        const float m0 = nw.x / nw.w, m1 = nw.y / nw.w, m2 = nw.z / nw.w;
        const float l2 = m0 * m0 + m1 * m1 + m2 * m2;
        float n0 = 0.0f, n1 = 0.0f, n2 = 0.0f;
        if (dn_finite(l2) && l2 != 0.0f) {
            const float l = sqrtf(l2);
            n0 = m0 / l; n1 = m1 / l; n2 = m2 / l;
        }
        guide[t] = make_float4(n0, n1, n2, __uint_as_float((uint32_t)nearest[rp]));
        const unsigned long long w = slot[t];
        trb_illum_ray r;
        if (w == ~0ull) { // no winner: a ray that hits nothing
            r.o[0] = r.o[1] = r.o[2] = 0.0f;
            r.d[0] = r.d[1] = r.d[2] = 0.5773502691896258f;
            r.min_t = 0.0f; r.max_t = 0.0f; r.time = 0.0f; r.key = 0u; r.sample = 0u;
        } else {
            const uint32_t j = (uint32_t)w;
            const float4 r0 = rec[4 * (size_t)j], r1 = rec[4 * (size_t)j + 1], r2 = rec[4 * (size_t)j + 2];
            const uint32_t id = __float_as_uint(r0.w);
            bool same = f.cam_same != 0u;
            const float* mc = inst[id].mat;
            const float* mp = mat_prev + 16 * (size_t)id;
            for (int k = 0; k < 16 && same; ++k) same = __float_as_uint(mc[k]) == __float_as_uint(mp[k]);
            if (same) {
                r.o[0] = r1.x; r.o[1] = r1.y; r.o[2] = r1.z;
                r.d[0] = r2.x; r.d[1] = r2.y; r.d[2] = r2.z;
            } else {
                const f3 pw = xf_point(mc, mk(r0.x, r0.y, r0.z));
                const f3 o = xf_point(f.cam_mat, splat(0.0f));
                const f3 d = unit(mk(pw.x - o.x, pw.y - o.y, pw.z - o.z));
                r.o[0] = o.x; r.o[1] = o.y; r.o[2] = o.z;
                r.d[0] = d.x; r.d[1] = d.y; r.d[2] = d.z;
            }
            r.min_t = 0.0f; r.max_t = finf();
            r.time = r1.w + f.dt;
            r.key = __float_as_uint(r2.w); r.sample = 0u;
        }
        r.pad = 0u;
        rays[t] = r;
    }
}

// Step 1, each stratum's (delta, m, c): the re-shaded luminance against the recorded one where there is a winner, else 0
__global__ void __launch_bounds__(256) k_gr_delta(uint32_t S, const float4* __restrict__ rec, const unsigned long long* __restrict__ slot,
                                                  const float* __restrict__ rgb, float4* __restrict__ dm, float* __restrict__ lam_s) {
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < S; t += gridDim.x * blockDim.x) {
        const unsigned long long w = slot[t];
        float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (w != ~0ull) {
            const float lc = gr_lum(rgb[3 * (size_t)t], rgb[3 * (size_t)t + 1], rgb[3 * (size_t)t + 2]);
            const float lp = rec[4 * (size_t)(uint32_t)w + 3].x;
            v = make_float4(lc - lp, lc > lp ? lc : lp, 1.0f, 0.0f);
        }
        dm[t] = v;
        if (lam_s) lam_s[t] = v.z > 0.0f && v.y > 0.0f ? fminf(1.0f, fabsf(v.x) / v.y) : 0.0f; // no a-trous pass
    }
}

// Step 2, one a-trous pass at a step of s strata over (delta, m, c); the last one (lam_s non-null) writes lambda instead
__global__ void __launch_bounds__(256) k_gr_atrous(uint32_t gw, uint32_t gh, int s, float normal_threshold, const float4* __restrict__ guide,
                                                   const float4* __restrict__ dm_in, float4* __restrict__ dm_out, float* __restrict__ lam_s) {
    const uint32_t S = gw * gh;
    const float h[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < S; t += gridDim.x * blockDim.x) {
        const int x = (int)(t % gw), y = (int)(t / gw);
        const float4 gp = guide[t];
        const bool p_nrm = gp.x != 0.0f || gp.y != 0.0f || gp.z != 0.0f;
        float W = 0.0f, sd = 0.0f, sm = 0.0f;
#pragma unroll
        for (int dy = -2; dy <= 2; ++dy) {
            const int qy = y + s * dy;
            if (qy < 0 || qy >= (int)gh) continue;
#pragma unroll
            for (int dx = -2; dx <= 2; ++dx) {
                const int qx = x + s * dx;
                if (qx < 0 || qx >= (int)gw) continue;
                const uint32_t q = (uint32_t)qy * gw + (uint32_t)qx;
                const float4 v = dm_in[q];
                if (!(v.z > 0.0f)) continue;
                if (q != t) {
                    const float4 gq = guide[q];
                    if (__float_as_uint(gq.w) != __float_as_uint(gp.w)) continue;
                    const bool q_nrm = gq.x != 0.0f || gq.y != 0.0f || gq.z != 0.0f;
                    if (q_nrm != p_nrm) continue;
                    if (p_nrm && !(gp.x * gq.x + gp.y * gq.y + gp.z * gq.z >= normal_threshold)) continue;
                }
                const float w = h[dx + 2] * h[dy + 2];
                W = W + w;
                sd = sd + w * v.x;
                sm = sm + w * v.y;
            }
        }
        float4 o = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (W > 0.0f) o = make_float4(sd / W, sm / W, 1.0f, 0.0f);
        if (lam_s) lam_s[t] = o.z > 0.0f && o.y > 0.0f ? fminf(1.0f, fabsf(o.x) / o.y) : 0.0f;
        else dm_out[t] = o;
    }
}

// Step 4, this frame's samples: one pixel per stratum picked by the draw (seed, s, GR_PICK_STREAM, 0), its camera ray as
// k_camera_rays generates sample 0 of 1, as a query ray (for the hit) and an illumination ray (for L)
template <bool ANIM>
__global__ void __launch_bounds__(256) k_gr_record(const __grid_constant__ DScene sc, uint32_t gw, uint32_t gh, uint32_t seed,
                                                   trb_query_ray* __restrict__ qrays, trb_illum_ray* __restrict__ irays) {
    const uint32_t S = gw * gh, W = (uint32_t)sc.width, H = (uint32_t)sc.height;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < S; t += gridDim.x * blockDim.x) {
        const uint32_t sx = t % gw, sy = t / gw;
        const uint32_t cw = min(GR_STRATUM, W - sx * GR_STRATUM), ch = min(GR_STRATUM, H - sy * GR_STRATUM);
        const uint32_t k = rng_absorb(rng_absorb(rng_absorb(rng_seed(seed), t), GR_PICK_STREAM), 0u) % (cw * ch);
        const uint32_t px = sx * GR_STRATUM + k % cw, py = sy * GR_STRATUM + k / cw, pixel = py * W + px;
        const PixelStreams ps = pixel_streams(seed, pixel);
        const uint32_t ip = permute_index(0u, 1u, ps.kpos);
        const float fx = ld_vdc(ip, ps.scr0) + (float)px, fy = ld_sobol(ip, ps.scr1) + (float)py;
        const float tm = ld_vdc(permute_index(0u, 1u, ps.ktime), ps.scrt);
        Ray r;
        const float time = camera_ray<ANIM>(sc, fx, fy, tm, r);
        trb_query_ray q;
        q.o[0] = r.o.x; q.o[1] = r.o.y; q.o[2] = r.o.z; q.d[0] = r.d.x; q.d[1] = r.d.y; q.d[2] = r.d.z;
        q.min_t = r.tmin; q.max_t = r.tmax; q.time = time; q.pad[0] = q.pad[1] = q.pad[2] = 0u;
        qrays[t] = q;
        trb_illum_ray l;
        l.o[0] = r.o.x; l.o[1] = r.o.y; l.o[2] = r.o.z; l.d[0] = r.d.x; l.d[1] = r.d.y; l.d[2] = r.d.z;
        l.min_t = r.tmin; l.max_t = r.tmax; l.time = time; l.key = pixel; l.sample = 0u; l.pad = 0u;
        irays[t] = l;
    }
}

// Step 4, the records of the write set: the hit's instance and object-space point (shutter-open inverse), the ray and L
__global__ void __launch_bounds__(256) k_gr_store(uint32_t S, const trb_intersection* __restrict__ hits, const trb_illum_ray* __restrict__ irays,
                                                  const float* __restrict__ rgb, const DInstance* __restrict__ inst, float4* __restrict__ rec) {
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < S; t += gridDim.x * blockDim.x) {
        const trb_intersection& hit = hits[t];
        const trb_illum_ray& l = irays[t];
        float4* o = rec + 4 * (size_t)t;
        if (hit.inst == TRB_MISS) {
            o[0] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(TRB_MISS));
            continue;
        }
        const f3 po = xf_point(inst[hit.inst].inv, mk(hit.p[0], hit.p[1], hit.p[2]));
        o[0] = make_float4(po.x, po.y, po.z, __uint_as_float(hit.inst));
        o[1] = make_float4(l.o[0], l.o[1], l.o[2], l.time);
        o[2] = make_float4(l.d[0], l.d[1], l.d[2], __uint_as_float(l.key));
        o[3] = make_float4(gr_lum(rgb[3 * (size_t)t], rgb[3 * (size_t)t + 1], rgb[3 * (size_t)t + 2]), 0.0f, 0.0f, 0.0f);
    }
}

} // namespace trb
