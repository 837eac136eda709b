/* The parity oracle's variance temporal denoiser — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into
 * oracle/_build/liboracle_variance_temporal.so and loaded by oracle_variance_temporal/pyvariancetemporal.py.
 *
 * This translation unit is the temporal gradient oracle (oracle_gradient/gradient.cpp, which includes the ray-query oracle and the
 * denoiser oracle), included whole, plus the contract of include/trb.h "Variance temporal denoising" (DESIGN.md §4) restated over its
 * CPU history: the tap gather and scene snapshot are gradient.cpp's (the gather of "Temporal denoising"), the a-trous filter is
 * denoise.cpp's, and v_f is step 2 of "Sample variance" restated here (oracle_variance/variance.cpp and oracle_temporal/temporal.cpp
 * cannot be included as well: each include chain defines oracle.cpp and denoise.cpp).
 *   orc_denoise_variance_temporal_lambda_frame  the contract over an explicit frame (orc_gradient_frame) with a caller lambda per
 *                                               stratum, so synthetic frames need no scene; the records are not touched
 *   orc_denoise_variance_temporal               the plain call with an oracle scene after orc_scene_update_frame (lambda 0)
 *   orc_denoise_variance_temporal_gradient      steps 1, 2 and 4 of "Temporal gradients" with an oracle scene around the blend
 * The history is gradient.cpp's orc_gradient_history (orc_gradient_history_create / _destroy / _reset) with ha holding ē and hb
 * (V, 0, 0); like the other oracles it has no family tag (a caller does not mix the families on one history).
 */
#include "../oracle_gradient/gradient.cpp"

namespace {

/* "Variance temporal denoising" with step 3's n' shortened by lambda (lam_s per stratum; lam_px per pixel out) */
void variance_lambda(uint32_t width, uint32_t height, const orc_gradient_frame* f, orc_gradient_history* h, const trb_denoise_frame* in,
                     const float* lum_w, const trb_denoise_params& p, int squarings, const GradPrm& t, const float* lam_s, float* rgbw,
                     float* motion, uint32_t* history_length, float* variance, float* lam_px) {
    const long W = width, H = height, N = W * H, gw = (W + 2) / 3;
    const float qnan = dm_from_bits(0x7fffffffu);
    /* 1: trb_denoise_variance's pixel */
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
            /* v_f: the variance of the pixel's weighted mean of l */
            const float V1 = lw[3], V2 = lw[2];
            float vf = qnan;
            if (V1 > 0.0f && V1 * V1 > V2) {
                const float m1 = lw[0] / V1, m2 = lw[1] / V1;
                const float s2 = m2 - m1 * m1;
                vf = (s2 > 0.0f ? s2 : 0.0f) * V2 / (V1 * V1 - V2);
            }
            const float len2 = m[0] * m[0] + m[1] * m[1] + m[2] * m[2];
            q.z = depth_of(in->nearest[i]);
            ok = ok && fin(len2) && fin(vf) && !std::isnan(q.z) && q.z != -INFINITY;
            if (!ok) continue;
            q.valid = true;
            v[i] = vf;
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
    /* 2-3 and 5: reproject, blend ē with 1 / n' and V with its square, the new history */
    std::vector<float> nha(N * 3), nhb(N * 3), nn(N * 3), nz(N);
    std::vector<uint32_t> ninst(N), nlen(N, 0u);
    for (long y = 0; y < H; ++y)
        for (long x = 0; x < W; ++x) {
            const long i = y * W + x;
            const float lam = lam_s[(y / 3) * gw + x / 3];
            if (lam_px) lam_px[i] = lam;
            const Px& P = px[i];
            float mx = qnan, my = qnan;
            uint32_t np = 0;
            if (P.valid) {
                const uint32_t id = (uint32_t)in->nearest[i];
                float S = 0.0f, sh[3] = {0, 0, 0}, sv[3] = {0, 0, 0};
                uint32_t len_prev = 0;
                gradient_gather(W, H, x, y, P, id, f, h, t, mx, my, S, sh, sv, len_prev);
                np = S > 0.0f ? std::min((uint32_t)std::floor((1.0f - lam) * (float)len_prev) + 1u, t.max_history) : 1u;
                if (np > 1) {
                    const float alpha = 1.0f / (float)np, beta = 1.0f - alpha;
                    for (int c = 0; c < 3; ++c) e[3 * i + c] = alpha * e[3 * i + c] + beta * (sh[c] / S);
                    v[i] = (alpha * alpha) * v[i] + (beta * beta) * (sv[0] / S);
                }
                if (fin(P.z)) {
                    for (int c = 0; c < 3; ++c) { nha[3 * i + c] = e[3 * i + c]; nn[3 * i + c] = P.n[c]; }
                    nhb[3 * i] = v[i]; nhb[3 * i + 1] = 0.0f; nhb[3 * i + 2] = 0.0f;
                    nz[i] = P.z; ninst[i] = id; nlen[i] = np;
                }
            }
            if (motion) { motion[2 * i] = std::isnan(mx) ? qnan : mx; motion[2 * i + 1] = std::isnan(my) ? qnan : my; }
            if (history_length) history_length[i] = np;
            if (variance) variance[i] = P.valid ? v[i] : qnan;
        }
    /* 4 */
    denoise_filter(W, H, p, squarings, px, std::move(e), std::move(v), rgbw);
    h->ha.swap(nha); h->hb.swap(nhb); h->n.swap(nn); h->z.swap(nz); h->inst.swap(ninst); h->len.swap(nlen);
    std::memcpy(h->cam_inv, f->cam_inv, 64);
    h->tan_fov = f->scaling[0];
    h->n_instances = f->n_instances;
    h->mats.assign(f->mat, f->mat + 16 * (size_t)f->n_instances);
    h->has_prev = true; h->bound = true; h->width = width; h->height = height;
}

bool frame_ok(const trb_denoise_frame* in, const float* lum_w) { return in && lum_w && in->colour && in->albedo_w && in->normal_w && in->nearest; }

}  // namespace

extern "C" {

int orc_denoise_variance_temporal_lambda_frame(uint32_t width, uint32_t height, const orc_gradient_frame* f, orc_gradient_history* h,
                                               const trb_denoise_frame* in, const float* lum_w, const trb_denoise_gradient_params* params,
                                               const float* lam_s, float* rgbw, float* motion, uint32_t* history_length, float* variance,
                                               float* lam_px) {
    trb_denoise_params p;
    int squarings;
    GradPrm t;
    if (!gradient_params(params, p, squarings, t)) return TRB_INVALID_ARG;
    if (!f || !h || !rgbw || !lam_s || !frame_ok(in, lum_w)) return TRB_INVALID_ARG;
    if (h->bound && (h->width != width || h->height != height)) return TRB_INVALID_ARG;
    variance_lambda(width, height, f, h, in, lum_w, p, squarings, t, lam_s, rgbw, motion, history_length, variance, lam_px);
    h->gr_valid = false;
    return TRB_OK;
}

int orc_denoise_variance_temporal(orc_scene* s, orc_gradient_history* h, const trb_denoise_frame* in, const float* lum_w,
                                  const trb_denoise_temporal_params* params, float* rgbw, float* motion, uint32_t* history_length, float* variance) {
    trb_denoise_gradient_params g{};
    if (params) g.temporal = *params;
    trb_denoise_params p;
    int squarings;
    GradPrm t;
    if (!gradient_params(params ? &g : nullptr, p, squarings, t)) return TRB_INVALID_ARG;
    if (!s || s->active_camera < 0) { g_err = "update_frame must be called before a temporal denoise"; return TRB_INVALID_ARG; }
    if (!h || !rgbw || !frame_ok(in, lum_w)) return TRB_INVALID_ARG;
    const uint32_t W = s->film.width, H = s->film.height;
    if (h->bound && (h->width != W || h->height != H)) return TRB_INVALID_ARG;
    orc_gradient_frame f;
    std::vector<float> inv, mat;
    scene_gradient_frame(s, f, inv, mat);
    const std::vector<float> lam((size_t)((W + 2) / 3) * ((H + 2) / 3), 0.0f);
    variance_lambda(W, H, &f, h, in, lum_w, p, squarings, t, lam.data(), rgbw, motion, history_length, variance, nullptr);
    h->gr_valid = false;
    return TRB_OK;
}

int orc_denoise_variance_temporal_gradient(orc_scene* s, orc_gradient_history* h, const trb_denoise_frame* in, const float* lum_w,
                                           const trb_denoise_gradient_params* params, uint32_t seed, float* rgbw, float* motion,
                                           uint32_t* history_length, float* variance, float* lam_px) {
    trb_denoise_params p;
    int squarings;
    GradPrm t;
    if (!gradient_params(params, p, squarings, t)) return TRB_INVALID_ARG;
    if (!s || s->active_camera < 0) { g_err = "update_frame must be called before a temporal denoise"; return TRB_INVALID_ARG; }
    if (!h || !rgbw || !frame_ok(in, lum_w)) return TRB_INVALID_ARG;
    const uint32_t W = s->film.width, H = s->film.height;
    if (h->bound && (h->width != W || h->height != H)) return TRB_INVALID_ARG;
    orc_gradient_frame f;
    std::vector<float> inv, mat;
    scene_gradient_frame(s, f, inv, mat);
    std::vector<float> lam;
    scene_lambda(s, h, f, in->normal_w, in->nearest, t, lam);
    variance_lambda(W, H, &f, h, in, lum_w, p, squarings, t, lam.data(), rgbw, motion, history_length, variance, lam_px);
    scene_record(s, h, f, seed);
    return TRB_OK;
}

}  // extern "C"
