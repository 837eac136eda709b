/* The parity oracle's moment gradients — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into
 * oracle/_build/liboracle_moment_gradient.so and loaded by oracle_moment_gradient/pymomentgradient.py.
 *
 * This translation unit is the temporal gradient oracle (oracle_gradient/gradient.cpp, which includes the ray-query oracle and the
 * denoiser oracle), included whole, plus the contract of include/trb.h "Moment gradients" (DESIGN.md §4) restated over its CPU history:
 * "Moment denoising" once more, with the lambda of step 3 (oracle_moments/moments.cpp cannot be included as well: both include chains
 * define oracle.cpp and denoise.cpp).
 *   orc_denoise_moments_lambda_frame  "Moment denoising" over an explicit frame (orc_gradient_frame) with a caller lambda per stratum,
 *                                     so synthetic frames need no scene; the records are not touched
 *   orc_denoise_moments_gradient      steps 1, 2 and 4 of "Temporal gradients" with an oracle scene after orc_scene_update_frame (its
 *                                     camera rays, ray-query records and trb_illumination), around that blend
 * The history is gradient.cpp's orc_gradient_history (orc_gradient_history_create / _destroy / _reset) with ha holding ē and hb
 * (mu1, mu2, 0); like the other oracles it has no family tag (a caller does not mix the half-film and moment calls on one history).
 */
#include "../oracle_gradient/gradient.cpp"

namespace {

/* "Moment denoising" with step 3's n' shortened by lambda (lam_s per stratum; lam_px per pixel out) */
void moments_lambda(uint32_t width, uint32_t height, const orc_gradient_frame* f, orc_gradient_history* h, const trb_denoise_frame* in,
                    const trb_denoise_params& p, int squarings, const GradPrm& t, const float* lam_s, float* rgbw, float* motion,
                    uint32_t* history_length, float* variance, float* lam_px) {
    const long W = width, H = height, N = W * H, gw = (W + 2) / 3;
    const float qnan = dm_from_bits(0x7fffffffu);
    /* 1: trb_denoise's pixel over one film */
    std::vector<Px> px(N);
    std::vector<float> e(N * 3, 0.0f);
    for (long y = 0; y < H; ++y)
        for (long x = 0; x < W; ++x) {
            const long i = y * W + x;
            Px& q = px[i];
            const float* A = in->colour + 4 * i;
            const float* al = in->albedo_w + 4 * i;
            const float* nw = in->normal_w + 4 * i;
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
            const float len2 = m[0] * m[0] + m[1] * m[1] + m[2] * m[2];
            q.z = depth_of(in->nearest[i]);
            ok = ok && fin(len2) && !std::isnan(q.z) && q.z != -INFINITY;
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
    /* 2-3 and 6, n' = min(floor((1 - lambda) len_prev) + 1, max_history) where there is history */
    std::vector<float> mu1(N, 0.0f), mu2(N, 0.0f), v(N, 0.0f);
    std::vector<uint32_t> nps(N, 0u);
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
                const float l = lum(&e[3 * i]);
                float S = 0.0f, sh[3] = {0, 0, 0}, sm[3] = {0, 0, 0};
                uint32_t len_prev = 0;
                gradient_gather(W, H, x, y, P, id, f, h, t, mx, my, S, sh, sm, len_prev);
                np = S > 0.0f ? std::min((uint32_t)std::floor((1.0f - lam) * (float)len_prev) + 1u, t.max_history) : 1u;
                mu1[i] = l; mu2[i] = l * l;
                if (np > 1) {
                    const float alpha = 1.0f / (float)np, beta = 1.0f - alpha;
                    for (int c = 0; c < 3; ++c) e[3 * i + c] = alpha * e[3 * i + c] + beta * (sh[c] / S);
                    mu1[i] = alpha * l + beta * (sm[0] / S);
                    mu2[i] = alpha * (l * l) + beta * (sm[1] / S);
                }
                nps[i] = np;
                if (fin(P.z)) {
                    for (int c = 0; c < 3; ++c) { nha[3 * i + c] = e[3 * i + c]; nn[3 * i + c] = P.n[c]; }
                    nhb[3 * i] = mu1[i]; nhb[3 * i + 1] = mu2[i]; nhb[3 * i + 2] = 0.0f;
                    nz[i] = P.z; ninst[i] = id; nlen[i] = np;
                }
            }
            if (motion) { motion[2 * i] = std::isnan(mx) ? qnan : mx; motion[2 * i + 1] = std::isnan(my) ? qnan : my; }
            if (history_length) history_length[i] = np;
        }
    /* 4 */
    const long R = TRB_DENOISE_MOMENTS_RADIUS;
    for (long y = 0; y < H; ++y)
        for (long x = 0; x < W; ++x) {
            const long i = y * W + x;
            const Px& P = px[i];
            if (!P.valid) { if (variance) variance[i] = qnan; continue; }
            float vi;
            if (nps[i] >= TRB_DENOISE_MOMENTS_MIN_HISTORY) {
                vi = mu2[i] - mu1[i] * mu1[i];
                vi = vi > 0.0f ? vi : 0.0f;
            } else {
                const float lp = lum(&e[3 * i]);
                const float sigma_l = p.sigma_luminance + TRB_DENOISE_EPS_LUMINANCE;
                float sw = 0.0f, s1 = 0.0f, s2 = 0.0f;
                for (long dy = -R; dy <= R; ++dy)
                    for (long dx = -R; dx <= R; ++dx) {
                        const long qx = x + dx, qy = y + dy;
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
                            const float along = P.gx * (float)dx + P.gy * (float)dy;
                            w_z = dm_expf(-(std::fabs(P.z - Q.z) / (p.sigma_depth * std::fabs(along) + TRB_DENOISE_EPS_DEPTH)));
                        }
                        const float w = w_l * w_n * w_z;
                        sw = sw + w;
                        s1 = s1 + w * mu1[j];
                        s2 = s2 + w * mu2[j];
                    }
                const float m1 = s1 / sw, m2 = s2 / sw;
                vi = m2 - m1 * m1;
                vi = vi > 0.0f ? vi : 0.0f;
                vi = vi * (4.0f / (float)nps[i]);
            }
            v[i] = vi;
            if (variance) variance[i] = vi;
        }
    /* 5 */
    denoise_filter(W, H, p, squarings, px, std::move(e), std::move(v), rgbw);
    h->ha.swap(nha); h->hb.swap(nhb); h->n.swap(nn); h->z.swap(nz); h->inst.swap(ninst); h->len.swap(nlen);
    std::memcpy(h->cam_inv, f->cam_inv, 64);
    h->tan_fov = f->scaling[0];
    h->n_instances = f->n_instances;
    h->mats.assign(f->mat, f->mat + 16 * (size_t)f->n_instances);
    h->has_prev = true; h->bound = true; h->width = width; h->height = height;
}

bool frame_ok(const trb_denoise_frame* in) { return in && in->colour && in->albedo_w && in->normal_w && in->nearest; }

}  // namespace

extern "C" {

int orc_denoise_moments_lambda_frame(uint32_t width, uint32_t height, const orc_gradient_frame* f, orc_gradient_history* h,
                                     const trb_denoise_frame* in, const trb_denoise_gradient_params* params, const float* lam_s, float* rgbw,
                                     float* motion, uint32_t* history_length, float* variance, float* lam_px) {
    trb_denoise_params p;
    int squarings;
    GradPrm t;
    if (!gradient_params(params, p, squarings, t)) return TRB_INVALID_ARG;
    if (!f || !h || !rgbw || !lam_s || !frame_ok(in)) return TRB_INVALID_ARG;
    if (h->bound && (h->width != width || h->height != height)) return TRB_INVALID_ARG;
    moments_lambda(width, height, f, h, in, p, squarings, t, lam_s, rgbw, motion, history_length, variance, lam_px);
    h->gr_valid = false;
    return TRB_OK;
}

int orc_denoise_moments_gradient(orc_scene* s, orc_gradient_history* h, const trb_denoise_frame* in, const trb_denoise_gradient_params* params,
                                 uint32_t seed, float* rgbw, float* motion, uint32_t* history_length, float* variance, float* lam_px) {
    trb_denoise_params p;
    int squarings;
    GradPrm t;
    if (!gradient_params(params, p, squarings, t)) return TRB_INVALID_ARG;
    if (!s || s->active_camera < 0) { g_err = "update_frame must be called before a temporal denoise"; return TRB_INVALID_ARG; }
    if (!h || !rgbw || !frame_ok(in)) return TRB_INVALID_ARG;
    const uint32_t W = s->film.width, H = s->film.height;
    if (h->bound && (h->width != W || h->height != H)) return TRB_INVALID_ARG;
    orc_gradient_frame f;
    std::vector<float> inv, mat;
    scene_gradient_frame(s, f, inv, mat);
    std::vector<float> lam;
    scene_lambda(s, h, f, in->normal_w, in->nearest, t, lam);
    moments_lambda(W, H, &f, h, in, p, squarings, t, lam.data(), rgbw, motion, history_length, variance, lam_px);
    scene_record(s, h, f, seed);
    return TRB_OK;
}

}  // extern "C"
