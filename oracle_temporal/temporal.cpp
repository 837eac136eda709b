/* The parity oracle's temporal denoiser — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into
 * oracle/_build/liboracle_temporal.so and loaded by oracle_temporal/pytemporal.py.
 *
 * This translation unit is the detmath oracle (oracle/oracle.cpp) and the denoiser oracle (oracle_denoise/denoise.cpp), both included
 * whole and unchanged, plus the contract of include/trb.h "Temporal denoising" (DESIGN.md §4) restated over a CPU history:
 *   orc_denoise_temporal_frame  one call of the contract over an explicit frame (camera and instance matrices as arrays), so synthetic
 *                               frames need no scene
 *   orc_denoise_temporal        the same with the frame of an oracle scene after orc_scene_update_frame: the camera's cam_world and
 *                               every instance's transform at shutter-open, from the oracle's own matrices
 *   orc_denoise_history_create / _destroy / _reset
 * The history holds one set (the contract's ping-pong is a detail of the device). There is no object generation: a caller that
 * renumbers instances resets the history.
 */
#include "../oracle/oracle.cpp"
#include "../oracle_denoise/denoise.cpp"

/* One frame as the contract sees it: row-major 4x4 matrices, inv / mat n_instances x 16 floats */
struct orc_temporal_frame {
    float px_to_cam[16], cam_mat[16], cam_inv[16], scaling[3];
    uint32_t n_instances;
    const float* inv;
    const float* mat;
};

struct orc_denoise_history {
    bool has_prev = false, bound = false;
    uint32_t width = 0, height = 0;
    std::vector<float> ha, hb, n, z;   // 3, 3, 3 and 1 per pixel
    std::vector<uint32_t> inst, len;   // len 0: "none"
    float cam_inv[16] = {}, tan_fov = 0;
    uint32_t n_instances = 0;
    std::vector<float> mats;           // n_instances x 16
};

namespace {

M4 m4_of(const float* m) { M4 r; for (int k = 0; k < 16; ++k) r.m[k] = m[k]; return r; }

struct TemporalPrm { uint32_t max_history; float depth_tolerance, normal_threshold; };

bool temporal_params(const trb_denoise_temporal_params* params, trb_denoise_params& p, int& squarings, TemporalPrm& t) {
    if (!denoise_params(params ? &params->spatial : nullptr, p, squarings)) return false;
    t = TemporalPrm{8u, 0.05f, 0.9f};
    if (params) t = TemporalPrm{params->max_history, params->depth_tolerance, params->normal_threshold};
    return t.max_history >= 1 && t.max_history <= 255 && t.depth_tolerance > 0.0f && fin(t.depth_tolerance) && t.normal_threshold >= -1.0f &&
           t.normal_threshold <= 1.0f;
}

/* Steps 1-3 of the contract for the valid pixel P at (x, y) with instance id: the motion (left as it is without one), S, the
 * tap-weighted sums sa and sb of the history's ha and hb (3 each, not yet divided by S) and len_prev. oracle_moments/moments.cpp
 * calls it over a history whose ha holds ē and hb (mu1, mu2, 0). */
void temporal_gather(long W, long H, long x, long y, const Px& P, uint32_t id, const orc_temporal_frame* f, const orc_denoise_history* h,
                     const TemporalPrm& t, float& mx, float& my, float& S, float* sa, float* sb, uint32_t& len_prev) {
    if (!(h->has_prev && id < h->n_instances && id < f->n_instances && fin(P.z))) return;
    const M4 cam_mat = m4_of(f->cam_mat), px_to_cam = m4_of(f->px_to_cam), cam_inv_prev = m4_of(h->cam_inv);
    const float aspect = (float)W / (float)H;
    float X0 = -1.0f, X1 = 1.0f, Y0 = -1.0f / aspect, Y1 = 1.0f / aspect;
    if (aspect > 1.0f) { X0 = -aspect; X1 = aspect; Y0 = -1.0f; Y1 = 1.0f; }
    const V3 pc = Transform::mul_point(px_to_cam, V3((float)x + 0.5f, (float)y + 0.5f, 0.0f));
    const V3 dir = Transform::mul_vector(cam_mat, normalized(V3(f->scaling[0], f->scaling[1], f->scaling[2]) * pc));
    const V3 o = Transform::mul_point(cam_mat, V3(0.0f));
    const V3 pw(o.x + P.z * dir.x, o.y + P.z * dir.y, o.z + P.z * dir.z);
    const V3 po = Transform::mul_point(m4_of(f->inv + 16 * (size_t)id), pw);
    const V3 pp = Transform::mul_point(m4_of(h->mats.data() + 16 * (size_t)id), po);
    const V3 q = Transform::mul_point(cam_inv_prev, pp);
    if (!(q.z > 0.0f)) return;
    const float X = q.x / (q.z * h->tan_fov), Y = q.y / (q.z * h->tan_fov);
    const float rx = (X - X0) / (X1 - X0) * (float)W, ry = (Y - Y1) / (Y0 - Y1) * (float)H;
    mx = rx - ((float)x + 0.5f); my = ry - ((float)y + 0.5f);
    const float ql = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
    const float cx = rx - 0.5f, cy = ry - 0.5f, fx = std::floor(cx), fy = std::floor(cy), ax = cx - fx, ay = cy - fy;
    const int ox[4] = {0, 1, 0, 1}, oy[4] = {0, 0, 1, 1};
    const float wts[4] = {(1.0f - ax) * (1.0f - ay), ax * (1.0f - ay), (1.0f - ax) * ay, ax * ay};
    for (int k = 0; k < 4; ++k) {
        const float tx = fx + (float)ox[k], ty = fy + (float)oy[k];
        if (!(tx >= 0.0f && tx <= (float)W - 1.0f && ty >= 0.0f && ty <= (float)H - 1.0f)) continue;
        const long j = (long)ty * W + (long)tx;
        if (h->len[j] == 0 || h->inst[j] != id) continue;
        if (!(std::fabs(h->z[j] - ql) <= t.depth_tolerance * ql)) continue;
        const float* tn = &h->n[3 * j];
        const bool t_nrm = tn[0] != 0.0f || tn[1] != 0.0f || tn[2] != 0.0f;
        if (t_nrm != P.has_n) continue;
        if (P.has_n && !(tn[0] * P.n[0] + tn[1] * P.n[1] + tn[2] * P.n[2] >= t.normal_threshold)) continue;
        const float w = wts[k];
        S = S + w;
        for (int c = 0; c < 3; ++c) {
            sa[c] = sa[c] + w * h->ha[3 * j + c];
            sb[c] = sb[c] + w * h->hb[3 * j + c];
        }
        if (w > 0.0f && h->len[j] > len_prev) len_prev = h->len[j];
    }
}

/* The frame of an oracle scene after orc_scene_update_frame: the camera's cam_world and every instance's transform at shutter-open,
 * from the oracle's own matrices (inv and mat hold the instances' matrices, which f points at); false without a frame */
bool scene_frame(orc_scene* s, orc_temporal_frame& f, std::vector<float>& inv, std::vector<float>& mat) {
    if (!s || s->active_camera < 0) { g_err = "update_frame must be called before a temporal denoise"; return false; }
    const Camera& cam = s->cameras[s->active_camera];
    const Transform cw = cam.cam_world.transform(cam.shutter_open);
    const size_t n = s->geom.instances.size();
    inv.assign(16 * n, 0.0f); mat.assign(16 * n, 0.0f);
    for (size_t k = 0; k < n; ++k) {
        const Transform t = s->geom.instances[k].transform.transform(cam.shutter_open);
        std::memcpy(&mat[16 * k], t.mat.m, 64); std::memcpy(&inv[16 * k], t.inv.m, 64);
    }
    std::memcpy(f.px_to_cam, cam.px_to_cam.mat.m, 64);
    std::memcpy(f.cam_mat, cw.mat.m, 64);
    std::memcpy(f.cam_inv, cw.inv.m, 64);
    f.scaling[0] = cam.scaling.x; f.scaling[1] = cam.scaling.y; f.scaling[2] = cam.scaling.z;
    f.n_instances = (uint32_t)n; f.inv = inv.data(); f.mat = mat.data();
    return true;
}

}  // namespace

extern "C" {

int orc_denoise_history_create(orc_denoise_history** out) { *out = new orc_denoise_history(); return TRB_OK; }
int orc_denoise_history_destroy(orc_denoise_history* h) { delete h; return TRB_OK; }
int orc_denoise_history_reset(orc_denoise_history* h) { h->has_prev = false; h->bound = false; return TRB_OK; }

int orc_denoise_temporal_frame(uint32_t width, uint32_t height, const orc_temporal_frame* f, orc_denoise_history* h, const trb_denoise_input* in,
                               const trb_denoise_temporal_params* params, float* rgbw, float* motion, uint32_t* history_length) {
    trb_denoise_params p;
    int squarings;
    TemporalPrm t;
    if (!temporal_params(params, p, squarings, t)) return TRB_INVALID_ARG;
    if (!f || !h || !in || !rgbw || !in->colour_a || !in->colour_b || !in->albedo_w || !in->normal_w || !in->nearest) return TRB_INVALID_ARG;
    if (h->bound && (h->width != width || h->height != height)) return TRB_INVALID_ARG;
    const long W = width, H = height, N = W * H;
    std::vector<Px> px;
    std::vector<float> e, v, ea, eb;
    denoise_prepare(W, H, in, px, e, v, &ea, &eb);
    const float qnan = dm_from_bits(0x7fffffffu);
    std::vector<float> nha(N * 3), nhb(N * 3), nn(N * 3), nz(N);
    std::vector<uint32_t> ninst(N), nlen(N, 0u);
    for (long y = 0; y < H; ++y)
        for (long x = 0; x < W; ++x) {
            const long i = y * W + x;
            Px& P = px[i];
            float mx = qnan, my = qnan;
            uint32_t np = 0;
            if (P.valid) {
                const uint32_t id = (uint32_t)in->nearest[i];
                float S = 0.0f, sa[3] = {0, 0, 0}, sb[3] = {0, 0, 0};
                uint32_t len_prev = 0;
                /* 1-3 */
                temporal_gather(W, H, x, y, P, id, f, h, t, mx, my, S, sa, sb, len_prev);
                /* 4 */
                np = S > 0.0f ? std::min(len_prev + 1, t.max_history) : 1u;
                if (np > 1) {
                    const float alpha = 1.0f / (float)np, beta = 1.0f - alpha;
                    for (int c = 0; c < 3; ++c) {
                        const float Ha = sa[c] / S, Hb = sb[c] / S;
                        e[3 * i + c] = alpha * e[3 * i + c] + beta * ((Ha + Hb) * 0.5f);
                        ea[3 * i + c] = alpha * ea[3 * i + c] + beta * Ha;
                        eb[3 * i + c] = alpha * eb[3 * i + c] + beta * Hb;
                    }
                    const float dl = lum(&ea[3 * i]) - lum(&eb[3 * i]);
                    v[i] = dl * dl * 0.25f;
                }
                /* 6 */
                if (fin(P.z)) {
                    for (int c = 0; c < 3; ++c) { nha[3 * i + c] = ea[3 * i + c]; nhb[3 * i + c] = eb[3 * i + c]; nn[3 * i + c] = P.n[c]; }
                    nz[i] = P.z; ninst[i] = id; nlen[i] = np;
                }
            }
            if (motion) { motion[2 * i] = std::isnan(mx) ? qnan : mx; motion[2 * i + 1] = std::isnan(my) ? qnan : my; }
            if (history_length) history_length[i] = np;
        }
    /* 5 */
    denoise_filter(W, H, p, squarings, px, std::move(e), std::move(v), rgbw);
    h->ha.swap(nha); h->hb.swap(nhb); h->n.swap(nn); h->z.swap(nz); h->inst.swap(ninst); h->len.swap(nlen);
    std::memcpy(h->cam_inv, f->cam_inv, 64);
    h->tan_fov = f->scaling[0];
    h->n_instances = f->n_instances;
    h->mats.assign(f->mat, f->mat + 16 * (size_t)f->n_instances);
    h->has_prev = true; h->bound = true; h->width = width; h->height = height;
    return TRB_OK;
}

int orc_denoise_temporal(orc_scene* s, orc_denoise_history* h, const trb_denoise_input* in, const trb_denoise_temporal_params* params,
                         float* rgbw, float* motion, uint32_t* history_length) {
    orc_temporal_frame f;
    std::vector<float> inv, mat;
    if (!scene_frame(s, f, inv, mat)) return TRB_INVALID_ARG;
    return orc_denoise_temporal_frame(s->film.width, s->film.height, &f, h, in, params, rgbw, motion, history_length);
}

}  // extern "C"
