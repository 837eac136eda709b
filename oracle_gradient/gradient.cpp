/* The parity oracle's temporal gradients — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into
 * oracle/_build/liboracle_gradient.so and loaded by oracle_gradient/pygradient.py.
 *
 * This translation unit is the ray-query oracle (oracle_queries/queries.cpp, which includes oracle/oracle.cpp) and the denoiser oracle
 * (oracle_denoise/denoise.cpp), both included whole and unchanged, plus the contract of include/trb.h "Temporal gradients" (DESIGN.md
 * §4) restated over a CPU history, on top of "Temporal denoising" restated once more with the lambda of step 3:
 *   orc_gradient_lambda_frame        steps 1-2 over an explicit frame and caller records, with the re-shaded luminances given by the
 *                                    caller (so synthetic frames need no scene): the winners, (delta, m) and lambda per stratum
 *   orc_denoise_temporal_lambda_frame "Temporal denoising" over an explicit frame with a caller lambda per stratum (step 3)
 *   orc_denoise_temporal_gradient    steps 1-4 with an oracle scene after orc_scene_update_frame: its camera rays, ray-query records
 *                                    and trb_illumination, then the blend
 *   orc_gradient_history_create / _destroy / _reset
 * The history holds one set of pixels and records (the ping-pong is a detail of the device). There is no object generation: a caller
 * that renumbers instances resets the history.
 */
#include "../oracle_queries/queries.cpp"
#include "../oracle_denoise/denoise.cpp"

/* One frame: row-major 4x4 matrices, inv / mat n_instances x 16 floats (oracle_temporal's orc_temporal_frame plus shutter_open) */
struct orc_gradient_frame {
    float px_to_cam[16], cam_mat[16], cam_inv[16], scaling[3];
    uint32_t n_instances;
    const float* inv;
    const float* mat;
    float shutter_open;
};

/* A gradient record as the header states it */
struct orc_gradient_record {
    float p_o[3];
    uint32_t inst;     /* TRB_MISS: none */
    float o[3], time;
    float d[3];
    uint32_t key;
    float lum;
    uint32_t pad[3];
};

struct orc_gradient_history {
    bool has_prev = false, bound = false;
    uint32_t width = 0, height = 0;
    std::vector<float> ha, hb, n, z;
    std::vector<uint32_t> inst, len;
    float cam_inv[16] = {}, tan_fov = 0;
    uint32_t n_instances = 0;
    std::vector<float> mats;
    bool gr_valid = false;
    std::vector<orc_gradient_record> rec;
    uint32_t gr_seed = 0;
    float gr_shutter_open = 0, gr_cam_mat[16] = {};
};

namespace {

M4 gm4(const float* m) { M4 r; for (int k = 0; k < 16; ++k) r.m[k] = m[k]; return r; }
float glum(float r, float g, float b) { return 0.2126f * r + 0.7152f * g + 0.0722f * b; }

struct GradPrm { uint32_t max_history; float depth_tolerance, normal_threshold; uint32_t iterations; };

bool gradient_params(const trb_denoise_gradient_params* params, trb_denoise_params& p, int& squarings, GradPrm& t) {
    if (!denoise_params(params ? &params->temporal.spatial : nullptr, p, squarings)) return false;
    t = GradPrm{8u, 0.05f, 0.9f, 3u};
    if (params) t = GradPrm{params->temporal.max_history, params->temporal.depth_tolerance, params->temporal.normal_threshold, params->iterations};
    return t.max_history >= 1 && t.max_history <= 255 && t.depth_tolerance > 0.0f && fin(t.depth_tolerance) && t.normal_threshold >= -1.0f &&
           t.normal_threshold <= 1.0f && t.iterations <= 6;
}

void window(uint32_t W, uint32_t H, float& X0, float& X1, float& Y0, float& Y1) {
    const float aspect = (float)W / (float)H;
    X0 = -1.0f; X1 = 1.0f; Y0 = -1.0f / aspect; Y1 = 1.0f / aspect;
    if (aspect > 1.0f) { X0 = -aspect; X1 = aspect; Y0 = -1.0f; Y1 = 1.0f; }
}

/* Step 1's forward projection and collision winners: slot[t] = min over kept records j of (dist bits << 32 | j), ~0 if none */
void project(uint32_t W, uint32_t H, const orc_gradient_frame* f, uint32_t n_prev, const orc_gradient_record* rec, size_t S,
             const uint64_t* nearest, float depth_tolerance, std::vector<uint64_t>& slot) {
    const uint32_t gw = (W + 2) / 3;
    float X0, X1, Y0, Y1;
    window(W, H, X0, X1, Y0, Y1);
    slot.assign(S, ~0ull);
    const M4 cam_inv = gm4(f->cam_inv), cam_mat = gm4(f->cam_mat);
    const float tan = f->scaling[0];
    for (size_t j = 0; j < S; ++j) {
        const orc_gradient_record& r = rec[j];
        if (r.inst == TRB_MISS || r.inst >= f->n_instances || r.inst >= n_prev) continue;
        const V3 pw = Transform::mul_point(gm4(f->mat + 16 * (size_t)r.inst), V3(r.p_o[0], r.p_o[1], r.p_o[2]));
        const V3 q = Transform::mul_point(cam_inv, pw);
        if (!(q.z > 0.0f)) continue;
        const float X = q.x / (q.z * tan), Y = q.y / (q.z * tan);
        const float rx = (X - X0) / (X1 - X0) * (float)W, ry = (Y - Y1) / (Y0 - Y1) * (float)H;
        if (!(rx >= 0.0f && rx < (float)W && ry >= 0.0f && ry < (float)H)) continue;
        const uint32_t px = (uint32_t)rx, py = (uint32_t)ry;
        if (px >= W || py >= H) continue;
        const uint64_t key = nearest[(size_t)py * W + px];
        if ((uint32_t)key != r.inst) continue;
        const float z = dm_from_bits((uint32_t)(key >> 32));
        const V3 o = Transform::mul_point(cam_mat, V3(0.0f));
        const float vx = pw.x - o.x, vy = pw.y - o.y, vz = pw.z - o.z;
        const float dist = std::sqrt(vx * vx + vy * vy + vz * vz);
        if (!(std::fabs(z - dist) <= depth_tolerance * z)) continue;
        const size_t t = (size_t)(py / 3) * gw + px / 3;
        uint32_t db;
        std::memcpy(&db, &dist, 4);
        slot[t] = std::min<uint64_t>(slot[t], ((uint64_t)db << 32) | j);
    }
}

/* Step 1's illumination ray of the winner j of stratum t */
trb_illum_ray reshade_ray(const orc_gradient_frame* f, const orc_gradient_record& r, const float* mat_prev, bool cam_same, float dt) {
    trb_illum_ray q{};
    const float* mc = f->mat + 16 * (size_t)r.inst;
    const float* mp = mat_prev + 16 * (size_t)r.inst;
    const bool same = cam_same && std::memcmp(mc, mp, 64) == 0;
    if (same) {
        for (int k = 0; k < 3; ++k) { q.o[k] = r.o[k]; q.d[k] = r.d[k]; }
    } else {
        const V3 pw = Transform::mul_point(gm4(mc), V3(r.p_o[0], r.p_o[1], r.p_o[2]));
        const V3 o = Transform::mul_point(gm4(f->cam_mat), V3(0.0f));
        const V3 d = normalized(V3(pw.x - o.x, pw.y - o.y, pw.z - o.z));
        q.o[0] = o.x; q.o[1] = o.y; q.o[2] = o.z; q.d[0] = d.x; q.d[1] = d.y; q.d[2] = d.z;
    }
    q.min_t = 0.0f; q.max_t = F32_INF; q.time = r.time + dt; q.key = r.key; q.sample = 0;
    return q;
}

/* Step 1's (delta, m, c) and step 2's reconstruction: lambda per stratum */
void reconstruct(uint32_t W, uint32_t H, const std::vector<uint64_t>& slot, const orc_gradient_record* rec, const float* l_cur,
                 const float* normal_w, const uint64_t* nearest, float normal_threshold, uint32_t iterations, float* dm_out, float* lam) {
    const uint32_t gw = (W + 2) / 3, gh = (H + 2) / 3, S = gw * gh;
    std::vector<float> d(S), m(S), c(S), n(3 * S);
    std::vector<uint32_t> id(S);
    for (uint32_t t = 0; t < S; ++t) {
        const uint32_t sx = t % gw, sy = t / gw;
        const size_t p = (size_t)std::min(sy * 3 + 1, H - 1) * W + std::min(sx * 3 + 1, W - 1);
        const float* nw = normal_w + 4 * p;
        const float m0 = nw[0] / nw[3], m1 = nw[1] / nw[3], m2 = nw[2] / nw[3];
        const float l2 = m0 * m0 + m1 * m1 + m2 * m2;
        n[3 * t] = n[3 * t + 1] = n[3 * t + 2] = 0.0f;
        if (fin(l2) && l2 != 0.0f) {
            const float l = std::sqrt(l2);
            n[3 * t] = m0 / l; n[3 * t + 1] = m1 / l; n[3 * t + 2] = m2 / l;
        }
        id[t] = (uint32_t)nearest[p];
        d[t] = m[t] = c[t] = 0.0f;
        if (slot[t] != ~0ull) {
            const float lc = l_cur[t], lp = rec[(uint32_t)slot[t]].lum;
            d[t] = lc - lp; m[t] = lc > lp ? lc : lp; c[t] = 1.0f;
        }
    }
    const float h[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    for (uint32_t it = 0; it < iterations; ++it) {
        const int s = 1 << it;
        std::vector<float> d2(S), m2(S), c2(S);
        for (uint32_t t = 0; t < S; ++t) {
            const int x = (int)(t % gw), y = (int)(t / gw);
            const bool p_nrm = n[3 * t] != 0.0f || n[3 * t + 1] != 0.0f || n[3 * t + 2] != 0.0f;
            float Wt = 0.0f, sd = 0.0f, sm = 0.0f;
            for (int dy = -2; dy <= 2; ++dy) {
                const int qy = y + s * dy;
                if (qy < 0 || qy >= (int)gh) continue;
                for (int dx = -2; dx <= 2; ++dx) {
                    const int qx = x + s * dx;
                    if (qx < 0 || qx >= (int)gw) continue;
                    const uint32_t q = (uint32_t)qy * gw + (uint32_t)qx;
                    if (!(c[q] > 0.0f)) continue;
                    if (q != t) {
                        if (id[q] != id[t]) continue;
                        const bool q_nrm = n[3 * q] != 0.0f || n[3 * q + 1] != 0.0f || n[3 * q + 2] != 0.0f;
                        if (q_nrm != p_nrm) continue;
                        if (p_nrm && !(n[3 * t] * n[3 * q] + n[3 * t + 1] * n[3 * q + 1] + n[3 * t + 2] * n[3 * q + 2] >= normal_threshold)) continue;
                    }
                    const float w = h[dx + 2] * h[dy + 2];
                    Wt = Wt + w;
                    sd = sd + w * d[q];
                    sm = sm + w * m[q];
                }
            }
            d2[t] = m2[t] = c2[t] = 0.0f;
            if (Wt > 0.0f) { d2[t] = sd / Wt; m2[t] = sm / Wt; c2[t] = 1.0f; }
        }
        d.swap(d2); m.swap(m2); c.swap(c2);
    }
    for (uint32_t t = 0; t < S; ++t) {
        lam[t] = c[t] > 0.0f && m[t] > 0.0f ? std::min(1.0f, std::fabs(d[t]) / m[t]) : 0.0f;
        if (dm_out) { dm_out[3 * t] = d[t]; dm_out[3 * t + 1] = m[t]; dm_out[3 * t + 2] = c[t]; }
    }
}

/* Steps 1-3 of "Temporal denoising" for the valid pixel P at (x, y) with instance id: the motion (left as it is without one), S, the
 * tap-weighted sums sa and sb of the history's ha and hb (3 each, not yet divided by S) and len_prev. oracle_moment_gradient calls it
 * over a history whose ha holds ē and hb (mu1, mu2, 0). */
void gradient_gather(long W, long H, long x, long y, const Px& P, uint32_t id, const orc_gradient_frame* f, const orc_gradient_history* h,
                     const GradPrm& t, float& mx, float& my, float& S, float* sa, float* sb, uint32_t& len_prev) {
    if (!(h->has_prev && id < h->n_instances && id < f->n_instances && fin(P.z))) return;
    const M4 cam_mat = gm4(f->cam_mat), px_to_cam = gm4(f->px_to_cam), cam_inv_prev = gm4(h->cam_inv);
    float X0, X1, Y0, Y1;
    window((uint32_t)W, (uint32_t)H, X0, X1, Y0, Y1);
    const V3 pc = Transform::mul_point(px_to_cam, V3((float)x + 0.5f, (float)y + 0.5f, 0.0f));
    const V3 dir = Transform::mul_vector(cam_mat, normalized(V3(f->scaling[0], f->scaling[1], f->scaling[2]) * pc));
    const V3 o = Transform::mul_point(cam_mat, V3(0.0f));
    const V3 pw(o.x + P.z * dir.x, o.y + P.z * dir.y, o.z + P.z * dir.z);
    const V3 po = Transform::mul_point(gm4(f->inv + 16 * (size_t)id), pw);
    const V3 pp = Transform::mul_point(gm4(h->mats.data() + 16 * (size_t)id), po);
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

/* "Temporal denoising" with step 3's lambda (lam_s per stratum; lam_px per pixel out) */
void temporal_lambda(uint32_t width, uint32_t height, const orc_gradient_frame* f, orc_gradient_history* h, const trb_denoise_input* in,
                     const trb_denoise_params& p, int squarings, const GradPrm& t, const float* lam_s, float* rgbw, float* motion,
                     uint32_t* history_length, float* lam_px) {
    const long W = width, H = height, N = W * H, gw = (W + 2) / 3;
    std::vector<Px> px;
    std::vector<float> e, v, ea, eb;
    denoise_prepare(W, H, in, px, e, v, &ea, &eb);
    const float qnan = dm_from_bits(0x7fffffffu);
    std::vector<float> nha(N * 3), nhb(N * 3), nn(N * 3), nz(N);
    std::vector<uint32_t> ninst(N), nlen(N, 0u);
    for (long y = 0; y < H; ++y)
        for (long x = 0; x < W; ++x) {
            const long i = y * W + x;
            const float lam = lam_s[(y / 3) * gw + x / 3];
            if (lam_px) lam_px[i] = lam;
            Px& P = px[i];
            float mx = qnan, my = qnan;
            uint32_t np = 0;
            if (P.valid) {
                const uint32_t id = (uint32_t)in->nearest[i];
                float S = 0.0f, sa[3] = {0, 0, 0}, sb[3] = {0, 0, 0};
                uint32_t len_prev = 0;
                gradient_gather(W, H, x, y, P, id, f, h, t, mx, my, S, sa, sb, len_prev);
                np = 1u;
                if (S > 0.0f) np = std::min((uint32_t)std::floor((1.0f - lam) * (float)len_prev) + 1u, t.max_history);
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
                if (fin(P.z)) {
                    for (int c = 0; c < 3; ++c) { nha[3 * i + c] = ea[3 * i + c]; nhb[3 * i + c] = eb[3 * i + c]; nn[3 * i + c] = P.n[c]; }
                    nz[i] = P.z; ninst[i] = id; nlen[i] = np;
                }
            }
            if (motion) { motion[2 * i] = std::isnan(mx) ? qnan : mx; motion[2 * i + 1] = std::isnan(my) ? qnan : my; }
            if (history_length) history_length[i] = np;
        }
    denoise_filter(W, H, p, squarings, px, std::move(e), std::move(v), rgbw);
    h->ha.swap(nha); h->hb.swap(nhb); h->n.swap(nn); h->z.swap(nz); h->inst.swap(ninst); h->len.swap(nlen);
    std::memcpy(h->cam_inv, f->cam_inv, 64);
    h->tan_fov = f->scaling[0];
    h->n_instances = f->n_instances;
    h->mats.assign(f->mat, f->mat + 16 * (size_t)f->n_instances);
    h->has_prev = true; h->bound = true; h->width = width; h->height = height;
}

}  // namespace

namespace {

/* The frame of an oracle scene after orc_scene_update_frame (the camera's active one): cam_world and every instance's transform at
 * shutter-open, from the oracle's own matrices (inv and mat hold the instances' matrices, which f points at) */
void scene_gradient_frame(orc_scene* s, orc_gradient_frame& f, std::vector<float>& inv, std::vector<float>& mat) {
    const Camera& cam = s->cameras[s->active_camera];
    const Transform cw = cam.cam_world.transform(cam.shutter_open);
    const size_t n = s->geom.instances.size();
    inv.assign(16 * n, 0.0f); mat.assign(16 * n, 0.0f);
    for (size_t k = 0; k < n; ++k) {
        const Transform tr = s->geom.instances[k].transform.transform(cam.shutter_open);
        std::memcpy(&mat[16 * k], tr.mat.m, 64); std::memcpy(&inv[16 * k], tr.inv.m, 64);
    }
    std::memcpy(f.px_to_cam, cam.px_to_cam.mat.m, 64);
    std::memcpy(f.cam_mat, cw.mat.m, 64);
    std::memcpy(f.cam_inv, cw.inv.m, 64);
    f.scaling[0] = cam.scaling.x; f.scaling[1] = cam.scaling.y; f.scaling[2] = cam.scaling.z;
    f.n_instances = (uint32_t)n; f.inv = inv.data(); f.mat = mat.data(); f.shutter_open = cam.shutter_open;
}

/* Steps 1-2 with the scene: the history's records re-shaded by orc_illumination, lambda per stratum (0 without valid records) */
void scene_lambda(orc_scene* s, const orc_gradient_history* h, const orc_gradient_frame& f, const float* normal_w, const uint64_t* nearest,
                  const GradPrm& t, std::vector<float>& lam) {
    const uint32_t W = s->film.width, H = s->film.height, S = ((W + 2) / 3) * ((H + 2) / 3);
    lam.assign(S, 0.0f);
    if (h->has_prev && h->gr_valid) {
        std::vector<uint64_t> slot;
        project(W, H, &f, h->n_instances, h->rec.data(), S, nearest, t.depth_tolerance, slot);
        const bool cam_same = std::memcmp(h->gr_cam_mat, f.cam_mat, 64) == 0;
        std::vector<trb_illum_ray> rays;
        std::vector<uint32_t> tgt;
        for (uint32_t k = 0; k < S; ++k)
            if (slot[k] != ~0ull) {
                rays.push_back(reshade_ray(&f, h->rec[(uint32_t)slot[k]], h->mats.data(), cam_same, f.shutter_open - h->gr_shutter_open));
                tgt.push_back(k);
            }
        std::vector<float> rgb(3 * rays.size()), lc(S, 0.0f);
        if (!rays.empty()) orc_illumination(s, rays.size(), rays.data(), 1, h->gr_seed, rgb.data(), 1, nullptr);
        for (size_t k = 0; k < rays.size(); ++k) lc[tgt[k]] = glum(rgb[3 * k], rgb[3 * k + 1], rgb[3 * k + 2]);
        reconstruct(W, H, slot, h->rec.data(), lc.data(), normal_w, nearest, t.normal_threshold, t.iterations, nullptr, lam.data());
    } else {
        std::vector<uint64_t> slot(S, ~0ull);
        std::vector<float> lc(S, 0.0f);
        reconstruct(W, H, slot, nullptr, lc.data(), normal_w, nearest, t.normal_threshold, t.iterations, nullptr, lam.data());
    }
}

/* Step 4 with the scene: this frame's samples at `seed` into the history's records, which become valid */
void scene_record(orc_scene* s, orc_gradient_history* h, const orc_gradient_frame& f, uint32_t seed) {
    const uint32_t W = s->film.width, H = s->film.height, gw = (W + 2) / 3, gh = (H + 2) / 3, S = gw * gh;
    const Camera& cam = s->cameras[s->active_camera];
    std::vector<trb_query_ray> q(S);
    std::vector<trb_illum_ray> il(S);
    for (uint32_t k = 0; k < S; ++k) {
        const uint32_t sx = k % gw, sy = k / gw, cwd = std::min(3u, W - 3 * sx), chd = std::min(3u, H - 3 * sy);
        const uint32_t pick = dm_rng(seed, k, 0xfffffffeu, 0u) % (cwd * chd);
        const uint32_t px = 3 * sx + pick % cwd, py = 3 * sy + pick / cwd, pixel = py * W + px;
        const PixelStreams st = pixel_streams(seed, pixel);
        const uint32_t ip = dm_permute(0, 1, st.kpos);
        const float fx = van_der_corput(ip, st.scr0) + (float)px, fy = sobol(ip, st.scr1) + (float)py;
        const float tm = van_der_corput(dm_permute(0, 1, st.ktime), st.scrt);
        const Ray r = cam.generate_ray(fx, fy, tm);
        q[k] = trb_query_ray{{r.o.x, r.o.y, r.o.z}, {r.d.x, r.d.y, r.d.z}, r.min_t, r.max_t, r.time, {0, 0, 0}};
        il[k] = trb_illum_ray{{r.o.x, r.o.y, r.o.z}, {r.d.x, r.d.y, r.d.z}, r.min_t, r.max_t, r.time, pixel, 0, 0};
    }
    std::vector<trb_intersection> hits(S);
    std::vector<float> rgb(3 * (size_t)S);
    orc_intersect_records(s, S, q.data(), hits.data(), nullptr);
    orc_illumination(s, S, il.data(), 1, seed, rgb.data(), 1, nullptr);
    h->rec.assign(S, orc_gradient_record{});
    for (uint32_t k = 0; k < S; ++k) {
        orc_gradient_record& r = h->rec[k];
        r.inst = hits[k].inst;
        if (r.inst == TRB_MISS) continue;
        const V3 po = Transform::mul_point(gm4(f.inv + 16 * (size_t)r.inst), V3(hits[k].p[0], hits[k].p[1], hits[k].p[2]));
        r.p_o[0] = po.x; r.p_o[1] = po.y; r.p_o[2] = po.z;
        for (int c = 0; c < 3; ++c) { r.o[c] = il[k].o[c]; r.d[c] = il[k].d[c]; }
        r.time = il[k].time; r.key = il[k].key;
        r.lum = glum(rgb[3 * k], rgb[3 * k + 1], rgb[3 * k + 2]);
    }
    h->gr_valid = true; h->gr_seed = seed; h->gr_shutter_open = f.shutter_open;
    std::memcpy(h->gr_cam_mat, f.cam_mat, 64);
}

}  // namespace

extern "C" {

int orc_gradient_history_create(orc_gradient_history** out) { *out = new orc_gradient_history(); return TRB_OK; }
int orc_gradient_history_destroy(orc_gradient_history* h) { delete h; return TRB_OK; }
int orc_gradient_history_reset(orc_gradient_history* h) { h->has_prev = false; h->bound = false; h->gr_valid = false; return TRB_OK; }

/* Steps 1-2 over caller records (S of them, the previous frame's snapshot being mat_prev / n_prev / cam_mat_prev / shutter_open_prev)
 * and caller re-shaded luminances l_cur per TARGET stratum: writes slot (S uint64), the rays step 1 would trace (S trb_illum_ray, zero
 * where no winner), dm (S x (delta, m, c) after reconstruction) and lambda (S floats). */
int orc_gradient_lambda_frame(uint32_t width, uint32_t height, const orc_gradient_frame* f, const orc_gradient_record* rec, uint32_t n_prev,
                              const float* mat_prev, const float* cam_mat_prev, float shutter_open_prev, const float* l_cur, const float* normal_w,
                              const uint64_t* nearest, float depth_tolerance, float normal_threshold, uint32_t iterations, uint64_t* slot_out,
                              trb_illum_ray* rays, float* dm, float* lambda) {
    if (!f || !rec || !l_cur || !normal_w || !nearest || !lambda || iterations > 6) return TRB_INVALID_ARG;
    const size_t S = (size_t)((width + 2) / 3) * ((height + 2) / 3);
    std::vector<uint64_t> slot;
    project(width, height, f, n_prev, rec, S, nearest, depth_tolerance, slot);
    const bool cam_same = std::memcmp(cam_mat_prev, f->cam_mat, 64) == 0;
    for (size_t t = 0; t < S; ++t) {
        if (slot_out) slot_out[t] = slot[t];
        if (rays) rays[t] = slot[t] == ~0ull ? trb_illum_ray{} : reshade_ray(f, rec[(uint32_t)slot[t]], mat_prev, cam_same, f->shutter_open - shutter_open_prev);
    }
    reconstruct(width, height, slot, rec, l_cur, normal_w, nearest, normal_threshold, iterations, dm, lambda);
    return TRB_OK;
}

/* "Temporal denoising" with step 3 over an explicit frame and a caller lambda per stratum; the records are not touched */
int orc_denoise_temporal_lambda_frame(uint32_t width, uint32_t height, const orc_gradient_frame* f, orc_gradient_history* h, const trb_denoise_input* in,
                                      const trb_denoise_gradient_params* params, const float* lam_s, float* rgbw, float* motion,
                                      uint32_t* history_length, float* lam_px) {
    trb_denoise_params p;
    int squarings;
    GradPrm t;
    if (!gradient_params(params, p, squarings, t)) return TRB_INVALID_ARG;
    if (!f || !h || !in || !rgbw || !lam_s || !in->colour_a || !in->colour_b || !in->albedo_w || !in->normal_w || !in->nearest) return TRB_INVALID_ARG;
    if (h->bound && (h->width != width || h->height != height)) return TRB_INVALID_ARG;
    temporal_lambda(width, height, f, h, in, p, squarings, t, lam_s, rgbw, motion, history_length, lam_px);
    h->gr_valid = false;
    return TRB_OK;
}

int orc_denoise_temporal_gradient(orc_scene* s, orc_gradient_history* h, const trb_denoise_input* in, const trb_denoise_gradient_params* params,
                                  uint32_t seed, float* rgbw, float* motion, uint32_t* history_length, float* lam_px) {
    trb_denoise_params p;
    int squarings;
    GradPrm t;
    if (!gradient_params(params, p, squarings, t)) return TRB_INVALID_ARG;
    if (!s || s->active_camera < 0) { g_err = "update_frame must be called before a temporal denoise"; return TRB_INVALID_ARG; }
    const uint32_t W = s->film.width, H = s->film.height;
    if (h->bound && (h->width != W || h->height != H)) return TRB_INVALID_ARG;
    orc_gradient_frame f;
    std::vector<float> inv, mat;
    scene_gradient_frame(s, f, inv, mat);
    std::vector<float> lam;
    scene_lambda(s, h, f, in->normal_w, in->nearest, t, lam);
    temporal_lambda(W, H, &f, h, in, p, squarings, t, lam.data(), rgbw, motion, history_length, lam_px);
    scene_record(s, h, f, seed);
    return TRB_OK;
}

}  // extern "C"
