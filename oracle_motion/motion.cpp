/* The motion-vector oracle — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into oracle/_build/liboracle_motion.so and
 * loaded by oracle_motion/pymotion.py.
 *
 * This translation unit is the ray-query oracle (oracle_queries/queries.cpp, included whole and unchanged) plus include/trb.h
 * "Motion vectors" restated over the oracle's own camera (Camera::generate_ray, the ray and its time), Scene::intersect (the hit's
 * instance and world point, as orc_intersect_records returns them) and AnimatedTransform::transform:
 *   orc_motion_samples  one trb_motion_sample per camera sample of a LowDiscrepancy render, in trb_camera_rays' order
 *   orc_motion_at       one per caller camera sample (raster x, y and time sample tm in [0, 1)), e.g. the slots an Adaptive render took
 * Both take the frame's (start, end) as trb_scene_update_frame was given them: an animated fov is sampled at their clamped midpoint.
 */
#include "../oracle_queries/queries.cpp"

namespace {
struct MotionFrame {
    const Camera* cam;
    float tan_now, tan_then, dt;
    float x0, x1, y0, y1, w, h;
};

/* tan(fov / 2) of the active camera for the frame (start, end) shifted by dt (Camera::update_frame's sampling) */
float motion_tan(const Camera& c, float start, float end, float dt) {
    float fov = c.fov;
    if (c.fov_animated) {
        float lo = c.fov_knots[c.fov_degree], hi = c.fov_knots[c.fov_knots.size() - 1 - c.fov_degree];
        float t = (start + end) / 2.0f + dt;
        t = t < lo ? lo : (t > hi ? hi : t);
        fov = c.fov_spline_point(t);
    }
    return tanf(to_radians(fov) / 2.0f);
}

MotionFrame motion_frame(const orc_scene* s, float dt, float start, float end) {
    MotionFrame f;
    f.cam = &s->cameras[s->active_camera];
    f.tan_now = motion_tan(*f.cam, start, end, 0.0f);
    f.tan_then = motion_tan(*f.cam, start, end, dt);
    f.dt = dt;
    const float aspect = (float)s->film.width / (float)s->film.height; /* Camera::new's screen window */
    if (aspect > 1.0f) { f.x0 = -aspect; f.x1 = aspect; f.y0 = -1.0f; f.y1 = 1.0f; }
    else { f.x0 = -1.0f; f.x1 = 1.0f; f.y0 = -1.0f / aspect; f.y1 = 1.0f / aspect; }
    f.w = (float)s->film.width; f.h = (float)s->film.height;
    return f;
}

/* step 3: r(tau, x); false unless x is in front of the camera */
bool raster_of(const MotionFrame& f, float tau, float tan_fov, V3 x, float& rx, float& ry) {
    const V3 q = Transform::mul_point(f.cam->cam_world.transform(tau).inv, x);
    const float X = q.x / (q.z * tan_fov), Y = q.y / (q.z * tan_fov);
    rx = (X - f.x0) / (f.x1 - f.x0) * f.w;
    ry = (Y - f.y1) / (f.y0 - f.y1) * f.h;
    return q.z > 0.0f;
}

/* steps 1-5 for the camera sample (sx, sy, tm) */
trb_motion_sample motion_of(const orc_scene* s, const MotionFrame& f, float sx, float sy, float tm) {
    trb_motion_sample o = {0.0f, 0.0f, 0.0f, 0u};
    Ray ray = f.cam->generate_ray(sx, sy, tm);
    const float t = ray.time;
    Hit hit;
    Counters cnt;
    if (!s->geom.intersect(ray, hit, cnt)) return o;
    const Transform M = s->geom.xf(hit.inst, t); /* the transform the trace used */
    const V3 po = Transform::mul_point(M.inv, hit.dg.p);
    const V3 p_now = M.point(po);
    const V3 p_then = s->geom.is_static[hit.inst] ? p_now : s->geom.instances[hit.inst].transform.transform(t + f.dt).point(po);
    float x0, y0, x1, y1;
    const bool v0 = raster_of(f, t, f.tan_now, p_now, x0, y0);
    const bool v1 = raster_of(f, t + f.dt, f.tan_then, p_then, x1, y1);
    if (v0 && v1) { o.dx = x1 - x0; o.dy = y1 - y0; o.valid = 1.0f; }
    return o;
}
} // namespace

extern "C" {

int orc_motion_samples(orc_scene* s, const trb_render_cfg* cfg, size_t n, float dt, float start, float end, trb_motion_sample* out) {
    if (s->active_camera < 0) { g_err = "update_frame must be called before rendering"; return TRB_INVALID_ARG; }
    const uint32_t spp = cfg->spp ? next_pow2(cfg->spp) : s->spp_pow2;
    const uint32_t s_first = cfg->sample_first, s_count = cfg->sample_count ? cfg->sample_count : spp - std::min(spp, s_first);
    if (s_first + s_count > spp) { g_err = "sample range exceeds spp"; return TRB_INVALID_ARG; }
    const auto blocks = s->block_list(cfg->block_start, cfg->block_count);
    if (n != blocks.size() * 64 * (size_t)s_count) { g_err = "output size mismatch"; return TRB_INVALID_ARG; }
    const MotionFrame f = motion_frame(s, dt, start, end);
    const uint32_t width = s->film.width;
#pragma omp parallel for schedule(dynamic, 1)
    for (long bi = 0; bi < (long)blocks.size(); ++bi) { /* render_impl's order: block, pixel row-major, sample */
        const uint32_t bx = blocks[bi].first * 8, by = blocks[bi].second * 8;
        size_t o = (size_t)bi * 64 * s_count;
        for (uint32_t py = by; py < by + 8; ++py)
            for (uint32_t px = bx; px < bx + 8; ++px) {
                const PixelStreams st = pixel_streams(cfg->seed, py * width + px);
                for (uint32_t si = s_first; si < s_first + s_count; ++si, ++o) {
                    const uint32_t ip = dm_permute(si, spp, st.kpos);
                    const float sx = van_der_corput(ip, st.scr0) + (float)px, sy = sobol(ip, st.scr1) + (float)py;
                    const float tm = van_der_corput(dm_permute(si, spp, st.ktime), st.scrt);
                    out[o] = motion_of(s, f, sx, sy, tm);
                }
            }
    }
    return TRB_OK;
}

int orc_motion_at(orc_scene* s, size_t n, const float* xyt, float dt, float start, float end, trb_motion_sample* out) {
    if (s->active_camera < 0) { g_err = "update_frame must be called before rendering"; return TRB_INVALID_ARG; }
    const MotionFrame f = motion_frame(s, dt, start, end);
#pragma omp parallel for schedule(dynamic, 1024)
    for (long i = 0; i < (long)n; ++i) out[i] = motion_of(s, f, xyt[3 * i], xyt[3 * i + 1], xyt[3 * i + 2]);
    return TRB_OK;
}

} // extern "C"
