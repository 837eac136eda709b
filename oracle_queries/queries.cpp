/* The parity oracle's ray queries — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into
 * oracle/_build/liboracle_queries.so and loaded by oracle_queries/pyqueries.py.
 *
 * This translation unit is the detmath oracle (oracle/oracle.cpp, included whole and unchanged, so every orc_* entry point is
 * here too) plus the three ray queries of the reference's public interface, over rays that carry their own time:
 *   orc_intersect_records  Scene::intersect (scene.rs:148-150) -> geometry::Intersection (intersection.rs): Hit::dg, which
 *                          SceneGeom::instance_intersect has already transformed to world space, the instance and its material
 *   orc_occluded           OcclusionTester::occluded (light/mod.rs:30-37): the closest-hit walk of SceneShade::occluded
 *   orc_illumination       thread_work's per-sample body (multithreaded.rs:95-103) along caller rays: Scene::intersect, then the
 *                          scene integrator's Integrator::illumination with the camera-sample stream (seed, key, sample + j)
 * Each ray is Ray::segment(o, d, min_t, max_t, time) and is traced against the TLAS of the current frame.
 * and the shading half of that interface, which traces nothing:
 *   orc_bsdf_eval / orc_bsdf_sample   Material::bsdf at a DifferentialGeometry built from a record's fields, then BSDF::eval and pdf,
 *                                     or BSDF::sample (bsdf.rs:66-125)
 *   orc_light_sample / orc_light_pdf  SceneShade::sample_incident and light_pdf (emitter.rs:164-204)
 *   orc_emitted                       SceneShade::radiance (emitter.rs:140-142)
 *   orc_scene_lights                  the light list of sample_one_light
 * and the film half:
 *   orc_film_write                    RenderTarget::write (render_target.rs:77-165), called once per region that has samples, regions
 *                                     in the Morton block list's order, each region's samples in input order
 */
#include "../oracle/oracle.cpp"

static inline Ray query_ray(const trb_query_ray& q) {
    return Ray::segment(V3(q.o[0], q.o[1], q.o[2]), V3(q.d[0], q.d[1], q.d[2]), q.min_t, q.max_t, q.time);
}
static inline void put3(float* dst, V3 v) { dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; }
static void query_stats(trb_stats* stats, const Counters& total) {
    if (!stats) return;
    memset(stats, 0, sizeof *stats);
    stats->rays_primary = total.rays[0]; stats->rays_shadow = total.rays[1];
    stats->node_tests = total.node_tests; stats->tri_tests = total.tri_tests; stats->inst_tests = total.inst_tests;
}

extern "C" {

int orc_intersect_records(orc_scene* s, size_t n, const trb_query_ray* rays, trb_intersection* out, trb_stats* stats) {
    Counters total;
#pragma omp parallel
    {
        Counters cnt;
#pragma omp for schedule(dynamic, 1024)
        for (long i = 0; i < (long)n; ++i) {
            Ray r = query_ray(rays[i]);
            Hit h;
            cnt.rays[0]++;
            const bool hit = s->geom.intersect(r, h, cnt);
            trb_intersection& o = out[i];
            memset(&o, 0, sizeof o);
            o.t = r.max_t;
            o.inst = hit ? h.inst : TRB_MISS;
            if (!hit) continue;
            o.prim = h.prim; o.material = s->geom.instances[h.inst].material;
            put3(o.p, h.dg.p); put3(o.n, h.dg.n); put3(o.ng, h.dg.ng);
            o.u = h.dg.u; o.v = h.dg.v; o.time = h.dg.time;
            put3(o.dp_du, h.dg.dp_du); put3(o.dp_dv, h.dg.dp_dv);
        }
#pragma omp critical
        total.add(cnt);
    }
    query_stats(stats, total);
    return TRB_OK;
}

int orc_occluded(orc_scene* s, size_t n, const trb_query_ray* rays, uint8_t* occluded, trb_stats* stats) {
    Counters total;
#pragma omp parallel
    {
        Counters cnt;
#pragma omp for schedule(dynamic, 1024)
        for (long i = 0; i < (long)n; ++i) occluded[i] = s->shade.occluded(query_ray(rays[i]), cnt) ? 1 : 0;
#pragma omp critical
        total.add(cnt);
    }
    query_stats(stats, total);
    return TRB_OK;
}

/* trb_illumination's contract: sample j of ray i counts one camera sample and one primary ray, intersects Ray::segment(o, d, min_t,
 * max_t, time) and on a hit runs SceneShade::illumination with PathSamples{seed, key, sample + j, max_depth + 1} — the stream
 * render_impl gives camera sample (seed, pixel, si). rgb[3i + c] = (c_0 + c_1 + ... in j order, each clamped first when `clamp`) / spp. */
int orc_illumination(orc_scene* s, size_t n, const trb_illum_ray* rays, uint32_t spp, uint32_t seed, float* rgb, uint32_t clamp, trb_stats* stats) {
    if (s->active_camera < 0) { g_err = "update_frame must be called before rendering"; return TRB_INVALID_ARG; }
    if (spp == 0) { g_err = "spp must be positive"; return TRB_INVALID_ARG; }
    Counters total;
#pragma omp parallel
    {
        Counters cnt;
#pragma omp for schedule(dynamic, 64)
        for (long i = 0; i < (long)n; ++i) {
            const trb_illum_ray& q = rays[i];
            Col sum(0.0f);
            for (uint32_t j = 0; j < spp; ++j) {
                Ray ray = Ray::segment(V3(q.o[0], q.o[1], q.o[2]), V3(q.d[0], q.d[1], q.d[2]), q.min_t, q.max_t, q.time);
                cnt.camera_samples++;
                cnt.rays[0]++;
                Hit hit;
                Col c(0.0f);
                if (s->geom.intersect(ray, hit, cnt)) {
                    PathSamples ps{seed, q.key, q.sample + j, s->shade.max_depth + 1};
                    c = s->shade.illumination(ray, hit, ps, cnt);
                }
                if (clamp) c = c.clamp();
                sum = j == 0 ? c : sum + c;
            }
            rgb[3 * i] = sum.r / (float)spp; rgb[3 * i + 1] = sum.g / (float)spp; rgb[3 * i + 2] = sum.b / (float)spp;
        }
#pragma omp critical
        total.add(cnt);
    }
    if (stats) {
        memset(stats, 0, sizeof *stats);
        stats->camera_samples = total.camera_samples;
        stats->rays_primary = total.rays[0]; stats->rays_shadow = total.rays[1]; stats->rays_mis = total.rays[2]; stats->rays_continuation = total.rays[3];
        stats->node_tests = total.node_tests; stats->tri_tests = total.tri_tests; stats->inst_tests = total.inst_tests;
    }
    return TRB_OK;
}

/* ---- shading queries: Material::bsdf with BSDF::eval / pdf / sample at a record, Light::sample_incident / pdf, Emitter::radiance.
 * Out-of-range indices (a missed record, material, light or instance past the scene's, a light that is not an emitter) give zeros. */
static bool record_bsdf(const orc_scene* s, const trb_intersection& r, BSDF& bsdf) {
    if (r.inst == TRB_MISS || r.material >= s->shade.materials.size()) return false;
    DG dg;
    dg.p = V3(r.p[0], r.p[1], r.p[2]); dg.n = V3(r.n[0], r.n[1], r.n[2]); dg.ng = V3(r.ng[0], r.ng[1], r.ng[2]);
    dg.u = r.u; dg.v = r.v; dg.time = r.time;
    dg.dp_du = V3(r.dp_du[0], r.dp_du[1], r.dp_du[2]); dg.dp_dv = V3(r.dp_dv[0], r.dp_dv[1], r.dp_dv[2]);
    s->shade.materials[r.material].bsdf(dg, bsdf);
    return true;
}
static bool is_light(const orc_scene* s, uint32_t li) { return li < s->geom.instances.size() && s->geom.instances[li].is_emitter(); }

int orc_bsdf_eval(orc_scene* s, size_t n, const trb_intersection* rec, const trb_bsdf_eval_query* q, float* out4) {
#pragma omp parallel for schedule(dynamic, 1024)
    for (long i = 0; i < (long)n; ++i) {
        float* o = out4 + 4 * i;
        o[0] = o[1] = o[2] = o[3] = 0.0f;
        BSDF bsdf;
        if (!record_bsdf(s, rec[i], bsdf)) continue;
        const V3 wo(q[i].wo[0], q[i].wo[1], q[i].wo[2]), wi(q[i].wi[0], q[i].wi[1], q[i].wi[2]);
        const Col f = bsdf.eval(wo, wi, q[i].bxdf);
        o[0] = f.r; o[1] = f.g; o[2] = f.b; o[3] = bsdf.pdf(wo, wi, q[i].bxdf);
    }
    return TRB_OK;
}

int orc_bsdf_sample(orc_scene* s, size_t n, const trb_intersection* rec, const trb_bsdf_sample_query* q, trb_bsdf_sample_result* out) {
#pragma omp parallel for schedule(dynamic, 1024)
    for (long i = 0; i < (long)n; ++i) {
        trb_bsdf_sample_result& o = out[i];
        memset(&o, 0, sizeof o);
        BSDF bsdf;
        if (!record_bsdf(s, rec[i], bsdf)) continue;
        Col f; V3 wi; float pdf; uint32_t sampled;
        bsdf.sample(V3(q[i].wo[0], q[i].wo[1], q[i].wo[2]), q[i].bxdf, q[i].u[0], q[i].u[1], q[i].u_comp, f, wi, pdf, sampled);
        o.f[0] = f.r; o.f[1] = f.g; o.f[2] = f.b; o.pdf = pdf; put3(o.wi, wi); o.sampled = sampled;
    }
    return TRB_OK;
}

int orc_light_sample(orc_scene* s, size_t n, const trb_light_query* q, trb_light_sample_result* out) {
    if (s->active_camera < 0) { g_err = "update_frame must be called before rendering"; return TRB_INVALID_ARG; }
#pragma omp parallel for schedule(dynamic, 1024)
    for (long i = 0; i < (long)n; ++i) {
        trb_light_sample_result& o = out[i];
        memset(&o, 0, sizeof o);
        if (!is_light(s, q[i].light)) continue;
        Col li; V3 wi; float pdf; Ray occl;
        s->shade.sample_incident(q[i].light, V3(q[i].p[0], q[i].p[1], q[i].p[2]), q[i].u[0], q[i].u[1], q[i].time, li, wi, pdf, occl);
        o.li[0] = li.r; o.li[1] = li.g; o.li[2] = li.b; o.pdf = pdf; put3(o.wi, wi);
        o.delta = s->geom.instances[q[i].light].kind == TRB_INST_EMITTER_POINT ? 1u : 0u;
        put3(o.shadow.o, occl.o); put3(o.shadow.d, occl.d);
        o.shadow.min_t = occl.min_t; o.shadow.max_t = occl.max_t; o.shadow.time = occl.time;
    }
    return TRB_OK;
}

int orc_light_pdf(orc_scene* s, size_t n, const trb_light_pdf_query* q, float* pdf) {
    if (s->active_camera < 0) { g_err = "update_frame must be called before rendering"; return TRB_INVALID_ARG; }
#pragma omp parallel for schedule(dynamic, 1024)
    for (long i = 0; i < (long)n; ++i)
        pdf[i] = is_light(s, q[i].light) ? s->shade.light_pdf(q[i].light, V3(q[i].p[0], q[i].p[1], q[i].p[2]), V3(q[i].wi[0], q[i].wi[1], q[i].wi[2]), q[i].time) : 0.0f;
    return TRB_OK;
}

int orc_emitted(orc_scene* s, size_t n, const trb_emit_query* q, float* rgb) {
#pragma omp parallel for schedule(dynamic, 1024)
    for (long i = 0; i < (long)n; ++i) {
        Col c(0.0f);
        if (is_light(s, q[i].inst)) c = s->shade.radiance(s->geom.instances[q[i].inst], V3(q[i].w[0], q[i].w[1], q[i].w[2]), V3(q[i].n[0], q[i].n[1], q[i].n[2]), q[i].time);
        rgb[3 * i] = c.r; rgb[3 * i + 1] = c.g; rgb[3 * i + 2] = c.b;
    }
    return TRB_OK;
}

/* the light list of sample_one_light: instance indices of the emitters in object order */
int orc_scene_lights(const orc_scene* s, uint32_t* inst) {
    for (size_t k = 0; k < s->shade.lights.size(); ++k) inst[k] = s->shade.lights[k];
    return TRB_OK;
}

/* ---- film writes: the samples grouped by region (index by * (width / 8) + bx; out-of-range indices skip the sample), then the
 * existing RenderTarget::write once per non-empty region in the order of BlockQueue::new's Morton list, one thread, no atomics. */
int orc_film_write(orc_scene* s, size_t n, const trb_sample* samples, const uint32_t* regions, float* film_rgbw) {
    const uint32_t nbx = s->film.width / 8, nr = nbx * (s->film.height / 8);
    std::vector<std::vector<ImageSample>> by_region(nr);
    for (size_t i = 0; i < n; ++i)
        if (regions[i] < nr) by_region[regions[i]].push_back(ImageSample{samples[i].x, samples[i].y, Col(samples[i].r, samples[i].g, samples[i].b)});
    for (const auto& b : s->block_list(0, 0)) {
        const std::vector<ImageSample>& v = by_region[b.second * nbx + b.first];
        if (v.empty()) continue;
        const int x0 = (int)b.first * 8, y0 = (int)b.second * 8;
        s->rt.write(v, x0, y0, x0 + 8, y0 + 8, film_rgbw, false);
    }
    return TRB_OK;
}

} // extern "C"
