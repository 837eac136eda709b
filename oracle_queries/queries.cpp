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

} // extern "C"
