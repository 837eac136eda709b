/* The parity oracle's ray queries — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into
 * oracle/_build/liboracle_queries.so and loaded by oracle_queries/pyqueries.py.
 *
 * This translation unit is the detmath oracle (oracle/oracle.cpp, included whole and unchanged, so every orc_* entry point is
 * here too) plus the two ray queries of the reference's public interface, over rays that carry their own time:
 *   orc_intersect_records  Scene::intersect (scene.rs:148-150) -> geometry::Intersection (intersection.rs): Hit::dg, which
 *                          SceneGeom::instance_intersect has already transformed to world space, the instance and its material
 *   orc_occluded           OcclusionTester::occluded (light/mod.rs:30-37): the closest-hit walk of SceneShade::occluded
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

} // extern "C"
