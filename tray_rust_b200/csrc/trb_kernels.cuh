// trb_kernels.cuh — the render hot path of tray_rust as sm_90a CUDA device code.
//
// Path covered (reference file:line in /root/reference):
//   sampler   src/sampler/ld.rs:33-119           (0,2)-sequence samples per pixel / per path
//   camera    src/film/camera.rs:150-157          Camera::generate_ray
//   intersect src/scene.rs:148 -> src/geometry/bvh.rs:81-130 (two levels), bbox.rs:75-104,
//             mesh.rs:136-198, sphere.rs:33-81, disk.rs:42-76, rectangle.rs:38-64,
//             receiver.rs:29-43 / emitter.rs:118-137
//   shading   src/material/*.rs -> src/bxdf/**; src/geometry/emitter.rs:140-204 (Light);
//             src/integrator/mod.rs:106-169, src/integrator/path.rs:45-119, src/mc.rs
//   film      src/exec/multithreaded.rs:98-111, src/film/render_target.rs:77-165
//
// Arithmetic contract: this TU is compiled with --fmad=false (Rust never contracts a*b+c), IEEE
// div/sqrt, and evaluates every expression in the reference's order; transcendentals come from
// trb_detmath.cuh. The result of each camera sample is therefore a pure function of
// (scene, seed, pixel, sample index) — independent of scheduling.
#pragma once
#include "trb_device.h"
#include "trb_detmath.cuh"
#include "trb_anim.h"
#include "trb_adaptive.h"
#include "../../include/trb.h"

namespace trb {

// ------------------------------------------------------------------------------------------
// small vector helpers (componentwise, no FMA)
// ------------------------------------------------------------------------------------------
struct f3 { float x, y, z; };
TRB_HD __forceinline__ f3 mk(float x, float y, float z) { f3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ f3 splat(float v) { return mk(v, v, v); }
__device__ __forceinline__ f3 operator+(f3 a, f3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ f3 operator-(f3 a, f3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ f3 operator*(f3 a, f3 b) { return mk(a.x * b.x, a.y * b.y, a.z * b.z); }
// a / b and sqrtf(a) under a name (div.rn / sqrt.rn, inlined). nvcc expands every IEEE division into ~15 instructions; calling
// them out of line would shrink the shade kernels, but every call then pays the call overhead on the hot path.
__device__ __forceinline__ float ieee_div(float a, float b) { return a / b; }
__device__ __forceinline__ float ieee_sqrt(float a) { return sqrtf(a); }
__device__ __forceinline__ f3 operator/(f3 a, f3 b) { return mk(ieee_div(a.x, b.x), ieee_div(a.y, b.y), ieee_div(a.z, b.z)); }
__device__ __forceinline__ f3 operator*(f3 a, float s) { return mk(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ f3 operator*(float s, f3 a) { return mk(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ f3 operator/(f3 a, float s) { return mk(ieee_div(a.x, s), ieee_div(a.y, s), ieee_div(a.z, s)); }
__device__ __forceinline__ f3 operator-(f3 a) { return mk(-a.x, -a.y, -a.z); }
__device__ __forceinline__ float dot3(f3 a, f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ f3 cross3(f3 a, f3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float len2(f3 a) { return a.x * a.x + a.y * a.y + a.z * a.z; }
__device__ __forceinline__ f3 unit(f3 a) { float l = ieee_sqrt(len2(a)); return mk(ieee_div(a.x, l), ieee_div(a.y, l), ieee_div(a.z, l)); } // Vector::normalized: 3 divides
__device__ __forceinline__ bool black(f3 c) { return c.x == 0.0f && c.y == 0.0f && c.z == 0.0f; }
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }
__device__ __forceinline__ float lerpf(float t, float a, float b) { return a * (1.0f - t) + b * t; }
__device__ __forceinline__ float finf() { return __int_as_float(0x7f800000); }

// Transform application (src/linalg/transform.rs:150-254), m row-major 4x4
__device__ __forceinline__ f3 xf_point(const float* __restrict__ m, f3 p) {
    f3 r = mk(m[0] * p.x + m[1] * p.y + m[2] * p.z + m[3], m[4] * p.x + m[5] * p.y + m[6] * p.z + m[7],
              m[8] * p.x + m[9] * p.y + m[10] * p.z + m[11]);
    float w = m[12] * p.x + m[13] * p.y + m[14] * p.z + m[15];
    if (fabsf(w - 1.0f) < TRB_EPS) return r / w; // sic: transform.rs:158-162
    return r;
}
__device__ __forceinline__ f3 xf_vector(const float* __restrict__ m, f3 v) {
    return mk(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[4] * v.x + m[5] * v.y + m[6] * v.z, m[8] * v.x + m[9] * v.y + m[10] * v.z);
}
// normal through the transpose of the OTHER matrix (transform.rs:231-242)
__device__ __forceinline__ f3 xf_normal_t(const float* __restrict__ m, f3 n) {
    return mk(m[0] * n.x + m[4] * n.y + m[8] * n.z, m[1] * n.x + m[5] * n.y + m[9] * n.z, m[2] * n.x + m[6] * n.y + m[10] * n.z);
}
// linalg::coordinate_system (src/linalg/mod.rs:96-108)
__device__ __forceinline__ void coord_system(f3 e1, f3& e2, f3& e3) {
    if (fabsf(e1.x) > fabsf(e1.y)) {
        float il = 1.0f / sqrtf(e1.x * e1.x + e1.z * e1.z);
        e2 = mk(-e1.z * il, 0.0f, e1.x * il);
    } else {
        float il = 1.0f / sqrtf(e1.y * e1.y + e1.z * e1.z);
        e2 = mk(0.0f, e1.z * il, -e1.y * il);
    }
    e3 = cross3(e1, e2);
}

// One 32-byte half of a node / triangle record through the read-only path. sm_90 has no 256-bit load, so this is two
// 128-bit LDG.E.128.CONSTANT issued back to back (the widest load Hopper has); records are 32-byte aligned, so each
// half is exactly one 32-byte sector.
__device__ __forceinline__ void ldg256(const void* p, float4& a, float4& b) {
    const float4* q = static_cast<const float4*>(p);
    a = __ldg(q);
    b = __ldg(q + 1);
}

struct Ray { f3 o, d; float tmin, tmax; };
struct HitRec { float t; uint32_t inst, prim; float b1, b2; };
struct Cnt { uint32_t node, tri, inst; };

// ------------------------------------------------------------------------------------------
// BBox::fast_intersect (src/geometry/bbox.rs:75-104), compares transcribed literally so the NaN
// behaviour (SURVEY A5) is the reference's.
// ------------------------------------------------------------------------------------------
TRB_HD __forceinline__ bool box_hit(const float4 lo, const float4 hi, f3 o, f3 inv, bool nx, bool ny, bool nz, float tmin_r, float tmax_r, float& t_entry) {
    // Branch-free form of the reference's early returns: every statement below is the reference's, in its order; the two
    // `return false` become flags, which cannot change the outcome (after either the result is false whatever follows)
    // and saves the divergent branches + reconvergence the warp would execute anyway for the lanes that go on.
    float tmin = ((nx ? hi.x : lo.x) - o.x) * inv.x;
    float tmax = ((nx ? lo.x : hi.x) - o.x) * inv.x;
    const float tymin = ((ny ? hi.y : lo.y) - o.y) * inv.y;
    const float tymax = ((ny ? lo.y : hi.y) - o.y) * inv.y;
    const bool miss_xy = tmin > tymax || tymin > tmax; // bbox.rs:87-89 `return false`
    if (tymin > tmin) tmin = tymin;
    if (tymax < tmax) tmax = tymax;
    const float tzmin = ((nz ? hi.z : lo.z) - o.z) * inv.z;
    const float tzmax = ((nz ? lo.z : hi.z) - o.z) * inv.z;
    const bool miss_z = tmin > tzmax || tzmin > tmax;  // bbox.rs:96-98 `return false`
    if (tzmin > tmin) tmin = tzmin;
    if (tzmax < tmax) tmax = tzmax;
    t_entry = tmin; // the only quantity a later, smaller max_t can still reject: `tmin < r.max_t` (bbox.rs:103)
    return !miss_xy && !miss_z && tmin < tmax_r && tmax > tmin_r;
}

// One visit of a DQuad record (trb_device.h): four box tests, then the reference's visit order. `next` is the first
// slot hit in that order (QUAD_EMPTY if none); the other hit slots come back farthest-first in e[0..2] so that the
// caller pushes them in this order and they pop nearest-first. Each entry = entry distance << 32 | reference.
// Host+device: trb_host_quad_check runs this very function against a literal bvh.rs:81-130 traversal.
struct QuadOut { uint32_t next; unsigned long long e0, e1, e2; bool p0, p1, p2; };
TRB_HD __forceinline__ void quad_visit(const float4 q0, const float4 q1, const float4 q2, const float4 q3, const float4 q4, const float4 q5, const float4 q6,
                                       const float4 q7, f3 o, f3 inv, bool nx, bool ny, bool nz, float tmin, float tmax, QuadOut& out) {
    const uint32_t r0 = f32_bits(q0.w), r1 = f32_bits(q2.w), r2 = f32_bits(q4.w), r3 = f32_bits(q6.w), meta = f32_bits(q1.w);
    float t0, t1, t2, t3;
    const bool h0 = box_hit(q0, q1, o, inv, nx, ny, nz, tmin, tmax, t0) && r0 != QUAD_EMPTY;
    const bool h1 = box_hit(q2, q3, o, inv, nx, ny, nz, tmin, tmax, t1) && r1 != QUAD_EMPTY;
    const bool h2 = box_hit(q4, q5, o, inv, nx, ny, nz, tmin, tmax, t2) && r2 != QUAD_EMPTY;
    const bool h3 = box_hit(q6, q7, o, inv, nx, ny, nz, tmin, tmax, t3) && r3 != QUAD_EMPTY;
    const uint32_t ap = meta & 3u, al = (meta >> 2) & 3u, ar = (meta >> 4) & 3u;
    const bool negp = ap == 0 ? nx : (ap == 1 ? ny : nz), negl = al == 0 ? nx : (al == 1 ? ny : nz), negr = ar == 0 ? nx : (ar == 1 ? ny : nz);
    // each half in its own near-first order (an empty slot never hits, so its position does not matter)
    const bool hla = negl ? h1 : h0, hlb = negl ? h0 : h1, hra = negr ? h3 : h2, hrb = negr ? h2 : h3;
    const uint32_t rla = negl ? r1 : r0, rlb = negl ? r0 : r1, rra = negr ? r3 : r2, rrb = negr ? r2 : r3;
    const float tla = negl ? t1 : t0, tlb = negl ? t0 : t1, tra = negr ? t3 : t2, trb_ = negr ? t2 : t3;
    // halves in P's near-first order
    const bool a0 = negp ? hra : hla, a1 = negp ? hrb : hlb, a2 = negp ? hla : hra, a3 = negp ? hlb : hrb;
    const uint32_t s0 = negp ? rra : rla, s1 = negp ? rrb : rlb, s2 = negp ? rla : rra, s3 = negp ? rlb : rrb;
    const float u1 = negp ? trb_ : tlb, u2 = negp ? tla : tra, u3 = negp ? tlb : trb_;
    out.next = a0 ? s0 : (a1 ? s1 : (a2 ? s2 : (a3 ? s3 : QUAD_EMPTY)));
    out.p0 = a3 && (a0 || a1 || a2); out.e0 = ((unsigned long long)f32_bits(u3) << 32) | s3;
    out.p1 = a2 && (a0 || a1);       out.e1 = ((unsigned long long)f32_bits(u2) << 32) | s2;
    out.p2 = a1 && a0;               out.e2 = ((unsigned long long)f32_bits(u1) << 32) | s1;
}

// solve_quadratic (src/linalg/mod.rs:78-94)
__device__ __forceinline__ bool solve_quadratic(float a, float b, float c, float& t0, float& t1) {
    float ds = b * b - 4.0f * a * c;
    if (ds < 0.0f) return false;
    float disc = sqrtf(ds);
    float q = b < 0.0f ? -0.5f * (b - disc) : -0.5f * (b + disc);
    float x = q / a, y = c / q;
    if (x > y) { t0 = y; t1 = x; } else { t0 = x; t1 = y; }
    return true;
}
// accept tests of the analytic shapes, object space; return t and shrink tmax
__device__ __forceinline__ bool sphere_t(float radius, f3 o, f3 d, float tmin, float& tmax) { // sphere.rs:33-55
    float a = len2(d);
    float b = 2.0f * dot3(d, o);
    float c = dot3(o, o) - radius * radius;
    float t0, t1;
    if (!solve_quadratic(a, b, c, t0, t1)) return false;
    if (t0 > tmax || t1 < tmin) return false;
    float th = t0;
    if (th < tmin) { th = t1; if (th > tmax) return false; }
    tmax = th;
    return true;
}
__device__ __forceinline__ bool disk_t(float radius, float inner, f3 o, f3 d, float tmin, float& tmax) { // disk.rs:42-68
    if (fabsf(d.z) == 0.0f) return false;
    float t = -o.z / d.z;
    if (t < tmin || t > tmax) return false;
    f3 p = o + d * t;
    float ds = p.x * p.x + p.y * p.y;
    if (ds > radius * radius || ds < inner * inner) return false;
    // disk.rs:60-66: phi = atan2(p.y, p.x) (+2pi if negative) can never exceed 2pi in fp32, and a NaN
    // phi fails both compares, so the test never rejects: omitted (DESIGN.md "dead code").
    tmax = t;
    return true;
}
__device__ __forceinline__ bool rect_t(float width, float height, f3 o, f3 d, float tmin, float& tmax) { // rectangle.rs:38-51
    if (fabsf(d.z) < 1e-8f) return false;
    float t = -o.z / d.z;
    if (t < tmin || t > tmax) return false;
    f3 p = o + d * t;
    float hw = width / 2.0f, hh = height / 2.0f;
    if (p.x >= -hw && p.x <= hw && p.y >= -hh && p.y <= hh) { tmax = t; return true; }
    return false;
}

__device__ __forceinline__ void load_xf(const float* __restrict__ src, float* dst) {
    const float4* s = reinterpret_cast<const float4*>(src);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float4 v = __ldg(s + i); dst[4 * i] = v.x; dst[4 * i + 1] = v.y; dst[4 * i + 2] = v.z; dst[4 * i + 3] = v.w; }
}

// AnimatedTransform::transform(ray.time) of a keyframed instance: the reference recomposes it per ray per instance
// (receiver.rs:30, emitter.rs:122,176,197); static instances use the matrices prepared by update_frame.
__device__ __noinline__ void eval_anim_xf(const DScene& sc, uint32_t first, uint32_t n, float time, float* inv16, float* mat16) {
    const trbh::Xf x = trbh::animated_xf(sc.splines, first, n, sc.keyframes, sc.knots, time, sc.level_xf);
#pragma unroll
    for (int i = 0; i < 16; ++i) { inv16[i] = x.inv.m[i]; if (mat16) mat16[i] = x.fwd.m[i]; }
}
// Keyframed instances in the wavefront pipeline: AnimatedTransform::transform(time) depends only on (instance, ray.time) and every ray
// of a path carries the camera ray's time, so k_wf_anim_table evaluates it ONCE per (path, keyframed instance) with the very same
// function (bit-identical) into a per-path row: entry `anim_slot` = 16 floats inverse + 16 floats forward. `row` == nullptr
// (megakernel, trb_intersect, Whitted): evaluate in place, per ray per instance, like the reference.
__device__ __forceinline__ void load_row(const float* __restrict__ src, float* dst) { // plain loads: the table is written by an earlier kernel of the same pass
    const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float4 v = s4[i]; dst[4 * i] = v.x; dst[4 * i + 1] = v.y; dst[4 * i + 2] = v.z; dst[4 * i + 3] = v.w; }
}
template <bool ANIM>
__device__ __forceinline__ void instance_inv(const DScene& sc, const DInstance& in, float time, float* inv16, const float* row = nullptr) {
    if (ANIM && (__ldg(&in.flags) & DI_ANIM_XF)) {
        if (row) load_row(row + 32 * __ldg(&in.anim_slot), inv16);
        else eval_anim_xf(sc, __ldg(&in.spline_first), __ldg(&in.n_splines), time, inv16, nullptr);
    } else load_xf(in.inv, inv16);
}
template <bool ANIM>
__device__ __forceinline__ void instance_inv_mat(const DScene& sc, const DInstance& in, float time, float* inv16, float* mat16, const float* row = nullptr) {
    if (ANIM && (__ldg(&in.flags) & DI_ANIM_XF)) {
        if (row) { const float* e = row + 32 * __ldg(&in.anim_slot); load_row(e, inv16); load_row(e + 16, mat16); }
        else eval_anim_xf(sc, __ldg(&in.spline_first), __ldg(&in.n_splines), time, inv16, mat16);
    } else { load_xf(in.inv, inv16); load_xf(in.mat, mat16); }
}
// AnimatedColor::color(time) of an emitter (animated_color.rs:52-78)
template <bool ANIM>
__device__ __forceinline__ void emission_at(const DScene& sc, const DInstance& in, float time, float& r, float& g, float& b) {
    if (ANIM && (__ldg(&in.flags) & DI_ANIM_EMISSION)) {
        float c[3];
        trbh::animated_color(sc.color_keys, __ldg(&in.emission_first), __ldg(&in.n_emission), time, c);
        r = c[0]; g = c[1]; b = c[2];
    } else { r = __ldg(&in.emission[0]); g = __ldg(&in.emission[1]); b = __ldg(&in.emission[2]); }
}

// ------------------------------------------------------------------------------------------
// Scene::intersect (scene.rs:148-150) = BVH<Instance>::intersect (bvh.rs:81-130) whose leaf callback
// is Instance::intersect (receiver.rs:29-43 / emitter.rs:118-137), which for meshes runs
// BVH<Triangle>::intersect with intersect_triangle (mesh.rs:136-170; only the accept test — normals,
// uv and derivatives are deferred to the final hit, surface_at()).
//
// GPU shape: ONE structured loop for both levels so a warp never serialises on "who is inside a
// mesh": the stack holds TLAS nodes, pending instances of a TLAS leaf (pushed in reverse so they
// pop in the reference's order) and, below a mesh's nodes, a RETURN marker that restores the world
// ray. Visit order, compares and the shrinking max_t are exactly the reference's, so hit indices,
// t and the test counters are bit-identical to the oracle. No early `return` inside the loop: every
// divergent branch reconverges at the loop head.
// ------------------------------------------------------------------------------------------
// `cur` / stack references: 2 tag bits + payload
//   00 interior record | 01 leaf (count << 25 | first slot) | 10 pending instance (slot in tlas_order) | 11 control
constexpr uint32_t ST_INSTANCE = 0x80000000u;
constexpr uint32_t ST_ROOT = 0xfffffffdu;   // test the current level's root box, then go to its reference
constexpr uint32_t ST_RETURN = 0xfffffffeu; // leave the mesh: restore the world ray
constexpr uint32_t ST_DONE = 0xffffffffu;
constexpr int STACK_DEPTH = 96;

// Where the wavefront trace kernel keeps the parts of a ray's state that are touched once or twice per ray, instead of in
// registers for the ray's whole life (13 registers -> one more resident CTA per SM): the world-space ray is re-read from the
// path state when a mesh is left (1/d recomputed by the same three IEEE divisions), and an accepted hit is written to the
// path's hit record at once (a later, nearer hit overwrites it; same thread, program order).
struct RayHome {
    const float4* org; const float4* dir; // this ray's origin / direction entries of the path state
    uint4* hit;                           // type 0 (continuation / primary): (inst, prim, b1, b2)
    float* a_w;                           // type 2 (MIS): the hit instance goes to wf.a[p].w
    int type;
};
// The traversal as an explicit state machine so that a warp can keep all lanes busy: scene_trace()
// runs it to completion for one ray; the wavefront trace kernel refills finished lanes with new rays.
struct TraceState {
    f3 wo, wd, winv;      // world ray and 1/d (bvh.rs:84)
    f3 o, d, inv;         // ray of the current level (world, or the mesh instance's object space)
    uint32_t neg;         // bit k: d[k] < 0 (bvh.rs:85)
    const DBvh* bvh;      // current level (root box + reference)
    const DPair* pairs;   // current level's records, kept in registers: no pointer chase per step (DQuad records when `quad`)
    bool quad;            // this level is traversed through the DQuad records (finite 1/d only, see trb_device.h)
    bool quads_ok;        // the kernel variant may use DQuad records at all
    bool exact_box;       // the current level's ray has a zero, NaN or infinite component: literal box_hit (see box_hit_finite)
    bool force_exact;     // test option "trace.exact_box": every ray takes the literal box_hit
    const DTri* tris;
    uint32_t level_inst;  // instance whose mesh is being traversed, TRB_MISS at the top level
    float tmin, tmax;
    float time;           // ray.time (only read for keyframed instances)
    const float* xf_row;  // this path's row of evaluated keyframed transforms (wavefront), nullptr: evaluate per instance test
    int sp;
    uint32_t cur;
    bool found, any_hit;
    uint32_t h_inst, h_prim;
    float h_b1, h_b2;
};
__device__ __forceinline__ uint32_t neg_mask(f3 d) { return (d.x < 0.0f ? 1u : 0u) | (d.y < 0.0f ? 2u : 0u) | (d.z < 0.0f ? 4u : 0u); }
__device__ __forceinline__ bool finite3(f3 v) { return fabsf(v.x) < finf() && fabsf(v.y) < finf() && fabsf(v.z) < finf(); }
__device__ __forceinline__ void trace_level(TraceState& t, const DBvh* bvh, const DPair* pairs, const DQuad* quads) {
    t.bvh = bvh;
    t.exact_box = t.force_exact || !(finite3(t.o) && finite3(t.d) && finite3(t.inv));
    t.quad = t.quads_ok && finite3(t.inv);
    t.pairs = t.quad ? reinterpret_cast<const DPair*>(quads) : pairs;
}
__device__ __forceinline__ void trace_init(const DScene& sc, TraceState& t, const Ray& ray, bool any_hit, float time, bool quads_ok = false, bool force_exact = false) {
    t.time = time; t.quads_ok = quads_ok; t.xf_row = nullptr; t.force_exact = force_exact;
    t.wo = ray.o; t.wd = ray.d;
    t.winv = mk(1.0f / ray.d.x, 1.0f / ray.d.y, 1.0f / ray.d.z);
    t.o = t.wo; t.d = t.wd; t.inv = t.winv;
    t.neg = neg_mask(t.d);
    trace_level(t, sc.tlas, sc.tlas_pairs, sc.tlas_quads);
    t.tris = nullptr; t.level_inst = TRB_MISS;
    t.tmin = ray.tmin; t.tmax = ray.tmax;
    t.sp = 0; t.cur = ST_ROOT; t.found = false; t.any_hit = any_hit;
    t.h_inst = TRB_MISS; t.h_prim = 0; t.h_b1 = 0.0f; t.h_b2 = 0.0f;
}
// Traversal stack storage. LocalStack: per-thread local memory. HybridStack: the 16 hottest entries live in shared
// memory ([entry][thread], conflict-free 8-byte accesses), deeper entries spill to local memory — pops no longer
// compete with node fetches for L1 (the trace kernel's second most frequent stall was the local-memory pop).
struct LocalStack {
    unsigned long long* s;
    __device__ __forceinline__ void put(int i, unsigned long long v) const { s[i] = v; }
    __device__ __forceinline__ unsigned long long get(int i) const { return s[i]; }
};
template <int SMEM_STACK>
struct HybridStack {
    unsigned long long* sm; // &smem[0][threadIdx.x], stride = blockDim.x = 128
    unsigned long long* lo;
    __device__ __forceinline__ void put(int i, unsigned long long v) const { if (i < SMEM_STACK) sm[i * 128] = v; else lo[i - SMEM_STACK] = v; }
    __device__ __forceinline__ unsigned long long get(int i) const { return i < SMEM_STACK ? sm[i * 128] : lo[i - SMEM_STACK]; }
};

// Pop the next reference. A node entry carries the entry distance of its box, computed when its parent was
// visited; the reference tests that box only now, against the current (smaller) max_t: `tmin < r.max_t`.
template <class Stack>
__device__ __forceinline__ uint32_t trace_pop(TraceState& t, const Stack& stack) {
    while (t.sp > 0) {
        const unsigned long long e = stack.get(--t.sp);
        const uint32_t ref = (uint32_t)e;
        if (ref & ST_INSTANCE) return ref; // pending instances and control entries are never culled
        if (__uint_as_float((uint32_t)(e >> 32)) < t.tmax) return ref;
    }
    return ST_DONE;
}
// One transition: visit an interior node (two box tests), a leaf, the root, a pending instance, or leave a mesh.
// WIDE: mesh leaf references carry no count (REF_LEAF | first slot); the leaf ends at the triangle marked TRI_LEAF_END.
template <bool STATS, bool ANIM, bool WIDE = false, class Stack>
__device__ __forceinline__ void trace_step(const DScene& sc, TraceState& t, const Stack& stack, Cnt& cnt, int* err) {
    const uint32_t cur = t.cur;
    const uint32_t tag = cur & REF_TAG;
    uint32_t next;
    if (tag == REF_INTERIOR) {
        const DPair* __restrict__ rec = t.pairs + cur;
        const float4 l_lo = __ldg(&rec->l_lo), l_hi = __ldg(&rec->l_hi), r_lo = __ldg(&rec->r_lo), r_hi = __ldg(&rec->r_hi);
        if (STATS) cnt.node += 2; // the reference tests the near child now and the far child when it pops it
        float tl, tr;
        const bool hl = box_hit(l_lo, l_hi, t.o, t.inv, (t.neg & 1u) != 0, (t.neg & 2u) != 0, (t.neg & 4u) != 0, t.tmin, t.tmax, tl);
        const bool hr = box_hit(r_lo, r_hi, t.o, t.inv, (t.neg & 1u) != 0, (t.neg & 2u) != 0, (t.neg & 4u) != 0, t.tmin, t.tmax, tr);
        const uint32_t axis = __float_as_uint(r_lo.w);
        const bool neg = ((t.neg >> axis) & 1u) != 0; // near child = second_child iff d[axis] < 0 (bvh.rs:111-117)
        const uint32_t ref_l = __float_as_uint(l_lo.w), ref_r = __float_as_uint(l_hi.w);
        const bool h_near = neg ? hr : hl, h_far = neg ? hl : hr;
        const uint32_t ref_near = neg ? ref_r : ref_l, ref_far = neg ? ref_l : ref_r;
        const float t_far = neg ? tl : tr;
        if (h_near) {
            next = ref_near;
            if (h_far) {
                if (t.sp >= STACK_DEPTH - 6) { *err = 1; t.sp = 0; next = ST_DONE; }
                else stack.put(t.sp++, ((unsigned long long)__float_as_uint(t_far) << 32) | ref_far);
            }
        } else if (h_far) next = ref_far; // nothing was tested in between, so max_t is unchanged: same outcome as pop + test
        else next = trace_pop(t, stack);
    } else if (tag == REF_LEAF) {
        const uint32_t a = cur & 0x01ffffffu, n = (cur >> 25) & 31u;
        if (t.level_inst == TRB_MISS) {
            for (uint32_t k = a + n; k-- > a;) stack.put(t.sp++, ST_INSTANCE | k); // pops as a, a+1, ... (bvh.rs:95-98)
        } else {
            const DTri* __restrict__ tris = t.tris;
            for (uint32_t k = WIDE ? (cur & ~REF_TAG) : a; WIDE || k < a + n; ++k) {
                const float4 v0 = __ldg(&tris[k].v0), q0 = __ldg(&tris[k].e0), q1 = __ldg(&tris[k].e1);
                if (STATS) cnt.tri++;
                const f3 e0 = mk(q0.x, q0.y, q0.z), e1 = mk(q1.x, q1.y, q1.z);
                const f3 s0 = cross3(t.d, e1);
                const float dd = dot3(s0, e0);
                const float div = 1.0f / dd;
                const f3 dv = t.o - mk(v0.x, v0.y, v0.z);
                const float b1 = dot3(dv, s0) * div;
                const f3 s1 = cross3(dv, e0);
                const float b2 = dot3(t.d, s1) * div;
                const float tt = dot3(e1, s1) * div;
                // mesh.rs:142-168: d == 0 -> miss; b1 in [0,1]; b2 >= 0 and b1+b2 <= 1; t in [min_t, max_t]
                const bool ok = dd != 0.0f && !(b1 < 0.0f || b1 > 1.0f) && !(b2 < 0.0f || b1 + b2 > 1.0f) && !(tt < t.tmin || tt > t.tmax);
                if (ok) { // last accepted wins, inclusive compare (Q9)
                    t.tmax = tt;
                    t.h_prim = __float_as_uint(v0.w); t.h_b1 = b1; t.h_b2 = b2; t.h_inst = t.level_inst;
                    t.found = true;
                    if (t.any_hit) t.sp = 0;
                }
                if (WIDE && __float_as_uint(q0.w) == TRI_LEAF_END) break;
            }
        }
        next = trace_pop(t, stack);
    } else if (cur == ST_ROOT) {
        const float4 lo = __ldg(&t.bvh->root_lo), hi = __ldg(&t.bvh->root_hi);
        if (STATS) cnt.node++;
        float te;
        next = box_hit(lo, hi, t.o, t.inv, (t.neg & 1u) != 0, (t.neg & 2u) != 0, (t.neg & 4u) != 0, t.tmin, t.tmax, te) ? __float_as_uint(lo.w) : trace_pop(t, stack);
    } else if (cur == ST_RETURN) {
        t.o = t.wo; t.d = t.wd; t.inv = t.winv;
        t.neg = neg_mask(t.d);
        t.bvh = sc.tlas; t.pairs = sc.tlas_pairs; t.level_inst = TRB_MISS;
        next = trace_pop(t, stack);
    } else {
        // Instance::intersect for one entry of a TLAS leaf
        const uint32_t ii = __ldg(&sc.tlas_order[cur & ~REF_TAG]);
        const DInstance& in = sc.instances[ii];
        if (STATS) cnt.inst++;
        const uint32_t kind = __ldg(&in.kind), shape = __ldg(&in.shape);
        next = ST_DONE;
        bool enter = false;
        if (kind != TRB_INST_EMITTER_POINT) { // point lights never intersect (emitter.rs:119-120)
            float m[16];
            instance_inv<ANIM>(sc, in, t.time, m, t.xf_row);
            const f3 lo_ = xf_point(m, t.wo), ld_ = xf_vector(m, t.wd); // inv_mul_ray: direction not renormalised
            if (shape == TRB_SHAPE_MESH) {
                const DMesh& me = sc.meshes[__ldg(&in.mesh)];
                t.o = lo_; t.d = ld_;
                t.inv = mk(1.0f / ld_.x, 1.0f / ld_.y, 1.0f / ld_.z);
                t.neg = neg_mask(ld_);
                t.bvh = &me.bvh; t.pairs = me.bvh.pairs; t.tris = me.tris; t.level_inst = ii;
                stack.put(t.sp++, ST_RETURN);
                next = ST_ROOT; // BVH<Triangle>::intersect starts by testing its root box
                enter = true;
            } else {
                const float p0 = __ldg(&in.p0), p1 = __ldg(&in.p1);
                float tt = t.tmax;
                bool h;
                if (shape == TRB_SHAPE_SPHERE) h = sphere_t(p0, lo_, ld_, t.tmin, tt);
                else if (shape == TRB_SHAPE_DISK) h = disk_t(p0, p1, lo_, ld_, t.tmin, tt);
                else h = rect_t(p0, p1, lo_, ld_, t.tmin, tt);
                if (h) {
                    t.tmax = tt; // receiver.rs:36
                    t.h_inst = ii; t.h_prim = 0; t.h_b1 = 0.0f; t.h_b2 = 0.0f;
                    t.found = true;
                    if (t.any_hit) t.sp = 0;
                }
            }
        }
        if (!enter) next = trace_pop(t, stack);
    }
    t.cur = next;
}

// ------------------------------------------------------------------------------------------
// The same state machine cut into three kinds of micro-step so that a warp can run them in PHASES
// (k_wf_trace, PHASED): per ray the sequence of operations — and therefore hits, t and the test
// counters — is exactly trace_step's; only *when* a lane takes its next micro-step changes.
//   node      one child-pair visit, or pop attempts                       (~64 per ray on C4)   step_nodes
//   triangle  one triangle of a mesh leaf                                  (~4.5 per ray)        step_triangle
//   other     level root box, TLAS leaf, instance entry, mesh return       (~6 per ray)          step_other
// In the flat loop a warp executes all three kinds of code every iteration with whatever lanes are in that
// state, so the triangle code and the pop loop run with only a few of the 32 lanes active.
// ------------------------------------------------------------------------------------------
constexpr uint32_t ST_POP = 0xfffffffcu; // control: take the next reference off the stack
constexpr uint32_t WF_TRACE_FORCE_EXACT_BOX = 0x40000000u; // k_wf_trace flag (option "trace.exact_box"): see TraceState::force_exact
constexpr int WF_BURST = 3;
__device__ __forceinline__ bool trace_is_node(uint32_t cur) { return (cur & REF_TAG) == REF_INTERIOR || cur == ST_POP; }
template <bool STATS, bool QUADS, class Stack>
__device__ __forceinline__ void step_nodes(TraceState& t, const Stack& stack, Cnt& cnt, int* err) {
    uint32_t cur = t.cur;
    if (QUADS && cur != ST_POP && t.quad) {
        const float4* __restrict__ rec = reinterpret_cast<const DQuad*>(t.pairs)[cur].q;
        float4 q0, q1, q2, q3, q4, q5, q6, q7;
        ldg256(rec, q0, q1); ldg256(rec + 2, q2, q3); ldg256(rec + 4, q4, q5); ldg256(rec + 6, q6, q7);
        QuadOut qo;
        quad_visit(q0, q1, q2, q3, q4, q5, q6, q7, t.o, t.inv, (t.neg & 1u) != 0, (t.neg & 2u) != 0, (t.neg & 4u) != 0, t.tmin, t.tmax, qo);
        cur = qo.next == QUAD_EMPTY ? ST_POP : qo.next;
        if (qo.p2) { // at least one more slot was hit
            if (t.sp >= STACK_DEPTH - 6) { *err = 1; t.sp = 0; cur = ST_DONE; }
            else {
                if (qo.p0) stack.put(t.sp++, qo.e0);
                if (qo.p1) stack.put(t.sp++, qo.e1);
                stack.put(t.sp++, qo.e2);
            }
        } else if (qo.p0 || qo.p1) {
            if (t.sp >= STACK_DEPTH - 6) { *err = 1; t.sp = 0; cur = ST_DONE; }
            else {
                if (qo.p0) stack.put(t.sp++, qo.e0);
                if (qo.p1) stack.put(t.sp++, qo.e1);
            }
        }
    } else if (cur != ST_POP) {
        const DPair* __restrict__ rec = t.pairs + cur;
        float4 l_lo, l_hi, r_lo, r_hi;
        ldg256(&rec->l_lo, l_lo, l_hi);
        ldg256(&rec->r_lo, r_lo, r_hi);
        if (STATS) cnt.node += 2;
        float tl, tr;
        const bool hl = box_hit(l_lo, l_hi, t.o, t.inv, (t.neg & 1u) != 0, (t.neg & 2u) != 0, (t.neg & 4u) != 0, t.tmin, t.tmax, tl);
        const bool hr = box_hit(r_lo, r_hi, t.o, t.inv, (t.neg & 1u) != 0, (t.neg & 2u) != 0, (t.neg & 4u) != 0, t.tmin, t.tmax, tr);
        const uint32_t axis = __float_as_uint(r_lo.w);
        const bool neg = ((t.neg >> axis) & 1u) != 0; // near child = second_child iff d[axis] < 0 (bvh.rs:111-117)
        const uint32_t ref_l = __float_as_uint(l_lo.w), ref_r = __float_as_uint(l_hi.w);
        const bool both = hl && hr;
        // both hit: the near child now, the far one on the stack; one hit: that child (nothing is tested in between, so
        // max_t is unchanged and the far child's deferred test has the same outcome); none: pop
        cur = both ? (neg ? ref_r : ref_l) : (hl ? ref_l : (hr ? ref_r : ST_POP));
        if (both) {
            if (t.sp >= STACK_DEPTH - 6) { *err = 1; t.sp = 0; cur = ST_DONE; }
            else stack.put(t.sp++, ((unsigned long long)__float_as_uint(neg ? tl : tr) << 32) | (neg ? ref_l : ref_r));
        }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) { // bounded: a lane with a long run of culled entries comes back next iteration
        if (cur == ST_POP) { // entry 0 of a PHASED kernel's stack is a ST_DONE sentinel (never culled): no empty-stack test
            const unsigned long long e = stack.get(--t.sp);
            const uint32_t ref = (uint32_t)e;
            if ((ref & ST_INSTANCE) || __uint_as_float((uint32_t)(e >> 32)) < t.tmax) cur = ref;
        }
    }
    t.cur = cur;
}
// BBox::fast_intersect for a ray whose origin, direction and 1/direction are all finite (TraceState::exact_box == false):
// then none of the six slab distances is NaN ((plane - o) is finite or ±inf, 1/d is finite and non-zero), near <= far on
// every axis (lo <= hi, near/far chosen by the sign of d, IEEE rounding is monotone), and the reference's sequence
//   reject if a > B || b > A;  m = max(a, b), M = min(A, B);  reject if m > C || c > M;  m = max(m, c), M = min(M, C)
// accepts exactly when max(a, b, c) <= min(A, B, C) — nine pairwise conditions of which the reference tests six and the
// other three (a <= A, b <= B, c <= C) hold by construction — with the same final tmin (up to the sign of a zero, which
// no compare sees). 23 instructions (6 select, 6 sub, 6 mul, 2 FMNMX3, 3 compares) instead of 33. Rays with a zero, NaN
// or infinite component keep the literal box_hit.
__device__ __forceinline__ bool box_hit_finite(const float4 lo, const float4 hi, f3 o, f3 inv, bool nx, bool ny, bool nz, float tmin_r, float tmax_r, float& t_entry) {
    const float ax = ((nx ? hi.x : lo.x) - o.x) * inv.x, bx = ((nx ? lo.x : hi.x) - o.x) * inv.x;
    const float ay = ((ny ? hi.y : lo.y) - o.y) * inv.y, by = ((ny ? lo.y : hi.y) - o.y) * inv.y;
    const float az = ((nz ? hi.z : lo.z) - o.z) * inv.z, bz = ((nz ? lo.z : hi.z) - o.z) * inv.z;
    const float m = fmaxf(fmaxf(ax, ay), az), M = fminf(fminf(bx, by), bz);
    t_entry = m;
    return m <= M && m < tmax_r && M > tmin_r;
}
// Self-test (trb_selftest_box): box_hit_finite against the literal box_hit on generated boxes and rays whose components are
// drawn from a table of awkward values (zeros of both signs, denormals, huge and tiny magnitudes, planes equal to the ray origin,
// degenerate boxes) mixed with random ones. For every all-finite ray the hit flags must agree and, on a hit, the entry
// distances must compare equal (a zero's sign may differ). out[0] = cases with an all-finite ray, out[1] = hits among
// them, out[2] = mismatches, out[3] = cases that take the literal path (a zero / NaN / infinite component).
__device__ __forceinline__ float selftest_value(uint32_t h) {
    const float table[16] = {0.0f, -0.0f, 1.0f, -1.0f, 0.5f, -0.5f, 1e-30f, -1e-30f, 1e30f, -1e30f, 3.0e38f, -3.0e38f, 1e-40f, -1e-40f, 2.0f, 1.17549435e-38f};
    if ((h & 3u) == 0) return table[(h >> 2) & 15u];
    const float u = (float)(h >> 8) * (1.0f / 16777216.0f);
    return (h & 4u) ? (u * 2.0f - 1.0f) * 30.0f : (u * 2.0f - 1.0f);
}
__global__ void k_selftest_box(uint32_t n, uint32_t seed, unsigned long long* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t h = rng_absorb(rng_seed(seed), i);
    float v[14];
    for (int k = 0; k < 14; ++k) { h = mix32(h + 0x9e3779b9u); v[k] = selftest_value(h); }
    const float4 lo = make_float4(fminf(v[0], v[3]), fminf(v[1], v[4]), fminf(v[2], v[5]), 0.0f), hi = make_float4(fmaxf(v[0], v[3]), fmaxf(v[1], v[4]), fmaxf(v[2], v[5]), 0.0f);
    f3 o = mk(v[6], v[7], v[8]);
    if ((h & 0x30u) == 0) o.x = lo.x;      // origin exactly on a plane
    if ((h & 0xc0u) == 0) o.y = hi.y;
    const f3 d = mk(v[9], v[10], v[11]);
    const f3 inv = mk(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
    const float tmin = (h & 0x100u) ? 0.0f : 0.001f, tmax = (h & 0x200u) ? finf() : fabsf(v[12]) * 40.0f;
    const bool nx = d.x < 0.0f, ny = d.y < 0.0f, nz = d.z < 0.0f;
    if (!(finite3(o) && finite3(d) && finite3(inv))) { atomicAdd(&out[3], 1ull); return; }
    float ta = 0.0f, tb = 0.0f;
    const bool a = box_hit(lo, hi, o, inv, nx, ny, nz, tmin, tmax, ta), b = box_hit_finite(lo, hi, o, inv, nx, ny, nz, tmin, tmax, tb);
    atomicAdd(&out[0], 1ull);
    if (a) atomicAdd(&out[1], 1ull);
    if (a != b || (a && !(ta == tb))) atomicAdd(&out[2], 1ull);
}
// step_nodes for pair records with box_hit_finite for the lanes whose ray is all-finite (operations per ray, hits, t and
// counters unchanged). The record's two halves are loaded where the lane uses them: hoisting the next record's load to the
// point where a lane first knows its next node makes lanes on different paths of the divergent push / pop code write the
// same registers, and the warp-wide scoreboard then serialises the loads.
template <bool STATS, bool FAST, class Stack>
__device__ __forceinline__ void step_nodes2(TraceState& t, const Stack& stack, Cnt& cnt, int* err) {
    uint32_t cur = t.cur;
    if (cur != ST_POP) {
        const DPair* __restrict__ rec = t.pairs + cur;
        float4 l_lo, l_hi, r_lo, r_hi;
        ldg256(&rec->l_lo, l_lo, l_hi);
        ldg256(&rec->r_lo, r_lo, r_hi);
        if (STATS) cnt.node += 2;
        const uint32_t axis = __float_as_uint(r_lo.w);
        const bool neg = ((t.neg >> axis) & 1u) != 0; // near child = second_child iff d[axis] < 0 (bvh.rs:111-117)
        const uint32_t ref_l = __float_as_uint(l_lo.w), ref_r = __float_as_uint(l_hi.w);
        const bool nx = (t.neg & 1u) != 0, ny = (t.neg & 2u) != 0, nz = (t.neg & 4u) != 0;
        float tl, tr;
        bool hl, hr;
        if (FAST && !t.exact_box) {
            hl = box_hit_finite(l_lo, l_hi, t.o, t.inv, nx, ny, nz, t.tmin, t.tmax, tl);
            hr = box_hit_finite(r_lo, r_hi, t.o, t.inv, nx, ny, nz, t.tmin, t.tmax, tr);
        } else {
            hl = box_hit(l_lo, l_hi, t.o, t.inv, nx, ny, nz, t.tmin, t.tmax, tl);
            hr = box_hit(r_lo, r_hi, t.o, t.inv, nx, ny, nz, t.tmin, t.tmax, tr);
        }
        const bool both = hl && hr;
        cur = both ? (neg ? ref_r : ref_l) : (hl ? ref_l : (hr ? ref_r : ST_POP));
        if (both) {
            if (t.sp >= STACK_DEPTH - 6) { *err = 1; t.sp = 0; cur = ST_DONE; }
            else stack.put(t.sp++, ((unsigned long long)__float_as_uint(neg ? tl : tr) << 32) | (neg ? ref_l : ref_r));
        }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) { // bounded pops (see step_nodes); entry 0 of the stack is the ST_DONE sentinel
        if (cur == ST_POP) {
            const unsigned long long e = stack.get(--t.sp);
            const uint32_t ref = (uint32_t)e;
            if ((ref & ST_INSTANCE) || __uint_as_float((uint32_t)(e >> 32)) < t.tmax) cur = ref;
        }
    }
    t.cur = cur;
}
template <bool HOME>
__device__ __forceinline__ void accept_hit(TraceState& t, const RayHome* home, uint32_t inst, uint32_t prim, float b1, float b2) {
    if (HOME) {
        if (home->type == 0) __stcs(home->hit, make_uint4(inst, prim, __float_as_uint(b1), __float_as_uint(b2)));
        else if (home->type == 2) __stcs(home->a_w, __uint_as_float(inst));
    } else { t.h_prim = prim; t.h_b1 = b1; t.h_b2 = b2; t.h_inst = inst; }
    t.found = true;
}
// WIDE: a mesh leaf reference is REF_LEAF | slot, and the next state is the next slot unless this triangle carries the leaf mark
template <bool STATS, bool HOME = false, bool WIDE = false>
__device__ __forceinline__ void step_triangle(TraceState& t, Cnt& cnt, const RayHome* home = nullptr) {
    const uint32_t cur = t.cur;
    const uint32_t a = WIDE ? (cur & ~REF_TAG) : (cur & 0x01ffffffu), n = (cur >> 25) & 31u;
    uint32_t next = n > 1 ? (REF_LEAF | ((n - 1) << 25) | (a + 1)) : ST_POP;
    if (WIDE || n != 0) {
        const DTri* __restrict__ tri = t.tris + a;
        float4 v0, q0, q1, qpad;
        ldg256(&tri->v0, v0, q0);
        ldg256(&tri->e1, q1, qpad);
        if (WIDE) next = __float_as_uint(q0.w) == TRI_LEAF_END ? ST_POP : cur + 1;
        if (STATS) cnt.tri++;
        const f3 e0 = mk(q0.x, q0.y, q0.z), e1 = mk(q1.x, q1.y, q1.z);
        const f3 s0 = cross3(t.d, e1);
        const float dd = dot3(s0, e0);
        const float div = 1.0f / dd;
        const f3 dv = t.o - mk(v0.x, v0.y, v0.z);
        const float b1 = dot3(dv, s0) * div;
        const f3 s1 = cross3(dv, e0);
        const float b2 = dot3(t.d, s1) * div;
        const float tt = dot3(e1, s1) * div;
        const bool ok = dd != 0.0f && !(b1 < 0.0f || b1 > 1.0f) && !(b2 < 0.0f || b1 + b2 > 1.0f) && !(tt < t.tmin || tt > t.tmax);
        if (ok) {
            t.tmax = tt;
            accept_hit<HOME>(t, home, t.level_inst, __float_as_uint(v0.w), b1, b2);
            if (t.any_hit) { t.sp = 0; next = ST_DONE; } // occlusion only: any accepted hit answers the query
        }
    }
    t.cur = next;
}
// HOME also FUSES the chains of non-node micro-steps every ray goes through (each one otherwise costs the lane a whole
// scheduling cycle of the phased loop): a TLAS leaf pushes all but its first instance and tests that one at once; entering a
// mesh tests the mesh's root box at once with the transformed ray (a miss leaves the traversal state untouched — what
// enter + root miss + pop RETURN + restore amounts to). Operations per ray, their order and the counters are unchanged.
template <bool STATS, bool ANIM, bool HOME = false, class Stack>
__device__ __forceinline__ void step_other(const DScene& sc, TraceState& t, const Stack& stack, Cnt& cnt, const RayHome* home = nullptr) {
    uint32_t cur = t.cur;
    uint32_t next = ST_POP;
    bool inst_now = false;
    if ((cur & REF_TAG) == REF_LEAF) { // TLAS leaf: its instances pop in the reference's order (bvh.rs:95-98)
        const uint32_t a = cur & 0x01ffffffu, n = (cur >> 25) & 31u;
        if (HOME) {
            for (uint32_t k = a + n; k-- > a + 1;) stack.put(t.sp++, ST_INSTANCE | k);
            cur = ST_INSTANCE | a; inst_now = n != 0;
        } else
            for (uint32_t k = a + n; k-- > a;) stack.put(t.sp++, ST_INSTANCE | k);
    } else if (cur == ST_ROOT) {
        const DBvh* bvh = t.bvh;
        if (HOME) bvh = t.level_inst == TRB_MISS ? sc.tlas : &sc.meshes[__ldg(&sc.instances[t.level_inst].mesh)].bvh; // (fused paths never get here for a mesh)
        const float4 lo = __ldg(&bvh->root_lo), hi = __ldg(&bvh->root_hi);
        if (STATS) cnt.node++;
        float te;
        if (box_hit(lo, hi, t.o, t.inv, (t.neg & 1u) != 0, (t.neg & 2u) != 0, (t.neg & 4u) != 0, t.tmin, t.tmax, te)) next = __float_as_uint(t.quad ? hi.w : lo.w);
    } else if (cur == ST_RETURN) {
        if (HOME) { // the world ray, as trace_init made it
            const float4 o4 = __ldcs(home->org), d4 = __ldcs(home->dir);
            t.o = mk(o4.x, o4.y, o4.z); t.d = mk(d4.x, d4.y, d4.z);
            t.inv = mk(1.0f / t.d.x, 1.0f / t.d.y, 1.0f / t.d.z);
        } else { t.o = t.wo; t.d = t.wd; t.inv = t.winv; }
        t.neg = neg_mask(t.d);
        trace_level(t, sc.tlas, sc.tlas_pairs, sc.tlas_quads);
        t.level_inst = TRB_MISS;
    } else inst_now = true;
    if (inst_now) { // Instance::intersect for one entry of a TLAS leaf
        const uint32_t ii = __ldg(&sc.tlas_order[cur & ~REF_TAG]);
        const DInstance& in = sc.instances[ii];
        if (STATS) cnt.inst++;
        const uint32_t kind = __ldg(&in.kind), shape = __ldg(&in.shape);
        if (kind != TRB_INST_EMITTER_POINT) {
            float m[16];
            instance_inv<ANIM>(sc, in, t.time, m, t.xf_row);
            const f3 lo_ = xf_point(m, HOME ? t.o : t.wo), ld_ = xf_vector(m, HOME ? t.d : t.wd); // at the top level the current ray IS the world ray
            if (shape == TRB_SHAPE_MESH) {
                const DMesh& me = sc.meshes[__ldg(&in.mesh)];
                const f3 inv_ = mk(1.0f / ld_.x, 1.0f / ld_.y, 1.0f / ld_.z);
                const uint32_t neg_ = neg_mask(ld_);
                bool enter = true;
                next = ST_ROOT;
                if (HOME) { // BVH<Triangle>::intersect starts by testing its root box: do it now
                    const float4 lo = __ldg(&me.bvh.root_lo), hi = __ldg(&me.bvh.root_hi);
                    if (STATS) cnt.node++;
                    float te;
                    enter = box_hit(lo, hi, lo_, inv_, (neg_ & 1u) != 0, (neg_ & 2u) != 0, (neg_ & 4u) != 0, t.tmin, t.tmax, te);
                    next = enter ? __float_as_uint(lo.w) : ST_POP;
                }
                if (enter) {
                    t.o = lo_; t.d = ld_; t.inv = inv_; t.neg = neg_;
                    trace_level(t, &me.bvh, me.bvh.pairs, me.bvh.quads);
                    t.tris = me.tris; t.level_inst = ii;
                    stack.put(t.sp++, ST_RETURN);
                }
            } else {
                const float p0 = __ldg(&in.p0), p1 = __ldg(&in.p1);
                float tt = t.tmax;
                bool h;
                if (shape == TRB_SHAPE_SPHERE) h = sphere_t(p0, lo_, ld_, t.tmin, tt);
                else if (shape == TRB_SHAPE_DISK) h = disk_t(p0, p1, lo_, ld_, t.tmin, tt);
                else h = rect_t(p0, p1, lo_, ld_, t.tmin, tt);
                if (h) {
                    t.tmax = tt;
                    accept_hit<HOME>(t, home, ii, 0u, 0.0f, 0.0f);
                    if (t.any_hit) { t.sp = 0; next = ST_DONE; }
                }
            }
        }
    }
    t.cur = next;
}

template <bool STATS, bool ANIM, bool WIDE = false>
__device__ __noinline__ bool scene_trace(const DScene& sc, Ray& ray, HitRec& hit, bool any_hit, Cnt& cnt, int* err, float time) {
    TraceState t;
    unsigned long long stack_mem[STACK_DEPTH];
    const LocalStack stack{stack_mem};
    trace_init(sc, t, ray, any_hit, time);
    while (t.cur != ST_DONE) trace_step<STATS, ANIM, WIDE>(sc, t, stack, cnt, err);
    ray.tmax = t.tmax;
    hit.t = t.tmax; hit.inst = t.h_inst; hit.prim = t.h_prim; hit.b1 = t.h_b1; hit.b2 = t.h_b2;
    return t.found;
}

// ------------------------------------------------------------------------------------------
// DifferentialGeometry of the final hit, transformed to world space (receiver.rs:36-41). Only the
// members the integrator reads: p, n, ng, dp_du (u, v feed constant textures only; dp_dv only feeds n).
// ------------------------------------------------------------------------------------------
struct Surf { f3 p, n, ng, dp_du; float u, v; }; // u, v: only filled when the scene has image textures (DScene::n_textures)

// RECORD (ray-query records, k_query_records): the whole DifferentialGeometry — u, v for every shape whatever the scene's
// textures, and dp_dv, transformed to world space into *dp_dv_world. The shading kernels instantiate RECORD = false only.
template <bool ANIM, bool RECORD = false>
__device__ __forceinline__ void surface_at(const DScene& sc, const Ray& ray, const HitRec& hit, Surf& s, float time, const float* xf_row = nullptr,
                                           f3* dp_dv_world = nullptr) {
    const DInstance& in = sc.instances[hit.inst];
    float m[16], w[16];
    instance_inv_mat<ANIM>(sc, in, time, m, w, xf_row);
    const f3 o = xf_point(m, ray.o), d = xf_vector(m, ray.d);
    const f3 p = o + d * hit.t; // ray.at(t) of the local ray
    const uint32_t shape = __ldg(&in.shape);
    f3 n, ng, dp_du;
    f3 dp_dv_rec; // RECORD only
    if (shape == TRB_SHAPE_MESH) {
        const DMesh& me = sc.meshes[__ldg(&in.mesh)];
        const uint32_t ia = __ldg(&me.indices[3 * hit.prim]), ib = __ldg(&me.indices[3 * hit.prim + 1]), ic = __ldg(&me.indices[3 * hit.prim + 2]);
        const float* P = me.positions; const float* N = me.normals; const float* T = me.texcoords;
        const f3 pa = mk(__ldg(P + 3 * ia), __ldg(P + 3 * ia + 1), __ldg(P + 3 * ia + 2));
        const f3 pb = mk(__ldg(P + 3 * ib), __ldg(P + 3 * ib + 1), __ldg(P + 3 * ib + 2));
        const f3 pc = mk(__ldg(P + 3 * ic), __ldg(P + 3 * ic + 1), __ldg(P + 3 * ic + 2));
        const f3 na = mk(__ldg(N + 3 * ia), __ldg(N + 3 * ia + 1), __ldg(N + 3 * ia + 2));
        const f3 nb = mk(__ldg(N + 3 * ib), __ldg(N + 3 * ib + 1), __ldg(N + 3 * ib + 2));
        const f3 nc = mk(__ldg(N + 3 * ic), __ldg(N + 3 * ic + 1), __ldg(N + 3 * ic + 2));
        const float b1 = hit.b1, b2 = hit.b2;
        const float b0 = 1.0f - b1 - b2;
        n = unit(unit(b0 * na + b1 * nb + b2 * nc)); // mesh.rs:174 normalises, DifferentialGeometry::with_normal normalises again
        ng = n;                                      // with_normal: n == ng
        const float tax = __ldg(T + 2 * ia), tay = __ldg(T + 2 * ia + 1), tbx = __ldg(T + 2 * ib), tby = __ldg(T + 2 * ib + 1);
        const float tcx = __ldg(T + 2 * ic), tcy = __ldg(T + 2 * ic + 1);
        s.u = b0 * tax + b1 * tbx + b2 * tcx; s.v = b0 * tay + b1 * tby + b2 * tcy;        // texcoord = bary-lerp (mesh.rs:178)
        const float du0 = tax - tcx, du1 = tbx - tcx, dv0 = tay - tcy, dv1 = tby - tcy; // mesh.rs:182-184
        const float det = du0 * dv1 - dv0 * du1;
        if (det == 0.0f) {
            f3 dp_dv;
            coord_system(unit(cross3(pc - pa, pb - pa)), dp_du, dp_dv); // cross(e[1], e[0])
            if (RECORD) dp_dv_rec = dp_dv;
        } else {
            const float idet = 1.0f / det;
            const f3 dp0 = pa - pc, dp1 = pb - pc;
            dp_du = (dv1 * dp0 - dv0 * dp1) * idet;
            if (RECORD) dp_dv_rec = (-du1 * dp0 + du0 * dp1) * idet;    // mesh.rs:194
        }
    } else if (shape == TRB_SHAPE_SPHERE) {
        n = unit(p); ng = n;                                            // sphere.rs:58, with_normal
        dp_du = mk(-TRB_PI * 2.0f * p.y, TRB_PI * 2.0f * p.x, 0.0f);    // sphere.rs:75
        if (RECORD || sc.n_textures) { // sphere.rs:59-73
            const float radius = __ldg(&in.p0);
            const float theta = dacos(clampf(p.z / radius, -1.0f, 1.0f));
            const float uu = datan2(p.x, p.y) / (2.0f * TRB_PI);
            s.u = uu < 0.0f ? uu + 1.0f : uu; s.v = theta / TRB_PI;
            if (RECORD) { // sphere.rs:64-66,77-78
                const float inv_z = 1.0f / sqrtf(p.x * p.x + p.y * p.y);
                const float cos_phi = p.x * inv_z, sin_phi = p.y * inv_z;
                dp_dv_rec = mk(p.z * cos_phi, p.z * sin_phi, -radius * dsin(theta)) * TRB_PI;
            }
        }
    } else if (shape == TRB_SHAPE_DISK) {
        const float radius = __ldg(&in.p0), inner = __ldg(&in.p1);
        const float hr = sqrtf(p.x * p.x + p.y * p.y);
        dp_du = mk(-TRB_PI * 2.0f * p.y, TRB_PI * 2.0f * p.x, 0.0f);    // disk.rs:71
        const f3 dp_dv = ((inner - radius) / hr) * mk(p.x, p.y, 0.0f);  // disk.rs:72
        n = unit(cross3(dp_du, dp_dv));                                  // DifferentialGeometry::new
        ng = unit(mk(0.0f, 0.0f, 1.0f));
        if (RECORD) dp_dv_rec = dp_dv;
        if (RECORD || sc.n_textures) { // disk.rs:60-70
            float phi = datan2(p.y, p.x);
            if (phi < 0.0f) phi += TRB_PI * 2.0f;
            s.u = phi / (2.0f * TRB_PI); s.v = 1.0f - (hr - inner) / (radius - inner);
        }
    } else {
        const float hw = __ldg(&in.p0) / 2.0f, hh = __ldg(&in.p1) / 2.0f;
        dp_du = mk(hw * 2.0f, 0.0f, 0.0f);                               // rectangle.rs:57-58
        const f3 dp_dv = mk(0.0f, hh * 2.0f, 0.0f);
        n = unit(cross3(dp_du, dp_dv));
        ng = unit(mk(0.0f, 0.0f, 1.0f));
        if (RECORD) dp_dv_rec = dp_dv;
        s.u = (p.x + hw) / (2.0f * hw); s.v = (p.y + hh) / (2.0f * hh);  // rectangle.rs:54-55
    }
    s.p = xf_point(w, p);
    s.n = xf_normal_t(m, n);
    s.ng = xf_normal_t(m, ng);
    s.dp_du = xf_vector(w, dp_du);
    if (RECORD) *dp_dv_world = xf_vector(w, dp_dv_rec);
}

// ------------------------------------------------------------------------------------------
// mc.rs
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void concentric_disk(float u0, float u1, float& ox, float& oy) { // mc.rs:22-51
    float s0 = 2.0f * u0 - 1.0f, s1 = 2.0f * u1 - 1.0f;
    if (s0 == 0.0f && s1 == 0.0f) { ox = s0; oy = s1; return; }
    float radius, theta;
    if (s0 >= -s1) {
        if (s0 > s1) { radius = s0; theta = s1 > 0.0f ? ieee_div(s1, s0) : 8.0f + ieee_div(s1, s0); }
        else { radius = s1; theta = 2.0f - ieee_div(s0, s1); }
    } else if (s0 <= s1) { radius = -s0; theta = 4.0f + ieee_div(s1, s0); }
    else { radius = -s1; theta = 6.0f - ieee_div(s0, s1); }
    theta = theta * TRB_PIO4;
    float sn, cs;
    dsincos(theta, sn, cs);
    ox = radius * cs; oy = radius * sn;
}
__device__ __forceinline__ f3 cos_hemisphere(float u0, float u1) { // mc.rs:11-16
    float dx, dy;
    concentric_disk(u0, u1, dx, dy);
    return mk(dx, dy, ieee_sqrt(fmaxf(0.0f, 1.0f - dx * dx - dy * dy)));
}
__device__ __forceinline__ float power_heuristic(float pf, float pg) { // mc.rs:56-60 with n_f = n_g = 1
    float f = 1.0f * pf, g = 1.0f * pg;
    return ieee_div(f * f, f * f + g * g);
}

// ------------------------------------------------------------------------------------------
// BxDFs (src/bxdf/**). Shading-space vectors; colours are rgb (alpha is never observable).
// ------------------------------------------------------------------------------------------
enum { BX_REFLECTION = 1, BX_TRANSMISSION = 2, BX_DIFFUSE = 4, BX_GLOSSY = 8, BX_SPECULAR = 16 }; // bxdf/mod.rs:37-41
constexpr uint32_t BX_ALL = 31, BX_NON_SPECULAR = BX_DIFFUSE | BX_GLOSSY | BX_REFLECTION | BX_TRANSMISSION;
enum { LK_LAMBERT, LK_OREN_NAYAR, LK_SPEC_REFL, LK_SPEC_TRANS, LK_TS, LK_MT, LK_MERL };
// Compile-time material kind of the split shade kernels' per-bucket instantiations (KIND = a TRB_MAT_* value, -1 = any): with the
// paths bucketed by kind, a kernel that only ever sees one kind is compiled with that kind's lobes alone (fewer live values,
// a fraction of the code). Same functions, same arithmetic: which lobes a Material has is data the specialised code knows already.
__host__ __device__ constexpr bool lk_in(int KIND, int lk) {
    return KIND < 0 ? true
         : KIND == TRB_MAT_MATTE ? (lk == LK_LAMBERT || lk == LK_OREN_NAYAR)
         : KIND == TRB_MAT_PLASTIC ? (lk == LK_LAMBERT || lk == LK_TS)
         : KIND == TRB_MAT_METAL ? lk == LK_TS
         : KIND == TRB_MAT_SPECULAR_METAL ? lk == LK_SPEC_REFL
         : KIND == TRB_MAT_GLASS ? (lk == LK_SPEC_REFL || lk == LK_SPEC_TRANS)
         : KIND == TRB_MAT_ROUGH_GLASS ? (lk == LK_TS || lk == LK_MT)
         : lk == LK_MERL;
}

struct Mat { // DMaterial in registers
    uint32_t type; f3 c0, c1; float roughness, width, eta, on_a, on_b; uint32_t merl_off;
};
__device__ __forceinline__ void load_mat(const DMaterial& m, Mat& o) {
    o.type = __ldg(&m.type);
    o.c0 = mk(__ldg(&m.c0[0]), __ldg(&m.c0[1]), __ldg(&m.c0[2]));
    o.c1 = mk(__ldg(&m.c1[0]), __ldg(&m.c1[1]), __ldg(&m.c1[2]));
    o.roughness = __ldg(&m.roughness); o.width = __ldg(&m.width); o.eta = __ldg(&m.eta);
    o.on_a = __ldg(&m.on_a); o.on_b = __ldg(&m.on_b); o.merl_off = __ldg(&m.merl_off);
}
// ---- image textures (texture/mod.rs:21-41 bilinear_interpolate, image.rs:14-48, animated_image.rs:18-60) ----
__device__ __forceinline__ f3 tex_texel(const DScene& sc, const DImage& im, uint32_t x, uint32_t y) { // Image::get_color: clamp to the last texel, c / 255
    x = min(x, im.width - 1u); y = min(y, im.height - 1u);
    const uchar4 t = __ldg(&sc.texels[im.offset + y * im.width + x]);
    return mk((float)t.x / 255.0f, (float)t.y / 255.0f, (float)t.z / 255.0f);
}
__device__ f3 tex_image_color(const DScene& sc, const DImage& im, float u, float v) { // Image::sample_color
    const float x = u * (float)im.width, y = v * (float)im.height;
    const uint32_t x0 = f2u(x), y0 = f2u(y);
    const f3 s00 = tex_texel(sc, im, x0, y0), s10 = tex_texel(sc, im, x0 + 1u, y0), s01 = tex_texel(sc, im, x0, y0 + 1u), s11 = tex_texel(sc, im, x0 + 1u, y0 + 1u);
    const float sx = x - (float)x0, sy = y - (float)y0;
    return s00 * (1.0f - sx) * (1.0f - sy) + s10 * sx * (1.0f - sy) + s01 * (1.0f - sx) * sy + s11 * sx * sy;
}
__device__ float tex_image_f32(const DScene& sc, const DImage& im, float u, float v) { // Image::sample_f32: channel 0
    const float x = u * (float)im.width, y = v * (float)im.height;
    const uint32_t x0 = f2u(x), y0 = f2u(y);
    const float s00 = tex_texel(sc, im, x0, y0).x, s10 = tex_texel(sc, im, x0 + 1u, y0).x, s01 = tex_texel(sc, im, x0, y0 + 1u).x, s11 = tex_texel(sc, im, x0 + 1u, y0 + 1u).x;
    const float sx = x - (float)x0, sy = y - (float)y0;
    return s00 * (1.0f - sx) * (1.0f - sy) + s10 * sx * (1.0f - sy) + s01 * (1.0f - sx) * sy + s11 * sx * sy;
}
// AnimatedImage::active_keyframes (animated_image.rs:23-37): lo and, between two keyframes, hi (else -1)
__device__ __forceinline__ void tex_active(const DScene& sc, const DTexture& t, float time, uint32_t& lo, int& hi) {
    uint32_t a = 0, b = t.n_images;
    while (a < b) { const uint32_t m = (a + b) / 2; if (__ldg(&sc.images[t.first_image + m].time) < time) a = m + 1; else b = m; }
    if (a < t.n_images && __ldg(&sc.images[t.first_image + a].time) == time) { lo = a; hi = -1; }
    else if (a == t.n_images) { lo = a - 1; hi = -1; }
    else if (a == 0) { lo = 0; hi = -1; }
    else { lo = a - 1; hi = (int)a; }
}
__device__ f3 tex_sample_color(const DScene& sc, uint32_t ti, float u, float v, float time) {
    const DTexture t = sc.textures[ti];
    if (t.n_images == 1) return tex_image_color(sc, sc.images[t.first_image], u, v);
    uint32_t lo; int hi;
    tex_active(sc, t, time, lo, hi);
    const DImage a = sc.images[t.first_image + lo];
    if (hi < 0) return tex_image_color(sc, a, u, v);
    const DImage b = sc.images[t.first_image + hi];
    const float x = (time - a.time) / (b.time - a.time);
    return tex_image_color(sc, a, u, v) * (1.0f - x) + tex_image_color(sc, b, u, v) * x; // linalg::lerp
}
__device__ float tex_sample_f32(const DScene& sc, uint32_t ti, float u, float v, float time) {
    const DTexture t = sc.textures[ti];
    if (t.n_images == 1) return tex_image_f32(sc, sc.images[t.first_image], u, v);
    uint32_t lo; int hi;
    tex_active(sc, t, time, lo, hi);
    const DImage a = sc.images[t.first_image + lo];
    if (hi < 0) return tex_image_f32(sc, a, u, v);
    const DImage b = sc.images[t.first_image + hi];
    const float x = (time - a.time) / (b.time - a.time);
    return tex_image_f32(sc, a, u, v) * (1.0f - x) + tex_image_f32(sc, b, u, v) * x;
}
// Material::bsdf's texture lookups: every parameter = texture.sample_*(hit.dg.u, hit.dg.v, hit.dg.time) (material/*.rs). Scenes without
// image textures (n_textures == 0: a uniform branch) read the constants prepared at scene creation.
__device__ __noinline__ void apply_textures(const DScene& sc, const DMaterial& dm, float u, float v, float time, Mat& o) {
    const uint32_t t0 = __ldg(&dm.tex[0]), t1 = __ldg(&dm.tex[1]), t2 = __ldg(&dm.tex[2]), t3 = __ldg(&dm.tex[3]);
    if (t0) o.c0 = tex_sample_color(sc, t0 - 1, u, v, time);
    if (t1) o.c1 = tex_sample_color(sc, t1 - 1, u, v, time);
    if (t3) o.eta = tex_sample_f32(sc, t3 - 1, u, v, time);
    if (t2) {
        o.roughness = tex_sample_f32(sc, t2 - 1, u, v, time);
        o.width = fmaxf(o.roughness, 0.000001f);              // Beckmann::new (beckmann.rs:19-22)
        float sigma = TRB_PI / 180.0f * o.roughness;          // OrenNayar::new (oren_nayar.rs:26-34), roughness in degrees
        sigma *= sigma;
        o.on_a = 1.0f - 0.5f * sigma / (sigma + 0.33f);
        o.on_b = 0.45f * sigma / (sigma + 0.09f);
    }
}
__device__ __forceinline__ void load_mat_at(const DScene& sc, uint32_t material, float u, float v, float time, Mat& o) {
    const DMaterial& dm = sc.materials[material];
    load_mat(dm, o);
    if (sc.n_textures) apply_textures(sc, dm, u, v, time, o);
}
// The lobes Material::bsdf allocates, in allocation order (material/{matte:52,plastic:59,metal:56,
// specular_metal:49,glass:51,rough_glass:57,merl:88}.rs). Returns false when lobe `i` does not exist.
// Material kind: the template argument where the caller is an instantiation for one kind, else the material's own field
template <int KIND>
__device__ __forceinline__ uint32_t mat_kind(const Mat& m) { return KIND >= 0 ? (uint32_t)KIND : m.type; }
template <int KIND = -1>
__device__ __forceinline__ bool lobe_of(const Mat& m, int i, int& kind, uint32_t& type, f3& col) {
    switch (mat_kind<KIND>(m)) {
        case TRB_MAT_MATTE:
            if (i != 0) return false;
            kind = m.roughness == 0.0f ? LK_LAMBERT : LK_OREN_NAYAR; type = BX_DIFFUSE | BX_REFLECTION; col = m.c0; return true;
        case TRB_MAT_PLASTIC: {
            const bool d = !black(m.c0), g = !black(m.c1);
            if (i == 0 && d) { kind = LK_LAMBERT; type = BX_DIFFUSE | BX_REFLECTION; col = m.c0; return true; }
            if (((i == 0 && !d) || (i == 1 && d)) && g) { kind = LK_TS; type = BX_GLOSSY | BX_REFLECTION; col = m.c1; return true; }
            return false;
        }
        case TRB_MAT_METAL:
            if (i != 0) return false;
            kind = LK_TS; type = BX_GLOSSY | BX_REFLECTION; col = splat(1.0f); return true;
        case TRB_MAT_SPECULAR_METAL:
            if (i != 0) return false;
            kind = LK_SPEC_REFL; type = BX_SPECULAR | BX_REFLECTION; col = splat(1.0f); return true;
        case TRB_MAT_GLASS: {
            const bool r = !black(m.c0), t = !black(m.c1);
            if (i == 0 && r) { kind = LK_SPEC_REFL; type = BX_SPECULAR | BX_REFLECTION; col = m.c0; return true; }
            if (((i == 0 && !r) || (i == 1 && r)) && t) { kind = LK_SPEC_TRANS; type = BX_SPECULAR | BX_TRANSMISSION; col = m.c1; return true; }
            return false;
        }
        case TRB_MAT_ROUGH_GLASS: {
            const bool r = !black(m.c0), t = !black(m.c1);
            if (i == 0 && r) { kind = LK_TS; type = BX_GLOSSY | BX_REFLECTION; col = m.c0; return true; }
            if (((i == 0 && !r) || (i == 1 && r)) && t) { kind = LK_MT; type = BX_GLOSSY | BX_TRANSMISSION; col = m.c1; return true; }
            return false;
        }
        default: // TRB_MAT_MERL
            if (i != 0) return false;
            kind = LK_MERL; type = BX_GLOSSY | BX_REFLECTION; col = splat(0.0f); return true;
    }
}
__device__ __forceinline__ bool type_matches(uint32_t type, uint32_t flags) { return (type & ~flags) == 0; } // is_subset

// trig helpers (bxdf/mod.rs:125-166)
__device__ __forceinline__ float sin2_theta(f3 v) { return fmaxf(0.0f, 1.0f - v.z * v.z); }
__device__ __forceinline__ float sin_theta(f3 v) { return ieee_sqrt(sin2_theta(v)); }
__device__ __forceinline__ float tan_theta(f3 v) { float s2 = sin2_theta(v); return s2 <= 0.0f ? 0.0f : ieee_div(ieee_sqrt(s2), v.z); }
__device__ __forceinline__ float cos_phi(f3 v) { float s = sin_theta(v); return s == 0.0f ? 1.0f : clampf(ieee_div(v.x, s), -1.0f, 1.0f); }
__device__ __forceinline__ float sin_phi(f3 v) { float s = sin_theta(v); return s == 0.0f ? 0.0f : clampf(ieee_div(v.y, s), -1.0f, 1.0f); }
__device__ __forceinline__ bool same_hemi(f3 a, f3 b) { return a.z * b.z > 0.0f; }

// fresnel.rs. Conductor for the metals, Dielectric(1, eta) for glass, Dielectric(1, 1.5) for plastic (Q16).
template <int KIND = -1>
__device__ __forceinline__ void dielectric_etas(const Mat& m, float& ei, float& et) { ei = 1.0f; et = mat_kind<KIND>(m) == TRB_MAT_PLASTIC ? 1.5f : m.eta; }
template <int KIND = -1>
__device__ __forceinline__ f3 fresnel(const Mat& m, float cos_i) {
    if (mat_kind<KIND>(m) == TRB_MAT_METAL || mat_kind<KIND>(m) == TRB_MAT_SPECULAR_METAL) { // fresnel.rs:19-28
        const float c = fabsf(cos_i);
        const f3 eta = m.c0, k = m.c1, one = splat(1.0f);
        const f3 a = (eta * eta + k * k) * c * c;
        const f3 r_par = (a - eta * c * 2.0f + one) / (a + eta * c * 2.0f + one);
        const f3 b = eta * eta + k * k;
        const f3 cc = splat(c * c);
        const f3 r_perp = (b - eta * c * 2.0f + cc) / (b + eta * c * 2.0f + cc);
        return (r_par + r_perp) * 0.5f;
    }
    float eta_i, eta_t;
    dielectric_etas<KIND>(m, eta_i, eta_t);
    const float ci = clampf(cos_i, -1.0f, 1.0f); // fresnel.rs:48-66
    const float ei = ci > 0.0f ? eta_i : eta_t, et = ci > 0.0f ? eta_t : eta_i;
    const float sin_t = ieee_div(ei, et) * ieee_sqrt(fmaxf(0.0f, 1.0f - ci * ci));
    if (sin_t >= 1.0f) return splat(1.0f);
    const float ct = ieee_sqrt(fmaxf(0.0f, 1.0f - sin_t * sin_t));
    const float aci = fabsf(ci);
    const float r_par = ieee_div(et * aci - ei * ct, et * aci + ei * ct); // fresnel.rs:10-14
    const float r_perp = ieee_div(ei * aci - et * ct, ei * aci + et * ct);
    return splat(0.5f * (r_par * r_par + r_perp * r_perp));
}
// microfacet/beckmann.rs
__device__ __forceinline__ float beck_d(float width, f3 wh) { // :26-35
    const float c2 = wh.z * wh.z;
    const float tan_sqr = ieee_div(sin2_theta(wh), c2);
    if (isinf(tan_sqr)) return 0.0f;
    const float c4 = c2 * c2;
    const float w2 = width * width;
    return ieee_div(dexp(ieee_div(-tan_sqr, w2)), TRB_PI * w2 * c4);
}
__device__ __forceinline__ f3 beck_sample(float width, float u0, float u1) { // :36-46
    float ls = dlog(1.0f - u0);
    if (isinf(ls)) ls = 0.0f;
    const float tan2 = -(width * width) * ls;
    const float phi = 2.0f * TRB_PI * u1;
    const float ct = ieee_div(1.0f, ieee_sqrt(1.0f + tan2));
    const float st = ieee_sqrt(fmaxf(0.0f, 1.0f - ct * ct));
    float sn, cs;
    dsincos(phi, sn, cs);
    return mk(st * cs, st * sn, ct); // linalg::spherical_dir
}
__device__ __forceinline__ float beck_pdf(float width, f3 wh) { return fabsf(wh.z) * beck_d(width, wh); }
__device__ __forceinline__ float beck_g1(float width, f3 v) { // :56-64
    const float a = ieee_div(1.0f, width * fabsf(tan_theta(v)));
    if (a < 1.6f) { const float a2 = a * a; return ieee_div(3.535f * a + 2.181f * a2, 1.0f + 2.276f * a + 2.577f * a2); }
    return 1.0f;
}
__device__ __forceinline__ bool refract3(f3 w, f3 n, float eta, f3& out) { // linalg/mod.rs:117-127
    const float c1 = dot3(n, w);
    const float s1 = fmaxf(0.0f, 1.0f - c1 * c1);
    const float s2 = eta * eta * s1;
    if (s2 >= 1.0f) return false;
    const float c2 = ieee_sqrt(1.0f - s2);
    out = eta * -w + (eta * c1 - c2) * n;
    return true;
}
// microfacet_transmission.rs helpers
template <int KIND = -1>
__device__ __forceinline__ void mt_etas(const Mat& m, f3 wo, float& e0, float& e1) { // :33-39
    float ei, et;
    dielectric_etas<KIND>(m, ei, et);
    if (wo.z > 0.0f) { e0 = ei; e1 = et; } else { e0 = et; e1 = ei; }
}
__device__ __forceinline__ float mt_jacobian(f3 wo, f3 wi, f3 wh, float e0, float e1) { // :40-49
    const float ih = dot3(wi, wh), oh = dot3(wo, wh);
    const float s = e1 * ih + e0 * oh;
    const float denom = s * s;
    if (denom != 0.0f) return fabsf(ieee_div(e0 * e0 * fabsf(oh), denom));
    return 0.0f;
}
__device__ __forceinline__ f3 mt_half(f3 wo, f3 wi, float e0, float e1) { return unit(-e1 * wi - e0 * wo); } // :50-52

__device__ __forceinline__ uint32_t merl_index(float val, float mx, uint32_t n) { // bxdf/merl.rs:42-44
    uint32_t i = f2u(val / mx * (float)n);
    return i > n - 1 ? n - 1 : i;
}
__device__ __noinline__ f3 merl_eval(const float* __restrict__ table, f3 wo, f3 wi_in) { // bxdf/merl.rs:47-82
    f3 wi = wi_in;
    f3 wh = wo + wi;
    if (wh.z < 0.0f) { wi = -wi; wh = -wh; }
    if (len2(wh) == 0.0f) return splat(0.0f);
    wh = unit(wh);
    const float theta_h = dacos(clampf(wh.z, -1.0f, 1.0f));
    const float cph = cos_phi(wh), sph = sin_phi(wh), cth = wh.z, sth = sin_theta(wh);
    const f3 whx = mk(cph * cth, sph * cth, -sth), why = mk(-sph, cph, 0.0f);
    const f3 wd = mk(dot3(wi, whx), dot3(wi, why), dot3(wi, wh));
    const float theta_d = dacos(clampf(wd.z, -1.0f, 1.0f));
    float phi_d = datan2(wd.y, wd.x);
    if (phi_d < 0.0f) phi_d = phi_d + TRB_PI * 2.0f;
    if (phi_d > TRB_PI) phi_d = phi_d - TRB_PI;
    const uint32_t ih = merl_index(ieee_sqrt(fmaxf(0.0f, 2.0f * theta_h / TRB_PI)), 1.0f, TRB_MERL_N_THETA_H);
    const uint32_t id = merl_index(theta_d, TRB_PI / 2.0f, TRB_MERL_N_THETA_D);
    const uint32_t ip = merl_index(phi_d, TRB_PI, TRB_MERL_N_PHI_D);
    const uint32_t i = ip + TRB_MERL_N_PHI_D * (id + ih * TRB_MERL_N_THETA_D);
    return mk(__ldg(table + 3 * i), __ldg(table + 3 * i + 1), __ldg(table + 3 * i + 2));
}

template <int KIND = -1>
__device__ f3 lobe_eval(const DScene& sc, const Mat& m, int kind, f3 col, f3 wo, f3 wi) {
    switch (kind) {
        case LK_LAMBERT: if (!lk_in(KIND, LK_LAMBERT)) break; return col * TRB_INV_PI; // lambertian.rs:32-34
        case LK_OREN_NAYAR: if (!lk_in(KIND, LK_OREN_NAYAR)) break; { // oren_nayar.rs:43-61
            const float so = sin_theta(wo), si = sin_theta(wi);
            float max_cos = 0.0f;
            if (si > 1e-4f && so > 1e-4f) max_cos = fmaxf(0.0f, cos_phi(wi) * cos_phi(wo) + sin_phi(wi) * sin_phi(wo));
            float sin_alpha, tan_beta;
            if (fabsf(wi.z) > fabsf(wo.z)) { sin_alpha = so; tan_beta = ieee_div(si, fabsf(wi.z)); }
            else { sin_alpha = si; tan_beta = ieee_div(so, fabsf(wo.z)); }
            return col * TRB_INV_PI * (m.on_a + m.on_b * max_cos * sin_alpha * tan_beta);
        }
        case LK_TS: if (!lk_in(KIND, LK_TS)) break; { // torrance_sparrow.rs:40-56
            const float cto = fabsf(wo.z), cti = fabsf(wi.z);
            if (cto == 0.0f || cti == 0.0f) return splat(0.0f);
            f3 wh = wi + wo;
            if (wh.x == 0.0f && wh.y == 0.0f && wh.z == 0.0f) return splat(0.0f);
            wh = unit(wh);
            const float d = beck_d(m.width, wh);
            const f3 f = fresnel<KIND>(m, dot3(wi, wh));
            const float g = beck_g1(m.width, wi) * beck_g1(m.width, wo);
            return col * f * d * g / (4.0f * cti * cto);
        }
        case LK_MT: if (!lk_in(KIND, LK_MT)) break; { // microfacet_transmission.rs:65-82
            if (same_hemi(wo, wi)) return splat(0.0f);
            if (wo.z == 0.0f || wi.z == 0.0f) return splat(0.0f);
            float e0, e1;
            mt_etas<KIND>(m, wo, e0, e1);
            const f3 wh = mt_half(wo, wi, e0, e1);
            const float d = beck_d(m.width, wh);
            const f3 f = splat(1.0f) - fresnel<KIND>(m, dot3(wi, wh));
            const float g = beck_g1(m.width, wi) * beck_g1(m.width, wo);
            const float ih = dot3(wi, wh);
            const float jac = mt_jacobian(wo, wi, wh, e0, e1);
            return col * ieee_div(fabsf(ih), fabsf(wi.z) * fabsf(wo.z)) * (f * g * d) * jac;
        }
        case LK_MERL: if (!lk_in(KIND, LK_MERL)) break; return merl_eval(sc.merl + m.merl_off, wo, wi);
        default: break; // specular lobes (specular_reflection.rs:38, specular_transmission.rs:38)
    }
    return splat(0.0f);
}
template <int KIND = -1>
__device__ float lobe_pdf(const Mat& m, int kind, f3 wo, f3 wi) {
    switch (kind) {
        case LK_TS: if (!lk_in(KIND, LK_TS)) break; { // torrance_sparrow.rs:73-81
            if (!same_hemi(wo, wi)) return 0.0f;
            const f3 wh = unit(wo + wi);
            const float jac = ieee_div(1.0f, 4.0f * fabsf(dot3(wo, wh)));
            return beck_pdf(m.width, wh) * jac;
        }
        case LK_MT: if (!lk_in(KIND, LK_MT)) break; { // microfacet_transmission.rs:100-108
            if (same_hemi(wo, wi)) return 0.0f;
            float e0, e1;
            mt_etas<KIND>(m, wo, e0, e1);
            const f3 wh = mt_half(wo, wi, e0, e1);
            return beck_pdf(m.width, wh) * mt_jacobian(wo, wi, wh, e0, e1);
        }
        default: break;
    }
    return same_hemi(wo, wi) ? fabsf(wi.z) * TRB_INV_PI : 0.0f; // BxDF::pdf default (bxdf/mod.rs:114-121)
}
template <int KIND = -1>
__device__ void lobe_sample(const DScene& sc, const Mat& m, int kind, f3 col, f3 wo, float u0, float u1, f3& f, f3& wi, float& pdf) {
    switch (kind) {
        case LK_SPEC_REFL: if (!lk_in(KIND, LK_SPEC_REFL)) break; { // specular_reflection.rs:39-50
            wi = mk(-wo.x, -wo.y, wo.z);
            if (wi.z != 0.0f) { f = fresnel<KIND>(m, wo.z) * col / fabsf(wi.z); pdf = 1.0f; }
            else { f = splat(0.0f); pdf = 0.0f; }
            return;
        }
        case LK_SPEC_TRANS: if (!lk_in(KIND, LK_SPEC_TRANS)) break; { // specular_transmission.rs:39-56
            float eta_i, eta_t;
            dielectric_etas<KIND>(m, eta_i, eta_t);
            const bool entering = wo.z > 0.0f;
            const float ei = entering ? eta_i : eta_t, et = entering ? eta_t : eta_i;
            const f3 n = entering ? mk(0.0f, 0.0f, 1.0f) : mk(0.0f, 0.0f, -1.0f);
            f3 r;
            if (refract3(wo, n, ei / et, r)) {
                wi = r;
                const f3 fr = splat(1.0f) - fresnel<KIND>(m, wi.z);
                f = fr * col / fabsf(wi.z); pdf = 1.0f;
            } else { f = splat(0.0f); wi = splat(0.0f); pdf = 0.0f; }
            return;
        }
        case LK_TS: if (!lk_in(KIND, LK_TS)) break; { // torrance_sparrow.rs:57-72
            if (wo.z == 0.0f) { f = splat(0.0f); wi = splat(0.0f); pdf = 0.0f; return; }
            f3 wh = beck_sample(m.width, u0, u1);
            if (!same_hemi(wo, wh)) wh = -wh;
            wi = 2.0f * dot3(wo, wh) * wh - wo; // linalg::reflect
            if (!same_hemi(wo, wi)) { f = splat(0.0f); wi = splat(0.0f); pdf = 0.0f; }
            else { f = lobe_eval<KIND>(sc, m, kind, col, wo, wi); pdf = lobe_pdf<KIND>(m, kind, wo, wi); }
            return;
        }
        case LK_MT: if (!lk_in(KIND, LK_MT)) break; { // microfacet_transmission.rs:83-99
            f3 wh = beck_sample(m.width, u0, u1);
            if (!same_hemi(wo, wh)) wh = -wh;
            float e0, e1;
            mt_etas<KIND>(m, wo, e0, e1);
            f3 r;
            if (refract3(wo, wh, e0 / e1, r) && !same_hemi(wo, r)) { wi = r; f = lobe_eval<KIND>(sc, m, kind, col, wo, wi); pdf = lobe_pdf<KIND>(m, kind, wo, wi); }
            else { f = splat(0.0f); wi = splat(0.0f); pdf = 0.0f; }
            return;
        }
        default: break;
    }
    // BxDF::sample default (bxdf/mod.rs:102-108): Lambertian, Oren-Nayar, Merl
    wi = cos_hemisphere(u0, u1);
    if (wo.z < 0.0f) wi.z *= -1.0f;
    f = lobe_eval<KIND>(sc, m, kind, col, wo, wi); pdf = lobe_pdf<KIND>(m, kind, wo, wi);
}

// bxdf::BSDF (bsdf.rs)
struct Frame { f3 p, n, tan, bitan; };
__device__ __forceinline__ void make_frame(const Surf& s, Frame& fr) { // bsdf.rs:38-44
    fr.n = unit(s.n);
    const f3 bt = unit(s.dp_du);
    fr.tan = cross3(fr.n, bt);
    fr.bitan = cross3(fr.tan, fr.n);
    fr.p = s.p;
}
__device__ __forceinline__ f3 to_shading(const Frame& fr, f3 v) { return mk(dot3(v, fr.bitan), dot3(v, fr.tan), dot3(v, fr.n)); }
__device__ __forceinline__ f3 from_shading(const Frame& fr, f3 v) {
    return mk(fr.bitan.x * v.x + fr.tan.x * v.y + fr.n.x * v.z, fr.bitan.y * v.x + fr.tan.y * v.y + fr.n.y * v.z,
              fr.bitan.z * v.x + fr.tan.z * v.y + fr.n.z * v.z);
}
template <int KIND = -1>
__device__ __noinline__ f3 bsdf_eval(const DScene& sc, const Mat& m, const Frame& fr, f3 wo_w, f3 wi_w, uint32_t flags) { // bsdf.rs:66-78
    const f3 wo = unit(to_shading(fr, wo_w)), wi = unit(to_shading(fr, wi_w));
    if (wo.z * wi.z > 0.0f) flags &= ~(uint32_t)BX_TRANSMISSION; else flags &= ~(uint32_t)BX_REFLECTION;
    f3 acc = splat(0.0f);
#pragma unroll 1
    for (int i = 0; i < 2; ++i) {
        int kind; uint32_t type; f3 col;
        if (lobe_of<KIND>(m, i, kind, type, col) && type_matches(type, flags)) acc = acc + lobe_eval<KIND>(sc, m, kind, col, wo, wi);
    }
    return acc;
}
template <int KIND = -1>
__device__ __noinline__ float bsdf_pdf(const Mat& m, const Frame& fr, f3 wo_w, f3 wi_w, uint32_t flags) { // bsdf.rs:114-125
    const f3 wo = unit(to_shading(fr, wo_w)), wi = unit(to_shading(fr, wi_w));
    float pdf = 0.0f; int n = 0;
#pragma unroll 1
    for (int i = 0; i < 2; ++i) {
        int kind; uint32_t type; f3 col;
        if (lobe_of<KIND>(m, i, kind, type, col) && type_matches(type, flags)) { pdf = pdf + lobe_pdf<KIND>(m, kind, wo, wi); n++; }
    }
    return n > 0 ? ieee_div(pdf, (float)n) : 0.0f;
}
template <int KIND = -1>
__device__ __noinline__ void bsdf_sample(const DScene& sc, const Mat& m, const Frame& fr, f3 wo_w, uint32_t flags, float u0, float u1, float uc,
                                         f3& f, f3& wi_w, float& pdf, uint32_t& sampled) { // bsdf.rs:85-112
    int n_matching = 0;
    for (int i = 0; i < 2; ++i) { int k; uint32_t t; f3 c; if (lobe_of<KIND>(m, i, k, t, c) && type_matches(t, flags)) n_matching++; }
    if (n_matching == 0) { f = splat(0.0f); wi_w = splat(0.0f); pdf = 0.0f; sampled = 0; return; }
    uint32_t comp = f2u(uc * (float)n_matching);
    if (comp > (uint32_t)n_matching - 1) comp = n_matching - 1;
    int kind = 0; uint32_t type = 0; f3 col = splat(0.0f);
    for (int i = 0, k = 0; i < 2; ++i) {
        int kk; uint32_t tt; f3 cc;
        if (lobe_of<KIND>(m, i, kk, tt, cc) && type_matches(tt, flags)) { if ((uint32_t)k == comp) { kind = kk; type = tt; col = cc; break; } k++; }
    }
    const f3 wo = unit(to_shading(fr, wo_w));
    f3 wi;
    lobe_sample<KIND>(sc, m, kind, col, wo, u0, u1, f, wi, pdf);
    if (len2(wi) == 0.0f) { f = splat(0.0f); wi_w = splat(0.0f); pdf = 0.0f; sampled = 0; return; }
    wi_w = unit(from_shading(fr, wi));
    const bool spec = (type & BX_SPECULAR) != 0;
    if (!spec && n_matching > 1) pdf = bsdf_pdf<KIND>(m, fr, wo_w, wi_w, flags);
    if (!spec) f = bsdf_eval<KIND>(sc, m, fr, wo_w, wi_w, flags);
    sampled = type;
}

// ------------------------------------------------------------------------------------------
// Sampleable shapes (sphere.rs:91-141, disk.rs:84-110, rectangle.rs:74-105), object space
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float shape_area(uint32_t shape, float p0, float p1) {
    if (shape == TRB_SHAPE_SPHERE) return 4.0f * TRB_PI * p0;          // sic (Q3)
    if (shape == TRB_SHAPE_DISK) return TRB_PI * (p0 * p0 - p1 * p1);
    return p0 * p1;
}
__device__ __forceinline__ void shape_sample_uniform(uint32_t shape, float p0, float p1, float u0, float u1, f3& p, f3& n) {
    if (shape == TRB_SHAPE_SPHERE) { // sphere.rs:92-95, mc::uniform_sample_sphere
        const float z = 1.0f - 2.0f * u0;
        const float r = ieee_sqrt(fmaxf(0.0f, 1.0f - z * z));
        const float phi = TRB_PI * 2.0f * u1;
        float sn, cs;
        dsincos(phi, sn, cs);
        p = splat(0.0f) + p0 * mk(cs * r, sn * r, z);
        n = unit(p);
    } else if (shape == TRB_SHAPE_DISK) { // disk.rs:85-90 (ignores inner radius, Q4)
        float dx, dy;
        concentric_disk(u0, u1, dx, dy);
        p = mk(dx * p0, dy * p0, 0.0f); n = mk(0.0f, 0.0f, 1.0f);
    } else { // rectangle.rs:77-80
        p = mk(u0 * p0 - p0 / 2.0f, u1 * p1 - p1 / 2.0f, 0.0f); n = mk(0.0f, 0.0f, 1.0f);
    }
}
__device__ void shape_sample(uint32_t shape, float p0, float p1, f3 pt, float u0, float u1, f3& p, f3& n) {
    if (shape != TRB_SHAPE_SPHERE) { shape_sample_uniform(shape, p0, p1, u0, u1, p, n); return; }
    const float dist_sqr = len2(pt - splat(0.0f)); // sphere.rs:99-124
    if (dist_sqr - p0 * p0 < 0.0001f) { shape_sample_uniform(shape, p0, p1, u0, u1, p, n); return; }
    const f3 wz = unit(splat(0.0f) - pt);
    f3 wx, wy;
    coord_system(wz, wx, wy);
    const float ctm = ieee_sqrt(fmaxf(0.0f, 1.0f - ieee_div(p0 * p0, dist_sqr)));
    const float ct = lerpf(u0, ctm, 1.0f); // mc::uniform_sample_cone_frame (mc.rs:77-83)
    const float st = ieee_sqrt(1.0f - ct * ct);
    const float phi = u1 * TRB_PI * 2.0f;
    float sn, cs;
    dsincos(phi, sn, cs);
    const f3 dir = unit(cs * st * wx + sn * st * wy + ct * wz);
    float tmax = finf();
    if (sphere_t(p0, pt, dir, 0.0f, tmax)) { p = pt + dir * tmax; n = unit(p); return; } // (dg.p, dg.ng)
    const float t = dot3(splat(0.0f) - pt, dir);
    p = pt + dir * t;
    n = unit(p);
}
__device__ float shape_pdf(uint32_t shape, float p0, float p1, f3 pt, f3 wi) {
    if (shape == TRB_SHAPE_SPHERE) { // sphere.rs:131-140
        const float dist_sqr = len2(pt - splat(0.0f));
        if (dist_sqr - p0 * p0 < 0.0001f) return ieee_div(1.0f, shape_area(shape, p0, p1));
        const float ctm = ieee_sqrt(fmaxf(0.0f, 1.0f - ieee_div(p0 * p0, dist_sqr)));
        return ieee_div(1.0f, TRB_PI * 2.0f * (1.0f - ctm)); // mc::uniform_cone_pdf
    }
    // disk.rs:97-110 / rectangle.rs:91-104: re-intersect from pt along wi on [0.001, inf)
    float tmax = finf();
    const bool hit = shape == TRB_SHAPE_DISK ? disk_t(p0, p1, pt, wi, 0.001f, tmax) : rect_t(p0, p1, pt, wi, 0.001f, tmax);
    if (!hit) return 0.0f;
    const f3 ph = pt + wi * tmax;
    f3 n; // d.n of DifferentialGeometry::new = normalize(cross(dp_du, dp_dv))
    if (shape == TRB_SHAPE_DISK) {
        const float hr = ieee_sqrt(ph.x * ph.x + ph.y * ph.y);
        const f3 dp_du = mk(-TRB_PI * 2.0f * ph.y, TRB_PI * 2.0f * ph.x, 0.0f);
        const f3 dp_dv = ((p1 - p0) / hr) * mk(ph.x, ph.y, 0.0f);
        n = unit(cross3(dp_du, dp_dv));
    } else {
        const float hw = p0 / 2.0f, hh = p1 / 2.0f;
        n = unit(cross3(mk(hw * 2.0f, 0.0f, 0.0f), mk(0.0f, hh * 2.0f, 0.0f)));
    }
    const f3 w = -wi;
    const float pdf = ieee_div(len2(pt - ph), fabsf(dot3(n, w)) * shape_area(shape, p0, p1));
    return isfinite(pdf) ? pdf : 0.0f;
}

// ------------------------------------------------------------------------------------------
// per-thread sampler state: the LowDiscrepancy sampler (ld.rs) on the counter RNG
// ------------------------------------------------------------------------------------------
struct PathRng {
    uint32_t h;   // hash state after (seed, pixel, sample)
    uint32_t len; // max_depth + 1 (path.rs:48)
    uint32_t off; // LD offset of ld::sample_2d / sample_1d: 0 for LowDiscrepancy (ld.rs:57,62), samples_taken for Adaptive (adaptive.rs:110,115)
    __device__ __forceinline__ uint32_t draw(uint32_t dim) const { return rng_absorb(h, dim); }
    __device__ __forceinline__ void two_d(uint32_t b, uint32_t d0, uint32_t d1, uint32_t dp, float& x, float& y) const {
        const uint32_t i = permute_index(b, len, draw(dp)) + off;
        x = ld_vdc(i, scramble_of(draw(d0)));
        y = ld_sobol(i, scramble_of(draw(d1)));
    }
    __device__ __forceinline__ float one_d(uint32_t b, uint32_t d0, uint32_t dp) const {
        return ld_vdc(permute_index(b, len, draw(dp)) + off, scramble_of(draw(d0)));
    }
};

struct RayCounts { uint32_t primary, shadow, mis, cont; };

// ------------------------------------------------------------------------------------------
// Integrator::estimate_direct (integrator/mod.rs:122-169) with sample_one_light's light choice
// already made; Light impl of Emitter (emitter.rs:160-204); OcclusionTester (light/mod.rs:21-37).
//
// Split in two so the two rays it needs can be traced elsewhere (inline in the megakernel, by the
// trace kernel in the wavefront pipeline) without changing a single operation:
//   direct_setup   everything up to the two rays: the shadow segment + the light-sample term A it
//                  enables, the BSDF-sampled MIS ray + the term B it enables
//   direct_resolve direct = occluded ? 0 : A;  if the MIS ray hit this light facing us: direct += B
// ------------------------------------------------------------------------------------------
struct DirectSetup {
    f3 a, b;             // contributions enabled by the shadow / MIS ray
    f3 shadow_d, mis_d;  // shadow segment p -> light sample (t in [0.001, 0.999]); MIS direction (t in [0.001, inf))
    bool has_shadow, has_mis;
};

template <bool ANIM, int KIND = -1>
__device__ __noinline__ void direct_setup(const DScene& sc, const Mat& m, const Frame& fr, f3 wo, uint32_t li, float l0, float l1, float b0, float b1,
                                          float bc, float time, DirectSetup& ds, const float* xf_row = nullptr) {
    ds.a = splat(0.0f); ds.b = splat(0.0f); ds.shadow_d = splat(0.0f); ds.mis_d = splat(0.0f); ds.has_shadow = false; ds.has_mis = false;
    const DInstance& light = sc.instances[li];
    const uint32_t kind = __ldg(&light.kind), shape = __ldg(&light.shape);
    const float p0 = __ldg(&light.p0), p1 = __ldg(&light.p1);
    f3 emission;
    emission_at<ANIM>(sc, light, time, emission.x, emission.y, emission.z); // self.emission.color(time)
    const bool delta = kind == TRB_INST_EMITTER_POINT;
    float linv[16], lmat[16];
    instance_inv_mat<ANIM>(sc, light, time, linv, lmat, xf_row); // self.transform.transform(time)
    const f3 p = fr.p;
    // --- light.sample_incident(&bsdf.p, ...) ---
    f3 lrad, wi, seg;
    float pdf_light;
    if (delta) { // emitter.rs:169-174
        const f3 pos = xf_point(lmat, splat(0.0f));
        wi = unit(pos - p);
        lrad = emission / len2(pos - p);
        pdf_light = 1.0f;
        seg = pos - p;
    } else { // emitter.rs:175-185 (object-space pdf and direction, Q5)
        const f3 pl = xf_point(linv, p);
        f3 ps, nl;
        shape_sample(shape, p0, p1, pl, l0, l1, ps, nl);
        const f3 wil = unit(ps - pl);
        pdf_light = shape_pdf(shape, p0, p1, pl, wil);
        lrad = dot3(-wil, nl) > 0.0f ? emission : splat(0.0f); // Emitter::radiance
        const f3 pw = xf_point(lmat, ps);
        wi = xf_vector(lmat, wil);
        seg = pw - p;
    }
    if (pdf_light > 0.0f && !black(lrad)) {
        ds.has_shadow = true; ds.shadow_d = seg; // OcclusionTester::test_points: Ray::segment(a, b - a, 0.001, 0.999)
        // evaluated only when unoccluded in the reference; a pure function of the same inputs, so hoisting it is exact
        const f3 f = bsdf_eval<KIND>(sc, m, fr, wo, wi, BX_NON_SPECULAR);
        if (!black(f)) {
            if (delta) ds.a = f * lrad * fabsf(dot3(wi, fr.n)) / pdf_light;
            else {
                const float pdf_bsdf = bsdf_pdf<KIND>(m, fr, wo, wi, BX_NON_SPECULAR);
                const float w = power_heuristic(pdf_light, pdf_bsdf);
                ds.a = f * lrad * fabsf(dot3(wi, fr.n)) * w / pdf_light;
            }
        }
    }
    if (!delta) { // --- BSDF sampling ---
        f3 f, wi2; float pdf_bsdf; uint32_t sampled;
        bsdf_sample<KIND>(sc, m, fr, wo, BX_NON_SPECULAR, b0, b1, bc, f, wi2, pdf_bsdf, sampled);
        if (pdf_bsdf > 0.0f && !black(f)) {
            float w = 1.0f;
            bool go = true;
            if (!(sampled & BX_SPECULAR)) { // light.pdf (emitter.rs:193-203)
                const f3 pl = xf_point(linv, p);
                const f3 wl = unit(xf_vector(linv, wi2));
                const float pl_pdf = shape_pdf(shape, p0, p1, pl, wl);
                if (pl_pdf == 0.0f) go = false; // `return direct_light` (Q7)
                else w = power_heuristic(pdf_bsdf, pl_pdf);
            }
            if (go) {
                ds.has_mis = true; ds.mis_d = wi2; // Ray::segment(p, w_i, 0.001, inf)
                ds.b = f * emission * fabsf(dot3(wi2, fr.n)) * w / pdf_bsdf; // used iff the ray hits this light from its front
            }
        }
    }
}
// Does the MIS ray's hit see the light's emitting side? e.radiance(&-w_i, &h.dg.p, &h.dg.ng) (integrator/mod.rs:156-162)
template <bool ANIM>
__device__ __forceinline__ bool mis_sees_light(const DScene& sc, f3 org, f3 mis_d, uint32_t li, uint32_t hit_inst, float hit_t, float time, const float* xf_row = nullptr) {
    if (hit_inst != li) return false;
    const DInstance& light = sc.instances[li];
    f3 le;
    emission_at<ANIM>(sc, light, time, le.x, le.y, le.z);
    if (black(le)) return false; // `if !li.is_black()`
    Ray mr; mr.o = org; mr.d = mis_d; mr.tmin = 0.001f; mr.tmax = hit_t;
    HitRec mh; mh.t = hit_t; mh.inst = hit_inst; mh.prim = 0; mh.b1 = 0.0f; mh.b2 = 0.0f; // area lights are analytic shapes
    Surf s;
    surface_at<ANIM>(sc, mr, mh, s, time, xf_row);
    return dot3(-mis_d, s.ng) > 0.0f;
}
__device__ __forceinline__ f3 direct_resolve(f3 a, f3 b, bool occluded, bool mis_ok) {
    f3 direct = occluded ? splat(0.0f) : a;
    if (mis_ok) direct = direct + b;
    return direct;
}

// ------------------------------------------------------------------------------------------
// One bounce of Path::illumination (path.rs:69-111) after the vertex has been found: emission,
// BSDF, direct-light setup, next direction, Russian roulette. Shared by both execution shapes.
// ------------------------------------------------------------------------------------------
struct BounceOut {
    DirectSetup ds;
    uint32_t light;      // instance index of the sampled light
    f3 t_before;         // path_throughput multiplying this bounce's direct light
    f3 throughput;       // after the BSDF sample (and Russian roulette)
    f3 next_d;           // ray.child direction
    f3 org;              // bsdf.p
    bool specular, terminate; // terminate: no continuation ray (black f / pdf 0 / RR / max depth)
};
// The three independent parts of a bounce (shared by the fused and the split shade kernels, so both run the same operations):
//   bounce_emission  path.rs:71-76   emitted light seen directly / through specular bounces (Q1: the FIRST hit's normal)
//   bounce_direct    path.rs:78-80   sample_one_light -> estimate_direct's set-up (integrator/mod.rs:106-169)
//   bounce_scatter   path.rs:82-111  BSDF sample for the next direction, throughput, Russian roulette
template <bool ANIM>
__device__ __forceinline__ void bounce_emission(const DScene& sc, uint32_t hit_inst, f3 ray_d, f3 first_ng, uint32_t bounce, bool prev_specular, f3 throughput_in,
                                                float time, f3& illum) {
    const DInstance& in = sc.instances[hit_inst];
    if (bounce == 0 || prev_specular) {
        if (__ldg(&in.kind) != TRB_INST_RECEIVER) {
            const f3 w = -ray_d;
            if (dot3(w, first_ng) > 0.0f) { // Emitter::radiance with the FIRST hit's normal (path.rs:73, Q1)
                f3 le;
                emission_at<ANIM>(sc, in, time, le.x, le.y, le.z);
                illum = illum + throughput_in * le;
            }
        }
    }
}
template <bool ANIM, int KIND = -1>
__device__ __forceinline__ void bounce_direct(const DScene& sc, const Mat& m, const Frame& fr, f3 wo, uint32_t bounce, uint32_t hsample, float time, DirectSetup& ds,
                                              uint32_t& light, const float* xf_row = nullptr, uint32_t ld_off = 0) {
    PathRng rng; rng.h = hsample; rng.len = sc.max_depth + 1; rng.off = ld_off;
    float l0, l1, b0, b1;
    rng.two_d(bounce, S_L0, S_L1, S_L_PERM, l0, l1);
    rng.two_d(bounce, S_B0, S_B1, S_B_PERM, b0, b1);
    const float lc = rng.one_d(bounce, S_LC, S_LC_PERM), bc = rng.one_d(bounce, S_BC, S_BC_PERM);
    uint32_t l = f2u(lc * (float)sc.n_lights); // sample_one_light (integrator/mod.rs:108-110), no xN (Q2)
    if (l > sc.n_lights - 1) l = sc.n_lights - 1;
    light = __ldg(&sc.lights[l]);
    direct_setup<ANIM, KIND>(sc, m, fr, wo, light, l0, l1, b0, b1, bc, time, ds, xf_row);
}
struct ScatterOut { f3 throughput, next_d; bool specular, terminate; };
template <int KIND = -1>
__device__ __forceinline__ void bounce_scatter(const DScene& sc, const Mat& m, const Frame& fr, f3 wo, uint32_t bounce, uint32_t hsample, f3 throughput_in, ScatterOut& o, uint32_t ld_off = 0) {
    PathRng rng; rng.h = hsample; rng.len = sc.max_depth + 1; rng.off = ld_off;
    float q0, q1;
    rng.two_d(bounce, S_P0, S_P1, S_P_PERM, q0, q1);
    const float qc = rng.one_d(bounce, S_PC, S_PC_PERM);
    f3 f, wi; float pdf; uint32_t sampled;
    bsdf_sample<KIND>(sc, m, fr, wo, BX_ALL, q0, q1, qc, f, wi, pdf, sampled);
    o.throughput = throughput_in; o.next_d = splat(0.0f); o.specular = false; o.terminate = true;
    if (black(f) || pdf == 0.0f) return;
    o.specular = (sampled & BX_SPECULAR) != 0;
    f3 t = throughput_in * f * fabsf(dot3(wi, fr.n)) / pdf;
    if (bounce > sc.min_depth) { // Russian roulette (path.rs:97-104), probability may exceed 1 (Q8)
        const float lum = 0.2126f * t.x + 0.7152f * t.y + 0.0722f * t.z;
        const float cont = fmaxf(0.5f, lum);
        if (unit_f32(rng.draw(S_RR + bounce)) > cont) { o.throughput = t; return; }
        t = t / cont;
    }
    o.throughput = t;
    if (bounce == sc.max_depth) return;
    o.next_d = unit(wi); // ray.child(&bsdf.p, &w_i.normalized()), min_t = 0.001
    o.terminate = false;
}
template <bool ANIM>
__device__ __forceinline__ void shade_bounce(const DScene& sc, const Surf& s, uint32_t hit_inst, f3 ray_d, f3 first_ng, uint32_t bounce, bool prev_specular,
                                             uint32_t hsample, f3 throughput_in, float time, f3& illum, BounceOut& o, const float* xf_row = nullptr,
                                             uint32_t ld_off = 0) {
    bounce_emission<ANIM>(sc, hit_inst, ray_d, first_ng, bounce, prev_specular, throughput_in, time, illum);
    Mat m;
    load_mat_at(sc, __ldg(&sc.instances[hit_inst].material), s.u, s.v, time, m);
    Frame fr;
    make_frame(s, fr);
    const f3 wo = -ray_d;
    bounce_direct<ANIM>(sc, m, fr, wo, bounce, hsample, time, o.ds, o.light, xf_row, ld_off);
    o.t_before = throughput_in;
    o.org = fr.p;
    ScatterOut so;
    bounce_scatter(sc, m, fr, wo, bounce, hsample, throughput_in, so, ld_off);
    o.throughput = so.throughput; o.next_d = so.next_d; o.specular = so.specular; o.terminate = so.terminate;
}

// ------------------------------------------------------------------------------------------
// One camera sample, megakernel shape: Camera::generate_ray + Scene::intersect + Path::illumination
// (multithreaded.rs:94-102, path.rs:45-119) with the rays traced inline.
// ------------------------------------------------------------------------------------------
// Returns the ray's time: frame_time = (shutter_close - shutter_open) * time + shutter_open.
template <bool ANIM>
__device__ __forceinline__ float camera_ray(const DScene& sc, float sx, float sy, float tm, Ray& ray) { // camera.rs:150-157
    const f3 pc = xf_point(sc.cam.px_to_cam, mk(sx, sy, 0.0f));
    const f3 pp = mk(sc.cam.scaling[0], sc.cam.scaling[1], sc.cam.scaling[2]) * pc;
    const f3 d = unit(pp);
    const float frame_time = (sc.cam.shutter_close - sc.cam.shutter_open) * tm + sc.cam.shutter_open;
    if (ANIM && sc.cam.animated) { // keyframed camera: cam_world.transform(frame_time) per ray
        float inv[16], mat[16];
        eval_anim_xf(sc, sc.cam.spline_first, sc.cam.n_splines, frame_time, inv, mat);
        ray.o = xf_point(mat, splat(0.0f));
        ray.d = xf_vector(mat, d);
    } else {
        ray.o = xf_point(sc.cam.cam_mat, splat(0.0f));
        ray.d = xf_vector(sc.cam.cam_mat, d);
    }
    ray.tmin = 0.0f; ray.tmax = finf();
    return frame_time;
}

template <bool STATS, bool ANIM, bool WIDE = false>
__device__ f3 radiance_of_sample(const DScene& sc, Ray ray, float time, uint32_t hpix_sample, bool ref_shadow, RayCounts& rc, Cnt& cnt, int* err) {
    HitRec hit;
    rc.primary++;
    if (!scene_trace<STATS, ANIM, WIDE>(sc, ray, hit, false, cnt, err, time)) return splat(0.0f); // multithreaded.rs:101-102
    f3 illum = splat(0.0f), throughput = splat(1.0f);
    bool specular_bounce = false;
    uint32_t bounce = 0;
    Surf s;
    surface_at<ANIM>(sc, ray, hit, s, time);
    const f3 first_ng = s.ng;
    for (;;) {
        BounceOut o;
        shade_bounce<ANIM>(sc, s, hit.inst, ray.d, first_ng, bounce, specular_bounce, hpix_sample, throughput, time, illum, o);
        bool occluded = false, mis_ok = false;
        if (o.ds.has_shadow) {
            Ray sr; sr.o = o.org; sr.d = o.ds.shadow_d; sr.tmin = 0.001f; sr.tmax = 0.999f;
            HitRec sh;
            rc.shadow++;
            occluded = scene_trace<STATS, ANIM, WIDE>(sc, sr, sh, !ref_shadow, cnt, err, time);
        }
        if (o.ds.has_mis) {
            Ray mr; mr.o = o.org; mr.d = o.ds.mis_d; mr.tmin = 0.001f; mr.tmax = finf();
            HitRec mh;
            rc.mis++;
            if (scene_trace<STATS, ANIM, WIDE>(sc, mr, mh, false, cnt, err, time)) mis_ok = mis_sees_light<ANIM>(sc, o.org, o.ds.mis_d, o.light, mh.inst, mh.t, time);
        }
        illum = illum + o.t_before * direct_resolve(o.ds.a, o.ds.b, occluded, mis_ok);
        throughput = o.throughput;
        specular_bounce = o.specular;
        if (o.terminate) break;
        ray.o = o.org; ray.d = o.next_d; ray.tmin = 0.001f; ray.tmax = finf();
        rc.cont++;
        if (!scene_trace<STATS, ANIM, WIDE>(sc, ray, hit, false, cnt, err, time)) break;
        surface_at<ANIM>(sc, ray, hit, s, time);
        bounce += 1;
    }
    return illum;
}

// pixel streams of LowDiscrepancy::get_samples / get_samples_1d (ld.rs:33-64)
struct PixelStreams { uint32_t scr0, scr1, kpos, scrt, ktime, hpix; };
__device__ __forceinline__ PixelStreams pixel_streams(uint32_t seed, uint32_t pixel) {
    PixelStreams p;
    p.hpix = rng_absorb(rng_seed(seed), pixel);
    const uint32_t hs = rng_absorb(p.hpix, PIXEL_STREAM);
    p.scr0 = scramble_of(rng_absorb(hs, PX_POS0));
    p.scr1 = scramble_of(rng_absorb(hs, PX_POS1));
    p.kpos = rng_absorb(hs, PX_POS_PERM);
    p.scrt = scramble_of(rng_absorb(hs, PX_TIME));
    p.ktime = rng_absorb(hs, PX_TIME_PERM);
    return p;
}

__device__ __forceinline__ void flush_stats(DStats* st, const RayCounts& rc, const Cnt& cnt, uint32_t samples, bool with_tests) {
    // warp-aggregate then one atomic per warp per counter
    unsigned long long v[8] = {samples, rc.primary, rc.shadow, rc.mis, rc.cont, cnt.node, cnt.tri, cnt.inst};
    const int n = with_tests ? 8 : 5;
    for (int i = 0; i < n; ++i) {
        unsigned long long x = v[i];
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if ((threadIdx.x & 31) == 0 && x) atomicAdd(&reinterpret_cast<unsigned long long*>(st)[i], x);
    }
}

// RenderTarget::write for one sample (render_target.rs:117-148) into the block's shared-memory tile
// RenderTarget::write hands a sample to a 2x2 lock block only if it lies within filter_pixel_width of the block's write
// range (render_target.rs:104-109) — on top of the per-pixel distance test. For the filters the reference's scenes use
// (reach width/inv_width <= filter_pixel_width) this never rejects and DScene::film_block_filter is 0.
__device__ __forceinline__ bool lock_block_takes(float s, int i, int lo, int hi, int fpw) {
    const int b0 = (i >> 1) << 1; // lock_size = (2, 2)
    const int w0 = max(lo, b0), w1 = min(hi + 1, b0 + 2);
    return s >= (float)(w0 - fpw) && s < (float)(w1 + fpw);
}

// LUM: the lum_w film's sums (include/trb.h "Sample variance"): c = (l, l * l, unused) and the third channel takes w * w
template <bool LUM = false>
__device__ __forceinline__ void splat_sample(const DScene& sc, float4* tile, const float* s_table, int T, int tx0, int ty0, int x_lo, int x_hi, int y_lo,
                                             int y_hi, uint32_t px, uint32_t py, float sx, float sy, f3 c) {
    const float img_x = sx - 0.5f, img_y = sy - 0.5f;
    // conservative loop bounds around the footprint |d| * inv_w <= w; the exact test is inside
    const int ry = (int)ceilf(sc.filter_h / sc.filter_inv_h) + 1, rx = (int)ceilf(sc.filter_w / sc.filter_inv_w) + 1;
    const int iy0 = max(y_lo, (int)py - ry), iy1 = min(y_hi, (int)py + ry + 1);
    const int ix0 = max(x_lo, (int)px - rx), ix1 = min(x_hi, (int)px + rx + 1);
    for (int iy = iy0; iy <= iy1; ++iy) {
        const float fy = fabsf((float)iy - img_y) * sc.filter_inv_h;
        if (fy > sc.filter_h) continue; // sic: normalised distance vs width (A7)
        if (sc.film_block_filter && !lock_block_takes(sy, iy, y_lo, y_hi, sc.fpw_y)) continue;
        const uint32_t fyi = min(f2u(fy * 16.0f), 15u);
        for (int ix = ix0; ix <= ix1; ++ix) {
            const float fx = fabsf((float)ix - img_x) * sc.filter_inv_w;
            if (fx > sc.filter_w) continue;
            if (sc.film_block_filter && !lock_block_takes(sx, ix, x_lo, x_hi, sc.fpw_x)) continue;
            const uint32_t fxi = min(f2u(fx * 16.0f), 15u);
            const float wgt = s_table[fyi * 16 + fxi];
            float* t = reinterpret_cast<float*>(&tile[(iy - ty0) * T + (ix - tx0)]);
            atomicAdd(t + 0, wgt * c.x);
            atomicAdd(t + 1, wgt * c.y);
            atomicAdd(t + 2, LUM ? wgt * wgt : wgt * c.z);
            atomicAdd(t + 3, wgt);
        }
    }
}

// ------------------------------------------------------------------------------------------
// k_render — persistent CTAs pull 8x8 blocks from the Morton-ordered queue with one atomic, exactly
// like the reference's worker threads (block_queue.rs:52-59). 128 threads = 64 pixels x 2 sample
// lanes; a warp is 32 neighbouring pixels at the same sample index (coherent primaries, and the 9x9
// film footprints of its lanes never collide at the same loop offset). The block's film footprint
// (8 + 2*fpw + 1)^2 is accumulated in shared memory and flushed once with global atomics.
// MODE 0: film; MODE 1: write trb_sample records instead (parity).
// ------------------------------------------------------------------------------------------
constexpr int RENDER_THREADS = 128;
constexpr int MAX_TILE = 25; // fpw <= 8

template <bool STATS, int MODE, bool ANIM, bool WIDE = false>
__global__ void __launch_bounds__(RENDER_THREADS) k_render(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, uint32_t flags) {
    extern __shared__ float4 tile[];           // T*T RGBW
    __shared__ float s_table[256];
    __shared__ uint32_t s_item;
    const int T = 9 + 2 * max(sc.fpw_x, sc.fpw_y);
    const bool ref_shadow = (flags & 4u) != 0;
    for (int i = threadIdx.x; i < 256; i += RENDER_THREADS) s_table[i] = sc.filter_table[i];
    RayCounts rc = {0, 0, 0, 0};
    Cnt cnt = {0, 0, 0};
    uint32_t my_samples = 0;
    const uint32_t pix = threadIdx.x & 63, lane_s = threadIdx.x >> 6;
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) s_item = atomicAdd(rp.work_counter, 1u);
        if (MODE == 0) for (int i = threadIdx.x; i < T * T; i += RENDER_THREADS) tile[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
        const uint32_t item = s_item;
        if (item >= rp.n_blocks) break;
        const uint2 blk = rp.blocks[item];
        const uint32_t bx = blk.x * 8, by = blk.y * 8;
        const uint32_t px = bx + (pix & 7), py = by + (pix >> 3); // row-major inside the block (ld.rs:47-52)
        const uint32_t pixel = py * sc.width + px;
        const PixelStreams ps = pixel_streams(rp.seed, pixel);
        // film range of this block (render_target.rs:79-82)
        const int x_lo = max((int)bx - sc.fpw_x, 0), x_hi = min((int)bx + 8 + sc.fpw_x, (int)sc.width - 1);
        const int y_lo = max((int)by - sc.fpw_y, 0), y_hi = min((int)by + 8 + sc.fpw_y, (int)sc.height - 1);
        const int tx0 = (int)bx - sc.fpw_x, ty0 = (int)by - sc.fpw_y;
        for (uint32_t si = rp.sample_first + lane_s; si < rp.sample_first + rp.sample_count; si += 2) {
            const uint32_t ip = permute_index(si, rp.spp, ps.kpos);
            const float sx = ld_vdc(ip, ps.scr0) + (float)px;
            const float sy = ld_sobol(ip, ps.scr1) + (float)py;
            const float tm = ld_vdc(permute_index(si, rp.spp, ps.ktime), ps.scrt);
            Ray ray;
            const float time = camera_ray<ANIM>(sc, sx, sy, tm, ray);
            my_samples++;
            f3 c = radiance_of_sample<STATS, ANIM, WIDE>(sc, ray, time, rng_absorb(ps.hpix, si), ref_shadow, rc, cnt, rp.error_flag);
            c = mk(clampf(c.x, 0.0f, 1.0f), clampf(c.y, 0.0f, 1.0f), clampf(c.z, 0.0f, 1.0f)); // multithreaded.rs:99 (Q12)
            if (MODE == 1) {
                trb_sample* out = reinterpret_cast<trb_sample*>(rp.samples_out) + ((size_t)item * 64 + pix) * rp.sample_count + (si - rp.sample_first);
                out->x = sx; out->y = sy; out->r = c.x; out->g = c.y; out->b = c.z;
            } else {
                splat_sample(sc, tile, s_table, T, tx0, ty0, x_lo, x_hi, y_lo, y_hi, px, py, sx, sy, c);
            }
        }
        if (MODE == 0) {
            __syncthreads();
            for (int i = threadIdx.x; i < T * T; i += RENDER_THREADS) {
                const int ix = tx0 + i % T, iy = ty0 + i / T;
                if (ix < x_lo || ix > x_hi || iy < y_lo || iy > y_hi) continue;
                const float4 v = tile[i];
                if (v.w == 0.0f && v.x == 0.0f && v.y == 0.0f && v.z == 0.0f) continue;
                float* dst = reinterpret_cast<float*>(rp.film + (size_t)iy * sc.width + ix);
                atomicAdd(dst + 0, v.x); atomicAdd(dst + 1, v.y); atomicAdd(dst + 2, v.z); atomicAdd(dst + 3, v.w);
            }
        }
    }
    if (rp.stats) flush_stats(rp.stats, rc, cnt, my_samples, STATS);
}

// ==========================================================================================
// Wavefront execution of the same path (DESIGN.md "Execution shape"). A pass of P camera samples
// lives in HBM as structure-of-arrays path state; per bounce round r:
//     k_wf_trace(r)  one thread per queued ray (continuation / shadow / MIS), lean registers, persistent
//                    warps that fetch 32 rays at a time from the round's queues
//     k_wf_shade(r)  one thread per live path: folds the previous bounce's shadow/MIS results into the
//                    radiance (direct_resolve), then shades the new vertex (shade_bounce) and queues up to
//                    three rays that all start at the vertex
// and finally k_wf_film splats each 8x8 block's samples through shared memory. Every camera sample
// performs exactly the operations of radiance_of_sample(), so results are bit-identical to the
// megakernel and to the oracle whatever the scheduling.
// ==========================================================================================
struct WfState {
    float4* org;     // (vertex = origin of this round's rays, flags)
    float4* cont;    // (continuation / primary direction, hit t)
    uint4* hit;      // continuation hit: (inst, prim, b1, b2)
    float4* shadow;  // (shadow segment, occluded flag)
    float4* mis;     // (MIS direction, hit t)
    float4* a;       // (light-sample term A, MIS hit instance)
    float4* b;       // (BSDF-sample term B, sampled light instance)
    float4* tprev;   // throughput multiplying this bounce's direct light
    float4* thr;     // path throughput
    float4* illum;   // radiance so far
    float4* ng;      // first hit's geometric normal (Q1)
    float4* rad;     // finished, clamped radiance per sample (film mode)
    uint32_t* q_active[2];
    uint32_t* q_ending[2]; // paths that have stopped scattering but still wait for their last shadow / MIS results (fused shade kernel)
    uint32_t* q_cont; uint32_t* q_shadow; uint32_t* q_mis;
    uint32_t* counters; // per round: WF_CNT words
    uint32_t n_paths;
    // ray-queue sorting (DESIGN.md "Ray sorting"): a counting sort of each round's rays by (octant, origin cell)
    uint32_t* q_sorted;  // the round's rays in sorted order: type << 30 | path   (type 0 continuation, 1 shadow, 2 MIS)
    uint32_t* sort_key;  // per queued ray: its bin
    uint32_t* sort_rank; // per queued ray: its arrival rank inside the bin
    uint32_t* sort_hist; // bins: counts (all zero between uses)
    uint32_t* sort_offs; // bins: exclusive prefix sums
    // split shading (k_wf_shade_a -> _b -> _c): the shading frame of the vertex (bsdf.rs:38-44) and the paths that reached it this round
    float4* f_p;         // (frame origin p, hit instance)
    float4* f_n;         // shading normal
    float4* f_t;         // tangent
    float4* f_b;         // bitangent
    uint32_t* q_mid;     // paths to shade this round (survived resolve / termination / miss): WF_MID_BUCKETS lists of n_paths entries, one per
                         // material kind, so that k_wf_shade_b / _c run one material's code at a time (whole warps of one kind, and the
                         // GPU's instruction caches hold one kind's code: the shade kernels are far larger than the instruction cache)
    uint32_t mid_keyed;  // 0: everything in bucket 0 (option shade.sort = 0)
    // keyframed scenes: per path, the evaluated transforms of every keyframed instance (32 floats each: inverse, forward); nullptr: none
    float* xf_tab;
    uint32_t n_anim;
    uint32_t* bounds;    // per round 8 words: min xyz, pad, max xyz, pad of the ray origins queued for that round (order-preserving uint encoding)
};
constexpr uint32_t WF_PATH_MASK = 0x3fffffffu;
constexpr int WF_SORT_MAX_BITS = 6; // origin grid up to 64^3 cells x 8 octants x 3 ray types = 6.3 M bins
enum { WF_N_ACTIVE = 0, WF_N_CONT = 1, WF_N_SHADOW = 2, WF_N_MIS = 3, WF_TRACE_HEAD = 4, WF_SHADE_HEAD = 5, WF_N_MID = 6, WF_SHADE_B_HEAD = 7, WF_SHADE_C_HEAD = 8,
       WF_N_ENDING = 9, WF_ENDING_HEAD = 10,
       WF_N_PATHS = 11, // Adaptive passes: the paths the pass really holds (k_wf_generate_ad), read by k_wf_anim_table<true> / 2<true>
       // split shading with the paths bucketed by material kind (k_wf_shade_a fills, _b and _c drain bucket after bucket)
       WF_MID_K = 12, WF_B_HEAD_K = 20, WF_C_HEAD_K = 28, WF_CNT = 36 };
constexpr uint32_t WF_MID_BUCKETS = 8;
enum { WF_F_SPECULAR = 1u, WF_F_TERMINATE = 2u, WF_F_SHADOW = 4u, WF_F_MIS = 8u };

// sample index p -> block item, pixel, sample (the canonical order of trb_camera_rays / trb_render_samples)
struct SampleId { uint32_t item, pix, si, px, py, pixel; };
__device__ __forceinline__ SampleId sample_id(const DScene& sc, const RenderParams& rp, uint32_t p) {
    SampleId id;
    const uint32_t s = p % rp.sample_count, q = p / rp.sample_count;
    id.pix = q & 63; id.item = q >> 6; id.si = rp.sample_first + s;
    const uint2 blk = rp.blocks[id.item];
    id.px = blk.x * 8 + (id.pix & 7); id.py = blk.y * 8 + (id.pix >> 3);
    id.pixel = id.py * sc.width + id.px;
    return id;
}
__device__ __forceinline__ void sample_position(const RenderParams& rp, const PixelStreams& ps, const SampleId& id, float& sx, float& sy, float& tm) {
    const uint32_t ip = permute_index(id.si, rp.spp, ps.kpos);
    sx = ld_vdc(ip, ps.scr0) + (float)id.px;
    sy = ld_sobol(ip, ps.scr1) + (float)id.py;
    tm = ld_vdc(permute_index(id.si, rp.spp, ps.ktime), ps.scrt);
}
// Adaptive sampler, round r (adaptive.rs:82-117): every round draws fresh scrambles and shuffle keys from the pixel stream
// (seed, pixel, 0xfffffffe - r, dim), next to LowDiscrepancy's (seed, pixel, 0xffffffff, dim); slots stay below 2^25.
__device__ __forceinline__ PixelStreams pixel_streams_round(uint32_t seed, uint32_t pixel, uint32_t round) {
    PixelStreams p;
    p.hpix = rng_absorb(rng_seed(seed), pixel);
    const uint32_t hs = rng_absorb(p.hpix, AD_PIXEL_STREAM0 - round);
    p.scr0 = scramble_of(rng_absorb(hs, PX_POS0));
    p.scr1 = scramble_of(rng_absorb(hs, PX_POS1));
    p.kpos = rng_absorb(hs, PX_POS_PERM);
    p.scrt = scramble_of(rng_absorb(hs, PX_TIME));
    p.ktime = rng_absorb(hs, PX_TIME_PERM);
    return p;
}
// entry s = si - sample_first of the round: position sample_02(perm_count(s) + offset), time vdc(perm_max(s) + offset)
// (thread_work sizes time_samples by max_spp and zips its first entries, multithreaded.rs:76,93-94)
__device__ __forceinline__ void sample_position_ad(const RenderParams& rp, const PixelStreams& ps, const SampleId& id, float& sx, float& sy, float& tm) {
    const uint32_t s = id.si - rp.sample_first;
    const uint32_t ip = permute_index(s, rp.ad_pos_len, ps.kpos) + rp.ld_offset;
    sx = ld_vdc(ip, ps.scr0) + (float)id.px;
    sy = ld_sobol(ip, ps.scr1) + (float)id.py;
    tm = ld_vdc(permute_index(s, rp.ad_time_len, ps.ktime) + rp.ld_offset, ps.scrt);
}
// blocks an Adaptive pass really covers: min(n_blocks, live - b0), 0 when the round's list ends before the pass starts
__device__ __forceinline__ uint32_t ad_pass_blocks(const RenderParams& rp) {
    const uint32_t live = *rp.ad_live;
    return live > rp.ad_b0 ? min(rp.n_blocks, live - rp.ad_b0) : 0u;
}

// warp-aggregated append: every lane of the warp must call it
__device__ __forceinline__ void wf_push(uint32_t* q, uint32_t* counter, bool want, uint32_t value) {
    const unsigned mask = __ballot_sync(0xffffffffu, want);
    if (mask == 0) return;
    const int lane = threadIdx.x & 31, leader = __ffs(mask) - 1;
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(counter, (uint32_t)__popc(mask));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (want) q[base + __popc(mask & ((1u << lane) - 1u))] = value;
}

// the same into one of several lists: lanes with equal keys are grouped (match.any), one atomic per group
__device__ __forceinline__ void wf_push_keyed(uint32_t* q, uint32_t stride, uint32_t* counters, bool want, uint32_t key, uint32_t value) {
    const unsigned mask = __ballot_sync(0xffffffffu, want);
    if (mask == 0 || !want) return;
    const unsigned peers = __match_any_sync(mask, key);
    const int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(&counters[key], (uint32_t)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    q[(size_t)key * stride + base + __popc(peers & ((1u << lane) - 1u))] = value;
}

template <bool ANIM>
__device__ __forceinline__ const float* wf_xf_row(const WfState& wf, uint32_t p) {
    return (ANIM && wf.xf_tab) ? wf.xf_tab + (size_t)p * wf.n_anim * 32 : nullptr;
}
// AnimatedTransform::transform(ray.time) once per (path, keyframed instance) — see instance_inv(). One thread per table entry.
// ADAPT: the pass's path count is the one k_wf_generate_ad found on the device (WF_N_PATHS), not the worst case wf.n_paths.
template <bool ADAPT = false>
__global__ void __launch_bounds__(128) k_wf_anim_table(const __grid_constant__ DScene sc, const __grid_constant__ WfState wf) {
    const size_t n = (size_t)(ADAPT ? wf.counters[WF_N_PATHS] : wf.n_paths) * wf.n_anim;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t p = (uint32_t)(i / wf.n_anim), k = (uint32_t)(i % wf.n_anim);
        const DInstance& in = sc.instances[__ldg(&sc.anim_instances[k])];
        float inv[16], mat[16];
        eval_anim_xf(sc, __ldg(&in.spline_first), __ldg(&in.n_splines), wf.thr[p].w, inv, mat);
        float4* dst = reinterpret_cast<float4*>(wf.xf_tab + i * 32);
#pragma unroll
        for (int q = 0; q < 4; ++q) dst[q] = make_float4(inv[4 * q], inv[4 * q + 1], inv[4 * q + 2], inv[4 * q + 3]);
#pragma unroll
        for (int q = 0; q < 4; ++q) dst[4 + q] = make_float4(mat[4 * q], mat[4 * q + 1], mat[4 * q + 2], mat[4 * q + 3]);
    }
}

// The same table with each DISTINCT keyframed spline evaluated once per path: the instances of a keyframed group carry copies of
// the group's spline (tr15.json: 28 keyframed instances, 8 distinct splines), and a level's transform
// Keyframe::transform(BSpline::point(clamp(time))) depends only on (the spline's content, time). Phase 1: one thread per
// (path, distinct spline) -> shared memory; phase 2: one thread per (path, keyframed instance) composes its stack in the
// reference's order from those and the precomputed one-control-point levels — the operations of trbh::animated_xf, so the rows
// are bit-identical to k_wf_anim_table's.
template <bool ADAPT = false>
__global__ void __launch_bounds__(128) k_wf_anim_table2(const __grid_constant__ DScene sc, const __grid_constant__ WfState wf, uint32_t per_iter) {
    extern __shared__ float s_lvl[]; // [path of this iteration][distinct spline][fwd 16 | inv 16]
    const uint32_t nu = sc.n_uniq_splines;
    const uint32_t n_paths = ADAPT ? wf.counters[WF_N_PATHS] : wf.n_paths; // as in k_wf_anim_table
    for (uint32_t p0 = blockIdx.x * per_iter; p0 < n_paths; p0 += gridDim.x * per_iter) {
        const uint32_t np = min(per_iter, n_paths - p0);
        for (uint32_t i = threadIdx.x; i < np * nu; i += blockDim.x) {
            const uint32_t lp = i / nu, u = i % nu;
            const trb_spline& sp = sc.splines[__ldg(&sc.uniq_splines[u])];
            const float time = wf.thr[p0 + lp].w;
            const float lo = sc.knots[sp.knot_first + sp.degree], hi = sc.knots[sp.knot_first + sp.n_knots - 1 - sp.degree];
            const trbh::Xf t = trbh::keyframe_xf(trbh::spline_point(sp, sc.keyframes, sc.knots, trbh::clampf_hd(time, lo, hi)));
            float* dst = s_lvl + (size_t)i * 32;
#pragma unroll
            for (int q = 0; q < 16; ++q) { dst[q] = t.fwd.m[q]; dst[16 + q] = t.inv.m[q]; }
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < np * wf.n_anim; i += blockDim.x) {
            const uint32_t lp = i / wf.n_anim, k = i % wf.n_anim;
            const DInstance& in = sc.instances[__ldg(&sc.anim_instances[k])];
            const uint32_t first = __ldg(&in.spline_first), count = __ldg(&in.n_splines);
            trbh::Xf acc = trbh::xf_identity();
            for (uint32_t s = first; s < first + count; ++s) {
                trbh::Xf t;
                if (sc.splines[s].n_ctrl == 1) t = sc.level_xf[s];
                else {
                    const float* src = s_lvl + ((size_t)lp * nu + __ldg(&sc.spline_uniq[s])) * 32;
#pragma unroll
                    for (int q = 0; q < 16; ++q) { t.fwd.m[q] = src[q]; t.inv.m[q] = src[16 + q]; }
                }
                acc = trbh::xf_compose(t, acc);
            }
            float4* dst = reinterpret_cast<float4*>(wf.xf_tab + ((size_t)(p0 + lp) * wf.n_anim + k) * 32);
#pragma unroll
            for (int q = 0; q < 4; ++q) dst[q] = make_float4(acc.inv.m[4 * q], acc.inv.m[4 * q + 1], acc.inv.m[4 * q + 2], acc.inv.m[4 * q + 3]);
#pragma unroll
            for (int q = 0; q < 4; ++q) dst[4 + q] = make_float4(acc.fwd.m[4 * q], acc.fwd.m[4 * q + 1], acc.fwd.m[4 * q + 2], acc.fwd.m[4 * q + 3]);
        }
        __syncthreads();
    }
}

// order-preserving float <-> uint (for atomicMin / atomicMax over floats of either sign)
__device__ __forceinline__ uint32_t f_ordered(float f) { const uint32_t u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float f_unordered(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }
// Bounding box of the ray origins a shade round queues, for the next round's sort grid: warp min/max, one atomic per warp and word.
__device__ __forceinline__ void wf_bounds_add(uint32_t* b, bool have, f3 o) {
    float lx = have ? o.x : finf(), ly = have ? o.y : finf(), lz = have ? o.z : finf();
    float hx = have ? o.x : -finf(), hy = have ? o.y : -finf(), hz = have ? o.z : -finf();
    if (__ballot_sync(0xffffffffu, have) == 0) return;
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        lx = fminf(lx, __shfl_xor_sync(0xffffffffu, lx, s)); ly = fminf(ly, __shfl_xor_sync(0xffffffffu, ly, s)); lz = fminf(lz, __shfl_xor_sync(0xffffffffu, lz, s));
        hx = fmaxf(hx, __shfl_xor_sync(0xffffffffu, hx, s)); hy = fmaxf(hy, __shfl_xor_sync(0xffffffffu, hy, s)); hz = fmaxf(hz, __shfl_xor_sync(0xffffffffu, hz, s));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(b + 0, f_ordered(lx)); atomicMin(b + 1, f_ordered(ly)); atomicMin(b + 2, f_ordered(lz));
        atomicMax(b + 4, f_ordered(hx)); atomicMax(b + 5, f_ordered(hy)); atomicMax(b + 6, f_ordered(hz));
    }
}

// ------------------------------------------------------------------------------------------
// Ray sorting. Bounce rays leave the shade kernel in path order, i.e. incoherent: neighbouring lanes of a trace warp
// start in different parts of the scene and head in different directions, so every lane fetches its own BVH records
// (one 32-byte sector per lane per load). Before each trace round
// the round's rays (continuation | shadow | MIS, kept in that order) are counting-sorted by
//     key = ray type, direction octant, Morton code of the origin's cell in a 2^bits grid over the origins' bounding box
// so that a warp's 32 rays share the traversal order (octant) and most of the path from the root to their leaf region:
// lanes then hit the same 128-byte lines. The order of rays never affects a result (each ray writes its own path's
// record), so parity is untouched.   count: key + arrival rank (one atomic per ray)  ->  scan: bin offsets  ->  scatter.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t spread3(uint32_t x) { // 10 bits -> every third bit
    x &= 0x3ffu; x = (x | (x << 16)) & 0x030000ffu; x = (x | (x << 8)) & 0x0300f00fu; x = (x | (x << 4)) & 0x030c30c3u; x = (x | (x << 2)) & 0x09249249u;
    return x;
}
struct RayRef { uint32_t type, p; };
__device__ __forceinline__ RayRef wf_ray_ref(const WfState& wf, uint32_t i, uint32_t n_cont, uint32_t n_shadow) {
    RayRef r;
    if (i < n_cont) { r.type = 0; r.p = wf.q_cont[i]; }
    else if (i < n_cont + n_shadow) { r.type = 1; r.p = wf.q_shadow[i - n_cont]; }
    else { r.type = 2; r.p = wf.q_mis[i - n_cont - n_shadow]; }
    return r;
}
__global__ void __launch_bounds__(256) k_wf_sort_count(const __grid_constant__ WfState wf, uint32_t round, uint32_t bits, uint32_t cell_major) {
    const uint32_t* cnt_r = wf.counters + round * WF_CNT;
    const uint32_t n_cont = cnt_r[WF_N_CONT], n_shadow = cnt_r[WF_N_SHADOW], total = n_cont + n_shadow + cnt_r[WF_N_MIS];
    const uint32_t* b = wf.bounds + round * 8;
    const f3 lo = mk(f_unordered(b[0]), f_unordered(b[1]), f_unordered(b[2])), hi = mk(f_unordered(b[4]), f_unordered(b[5]), f_unordered(b[6]));
    const float cells = (float)(1u << bits);
    const float sx = hi.x > lo.x ? cells / (hi.x - lo.x) : 0.0f, sy = hi.y > lo.y ? cells / (hi.y - lo.y) : 0.0f, sz = hi.z > lo.z ? cells / (hi.z - lo.z) : 0.0f;
    const uint32_t cmax = (1u << bits) - 1u, nb = 8u << (3u * bits);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const RayRef r = wf_ray_ref(wf, i, n_cont, n_shadow);
        const float4 o4 = wf.org[r.p];
        const float4 d4 = r.type == 0 ? wf.cont[r.p] : (r.type == 1 ? wf.shadow[r.p] : wf.mis[r.p]);
        const uint32_t cx = min(cmax, __float2uint_rz(fmaxf(0.0f, (o4.x - lo.x) * sx))), cy = min(cmax, __float2uint_rz(fmaxf(0.0f, (o4.y - lo.y) * sy))),
                       cz = min(cmax, __float2uint_rz(fmaxf(0.0f, (o4.z - lo.z) * sz)));
        const uint32_t m = spread3(cx) | (spread3(cy) << 1) | (spread3(cz) << 2);
        const uint32_t oct = (d4.x < 0.0f ? 1u : 0u) | (d4.y < 0.0f ? 2u : 0u) | (d4.z < 0.0f ? 4u : 0u);
        const uint32_t key = r.type * nb + (cell_major ? ((m << 3) | oct) : ((oct << (3u * bits)) | m));
        wf.sort_key[i] = key;
        wf.sort_rank[i] = atomicAdd(&wf.sort_hist[key], 1u);
    }
}
// Exclusive prefix sum over the 3 * 8 * 8^bits bins, one CTA; leaves the histogram zeroed for the next round.
__global__ void __launch_bounds__(1024) k_wf_sort_scan(const __grid_constant__ WfState wf, uint32_t n_bins) {
    __shared__ uint32_t part[1024];
    const uint32_t chunk = (n_bins + 1023u) / 1024u, b0 = min(n_bins, threadIdx.x * chunk), b1 = min(n_bins, b0 + chunk);
    uint32_t sum = 0;
    for (uint32_t k = b0; k < b1; ++k) sum += wf.sort_hist[k];
    part[threadIdx.x] = sum;
    __syncthreads();
    for (uint32_t s = 1; s < 1024; s <<= 1) { // Hillis-Steele inclusive scan of the 1024 partial sums
        const uint32_t v = threadIdx.x >= s ? part[threadIdx.x - s] : 0u;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = part[threadIdx.x] - sum;
    for (uint32_t k = b0; k < b1; ++k) { const uint32_t c = wf.sort_hist[k]; wf.sort_offs[k] = run; wf.sort_hist[k] = 0u; run += c; }
}
__global__ void __launch_bounds__(256) k_wf_sort_scatter(const __grid_constant__ WfState wf, uint32_t round) {
    const uint32_t* cnt_r = wf.counters + round * WF_CNT;
    const uint32_t n_cont = cnt_r[WF_N_CONT], n_shadow = cnt_r[WF_N_SHADOW], total = n_cont + n_shadow + cnt_r[WF_N_MIS];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const RayRef r = wf_ray_ref(wf, i, n_cont, n_shadow);
        wf.q_sorted[wf.sort_offs[wf.sort_key[i]] + wf.sort_rank[i]] = (r.type << 30) | r.p;
    }
}

template <bool ANIM>
__global__ void __launch_bounds__(256) k_wf_generate(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf) {
    const uint32_t n = wf.n_paths;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const SampleId id = sample_id(sc, rp, p);
        const PixelStreams ps = pixel_streams(rp.seed, id.pixel);
        float sx, sy, tm;
        sample_position(rp, ps, id, sx, sy, tm);
        Ray ray;
        const float time = camera_ray<ANIM>(sc, sx, sy, tm, ray);
        wf.org[p] = make_float4(ray.o.x, ray.o.y, ray.o.z, __uint_as_float(0u));
        wf.cont[p] = make_float4(ray.d.x, ray.d.y, ray.d.z, finf());
        wf.thr[p] = make_float4(1.0f, 1.0f, 1.0f, time); // .w: the path's ray.time (every child ray inherits it)
        wf.illum[p] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        wf.q_cont[p] = p;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        wf.counters[WF_N_ACTIVE] = n; wf.counters[WF_N_CONT] = n;
        if (rp.stats) { atomicAdd(&rp.stats->camera_samples, (unsigned long long)n); }
    }
    if (wf.bounds && blockIdx.x == 0 && threadIdx.x < 64) { // empty origin boxes for every round's sort grid (nullptr: sorting off)
        uint32_t* b = wf.bounds + threadIdx.x * 8;
        b[0] = b[1] = b[2] = b[3] = 0xffffffffu; b[4] = b[5] = b[6] = b[7] = 0u;
    }
}

// Trace round r: the rays queued by shade round r-1 (round 0: the primary rays). Persistent warps: a lane
// whose ray has finished writes its result and, once enough lanes of the warp are idle, the idle lanes
// fetch new rays with one warp-aggregated atomic, so rays of very different lengths (an any-hit shadow
// ray vs. a continuation ray crossing the whole mesh) do not leave the warp mostly empty.
//
// PHASED: the warp alternates bursts of node micro-steps with one non-node micro-step (triangle / root / instance /
// return) that runs only once enough lanes are waiting for one (or no lane has node work left), so triangle tests and
// instance entries execute with several lanes instead of the two that happen to be there, and the scheduling
// ballots are paid once per burst.
template <bool STATS, int MINB, int SMEM_STACK, bool ANIM, bool PHASED, bool QUADS, int PIPE = 0>
__global__ void __launch_bounds__(128, MINB) k_wf_trace(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf,
                                                         uint32_t round, uint32_t flags, int WF_REFILL_IDLE, uint32_t sched, const uint32_t* __restrict__ q_sorted) {
    constexpr bool HOME = PHASED && (PIPE & 32) != 0; // RayHome: world ray and hit record live in the path state, not in registers
    constexpr bool QUERY = (PIPE & 64) != 0;          // ray queries (k_query_load): each ray's [min_t, max_t] is org.w and the direction entry's .w
    constexpr bool WIDE = (PIPE & 128) != 0;          // wide mesh leaf references (trb_device.h DPair)
    uint32_t* cnt_r = wf.counters + round * WF_CNT;
    const uint32_t n_cont = cnt_r[WF_N_CONT], n_shadow = cnt_r[WF_N_SHADOW], n_mis = cnt_r[WF_N_MIS];
    const uint32_t total = n_cont + n_shadow + n_mis;
    const bool shadow_any = (flags & 4u) == 0; // TRB_RENDER_REFERENCE_SHADOW clears it
    const int lane = threadIdx.x & 31;
    const unsigned lt_mask = (1u << lane) - 1u;
    Cnt cnt = {0, 0, 0};
    TraceState t;
    __shared__ unsigned long long s_stack[SMEM_STACK * 128];
    unsigned long long stack_lo[STACK_DEPTH - SMEM_STACK];
    const HybridStack<SMEM_STACK> stack{s_stack + threadIdx.x, stack_lo};
    t.cur = ST_DONE;
    bool have = false, exhausted = false;
    uint32_t p = 0;
    int type = 0;
    for (;;) {
        // ---- retire finished rays ----
        if (HOME && have && t.cur == ST_DONE) { // the direction entries stay as they are: only the result words are written
            if (type == 0) {
                __stcs(&wf.cont[p].w, t.tmax);
                if (!t.found) __stcs(&wf.hit[p], make_uint4(TRB_MISS, 0u, 0u, 0u));
            } else if (type == 1) __stcs(&wf.shadow[p].w, __uint_as_float(t.found ? 1u : 0u));
            else {
                __stcs(&wf.mis[p].w, t.tmax);
                if (!t.found) __stcs(&wf.a[p].w, __uint_as_float(TRB_MISS));
            }
            have = false;
        } else if (have && t.cur == ST_DONE) {
            if (type == 0) {
                __stcs(&wf.cont[p], make_float4(t.wd.x, t.wd.y, t.wd.z, t.tmax));
                __stcs(&wf.hit[p], make_uint4(t.found ? t.h_inst : TRB_MISS, t.h_prim, __float_as_uint(t.h_b1), __float_as_uint(t.h_b2)));
            } else if (type == 1) {
                __stcs(&wf.shadow[p], make_float4(t.wd.x, t.wd.y, t.wd.z, __uint_as_float(t.found ? 1u : 0u)));
            } else {
                __stcs(&wf.mis[p], make_float4(t.wd.x, t.wd.y, t.wd.z, t.tmax));
                float4 a4 = __ldcs(&wf.a[p]);
                a4.w = __uint_as_float(t.found ? t.h_inst : TRB_MISS);
                __stcs(&wf.a[p], a4);
            }
            have = false;
        }
        // ---- refill idle lanes ----
        const unsigned idle = __ballot_sync(0xffffffffu, !have);
        if (idle != 0 && !exhausted && (__popc(idle) >= WF_REFILL_IDLE || idle == 0xffffffffu)) {
            const int leader = __ffs(idle) - 1;
            uint32_t base = 0;
            if (lane == leader) base = atomicAdd(&cnt_r[WF_TRACE_HEAD], (uint32_t)__popc(idle));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (base >= total) exhausted = true;
            else if (!have) {
                const uint32_t i = base + __popc(idle & lt_mask);
                if (i < total) {
                    if (q_sorted) { const uint32_t e = __ldg(&q_sorted[i]); type = (int)(e >> 30); p = e & WF_PATH_MASK; } // sorted by (type, octant, origin cell)
                    else if (i < n_cont) { type = 0; p = wf.q_cont[i]; }
                    else if (i < n_cont + n_shadow) { type = 1; p = wf.q_shadow[i - n_cont]; }
                    else { type = 2; p = wf.q_mis[i - n_cont - n_shadow]; }
                    const float4 o4 = __ldcs(&wf.org[p]);
                    const float4 d4 = __ldcs(type == 0 ? &wf.cont[p] : (type == 1 ? &wf.shadow[p] : &wf.mis[p])); // streamed: keep L2 for the BVH
                    Ray ray; ray.o = mk(o4.x, o4.y, o4.z); ray.d = mk(d4.x, d4.y, d4.z);
                    ray.tmin = QUERY ? o4.w : ((type == 0 && round == 0) ? 0.0f : 0.001f);
                    ray.tmax = QUERY ? d4.w : (type == 1 ? 0.999f : finf());
                    trace_init(sc, t, ray, type == 1 && shadow_any, ANIM ? __ldg(&wf.thr[p].w) : 0.0f, QUADS && PHASED, (flags & WF_TRACE_FORCE_EXACT_BOX) != 0);
                    t.xf_row = wf_xf_row<ANIM>(wf, p);
                    if (PHASED) { stack.put(0, (unsigned long long)ST_DONE); t.sp = 1; } // bottom sentinel: popping it ends the ray
                    if (HOME) { // the TLAS root box is every ray's first test: do it here, with all refilled lanes, instead of as a non-node micro-step
                        const float4 lo = __ldg(&sc.tlas->root_lo), hi = __ldg(&sc.tlas->root_hi);
                        if (STATS) cnt.node++;
                        float te;
                        t.cur = box_hit(lo, hi, t.o, t.inv, (t.neg & 1u) != 0, (t.neg & 2u) != 0, (t.neg & 4u) != 0, t.tmin, t.tmax, te) ? __float_as_uint(lo.w) : ST_POP;
                    }
                    have = true;
                }
            }
        }
        const unsigned busy0 = __ballot_sync(0xffffffffu, have);
        if (busy0 == 0) { if (exhausted) break; else continue; }
        // ---- traverse until enough lanes have finished ----
        if (PHASED) {
            // `sched`: quorum of lanes waiting for a non-node micro-step (triangle / root / instance / return); WF_BURST node
            // micro-steps per scheduling decision. An idle lane has cur == ST_DONE.
            const int thr_o = (int)(sched & 255u);
            for (;;) {
#pragma unroll
                for (int k = 0; k < WF_BURST; ++k)
                    if (trace_is_node(t.cur)) {
                        if (PIPE != 0 && !QUADS) step_nodes2<STATS, (PIPE & 1) != 0>(t, stack, cnt, rp.error_flag);
                        else step_nodes<STATS, QUADS>(t, stack, cnt, rp.error_flag);
                    }
                const bool is_a = trace_is_node(t.cur), is_o = !is_a && t.cur != ST_DONE;
                const unsigned m_a = __ballot_sync(0xffffffffu, is_a), m_o = __ballot_sync(0xffffffffu, is_o);
                if ((m_a | m_o) == 0) break;
                if (!exhausted && 32 - __popc(m_a | m_o) >= WF_REFILL_IDLE) break;
                if (m_o != 0 && (m_a == 0 || __popc(m_o) >= thr_o)) {
                    if (is_o) {
                        const RayHome home{&wf.org[p], type == 0 ? &wf.cont[p] : (type == 1 ? &wf.shadow[p] : &wf.mis[p]), &wf.hit[p], &wf.a[p].w, type};
                        if ((t.cur & REF_TAG) == REF_LEAF && t.level_inst != TRB_MISS) step_triangle<STATS, HOME, WIDE>(t, cnt, &home);
                        else step_other<STATS, ANIM, HOME>(sc, t, stack, cnt, &home);
                    }
                }
            }
        } else {
            for (;;) {
                if (have && t.cur != ST_DONE) trace_step<STATS, ANIM, WIDE>(sc, t, stack, cnt, rp.error_flag);
                const unsigned running = __ballot_sync(0xffffffffu, have && t.cur != ST_DONE);
                if (running == 0) break;
                if (!exhausted && 32 - __popc(running) >= WF_REFILL_IDLE) break;
            }
        }
    }
    if (rp.stats) {
        if (STATS) {
            unsigned long long v[3] = {cnt.node, cnt.tri, cnt.inst};
            for (int k = 0; k < 3; ++k) {
                unsigned long long x = v[k];
                for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
                if (lane == 0 && x) atomicAdd(&rp.stats->node_tests + k, x);
            }
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            atomicAdd(round == 0 ? &rp.stats->rays_primary : &rp.stats->rays_continuation, (unsigned long long)n_cont);
            atomicAdd(&rp.stats->rays_shadow, (unsigned long long)n_shadow);
            atomicAdd(&rp.stats->rays_mis, (unsigned long long)n_mis);
        }
    }
}

// per-sample clamp (multithreaded.rs:99, Q12) and hand-over to the film (MODE 0) or the parity records (MODE 1); MODE 2 (illumination
// queries) keeps the integrator's unclamped radiance: k_illum_reduce clamps on request
__device__ __forceinline__ void finish_sample(const DScene& sc, const RenderParams& rp, const WfState& wf, uint32_t p, f3 illum, int mode) {
    if (mode == 2) { wf.rad[p] = make_float4(illum.x, illum.y, illum.z, 1.0f); return; }
    const f3 c = mk(clampf(illum.x, 0.0f, 1.0f), clampf(illum.y, 0.0f, 1.0f), clampf(illum.z, 0.0f, 1.0f)); // multithreaded.rs:99 (Q12)
    if (mode == 0) wf.rad[p] = make_float4(c.x, c.y, c.z, 1.0f);
    else {
        const SampleId id = sample_id(sc, rp, p);
        const PixelStreams ps = pixel_streams(rp.seed, id.pixel);
        float sx, sy, tm;
        sample_position(rp, ps, id, sx, sy, tm);
        trb_sample* out = reinterpret_cast<trb_sample*>(rp.samples_out) + p;
        out->x = sx; out->y = sy; out->r = c.x; out->g = c.y; out->b = c.z;
    }
}
// Illumination queries (MODE 2 of the shade kernels): k_illum_load leaves each path's stream hash (seed, key, sample) in
// wf.illum[p].w, which the shade kernels carry along instead of deriving it from sample_id, and min_t in wf.org[p].w, which
// round 0 must not read as the path's WF_F_* flags.
template <int MODE>
__device__ __forceinline__ uint32_t wf_flags(float4 o4, uint32_t round) { return (MODE == 2 && round == 0) ? 0u : __float_as_uint(o4.w); }
template <int MODE>
__device__ __forceinline__ uint32_t wf_stream(const DScene& sc, const RenderParams& rp, const WfState& wf, uint32_t p) {
    if (MODE == 2) return __float_as_uint(wf.illum[p].w);
    const SampleId id = sample_id(sc, rp, p);
    return rng_absorb(rng_absorb(rng_seed(rp.seed), id.pixel), id.si);
}

// Shade round r (== bounce r of every live path). MODE 0: finished samples go to wf.rad; MODE 1: to trb_sample records;
// MODE 2: illumination queries, unclamped to wf.rad.
template <int MODE, bool ANIM, int MINB>
__global__ void __launch_bounds__(128, MINB) k_wf_shade(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf,
                                                   uint32_t round) {
    uint32_t* cnt_r = wf.counters + round * WF_CNT;
    uint32_t* cnt_n = wf.counters + (round + 1) * WF_CNT;
    const uint32_t n = cnt_r[WF_N_ACTIVE];
    const uint32_t* __restrict__ act = wf.q_active[round & 1];
    uint32_t* act_next = wf.q_active[(round + 1) & 1];
    uint32_t* ending_next = wf.q_ending[(round + 1) & 1];
    const int lane = threadIdx.x & 31;
    // Paths whose last bounce ended them (black BSDF sample, Russian roulette, max depth) only have the direct light of that bounce
    // left to fold in. They come in their own list so that the warps doing the expensive shading below are not one third empty:
    // this loop is a few loads and one direct_resolve per path.
    if (round > 0) {
        const uint32_t n_end = cnt_r[WF_N_ENDING];
        const uint32_t* __restrict__ ending = wf.q_ending[round & 1];
        for (;;) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(&cnt_r[WF_ENDING_HEAD], 32u);
            base = __shfl_sync(0xffffffffu, base, 0);
            if (base >= n_end) break;
            const uint32_t i = base + lane;
            if (i < n_end) {
                const uint32_t p = ending[i];
                const float4 o4 = wf.org[p];
                const uint32_t fl = __float_as_uint(o4.w);
                const float4 il4 = wf.illum[p];
                const float4 a4 = wf.a[p], b4 = wf.b[p], t4 = wf.tprev[p];
                bool occluded = false, mis_ok = false;
                if (fl & WF_F_SHADOW) occluded = __float_as_uint(wf.shadow[p].w) != 0u;
                if (fl & WF_F_MIS) {
                    const float4 m4 = wf.mis[p];
                    mis_ok = mis_sees_light<ANIM>(sc, mk(o4.x, o4.y, o4.z), mk(m4.x, m4.y, m4.z), __float_as_uint(b4.w), __float_as_uint(a4.w), m4.w, wf.thr[p].w, wf_xf_row<ANIM>(wf, p));
                }
                const f3 illum = mk(il4.x, il4.y, il4.z) + mk(t4.x, t4.y, t4.z) * direct_resolve(mk(a4.x, a4.y, a4.z), mk(b4.x, b4.y, b4.z), occluded, mis_ok);
                finish_sample(sc, rp, wf, p, illum, MODE);
            }
        }
    }
    for (;;) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&cnt_r[WF_SHADE_HEAD], 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= n) break;
        const uint32_t i = base + lane;
        const bool valid = i < n;
        uint32_t p = 0;
        bool push_cont = false, push_shadow = false, push_mis = false, push_active = false, push_ending = false;
        f3 new_org = splat(0.0f);
        if (valid) {
            p = round == 0 ? i : act[i];
            const float4 o4 = wf.org[p];
            const uint32_t fl = wf_flags<MODE>(o4, round);
            const f3 org = mk(o4.x, o4.y, o4.z);
            float4 il4 = wf.illum[p];
            f3 illum = mk(il4.x, il4.y, il4.z);
            bool done = false;
            const float4 th4 = wf.thr[p];
            const float time = th4.w;
            const float* xf_row = wf_xf_row<ANIM>(wf, p);
            if (round > 0) { // fold in the direct light of the previous bounce (estimate_direct's two ray results)
                const float4 a4 = wf.a[p], b4 = wf.b[p], t4 = wf.tprev[p];
                bool occluded = false, mis_ok = false;
                if (fl & WF_F_SHADOW) occluded = __float_as_uint(wf.shadow[p].w) != 0u;
                if (fl & WF_F_MIS) {
                    const float4 m4 = wf.mis[p];
                    mis_ok = mis_sees_light<ANIM>(sc, org, mk(m4.x, m4.y, m4.z), __float_as_uint(b4.w), __float_as_uint(a4.w), m4.w, time, xf_row);
                }
                illum = illum + mk(t4.x, t4.y, t4.z) * direct_resolve(mk(a4.x, a4.y, a4.z), mk(b4.x, b4.y, b4.z), occluded, mis_ok);
                done = (fl & WF_F_TERMINATE) != 0;
            }
            if (!done) {
                const float4 c4 = wf.cont[p];
                const uint4 h4 = wf.hit[p];
                if (h4.x == TRB_MISS) done = true; // primary miss: black sample (multithreaded.rs:101-102); later: `None => break`
                else {
                    Ray ray; ray.o = org; ray.d = mk(c4.x, c4.y, c4.z); ray.tmin = 0.0f; ray.tmax = c4.w;
                    HitRec h; h.t = c4.w; h.inst = h4.x; h.prim = h4.y; h.b1 = __uint_as_float(h4.z); h.b2 = __uint_as_float(h4.w);
                    Surf s;
                    surface_at<ANIM>(sc, ray, h, s, time, xf_row);
                    f3 first_ng;
                    if (round == 0) { first_ng = s.ng; wf.ng[p] = make_float4(s.ng.x, s.ng.y, s.ng.z, 0.0f); }
                    else { const float4 n4 = wf.ng[p]; first_ng = mk(n4.x, n4.y, n4.z); }
                    const uint32_t hs = MODE == 2 ? __float_as_uint(il4.w) : wf_stream<MODE>(sc, rp, wf, p);
                    BounceOut o;
                    shade_bounce<ANIM>(sc, s, h.inst, ray.d, first_ng, round, (fl & WF_F_SPECULAR) != 0, hs, mk(th4.x, th4.y, th4.z), time, illum, o, xf_row, rp.ld_offset);
                    const uint32_t nf = (o.specular ? WF_F_SPECULAR : 0u) | (o.terminate ? WF_F_TERMINATE : 0u) | (o.ds.has_shadow ? WF_F_SHADOW : 0u) |
                                        (o.ds.has_mis ? WF_F_MIS : 0u);
                    push_cont = !o.terminate; push_shadow = o.ds.has_shadow; push_mis = o.ds.has_mis;
                    push_active = push_cont || push_shadow || push_mis;
                    push_ending = push_active && o.terminate; // nothing left to shade: next round only resolves its shadow / MIS rays
                    if (push_active) {
                        new_org = o.org;
                        wf.org[p] = make_float4(o.org.x, o.org.y, o.org.z, __uint_as_float(nf));
                        if (push_cont) wf.cont[p] = make_float4(o.next_d.x, o.next_d.y, o.next_d.z, finf());
                        if (push_shadow) wf.shadow[p] = make_float4(o.ds.shadow_d.x, o.ds.shadow_d.y, o.ds.shadow_d.z, 0.0f);
                        if (push_mis) wf.mis[p] = make_float4(o.ds.mis_d.x, o.ds.mis_d.y, o.ds.mis_d.z, finf());
                        wf.a[p] = make_float4(o.ds.a.x, o.ds.a.y, o.ds.a.z, __uint_as_float(TRB_MISS));
                        wf.b[p] = make_float4(o.ds.b.x, o.ds.b.y, o.ds.b.z, __uint_as_float(o.light));
                        wf.tprev[p] = make_float4(o.t_before.x, o.t_before.y, o.t_before.z, 0.0f);
                        wf.thr[p] = make_float4(o.throughput.x, o.throughput.y, o.throughput.z, time);
                        wf.illum[p] = make_float4(illum.x, illum.y, illum.z, MODE == 2 ? il4.w : 0.0f);
                    } else done = true; // nothing pending: direct light of this bounce is zero, the path ends here
                }
            }
            if (done && MODE == 2) finish_sample(sc, rp, wf, p, illum, MODE);
            else if (done) { // per-sample clamp (multithreaded.rs:99, Q12) and hand-over to the film
                const f3 c = mk(clampf(illum.x, 0.0f, 1.0f), clampf(illum.y, 0.0f, 1.0f), clampf(illum.z, 0.0f, 1.0f));
                if (MODE == 0) wf.rad[p] = make_float4(c.x, c.y, c.z, 1.0f);
                else {
                    const SampleId id = sample_id(sc, rp, p);
                    const PixelStreams ps = pixel_streams(rp.seed, id.pixel);
                    float sx, sy, tm;
                    sample_position(rp, ps, id, sx, sy, tm);
                    trb_sample* out = reinterpret_cast<trb_sample*>(rp.samples_out) + p;
                    out->x = sx; out->y = sy; out->r = c.x; out->g = c.y; out->b = c.z;
                }
            }
        }
        wf_push(wf.q_cont, &cnt_n[WF_N_CONT], push_cont, p);
        wf_push(wf.q_shadow, &cnt_n[WF_N_SHADOW], push_shadow, p);
        wf_push(wf.q_mis, &cnt_n[WF_N_MIS], push_mis, p);
        wf_push(act_next, &cnt_n[WF_N_ACTIVE], push_active && !push_ending, p);
        wf_push(ending_next, &cnt_n[WF_N_ENDING], push_ending, p);
        if (wf.bounds) wf_bounds_add(wf.bounds + (round + 1) * 8, push_active, new_org); // ray sorting's origin boxes (nullptr: sorting off)
    }
}

// ------------------------------------------------------------------------------------------
// The two other integrators of the reference (SURVEY 8f N4): Whitted (integrator/whitted.rs:41-70 with
// Integrator::specular_reflection / specular_transmission, integrator/mod.rs:41-103) and NormalsDebug
// (integrator/normals_debug.rs:28-36). Not the performance path: one thread per camera sample, the recursion of the
// reference kept as a recursion (post-order float sums must associate exactly like the Rust code), rays traced inline.
// Sampler: every call of the reference asks for fresh 1-element arrays; node n of the recursion tree (root 1, reflection
// child 2n, transmission child 2n + 1) draws dimension S_WHITTED + 8n + slot of the camera sample's stream (detmath contract).
// ------------------------------------------------------------------------------------------
constexpr uint32_t S_WHITTED = 4096;
__device__ __forceinline__ void whitted_2d(uint32_t hs, uint32_t node, uint32_t slot, float& x, float& y) {
    x = ld_vdc(0, scramble_of(rng_absorb(hs, S_WHITTED + 8 * node + slot)));
    y = ld_sobol(0, scramble_of(rng_absorb(hs, S_WHITTED + 8 * node + slot + 1)));
}
__device__ __forceinline__ float whitted_1d(uint32_t hs, uint32_t node, uint32_t slot) { return ld_vdc(0, scramble_of(rng_absorb(hs, S_WHITTED + 8 * node + slot))); }

// Light::sample_incident of Emitter (emitter.rs:160-190): radiance arriving at p, direction, pdf and the occlusion segment
template <bool ANIM>
__device__ __noinline__ void light_sample_incident(const DScene& sc, uint32_t li, f3 p, float u0, float u1, float time, f3& lrad, f3& wi, float& pdf, f3& seg) {
    const DInstance& light = sc.instances[li];
    const uint32_t kind = __ldg(&light.kind), shape = __ldg(&light.shape);
    const float p0 = __ldg(&light.p0), p1 = __ldg(&light.p1);
    f3 emission;
    emission_at<ANIM>(sc, light, time, emission.x, emission.y, emission.z);
    float linv[16], lmat[16];
    instance_inv_mat<ANIM>(sc, light, time, linv, lmat);
    if (kind == TRB_INST_EMITTER_POINT) { // emitter.rs:169-174
        const f3 pos = xf_point(lmat, splat(0.0f));
        wi = unit(pos - p);
        lrad = emission / len2(pos - p);
        pdf = 1.0f;
        seg = pos - p;
        return;
    }
    const f3 pl = xf_point(linv, p); // emitter.rs:175-185 (object-space pdf and direction, Q5)
    f3 ps, nl;
    shape_sample(shape, p0, p1, pl, u0, u1, ps, nl);
    const f3 wil = unit(ps - pl);
    pdf = shape_pdf(shape, p0, p1, pl, wil);
    lrad = dot3(-wil, nl) > 0.0f ? emission : splat(0.0f);
    const f3 pw = xf_point(lmat, ps);
    wi = xf_vector(lmat, wil);
    seg = pw - p;
}

template <bool ANIM, bool WIDE = false>
__device__ f3 whitted_illum(const DScene& sc, const Ray& ray, uint32_t depth, const HitRec& hit, uint32_t node, uint32_t hs, float time, bool ref_shadow,
                            RayCounts& rc, Cnt& cnt, int* err) {
    Surf s;
    surface_at<ANIM>(sc, ray, hit, s, time);
    const DInstance& in = sc.instances[hit.inst];
    Mat m;
    load_mat_at(sc, __ldg(&in.material), s.u, s.v, time, m);
    Frame fr;
    make_frame(s, fr);
    const f3 wo = -ray.d;
    float u0, u1;
    whitted_2d(hs, node, 0, u0, u1);
    f3 illum = splat(0.0f);
    if (depth == 0 && __ldg(&in.kind) != TRB_INST_RECEIVER) { // whitted.rs:49-54
        if (dot3(-ray.d, s.ng) > 0.0f) { f3 le; emission_at<ANIM>(sc, in, time, le.x, le.y, le.z); illum = illum + le; }
        else illum = illum + splat(0.0f);
    }
    for (uint32_t k = 0; k < sc.n_lights; ++k) { // whitted.rs:56-62: every light, the same 2-D sample
        f3 lrad, wi, seg; float pdf;
        light_sample_incident<ANIM>(sc, __ldg(&sc.lights[k]), s.p, u0, u1, time, lrad, wi, pdf, seg);
        const f3 f = bsdf_eval(sc, m, fr, wo, wi, BX_ALL);
        if (!black(lrad) && !black(f)) {
            Ray sr; sr.o = s.p; sr.d = seg; sr.tmin = 0.001f; sr.tmax = 0.999f;
            HitRec sh;
            rc.shadow++;
            if (!scene_trace<true, ANIM, WIDE>(sc, sr, sh, !ref_shadow, cnt, err, time)) illum = illum + f * lrad * fabsf(dot3(wi, fr.n)) / pdf;
        }
    }
    if (depth < sc.max_depth) {
#pragma unroll 1
        for (int which = 0; which < 2; ++which) { // specular_reflection, then specular_transmission (integrator/mod.rs:41-103)
            const uint32_t flags = BX_SPECULAR | (which == 0 ? BX_REFLECTION : BX_TRANSMISSION), slot = which == 0 ? 2u : 5u;
            float v0, v1;
            whitted_2d(hs, node, slot, v0, v1);
            const float vc = whitted_1d(hs, node, slot + 2);
            f3 f, wi; float pdf; uint32_t sampled;
            bsdf_sample(sc, m, fr, wo, flags, v0, v1, vc, f, wi, pdf, sampled);
            f3 out = splat(0.0f);
            if (pdf > 0.0f && !black(f) && fabsf(dot3(wi, fr.n)) != 0.0f) {
                Ray r2; r2.o = fr.p; r2.d = wi; r2.tmin = 0.001f; r2.tmax = finf();
                HitRec h2;
                rc.cont++;
                if (scene_trace<true, ANIM, WIDE>(sc, r2, h2, false, cnt, err, time)) {
                    const f3 li = whitted_illum<ANIM, WIDE>(sc, r2, depth + 1, h2, 2 * node + (uint32_t)which, hs, time, ref_shadow, rc, cnt, err);
                    out = f * li * fabsf(dot3(wi, fr.n)) / pdf;
                }
            }
            illum = illum + out;
        }
    }
    return illum;
}

// One camera sample per thread for the Whitted / NormalsDebug integrators; radiance to wf.rad (MODE 0, then the film kernel) or to trb_sample records (MODE 1).
// MODE 2 (illumination queries): path p is sample p % rp.spp of the caller's ray rays[p / rp.spp], whose key and sample index key the
// streams; the unclamped radiance goes to rad[p] (then k_illum_reduce).
template <int MODE, bool ANIM, bool WIDE = false>
__global__ void __launch_bounds__(128) k_simple_integrator(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, float4* rad, uint32_t n_paths,
                                                           uint32_t integrator, uint32_t flags, const trb_illum_ray* __restrict__ rays) {
    RayCounts rc = {0, 0, 0, 0};
    Cnt cnt = {0, 0, 0};
    uint32_t mine = 0;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n_paths; p += gridDim.x * blockDim.x) {
        Ray ray;
        float time, sx = 0.0f, sy = 0.0f;
        uint32_t hpix, si;
        if (MODE == 2) {
            const trb_illum_ray& q = rays[p / rp.spp];
            ray.o = mk(q.o[0], q.o[1], q.o[2]); ray.d = mk(q.d[0], q.d[1], q.d[2]); ray.tmin = q.min_t; ray.tmax = q.max_t;
            time = q.time;
            hpix = rng_absorb(rng_seed(rp.seed), q.key); si = q.sample + p % rp.spp;
        } else {
            const SampleId id = sample_id(sc, rp, p);
            const PixelStreams ps = pixel_streams(rp.seed, id.pixel);
            hpix = ps.hpix; si = id.si;
            float tm;
            sample_position(rp, ps, id, sx, sy, tm);
            time = camera_ray<ANIM>(sc, sx, sy, tm, ray);
        }
        mine++; rc.primary++;
        HitRec hit;
        f3 c = splat(0.0f);
        if (scene_trace<true, ANIM, WIDE>(sc, ray, hit, false, cnt, rp.error_flag, time)) {
            if (integrator == TRB_INTEGRATOR_NORMALS_DEBUG) { // (bsdf.n + 1) / 2
                Surf s;
                surface_at<ANIM>(sc, ray, hit, s, time);
                Frame fr;
                make_frame(s, fr);
                c = (fr.n + splat(1.0f)) / 2.0f;
            } else c = whitted_illum<ANIM, WIDE>(sc, ray, 0, hit, 1, rng_absorb(hpix, si), time, (flags & 4u) != 0, rc, cnt, rp.error_flag);
        }
        if (MODE == 2) { rad[p] = make_float4(c.x, c.y, c.z, 1.0f); continue; }
        c = mk(clampf(c.x, 0.0f, 1.0f), clampf(c.y, 0.0f, 1.0f), clampf(c.z, 0.0f, 1.0f)); // multithreaded.rs:99 (Q12)
        if (MODE == 0) rad[p] = make_float4(c.x, c.y, c.z, 1.0f);
        else { trb_sample* out = reinterpret_cast<trb_sample*>(rp.samples_out) + p; out->x = sx; out->y = sy; out->r = c.x; out->g = c.y; out->b = c.z; }
    }
    if (rp.stats) flush_stats(rp.stats, rc, cnt, mine, true);
}

// ------------------------------------------------------------------------------------------
// Split shading: the same bounce as k_wf_shade in three kernels, so that each part keeps fewer values live (the fused
// kernel needs 128 registers: 4 CTAs per SM, 25 % of the warp slots) and its code stays resident in the instruction cache.
//   k_wf_shade_a  fold the previous bounce's shadow / MIS results into the radiance (direct_resolve), end terminated or
//                 escaped paths, else build the vertex: surface_at, emission (Q1), shading frame -> f_p/f_n/f_t/f_b, q_mid
//   k_wf_shade_b  direct lighting set-up of the vertex: light choice, direct_setup -> A, B, shadow and MIS rays
//   k_wf_shade_c  BSDF sample, throughput, Russian roulette -> continuation ray; decides whether the path goes on
// Every value is computed by the same device functions in the same order as in the fused kernel: bit-identical results.
// ------------------------------------------------------------------------------------------
// the shading frame k_wf_shade_a left: f_p.w the hit's material index, f_n.w / f_t.w the hit's (u, v), f_b.w the path's stream hash
__device__ __forceinline__ void load_frame(const WfState& wf, uint32_t p, Frame& fr, uint32_t& material, uint32_t& hs, float& u, float& v) {
    const float4 a = wf.f_p[p], n = wf.f_n[p], t = wf.f_t[p], b = wf.f_b[p];
    fr.p = mk(a.x, a.y, a.z); material = __float_as_uint(a.w); u = n.w; v = t.w; hs = __float_as_uint(b.w);
    fr.n = mk(n.x, n.y, n.z); fr.tan = mk(t.x, t.y, t.z); fr.bitan = mk(b.x, b.y, b.z);
}

template <int MODE, bool ANIM, int MINB>
__global__ void __launch_bounds__(128, MINB) k_wf_shade_a(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf,
                                                     uint32_t round) {
    uint32_t* cnt_r = wf.counters + round * WF_CNT;
    const uint32_t n = cnt_r[WF_N_ACTIVE];
    const uint32_t* __restrict__ act = wf.q_active[round & 1];
    const int lane = threadIdx.x & 31;
    for (;;) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&cnt_r[WF_SHADE_HEAD], 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= n) break;
        const uint32_t i = base + lane;
        uint32_t p = 0, mid_key = 0;
        bool push_mid = false;
        if (i < n) {
            p = round == 0 ? i : act[i];
            const float4 o4 = wf.org[p];
            const uint32_t fl = wf_flags<MODE>(o4, round);
            const f3 org = mk(o4.x, o4.y, o4.z);
            const float4 il4 = wf.illum[p];
            f3 illum = mk(il4.x, il4.y, il4.z);
            bool done = false;
            const float4 th4 = wf.thr[p];
            const float time = th4.w;
            const float* xf_row = wf_xf_row<ANIM>(wf, p);
            if (round > 0) { // fold in the direct light of the previous bounce (estimate_direct's two ray results)
                const float4 a4 = wf.a[p], b4 = wf.b[p], t4 = wf.tprev[p];
                bool occluded = false, mis_ok = false;
                if (fl & WF_F_SHADOW) occluded = __float_as_uint(wf.shadow[p].w) != 0u;
                if (fl & WF_F_MIS) {
                    const float4 m4 = wf.mis[p];
                    mis_ok = mis_sees_light<ANIM>(sc, org, mk(m4.x, m4.y, m4.z), __float_as_uint(b4.w), __float_as_uint(a4.w), m4.w, time, xf_row);
                }
                illum = illum + mk(t4.x, t4.y, t4.z) * direct_resolve(mk(a4.x, a4.y, a4.z), mk(b4.x, b4.y, b4.z), occluded, mis_ok);
                done = (fl & WF_F_TERMINATE) != 0;
            }
            if (!done) {
                const float4 c4 = wf.cont[p];
                const uint4 h4 = wf.hit[p];
                if (h4.x == TRB_MISS) done = true; // primary miss: black sample (multithreaded.rs:101-102); later: `None => break`
                else {
                    const uint32_t material = __ldg(&sc.instances[h4.x].material); // handed to _b / _c in f_p.w
                    Ray ray; ray.o = org; ray.d = mk(c4.x, c4.y, c4.z); ray.tmin = 0.0f; ray.tmax = c4.w;
                    HitRec h; h.t = c4.w; h.inst = h4.x; h.prim = h4.y; h.b1 = __uint_as_float(h4.z); h.b2 = __uint_as_float(h4.w);
                    Surf s;
                    surface_at<ANIM>(sc, ray, h, s, time, xf_row);
                    f3 first_ng;
                    if (round == 0) { first_ng = s.ng; wf.ng[p] = make_float4(s.ng.x, s.ng.y, s.ng.z, 0.0f); }
                    else { const float4 n4 = wf.ng[p]; first_ng = mk(n4.x, n4.y, n4.z); }
                    bounce_emission<ANIM>(sc, h.inst, ray.d, first_ng, round, (fl & WF_F_SPECULAR) != 0, mk(th4.x, th4.y, th4.z), time, illum);
                    Frame fr;
                    make_frame(s, fr);
                    const uint32_t hs = MODE == 2 ? __float_as_uint(il4.w) : wf_stream<MODE>(sc, rp, wf, p); // handed to _b / _c in f_b.w
                    wf.f_p[p] = make_float4(fr.p.x, fr.p.y, fr.p.z, __uint_as_float(material));
                    wf.f_n[p] = make_float4(fr.n.x, fr.n.y, fr.n.z, s.u); // .w: the hit's (u, v) for image textures
                    wf.f_t[p] = make_float4(fr.tan.x, fr.tan.y, fr.tan.z, s.v);
                    wf.f_b[p] = make_float4(fr.bitan.x, fr.bitan.y, fr.bitan.z, __uint_as_float(hs));
                    wf.illum[p] = make_float4(illum.x, illum.y, illum.z, MODE == 2 ? il4.w : 0.0f);
                    push_mid = true;
                    if (wf.mid_keyed) mid_key = __ldg(&sc.materials[material].type) & (WF_MID_BUCKETS - 1u);
                }
            }
            if (done) finish_sample(sc, rp, wf, p, illum, MODE);
        }
        wf_push_keyed(wf.q_mid, wf.n_paths, &cnt_r[WF_MID_K], push_mid, mid_key, p);
    }
}

// KIND >= 0: the instantiation compiled for that material kind alone; it drains that kind's bucket. KIND = -1: any kind; drains the
// buckets of `bucket_mask` (the kinds the scene uses that have no instantiation of their own). Every mode shades alike here: the
// stream hash comes with the frame.
template <bool ANIM, int MINB, int KIND = -1>
__global__ void __launch_bounds__(128, MINB) k_wf_shade_b(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf,
                                                     uint32_t round, uint32_t bucket_mask) {
    uint32_t* cnt_r = wf.counters + round * WF_CNT;
    uint32_t* cnt_n = wf.counters + (round + 1) * WF_CNT;
    const int lane = threadIdx.x & 31;
    for (uint32_t bucket = 0; bucket < WF_MID_BUCKETS; ++bucket) {
    if (!((bucket_mask >> bucket) & 1u)) continue;
    const uint32_t n = cnt_r[WF_MID_K + bucket];
    const uint32_t* __restrict__ q_mid = wf.q_mid + (size_t)bucket * wf.n_paths;
    for (;;) {
        if (n == 0) break;
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&cnt_r[WF_B_HEAD_K + bucket], 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= n) break;
        const uint32_t i = base + lane;
        uint32_t p = 0;
        bool push_shadow = false, push_mis = false;
        if (i < n) {
            p = q_mid[i];
            Frame fr; uint32_t material, hs; float tu, tv;
            load_frame(wf, p, fr, material, hs, tu, tv);
            const float4 c4 = wf.cont[p], th4 = wf.thr[p];
            const f3 wo = -mk(c4.x, c4.y, c4.z);
            Mat m;
            load_mat_at(sc, material, tu, tv, th4.w, m);
            DirectSetup ds; uint32_t light;
            bounce_direct<ANIM, KIND>(sc, m, fr, wo, round, hs, th4.w, ds, light, wf_xf_row<ANIM>(wf, p), rp.ld_offset);
            push_shadow = ds.has_shadow; push_mis = ds.has_mis;
            wf.org[p] = make_float4(fr.p.x, fr.p.y, fr.p.z, __uint_as_float((push_shadow ? WF_F_SHADOW : 0u) | (push_mis ? WF_F_MIS : 0u)));
            if (push_shadow) wf.shadow[p] = make_float4(ds.shadow_d.x, ds.shadow_d.y, ds.shadow_d.z, 0.0f);
            if (push_mis) wf.mis[p] = make_float4(ds.mis_d.x, ds.mis_d.y, ds.mis_d.z, finf());
            wf.a[p] = make_float4(ds.a.x, ds.a.y, ds.a.z, __uint_as_float(TRB_MISS));
            wf.b[p] = make_float4(ds.b.x, ds.b.y, ds.b.z, __uint_as_float(light));
            wf.tprev[p] = make_float4(th4.x, th4.y, th4.z, 0.0f); // path_throughput multiplying this bounce's direct light
        }
        wf_push(wf.q_shadow, &cnt_n[WF_N_SHADOW], push_shadow, p);
        wf_push(wf.q_mis, &cnt_n[WF_N_MIS], push_mis, p);
    }
    }
}

template <int MODE, bool ANIM, int MINB, int KIND = -1>
__global__ void __launch_bounds__(128, MINB) k_wf_shade_c(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf,
                                                     uint32_t round, uint32_t bucket_mask) {
    uint32_t* cnt_r = wf.counters + round * WF_CNT;
    uint32_t* cnt_n = wf.counters + (round + 1) * WF_CNT;
    uint32_t* act_next = wf.q_active[(round + 1) & 1];
    const int lane = threadIdx.x & 31;
    for (uint32_t bucket = 0; bucket < WF_MID_BUCKETS; ++bucket) {
    if (!((bucket_mask >> bucket) & 1u)) continue;
    const uint32_t n = cnt_r[WF_MID_K + bucket];
    const uint32_t* __restrict__ q_mid = wf.q_mid + (size_t)bucket * wf.n_paths;
    for (;;) {
        if (n == 0) break;
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&cnt_r[WF_C_HEAD_K + bucket], 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= n) break;
        const uint32_t i = base + lane;
        uint32_t p = 0;
        bool push_cont = false, push_active = false;
        f3 new_org = splat(0.0f);
        if (i < n) {
            p = q_mid[i];
            Frame fr; uint32_t material, hs; float tu, tv;
            load_frame(wf, p, fr, material, hs, tu, tv);
            const float4 c4 = wf.cont[p], th4 = wf.thr[p];
            const f3 wo = -mk(c4.x, c4.y, c4.z);
            Mat m;
            load_mat_at(sc, material, tu, tv, th4.w, m);
            ScatterOut so;
            bounce_scatter<KIND>(sc, m, fr, wo, round, hs, mk(th4.x, th4.y, th4.z), so, rp.ld_offset);
            const uint32_t fb = __float_as_uint(wf.org[p].w); // WF_F_SHADOW | WF_F_MIS from k_wf_shade_b
            push_cont = !so.terminate;
            push_active = push_cont || (fb & (WF_F_SHADOW | WF_F_MIS)) != 0u;
            if (push_active) {
                new_org = fr.p;
                wf.org[p] = make_float4(fr.p.x, fr.p.y, fr.p.z, __uint_as_float(fb | (so.specular ? WF_F_SPECULAR : 0u) | (so.terminate ? WF_F_TERMINATE : 0u)));
                if (push_cont) wf.cont[p] = make_float4(so.next_d.x, so.next_d.y, so.next_d.z, finf());
                wf.thr[p] = make_float4(so.throughput.x, so.throughput.y, so.throughput.z, th4.w);
            } else { // nothing pending: the direct light of this bounce is zero, the path ends here
                const float4 il4 = wf.illum[p];
                finish_sample(sc, rp, wf, p, mk(il4.x, il4.y, il4.z), MODE);
            }
        }
        wf_push(wf.q_cont, &cnt_n[WF_N_CONT], push_cont, p);
        wf_push(act_next, &cnt_n[WF_N_ACTIVE], push_active, p);
        if (wf.bounds) wf_bounds_add(wf.bounds + (round + 1) * 8, push_active, new_org); // ray sorting's origin boxes (nullptr: sorting off)
    }
    }
}

// The per-sample value of the lum_w film (include/trb.h "Sample variance"): l = L(c / max(a, TRB_DENOISE_EPS_ALBEDO)) of the sample's
// radiance c and the albedo a of its AOV record, as (l, l * l, 0)
__device__ __forceinline__ f3 lum_sample(float4 c, float4 a) {
    const float d0 = a.x > TRB_DENOISE_EPS_ALBEDO ? a.x : TRB_DENOISE_EPS_ALBEDO, d1 = a.y > TRB_DENOISE_EPS_ALBEDO ? a.y : TRB_DENOISE_EPS_ALBEDO,
                d2 = a.z > TRB_DENOISE_EPS_ALBEDO ? a.z : TRB_DENOISE_EPS_ALBEDO;
    const float l = 0.2126f * (c.x / d0) + 0.7152f * (c.y / d1) + 0.0722f * (c.z / d2);
    return mk(l, l * l, 0.0f);
}

// RenderTarget::write for a whole pass: one CTA per 8x8 block, footprint accumulated in shared memory.
// LUM: the lum_w film instead of the colour film, from the radiance (wf.rad) and the albedo half of each sample's AOV record (alb,
// indexed like wf.rad); the same weights, window and lock-block rule, with (w l, w l^2, w^2, w) in place of (w c, w).
template <bool ADAPT = false, bool LUM = false>
__global__ void __launch_bounds__(RENDER_THREADS) k_wf_film(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf,
                                                            const float4* __restrict__ alb = nullptr) {
    extern __shared__ float4 tile[];
    __shared__ float s_table[256];
    const int T = 9 + 2 * max(sc.fpw_x, sc.fpw_y);
    for (int i = threadIdx.x; i < 256; i += RENDER_THREADS) s_table[i] = sc.filter_table[i];
    const uint32_t pix = threadIdx.x & 63, lane_s = threadIdx.x >> 6;
    uint32_t n_live = 0; // ADAPT: the blocks this pass really covers; the LowDiscrepancy loop reads rp.n_blocks as before
    if (ADAPT) n_live = ad_pass_blocks(rp);
    for (uint32_t item = blockIdx.x; item < (ADAPT ? n_live : rp.n_blocks); item += gridDim.x) {
        __syncthreads();
        for (int i = threadIdx.x; i < T * T; i += RENDER_THREADS) tile[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
        const uint2 blk = rp.blocks[item];
        const uint32_t bx = blk.x * 8, by = blk.y * 8;
        SampleId id; id.item = item; id.pix = pix; id.px = bx + (pix & 7); id.py = by + (pix >> 3); id.pixel = id.py * sc.width + id.px;
        const PixelStreams ps = ADAPT ? pixel_streams_round(rp.seed, id.pixel, rp.ad_round) : pixel_streams(rp.seed, id.pixel);
        const bool on = !ADAPT || (rp.ad_state[id.pixel].x & trbh::AD_ACTIVE) != 0u; // Adaptive: pixels that took this round's samples
        const int x_lo = max((int)bx - sc.fpw_x, 0), x_hi = min((int)bx + 8 + sc.fpw_x, (int)sc.width - 1);
        const int y_lo = max((int)by - sc.fpw_y, 0), y_hi = min((int)by + 8 + sc.fpw_y, (int)sc.height - 1);
        const int tx0 = (int)bx - sc.fpw_x, ty0 = (int)by - sc.fpw_y;
        for (uint32_t s = lane_s; on && s < rp.sample_count; s += 2) {
            id.si = rp.sample_first + s;
            float sx, sy, tm;
            if (ADAPT) sample_position_ad(rp, ps, id, sx, sy, tm);
            else sample_position(rp, ps, id, sx, sy, tm);
            const size_t p = ((size_t)item * 64 + pix) * rp.sample_count + s;
            const float4 c4 = wf.rad[p];
            if (LUM) splat_sample<true>(sc, tile, s_table, T, tx0, ty0, x_lo, x_hi, y_lo, y_hi, id.px, id.py, sx, sy, lum_sample(c4, alb[p]));
            else splat_sample(sc, tile, s_table, T, tx0, ty0, x_lo, x_hi, y_lo, y_hi, id.px, id.py, sx, sy, mk(c4.x, c4.y, c4.z));
        }
        __syncthreads();
        for (int i = threadIdx.x; i < T * T; i += RENDER_THREADS) {
            const int ix = tx0 + i % T, iy = ty0 + i / T;
            if (ix < x_lo || ix > x_hi || iy < y_lo || iy > y_hi) continue;
            const float4 v = tile[i];
            if (v.w == 0.0f && v.x == 0.0f && v.y == 0.0f && v.z == 0.0f) continue;
            float* dst = reinterpret_cast<float*>(rp.film + (size_t)iy * sc.width + ix);
            atomicAdd(dst + 0, v.x); atomicAdd(dst + 1, v.y); atomicAdd(dst + 2, v.z); atomicAdd(dst + 3, v.w);
        }
    }
}

// ------------------------------------------------------------------------------------------
// AOVs (DESIGN.md §4 "AOVs"): one trb_aov_sample per camera sample from its primary hit, computed between the round-0 trace and the
// round-0 shade from the path state those two kernels share. The films are written by the colour film's own kernel (k_wf_film_v2 or
// k_wf_film) over the records' two halves, nearest by k_wf_nearest.
// ------------------------------------------------------------------------------------------
// Albedo of Material::bsdf's lobes (lobe_of, allocation order): colour x Fresnel factor at normal incidence, summed left to right,
// each channel clamped to [0, 1]. MERL has no colour term: pi * BSDF::eval(n, n) over all lobes.
__device__ __noinline__ f3 aov_albedo(const DScene& sc, const Mat& m, const Frame& fr) {
    f3 acc = splat(0.0f);
    if (m.type == TRB_MAT_MERL) acc = bsdf_eval(sc, m, fr, fr.n, fr.n, BX_ALL) * TRB_PI;
    else {
        const f3 F = fresnel(m, 1.0f);
#pragma unroll 1
        for (int i = 0; i < 2; ++i) {
            int kind; uint32_t type; f3 col;
            if (!lobe_of(m, i, kind, type, col)) continue;
            if (kind == LK_LAMBERT || kind == LK_OREN_NAYAR) acc = acc + col;
            else if (type & BX_TRANSMISSION) acc = acc + col * (splat(1.0f) - F);
            else acc = acc + col * F;
        }
    }
    return mk(clampf(acc.x, 0.0f, 1.0f), clampf(acc.y, 0.0f, 1.0f), clampf(acc.z, 0.0f, 1.0f));
}

// Per path of the pass (round 0: every path, path p = sample p of the pass): the camera ray (org, cont), its hit t (cont.w) and hit
// record, the path's time (thr.w) and keyframed transforms. Writes the record's two halves, (albedo, depth) to lo[p * step] and
// (n, inst bits) to hi[p * step]: step 2 with hi = lo + 1 is a trb_aov_sample array, step 1 two float4 arrays the film kernels read
// as they read wf.rad. Reads nothing the shade kernels write and writes nothing they read.
template <bool ANIM>
__device__ __forceinline__ void wf_aov_paths(const DScene& sc, const WfState& wf, uint32_t n, float4* __restrict__ lo_out, float4* __restrict__ hi_out,
                                             uint32_t step) {
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const uint4 h4 = wf.hit[p];
        float4 lo = make_float4(0.0f, 0.0f, 0.0f, finf()), hi = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(TRB_MISS));
        if (h4.x != TRB_MISS) {
            const float4 o4 = wf.org[p], c4 = wf.cont[p];
            const float time = wf.thr[p].w;
            Ray ray; ray.o = mk(o4.x, o4.y, o4.z); ray.d = mk(c4.x, c4.y, c4.z); ray.tmin = 0.0f; ray.tmax = c4.w;
            HitRec h; h.t = c4.w; h.inst = h4.x; h.prim = h4.y; h.b1 = __uint_as_float(h4.z); h.b2 = __uint_as_float(h4.w);
            Surf s;
            surface_at<ANIM>(sc, ray, h, s, time, wf_xf_row<ANIM>(wf, p));
            Frame fr;
            make_frame(s, fr);
            Mat m;
            load_mat_at(sc, __ldg(&sc.instances[h.inst].material), s.u, s.v, time, m);
            const f3 a = aov_albedo(sc, m, fr);
            lo = make_float4(a.x, a.y, a.z, c4.w);
            hi = make_float4(fr.n.x, fr.n.y, fr.n.z, __uint_as_float(h4.x));
        }
        lo_out[(size_t)p * step] = lo;
        hi_out[(size_t)p * step] = hi;
    }
}
template <bool ANIM>
__global__ void __launch_bounds__(128) k_wf_aov(const __grid_constant__ DScene sc, const __grid_constant__ WfState wf, float4* __restrict__ lo_out,
                                                float4* __restrict__ hi_out, uint32_t step) {
    wf_aov_paths<ANIM>(sc, wf, wf.n_paths, lo_out, hi_out, step);
}
// k_wf_aov for an Adaptive pass (DESIGN.md §4 "Adaptive AOVs"), which is launched for the worst-case path count: only the paths it
// really holds (WF_N_PATHS, written by k_wf_generate_ad), since the paths past them keep stale state of earlier passes. The paths of
// pixels that are not sampling this round enter as primary misses and give miss records, which no film or slot reads.
template <bool ANIM>
__global__ void __launch_bounds__(128) k_wf_aov_ad(const __grid_constant__ DScene sc, const __grid_constant__ WfState wf, float4* __restrict__ lo_out,
                                                   float4* __restrict__ hi_out) {
    wf_aov_paths<ANIM>(sc, wf, wf.counters[WF_N_PATHS], lo_out, hi_out, 1u);
}

// nearest: per camera sample of the pass, atomicMin(float_bits(depth) << 32 | inst) on the pixel the sample was taken for
__global__ void __launch_bounds__(256) k_wf_nearest(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const float4* __restrict__ lo,
                                                    const float4* __restrict__ hi, uint32_t n, unsigned long long* __restrict__ nearest) {
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const SampleId id = sample_id(sc, rp, p);
        atomicMin(&nearest[id.pixel], ((unsigned long long)__float_as_uint(lo[p].w) << 32) | __float_as_uint(hi[p].w));
    }
}
// k_wf_nearest for an Adaptive pass: the blocks it really covers (ad_pass_blocks) and the pixels that sampled this round. Runs
// before k_ad_decide, which clears the flag of a pixel that stops.
__global__ void __launch_bounds__(256) k_wf_nearest_ad(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const float4* __restrict__ lo,
                                                       const float4* __restrict__ hi, unsigned long long* __restrict__ nearest) {
    const uint32_t n = ad_pass_blocks(rp) * 64 * rp.sample_count;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const SampleId id = sample_id(sc, rp, p);
        if (!(rp.ad_state[id.pixel].x & trbh::AD_ACTIVE)) continue;
        atomicMin(&nearest[id.pixel], ((unsigned long long)__float_as_uint(lo[p].w) << 32) | __float_as_uint(hi[p].w));
    }
}

// ------------------------------------------------------------------------------------------
// Motion vectors (include/trb.h "Motion vectors"): one (v dx, v dy, v, 0) record per camera sample from its primary hit, between the
// round-0 trace and shade like k_wf_aov. Since dx = dy = 0 where v = 0, the record is also the value the motion_w film adds per unit
// weight: the colour film's kernel reads it in place of the radiance.
// ------------------------------------------------------------------------------------------
// The raster projection at the two times: the world -> camera matrix of a static camera (the frame's cam_world inverse; a keyframed
// camera evaluates its own at each time), tan(fov / 2) at t and at t + dt, camera_setup's screen window and the film size.
struct MotionCam {
    float cam_inv[16];
    float tan_now, tan_then, dt;
    float x0, x1, y0, y1, w, h;
};
// r(tau, x): camera_ray's raster -> camera mapping inverted, as dn_reproject inverts it; false unless x is in front of the camera
template <bool ANIM>
__device__ __forceinline__ bool motion_raster(const DScene& sc, const MotionCam& mc, float tau, float tan_fov, f3 x, float& rx, float& ry) {
    float inv[16];
    if (ANIM && sc.cam.animated) {
        float mat[16];
        eval_anim_xf(sc, sc.cam.spline_first, sc.cam.n_splines, tau, inv, mat);
    } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) inv[i] = mc.cam_inv[i];
    }
    const f3 q = xf_point(inv, x);
    const float X = q.x / (q.z * tan_fov), Y = q.y / (q.z * tan_fov);
    rx = (X - mc.x0) / (mc.x1 - mc.x0) * mc.w;
    ry = (Y - mc.y1) / (mc.y0 - mc.y1) * mc.h;
    return q.z > 0.0f;
}
// Per path of the pass (round 0): the hit's world point as surface_at computes it, p_o = M_i(t)^-1 p through the transform the trace
// and the transform table use, then r(t + dt, M_i(t + dt) p_o) - r(t, M_i(t) p_o). ANIM false: no keyframed transform at all, so the
// two points are one (a static scene's records are (0, 0, v) unless the fov is animated).
template <bool ANIM>
__device__ __forceinline__ void wf_motion_paths(const DScene& sc, const WfState& wf, const MotionCam& mc, uint32_t n, float4* __restrict__ out) {
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const uint4 h4 = wf.hit[p];
        float4 rec = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (h4.x != TRB_MISS) {
            const float4 o4 = wf.org[p], c4 = wf.cont[p];
            const float time = wf.thr[p].w;
            const DInstance& in = sc.instances[h4.x];
            float m[16], w[16];
            instance_inv_mat<ANIM>(sc, in, time, m, w, wf_xf_row<ANIM>(wf, p));
            const f3 o = xf_point(m, mk(o4.x, o4.y, o4.z)), d = xf_vector(m, mk(c4.x, c4.y, c4.z));
            const f3 pw = xf_point(w, o + d * c4.w); // surface_at's s.p
            const f3 po = xf_point(m, pw);
            const f3 p_now = xf_point(w, po);
            f3 p_then = p_now;
            if (ANIM && (__ldg(&in.flags) & DI_ANIM_XF)) {
                float inv2[16], mat2[16];
                eval_anim_xf(sc, __ldg(&in.spline_first), __ldg(&in.n_splines), time + mc.dt, inv2, mat2);
                p_then = xf_point(mat2, po);
            }
            float x0, y0, x1, y1;
            const bool v0 = motion_raster<ANIM>(sc, mc, time, mc.tan_now, p_now, x0, y0);
            const bool v1 = motion_raster<ANIM>(sc, mc, time + mc.dt, mc.tan_then, p_then, x1, y1);
            if (v0 && v1) rec = make_float4(x1 - x0, y1 - y0, 1.0f, 0.0f);
        }
        out[p] = rec;
    }
}
template <bool ANIM>
__global__ void __launch_bounds__(128) k_wf_motion(const __grid_constant__ DScene sc, const __grid_constant__ WfState wf, const __grid_constant__ MotionCam mc,
                                                   float4* __restrict__ out) {
    wf_motion_paths<ANIM>(sc, wf, mc, wf.n_paths, out);
}
// k_wf_motion for an Adaptive pass: the paths it really holds (WF_N_PATHS), as k_wf_aov_ad
template <bool ANIM>
__global__ void __launch_bounds__(128) k_wf_motion_ad(const __grid_constant__ DScene sc, const __grid_constant__ WfState wf, const __grid_constant__ MotionCam mc,
                                                      float4* __restrict__ out) {
    wf_motion_paths<ANIM>(sc, wf, mc, wf.counters[WF_N_PATHS], out);
}

// LowDiscrepancy::get_samples + get_samples_1d + Camera::generate_ray only (parity of S2 / C)
// k_wf_film without shared-memory atomics (opt-in: TRB_FILM_V2=1; validated by tools/film_check.py). Each of the CTA's
// four warps splats into its OWN copy of the tile. Inside a warp the 32 lanes are 32 different pixels walking the footprint
// in lockstep (same (dy, dx) offset at the same time, __syncwarp per offset), so their targets are always 32 different tile
// pixels and a plain 16-byte read-modify-write is race-free; the four copies are summed at the flush. Same weights and
// products as RenderTarget::write; only the order of the float additions differs (the film bar is an RMSE tolerance).
// LUM: the lum_w film, as for k_wf_film.
template <bool ADAPT = false, bool LUM = false>
__global__ void __launch_bounds__(RENDER_THREADS) k_wf_film_v2(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf,
                                                               const float4* __restrict__ alb = nullptr) {
    extern __shared__ float4 tiles[]; // 4 x T*T
    __shared__ float s_table[256];
    const int T = 9 + 2 * max(sc.fpw_x, sc.fpw_y);
    for (int i = threadIdx.x; i < 256; i += RENDER_THREADS) s_table[i] = sc.filter_table[i];
    const uint32_t pix = threadIdx.x & 63, lane_s = threadIdx.x >> 6;
    float4* mine = tiles + (threadIdx.x >> 5) * (T * T);
    const int ry = (int)ceilf(sc.filter_h / sc.filter_inv_h) + 1, rx = (int)ceilf(sc.filter_w / sc.filter_inv_w) + 1;
    uint32_t n_live = 0; // ADAPT: the blocks this pass really covers (CTA-uniform: the per-offset __syncwarp lockstep is untouched)
    if (ADAPT) n_live = ad_pass_blocks(rp);
    for (uint32_t item = blockIdx.x; item < (ADAPT ? n_live : rp.n_blocks); item += gridDim.x) {
        __syncthreads();
        for (int i = threadIdx.x; i < 4 * T * T; i += RENDER_THREADS) tiles[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
        const uint2 blk = rp.blocks[item];
        const uint32_t bx = blk.x * 8, by = blk.y * 8;
        SampleId id; id.item = item; id.pix = pix; id.px = bx + (pix & 7); id.py = by + (pix >> 3); id.pixel = id.py * sc.width + id.px;
        const PixelStreams ps = ADAPT ? pixel_streams_round(rp.seed, id.pixel, rp.ad_round) : pixel_streams(rp.seed, id.pixel);
        // Adaptive: a pixel that took no samples this round walks the footprint with the others (the __syncwarp lockstep below
        // is what makes the plain read-modify-write race-free) but writes nothing
        const bool on = !ADAPT || (rp.ad_state[id.pixel].x & trbh::AD_ACTIVE) != 0u;
        const int x_lo = max((int)bx - sc.fpw_x, 0), x_hi = min((int)bx + 8 + sc.fpw_x, (int)sc.width - 1);
        const int y_lo = max((int)by - sc.fpw_y, 0), y_hi = min((int)by + 8 + sc.fpw_y, (int)sc.height - 1);
        const int tx0 = (int)bx - sc.fpw_x, ty0 = (int)by - sc.fpw_y;
        for (uint32_t s = lane_s; s < rp.sample_count; s += 2) { // uniform trip count inside a warp (one lane_s per warp)
            id.si = rp.sample_first + s;
            float sx, sy, tm;
            if (ADAPT) sample_position_ad(rp, ps, id, sx, sy, tm);
            else sample_position(rp, ps, id, sx, sy, tm);
            float4 c4 = on ? wf.rad[((size_t)item * 64 + pix) * rp.sample_count + s] : make_float4(0.f, 0.f, 0.f, 0.f);
            if (LUM && on) {
                const f3 l = lum_sample(c4, alb[((size_t)item * 64 + pix) * rp.sample_count + s]);
                c4 = make_float4(l.x, l.y, l.z, 0.f);
            }
            const float img_x = sx - 0.5f, img_y = sy - 0.5f;
            for (int dy = -ry; dy <= ry + 1; ++dy) {
                const int iy = (int)id.py + dy;
                const float fy = fabsf((float)iy - img_y) * sc.filter_inv_h;
                const bool vy = iy >= y_lo && iy <= y_hi && !(fy > sc.filter_h) && // sic: normalised distance vs width (A7)
                                (!sc.film_block_filter || lock_block_takes(sy, iy, y_lo, y_hi, sc.fpw_y));
                const uint32_t fyi = min(f2u(fy * 16.0f), 15u);
                for (int dx = -rx; dx <= rx + 1; ++dx) {
                    const int ix = (int)id.px + dx;
                    const float fx = fabsf((float)ix - img_x) * sc.filter_inv_w;
                    if (on && vy && ix >= x_lo && ix <= x_hi && !(fx > sc.filter_w) && (!sc.film_block_filter || lock_block_takes(sx, ix, x_lo, x_hi, sc.fpw_x))) {
                        const uint32_t fxi = min(f2u(fx * 16.0f), 15u);
                        const float wgt = s_table[fyi * 16 + fxi];
                        float4* t = &mine[(iy - ty0) * T + (ix - tx0)];
                        float4 a = *t;
                        a.x += wgt * c4.x; a.y += wgt * c4.y; a.z += LUM ? wgt * wgt : wgt * c4.z; a.w += wgt;
                        *t = a;
                    }
                    __syncwarp(); // lockstep per offset: no lane starts (dy, dx + 1) before all finished (dy, dx)
                }
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < T * T; i += RENDER_THREADS) {
            const int ix = tx0 + i % T, iy = ty0 + i / T;
            if (ix < x_lo || ix > x_hi || iy < y_lo || iy > y_hi) continue;
            const float4 a = tiles[i], b = tiles[T * T + i], c = tiles[2 * T * T + i], d = tiles[3 * T * T + i];
            const float4 v = make_float4((a.x + b.x) + (c.x + d.x), (a.y + b.y) + (c.y + d.y), (a.z + b.z) + (c.z + d.z), (a.w + b.w) + (c.w + d.w));
            if (v.w == 0.0f && v.x == 0.0f && v.y == 0.0f && v.z == 0.0f) continue;
            float* dst = reinterpret_cast<float*>(rp.film + (size_t)iy * sc.width + ix);
            atomicAdd(dst + 0, v.x); atomicAdd(dst + 1, v.y); atomicAdd(dst + 2, v.z); atomicAdd(dst + 3, v.w);
        }
    }
}

template <bool ANIM>
__global__ void k_camera_rays(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, trb_ray* rays, float* xy) {
    const size_t n = (size_t)rp.n_blocks * 64 * rp.sample_count;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t s = (uint32_t)(i % rp.sample_count), pix = (uint32_t)((i / rp.sample_count) % 64), item = (uint32_t)(i / ((size_t)64 * rp.sample_count));
        const uint2 blk = rp.blocks[item];
        const uint32_t px = blk.x * 8 + (pix & 7), py = blk.y * 8 + (pix >> 3);
        const PixelStreams ps = pixel_streams(rp.seed, py * sc.width + px);
        const uint32_t si = rp.sample_first + s;
        const uint32_t ip = permute_index(si, rp.spp, ps.kpos);
        const float sx = ld_vdc(ip, ps.scr0) + (float)px, sy = ld_sobol(ip, ps.scr1) + (float)py;
        const float tm = ld_vdc(permute_index(si, rp.spp, ps.ktime), ps.scrt);
        Ray r;
        camera_ray<ANIM>(sc, sx, sy, tm, r);
        rays[i].o[0] = r.o.x; rays[i].o[1] = r.o.y; rays[i].o[2] = r.o.z;
        rays[i].d[0] = r.d.x; rays[i].d[1] = r.d.y; rays[i].d[2] = r.d.z;
        rays[i].min_t = r.tmin; rays[i].max_t = r.tmax;
        xy[2 * i] = sx; xy[2 * i + 1] = sy;
    }
}

// Scene::intersect over a ray batch (trb_intersect): one ray per thread, grid-stride.
template <bool STATS, bool ANIM, bool WIDE = false>
__global__ void __launch_bounds__(128) k_intersect(const __grid_constant__ DScene sc, size_t n, const trb_ray* __restrict__ rays, trb_hit* __restrict__ hits,
                                                    DStats* stats, int* err) {
    Cnt cnt = {0, 0, 0};
    RayCounts rc = {0, 0, 0, 0};
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(rays + i)), b = __ldg(reinterpret_cast<const float4*>(rays + i) + 1);
        Ray r; r.o = mk(a.x, a.y, a.z); r.d = mk(a.w, b.x, b.y); r.tmin = b.z; r.tmax = b.w;
        HitRec h;
        const bool hit = scene_trace<STATS, ANIM, WIDE>(sc, r, h, false, cnt, err, sc.cam.shutter_open); // batch rays carry no time: the frame's shutter-open time
        rc.primary++;
        uint4 o; o.x = __float_as_uint(r.tmax); o.y = hit ? h.inst : TRB_MISS; o.z = hit ? h.prim : 0u; o.w = 0u;
        *reinterpret_cast<uint4*>(hits + i) = o;
    }
    if (stats) flush_stats(stats, rc, cnt, 0, STATS);
}

// ------------------------------------------------------------------------------------------
// Ray queries (trb_intersect_records / trb_occluded) on the render's trace kernel: one pass = k_query_load writes the pass's
// rays into the path state as round 0 of a wavefront (continuation rays for records, shadow rays for occlusion), keyframed
// scenes fill the transform table from each ray's time (k_wf_anim_table[2], unchanged), k_wf_trace runs with PIPE bit 64 (each
// ray's own [min_t, max_t]), then k_query_records / k_query_occluded read the results out of the path state.
// ------------------------------------------------------------------------------------------
template <bool OCCLUSION>
__global__ void __launch_bounds__(256) k_query_load(const __grid_constant__ WfState wf, const trb_query_ray* __restrict__ rays) {
    const uint32_t n = wf.n_paths;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const float4* r = reinterpret_cast<const float4*>(rays + p); // (o, d.x) (d.yz, min_t, max_t) (time, pad)
        const float4 a = __ldg(r), b = __ldg(r + 1), c = __ldg(r + 2);
        wf.org[p] = make_float4(a.x, a.y, a.z, b.z);
        (OCCLUSION ? wf.shadow : wf.cont)[p] = make_float4(a.w, b.x, b.y, b.w);
        wf.thr[p] = make_float4(0.0f, 0.0f, 0.0f, c.x); // .w: ray.time, as k_wf_generate leaves it for the transform table and the trace
        (OCCLUSION ? wf.q_shadow : wf.q_cont)[p] = p;
    }
    if (blockIdx.x == 0 && threadIdx.x < WF_CNT) wf.counters[threadIdx.x] = threadIdx.x == (OCCLUSION ? WF_N_SHADOW : WF_N_CONT) ? n : 0u;
}
// geometry::Intersection of each ray (scene.rs:148-150): the DifferentialGeometry of Receiver / Emitter::intersect in world space
// (receiver.rs:36-41, emitter.rs:128-134), built by surface_at's shape code from the trace kernel's (t, inst, prim, b1, b2)
template <bool ANIM>
__global__ void __launch_bounds__(128) k_query_records(const __grid_constant__ DScene sc, const __grid_constant__ WfState wf, trb_intersection* __restrict__ out) {
    const uint32_t n = wf.n_paths;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const float4 o4 = wf.org[p], d4 = wf.cont[p];
        const uint4 h4 = wf.hit[p];
        float4 q[6] = {make_float4(d4.w, __uint_as_float(TRB_MISS), 0.0f, 0.0f), make_float4(0.0f, 0.0f, 0.0f, 0.0f), make_float4(0.0f, 0.0f, 0.0f, 0.0f),
                       make_float4(0.0f, 0.0f, 0.0f, 0.0f), make_float4(0.0f, 0.0f, 0.0f, 0.0f), make_float4(0.0f, 0.0f, 0.0f, 0.0f)};
        if (h4.x != TRB_MISS) {
            Ray ray; ray.o = mk(o4.x, o4.y, o4.z); ray.d = mk(d4.x, d4.y, d4.z); ray.tmin = o4.w; ray.tmax = d4.w;
            HitRec hit; hit.t = d4.w; hit.inst = h4.x; hit.prim = h4.y; hit.b1 = __uint_as_float(h4.z); hit.b2 = __uint_as_float(h4.w);
            const float time = wf.thr[p].w;
            Surf s;
            f3 dp_dv;
            surface_at<ANIM, true>(sc, ray, hit, s, time, wf_xf_row<ANIM>(wf, p), &dp_dv);
            const uint32_t material = __ldg(&sc.instances[hit.inst].material);
            // t inst prim material | p n.x | n.yz ng.xy | ng.z u v time | dp_du dp_dv.x | dp_dv.yz pad
            q[0] = make_float4(d4.w, __uint_as_float(hit.inst), __uint_as_float(hit.prim), __uint_as_float(material));
            q[1] = make_float4(s.p.x, s.p.y, s.p.z, s.n.x);
            q[2] = make_float4(s.n.y, s.n.z, s.ng.x, s.ng.y);
            q[3] = make_float4(s.ng.z, s.u, s.v, time);
            q[4] = make_float4(s.dp_du.x, s.dp_du.y, s.dp_du.z, dp_dv.x);
            q[5] = make_float4(dp_dv.y, dp_dv.z, 0.0f, 0.0f);
        }
        float4* dst = reinterpret_cast<float4*>(out + p);
#pragma unroll
        for (int k = 0; k < 6; ++k) dst[k] = q[k];
    }
}
__global__ void __launch_bounds__(256) k_query_occluded(const __grid_constant__ WfState wf, uint8_t* __restrict__ out) {
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < wf.n_paths; p += gridDim.x * blockDim.x) out[p] = __float_as_uint(wf.shadow[p].w) != 0u ? 1 : 0;
}

// ------------------------------------------------------------------------------------------
// Illumination queries (trb_illumination): Integrator::illumination along caller rays on the render's wavefront. Path p of a pass
// is sample j = p % spp of ray i = p / spp. k_illum_load writes it as a round-0 path the way k_wf_generate writes a camera sample:
// the ray with its [min_t, max_t] as PIPE bit 64 of k_wf_trace reads them (min_t in org.w: the MODE 2 shade kernels do not take
// it for flags), throughput (1, 1, 1, time), and in illum.w the hash of the camera-sample stream (seed, key, sample + j) that
// the render derives from (seed, pixel, si). The bounce rounds then run the render's trace and MODE 2 shade kernels, which
// leave each sample's unclamped radiance in wf.rad; k_illum_reduce averages each ray's spp samples.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_illum_load(const __grid_constant__ WfState wf, const trb_illum_ray* __restrict__ rays, uint32_t spp, uint32_t seed,
                                                    DStats* stats) {
    const uint32_t n = wf.n_paths, hseed = rng_seed(seed);
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const float4* r = reinterpret_cast<const float4*>(rays + p / spp); // (o, d.x) (d.yz, min_t, max_t) (time, key, sample, pad)
        const float4 a = __ldg(r), b = __ldg(r + 1), c = __ldg(r + 2);
        const uint32_t hs = rng_absorb(rng_absorb(hseed, __float_as_uint(c.y)), __float_as_uint(c.z) + p % spp);
        wf.org[p] = make_float4(a.x, a.y, a.z, b.z);
        wf.cont[p] = make_float4(a.w, b.x, b.y, b.w);
        wf.thr[p] = make_float4(1.0f, 1.0f, 1.0f, c.x);
        wf.illum[p] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(hs));
        wf.q_cont[p] = p;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { // as k_wf_generate: the host zeroed every round's counters
        wf.counters[WF_N_ACTIVE] = n; wf.counters[WF_N_CONT] = n;
        if (stats) atomicAdd(&stats->camera_samples, (unsigned long long)n);
    }
    if (wf.bounds && blockIdx.x == 0 && threadIdx.x < 64) {
        uint32_t* b = wf.bounds + threadIdx.x * 8;
        b[0] = b[1] = b[2] = b[3] = 0xffffffffu; b[4] = b[5] = b[6] = b[7] = 0u;
    }
}
// rgb[3i + c] = (sum over j in order of sample j's radiance, each clamped to [0, 1] first if asked) / spp
__global__ void __launch_bounds__(128) k_illum_reduce(const float4* __restrict__ rad, uint32_t n_rays, uint32_t spp, uint32_t clamp, float* __restrict__ rgb) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_rays; i += gridDim.x * blockDim.x) {
        const float4* r = rad + (size_t)i * spp;
        f3 sum = splat(0.0f);
        for (uint32_t j = 0; j < spp; ++j) {
            const float4 v = r[j];
            const f3 c = clamp ? mk(clampf(v.x, 0.0f, 1.0f), clampf(v.y, 0.0f, 1.0f), clampf(v.z, 0.0f, 1.0f)) : mk(v.x, v.y, v.z);
            sum = j == 0 ? c : sum + c; // starts at sample 0, not at 0.0f: one sample returns its own bits, -0.0 included
        }
        const float k = (float)spp;
        rgb[3 * (size_t)i] = sum.x / k; rgb[3 * (size_t)i + 1] = sum.y / k; rgb[3 * (size_t)i + 2] = sum.z / k;
    }
}

// ------------------------------------------------------------------------------------------
// Shading queries (trb_bsdf_eval / trb_bsdf_sample / trb_light_sample / trb_light_pdf / trb_emitted): the render's shading functions
// on caller inputs, one query per thread, grid-stride, 16-byte loads of every query and record. Nothing is traced. An index out of
// range (a missed record, a material, light or instance past the scene's, a light that is not an emitter) writes zeros and reads
// nothing else.
// ------------------------------------------------------------------------------------------
// Material::bsdf(&Intersection) (material/*.rs, bsdf.rs:38-44) at record r: the material's parameters sampled at (u, v, time), the
// frame from n and dp_du. The record is already in world space, so no transform is involved.
__device__ __forceinline__ bool record_bsdf(const DScene& sc, uint32_t n_materials, const trb_intersection* rec, Mat& m, Frame& fr) {
    const float4* r = reinterpret_cast<const float4*>(rec); // t inst prim material | p n.x | n.yz ng.xy | ng.z u v time | dp_du dp_dv.x
    const float4 a = __ldg(r);
    if (__float_as_uint(a.y) == TRB_MISS || __float_as_uint(a.w) >= n_materials) return false;
    const float4 b = __ldg(r + 1), c = __ldg(r + 2), d = __ldg(r + 3), e = __ldg(r + 4);
    Surf s;
    s.p = mk(b.x, b.y, b.z); s.n = mk(b.w, c.x, c.y); s.ng = mk(c.z, c.w, d.x); s.u = d.y; s.v = d.z; s.dp_du = mk(e.x, e.y, e.z);
    load_mat_at(sc, __float_as_uint(a.w), d.y, d.z, d.w, m);
    make_frame(s, fr);
    return true;
}
// out[i] = (BSDF::eval(wo, wi, bxdf), BSDF::pdf(wo, wi, bxdf)) (bsdf.rs:66-78, 114-125)
__global__ void __launch_bounds__(128) k_bsdf_eval(const __grid_constant__ DScene sc, uint32_t n_materials, size_t n, const trb_intersection* __restrict__ rec,
                                                   const trb_bsdf_eval_query* __restrict__ q, float4* __restrict__ out) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float4 o = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        Mat m; Frame fr;
        if (record_bsdf(sc, n_materials, rec + i, m, fr)) {
            const float4* qq = reinterpret_cast<const float4*>(q + i); // (wo, bxdf) (wi, pad)
            const float4 a = __ldg(qq), b = __ldg(qq + 1);
            const f3 wo = mk(a.x, a.y, a.z), wi = mk(b.x, b.y, b.z);
            const uint32_t flags = __float_as_uint(a.w);
            const f3 f = bsdf_eval(sc, m, fr, wo, wi, flags);
            o = make_float4(f.x, f.y, f.z, bsdf_pdf(m, fr, wo, wi, flags));
        }
        out[i] = o;
    }
}
// out[i] = BSDF::sample(wo, bxdf, Sample { two_d: u, one_d: u_comp }) (bsdf.rs:85-112): (f, pdf) (wi, sampled type bits)
__global__ void __launch_bounds__(128) k_bsdf_sample(const __grid_constant__ DScene sc, uint32_t n_materials, size_t n, const trb_intersection* __restrict__ rec,
                                                     const trb_bsdf_sample_query* __restrict__ q, trb_bsdf_sample_result* __restrict__ out) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float4 o0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), o1 = o0;
        Mat m; Frame fr;
        if (record_bsdf(sc, n_materials, rec + i, m, fr)) {
            const float4* qq = reinterpret_cast<const float4*>(q + i); // (wo, bxdf) (u, u_comp, pad)
            const float4 a = __ldg(qq), b = __ldg(qq + 1);
            f3 f, wi; float pdf; uint32_t sampled;
            bsdf_sample(sc, m, fr, mk(a.x, a.y, a.z), __float_as_uint(a.w), b.x, b.y, b.z, f, wi, pdf, sampled);
            o0 = make_float4(f.x, f.y, f.z, pdf);
            o1 = make_float4(wi.x, wi.y, wi.z, __uint_as_float(sampled));
        }
        float4* dst = reinterpret_cast<float4*>(out + i);
        dst[0] = o0; dst[1] = o1;
    }
}
// Is `li` an emitter of the scene? (anything else gives a zero result)
__device__ __forceinline__ bool is_light(const DScene& sc, uint32_t li) { return li < sc.n_instances && __ldg(&sc.instances[li].kind) != TRB_INST_RECEIVER; }
// out[i] = Light::sample_incident(p, u, time) of light q.light (emitter.rs:164-190): (Li, pdf) (wi, delta_light) and the
// OcclusionTester as a ray, test_points(p, p_light, time) = Ray::segment(p, p_light - p, 0.001, 0.999, time) (light/mod.rs:21-23)
template <bool ANIM>
__global__ void __launch_bounds__(128) k_light_sample(const __grid_constant__ DScene sc, size_t n, const trb_light_query* __restrict__ q, trb_light_sample_result* __restrict__ out) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float4* qq = reinterpret_cast<const float4*>(q + i); // (p, time) (u, light, pad)
        const float4 a = __ldg(qq), b = __ldg(qq + 1);
        const uint32_t li = __float_as_uint(b.z);
        const float4 z = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        float4 o[5] = {z, z, z, z, z};
        if (is_light(sc, li)) {
            const f3 p = mk(a.x, a.y, a.z);
            f3 lrad, wi, seg; float pdf;
            light_sample_incident<ANIM>(sc, li, p, b.x, b.y, a.w, lrad, wi, pdf, seg);
            const uint32_t delta = __ldg(&sc.instances[li].kind) == TRB_INST_EMITTER_POINT ? 1u : 0u;
            // li pdf | wi delta | shadow: (o, d.x) (d.yz, min_t, max_t) (time, pad)
            o[0] = make_float4(lrad.x, lrad.y, lrad.z, pdf);
            o[1] = make_float4(wi.x, wi.y, wi.z, __uint_as_float(delta));
            o[2] = make_float4(p.x, p.y, p.z, seg.x);
            o[3] = make_float4(seg.y, seg.z, 0.001f, 0.999f);
            o[4] = make_float4(a.w, 0.0f, 0.0f, 0.0f);
        }
        float4* dst = reinterpret_cast<float4*>(out + i);
#pragma unroll
        for (int k = 0; k < 5; ++k) dst[k] = o[k];
    }
}
// Light::pdf of Emitter (emitter.rs:193-203): 0 for a point light, else the shape's pdf of the object-space point and normalised
// direction — the operations of direct_setup's MIS weight, with the light's transform at `time`
template <bool ANIM>
__device__ __noinline__ float light_pdf(const DScene& sc, uint32_t li, f3 p, f3 wi, float time) {
    const DInstance& light = sc.instances[li];
    if (__ldg(&light.kind) == TRB_INST_EMITTER_POINT) return 0.0f;
    float linv[16];
    instance_inv<ANIM>(sc, light, time, linv);
    const f3 pl = xf_point(linv, p);
    const f3 wl = unit(xf_vector(linv, wi));
    return shape_pdf(__ldg(&light.shape), __ldg(&light.p0), __ldg(&light.p1), pl, wl);
}
template <bool ANIM>
__global__ void __launch_bounds__(128) k_light_pdf(const __grid_constant__ DScene sc, size_t n, const trb_light_pdf_query* __restrict__ q, float* __restrict__ pdf) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float4* qq = reinterpret_cast<const float4*>(q + i); // (p, time) (wi, light)
        const float4 a = __ldg(qq), b = __ldg(qq + 1);
        const uint32_t li = __float_as_uint(b.w);
        pdf[i] = is_light(sc, li) ? light_pdf<ANIM>(sc, li, mk(a.x, a.y, a.z), mk(b.x, b.y, b.z), a.w) : 0.0f;
    }
}
// rgb[3i..3i+2] = Emitter::radiance(w, _, n, time) (emitter.rs:140-142) of instance q.inst: its emission at `time` when
// dot(w, n) > 0, else black; black for a receiver
template <bool ANIM>
__global__ void __launch_bounds__(128) k_emitted(const __grid_constant__ DScene sc, size_t n, const trb_emit_query* __restrict__ q, float* __restrict__ rgb) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float4* qq = reinterpret_cast<const float4*>(q + i); // (w, time) (n, inst)
        const float4 a = __ldg(qq), b = __ldg(qq + 1);
        const uint32_t inst = __float_as_uint(b.w);
        f3 le = splat(0.0f);
        if (is_light(sc, inst) && dot3(mk(a.x, a.y, a.z), mk(b.x, b.y, b.z)) > 0.0f) emission_at<ANIM>(sc, sc.instances[inst], a.w, le.x, le.y, le.z);
        rgb[3 * i] = le.x; rgb[3 * i + 1] = le.y; rgb[3 * i + 2] = le.z;
    }
}

// ------------------------------------------------------------------------------------------
// Scene::update_frame on the device (SURVEY 8f N1; scene.rs:152-176, bvh.rs:61-78): per instance the world transform at the
// shutter-open time and its bounds over the shutter interval (animation_bounds, animated_transform.rs:57-70: 128 time
// samples when every stacked level is keyframed, one box otherwise — Q22), then BVH<Instance>::rebuild with the reference's
// SAH builder (the same bvh_build_arrays the host runs, on one thread for the tens of instances of most scenes; the level builder
// of trb_bvh_build.cuh writes the same bytes for scenes of many instances) and the child-pair records the trace kernel walks. Nothing is uploaded per frame but the camera block inside the kernel parameters.
// ------------------------------------------------------------------------------------------
struct FrameBuild {
    DInstance* instances;          // in/out: static fields set at scene creation; inv / mat written here
    trbh::Box3* bounds;            // out [n]
    uint32_t n;
    float shutter_open, shutter_close;
    // TLAS build
    float* cx; float* cy; float* cz; uint32_t* idx; uint32_t* task; uint32_t* rec_of; // scratch
    trb_bvh_node* nodes; uint32_t* order; uint32_t* counts; // out: reference-order nodes, ordered_geom, {n_nodes, n_order, pack ok, bounds not buildable}
    DPair* pairs; DBvh* hdr;                                // out: traversal records + header
};
__device__ __forceinline__ trbh::Box3 shape_bounds_dev(const DScene& sc, const DInstance& in) {
    trbh::Box3 b;
    const float p0 = in.p0, p1 = in.p1;
    switch (in.shape) {
        case TRB_SHAPE_SPHERE: for (int i = 0; i < 3; ++i) { b.lo[i] = -p0; b.hi[i] = p0; } break;                               // sphere.rs:84-88
        case TRB_SHAPE_DISK: b.lo[0] = b.lo[1] = -p0; b.hi[0] = b.hi[1] = p0; b.lo[2] = -0.1f; b.hi[2] = 0.1f; break;            // disk.rs:79-81
        case TRB_SHAPE_RECT: { const float hw = p0 / 2.0f, hh = p1 / 2.0f; b.lo[0] = -hw; b.lo[1] = -hh; b.hi[0] = hw; b.hi[1] = hh; b.lo[2] = b.hi[2] = 0.0f; break; } // rectangle.rs:67-71
        case TRB_SHAPE_MESH: { const DBvh& h = sc.meshes[in.mesh].bvh; b.lo[0] = h.root_lo.x; b.lo[1] = h.root_lo.y; b.lo[2] = h.root_lo.z; b.hi[0] = h.root_hi.x; b.hi[1] = h.root_hi.y; b.hi[2] = h.root_hi.z; break; } // mesh.rs:87-90
        default: for (int i = 0; i < 3; ++i) b.lo[i] = b.hi[i] = 0.0f;                                                          // point light (emitter.rs:152)
    }
    return b;
}
__global__ void __launch_bounds__(64) k_frame_instances(const __grid_constant__ DScene sc, const __grid_constant__ FrameBuild fb) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= fb.n) return;
    DInstance& in = fb.instances[i];
    const uint32_t first = in.xf_first, cnt = in.xf_count;
    const trbh::Xf w = trbh::animated_xf(sc.splines, first, cnt, sc.keyframes, sc.knots, fb.shutter_open, sc.level_xf);
#pragma unroll
    for (int k = 0; k < 16; ++k) { in.inv[k] = w.inv.m[k]; in.mat[k] = w.fwd.m[k]; }
    const trbh::Box3 local = shape_bounds_dev(sc, in);
    trbh::Box3 acc;
    if (!trbh::xf_is_animated(sc.splines, first, cnt)) acc = trbh::arvo_bounds(w.fwd, local);
    else {
        acc = trbh::box_empty_hd();
        for (int k = 0; k < 128; ++k) {
            const float u = (float)k / 127.0f;
            const float time = fb.shutter_open * (1.0f - u) + fb.shutter_close * u; // linalg::lerp
            const trbh::Xf x = trbh::animated_xf(sc.splines, first, cnt, sc.keyframes, sc.knots, time, sc.level_xf);
            trbh::box_grow_hd(acc, trbh::arvo_bounds(x.fwd, local));
        }
    }
    fb.bounds[i] = acc;
}
__global__ void k_tlas_build(const __grid_constant__ FrameBuild fb) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    bool buildable = true; // trb_host.h bvh_bound_buildable: the build below would not end otherwise
    if (fb.n > 4u) for (uint32_t i = 0; i < 6u * fb.n; ++i) buildable = buildable && trbh::bvh_bound_buildable(reinterpret_cast<const float*>(fb.bounds)[i]);
    fb.counts[3] = buildable ? 0u : 1u;
    if (!buildable) return;
    trbh::BvhBuildArrays B{fb.bounds, fb.n, 4u, fb.cx, fb.cy, fb.cz, fb.idx, fb.task, fb.nodes, fb.order, 0u, 0u}; // max_geom 4 (scene.rs:141)
    trbh::bvh_build_arrays(B);
    // child-pair records (trb_device.h DPair): pure re-layout of the reference-order tree
    const trb_bvh_node* in = fb.nodes;
    uint32_t n_rec = 0;
    bool ok = true;
    for (uint32_t i = 0; i < B.n_nodes; ++i) if (!(in[i].b & TRB_BVH_LEAF)) fb.rec_of[i] = n_rec++;
    auto ref_of = [&](uint32_t i) -> uint32_t {
        if (in[i].b & TRB_BVH_LEAF) {
            const uint32_t cnt = in[i].b & ~TRB_BVH_LEAF, first = in[i].a;
            if (cnt > 31 || first >= (1u << 25)) ok = false;
            return REF_LEAF | (cnt << 25) | first;
        }
        return REF_INTERIOR | fb.rec_of[i];
    };
    for (uint32_t i = 0; i < B.n_nodes; ++i) {
        if (in[i].b & TRB_BVH_LEAF) continue;
        const trb_bvh_node& l = in[i + 1];
        const trb_bvh_node& r = in[in[i].a];
        DPair& p = fb.pairs[fb.rec_of[i]];
        p.l_lo = make_float4(l.bmin[0], l.bmin[1], l.bmin[2], __uint_as_float(ref_of(i + 1)));
        p.l_hi = make_float4(l.bmax[0], l.bmax[1], l.bmax[2], __uint_as_float(ref_of(in[i].a)));
        p.r_lo = make_float4(r.bmin[0], r.bmin[1], r.bmin[2], __uint_as_float(in[i].b));
        p.r_hi = make_float4(r.bmax[0], r.bmax[1], r.bmax[2], 0.f);
    }
    fb.hdr->pairs = fb.pairs;
    fb.hdr->root_lo = make_float4(in[0].bmin[0], in[0].bmin[1], in[0].bmin[2], __uint_as_float(ref_of(0)));
    fb.hdr->root_hi = make_float4(in[0].bmax[0], in[0].bmax[1], in[0].bmax[2], 0.f);
    fb.counts[0] = B.n_nodes; fb.counts[1] = B.n_order; fb.counts[2] = ok ? 1u : 0u;
}

// RenderTarget::get_render (render_target.rs:185-210) + Colorf::to_srgb (color.rs:59-72)
__global__ void k_srgb8(size_t n, const float4* __restrict__ film, uint8_t* __restrict__ rgb8) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float4 c = film[i];
        uint8_t o[3];
        srgb8_pixel(c.x, c.y, c.z, c.w, o); // trb_detmath.cuh, shared with trb_host_film_to_srgb8
        rgb8[3 * i] = o[0]; rgb8[3 * i + 1] = o[1]; rgb8[3 * i + 2] = o[2];
    }
}

// ==========================================================================================
// Adaptive sampler (src/sampler/adaptive.rs driven by thread_work, multithreaded.rs:72-114; DESIGN.md §2 and §5). A render is
// a sequence of rounds over the selected blocks; a round is cut into passes by block sub-ranges only, so one pass holds all of a
// pixel's samples of the round. Per pass: k_wf_generate_ad, the unchanged trace / shade rounds (the per-path sample arrays get
// the round's LD offset), the film kernels' ADAPT variant, then k_ad_decide. Between rounds k_ad_compact keeps the blocks that
// still have a pixel sampling. The rounds are driven by the device: the host enqueues every round with the passes the whole
// selection would need, and each pass reads the live length of its round's list (RenderParams::ad_live, ad_pass_blocks) and
// does nothing past it.
// ==========================================================================================
// A pass's path p = (block, pixel, entry) as in LowDiscrepancy, slot = sample_first + entry. Only the paths of pixels that are
// still sampling are queued for the primary trace (warp-aggregated push) and counted as camera samples; the others enter shade
// round 0 as primary misses, which only writes a black sample that neither the film nor the decision reads. The pass's real
// path count goes to WF_N_ACTIVE (shade round 0) and WF_N_PATHS (the keyframed tables); an empty pass leaves every count 0.
template <bool ANIM>
__global__ void __launch_bounds__(256) k_wf_generate_ad(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf) {
    const uint32_t n = ad_pass_blocks(rp) * 64 * rp.sample_count;
    if (n == 0) return;
    const uint32_t lane = threadIdx.x & 31, stride = gridDim.x * blockDim.x;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p - lane < n; p += stride) { // whole warps iterate (wf_push)
        bool on = false;
        if (p < n) {
            const SampleId id = sample_id(sc, rp, p);
            on = (rp.ad_state[id.pixel].x & trbh::AD_ACTIVE) != 0u;
            float time = 0.0f;
            if (on) {
                const PixelStreams ps = pixel_streams_round(rp.seed, id.pixel, rp.ad_round);
                float sx, sy, tm;
                sample_position_ad(rp, ps, id, sx, sy, tm);
                Ray ray;
                time = camera_ray<ANIM>(sc, sx, sy, tm, ray);
                wf.org[p] = make_float4(ray.o.x, ray.o.y, ray.o.z, __uint_as_float(0u));
                wf.cont[p] = make_float4(ray.d.x, ray.d.y, ray.d.z, finf());
            } else {
                wf.org[p] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(0u));
                wf.cont[p] = make_float4(0.0f, 0.0f, 0.0f, finf());
                wf.hit[p] = make_uint4(TRB_MISS, 0u, 0u, 0u);
            }
            wf.thr[p] = make_float4(1.0f, 1.0f, 1.0f, time);
            wf.illum[p] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
        const unsigned m = __ballot_sync(0xffffffffu, on);
        wf_push(wf.q_cont, &wf.counters[WF_N_CONT], on, p);
        if (lane == 0 && m && rp.stats) atomicAdd(&rp.stats->camera_samples, (unsigned long long)__popc(m));
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { wf.counters[WF_N_ACTIVE] = n; wf.counters[WF_N_PATHS] = n; } // shade round 0 walks every path of the pass
    if (wf.bounds && blockIdx.x == 0 && threadIdx.x < 64) { // empty origin boxes for every round's sort grid (nullptr: sorting off)
        uint32_t* b = wf.bounds + threadIdx.x * 8;
        b[0] = b[1] = b[2] = b[3] = 0xffffffffu; b[4] = b[5] = b[6] = b[7] = 0u;
    }
}

// report_results for every pixel of the pass that sampled this round: fold the round's luminances in slot order into the
// 16-byte state (trb_adaptive.h), decide, flag the block when the pixel goes on. With samples_out: the parity records
// (trb_render_samples_adaptive), max_per_pixel slots per pixel in the caller's block order.
__global__ void __launch_bounds__(128) k_ad_decide(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const __grid_constant__ WfState wf,
                                                   uint32_t* block_flags) {
    trbh::AdSchedule sch;
    sch.min = rp.ad_min; sch.max = rp.ad_max; sch.step = rp.ad_step; sch.max_per_pixel = rp.ad_max_per_pixel; sch.rounds = 0;
    const uint32_t n = ad_pass_blocks(rp) * 64;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        SampleId id;
        id.item = t >> 6; id.pix = t & 63;
        const uint2 blk = rp.blocks[id.item];
        id.px = blk.x * 8 + (id.pix & 7); id.py = blk.y * 8 + (id.pix >> 3); id.pixel = id.py * sc.width + id.px;
        const uint4 st4 = rp.ad_state[id.pixel];
        if (!(st4.x & trbh::AD_ACTIVE)) continue;
        trbh::AdPixel st; st.taken = st4.x; st.avg = __uint_as_float(st4.y); st.lmin = __uint_as_float(st4.z); st.lmax = __uint_as_float(st4.w);
        PixelStreams ps;
        if (rp.samples_out) ps = pixel_streams_round(rp.seed, id.pixel, rp.ad_round);
        for (uint32_t s = 0; s < rp.sample_count; ++s) {
            const float4 c = wf.rad[(size_t)t * rp.sample_count + s];
            const uint32_t slot = rp.sample_first + s;
            trbh::ad_add(st, slot, trbh::ad_luminance(c.x, c.y, c.z), rp.ad_round == 0);
            if (rp.samples_out) {
                id.si = slot;
                float sx, sy, tm;
                sample_position_ad(rp, ps, id, sx, sy, tm);
                trb_sample* out = reinterpret_cast<trb_sample*>(rp.samples_out) + ((size_t)rp.ad_block_index[id.item] * 64 + id.pix) * rp.ad_max_per_pixel + slot;
                out->x = sx; out->y = sy; out->r = c.x; out->g = c.y; out->b = c.z;
            }
        }
        const bool more = trbh::ad_finish(st, sch, rp.ad_round);
        rp.ad_state[id.pixel] = make_uint4(st.taken, __float_as_uint(st.avg), __float_as_uint(st.lmin), __float_as_uint(st.lmax));
        if (more) block_flags[id.item] = 1u;
    }
}

// The AOV records of a pass (k_wf_aov_ad: lo, hi indexed by path) into the parity layout of k_ad_decide's samples_out
// (trb_render_samples_adaptive_aov): path t * sample_count + s of a pixel sampling this round goes to slot sample_first + s.
// Runs before k_ad_decide, which clears the flag of a pixel that stops.
__global__ void __launch_bounds__(128) k_ad_aov_slots(const __grid_constant__ DScene sc, const __grid_constant__ RenderParams rp, const float4* __restrict__ lo,
                                                      const float4* __restrict__ hi, trb_aov_sample* __restrict__ out) {
    const uint32_t n = ad_pass_blocks(rp) * 64;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        const uint32_t item = t >> 6, pix = t & 63;
        const uint2 blk = rp.blocks[item];
        const uint32_t pixel = (blk.y * 8 + (pix >> 3)) * sc.width + blk.x * 8 + (pix & 7);
        if (!(rp.ad_state[pixel].x & trbh::AD_ACTIVE)) continue;
        float4* dst = reinterpret_cast<float4*>(out + ((size_t)rp.ad_block_index[item] * 64 + pix) * rp.ad_max_per_pixel + rp.sample_first);
        for (uint32_t s = 0; s < rp.sample_count; ++s) {
            const size_t p = (size_t)t * rp.sample_count + s;
            dst[2 * s] = lo[p];
            dst[2 * s + 1] = hi[p];
        }
    }
}

// Start of a render: every pixel of the selected blocks samples round 0; the round list starts as the selection.
__global__ void k_ad_init(const __grid_constant__ DScene sc, const uint2* blocks, uint32_t n_blocks, uint4* state, uint2* list, uint32_t* list_index,
                          uint32_t* list_count) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *list_count = n_blocks;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_blocks * 64; t += gridDim.x * blockDim.x) {
        const uint2 blk = blocks[t >> 6];
        const uint32_t pixel = (blk.y * 8 + ((t & 63) >> 3)) * sc.width + blk.x * 8 + (t & 7);
        const trbh::AdPixel p = trbh::ad_initial();
        state[pixel] = make_uint4(p.taken, __float_as_uint(p.avg), __float_as_uint(p.lmin), __float_as_uint(p.lmax));
        if ((t & 63) == 0) { list[t >> 6] = blk; list_index[t >> 6] = t >> 6; }
    }
}

// Order-preserving compaction of the round's block list to the blocks flagged by k_ad_decide (one CTA; at most ~32 K blocks
// at 1080p). Clears the flags it read. in_count / out_count: the lists' lengths, which stay on the device (one word per list,
// so a round reads its input length while it writes its output length).
__global__ void __launch_bounds__(1024) k_ad_compact(uint32_t* flags, const uint32_t* in_count, const uint2* in_list, const uint32_t* in_index,
                                                     uint2* out_list, uint32_t* out_index, uint32_t* out_count) {
    __shared__ uint32_t part[1024];
    __shared__ uint32_t base;
    const uint32_t n = *in_count;
    if (threadIdx.x == 0) base = 0;
    for (uint32_t c0 = 0; c0 < n; c0 += 1024) {
        const uint32_t i = c0 + threadIdx.x;
        const uint32_t f = i < n && flags[i] ? 1u : 0u;
        __syncthreads();
        part[threadIdx.x] = f;
        __syncthreads();
        for (uint32_t s = 1; s < 1024; s <<= 1) { // Hillis-Steele inclusive scan
            const uint32_t v = threadIdx.x >= s ? part[threadIdx.x - s] : 0u;
            __syncthreads();
            part[threadIdx.x] += v;
            __syncthreads();
        }
        if (f) { const uint32_t o = base + part[threadIdx.x] - 1u; out_list[o] = in_list[i]; out_index[o] = in_index[i]; }
        if (i < n) flags[i] = 0u;
        __syncthreads();
        if (threadIdx.x == 1023) base += part[1023];
    }
    __syncthreads();
    if (threadIdx.x == 0) *out_count = base;
}

// Samples per pixel of the selected blocks (the reference's per-pixel count: samples_taken when report_results let go), written
// at spp[y * width + x]; other pixels are not touched
__global__ void k_ad_pixel_spp(const __grid_constant__ DScene sc, const uint2* blocks, uint32_t n_blocks, const uint4* state, uint32_t* spp) {
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_blocks * 64; t += gridDim.x * blockDim.x) {
        const uint2 blk = blocks[t >> 6];
        const uint32_t pixel = (blk.y * 8 + ((t & 63) >> 3)) * sc.width + blk.x * 8 + (t & 7);
        spp[pixel] = state[pixel].x & ~trbh::AD_ACTIVE;
    }
}

// ------------------------------------------------------------------------------------------
// Caller film writes (trb_film_write; DESIGN.md §5): RenderTarget::write (render_target.rs:77-165) once per region that has
// samples, regions in Morton-list order, each region's samples in input order — without float atomics. The samples are
// stable-sorted by region (CUB radix sort, launched from trb_api.cu), then one CTA per target 8x8 block gathers, for each of
// its 64 pixels (one owner thread each), the sum S_r of every candidate region r in Morton order and adds it to the film.
// ------------------------------------------------------------------------------------------
// Sort keys: the sample's region, or n_regions for a region out of range (sorted last, never written); values: input positions.
__global__ void k_film_keys(uint32_t n, const uint32_t* __restrict__ regions, uint32_t n_regions, uint32_t* __restrict__ keys,
                            uint32_t* __restrict__ order) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t r = regions[i];
        keys[i] = r < n_regions ? r : n_regions;
        order[i] = i;
    }
}

// start[r] = the first sorted position whose key is >= r, for r in [0, n_regions]: region r's samples are [start[r], start[r + 1]).
__global__ void k_film_starts(uint32_t n, const uint32_t* __restrict__ keys, uint32_t n_regions, uint32_t* __restrict__ start) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= n_regions; r += gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = n;
        while (lo < hi) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (keys[mid] < r) lo = mid + 1; else hi = mid;
        }
        start[r] = lo;
    }
}

// morton.rs: the Morton code of block (x, y). Codes of distinct blocks differ, so ordering blocks by code is their order in
// BlockQueue::new's stably sorted list (block_queue.rs:28-46).
__device__ __forceinline__ uint32_t morton_block(uint32_t x, uint32_t y) {
    auto part = [](uint32_t v) {
        v &= 0x0000ffffu; v = (v ^ (v << 8)) & 0x00ff00ffu; v = (v ^ (v << 4)) & 0x0f0f0f0fu;
        v = (v ^ (v << 2)) & 0x33333333u; return (v ^ (v << 1)) & 0x55555555u;
    };
    return (part(y) << 1) + part(x);
}

constexpr int FILM_WRITE_THREADS = 64; // one thread per pixel of the target block
constexpr int FILM_CHUNK = 512;        // samples staged in shared memory at a time

// One CTA per target 8x8 block. Candidate regions are those whose write range [start - fpw, start + 8 + fpw] (inclusive,
// clipped to the image; render_target.rs:79-82) reaches the block: the 3x3 neighbours for fpw <= 7, 4x4 (two blocks to the
// left and above) for fpw = 8. Per candidate with samples, each pixel inside its write range sums weight * c and weight over
// the region's samples in input order (the lock-block test of render_target.rs:105-110 always applies here: caller positions
// may be anywhere, NaN included), then adds that sum to its film value, as RenderTarget::write adds filtered_samples.
__global__ void __launch_bounds__(FILM_WRITE_THREADS) k_film_gather(const __grid_constant__ DScene sc, const trb_sample* __restrict__ samples,
                                                                    const uint32_t* __restrict__ order, const uint32_t* __restrict__ start,
                                                                    float* __restrict__ film) {
    __shared__ float s_table[256];
    __shared__ float s_x[FILM_CHUNK], s_y[FILM_CHUNK], s_r[FILM_CHUNK], s_g[FILM_CHUNK], s_b[FILM_CHUNK];
    __shared__ uint32_t s_cand[16], s_code[16];
    __shared__ int s_ncand;
    const uint32_t nbx = sc.width / 8, nby = sc.height / 8;
    const uint32_t tbx = blockIdx.x % nbx, tby = blockIdx.x / nbx;
    for (int i = threadIdx.x; i < 256; i += FILM_WRITE_THREADS) s_table[i] = sc.filter_table[i];
    if (threadIdx.x == 0) { // the candidate regions with samples, sorted by Morton code (insertion sort of at most 16)
        int nc = 0;
        const uint32_t bx0 = (uint32_t)max((int)tbx - (8 + sc.fpw_x) / 8, 0), bx1 = min(tbx + (uint32_t)(7 + sc.fpw_x) / 8, nbx - 1);
        const uint32_t by0 = (uint32_t)max((int)tby - (8 + sc.fpw_y) / 8, 0), by1 = min(tby + (uint32_t)(7 + sc.fpw_y) / 8, nby - 1);
        for (uint32_t by = by0; by <= by1; ++by)
            for (uint32_t bx = bx0; bx <= bx1; ++bx) {
                const uint32_t r = by * nbx + bx;
                if (start[r + 1] == start[r]) continue; // no samples: RenderTarget::write is not called for it
                const uint32_t code = morton_block(bx, by);
                int k = nc++;
                for (; k > 0 && s_code[k - 1] > code; --k) { s_code[k] = s_code[k - 1]; s_cand[k] = s_cand[k - 1]; }
                s_code[k] = code; s_cand[k] = r;
            }
        s_ncand = nc;
    }
    __syncthreads();
    const int ix = (int)(tbx * 8 + (threadIdx.x & 7)), iy = (int)(tby * 8 + (threadIdx.x >> 3));
    float* px = film + ((size_t)iy * sc.width + ix) * 4;
    float f0 = px[0], f1 = px[1], f2 = px[2], f3v = px[3];
    bool touched = false;
    const int nc = s_ncand;
    for (int c = 0; c < nc; ++c) {
        const uint32_t r = s_cand[c];
        const int rx = (int)(r % nbx) * 8, ry = (int)(r / nbx) * 8;
        const int x_lo = max(rx - sc.fpw_x, 0), x_hi = min(rx + 8 + sc.fpw_x, (int)sc.width - 1);
        const int y_lo = max(ry - sc.fpw_y, 0), y_hi = min(ry + 8 + sc.fpw_y, (int)sc.height - 1);
        const bool in = ix >= x_lo && ix <= x_hi && iy >= y_lo && iy <= y_hi;
        float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f; // filtered_samples[px] (render_target.rs:112-114)
        const uint32_t s0 = start[r], s1 = start[r + 1];
        for (uint32_t b = s0; b < s1; b += FILM_CHUNK) {
            const uint32_t cnt = min(s1 - b, (uint32_t)FILM_CHUNK);
            __syncthreads();
            for (uint32_t j = threadIdx.x; j < cnt; j += FILM_WRITE_THREADS) {
                const trb_sample* sp = samples + order[b + j];
                s_x[j] = sp->x; s_y[j] = sp->y; s_r[j] = sp->r; s_g[j] = sp->g; s_b[j] = sp->b;
            }
            __syncthreads();
            if (!in) continue;
            for (uint32_t j = 0; j < cnt; ++j) {
                const float sx = s_x[j], sy = s_y[j];
                if (!lock_block_takes(sx, ix, x_lo, x_hi, sc.fpw_x) || !lock_block_takes(sy, iy, y_lo, y_hi, sc.fpw_y)) continue;
                const float fy = fabsf((float)iy - (sy - 0.5f)) * sc.filter_inv_h;
                if (fy > sc.filter_h) continue; // sic: normalised distance vs width (A7)
                const float fx = fabsf((float)ix - (sx - 0.5f)) * sc.filter_inv_w;
                if (fx > sc.filter_w) continue;
                const uint32_t fyi = min(f2u(fy * 16.0f), 15u), fxi = min(f2u(fx * 16.0f), 15u);
                const float wgt = s_table[fyi * 16 + fxi];
                a0 += wgt * s_r[j];
                a1 += wgt * s_g[j];
                a2 += wgt * s_b[j];
                a3 += wgt;
            }
        }
        if (in) { f0 += a0; f1 += a1; f2 += a2; f3v += a3; touched = true; } // pixels[px] += filtered_samples[px] (:153-161)
    }
    if (touched) { px[0] = f0; px[1] = f1; px[2] = f2; px[3] = f3v; }
}

} // namespace trb
