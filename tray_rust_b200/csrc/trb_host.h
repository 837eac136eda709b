// trb_host.h — host side of the GPU render path: the per-frame preparation the reference does inside
// Scene::load_file / Scene::update_frame, restated in C++ so the kernels receive flat arrays.
//
//   Mat4 / Xf            src/linalg/matrix4.rs, src/linalg/transform.rs
//   keyframe_xf          src/linalg/keyframe.rs:60-63, src/linalg/quaternion.rs:65-84
//   instance_world_xf    src/linalg/animated_transform.rs:40-56 (static instances)
//   arvo_bounds          src/linalg/transform.rs:256-281
//   BvhBuilder           src/geometry/bvh.rs:139-267, src/partition.rs:9-38
//   CameraSetup          src/film/camera.rs:64-91,127-144
//   filter_table         src/film/render_target.rs:41-59, src/film/filter/*.rs
//   morton_blocks        src/sampler/block_queue.rs:28-46, src/sampler/morton.rs
//
// Host arithmetic is compiled with -ffp-contract=off: every matrix the kernels read must carry the
// reference's bits (SURVEY Q14: the renderer uses the T*R*S recomposition, not the JSON matrix).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/trb.h"

// Functions marked TRB_HD are shared by the host (per-frame preparation, TLAS bounds) and the device (per-ray
// evaluation of animated transforms); both compilers evaluate them without FMA contraction, so the bits agree.
#ifdef __CUDACC__
#define TRB_HD __host__ __device__
#else
#define TRB_HD
#endif

namespace trbh {

constexpr float kPi = 3.14159265358979323846f;
constexpr float kEps = 1.1920929e-7f;

struct Mat4 { float m[16]; };

TRB_HD inline Mat4 mat_identity() { Mat4 r; for (int i = 0; i < 16; ++i) r.m[i] = 0.0f; r.m[0] = r.m[5] = r.m[10] = r.m[15] = 1.0f; return r; }
TRB_HD inline Mat4 mat_mul(const Mat4& a, const Mat4& b) { // matrix4.rs:232-247
    Mat4 r;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            r.m[4 * i + j] = a.m[4 * i] * b.m[j] + a.m[4 * i + 1] * b.m[4 + j] + a.m[4 * i + 2] * b.m[8 + j] + a.m[4 * i + 3] * b.m[12 + j];
    return r;
}
// 3x3 sub-determinant helper: returns x*y*z with the reference's left-to-right product order
TRB_HD inline float p3(float x, float y, float z) { return x * y * z; }
// Matrix4::inverse (matrix4.rs:48-172): cofactor expansion, each cofactor a 6-term signed sum in the source order.
TRB_HD inline Mat4 mat_inverse(const Mat4& s) {
    const float* a = s.m;
    Mat4 out;
    float* v = out.m;
    v[0] = p3(a[5], a[10], a[15]) - p3(a[5], a[11], a[14]) - p3(a[9], a[6], a[15]) + p3(a[9], a[7], a[14]) + p3(a[13], a[6], a[11]) - p3(a[13], a[7], a[10]);
    v[4] = p3(-a[4], a[10], a[15]) + p3(a[4], a[11], a[14]) + p3(a[8], a[6], a[15]) - p3(a[8], a[7], a[14]) - p3(a[12], a[6], a[11]) + p3(a[12], a[7], a[10]);
    v[8] = p3(a[4], a[9], a[15]) - p3(a[4], a[11], a[13]) - p3(a[8], a[5], a[15]) + p3(a[8], a[7], a[13]) + p3(a[12], a[5], a[11]) - p3(a[12], a[7], a[9]);
    v[12] = p3(-a[4], a[9], a[14]) + p3(a[4], a[10], a[13]) + p3(a[8], a[5], a[14]) - p3(a[8], a[6], a[13]) - p3(a[12], a[5], a[10]) + p3(a[12], a[6], a[9]);
    v[1] = p3(-a[1], a[10], a[15]) + p3(a[1], a[11], a[14]) + p3(a[9], a[2], a[15]) - p3(a[9], a[3], a[14]) - p3(a[13], a[2], a[11]) + p3(a[13], a[3], a[10]);
    v[5] = p3(a[0], a[10], a[15]) - p3(a[0], a[11], a[14]) - p3(a[8], a[2], a[15]) + p3(a[8], a[3], a[14]) + p3(a[12], a[2], a[11]) - p3(a[12], a[3], a[10]);
    v[9] = p3(-a[0], a[9], a[15]) + p3(a[0], a[11], a[13]) + p3(a[8], a[1], a[15]) - p3(a[8], a[3], a[13]) - p3(a[12], a[1], a[11]) + p3(a[12], a[3], a[9]);
    v[13] = p3(a[0], a[9], a[14]) - p3(a[0], a[10], a[13]) - p3(a[8], a[1], a[14]) + p3(a[8], a[2], a[13]) + p3(a[12], a[1], a[10]) - p3(a[12], a[2], a[9]);
    v[2] = p3(a[1], a[6], a[15]) - p3(a[1], a[7], a[14]) - p3(a[5], a[2], a[15]) + p3(a[5], a[3], a[14]) + p3(a[13], a[2], a[7]) - p3(a[13], a[3], a[6]);
    v[6] = p3(-a[0], a[6], a[15]) + p3(a[0], a[7], a[14]) + p3(a[4], a[2], a[15]) - p3(a[4], a[3], a[14]) - p3(a[12], a[2], a[7]) + p3(a[12], a[3], a[6]);
    v[10] = p3(a[0], a[5], a[15]) - p3(a[0], a[7], a[13]) - p3(a[4], a[1], a[15]) + p3(a[4], a[3], a[13]) + p3(a[12], a[1], a[7]) - p3(a[12], a[3], a[5]);
    v[14] = p3(-a[0], a[5], a[14]) + p3(a[0], a[6], a[13]) + p3(a[4], a[1], a[14]) - p3(a[4], a[2], a[13]) - p3(a[12], a[1], a[6]) + p3(a[12], a[2], a[5]);
    v[3] = p3(-a[1], a[6], a[11]) + p3(a[1], a[7], a[10]) + p3(a[5], a[2], a[11]) - p3(a[5], a[3], a[10]) - p3(a[9], a[2], a[7]) + p3(a[9], a[3], a[6]);
    v[7] = p3(a[0], a[6], a[11]) - p3(a[0], a[7], a[10]) - p3(a[4], a[2], a[11]) + p3(a[4], a[3], a[10]) + p3(a[8], a[2], a[7]) - p3(a[8], a[3], a[6]);
    v[11] = p3(-a[0], a[5], a[11]) + p3(a[0], a[7], a[9]) + p3(a[4], a[1], a[11]) - p3(a[4], a[3], a[9]) - p3(a[8], a[1], a[7]) + p3(a[8], a[3], a[5]);
    v[15] = p3(a[0], a[5], a[10]) - p3(a[0], a[6], a[9]) - p3(a[4], a[1], a[10]) + p3(a[4], a[2], a[9]) + p3(a[8], a[1], a[6]) - p3(a[8], a[2], a[5]);
    float det = a[0] * v[0] + a[1] * v[4] + a[2] * v[8] + a[3] * v[12];
    det = 1.0f / det;
    for (int i = 0; i < 16; ++i) v[i] *= det;
    return out;
}

// Transform {mat, inv} (transform.rs:10-15)
struct Xf { Mat4 fwd, inv; };
TRB_HD inline Xf xf_identity() { return Xf{mat_identity(), mat_identity()}; }
TRB_HD inline Xf xf_compose(const Xf& l, const Xf& r) { return Xf{mat_mul(l.fwd, r.fwd), mat_mul(r.inv, l.inv)}; } // transform.rs:191-197
TRB_HD inline Xf xf_translate(const float t[3]) {
    Xf x = xf_identity();
    for (int i = 0; i < 3; ++i) { x.fwd.m[4 * i + 3] = t[i]; x.inv.m[4 * i + 3] = -t[i]; }
    return x;
}
TRB_HD inline Xf xf_scale(const float s[3]) {
    Xf x = xf_identity();
    for (int i = 0; i < 3; ++i) { x.fwd.m[5 * i] = s[i]; x.inv.m[5 * i] = 1.0f / s[i]; }
    return x;
}
TRB_HD inline Xf xf_from_mat(const Mat4& m) { return Xf{m, mat_inverse(m)}; }
TRB_HD inline Xf xf_inverse(const Xf& x) { return Xf{x.inv, x.fwd}; }

// Quaternion::to_matrix (quaternion.rs:65-84): the rotation matrix of (x,y,z,w). The source writes the
// transposed literal and transposes it; element (r,c) below is the source literal's (c,r).
TRB_HD inline Mat4 quat_matrix(const float q[4]) {
    const float x = q[0], y = q[1], z = q[2], w = q[3];
    Mat4 r = mat_identity();
    r.m[0] = 1.0f - 2.0f * (y * y + z * z); r.m[1] = 2.0f * (x * y - z * w);        r.m[2] = 2.0f * (x * z + y * w);
    r.m[4] = 2.0f * (x * y + z * w);        r.m[5] = 1.0f - 2.0f * (x * x + z * z); r.m[6] = 2.0f * (y * z - x * w);
    r.m[8] = 2.0f * (x * z - y * w);        r.m[9] = 2.0f * (y * z + x * w);        r.m[10] = 1.0f - 2.0f * (x * x + y * y);
    return r;
}
// Keyframe::transform (keyframe.rs:60-63): (translate * from_mat(rot)) * scale
TRB_HD inline Xf keyframe_xf(const trb_keyframe& k) {
    return xf_compose(xf_compose(xf_translate(k.translation), xf_from_mat(quat_matrix(k.rotation))), xf_scale(k.scaling));
}

struct Box3 { float lo[3], hi[3]; };
inline Box3 box_empty() { Box3 b; for (int i = 0; i < 3; ++i) { b.lo[i] = INFINITY; b.hi[i] = -INFINITY; } return b; }
inline void box_grow(Box3& b, const Box3& o) { for (int i = 0; i < 3; ++i) { b.lo[i] = fminf(b.lo[i], o.lo[i]); b.hi[i] = fmaxf(b.hi[i], o.hi[i]); } }
inline void box_grow_pt(Box3& b, const float p[3]) { for (int i = 0; i < 3; ++i) { b.lo[i] = fminf(b.lo[i], p[i]); b.hi[i] = fmaxf(b.hi[i], p[i]); } }
inline float box_area(const Box3& b) { // bbox.rs:66-69
    const float dx = b.hi[0] - b.lo[0], dy = b.hi[1] - b.lo[1], dz = b.hi[2] - b.lo[2];
    return 2.0f * (dx * dy + dx * dz + dy * dz);
}
inline int box_longest_axis(const Box3& b) { // bbox.rs:47-56
    const float dx = b.hi[0] - b.lo[0], dy = b.hi[1] - b.lo[1], dz = b.hi[2] - b.lo[2];
    if (dx > dy && dx > dz) return 0;
    return dy > dz ? 1 : 2;
}
// Transform * BBox (Arvo), transform.rs:256-281
TRB_HD inline Box3 arvo_bounds(const Mat4& m, const Box3& b) {
    Box3 o;
    for (int i = 0; i < 3; ++i) o.lo[i] = o.hi[i] = m.m[4 * i + 3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const float x = m.m[4 * i + j] * b.lo[j], y = m.m[4 * i + j] * b.hi[j];
            if (x < y) { o.lo[i] += x; o.hi[i] += y; } else { o.lo[i] += y; o.hi[i] += x; }
        }
    return o;
}

// ---------------------------------------------------------------------------------------------
// SAH BVH2 in the reference's exact topology and order (bvh.rs:139-267, partition.rs:9-38), emitting the flattened
// pre-order array directly (the reference builds a pointer tree and flattens it depth-first; both visit nodes in the same
// order). ONE implementation for the host (per-mesh BLAS at load time, TLAS when the device path is off) and the device
// (TLAS per update_frame, k_tlas_build): iterative with an explicit task stack — device recursion would need a stack
// reservation for every resident thread — on caller-provided arrays.
// ---------------------------------------------------------------------------------------------
TRB_HD inline Box3 box_empty_hd() { Box3 b; for (int i = 0; i < 3; ++i) { b.lo[i] = INFINITY; b.hi[i] = -INFINITY; } return b; }
TRB_HD inline void box_grow_hd(Box3& b, const Box3& o) { for (int i = 0; i < 3; ++i) { b.lo[i] = fminf(b.lo[i], o.lo[i]); b.hi[i] = fmaxf(b.hi[i], o.hi[i]); } }
TRB_HD inline float box_area_hd(const Box3& b) { // bbox.rs:66-69
    const float dx = b.hi[0] - b.lo[0], dy = b.hi[1] - b.lo[1], dz = b.hi[2] - b.lo[2];
    return 2.0f * (dx * dy + dx * dz + dy * dz);
}
TRB_HD inline uint32_t sat_u32_hd(float f) { if (!(f > 0.0f)) return 0; if (f >= 4294967296.0f) return 0xffffffffu; return (uint32_t)f; }

struct BvhBuildArrays {
    const Box3* boxes; uint32_t n; uint32_t max_geom;
    float* cx; float* cy; float* cz;   // scratch [n]: centroids = lo*0.5 + hi*0.5 (bbox.rs:58-61 via linalg::lerp)
    uint32_t* idx;                     // scratch [n]
    uint32_t* task;                    // scratch [3 * n]: pending right subtrees (begin, end, parent)
    trb_bvh_node* nodes;               // out [2 * n]
    uint32_t* order;                   // out [n]: ordered_geom
    uint32_t n_nodes, n_order;
};

TRB_HD inline void bvh_build_arrays(BvhBuildArrays& B) {
    const Box3* boxes = B.boxes;
    uint32_t* idx = B.idx;
    for (uint32_t i = 0; i < B.n; ++i) {
        B.cx[i] = boxes[i].lo[0] * (1.0f - 0.5f) + boxes[i].hi[0] * 0.5f;
        B.cy[i] = boxes[i].lo[1] * (1.0f - 0.5f) + boxes[i].hi[1] * 0.5f;
        B.cz[i] = boxes[i].lo[2] * (1.0f - 0.5f) + boxes[i].hi[2] * 0.5f;
        idx[i] = i;
    }
    B.n_nodes = 0; B.n_order = 0;
    uint32_t n_task = 0;
    uint32_t begin = 0, end = B.n, parent = 0xffffffffu; // the range being emitted; parent != ~0: this node is that interior's second child
    for (;;) {
        // ---- BVH::build (bvh.rs:139-232) over idx[begin, end): emit one node, descend into its first child or pop a pending second child
        const uint32_t n = end - begin;
        const uint32_t me = B.n_nodes++;
        if (parent != 0xffffffffu) B.nodes[parent].a = me; // second_child index (bvh.rs:259-262)
        Box3 bounds = box_empty_hd();
        for (uint32_t i = begin; i < end; ++i) box_grow_hd(bounds, boxes[idx[i]]);
        bool is_leaf = false;
        int axis = 0;
        uint32_t mid = begin + n / 2;
        if (n == 1) is_leaf = true;
        else {
            Box3 cb = box_empty_hd();
            for (uint32_t i = begin; i < end; ++i) {
                const uint32_t g = idx[i];
                cb.lo[0] = fminf(cb.lo[0], B.cx[g]); cb.hi[0] = fmaxf(cb.hi[0], B.cx[g]);
                cb.lo[1] = fminf(cb.lo[1], B.cy[g]); cb.hi[1] = fmaxf(cb.hi[1], B.cy[g]);
                cb.lo[2] = fminf(cb.lo[2], B.cz[g]); cb.hi[2] = fmaxf(cb.hi[2], B.cz[g]);
            }
            { // bbox.rs:47-56 max_extent
                const float dx = cb.hi[0] - cb.lo[0], dy = cb.hi[1] - cb.lo[1], dz = cb.hi[2] - cb.lo[2];
                axis = (dx > dy && dx > dz) ? 0 : (dy > dz ? 1 : 2);
            }
            const float* cen = axis == 0 ? B.cx : (axis == 1 ? B.cy : B.cz);
            if (fabsf(cb.hi[axis] - cb.lo[axis]) < kEps) { // coincident centroids (bvh.rs:156-166)
                if (n < B.max_geom) is_leaf = true;
            } else if (n < 5) { // stable sort by centroid, median split (bvh.rs:169-178); insertion sort == stable
                for (uint32_t i = begin + 1; i < end; ++i) {
                    const uint32_t g = idx[i];
                    const float key = cen[g];
                    uint32_t j = i;
                    while (j > begin && cen[idx[j - 1]] > key) { idx[j] = idx[j - 1]; --j; }
                    idx[j] = g;
                }
            } else {
                const float cmin = cb.lo[axis], cmax = cb.hi[axis];
                uint32_t count[12];
                Box3 bb[12];
                for (int k = 0; k < 12; ++k) { count[k] = 0; bb[k] = box_empty_hd(); }
                for (uint32_t i = begin; i < end; ++i) {
                    uint32_t k = sat_u32_hd((cen[idx[i]] - cmin) / (cmax - cmin) * 12.0f);
                    if (k >= 12) k = 11;
                    count[k]++;
                    box_grow_hd(bb[k], boxes[idx[i]]);
                }
                float best_cost = INFINITY; int best = 0;
                const float total_area = box_area_hd(bounds);
                for (int sp = 0; sp < 11; ++sp) { // cost of splitting after bucket sp (bvh.rs:191-206)
                    Box3 lb = box_empty_hd(), rb = box_empty_hd();
                    uint32_t lc = 0, rc = 0;
                    for (int k = 0; k <= sp; ++k) { box_grow_hd(lb, bb[k]); lc += count[k]; }
                    for (int k = sp + 1; k < 12; ++k) { box_grow_hd(rb, bb[k]); rc += count[k]; }
                    const float cost = 0.125f + ((float)lc * box_area_hd(lb) + (float)rc * box_area_hd(rb)) / total_area;
                    if (cost < best_cost) { best_cost = cost; best = sp; }
                }
                if (n > B.max_geom || best_cost < (float)n) {
                    // partition.rs:9-38: two-ended, swaps the first "false" from the front with the first "true" from the back
                    uint32_t lo = begin, hi = end, split = begin;
                    for (;;) {
                        long f = -1, bk = -1;
                        while (lo < hi) { const uint32_t p = lo++; uint32_t k = sat_u32_hd((cen[idx[p]] - cmin) / (cmax - cmin) * 12.0f); if (k >= 12) k = 11; if (k > (uint32_t)best) { f = p; break; } split++; }
                        while (lo < hi) { const uint32_t p = --hi; uint32_t k = sat_u32_hd((cen[idx[p]] - cmin) / (cmax - cmin) * 12.0f); if (k >= 12) k = 11; if (k <= (uint32_t)best) { bk = p; break; } }
                        if (f < 0 || bk < 0) break;
                        const uint32_t tmp = idx[f]; idx[f] = idx[bk]; idx[bk] = tmp;
                        split++;
                    }
                    mid = split;
                } else is_leaf = true;
            }
        }
        trb_bvh_node& nd = B.nodes[me];
        for (int i = 0; i < 3; ++i) { nd.bmin[i] = bounds.lo[i]; nd.bmax[i] = bounds.hi[i]; }
        if (is_leaf) {
            nd.a = B.n_order; nd.b = TRB_BVH_LEAF | n;
            for (uint32_t i = begin; i < end; ++i) B.order[B.n_order++] = idx[i];
            if (n_task == 0) break;
            n_task--;
            begin = B.task[3 * n_task]; end = B.task[3 * n_task + 1]; parent = B.task[3 * n_task + 2];
        } else {
            nd.a = 0; nd.b = (uint32_t)axis;
            B.task[3 * n_task] = mid; B.task[3 * n_task + 1] = end; B.task[3 * n_task + 2] = me; n_task++; // second child later
            end = mid; parent = 0xffffffffu;                                                                 // first child = next node (bvh.rs:255)
        }
    }
    // BuildNode::interior: an interior node's bounds are the union of its children's (bvh.rs:358-362); children follow their parent
    for (uint32_t i = B.n_nodes; i-- > 0;) {
        trb_bvh_node& nd = B.nodes[i];
        if (nd.b & TRB_BVH_LEAF) continue;
        const trb_bvh_node& l = B.nodes[i + 1];
        const trb_bvh_node& r = B.nodes[nd.a];
        for (int k = 0; k < 3; ++k) { nd.bmin[k] = fminf(l.bmin[k], r.bmin[k]); nd.bmax[k] = fmaxf(l.bmax[k], r.bmax[k]); }
    }
}

// When bvh_build_arrays ends. A split that returns `begin` or `end` never shrinks its range: the first child is then empty (n = 0:
// no leaf case matches, and it splits into itself again) or the whole range, and either repeats for ever while the task stack grows
// past its array. It happens exactly where a node of more than max_geom elements has all its centroids in one bucket, which takes a
// centroid extent that is infinite or NaN: with a finite extent of at least kEps the element at cmin lands in bucket 0 and the one at
// cmax in bucket 11, and every split candidate (0..10) separates them. Bounds of magnitude at most 2^126 keep every centroid, and
// the difference of any two, finite. Trees of at most four elements never reach the buckets. The frame's instance tree is
// therefore built only over bounds that pass this test (or over at most four instances); the reference never finishes otherwise.
TRB_HD inline bool bvh_bound_buildable(float v) { return fabsf(v) <= 8.507059173023462e37f; } // 2^126; false for NaN

struct BvhBuilder { // host convenience over bvh_build_arrays
    std::vector<trb_bvh_node> nodes;
    std::vector<uint32_t> order; // ordered_geom
    void build(const std::vector<Box3>& b, uint32_t max_geom) {
        const size_t n = b.size();
        std::vector<float> cx(n), cy(n), cz(n);
        std::vector<uint32_t> idx(n), task(3 * n + 3);
        nodes.assign(2 * n, trb_bvh_node{}); order.assign(n, 0u);
        BvhBuildArrays B{b.data(), (uint32_t)n, max_geom, cx.data(), cy.data(), cz.data(), idx.data(), task.data(), nodes.data(), order.data(), 0, 0};
        bvh_build_arrays(B);
        nodes.resize(B.n_nodes); order.resize(B.n_order);
    }
};

// ---------------------------------------------------------------------------------------------
// film: filter table (render_target.rs:50-58), Mitchell-Netravali (mitchell_netravali.rs:35-55), Gaussian (gaussian.rs)
// ---------------------------------------------------------------------------------------------
inline float clamp01(float x) { return x < 0.0f ? 0.0f : (x > 1.0f ? 1.0f : x); }
inline float mitchell_1d(float x, float b, float c) {
    const float ax = fabsf(x);
    if (x >= 2.0f) return 0.0f; // signed x, as in the source
    if (x >= 1.0f)
        return 1.0f / 6.0f * ((-b - 6.0f * c) * powf(ax, 3.0f) + (6.0f * b + 30.0f * c) * powf(ax, 2.0f) + (-12.0f * b - 48.0f * c) * ax + (8.0f * b + 24.0f * c));
    return 1.0f / 6.0f * ((12.0f - 9.0f * b - 6.0f * c) * powf(ax, 3.0f) + (-18.0f + 12.0f * b + 6.0f * c) * powf(ax, 2.0f) + (6.0f - 2.0f * b));
}
inline void filter_table(const trb_film& f, float* table256) {
    const float inv_w = 1.0f / f.filter_w, inv_h = 1.0f / f.filter_h;
    const float b = clamp01(f.filter_b), c = clamp01(f.filter_c);
    const float alpha = f.filter_b;
    const float ex = expf(-alpha * f.filter_w * f.filter_w), ey = expf(-alpha * f.filter_h * f.filter_h);
    for (int y = 0; y < 16; ++y) {
        const float fy = ((float)y + 0.5f) * f.filter_h / 16.0f;
        for (int x = 0; x < 16; ++x) {
            const float fx = ((float)x + 0.5f) * f.filter_w / 16.0f;
            float w;
            if (f.filter_type == TRB_FILTER_MITCHELL_NETRAVALI) w = mitchell_1d(2.0f * fx * inv_w, b, c) * mitchell_1d(2.0f * fy * inv_h, b, c);
            else w = fmaxf(0.0f, expf(-alpha * fx * fx) - ex) * fmaxf(0.0f, expf(-alpha * fy * fy) - ey);
            table256[y * 16 + x] = w;
        }
    }
}

// sampler::morton + BlockQueue::new (morton.rs, block_queue.rs:28-46)
inline uint32_t spread_bits(uint32_t x) {
    x &= 0x0000ffffu; x = (x ^ (x << 8)) & 0x00ff00ffu; x = (x ^ (x << 4)) & 0x0f0f0f0fu; x = (x ^ (x << 2)) & 0x33333333u;
    return (x ^ (x << 1)) & 0x55555555u;
}
inline std::vector<uint32_t> morton_blocks(uint32_t w, uint32_t h, uint32_t start, uint32_t count, uint32_t shard_index = 0,
                                           uint32_t shard_count = 0, uint32_t shard_chunk = 0) {
    const uint32_t nbx = w / 8, nby = h / 8;
    std::vector<std::pair<uint32_t, uint32_t>> keyed(nbx * nby); // (morton, linear)
    for (uint32_t i = 0; i < nbx * nby; ++i) keyed[i] = {(spread_bits(i / nbx) << 1) + spread_bits(i % nbx), i};
    std::stable_sort(keyed.begin(), keyed.end(), [](const std::pair<uint32_t, uint32_t>& a, const std::pair<uint32_t, uint32_t>& b) { return a.first < b.first; });
    std::vector<uint32_t> out;
    size_t b0 = 0, b1 = keyed.size();
    if (count > 0) { b0 = std::min<size_t>(start, keyed.size()); b1 = std::min<size_t>(keyed.size(), (size_t)start + count); }
    const uint32_t chunk = shard_chunk ? shard_chunk : 1;
    for (size_t i = b0; i < b1; ++i) {
        if (shard_count > 1 && ((i - b0) / chunk) % shard_count != shard_index) continue; // interleaved multi-GPU sharding
        out.push_back(keyed[i].second % nbx); out.push_back(keyed[i].second / nbx);
    }
    return out;
}

// Camera::new (camera.rs:64-91): returns proj_div_inv * raster_screen and the fov scaling
inline void camera_setup(float fov, uint32_t w, uint32_t h, Mat4& px_to_cam, float scaling[3]) {
    const float aspect = (float)w / (float)h;
    float scr[4];
    if (aspect > 1.0f) { scr[0] = -aspect; scr[1] = aspect; scr[2] = -1.0f; scr[3] = 1.0f; }
    else { scr[0] = -1.0f; scr[1] = 1.0f; scr[2] = -1.0f / aspect; scr[3] = 1.0f / aspect; }
    const float s0[3] = {(float)w, (float)h, 1.0f};
    const float s1[3] = {1.0f / (scr[1] - scr[0]), 1.0f / (scr[2] - scr[3]), 1.0f};
    const float t0[3] = {-scr[0], -scr[3], 0.0f};
    const Xf screen_raster = xf_compose(xf_compose(xf_scale(s0), xf_scale(s1)), xf_translate(t0));
    const Xf raster_screen = xf_inverse(screen_raster);
    const float far = 1.0f, near = 1000.0f;
    Mat4 proj = mat_identity();
    proj.m[10] = far / (far - near); proj.m[11] = -far * near / (far - near); proj.m[14] = 1.0f; proj.m[15] = 0.0f;
    const Xf proj_div_inv = xf_inverse(xf_from_mat(proj));
    px_to_cam = xf_compose(proj_div_inv, raster_screen).fwd;
    const float tan_fov = tanf(kPi / 180.0f * fov / 2.0f); // f32::tan(linalg::to_radians(fov) / 2.0)
    scaling[0] = tan_fov; scaling[1] = tan_fov; scaling[2] = 1.0f;
}

} // namespace trbh
