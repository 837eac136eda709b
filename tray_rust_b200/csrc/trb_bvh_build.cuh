// trb_bvh_build.cuh — the reference's SAH BVH (bvh.rs:139-267, partition.rs:9-38) built on the device. The output is the
// host builder's (trbh::bvh_build_arrays): the same preorder trb_bvh_node array and the same ordered_geom, bit for bit but for
// the sign of a bound that ties between -0 and +0 (below).
//
// Shape of the build:
//   - Nodes of more than SMALL elements are built level by level over the whole array: per level, segmented reductions
//     (k_bvh_bounds, k_bvh_bins), one thread per node for each decision (k_bvh_axis, k_bvh_split), a prefix-sum partition
//     (k_bvh_flags, CUB scan, k_bvh_ranks, k_bvh_swap) and the children (k_bvh_children). The host reads the open-node count
//     once per level.
//   - A node of at most SMALL elements is a subtree one thread builds with the serial algorithm (k_bvh_small).
//   - The level nodes form a "top tree"; subtree node counts are summed bottom-up and preorder indices assigned top-down, one
//     launch per level (k_bvh_size, k_bvh_pre), then the nodes are written (k_bvh_emit, k_bvh_copy) and the interior bounds
//     recomputed from the children, left first, bottom-up (k_bvh_ibounds).
//
// Folds with signed zeros. Every fold here follows glibc's fminf / fmaxf: NaN operands are skipped and, when both are zeros
// of different sign, the FIRST operand is returned (fminf(+0, -0) = +0, fminf(-0, +0) = -0), so a bound is the first element
// (in the node's current order) holding the extreme value, ±0 being one value. CUDA's fminf compiles to PTX min.f32, which
// the PTX ISA orders with -0.0 < +0.0, so it is not used for boxes here: hmin / hmax restate glibc, and the parallel
// reductions reduce (ordered value with ±0 collapsed, position) pairs with 64-bit atomicMin / atomicMax, keeping the first
// position among equal values, and then read the winner's own bits. The host builder's zero signs do not follow one rule
// (where GCC lowers a fold inline the second operand wins; DESIGN.md §4 "Mesh BVH build"), so a bound that ties between -0
// and +0 may differ from the host's in its sign; every other bit, the topology and the order are the host's.
// Centroid bounds are reduced as plain values: their zero signs never reach a result (c - cmin and cmax - cmin give the
// same bucket for either sign, and the axis and coincidence tests compare magnitudes).
//
// The frame's instance tree (trb_scene_update_frame) is also built by one device thread running trbh::bvh_build_arrays
// (k_tlas_build), whose fminf / fmaxf are min.f32 / max.f32: a NaN operand is skipped and -0.0 orders below +0.0. The two rules
// differ only where a fold meets both zeros, and an instance bound is never -0: arvo_bounds starts each bound from the composed
// translation and adds products to it, a sum is -0 only when both operands are, and the translation entry of keyframe_xf and of
// every xf_compose of such transforms contains the term 1 * (+0) or ends in a term that is itself never -0 (DESIGN.md §4
// "`update_frame` on the device" has the induction). So this builder reproduces that kernel's bytes with the one rule above, which
// tests/test_tlas_build_gpu.py checks builder against builder, together with the absence of -0 bounds.
//
// The serial-subtree threshold (`small`, at least 4: the level kernels have no n == 1 and n < 5 cases) is an argument of the
// build: both phases run the same algorithm, so the tree does not depend on it. Meshes pass SMALL.
//
// Partition as a closed form (partition.rs:9-38). Let pred(x) = bucket(x) <= best, P the number of elements of [b, e) with
// pred true, L the positions of [b, b+P) with pred false in ascending order and R the positions of [b+P, e) with pred
// true in descending order; |L| = |R| because both equal P minus the trues in [b, b+P). The two-ended loop swaps L[k]
// with R[k] for every k and returns b+P. Proof, by induction on the loop's rounds: entering round k, the front cursor
// has passed exactly L[0..k) (each was swapped, and every true it stepped over stays in place) and the back cursor has
// passed exactly R[0..k). The front scan stops at the next false, which is L[k] if k < |L|; since every true ahead of
// it in [b, b+P) is left alone, it cannot cross b+P before exhausting L. The back scan stops at the next true from the
// end, R[k] if k < |R|, and never crosses b+P while an L remains, because the positions below b+P that it could reach are
// all at or after L[k]'s cursor. When L is exhausted the front cursor walks the remaining trues up to b+P and then meets
// only falses, or meets the back cursor; either way the loop ends with split = b+P. tests/test_device_bvh_cpu.py checks
// the closed form against a literal two-ended partition.
#pragma once
#include <cub/device/device_scan.cuh>
#include "trb_device.h"
#include "trb_host.h"

namespace trb {
namespace bvhb {

constexpr uint32_t SMALL = 1024;   // meshes: a node of at most SMALL elements is one thread's serial subtree
constexpr uint32_t NONE = 0xffffffffu;
enum : uint32_t { K_SAH = 0, K_LEAF = 1, K_KEEP = 2, K_PART = 3 }; // open node: undecided SAH, leaf, split in place, partition
enum : uint32_t { T_LEAF = 0, T_INTERIOR = 1, T_SMALL = 2 };        // top-tree node kinds

// glibc fminf / fmaxf: a NaN operand is skipped; between equal values (±0) the first operand is returned
__device__ __forceinline__ float hmin(float a, float b) { if (isnan(a)) return b; if (isnan(b)) return a; return b < a ? b : a; }
__device__ __forceinline__ float hmax(float a, float b) { if (isnan(a)) return b; if (isnan(b)) return a; return b > a ? b : a; }
__device__ __forceinline__ void hgrow(trbh::Box3& b, const trbh::Box3& o) {
    for (int i = 0; i < 3; ++i) { b.lo[i] = hmin(b.lo[i], o.lo[i]); b.hi[i] = hmax(b.hi[i], o.hi[i]); }
}
__device__ __forceinline__ trbh::Box3 load_box(const float* boxes, uint32_t g) {
    trbh::Box3 b;
    for (int i = 0; i < 3; ++i) { b.lo[i] = boxes[6 * (size_t)g + i]; b.hi[i] = boxes[6 * (size_t)g + 3 + i]; }
    return b;
}
// order-preserving key of a non-NaN float, -0 and +0 mapped to one key
__device__ __forceinline__ uint32_t okey(float v) {
    const uint32_t u = __float_as_uint(v == 0.0f ? 0.0f : v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float okey_inv(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }
__device__ __forceinline__ uint32_t bucket(float c, float cmin, float cmax) { // bvh.rs:183-186
    uint32_t k = trbh::sat_u32_hd((c - cmin) / (cmax - cmin) * 12.0f);
    return k >= 12 ? 11 : k;
}

// Reductions over the lanes of `grp` (lanes sharing one destination); the lowest lane of the group writes.
// Pair keys: min = value key << 32 | position, max = value key << 32 | ~position; empty = ~0 / 0.
__device__ __forceinline__ void red_min(unsigned grp, bool lead, float v, uint32_t pos, unsigned long long* dst) {
    const uint32_t k = isnan(v) ? 0xffffffffu : okey(v);
    const uint32_t km = __reduce_min_sync(grp, k);
    const uint32_t pm = __reduce_min_sync(grp, k == km ? pos : 0xffffffffu);
    if (lead && km != 0xffffffffu) atomicMin(dst, ((unsigned long long)km << 32) | pm);
}
__device__ __forceinline__ void red_max(unsigned grp, bool lead, float v, uint32_t pos, unsigned long long* dst) {
    const uint32_t k = isnan(v) ? 0u : okey(v);
    const uint32_t km = __reduce_max_sync(grp, k);
    const uint32_t pm = __reduce_min_sync(grp, k == km ? pos : 0xffffffffu);
    if (lead && km != 0u) atomicMax(dst, ((unsigned long long)km << 32) | (0xffffffffu - pm));
}
// the bits of the winning element (positions index the current order idx[])
__device__ __forceinline__ float dec_lo(unsigned long long key, const float* boxes, const uint32_t* idx, int c) {
    return key == ~0ull ? INFINITY : boxes[6 * (size_t)idx[(uint32_t)key] + c];
}
__device__ __forceinline__ float dec_hi(unsigned long long key, const float* boxes, const uint32_t* idx, int c) {
    return key == 0ull ? -INFINITY : boxes[6 * (size_t)idx[0xffffffffu - (uint32_t)key] + 3 + c];
}

struct Bin { unsigned long long lo[3], hi[3]; uint32_t cnt, pad; };
struct Open {                                  // a node of more than `small` elements, open at this level
    uint32_t begin, end, tn, kind;             // range of idx[], top-tree node, decision
    uint32_t axis, best, mid, pad;             // mid: first slot of the second child
    float cmin, cmax;
    uint32_t clo[3], chi[3];                   // centroid bounds (value keys)
    unsigned long long lo[3], hi[3];           // node bounds (pair keys)
    Bin bins[12];
};
struct TNode { uint32_t begin, end, left, kind, axis, size, pre, pad; float lo[3], hi[3]; }; // right child = left + 1
struct Counters { uint32_t n_tree, n_next, n_small, empty; }; // empty: a split left a child of no elements

__device__ void open_init(Open& o, uint32_t begin, uint32_t end, uint32_t tn) {
    o.begin = begin; o.end = end; o.tn = tn; o.kind = K_SAH;
    for (int i = 0; i < 3; ++i) { o.clo[i] = 0xffffffffu; o.chi[i] = 0u; o.lo[i] = ~0ull; o.hi[i] = 0ull; }
    for (int k = 0; k < 12; ++k) {
        for (int i = 0; i < 3; ++i) { o.bins[k].lo[i] = ~0ull; o.bins[k].hi[i] = 0ull; }
        o.bins[k].cnt = 0;
    }
}

// centroids (bbox.rs:58-61 via linalg::lerp) and the identity order
__global__ void k_bvh_init(const float* __restrict__ boxes, uint32_t n, float* __restrict__ cen, uint32_t* __restrict__ idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int c = 0; c < 3; ++c)
        cen[(size_t)c * n + i] = __fadd_rn(__fmul_rn(boxes[6 * (size_t)i + c], 1.0f - 0.5f), __fmul_rn(boxes[6 * (size_t)i + 3 + c], 0.5f));
    idx[i] = i;
}

__global__ void k_bvh_root(uint32_t n, uint32_t small, TNode* tn, Open* op, uint32_t* small_list, Counters* cnt) {
    TNode& t = tn[0];
    t.begin = 0; t.end = n; t.pre = 0;
    if (n > small) { t.kind = T_INTERIOR; open_init(op[0], 0, n, 0); *cnt = Counters{1, 1, 0, 0}; }
    else { t.kind = T_SMALL; small_list[0] = 0; *cnt = Counters{1, 0, 1, 0}; }
}

__global__ void k_bvh_seg(const Open* __restrict__ op, uint32_t* __restrict__ seg) {
    const Open& o = op[blockIdx.x];
    for (uint32_t p = o.begin + threadIdx.x; p < o.end; p += blockDim.x) seg[p] = blockIdx.x;
}

// node bounds and centroid bounds of every open node
__global__ void k_bvh_bounds(uint32_t n, const uint32_t* __restrict__ seg, const uint32_t* __restrict__ idx, const float* __restrict__ boxes,
                             const float* __restrict__ cen, Open* op) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t s = p < n ? seg[p] : NONE;
    const unsigned act = __ballot_sync(0xffffffffu, s != NONE);
    if (s == NONE) return;
    const unsigned grp = __match_any_sync(act, s);
    const bool lead = (int)(threadIdx.x & 31) == __ffs(grp) - 1;
    const uint32_t g = idx[p];
    Open& o = op[s];
    for (int c = 0; c < 3; ++c) {
        const float x = cen[(size_t)c * n + g];
        const uint32_t klo = __reduce_min_sync(grp, isnan(x) ? 0xffffffffu : okey(x));
        const uint32_t khi = __reduce_max_sync(grp, isnan(x) ? 0u : okey(x));
        if (lead) { atomicMin(&o.clo[c], klo); atomicMax(&o.chi[c], khi); }
        red_min(grp, lead, boxes[6 * (size_t)g + c], p, &o.lo[c]);
        red_max(grp, lead, boxes[6 * (size_t)g + 3 + c], p, &o.hi[c]);
    }
}

// split axis (bvh.rs:147-166): max_extent of the centroid bounds; coincident centroids make a leaf or split in place
__global__ void k_bvh_axis(Open* op, uint32_t n_open, uint32_t max_geom) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_open) return;
    Open& o = op[j];
    float lo[3], hi[3];
    for (int c = 0; c < 3; ++c) {
        lo[c] = o.clo[c] == 0xffffffffu ? INFINITY : okey_inv(o.clo[c]);
        hi[c] = o.chi[c] == 0u ? -INFINITY : okey_inv(o.chi[c]);
    }
    const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
    const uint32_t axis = (dx > dy && dx > dz) ? 0 : (dy > dz ? 1 : 2);
    const uint32_t n = o.end - o.begin;
    o.axis = axis; o.cmin = lo[axis]; o.cmax = hi[axis];
    if (fabsf(hi[axis] - lo[axis]) < trbh::kEps) { o.kind = n < max_geom ? K_LEAF : K_KEEP; o.mid = o.begin + n / 2; }
}

// the 12 SAH buckets of every undecided node
__global__ void k_bvh_bins(uint32_t n, const uint32_t* __restrict__ seg, const uint32_t* __restrict__ idx, const float* __restrict__ boxes,
                           const float* __restrict__ cen, Open* op) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t s = p < n ? seg[p] : NONE;
    if (s != NONE && op[s].kind != K_SAH) s = NONE;
    const unsigned act = __ballot_sync(0xffffffffu, s != NONE);
    if (s == NONE) return;
    Open& o = op[s];
    const uint32_t g = idx[p];
    const uint32_t k = bucket(cen[(size_t)o.axis * n + g], o.cmin, o.cmax);
    const unsigned grp = __match_any_sync(act, ((unsigned long long)s << 4) | k);
    const bool lead = (int)(threadIdx.x & 31) == __ffs(grp) - 1;
    Bin& b = o.bins[k];
    if (lead) atomicAdd(&b.cnt, (uint32_t)__popc(grp));
    for (int c = 0; c < 3; ++c) {
        red_min(grp, lead, boxes[6 * (size_t)g + c], p, &b.lo[c]);
        red_max(grp, lead, boxes[6 * (size_t)g + 3 + c], p, &b.hi[c]);
    }
}

// SAH costs of splits after buckets 0..10 (bvh.rs:180-215), folded as the host folds them
__global__ void k_bvh_split(Open* op, uint32_t n_open, uint32_t max_geom, const uint32_t* __restrict__ idx, const float* __restrict__ boxes) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_open || op[j].kind != K_SAH) return;
    Open& o = op[j];
    trbh::Box3 bounds, bb[12];
    uint32_t count[12];
    for (int c = 0; c < 3; ++c) { bounds.lo[c] = dec_lo(o.lo[c], boxes, idx, c); bounds.hi[c] = dec_hi(o.hi[c], boxes, idx, c); }
    for (int k = 0; k < 12; ++k) {
        count[k] = o.bins[k].cnt;
        for (int c = 0; c < 3; ++c) { bb[k].lo[c] = dec_lo(o.bins[k].lo[c], boxes, idx, c); bb[k].hi[c] = dec_hi(o.bins[k].hi[c], boxes, idx, c); }
    }
    float best_cost = INFINITY;
    int best = 0;
    const float total_area = trbh::box_area_hd(bounds);
    for (int sp = 0; sp < 11; ++sp) {
        trbh::Box3 lb = trbh::box_empty_hd(), rb = trbh::box_empty_hd();
        uint32_t lc = 0, rc = 0;
        for (int k = 0; k <= sp; ++k) { hgrow(lb, bb[k]); lc += count[k]; }
        for (int k = sp + 1; k < 12; ++k) { hgrow(rb, bb[k]); rc += count[k]; }
        const float cost = 0.125f + ((float)lc * trbh::box_area_hd(lb) + (float)rc * trbh::box_area_hd(rb)) / total_area;
        if (cost < best_cost) { best_cost = cost; best = sp; }
    }
    const uint32_t n = o.end - o.begin;
    if (n > max_geom || best_cost < (float)n) {
        uint32_t lc = 0;
        for (int k = 0; k <= best; ++k) lc += count[k];
        o.kind = K_PART; o.best = (uint32_t)best; o.mid = o.begin + lc;
    } else o.kind = K_LEAF;
}

// partition flags: 1 for a false in [b, b+P), 1 << 32 for a true in [b+P, e); f[n] = 0 ends the scan
__global__ void k_bvh_flags(uint32_t n, const uint32_t* __restrict__ seg, const uint32_t* __restrict__ idx, const float* __restrict__ cen,
                            const Open* __restrict__ op, unsigned long long* __restrict__ f) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p > n) return;
    unsigned long long v = 0;
    const uint32_t s = p < n ? seg[p] : NONE;
    if (s != NONE && op[s].kind == K_PART) {
        const Open& o = op[s];
        const bool pred = bucket(cen[(size_t)o.axis * n + idx[p]], o.cmin, o.cmax) <= o.best;
        if (p < o.mid) v = pred ? 0ull : 1ull;
        else v = pred ? (1ull << 32) : 0ull;
    }
    f[p] = v;
}

// after the exclusive scan of the flags: L[k] -> tmp[b + k], R's ascending rank r -> tmp[b + P + r]
__global__ void k_bvh_ranks(uint32_t n, const uint32_t* __restrict__ seg, const Open* __restrict__ op, const unsigned long long* __restrict__ f,
                            uint32_t* __restrict__ tmp) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t s = p < n ? seg[p] : NONE;
    if (s == NONE || op[s].kind != K_PART) return;
    const Open& o = op[s];
    const unsigned long long d = f[p + 1] - f[p];
    if (p < o.mid) { if ((uint32_t)d) tmp[o.begin + (uint32_t)(f[p] - f[o.begin])] = p; }
    else if (d >> 32) tmp[o.mid + (uint32_t)((f[p] - f[o.mid]) >> 32)] = p;
}

// swap L[k] with R[k] (R descending = ascending rank m - 1 - k)
__global__ void k_bvh_swap(uint32_t n, const uint32_t* __restrict__ seg, const Open* __restrict__ op, const unsigned long long* __restrict__ f,
                           const uint32_t* __restrict__ tmp, uint32_t* __restrict__ idx) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t s = p < n ? seg[p] : NONE;
    if (s == NONE || op[s].kind != K_PART) return;
    const Open& o = op[s];
    if (p >= o.mid) return;
    const uint32_t m = (uint32_t)(f[o.mid] - f[o.begin]), k = p - o.begin;
    if (k >= m) return;
    const uint32_t pl = tmp[o.begin + k], pr = tmp[o.mid + (m - 1 - k)];
    const uint32_t t = idx[pl]; idx[pl] = idx[pr]; idx[pr] = t;
}

// leaves take their bounds; interior nodes get two children, each opened at the next level or left to a serial subtree
__global__ void k_bvh_children(const Open* __restrict__ op, uint32_t n_open, uint32_t small, TNode* tn, Open* next, uint32_t* small_list, Counters* cnt,
                               const uint32_t* __restrict__ idx, const float* __restrict__ boxes) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_open) return;
    const Open& o = op[j];
    TNode& t = tn[o.tn];
    if (o.kind == K_LEAF) {
        t.kind = T_LEAF;
        for (int c = 0; c < 3; ++c) { t.lo[c] = dec_lo(o.lo[c], boxes, idx, c); t.hi[c] = dec_hi(o.hi[c], boxes, idx, c); }
        return;
    }
    if (o.mid == o.begin || o.mid == o.end) { t.kind = T_LEAF; atomicExch(&cnt->empty, 1u); return; }
    t.kind = T_INTERIOR; t.axis = o.axis;
    const uint32_t l = atomicAdd(&cnt->n_tree, 2u);
    t.left = l;
    const uint32_t b[3] = {o.begin, o.mid, o.end};
    for (int i = 0; i < 2; ++i) {
        TNode& ch = tn[l + i];
        ch.begin = b[i]; ch.end = b[i + 1];
        if (b[i + 1] - b[i] > small) { ch.kind = T_INTERIOR; open_init(next[atomicAdd(&cnt->n_next, 1u)], b[i], b[i + 1], l + i); }
        else { ch.kind = T_SMALL; small_list[atomicAdd(&cnt->n_small, 1u)] = l + i; }
    }
}

// One thread builds the subtree of idx[b0, e0) with bvh_build_arrays' algorithm (folds through hmin / hmax). Its nodes
// go to out[0, count) in local preorder (an interior `a` is local, a leaf `a` is the global slot); `task` holds 3 * (e0 - b0) words.
// Returns NONE, having stopped, where a split leaves a child of no elements.
__device__ uint32_t serial_build(uint32_t b0, uint32_t e0, uint32_t max_geom, const float* __restrict__ boxes, const float* __restrict__ cen,
                                 uint32_t nall, uint32_t* idx, uint32_t* task, trb_bvh_node* out) {
    uint32_t n_nodes = 0, n_task = 0;
    uint32_t begin = b0, end = e0, parent = NONE;
    for (;;) {
        const uint32_t n = end - begin;
        if (n == 0) return NONE;
        const uint32_t me = n_nodes++;
        if (parent != NONE) out[parent].a = me;
        trbh::Box3 bounds = trbh::box_empty_hd();
        for (uint32_t i = begin; i < end; ++i) hgrow(bounds, load_box(boxes, idx[i]));
        bool is_leaf = false;
        int axis = 0;
        uint32_t mid = begin + n / 2;
        if (n == 1) is_leaf = true;
        else {
            trbh::Box3 cb = trbh::box_empty_hd();
            for (uint32_t i = begin; i < end; ++i) {
                const uint32_t g = idx[i];
                for (int c = 0; c < 3; ++c) { const float x = cen[(size_t)c * nall + g]; cb.lo[c] = hmin(cb.lo[c], x); cb.hi[c] = hmax(cb.hi[c], x); }
            }
            const float dx = cb.hi[0] - cb.lo[0], dy = cb.hi[1] - cb.lo[1], dz = cb.hi[2] - cb.lo[2];
            axis = (dx > dy && dx > dz) ? 0 : (dy > dz ? 1 : 2);
            const float* ca = cen + (size_t)axis * nall;
            if (fabsf(cb.hi[axis] - cb.lo[axis]) < trbh::kEps) {
                if (n < max_geom) is_leaf = true;
            } else if (n < 5) {
                for (uint32_t i = begin + 1; i < end; ++i) {
                    const uint32_t g = idx[i];
                    const float key = ca[g];
                    uint32_t j = i;
                    while (j > begin && ca[idx[j - 1]] > key) { idx[j] = idx[j - 1]; --j; }
                    idx[j] = g;
                }
            } else {
                const float cmin = cb.lo[axis], cmax = cb.hi[axis];
                uint32_t count[12];
                trbh::Box3 bb[12];
                for (int k = 0; k < 12; ++k) { count[k] = 0; bb[k] = trbh::box_empty_hd(); }
                for (uint32_t i = begin; i < end; ++i) {
                    const uint32_t k = bucket(ca[idx[i]], cmin, cmax);
                    count[k]++;
                    hgrow(bb[k], load_box(boxes, idx[i]));
                }
                float best_cost = INFINITY;
                int best = 0;
                const float total_area = trbh::box_area_hd(bounds);
                for (int sp = 0; sp < 11; ++sp) {
                    trbh::Box3 lb = trbh::box_empty_hd(), rb = trbh::box_empty_hd();
                    uint32_t lc = 0, rc = 0;
                    for (int k = 0; k <= sp; ++k) { hgrow(lb, bb[k]); lc += count[k]; }
                    for (int k = sp + 1; k < 12; ++k) { hgrow(rb, bb[k]); rc += count[k]; }
                    const float cost = 0.125f + ((float)lc * trbh::box_area_hd(lb) + (float)rc * trbh::box_area_hd(rb)) / total_area;
                    if (cost < best_cost) { best_cost = cost; best = sp; }
                }
                if (n > max_geom || best_cost < (float)n) {
                    uint32_t lo = begin, hi = end, split = begin;
                    for (;;) {
                        uint32_t f = NONE, bk = NONE;
                        while (lo < hi) { const uint32_t p = lo++; if (bucket(ca[idx[p]], cmin, cmax) > (uint32_t)best) { f = p; break; } split++; }
                        while (lo < hi) { const uint32_t p = --hi; if (bucket(ca[idx[p]], cmin, cmax) <= (uint32_t)best) { bk = p; break; } }
                        if (f == NONE || bk == NONE) break;
                        const uint32_t tmp = idx[f]; idx[f] = idx[bk]; idx[bk] = tmp;
                        split++;
                    }
                    mid = split;
                } else is_leaf = true;
            }
        }
        trb_bvh_node& nd = out[me];
        for (int i = 0; i < 3; ++i) { nd.bmin[i] = bounds.lo[i]; nd.bmax[i] = bounds.hi[i]; }
        if (is_leaf) {
            nd.a = begin; nd.b = TRB_BVH_LEAF | n;
            if (n_task == 0) break;
            n_task--;
            begin = task[3 * n_task]; end = task[3 * n_task + 1]; parent = task[3 * n_task + 2];
        } else {
            nd.a = 0; nd.b = (uint32_t)axis;
            task[3 * n_task] = mid; task[3 * n_task + 1] = end; task[3 * n_task + 2] = me; n_task++;
            end = mid; parent = NONE;
        }
    }
    for (uint32_t i = n_nodes; i-- > 0;) {
        trb_bvh_node& nd = out[i];
        if (nd.b & TRB_BVH_LEAF) continue;
        const trb_bvh_node& l = out[i + 1];
        const trb_bvh_node& r = out[nd.a];
        for (int k = 0; k < 3; ++k) { nd.bmin[k] = hmin(l.bmin[k], r.bmin[k]); nd.bmax[k] = hmax(l.bmax[k], r.bmax[k]); }
    }
    return n_nodes;
}

__global__ void k_bvh_small(const uint32_t* __restrict__ small_list, uint32_t n_small, TNode* tn, Counters* cnt, uint32_t max_geom, const float* __restrict__ boxes,
                            const float* __restrict__ cen, uint32_t n, uint32_t* idx, uint32_t* task, trb_bvh_node* snodes) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_small) return;
    TNode& t = tn[small_list[j]];
    t.size = serial_build(t.begin, t.end, max_geom, boxes, cen, n, idx, task + 3 * (size_t)t.begin, snodes + 2 * (size_t)t.begin);
    if (t.size == NONE) { t.size = 0; atomicExch(&cnt->empty, 1u); }
}

// subtree node counts of one level of the top tree (children done first)
__global__ void k_bvh_size(TNode* tn, uint32_t first, uint32_t last) {
    const uint32_t i = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= last) return;
    TNode& t = tn[i];
    if (t.kind == T_LEAF) t.size = 1;
    else if (t.kind == T_INTERIOR) t.size = 1 + tn[t.left].size + tn[t.left + 1].size;
}
// preorder indices of the children of one level (bvh.rs:248-267: first child next, second after the first's subtree)
__global__ void k_bvh_pre(TNode* tn, uint32_t first, uint32_t last) {
    const uint32_t i = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= last) return;
    const TNode& t = tn[i];
    if (t.kind != T_INTERIOR) return;
    tn[t.left].pre = t.pre + 1;
    tn[t.left + 1].pre = t.pre + 1 + tn[t.left].size;
}
__global__ void k_bvh_emit(const TNode* __restrict__ tn, uint32_t n_tree, trb_bvh_node* nodes) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_tree) return;
    const TNode& t = tn[i];
    trb_bvh_node& nd = nodes[t.pre];
    if (t.kind == T_LEAF) {
        for (int c = 0; c < 3; ++c) { nd.bmin[c] = t.lo[c]; nd.bmax[c] = t.hi[c]; }
        nd.a = t.begin; nd.b = TRB_BVH_LEAF | (t.end - t.begin);
    } else if (t.kind == T_INTERIOR) { nd.a = tn[t.left + 1].pre; nd.b = t.axis; }
}
// one CTA per serial subtree: move its nodes to their preorder place
__global__ void k_bvh_copy(const uint32_t* __restrict__ small_list, const TNode* __restrict__ tn, const trb_bvh_node* __restrict__ snodes,
                           trb_bvh_node* nodes) {
    const TNode& t = tn[small_list[blockIdx.x]];
    for (uint32_t i = threadIdx.x; i < t.size; i += blockDim.x) {
        trb_bvh_node nd = snodes[2 * (size_t)t.begin + i];
        if (!(nd.b & TRB_BVH_LEAF)) nd.a += t.pre;
        nodes[t.pre + i] = nd;
    }
}
// BuildNode::interior (bvh.rs:358-362): the union of the children, left first; one level of the top tree, deepest first
__global__ void k_bvh_ibounds(const TNode* __restrict__ tn, uint32_t first, uint32_t last, trb_bvh_node* nodes) {
    const uint32_t i = first + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= last || tn[i].kind != T_INTERIOR) return;
    trb_bvh_node& nd = nodes[tn[i].pre];
    const trb_bvh_node& l = nodes[tn[i].pre + 1];
    const trb_bvh_node& r = nodes[nd.a];
    for (int k = 0; k < 3; ++k) { nd.bmin[k] = hmin(l.bmin[k], r.bmin[k]); nd.bmax[k] = hmax(l.bmax[k], r.bmax[k]); }
}

// ---- mesh helpers of trb_scene_create
// Triangle::bounds (mesh.rs:128-134): lo = hi = pa, grown with pb and pc
__global__ void k_tri_boxes(const float* __restrict__ pos, const uint32_t* __restrict__ tri, uint32_t n_tris, float* __restrict__ boxes) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tris) return;
    float lo[3], hi[3];
    for (int v = 0; v < 3; ++v) {
        const float* p = pos + 3 * (size_t)tri[3 * (size_t)t + v];
        for (int c = 0; c < 3; ++c) {
            if (v == 0) lo[c] = hi[c] = p[c];
            else { lo[c] = hmin(lo[c], p[c]); hi[c] = hmax(hi[c], p[c]); }
        }
    }
    for (int c = 0; c < 3; ++c) { boxes[6 * (size_t)t + c] = lo[c]; boxes[6 * (size_t)t + 3 + c] = hi[c]; }
}
// the leaf-ordered triangle records (trb_device.h DTri); the leaf-end marks are added by k_tri_leaf_marks
__global__ void k_tri_pack(const float* __restrict__ pos, const uint32_t* __restrict__ tri, const uint32_t* __restrict__ order, uint32_t n_tris,
                           DTri* __restrict__ out) {
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= n_tris) return;
    const uint32_t t = order[slot];
    const float* pa = pos + 3 * (size_t)tri[3 * (size_t)t];
    const float* pb = pos + 3 * (size_t)tri[3 * (size_t)t + 1];
    const float* pc = pos + 3 * (size_t)tri[3 * (size_t)t + 2];
    DTri r;
    r.v0 = make_float4(pa[0], pa[1], pa[2], __uint_as_float(t));
    r.e0 = make_float4(pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2], 0.f);
    r.e1 = make_float4(pc[0] - pa[0], pc[1] - pa[1], pc[2] - pa[2], 0.f);
    r.pad = make_float4(0.f, 0.f, 0.f, 0.f);
    out[slot] = r;
}
__global__ void k_tri_leaf_marks(const trb_bvh_node* __restrict__ nodes, uint32_t n_nodes, DTri* tris) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    const trb_bvh_node nd = nodes[i];
    const uint32_t cnt = nd.b & ~TRB_BVH_LEAF;
    if ((nd.b & TRB_BVH_LEAF) && cnt) tris[(size_t)nd.a + cnt - 1].e0.w = __uint_as_float(TRI_LEAF_END);
}
// *bad = 1 where some of the n indices is >= n_verts: trb_scene_create's "mesh index out of range" for indices that are already on the
// device (trb_scene_replace_meshes_device), read once where they are. idx is a cudaMalloc'd buffer, so 16-byte aligned: vector loads
// over the body, a scalar tail, and one atomic per warp that found an index out of range. Grid-stride; blockDim a multiple of 32.
__global__ void k_mesh_index_check(const uint32_t* __restrict__ idx, size_t n, uint32_t n_verts, uint32_t* bad) {
    const size_t n4 = n / 4, stride = (size_t)gridDim.x * blockDim.x, t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const uint4* __restrict__ v = reinterpret_cast<const uint4*>(idx);
    bool out = false;
    for (size_t i = t; i < n4; i += stride) {
        const uint4 q = v[i];
        out |= (q.x >= n_verts) | (q.y >= n_verts) | (q.z >= n_verts) | (q.w >= n_verts);
    }
    for (size_t i = 4 * n4 + t; i < n; i += stride) out |= idx[i] >= n_verts;
    if (__any_sync(0xffffffffu, out) && (threadIdx.x & 31) == 0) atomicOr(bad, 1u);
}

// ---- mesh helpers of trb_scene_update_mesh: the DPair records (trb_device.h) of a preorder tree still on the device
// rec[i] = 1 for an interior node, rec[n] = 0; an exclusive scan then gives each interior node its record index and rec[n] the count
__global__ void k_pair_flags(const trb_bvh_node* __restrict__ nodes, uint32_t n, uint32_t* __restrict__ rec) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    rec[i] = i < n && !(nodes[i].b & TRB_BVH_LEAF) ? 1u : 0u;
}
// One record per interior node in the layout of trb_api.cu's pack_pairs, leaves referenced in the narrow or the wide form.
// *narrow_bad is set where a leaf does not fit the narrow reference, whichever form was asked for, so the caller learns which
// form the tree needs. Every leaf fits the wide reference: a mesh holds at most 2^30 triangles and a leaf at least one.
__device__ __forceinline__ uint32_t pair_ref(const trb_bvh_node& nd, uint32_t rec, bool wide) {
    if (!(nd.b & TRB_BVH_LEAF)) return REF_INTERIOR | rec;
    const uint32_t cnt = nd.b & ~TRB_BVH_LEAF, first = nd.a;
    return wide ? (REF_LEAF | (first & ~REF_TAG)) : (REF_LEAF | (cnt << 25) | first);
}
__global__ void k_pair_pack(const trb_bvh_node* __restrict__ nodes, uint32_t n, const uint32_t* __restrict__ rec, bool wide,
                            DPair* __restrict__ out, uint32_t* narrow_bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const trb_bvh_node nd = nodes[i];
    if (nd.b & TRB_BVH_LEAF) {
        if ((nd.b & ~TRB_BVH_LEAF) > 31 || nd.a >= (1u << 25)) *narrow_bad = 1u;
        return;
    }
    const trb_bvh_node l = nodes[i + 1], r = nodes[nd.a];
    DPair p;
    p.l_lo = make_float4(l.bmin[0], l.bmin[1], l.bmin[2], __uint_as_float(pair_ref(l, rec[i + 1], wide)));
    p.l_hi = make_float4(l.bmax[0], l.bmax[1], l.bmax[2], __uint_as_float(pair_ref(r, rec[nd.a], wide)));
    p.r_lo = make_float4(r.bmin[0], r.bmin[1], r.bmin[2], __uint_as_float(nd.b));
    p.r_hi = make_float4(r.bmax[0], r.bmax[1], r.bmax[2], 0.f);
    out[rec[i]] = p;
}

// ---- mesh helpers of trb_scene_refit_mesh: new positions through the kept tree (DESIGN.md §4 "Mesh refits")
// The leaf-ordered triangle records from new positions with k_tri_pack's arithmetic. Each slot keeps its triangle index and its
// leaf-end mark, so the tree's ordered_geom is never needed on the device.
__global__ void k_refit_tris(const float* __restrict__ pos, const uint32_t* __restrict__ tri, uint32_t n_tris, DTri* tris) {
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= n_tris) return;
    const uint32_t t = __float_as_uint(tris[slot].v0.w);
    const float mark = tris[slot].e0.w;
    const float* pa = pos + 3 * (size_t)tri[3 * (size_t)t];
    const float* pb = pos + 3 * (size_t)tri[3 * (size_t)t + 1];
    const float* pc = pos + 3 * (size_t)tri[3 * (size_t)t + 2];
    DTri r;
    r.v0 = make_float4(pa[0], pa[1], pa[2], __uint_as_float(t));
    r.e0 = make_float4(pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2], mark);
    r.e1 = make_float4(pc[0] - pa[0], pc[1] - pa[1], pc[2] - pa[2], 0.f);
    r.pad = make_float4(0.f, 0.f, 0.f, 0.f);
    tris[slot] = r;
}
// The parent of every record as (parent record << 1 | side), side 0 for the first child (l), 1 for the second (r); the root record 0
// has none. Records number the interior nodes in preorder (pack_pairs), so n_rec < 2^30 and the link fits 31 bits.
__global__ void k_refit_parents(const DPair* __restrict__ pairs, uint32_t n_rec, uint32_t* __restrict__ parent) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rec) return;
    if (r == 0) parent[0] = NONE;
    const uint32_t lref = __float_as_uint(pairs[r].l_lo.w), rref = __float_as_uint(pairs[r].l_hi.w);
    if ((lref & REF_TAG) == REF_INTERIOR) parent[lref & ~REF_TAG] = r << 1;
    if ((rref & REF_TAG) == REF_INTERIOR) parent[rref & ~REF_TAG] = r << 1 | 1u;
}
// The fold of bvh.rs:143 over one leaf: BBox::new() grown with Triangle::bounds (mesh.rs:128-134) of each of its triangles, in slot
// order, from the mesh's positions. A narrow reference carries the count, a wide one runs to the slot marked TRI_LEAF_END.
__device__ __forceinline__ trbh::Box3 refit_leaf_box(uint32_t ref, bool wide, const DTri* __restrict__ tris, const uint32_t* __restrict__ tri,
                                                     const float* __restrict__ pos) {
    trbh::Box3 b;
    for (int c = 0; c < 3; ++c) { b.lo[c] = INFINITY; b.hi[c] = -INFINITY; }
    const uint32_t first = wide ? (ref & ~REF_TAG) : (ref & ((1u << 25) - 1u)), cnt = wide ? NONE : (ref >> 25) & 31u;
    for (uint32_t j = 0; j < cnt; ++j) {
        const uint32_t slot = first + j, t = __float_as_uint(tris[slot].v0.w);
        trbh::Box3 tb;
        for (int v = 0; v < 3; ++v) {
            const float* p = pos + 3 * (size_t)tri[3 * (size_t)t + v];
            for (int c = 0; c < 3; ++c) {
                if (v == 0) tb.lo[c] = tb.hi[c] = p[c];
                else { tb.lo[c] = hmin(tb.lo[c], p[c]); tb.hi[c] = hmax(tb.hi[c], p[c]); }
            }
        }
        hgrow(b, tb);
        if (wide && __float_as_uint(tris[slot].e0.w) == TRI_LEAF_END) break;
    }
    return b;
}
__device__ __forceinline__ void refit_store(DPair* pairs, uint32_t rec, uint32_t side, const trbh::Box3& b) {
    float* f = reinterpret_cast<float*>(pairs + rec) + 8 * side; // side 0: l_lo / l_hi, side 1: r_lo / r_hi; the w words stay
    for (int c = 0; c < 3; ++c) { f[c] = b.lo[c]; f[4 + c] = b.hi[c]; }
}
// Node boxes, bottom-up, in place in the DPair records (Karras 2012). The thread of record r writes the boxes of r's leaf children and
// then arrives at r once per box written; the box of an interior child is written into r by the thread that completed that child,
// which then arrives at r once. The arrival that brings r's counter to 2 owns r: it unions r's two boxes (first child first) into the
// box of r's node, writes it into the parent's slot, and arrives there. Every box is therefore written once, by one thread, from
// operands that are final when it reads them, and the result does not depend on the schedule.
// Ordering: each box is stored, then __threadfence() (release), then the arrival's atomicAdd. The owning arrival issues
// __threadfence() (acquire) before it reads the record, and reads it with ld.global.cg (from L2, never a stale L1 line).
// The root record's box goes into the mesh header (root_lo / root_hi xyz; the w words stay). A tree that is one leaf has no record:
// thread 0 folds that leaf into the header. `count` holds n_rec zeros.
__global__ void k_refit_nodes(DPair* pairs, uint32_t n_rec, const uint32_t* __restrict__ parent, uint32_t* count, bool wide,
                              const DTri* __restrict__ tris, const uint32_t* __restrict__ tri, const float* __restrict__ pos, DBvh* hdr) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    auto store_root = [&](const trbh::Box3& b) {
        float* lo = reinterpret_cast<float*>(&hdr->root_lo);
        float* hi = reinterpret_cast<float*>(&hdr->root_hi);
        for (int c = 0; c < 3; ++c) { lo[c] = b.lo[c]; hi[c] = b.hi[c]; }
    };
    if (n_rec == 0) {
        if (r == 0) store_root(refit_leaf_box(__float_as_uint(hdr->root_lo.w), wide, tris, tri, pos));
        return;
    }
    if (r >= n_rec) return;
    const uint32_t lref = __float_as_uint(pairs[r].l_lo.w), rref = __float_as_uint(pairs[r].l_hi.w);
    uint32_t arrivals = 0;
    if ((lref & REF_TAG) == REF_LEAF) { refit_store(pairs, r, 0, refit_leaf_box(lref, wide, tris, tri, pos)); ++arrivals; }
    if ((rref & REF_TAG) == REF_LEAF) { refit_store(pairs, r, 1, refit_leaf_box(rref, wide, tris, tri, pos)); ++arrivals; }
    if (arrivals == 0) return;
    __threadfence();
    uint32_t node = r;
    if (atomicAdd(&count[node], arrivals) + arrivals != 2u) return;
    for (;;) {
        __threadfence();
        const float4 llo = __ldcg(&pairs[node].l_lo), lhi = __ldcg(&pairs[node].l_hi), rlo = __ldcg(&pairs[node].r_lo), rhi = __ldcg(&pairs[node].r_hi);
        trbh::Box3 b;
        b.lo[0] = hmin(llo.x, rlo.x); b.lo[1] = hmin(llo.y, rlo.y); b.lo[2] = hmin(llo.z, rlo.z);
        b.hi[0] = hmax(lhi.x, rhi.x); b.hi[1] = hmax(lhi.y, rhi.y); b.hi[2] = hmax(lhi.z, rhi.z);
        if (node == 0) { store_root(b); return; }
        const uint32_t p = parent[node];
        refit_store(pairs, p >> 1, p & 1u, b);
        __threadfence();
        node = p >> 1;
        if (atomicAdd(&count[node], 1u) != 1u) return;
    }
}

// ---- instance-tree helpers of trb_scene_update_frame (the level builder's counterpart of k_tlas_build's head and tail)
// *bad = 1 where some bound fails trbh::bvh_bound_buildable
__global__ void k_bounds_check(const float* __restrict__ bounds, size_t n_floats, uint32_t* bad) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < n_floats && !trbh::bvh_bound_buildable(bounds[i])) *bad = 1u;
}
// the traversal header and the frame's counts {n_nodes, n_order, pack ok, 0: the build accepted the bounds}, after k_pair_pack in the narrow form
__global__ void k_tlas_header(const trb_bvh_node* __restrict__ nodes, const uint32_t* __restrict__ rec, uint32_t n_nodes, uint32_t n_order,
                              const uint32_t* __restrict__ narrow_bad, DPair* pairs, DBvh* hdr, uint32_t* counts) {
    const trb_bvh_node root = nodes[0];
    hdr->pairs = pairs;
    hdr->root_lo = make_float4(root.bmin[0], root.bmin[1], root.bmin[2], __uint_as_float(pair_ref(root, rec[0], false)));
    hdr->root_hi = make_float4(root.bmax[0], root.bmax[1], root.bmax[2], 0.f);
    counts[0] = n_nodes; counts[1] = n_order; counts[2] = *narrow_bad ? 0u : 1u; counts[3] = 0u;
}

// ---- host driver
inline size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }
struct Scratch {
    float* cen; uint32_t* seg; unsigned long long* f; uint32_t* tmp; uint32_t* small_list; trb_bvh_node* snodes;
    Open* open[2]; Counters* cnt; void* cub; size_t cub_bytes; size_t bytes;
};
inline uint32_t open_cap(uint32_t n, uint32_t small = SMALL) { return n / (small + 1) + 1; } // open nodes are disjoint and hold more than `small` elements each
// Carves the scratch of an n-box build from `base` (base = nullptr: only sizes it). f and tmp are adjacent: after the level
// loop their 12n + 8 bytes hold the serial subtrees' task stacks (3n words).
inline Scratch scratch_layout(uint32_t n, char* base, uint32_t small = SMALL) {
    Scratch s{};
    size_t off = 0;
    auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align_up(bytes); return p; };
    s.cen = (float*)take(3 * (size_t)n * 4);
    s.seg = (uint32_t*)take((size_t)n * 4);
    s.f = (unsigned long long*)(base ? base + off : nullptr);
    off += ((size_t)n + 1) * 8; // tmp directly after f
    s.tmp = (uint32_t*)take((size_t)n * 4);
    s.small_list = (uint32_t*)take((size_t)n * 4);
    s.snodes = (trb_bvh_node*)take(2 * (size_t)n * sizeof(trb_bvh_node));
    s.open[0] = (Open*)take(open_cap(n, small) * sizeof(Open));
    s.open[1] = (Open*)take(open_cap(n, small) * sizeof(Open));
    s.cnt = (Counters*)take(sizeof(Counters));
    cub::DeviceScan::ExclusiveSum(nullptr, s.cub_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n + 1);
    s.cub = take(s.cub_bytes);
    s.bytes = off;
    return s;
}
// device bytes an n-box build allocates, besides its nodes and order outputs (the top tree is small and grows on demand)
inline size_t build_scratch_bytes(uint32_t n, uint32_t small = SMALL) {
    return scratch_layout(n, nullptr, small).bytes + (size_t)(4 * open_cap(n, small) + 64) * sizeof(TNode);
}
// A build that must not allocate runs in memory its caller keeps: `base` of scratch_layout(n, nullptr, small).bytes and a top tree of
// top_cap(n) nodes, which no build outgrows (the top tree is a binary tree whose leaves hold disjoint, non-empty ranges of the n boxes).
inline size_t top_cap(uint32_t n) { return 2 * (size_t)n; }
struct OwnedScratch { char* base; TNode* tn; };
// What a caller timing the build's phases gets back: events recorded after the level loop and after the serial subtrees (recorded
// only when non-null), and the number of levels.
struct BuildTrace { cudaEvent_t after_levels = nullptr, after_small = nullptr; uint32_t levels = 0; };

#define BVHB_TRY(call) do { const cudaError_t e_ = (call); if (e_ != cudaSuccess) { err = e_; goto done; } } while (0)

// Builds the BVH of the n boxes at d_boxes (6 floats each) on `st`: nodes to d_nodes (room for 2n - 1),
// their count to the device word d_n_nodes (and to *h_n_nodes when given), ordered_geom to d_order. Nodes of more than `small` (>= 4)
// boxes are split level by level, the rest by one thread each. Synchronises `st` once per level and once at the end. Scratch is
// `own` when given, else allocated on `st` for this call and freed. *empty is set where the reference's build would split a node into
// a child of no elements (a node of more than max_geom boxes whose centroids all fall in one bucket, which infinite coordinates cause):
// the reference and the host builder never finish such a build, so the output is then not a tree and the caller reports an error.
// With `refuse`, *empty is also set, and no serial subtree is started, where more than max_geom boxes hold a bound that fails
// trbh::bvh_bound_buildable: the serial subtrees, like bvh_build_arrays, never end on a split that keeps every element on one side.
inline cudaError_t build_device(const float* d_boxes, uint32_t n, uint32_t max_geom, uint32_t* d_n_nodes, trb_bvh_node* d_nodes,
                                uint32_t* d_order, cudaStream_t st, unsigned long long* launches, bool* empty, uint32_t small = SMALL,
                                const OwnedScratch* own = nullptr, uint32_t* h_n_nodes = nullptr, BuildTrace* trace = nullptr, bool refuse = false) {
    cudaError_t err = cudaSuccess;
    char* base = own ? own->base : nullptr;
    TNode* tn = own ? own->tn : nullptr;
    Scratch s = scratch_layout(n, nullptr, small);
    size_t cap = own ? top_cap(n) : 4 * (size_t)open_cap(n, small) + 64;
    uint32_t n_tree = 1, n_open, n_small, h_nodes = 0;
    std::vector<uint32_t> lvl{0u, 1u}; // the top tree's levels: level L is nodes [lvl[L], lvl[L + 1])
    Counters hc{};
    auto grid = [](size_t k, unsigned b) { return (unsigned)((k + b - 1) / b); };
    if (!own) {
        BVHB_TRY(cudaMallocAsync((void**)&base, s.bytes, st));
        BVHB_TRY(cudaMallocAsync((void**)&tn, cap * sizeof(TNode), st));
    }
    s = scratch_layout(n, base, small);
    k_bvh_init<<<grid(n, 256), 256, 0, st>>>(d_boxes, n, s.cen, d_order);
    k_bvh_root<<<1, 1, 0, st>>>(n, small, tn, s.open[0], s.small_list, s.cnt);
    *launches += 2;
    if (refuse && n > max_geom) { // the flag is read with the first level's counters, or before the serial subtrees when there is no level
        k_bounds_check<<<grid(6 * (size_t)n, 256), 256, 0, st>>>(d_boxes, 6 * (size_t)n, &s.cnt->empty);
        ++*launches;
    }
    n_open = n > small ? 1 : 0;
    *empty = false;
    for (int cur = 0; n_open && !hc.empty; cur ^= 1) {
        if (n_tree + 2 * (size_t)n_open > cap) { // room for this level's children
            if (own) { err = cudaErrorInvalidValue; goto done; } // top_cap(n) nodes hold every top tree
            const size_t ncap = std::max(2 * cap, n_tree + 2 * (size_t)n_open);
            TNode* t2 = nullptr;
            BVHB_TRY(cudaMallocAsync((void**)&t2, ncap * sizeof(TNode), st));
            BVHB_TRY(cudaMemcpyAsync(t2, tn, n_tree * sizeof(TNode), cudaMemcpyDeviceToDevice, st));
            BVHB_TRY(cudaFreeAsync(tn, st));
            tn = t2; cap = ncap;
        }
        Open* op = s.open[cur];
        BVHB_TRY(cudaMemsetAsync(s.seg, 0xff, (size_t)n * 4, st));
        k_bvh_seg<<<n_open, 256, 0, st>>>(op, s.seg);
        k_bvh_bounds<<<grid(n, 256), 256, 0, st>>>(n, s.seg, d_order, d_boxes, s.cen, op);
        k_bvh_axis<<<grid(n_open, 128), 128, 0, st>>>(op, n_open, max_geom);
        k_bvh_bins<<<grid(n, 256), 256, 0, st>>>(n, s.seg, d_order, d_boxes, s.cen, op);
        k_bvh_split<<<grid(n_open, 64), 64, 0, st>>>(op, n_open, max_geom, d_order, d_boxes);
        k_bvh_flags<<<grid((size_t)n + 1, 256), 256, 0, st>>>(n, s.seg, d_order, s.cen, op, s.f);
        BVHB_TRY(cub::DeviceScan::ExclusiveSum(s.cub, s.cub_bytes, s.f, s.f, (int)n + 1, st));
        k_bvh_ranks<<<grid(n, 256), 256, 0, st>>>(n, s.seg, op, s.f, s.tmp);
        k_bvh_swap<<<grid(n, 256), 256, 0, st>>>(n, s.seg, op, s.f, s.tmp, d_order);
        BVHB_TRY(cudaMemsetAsync(&s.cnt->n_next, 0, 4, st));
        k_bvh_children<<<grid(n_open, 128), 128, 0, st>>>(op, n_open, small, tn, s.open[cur ^ 1], s.small_list, s.cnt, d_order, d_boxes);
        *launches += 10;
        BVHB_TRY(cudaGetLastError());
        BVHB_TRY(cudaMemcpyAsync(&hc, s.cnt, sizeof hc, cudaMemcpyDeviceToHost, st));
        BVHB_TRY(cudaStreamSynchronize(st));
        n_tree = hc.n_tree; n_open = hc.n_next;
        lvl.push_back(n_tree);
        if (trace) trace->levels++;
    }
    BVHB_TRY(cudaMemcpyAsync(&hc, s.cnt, sizeof hc, cudaMemcpyDeviceToHost, st));
    BVHB_TRY(cudaStreamSynchronize(st));
    if (hc.empty) { *empty = true; goto done; } // nodes are left open: there is no tree to number
    if (trace && trace->after_levels) BVHB_TRY(cudaEventRecord(trace->after_levels, st));
    n_small = hc.n_small;
    if (n_small) k_bvh_small<<<grid(n_small, 64), 64, 0, st>>>(s.small_list, n_small, tn, s.cnt, max_geom, d_boxes, s.cen, n, d_order, (uint32_t*)s.f, s.snodes);
    if (trace && trace->after_small) BVHB_TRY(cudaEventRecord(trace->after_small, st));
    while (lvl.size() > 1 && lvl[lvl.size() - 2] == lvl.back()) lvl.pop_back(); // a last level that opened no node
    for (size_t L = lvl.size() - 1; L-- > 0;) k_bvh_size<<<grid(lvl[L + 1] - lvl[L], 128), 128, 0, st>>>(tn, lvl[L], lvl[L + 1]);
    for (size_t L = 0; L + 1 < lvl.size(); ++L) k_bvh_pre<<<grid(lvl[L + 1] - lvl[L], 128), 128, 0, st>>>(tn, lvl[L], lvl[L + 1]);
    k_bvh_emit<<<grid(n_tree, 128), 128, 0, st>>>(tn, n_tree, d_nodes);
    if (n_small) k_bvh_copy<<<n_small, 128, 0, st>>>(s.small_list, tn, s.snodes, d_nodes);
    for (size_t L = lvl.size() - 1; L-- > 0;) k_bvh_ibounds<<<grid(lvl[L + 1] - lvl[L], 128), 128, 0, st>>>(tn, lvl[L], lvl[L + 1], d_nodes);
    *launches += 3 + 3 * (lvl.size() - 1);
    BVHB_TRY(cudaGetLastError());
    BVHB_TRY(cudaMemcpyAsync(d_n_nodes, &tn[0].size, 4, cudaMemcpyDeviceToDevice, st));
    if (h_n_nodes) BVHB_TRY(cudaMemcpyAsync(&h_nodes, &tn[0].size, 4, cudaMemcpyDeviceToHost, st));
    BVHB_TRY(cudaMemcpyAsync(&hc, s.cnt, sizeof hc, cudaMemcpyDeviceToHost, st));
    BVHB_TRY(cudaStreamSynchronize(st));
    *empty = hc.empty != 0;
    if (h_n_nodes) *h_n_nodes = h_nodes;
done:
    if (!own) {
        if (tn) { const cudaError_t e = cudaFreeAsync(tn, st); if (err == cudaSuccess) err = e; }
        if (base) { const cudaError_t e = cudaFreeAsync(base, st); if (err == cudaSuccess) err = e; }
    }
    return err;
}
#undef BVHB_TRY

} // namespace bvhb
} // namespace trb
