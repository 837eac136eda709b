// trb_api.cu — the C ABI of include/trb.h: scene upload, per-frame update and kernel launches.
// Everything that touches device memory lives here; there is no CPU rendering path in this library.
#include <chrono>
#include <dlfcn.h>
#include <nccl.h>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <thread>
#include <cub/device/device_radix_sort.cuh>
#include "trb_host.h"
#include "trb_kernels.cuh"
#include "trb_bvh_build.cuh"
#include "trb_denoise.cuh"

using namespace trbh;

namespace {

thread_local std::string g_error;
unsigned long long g_launches = 0; // kernels launched by this library (bench.py reports it as gpu_launches)
trb_status fail(trb_status s, const std::string& msg) { g_error = msg; return s; }

#define CU(call)                                                                                                   \
    do {                                                                                                           \
        cudaError_t e_ = (call);                                                                                   \
        if (e_ != cudaSuccess) return fail(e_ == cudaErrorMemoryAllocation ? TRB_OOM : TRB_CUDA,                   \
                                           std::string(#call) + ": " + cudaGetErrorString(e_));                    \
    } while (0)

struct DeviceArena { // owns every cudaMalloc of a scene
    std::vector<void*> ptrs;
    ~DeviceArena() { for (void* p : ptrs) cudaFree(p); }
    template <class T>
    cudaError_t upload(const T* host, size_t n, T** out) {
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, std::max<size_t>(1, n) * sizeof(T));
        if (e != cudaSuccess) return e;
        ptrs.push_back(d);
        if (n) e = cudaMemcpy(d, host, n * sizeof(T), cudaMemcpyHostToDevice);
        *out = static_cast<T*>(d);
        return e;
    }
    template <class T>
    cudaError_t alloc(size_t n, T** out) {
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, std::max<size_t>(1, n) * sizeof(T));
        if (e != cudaSuccess) return e;
        ptrs.push_back(d);
        *out = static_cast<T*>(d);
        return e;
    }
    void release(const void* p) { // frees one allocation of this arena (a mesh buffer that an update replaced)
        for (size_t i = 0; i < ptrs.size(); ++i)
            if (ptrs[i] == p) { cudaFree(ptrs[i]); ptrs[i] = ptrs.back(); ptrs.pop_back(); return; }
    }
};

// A failed CUDA call as TRB_OOM (out of memory) or TRB_CUDA, with `what` leading the message; the call's error is cleared
trb_status cuda_fail(cudaError_t e, const char* what) {
    cudaGetLastError();
    return fail(e == cudaErrorMemoryAllocation ? TRB_OOM : TRB_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

// A device allocation of `bytes`; a failure is cuda_fail's and leaves *p null
trb_status device_alloc(void** p, size_t bytes, const char* what) {
    const cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaSuccess) return TRB_OK;
    *p = nullptr;
    return cuda_fail(e, what);
}

// A per-call device temporary, freed with the scope
struct DeviceBuffer {
    void* p = nullptr;
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    ~DeviceBuffer() { reset(); }
    trb_status alloc(size_t bytes, const char* what) { return device_alloc(&p, bytes, what); }
    cudaError_t reset() { const cudaError_t e = p ? cudaFree(p) : cudaSuccess; p = nullptr; return e; }
    template <class T> T* as() const { return static_cast<T*>(p); }
};

using Span = std::pair<const void*, size_t>;
using OutSpan = std::pair<void*, size_t>;

// The blocking host form of a call. Each input span is copied into a device buffer of its own, and each output span whose host pointer
// is not null gets one; enqueue(d) runs on the default stream with d the buffers of the inputs, then of the outputs (a null output's
// holds null), and the outputs are copied back. Passes a failed enqueue left in flight still read the buffers, so the device is
// drained before they are freed.
template <class Enqueue>
trb_status run_staged(std::initializer_list<Span> ins, std::initializer_list<OutSpan> outs, Enqueue enqueue) {
    std::vector<DeviceBuffer> d(ins.size() + outs.size());
    DeviceBuffer* b = d.data();
    trb_status r;
    for (const Span& in : ins) {
        if ((r = b->alloc(in.second, "host-form staging")) != TRB_OK) return r;
        CU(cudaMemcpy(b->p, in.first, in.second, cudaMemcpyHostToDevice));
        ++b;
    }
    for (const OutSpan& out : outs) {
        if (out.first && (r = b->alloc(out.second, "host-form staging")) != TRB_OK) return r;
        ++b;
    }
    if ((r = enqueue(d.data())) != TRB_OK) { cudaDeviceSynchronize(); return r; }
    b = d.data() + ins.size();
    for (const OutSpan& out : outs) {
        if (out.first) CU(cudaMemcpy(out.first, b->p, out.second, cudaMemcpyDeviceToHost));
        ++b;
    }
    return TRB_OK;
}

// The device forms' alignment check: TRB_INVALID_ARG with `msg` unless every pointer is a multiple of its alignment (a power of two)
trb_status check_aligned(std::initializer_list<std::pair<const void*, uintptr_t>> ptrs, const char* msg) {
    for (const auto& [p, align] : ptrs)
        if (reinterpret_cast<uintptr_t>(p) & (align - 1)) return fail(TRB_INVALID_ARG, msg);
    return TRB_OK;
}

// Whether two buffers overlap (a null one overlaps nothing)
bool spans_overlap(Span a, Span b) {
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(a.first), b0 = reinterpret_cast<uintptr_t>(b.first);
    return a.first && b.first && a0 < b0 + b.second && b0 < a0 + a.second;
}
bool overlaps_any(Span a, std::initializer_list<Span> others) {
    for (const Span& b : others) if (spans_overlap(a, b)) return true;
    return false;
}

struct HostMesh {
    std::vector<trb_bvh_node> nodes;
    std::vector<uint32_t> order;
    Box3 bounds;
    uint32_t n_verts = 0;
    bool narrow = true;    // every leaf fits the narrow reference (pack_pairs)
    size_t pair_cap = 0;   // DPair records the mesh's record buffer holds
    // trb_scene_refit_mesh: the boxes of `nodes` are stale once a refit rewrote the device records (refresh_host_tree reads them back
    // when a host reader needs them). d_refit holds, per record, its parent link (k_refit_parents) and then its arrival counter; it
    // follows the topology, so a rebuild or a removal of the mesh releases it.
    bool stale = false;
    uint32_t* d_refit = nullptr;
};

uint32_t pow2_ceil(uint32_t v) { uint32_t p = 1; while (p < v) p <<= 1; return p; }

// Re-layout of the reference-order flat tree into child-pair records (trb_device.h DPair). Pure layout: no box,
// child order or primitive order changes. Returns false if a leaf does not fit the 25-bit slot / 5-bit count fields, or,
// `wide` (mesh levels only: REF_LEAF | first slot, the leaf's end is marked in its last DTri), if a leaf is empty or ends past 2^30.
float bits_f(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
constexpr uint32_t QUAD_EMPTY_HOST = 0xffffffffu;
bool pack_pairs(const std::vector<trb_bvh_node>& in, std::vector<trb::DPair>& out, trb::DBvh& hdr, bool wide = false) {
    std::vector<uint32_t> rec_of(in.size(), 0);
    uint32_t n_rec = 0;
    for (size_t i = 0; i < in.size(); ++i) if (!(in[i].b & TRB_BVH_LEAF)) rec_of[i] = n_rec++;
    bool ok = n_rec < (1u << 30);
    auto ref_of = [&](uint32_t i) -> uint32_t {
        if (in[i].b & TRB_BVH_LEAF) {
            const uint32_t cnt = in[i].b & ~TRB_BVH_LEAF, first = in[i].a;
            if (wide) {
                if (cnt == 0 || (uint64_t)first + cnt > (1u << 30)) ok = false;
                return trb::REF_LEAF | (first & ~trb::REF_TAG);
            }
            if (cnt > 31 || first >= (1u << 25)) ok = false;
            return trb::REF_LEAF | (cnt << 25) | first;
        }
        return trb::REF_INTERIOR | rec_of[i];
    };
    out.resize(n_rec);
    for (size_t i = 0; i < in.size(); ++i) {
        if (in[i].b & TRB_BVH_LEAF) continue;
        const trb_bvh_node& l = in[i + 1];
        const trb_bvh_node& r = in[in[i].a];
        trb::DPair& p = out[rec_of[i]];
        p.l_lo = make_float4(l.bmin[0], l.bmin[1], l.bmin[2], bits_f(ref_of((uint32_t)i + 1)));
        p.l_hi = make_float4(l.bmax[0], l.bmax[1], l.bmax[2], bits_f(ref_of(in[i].a)));
        p.r_lo = make_float4(r.bmin[0], r.bmin[1], r.bmin[2], bits_f(in[i].b));
        p.r_hi = make_float4(r.bmax[0], r.bmax[1], r.bmax[2], 0.f);
    }
    hdr.root_lo = make_float4(in[0].bmin[0], in[0].bmin[1], in[0].bmin[2], bits_f(ref_of(0)));
    hdr.root_hi = make_float4(in[0].bmax[0], in[0].bmax[1], in[0].bmax[2], 0.f);
    return ok;
}
// Whether every leaf of a mesh tree fits the narrow reference (count << 25 | first slot). A scene whose meshes all fit uses the
// narrow form unless the option trace.wide_leaf asks for the wide one.
bool leaves_fit_narrow(const std::vector<trb_bvh_node>& in) {
    for (const trb_bvh_node& n : in)
        if ((n.b & TRB_BVH_LEAF) && ((n.b & ~TRB_BVH_LEAF) > 31 || n.a >= (1u << 25))) return false;
    return true;
}

// Collapse pairs of levels of the reference-order tree into DQuad records (trb_device.h). Layout only: boxes, child
// order and primitive order are the reference's. A child whose box is not inside its parent's (cannot happen for boxes
// built as unions, checked anyway) is kept as a one-slot half so the containment argument never has to be trusted.
// Returns the root reference in DQuad index space.
bool pack_quads(const std::vector<trb_bvh_node>& in, std::vector<trb::DQuad>& out, uint32_t& root_ref) {
    out.clear();
    bool ok = true;
    auto is_leaf = [&](uint32_t i) { return (in[i].b & TRB_BVH_LEAF) != 0; };
    auto leaf_ref = [&](uint32_t i) -> uint32_t {
        const uint32_t cnt = in[i].b & ~TRB_BVH_LEAF, first = in[i].a;
        if (cnt > 31 || first >= (1u << 25)) ok = false;
        return trb::REF_LEAF | (cnt << 25) | first;
    };
    auto inside = [&](uint32_t c, uint32_t p) {
        for (int k = 0; k < 3; ++k) if (!(in[c].bmin[k] >= in[p].bmin[k] && in[c].bmax[k] <= in[p].bmax[k])) return false;
        return true;
    };
    if (in.empty()) { root_ref = QUAD_EMPTY_HOST; return true; }
    if (is_leaf(0)) { root_ref = leaf_ref(0); return ok; }
    // quad roots in depth-first order (a record is followed by the records below its first slots: locality for near-first descent)
    std::vector<uint32_t> quad_of(in.size(), 0xffffffffu), order, todo{0};
    while (!todo.empty()) {
        const uint32_t p = todo.back(); todo.pop_back();
        quad_of[p] = (uint32_t)order.size(); order.push_back(p);
        uint32_t kids[4]; int nk = 0;
        for (uint32_t c : {p + 1, in[p].a}) {
            if (is_leaf(c)) continue;
            const uint32_t g0 = c + 1, g1 = in[c].a;
            if (inside(g0, c) && inside(g1, c)) { if (!is_leaf(g0)) kids[nk++] = g0; if (!is_leaf(g1)) kids[nk++] = g1; }
            else kids[nk++] = c;
        }
        for (int k = nk; k-- > 0;) todo.push_back(kids[k]);
    }
    if (order.size() >= (1u << 30)) return false;
    out.resize(order.size());
    auto slot = [&](trb::DQuad& q, int k, uint32_t node, bool empty) {
        if (empty) { q.q[2 * k] = make_float4(0.f, 0.f, 0.f, bits_f(0xffffffffu)); q.q[2 * k + 1] = make_float4(0.f, 0.f, 0.f, 0.f); return; }
        const uint32_t ref = is_leaf(node) ? leaf_ref(node) : (trb::REF_INTERIOR | quad_of[node]);
        q.q[2 * k] = make_float4(in[node].bmin[0], in[node].bmin[1], in[node].bmin[2], bits_f(ref));
        q.q[2 * k + 1] = make_float4(in[node].bmax[0], in[node].bmax[1], in[node].bmax[2], 0.f);
    };
    for (size_t qi = 0; qi < order.size(); ++qi) {
        const uint32_t p = order[qi];
        trb::DQuad& q = out[qi];
        uint32_t axes[2] = {0, 0};
        int h = 0;
        for (uint32_t c : {p + 1, in[p].a}) {
            bool split = false;
            if (!is_leaf(c)) { const uint32_t g0 = c + 1, g1 = in[c].a; split = inside(g0, c) && inside(g1, c); }
            if (split) { slot(q, 2 * h, c + 1, false); slot(q, 2 * h + 1, in[c].a, false); axes[h] = in[c].b & 3u; }
            else { slot(q, 2 * h, c, false); slot(q, 2 * h + 1, 0, true); }
            ++h;
        }
        q.q[1].w = bits_f((in[p].b & 3u) | axes[0] << 2 | axes[1] << 4);
    }
    root_ref = trb::REF_INTERIOR | quad_of[0];
    return ok;
}

} // namespace

namespace {
// Launch-shape knobs of the wavefront pipeline. Read ONCE from the environment when the scene is created (developer
// sweeps), changed afterwards only through trb_scene_set_option: the launch path never touches getenv.
struct Tuning {
    int refill = 8;            // trace: idle lanes that trigger a warp refill
    unsigned trace_grid = 0;   // trace: CTAs per SM launched (0 = twice what the chosen variant keeps resident)
    uint32_t sched = 6;        // trace: quorum of the phased loop (0 = flat state machine)
    int quads = 0;             // trace: DQuad two-level records
    int exact_box = 0;         // trace: test option — every ray takes the literal BBox::fast_intersect transcription (box_hit) instead of box_hit_finite
    int wide_leaf = 0;         // trace: test option — 1: wide mesh leaf references for every scene; 0: only where a mesh leaf does not fit the narrow form
    int pipe = 36;             // trace: kernel variant. 0 = round-1 kernel; 1 = + box_hit_finite; 33 = + RayHome + fused non-node chains at 7 CTAs per SM; 34 / 35 / 36 / 37 = the same at 8 / 8 / 9 / 9 CTAs with 16 / 12 / 12 / 8 stack entries in shared memory
    int film_v2 = 1;           // film: per-warp private tiles (0 = shared-memory atomics)
    int sort = 0;              // ray queues: 0 = path order; 1 / 2 = counting sort by (octant, origin cell) / (cell, octant) before each trace round
    int sort_bits = 5;         // bits per axis of the origin cell grid
    int sort_min_round = 1;    // first bounce round whose queues are sorted (round 0 = primary rays, already coherent)
    int shade_anim_occ = 4;    // keyframed shade kernel variant: resident CTAs per SM it is compiled for (3 or 4)
    int frame_device = 1;      // Scene::update_frame on the device (instance transforms, animation bounds, TLAS SAH build); 0 = on the host
    int anim_table = 2;        // keyframed scenes: evaluate each keyframed instance's transform once per path (0 = per ray per instance, like the reference; 1 = one thread per (path, instance) evaluates the whole stack; 2 = each distinct keyframed spline once per path, then the stacks)
    int shade_split = -1;      // shading as three kernels (surface | direct light | BSDF sample) instead of one: 1 / 0, -1 = per scene — split
                               // when the scene mixes material kinds or uses MERL, fused for other one-material scenes
    int shade_sort = 1;        // split shading: bucket the paths by material kind between k_wf_shade_a and _b / _c
    int shade_kind = 1;        // split shading with buckets: the matte bucket goes through _b / _c instantiations compiled for matte alone
    uint64_t pass_paths = 1ull << 24; // camera samples per wavefront pass (the frame is rendered in additive passes)
    int build_device = 1;      // scene creation: mesh BVHs built on the device (trb_bvh_build.cuh); 0 = on the host, as when the build's scratch does not fit
    long long tlas_min = -1;   // frame: test option — the instance count from which the device frame path builds the instance tree with the level
                               // builder instead of one thread; -1 = kTlasLevelMin. The tree does not depend on it
    int frame_time = 0;        // TRB_FRAME_TIME=1: trb_scene_update_frame prints its phases to stderr
    int tlas_small = 8;        // frame: the level builder's serial-subtree threshold (TRB_FRAME_TLAS_SMALL; swept below; the tree does not depend on it)
};
// The instance tree of a frame (device path). One thread (k_tlas_build) is two launches and no synchronisation but the final
// read-back; the level builder (bvhb::build_device) is tens of launches and a stream synchronisation per level, and overtakes it
// once the serial build costs more than those. tools/tlas_bench.py, scene_instances(k), NVIDIA H100 80GB HBM3 at a 700 W limit, median
// of five update_frame calls alternating the two, two calls of the tool, one-thread / level builder in ms: k = 10: 0.19-0.44 / 0.57-0.82;
// 100: 0.78-0.88 / 1.30-1.70; 10^3: 6.62-6.83 / 1.90-2.22; 10^4: 87.0-87.9 / 2.44-2.60; 10^5: 1167 / 3.95-4.09. The one-thread build
// grows by about 6.5 us per instance and the level builder by a level (about 0.1 ms) per doubling, so the two meet near 200 instances;
// the level builder runs from 256, where interpolation puts it at 1.4 ms against 1.8 ms.
constexpr uint32_t kTlasLevelMin = 256;
// Tuning::tlas_small, the level builder's serial-subtree threshold for the instance tree (meshes use bvhb::SMALL = 1024, but a thousand
// boxes cost one thread about 6 ms, the k = 10^3 figure above, which a frame cannot hide). Swept with
// TRB_FRAME_TLAS_SMALL under tools/tlas_bench.py on an NVIDIA H100 80GB HBM3 at a 700 W limit, update_frame in ms at 10^3 / 10^5 instances:
// 8: 1.79 / 3.32; 16: 2.28 / 4.00; 32: 3.36 / 5.13; 64: 5.49 / 8.71; 128: 8.49 / 17.1; 1024: 19.3 / 178. At 8 the level loop (17 levels,
// 2.29 ms at 10^5) outweighs the serial subtrees (0.30 ms); at 32 it is the reverse (1.79 / 2.42 ms).
int env_int(const char* name, int dflt) { const char* v = getenv(name); return v ? (int)strtol(v, nullptr, 0) : dflt; }
void tuning_from_env(Tuning& t) {
    t.refill = env_int("TRB_REFILL", t.refill); t.trace_grid = (unsigned)env_int("TRB_TRACE_GRID", (int)t.trace_grid);
    t.sched = (uint32_t)env_int("TRB_TRACE_SCHED", (int)t.sched); t.quads = env_int("TRB_TRACE_QUADS", t.quads); t.pipe = env_int("TRB_TRACE_PIPE", t.pipe);
    t.wide_leaf = env_int("TRB_TRACE_WIDE_LEAF", t.wide_leaf);
    t.film_v2 = env_int("TRB_FILM_V2", t.film_v2); t.sort = env_int("TRB_SORT", t.sort); t.sort_bits = env_int("TRB_SORT_BITS", t.sort_bits);
    t.sort_min_round = env_int("TRB_SORT_MIN_ROUND", t.sort_min_round); t.shade_split = env_int("TRB_SHADE_SPLIT", t.shade_split); t.anim_table = env_int("TRB_ANIM_TABLE", t.anim_table); t.frame_device = env_int("TRB_FRAME_DEVICE", t.frame_device);
    if (getenv("TRB_PASS_PATHS")) t.pass_paths = strtoull(getenv("TRB_PASS_PATHS"), nullptr, 0);
    t.build_device = env_int("TRB_BUILD_DEVICE", t.build_device);
    t.tlas_min = env_int("TRB_FRAME_TLAS_MIN", (int)t.tlas_min); t.frame_time = env_int("TRB_FRAME_TIME", t.frame_time);
    t.tlas_small = std::max(4, env_int("TRB_FRAME_TLAS_SMALL", t.tlas_small)); // the level kernels have no case for fewer than five boxes
}

} // namespace

struct BlockList { // one selection of the Morton block list, resident on the device (never overwritten in place: kernels in flight may read it)
    uint32_t key[5];
    std::vector<uint32_t> host; // (bx, by) pairs
    uint2* dev = nullptr;
};

struct trb_scene {
    int device = 0;
    int sm_count = 0;          // cudaDeviceProp::multiProcessorCount of `device`, read when the scene is created
    Tuning tune;
    // deep copy of the description
    trb_film film{};
    trb_integrator integrator{};
    std::vector<trb_camera> cameras;
    std::vector<trb_instance> instances;
    std::vector<trb_spline> splines;
    std::vector<trb_keyframe> keyframes;
    std::vector<float> knots;
    std::vector<trb_color_key> color_keys;
    std::vector<float> fov_floats;
    std::vector<trb_material> materials;
    uint32_t n_merl = 0;                 // MERL tables of the description (a material edit is checked against it)
    std::vector<HostMesh> meshes;
    std::vector<trb::DMesh> dmeshes;     // the device mesh headers (d_meshes), kept to re-pack the node records (trace.wide_leaf)
    trb::DMesh* d_meshes = nullptr;
    bool needs_wide = false;             // some mesh leaf does not fit the narrow reference (a mesh of more than 2^25 triangles)
    bool quads_dropped = false;          // trb_scene_update_mesh rebuilt a mesh, which has no DQuad records (trace.quads) since
    bool wide_leaf = false;              // the mesh node records hold wide leaf references: the WIDE kernel instantiations run
    uint32_t spp_pow2 = 1;
    uint32_t n_anim = 0;                 // instances whose transform stack is keyframed (evaluated per path into WfState::xf_tab)
    std::vector<uint32_t> anim_list;     // those instances, and whether any instance's transform or emission depends on time: properties
    bool inst_any_anim = false;          // of the object section (static_instance_records), kept so that a frame need not rebuild the records
    bool frame_set = false; uint32_t last_frame = 0; float last_start = 0, last_end = 0; // the arguments of the last update_frame (re-run when an option changes what it builds)
    uint32_t material_kinds = 0;         // bit k: some hittable instance's material is of kind k (TRB_MAT_*)
    bool mixed_materials = false;        // the hittable instances use >= 2 material kinds or a MERL table: the split shade kernels with material buckets win (Tuning::shade_split = -1)
    bool anim_emission = false;          // some emitter's colour is keyframed (ds.has_anim is only known after update_frame; trb_emitted runs before it)
    uint32_t* d_anim_instances = nullptr;
    // per-frame host state
    int active_camera = -1;
    float shutter_open = 0, shutter_close = 0;
    std::vector<Xf> world; // instance world transforms of the current frame
    std::vector<trb_bvh_node> tlas_nodes;
    std::vector<uint32_t> tlas_order;
    float table[256];
    // device
    DeviceArena arena;
    trb::DScene ds{};
    trb::DInstance* d_instances = nullptr;
    trb::DPair* d_tlas = nullptr;
    trb::DQuad* d_tlas_quads = nullptr;
    trb::DBvh* d_tlas_hdr = nullptr;
    uint32_t* d_tlas_order = nullptr;
    size_t tlas_capacity = 0;
    // device-side update_frame (k_frame_instances / k_tlas_build): reference-order nodes, instance bounds, builder scratch
    trb_bvh_node* d_tlas_nodes = nullptr;
    float* d_bounds = nullptr;           // n x Box3 (6 floats)
    float* d_build_f = nullptr;
    uint32_t* d_build_u = nullptr;
    uint32_t* d_build_counts = nullptr;
    char* d_build_level = nullptr;       // the level builder's scratch, top tree and scan storage (LevelScratch) for tlas_capacity - 1 instances,
                                         // allocated with the first frame that runs it and released where the capacity grows
    uint32_t tlas_n_nodes = 0;
    bool instances_static_uploaded = false, host_frame_stale = false;
    std::vector<BlockList> block_lists;
    uint32_t* d_counter = nullptr;
    int* d_error = nullptr;
    trb::DStats* d_stats = nullptr;
    float4* d_film = nullptr;
    float* h_film_staging = nullptr; // pinned
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool frame_ready = false;
    // wavefront path state (grown on demand, owned outside the arena so it can be re-sized)
    trb::WfState wf{};
    size_t wf_capacity = 0;
    std::vector<void*> wf_allocs;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> trace_events; // TRB_RENDER_TIME_TRACE
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> event_pool;
    // Adaptive sampler (trb_render_adaptive), allocated on first use: per-pixel state (trbh::AdPixel), the round's block list
    // twice (compaction ping-pong) with each block's index in the selection, per-block "still sampling" flags
    uint4* d_ad_state = nullptr;
    uint2* d_ad_list[2] = {nullptr, nullptr};
    uint32_t* d_ad_index[2] = {nullptr, nullptr};
    uint32_t* d_ad_flags = nullptr;
    uint32_t* d_ad_count = nullptr;
    uint32_t* d_ad_spp = nullptr;
    // caller film writes (trb_film_write): sort keys and sample order (double-buffered), region starts, CUB's temporary storage
    void* d_film_scratch = nullptr;
    size_t film_scratch_bytes = 0;
    // AOV records of a film render's pass (trb_render_aov*), allocated by the first AOV render at the path-state capacity: per path
    // (albedo, depth) in d_aov[p] and (n, inst bits) in d_aov[aov_capacity + p], 32 bytes
    float4* d_aov = nullptr;
    size_t aov_capacity = 0;
    // motion records of a film render's pass (trb_render_*aov_motion*), allocated by the first motion render at the path-state capacity:
    // per path (v dx, v dy, v, 0), 16 bytes
    float4* d_motion = nullptr;
    size_t motion_capacity = 0;
    // denoiser scratch (trb_denoise*; trb::DnScratch), allocated by the first denoise for the film's pixel count and released with the film;
    // denoise_moments: it also holds the moment records of trb_denoise_moments* (trb::DN_MOMENTS_BYTES_PER_PIXEL)
    void* d_denoise = nullptr;
    size_t denoise_pixels = 0;
    bool denoise_moments = false;
    // the AOV films of a sharded or group AOV render (trb_render_sharded_aov, trb_group_render_aov and their Adaptive forms), allocated
    // by the first such render for the film's pixel count and released with the film: per pixel albedo_w, then normal_w (float4 each),
    // then nearest (uint64), each a whole-film run, so that the NCCL reduce can sum both films in one call
    void* d_shard_aov = nullptr;
    // temporal denoising (trb_denoise_temporal*): the inverse of the camera's cam_world at the current frame's shutter-open, and the
    // object generation, counted up by the calls that renumber instances (replace_objects, replace_meshes with an object section)
    float cam_inv[16] = {};
    uint64_t object_generation = 0;
    ~trb_scene() {
        for (void* p : {(void*)d_ad_state, (void*)d_ad_list[0], (void*)d_ad_list[1], (void*)d_ad_index[0], (void*)d_ad_index[1], (void*)d_ad_flags,
                        (void*)d_ad_count, (void*)d_ad_spp, d_film_scratch, (void*)d_aov, (void*)d_motion, d_denoise, d_shard_aov}) if (p) cudaFree(p);
        for (auto& b : block_lists) cudaFree(b.dev);
        for (void* p : wf_allocs) cudaFree(p);
        for (auto& e : trace_events) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
        for (auto& e : event_pool) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
        if (h_film_staging) cudaFreeHost(h_film_staging);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
    }
};

namespace {

Box3 shape_bounds(const trb_scene& s, const trb_instance& in) {
    Box3 b;
    switch (in.shape) {
        case TRB_SHAPE_SPHERE: for (int i = 0; i < 3; ++i) { b.lo[i] = -in.p0; b.hi[i] = in.p0; } break;          // sphere.rs:84-88
        case TRB_SHAPE_DISK: b.lo[0] = b.lo[1] = -in.p0; b.hi[0] = b.hi[1] = in.p0; b.lo[2] = -0.1f; b.hi[2] = 0.1f; break; // disk.rs:79-81
        case TRB_SHAPE_RECT: { const float hw = in.p0 / 2.0f, hh = in.p1 / 2.0f; b.lo[0] = -hw; b.lo[1] = -hh; b.hi[0] = hw; b.hi[1] = hh; b.lo[2] = b.hi[2] = 0.0f; break; } // rectangle.rs:67-71
        case TRB_SHAPE_MESH: b = s.meshes[in.mesh].bounds; break;                                                   // mesh.rs:87-90
        default: for (int i = 0; i < 3; ++i) b.lo[i] = b.hi[i] = 0.0f;                                            // point light (emitter.rs:152)
    }
    return b;
}

// One material of a description (trb_scene_create, trb_scene_update_materials)
trb_status validate_material(const trb_material& m, uint32_t n_merl, uint32_t n_textures) {
    if (m.type > TRB_MAT_MERL) return fail(TRB_INVALID_ARG, "unrecognized material type");
    if (m.type == TRB_MAT_MERL && m.merl >= n_merl) return fail(TRB_INVALID_ARG, "merl table index out of range");
    for (int k = 0; k < 4; ++k) if (m.tex[k] > n_textures) return fail(TRB_INVALID_ARG, "texture index out of range");
    return TRB_OK;
}

// The object section of a description (trb_scene_create, trb_scene_replace_objects); mesh and material indices against the counts given
trb_status validate_objects(const trb_scene_objects& o, uint32_t n_meshes, uint32_t n_materials) {
    if (o.n_instances == 0) return fail(TRB_INVALID_ARG, "Aborting: the scene does not have any objects!"); // scene.rs:134
    if (o.n_cameras == 0) return fail(TRB_INVALID_ARG, "Error: A camera is required!");
    if (!o.cameras || !o.instances || (o.n_splines && !o.splines) || (o.n_keyframes && !o.keyframes) || (o.n_knots && !o.knots) ||
        (o.n_color_keys && !o.color_keys) || (o.n_fov_floats && !o.fov_floats))
        return fail(TRB_INVALID_ARG, "null array with a non-zero count");
    bool light = false;
    for (uint32_t i = 0; i < o.n_instances; ++i) {
        const trb_instance& in = o.instances[i];
        if (in.kind > TRB_INST_EMITTER_POINT || in.shape > TRB_SHAPE_MESH) return fail(TRB_INVALID_ARG, "unknown instance kind/shape");
        if (in.kind != TRB_INST_EMITTER_POINT && in.shape == TRB_SHAPE_NONE) return fail(TRB_INVALID_ARG, "instance without geometry");
        if (in.kind == TRB_INST_EMITTER_AREA && in.shape == TRB_SHAPE_MESH)
            return fail(TRB_INVALID_ARG, "Geometry of type 'mesh' is not sampleable and can't be used for area light geometry"); // scene.rs:577-579
        if (in.shape == TRB_SHAPE_MESH && in.mesh >= n_meshes) return fail(TRB_INVALID_ARG, "mesh index out of range");
        if (in.kind != TRB_INST_EMITTER_POINT && in.material >= n_materials) return fail(TRB_INVALID_ARG, "material index out of range");
        if ((uint64_t)in.spline_first + in.n_splines > o.n_splines) return fail(TRB_INVALID_ARG, "spline range out of bounds");
        if (in.kind != TRB_INST_RECEIVER) {
            light = true;
            if (in.n_emission == 0 || (uint64_t)in.emission_first + in.n_emission > o.n_color_keys) return fail(TRB_INVALID_ARG, "An emission color is required for emitters");
        }
    }
    for (uint32_t k = 0; k < o.n_splines; ++k) { // BSpline::new's invariants (bspline 0.2.2) + the device evaluator's degree cap
        const trb_spline& sp = o.splines[k];
        if (sp.n_ctrl == 0 || (uint64_t)sp.ctrl_first + sp.n_ctrl > o.n_keyframes) return fail(TRB_INVALID_ARG, "spline control points out of bounds");
        if (sp.n_ctrl > 1) {
            if ((uint64_t)sp.knot_first + sp.n_knots > o.n_knots) return fail(TRB_INVALID_ARG, "spline knots out of bounds");
            if (sp.n_ctrl <= sp.degree) return fail(TRB_INVALID_ARG, "Too few control points for curve"); // BSpline::new panics with this message
            if ((uint64_t)sp.n_knots != (uint64_t)sp.n_ctrl + sp.degree + 1) return fail(TRB_INVALID_ARG, "Invalid B-spline: knots.len() != control_points.len() + degree + 1");
            if (sp.degree > (uint32_t)trbh::kMaxSplineDegree) return fail(TRB_UNSUPPORTED, "B-spline degree above 5");
            for (uint32_t i = 0; i < sp.n_knots; ++i) if (o.knots[sp.knot_first + i] != o.knots[sp.knot_first + i]) return fail(TRB_INVALID_ARG, "NaN knot in B-spline"); // BSpline::new sorts with partial_cmp().unwrap(): panics on NaN
        }
    }
    if (!light) return fail(TRB_INVALID_ARG, "At least one light is required"); // multithreaded.rs:39
    for (uint32_t i = 0; i < o.n_cameras; ++i) {
        const trb_camera& c = o.cameras[i];
        if (c.n_fov_ctrl) { // CameraFov::Animated (camera.rs:95-125)
            if ((uint64_t)c.fov_ctrl_first + c.n_fov_ctrl > o.n_fov_floats || (uint64_t)c.fov_knot_first + c.n_fov_knots > o.n_fov_floats) return fail(TRB_INVALID_ARG, "fov spline out of bounds");
            if (c.n_fov_ctrl <= c.fov_degree) return fail(TRB_INVALID_ARG, "Too few control points for curve");
            if ((uint64_t)c.n_fov_knots != (uint64_t)c.n_fov_ctrl + c.fov_degree + 1) return fail(TRB_INVALID_ARG, "Invalid B-spline: knots.len() != control_points.len() + degree + 1");
            for (uint32_t i = 0; i < c.n_fov_knots; ++i) if (o.fov_floats[c.fov_knot_first + i] != o.fov_floats[c.fov_knot_first + i]) return fail(TRB_INVALID_ARG, "NaN knot in B-spline");
            if (c.fov_degree > (uint32_t)trbh::kMaxSplineDegree) return fail(TRB_UNSUPPORTED, "B-spline degree above 5");
        }
        if ((uint64_t)c.spline_first + c.n_splines > o.n_splines) return fail(TRB_INVALID_ARG, "camera spline range out of bounds");
    }
    return TRB_OK;
}

trb_scene_objects desc_objects(const trb_scene_desc& d) {
    return {d.n_cameras, d.cameras, d.n_instances, d.instances, d.n_splines, d.splines, d.n_keyframes, d.keyframes,
            d.n_knots, d.knots, d.n_color_keys, d.color_keys, d.n_fov_floats, d.fov_floats};
}

// One mesh of a description (trb_scene_create, trb_scene_replace_meshes). Device arrays (`device`) are not read here: their indices
// are checked on the device once copied (setup_mesh), with the same message.
trb_status validate_mesh(const trb_mesh& m, bool device) {
    if (m.n_tris == 0 || m.n_verts == 0) return fail(TRB_INVALID_ARG, "empty mesh");
    // the wide leaf references hold a 30-bit slot; the kernels index vertex attributes as 3 * index in 32 bits
    if (m.n_tris > (1u << 30)) return fail(TRB_UNSUPPORTED, "mesh too large for the wide leaf encoding (2^30 triangles)");
    if (m.n_verts > 0xffffffffu / 3) return fail(TRB_UNSUPPORTED, "mesh has too many vertices (more than (2^32 - 1) / 3)");
    if (!m.positions || !m.normals || !m.texcoords || !m.indices) return fail(TRB_INVALID_ARG, "Normals and texture coordinates are required!"); // mesh.rs:57-61
    if (!device)
        for (size_t k = 0; k < 3 * (size_t)m.n_tris; ++k) if (m.indices[k] >= m.n_verts) return fail(TRB_INVALID_ARG, "mesh index out of range");
    return TRB_OK;
}

// The film and the integrator of a description (trb_scene_create, trb_scene_replace_settings)
trb_status validate_settings(const trb_film& f, const trb_integrator& in) {
    if (f.width == 0 || f.height == 0 || f.width % 8 || f.height % 8)
        return fail(TRB_INVALID_ARG, "Image not evenly divided by blocks of (8, 8)"); // block_queue.rs:29-31
    if (f.frames == 0) return fail(TRB_INVALID_ARG, "film.frames must be >= 1");
    if (in.type > TRB_INTEGRATOR_NORMALS_DEBUG) return fail(TRB_INVALID_ARG, "Unrecognized integrator type"); // scene.rs:313
    if (in.type == TRB_INTEGRATOR_PATH && in.max_depth > 57u) return fail(TRB_UNSUPPORTED, "max_depth > 57");
    if (in.type == TRB_INTEGRATOR_WHITTED && in.max_depth > 24u) return fail(TRB_UNSUPPORTED, "whitted max_depth > 24 (device recursion stack)");
    if (!(f.filter_w > 0.0f && f.filter_h > 0.0f)) return fail(TRB_INVALID_ARG, "filter width/height must be positive");
    if (floorf(f.filter_w / 0.5f) > 8.0f || floorf(f.filter_h / 0.5f) > 8.0f) return fail(TRB_UNSUPPORTED, "filter wider than 4 pixels");
    return TRB_OK;
}

trb_scene_materials desc_materials(const trb_scene_desc& d) {
    return {d.n_materials, d.materials, d.n_merl, d.merl_tables, d.n_textures, d.textures, d.n_images, d.images};
}

// The material section of a description (trb_scene_create, trb_scene_replace_materials): materials against its own MERL and texture
// counts, texture image ranges, images and the texel limit. Images in device memory are checked the same way (their pixels are not read).
trb_status validate_materials(const trb_scene_materials& m) {
    for (uint32_t i = 0; i < m.n_materials; ++i) {
        const trb_status r = validate_material(m.materials[i], m.n_merl, m.n_textures);
        if (r != TRB_OK) return r;
    }
    uint64_t texels = 0;
    for (uint32_t i = 0; i < m.n_textures; ++i)
        if (m.textures[i].n_images == 0 || (uint64_t)m.textures[i].first_image + m.textures[i].n_images > m.n_images) return fail(TRB_INVALID_ARG, "texture image range out of bounds");
    for (uint32_t i = 0; i < m.n_images; ++i) {
        if (m.images[i].width == 0 || m.images[i].height == 0 || !m.images[i].rgba8) return fail(TRB_INVALID_ARG, "empty image");
        texels += (uint64_t)m.images[i].width * m.images[i].height;
    }
    if (texels >= (1ull << 32)) return fail(TRB_UNSUPPORTED, "more than 2^32 texels of image textures");
    return TRB_OK;
}

trb_status validate(const trb_scene_desc* d) {
    if (!d) return fail(TRB_INVALID_ARG, "null scene description");
    if (d->abi_version != TRB_ABI_VERSION) return fail(TRB_INVALID_ARG, "trb_scene_desc.abi_version mismatch");
    { const trb_status r = validate_settings(d->film, d->integrator); if (r != TRB_OK) return r; }
    { const trb_status r = validate_objects(desc_objects(*d), d->n_meshes, d->n_materials); if (r != TRB_OK) return r; }
    { const trb_status r = validate_materials(desc_materials(*d)); if (r != TRB_OK) return r; }
    for (uint32_t i = 0; i < d->n_meshes; ++i) {
        const trb_status r = validate_mesh(d->meshes[i], false);
        if (r != TRB_OK) return r;
    }
    return TRB_OK;
}

// The selected, sharded block list on the device. Lists are cached per selection and never overwritten in place, so a
// pass still in flight on a caller stream keeps reading valid memory when the next call selects other blocks.
trb_status ensure_blocks(trb_scene* s, const trb_render_cfg* cfg, const uint2** d_blocks, uint32_t* n_blocks) {
    if (cfg->shard_count > 1 && cfg->shard_index >= cfg->shard_count) return fail(TRB_INVALID_ARG, "shard_index must be < shard_count");
    const uint32_t key[5] = {cfg->block_start, cfg->block_count, cfg->shard_index, cfg->shard_count, cfg->shard_chunk};
    for (const BlockList& b : s->block_lists)
        if (std::memcmp(b.key, key, sizeof key) == 0) { *d_blocks = b.dev; *n_blocks = (uint32_t)(b.host.size() / 2); return TRB_OK; }
    if (s->block_lists.size() >= 16) { // bounded cache: retire everything once nothing can be reading it any more
        CU(cudaDeviceSynchronize());
        for (BlockList& b : s->block_lists) cudaFree(b.dev);
        s->block_lists.clear();
    }
    BlockList bl;
    std::memcpy(bl.key, key, sizeof key);
    bl.host = morton_blocks(s->film.width, s->film.height, cfg->block_start, cfg->block_count, cfg->shard_index, cfg->shard_count, cfg->shard_chunk);
    const size_t n = bl.host.size() / 2;
    CU(cudaMalloc(reinterpret_cast<void**>(&bl.dev), std::max<size_t>(1, n) * sizeof(uint2)));
    if (n) { cudaError_t e = cudaMemcpy(bl.dev, bl.host.data(), n * sizeof(uint2), cudaMemcpyHostToDevice); if (e != cudaSuccess) { cudaFree(bl.dev); CU(e); } }
    s->block_lists.push_back(std::move(bl));
    *d_blocks = s->block_lists.back().dev; *n_blocks = (uint32_t)n;
    return TRB_OK;
}

trb_status resolve_samples(const trb_scene* s, const trb_render_cfg* cfg, uint32_t& spp, uint32_t& first, uint32_t& count) {
    if (cfg->spp > (1u << 31)) return fail(TRB_INVALID_ARG, "spp too large");
    spp = cfg->spp ? pow2_ceil(cfg->spp) : s->spp_pow2; // ld.rs:22-26
    first = cfg->sample_first;
    if (first > spp) return fail(TRB_INVALID_ARG, "sample_first exceeds spp");
    count = cfg->sample_count ? cfg->sample_count : spp - first;
    if ((uint64_t)first + count > spp) return fail(TRB_INVALID_ARG, "sample range exceeds spp");
    return TRB_OK;
}

// The instantiation of a kernel that traces through scene_trace for the scene's animation and mesh leaf form
template <int MODE>
auto simple_integrator_kernel(const trb_scene* s) {
    const bool anim = s->ds.has_anim != 0;
    if (s->wide_leaf) return anim ? trb::k_simple_integrator<MODE, true, true> : trb::k_simple_integrator<MODE, false, true>;
    return anim ? trb::k_simple_integrator<MODE, true> : trb::k_simple_integrator<MODE, false>;
}
template <bool STATS>
auto intersect_kernel(const trb_scene* s) {
    const bool anim = s->ds.has_anim != 0;
    if (s->wide_leaf) return anim ? trb::k_intersect<STATS, true, true> : trb::k_intersect<STATS, false, true>;
    return anim ? trb::k_intersect<STATS, true> : trb::k_intersect<STATS, false>;
}

template <bool STATS, int MODE, bool ANIM>
trb_status launch_render_t(trb_scene* s, const trb::RenderParams& rp, uint32_t flags, cudaStream_t st) {
    const int T = 9 + 2 * std::max(s->ds.fpw_x, s->ds.fpw_y);
    const size_t smem = (size_t)T * T * sizeof(float4);
    const auto kernel = s->wide_leaf ? trb::k_render<STATS, MODE, ANIM, true> : trb::k_render<STATS, MODE, ANIM>;
    int per_sm = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, trb::RENDER_THREADS, smem));
    const uint32_t grid = std::max(1u, std::min<uint32_t>(rp.n_blocks, (uint32_t)(std::max(1, per_sm) * s->sm_count)));
    kernel<<<grid, trb::RENDER_THREADS, smem, st>>>(s->ds, rp, flags);
    g_launches++;
    CU(cudaGetLastError());
    return TRB_OK;
}
// The AOVs a render asks for (DESIGN.md §4 "AOVs"): samples = the caller's device records (per-sample mode), else the film outputs
// (any may be nullptr); lum_w: the sample-variance film of the *_lum renders (include/trb.h "Sample variance"); motion_samples (the
// caller's device records, per-sample mode) or motion_w (the film) with dt: the motion vectors of the *_motion renders (include/trb.h
// "Motion vectors")
struct AovRequest {
    trb_aov_sample* samples; float4* albedo_w; float4* normal_w; unsigned long long* nearest; float4* lum_w = nullptr;
    trb_motion_sample* motion_samples = nullptr; float4* motion_w = nullptr; float dt = 0.0f;
};

// the path-indexed AOV records of film passes, at the path-state capacity
trb_status ensure_aov(trb_scene* s) {
    if (s->aov_capacity >= s->wf_capacity) return TRB_OK;
    CU(cudaDeviceSynchronize()); // a pass still in flight owns the old buffer
    if (s->d_aov) cudaFree(s->d_aov);
    s->d_aov = nullptr; s->aov_capacity = 0;
    const trb_status r = device_alloc(reinterpret_cast<void**>(&s->d_aov), s->wf_capacity * 2 * sizeof(float4), "AOV records");
    if (r != TRB_OK) return r;
    s->aov_capacity = s->wf_capacity;
    return TRB_OK;
}
// the path-indexed motion records of film passes, likewise; only the renders with a motion_w film allocate them
trb_status ensure_motion(trb_scene* s) {
    if (s->motion_capacity >= s->wf_capacity) return TRB_OK;
    CU(cudaDeviceSynchronize());
    if (s->d_motion) cudaFree(s->d_motion);
    s->d_motion = nullptr; s->motion_capacity = 0;
    const trb_status r = device_alloc(reinterpret_cast<void**>(&s->d_motion), s->wf_capacity * sizeof(float4), "motion records");
    if (r != TRB_OK) return r;
    s->motion_capacity = s->wf_capacity;
    return TRB_OK;
}

// The projection of the motion records at this frame (include/trb.h "Motion vectors"). An animated fov is sampled once per frame at
// the clamped mid-frame time, as trb_scene_update_frame samples it (camera.rs:134-141); at t + dt it is sampled at mid-frame + dt, so
// dt = 0 gives the frame's own fov and dt = -(one frame) the previous frame's.
float motion_tan(const trb_scene* s, float dt) {
    const trb_camera& c = s->cameras[s->active_camera];
    float fov = c.fov;
    if (c.n_fov_ctrl) {
        const float* kn = s->fov_floats.data() + c.fov_knot_first;
        const float lo = kn[c.fov_degree], hi = kn[c.n_fov_knots - 1 - c.fov_degree];
        float t = (s->last_start + s->last_end) / 2.0f + dt;
        t = t < lo ? lo : (t > hi ? hi : t);
        fov = trbh::spline_point_f32(c.fov_degree, s->fov_floats.data() + c.fov_ctrl_first, kn, c.n_fov_knots, t);
    }
    Mat4 px_to_cam; float scaling[3];
    trbh::camera_setup(fov, s->film.width, s->film.height, px_to_cam, scaling);
    return scaling[0];
}
trb::MotionCam motion_camera(const trb_scene* s, float dt) {
    trb::MotionCam mc{};
    std::memcpy(mc.cam_inv, s->cam_inv, 64);
    mc.tan_now = motion_tan(s, 0.0f);
    mc.tan_then = motion_tan(s, dt);
    mc.dt = dt;
    const float aspect = (float)s->film.width / (float)s->film.height; // camera_setup's screen window
    if (aspect > 1.0f) { mc.x0 = -aspect; mc.x1 = aspect; mc.y0 = -1.0f; mc.y1 = 1.0f; }
    else { mc.x0 = -1.0f; mc.x1 = 1.0f; mc.y0 = -1.0f / aspect; mc.y1 = 1.0f / aspect; }
    mc.w = (float)s->film.width; mc.h = (float)s->film.height;
    return mc;
}

trb_status ensure_wavefront(trb_scene* s, size_t n_paths) {
    if (n_paths <= s->wf_capacity) return TRB_OK;
    CU(cudaDeviceSynchronize()); // a pass still in flight owns the old buffers
    for (void* p : s->wf_allocs) cudaFree(p);
    s->wf_allocs.clear(); s->wf_capacity = 0;
    const size_t cap = n_paths;
    cudaError_t err = cudaSuccess;
    auto grab = [&](size_t bytes, void** out) {
        if (err != cudaSuccess) return;
        err = cudaMalloc(out, bytes);
        if (err == cudaSuccess) s->wf_allocs.push_back(*out);
    };
    trb::WfState& w = s->wf;
    float4** f4[] = {&w.org, &w.cont, &w.shadow, &w.mis, &w.a, &w.b, &w.tprev, &w.thr, &w.illum, &w.ng, &w.rad, &w.f_p, &w.f_n, &w.f_t, &w.f_b};
    for (float4** q : f4) grab(cap * sizeof(float4), reinterpret_cast<void**>(q));
    grab(cap * sizeof(uint4), reinterpret_cast<void**>(&w.hit));
    uint32_t** u1[] = {&w.q_active[0], &w.q_active[1], &w.q_ending[0], &w.q_ending[1], &w.q_cont, &w.q_shadow, &w.q_mis};
    for (uint32_t** q : u1) grab(cap * sizeof(uint32_t), reinterpret_cast<void**>(q));
    grab(cap * trb::WF_MID_BUCKETS * sizeof(uint32_t), reinterpret_cast<void**>(&w.q_mid)); // one list per material kind (split shading)
    grab(64 * trb::WF_CNT * sizeof(uint32_t), reinterpret_cast<void**>(&w.counters));
    // ray sorting: up to three rays per path and round; bins for the finest grid the options allow
    const size_t max_bins = (size_t)3 * (8u << (3 * trb::WF_SORT_MAX_BITS));
    uint32_t** u3[] = {&w.q_sorted, &w.sort_key, &w.sort_rank};
    for (uint32_t** q : u3) grab(3 * cap * sizeof(uint32_t), reinterpret_cast<void**>(q));
    grab(max_bins * sizeof(uint32_t), reinterpret_cast<void**>(&w.sort_hist));
    grab(max_bins * sizeof(uint32_t), reinterpret_cast<void**>(&w.sort_offs));
    grab(64 * 8 * sizeof(uint32_t), reinterpret_cast<void**>(&w.bounds));
    w.xf_tab = nullptr; w.n_anim = s->n_anim;
    if (s->n_anim) grab(cap * (size_t)s->n_anim * 32 * sizeof(float), reinterpret_cast<void**>(&w.xf_tab)); // per-path keyframed transforms (128 B per path and keyframed instance)
    if (err == cudaSuccess) err = cudaMemset(w.sort_hist, 0, max_bins * sizeof(uint32_t)); // invariant: all zero between sorts (the scan clears what it reads)
    if (err != cudaSuccess) {
        for (void* p : s->wf_allocs) cudaFree(p);
        s->wf_allocs.clear();
        return cuda_fail(err, "wavefront state");
    }
    s->wf_capacity = cap;
    return TRB_OK;
}

// AnimatedTransform::transform(ray.time) once per (path, keyframed instance) of a pass of n_paths paths whose times are in
// wf.thr[].w. Leaves wf.xf_tab == nullptr when there is no table (static scene, or option anim.table 0): the trace kernel then
// evaluates the transforms per instance test. adapt: an Adaptive pass, whose live path count the device holds.
void launch_anim_table(trb_scene* s, trb::WfState& wf, size_t n_paths, bool adapt, cudaStream_t st) {
    if (!(s->ds.has_anim && wf.xf_tab && s->tune.anim_table)) { wf.xf_tab = nullptr; return; }
    const size_t items = n_paths * wf.n_anim;
    const uint32_t nu = s->ds.n_uniq_splines;
    if (s->tune.anim_table >= 2 && nu > 0 && nu <= 256) { // each distinct keyframed spline once per path, in shared memory; then the stacks
        const uint32_t per_iter = std::max(1u, std::min(32u, 128u / nu));
        const size_t smem = (size_t)per_iter * nu * 32 * sizeof(float);
        const unsigned grid = (unsigned)std::min<size_t>((n_paths + per_iter - 1) / per_iter, (size_t)s->sm_count * 16);
        if (adapt) trb::k_wf_anim_table2<true><<<grid, 128, smem, st>>>(s->ds, wf, per_iter); // Adaptive: the pass's live paths
        else trb::k_wf_anim_table2<<<grid, 128, smem, st>>>(s->ds, wf, per_iter);
    } else {
        const unsigned grid = (unsigned)std::min<size_t>((items + 127) / 128, (size_t)s->sm_count * 16);
        if (adapt) trb::k_wf_anim_table<true><<<grid, 128, 0, st>>>(s->ds, wf);
        else trb::k_wf_anim_table<<<grid, 128, 0, st>>>(s->ds, wf);
    }
    g_launches++;
}

// The default trace variant (trace.pipe 36: box_hit_finite + RayHome) with PIPE bit 64: each ray's own [min_t, max_t] from the
// path state (k_query_load, k_illum_load). The ray queries' only trace, and round 0 of the illumination queries.
void launch_query_trace(trb_scene* s, const trb::RenderParams& rp, const trb::WfState& wf, uint32_t tflags, bool stats, const uint32_t* q_sorted,
                        cudaStream_t st) {
    const Tuning& tu = s->tune;
    const bool anim = s->ds.has_anim != 0;
    const unsigned resident = stats ? 4u : (anim ? 8u : 9u); // as for renders: two rounds of what is resident per SM
    const unsigned tgrid = (unsigned)s->sm_count * (tu.trace_grid ? tu.trace_grid : 2u * resident);
    const uint32_t sched = std::max(1u, tu.sched);
    if (s->wide_leaf) { // PIPE bit 128: wide mesh leaf references
        if (anim) {
            if (stats) trb::k_wf_trace<true, 4, 16, true, true, false, 225><<<tgrid, 128, 0, st>>>(s->ds, rp, wf, 0, tflags, tu.refill, sched, q_sorted);
            else trb::k_wf_trace<false, 8, 12, true, true, false, 225><<<tgrid, 128, 0, st>>>(s->ds, rp, wf, 0, tflags, tu.refill, sched, q_sorted);
        } else if (stats) trb::k_wf_trace<true, 4, 16, false, true, false, 225><<<tgrid, 128, 0, st>>>(s->ds, rp, wf, 0, tflags, tu.refill, sched, q_sorted);
        else trb::k_wf_trace<false, 9, 12, false, true, false, 225><<<tgrid, 128, 0, st>>>(s->ds, rp, wf, 0, tflags, tu.refill, sched, q_sorted);
    } else if (anim) {
        if (stats) trb::k_wf_trace<true, 4, 16, true, true, false, 97><<<tgrid, 128, 0, st>>>(s->ds, rp, wf, 0, tflags, tu.refill, sched, q_sorted);
        else trb::k_wf_trace<false, 8, 12, true, true, false, 97><<<tgrid, 128, 0, st>>>(s->ds, rp, wf, 0, tflags, tu.refill, sched, q_sorted);
    } else if (stats) trb::k_wf_trace<true, 4, 16, false, true, false, 97><<<tgrid, 128, 0, st>>>(s->ds, rp, wf, 0, tflags, tu.refill, sched, q_sorted);
    else trb::k_wf_trace<false, 9, 12, false, true, false, 97><<<tgrid, 128, 0, st>>>(s->ds, rp, wf, 0, tflags, tu.refill, sched, q_sorted);
}

// The shade kernels of one bounce round, chosen per scene (split or fused, material buckets). MODE 0: film, 1: parity records,
// 2: illumination queries. Counts the round's trace launch with its own.
template <int MODE>
void launch_shade(trb_scene* s, const trb::RenderParams& rp, const trb::WfState& wf, uint32_t round, cudaStream_t st) {
    const Tuning& tu = s->tune;
    const bool anim = s->ds.has_anim != 0;
    const unsigned shade_grid = (unsigned)s->sm_count * 4;
    // per scene (shade_split < 0): split when the scene mixes material kinds, and also when it is all matte — the matte instantiations of
    // _b / _c carry less code and fewer live values than the fused kernel; other one-kind scenes stay fused
    const bool split_auto = s->mixed_materials || (tu.shade_sort && tu.shade_kind && s->material_kinds == (1u << TRB_MAT_MATTE));
    if (tu.shade_split > 0 || (tu.shade_split < 0 && split_auto)) { // three kernels with fewer live values each (DESIGN.md "Split shading"); same device functions, same results
        // with the material buckets, _b and _c run once per kind that has an instantiation of its own (matte: the commonest), and once
        // for the other kinds the scene uses
        const uint32_t all = 0xffu, own = (tu.shade_sort && tu.shade_kind) ? (s->material_kinds & (1u << TRB_MAT_MATTE)) : 0u;
        const uint32_t rest = tu.shade_sort ? (s->material_kinds & ~own) : all;
        if (anim) {
            trb::k_wf_shade_a<MODE, true, 3><<<shade_grid, 128, 0, st>>>(s->ds, rp, wf, round);
            if (own) trb::k_wf_shade_b<true, 4, TRB_MAT_MATTE><<<shade_grid, 128, 0, st>>>(s->ds, rp, wf, round, own);
            if (rest) trb::k_wf_shade_b<true, 3><<<shade_grid, 128, 0, st>>>(s->ds, rp, wf, round, rest);
            if (own) trb::k_wf_shade_c<MODE, true, 6, TRB_MAT_MATTE><<<(unsigned)s->sm_count * 6, 128, 0, st>>>(s->ds, rp, wf, round, own);
            if (rest) trb::k_wf_shade_c<MODE, true, 4><<<shade_grid, 128, 0, st>>>(s->ds, rp, wf, round, rest);
        } else {
            const unsigned ga = (unsigned)s->sm_count * 6, gb = (unsigned)s->sm_count * 5, gc = (unsigned)s->sm_count * 6;
            trb::k_wf_shade_a<MODE, false, 6><<<ga, 128, 0, st>>>(s->ds, rp, wf, round);
            if (own) trb::k_wf_shade_b<false, 5, TRB_MAT_MATTE><<<gb, 128, 0, st>>>(s->ds, rp, wf, round, own);
            if (rest) trb::k_wf_shade_b<false, 5><<<gb, 128, 0, st>>>(s->ds, rp, wf, round, rest);
            if (own) trb::k_wf_shade_c<MODE, false, 6, TRB_MAT_MATTE><<<gc, 128, 0, st>>>(s->ds, rp, wf, round, own);
            if (rest) trb::k_wf_shade_c<MODE, false, 6><<<gc, 128, 0, st>>>(s->ds, rp, wf, round, rest);
        }
        g_launches += 4;
        return;
    }
    if (anim) { // keyframed variant: 168 registers at 3 CTAs per SM, or capped to 128 (some spills) at 4
        if constexpr (MODE == 1) trb::k_wf_shade<1, true, 3><<<shade_grid, 128, 0, st>>>(s->ds, rp, wf, round);
        else if constexpr (MODE == 2) trb::k_wf_shade<2, true, 4><<<shade_grid, 128, 0, st>>>(s->ds, rp, wf, round);
        else if (tu.shade_anim_occ >= 4) trb::k_wf_shade<0, true, 4><<<shade_grid, 128, 0, st>>>(s->ds, rp, wf, round);
        else trb::k_wf_shade<0, true, 3><<<shade_grid, 128, 0, st>>>(s->ds, rp, wf, round);
    } else trb::k_wf_shade<MODE, false, 4><<<shade_grid, 128, 0, st>>>(s->ds, rp, wf, round);
    g_launches += 2;
}

// The bounce rounds of a wavefront pass whose round-0 paths are in place (k_wf_generate or k_illum_load, then the transform
// table): per round the optional ray sort, the trace, the shade kernels (DESIGN.md "Execution shape"). mode as launch_shade; the
// illumination queries' round 0 traces each ray's own [min_t, max_t] (launch_query_trace).
trb_status wavefront_rounds(trb_scene* s, const trb::RenderParams& rp, const trb::WfState& wf, uint32_t flags, int mode, cudaStream_t st,
                            const AovRequest* aov = nullptr) {
    const Tuning& tu = s->tune;
    const bool stats = (flags & TRB_RENDER_STATS) != 0, anim = s->ds.has_anim != 0;
    const uint32_t rounds = s->integrator.max_depth + 2; // bounces 0..max_depth, plus the round that only resolves
    const int refill = tu.refill;
    // persistent CTAs: two rounds of what is resident per SM (9 for the default variant, 7 keyframed, 4 with counters) unless set
    const unsigned resident = (flags & TRB_RENDER_STATS) ? 4u : (tu.pipe == 0 || tu.pipe == 1 || tu.pipe == 33 ? 7u : (tu.pipe == 34 || tu.pipe == 35 || s->ds.has_anim ? 8u : 9u));
    const unsigned tgrid = (unsigned)s->sm_count * (tu.trace_grid ? tu.trace_grid : 2u * resident);
    const uint32_t sched = tu.sched;   // 0 = flat state machine; else the quorum of the phased loop (see k_wf_trace)
    const bool quads = tu.quads != 0;  // DQuad two-level records (never in the STATS variants: their counters are the reference's)
    const uint32_t tflags = flags | (tu.exact_box ? trb::WF_TRACE_FORCE_EXACT_BOX : 0u);
    // a scene with wide mesh leaves runs the default trace variant only: the option-selected experimental ones have no wide form
    if (s->wide_leaf && (sched == 0 || quads || tu.pipe == 0 || tu.pipe == 1 || (tu.pipe >= 33 && tu.pipe <= 35) || tu.pipe == 37))
        return fail(TRB_UNSUPPORTED, "trace.quads, trace.sched 0 and the experimental trace.pipe variants do not read wide mesh leaves (trace.wide_leaf)");
    if (quads && s->quads_dropped) return fail(TRB_UNSUPPORTED, "trace.quads reads DQuad records, which a mesh updated by trb_scene_update_mesh does not have");
    for (uint32_t round = 0; round < rounds; ++round) {
        const uint32_t* q_sorted = nullptr;
        if (tu.sort && (int)round >= tu.sort_min_round) { // counting sort of this round's rays by (type, octant, origin cell): DESIGN.md "Ray sorting"
            const uint32_t bits = (uint32_t)std::min(trb::WF_SORT_MAX_BITS, std::max(1, tu.sort_bits));
            const unsigned sgrid = (unsigned)s->sm_count * 8;
            trb::k_wf_sort_count<<<sgrid, 256, 0, st>>>(wf, round, bits, tu.sort == 2 ? 1u : 0u);
            trb::k_wf_sort_scan<<<1, 1024, 0, st>>>(wf, 3u * (8u << (3u * bits)));
            trb::k_wf_sort_scatter<<<sgrid, 256, 0, st>>>(wf, round);
            g_launches += 3;
            q_sorted = wf.q_sorted;
        }
        std::pair<cudaEvent_t, cudaEvent_t> ev{nullptr, nullptr};
        if (flags & TRB_RENDER_TIME_TRACE) {
            if (!s->event_pool.empty()) { ev = s->event_pool.back(); s->event_pool.pop_back(); }
            else { CU(cudaEventCreate(&ev.first)); CU(cudaEventCreate(&ev.second)); }
            CU(cudaEventRecord(ev.first, st));
        }
#define TRB_TRACE_LAUNCH(ST, MB, SS, AN, PH, QD, PIPE) trb::k_wf_trace<ST, MB, SS, AN, PH, QD, PIPE><<<tgrid, 128, 0, st>>>(s->ds, rp, wf, round, tflags, refill, sched, q_sorted)
        // PIPE 33 = box_hit_finite + RayHome + fused non-node chains (trb_kernels.cuh); tu.pipe picks the variant and how many
        // CTAs per SM it is compiled for: 36 (default) = 9 CTAs / 12 stack entries in shared memory. The STATS and keyframed
        // variants run the same code at their own occupancy, so the parity tests' counters cover it.
        const bool v2 = tu.pipe != 0;
        if (mode == 2 && round == 0) launch_query_trace(s, rp, wf, tflags, stats, q_sorted, st);
        else if (s->wide_leaf) { // the default variant and its STATS and keyframed forms with PIPE bit 128 (wide mesh leaf references)
            if (anim) { if (stats) TRB_TRACE_LAUNCH(true, 4, 16, true, true, false, 161); else TRB_TRACE_LAUNCH(false, 8, 12, true, true, false, 161); }
            else if (stats) TRB_TRACE_LAUNCH(true, 4, 16, false, true, false, 161);
            else TRB_TRACE_LAUNCH(false, 9, 12, false, true, false, 161);
        } else if (anim) {
            if (stats) { if (v2) TRB_TRACE_LAUNCH(true, 4, 16, true, true, false, 33); else TRB_TRACE_LAUNCH(true, 4, 16, true, true, false, 0); }
            else if (!v2) TRB_TRACE_LAUNCH(false, 7, 16, true, true, false, 0);
            else if (tu.pipe == 33) TRB_TRACE_LAUNCH(false, 7, 16, true, true, false, 33);
            else if (tu.pipe == 37) TRB_TRACE_LAUNCH(false, 9, 12, true, true, false, 33);
            else TRB_TRACE_LAUNCH(false, 8, 12, true, true, false, 33); // keyframed default: 8 CTAs per SM
        } else if (stats) {
            if (sched == 0) TRB_TRACE_LAUNCH(true, 4, 16, false, false, false, 0);
            else if (v2) TRB_TRACE_LAUNCH(true, 4, 16, false, true, false, 33); else TRB_TRACE_LAUNCH(true, 4, 16, false, true, false, 0);
        } else if (sched == 0) TRB_TRACE_LAUNCH(false, 7, 16, false, false, false, 0); // flat state machine (no phases)
        else if (quads) TRB_TRACE_LAUNCH(false, 7, 16, false, true, true, 0);
        else switch (tu.pipe) {
            case 0: TRB_TRACE_LAUNCH(false, 7, 16, false, true, false, 0); break;  // round-1 kernel
            case 1: TRB_TRACE_LAUNCH(false, 7, 16, false, true, false, 1); break;  // + box_hit_finite only
            case 33: TRB_TRACE_LAUNCH(false, 7, 16, false, true, false, 33); break;
            case 34: TRB_TRACE_LAUNCH(false, 8, 16, false, true, false, 33); break;
            case 35: TRB_TRACE_LAUNCH(false, 8, 12, false, true, false, 33); break;
            case 37: TRB_TRACE_LAUNCH(false, 9, 8, false, true, false, 33); break;
            default: TRB_TRACE_LAUNCH(false, 9, 12, false, true, false, 33); break; // 36
        }
#undef TRB_TRACE_LAUNCH
        if (ev.first) { CU(cudaEventRecord(ev.second, st)); s->trace_events.push_back(ev); }
        if (aov && round == 0) { // the primary hits, before the round-0 shade overwrites them
            const unsigned agrid = (unsigned)std::min<size_t>((wf.n_paths + 127) / 128, (size_t)s->sm_count * 16);
            float4* lo = mode == 1 ? reinterpret_cast<float4*>(aov->samples) : s->d_aov;
            float4* hi = mode == 1 ? lo + 1 : s->d_aov + s->aov_capacity;
            const uint32_t step = mode == 1 ? 2u : 1u;
            if (rp.ad_state) { // Adaptive pass (always mode 0): the paths the pass really holds
                if (anim) trb::k_wf_aov_ad<true><<<agrid, 128, 0, st>>>(s->ds, wf, lo, hi);
                else trb::k_wf_aov_ad<false><<<agrid, 128, 0, st>>>(s->ds, wf, lo, hi);
            } else if (anim) trb::k_wf_aov<true><<<agrid, 128, 0, st>>>(s->ds, wf, lo, hi, step);
            else trb::k_wf_aov<false><<<agrid, 128, 0, st>>>(s->ds, wf, lo, hi, step);
            g_launches++;
            if (aov->motion_samples || aov->motion_w) { // the motion records from the same primary hits
                const trb::MotionCam mc = motion_camera(s, aov->dt);
                float4* mo = mode == 1 ? reinterpret_cast<float4*>(aov->motion_samples) : s->d_motion;
                if (rp.ad_state) {
                    if (anim) trb::k_wf_motion_ad<true><<<agrid, 128, 0, st>>>(s->ds, wf, mc, mo);
                    else trb::k_wf_motion_ad<false><<<agrid, 128, 0, st>>>(s->ds, wf, mc, mo);
                } else if (anim) trb::k_wf_motion<true><<<agrid, 128, 0, st>>>(s->ds, wf, mc, mo);
                else trb::k_wf_motion<false><<<agrid, 128, 0, st>>>(s->ds, wf, mc, mo);
                g_launches++;
            }
        }
        if (mode == 0) launch_shade<0>(s, rp, wf, round, st);
        else if (mode == 1) launch_shade<1>(s, rp, wf, round, st);
        else launch_shade<2>(s, rp, wf, round, st);
    }
    CU(cudaGetLastError());
    return TRB_OK;
}

// One wavefront pass over rp's blocks x samples: generate, then (trace, shade) per bounce round, then the film
// (DESIGN.md "Execution shape"). n_paths = blocks * 64 * sample_count must fit the allocated path state.
trb_status launch_wavefront(trb_scene* s, const trb::RenderParams& rp, uint32_t flags, int mode, cudaStream_t st, const AovRequest* aov = nullptr) {
    const size_t n_paths = (size_t)rp.n_blocks * 64 * rp.sample_count;
    if (n_paths > s->wf_capacity || n_paths >= (1ull << 30)) return fail(TRB_INVALID_ARG, "pass larger than the wavefront state");
    const Tuning& tu = s->tune;
    trb::WfState wf = s->wf;
    wf.n_paths = (uint32_t)n_paths; // Adaptive passes: the worst case (the stride of the q_mid lists); their kernels read the live count on the device
    wf.mid_keyed = s->tune.shade_sort ? 1u : 0u;
    if (!tu.sort) wf.bounds = nullptr; // the origin boxes only size the ray sort's grid: no box updates when sorting is off
    if (s->integrator.type != TRB_INTEGRATOR_PATH) { // Whitted / NormalsDebug: one thread per camera sample, then the same film kernel
        const unsigned grid = (unsigned)std::min<size_t>((n_paths + 127) / 128, (size_t)s->sm_count * 8);
        const auto kernel = mode == 0 ? simple_integrator_kernel<0>(s) : simple_integrator_kernel<1>(s);
        kernel<<<grid, 128, 0, st>>>(s->ds, rp, wf.rad, wf.n_paths, s->integrator.type, flags, nullptr);
        g_launches++;
        if (mode == 0) {
            const int T = 9 + 2 * std::max(s->ds.fpw_x, s->ds.fpw_y);
            const unsigned film_grid = std::min<unsigned>(rp.n_blocks, (unsigned)s->sm_count * 8);
            if (tu.film_v2) trb::k_wf_film_v2<<<film_grid, trb::RENDER_THREADS, (size_t)4 * T * T * sizeof(float4), st>>>(s->ds, rp, wf);
            else trb::k_wf_film<<<film_grid, trb::RENDER_THREADS, (size_t)T * T * sizeof(float4), st>>>(s->ds, rp, wf);
            g_launches++;
        }
        CU(cudaGetLastError());
        return TRB_OK;
    }
    CU(cudaMemsetAsync(wf.counters, 0, 64 * trb::WF_CNT * sizeof(uint32_t), st));
    const unsigned gen_grid = (unsigned)std::min<size_t>((n_paths + 255) / 256, (size_t)s->sm_count * 8);
    const bool anim = s->ds.has_anim != 0; // static scenes run kernels with no animation code in them at all
    if (rp.ad_state) { // Adaptive sampler round: only the pixels still sampling queue their paths
        if (anim) trb::k_wf_generate_ad<true><<<gen_grid, 256, 0, st>>>(s->ds, rp, wf);
        else trb::k_wf_generate_ad<false><<<gen_grid, 256, 0, st>>>(s->ds, rp, wf);
    } else if (anim) trb::k_wf_generate<true><<<gen_grid, 256, 0, st>>>(s->ds, rp, wf);
    else trb::k_wf_generate<false><<<gen_grid, 256, 0, st>>>(s->ds, rp, wf);
    g_launches++;
    launch_anim_table(s, wf, n_paths, rp.ad_state != nullptr, st);
    const trb_status r = wavefront_rounds(s, rp, wf, flags, mode, st, aov);
    if (r != TRB_OK) return r;
    if (mode == 0 && rp.film) { // (an Adaptive parity dump has no film: its records are written by k_ad_decide)
        const int T = 9 + 2 * std::max(s->ds.fpw_x, s->ds.fpw_y);
        const unsigned film_grid = std::min<unsigned>(rp.n_blocks, (unsigned)s->sm_count * 8);
        if (rp.ad_state) {
            if (tu.film_v2) trb::k_wf_film_v2<true><<<film_grid, trb::RENDER_THREADS, (size_t)4 * T * T * sizeof(float4), st>>>(s->ds, rp, wf);
            else trb::k_wf_film<true><<<film_grid, trb::RENDER_THREADS, (size_t)T * T * sizeof(float4), st>>>(s->ds, rp, wf);
        } else if (tu.film_v2) trb::k_wf_film_v2<<<film_grid, trb::RENDER_THREADS, (size_t)4 * T * T * sizeof(float4), st>>>(s->ds, rp, wf);
        else trb::k_wf_film<<<film_grid, trb::RENDER_THREADS, (size_t)T * T * sizeof(float4), st>>>(s->ds, rp, wf);
        g_launches++;
        if (aov) { // the colour film's kernel over each half of the AOV records in place of the radiance: the same weights and order
            trb::RenderParams ra = rp;
            trb::WfState wa = wf;
            const std::pair<float4*, float4*> films[2] = {{aov->albedo_w, s->d_aov}, {aov->normal_w, s->d_aov + s->aov_capacity}};
            for (const auto& f : films) {
                if (!f.first) continue;
                ra.film = f.first; wa.rad = f.second;
                if (rp.ad_state) { // Adaptive: the live blocks and the pixels that sampled this round, as for the colour film
                    if (tu.film_v2) trb::k_wf_film_v2<true><<<film_grid, trb::RENDER_THREADS, (size_t)4 * T * T * sizeof(float4), st>>>(s->ds, ra, wa);
                    else trb::k_wf_film<true><<<film_grid, trb::RENDER_THREADS, (size_t)T * T * sizeof(float4), st>>>(s->ds, ra, wa);
                } else if (tu.film_v2) trb::k_wf_film_v2<<<film_grid, trb::RENDER_THREADS, (size_t)4 * T * T * sizeof(float4), st>>>(s->ds, ra, wa);
                else trb::k_wf_film<<<film_grid, trb::RENDER_THREADS, (size_t)T * T * sizeof(float4), st>>>(s->ds, ra, wa);
                g_launches++;
            }
            if (aov->lum_w) { // the colour film's kernel once more, over the radiance and the records' albedo half together
                ra.film = aov->lum_w;
                if (rp.ad_state) {
                    if (tu.film_v2) trb::k_wf_film_v2<true, true><<<film_grid, trb::RENDER_THREADS, (size_t)4 * T * T * sizeof(float4), st>>>(s->ds, ra, wf, s->d_aov);
                    else trb::k_wf_film<true, true><<<film_grid, trb::RENDER_THREADS, (size_t)T * T * sizeof(float4), st>>>(s->ds, ra, wf, s->d_aov);
                } else if (tu.film_v2) trb::k_wf_film_v2<false, true><<<film_grid, trb::RENDER_THREADS, (size_t)4 * T * T * sizeof(float4), st>>>(s->ds, ra, wf, s->d_aov);
                else trb::k_wf_film<false, true><<<film_grid, trb::RENDER_THREADS, (size_t)T * T * sizeof(float4), st>>>(s->ds, ra, wf, s->d_aov);
                g_launches++;
            }
            if (aov->motion_w) { // the colour film's kernel over the motion records, which are (v dx, v dy, v, 0) already
                ra.film = aov->motion_w; wa.rad = s->d_motion;
                if (rp.ad_state) {
                    if (tu.film_v2) trb::k_wf_film_v2<true><<<film_grid, trb::RENDER_THREADS, (size_t)4 * T * T * sizeof(float4), st>>>(s->ds, ra, wa);
                    else trb::k_wf_film<true><<<film_grid, trb::RENDER_THREADS, (size_t)T * T * sizeof(float4), st>>>(s->ds, ra, wa);
                } else if (tu.film_v2) trb::k_wf_film_v2<<<film_grid, trb::RENDER_THREADS, (size_t)4 * T * T * sizeof(float4), st>>>(s->ds, ra, wa);
                else trb::k_wf_film<<<film_grid, trb::RENDER_THREADS, (size_t)T * T * sizeof(float4), st>>>(s->ds, ra, wa);
                g_launches++;
            }
            if (aov->nearest) {
                const unsigned ngrid = (unsigned)std::min<size_t>((n_paths + 255) / 256, (size_t)s->sm_count * 8);
                if (rp.ad_state) trb::k_wf_nearest_ad<<<ngrid, 256, 0, st>>>(s->ds, rp, s->d_aov, s->d_aov + s->aov_capacity, aov->nearest);
                else trb::k_wf_nearest<<<ngrid, 256, 0, st>>>(s->ds, rp, s->d_aov, s->d_aov + s->aov_capacity, (uint32_t)n_paths, aov->nearest);
                g_launches++;
            }
        }
    }
    CU(cudaGetLastError());
    return TRB_OK;
}

// Exec::render renders every selected block at the full spp in one call (multithreaded.rs:55-114). The wavefront keeps
// 212 B of path state per camera sample in HBM, so a frame is cut into additive passes of at most `pass_paths` camera
// samples (fewer if device memory is short): all selected blocks x a sample sub-range, or — for images with more than
// pass_paths / 64 blocks — a block sub-range x one sample. A camera sample's radiance is a pure function of
// (scene, seed, pixel, sample index), so the split changes nothing but the order of the film's float additions.
trb_status render_passes(trb_scene* s, trb::RenderParams rp, uint32_t flags, int mode, cudaStream_t st, const AovRequest* aov = nullptr) {
    const uint32_t nb = rp.n_blocks, first = rp.sample_first, count = rp.sample_count;
    const uint2* blocks = rp.blocks;
    const uint64_t total = (uint64_t)nb * 64 * count;
    uint64_t want = std::min<uint64_t>(total, std::min<uint64_t>(std::max<uint64_t>(s->tune.pass_paths, 64), (1ull << 30) - 64));
    if (mode == 1) { // per-sample records are indexed by the path number of ONE pass
        if (total >= (1ull << 30)) return fail(TRB_INVALID_ARG, "sample buffer too large: blocks*64*sample_count must be < 2^30; select fewer blocks or samples");
        want = total;
    }
    want = ((want + 63) / 64) * 64;
    if (want > s->wf_capacity) {
        trb_status r;
        while ((r = ensure_wavefront(s, (size_t)want)) == TRB_OOM && want > (1u << 16) && mode == 0) want = ((want / 2 + 63) / 64) * 64;
        if (r != TRB_OK) return r;
    }
    if (aov && mode == 0) {
        trb_status r = ensure_aov(s);
        if (r == TRB_OK && aov->motion_w) r = ensure_motion(s);
        if (r != TRB_OK) return r;
    }
    const uint64_t cap = std::max<uint64_t>(want, 64);  // paths per pass actually used (a larger state left by an earlier call is not required)
    uint32_t bp, sp;
    if ((uint64_t)nb * 64 <= cap) { bp = nb; sp = (uint32_t)std::min<uint64_t>(count, cap / ((uint64_t)nb * 64)); }
    else { bp = (uint32_t)(cap / 64); sp = 1; }
    for (uint32_t b0 = 0; b0 < nb; b0 += bp)
        for (uint32_t s0 = 0; s0 < count; s0 += sp) {
            rp.blocks = blocks + b0; rp.n_blocks = std::min(bp, nb - b0);
            rp.sample_first = first + s0; rp.sample_count = std::min(sp, count - s0);
            trb_status r = launch_wavefront(s, rp, flags, mode, st, aov);
            if (r != TRB_OK) return r;
        }
    return TRB_OK;
}

// ---- Adaptive sampler (DESIGN.md §2 "Adaptive sampler", §5) ----------------------------------------------------------
trb_status adaptive_check(const trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, trbh::AdSchedule& sch) {
    if (cfg->spp || cfg->sample_first || cfg->sample_count)
        return fail(TRB_INVALID_ARG, "the Adaptive sampler owns the sample schedule: spp, sample_first and sample_count must be 0");
    if (!trbh::ad_schedule(ad->min_spp, ad->max_spp, sch))
        return fail(TRB_INVALID_ARG, "Adaptive sampler: max_spp < min_spp after rounding up to powers of two (the reference panics), or more than 2^24");
    if (s->integrator.type != TRB_INTEGRATOR_PATH) return fail(TRB_UNSUPPORTED, "the Adaptive sampler is built for the path integrator only");
    if (cfg->flags & TRB_RENDER_MEGAKERNEL) return fail(TRB_UNSUPPORTED, "the Adaptive sampler runs on the wavefront pipeline only");
    return TRB_OK;
}

trb_status ensure_adaptive(trb_scene* s) {
    if (s->d_ad_state) return TRB_OK;
    const size_t npx = (size_t)s->film.width * s->film.height, nblk = npx / 64;
    CU(cudaMalloc(reinterpret_cast<void**>(&s->d_ad_state), npx * sizeof(uint4)));
    for (int k = 0; k < 2; ++k) {
        CU(cudaMalloc(reinterpret_cast<void**>(&s->d_ad_list[k]), std::max<size_t>(1, nblk) * sizeof(uint2)));
        CU(cudaMalloc(reinterpret_cast<void**>(&s->d_ad_index[k]), std::max<size_t>(1, nblk) * sizeof(uint32_t)));
    }
    CU(cudaMalloc(reinterpret_cast<void**>(&s->d_ad_flags), std::max<size_t>(1, nblk) * sizeof(uint32_t)));
    CU(cudaMemset(s->d_ad_flags, 0, std::max<size_t>(1, nblk) * sizeof(uint32_t)));
    CU(cudaMalloc(reinterpret_cast<void**>(&s->d_ad_count), 2 * sizeof(uint32_t))); // live length of each block list
    CU(cudaMalloc(reinterpret_cast<void**>(&s->d_ad_spp), npx * sizeof(uint32_t)));
    return TRB_OK;
}

// thread_work with the Adaptive sampler over the selected blocks: round 0 over all of them, round k over the blocks that still
// have a pixel sampling, each round cut into passes of whole blocks (a pass holds all of a pixel's samples of the round, so
// k_ad_decide sees them together). rp carries the film or the parity records, stats, seed. Enqueued on st with no host
// synchronisation: the host cannot know how many blocks a round keeps, so it enqueues every round of the schedule with the
// passes the whole selection would need, and each pass clamps itself to the round's live block count, which k_ad_init /
// k_ad_compact keep on the device (DESIGN.md §5 "Adaptive rounds"). Afterwards d_spp[y * width + x] holds the sample count
// of each selected pixel (d_spp: width*height u32, or nullptr). aov (nullptr: none): the AOV films of rp's film, or with
// rp.film == nullptr the AOV records in samples_out's slot layout (DESIGN.md §4 "Adaptive AOVs").
trb_status render_adaptive_rounds(trb_scene* s, const trbh::AdSchedule& sch, trb::RenderParams rp, const uint2* d_blocks, uint32_t nb, uint32_t flags,
                                  cudaStream_t st, uint32_t* d_spp, const AovRequest* aov = nullptr) {
    trb_status r = ensure_adaptive(s);
    if (r != TRB_OK) return r;
    const uint64_t per_block = (uint64_t)64 * std::max(sch.min, sch.step); // paths of one block in the largest round
    if (per_block >= (1ull << 30)) return fail(TRB_INVALID_ARG, "Adaptive sampler: one block of one round exceeds 2^30 paths");
    uint64_t want = std::min<uint64_t>((uint64_t)nb * per_block, std::min<uint64_t>(std::max<uint64_t>(s->tune.pass_paths, 64), (1ull << 30) - 64));
    want = ((std::max(want, per_block) + 63) / 64) * 64;
    if (want > s->wf_capacity) {
        while ((r = ensure_wavefront(s, (size_t)want)) == TRB_OOM && want / 2 >= per_block && want > (1u << 16)) want = ((want / 2 + 63) / 64) * 64;
        if (r != TRB_OK) return r;
    }
    if (aov && (r = ensure_aov(s)) != TRB_OK) return r;
    if (aov && aov->motion_w && (r = ensure_motion(s)) != TRB_OK) return r;
    const uint64_t cap = want;
    rp.ad_state = s->d_ad_state;
    rp.ad_min = sch.min; rp.ad_max = sch.max; rp.ad_step = sch.step; rp.ad_max_per_pixel = sch.max_per_pixel;
    rp.spp = sch.max; rp.ad_time_len = sch.max;
    const unsigned init_grid = (unsigned)std::min<size_t>(((size_t)nb * 64 + 255) / 256, (size_t)s->sm_count * 8);
    trb::k_ad_init<<<std::max(1u, init_grid), 256, 0, st>>>(s->ds, d_blocks, nb, s->d_ad_state, s->d_ad_list[0], s->d_ad_index[0], s->d_ad_count);
    g_launches++;
    for (uint32_t round = 0; round < sch.rounds; ++round) {
        const int cur = round & 1; // round r reads list r % 2 and (compaction) writes the other one
        const uint32_t count = trbh::ad_count(sch, round);
        rp.ad_round = round; rp.sample_first = trbh::ad_slot_base(sch, round); rp.sample_count = count;
        rp.ld_offset = trbh::ad_offset(sch, round); rp.ad_pos_len = count;
        rp.ad_live = s->d_ad_count + cur;
        const uint32_t bp = (uint32_t)std::max<uint64_t>(1, cap / ((uint64_t)64 * count));
        for (uint32_t b0 = 0; b0 < nb; b0 += bp) { // worst case: the whole selection is still live; passes past the live count exit at once
            rp.blocks = s->d_ad_list[cur] + b0; rp.n_blocks = std::min(bp, nb - b0); rp.ad_block_index = s->d_ad_index[cur] + b0; rp.ad_b0 = b0;
            r = launch_wavefront(s, rp, flags, 0, st, aov);
            if (r != TRB_OK) return r;
            const unsigned dgrid = (unsigned)std::min<size_t>(((size_t)rp.n_blocks * 64 + 127) / 128, (size_t)s->sm_count * 16);
            if (aov && aov->samples) {
                trb::k_ad_aov_slots<<<dgrid, 128, 0, st>>>(s->ds, rp, s->d_aov, s->d_aov + s->aov_capacity, aov->samples);
                g_launches++;
            }
            trb::k_ad_decide<<<dgrid, 128, 0, st>>>(s->ds, rp, s->wf, s->d_ad_flags + b0);
            g_launches++;
        }
        if (round + 1 == sch.rounds) break;
        trb::k_ad_compact<<<1, 1024, 0, st>>>(s->d_ad_flags, s->d_ad_count + cur, s->d_ad_list[cur], s->d_ad_index[cur], s->d_ad_list[cur ^ 1],
                                              s->d_ad_index[cur ^ 1], s->d_ad_count + (cur ^ 1));
        g_launches++;
    }
    if (d_spp) {
        const unsigned sgrid = (unsigned)std::min<size_t>(((size_t)nb * 64 + 255) / 256, (size_t)s->sm_count * 8);
        trb::k_ad_pixel_spp<<<std::max(1u, sgrid), 256, 0, st>>>(s->ds, d_blocks, nb, s->d_ad_state, d_spp);
        g_launches++;
    }
    CU(cudaGetLastError());
    return TRB_OK;
}

// the selection's host block list (bx, by pairs) of a device list made by ensure_blocks
const std::vector<uint32_t>* host_blocks(const trb_scene* s, const uint2* d_blocks) {
    for (const BlockList& b : s->block_lists) if (b.dev == d_blocks) return &b.host;
    return nullptr;
}
// d_ad_spp (image layout, written by k_ad_pixel_spp) -> pixel_spp[y * width + x] for the selected pixels only
trb_status adaptive_pixel_spp_out(trb_scene* s, const uint2* d_blocks, uint32_t nb, uint32_t* pixel_spp) {
    if (!pixel_spp || nb == 0) return TRB_OK;
    const std::vector<uint32_t>* hb = host_blocks(s, d_blocks);
    if (!hb) return fail(TRB_CUDA, "block list not found");
    std::vector<uint32_t> v((size_t)s->film.width * s->film.height);
    CU(cudaMemcpy(v.data(), s->d_ad_spp, v.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    for (uint32_t b = 0; b < nb; ++b)
        for (uint32_t k = 0; k < 64; ++k) {
            const size_t pixel = ((*hb)[2 * b + 1] * 8 + k / 8) * (size_t)s->film.width + (*hb)[2 * b] * 8 + k % 8;
            pixel_spp[pixel] = v[pixel];
        }
    return TRB_OK;
}

trb_status launch_render(trb_scene* s, const trb::RenderParams& rp, uint32_t flags, int mode, cudaStream_t st, const AovRequest* aov = nullptr) {
    if (!(flags & TRB_RENDER_MEGAKERNEL) || s->integrator.type != TRB_INTEGRATOR_PATH) return render_passes(s, rp, flags, mode, st, aov);
    const bool stats = (flags & TRB_RENDER_STATS) != 0;
    CU(cudaMemsetAsync(rp.work_counter, 0, sizeof(uint32_t), st));
    if (s->ds.has_anim) {
        if (mode == 0) return stats ? launch_render_t<true, 0, true>(s, rp, flags, st) : launch_render_t<false, 0, true>(s, rp, flags, st);
        return stats ? launch_render_t<true, 1, true>(s, rp, flags, st) : launch_render_t<false, 1, true>(s, rp, flags, st);
    }
    if (mode == 0) return stats ? launch_render_t<true, 0, false>(s, rp, flags, st) : launch_render_t<false, 0, false>(s, rp, flags, st);
    return stats ? launch_render_t<true, 1, false>(s, rp, flags, st) : launch_render_t<false, 1, false>(s, rp, flags, st);
}

void stats_out(const trb::DStats& d, trb_stats* o) {
    o->camera_samples = d.camera_samples; o->rays_primary = d.rays_primary; o->rays_shadow = d.rays_shadow; o->rays_mis = d.rays_mis;
    o->rays_continuation = d.rays_continuation; o->node_tests = d.node_tests; o->tri_tests = d.tri_tests; o->inst_tests = d.inst_tests;
}

// A host form's trb_stats (none when stats is null): the scene's counters, the kernel time between its events and update_ms
trb_status stats_readback(trb_scene* s, trb_stats* stats, float update_ms) {
    if (!stats) return TRB_OK;
    trb::DStats h;
    CU(cudaMemcpy(&h, s->d_stats, sizeof h, cudaMemcpyDeviceToHost));
    std::memset(stats, 0, sizeof *stats);
    stats_out(h, stats);
    CU(cudaEventElapsedTime(&stats->kernel_ms, s->ev0, s->ev1));
    stats->update_ms = update_ms;
    return TRB_OK;
}

trb_status check_error_flag(trb_scene* s) {
    int e = 0;
    CU(cudaMemcpy(&e, s->d_error, sizeof e, cudaMemcpyDeviceToHost));
    if (e) { CU(cudaMemset(s->d_error, 0, sizeof(int))); return fail(TRB_CUDA, "BVH traversal stack overflow (depth > 64; the reference would panic)"); }
    return TRB_OK;
}

// run_staged for the host forms that report counters (trb_intersect, the ray and illumination queries, the sample renders): the
// scene's counters cleared and its events recorded around enqueue, then the traversal error flag checked
template <class Enqueue>
trb_status run_counted(trb_scene* s, std::initializer_list<Span> ins, std::initializer_list<OutSpan> outs, Enqueue enqueue) {
    const trb_status r = run_staged(ins, outs, [&](const DeviceBuffer* d) {
        CU(cudaMemsetAsync(s->d_stats, 0, sizeof(trb::DStats), 0));
        CU(cudaEventRecord(s->ev0, 0));
        const trb_status q = enqueue(d);
        if (q == TRB_OK) CU(cudaEventRecord(s->ev1, 0));
        return q;
    });
    return r != TRB_OK ? r : check_error_flag(s);
}

// ---- ray queries (trb_intersect_records / trb_occluded; DESIGN.md §5 "Ray queries") ---------------------------------------
// Argument checks shared by the four entry points. `allowed`: the flag bits the query accepts; device buffers are read and
// written with 16-byte accesses (`out16`: the output buffer too).
trb_status query_check(const trb_scene* s, size_t n, const void* rays, const void* out, uint32_t flags, uint32_t allowed, bool device, bool out16) {
    if (!s || (n && (!rays || !out))) return fail(TRB_INVALID_ARG, "null argument");
    if (flags & ~allowed) return fail(TRB_INVALID_ARG, "unsupported flag bits for a ray query");
    if (device && n) { const trb_status r = check_aligned({{rays, 16}, {out, out16 ? 16 : 1}}, "device query buffers must be 16-byte aligned"); if (r != TRB_OK) return r; }
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering"); // scene.rs:179
    return TRB_OK;
}

// Enqueue the queries on st in passes of at most pass.paths rays (the path state grows as for renders, halving on OOM). Each pass:
// k_query_load -> keyframed transform table -> k_wf_trace (default variant, PIPE bit 64) -> k_query_records (d_out) or
// k_query_occluded (d_occ). The rays of a pass are round 0 of a wavefront: continuation rays for records, shadow rays for occlusion.
trb_status query_passes(trb_scene* s, size_t n, const trb_query_ray* d_rays, trb_intersection* d_out, uint8_t* d_occ, uint32_t flags,
                        trb::DStats* d_stats, cudaStream_t st) {
    uint64_t want = std::min<uint64_t>(n, std::min<uint64_t>(std::max<uint64_t>(s->tune.pass_paths, 64), (1ull << 30) - 64));
    want = ((want + 63) / 64) * 64;
    if (want > s->wf_capacity) {
        trb_status r;
        while ((r = ensure_wavefront(s, (size_t)want)) == TRB_OOM && want > (1u << 16)) want = ((want / 2 + 63) / 64) * 64;
        if (r != TRB_OK) return r;
    }
    const Tuning& tu = s->tune;
    const bool stats = (flags & TRB_RENDER_STATS) != 0, anim = s->ds.has_anim != 0, occl = d_occ != nullptr;
    trb::RenderParams rp{};
    rp.stats = d_stats; rp.error_flag = s->d_error;
    const uint32_t tflags = (flags & TRB_RENDER_REFERENCE_SHADOW) | (tu.exact_box ? trb::WF_TRACE_FORCE_EXACT_BOX : 0u);
    for (size_t b = 0; b < n; b += want) {
        const size_t m = std::min<size_t>(want, n - b);
        trb::WfState wf = s->wf;
        wf.n_paths = (uint32_t)m;
        const unsigned lgrid = (unsigned)std::min<size_t>((m + 255) / 256, (size_t)s->sm_count * 8);
        if (occl) trb::k_query_load<true><<<lgrid, 256, 0, st>>>(wf, d_rays + b);
        else trb::k_query_load<false><<<lgrid, 256, 0, st>>>(wf, d_rays + b);
        g_launches++;
        launch_anim_table(s, wf, m, false, st);
        launch_query_trace(s, rp, wf, tflags, stats, nullptr, st);
        g_launches++;
        if (occl) trb::k_query_occluded<<<lgrid, 256, 0, st>>>(wf, d_occ + b);
        else {
            const unsigned rgrid = (unsigned)std::min<size_t>((m + 127) / 128, (size_t)s->sm_count * 16);
            if (anim) trb::k_query_records<true><<<rgrid, 128, 0, st>>>(s->ds, wf, d_out + b);
            else trb::k_query_records<false><<<rgrid, 128, 0, st>>>(s->ds, wf, d_out + b);
        }
        g_launches++;
    }
    CU(cudaGetLastError());
    return TRB_OK;
}

// Enqueue the illumination queries on st (DESIGN.md §5 "Illumination queries"). A pass holds whole rays, floor(pass paths / spp) of
// them, so that k_illum_reduce finds all of a ray's samples in the pass; the path state grows as for renders, halving on OOM.
// Path integrator: k_illum_load -> keyframed transform table -> the render's bounce rounds (wavefront_rounds, mode 2). Whitted
// and NormalsDebug: k_simple_integrator<2> reads the caller's rays itself. Then k_illum_reduce writes each ray's mean.
trb_status illum_passes(trb_scene* s, size_t n, const trb_illum_ray* d_rays, uint32_t spp, uint32_t seed, float* d_rgb, uint32_t flags,
                        trb::DStats* d_stats, cudaStream_t st) {
    uint64_t want = std::min<uint64_t>((uint64_t)n * spp, std::min<uint64_t>(std::max<uint64_t>(s->tune.pass_paths, 64), (1ull << 30) - 64));
    want = ((std::max<uint64_t>(want, spp) + 63) / 64) * 64;
    if (want > s->wf_capacity) {
        trb_status r;
        while ((r = ensure_wavefront(s, (size_t)want)) == TRB_OOM && want / 2 >= spp && want > (1u << 16)) want = ((want / 2 + 63) / 64) * 64;
        if (r != TRB_OK) return r;
    }
    const size_t per = (size_t)(want / spp); // rays per pass
    const bool anim = s->ds.has_anim != 0;
    trb::RenderParams rp{}; // LD offset 0; no blocks: the MODE 2 kernels never call sample_id
    rp.stats = d_stats; rp.error_flag = s->d_error; rp.seed = seed; rp.spp = spp;
    for (size_t b = 0; b < n; b += per) {
        const size_t m = std::min(per, n - b);
        trb::WfState wf = s->wf;
        wf.n_paths = (uint32_t)(m * spp);
        wf.mid_keyed = s->tune.shade_sort ? 1u : 0u;
        if (!s->tune.sort) wf.bounds = nullptr; // as launch_wavefront
        if (s->integrator.type != TRB_INTEGRATOR_PATH) {
            const unsigned grid = (unsigned)std::min<size_t>((wf.n_paths + 127) / 128, (size_t)s->sm_count * 8);
            simple_integrator_kernel<2>(s)<<<grid, 128, 0, st>>>(s->ds, rp, wf.rad, wf.n_paths, s->integrator.type, flags, d_rays + b);
            g_launches++;
        } else {
            CU(cudaMemsetAsync(wf.counters, 0, 64 * trb::WF_CNT * sizeof(uint32_t), st));
            const unsigned lgrid = (unsigned)std::min<size_t>((wf.n_paths + 255) / 256, (size_t)s->sm_count * 8);
            trb::k_illum_load<<<lgrid, 256, 0, st>>>(wf, d_rays + b, spp, seed, d_stats);
            g_launches++;
            launch_anim_table(s, wf, wf.n_paths, false, st);
            const trb_status r = wavefront_rounds(s, rp, wf, flags, 2, st);
            if (r != TRB_OK) return r;
        }
        const unsigned rgrid = (unsigned)std::min<size_t>((m + 127) / 128, (size_t)s->sm_count * 16);
        trb::k_illum_reduce<<<rgrid, 128, 0, st>>>(wf.rad, (uint32_t)m, spp, (flags & TRB_QUERY_CLAMP) ? 1u : 0u, d_rgb + 3 * b);
        g_launches++;
    }
    CU(cudaGetLastError());
    return TRB_OK;
}

trb_status illum_check(const trb_scene* s, size_t n, const void* rays, uint32_t spp, const void* rgb, uint32_t flags, bool device) {
    if (spp == 0 || spp > 65536) return fail(TRB_INVALID_ARG, "spp must be in [1, 65536]");
    if (device && n) { const trb_status r = check_aligned({{rgb, 4}}, "the device rgb buffer must be 4-byte aligned"); if (r != TRB_OK) return r; }
    return query_check(s, n, rays, rgb, flags, TRB_RENDER_STATS | TRB_RENDER_REFERENCE_SHADOW | TRB_QUERY_CLAMP, device, false);
}

// The host form of a ray or illumination query: the rays staged, enqueue(d_rays, d_out) counted (run_counted), the results and the
// counters read back; no rays leave zero counters
template <class Enqueue>
trb_status run_query(trb_scene* s, size_t n, Span rays, OutSpan out, trb_stats* stats, Enqueue enqueue) {
    if (n == 0) { if (stats) std::memset(stats, 0, sizeof *stats); return TRB_OK; }
    CU(cudaSetDevice(s->device));
    const trb_status r = run_counted(s, {rays}, {out}, [&](const DeviceBuffer* d) { return enqueue(d[0].p, d[1].p); });
    return r != TRB_OK ? r : stats_readback(s, stats, 0.f);
}

// The static part of the device instance records (everything but the matrices, which update_frame writes); keyframed / animated flags
// are scene properties. anim_list: the keyframed instances. Returns whether any instance's transform or emission depends on time.
bool static_instance_records(const trb_scene* s, std::vector<trb::DInstance>& di, std::vector<uint32_t>& anim_list) {
    const size_t n = s->instances.size();
    bool any_anim = false;
    di.assign(n, trb::DInstance{});
    anim_list.clear();
    for (size_t i = 0; i < n; ++i) {
        const trb_instance& in = s->instances[i];
        trb::DInstance& o = di[i];
        std::memset(&o, 0, sizeof o);
        o.kind = in.kind; o.shape = in.shape; o.p0 = in.p0; o.p1 = in.p1; o.mesh = in.mesh; o.material = in.material;
        o.xf_first = in.spline_first; o.xf_count = in.n_splines;
        if (!trbh::xf_is_static(s->splines.data(), in.spline_first, in.n_splines)) {
            o.flags |= trb::DI_ANIM_XF; o.spline_first = in.spline_first; o.n_splines = in.n_splines; any_anim = true;
            o.anim_slot = (uint32_t)anim_list.size(); anim_list.push_back((uint32_t)i);
        }
        if (in.kind != TRB_INST_RECEIVER) {
            for (int k = 0; k < 3; ++k) o.emission[k] = s->color_keys[in.emission_first].rgba[k];
            if (in.n_emission > 1) { o.flags |= trb::DI_ANIM_EMISSION; o.emission_first = in.emission_first; o.n_emission = in.n_emission; any_anim = true; }
        }
    }
    return any_anim;
}

// The device record of a material: what Material::bsdf recomputes per hit from constant textures, precomputed
trb::DMaterial device_material(const trb_material& m) {
    trb::DMaterial o;
    std::memset(&o, 0, sizeof o);
    o.type = m.type;
    for (int k = 0; k < 3; ++k) { o.c0[k] = m.c0[k]; o.c1[k] = m.c1[k]; }
    o.roughness = m.roughness; o.eta = m.eta;
    o.width = fmaxf(m.roughness, 0.000001f);         // Beckmann::new (beckmann.rs:19-22)
    float sigma = kPi / 180.0f * m.roughness;        // OrenNayar::new (oren_nayar.rs:26-34), roughness in degrees
    sigma *= sigma;
    o.on_a = 1.0f - 0.5f * sigma / (sigma + 0.33f);
    o.on_b = 0.45f * sigma / (sigma + 0.09f);
    o.merl_off = m.type == TRB_MAT_MERL ? m.merl * TRB_MERL_TABLE_FLOATS : 0;
    for (int k = 0; k < 4; ++k) o.tex[k] = m.tex[k];
    return o;
}

// The material kinds of the hittable instances, which choose the shading kernels (launch_shade)
void material_shape(trb_scene* s) {
    uint32_t kinds = 0;
    for (const trb_instance& in : s->instances) if (in.kind != TRB_INST_EMITTER_POINT && in.material < s->materials.size()) kinds |= 1u << s->materials[in.material].type;
    // two kinds are enough: with the material buckets the split kernels run one kind's code at a time, the fused kernel runs every
    // kind a warp holds
    s->mixed_materials = __builtin_popcount(kinds) >= 2 || (kinds & (1u << TRB_MAT_MERL)) != 0;
    s->material_kinds = kinds;
}

// DScene::level_xf of spline k: Keyframe::transform of a one-control-point level (identity, unused, for keyframed splines)
Xf level_transform(const trb_scene* s, size_t k) {
    return s->splines[k].n_ctrl == 1 ? keyframe_xf(s->keyframes[s->splines[k].ctrl_first]) : xf_identity();
}

// Distinct keyframed splines by content (degree, knots, control keyframes compared bit for bit): uniq_of per spline (0xffffffff for
// one-control-point levels), uniq_list a representative spline of each (DScene::spline_uniq, uniq_splines)
void spline_dedup(const trb_scene* s, std::vector<uint32_t>& uniq_of, std::vector<uint32_t>& uniq_list) {
    uniq_of.assign(s->splines.size(), 0xffffffffu);
    uniq_list.clear();
    auto same = [&](const trb_spline& a, const trb_spline& b) {
        return a.degree == b.degree && a.n_ctrl == b.n_ctrl && a.n_knots == b.n_knots &&
               memcmp(&s->keyframes[a.ctrl_first], &s->keyframes[b.ctrl_first], a.n_ctrl * sizeof(trb_keyframe)) == 0 &&
               memcmp(&s->knots[a.knot_first], &s->knots[b.knot_first], a.n_knots * sizeof(float)) == 0;
    };
    for (size_t k = 0; k < s->splines.size(); ++k) {
        if (s->splines[k].n_ctrl <= 1) continue;
        for (size_t u = 0; u < uniq_list.size() && uniq_of[k] == 0xffffffffu; ++u)
            if (same(s->splines[k], s->splines[uniq_list[u]])) uniq_of[k] = (uint32_t)u;
        if (uniq_of[k] == 0xffffffffu) { uniq_of[k] = (uint32_t)uniq_list.size(); uniq_list.push_back((uint32_t)k); }
    }
}

// ---- shading queries (trb_bsdf_eval / trb_bsdf_sample / trb_light_sample / trb_light_pdf / trb_emitted; DESIGN.md §5) ------------------
// Argument checks: `a` and `b` are the input buffers (the light and emission queries have one and pass it twice), read with 16-byte
// loads on the device; `out_align` is the device output's required alignment. `frame`: the query reads the instance matrices.
trb_status shade_check(const trb_scene* s, size_t n, const void* a, const void* b, const void* out, uintptr_t out_align, bool device, bool frame) {
    if (!s || (n && (!a || !b || !out))) return fail(TRB_INVALID_ARG, "null argument");
    if (device && n) {
        const trb_status r = check_aligned({{a, 16}, {b, 16}, {out, out_align}}, out_align == 16 ? "device query buffers must be 16-byte aligned"
                                                                                                 : "device query buffers must be 16-byte aligned, the float output 4-byte aligned");
        if (r != TRB_OK) return r;
    }
    if (frame && !s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering"); // scene.rs:179
    return TRB_OK;
}

// One thread per query, grid-stride: at most 16 CTAs of 128 threads per SM
inline unsigned shade_grid(const trb_scene* s, size_t n) { return (unsigned)std::min<size_t>((n + 127) / 128, (size_t)s->sm_count * 16); }

trb_status launch_bsdf_eval(trb_scene* s, size_t n, const trb_intersection* d_rec, const trb_bsdf_eval_query* d_q, float* d_out, cudaStream_t st) {
    trb::k_bsdf_eval<<<shade_grid(s, n), 128, 0, st>>>(s->ds, (uint32_t)s->materials.size(), n, d_rec, d_q, reinterpret_cast<float4*>(d_out));
    g_launches++;
    CU(cudaGetLastError());
    return TRB_OK;
}
trb_status launch_bsdf_sample(trb_scene* s, size_t n, const trb_intersection* d_rec, const trb_bsdf_sample_query* d_q, trb_bsdf_sample_result* d_out,
                              cudaStream_t st) {
    trb::k_bsdf_sample<<<shade_grid(s, n), 128, 0, st>>>(s->ds, (uint32_t)s->materials.size(), n, d_rec, d_q, d_out);
    g_launches++;
    CU(cudaGetLastError());
    return TRB_OK;
}
trb_status launch_light_sample(trb_scene* s, size_t n, const trb_light_query* d_q, trb_light_sample_result* d_out, cudaStream_t st) {
    if (s->ds.has_anim) trb::k_light_sample<true><<<shade_grid(s, n), 128, 0, st>>>(s->ds, n, d_q, d_out);
    else trb::k_light_sample<false><<<shade_grid(s, n), 128, 0, st>>>(s->ds, n, d_q, d_out);
    g_launches++;
    CU(cudaGetLastError());
    return TRB_OK;
}
trb_status launch_light_pdf(trb_scene* s, size_t n, const trb_light_pdf_query* d_q, float* d_pdf, cudaStream_t st) {
    if (s->ds.has_anim) trb::k_light_pdf<true><<<shade_grid(s, n), 128, 0, st>>>(s->ds, n, d_q, d_pdf);
    else trb::k_light_pdf<false><<<shade_grid(s, n), 128, 0, st>>>(s->ds, n, d_q, d_pdf);
    g_launches++;
    CU(cudaGetLastError());
    return TRB_OK;
}
trb_status launch_emitted(trb_scene* s, size_t n, const trb_emit_query* d_q, float* d_rgb, cudaStream_t st) {
    if (s->ds.has_anim || s->anim_emission) trb::k_emitted<true><<<shade_grid(s, n), 128, 0, st>>>(s->ds, n, d_q, d_rgb);
    else trb::k_emitted<false><<<shade_grid(s, n), 128, 0, st>>>(s->ds, n, d_q, d_rgb);
    g_launches++;
    CU(cudaGetLastError());
    return TRB_OK;
}

// ---- caller film writes (trb_film_write / trb_film_write_device; DESIGN.md §5) --------------------------------------------------
// Argument checks, before anything is read: n < 2^32 (the sort and the region starts index with 32 bits), buffers present when
// n > 0, device buffers 4-byte aligned.
trb_status film_check(const trb_scene* s, size_t n, const void* samples, const void* regions, const void* film, bool device) {
    if (!s) return fail(TRB_INVALID_ARG, "null argument");
    if ((uint64_t)n >= (1ull << 32)) return fail(TRB_INVALID_ARG, "film writes take fewer than 2^32 samples");
    if (n && (!samples || !regions || !film)) return fail(TRB_INVALID_ARG, "null argument");
    if (device && n) return check_aligned({{samples, 4}, {regions, 4}, {film, 4}}, "device film-write buffers must be 4-byte aligned");
    return TRB_OK;
}

// Enqueue one film write on `st`: keys, a stable radix sort of the sample order by region (CUB; its kernels are not counted in
// g_launches), region starts, the gather. The scratch space is per scene and only grows; growing it drains the device once. There
// is no splitting into passes: a split would change the order of the additions, so a write that does not fit is TRB_OOM.
trb_status film_write_enqueue(trb_scene* s, uint32_t n, const trb_sample* d_samples, const uint32_t* d_regions, float* d_film, cudaStream_t st) {
    const uint32_t nr = (s->film.width / 8) * (s->film.height / 8);
    const int bits = 32 - __builtin_clz(nr); // keys are 0 .. nr (nr = out of range)
    size_t temp = 0;
    cub::DoubleBuffer<uint32_t> keys(nullptr, nullptr), order(nullptr, nullptr);
    CU(cub::DeviceRadixSort::SortPairs(nullptr, temp, keys, order, n, 0, bits, st));
    const size_t a = ((size_t)n * 4 + 255) / 256 * 256, sb = ((size_t)(nr + 1) * 4 + 255) / 256 * 256;
    const size_t need = 4 * a + sb + temp;
    if (need > s->film_scratch_bytes) {
        CU(cudaDeviceSynchronize()); // a write still in flight owns the old scratch
        cudaFree(s->d_film_scratch);
        s->d_film_scratch = nullptr; s->film_scratch_bytes = 0;
        const trb_status r = device_alloc(&s->d_film_scratch, need, "film write scratch");
        if (r != TRB_OK) return r;
        s->film_scratch_bytes = need;
    }
    char* base = static_cast<char*>(s->d_film_scratch);
    uint32_t* k0 = reinterpret_cast<uint32_t*>(base);
    uint32_t* o0 = reinterpret_cast<uint32_t*>(base + 2 * a);
    keys = cub::DoubleBuffer<uint32_t>(k0, reinterpret_cast<uint32_t*>(base + a));
    order = cub::DoubleBuffer<uint32_t>(o0, reinterpret_cast<uint32_t*>(base + 3 * a));
    uint32_t* d_start = reinterpret_cast<uint32_t*>(base + 4 * a);
    trb::k_film_keys<<<(unsigned)std::min<size_t>(((size_t)n + 255) / 256, (size_t)s->sm_count * 8), 256, 0, st>>>(n, d_regions, nr, k0, o0);
    g_launches++;
    CU(cudaGetLastError());
    CU(cub::DeviceRadixSort::SortPairs(base + 4 * a + sb, temp, keys, order, n, 0, bits, st));
    trb::k_film_starts<<<(nr + 1 + 255) / 256, 256, 0, st>>>(n, keys.Current(), nr, d_start);
    g_launches++;
    CU(cudaGetLastError());
    trb::k_film_gather<<<nr, trb::FILM_WRITE_THREADS, 0, st>>>(s->ds, d_samples, order.Current(), d_start, d_film);
    g_launches++;
    CU(cudaGetLastError());
    return TRB_OK;
}

// k_camera_rays over the selection of cfg into device buffers of n = blocks * 64 * sample_count records, enqueued on st
trb_status camera_rays_enqueue(trb_scene* s, const trb_render_cfg* cfg, size_t n, trb_ray* d_rays, float* d_xy, cudaStream_t st) {
    uint32_t spp, first, count, nb;
    const uint2* d_blocks = nullptr;
    trb_status r = resolve_samples(s, cfg, spp, first, count);
    if (r != TRB_OK) return r;
    r = ensure_blocks(s, cfg, &d_blocks, &nb);
    if (r != TRB_OK) return r;
    if (n != (size_t)nb * 64 * count) return fail(TRB_INVALID_ARG, "ray buffer size must be blocks*64*sample_count");
    if (n == 0) return TRB_OK;
    trb::RenderParams rp{};
    rp.blocks = d_blocks; rp.n_blocks = nb; rp.spp = spp; rp.sample_first = first; rp.sample_count = count; rp.seed = cfg->seed;
    const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)s->sm_count * 8);
    if (s->ds.has_anim) trb::k_camera_rays<true><<<grid, 256, 0, st>>>(s->ds, rp, d_rays, d_xy);
    else trb::k_camera_rays<false><<<grid, 256, 0, st>>>(s->ds, rp, d_rays, d_xy);
    g_launches++;
    CU(cudaGetLastError());
    return TRB_OK;
}

// One mesh's DPair records in one leaf form, narrow or wide (trb_device.h), packed from its host tree into its record buffer, and
// the root reference into its header (dh.root_lo)
trb_status pack_mesh_nodes(const HostMesh& hm, trb::DBvh& dh, bool wide) {
    std::vector<trb::DPair> pn;
    trb::DBvh hdr{};
    if (!pack_pairs(hm.nodes, pn, hdr, wide))
        return fail(TRB_UNSUPPORTED, wide ? "mesh too large for the wide leaf encoding (2^30 triangles)" : "mesh too large for the leaf encoding (2^25 triangles)");
    if (!pn.empty()) CU(cudaMemcpy(const_cast<trb::DPair*>(dh.pairs), pn.data(), pn.size() * sizeof(trb::DPair), cudaMemcpyHostToDevice));
    dh.root_lo = hdr.root_lo;
    return TRB_OK;
}

// The boxes of a refit mesh's host tree, read back from its device records (either leaf form: only the boxes are read). Record k
// belongs to the k-th interior node in preorder and holds the boxes of its two children; the root box is hm.bounds.
trb_status refresh_host_tree(HostMesh& hm, const trb::DMesh& dm) {
    if (!hm.stale) return TRB_OK;
    std::vector<trb::DPair> pn((hm.nodes.size() - 1) / 2); // a binary tree of n nodes has (n - 1) / 2 interior ones
    if (!pn.empty()) CU(cudaMemcpy(pn.data(), dm.bvh.pairs, pn.size() * sizeof(trb::DPair), cudaMemcpyDeviceToHost));
    auto set = [](trb_bvh_node& n, const float4& lo, const float4& hi) {
        n.bmin[0] = lo.x; n.bmin[1] = lo.y; n.bmin[2] = lo.z; n.bmax[0] = hi.x; n.bmax[1] = hi.y; n.bmax[2] = hi.z;
    };
    set(hm.nodes[0], make_float4(hm.bounds.lo[0], hm.bounds.lo[1], hm.bounds.lo[2], 0.f), make_float4(hm.bounds.hi[0], hm.bounds.hi[1], hm.bounds.hi[2], 0.f));
    size_t k = 0;
    for (size_t i = 0; i < hm.nodes.size(); ++i) {
        if (hm.nodes[i].b & TRB_BVH_LEAF) continue;
        const trb::DPair& p = pn[k++];
        set(hm.nodes[i + 1], p.l_lo, p.l_hi);
        set(hm.nodes[hm.nodes[i].a], p.r_lo, p.r_hi);
    }
    hm.stale = false;
    return TRB_OK;
}

// Packs every mesh's DPair records in one leaf form into the buffers allocated when the mesh was set up (setup_mesh), and uploads
// the mesh headers. Kernels still in flight may read the records, so the device is drained first.
trb_status upload_mesh_nodes(trb_scene* s, bool wide) {
    CU(cudaDeviceSynchronize());
    for (size_t mi = 0; mi < s->meshes.size(); ++mi) {
        { const trb_status r = refresh_host_tree(s->meshes[mi], s->dmeshes[mi]); if (r != TRB_OK) return r; }
        const trb_status r = pack_mesh_nodes(s->meshes[mi], s->dmeshes[mi].bvh, wide);
        if (r != TRB_OK) return r;
    }
    if (!s->dmeshes.empty()) CU(cudaMemcpy(s->d_meshes, s->dmeshes.data(), s->dmeshes.size() * sizeof(trb::DMesh), cudaMemcpyHostToDevice));
    s->wide_leaf = wide;
    return TRB_OK;
}

// BVH<Triangle> of one uploaded mesh (max_geom 16, mesh.rs:44) into hm.nodes / hm.order, and its leaf-ordered triangle records with
// their leaf-end marks into dtris. The triangle boxes are computed on the device. The SAH build runs on the device, or on the host
// (BvhBuilder over the boxes read back) when `on_device` is off or its scratch does not fit in free device memory, which keeps the
// largest meshes loadable. Every scratch buffer is freed before returning, except that with `keep` the device-built node array is
// handed to the caller (keep stays empty after a host build). `ev_built` / `ev_read` (optional) are recorded on the default stream
// once the tree is built and once it has been read back to the host (a host build records both after building).
trb_status build_mesh_bvh(bool on_device, const float* dp, const uint32_t* di, uint32_t n, HostMesh& hm, trb::DTri* dtris,
                          DeviceBuffer* keep = nullptr, cudaEvent_t ev_built = nullptr, cudaEvent_t ev_read = nullptr) {
    DeviceBuffer boxes, order, nodes; // order: + one word, the node count
    bool built = false;               // nodes holds the device-built tree
    const auto grid = [](size_t k) { return (unsigned)((k + 255) / 256); };
    trb_status r;
    if ((r = boxes.alloc(24 * (size_t)n, "mesh BVH scratch")) != TRB_OK || (r = order.alloc(4 * ((size_t)n + 1), "mesh BVH scratch")) != TRB_OK) return r;
    float* d_boxes = boxes.as<float>();
    uint32_t* d_order = order.as<uint32_t>();
    trb::bvhb::k_tri_boxes<<<grid(n), 256>>>(dp, di, n, d_boxes);
    ++g_launches;
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    const size_t need = trb::bvhb::build_scratch_bytes(n) + (2 * (size_t)n - 1) * sizeof(trb_bvh_node) + ((size_t)64 << 20);
    if (on_device && need <= free_b) {
        if ((r = nodes.alloc((2 * (size_t)n - 1) * sizeof(trb_bvh_node), "mesh BVH scratch")) != TRB_OK) return r;
        bool empty = false;
        CU(trb::bvhb::build_device(d_boxes, n, 16, d_order + n, nodes.as<trb_bvh_node>(), d_order, 0, &g_launches, &empty));
        if (empty) return fail(TRB_INVALID_ARG, "mesh triangles with infinite coordinates: the SAH build would split a node into an empty child");
        built = true;
        if (ev_built) CU(cudaEventRecord(ev_built, 0));
        uint32_t nn = 0;
        CU(cudaMemcpy(&nn, d_order + n, 4, cudaMemcpyDeviceToHost));
        hm.nodes.resize(nn);
        hm.order.resize(n);
        CU(cudaMemcpy(hm.nodes.data(), nodes.p, (size_t)nn * sizeof(trb_bvh_node), cudaMemcpyDeviceToHost));
        CU(cudaMemcpy(hm.order.data(), d_order, 4 * (size_t)n, cudaMemcpyDeviceToHost));
        if (ev_read) CU(cudaEventRecord(ev_read, 0));
    } else {
        {
            std::vector<Box3> tb(n);
            CU(cudaMemcpy(tb.data(), d_boxes, 24 * (size_t)n, cudaMemcpyDeviceToHost));
            BvhBuilder bb;
            bb.build(tb, 16);
            hm.nodes = std::move(bb.nodes); hm.order = std::move(bb.order);
        }
        if (ev_built) CU(cudaEventRecord(ev_built, 0));
        if (ev_read) CU(cudaEventRecord(ev_read, 0));
        CU(cudaMemcpy(d_order, hm.order.data(), 4 * (size_t)n, cudaMemcpyHostToDevice));
    }
    CU(boxes.reset());
    trb::bvhb::k_tri_pack<<<grid(n), 256>>>(dp, di, d_order, n, dtris);
    ++g_launches;
    if (!built) { // host build: the marks are set from the host tree, a chunk of nodes at a time
        const size_t chunk = std::min<size_t>(hm.nodes.size(), (size_t)1 << 22);
        if ((r = nodes.alloc(chunk * sizeof(trb_bvh_node), "mesh BVH scratch")) != TRB_OK) return r;
        for (size_t i = 0; i < hm.nodes.size(); i += chunk) {
            const size_t k = std::min(chunk, hm.nodes.size() - i);
            CU(cudaMemcpy(nodes.p, hm.nodes.data() + i, k * sizeof(trb_bvh_node), cudaMemcpyHostToDevice));
            trb::bvhb::k_tri_leaf_marks<<<grid(k), 256>>>(nodes.as<trb_bvh_node>(), (uint32_t)k, dtris);
            ++g_launches;
        }
    } else {
        trb::bvhb::k_tri_leaf_marks<<<grid(hm.nodes.size()), 256>>>(nodes.as<trb_bvh_node>(), (uint32_t)hm.nodes.size(), dtris);
        ++g_launches;
    }
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize());
    if (keep && built) std::swap(keep->p, nodes.p);
    return TRB_OK;
}

// DPair records of a device-built mesh tree (d_nodes, n nodes) in one leaf form, with pack_pairs' layout, on the default stream.
// The interior nodes are ranked first (an exclusive scan of their flags); `records(n_rec, &out)` then supplies room for the n_rec
// records. *fits_narrow: whether every leaf fits the narrow reference. Scratch is freed before returning.
template <class Records>
trb_status pack_pairs_device(const trb_bvh_node* d_nodes, uint32_t n, bool wide, Records records, bool* fits_narrow) {
    DeviceBuffer rec, scan; // rec: n + 1 ranks, then the narrow-misfit word
    const auto grid = [](size_t k) { return (unsigned)((k + 255) / 256); };
    size_t cub_bytes = 0;
    CU(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)n + 1));
    trb_status r;
    if ((r = rec.alloc(4 * ((size_t)n + 2), "node record scratch")) != TRB_OK || (r = scan.alloc(std::max<size_t>(1, cub_bytes), "node record scratch")) != TRB_OK)
        return r;
    uint32_t* d_rec = rec.as<uint32_t>();
    CU(cudaMemset(d_rec + n + 1, 0, 4));
    trb::bvhb::k_pair_flags<<<grid((size_t)n + 1), 256>>>(d_nodes, n, d_rec);
    ++g_launches;
    CU(cub::DeviceScan::ExclusiveSum(scan.p, cub_bytes, d_rec, d_rec, (int)n + 1));
    uint32_t n_rec = 0;
    CU(cudaMemcpy(&n_rec, d_rec + n, 4, cudaMemcpyDeviceToHost));
    trb::DPair* out = nullptr;
    if ((r = records(n_rec, &out)) != TRB_OK) return r;
    trb::bvhb::k_pair_pack<<<grid(n), 256>>>(d_nodes, n, d_rec, wide, out, d_rec + n + 1);
    ++g_launches;
    CU(cudaGetLastError());
    uint32_t bad = 0;
    CU(cudaMemcpy(&bad, d_rec + n + 1, 4, cudaMemcpyDeviceToHost));
    *fits_narrow = bad == 0;
    return TRB_OK;
}

// One mesh of a description into fresh buffers of `arena` (trb_scene_create, trb_scene_replace_meshes), checked by validate_mesh: the
// four arrays uploaded or, with `device`, copied from the caller's device arrays on `st` and the indices checked there
// (k_mesh_index_check, flag read before anything else is built); BVH<Triangle> with max_geom 16 (mesh.rs:44) and the leaf-ordered
// triangle records (build_mesh_bvh); the bounds; DQuad records (trace.quads) where every leaf fits the narrow reference; and room
// for one DPair record per interior node (both leaf forms have one), which pack_mesh_nodes fills in the scene's form.
trb_status setup_mesh(trb_scene* s, DeviceArena& arena, const trb_mesh& m, bool device, cudaStream_t st, HostMesh& hm, trb::DMesh& dm) {
    hm.n_verts = m.n_verts;
    float *dp, *dn, *dt; uint32_t* di; trb::DPair* dnodes; trb::DTri* dtris;
    const size_t nv = m.n_verts, ni = 3 * (size_t)m.n_tris;
    if (!device) {
        CU(arena.upload(m.positions, 3 * nv, &dp));
        CU(arena.upload(m.normals, 3 * nv, &dn));
        CU(arena.upload(m.texcoords, 2 * nv, &dt));
        CU(arena.upload(m.indices, ni, &di));
    } else {
        CU(arena.alloc(3 * nv, &dp)); CU(arena.alloc(3 * nv, &dn)); CU(arena.alloc(2 * nv, &dt)); CU(arena.alloc(ni, &di));
        uint32_t* d_bad = nullptr;
        CU(arena.alloc(1, &d_bad));
        CU(cudaMemcpyAsync(dp, m.positions, 3 * nv * sizeof(float), cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(dn, m.normals, 3 * nv * sizeof(float), cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(dt, m.texcoords, 2 * nv * sizeof(float), cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(di, m.indices, ni * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
        CU(cudaMemsetAsync(d_bad, 0, sizeof(uint32_t), st));
        const unsigned blocks = (unsigned)std::max<size_t>(1, std::min<size_t>((ni / 4 + 255) / 256, (size_t)s->sm_count * 8));
        trb::bvhb::k_mesh_index_check<<<blocks, 256, 0, st>>>(di, ni, m.n_verts, d_bad);
        ++g_launches;
        CU(cudaGetLastError());
        uint32_t bad = 0;
        CU(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        arena.release(d_bad);
        if (bad) return fail(TRB_INVALID_ARG, "mesh index out of range");
    }
    CU(arena.alloc(m.n_tris, &dtris));
    { const trb_status r = build_mesh_bvh(s->tune.build_device != 0, dp, di, m.n_tris, hm, dtris); if (r != TRB_OK) return r; }
    for (int k = 0; k < 3; ++k) { hm.bounds.lo[k] = hm.nodes[0].bmin[k]; hm.bounds.hi[k] = hm.nodes[0].bmax[k]; }
    size_t n_rec = 0;
    for (const trb_bvh_node& n : hm.nodes) if (!(n.b & TRB_BVH_LEAF)) ++n_rec;
    trb::DBvh& hdr = dm.bvh;
    hdr.quads = nullptr;
    hdr.root_hi = make_float4(hm.bounds.hi[0], hm.bounds.hi[1], hm.bounds.hi[2], bits_f(QUAD_EMPTY_HOST));
    hm.narrow = leaves_fit_narrow(hm.nodes);
    if (hm.narrow) { // DQuad records (trace.quads) hold narrow leaves only: a mesh that needs the wide form skips them
        std::vector<trb::DQuad> qn;
        uint32_t qroot = 0;
        if (!pack_quads(hm.nodes, qn, qroot)) return fail(TRB_UNSUPPORTED, "mesh too large for the leaf encoding (2^25 triangles)");
        hdr.root_hi.w = bits_f(qroot);
        trb::DQuad* dquads;
        CU(arena.upload(qn.data(), qn.size(), &dquads));
        hdr.quads = dquads;
    }
    CU(arena.alloc(n_rec, &dnodes));
    hm.pair_cap = n_rec;
    hdr.pairs = dnodes;
    dm.positions = dp; dm.normals = dn; dm.texcoords = dt; dm.indices = di; dm.tris = dtris;
    dm.n_nodes = (uint32_t)hm.nodes.size(); dm.n_tris = m.n_tris;
    return TRB_OK;
}

// n floats of a caller's array into a mesh buffer: from host memory, or from device memory read on `st` (complete on return)
cudaError_t mesh_copy_in(const float* dst, const float* src, size_t n, bool device, cudaStream_t st) {
    if (!device) return cudaMemcpy(const_cast<float*>(dst), src, n * sizeof(float), cudaMemcpyHostToDevice);
    const cudaError_t e = cudaMemcpyAsync(const_cast<float*>(dst), src, n * sizeof(float), cudaMemcpyDeviceToDevice, st);
    return e != cudaSuccess ? e : cudaStreamSynchronize(st);
}
// The attribute half of trb_scene_update_mesh and trb_scene_refit_mesh: normals and / or texcoords copied in place. The caller has
// drained the device.
trb_status copy_mesh_attributes(trb_scene* s, uint32_t mi, const float* nrm, const float* uv, bool device, cudaStream_t st) {
    const trb::DMesh& dm = s->dmeshes[mi];
    const size_t nv = s->meshes[mi].n_verts;
    if (nrm) CU(mesh_copy_in(dm.normals, nrm, 3 * nv, device, st));
    if (uv) CU(mesh_copy_in(dm.texcoords, uv, 2 * nv, device, st));
    return TRB_OK;
}

// trb_scene_update_mesh(_device): `device` says the caller's arrays are device memory, read on `st`. New positions are copied
// into a fresh buffer and the tree and triangle records are built into fresh buffers, so a failed build or allocation leaves the
// scene as it was; the live buffers are replaced only after the build succeeded and the device was drained. The node records are
// written into the live record buffer when the new tree fits it, so a CUDA error from the packing on (a device fault, not a
// property of the input) may leave the scene half updated. TRB_MESH_UPDATE_TIME=1 prints the phases, timed with CUDA events on the
// default stream (every phase ends at a synchronisation point, so they are also wall time), to stderr: build, read-back (the tree to
// the host), triangle records (k_tri_pack, k_tri_leaf_marks), pack (node records), frame refresh.
trb_status update_mesh(trb_scene* s, uint32_t mi, const float* pos, const float* nrm, const float* uv, bool device, cudaStream_t st) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    if (mi >= s->meshes.size()) return fail(TRB_INVALID_ARG, "mesh index out of range");
    if (!pos && !nrm && !uv) return TRB_OK;
    CU(cudaSetDevice(s->device));
    HostMesh& hm = s->meshes[mi];
    trb::DMesh& dm = s->dmeshes[mi];
    const size_t nv = hm.n_verts;
    auto copy_in = [&](const float* dst, const float* src, size_t n) { return mesh_copy_in(dst, src, n, device, st); };
    struct PhaseEvents {
        cudaEvent_t e[6] = {};
        ~PhaseEvents() { for (cudaEvent_t x : e) if (x) cudaEventDestroy(x); }
    } ev;
    const bool timing = pos && getenv("TRB_MESH_UPDATE_TIME") != nullptr;
    if (timing) for (cudaEvent_t& x : ev.e) CU(cudaEventCreate(&x));
    auto mark = [&](int k) { if (timing) cudaEventRecord(ev.e[k], 0); };
    auto report = [&]() {
        if (!timing) return;
        mark(5);
        cudaEventSynchronize(ev.e[5]);
        static const char* const phase[5] = {"build", "read-back", "triangle records", "pack", "frame refresh"};
        for (int k = 0; k < 5; ++k) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, ev.e[k], ev.e[k + 1]);
            fprintf(stderr, "trb_scene_update_mesh %s %.3f ms\n", phase[k], ms);
        }
    };
    if (pos) {
        float* d_pos = nullptr;
        trb::DTri* d_tris = nullptr;
        DeviceBuffer d_nodes; // the device-built tree (empty after a host build)
        HostMesh nm;
        auto build = [&]() -> trb_status {
            CU(s->arena.alloc(3 * nv, &d_pos));
            CU(s->arena.alloc(dm.n_tris, &d_tris));
            mark(0);
            CU(copy_in(d_pos, pos, 3 * nv));
            return build_mesh_bvh(s->tune.build_device != 0, d_pos, dm.indices, dm.n_tris, nm, d_tris, &d_nodes, ev.e[1], ev.e[2]);
        };
        { const trb_status r = build(); if (r != TRB_OK) { s->arena.release(d_pos); s->arena.release(d_tris); return r; } }
        mark(3);
        // the device is drained (build_mesh_bvh ends with a device synchronisation): nothing in flight reads what is replaced below
        trb::DPair* pairs = const_cast<trb::DPair*>(dm.bvh.pairs);
        size_t cap = hm.pair_cap;
        auto records = [&](uint32_t n_rec, trb::DPair** out) -> trb_status {
            if (n_rec > cap) { // the new tree has more interior nodes than the buffer holds: a larger one replaces it at the commit
                trb::DPair* grown = nullptr;
                CU(s->arena.alloc(n_rec, &grown));
                pairs = grown; cap = n_rec;
            }
            *out = pairs;
            return TRB_OK;
        };
        bool narrow = true;
        trb_status r = TRB_OK;
        if (d_nodes.p) {
            r = pack_pairs_device(d_nodes.as<trb_bvh_node>(), (uint32_t)nm.nodes.size(), s->wide_leaf, records, &narrow);
            d_nodes.reset();
        } else { // host build: the records are packed on the host, as at creation. A tree that does not fit the scene's narrow form is
                 // packed wide (the form changes below and every mesh is re-packed): either way the buffer is sized for its interior nodes
            narrow = leaves_fit_narrow(nm.nodes);
            std::vector<trb::DPair> pn;
            trb::DBvh hdr{};
            pack_pairs(nm.nodes, pn, hdr, s->wide_leaf || !narrow);
            trb::DPair* out = nullptr;
            r = records((uint32_t)pn.size(), &out);
            if (r == TRB_OK && !pn.empty()) {
                const cudaError_t e = cudaMemcpy(out, pn.data(), pn.size() * sizeof(trb::DPair), cudaMemcpyHostToDevice);
                if (e != cudaSuccess) r = fail(TRB_CUDA, std::string("cudaMemcpy(node records): ") + cudaGetErrorString(e));
            }
        }
        if (r != TRB_OK) {
            s->arena.release(d_pos); s->arena.release(d_tris);
            if (pairs != dm.bvh.pairs) s->arena.release(pairs);
            return r;
        }
        mark(4);
        // commit: positions, triangle records, tree and header
        s->arena.release(dm.positions);
        s->arena.release(dm.tris);
        if (pairs != dm.bvh.pairs) s->arena.release(dm.bvh.pairs);
        if (dm.bvh.quads) s->arena.release(dm.bvh.quads);
        if (hm.d_refit) s->arena.release(hm.d_refit); // the refit's parent links follow the old topology
        hm.nodes = std::move(nm.nodes); hm.order = std::move(nm.order);
        hm.narrow = narrow; hm.pair_cap = cap; hm.stale = false; hm.d_refit = nullptr;
        for (int k = 0; k < 3; ++k) { hm.bounds.lo[k] = hm.nodes[0].bmin[k]; hm.bounds.hi[k] = hm.nodes[0].bmax[k]; }
        const trb_bvh_node& root = hm.nodes[0];
        uint32_t root_ref = trb::REF_INTERIOR; // record 0
        if (root.b & TRB_BVH_LEAF)
            root_ref = s->wide_leaf ? (trb::REF_LEAF | (root.a & ~trb::REF_TAG)) : (trb::REF_LEAF | ((root.b & ~TRB_BVH_LEAF) << 25) | root.a);
        dm.positions = d_pos; dm.tris = d_tris; dm.n_nodes = (uint32_t)hm.nodes.size();
        dm.bvh.pairs = pairs; dm.bvh.quads = nullptr; // DQuad records (trace.quads) are built at creation only
        dm.bvh.root_lo = make_float4(hm.bounds.lo[0], hm.bounds.lo[1], hm.bounds.lo[2], bits_f(root_ref));
        dm.bvh.root_hi = make_float4(hm.bounds.hi[0], hm.bounds.hi[1], hm.bounds.hi[2], bits_f(QUAD_EMPTY_HOST));
        s->quads_dropped = true;
        s->needs_wide = false;
        for (const HostMesh& m : s->meshes) if (!m.narrow) s->needs_wide = true;
        const bool wide = s->needs_wide || s->tune.wide_leaf != 0;
        if (wide != s->wide_leaf) { // the scene's leaf form changes with this tree: every mesh is re-packed, headers included
            const trb_status rw = upload_mesh_nodes(s, wide);
            if (rw != TRB_OK) return rw;
        } else CU(cudaMemcpy(s->d_meshes + mi, &dm, sizeof dm, cudaMemcpyHostToDevice));
    } else CU(cudaDeviceSynchronize()); // kernels in flight may read the attributes overwritten below
    { const trb_status r = copy_mesh_attributes(s, mi, nrm, uv, device, st); if (r != TRB_OK) return r; }
    if (pos && s->frame_set) { // instance bounds and the TLAS over the new mesh bounds
        const trb_status r = trb_scene_update_frame(s, s->last_frame, s->last_start, s->last_end);
        if (r != TRB_OK) return r;
    }
    report();
    return TRB_OK;
}

// trb_scene_refit_mesh(_device): new positions through the mesh's kept tree (DESIGN.md §4 "Mesh refits"). Without positions it is
// update_mesh's attribute copy. With them: the device is drained, the positions are copied in place, the triangle records rewritten
// (k_refit_tris) and the node boxes recomputed bottom-up in the records (k_refit_nodes, after k_refit_parents on a mesh's first refit),
// all on `st`; the root box (the header's 24 bytes) is the only read-back. The host tree is marked stale instead of being copied back.
// Nothing here depends on the values of the positions, so the call fails only on a CUDA error.
trb_status refit_mesh(trb_scene* s, uint32_t mi, const float* pos, const float* nrm, const float* uv, bool device, cudaStream_t st) {
    if (!pos) return update_mesh(s, mi, nullptr, nrm, uv, device, st);
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    if (mi >= s->meshes.size()) return fail(TRB_INVALID_ARG, "mesh index out of range");
    CU(cudaSetDevice(s->device));
    HostMesh& hm = s->meshes[mi];
    trb::DMesh& dm = s->dmeshes[mi];
    const uint32_t n_rec = (uint32_t)((hm.nodes.size() - 1) / 2);
    const auto grid = [](size_t k) { return (unsigned)std::max<size_t>(1, (k + 255) / 256); };
    CU(cudaDeviceSynchronize()); // kernels in flight read the positions, triangle records, node records and header rewritten below
    if (!hm.d_refit) {
        uint32_t* links = nullptr;
        CU(s->arena.alloc(2 * (size_t)n_rec, &links));
        hm.d_refit = links;
        trb::bvhb::k_refit_parents<<<grid(n_rec), 256, 0, st>>>(dm.bvh.pairs, n_rec, hm.d_refit);
        ++g_launches;
    }
    CU(mesh_copy_in(dm.positions, pos, 3 * (size_t)hm.n_verts, device, st));
    if (dm.bvh.quads) { s->arena.release(dm.bvh.quads); dm.bvh.quads = nullptr; } // DQuad records (trace.quads) are built at creation only
    dm.bvh.root_hi.w = bits_f(QUAD_EMPTY_HOST);
    s->quads_dropped = true;
    trb::DMesh* d_dm = s->d_meshes + mi;
    CU(cudaMemcpyAsync(d_dm, &dm, sizeof dm, cudaMemcpyHostToDevice, st));
    if (n_rec) CU(cudaMemsetAsync(hm.d_refit + n_rec, 0, 4 * (size_t)n_rec, st));
    trb::bvhb::k_refit_tris<<<grid(dm.n_tris), 256, 0, st>>>(dm.positions, dm.indices, dm.n_tris, const_cast<trb::DTri*>(dm.tris));
    trb::bvhb::k_refit_nodes<<<grid(n_rec), 256, 0, st>>>(const_cast<trb::DPair*>(dm.bvh.pairs), n_rec, hm.d_refit, hm.d_refit + n_rec,
                                                          s->wide_leaf, dm.tris, dm.indices, dm.positions, &d_dm->bvh);
    g_launches += 2;
    CU(cudaGetLastError());
    trb::DBvh hdr{};
    CU(cudaMemcpyAsync(&hdr, &d_dm->bvh, sizeof hdr, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    dm.bvh.root_lo = hdr.root_lo; dm.bvh.root_hi = hdr.root_hi;
    for (int k = 0; k < 3; ++k) { hm.bounds.lo[k] = (&hdr.root_lo.x)[k]; hm.bounds.hi[k] = (&hdr.root_hi.x)[k]; }
    hm.stale = true;
    { const trb_status r = copy_mesh_attributes(s, mi, nrm, uv, device, st); if (r != TRB_OK) return r; }
    if (s->frame_set) return trb_scene_update_frame(s, s->last_frame, s->last_start, s->last_end); // instance bounds and the TLAS
    return TRB_OK;
}

// ---- description edits (trb_scene_update_keyframes / _color_keys / _materials; DESIGN.md §4 "Scene edits") ----------------------
// The argument checks, before anything is read: entries [first, first + count) of an array of n. *done: nothing to do (count 0).
trb_status edit_check(const trb_scene* s, uint32_t first, uint32_t count, const void* a, size_t n, bool device, bool* done) {
    *done = false;
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    if (count == 0) { *done = true; return TRB_OK; }
    if (!a) return fail(TRB_INVALID_ARG, "null array");
    if ((uint64_t)first + count > n) return fail(TRB_INVALID_ARG, "edit range out of bounds");
    return device ? check_aligned({{a, 4}}, "device array must be 4-byte aligned") : TRB_OK;
}

// The host mirror, the device keyframe table, the level transforms of the one-control-point splines whose point was edited and, when
// a keyframed spline's control points were edited, the distinct-spline tables; then the frame, as update_frame built it
trb_status update_keyframes(trb_scene* s, uint32_t first, uint32_t count, const trb_keyframe* kf) {
    CU(cudaSetDevice(s->device));
    CU(cudaDeviceSynchronize()); // kernels in flight may read what is overwritten below
    std::copy(kf, kf + count, s->keyframes.begin() + first);
    CU(cudaMemcpy(const_cast<trb_keyframe*>(s->ds.keyframes) + first, kf, count * sizeof(trb_keyframe), cudaMemcpyHostToDevice));
    const uint64_t last = (uint64_t)first + count;
    size_t lo = s->splines.size(), hi = 0;
    bool keyed = false;
    for (size_t k = 0; k < s->splines.size(); ++k) {
        const trb_spline& sp = s->splines[k];
        if (sp.ctrl_first >= last || (uint64_t)sp.ctrl_first + sp.n_ctrl <= first) continue;
        if (sp.n_ctrl == 1) { lo = std::min(lo, k); hi = std::max(hi, k); }
        else keyed = true;
    }
    if (lo <= hi) { // the span between the first and the last edited level
        std::vector<Xf> level(hi - lo + 1);
        for (size_t k = lo; k <= hi; ++k) level[k - lo] = level_transform(s, k);
        CU(cudaMemcpy(const_cast<Xf*>(s->ds.level_xf) + lo, level.data(), level.size() * sizeof(Xf), cudaMemcpyHostToDevice));
    }
    if (keyed) {
        std::vector<uint32_t> uniq_of, uniq_list;
        spline_dedup(s, uniq_of, uniq_list);
        CU(cudaMemcpy(const_cast<uint32_t*>(s->ds.spline_uniq), uniq_of.data(), uniq_of.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
        CU(cudaMemcpy(const_cast<uint32_t*>(s->ds.uniq_splines), uniq_list.data(), uniq_list.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
        s->ds.n_uniq_splines = (uint32_t)uniq_list.size();
    }
    if (s->frame_set) return trb_scene_update_frame(s, s->last_frame, s->last_start, s->last_end);
    return TRB_OK;
}

// The host mirror, the device colour-key table and the static emission of the instance records whose first key was edited. Only
// the emission fields are written: the device frame path uploads the rest of the records once and then writes the matrices alone.
trb_status update_color_keys(trb_scene* s, uint32_t first, uint32_t count, const trb_color_key* keys) {
    CU(cudaSetDevice(s->device));
    CU(cudaDeviceSynchronize());
    std::copy(keys, keys + count, s->color_keys.begin() + first);
    CU(cudaMemcpy(const_cast<trb_color_key*>(s->ds.color_keys) + first, keys, count * sizeof(trb_color_key), cudaMemcpyHostToDevice));
    std::vector<trb::DInstance> di;
    std::vector<uint32_t> anim_list;
    static_instance_records(s, di, anim_list);
    size_t lo = di.size(), hi = 0;
    for (size_t i = 0; i < di.size(); ++i) {
        const trb_instance& in = s->instances[i];
        if (in.kind != TRB_INST_RECEIVER && in.emission_first >= first && in.emission_first - first < count) { lo = std::min(lo, i); hi = std::max(hi, i); }
    }
    if (lo <= hi)
        CU(cudaMemcpy2D(s->d_instances[lo].emission, sizeof(trb::DInstance), di[lo].emission, sizeof(trb::DInstance), sizeof di[lo].emission,
                        hi - lo + 1, cudaMemcpyHostToDevice));
    return TRB_OK;
}

// Checked as trb_scene_create checks them; then the host mirror, the device records and the shading shape (material_shape)
trb_status update_materials(trb_scene* s, uint32_t first, uint32_t count, const trb_material* m) {
    for (uint32_t i = 0; i < count; ++i) {
        const trb_status r = validate_material(m[i], s->n_merl, s->ds.n_textures);
        if (r != TRB_OK) return r;
    }
    std::vector<trb::DMaterial> dm(count);
    for (uint32_t i = 0; i < count; ++i) dm[i] = device_material(m[i]);
    CU(cudaSetDevice(s->device));
    CU(cudaDeviceSynchronize());
    std::copy(m, m + count, s->materials.begin() + first);
    CU(cudaMemcpy(const_cast<trb::DMaterial*>(s->ds.materials) + first, dm.data(), count * sizeof(trb::DMaterial), cudaMemcpyHostToDevice));
    material_shape(s);
    return TRB_OK;
}


// ---- the object section (trb_scene_create, trb_scene_replace_objects; DESIGN.md §4 "Object replacement") ------------------------
// Makes `o`, already checked by validate_objects, the scene's object section: the host copy (knots sorted as BSpline::new sorts
// them), the light list, the instance records without matrices (so that trb_emitted runs before the first update_frame), the
// animation tables, and what the kernels' choice depends on (n_anim, material_shape, anim_emission). Needs the scene's meshes and
// materials in place. The new device buffers are complete before DScene is switched over and the ones they replace are released, so
// a failure leaves the scene as it was. set_objects is stage_objects, which builds all of that without touching the scene, then
// commit_objects, which switches the scene over; the caller has drained the device before the commit.
struct StagedObjects {
    std::vector<trb_camera> cameras;
    std::vector<trb_instance> instances;
    std::vector<trb_spline> splines;
    std::vector<trb_keyframe> keyframes;
    std::vector<float> knots, fov_floats;
    std::vector<trb_color_key> color_keys;
    std::vector<uint32_t> anim_list;
    bool inst_any_anim = false;
    uint32_t n_lights = 0, n_uniq = 0;
    DeviceArena fresh; // frees what it holds unless committed
    uint32_t *d_lights = nullptr, *d_anim = nullptr, *d_uo = nullptr, *d_ul = nullptr;
    trb::DInstance* d_inst = nullptr;
    trb_spline* d_sp = nullptr; trb_keyframe* d_kf = nullptr; float* d_kn = nullptr; trb_color_key* d_ck = nullptr; Xf* d_lv = nullptr;
};

trb_status stage_objects(trb_scene* s, const trb_scene_objects& o, StagedObjects& g) {
    g.cameras.assign(o.cameras, o.cameras + o.n_cameras);
    g.instances.assign(o.instances, o.instances + o.n_instances);
    g.splines.assign(o.splines, o.splines + o.n_splines);
    g.keyframes.assign(o.keyframes, o.keyframes + o.n_keyframes);
    g.knots.assign(o.knots, o.knots + o.n_knots); g.fov_floats.assign(o.fov_floats, o.fov_floats + o.n_fov_floats);
    g.color_keys.assign(o.color_keys, o.color_keys + o.n_color_keys);
    for (const trb_spline& sp : g.splines) // BSpline::new sorts its knots (bspline 0.2.2); ranges were bounds-checked by validate_objects()
        if (sp.n_ctrl > 1) std::stable_sort(g.knots.begin() + sp.knot_first, g.knots.begin() + sp.knot_first + sp.n_knots);
    for (const trb_camera& c : g.cameras)
        if (c.n_fov_ctrl) std::stable_sort(g.fov_floats.begin() + c.fov_knot_first, g.fov_floats.begin() + c.fov_knot_first + c.n_fov_knots);
    // the helpers below read the section from the scene: it is swapped in while they run and swapped out again before returning
    auto swap_host = [&] {
        s->cameras.swap(g.cameras); s->instances.swap(g.instances); s->splines.swap(g.splines); s->keyframes.swap(g.keyframes);
        s->knots.swap(g.knots); s->fov_floats.swap(g.fov_floats); s->color_keys.swap(g.color_keys);
    };
    swap_host();
    std::vector<uint32_t> lights;
    for (uint32_t i = 0; i < o.n_instances; ++i) if (s->instances[i].kind != TRB_INST_RECEIVER) lights.push_back(i); // multithreaded.rs:33-38
    std::vector<trb::DInstance> di;
    std::vector<uint32_t> uniq_of, uniq_list;
    g.inst_any_anim = static_instance_records(s, di, g.anim_list);
    std::vector<Xf> level(s->splines.size());
    for (size_t k = 0; k < level.size(); ++k) level[k] = level_transform(s, k);
    spline_dedup(s, uniq_of, uniq_list);
    // room for every keyframed spline: a keyframe edit can make splines that were equal distinct (trb_scene_update_keyframes)
    const size_t n_keyed = (size_t)std::count_if(s->splines.begin(), s->splines.end(), [](const trb_spline& sp) { return sp.n_ctrl > 1; });
    g.n_lights = (uint32_t)lights.size(); g.n_uniq = (uint32_t)uniq_list.size();
    const trb_status r = [&]() -> trb_status {
        CU(g.fresh.upload(lights.data(), lights.size(), &g.d_lights));
        CU(g.fresh.upload(di.data(), di.size(), &g.d_inst));
        CU(g.fresh.alloc(di.size(), &g.d_anim)); // update_frame fills it
        if (!s->splines.empty()) CU(g.fresh.upload(s->splines.data(), s->splines.size(), &g.d_sp));
        if (!s->keyframes.empty()) CU(g.fresh.upload(s->keyframes.data(), s->keyframes.size(), &g.d_kf));
        if (!s->knots.empty()) CU(g.fresh.upload(s->knots.data(), s->knots.size(), &g.d_kn));
        if (!s->color_keys.empty()) CU(g.fresh.upload(s->color_keys.data(), s->color_keys.size(), &g.d_ck));
        if (!level.empty()) CU(g.fresh.upload(level.data(), level.size(), &g.d_lv));
        if (!uniq_of.empty()) CU(g.fresh.upload(uniq_of.data(), uniq_of.size(), &g.d_uo));
        if (n_keyed) {
            CU(g.fresh.alloc(n_keyed, &g.d_ul));
            CU(cudaMemcpy(g.d_ul, uniq_list.data(), uniq_list.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
        }
        return TRB_OK;
    }();
    swap_host();
    return r;
}

// Needs the scene's meshes and materials in place (material_shape reads the materials)
void commit_objects(trb_scene* s, StagedObjects& g) {
    s->cameras.swap(g.cameras); s->instances.swap(g.instances); s->splines.swap(g.splines); s->keyframes.swap(g.keyframes);
    s->knots.swap(g.knots); s->fov_floats.swap(g.fov_floats); s->color_keys.swap(g.color_keys);
    trb::DScene& ds = s->ds;
    for (const void* p : {(const void*)ds.lights, (const void*)s->d_instances, (const void*)s->d_anim_instances, (const void*)ds.splines,
                          (const void*)ds.keyframes, (const void*)ds.knots, (const void*)ds.color_keys, (const void*)ds.level_xf,
                          (const void*)ds.spline_uniq, (const void*)ds.uniq_splines}) s->arena.release(p);
    s->arena.ptrs.insert(s->arena.ptrs.end(), g.fresh.ptrs.begin(), g.fresh.ptrs.end());
    g.fresh.ptrs.clear();
    s->d_instances = g.d_inst; s->d_anim_instances = g.d_anim;
    ds.instances = g.d_inst; ds.n_instances = (uint32_t)s->instances.size(); ds.lights = g.d_lights; ds.n_lights = g.n_lights;
    ds.splines = g.d_sp; ds.keyframes = g.d_kf; ds.knots = g.d_kn; ds.color_keys = g.d_ck; ds.level_xf = g.d_lv;
    ds.spline_uniq = g.d_uo; ds.uniq_splines = g.d_ul; ds.n_uniq_splines = g.n_uniq;
    ds.has_anim = 0; ds.anim_instances = nullptr; ds.n_anim_instances = 0; // update_frame sets them
    s->n_anim = (uint32_t)g.anim_list.size();
    s->anim_list.swap(g.anim_list); s->inst_any_anim = g.inst_any_anim;
    material_shape(s);
    s->anim_emission = false;
    for (const trb_instance& in : s->instances) if (in.kind != TRB_INST_RECEIVER && in.n_emission > 1) s->anim_emission = true;
}

trb_status set_objects(trb_scene* s, const trb_scene_objects& o) {
    StagedObjects g;
    const trb_status r = stage_objects(s, o, g);
    if (r != TRB_OK) return r;
    commit_objects(s, g);
    return TRB_OK;
}

// After a new object section was committed: nothing of the old instance list's frame survives, and the camera is selected as on a
// new scene's first frame (scene.rs:153-166). The caller re-runs the frame that had been set.
void objects_replaced(trb_scene* s) {
    s->frame_ready = false; s->instances_static_uploaded = false; s->host_frame_stale = false;
    s->world.clear(); s->tlas_nodes.clear(); s->tlas_order.clear(); s->tlas_n_nodes = 0;
    s->active_camera = -1;
    if (s->wf.n_anim != s->n_anim) s->wf_capacity = 0; // WfState::xf_tab is sized by n_anim: ensure_wavefront allocates the state anew
}

// The checks of a new object section against a scene whose meshes and materials will number n_meshes and n_materials:
// trb_scene_create's, and that the frame that has been set can be set again
trb_status check_objects(const trb_scene* s, const trb_scene_objects& o, uint32_t n_meshes, uint32_t n_materials) {
    const trb_status v = validate_objects(o, n_meshes, n_materials);
    if (v != TRB_OK) return v;
    if (s->frame_set && o.cameras[0].active_at > s->last_frame) return fail(TRB_INVALID_ARG, "no camera is active at this frame");
    return TRB_OK;
}

// Checked as trb_scene_create checks the section; then set_objects, the state that was sized or built for the old section, and the frame
trb_status replace_objects(trb_scene* s, const trb_scene_objects& o) {
    const trb_status v = check_objects(s, o, (uint32_t)s->meshes.size(), (uint32_t)s->materials.size());
    if (v != TRB_OK) return v;
    CU(cudaSetDevice(s->device));
    CU(cudaDeviceSynchronize()); // passes enqueued by the _device calls may still read the buffers released below
    const trb_status r = set_objects(s, o);
    if (r != TRB_OK) return r;
    objects_replaced(s);
    if (s->frame_set) return trb_scene_update_frame(s, s->last_frame, s->last_start, s->last_end);
    return TRB_OK;
}

// ---- the mesh section (trb_scene_replace_meshes; DESIGN.md §4 "Mesh replacement") -----------------------------------------------
// Checks everything first (keep entries, new meshes as creation checks them, the object section or the current instances against the
// new mesh count); builds every new mesh, the new header array and the staged object section into fresh buffers; and only then drains
// the device, switches the scene over and releases what was replaced. Kept meshes move with their buffers, trees and records; their
// records are re-packed only when the scene's leaf form changes with the new list.
trb_status replace_meshes(trb_scene* s, const trb_scene_meshes& sec, const trb_scene_objects* o, bool device, cudaStream_t st) {
    const uint32_t n = sec.n_meshes, n_old = (uint32_t)s->meshes.size();
    if (n && !sec.keep) return fail(TRB_INVALID_ARG, "null keep array with a non-zero mesh count");
    std::vector<char> named(n_old, 0);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t k = sec.keep[i];
        if (k == TRB_MESH_NEW) { if (!sec.meshes) return fail(TRB_INVALID_ARG, "null meshes array with a new mesh"); continue; }
        if (k >= n_old) return fail(TRB_INVALID_ARG, "kept mesh index out of range");
        if (named[k]) return fail(TRB_INVALID_ARG, "a mesh is kept twice");
        named[k] = 1;
    }
    if (o) { const trb_status v = check_objects(s, *o, n, (uint32_t)s->materials.size()); if (v != TRB_OK) return v; }
    else
        for (const trb_instance& in : s->instances)
            if (in.shape == TRB_SHAPE_MESH && in.mesh >= n) return fail(TRB_INVALID_ARG, "mesh index out of range");
    for (uint32_t i = 0; i < n; ++i)
        if (sec.keep[i] == TRB_MESH_NEW) { const trb_status v = validate_mesh(sec.meshes[i], device); if (v != TRB_OK) return v; }
    CU(cudaSetDevice(s->device));

    // build: new meshes, the leaf form of the new list, new meshes' node records in it, the header array, the object section
    DeviceArena fresh; // frees what it holds if anything below fails
    std::vector<HostMesh> built(n);
    std::vector<trb::DMesh> dmeshes(n);
    bool needs_wide = false;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t k = sec.keep[i];
        if (k != TRB_MESH_NEW) { dmeshes[i] = s->dmeshes[k]; needs_wide |= !s->meshes[k].narrow; continue; }
        const trb_status r = setup_mesh(s, fresh, sec.meshes[i], device, st, built[i], dmeshes[i]);
        if (r != TRB_OK) return r;
        needs_wide |= !built[i].narrow;
    }
    const bool wide = needs_wide || s->tune.wide_leaf != 0, repack = wide != s->wide_leaf;
    if (!repack) // otherwise every mesh is packed below, once the kept ones' records are no longer read
        for (uint32_t i = 0; i < n; ++i)
            if (sec.keep[i] == TRB_MESH_NEW) { const trb_status r = pack_mesh_nodes(built[i], dmeshes[i].bvh, wide); if (r != TRB_OK) return r; }
    trb::DMesh* d_meshes = nullptr;
    CU(fresh.upload(dmeshes.data(), dmeshes.size(), &d_meshes));
    StagedObjects g;
    if (o) { const trb_status r = stage_objects(s, *o, g); if (r != TRB_OK) return r; }

    // switch: passes enqueued by the _device calls may still read the buffers released here
    CU(cudaDeviceSynchronize());
    for (uint32_t k = 0; k < n_old; ++k) {
        if (named[k]) continue;
        const trb::DMesh& dm = s->dmeshes[k];
        for (const void* p : {(const void*)dm.positions, (const void*)dm.normals, (const void*)dm.texcoords, (const void*)dm.indices,
                              (const void*)dm.tris, (const void*)dm.bvh.pairs, (const void*)dm.bvh.quads, (const void*)s->meshes[k].d_refit})
            if (p) s->arena.release(p);
    }
    s->arena.release(s->d_meshes);
    s->arena.ptrs.insert(s->arena.ptrs.end(), fresh.ptrs.begin(), fresh.ptrs.end());
    fresh.ptrs.clear();
    std::vector<HostMesh> meshes(n);
    for (uint32_t i = 0; i < n; ++i) meshes[i] = std::move(sec.keep[i] == TRB_MESH_NEW ? built[i] : s->meshes[sec.keep[i]]);
    s->meshes.swap(meshes); s->dmeshes.swap(dmeshes);
    s->d_meshes = d_meshes; s->ds.meshes = d_meshes;
    s->needs_wide = needs_wide;
    s->quads_dropped = false; // a narrow mesh without DQuad records was rebuilt by trb_scene_update_mesh
    for (uint32_t i = 0; i < n; ++i) if (s->meshes[i].narrow && !s->dmeshes[i].bvh.quads) s->quads_dropped = true;
    if (o) { commit_objects(s, g); objects_replaced(s); }
    else { s->instances_static_uploaded = false; s->frame_ready = false; } // the instances' mesh bounds changed
    if (repack) { const trb_status r = upload_mesh_nodes(s, wide); if (r != TRB_OK) return r; }
    if (s->frame_set) return trb_scene_update_frame(s, s->last_frame, s->last_start, s->last_end);
    return TRB_OK;
}

// ---- film, integrator and material section (trb_scene_create, trb_scene_replace_settings / _materials; DESIGN.md §4 "Settings
// replacement" and "Material replacement") ---------------------------------------------------------------------------------------
// Each part is staged into fresh buffers without touching the scene, then committed once the device has been drained, so creation
// and replacement run the same code and a failed replacement leaves the scene as it was.

// k_simple_integrator (Whitted and NormalsDebug) is recursive, so its stack is the context's limit, not a size ptxas computed: the
// reference's recursion is kept as device recursion (one frame per ray depth), and even NormalsDebug's one scene_trace call (kernel
// frame + scene_trace's, about 1.8 KB on sm_90a) needs more than CUDA's default 1 KB. The limit is raised, never lowered.
trb_status raise_stack_limit(const trb_integrator& in) {
    if (in.type != TRB_INTEGRATOR_WHITTED && in.type != TRB_INTEGRATOR_NORMALS_DEBUG) return TRB_OK;
    size_t have = 0;
    CU(cudaDeviceGetLimit(&have, cudaLimitStackSize));
    const size_t need = 4096 + (size_t)2048 * (in.max_depth + 2);
    if (have < need) CU(cudaDeviceSetLimit(cudaLimitStackSize, need));
    return TRB_OK;
}

// The film's filter table (host and device), the device film of trb_render and its pinned host staging
struct StagedFilm {
    trb_film film{};
    float table[256];
    DeviceArena fresh; // frees what it holds unless committed
    float* d_table = nullptr;
    float4* d_film = nullptr;
    float* h_staging = nullptr; // pinned; freed unless committed
    ~StagedFilm() { if (h_staging) cudaFreeHost(h_staging); }
};

trb_status stage_film(const trb_film& f, StagedFilm& g) {
    g.film = f;
    filter_table(f, g.table);
    const size_t npx = (size_t)f.width * f.height;
    CU(g.fresh.upload(g.table, 256, &g.d_table));
    CU(g.fresh.alloc(npx, &g.d_film));
    CU(cudaMallocHost(&g.h_staging, npx * 4 * sizeof(float)));
    return TRB_OK;
}

// Also retires what was made for the old film: the Morton block lists (keyed by the selection, not by the film size) and the Adaptive
// sampler's per-pixel and per-block state (sized by the pixel count; ensure_adaptive allocates it anew), the denoiser's scratch and the
// sharded renders' AOV films (both sized by the pixel count and allocated anew by their next use). The caller has drained the device.
void commit_film(trb_scene* s, StagedFilm& g) {
    trb::DScene& ds = s->ds;
    s->arena.release(ds.filter_table); s->arena.release(s->d_film);
    s->arena.ptrs.insert(s->arena.ptrs.end(), g.fresh.ptrs.begin(), g.fresh.ptrs.end());
    g.fresh.ptrs.clear();
    if (s->h_film_staging) cudaFreeHost(s->h_film_staging);
    s->h_film_staging = g.h_staging; g.h_staging = nullptr;
    s->d_film = g.d_film;
    const trb_film& f = g.film;
    s->film = f;
    std::memcpy(s->table, g.table, sizeof s->table);
    s->spp_pow2 = pow2_ceil(std::max(1u, f.samples));
    ds.width = f.width; ds.height = f.height;
    ds.filter_w = f.filter_w; ds.filter_h = f.filter_h;
    ds.filter_inv_w = 1.0f / f.filter_w; ds.filter_inv_h = 1.0f / f.filter_h;
    ds.fpw_x = (int)floorf(f.filter_w / 0.5f); ds.fpw_y = (int)floorf(f.filter_h / 0.5f); // render_target.rs:48-49
    // the per-pixel test accepts |d| <= w / inv_w; the lock-block filter of render_target.rs:104-109 can only reject beyond fpw - 0.5
    ds.film_block_filter = (f.filter_w / ds.filter_inv_w <= (float)ds.fpw_x && f.filter_h / ds.filter_inv_h <= (float)ds.fpw_y) ? 0u : 1u;
    ds.filter_table = g.d_table;
    for (BlockList& b : s->block_lists) cudaFree(b.dev);
    s->block_lists.clear();
    for (void** p : {(void**)&s->d_ad_state, (void**)&s->d_ad_list[0], (void**)&s->d_ad_list[1], (void**)&s->d_ad_index[0],
                     (void**)&s->d_ad_index[1], (void**)&s->d_ad_flags, (void**)&s->d_ad_count, (void**)&s->d_ad_spp, &s->d_denoise, &s->d_shard_aov}) {
        if (*p) cudaFree(*p);
        *p = nullptr;
    }
    s->denoise_pixels = 0;
}

// The material records, MERL tables and image textures, and the counts they are checked against
struct StagedMaterials {
    std::vector<trb_material> materials;
    uint32_t n_merl = 0, n_textures = 0;
    DeviceArena fresh; // frees what it holds unless committed
    trb::DMaterial* d_mats = nullptr;
    float* d_merl = nullptr;
    trb::DImage* d_img = nullptr; trb::DTexture* d_tex = nullptr; uchar4* d_tx = nullptr;
};

// `m` checked by validate_materials. With `device` the MERL tables and the images' texels are device memory on the scene's GPU,
// copied on `st`; otherwise host memory.
trb_status stage_materials(const trb_scene_materials& m, bool device, cudaStream_t st, StagedMaterials& g) {
    g.materials.assign(m.materials, m.materials + m.n_materials);
    g.n_merl = m.n_merl; g.n_textures = m.n_textures;
    // precompute what Material::bsdf recomputes per hit from constant textures
    std::vector<trb::DMaterial> dmats(m.n_materials);
    for (uint32_t i = 0; i < m.n_materials; ++i) dmats[i] = device_material(m.materials[i]);
    CU(g.fresh.upload(dmats.data(), dmats.size(), &g.d_mats));
    auto copy = [&](void* dst, const void* src, size_t bytes) {
        return device ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st) : cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
    };
    CU(g.fresh.alloc((size_t)m.n_merl * TRB_MERL_TABLE_FLOATS, &g.d_merl));
    for (uint32_t i = 0; i < m.n_merl; ++i)
        CU(copy(g.d_merl + (size_t)i * TRB_MERL_TABLE_FLOATS, m.merl_tables[i], sizeof(float) * TRB_MERL_TABLE_FLOATS));
    // image textures: every frame's RGBA8 texels in one array (texture/image.rs)
    std::vector<trb::DImage> dimg(m.n_images);
    std::vector<trb::DTexture> dtex(m.n_textures);
    size_t n_tx = 0;
    for (uint32_t i = 0; i < m.n_images; ++i) {
        const trb_image& im = m.images[i];
        dimg[i].width = im.width; dimg[i].height = im.height; dimg[i].offset = (uint32_t)n_tx; dimg[i].time = im.time;
        n_tx += (size_t)im.width * im.height;
    }
    for (uint32_t i = 0; i < m.n_textures; ++i) { dtex[i].first_image = m.textures[i].first_image; dtex[i].n_images = m.textures[i].n_images; }
    CU(g.fresh.upload(dimg.data(), dimg.size(), &g.d_img));
    CU(g.fresh.upload(dtex.data(), dtex.size(), &g.d_tex));
    CU(g.fresh.alloc(n_tx, &g.d_tx));
    for (uint32_t i = 0; i < m.n_images; ++i)
        CU(copy(g.d_tx + dimg[i].offset, m.images[i].rgba8, (size_t)m.images[i].width * m.images[i].height * 4));
    if (device) CU(cudaStreamSynchronize(st));
    return TRB_OK;
}

// Also the shading shape (material_shape), which needs the object section in place. The caller has drained the device.
void commit_materials(trb_scene* s, StagedMaterials& g) {
    trb::DScene& ds = s->ds;
    for (const void* p : {(const void*)ds.materials, (const void*)ds.merl, (const void*)ds.images, (const void*)ds.textures,
                          (const void*)ds.texels}) s->arena.release(p);
    s->arena.ptrs.insert(s->arena.ptrs.end(), g.fresh.ptrs.begin(), g.fresh.ptrs.end());
    g.fresh.ptrs.clear();
    s->materials.swap(g.materials); s->n_merl = g.n_merl;
    ds.materials = g.d_mats; ds.merl = g.d_merl;
    ds.images = g.d_img; ds.textures = g.d_tex; ds.texels = g.d_tx; ds.n_textures = g.n_textures;
    material_shape(s);
}

// trb_scene_replace_settings: checked as trb_scene_create checks the film and the integrator; the new film staged and the stack limit
// raised before the device is drained and anything switched; then the frame, whose camera depends on the film size
trb_status replace_settings(trb_scene* s, const trb_film* film, const trb_integrator* integrator) {
    const trb_integrator in = integrator ? *integrator : s->integrator;
    { const trb_status v = validate_settings(film ? *film : s->film, in); if (v != TRB_OK) return v; }
    CU(cudaSetDevice(s->device));
    StagedFilm g;
    if (film) { const trb_status r = stage_film(*film, g); if (r != TRB_OK) return r; }
    if (integrator) { const trb_status r = raise_stack_limit(in); if (r != TRB_OK) return r; }
    CU(cudaDeviceSynchronize()); // passes enqueued by the _device calls may still read the buffers released below
    if (film) commit_film(s, g);
    s->integrator = in;
    s->ds.min_depth = in.min_depth; s->ds.max_depth = in.max_depth;
    if (s->frame_set) return trb_scene_update_frame(s, s->last_frame, s->last_start, s->last_end);
    return TRB_OK;
}

// trb_scene_replace_materials(_device): checks everything first (null arrays, the section as creation checks it, the object section or
// the current instances against the new material count), stages the section and the object section, and only then drains the device
// and switches the scene over
trb_status replace_materials(trb_scene* s, const trb_scene_materials& m, const trb_scene_objects* o, bool device, cudaStream_t st) {
    if ((m.n_materials && !m.materials) || (m.n_merl && !m.merl_tables) || (m.n_textures && !m.textures) || (m.n_images && !m.images))
        return fail(TRB_INVALID_ARG, "null array with a non-zero count");
    for (uint32_t i = 0; i < m.n_merl; ++i) if (!m.merl_tables[i]) return fail(TRB_INVALID_ARG, "null MERL table");
    { const trb_status v = validate_materials(m); if (v != TRB_OK) return v; }
    if (o) { const trb_status v = check_objects(s, *o, (uint32_t)s->meshes.size(), m.n_materials); if (v != TRB_OK) return v; }
    else
        for (const trb_instance& in : s->instances)
            if (in.kind != TRB_INST_EMITTER_POINT && in.material >= m.n_materials) return fail(TRB_INVALID_ARG, "material index out of range");
    CU(cudaSetDevice(s->device));
    StagedMaterials g;
    { const trb_status r = stage_materials(m, device, st, g); if (r != TRB_OK) return r; }
    StagedObjects go;
    if (o) { const trb_status r = stage_objects(s, *o, go); if (r != TRB_OK) return r; }
    CU(cudaDeviceSynchronize()); // passes enqueued by the _device calls may still read the buffers released below
    commit_materials(s, g);
    if (o) { commit_objects(s, go); objects_replaced(s); }
    if (s->frame_set) return trb_scene_update_frame(s, s->last_frame, s->last_start, s->last_end);
    return TRB_OK;
}

} // namespace

extern "C" {

trb_status trb_scene_update_keyframes(trb_scene* s, uint32_t first, uint32_t count, const trb_keyframe* keyframes) {
    bool done;
    const trb_status r = edit_check(s, first, count, keyframes, s ? s->keyframes.size() : 0, false, &done);
    return r != TRB_OK || done ? r : update_keyframes(s, first, count, keyframes);
}
trb_status trb_scene_update_keyframes_device(trb_scene* s, uint32_t first, uint32_t count, const trb_keyframe* d_keyframes, void* cuda_stream) {
    bool done;
    const trb_status r = edit_check(s, first, count, d_keyframes, s ? s->keyframes.size() : 0, true, &done);
    if (r != TRB_OK || done) return r;
    CU(cudaSetDevice(s->device));
    const cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    std::vector<trb_keyframe> kf(count);
    CU(cudaMemcpyAsync(kf.data(), d_keyframes, count * sizeof(trb_keyframe), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    return update_keyframes(s, first, count, kf.data());
}
trb_status trb_scene_update_color_keys(trb_scene* s, uint32_t first, uint32_t count, const trb_color_key* keys) {
    bool done;
    const trb_status r = edit_check(s, first, count, keys, s ? s->color_keys.size() : 0, false, &done);
    return r != TRB_OK || done ? r : update_color_keys(s, first, count, keys);
}
trb_status trb_scene_update_materials(trb_scene* s, uint32_t first, uint32_t count, const trb_material* materials) {
    bool done;
    const trb_status r = edit_check(s, first, count, materials, s ? s->materials.size() : 0, false, &done);
    return r != TRB_OK || done ? r : update_materials(s, first, count, materials);
}

trb_status trb_scene_update_mesh(trb_scene* s, uint32_t mesh, const float* positions, const float* normals, const float* texcoords) {
    return update_mesh(s, mesh, positions, normals, texcoords, false, nullptr);
}
trb_status trb_scene_update_mesh_device(trb_scene* s, uint32_t mesh, const float* d_positions, const float* d_normals, const float* d_texcoords,
                                        void* cuda_stream) {
    return update_mesh(s, mesh, d_positions, d_normals, d_texcoords, true, static_cast<cudaStream_t>(cuda_stream));
}
trb_status trb_scene_refit_mesh(trb_scene* s, uint32_t mesh, const float* positions, const float* normals, const float* texcoords) {
    return refit_mesh(s, mesh, positions, normals, texcoords, false, nullptr);
}
trb_status trb_scene_refit_mesh_device(trb_scene* s, uint32_t mesh, const float* d_positions, const float* d_normals, const float* d_texcoords,
                                       void* cuda_stream) {
    return refit_mesh(s, mesh, d_positions, d_normals, d_texcoords, true, static_cast<cudaStream_t>(cuda_stream));
}

trb_status trb_scene_replace_objects(trb_scene* s, const trb_scene_objects* objects) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    if (!objects) return fail(TRB_INVALID_ARG, "null objects");
    const trb_status r = replace_objects(s, *objects);
    if (r == TRB_OK) s->object_generation++;
    return r;
}

trb_status trb_scene_replace_meshes(trb_scene* s, const trb_scene_meshes* meshes, const trb_scene_objects* objects) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    if (!meshes) return fail(TRB_INVALID_ARG, "null meshes");
    const trb_status r = replace_meshes(s, *meshes, objects, false, nullptr);
    if (r == TRB_OK && objects) s->object_generation++;
    return r;
}
trb_status trb_scene_replace_meshes_device(trb_scene* s, const trb_scene_meshes* meshes, const trb_scene_objects* objects, void* cuda_stream) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    if (!meshes) return fail(TRB_INVALID_ARG, "null meshes");
    const trb_status r = replace_meshes(s, *meshes, objects, true, static_cast<cudaStream_t>(cuda_stream));
    if (r == TRB_OK && objects) s->object_generation++;
    return r;
}

trb_status trb_scene_replace_settings(trb_scene* s, const trb_film* film, const trb_integrator* integrator) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    return replace_settings(s, film, integrator);
}

trb_status trb_scene_replace_materials(trb_scene* s, const trb_scene_materials* materials, const trb_scene_objects* objects) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    if (!materials) return fail(TRB_INVALID_ARG, "null materials");
    return replace_materials(s, *materials, objects, false, nullptr);
}
trb_status trb_scene_replace_materials_device(trb_scene* s, const trb_scene_materials* materials, const trb_scene_objects* objects,
                                              void* cuda_stream) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    if (!materials) return fail(TRB_INVALID_ARG, "null materials");
    return replace_materials(s, *materials, objects, true, static_cast<cudaStream_t>(cuda_stream));
}

const char* trb_last_error(void) { return g_error.c_str(); }
void trb_internal_set_error(const char* msg) { g_error = msg ? msg : ""; } // used by trb_loader.cpp
uint32_t trb_abi_version(void) { return TRB_ABI_VERSION; }
unsigned long long trb_launch_count(void) { return g_launches; }

trb_status trb_scene_set_option(trb_scene* s, const char* name, long long value) {
    if (!s || !name) return fail(TRB_INVALID_ARG, "null argument");
    Tuning& t = s->tune;
    const std::string k(name);
    if (k == "trace.refill") t.refill = (int)value;
    else if (k == "trace.occupancy" || k == "trace.smem_stack") {} // round-1 knobs: the variant (trace.pipe) now fixes both
    else if (k == "trace.grid") t.trace_grid = (unsigned)std::max<long long>(0, value);
    else if (k == "trace.sched") t.sched = (uint32_t)value;
    else if (k == "trace.quads" || k == "frame.device") { // both decide what update_frame builds (the DQuad TLAS records exist on the host path only): rebuild the current frame
        int& field = k == "trace.quads" ? t.quads : t.frame_device;
        const bool changed = (field != 0) != (value != 0);
        field = (int)value;
        if (changed && s->frame_set) return trb_scene_update_frame(s, s->last_frame, s->last_start, s->last_end);
    }
    else if (k == "frame.tlas_min") { // which builder makes the instance tree: rebuild the current frame with the one now chosen
        const bool changed = t.tlas_min != value;
        t.tlas_min = value;
        if (changed && s->frame_set) return trb_scene_update_frame(s, s->last_frame, s->last_start, s->last_end);
    }
    else if (k == "trace.pipe") t.pipe = (int)value;
    else if (k == "trace.exact_box") t.exact_box = (int)value;
    else if (k == "trace.wide_leaf") { // re-pack the mesh node records when the form changes (a mesh that needs the wide form keeps it)
        t.wide_leaf = (int)value;
        const bool wide = s->needs_wide || value != 0;
        if (wide != s->wide_leaf) { CU(cudaSetDevice(s->device)); return upload_mesh_nodes(s, wide); }
    }
    else if (k == "film.v2") t.film_v2 = (int)value;
    else if (k == "sort.mode") t.sort = (int)value;
    else if (k == "sort.bits") t.sort_bits = (int)std::min<long long>(6, std::max<long long>(1, value));
    else if (k == "sort.min_round") t.sort_min_round = (int)value;
    else if (k == "shade.split") t.shade_split = (int)value;
    else if (k == "shade.sort") t.shade_sort = (int)value;
    else if (k == "shade.kind") t.shade_kind = (int)value;
    else if (k == "anim.table") t.anim_table = (int)value;
    else if (k == "shade.anim_occupancy") t.shade_anim_occ = (int)value;
    else if (k == "pass.paths") { if (value < 64) return fail(TRB_INVALID_ARG, "pass.paths must be >= 64"); t.pass_paths = (uint64_t)value; }
    else return fail(TRB_INVALID_ARG, "unknown option: " + k);
    return TRB_OK;
}

trb_status trb_scene_check_error(trb_scene* s) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    CU(cudaSetDevice(s->device));
    CU(cudaDeviceSynchronize());
    return check_error_flag(s);
}

trb_status trb_scene_trace_time(trb_scene* s, float* total_ms, uint32_t* n_launches) {
    if (!s || !total_ms || !n_launches) return fail(TRB_INVALID_ARG, "null argument");
    CU(cudaSetDevice(s->device));
    float total = 0.f;
    for (auto& e : s->trace_events) {
        CU(cudaEventSynchronize(e.second));
        float ms = 0.f;
        CU(cudaEventElapsedTime(&ms, e.first, e.second));
        total += ms;
        s->event_pool.push_back(e);
    }
    *total_ms = total; *n_launches = (uint32_t)s->trace_events.size();
    s->trace_events.clear();
    return TRB_OK;
}

trb_status trb_scene_create(const trb_scene_desc* d, int device, trb_scene** out) {
    if (!out) return fail(TRB_INVALID_ARG, "null out pointer");
    *out = nullptr;
    trb_status v = validate(d);
    if (v != TRB_OK) return v;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(TRB_NO_DEVICE, "no CUDA device: tray_rust_b200 has no CPU fallback");
    if (device < 0 || device >= ndev) return fail(TRB_INVALID_ARG, "device ordinal out of range");
    CU(cudaSetDevice(device));
    std::unique_ptr<trb_scene> s(new trb_scene);
    s->device = device;
    tuning_from_env(s->tune);
    { const trb_status r = raise_stack_limit(d->integrator); if (r != TRB_OK) return r; }
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    s->sm_count = prop.multiProcessorCount;
    s->integrator = d->integrator;

    // meshes: BVH<Triangle> with max_geom 16 (mesh.rs:44), then leaf-ordered triangle records
    s->dmeshes.resize(d->n_meshes);
    s->meshes.resize(d->n_meshes);
    for (uint32_t mi = 0; mi < d->n_meshes; ++mi) {
        const trb_status r = setup_mesh(s.get(), s->arena, d->meshes[mi], false, nullptr, s->meshes[mi], s->dmeshes[mi]);
        if (r != TRB_OK) return r;
        if (!s->meshes[mi].narrow) s->needs_wide = true;
    }
    CU(s->arena.alloc(s->dmeshes.size(), &s->d_meshes));
    { const trb_status r = upload_mesh_nodes(s.get(), s->needs_wide || s->tune.wide_leaf != 0); if (r != TRB_OK) return r; }
    s->ds.meshes = s->d_meshes;
    {
        StagedMaterials g;
        const trb_status r = stage_materials(desc_materials(*d), false, nullptr, g);
        if (r != TRB_OK) return r;
        commit_materials(s.get(), g);
    }
    {
        StagedFilm g;
        const trb_status r = stage_film(d->film, g);
        if (r != TRB_OK) return r;
        commit_film(s.get(), g);
    }
    CU(s->arena.alloc(1, &s->d_counter));
    CU(s->arena.alloc(1, &s->d_error));
    CU(cudaMemset(s->d_error, 0, sizeof(int)));
    CU(s->arena.alloc(1, &s->d_stats));
    CU(cudaEventCreate(&s->ev0));
    CU(cudaEventCreate(&s->ev1));
    s->ds.min_depth = d->integrator.min_depth; s->ds.max_depth = d->integrator.max_depth;
    { const trb_status r = set_objects(s.get(), desc_objects(*d)); if (r != TRB_OK) return r; }
    // Scene::load_file builds the BVH<Instance> for [0, scene_time] (scene.rs:141); the first render rebuilds it
    *out = s.release();
    return TRB_OK;
}

void trb_scene_destroy(trb_scene* s) {
    if (!s) return;
    cudaSetDevice(s->device);
    delete s;
}

trb_status trb_scene_info(const trb_scene* s, uint32_t* w, uint32_t* h, uint32_t* spp, uint32_t* n_blocks, uint32_t* n_inst, uint32_t* n_lights) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    if (w) *w = s->film.width; if (h) *h = s->film.height; if (spp) *spp = s->spp_pow2;
    if (n_blocks) *n_blocks = (s->film.width / 8) * (s->film.height / 8);
    if (n_inst) *n_inst = (uint32_t)s->instances.size(); if (n_lights) *n_lights = s->ds.n_lights;
    return TRB_OK;
}

namespace {
// The level builder's memory for frames of up to n instances (the scene's instance capacity), carved from trb_scene::d_build_level: the build's scratch and top tree
// (bvhb::OwnedScratch), then the record ranks (one per node and one past the end), the narrow-misfit word and the scan's storage
struct LevelScratch {
    trb::bvhb::OwnedScratch own; uint32_t* rec; uint32_t* narrow_bad; void* cub; size_t cub_bytes; size_t bytes;
    LevelScratch(uint32_t n, uint32_t small, char* base) {
        size_t off = 0;
        auto take = [&](size_t b) { char* p = base ? base + off : nullptr; off += trb::bvhb::align_up(b); return p; };
        own.base = take(trb::bvhb::scratch_layout(n, nullptr, small).bytes);
        own.tn = (trb::bvhb::TNode*)take(trb::bvhb::top_cap(n) * sizeof(trb::bvhb::TNode));
        rec = (uint32_t*)take(4 * (2 * (size_t)n + 1));
        narrow_bad = (uint32_t*)take(4);
        cub_bytes = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, 2 * (int)n);
        cub = take(cub_bytes);
        bytes = off;
    }
};
// TRB_FRAME_TIME=1: the phases of the device frame path, timed with CUDA events on the default stream, to stderr
struct FrameEvents {
    cudaEvent_t e[6] = {};
    ~FrameEvents() { for (cudaEvent_t x : e) if (x) cudaEventDestroy(x); }
};
} // namespace

trb_status trb_scene_update_frame(trb_scene* s, uint32_t frame, float start, float end) {
    if (!s) return fail(TRB_INVALID_ARG, "null scene");
    CU(cudaSetDevice(s->device));
    // A frame boundary: passes enqueued with trb_render_device may still be reading the instances / TLAS this call
    // overwrites, so the device is drained first (the reference's update_frame likewise runs between renders, scene.rs:152).
    CU(cudaDeviceSynchronize());
    const auto t_host = std::chrono::steady_clock::now();
    s->frame_set = true; s->last_frame = frame; s->last_start = start; s->last_end = end;
    // camera selection (scene.rs:153-166)
    int cam;
    if (s->active_camera >= 0) {
        cam = s->active_camera;
        if (cam != (int)s->cameras.size() - 1 && s->cameras[cam + 1].active_at == frame) cam += 1;
    } else {
        int c = 0;
        for (const trb_camera& x : s->cameras) { if (x.active_at <= frame) c++; else break; }
        if (c == 0) return fail(TRB_INVALID_ARG, "no camera is active at this frame");
        cam = c - 1;
    }
    s->active_camera = cam;
    const trb_camera& c = s->cameras[cam];
    s->shutter_open = start;                                  // camera.rs:127-129
    s->shutter_close = start + c.shutter_size * (end - start);
    Mat4 px_to_cam; float scaling[3];
    float fov = c.fov;
    if (c.n_fov_ctrl) { // sampled once per frame at the clamped mid-frame time (camera.rs:134-141)
        const float* kn = s->fov_floats.data() + c.fov_knot_first;
        const float lo = kn[c.fov_degree], hi = kn[c.n_fov_knots - 1 - c.fov_degree];
        float t = (start + end) / 2.0f;
        t = t < lo ? lo : (t > hi ? hi : t);
        fov = trbh::spline_point_f32(c.fov_degree, s->fov_floats.data() + c.fov_ctrl_first, kn, c.n_fov_knots, t);
    }
    camera_setup(fov, s->film.width, s->film.height, px_to_cam, scaling);
    // cam_world.transform(frame_time): a keyframed camera is evaluated per ray on the device (camera.rs:156)
    const bool cam_static = trbh::xf_is_static(s->splines.data(), c.spline_first, c.n_splines);
    const Xf cam_world = trbh::animated_xf(s->splines.data(), c.spline_first, c.n_splines, s->keyframes.data(), s->knots.data(), s->shutter_open);
    s->ds.cam.animated = cam_static ? 0u : 1u; s->ds.cam.spline_first = c.spline_first; s->ds.cam.n_splines = c.n_splines;
    bool any_anim = !cam_static;
    std::memcpy(s->ds.cam.px_to_cam, px_to_cam.m, 64);
    std::memcpy(s->ds.cam.cam_mat, cam_world.fwd.m, 64);
    std::memcpy(s->cam_inv, cam_world.inv.m, 64);
    std::memcpy(s->ds.cam.scaling, scaling, 12);
    s->ds.cam.shutter_open = s->shutter_open; s->ds.cam.shutter_close = s->shutter_close;

    // instance transforms + bounds, then BVH<Instance>::rebuild(shutter_open, shutter_close) (scene.rs:175, bvh.rs:61-78)
    const size_t n = s->instances.size();
    const bool device_path = s->tune.frame_device && !s->tune.quads;
    const std::vector<uint32_t>& anim_list = s->anim_list;
    std::vector<trb::DInstance> di; // the static records, where this frame uploads them: a frame on the device writes the matrices alone
    if (!device_path || !s->instances_static_uploaded) { std::vector<uint32_t> unused; static_instance_records(s, di, unused); }
    if (s->inst_any_anim) any_anim = true;
    s->ds.has_anim = any_anim ? 1u : 0u;
    if (n + 1 > s->tlas_capacity) { // a tree over n instances has < n interior records and < 2n nodes
        for (const void* p : {(const void*)s->d_tlas_quads, (const void*)s->d_tlas, (const void*)s->d_tlas_order, (const void*)s->d_tlas_nodes,
                              (const void*)s->d_bounds, (const void*)s->d_build_f, (const void*)s->d_build_u, (const void*)s->d_build_counts,
                              (const void*)s->d_build_level})
            s->arena.release(p); // grown after trb_scene_replace_objects added instances (the device was drained above)
        s->tlas_capacity = 0; s->frame_ready = false; s->d_build_level = nullptr;
        CU(s->arena.alloc(n + 1, &s->d_tlas_quads));
        CU(s->arena.alloc(n + 1, &s->d_tlas));
        CU(s->arena.alloc(n, &s->d_tlas_order));
        CU(s->arena.alloc(2 * n + 2, &s->d_tlas_nodes));
        CU(s->arena.alloc(6 * n, &s->d_bounds));
        CU(s->arena.alloc(3 * n, &s->d_build_f));
        CU(s->arena.alloc(7 * n + 8, &s->d_build_u));
        CU(s->arena.alloc(4, &s->d_build_counts));
        s->tlas_capacity = n + 1;
    }
    if (!s->d_tlas_hdr) CU(s->arena.alloc(1, &s->d_tlas_hdr));
    if (!anim_list.empty()) CU(cudaMemcpy(s->d_anim_instances, anim_list.data(), anim_list.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    s->ds.anim_instances = s->d_anim_instances; s->ds.n_anim_instances = (uint32_t)anim_list.size();
    s->ds.tlas = s->d_tlas_hdr; s->ds.tlas_pairs = s->d_tlas; s->ds.tlas_quads = s->d_tlas_quads; s->ds.tlas_order = s->d_tlas_order;

    if (device_path) {
        // ---- device path: transforms, animation bounds, SAH build and record packing all on the GPU (k_frame_instances, then
        // k_tlas_build or, from tlas_min instances, the level builder)
        const long long tlas_min = s->tune.tlas_min < 0 ? (long long)kTlasLevelMin : s->tune.tlas_min;
        const bool level = n > 0 && (long long)n >= tlas_min;
        FrameEvents ev;
        const bool timing = s->tune.frame_time != 0;
        if (timing) for (cudaEvent_t& x : ev.e) CU(cudaEventCreate(&x));
        const unsigned long long launches0 = g_launches;
        trb::bvhb::BuildTrace trace;
        auto mark = [&](int k) { if (timing) cudaEventRecord(ev.e[k], 0); };
        auto report = [&](float host_ms) {
            if (!timing) return;
            cudaEventSynchronize(ev.e[5]);
            auto ms = [&](int a, int b) { float t = 0.f; cudaEventElapsedTime(&t, ev.e[a], ev.e[b]); return t; };
            fprintf(stderr, "trb_scene_update_frame instances %zu builder %s\n", n, level ? "level" : "one-thread");
            fprintf(stderr, "trb_scene_update_frame host before the first launch %.3f ms\n", host_ms);
            fprintf(stderr, "trb_scene_update_frame k_frame_instances %.3f ms\n", ms(0, 1));
            if (level) {
                fprintf(stderr, "trb_scene_update_frame level loop %.3f ms\n", ms(1, 2));
                fprintf(stderr, "trb_scene_update_frame serial subtrees %.3f ms\n", ms(2, 3));
                fprintf(stderr, "trb_scene_update_frame numbering and emit %.3f ms\n", ms(3, 4));
                fprintf(stderr, "trb_scene_update_frame record packing %.3f ms\n", ms(4, 5));
            } else fprintf(stderr, "trb_scene_update_frame k_tlas_build %.3f ms\n", ms(1, 5));
            fprintf(stderr, "trb_scene_update_frame levels %u launches %llu\n", trace.levels, g_launches - launches0);
        };
        if (!s->instances_static_uploaded) { CU(cudaMemcpy(s->d_instances, di.data(), n * sizeof(trb::DInstance), cudaMemcpyHostToDevice)); s->instances_static_uploaded = true; }
        trb::FrameBuild fb{};
        fb.instances = s->d_instances; fb.bounds = reinterpret_cast<trbh::Box3*>(s->d_bounds); fb.n = (uint32_t)n;
        fb.shutter_open = s->shutter_open; fb.shutter_close = s->shutter_close;
        fb.cx = s->d_build_f; fb.cy = s->d_build_f + n; fb.cz = s->d_build_f + 2 * n;
        fb.idx = s->d_build_u; fb.task = s->d_build_u + n; fb.rec_of = s->d_build_u + 4 * n + 4;
        fb.nodes = s->d_tlas_nodes; fb.order = s->d_tlas_order; fb.counts = s->d_build_counts; fb.pairs = s->d_tlas; fb.hdr = s->d_tlas_hdr;
        // sized like the other frame buffers, by the capacity: a later frame of more instances within it runs in the same memory
        const uint32_t cap_n = (uint32_t)(s->tlas_capacity - 1), small = (uint32_t)s->tune.tlas_small;
        if (level && !s->d_build_level) CU(s->arena.alloc(LevelScratch(cap_n, small, nullptr).bytes, &s->d_build_level));
        const float host_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_host).count();
        mark(0);
        trb::k_frame_instances<<<(unsigned)((n + 63) / 64), 64>>>(s->ds, fb);
        ++g_launches;
        mark(1);
        uint32_t counts[4] = {0, 0, 0, 0};
        static const char* const not_buildable = "the instance tree cannot be built: an instance's bounds are infinite, NaN or beyond 2^126";
        if (!level) {
            trb::k_tlas_build<<<1, 1>>>(fb);
            ++g_launches;
            CU(cudaGetLastError());
        } else {
            const auto grid = [](size_t k) { return (unsigned)((k + 255) / 256); };
            const LevelScratch ls(cap_n, small, s->d_build_level);
            const uint32_t n32 = (uint32_t)n;
            bool empty = false;
            uint32_t n_nodes = 0;
            trace.after_levels = ev.e[2]; trace.after_small = ev.e[3];
            // bounds the build would not end on are refused inside it, before any serial subtree runs (trb_host.h bvh_bound_buildable)
            CU(trb::bvhb::build_device(s->d_bounds, n32, 4u /* scene.rs:141 */, s->d_build_counts, s->d_tlas_nodes, s->d_tlas_order, 0, &g_launches, &empty,
                                       small, &ls.own, &n_nodes, &trace, true));
            if (empty) { s->frame_ready = false; return fail(TRB_INVALID_ARG, not_buildable); }
            mark(4);
            // the child-pair records and the header, as k_tlas_build's tail writes them
            CU(cudaMemsetAsync(ls.narrow_bad, 0, 4, 0));
            trb::bvhb::k_pair_flags<<<grid((size_t)n_nodes + 1), 256>>>(s->d_tlas_nodes, n_nodes, ls.rec);
            size_t cub_bytes = ls.cub_bytes;
            CU(cub::DeviceScan::ExclusiveSum(ls.cub, cub_bytes, ls.rec, ls.rec, (int)n_nodes + 1, 0));
            trb::bvhb::k_pair_pack<<<grid(n_nodes), 256>>>(s->d_tlas_nodes, n_nodes, ls.rec, false, s->d_tlas, ls.narrow_bad);
            trb::bvhb::k_tlas_header<<<1, 1>>>(s->d_tlas_nodes, ls.rec, n_nodes, n32, ls.narrow_bad, s->d_tlas, s->d_tlas_hdr, s->d_build_counts);
            g_launches += 3;
            CU(cudaGetLastError());
        }
        mark(5);
        CU(cudaMemcpy(counts, s->d_build_counts, sizeof counts, cudaMemcpyDeviceToHost)); // also the frame's last synchronisation point
        report(host_ms);
        if (counts[3]) { s->frame_ready = false; return fail(TRB_INVALID_ARG, not_buildable); }
        if (!counts[2]) return fail(TRB_UNSUPPORTED, "too many instances for the leaf encoding");
        s->tlas_n_nodes = counts[0];
        s->host_frame_stale = true; // world transforms / TLAS nodes are fetched from the device when a getter asks for them
        s->frame_ready = true;
        return TRB_OK;
    }

    // ---- host path (kept for the DQuad experiment and as an independent check of the device path)
    s->world.resize(n);
    std::vector<Box3> bounds(n);
    for (size_t i = 0; i < n; ++i) {
        const trb_instance& in = s->instances[i];
        // world[i] = transform(shutter_open): exact for static instances; keyframed ones are re-evaluated per ray / per path on the device
        s->world[i] = trbh::animated_xf(s->splines.data(), in.spline_first, in.n_splines, s->keyframes.data(), s->knots.data(), s->shutter_open);
        const Box3 local = shape_bounds(*s, in);
        if (!trbh::xf_is_animated(s->splines.data(), in.spline_first, in.n_splines)) { // animation_bounds (animated_transform.rs:57-70, Q22)
            bounds[i] = arvo_bounds(s->world[i].fwd, local);
        } else {
            Box3 acc = box_empty();
            for (int k = 0; k < 128; ++k) {
                const float u = (float)k / 127.0f;
                const float time = s->shutter_open * (1.0f - u) + s->shutter_close * u; // linalg::lerp
                const Xf x = trbh::animated_xf(s->splines.data(), in.spline_first, in.n_splines, s->keyframes.data(), s->knots.data(), time);
                box_grow(acc, arvo_bounds(x.fwd, local));
            }
            bounds[i] = acc;
        }
        std::memcpy(di[i].inv, s->world[i].inv.m, 64);
        std::memcpy(di[i].mat, s->world[i].fwd.m, 64);
    }
    BvhBuilder bb;
    bb.build(bounds, 4);
    s->tlas_nodes = bb.nodes; s->tlas_order = bb.order;
    s->host_frame_stale = false; s->instances_static_uploaded = false;
    std::vector<trb::DPair> pn;
    trb::DBvh hdr{};
    if (!pack_pairs(s->tlas_nodes, pn, hdr)) return fail(TRB_UNSUPPORTED, "too many instances for the leaf encoding");
    std::vector<trb::DQuad> qn;
    uint32_t qroot = 0;
    if (!pack_quads(s->tlas_nodes, qn, qroot)) return fail(TRB_UNSUPPORTED, "too many instances for the leaf encoding");
    hdr.root_hi.w = bits_f(qroot);
    if (!pn.empty()) CU(cudaMemcpy(s->d_tlas, pn.data(), pn.size() * sizeof(trb::DPair), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_tlas_order, s->tlas_order.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_instances, di.data(), n * sizeof(trb::DInstance), cudaMemcpyHostToDevice));
    if (!qn.empty()) CU(cudaMemcpy(s->d_tlas_quads, qn.data(), qn.size() * sizeof(trb::DQuad), cudaMemcpyHostToDevice));
    hdr.pairs = s->d_tlas; hdr.quads = s->d_tlas_quads;
    CU(cudaMemcpy(s->d_tlas_hdr, &hdr, sizeof hdr, cudaMemcpyHostToDevice));
    s->frame_ready = true;
    return TRB_OK;
}

namespace {
// trb_render_device's body; aov: the AOV outputs of trb_render_aov_device (nullptr: none)
trb_status render_device(trb_scene* s, const trb_render_cfg* cfg, float* d_film, trb_stats* d_stats, cudaStream_t st, const AovRequest* aov) {
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering"); // scene.rs:179
    CU(cudaSetDevice(s->device));
    uint32_t spp, first, count, nb;
    const uint2* d_blocks = nullptr;
    trb_status r = resolve_samples(s, cfg, spp, first, count);
    if (r != TRB_OK) return r;
    r = ensure_blocks(s, cfg, &d_blocks, &nb);
    if (r != TRB_OK) return r;
    if (nb == 0 || count == 0) return TRB_OK; // "Warning: This block queue is empty!" (block_queue.rs:42-44)
    trb::RenderParams rp{};
    rp.blocks = d_blocks; rp.n_blocks = nb; rp.spp = spp; rp.sample_first = first; rp.sample_count = count; rp.seed = cfg->seed;
    rp.work_counter = s->d_counter; rp.film = reinterpret_cast<float4*>(d_film); rp.stats = reinterpret_cast<trb::DStats*>(d_stats);
    rp.error_flag = s->d_error;
    return launch_render(s, rp, cfg->flags, 0, st, aov);
}

// The AOV renders run the path integrator's wavefront only (DESIGN.md §4 "AOVs")
trb_status aov_supported(const trb_scene* s, const trb_render_cfg* cfg) {
    if (s->integrator.type != TRB_INTEGRATOR_PATH) return fail(TRB_UNSUPPORTED, "AOVs are rendered by the path integrator only");
    if (cfg->flags & TRB_RENDER_MEGAKERNEL) return fail(TRB_UNSUPPORTED, "AOVs are rendered on the wavefront pipeline only, not with TRB_RENDER_MEGAKERNEL");
    return TRB_OK;
}

// additive, like film::Image::add_pixels (image.rs:21-33); a 33 MB read-modify-write: split over a few host threads
void add_film(float* film, const float* src, size_t n) {
    const unsigned nt = n >= (1u << 20) ? std::min(8u, std::max(1u, std::thread::hardware_concurrency())) : 1u;
    auto add = [film, src](size_t a, size_t b) { for (size_t i = a; i < b; ++i) film[i] += src[i]; };
    std::vector<std::thread> th;
    for (unsigned k = 1; k < nt; ++k) th.emplace_back(add, n * k / nt, n * (k + 1) / nt);
    add(0, n / nt);
    for (auto& t : th) t.join();
}

// The device side of a host AOV render (trb_render_aov, trb_render_adaptive_aov): films from zero, added into the caller's
// afterwards; nearest from the caller's. lum_w (the *_lum renders) and motion_w (the *_motion renders, with dt): staged as albedo_w
// and normal_w.
struct HostAov {
    DeviceBuffer albedo, normal, nearest, lum, motion;
    AovRequest req{nullptr, nullptr, nullptr, nullptr};
    const trb_aov_film* aov = nullptr; // nullptr: no AOV output asked for
    float* lum_w = nullptr;
    float* motion_w = nullptr;
    trb_status stage(const trb_aov_film* a, size_t npx, float* lum_host = nullptr, float* motion_host = nullptr, float dt = 0.0f) {
        if (!a || !(a->albedo_w || a->normal_w || a->nearest || lum_host || motion_host)) return TRB_OK;
        aov = a;
        lum_w = lum_host;
        motion_w = motion_host;
        trb_status r;
        for (auto [h, d] : {std::pair<const float*, DeviceBuffer*>{a->albedo_w, &albedo}, {a->normal_w, &normal}, {lum_host, &lum},
                            {motion_host, &motion}}) {
            if (!h) continue;
            if ((r = d->alloc(npx * sizeof(float4), "AOV films")) != TRB_OK) return r;
            CU(cudaMemsetAsync(d->p, 0, npx * sizeof(float4), 0));
        }
        if (a->nearest) {
            if ((r = nearest.alloc(npx * sizeof(uint64_t), "AOV films")) != TRB_OK) return r;
            CU(cudaMemcpy(nearest.p, a->nearest, npx * sizeof(uint64_t), cudaMemcpyHostToDevice));
        }
        req = {nullptr, albedo.as<float4>(), normal.as<float4>(), nearest.as<unsigned long long>(), lum.as<float4>(), nullptr, motion.as<float4>(), dt};
        return TRB_OK;
    }
    const AovRequest* request() const { return aov ? &req : nullptr; }
    trb_status unstage(size_t npx) {
        if (!aov) return TRB_OK;
        std::vector<float> h;
        for (auto [dst, src] : {std::pair<float*, void*>{aov->albedo_w, albedo.p}, std::pair<float*, void*>{aov->normal_w, normal.p},
                                std::pair<float*, void*>{lum_w, lum.p}, std::pair<float*, void*>{motion_w, motion.p}}) {
            if (!dst) continue;
            h.resize(npx * 4);
            CU(cudaMemcpy(h.data(), src, npx * sizeof(float4), cudaMemcpyDeviceToHost));
            add_film(dst, h.data(), npx * 4);
        }
        if (aov->nearest) CU(cudaMemcpy(aov->nearest, nearest.p, npx * sizeof(uint64_t), cudaMemcpyDeviceToHost));
        return TRB_OK;
    }
};

// trb_render's body; aov: the host AOV outputs of trb_render_aov (nullptr: none)
trb_status render_host(trb_scene* s, const trb_render_cfg* cfg, float* film, const trb_aov_film* aov, trb_stats* stats, float* lum_w = nullptr,
                       float* motion_w = nullptr, float dt = 0.0f) {
    CU(cudaSetDevice(s->device));
    float update_ms = 0.f;
    if (!(cfg->flags & TRB_RENDER_NO_UPDATE)) { // Exec::render: scene.update_frame first (multithreaded.rs:57-60)
        auto t0 = std::chrono::steady_clock::now();
        const float step = s->film.scene_time / (float)s->film.frames;
        trb_status r = trb_scene_update_frame(s, cfg->current_frame, (float)cfg->current_frame * step, ((float)cfg->current_frame + 1.0f) * step);
        if (r != TRB_OK) return r;
        update_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    const size_t npx = (size_t)s->film.width * s->film.height;
    CU(cudaMemsetAsync(s->d_film, 0, npx * sizeof(float4), 0));
    CU(cudaMemsetAsync(s->d_stats, 0, sizeof(trb::DStats), 0));
    HostAov ha;
    trb_status r = ha.stage(aov, npx, lum_w, motion_w, dt);
    if (r != TRB_OK) return r;
    CU(cudaEventRecord(s->ev0, 0));
    r = render_device(s, cfg, reinterpret_cast<float*>(s->d_film), reinterpret_cast<trb_stats*>(s->d_stats), 0, ha.request());
    if (r != TRB_OK) { if (ha.aov) cudaDeviceSynchronize(); return r; } // passes already enqueued still write the AOV films
    CU(cudaEventRecord(s->ev1, 0));
    CU(cudaMemcpyAsync(s->h_film_staging, s->d_film, npx * sizeof(float4), cudaMemcpyDeviceToHost, 0));
    CU(cudaStreamSynchronize(0));
    r = check_error_flag(s);
    if (r != TRB_OK) return r;
    add_film(film, s->h_film_staging, npx * 4);
    if ((r = ha.unstage(npx)) != TRB_OK) return r;
    return stats_readback(s, stats, update_ms);
}

// trb_render_samples' body; aov: the host AOV records of trb_render_samples_aov (nullptr: none)
trb_status render_samples(trb_scene* s, const trb_render_cfg* cfg, size_t n, trb_sample* samples, trb_aov_sample* aov, trb_stats* stats,
                          trb_motion_sample* motion = nullptr, float dt = 0.0f) {
    CU(cudaSetDevice(s->device));
    uint32_t spp, first, count, nb;
    const uint2* d_blocks = nullptr;
    trb_status r = resolve_samples(s, cfg, spp, first, count);
    if (r != TRB_OK) return r;
    r = ensure_blocks(s, cfg, &d_blocks, &nb);
    if (r != TRB_OK) return r;
    if (n != (size_t)nb * 64 * count) return fail(TRB_INVALID_ARG, "sample buffer size must be blocks*64*sample_count");
    if (n == 0) return TRB_OK;
    trb::RenderParams rp{};
    rp.blocks = d_blocks; rp.n_blocks = nb; rp.spp = spp; rp.sample_first = first; rp.sample_count = count; rp.seed = cfg->seed;
    rp.work_counter = s->d_counter; rp.film = nullptr; rp.stats = s->d_stats; rp.error_flag = s->d_error;
    r = run_counted(s, {}, {{samples, n * sizeof(trb_sample)}, {aov, n * sizeof(trb_aov_sample)}, {motion, n * sizeof(trb_motion_sample)}},
                    [&](const DeviceBuffer* d) {
        rp.samples_out = d[0].as<trb_sample>();
        const AovRequest req{d[1].as<trb_aov_sample>(), nullptr, nullptr, nullptr, nullptr, d[2].as<trb_motion_sample>(), nullptr, dt};
        return launch_render(s, rp, cfg->flags, 1, 0, aov ? &req : nullptr);
    });
    return r != TRB_OK ? r : stats_readback(s, stats, 0.f);
}
} // namespace

trb_status trb_render_device(trb_scene* s, const trb_render_cfg* cfg, float* d_film, trb_stats* d_stats, void* stream) {
    if (!s || !cfg || !d_film) return fail(TRB_INVALID_ARG, "null argument");
    return render_device(s, cfg, d_film, d_stats, static_cast<cudaStream_t>(stream), nullptr);
}

trb_status trb_render(trb_scene* s, const trb_render_cfg* cfg, float* film, trb_stats* stats) {
    if (!s || !cfg || !film) return fail(TRB_INVALID_ARG, "null argument");
    return render_host(s, cfg, film, nullptr, stats);
}

trb_status trb_render_samples(trb_scene* s, const trb_render_cfg* cfg, size_t n, trb_sample* samples, trb_stats* stats) {
    if (!s || !cfg || !samples) return fail(TRB_INVALID_ARG, "null argument");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering");
    return render_samples(s, cfg, n, samples, nullptr, stats);
}

trb_status trb_render_aov_device(trb_scene* s, const trb_render_cfg* cfg, float* d_film, const trb_aov_film* d_aov, trb_stats* d_stats, void* stream) {
    if (!s || !cfg || !d_film || !d_aov) return fail(TRB_INVALID_ARG, "null argument");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering");
    trb_status r = aov_supported(s, cfg);
    if (r == TRB_OK)
        r = check_aligned({{d_film, 16}, {d_aov->albedo_w, 16}, {d_aov->normal_w, 16}, {d_aov->nearest, 8}},
                          "device films must be 16-byte aligned, the nearest buffer 8-byte aligned");
    if (r != TRB_OK) return r;
    const AovRequest req{nullptr, reinterpret_cast<float4*>(d_aov->albedo_w), reinterpret_cast<float4*>(d_aov->normal_w),
                         reinterpret_cast<unsigned long long*>(d_aov->nearest)};
    const bool with_aov = d_aov->albedo_w || d_aov->normal_w || d_aov->nearest;
    return render_device(s, cfg, d_film, d_stats, static_cast<cudaStream_t>(stream), with_aov ? &req : nullptr);
}

trb_status trb_render_aov(trb_scene* s, const trb_render_cfg* cfg, float* film, const trb_aov_film* aov, trb_stats* stats) {
    if (!s || !cfg || !film || !aov) return fail(TRB_INVALID_ARG, "null argument");
    const trb_status r = aov_supported(s, cfg);
    if (r != TRB_OK) return r;
    return render_host(s, cfg, film, aov, stats);
}

trb_status trb_render_samples_aov(trb_scene* s, const trb_render_cfg* cfg, size_t n, trb_sample* samples, trb_aov_sample* aov, trb_stats* stats) {
    if (!s || !cfg || !samples || !aov) return fail(TRB_INVALID_ARG, "null argument");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering");
    const trb_status r = aov_supported(s, cfg);
    if (r != TRB_OK) return r;
    return render_samples(s, cfg, n, samples, aov, stats);
}

trb_status trb_render_aov_lum_device(trb_scene* s, const trb_render_cfg* cfg, float* d_film, const trb_aov_film* d_aov, float* d_lum_w, trb_stats* d_stats,
                                     void* stream) {
    if (!s || !cfg || !d_film || !d_aov || !d_lum_w) return fail(TRB_INVALID_ARG, "null argument");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering");
    trb_status r = aov_supported(s, cfg);
    if (r == TRB_OK)
        r = check_aligned({{d_film, 16}, {d_aov->albedo_w, 16}, {d_aov->normal_w, 16}, {d_lum_w, 16}, {d_aov->nearest, 8}},
                          "device films must be 16-byte aligned, the nearest buffer 8-byte aligned");
    if (r != TRB_OK) return r;
    const AovRequest req{nullptr, reinterpret_cast<float4*>(d_aov->albedo_w), reinterpret_cast<float4*>(d_aov->normal_w),
                         reinterpret_cast<unsigned long long*>(d_aov->nearest), reinterpret_cast<float4*>(d_lum_w)};
    return render_device(s, cfg, d_film, d_stats, static_cast<cudaStream_t>(stream), &req);
}

trb_status trb_render_aov_lum(trb_scene* s, const trb_render_cfg* cfg, float* film, const trb_aov_film* aov, float* lum_w, trb_stats* stats) {
    if (!s || !cfg || !film || !aov || !lum_w) return fail(TRB_INVALID_ARG, "null argument");
    const trb_status r = aov_supported(s, cfg);
    if (r != TRB_OK) return r;
    return render_host(s, cfg, film, aov, stats, lum_w);
}

// ---- motion vectors (include/trb.h "Motion vectors") ----------------------------------------------------------------------------
namespace {
trb_status motion_dt(float dt) { return std::isfinite(dt) ? TRB_OK : fail(TRB_INVALID_ARG, "motion dt must be finite"); }
} // namespace

trb_status trb_render_aov_motion_device(trb_scene* s, const trb_render_cfg* cfg, float* d_film, const trb_aov_film* d_aov, float* d_lum_w, float* d_motion_w,
                                        float dt, trb_stats* d_stats, void* stream) {
    if (!s || !cfg || !d_film || !d_aov || !d_motion_w) return fail(TRB_INVALID_ARG, "null argument");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering");
    trb_status r = aov_supported(s, cfg);
    if (r == TRB_OK)
        r = check_aligned({{d_film, 16}, {d_aov->albedo_w, 16}, {d_aov->normal_w, 16}, {d_lum_w, 16}, {d_motion_w, 16}, {d_aov->nearest, 8}},
                          "device films must be 16-byte aligned, the nearest buffer 8-byte aligned");
    if (r == TRB_OK) r = motion_dt(dt);
    if (r != TRB_OK) return r;
    const AovRequest req{nullptr, reinterpret_cast<float4*>(d_aov->albedo_w), reinterpret_cast<float4*>(d_aov->normal_w),
                         reinterpret_cast<unsigned long long*>(d_aov->nearest), reinterpret_cast<float4*>(d_lum_w), nullptr,
                         reinterpret_cast<float4*>(d_motion_w), dt};
    return render_device(s, cfg, d_film, d_stats, static_cast<cudaStream_t>(stream), &req);
}

trb_status trb_render_aov_motion(trb_scene* s, const trb_render_cfg* cfg, float* film, const trb_aov_film* aov, float* lum_w, float* motion_w, float dt,
                                 trb_stats* stats) {
    if (!s || !cfg || !film || !aov || !motion_w) return fail(TRB_INVALID_ARG, "null argument");
    trb_status r = aov_supported(s, cfg);
    if (r == TRB_OK) r = motion_dt(dt);
    if (r != TRB_OK) return r;
    return render_host(s, cfg, film, aov, stats, lum_w, motion_w, dt);
}

trb_status trb_render_samples_aov_motion(trb_scene* s, const trb_render_cfg* cfg, size_t n, trb_sample* samples, trb_aov_sample* aov,
                                         trb_motion_sample* motion, float dt, trb_stats* stats) {
    if (!s || !cfg || !samples || !aov || !motion) return fail(TRB_INVALID_ARG, "null argument");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering");
    trb_status r = aov_supported(s, cfg);
    if (r == TRB_OK) r = motion_dt(dt);
    if (r != TRB_OK) return r;
    return render_samples(s, cfg, n, samples, aov, stats, motion, dt);
}

namespace {
// trb_denoise_params, NULL meaning the defaults (include/trb.h "Denoising"); checked before anything else, so no scene is needed
trb_status denoise_params(const trb_denoise_params* p, trb::DnParams& out) {
    const trb_denoise_params d = p ? *p : trb_denoise_params{5, 128, 4.0f, 1.0f};
    if (d.iterations > 10) return fail(TRB_INVALID_ARG, "denoise iterations must be 0 to 10");
    if (d.normal_power < 1 || d.normal_power > 1024 || (d.normal_power & (d.normal_power - 1)))
        return fail(TRB_INVALID_ARG, "denoise normal_power must be a power of two from 1 to 1024");
    if (!(d.sigma_luminance > 0.0f) || !std::isfinite(d.sigma_luminance)) return fail(TRB_INVALID_ARG, "denoise sigma_luminance must be finite and > 0");
    if (!(d.sigma_depth > 0.0f) || !std::isfinite(d.sigma_depth)) return fail(TRB_INVALID_ARG, "denoise sigma_depth must be finite and > 0");
    out.iterations = d.iterations;
    out.normal_squarings = (uint32_t)__builtin_ctz(d.normal_power);
    out.sigma_l = d.sigma_luminance; out.sigma_z = d.sigma_depth;
    return TRB_OK;
}

// The argument checks of both forms: parameters, null pointers, an output overlapping an input
trb_status denoise_check(const trb_scene* s, const trb_denoise_input* in, const trb_denoise_params* params, const float* out, trb::DnParams& prm) {
    const trb_status r = denoise_params(params, prm);
    if (r != TRB_OK) return r;
    if (!s || !in || !out || !in->colour_a || !in->colour_b || !in->albedo_w || !in->normal_w || !in->nearest) return fail(TRB_INVALID_ARG, "null argument");
    prm.width = (int)s->film.width; prm.height = (int)s->film.height;
    const size_t npx = (size_t)s->film.width * s->film.height, fb = npx * sizeof(float4);
    if (overlaps_any({out, fb}, {{in->colour_a, fb}, {in->colour_b, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}}))
        return fail(TRB_INVALID_ARG, "the denoise output overlaps an input");
    return TRB_OK;
}

// The scene's denoise scratch for the film's npx pixels, and with `mom` the moment records after it. The scratch is per scene and sized
// by the film; growing it drains the device once.
trb_status denoise_scratch(trb_scene* s, size_t npx, trb::DnScratch& sc, float4** mom = nullptr) {
    const size_t mom_off = (npx * trb::DN_BYTES_PER_PIXEL + 15) & ~(size_t)15;
    if (s->denoise_pixels < npx || (mom && !s->denoise_moments)) {
        if (s->d_denoise) {
            CU(cudaDeviceSynchronize()); // a denoise still in flight owns the old scratch
            cudaFree(s->d_denoise);
        }
        s->d_denoise = nullptr; s->denoise_pixels = 0; s->denoise_moments = false;
        const trb_status r = device_alloc(&s->d_denoise, mom ? mom_off + npx * sizeof(float4) : npx * trb::DN_BYTES_PER_PIXEL, "denoise scratch");
        if (r != TRB_OK) return r;
        s->denoise_pixels = npx; s->denoise_moments = mom != nullptr;
    }
    float4* base = static_cast<float4*>(s->d_denoise);
    sc = trb::DnScratch{base, base + npx, {base + 2 * npx, base + 3 * npx}, reinterpret_cast<float2*>(base + 4 * npx)};
    if (mom) *mom = reinterpret_cast<float4*>(static_cast<char*>(s->d_denoise) + mom_off);
    return TRB_OK;
}

// The N a-trous launches after k_dn_prepare or k_dn_temporal wrote the scratch
trb_status denoise_atrous(const trb::DnParams& prm, const trb::DnScratch& sc, float4* out, cudaStream_t st) {
    const dim3 block(32, 8), grid((prm.width + 31) / 32, (prm.height + 7) / 8);
    for (uint32_t i = 0; i < prm.iterations; ++i) {
        const bool last = i + 1 == prm.iterations;
        trb::k_dn_atrous<<<grid, block, 0, st>>>(prm, 1 << i, sc.guide, sc.grad, sc.divisor, sc.ev[i & 1], last ? nullptr : sc.ev[(i + 1) & 1],
                                                 last ? out : nullptr);
        g_launches++;
        CU(cudaGetLastError());
    }
    return TRB_OK;
}

// Enqueue the 1 + N denoise launches on `st`
trb_status denoise_enqueue(trb_scene* s, const trb::DnParams& prm, const trb_denoise_input& in, float* d_out, cudaStream_t st) {
    const size_t npx = (size_t)prm.width * prm.height;
    if (npx == 0) return TRB_OK;
    trb::DnScratch sc;
    const trb_status r = denoise_scratch(s, npx, sc);
    if (r != TRB_OK) return r;
    float4* out = reinterpret_cast<float4*>(d_out);
    const dim3 block(32, 8), grid((prm.width + 31) / 32, (prm.height + 7) / 8);
    trb::k_dn_prepare<<<grid, block, 0, st>>>(prm, reinterpret_cast<const float4*>(in.colour_a), reinterpret_cast<const float4*>(in.colour_b),
                                              reinterpret_cast<const float4*>(in.albedo_w), reinterpret_cast<const float4*>(in.normal_w),
                                              reinterpret_cast<const unsigned long long*>(in.nearest), sc, out);
    g_launches++;
    CU(cudaGetLastError());
    return denoise_atrous(prm, sc, out, st);
}
} // namespace

trb_status trb_denoise_device(trb_scene* s, const trb_denoise_input* d_in, const trb_denoise_params* params, float* d_out, void* stream) {
    trb::DnParams prm{};
    trb_status r = denoise_check(s, d_in, params, d_out, prm);
    if (r == TRB_OK)
        r = check_aligned({{d_in->colour_a, 16}, {d_in->colour_b, 16}, {d_in->albedo_w, 16}, {d_in->normal_w, 16}, {d_out, 16}, {d_in->nearest, 8}},
                          "device films must be 16-byte aligned, the nearest buffer 8-byte aligned");
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    return denoise_enqueue(s, prm, *d_in, d_out, static_cast<cudaStream_t>(stream));
}

trb_status trb_denoise(trb_scene* s, const trb_denoise_input* in, const trb_denoise_params* params, float* out) {
    trb::DnParams prm{};
    trb_status r = denoise_check(s, in, params, out, prm);
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)prm.width * prm.height, fb = npx * sizeof(float4);
    return run_staged({{in->colour_a, fb}, {in->colour_b, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}}, {{out, fb}},
                      [&](const DeviceBuffer* d) {
                          const trb_denoise_input d_in{d[0].as<float>(), d[1].as<float>(), d[2].as<float>(), d[3].as<float>(), d[4].as<uint64_t>()};
                          return denoise_enqueue(s, prm, d_in, d[5].as<float>(), 0);
                      });
}

// ---- sample-variance denoising (include/trb.h "Sample variance", DESIGN.md §4) -----------------------------------------------------
namespace {
// The checks of both forms: parameters, null pointers, an output overlapping an input or the other output
trb_status variance_check(const trb_scene* s, const trb_denoise_frame* in, const float* lum_w, const trb_denoise_params* params, const float* rgbw,
                          const float* variance, trb::DnParams& prm) {
    const trb_status r = denoise_params(params, prm);
    if (r != TRB_OK) return r;
    if (!s || !in || !lum_w || !rgbw || !in->colour || !in->albedo_w || !in->normal_w || !in->nearest) return fail(TRB_INVALID_ARG, "null argument");
    prm.width = (int)s->film.width; prm.height = (int)s->film.height;
    const size_t npx = (size_t)s->film.width * s->film.height, fb = npx * sizeof(float4);
    for (const Span o : {Span{rgbw, fb}, Span{variance, npx * sizeof(float)}})
        if (overlaps_any(o, {{in->colour, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}, {lum_w, fb}}))
            return fail(TRB_INVALID_ARG, "the denoise output overlaps an input");
    if (spans_overlap({rgbw, fb}, {variance, npx * sizeof(float)})) return fail(TRB_INVALID_ARG, "the denoise outputs overlap");
    return TRB_OK;
}

// k_dn_variance_prepare and the N a-trous launches on `st`
trb_status variance_enqueue(trb_scene* s, const trb::DnParams& prm, const trb_denoise_frame& in, const float* lum_w, float* d_rgbw, float* d_var,
                            cudaStream_t st) {
    const size_t npx = (size_t)prm.width * prm.height;
    if (npx == 0) return TRB_OK;
    trb::DnScratch sc;
    const trb_status r = denoise_scratch(s, npx, sc);
    if (r != TRB_OK) return r;
    float4* out = reinterpret_cast<float4*>(d_rgbw);
    const dim3 block(32, 8), grid((prm.width + 31) / 32, (prm.height + 7) / 8);
    trb::k_dn_variance_prepare<<<grid, block, 0, st>>>(prm, reinterpret_cast<const float4*>(in.colour), reinterpret_cast<const float4*>(lum_w),
                                                       reinterpret_cast<const float4*>(in.albedo_w), reinterpret_cast<const float4*>(in.normal_w),
                                                       reinterpret_cast<const unsigned long long*>(in.nearest), sc, out, d_var);
    g_launches++;
    CU(cudaGetLastError());
    return denoise_atrous(prm, sc, out, st);
}
} // namespace

trb_status trb_denoise_variance_device(trb_scene* s, const trb_denoise_frame* d_in, const float* d_lum_w, const trb_denoise_params* params, float* d_rgbw,
                                       float* d_variance, void* stream) {
    trb::DnParams prm{};
    trb_status r = variance_check(s, d_in, d_lum_w, params, d_rgbw, d_variance, prm);
    if (r == TRB_OK)
        r = check_aligned({{d_in->colour, 16}, {d_in->albedo_w, 16}, {d_in->normal_w, 16}, {d_lum_w, 16}, {d_rgbw, 16}, {d_in->nearest, 8}, {d_variance, 4}},
                          "device films must be 16-byte aligned, the nearest buffer 8-byte aligned, variance 4-byte aligned");
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    return variance_enqueue(s, prm, *d_in, d_lum_w, d_rgbw, d_variance, static_cast<cudaStream_t>(stream));
}

trb_status trb_denoise_variance(trb_scene* s, const trb_denoise_frame* in, const float* lum_w, const trb_denoise_params* params, float* rgbw, float* variance) {
    trb::DnParams prm{};
    trb_status r = variance_check(s, in, lum_w, params, rgbw, variance, prm);
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)prm.width * prm.height, fb = npx * sizeof(float4);
    return run_staged({{in->colour, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}, {lum_w, fb}},
                      {{rgbw, fb}, {variance, npx * sizeof(float)}}, [&](const DeviceBuffer* d) {
                          return variance_enqueue(s, prm, {d[0].as<float>(), d[1].as<float>(), d[2].as<float>(), d[3].as<uint64_t>()}, d[4].as<float>(),
                                                  d[5].as<float>(), d[6].as<float>(), 0);
                      });
}

// ---- temporal denoising (include/trb.h "Temporal denoising", DESIGN.md §4) -------------------------------------------------------
// The history families: what a set's records hold. A call finds no history in a set written by another family.
enum DnFamily : uint8_t {
    DN_HALVES,   // trb_denoise_temporal*: (ē_a, z), (ē_b, inst)
    DN_MOMENTS,  // trb_denoise_moments*: (ē, z), (mu1, mu2, 0, inst)
    DN_VARIANCE, // trb_denoise_variance_temporal*: (ē, z), (V, 0, 0, inst)
};

// Two per-pixel history sets (trb::DnHistory, 48 B per pixel each) and two instance snapshots (64 B per instance each); `cur` is the
// set the next call reads. The host fields describe the frame the read set was written at.
struct trb_denoise_history {
    trb_scene* scene = nullptr;
    int device = 0;
    void* d_px = nullptr;          // 2 sets x 3 float4 arrays of px_capacity pixels
    size_t px_capacity = 0;
    float* d_mats = nullptr;       // 2 sets x mat_capacity x 16 floats
    size_t mat_capacity = 0;
    uint32_t cur = 0;
    bool bound = false;            // the film size is taken (first call after create / reset)
    uint32_t width = 0, height = 0;
    bool has_prev = false;         // the read set holds a frame
    float cam_inv[16] = {}, tan_fov = 0;
    uint32_t n_instances = 0;
    uint64_t generation = 0;
    DnFamily family = DN_HALVES;   // the family of the calls that wrote the read set
    // temporal gradients: two record sets and the per-call stratum buffers (trb::GrBuffers) for gr_capacity strata; the records of
    // the read set are valid only after a gradient call, and were written at gr_seed, gr_shutter_open and gr_cam_mat
    void* d_gr = nullptr;
    size_t gr_capacity = 0;
    bool gr_valid = false;
    uint32_t gr_seed = 0;
    float gr_shutter_open = 0, gr_cam_mat[16] = {};
    ~trb_denoise_history() {
        if (d_px) cudaFree(d_px);
        if (d_mats) cudaFree(d_mats);
        if (d_gr) cudaFree(d_gr);
    }
    trb::DnHistory set(uint32_t k) const {
        float4* base = static_cast<float4*>(d_px) + (size_t)k * 3 * px_capacity;
        return trb::DnHistory{base, base + px_capacity, base + 2 * px_capacity};
    }
};

trb_status trb_denoise_history_create(trb_scene* s, trb_denoise_history** out) {
    if (!s || !out) return fail(TRB_INVALID_ARG, "null argument");
    trb_denoise_history* h = new (std::nothrow) trb_denoise_history();
    if (!h) return fail(TRB_OOM, "denoise history");
    h->scene = s; h->device = s->device;
    *out = h;
    return TRB_OK;
}

trb_status trb_denoise_history_destroy(trb_denoise_history* h) {
    if (!h) return TRB_OK;
    cudaSetDevice(h->device);
    delete h; // cudaFree waits for the calls still reading the buffers
    return TRB_OK;
}

trb_status trb_denoise_history_reset(trb_denoise_history* h) {
    if (!h) return fail(TRB_INVALID_ARG, "null history");
    h->has_prev = false; h->bound = false; h->width = h->height = 0; h->gr_valid = false;
    return TRB_OK;
}

namespace {
// trb_denoise_temporal_params, NULL meaning the defaults; checked before anything else
trb_status temporal_params(const trb_denoise_temporal_params* p, trb::DnParams& prm, trb::DnTemporal& tp) {
    const trb_status r = denoise_params(p ? &p->spatial : nullptr, prm);
    if (r != TRB_OK) return r;
    const uint32_t max_history = p ? p->max_history : 8u;
    const float depth_tolerance = p ? p->depth_tolerance : 0.05f, normal_threshold = p ? p->normal_threshold : 0.9f;
    if (max_history < 1 || max_history > 255) return fail(TRB_INVALID_ARG, "temporal denoise max_history must be 1 to 255");
    if (!(depth_tolerance > 0.0f) || !std::isfinite(depth_tolerance)) return fail(TRB_INVALID_ARG, "temporal denoise depth_tolerance must be finite and > 0");
    if (!(normal_threshold >= -1.0f && normal_threshold <= 1.0f)) return fail(TRB_INVALID_ARG, "temporal denoise normal_threshold must be in [-1, 1]");
    tp.max_history = max_history; tp.depth_tolerance = depth_tolerance; tp.normal_threshold = normal_threshold;
    return TRB_OK;
}

// The checks shared by the half-film and moment calls after their parameters and null pointers: outputs outs[first..] overlapping an
// input or an earlier output, the history's scene and film size, a frame
trb_status history_call_check(const trb_scene* s, const trb_denoise_history* h, const Span* ins, size_t nin, const Span* outs, size_t nout,
                              size_t first) {
    for (size_t k = first; k < nout; ++k) {
        for (size_t j = 0; j < nin; ++j)
            if (spans_overlap(outs[k], ins[j]))
                return fail(TRB_INVALID_ARG, k == 0 ? "the denoise output overlaps an input" : "a temporal denoise output overlaps an input");
        for (size_t j = 0; j < k; ++j)
            if (spans_overlap(outs[k], outs[j]))
                return fail(TRB_INVALID_ARG, "two temporal denoise outputs overlap");
    }
    if (h->scene != s) return fail(TRB_INVALID_ARG, "the denoise history belongs to another scene");
    if (h->bound && (h->width != s->film.width || h->height != s->film.height))
        return fail(TRB_INVALID_ARG, "the denoise history was written at another film size: reset it");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "update_frame must be called before a temporal denoise");
    return TRB_OK;
}

// The checks of both forms after the parameters: null pointers, the history's scene and film size, a frame, overlapping outputs
trb_status temporal_check(const trb_scene* s, const trb_denoise_history* h, const trb_denoise_input* in, const trb_denoise_temporal_params* params,
                          const trb_denoise_temporal_output* out, trb::DnParams& prm, trb::DnTemporal& tp) {
    trb_status r = temporal_params(params, prm, tp);
    if (r != TRB_OK) return r;
    if (!s || !h || !in || !out || !out->rgbw) return fail(TRB_INVALID_ARG, "null argument");
    r = denoise_check(s, in, params ? &params->spatial : nullptr, out->rgbw, prm);
    if (r != TRB_OK) return r;
    const size_t npx = (size_t)s->film.width * s->film.height;
    const Span ins[5] = {{in->colour_a, npx * sizeof(float4)}, {in->colour_b, npx * sizeof(float4)}, {in->albedo_w, npx * sizeof(float4)},
                         {in->normal_w, npx * sizeof(float4)}, {in->nearest, npx * sizeof(uint64_t)}};
    const Span outs[3] = {{out->rgbw, npx * sizeof(float4)}, {out->motion, npx * sizeof(float2)}, {out->history_length, npx * sizeof(uint32_t)}};
    return history_call_check(s, h, ins, 5, outs, 3, 1); // denoise_check tested rgbw
}

// The gradient buffers of G strata, carved out of one allocation at 256-byte offsets: two record sets (64 B per stratum each), the
// winner slots, the re-shade rays and radiance, the record query and illumination rays, their hits and radiance, two (delta, m, c)
// buffers, the stratum guides and lambda: 456 B per stratum
struct GrBuffers {
    float4* rec[2];
    unsigned long long* slot;
    trb_illum_ray* reshade;
    float* reshade_rgb;
    trb_query_ray* qrays;
    trb_illum_ray* irays;
    trb_intersection* hits;
    float* rgb;
    float4* dm[2];
    float4* guide;
    float* lam;
};
size_t gr_layout(size_t G, char* base, GrBuffers* b) {
    size_t off = 0;
    auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += (bytes + 255) & ~(size_t)255; return p; };
    char* r0 = take(G * 64); char* r1 = take(G * 64); char* sl = take(G * 8); char* rs = take(G * sizeof(trb_illum_ray));
    char* rsc = take(G * 12); char* q = take(G * sizeof(trb_query_ray)); char* il = take(G * sizeof(trb_illum_ray));
    char* hi = take(G * sizeof(trb_intersection)); char* rgb = take(G * 12); char* d0 = take(G * 16); char* d1 = take(G * 16);
    char* gd = take(G * 16); char* lm = take(G * 4);
    if (b) *b = GrBuffers{{reinterpret_cast<float4*>(r0), reinterpret_cast<float4*>(r1)}, reinterpret_cast<unsigned long long*>(sl),
                          reinterpret_cast<trb_illum_ray*>(rs), reinterpret_cast<float*>(rsc), reinterpret_cast<trb_query_ray*>(q),
                          reinterpret_cast<trb_illum_ray*>(il), reinterpret_cast<trb_intersection*>(hi), reinterpret_cast<float*>(rgb),
                          {reinterpret_cast<float4*>(d0), reinterpret_cast<float4*>(d1)}, reinterpret_cast<float4*>(gd), reinterpret_cast<float*>(lm)};
    return off;
}

// A gradient call's own arguments (trb_denoise_temporal_gradient*, trb_denoise_moments_gradient*)
struct GradCall {
    uint32_t iterations;
    uint32_t seed;
    float* lambda;   // per-pixel output, may be null
};

// Steps 1-2 of "Temporal gradients": re-shade the read set's records in this frame, reconstruct lambda on the stratum grid into b.lam.
// nearest and normal_w are the frame's AOVs (trb_denoise_input's or trb_denoise_frame's).
trb_status gradient_lambda(trb_scene* s, trb_denoise_history* h, const GradCall& gc, const trb::DnTemporal& tp, const GrBuffers& b,
                           const float* mats_rd, const uint64_t* nearest_in, const float* normal_w, bool valid, cudaStream_t st) {
    const uint32_t W = s->film.width, H = s->film.height, gw = (W + 2) / 3, gh = (H + 2) / 3, S = gw * gh;
    const unsigned grid = (unsigned)std::min<size_t>((S + 255) / 256, (size_t)s->sm_count * 8);
    trb::GrFrame f{};
    std::memcpy(f.cam_mat, s->ds.cam.cam_mat, 64);
    std::memcpy(f.cam_inv, s->cam_inv, 64);
    f.tan_cur = s->ds.cam.scaling[0];
    f.x0 = tp.x0; f.x1 = tp.x1; f.y0 = tp.y0; f.y1 = tp.y1; f.w = (float)W; f.h = (float)H;
    f.width = W; f.height = H; f.gw = gw; f.gh = gh;
    f.n_cur = tp.n_cur; f.n_prev = valid ? tp.n_prev : 0u;
    f.cam_same = std::memcmp(h->gr_cam_mat, s->ds.cam.cam_mat, 64) == 0 ? 1u : 0u;
    f.dt = s->shutter_open - h->gr_shutter_open;
    f.depth_tolerance = tp.depth_tolerance; f.normal_threshold = tp.normal_threshold;
    const float4* rec = b.rec[h->cur];
    const unsigned long long* nearest = reinterpret_cast<const unsigned long long*>(nearest_in);
    CU(cudaMemsetAsync(b.slot, 0xff, (size_t)S * 8, st));
    if (valid) {
        trb::k_gr_project<<<grid, 256, 0, st>>>(f, rec, s->d_instances, nearest, b.slot);
        g_launches++;
    }
    trb::k_gr_resolve<<<grid, 256, 0, st>>>(f, rec, s->d_instances, mats_rd, b.slot, reinterpret_cast<const float4*>(normal_w), nearest, b.reshade,
                                            b.guide);
    g_launches++;
    CU(cudaGetLastError());
    if (valid) {
        const trb_status r = illum_passes(s, S, b.reshade, 1, h->gr_seed, b.reshade_rgb, TRB_QUERY_CLAMP, nullptr, st);
        if (r != TRB_OK) return r;
    } else {
        CU(cudaMemsetAsync(b.reshade_rgb, 0, (size_t)S * 12, st));
    }
    trb::k_gr_delta<<<grid, 256, 0, st>>>(S, rec, b.slot, b.reshade_rgb, b.dm[0], gc.iterations == 0 ? b.lam : nullptr);
    g_launches++;
    for (uint32_t i = 0; i < gc.iterations; ++i) {
        const bool last = i + 1 == gc.iterations;
        trb::k_gr_atrous<<<grid, 256, 0, st>>>(gw, gh, 1 << i, tp.normal_threshold, b.guide, b.dm[i & 1], last ? nullptr : b.dm[(i + 1) & 1],
                                               last ? b.lam : nullptr);
        g_launches++;
    }
    CU(cudaGetLastError());
    return TRB_OK;
}

// After step 4: the write set's records are valid, written at the call's seed and this frame's shutter_open and camera
void gradient_commit(const trb_scene* s, trb_denoise_history* h, const GradCall& gc) {
    h->gr_valid = true; h->gr_seed = gc.seed; h->gr_shutter_open = s->shutter_open;
    std::memcpy(h->gr_cam_mat, s->ds.cam.cam_mat, 64);
}

// Step 4: this frame's samples into the write set's records
trb_status gradient_record(trb_scene* s, const GradCall& gc, const GrBuffers& b, uint32_t wr, cudaStream_t st) {
    const uint32_t W = s->film.width, H = s->film.height, gw = (W + 2) / 3, gh = (H + 2) / 3, S = gw * gh;
    const unsigned grid = (unsigned)std::min<size_t>((S + 255) / 256, (size_t)s->sm_count * 8);
    if (s->ds.has_anim) trb::k_gr_record<true><<<grid, 256, 0, st>>>(s->ds, gw, gh, gc.seed, b.qrays, b.irays);
    else trb::k_gr_record<false><<<grid, 256, 0, st>>>(s->ds, gw, gh, gc.seed, b.qrays, b.irays);
    g_launches++;
    CU(cudaGetLastError());
    trb_status r = query_passes(s, S, b.qrays, b.hits, nullptr, 0u, nullptr, st);
    if (r != TRB_OK) return r;
    r = illum_passes(s, S, b.irays, 1, gc.seed, b.rgb, TRB_QUERY_CLAMP, nullptr, st);
    if (r != TRB_OK) return r;
    trb::k_gr_store<<<grid, 256, 0, st>>>(S, b.hits, b.irays, b.rgb, s->d_instances, b.rec[wr]);
    g_launches++;
    CU(cudaGetLastError());
    return TRB_OK;
}

// The sets and snapshots of a history call: the one read, the one written, and the matrices of each
struct HistorySets {
    uint32_t rd, wr;
    float* mats_rd;
};

// What a history call does before its kernels, for npx > 0 pixels: grow the history (and, with gc, its gradient buffers) where
// needed, fill tp's current frame and the read set's snapshot (has_prev only for a history of the call's family), and copy this
// frame's instance transforms into the write snapshot on `st`
trb_status history_begin(trb_scene* s, trb_denoise_history* h, const trb::DnParams& prm, trb::DnTemporal& tp, DnFamily family, const GradCall* gc,
                         HistorySets& hs, cudaStream_t st) {
    const size_t npx = (size_t)prm.width * prm.height, n = s->instances.size();
    trb_status r;
    // the pixel sets are bound to one film size, so they only grow while the history is empty: nothing to keep. A new buffer is
    // allocated before the old one is released, so a failure leaves the history as it was.
    if (h->px_capacity < npx) {
        void* p = nullptr;
        r = device_alloc(&p, 2 * 3 * npx * sizeof(float4), "denoise history");
        if (r != TRB_OK) return r;
        if (h->d_px) { CU(cudaDeviceSynchronize()); cudaFree(h->d_px); } // a call still in flight owns the old sets
        h->d_px = p; h->px_capacity = npx; h->has_prev = false;
    }
    if (h->mat_capacity < n) { // both snapshots, the read one copied to its place in the new buffer
        void* p = nullptr;
        r = device_alloc(&p, 2 * n * 16 * sizeof(float), "denoise history snapshot");
        if (r != TRB_OK) return r;
        if (h->d_mats) {
            CU(cudaDeviceSynchronize());
            const size_t rows = std::min<size_t>(h->n_instances, h->mat_capacity);
            if (rows)
                CU(cudaMemcpy(static_cast<float*>(p) + (size_t)h->cur * n * 16, h->d_mats + (size_t)h->cur * h->mat_capacity * 16, rows * 64,
                              cudaMemcpyDeviceToDevice));
            cudaFree(h->d_mats);
        }
        h->d_mats = static_cast<float*>(p); h->mat_capacity = n;
    }
    const size_t S = (size_t)((prm.width + 2) / 3) * ((prm.height + 2) / 3);
    if (gc && h->gr_capacity < S) { // like the pixel sets: bound to one film size, so the records are not kept
        void* p = nullptr;
        r = device_alloc(&p, gr_layout(S, nullptr, nullptr), "denoise history gradients");
        if (r != TRB_OK) return r;
        if (h->d_gr) { CU(cudaDeviceSynchronize()); cudaFree(h->d_gr); }
        h->d_gr = p; h->gr_capacity = S; h->gr_valid = false;
    }
    // the current frame, and the snapshot the read set was written at
    std::memcpy(tp.px_to_cam, s->ds.cam.px_to_cam, 64);
    std::memcpy(tp.cam_mat, s->ds.cam.cam_mat, 64);
    std::memcpy(tp.scaling, s->ds.cam.scaling, 12);
    tp.n_cur = (uint32_t)n;
    std::memcpy(tp.cam_inv_prev, h->cam_inv, 64);
    tp.tan_prev = h->tan_fov;
    tp.w_prev = (float)prm.width; tp.h_prev = (float)prm.height;
    const float aspect = (float)s->film.width / (float)s->film.height; // camera_setup's screen window
    if (aspect > 1.0f) { tp.x0 = -aspect; tp.x1 = aspect; tp.y0 = -1.0f; tp.y1 = 1.0f; }
    else { tp.x0 = -1.0f; tp.x1 = 1.0f; tp.y0 = -1.0f / aspect; tp.y1 = 1.0f / aspect; }
    tp.n_prev = h->n_instances;
    tp.has_prev = h->has_prev && h->generation == s->object_generation && h->family == family ? 1u : 0u;
    hs.rd = h->cur; hs.wr = h->cur ^ 1u;
    hs.mats_rd = h->d_mats + (size_t)hs.rd * h->mat_capacity * 16;
    float* mats_wr = h->d_mats + (size_t)hs.wr * h->mat_capacity * 16;
    // this frame's object -> world matrices into the write snapshot: DInstance.mat, 64-byte rows at the records' 208-byte pitch
    CU(cudaMemcpy2DAsync(mats_wr, 64, reinterpret_cast<const char*>(s->d_instances) + offsetof(trb::DInstance, mat), sizeof(trb::DInstance), 64, n,
                         cudaMemcpyDeviceToDevice, st));
    return TRB_OK;
}

// After a history call's kernels: the history switches to the set just written, and the snapshot becomes the current frame's
void history_commit(trb_scene* s, trb_denoise_history* h, const HistorySets& hs, DnFamily family) {
    h->cur = hs.wr; h->has_prev = true; h->bound = true; h->width = s->film.width; h->height = s->film.height;
    std::memcpy(h->cam_inv, s->cam_inv, 64);
    h->tan_fov = s->ds.cam.scaling[0];
    h->n_instances = (uint32_t)s->instances.size();
    h->generation = s->object_generation;
    h->family = family;
}

// k_dn_temporal (or, with gc, the gradient steps around k_dn_temporal_grad) and the a-trous launches on `st`, then the history's
// switch to the set just written
trb_status temporal_enqueue(trb_scene* s, trb_denoise_history* h, trb::DnParams& prm, trb::DnTemporal& tp, const trb_denoise_input& in,
                            const trb_denoise_temporal_output& out, cudaStream_t st, const GradCall* gc = nullptr) {
    const size_t npx = (size_t)prm.width * prm.height;
    if (npx == 0) return TRB_OK;
    trb::DnScratch sc;
    trb_status r = denoise_scratch(s, npx, sc);
    if (r != TRB_OK) return r;
    HistorySets hs;
    r = history_begin(s, h, prm, tp, DN_HALVES, gc, hs, st);
    if (r != TRB_OK) return r;
    const uint32_t rd = hs.rd, wr = hs.wr;
    const float* mats_rd = hs.mats_rd;
    float4* rgbw = reinterpret_cast<float4*>(out.rgbw);
    const dim3 block(32, 8), grid((prm.width + 31) / 32, (prm.height + 7) / 8);
    if (!gc) {
        trb::k_dn_temporal<<<grid, block, 0, st>>>(prm, tp, reinterpret_cast<const float4*>(in.colour_a), reinterpret_cast<const float4*>(in.colour_b),
                                                   reinterpret_cast<const float4*>(in.albedo_w), reinterpret_cast<const float4*>(in.normal_w),
                                                   reinterpret_cast<const unsigned long long*>(in.nearest), sc, rgbw, s->d_instances, mats_rd,
                                                   h->set(rd), h->set(wr), reinterpret_cast<float2*>(out.motion), out.history_length);
        g_launches++;
        CU(cudaGetLastError());
        r = denoise_atrous(prm, sc, rgbw, st);
        if (r != TRB_OK) return r;
        h->gr_valid = false;
    } else {
        GrBuffers b;
        gr_layout(h->gr_capacity, static_cast<char*>(h->d_gr), &b);
        const bool valid = tp.has_prev && h->gr_valid;
        r = gradient_lambda(s, h, *gc, tp, b, mats_rd, in.nearest, in.normal_w, valid, st);
        if (r != TRB_OK) return r;
        trb::k_dn_temporal_grad<<<grid, block, 0, st>>>(prm, tp, reinterpret_cast<const float4*>(in.colour_a), reinterpret_cast<const float4*>(in.colour_b),
                                                        reinterpret_cast<const float4*>(in.albedo_w), reinterpret_cast<const float4*>(in.normal_w),
                                                        reinterpret_cast<const unsigned long long*>(in.nearest), sc, rgbw, s->d_instances, mats_rd,
                                                        h->set(rd), h->set(wr), reinterpret_cast<float2*>(out.motion), out.history_length, b.lam,
                                                        (uint32_t)((prm.width + 2) / 3), gc->lambda);
        g_launches++;
        CU(cudaGetLastError());
        r = denoise_atrous(prm, sc, rgbw, st);
        if (r != TRB_OK) return r;
        r = gradient_record(s, *gc, b, wr, st);
        if (r != TRB_OK) return r;
        gradient_commit(s, h, *gc);
    }
    history_commit(s, h, hs, DN_HALVES);
    return TRB_OK;
}
} // namespace

trb_status trb_denoise_temporal_device(trb_scene* s, trb_denoise_history* h, const trb_denoise_input* d_in, const trb_denoise_temporal_params* params,
                                       const trb_denoise_temporal_output* d_out, void* stream) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    trb_status r = temporal_check(s, h, d_in, params, d_out, prm, tp);
    if (r == TRB_OK)
        r = check_aligned({{d_in->colour_a, 16}, {d_in->colour_b, 16}, {d_in->albedo_w, 16}, {d_in->normal_w, 16}, {d_out->rgbw, 16}, {d_in->nearest, 8},
                           {d_out->motion, 8}, {d_out->history_length, 4}},
                          "device films must be 16-byte aligned, nearest and motion 8-byte, history_length 4-byte");
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    return temporal_enqueue(s, h, prm, tp, *d_in, *d_out, static_cast<cudaStream_t>(stream));
}

trb_status trb_denoise_temporal(trb_scene* s, trb_denoise_history* h, const trb_denoise_input* in, const trb_denoise_temporal_params* params,
                                const trb_denoise_temporal_output* out) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    trb_status r = temporal_check(s, h, in, params, out, prm, tp);
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)prm.width * prm.height, fb = npx * sizeof(float4);
    return run_staged({{in->colour_a, fb}, {in->colour_b, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}},
                      {{out->rgbw, fb}, {out->motion, npx * sizeof(float2)}, {out->history_length, npx * sizeof(uint32_t)}}, [&](const DeviceBuffer* d) {
                          const trb_denoise_input d_in{d[0].as<float>(), d[1].as<float>(), d[2].as<float>(), d[3].as<float>(), d[4].as<uint64_t>()};
                          return temporal_enqueue(s, h, prm, tp, d_in, {d[5].as<float>(), d[6].as<float>(), d[7].as<uint32_t>()}, 0);
                      });
}

namespace {
// trb_denoise_gradient_params, NULL meaning the defaults; checked before anything else
trb_status gradient_check(const trb_scene* s, const trb_denoise_history* h, const trb_denoise_input* in, const trb_denoise_gradient_params* params,
                          const trb_denoise_gradient_output* out, trb::DnParams& prm, trb::DnTemporal& tp, GradCall& gc) {
    const uint32_t iterations = params ? params->iterations : 3u;
    trb_status r = temporal_params(params ? &params->temporal : nullptr, prm, tp);
    if (r != TRB_OK) return r;
    if (iterations > 6) return fail(TRB_INVALID_ARG, "temporal gradient iterations must be 0 to 6");
    if (!out) return fail(TRB_INVALID_ARG, "null argument");
    const trb_denoise_temporal_output o{out->rgbw, out->motion, out->history_length};
    r = temporal_check(s, h, in, params ? &params->temporal : nullptr, &o, prm, tp);
    if (r != TRB_OK) return r;
    const size_t npx = (size_t)s->film.width * s->film.height, fb = npx * sizeof(float4);
    if (overlaps_any({out->lambda, npx * sizeof(float)}, {{in->colour_a, fb}, {in->colour_b, fb}, {in->albedo_w, fb}, {in->normal_w, fb},
                                                          {in->nearest, npx * sizeof(uint64_t)}, {out->rgbw, fb}, {out->motion, npx * sizeof(float2)},
                                                          {out->history_length, npx * sizeof(uint32_t)}}))
        return fail(TRB_INVALID_ARG, "the lambda output overlaps another buffer");
    gc.iterations = iterations;
    gc.lambda = out->lambda;
    return TRB_OK;
}
} // namespace

trb_status trb_denoise_temporal_gradient_device(trb_scene* s, trb_denoise_history* h, const trb_denoise_input* d_in,
                                                const trb_denoise_gradient_params* params, uint32_t seed, const trb_denoise_gradient_output* d_out,
                                                void* stream) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    GradCall gc{};
    trb_status r = gradient_check(s, h, d_in, params, d_out, prm, tp, gc);
    if (r == TRB_OK)
        r = check_aligned({{d_in->colour_a, 16}, {d_in->colour_b, 16}, {d_in->albedo_w, 16}, {d_in->normal_w, 16}, {d_out->rgbw, 16}, {d_in->nearest, 8},
                           {d_out->motion, 8}, {d_out->history_length, 4}, {d_out->lambda, 4}},
                          "device films must be 16-byte aligned, nearest and motion 8-byte, history_length and lambda 4-byte");
    if (r != TRB_OK) return r;
    gc.seed = seed;
    CU(cudaSetDevice(s->device));
    const trb_denoise_temporal_output o{d_out->rgbw, d_out->motion, d_out->history_length};
    return temporal_enqueue(s, h, prm, tp, *d_in, o, static_cast<cudaStream_t>(stream), &gc);
}

trb_status trb_denoise_temporal_gradient(trb_scene* s, trb_denoise_history* h, const trb_denoise_input* in, const trb_denoise_gradient_params* params,
                                         uint32_t seed, const trb_denoise_gradient_output* out) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    GradCall gc{};
    trb_status r = gradient_check(s, h, in, params, out, prm, tp, gc);
    if (r != TRB_OK) return r;
    gc.seed = seed;
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)prm.width * prm.height, fb = npx * sizeof(float4);
    return run_staged({{in->colour_a, fb}, {in->colour_b, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}},
                      {{out->rgbw, fb}, {out->motion, npx * sizeof(float2)}, {out->history_length, npx * sizeof(uint32_t)}, {out->lambda, npx * sizeof(float)}},
                      [&](const DeviceBuffer* d) {
                          const trb_denoise_input d_in{d[0].as<float>(), d[1].as<float>(), d[2].as<float>(), d[3].as<float>(), d[4].as<uint64_t>()};
                          gc.lambda = d[8].as<float>();
                          return temporal_enqueue(s, h, prm, tp, d_in, {d[5].as<float>(), d[6].as<float>(), d[7].as<uint32_t>()}, 0, &gc);
                      });
}

// ---- moment denoising (include/trb.h "Moment denoising", DESIGN.md §4) -----------------------------------------------------------
namespace {
// The checks of both forms after the parameters: null pointers, overlapping outputs, the history's scene and film size, a frame.
// variance: a trb_denoise_variance_temporal* call, whose lum_w is one more required input.
trb_status moments_check(const trb_scene* s, const trb_denoise_history* h, const trb_denoise_frame* in, const trb_denoise_temporal_params* params,
                         const trb_denoise_moments_output* out, trb::DnParams& prm, trb::DnTemporal& tp, bool variance = false,
                         const float* lum_w = nullptr) {
    trb_status r = temporal_params(params, prm, tp);
    if (r != TRB_OK) return r;
    if (!s || !h || !in || !out || !out->rgbw || !in->colour || !in->albedo_w || !in->normal_w || !in->nearest || (variance && !lum_w))
        return fail(TRB_INVALID_ARG, "null argument");
    prm.width = (int)s->film.width; prm.height = (int)s->film.height;
    const size_t npx = (size_t)s->film.width * s->film.height;
    const Span ins[5] = {{in->colour, npx * sizeof(float4)}, {in->albedo_w, npx * sizeof(float4)}, {in->normal_w, npx * sizeof(float4)},
                         {in->nearest, npx * sizeof(uint64_t)}, {lum_w, npx * sizeof(float4)}};
    const Span outs[4] = {{out->rgbw, npx * sizeof(float4)}, {out->motion, npx * sizeof(float2)}, {out->history_length, npx * sizeof(uint32_t)},
                          {out->variance, npx * sizeof(float)}};
    return history_call_check(s, h, ins, variance ? 5 : 4, outs, 4, 0);
}

// k_dn_temporal_moments (or, with gc, the gradient steps around k_dn_temporal_moments_grad), k_dn_moments_variance and the a-trous
// launches on `st`, then the history's switch to the set just written. With lum_w (trb_denoise_variance_temporal*),
// k_dn_temporal_variance or k_dn_temporal_variance_grad takes the place of the moment kernels, and the history is of the variance
// family.
trb_status moments_enqueue(trb_scene* s, trb_denoise_history* h, trb::DnParams& prm, trb::DnTemporal& tp, const trb_denoise_frame& in,
                           const trb_denoise_moments_output& out, cudaStream_t st, const GradCall* gc = nullptr, const float* lum_w = nullptr) {
    const size_t npx = (size_t)prm.width * prm.height;
    if (npx == 0) return TRB_OK;
    const DnFamily family = lum_w ? DN_VARIANCE : DN_MOMENTS;
    trb::DnScratch sc;
    float4* mom = nullptr;
    trb_status r = denoise_scratch(s, npx, sc, lum_w ? nullptr : &mom);
    if (r != TRB_OK) return r;
    HistorySets hs;
    r = history_begin(s, h, prm, tp, family, gc, hs, st);
    if (r != TRB_OK) return r;
    float4* rgbw = reinterpret_cast<float4*>(out.rgbw);
    const dim3 block(32, 8), grid((prm.width + 31) / 32, (prm.height + 7) / 8);
    const float4* col = reinterpret_cast<const float4*>(in.colour);
    const float4* lum = reinterpret_cast<const float4*>(lum_w);
    const float4* alb = reinterpret_cast<const float4*>(in.albedo_w);
    const float4* nrm = reinterpret_cast<const float4*>(in.normal_w);
    const unsigned long long* nearest = reinterpret_cast<const unsigned long long*>(in.nearest);
    float2* motion = reinterpret_cast<float2*>(out.motion);
    GrBuffers b{};
    if (!gc) {
        if (lum_w)
            trb::k_dn_temporal_variance<<<grid, block, 0, st>>>(prm, tp, col, lum, alb, nrm, nearest, sc, rgbw, s->d_instances, hs.mats_rd, h->set(hs.rd),
                                                                h->set(hs.wr), motion, out.history_length, out.variance);
        else
            trb::k_dn_temporal_moments<<<grid, block, 0, st>>>(prm, tp, col, alb, nrm, nearest, sc, mom, rgbw, s->d_instances, hs.mats_rd, h->set(hs.rd),
                                                               h->set(hs.wr), motion, out.history_length);
    } else {
        gr_layout(h->gr_capacity, static_cast<char*>(h->d_gr), &b);
        r = gradient_lambda(s, h, *gc, tp, b, hs.mats_rd, in.nearest, in.normal_w, tp.has_prev && h->gr_valid, st);
        if (r != TRB_OK) return r;
        const uint32_t gw = (uint32_t)((prm.width + 2) / 3);
        if (lum_w)
            trb::k_dn_temporal_variance_grad<<<grid, block, 0, st>>>(prm, tp, col, lum, alb, nrm, nearest, sc, rgbw, s->d_instances, hs.mats_rd,
                                                                     h->set(hs.rd), h->set(hs.wr), motion, out.history_length, out.variance, b.lam, gw,
                                                                     gc->lambda);
        else
            trb::k_dn_temporal_moments_grad<<<grid, block, 0, st>>>(prm, tp, col, alb, nrm, nearest, sc, mom, rgbw, s->d_instances, hs.mats_rd,
                                                                    h->set(hs.rd), h->set(hs.wr), motion, out.history_length, b.lam, gw, gc->lambda);
    }
    g_launches++;
    if (!lum_w) {
        trb::k_dn_moments_variance<<<grid, block, 0, st>>>(prm, sc.guide, sc.grad, mom, sc.ev[0], out.variance);
        g_launches++;
    }
    CU(cudaGetLastError());
    r = denoise_atrous(prm, sc, rgbw, st);
    if (r != TRB_OK) return r;
    if (gc) {
        r = gradient_record(s, *gc, b, hs.wr, st);
        if (r != TRB_OK) return r;
        gradient_commit(s, h, *gc);
    } else {
        h->gr_valid = false;
    }
    history_commit(s, h, hs, family);
    return TRB_OK;
}
} // namespace

trb_status trb_denoise_moments_device(trb_scene* s, trb_denoise_history* h, const trb_denoise_frame* d_in, const trb_denoise_temporal_params* params,
                                      const trb_denoise_moments_output* d_out, void* stream) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    trb_status r = moments_check(s, h, d_in, params, d_out, prm, tp);
    if (r == TRB_OK)
        r = check_aligned({{d_in->colour, 16}, {d_in->albedo_w, 16}, {d_in->normal_w, 16}, {d_out->rgbw, 16}, {d_in->nearest, 8}, {d_out->motion, 8},
                           {d_out->history_length, 4}, {d_out->variance, 4}},
                          "device films must be 16-byte aligned, nearest and motion 8-byte, history_length and variance 4-byte");
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    return moments_enqueue(s, h, prm, tp, *d_in, *d_out, static_cast<cudaStream_t>(stream));
}

trb_status trb_denoise_moments(trb_scene* s, trb_denoise_history* h, const trb_denoise_frame* in, const trb_denoise_temporal_params* params,
                               const trb_denoise_moments_output* out) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    trb_status r = moments_check(s, h, in, params, out, prm, tp);
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)prm.width * prm.height, fb = npx * sizeof(float4);
    return run_staged({{in->colour, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}},
                      {{out->rgbw, fb}, {out->motion, npx * sizeof(float2)}, {out->history_length, npx * sizeof(uint32_t)}, {out->variance, npx * sizeof(float)}},
                      [&](const DeviceBuffer* d) {
                          return moments_enqueue(s, h, prm, tp, {d[0].as<float>(), d[1].as<float>(), d[2].as<float>(), d[3].as<uint64_t>()},
                                                 {d[4].as<float>(), d[5].as<float>(), d[6].as<uint32_t>(), d[7].as<float>()}, 0);
                      });
}

// ---- moment gradients (include/trb.h "Moment gradients", DESIGN.md §4) -------------------------------------------------------------
namespace {
// trb_denoise_gradient_params (NULL meaning the defaults) first, then moments_check and the lambda output's overlaps (variance, lum_w:
// as for moments_check)
trb_status moments_gradient_check(const trb_scene* s, const trb_denoise_history* h, const trb_denoise_frame* in, const trb_denoise_gradient_params* params,
                                  const trb_denoise_moments_gradient_output* out, trb::DnParams& prm, trb::DnTemporal& tp, GradCall& gc,
                                  bool variance = false, const float* lum_w = nullptr) {
    const uint32_t iterations = params ? params->iterations : 3u;
    trb_status r = temporal_params(params ? &params->temporal : nullptr, prm, tp);
    if (r != TRB_OK) return r;
    if (iterations > 6) return fail(TRB_INVALID_ARG, "temporal gradient iterations must be 0 to 6");
    if (!out) return fail(TRB_INVALID_ARG, "null argument");
    const trb_denoise_moments_output o{out->rgbw, out->motion, out->history_length, out->variance};
    r = moments_check(s, h, in, params ? &params->temporal : nullptr, &o, prm, tp, variance, lum_w);
    if (r != TRB_OK) return r;
    const size_t npx = (size_t)s->film.width * s->film.height, fb = npx * sizeof(float4);
    if (overlaps_any({out->lambda, npx * sizeof(float)}, {{in->colour, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)},
                                                          {out->rgbw, fb}, {out->motion, npx * sizeof(float2)}, {out->history_length, npx * sizeof(uint32_t)},
                                                          {out->variance, npx * sizeof(float)}, {lum_w, fb}}))
        return fail(TRB_INVALID_ARG, "the lambda output overlaps another buffer");
    gc.iterations = iterations;
    gc.lambda = out->lambda;
    return TRB_OK;
}
} // namespace

trb_status trb_denoise_moments_gradient_device(trb_scene* s, trb_denoise_history* h, const trb_denoise_frame* d_in, const trb_denoise_gradient_params* params,
                                               uint32_t seed, const trb_denoise_moments_gradient_output* d_out, void* stream) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    GradCall gc{};
    trb_status r = moments_gradient_check(s, h, d_in, params, d_out, prm, tp, gc);
    if (r == TRB_OK)
        r = check_aligned({{d_in->colour, 16}, {d_in->albedo_w, 16}, {d_in->normal_w, 16}, {d_out->rgbw, 16}, {d_in->nearest, 8}, {d_out->motion, 8},
                           {d_out->history_length, 4}, {d_out->variance, 4}, {d_out->lambda, 4}},
                          "device films must be 16-byte aligned, nearest and motion 8-byte, history_length, variance and lambda 4-byte");
    if (r != TRB_OK) return r;
    gc.seed = seed;
    CU(cudaSetDevice(s->device));
    const trb_denoise_moments_output o{d_out->rgbw, d_out->motion, d_out->history_length, d_out->variance};
    return moments_enqueue(s, h, prm, tp, *d_in, o, static_cast<cudaStream_t>(stream), &gc);
}

trb_status trb_denoise_moments_gradient(trb_scene* s, trb_denoise_history* h, const trb_denoise_frame* in, const trb_denoise_gradient_params* params,
                                        uint32_t seed, const trb_denoise_moments_gradient_output* out) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    GradCall gc{};
    trb_status r = moments_gradient_check(s, h, in, params, out, prm, tp, gc);
    if (r != TRB_OK) return r;
    gc.seed = seed;
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)prm.width * prm.height, fb = npx * sizeof(float4);
    return run_staged({{in->colour, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}},
                      {{out->rgbw, fb}, {out->motion, npx * sizeof(float2)}, {out->history_length, npx * sizeof(uint32_t)}, {out->variance, npx * sizeof(float)},
                       {out->lambda, npx * sizeof(float)}},
                      [&](const DeviceBuffer* d) {
                          gc.lambda = d[8].as<float>();
                          return moments_enqueue(s, h, prm, tp, {d[0].as<float>(), d[1].as<float>(), d[2].as<float>(), d[3].as<uint64_t>()},
                                                 {d[4].as<float>(), d[5].as<float>(), d[6].as<uint32_t>(), d[7].as<float>()}, 0, &gc);
                      });
}

// ---- variance temporal denoising (include/trb.h "Variance temporal denoising", DESIGN.md §4) ---------------------------------------
// The moment calls' checks and enqueue with lum_w: one more input, and the variance kernels in place of the moment ones
trb_status trb_denoise_variance_temporal_device(trb_scene* s, trb_denoise_history* h, const trb_denoise_frame* d_in, const float* d_lum_w,
                                                const trb_denoise_temporal_params* params, const trb_denoise_moments_output* d_out, void* stream) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    trb_status r = moments_check(s, h, d_in, params, d_out, prm, tp, true, d_lum_w);
    if (r == TRB_OK)
        r = check_aligned({{d_in->colour, 16}, {d_in->albedo_w, 16}, {d_in->normal_w, 16}, {d_lum_w, 16}, {d_out->rgbw, 16}, {d_in->nearest, 8},
                           {d_out->motion, 8}, {d_out->history_length, 4}, {d_out->variance, 4}},
                          "device films must be 16-byte aligned, nearest and motion 8-byte, history_length and variance 4-byte");
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    return moments_enqueue(s, h, prm, tp, *d_in, *d_out, static_cast<cudaStream_t>(stream), nullptr, d_lum_w);
}

trb_status trb_denoise_variance_temporal(trb_scene* s, trb_denoise_history* h, const trb_denoise_frame* in, const float* lum_w,
                                         const trb_denoise_temporal_params* params, const trb_denoise_moments_output* out) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    trb_status r = moments_check(s, h, in, params, out, prm, tp, true, lum_w);
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)prm.width * prm.height, fb = npx * sizeof(float4);
    return run_staged({{in->colour, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}, {lum_w, fb}},
                      {{out->rgbw, fb}, {out->motion, npx * sizeof(float2)}, {out->history_length, npx * sizeof(uint32_t)}, {out->variance, npx * sizeof(float)}},
                      [&](const DeviceBuffer* d) {
                          return moments_enqueue(s, h, prm, tp, {d[0].as<float>(), d[1].as<float>(), d[2].as<float>(), d[3].as<uint64_t>()},
                                                 {d[5].as<float>(), d[6].as<float>(), d[7].as<uint32_t>(), d[8].as<float>()}, 0, nullptr, d[4].as<float>());
                      });
}

trb_status trb_denoise_variance_temporal_gradient_device(trb_scene* s, trb_denoise_history* h, const trb_denoise_frame* d_in, const float* d_lum_w,
                                                         const trb_denoise_gradient_params* params, uint32_t seed,
                                                         const trb_denoise_moments_gradient_output* d_out, void* stream) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    GradCall gc{};
    trb_status r = moments_gradient_check(s, h, d_in, params, d_out, prm, tp, gc, true, d_lum_w);
    if (r == TRB_OK)
        r = check_aligned({{d_in->colour, 16}, {d_in->albedo_w, 16}, {d_in->normal_w, 16}, {d_lum_w, 16}, {d_out->rgbw, 16}, {d_in->nearest, 8},
                           {d_out->motion, 8}, {d_out->history_length, 4}, {d_out->variance, 4}, {d_out->lambda, 4}},
                          "device films must be 16-byte aligned, nearest and motion 8-byte, history_length, variance and lambda 4-byte");
    if (r != TRB_OK) return r;
    gc.seed = seed;
    CU(cudaSetDevice(s->device));
    const trb_denoise_moments_output o{d_out->rgbw, d_out->motion, d_out->history_length, d_out->variance};
    return moments_enqueue(s, h, prm, tp, *d_in, o, static_cast<cudaStream_t>(stream), &gc, d_lum_w);
}

trb_status trb_denoise_variance_temporal_gradient(trb_scene* s, trb_denoise_history* h, const trb_denoise_frame* in, const float* lum_w,
                                                  const trb_denoise_gradient_params* params, uint32_t seed,
                                                  const trb_denoise_moments_gradient_output* out) {
    trb::DnParams prm{};
    trb::DnTemporal tp{};
    GradCall gc{};
    trb_status r = moments_gradient_check(s, h, in, params, out, prm, tp, gc, true, lum_w);
    if (r != TRB_OK) return r;
    gc.seed = seed;
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)prm.width * prm.height, fb = npx * sizeof(float4);
    return run_staged({{in->colour, fb}, {in->albedo_w, fb}, {in->normal_w, fb}, {in->nearest, npx * sizeof(uint64_t)}, {lum_w, fb}},
                      {{out->rgbw, fb}, {out->motion, npx * sizeof(float2)}, {out->history_length, npx * sizeof(uint32_t)}, {out->variance, npx * sizeof(float)},
                       {out->lambda, npx * sizeof(float)}},
                      [&](const DeviceBuffer* d) {
                          gc.lambda = d[9].as<float>();
                          return moments_enqueue(s, h, prm, tp, {d[0].as<float>(), d[1].as<float>(), d[2].as<float>(), d[3].as<uint64_t>()},
                                                 {d[5].as<float>(), d[6].as<float>(), d[7].as<uint32_t>(), d[8].as<float>()}, 0, &gc, d[4].as<float>());
                      });
}

trb_status trb_adaptive_schedule(const trb_adaptive* ad, uint32_t* min_spp, uint32_t* max_spp, uint32_t* step, uint32_t* max_per_pixel) {
    if (!ad) return fail(TRB_INVALID_ARG, "null argument");
    trbh::AdSchedule sch;
    if (!trbh::ad_schedule(ad->min_spp, ad->max_spp, sch))
        return fail(TRB_INVALID_ARG, "Adaptive sampler: max_spp < min_spp after rounding up to powers of two (the reference panics), or more than 2^24");
    if (min_spp) *min_spp = sch.min;
    if (max_spp) *max_spp = sch.max;
    if (step) *step = sch.step;
    if (max_per_pixel) *max_per_pixel = sch.max_per_pixel;
    return TRB_OK;
}

trb_status trb_host_adaptive_decide(const trb_adaptive* ad, const float* lum, size_t n, uint32_t* samples_taken, float* avg) {
    if (!ad || (n && !lum) || !samples_taken) return fail(TRB_INVALID_ARG, "null argument");
    trbh::AdSchedule sch;
    if (!trbh::ad_schedule(ad->min_spp, ad->max_spp, sch)) return fail(TRB_INVALID_ARG, "Adaptive sampler: max_spp < min_spp after rounding up to powers of two");
    trbh::AdPixel p = trbh::ad_initial();
    for (uint32_t round = 0; round < sch.rounds; ++round) {
        const uint32_t first = trbh::ad_slot_base(sch, round), count = trbh::ad_count(sch, round);
        if ((uint64_t)first + count > n) return fail(TRB_INVALID_ARG, "luminance sequence ends before the pixel stops sampling");
        for (uint32_t k = 0; k < count; ++k) trbh::ad_add(p, first + k, lum[first + k], round == 0);
        if (!trbh::ad_finish(p, sch, round)) break;
    }
    *samples_taken = p.taken & ~trbh::AD_ACTIVE;
    if (avg) *avg = p.avg;
    return TRB_OK;
}

namespace {
// trb_render_adaptive's body; aov: the host AOV outputs of trb_render_adaptive_aov (nullptr: none)
trb_status render_adaptive_host(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* film, const trb_aov_film* aov, uint32_t* pixel_spp,
                                trb_stats* stats, float* lum_w = nullptr, float* motion_w = nullptr, float dt = 0.0f) {
    trbh::AdSchedule sch;
    trb_status r = adaptive_check(s, cfg, ad, sch);
    if (r != TRB_OK) return r;
    CU(cudaSetDevice(s->device));
    float update_ms = 0.f;
    if (!(cfg->flags & TRB_RENDER_NO_UPDATE)) { // Exec::render: scene.update_frame first (multithreaded.rs:57-60)
        auto t0 = std::chrono::steady_clock::now();
        const float step = s->film.scene_time / (float)s->film.frames;
        r = trb_scene_update_frame(s, cfg->current_frame, (float)cfg->current_frame * step, ((float)cfg->current_frame + 1.0f) * step);
        if (r != TRB_OK) return r;
        update_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering"); // scene.rs:179
    uint32_t nb;
    const uint2* d_blocks = nullptr;
    r = ensure_blocks(s, cfg, &d_blocks, &nb);
    if (r != TRB_OK) return r;
    const size_t npx = (size_t)s->film.width * s->film.height;
    CU(cudaMemsetAsync(s->d_film, 0, npx * sizeof(float4), 0));
    CU(cudaMemsetAsync(s->d_stats, 0, sizeof(trb::DStats), 0));
    HostAov ha;
    if ((r = ha.stage(aov, npx, lum_w, motion_w, dt)) != TRB_OK) return r;
    CU(cudaEventRecord(s->ev0, 0));
    if (nb) { // an empty selection renders nothing (block_queue.rs:42-44)
        r = ensure_adaptive(s);
        if (r != TRB_OK) return r;
        trb::RenderParams rp{};
        rp.seed = cfg->seed; rp.work_counter = s->d_counter; rp.film = s->d_film; rp.stats = s->d_stats; rp.error_flag = s->d_error;
        r = render_adaptive_rounds(s, sch, rp, d_blocks, nb, cfg->flags, 0, pixel_spp ? s->d_ad_spp : nullptr, ha.request());
        if (r != TRB_OK) { if (ha.aov) cudaDeviceSynchronize(); return r; } // passes already enqueued still write the AOV films
    }
    CU(cudaEventRecord(s->ev1, 0));
    CU(cudaMemcpyAsync(s->h_film_staging, s->d_film, npx * sizeof(float4), cudaMemcpyDeviceToHost, 0));
    CU(cudaStreamSynchronize(0));
    r = check_error_flag(s);
    if (r != TRB_OK) return r;
    add_film(film, s->h_film_staging, npx * 4);
    if ((r = ha.unstage(npx)) != TRB_OK) return r;
    r = adaptive_pixel_spp_out(s, d_blocks, nb, pixel_spp);
    return r != TRB_OK ? r : stats_readback(s, stats, update_ms);
}

// trb_render_samples_adaptive's body; aov: the host AOV records of trb_render_samples_adaptive_aov (nullptr: none)
trb_status render_samples_adaptive(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, size_t n, trb_sample* samples, trb_aov_sample* aov,
                                   uint32_t* pixel_spp, trb_stats* stats) {
    trbh::AdSchedule sch;
    trb_status r = adaptive_check(s, cfg, ad, sch);
    if (r != TRB_OK) return r;
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering");
    CU(cudaSetDevice(s->device));
    uint32_t nb;
    const uint2* d_blocks = nullptr;
    r = ensure_blocks(s, cfg, &d_blocks, &nb);
    if (r != TRB_OK) return r;
    if (n != (size_t)nb * 64 * sch.max_per_pixel) return fail(TRB_INVALID_ARG, "sample buffer size must be blocks*64*max_per_pixel");
    if (n == 0) return TRB_OK;
    r = ensure_adaptive(s);
    if (r != TRB_OK) return r;
    trb::RenderParams rp{};
    rp.seed = cfg->seed; rp.work_counter = s->d_counter; rp.film = nullptr; rp.stats = s->d_stats; rp.error_flag = s->d_error;
    r = run_counted(s, {}, {{samples, n * sizeof(trb_sample)}, {aov, n * sizeof(trb_aov_sample)}}, [&](const DeviceBuffer* d) {
        CU(cudaMemsetAsync(d[0].p, 0, n * sizeof(trb_sample), 0)); // unused slots stay zero
        if (aov) CU(cudaMemsetAsync(d[1].p, 0, n * sizeof(trb_aov_sample), 0));
        rp.samples_out = d[0].as<trb_sample>();
        const AovRequest req{d[1].as<trb_aov_sample>(), nullptr, nullptr, nullptr};
        return render_adaptive_rounds(s, sch, rp, d_blocks, nb, cfg->flags, 0, pixel_spp ? s->d_ad_spp : nullptr, aov ? &req : nullptr);
    });
    if (r == TRB_OK) r = adaptive_pixel_spp_out(s, d_blocks, nb, pixel_spp);
    return r != TRB_OK ? r : stats_readback(s, stats, 0.f);
}

// trb_render_adaptive_device's body; aov: the device AOV outputs of trb_render_adaptive_aov_device (nullptr: none)
trb_status render_adaptive_device(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* d_film, const AovRequest* aov, uint32_t* d_pixel_spp,
                                  trb_stats* d_stats, cudaStream_t st) {
    trbh::AdSchedule sch;
    trb_status r = adaptive_check(s, cfg, ad, sch);
    if (r != TRB_OK) return r;
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering"); // scene.rs:179
    CU(cudaSetDevice(s->device));
    uint32_t nb;
    const uint2* d_blocks = nullptr;
    r = ensure_blocks(s, cfg, &d_blocks, &nb);
    if (r != TRB_OK) return r;
    if (nb == 0) return TRB_OK; // "Warning: This block queue is empty!" (block_queue.rs:42-44)
    trb::RenderParams rp{};
    rp.seed = cfg->seed; rp.work_counter = s->d_counter; rp.film = reinterpret_cast<float4*>(d_film); rp.stats = reinterpret_cast<trb::DStats*>(d_stats);
    rp.error_flag = s->d_error;
    return render_adaptive_rounds(s, sch, rp, d_blocks, nb, cfg->flags, st, d_pixel_spp, aov);
}
} // namespace

trb_status trb_render_adaptive(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* film, uint32_t* pixel_spp, trb_stats* stats) {
    if (!s || !cfg || !ad || !film) return fail(TRB_INVALID_ARG, "null argument");
    return render_adaptive_host(s, cfg, ad, film, nullptr, pixel_spp, stats);
}

trb_status trb_render_samples_adaptive(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, size_t n, trb_sample* samples, uint32_t* pixel_spp,
                                       trb_stats* stats) {
    if (!s || !cfg || !ad || !samples) return fail(TRB_INVALID_ARG, "null argument");
    return render_samples_adaptive(s, cfg, ad, n, samples, nullptr, pixel_spp, stats);
}

trb_status trb_render_adaptive_device(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* d_film, uint32_t* d_pixel_spp,
                                      trb_stats* d_stats, void* stream) {
    if (!s || !cfg || !ad || !d_film) return fail(TRB_INVALID_ARG, "null argument");
    return render_adaptive_device(s, cfg, ad, d_film, nullptr, d_pixel_spp, d_stats, static_cast<cudaStream_t>(stream));
}

// The AOV forms: adaptive_check's statuses cover aov_supported's (the path integrator on the wavefront only)
trb_status trb_render_adaptive_aov(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* film, const trb_aov_film* aov, uint32_t* pixel_spp,
                                   trb_stats* stats) {
    if (!s || !cfg || !ad || !film || !aov) return fail(TRB_INVALID_ARG, "null argument");
    return render_adaptive_host(s, cfg, ad, film, aov, pixel_spp, stats);
}

trb_status trb_render_adaptive_aov_device(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* d_film, const trb_aov_film* d_aov,
                                          uint32_t* d_pixel_spp, trb_stats* d_stats, void* stream) {
    if (!s || !cfg || !ad || !d_film || !d_aov) return fail(TRB_INVALID_ARG, "null argument");
    const trb_status r = check_aligned({{d_film, 16}, {d_aov->albedo_w, 16}, {d_aov->normal_w, 16}, {d_aov->nearest, 8}},
                                       "device films must be 16-byte aligned, the nearest buffer 8-byte aligned");
    if (r != TRB_OK) return r;
    const AovRequest req{nullptr, reinterpret_cast<float4*>(d_aov->albedo_w), reinterpret_cast<float4*>(d_aov->normal_w),
                         reinterpret_cast<unsigned long long*>(d_aov->nearest)};
    const bool with_aov = d_aov->albedo_w || d_aov->normal_w || d_aov->nearest;
    return render_adaptive_device(s, cfg, ad, d_film, with_aov ? &req : nullptr, d_pixel_spp, d_stats, static_cast<cudaStream_t>(stream));
}

trb_status trb_render_adaptive_aov_lum(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* film, const trb_aov_film* aov, float* lum_w,
                                       uint32_t* pixel_spp, trb_stats* stats) {
    if (!s || !cfg || !ad || !film || !aov || !lum_w) return fail(TRB_INVALID_ARG, "null argument");
    return render_adaptive_host(s, cfg, ad, film, aov, pixel_spp, stats, lum_w);
}

trb_status trb_render_adaptive_aov_lum_device(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* d_film, const trb_aov_film* d_aov,
                                              float* d_lum_w, uint32_t* d_pixel_spp, trb_stats* d_stats, void* stream) {
    if (!s || !cfg || !ad || !d_film || !d_aov || !d_lum_w) return fail(TRB_INVALID_ARG, "null argument");
    const trb_status r = check_aligned({{d_film, 16}, {d_aov->albedo_w, 16}, {d_aov->normal_w, 16}, {d_lum_w, 16}, {d_aov->nearest, 8}},
                                       "device films must be 16-byte aligned, the nearest buffer 8-byte aligned");
    if (r != TRB_OK) return r;
    const AovRequest req{nullptr, reinterpret_cast<float4*>(d_aov->albedo_w), reinterpret_cast<float4*>(d_aov->normal_w),
                         reinterpret_cast<unsigned long long*>(d_aov->nearest), reinterpret_cast<float4*>(d_lum_w)};
    return render_adaptive_device(s, cfg, ad, d_film, &req, d_pixel_spp, d_stats, static_cast<cudaStream_t>(stream));
}

trb_status trb_render_adaptive_aov_motion(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* film, const trb_aov_film* aov, float* lum_w,
                                          float* motion_w, float dt, uint32_t* pixel_spp, trb_stats* stats) {
    if (!s || !cfg || !ad || !film || !aov || !motion_w) return fail(TRB_INVALID_ARG, "null argument");
    const trb_status r = motion_dt(dt);
    if (r != TRB_OK) return r;
    return render_adaptive_host(s, cfg, ad, film, aov, pixel_spp, stats, lum_w, motion_w, dt);
}

trb_status trb_render_adaptive_aov_motion_device(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, float* d_film, const trb_aov_film* d_aov,
                                                 float* d_lum_w, float* d_motion_w, float dt, uint32_t* d_pixel_spp, trb_stats* d_stats, void* stream) {
    if (!s || !cfg || !ad || !d_film || !d_aov || !d_motion_w) return fail(TRB_INVALID_ARG, "null argument");
    trb_status r = check_aligned({{d_film, 16}, {d_aov->albedo_w, 16}, {d_aov->normal_w, 16}, {d_lum_w, 16}, {d_motion_w, 16}, {d_aov->nearest, 8}},
                                 "device films must be 16-byte aligned, the nearest buffer 8-byte aligned");
    if (r == TRB_OK) r = motion_dt(dt);
    if (r != TRB_OK) return r;
    const AovRequest req{nullptr, reinterpret_cast<float4*>(d_aov->albedo_w), reinterpret_cast<float4*>(d_aov->normal_w),
                         reinterpret_cast<unsigned long long*>(d_aov->nearest), reinterpret_cast<float4*>(d_lum_w), nullptr,
                         reinterpret_cast<float4*>(d_motion_w), dt};
    return render_adaptive_device(s, cfg, ad, d_film, &req, d_pixel_spp, d_stats, static_cast<cudaStream_t>(stream));
}

trb_status trb_render_samples_adaptive_aov(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, size_t n, trb_sample* samples, trb_aov_sample* aov,
                                           uint32_t* pixel_spp, trb_stats* stats) {
    if (!s || !cfg || !ad || !samples || !aov) return fail(TRB_INVALID_ARG, "null argument");
    return render_samples_adaptive(s, cfg, ad, n, samples, aov, pixel_spp, stats);
}

trb_status trb_camera_rays(trb_scene* s, const trb_render_cfg* cfg, size_t n, trb_ray* rays, float* xy) {
    if (!s || !cfg || !rays || !xy) return fail(TRB_INVALID_ARG, "null argument");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering");
    CU(cudaSetDevice(s->device));
    uint32_t spp, first, count, nb;
    const uint2* d_blocks = nullptr;
    trb_status r = resolve_samples(s, cfg, spp, first, count);
    if (r != TRB_OK) return r;
    r = ensure_blocks(s, cfg, &d_blocks, &nb);
    if (r != TRB_OK) return r;
    if (n != (size_t)nb * 64 * count) return fail(TRB_INVALID_ARG, "ray buffer size must be blocks*64*sample_count");
    if (n == 0) return TRB_OK;
    trb::RenderParams rp{};
    rp.blocks = d_blocks; rp.n_blocks = nb; rp.spp = spp; rp.sample_first = first; rp.sample_count = count; rp.seed = cfg->seed;
    return run_staged({}, {{rays, n * sizeof(trb_ray)}, {xy, n * 2 * sizeof(float)}}, [&](const DeviceBuffer* d) {
        const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)s->sm_count * 8);
        if (s->ds.has_anim) trb::k_camera_rays<true><<<grid, 256>>>(s->ds, rp, d[0].as<trb_ray>(), d[1].as<float>());
        else trb::k_camera_rays<false><<<grid, 256>>>(s->ds, rp, d[0].as<trb_ray>(), d[1].as<float>());
        CU(cudaGetLastError());
        return TRB_OK;
    });
}

trb_status trb_intersect_device(trb_scene* s, size_t n, const trb_ray* d_rays, trb_hit* d_hits, trb_stats* d_stats, void* stream) {
    if (!s || (n && (!d_rays || !d_hits))) return fail(TRB_INVALID_ARG, "null argument");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before intersecting");
    if (n == 0) return TRB_OK;
    CU(cudaSetDevice(s->device));
    const unsigned grid = (unsigned)std::min<size_t>((n + 127) / 128, (size_t)s->sm_count * 16);
    g_launches++;
    intersect_kernel<false>(s)<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(s->ds, n, d_rays, d_hits, reinterpret_cast<trb::DStats*>(d_stats), s->d_error);
    CU(cudaGetLastError());
    return TRB_OK;
}

trb_status trb_intersect(trb_scene* s, size_t n, const trb_ray* rays, trb_hit* hits, trb_stats* stats) {
    if (!s || (n && (!rays || !hits))) return fail(TRB_INVALID_ARG, "null argument");
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before intersecting");
    if (n == 0) return TRB_OK;
    return run_query(s, n, {rays, n * sizeof(trb_ray)}, {hits, n * sizeof(trb_hit)}, stats, [&](void* d_rays, void* d_hits) {
        const unsigned grid = (unsigned)std::min<size_t>((n + 127) / 128, (size_t)s->sm_count * 16);
        intersect_kernel<true>(s)<<<grid, 128>>>(s->ds, n, static_cast<const trb_ray*>(d_rays), static_cast<trb_hit*>(d_hits), s->d_stats,
                                                 s->d_error); // host variant always counts tests
        CU(cudaGetLastError());
        return TRB_OK;
    });
}

trb_status trb_intersect_records(trb_scene* s, size_t n, const trb_query_ray* rays, trb_intersection* out, uint32_t flags, trb_stats* stats) {
    const trb_status r = query_check(s, n, rays, out, flags, TRB_RENDER_STATS, false, false);
    return r != TRB_OK ? r : run_query(s, n, {rays, n * sizeof(trb_query_ray)}, {out, n * sizeof(trb_intersection)}, stats, [&](const void* d_rays, void* d_out) {
        return query_passes(s, n, static_cast<const trb_query_ray*>(d_rays), static_cast<trb_intersection*>(d_out), nullptr, flags, s->d_stats, 0);
    });
}

trb_status trb_intersect_records_device(trb_scene* s, size_t n, const trb_query_ray* d_rays, trb_intersection* d_out, uint32_t flags,
                                        trb_stats* d_stats, void* stream) {
    const trb_status r = query_check(s, n, d_rays, d_out, flags, TRB_RENDER_STATS, true, true);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return query_passes(s, n, d_rays, d_out, nullptr, flags, reinterpret_cast<trb::DStats*>(d_stats), static_cast<cudaStream_t>(stream));
}

trb_status trb_occluded(trb_scene* s, size_t n, const trb_query_ray* rays, uint8_t* occluded, uint32_t flags, trb_stats* stats) {
    const trb_status r = query_check(s, n, rays, occluded, flags, TRB_RENDER_STATS | TRB_RENDER_REFERENCE_SHADOW, false, false);
    return r != TRB_OK ? r : run_query(s, n, {rays, n * sizeof(trb_query_ray)}, {occluded, n}, stats, [&](const void* d_rays, void* d_out) {
        return query_passes(s, n, static_cast<const trb_query_ray*>(d_rays), nullptr, static_cast<uint8_t*>(d_out), flags, s->d_stats, 0);
    });
}

trb_status trb_occluded_device(trb_scene* s, size_t n, const trb_query_ray* d_rays, uint8_t* d_occluded, uint32_t flags, trb_stats* d_stats,
                               void* stream) {
    const trb_status r = query_check(s, n, d_rays, d_occluded, flags, TRB_RENDER_STATS | TRB_RENDER_REFERENCE_SHADOW, true, false);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return query_passes(s, n, d_rays, nullptr, d_occluded, flags, reinterpret_cast<trb::DStats*>(d_stats), static_cast<cudaStream_t>(stream));
}

trb_status trb_illumination(trb_scene* s, size_t n, const trb_illum_ray* rays, uint32_t spp, uint32_t seed, float* rgb, uint32_t flags, trb_stats* stats) {
    const trb_status r = illum_check(s, n, rays, spp, rgb, flags, false);
    return r != TRB_OK ? r : run_query(s, n, {rays, n * sizeof(trb_illum_ray)}, {rgb, n * 3 * sizeof(float)}, stats, [&](const void* d_rays, void* d_rgb) {
        return illum_passes(s, n, static_cast<const trb_illum_ray*>(d_rays), spp, seed, static_cast<float*>(d_rgb), flags, s->d_stats, 0);
    });
}

trb_status trb_illumination_device(trb_scene* s, size_t n, const trb_illum_ray* d_rays, uint32_t spp, uint32_t seed, float* d_rgb, uint32_t flags,
                                   trb_stats* d_stats, void* stream) {
    const trb_status r = illum_check(s, n, d_rays, spp, d_rgb, flags, true);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return illum_passes(s, n, d_rays, spp, seed, d_rgb, flags, reinterpret_cast<trb::DStats*>(d_stats), static_cast<cudaStream_t>(stream));
}

trb_status trb_bsdf_eval(trb_scene* s, size_t n, const trb_intersection* rec, const trb_bsdf_eval_query* q, float* out4) {
    const trb_status r = shade_check(s, n, rec, q, out4, 16, false, false);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return run_staged({{rec, n * sizeof *rec}, {q, n * sizeof *q}}, {{out4, n * 4 * sizeof(float)}}, [&](const DeviceBuffer* d) {
        return launch_bsdf_eval(s, n, d[0].as<trb_intersection>(), d[1].as<trb_bsdf_eval_query>(), d[2].as<float>(), 0);
    });
}

trb_status trb_bsdf_eval_device(trb_scene* s, size_t n, const trb_intersection* d_rec, const trb_bsdf_eval_query* d_q, float* d_out4, void* stream) {
    const trb_status r = shade_check(s, n, d_rec, d_q, d_out4, 16, true, false);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return launch_bsdf_eval(s, n, d_rec, d_q, d_out4, static_cast<cudaStream_t>(stream));
}

trb_status trb_bsdf_sample(trb_scene* s, size_t n, const trb_intersection* rec, const trb_bsdf_sample_query* q, trb_bsdf_sample_result* out) {
    const trb_status r = shade_check(s, n, rec, q, out, 16, false, false);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return run_staged({{rec, n * sizeof *rec}, {q, n * sizeof *q}}, {{out, n * sizeof *out}}, [&](const DeviceBuffer* d) {
        return launch_bsdf_sample(s, n, d[0].as<trb_intersection>(), d[1].as<trb_bsdf_sample_query>(), d[2].as<trb_bsdf_sample_result>(), 0);
    });
}

trb_status trb_bsdf_sample_device(trb_scene* s, size_t n, const trb_intersection* d_rec, const trb_bsdf_sample_query* d_q, trb_bsdf_sample_result* d_out,
                                  void* stream) {
    const trb_status r = shade_check(s, n, d_rec, d_q, d_out, 16, true, false);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return launch_bsdf_sample(s, n, d_rec, d_q, d_out, static_cast<cudaStream_t>(stream));
}

trb_status trb_light_sample(trb_scene* s, size_t n, const trb_light_query* q, trb_light_sample_result* out) {
    const trb_status r = shade_check(s, n, q, q, out, 16, false, true);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return run_staged({{q, n * sizeof *q}}, {{out, n * sizeof *out}}, [&](const DeviceBuffer* d) {
        return launch_light_sample(s, n, d[0].as<trb_light_query>(), d[1].as<trb_light_sample_result>(), 0);
    });
}

trb_status trb_light_sample_device(trb_scene* s, size_t n, const trb_light_query* d_q, trb_light_sample_result* d_out, void* stream) {
    const trb_status r = shade_check(s, n, d_q, d_q, d_out, 16, true, true);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return launch_light_sample(s, n, d_q, d_out, static_cast<cudaStream_t>(stream));
}

trb_status trb_light_pdf(trb_scene* s, size_t n, const trb_light_pdf_query* q, float* pdf) {
    const trb_status r = shade_check(s, n, q, q, pdf, 4, false, true);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return run_staged({{q, n * sizeof *q}}, {{pdf, n * sizeof(float)}}, [&](const DeviceBuffer* d) {
        return launch_light_pdf(s, n, d[0].as<trb_light_pdf_query>(), d[1].as<float>(), 0);
    });
}

trb_status trb_light_pdf_device(trb_scene* s, size_t n, const trb_light_pdf_query* d_q, float* d_pdf, void* stream) {
    const trb_status r = shade_check(s, n, d_q, d_q, d_pdf, 4, true, true);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return launch_light_pdf(s, n, d_q, d_pdf, static_cast<cudaStream_t>(stream));
}

trb_status trb_emitted(trb_scene* s, size_t n, const trb_emit_query* q, float* rgb) {
    const trb_status r = shade_check(s, n, q, q, rgb, 4, false, false);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return run_staged({{q, n * sizeof *q}}, {{rgb, n * 3 * sizeof(float)}}, [&](const DeviceBuffer* d) {
        return launch_emitted(s, n, d[0].as<trb_emit_query>(), d[1].as<float>(), 0);
    });
}

trb_status trb_emitted_device(trb_scene* s, size_t n, const trb_emit_query* d_q, float* d_rgb, void* stream) {
    const trb_status r = shade_check(s, n, d_q, d_q, d_rgb, 4, true, false);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return launch_emitted(s, n, d_q, d_rgb, static_cast<cudaStream_t>(stream));
}

trb_status trb_scene_lights(const trb_scene* s, uint32_t* inst) {
    if (!s || (s->ds.n_lights && !inst)) return fail(TRB_INVALID_ARG, "null argument");
    uint32_t k = 0;
    for (uint32_t i = 0; i < (uint32_t)s->instances.size(); ++i) if (s->instances[i].kind != TRB_INST_RECEIVER) inst[k++] = i; // as trb_scene_create builds ds.lights
    return TRB_OK;
}

trb_status trb_film_write(trb_scene* s, size_t n, const trb_sample* samples, const uint32_t* regions, float* film_rgbw) {
    const trb_status r = film_check(s, n, samples, regions, film_rgbw, false);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    const size_t film_bytes = (size_t)s->film.width * s->film.height * 4 * sizeof(float);
    return run_staged({{samples, n * sizeof(trb_sample)}, {regions, n * sizeof(uint32_t)}}, {{film_rgbw, film_bytes}}, [&](const DeviceBuffer* d) {
        CU(cudaMemcpy(d[2].p, film_rgbw, film_bytes, cudaMemcpyHostToDevice)); // the samples are added to the caller's film
        return film_write_enqueue(s, (uint32_t)n, d[0].as<trb_sample>(), d[1].as<uint32_t>(), d[2].as<float>(), 0);
    });
}

trb_status trb_film_write_device(trb_scene* s, size_t n, const trb_sample* d_samples, const uint32_t* d_regions, float* d_film_rgbw, void* stream) {
    const trb_status r = film_check(s, n, d_samples, d_regions, d_film_rgbw, true);
    if (r != TRB_OK || n == 0) return r;
    CU(cudaSetDevice(s->device));
    return film_write_enqueue(s, (uint32_t)n, d_samples, d_regions, d_film_rgbw, static_cast<cudaStream_t>(stream));
}

trb_status trb_camera_rays_device(trb_scene* s, const trb_render_cfg* cfg, size_t n, trb_ray* d_rays, float* d_xy, void* stream) {
    if (!s || !cfg || (n && (!d_rays || !d_xy))) return fail(TRB_INVALID_ARG, "null argument");
    { const trb_status r = check_aligned({{d_rays, 4}, {d_xy, 4}}, "device ray buffers must be 4-byte aligned"); if (r != TRB_OK) return r; }
    if (!s->frame_ready) return fail(TRB_INVALID_ARG, "Update frame must be called before rendering");
    CU(cudaSetDevice(s->device));
    return camera_rays_enqueue(s, cfg, n, d_rays, d_xy, static_cast<cudaStream_t>(stream));
}

trb_status trb_film_to_srgb8(trb_scene* s, const float* film, uint8_t* rgb8) {
    if (!s || !film || !rgb8) return fail(TRB_INVALID_ARG, "null argument");
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)s->film.width * s->film.height;
    return run_staged({}, {{rgb8, npx * 3}}, [&](const DeviceBuffer* d) {
        CU(cudaMemcpy(s->d_film, film, npx * sizeof(float4), cudaMemcpyHostToDevice)); // the input goes through the scene's device film
        trb::k_srgb8<<<(unsigned)std::min<size_t>((npx + 255) / 256, (size_t)s->sm_count * 16), 256>>>(npx, s->d_film, d[0].as<uint8_t>());
        CU(cudaGetLastError());
        return TRB_OK;
    });
}

trb_status trb_host_film_to_srgb8(uint32_t width, uint32_t height, const float* film, uint8_t* rgb8) {
    const size_t npx = (size_t)width * height;
    if (npx && (!film || !rgb8)) return fail(TRB_INVALID_ARG, "null argument");
    for (size_t i = 0; i < npx; ++i) trb::srgb8_pixel(film[4 * i], film[4 * i + 1], film[4 * i + 2], film[4 * i + 3], rgb8 + 3 * i);
    return TRB_OK;
}

trb_status trb_block_list(const trb_scene* s, uint32_t start, uint32_t count, uint32_t* n_out, uint32_t* xy, uint32_t cap) {
    if (!s || !n_out) return fail(TRB_INVALID_ARG, "null argument");
    std::vector<uint32_t> b = morton_blocks(s->film.width, s->film.height, start, count);
    *n_out = (uint32_t)(b.size() / 2);
    if (xy) std::memcpy(xy, b.data(), sizeof(uint32_t) * std::min<size_t>(b.size(), 2 * (size_t)cap));
    return TRB_OK;
}

trb_status trb_scene_get_bvh(const trb_scene* s, int which, uint32_t* n_nodes, trb_bvh_node* nodes, uint32_t* n_ordered, uint32_t* ordered) {
    if (!s || !n_nodes || !n_ordered) return fail(TRB_INVALID_ARG, "null argument");
    const std::vector<trb_bvh_node>* nn; const std::vector<uint32_t>* oo;
    std::vector<trb_bvh_node> dev_nodes; std::vector<uint32_t> dev_order;
    if (which < 0) {
        if (!s->frame_ready) return fail(TRB_INVALID_ARG, "update_frame first");
        if (s->host_frame_stale) { // the frame was prepared on the device: read its TLAS back
            CU(cudaSetDevice(s->device));
            dev_nodes.resize(s->tlas_n_nodes); dev_order.resize(s->instances.size());
            CU(cudaMemcpy(dev_nodes.data(), s->d_tlas_nodes, dev_nodes.size() * sizeof(trb_bvh_node), cudaMemcpyDeviceToHost));
            CU(cudaMemcpy(dev_order.data(), s->d_tlas_order, dev_order.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
            nn = &dev_nodes; oo = &dev_order;
        } else { nn = &s->tlas_nodes; oo = &s->tlas_order; }
    }
    else {
        if ((size_t)which >= s->meshes.size()) return fail(TRB_INVALID_ARG, "mesh index out of range");
        if (s->meshes[which].stale) { // a refit left the boxes on the device: refreshing the host copy does not change the scene
            trb_scene* ms = const_cast<trb_scene*>(s);
            CU(cudaSetDevice(s->device));
            const trb_status r = refresh_host_tree(ms->meshes[which], ms->dmeshes[which]);
            if (r != TRB_OK) return r;
        }
        nn = &s->meshes[which].nodes; oo = &s->meshes[which].order;
    }
    *n_nodes = (uint32_t)nn->size(); *n_ordered = (uint32_t)oo->size();
    if (nodes) std::memcpy(nodes, nn->data(), nn->size() * sizeof(trb_bvh_node));
    if (ordered) std::memcpy(ordered, oo->data(), oo->size() * sizeof(uint32_t));
    return TRB_OK;
}

trb_status trb_scene_get_transform(const trb_scene* s, uint32_t inst, float* mat16, float* inv16) {
    if (!s || !s->frame_ready || inst >= s->instances.size()) return fail(TRB_INVALID_ARG, "bad instance / update_frame first");
    if (s->host_frame_stale) { // prepared on the device
        trb::DInstance di;
        CU(cudaSetDevice(s->device));
        CU(cudaMemcpy(&di, s->d_instances + inst, sizeof di, cudaMemcpyDeviceToHost));
        std::memcpy(mat16, di.mat, 64); std::memcpy(inv16, di.inv, 64);
        return TRB_OK;
    }
    std::memcpy(mat16, s->world[inst].fwd.m, 64); std::memcpy(inv16, s->world[inst].inv.m, 64);
    return TRB_OK;
}

trb_status trb_scene_get_filter_table(const trb_scene* s, float* t) {
    if (!s || !t) return fail(TRB_INVALID_ARG, "null argument");
    std::memcpy(t, s->table, sizeof s->table);
    return TRB_OK;
}

trb_status trb_host_build_bvh(const float* boxes6, uint32_t n, uint32_t max_geom, uint32_t* n_nodes, trb_bvh_node* nodes, uint32_t* ordered) {
    if (!boxes6 || n == 0 || !n_nodes) return fail(TRB_INVALID_ARG, "empty geometry"); // bvh.rs:35 assert!(!geometry.is_empty())
    std::vector<Box3> b(n);
    for (uint32_t i = 0; i < n; ++i) for (int k = 0; k < 3; ++k) { b[i].lo[k] = boxes6[6 * i + k]; b[i].hi[k] = boxes6[6 * i + 3 + k]; }
    BvhBuilder bb;
    bb.build(b, max_geom);
    *n_nodes = (uint32_t)bb.nodes.size();
    if (nodes) std::memcpy(nodes, bb.nodes.data(), bb.nodes.size() * sizeof(trb_bvh_node));
    if (ordered) std::memcpy(ordered, bb.order.data(), bb.order.size() * sizeof(uint32_t));
    return TRB_OK;
}

static trb_status bvh_device_check(int device, uint32_t n) {
    if (n >= (1u << 31)) return fail(TRB_UNSUPPORTED, "more than 2^31 - 1 boxes");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(TRB_NO_DEVICE, "no CUDA device: tray_rust_b200 has no CPU fallback"); }
    if (device < 0 || device >= ndev) return fail(TRB_INVALID_ARG, "device ordinal out of range");
    CU(cudaSetDevice(device));
    return TRB_OK;
}

trb_status trb_build_bvh_device(int device, const float* d_boxes6, uint32_t n, uint32_t max_geom, uint32_t* d_n_nodes, trb_bvh_node* d_nodes,
                                uint32_t* d_ordered, void* cuda_stream) {
    if (!d_boxes6 || n == 0 || !d_n_nodes || !d_nodes || !d_ordered) return fail(TRB_INVALID_ARG, "null buffer or empty geometry");
    const trb_status c = bvh_device_check(device, n);
    if (c != TRB_OK) return c;
    bool empty = false;
    CU(trb::bvhb::build_device(d_boxes6, n, max_geom, d_n_nodes, d_nodes, d_ordered, (cudaStream_t)cuda_stream, &g_launches, &empty));
    if (empty) return fail(TRB_INVALID_ARG, "the SAH build would split a node into an empty child (infinite coordinates)");
    return TRB_OK;
}

trb_status trb_build_bvh(int device, const float* boxes6, uint32_t n, uint32_t max_geom, uint32_t* n_nodes, trb_bvh_node* nodes, uint32_t* ordered) {
    if (!boxes6 || n == 0 || !n_nodes) return fail(TRB_INVALID_ARG, "empty geometry"); // bvh.rs:35 assert!(!geometry.is_empty())
    const trb_status c = bvh_device_check(device, n);
    if (c != TRB_OK) return c;
    DeviceBuffer order, tree; // order: + one word, the node count; both outlive run_staged's drain
    return run_staged({{boxes6, 24 * (size_t)n}}, {}, [&](const DeviceBuffer* d) {
        trb_status r;
        if ((r = order.alloc(4 * ((size_t)n + 1), "BVH build scratch")) != TRB_OK || (r = tree.alloc((2 * (size_t)n - 1) * sizeof(trb_bvh_node), "BVH build scratch")) != TRB_OK)
            return r;
        uint32_t* d_order = order.as<uint32_t>();
        bool empty = false;
        CU(trb::bvhb::build_device(d[0].as<float>(), n, max_geom, d_order + n, tree.as<trb_bvh_node>(), d_order, 0, &g_launches, &empty));
        if (empty) return fail(TRB_INVALID_ARG, "the SAH build would split a node into an empty child (infinite coordinates)");
        CU(cudaMemcpy(n_nodes, d_order + n, 4, cudaMemcpyDeviceToHost));
        if (nodes) CU(cudaMemcpy(nodes, tree.p, (size_t)*n_nodes * sizeof(trb_bvh_node), cudaMemcpyDeviceToHost));
        if (ordered) CU(cudaMemcpy(ordered, d_order, 4 * (size_t)n, cudaMemcpyDeviceToHost));
        return TRB_OK;
    });
}

trb_status trb_host_keyframe_transform(const trb_keyframe* kf, float* mat16, float* inv16) {
    if (!kf || !mat16 || !inv16) return fail(TRB_INVALID_ARG, "null argument");
    const Xf x = keyframe_xf(*kf);
    std::memcpy(mat16, x.fwd.m, 64); std::memcpy(inv16, x.inv.m, 64);
    return TRB_OK;
}

// Layout check without a GPU: every ray is traversed (a) literally like bvh.rs:81-130 over the reference-order nodes and
// (b) through the DQuad records with quad_visit — the function the trace kernel runs — and the two must visit the same
// leaves in the same order with the same max_t history. Leaves "hit" pseudo-randomly (a hash of leaf and ray decides a
// distance) so that max_t shrinks during the walk. Returns the number of rays whose walks differ.
trb_status trb_selftest_box(uint32_t n_cases, uint32_t seed, uint64_t out[4]) {
    if (!out || n_cases == 0) return fail(TRB_INVALID_ARG, "null argument");
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) { cudaGetLastError(); return fail(TRB_NO_DEVICE, "no CUDA device"); }
    return run_staged({}, {{out, 4 * sizeof(uint64_t)}}, [&](const DeviceBuffer* d) {
        CU(cudaMemset(d[0].p, 0, 4 * sizeof(unsigned long long)));
        trb::k_selftest_box<<<(n_cases + 255) / 256, 256>>>(n_cases, seed, d[0].as<unsigned long long>());
        g_launches++;
        return TRB_OK;
    });
}

trb_status trb_host_quad_check(const trb_bvh_node* nodes, uint32_t n_nodes, const trb_ray* rays, uint32_t n_rays, uint32_t* mismatches,
                               uint64_t* leaf_visits, uint64_t* quad_visits) {
    if (!nodes || !rays || !mismatches || n_nodes == 0) return fail(TRB_INVALID_ARG, "null argument");
    const std::vector<trb_bvh_node> in(nodes, nodes + n_nodes);
    std::vector<trb::DQuad> quads;
    uint32_t qroot = 0;
    if (!pack_quads(in, quads, qroot)) return fail(TRB_UNSUPPORTED, "leaf encoding");
    uint32_t bad = 0; uint64_t nl = 0, nq = 0;
    auto leaf_hit = [](uint32_t first, uint32_t ray, float tmin, float& tmax) {
        uint32_t h = (first * 0x9E3779B1u) ^ (ray * 0x85EBCA77u); h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
        if ((h & 3u) == 0) { const float tc = tmin + (float)(h >> 8) * (1.0f / 16777216.0f) * 40.0f; if (tc >= tmin && tc <= tmax) tmax = tc; }
    };
    for (uint32_t ri = 0; ri < n_rays; ++ri) {
        const trb_ray& r = rays[ri];
        const trb::f3 o = trb::mk(r.o[0], r.o[1], r.o[2]);
        const trb::f3 inv = trb::mk(1.0f / r.d[0], 1.0f / r.d[1], 1.0f / r.d[2]);
        const bool nx = r.d[0] < 0.0f, ny = r.d[1] < 0.0f, nz = r.d[2] < 0.0f;
        const bool neg[3] = {nx, ny, nz};
        if (!(std::isfinite(inv.x) && std::isfinite(inv.y) && std::isfinite(inv.z))) continue; // these rays take the DPair path
        // (a) the reference loop
        std::vector<uint32_t> seq_a, seq_b;
        float tmax_a = r.max_t, tmax_b = r.max_t;
        {
            uint32_t stack[64]; int sp = 0; uint32_t cur = 0;
            for (;;) {
                const trb_bvh_node& n = in[cur];
                float te;
                const float4 lo = make_float4(n.bmin[0], n.bmin[1], n.bmin[2], 0.f), hi = make_float4(n.bmax[0], n.bmax[1], n.bmax[2], 0.f);
                if (trb::box_hit(lo, hi, o, inv, nx, ny, nz, r.min_t, tmax_a, te)) {
                    if (n.b & TRB_BVH_LEAF) {
                        seq_a.push_back(n.a); leaf_hit(n.a, ri, r.min_t, tmax_a);
                        if (sp == 0) break;
                        cur = stack[--sp];
                    } else {
                        if (neg[n.b & 3u]) { stack[sp++] = cur + 1; cur = n.a; } else { stack[sp++] = n.a; cur += 1; }
                    }
                } else { if (sp == 0) break; cur = stack[--sp]; }
            }
        }
        // (b) root box, then DQuad records with a stack of (entry distance, reference)
        {
            const trb_bvh_node& n = in[0];
            float te;
            const float4 lo = make_float4(n.bmin[0], n.bmin[1], n.bmin[2], 0.f), hi = make_float4(n.bmax[0], n.bmax[1], n.bmax[2], 0.f);
            std::vector<unsigned long long> stack;
            uint32_t cur = trb::box_hit(lo, hi, o, inv, nx, ny, nz, r.min_t, tmax_b, te) ? qroot : 0xffffffffu;
            for (;;) {
                if (cur == 0xffffffffu) { // pop
                    bool got = false;
                    while (!stack.empty()) {
                        const unsigned long long e = stack.back(); stack.pop_back();
                        float tent; const uint32_t tb = (uint32_t)(e >> 32); std::memcpy(&tent, &tb, 4);
                        if (tent < tmax_b) { cur = (uint32_t)e; got = true; break; }
                    }
                    if (!got) break;
                }
                if ((cur & trb::REF_TAG) == trb::REF_LEAF) {
                    const uint32_t first = cur & 0x01ffffffu;
                    seq_b.push_back(first); leaf_hit(first, ri, r.min_t, tmax_b);
                    cur = 0xffffffffu;
                } else {
                    const float4* q = quads[cur].q;
                    trb::QuadOut qo;
                    trb::quad_visit(q[0], q[1], q[2], q[3], q[4], q[5], q[6], q[7], o, inv, nx, ny, nz, r.min_t, tmax_b, qo);
                    ++nq;
                    if (qo.p0) stack.push_back(qo.e0);
                    if (qo.p1) stack.push_back(qo.e1);
                    if (qo.p2) stack.push_back(qo.e2);
                    cur = qo.next;
                }
            }
        }
        nl += seq_a.size();
        if (seq_a != seq_b || std::memcmp(&tmax_a, &tmax_b, 4) != 0) ++bad;
    }
    *mismatches = bad;
    if (leaf_visits) *leaf_visits = nl;
    if (quad_visits) *quad_visits = nq;
    return TRB_OK;
}

trb_status trb_host_animated_transform(const trb_scene_desc* d, uint32_t first, uint32_t count, float time, float* mat16, float* inv16) {
    if (!d || !mat16 || !inv16) return fail(TRB_INVALID_ARG, "null argument");
    const trb_status r = validate(d);
    if (r != TRB_OK) return r;
    if ((uint64_t)first + count > d->n_splines) return fail(TRB_INVALID_ARG, "spline range out of bounds");
    std::vector<float> knots(d->knots, d->knots + d->n_knots); // BSpline::new sorts its knots
    for (uint32_t k = first; k < first + count; ++k)
        if (d->splines[k].n_ctrl > 1) std::stable_sort(knots.begin() + d->splines[k].knot_first, knots.begin() + d->splines[k].knot_first + d->splines[k].n_knots);
    const Xf x = trbh::animated_xf(d->splines, first, count, d->keyframes, knots.data(), time);
    std::memcpy(mat16, x.fwd.m, 64); std::memcpy(inv16, x.inv.m, 64);
    return TRB_OK;
}

trb_status trb_host_animated_color(const trb_scene_desc* d, uint32_t first, uint32_t count, float time, float* rgb3) {
    if (!d || !rgb3) return fail(TRB_INVALID_ARG, "null argument");
    if (count == 0 || (uint64_t)first + count > d->n_color_keys) return fail(TRB_INVALID_ARG, "colour key range out of bounds");
    trbh::animated_color(d->color_keys, first, count, time, rgb3);
    return TRB_OK;
}


// ---------------------------------------------------------------------------------------------------------------
// Multi-GPU (SURVEY 8e): tile sharding + one film SUM-reduce per frame with NCCL called directly (no torch).
// libnccl is resolved at run time so that the single-GPU library has no link-time dependency on it.
// ---------------------------------------------------------------------------------------------------------------
} // extern "C"

namespace {
struct NcclApi {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Reduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;
trb_status nccl_load() {
    if (g_nccl.lib) return TRB_OK;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD); // the copy the process already uses (e.g. PyTorch's)
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return fail(TRB_NCCL, std::string("cannot load libnccl.so.2: ") + (dlerror() ? dlerror() : "not found"));
    NcclApi a; a.lib = h;
#define TRB_SYM(field, name) a.field = reinterpret_cast<decltype(a.field)>(dlsym(h, name)); if (!a.field) return fail(TRB_NCCL, "libnccl lacks " name)
    TRB_SYM(GetUniqueId, "ncclGetUniqueId"); TRB_SYM(CommInitRank, "ncclCommInitRank"); TRB_SYM(CommInitAll, "ncclCommInitAll");
    TRB_SYM(CommDestroy, "ncclCommDestroy"); TRB_SYM(Reduce, "ncclReduce"); TRB_SYM(GroupStart, "ncclGroupStart"); TRB_SYM(GroupEnd, "ncclGroupEnd");
    TRB_SYM(GetErrorString, "ncclGetErrorString");
#undef TRB_SYM
    g_nccl = a;
    return TRB_OK;
}
#define NC(call)                                                                                                   \
    do {                                                                                                           \
        ncclResult_t r_ = (call);                                                                                  \
        if (r_ != ncclSuccess) return fail(TRB_NCCL, std::string(#call) + ": " + g_nccl.GetErrorString(r_));       \
    } while (0)
} // namespace

struct trb_comm { ncclComm_t comm = nullptr; int n_ranks = 1, rank = 0, device = 0; };
struct trb_group { std::vector<trb_scene*> scenes; std::vector<ncclComm_t> comms; std::vector<int> devices; };

namespace {
// this rank's shard of the selected block list inside cfg (interleaved chunks unless the caller asked for the reference's contiguous ranges)
trb_status shard_cfg(const trb_scene* s, const trb_render_cfg* in, int rank, int n_ranks, trb_render_cfg* out, bool* empty) {
    *out = *in; *empty = false;
    if (n_ranks <= 1) { out->shard_index = out->shard_count = out->shard_chunk = 0; return TRB_OK; }
    if (in->shard_count == 0xffffffffu) { // exec/distrib/master.rs:91-93,218-224: floor(B / W) blocks each, the remainder to the last worker
        const uint32_t all = (s->film.width / 8) * (s->film.height / 8);
        const uint32_t sel0 = in->block_count ? std::min(in->block_start, all) : 0u;
        const uint32_t sel = in->block_count ? (uint32_t)std::min<uint64_t>(all - sel0, in->block_count) : all;
        const uint32_t per = sel / (uint32_t)n_ranks, start = sel0 + (uint32_t)rank * per;
        const uint32_t count = rank == n_ranks - 1 ? sel0 + sel - start : per;
        out->block_start = start; out->block_count = count; out->shard_index = out->shard_count = out->shard_chunk = 0;
        *empty = count == 0; // block_count 0 would mean "all blocks" (block_queue.rs:39-41): an idle rank must not render
        return TRB_OK;
    }
    out->shard_index = (uint32_t)rank; out->shard_count = (uint32_t)n_ranks; out->shard_chunk = in->shard_chunk ? in->shard_chunk : 32u;
    return TRB_OK;
}
// The scene's AOV films of a sharded or group AOV render (trb_scene::d_shard_aov), allocated on first use
trb_status shard_aov_films(trb_scene* s, AovRequest& req) {
    const size_t npx = (size_t)s->film.width * s->film.height;
    if (!s->d_shard_aov) {
        const trb_status r = device_alloc(&s->d_shard_aov, npx * (2 * sizeof(float4) + sizeof(uint64_t)), "AOV films");
        if (r != TRB_OK) return r;
    }
    float4* f = static_cast<float4*>(s->d_shard_aov);
    req = {nullptr, f, f + npx, reinterpret_cast<unsigned long long*>(f + 2 * npx)};
    return TRB_OK;
}
// Exec::render on one replica with the film left on the device: update_frame, clear, all passes of this shard (LowDiscrepancy,
// or the Adaptive sampler's rounds when `ad` is set). With `aov` it also renders the three AOVs into the scene's AOV films,
// cleared first (albedo_w and normal_w to zero, nearest to all ones), so that an empty shard contributes nothing to the reduce.
trb_status render_to_device_film(trb_scene* s, const trb_render_cfg* cfg, const trb_adaptive* ad, bool empty, cudaStream_t st, bool aov = false) {
    CU(cudaSetDevice(s->device));
    if (!(cfg->flags & TRB_RENDER_NO_UPDATE)) {
        const float step = s->film.scene_time / (float)s->film.frames;
        trb_status r = trb_scene_update_frame(s, cfg->current_frame, (float)cfg->current_frame * step, ((float)cfg->current_frame + 1.0f) * step);
        if (r != TRB_OK) return r;
    }
    const size_t npx = (size_t)s->film.width * s->film.height;
    CU(cudaMemsetAsync(s->d_film, 0, npx * sizeof(float4), st));
    CU(cudaMemsetAsync(s->d_stats, 0, sizeof(trb::DStats), st));
    AovRequest req{nullptr, nullptr, nullptr, nullptr};
    if (aov) {
        trb_status r = shard_aov_films(s, req);
        if (r != TRB_OK) return r;
        CU(cudaMemsetAsync(req.albedo_w, 0, 2 * npx * sizeof(float4), st)); // albedo_w and normal_w
        CU(cudaMemsetAsync(req.nearest, 0xff, npx * sizeof(uint64_t), st));
    }
    if (empty) return TRB_OK;
    if (ad) { // per-pixel counts to d_ad_spp, for shard_pixel_spp_out
        trb_status r = ensure_adaptive(s);
        if (r != TRB_OK) return r;
        if (aov)
            return render_adaptive_device(s, cfg, ad, reinterpret_cast<float*>(s->d_film), &req, s->d_ad_spp, reinterpret_cast<trb_stats*>(s->d_stats), st);
        return trb_render_adaptive_device(s, cfg, ad, reinterpret_cast<float*>(s->d_film), s->d_ad_spp, reinterpret_cast<trb_stats*>(s->d_stats), st);
    }
    if (aov) return render_device(s, cfg, reinterpret_cast<float*>(s->d_film), reinterpret_cast<trb_stats*>(s->d_stats), st, &req);
    return trb_render_device(s, cfg, reinterpret_cast<float*>(s->d_film), reinterpret_cast<trb_stats*>(s->d_stats), st);
}
// the Adaptive sampler's per-pixel counts of this replica's shard -> pixel_spp (host, width*height; other entries untouched)
trb_status shard_pixel_spp_out(trb_scene* s, const trb_render_cfg* mine, bool empty, uint32_t* pixel_spp) {
    if (!pixel_spp || empty) return TRB_OK;
    CU(cudaSetDevice(s->device));
    uint32_t nb;
    const uint2* d_blocks = nullptr;
    trb_status r = ensure_blocks(s, mine, &d_blocks, &nb); // the list the render used (cached per selection)
    if (r != TRB_OK) return r;
    return adaptive_pixel_spp_out(s, d_blocks, nb, pixel_spp);
}
trb_status film_to_host_add(trb_scene* s, float* film, cudaStream_t st) {
    const size_t npx = (size_t)s->film.width * s->film.height;
    CU(cudaMemcpyAsync(s->h_film_staging, s->d_film, npx * sizeof(float4), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    add_film(film, s->h_film_staging, npx * 4);
    return TRB_OK;
}
// The AOV films of a sharded or group AOV render, reduced into `root`'s: albedo_w and normal_w (one run of 8 floats per pixel) summed
// like the colour film, nearest min-reduced. Exact for nearest: a sample writes only its own pixel and the shards own disjoint pixels,
// so each pixel's key comes from one replica and the others hold all ones (DESIGN.md §4 "Multi-GPU AOVs"). Inside the caller's
// ncclGroupStart/End, next to the colour film's reduce.
trb_status reduce_aov_films(trb_scene* s, ncclComm_t comm, int root, cudaStream_t st) {
    const size_t npx = (size_t)s->film.width * s->film.height;
    float4* f = static_cast<float4*>(s->d_shard_aov);
    NC(g_nccl.Reduce(f, f, npx * 8, ncclFloat, ncclSum, root, comm, st));
    NC(g_nccl.Reduce(f + 2 * npx, f + 2 * npx, npx, ncclUint64, ncclMin, root, comm, st));
    return TRB_OK;
}
// The root's AOV films into the caller's host buffers, as trb_render_aov leaves them: albedo_w and normal_w added into, nearest
// min-merged with what the caller's buffer holds; a NULL member (or a NULL aov) is skipped
trb_status aov_films_to_host(trb_scene* s, const trb_aov_film* aov) {
    if (!aov) return TRB_OK;
    CU(cudaSetDevice(s->device));
    const size_t npx = (size_t)s->film.width * s->film.height;
    const float4* f = static_cast<const float4*>(s->d_shard_aov);
    std::vector<float> h;
    for (auto [dst, src] : {std::pair<float*, const float4*>{aov->albedo_w, f}, {aov->normal_w, f + npx}}) {
        if (!dst) continue;
        h.resize(npx * 4);
        CU(cudaMemcpy(h.data(), src, npx * sizeof(float4), cudaMemcpyDeviceToHost));
        add_film(dst, h.data(), npx * 4);
    }
    if (aov->nearest) {
        std::vector<uint64_t> v(npx);
        CU(cudaMemcpy(v.data(), f + 2 * npx, npx * sizeof(uint64_t), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < npx; ++i) aov->nearest[i] = std::min(aov->nearest[i], v[i]);
    }
    return TRB_OK;
}
} // namespace

extern "C" {

trb_status trb_nccl_unique_id(void* id128) {
    if (!id128) return fail(TRB_INVALID_ARG, "null argument");
    trb_status r = nccl_load();
    if (r != TRB_OK) return r;
    ncclUniqueId id;
    NC(g_nccl.GetUniqueId(&id));
    static_assert(sizeof(ncclUniqueId) == TRB_NCCL_UNIQUE_ID_BYTES, "ncclUniqueId size");
    std::memcpy(id128, &id, sizeof id);
    return TRB_OK;
}

trb_status trb_comm_create(const void* id128, int n_ranks, int rank, int device, trb_comm** out) {
    if (!id128 || !out || n_ranks < 1 || rank < 0 || rank >= n_ranks) return fail(TRB_INVALID_ARG, "bad communicator arguments");
    *out = nullptr;
    trb_status r = nccl_load();
    if (r != TRB_OK) return r;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(TRB_NO_DEVICE, "no CUDA device: tray_rust_b200 has no CPU fallback");
    if (device < 0 || device >= ndev) return fail(TRB_INVALID_ARG, "device ordinal out of range");
    CU(cudaSetDevice(device));
    ncclUniqueId id;
    std::memcpy(&id, id128, sizeof id);
    std::unique_ptr<trb_comm> c(new trb_comm);
    c->n_ranks = n_ranks; c->rank = rank; c->device = device;
    NC(g_nccl.CommInitRank(&c->comm, n_ranks, id, rank));
    *out = c.release();
    return TRB_OK;
}

void trb_comm_destroy(trb_comm* c) {
    if (!c) return;
    if (c->comm && g_nccl.CommDestroy) { cudaSetDevice(c->device); g_nccl.CommDestroy(c->comm); }
    delete c;
}

trb_status trb_comm_info(const trb_comm* c, int* n_ranks, int* rank) {
    if (!c) return fail(TRB_INVALID_ARG, "null communicator");
    if (n_ranks) *n_ranks = c->n_ranks;
    if (rank) *rank = c->rank;
    return TRB_OK;
}

trb_status trb_comm_reduce_film(trb_comm* c, float* d_film, size_t n, int root, void* stream) {
    if (!c || !d_film || root < 0 || root >= c->n_ranks) return fail(TRB_INVALID_ARG, "bad reduce arguments");
    if (c->n_ranks == 1) return TRB_OK;
    CU(cudaSetDevice(c->device));
    NC(g_nccl.Reduce(d_film, d_film, n, ncclFloat, ncclSum, root, c->comm, static_cast<cudaStream_t>(stream)));
    return TRB_OK;
}

} // extern "C"

namespace {
// trb_render_sharded (ad == nullptr) and trb_render_sharded_adaptive; with `with_aov` their AOV forms, whose host AOV films `aov`
// are the root's only (every rank renders and reduces all three AOVs)
trb_status render_sharded(trb_scene* s, trb_comm* c, const trb_render_cfg* cfg, const trb_adaptive* ad, int root, float* film, uint32_t* pixel_spp,
                          trb_stats* stats, bool with_aov = false, const trb_aov_film* aov = nullptr) {
    if (!s || !c || !cfg || root < 0 || root >= c->n_ranks) return fail(TRB_INVALID_ARG, "null or bad argument");
    if (c->rank == root && !film) return fail(TRB_INVALID_ARG, "the root rank needs a film buffer");
    if (with_aov && c->rank == root && !aov) return fail(TRB_INVALID_ARG, "null argument");
    if (c->device != s->device) return fail(TRB_INVALID_ARG, "scene and communicator live on different devices");
    if (ad) { // before sharding: a rank whose shard is empty answers like the others
        trbh::AdSchedule sch;
        trb_status r = adaptive_check(s, cfg, ad, sch);
        if (r != TRB_OK) return r;
    } else if (with_aov) { // adaptive_check's statuses cover aov_supported's
        trb_status r = aov_supported(s, cfg);
        if (r != TRB_OK) return r;
    }
    trb_render_cfg mine; bool empty;
    trb_status r = shard_cfg(s, cfg, c->rank, c->n_ranks, &mine, &empty);
    if (r != TRB_OK) return r;
    auto t0 = std::chrono::steady_clock::now();
    CU(cudaSetDevice(s->device));
    CU(cudaEventRecord(s->ev0, 0));
    r = render_to_device_film(s, &mine, ad, empty, nullptr, with_aov);
    if (r != TRB_OK) return r;
    CU(cudaEventRecord(s->ev1, 0));
    const size_t nfl = (size_t)s->film.width * s->film.height * 4;
    if (with_aov && c->n_ranks > 1) { // ONE NCCL group per frame: the colour film and the three AOVs
        NC(g_nccl.GroupStart());
        NC(g_nccl.Reduce(s->d_film, s->d_film, nfl, ncclFloat, ncclSum, root, c->comm, nullptr));
        r = reduce_aov_films(s, c->comm, root, nullptr);
        NC(g_nccl.GroupEnd());
    } else {
        r = trb_comm_reduce_film(c, reinterpret_cast<float*>(s->d_film), nfl, root, nullptr); // ONE reduce per frame
    }
    if (r != TRB_OK) return r;
    if (c->rank == root) {
        r = film_to_host_add(s, film, nullptr);
        if (r == TRB_OK && with_aov) r = aov_films_to_host(s, aov);
        if (r != TRB_OK) return r;
    }
    else CU(cudaStreamSynchronize(nullptr));
    r = check_error_flag(s);
    if (r != TRB_OK) return r;
    if (ad) { r = shard_pixel_spp_out(s, &mine, empty, pixel_spp); if (r != TRB_OK) return r; }
    if ((r = stats_readback(s, stats, 0.f)) != TRB_OK) return r;
    if (stats) stats->update_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count() - stats->kernel_ms;
    return TRB_OK;
}
} // namespace

extern "C" {

trb_status trb_render_sharded(trb_scene* s, trb_comm* c, const trb_render_cfg* cfg, int root, float* film, trb_stats* stats) {
    return render_sharded(s, c, cfg, nullptr, root, film, nullptr, stats);
}

trb_status trb_render_sharded_adaptive(trb_scene* s, trb_comm* c, const trb_render_cfg* cfg, const trb_adaptive* ad, int root, float* film,
                                       uint32_t* pixel_spp, trb_stats* stats) {
    if (!ad) return fail(TRB_INVALID_ARG, "null argument");
    return render_sharded(s, c, cfg, ad, root, film, pixel_spp, stats);
}

trb_status trb_render_sharded_aov(trb_scene* s, trb_comm* c, const trb_render_cfg* cfg, int root, float* film, const trb_aov_film* aov, trb_stats* stats) {
    return render_sharded(s, c, cfg, nullptr, root, film, nullptr, stats, true, aov);
}

trb_status trb_render_sharded_adaptive_aov(trb_scene* s, trb_comm* c, const trb_render_cfg* cfg, const trb_adaptive* ad, int root, float* film,
                                           const trb_aov_film* aov, uint32_t* pixel_spp, trb_stats* stats) {
    if (!ad) return fail(TRB_INVALID_ARG, "null argument");
    return render_sharded(s, c, cfg, ad, root, film, pixel_spp, stats, true, aov);
}

trb_status trb_group_create(const trb_scene_desc* desc, const int* devices, int n, trb_group** out) {
    if (!out || !devices || n < 1) return fail(TRB_INVALID_ARG, "bad group arguments");
    *out = nullptr;
    for (int i = 0; i < n; ++i) for (int j = 0; j < i; ++j) if (devices[i] == devices[j]) return fail(TRB_INVALID_ARG, "duplicate device in group");
    std::unique_ptr<trb_group> g(new trb_group);
    g->devices.assign(devices, devices + n);
    auto cleanup = [&]() { for (trb_scene* s : g->scenes) trb_scene_destroy(s); g->scenes.clear(); };
    // replicas are built concurrently (the per-mesh SAH build is host work)
    std::vector<trb_scene*> scenes(n, nullptr);
    std::vector<trb_status> rc(n, TRB_OK);
    std::vector<std::string> msg(n);
    std::vector<std::thread> th;
    for (int i = 0; i < n; ++i) th.emplace_back([&, i]() { rc[i] = trb_scene_create(desc, devices[i], &scenes[i]); if (rc[i] != TRB_OK) msg[i] = trb_last_error(); });
    for (auto& t : th) t.join();
    g->scenes = scenes;
    for (int i = 0; i < n; ++i) if (rc[i] != TRB_OK) { g->scenes.erase(std::remove(g->scenes.begin(), g->scenes.end(), nullptr), g->scenes.end()); cleanup(); return fail(rc[i], msg[i]); }
    if (n > 1) {
        trb_status r = nccl_load();
        if (r != TRB_OK) { cleanup(); return r; }
        g->comms.resize(n);
        ncclResult_t e = g_nccl.CommInitAll(g->comms.data(), n, devices);
        if (e != ncclSuccess) { cleanup(); return fail(TRB_NCCL, std::string("ncclCommInitAll: ") + g_nccl.GetErrorString(e)); }
    }
    *out = g.release();
    return TRB_OK;
}

trb_status trb_group_load_json(const char* path, uint32_t w, uint32_t h, uint32_t spp, const int* devices, int n, trb_group** out) {
    trb_scene_desc* d = nullptr;
    trb_status r = trb_desc_load_json(path, w, h, spp, &d);
    if (r != TRB_OK) return r;
    r = trb_group_create(d, devices, n, out);
    const std::string keep = g_error;
    trb_desc_free(d);
    g_error = keep;
    return r;
}

trb_scene* trb_group_scene(trb_group* g, int i) { return (g && i >= 0 && i < (int)g->scenes.size()) ? g->scenes[i] : nullptr; }

void trb_group_destroy(trb_group* g) {
    if (!g) return;
    for (size_t i = 0; i < g->comms.size(); ++i) if (g->comms[i]) { cudaSetDevice(g->devices[i]); g_nccl.CommDestroy(g->comms[i]); }
    for (trb_scene* s : g->scenes) trb_scene_destroy(s);
    delete g;
}

} // extern "C"

namespace {
// trb_group_render (ad == nullptr) and trb_group_render_adaptive; with `aov` their AOV forms
trb_status group_render(trb_group* g, const trb_render_cfg* cfg, const trb_adaptive* ad, float* film, uint32_t* pixel_spp, trb_stats* stats,
                        const trb_aov_film* aov = nullptr) {
    if (!g || !cfg || !film) return fail(TRB_INVALID_ARG, "null argument");
    const int n = (int)g->scenes.size();
    for (const trb_scene* s : g->scenes) // the film reduce is sized by replica 0 (trb_scene_replace_settings edits one replica at a time)
        if (s->film.width != g->scenes[0]->film.width || s->film.height != g->scenes[0]->film.height)
            return fail(TRB_INVALID_ARG, "the group's replicas have different film sizes");
    if (n == 1 && aov)
        return ad ? trb_render_adaptive_aov(g->scenes[0], cfg, ad, film, aov, pixel_spp, stats) : trb_render_aov(g->scenes[0], cfg, film, aov, stats);
    if (n == 1) return ad ? trb_render_adaptive(g->scenes[0], cfg, ad, film, pixel_spp, stats) : trb_render(g->scenes[0], cfg, film, stats);
    if (ad) {
        trbh::AdSchedule sch;
        trb_status r = adaptive_check(g->scenes[0], cfg, ad, sch);
        if (r != TRB_OK) return r;
    }
    if (aov) // every replica, before any renders (adaptive_check's statuses cover aov_supported's on replica 0)
        for (const trb_scene* s : g->scenes) { const trb_status r = aov_supported(s, cfg); if (r != TRB_OK) return r; }
    auto t0 = std::chrono::steady_clock::now();
    // enqueue every replica's shard (update_frame is host work per replica; the kernels of all devices then run concurrently)
    std::vector<trb_status> rc(n, TRB_OK);
    std::vector<std::string> msg(n);
    std::vector<trb_render_cfg> mine(n);
    std::vector<char> empty(n, 0);
    std::vector<std::thread> th;
    for (int i = 0; i < n; ++i) th.emplace_back([&, i]() {
        bool e = false;
        rc[i] = shard_cfg(g->scenes[i], cfg, i, n, &mine[i], &e);
        empty[i] = e;
        if (rc[i] == TRB_OK) { cudaSetDevice(g->scenes[i]->device); cudaEventRecord(g->scenes[i]->ev0, 0); rc[i] = render_to_device_film(g->scenes[i], &mine[i], ad, e, nullptr, aov != nullptr); cudaEventRecord(g->scenes[i]->ev1, 0); }
        if (rc[i] != TRB_OK) msg[i] = trb_last_error();
    });
    for (auto& t : th) t.join();
    for (int i = 0; i < n; ++i) if (rc[i] != TRB_OK) return fail(rc[i], msg[i]);
    const size_t nfl = (size_t)g->scenes[0]->film.width * g->scenes[0]->film.height * 4;
    NC(g_nccl.GroupStart()); // ONE reduce per frame, root = devices[0] (with the AOVs: one NCCL group of the colour film and the three AOVs)
    for (int i = 0; i < n; ++i) {
        CU(cudaSetDevice(g->scenes[i]->device));
        NC(g_nccl.Reduce(g->scenes[i]->d_film, g->scenes[i]->d_film, nfl, ncclFloat, ncclSum, 0, g->comms[i], nullptr));
        if (aov) { const trb_status r = reduce_aov_films(g->scenes[i], g->comms[i], 0, nullptr); if (r != TRB_OK) return r; }
    }
    NC(g_nccl.GroupEnd());
    CU(cudaSetDevice(g->scenes[0]->device));
    trb_status r = film_to_host_add(g->scenes[0], film, nullptr);
    if (r == TRB_OK && aov) r = aov_films_to_host(g->scenes[0], aov);
    if (r != TRB_OK) return r;
    float kernel_ms = 0.f;
    if (stats) std::memset(stats, 0, sizeof *stats);
    for (int i = 0; i < n; ++i) {
        CU(cudaSetDevice(g->scenes[i]->device));
        CU(cudaDeviceSynchronize());
        r = check_error_flag(g->scenes[i]);
        if (r != TRB_OK) return r;
        if (ad) { r = shard_pixel_spp_out(g->scenes[i], &mine[i], empty[i] != 0, pixel_spp); if (r != TRB_OK) return r; } // the replicas' pixels are disjoint
        if (stats) {
            trb_stats one;
            if ((r = stats_readback(g->scenes[i], &one, 0.f)) != TRB_OK) return r;
            stats->camera_samples += one.camera_samples; stats->rays_primary += one.rays_primary; stats->rays_shadow += one.rays_shadow; stats->rays_mis += one.rays_mis;
            stats->rays_continuation += one.rays_continuation; stats->node_tests += one.node_tests; stats->tri_tests += one.tri_tests; stats->inst_tests += one.inst_tests;
            kernel_ms = std::max(kernel_ms, one.kernel_ms);
        }
    }
    if (stats) { stats->kernel_ms = kernel_ms; stats->update_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count() - kernel_ms; }
    return TRB_OK;
}
} // namespace

extern "C" {

trb_status trb_group_render(trb_group* g, const trb_render_cfg* cfg, float* film, trb_stats* stats) {
    return group_render(g, cfg, nullptr, film, nullptr, stats);
}

trb_status trb_group_render_adaptive(trb_group* g, const trb_render_cfg* cfg, const trb_adaptive* ad, float* film, uint32_t* pixel_spp, trb_stats* stats) {
    if (!ad) return fail(TRB_INVALID_ARG, "null argument");
    return group_render(g, cfg, ad, film, pixel_spp, stats);
}

trb_status trb_group_render_aov(trb_group* g, const trb_render_cfg* cfg, float* film, const trb_aov_film* aov, trb_stats* stats) {
    if (!aov) return fail(TRB_INVALID_ARG, "null argument");
    return group_render(g, cfg, nullptr, film, nullptr, stats, aov);
}

trb_status trb_group_render_adaptive_aov(trb_group* g, const trb_render_cfg* cfg, const trb_adaptive* ad, float* film, const trb_aov_film* aov,
                                         uint32_t* pixel_spp, trb_stats* stats) {
    if (!ad || !aov) return fail(TRB_INVALID_ARG, "null argument");
    return group_render(g, cfg, ad, film, pixel_spp, stats, aov);
}

} // extern "C"
