// trb_device.h — device-resident scene layout (HBM), shared by the host code that fills it and the
// kernels that read it. See DESIGN.md "Data layout in HBM".
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/trb.h"
#include "trb_host.h" // trbh::Xf (host+device math shared with the per-frame host code)

namespace trb {

// One BVH node, 32 B, read as two 16-byte vector loads. Topology and order are the reference's
// (src/geometry/bvh.rs:248-267): node i's first child is i+1.
//   lo = (bmin.xyz, a)   interior: a = second_child            leaf: a = first primitive slot
//   hi = (bmax.xyz, b)   interior: b = split axis (0,1,2)      leaf: b = 0x80000000 | count
struct DNode { float4 lo, hi; };
constexpr uint32_t LEAF_BIT = 0x80000000u;

// Traversal layout: one 64-byte record per INTERIOR node of the reference tree holding BOTH children's
// boxes, so one fetch (four 16-byte loads, two 32-byte sectors) feeds two box tests and the dependent-load
// chain per ray is half as long. Topology, child order and every compare are unchanged (DESIGN.md
// "Node layout"). A child reference is 2 tag bits + 30 payload bits:
//   REF_INTERIOR | record index        REF_LEAF | count << 25 | first primitive slot     (narrow leaves)
//                                      REF_LEAF | first triangle slot (30 bits)          (wide mesh leaves)
// A wide leaf ends at the triangle that carries TRI_LEAF_END (DTri). A scene uses one form for all its meshes, and the
// host launches the kernel instantiations of that form (template flag WIDE); TLAS leaves are always narrow.
struct DPair {
    float4 l_lo; // left  (= first child, index+1) min, w = left reference
    float4 l_hi; // left  max,                       w = right reference
    float4 r_lo; // right (= second_child) min,      w = split axis of this node
    float4 r_hi; // right max
};
constexpr uint32_t REF_TAG = 0xc0000000u, REF_INTERIOR = 0x00000000u, REF_LEAF = 0x40000000u;

// Two levels of the reference tree in one 128-byte record: for an interior node P with children L (= first
// child) and R (= second_child), the four slots hold the boxes of L's children and R's children (a child that is
// a leaf occupies one slot with its own box; the other slot of that half is empty). A visit tests four boxes from one
// fetch, so the dependent-load chain per ray is half as long again. The boxes of L and R themselves are not tested:
// a child's box lies inside its parent's, and for a ray with finite 1/d every compare of BBox::fast_intersect is
// monotone in the box, so "grandchild hit" implies "child hit" at the same max_t (rays with a zero direction
// component use the DPair path). Visit ORDER is the reference's: near half first (P's axis), near slot first
// inside each half (that child's axis); entries are re-tested against the shrunken max_t when popped.
//   slot k: q[2k] = (lo.xyz, ref_k), q[2k+1] = (hi.xyz, -)   slots 0,1 = L's half, 2,3 = R's half
//   q[1].w = axis(P) | axis(L) << 2 | axis(R) << 4          ref = QUAD_EMPTY: unused slot
struct DQuad { float4 q[8]; };
constexpr uint32_t QUAD_EMPTY = 0xffffffffu;

struct DBvh {
    const DPair* pairs;
    const DQuad* quads;
    float4 root_lo; // root box min, w = root reference (DPair index space)
    float4 root_hi; // root box max, w = root reference (DQuad index space)
};
static_assert(sizeof(DBvh) == 48, "DBvh layout");

// One triangle in LEAF ORDER (slot k of the BLAS == ordered_geom[k]), padded to 64 B so that it is two aligned
// 32-byte loads (one L1TEX tag lookup each) and never straddles a 128-byte line:
// v0 = (pa.xyz, triangle index), e0 = (pb-pa, leaf mark), e1 = (pc-pa, 0) (the same single IEEE subtraction the
// reference performs per test, mesh.rs:140, hoisted to load time). The leaf mark is a bit pattern, never read as a
// float: TRI_LEAF_END on the last slot of every mesh leaf, 0 elsewhere. The wide mesh leaf references (no count,
// see DPair) walk a leaf up to the marked slot.
struct alignas(64) DTri { float4 v0, e0, e1, pad; };
static_assert(sizeof(DTri) == 64, "DTri layout");
constexpr uint32_t TRI_LEAF_END = 0xffffffffu;

struct DMesh {
    const float* positions; // 3 per vertex
    const float* normals;   // 3 per vertex
    const float* texcoords; // 2 per vertex
    const uint32_t* indices; // 3 per triangle
    DBvh bvh;               // BVH<Triangle>, max_geom 16 (mesh.rs:44)
    const DTri* tris;       // leaf order
    uint32_t n_nodes, n_tris;
};

// geometry::Instance with its world transform at the current frame (static instances: recomposed
// once per update_frame instead of once per ray — bit-identical, DESIGN.md "X1").
struct alignas(16) DInstance { // 208 B: the two matrices are read as 16-byte vectors
    float inv[16];  // world -> object, row-major 4x4 (last row kept: transform.rs:150-162 divides by w)
    float mat[16];  // object -> world
    uint32_t kind, shape;
    float p0, p1;
    uint32_t mesh, material;
    float emission[3];       // static emission (one colour key)
    uint32_t flags;          // DI_ANIM_XF: transform depends on ray time; DI_ANIM_EMISSION: keyframed emission
    uint32_t spline_first, n_splines;     // AnimatedTransform (into DScene::splines) when DI_ANIM_XF
    uint32_t emission_first, n_emission;  // colour keys (into DScene::color_keys) when DI_ANIM_EMISSION
    uint32_t anim_slot;      // index among the keyframed instances (DScene::anim_instances) when DI_ANIM_XF
    uint32_t pad;
    uint32_t xf_first, xf_count;  // the instance's whole transform stack (every level), for the per-frame device update
    uint32_t pad2[2];
};
constexpr uint32_t DI_ANIM_XF = 1u, DI_ANIM_EMISSION = 2u;
static_assert(sizeof(DInstance) == 208, "DInstance must stay 16-byte sized");

struct DMaterial {
    uint32_t type;
    float c0[3], c1[3];
    float roughness; // as given
    float width;     // Beckmann::new: max(roughness, 1e-6) (beckmann.rs:19-22)
    float eta;
    float on_a, on_b; // OrenNayar::new (oren_nayar.rs:26-34)
    uint32_t merl_off; // float offset into merl
    uint32_t pad;
    uint32_t tex[4];   // 1 + texture index bound to c0 / c1 / roughness / eta (0 = the constant), LoadedTextures::find_color / find_scalar
};

// texture::Image / AnimatedImage frames (src/texture/image.rs, animated_image.rs): RGBA8 texels of all images in one array
struct DImage { uint32_t width, height, offset; float time; }; // offset: first texel in DScene::texels
struct DTexture { uint32_t first_image, n_images; };

struct DCamera {
    float px_to_cam[16]; // proj_div_inv * raster_screen (camera.rs:152)
    float cam_mat[16];   // cam_world at the frame (static camera)
    float scaling[3];
    float shutter_open, shutter_close;
    uint32_t animated, spline_first, n_splines; // keyframed cam_world: evaluated at each ray's time (camera.rs:156)
};

struct DStats { // mirrors trb_stats' integer part
    unsigned long long camera_samples, rays_primary, rays_shadow, rays_mis, rays_continuation, node_tests, tri_tests, inst_tests;
};

struct DScene {
    const DBvh* tlas;            // BVH<Instance>, max_geom 4 (scene.rs:141); header in global memory like the meshes'
    const DPair* tlas_pairs;     // == tlas->pairs
    const DQuad* tlas_quads;     // == tlas->quads
    const uint32_t* tlas_order;  // ordered_geom
    const DInstance* instances;
    const DMesh* meshes;
    const DMaterial* materials;
    const float* merl;
    const uint32_t* lights;      // instance indices of the emitters, object order
    uint32_t n_instances, n_lights;
    uint32_t width, height;
    uint32_t min_depth, max_depth;
    DCamera cam;
    // film filter (render_target.rs:41-75)
    float filter_w, filter_h, filter_inv_w, filter_inv_h;
    int fpw_x, fpw_y;
    uint32_t film_block_filter; // the 2x2 lock-block sample filter of RenderTarget::write can reject (wide filters only)
    const float* filter_table; // 256 floats
    // animation (SURVEY 8f N1): the AnimatedTransform / AnimatedColor tables of the scene description, evaluated per ray
    const trb_spline* splines;
    const trb_keyframe* keyframes;
    const float* knots;
    const trb_color_key* color_keys;
    const trbh::Xf* level_xf; // per spline: Keyframe::transform of a one-control-point level (else unused)
    // distinct keyframed splines (by content): instances of one keyframed group carry copies of the group's spline, and
    // Keyframe::transform(BSpline::point(time)) of a spline is a pure function of (its content, time) — evaluated once per path and
    // distinct spline (k_wf_anim_table)
    const uint32_t* spline_uniq;  // per spline: index into uniq_splines, 0xffffffff for one-control-point levels
    const uint32_t* uniq_splines; // per distinct keyframed spline: a representative index into `splines`
    uint32_t n_uniq_splines;
    uint32_t has_anim; // any instance / camera / emission depends on time
    const uint32_t* anim_instances; // instance indices with DI_ANIM_XF, in instance order
    uint32_t n_anim_instances;
    // image textures (SURVEY 8f N3): sampled in Material::bsdf at the hit's (u, v, time)
    const DTexture* textures;
    const DImage* images;
    const uchar4* texels;
    uint32_t n_textures;
};

struct RenderParams {
    const uint2* blocks;   // Morton-ordered (bx, by) list after select_blocks
    uint32_t n_blocks;
    uint32_t spp;          // pow2
    uint32_t sample_first, sample_count;
    uint32_t seed;
    uint32_t* work_counter;
    float4* film;          // RGBW, row-major
    void* samples_out;     // trb_sample*, mode 1
    DStats* stats;
    int* error_flag;
    // Adaptive sampler round (zero for LowDiscrepancy): entry s of the round is sample_02(perm_pos(s) + ld_offset) at slot
    // sample_first + s (DESIGN.md §2 "Adaptive sampler"). The per-path sample arrays read ld_offset, LowDiscrepancy's is 0.
    uint32_t ld_offset;
    uint32_t ad_pos_len, ad_time_len; // permutation lengths of the positions (the round's count) and the times (max_spp)
    uint32_t ad_round;                // round index: pixel streams (seed, pixel, 0xfffffffe - round, dim)
    uint4* ad_state;                  // per image pixel trbh::AdPixel; nullptr: LowDiscrepancy
    const uint32_t* ad_block_index;   // index of each pass block in the caller's selected block list (parity records)
    uint32_t ad_min, ad_max, ad_step, ad_max_per_pixel;
    // Adaptive passes are enqueued for the worst case: the pass covers blocks [ad_b0, ad_b0 + n_blocks) of the round's list,
    // and *ad_live (written on the device by k_ad_init / k_ad_compact) is how many blocks that list really holds
    const uint32_t* ad_live;
    uint32_t ad_b0;
};

} // namespace trb
