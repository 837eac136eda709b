/* trb.h — C ABI of the H100-native (sm_90a) render path for tray_rust.
 *
 * This is the drop-in boundary for ONE path of the reference: the call
 *     Exec::render(&mut self, scene: &mut Scene, rt: &mut RenderTarget, config: &Config)
 * (/root/reference/src/exec/mod.rs:41-49; sole implementation
 * exec::MultiThreaded, src/exec/multithreaded.rs:54-114) and the data it consumes
 * (Scene, src/scene.rs:93-98) and produces (the RGBW f32 film in the layout of
 * RenderTarget::get_renderf32, src/film/render_target.rs:243-265).
 *
 * Everything here is plain C: POD structs, pointers and sizes. No torch types, no
 * C++ types, no callbacks into the host. The library owns all device memory behind
 * the opaque trb_scene handle; host buffers are borrowed for the duration of a call.
 *
 * All entry points return trb_status; on failure trb_last_error() (thread-local)
 * describes why. The conditions the reference panics on (image not a multiple of the
 * 8x8 block, no lights, empty scene, unknown types) are reported as
 * TRB_INVALID_ARG / TRB_UNSUPPORTED instead of aborting the process.
 */
#ifndef TRB_H
#define TRB_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TRB_ABI_VERSION 4u

typedef enum trb_status {
    TRB_OK = 0,
    TRB_INVALID_ARG = 1, /* what the reference would panic!/assert! on */
    TRB_CUDA = 2,        /* a CUDA runtime call or kernel failed */
    TRB_OOM = 3,
    TRB_UNSUPPORTED = 4, /* valid in the reference, not in this build (see DESIGN.md) */
    TRB_IO = 5,
    TRB_NO_DEVICE = 6,   /* no CUDA device: this library has no CPU fallback */
    TRB_NCCL = 7         /* an NCCL call failed, or libnccl.so.2 could not be loaded */
} trb_status;

/* ---------------------------------------------------------------------------------
 * Scene description (source-level, nothing derived: no matrices, no BVH).
 * It is the FFI-safe flattening of `Scene` + `RenderTarget` construction arguments
 * (src/scene.rs:93-146). Every array is caller-owned and deep-copied by
 * trb_scene_create.
 * ------------------------------------------------------------------------------- */

/* linalg::Keyframe (src/linalg/keyframe.rs:14-21): translation, rotation quaternion
 * (v.x, v.y, v.z, w), scaling. The reference stores EVERY transform this way (even a
 * static JSON one, src/linalg/animated_transform.rs:34-37) and recomposes T*R*S per
 * ray (keyframe.rs:60-63), so the TRS triple — not a matrix — is the ABI. */
typedef struct trb_keyframe {
    float translation[3];
    float rotation[4];
    float scaling[3];
} trb_keyframe;

/* bspline::BSpline<Keyframe> (animated_transform.rs:22-37): control points
 * keyframes[ctrl_first .. ctrl_first+n_ctrl), knots[knot_first .. knot_first+n_knots). */
typedef struct trb_spline {
    uint32_t degree;
    uint32_t n_ctrl;
    uint32_t ctrl_first;
    uint32_t n_knots;
    uint32_t knot_first;
} trb_spline;

/* film::ColorKeyframe (src/film/animated_color.rs:12-17), sorted by time. */
typedef struct trb_color_key {
    float rgba[4];
    float time;
} trb_color_key;

enum { /* geometry::Instance / EmitterType (src/geometry/instance.rs:81-84, emitter.rs:74-79) */
    TRB_INST_RECEIVER = 0,
    TRB_INST_EMITTER_AREA = 1,
    TRB_INST_EMITTER_POINT = 2
};
enum { /* shapes reachable from scene.rs:513-580 */
    TRB_SHAPE_NONE = 0,   /* point light */
    TRB_SHAPE_SPHERE = 1, /* p0 = radius                       (geometry/sphere.rs)    */
    TRB_SHAPE_DISK = 2,   /* p0 = radius, p1 = inner_radius    (geometry/disk.rs)      */
    TRB_SHAPE_RECT = 3,   /* p0 = width,  p1 = height; "plane" = 2x2 (scene.rs:527-528) */
    TRB_SHAPE_MESH = 4    /* mesh = index into meshes          (geometry/mesh.rs)      */
};

/* One geometry::Instance in JSON object order (group members flattened in place,
 * scene.rs:496-505). The AnimatedTransform is splines[spline_first .. +n_splines) in
 * application order (animated_transform.rs:42-54: transform = t_i * transform). */
typedef struct trb_instance {
    uint32_t kind;
    uint32_t shape;
    float p0, p1;
    uint32_t mesh;
    uint32_t material;
    uint32_t spline_first, n_splines;
    uint32_t emission_first, n_emission; /* color keys; emitters only */
} trb_instance;

/* geometry::Mesh buffers as produced by Mesh::load_obj (mesh.rs:49-76): positions and
 * normals 3 floats per vertex, texcoords 2 floats per vertex, 3 indices per triangle. */
typedef struct trb_mesh {
    uint32_t n_verts;
    uint32_t n_tris;
    const float* positions;
    const float* normals;
    const float* texcoords;
    const uint32_t* indices;
} trb_mesh;

/* texture::Image / texture::AnimatedImage (src/texture/image.rs:36-48, animated_image.rs): what scene.rs:317-394 builds for
 * "image", "animated_image" and "movie" textures. A frame is RGBA8 with the semantics of image::DynamicImage::get_pixel
 * (grey -> (l, l, l, 255), RGB -> alpha 255), row-major from the top; one frame = Image, two or more = AnimatedImage whose
 * frames carry their keyframe times in the order given. */
typedef struct trb_image {
    uint32_t width, height;
    const uint8_t* rgba8; /* width * height * 4 bytes */
    float time;
    uint32_t pad;
} trb_image;
typedef struct trb_texture {
    uint32_t first_image, n_images; /* images[first_image .. first_image + n_images) */
} trb_texture;

enum { /* material types (src/material/); every colour / scalar parameter is a constant or a texture (texture/mod.rs) */
    TRB_MAT_MATTE = 0,          /* c0 = diffuse, roughness (degrees; 0 => Lambertian) */
    TRB_MAT_PLASTIC = 1,        /* c0 = diffuse, c1 = gloss, roughness                */
    TRB_MAT_METAL = 2,          /* c0 = refractive_index, c1 = absorption_coefficient, roughness */
    TRB_MAT_SPECULAR_METAL = 3, /* c0 = refractive_index, c1 = absorption_coefficient */
    TRB_MAT_GLASS = 4,          /* c0 = reflect, c1 = transmit, eta                   */
    TRB_MAT_ROUGH_GLASS = 5,    /* c0 = reflect, c1 = transmit, eta, roughness        */
    TRB_MAT_MERL = 6            /* merl = index into merl_tables                       */
};
typedef struct trb_material {
    uint32_t type;
    float c0[3];
    float c1[3];
    float roughness;
    float eta;
    uint32_t merl;
    /* LoadedTextures::find_color / find_scalar (scene.rs:45-87): a parameter given as a texture NAME in the JSON is sampled at the
     * hit's (u, v, time) in Material::bsdf. tex[k] = 1 + index into trb_scene_desc.textures, 0 = the constant above;
     * k: 0 = c0, 1 = c1 (sample_color), 2 = roughness, 3 = eta (sample_f32). */
    uint32_t tex[4];
} trb_material;

#define TRB_MERL_N_THETA_H 90u
#define TRB_MERL_N_THETA_D 90u
#define TRB_MERL_N_PHI_D 180u
#define TRB_MERL_TABLE_FLOATS (90u * 90u * 180u * 3u) /* interleaved RGB f32 as built by material::Merl::load_file (merl.rs:51-84) */

/* film::Camera construction arguments (src/film/camera.rs:64-91). Animated fov
 * (camera.rs:95-125): fov_ctrl/fov_knots non-empty. */
typedef struct trb_camera {
    uint32_t spline_first, n_splines; /* cam_world AnimatedTransform */
    float fov;                        /* degrees */
    float shutter_size;               /* default 0.5 (scene.rs:197-200) */
    uint32_t active_at;
    uint32_t fov_degree, n_fov_ctrl, fov_ctrl_first, n_fov_knots, fov_knot_first; /* into fov_floats */
} trb_camera;

enum { TRB_FILTER_MITCHELL_NETRAVALI = 0, TRB_FILTER_GAUSSIAN = 1 };
typedef struct trb_film {
    uint32_t width, height;  /* multiples of 8 (block_queue.rs:29-31) and of 2 (render_target.rs:43-45) */
    uint32_t samples;        /* spp; rounded up to a power of two (ld.rs:22-26) */
    uint32_t frames, start_frame, end_frame;
    float scene_time;
    uint32_t filter_type;
    float filter_w, filter_h;
    float filter_b, filter_c; /* Mitchell-Netravali b,c; Gaussian: filter_b = alpha */
} trb_film;

enum {
    TRB_INTEGRATOR_PATH = 0,          /* integrator/path.rs:35-43: min_depth, max_depth */
    TRB_INTEGRATOR_WHITTED = 1,       /* integrator/whitted.rs:29-38: max_depth = recursion limit (the JSON loader reads it from
                                         "min_depth", like scene.rs:305-309); min_depth unused */
    TRB_INTEGRATOR_NORMALS_DEBUG = 2  /* integrator/normals_debug.rs:25-36: (shading normal + 1) / 2 */
};
typedef struct trb_integrator {
    uint32_t type;
    uint32_t min_depth, max_depth;
} trb_integrator;

typedef struct trb_scene_desc {
    uint32_t abi_version; /* TRB_ABI_VERSION */
    trb_film film;
    trb_integrator integrator;
    uint32_t n_cameras;   const trb_camera* cameras;     /* sorted by active_at (scene.rs:190) */
    uint32_t n_instances; const trb_instance* instances; /* JSON object order == light order (Q20) */
    uint32_t n_splines;   const trb_spline* splines;
    uint32_t n_keyframes; const trb_keyframe* keyframes;
    uint32_t n_knots;     const float* knots;
    uint32_t n_color_keys; const trb_color_key* color_keys;
    uint32_t n_meshes;    const trb_mesh* meshes;
    uint32_t n_materials; const trb_material* materials;
    uint32_t n_merl;      const float* const* merl_tables; /* each TRB_MERL_TABLE_FLOATS floats */
    uint32_t n_fov_floats; const float* fov_floats;
    uint32_t n_textures;  const trb_texture* textures;
    uint32_t n_images;    const trb_image* images;
} trb_scene_desc;

/* ---------------------------------------------------------------------------------
 * Render configuration = exec::Config (src/exec/mod.rs:17-37) minus paths/threads,
 * plus what the reference leaves to the OS: the RNG seed (multithreaded.rs:79 seeds
 * StdRng from the OS; see DESIGN.md "RNG") and a sample sub-range so a frame can be
 * rendered in additive passes.
 * ------------------------------------------------------------------------------- */
enum {
    TRB_RENDER_STATS = 1u,            /* also count BVH node / triangle / instance tests */
    TRB_RENDER_NO_UPDATE = 2u,        /* skip Scene::update_frame (caller already did it) */
    TRB_RENDER_REFERENCE_SHADOW = 4u, /* trace shadow rays as full closest-hit like light/mod.rs:30-37 instead of
                                         stopping at the first accepted hit (same boolean, fewer tests) */
    TRB_RENDER_MEGAKERNEL = 8u,       /* one persistent kernel per pass instead of the wavefront pipeline (same results) */
    TRB_RENDER_TIME_TRACE = 16u       /* bracket every trace-kernel launch with CUDA events (read with trb_scene_trace_time) */
};
typedef struct trb_render_cfg {
    uint32_t spp;           /* Config.spp; 0 = film.samples. Rounded up to pow2 like ld.rs:22-26 */
    uint32_t sample_first;  /* render sample indices [sample_first, sample_first+sample_count) */
    uint32_t sample_count;  /* of each pixel's spp; 0 = all */
    uint32_t block_start;   /* Config.select_blocks.0 (index into the Morton-sorted 8x8 block list) */
    uint32_t block_count;   /* Config.select_blocks.1; 0 = all blocks (block_queue.rs:39-41) */
    uint32_t current_frame; /* Config.current_frame */
    uint32_t seed;
    uint32_t flags;
    /* Optional interleaved sharding of the selected block list for multi-GPU load balance: keep block j (index in the
     * list after select_blocks) iff (j / shard_chunk) % shard_count == shard_index. shard_count <= 1 disables it. The
     * reference shards by contiguous ranges only (master.rs:91-93); the union and the summed film are the same. */
    uint32_t shard_index, shard_count, shard_chunk;
} trb_render_cfg;

typedef struct trb_stats {
    uint64_t camera_samples;
    uint64_t rays_primary;      /* multithreaded.rs:97        */
    uint64_t rays_shadow;       /* light/mod.rs:30-37         */
    uint64_t rays_mis;          /* integrator/mod.rs:156-157  */
    uint64_t rays_continuation; /* integrator/path.rs:112     */
    uint64_t node_tests;        /* BBox::fast_intersect calls (TLAS + BLAS); TRB_RENDER_STATS only */
    uint64_t tri_tests;         /* intersect_triangle calls;                 TRB_RENDER_STATS only */
    uint64_t inst_tests;        /* Instance::intersect calls;                TRB_RENDER_STATS only */
    float kernel_ms;            /* device time of the render kernels of this call (CUDA events) */
    float update_ms;            /* host time of Scene::update_frame + upload */
} trb_stats;

/* linalg::Ray without depth/time (src/linalg/ray.rs:9-22): 32 bytes. */
typedef struct trb_ray {
    float o[3];
    float d[3];
    float min_t, max_t;
} trb_ray;

/* Result of Scene::intersect (scene.rs:148-150): ray.max_t after traversal, the
 * instance hit (index into instances) and, for meshes, the triangle index.
 * inst == TRB_MISS when nothing was hit. 16 bytes. */
#define TRB_MISS 0xffffffffu
typedef struct trb_hit {
    float t;
    uint32_t inst;
    uint32_t prim;
    uint32_t pad;
} trb_hit;

/* linalg::Ray with its time (src/linalg/ray.rs:9-22) for the ray queries: the segment [min_t, max_t] of o + t*d,
 * traced at `time`. 48 bytes (three 16-byte loads); pad is ignored. */
typedef struct trb_query_ray {
    float o[3];
    float d[3];
    float min_t, max_t;
    float time;
    uint32_t pad[3];
} trb_query_ray;

/* geometry::Intersection (src/geometry/intersection.rs) of one ray query: ray.max_t after the query (the input max_t on a
 * miss), the instance and, for meshes, the triangle hit, the instance's material, and the hit's DifferentialGeometry
 * (differential_geometry.rs) in world space, transformed as Receiver / Emitter::intersect do (receiver.rs:36-41: p as a
 * point, n and ng as normals, dp_du and dp_dv as vectors). On a miss inst == TRB_MISS and every field after it is 0.
 * 96 bytes. */
typedef struct trb_intersection {
    float t;
    uint32_t inst;
    uint32_t prim;      /* triangle index for meshes, else 0 */
    uint32_t material;  /* trb_instance.material of the hit instance */
    float p[3], n[3], ng[3];
    float u, v, time;   /* time: the ray's */
    float dp_du[3], dp_dv[3];
    uint32_t pad[2];
} trb_intersection;

/* A caller's ray for trb_illumination: linalg::Ray (src/linalg/ray.rs) with its time, plus the key of its sample streams.
 * d is used as given (the reference does not normalise a caller's ray); [min_t, max_t] bounds the primary intersection only,
 * child rays start at 0.001 as Ray::child does (path.rs:109-110); time is ray.time of the whole path (keyframed transforms,
 * AnimatedColor emission). Sample j of the ray draws from the camera-sample stream (seed, key, sample + j): key plays the role
 * of the render's pixel index, sample of its sample index. 48 bytes (three 16-byte loads); pad is ignored. */
typedef struct trb_illum_ray {
    float o[3];
    float d[3];
    float min_t, max_t;
    float time;
    uint32_t key;
    uint32_t sample;
    uint32_t pad;
} trb_illum_ray;
enum { TRB_QUERY_CLAMP = 32u }; /* trb_illumination: clamp each sample to [0, 1] before averaging, as thread_work does (multithreaded.rs:99) */

/* Per camera sample record for parity tests: film position and the clamped radiance
 * pushed as ImageSample (multithreaded.rs:98-102). */
typedef struct trb_sample {
    float x, y;
    float r, g, b;
} trb_sample;

/* Flattened BVH node in the reference's order (bvh.rs:248-267): interior: a =
 * second_child, b = axis (0,1,2); leaf: a = geom_offset, b = 0x80000000 | ngeom. */
typedef struct trb_bvh_node {
    float bmin[3];
    float bmax[3];
    uint32_t a;
    uint32_t b;
} trb_bvh_node;
#define TRB_BVH_LEAF 0x80000000u

typedef struct trb_scene trb_scene;

/* -- lifecycle -------------------------------------------------------------------- */

/* ≙ the construction half of Scene::load_file (scene.rs:101-146): builds each mesh's
 * BVH<Triangle> (mesh.rs:44, max_geom 16) and uploads the scene to `device`
 * (cudaSetDevice ordinal). */
trb_status trb_scene_create(const trb_scene_desc* desc, int device, trb_scene** out);

/* ≙ Scene::load_file(file) (scene.rs:101): JSON + OBJ + MERL loading, then
 * trb_scene_create. width/height/spp > 0 override film.width/height/samples (the
 * BASELINE.json configs do this). */
trb_status trb_scene_load_json(const char* path, uint32_t width, uint32_t height, uint32_t spp,
                               int device, trb_scene** out);

void trb_scene_destroy(trb_scene* scene);

/* film dimensions and rounded spp of a scene */
trb_status trb_scene_info(const trb_scene* scene, uint32_t* width, uint32_t* height, uint32_t* spp,
                          uint32_t* n_blocks, uint32_t* n_instances, uint32_t* n_lights);

/* ≙ Scene::update_frame(frame, start, end) (scene.rs:152-176): selects the camera,
 * sets the shutter interval, recomposes instance transforms, rebuilds the
 * BVH<Instance> (max_geom 4) for the shutter interval and uploads it. */
trb_status trb_scene_update_frame(trb_scene* scene, uint32_t frame, float start, float end);

/* Replace the vertex attributes of mesh `mesh` (n_verts of the description, indices and triangle count unchanged). Each of
 * positions (3 floats per vertex), normals (3) and texcoords (2) may be NULL to keep the current array. New positions rebuild
 * the mesh's BVH<Triangle> (max_geom 16), its leaf-ordered triangle records and node records, and, if a frame has been set,
 * re-run trb_scene_update_frame with its last arguments. Afterwards the scene equals one created from the description with
 * these arrays, except that the mesh has no records for the trace.quads experiment (it then returns TRB_UNSUPPORTED).
 * Drains the device before it overwrites anything that kernels read; returns when the update is complete.
 * Statuses: a null scene or a mesh index out of range is TRB_INVALID_ARG; all three arrays NULL is TRB_OK and changes nothing.
 * Positions that trb_scene_create would reject get its status and message (TRB_INVALID_ARG for triangles with infinite
 * coordinates that make the build split a node into an empty child). A failed update leaves the scene as it was, with one
 * exception: a CUDA error (a device fault, not a property of the input) reported once the node records are being written may leave
 * it half updated. */
trb_status trb_scene_update_mesh(trb_scene* scene, uint32_t mesh, const float* positions, const float* normals, const float* texcoords);
/* The same from device buffers on the scene's GPU: the caller's arrays are read on cuda_stream (a cudaStream_t; NULL = default
 * stream), so a producer on that stream needs no host copy. */
trb_status trb_scene_update_mesh_device(trb_scene* scene, uint32_t mesh, const float* d_positions, const float* d_normals,
                                        const float* d_texcoords, void* cuda_stream);

/* Refit mesh `mesh` to new vertex positions: the mesh's BVH<Triangle> keeps the partition its build chose (same nodes, order,
 * second_child, axis, geom_offset, ngeom and ordered_geom) and each node's box becomes the fold of bvh.rs:143 over that node's
 * triangles at the new positions: BBox::new() unioned with Triangle::bounds of each of them (a bound tied between -0.0 and +0.0 may
 * carry either sign; NaN components are dropped as fminf / fmaxf drop them). The triangle and node records are rewritten on the device
 * and, if a frame has been set, trb_scene_update_frame is re-run with its last arguments; renders, counters and queries then follow
 * the reference's traversal over that tree. The mesh then has no records for the trace.quads experiment (it returns TRB_UNSUPPORTED).
 * Arguments, the stream rule and the statuses are trb_scene_update_mesh's; positions NULL is exactly its attribute copy. The refit
 * depends on no value of the positions, so it does not fail on them: positions that a rebuild refuses refit fine. The frame it re-runs
 * keeps trb_scene_update_frame's rule, which refuses infinite or NaN instance bounds among more than four instances; the mesh is then
 * refit and the call returns that status with no frame set. Otherwise a failed call leaves the scene as it was, except for a CUDA
 * error (a device fault), which may leave it half refit. A refit tree is correct however far the mesh has moved, but slower to trace
 * as it deforms: trb_scene_update_mesh rebuilds it. */
trb_status trb_scene_refit_mesh(trb_scene* scene, uint32_t mesh, const float* positions, const float* normals, const float* texcoords);
/* The same from device buffers on the scene's GPU, read on cuda_stream (a cudaStream_t; NULL = default stream); returns when complete. */
trb_status trb_scene_refit_mesh_device(trb_scene* scene, uint32_t mesh, const float* d_positions, const float* d_normals,
                                       const float* d_texcoords, void* cuda_stream);

/* Scene edits: replace entries [first, first + count) of one array of the description. The structure of the scene (counts, index
 * ranges, which instance is a light, which spline is keyframed) stays; only the values change (trb_scene_replace_objects, below,
 * changes the structure). After a successful call the scene
 * equals trb_scene_create on the description with those entries replaced and, if a frame has been set, that scene after
 * trb_scene_update_frame with the last arguments given: TLAS, transforms, renders and their counters, Adaptive per-pixel counts,
 * ray, illumination and shading queries, and the light list; films to rounding (they are added with atomics).
 * Statuses: a null scene, a null array with count > 0, or a range past the end of the array (first + count computed in 64 bits) is
 * TRB_INVALID_ARG; count 0 is TRB_OK and changes nothing, even with a null array. Each call drains the device before it overwrites
 * anything that kernels read, and returns when the edit is complete. A failed call leaves the scene as it was, with one exception: a
 * CUDA error (a device fault, not a property of the input) reported once the writes have begun may leave it half edited. */
/* Replace keyframes[first .. first + count): the TRS control points of instance, group and camera transforms (trb_spline.ctrl_first
 * indexes this array). Splines, knots and every other array keep their structure. If a frame has been set, it is rebuilt. */
trb_status trb_scene_update_keyframes(trb_scene* scene, uint32_t first, uint32_t count, const trb_keyframe* keyframes);
/* The same from a device array on the scene's GPU, read on cuda_stream (a cudaStream_t; NULL = default stream); returns when complete.
 * A pointer that is not 4-byte aligned is TRB_INVALID_ARG. */
trb_status trb_scene_update_keyframes_device(trb_scene* scene, uint32_t first, uint32_t count, const trb_keyframe* d_keyframes,
                                             void* cuda_stream);
/* Replace color_keys[first .. first + count): emission colours and their key times (AnimatedColor). The frame is not rebuilt. */
trb_status trb_scene_update_color_keys(trb_scene* scene, uint32_t first, uint32_t count, const trb_color_key* keys);
/* Replace materials[first .. first + count): type, colours, roughness, eta, MERL table, texture bindings. They are checked as
 * trb_scene_create checks them, with its statuses and messages. The frame is not rebuilt. */
trb_status trb_scene_update_materials(trb_scene* scene, uint32_t first, uint32_t count, const trb_material* materials);

/* The object section of a trb_scene_desc: everything Scene::load_file builds from "camera(s)" and "objects"
 * (scene.rs:185-260, 480-628). Same field meanings, same index conventions as in trb_scene_desc. */
typedef struct trb_scene_objects {
    uint32_t n_cameras;    const trb_camera* cameras;
    uint32_t n_instances;  const trb_instance* instances;
    uint32_t n_splines;    const trb_spline* splines;
    uint32_t n_keyframes;  const trb_keyframe* keyframes;
    uint32_t n_knots;      const float* knots;
    uint32_t n_color_keys; const trb_color_key* color_keys;
    uint32_t n_fov_floats; const float* fov_floats;
} trb_scene_objects;

/* Object replacement: replace the scene's cameras, instances, splines, keyframes, knots, colour keys and fov floats with the seven
 * arrays of `objects`. Every count may differ from the scene's current one, in either direction, so objects, lights and cameras can
 * be added and removed, instances bound to another mesh, material or shape, receivers turned into emitters and static transforms
 * into keyframed ones. trb_instance.mesh and .material index the scene's existing meshes and materials, which stay as they are
 * with their trees, as do the MERL tables, textures, film, integrator and options. After a successful call the scene equals
 * trb_scene_create on the description with the seven arrays replaced and, if a frame has been set, that scene after
 * trb_scene_update_frame with the last arguments given (the camera is selected as on a new scene's first frame), on everything the
 * scene edits above list.
 * The section is checked before anything is written, by the code that checks it in trb_scene_create, with the same statuses and
 * messages; mesh and material indices are checked against the scene's counts. A null scene or null `objects`, or a null array with a
 * non-zero count, is TRB_INVALID_ARG, as is a section none of whose cameras is active at the frame that has been set. The call
 * drains the device before it frees or overwrites anything that kernels read, and returns when the replacement is complete. A
 * failed call leaves the scene as it was, with one exception: a CUDA error (a device fault, not a property of the input) reported
 * once the scene has been switched to the new section, while the frame is rebuilt, may leave it without a frame. */
trb_status trb_scene_replace_objects(trb_scene* scene, const trb_scene_objects* objects);

/* The mesh section of a trb_scene_desc, as trb_scene_replace_meshes takes it: mesh i of the new list is the scene's current mesh
 * keep[i], which keeps its buffers and trees, or, where keep[i] is TRB_MESH_NEW, the arrays of meshes[i] (read only there). */
#define TRB_MESH_NEW 0xffffffffu
typedef struct trb_scene_meshes {
    uint32_t n_meshes;
    const trb_mesh* meshes;   /* meshes[i] is read only where keep[i] == TRB_MESH_NEW */
    const uint32_t* keep;     /* keep[i]: index of the scene's current mesh that becomes mesh i, or TRB_MESH_NEW */
} trb_scene_meshes;

/* Mesh replacement: replace the scene's meshes with the list `meshes` describes, of any length. A kept mesh (keep[i] an index of the
 * current list) may move to another index and is neither uploaded nor built again; a new one is uploaded and its BVH<Triangle>
 * (max_geom 16) built as trb_scene_create builds it; a current mesh that no keep entry names is released. With `objects` the object
 * section is replaced in the same call, as trb_scene_replace_objects replaces it (what renumbered meshes need); with `objects` NULL
 * the instances stay and their mesh indices index the new list. After a successful call the scene equals trb_scene_create on the
 * description with the mesh section (and the object section, if given) replaced and, if a frame has been set, that scene after
 * trb_scene_update_frame with the last arguments given, on everything the scene edits above list.
 * Statuses: a null scene or null `meshes`, a null keep with n_meshes > 0, a null meshes array where some keep[i] is TRB_MESH_NEW, a
 * keep entry past the current list or naming a mesh twice, an instance whose mesh index is past the new list, or a section none of
 * whose cameras is active at the frame that has been set is TRB_INVALID_ARG. New meshes and `objects` are checked by the code that
 * checks them in trb_scene_create, with its statuses and messages. Every new buffer is built before the scene is switched over, so a
 * failed call leaves the scene as it was, with one exception: a CUDA error (a device fault, not a property of the input) reported
 * once the scene has been switched, while node records are re-packed or the frame is rebuilt. Drains the device before it frees or
 * overwrites anything kernels read; returns when the replacement is complete. */
trb_status trb_scene_replace_meshes(trb_scene* scene, const trb_scene_meshes* meshes, const trb_scene_objects* objects);
/* The same with the four arrays of each new mesh in device memory on the scene's GPU, read on cuda_stream (a cudaStream_t; NULL =
 * default stream); `meshes`, its two arrays and `objects` stay host memory. The indices are checked on the device. */
trb_status trb_scene_replace_meshes_device(trb_scene* scene, const trb_scene_meshes* meshes, const trb_scene_objects* objects,
                                           void* cuda_stream);

/* Settings replacement: replace the scene's film (`film`) and / or integrator (`integrator`); NULL keeps the current one. A new film
 * rebuilds the filter table (trb_scene_get_filter_table), the device film and its host staging, the block lists and the Adaptive
 * sampler's state, and sets the rounded spp from film.samples; a new integrator sets the type and depths and raises the context's
 * stack limit for Whitted and NormalsDebug as trb_scene_create does (it is never lowered). After a successful call the scene equals
 * trb_scene_create on the description with the film and integrator replaced and, if a frame has been set, that scene after
 * trb_scene_update_frame with the last arguments given (the camera's pixel transform follows the film size), on everything the scene
 * edits above list. Statuses: a null scene is TRB_INVALID_ARG; the film and integrator are checked by the code that checks them in
 * trb_scene_create, with its statuses and messages. A failed call leaves the scene as it was, with one exception: a CUDA error (a
 * device fault, not a property of the input) reported while the frame is rebuilt. Drains the device before it frees anything kernels
 * read; returns when the replacement is complete. The replicas of a trb_group are edited one by one (trb_group_scene); the group
 * renders refuse replicas of different film sizes with TRB_INVALID_ARG. */
trb_status trb_scene_replace_settings(trb_scene* scene, const trb_film* film, const trb_integrator* integrator);

/* The material section of a trb_scene_desc, as trb_scene_replace_materials takes it. Same field meanings, same index conventions. */
typedef struct trb_scene_materials {
    uint32_t n_materials; const trb_material* materials;
    uint32_t n_merl;      const float* const* merl_tables; /* each TRB_MERL_TABLE_FLOATS floats */
    uint32_t n_textures;  const trb_texture* textures;
    uint32_t n_images;    const trb_image* images;
} trb_scene_materials;

/* Material replacement: replace the scene's materials, MERL tables, textures and images with the section `materials`, of any counts.
 * With `objects` the object section is replaced in the same call, as trb_scene_replace_objects replaces it (what renumbered materials
 * need); with `objects` NULL the instances stay and their material indices index the new list. The shading kernels (fused or split)
 * and the texture coordinates follow the new section as on a new scene. After a successful call the scene equals trb_scene_create on
 * the description with the material section (and the object section, if given) replaced and, if a frame has been set, that scene
 * after trb_scene_update_frame with the last arguments given, on everything the scene edits above list.
 * Statuses: a null scene or null `materials`, a null array with a non-zero count, a null MERL table, an instance whose material index
 * is past the new list, or a section none of whose cameras is active at the frame that has been set is TRB_INVALID_ARG. The section
 * and `objects` are checked by the code that checks them in trb_scene_create, with its statuses and messages. Every new buffer is
 * built before the scene is switched over, so a failed call leaves the scene as it was, with one exception: a CUDA error (a device
 * fault, not a property of the input) reported while the frame is rebuilt. Drains the device before it frees anything kernels read;
 * returns when the replacement is complete. */
trb_status trb_scene_replace_materials(trb_scene* scene, const trb_scene_materials* materials, const trb_scene_objects* objects);
/* The same with the MERL tables and each image's rgba8 in device memory on the scene's GPU, read on cuda_stream (a cudaStream_t;
 * NULL = default stream) with device-to-device copies; `materials`, its arrays of structs and `objects` stay host memory. */
trb_status trb_scene_replace_materials_device(trb_scene* scene, const trb_scene_materials* materials, const trb_scene_objects* objects,
                                              void* cuda_stream);

/* -- the hot path ------------------------------------------------------------------ */

/* ≙ Exec::render (exec/mod.rs:48; multithreaded.rs:55-70). Renders the selected
 * blocks at the selected samples — with sample_count = 0 the WHOLE spp of the frame,
 * like MultiThreaded::render — on the scene's GPU and ADDS the RGBW film (row-major,
 * width*height*4 floats, layout of get_renderf32 render_target.rs:243-265) into the
 * HOST buffer `film_rgbw` — additive like film::Image::add_pixels (film/image.rs:21-33).
 * Internally the frame is rendered in additive passes sized to the free device memory
 * (212 B of path state per camera sample in flight); the film is accumulated on the
 * device and copied to the host once. Includes update_frame unless
 * TRB_RENDER_NO_UPDATE. Blocking. */
trb_status trb_render(trb_scene* scene, const trb_render_cfg* cfg, float* film_rgbw, trb_stats* stats);

/* Same, but the film is a DEVICE buffer on the scene's GPU (accumulated into), and the
 * work is enqueued on `cuda_stream` (a cudaStream_t; NULL = default stream) without
 * host synchronisation. Never calls update_frame. `stats` (may be NULL) is a DEVICE
 * pointer to a trb_stats the kernels accumulate ray counters into.
 * Synchronisation contract: passes of one scene must be enqueued on ONE stream at a time
 * (they share the scene's path-state buffers); trb_scene_update_frame drains the device
 * before it touches the instance / TLAS buffers; a traversal-stack overflow (the reference
 * panics) is latched on the device and reported by trb_scene_check_error or by the next
 * host-buffer call (trb_render / trb_intersect / trb_render_samples). */
trb_status trb_render_device(trb_scene* scene, const trb_render_cfg* cfg, float* d_film_rgbw,
                             trb_stats* d_stats, void* cuda_stream);

/* -- multi-GPU: tile sharding + ONE film SUM-reduce per frame (SURVEY 8e) -------------
 *
 * The reference's distributed mode gives worker r of W the blocks [r*floor(B/W), ...) of the Morton block list
 * (exec/distrib/master.rs:88-93,218-224), every worker renders its blocks at full spp with the scene replicated
 * (worker.rs:37-89), and the master adds the workers' films (film/image.rs:21-50, master.rs:124-163). Here the
 * exchange is one ncclReduce(SUM, fp32) of the RGBW film over NVLink at frame end. libnccl.so.2 is resolved at run
 * time (the copy already loaded in the process, else the system one): a single-GPU user never needs it.
 *
 * Two shapes:
 *   one process per GPU  trb_nccl_unique_id (rank 0; ship the 128 bytes to the other ranks by any means)
 *                        -> trb_comm_create on every rank -> trb_render_sharded per frame
 *   one process, n GPUs  trb_group_create / trb_group_load_json -> trb_group_render per frame
 */
#define TRB_NCCL_UNIQUE_ID_BYTES 128
typedef struct trb_comm trb_comm;
typedef struct trb_group trb_group;

trb_status trb_nccl_unique_id(void* id128);
/* ncclCommInitRank on `device`: collective over the n_ranks processes. */
trb_status trb_comm_create(const void* id128, int n_ranks, int rank, int device, trb_comm** out);
void trb_comm_destroy(trb_comm* comm);
trb_status trb_comm_info(const trb_comm* comm, int* n_ranks, int* rank);
/* SUM-reduce `n_floats` of a DEVICE film into rank `root`'s buffer (in place), enqueued on cuda_stream. */
trb_status trb_comm_reduce_film(trb_comm* comm, float* d_film_rgbw, size_t n_floats, int root, void* cuda_stream);

/* ≙ Exec::render of one rank of the distributed mode + the master's film sum: renders this rank's share of the
 * selected blocks (interleaved chunks of cfg->shard_chunk blocks, default 32, rank = shard index; cfg->shard_count
 * == 0xffffffff selects the reference's contiguous ranges instead), all samples, film kept on the device, then ONE
 * reduce to `root`; on the root the summed film is ADDED into the host buffer `film_rgbw` (ignored elsewhere, may
 * be NULL). `stats` receives this rank's counters. Blocking. */
trb_status trb_render_sharded(trb_scene* scene, trb_comm* comm, const trb_render_cfg* cfg, int root, float* film_rgbw,
                              trb_stats* stats);

/* One process driving n GPUs: a scene replica per device (trb_scene_create on each) plus communicators from
 * ncclCommInitAll. trb_group_render ≙ Exec::render on all of them: tile-sharded, one reduce to devices[0], film
 * ADDED into the host buffer; `stats` is the sum over the devices. */
trb_status trb_group_create(const trb_scene_desc* desc, const int* devices, int n_devices, trb_group** out);
trb_status trb_group_load_json(const char* path, uint32_t width, uint32_t height, uint32_t spp, const int* devices,
                               int n_devices, trb_group** out);
trb_status trb_group_render(trb_group* group, const trb_render_cfg* cfg, float* film_rgbw, trb_stats* stats);
trb_scene* trb_group_scene(trb_group* group, int index); /* borrowed: replica `index` (film_to_srgb8, info, options) */
void trb_group_destroy(trb_group* group);

/* ≙ Scene::intersect (scene.rs:148-150) for a batch of rays: closest hit through the
 * two-level BVH in the reference's traversal order. Host buffers. */
trb_status trb_intersect(trb_scene* scene, size_t n, const trb_ray* rays, trb_hit* hits, trb_stats* stats);

/* Device-buffer variant of trb_intersect, enqueued on cuda_stream. */
trb_status trb_intersect_device(trb_scene* scene, size_t n, const trb_ray* d_rays, trb_hit* d_hits,
                                trb_stats* d_stats, void* cuda_stream);

/* -- ray queries on the render's trace kernel ------------------------------------------
 * ≙ Scene::intersect (scene.rs:148-150) for a batch of rays, each traced at its own `time` with the reference's inclusive
 * [min_t, max_t] tests, returning the whole geometry::Intersection. The rays run through the wavefront trace kernel the
 * renders use, in passes of at most "pass.paths" rays (trb_scene_set_option). The TLAS is the one trb_scene_update_frame built
 * for the current shutter interval: a time outside that interval is traced against those boxes, exactly as the reference
 * would trace it. flags: TRB_RENDER_STATS also counts node / triangle / instance tests; stats->rays_primary counts the
 * queries. TRB_INVALID_ARG for null arguments, other flag bits, or before the first update_frame ("Update frame must be
 * called before rendering"); n == 0 is TRB_OK. A traversal-stack overflow returns TRB_CUDA. Host buffers; blocking. */
trb_status trb_intersect_records(trb_scene* scene, size_t n, const trb_query_ray* rays, trb_intersection* out, uint32_t flags,
                                 trb_stats* stats);

/* Device-buffer variant of trb_intersect_records, enqueued on cuda_stream (a cudaStream_t; NULL = default stream) without host
 * synchronisation. d_rays and d_out must be 16-byte aligned; d_stats (may be NULL) is a DEVICE trb_stats the kernels accumulate
 * into. A call that needs more path state than earlier calls grows it and synchronises the device once, as trb_render_device
 * does; the same one-stream-per-scene rule applies, and a traversal-stack overflow is reported by trb_scene_check_error. */
trb_status trb_intersect_records_device(trb_scene* scene, size_t n, const trb_query_ray* d_rays, trb_intersection* d_out, uint32_t flags,
                                        trb_stats* d_stats, void* cuda_stream);

/* ≙ OcclusionTester::occluded (light/mod.rs:30-37) for a batch: occluded[i] = 1 iff Scene::intersect finds a hit on ray i's
 * segment at its time, else 0. Callers build the segment as OcclusionTester::test_points / test_ray do (light/mod.rs:21-28).
 * By default a ray stops at its first accepted hit (same booleans, fewer tests); TRB_RENDER_REFERENCE_SHADOW walks to the
 * closest hit like the reference, so the test counters of TRB_RENDER_STATS equal its. stats->rays_shadow counts the queries.
 * Statuses, passes and TLAS as trb_intersect_records. Host buffers; blocking. */
trb_status trb_occluded(trb_scene* scene, size_t n, const trb_query_ray* rays, uint8_t* occluded, uint32_t flags, trb_stats* stats);

/* Device-buffer variant of trb_occluded, with trb_intersect_records_device's contract (d_rays 16-byte aligned). */
trb_status trb_occluded_device(trb_scene* scene, size_t n, const trb_query_ray* d_rays, uint8_t* d_occluded, uint32_t flags,
                               trb_stats* d_stats, void* cuda_stream);

/* ≙ the per-sample body of thread_work (multithreaded.rs:95-103) along caller rays: sample j (0 <= j < spp) of ray i runs
 * Scene::intersect and, on a hit, the scene integrator's Integrator::illumination (Path, Whitted or NormalsDebug); a miss is
 * black. Its per-path sample arrays, Russian roulette and Whitted node streams come from the camera-sample stream
 * (seed, rays[i].key, rays[i].sample + j mod 2^32) with LD offset 0, so a trb_camera_rays ray submitted with key = its pixel,
 * sample = its sample index, spp = 1 and TRB_QUERY_CLAMP returns trb_render_samples' r, g, b bits.
 * rgb[3i + c] = (sum of the spp samples' radiance, added in sample order) / spp in float32; each sample is clamped to [0, 1]
 * first only with TRB_QUERY_CLAMP. flags: TRB_RENDER_STATS, TRB_RENDER_REFERENCE_SHADOW, TRB_QUERY_CLAMP; anything else is
 * TRB_INVALID_ARG. stats: camera_samples = rays_primary = n * spp, shadow / MIS / continuation rays as a render counts them.
 * The paths run on the render's wavefront kernels in passes of at most "pass.paths" samples holding whole rays. TRB_INVALID_ARG
 * for null arguments, spp == 0 or > 65536, or before the first update_frame; n == 0 is TRB_OK. TLAS as trb_intersect_records.
 * Host buffers; blocking. */
trb_status trb_illumination(trb_scene* scene, size_t n, const trb_illum_ray* rays, uint32_t spp, uint32_t seed, float* rgb, uint32_t flags,
                            trb_stats* stats);

/* Device-buffer variant of trb_illumination, with trb_intersect_records_device's contract: d_rays 16-byte aligned, d_rgb 4-byte
 * aligned, d_stats NULL or a DEVICE trb_stats, enqueued on cuda_stream without host synchronisation. */
trb_status trb_illumination_device(trb_scene* scene, size_t n, const trb_illum_ray* d_rays, uint32_t spp, uint32_t seed, float* d_rgb,
                                   uint32_t flags, trb_stats* d_stats, void* cuda_stream);

/* -- shading queries: the render's BSDF and light functions on caller inputs ---------------------------------------------
 * Material::bsdf with BSDF::eval / pdf / sample, Light::sample_incident / pdf and Emitter::radiance (bsdf.rs:66-125, light/mod.rs:43-53,
 * emitter.rs:140-204) for batches of queries, on the device code the renders run, so they return the render's bits. They trace
 * nothing: a caller composes them with trb_intersect_records and trb_occluded into an integrator of its own.
 *
 * A BSDF query i builds Material::bsdf at record rec[i] (a trb_intersection as trb_intersect_records returns it, or filled in by the
 * caller): material rec.material, textures sampled at (rec.u, rec.v, rec.time), shading frame from rec.n and rec.dp_du (bsdf.rs:38-44);
 * no other field is read. `bxdf` is the EnumSet<BxDFType> of the call (bxdf/mod.rs:37-41), TRB_BXDF_ALL for every lobe.
 * A light query names its light by instance index (trb_scene_lights lists them in light order); its transform and emission are
 * evaluated at the query's time.
 *
 * Out-of-range inputs are not errors: the query writes an all-zero output and reads nothing out of bounds. That is a record with
 * inst == TRB_MISS or material >= the scene's material count, a light or inst >= the instance count, and a light that is not an
 * emitter.
 * Statuses: TRB_INVALID_ARG for null arguments with n > 0 and for unaligned device buffers; n == 0 is TRB_OK. The light queries read the
 * instance matrices of trb_scene_update_frame and return TRB_INVALID_ARG before the first one; the BSDF queries and trb_emitted work
 * right after scene creation. The host forms take host buffers and block. The _device forms take device buffers on the scene's GPU
 * (queries, records and 16-byte outputs 16-byte aligned, float outputs 4-byte aligned) and enqueue one kernel on cuda_stream (a
 * cudaStream_t; NULL = default stream) without host synchronisation, under trb_render_device's one-stream-per-scene rule. */
enum { /* bxdf::BxDFType (bxdf/mod.rs:37-41) */
    TRB_BXDF_REFLECTION = 1u,
    TRB_BXDF_TRANSMISSION = 2u,
    TRB_BXDF_DIFFUSE = 4u,
    TRB_BXDF_GLOSSY = 8u,
    TRB_BXDF_SPECULAR = 16u,
    TRB_BXDF_ALL = 31u
};

/* BSDF::eval / pdf arguments: w_o, the lobe set, w_i (world space, used as given). 32 bytes; pad is ignored. */
typedef struct trb_bsdf_eval_query {
    float wo[3];
    uint32_t bxdf;
    float wi[3];
    uint32_t pad;
} trb_bsdf_eval_query;

/* BSDF::sample arguments: w_o, the lobe set and Sample { two_d: u, one_d: u_comp } (u_comp chooses the lobe). 32 bytes. */
typedef struct trb_bsdf_sample_query {
    float wo[3];
    uint32_t bxdf;
    float u[2];
    float u_comp;
    uint32_t pad;
} trb_bsdf_sample_query;

/* BSDF::sample's (f, w_i, pdf, sampled type) (bsdf.rs:85-111); sampled = the chosen lobe's type bits, 0 when nothing was sampled.
 * 32 bytes. */
typedef struct trb_bsdf_sample_result {
    float f[3];
    float pdf;
    float wi[3];
    uint32_t sampled;
} trb_bsdf_sample_result;

/* Light::sample_incident arguments: the receiving point, the time, the 2-D sample and the light's instance index. 32 bytes. */
typedef struct trb_light_query {
    float p[3];
    float time;
    float u[2];
    uint32_t light;
    uint32_t pad;
} trb_light_query;

/* Light::sample_incident's (Li, w_i, pdf, OcclusionTester) (emitter.rs:164-190) and delta_light() (1 for point lights). shadow is the
 * OcclusionTester as a ray: test_points(p, p_light, time) = Ray::segment(p, p_light - p, 0.001, 0.999, time) (light/mod.rs:21-23), ready
 * for trb_occluded. 80 bytes. */
typedef struct trb_light_sample_result {
    float li[3];
    float pdf;
    float wi[3];
    uint32_t delta;
    trb_query_ray shadow;
} trb_light_sample_result;

/* Light::pdf arguments: p, time, w_i, the light's instance index. 32 bytes. */
typedef struct trb_light_pdf_query {
    float p[3];
    float time;
    float wi[3];
    uint32_t light;
} trb_light_pdf_query;

/* Emitter::radiance arguments: the outgoing direction w, time, the surface normal n, the instance index. 32 bytes. */
typedef struct trb_emit_query {
    float w[3];
    float time;
    float n[3];
    uint32_t inst;
} trb_emit_query;

/* out4[4i .. 4i+3] = BSDF::eval(wo, wi, bxdf) r, g, b, then BSDF::pdf(wo, wi, bxdf), of Material::bsdf at rec[i]. */
trb_status trb_bsdf_eval(trb_scene* scene, size_t n, const trb_intersection* rec, const trb_bsdf_eval_query* q, float* out4);
trb_status trb_bsdf_eval_device(trb_scene* scene, size_t n, const trb_intersection* d_rec, const trb_bsdf_eval_query* d_q, float* d_out4,
                                void* cuda_stream);

/* out[i] = BSDF::sample(wo, bxdf, (u, u_comp)) of Material::bsdf at rec[i]. */
trb_status trb_bsdf_sample(trb_scene* scene, size_t n, const trb_intersection* rec, const trb_bsdf_sample_query* q, trb_bsdf_sample_result* out);
trb_status trb_bsdf_sample_device(trb_scene* scene, size_t n, const trb_intersection* d_rec, const trb_bsdf_sample_query* d_q,
                                  trb_bsdf_sample_result* d_out, void* cuda_stream);

/* out[i] = Light::sample_incident(p, u, time) of instance q[i].light. */
trb_status trb_light_sample(trb_scene* scene, size_t n, const trb_light_query* q, trb_light_sample_result* out);
trb_status trb_light_sample_device(trb_scene* scene, size_t n, const trb_light_query* d_q, trb_light_sample_result* d_out, void* cuda_stream);

/* pdf[i] = Light::pdf(p, wi, time) of instance q[i].light (emitter.rs:193-203): 0 for point lights and for directions that miss the
 * light's shape. */
trb_status trb_light_pdf(trb_scene* scene, size_t n, const trb_light_pdf_query* q, float* pdf);
trb_status trb_light_pdf_device(trb_scene* scene, size_t n, const trb_light_pdf_query* d_q, float* d_pdf, void* cuda_stream);

/* rgb[3i .. 3i+2] = Emitter::radiance(w, _, n, time) of instance q[i].inst (its emission when dot(w, n) > 0, else black); black when the
 * instance is a receiver. This is the emitted term of Path::illumination (path.rs:71-74) and of the MIS ray (integrator/mod.rs:156-162);
 * the caller chooses the normal. */
trb_status trb_emitted(trb_scene* scene, size_t n, const trb_emit_query* q, float* rgb);
trb_status trb_emitted_device(trb_scene* scene, size_t n, const trb_emit_query* d_q, float* d_rgb, void* cuda_stream);

/* The light list of sample_one_light (integrator/mod.rs:106-111): the instance indices of the emitters in object order (Q20),
 * n_lights of them (trb_scene_info). Host buffer; no device work. */
trb_status trb_scene_lights(const trb_scene* scene, uint32_t* inst);

/* ≙ LowDiscrepancy::get_samples + get_samples_1d + Camera::generate_ray
 * (ld.rs:33-64, camera.rs:150-157) for the selected blocks/samples: writes one ray and
 * one film position per camera sample, in block-list order, pixel row-major within the
 * block, sample index minor. Host buffers sized n = blocks*64*sample_count. */
trb_status trb_camera_rays(trb_scene* scene, const trb_render_cfg* cfg, size_t n, trb_ray* rays, float* xy);

/* Parity/debug variant of trb_render: instead of splatting, writes the clamped
 * radiance of every camera sample (same order as trb_camera_rays). Host buffer. */
trb_status trb_render_samples(trb_scene* scene, const trb_render_cfg* cfg, size_t n, trb_sample* samples,
                              trb_stats* stats);

/* -- AOVs: denoiser guide images and per-pixel depth / object id from the render's own primary hits (DESIGN.md §4 "AOVs") --------
 * For every camera sample of a render, one record from the sample's primary hit (the trb_camera_rays ray, traced by Scene::intersect):
 *   depth   the hit's t, as trb_intersect_records gives it for that ray; +inf on a miss
 *   inst    the instance hit, or TRB_MISS
 *   n       the unit world-space shading normal of the BSDF frame (bsdf.rs:38-44, what NormalsDebug shows as (n + 1) / 2); not flipped
 *           toward the camera; 0 on a miss
 *   albedo  Material::bsdf's lobes at the hit, textured: the sum, in lobe order, of each lobe's colour times its Fresnel factor at
 *           normal incidence (diffuse lobes 1, reflection F(1), transmission 1 - F(1)); MERL: pi * BSDF::eval(n, n, all lobes). Each
 *           channel clamped to [0, 1]. Emission is not part of it. 0 on a miss.
 * 32 bytes. */
typedef struct trb_aov_sample {
    float albedo[3];
    float depth;
    float n[3];
    uint32_t inst;
} trb_aov_sample;

/* AOV outputs of a film render; any may be NULL (not rendered).
 *   albedo_w, normal_w  RGBW films (width*height*4 floats, the colour film's layout). Each sample adds w * value and w with the colour
 *                       film's weights (RenderTarget::write: filter table, filter_pixel_width window, 2x2 lock blocks); a miss adds w
 *                       with a zero value, so their W equals the colour film's W up to float addition order. Added into.
 *   nearest             width*height uint64: each sample does atomicMin(pixel, float_bits(depth) << 32 | inst) on the pixel it was
 *                       taken for. Initialise it to all ones; a pixel whose samples all missed holds 0x7f800000ffffffff. The result
 *                       does not depend on the order of samples, passes or calls. */
typedef struct trb_aov_film {
    float* albedo_w;
    float* normal_w;
    uint64_t* nearest;
} trb_aov_film;

/* trb_render that also renders the AOVs into the HOST buffers of `aov` (same sizes as above; nearest is read and written). The colour
 * film, samples and every trb_stats counter equal trb_render's with the same cfg. Path integrator on the wavefront only: Whitted,
 * NormalsDebug and TRB_RENDER_MEGAKERNEL give TRB_UNSUPPORTED. The first AOV render allocates 32 B of AOV record per path in flight
 * (TRB_OOM if that does not fit); plain renders never do. Blocking. */
trb_status trb_render_aov(trb_scene* scene, const trb_render_cfg* cfg, float* film_rgbw, const trb_aov_film* aov, trb_stats* stats);

/* trb_render_aov with the contract of trb_render_device: the film and the outputs of `d_aov` (a host struct of DEVICE pointers) are
 * device buffers on the scene's GPU, enqueued on cuda_stream without host synchronisation. TRB_INVALID_ARG for a film or an AOV
 * film that is not 16-byte aligned, or a nearest buffer that is not 8-byte aligned. */
trb_status trb_render_aov_device(trb_scene* scene, const trb_render_cfg* cfg, float* d_film_rgbw, const trb_aov_film* d_aov,
                                 trb_stats* d_stats, void* cuda_stream);

/* trb_render_samples that also writes each camera sample's AOV record into the HOST buffer aov[n], in the same order. samples[] and
 * the stats equal trb_render_samples'. The statuses of trb_render_samples and trb_render_aov. */
trb_status trb_render_samples_aov(trb_scene* scene, const trb_render_cfg* cfg, size_t n, trb_sample* samples, trb_aov_sample* aov,
                                  trb_stats* stats);

/* -- Denoising: an edge-avoiding a-trous filter over two half renders and their AOVs (DESIGN.md §4 "Denoising") -----------------
 * SVGF's spatial filter (Schied et al. 2017, §4.4-4.5; Dammertz et al. 2010) with the variance taken from two half-buffers and the
 * colour demodulated by the albedo. Render samples [0, n) of a frame into colour_a and [n, 2n) into colour_b (trb_render_cfg's
 * sample_first / sample_count), with albedo_w, normal_w and nearest accumulated over both (trb_render_aov). All five are the scene's
 * film layout: width*height RGBW float films, width*height uint64 nearest. Per pixel p, float32, left to right, never contracted:
 *   W     = A.w + B.w. W <= 0: the output is (0, 0, 0, 0) and p is never a neighbour (blocks a block-range render did not render).
 *   c     = (A.rgb + B.rgb) / W,  c_a = A.rgb / A.w,  c_b = B.rgb / B.w
 *   d     = max(albedo_w.rgb / albedo_w.w, TRB_DENOISE_EPS_ALBEDO) per channel;  e = c / d,  e_a = c_a / d,  e_b = c_b / d
 *   v     = (L(e_a) - L(e_b))^2 * 0.25,  L(x) = 0.2126 x.r + 0.7152 x.g + 0.0722 x.b
 *   m     = normal_w.rgb / normal_w.w, len2 = m.x^2 + m.y^2 + m.z^2; n = m / sqrt(len2) per component, or "no normal" if len2 == 0
 *   z     = the float in nearest's high 32 bits (+inf: a miss)
 *   Unless c, albedo, m, len2, e and v are all finite and z is neither NaN nor -inf, p is copied through: (c, 1), never a neighbour.
 *   dz    = (gx, gy), per axis the central difference (z[+1] - z[-1]) * 0.5 when both neighbours are inside the image with finite z,
 *           else z[+1] - z or z - z[-1] for the one that is, else 0; 0 when z is infinite
 * Iteration i = 0 .. N-1, step s = 2^i, over the valid pixels, from (e, v):
 *   g     = sum k(dx) k(dy) v(q) / sum k(dx) k(dy) over the 3x3 q = p + (dx, dy) inside the image and valid, k = (1/4, 1/2, 1/4)
 *   for the 25 taps q = p + s (dx, dy), dy then dx from -2 to 2, inside the image and valid, h = (1/16, 1/4, 3/8, 1/4, 1/16):
 *     w_l = exp(-(|L(e(p)) - L(e(q))| / (sigma_luminance * sqrt(g) + TRB_DENOISE_EPS_LUMINANCE)))
 *     w_n = max(0, n_p . n_q) squared log2(normal_power) times; 1 when neither has a normal, 0 when one has
 *     w_z = exp(-(|z_p - z_q| / (sigma_depth * |gx * s dx + gy * s dy| + TRB_DENOISE_EPS_DEPTH))); 1 when both z are infinite,
 *           0 when one is
 *     w   = h(dx) h(dy) * w_l * w_n * w_z
 *   e'(p) = sum w e(q) / sum w,  v'(p) = sum w^2 v(q) / (sum w)^2
 * The output of a valid pixel is (e_N * d, 1): an RGBW film that trb_film_to_srgb8 and trb_host_film_to_srgb8 take as it is. Every NaN
 * the output holds is written as 0x7fffffff, whatever NaN the inputs carried. exp is
 * the library's deterministic exp; sums run in tap order without atomics, so the output is bit-reproducible. */
#define TRB_DENOISE_EPS_ALBEDO 1e-3f
#define TRB_DENOISE_EPS_LUMINANCE 1e-6f
#define TRB_DENOISE_EPS_DEPTH 1e-2f

/* The five inputs, all required: host pointers for trb_denoise, device pointers for trb_denoise_device. */
typedef struct trb_denoise_input {
    const float* colour_a;
    const float* colour_b;
    const float* albedo_w;
    const float* normal_w;
    const uint64_t* nearest;
} trb_denoise_input;

/* NULL means the defaults: 5 iterations (0-10; 0 = demodulate and remodulate only), normal_power 128 (a power of two, 1-1024),
 * sigma_luminance 4 and sigma_depth 1 (finite, > 0). Anything else is TRB_INVALID_ARG. */
typedef struct trb_denoise_params {
    uint32_t iterations;
    uint32_t normal_power;
    float sigma_luminance;
    float sigma_depth;
} trb_denoise_params;

/* Denoise HOST films into the HOST RGBW film out_rgbw (width*height*4 floats, overwritten). The inputs are staged per call; blocking.
 * The scene keeps 72 bytes of scratch per pixel, allocated by its first denoise (TRB_OOM if that does not fit) and released when
 * trb_scene_replace_settings changes the film; renders never allocate it. TRB_INVALID_ARG for a null argument, bad parameters or an
 * output that overlaps an input. */
trb_status trb_denoise(trb_scene* scene, const trb_denoise_input* in, const trb_denoise_params* params, float* out_rgbw);

/* trb_denoise with DEVICE buffers on the scene's GPU (films and output 16-byte aligned, nearest 8-byte aligned; TRB_INVALID_ARG
 * otherwise), enqueued on cuda_stream (a cudaStream_t; NULL = default stream) under trb_render_device's one-stream rule. No host
 * synchronisation, except once when the scratch grows. */
trb_status trb_denoise_device(trb_scene* scene, const trb_denoise_input* d_in, const trb_denoise_params* params, float* d_out_rgbw,
                              void* cuda_stream);

/* -- Temporal denoising: reproject each pixel's history through the scene's motion and accumulate the half-buffers over frames -----
 * (DESIGN.md §4 "Temporal denoising"). SVGF's temporal half (Schied et al. 2017, §4.1-4.2) over trb_denoise's inputs, with the
 * variance still taken from the two halves: two half histories blended with the same weights are two independent estimates of one
 * mean, so (L(ē_a) - L(ē_b))^2 / 4 stays the variance of their mean, and it shrinks as the history grows.
 *
 * A trb_denoise_history belongs to one scene (another scene is TRB_INVALID_ARG). It is empty after create and after reset, and it
 * takes the film size of the first call that uses it: a later call with another film size (trb_scene_replace_settings) is
 * TRB_INVALID_ARG until it is reset. Per pixel it holds H_a, H_b (the demodulated accumulated halves), the unit normal n, the depth
 * z, the instance inst and len (frames accumulated), or "none"; two such sets, each call reading one and writing the other. It also
 * holds a snapshot of the frame it was written at: the inverse of the camera's cam_world at shutter-open, tan(fov / 2), the film size,
 * every instance's world transform at shutter-open (object -> world), the instance count, and the scene's object generation, a counter
 * that trb_scene_replace_objects and trb_scene_replace_meshes with an object section (the calls that renumber instances) increment.
 * A history of another generation is treated as empty.
 *
 * The inputs are trb_denoise's, rendered at the scene's current frame (the last update_frame; a render with current_frame sets it).
 * Per pixel p = (x, y), float32, left to right, never contracted: validity, e, e_a, e_b, v, d, n, z and dz are trb_denoise's. A pixel
 * trb_denoise does not filter is written as trb_denoise writes it, stores "none", has motion (NaN, NaN) and history_length 0.
 * Otherwise, with i = the low 32 bits of nearest:
 *   1. o, dir = camera_ray's arithmetic through (x + 0.5, y + 0.5) with the current frame's cam_world at shutter-open (not a keyframed
 *      camera's per-ray transform): pc = px_to_cam . (x + 0.5, y + 0.5, 0), dir = cam_world (vector) . unit(tan * pc.x, tan * pc.y,
 *      1 * pc.z), o = cam_world (point) . 0; p_w = o + z * dir per component.
 *   2. Motion, when the history is not empty, its generation is the scene's, i is below the snapshot's and the scene's instance count
 *      and z is finite: p_o = inv_cur[i] . p_w, p' = mat_prev[i] . p_o, q = cam_inv_prev . p' (points, applied as the trace kernels
 *      apply an instance's inverse: divided by w when |w - 1| < FLT_EPSILON). If q.z > 0:
 *        X = q.x / (q.z * tan_prev), Y = q.y / (q.z * tan_prev)
 *        r = ((X - X0) / (X1 - X0) * w_prev, (Y - Y1) / (Y0 - Y1) * h_prev), with a = (float)w_prev / (float)h_prev and
 *            (X0, X1, Y0, Y1) = a > 1 ? (-a, a, -1, 1) : (-1, 1, -1 / a, 1 / a): the inverse of camera_ray's raster -> camera
 *            mapping up to rounding, since camera space directions are (tan X, tan Y, 1) up to scale
 *        motion = r - (x + 0.5, y + 0.5); |q| = sqrt(q.x^2 + q.y^2 + q.z^2) is the depth the previous frame's ray would record.
 *      Otherwise motion is (NaN, NaN) and there is no history.
 *   3. c = r - 0.5, f = (floor(c.x), floor(c.y)), a = c - f. Taps t = f + (0,0), (1,0), (0,1), (1,1) in that order, with weights
 *      (1 - a.x) * (1 - a.y), a.x * (1 - a.y), (1 - a.x) * a.y, a.x * a.y. A tap counts when it is inside the image (tested on the
 *      float coordinates), is not "none", has inst == i, |z_t - |q|| <= depth_tolerance * |q|, and n_t . n >= normal_threshold when
 *      both have a normal (passing when neither has one, failing when one has). S = the sum of the counted weights in tap order; if
 *      S > 0, H_a' = (sum of w * H_a in tap order) / S per channel, H_b' likewise, len_prev = the largest len of a counted tap with
 *      w > 0. S <= 0: no history.
 *   4. n' = min(len_prev + 1, max_history), or 1 without history. n' == 1: ē_a = e_a, ē_b = e_b, and e, v are trb_denoise's (so the
 *      output is trb_denoise's, bit for bit). Otherwise alpha = 1 / (float)n', per channel
 *        ē_a = alpha * e_a + (1 - alpha) * H_a',  ē_b likewise,  ē = alpha * e + (1 - alpha) * ((H_a' + H_b') * 0.5)
 *        v = (L(ē_a) - L(ē_b))^2 * 0.25
 *   5. (ē, v) replaces (e, v) in trb_denoise's a-trous iterations; the output is remodulated by d as there.
 *   6. A filtered pixel with finite z stores (ē_a, ē_b, n, z, i, n'); every other pixel stores "none". The snapshot becomes the
 *      current frame's.
 * Every NaN written to rgbw or motion is 0x7fffffff. Motion covers rigid instance transforms and the camera, not the deformation of
 * trb_scene_update_mesh / trb_scene_refit_mesh: the depth and normal tests reject what moved too far, and what they accept may ghost.
 * Misses have no history. A history last written by trb_denoise_moments* holds moments, not halves: these calls treat it as empty
 * (as for another object generation), so the first one after it filters as trb_denoise does. */
typedef struct trb_denoise_history trb_denoise_history;

/* NULL means: trb_denoise's defaults for `spatial`, max_history 8 (1-255), depth_tolerance 0.05 (finite, > 0), normal_threshold 0.9
 * (in [-1, 1]). `spatial` takes trb_denoise's ranges. Anything out of range is TRB_INVALID_ARG. These defaults have not been tuned. */
typedef struct trb_denoise_temporal_params {
    trb_denoise_params spatial;
    uint32_t max_history;
    float depth_tolerance;
    float normal_threshold;
    uint32_t pad; /* ignored */
} trb_denoise_temporal_params;

/* rgbw (width*height*4 floats) is required; motion (width*height*2 floats) and history_length (width*height uint32) may be NULL. */
typedef struct trb_denoise_temporal_output {
    float* rgbw;
    float* motion;
    uint32_t* history_length;
} trb_denoise_temporal_output;

/* An empty history for `scene`'s temporal denoising. Its per-pixel buffers (96 bytes per pixel) and the instance snapshot (64 bytes
 * per instance, twice) are allocated by its first call and grown where a call needs more (draining the device once, TRB_OOM if it does
 * not fit). Destroy it before its scene. */
trb_status trb_denoise_history_create(trb_scene* scene, trb_denoise_history** out);
trb_status trb_denoise_history_destroy(trb_denoise_history* history);
/* Empty the history and forget its film size; the next call filters as trb_denoise does. */
trb_status trb_denoise_history_reset(trb_denoise_history* history);

/* Denoise a frame with its history: HOST inputs and outputs, staged per call; blocking. Parameters are checked first (no scene is
 * needed to refuse them); then TRB_INVALID_ARG for a null scene, history, input or out->rgbw, a history of another scene or film size,
 * a scene without a frame, or an output overlapping an input or another output; TRB_OOM when scratch or history does not fit. A call
 * that fails leaves the history as it was. */
trb_status trb_denoise_temporal(trb_scene* scene, trb_denoise_history* history, const trb_denoise_input* in,
                                const trb_denoise_temporal_params* params, const trb_denoise_temporal_output* out);

/* trb_denoise_temporal with DEVICE buffers (films and rgbw 16-byte, nearest and motion 8-byte, history_length 4-byte aligned;
 * TRB_INVALID_ARG otherwise), enqueued on cuda_stream under trb_render_device's one-stream rule: 1 + iterations kernel launches and
 * one copy of the instance transforms. No host synchronisation, except once when the scratch or the history grows. */
trb_status trb_denoise_temporal_device(trb_scene* scene, trb_denoise_history* history, const trb_denoise_input* d_in,
                                       const trb_denoise_temporal_params* params, const trb_denoise_temporal_output* d_out,
                                       void* cuda_stream);

/* -- Temporal gradients: re-shade last frame's samples in this frame and shorten the history where the shading changed -------------
 * (DESIGN.md §4 "Temporal gradients"). A-SVGF's temporal gradients (Schied, Peters, Dachsbacher 2018) on top of trb_denoise_temporal:
 * a sample's radiance is a pure function of (scene, seed, key, sample), so one sample of the previous frame traced again in the
 * current scene with the same random numbers differs from its recorded value only where the shading changed.
 *
 * Strata: the film is cut into 3x3 strata from (0, 0), the last column and row possibly smaller; gw = ceil(W / 3), gh = ceil(H / 3),
 * S = gw * gh, stratum s = (s mod gw, s div gw). Its representative pixel is (min(3 sx + 1, W - 1), min(3 sy + 1, H - 1)).
 * The history gains one gradient record per stratum, in two sets read and written like the pixel sets: the hit's instance i and its
 * object-space point p_o, the camera ray (o, d, time), its key (the pixel index) and L_prev, the luminance L(x) = 0.2126 x.r +
 * 0.7152 x.g + 0.0722 x.b of the sample's radiance clamped to [0, 1] per channel; plus the frame's cam_world at shutter-open, its
 * shutter_open and the call's seed. The records are valid only if the previous call on the history was a gradient call of the same
 * object generation and film size; otherwise (first call, after reset, after trb_denoise_temporal or trb_denoise_moments, after
 * replace_objects, after trb_denoise_moments_gradient, whose history is of the moment family) there are
 * no gradients and lambda is 0 everywhere. Per call, float32, left to right, never contracted:
 *   1. Re-shade. For each valid record j (i below both instance counts): p_w' = mat_cur[i] . p_o, q = cam_inv_cur . p_w' (points as
 *      in "Temporal denoising"). Kept if q.z > 0, r = ((X - X0) / (X1 - X0) * W, (Y - Y1) / (Y0 - Y1) * H) with X = q.x / (q.z tan),
 *      Y = q.y / (q.z tan) lies in [0, W) x [0, H), the current nearest at pixel floor(r) has instance i, and |z - dist| <=
 *      depth_tolerance * z with dist = sqrt(v.x^2 + v.y^2 + v.z^2), v = p_w' - o_cur, o_cur = cam_world_cur . 0. Target stratum
 *      t = floor(r) / 3 per axis; its winner is the smallest (float bits of dist) << 32 | j (a 64-bit atomicMin, so scheduling
 *      does not matter). The winner's illumination ray: the recorded (o, d) if cam_world and mat[i] at shutter-open are both bit
 *      for bit the snapshot's, else o = o_cur, d = unit(p_w' - o_cur) (Vector::normalized); [0, +inf); time = rec.time +
 *      (shutter_open_cur - shutter_open_prev) (exactly rec.time when the shutter did not move); key and sample 0 from the record,
 *      traced by trb_illumination at the record's seed with TRB_QUERY_CLAMP and spp 1. L_cur = L(its radiance). The target gets
 *      delta = L_cur - L_prev, m = max(L_cur, L_prev), c = 1; a stratum without a winner gets (0, 0, 0).
 *   2. Reconstruct: `iterations` a-trous passes k = 0 .. N-1 on the stratum grid, step 2^k strata, taps dy then dx from -2 to 2 inside
 *      the grid with h = (1/16, 1/4, 3/8, 1/4, 1/16). A tap q counts when c_q > 0 and, for q != p, the representative pixels of p
 *      and q have the same instance (the low 32 bits of nearest) and their normals (normal_w.rgb / normal_w.w, unit as in
 *      trb_denoise; none if its length is 0 or not finite) both lack one or have n_p . n_q >= normal_threshold. W = sum h(dx) h(dy)
 *      over counted taps; W > 0: delta' = sum w delta / W, m' = sum w m / W, c' = 1; else (0, 0, 0). Then
 *      lambda = c > 0 && m > 0 ? min(1, |delta| / m) : 0.
 *   3. Blend: "Temporal denoising" with one change at step 4, lambda taken from the pixel's stratum: where there is history,
 *      len_adj = (uint32)floorf((1 - lambda) * (float)len_prev) and n' = min(len_adj + 1, max_history). Lambda 0 gives
 *      trb_denoise_temporal's pixel, lambda 1 trb_denoise's (n' = 1). The history stores n'.
 *   4. Record: in stratum s the pixel k = h mod (cw * ch) (row-major in the stratum, cw x ch its size), h = rng_absorb(rng_absorb(
 *      rng_absorb(rng_seed(seed), s), 0xfffffffe), 0) (the counter hash of the sample streams); its camera ray as trb_camera_rays
 *      generates sample 0 of 1 (with the ray's time), its hit as trb_intersect_records returns it (p_o = inv[i] . p at
 *      shutter-open) and L as step 1 computes it at `seed`. A miss leaves the record invalid.
 * Cost: about 2 S illumination samples and S ray queries per call on top of trb_denoise_temporal. */
typedef struct trb_denoise_gradient_params {
    trb_denoise_temporal_params temporal; /* as trb_denoise_temporal: same ranges and defaults */
    uint32_t iterations;                  /* gradient a-trous passes on the stratum grid: 0-6, default 3 */
    uint32_t pad[3];                      /* ignored */
} trb_denoise_gradient_params;            /* NULL: all defaults */

/* trb_denoise_temporal_output's three buffers, plus lambda (width*height floats, may be NULL): each pixel's lambda. */
typedef struct trb_denoise_gradient_output {
    float* rgbw;
    float* motion;
    uint32_t* history_length;
    float* lambda;
} trb_denoise_gradient_output;

/* trb_denoise_temporal with temporal gradients: the same inputs, history, checks and statuses (parameters first, and a failed call
 * leaves the history as it was), plus TRB_INVALID_ARG for iterations above 6 or a lambda output that overlaps another buffer.
 * `seed` seeds this frame's gradient samples (render_denoised_temporal passes the frame's seed). HOST buffers; blocking. The
 * history grows by 128 bytes of records and 328 bytes of per-call buffers per stratum. */
trb_status trb_denoise_temporal_gradient(trb_scene* scene, trb_denoise_history* history, const trb_denoise_input* in,
                                         const trb_denoise_gradient_params* params, uint32_t seed, const trb_denoise_gradient_output* out);

/* The same with DEVICE buffers (the alignment of trb_denoise_temporal_device, lambda 4-byte aligned), enqueued on cuda_stream under
 * trb_render_device's one-stream rule. No host synchronisation, except when scratch, history or the wavefront state grows. */
trb_status trb_denoise_temporal_gradient_device(trb_scene* scene, trb_denoise_history* history, const trb_denoise_input* d_in,
                                                const trb_denoise_gradient_params* params, uint32_t seed,
                                                const trb_denoise_gradient_output* d_out, void* cuda_stream);

/* -- Moment denoising: one film per frame, the variance from temporally accumulated luminance moments -------------------------------
 * (DESIGN.md §4 "Moment denoising"). SVGF's variance estimate (Schied et al. 2017, §4.2-4.3) in place of the two half films: each
 * pixel accumulates the first two moments of its luminance over its reprojected history, and where that history is shorter than
 * TRB_DENOISE_MOMENTS_MIN_HISTORY frames the variance is estimated spatially over a 7x7 window instead. So a frame needs one render at
 * any sample count, 1 spp included: colour is trb_render_aov's film of the frame's whole sample range, albedo_w, normal_w and nearest
 * its AOVs. The history is a trb_denoise_history as in "Temporal denoising" (same scene, film size, snapshot and generation rules);
 * its per-pixel sets hold (ē, z), (mu1, mu2, inst) and (n, n') in the same 96 bytes per pixel. A history last written by the other
 * family (trb_denoise_temporal* against trb_denoise_moments*) is treated as empty, as for another object generation.
 * Per pixel p = (x, y), float32, left to right, never contracted, L(x) = 0.2126 x.r + 0.7152 x.g + 0.0722 x.b:
 *   1. W = colour.w. W <= 0: the output is (0, 0, 0, 0), p is never a neighbour. c = colour.rgb / W; d, m, len2, n, z and dz are
 *      trb_denoise's; e = c / d, l = L(e). Unless c, albedo, m, len2 and e are all finite and z is neither NaN nor -inf, p is copied
 *      through as (c, 1) and is never a neighbour. Such pixels and W <= 0 ones store "none", have motion (NaN, NaN), history_length 0
 *      and variance NaN.
 *   2. Reprojection: steps 1-3 of "Temporal denoising", unchanged (the same motion, taps and instance, depth and normal tests), with
 *      H' = (sum of w * ē_t in tap order) / S per channel, M1' = (sum of w * mu1_t) / S, M2' = (sum of w * mu2_t) / S and len_prev.
 *   3. n' = min(len_prev + 1, max_history), or 1 without history. n' > 1: alpha = 1 / (float)n',
 *        ē = alpha * e + (1 - alpha) * H' per channel,  mu1 = alpha * l + (1 - alpha) * M1',  mu2 = alpha * (l * l) + (1 - alpha) * M2'
 *      n' == 1: ē = e, mu1 = l, mu2 = l * l. (The colour and the moments share the weight 1 / n'.)
 *   4. n' >= TRB_DENOISE_MOMENTS_MIN_HISTORY: v = max(0, mu2 - mu1 * mu1). Otherwise, over the 7x7 taps q = p + (dx, dy), dy then dx
 *      from -TRB_DENOISE_MOMENTS_RADIUS to TRB_DENOISE_MOMENTS_RADIUS, inside the image and filtered (p's own tap included, so the sum
 *      is > 0), with ē, mu1, mu2 of step 3 at q:
 *        w_l = exp(-(|L(ē_p) - L(ē_q)| / (sigma_luminance + TRB_DENOISE_EPS_LUMINANCE)))
 *        w_n, w_z = trb_denoise's at step s = 1 (w_z's denominator sigma_depth * |gx * dx + gy * dy| + TRB_DENOISE_EPS_DEPTH)
 *        w = w_l * w_n * w_z;  Sw, S1 = sum w * mu1, S2 = sum w * mu2 in tap order
 *        v = max(0, S2 / Sw - (S1 / Sw) * (S1 / Sw)) * (4 / (float)n')   (SVGF's boost of short histories)
 *   5. (ē, v) goes into trb_denoise's a-trous iterations; the output is remodulated by d as there (iterations 0: ē * d).
 *   6. A filtered pixel with finite z stores (ē, z), (mu1, mu2, i), (n, n'); every other pixel stores "none". The snapshot becomes the
 *      current frame's. Gradient records (trb_denoise_temporal_gradient) become invalid.
 * max_history 1 makes every call a single-frame spatial denoiser of one film (n' = 1 everywhere). Every NaN written to rgbw, motion
 * or variance is 0x7fffffff. The scene's denoise scratch grows to 88 bytes per pixel for moment calls (72 for every other denoise). */
#define TRB_DENOISE_MOMENTS_MIN_HISTORY 4
#define TRB_DENOISE_MOMENTS_RADIUS 3

/* One colour film of the frame at any sample count and its AOVs, all required: host pointers for trb_denoise_moments, device
 * pointers for trb_denoise_moments_device. The scene's film layout, as trb_denoise_input. */
typedef struct trb_denoise_frame {
    const float* colour;
    const float* albedo_w;
    const float* normal_w;
    const uint64_t* nearest;
} trb_denoise_frame;

/* rgbw (width*height*4 floats) is required; motion (width*height*2 floats), history_length (width*height uint32) and variance
 * (width*height floats: each pixel's v of step 4, the variance the a-trous iterations start from) may be NULL. */
typedef struct trb_denoise_moments_output {
    float* rgbw;
    float* motion;
    uint32_t* history_length;
    float* variance;
} trb_denoise_moments_output;

/* Denoise a frame of one film with its history: HOST inputs and outputs, staged per call; blocking. The parameters are
 * trb_denoise_temporal's, checked first (no scene is needed to refuse them); then TRB_INVALID_ARG for a null scene, history, input
 * member or out->rgbw, a history of another scene or film size, a scene without a frame, or an output overlapping an input or another
 * output; TRB_OOM when scratch or history does not fit. A call that fails leaves the history as it was. */
trb_status trb_denoise_moments(trb_scene* scene, trb_denoise_history* history, const trb_denoise_frame* in,
                               const trb_denoise_temporal_params* params, const trb_denoise_moments_output* out);

/* trb_denoise_moments with DEVICE buffers (colour, albedo_w, normal_w and rgbw 16-byte, nearest and motion 8-byte, history_length and
 * variance 4-byte aligned; TRB_INVALID_ARG otherwise), enqueued on cuda_stream under trb_render_device's one-stream rule: 2 +
 * iterations kernel launches and one copy of the instance transforms. No host synchronisation, except once when the scratch or the
 * history grows. */
trb_status trb_denoise_moments_device(trb_scene* scene, trb_denoise_history* history, const trb_denoise_frame* d_in,
                                      const trb_denoise_temporal_params* params, const trb_denoise_moments_output* d_out,
                                      void* cuda_stream);

/* -- Sample variance: denoise one render with the variance of its own samples (DESIGN.md §4 "Sample variance") ------------------
 * The lum_w film. trb_render_aov_lum and trb_render_adaptive_aov_lum (and their _device forms) add one more AOV film, in the colour
 * film's layout (width*height RGBW floats, added into). Per camera sample, float32, left to right, never contracted, with c the
 * radiance the colour film adds for the sample and a the albedo of its AOV record (0 on a miss):
 *   d = max(a, TRB_DENOISE_EPS_ALBEDO) per channel,  l = L(c / d) = 0.2126 (c.r / d.r) + 0.7152 (c.g / d.g) + 0.0722 (c.b / d.b)
 *   the sample adds (w * l, w * (l * l), w * w, w) with the colour film's weights w (RenderTarget::write: filter table,
 *   filter_pixel_width window, 2x2 lock blocks); Mitchell's w can be negative, w * w is not. lum_w.w is the colour film's W up to
 *   float addition order. An Adaptive render adds every sample of every round under the colour film's Adaptive rules.
 * Each sample is demodulated by its own albedo, not by the pixel's filtered one: albedo changes inside a pixel's footprint are
 * antialiasing, not noise, and do not raise the variance.
 *
 * trb_denoise_variance: trb_denoise's filter over one film with v from lum_w. Per pixel p, float32, left to right, never contracted:
 *   1. W = colour.w. W <= 0: the output is (0, 0, 0, 0) and p is never a neighbour. c = colour.rgb / W; d, m, len2, n, z, dz and
 *      e = c / d are trb_denoise's.
 *   2. V1 = lum_w.w, V2 = lum_w.z, m1 = lum_w.x / V1, m2 = lum_w.y / V1. If V1 > 0 and V1 * V1 > V2:
 *        v = max(0, m2 - m1 * m1) * V2 / (V1 * V1 - V2),   max(0, x) = x > 0 ? x : 0
 *      otherwise (at most one effective sample) v = NaN. For independent samples this is the unbiased estimate of the variance of
 *      the pixel's weighted mean of l (reliability weights); with equal weights it is s^2 / n. LowDiscrepancy's stratified samples
 *      have a smaller true variance than independent ones, so v overestimates it and errs toward blurring.
 *   3. Unless c, albedo, m, len2, e and v are all finite and z is neither NaN nor -inf, p is copied through as (c, 1) and is never
 *      a neighbour.
 *   4. (e, v) goes into trb_denoise's a-trous iterations unchanged; the output is (e_N * d, 1) (iterations 0: e * d). Every NaN
 *      written to rgbw or variance is 0x7fffffff. variance (may be NULL; width*height floats) receives v, or NaN where p is not
 *      filtered.
 * No history: a still image, or any frame on its own. The scene's denoise scratch is trb_denoise's 72 bytes per pixel.
 * The Adaptive forms, trb_render_adaptive_aov_lum*, are declared with the Adaptive AOVs below. */

/* trb_render_aov with the lum_w film (HOST, width*height*4 floats, added into; required). The colour film, the AOVs and every
 * trb_stats counter equal trb_render_aov's with the same cfg, and so do the statuses. The AOV records are computed even when
 * aov's three members are NULL. Blocking. */
trb_status trb_render_aov_lum(trb_scene* scene, const trb_render_cfg* cfg, float* film_rgbw, const trb_aov_film* aov, float* lum_w,
                              trb_stats* stats);
/* trb_render_aov_device with the DEVICE lum_w film (16-byte aligned, else TRB_INVALID_ARG). */
trb_status trb_render_aov_lum_device(trb_scene* scene, const trb_render_cfg* cfg, float* d_film_rgbw, const trb_aov_film* d_aov, float* d_lum_w,
                                     trb_stats* d_stats, void* cuda_stream);

/* Denoise one film with its lum_w film: HOST inputs and outputs (rgbw required, width*height*4 floats, overwritten; variance may be
 * NULL), staged per call; blocking. The parameters are trb_denoise's, checked first (no scene is needed to refuse them); then
 * TRB_INVALID_ARG for a null scene, input member, lum_w or rgbw, or an output overlapping an input or the other output; TRB_OOM when
 * the scratch does not fit. */
trb_status trb_denoise_variance(trb_scene* scene, const trb_denoise_frame* in, const float* lum_w, const trb_denoise_params* params,
                                float* out_rgbw, float* out_variance);
/* The same with DEVICE buffers (films, lum_w and rgbw 16-byte, nearest 8-byte, variance 4-byte aligned; TRB_INVALID_ARG otherwise),
 * enqueued on cuda_stream under trb_render_device's one-stream rule: 1 + iterations kernel launches. No host synchronisation, except
 * once when the scratch grows. */
trb_status trb_denoise_variance_device(trb_scene* scene, const trb_denoise_frame* d_in, const float* d_lum_w, const trb_denoise_params* params,
                                       float* d_out_rgbw, float* d_out_variance, void* cuda_stream);

/* -- Moment gradients: temporal gradients on the moment denoiser, so a 1-spp history drops where the lighting changed -------------
 * (DESIGN.md §4 "Moment gradients"). A-SVGF (Schied, Peters, Dachsbacher 2018) is SVGF at one sample per pixel with temporal
 * gradients: "Moment denoising" with the lambda of "Temporal gradients". Per call:
 *   - steps 1, 2 and 4 of "Temporal gradients" run unchanged: re-shade the previous records at the previous seed, reconstruct lambda
 *     on the 3x3 stratum grid (normal_w and nearest of the frame), and record this frame's samples at `seed`;
 *   - "Moment denoising" runs with one change at step 3: where there is history, n' = min((uint32)floorf((1 - lambda) *
 *     (float)len_prev) + 1, max_history) with lambda taken from the pixel's stratum, and ē, mu1 and mu2 blend with that 1 / n'.
 *     A shortened history falls below TRB_DENOISE_MOMENTS_MIN_HISTORY exactly where the lighting changed, so step 4's 7x7 spatial
 *     variance with its 4 / n' boost takes over there. Lambda 0 everywhere gives trb_denoise_moments's pixel bit for bit, lambda 1
 *     its max_history 1 pixel.
 * The records are valid only if the previous call on the history was a moment gradient call of the same object generation and film
 * size; otherwise (first call, after reset, after replace_objects, trb_denoise_moments or any half-film call) lambda is 0
 * everywhere. A half-film call (trb_denoise_temporal*, trb_denoise_temporal_gradient*) after a moment gradient call finds no
 * history, as after trb_denoise_moments. The history and scratch sizes are those of the two calls combined: 96 bytes per pixel,
 * 456 bytes per stratum and 88 bytes per pixel of scratch. */

/* trb_denoise_moments_output's four buffers, plus lambda (width*height floats, may be NULL): each pixel's lambda. */
typedef struct trb_denoise_moments_gradient_output {
    float* rgbw;
    float* motion;
    uint32_t* history_length;
    float* variance;
    float* lambda;
} trb_denoise_moments_gradient_output;

/* trb_denoise_moments with temporal gradients: the same inputs, history, checks and statuses (the parameters first, with no scene
 * needed, and a failed call leaves the history as it was), plus TRB_INVALID_ARG for iterations above 6 or a lambda output that
 * overlaps another buffer. `seed` seeds this frame's gradient samples (render_denoised_moments(gradients=True) passes the frame's
 * seed). HOST buffers; blocking. */
trb_status trb_denoise_moments_gradient(trb_scene* scene, trb_denoise_history* history, const trb_denoise_frame* in,
                                        const trb_denoise_gradient_params* params, uint32_t seed,
                                        const trb_denoise_moments_gradient_output* out);

/* The same with DEVICE buffers (the alignment of trb_denoise_moments_device, lambda 4-byte aligned), enqueued on cuda_stream under
 * trb_render_device's one-stream rule. No host synchronisation, except when scratch, history or the wavefront state grows. */
trb_status trb_denoise_moments_gradient_device(trb_scene* scene, trb_denoise_history* history, const trb_denoise_frame* d_in,
                                               const trb_denoise_gradient_params* params, uint32_t seed,
                                               const trb_denoise_moments_gradient_output* d_out, void* cuda_stream);

/* -- Variance temporal denoising: animations denoised with the variance of their own samples, carried through the history ---------
 * (DESIGN.md §4 "Variance temporal denoising"). "Sample variance" over a history: each frame's lum_w film gives the variance v_f of
 * the frame's pixel mean, and for the blend ē = alpha e + (1 - alpha) H' of independent frames the history carries V' = Var(H'), so
 * Var(ē) = alpha^2 v_f + (1 - alpha)^2 V' exactly, for any sequence of alpha. One render per frame at 2 spp or more (LowDiscrepancy
 * or Adaptive), a variance that shrinks as the history grows, and no spatial estimate. The inputs are a trb_denoise_frame and the
 * lum_w film of the same render (trb_render_aov_lum* or trb_render_adaptive_aov_lum*) at the scene's current frame; the history is a
 * trb_denoise_history with the scene, film size, snapshot and generation rules of "Temporal denoising". Per pixel p, float32, left to
 * right, never contracted:
 *   1. W, c, d, e, n, z, dz and v_f are trb_denoise_variance's steps 1-3 (v_f from lum_w). A pixel that call does not filter (W <= 0,
 *      anything non-finite, or v_f NaN: at most one effective sample) is written exactly as it writes it, stores "none", and has
 *      motion (NaN, NaN), history_length 0 and variance NaN.
 *   2. Reprojection: steps 1-3 of "Temporal denoising", unchanged, over this family's sets: H' = (sum of w * ē_t in tap order) / S per
 *      channel, V' = (sum of w * V_t in tap order) / S, and len_prev.
 *   3. n' = min(len_prev + 1, max_history), or 1 without history; in the gradient form, where there is history, n' =
 *      min((uint32)floorf((1 - lambda) * (float)len_prev) + 1, max_history) with lambda from the pixel's stratum ("Temporal
 *      gradients" steps 1, 2 and 4 run unchanged around it). n' > 1: alpha = 1 / (float)n', beta = 1 - alpha,
 *        ē = alpha * e + beta * H' per channel,  V = (alpha * alpha) * v_f + (beta * beta) * V'
 *      n' == 1: ē = e, V = v_f.
 *   4. (ē, V) goes into trb_denoise's a-trous iterations unchanged; the output is remodulated by d (iterations 0: ē * d).
 *   5. A filtered pixel with finite z stores (ē, z), (V, 0, 0, i), (n, n'): 96 bytes per pixel, as the other families. variance
 *      receives V. Every NaN written to rgbw, motion or variance is 0x7fffffff.
 * An empty history or max_history 1 gives trb_denoise_variance's rgbw and variance bit for bit; in the gradient form lambda 0
 * everywhere gives the plain call's pixel, lambda 1 trb_denoise_variance's.
 * History families: the half-film calls (trb_denoise_temporal*), the moment calls (trb_denoise_moments*) and these calls each treat
 * a history last written by another family as empty. Gradient records are valid only after a variance gradient call of the same
 * object generation and film size; a plain variance call invalidates them. The scene's denoise scratch is 72 bytes per pixel. */

/* Denoise a frame of one film with its lum_w film and its history: HOST inputs and outputs (lum_w width*height*4 floats), staged per
 * call; blocking. The parameters are trb_denoise_temporal's, checked first (no scene is needed to refuse them); then TRB_INVALID_ARG
 * for a null scene, history, input member, lum_w or out->rgbw, a history of another scene or film size, a scene without a frame, or
 * an output overlapping an input or another output; TRB_OOM when scratch or history does not fit. A call that fails leaves the
 * history as it was. */
trb_status trb_denoise_variance_temporal(trb_scene* scene, trb_denoise_history* history, const trb_denoise_frame* in, const float* lum_w,
                                         const trb_denoise_temporal_params* params, const trb_denoise_moments_output* out);

/* The same with DEVICE buffers (the alignment of trb_denoise_moments_device, lum_w 16-byte aligned; TRB_INVALID_ARG otherwise),
 * enqueued on cuda_stream under trb_render_device's one-stream rule: 1 + iterations kernel launches and one copy of the instance
 * transforms. No host synchronisation, except once when the scratch or the history grows. */
trb_status trb_denoise_variance_temporal_device(trb_scene* scene, trb_denoise_history* history, const trb_denoise_frame* d_in,
                                                const float* d_lum_w, const trb_denoise_temporal_params* params,
                                                const trb_denoise_moments_output* d_out, void* cuda_stream);

/* trb_denoise_variance_temporal with temporal gradients: the same inputs, history, checks and statuses (the parameters first, and a
 * failed call leaves the history as it was), plus TRB_INVALID_ARG for iterations above 6 or a lambda output that overlaps another
 * buffer. `seed` seeds this frame's gradient samples. HOST buffers; blocking. */
trb_status trb_denoise_variance_temporal_gradient(trb_scene* scene, trb_denoise_history* history, const trb_denoise_frame* in,
                                                  const float* lum_w, const trb_denoise_gradient_params* params, uint32_t seed,
                                                  const trb_denoise_moments_gradient_output* out);

/* The same with DEVICE buffers (the alignment of trb_denoise_variance_temporal_device, lambda 4-byte aligned), enqueued on
 * cuda_stream under trb_render_device's one-stream rule: trb_denoise_moments_gradient_device's launches without its variance kernel.
 * No host synchronisation, except when scratch, history or the wavefront state grows. */
trb_status trb_denoise_variance_temporal_gradient_device(trb_scene* scene, trb_denoise_history* history, const trb_denoise_frame* d_in,
                                                         const float* d_lum_w, const trb_denoise_gradient_params* params, uint32_t seed,
                                                         const trb_denoise_moments_gradient_output* d_out, void* cuda_stream);

/* trb_camera_rays with DEVICE buffers on the scene's GPU (4-byte aligned), enqueued on cuda_stream (a cudaStream_t; NULL = default
 * stream) without host synchronisation: the same kernel, so the same bits. The checks and statuses of trb_camera_rays, plus
 * TRB_INVALID_ARG for unaligned buffers; before the first update_frame it is TRB_INVALID_ARG. */
trb_status trb_camera_rays_device(trb_scene* scene, const trb_render_cfg* cfg, size_t n, trb_ray* d_rays, float* d_xy,
                                  void* cuda_stream);

/* -- film writes: RenderTarget::write (render_target.rs:77-165) for caller samples ---------------------------------------------
 * samples[i] is an ImageSample: film position (x, y) and colour (r, g, b); trb_render_samples' output goes straight in.
 * regions[i] is the Region `write` receives for the sample: the 8x8 block with row-major index by * (width / 8) + bx. A region
 * index >= the block count skips the sample. Regions are not derived from floor(x): a low-discrepancy position vdc + px can round
 * up to exactly px + 1, into the next pixel and sometimes the next block, and the render writes that sample with the block it came
 * from, so only an explicit region reproduces the render.
 * Order: the result equals, bit for bit, the film left by this sequence of reference calls: start from the caller's film, call
 * RenderTarget::write once per region that has at least one sample, regions in the order of the scene's Morton block list
 * (block_queue.rs:28-46, trb_block_list), each region's samples in input order. That is the order a one-thread
 * MultiThreaded::render writes in, so trb_render_samples of a whole frame written with this call gives the film of a one-thread
 * reference render. Consequences: a pixel inside the write range [start - fpw, start + 8 + fpw] (clipped to the image) of a
 * non-empty region gets += S_r even when S_r is zero, which turns -0.0 into +0.0; pixels outside every write range keep their
 * bits; two calls compose as two sequences of writes; splitting one block's samples across calls changes the last bits.
 * Film: RGBW, row-major, width*height*4 floats (get_renderf32 layout), added into in place like trb_render. The filter is fixed
 * when the scene is created, so no update_frame is needed. No float atomics: the result does not depend on scheduling.
 * Statuses: TRB_INVALID_ARG for null arguments with n > 0, unaligned device buffers (4 bytes) and n >= 2^32 (checked before
 * anything is read); n == 0 is TRB_OK. The sort needs about 16 bytes of scratch per sample on the device (kept by the scene and
 * grown on demand); TRB_OOM when it does not fit: the write is never split into passes, because a split would change the result.
 * The host form takes host buffers and blocks. The _device form takes device buffers on the scene's GPU and enqueues on
 * cuda_stream under trb_render_device's one-stream-per-scene rule, without host synchronisation except once, when the scratch
 * space grows. */
trb_status trb_film_write(trb_scene* scene, size_t n, const trb_sample* samples, const uint32_t* regions, float* film_rgbw);
trb_status trb_film_write_device(trb_scene* scene, size_t n, const trb_sample* d_samples, const uint32_t* d_regions,
                                 float* d_film_rgbw, void* cuda_stream);

/* ≙ RenderTarget::get_render (render_target.rs:185-210): rgb/weight, clamp, sRGB,
 * (c*255) as u8; pixels with weight <= 0 stay 0. Host buffers; runs on the scene's GPU. */
trb_status trb_film_to_srgb8(trb_scene* scene, const float* film_rgbw, uint8_t* rgb8);

/* The same conversion on the host, with no scene and no device: ≙ Image::get_srgb8 (film/image.rs:53-67), which the distributed
 * master applies to the blocks its workers sent. film_rgbw holds width*height RGBW pixels, rgb8 receives width*height*3 bytes.
 * The bytes equal trb_film_to_srgb8's for the same film, bit for bit (one per-pixel function compiled for both sides), including
 * weights <= 0 or NaN (black), infinities and NaN colours. TRB_INVALID_ARG for null buffers with width*height > 0. */
trb_status trb_host_film_to_srgb8(uint32_t width, uint32_t height, const float* film_rgbw, uint8_t* rgb8);

/* ≙ image::save_buffer(path, &img, w, h, image::RGB(8)) for the frames written by main.rs:95-103 and by the distributed
 * master (exec/distrib/master.rs:137-142): an 8-bit RGB PNG (stored deflate blocks; host only, no device needed). */
trb_status trb_write_png(const char* path, const uint8_t* rgb8, uint32_t width, uint32_t height);

/* -- Adaptive sampler (sampler/adaptive.rs) ------------------------------------------
 * min_spp samples per pixel, then `step` more per round while the pixel's samples disagree (some sample's
 * |luminance - average| / average > 0.5), until samples_taken >= max_spp. min_spp and max_spp are rounded up to powers of
 * two (0 -> 1), step = ((max - min) / 5) rounded up to a power of two; a pixel ends with at most max_per_pixel samples,
 * which can exceed max_spp (min 4, max 64: step 16, up to 68). Path integrator, wavefront pipeline only. */
typedef struct trb_adaptive {
    uint32_t min_spp, max_spp;
} trb_adaptive;

/* Exec::render with the Adaptive sampler: every selected block, all rounds, one blocking call; the film is ADDED to
 * film_rgbw like trb_render. cfg->spp, sample_first and sample_count must be 0 (the sampler owns the schedule).
 * pixel_spp (width*height, or NULL) receives the sample count of each pixel of the selected blocks; other entries are
 * left as they are. TRB_INVALID_ARG when max < min after rounding; TRB_UNSUPPORTED for the Whitted / NormalsDebug
 * integrators and TRB_RENDER_MEGAKERNEL. */
trb_status trb_render_adaptive(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* film_rgbw,
                               uint32_t* pixel_spp, trb_stats* stats);

/* Parity variant of trb_render_adaptive: the clamped sample of every (block, pixel, slot) in the trb_render_samples order
 * with max_per_pixel slots per pixel: n = blocks*64*max_per_pixel, slots a pixel did not take are zero. Does not update
 * the frame. */
trb_status trb_render_samples_adaptive(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, size_t n,
                                       trb_sample* samples, uint32_t* pixel_spp, trb_stats* stats);

/* trb_render_adaptive with the contract of trb_render_device: the film is a DEVICE buffer on the scene's GPU (accumulated
 * into), every round is enqueued on `cuda_stream` (a cudaStream_t; NULL = default stream) without host synchronisation,
 * and update_frame is never called. The rounds are driven by the device: the host enqueues every round of the schedule
 * with the passes the whole selection would need, and passes past a round's live blocks return at once. `d_pixel_spp`
 * is NULL or a DEVICE buffer of width*height u32 with the layout of trb_render_adaptive's pixel_spp; only the selected
 * pixels are written. `d_stats` (may be NULL) is a DEVICE trb_stats the kernels accumulate into. The first call on a
 * scene allocates the sampler's per-pixel state (20 B per pixel), and a call that needs more path state than earlier
 * calls grows it, as trb_render_device does; both synchronise the device once. Same one-stream-per-scene rule as
 * trb_render_device; the same argument checks and statuses as trb_render_adaptive. */
trb_status trb_render_adaptive_device(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* d_film_rgbw,
                                      uint32_t* d_pixel_spp, trb_stats* d_stats, void* cuda_stream);

/* -- AOVs of Adaptive renders (DESIGN.md §4 "Adaptive AOVs") -------------------------------------------------------------
 * trb_render_adaptive that also renders the AOVs (trb_aov_sample, trb_aov_film) of every sample it takes into the HOST buffers of
 * `aov`: albedo_w and normal_w are added into with the colour film's weights, so their W equals the colour film's W up to float
 * addition order; nearest is read and written (initialise it to all ones); any of the three may be NULL. The colour film,
 * pixel_spp and every trb_stats counter equal trb_render_adaptive's with the same arguments. Statuses: trb_render_adaptive's
 * (TRB_INVALID_ARG for a non-zero spp, sample_first or sample_count, or max < min after rounding; TRB_UNSUPPORTED for the
 * Whitted / NormalsDebug integrators and TRB_RENDER_MEGAKERNEL), which include trb_render_aov's. The first AOV render allocates
 * 32 B of AOV record per path in flight, as trb_render_aov does. Blocking. */
trb_status trb_render_adaptive_aov(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* film_rgbw,
                                   const trb_aov_film* aov, uint32_t* pixel_spp, trb_stats* stats);

/* trb_render_adaptive_aov with the contract of trb_render_adaptive_device: the film, d_pixel_spp, d_stats and the outputs of
 * `d_aov` (a host struct of DEVICE pointers) are device buffers on the scene's GPU; every round is enqueued on cuda_stream without
 * host synchronisation, and update_frame is never called. TRB_INVALID_ARG for a film or an AOV film that is not 16-byte aligned,
 * or a nearest buffer that is not 8-byte aligned, as trb_render_aov_device. */
trb_status trb_render_adaptive_aov_device(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* d_film_rgbw,
                                          const trb_aov_film* d_aov, uint32_t* d_pixel_spp, trb_stats* d_stats, void* cuda_stream);

/* trb_render_samples_adaptive that also writes the AOV record of every (block, pixel, slot) into the HOST buffer aov[n], in the
 * same layout: n = blocks*64*max_per_pixel, slots a pixel did not take are zero. samples[], pixel_spp and the stats equal
 * trb_render_samples_adaptive's. Does not update the frame. */
trb_status trb_render_samples_adaptive_aov(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, size_t n,
                                           trb_sample* samples, trb_aov_sample* aov, uint32_t* pixel_spp, trb_stats* stats);

/* trb_render_adaptive_aov with the HOST lum_w film of "Sample variance" (width*height*4 floats, added into; required): the film,
 * AOVs, pixel_spp, counters and statuses are trb_render_adaptive_aov's. */
trb_status trb_render_adaptive_aov_lum(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* film_rgbw,
                                       const trb_aov_film* aov, float* lum_w, uint32_t* pixel_spp, trb_stats* stats);
/* trb_render_adaptive_aov_device with the DEVICE lum_w film (16-byte aligned, else TRB_INVALID_ARG). */
trb_status trb_render_adaptive_aov_lum_device(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* d_film_rgbw,
                                              const trb_aov_film* d_aov, float* d_lum_w, uint32_t* d_pixel_spp, trb_stats* d_stats,
                                              void* cuda_stream);

/* -- Motion vectors: each camera sample's screen-space motion to another time, from the scene's own animation (DESIGN.md §4
 * "Motion vectors") -------------------------------------------------------------------------------------------------------------
 * For one camera sample: its trb_camera_rays ray, that ray's time t, and its hit as trb_intersect_records returns it (instance i,
 * world point p). dt is the caller's time offset, a finite float. Per sample, float32, left to right, never contracted:
 *   1. p_o = M_i(t)^-1 . p, the hit in instance i's object space through the transform the trace uses (the per-path transform table of
 *      a keyframed instance, the frame's fixed matrices of a static one).
 *   2. p_now = M_i(t) . p_o and p_then = M_i(t + dt) . p_o, where M_i(tau) is a keyframed instance's AnimatedTransform at tau (as
 *      eval_anim_xf evaluates it) and a static instance's fixed transform. p_now is p sent through the same transforms as p_then, so
 *      that both terms of step 4 go through the same arithmetic.
 *   3. r(tau, x) projects the world point x to raster coordinates with the camera active for the current frame at time tau, inverting
 *      camera_ray's raster -> camera mapping: q = cam_world(tau)^-1 . x, X = q.x / (q.z * tan_tau), Y = q.y / (q.z * tan_tau),
 *      r = ((X - x0) / (x1 - x0) * width, (Y - y1) / (y0 - y1) * height) with camera_setup's screen window (x0, x1, y0, y1).
 *      tan_tau = tan(fov / 2); an animated fov is sampled once per frame at the clamped mid-frame time m (camera.rs:134-141), so
 *      tan_t is the frame's own and tan_{t+dt} is the spline's at clamp(m + dt): one frame back gives the previous frame's fov.
 *   4. m = r(t + dt, p_then) - r(t, p_now), in pixels. A scene with nothing keyframed, and any scene at dt = 0, gives (0, 0) exactly.
 *   5. valid = 1 where the hit is in front of the camera (q.z > 0) at both times; else valid = 0 and m = (0, 0). A miss is invalid.
 * dt = -(scene_time / frames) gives the backward vectors a temporal filter wants (previous position minus current, the sign of the
 * temporal denoisers' motion output); +scene_time / frames gives forward flow.
 * Not seen: edits made between calls (trb_scene_update_keyframes, trb_scene_replace_objects, mesh updates and refits) and a camera cut
 * between t and t + dt: the motion is that of the current scene and the current frame's camera. Deforming meshes do not move.
 * Path integrator on the wavefront only: Whitted, NormalsDebug and TRB_RENDER_MEGAKERNEL give TRB_UNSUPPORTED; a non-finite dt is
 * TRB_INVALID_ARG, checked before anything is enqueued. The first motion render allocates 16 B of record per path in flight. */

/* One sample's motion: valid is 1.0f or 0.0f, so a record is (v dx, v dy, v, 0), the value the motion_w film adds per unit weight.
 * 16 bytes. */
typedef struct trb_motion_sample {
    float dx, dy;
    float valid;
    uint32_t reserved; /* 0 */
} trb_motion_sample;

/* trb_render_samples_aov that also writes each camera sample's motion record into the HOST buffer motion[n], in the same order.
 * samples[], aov[] and the stats equal trb_render_samples_aov's; its statuses, plus dt's. */
trb_status trb_render_samples_aov_motion(trb_scene* scene, const trb_render_cfg* cfg, size_t n, trb_sample* samples, trb_aov_sample* aov,
                                         trb_motion_sample* motion, float dt, trb_stats* stats);

/* The motion_w film: RGBW in the colour film's layout (width*height*4 floats, added into). Each sample adds (w v dx, w v dy, w v, w)
 * with the colour film's weights (RenderTarget::write: filter table, filter_pixel_width window, 2x2 lock blocks); it is the colour
 * film's kernel over the records in place of the radiance. A pixel's motion is (x / z, y / z) where z > 0; w is the colour film's W
 * up to float addition order.
 * trb_render_aov_lum with the HOST motion_w film (required) and lum_w (may be NULL: not rendered). The colour film, the AOVs, lum_w and
 * every trb_stats counter equal trb_render_aov_lum's (trb_render_aov's without lum_w); so do the statuses, plus dt's. Blocking. */
trb_status trb_render_aov_motion(trb_scene* scene, const trb_render_cfg* cfg, float* film_rgbw, const trb_aov_film* aov, float* lum_w,
                                 float* motion_w, float dt, trb_stats* stats);
/* The same with DEVICE buffers under trb_render_aov_lum_device's contract; d_motion_w (required) and d_lum_w 16-byte aligned, else
 * TRB_INVALID_ARG. */
trb_status trb_render_aov_motion_device(trb_scene* scene, const trb_render_cfg* cfg, float* d_film_rgbw, const trb_aov_film* d_aov,
                                        float* d_lum_w, float* d_motion_w, float dt, trb_stats* d_stats, void* cuda_stream);
/* trb_render_adaptive_aov_lum with the HOST motion_w film (required; lum_w may be NULL): every sample of every round adds to it under
 * the colour film's Adaptive rules. The film, AOVs, lum_w, pixel_spp, counters and statuses are trb_render_adaptive_aov_lum's (or
 * trb_render_adaptive_aov's), plus dt's. */
trb_status trb_render_adaptive_aov_motion(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* film_rgbw,
                                          const trb_aov_film* aov, float* lum_w, float* motion_w, float dt, uint32_t* pixel_spp,
                                          trb_stats* stats);
/* The same with DEVICE buffers (d_motion_w and d_lum_w 16-byte aligned, else TRB_INVALID_ARG). */
trb_status trb_render_adaptive_aov_motion_device(trb_scene* scene, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* d_film_rgbw,
                                                 const trb_aov_film* d_aov, float* d_lum_w, float* d_motion_w, float dt,
                                                 uint32_t* d_pixel_spp, trb_stats* d_stats, void* cuda_stream);

/* trb_render_sharded with the Adaptive sampler: this rank's shard (interleaved chunks, or the reference's contiguous
 * ranges with cfg->shard_count == 0xffffffff) runs the Adaptive rounds into the device film, then ONE reduce to `root`,
 * whose host film_rgbw the summed film is ADDED to. pixel_spp (width*height, or NULL) receives the counts of this rank's
 * own pixels only; other entries are left as they are. Blocking. */
trb_status trb_render_sharded_adaptive(trb_scene* scene, trb_comm* comm, const trb_render_cfg* cfg, const trb_adaptive* adaptive,
                                       int root, float* film_rgbw, uint32_t* pixel_spp, trb_stats* stats);

/* trb_group_render with the Adaptive sampler: the replicas run their shards' rounds concurrently, then one reduce to
 * devices[0]; each replica's pixel counts are written into the one pixel_spp (the shards are disjoint). Blocking. */
trb_status trb_group_render_adaptive(trb_group* group, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* film_rgbw,
                                     uint32_t* pixel_spp, trb_stats* stats);

/* -- AOVs of multi-GPU renders (DESIGN.md §4 "Multi-GPU AOVs") ----------------------------------------------------------
 * trb_render_sharded, trb_render_sharded_adaptive, trb_group_render and trb_group_render_adaptive that also render the AOVs
 * (trb_aov_film). Every rank or replica renders albedo_w, normal_w and nearest of its own shard into device films the scene owns
 * (allocated by the first such render, 40 B per pixel, released with the film), and ONE NCCL group per frame reduces the colour film
 * and the three AOVs to the root: the films summed, nearest min-reduced (exact: the shards own disjoint pixels). The root (the
 * group: the caller) then holds what trb_render_aov / trb_render_adaptive_aov give on one GPU: film_rgbw, albedo_w and normal_w
 * added into, nearest read and min-merged, a NULL member of `aov` skipped; the sums equal one-GPU output up to float addition order,
 * nearest and pixel_spp exactly. On a sharded call the non-root ranks may pass film_rgbw and aov as NULL. A one-rank communicator
 * performs no reduce, and a group of one device calls trb_render_aov / trb_render_adaptive_aov on its replica.
 * Every check that depends only on arguments all ranks share (null arguments, trb_render_aov's and trb_render_adaptive's statuses,
 * the group's film sizes) fails on every rank before any rank renders, so no rank is left waiting in the reduce. Blocking. */
trb_status trb_render_sharded_aov(trb_scene* scene, trb_comm* comm, const trb_render_cfg* cfg, int root, float* film_rgbw,
                                  const trb_aov_film* aov, trb_stats* stats);
trb_status trb_render_sharded_adaptive_aov(trb_scene* scene, trb_comm* comm, const trb_render_cfg* cfg, const trb_adaptive* adaptive, int root,
                                           float* film_rgbw, const trb_aov_film* aov, uint32_t* pixel_spp, trb_stats* stats);
trb_status trb_group_render_aov(trb_group* group, const trb_render_cfg* cfg, float* film_rgbw, const trb_aov_film* aov, trb_stats* stats);
trb_status trb_group_render_adaptive_aov(trb_group* group, const trb_render_cfg* cfg, const trb_adaptive* adaptive, float* film_rgbw,
                                         const trb_aov_film* aov, uint32_t* pixel_spp, trb_stats* stats);

/* The rounded schedule of Adaptive::new (adaptive.rs:34-49); any output may be NULL. Host only. */
trb_status trb_adaptive_schedule(const trb_adaptive* adaptive, uint32_t* min_spp, uint32_t* max_spp, uint32_t* step,
                                 uint32_t* max_per_pixel);

/* The per-pixel decision the device runs (csrc/trb_adaptive.h), over a caller-given luminance sequence lum[0..n) in slot
 * order: the pixel's final sample count and average luminance. TRB_INVALID_ARG when the sequence ends before the pixel
 * stops sampling. Host only. */
trb_status trb_host_adaptive_decide(const trb_adaptive* adaptive, const float* lum, size_t n, uint32_t* samples_taken,
                                    float* avg);

/* -- introspection for parity tests ------------------------------------------------ */

/* The Morton-sorted 8x8 block list (block_queue.rs:28-46) after select_blocks: pairs (bx,by). */
trb_status trb_block_list(const trb_scene* scene, uint32_t block_start, uint32_t block_count,
                          uint32_t* n_out, uint32_t* xy_pairs, uint32_t capacity);

/* Flattened BVH in the reference's node order. which = -1: BVH<Instance> (after
 * update_frame); which >= 0: the BVH<Triangle> of mesh `which`. Pass NULL buffers to
 * query sizes. `ordered` is bvh.rs `ordered_geom`. */
trb_status trb_scene_get_bvh(const trb_scene* scene, int which, uint32_t* n_nodes, trb_bvh_node* nodes,
                             uint32_t* n_ordered, uint32_t* ordered);

/* World transform (mat, inv: 16 floats each, row-major) of instance i after update_frame. */
trb_status trb_scene_get_transform(const trb_scene* scene, uint32_t inst, float* mat16, float* inv16);

/* The 16x16 filter table (render_target.rs:50-57). */
trb_status trb_scene_get_filter_table(const trb_scene* scene, float* table256);

/* -- host-only helpers (no device needed; used by the CPU test-suite) ---------------- */

/* BVH::new over `n` boxes (6 floats each: min xyz, max xyz) with the reference's SAH
 * build (bvh.rs:139-267). Pass NULL buffers to query sizes. */
trb_status trb_host_build_bvh(const float* boxes6, uint32_t n, uint32_t max_geom, uint32_t* n_nodes,
                              trb_bvh_node* nodes, uint32_t* ordered);

/* trb_host_build_bvh run on GPU `device`, with the same arguments and statuses and the same output (the same nodes in the
 * same order, the same ordered_geom), bit for bit except that a bound which ties between -0.0 and +0.0 may carry the other
 * zero. Host buffers; NULL nodes / ordered query sizes. n >= 2^31 is TRB_UNSUPPORTED; without a GPU the result is
 * TRB_NO_DEVICE. Boxes on which the reference's build would split a node into an empty child (more than max_geom boxes
 * whose centroids all fall in one bucket, from infinite or NaN coordinates) give TRB_INVALID_ARG. */
trb_status trb_build_bvh(int device, const float* boxes6, uint32_t n, uint32_t max_geom, uint32_t* n_nodes,
                         trb_bvh_node* nodes, uint32_t* ordered);

/* trb_build_bvh with DEVICE buffers on GPU `device` (4-byte aligned): d_nodes has room for 2n - 1 nodes, d_ordered for
 * n words, and the node count is written to the device word d_n_nodes. The work is enqueued on cuda_stream (a
 * cudaStream_t; NULL = default stream), and no other stream is touched. The one exception to asynchrony: the build
 * proceeds level by level over its nodes of more than 1024 boxes and reads the number of such nodes back, so it
 * synchronises cuda_stream once per level (the call returns with the rest of the work enqueued). Scratch memory is
 * allocated and freed stream-ordered on cuda_stream. Null buffers or n == 0: TRB_INVALID_ARG. */
trb_status trb_build_bvh_device(int device, const float* d_boxes6, uint32_t n, uint32_t max_geom, uint32_t* d_n_nodes,
                                trb_bvh_node* d_nodes, uint32_t* d_ordered, void* cuda_stream);

/* Keyframe::transform (keyframe.rs:60-63): T * R * S and its inverse, row-major. */
trb_status trb_host_keyframe_transform(const trb_keyframe* kf, float* mat16, float* inv16);

/* Self-check of the two-level node records the trace kernel walks (csrc/trb_device.h DQuad): for every ray
 * with a finite 1/d, a literal BVH::intersect walk (bvh.rs:81-130) over `nodes` and a walk through the packed
 * records must visit the same leaves in the same order. Host only. */
trb_status trb_host_quad_check(const trb_bvh_node* nodes, uint32_t n_nodes, const trb_ray* rays, uint32_t n_rays,
                               uint32_t* mismatches, uint64_t* leaf_visits, uint64_t* quad_visits);

/* Device self-check of the trace kernel's short box test (csrc/trb_kernels.cuh box_hit_finite, used for rays whose origin,
 * direction and 1/direction are all finite) against the literal transcription of BBox::fast_intersect (bbox.rs:75-104) on
 * n_cases generated boxes and rays built from awkward values (signed zeros, denormals, huge / tiny magnitudes, origins on box
 * planes, flat boxes). out[0] = cases with an all-finite ray, out[1] = hits among them, out[2] = MISMATCHES (must be 0),
 * out[3] = cases that take the literal path. Needs a GPU (TRB_NO_DEVICE otherwise). */
trb_status trb_selftest_box(uint32_t n_cases, uint32_t seed, uint64_t out[4]);

/* AnimatedTransform::transform(time) (animated_transform.rs:40-56) of the transform stack
 * desc->splines[first .. first+count): the same code the device runs per ray for keyframed
 * instances, compiled for the host. AnimatedColor::color(time) (animated_color.rs:52-78) of
 * desc->color_keys[first .. first+count) likewise. */
trb_status trb_host_animated_transform(const trb_scene_desc* desc, uint32_t first, uint32_t count, float time,
                                       float* mat16, float* inv16);
trb_status trb_host_animated_color(const trb_scene_desc* desc, uint32_t first, uint32_t count, float time, float* rgb3);

/* The JSON loader alone (Scene::load_file up to the flattened description): the result is
 * owned by the library; release with trb_desc_free. */
trb_status trb_desc_load_json(const char* path, uint32_t width, uint32_t height, uint32_t spp,
                              trb_scene_desc** out);
void trb_desc_free(trb_scene_desc* desc);

/* Drains the scene's device and reports a latched traversal-stack overflow of passes enqueued with
 * trb_render_device / trb_intersect_device (TRB_CUDA), else TRB_OK. */
trb_status trb_scene_check_error(trb_scene* scene);

/* Launch-shape options of the wavefront pipeline (results never depend on them; DESIGN.md "Launch options"):
 * "pass.paths" camera samples per pass; "trace.pipe" trace-kernel variant (36 = default: 9 CTAs per SM; 0 = the round-1 kernel),
 * "trace.refill", "trace.grid", "trace.sched", "trace.quads", "trace.exact_box" (test: every ray takes the literal box test);
 * "shade.split" -1 per scene / 0 fused / 1 split, "shade.sort" 0/1 material buckets between the split kernels, "shade.kind" 0/1 the
 * matte instantiations of the split kernels, "shade.anim_occupancy" 3/4; "anim.table" 0/1/2, "frame.device" 0/1; "film.v2" 0/1;
 * "sort.mode" 0/1/2 ray-queue sorting, "sort.bits", "sort.min_round". "trace.quads" and "frame.device" re-run update_frame for the
 * current frame (they change what it builds). Defaults can also be preset by TRB_* environment variables, read once by
 * trb_scene_create. */
trb_status trb_scene_set_option(trb_scene* scene, const char* name, long long value);

/* Device time spent in the dominant kernel (k_wf_trace) by launches made with TRB_RENDER_TIME_TRACE since the last
 * call, measured with CUDA events on the launching stream; synchronises those events. */
trb_status trb_scene_trace_time(trb_scene* scene, float* total_ms, uint32_t* n_launches);

/* Number of CUDA kernels this library has launched in this process (monotonic). */
unsigned long long trb_launch_count(void);

const char* trb_last_error(void);
uint32_t trb_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* TRB_H */
