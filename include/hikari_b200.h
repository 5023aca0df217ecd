/* hikari_b200.h — the C ABI of libhikari_b200.so: the drop-in boundary for bevy-hikari's per-frame GPU path.
 *
 * The reference has no FFI; its hot path sits behind three Bevy render-graph nodes that encode wgpu compute
 * dispatches.  Each entry point below replaces one of those Rust call sites (file:line under /root/reference):
 *
 *   hk_context_create / _resize   prepare_light_textures + ReservoirCache        src/light.rs:307-383
 *                                 prepass_textures_system                        src/prepass.rs:285-428
 *                                 prepare_post_process_textures                  src/post_process.rs:635-747
 *   hk_scene_upload               MeshRenderAssets/InstanceRenderAssets/MaterialRenderAssets::write_buffer
 *                                 (the 9 storage buffers of bind group 2)        src/mesh_material/mod.rs:684-808
 *                                 texture array of bind group 3                  src/mesh_material/mod.rs:760-799
 *   hk_set_noise                  NoiseTextures::as_bind_group (bind group 4)    src/lib.rs:518-598
 *   hk_prepass_run                PrepassNode::run                               src/prepass.rs:769-851
 *   hk_light_run                  LightNode::run                                 src/light.rs:590-702
 *   hk_post_process_run           PostProcessNode::run (denoise + tone mapping)  src/post_process.rs:1140-1234
 *   hk_render_frame               the three nodes in graph order                 src/lib.rs:258-365
 *   hk_get_output / hk_readback   the texture views later nodes bind             src/light.rs:297-304,
 *                                                                                src/post_process.rs:622-633
 *
 * Conventions: plain C, plain pointers and sizes, no C++/torch types.  Every function returns HK_OK (0) or a
 * negative HK_ERR_* and never throws or aborts; hk_last_error() gives the message.  Like the reference nodes
 * (src/light.rs:606-617) a frame with missing inputs is skipped, but here that is reported as HK_ERR_NOT_READY
 * instead of silently returning Ok.  One context = one GPU = one CUDA stream = one caller thread at a time.
 * All work is stream-ordered and asynchronous until hk_sync()/hk_readback().  There is no CPU fallback:
 * without a CUDA device hk_context_create fails.
 */
#ifndef HIKARI_B200_H
#define HIKARI_B200_H
#include <stddef.h>
#include <stdint.h>
#include "hk_layout.h"

#ifdef __cplusplus
extern "C" {
#endif

#define HK_OK 0
#define HK_ERR_INVALID_ARGUMENT (-1)
#define HK_ERR_CUDA (-2)
#define HK_ERR_NOT_READY (-3)     /* scene / noise not uploaded yet (reference: node returns Ok(()) and skips) */
#define HK_ERR_OUT_OF_MEMORY (-4)
#define HK_ERR_UNSUPPORTED (-5)

typedef struct hk_context hk_context;

/* One RGBA8 texture of the bindless array (src/mesh_material/material.rs:55-87). */
typedef struct hk_texture_desc {
    const uint8_t* rgba8;      /* width*height*4, row-major, already linearised the way the wgpu format would */
    uint32_t width, height;
    uint32_t address_mode_u;   /* 0 = repeat, 1 = clamp-to-edge, 2 = mirror-repeat */
    uint32_t address_mode_v;
    uint32_t filter_linear;    /* 0 = nearest, 1 = bilinear (mip level 0 only, light.wgsl:756) */
    uint32_t srgb;             /* 1 = decode sRGB -> linear on fetch (Rgba8UnormSrgb) */
} hk_texture_desc;

/* The nine storage buffers of src/shaders/mesh_material_bindings.wgsl:5-22, host pointers, copied before return. */
typedef struct hk_scene_desc {
    const hk_vertex* vertices;           uint32_t vertex_count;
    const hk_primitive* primitives;      uint32_t primitive_count;
    const hk_node* asset_nodes;          uint32_t asset_node_count;      /* Nodes.count (mesh.rs:56) */
    const hk_alias_entry* alias_table;   uint32_t alias_count;
    const hk_instance* instances;        uint32_t instance_count;
    const hk_node* instance_nodes;       uint32_t instance_node_count;   /* Nodes.count (instance.rs:94) */
    const hk_material* materials;        uint32_t material_count;
    const hk_node* emissive_nodes;       uint32_t emissive_node_count;   /* Nodes.count (instance.rs:97) */
    const hk_emissive* emissives;        uint32_t emissive_count;
    const hk_texture_desc* textures;     uint32_t texture_count;         /* 0 => NO_TEXTURE variant (light.rs:141-143) */
    /* PreviousMeshUniform::transform of every instance (instance.rs:111-128, bound as `previous_mesh` in prepass.wgsl:7-8):
     * instance_count column-major mat4 (16 floats each), the model matrix of the previous frame.  NULL = nothing moved.
     * Only feeds the motion vectors of the G-buffer (prepass.wgsl:52,99). */
    const float* previous_instance_models;
} hk_scene_desc;

/* What bind group 0 carries each frame (src/prepass.rs:81-125, src/light.rs:630-639) + the settings that pick passes. */
typedef struct hk_frame_inputs {
    hk_frame_uniform frame;          /* FrameUniform::extract_component, src/view.rs:141-193 */
    hk_view view;
    hk_previous_view previous_view;
    hk_lights lights;
    uint32_t denoise;                /* HikariSettings::denoise (src/lib.rs:428) */
    uint32_t taa_jitter;             /* 1 = TEMPORAL_ANTI_ALIASING jitter in the prepass (prepass.wgsl:52-54) */
    uint32_t smaa_tu4x;              /* 1 = Upscale::SmaaTu4x: SMAA_TU4X jitter index rule (prepass.wgsl:31-35) */
    uint32_t temporal_upscalers;     /* 1 = hk_post_process_run continues past tone mapping with smaa_tu4x + smaa_tu4x_extrapolate
                                        (when smaa_tu4x) and taa_jasmine (when taa_jitter) — post_process.rs:1236-1277, the
                                        "next" rows K11/K12 of SURVEY.md 8(f).  0 = the hot path ends at tone mapping.
                                        Tiles: see hk_context_enable_tile_upscalers. */
    uint32_t fsr1;                   /* 1 = Upscale::Fsr1 (lib.rs:476-483): with temporal_upscalers, hk_post_process_run ends with
                                        FSR 1.0 EASU (render size -> camera target size; input = taa_output when taa_jitter else
                                        the tone-mapped image, post_process.rs:1037-1040) and RCAS (post_process.rs:1279-1308).
                                        Excludes smaa_tu4x.  Full-frame contexts only. */
    float fsr_sharpness;             /* Upscale::sharpness(), lib.rs:507-512: RCAS stops, 0 = sharpest (FsrConstantsUniform) */
} hk_frame_inputs;

/* Identifiers for hk_get_output / hk_readback / hk_upload_state.  Read-back formats are the reference's texture /
 * buffer formats (src/prepass.rs:43-47, src/light.rs:29-31,51-60, src/post_process.rs:29), row-major, tightly packed,
 * rows [row_begin,row_end) of the context's band. */
enum {
    HK_OUT_TONE_MAPPED = 0,      /* Rgba16Float, 8 B/px   post_process.rs:974-981 */
    HK_OUT_RENDER_DIRECT = 1,    /* Rgba16Float           light.rs:372 render[0] */
    HK_OUT_RENDER_EMISSIVE = 2,
    HK_OUT_RENDER_INDIRECT = 3,
    HK_OUT_VARIANCE_DIRECT = 4,  /* R32Float              light.rs:371 variance[0] */
    HK_OUT_VARIANCE_EMISSIVE = 5,
    HK_OUT_VARIANCE_INDIRECT = 6,
    HK_OUT_ALBEDO = 7,           /* Rgba16Float           light.rs:373 */
    HK_OUT_DENOISED_DIRECT = 8,  /* Rgba16Float           post_process.rs:714 denoise_render[0] */
    HK_OUT_DENOISED_EMISSIVE = 9,
    HK_OUT_DENOISED_INDIRECT = 10,
    HK_OUT_UPSCALED = 11,        /* Rgba16Float   post_process.rs:718-724 upscale_output[0]: ceil(size * 2 / ratio) (SMAA TU4x; <= 2x render size) or the camera
                                    target size (Fsr1: the EASU result) */
    HK_OUT_TAA = 12,             /* Rgba16Float, the extent of HK_OUT_UPSCALED with SMAA TU4x else render size   post_process.rs:726-731 taa_output[current] */
    HK_OUT_FSR_SHARPENED = 13,   /* Rgba16Float, camera target size   upscale_output[1]: the RCAS result, what the overlay presents
                                    under Upscale::Fsr1 (overlay.rs:228) */
    HK_OUT_GBUFFER_POSITION = 16,           /* Rgba32Float 16 B/px */
    HK_OUT_GBUFFER_NORMAL = 17,             /* Rgba8Snorm   4 B/px */
    HK_OUT_GBUFFER_DEPTH_GRADIENT = 18,     /* Rg32Float    8 B/px */
    HK_OUT_GBUFFER_INSTANCE_MATERIAL = 19,  /* Rg32Float    8 B/px (id + 0.5) */
    HK_OUT_GBUFFER_VELOCITY_UV = 20,        /* Rgba32Float 16 B/px */
    HK_OUT_RESERVOIR_0 = 32      /* .. HK_OUT_RESERVOIR_0+9 : PackedReservoir 64 B/px, buffer index as in light.rs:518 */
};

/* Per-frame counters and timings (SURVEY.md 8(d): rays = traverse_top calls + stand-alone traverse_bottom calls). */
typedef struct hk_frame_stats {
    uint64_t primary_rays;       /* G-buffer rays (the reference rasterises these) */
    uint64_t tlas_rays;          /* traverse_top calls of the light passes (light.wgsl:442) */
    uint64_t blas_rays;          /* stand-alone traverse_bottom calls (light.wgsl:687) */
    float ms_prepass, ms_light, ms_post_process, ms_total;   /* CUDA-event times of the last frame, if enabled */
    uint32_t kernel_launches;    /* kernels launched by the last hk_render_frame */
    uint32_t timed_frames;       /* hk_set_profiling_kernel mode: frames averaged into ms_kernel[kernel]; 0 otherwise */
    float ms_kernel[16];         /* per-kernel CUDA-event times of the last hk_render_frame, index = HK_K_*; 0 = not run */
    uint32_t wide_traversal;     /* rays that walk the scene's 4-wide trees (HK_TUNE_WIDE_TRAVERSAL): bit 0 = primary rays, bit 1 = light passes */
    uint32_t wide_stack_need;    /* bound on the stack entries a walk of the uploaded scene's trees can need; 0 = no trees */
} hk_frame_stats;

enum {   /* indices into hk_frame_stats.ms_kernel */
    HK_K_GBUFFER = 0,            /* primary rays + albedo (replaces the raster prepass and full_screen_albedo) */
    HK_K_DIRECT = 1,             /* direct_lit, sun */
    HK_K_EMISSIVE = 2,           /* direct_lit, EMISSIVE_LIT */
    HK_K_EMISSIVE_SPATIAL = 3,   /* spatial_reuse, EMISSIVE_LIT */
    HK_K_INDIRECT = 4,           /* indirect_lit_ambient */
    HK_K_INDIRECT_SPATIAL = 5,   /* spatial_reuse */
    HK_K_DEMODULATION = 6,
    HK_K_DENOISE_0 = 7, HK_K_DENOISE_1 = 8, HK_K_DENOISE_2 = 9, HK_K_DENOISE_3 = 10,   /* level 3 includes tone mapping when fused */
    HK_K_TONE_MAPPING = 11,
    HK_K_SMAA_TU4X = 12,         /* smaa_tu4x + smaa_tu4x_extrapolate (only with temporal_upscalers) */
    HK_K_TAA = 13,               /* taa_jasmine (only with temporal_upscalers) */
    HK_K_FSR1 = 14,              /* FSR 1.0 EASU + RCAS (only with temporal_upscalers and fsr1) */
    HK_K_COUNT = 15,
    HK_K_TRACE_RAYS = 15         /* kernel time of the last hk_trace_rays call (always filled) */
};

typedef struct hk_ray {   /* test hook input: a world-space ray exactly as traverse_top takes it */
    float origin[3];    float max_distance;
    float direction[3]; float early_distance;
    uint32_t exclude_instance; uint32_t _pad[3];
} hk_ray;
typedef struct hk_hit {   /* light.wgsl:270-279 */
    float u, v, distance;
    uint32_t instance_index, primitive_index;
} hk_hit;

/* width x height = the camera target (HikariSettings upscale ratio 1: render size == target size).
 * [row_begin,row_end) = the band of rows this context owns (whole frame: 0,height).  The context renders the band
 * plus the ghost rows it needs so that owned rows are bit-identical to an unsharded render (SURVEY.md 8(e)).
 * cuda_stream: a cudaStream_t to run on, or NULL to let the context create its own. */
int hk_context_create(hk_context** out, int cuda_device, uint32_t width, uint32_t height,
                      uint32_t row_begin, uint32_t row_end, void* cuda_stream);
/* Same, for a rectangular tile [col_begin,col_end) x [row_begin,row_end) of the frame (2-D sharding: vertical strips balance
 * sky / ground far better than row bands and 4x2 tiles halve the ghost area at 8 GPUs). */
int hk_context_create_tile(hk_context** out, int cuda_device, uint32_t width, uint32_t height, uint32_t col_begin, uint32_t col_end,
                           uint32_t row_begin, uint32_t row_end, void* cuda_stream);
void hk_context_destroy(hk_context* ctx);
int hk_context_resize(hk_context* ctx, uint32_t width, uint32_t height, uint32_t row_begin, uint32_t row_end);
int hk_context_resize_tile(hk_context* ctx, uint32_t width, uint32_t height, uint32_t col_begin, uint32_t col_end,
                           uint32_t row_begin, uint32_t row_end);
int hk_reset_temporal_state(hk_context* ctx);   /* zero reservoirs, as re-allocation does in light.rs:342-363 */

int hk_scene_upload(hk_context* ctx, const hk_scene_desc* scene);
/* The per-frame part of the scene, for animated instances and materials: replaces instances, instance_nodes (TLAS), emissives,
 * emissive_nodes, alias_table and previous_instance_models — what MeshMaterialRenderAssets / InstanceRenderAssets::set +
 * write_buffer rewrite when an instance event fires (instance.rs:352-437) — and, when `materials` is not NULL, the material
 * records (material.rs:139-203; texture indices keep referring to the uploaded textures).  Meshes, BLAS nodes and textures
 * of the last hk_scene_upload stay in place.  Only those members of `scene` are read. */
int hk_scene_update_instances(hk_context* ctx, const hk_scene_desc* scene);
/* The same per-frame part REBUILT ON THE DEVICE from what actually changed — one model matrix per instance (SURVEY 8(f) rank 2; the
 * reference does this on the CPU whenever anything moves, instance.rs:352-437, and lists asynchronous acceleration-structure builds as
 * to do, README.md:27).  For the instances of the last hk_scene_upload / hk_scene_update_instances, same order, same number:
 *   models            instance_count column-major mat4: GlobalTransform::compute_matrix() (instance.rs:287)
 *   previous_models   PreviousMeshUniform::transform of every instance (instance.rs:111-128), or NULL = the model each instance had
 *                     until this call (then call once per frame while anything moves, and once more after it stopped)
 *   mesh_aabbs        instance_count x {center[3], half_extents[3]}: the bevy `Aabb` of each instance's mesh (instance.rs:293-296)
 * Kernels on the context's stream recompute every instance's world AABB, model / inverse-transpose matrices and traversal record,
 * rebuild the TLAS (bvh 0.7.1's bucketed SAH build + flatten_custom, one warp per tree node), every emissive's bounding sphere and
 * surface area and the emissive BVH: record for record what host/hikari.cpp (= the reference's CPU path) produces
 * (tests/test_gpu_scene_update.py), without a host round trip: the arrays are staged through pinned memory owned by the context and
 * are the caller's again on return.  Unchanged by this call, hence the caller's to watch: the SET of instances / meshes / materials
 * and the alias tables, which the reference rebuilds when an emissive instance's scale moved by more than 0.01 (instance.rs:385-397;
 * hikari::MeshMaterialWorld::prepare_instance_transforms checks both and says when hk_scene_update_instances is needed instead).
 * HK_ERR_UNSUPPORTED if the uploaded TLAS / emissive BVH is not in bvh 0.7.1's layout.  When rays walk the 4-wide trees
 * (HK_TUNE_WIDE_TRAVERSAL in effect for this scene) the 4-wide TLAS is re-derived on the host from the records just built, which
 * costs one small read-back and a stream synchronisation; otherwise the call never waits for the device. */
int hk_scene_update_transforms(hk_context* ctx, const float* models, const float* previous_models, const float* mesh_aabbs,
                               uint32_t instance_count);
/* Test / debugging aid: the per-frame scene buffers as they are on the device, in the layouts of hk_layout.h. */
enum { HK_SCENE_INSTANCES = 0, HK_SCENE_INSTANCE_NODES = 1, HK_SCENE_EMISSIVES = 2, HK_SCENE_EMISSIVE_NODES = 3,
       HK_SCENE_PREVIOUS_MODELS = 4 /* 64 B per instance; empty when nothing moved */, HK_SCENE_INSTANCE_MOVED = 5 /* uint32 per instance */ };
int hk_scene_buffer_bytes(hk_context* ctx, int which, size_t* bytes);
int hk_scene_readback(hk_context* ctx, int which, void* host, size_t bytes);   /* bytes = hk_scene_buffer_bytes */
int hk_set_noise(hk_context* ctx, const uint8_t* rgba8_64x64x16);   /* 16 textures of 64x64 RGBA8, lib.rs:189-219 */

/* The five G-buffer render targets of a host-side raster prepass (src/prepass.rs:285-306; formats src/prepass.rs:43-47), as DEVICE
 * pointers (e.g. the CUDA mapping of the Vulkan images through external memory) with their row pitches, covering the context's owned
 * rectangle, row-major.  hk_import_gbuffer replaces hk_prepass_run for such a host: it swaps current <-> previous like the prepass
 * (prepass.rs:427) and copies the planes device-to-device, stream-ordered; then hk_light_run (which starts with full_screen_albedo,
 * light.rs:645-653) and hk_post_process_run.  ids are stored as id + 0.5 (prepass.wgsl:97); background texels are all zero. */
typedef struct hk_gbuffer_desc {
    const void* position;           size_t position_pitch_bytes;            /* Rgba32Float: world position, w = NDC depth (0 = background) */
    const void* normal;             size_t normal_pitch_bytes;              /* Rgba8Snorm */
    const void* depth_gradient;     size_t depth_gradient_pitch_bytes;      /* Rg32Float */
    const void* instance_material;  size_t instance_material_pitch_bytes;   /* Rg32Float: instance + 0.5, material + 0.5 */
    const void* velocity_uv;        size_t velocity_uv_pitch_bytes;         /* Rgba32Float: velocity.xy, uv */
} hk_gbuffer_desc;
int hk_import_gbuffer(hk_context* ctx, const hk_gbuffer_desc* gbuffer);
int hk_prepass_run(hk_context* ctx, const hk_frame_inputs* in);
int hk_light_run(hk_context* ctx, const hk_frame_inputs* in);
int hk_post_process_run(hk_context* ctx, const hk_frame_inputs* in);
int hk_render_frame(hk_context* ctx, const hk_frame_inputs* in);     /* prepass -> light -> post process */
/* Test hook: ONE pass on whatever the planes hold (hk_upload_state), for per-pass comparison with the oracle from identical inputs.
 * pass: 0 albedo, 1 direct_lit sun, 2 direct_lit emissive, 3 spatial_reuse emissive, 4 indirect_lit_ambient, 5 spatial_reuse indirect,
 * 6 denoise chain (all signals; writes HK_OUT_DENOISED_*), 7 tone mapping. */
int hk_run_pass(hk_context* ctx, const hk_frame_inputs* in, int pass, int arg);

int hk_get_output(hk_context* ctx, int which, void** device_ptr, size_t* bytes);  /* final images only: HK_OUT_TONE_MAPPED (owned
                                                                                     rectangle), HK_OUT_UPSCALED, HK_OUT_TAA */
/* Pixels of the rectangle hk_readback / hk_get_output transfer for `which`, under the settings of the last frame run:
 * deferred-size planes (G-buffer, albedo) = the owned rectangle; render-size planes = ceil(size / upscale_ratio)
 * (light.rs:622-624); HK_OUT_UPSCALED (and HK_OUT_TAA after smaa_tu4x) = ceil(size * (2 / ratio)) as create_texture computes it (post_process.rs:663-667,
 * 711-731): twice the render size except where the two ceilings disagree (ratio 2 on an odd width W: W, not W + 1). */
int hk_output_extent(hk_context* ctx, int which, uint32_t* width, uint32_t* height);
int hk_readback(hk_context* ctx, int which, void* host, size_t bytes);            /* synchronises */
/* Pipelined read-back of a final image (HK_OUT_TONE_MAPPED / HK_OUT_UPSCALED / HK_OUT_TAA / HK_OUT_FSR_SHARPENED) for a presentation loop: the
 * copy into `pinned_host` (page-locked memory) is queued on an internal copy stream behind all work submitted so far and
 * the call returns at once.  The next frame can be submitted immediately — on the device, its first write to a final
 * image waits for the copy.  hk_readback_wait blocks the host until the last queued copy has landed.  One copy may be
 * in flight per context. */
int hk_readback_async(hk_context* ctx, int which, void* pinned_host, size_t bytes);
int hk_readback_wait(hk_context* ctx);
int hk_upload_state(hk_context* ctx, int which, const void* host, size_t bytes);  /* inverse of hk_readback (tests) */
int hk_sync(hk_context* ctx);

/* Exact tiling under camera motion.  A tile's ghost pixels compute their own temporal history, which is exact only while
 * the camera is static.  hk_halo_pull(dst, src), called after both contexts have finished a frame (and before either
 * starts the next), overwrites the reservoirs of `dst`'s ghost pixels that `src` owns with `src`'s values (stream-ordered
 * on `dst`; `src` may be on a peer GPU of the same process).  With every neighbour pulled, the next frame's temporal passes
 * read exactly what an unsharded render would, provided the per-frame reprojection stays within the motion margin:
 * hk_context_set_motion_margin widens the ghost ring from 36 to 36 + `pixels` (re-allocates and clears the tile's state). */
int hk_context_set_motion_margin(hk_context* ctx, uint32_t pixels);
int hk_halo_pull(hk_context* dst, hk_context* src);
/* The temporal upscalers (hk_frame_inputs.temporal_upscalers) on a TILE: allocates the tile's copies of the tone-mapped,
 * upscaled and TAA images over its allocation (re-allocates and clears the tile's state).  Needs upscale_ratio 1, a
 * motion margin of at least 4 pixels + the per-frame motion, and hk_halo_pull from every neighbour after each frame (it
 * also carries the tone-mapped and TAA history of the ghost ring).  HK_OUT_UPSCALED / HK_OUT_TAA then serve the owned part. */
int hk_context_enable_tile_upscalers(hk_context* ctx, int enabled);
/* The same between processes (one process per GPU): the owner exports a descriptor — CUDA IPC handles of its forty
 * reservoir quarter-planes (and, with tile upscalers, its four history images) and its tile rectangles — which travels to the neighbour by any channel; the neighbour imports it
 * once (maps the planes; peer access over NVLink) and pulls after every frame.  Re-export after hk_context_resize* or
 * hk_context_set_motion_margin (the planes are re-allocated).  Imported peers are released with the importing context. */
typedef struct hk_halo_descriptor {
    uint8_t plane_handles[44][64];   /* reservoir r, quarter q at [4 * r + q]; [40..41] tone-mapped ring, [42..43] TAA history (tile upscalers) */
    int32_t has_images;              /* 1 = entries 40..43 are valid (hk_context_enable_tile_upscalers on the exporter) */
    int32_t frame[2];                /* width, height */
    int32_t allocated[4];            /* col_begin, col_end, row_begin, row_end of the allocation (owned + ghosts) */
    int32_t owned[4];
} hk_halo_descriptor;
typedef struct hk_halo_peer hk_halo_peer;
int hk_halo_export(hk_context* ctx, hk_halo_descriptor* out);
int hk_halo_import(hk_context* ctx, const hk_halo_descriptor* remote, hk_halo_peer** out);
int hk_halo_pull_peer(hk_context* ctx, hk_halo_peer* peer);

/* Frame assembly for tiled (multi-GPU) rendering.  With a frame target set, every owned pixel of the tone-mapped image is
 * also stored into the full-frame Rgba16Float buffer `frame` (pitch in pixels) at its position in the frame, by the last
 * kernel of hk_render_frame / hk_post_process_run itself.  `frame` may live on another GPU — same process (peer access is
 * enabled on demand) or another process (hk_frame_open of a handle from hk_frame_alloc; CUDA IPC) — so that the store
 * over NVLink is the transfer and no gather pass or collective touches the pixels.  The caller orders "all tiles have
 * landed" (an event, or a barrier across ranks) before consuming the frame.  NULL clears the target.  upscale_ratio 1 only. */
int hk_set_frame_target(hk_context* ctx, void* frame_device_ptr, uint32_t pitch_pixels);
int hk_frame_alloc(hk_context* ctx, void** device_ptr, uint8_t ipc_handle[64]);        /* width x height x 8 B, zeroed; freed with the context */
int hk_frame_open(hk_context* ctx, const uint8_t ipc_handle[64], void** device_ptr);   /* map a frame of another process; closed with the context */
int hk_frame_read(hk_context* ctx, const void* frame_device_ptr, void* host, size_t bytes);   /* synchronous D2H of an assembled frame */

int hk_trace_rays(hk_context* ctx, const hk_ray* rays, size_t n, hk_hit* hits);   /* F3/F4 parity hook */
int hk_set_profiling(hk_context* ctx, int count_rays, int time_passes);
/* Low-overhead timing of ONE kernel (HK_K_* index): only its launch is bracketed with CUDA events (2 records per frame), kept in
 * a ring of 256 frames; hk_get_stats then reports the MEAN duration over the frames rendered since this call in ms_kernel[kernel]
 * (timed_frames = how many).  bench.py uses it to measure the dominant kernel live inside the timed region without the ~30 event
 * records of full pass timing.  kernel < 0 restores per-pass timing as selected by hk_set_profiling. */
int hk_set_profiling_kernel(hk_context* ctx, int kernel);
/* Implementation choices.  Keys 1-3 do not change a single output value (both forms are held to the same parity suite); key 4 is
 * the image-exact traversal mode, which keeps every image but not every record (below).
 * HK_TUNE_POOLED_INDIRECT: 1 = the indirect pass runs as kc_indirect (per-CTA shared-memory ray pool, dynamic fetch, TMA-staged scene
 * records, kernels_pool.cu), 0 = per pixel, k_indirect_path + k_indirect_restir (default, DESIGN.md 4).
 * HK_TUNE_TILED_SPATIAL: 1 (default) = spatial_reuse runs as kc_spatial (neighbourhood depth + reservoir-quarter tiles staged in shared
 * memory by TMA, kernels_spatial.cu) whenever the upscale ratio is 1, 0 = as k_spatial (gathers from global memory).
 * HK_TUNE_TILED_DENOISE: 1 (default) = the a-trous levels run as kc_denoise (the nine taps' planes staged by TMA, kernels_post.cu) at
 * upscale ratio 1, 0 = as k_denoise.
 * HK_TUNE_WIDE_TRAVERSAL: which rays walk 4-wide trees derived at hk_scene_upload / hk_scene_update_instances from the uploaded flat
 * BVHs (instance.rs:352-437, mod.rs:185-201) front to back with a short stack (csrc/hk_wide.cuh) instead of the flat arrays in the
 * reference's fixed order (light.wgsl:400-486): 0 = none, 1 = the primary rays of the prepass when the scene's trees have at least 256
 * nodes (default in libhikari_b200.so, the tolerance build: the ordered walk is meant for these coherent rays, not for the incoherent
 * rays of the light passes), 3 = every ray of the prepass and the light passes, whatever the
 * scene's size (A/B runs and the mode's tests).  Box and triangle tests, their arithmetic and the tie rule (first in array order
 * among equidistant hits) are the reference's, so G-buffer ids, hit distances and every image are the exact walk's except for rays
 * whose two nearest hits tie within the rounding of a box test; under 3 the any-hit OCCLUDER a shadow ray reports (stored with
 * zero-radiance samples, read by no image) depends on the order and differs.  Default 0 in libhikari_b200_exact.so.  A scene whose
 * flat arrays are not bvh 0.7.1's flatten_custom layout, or whose trees could overflow the walk's stack, silently keeps the
 * reference's walk (hk_frame_stats.wide_traversal: bit 0 = primary rays, bit 1 = light passes). */
enum { HK_TUNE_POOLED_INDIRECT = 1, HK_TUNE_TILED_SPATIAL = 2, HK_TUNE_TILED_DENOISE = 3, HK_TUNE_WIDE_TRAVERSAL = 4 };
int hk_set_tuning(hk_context* ctx, int key, int value);
int hk_set_keep_intermediates(hk_context* ctx, int keep);   /* 1: hk_render_frame also writes HK_OUT_DENOISED_* */
int hk_get_stats(hk_context* ctx, hk_frame_stats* out);
int hk_band_rows(hk_context* ctx, uint32_t* alloc_row_begin, uint32_t* alloc_row_end); /* owned rows +- ghost rows */
int hk_tile_rect(hk_context* ctx, uint32_t allocated[4], uint32_t owned[4]);            /* x0, x1, y0, y1 of each */

const char* hk_last_error(hk_context* ctx);    /* ctx may be NULL: error of the last failed hk_context_create */
const char* hk_version(void);

#ifdef __cplusplus
}
#endif
#endif
