// context.cu — implementation of the C ABI in include/hikari_b200.h: device memory ownership, scene upload, pass
// scheduling on one CUDA stream (what LightNode::run / PostProcessNode::run do with a wgpu command encoder,
// src/light.rs:590-702, src/post_process.rs:1140-1234), read-back / state upload for tests.
#include <cuda_runtime.h>
#ifndef HK_EMU
#include <cuda.h>            // CUtensorMap + the enums of cuTensorMapEncodeTiled (types only: the entry point is looked up at run time)
#endif
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <set>
#include <string>
#include <unordered_set>
#include <vector>

#include "hikari_b200.h"
#include "hk_kernels.h"
#include "wide_build.h"

#ifndef HK_POOLED_INDIRECT
#define HK_POOLED_INDIRECT 0     // default of hk_set_tuning(HK_TUNE_POOLED_INDIRECT): 0 = per-pixel k_indirect_path + k_indirect_restir, 1 = kc_indirect (ray pool).
#endif                            // Same values either way; the per-pixel form is the default.

#ifndef HK_WIDE_TRAVERSAL_DEFAULT
#define HK_WIDE_TRAVERSAL_DEFAULT 1   // default of hk_set_tuning(HK_TUNE_WIDE_TRAVERSAL) in the tolerance build (libhikari_b200.so): 1 = primary rays; the exact
#endif                                // flavour (and the kernel-logic emulation) default to the reference's walk whatever this says
int hk_tolerance_build();             // kernels_post.cu: 1 when that unit was compiled with the tolerance flags (build.py FAST_FLAGS)

using namespace hkd;

// Rows a band needs beyond the rows it owns so that owned pixels equal an unsharded render (SURVEY.md 8(e)):
// a-trous reach 8+4+2+1 = 15 (+1 for the 3x3 variance blur), spatial reuse radius 20 on top of that.
static const int GHOST_DEMOD = 15, GHOST_L0 = 7, GHOST_L1 = 3, GHOST_L2 = 1;
static const int GHOST_SPATIAL = GHOST_DEMOD + 1;           // 16
static const int GHOST_TEMPORAL = GHOST_SPATIAL + 20;       // 36
// Temporal upscalers on a tile: taa_jasmine reads the upscaled image 1 output texel around a pixel, smaa_tu4x_extrapolate the
// diagonal texels of the neighbouring render pixels, smaa_tu4x the current tone-mapped image up to 2 render pixels away:
// smaa runs on owned + 2, extrapolate on owned + 1, and the tone-mapped image (with everything upstream) on owned + 4.
static const int RING_SMAA = 2, RING_EXTRAPOLATE = 1, RING_TONE = 4;

struct hk_halo_peer {   // a neighbour tile of another process, mapped through CUDA IPC (hk_halo_import)
    Planes planes;       // only reservoir[] (and tone_ring_db[] / taa_output[] when exported) are filled
    Band band;
    void* mapped[44];
};

// The scene a context renders: meshes, BLAS nodes, materials, textures, the per-frame instance half, the 4-wide trees and the host
// copies that validate later updates.  The reference keeps one such set for the whole render world (MeshMaterialBindGroup,
// mesh_material/mod.rs:677-681) and every camera's LightNode binds it (light.rs:641-642); here several contexts attach to one scene
// (hk_shared_scene_create), or hk_scene_upload gives a context a private one on the context's own stream.
struct hk_shared_scene {
    int device = 0;
    cudaStream_t stream = nullptr;         // uploads and updates run here
    bool own_stream = false;
    bool handle = true;                    // the creator's hk_shared_scene handle is alive (a private scene has none)
    hk_context* owner = nullptr;           // private scene: the one context whose hk_scene_upload / hk_scene_update_* write it
    std::vector<hk_context*> attached;     // the scene is freed when the handle is gone and the last context detached
    uint64_t version = 0;                  // bumped by every upload / update
    cudaEvent_t ev_ready = nullptr;        // recorded after an update when an attached context runs on another stream
    std::vector<void*> scene_allocations;  // scene buffers: meshes, BLAS nodes, materials, textures
    struct DevBuf { void* p = nullptr; size_t cap = 0; } ibuf[20];  // scene buffers rewritten by hk_scene_update_instances (grow-only);
                                                                    // 14-19: staging + scratch of hk_scene_update_transforms
                                                                    // (15: DeviceScene::wide_state, 16: kc_build_wide_tlas's scratch)
    // hk_scene_update_transforms: what the last full upload fixed, and pinned staging (two slots, so that the host never waits for
    // the copy of the previous call unless it is two calls behind)
    uint32_t scene_instance_count = 0, scene_emissive_count = 0;
    std::vector<uint32_t> wide_mesh_of;                     // per instance: index into wide_meshes
    struct PinBuf { void* p = nullptr; size_t cap = 0; cudaEvent_t ev = nullptr; bool used = false; } pin[2];
    int pin_slot = 0;
    // image-exact traversal mode (hk_wide.cuh): 4-wide trees of the meshes the instances use, rebuilt only when that set changes
    struct WideMesh { uint32_t base = 0, root = 0xFFFFFFFFu, need = 0; bool ok = false; };
    std::vector<std::array<uint32_t, 3>> wide_mesh_keys;    // (node_offset, node_count, primitive) in first-use order
    std::vector<WideMesh> wide_meshes;                      // parallel to wide_mesh_keys
    uint32_t wide_blas_node_count = 0;
    uint32_t wide_tlas_node_count = 0;     // of the last host derivation (upload / instance update): wide_primary's size rule
    uint32_t wide_stack_need = 0;          // of the last host derivation
    bool wide_blas_ok = false;             // every instance's mesh has a 4-wide tree ...
    uint32_t wide_blas_need = 0;           // ... and the deepest of them needs this much stack
    bool wide_on_device = false;           // the 4-wide TLAS was last derived on the device: its verdict is in ibuf[15] only
    bool mesh_boxes_match = false;         // BLAS half of DeviceScene::leaf_boxes_match
    uint32_t scene_material_count = 0, scene_asset_node_count = 0, scene_primitive_count = 0, scene_vertex_count = 0, scene_texture_count = 0;
    std::vector<hk_node> host_asset_nodes;                 // copy of the uploaded BLAS records: index validation of later instance updates
    std::vector<uint32_t> host_primitive_vertex_index;     // 3 per primitive (hk_primitive_vertex::index), same purpose
    std::vector<float> host_primitive_box;                 // 6 per primitive (min xyz, max xyz): what a BLAS leaf's navigator must enclose
    std::set<std::array<uint32_t, 4>> mesh_range_checked;   // hk_mesh_index values whose leaves have been validated
    // the vertex, primitive and BLAS buffers as hk_scene_add_meshes grows them: those of the upload (scene_allocations, freed with
    // them), then stream-ordered allocations of the scene's stream (`async`), replaced in stream order when they grow again.  The
    // BLAS records past host_asset_nodes were built on the device and have no host copy (nor a 4-wide tree).
    struct MeshBuf { void* p = nullptr; size_t cap = 0; bool async = false; } mbuf[3];
    DeviceScene scene{};
    bool ready = false;
    std::string error;
};

struct hk_context {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    Band band{};
    size_t band_pixels = 0, owned_pixels = 0;
    std::vector<void*> allocations;        // per-pixel planes
    // the scene this context renders (hk_context_attach_scene, or the private one of hk_scene_upload); stream ordering against it
    // only when it runs on another stream: the version of it this stream has waited for, and "the last frame is done reading it"
    hk_shared_scene* sc = nullptr;
    uint64_t scene_seen = 0;
    cudaEvent_t ev_released = nullptr;
    bool released_recorded = false;
    Planes planes{};
    // the light node's indirect pipeline runs on its own stream beside the sun and emissive ones (run_light), forked from and
    // joined back into `stream` within the node, so every other ordering rule of the context only ever sees `stream`;
    // it has its own scatter scratch, the other two share planes.scatter_*
    cudaStream_t indirect_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    uint32_t* indirect_scatter_key = nullptr;
    ReservoirPlanes indirect_scatter_value{};
    bool noise_ready = false;
    bool planes_ready = false;         // allocate_planes completed: every pointer of `planes` is valid
    // TMA descriptors of kc_spatial's tiles (hk_tile.cuh): [0] indirect (radius 20, box 56), [1] emissive (radius 10, box 36);
    // q3 maps per buffer parity: the temporal reservoir the spatial pass reuses is reservoir[base + 1 - (frame.number & 1)]
    TileMap tm_depth[2], tm_q3[2][2];
    TileMap tm_denoise[4][5];          // kc_denoise, per level: tap geometry, instance, the level's three signal planes (box = 16 + 2 x apron)
    bool tile_maps_ready = false;
    bool full_frame = true;            // the context owns the whole frame (no tile): upscale_ratio > 1 and the upscalers need it
    int last_up_w = 0, last_up_h = 0;   // Band::OW / OH of the last frame
    bool last_scaled = false;           // the last frame ran at upscale_ratio != 1: render-size planes are tight RW x RH (even where RW x RH == W x H:
                                        // ceil(3 / 1.25) = 3), not strided like the deferred-size planes
    int last_render_w = 0, last_render_h = 0; bool last_smaa = false, last_upscalers = false, last_fsr = false; uint32_t last_number = 0;   // of the last frame, for read-back sizes
    int gbuffer_current = 0;           // index of the "current" position / velocity_uv planes; toggled by every prepass
    uint8_t* noise = nullptr;
    Counters* counters = nullptr;
    SpatialTable* spatial_tables = nullptr;
    SpatialTable spatial_tables_host[2];  // the same two tables on the host: kc_spatial takes its table as a kernel parameter
    bool count_rays = false, time_passes = false, keep_intermediates = false;
    bool pooled_indirect = HK_POOLED_INDIRECT != 0;   // hk_set_tuning(HK_TUNE_POOLED_INDIRECT)
    bool tiled_denoise = true;                        // hk_set_tuning(HK_TUNE_TILED_DENOISE): kc_denoise (TMA tiles) vs k_denoise (gathers)
    bool tiled_spatial = true;                        // hk_set_tuning(HK_TUNE_TILED_SPATIAL): kc_spatial (TMA tiles) vs k_spatial (gathers)
    int wide_traversal = 0;                           // hk_set_tuning(HK_TUNE_WIDE_TRAVERSAL): 0 = the reference's fixed-order walk, 1 = primary rays
                                                      // walk the 4-wide trees (scenes deep enough to gain), 3 = every ray does
    // pipelined read-back (hk_readback_async): copy stream + "frame submitted" / "copy landed" events
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_submitted = nullptr, ev_copied = nullptr;
    bool copy_in_flight = false;      // a copy has been queued and the compute stream has not yet been ordered behind it
    bool copy_unwaited = false;       // ... and the host has not waited for it
    uint2* frame_target = nullptr; uint32_t frame_pitch = 0;   // hk_set_frame_target
    bool tile_upscalers = false;      // tile context with planes for the temporal upscalers (hk_context_enable_tile_upscalers)
    int motion_margin = 0;            // extra ghost pixels for exact tiling under camera motion (hk_context_set_motion_margin)
    std::vector<void*> frames_owned, frames_opened;            // hk_frame_alloc / hk_frame_open
    std::vector<hk_halo_peer*> halo_peers;                     // hk_halo_import
    float trace_ms = 0.0f;            // kernel time of the last hk_trace_rays (ms_kernel[HK_K_TRACE_RAYS])
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t kev[HK_K_COUNT][2] = {};   // per-kernel begin/end
    // hk_set_profiling_kernel: only ONE kernel is bracketed with events (2 records per frame instead of 28 + 4), into a ring, so
    // that a timed region can carry the dominant kernel's live duration without synchronising per frame or perturbing the frame
    int time_only = -1;                    // -1 = every kernel (time_passes), else the HK_K_* index
    static const int RING = 256;
    cudaEvent_t ring[RING][2] = {};
    uint32_t ring_frames = 0;              // frames recorded since hk_set_profiling_kernel
    bool ring_hit = false;                 // the selected kernel ran in the current frame
    bool kran[HK_K_COUNT] = {};
    hk_frame_stats stats{};
    uint32_t launches = 0;
    std::string error;
};

static std::string g_create_error;

static int set_error(hk_context* c, int code, const std::string& msg) {
    if (c) c->error = msg; else g_create_error = msg;
    return code;
}
static int set_error(hk_shared_scene* s, int code, const std::string& msg) {
    if (s) s->error = msg; else g_create_error = msg;
    return code;
}
static int set_error(std::nullptr_t, int code, const std::string& msg) {   // a failed create: hk_last_error(NULL)
    g_create_error = msg;
    return code;
}
#define HK_CUDA_ON(obj, call)                                                                              \
    do {                                                                                                   \
        cudaError_t e__ = (call);                                                                          \
        if (e__ != cudaSuccess)                                                                            \
            return set_error(obj, e__ == cudaErrorMemoryAllocation ? HK_ERR_OUT_OF_MEMORY : HK_ERR_CUDA,   \
                             std::string(#call) + ": " + cudaGetErrorString(e__));                         \
    } while (0)
#define HK_CUDA(call) HK_CUDA_ON(ctx, call)     // in functions of a context
#define HK_SCUDA(call) HK_CUDA_ON(sc, call)     // in functions of a scene

template <class T>
static cudaError_t alloc_plane(hk_context* ctx, T** out, size_t count, std::vector<void*>& list) {
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, count * sizeof(T) + 16);
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(p, 0, count * sizeof(T), ctx->stream);
    list.push_back(p);
    *out = reinterpret_cast<T*>(p);
    return e;
}

static void free_list(std::vector<void*>& list) {
    for (void* p : list) cudaFree(p);
    list.clear();
}

// ------------------------------------------------------------------------------------------------ scene ownership + ordering
// A scene and the contexts attached to it may run on different streams.  Then every scene update first makes the scene's stream
// wait for each such context's "released" event (recorded after the last launch of a frame entry point that reads the scene),
// rewrites its buffers, records "ready" and bumps the version; a context's stream waits for "ready" before its first launch that
// reads a new version.  When a context runs on the scene's own stream — always the case for a private scene — stream order already
// says all of this and no event is recorded or waited for.
static bool scene_cross(const hk_shared_scene* sc) {      // some attached context runs on another stream
    for (const hk_context* c : sc->attached)
        if (c->stream != sc->stream) return true;
    return false;
}
static void scene_begin_write(hk_shared_scene* sc) {
    for (hk_context* c : sc->attached)
        if (c->stream != sc->stream && c->released_recorded) cudaStreamWaitEvent(sc->stream, c->ev_released, 0);
}
static void scene_end_write(hk_shared_scene* sc) {
    sc->version += 1;
    if (scene_cross(sc) && (sc->ev_ready || cudaEventCreateWithFlags(&sc->ev_ready, cudaEventDisableTiming) == cudaSuccess))
        cudaEventRecord(sc->ev_ready, sc->stream);
}
// before a scene buffer is freed: the released events the scene's stream waits for have completed (grow-only re-allocations and
// full re-uploads are rare; on the scene's own stream cudaFree is ordered as it always was)
static void scene_before_free(hk_shared_scene* sc) {
    if (scene_cross(sc)) cudaStreamSynchronize(sc->stream);
}
// stream-ordered allocations on the scene's stream: hk_scene_add_meshes returns without waiting for the device, and a buffer it
// replaces is released only after the frames in flight that read it (the emulation of tests/emu runs every launch synchronously)
static cudaError_t malloc_on_stream(void** p, size_t bytes, cudaStream_t st) {
#ifdef HK_EMU
    (void)st;
    return cudaMalloc(p, bytes);
#else
    return cudaMallocAsync(p, bytes, st);
#endif
}
static void free_on_stream(void* p, cudaStream_t st) {
#ifdef HK_EMU
    (void)st;
    cudaFree(p);
#else
    cudaFreeAsync(p, st);
#endif
}
static void free_mesh_bufs(hk_shared_scene* sc) {      // (after the scene's stream is idle)
    for (auto& b : sc->mbuf) {
        if (b.async && b.p) cudaFree(b.p);
        b = hk_shared_scene::MeshBuf();
    }
}
static void scene_free(hk_shared_scene* sc) {
    cudaSetDevice(sc->device);
    if (sc->stream) cudaStreamSynchronize(sc->stream);
    free_list(sc->scene_allocations);
    free_mesh_bufs(sc);
    for (auto& b : sc->ibuf) { if (b.p) cudaFree(b.p); b.p = nullptr; b.cap = 0; }
    for (auto& b : sc->pin) { if (b.p) cudaFreeHost(b.p); if (b.ev) cudaEventDestroy(b.ev); b = hk_shared_scene::PinBuf(); }
    if (sc->ev_ready) cudaEventDestroy(sc->ev_ready);
    if (sc->own_stream && sc->stream) cudaStreamDestroy(sc->stream);
    delete sc;
}
static int attach_scene(hk_context* ctx, hk_shared_scene* sc) {
    if (sc->stream != ctx->stream) {      // frames of this context wait for whatever the scene's stream has queued so far
        if (!ctx->ev_released) HK_CUDA(cudaEventCreateWithFlags(&ctx->ev_released, cudaEventDisableTiming));
        if (!sc->ev_ready) HK_CUDA(cudaEventCreateWithFlags(&sc->ev_ready, cudaEventDisableTiming));
        HK_CUDA(cudaEventRecord(sc->ev_ready, sc->stream));
        HK_CUDA(cudaStreamWaitEvent(ctx->stream, sc->ev_ready, 0));
    }
    sc->attached.push_back(ctx);
    ctx->sc = sc;
    ctx->scene_seen = sc->version;
    ctx->released_recorded = false;
    return HK_OK;
}
static void detach_scene(hk_context* ctx) {
    hk_shared_scene* sc = ctx->sc;
    if (!sc) return;
    if (sc->stream != ctx->stream && ctx->released_recorded) cudaStreamWaitEvent(sc->stream, ctx->ev_released, 0);
    sc->attached.erase(std::remove(sc->attached.begin(), sc->attached.end(), ctx), sc->attached.end());
    if (sc->owner == ctx) sc->owner = nullptr;
    ctx->sc = nullptr;
    ctx->released_recorded = false;
    if (!sc->handle && sc->attached.empty()) scene_free(sc);
}
static bool scene_ready(const hk_context* ctx) { return ctx->sc && ctx->sc->ready; }
// Brackets the launches of a frame entry point that read the scene: waits for a new version first, records "released" at the end.
struct SceneUse {
    hk_context* c;
    explicit SceneUse(hk_context* ctx) : c(ctx) {
        hk_shared_scene* sc = c->sc;
        if (sc->stream != c->stream && c->scene_seen != sc->version) {
            if (sc->ev_ready) cudaStreamWaitEvent(c->stream, sc->ev_ready, 0);
            c->scene_seen = sc->version;
        }
    }
    ~SceneUse() {
        if (c->sc->stream == c->stream) return;
        cudaEventRecord(c->ev_released, c->stream);
        c->released_recorded = true;
    }
};

// One TMA descriptor: a 2-D tensor of `width` x `height` elements of `elem_bytes` (row pitch `pitch_bytes`) read in boxes of
// box_w x box_h elements, no swizzle, zero fill outside.  Encoded by the driver (cuTensorMapEncodeTiled, looked up through the
// runtime so that the library does not link libcuda); the kernel-logic emulation keeps a plain description in the same bytes.
static bool make_tile_map(TileMap* out, void* base, uint32_t elem_bytes, uint64_t width, uint64_t height, uint64_t pitch_bytes, uint32_t box_w, uint32_t box_h) {
    memset(out, 0, sizeof(*out));
#ifdef HK_EMU
    TileMapEmu m{static_cast<const unsigned char*>(base), elem_bytes, (uint32_t)width, (uint32_t)height, (uint32_t)pitch_bytes, box_w, box_h};
    static_assert(sizeof(TileMapEmu) <= sizeof(TileMap), "emulated descriptor fits");
    memcpy(out->bytes, &m, sizeof(m));
    return true;
#else
    typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeTiled encode = nullptr;
    static bool looked_up = false;
    if (!looked_up) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            encode = reinterpret_cast<EncodeTiled>(fn);
        cudaGetLastError();
        looked_up = true;
    }
    if (!encode) return false;
    static_assert(sizeof(CUtensorMap) == sizeof(TileMap), "CUtensorMap is 128 bytes");
    const cuuint64_t dims[2] = {width, height};
    const cuuint64_t strides[1] = {pitch_bytes};
    const cuuint32_t box[2] = {box_w, box_h};
    const cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType dt = elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8;
    return encode(reinterpret_cast<CUtensorMap*>(out), dt, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
#endif
}
static bool make_spatial_tile_maps(hk_context* ctx) {
    const Band& b = ctx->band;
    const uint64_t rows = (uint64_t)(b.a1 - b.a0), pitch = (uint64_t)b.AW;
    bool ok = true;
    for (int v = 0; v < 2 && ok; ++v) {
        const uint32_t bh = 16u + 2u * (v ? 10u : 20u), bw = (uint32_t)tile_box_width((int)bh);      // kernels_spatial.cu SpatialTile
        ok = make_tile_map(&ctx->tm_depth[v], ctx->planes.depth, 4, pitch, rows, pitch * 4, bw, bh);
        for (int parity = 0; parity < 2 && ok; ++parity)      // quarter 3 as rows of u32, 4 per pixel
            ok = make_tile_map(&ctx->tm_q3[v][parity], ctx->planes.reservoir[(v ? 2 : 6) + parity].q[3], 4, pitch * 4, rows, pitch * 16, bw * 4, bh);
    }
    for (int level = 0; level < 4 && ok; ++level) {          // kernels_post.cu DenoiseTile<LEVEL>
        const uint32_t step = 8u >> level, bh = 16u + 2u * step, bw = (uint32_t)tile_box_width((int)bh);
        ok = make_tile_map(&ctx->tm_denoise[level][0], ctx->planes.dn_geometry, 4, pitch * 4, rows, pitch * 16, bw * 4, bh) &&
             make_tile_map(&ctx->tm_denoise[level][1], ctx->planes.dn_instance, 4, pitch, rows, pitch * 4, bw, bh);
        for (int sgl = 0; sgl < 3 && ok; ++sgl)
            ok = make_tile_map(&ctx->tm_denoise[level][2 + sgl], ctx->planes.dn_internal[level][sgl], 4, pitch * 2, rows, pitch * 8, bw * 2, bh);
    }
    return ok;
}

static int allocate_planes(hk_context* ctx, uint32_t width, uint32_t height, uint32_t col_begin, uint32_t col_end,
                           uint32_t row_begin, uint32_t row_end) {
    if (width == 0 || height == 0 || row_begin >= row_end || row_end > height || col_begin >= col_end || col_end > width)
        return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "bad size or tile rectangle");
    // Everything derived from the old planes dies with them: the read-back geometry of the last frame, the frame target
    // (validated against the old width) and the "planes are usable" flag, which only a complete allocation sets again —
    // a cudaMalloc failing half-way leaves the context refusing to render instead of holding dangling pointers.
    ctx->planes_ready = false;
    ctx->last_render_w = ctx->last_render_h = 0; ctx->last_up_w = ctx->last_up_h = 0; ctx->last_number = 0; ctx->last_scaled = false;
    ctx->last_smaa = ctx->last_upscalers = ctx->last_fsr = false;
    ctx->frame_target = nullptr; ctx->frame_pitch = 0;
    free_list(ctx->allocations);
    ctx->planes = Planes{};
    Band b;
    b.W = (int)width; b.H = (int)height; b.r0 = (int)row_begin; b.r1 = (int)row_end; b.cx0 = (int)col_begin; b.cx1 = (int)col_end;
    const int ghost = GHOST_TEMPORAL + ctx->motion_margin;
    b.a0 = b.r0 - ghost < 0 ? 0 : b.r0 - ghost;
    b.a1 = b.r1 + ghost > b.H ? b.H : b.r1 + ghost;
    b.ax0 = b.cx0 - ghost < 0 ? 0 : b.cx0 - ghost;
    b.ax1 = b.cx1 + ghost > b.W ? b.W : b.cx1 + ghost;
    b.AW = hk_plane_pitch(b.ax1 - b.ax0);
    b.RW = b.W; b.RH = b.H; b.RS = b.AW; b.OW = 2 * b.W; b.OH = 2 * b.H;
    ctx->band = b;
    const size_t n = (size_t)b.AW * (size_t)(b.a1 - b.a0);
    ctx->band_pixels = n;
    ctx->owned_pixels = (size_t)(b.cx1 - b.cx0) * (size_t)(b.r1 - b.r0);
    Planes& p = ctx->planes;
    auto& L = ctx->allocations;
    ctx->full_frame = (b.cx0 == 0 && b.cx1 == b.W && b.r0 == 0 && b.r1 == b.H);
    ctx->gbuffer_current = 0;
    HK_CUDA(alloc_plane(ctx, &p.pos_depth_db[0], n, L));
    HK_CUDA(alloc_plane(ctx, &p.pos_depth_db[1], n, L));
    HK_CUDA(alloc_plane(ctx, &p.velocity_uv_db[0], n, L));
    HK_CUDA(alloc_plane(ctx, &p.velocity_uv_db[1], n, L));
    p.pos_depth = p.pos_depth_db[0];
    p.velocity_uv = p.velocity_uv_db[0];
    HK_CUDA(alloc_plane(ctx, &p.depth, n, L));
    HK_CUDA(alloc_plane(ctx, &p.normal, n, L));
    HK_CUDA(alloc_plane(ctx, &p.depth_gradient, n, L));
    HK_CUDA(alloc_plane(ctx, &p.instance_material, n, L));
    HK_CUDA(alloc_plane(ctx, &p.albedo, n, L));
    HK_CUDA(alloc_plane(ctx, &p.dn_geometry, n, L));
    HK_CUDA(alloc_plane(ctx, &p.dn_instance, n, L));
    for (int i = 0; i < 3; ++i) {
        HK_CUDA(alloc_plane(ctx, &p.render[i], n, L));
        HK_CUDA(alloc_plane(ctx, &p.variance[i], n, L));
        HK_CUDA(alloc_plane(ctx, &p.dn_variance[i], n, L));
        HK_CUDA(alloc_plane(ctx, &p.dn_render[i], n, L));
        for (int l = 0; l < 4; ++l) HK_CUDA(alloc_plane(ctx, &p.dn_internal[l][i], n, L));
    }
    for (int r = 0; r < 10; ++r)
        for (int q = 0; q < 4; ++q) HK_CUDA(alloc_plane(ctx, &p.reservoir[r].q[q], n, L));
    HK_CUDA(alloc_plane(ctx, &p.scatter_key, n, L));   // zero = no claim; k_scatter_resolve re-zeroes what it consumes
    for (int q = 0; q < 4; ++q) HK_CUDA(alloc_plane(ctx, &p.scatter_value.q[q], n, L));
    ctx->indirect_scatter_key = nullptr; ctx->indirect_scatter_value = ReservoirPlanes{};
    HK_CUDA(alloc_plane(ctx, &ctx->indirect_scatter_key, n, L));
    for (int q = 0; q < 4; ++q) HK_CUDA(alloc_plane(ctx, &ctx->indirect_scatter_value.q[q], n, L));
    HK_CUDA(alloc_plane(ctx, &p.tone_mapped_db[0], ctx->owned_pixels, L));
    HK_CUDA(alloc_plane(ctx, &p.tone_mapped_db[1], ctx->owned_pixels, L));
    p.tone_mapped = p.tone_mapped_db[0];
    p.upscale_output = nullptr; p.upscale_sharpen_output = nullptr; p.taa_output[0] = p.taa_output[1] = nullptr;
    p.tone_ring_db[0] = p.tone_ring_db[1] = nullptr;
    if (!ctx->full_frame && ctx->tile_upscalers) {   // every image over the allocation (owned + ring + halo)
        HK_CUDA(alloc_plane(ctx, &p.tone_ring_db[0], n, L));
        HK_CUDA(alloc_plane(ctx, &p.tone_ring_db[1], n, L));
    }
    if (ctx->full_frame || ctx->tile_upscalers) {   // temporal upscalers (K11/K12)
        HK_CUDA(alloc_plane(ctx, &p.upscale_output, 4 * n, L));
        HK_CUDA(alloc_plane(ctx, &p.taa_output[0], 4 * n, L));
        HK_CUDA(alloc_plane(ctx, &p.taa_output[1], 4 * n, L));
    }
    if (ctx->full_frame) HK_CUDA(alloc_plane(ctx, &p.upscale_sharpen_output, n, L));   // FSR RCAS result (Upscale::Fsr1)
    ctx->tile_maps_ready = make_spatial_tile_maps(ctx);     // false: no TMA descriptors (old driver) -> the gather form of the pass
    ctx->planes_ready = true;
    return HK_OK;
}

extern "C" {

const char* hk_version(void) { return "hikari_b200 0.1 (sm_90a)"; }

const char* hk_last_error(hk_context* ctx) { return ctx ? ctx->error.c_str() : g_create_error.c_str(); }

int hk_context_create(hk_context** out, int cuda_device, uint32_t width, uint32_t height, uint32_t row_begin, uint32_t row_end,
                      void* cuda_stream) {
    return hk_context_create_tile(out, cuda_device, width, height, 0, width, row_begin, row_end, cuda_stream);
}

int hk_context_create_tile(hk_context** out, int cuda_device, uint32_t width, uint32_t height, uint32_t col_begin, uint32_t col_end,
                           uint32_t row_begin, uint32_t row_end, void* cuda_stream) {
    hk_context* ctx = nullptr;
    if (!out) return set_error(nullptr, HK_ERR_INVALID_ARGUMENT, "out == NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return set_error(nullptr, HK_ERR_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(e) +
                                                   " (this library has no CPU fallback)");
    if (cuda_device < 0 || cuda_device >= ndev) return set_error(nullptr, HK_ERR_INVALID_ARGUMENT, "bad cuda_device");
    HK_CUDA(cudaSetDevice(cuda_device));
    hk_context* c = new hk_context();
    c->device = cuda_device;
    // defaults of hk_set_tuning from the environment (A/B runs of one build: HK_TUNE_POOLED_INDIRECT=1, HK_TUNE_TILED_SPATIAL=0)
    if (const char* e = getenv("HK_TUNE_POOLED_INDIRECT")) c->pooled_indirect = atoi(e) != 0;
    if (const char* e = getenv("HK_TUNE_TILED_SPATIAL")) c->tiled_spatial = atoi(e) != 0;
    if (const char* e = getenv("HK_TUNE_TILED_DENOISE")) c->tiled_denoise = atoi(e) != 0;
    c->wide_traversal = hk_tolerance_build() != 0 ? HK_WIDE_TRAVERSAL_DEFAULT : 0;      // the exact flavour keeps the reference's walk
    if (const char* e = getenv("HK_TUNE_WIDE_TRAVERSAL")) c->wide_traversal = atoi(e) & 3;
    ctx = c;
    if (cuda_stream) c->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
    else {
        e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
        if (e != cudaSuccess) { delete c; return set_error(nullptr, HK_ERR_CUDA, cudaGetErrorString(e)); }
        c->own_stream = true;
    }
    int rc = HK_OK;
    {   // at the default priority, as the streams a host usually renders on: the block scheduler interleaves the two branches' CTAs
        // freely (a higher priority for either branch measured slower, DESIGN.md §4a-6)
        if (cudaStreamCreateWithFlags(&c->indirect_stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming) != cudaSuccess)
            rc = set_error(c, HK_ERR_CUDA, "indirect light stream");
    }
    if (rc == HK_OK) rc = allocate_planes(c, width, height, col_begin, col_end, row_begin, row_end);
    if (rc == HK_OK) {
        void* p = nullptr;
        if (cudaMalloc(&p, sizeof(Counters)) != cudaSuccess) rc = set_error(c, HK_ERR_OUT_OF_MEMORY, "counters");
        else { c->counters = reinterpret_cast<Counters*>(p); cudaMemsetAsync(p, 0, sizeof(Counters), c->stream); }
    }
    if (rc == HK_OK) {   // per-neighbour constants of spatial_reuse, light.wgsl:246-253,1566-1572,1609-1620
        SpatialTable t[2];
        memset(t, 0, sizeof(t));
        for (int v = 0; v < 2; ++v) {
            const uint32_t count = v ? 8u : 16u;
            const float range = v ? 10.0f : 20.0f;
            const uint32_t taps = 4u;
            for (uint32_t i = 1; i <= count; ++i) {
                t[v].phase[i] = (float)i * hk::GOLDEN_RATIO;
                const float rad = sqrtf((float)i / (float)count) * range;
                t[v].radius[i] = rad;
                const float tap_interval = hk::fmax_(1.0f, rad / (float)(taps + 1u));
                const uint32_t tap_count = hk::f32_to_u32(rad / tap_interval);
                t[v].tap_count[i] = tap_count > 6u ? 6u : tap_count;   // never above 5 (radius / (radius / 5))
                for (uint32_t j = 1; j <= t[v].tap_count[i]; ++j) {
                    t[v].tap_dist[i][j - 1] = (float)j * tap_interval;
                    t[v].tap_ratio[i][j - 1] = (float)j / (float)(tap_count + 1u);
                }
            }
        }
        memcpy(c->spatial_tables_host, t, sizeof(t));
        void* p = nullptr;
        if (cudaMalloc(&p, sizeof(t)) != cudaSuccess) rc = set_error(c, HK_ERR_OUT_OF_MEMORY, "spatial tables");
        else {
            c->spatial_tables = reinterpret_cast<SpatialTable*>(p);
            if (cudaMemcpy(p, t, sizeof(t), cudaMemcpyHostToDevice) != cudaSuccess) rc = set_error(c, HK_ERR_CUDA, "spatial tables upload");
        }
    }
    if (rc == HK_OK)
        for (int i = 0; i < 4; ++i)
            if (cudaEventCreate(&c->ev[i]) != cudaSuccess) rc = set_error(c, HK_ERR_CUDA, "cudaEventCreate");
    if (rc == HK_OK)
        for (int i = 0; i < HK_K_COUNT; ++i)
            for (int j = 0; j < 2; ++j)
                if (cudaEventCreate(&c->kev[i][j]) != cudaSuccess) rc = set_error(c, HK_ERR_CUDA, "cudaEventCreate");
    if (rc != HK_OK) {
        g_create_error = c->error;
        hk_context_destroy(c);
        return rc;
    }
    *out = c;
    return HK_OK;
}

void hk_context_destroy(hk_context* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    if (ctx->copy_stream) { cudaStreamSynchronize(ctx->copy_stream); cudaStreamDestroy(ctx->copy_stream); }
    for (void* p : ctx->frames_opened) cudaIpcCloseMemHandle(p);
    for (hk_halo_peer* peer : ctx->halo_peers) {
        for (void* p : peer->mapped) if (p) cudaIpcCloseMemHandle(p);
        delete peer;
    }
    for (void* p : ctx->frames_owned) cudaFree(p);
    if (ctx->ev_submitted) cudaEventDestroy(ctx->ev_submitted);
    if (ctx->ev_copied) cudaEventDestroy(ctx->ev_copied);
    free_list(ctx->allocations);
    detach_scene(ctx);                     // frees a private scene, and a shared one whose handle and other contexts are gone
    if (ctx->ev_released) cudaEventDestroy(ctx->ev_released);
    if (ctx->noise) cudaFree(ctx->noise);
    if (ctx->counters) cudaFree(ctx->counters);
    if (ctx->spatial_tables) cudaFree(ctx->spatial_tables);
    for (int i = 0; i < 4; ++i) if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
    for (int i = 0; i < HK_K_COUNT; ++i)
        for (int j = 0; j < 2; ++j) if (ctx->kev[i][j]) cudaEventDestroy(ctx->kev[i][j]);
    for (int i = 0; i < hk_context::RING; ++i)
        for (int j = 0; j < 2; ++j) if (ctx->ring[i][j]) cudaEventDestroy(ctx->ring[i][j]);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    if (ctx->indirect_stream) cudaStreamDestroy(ctx->indirect_stream);   // idle: its work is joined into `stream`, synchronised above
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int hk_context_resize(hk_context* ctx, uint32_t width, uint32_t height, uint32_t row_begin, uint32_t row_end) {
    return hk_context_resize_tile(ctx, width, height, 0, width, row_begin, row_end);
}
int hk_context_resize_tile(hk_context* ctx, uint32_t width, uint32_t height, uint32_t col_begin, uint32_t col_end,
                           uint32_t row_begin, uint32_t row_end) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    // The reference re-allocates (and zeroes) the reservoirs only when size.x * size.y changes (light.rs:342-363); a host that
    // calls resize every frame (prepare_light_textures runs every frame) must not lose its temporal state or pay ~100 cudaMallocs.
    const Band& b = ctx->band;
    if (ctx->planes_ready && (int)width == b.W && (int)height == b.H && (int)col_begin == b.cx0 && (int)col_end == b.cx1 &&
        (int)row_begin == b.r0 && (int)row_end == b.r1)
        return HK_OK;
    HK_CUDA(cudaSetDevice(ctx->device));
    HK_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ctx->copy_stream) HK_CUDA(cudaStreamSynchronize(ctx->copy_stream));
    ctx->copy_in_flight = ctx->copy_unwaited = false;
    return allocate_planes(ctx, width, height, col_begin, col_end, row_begin, row_end);  // zeroed planes (light.rs:342-363)
}

int hk_reset_temporal_state(hk_context* ctx) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    if (!ctx->planes_ready) return set_error(ctx, HK_ERR_NOT_READY, "per-pixel planes are not allocated (a resize failed)");
    HK_CUDA(cudaSetDevice(ctx->device));
    for (int r = 0; r < 10; ++r)
        for (int q = 0; q < 4; ++q) HK_CUDA(cudaMemsetAsync(ctx->planes.reservoir[r].q[q], 0, ctx->band_pixels * sizeof(uint4), ctx->stream));
    return HK_OK;
}

}  // extern "C"

template <class T>
static cudaError_t upload(hk_shared_scene* sc, const T** dst, const T* src, uint32_t count) {
    void* p = nullptr;
    size_t bytes = (size_t)count * sizeof(T);
    cudaError_t e = cudaMalloc(&p, bytes + 64);   // +64: 16-byte vector loads at the tail stay in bounds
    if (e != cudaSuccess) return e;
    sc->scene_allocations.push_back(p);
    e = cudaMemsetAsync(p, 0, bytes + 64, sc->stream);
    if (e != cudaSuccess) return e;
    if (bytes) e = cudaMemcpyAsync(p, src, bytes, cudaMemcpyHostToDevice, sc->stream);
    *dst = reinterpret_cast<const T*>(p);
    return e;
}


// copy into a grow-only device buffer (per-frame updates must not pay cudaMalloc/cudaFree)
template <class T>
static cudaError_t upload_into(hk_shared_scene* sc, hk_shared_scene::DevBuf& b, const T** dst, const T* src, size_t count) {
    const size_t bytes = count * sizeof(T), need = bytes + 64;   // +64: 16-byte vector loads at the tail stay in bounds
    cudaError_t e = cudaSuccess;
    if (b.cap < need) {
        if (b.p) { scene_before_free(sc); cudaFree(b.p); }
        b.p = nullptr; b.cap = 0;
        const size_t cap = need + need / 2;
        e = cudaMalloc(&b.p, cap);
        if (e != cudaSuccess) return e;
        b.cap = cap;
    }
    if (bytes) e = cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, sc->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(static_cast<char*>(b.p) + bytes, 0, 64, sc->stream);
    *dst = reinterpret_cast<const T*>(b.p);
    return e;
}

// grow-only device scratch
static cudaError_t ensure_buf(hk_shared_scene* sc, hk_shared_scene::DevBuf& b, size_t bytes) {
    const size_t need = bytes + 64;
    if (b.cap >= need) return cudaSuccess;
    if (b.p) { scene_before_free(sc); cudaFree(b.p); }
    b.p = nullptr; b.cap = 0;
    const size_t cap = need + need / 2;
    cudaError_t e = cudaMalloc(&b.p, cap);
    if (e == cudaSuccess) b.cap = cap;
    return e;
}

// The 4-wide tree over the instances (the half of upload_wide that every instance update repeats) from the flat TLAS in `nodes`
// (host memory) and the instances' boxes (6 floats each, or null when the navigators carry them by construction); the meshes' trees
// and sc->wide_mesh_of are those of the last upload_wide.
static int upload_wide_tlas(hk_shared_scene* sc, const hk_node* nodes, uint32_t node_count, uint32_t instance_count, const float* instance_box,
                            DeviceScene& d) {
    d.wide_ready = 0u; d.wide_tlas_root = WIDE_EMPTY;
    sc->wide_on_device = false;
    hkw::WideTree tlas = hkw::build_wide(nodes, node_count, instance_count, instance_box);
    bool blas_ok = sc->wide_mesh_of.size() == instance_count;
    uint32_t blas_need = 0;
    std::vector<uint2> entry(instance_count);
    for (uint32_t i = 0; i < instance_count && sc->wide_mesh_of.size() == instance_count; ++i) {
        const hk_shared_scene::WideMesh& m = sc->wide_meshes[sc->wide_mesh_of[i]];
        blas_ok = blas_ok && m.ok;
        entry[i] = make_uint2(m.base, m.root);
        blas_need = std::max(blas_need, m.need);
    }
    const bool ok = tlas.ok && blas_ok;
    sc->wide_blas_ok = blas_ok;
    sc->wide_blas_need = blas_need;
    if (!tlas.ok) { tlas.nodes.clear(); tlas.rank.assign(instance_count, 0u); }
    sc->wide_tlas_node_count = (uint32_t)tlas.nodes.size();
    // hk_scene_update_transforms re-derives the tree into the same buffers on the device: sized here for the largest tree over these
    // instances (n - 1 nodes, n ranks) with its scratch, so that the update allocates nothing
    const size_t max_nodes = instance_count > 1u ? instance_count - 1u : 1u;
    HK_SCUDA(ensure_buf(sc, sc->ibuf[9], sizeof(hk_wide_node) * max_nodes));
    HK_SCUDA(ensure_buf(sc, sc->ibuf[12], sizeof(uint32_t) * (size_t)instance_count));
    HK_SCUDA(ensure_buf(sc, sc->ibuf[16], hk_wide_tlas_scratch_bytes(instance_count)));
    HK_SCUDA(upload_into(sc, sc->ibuf[9], &d.wide_tlas, tlas.nodes.data(), tlas.nodes.size()));
    HK_SCUDA(upload_into(sc, sc->ibuf[11], &d.wide_instance, entry.data(), entry.size()));
    HK_SCUDA(upload_into(sc, sc->ibuf[12], &d.wide_instance_rank, tlas.rank.data(), tlas.rank.size()));
    // pending TLAS siblings + the BLAS marker + pending BLAS siblings, and the three pushes a node step makes before it pops
    sc->wide_stack_need = tlas.stack_need + 1u + blas_need + 3u;
    const bool ready = ok && sc->wide_stack_need <= (uint32_t)HK_WIDE_STACK;
    const uint32_t state[3] = {ready ? 1u : 0u, sc->wide_stack_need, sc->wide_tlas_node_count};
    HK_SCUDA(upload_into(sc, sc->ibuf[15], &d.wide_state, state, 3));
    HK_SCUDA(cudaStreamSynchronize(sc->stream));
    if (ready) {
        d.wide_tlas_root = tlas.root;
        d.wide_ready = 1u;
    }
    return HK_OK;
}

// The 4-wide trees of the image-exact traversal mode (hk_wide.cuh / wide_build.h) for the scene in `s`: one tree per distinct mesh
// (rebuilt only when the set of meshes in use changes), one over the instances (every call), the per-instance entry points and the
// array-order ranks that settle ties.  d.wide_ready stays 0 — and every launch keeps the reference's walk — when a flat array is not
// in bvh 0.7.1's layout or the trees could ask for more stack than the walk has.
static int upload_wide(hk_shared_scene* sc, const hk_scene_desc* s, DeviceScene& d) {
    d.wide_ready = 0u; d.wide_tlas_root = WIDE_EMPTY;
    sc->wide_stack_need = 0;
    std::vector<std::array<uint32_t, 3>> keys;
    std::vector<uint32_t> mesh_of(s->instance_count);
    for (uint32_t i = 0; i < s->instance_count; ++i) {
        const hk_mesh_index& m = s->instances[i].mesh;
        const std::array<uint32_t, 3> key = {m.node_offset, m.node_count, m.primitive};
        size_t k = 0;
        while (k < keys.size() && keys[k] != key) ++k;      // few distinct meshes (3 in the city, 1 per instance in scene.rs)
        if (k == keys.size()) keys.push_back(key);
        mesh_of[i] = (uint32_t)k;
    }
    if (keys != sc->wide_mesh_keys || sc->ibuf[10].p == nullptr) {
        std::vector<hk_wide_node> all;
        std::vector<hk_shared_scene::WideMesh> meshes(keys.size());
        std::vector<uint32_t> prim_rank(sc->scene_primitive_count, 0u);
        for (size_t k = 0; k < keys.size(); ++k) {
            if ((uint64_t)keys[k][0] + keys[k][1] > sc->host_asset_nodes.size()) continue;   // built on the device: no 4-wide tree
            const hk_node* flat = sc->host_asset_nodes.data() + keys[k][0];
            uint32_t shapes = 0;
            for (uint32_t r = 0; r < keys[k][1]; ++r)
                if (flat[r].entry_index >= 0x80000000u) shapes = std::max(shapes, flat[r].entry_index - 0x80000000u + 1u);
            hkw::WideTree t = hkw::build_wide(flat, keys[k][1], shapes, sc->host_primitive_box.data() + 6 * (size_t)keys[k][2]);
            meshes[k].ok = t.ok;
            if (!t.ok) continue;
            if (t.root == WIDE_EMPTY) {      // a mesh without records: WIDE_EMPTY as its entry point would end the whole walk, not
                t.nodes.assign(1, hkw::empty_node());       // just the instance; a node without children returns to the TLAS
                t.root = 0;
            }
            meshes[k].base = (uint32_t)all.size(); meshes[k].root = t.root; meshes[k].need = t.stack_need;
            all.insert(all.end(), t.nodes.begin(), t.nodes.end());
            for (uint32_t sh = 0; sh < shapes; ++sh)
                if (t.rank[sh] != 0xFFFFFFFFu && (uint64_t)keys[k][2] + sh < prim_rank.size()) prim_rank[keys[k][2] + sh] = t.rank[sh];
        }
        HK_SCUDA(upload_into(sc, sc->ibuf[10], &d.wide_blas, all.data(), all.size()));
        HK_SCUDA(upload_into(sc, sc->ibuf[13], &d.wide_primitive_rank, prim_rank.data(), prim_rank.size()));
        HK_SCUDA(cudaStreamSynchronize(sc->stream));      // the staging vectors die at the end of this block
        sc->wide_mesh_keys = keys; sc->wide_meshes = meshes; sc->wide_blas_node_count = (uint32_t)all.size();
    } else {
        d.wide_blas = reinterpret_cast<const hk_wide_node*>(sc->ibuf[10].p);
        d.wide_primitive_rank = reinterpret_cast<const uint32_t*>(sc->ibuf[13].p);
    }
    sc->wide_mesh_of = mesh_of;
    std::vector<float> instance_box(6 * (size_t)s->instance_count);
    for (uint32_t i = 0; i < s->instance_count; ++i)
        for (int c = 0; c < 3; ++c) { instance_box[6 * (size_t)i + c] = s->instances[i].min[c]; instance_box[6 * (size_t)i + 3 + c] = s->instances[i].max[c]; }
    return upload_wide_tlas(sc, s->instance_nodes, s->instance_node_count, s->instance_count, instance_box.data(), d);
}

// Validation + upload of the per-frame half of the scene (instances, TLAS, emissives, emissive BVH, alias tables,
// previous model matrices) into `d`.  Frees the previous copies.
static int upload_instances(hk_shared_scene* sc, const hk_scene_desc* s, DeviceScene& d) {
    // materials travel with the per-frame half when given (material.rs:139-203 rewrites them whenever a material changes)
    const bool new_materials = s->materials != nullptr && s->material_count > 0;
    const uint32_t material_count = new_materials ? s->material_count : sc->scene_material_count;
    if ((s->instance_count && !s->instances) || (s->instance_node_count && !s->instance_nodes) ||
        (s->emissive_node_count && !s->emissive_nodes) || (s->emissive_count && !s->emissives) || (s->alias_count && !s->alias_table))
        return set_error(sc, HK_ERR_INVALID_ARGUMENT, "scene buffer pointer is NULL with a non-zero count");
    // Validate every index the kernels follow, once, so that they can skip bounds checks (wgpu's robust buffer access would clamp
    // a bad index; here a malformed host buffer is refused instead of read out of bounds).
    for (uint32_t i = 0; i < s->instance_count; ++i) {
        const hk_instance& in = s->instances[i];
        if (in.material >= material_count || (uint64_t)in.mesh.node_offset + in.mesh.node_count > sc->scene_asset_node_count)
            return set_error(sc, HK_ERR_INVALID_ARGUMENT, "instance references a material / node range out of bounds");
        if (in.mesh.primitive > sc->scene_primitive_count || in.mesh.vertex > sc->scene_vertex_count)
            return set_error(sc, HK_ERR_INVALID_ARGUMENT, "instance references a primitive / vertex range out of bounds");
        // every leaf of the instance's BLAS must name a primitive inside the primitive buffer, and every link a record of its range
        const std::array<uint32_t, 4> mesh_key = {in.mesh.vertex, in.mesh.primitive, in.mesh.node_offset, in.mesh.node_count};
        if (!sc->mesh_range_checked.count(mesh_key)) {
            const std::vector<hk_node>& nodes = sc->host_asset_nodes;
            if ((uint64_t)in.mesh.node_offset + in.mesh.node_count > nodes.size())     // records built on the device: only as added
                return set_error(sc, HK_ERR_INVALID_ARGUMENT, "instance references a BLAS range that is not one hk_scene_add_meshes returned");
            for (uint32_t k = 0; k < in.mesh.node_count; ++k) {
                const hk_node& nd = nodes[in.mesh.node_offset + k];
                if (nd.entry_index >= 0x80000000u) {
                    const uint64_t pid = (uint64_t)in.mesh.primitive + (nd.entry_index - 0x80000000u);
                    if (pid >= sc->scene_primitive_count)
                        return set_error(sc, HK_ERR_INVALID_ARGUMENT, "BLAS leaf references a primitive out of bounds");
                    const uint32_t* vi = &sc->host_primitive_vertex_index[3 * pid];
                    for (int c = 0; c < 3; ++c)
                        if ((uint64_t)in.mesh.vertex + vi[c] >= sc->scene_vertex_count)
                            return set_error(sc, HK_ERR_INVALID_ARGUMENT, "primitive references a vertex out of bounds");
                } else if (nd.entry_index > in.mesh.node_count) {
                    return set_error(sc, HK_ERR_INVALID_ARGUMENT, "BLAS entry link out of its mesh's node range");
                }
            }
            sc->mesh_range_checked.insert(mesh_key);
        }
    }
    if (new_materials && sc->scene_texture_count != 0xFFFFFFFFu) {
        for (uint32_t i = 0; i < s->material_count; ++i) {
            const hk_material& m = s->materials[i];
            const uint32_t ids[5] = {m.base_color_texture, m.emissive_texture, m.metallic_roughness_texture, m.normal_map_texture, m.occlusion_texture};
            for (uint32_t id : ids)
                if (id != 0xFFFFFFFFu && id >= sc->scene_texture_count)
                    return set_error(sc, HK_ERR_INVALID_ARGUMENT, "material references a texture out of bounds");
        }
    }
    for (uint32_t i = 0; i < s->instance_node_count; ++i) {
        const hk_node& nd = s->instance_nodes[i];
        if (nd.entry_index >= 0x80000000u) {
            if (nd.entry_index - 0x80000000u >= s->instance_count)
                return set_error(sc, HK_ERR_INVALID_ARGUMENT, "TLAS leaf references an instance out of bounds");
        }
    }
    for (uint32_t i = 0; i < s->emissive_node_count; ++i) {
        const hk_node& nd = s->emissive_nodes[i];
        if (nd.entry_index >= 0x80000000u && nd.entry_index - 0x80000000u >= s->emissive_count)
            return set_error(sc, HK_ERR_INVALID_ARGUMENT, "emissive BVH leaf references an emissive out of bounds");
    }
    for (uint32_t i = 0; i < s->emissive_count; ++i) {
        const hk_emissive& em = s->emissives[i];
        if (em.instance >= s->instance_count || (uint64_t)em.alias_table_offset + em.alias_table_count > s->alias_count || em.alias_table_count == 0)
            return set_error(sc, HK_ERR_INVALID_ARGUMENT, "emissive references an instance / alias-table slice out of bounds");
        // alias entries index triangles of the emissive instance's mesh
        const hk_instance& ei = s->instances[em.instance];
        for (uint32_t k = 0; k < em.alias_table_count; ++k)
            if ((uint64_t)ei.mesh.primitive + s->alias_table[em.alias_table_offset + k].index >= sc->scene_primitive_count)
                return set_error(sc, HK_ERR_INVALID_ARGUMENT, "alias-table entry references a primitive out of bounds");
    }
    // Does every leaf record sit right behind a navigator whose box is the shape's own AABB?  (true for bvh 0.7.1's
    // flatten_custom, which is what the reference uploads; then the kernels skip the re-derived leaf box test.)
    bool boxes_match = sc->mesh_boxes_match;
    auto same3 = [](const float* a, const float* b) { return a[0] == b[0] && a[1] == b[1] && a[2] == b[2]; };
    for (uint32_t i = 1; i < s->instance_node_count && boxes_match; ++i) {
        const hk_node& leaf = s->instance_nodes[i];
        if (leaf.entry_index < 0x80000000u) continue;
        const hk_node& nav = s->instance_nodes[i - 1];
        uint32_t id = leaf.entry_index - 0x80000000u;
        boxes_match = nav.entry_index == i && id < s->instance_count && same3(nav.min, s->instances[id].min) &&
                      same3(nav.max, s->instances[id].max);
    }
    HK_SCUDA(cudaStreamSynchronize(sc->stream));   // frames in flight still read the buffers that are overwritten below
    d.leaf_boxes_match = boxes_match ? 1u : 0u;
    if (new_materials) {
        HK_SCUDA(upload_into(sc, sc->ibuf[7], &d.materials, s->materials, s->material_count));
        sc->scene_material_count = s->material_count;
    }
    HK_SCUDA(upload_into(sc, sc->ibuf[0], &d.alias_table, s->alias_table, s->alias_count));
    HK_SCUDA(upload_into(sc, sc->ibuf[1], &d.instances, s->instances, s->instance_count));
    HK_SCUDA(upload_into(sc, sc->ibuf[2], &d.instance_nodes, s->instance_nodes, s->instance_node_count));
    HK_SCUDA(upload_into(sc, sc->ibuf[3], &d.emissive_nodes, s->emissive_nodes, s->emissive_node_count));
    HK_SCUDA(upload_into(sc, sc->ibuf[4], &d.emissives, s->emissives, s->emissive_count));
    {   // compact traversal records + what the pooled kernels stage into shared memory (hk_pool.cuh)
        std::vector<hk_instance_trav> trav(s->instance_count);
        for (uint32_t i = 0; i < s->instance_count; ++i) {
            memcpy(trav[i].inverse_transpose_model, s->instances[i].inverse_transpose_model, 64);
            trav[i].mesh[0] = s->instances[i].mesh.vertex; trav[i].mesh[1] = s->instances[i].mesh.primitive;
            trav[i].mesh[2] = s->instances[i].mesh.node_offset; trav[i].mesh[3] = s->instances[i].mesh.node_count;
        }
        HK_SCUDA(upload_into(sc, sc->ibuf[8], &d.instance_trav, trav.data(), trav.size()));
        HK_SCUDA(cudaStreamSynchronize(sc->stream));      // `trav` dies at the end of this block
        StagePlan plan{};
        const uint32_t budget = (uint32_t)HK_STAGE_F4;
        const uint64_t tlas = 2ull * s->instance_node_count, itrav = 5ull * s->instance_count;
        if (s->instance_node_count && tlas + itrav <= budget) {
            plan.tlas_f4 = 0; plan.tlas_count = s->instance_node_count;
            plan.itrav_f4 = (uint32_t)tlas; plan.itrav_count = s->instance_count;
            const uint64_t used = tlas + itrav, blas = 2ull * sc->scene_asset_node_count, prim = 3ull * sc->scene_primitive_count;
            if (sc->scene_asset_node_count && used + blas + prim <= budget) {     // small scene: walked entirely out of shared memory
                plan.blas_f4 = (uint32_t)used; plan.blas_count = sc->scene_asset_node_count;
                plan.prim_f4 = (uint32_t)(used + blas); plan.prim_count = sc->scene_primitive_count;
            }
        }
        d.stage = plan;
    }
    d.instance_node_count = s->instance_node_count;
    d.emissive_node_count = s->emissive_node_count;
    d.previous_models = nullptr;
    d.instance_moved = nullptr;
    std::vector<uint32_t> moved;
    if (s->previous_instance_models && s->instance_count) {
        moved.resize(s->instance_count);
        bool any = false;
        for (uint32_t i = 0; i < s->instance_count; ++i) {
            moved[i] = memcmp(s->previous_instance_models + 16 * (size_t)i, s->instances[i].model, 64) != 0 ? 1u : 0u;
            any = any || moved[i];
        }
        if (any) {
            HK_SCUDA(upload_into(sc, sc->ibuf[5], &d.previous_models, reinterpret_cast<const float4*>(s->previous_instance_models), 4 * (size_t)s->instance_count));
            HK_SCUDA(upload_into(sc, sc->ibuf[6], &d.instance_moved, moved.data(), s->instance_count));
        }
    }
    HK_SCUDA(cudaStreamSynchronize(sc->stream));      // caller's arrays (and `moved`) may be freed after return
    sc->scene_instance_count = s->instance_count;
    sc->scene_emissive_count = s->emissive_count;
    return upload_wide(sc, s, d);
}

// A model matrix with an infinite or NaN entry has no world box and no place in the TLAS (the SAH build's bucket of a NaN centre is
// undefined, and differently so on the host and the device): refused on the host, before anything is built, launched or freed, so
// that the scene stays as it was.  Singular but finite models (an axis scaled to zero) are accepted, as the reference accepts them.
static int check_models(hk_shared_scene* sc, const float* models, size_t stride_floats, uint32_t n, const char* what) {
    for (uint32_t i = 0; i < n; ++i) {
        const float* m = models + stride_floats * (size_t)i;
        for (int k = 0; k < 16; ++k) {
            uint32_t bits;
            memcpy(&bits, m + k, 4);
            if ((bits & 0x7f800000u) == 0x7f800000u)
                return set_error(sc, HK_ERR_INVALID_ARGUMENT, std::string(what) + ": instance " + std::to_string(i) + " has a non-finite model matrix (entry " +
                                                              std::to_string(k) + ")");
        }
    }
    return HK_OK;
}
static int check_instance_models(hk_shared_scene* sc, const hk_scene_desc* s, const char* what) {
    if (!s->instance_count || !s->instances) return HK_OK;     // (a NULL pointer is reported by upload_instances)
    static_assert(sizeof(hk_instance) % sizeof(float) == 0, "instance records are float-aligned");
    return check_models(sc, s->instances[0].model, sizeof(hk_instance) / sizeof(float), s->instance_count, what);
}

static int scene_upload(hk_shared_scene* sc, const hk_scene_desc* s) {
    if ((s->vertex_count && !s->vertices) || (s->primitive_count && !s->primitives) ||
        (s->material_count && !s->materials) || (s->asset_node_count && !s->asset_nodes) || (s->texture_count && !s->textures))
        return set_error(sc, HK_ERR_INVALID_ARGUMENT, "scene buffer pointer is NULL with a non-zero count");
    if (const int rc = check_instance_models(sc, s, "hk_scene_upload")) return rc;
    bool boxes_match = true;
    auto same3 = [](const float* a, const float* b) { return a[0] == b[0] && a[1] == b[1] && a[2] == b[2]; };
    std::unordered_set<uint32_t> checked;   // mesh node ranges repeat across instances: check each once
    for (uint32_t m = 0; m < s->instance_count && boxes_match && s->instances; ++m) {
        const hk_mesh_index& mi = s->instances[m].mesh;
        if ((uint64_t)mi.node_offset + mi.node_count > s->asset_node_count) break;   // reported by upload_instances
        if (!checked.insert(mi.node_offset).second) continue;
        for (uint32_t i = 1; i < mi.node_count && boxes_match; ++i) {
            const hk_node& leaf = s->asset_nodes[mi.node_offset + i];
            if (leaf.entry_index < 0x80000000u) continue;
            const hk_node& nav = s->asset_nodes[mi.node_offset + i - 1];
            uint64_t pid = (uint64_t)mi.primitive + (leaf.entry_index - 0x80000000u);
            if (nav.entry_index != i || pid >= s->primitive_count) { boxes_match = false; break; }
            const hk_primitive& p = s->primitives[pid];
            float mn[3], mx[3];
            for (int c = 0; c < 3; ++c) {
                mn[c] = fminf(p.vertices[0].position[c], fminf(p.vertices[1].position[c], p.vertices[2].position[c]));
                mx[c] = fmaxf(p.vertices[0].position[c], fmaxf(p.vertices[1].position[c], p.vertices[2].position[c]));
            }
            boxes_match = same3(nav.min, mn) && same3(nav.max, mx);
        }
    }
    HK_SCUDA(cudaSetDevice(sc->device));
    HK_SCUDA(cudaStreamSynchronize(sc->stream));     // (after scene_begin_write: also every attached camera's last read)
    free_list(sc->scene_allocations);
    free_mesh_bufs(sc);
    sc->ready = false;
    sc->mesh_boxes_match = boxes_match;
    sc->scene_material_count = 0;
    sc->scene_asset_node_count = s->asset_node_count;
    sc->scene_primitive_count = s->primitive_count;
    sc->scene_vertex_count = s->vertex_count;
    sc->scene_texture_count = s->texture_count;
    sc->host_asset_nodes.assign(s->asset_nodes, s->asset_nodes + s->asset_node_count);
    sc->mesh_range_checked.clear();
    sc->wide_mesh_keys.clear(); sc->wide_meshes.clear();     // new asset nodes: the meshes' 4-wide trees are rebuilt
    sc->host_primitive_vertex_index.resize(3 * (size_t)s->primitive_count);
    for (uint32_t i = 0; i < s->primitive_count; ++i)
        for (int c = 0; c < 3; ++c) sc->host_primitive_vertex_index[3 * (size_t)i + c] = s->primitives[i].vertices[c].index;
    sc->host_primitive_box.resize(6 * (size_t)s->primitive_count);
    for (uint32_t i = 0; i < s->primitive_count; ++i) {
        const hk_primitive& p = s->primitives[i];
        for (int c = 0; c < 3; ++c) {
            sc->host_primitive_box[6 * (size_t)i + c] = fminf(p.vertices[0].position[c], fminf(p.vertices[1].position[c], p.vertices[2].position[c]));
            sc->host_primitive_box[6 * (size_t)i + 3 + c] = fmaxf(p.vertices[0].position[c], fmaxf(p.vertices[1].position[c], p.vertices[2].position[c]));
        }
    }
    // primitives index vertices relative to their mesh's vertex base: the largest index of each mesh is checked per instance
    // below through mesh.vertex + index < vertex_count for the primitives of its leaves
    DeviceScene d{};
    HK_SCUDA(upload(sc, &d.vertices, s->vertices, s->vertex_count));
    HK_SCUDA(upload(sc, &d.primitives, s->primitives, s->primitive_count));
    HK_SCUDA(upload(sc, &d.asset_nodes, s->asset_nodes, s->asset_node_count));
    sc->mbuf[0] = {const_cast<hk_vertex*>(d.vertices), sizeof(hk_vertex) * (size_t)s->vertex_count, false};
    sc->mbuf[1] = {const_cast<hk_primitive*>(d.primitives), sizeof(hk_primitive) * (size_t)s->primitive_count, false};
    sc->mbuf[2] = {const_cast<hk_node*>(d.asset_nodes), sizeof(hk_node) * (size_t)s->asset_node_count, false};
    d.materials = nullptr;           // uploaded with the per-frame half below
    d.texture_count = s->texture_count;
    d.textures = nullptr;
    if (s->texture_count) {
        // decode to linear float4 texels on the host (sRGB LUT built with the same libm call as the oracle's)
        float srgb_lut[256], lin_lut[256];
        for (int i = 0; i < 256; ++i) {
            double v = i / 255.0;
            lin_lut[i] = (float)v;
            srgb_lut[i] = (float)(v <= 0.04045 ? v / 12.92 : pow((v + 0.055) / 1.055, 2.4));
        }
        std::vector<uint4> info(s->texture_count);
        size_t total = 0;
        for (uint32_t t = 0; t < s->texture_count; ++t) {
            const hk_texture_desc& td = s->textures[t];
            if (!td.rgba8 || !td.width || !td.height) return set_error(sc, HK_ERR_INVALID_ARGUMENT, "bad texture");
            info[t] = make_uint4((uint32_t)total, td.width, td.height,
                                 (td.address_mode_u & 3u) | ((td.address_mode_v & 3u) << 2) | (td.filter_linear ? 16u : 0u));
            total += (size_t)td.width * td.height;
        }
        if (total > 0xFFFFFFFFull) return set_error(sc, HK_ERR_UNSUPPORTED, "texture atlas too large");
        std::vector<float4> texels(total);
        for (uint32_t t = 0; t < s->texture_count; ++t) {
            const hk_texture_desc& td = s->textures[t];
            const float* lut = td.srgb ? srgb_lut : lin_lut;
            float4* dst = texels.data() + info[t].x;
            size_t n = (size_t)td.width * td.height;
            for (size_t i = 0; i < n; ++i)
                dst[i] = make_float4(lut[td.rgba8[4 * i]], lut[td.rgba8[4 * i + 1]], lut[td.rgba8[4 * i + 2]], lin_lut[td.rgba8[4 * i + 3]]);
        }
        HK_SCUDA(upload(sc, &d.texture_texels, texels.data(), (uint32_t)total));
        HK_SCUDA(upload(sc, &d.texture_info, info.data(), s->texture_count));
        HK_SCUDA(cudaStreamSynchronize(sc->stream));  // host staging vectors die at scope exit
    }
    int rc = upload_instances(sc, s, d);
    if (rc != HK_OK) return rc;
    sc->scene = d;
    sc->ready = true;
    return HK_OK;
}

static int scene_update_instances(hk_shared_scene* sc, const hk_scene_desc* s) {
    if (!sc->ready) return set_error(sc, HK_ERR_NOT_READY, "hk_scene_update_instances needs a scene from hk_scene_upload");
    if (const int rc = check_instance_models(sc, s, "hk_scene_update_instances")) return rc;
    HK_SCUDA(cudaSetDevice(sc->device));
    DeviceScene d = sc->scene;
    int rc = upload_instances(sc, s, d);
    if (rc != HK_OK) {   // validation fails before anything is freed; a CUDA failure may leave freed buffers behind
        if (rc != HK_ERR_INVALID_ARGUMENT) sc->ready = false;
        return rc;
    }
    sc->scene = d;
    return HK_OK;
}

extern "C" {      // (defined with the scheduling below)
static bool wide_primary(const hk_context* ctx);
static bool wide_light(const hk_context* ctx);
}

// The next of the scene's two pinned staging slots with room for `bytes`; waits only for the copy made from it two calls ago.
// The caller records pin.ev after its copy and sets pin.used.
static int pinned_slot(hk_shared_scene* sc, size_t bytes, hk_shared_scene::PinBuf** out) {
    hk_shared_scene::PinBuf& pin = sc->pin[sc->pin_slot];
    sc->pin_slot ^= 1;
    if (!pin.ev) HK_SCUDA(cudaEventCreateWithFlags(&pin.ev, cudaEventDisableTiming));
    if (pin.used) HK_SCUDA(cudaEventSynchronize(pin.ev));          // the copy made from this slot two calls ago
    if (pin.cap < bytes) {
        if (pin.p) cudaFreeHost(pin.p);
        pin.p = nullptr; pin.cap = 0;
        HK_SCUDA(cudaMallocHost(&pin.p, bytes + bytes / 2));
        pin.cap = bytes + bytes / 2;
    }
    *out = &pin;
    return HK_OK;
}

// SURVEY 8(f) rank 2 — the per-frame half of the scene rebuilt on the device (kernels_scene.cu) from the model matrices alone.
static int scene_update_transforms(hk_shared_scene* sc, const float* models, const float* previous_models, const float* mesh_aabbs,
                                   uint32_t instance_count, uint32_t* launches) {
    if (!sc->ready) return set_error(sc, HK_ERR_NOT_READY, "hk_scene_update_transforms needs a scene from hk_scene_upload");
    if (instance_count != sc->scene_instance_count)
        return set_error(sc, HK_ERR_INVALID_ARGUMENT, "hk_scene_update_transforms moves the instances of the last upload: their number must be unchanged "
                                                       "(a changed set goes through hk_scene_update_instances)");
    const uint32_t n = instance_count, ne = sc->scene_emissive_count;
    if (n == 0u) return HK_OK;
    if (const int rc = check_models(sc, models, 16, n, "hk_scene_update_transforms")) return rc;
    for (uint32_t i = 0; i < n; ++i)          // a non-finite mesh AABB gives a non-finite centre just as a model does
        for (int k = 0; k < 6; ++k) {
            uint32_t bits;
            memcpy(&bits, mesh_aabbs + 6 * (size_t)i + k, 4);
            if ((bits & 0x7f800000u) == 0x7f800000u)
                return set_error(sc, HK_ERR_INVALID_ARGUMENT, "hk_scene_update_transforms: instance " + std::to_string(i) +
                                                              " has a non-finite mesh AABB (entry " + std::to_string(k) + ")");
        }
    DeviceScene d = sc->scene;
    // the arrays being rebuilt in place must have bvh 0.7.1's sizes (3 m - 2 records over m >= 2 shapes, 1 over one)
    const uint32_t tlas_records = n == 1u ? 1u : 3u * n - 2u, em_records = ne == 0u ? 0u : (ne == 1u ? 1u : 3u * ne - 2u);
    if (d.instance_node_count != tlas_records || d.emissive_node_count != em_records)
        return set_error(sc, HK_ERR_UNSUPPORTED, "the uploaded TLAS / emissive BVH is not in bvh 0.7.1's flatten_custom layout: use hk_scene_update_instances");
    HK_SCUDA(cudaSetDevice(sc->device));
    const size_t mbytes = 64u * (size_t)n, abytes = 24u * (size_t)n;
    const size_t stage_bytes = mbytes * (previous_models ? 2u : 1u) + abytes;
    // pinned staging: the caller's arrays are free on return and the host does not wait for the frames in flight
    hk_shared_scene::PinBuf* slot = nullptr;
    if (const int rc = pinned_slot(sc, stage_bytes, &slot)) return rc;
    hk_shared_scene::PinBuf& pin = *slot;
    // staging layout: models | previous models (optional) | mesh AABBs — the two matrix arrays are read as float4 and must stay
    // 16-byte aligned for every n (24 n bytes of AABBs in between misaligned `previous` for odd n: a misaligned-address fault on
    // the device that the host emulation did not see)
    const size_t aoff = mbytes * (previous_models ? 2u : 1u);
    uint8_t* hp = static_cast<uint8_t*>(pin.p);
    memcpy(hp, models, mbytes);
    if (previous_models) memcpy(hp + mbytes, previous_models, mbytes);
    memcpy(hp + aoff, mesh_aabbs, abytes);
    const uint32_t nmax = n > ne ? n : ne;
    HK_SCUDA(ensure_buf(sc, sc->ibuf[14], stage_bytes));
    HK_SCUDA(ensure_buf(sc, sc->ibuf[5], mbytes));
    HK_SCUDA(ensure_buf(sc, sc->ibuf[6], 4u * (size_t)n));
    HK_SCUDA(ensure_buf(sc, sc->ibuf[17], 16u * (size_t)nmax));
    HK_SCUDA(ensure_buf(sc, sc->ibuf[18], 16u * (size_t)nmax));
    HK_SCUDA(ensure_buf(sc, sc->ibuf[19], hk_scene_bvh_scratch_bytes(nmax)));
    uint8_t* dp = static_cast<uint8_t*>(sc->ibuf[14].p);
    HK_SCUDA(cudaMemcpyAsync(dp, hp, stage_bytes, cudaMemcpyHostToDevice, sc->stream));
    HK_SCUDA(cudaEventRecord(pin.ev, sc->stream));
    pin.used = true;
    hk_instance* instances = static_cast<hk_instance*>(sc->ibuf[1].p);
    hk_emissive* emissives = static_cast<hk_emissive*>(sc->ibuf[4].p);
    float4* box_lo = static_cast<float4*>(sc->ibuf[17].p);
    float4* box_hi = static_cast<float4*>(sc->ibuf[18].p);
    hk_launch_scene_instances(n, reinterpret_cast<const float4*>(dp), previous_models ? reinterpret_cast<const float4*>(dp + mbytes) : nullptr,
                              reinterpret_cast<const float*>(dp + aoff), instances, static_cast<hk_instance_trav*>(sc->ibuf[8].p),
                              static_cast<float4*>(sc->ibuf[5].p), static_cast<uint32_t*>(sc->ibuf[6].p), box_lo, box_hi, sc->stream);
    hk_launch_build_flat_bvh(n, box_lo, box_hi, sc->ibuf[19].p, static_cast<hk_node*>(sc->ibuf[2].p),
                             reinterpret_cast<uint8_t*>(instances) + offsetof(hk_instance, node_index), (uint32_t)sizeof(hk_instance), sc->stream);
    bool wide = false;          // the 4-wide TLAS is re-derived when any attached camera walks the wide trees
    for (const hk_context* c : sc->attached) wide = wide || wide_primary(c) || wide_light(c);
    if (wide) {
        // image-exact traversal mode in use: its 4-wide TLAS is derived on the device from the records just built, into the buffers
        // upload_wide_tlas sized for these instances (leaf navigators = instance boxes, as built).  Whether it fits the walk's stack
        // is known only there: the WIDE launches read the verdict (DeviceScene::wide_state), the host never waits for it
        hk_launch_build_wide_tlas(n, static_cast<const hk_node*>(sc->ibuf[2].p), sc->wide_blas_ok, 1u + sc->wide_blas_need + 3u, sc->ibuf[16].p,
                                  static_cast<hk_wide_node*>(sc->ibuf[9].p), static_cast<uint32_t*>(sc->ibuf[12].p),
                                  static_cast<uint32_t*>(sc->ibuf[15].p), sc->stream);
    }
    if (ne) {
        hk_launch_scene_emissives(ne, emissives, instances, d.materials, d.primitives, d.vertices, box_lo, box_hi, sc->stream);
        hk_launch_build_flat_bvh(ne, box_lo, box_hi, sc->ibuf[19].p, static_cast<hk_node*>(sc->ibuf[3].p),
                                 reinterpret_cast<uint8_t*>(emissives) + offsetof(hk_emissive, node_index), (uint32_t)sizeof(hk_emissive), sc->stream);
    }
    HK_SCUDA(cudaGetLastError());
    *launches = (ne ? 4u : 2u) + (wide ? 1u : 0u);
    d.previous_models = static_cast<const float4*>(sc->ibuf[5].p);
    d.instance_moved = static_cast<const uint32_t*>(sc->ibuf[6].p);
    d.leaf_boxes_match = sc->mesh_boxes_match ? 1u : 0u;       // every navigator carries its instance's own box by construction
    d.wide_ready = 0u; d.wide_tlas_root = WIDE_EMPTY;
    if (wide) {
        d.wide_tlas = static_cast<const hk_wide_node*>(sc->ibuf[9].p);
        d.wide_instance_rank = static_cast<const uint32_t*>(sc->ibuf[12].p);
        d.wide_state = static_cast<const uint32_t*>(sc->ibuf[15].p);
        d.wide_tlas_root = n == 1u ? WIDE_LEAF : 0u;      // what build_wide returns for bvh 0.7.1's layout
        d.wide_ready = sc->wide_blas_ok ? 1u : 0u;         // the meshes' half; the TLAS's half is wide_state[0]
        sc->wide_on_device = true;
    }
    sc->scene = d;
    return HK_OK;
}

// SURVEY 8(f) rank 2, the meshes: GpuMesh::try_from for meshes added to a live scene, on the device (kernels_scene.cu).  Everything
// the kernels rely on is checked here first, in one pass over the caller's arrays, so that a refused call launches nothing and
// leaves the scene as it was.
static int scene_add_meshes(hk_shared_scene* sc, const hk_mesh_source* meshes, uint32_t n, hk_mesh_index* out, uint32_t* launches) {
    if (!sc->ready) return set_error(sc, HK_ERR_NOT_READY, "hk_scene_add_meshes needs a scene from hk_scene_upload");
    if (n == 0u) return HK_OK;
    std::vector<MeshJob> jobs(n);
    std::vector<hk_mesh_index> index(n);
    uint64_t nv_total = 0, np_total = 0, ni_total = 0, nodes_total = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const hk_mesh_source& m = meshes[i];
        auto refuse = [&](const std::string& why) {
            return set_error(sc, HK_ERR_INVALID_ARGUMENT, "hk_scene_add_meshes: mesh " + std::to_string(i) + ": " + why);
        };
        if (!m.positions || !m.position_count) return refuse("MissingAttribute(ATTRIBUTE_POSITION)");      // mod.rs:301-308
        if (!m.normals || !m.normal_count) return refuse("MissingAttribute(ATTRIBUTE_NORMAL)");
        if (!m.uvs || !m.uv_count) return refuse("MissingAttribute(ATTRIBUTE_UV_0)");
        if (m.topology != HK_TOPOLOGY_TRIANGLE_LIST && m.topology != HK_TOPOLOGY_TRIANGLE_STRIP)
            return refuse("IncompatiblePrimitiveTopology (topology " + std::to_string(m.topology) + ")");
        const uint32_t nv = std::min(m.position_count, std::min(m.normal_count, m.uv_count));     // multizip
        const bool strip = m.topology == HK_TOPOLOGY_TRIANGLE_STRIP, indexed = m.indices != nullptr;
        const uint64_t ni = indexed ? m.index_count : nv;
        if (!strip && ni % 3u != 0u) return refuse("IncompatiblePrimitiveTopology (a short chunk: " + std::to_string(ni) + " indices in a triangle list)");
        const uint64_t np = strip ? (ni >= 3u ? ni - 2u : 0u) : ni / 3u;
        if (np == 0u) return refuse("NoPrimitive");
        if (np >= 0x80000000ull) return refuse(std::to_string(np) + " primitives do not fit the BLAS leaf flag (0x80000000)");
        if (indexed)
            for (uint32_t k = 0; k < m.index_count; ++k)
                if (m.indices[k] >= nv)
                    return refuse("index " + std::to_string(k) + " = " + std::to_string(m.indices[k]) + " is not below the vertex count " + std::to_string(nv));
        const uint64_t nodes = np == 1u ? 1u : 3u * np - 2u;
        const uint64_t v0 = (uint64_t)sc->scene_vertex_count + nv_total, p0 = (uint64_t)sc->scene_primitive_count + np_total;
        const uint64_t n0 = (uint64_t)sc->scene_asset_node_count + nodes_total;
        if (v0 + nv > 0xFFFFFFFFull || p0 + np > 0xFFFFFFFFull || n0 + nodes > 0xFFFFFFFFull || ni_total + (indexed ? ni : 0u) > 0xFFFFFFFFull)
            return refuse("the scene's vertex / primitive / BLAS record offsets would not fit 32 bits");
        index[i] = hk_mesh_index{(uint32_t)v0, (uint32_t)p0, (uint32_t)n0, (uint32_t)nodes};
        jobs[i] = MeshJob{(uint32_t)nv_total, (uint32_t)ni_total, indexed ? 1u : 0u, strip ? 1u : 0u, (uint32_t)np_total, (uint32_t)np,
                          (uint32_t)v0, (uint32_t)p0, (uint32_t)n0};
        nv_total += nv; np_total += np; nodes_total += nodes;
        if (indexed) ni_total += ni;
    }
    HK_SCUDA(cudaSetDevice(sc->device));
    // staging: jobs | positions | normals | uvs | indices, each 16-byte aligned
    auto align16 = [](size_t x) { return (x + 15u) & ~(size_t)15u; };
    const size_t o_pos = align16(sizeof(MeshJob) * (size_t)n), o_nrm = o_pos + align16(12u * nv_total), o_uv = o_nrm + align16(12u * nv_total);
    const size_t o_idx = o_uv + align16(8u * nv_total), stage_bytes = o_idx + align16(4u * ni_total);
    hk_shared_scene::PinBuf* slot = nullptr;
    if (const int rc = pinned_slot(sc, stage_bytes, &slot)) return rc;
    uint8_t* hp = static_cast<uint8_t*>(slot->p);
    memcpy(hp, jobs.data(), sizeof(MeshJob) * (size_t)n);
    for (uint32_t i = 0; i < n; ++i) {
        const hk_mesh_source& m = meshes[i];
        const MeshJob& j = jobs[i];
        const size_t nv = (i + 1u < n ? jobs[i + 1u].src_vertex : nv_total) - j.src_vertex;
        memcpy(hp + o_pos + 12u * (size_t)j.src_vertex, m.positions, 12u * nv);
        memcpy(hp + o_nrm + 12u * (size_t)j.src_vertex, m.normals, 12u * nv);
        memcpy(hp + o_uv + 8u * (size_t)j.src_vertex, m.uvs, 8u * nv);
        if (j.indexed) memcpy(hp + o_idx + 4u * (size_t)j.src_index, m.indices, 4u * (size_t)m.index_count);
    }
    // the scene's buffers, grown where needed: a new allocation takes the records the frames read so far, in stream order.  Every
    // allocation is made before anything is copied or released, so that a failed one leaves the scene on its old buffers.
    const size_t rec[3] = {sizeof(hk_vertex), sizeof(hk_primitive), sizeof(hk_node)};
    const uint64_t have[3] = {sc->scene_vertex_count, sc->scene_primitive_count, sc->scene_asset_node_count};
    const uint64_t add[3] = {nv_total, np_total, nodes_total};
    size_t need[3], cap[3];
    void* grown[3] = {nullptr, nullptr, nullptr};
    void* block = nullptr;       // staged copy + build scratch, released in stream order behind the build
    const size_t scratch_off = align16(stage_bytes);
    cudaError_t e = malloc_on_stream(&block, scratch_off + hk_blas_scratch_bytes((uint32_t)np_total), sc->stream);
    for (int b = 0; b < 3 && e == cudaSuccess; ++b) {
        need[b] = rec[b] * (size_t)(have[b] + add[b]) + 64u;        // +64: 16-byte vector loads at the tail stay in bounds
        cap[b] = need[b] + need[b] / 2u;
        if (sc->mbuf[b].cap < need[b]) e = malloc_on_stream(&grown[b], cap[b], sc->stream);
    }
    if (e != cudaSuccess) {
        for (void* p : grown) if (p) free_on_stream(p, sc->stream);
        if (block) free_on_stream(block, sc->stream);
        HK_SCUDA(e);
    }
    void* retired[3] = {nullptr, nullptr, nullptr};      // released behind the build, once the new pointers are published
    for (int b = 0; b < 3; ++b) {
        if (!grown[b]) continue;
        hk_shared_scene::MeshBuf& mb = sc->mbuf[b];
        HK_SCUDA(cudaMemcpyAsync(grown[b], mb.p, rec[b] * (size_t)have[b], cudaMemcpyDeviceToDevice, sc->stream));
        HK_SCUDA(cudaMemsetAsync(static_cast<uint8_t*>(grown[b]) + need[b] - 64u, 0, 64u, sc->stream));
        if (mb.async) retired[b] = mb.p;      // an upload's buffer goes with the upload's allocations
        mb = hk_shared_scene::MeshBuf{grown[b], cap[b], true};
    }
    uint8_t* dp = static_cast<uint8_t*>(block);
    HK_SCUDA(cudaMemcpyAsync(dp, hp, stage_bytes, cudaMemcpyHostToDevice, sc->stream));
    HK_SCUDA(cudaEventRecord(slot->ev, sc->stream));
    slot->used = true;
    hk_vertex* vertices = static_cast<hk_vertex*>(sc->mbuf[0].p);
    hk_primitive* primitives = static_cast<hk_primitive*>(sc->mbuf[1].p);
    hk_node* nodes = static_cast<hk_node*>(sc->mbuf[2].p);
    *launches = (uint32_t)hk_launch_build_meshes(n, reinterpret_cast<const MeshJob*>(dp), (uint32_t)nv_total, (uint32_t)np_total,
                                                  reinterpret_cast<const float*>(dp + o_pos), reinterpret_cast<const float*>(dp + o_nrm),
                                                  reinterpret_cast<const float*>(dp + o_uv), reinterpret_cast<const uint32_t*>(dp + o_idx),
                                                  dp + scratch_off, vertices, primitives, nodes, sc->stream);
    HK_SCUDA(cudaGetLastError());
    free_on_stream(block, sc->stream);
    // host copies that validate later instance updates; the new BLAS ranges are checked by construction
    sc->host_primitive_vertex_index.resize(3u * (size_t)(sc->scene_primitive_count + np_total));
    sc->host_primitive_box.resize(6u * (size_t)(sc->scene_primitive_count + np_total));
    for (uint32_t i = 0; i < n; ++i) {
        const hk_mesh_source& m = meshes[i];
        const MeshJob& j = jobs[i];
        for (uint32_t p = 0; p < j.shapes; ++p) {
            uint32_t id[3];
            for (uint32_t k = 0; k < 3u; ++k) {
                const uint32_t at = j.strip ? p + k : 3u * p + k;
                id[k] = j.indexed ? m.indices[at] : at;
            }
            if (j.strip && (p & 1u)) std::swap(id[0], id[1]);
            const size_t g = (size_t)j.dst_primitive + p;
            for (int c = 0; c < 3; ++c) {
                sc->host_primitive_vertex_index[3u * g + c] = id[c];
                const float a = m.positions[3u * (size_t)id[0] + c], b = m.positions[3u * (size_t)id[1] + c], e = m.positions[3u * (size_t)id[2] + c];
                sc->host_primitive_box[6u * g + c] = fminf(a, fminf(b, e));
                sc->host_primitive_box[6u * g + 3u + c] = fmaxf(a, fmaxf(b, e));
            }
        }
        sc->mesh_range_checked.insert({index[i].vertex, index[i].primitive, index[i].node_offset, index[i].node_count});
        out[i] = index[i];
    }
    sc->scene_vertex_count += (uint32_t)nv_total;
    sc->scene_primitive_count += (uint32_t)np_total;
    sc->scene_asset_node_count += (uint32_t)nodes_total;
    DeviceScene d = sc->scene;          // published behind the launches above: frames enqueued from now on read the grown buffers
    d.vertices = vertices; d.primitives = primitives; d.asset_nodes = nodes;
    sc->scene = d;
    for (void* p : retired) if (p) free_on_stream(p, sc->stream);
    return HK_OK;
}

// {ready, stack need, TLAS node count} of the scene's 4-wide TLAS.  After a derivation on the device they exist only there
// and are read back: a query (hk_get_stats, hk_scene_readback), not a frame call, so it may wait for the scene's stream.
static cudaError_t wide_tlas_state(hk_shared_scene* sc, uint32_t out[3]) {
    if (!sc->wide_on_device) {
        out[0] = sc->scene.wide_ready; out[1] = sc->wide_stack_need; out[2] = sc->wide_tlas_node_count;
        return cudaSuccess;
    }
    cudaError_t e = cudaMemcpyAsync(out, sc->ibuf[15].p, 3u * sizeof(uint32_t), cudaMemcpyDeviceToHost, sc->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(sc->stream);
    return e;
}

// Test / debugging aid: the per-frame scene buffers as they are on the device (what hk_scene_update_transforms built in place).
static bool scene_buffer(hk_shared_scene* sc, int which, const void** src, size_t* have) {
    const DeviceScene& d = sc->scene;
    switch (which) {
        case HK_SCENE_WIDE_TLAS: {
            uint32_t state[3] = {0u, 0u, 0u};
            if (wide_tlas_state(sc, state) != cudaSuccess) return false;
            *src = d.wide_tlas; *have = d.wide_tlas ? sizeof(hk_wide_node) * (size_t)state[2] : 0u;
            return true;
        }
        case HK_SCENE_WIDE_INSTANCE_RANK:
            *src = d.wide_instance_rank; *have = d.wide_instance_rank ? 4u * (size_t)sc->scene_instance_count : 0u; return true;
        case HK_SCENE_INSTANCES: *src = d.instances; *have = sizeof(hk_instance) * (size_t)sc->scene_instance_count; return true;
        case HK_SCENE_INSTANCE_NODES: *src = d.instance_nodes; *have = sizeof(hk_node) * (size_t)d.instance_node_count; return true;
        case HK_SCENE_EMISSIVES: *src = d.emissives; *have = sizeof(hk_emissive) * (size_t)sc->scene_emissive_count; return true;
        case HK_SCENE_EMISSIVE_NODES: *src = d.emissive_nodes; *have = sizeof(hk_node) * (size_t)d.emissive_node_count; return true;
        case HK_SCENE_PREVIOUS_MODELS: *src = d.previous_models; *have = d.previous_models ? 64u * (size_t)sc->scene_instance_count : 0u; return true;
        case HK_SCENE_INSTANCE_MOVED: *src = d.instance_moved; *have = d.instance_moved ? 4u * (size_t)sc->scene_instance_count : 0u; return true;
        case HK_SCENE_VERTICES: *src = d.vertices; *have = sizeof(hk_vertex) * (size_t)sc->scene_vertex_count; return true;
        case HK_SCENE_PRIMITIVES: *src = d.primitives; *have = sizeof(hk_primitive) * (size_t)sc->scene_primitive_count; return true;
        case HK_SCENE_ASSET_NODES: *src = d.asset_nodes; *have = sizeof(hk_node) * (size_t)sc->scene_asset_node_count; return true;
        default: return false;
    }
}

// The scene that a context's hk_scene_upload / hk_scene_update_* write: its private one.  A context rendering a shared scene is
// refused (the scene is updated through its handle); a context without a scene gets a private one on its own stream at upload.
static int private_scene(hk_context* ctx, bool create, hk_shared_scene** out) {
    *out = nullptr;
    if (ctx->sc && ctx->sc->owner != ctx)
        return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "the context renders a shared scene: upload and update it through its hk_shared_scene handle");
    if (!ctx->sc && create) {
        hk_shared_scene* sc = new hk_shared_scene();
        sc->device = ctx->device;
        sc->stream = ctx->stream;
        sc->handle = false;
        sc->owner = ctx;
        attach_scene(ctx, sc);       // same stream: records nothing, cannot fail
    }
    *out = ctx->sc;
    return HK_OK;
}
static int scene_result(hk_context* ctx, hk_shared_scene* sc, int rc) {   // a scene's error, reported on the context that asked
    if (rc != HK_OK) ctx->error = sc->error;
    return rc;
}
static int do_upload(hk_shared_scene* sc, const hk_scene_desc* s) {
    scene_begin_write(sc);
    const int rc = scene_upload(sc, s);
    scene_end_write(sc);
    return rc;
}
static int do_update_instances(hk_shared_scene* sc, const hk_scene_desc* s) {
    if (!sc->ready) return set_error(sc, HK_ERR_NOT_READY, "hk_scene_update_instances needs a scene from hk_scene_upload");
    scene_begin_write(sc);
    const int rc = scene_update_instances(sc, s);
    scene_end_write(sc);
    return rc;
}
static int do_update_transforms(hk_shared_scene* sc, const float* models, const float* previous_models, const float* mesh_aabbs,
                                uint32_t instance_count, uint32_t* launches) {
    if (!sc->ready) return set_error(sc, HK_ERR_NOT_READY, "hk_scene_update_transforms needs a scene from hk_scene_upload");
    scene_begin_write(sc);
    const int rc = scene_update_transforms(sc, models, previous_models, mesh_aabbs, instance_count, launches);
    scene_end_write(sc);
    return rc;
}
static int do_add_meshes(hk_shared_scene* sc, const hk_mesh_source* meshes, uint32_t n, hk_mesh_index* out, uint32_t* launches) {
    if (!sc->ready) return set_error(sc, HK_ERR_NOT_READY, "hk_scene_add_meshes needs a scene from hk_scene_upload");
    scene_begin_write(sc);
    const int rc = scene_add_meshes(sc, meshes, n, out, launches);
    scene_end_write(sc);
    return rc;
}

extern "C" {

int hk_scene_upload(hk_context* ctx, const hk_scene_desc* s) {
    if (!ctx || !s) return HK_ERR_INVALID_ARGUMENT;
    hk_shared_scene* sc = nullptr;
    int rc = private_scene(ctx, true, &sc);
    if (rc != HK_OK) return rc;
    return scene_result(ctx, sc, do_upload(sc, s));
}
int hk_scene_update_instances(hk_context* ctx, const hk_scene_desc* s) {
    if (!ctx || !s) return HK_ERR_INVALID_ARGUMENT;
    hk_shared_scene* sc = nullptr;
    int rc = private_scene(ctx, false, &sc);
    if (rc != HK_OK) return rc;
    if (!sc) return set_error(ctx, HK_ERR_NOT_READY, "hk_scene_update_instances needs a scene from hk_scene_upload");
    return scene_result(ctx, sc, do_update_instances(sc, s));
}
int hk_scene_update_transforms(hk_context* ctx, const float* models, const float* previous_models, const float* mesh_aabbs, uint32_t instance_count) {
    if (!ctx || (instance_count && (!models || !mesh_aabbs))) return HK_ERR_INVALID_ARGUMENT;
    hk_shared_scene* sc = nullptr;
    int rc = private_scene(ctx, false, &sc);
    if (rc != HK_OK) return rc;
    if (!sc) return set_error(ctx, HK_ERR_NOT_READY, "hk_scene_update_transforms needs a scene from hk_scene_upload");
    uint32_t launches = 0;
    rc = scene_result(ctx, sc, do_update_transforms(sc, models, previous_models, mesh_aabbs, instance_count, &launches));
    ctx->launches += launches;
    return rc;
}

int hk_scene_add_meshes(hk_context* ctx, const hk_mesh_source* meshes, uint32_t mesh_count, hk_mesh_index* out) {
    if (!ctx || (mesh_count && (!meshes || !out))) return HK_ERR_INVALID_ARGUMENT;
    hk_shared_scene* sc = nullptr;
    int rc = private_scene(ctx, false, &sc);
    if (rc != HK_OK) return rc;
    if (!sc) return set_error(ctx, HK_ERR_NOT_READY, "hk_scene_add_meshes needs a scene from hk_scene_upload");
    uint32_t launches = 0;
    rc = scene_result(ctx, sc, do_add_meshes(sc, meshes, mesh_count, out, &launches));
    ctx->launches += launches;
    return rc;
}

int hk_shared_scene_create(hk_shared_scene** out, int cuda_device, void* cuda_stream) {
    if (!out) return set_error(nullptr, HK_ERR_INVALID_ARGUMENT, "out == NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return set_error(nullptr, HK_ERR_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(e) +
                                                   " (this library has no CPU fallback)");
    if (cuda_device < 0 || cuda_device >= ndev) return set_error(nullptr, HK_ERR_INVALID_ARGUMENT, "bad cuda_device");
    e = cudaSetDevice(cuda_device);
    if (e != cudaSuccess) return set_error(nullptr, HK_ERR_CUDA, cudaGetErrorString(e));
    hk_shared_scene* sc = new hk_shared_scene();
    sc->device = cuda_device;
    if (cuda_stream) sc->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
    else {
        e = cudaStreamCreateWithFlags(&sc->stream, cudaStreamNonBlocking);
        if (e != cudaSuccess) { delete sc; return set_error(nullptr, HK_ERR_CUDA, cudaGetErrorString(e)); }
        sc->own_stream = true;
    }
    *out = sc;
    return HK_OK;
}
void hk_shared_scene_destroy(hk_shared_scene* sc) {
    if (!sc) return;
    sc->handle = false;
    if (sc->attached.empty()) scene_free(sc);
}
int hk_shared_scene_upload(hk_shared_scene* sc, const hk_scene_desc* s) {
    if (!sc || !s) return HK_ERR_INVALID_ARGUMENT;
    return do_upload(sc, s);
}
int hk_shared_scene_update_instances(hk_shared_scene* sc, const hk_scene_desc* s) {
    if (!sc || !s) return HK_ERR_INVALID_ARGUMENT;
    return do_update_instances(sc, s);
}
int hk_shared_scene_update_transforms(hk_shared_scene* sc, const float* models, const float* previous_models, const float* mesh_aabbs,
                                      uint32_t instance_count) {
    if (!sc || (instance_count && (!models || !mesh_aabbs))) return HK_ERR_INVALID_ARGUMENT;
    uint32_t launches = 0;
    return do_update_transforms(sc, models, previous_models, mesh_aabbs, instance_count, &launches);
}
int hk_shared_scene_add_meshes(hk_shared_scene* sc, const hk_mesh_source* meshes, uint32_t mesh_count, hk_mesh_index* out) {
    if (!sc || (mesh_count && (!meshes || !out))) return HK_ERR_INVALID_ARGUMENT;
    uint32_t launches = 0;
    return do_add_meshes(sc, meshes, mesh_count, out, &launches);
}
const char* hk_shared_scene_last_error(hk_shared_scene* sc) { return sc ? sc->error.c_str() : g_create_error.c_str(); }

int hk_context_attach_scene(hk_context* ctx, hk_shared_scene* sc) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    if (sc && sc->device != ctx->device) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "the scene lives on another device than the context");
    if (sc && sc->owner) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "a private scene cannot be attached to another context");
    if (sc == ctx->sc) return HK_OK;
    HK_CUDA(cudaSetDevice(ctx->device));
    detach_scene(ctx);
    return sc ? attach_scene(ctx, sc) : HK_OK;
}

int hk_scene_buffer_bytes(hk_context* ctx, int which, size_t* bytes) {
    if (!ctx || !bytes) return HK_ERR_INVALID_ARGUMENT;
    if (!scene_ready(ctx)) return set_error(ctx, HK_ERR_NOT_READY, "no scene");
    const void* src = nullptr;
    if (!scene_buffer(ctx->sc, which, &src, bytes)) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "unknown scene buffer");
    return HK_OK;
}
int hk_scene_readback(hk_context* ctx, int which, void* host, size_t bytes) {
    if (!ctx || (!host && bytes)) return HK_ERR_INVALID_ARGUMENT;
    if (!scene_ready(ctx)) return set_error(ctx, HK_ERR_NOT_READY, "no scene");
    const void* src = nullptr;
    size_t have = 0;
    if (!scene_buffer(ctx->sc, which, &src, &have)) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "unknown scene buffer");
    if (bytes != have) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "size mismatch");
    HK_CUDA(cudaSetDevice(ctx->device));
    if (bytes) HK_CUDA(cudaMemcpyAsync(host, src, bytes, cudaMemcpyDeviceToHost, ctx->sc->stream));   // behind the scene's updates
    HK_CUDA(cudaStreamSynchronize(ctx->sc->stream));
    return HK_OK;
}

int hk_set_noise(hk_context* ctx, const uint8_t* rgba) {
    if (!ctx || !rgba) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    const size_t bytes = 16u * 64u * 64u * 4u;
    if (!ctx->noise) { void* p = nullptr; HK_CUDA(cudaMalloc(&p, bytes)); ctx->noise = reinterpret_cast<uint8_t*>(p); }
    HK_CUDA(cudaMemcpyAsync(ctx->noise, rgba, bytes, cudaMemcpyHostToDevice, ctx->stream));
    HK_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->noise_ready = true;
    return HK_OK;
}

// ------------------------------------------------------------------------------------------------ scheduling
static int make_params(hk_context* ctx, const hk_frame_inputs* in, KParams& P) {
    if (!ctx || !in) return HK_ERR_INVALID_ARGUMENT;
    if (!scene_ready(ctx) || !ctx->noise_ready) return set_error(ctx, HK_ERR_NOT_READY, "scene or noise not uploaded");
    if (!ctx->planes_ready) return set_error(ctx, HK_ERR_NOT_READY, "per-pixel planes are not allocated (a resize failed)");
    const bool ratio1 = in->frame.upscale_ratio == 1.0f;
    if (!(in->frame.upscale_ratio >= 1.0f && in->frame.upscale_ratio <= 2.0f))
        return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "upscale_ratio must be in [1, 2] (Upscale::ratio clamps, lib.rs:501-505)");
    if (!ratio1 && !ctx->full_frame)
        return set_error(ctx, HK_ERR_UNSUPPORTED, "upscale_ratio != 1 needs a full-frame context (no tile)");
    if (in->temporal_upscalers && !ctx->full_frame && (!ctx->tile_upscalers || ctx->motion_margin < RING_TONE))
        return set_error(ctx, HK_ERR_UNSUPPORTED, "the temporal upscalers on a tile need a full-frame context, or hk_context_enable_tile_upscalers "
                                                  "and a motion margin of at least 4 pixels + the per-frame motion");
    if (in->temporal_upscalers && in->fsr1 && in->smaa_tu4x)
        return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "fsr1 and smaa_tu4x are the two variants of one enum (Upscale, lib.rs:475-490)");
    if (in->temporal_upscalers && in->fsr1 && !ctx->full_frame)
        return set_error(ctx, HK_ERR_UNSUPPORTED, "FSR1 needs a full-frame context (no tile)");
    if (in->frame.direct_validate_interval == 0 || in->frame.emissive_validate_interval == 0)
        return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "validate interval must be >= 1");
    if (cudaSetDevice(ctx->device) != cudaSuccess) return set_error(ctx, HK_ERR_CUDA, "cudaSetDevice");
    P.in = *in;
    P.scene = ctx->sc->scene;      // the attached scene as it is now (stream order: SceneUse)
    P.planes = ctx->planes;
    P.planes.pos_depth = ctx->planes.pos_depth_db[ctx->gbuffer_current];
    P.planes.velocity_uv = ctx->planes.velocity_uv_db[ctx->gbuffer_current];
    // tone_mapping_output alternates every frame in the reference (post_process.rs:979); only smaa_tu4x reads the other one,
    // so the pointer hk_get_output hands out stays fixed unless the temporal upscalers are on
    P.planes.tone_mapped = ctx->planes.tone_mapped_db[in->temporal_upscalers ? (in->frame.number % 2u) : 0u];
    ctx->last_upscalers = in->temporal_upscalers != 0;
    P.band = ctx->band;
    P.ratio1 = ratio1 ? 1 : 0;
    P.jitter_sign = ((in->frame.number & 1u) == 0u) ? -1.0f : 1.0f;
    P.ratio_m1 = in->frame.upscale_ratio - 1.0f;
    P.gbuffer_current = ctx->gbuffer_current;
    P.frame_target = ratio1 ? ctx->frame_target : nullptr;   // the assembled frame has the output size = render size at ratio 1
    P.frame_pitch = ctx->frame_pitch;
    P.tile_images = (!ctx->full_frame && in->temporal_upscalers) ? 1 : 0;
    if (!ratio1) {   // scaled_size = (ratio.recip() * size).ceil(), light.rs:622-624; render-size planes use stride RW
        const float scale = 1.0f / in->frame.upscale_ratio;
        P.band.RW = (int)ceilf(scale * (float)P.band.W);
        P.band.RH = (int)ceilf(scale * (float)P.band.H);
        P.band.RS = P.band.RW;
    }
    {   // upscale_output after SMAA TU4x: create_texture(format, scale) with scale = ratio.recip() * 2 (post_process.rs:663-667,711,717)
        const float scale2 = (1.0f / in->frame.upscale_ratio) * 2.0f;
        P.band.OW = (int)ceilf((float)P.band.W * scale2);
        P.band.OH = (int)ceilf((float)P.band.H * scale2);
    }
    ctx->last_up_w = P.band.OW; ctx->last_up_h = P.band.OH; ctx->last_scaled = !ratio1;
    P.inv_rw = 1.0f / (float)P.band.RW; P.inv_rh = 1.0f / (float)P.band.RH;
    ctx->last_render_w = P.band.RW; ctx->last_render_h = P.band.RH; ctx->last_smaa = in->smaa_tu4x != 0; ctx->last_number = in->frame.number;
    ctx->last_fsr = in->temporal_upscalers && in->fsr1;
    P.counters = ctx->count_rays ? ctx->counters : nullptr;
    P.noise = ctx->noise;
    float s, c;
    hk::sincos_(in->frame.solar_angle, &s, &c);
    P.cos_solar_angle = c;
    P.random_frame = hk::random_float(in->frame.number);
    P.spatial_tables = ctx->spatial_tables;
    return HK_OK;
}
static void rows_deferred(const hk_context* ctx, KParams& P, int ghost) {   // deferred-space launches (G-buffer, albedo)
    const Band& b = ctx->band;
    P.band.cx0 = b.cx0; P.band.cx1 = b.cx1; P.band.r0 = b.r0; P.band.r1 = b.r1;
    P.row_lo = b.r0 - ghost < b.a0 ? b.a0 : b.r0 - ghost;
    P.row_hi = b.r1 + ghost > b.a1 ? b.a1 : b.r1 + ghost;
    P.col_lo = b.cx0 - ghost < b.ax0 ? b.ax0 : b.cx0 - ghost;
    P.col_hi = b.cx1 + ghost > b.ax1 ? b.ax1 : b.cx1 + ghost;
}
static void rows(const hk_context* ctx, KParams& P, int ghost) {   // owned rectangle grown by `ghost`, clamped to the allocation
    if (!P.ratio1) {   // full-frame context at render size: no ghosts, the owned rectangle is the render rectangle
        P.band.cx0 = 0; P.band.cx1 = P.band.RW; P.band.r0 = 0; P.band.r1 = P.band.RH;
        P.row_lo = 0; P.row_hi = P.band.RH; P.col_lo = 0; P.col_hi = P.band.RW;
        return;
    }
    const Band& b = ctx->band;
    P.row_lo = b.r0 - ghost < b.a0 ? b.a0 : b.r0 - ghost;
    P.row_hi = b.r1 + ghost > b.a1 ? b.a1 : b.r1 + ghost;
    P.col_lo = b.cx0 - ghost < b.ax0 ? b.ax0 : b.cx0 - ghost;
    P.col_hi = b.cx1 + ghost > b.ax1 ? b.ax1 : b.cx1 + ghost;
}
// Which rays walk the 4-wide trees (hk_wide.cuh).  The ordered walk is meant for the coherent closest-hit rays of the prepass; the
// incoherent rays of the light passes keep the flat walk, whose kernels are instruction-fetch bound and would grow by the walk's code;
// a scene as small as cornell gains nothing either way.
#ifndef HK_WIDE_MIN_NODES
#define HK_WIDE_MIN_NODES 256
#endif
static bool wide_primary(const hk_context* ctx) {
    if (!scene_ready(ctx) || !ctx->sc->scene.wide_ready) return false;
    if (ctx->wide_traversal == 3) return true;
    return ctx->wide_traversal == 1 && ctx->sc->wide_blas_node_count + ctx->sc->wide_tlas_node_count >= (uint32_t)HK_WIDE_MIN_NODES;
}
static bool wide_light(const hk_context* ctx) { return scene_ready(ctx) && ctx->sc->scene.wide_ready && ctx->wide_traversal == 3; }

static int check_launch(hk_context* ctx) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(ctx, HK_ERR_CUDA, std::string("kernel launch: ") + cudaGetErrorString(e));
    return HK_OK;
}

struct KernelTimer {  // brackets one launch (on `st`, the context's stream by default) with events when pass timing is on
    hk_context* c; int k; cudaStream_t s;
    KernelTimer(hk_context* ctx, int kernel, cudaStream_t st = nullptr) : c(ctx), k(kernel), s(st ? st : ctx->stream) {
        c->launches += 1;
        if (c->time_only >= 0) {
            if (c->time_only == k && c->ring[0][0]) { cudaEventRecord(c->ring[c->ring_frames % hk_context::RING][0], s); c->ring_hit = true; }
        } else if (c->time_passes) { cudaEventRecord(c->kev[k][0], s); c->kran[k] = true; }
    }
    ~KernelTimer() {
        if (c->time_only >= 0) {
            if (c->time_only == k && c->ring[0][0]) cudaEventRecord(c->ring[c->ring_frames % hk_context::RING][1], s);
        } else if (c->time_passes) cudaEventRecord(c->kev[k][1], s);
    }
};

static int run_prepass(hk_context* ctx, KParams& P) {
    // prepass_textures_system swaps current <-> previous before rendering (prepass.rs:427)
    ctx->gbuffer_current ^= 1;
    P.gbuffer_current = ctx->gbuffer_current;
    P.planes.pos_depth = ctx->planes.pos_depth_db[ctx->gbuffer_current];
    P.planes.velocity_uv = ctx->planes.velocity_uv_db[ctx->gbuffer_current];
    rows_deferred(ctx, P, GHOST_TEMPORAL + ctx->motion_margin);
    { KernelTimer t(ctx, HK_K_GBUFFER); hk_launch_gbuffer(P, ctx->count_rays, wide_primary(ctx), ctx->stream); }
    return check_launch(ctx);
}
static int ring_of(const KParams& P) { return P.tile_images ? RING_TONE : 0; }   // extra reach of every pass when a tile feeds the upscalers
// spatial_reuse of one pipeline: the TMA-tiled kernel when descriptors exist and render space == G-buffer space, else the gather form
static void launch_spatial(hk_context* ctx, const KParams& P, bool emissive, cudaStream_t st = nullptr) {
    const int v = emissive ? 1 : 0, parity = 1 - (int)(P.in.frame.number & 1u);
    const bool tiled = ctx->tile_maps_ready && ctx->tiled_spatial;
    hk_launch_spatial(P, emissive, tiled ? &ctx->tm_depth[v] : nullptr, tiled ? &ctx->tm_q3[v][parity] : nullptr, ctx->spatial_tables_host[v],
                      st ? st : ctx->stream);
}
static const TileMap* denoise_maps(hk_context* ctx, int level) { return (ctx->tile_maps_ready && ctx->tiled_denoise) ? ctx->tm_denoise[level] : nullptr; }
static int run_light(hk_context* ctx, KParams& P) {  // LightNode::run order, light.rs:645-699 (albedo is fused in the prepass)
    const hk_frame_uniform& f = P.in.frame;
    const int GHOST_SPATIAL = ::GHOST_SPATIAL + ring_of(P);
    // The three pipelines read the same G-buffer and write only their own signal's planes (DESIGN.md §4a-6).  The indirect one,
    // with a scatter scratch of its own, runs on indirect_stream beside the sun and emissive ones: each branch's CTAs fill the SMs
    // the other leaves idle while a kernel drains at a launch boundary.  Per-kernel pass timing keeps the serial order on one stream,
    // so that each bracket holds one kernel alone.
    const bool serial = ctx->time_passes && ctx->time_only < 0;
    const cudaStream_t side = serial ? ctx->stream : ctx->indirect_stream;
    KParams I = P;   // rows() rewrites the launch rectangle: each branch has its own copy
    I.planes.scatter_key = ctx->indirect_scatter_key;
    I.planes.scatter_value = ctx->indirect_scatter_value;
    auto indirect = [&]() {
        rows(ctx, I, GHOST_TEMPORAL + ctx->motion_margin);
        { KernelTimer t(ctx, HK_K_INDIRECT, side);   // the per-pixel form's two kernels (path, then ReSTIR tail) count as one launch, as the pooled one
          if (ctx->pooled_indirect) hk_launch_indirect_pool(I, f.indirect_bounces >= 2, ctx->count_rays, side);
          else hk_launch_indirect(I, f.indirect_bounces >= 2, ctx->count_rays, wide_light(ctx), side);
          hk_launch_scatter_resolve(I, 2, side); ctx->launches += 1; }
        if (f.indirect_spatial_reuse) { rows(ctx, I, GHOST_SPATIAL); KernelTimer t(ctx, HK_K_INDIRECT_SPATIAL, side); launch_spatial(ctx, I, false, side); }
    };
    if (!serial) {
        HK_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
        HK_CUDA(cudaStreamWaitEvent(side, ctx->ev_fork, 0));
        indirect();
    }
    rows(ctx, P, GHOST_TEMPORAL + ctx->motion_margin);
    // each temporal pass is followed by the resolve of its scatter writes (all allocated rows can be targets)
    { KernelTimer t(ctx, HK_K_DIRECT); hk_launch_direct(P, false, ctx->count_rays, wide_light(ctx), ctx->stream);
      hk_launch_scatter_resolve(P, 0, ctx->stream); ctx->launches += 1; }
    { KernelTimer t(ctx, HK_K_EMISSIVE); hk_launch_direct(P, true, ctx->count_rays, wide_light(ctx), ctx->stream);
      hk_launch_scatter_resolve(P, 1, ctx->stream); ctx->launches += 1; }
    if (f.emissive_spatial_reuse) { rows(ctx, P, GHOST_SPATIAL); KernelTimer t(ctx, HK_K_EMISSIVE_SPATIAL); launch_spatial(ctx, P, true); }
    if (serial) indirect();
    else {   // join before the node returns: the post node, read-backs, scene updates and hk_sync order behind `stream` alone
        HK_CUDA(cudaEventRecord(ctx->ev_join, side));
        HK_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    }
    return check_launch(ctx);
}
// the kernels below overwrite the final images: a pipelined read-back of the previous frame must have left them first
static void order_behind_copy(hk_context* ctx) {
    if (!ctx->copy_in_flight) return;
    cudaStreamWaitEvent(ctx->stream, ctx->ev_copied, 0);
    ctx->copy_in_flight = false;
}
static int run_post(hk_context* ctx, KParams& P, bool fuse) {  // PostProcessNode::run, post_process.rs:1190-1234
    const int ring = ring_of(P);
    const int GHOST_DEMOD = ::GHOST_DEMOD + ring, GHOST_L0 = ::GHOST_L0 + ring, GHOST_L1 = ::GHOST_L1 + ring, GHOST_L2 = ::GHOST_L2 + ring;
    if (P.in.denoise) {
        const int signals = (P.in.frame.indirect_bounces == 0) ? 2 : 3;  // post_process.rs:949-954
        { rows(ctx, P, GHOST_DEMOD); KernelTimer t(ctx, HK_K_DEMODULATION); hk_launch_demodulation(P, signals, ctx->stream); }
        { rows(ctx, P, GHOST_L0); KernelTimer t(ctx, HK_K_DENOISE_0); hk_launch_denoise_level(P, 0, signals, false, false, denoise_maps(ctx, 0), ctx->stream); }
        { rows(ctx, P, GHOST_L1); KernelTimer t(ctx, HK_K_DENOISE_1); hk_launch_denoise_level(P, 1, signals, false, false, denoise_maps(ctx, 1), ctx->stream); }
        { rows(ctx, P, GHOST_L2); KernelTimer t(ctx, HK_K_DENOISE_2); hk_launch_denoise_level(P, 2, signals, false, false, denoise_maps(ctx, 2), ctx->stream); }
        if (fuse) order_behind_copy(ctx);
        { rows(ctx, P, ring); KernelTimer t(ctx, HK_K_DENOISE_3);
          hk_launch_denoise_level(P, 3, signals, fuse, !fuse || ctx->keep_intermediates, denoise_maps(ctx, 3), ctx->stream); }
        if (!fuse) { order_behind_copy(ctx); KernelTimer t(ctx, HK_K_TONE_MAPPING); hk_launch_tone_mapping(P, ctx->stream); }
    } else {
        rows(ctx, P, ring);
        order_behind_copy(ctx);
        KernelTimer t(ctx, HK_K_TONE_MAPPING);
        hk_launch_tone_mapping(P, ctx->stream);
    }
    if (P.in.temporal_upscalers) {   // post_process.rs:1236-1277
        const bool smaa = P.in.smaa_tu4x != 0;
        if (smaa) {
            KernelTimer t(ctx, HK_K_SMAA_TU4X);
            rows(ctx, P, P.tile_images ? RING_SMAA : 0);
            hk_launch_smaa_tu4x(P, ctx->stream);
            rows(ctx, P, P.tile_images ? RING_EXTRAPOLATE : 0);
            hk_launch_smaa_tu4x_extrapolate(P, ctx->stream);
            ctx->launches += 1;
        }
        if (P.in.taa_jitter) {   // over the output pixels of the owned rectangle
            rows(ctx, P, 0);
            const int k = smaa ? 2 : 1;
            P.row_lo *= k; P.row_hi *= k; P.col_lo *= k; P.col_hi *= k;
            KernelTimer t(ctx, HK_K_TAA); hk_launch_taa_jasmine(P, smaa, ctx->stream);
        }
        if (P.in.fsr1) {   // post_process.rs:1279-1308: EASU then RCAS over the camera target (full-frame context, checked above)
            P.row_lo = 0; P.row_hi = P.band.H; P.col_lo = 0; P.col_hi = P.band.W;
            KernelTimer t(ctx, HK_K_FSR1);
            hk_launch_fsr_easu(P, ctx->stream);
            hk_launch_fsr_rcas(P, ctx->stream);
            ctx->launches += 1;
        }
    }
    return check_launch(ctx);
}

int hk_prepass_run(hk_context* ctx, const hk_frame_inputs* in) {
    KParams P; int rc = make_params(ctx, in, P); if (rc) return rc;
    SceneUse use(ctx);
    ctx->launches = 0;
    return run_prepass(ctx, P);
}
// A host that rasterises its own prepass (bevy-hikari's PrepassNode writes five render targets, prepass.rs:285-306, prepass.wgsl:76-99)
// hands them over as DEVICE pointers: no host copy, no primary rays.  The planes are copied plane by plane, device to device, on the
// context's stream into the context's own layout (52 B/px: 0.03 ms at 1080p), after the current <-> previous swap PrepassNode::run
// is preceded by (prepass.rs:427).  hk_light_run + hk_post_process_run then run the path on them.
int hk_import_gbuffer(hk_context* ctx, const hk_gbuffer_desc* g) {
    if (!ctx || !g) return HK_ERR_INVALID_ARGUMENT;
    if (!ctx->planes_ready) return set_error(ctx, HK_ERR_NOT_READY, "per-pixel planes are not allocated (a resize failed)");
    if (!g->position || !g->normal || !g->depth_gradient || !g->instance_material || !g->velocity_uv)
        return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "hk_import_gbuffer: all five planes are required");
    const Band& b = ctx->band;
    const size_t ow = (size_t)(b.cx1 - b.cx0), oh = (size_t)(b.r1 - b.r0);
    const size_t pitch[5] = {g->position_pitch_bytes, g->normal_pitch_bytes, g->depth_gradient_pitch_bytes, g->instance_material_pitch_bytes, g->velocity_uv_pitch_bytes};
    const size_t bpp[5] = {16, 4, 8, 8, 16};
    for (int i = 0; i < 5; ++i)
        if (pitch[i] < ow * bpp[i]) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "hk_import_gbuffer: a row pitch is smaller than the owned rectangle's row");
    HK_CUDA(cudaSetDevice(ctx->device));
    ctx->gbuffer_current ^= 1;
    Planes& p = ctx->planes;
    const size_t first = (size_t)(b.r0 - b.a0) * (size_t)b.AW + (size_t)(b.cx0 - b.ax0);
    void* dst[5] = {p.pos_depth_db[ctx->gbuffer_current] + first, p.normal + first, p.depth_gradient + first, p.instance_material + first,
                    p.velocity_uv_db[ctx->gbuffer_current] + first};
    const void* src[5] = {g->position, g->normal, g->depth_gradient, g->instance_material, g->velocity_uv};
    for (int i = 0; i < 5; ++i)
        HK_CUDA(cudaMemcpy2DAsync(dst[i], (size_t)b.AW * bpp[i], src[i], pitch[i], ow * bpp[i], oh, cudaMemcpyDeviceToDevice, ctx->stream));
    return HK_OK;
}
int hk_light_run(hk_context* ctx, const hk_frame_inputs* in) {
    KParams P; int rc = make_params(ctx, in, P); if (rc) return rc;
    SceneUse use(ctx);
    ctx->launches = 0;
    // LightNode::run starts with full_screen_albedo (light.rs:645-653).  hk_render_frame has it fused into the G-buffer
    // kernel; the stand-alone node recomputes it from whatever G-buffer is current (e.g. one supplied with hk_upload_state).
    rows_deferred(ctx, P, GHOST_TEMPORAL + ctx->motion_margin);
    hk_launch_albedo(P, ctx->stream);
    ctx->launches += 1;
    return run_light(ctx, P);
}
int hk_post_process_run(hk_context* ctx, const hk_frame_inputs* in) {
    KParams P; int rc = make_params(ctx, in, P); if (rc) return rc;
    ctx->launches = 0;
    return run_post(ctx, P, false);
}
// Test hook: ONE pass of the path on whatever the planes hold (e.g. state uploaded with hk_upload_state), so that a pass can be
// compared with the oracle's from identical inputs.  Pass ids as oracle/hk_oracle.cpp hko_run_pass: 0 albedo, 1 direct_lit (sun),
// 2 direct_lit (emissive), 3 spatial_reuse (emissive), 4 indirect_lit_ambient, 5 spatial_reuse (indirect), 6 the denoise chain
// (demodulation + four levels, all signals at once; level 3 writes HK_OUT_DENOISED_*), 7 tone mapping.
int hk_run_pass(hk_context* ctx, const hk_frame_inputs* in, int pass, int arg) {
    (void)arg;
    KParams P; int rc = make_params(ctx, in, P); if (rc) return rc;
    SceneUse use(ctx);
    ctx->launches = 0;
    const hk_frame_uniform& f = P.in.frame;
    const int GS = ::GHOST_SPATIAL + ring_of(P), GT = GHOST_TEMPORAL + ctx->motion_margin;
    switch (pass) {
        case 0: rows_deferred(ctx, P, GT); hk_launch_albedo(P, ctx->stream); break;
        case 1: rows(ctx, P, GT); hk_launch_direct(P, false, ctx->count_rays, wide_light(ctx), ctx->stream); hk_launch_scatter_resolve(P, 0, ctx->stream); break;
        case 2: rows(ctx, P, GT); hk_launch_direct(P, true, ctx->count_rays, wide_light(ctx), ctx->stream); hk_launch_scatter_resolve(P, 1, ctx->stream); break;
        case 3: rows(ctx, P, GS); launch_spatial(ctx, P, true); break;
        case 4:
            rows(ctx, P, GT);
            if (ctx->pooled_indirect) hk_launch_indirect_pool(P, f.indirect_bounces >= 2, ctx->count_rays, ctx->stream);
            else hk_launch_indirect(P, f.indirect_bounces >= 2, ctx->count_rays, wide_light(ctx), ctx->stream);
            hk_launch_scatter_resolve(P, 2, ctx->stream);
            break;
        case 5: rows(ctx, P, GS); launch_spatial(ctx, P, false); break;
        case 6: {
            const int ring = ring_of(P), signals = (f.indirect_bounces == 0) ? 2 : 3;
            rows(ctx, P, ::GHOST_DEMOD + ring); hk_launch_demodulation(P, signals, ctx->stream);
            rows(ctx, P, ::GHOST_L0 + ring); hk_launch_denoise_level(P, 0, signals, false, false, denoise_maps(ctx, 0), ctx->stream);
            rows(ctx, P, ::GHOST_L1 + ring); hk_launch_denoise_level(P, 1, signals, false, false, denoise_maps(ctx, 1), ctx->stream);
            rows(ctx, P, ::GHOST_L2 + ring); hk_launch_denoise_level(P, 2, signals, false, false, denoise_maps(ctx, 2), ctx->stream);
            rows(ctx, P, ring); hk_launch_denoise_level(P, 3, signals, false, true, denoise_maps(ctx, 3), ctx->stream);
            break;
        }
        case 7: rows(ctx, P, ring_of(P)); order_behind_copy(ctx); hk_launch_tone_mapping(P, ctx->stream); break;
        default: return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "unknown pass id");
    }
    return check_launch(ctx);
}
int hk_render_frame(hk_context* ctx, const hk_frame_inputs* in) {
    KParams P; int rc = make_params(ctx, in, P); if (rc) return rc;
    SceneUse use(ctx);
    ctx->launches = 0;
    for (int i = 0; i < HK_K_COUNT; ++i) ctx->kran[i] = false;
    ctx->ring_hit = false;
    const bool t = ctx->time_passes && ctx->time_only < 0;
    if (ctx->count_rays) HK_CUDA(cudaMemsetAsync(ctx->counters, 0, sizeof(Counters), ctx->stream));
    if (t) cudaEventRecord(ctx->ev[0], ctx->stream);
    rc = run_prepass(ctx, P); if (rc) return rc;
    if (t) cudaEventRecord(ctx->ev[1], ctx->stream);
    rc = run_light(ctx, P); if (rc) return rc;
    if (t) cudaEventRecord(ctx->ev[2], ctx->stream);
    rc = run_post(ctx, P, true); if (rc) return rc;
    if (t) cudaEventRecord(ctx->ev[3], ctx->stream);
    if (ctx->ring_hit) ctx->ring_frames += 1;
    return HK_OK;
}

int hk_sync(hk_context* ctx) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    HK_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ctx->copy_unwaited) { HK_CUDA(cudaEventSynchronize(ctx->ev_copied)); ctx->copy_unwaited = false; }
    return HK_OK;
}

int hk_set_profiling(hk_context* ctx, int count_rays, int time_passes) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    ctx->count_rays = count_rays != 0;
    ctx->time_passes = time_passes != 0;
    return HK_OK;
}
int hk_set_tuning(hk_context* ctx, int key, int value) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    switch (key) {
        case HK_TUNE_POOLED_INDIRECT: ctx->pooled_indirect = value != 0; return HK_OK;
        case HK_TUNE_TILED_SPATIAL: ctx->tiled_spatial = value != 0; return HK_OK;
        case HK_TUNE_TILED_DENOISE: ctx->tiled_denoise = value != 0; return HK_OK;
        case HK_TUNE_WIDE_TRAVERSAL:
            if (value < 0 || value > 3 || value == 2) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "HK_TUNE_WIDE_TRAVERSAL takes 0, 1 or 3");
            ctx->wide_traversal = value; return HK_OK;
        default: return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "unknown tuning key");
    }
}
int hk_set_profiling_kernel(hk_context* ctx, int kernel) {
    if (!ctx || kernel >= HK_K_COUNT) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    ctx->time_only = kernel < 0 ? -1 : kernel;
    ctx->ring_frames = 0;
    if (kernel >= 0 && !ctx->ring[0][0])
        for (int i = 0; i < hk_context::RING; ++i)
            for (int j = 0; j < 2; ++j) HK_CUDA(cudaEventCreate(&ctx->ring[i][j]));
    return HK_OK;
}
int hk_set_keep_intermediates(hk_context* ctx, int keep) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    ctx->keep_intermediates = keep != 0;
    return HK_OK;
}

int hk_get_stats(hk_context* ctx, hk_frame_stats* out) {
    if (!ctx || !out) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    HK_CUDA(cudaStreamSynchronize(ctx->stream));
    memset(out, 0, sizeof(*out));
    if (ctx->count_rays) {
        Counters h;
        HK_CUDA(cudaMemcpy(&h, ctx->counters, sizeof(h), cudaMemcpyDeviceToHost));
        out->primary_rays = h.primary; out->tlas_rays = h.tlas; out->blas_rays = h.blas;
    }
    if (ctx->time_only >= 0) {   // mean live duration of the one selected kernel over the frames recorded in the ring
        const uint32_t n = ctx->ring_frames < (uint32_t)hk_context::RING ? ctx->ring_frames : (uint32_t)hk_context::RING;
        double sum = 0.0;
        for (uint32_t i = 0; i < n; ++i) { float ms = 0.0f; cudaEventElapsedTime(&ms, ctx->ring[i][0], ctx->ring[i][1]); sum += ms; }
        if (n) out->ms_kernel[ctx->time_only] = (float)(sum / n);
        out->timed_frames = n;
    } else if (ctx->time_passes) {
        cudaEventElapsedTime(&out->ms_prepass, ctx->ev[0], ctx->ev[1]);
        cudaEventElapsedTime(&out->ms_light, ctx->ev[1], ctx->ev[2]);
        cudaEventElapsedTime(&out->ms_post_process, ctx->ev[2], ctx->ev[3]);
        cudaEventElapsedTime(&out->ms_total, ctx->ev[0], ctx->ev[3]);
        for (int i = 0; i < HK_K_COUNT; ++i)
            if (ctx->kran[i]) cudaEventElapsedTime(&out->ms_kernel[i], ctx->kev[i][0], ctx->kev[i][1]);
    }
    out->ms_kernel[HK_K_TRACE_RAYS] = ctx->trace_ms;
    out->kernel_launches = ctx->launches;
    out->wide_traversal = (wide_primary(ctx) ? 1u : 0u) | (wide_light(ctx) ? 2u : 0u);
    out->wide_stack_need = ctx->sc ? ctx->sc->wide_stack_need : 0u;
    if (ctx->sc && ctx->sc->wide_on_device) {      // the last 4-wide TLAS was derived on the device: so are its verdict and stack need
        uint32_t state[3];
        HK_CUDA(wide_tlas_state(ctx->sc, state));
        if (!state[0]) out->wide_traversal = 0u;
        out->wide_stack_need = state[1];
    }
    return HK_OK;
}

int hk_band_rows(hk_context* ctx, uint32_t* a0, uint32_t* a1) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    if (a0) *a0 = (uint32_t)ctx->band.a0;
    if (a1) *a1 = (uint32_t)ctx->band.a1;
    return HK_OK;
}
int hk_tile_rect(hk_context* ctx, uint32_t allocated[4], uint32_t owned[4]) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    const Band& b = ctx->band;
    if (allocated) { allocated[0] = b.ax0; allocated[1] = b.ax1; allocated[2] = b.a0; allocated[3] = b.a1; }
    if (owned) { owned[0] = b.cx0; owned[1] = b.cx1; owned[2] = b.r0; owned[3] = b.r1; }
    return HK_OK;
}

}  // extern "C"

// ----------------------------------------------------------------------------------------- outputs / state
// owned rectangle of a reservoir buffer <-> the reference's AoS PackedReservoir layout
__global__ void k_gather_reservoir(ReservoirPlanes b, Band band, size_t n, uint4* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int ow = band.cx1 - band.cx0;
    const size_t src = band_index(band, band.cx0 + (int)(i % (size_t)ow), band.r0 + (int)(i / (size_t)ow));
    for (int q = 0; q < 4; ++q) out[4 * i + q] = b.q[q][src];
}
__global__ void k_scatter_reservoir(ReservoirPlanes b, Band band, size_t n, const uint4* in) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int ow = band.cx1 - band.cx0;
    const size_t dst = band_index(band, band.cx0 + (int)(i % (size_t)ow), band.r0 + (int)(i / (size_t)ow));
    for (int q = 0; q < 4; ++q) b.q[q][dst] = in[4 * i + q];
}

// Where a read-back / upload plane lives: device pointer of its first transferred pixel, bytes per pixel, the
// rectangle (width x height, in pixels) that is transferred and the row pitch of the plane in pixels.
struct PlaneView { void* ptr; size_t bpp, w, h, pitch; };
static bool plane_view(hk_context* ctx, int which, PlaneView* v) {
    if (!ctx->planes_ready) return false;
    const Planes& p = ctx->planes;
    const Band& b = ctx->band;
    const size_t ow = (size_t)(b.cx1 - b.cx0), oh = (size_t)(b.r1 - b.r0);
    const bool scaled = ctx->last_render_w != 0 && ctx->last_scaled;   // ratio > 1 (full frame)
    const size_t rw = scaled ? (size_t)ctx->last_render_w : ow, rh = scaled ? (size_t)ctx->last_render_h : oh;
    const size_t first_def = (size_t)(b.r0 - b.a0) * (size_t)b.AW + (size_t)(b.cx0 - b.ax0);
    const size_t first_ren = scaled ? 0 : first_def;
    const size_t pitch_ren = scaled ? rw : (size_t)b.AW;
    auto deferred = [&](void* base, size_t bpp) { *v = PlaneView{(char*)base + first_def * bpp, bpp, ow, oh, (size_t)b.AW}; return true; };
    auto render = [&](void* base, size_t bpp) { *v = PlaneView{(char*)base + first_ren * bpp, bpp, rw, rh, pitch_ren}; return true; };
    const uint32_t cur = ctx->last_number % 2u;
    switch (which) {
        case HK_OUT_TONE_MAPPED: *v = PlaneView{p.tone_mapped_db[ctx->last_upscalers ? cur : 0u], 8, rw, rh, rw}; return true;
        // upscaled images: a full-frame context stores them tightly; a tile over k x its allocation, of which the owned part is served
        case HK_OUT_FSR_SHARPENED:
            if (!p.upscale_sharpen_output) return false;
            *v = PlaneView{p.upscale_sharpen_output, 8, (size_t)b.W, (size_t)b.H, (size_t)b.W}; return true;
        case HK_OUT_UPSCALED: case HK_OUT_TAA: {
            uint2* base = which == HK_OUT_UPSCALED ? p.upscale_output : p.taa_output[cur];
            if (!base) return false;
            if (which == HK_OUT_UPSCALED && ctx->last_fsr) { *v = PlaneView{base, 8, (size_t)b.W, (size_t)b.H, (size_t)b.W}; return true; }
            const size_t k = (which == HK_OUT_UPSCALED || ctx->last_smaa) ? 2 : 1;
            if (ctx->full_frame) {
                const size_t uw = ctx->last_up_w ? (size_t)ctx->last_up_w : 2 * rw, uh = ctx->last_up_h ? (size_t)ctx->last_up_h : 2 * rh;
                if (k == 2) *v = PlaneView{base, 8, uw, uh, uw};   // stored tightly at OW x OH
                else *v = PlaneView{base, 8, rw, rh, rw};
                return true;
            }
            const size_t pitch = k * (size_t)b.AW, first = (k * (size_t)(b.r0 - b.a0)) * pitch + k * (size_t)(b.cx0 - b.ax0);
            *v = PlaneView{base + first, 8, k * ow, k * oh, pitch};
            return true;
        }
        case HK_OUT_RENDER_DIRECT: case HK_OUT_RENDER_EMISSIVE: case HK_OUT_RENDER_INDIRECT: return render(p.render[which - HK_OUT_RENDER_DIRECT], 8);
        case HK_OUT_VARIANCE_DIRECT: case HK_OUT_VARIANCE_EMISSIVE: case HK_OUT_VARIANCE_INDIRECT: return render(p.variance[which - HK_OUT_VARIANCE_DIRECT], 4);
        case HK_OUT_DENOISED_DIRECT: case HK_OUT_DENOISED_EMISSIVE: case HK_OUT_DENOISED_INDIRECT: return render(p.dn_render[which - HK_OUT_DENOISED_DIRECT], 8);
        case HK_OUT_ALBEDO: return deferred(p.albedo, 8);
        case HK_OUT_GBUFFER_POSITION: return deferred(p.pos_depth_db[ctx->gbuffer_current], 16);
        case HK_OUT_GBUFFER_NORMAL: return deferred(p.normal, 4);
        case HK_OUT_GBUFFER_DEPTH_GRADIENT: return deferred(p.depth_gradient, 8);
        case HK_OUT_GBUFFER_INSTANCE_MATERIAL: return deferred(p.instance_material, 8);
        case HK_OUT_GBUFFER_VELOCITY_UV: return deferred(p.velocity_uv_db[ctx->gbuffer_current], 16);
    }
    return false;
}

extern "C" {

int hk_get_output(hk_context* ctx, int which, void** device_ptr, size_t* bytes) {
    if (!ctx || !device_ptr) return HK_ERR_INVALID_ARGUMENT;
    PlaneView v;
    if ((which != HK_OUT_TONE_MAPPED && which != HK_OUT_UPSCALED && which != HK_OUT_TAA && which != HK_OUT_FSR_SHARPENED) || !plane_view(ctx, which, &v))
        return set_error(ctx, HK_ERR_UNSUPPORTED, "only the final images (tone-mapped, upscaled, TAA, FSR-sharpened) are exposed as device pointers");
    *device_ptr = v.ptr;
    if (bytes) *bytes = v.w * v.h * v.bpp;
    return HK_OK;
}

int hk_output_extent(hk_context* ctx, int which, uint32_t* width, uint32_t* height) {
    if (!ctx || !width || !height) return HK_ERR_INVALID_ARGUMENT;
    PlaneView v;
    if (which >= HK_OUT_RESERVOIR_0 && which < HK_OUT_RESERVOIR_0 + 10) {
        if (!plane_view(ctx, HK_OUT_RENDER_DIRECT, &v)) return HK_ERR_INVALID_ARGUMENT;
    } else if (!plane_view(ctx, which, &v)) {
        return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "unknown plane id");
    }
    *width = (uint32_t)v.w; *height = (uint32_t)v.h;
    return HK_OK;
}

static int transfer(hk_context* ctx, int which, void* host, size_t bytes, bool to_host) {
    if (!ctx || !host) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    if (!ctx->planes_ready) return set_error(ctx, HK_ERR_NOT_READY, "per-pixel planes are not allocated (a resize failed)");
    if (which >= HK_OUT_RESERVOIR_0 && which < HK_OUT_RESERVOIR_0 + 10) {
        Band rb = ctx->band;   // rectangle of the reservoir buffer in render space
        if (ctx->last_render_w != 0 && ctx->last_scaled) {
            rb.cx0 = 0; rb.cx1 = ctx->last_render_w; rb.r0 = 0; rb.r1 = ctx->last_render_h; rb.a0 = 0; rb.ax0 = 0; rb.AW = ctx->last_render_w;
        }
        const size_t n = (size_t)(rb.cx1 - rb.cx0) * (size_t)(rb.r1 - rb.r0);
        if (bytes != n * 64) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "size mismatch");
        uint4* tmp = nullptr;
        HK_CUDA(cudaMalloc(reinterpret_cast<void**>(&tmp), bytes));
        const unsigned blocks = (unsigned)((n + 255) / 256);
        cudaError_t e;
        if (to_host) {
            k_gather_reservoir<<<blocks, 256, 0, ctx->stream>>>(ctx->planes.reservoir[which - HK_OUT_RESERVOIR_0], rb, n, tmp);
            e = cudaMemcpyAsync(host, tmp, bytes, cudaMemcpyDeviceToHost, ctx->stream);
        } else {
            e = cudaMemcpyAsync(tmp, host, bytes, cudaMemcpyHostToDevice, ctx->stream);
            k_scatter_reservoir<<<blocks, 256, 0, ctx->stream>>>(ctx->planes.reservoir[which - HK_OUT_RESERVOIR_0], rb, n, tmp);
        }
        cudaError_t e2 = cudaStreamSynchronize(ctx->stream);
        cudaFree(tmp);
        HK_CUDA(e);
        HK_CUDA(e2);
        return HK_OK;
    }
    PlaneView v;
    if (!plane_view(ctx, which, &v)) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "unknown plane id");
    if (bytes != v.w * v.h * v.bpp) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "size mismatch");
    if (to_host) HK_CUDA(cudaMemcpy2DAsync(host, v.w * v.bpp, v.ptr, v.pitch * v.bpp, v.w * v.bpp, v.h, cudaMemcpyDeviceToHost, ctx->stream));
    else HK_CUDA(cudaMemcpy2DAsync(v.ptr, v.pitch * v.bpp, host, v.w * v.bpp, v.w * v.bpp, v.h, cudaMemcpyHostToDevice, ctx->stream));
    if (!to_host && which == HK_OUT_GBUFFER_POSITION) {      // the planar copy of the depth follows an uploaded position plane
        KParams P{};
        P.planes = ctx->planes; P.planes.pos_depth = ctx->planes.pos_depth_db[ctx->gbuffer_current]; P.band = ctx->band;
        P.row_lo = ctx->band.r0; P.row_hi = ctx->band.r1; P.col_lo = ctx->band.cx0; P.col_hi = ctx->band.cx1;
        hk_launch_extract_depth(P, ctx->stream);
    }
    HK_CUDA(cudaStreamSynchronize(ctx->stream));
    return HK_OK;
}
int hk_readback(hk_context* ctx, int which, void* host, size_t bytes) { return transfer(ctx, which, host, bytes, true); }

int hk_readback_async(hk_context* ctx, int which, void* pinned_host, size_t bytes) {
    if (!ctx || !pinned_host) return HK_ERR_INVALID_ARGUMENT;
    PlaneView v;
    if ((which != HK_OUT_TONE_MAPPED && which != HK_OUT_UPSCALED && which != HK_OUT_TAA && which != HK_OUT_FSR_SHARPENED) || !plane_view(ctx, which, &v))
        return set_error(ctx, HK_ERR_UNSUPPORTED, "hk_readback_async serves the final images (tone-mapped, upscaled, TAA, FSR-sharpened)");
    if (bytes != v.w * v.h * v.bpp) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "size mismatch");
    HK_CUDA(cudaSetDevice(ctx->device));
    if (!ctx->copy_stream) {
        HK_CUDA(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
        HK_CUDA(cudaEventCreateWithFlags(&ctx->ev_submitted, cudaEventDisableTiming));
        HK_CUDA(cudaEventCreateWithFlags(&ctx->ev_copied, cudaEventDisableTiming));
    }
    if (ctx->copy_unwaited) HK_CUDA(cudaEventSynchronize(ctx->ev_copied));   // one copy in flight: the previous one must have landed
    HK_CUDA(cudaEventRecord(ctx->ev_submitted, ctx->stream));
    HK_CUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_submitted, 0));
    HK_CUDA(cudaMemcpy2DAsync(pinned_host, v.w * v.bpp, v.ptr, v.pitch * v.bpp, v.w * v.bpp, v.h, cudaMemcpyDeviceToHost, ctx->copy_stream));
    HK_CUDA(cudaEventRecord(ctx->ev_copied, ctx->copy_stream));
    ctx->copy_in_flight = true;
    ctx->copy_unwaited = true;
    return HK_OK;
}
// ------------------------------------------------------------------------------------------ halo exchange
static int halo_rect(hk_context* ctx, const Band& d, const Band& s, int& x0, int& x1, int& y0, int& y1);
int hk_context_set_motion_margin(hk_context* ctx, uint32_t pixels) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    if (pixels > 256u) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "motion margin above 256 pixels");
    HK_CUDA(cudaSetDevice(ctx->device));
    HK_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->motion_margin = (int)pixels;
    const Band b = ctx->band;
    return allocate_planes(ctx, (uint32_t)b.W, (uint32_t)b.H, (uint32_t)b.cx0, (uint32_t)b.cx1, (uint32_t)b.r0, (uint32_t)b.r1);
}
int hk_context_enable_tile_upscalers(hk_context* ctx, int enabled) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    HK_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->tile_upscalers = enabled != 0;
    const Band b = ctx->band;
    return allocate_planes(ctx, (uint32_t)b.W, (uint32_t)b.H, (uint32_t)b.cx0, (uint32_t)b.cx1, (uint32_t)b.r0, (uint32_t)b.r1);
}
// the images the temporal upscalers carry from frame to frame (tiles): tone-mapped ring planes and TAA history
static void halo_pull_images(hk_context* dst, const Planes& sp, const Band& sb, int x0, int x1, int y0, int y1) {
    const Planes& dp = dst->planes;
    if (!dp.tone_ring_db[0] || !sp.tone_ring_db[0]) return;
    const int k = dst->last_smaa ? 2 : 1;
    for (int i = 0; i < 2; ++i) {
        hk_launch_halo_copy_image(dp.tone_ring_db[i], dst->band, sp.tone_ring_db[i], sb, 1, x0, x1, y0, y1, dst->stream);
        hk_launch_halo_copy_image(dp.taa_output[i], dst->band, sp.taa_output[i], sb, k, x0, x1, y0, y1, dst->stream);
    }
}
int hk_halo_pull(hk_context* dst, hk_context* src) {
    if (!dst || !src) return HK_ERR_INVALID_ARGUMENT;
    if (dst == src) return HK_OK;
    hk_context* ctx = dst;   // errors are reported on the pulling context
    const Band& d = dst->band;
    const Band& s = src->band;
    int x0, x1, y0, y1;
    int rc = halo_rect(dst, d, s, x0, x1, y0, y1);
    if (rc != HK_OK) return rc;
    if (x0 >= x1 || y0 >= y1) return HK_OK;
    HK_CUDA(cudaSetDevice(dst->device));
    if (src->device != dst->device) {
        int can = 0;
        HK_CUDA(cudaDeviceCanAccessPeer(&can, dst->device, src->device));
        if (!can) return set_error(dst, HK_ERR_UNSUPPORTED, "no peer access between the two contexts' GPUs");
        cudaError_t e = cudaDeviceEnablePeerAccess(src->device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) HK_CUDA(e);
        cudaGetLastError();
    }
    hk_launch_halo_copy(dst->planes, d, src->planes, s, x0, x1, y0, y1, dst->stream);
    halo_pull_images(dst, src->planes, s, x0, x1, y0, y1);
    return check_launch(dst);
}

static int halo_rect(hk_context* ctx, const Band& d, const Band& s, int& x0, int& x1, int& y0, int& y1) {
    if (d.W != s.W || d.H != s.H) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "hk_halo_pull: the two contexts render different frames");
    x0 = std::max(d.ax0, s.cx0); x1 = std::min(d.ax1, s.cx1); y0 = std::max(d.a0, s.r0); y1 = std::min(d.a1, s.r1);
    if (x0 < x1 && y0 < y1 && x0 < d.cx1 && x1 > d.cx0 && y0 < d.r1 && y1 > d.r0)
        return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "hk_halo_pull: the owned rectangles of the two contexts overlap");
    return HK_OK;
}
int hk_halo_export(hk_context* ctx, hk_halo_descriptor* out) {
    if (!ctx || !out) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    memset(out, 0, sizeof(*out));
    for (int r = 0; r < 10; ++r)
        for (int q = 0; q < 4; ++q) {
            cudaIpcMemHandle_t h;
            HK_CUDA(cudaIpcGetMemHandle(&h, ctx->planes.reservoir[r].q[q]));
            memcpy(out->plane_handles[4 * r + q], &h, 64);
        }
    if (ctx->planes.tone_ring_db[0]) {
        uint2* images[4] = {ctx->planes.tone_ring_db[0], ctx->planes.tone_ring_db[1], ctx->planes.taa_output[0], ctx->planes.taa_output[1]};
        for (int i = 0; i < 4; ++i) {
            cudaIpcMemHandle_t h;
            HK_CUDA(cudaIpcGetMemHandle(&h, images[i]));
            memcpy(out->plane_handles[40 + i], &h, 64);
        }
        out->has_images = 1;
    }
    const Band& b = ctx->band;
    out->frame[0] = b.W; out->frame[1] = b.H;
    out->allocated[0] = b.ax0; out->allocated[1] = b.ax1; out->allocated[2] = b.a0; out->allocated[3] = b.a1;
    out->owned[0] = b.cx0; out->owned[1] = b.cx1; out->owned[2] = b.r0; out->owned[3] = b.r1;
    return HK_OK;
}
int hk_halo_import(hk_context* ctx, const hk_halo_descriptor* remote, hk_halo_peer** out) {
    if (!ctx || !remote || !out) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    hk_halo_peer* peer = new hk_halo_peer();
    memset(peer->mapped, 0, sizeof(peer->mapped));
    Band& b = peer->band;
    b = Band{};
    b.W = remote->frame[0]; b.H = remote->frame[1];
    b.ax0 = remote->allocated[0]; b.ax1 = remote->allocated[1]; b.a0 = remote->allocated[2]; b.a1 = remote->allocated[3];
    b.cx0 = remote->owned[0]; b.cx1 = remote->owned[1]; b.r0 = remote->owned[2]; b.r1 = remote->owned[3];
    b.AW = hk_plane_pitch(b.ax1 - b.ax0); b.RW = b.W; b.RH = b.H; b.RS = b.AW; b.OW = 2 * b.W; b.OH = 2 * b.H;
    peer->planes = Planes{};
    const int handles = remote->has_images ? 44 : 40;
    for (int i = 0; i < handles; ++i) {
        cudaIpcMemHandle_t h;
        memcpy(&h, remote->plane_handles[i], 64);
        void* p = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
            for (void* m : peer->mapped) if (m) cudaIpcCloseMemHandle(m);
            delete peer;
            return set_error(ctx, HK_ERR_CUDA, std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
        }
        peer->mapped[i] = p;
        if (i < 40) peer->planes.reservoir[i / 4].q[i % 4] = static_cast<uint4*>(p);
        else if (i < 42) peer->planes.tone_ring_db[i - 40] = static_cast<uint2*>(p);
        else peer->planes.taa_output[i - 42] = static_cast<uint2*>(p);
    }
    ctx->halo_peers.push_back(peer);
    *out = peer;
    return HK_OK;
}
int hk_halo_pull_peer(hk_context* ctx, hk_halo_peer* peer) {
    if (!ctx || !peer) return HK_ERR_INVALID_ARGUMENT;
    int x0, x1, y0, y1;
    int rc = halo_rect(ctx, ctx->band, peer->band, x0, x1, y0, y1);
    if (rc != HK_OK) return rc;
    if (x0 >= x1 || y0 >= y1) return HK_OK;
    HK_CUDA(cudaSetDevice(ctx->device));
    hk_launch_halo_copy(ctx->planes, ctx->band, peer->planes, peer->band, x0, x1, y0, y1, ctx->stream);
    halo_pull_images(ctx, peer->planes, peer->band, x0, x1, y0, y1);
    return check_launch(ctx);
}

// ------------------------------------------------------------------------------------------ frame assembly
int hk_set_frame_target(hk_context* ctx, void* frame_device_ptr, uint32_t pitch_pixels) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    if (!frame_device_ptr) { ctx->frame_target = nullptr; ctx->frame_pitch = 0; return HK_OK; }
    if (pitch_pixels < (uint32_t)ctx->band.W) return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "frame target pitch is smaller than the frame width");
    HK_CUDA(cudaSetDevice(ctx->device));
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, frame_device_ptr) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        return set_error(ctx, HK_ERR_INVALID_ARGUMENT, "frame target is not device memory");
    }
    if (attr.device != ctx->device) {   // same-process peer (cross-process mappings from hk_frame_open are already accessible)
        int can = 0;
        HK_CUDA(cudaDeviceCanAccessPeer(&can, ctx->device, attr.device));
        if (!can) return set_error(ctx, HK_ERR_UNSUPPORTED, "no peer access between the context's GPU and the frame target's GPU");
        cudaError_t e = cudaDeviceEnablePeerAccess(attr.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) HK_CUDA(e);
        cudaGetLastError();
    }
    ctx->frame_target = static_cast<uint2*>(frame_device_ptr);
    ctx->frame_pitch = pitch_pixels;
    return HK_OK;
}
int hk_frame_alloc(hk_context* ctx, void** device_ptr, uint8_t ipc_handle[64]) {
    if (!ctx || !device_ptr) return HK_ERR_INVALID_ARGUMENT;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
    HK_CUDA(cudaSetDevice(ctx->device));
    const size_t bytes = (size_t)ctx->band.W * (size_t)ctx->band.H * 8u;
    void* p = nullptr;
    HK_CUDA(cudaMalloc(&p, bytes));
    ctx->frames_owned.push_back(p);
    HK_CUDA(cudaMemsetAsync(p, 0, bytes, ctx->stream));
    HK_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ipc_handle) {
        cudaIpcMemHandle_t h;
        HK_CUDA(cudaIpcGetMemHandle(&h, p));
        memcpy(ipc_handle, &h, 64);
    }
    *device_ptr = p;
    return HK_OK;
}
int hk_frame_open(hk_context* ctx, const uint8_t ipc_handle[64], void** device_ptr) {
    if (!ctx || !ipc_handle || !device_ptr) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, ipc_handle, 64);
    void* p = nullptr;
    HK_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    ctx->frames_opened.push_back(p);
    *device_ptr = p;
    return HK_OK;
}
int hk_frame_read(hk_context* ctx, const void* frame_device_ptr, void* host, size_t bytes) {
    if (!ctx || !frame_device_ptr || !host) return HK_ERR_INVALID_ARGUMENT;
    HK_CUDA(cudaSetDevice(ctx->device));
    HK_CUDA(cudaMemcpyAsync(host, frame_device_ptr, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    HK_CUDA(cudaStreamSynchronize(ctx->stream));
    return HK_OK;
}

int hk_readback_wait(hk_context* ctx) {
    if (!ctx) return HK_ERR_INVALID_ARGUMENT;
    if (!ctx->copy_unwaited) return HK_OK;
    HK_CUDA(cudaSetDevice(ctx->device));
    HK_CUDA(cudaEventSynchronize(ctx->ev_copied));
    ctx->copy_unwaited = false;
    return HK_OK;
}
int hk_upload_state(hk_context* ctx, int which, const void* host, size_t bytes) {
    return transfer(ctx, which, const_cast<void*>(host), bytes, false);
}

int hk_trace_rays(hk_context* ctx, const hk_ray* rays, size_t n, hk_hit* hits) {
    if (!ctx || (n && (!rays || !hits))) return HK_ERR_INVALID_ARGUMENT;
    if (!scene_ready(ctx)) return set_error(ctx, HK_ERR_NOT_READY, "scene not uploaded");
    if (n == 0) return HK_OK;
    HK_CUDA(cudaSetDevice(ctx->device));
    SceneUse use(ctx);
    hk_ray* d_rays = nullptr; hk_hit* d_hits = nullptr;
    HK_CUDA(cudaMalloc(reinterpret_cast<void**>(&d_rays), n * sizeof(hk_ray)));
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&d_hits), n * sizeof(hk_hit));
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_rays, rays, n * sizeof(hk_ray), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) {
        cudaEventRecord(ctx->ev[0], ctx->stream);
        hk_launch_trace_rays(ctx->sc->scene, d_rays, n, d_hits, wide_light(ctx), ctx->stream);
        cudaEventRecord(ctx->ev[1], ctx->stream);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(hits, d_hits, n * sizeof(hk_hit), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) cudaEventElapsedTime(&ctx->trace_ms, ctx->ev[0], ctx->ev[1]);
    cudaFree(d_rays); cudaFree(d_hits);
    HK_CUDA(e);
    return HK_OK;
}

}  // extern "C"
