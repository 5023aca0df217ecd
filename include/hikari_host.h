/* hikari_host.h — C view of the host mirror (bevy_hikari_b200/host/hikari.hpp) for ctypes / other-language callers.
 * Everything here sits ABOVE the drop-in boundary (include/hikari_b200.h): it restates, in C++, the Rust host code
 * of the reference for this path (settings -> uniform, mesh/instance/material preparation, node order) because no
 * Rust toolchain exists in this image.  A real Bevy host would keep its own Rust versions of these and bind only
 * hikari_b200.h (see INTEGRATION.md). */
#ifndef HIKARI_HOST_H
#define HIKARI_HOST_H
#include "hikari_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { HIKARI_TAA_JASMINE = 0, HIKARI_TAA_NONE = 1 };              /* src/lib.rs:466-471 */
enum { HIKARI_UPSCALE_FSR1 = 0, HIKARI_UPSCALE_SMAA_TU4X = 1 };    /* src/lib.rs:473-487 */

typedef struct hikari_settings {   /* HikariSettings, src/lib.rs:399-433, same field names */
    uint32_t direct_validate_interval;
    uint32_t emissive_validate_interval;
    uint32_t max_temporal_reuse_count;
    uint32_t max_spatial_reuse_count;
    float max_reservoir_lifetime;
    float solar_angle;
    uint32_t indirect_bounces;
    float max_indirect_luminance;
    float clear_color[4];
    uint32_t temporal_reuse;
    uint32_t emissive_spatial_reuse;
    uint32_t indirect_spatial_reuse;
    uint32_t denoise;
    uint32_t taa;
    uint32_t upscale_kind;
    float upscale_ratio;
    float upscale_sharpness;
} hikari_settings;

typedef struct hikari_world hikari_world;     /* MeshMaterialPlugin's render-world resources */
typedef struct hikari_plugin hikari_plugin;   /* HikariPlugin + one camera */

void hikari_settings_default(hikari_settings* out);                       /* HikariSettings::default(), lib.rs:435-455 */
float hikari_upscale_ratio(const hikari_settings* s);                     /* Upscale::ratio(), lib.rs:501-505 */
void hikari_make_frame_inputs(const hikari_settings* s, uint64_t frame_counter, const hk_view* view,
                              const hk_previous_view* previous_view, const hk_lights* lights, hk_frame_inputs* out);
const char* hikari_graph_name(void);                                      /* graph::NAME, lib.rs:44 */

hikari_world* hikari_world_create(void);
void hikari_world_destroy(hikari_world* w);
/* topology: 0 = TriangleList, 1 = TriangleStrip, 2 = anything else.  NULL attribute => PrepareMeshError (mod.rs:301-308). */
uint32_t hikari_world_add_mesh(hikari_world* w, const float* positions, const float* normals, const float* uvs,
                               uint32_t vertex_count, const uint32_t* indices, uint32_t index_count, uint32_t topology);
/* The same for a mesh whose BLAS is built on the device (hikari_plugin_add_meshes / hikari_shared_scene_add_meshes): prepare keeps its
 * vertices and primitives on the host, for the alias tables, gives it the hk_mesh_index the device gives it and builds no BVH.  Device
 * meshes follow every host mesh, and are added to the scene in world order after the world's upload (which never carries them). */
uint32_t hikari_world_add_device_mesh(hikari_world* w, const float* positions, const float* normals, const float* uvs,
                                      uint32_t vertex_count, const uint32_t* indices, uint32_t index_count, uint32_t topology);
uint32_t hikari_world_add_material(hikari_world* w, const hk_material* m);
/* a modified StandardMaterial asset: set, then hikari_world_prepare_materials (material.rs:139-203) and
 * hikari_world_prepare_instances (emissive list / alias tables depend on the materials), then hikari_plugin_update_instances */
void hikari_world_set_material(hikari_world* w, uint32_t id, const hk_material* m);
void hikari_world_prepare_materials(hikari_world* w);
uint32_t hikari_world_add_texture(hikari_world* w, const hk_texture_desc* t);
uint32_t hikari_world_add_instance(hikari_world* w, uint32_t mesh, uint32_t material, const float* transform16, uint32_t visible);
void hikari_world_prepare(hikari_world* w);                               /* prepare_mesh_assets -> materials -> instances */
/* animated instances: a user system moving an entity (Update), previous_transform_system (transform.rs:31-44, once per
 * frame in PostUpdate), then prepare_instances (instance.rs:245-444) which rebuilds instances / TLAS / emissives / alias
 * tables (cached per entity while the scale stays within 0.01, instance.rs:385-397) and PreviousMeshUniform */
void hikari_world_set_instance_transform(hikari_world* w, uint32_t instance, const float* transform16);
void hikari_world_set_instance_visible(hikari_world* w, uint32_t instance, uint32_t visible);
void hikari_world_previous_transform_system(hikari_world* w);
void hikari_world_prepare_instances(hikari_world* w);
void hikari_world_scene_desc(hikari_world* w, hk_scene_desc* out);        /* pointers valid until the next prepare */
/* The transforms-only form of prepare_instances, for hk_scene_update_transforms (the device rebuilds AABBs / TLAS / emissives itself):
 * 1 + the three arrays that call takes (valid until the next call) when only transforms changed since the last prepare_instances;
 * 0 when the kept set of instances changed or an emissive's alias table must be rebuilt (scale moved by more than 0.01,
 * instance.rs:385-397): then hikari_world_prepare_instances + hikari_plugin_update_instances. */
int hikari_world_prepare_instance_transforms(hikari_world* w, const float** models, const float** previous_models, const float** mesh_aabbs,
                                             uint32_t* instance_count);
int hikari_world_mesh_error(hikari_world* w, uint32_t mesh);              /* PrepareMeshError as int, 0 = ok */

/* Run-time glTF 2.0 ingest (.glb, or .gltf with side-car / data: buffers) into the world: meshes (one per glTF primitive; triangle
 * lists and strips), materials, instances (depth-first node order, world matrices in glam f32 arithmetic, x parent_transform16 or
 * identity when NULL) and textures (one per image and colour space; sampler wrap modes / filter) — the rules of
 * src/mesh_material/{mesh,material,instance}.rs + bevy_gltf, see host/gltf_ingest.cpp.  Call hikari_world_prepare afterwards.
 * PNG images are decoded by the library; anything else is handed to `decoder` (NULL = such a file fails), called twice per image:
 * first with rgba_out = NULL to report *width / *height, then with a width*height*4-byte buffer to fill; returns non-zero on success.
 * Returns 1 on success; on failure 0 and the reason in `error` (truncated to error_capacity).  `counts` (may be NULL) receives the
 * ids the world assigned: each range is contiguous. */
typedef int (*hikari_image_decoder)(const uint8_t* bytes, size_t size, const char* mime_type, void* user, uint8_t* rgba_out,
                                    uint32_t* width, uint32_t* height);
typedef struct hikari_gltf_counts {
    uint32_t first_mesh, mesh_count, first_material, material_count, first_instance, instance_count, first_texture, texture_count;
} hikari_gltf_counts;
int hikari_world_load_gltf(hikari_world* w, const char* path, const float* parent_transform16, hikari_image_decoder decoder, void* user,
                           hikari_gltf_counts* counts, char* error, size_t error_capacity);
/* the library's PNG decoder on its own (8 / 16-bit grey, grey+alpha, RGB, RGBA, palette, 1/2/4-bit grey and palette; non-interlaced):
 * rgba_out may be NULL to query the size */
int hikari_decode_png(const uint8_t* bytes, size_t size, uint8_t* rgba_out, uint32_t* width, uint32_t* height);
/* Mesh::from(shape::*) of bevy 0.9 added as a mesh (returns its id; 0xFFFFFFFF = unknown kind).  params: PLANE {size};
 * UV_SPHERE {radius, sectors, stacks}; BOX {x_length, y_length, z_length} (shape::Cube{size} = BOX {size, size, size}). */
enum { HIKARI_SHAPE_PLANE = 0, HIKARI_SHAPE_UV_SPHERE = 1, HIKARI_SHAPE_BOX = 2 };
uint32_t hikari_world_add_shape(hikari_world* w, uint32_t kind, const float* params);

hikari_plugin* hikari_plugin_create(void);
void hikari_plugin_destroy(hikari_plugin* p);
int hikari_plugin_build(hikari_plugin* p, int cuda_device, uint32_t width, uint32_t height, uint32_t row_begin,
                        uint32_t row_end, const uint8_t* noise_rgba8_64x64x16, void* cuda_stream);
int hikari_plugin_build_tile(hikari_plugin* p, int cuda_device, uint32_t width, uint32_t height, uint32_t col_begin, uint32_t col_end,
                             uint32_t row_begin, uint32_t row_end, const uint8_t* noise_rgba8_64x64x16, void* cuda_stream);
int hikari_plugin_upload_scene(hikari_plugin* p, hikari_world* w);
int hikari_plugin_update_instances(hikari_plugin* p, hikari_world* w);   /* hk_scene_update_instances: instance-level buffers only */
/* animated instances, device-side: hk_scene_update_transforms when hikari_world_prepare_instance_transforms allows it, else
 * prepare_instances + hk_scene_update_instances; *used_device_path (may be NULL) says which */
int hikari_plugin_update_transforms(hikari_plugin* p, hikari_world* w, int* used_device_path);
/* hk_scene_add_meshes for the world's device meshes `mesh_ids`; out (may be NULL) receives their hk_mesh_index */
int hikari_plugin_add_meshes(hikari_plugin* p, hikari_world* w, const uint32_t* mesh_ids, uint32_t n, hk_mesh_index* out);
int hikari_plugin_run_frame(hikari_plugin* p, const hikari_settings* s, const hk_view* view,
                            const hk_previous_view* previous_view, const hk_lights* lights);
hk_context* hikari_plugin_context(hikari_plugin* p);
uint64_t hikari_plugin_frame_counter(hikari_plugin* p);
void hikari_plugin_set_frame_counter(hikari_plugin* p, uint64_t v);
/* 1 = run_frame continues past tone mapping with smaa_tu4x / taa_jasmine as the settings select (post_process.rs:1236-1277) */
void hikari_plugin_set_temporal_upscalers(hikari_plugin* p, int enabled);

/* HikariScene: one scene, uploaded and animated once per frame, that several cameras render (hk_shared_scene, hikari_b200.h).
 * build creates it on `cuda_stream` (NULL: a stream of its own); upload / update_instances / update_transforms are those of
 * hikari_plugin_*, for every attached camera at once.  Errors: hk_shared_scene_last_error(hikari_shared_scene_handle(s)).
 * destroy drops the handle; the scene lives on while a camera renders it. */
typedef struct hikari_shared_scene hikari_shared_scene;
hikari_shared_scene* hikari_shared_scene_create(void);
void hikari_shared_scene_destroy(hikari_shared_scene* s);
int hikari_shared_scene_build(hikari_shared_scene* s, int cuda_device, void* cuda_stream);
int hikari_shared_scene_upload(hikari_shared_scene* s, hikari_world* w);
int hikari_shared_scene_update_instances(hikari_shared_scene* s, hikari_world* w);
int hikari_shared_scene_update_transforms(hikari_shared_scene* s, hikari_world* w, int* used_device_path);
int hikari_shared_scene_add_meshes(hikari_shared_scene* s, hikari_world* w, const uint32_t* mesh_ids, uint32_t n, hk_mesh_index* out);
hk_shared_scene* hikari_shared_scene_handle(hikari_shared_scene* s);
/* the camera renders `s` from its next frame on, keeping its reservoirs (hk_context_attach_scene); its own upload / update calls
 * are refused while it does.  s = NULL: back to a private scene, HK_ERR_NOT_READY until hikari_plugin_upload_scene. */
int hikari_plugin_attach_scene(hikari_plugin* p, hikari_shared_scene* s);

#ifdef __cplusplus
}
#endif
#endif
