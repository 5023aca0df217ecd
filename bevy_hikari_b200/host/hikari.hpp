// hikari.hpp — host side of the drop-in, in C++ because the reference's host language (Rust) is not available in
// this image.  It mirrors the reference's plugin surface for the hot path — same type names, same field names,
// same defaults, same error behaviour — and sits strictly ABOVE the C ABI of include/hikari_b200.h: nothing in
// here touches CUDA; it only prepares the bytes the C ABI takes and calls hk_*().  Two libraries: libhikari_host.so holds
// everything up to and including make_frame_inputs (pure CPU, no CUDA dependency); the nodes and HikariPlugin, which call
// hk_*(), are linked into libhikari_b200.so (hikari_plugin.cpp), which depends on libhikari_host.so.
//
//   hikari::HikariSettings / Taa / Upscale / HikariUniversalSettings      src/lib.rs:372-513
//   hikari::graph::NAME, graph::node::*                                   src/lib.rs:43-51
//   hikari::FrameCounter, FrameUniform::extract_component                 src/view.rs:75-193
//   hikari::Mesh -> GpuMesh::try_from, build_alias_table                  src/mesh_material/mod.rs:310-467
//   hikari::MeshMaterialWorld::{prepare_mesh_assets,prepare_material_assets,prepare_instances}
//                                                                         src/mesh_material/{mesh,material,instance}.rs
//   hikari::PrepassNode / LightNode / PostProcessNode ::run               src/prepass.rs:769, src/light.rs:590,
//                                                                         src/post_process.rs:1140
//   hikari::HikariPlugin                                                  src/lib.rs:95-370
#pragma once
#include <array>
#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "hikari_b200.h"

namespace hikari {

namespace graph {
constexpr const char* NAME = "hikari";                       // lib.rs:44
namespace node {
constexpr const char* PREPASS = "hikari_prepass";            // lib.rs:46-49
constexpr const char* LIGHT = "hikari_light";
constexpr const char* POST_PROCESS = "hikari_post_process";
constexpr const char* OVERLAY = "hikari_overlay";
}  // namespace node
}  // namespace graph

constexpr uint32_t WORKGROUP_SIZE = 8;        // lib.rs:53
constexpr size_t NOISE_TEXTURE_COUNT = 16;    // lib.rs:54

enum class Taa { Jasmine, None };             // lib.rs:466-471 (default Jasmine)

struct Upscale {                              // lib.rs:473-513
    enum Kind { Fsr1, SmaaTu4x } kind = SmaaTu4x;
    float ratio_value = 2.0f;
    float sharpness_value = 0.0f;
    static Upscale fsr1(float ratio, float sharpness) { return Upscale{Fsr1, ratio, sharpness}; }
    static Upscale smaa_tu4x(float ratio) { return Upscale{SmaaTu4x, ratio, 0.0f}; }
    static Upscale SMAA_TU_1_0() { return smaa_tu4x(1.0f); }
    static Upscale SMAA_TU_2_0() { return smaa_tu4x(2.0f); }
    float ratio() const { return ratio_value < 1.0f ? 1.0f : (ratio_value > 2.0f ? 2.0f : ratio_value); }  // clamp(1,2)
    float sharpness() const { return kind == Fsr1 ? sharpness_value : 0.0f; }
};

struct HikariUniversalSettings {              // lib.rs:372-389
    bool build_mesh_acceleration_structure = true;
    bool build_instance_acceleration_structure = true;
};

struct HikariSettings {                       // lib.rs:399-455 (defaults lib.rs:435-455)
    size_t direct_validate_interval = 3;
    size_t emissive_validate_interval = 5;
    size_t max_temporal_reuse_count = 50;
    size_t max_spatial_reuse_count = 800;
    float max_reservoir_lifetime = 100.0f;
    float solar_angle = 0.046f;
    size_t indirect_bounces = 1;
    float max_indirect_luminance = 10.0f;
    std::array<float, 4> clear_color = {0.4f, 0.4f, 0.4f, 1.0f};
    bool temporal_reuse = true;
    bool emissive_spatial_reuse = false;
    bool indirect_spatial_reuse = true;
    bool denoise = true;
    Taa taa = Taa::Jasmine;
    Upscale upscale = Upscale::SMAA_TU_2_0();
};

struct FrameCounter { size_t value = 0; };    // view.rs:75-77, +1 per frame (view.rs:89-103)

struct FrameUniform : hk_frame_uniform {      // view.rs:105-193
    static FrameUniform extract_component(const HikariSettings& settings, const FrameCounter& counter);
};

// ------------------------------------------------------------------------------------------ mesh assets
enum class PrimitiveTopology { TriangleList, TriangleStrip, Other };
enum class PrepareMeshError {                 // mod.rs:301-308
    Ok = 0, MissingAttributePosition, MissingAttributeNormal, MissingAttributeUV, IncompatiblePrimitiveTopology, NoPrimitive
};

struct Mesh {                                 // the slice of bevy::render::mesh::Mesh that try_from reads
    std::vector<std::array<float, 3>> positions;   // ATTRIBUTE_POSITION
    std::vector<std::array<float, 3>> normals;     // ATTRIBUTE_NORMAL
    std::vector<std::array<float, 2>> uvs;         // ATTRIBUTE_UV_0
    std::vector<uint32_t> indices;                 // empty = non-indexed
    bool has_indices = true;
    PrimitiveTopology topology = PrimitiveTopology::TriangleList;
};

struct GpuMesh {                              // mod.rs:310-315
    std::vector<hk_vertex> vertices;
    std::vector<hk_primitive> primitives;     // already "compact" (mod.rs:121-145)
    std::vector<hk_node> nodes;
    // mod.rs:379-467; build_bvh = false: records only, for a mesh whose BLAS is built on the device (hk_scene_add_meshes)
    static PrepareMeshError try_from(const Mesh& mesh, GpuMesh* out, bool build_bvh = true);
    std::vector<float> transformed_primitive_areas(const float transform[16]) const;       // mod.rs:318-328
    std::vector<hk_alias_entry> build_alias_table(const float transform[16]) const;        // mod.rs:330-376
};

struct StandardMaterial {                     // the slice of bevy_pbr::StandardMaterial that material.rs:139-203 reads
    std::array<float, 4> base_color = {1, 1, 1, 1};       // Color::as_rgba_f32 components (material.rs:168)
    std::array<float, 4> emissive = {0, 0, 0, 1};
    float perceptual_roughness = 0.089f;
    float metallic = 0.01f;
    float reflectance = 0.5f;
    uint32_t base_color_texture = 0xFFFFFFFFu, emissive_texture = 0xFFFFFFFFu, metallic_roughness_texture = 0xFFFFFFFFu;
    uint32_t normal_map_texture = 0xFFFFFFFFu, occlusion_texture = 0xFFFFFFFFu;
};

struct InstanceDesc {                         // one (Entity, Handle<Mesh>, Handle<M>, GlobalTransform) — instance.rs:176-220
    uint32_t mesh = 0, material = 0;
    float transform[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    bool visible = true;
    // GlobalTransformQueue([current, previous]) (transform.rs:19-20); absent until previous_transform_system has seen the entity
    bool has_queue = false;
    float queue[2][16] = {};
};

// Flattened skip-link BVH over boxes (bvh 0.7.1 BVH::build + flatten_custom(&GpuNode::pack); mod.rs:458-459).
std::vector<hk_node> build_flat_bvh(const std::vector<std::array<float, 3>>& aabb_min,
                                    const std::vector<std::array<float, 3>>& aabb_max,
                                    std::vector<uint32_t>* shape_node_index);

// The render-world resources of MeshMaterialPlugin: owns the nine buffers handed to hk_scene_upload().
class MeshMaterialWorld {
public:
    HikariUniversalSettings universal_settings;
    uint32_t add_mesh(const Mesh& mesh);                   // Assets<Mesh>::add + extract (mesh.rs:77-104); id = asset order
    // A mesh whose BLAS lives on the device (HikariScene::add_meshes builds it there): prepare_mesh_assets keeps its vertices and
    // primitives on the host (the alias tables of emissive instances need the primitives' areas) and gives it the hk_mesh_index the
    // device gives it, but builds no BVH.  Device meshes come after every host mesh of the world, and are added to the scene in
    // world order after the world's upload; scene_desc() holds the host meshes only, so that upload never carries their records.
    uint32_t add_device_mesh(const Mesh& mesh);
    const Mesh& mesh(uint32_t id) const { return meshes_[id]; }
    bool is_device_mesh(uint32_t id) const { return id < device_mesh_.size() && device_mesh_[id]; }
    uint32_t add_material(const StandardMaterial& m);      // id = rank in the BTreeMap (material.rs:162-165)
    void set_material(uint32_t id, const StandardMaterial& m);   // Assets<StandardMaterial> modified -> prepare_material_assets + prepare_instances
    uint32_t add_texture(const hk_texture_desc& t, const uint8_t* pixels);
    uint32_t add_instance(const InstanceDesc& inst);       // id = rank in BTreeMap<Entity,..> (instance.rs:231-239)
    void prepare_mesh_assets();                            // mesh.rs:106-166
    void prepare_material_assets();                        // material.rs:139-203
    void prepare_instances();                              // instance.rs:245-444
    void prepare();                                        // the three, in RenderStage::Prepare order (mod.rs:42-55)
    // Animated instances.  set_instance_transform changes an entity's GlobalTransform (a user system in Update);
    // previous_transform_system is the PostUpdate system of transform.rs:31-44, run once per frame: every entity's queue
    // becomes [current matrix, former queue[0]] ([m, m] the first time).  prepare_instances then rebuilds instances, TLAS,
    // emissives and alias tables (instance.rs:352-437) and PreviousMeshUniform (instance.rs:111-128).
    void set_instance_transform(uint32_t instance, const float transform[16]);
    void set_instance_visible(uint32_t instance, bool visible);
    void previous_transform_system();
    // The transforms-only form of prepare_instances for hk_scene_update_transforms (the device rebuilds AABBs, TLAS, emissives and
    // the emissive BVH itself): fills transform_models / transform_previous (16 floats per kept instance: GlobalTransform and
    // PreviousMeshUniform::transform) and transform_aabbs (6 floats: centre and half extents of the mesh's Aabb, instance.rs:293-296)
    // and returns true — or returns false when the device path does not apply and prepare_instances + hk_scene_update_instances must
    // run instead: the kept SET of (entity, mesh, material) differs from the last prepare_instances, or an emissive instance's
    // alias table would be rebuilt (scale moved by more than 0.01 from the cached one, instance.rs:385-397).  Does not touch the
    // buffers of scene_desc(): after a device update they describe the last prepare_instances, not the device.
    bool prepare_instance_transforms();
    std::vector<float> transform_models, transform_previous, transform_aabbs;
    std::vector<float> previous_models;                    // 16 floats per entry of `instances`, queue[1] (or the model itself)
    hk_scene_desc scene_desc() const;                      // views into the vectors below; valid until the next prepare()
    const std::vector<PrepareMeshError>& mesh_errors() const { return mesh_errors_; }

    std::vector<hk_vertex> vertices;
    std::vector<hk_primitive> primitives;
    std::vector<hk_node> asset_nodes;
    std::vector<hk_alias_entry> alias_table;
    std::vector<hk_instance> instances;
    std::vector<hk_node> instance_nodes;
    std::vector<hk_material> materials;
    std::vector<hk_node> emissive_nodes;
    std::vector<hk_emissive> emissives;

private:
    std::vector<Mesh> meshes_;
    std::vector<bool> device_mesh_;                         // per mesh: its BLAS is built on the device
    uint32_t host_vertex_count_ = 0, host_primitive_count_ = 0;   // the records of the host meshes (scene_desc)
    std::vector<GpuMesh> gpu_meshes_;
    std::vector<bool> mesh_ok_;
    std::vector<PrepareMeshError> mesh_errors_;
    std::vector<hk_mesh_index> mesh_index_;
    std::vector<StandardMaterial> materials_in_;
    std::vector<InstanceDesc> instances_in_;
    struct CachedAliasTable { bool valid = false; float scale[3] = {0, 0, 0}; std::vector<hk_alias_entry> table; };
    struct KeptInstance { uint32_t entity, mesh, material; };
    std::vector<KeptInstance> kept_;                       // the instances of the last prepare_instances, in buffer order
    std::vector<std::array<float, 6>> mesh_aabb_;          // per mesh: centre | half extents, filled on first use
    std::vector<bool> mesh_aabb_ok_;
    std::vector<CachedAliasTable> alias_table_cache_;      // per entity: Local<HashMap<Entity, (Vec3, Vec<GpuAliasEntry>)>>, instance.rs:253,386-397
    std::vector<hk_texture_desc> textures_;
    std::vector<std::vector<uint8_t>> texture_pixels_;
};

// ------------------------------------------------------------------------------------------------ scene ingest (gltf_ingest.cpp)
// Run-time glTF 2.0 ingest into a MeshMaterialWorld: what `asset_server.load("x.glb#Scene0")` + the extraction systems of
// src/mesh_material/{mesh,material,instance}.rs hand the render world.  One Mesh per glTF primitive, one StandardMaterial per glTF
// material (+ StandardMaterial::default() for primitives without one), one instance per (node, primitive) in depth-first node order
// with the node's world matrix (x `parent_transform`, NULL = identity), one texture per (image, colour space): base colour and
// emissive sRGB, metallic-roughness / normal / occlusion linear (material.rs:55-87), wrap modes and mag filter from the sampler.
// PNG is decoded here; other encodings (JPEG) by `decoder` (NULL = fail on them), as image decoding is the host app's job.
struct GltfImage { std::vector<uint8_t> rgba; uint32_t width = 0, height = 0; };
typedef bool (*GltfImageDecoder)(const uint8_t* bytes, size_t size, const char* mime_type, void* user, GltfImage* out);
struct GltfLoadResult {
    std::vector<uint32_t> meshes, materials, instances, textures;    // ids the world assigned, in glTF order
    std::string error;
};
bool load_gltf(MeshMaterialWorld& world, const char* path, const float* parent_transform, GltfImageDecoder decoder, void* user,
               GltfLoadResult* out);
bool decode_png_rgba8(const uint8_t* bytes, size_t size, GltfImage* out);
// Mesh::from(shape::Plane / UVSphere / Box) of bevy 0.9, the generators the reference's examples spawn (scene.rs:86-113, city.rs:64-90)
namespace shape {
Mesh plane(float size);
Mesh uv_sphere(float radius, uint32_t sectors, uint32_t stacks);
Mesh box(float x_length, float y_length, float z_length);      // shape::Cube { size } = box(size, size, size)
}  // namespace shape

// ------------------------------------------------------------------------------------------------ nodes
struct ViewInputs {                           // what the render graph resolves for the "view" slot (light.rs:596-617)
    hk_view view;
    hk_previous_view previous_view;
    hk_lights lights;
};
hk_frame_inputs make_frame_inputs(const HikariSettings& settings, const FrameCounter& counter, const ViewInputs& view);

struct PrepassNode { static int run(hk_context* ctx, const hk_frame_inputs& in); };       // prepass.rs:769-851
struct LightNode { static int run(hk_context* ctx, const hk_frame_inputs& in); };         // light.rs:590-702
struct PostProcessNode { static int run(hk_context* ctx, const hk_frame_inputs& in); };   // post_process.rs:1140-1234

// HikariScene: the scene buffers of the render world (MeshMaterialBindGroup, mesh_material/mod.rs:677-681), uploaded and animated
// once per frame whatever the number of cameras.  create() makes a shared scene (hk_shared_scene) that cameras attach to with
// HikariPlugin::attach_scene; inside HikariPlugin the same class drives the camera's private scene through its context, so the
// upload / update logic (and the fallback of update_transforms) exists once.
class HikariScene {
public:
    HikariScene() = default;
    ~HikariScene();
    HikariScene(const HikariScene&) = delete;
    HikariScene& operator=(const HikariScene&) = delete;
    int create(int cuda_device, void* cuda_stream);         // cuda_stream NULL: the scene creates its own
    int upload(const MeshMaterialWorld& world);
    // instance-level buffers only (hk_scene_update_instances): what instance.rs:427-435 rewrites when instances change
    int update_instances(const MeshMaterialWorld& world);
    // Animated instances through the device-side rebuild (hk_scene_update_transforms) whenever only transforms changed since the
    // last prepare_instances; otherwise world.prepare_instances() + hk_scene_update_instances.  *used_device_path says which.
    int update_transforms(MeshMaterialWorld& world, bool* used_device_path = nullptr);
    // hk_scene_add_meshes for the world's device meshes `ids` (in world order, each once): their records and BLAS are built on the
    // device; out (may be NULL) receives their hk_mesh_index, which prepare_mesh_assets gives them as well
    int add_meshes(const MeshMaterialWorld& world, const uint32_t* ids, uint32_t n, hk_mesh_index* out);
    hk_shared_scene* handle() const { return scene_; }      // NULL for a camera's private scene
    std::string last_error() const;

private:
    friend class HikariPlugin;
    hk_shared_scene* scene_ = nullptr;   // a shared scene of its own, or
    hk_context* ctx_ = nullptr;          // the context whose private scene the hk_scene_* calls write
    int upload_desc(const hk_scene_desc& d);
    int update_instances_desc(const hk_scene_desc& d);
    int update_transforms_arrays(const float* models, const float* previous_models, const float* mesh_aabbs, uint32_t instance_count);
};

// HikariPlugin: owns the context of one camera, uploads noise + scene, runs the "hikari" sub-graph each frame.
class HikariPlugin {                          // lib.rs:95-370
public:
    HikariPlugin() = default;
    ~HikariPlugin();
    HikariPlugin(const HikariPlugin&) = delete;
    HikariPlugin& operator=(const HikariPlugin&) = delete;
    int build(int cuda_device, uint32_t width, uint32_t height, uint32_t row_begin, uint32_t row_end,
              const uint8_t* noise_rgba8_64x64x16, void* cuda_stream);
    // same for a rectangular tile of the camera target (multi-GPU sharding in two dimensions)
    int build_tile(int cuda_device, uint32_t width, uint32_t height, uint32_t col_begin, uint32_t col_end, uint32_t row_begin,
                   uint32_t row_end, const uint8_t* noise_rgba8_64x64x16, void* cuda_stream);
    int upload_scene(const MeshMaterialWorld& world);
    // instance-level buffers only (hk_scene_update_instances): what instance.rs:427-435 rewrites when instances change
    int update_instances(const MeshMaterialWorld& world);
    // Animated instances through the device-side rebuild (hk_scene_update_transforms) whenever only transforms changed since the
    // last prepare_instances; otherwise world.prepare_instances() + hk_scene_update_instances.  *used_device_path says which.
    int update_transforms(MeshMaterialWorld& world, bool* used_device_path = nullptr);
    // HikariScene::add_meshes on the camera's private scene
    int add_meshes(const MeshMaterialWorld& world, const uint32_t* ids, uint32_t n, hk_mesh_index* out);
    // Render `scene` (a HikariScene after create()) instead of the camera's private scene; the reservoirs are kept.  From then on the
    // plugin's own upload / update calls are refused: the scene is updated once per frame through `scene` for every camera.
    int attach_scene(HikariScene& scene);
    // Back to a private scene (HK_ERR_NOT_READY until the next upload_scene).
    int detach_scene();
    // One frame of the camera's sub-graph: PREPASS -> LIGHT -> POST_PROCESS (lib.rs:258-365).  Increments the counter
    // first, as frame_counter_system does in PostUpdate (view.rs:89-103).
    int run_frame(const HikariSettings& settings, const ViewInputs& view);
    hk_context* context() const { return ctx_; }
    FrameCounter counter;
    // Run the temporal upscalers after tone mapping — smaa_tu4x (+ extrapolate) under Upscale::SmaaTu4x, taa_jasmine under
    // Taa::Jasmine, FSR1 EASU + RCAS under Upscale::Fsr1 — exactly when `settings` select them, as PostProcessNode::run does
    // (post_process.rs:1236-1308).  On by default: HikariSettings::default() then gives the reference's default pipeline end to
    // end.  A caller that ends the path at the tone-mapped image (the sharded benchmark; SURVEY 8(d) runs SmaaTu4x{ratio 1}
    // without the upscale passes) sets it to false; run_frame then also drops the prepass jitter those passes would resolve.
    // Tiles: the upscalers need hk_context_enable_tile_upscalers + a motion margin (HK_ERR_UNSUPPORTED otherwise), and
    // upscale ratios above 1 / FSR1 need a full-frame context.
    bool temporal_upscalers = true;
    std::string last_error() const;

private:
    hk_context* ctx_ = nullptr;
    HikariScene scene_;                  // the private scene, through ctx_
};

}  // namespace hikari
