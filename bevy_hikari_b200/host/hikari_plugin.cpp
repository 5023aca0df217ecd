// hikari_plugin.cpp — the part of the host mirror that CALLS the C ABI: the three render-graph nodes and HikariPlugin.
// Linked into libhikari_b200.so; everything else of the mirror (scene preparation, settings, frame uniforms) is in
// libhikari_host.so, which has no CUDA dependency at all (the CPU reference arm of bench.py loads only that one).
#include <algorithm>

#include "hikari.hpp"

namespace hikari {

int PrepassNode::run(hk_context* ctx, const hk_frame_inputs& in) { return hk_prepass_run(ctx, &in); }
int LightNode::run(hk_context* ctx, const hk_frame_inputs& in) { return hk_light_run(ctx, &in); }
int PostProcessNode::run(hk_context* ctx, const hk_frame_inputs& in) { return hk_post_process_run(ctx, &in); }

HikariScene::~HikariScene() { if (scene_) hk_shared_scene_destroy(scene_); }
int HikariScene::create(int cuda_device, void* cuda_stream) {
    if (scene_) { hk_shared_scene_destroy(scene_); scene_ = nullptr; }
    ctx_ = nullptr;
    return hk_shared_scene_create(&scene_, cuda_device, cuda_stream);
}
int HikariScene::upload_desc(const hk_scene_desc& d) {
    if (scene_) return hk_shared_scene_upload(scene_, &d);
    return ctx_ ? hk_scene_upload(ctx_, &d) : HK_ERR_NOT_READY;
}
int HikariScene::update_instances_desc(const hk_scene_desc& d) {
    if (scene_) return hk_shared_scene_update_instances(scene_, &d);
    return ctx_ ? hk_scene_update_instances(ctx_, &d) : HK_ERR_NOT_READY;
}
int HikariScene::update_transforms_arrays(const float* models, const float* previous_models, const float* mesh_aabbs, uint32_t instance_count) {
    if (scene_) return hk_shared_scene_update_transforms(scene_, models, previous_models, mesh_aabbs, instance_count);
    return ctx_ ? hk_scene_update_transforms(ctx_, models, previous_models, mesh_aabbs, instance_count) : HK_ERR_NOT_READY;
}
int HikariScene::upload(const MeshMaterialWorld& world) { return upload_desc(world.scene_desc()); }
int HikariScene::update_instances(const MeshMaterialWorld& world) { return update_instances_desc(world.scene_desc()); }
int HikariScene::update_transforms(MeshMaterialWorld& world, bool* used_device_path) {
    if (!scene_ && !ctx_) return HK_ERR_NOT_READY;
    if (world.prepare_instance_transforms()) {
        int rc = update_transforms_arrays(world.transform_models.data(), world.transform_previous.data(), world.transform_aabbs.data(),
                                          (uint32_t)(world.transform_models.size() / 16));
        if (rc != HK_ERR_UNSUPPORTED) {      // (a TLAS that is not in bvh 0.7.1's layout keeps the host path)
            if (used_device_path) *used_device_path = true;
            return rc;
        }
    }
    if (used_device_path) *used_device_path = false;
    world.prepare_instances();
    return update_instances(world);
}
int HikariScene::add_meshes(const MeshMaterialWorld& world, const uint32_t* ids, uint32_t n, hk_mesh_index* out) {
    if (!scene_ && !ctx_) return HK_ERR_NOT_READY;
    std::vector<hk_mesh_source> src(n);
    for (uint32_t i = 0; i < n; ++i) {
        const Mesh& m = world.mesh(ids[i]);
        hk_mesh_source& s = src[i];
        s.positions = m.positions.empty() ? nullptr : m.positions[0].data(); s.position_count = (uint32_t)m.positions.size();
        s.normals = m.normals.empty() ? nullptr : m.normals[0].data(); s.normal_count = (uint32_t)m.normals.size();
        s.uvs = m.uvs.empty() ? nullptr : m.uvs[0].data(); s.uv_count = (uint32_t)m.uvs.size();
        static const uint32_t none = 0;
        s.indices = m.has_indices ? (m.indices.empty() ? &none : m.indices.data()) : nullptr;
        s.index_count = (uint32_t)m.indices.size();
        s.topology = m.topology == PrimitiveTopology::TriangleList ? HK_TOPOLOGY_TRIANGLE_LIST
                     : (m.topology == PrimitiveTopology::TriangleStrip ? HK_TOPOLOGY_TRIANGLE_STRIP : 0xFFFFFFFFu);
    }
    std::vector<hk_mesh_index> got(n);
    const int rc = scene_ ? hk_shared_scene_add_meshes(scene_, src.data(), n, got.data()) : hk_scene_add_meshes(ctx_, src.data(), n, got.data());
    if (rc == HK_OK && out) std::copy(got.begin(), got.end(), out);
    return rc;
}
std::string HikariScene::last_error() const {
    if (scene_) return hk_shared_scene_last_error(scene_);
    return ctx_ ? hk_last_error(ctx_) : "";
}

HikariPlugin::~HikariPlugin() { if (ctx_) hk_context_destroy(ctx_); }
int HikariPlugin::build(int cuda_device, uint32_t width, uint32_t height, uint32_t row_begin, uint32_t row_end,
                        const uint8_t* noise, void* cuda_stream) {
    return build_tile(cuda_device, width, height, 0, width, row_begin, row_end, noise, cuda_stream);
}
int HikariPlugin::build_tile(int cuda_device, uint32_t width, uint32_t height, uint32_t col_begin, uint32_t col_end,
                             uint32_t row_begin, uint32_t row_end, const uint8_t* noise, void* cuda_stream) {
    if (ctx_) { hk_context_destroy(ctx_); ctx_ = nullptr; }
    scene_.ctx_ = nullptr;
    int e = hk_context_create_tile(&ctx_, cuda_device, width, height, col_begin, col_end, row_begin, row_end, cuda_stream);
    if (e != HK_OK) return e;
    scene_.ctx_ = ctx_;
    counter.value = 0;
    return hk_set_noise(ctx_, noise);
}
int HikariPlugin::upload_scene(const MeshMaterialWorld& world) { return scene_.upload(world); }
int HikariPlugin::update_instances(const MeshMaterialWorld& world) { return scene_.update_instances(world); }
int HikariPlugin::update_transforms(MeshMaterialWorld& world, bool* used_device_path) { return scene_.update_transforms(world, used_device_path); }
int HikariPlugin::add_meshes(const MeshMaterialWorld& world, const uint32_t* ids, uint32_t n, hk_mesh_index* out) {
    return scene_.add_meshes(world, ids, n, out);
}
int HikariPlugin::attach_scene(HikariScene& scene) {
    if (!ctx_) return HK_ERR_NOT_READY;
    if (!scene.handle()) return HK_ERR_INVALID_ARGUMENT;     // a camera's private scene is not shared
    return hk_context_attach_scene(ctx_, scene.handle());
}
int HikariPlugin::detach_scene() { return ctx_ ? hk_context_attach_scene(ctx_, nullptr) : HK_ERR_NOT_READY; }
int HikariPlugin::run_frame(const HikariSettings& settings, const ViewInputs& view) {
    if (!ctx_) return HK_ERR_NOT_READY;
    counter.value += 1;
    hk_frame_inputs in = make_frame_inputs(settings, counter, view);
    // The reference runs smaa_tu4x / taa_jasmine / FSR1 whenever the settings select them (post_process.rs:1236-1308), so that
    // is the default here too.  A caller that ends the path at the tone-mapped image (the sharded benchmark) opts out; the
    // prepass jitter only makes sense with the passes that resolve it, so it is switched off with them.
    in.temporal_upscalers = temporal_upscalers ? 1u : 0u;
    if (!temporal_upscalers) in.taa_jitter = 0u;
    return hk_render_frame(ctx_, &in);
}
std::string HikariPlugin::last_error() const { return hk_last_error(ctx_); }

}  // namespace hikari
