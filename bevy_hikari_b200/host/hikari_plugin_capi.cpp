// hikari_plugin_capi.cpp — extern "C" shims of HikariPlugin (declared in include/hikari_host.h); linked into
// libhikari_b200.so next to the C ABI they call.
#include <string.h>

#include "hikari.hpp"
#include "hikari_host.h"
#include "hikari_settings_convert.hpp"

using namespace hikari;

static MeshMaterialWorld* W(hikari_world* w) { return reinterpret_cast<MeshMaterialWorld*>(w); }

extern "C" {

// ---------------------------------------------------------------------------------------------- plugin
hikari_plugin* hikari_plugin_create(void) { return reinterpret_cast<hikari_plugin*>(new HikariPlugin()); }
void hikari_plugin_destroy(hikari_plugin* p) { delete reinterpret_cast<HikariPlugin*>(p); }
static HikariPlugin* P(hikari_plugin* p) { return reinterpret_cast<HikariPlugin*>(p); }
int hikari_plugin_build(hikari_plugin* p, int cuda_device, uint32_t width, uint32_t height, uint32_t row_begin,
                        uint32_t row_end, const uint8_t* noise, void* cuda_stream) {
    return P(p)->build(cuda_device, width, height, row_begin, row_end, noise, cuda_stream);
}
int hikari_plugin_build_tile(hikari_plugin* p, int cuda_device, uint32_t width, uint32_t height, uint32_t col_begin, uint32_t col_end,
                             uint32_t row_begin, uint32_t row_end, const uint8_t* noise, void* cuda_stream) {
    return P(p)->build_tile(cuda_device, width, height, col_begin, col_end, row_begin, row_end, noise, cuda_stream);
}
int hikari_plugin_upload_scene(hikari_plugin* p, hikari_world* w) { return P(p)->upload_scene(*W(w)); }
int hikari_plugin_update_instances(hikari_plugin* p, hikari_world* w) { return P(p)->update_instances(*W(w)); }
int hikari_plugin_update_transforms(hikari_plugin* p, hikari_world* w, int* used_device_path) {
    bool used = false;
    int rc = P(p)->update_transforms(*W(w), &used);
    if (used_device_path) *used_device_path = used ? 1 : 0;
    return rc;
}
int hikari_plugin_run_frame(hikari_plugin* p, const hikari_settings* s, const hk_view* view,
                            const hk_previous_view* previous_view, const hk_lights* lights) {
    ViewInputs v;
    v.view = *view; v.previous_view = *previous_view; v.lights = *lights;
    return P(p)->run_frame(to_cpp(s), v);
}
int hikari_plugin_add_meshes(hikari_plugin* p, hikari_world* w, const uint32_t* mesh_ids, uint32_t n, hk_mesh_index* out) {
    return P(p)->add_meshes(*W(w), mesh_ids, n, out);
}
hk_context* hikari_plugin_context(hikari_plugin* p) { return P(p)->context(); }
uint64_t hikari_plugin_frame_counter(hikari_plugin* p) { return P(p)->counter.value; }
void hikari_plugin_set_frame_counter(hikari_plugin* p, uint64_t v) { P(p)->counter.value = (size_t)v; }
void hikari_plugin_set_temporal_upscalers(hikari_plugin* p, int enabled) { P(p)->temporal_upscalers = enabled != 0; }

// ---------------------------------------------------------------------------------------------- shared scene
static HikariScene* S(hikari_shared_scene* s) { return reinterpret_cast<HikariScene*>(s); }
hikari_shared_scene* hikari_shared_scene_create(void) { return reinterpret_cast<hikari_shared_scene*>(new HikariScene()); }
void hikari_shared_scene_destroy(hikari_shared_scene* s) { delete S(s); }
int hikari_shared_scene_build(hikari_shared_scene* s, int cuda_device, void* cuda_stream) { return S(s)->create(cuda_device, cuda_stream); }
int hikari_shared_scene_upload(hikari_shared_scene* s, hikari_world* w) { return S(s)->upload(*W(w)); }
int hikari_shared_scene_update_instances(hikari_shared_scene* s, hikari_world* w) { return S(s)->update_instances(*W(w)); }
int hikari_shared_scene_update_transforms(hikari_shared_scene* s, hikari_world* w, int* used_device_path) {
    bool used = false;
    int rc = S(s)->update_transforms(*W(w), &used);
    if (used_device_path) *used_device_path = used ? 1 : 0;
    return rc;
}
int hikari_shared_scene_add_meshes(hikari_shared_scene* s, hikari_world* w, const uint32_t* mesh_ids, uint32_t n, hk_mesh_index* out) {
    return S(s)->add_meshes(*W(w), mesh_ids, n, out);
}
hk_shared_scene* hikari_shared_scene_handle(hikari_shared_scene* s) { return S(s)->handle(); }
int hikari_plugin_attach_scene(hikari_plugin* p, hikari_shared_scene* s) { return s ? P(p)->attach_scene(*S(s)) : P(p)->detach_scene(); }

}  // extern "C"
