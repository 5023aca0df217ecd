// hikari_capi.cpp — thin extern "C" shims over the C++ host mirror (hikari.hpp) so that Python (ctypes) tests,
// bench.py and __graft_entry__ can drive the same objects a Bevy app would.  Declared in include/hikari_host.h.
#include <string.h>

#include "hikari.hpp"
#include "hikari_host.h"

using namespace hikari;

#include "hikari_settings_convert.hpp"

extern "C" {

void hikari_settings_default(hikari_settings* out) {
    HikariSettings d;
    out->direct_validate_interval = (uint32_t)d.direct_validate_interval;
    out->emissive_validate_interval = (uint32_t)d.emissive_validate_interval;
    out->max_temporal_reuse_count = (uint32_t)d.max_temporal_reuse_count;
    out->max_spatial_reuse_count = (uint32_t)d.max_spatial_reuse_count;
    out->max_reservoir_lifetime = d.max_reservoir_lifetime;
    out->solar_angle = d.solar_angle;
    out->indirect_bounces = (uint32_t)d.indirect_bounces;
    out->max_indirect_luminance = d.max_indirect_luminance;
    for (int i = 0; i < 4; ++i) out->clear_color[i] = d.clear_color[i];
    out->temporal_reuse = d.temporal_reuse;
    out->emissive_spatial_reuse = d.emissive_spatial_reuse;
    out->indirect_spatial_reuse = d.indirect_spatial_reuse;
    out->denoise = d.denoise;
    out->taa = d.taa == Taa::None ? HIKARI_TAA_NONE : HIKARI_TAA_JASMINE;
    out->upscale_kind = d.upscale.kind == Upscale::Fsr1 ? HIKARI_UPSCALE_FSR1 : HIKARI_UPSCALE_SMAA_TU4X;
    out->upscale_ratio = d.upscale.ratio_value;
    out->upscale_sharpness = d.upscale.sharpness_value;
}

float hikari_upscale_ratio(const hikari_settings* s) { return to_cpp(s).upscale.ratio(); }

void hikari_make_frame_inputs(const hikari_settings* s, uint64_t frame_counter, const hk_view* view,
                              const hk_previous_view* previous_view, const hk_lights* lights, hk_frame_inputs* out) {
    ViewInputs v;
    v.view = *view; v.previous_view = *previous_view; v.lights = *lights;
    FrameCounter c; c.value = (size_t)frame_counter;
    *out = make_frame_inputs(to_cpp(s), c, v);
}

const char* hikari_graph_name(void) { return graph::NAME; }

// ----------------------------------------------------------------------------------------------- world
hikari_world* hikari_world_create(void) { return reinterpret_cast<hikari_world*>(new MeshMaterialWorld()); }
void hikari_world_destroy(hikari_world* w) { delete reinterpret_cast<MeshMaterialWorld*>(w); }
static MeshMaterialWorld* W(hikari_world* w) { return reinterpret_cast<MeshMaterialWorld*>(w); }

static Mesh make_mesh(const float* positions, const float* normals, const float* uvs, uint32_t vertex_count, const uint32_t* indices,
                      uint32_t index_count, uint32_t topology) {
    Mesh m;
    if (positions) { m.positions.resize(vertex_count); memcpy(m.positions.data(), positions, 12u * vertex_count); }
    if (normals) { m.normals.resize(vertex_count); memcpy(m.normals.data(), normals, 12u * vertex_count); }
    if (uvs) { m.uvs.resize(vertex_count); memcpy(m.uvs.data(), uvs, 8u * vertex_count); }
    m.has_indices = indices != nullptr;
    if (indices) m.indices.assign(indices, indices + index_count);
    m.topology = topology == 0 ? PrimitiveTopology::TriangleList
                               : (topology == 1 ? PrimitiveTopology::TriangleStrip : PrimitiveTopology::Other);
    return m;
}
uint32_t hikari_world_add_mesh(hikari_world* w, const float* positions, const float* normals, const float* uvs,
                               uint32_t vertex_count, const uint32_t* indices, uint32_t index_count, uint32_t topology) {
    return W(w)->add_mesh(make_mesh(positions, normals, uvs, vertex_count, indices, index_count, topology));
}
uint32_t hikari_world_add_device_mesh(hikari_world* w, const float* positions, const float* normals, const float* uvs,
                                      uint32_t vertex_count, const uint32_t* indices, uint32_t index_count, uint32_t topology) {
    return W(w)->add_device_mesh(make_mesh(positions, normals, uvs, vertex_count, indices, index_count, topology));
}
static StandardMaterial to_standard_material(const hk_material* m);
void hikari_world_set_material(hikari_world* w, uint32_t id, const hk_material* m) { W(w)->set_material(id, to_standard_material(m)); }
void hikari_world_prepare_materials(hikari_world* w) { W(w)->prepare_material_assets(); }
uint32_t hikari_world_add_material(hikari_world* w, const hk_material* m) { return W(w)->add_material(to_standard_material(m)); }
static StandardMaterial to_standard_material(const hk_material* m) {
    StandardMaterial s;
    memcpy(s.base_color.data(), m->base_color, 16);
    memcpy(s.emissive.data(), m->emissive, 16);
    s.perceptual_roughness = m->perceptual_roughness; s.metallic = m->metallic; s.reflectance = m->reflectance;
    s.base_color_texture = m->base_color_texture; s.emissive_texture = m->emissive_texture;
    s.metallic_roughness_texture = m->metallic_roughness_texture; s.normal_map_texture = m->normal_map_texture;
    s.occlusion_texture = m->occlusion_texture;
    return s;
}
uint32_t hikari_world_add_texture(hikari_world* w, const hk_texture_desc* t) { return W(w)->add_texture(*t, t->rgba8); }
uint32_t hikari_world_add_instance(hikari_world* w, uint32_t mesh, uint32_t material, const float* transform16, uint32_t visible) {
    InstanceDesc d;
    d.mesh = mesh; d.material = material; d.visible = visible != 0;
    memcpy(d.transform, transform16, 64);
    return W(w)->add_instance(d);
}
void hikari_world_prepare(hikari_world* w) { W(w)->prepare(); }
void hikari_world_prepare_instances(hikari_world* w) { W(w)->prepare_instances(); }
void hikari_world_set_instance_transform(hikari_world* w, uint32_t instance, const float* transform16) { W(w)->set_instance_transform(instance, transform16); }
void hikari_world_set_instance_visible(hikari_world* w, uint32_t instance, uint32_t visible) { W(w)->set_instance_visible(instance, visible != 0); }
void hikari_world_previous_transform_system(hikari_world* w) { W(w)->previous_transform_system(); }
void hikari_world_scene_desc(hikari_world* w, hk_scene_desc* out) { *out = W(w)->scene_desc(); }
int hikari_world_prepare_instance_transforms(hikari_world* w, const float** models, const float** previous_models, const float** mesh_aabbs,
                                             uint32_t* instance_count) {
    MeshMaterialWorld* world = W(w);
    if (!world->prepare_instance_transforms()) return 0;
    *models = world->transform_models.data(); *previous_models = world->transform_previous.data();
    *mesh_aabbs = world->transform_aabbs.data(); *instance_count = (uint32_t)(world->transform_models.size() / 16);
    return 1;
}
int hikari_world_mesh_error(hikari_world* w, uint32_t mesh) {
    const auto& e = W(w)->mesh_errors();
    return mesh < e.size() ? (int)e[mesh] : -1;
}

}  // extern "C"
