"""numpy dtypes of the records in include/hk_layout.h (std430 layouts of the reference,
src/shaders/mesh_material_types.wgsl:3-83, src/shaders/light.wgsl:35-43, src/shaders/mesh_view_types.wgsl:3-25)
and ctypes mirrors of the structs in include/hikari_b200.h."""
import ctypes as C

import numpy as np

f4, u4 = np.float32, np.uint32

NODE = np.dtype({"names": ["min", "entry_index", "max", "exit_index"],
                 "formats": [(f4, 3), u4, (f4, 3), u4], "offsets": [0, 12, 16, 28], "itemsize": 32})
PRIMITIVE_VERTEX = np.dtype({"names": ["position", "index"], "formats": [(f4, 3), u4], "offsets": [0, 12], "itemsize": 16})
PRIMITIVE = np.dtype({"names": ["vertices"], "formats": [(PRIMITIVE_VERTEX, 3)], "offsets": [0], "itemsize": 48})
VERTEX = np.dtype({"names": ["position", "u", "normal", "v"], "formats": [(f4, 3), f4, (f4, 3), f4],
                   "offsets": [0, 12, 16, 28], "itemsize": 32})
MESH_INDEX = np.dtype({"names": ["vertex", "primitive", "node_offset", "node_count"], "formats": [u4] * 4,
                       "offsets": [0, 4, 8, 12], "itemsize": 16})
INSTANCE = np.dtype({"names": ["min", "material", "max", "node_index", "model", "inverse_transpose_model", "mesh"],
                     "formats": [(f4, 3), u4, (f4, 3), u4, (f4, 16), (f4, 16), MESH_INDEX],
                     "offsets": [0, 12, 16, 28, 32, 96, 160], "itemsize": 176})
MATERIAL = np.dtype({"names": ["base_color", "base_color_texture", "emissive", "emissive_texture", "perceptual_roughness",
                               "metallic", "metallic_roughness_texture", "reflectance", "normal_map_texture",
                               "occlusion_texture"],
                     "formats": [(f4, 4), u4, (f4, 4), u4, f4, f4, u4, f4, u4, u4],
                     "offsets": [0, 16, 32, 48, 52, 56, 60, 64, 68, 72], "itemsize": 80})
ALIAS_ENTRY = np.dtype({"names": ["prob", "index"], "formats": [f4, u4], "offsets": [0, 4], "itemsize": 8})
EMISSIVE = np.dtype({"names": ["emissive", "position", "radius", "instance", "alias_table_offset", "alias_table_count",
                               "surface_area", "node_index"],
                     "formats": [(f4, 4), (f4, 3), f4, u4, u4, u4, f4, u4],
                     "offsets": [0, 16, 28, 32, 40, 44, 48, 52], "itemsize": 64})
PACKED_RESERVOIR = np.dtype({"names": ["radiance", "random", "visible_position", "sample_position", "visible_normal",
                                       "sample_normal", "reservoir"],
                             "formats": [(u4, 2), (u4, 2), (f4, 4), (f4, 4), u4, u4, (u4, 2)],
                             "offsets": [0, 8, 16, 32, 48, 52, 56], "itemsize": 64})

assert NODE.itemsize == 32 and PRIMITIVE.itemsize == 48 and VERTEX.itemsize == 32 and INSTANCE.itemsize == 176
assert MATERIAL.itemsize == 80 and EMISSIVE.itemsize == 64 and PACKED_RESERVOIR.itemsize == 64

SCENE_BUFFERS = (("vertices", VERTEX), ("primitives", PRIMITIVE), ("asset_nodes", NODE), ("alias_table", ALIAS_ENTRY),
                 ("instances", INSTANCE), ("instance_nodes", NODE), ("materials", MATERIAL), ("emissive_nodes", NODE),
                 ("emissives", EMISSIVE))


# ------------------------------------------------------------------------------------------ ctypes structs
class FrameUniform(C.Structure):
    _fields_ = [("kernel", (C.c_float * 4) * 3), ("halton", (C.c_float * 4) * 8), ("clear_color", C.c_float * 4),
                ("number", C.c_uint32), ("direct_validate_interval", C.c_uint32), ("emissive_validate_interval", C.c_uint32),
                ("indirect_bounces", C.c_uint32), ("temporal_reuse", C.c_uint32), ("emissive_spatial_reuse", C.c_uint32),
                ("indirect_spatial_reuse", C.c_uint32), ("max_temporal_reuse_count", C.c_uint32),
                ("max_spatial_reuse_count", C.c_uint32), ("max_reservoir_lifetime", C.c_float), ("solar_angle", C.c_float),
                ("max_indirect_luminance", C.c_float), ("upscale_ratio", C.c_float), ("_pad", C.c_uint32 * 3)]


class PreviousView(C.Structure):
    _fields_ = [("view_proj", C.c_float * 16), ("inverse_view_proj", C.c_float * 16)]


class View(C.Structure):
    _fields_ = [("view_proj", C.c_float * 16), ("inverse_view_proj", C.c_float * 16), ("view", C.c_float * 16),
                ("inverse_view", C.c_float * 16), ("projection", C.c_float * 16), ("inverse_projection", C.c_float * 16),
                ("world_position", C.c_float * 3), ("_pad0", C.c_float), ("viewport", C.c_float * 4)]


class Lights(C.Structure):
    _fields_ = [("directional_color", C.c_float * 4), ("direction_to_light", C.c_float * 3), ("_pad0", C.c_float),
                ("ambient_color", C.c_float * 4)]


class FrameInputs(C.Structure):
    _fields_ = [("frame", FrameUniform), ("view", View), ("previous_view", PreviousView), ("lights", Lights),
                ("denoise", C.c_uint32), ("taa_jitter", C.c_uint32), ("smaa_tu4x", C.c_uint32), ("temporal_upscalers", C.c_uint32),
                ("fsr1", C.c_uint32), ("fsr_sharpness", C.c_float)]


class TextureDesc(C.Structure):
    _fields_ = [("rgba8", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32), ("address_mode_u", C.c_uint32),
                ("address_mode_v", C.c_uint32), ("filter_linear", C.c_uint32), ("srgb", C.c_uint32)]


class SceneDesc(C.Structure):
    _fields_ = [("vertices", C.c_void_p), ("vertex_count", C.c_uint32),
                ("primitives", C.c_void_p), ("primitive_count", C.c_uint32),
                ("asset_nodes", C.c_void_p), ("asset_node_count", C.c_uint32),
                ("alias_table", C.c_void_p), ("alias_count", C.c_uint32),
                ("instances", C.c_void_p), ("instance_count", C.c_uint32),
                ("instance_nodes", C.c_void_p), ("instance_node_count", C.c_uint32),
                ("materials", C.c_void_p), ("material_count", C.c_uint32),
                ("emissive_nodes", C.c_void_p), ("emissive_node_count", C.c_uint32),
                ("emissives", C.c_void_p), ("emissive_count", C.c_uint32),
                ("textures", C.c_void_p), ("texture_count", C.c_uint32),
                ("previous_instance_models", C.c_void_p)]


class FrameStats(C.Structure):
    _fields_ = [("primary_rays", C.c_uint64), ("tlas_rays", C.c_uint64), ("blas_rays", C.c_uint64),
                ("ms_prepass", C.c_float), ("ms_light", C.c_float), ("ms_post_process", C.c_float), ("ms_total", C.c_float),
                ("kernel_launches", C.c_uint32), ("timed_frames", C.c_uint32), ("ms_kernel", C.c_float * 16),
                ("wide_traversal", C.c_uint32), ("wide_stack_need", C.c_uint32)]


KERNEL_NAMES = ["gbuffer", "direct", "emissive", "emissive_spatial", "indirect", "indirect_spatial", "demodulation",
                "denoise_0", "denoise_1", "denoise_2", "denoise_3", "tone_mapping", "smaa_tu4x", "taa", "fsr1"]


RAY = np.dtype({"names": ["origin", "max_distance", "direction", "early_distance", "exclude_instance"],
                "formats": [(f4, 3), f4, (f4, 3), f4, u4], "offsets": [0, 12, 16, 28, 32], "itemsize": 48})
HIT = np.dtype({"names": ["u", "v", "distance", "instance_index", "primitive_index"],
                "formats": [f4, f4, f4, u4, u4], "offsets": [0, 4, 8, 12, 16], "itemsize": 20})

assert C.sizeof(FrameUniform) == 256 and C.sizeof(PreviousView) == 128
assert C.sizeof(View) == 6 * 64 + 32 and C.sizeof(Lights) == 48

# hk_get_output / hk_readback identifiers (include/hikari_b200.h)
OUT_TONE_MAPPED, OUT_RENDER_DIRECT, OUT_RENDER_EMISSIVE, OUT_RENDER_INDIRECT = 0, 1, 2, 3
OUT_VARIANCE_DIRECT, OUT_VARIANCE_EMISSIVE, OUT_VARIANCE_INDIRECT, OUT_ALBEDO = 4, 5, 6, 7
OUT_DENOISED_DIRECT, OUT_DENOISED_EMISSIVE, OUT_DENOISED_INDIRECT = 8, 9, 10
OUT_UPSCALED, OUT_TAA, OUT_FSR_SHARPENED = 11, 12, 13
OUT_GBUFFER_POSITION, OUT_GBUFFER_NORMAL, OUT_GBUFFER_DEPTH_GRADIENT = 16, 17, 18
OUT_GBUFFER_INSTANCE_MATERIAL, OUT_GBUFFER_VELOCITY_UV = 19, 20
OUT_RESERVOIR_0 = 32
SCENE_INSTANCES, SCENE_INSTANCE_NODES, SCENE_EMISSIVES, SCENE_EMISSIVE_NODES, SCENE_PREVIOUS_MODELS, SCENE_INSTANCE_MOVED = range(6)   # hk_scene_readback
SCENE_WIDE_TLAS, SCENE_WIDE_INSTANCE_RANK = 6, 7
SCENE_VERTICES, SCENE_PRIMITIVES, SCENE_ASSET_NODES = 8, 9, 10
TOPOLOGY_TRIANGLE_LIST, TOPOLOGY_TRIANGLE_STRIP = 0, 1


class MeshSource(C.Structure):
    """hk_mesh_source (include/hikari_b200.h): one mesh for hk_scene_add_meshes."""
    _fields_ = [("positions", C.c_void_p), ("position_count", C.c_uint32), ("normals", C.c_void_p), ("normal_count", C.c_uint32),
                ("uvs", C.c_void_p), ("uv_count", C.c_uint32), ("indices", C.c_void_p), ("index_count", C.c_uint32),
                ("topology", C.c_uint32)]
WIDE_NODE = np.dtype([("lo_x", f4, 4), ("lo_y", f4, 4), ("lo_z", f4, 4), ("hi_x", f4, 4), ("hi_y", f4, 4), ("hi_z", f4, 4),
                      ("child", u4, 4), ("pad", u4, 4)])      # hk_wide_node (csrc/hk_wide.cuh), 128 bytes
assert WIDE_NODE.itemsize == 128

# bytes per pixel and numpy view of each read-back plane
OUT_FORMATS = {}
for _k in (0, 1, 2, 3, 7, 8, 9, 10, 11, 12, 13):
    OUT_FORMATS[_k] = (8, np.float16, 4)
for _k in (4, 5, 6):
    OUT_FORMATS[_k] = (4, np.float32, 1)
OUT_FORMATS[16] = (16, np.float32, 4)
OUT_FORMATS[17] = (4, np.int8, 4)
OUT_FORMATS[18] = (8, np.float32, 2)
OUT_FORMATS[19] = (8, np.float32, 2)
OUT_FORMATS[20] = (16, np.float32, 4)
for _k in range(32, 42):
    OUT_FORMATS[_k] = (64, PACKED_RESERVOIR, 1)
