"""ctypes bindings of libhikari_b200.so (include/hikari_b200.h + include/hikari_host.h).

The library is the product: if it is missing this module raises — there is no Python / CPU fallback for the path."""
import ctypes as C
import os

from . import layout as L

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libhikari_b200.so")   # the product library (CUDA + C ABI); there is no fallback if it is missing
EXACT_LIB_PATH = os.path.join(HERE, "libhikari_b200_exact.so")   # same sources, exact arithmetic in every unit: the 0-ulp parity suite
DEFAULT_FLAVOR = "product"    # tests/conftest.py switches the default to "exact"; the tolerance gate asks for "product" explicitly
HOST_LIB_PATH = os.path.join(HERE, "libhikari_host.so")   # the host mirror up to hikari_make_frame_inputs: pure CPU, no CUDA

HK_OK = 0
HK_ERR_INVALID_ARGUMENT, HK_ERR_CUDA, HK_ERR_NOT_READY, HK_ERR_OUT_OF_MEMORY, HK_ERR_UNSUPPORTED = -1, -2, -3, -4, -5

# every symbol the two headers declare: name -> (restype, argtypes)
_P = C.c_void_p
_U32, _I, _SZ, _U64 = C.c_uint32, C.c_int, C.c_size_t, C.c_uint64


class Settings(C.Structure):
    """hikari_settings (include/hikari_host.h) == HikariSettings, src/lib.rs:399-433."""
    _fields_ = [("direct_validate_interval", _U32), ("emissive_validate_interval", _U32),
                ("max_temporal_reuse_count", _U32), ("max_spatial_reuse_count", _U32),
                ("max_reservoir_lifetime", C.c_float), ("solar_angle", C.c_float), ("indirect_bounces", _U32),
                ("max_indirect_luminance", C.c_float), ("clear_color", C.c_float * 4), ("temporal_reuse", _U32),
                ("emissive_spatial_reuse", _U32), ("indirect_spatial_reuse", _U32), ("denoise", _U32), ("taa", _U32),
                ("upscale_kind", _U32), ("upscale_ratio", C.c_float), ("upscale_sharpness", C.c_float)]


SYMBOLS = {
    # include/hikari_b200.h
    "hk_context_create": (_I, [C.POINTER(_P), _I, _U32, _U32, _U32, _U32, _P]),
    "hk_context_create_tile": (_I, [C.POINTER(_P), _I, _U32, _U32, _U32, _U32, _U32, _U32, _P]),
    "hk_context_destroy": (None, [_P]),
    "hk_context_resize": (_I, [_P, _U32, _U32, _U32, _U32]),
    "hk_context_resize_tile": (_I, [_P, _U32, _U32, _U32, _U32, _U32, _U32]),
    "hk_reset_temporal_state": (_I, [_P]),
    "hk_scene_upload": (_I, [_P, C.POINTER(L.SceneDesc)]),
    "hk_scene_update_instances": (_I, [_P, C.POINTER(L.SceneDesc)]),
    "hk_set_noise": (_I, [_P, _P]),
    "hk_import_gbuffer": (_I, [_P, _P]),
    "hk_prepass_run": (_I, [_P, C.POINTER(L.FrameInputs)]),
    "hk_light_run": (_I, [_P, C.POINTER(L.FrameInputs)]),
    "hk_post_process_run": (_I, [_P, C.POINTER(L.FrameInputs)]),
    "hk_render_frame": (_I, [_P, C.POINTER(L.FrameInputs)]),
    "hk_get_output": (_I, [_P, _I, C.POINTER(_P), C.POINTER(_SZ)]),
    "hk_output_extent": (_I, [_P, _I, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "hk_readback": (_I, [_P, _I, _P, _SZ]),
    "hk_readback_async": (_I, [_P, _I, _P, _SZ]),
    "hk_readback_wait": (_I, [_P]),
    "hk_context_set_motion_margin": (_I, [_P, _U32]),
    "hk_halo_pull": (_I, [_P, _P]),
    "hk_context_enable_tile_upscalers": (_I, [_P, _I]),
    "hk_halo_export": (_I, [_P, _P]),
    "hk_halo_import": (_I, [_P, _P, C.POINTER(_P)]),
    "hk_halo_pull_peer": (_I, [_P, _P]),
    "hk_set_frame_target": (_I, [_P, _P, _U32]),
    "hk_frame_alloc": (_I, [_P, C.POINTER(_P), _P]),
    "hk_frame_open": (_I, [_P, _P, C.POINTER(_P)]),
    "hk_frame_read": (_I, [_P, _P, _P, _SZ]),
    "hk_upload_state": (_I, [_P, _I, _P, _SZ]),
    "hk_scene_update_transforms": (_I, [_P, _P, _P, _P, _U32]),
    "hk_scene_add_meshes": (_I, [_P, _P, _U32, _P]),
    "hk_scene_readback": (_I, [_P, _I, _P, _SZ]),
    "hk_scene_buffer_bytes": (_I, [_P, _I, C.POINTER(_SZ)]),
    "hk_shared_scene_create": (_I, [C.POINTER(_P), _I, _P]),
    "hk_shared_scene_destroy": (None, [_P]),
    "hk_shared_scene_upload": (_I, [_P, C.POINTER(L.SceneDesc)]),
    "hk_shared_scene_update_instances": (_I, [_P, C.POINTER(L.SceneDesc)]),
    "hk_shared_scene_update_transforms": (_I, [_P, _P, _P, _P, _U32]),
    "hk_shared_scene_add_meshes": (_I, [_P, _P, _U32, _P]),
    "hk_shared_scene_last_error": (C.c_char_p, [_P]),
    "hk_context_attach_scene": (_I, [_P, _P]),
    "hk_sync": (_I, [_P]),
    "hk_trace_rays": (_I, [_P, _P, _SZ, _P]),
    "hk_set_profiling": (_I, [_P, _I, _I]),
    "hk_set_profiling_kernel": (_I, [_P, _I]),
    "hk_set_tuning": (_I, [_P, _I, _I]),
    "hk_run_pass": (_I, [_P, C.POINTER(L.FrameInputs), _I, _I]),
    "hk_set_keep_intermediates": (_I, [_P, _I]),
    "hk_get_stats": (_I, [_P, C.POINTER(L.FrameStats)]),
    "hk_band_rows": (_I, [_P, C.POINTER(_U32), C.POINTER(_U32)]),
    "hk_tile_rect": (_I, [_P, C.POINTER(_U32 * 4), C.POINTER(_U32 * 4)]),
    "hk_last_error": (C.c_char_p, [_P]),
    "hk_version": (C.c_char_p, []),
    # include/hikari_host.h
    "hikari_settings_default": (None, [C.POINTER(Settings)]),
    "hikari_upscale_ratio": (C.c_float, [C.POINTER(Settings)]),
    "hikari_make_frame_inputs": (None, [C.POINTER(Settings), _U64, C.POINTER(L.View), C.POINTER(L.PreviousView),
                                        C.POINTER(L.Lights), C.POINTER(L.FrameInputs)]),
    "hikari_graph_name": (C.c_char_p, []),
    "hikari_world_create": (_P, []),
    "hikari_world_destroy": (None, [_P]),
    "hikari_world_add_mesh": (_U32, [_P, _P, _P, _P, _U32, _P, _U32, _U32]),
    "hikari_world_add_device_mesh": (_U32, [_P, _P, _P, _P, _U32, _P, _U32, _U32]),
    "hikari_world_add_material": (_U32, [_P, _P]),
    "hikari_world_add_texture": (_U32, [_P, C.POINTER(L.TextureDesc)]),
    "hikari_world_add_instance": (_U32, [_P, _U32, _U32, _P, _U32]),
    "hikari_world_set_material": (None, [_P, _U32, _P]),
    "hikari_world_prepare_materials": (None, [_P]),
    "hikari_world_prepare": (None, [_P]),
    "hikari_world_prepare_instances": (None, [_P]),
    "hikari_world_set_instance_transform": (None, [_P, _U32, _P]),
    "hikari_world_set_instance_visible": (None, [_P, _U32, _U32]),
    "hikari_world_previous_transform_system": (None, [_P]),
    "hikari_world_scene_desc": (None, [_P, C.POINTER(L.SceneDesc)]),
    "hikari_world_mesh_error": (_I, [_P, _U32]),
    "hikari_world_prepare_instance_transforms": (_I, [_P, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), C.POINTER(_U32)]),
    "hikari_world_load_gltf": (_I, [_P, C.c_char_p, _P, _P, _P, _P, C.c_char_p, _SZ]),
    "hikari_decode_png": (_I, [_P, _SZ, _P, C.POINTER(_U32), C.POINTER(_U32)]),
    "hikari_world_add_shape": (_U32, [_P, _U32, _P]),
    "hikari_plugin_create": (_P, []),
    "hikari_plugin_destroy": (None, [_P]),
    "hikari_plugin_build": (_I, [_P, _I, _U32, _U32, _U32, _U32, _P, _P]),
    "hikari_plugin_build_tile": (_I, [_P, _I, _U32, _U32, _U32, _U32, _U32, _U32, _P, _P]),
    "hikari_plugin_upload_scene": (_I, [_P, _P]),
    "hikari_plugin_update_instances": (_I, [_P, _P]),
    "hikari_plugin_update_transforms": (_I, [_P, _P, C.POINTER(_I)]),
    "hikari_plugin_add_meshes": (_I, [_P, _P, _P, _U32, _P]),
    "hikari_plugin_run_frame": (_I, [_P, C.POINTER(Settings), C.POINTER(L.View), C.POINTER(L.PreviousView), C.POINTER(L.Lights)]),
    "hikari_plugin_context": (_P, [_P]),
    "hikari_plugin_frame_counter": (_U64, [_P]),
    "hikari_plugin_set_frame_counter": (None, [_P, _U64]),
    "hikari_plugin_set_temporal_upscalers": (None, [_P, _I]),
    "hikari_shared_scene_create": (_P, []),
    "hikari_shared_scene_destroy": (None, [_P]),
    "hikari_shared_scene_build": (_I, [_P, _I, _P]),
    "hikari_shared_scene_upload": (_I, [_P, _P]),
    "hikari_shared_scene_update_instances": (_I, [_P, _P]),
    "hikari_shared_scene_update_transforms": (_I, [_P, _P, C.POINTER(_I)]),
    "hikari_shared_scene_add_meshes": (_I, [_P, _P, _P, _U32, _P]),
    "hikari_shared_scene_handle": (_P, [_P]),
    "hikari_plugin_attach_scene": (_I, [_P, _P]),
}

_lib = None
_host_lib = None
# symbols of include/hikari_host.h that live in libhikari_host.so (no CUDA behind them)
HOST_ONLY = [n for n in SYMBOLS if n.startswith("hikari_") and not n.startswith(("hikari_plugin_", "hikari_shared_scene_"))]


def host_lib():
    """libhikari_host.so alone: scene preparation, settings, frame uniforms.  CPU-only consumers (bench.py --impl reference,
    the oracle's tests) use this and never map the CUDA library."""
    global _host_lib
    if _host_lib is None:
        if not os.path.exists(HOST_LIB_PATH):
            raise RuntimeError(f"{HOST_LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _host_lib = C.CDLL(HOST_LIB_PATH, mode=C.RTLD_GLOBAL)
        for name in HOST_ONLY:
            fn = getattr(_host_lib, name)
            fn.restype, fn.argtypes = SYMBOLS[name]
    return _host_lib


def lib(flavor=None):
    """the CUDA library: flavor "product" (tolerance build of the units that trace no rays, bevy_hikari_b200/build.py) or "exact";
    None = DEFAULT_FLAVOR.  An explicit LIB_PATH override (bench.py --lib, the kernel-logic emulation) serves both."""
    global _lib
    flavor = flavor or DEFAULT_FLAVOR
    if _lib is None:
        _lib = {}
    path = LIB_PATH
    if flavor == "exact" and LIB_PATH == os.path.join(HERE, "libhikari_b200.so"):
        path = EXACT_LIB_PATH
    if path not in _lib:
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(nvcc, sm_90a). There is no fallback path.")
        host_lib()                 # dependency of the CUDA library (also found through its $ORIGIN rpath)
        h = C.CDLL(path)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(h, name)   # AttributeError if the library does not export a declared symbol
            fn.restype, fn.argtypes = res, args
        _lib[path] = h
    return _lib[path]


class HikariError(RuntimeError):
    pass


def check(rc, ctx=None, handle=None):
    if rc != HK_OK:
        msg = (handle or lib()).hk_last_error(ctx)
        raise HikariError(f"hk error {rc}: {msg.decode() if msg else ''}")
