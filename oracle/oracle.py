"""ORACLE (test infrastructure): ctypes wrapper of oracle/libhk_oracle.so, the CPU restatement of the reference's
per-frame passes (oracle/hk_oracle.cpp).  Imported only by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs — never by the product package."""
import ctypes as C
import os
import subprocess

import numpy as np

from bevy_hikari_b200 import layout as L

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libhk_oracle.so")
_P, _I, _U32, _SZ = C.c_void_p, C.c_int, C.c_uint32, C.c_size_t


def build(force=False):
    src = [os.path.join(HERE, "hk_oracle.cpp")] + [os.path.join(HERE, "..", "include", h)
                                                   for h in ("hk_math.h", "hk_layout.h", "hikari_b200.h")]
    if force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in src):
        r = subprocess.run(["make", "-C", HERE, "-B", "libhk_oracle.so"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("oracle build failed:\n" + r.stdout + r.stderr)
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        _lib = C.CDLL(LIB_PATH)
        sig = {
            "hko_context_create": (_I, [C.POINTER(_P), _U32, _U32, _I]),
            "hko_context_destroy": (None, [_P]),
            "hko_reset_temporal_state": (_I, [_P]),
            "hko_scene_upload": (_I, [_P, C.POINTER(L.SceneDesc)]),
            "hko_scene_update_instances": (_I, [_P, C.POINTER(L.SceneDesc)]),
            "hko_set_noise": (_I, [_P, _P]),
            "hko_prepass_run": (_I, [_P, C.POINTER(L.FrameInputs)]),
            "hko_light_run": (_I, [_P, C.POINTER(L.FrameInputs)]),
            "hko_post_process_run": (_I, [_P, C.POINTER(L.FrameInputs)]),
            "hko_render_frame": (_I, [_P, C.POINTER(L.FrameInputs)]),
            "hko_run_pass": (_I, [_P, C.POINTER(L.FrameInputs), _I, _I]),
            "hko_output_extent": (_I, [_P, _I, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
            "hko_readback": (_I, [_P, _I, _P, _SZ]),
            "hko_upload_state": (_I, [_P, _I, _P, _SZ]),
            "hko_trace_rays": (_I, [_P, _P, _SZ, _P]),
            "hko_get_stats": (_I, [_P, C.POINTER(L.FrameStats)]),
            "hko_trace_steps": (_I, [_P, _P, _SZ, _P]),
            "hko_last_error": (C.c_char_p, [_P]),
            "hko_math_lit": (None, [_P, _P, C.c_float, _P, _P, _P, _P, _P]),
            "hko_math_env_brdf_approx": (None, [_P, C.c_float, C.c_float, _P]),
            "hko_math_perceptual_roughness_to_roughness": (C.c_float, [C.c_float]),
            "hko_math_exp2": (C.c_float, [C.c_float]),
            "hko_math_exp": (C.c_float, [C.c_float]),
            "hko_math_sincos": (None, [C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
            "hko_math_pack2x16float": (_U32, [C.c_float, C.c_float]),
            "hko_math_f16_to_f32": (C.c_float, [C.c_uint16]),
            "hko_math_pack4x8snorm": (_U32, [C.c_float] * 4),
            "hko_math_pack2x16unorm": (_U32, [C.c_float, C.c_float]),
            "hko_math_hash": (_U32, [_U32]),
            "hko_math_unsnorm8": (C.c_float, [_U32]),
            "hko_math_unorm8": (C.c_float, [_U32]),
            "hko_math_unorm16": (C.c_float, [_U32]),
            "hko_math_normal_basis": (None, [_P, _P]),
            "hko_pack_reservoir_roundtrip": (None, [_P, _P]),
            "hko_math_batch": (None, [_I, _P, _P, _SZ]),
            "hko_math_batch_range": (None, [_I, _U32, _P, _SZ]),
            "hko_spatial_digest": (None, [_U32, C.c_float, _I, _I, _U32, _P]),
            "hko_deferred_digest": (None, [_I, _I, C.c_float, _U32, _P]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(_lib, name)
            fn.restype, fn.argtypes = res, args
    return _lib


PASS_ALBEDO, PASS_DIRECT, PASS_EMISSIVE, PASS_EMISSIVE_SPATIAL, PASS_INDIRECT, PASS_INDIRECT_SPATIAL, PASS_DENOISE, PASS_TONE_MAPPING = range(8)


def usable_cpus():
    """Host cores this process may really use: the affinity mask capped by the cgroup CPU quota.  os.cpu_count() reports the whole
    machine (128 hardware threads on the GPU box against a 16-CPU quota); an OpenMP team of that size under the quota spends its time
    being throttled at barriers, which made the device suite's checker several times slower than the thing it checks."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    for path, parse in (("/sys/fs/cgroup/cpu.max", lambda t: None if t.split()[0] == "max" else float(t.split()[0]) / float(t.split()[1])),
                        ("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", None)):
        try:
            text = open(path).read()
            if parse is None:
                quota = int(text)
                period = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
                cap = quota / period if quota > 0 else None
            else:
                cap = parse(text)
            if cap:
                n = min(n, max(1, int(cap)))
            break
        except Exception:
            continue
    return max(1, n)


class Oracle:
    def __init__(self, width, height, noise, threads=None):
        self.width, self.height = width, height
        p = _P()
        threads = threads or usable_cpus()
        self.threads = threads
        rc = lib().hko_context_create(C.byref(p), width, height, threads)
        assert rc == 0
        self.ctx = p
        noise = np.ascontiguousarray(noise, np.uint8)
        assert lib().hko_set_noise(self.ctx, noise.ctypes.data) == 0

    def close(self):
        if getattr(self, "ctx", None):
            lib().hko_context_destroy(self.ctx)
            self.ctx = None

    __del__ = close

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(f"oracle error {rc}: {lib().hko_last_error(self.ctx).decode()}")

    def upload_scene_desc(self, desc): self._check(lib().hko_scene_upload(self.ctx, C.byref(desc)))
    def update_instances_desc(self, desc): self._check(lib().hko_scene_update_instances(self.ctx, C.byref(desc)))
    def reset_temporal_state(self): self._check(lib().hko_reset_temporal_state(self.ctx))
    def prepass(self, inputs): self._check(lib().hko_prepass_run(self.ctx, C.byref(inputs)))
    def light(self, inputs): self._check(lib().hko_light_run(self.ctx, C.byref(inputs)))
    def post_process(self, inputs): self._check(lib().hko_post_process_run(self.ctx, C.byref(inputs)))
    def render_frame(self, inputs): self._check(lib().hko_render_frame(self.ctx, C.byref(inputs)))
    def run_pass(self, inputs, which, arg=0): self._check(lib().hko_run_pass(self.ctx, C.byref(inputs), which, arg))

    def readback(self, which):
        from bevy_hikari_b200.plugin import view_plane
        bpp, dt, comps = L.OUT_FORMATS[which]
        w, h = C.c_uint32(), C.c_uint32()
        self._check(lib().hko_output_extent(self.ctx, which, C.byref(w), C.byref(h)))
        raw = np.empty(w.value * h.value * bpp, np.uint8)
        self._check(lib().hko_readback(self.ctx, which, raw.ctypes.data, raw.size))
        return view_plane(raw, which, h.value, w.value)

    def upload_state(self, which, array):
        a = np.ascontiguousarray(array)
        self._check(lib().hko_upload_state(self.ctx, which, a.ctypes.data, a.nbytes))

    def trace_rays(self, rays):
        rays = np.ascontiguousarray(rays, L.RAY)
        hits = np.zeros(len(rays), L.HIT)
        self._check(lib().hko_trace_rays(self.ctx, rays.ctypes.data, len(rays), hits.ctypes.data))
        return hits

    def trace_steps(self, rays):
        rays = np.ascontiguousarray(rays, L.RAY)
        steps = np.zeros((len(rays), 3), np.uint32)
        self._check(lib().hko_trace_steps(self.ctx, rays.ctypes.data, len(rays), steps.ctypes.data))
        return steps

    def stats(self):
        s = L.FrameStats()
        self._check(lib().hko_get_stats(self.ctx, C.byref(s)))
        return s
