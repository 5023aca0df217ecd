#!/usr/bin/env python
"""Randomised parity campaign: CUDA kernel logic (emulated on the host, tests/emu/) against the oracle over random scenes,
sizes, settings, camera motion and instance animation.  Any mismatch prints the seed and the differing planes.
usage: HK_EMULATE_KERNELS=1 python tools/fuzz_parity.py [first_seed] [count]        (on a GPU box: without the variable)"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if os.environ.get("HK_EMULATE_KERNELS"):
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    from bevy_hikari_b200 import _ffi
    _ffi.LIB_PATH = build_emu.build()
from bevy_hikari_b200 import layout as L  # noqa: E402
from bevy_hikari_b200 import plugin  # noqa: E402
from tests.conftest import Animation, Bench, rotation_y_about  # noqa: E402
from tests.test_gpu_parity import ALL_PLANES, DENOISED, mismatch  # noqa: E402


def draw_tuning(seed):
    """hk_set_tuning switches that leave every output bit-exact: pooled indirect pass, tiled or gathered spatial reuse, tiled or
    gathered denoise.  From a stream of its own, so that a seed still draws the scene, size and settings it always drew."""
    rng = np.random.default_rng(seed + 2 ** 20)
    return {plugin.TUNE_POOLED_INDIRECT: int(rng.integers(0, 2)), plugin.TUNE_TILED_SPATIAL: int(rng.integers(0, 2)),
            plugin.TUNE_TILED_DENOISE: int(rng.integers(0, 2))}


def apply_tuning(devices, tuning):
    for d in devices:
        for k, v in tuning.items():
            d.set_tuning(k, v)


def one_case(seed):
    rng = np.random.default_rng(seed)
    scene = rng.choice(["cornell", "cornell", "city", "simple", "minimal"])
    if os.environ.get("HK_FUZZ_SOUP"):      # random triangle soups (degenerate triangles, mirrored / non-uniform instances, several lights)
        from bevy_hikari_b200 import scenes
        scene = f"soup{seed}"
        scenes.SCENE_BUILDERS[scene] = (lambda seed=seed: scenes.soup(seed))
    w, h = int(rng.integers(1, 97)), int(rng.integers(1, 73))
    ratio = float(rng.choice([1.0, 1.0, 1.0, 1.25, 1.5, 2.0]))
    settings = dict(
        indirect_bounces=int(rng.integers(0, 5)), temporal_reuse=int(rng.integers(0, 2)), emissive_spatial_reuse=int(rng.integers(0, 2)),
        indirect_spatial_reuse=int(rng.integers(0, 2)), denoise=int(rng.integers(0, 2)),
        direct_validate_interval=int(rng.integers(1, 6)), emissive_validate_interval=int(rng.integers(1, 6)),
        max_temporal_reuse_count=int(rng.choice([1, 2, 8, 50, 200])), max_spatial_reuse_count=int(rng.choice([1, 10, 800])),
        max_reservoir_lifetime=float(rng.choice([0.5, 1.0, 2.0, 100.0])), solar_angle=float(rng.choice([0.0, 0.046, 0.3])),
        max_indirect_luminance=float(rng.choice([0.1, 10.0, 1e6])),
        taa=int(rng.integers(0, 2)), upscale_kind=int(rng.integers(0, 2)), upscale_ratio=ratio,
        upscale_sharpness=float(rng.choice([0.0, 0.2, 1.0, 2.0])))
    upscalers = bool(rng.integers(0, 2))
    b = Bench(str(scene), w, h, **settings)
    dev, orc = b.device(), b.oracle()
    dev.set_keep_intermediates(True)
    tuning = draw_tuning(seed)
    apply_tuning([dev], tuning)
    step = tuple(rng.uniform(-0.08, 0.08, 3)) if rng.integers(0, 2) else (0.0, 0.0, 0.0)
    an = None
    if rng.integers(0, 2):
        n_inst = len(b.scene.inst_transform)
        ids = rng.choice(n_inst, size=min(2, n_inst), replace=False)
        a, t = rng.uniform(-0.2, 0.2), rng.uniform(-0.05, 0.05, 3)
        an = Animation(b, {int(i): (lambda f, a=a, t=t: rotation_y_about(a * f, (0.0, 0.5, 0.0), tuple(t * f))) for i in ids})
    planes = ALL_PLANES + (DENOISED if settings["denoise"] else [])
    if upscalers:
        # Upscale::SmaaTu4x: upscale_output[0]; Upscale::Fsr1: the EASU and RCAS images
        planes = planes + ([L.OUT_UPSCALED] if settings["upscale_kind"] == plugin.UPSCALE_SMAA_TU4X else [L.OUT_UPSCALED, L.OUT_FSR_SHARPENED]) + \
                 ([L.OUT_TAA] if settings["taa"] == plugin.TAA_JASMINE else [])
    frames = int(rng.integers(2, 7))
    for f in range(1, frames + 1):
        if an:
            wld = an.step(f)
            dev.update_instances(wld)
            orc.update_instances_desc(wld.scene_desc())
        inp = b.moving_inputs(f, step=step)
        inp.temporal_upscalers = 1 if upscalers else 0
        dev.render_frame(inp)
        orc.render_frame(inp)
        bad = {k: mismatch(dev.readback(k), orc.readback(k)) for k in planes}
        bad = {k: v for k, v in bad.items() if v}
        if bad:
            return f"seed {seed}: {scene} {w}x{h} frame {f} {settings} upscalers={upscalers} step={step} animated={an is not None} tuning={tuning} -> {bad}"
    return None


def tile_case(seed):
    """random partition of the frame into strips / a grid of tiles, static camera: every tile's owned pixels equal the
    unsharded render (tone-mapped image, radiance, the reservoirs written this frame)"""
    rng = np.random.default_rng(seed)
    scene = rng.choice(["cornell", "city", "simple"])
    w, h = int(rng.integers(40, 161)), int(rng.integers(40, 121))
    settings = dict(indirect_bounces=int(rng.integers(0, 3)), emissive_spatial_reuse=int(rng.integers(0, 2)),
                    indirect_spatial_reuse=int(rng.integers(0, 2)), denoise=int(rng.integers(0, 2)), taa=plugin.TAA_NONE, upscale_ratio=1.0)
    b = Bench(str(scene), w, h, **settings)
    xs = sorted({0, w} | {int(x) for x in rng.integers(1, w, size=int(rng.integers(0, 3)))})
    ys = sorted({0, h} | {int(y) for y in rng.integers(1, h, size=int(rng.integers(0, 3)))})
    rects = [(x0, x1, y0, y1) for x0, x1 in zip(xs[:-1], xs[1:]) for y0, y1 in zip(ys[:-1], ys[1:])]
    full = b.device()
    tiles = [b.device(r[2], r[3], r[0], r[1]) for r in rects]
    tuning = draw_tuning(seed)
    apply_tuning([full] + tiles, tuning)
    halo = bool(os.environ.get("HK_FUZZ_HALO"))       # moving camera + motion margin + halo pulls after every frame
    step = tuple(rng.uniform(-0.05, 0.05, 3)) if halo else (0.0, 0.0, 0.0)
    upscalers = halo and bool(rng.integers(0, 2))     # ... and the temporal upscalers on the tiles
    if upscalers:
        b.settings.taa = int(rng.integers(0, 2))
        b.settings.upscale_kind = int(rng.integers(0, 2))
    if halo:
        for t in tiles:
            t.set_motion_margin(16)
            if upscalers:
                t.enable_tile_upscalers()
    planes = [L.OUT_TONE_MAPPED, L.OUT_RENDER_DIRECT, L.OUT_RENDER_EMISSIVE, L.OUT_RENDER_INDIRECT] + [L.OUT_RESERVOIR_0 + i for i in range(10)]
    scaled = []
    if upscalers:
        smaa = b.settings.upscale_kind == plugin.UPSCALE_SMAA_TU4X
        scaled = ([(L.OUT_UPSCALED, 2)] if smaa else []) + ([(L.OUT_TAA, 2 if smaa else 1)] if b.settings.taa == plugin.TAA_JASMINE else [])
    for f in range(1, int(rng.integers(3, 7))):
        if f > 1 and halo:
            for t in tiles:
                for other in tiles:
                    if other is not t:
                        t.halo_pull(other)
        inp = b.moving_inputs(f, step=step)
        inp.temporal_upscalers = 1 if upscalers else 0
        inp.fsr1 = 0          # FSR1 needs a full-frame context; on tiles Upscale::Fsr1 here means "TAA only"
        full.render_frame(inp)
        for t in tiles:
            t.render_frame(inp)
        for k in planes:
            whole = full.readback(k)
            for r, t in zip(rects, tiles):
                if mismatch(t.readback(k), whole[r[2]:r[3], r[0]:r[1]]):
                    return f"tile seed {seed}: {scene} {w}x{h} rects {rects} frame {f} plane {k} {settings} tuning={tuning}"
        for k, sc in scaled:
            whole = full.readback(k)
            for r, t in zip(rects, tiles):
                if mismatch(t.readback(k), whole[sc * r[2]:sc * r[3], sc * r[0]:sc * r[1]]):
                    return f"tile seed {seed}: {scene} {w}x{h} rects {rects} frame {f} upscaled plane {k} {settings} tuning={tuning}"
    return None


if __name__ == "__main__":
    first = int(sys.argv[1]) if len(sys.argv) > 1 else 0
    count = int(sys.argv[2]) if len(sys.argv) > 2 else 50
    failures = 0
    for seed in range(first, first + count):
        try:
            msg = tile_case(seed) if (os.environ.get("HK_FUZZ_TILES") or os.environ.get("HK_FUZZ_HALO")) else one_case(seed)
        except Exception as e:   # API errors are findings too
            msg = f"seed {seed}: exception {e!r}"
        if msg:
            failures += 1
            print(msg, flush=True)
    print(f"{count} cases, {failures} failures")
    sys.exit(1 if failures else 0)
