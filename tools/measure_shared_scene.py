#!/usr/bin/env python
"""Several cameras, one scene: a private scene per camera (N uploads, N copies in device memory, N update_transforms per frame)
against one SharedScene (hk_shared_scene) that every camera attaches to.  Two workloads:

  scene_1080p_minimap   scene.rs (the "town" scene) at 1920 x 1080 + a 480 x 270 second camera, the emissive sphere animated
  city_split_screen     the city as two 1920 x 2160 cameras side by side (split screen), the city animation

Per workload and arm it records the device memory the SECOND camera adds (torch.cuda.mem_get_info around its creation + upload or
attach), the host time per frame of the scene update(s) (perf_counter around the update calls: with the device idle before the
call, and inside the timed run, where it also waits for frames in flight) and the wall time per frame of both
cameras (updates + two hk_render_frame, synchronised once per run of frames), with every camera and the scene on ONE stream and with
each on a stream of its own.  The arms alternate within one process, repeated --reps times; medians are reported.

    python tools/measure_shared_scene.py --out profiles/h100_shared_scene.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bevy_hikari_b200 import plugin  # noqa: E402
from tests.conftest import Animation, Bench, city_animation, rotation_y_about  # noqa: E402


def town_animation(bench):
    w = bench.world
    em = int(w.buffers()["emissives"]["instance"][0])     # the emissive earth sphere at (2, 2, 0) (scene.rs:85-107)
    return Animation(bench, {em: lambda f: rotation_y_about(0.1 * f, (2.0, 2.0, 0.0), (0.0, 0.05 * np.sin(0.5 * f), 0.0))})


WORKLOADS = {
    "scene_1080p_minimap": dict(scene="town", config="scene_1080p", cameras=[(1920, 1080), (480, 270)], animation=town_animation),
    "city_split_screen": dict(scene="city", config="city_4k", cameras=[(1920, 2160), (1920, 2160)], animation=city_animation),
}


def free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def run_arm(spec, shared, one_stream, frames, warmup):
    benches = [Bench(spec["scene"], w, h, config=spec["config"]) for w, h in spec["cameras"]]
    world = benches[0].world
    stream = torch.cuda.Stream() if one_stream else None
    sptr = stream.cuda_stream if stream is not None else None
    scene = None
    devs, second_camera_bytes = [], 0
    if shared:
        scene = plugin.SharedScene(0, sptr)
        scene.upload(world)
    for i, b in enumerate(benches):
        before = free_bytes()
        d = plugin.HikariPlugin(b.width, b.height, 0, 0, None, sptr)
        d.set_temporal_upscalers(False)
        if shared:
            d.attach_scene(scene)
        else:
            d.upload_scene(world)
        after = free_bytes()
        if i == 1:
            second_camera_bytes = before - after
        devs.append(d)
    an = spec["animation"](benches[0])
    update_s, idle_s = [], []
    for f in range(1, warmup + frames + 1):
        for k, track in an.tracks.items():
            world.set_instance_transform(k, an.compose(track(f), an.base[k]))
        world.previous_transform_system()
        if f == warmup + 1:
            torch.cuda.synchronize()
            t_run = time.perf_counter()
        t0 = time.perf_counter()
        if shared:
            assert scene.update_transforms(world)
        else:
            models, previous, aabbs = world.prepare_instance_transforms()
            for d in devs:
                d.update_transforms_arrays(models, aabbs, previous)
        t1 = time.perf_counter()
        for d, b in zip(devs, benches):
            d.render_frame(b.inputs(f))
        if f > warmup:
            update_s.append(t1 - t0)
    for d in devs:
        d.sync()
    torch.cuda.synchronize()
    frame_s = (time.perf_counter() - t_run) / frames
    # the update(s) alone with the device idle before each call: the host's own work, without the back-pressure of the frames in
    # flight that the frame time above contains (the pinned staging slot of two calls before)
    for f in range(warmup + frames + 1, warmup + frames + 9):
        for k, track in an.tracks.items():
            world.set_instance_transform(k, an.compose(track(f), an.base[k]))
        world.previous_transform_system()
        for d in devs:
            d.sync()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if shared:
            assert scene.update_transforms(world)
        else:
            models, previous, aabbs = world.prepare_instance_transforms()
            for d in devs:
                d.update_transforms_arrays(models, aabbs, previous)
        idle_s.append(time.perf_counter() - t0)
        for d, b in zip(devs, benches):
            d.render_frame(b.inputs(f))
    wide = [int(d.stats().wide_traversal) for d in devs]
    for d in devs:
        d.close()
    if scene is not None:
        scene.close()
    return {"second_camera_mib": second_camera_bytes / 2**20, "update_host_ms_in_flight": 1e3 * statistics.median(update_s),
            "update_host_ms_idle": 1e3 * statistics.median(idle_s), "ms_per_frame_both_cameras": 1e3 * frame_s, "wide_traversal": wide}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except Exception as e:   # pragma: no cover
        power = f"unavailable ({e})"
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": power, "frames": args.frames, "warmup": args.warmup,
              "reps": args.reps, "workloads": {}}
    for name, spec in WORKLOADS.items():
        samples = {}
        for rep in range(args.reps):
            for streams in ("one_stream", "two_streams"):
                for arm in (("private", "shared") if rep % 2 == 0 else ("shared", "private")):      # alternate the arms
                    r = run_arm(spec, arm == "shared", streams == "one_stream", args.frames, args.warmup)
                    samples.setdefault((arm, streams), []).append(r)
                    print(name, rep, arm, streams, json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()}), flush=True)
        out = {}
        for (arm, streams), rs in samples.items():
            out.setdefault(arm, {})[streams] = {
                "ms_per_frame_both_cameras": round(statistics.median(r["ms_per_frame_both_cameras"] for r in rs), 3),
                "ms_per_frame_spread": [round(min(r["ms_per_frame_both_cameras"] for r in rs), 3),
                                        round(max(r["ms_per_frame_both_cameras"] for r in rs), 3)],
                "update_host_ms_idle": round(statistics.median(r["update_host_ms_idle"] for r in rs), 3),
                "update_host_ms_in_flight": round(statistics.median(r["update_host_ms_in_flight"] for r in rs), 3),
                "wide_traversal_per_camera": rs[0]["wide_traversal"],
                "second_camera_mib": round(statistics.median(r["second_camera_mib"] for r in rs), 1)}
        result["workloads"][name] = {"cameras": spec["cameras"], "scene": spec["scene"], "config": spec["config"], **out}
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text + "\n")


if __name__ == "__main__":
    main()
