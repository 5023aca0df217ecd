#!/usr/bin/env python
"""Time hk_scene_add_meshes against the host mirror's GpuMesh::try_from, and write profiles/h100_mesh_build.json (or --out).

For each mesh set — town's largest mesh (scene.rs), the city's houses, a seeded soup of 2^20 triangles — it records
  * device_ms      CUDA events on the scene's stream around the work the call enqueues: copies, packing and BLAS build.  The stream
                   is held by a spin kernel (torch.cuda._sleep) until after the call has returned, so the host's part of the call
                   (validation, host copies, staging) is not in it; median
  * span_ms        the same events without the spin kernel: from before the call to its last kernel, host part included, median
  * host_try_from_ms  the host mirror building the same meshes (MeshMaterialWorld::prepare_mesh_assets = GpuMesh::try_from), median
  * call_ms        the host time of the call itself while four 4K frames are queued on the same stream (the call does not wait
                   for them), median over calls whose pinned staging slot is already large enough
  * first_call_ms  the same for the scene's first call, which allocates its pinned staging slot
with the card's name and power limit read in the same run.  Needs a GPU: nothing here falls back to the CPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


GATE_S = 0.5       # seconds the spin kernel holds the stream: longer than the host part of any call measured here


def soup(tris, seed, spread=100.0):
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-spread, spread, (tris, 3)).astype(np.float32)
    pos = (centres[:, None, :] + rng.normal(0, 0.05, (tris, 3, 3))).astype(np.float32).reshape(-1, 3)
    return (pos, rng.normal(size=pos.shape).astype(np.float32), rng.random((len(pos), 2)).astype(np.float32), None)


def mesh_sets():
    from bevy_hikari_b200 import scenes
    town = scenes._load_npz("town")[0]
    largest = max(town, key=lambda m: len(m[3]))
    houses = scenes._load_npz("house2")[0] + scenes._load_npz("house3")[0]
    return {"town_largest": [largest], "city_houses": houses, "soup_1M": [soup(1 << 20, 11)]}


def host_try_from_ms(meshes, reps):
    from bevy_hikari_b200 import plugin
    times = []
    for _ in range(reps):
        w = plugin.World()
        for m in meshes:
            w.add_mesh(m[0], m[1], m[2], m[3])
        t0 = time.perf_counter()
        w.prepare()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_mesh_build.json"))
    args = ap.parse_args()
    import torch
    from bevy_hikari_b200 import plugin
    from tests.test_gpu_mesh_build import base_world
    from tests.conftest import Bench
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh_build needs a GPU")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    stream = torch.cuda.Stream()
    result = {"gpu": smi, "reps": args.reps, "sets": {}}
    bench = Bench("cornell", 3840, 2160, config="cornell_1080p")
    for name, meshes in mesh_sets().items():
        tris = int(sum((len(m[3]) // 3) if m[3] is not None else len(m[0]) // 3 for m in meshes))
        dev_ms, span_ms, call_ms, held = [], [], [], []
        for r in range(args.reps + 1):             # the first round warms up
            for gate in (False, True):
                dev = plugin.HikariPlugin(64, 64, 0, 0, None, stream.cuda_stream)
                dev.upload_scene(base_world())
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                if gate:
                    with torch.cuda.stream(stream):
                        torch.cuda._sleep(int(GATE_S * 1.98e9))
                e0.record(stream)
                t0 = time.perf_counter()
                dev.add_mesh_sources(meshes)
                returned = time.perf_counter() - t0
                e1.record(stream)
                torch.cuda.synchronize()
                if r:
                    (dev_ms if gate else span_ms).append(e0.elapsed_time(e1))
                    if gate:
                        held.append(returned < GATE_S)
                dev.close()
        cam = plugin.HikariPlugin(bench.width, bench.height, 0, 0, None, stream.cuda_stream)
        cam.upload_scene(bench.world)
        for r in range(args.reps + 2):             # the first two calls allocate the scene's two pinned staging slots
            cam.render_frame(bench.inputs(2 * r + 1))
            torch.cuda.synchronize()
            for f in range(4):
                cam.render_frame(bench.inputs(2 * r + 2))      # four 4K frames queued
            t0 = time.perf_counter()
            cam.add_mesh_sources(meshes)
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            if r >= 2:
                call_ms.append((t1 - t0) * 1e3)
            elif r == 0:
                first_call_ms = (t1 - t0) * 1e3
        cam.close()
        host = host_try_from_ms(meshes, max(1, min(args.reps, 3)))
        result["sets"][name] = {"meshes": len(meshes), "triangles": tris, "device_ms": float(np.median(dev_ms)),
                                "device_ms_call_returned_before_the_stream_ran": all(held), "span_ms": float(np.median(span_ms)),
                                "host_try_from_ms": host, "call_ms_with_4_frames_queued": float(np.median(call_ms)),
                                "first_call_ms_with_4_frames_queued": first_call_ms}
        print(name, result["sets"][name], flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(result, open(args.out, "w"), indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
