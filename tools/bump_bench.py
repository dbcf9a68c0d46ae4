#!/usr/bin/env python
"""Cost of the bump mapping (GfxFrameParams::enableBumpMapping) on one GPU, switch off against switch on:
  * the config-2 ReSTIR DI frame (bistro-class city, 1920x1080; no bump table, so every material reads the reference's default
    texel, as in the apps): G-buffer kernel ms and whole-frame ms;
  * the baseline path tracer (maxPathLength 5) on small_city_scene_bumped at 1920x1080: G-buffer and path-tracer kernel ms, rays/s.
Per-kernel times come from the library's CUDA-event timing (gfx_timing_enable); frame times from CUDA events without it.  The
card's name and power limit are read in the same run.  Prints one JSON line."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from gfxexp_b200 import abi, engine, scenes

W, H = 1920, 1080


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0) + ", power limit not read"
    return q


def _timed(ctx, run, reps):
    """(ms per call of run() from CUDA events, {kernel: ms per call} from the library's timing in a separate pass)"""
    run(0)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for i in range(reps):
        run(1 + i)
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / reps
    ctx.timing_enable(True)
    ctx.timing_read()
    for i in range(reps):
        run(1 + reps + i)
    kernels = {k: v[0] / reps for k, v in ctx.timing_read().items()}
    ctx.timing_enable(False)
    return ms, kernels


def restir(ctx, scene, bump, reps):
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(W, H)
    p = abi.default_frame_params(scene, W, H)
    p.enableBumpMapping = bump

    def run(f):
        p.numAccumFrames = f
        ctx.build_light_distributions(f % 2)
        for kind, pid in engine.restir_frame_passes(p, f, 1, True, False):
            ctx.gbuffer(p) if kind == "gbuffer" else ctx.restir(p, pid)
    ms, k = _timed(ctx, run, reps)
    return {"frame_ms": ms, "gbuffer_ms": k.get("gbuffer")}


def pathtrace(ctx, scene, bump, reps):
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(W, H)
    ctx.build_light_distributions(0)
    p = abi.default_frame_params(scene, W, H)
    p.enableBumpMapping = bump

    def run(f):
        p.numAccumFrames = f
        ctx.gbuffer(p)
        ctx.pathtrace(p)
    run(0)
    torch.cuda.synchronize()
    ctx.read_stats(reset=True)
    ms, k = _timed(ctx, run, reps)
    rays = ctx.read_stats()[0] / (2 * reps + 1)
    pt = {name: v for name, v in k.items() if name != "gbuffer"}
    return {"frame_ms": ms, "gbuffer_ms": k.get("gbuffer"), "pathtrace_kernels_ms": sum(pt.values()), "kernels": pt,
            "rays_per_frame": rays, "mrays_per_s": rays / (ms * 1e3)}


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 20
    ctx = engine.Context(0)
    out = {"card": _card(), "size": [W, H], "reps": reps}
    config2 = scenes.bistro_class_scene()
    bumped = scenes.small_city_scene_bumped()
    for bump in (0, 1, 0, 1):  # alternating, twice
        key = "on" if bump else "off"
        out.setdefault("restir_config2_" + key, []).append(restir(ctx, config2, bump, reps))
        out.setdefault("pathtrace_bumped_" + key, []).append(pathtrace(ctx, bumped, bump, reps))
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
