#!/usr/bin/env python
"""Cost of the SVGF app's debug views (gfx_svgf_debug_visualize) at 1920x1080 on the bistro-class city, on cuda:0.  A few
SVGF-app frames first put the planes in the state a user of the display would see; then CUDA events time `--iters`
back-to-back launches of each view after warm-up.  Each view is one per-pixel pass: the bytes it needs per pixel (the planes
it reads, 16 B written) over the kernel time give its achieved bandwidth, which is set against the H100 SXM data sheet's
3.35 TB/s of HBM3.  Prints one JSON line with the card's name and power limit, read in the same call.

    python tools/svgf_views_bench.py [--iters 500] [--warmup 20] [--small]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from gfxexp_b200 import abi, engine, scenes

# the bytes each view reads per pixel (float4 planes, the float2 prevScreenPos); every view writes one float4
READ_BYTES = {"noisy_beauty": 32, "noisy_beauty_unmodulated": 16, "variance": 16, "filtered_variance": 16, "albedo": 16,
              "normal": 16, "motion_vector": 8, "sample_count": 16}
WRITE_BYTES = 16
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet, HBM3


def _power_limit_w():
    try:  # a read-only query
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--small", action="store_true", help="small city at 640x360 (a quick check, not the reported figure)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    scene = scenes.small_city_scene() if args.small else scenes.bistro_class_scene()
    w, h = (640, 360) if args.small else (1920, 1080)
    ctx = engine.Context(0)
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(w, h)
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = 5
    for frame in range(4):
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame):
            engine.run_svgf_app_pass(ctx, p, kind, pass_id, stage)
    ctx.synchronize()
    names = ["noisy_beauty", "variance", "filtered_variance", "albedo", "normal", "motion_vector", "sample_count"]
    ms = {}
    assert p.svgfFlags & abi.SVGF_MODULATE_ALBEDO  # the app's default (svgf_main.cpp:1735): Noisy Beauty reads the albedo too
    for view, name in enumerate(names):
        ms[name] = _time(lambda: ctx.svgf_debug_visualize(p, view), args.iters, args.warmup)
    p.svgfFlags &= ~abi.SVGF_MODULATE_ALBEDO
    ms["noisy_beauty_unmodulated"] = _time(lambda: ctx.svgf_debug_visualize(p, abi.SVGF_VIEW_NOISY_BEAUTY), args.iters, args.warmup)
    pixels = w * h
    views = {}
    for name, t in ms.items():
        nbytes = pixels * (READ_BYTES[name] + WRITE_BYTES)
        views[name] = {"ms": round(t, 4), "bytes": nbytes, "GB_per_s": round(nbytes / (t * 1e-3) / 1e9, 1),
                       "share_of_hbm_peak": round(nbytes / (t * 1e-3) / HBM_BYTES_PER_S, 3)}
    print(json.dumps({"bench": "svgf_views", "scene": scene.name, "width": w, "height": h, "iters": args.iters,
                      "warmup": args.warmup, "views": views, "gpu": torch.cuda.get_device_name(0),
                      "power_limit_w": _power_limit_w()}))
    ctx.close()


if __name__ == "__main__":
    main()
