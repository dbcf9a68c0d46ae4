#!/usr/bin/env python
"""The SVGF app's frame (svgf_main.cpp:1980-2172) at 1920x1080 on the bistro-class city: light distributions, G-buffer, the
app's path tracer (GFX_PT_SVGF, maxPathLength 5, specular mollification on), temporal accumulation, variance, 5 a-trous
stages, background, albedo modulation + TAA.  After warm-up, CUDA events time whole frames; gfx_timing_enable /
gfx_timing_read give the per-kernel times of one more pass over as many frames, and the device ray counter, read around
every path tracer launch of that pass, its rays.  Prints one JSON line with the card's name and power limit, read in the same call.
--taa-jitter turns on the app's TAA sub-pixel jitter (GFX_SVGF_SUBPIXEL_JITTER), which moves the G-buffer's primary rays and
the background's environment lookups off the pixel centres.

    python tools/svgf_app_bench.py [--frames N] [--warmup W] [--small] [--taa-jitter]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from gfxexp_b200 import abi, engine, scenes


def _power_limit_w():
    try:  # a read-only query
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--small", action="store_true", help="small city at 640x360 (a quick check, not the reported figure)")
    ap.add_argument("--taa-jitter", action="store_true", help="the app's TAA sub-pixel jitter (GFX_SVGF_SUBPIXEL_JITTER)")
    args = ap.parse_args()
    scene = scenes.small_city_scene() if args.small else scenes.bistro_class_scene()
    w, h = (640, 360) if args.small else (1920, 1080)
    ctx = engine.Context(0)
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(w, h)
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = 5
    frame = 0

    pt_rays = [0]

    def run(n, count_rays=False):
        nonlocal frame
        for _ in range(n):
            for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame, mollify=True, taa_jitter=args.taa_jitter):
                if count_rays and kind == "pathtrace":
                    ctx.read_stats(reset=True)  # the G-buffer's primary rays go to the same counter
                engine.run_svgf_app_pass(ctx, p, kind, pass_id, stage)
                if count_rays and kind == "pathtrace":
                    pt_rays[0] += ctx.read_stats(reset=True)[0]
            frame += 1

    run(args.warmup)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    run(args.frames)
    ev[1].record()
    torch.cuda.synchronize()
    frame_ms = ev[0].elapsed_time(ev[1]) / args.frames
    # per-kernel times and the path tracer's rays: a second pass with an event pair around every launch and a counter read
    # around the path tracer (slower frames, not the frame figure)
    ctx.timing_enable(True)
    ctx.timing_read()
    run(args.frames, count_rays=True)
    torch.cuda.synchronize()
    rays = pt_rays[0] / args.frames
    kernels = {k: round(ms / args.frames, 4) for k, (ms, _) in sorted(ctx.timing_read().items())}
    ctx.timing_enable(False)
    pt_ms = sum(v for k, v in kernels.items() if k.startswith("pt_"))
    print(json.dumps({"bench": "svgf_app_frame", "scene": scene.name, "width": w, "height": h, "max_path_length": 5,
                      "mollify_specular": True, "taa_jitter": args.taa_jitter, "frames": args.frames, "warmup": args.warmup, "frame_ms": round(frame_ms, 4),
                      "pathtrace_ms": round(pt_ms, 4), "pathtrace_rays_per_frame": rays,
                      "pathtrace_Mrays_per_s": round(rays / (pt_ms * 1e-3) / 1e6, 1) if pt_ms > 0 else None,
                      "kernel_ms": kernels, "gpu": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w()}))
    ctx.close()


if __name__ == "__main__":
    main()
