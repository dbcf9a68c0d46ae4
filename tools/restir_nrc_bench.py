#!/usr/bin/env python
"""The ReSTIR DI + NRC frame at 1920x1080 on the config-2 scene (bistro_class), old against combined, in one process on cuda:0:

  old       StripDriver.render_restir_nrc_frame(combined=False): ReSTIR DI, then GFX_PT_NRC blended over it
  combined  ... (combined=True): ReSTIR DI, then GFX_PT_NRC_INDIRECT added to it (one estimator)

The two are timed in alternating blocks of frames on the same driver (CUDA events around each block, training overlapped as in
bench.py's north_star_frame), then a few frames of each run with the library's kernel timers on (nrc_first_hit, nrc_trace_shadow,
...) and with gfx_stats_read's ray counter.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from gfxexp_b200 import abi, engine, multigpu, scenes

W, H = 1920, 1080


def _power_limit_w():
    try:  # a read-only query
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=6, help="timed blocks per frame kind, alternating")
    ap.add_argument("--frames", type=int, default=10, help="frames per block")
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("restir_nrc_bench needs a GPU")
    scene = scenes.bistro_class_scene()
    ctx = engine.Context(0)
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(W, H)
    p = abi.default_frame_params(scene, W, H)
    net = engine.NeuralRadianceCache(ctx, 2, 1e-2)
    driver = multigpu.StripDriver(ctx, p, W, H, 0, 1)
    driver.enable_nrc(net)
    rng = np.random.default_rng(0)
    frame = [0]

    def run(combined, n):
        for _ in range(n):
            p.numAccumFrames = frame[0]
            driver.render_restir_nrc_frame(frame[0], [int(rng.integers(0, 2 ** 32)) for _ in range(2)], combined=combined)
            frame[0] += 1

    kinds = {"old": False, "combined": True}
    for combined in kinds.values():
        run(combined, args.warmup)
    driver.wait_training()
    torch.cuda.synchronize()
    ms = {k: [] for k in kinds}
    for b in range(args.blocks):
        for k, combined in (kinds.items() if b % 2 == 0 else reversed(list(kinds.items()))):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(combined, args.frames)
            driver.wait_training()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / args.frames)

    # kernel times and rays, in stream order
    driver.train_stream = None
    result = {"what": "ReSTIR DI + NRC frame, 1920x1080, bistro_class scene, 1 GPU: old (GFX_PT_NRC blended over ReSTIR DI) "
                      "against combined (GFX_PT_NRC_INDIRECT added to ReSTIR DI)",
              "device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(),
              "blocks": args.blocks, "frames_per_block": args.frames}
    reps = 4
    for k, combined in kinds.items():
        ctx.timing_enable(True)
        ctx.timing_read()
        ctx.read_stats(reset=True)
        run(combined, reps)
        torch.cuda.synchronize()
        rays = ctx.read_stats(reset=True)[0] / reps
        timing = ctx.timing_read()
        ctx.timing_enable(False)
        nrc = {lbl: t / reps for lbl, (t, _) in sorted(timing.items()) if lbl.startswith("nrc_")}
        result[k] = {"ms_per_frame_median": float(np.median(ms[k])), "ms_per_frame_blocks": [round(v, 4) for v in ms[k]],
                     "rays_per_frame": rays, "nrc_kernel_ms_per_frame": {lbl: round(v, 4) for lbl, v in nrc.items()}}
    result["combined_minus_old_ms"] = result["combined"]["ms_per_frame_median"] - result["old"]["ms_per_frame_median"]
    result["rays_saved_per_frame"] = result["old"]["rays_per_frame"] - result["combined"]["rays_per_frame"]
    net.close()
    ctx.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
