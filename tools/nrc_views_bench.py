"""Cost of the NRC debug views at 1920x1080 on cuda:0: the visualizePrediction pass (GFX_PT_NRC_VISUALIZE_PREDICTION), the
inference of its W*H queries (gfx_nrc_frame_infer), and gfx_present_launch of the prediction, path-length, flow and ReGIR-cell
views beside the plain tone-mapped COLOR present.  CUDA events around `--iters` back-to-back calls of each, after a few NRC
frames so that the network and the buffers are in the state a user of the display would see.  Prints one JSON line with the
card's name and power limit, read in the same call.

    python tools/nrc_views_bench.py [--iters 200] [--width 1920 --height 1080]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gfxexp_b200 import abi, engine, scenes  # noqa: E402


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return out or "unknown"


def _time(fn, iters):
    for _ in range(3):
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
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    w, h = args.width, args.height
    scene = scenes.small_city_scene()
    ctx = engine.Context(0)
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(w, h)
    net = engine.NeuralRadianceCache(ctx, 2, 1e-2)
    p = abi.default_frame_params(scene, w, h)
    rng = np.random.default_rng(1)
    for f in range(4):
        p.numAccumFrames = f
        ctx.build_light_distributions(f % 2)
        ctx.nrc_frame(net, p, f, [int(rng.integers(0, 2 ** 32)) for _ in range(2)], train=True)
    ctx.synchronize()
    pp = {}
    for name, mode, flags in [("present_color", abi.PRESENT_COLOR, 0), ("present_prediction", abi.PRESENT_NRC_PREDICTION, 0),
                              ("present_path_length", abi.PRESENT_NRC_PATH_LENGTH, abi.PRESENT_NRC_TRAINING_PATHS),
                              ("present_flow", abi.PRESENT_FLOW, 0), ("present_cells", abi.PRESENT_COLOR, abi.PRESENT_REGIR_CELLS)]:
        pp[name] = abi.GfxPresentParams(abi.BUF_BEAUTY_ACCUM, 0, mode, flags | abi.PRESENT_TONE_MAP | abi.PRESENT_SRGB_GAMMA, 1.0, 1.0,
                                        C.pointer(p), 0.1, 0.5)

    def present(name):
        return lambda: ctx._check(ctx.lib.gfx_present_launch(ctx.h, None, C.byref(pp[name])), "gfx_present_launch")

    ms = {"visualize_pass": _time(lambda: ctx.pathtrace(p, abi.PT_NRC_VISUALIZE_PREDICTION), args.iters),
          "frame_infer_wxh": _time(lambda: ctx.nrc_frame_infer(net), args.iters)}
    for name in pp:
        ms[name] = _time(present(name), args.iters)
    ms["prediction_view_total"] = ms["visualize_pass"] + ms["frame_infer_wxh"] + ms["present_prediction"]
    print(json.dumps({"width": w, "height": h, "queries": (w * h + 127) // 128 * 128, "card": _card(),
                      "ms": {k: round(v, 4) for k, v in ms.items()}}))
    net.close()
    ctx.close()


if __name__ == "__main__":
    main()
