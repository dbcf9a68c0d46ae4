#!/usr/bin/env python
"""NRC network micro-benchmark (config 3 sizes): inference batch = pad128(1920*1080 + tiles) ~ 2.2 M queries,
training 4 x 16 384 samples (neural_radiance_caching_main.cpp:2304-2316,2350-2365).  Prints one JSON line:
ms per inference launch, achieved TFLOP/s on the padded MLP (18 432 FLOP/query) and compulsory-HBM GB/s.

--position-encoding tri: the triangle-wave network (gfx_nrc_create_with_encoding) is timed as well, on the same queries and
training batch, and reported next to the hash-grid network's figures under "tri_*", with the GPU's name and power limit.
--queries N: the inference batch (default pad128(1920 * 1080 * 17 / 16)); 2116608 is the batch the stored tiny-cuda-nn timings
of tests/golden/make_golden_tcnn*.py use."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from gfxexp_b200 import abi, engine


def _time(net, q, out, n, tq, tt, nt):
    """ms per inference launch of n queries, ms per training step of nt samples"""
    for _ in range(3):
        net.infer(q, out, n)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    reps = 20
    ev[0].record()
    for _ in range(reps):
        net.infer(q, out, n)
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1]) / reps
    for _ in range(3):
        net.train(tq, tt, nt)
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(reps):
        net.train(tq, tt, nt)
    ev[1].record()
    torch.cuda.synchronize()
    tms = ev[0].elapsed_time(ev[1]) / reps
    return ms, tms


def _power_limit_w():
    try:  # a read-only query
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--position-encoding", choices=("hash", "tri"), default="hash")
    ap.add_argument("--queries", type=int, default=((1920 * 1080 + 1920 * 1080 // 16 + 127) // 128) * 128)
    args = ap.parse_args()
    ctx = engine.Context(0)
    net = engine.NeuralRadianceCache(ctx, 2, 1e-2)
    net.set_params(engine.random_nrc_params(net.num_params, 64 * 64 * 2 + 16 * 64, grid_amplitude=0.1))
    n = (args.queries + 127) // 128 * 128
    q = torch.rand((n, 14), device="cuda")
    out = torch.empty((n, 3), device="cuda")
    nt = 16384
    tq, tt = torch.rand((nt, 14), device="cuda"), torch.rand((nt, 3), device="cuda")
    ms, tms = _time(net, q, out, n, tq, tt, nt)
    peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json"))) \
        if os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")) else {"bf16_tflops": 1590.0, "hbm_gbs": 6650.0}
    flops = 18432.0 * n
    result = {
        "nrc_infer_queries": n, "nrc_infer_ms": ms, "nrc_infer_tflops": flops / (ms * 1e-3) / 1e12,
        "tensor_frac_of_measured_bf16_peak": flops / (ms * 1e-3) / 1e12 / peaks["bf16_tflops"],
        "nrc_infer_hbm_GBps": 68.0 * n / (ms * 1e-3) / 1e9, "hbm_frac": 68.0 * n / (ms * 1e-3) / 1e9 / peaks["hbm_gbs"],
        "nrc_infer_Mqueries_per_s": n / (ms * 1e-3) / 1e6,
        "nrc_train_step_ms_16384": tms, "nrc_train_tflops": 55296.0 * nt / (tms * 1e-3) / 1e12}
    if args.position_encoding == "tri":
        net.close()
        tri = engine.NeuralRadianceCache(ctx, 2, 1e-2, position_encoding=abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE)
        tri.set_params(engine.random_nrc_params(tri.num_params, tri.num_params))
        tri_ms, tri_tms = _time(tri, q, out, n, tq, tt, nt)
        result.update({"tri_nrc_infer_ms": tri_ms, "tri_nrc_infer_Mqueries_per_s": n / (tri_ms * 1e-3) / 1e6,
                       "tri_nrc_train_step_ms_16384": tri_tms, "gpu": torch.cuda.get_device_name(0),
                       "power_limit_w": _power_limit_w()})
        tri.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
