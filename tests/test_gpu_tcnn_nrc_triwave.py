"""The triangle-wave NRC network against the reference's own code: tiny-cuda-nn's NetworkWithInputEncoding + Trainer built from
network_interface.cu's PositionEncoding::TriangleWave config, whose results are stored in tests/golden/tcnn_nrc_triwave.npz.
tests/tcnn_nrc_triwave_check.py does the work in a child process and prints one JSON line; the bars:

  * the initial fp32 master weights bit for bit (and equal to the hash-grid network's matrices), the training halves identical,
    the EMA weights zero;
  * tiny-cuda-nn's Composite encoding (triangle wave, one-blob, identity, ones) equal, half for half, to the oracle's and to
    gfx_nrc_encode_debug's;
  * inferred radiance within 1e-3 relative L2 of tiny-cuda-nn's, the half-accumulating oracle within 1e-4 of it, ours within 1e-4
    of the fp32 oracle; after four training steps within 1e-3;
  * one step's matrix gradients within 2.5e-3, and within 1e-4 of the fp32 oracle;
  * the losses of four steps within 1e-4 relative."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_triangle_wave_network_matches_tiny_cuda_nn():
    proc = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "tcnn_nrc_triwave_check.py")], capture_output=True,
                          text=True, timeout=400)
    line = proc.stdout.strip().splitlines()[-1] if proc.stdout.strip() else ""
    assert proc.returncode == 0, f"rc={proc.returncode} {line[:400]} {proc.stderr[-600:]}"
    r = json.loads(line)
    init = r["init"]
    assert init["master_mismatches"] == 0 and init["hash_grid_matrix_mismatches"] == 0, init
    assert init["training_half_mismatches"] == 0 and init["inference_all_zero"], init
    enc = r["encoding"]
    assert enc["width"] == 64 and enc["oracle_mismatches"] == 0 and enc["ours_mismatches"] == 0, enc
    fwd = r["forward"]
    assert fwd["ours_vs_tcnn"] <= 1e-3, fwd
    assert fwd["oracle_halfacc_vs_tcnn"] <= 1e-4, fwd
    assert fwd["ours_vs_oracle_fp32acc"] <= 1e-4, fwd
    g = r["gradients"]
    for name in ("W0", "W1", "W2"):
        assert g[name]["ours_vs_tcnn"] <= 2.5e-3, (name, g[name])
        assert g[name]["ours_vs_oracle_fp32acc"] <= 1e-4, (name, g[name])
    losses = r["weights"]["losses"]
    for a, b in zip(losses["ours"], losses["tcnn"]):
        assert abs(a - b) <= 1e-4 * abs(b), losses
    assert r["weights"]["inference_after_training_ours_vs_tcnn"] <= 1e-3, r["weights"]
