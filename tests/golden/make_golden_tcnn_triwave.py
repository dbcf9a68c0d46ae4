#!/usr/bin/env python
"""Records what the reference's own tiny-cuda-nn computes with the triangle-wave NRC network (NeuralRadianceCache::initialize
with PositionEncoding::TriangleWave, depth 2, learning rate 1e-2) for the inputs of tests/tcnn_nrc_triwave_check.py, so that the
check compares against stored vectors and runs anywhere.  Needs a GPU, oracle/_ref/libtcnn_nrc.so (oracle/ref_tcnn/Makefile) and
oracle/_ref/libtcnn_nrc_encode.so (oracle/ref_tcnn/Makefile.encode).

Writes tests/golden/tcnn_nrc_triwave.npz (or into the directory given as the first argument); tcnn_nrc.npz and tcnn_ref.npz are
left alone.  The network has 9 216 parameters, all of them stored.  Prints tiny-cuda-nn's triangle-wave timings on the same GPU
as one JSON line.
Usage: python tests/golden/make_golden_tcnn_triwave.py [OUT_DIR]"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

import make_golden_tcnn as MG
import tcnn_nrc_check as NC
import tcnn_nrc_triwave_check as TW
from gfxexp_b200 import engine

TRIANGLE_WAVE = 0  # PositionEncoding::TriangleWave


class TcnnNrcTriWave(MG.TcnnNrc):
    """tiny-cuda-nn's network and trainer from the triangle-wave config (tcnn_nrc_create's posEnc 0)"""

    def __init__(self):
        super().__init__()  # binds the library (and creates a hash-grid network, released here)
        self.lib.tcnn_nrc_destroy(self.h)
        self.h = C.c_void_p()
        self._ok(self.lib.tcnn_nrc_create(TRIANGLE_WAVE, NC.HIDDEN, NC.LR, C.byref(self.h)))
        self.num_params = self.lib.tcnn_nrc_num_params(self.h)


def tcnn_encode(q):
    """the triangle-wave network's own Composite encoding (tcnn_nrc_encode.cu): [n][64] half bits"""
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libtcnn_nrc_encode.so"))
    lib.tcnn_nrc_encode.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
    q = np.ascontiguousarray(q, dtype=np.float32)
    out = np.empty((q.shape[0], 64), dtype=np.uint16)
    width = C.c_uint32()
    assert lib.tcnn_nrc_encode(TRIANGLE_WAVE, NC.HIDDEN, q.ctypes.data, q.shape[0], out.ctypes.data, C.byref(width)) == 0
    assert width.value == 64, width.value
    return out


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.dirname(os.path.abspath(__file__))
    os.makedirs(out_dir, exist_ok=True)
    ref = TcnnNrcTriWave()
    P = ref.num_params
    M = NC.num_matrix_weights()
    assert P == M, (P, M)
    g = {"init_master": ref.read(0), "init_training": ref.read(1), "init_inference_all_zero": np.array(not ref.read(2).any())}
    g["encoding"] = tcnn_encode(TW.encode_queries())
    # the same draws, in the same order, as tcnn_nrc_triwave_check.main()
    rng = np.random.default_rng(29)
    master = engine.random_nrc_params(P, M, seed=31).astype(np.float32)
    ref.set_params(master)
    g["forward"] = ref.infer(NC.queries(rng, TW.N_FORWARD))
    qt = NC.queries(rng, TW.N_TRAIN)
    loss, grad = ref.forward_backward(qt, NC.targets(qt))
    g["loss"], g["gradients"] = np.array(loss, dtype=np.float32), grad
    ref2 = TcnnNrcTriWave()
    ref2.set_params(master)
    losses = []
    for _ in range(4):
        qs = NC.queries(rng, TW.N_TRAIN)
        losses.append(ref2.train(qs, NC.targets(qs)))
    g["losses"] = np.array(losses, dtype=np.float32)
    g["training"], g["inference"] = ref2.read(1), ref2.read(2)
    g["forward_after_training"] = ref2.infer(NC.queries(rng, TW.N_FORWARD))
    np.savez_compressed(os.path.join(out_dir, "tcnn_nrc_triwave.npz"), **g)

    # tiny-cuda-nn's triangle-wave network at a 1080p frame's query count (pad128(1920 * 1080 + 1920 * 1080 / 48)) and a
    # training batch
    n_big = 2_116_608
    t_inf = ref2.time_infer(NC.queries(rng, n_big), 3, 20)
    qt2 = NC.queries(rng, TW.N_TRAIN)
    t_tr = ref2.time_train(qt2, NC.targets(qt2), 3, 40)
    print(json.dumps({"position_encoding": "triangle_wave", "tcnn_infer_ms": t_inf, "infer_queries": n_big,
                      "tcnn_train_step_ms": t_tr, "train_samples": TW.N_TRAIN, "gpu": torch.cuda.get_device_name(0)}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
