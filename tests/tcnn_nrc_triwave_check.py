#!/usr/bin/env python
"""Pins the triangle-wave NRC network (gfx_nrc_create_with_encoding(GFX_NRC_POSITION_ENCODING_TRIANGLE_WAVE, 2, 1e-2)) against
the reference's own code: tiny-cuda-nn's NetworkWithInputEncoding + Trainer built from neural_radiance_caching/network_interface.cu's
posEnc == TriangleWave config (oracle/ref_tcnn/tcnn_nrc.cu, tcnn_nrc_encode.cu), whose results on the inputs below are stored in
tests/golden/tcnn_nrc_triwave.npz (tests/golden/make_golden_tcnn_triwave.py; the network has only 9 216 parameters, all kept).
Runs on a GPU in its own process and prints ONE JSON line:

  init        tcnn's pcg32{1337} initial parameters vs ours, and vs the hash-grid network's matrices
  encoding    tiny-cuda-nn's Composite encoding vs the oracle's and gfx_nrc_encode_debug's, half for half
  forward     relative L2 of the inferred radiance: ours / the oracle (fp32 and half accumulation) vs tcnn
  gradients   one training step from identical weights: loss and relative L2 per weight matrix
  weights     the losses of four training steps, the weights after them and the inference after them

Usage: python tests/tcnn_nrc_triwave_check.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np

import tcnn_nrc_check as NC

HIDDEN, LR = NC.HIDDEN, NC.LR
N_ENCODE, N_FORWARD, N_TRAIN = 4096, 4096, NC.N_TRAIN
GOLDEN = os.path.join(ROOT, "tests", "golden", "tcnn_nrc_triwave.npz")


def adversarial_positions(n, seed):
    """positions where the triangle wave's floor and fold go wrong if anything is off: 0 and 1, multiples of 2^-k that make
    val = x + f / 4 an exact integer or half-integer, negative values, values above 1, tiny and large magnitudes"""
    f = np.float32
    rng = np.random.default_rng(seed)
    p = rng.uniform(0.0, 1.0, size=(n, 3)).astype(f)
    special = [0.0, 1.0, -0.0, -1.0, 0.5, 0.25, 0.125, 2.0 ** -11, 2.0 ** -12, 1.0 - 2.0 ** -24, 1.0 + 2.0 ** -23, 2.0, 3.75,
               -0.5, -0.25, -2.0 ** -13, 1e-30, -1e-30, 1000.5, -1000.25, 65504.0, 1e7]
    k = len(special)
    p[:k] = np.array(special, dtype=f)[:, None]
    rows = k
    for e in range(1, 15):  # multiples of 2^-e: x = p 2^(f-1) hits integers / half-integers for many f
        m = rng.integers(-2 ** (e + 1), 2 ** (e + 1) + 1, size=(16, 3))
        p[rows:rows + 16] = (m / 2.0 ** e).astype(f)
        rows += 16
    p[rows:rows + 64] = rng.uniform(-3.0, 3.0, size=(64, 3)).astype(f)
    return p


def encode_queries():
    q = NC.queries(np.random.default_rng(41), N_ENCODE)
    q[:, :3] = adversarial_positions(N_ENCODE, 42)
    return np.ascontiguousarray(q)


def layer_slices(num_matrix_weights):
    out = {f"W{l}": slice(64 * 64 * l, 64 * 64 * (l + 1)) for l in range(HIDDEN)}
    out[f"W{HIDDEN}"] = slice(64 * 64 * HIDDEN, num_matrix_weights)
    return out


def main():
    import torch

    import oracle_nrc_triwave as OW
    from gfxexp_b200 import abi, engine
    tri = abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE
    rel_l2 = NC.rel_l2
    result = {}
    ref = np.load(GOLDEN)
    ctx = engine.Context(0)
    ours = engine.NeuralRadianceCache(ctx, HIDDEN, LR, position_encoding=tri)
    P = ours.num_params
    onet = OW.OracleNrcTriWave(HIDDEN, LR)
    M = onet.num_matrix_weights
    assert P == M == NC.num_matrix_weights()
    slices = layer_slices(M)

    # ---- init: Trainer{seed 1337}; the same pcg32 prefix as the hash-grid network's
    hash_net = engine.NeuralRadianceCache(ctx, HIDDEN, LR)
    hash_master = hash_net.read(abi.NRC_READ_MASTER)[:M]
    hash_net.close()
    our_master = ours.read(abi.NRC_READ_MASTER)
    result["init"] = {"params": int(P),
                      "master_mismatches": int((ref["init_master"].view(np.uint32) != our_master.view(np.uint32)).sum()),
                      "hash_grid_matrix_mismatches": int((hash_master.view(np.uint32) != our_master.view(np.uint32)).sum()),
                      "training_half_mismatches": int((ref["init_training"].view(np.uint16) !=
                                                       ours.read(abi.NRC_READ_TRAINING).view(np.uint16)).sum()),
                      "inference_all_zero": bool(ref["init_inference_all_zero"] and not ours.read(abi.NRC_READ_INFERENCE).any())}

    # ---- the Composite encoding, half for half
    qe = encode_queries()
    ref_enc = ref["encoding"]
    orc_enc = onet.encode(qe).view(np.uint16)
    our_enc = ours.encode(torch.from_numpy(qe).cuda(), N_ENCODE).view(np.uint16)
    result["encoding"] = {"n": N_ENCODE, "width": int(ref_enc.shape[1]), "oracle_mismatches": int((orc_enc != ref_enc).sum()),
                          "ours_mismatches": int((our_enc != ref_enc).sum())}

    # ---- forward and one training step from identical, half-representable weights
    rng = np.random.default_rng(29)
    params = engine.random_nrc_params(P, M, seed=31)
    master = params.astype(np.float32)
    ours.set_params(params)
    onet.set_params(params)
    q = NC.queries(rng, N_FORWARD)
    ref_out = ref["forward"]
    dq = torch.from_numpy(q).cuda()
    dout = torch.empty((N_FORWARD, 3), device="cuda")
    ours.infer(dq, dout, N_FORWARD)
    torch.cuda.synchronize()
    our_out = dout.cpu().numpy()
    o32 = onet.infer(q)
    onet.set_accumulate_half(True)
    o16 = onet.infer(q)
    onet.set_accumulate_half(False)
    result["forward"] = {"n": N_FORWARD, "ours_vs_tcnn": rel_l2(our_out, ref_out), "oracle_fp32acc_vs_tcnn": rel_l2(o32, ref_out),
                         "oracle_halfacc_vs_tcnn": rel_l2(o16, ref_out), "ours_vs_oracle_fp32acc": rel_l2(our_out, o32)}

    qt = NC.queries(rng, N_TRAIN)
    tt = NC.targets(qt)
    ref_grad = ref["gradients"].astype(np.float32)
    ours.keep_gradients(True)
    our_loss = ours.train(torch.from_numpy(qt).cuda(), torch.from_numpy(tt).cuda(), N_TRAIN, want_loss=True)
    our_grad = ours.read(abi.NRC_READ_GRADIENTS)
    o_loss32 = onet.train(qt, tt)
    o_grad32 = onet.get_gradients()
    onet.set_params(params)
    onet.set_accumulate_half(True)
    o_loss16 = onet.train(qt, tt)
    o_grad16 = onet.get_gradients()
    onet.set_accumulate_half(False)
    grads = {"loss": {"tcnn": float(ref["loss"]), "ours": our_loss, "oracle_fp32acc": o_loss32, "oracle_halfacc": o_loss16}}
    for name, sl in slices.items():
        grads[name] = {"ours_vs_tcnn": rel_l2(our_grad[sl], ref_grad[sl]), "oracle_fp32acc_vs_tcnn": rel_l2(o_grad32[sl], ref_grad[sl]),
                       "oracle_halfacc_vs_tcnn": rel_l2(o_grad16[sl], ref_grad[sl]),
                       "ours_vs_oracle_fp32acc": rel_l2(our_grad[sl], o_grad32[sl])}
    result["gradients"] = grads

    # ---- four full training steps (forward, loss, backward, Adam with epsilon 1e-8, EMA) from the same start
    ours.set_params(params)
    onet.set_params(params)
    losses = {"tcnn": [float(x) for x in ref["losses"]], "ours": [], "oracle_fp32acc": []}
    for _ in range(4):
        qs = NC.queries(rng, N_TRAIN)
        ts = NC.targets(qs)
        losses["ours"].append(ours.train(torch.from_numpy(qs).cuda(), torch.from_numpy(ts).cuda(), N_TRAIN, want_loss=True))
        losses["oracle_fp32acc"].append(onet.train(qs, ts))
    weights = {"losses": losses}
    ref_tr, ref_inf = ref["training"].astype(np.float32), ref["inference"].astype(np.float32)
    our_tr = ours.read(abi.NRC_READ_TRAINING).astype(np.float32)
    our_inf = ours.read(abi.NRC_READ_INFERENCE).astype(np.float32)
    orc_tr = onet.get_params(ema=False).astype(np.float32)
    for name, sl in slices.items():
        weights[name] = {"inference_ours_vs_tcnn": rel_l2(our_inf[sl], ref_inf[sl]),
                         "update_ours_vs_tcnn": rel_l2(our_tr[sl] - master[sl], ref_tr[sl] - master[sl]),
                         "update_oracle_vs_tcnn": rel_l2(orc_tr[sl] - master[sl], ref_tr[sl] - master[sl])}
    qa = NC.queries(rng, N_FORWARD)
    ours.infer(torch.from_numpy(qa).cuda(), dout, N_FORWARD)
    torch.cuda.synchronize()
    weights["inference_after_training_ours_vs_tcnn"] = rel_l2(dout.cpu().numpy(), ref["forward_after_training"])
    weights["inference_after_training_oracle_vs_tcnn"] = rel_l2(onet.infer(qa), ref["forward_after_training"])
    result["weights"] = weights
    ours.close()
    ctx.close()
    print(json.dumps(result))
    return 0


if __name__ == "__main__":
    sys.exit(main())
