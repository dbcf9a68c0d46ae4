"""The triangle-wave NRC network's oracle (oracle/nrc_triwave.cpp, tests/oracle_nrc_triwave.py), pinned without a GPU: its
encoding against a float32 transcription of tiny-cuda-nn's triangle_wave_encoding (encodings/triangle_wave.h:47-81) bit for bit,
the AoS one-blob against a transcription of kernel_one_blob, the whole encoding against tiny-cuda-nn's stored output, the
parameter count, the matrix gradients against finite differences, loss descent, and the NRC strip frames with a triangle-wave
net at world_size 2 over gloo."""
import os
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

from gfxexp_b200 import abi, engine
from tests import oracle_nrc_triwave as OW
from tests.tcnn_nrc_triwave_check import adversarial_positions

TRI, HASH = abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE, abi.NRC_POSITION_ENCODING_HASH_GRID


def _queries(n, seed=0):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.02, 0.98, size=(n, 14)).astype(np.float32)


def triangle_wave_numpy(p):
    """triangle_wave_encoding in float32, one IEEE rounding per operation: [n][3] -> [n][36] float16, column 12 d + f"""
    f32 = np.float32
    out = np.empty((p.shape[0], 36), dtype=np.float16)
    for d in range(3):
        for fr in range(12):
            x = np.ldexp(p[:, d], fr - 1).astype(f32)
            val = (x + f32(fr * 0.25)).astype(f32)
            r = ((np.abs(((val - np.floor(val)).astype(f32) - f32(0.5)).astype(f32)) * f32(4)).astype(f32) - f32(1)).astype(f32)
            out[:, 12 * d + fr] = r.astype(np.float16)
    return out


def test_triangle_wave_columns_match_tiny_cuda_nn_bit_for_bit(oracle):
    n = 4096
    q = _queries(n, 1)
    q[:, :3] = adversarial_positions(n, 2)
    net = OW.OracleNrcTriWave(2, 1e-2)
    got = net.encode(q).view(np.uint16)
    want = triangle_wave_numpy(q[:, :3]).view(np.uint16)
    bad = np.argwhere(got[:, :36] != want)
    assert bad.size == 0, f"{len(bad)} halves differ, first {bad[:5].tolist()}"
    # the folds are exercised: exact -1 and +1 and values in between all occur
    e = got[:, :36].view(np.float16).astype(np.float32)
    assert (e == -1.0).any() and (e == 1.0).any() and ((e > -1) & (e < 1)).mean() > 0.5


def _quartic_cdf_contracted(x):
    """quartic_cdf with the three FMAs nvcc contracts it into in the reference's build (float32 operands; the products are exact
    in float64, so a*b+c rounded once from float64 stands for the FMA)"""
    f, d = np.float32, np.float64
    u = (x * f(4.0)).astype(f)
    u2 = (u * u).astype(f)
    u4 = (u2 * u2).astype(f)
    a = (d(-(f(2.0) / f(3.0))) * u2.astype(d) + 1.0).astype(f)
    inner = (d(f(1.0) / f(5.0)) * u4.astype(d) + a.astype(d)).astype(f)
    v = ((f(f(15.0) / f(16.0)) * u).astype(f).astype(d) * inner.astype(d) + 0.5).astype(f)
    return np.maximum(f(0.0), np.minimum(f(1.0), v)).astype(f)


def one_blob_aos_numpy(x5):
    """kernel_one_blob / one_blob_subwarp_aligned (oneblob.h:47-108), the AoS one-blob the triangle-wave Composite runs:
    [n][5] -> [n][20] float16"""
    f = np.float32
    out = np.empty((x5.shape[0], 20), dtype=np.float16)
    for d in range(5):
        x = x5[:, d]
        left = []
        for k in range(4):
            t = (f(0.25 * k) - x).astype(f)
            left.append(((_quartic_cdf_contracted(t) + _quartic_cdf_contracted((t - f(1.0)).astype(f))).astype(f) +
                         _quartic_cdf_contracted((t + f(1.0)).astype(f))).astype(f))
        for k in range(4):
            right = left[k + 1] if k < 3 else (left[0] + f(1.0)).astype(f)
            out[:, 4 * d + k] = (right - left[k]).astype(f).astype(np.float16)
    return out


def test_tail_is_the_aos_one_blob_identity_and_ones(oracle):
    """TriangleWave prefers AoS, so the reference's triangle-wave Composite runs OneBlob's AoS kernel, whose last bin is closed
    by "first boundary + 1" - not the hash-grid network's SoA one-blob.  Identity and ones are the hash-grid network's."""
    rng = np.random.default_rng(3)
    n = 2048
    q = rng.uniform(-0.2, 1.2, size=(n, 14)).astype(np.float32)
    q[:, 3:8] = rng.uniform(-np.pi, np.pi, size=(n, 5))
    q[:200, 3:8] = rng.choice(np.array([0.0, 0.25, 0.5, 0.75, 1.0, -1.0], dtype=np.float32), size=(200, 5))
    tri = OW.OracleNrcTriWave(2, 1e-2)
    hg = oracle.OracleNrc(2, 1e-2)
    hg.set_params(np.zeros(hg.num_params, dtype=np.float16))
    et, eh = tri.encode(q).view(np.uint16), hg.encode(q).view(np.uint16)
    assert np.array_equal(et[:, 36:56], one_blob_aos_numpy(q[:, 3:8]).view(np.uint16))
    assert np.array_equal(et[:, 56:62], eh[:, 52:58])
    assert (et[:, 62:].view(np.float16) == 1.0).all()
    assert not np.array_equal(et[:, 36:56], eh[:, 32:52])  # the two one-blob kernels do differ


def test_encoding_equals_tiny_cuda_nns_stored_encoding(oracle):
    """the stored output of the reference network's own Composite encoding (tests/golden/tcnn_nrc_triwave.npz), half for half"""
    from tests.tcnn_nrc_triwave_check import GOLDEN, N_ENCODE, encode_queries
    want = np.load(GOLDEN)["encoding"]
    assert want.shape == (N_ENCODE, 64)
    got = OW.OracleNrcTriWave(2, 1e-2).encode(encode_queries()).view(np.uint16)
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{len(bad)} halves differ, first {bad[:5].tolist()}"


def test_parameter_count_is_the_matrix_weights(oracle):
    for hidden in range(1, 8):
        net = OW.OracleNrcTriWave(hidden, 1e-2)
        assert net.num_matrix_weights == 64 * 64 * hidden + 16 * 64
        assert net.num_params == net.num_matrix_weights, hidden
    # the default stays the hash grid
    assert oracle.OracleNrc(2, 1e-2).num_params == 64 * 64 * 2 + 16 * 64 + (4096 + 15 * 32768) * 2


def _forward64(x, w, hidden):
    """the network in float64 without intermediate roundings: x [n][64], w = the matrix weights"""
    h = x
    for l in range(hidden):
        h = np.maximum(h @ w[64 * 64 * l:64 * 64 * (l + 1)].reshape(64, 64).T, 0.0)
    return (h @ w[64 * 64 * hidden:].reshape(16, 64).T)[:, :3]


def test_matrix_gradients_match_finite_differences(oracle):
    """RelativeL2Luminance's gradient holds the luminance denominator fixed (relative_l2_luminance.h:41-88), so the finite
    differences are taken of sum (y - t)^2 / denom0 / (3 n) with denom0 from the unperturbed output.  The oracle's gradients
    (loss-scaled by 128, fp16 activations) must match the float64 directional derivatives along random directions, matrix by
    matrix, within 2 %."""
    hidden, n = 2, 512
    net = OW.OracleNrcTriWave(hidden, 1e-2)
    params = engine.random_nrc_params(net.num_params, net.num_matrix_weights, seed=4)
    net.set_params(params)
    q = _queries(n, 5)
    t = np.stack([0.5 + 0.4 * np.sin(6 * q[:, 0]), q[:, 1] * q[:, 8], 0.3 + 0.5 * q[:, 2]], axis=1)
    x = net.encode(q).astype(np.float64)
    w = params.astype(np.float64)
    y0 = _forward64(x, w, hidden)
    lum = y0 @ np.array([0.299, 0.587, 0.114])
    denom0 = (lum * lum + 0.01)[:, None]

    def loss(wv):
        return float((((_forward64(x, wv, hidden) - t) ** 2) / denom0).sum() / (3 * n))

    net.train(q, t.astype(np.float32))
    g = net.get_gradients() / 128.0
    rng = np.random.default_rng(6)
    bounds = [(64 * 64 * l, 64 * 64 * (l + 1)) for l in range(hidden)] + [(64 * 64 * hidden, net.num_matrix_weights)]
    eps = 1e-4
    for lo, hi in bounds:
        for _ in range(3):
            d = np.zeros_like(w)
            d[lo:hi] = rng.standard_normal(hi - lo)
            fd = (loss(w + eps * d) - loss(w - eps * d)) / (2 * eps)
            an = float(g @ d)
            assert abs(fd - an) <= 2e-2 * abs(fd) + 1e-7, (lo, fd, an)


def test_training_learns_target(oracle):
    net = OW.OracleNrcTriWave(2, 1e-2)
    net.set_params(engine.random_nrc_params(net.num_params, net.num_matrix_weights))
    q = _queries(2048, 3)
    target = np.stack([0.5 + 0.4 * np.sin(6 * q[:, 0]), q[:, 1] * q[:, 8], 0.3 + 0.5 * q[:, 2]], axis=1).astype(np.float32)
    losses = [net.train(q, target) for _ in range(40)]
    assert np.isfinite(losses).all()
    assert losses[-1] < 0.25 * losses[0], losses[::8]
    pred = net.infer(q)
    assert np.mean((pred - target) ** 2) < 0.05


def test_oracle_for_each_encoding():
    import pytest
    assert isinstance(OW.oracle_nrc(2, 1e-2, TRI), OW.OracleNrcTriWave)
    assert OW.oracle_nrc(2, 1e-2, HASH).num_params == 64 * 64 * 2 + 16 * 64 + (4096 + 15 * 32768) * 2
    with pytest.raises(ValueError):
        OW.oracle_nrc(2, 1e-2, 2)


# ---- the NRC strip frames with a triangle-wave net (tests/test_multigpu_cpu.py's setup), world_size 2 over gloo ---------------
def _nrc_setup_tri():
    from tests import test_multigpu_cpu as T
    O, oframe, _, p = T._nrc_setup()
    onet = OW.OracleNrcTriWave(2, 1e-2)
    onet.set_params(engine.random_nrc_params(onet.num_params, onet.num_matrix_weights))
    return T, O, oframe, onet, p


def _worker_nrc_tri(rank, world, port, result_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    T, O, oframe, onet, p = _nrc_setup_tri()
    oframe.nrc_shard(rank, world)
    rows = (rank * T.NRC_H // world, (rank + 1) * T.NRC_H // world)
    out = {}
    for f in range(T.NRC_FRAMES):
        T._nrc_frame(O, oframe, onet, p, f, rows)
        out[f"beauty{f}"] = oframe.buffer(abi.BUF_BEAUTY_ACCUM)[rows[0]:rows[1]].copy()
        out[f"records{f}"] = oframe.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 0).copy()
        out[f"targets{f}"] = oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0).copy()
    out["weights"] = onet.get_master()
    np.savez(result_path + f".{rank}.npz", **out)
    dist.barrier()
    dist.destroy_process_group()


def test_nrc_strips_with_triangle_wave_net_equal_single_process(tmp_path):
    """images, records and trained weights of both ranks equal the unsharded frames bit for bit"""
    from tests import test_multigpu_cpu as T
    result = str(tmp_path / "nrc_tri")
    mp.spawn(_worker_nrc_tri, args=(2, T._free_port(), result), nprocs=2, join=True)
    T, O, oframe, onet, p = _nrc_setup_tri()
    got = [np.load(result + f".{r}.npz") for r in range(2)]
    for f in range(T.NRC_FRAMES):
        T._nrc_frame(O, oframe, onet, p, f)
        st = oframe.linear_buffer(abi.BUF_NRC_STATE)[:8, 0]
        ntrain = min(int(st[f % 2]), abi.NRC_TRAIN_BUFFER_SIZE)
        assert ntrain > 30, "vacuous: no training vertices"
        beauty = oframe.buffer(abi.BUF_BEAUTY_ACCUM)
        for r in range(2):
            rows = slice(r * T.NRC_H // 2, (r + 1) * T.NRC_H // 2)
            assert np.array_equal(got[r][f"beauty{f}"].view(np.uint32), beauty[rows].view(np.uint32)), f"frame {f} rank {r}: image"
            assert np.array_equal(got[r][f"records{f}"][:ntrain].view(np.uint32),
                                  oframe.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 0)[:ntrain].view(np.uint32)), f"frame {f} rank {r}"
            assert np.array_equal(got[r][f"targets{f}"][:ntrain].view(np.uint32),
                                  oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain].view(np.uint32)), f"frame {f} rank {r}"
    want = onet.get_master()
    for r in range(2):
        assert np.array_equal(got[r]["weights"].view(np.uint32), want.view(np.uint32)), f"rank {r}: trained weights"
