"""GPU parity: the NRC network (fused hash-grid/one-blob/identity encoding + wgmma MLP inference and training step;
the CUDA-core training kernel is the A/B arm and the deep-network fallback) vs the CPU oracle.  Tensor-core accumulation order is hardware-defined, so the bar is
<= 1e-3 relative L2 on inference (BASELINE.json north_star) and agreement of gradients, loss curves and weights on training.
Between the GPU's own inference paths (fused / split kernels, launch sizes, aligned or not) the radiance is compared bit for bit."""
import re

import numpy as np
import pytest

from gfxexp_b200 import abi, engine

pytestmark = pytest.mark.gpu


def _queries(n, seed=0):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.0, 1.0, size=(n, 14)).astype(np.float32)


def _tile_queries(num_tiles, seed):
    """distinct random queries in every 128-query tile, each tile with the rows where encodings go wrong: grid corners, cell
    boundaries of the coarsest and of a fine level, one-blob bin boundaries"""
    rng = np.random.default_rng(seed)
    q = _queries(num_tiles * 128, seed).reshape(num_tiles, 128, 14)
    q[:, :8, :3] = 0.0
    q[:, 8:16, :3] = 1.0
    q[:, 16:32, :3] = rng.integers(0, 17, size=(num_tiles, 16, 3)) / 16.0
    q[:, 32:48, :3] = rng.integers(0, 513, size=(num_tiles, 16, 3)) / 512.0
    q[:, 48:64, 3:8] = rng.choice([0.0, 0.25, 0.5, 0.75, 1.0], size=(num_tiles, 16, 5))
    return np.ascontiguousarray(q.reshape(-1, 14))


def _misaligned(t):
    """a copy of t that starts 4 bytes past a 16-byte boundary, which the split path's TMA bulk copies cannot take: inference
    on it runs the fused kernel"""
    import torch
    storage = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    storage[1:] = t.reshape(-1)
    view = storage[1:].view(t.shape)
    assert view.data_ptr() % 16 == 4
    return view


def _rel_l2(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-20))


def _same_bits(got, want, tag):
    g, w = np.ascontiguousarray(got).view(np.uint32), np.ascontiguousarray(want).view(np.uint32)
    bad = np.argwhere(g != w)
    assert bad.size == 0, f"{tag}: {len(bad)} values differ, first at {bad[:4].tolist()}"


@pytest.mark.parametrize("hidden,amp", [(1, 0.5), (2, 1e-4), (2, 0.5), (3, 0.5), (4, 0.5), (5, 0.5), (6, 0.5), (7, 0.5)])
def test_inference_matches_oracle(gfx_ctx, oracle, hidden, amp):
    import torch
    onet = oracle.OracleNrc(hidden, 1e-2)
    params = engine.random_nrc_params(onet.num_params, onet.num_matrix_weights, seed=7 + hidden, grid_amplitude=amp)
    onet.set_params(params)
    gnet = engine.NeuralRadianceCache(gfx_ctx, hidden, 1e-2)
    assert gnet.num_params == onet.num_params
    gnet.set_params(params)
    n = 128 * 300
    q = _queries(n, 5)
    q[:64, :3] = 0.0      # grid corners / cell boundaries
    q[64:128, :3] = 1.0
    dq = torch.from_numpy(q).cuda()
    out = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    gnet.infer(dq, out, n)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    want = onet.infer(q)
    assert np.isfinite(got).all()
    assert _rel_l2(got, want) <= 1e-3, _rel_l2(got, want)
    gnet.close()


def test_split_encoding_is_bit_exact(gfx_ctx, oracle):
    """the encoded network input of the split inference path (positions packed, one hash-grid level per CTA with the level's
    table staged in shared memory by TMA, one-blob + identity in the MLP kernel) equals the oracle's - which is pinned bit for
    bit against tiny-cuda-nn's kernel_grid / kernel_one_blob_soa (tests/test_gpu_tcnn_ref.py) - in every half"""
    import torch
    onet = oracle.OracleNrc(2, 1e-2)
    params = engine.random_nrc_params(onet.num_params, onet.num_matrix_weights, seed=3, grid_amplitude=0.5)
    onet.set_params(params)
    gnet = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    gnet.set_params(params)
    n = 128 * 150 + 128  # not a multiple of the replica count
    q = _queries(n, 9)
    rng = np.random.default_rng(4)
    q[:64, :3] = 0.0
    q[64:128, :3] = 1.0
    q[128:256, :3] = (rng.integers(0, 17, size=(128, 3)) / 16.0).astype(np.float32)   # level-0 cell corners
    q[256:384, :3] = (rng.integers(0, 513, size=(128, 3)) / 512.0).astype(np.float32)  # finer cell corners
    q[384:512, 3:8] = rng.choice([0.0, 0.25, 0.5, 0.75, 1.0], size=(128, 5)).astype(np.float32)
    got = gnet.encode(torch.from_numpy(q).cuda(), n).view(np.uint16)
    want = onet.encode(q).view(np.uint16).reshape(n, 64)
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{len(bad)} halves differ, first {bad[:5].tolist()}"
    gnet.close()


@pytest.mark.parametrize("hidden", [2, 7])  # k_nrcInferMlp runs 3 CTAs per SM at depth 2, 2 at depth 7
def test_frame_sized_batch_matches_one_tile_per_cta(gfx_ctx, oracle, hidden):
    """Both inference kernels are persistent: k_nrcInferMlp's grid is SMs x (CTAs per SM), k_nrcInfer's 6 x SMs, and a CTA walks
    the tiles with that stride.  At a 1080p frame's ~17 000 tiles every CTA handles dozens, through the double-buffered TMA
    stage (prefetch into the other buffer, mbarrier parity flip on reuse) and the output staging buffer that the previous tile's
    bulk store must have drained.  A batch with at least 3 tiles per CTA of either kernel must give the same bits as launches
    of at most SMs tiles, in which every CTA handles a single tile, and the oracle's radiance at the inference bar.  k_nrcInfer
    runs on a copy of the queries that is not 16-byte aligned."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    num_tiles = max(4096, 3 * 6 * sms)
    n = num_tiles * 128
    q = _tile_queries(num_tiles, 31 + hidden)
    onet = oracle.OracleNrc(hidden, 1e-2)
    params = engine.random_nrc_params(onet.num_params, onet.num_matrix_weights, seed=40 + hidden, grid_amplitude=0.5)
    onet.set_params(params)
    gnet = engine.NeuralRadianceCache(gfx_ctx, hidden, 1e-2)
    gnet.set_params(params)
    dq = torch.from_numpy(q).cuda()
    whole, chunked, fused = (torch.full((n, 3), float("nan"), device="cuda") for _ in range(3))
    gnet.infer(dq, whole, n)
    step = sms * 128
    for lo in range(0, n, step):
        m = min(step, n - lo)
        gnet.infer(dq[lo:lo + m], chunked[lo:lo + m], m)
    gnet.infer(_misaligned(dq), fused, n)
    torch.cuda.synchronize()
    whole, chunked, fused = (t.cpu().numpy() for t in (whole, chunked, fused))
    assert np.isfinite(whole).all()
    _same_bits(whole, chunked, "split path: whole batch vs one tile per CTA")
    _same_bits(fused, whole, "fused path vs split path")
    want = onet.infer(q)
    assert _rel_l2(whole, want) <= 1e-3, _rel_l2(whole, want)
    gnet.close()


def test_unaligned_buffers_take_the_fused_path(gfx_ctx):
    """queries or radiance that are not 16-byte aligned cannot go through the TMA bulk copies of the split path; the fused kernel
    takes them, gives the same bits and writes nothing outside the output rows"""
    import torch
    n = 128 * 77
    gnet = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    gnet.set_params(engine.random_nrc_params(gnet.num_params, 64 * 64 * 2 + 16 * 64, seed=8, grid_amplitude=0.5))
    dq = torch.from_numpy(_tile_queries(77, 13)).cuda()
    aligned = torch.empty((n, 3), device="cuda")
    gnet.infer(dq, aligned, n)
    sentinel = -12345.0
    for q_offset, out_offset in ((1, 0), (0, 1), (1, 1)):
        q_storage = torch.empty(n * 14 + 1, device="cuda")
        q_storage[q_offset:q_offset + n * 14] = dq.view(-1)
        qv = q_storage[q_offset:q_offset + n * 14].view(n, 14)
        out_storage = torch.full((n * 3 + 2,), sentinel, device="cuda")
        out = out_storage[out_offset:out_offset + n * 3].view(n, 3)
        assert qv.data_ptr() % 16 == 4 * q_offset and out.data_ptr() % 16 == 4 * out_offset
        gnet.infer(qv, out, n)
        torch.cuda.synchronize()
        _same_bits(out.cpu().numpy(), aligned.cpu().numpy(), f"query offset {4 * q_offset} B, output offset {4 * out_offset} B")
        rest = torch.cat([out_storage[:out_offset], out_storage[out_offset + n * 3:]])
        assert (rest == sentinel).all(), rest
    gnet.close()


def test_infer_rejects_unpadded_batch(gfx_ctx):
    import torch
    gnet = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    dq = torch.zeros((100, 14), device="cuda")
    out = torch.zeros((100, 3), device="cuda")
    with pytest.raises(engine.GfxError):
        gnet.infer(dq, out, 100)  # network_interface.cu:143 requires numData % 128 == 0
    gnet.close()


def test_training_tracks_oracle(gfx_ctx, oracle):
    import torch
    onet = oracle.OracleNrc(2, 1e-2)
    params = engine.random_nrc_params(onet.num_params, onet.num_matrix_weights, seed=11)
    onet.set_params(params)
    gnet = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    gnet.set_params(params)
    n = 4096
    q = _queries(n, 9)
    target = np.stack([0.5 + 0.4 * np.sin(6 * q[:, 0]), q[:, 1] * q[:, 8], 0.3 + 0.5 * q[:, 2]], axis=1).astype(np.float32)
    dq, dt = torch.from_numpy(q).cuda(), torch.from_numpy(target).cuda()
    gl, ol = [], []
    for _ in range(12):
        gl.append(gnet.train(dq, dt, n, want_loss=True))
        ol.append(onet.train(q, target))
    gl, ol = np.array(gl), np.array(ol)
    assert np.isfinite(gl).all()
    assert np.abs(gl - ol).max() <= 0.05 * ol.max(), (gl, ol)
    assert gl[-1] < 0.5 * gl[0]
    # inference after training (EMA weights) agrees
    out = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    gnet.infer(dq, out, n)
    torch.cuda.synchronize()
    assert _rel_l2(out.cpu().numpy(), onet.infer(q)) <= 2e-2
    gnet.close()


def _train_targets(q):
    return np.stack([0.5 + 0.4 * np.sin(6 * q[:, 0]), q[:, 1] * q[:, 8], 0.3 + 0.5 * q[:, 2]], axis=1).astype(np.float32)


def _parameter_slices(hidden, num_matrix_weights, num_params):
    out = {f"W{l}": slice(64 * 64 * l, 64 * 64 * (l + 1)) for l in range(hidden)}
    out[f"W{hidden}"] = slice(64 * 64 * hidden, num_matrix_weights)
    out["grid"] = slice(num_matrix_weights, num_params)
    return out


def _cuda_core_training_smem(hidden):
    """dynamic shared memory of k_nrcTrain: the fp16 weights and (hidden + 2) activation / gradient tiles of 128 rows x 66"""
    return (64 * 64 * hidden + 16 * 64 + (hidden + 2) * 128 * 66) * 2


# the depth chooses the training kernel: the wgmma kernel for 1..3 hidden layers, the CUDA-core kernel for 4..8
@pytest.mark.parametrize("hidden", [1, 2, 3, 4, 5, 6, 7, 8])
def test_training_step_matches_oracle(gfx_ctx, oracle, hidden):
    """One training step from the same weights, on a batch of 16 384 and on one of 128 x 37 samples (not a multiple of the SM
    count): the loss within 1e-4 relative of the fp32-accumulating oracle's, and the gradient of every weight matrix within 1e-4
    relative L2, of the hash grid within 1e-3 - the bars of the depth-2 check against tiny-cuda-nn (tests/test_gpu_tcnn_nrc.py).
    Where the wgmma kernel's accumulation order flips more fp16 roundings than that (the smaller batch, other depths than 2), the
    gradient must still be no further from the oracle than the oracle's own rounding spread on the same step: its
    half-accumulating mode against its fp32 one.  Then four full steps (Adam, EMA): what they changed in the training and the
    inference weights, per matrix, within the 2e-2 of test_training_tracks_oracle.
    A depth whose kernels do not fit in shared memory must be refused when the network is created, not when it first trains."""
    import torch
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    try:
        gnet = engine.NeuralRadianceCache(gfx_ctx, hidden, 1e-2)
    except engine.GfxError as e:
        assert _cuda_core_training_smem(hidden) > limit, e
        assert re.search(f"{hidden} hidden layers need .* k_nrcTrain, more than the device's limit of {limit} bytes", str(e)), e
        return
    onet = oracle.OracleNrc(hidden, 1e-2)
    params = engine.random_nrc_params(onet.num_params, onet.num_matrix_weights, seed=50 + hidden, grid_amplitude=0.5)
    gnet.keep_gradients(True)
    slices = _parameter_slices(hidden, onet.num_matrix_weights, onet.num_params)
    for n, seed in ((16384, 61), (128 * 37, 62)):
        q = _queries(n, seed)
        t = _train_targets(q)
        gnet.set_params(params)
        onet.set_params(params)
        loss = gnet.train(torch.from_numpy(q).cuda(), torch.from_numpy(t).cuda(), n, want_loss=True)
        grads = gnet.read(abi.NRC_READ_GRADIENTS)
        oloss = onet.train(q, t)
        ograds = onet.get_gradients()
        assert abs(loss - oloss) <= 1e-4 * abs(oloss), (n, loss, oloss)
        over = {}
        for name, sl in slices.items():
            rel = _rel_l2(grads[sl], ograds[sl])
            if rel > (1e-3 if name == "grid" else 1e-4):
                over[name] = rel
        if over:
            onet.set_params(params)
            onet.set_accumulate_half(True)
            onet.train(q, t)
            spread = onet.get_gradients()
            onet.set_accumulate_half(False)
            for name, rel in over.items():
                own = _rel_l2(spread[slices[name]], ograds[slices[name]])
                assert rel <= own, (n, name, rel, own)

    gnet.set_params(params)
    onet.set_params(params)
    for step in range(4):
        q = _queries(16384, 70 + step)
        t = _train_targets(q)
        gnet.train(torch.from_numpy(q).cuda(), torch.from_numpy(t).cuda(), 16384)
        onet.train(q, t)
    start = params.astype(np.float32)
    for which, ema in ((abi.NRC_READ_TRAINING, False), (abi.NRC_READ_INFERENCE, True)):
        got = gnet.read(which).astype(np.float32)
        want = onet.get_params(ema=ema).astype(np.float32)
        for name, sl in slices.items():
            # on the update rather than the weights: the weights' relative difference is smaller by |update| / |weights|
            rel = _rel_l2(got[sl] - start[sl], want[sl] - start[sl])
            assert rel <= 2e-2, ("EMA" if ema else "training", name, rel)
    gnet.close()


def test_tensor_core_training_is_deterministic(gfx_ctx):
    import torch
    n = 4096
    q = _queries(n, 22)
    target = np.stack([q[:, 0], q[:, 1], q[:, 2]], axis=1).astype(np.float32)
    dq, dt = torch.from_numpy(q).cuda(), torch.from_numpy(target).cuda()
    outs = []
    for _ in range(2):
        net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
        net.set_params(engine.random_nrc_params(net.num_params, 64 * 64 * 2 + 16 * 64, seed=5))
        for _ in range(6):
            net.train(dq, dt, n)
        out = torch.empty((n, 3), dtype=torch.float32, device="cuda")
        net.infer(dq, out, n)
        torch.cuda.synchronize()
        outs.append(out.cpu().numpy())
        net.close()
    assert np.array_equal(outs[0], outs[1])
