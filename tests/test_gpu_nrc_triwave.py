"""GPU parity of the triangle-wave NRC network (gfx_nrc_create_with_encoding(GFX_NRC_POSITION_ENCODING_TRIANGLE_WAVE, ...)) with
the CPU oracle: inference at every trainable depth, the persistent inference kernel at frame-sized batches, unaligned buffers,
one training step on both training kernels at every depth, determinism, and the NRC frame launches with a triangle-wave net.
The bars are those of tests/test_gpu_nrc.py and tests/test_gpu_nrc_frame.py."""
import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_nrc_triwave as OW
from tests.test_gpu_nrc import _misaligned, _queries, _rel_l2, _same_bits, _tile_queries, _train_targets
from tests.test_gpu_nrc_frame import SEEDED_TILE, _compare_pathtrace, _same, _seeded_preprocess

pytestmark = pytest.mark.gpu
TRI = abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE


def _nets(gfx_ctx, oracle, hidden, seed):
    onet = OW.OracleNrcTriWave(hidden, 1e-2)
    params = engine.random_nrc_params(onet.num_params, onet.num_matrix_weights, seed=seed)
    onet.set_params(params)
    gnet = engine.NeuralRadianceCache(gfx_ctx, hidden, 1e-2, position_encoding=TRI)
    assert gnet.num_params == onet.num_params == onet.num_matrix_weights
    gnet.set_params(params)
    return gnet, onet, params


def test_unknown_encoding_is_rejected(gfx_ctx):
    import ctypes as C
    h = C.c_void_p()
    assert gfx_ctx.lib.gfx_nrc_create_with_encoding(gfx_ctx.h, 2, 2, 1e-2, C.byref(h)) != 0 and not h.value
    assert gfx_ctx.lib.gfx_nrc_create_with_encoding(gfx_ctx.h, -1, 2, 1e-2, C.byref(h)) != 0 and not h.value


@pytest.mark.parametrize("hidden", [1, 2, 3, 4, 5, 6, 7])
def test_inference_matches_oracle(gfx_ctx, oracle, hidden):
    import torch
    gnet, onet, _ = _nets(gfx_ctx, oracle, hidden, 7 + hidden)
    n = 128 * 300
    q = _tile_queries(300, 5)
    q[:1024, :3] = np.random.default_rng(1).uniform(-2.0, 3.0, size=(1024, 3))  # outside the unit cube
    out = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    gnet.infer(torch.from_numpy(q).cuda(), out, n)
    torch.cuda.synchronize()
    got, want = out.cpu().numpy(), onet.infer(q)
    assert np.isfinite(got).all()
    assert _rel_l2(got, want) <= 1e-3, _rel_l2(got, want)
    gnet.close()


def test_encoding_is_bit_exact(gfx_ctx, oracle):
    """gfx_nrc_encode_debug (the nrcEncodeTriWave the inference and training kernels run) equals the oracle's encoding, which
    tests/test_oracle_nrc_triwave.py pins against triangle_wave_encoding bit for bit"""
    import torch
    from tests.tcnn_nrc_triwave_check import adversarial_positions
    gnet, onet, _ = _nets(gfx_ctx, oracle, 2, 3)
    n = 128 * 64
    q = _tile_queries(64, 9)
    q[:4096, :3] = adversarial_positions(4096, 11)
    got = gnet.encode(torch.from_numpy(q).cuda(), n).view(np.uint16)
    want = onet.encode(q).view(np.uint16)
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{len(bad)} halves differ, first {bad[:5].tolist()}"
    gnet.close()


@pytest.mark.parametrize("hidden", [2, 7])
def test_frame_sized_batch_matches_one_tile_per_cta(gfx_ctx, oracle, hidden):
    """A batch with at least 3 tiles per CTA gives the same bits as launches in which every CTA handles one tile: on the
    persistent kernel (double-buffered TMA stage, output staging), and on the fused kernel, which takes a copy of the queries
    that is not 16-byte aligned"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    num_tiles = max(4096, 3 * 6 * sms)
    n = num_tiles * 128
    q = _tile_queries(num_tiles, 31 + hidden)
    gnet, onet, _ = _nets(gfx_ctx, oracle, hidden, 40 + hidden)
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
    _same_bits(whole, chunked, "whole batch vs one tile per CTA")
    _same_bits(fused, whole, "fused kernel vs persistent kernel")
    assert _rel_l2(whole, onet.infer(q)) <= 1e-3
    gnet.close()


def test_unaligned_buffers(gfx_ctx, oracle):
    """queries or radiance that are not 16-byte aligned take the one-kernel path with L2 loads: same bits, nothing written
    outside the output"""
    import torch
    n = 128 * 77
    gnet, _, _ = _nets(gfx_ctx, oracle, 2, 8)
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
        gnet.infer(qv, out, n)
        torch.cuda.synchronize()
        _same_bits(out.cpu().numpy(), aligned.cpu().numpy(), f"query offset {4 * q_offset} B, output offset {4 * out_offset} B")
        rest = torch.cat([out_storage[:out_offset], out_storage[out_offset + n * 3:]])
        assert (rest == sentinel).all(), rest
    gnet.close()


@pytest.mark.parametrize("hidden", [1, 2, 3, 4, 5, 6, 7])
def test_training_step_matches_oracle(gfx_ctx, oracle, hidden):
    """One step on 16 384 and on 128 x 37 samples: the loss within 1e-4 relative, every matrix gradient within 1e-4 relative L2
    or, where the accumulation order flips more fp16 roundings, within the oracle's own half-vs-fp32 accumulation spread or
    2.5e-4, whichever is larger (the triangle wave's inputs are of order 1, not 1e-4 like a fresh hash grid's, so the
    pre-activations and their roundings are larger; the bar against tiny-cuda-nn itself is 2.5e-3).  Then four Adam
    (epsilon 1e-8) / EMA steps, per matrix, within 2e-2 on the update."""
    import torch
    gnet, onet, params = _nets(gfx_ctx, oracle, hidden, 50 + hidden)
    gnet.keep_gradients(True)
    M = onet.num_matrix_weights
    slices = {f"W{l}": slice(64 * 64 * l, 64 * 64 * (l + 1)) for l in range(hidden)}
    slices[f"W{hidden}"] = slice(64 * 64 * hidden, M)
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
        over = {name: _rel_l2(grads[sl], ograds[sl]) for name, sl in slices.items() if _rel_l2(grads[sl], ograds[sl]) > 1e-4}
        if over:
            onet.set_params(params)
            onet.set_accumulate_half(True)
            onet.train(q, t)
            spread = onet.get_gradients()
            onet.set_accumulate_half(False)
            for name, rel in over.items():
                own = _rel_l2(spread[slices[name]], ograds[slices[name]])
                assert rel <= max(own, 2.5e-4), (n, name, rel, own)
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
            rel = _rel_l2(got[sl] - start[sl], want[sl] - start[sl])
            assert rel <= 2e-2, ("EMA" if ema else "training", name, rel)
    gnet.close()


@pytest.mark.parametrize("hidden", [2, 4])
def test_training_is_deterministic(gfx_ctx, oracle, hidden):
    """the 64-bit fixed-point gradient accumulation of both training kernels (wgmma at 2 hidden layers, CUDA cores at 4): two
    runs of four steps give the same weights, bit for bit"""
    import torch
    n = 16384
    q = _queries(n, 22)
    dq, dt = torch.from_numpy(q).cuda(), torch.from_numpy(_train_targets(q)).cuda()
    runs = []
    for _ in range(2):
        gnet, _, _ = _nets(gfx_ctx, oracle, hidden, 5)
        for _ in range(4):
            gnet.train(dq, dt, n)
        runs.append((gnet.read(abi.NRC_READ_MASTER), gnet.read(abi.NRC_READ_INFERENCE)))
        gnet.close()
    assert np.array_equal(runs[0][0].view(np.uint32), runs[1][0].view(np.uint32))
    assert np.array_equal(runs[0][1].view(np.uint16), runs[1][1].view(np.uint16))


def test_fresh_network_is_tcnn_trainer_state(gfx_ctx):
    """Trainer{seed 1337}: the matrices are the hash-grid network's (the same pcg32 prefix), nothing follows them, the EMA
    weights are zero"""
    tri = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2, position_encoding=TRI)
    hg = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    M = 64 * 64 * 2 + 16 * 64
    assert tri.num_params == M
    assert np.array_equal(tri.read(abi.NRC_READ_MASTER).view(np.uint32), hg.read(abi.NRC_READ_MASTER)[:M].view(np.uint32))
    assert np.array_equal(tri.read(abi.NRC_READ_TRAINING).view(np.uint16), hg.read(abi.NRC_READ_TRAINING)[:M].view(np.uint16))
    assert not tri.read(abi.NRC_READ_INFERENCE).any()
    tri.close()
    hg.close()


@pytest.mark.parametrize("w,h,strips", [(192, 108, [(0, 34), (34, 80), (80, 108)]),
                                         (1920, 1080, [(0, 360), (360, 1001), (1001, 1080)]),
                                         (3840, 2160, [(0, 720), (720, 2002), (2002, 2160)])])
def test_frame_inference_matches_direct_inference(gfx_ctx, oracle, w, h, strips):
    """gfx_nrc_frame_infer with a triangle-wave net: the device-side query count, a NaN sentinel beyond it, the bits of
    gfx_nrc_infer on the same queries; gfx_nrc_frame_infer_rows over three strips: the same bits, nothing else written"""
    import torch
    scene = scenes.small_city_scene()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    gfx_ctx.build_light_distributions(0)
    net, _, _ = _nets(gfx_ctx, oracle, 2, 19)
    p = abi.default_frame_params(scene, w, h)
    tile = SEEDED_TILE.get((w, h))
    gfx_ctx.gbuffer(p)
    _seeded_preprocess(gfx_ctx, p, tile, (0x2545F491, 0x9E3779B9))
    gfx_ctx.pathtrace(p, abi.PT_NRC)
    n, capacity = w * h, abi.nrc_query_capacity(w, h)
    sentinel = np.full((capacity, 3), 0x7FC0DEAD, dtype=np.uint32).view(np.float32)
    gfx_ctx.upload(abi.BUF_NRC_INFERRED_RADIANCE, 0, sentinel)
    gfx_ctx.nrc_frame_infer(net)
    frame = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
    st = gfx_ctx.download_linear(abi.BUF_NRC_STATE)[:, 0]
    count, num_suffix = int(st[abi.NRC_STATE_NUM_INFERENCE_QUERIES]), int(st[abi.NRC_STATE_NUM_SUFFIX_QUERIES])
    assert count % 128 == 0 and n < count <= capacity and count == n + num_suffix
    if tile is not None:
        assert st[abi.NRC_STATE_TILE_SIZE] == tile and count == capacity == n + ((w + 3) // 4) * ((h + 3) // 4), (count, capacity)
    _same(frame[count:], sentinel[count:], "rows beyond the device-side query count")
    queries = torch.from_numpy(gfx_ctx.download_linear(abi.BUF_NRC_INFERENCE_QUERY)[:count]).cuda()
    direct = torch.empty((count, 3), device="cuda")
    step = torch.cuda.get_device_properties(0).multi_processor_count * 128
    for lo in range(0, count, step):
        m = min(step, count - lo)
        net.infer(queries[lo:lo + m], direct[lo:lo + m], m)
    torch.cuda.synchronize()
    _same(frame[:count], direct.cpu().numpy(), "frame inference vs gfx_nrc_infer")
    for lo, hi in strips:
        gfx_ctx.upload(abi.BUF_NRC_INFERRED_RADIANCE, 0, sentinel)
        gfx_ctx._check(gfx_ctx.lib.gfx_nrc_frame_infer_rows(gfx_ctx.h, net.h, None, lo, hi), "gfx_nrc_frame_infer_rows")
        got = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
        first, end = lo * w, lo * w + ((hi - lo) * w + 127) // 128 * 128
        _same(got[first:hi * w], frame[first:hi * w], f"rows {lo}..{hi}: pixel queries")
        _same(got[n:n + num_suffix], frame[n:n + num_suffix], f"rows {lo}..{hi}: suffix queries")
        _same(got[:first], sentinel[:first], f"rows {lo}..{hi}: before the strip")
        _same(got[end:n], sentinel[end:n], f"rows {lo}..{hi}: after the strip")
        _same(got[n + num_suffix:], sentinel[n + num_suffix:], f"rows {lo}..{hi}: beyond the suffix queries")
    net.close()


def test_nrc_frames_bit_exact(gfx_ctx, oracle):
    """three NRC frames with a triangle-wave net: the GPU's predictions within the inference bar of the oracle's; accumulate,
    propagate and shuffle on those predictions equal the oracle's bit for bit; the frame's training tracks the oracle's"""
    scene = scenes.small_city_scene()
    w, h = 192, 108
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    gfx_ctx.build_light_distributions(0)
    oframe = oracle.OracleFrame(oracle.OracleScene(scene), w, h)
    net, onet, _ = _nets(gfx_ctx, oracle, 2, 1337)
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = 5
    p.radianceScale = 2.0
    rng = np.random.default_rng(7)
    n = w * h
    for frame in range(3):
        p.frameIndex, p.bufferIndex, p.numAccumFrames = frame, frame % 2, frame
        offsets = [int(rng.integers(0, 2 ** 32)) for _ in range(2)]
        gfx_ctx.gbuffer(p)
        gfx_ctx.nrc_preprocess(p, offsets[0], offsets[1], frame == 0)
        gfx_ctx.pathtrace(p, abi.PT_NRC)
        oframe.gbuffer(p)
        oframe.nrc_preprocess(p, offsets[0], offsets[1], frame == 0)
        oframe.pathtrace(p, abi.PT_NRC)
        ntrain, has_query, suffix_query = _compare_pathtrace(gfx_ctx, oframe, p, f"frame {frame}")
        gfx_ctx.nrc_frame_infer(net)
        pred = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
        q = oframe.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)
        rows = np.concatenate([np.flatnonzero(has_query), n + np.flatnonzero(suffix_query)])
        assert _rel_l2(pred[rows], onet.infer(q[rows])) <= 1e-3
        oframe.linear_buffer(abi.BUF_NRC_INFERRED_RADIANCE, copy=False)[:] = pred
        gfx_ctx.nrc_accumulate(p)
        oframe.nrc_accumulate(p)
        _same(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), oframe.buffer(abi.BUF_BEAUTY_ACCUM), f"frame {frame} beauty")
        gfx_ctx.nrc_propagate(p)
        oframe.nrc_propagate(p)
        _same(gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain], oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain],
              f"frame {frame} propagated targets")
        gfx_ctx.nrc_shuffle(p)
        oframe.nrc_shuffle(p)
        tq_g, tt_g = gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_QUERY, 1), gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_TARGET, 1)
        m = abi.NRC_TRAINING_DATA_PER_FRAME
        _same(tq_g[:m], oframe.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 1)[:m], f"frame {frame} shuffled queries")
        _same(tt_g[:m], oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 1)[:m], f"frame {frame} shuffled targets")
        loss = gfx_ctx.nrc_frame_train(net, want_loss=True)
        oloss = None
        for step in range(4):
            sl = slice(step * 16384, (step + 1) * 16384)
            oloss = onet.train(tq_g[sl], tt_g[sl])
        assert np.isfinite(loss) and abs(loss - oloss) <= 0.05 * abs(oloss) + 1e-4, (loss, oloss)
    net.close()
