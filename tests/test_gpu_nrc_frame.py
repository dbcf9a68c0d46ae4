"""GPU parity: the NRC path tracer and its bookkeeping kernels vs the CPU oracle (SURVEY.md §8a rows N1-N3).
Everything the path tracer writes is compared bit for bit - including the indices of the training records, which
the library allocates in a canonical order (tile order per path vertex) instead of the reference's atomicAdd.
The network is then run on the GPU, its predictions are handed to the oracle, and accumulate / propagate /
shuffle are compared bit for bit again."""
import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import nrc_records

pytestmark = pytest.mark.gpu


def _same(got, want, tag):
    g, w = np.ascontiguousarray(got), np.ascontiguousarray(want)
    g = g.view(np.uint32) if g.dtype.itemsize == 4 else g
    w = w.view(np.uint32) if w.dtype.itemsize == 4 else w
    if not np.array_equal(g, w):
        bad = np.argwhere(g != w)
        raise AssertionError(f"{tag}: {len(bad)} elements differ, first {bad[:4].tolist()}: "
                             f"{got[tuple(bad[0])]} vs {want[tuple(bad[0])]}")


def _compare_pathtrace(ctx, oframe, p, tag):
    w, h = oframe.W, oframe.H
    n = w * h
    _same(ctx.download(abi.BUF_RNG), oframe.buffer(abi.BUF_RNG), f"{tag} rng")
    st_g = ctx.download_linear(abi.BUF_NRC_STATE)[:, 0]
    st_o = oframe.linear_buffer(abi.BUF_NRC_STATE)[:, 0]
    _same(st_g[:8], st_o[:8], f"{tag} state (numTrainingData, tileSize, offsets)")
    assert st_g[abi.NRC_STATE_NUM_INFERENCE_QUERIES] == st_o[abi.NRC_STATE_NUM_INFERENCE_QUERIES]
    ntrain = min(int(st_o[p.bufferIndex]), abi.NRC_TRAIN_BUFFER_SIZE)
    assert ntrain > 0
    _same(ctx.download_linear(abi.BUF_NRC_FRAME_CONTRIBUTION), oframe.linear_buffer(abi.BUF_NRC_FRAME_CONTRIBUTION), f"{tag} contribution")
    ti_g = ctx.download_linear(abi.BUF_NRC_TERMINAL_INFO)
    ti_o = oframe.linear_buffer(abi.BUF_NRC_TERMINAL_INFO)
    _same(ti_g, ti_o, f"{tag} terminal info")
    _same(ctx.download_linear(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL), oframe.linear_buffer(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL), f"{tag} suffix terminals")
    _same(ctx.download_linear(abi.BUF_NRC_TRAIN_VERTEX_INFO)[:ntrain], oframe.linear_buffer(abi.BUF_NRC_TRAIN_VERTEX_INFO)[:ntrain], f"{tag} vertex infos")
    _same(ctx.download_linear(abi.BUF_NRC_TRAIN_QUERY, 0)[:ntrain], oframe.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 0)[:ntrain], f"{tag} train queries")
    _same(ctx.download_linear(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain], oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain], f"{tag} train targets")
    # inference queries: only rows that were written this frame are defined
    q_g = ctx.download_linear(abi.BUF_NRC_INFERENCE_QUERY)
    q_o = oframe.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)
    has_query = (ti_o[:, 3] & 1).astype(bool)
    _same(q_g[:n][has_query], q_o[:n][has_query], f"{tag} pixel queries")
    suffix = oframe.linear_buffer(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL)[:, 0]
    suffix_query = ((suffix >> 23) & 1).astype(bool)
    _same(q_g[n:n + len(suffix)][suffix_query], q_o[n:n + len(suffix)][suffix_query], f"{tag} suffix queries")
    return ntrain, has_query, suffix_query


@pytest.mark.parametrize("max_path_length,scene_name", [(5, "small_city_scene"), (0, "small_city_scene"), (5, "small_interior_scene"),
                                                        (5, "small_city_scene_env"), (5, "small_city_scene_textured")])
def test_nrc_frames_bit_exact(gfx_ctx, oracle, max_path_length, scene_name):
    scene = getattr(scenes, scene_name)()
    w, h = 192, 108
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    gfx_ctx.build_light_distributions(0)
    oscene = oracle.OracleScene(scene)
    oframe = oracle.OracleFrame(oscene, w, h)
    net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    onet = oracle.OracleNrc(2, 1e-2)
    params = engine.random_nrc_params(net.num_params, onet.num_matrix_weights, grid_amplitude=0.1)
    net.set_params(params)
    onet.set_params(params)
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = max_path_length
    p.radianceScale = 2.0
    rng = np.random.default_rng(7)
    n = w * h
    for frame in range(3):
        p.frameIndex, p.bufferIndex, p.numAccumFrames = frame, frame % 2, frame
        offsets = [int(rng.integers(0, 2 ** 32)) for _ in range(2)]
        # --- path tracer
        gfx_ctx.gbuffer(p)
        gfx_ctx.nrc_preprocess(p, offsets[0], offsets[1], frame == 0)
        gfx_ctx.pathtrace(p, abi.PT_NRC)
        oframe.gbuffer(p)
        oframe.nrc_preprocess(p, offsets[0], offsets[1], frame == 0)
        oframe.pathtrace(p, abi.PT_NRC)
        ntrain, has_query, suffix_query = _compare_pathtrace(gfx_ctx, oframe, p, f"frame {frame}")
        assert has_query.mean() > 0.3

        # --- inference: wgmma MLP vs the oracle network on the real queries (tolerance of the fp16 path)
        gfx_ctx.nrc_frame_infer(net)
        pred = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
        q = oframe.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)
        rows = np.concatenate([np.flatnonzero(has_query), n + np.flatnonzero(suffix_query)])
        want = onet.infer(q[rows])
        rel = np.linalg.norm(pred[rows] - want) / max(np.linalg.norm(want), 1e-12)
        assert rel <= 1e-3, rel
        # the oracle continues from the GPU's predictions
        oframe.linear_buffer(abi.BUF_NRC_INFERRED_RADIANCE, copy=False)[:] = pred

        # --- accumulate / propagate / shuffle
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
        st_g = gfx_ctx.download_linear(abi.BUF_NRC_STATE)[:, 0]
        st_o = oframe.linear_buffer(abi.BUF_NRC_STATE)[:, 0]
        _same(st_g[8:20], st_o[8:20], f"frame {frame} target min/max")
        # targetAvg is a float-atomic sum in the reference (no defined order): tolerance
        np.testing.assert_allclose(st_g[20:26].view(np.float32), st_o[20:26].view(np.float32), rtol=1e-4, atol=1e-7)

        # --- training on the shuffled records (both sides the same data)
        loss = gfx_ctx.nrc_frame_train(net, want_loss=True)
        oloss = None
        for step in range(4):
            sl = slice(step * 16384, (step + 1) * 16384)
            oloss = onet.train(tq_g[sl], tt_g[sl])
        assert np.isfinite(loss) and abs(loss - oloss) <= 0.05 * abs(oloss) + 1e-4, (loss, oloss)
    net.close()


def _seeded_preprocess(gfx_ctx, p, tile, offsets):
    """the NRC preprocess of a new sequence (tile 8), or with `tile` seeded as the previous frame's tile size"""
    if tile is not None:
        st = gfx_ctx.download_linear(abi.BUF_NRC_STATE)
        gfx_ctx.upload(abi.BUF_NRC_STATE, 0, nrc_records.seeded_state(st, p.bufferIndex, tile))
    gfx_ctx.nrc_preprocess(p, offsets[0], offsets[1], tile is None)


# 4K with 4x4 tiles has every suffix slot in use: 3840 * 2160 + 518 400 = 8 812 800 queries
SEEDED_TILE = {(3840, 2160): 4}


@pytest.mark.parametrize("w,h,strips", [(192, 108, [(0, 34), (34, 80), (80, 108)]),
                                         (1920, 1080, [(0, 360), (360, 1001), (1001, 1080)]),
                                         (3840, 2160, [(0, 720), (720, 2002), (2002, 2160)])])
def test_frame_inference_matches_direct_inference(gfx_ctx, w, h, strips):
    """gfx_nrc_frame_infer infers as many queries as the device-side count in the state block says (pixels + training-suffix
    slots, padded to the 128-query tile) and leaves the rows beyond it alone; its predictions are the bits gfx_nrc_infer gives
    the same queries in launches of one tile per CTA.  gfx_nrc_frame_infer_rows (one strip of rows of a frame split across GPUs)
    gives the same bits on the strip's pixel rows and on every suffix query, and writes nothing else."""
    import torch
    scene = scenes.small_city_scene()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    gfx_ctx.build_light_distributions(0)
    net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    net.set_params(engine.random_nrc_params(net.num_params, 64 * 64 * 2 + 16 * 64, seed=19, grid_amplitude=0.1))
    p = abi.default_frame_params(scene, w, h)
    tile = SEEDED_TILE.get((w, h))
    gfx_ctx.gbuffer(p)
    _seeded_preprocess(gfx_ctx, p, tile, (0x2545F491, 0x9E3779B9))
    gfx_ctx.pathtrace(p, abi.PT_NRC)
    n, capacity = w * h, abi.nrc_query_capacity(w, h)
    sentinel = np.full((capacity, 3), 0x7FC0DEAD, dtype=np.uint32).view(np.float32)  # a NaN no kernel produces

    gfx_ctx.upload(abi.BUF_NRC_INFERRED_RADIANCE, 0, sentinel)
    gfx_ctx.nrc_frame_infer(net)
    frame = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
    st = gfx_ctx.download_linear(abi.BUF_NRC_STATE)[:, 0]
    count, num_suffix = int(st[abi.NRC_STATE_NUM_INFERENCE_QUERIES]), int(st[abi.NRC_STATE_NUM_SUFFIX_QUERIES])
    assert count % 128 == 0 and n < count <= capacity and count == n + num_suffix, (count, num_suffix, capacity)
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
    _same(frame[:count], direct.cpu().numpy(), "frame inference vs gfx_nrc_infer in single-wave launches")

    for lo, hi in strips:
        gfx_ctx.upload(abi.BUF_NRC_INFERRED_RADIANCE, 0, sentinel)
        gfx_ctx._check(gfx_ctx.lib.gfx_nrc_frame_infer_rows(gfx_ctx.h, net.h, None, lo, hi), "gfx_nrc_frame_infer_rows")
        got = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
        first, end = lo * w, lo * w + ((hi - lo) * w + 127) // 128 * 128  # the strip's pixels, padded to whole tiles
        _same(got[first:hi * w], frame[first:hi * w], f"rows {lo}..{hi}: pixel queries")
        _same(got[n:n + num_suffix], frame[n:n + num_suffix], f"rows {lo}..{hi}: suffix queries")
        _same(got[:first], sentinel[:first], f"rows {lo}..{hi}: pixels before the strip")
        _same(got[end:n], sentinel[end:n], f"rows {lo}..{hi}: pixels after the strip")
        _same(got[n + num_suffix:], sentinel[n + num_suffix:], f"rows {lo}..{hi}: beyond the suffix queries")
    net.close()


def test_nrc_frame_wrapper_and_tile_controller(gfx_ctx):
    """the one-call frame (no host read-backs) keeps the training-record count near 65 536 * (tile area ratio)
    and produces a finite image"""
    scene = scenes.small_city_scene()
    w, h = 320, 180
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    gfx_ctx.build_light_distributions(0)
    net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    net.set_params(engine.random_nrc_params(net.num_params, 64 * 64 * 2 + 16 * 64, grid_amplitude=0.1))
    p = abi.default_frame_params(scene, w, h)
    rng = np.random.default_rng(3)
    losses = []
    for frame in range(8):
        p.numAccumFrames = frame
        losses.append(gfx_ctx.nrc_frame(net, p, frame, [int(rng.integers(0, 2 ** 32)) for _ in range(2)], train=True, want_loss=True))
    st = gfx_ctx.download_linear(abi.BUF_NRC_STATE)[:, 0]
    tile = st[abi.NRC_STATE_TILE_SIZE + 2 * (7 % 2)]
    assert tile == 4  # a 320x180 frame cannot reach 65 536 records even with the smallest tiles
    assert st[7 % 2] > 320 * 180 // 16
    beauty = gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)[..., :3]
    assert np.isfinite(beauty).all() and beauty.mean() > 1e-3
    assert all(np.isfinite(l) for l in losses)
    net.close()
