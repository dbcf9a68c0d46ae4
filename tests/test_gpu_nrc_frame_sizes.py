"""GPU parity of the NRC frame at the sizes it ships at (1080p, and 3840x2160 as in bench.py's config 5), where its control flow
differs from the 192x108 frames of test_gpu_nrc_frame.py: the training buffer of 131 072 records overflows (a ray-gen vertex past
it starts no chain, a bounce vertex past it ends its suffix with a query), k_nrcCommitScan numbers a chunk of tiles per thread,
and the tile-size controller gives sizes that are not powers of two or hits its clamp.  Every frame is compared with the CPU
oracle bit for bit as in test_nrc_frames_bit_exact, its records are checked against the chain rules of tests/nrc_records.py,
and every case asserts that the branch it targets ran."""
import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import nrc_records
from tests.test_gpu_nrc_frame import _compare_pathtrace, _same

pytestmark = pytest.mark.gpu

BUF = abi.NRC_TRAIN_BUFFER_SIZE

# case: scene, W, H, one seed per frame: None lets the controller act (a new sequence on frame 0), (tile, count) writes the
# previous buffer's tile size and record count first, which the controller turns into clamp(tile * sqrt(count / 65536), 4, 128)
CASES = {
    "1080p": ("small_city_scene", 1920, 1080, [None, None, None]),
    "4k": ("small_city_scene", 3840, 2160, [None, None, None]),
    "1080p_tile4": ("small_city_scene", 1920, 1080, [(4, 65536)]),
    "4k_tile5_then_controller": ("small_city_scene", 3840, 2160, [(5, 65536), None]),
    "ragged_tile4": ("small_city_scene", 1283, 721, [(4, 65536)]),
    "ragged_clamped_to_128": ("small_city_scene", 1283, 721, [(100, 4 * 65536)]),
    "env_1080p": ("small_city_scene_env", 1920, 1080, [None, None, None]),
}


@pytest.fixture(scope="module")
def oracle_scenes(oracle):
    built = {}

    def get(name):
        if name not in built:
            built[name] = oracle.OracleScene(getattr(scenes, name)())
        return built[name]
    return get


def _frames(gfx_ctx, oracle, oscene, scene, w, h, seeds):
    """runs the frames of a case on both sides, compares them, and returns per frame the record summary of the GPU's buffers
    and the pixels whose training path found no primary hit"""
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    gfx_ctx.build_light_distributions(0)
    oframe = oracle.OracleFrame(oscene, w, h)
    net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    onet = oracle.OracleNrc(2, 1e-2)
    params = engine.random_nrc_params(net.num_params, onet.num_matrix_weights, grid_amplitude=0.1)
    net.set_params(params)
    onet.set_params(params)
    p = abi.default_frame_params(scene, w, h)
    p.radianceScale = 2.0
    rng = np.random.default_rng(11)
    n = w * h
    out = []
    for frame, seed in enumerate(seeds):
        tag = f"{w}x{h} frame {frame}"
        p.frameIndex, p.bufferIndex, p.numAccumFrames = frame, frame % 2, frame
        offsets = [int(rng.integers(0, 2 ** 32)) for _ in range(2)]
        gfx_ctx.gbuffer(p)
        oframe.gbuffer(p)
        if seed is not None:
            st = oframe.linear_buffer(abi.BUF_NRC_STATE, copy=False)
            st[:] = nrc_records.seeded_state(st, p.bufferIndex, seed[0], seed[1])
            gfx_ctx.upload(abi.BUF_NRC_STATE, 0, st)
        new_sequence = frame == 0 and seed is None
        gfx_ctx.nrc_preprocess(p, offsets[0], offsets[1], new_sequence)
        gfx_ctx.pathtrace(p, abi.PT_NRC)
        oframe.nrc_preprocess(p, offsets[0], offsets[1], new_sequence)
        oframe.pathtrace(p, abi.PT_NRC)
        ntrain, has_query, suffix_query = _compare_pathtrace(gfx_ctx, oframe, p, tag)
        hit = gfx_ctx.download(abi.BUF_GBUFFER0, p.bufferIndex)[..., 0] != 0xFFFFFFFF
        state = gfx_ctx.download_linear(abi.BUF_NRC_STATE)[:, 0]
        rec = nrc_records.check_records(gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_VERTEX_INFO),
                                        gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL), state, p.bufferIndex, hit)
        is_train, _ = nrc_records.training_pixels(state, p.bufferIndex, w, h)
        rec["missed_training_pixels"] = int((is_train & ~hit).sum())
        out.append(rec)

        gfx_ctx.nrc_frame_infer(net)
        pred = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
        q = oframe.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)
        rows = np.concatenate([np.flatnonzero(has_query), n + np.flatnonzero(suffix_query)])
        want = onet.infer(q[rows])
        rel = np.linalg.norm(pred[rows] - want) / max(np.linalg.norm(want), 1e-12)
        assert rel <= 1e-3, (tag, rel)
        oframe.linear_buffer(abi.BUF_NRC_INFERRED_RADIANCE, copy=False)[:] = pred

        gfx_ctx.nrc_accumulate(p)
        oframe.nrc_accumulate(p)
        _same(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), oframe.buffer(abi.BUF_BEAUTY_ACCUM), f"{tag} beauty")
        gfx_ctx.nrc_propagate(p)
        oframe.nrc_propagate(p)
        _same(gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain], oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain],
              f"{tag} propagated targets")
        gfx_ctx.nrc_shuffle(p)
        oframe.nrc_shuffle(p)
        tq_g, tt_g = gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_QUERY, 1), gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_TARGET, 1)
        m = abi.NRC_TRAINING_DATA_PER_FRAME
        _same(tq_g[:m], oframe.linear_buffer(abi.BUF_NRC_TRAIN_QUERY, 1)[:m], f"{tag} shuffled queries")
        _same(tt_g[:m], oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 1)[:m], f"{tag} shuffled targets")
        st_g = gfx_ctx.download_linear(abi.BUF_NRC_STATE)[:, 0]
        st_o = oframe.linear_buffer(abi.BUF_NRC_STATE)[:, 0]
        _same(st_g[:20], st_o[:20], f"{tag} state words 0..19")
        np.testing.assert_allclose(st_g[20:26].view(np.float32), st_o[20:26].view(np.float32), rtol=1e-4, atol=1e-7)

        loss = gfx_ctx.nrc_frame_train(net, want_loss=True)
        oloss = None
        for step in range(4):
            sl = slice(step * 16384, (step + 1) * 16384)
            oloss = onet.train(tq_g[sl], tt_g[sl])
        assert np.isfinite(loss) and abs(loss - oloss) <= 0.05 * abs(oloss) + 1e-4, (tag, loss, oloss)
    net.close()
    onet.close()
    oframe.close()
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_nrc_frames_at_frame_size(gfx_ctx, oracle, oracle_scenes, case):
    scene_name, w, h, seeds = CASES[case]
    r = _frames(gfx_ctx, oracle, oracle_scenes(scene_name), getattr(scenes, scene_name)(), w, h, seeds)
    tiles = [x["tile_size"][0] for x in r]
    assert all(x["tile_size"][0] == x["tile_size"][1] for x in r)
    if case != "ragged_clamped_to_128":  # more tiles than the commit scan's 1024 threads: each thread numbers a chunk
        assert all(x["num_tiles"] > 1024 for x in r), [x["num_tiles"] for x in r]
    if case == "1080p":
        assert tiles == [8, 7, 7], tiles            # ragged: 1920 % 7 = 2, 1080 % 7 = 2
        assert all(0 < x["num_training_data"] < BUF for x in r)
    elif case == "4k":
        assert tiles == [8, 14, 14], tiles
        assert r[0]["num_training_data"] > BUF and r[0]["bounce_vertices_past_buffer"] > 50000, r[0]
        assert r[0]["query_terminals"] > 50000 and r[0]["chainless_tiles"] == 0, r[0]
    elif case == "1080p_tile4":
        assert tiles == [4]
        assert r[0]["num_training_data"] > BUF and r[0]["bounce_vertices_past_buffer"] > 50000, r[0]
    elif case == "4k_tile5_then_controller":
        assert r[0]["hit_training_tiles"] > BUF, r[0]
        assert r[0]["chainless_tiles"] == r[0]["hit_training_tiles"] - BUF > 100000, r[0]
        assert r[0]["bounce_vertices_past_buffer"] > 0, r[0]
        # the controller acts on a count far past the buffer
        assert r[0]["num_training_data"] > 4 * BUF
        assert tiles[1] == int(5 * np.sqrt(r[0]["num_training_data"] / 65536)) > 8, (tiles, r[0])
    elif case == "ragged_tile4":
        assert tiles == [4] and r[0]["num_tiles"] == 321 * 181   # W % 4 = 3, H % 4 = 1
    elif case == "ragged_clamped_to_128":
        assert tiles == [128] and r[0]["num_tiles"] == 11 * 6    # 100 * sqrt(4) = 200, clamped
    elif case == "env_1080p":
        assert tiles[0] == 8
        assert all(x["missed_training_pixels"] > 100 for x in r), [x["missed_training_pixels"] for x in r]
