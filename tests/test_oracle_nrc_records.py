"""The oracle's NRC training records obey the chain rules of tests/nrc_records.py at frame sizes where the training buffer
overflows: a GPU mismatch at those sizes can then be blamed on the right side.  Tile sizes are seeded through the state block
(the previous buffer's record count and tile size), so each case reaches its branch in one frame."""
import numpy as np
import pytest

from gfxexp_b200 import abi, scenes
from tests import nrc_records

OFFSETS = (0x2545F491, 0x9E3779B9)


@pytest.fixture(scope="module")
def city(oracle):
    scene = scenes.small_city_scene()
    return scene, oracle.OracleScene(scene)


def _records(oracle, city, w, h, tile, frames=1):
    """path-traces `frames` frames of a new sequence, the first seeded to `tile` unless it is None; checks and returns the
    records of every frame"""
    scene, oscene = city
    oframe = oracle.OracleFrame(oscene, w, h)
    p = abi.default_frame_params(scene, w, h)
    out = []
    for frame in range(frames):
        p.frameIndex, p.bufferIndex = frame + 1, (frame + 1) % 2
        oframe.gbuffer(p)
        if frame == 0 and tile is not None:
            st = oframe.linear_buffer(abi.BUF_NRC_STATE, copy=False)
            st[:] = nrc_records.seeded_state(st, p.bufferIndex, tile)
        oframe.nrc_preprocess(p, OFFSETS[0] + frame, OFFSETS[1] + frame, frame == 0 and tile is None)
        oframe.pathtrace(p, abi.PT_NRC)
        hit = oframe.buffer(abi.BUF_GBUFFER0, p.bufferIndex)[..., 0] != 0xFFFFFFFF
        out.append(nrc_records.check_records(oframe.linear_buffer(abi.BUF_NRC_TRAIN_VERTEX_INFO),
                                             oframe.linear_buffer(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL),
                                             oframe.linear_buffer(abi.BUF_NRC_STATE)[:, 0], p.bufferIndex, hit))
    return out


def test_records_of_a_small_frame(oracle, city):
    """192x108 from a new sequence: tile 8, then the controller's 4; nothing overflows"""
    r = _records(oracle, city, 192, 108, None, frames=3)
    assert [x["tile_size"] for x in r] == [(8, 8), (4, 4), (4, 4)]
    assert all(0 < x["num_training_data"] < abi.NRC_TRAIN_BUFFER_SIZE for x in r)
    assert all(x["chainless_tiles"] == 0 and x["bounce_vertices_past_buffer"] == 0 for x in r)


def test_records_at_1080p_with_4x4_tiles(oracle, city):
    """129 600 tiles fit the ray-gen vertices, but bounce vertices run past the buffer and end their suffix with a query"""
    (r,) = _records(oracle, city, 1920, 1080, 4)
    assert r["tile_size"] == (4, 4) and r["num_tiles"] == 129600
    assert r["num_training_data"] > 200000, r
    assert r["chainless_tiles"] == 0 and r["bounce_vertices_past_buffer"] > 50000, r


def test_records_at_4k_with_5x5_tiles(oracle, city):
    """331 776 tiles: more hit training tiles than records, so the ones after the first 131 072 in tile order start no chain"""
    (r,) = _records(oracle, city, 3840, 2160, 5)
    assert r["tile_size"] == (5, 5) and r["hit_training_tiles"] > abi.NRC_TRAIN_BUFFER_SIZE, r
    assert r["chainless_tiles"] == r["hit_training_tiles"] - abi.NRC_TRAIN_BUFFER_SIZE > 100000, r
    assert r["num_training_data"] > 500000 and r["bounce_vertices_past_buffer"] > 0, r


def test_records_of_a_ragged_frame(oracle, city):
    """1283x721 with 7x7 tiles: the right column of tiles is 2 pixels wide, W % 4 = 3 and H % 4 = 1"""
    (r,) = _records(oracle, city, 1283, 721, 7)
    assert r["tile_size"] == (7, 7) and r["num_tiles"] == 184 * 103
    assert 0 < r["num_training_data"] < abi.NRC_TRAIN_BUFFER_SIZE, r


def test_record_rules_catch_a_record_on_no_chain(oracle, city):
    """the checker itself: a terminal that loses its chain, a prev that skips a vertex, two records swapped each fail"""
    scene, oscene = city
    w, h = 192, 108
    oframe = oracle.OracleFrame(oscene, w, h)
    p = abi.default_frame_params(scene, w, h)
    oframe.gbuffer(p)
    oframe.nrc_preprocess(p, *OFFSETS, True)
    oframe.pathtrace(p, abi.PT_NRC)
    vi = oframe.linear_buffer(abi.BUF_NRC_TRAIN_VERTEX_INFO)
    st = oframe.linear_buffer(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL)[:, 0]
    state = oframe.linear_buffer(abi.BUF_NRC_STATE)[:, 0]
    hit = oframe.buffer(abi.BUF_GBUFFER0, 0)[..., 0] != 0xFFFFFFFF
    r = nrc_records.check_records(vi, st, state, 0, hit)
    assert r["num_training_data"] > 100
    tile = int(np.flatnonzero((st & nrc_records.INVALID) != nrc_records.INVALID)[0])
    cut = st.copy()
    cut[tile] |= nrc_records.INVALID
    with pytest.raises(AssertionError, match="not 1"):
        nrc_records.check_records(vi, cut, state, 0, hit)
    n = min(int(state[0]), abi.NRC_TRAIN_BUFFER_SIZE)
    prev, plen = vi[:n, 3] & nrc_records.INVALID, vi[:n, 3] >> 23
    skip = vi.copy()
    rec = int(np.flatnonzero(plen == 3)[0])
    skip[rec, 3] = (3 << 23) | prev[prev[rec]]
    with pytest.raises(AssertionError, match="path length"):
        nrc_records.check_records(skip, st, state, 0, hit)
    swapped = vi.copy()
    a, b = np.flatnonzero(plen == 2)[[0, -1]]
    swapped[a, 3], swapped[b, 3] = vi[b, 3], vi[a, 3]
    with pytest.raises(AssertionError, match="order"):
        nrc_records.check_records(swapped, st, state, 0, hit)
