"""The rules every NRC frame's training records obey, checked with numpy on the buffers the path tracer wrote (oracle or GPU).

Records are numbered in the canonical order "path vertex first, tile second" (oracle/nrc_pathtrace.inl header): the ray-gen
round commits first, in tile order, so once the buffer of NRC_TRAIN_BUFFER_SIZE records is full, the hit training tiles after
the first NRC_TRAIN_BUFFER_SIZE in tile order start no chain, and a bounce vertex past the buffer ends its suffix with a query.
"""
import numpy as np

from gfxexp_b200 import abi

INVALID = 0x7FFFFF  # kInvalidVertexDataIndex: the 23-bit prev field of a chain's first record or an empty terminal


def seeded_state(state, buffer_index, tile_size, num_training_data=abi.NRC_TRAINING_DATA_PER_FRAME):
    """the state words with the previous buffer's record count and tile size set, so that the next preprocess of buffer
    `buffer_index` with new_sequence=False gives clamp(tile_size * sqrt(num_training_data / 65536), 4, 128): tile_size itself
    with the default count"""
    s = np.array(state, dtype=np.uint32).reshape(32, 1)
    prev = (buffer_index + 1) % 2
    s[abi.NRC_STATE_NUM_TRAINING_DATA + prev] = num_training_data
    s[abi.NRC_STATE_TILE_SIZE + 2 * prev:abi.NRC_STATE_TILE_SIZE + 2 * prev + 2] = tile_size
    return s


def training_pixels(state, buffer_index, w, h):
    """[h, w] bool: the one pixel per tile that traces the training path, and the linear tile index of every pixel"""
    tsx, tsy = (int(v) for v in state[abi.NRC_STATE_TILE_SIZE + 2 * buffer_index:abi.NRC_STATE_TILE_SIZE + 2 * buffer_index + 2])
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    local = (y % tsy) * tsx + (x % tsx)
    is_train = (local + int(state[abi.NRC_STATE_OFFSET_TRAINING_PATH])) % (tsx * tsy) == 0
    tile = (y // tsy) * ((w + tsx - 1) // tsx) + x // tsx
    return is_train, tile


def check_records(vertex_info, suffix_terminal, state, buffer_index, primary_hit):
    """Asserts the record invariants of one path-traced frame and returns what the frame reached.

    vertex_info: BUF_NRC_TRAIN_VERTEX_INFO [NRC_TRAIN_BUFFER_SIZE, 4] uint32; suffix_terminal: BUF_NRC_TRAIN_SUFFIX_TERMINAL;
    state: BUF_NRC_STATE words; primary_hit: [H, W] bool, the G-buffer of buffer_index has a hit.
    - every prev index is smaller than its record's index;
    - along a chain the path length grows by exactly 1, and every chain starts at path length 1;
    - the chains that end in the suffix terminals partition [0, min(N, NRC_TRAIN_BUFFER_SIZE)): every record lies on one;
    - record indices are sorted by (path length, tile);
    - no terminal or prev points at or past min(N, NRC_TRAIN_BUFFER_SIZE), and the ray-gen records are the first hit training
      tiles in tile order: the hit training tiles after the first NRC_TRAIN_BUFFER_SIZE start no chain."""
    b = buffer_index
    h, w = primary_hit.shape
    state = np.asarray(state).reshape(-1)
    n = int(state[abi.NRC_STATE_NUM_TRAINING_DATA + b])
    m = min(n, abi.NRC_TRAIN_BUFFER_SIZE)
    tsx, tsy = int(state[abi.NRC_STATE_TILE_SIZE + 2 * b]), int(state[abi.NRC_STATE_TILE_SIZE + 2 * b + 1])
    num_tiles = ((w + tsx - 1) // tsx) * ((h + tsy - 1) // tsy)

    vi = np.asarray(vertex_info)[:m, 3].astype(np.int64)
    prev, plen = vi & INVALID, vi >> 23
    idx = np.arange(m)
    linked = prev != INVALID
    bad = np.flatnonzero(linked & (prev >= idx))
    assert not len(bad), f"records {bad[:4].tolist()} point at prev {prev[bad[:4]].tolist()}: not an earlier record"
    bad = np.flatnonzero(~linked & (plen != 1))
    assert not len(bad), f"records {bad[:4].tolist()} start a chain at path length {plen[bad[:4]].tolist()}, not 1"
    bad = np.flatnonzero(linked & (plen != plen[np.where(linked, prev, 0)] + 1))
    assert not len(bad), f"records {bad[:4].tolist()}: path length {plen[bad[:4]].tolist()} after {plen[prev[bad[:4]]].tolist()}"

    st = np.asarray(suffix_terminal).reshape(-1).astype(np.int64)
    assert (st[num_tiles:] == INVALID).all(), "a terminal slot beyond this frame's tiles was written"
    st = st[:num_tiles]
    tprev, tquery, tlen = st & INVALID, (st >> 23) & 1, st >> 24
    tlinked = tprev != INVALID
    bad = np.flatnonzero(tlinked & (tprev >= m))
    assert not len(bad), f"terminals of tiles {bad[:4].tolist()} point at {tprev[bad[:4]].tolist()}, past the {m} records"
    safe = np.where(tlinked, np.minimum(tprev, max(m - 1, 0)), 0)
    last = plen[safe] if m else np.zeros_like(tprev)
    bad = np.flatnonzero(tlinked & (tquery == 1) & (tlen != last + 1))
    assert not len(bad), f"query terminals of tiles {bad[:4].tolist()}: path length {tlen[bad[:4]].tolist()} after {last[bad[:4]].tolist()}"
    bad = np.flatnonzero(tlinked & (tlen < last))
    assert not len(bad), f"terminals of tiles {bad[:4].tolist()} end before their last record"

    refs = np.bincount(prev[linked], minlength=m) + np.bincount(tprev[tlinked], minlength=m)
    bad = np.flatnonzero(refs != 1)
    assert not len(bad), f"records {bad[:4].tolist()} are followed by {refs[bad[:4]].tolist()} records or terminals, not 1"

    # the tile of every record, from its chain's terminal back (a record's successor has the next path length)
    tile = np.full(m, -1, dtype=np.int64)
    tile[tprev[tlinked]] = np.flatnonzero(tlinked)
    for length in range(int(plen.max()) if m else 0, 1, -1):
        r = np.flatnonzero(plen == length)
        tile[prev[r]] = tile[r]
    key = plen * num_tiles + tile
    bad = np.flatnonzero(np.diff(key) <= 0)
    assert not len(bad), (f"records {bad[:4].tolist()} and their successors are out of (path length, tile) order: "
                          f"{[(int(plen[i]), int(tile[i]), int(plen[i + 1]), int(tile[i + 1])) for i in bad[:4]]}")

    is_train, pixel_tile = training_pixels(state, b, w, h)
    hit_tiles = np.sort(pixel_tile[is_train & primary_hit])
    assert np.array_equal(tile[plen == 1], hit_tiles[:abi.NRC_TRAIN_BUFFER_SIZE]), "ray-gen records are not the first hit training tiles"
    chainless = hit_tiles[~tlinked[hit_tiles]]
    assert np.array_equal(chainless, hit_tiles[abi.NRC_TRAIN_BUFFER_SIZE:]), \
        f"{len(chainless)} hit training tiles start no chain, want the {max(len(hit_tiles) - abi.NRC_TRAIN_BUFFER_SIZE, 0)} past the buffer"
    others = np.ones(num_tiles, dtype=bool)
    others[hit_tiles] = False
    assert (st[others] == INVALID).all(), "a tile without a hit training pixel has a terminal"
    # the ray-gen vertices are numbers 0 .. hit tiles - 1, so the bounce vertices numbered past the buffer are the rest
    return dict(num_training_data=n, tile_size=(tsx, tsy), num_tiles=num_tiles, hit_training_tiles=len(hit_tiles),
                chainless_tiles=len(chainless), query_terminals=int(tquery.sum()),
                bounce_vertices_past_buffer=max(n - max(len(hit_tiles), abi.NRC_TRAIN_BUFFER_SIZE), 0))
