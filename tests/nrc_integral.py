"""The NRC path tracer against a closed form - TEST INFRASTRUCTURE shared by tests/test_oracle_nrc_integral.py (CPU oracle)
and tests/test_gpu_nrc_integral.py (library).

A closed box seen from inside: every face an inward-facing Lambertian emitter of emitted radiance e (emittance / pi, as the
path tracers convert it) and albedo rho_c.  The radiance leaving every point in every direction is L_c = e / (1 - rho_c), the
scattered part rho_c L_c.  A network whose output is the constant radianceScale * L_c is an exact cache: accumulate and
propagate divide by radianceScale and multiply by the query's diffuse + specularF0 = rho_c + 0 (Lambert has F0 = 0), which
gives rho_c L_c, the scattered radiance at the terminal vertex.  With that cache every estimator branch of the NRC frame -
Russian roulette, the spread heuristic's cache termination, unbiased tiles, the buffer-full suffix query, a training suffix's
cache query, NEE + BSDF sampling with MIS at every vertex - has expectation L, so a wrong weight in any branch is a bias
against one known number.  Paths are cut at 62 rounds (kMaxNrcRounds): with rho <= 0.75 what that drops is below
0.75^61 ~ 2.4e-8 of L, far inside the float32 slack below.

Grouping rule: results are grouped only by facts decided before the random draws that follow them - per pixel whether it
traces the tile's training path and whether its tile is unbiased (both in the terminal info, set from the frame's offsets
before any draw); per training record its path length and its tile's class.  Grouping by an outcome - the terminal's
hasQuery or path length, a suffix's hasQuery - conditions on the sampled distances (the spread heuristic) and on the MIS
weights, and such groups have biased means even for a correct estimator.

Standard errors take the tile as the independent unit for records (the records of one chain are correlated) and the pixel
for pixels (each pixel has its own RNG stream).  Every mean must equal L within 5 SE + SLACK * L."""
from __future__ import annotations

import math

import numpy as np

from gfxexp_b200 import abi, scenes

F32 = np.float32
RHO = np.array([0.5, 0.75, 0.5], dtype=F32)
EMITTANCE = F32(math.pi * 0.25)               # e = emittance / pi = 0.25 up to float32 rounding
E = float(F32(EMITTANCE / F32(math.pi)))       # the emitted radiance as the path tracers compute it, in float32
L = E / (1.0 - RHO.astype(np.float64))        # (0.5, 1, 0.5)
RADIANCE_SCALE = 2.0
# float32 slack, relative to L: a path of up to ~60 vertices rounds a few operations per vertex (2^-24 each), MIS weights
# pow2(a) / (pow2(a) + pow2(b)) are float32 and their NEE + implicit pair sums to 1 only to a few ulps, and e itself is float32.
# 1e-4 bounds all of it with a wide margin; it is more than 100 times smaller than the biases the negative controls show.
SLACK = 1e-4
NSE = 5.0


def emissive_box_scene(size=(4.0, 3.0, 6.0), tess: int = 2) -> scenes.Scene:
    """scenes.make_box turned inside out (winding and normals reversed, so its faces face inwards), one emissive Lambertian
    material, the camera inside looking towards a corner so that the view sees four faces at grazing to normal incidence"""
    mats = np.zeros(1, dtype=scenes.MATERIAL_DTYPE)
    mats[0]["bsdfType"] = scenes.BSDF_LAMBERT
    mats[0]["p0"] = RHO
    mats[0]["emittance"] = EMITTANCE
    mats[0]["hasEmittance"] = 1
    box = scenes.make_box(tess, size, 0)
    box.triangles = np.ascontiguousarray(box.triangles[:, ::-1])
    box.normals = np.ascontiguousarray(-box.normals)
    eye = np.array([0.4, 1.3, -1.2])
    orientation = scenes.look_at_orientation(eye, (1.7, 2.4, 2.9))
    return scenes.Scene([box], mats, [scenes.make_instance([0])], eye.astype(F32), orientation, math.radians(80.0),
                        "emissive_box")


def truncated_series(n: int) -> np.ndarray:
    """e * sum_{k < n} rho^k: the baseline path tracer at maxPathLength n (the primary vertex's emission is k = 0, the light
    after k scatterings is term k, the last one the NEE + implicit hit of vertex n - 1)"""
    rho = RHO.astype(np.float64)
    return E * (1.0 - rho ** n) / (1.0 - rho)


def constant_params(num_params: int, num_matrix_weights: int, num_hidden_layers: int, value) -> np.ndarray:
    """fp16 parameters, in the layout of engine.random_nrc_params / OracleNrc (matrices [out][in] in layer order, then the
    hash-grid table), of a network that outputs `value` for every query: the first layer reads features 62 and 63, which are
    ones in both position encodings, with weight 1/2 each, so hidden neuron 0 is 1 through every ReLU layer and the rest are
    0; output row c is value[c], rounded to half, on neuron 0.  Every grid entry is 0."""
    p = np.zeros(num_params, dtype=np.float16)
    p[62] = p[63] = 0.5
    for layer in range(1, num_hidden_layers):
        p[layer * 64 * 64] = 1.0
    out = num_hidden_layers * 64 * 64
    for c in range(3):
        p[out + c * 64] = value[c]
    assert num_matrix_weights == out + 16 * 64 and num_params >= num_matrix_weights
    return p


def check_queries(n: int = 4096, seed: int = 5) -> np.ndarray:
    """random radiance queries, positions and angles well outside their normalised ranges included"""
    rng = np.random.default_rng(seed)
    q = rng.uniform(0.0, 1.0, size=(n, 14))
    q[:, 0:3] = rng.uniform(-2.0, 3.0, size=(n, 3))
    q[:, 3:7] = rng.uniform(-7.0, 7.0, size=(n, 4))
    return q.astype(F32)


def clustered_mean(values: np.ndarray, clusters: np.ndarray):
    """(mean, standard error, n) of `values` [n] whose correlated members share a cluster id: the ratio estimator over
    clusters, its variance from the spread of the cluster sums around mean * cluster size"""
    values = np.asarray(values, dtype=np.float64)
    _, inv = np.unique(clusters, return_inverse=True)
    sums = np.bincount(inv, weights=values)
    counts = np.bincount(inv).astype(np.float64)
    k = len(sums)
    mean = sums.sum() / counts.sum()
    resid = sums - mean * counts
    se = math.sqrt(k / max(k - 1, 1) * float((resid ** 2).sum())) / counts.sum()
    return mean, se, len(values)


def group_report(name: str, values: np.ndarray, clusters: np.ndarray, expected, slack: float = SLACK, min_n: int = 30):
    """per channel (mean, se, n, ok) of a group against `expected` [3]; nothing for a group of fewer than min_n samples"""
    out = []
    if len(values) < min_n:
        return out
    for c in range(3):
        mean, se, n = clustered_mean(values[:, c], clusters)
        ok = abs(mean - expected[c]) <= NSE * se + slack * expected[c]
        out.append((name, c, mean, se, n, bool(ok)))
    return out


def format_report(rows) -> str:
    return "\n".join(f"{name} ch{c}: mean {mean:.5f} se {se:.1e} n {n} expected {float(L[c]):.5f}{'' if ok else '  FAIL'}"
                     for name, c, mean, se, n, ok in rows)


# ---- one frame's buffers ----------------------------------------------------------------------------------------------
def pixel_groups(terminal_info: np.ndarray):
    """{group: bool mask [W*H]} from the pixel flags of the terminal info (bit 9 training pixel, bit 10 unbiased tile)"""
    w = terminal_info[:, 3]
    train = ((w >> 9) & 1).astype(bool)
    unbiased = ((w >> 10) & 1).astype(bool)
    return {"training pixels, biased tiles": train & ~unbiased, "training pixels, unbiased tiles": train & unbiased,
            "other pixels": ~train}


def record_tiles(suffix_terminal: np.ndarray, vertex_info: np.ndarray, ntrain: int) -> np.ndarray:
    """the tile of every training record [ntrain], by walking each tile's chain back from its suffix terminal; every record
    must be on exactly one chain"""
    invalid = 0x7FFFFF
    tile_of = np.full(ntrain, -1, dtype=np.int64)
    cur = (suffix_terminal.reshape(-1) & invalid).astype(np.int64)
    tiles = np.arange(len(cur))
    for _ in range(64):
        live = cur != invalid
        if not live.any():
            break
        cur, tiles = cur[live], tiles[live]
        assert (cur < ntrain).all() and (tile_of[cur] == -1).all(), "a record on two chains or beyond the record count"
        tile_of[cur] = tiles
        cur = (vertex_info[cur, 3] & invalid).astype(np.int64)
    assert (tile_of >= 0).all(), f"{int((tile_of < 0).sum())} records on no chain"
    return tile_of


def unbiased_tile(state: np.ndarray, buffer_index: int, width: int, tiles: np.ndarray) -> np.ndarray:
    tsx = int(state[abi.NRC_STATE_TILE_SIZE + 2 * buffer_index])
    ntx = (width + tsx - 1) // tsx
    tx, ty = tiles % ntx, tiles // ntx
    return ((ty % 4) * 4 + (tx % 4) + int(state[abi.NRC_STATE_OFFSET_UNBIASED_TILE])) % 16 == 0


RECORD_LENGTHS = {"1": (1, 1), "2": (2, 2), "3-5": (3, 5), ">=6": (6, 255)}


def record_groups(vertex_info: np.ndarray, unbiased: np.ndarray):
    length = (vertex_info[:, 3] >> 23) & 0xFF
    for name, (lo, hi) in RECORD_LENGTHS.items():
        sel = (length >= lo) & (length <= hi)
        yield f"records of length {name}, biased tiles", sel & ~unbiased
        yield f"records of length {name}, unbiased tiles", sel & unbiased


def shuffler_states(num_shuffles: int) -> np.ndarray:
    """the shufflers' LCG (neural_radiance_caching_main.cpp:1187-1193, nrc_setup_kernels.cu:150-152) after `num_shuffles`
    gfx_nrc_shuffle calls: seeded from 471313181, one step per entry, then one more step per call"""
    m = abi.NRC_TRAINING_DATA_PER_FRAME
    s = np.empty(m, dtype=np.uint64)
    lcg = 471313181
    for i in range(m):
        lcg = (lcg * 1103515245 + 12345) % (1 << 31)
        s[i] = lcg
    for _ in range(num_shuffles):
        s = (s * np.uint64(1103515245) + np.uint64(12345)) % np.uint64(1 << 31)
    return s


def check_shuffle(q0, t0, q1, t1, state, buffer_index: int, ntrain_total: int, num_shuffles: int, radiance_scale: float):
    """gfx_nrc_shuffle restated: row lcg % 65536 of buffer 1 holds record i % min(count, 131072) of buffer 0, its target times
    radianceScale clamped to 1e6; the state block's target min / max are exact, the average (float atomics in no defined
    order) within 1e-4 relative"""
    m = abi.NRC_TRAINING_DATA_PER_FRAME
    dst = (shuffler_states(num_shuffles) % np.uint64(m)).astype(np.int64)
    src = np.arange(m) % min(ntrain_total, abi.NRC_TRAIN_BUFFER_SIZE)
    assert np.isfinite(q0[src]).all() and np.isfinite(t0[src]).all()
    want_t = np.minimum(t0[src] * F32(radiance_scale), F32(1e6)).astype(F32)
    assert np.array_equal(t1[dst].view(np.uint32), want_t.view(np.uint32)), "shuffled targets"
    assert np.array_equal(q1[dst].view(np.uint32), q0[src].view(np.uint32)), "shuffled queries"
    s = state.reshape(-1)
    tsrc = t0[src]
    for c in range(3):
        assert s[abi.NRC_STATE_TARGET_MIN + 6 * buffer_index + c] == tsrc[:, c].min().view(np.uint32), f"target min {c}"
        assert s[abi.NRC_STATE_TARGET_MAX + 6 * buffer_index + c] == tsrc[:, c].max().view(np.uint32), f"target max {c}"
        avg = float(s[abi.NRC_STATE_TARGET_AVG + 3 * buffer_index + c:][:1].view(F32)[0])
        want = float(tsrc[:, c].astype(np.float64).sum() / m)
        assert abs(avg - want) <= 1e-4 * abs(want) + 1e-9, (c, avg, want)


def double_counted_beauty(beauty: np.ndarray, terminal_info: np.ndarray, inferred: np.ndarray, queries: np.ndarray,
                          radiance_scale: float) -> np.ndarray:
    """Negative control: the estimator before the training continuation stopped adding to the rendering radiance, restated
    in expectation over the downloaded buffers.  A training pixel whose rendering path ended in the cache went on adding the
    light its continuation found beyond the terminal vertex - an unbiased estimate of what the cache term alpha * cache
    already holds - so in expectation it showed alpha * cache twice.  `beauty` is one frame's (numAccumFrames 0)."""
    n = beauty.shape[0]
    t = terminal_info[:n]
    twice = ((t[:, 3] & 1) != 0) & (((t[:, 3] >> 9) & 1) != 0)
    alpha = t[:, :3].view(F32).astype(np.float64)
    cache = np.maximum(inferred[:n].astype(np.float64), 0.0) / radiance_scale * (queries[:n, 8:11] + queries[:n, 11:14])
    out = beauty.astype(np.float64).copy()
    out[twice] += alpha[twice] * cache[twice]
    return out


# ---- running frames ---------------------------------------------------------------------------------------------------
class OracleBackend:
    """the CPU oracle's NRC frame (tests/oracle_lib.py) with the CPU network of either position encoding"""

    def __init__(self, scene, width: int, height: int, encoding: int, num_hidden_layers: int = 2):
        from tests import oracle_lib, oracle_nrc_triwave
        self.oscene = oracle_lib.OracleScene(scene)
        self.frame = oracle_lib.OracleFrame(self.oscene, width, height)
        self.net = oracle_nrc_triwave.oracle_nrc(num_hidden_layers, 1e-2, encoding)
        self.num_params, self.num_matrix_weights = self.net.num_params, self.net.num_matrix_weights

    def set_params(self, params):
        self.net.set_params(params)

    def infer_queries(self, q):
        return self.net.infer(q)

    def linear(self, buffer_id, index=0):
        return self.frame.linear_buffer(buffer_id, index)

    def set_linear(self, buffer_id, index, data):
        self.frame.linear_buffer(buffer_id, index, copy=False)[:] = data

    def beauty(self):
        return self.frame.buffer(abi.BUF_BEAUTY_ACCUM)

    def frame_infer(self):
        count = int(self.linear(abi.BUF_NRC_STATE)[abi.NRC_STATE_NUM_INFERENCE_QUERIES, 0])
        pred = self.net.infer(self.linear(abi.BUF_NRC_INFERENCE_QUERY)[:count])
        self.frame.linear_buffer(abi.BUF_NRC_INFERRED_RADIANCE, copy=False)[:count] = pred

    def __getattr__(self, name):  # gbuffer, pathtrace, nrc_preprocess / accumulate / propagate / shuffle
        return getattr(self.frame, name)


class GpuBackend:
    """the library's NRC frame on a context (one gfx_ctx for the session) and a NeuralRadianceCache"""

    def __init__(self, ctx, scene, width: int, height: int, encoding: int, num_hidden_layers: int = 2):
        from gfxexp_b200 import engine
        self.ctx = ctx
        ctx.upload_scene(scene)
        ctx.build_bvh()
        ctx.create_frame(width, height)
        ctx.build_light_distributions(0)
        self.net = engine.NeuralRadianceCache(ctx, num_hidden_layers, 1e-2, encoding)
        self.num_params = self.net.num_params
        self.num_matrix_weights = num_hidden_layers * 64 * 64 + 16 * 64

    def close(self):
        self.net.close()

    def set_params(self, params):
        self.net.set_params(params)

    def infer_queries(self, q):
        import torch
        qd = torch.from_numpy(np.ascontiguousarray(q)).cuda()
        out = torch.empty((q.shape[0], 3), dtype=torch.float32, device="cuda")
        self.net.infer(qd, out, q.shape[0])
        torch.cuda.synchronize()
        return out.cpu().numpy()

    def linear(self, buffer_id, index=0):
        return self.ctx.download_linear(buffer_id, index)

    def set_linear(self, buffer_id, index, data):
        self.ctx.upload(buffer_id, index, data)

    def beauty(self):
        return self.ctx.download(abi.BUF_BEAUTY_ACCUM)

    def frame_infer(self):
        self.ctx.nrc_frame_infer(self.net)

    def __getattr__(self, name):
        return getattr(self.ctx, name)


def self_check(backend, params, value):
    """the installed network returns exactly `value` (rounded to half) on random queries, out-of-range ones included"""
    backend.set_params(params)
    got = backend.infer_queries(check_queries())
    want = np.broadcast_to(np.asarray(value, dtype=np.float16).astype(F32), got.shape)
    assert np.array_equal(got, want), (got[:2], want[0])


def offsets(frame: int):
    rng = np.random.default_rng(1000 + frame)
    return [int(v) for v in rng.integers(0, 2 ** 32, size=2)]


class Samples:
    """per group: the samples [n, 3] and their cluster ids"""

    def __init__(self):
        self.values, self.clusters = {}, {}

    def add(self, name, values, clusters):
        self.values.setdefault(name, []).append(np.asarray(values, dtype=np.float64).reshape(-1, 3))
        self.clusters.setdefault(name, []).append(np.asarray(clusters, dtype=np.int64).reshape(-1))

    def report(self, expected=L, min_n: int = 30):
        rows = []
        for name in self.values:
            rows += group_report(name, np.concatenate(self.values[name]), np.concatenate(self.clusters[name]), expected,
                                 min_n=min_n)
        return rows


def run_nrc(backend, scene, width: int, height: int, frames: int, cache_scale: float = 1.0, seed_tile=None,
            num_hidden_layers: int = 2):
    """`frames` GFX_PT_NRC frames with the constant cache radianceScale * L * cache_scale (never trained): G-buffer, preprocess
    (each frame its own tile offsets; seed_tile: that tile size, so that small tiles fill the record buffer), path tracing,
    frame inference, accumulate with numAccumFrames 0 (the beauty is the frame's estimate), propagate, shuffle.  Returns
    (pixel samples, record samples, negative-control pixel samples of the double count, buffer-full frames); checks the
    shuffle exactly and every target finite and non-negative on the way."""
    from tests import nrc_records
    value = RADIANCE_SCALE * L * cache_scale
    params = constant_params(backend.num_params, backend.num_matrix_weights, num_hidden_layers, value)
    self_check(backend, params, value)
    p = abi.default_frame_params(scene, width, height)
    p.maxPathLength = 0
    p.radianceScale = RADIANCE_SCALE
    n = width * height
    pixels, records, doubled = Samples(), Samples(), Samples()
    full_frames = 0
    for f in range(frames):
        p.frameIndex, p.bufferIndex, p.numAccumFrames = f, f % 2, 0
        backend.gbuffer(p)
        if seed_tile is not None:
            backend.set_linear(abi.BUF_NRC_STATE, 0, nrc_records.seeded_state(backend.linear(abi.BUF_NRC_STATE), p.bufferIndex,
                                                                            seed_tile))
        o = offsets(f)
        backend.nrc_preprocess(p, o[0], o[1], f == 0 and seed_tile is None)
        backend.pathtrace(p, abi.PT_NRC)
        backend.frame_infer()
        backend.nrc_accumulate(p)
        ti = backend.linear(abi.BUF_NRC_TERMINAL_INFO)
        beauty = backend.beauty()[..., :3].reshape(n, 3)
        assert np.isfinite(beauty).all()
        ids = f * n + np.arange(n)
        groups = pixel_groups(ti)
        dc = double_counted_beauty(beauty, ti, backend.linear(abi.BUF_NRC_INFERRED_RADIANCE),
                                   backend.linear(abi.BUF_NRC_INFERENCE_QUERY), RADIANCE_SCALE)
        for name, sel in groups.items():
            pixels.add(name, beauty[sel], ids[sel])
            doubled.add(name, dc[sel], ids[sel])

        backend.nrc_propagate(p)
        state = backend.linear(abi.BUF_NRC_STATE)[:, 0]
        total = int(state[p.bufferIndex])
        ntrain = min(total, abi.NRC_TRAIN_BUFFER_SIZE)
        full_frames += total > abi.NRC_TRAIN_BUFFER_SIZE
        q0 = backend.linear(abi.BUF_NRC_TRAIN_QUERY, 0)[:ntrain]
        t0 = backend.linear(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain]
        vi = backend.linear(abi.BUF_NRC_TRAIN_VERTEX_INFO)[:ntrain]
        assert np.isfinite(t0).all() and (t0 >= 0).all(), "a training target is not finite or negative"
        tiles = record_tiles(backend.linear(abi.BUF_NRC_TRAIN_SUFFIX_TERMINAL), vi, ntrain)
        unbiased = unbiased_tile(state, p.bufferIndex, width, tiles)
        for name, sel in record_groups(vi, unbiased):
            records.add(name, t0[sel], f * n + tiles[sel])

        backend.nrc_shuffle(p)
        check_shuffle(q0, t0, backend.linear(abi.BUF_NRC_TRAIN_QUERY, 1), backend.linear(abi.BUF_NRC_TRAIN_TARGET, 1),
                      backend.linear(abi.BUF_NRC_STATE), p.bufferIndex, total, f + 1, RADIANCE_SCALE)
    return pixels, records, doubled, full_frames


def run_baseline(backend, scene, width: int, height: int, frames: int, max_path_length: int) -> Samples:
    """the baseline path tracer (GFX_PT_BASELINE), `frames` frames accumulated; one sample per pixel"""
    p = abi.default_frame_params(scene, width, height)
    p.maxPathLength = max_path_length
    for f in range(frames):
        p.frameIndex, p.bufferIndex, p.numAccumFrames = f, f % 2, f
        backend.gbuffer(p)
        backend.pathtrace(p)
    s = Samples()
    b = backend.beauty()[..., :3].reshape(-1, 3)
    s.add("all pixels", b, np.arange(len(b)))
    return s


def baseline_series(max_path_length: int) -> np.ndarray:
    """the baseline path tracer's expectation at maxPathLength n (0: the hosts' default 5, pathtrace.cu)"""
    return truncated_series(max_path_length or 5)
