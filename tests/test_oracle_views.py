"""The oracle's debug views against numpy transcriptions of the reference kernels they restate:
visualizeToOutputBuffer of the NRC app (neural_radiance_caching/gpu_kernels/copy_buffers.cu:32-130), calcCellColor of the
ReGIR app (regir/gpu_kernels/copy_buffers.cu:30-76), and the visualizePrediction pass
(neural_radiance_caching/gpu_kernels/optix_pathtracing_kernels.cu:702-778) on a rendered G-buffer."""
import numpy as np
import pytest

from gfxexp_b200 import abi, scenes
from tests import oracle_views as V

f32 = np.float32
W, H = 37, 23


def _pack(v):
    """min(uint(v * 255), 255) per channel with CUDA's saturating conversion (NaN and negatives -> 0)"""
    s = (v.astype(f32) * f32(255)).astype(np.float64)
    s = np.where(s > 0, np.minimum(np.trunc(np.nan_to_num(s, nan=0.0, posinf=1e10)), 255), 0).astype(np.uint32)
    return s[..., 0] | (s[..., 1] << 8) | (s[..., 2] << 16) | (s[..., 3] << 24)


def _buffers(seed):
    rng = np.random.default_rng(seed)
    n = W * H
    ti = np.zeros((n, 4), dtype=np.uint32)
    ti[:, :3] = rng.uniform(-0.5, 2.0, (n, 3)).astype(f32).view(np.uint32)
    has_query = rng.integers(0, 2, n)
    path_length = np.arange(n) % 32                        # 0 .. 31
    bits = rng.integers(0, 4, n)                           # every combination of training / unbiased
    ti[:, 3] = has_query | (path_length << 1) | ((bits & 1) << 9) | ((bits >> 1) << 10)
    pred = rng.uniform(-1.0, 3.0, (n, 3)).astype(f32)
    pred[rng.random((n, 3)) < 0.1] = np.nan               # negative and NaN predictions
    query = rng.uniform(0.0, 1.0, (n, 14)).astype(f32)
    mv = rng.uniform(-20.0, 20.0, (n, 2)).astype(f32)     # clamps at both ends with scale 0.1, offset 0.5
    mv[::7] = [[-1e3, 1e3]]
    gb2 = np.zeros((n, 4), dtype=f32)
    gb2[:, :3] = rng.uniform(-5.0, 5.0, (n, 3))
    rgba = rng.uniform(0.0, 1.5, (H, W, 4)).astype(f32)
    return ti, pred, query, mv, gb2, rgba


def _numpy_views(mode, flags, p, ti, pred, query, mv, gb2, rgba, scale, offset):
    """the view value per pixel, transcribed from copy_buffers.cu in float32"""
    n = W * H
    v = rgba.reshape(n, 4).copy() if mode == abi.PRESENT_COLOR else np.zeros((n, 4), dtype=f32)
    alpha = ti[:, :3].view(f32)
    if mode == abi.PRESENT_NRC_PREDICTION:                 # :52-67
        rad = np.fmax(pred, f32(0))
        if p.radianceScale > 0:
            rad = rad * (f32(1) / f32(p.radianceScale))  # RGB /= s multiplies by the reciprocal
        rad = rad * (query[:, 8:11] + query[:, 11:14])
        rad = np.where((ti[:, 3] & 1).astype(bool)[:, None], rad, f32(0))
        v[:, :3] = alpha * rad
        v[:, 3] = 1
    elif mode == abi.PRESENT_FLOW:                         # :87-94
        v[:, :2] = np.fmin(np.fmax(f32(scale) * mv + f32(offset), f32(0)), f32(1))
        v[:, 2] = f32(offset)
        v[:, 3] = 1
    elif mode == abi.PRESENT_NRC_PATH_LENGTH:              # :96-112
        pl = ((ti[:, 3] >> 1) & 0xFF).astype(np.int64)
        t = np.minimum((pl - 1).astype(f32) / f32(5), f32(1))
        lo = t < f32(0.5)
        tt = np.where(lo, f32(2) * t, f32(2) * (t - f32(0.5))).astype(f32)
        one_m = (f32(1) - tt).astype(f32)
        zero = f32(0)
        # B * (1 - tt) + G * tt  /  G * (1 - tt) + R * tt, componentwise
        v[:, 0] = np.where(lo, zero * one_m + zero * tt, zero * one_m + f32(1) * tt)
        v[:, 1] = np.where(lo, zero * one_m + f32(1) * tt, f32(1) * one_m + zero * tt)
        v[:, 2] = np.where(lo, f32(1) * one_m + zero * tt, zero * one_m + zero * tt)
        v[:, 3] = 1
    elif mode == abi.PRESENT_COLOR and flags & abi.PRESENT_REGIR_CELLS:
        v[:, :3] *= _numpy_cell_color(p, gb2[:, :3])
    if flags & abi.PRESENT_NRC_TRAINING_PATHS:             # :118-127
        train = ((ti[:, 3] >> 9) & 1).astype(bool)
        unbiased = ((ti[:, 3] >> 10) & 1).astype(bool) & ~train
        v[train] *= np.array([1, 0.25, 1, 1], dtype=f32)
        v[unbiased] *= np.array([0.25, 1, 0.25, 1], dtype=f32)
    return v.reshape(H, W, 4)


def _pcg32_floats(state, k):
    out = []
    for _ in range(k):
        old = state
        state = (old * 6364136223846793005 + 1) & (2 ** 64 - 1)
        xorshifted = (((old >> 18) ^ old) >> 27) & 0xFFFFFFFF
        rot = old >> 59
        r = ((xorshifted >> rot) | (xorshifted << ((-rot) & 31))) & 0xFFFFFFFF
        out.append(np.array([(r >> 9) | 0x3F800000], dtype=np.uint32).view(f32)[0] - f32(1))
    return out


def _hsv_to_rgb(h, s, v):                                  # basic_types.h:5365-5388
    if s == 0:
        return [v, v, v]
    hm = f32(h - np.floor(h))
    hi = int(f32(hm * f32(6)))
    f = f32(hm * f32(6) - f32(hi))
    m, n, k = f32(v * (f32(1) - s)), f32(v * (f32(1) - s * f)), f32(v * (f32(1) - s * (f32(1) - f)))
    return [[v, k, m], [n, v, m], [m, v, k], [m, n, v], [k, m, v], [v, m, n]][hi] if hi < 6 else [0, 0, 0]


def _numpy_cell_color(p, positions):
    dim = list(p.regirGridDim)
    if 0 in dim:
        dim = [32, 8, 32]
    lo = np.array(p.sceneAabbMin, dtype=f32)
    cell = (np.array(p.sceneAabbMax, dtype=f32) - lo) / np.array(dim, dtype=f32)
    out = np.zeros((len(positions), 3), dtype=f32)
    for i, pos in enumerate(positions.astype(f32)):
        q = (pos - lo) / cell
        idx = [min(int(min(c, 4294967295.0)) if c > 0 else 0, d - 1) for c, d in zip(q, dim)]
        lin = idx[2] * dim[0] * dim[1] + idx[1] * dim[0] + idx[0]
        h = 2166136261
        for b in lin.to_bytes(4, "little"):
            h = ((16777619 * h) & 0xFFFFFFFF) ^ b
        u = _pcg32_floats((h << 32) | 3018421212, 3)
        out[i] = _hsv_to_rgb(u[0], f32(f32(0.5) + f32(0.5) * u[1]), f32(f32(0.5) + f32(0.5) * u[2]))
    return out


def _params(radiance_scale=0.0, grid=(0, 0, 0)):
    p = abi.default_frame_params(scenes.tiny_city_scene(), W, H)
    p.radianceScale = radiance_scale
    p.sceneAabbMin[:] = [-4.0, -1.0, -3.0]
    p.sceneAabbMax[:] = [4.0, 3.0, 5.0]
    p.regirGridDim[:] = list(grid)
    return p


@pytest.mark.parametrize("mode,flags", [(abi.PRESENT_NRC_PREDICTION, 0), (abi.PRESENT_NRC_PATH_LENGTH, 0), (abi.PRESENT_FLOW, 0),
                                        (abi.PRESENT_COLOR, abi.PRESENT_NRC_TRAINING_PATHS),
                                        (abi.PRESENT_NRC_PREDICTION, abi.PRESENT_NRC_TRAINING_PATHS),
                                        (abi.PRESENT_COLOR, abi.PRESENT_REGIR_CELLS),
                                        (abi.PRESENT_COLOR, abi.PRESENT_REGIR_CELLS | abi.PRESENT_NRC_TRAINING_PATHS),
                                        (abi.PRESENT_FLOW, abi.PRESENT_REGIR_CELLS)])
@pytest.mark.parametrize("radiance_scale", [0.0, 4.0])
def test_views_match_numpy_transcription(oracle, mode, flags, radiance_scale):
    ti, pred, query, mv, gb2, rgba = _buffers(11)
    p = _params(radiance_scale, (5, 3, 4))
    for flip in (0, abi.PRESENT_FLIP_Y):
        got = V.present_views(p, mode, flags | flip, rgba=rgba, terminal_info=ti, inferred_radiance=pred,
                                   inference_query=query, gbuffer1=mv, gbuffer2=gb2, alpha_override=-1.0,
                                   motion_vector_scale=0.1, motion_vector_offset=0.5)
        want = _pack(_numpy_views(mode, flags, p, ti, pred, query, mv, gb2, rgba, 0.1, 0.5))
        if flip:
            want = want[::-1]
        assert got.shape == (H, W)
        bad = np.argwhere(got != want)
        assert len(bad) == 0, f"mode {mode} flags {flags | flip}: {len(bad)} pixels differ, first {bad[:3].tolist()}"


def test_views_tone_map_after_tint(oracle):
    """the tints come before the alpha override, tone map and gamma: a tinted view presented with those equals the
    plain present of the tinted float image"""
    ti, pred, query, mv, gb2, rgba = _buffers(5)
    p = _params(2.0)
    flags = abi.PRESENT_NRC_TRAINING_PATHS | abi.PRESENT_TONE_MAP | abi.PRESENT_SRGB_GAMMA
    got = V.present_views(p, abi.PRESENT_NRC_PREDICTION, flags, terminal_info=ti, inferred_radiance=pred,
                               inference_query=query, brightness_scale=3.0, alpha_override=0.5, width=W, height=H)
    tinted = _numpy_views(abi.PRESENT_NRC_PREDICTION, flags, p, ti, pred, query, mv, gb2, rgba, 0.1, 0.5)
    want = oracle.present(tinted, abi.PRESENT_COLOR, abi.PRESENT_TONE_MAP | abi.PRESENT_SRGB_GAMMA, 3.0, 0.5)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("grid", [(0, 0, 0), (5, 3, 4), (1, 1, 1)])
def test_cell_color_matches_numpy_transcription(oracle, grid):
    p = _params(0.0, grid)
    rng = np.random.default_rng(3)
    inside = rng.uniform([-4, -1, -3], [4, 3, 5], (200, 3))
    on = np.array([[-4, -1, -3], [4, 3, 5], [0, 1, 1], [-4, 3, 5], [4, -1, -3]], dtype=f32)
    outside = np.array([[-100, -100, -100], [100, 100, 100], [-4.5, 1, 1], [0, 3.5, 0], [np.nan, 0, 0],
                        [np.inf, -np.inf, 0]], dtype=f32)
    pos = np.concatenate([inside, on, outside]).astype(f32)
    got = V.regir_cell_color(p, pos)
    want = _numpy_cell_color(p, pos)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert (got >= 0).all() and (got <= 1).all()
    if grid != (1, 1, 1):
        assert len(np.unique(got[:200], axis=0)) > 5  # neighbouring cells get different colours


@pytest.mark.parametrize("scene_name", ["small_interior_scene", "small_city_scene_env"])
def test_visualize_prediction_pass(oracle, scene_name):
    """the oracle's visualizePrediction on a rendered G-buffer: a query row per hit, miss rows untouched, positions
    normalised into the scene box, finite predictions of the oracle network"""
    scene = getattr(scenes, scene_name)()
    w, h = 48, 32
    oframe = V.ViewsFrame(scene, w, h)
    p = abi.default_frame_params(scene, w, h)
    p.bufferIndex = 1
    oframe.gbuffer(p)
    q = oframe.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY, copy=False)
    sentinel = np.uint32(0x7FC0DEAD)
    q.view(np.uint32)[:] = sentinel
    oframe.nrc_visualize_prediction(p)
    n = w * h
    hit = oframe.buffer(abi.BUF_GBUFFER0, 1)[..., 0].reshape(-1) != 0xFFFFFFFF
    assert hit.any()
    if scene_name == "small_city_scene_env":
        assert not hit.all()
    ti = oframe.linear_buffer(abi.BUF_NRC_TERMINAL_INFO)
    assert np.array_equal((ti[:, 3] & 1).astype(bool), hit)
    assert (ti[:, 3] >> 1 & 0xFF == 1).all() and (ti[:, 3] >> 9 == 0).all()
    assert (ti[:, :3].view(f32) == 1).all()
    q = oframe.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)
    assert (q[:n][~hit].view(np.uint32) == sentinel).all()
    assert (q[n:].view(np.uint32) == sentinel).all()
    rows = q[:n][hit]
    assert np.isfinite(rows).all()
    assert (rows[:, :3] >= 0).all() and (rows[:, :3] <= 1).all()
    st = oframe.linear_buffer(abi.BUF_NRC_STATE)[:, 0]
    assert st[abi.NRC_STATE_NUM_INFERENCE_QUERIES] == (n + 127) // 128 * 128
    onet = oracle.OracleNrc(2, 1e-2)
    pred = onet.infer(rows)
    assert np.isfinite(pred).all()
