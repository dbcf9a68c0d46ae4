"""GPU: light sampling as the renderers call it (gfx_light_sample_debug) against the CPU oracle (orc_light_sample_debug), on the
emitter layouts and environment maps of tests/light_scenes.py, bit for bit apart from NaN payloads (x86 and sm_90a write different
NaN bits).  The oracle side is checked against float64 and its own densities in test_oracle_light_sampling.py.  Also: the dark
early-out of the RIS candidate loop (sampleLightUnlessDark, classifyLight + finishLightSample) against the plain sample and the
float64 geometry, the pick after gfx_scene_update_instances, the instance-count limits, and renders under a sky with black rows."""
import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import light_ref as R
from tests import light_scenes as LS

pytestmark = pytest.mark.gpu

N_LATTICE = 1 << 23
KEY_NONE = 0x40000000
GFX_ERR_INVALID_ARGUMENT, GFX_ERR_UNSUPPORTED = -1, -6  # include/gfxb200.h


def _same(got, want, tag):
    g, w = got.view(np.uint32), want.view(np.uint32)
    eq = (g == w) | (np.isnan(got) & np.isnan(want))
    assert eq.all(), f"{tag}: {np.count_nonzero(~eq.all(axis=-1))} records differ, first {np.argwhere(~eq)[:4].tolist()}"


def _records(rng, n, env=False):
    rec = rng.random((n, 3), dtype=np.float32)
    rec[:64, 0] = np.array([0.0, 0.99999994, 0.5, 2.0 ** -23] * 16, dtype=np.float32)
    return rec


def _hit_records(em, rng, n):
    k = rng.integers(0, em.prob.size, n)
    rec = np.zeros((n, 5), dtype=np.float32)
    rec[:, 0] = em.inst[k].astype(np.uint32).view(np.float32)
    rec[:, 1] = em.geom[k].astype(np.uint32).view(np.float32)
    rec[:, 2] = em.prim[k].astype(np.uint32).view(np.float32)
    b = rng.random((n, 2), dtype=np.float32) * 0.5
    rec[:, 3:] = b
    return rec


def _split_records(n_cand, ul):
    rec = np.zeros((ul.size * n_cand, 3), dtype=np.float32)
    rec[:, 0] = np.repeat(np.arange(n_cand, dtype=np.uint32), ul.size).view(np.float32)
    rec[:, 1] = np.uint32(n_cand).view(np.float32)
    rec[:, 2] = np.tile(ul, n_cand)
    return rec


@pytest.mark.parametrize("name", list(LS.EMITTER_SCENES))
def test_emitter_ops_bit_exact(gfx_ctx, oracle, name):
    scene = LS.EMITTER_SCENES[name]()
    scene.env_map = LS.env_map("37x19")
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_light_distributions()
    osc = oracle.OracleScene(scene, build_bvh=False)
    em = R.emitters(scene)
    rng = np.random.default_rng(11)
    rec = _records(rng, 1 << 18)
    _same(gfx_ctx.light_sample_debug(0, rec), osc.light_sample_debug(0, rec), f"{name} op 0")
    hits = _hit_records(em, rng, 1 << 16)
    for env in (False, True):
        _same(gfx_ctx.light_sample_debug(5, hits, enable_env=env), osc.light_sample_debug(5, hits, enable_env=env), f"{name} op 5 env {env}")
        ul = rng.random(1 << 14, dtype=np.float32)
        for n in (32, 30):
            r6 = _split_records(n, ul)
            _same(gfx_ctx.light_sample_debug(6, r6, enable_env=env), osc.light_sample_debug(6, r6, enable_env=env), f"{name} op 6")
        _same(gfx_ctx.light_sample_debug(7, ul[:, None], enable_env=env), osc.light_sample_debug(7, ul[:, None], enable_env=env),
              f"{name} op 7")


@pytest.mark.parametrize("kind", [k for k in LS.ENV_KINDS])
def test_env_ops_bit_exact(gfx_ctx, oracle, kind):
    scene = LS.single_triangle()
    scene.env_map = LS.env_map(kind)
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_light_distributions()
    osc = oracle.OracleScene(scene, build_bvh=False)
    rng = np.random.default_rng(12)
    u = rng.random((1 << 17, 2), dtype=np.float32)
    u[:4] = [[0.0, 0.0], [0.99999994, 0.99999994], [0.5, 0.0], [0.0, 0.5]]
    dirs = R.from_polar_y_up(rng.uniform(0, 2 * np.pi, 1 << 17), np.arccos(rng.uniform(-1, 1, 1 << 17))).astype(np.float32)
    miss = np.concatenate([dirs, rng.random((dirs.shape[0], 1), dtype=np.float32) * 3, np.full((dirs.shape[0], 1), 0.25, np.float32)], 1)
    for rot in (0.0, 0.7, -3.0, 10.0):
        _same(gfx_ctx.light_sample_debug(3, u, env_rotation=rot, env_power=1.5, enable_env=True),
              osc.light_sample_debug(3, u, env_rotation=rot, env_power=1.5, enable_env=True), f"{kind} op 3 rotation {rot}")
        _same(gfx_ctx.light_sample_debug(4, miss, env_rotation=rot, enable_env=True),
              osc.light_sample_debug(4, miss, env_rotation=rot, enable_env=True), f"{kind} op 4 rotation {rot}")
    out = gfx_ctx.light_sample_debug(4, miss, enable_env=True)
    if kind.startswith("black"):  # density 0 (finite) in the black rows / columns / map, never NaN
        assert not np.isnan(out[:, :2]).any()


@pytest.mark.parametrize("name", ["spread_weights", "guide_sizes", "scaled_instances"])
def test_lattice_counts_equal_the_oracle(gfx_ctx, oracle, name):
    """the flattened pick's keys over the whole PCG32 lattice (gfx_light_pick_debug) against the oracle's sampleLight"""
    import torch
    scene = LS.EMITTER_SCENES[name]()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_light_distributions()
    osc = oracle.OracleScene(scene, build_bvh=False)
    ul = (np.arange(N_LATTICE, dtype=np.float64) * 2.0 ** -23).astype(np.float32)
    d_ul = torch.from_numpy(ul).cuda()
    flat = torch.empty(N_LATTICE, dtype=torch.int32, device="cuda")
    chain = torch.empty_like(flat)
    gfx_ctx._check(gfx_ctx.lib.gfx_light_pick_debug(gfx_ctx.h, None, d_ul.data_ptr(), N_LATTICE, flat.data_ptr(), chain.data_ptr()),
                   "gfx_light_pick_debug")
    torch.cuda.synchronize()
    keys = flat.cpu().numpy().view(np.uint32)
    want = np.concatenate([osc.light_sample_debug(0, ul[lo:lo + (1 << 21), None])[:, 0].view(np.uint32)
                           for lo in range(0, N_LATTICE, 1 << 21)])
    assert np.array_equal(keys, want), f"{np.count_nonzero(keys != want)} lattice points differ"
    n = R.emitters(scene).prob.size
    live = (keys & KEY_NONE) == 0
    assert np.array_equal(np.bincount(keys[live], minlength=n), np.bincount(want[live], minlength=n))


def test_pick_after_a_scale_change_equals_a_fresh_upload(gfx_ctx):
    scene = LS.scaled_instances()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_light_distributions()
    moved = [scenes.make_instance(i.mesh_slots, tuple(i.transform[:, 3]), scale=s) for i, s in zip(scene.instances[:4], (2.0, 0.25, 0.5, 1.0))]
    new_insts = moved + scene.instances[4:]
    gfx_ctx.update_instances(abi.make_instance_descs(new_insts))
    with pytest.raises(engine.GfxError):  # the pick of the old transforms is not served
        gfx_ctx.light_sample_debug(0, np.zeros((1, 3), np.float32))
    gfx_ctx.build_light_distributions()
    ul = (np.arange(0, N_LATTICE, 7, dtype=np.float64) * 2.0 ** -23).astype(np.float32)
    rec = np.stack([ul, np.full_like(ul, 0.3), np.full_like(ul, 0.6)], 1)
    updated = gfx_ctx.light_sample_debug(0, rec)
    fresh_scene = LS.scaled_instances()
    fresh_scene.instances = new_insts
    gfx_ctx.upload_scene(fresh_scene)
    gfx_ctx.build_light_distributions()
    _same(updated, gfx_ctx.light_sample_debug(0, rec), "update_instances vs fresh upload")


def test_instance_count_limits(gfx_ctx):
    for n, ok in ((28000, True), (28001, False)):
        gfx_ctx.upload_scene(LS.many_instances(n))
        rc = gfx_ctx.lib.gfx_light_dist_build(gfx_ctx.h, None, 0)
        assert (rc == 0) == ok, (n, rc)
        if not ok:
            assert rc == GFX_ERR_UNSUPPORTED


def test_nan_texel_is_refused(gfx_ctx):
    scene = LS.single_triangle()
    scene.env_map = LS.env_map("37x19")
    scene.env_map[3, 4, 1] = np.nan
    arrays = abi.SceneArrays(scene)
    assert gfx_ctx.lib.gfx_scene_upload(gfx_ctx.h, abi.C.byref(arrays.desc)) == GFX_ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("name", ["single_triangle", "guide_sizes", "degenerate_light"])
def test_dark_cull(gfx_ctx, name):
    """Shading points around each light (in a box, on its plane, inside its bounding sphere, on the triangle), vOutLocalZ in
    {+-1, +-1e-3, +-1e-7, +0, -0}, normals +- the light's.  Ops 1 (sampleLightUnlessDark) and 2 (classifyLight + finishLightSample)
    decide alike; not dark, they are op 0 bit for bit; dark, the float64 geometry has the sample below the shading horizon or
    behind the emitter by more than the cull's 1e-3 cosine margin (a little less for the sphere test's bound: 1e-3 / 2)."""
    scene = LS.EMITTER_SCENES[name]()
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_light_distributions()
    em = R.emitters(scene)
    rng = np.random.default_rng(13)
    lights = np.flatnonzero(em.prob > 1e-6)
    lights = lights[rng.integers(0, lights.size, 512)]
    pick0 = np.cumsum(em.prob)
    # a lattice point inside each chosen light's piece (probe the flattened pick, which op 0 reports)
    probe = np.clip(pick0[lights] - 0.5 * em.prob[lights], 0, 0.99999994).astype(np.float32)
    keys = gfx_ctx.light_sample_debug(0, probe[:, None])[:, 0].view(np.uint32)
    lights, probe = lights[keys == lights], probe[keys == lights]
    per = 48
    n = lights.size * per
    L = np.repeat(lights, per)
    wv = em.world[L]
    c = wv.mean(axis=1)
    nl = np.cross(wv[:, 1] - wv[:, 0], wv[:, 2] - wv[:, 0])
    nl /= np.linalg.norm(nl, axis=1, keepdims=True)
    r = np.linalg.norm(wv - c[:, None], axis=2).max(axis=1)
    kind = rng.integers(0, 4, n)
    box = c + rng.uniform(-3, 3, (n, 3)) * np.maximum(r, 0.1)[:, None]
    plane = box - np.sum((box - c) * nl, axis=1, keepdims=True) * nl
    ball = c + rng.normal(size=(n, 3)) * (0.5 * r)[:, None]
    a, b, cc = R.square_to_triangle(rng.random(n), rng.random(n))
    ontri = a[:, None] * wv[:, 0] + b[:, None] * wv[:, 1] + cc[:, None] * wv[:, 2]
    sp = np.select([kind[:, None] == k for k in range(4)], [box, plane, ball, ontri])
    sn = nl * rng.choice([-1.0, 1.0], n)[:, None]
    tilt = rng.normal(size=(n, 3)) * 0.3 * (rng.random(n) < 0.5)[:, None]
    sn = (sn + tilt) / np.linalg.norm(sn + tilt, axis=1, keepdims=True)
    sp, sn = sp.astype(np.float32).astype(np.float64), sn.astype(np.float32).astype(np.float64)  # what the device receives
    vz = rng.choice(np.array([1, -1, 1e-3, -1e-3, 1e-7, -1e-7, 0.0, -0.0], dtype=np.float32), n)
    u = rng.random((n, 2), dtype=np.float32)
    rec = np.concatenate([np.repeat(probe, per)[:, None], u, sp.astype(np.float32), sn.astype(np.float32), vz[:, None]], 1).astype(np.float32)
    o0, o1, o2 = (gfx_ctx.light_sample_debug(op, rec) for op in (0, 1, 2))
    dark1, dark2 = o1[:, 12] > 0, o2[:, 12] > 0
    fin = np.isfinite(o0[:, 10])
    assert np.array_equal(dark1[fin], dark2[fin]), f"{name}: ops 1 and 2 decide differently on {np.count_nonzero(dark1 != dark2)} records"
    # A light of infinite density (degenerate_light: a world-space area of 0): the steps 1 and 2 of sampleLightUnlessDark test
    # density > 0 and may cull it, classifyLight's cullable bit needs a finite density and leaves it to the exact path.  Both
    # add RGB(0) to the reservoir (the sample is dark by the margin checked below); pinned: only op 1 culls more.
    assert not (dark2 & ~dark1).any()
    _same(o1[~dark1, :12], o0[~dark1, :12], f"{name}: op 1 not dark vs op 0")
    _same(o2[~dark2, :12], o0[~dark2, :12], f"{name}: op 2 not dark vs op 0")
    assert dark1.mean() > 0.1, f"{name}: the cull never fires ({dark1.mean():.3f})"
    # the float64 geometry of each dark decision (op 2's are a subset of op 1's): the sample point of op 0
    pos = o0[dark1, 1:4].astype(np.float64)
    d = pos - sp[dark1]
    dist = np.linalg.norm(d, axis=1)
    below = -(np.sum(d * sn[dark1], axis=1) * np.sign(vz[dark1].astype(np.float64))) / dist
    lnorm = o0[dark1, 4:7].astype(np.float64)
    behind = np.sum(d * lnorm, axis=1) / dist
    margin = np.maximum(below, behind)
    assert np.all(margin > 0.5e-3), f"{name}: a dark decision within the margin: {margin.min():.3g}"


# ---- renders under a sky whose ground rows are black ---------------------------------------------------------------------------
def test_black_ground_pathtrace(gfx_ctx, oracle):
    """the baseline path tracer at maxPathLength 4, 4 frames at 64 x 40: finite and equal to the oracle (before the fix, 2 NaN
    pixels: the miss program's MIS weight along the black rows was 0 / 0)"""
    scene = LS.sky_with_black_ground()
    w, h = 64, 40
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    oframe = oracle.OracleFrame(oracle.OracleScene(scene), w, h)
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = 4
    gfx_ctx.build_light_distributions(0)
    for frame in range(4):
        p.numAccumFrames = p.frameIndex = frame
        gfx_ctx.gbuffer(p)
        gfx_ctx.pathtrace(p)
        oframe.gbuffer(p)
        oframe.pathtrace(p)
        got, want = gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), oframe.buffer(abi.BUF_BEAUTY_ACCUM)
        assert np.isfinite(got).all(), f"frame {frame}: {np.count_nonzero(~np.isfinite(got))} non-finite values"
        _same(got, want, f"beauty frame {frame}")


def test_black_ground_nrc_pathtrace(gfx_ctx, oracle):
    from tests.test_gpu_nrc_frame import _compare_pathtrace
    scene = LS.sky_with_black_ground()
    w, h = 96, 64
    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(w, h)
    gfx_ctx.build_light_distributions(0)
    oframe = oracle.OracleFrame(oracle.OracleScene(scene), w, h)
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = 5
    for frame in range(2):
        p.frameIndex, p.bufferIndex, p.numAccumFrames = frame, frame % 2, frame
        gfx_ctx.gbuffer(p)
        gfx_ctx.nrc_preprocess(p, 17 + frame, 91 + frame, frame == 0)
        gfx_ctx.pathtrace(p, abi.PT_NRC)
        oframe.gbuffer(p)
        oframe.nrc_preprocess(p, 17 + frame, 91 + frame, frame == 0)
        oframe.pathtrace(p, abi.PT_NRC)
        _compare_pathtrace(gfx_ctx, oframe, p, f"frame {frame}")
        assert np.isfinite(gfx_ctx.download_linear(abi.BUF_NRC_FRAME_CONTRIBUTION)).all()


def test_black_ground_svgf_app(gfx_ctx):
    from tests.test_gpu_svgf_app import _run
    _run(gfx_ctx, LS.sky_with_black_ground(), 96, 64, 3)
