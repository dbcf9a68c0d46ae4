"""GPU parity of the bump mapping (GfxFrameParams::enableBumpMapping, GfxSceneDesc::bumpMaps) on small_city_scene_bumped:
every renderer that tilts its shading frames, bit for bit against the CPU oracle with the switch on; the switch off gives the
buffers of the same scene without a bump table; the software gather equals the texture unit's tld4; the C++ host's
-bump-mapping equals the Python host."""
import os
import subprocess

import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_bump as B
from tests import test_gpu_host_cpp as HOSTS
from tests import test_gpu_nrc_frame as NRC
from tests import test_gpu_nrc_views as NRCV
from tests import test_gpu_restir_rearch as REARCH

pytestmark = pytest.mark.gpu

W, H = 160, 96


def _same(got, want, tag):
    g, w = np.ascontiguousarray(got), np.ascontiguousarray(want)
    g = g.view(np.uint32) if g.dtype.itemsize == 4 else g
    w = w.view(np.uint32) if w.dtype.itemsize == 4 else w
    if not np.array_equal(g, w):
        bad = np.argwhere(g != w)
        raise AssertionError(f"{tag}: {len(bad)} elements differ, first {bad[:4].tolist()}")


@pytest.fixture(scope="module")
def bumped():
    return scenes.small_city_scene_bumped()


def _setup(ctx, scene, w=W, h=H):
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(w, h)
    oframe = B.OracleFrame(B.OracleScene(scene), w, h)
    p = abi.default_frame_params(scene, w, h)
    p.enableBumpMapping = 1
    return oframe, p


def _gbuffer_same(ctx, oframe, p, tag):
    for buf in (abi.BUF_GBUFFER0, abi.BUF_GBUFFER1, abi.BUF_GBUFFER2, abi.BUF_GBUFFER3):
        _same(ctx.download(buf, p.bufferIndex), oframe.buffer(buf, p.bufferIndex), f"{tag} G-buffer {buf}")
    _same(ctx.download(abi.BUF_ALBEDO_ACCUM), oframe.buffer(abi.BUF_ALBEDO_ACCUM), f"{tag} albedo")
    _same(ctx.download(abi.BUF_NORMAL_ACCUM), oframe.buffer(abi.BUF_NORMAL_ACCUM), f"{tag} normal")


@pytest.mark.parametrize("unbiased", [False, True])
def test_gbuffer_and_restir_bit_exact(gfx_ctx, bumped, unbiased):
    oframe, p = _setup(gfx_ctx, bumped)
    for f in range(3):
        p.numAccumFrames = f
        gfx_ctx.build_light_distributions(f % 2)
        for kind, pid in engine.restir_frame_passes(p, f, 1, True, unbiased):
            if kind == "gbuffer":
                gfx_ctx.gbuffer(p)
                oframe.gbuffer(p)
                _gbuffer_same(gfx_ctx, oframe, p, f"frame {f}")
            else:
                gfx_ctx.restir(p, pid)
                oframe.restir(p, pid)
        _same(gfx_ctx.download(abi.BUF_RNG), oframe.buffer(abi.BUF_RNG), f"frame {f} rng")
        _same(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), oframe.buffer(abi.BUF_BEAUTY_ACCUM), f"frame {f} beauty")
    assert np.isfinite(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)).all()


def test_rearch_bit_exact(gfx_ctx, bumped):
    def configure(p):
        p.enableBumpMapping = 1
        return dict(temporal=True, spatial=True, unbiased=False)
    REARCH._run(gfx_ctx, B, bumped, W, H, 3, configure)  # the rearchitected passes on frames of the bump oracle


@pytest.mark.parametrize("variant", [abi.PT_BASELINE, abi.PT_REGIR])
def test_path_tracers_bit_exact(gfx_ctx, bumped, variant):
    oframe, p = _setup(gfx_ctx, bumped)
    for f in range(3):
        p.frameIndex, p.bufferIndex, p.numAccumFrames = f, f % 2, f
        gfx_ctx.build_light_distributions(f % 2)
        gfx_ctx.gbuffer(p)
        oframe.gbuffer(p)
        if variant == abi.PT_REGIR:
            gfx_ctx.regir_build_cells(p, f, f > 0)
            oframe.regir_build_cells(p, f, f > 0)
        gfx_ctx.pathtrace(p, variant)
        oframe.pathtrace(p, variant)
        if variant == abi.PT_REGIR:
            gfx_ctx.regir_update_access(p, f)
            oframe.regir_update_access(p, f)
        _same(gfx_ctx.download(abi.BUF_RNG), oframe.buffer(abi.BUF_RNG), f"frame {f} rng")
        _same(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), oframe.buffer(abi.BUF_BEAUTY_ACCUM), f"frame {f} beauty")
    beauty = gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)[..., :3]
    assert np.isfinite(beauty).all() and beauty.mean() > 1e-3


def test_nrc_frame_bit_exact(gfx_ctx, oracle, bumped):
    """path tracer (training records, counters, queries), inference, accumulation (beauty) and propagation"""
    oframe, p = _setup(gfx_ctx, bumped)
    gfx_ctx.build_light_distributions(0)
    net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    onet = oracle.OracleNrc(2, 1e-2)
    params = engine.random_nrc_params(net.num_params, onet.num_matrix_weights, grid_amplitude=0.1)
    net.set_params(params)
    onet.set_params(params)
    p.radianceScale = 2.0
    rng = np.random.default_rng(11)
    for f in range(3):
        p.frameIndex, p.bufferIndex, p.numAccumFrames = f, f % 2, f
        offsets = [int(rng.integers(0, 2 ** 32)) for _ in range(2)]
        gfx_ctx.gbuffer(p)
        gfx_ctx.nrc_preprocess(p, offsets[0], offsets[1], f == 0)
        gfx_ctx.pathtrace(p, abi.PT_NRC)
        oframe.gbuffer(p)
        oframe.nrc_preprocess(p, offsets[0], offsets[1], f == 0)
        oframe.pathtrace(p, abi.PT_NRC)
        ntrain, _, _ = NRC._compare_pathtrace(gfx_ctx, oframe, p, f"frame {f}")
        gfx_ctx.nrc_frame_infer(net)
        oframe.linear_buffer(abi.BUF_NRC_INFERRED_RADIANCE, copy=False)[:] = gfx_ctx.download_linear(abi.BUF_NRC_INFERRED_RADIANCE)
        gfx_ctx.nrc_accumulate(p)
        oframe.nrc_accumulate(p)
        _same(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM), oframe.buffer(abi.BUF_BEAUTY_ACCUM), f"frame {f} beauty")
        gfx_ctx.nrc_propagate(p)
        oframe.nrc_propagate(p)
        _same(gfx_ctx.download_linear(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain], oframe.linear_buffer(abi.BUF_NRC_TRAIN_TARGET, 0)[:ntrain],
              f"frame {f} propagated targets")
    net.close()


def test_nrc_visualize_prediction_bit_exact(gfx_ctx, bumped):
    net, p = NRCV._setup(gfx_ctx, bumped, W, H)
    p.enableBumpMapping = 1
    oframe = B.OracleFrame(B.OracleScene(bumped), W, H)
    n = W * H
    for f in range(2):
        p.numAccumFrames = f
        gfx_ctx.build_light_distributions(f % 2)
        gfx_ctx.nrc_frame(net, p, f, NRCV._offsets(f), train=True)
        NRCV._sentinel_queries(gfx_ctx)
        gfx_ctx.pathtrace(p, abi.PT_NRC_VISUALIZE_PREDICTION)
        oframe.gbuffer(p)
        oframe.nrc_visualize_prediction(p)
        ti = gfx_ctx.download_linear(abi.BUF_NRC_TERMINAL_INFO)
        _same(ti, oframe.linear_buffer(abi.BUF_NRC_TERMINAL_INFO), f"frame {f} terminal info")
        hit = (ti[:, 3] & 1).astype(bool)
        assert hit.mean() > 0.3
        _same(gfx_ctx.download_linear(abi.BUF_NRC_INFERENCE_QUERY)[:n][hit], oframe.linear_buffer(abi.BUF_NRC_INFERENCE_QUERY)[:n][hit],
              f"frame {f} queries")
    net.close()


def test_full_size_frame_on_an_oracle_strip(gfx_ctx, bumped):
    """1920x1080: the G-buffer and one ReSTIR frame against the oracle on rows 500..579, compared on the inner rows 530..549
    (whose 20-pixel spatial neighbourhood lies inside the strip)"""
    w, h = 1920, 1080
    oframe, p = _setup(gfx_ctx, bumped, w, h)
    po = abi.default_frame_params(bumped, w, h)
    po.enableBumpMapping = 1
    po.tileOriginY, po.tileRows = 500, 80
    gfx_ctx.build_light_distributions(0)
    for kind, pid in engine.restir_frame_passes(p, 0, 1, True, False):
        gfx_ctx.gbuffer(p) if kind == "gbuffer" else gfx_ctx.restir(p, pid)
    for kind, pid in engine.restir_frame_passes(po, 0, 1, True, False):
        oframe.gbuffer(po) if kind == "gbuffer" else oframe.restir(po, pid)
    for buf in (abi.BUF_GBUFFER0, abi.BUF_GBUFFER2, abi.BUF_GBUFFER3):
        _same(gfx_ctx.download(buf, 0)[500:580], oframe.buffer(buf, 0)[500:580], f"G-buffer {buf}")
    _same(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)[530:550], oframe.buffer(abi.BUF_BEAUTY_ACCUM)[530:550], "beauty")


def _frame_buffers(ctx, scene, bump):
    """every buffer of a ReSTIR, a path-traced and an NRC frame of `scene`"""
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(W, H)  # seeds the RNG
    p = abi.default_frame_params(scene, W, H)
    p.enableBumpMapping = bump
    out = []
    ctx.build_light_distributions(0)
    for kind, pid in engine.restir_frame_passes(p, 0, 1, True, False):
        ctx.gbuffer(p) if kind == "gbuffer" else ctx.restir(p, pid)
    out += [ctx.download(b, i) for b in (abi.BUF_GBUFFER0, abi.BUF_GBUFFER1, abi.BUF_GBUFFER2, abi.BUF_GBUFFER3,
                                         abi.BUF_RESERVOIR, abi.BUF_RESERVOIR_INFO) for i in (0, 1)]
    out += [ctx.download(b) for b in (abi.BUF_RNG, abi.BUF_BEAUTY_ACCUM, abi.BUF_ALBEDO_ACCUM, abi.BUF_NORMAL_ACCUM)]
    p.numAccumFrames = 0
    ctx.gbuffer(p)
    ctx.pathtrace(p, abi.PT_BASELINE)
    out += [ctx.download(abi.BUF_BEAUTY_ACCUM), ctx.download(abi.BUF_RNG)]
    ctx.nrc_preprocess(p, 12345, 678, True)
    ctx.pathtrace(p, abi.PT_NRC)
    out += [ctx.download_linear(b) for b in (abi.BUF_NRC_TERMINAL_INFO, abi.BUF_NRC_FRAME_CONTRIBUTION, abi.BUF_NRC_STATE)]
    out += [ctx.download(abi.BUF_RNG)]
    return out


def test_switch_off_equals_no_bump_table(gfx_ctx, bumped):
    plain = scenes.small_city_scene_bumped()
    plain.bump_maps = None
    off = _frame_buffers(gfx_ctx, bumped, 0)
    ref = _frame_buffers(gfx_ctx, plain, 0)
    for k, (a, b) in enumerate(zip(off, ref)):
        _same(a, b, f"buffer #{k}")
    on = _frame_buffers(gfx_ctx, bumped, 1)
    assert not np.array_equal(on[6].view(np.uint32), off[6].view(np.uint32))  # the shading normals of G-buffer 3 move


def _bump_debug(ctx, op, mat, inp, width):
    import torch
    a = torch.from_numpy(np.ascontiguousarray(inp, dtype=np.float32)).cuda()
    out = torch.zeros((a.shape[0], width), dtype=torch.float32, device="cuda")
    ctx._check(ctx.lib.gfx_bump_debug(ctx.h, None, op, mat, a.data_ptr(), a.shape[0], out.data_ptr()), "gfx_bump_debug")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _fraction_ties(scene, tex, rng):
    """coordinates whose footprint fraction in u is exactly 255.5 / 256 or one float either side (where the texture unit's 8-bit
    position decides whether the footprint moves on), with random v"""
    w = 1 if tex == abi.NO_BUMP_MAP else scene.textures[tex].shape[1]
    out = []
    for i in range(w):
        u0 = np.float32((i + 0.5 + 255.5 / 256) / w)
        for k in range(-40, 41):
            u = np.float32(u0 + np.float32(k) * np.spacing(u0))
            xB = (u - np.floor(u)) * np.float32(w) - np.float32(0.5)
            f = (xB - np.floor(xB)) * np.float32(256)
            if abs(float(f) - 255.5) <= 2e-3:
                out.append((u, rng.uniform(-2.0, 3.0)))
    assert out
    return np.asarray(out, dtype=np.float32)


def _in_tie_band(scene, tex, coords):
    H, W = (1, 1) if tex == abi.NO_BUMP_MAP else scene.textures[tex].shape[:2]
    band = np.zeros(coords.shape[0], dtype=bool)
    for c, n in ((coords[:, 0], W), (coords[:, 1], H)):
        xB = (c - np.floor(c)) * np.float32(n) - np.float32(0.5)
        band |= np.abs((xB - np.floor(xB)).astype(np.float64) * 256 - 255.5) < 0.01
    return band


def test_software_gather_equals_texture_unit(gfx_ctx, bumped):
    """tex2Dgather on a uchar4 cudaArray (normalised float, wrap, linear) returns exactly the texels the kernels' software
    gather picks, in the same order - for every map of the scene and the default texel; and the device's readModifiedNormal /
    applyBumpMapping equal the oracle's"""
    gfx_ctx.upload_scene(bumped)
    oscene = B.OracleScene(bumped, build_bvh=False)
    rng = np.random.default_rng(4)
    uv = rng.uniform(-3.0, 4.0, (200000, 2)).astype(np.float32)
    uv[:4096] = (rng.integers(-64, 64, (4096, 2)) / np.float32(64)).astype(np.float32)  # on and next to texel boundaries
    mats = {}
    for m in range(bumped.materials.shape[0]):
        mats.setdefault(int(bumped.bump_maps[m, 0]), m)
    assert len(mats) == 5
    for tex, m in mats.items():
        coords = np.concatenate([uv, _fraction_ties(bumped, tex, rng)])
        g = _bump_debug(gfx_ctx, 2, m, coords, 8)
        # Within 0.01 / 256 texel of the fraction 255.5 / 256 the texture unit's own fixed-point position decides whether the
        # footprint moves on, and a float32 restatement cannot know it; everywhere else the four texels and their order agree.
        band = _in_tie_band(bumped, tex, coords)
        _same(g[~band, :4], g[~band, 4:], f"texture {tex}: software vs hardware gather")
        assert band.sum() < 1000 and band[:uv.shape[0]].mean() < 1e-3
        for op, width in ((0, 3), (2, 4)):
            want = oscene.bump_query(op, m, uv, width)
            _same(_bump_debug(gfx_ctx, op, m, uv, 8 if op == 2 else 3)[:, :width], want, f"texture {tex} op {op}")
    frames = rng.normal(size=(50000, 12)).astype(np.float32)
    frames[:1000, :2] *= np.float32(1e-4)
    want = oscene.bump_query(1, 0, frames, 9)
    _same(_bump_debug(gfx_ctx, 1, 0, frames, 9), want, "applyBumpMapping")


def test_cpp_host_bump_mapping_matches_python_host(gfx_ctx, tmp_path, monkeypatch):
    """gfx_headless -bump-mapping: the scene file carries no textures, so every material reads the default texel"""
    scene = scenes.tiny_city_scene()
    scene_path = str(tmp_path / "scene.bin")
    scenes.save_scene_bin(scene, scene_path, HOSTS.W, HOSTS.H)  # the file's defaults keep the switch off
    params_path = str(tmp_path / "nrc.f16")
    probe = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2)
    engine.random_nrc_params(probe.num_params, 64 * 64 * 2 + 16 * 64, grid_amplitude=0.1).tofile(params_path)
    probe.close()
    default_frame_params = abi.default_frame_params

    def with_bump(*args, **kwargs):
        p = default_frame_params(*args, **kwargs)
        p.enableBumpMapping = 1
        return p
    monkeypatch.setattr(abi, "default_frame_params", with_bump)
    for renderer in ("restir", "pathtrace", "regir", "nrc"):
        out_path = str(tmp_path / f"{renderer}.raw")
        cmd = [HOSTS.HOST, scene_path, renderer, str(HOSTS.W), str(HOSTS.H), str(HOSTS.FRAMES), out_path]
        cmd += ([params_path] if renderer == "nrc" else []) + ["-bump-mapping"]
        res = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stderr
        got = np.fromfile(out_path, dtype=np.float32).reshape(HOSTS.H, HOSTS.W, 4)
        want = HOSTS._python_host(gfx_ctx, scene, renderer)
        _same(got, want, f"{renderer}: C++ host with -bump-mapping vs Python host")
        monkeypatch.setattr(abi, "default_frame_params", default_frame_params)
        off = HOSTS._python_host(gfx_ctx, scene, renderer)
        monkeypatch.setattr(abi, "default_frame_params", with_bump)
        assert not np.array_equal(got.view(np.uint32), off.view(np.uint32)), f"{renderer}: the switch changed nothing"
    assert os.path.exists(HOSTS.HOST)
