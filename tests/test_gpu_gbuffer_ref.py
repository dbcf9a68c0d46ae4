"""The device's G-buffer pass (gfxexp_b200/csrc/gbuffer.cu) on the seeded scenes of tests/gbuffer_scenes.py: bit for bit
against the oracle on every kernel form - k_gbuffer<false / true> (bump off / on) and k_gbufferSubPixelJitter<false / true> -
at the CPU test's sizes and strips, the form no oracle covers (the TAA jitter with the bump) against the float64 restatement
(tests/gbuffer_ref.py), a 1920x1080 frame within the restatement's bars on row windows, and the ray counter on partial tiles."""
import numpy as np
import pytest

from gfxexp_b200 import abi
from tests import gbuffer_ref as R, gbuffer_scenes as S, oracle_bump, oracle_lib, oracle_svgf_taa_jitter
from tests.test_oracle_gbuffer_ref import PLANES, SENTINEL, SIZES, check, frame_params

pytestmark = pytest.mark.gpu


def _device(ctx, sc, W, H, seed=591842031321323413):
    """the scene and a frame whose G-buffer planes hold SENTINEL (the PCG32 states keep their seeding)"""
    ctx.upload_scene(sc)
    ctx.build_bvh()
    ctx.create_frame(W, H, seed)
    for b in PLANES[:-1]:
        dtype, comps, _ = abi.BUFFER_LAYOUT[b]
        for idx in (0, 1) if b < abi.BUF_RNG else (0,):
            ctx.upload(b, idx, np.full(H * W * comps * np.dtype(dtype).itemsize // 4, SENTINEL, np.uint32))


def _dev_planes(ctx, idx=0):
    return {b: ctx.download(b, idx if b < abi.BUF_RNG else 0) for b in PLANES}


def _same(dev, orc, what):
    for b in PLANES:
        got, want = dev[b].view(np.uint32), orc[b].view(np.uint32)
        assert np.array_equal(got, want), f"{what}: buffer {b} differs at {np.count_nonzero(got != want)} words"


def _oracle_frame(form, sc, W, H, seed=591842031321323413):
    if form in ("bump", "taa_bump"):
        return oracle_bump.OracleFrame(oracle_bump.OracleScene(sc), W, H, seed)
    if form == "taa":
        return oracle_svgf_taa_jitter.Frame(sc, W, H, seed)
    return oracle_lib.OracleFrame(oracle_lib.OracleScene(sc), W, H, seed)


def _params(form, sc, W, H):
    p = frame_params(sc, W, H)
    if form in ("bump", "taa_bump"):
        p.enableBumpMapping = 1
    if form in ("taa", "taa_bump"):
        p.svgfFlags = abi.SVGF_ENABLE_TAA | abi.SVGF_SUBPIXEL_JITTER
        p.taaHistoryLength, p.frameIndex = 4, 6
    if form == "jitter":
        p.enableJittering = 1
    return p


@pytest.mark.parametrize("form", ["plain", "jitter", "bump", "taa"])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_bit_exact_with_oracle(gfx_ctx, form, size):
    """k_gbuffer<false> (plain, enableJittering), k_gbuffer<true> (bump), k_gbufferSubPixelJitter<false> (taa)"""
    W, H = size
    sc = S.scene(bump=form == "bump")
    _device(gfx_ctx, sc, W, H)
    f = _oracle_frame(form, sc, W, H)
    if form == "jitter":
        gfx_ctx.upload(abi.BUF_RNG, 0, f.buffer(abi.BUF_RNG, 0))
    p = _params(form, sc, W, H)
    gfx_ctx.read_stats(reset=True)
    gfx_ctx.gbuffer(p)
    f.gbuffer(p)
    _same(_dev_planes(gfx_ctx), {b: f.buffer(b, 0) for b in PLANES}, f"{form} {W}x{H}")
    assert gfx_ctx.read_stats()[0] == W * H


def test_taa_jitter_with_bump_equals_restatement(gfx_ctx):
    """k_gbufferSubPixelJitter<true>: no oracle restates the TAA jitter together with the bump"""
    W, H = 67, 45
    sc = S.scene(bump=True)
    _device(gfx_ctx, sc, W, H)
    p = _params("taa_bump", sc, W, H)
    gfx_ctx.gbuffer(p)
    check(R.gbuffer(R.Scene64(sc), p, W, H, bump=True), _dev_planes(gfx_ctx), "taa + bump")


@pytest.mark.parametrize("form", ["plain", "jitter", "bump", "taa"])
@pytest.mark.parametrize("strip", [(3, 6), (11, 40), (22, 1)], ids=lambda s: f"{s[0]}+{s[1]}")
def test_strips_bit_exact_with_oracle(gfx_ctx, form, strip):
    """strips that start off the 8-row block grid and run past H: the oracle's bits inside, the sentinel outside, and one ray
    counted per pixel of the strip although the partial tiles' lanes outside the image run countRays too"""
    W, H = 29, 23
    sc = S.scene(bump=form == "bump")
    _device(gfx_ctx, sc, W, H)
    p = _params(form, sc, W, H)
    p.tileOriginY, p.tileRows = strip
    rng_in = gfx_ctx.download(abi.BUF_RNG, 0)
    gfx_ctx.read_stats(reset=True)
    gfx_ctx.gbuffer(p)
    dev = _dev_planes(gfx_ctx)
    y1 = min(H, strip[0] + strip[1])
    assert gfx_ctx.read_stats()[0] == W * (y1 - strip[0])
    for b in PLANES:
        v = dev[b].view(np.uint32)
        keep = rng_in.view(np.uint32) if b == abi.BUF_RNG else np.full_like(v, SENTINEL)
        assert (v[:strip[0]] == keep[:strip[0]]).all() and (v[y1:] == keep[y1:]).all(), b
    ref = R.gbuffer(R.Scene64(sc), p, W, H, rng_in=rng_in, bump=form == "bump")
    check(ref, dev, f"{form} strip {strip}")
    f = _oracle_frame(form, sc, W, H)
    if form == "jitter":
        f.buffer(abi.BUF_RNG, 0, copy=False)[...] = rng_in
    f.gbuffer(p)
    for b in PLANES:
        got, want = dev[b].view(np.uint32)[strip[0]:y1], f.buffer(b, 0).view(np.uint32)[strip[0]:y1]
        assert np.array_equal(got, want), f"{form} strip {strip}: buffer {b}"


def test_two_animated_frames_bit_exact(gfx_ctx):
    from tests.test_oracle_gbuffer_ref import _animated
    sc = S.scene()
    W, H = 61, 41
    osc = oracle_lib.OracleScene(sc)
    f = oracle_lib.OracleFrame(osc, W, H)
    _device(gfx_ctx, sc, W, H)
    gfx_ctx.gbuffer(frame_params(sc, W, H))
    sc1, moved, p1 = _animated(sc, osc, W, H, f)
    gfx_ctx.update_instances(abi.make_instance_descs(moved))
    gfx_ctx.build_bvh()
    gfx_ctx.gbuffer(p1)
    f.gbuffer(p1)
    dev = _dev_planes(gfx_ctx, 1)
    orc = {b: f.buffer(b, 1 if b < abi.BUF_RNG else 0) for b in PLANES}
    _same(dev, orc, "frame 1")
    check(R.gbuffer(R.Scene64(sc1, prev_instances=sc.instances), p1, W, H), dev, "frame 1")


@pytest.mark.parametrize("form", ["plain", "bump", "taa"])
def test_1080p_within_restatement(gfx_ctx, form):
    """a 1920x1080 frame: the first, a middle and the last 8 rows within the restatement's bars"""
    W, H = 1920, 1080
    sc = S.scene(bump=form == "bump")
    _device(gfx_ctx, sc, W, H)
    p = _params(form, sc, W, H)
    gfx_ctx.read_stats(reset=True)
    gfx_ctx.gbuffer(p)
    assert gfx_ctx.read_stats()[0] == W * H
    dev = _dev_planes(gfx_ctx)
    s64 = R.Scene64(sc)
    for y0 in (0, 536, H - 8):
        check(R.gbuffer(s64, p, W, H, rows=(y0, y0 + 8), bump=form == "bump"), dev, f"{form} 1080p rows {y0}")
