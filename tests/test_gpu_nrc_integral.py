"""The library's NRC frame against the closed form of tests/nrc_integral.py: an emissive box seen from inside, with the network
installed as the exact cache radianceScale * L (never trained).  The grouping rule and the bound (5 SE + 1e-4 L) are the
helper's.

Sizes: 97x61 (ragged tiles), 192x108, and 1920x1080 with the tile size seeded to 4, which fills the record buffer during the
second round, so that most training suffixes end in the buffer-full branch (k_nrcCommitScatter's suffix query); both position
encodings; maxPathLength 0, radianceScale 2, several frames with different tile offsets.

  pixels after gfx_nrc_frame_infer + gfx_nrc_accumulate: training pixels of biased tiles, of unbiased tiles, the other pixels
  records after gfx_nrc_propagate: the targets by record path length (1, 2, 3-5, >= 6) and tile class; all finite and >= 0
  shuffle: buffer 1 is buffer 0 permuted by the shufflers' LCG (restated in numpy) and scaled by radianceScale, bit for bit;
  target min / max exact, the float-atomic average within 1e-4 relative
  ReSTIR DI + NRC: unbiased ReSTIR DI, GFX_PT_NRC_INDIRECT and the additive accumulate over 8 frames, through the context's
  launches and through StripDriver.render_restir_nrc_frame(combined=True)
  control: the baseline path tracer at maxPathLength 2, 4 and 0 (= 5) averages e * sum_{k<n} rho^k
  negative controls: a cache scaled by 0.9 and the double count of training pixels whose rendering path ended in the cache
  (restated in expectation over the buffers) fail the same bound"""
import numpy as np
import pytest

from gfxexp_b200 import abi, engine, multigpu
from tests import nrc_integral as I

pytestmark = pytest.mark.gpu

HASH, TRIWAVE = abi.NRC_POSITION_ENCODING_HASH_GRID, abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE
# (width, height, frames, seeded tile size)
SIZES = {"97x61": (97, 61, 16, None), "192x108": (192, 108, 8, None), "1920x1080": (1920, 1080, 3, 4)}


def _failures(rows):
    return [r for r in rows if not r[5]]


@pytest.mark.parametrize("encoding", [HASH, TRIWAVE])
@pytest.mark.parametrize("size", list(SIZES))
def test_nrc_frame_averages_the_closed_form(gfx_ctx, size, encoding):
    w, h, frames, tile = SIZES[size]
    scene = I.emissive_box_scene()
    b = I.GpuBackend(gfx_ctx, scene, w, h, encoding)
    pixels, records, doubled, full = I.run_nrc(b, scene, w, h, frames, seed_tile=tile)
    b.close()
    rows = pixels.report() + records.report(min_n=10)
    print(f"{size} encoding {encoding}\n" + I.format_report(rows))
    names = {r[0] for r in rows}
    assert {"training pixels, biased tiles", "training pixels, unbiased tiles", "other pixels"} <= names
    assert {"records of length 1, biased tiles", "records of length 2, biased tiles", "records of length 1, unbiased tiles"} <= names
    assert not _failures(rows), I.format_report(rows)
    if tile is not None:
        assert full == frames, "the record buffer did not fill"
    bad = {r[0] for r in _failures(doubled.report())}
    assert {"training pixels, biased tiles", "training pixels, unbiased tiles"} <= bad, I.format_report(doubled.report())
    assert "other pixels" not in bad


def test_nrc_frame_with_a_wrong_cache_fails(gfx_ctx):
    scene = I.emissive_box_scene()
    b = I.GpuBackend(gfx_ctx, scene, 192, 108, HASH)
    pixels, records, _, _ = I.run_nrc(b, scene, 192, 108, 4, cache_scale=0.9)
    b.close()
    bad = {r[0] for r in _failures(pixels.report() + records.report(min_n=10))}
    assert {"other pixels", "training pixels, biased tiles", "records of length 1, biased tiles"} <= bad, bad


def _frame_values(beauties):
    """each frame's own estimate D + I from the running mean: B_f = (1 - w) B_{f-1} + w (D + I), w = 1 / (1 + f)"""
    out, prev = [], None
    for f, b in enumerate(beauties):
        b = b.astype(np.float64)
        w = 1.0 / (1 + f)
        out.append(b if prev is None else (b - (1 - w) * prev) / w)
        prev = b
    return out


@pytest.mark.parametrize("driver", ["context", "strip_driver"])
def test_restir_nrc_frame_averages_the_closed_form(gfx_ctx, driver):
    """8 frames of unbiased ReSTIR DI (temporal reuse, no spatial pass, so pixels stay independent of each other) + the NRC
    light beyond the primary vertex; a pixel's frames are correlated by the temporal reuse, so the pixel is the unit of the SE"""
    w, h, frames = 192, 108, 8
    scene = I.emissive_box_scene()
    b = I.GpuBackend(gfx_ctx, scene, w, h, HASH)
    value = I.RADIANCE_SCALE * I.L
    b.set_params(I.constant_params(b.num_params, b.num_matrix_weights, 2, value))
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = 0
    p.radianceScale = I.RADIANCE_SCALE
    strip = None
    if driver == "strip_driver":
        strip = multigpu.StripDriver(gfx_ctx, p, w, h, 0, 1)
        strip.enable_nrc(b.net, overlap_training=False)
    beauties, flags = [], []
    for f in range(frames):
        p.numAccumFrames = f
        off = I.offsets(f)
        if strip is not None:
            strip.render_restir_nrc_frame(f, off, num_spatial_passes=0, unbiased=True, train=False, combined=True)
        else:
            gfx_ctx.build_light_distributions(f % 2)
            for kind, pid in engine.restir_frame_passes(p, f, 0, True, True):
                gfx_ctx.gbuffer(p) if kind == "gbuffer" else gfx_ctx.restir(p, pid)
            gfx_ctx.nrc_preprocess(p, off[0], off[1], f == 0)
            gfx_ctx.pathtrace(p, abi.PT_NRC_INDIRECT)
            gfx_ctx.nrc_frame_infer(b.net)
            gfx_ctx.nrc_accumulate(p)
        gfx_ctx.synchronize()
        beauties.append(gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)[..., :3].reshape(-1, 3))
        flags.append(gfx_ctx.download_linear(abi.BUF_NRC_TERMINAL_INFO))
    b.close()
    s = I.Samples()
    ids = np.arange(w * h)
    for v, ti in zip(_frame_values(beauties), flags):
        assert np.isfinite(v).all()
        for name, sel in I.pixel_groups(ti).items():
            s.add(name, v[sel], ids[sel])
    rows = s.report()
    print(f"ReSTIR DI + NRC ({driver})\n" + I.format_report(rows))
    assert len(rows) == 9 and not _failures(rows), I.format_report(rows)


@pytest.mark.parametrize("max_path_length", [2, 4, 0])
def test_baseline_path_tracer_control(gfx_ctx, max_path_length):
    w, h = 192, 108
    scene = I.emissive_box_scene()
    b = I.GpuBackend(gfx_ctx, scene, w, h, HASH)
    rows = I.run_baseline(b, scene, w, h, 8, max_path_length).report(I.baseline_series(max_path_length))
    b.close()
    assert not _failures(rows), I.format_report(rows)
