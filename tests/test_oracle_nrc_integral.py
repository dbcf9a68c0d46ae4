"""The CPU oracle's NRC frame (oracle/nrc_pathtrace.inl) against the closed form of tests/nrc_integral.py: an emissive box
seen from inside, with a network installed as the exact cache radianceScale * L.  The grouping rule and the bound (5 SE +
1e-4 L) are the helper's; tests/test_gpu_nrc_integral.py runs the same checks on the library at frame sizes up to 1080p.

  pixels: training pixels of biased tiles, of unbiased tiles, and the other pixels each average L
  records: the propagated training targets, by record path length and tile class, average L; all finite and >= 0
  shuffle: buffer 1 is buffer 0 permuted by the shufflers' LCG and scaled by radianceScale, bit for bit; target min / max
  negative controls: a cache scaled by 0.9 and the double count of training pixels whose rendering path ended in the cache
  (restated in expectation over the buffers) fail the same bound
  control: the baseline path tracer at maxPathLength 2, 4 and 0 (= 5) averages e * sum_{k<n} rho^k"""
import numpy as np
import pytest

from gfxexp_b200 import abi
from tests import nrc_integral as I

W, H, FRAMES = 160, 96, 8


def _failures(rows):
    return [r for r in rows if not r[5]]


@pytest.mark.parametrize("encoding", [abi.NRC_POSITION_ENCODING_HASH_GRID, abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE])
def test_nrc_frame_averages_the_closed_form(oracle, encoding):
    scene = I.emissive_box_scene()
    b = I.OracleBackend(scene, W, H, encoding)
    pixels, records, doubled, _ = I.run_nrc(b, scene, W, H, FRAMES)
    rows = pixels.report() + records.report(min_n=10)
    assert not _failures(rows), I.format_report(rows)
    # the double count inflates the training pixels whose rendering path ended in the cache
    rows = doubled.report()
    bad = {r[0] for r in _failures(rows)}
    assert {"training pixels, biased tiles", "training pixels, unbiased tiles"} <= bad, I.format_report(rows)
    assert "other pixels" not in bad, I.format_report(rows)


def test_nrc_frame_with_a_wrong_cache_fails(oracle):
    scene = I.emissive_box_scene()
    b = I.OracleBackend(scene, W, H, abi.NRC_POSITION_ENCODING_HASH_GRID)
    pixels, records, _, _ = I.run_nrc(b, scene, W, H, 4, cache_scale=0.9)
    bad = {r[0] for r in _failures(pixels.report() + records.report(min_n=10))}
    assert {"other pixels", "training pixels, biased tiles", "records of length 1, biased tiles"} <= bad, bad


@pytest.mark.parametrize("max_path_length", [2, 4, 0])
def test_baseline_path_tracer_control(oracle, max_path_length):
    scene = I.emissive_box_scene()
    b = I.OracleBackend(scene, W, H, abi.NRC_POSITION_ENCODING_HASH_GRID)
    rows = I.run_baseline(b, scene, W, H, 4, max_path_length).report(I.baseline_series(max_path_length))
    assert not _failures(rows), I.format_report(rows)


def test_buffer_full_suffixes_average_the_closed_form(oracle):
    """1080p with 4x4 tiles: the record buffer fills during the second round, so most training suffixes end in the buffer-full
    branch with a query at their staged vertex while the path traces on; the vertices after it must feed no record"""
    scene = I.emissive_box_scene()
    b = I.OracleBackend(scene, 1920, 1080, abi.NRC_POSITION_ENCODING_HASH_GRID)
    pixels, records, _, full = I.run_nrc(b, scene, 1920, 1080, 1, seed_tile=4)
    assert full == 1
    rows = pixels.report() + records.report(min_n=10)
    assert not _failures(rows), I.format_report(rows)
