"""The shading layer on the GPU (gfx_shading_debug) equals shading.cuh built for the CPU (tests/cpp/shading_host.cpp) bit for
bit, over the inputs of test_shading_host.py: every grid material with REGULARIZE off and on, view directions on and below the
horizon, the PCG lattice and the u edges; and the warps, encoders, frames and ray offsets.  The CPU build is held to the oracle
and to float64 there, so this closes the chain from the device kernels to the reference's formulas."""
import numpy as np
import pytest

from tests import shading_ops as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def runners(gfx_ctx, tmp_path_factory):
    return S.build_host(tmp_path_factory.mktemp("shading_host")), S.device_runner(gfx_ctx)


def _same(host, dev, op, mat, rec, what):
    """bit for bit, except that a NaN equals a NaN: the x86 and sm_90a NaN payloads differ (0xFFC00000 / 0x7FFFFFFF)"""
    a, b = host(op, mat, rec), dev(op, mat, rec)
    differ = (a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b))
    bad = np.flatnonzero(differ.any(1))
    assert bad.size == 0, (f"{what} op {op}: {bad.size} records differ, first {rec[bad[0]].tolist()} -> host "
                           f"{a[bad[0]].tolist()} device {b[bad[0]].tolist()}")


@pytest.mark.parametrize("op", S.BSDF_OPS, ids=["evaluate", "evaluatePDF", "sampleThroughput", "DHReflectance"])
def test_bsdf_ops_bit_exact(runners, op):
    host, dev = runners
    for name, mat in S.materials():
        _same(host, dev, op, mat, S.bsdf_inputs(host, mat)[op], name)


@pytest.mark.parametrize("family", ["warps", "polar", "codes", "frames"])
def test_helper_ops_bit_exact(runners, family):
    host, dev = runners
    ops = {"warps": (S.CONCENTRIC_DISK, S.COSINE_HEMISPHERE), "polar": (S.TO_POLAR, S.FROM_POLAR, S.ENCODE_VECTOR, S.DECODE_VECTOR),
           "codes": (S.ENCODE_BARYCENTRIC, S.DECODE_BARYCENTRIC, S.ENCODE_TEXCOORDS, S.DECODE_TEXCOORDS),
           "frames": (S.COORDINATE_SYSTEM, S.OFFSET_RAY_ORIGIN)}[family]
    ins = S.helper_inputs()
    for op in ops:
        _same(host, dev, op, S.material(0, 0.0), ins[op], family)


def test_invalid_op_is_refused(gfx_ctx):
    import torch
    a = torch.zeros((4, 8), device="cuda")
    mat = S.material(0, 0.5)
    assert gfx_ctx.lib.gfx_shading_debug(gfx_ctx.h, None, 16, mat.ctypes.data, a.data_ptr(), 4, a.data_ptr()) != 0
    assert gfx_ctx.lib.gfx_shading_debug(gfx_ctx.h, None, -1, mat.ctypes.data, a.data_ptr(), 4, a.data_ptr()) != 0
