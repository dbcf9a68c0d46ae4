"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/gfxb200.h declares, and refuses to run without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from gfxexp_b200 import abi, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "gfxb200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(gfx_[a-z0-9_]+)\s*\(", text)))


def test_header_and_python_mirror_agree():
    assert _declared_symbols() == sorted(abi.EXPORTED_SYMBOLS)


def test_library_exports_every_declared_symbol():
    lib = abi.load_library()
    for name in _declared_symbols():
        assert hasattr(lib, name), f"{name} declared in gfxb200.h but not exported"


def test_trace_debug_hook():
    """gfx_trace_debug(ctx, stream, rays, n, hits, mode, kernel): the test hook of the three traversal kernels"""
    assert "gfx_trace_debug" in _declared_symbols()
    restype, argtypes = abi._DECLS["gfx_trace_debug"]
    assert restype is C.c_int and argtypes[-2:] == [C.c_int, C.c_int] and len(argtypes) == 7


def test_pod_sizes_match_reference_layouts():
    # CompressedInternalNode_T<8> 80 B, TriangleStorage 48 B, HitObject 32 B
    # (common/common_shared.h:915-917,1025,1065-1078)
    assert abi.NODE_DTYPE.itemsize == 80
    assert abi.TRI_DTYPE.itemsize == 48
    assert abi.HIT_DTYPE.itemsize == 32
    assert C.sizeof(abi.GfxMaterialDesc) == 48
    assert C.sizeof(abi.GfxInstanceDesc) == 4 * (12 + 12 + 9 + 1 + 2)
    assert C.sizeof(abi.GfxCamera) == 4 * 14


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(engine.GfxError):
        engine.Context(0)


def test_missing_library_fails_loudly(tmp_path):
    with pytest.raises(OSError):
        abi.load_library(str(tmp_path / "nope.so"))
