"""ctypes binding of oracle/liborc_views.so (oracle/views.cpp, built by oracle/Makefile.views) — TEST INFRASTRUCTURE.

The CPU restatement of the NRC and ReGIR apps' debug views: the views of gfx_present_launch on host copies of the buffers it
reads, the ReGIR cell colour, and the visualizePrediction pass.  The library carries its own copy of the oracle renderer, so
the pass runs on a ViewsFrame of this module (G-buffer + NRC buffers), not on an oracle_lib.OracleFrame.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gfxexp_b200 import abi
from tests import oracle_lib

LIB = os.path.join(oracle_lib.ORACLE_DIR, "liborc_views.so")
_lib = None


class OrcViewInputs(C.Structure):
    _fields_ = [("terminalInfo", C.c_void_p), ("inferredRadiance", C.c_void_p), ("inferenceQuery", C.c_void_p),
                ("gbuffer1", C.c_void_p), ("gbuffer2", C.c_void_p)]


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "Makefile.views"], stdout=subprocess.DEVNULL)
        L = C.CDLL(LIB)
        vp = C.c_void_p
        L.orc_present_views.argtypes = [vp, C.c_uint32, C.c_uint32, C.POINTER(abi.GfxPresentParams), C.POINTER(OrcViewInputs), vp]
        L.orc_regir_cell_color.argtypes = [C.POINTER(abi.GfxFrameParams), vp, C.c_uint32, vp]
        L.orc_scene_create.restype = vp
        L.orc_scene_create.argtypes = [C.POINTER(abi.GfxSceneDesc), C.POINTER(oracle_lib.OrcBuildConfig), C.c_int]
        L.orc_scene_destroy.argtypes = [vp]
        L.orc_frame_create.restype = vp
        L.orc_frame_create.argtypes = [vp, C.c_uint32, C.c_uint32]
        L.orc_frame_destroy.argtypes = [vp]
        L.orc_rng_seed.argtypes = [vp, C.c_uint64]
        L.orc_buffer_ptr.restype = vp
        L.orc_buffer_ptr.argtypes = [vp, C.c_int, C.c_uint32, C.POINTER(C.c_size_t)]
        L.orc_gbuffer.argtypes = [vp, C.POINTER(abi.GfxFrameParams), C.c_int]
        L.orc_nrc_visualize_prediction.argtypes = [vp, C.POINTER(abi.GfxFrameParams)]
        _lib = L
    return _lib


def present_views(params, mode: int, flags: int, rgba=None, terminal_info=None, inferred_radiance=None, inference_query=None,
                  gbuffer1=None, gbuffer2=None, brightness_scale: float = 1.0, alpha_override: float = 1.0,
                  motion_vector_scale: float = 0.1, motion_vector_offset: float = 0.5, width: int = 0,
                  height: int = 0) -> np.ndarray:
    """the debug views of gfx_present_launch on host copies of the buffers it reads -> RGBA8 [H, W]; params = the
    GfxFrameParams the view is given, the buffers in their download layouts (None = not read)"""
    keep = []

    def ptr(a, dtype):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=dtype)
        keep.append(a)
        return a.ctypes.data

    h, w = (rgba.shape[:2] if rgba is not None else (height, width))
    out = np.empty((h, w), dtype=np.uint32)
    pp = abi.GfxPresentParams(0, 0, mode, flags, brightness_scale, alpha_override, C.pointer(params),
                              motion_vector_scale, motion_vector_offset)
    ins = OrcViewInputs(ptr(terminal_info, np.uint32), ptr(inferred_radiance, np.float32), ptr(inference_query, np.float32),
                        ptr(gbuffer1, np.float32), ptr(gbuffer2, np.float32))
    lib().orc_present_views(ptr(rgba, np.float32), w, h, C.byref(pp), C.byref(ins), out.ctypes.data_as(C.c_void_p))
    return out


def regir_cell_color(params, positions: np.ndarray) -> np.ndarray:
    """calcCellColor (regir/gpu_kernels/copy_buffers.cu:62-76) of [n, 3] positions over the ReGIR grid of params"""
    pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
    out = np.empty_like(pos)
    lib().orc_regir_cell_color(C.byref(params), pos.ctypes.data, pos.shape[0], out.ctypes.data)
    return out


class ViewsFrame:
    """a scene + frame of the views library: its G-buffer pass and the visualizePrediction pass"""

    def __init__(self, scene, width: int, height: int, seed: int = 591842031321323413):
        self.arrays = abi.SceneArrays(scene)
        self.cfg = oracle_lib.reference_build_config()
        self.scene = lib().orc_scene_create(C.byref(self.arrays.desc), C.byref(self.cfg), 0)
        assert self.scene
        self.W, self.H = width, height
        self.h = lib().orc_frame_create(self.scene, width, height)
        lib().orc_rng_seed(self.h, seed)

    def close(self):
        if self.h:
            lib().orc_frame_destroy(self.h)
            lib().orc_scene_destroy(self.scene)
            self.h = None

    def __del__(self):
        self.close()

    def gbuffer(self, params, threads: int = 0):
        lib().orc_gbuffer(self.h, C.byref(params), threads)

    def nrc_visualize_prediction(self, params):
        """GFX_PT_NRC_VISUALIZE_PREDICTION: the primary hits' radiance queries and the terminal infos"""
        lib().orc_nrc_visualize_prediction(self.h, C.byref(params))

    def buffer(self, buffer_id: int, index: int = 0) -> np.ndarray:
        nbytes = C.c_size_t()
        ptr = lib().orc_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        dtype, comps, _ = abi.BUFFER_LAYOUT[buffer_id]
        arr = np.frombuffer((C.c_uint8 * nbytes.value).from_address(ptr), dtype=dtype).copy()
        return arr.reshape(self.H, self.W, comps) if comps > 1 else arr.reshape(self.H, self.W)

    def linear_buffer(self, buffer_id: int, index: int = 0, copy: bool = True) -> np.ndarray:
        """NRC buffers as [rows, cols]; copy=False returns a writable view of the library's memory"""
        nbytes = C.c_size_t()
        ptr = lib().orc_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        dtype, cols, rows = abi.linear_buffer_layout(buffer_id, self.W, self.H)
        assert nbytes.value == rows * cols * np.dtype(dtype).itemsize, (buffer_id, nbytes.value, rows, cols)
        arr = np.frombuffer((C.c_uint8 * nbytes.value).from_address(ptr), dtype=dtype).reshape(rows, cols)
        return arr.copy() if copy else arr
