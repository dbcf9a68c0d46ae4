"""ctypes binding of oracle/liborc_bump.so (oracle/bump.cpp, built by oracle/Makefile.bump) — TEST INFRASTRUCTURE.

The CPU restatement of the bump mapping (GfxFrameParams::enableBumpMapping, GfxSceneDesc::bumpMaps).  The library carries its
own copy of the oracle renderer whose G-buffer pass, path tracers and visualizePrediction pass tilt the shading frames, so a
frame with bump mapping runs on an OracleScene / OracleFrame of this module (the same methods as oracle_lib's), not on
oracle_lib's.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gfxexp_b200 import abi
from tests import oracle_lib
from tests.oracle_lib import ORC_NOT_READY

LIB = os.path.join(oracle_lib.ORACLE_DIR, "liborc_bump.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "Makefile.bump"], stdout=subprocess.DEVNULL)
        L = C.CDLL(LIB)
        vp, pp = C.c_void_p, C.POINTER(abi.GfxFrameParams)
        L.orc_scene_create.restype = vp
        L.orc_scene_create.argtypes = [C.POINTER(abi.GfxSceneDesc), C.POINTER(oracle_lib.OrcBuildConfig), C.c_int]
        L.orc_scene_destroy.argtypes = [vp]
        L.orc_bump_attach.argtypes = [vp, C.POINTER(abi.GfxSceneDesc)]
        L.orc_bump_detach.argtypes = [vp]
        L.orc_bump_query.restype = C.c_int
        L.orc_bump_query.argtypes = [vp, C.c_int, C.c_uint32, vp, C.c_uint32, vp]
        L.orc_bump_dm_atan.argtypes = [vp, vp, C.c_size_t]
        L.orc_frame_create.restype = vp
        L.orc_frame_create.argtypes = [vp, C.c_uint32, C.c_uint32]
        L.orc_frame_destroy.argtypes = [vp]
        L.orc_rng_seed.argtypes = [vp, C.c_uint64]
        L.orc_restir_setup_neighbor_table.argtypes = [vp]
        L.orc_buffer_ptr.restype = vp
        L.orc_buffer_ptr.argtypes = [vp, C.c_int, C.c_uint32, C.POINTER(C.c_size_t)]
        L.orc_bump_gbuffer.argtypes = [vp, pp, C.c_int]
        L.orc_restir.argtypes = [vp, pp, C.c_int, C.c_int]
        L.orc_restir_rearch.restype = C.c_uint64
        L.orc_restir_rearch.argtypes = [vp, pp, C.c_int, C.c_int]
        L.orc_bump_pathtrace.restype = C.c_uint64
        L.orc_bump_pathtrace.argtypes = [vp, pp, C.c_int, C.c_int]
        L.orc_regir_build_cells.argtypes = [vp, pp, C.c_uint32, C.c_int, C.c_int]
        L.orc_regir_update_access.argtypes = [vp, pp, C.c_uint32]
        L.orc_nrc_preprocess.argtypes = [vp, pp, C.c_uint32, C.c_uint32, C.c_int]
        for name in ("orc_nrc_accumulate", "orc_nrc_propagate", "orc_nrc_shuffle", "orc_bump_nrc_visualize_prediction"):
            getattr(L, name).argtypes = [vp, pp]
        _lib = L
    return _lib


def dm_atan(x: np.ndarray) -> np.ndarray:
    x = np.ascontiguousarray(x, dtype=np.float32)
    y = np.empty_like(x)
    lib().orc_bump_dm_atan(x.ctypes.data, y.ctypes.data, x.size)
    return y


class OracleScene:
    def __init__(self, scene, cfg=None, build_bvh: bool = True):
        self.arrays = abi.SceneArrays(scene)
        self.cfg = cfg or oracle_lib.reference_build_config()
        self.h = lib().orc_scene_create(C.byref(self.arrays.desc), C.byref(self.cfg), 0 if build_bvh else -1)
        assert self.h
        lib().orc_bump_attach(self.h, C.byref(self.arrays.desc))

    def close(self):
        if self.h:
            lib().orc_bump_detach(self.h)
            lib().orc_scene_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def bump_query(self, op: int, mat: int, inp: np.ndarray, width: int) -> np.ndarray:
        """op 0 readModifiedNormal of material mat at [n, 2] (u, v) -> [n, 3]; 1 applyBumpMapping of [n, 12] (modified normal,
        tangent, bitangent, normal) -> [n, 9]; 2 the height-map gather at [n, 2] (u, v) -> [n, 4]"""
        inp = np.ascontiguousarray(inp, dtype=np.float32)
        out = np.zeros((inp.shape[0], width), dtype=np.float32)
        assert lib().orc_bump_query(self.h, op, mat, inp.ctypes.data, inp.shape[0], out.ctypes.data) == 0
        return out


class OracleFrame:
    def __init__(self, oscene: OracleScene, width: int, height: int, seed: int = 591842031321323413):
        self.oscene = oscene
        self.W, self.H = width, height
        self.h = lib().orc_frame_create(oscene.h, width, height)
        lib().orc_rng_seed(self.h, seed)
        lib().orc_restir_setup_neighbor_table(self.h)

    def close(self):
        if self.h:
            lib().orc_frame_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _raw(self, buffer_id: int, index: int):
        nbytes = C.c_size_t()
        ptr = lib().orc_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        return (C.c_uint8 * nbytes.value).from_address(ptr), nbytes.value

    def buffer(self, buffer_id: int, index: int = 0) -> np.ndarray:
        raw, _ = self._raw(buffer_id, index)
        dtype, comps, planes = abi.BUFFER_LAYOUT[buffer_id]
        arr = np.frombuffer(raw, dtype=dtype).copy()
        if planes > 1:
            return arr.reshape(planes, self.H, self.W, comps)
        return arr.reshape(self.H, self.W, comps) if comps > 1 else arr.reshape(self.H, self.W)

    def linear_buffer(self, buffer_id: int, index: int = 0, copy: bool = True, params=None) -> np.ndarray:
        raw, nbytes = self._raw(buffer_id, index)
        dtype, cols, rows = abi.linear_buffer_layout(buffer_id, self.W, self.H, params)
        assert nbytes == rows * cols * np.dtype(dtype).itemsize, (buffer_id, nbytes, rows, cols)
        arr = np.frombuffer(raw, dtype=dtype).reshape(rows, cols)
        return arr.copy() if copy else arr

    def gbuffer(self, params, threads: int = 0):
        lib().orc_bump_gbuffer(self.h, C.byref(params), threads)

    def restir(self, params, pass_id: int, threads: int = 0):
        lib().orc_restir(self.h, C.byref(params), pass_id, threads)

    def restir_rearch(self, params, pass_id: int, threads: int = 0) -> int:
        return int(lib().orc_restir_rearch(self.h, C.byref(params), pass_id, threads))

    def pathtrace(self, params, variant: int = 0, threads: int = 0) -> int:
        rays = int(lib().orc_bump_pathtrace(self.h, C.byref(params), variant, threads))
        if rays == ORC_NOT_READY:
            raise RuntimeError("orc_bump_pathtrace(GFX_PT_REGIR): call regir_build_cells first")
        return rays

    def regir_build_cells(self, params, frame_index: int, temporal: bool, threads: int = 0):
        lib().orc_regir_build_cells(self.h, C.byref(params), frame_index & 0xFFFFFFFF, 1 if temporal else 0, threads)

    def regir_update_access(self, params, frame_index: int):
        lib().orc_regir_update_access(self.h, C.byref(params), frame_index & 0xFFFFFFFF)

    def nrc_preprocess(self, params, offset_unbiased_tile: int, offset_training_path: int, new_sequence: bool):
        lib().orc_nrc_preprocess(self.h, C.byref(params), offset_unbiased_tile, offset_training_path, 1 if new_sequence else 0)

    def nrc_accumulate(self, params):
        lib().orc_nrc_accumulate(self.h, C.byref(params))

    def nrc_propagate(self, params):
        lib().orc_nrc_propagate(self.h, C.byref(params))

    def nrc_shuffle(self, params):
        lib().orc_nrc_shuffle(self.h, C.byref(params))

    def nrc_visualize_prediction(self, params):
        lib().orc_bump_nrc_visualize_prediction(self.h, C.byref(params))
