"""ctypes binding of oracle/liborc_nrc_triwave.so — TEST INFRASTRUCTURE: the CPU restatement of the triangle-wave NRC network
(oracle/nrc_triwave.cpp), with the interface of tests/oracle_lib.OracleNrc.  oracle_nrc() picks the oracle of either position
encoding."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gfxexp_b200 import abi

ORACLE_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")
TRIWAVE_LIB = os.path.join(ORACLE_DIR, "liborc_nrc_triwave.so")
_lib = None


def build_oracle(force: bool = False) -> str:
    if force or not os.path.exists(TRIWAVE_LIB):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-f", "Makefile.triwave"], stdout=subprocess.DEVNULL)
    return TRIWAVE_LIB


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(build_oracle())
        vp, u32 = C.c_void_p, C.c_uint32
        L.orc_nrctw_create.restype = vp
        L.orc_nrctw_create.argtypes = [u32, C.c_float]
        L.orc_nrctw_destroy.argtypes = [vp]
        L.orc_nrctw_num_params.restype = u32
        L.orc_nrctw_num_params.argtypes = [vp]
        L.orc_nrctw_set_params.argtypes = [vp, vp]
        L.orc_nrctw_get_params.argtypes = [vp, vp, C.c_int]
        L.orc_nrctw_set_accumulate_half.argtypes = [vp, C.c_int]
        L.orc_nrctw_get_master.argtypes = [vp, vp]
        L.orc_nrctw_get_gradients.restype = C.c_int
        L.orc_nrctw_get_gradients.argtypes = [vp, vp]
        L.orc_nrctw_encode.argtypes = [vp, vp, u32, vp]
        L.orc_nrctw_infer.argtypes = [vp, vp, vp, u32]
        L.orc_nrctw_train.restype = C.c_float
        L.orc_nrctw_train.argtypes = [vp, vp, vp, u32]
        _lib = L
    return _lib


class OracleNrcTriWave:
    """CPU restatement of NeuralRadianceCache::initialize(PositionEncoding::TriangleWave, ...) — see oracle/nrc_triwave.cpp."""
    position_encoding = abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE

    def __init__(self, num_hidden_layers: int = 2, learning_rate: float = 1e-2):
        self._lib = lib()
        self.h = self._lib.orc_nrctw_create(num_hidden_layers, learning_rate)
        self.num_params = self._lib.orc_nrctw_num_params(self.h)
        self.num_matrix_weights = self.num_params  # the encoding has no parameters

    def close(self):
        if self.h:
            self._lib.orc_nrctw_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def set_params(self, params_f16: np.ndarray):
        p = np.ascontiguousarray(params_f16, dtype=np.float16)
        assert p.shape[0] == self.num_params
        self._lib.orc_nrctw_set_params(self.h, p.ctypes.data)

    def get_params(self, ema: bool = True) -> np.ndarray:
        out = np.empty(self.num_params, dtype=np.float16)
        self._lib.orc_nrctw_get_params(self.h, out.ctypes.data, 1 if ema else 0)
        return out

    def set_accumulate_half(self, on: bool):
        """fully-connected layers with tiny-cuda-nn's half accumulator fragments instead of fp32"""
        self._lib.orc_nrctw_set_accumulate_half(self.h, 1 if on else 0)

    def get_master(self) -> np.ndarray:
        out = np.empty(self.num_params, dtype=np.float32)
        self._lib.orc_nrctw_get_master(self.h, out.ctypes.data)
        return out

    def get_gradients(self) -> np.ndarray:
        out = np.empty(self.num_params, dtype=np.float32)
        assert self._lib.orc_nrctw_get_gradients(self.h, out.ctypes.data) == 0, "no training step yet"
        return out

    def encode(self, queries: np.ndarray) -> np.ndarray:
        q = np.ascontiguousarray(queries, dtype=np.float32)
        out = np.empty((q.shape[0], 64), dtype=np.float16)
        self._lib.orc_nrctw_encode(self.h, q.ctypes.data, q.shape[0], out.ctypes.data)
        return out

    def infer(self, queries: np.ndarray) -> np.ndarray:
        q = np.ascontiguousarray(queries, dtype=np.float32)
        out = np.empty((q.shape[0], 3), dtype=np.float32)
        self._lib.orc_nrctw_infer(self.h, q.ctypes.data, out.ctypes.data, q.shape[0])
        return out

    def train(self, queries: np.ndarray, targets: np.ndarray) -> float:
        q = np.ascontiguousarray(queries, dtype=np.float32)
        t = np.ascontiguousarray(targets, dtype=np.float32)
        return float(self._lib.orc_nrctw_train(self.h, q.ctypes.data, t.ctypes.data, q.shape[0]))


def oracle_nrc(num_hidden_layers: int = 2, learning_rate: float = 1e-2,
               position_encoding: int = abi.NRC_POSITION_ENCODING_HASH_GRID):
    """the oracle network for either of gfx_nrc_create_with_encoding's position encodings"""
    if position_encoding == abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE:
        return OracleNrcTriWave(num_hidden_layers, learning_rate)
    if position_encoding == abi.NRC_POSITION_ENCODING_HASH_GRID:
        from tests import oracle_lib
        return oracle_lib.OracleNrc(num_hidden_layers, learning_rate)
    raise ValueError(f"unknown position encoding {position_encoding}")
