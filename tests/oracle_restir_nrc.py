"""ctypes binding of oracle/liborc_restir_nrc.so (oracle/restir_nrc.cpp, built by oracle/Makefile.restir_nrc) — TEST INFRASTRUCTURE.

The CPU restatement of GFX_PT_NRC_INDIRECT and of the additive gfx_nrc_accumulate after it (ReSTIR DI + NRC as one estimator).
The library carries its own copy of the oracle renderer (bump.cpp's, so GfxFrameParams::enableBumpMapping works), so a frame runs
on an OracleScene / OracleFrame of this module: the same methods as oracle_bump's, with pathtrace(PT_NRC or PT_NRC_INDIRECT).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gfxexp_b200 import abi
from tests import oracle_lib

LIB = os.path.join(oracle_lib.ORACLE_DIR, "liborc_restir_nrc.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "Makefile.restir_nrc"], stdout=subprocess.DEVNULL)
        L = C.CDLL(LIB)
        vp, pp = C.c_void_p, C.POINTER(abi.GfxFrameParams)
        L.orc_scene_create.restype = vp
        L.orc_scene_create.argtypes = [C.POINTER(abi.GfxSceneDesc), C.POINTER(oracle_lib.OrcBuildConfig), C.c_int]
        L.orc_scene_destroy.argtypes = [vp]
        L.orc_bump_attach.argtypes = [vp, C.POINTER(abi.GfxSceneDesc)]
        L.orc_bump_detach.argtypes = [vp]
        L.orc_frame_create.restype = vp
        L.orc_frame_create.argtypes = [vp, C.c_uint32, C.c_uint32]
        L.orc_rnc_frame_destroy.argtypes = [vp]
        L.orc_rng_seed.argtypes = [vp, C.c_uint64]
        L.orc_restir_setup_neighbor_table.argtypes = [vp]
        L.orc_buffer_ptr.restype = vp
        L.orc_buffer_ptr.argtypes = [vp, C.c_int, C.c_uint32, C.POINTER(C.c_size_t)]
        L.orc_bump_gbuffer.argtypes = [vp, pp, C.c_int]
        L.orc_restir.argtypes = [vp, pp, C.c_int, C.c_int]
        L.orc_restir_rearch.restype = C.c_uint64
        L.orc_restir_rearch.argtypes = [vp, pp, C.c_int, C.c_int]
        L.orc_rnc_pathtrace.restype = C.c_uint64
        L.orc_rnc_pathtrace.argtypes = [vp, pp, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
        L.orc_bump_pathtrace.restype = C.c_uint64
        L.orc_bump_pathtrace.argtypes = [vp, pp, C.c_int, C.c_int]
        L.orc_nrc_set_shard.argtypes = [vp, C.c_int, C.c_int, oracle_lib.NRC_EXCHANGE_FN, oracle_lib.NRC_SUM_FN, vp]
        L.orc_nrc_preprocess.argtypes = [vp, pp, C.c_uint32, C.c_uint32, C.c_int]
        for name in ("orc_rnc_nrc_accumulate", "orc_nrc_propagate", "orc_nrc_shuffle"):
            getattr(L, name).argtypes = [vp, pp]
        _lib = L
    return _lib


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


class OracleFrame:
    def __init__(self, oscene: OracleScene, width: int, height: int, seed: int = 591842031321323413):
        self.oscene = oscene
        self.W, self.H = width, height
        self.h = lib().orc_frame_create(oscene.h, width, height)
        lib().orc_rng_seed(self.h, seed)
        lib().orc_restir_setup_neighbor_table(self.h)
        self.skipped_shadow_rays = 0
        self.skipped_contributing_shadow_rays = 0

    def close(self):
        if self.h:
            lib().orc_rnc_frame_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _raw(self, buffer_id: int, index: int):
        nbytes = C.c_size_t()
        ptr = lib().orc_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        return (C.c_uint8 * nbytes.value).from_address(ptr), nbytes.value

    def buffer(self, buffer_id: int, index: int = 0, copy: bool = True) -> np.ndarray:
        raw, _ = self._raw(buffer_id, index)
        dtype, comps, planes = abi.BUFFER_LAYOUT[buffer_id]
        arr = np.frombuffer(raw, dtype=dtype)
        arr = arr.copy() if copy else arr
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

    def pathtrace(self, params, variant: int = abi.PT_NRC_INDIRECT, threads: int = 0) -> int:
        """PT_NRC or PT_NRC_INDIRECT; returns the rays traced.  skipped_shadow_rays: the primary vertices that drew a light
        sample but traced no shadow ray (PT_NRC_INDIRECT's non-training primary hits); skipped_contributing_shadow_rays: those of
        them whose sample has a non-zero unshadowed contribution - the library queues a shadow ray only for such a sample, so
        this is what its ray counter drops from PT_NRC to PT_NRC_INDIRECT"""
        assert variant in (abi.PT_NRC, abi.PT_NRC_INDIRECT)
        skipped = (C.c_uint64 * 2)()
        rays = int(lib().orc_rnc_pathtrace(self.h, C.byref(params), variant, threads, skipped))
        self.skipped_shadow_rays, self.skipped_contributing_shadow_rays = int(skipped[0]), int(skipped[1])
        return rays

    def bump_pathtrace_nrc(self, params, threads: int = 0) -> int:
        """the bump oracle's own GFX_PT_NRC restatement (oracle/bump.cpp), which pathtrace(PT_NRC) must reproduce"""
        return int(lib().orc_bump_pathtrace(self.h, C.byref(params), abi.PT_NRC, threads))

    def nrc_shard(self, rank: int, world: int):
        """the oracle's gfx_nrc_shard over the default torch.distributed group (gloo), as oracle_lib.OracleFrame.nrc_shard"""
        import torch
        import torch.distributed as dist

        def exchange(_user, mine, num_words, out):
            t = torch.tensor([mine[i] for i in range(num_words)], dtype=torch.int64)
            gathered = [torch.zeros_like(t) for _ in range(world)]
            dist.all_gather(gathered, t)
            for r in range(world):
                for i in range(num_words):
                    out[r * num_words + i] = int(gathered[r][i])

        def total(_user, words, num_words):
            a = np.ctypeslib.as_array(words, shape=(num_words,))
            t = torch.from_numpy(a.astype(np.int64))  # every word is non-zero on one rank only: the sum fits 32 bits again
            dist.all_reduce(t)
            a[:] = t.numpy().astype(np.uint32)
        self._shard_callbacks = (oracle_lib.NRC_EXCHANGE_FN(exchange), oracle_lib.NRC_SUM_FN(total))  # keep the thunks alive
        lib().orc_nrc_set_shard(self.h, rank, world, self._shard_callbacks[0], self._shard_callbacks[1], None)

    def nrc_preprocess(self, params, offset_unbiased_tile: int, offset_training_path: int, new_sequence: bool):
        lib().orc_nrc_preprocess(self.h, C.byref(params), offset_unbiased_tile, offset_training_path, 1 if new_sequence else 0)

    def nrc_accumulate(self, params):
        lib().orc_rnc_nrc_accumulate(self.h, C.byref(params))

    def nrc_propagate(self, params):
        lib().orc_nrc_propagate(self.h, C.byref(params))

    def nrc_shuffle(self, params):
        lib().orc_nrc_shuffle(self.h, C.byref(params))
