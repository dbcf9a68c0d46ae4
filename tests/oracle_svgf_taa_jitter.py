"""ctypes binding of oracle/liborc_svgf_taa_jitter.so (oracle/svgf_taa_jitter.cpp, built by oracle/Makefile.svgf_taa_jitter) —
TEST INFRASTRUCTURE.

The CPU restatement of the SVGF app's frame with its TAA sub-pixel jitter (GFX_SVGF_SUBPIXEL_JITTER): the library carries its
own copy of the SVGF app's oracle (tests/oracle_svgf_app.py), so the G-buffer, the path tracers and the SVGF passes run on a
Frame / Svgf of this module.  Frames the jitter does not apply to run the same code as there.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gfxexp_b200 import abi
from tests import oracle_lib

LIB = os.path.join(oracle_lib.ORACLE_DIR, "liborc_svgf_taa_jitter.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "Makefile.svgf_taa_jitter"], stdout=subprocess.DEVNULL)
        L = C.CDLL(LIB)
        vp = C.c_void_p
        P = C.POINTER(abi.GfxFrameParams)
        L.orc_scene_create.restype = vp
        L.orc_scene_create.argtypes = [C.POINTER(abi.GfxSceneDesc), C.POINTER(oracle_lib.OrcBuildConfig), C.c_int]
        L.orc_scene_destroy.argtypes = [vp]
        L.orc_frame_create.restype = vp
        L.orc_frame_create.argtypes = [vp, C.c_uint32, C.c_uint32]
        L.orc_frame_destroy.argtypes = [vp]
        L.orc_rng_seed.argtypes = [vp, C.c_uint64]
        L.orc_buffer_ptr.restype = vp
        L.orc_buffer_ptr.argtypes = [vp, C.c_int, C.c_uint32, C.POINTER(C.c_size_t)]
        L.orc_gbuffer_taa_jitter.restype = C.c_int
        L.orc_gbuffer_taa_jitter.argtypes = [vp, P, C.c_int]
        L.orc_svgf_app_pathtrace.restype = C.c_uint64
        L.orc_svgf_app_pathtrace.argtypes = [vp, P, C.c_int]
        L.orc_svgf_create.restype = vp
        L.orc_svgf_create.argtypes = [vp, C.c_uint32, C.c_uint32]
        L.orc_svgf_destroy.argtypes = [vp]
        L.orc_svgf_buffer_ptr.restype = vp
        L.orc_svgf_buffer_ptr.argtypes = [vp, C.c_int, C.c_uint32, C.POINTER(C.c_size_t)]
        L.orc_svgf_pass.argtypes = [vp, P, C.c_int, C.c_uint32, C.c_int]
        L.orc_svgf_app_feedback_noisy_lighting.argtypes = [vp, P, C.c_uint32, C.c_uint32]
        L.orc_svgf_fill_background_taa_jitter.restype = C.c_int
        L.orc_svgf_fill_background_taa_jitter.argtypes = [vp, vp, P, C.c_uint32, C.c_int]
        L.orc_svgf_subpixel_offset.argtypes = [C.c_uint32, C.POINTER(C.c_float)]
        _lib = L
    return _lib


def subpixel_offset(i: int):
    """the app's subPixelOffsets[i] = (halton(2, i), halton(3, i)) as the oracle computes it"""
    out = (C.c_float * 2)()
    lib().orc_svgf_subpixel_offset(i, out)
    return np.float32(out[0]), np.float32(out[1])


def _view(ptr, nbytes, buffer_id, h, w):
    dtype, comps, _ = abi.BUFFER_LAYOUT[buffer_id]
    arr = np.frombuffer((C.c_uint8 * nbytes).from_address(ptr), dtype=dtype).copy()
    return arr.reshape(h, w, comps) if comps > 1 else arr.reshape(h, w)


class Frame:
    """a scene + frame of this library: the G-buffer pass (jittered when the frame asks for it) and GFX_PT_SVGF"""

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
        rc = lib().orc_gbuffer_taa_jitter(self.h, C.byref(params), threads)
        assert rc == 0, "GFX_SVGF_SUBPIXEL_JITTER together with enableJittering"

    def pathtrace(self, params, variant: int = abi.PT_SVGF, threads: int = 0) -> int:
        assert variant == abi.PT_SVGF
        return int(lib().orc_svgf_app_pathtrace(self.h, C.byref(params), threads))

    def buffer(self, buffer_id: int, index: int = 0) -> np.ndarray:
        nbytes = C.c_size_t()
        ptr = lib().orc_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        return _view(ptr, nbytes.value, buffer_id, self.H, self.W)


class Svgf:
    """the SVGF app's passes on a Frame of this library, the background through the jitter's sample"""

    def __init__(self, frame: Frame):
        self.frame = frame
        self.W, self.H = frame.W, frame.H
        self.h = lib().orc_svgf_create(frame.h, frame.W, frame.H)

    def close(self):
        if self.h:
            lib().orc_svgf_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def run(self, params, pass_id: int, stage: int = 0, threads: int = 0):
        if pass_id == abi.SVGF_FEEDBACK_NOISY_LIGHTING:
            lib().orc_svgf_app_feedback_noisy_lighting(self.h, C.byref(params), self.W, self.H)
        elif pass_id == abi.SVGF_FILL_BACKGROUND:
            rc = lib().orc_svgf_fill_background_taa_jitter(self.h, self.frame.h, C.byref(params), stage, threads)
            assert rc == 0, "GFX_SVGF_SUBPIXEL_JITTER together with enableJittering"
        else:
            lib().orc_svgf_pass(self.h, C.byref(params), pass_id, stage, threads)

    def buffer(self, buffer_id: int, index: int = 0) -> np.ndarray:
        nbytes = C.c_size_t()
        ptr = lib().orc_svgf_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        return _view(ptr, nbytes.value, buffer_id, self.H, self.W)
