"""ctypes binding of oracle/liborc_svgf_views.so (oracle/svgf_views.cpp, built by oracle/Makefile.svgf_views) — TEST
INFRASTRUCTURE.

The CPU restatement of the SVGF app's debug views (gfx_svgf_debug_visualize, debugVisualize of svgf/gpu_kernels/visualize.cu).
The library carries its own copy of the SVGF app's oracle with its TAA jitter (tests/oracle_svgf_taa_jitter.py), so the frame
and the SVGF passes run on a Frame / Svgf of this module, and Svgf.debug_visualize reads that Svgf's planes.  view_planes runs
the views on planes given as arrays.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gfxexp_b200 import abi
from tests import oracle_lib

LIB = os.path.join(oracle_lib.ORACLE_DIR, "liborc_svgf_views.so")
_lib = None


class OrcSvgfViewPlanes(C.Structure):
    _fields_ = [("lighting", C.c_void_p * 2), ("albedo", C.c_void_p), ("normal", C.c_void_p), ("prevScreenPos", C.c_void_p),
                ("moments", C.c_void_p)]


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", oracle_lib.ORACLE_DIR, "-f", "Makefile.svgf_views"], stdout=subprocess.DEVNULL)
        L = C.CDLL(LIB)
        vp = C.c_void_p
        u32 = C.c_uint32
        P = C.POINTER(abi.GfxFrameParams)
        L.orc_scene_create.restype = vp
        L.orc_scene_create.argtypes = [C.POINTER(abi.GfxSceneDesc), C.POINTER(oracle_lib.OrcBuildConfig), C.c_int]
        L.orc_scene_destroy.argtypes = [vp]
        L.orc_frame_create.restype = vp
        L.orc_frame_create.argtypes = [vp, u32, u32]
        L.orc_frame_destroy.argtypes = [vp]
        L.orc_rng_seed.argtypes = [vp, C.c_uint64]
        L.orc_buffer_ptr.restype = vp
        L.orc_buffer_ptr.argtypes = [vp, C.c_int, u32, C.POINTER(C.c_size_t)]
        L.orc_gbuffer_taa_jitter.restype = C.c_int
        L.orc_gbuffer_taa_jitter.argtypes = [vp, P, C.c_int]
        L.orc_svgf_app_pathtrace.restype = C.c_uint64
        L.orc_svgf_app_pathtrace.argtypes = [vp, P, C.c_int]
        L.orc_svgf_create.restype = vp
        L.orc_svgf_create.argtypes = [vp, u32, u32]
        L.orc_svgf_destroy.argtypes = [vp]
        L.orc_svgf_buffer_ptr.restype = vp
        L.orc_svgf_buffer_ptr.argtypes = [vp, C.c_int, u32, C.POINTER(C.c_size_t)]
        L.orc_svgf_pass.argtypes = [vp, P, C.c_int, u32, C.c_int]
        L.orc_svgf_app_feedback_noisy_lighting.argtypes = [vp, P, u32, u32]
        L.orc_svgf_fill_background_taa_jitter.restype = C.c_int
        L.orc_svgf_fill_background_taa_jitter.argtypes = [vp, vp, P, u32, C.c_int]
        L.orc_svgf_view_planes.restype = C.c_int
        L.orc_svgf_view_planes.argtypes = [C.POINTER(OrcSvgfViewPlanes), u32, u32, u32, u32, C.c_int, C.c_int, C.c_float,
                                           C.c_float, u32, vp]
        L.orc_svgf_view_inputs.argtypes = [vp, P, vp, vp]
        L.orc_svgf_debug_visualize.restype = C.c_int
        L.orc_svgf_debug_visualize.argtypes = [vp, vp, P, C.c_int, C.c_float, C.c_float, u32, vp]
        _lib = L
    return _lib


def _view(ptr, nbytes, buffer_id, h, w):
    dtype, comps, _ = abi.BUFFER_LAYOUT[buffer_id]
    arr = np.frombuffer((C.c_uint8 * nbytes).from_address(ptr), dtype=dtype).copy()
    return arr.reshape(h, w, comps) if comps > 1 else arr.reshape(h, w)


def _c(a, dtype):
    a = np.ascontiguousarray(a, dtype=dtype)
    return a, a.ctypes.data


def view_planes(lighting0, lighting1, albedo, normal, prev_screen_pos, moments, view: int, modulate_albedo: bool = False,
                offset: float = 0.5, scale: float = 0.1, num_filtering_stages: int = 5, out=None, rows=None) -> np.ndarray:
    """orc_svgf_view_planes on [H, W, 4] float32 planes (lighting 0 / 1, albedo, normal), [H, W, 2] float32 prevScreenPos and
    [H, W, 4] uint32 moments; rows = (y0, y1) (all rows by default) of out (zeros by default) are written"""
    h, w = np.shape(albedo)[:2]
    keep = [_c(lighting0, np.float32), _c(lighting1, np.float32), _c(albedo, np.float32), _c(normal, np.float32),
            _c(prev_screen_pos, np.float32), _c(moments, np.uint32)]
    planes = OrcSvgfViewPlanes((C.c_void_p * 2)(keep[0][1], keep[1][1]), keep[2][1], keep[3][1], keep[4][1], keep[5][1])
    out = np.zeros((h, w, 4), dtype=np.float32) if out is None else np.ascontiguousarray(out, dtype=np.float32).copy()
    y0, y1 = rows if rows is not None else (0, h)
    rc = lib().orc_svgf_view_planes(C.byref(planes), w, h, y0, y1, view, 1 if modulate_albedo else 0, offset, scale,
                                    num_filtering_stages, out.ctypes.data)
    if rc != 0:
        raise ValueError(f"view {view} is not one of the SVGF app's debug views 0..6")
    return out


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

    def view_inputs(self, params):
        """(normal [H, W, 4], prevScreenPos [H, W, 2]) of the rows of params, as the temporal pass and the background fill
        write them; zeros elsewhere"""
        normal = np.zeros((self.H, self.W, 4), dtype=np.float32)
        psp = np.zeros((self.H, self.W, 2), dtype=np.float32)
        lib().orc_svgf_view_inputs(self.h, C.byref(params), normal.ctypes.data, psp.ctypes.data)
        return normal, psp


class Svgf:
    """the SVGF app's passes on a Frame of this library, and its debug views into a buffer of its own"""

    def __init__(self, frame: Frame):
        self.frame = frame
        self.W, self.H = frame.W, frame.H
        self.h = lib().orc_svgf_create(frame.h, frame.W, frame.H)
        self.debug = None  # BUF_SVGF_DEBUG_VISUALIZE, allocated and zeroed by the first view

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

    def debug_visualize(self, params, view: int, offset: float = 0.5, scale: float = 0.1, num_filtering_stages: int = 5):
        if self.debug is None:
            self.debug = np.zeros((self.H, self.W, 4), dtype=np.float32)
        rc = lib().orc_svgf_debug_visualize(self.h, self.frame.h, C.byref(params), view, offset, scale, num_filtering_stages,
                                            self.debug.ctypes.data)
        if rc != 0:
            raise ValueError(f"view {view} is not one of the SVGF app's debug views 0..6")

    def buffer(self, buffer_id: int, index: int = 0) -> np.ndarray:
        if buffer_id == abi.BUF_SVGF_DEBUG_VISUALIZE:
            if self.debug is None:
                raise ValueError("no debug view has been computed yet")
            return self.debug.copy()
        nbytes = C.c_size_t()
        ptr = lib().orc_svgf_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        return _view(ptr, nbytes.value, buffer_id, self.H, self.W)
