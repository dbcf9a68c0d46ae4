"""ctypes binding of oracle/liboracle.so — TEST INFRASTRUCTURE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import
this module.  The product package (gfxexp_b200) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gfxexp_b200 import abi

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(_ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liboracle.so")
ORC_NOT_READY = (1 << 64) - 1   # orc_pathtrace(GFX_PT_REGIR) before a ReGIR build (oracle.h)


class OrcBuildConfig(C.Structure):
    _fields_ = [("splittingBudget", C.c_float), ("intNodeTravCost", C.c_float), ("primIntersectCost", C.c_float),
                ("minNumPrimsPerLeaf", C.c_uint32), ("maxNumPrimsPerLeaf", C.c_uint32)]


class OrcTraversalStats(C.Structure):
    _fields_ = [("numAabbTests", C.c_uint64), ("numTriTests", C.c_uint64), ("numIntNodes", C.c_uint64),
                ("maxStackDepth", C.c_int32), ("numHits", C.c_uint32)]


TRACE_FIRST_FOUND, TRACE_CANONICAL, TRACE_BRUTE_FORCE, TRACE_ANY = range(4)


def reference_build_config() -> OrcBuildConfig:
    """nrtdsm/nrtdsm_sandbox.cpp:3177-3184: budget .3, trav 1.2, isect 1.0, leaf 1..128."""
    return OrcBuildConfig(0.3, 1.2, 1.0, 1, 128)


def build_oracle(force: bool = False) -> str:
    if force or not os.path.exists(ORACLE_LIB):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-j8"], stdout=subprocess.DEVNULL)
    return ORACLE_LIB


_lib = None


NRC_EXCHANGE_FN = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_uint32))
NRC_SUM_FN = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_uint32), C.c_uint64)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build_oracle()
        L = C.CDLL(ORACLE_LIB)
        vp = C.c_void_p
        L.orc_scene_create.restype = vp
        L.orc_scene_create.argtypes = [C.POINTER(abi.GfxSceneDesc), C.POINTER(OrcBuildConfig), C.c_int]
        L.orc_scene_destroy.argtypes = [vp]
        L.orc_scene_update_instances.restype = C.c_int
        L.orc_scene_update_instances.argtypes = [vp, C.POINTER(abi.GfxInstanceDesc), C.c_uint32]
        L.orc_scene_build_seconds.restype = C.c_double
        L.orc_scene_build_seconds.argtypes = [vp]
        L.orc_bvh_info.argtypes = [vp, C.POINTER(abi.GfxBvhInfo)]
        L.orc_bvh_export.argtypes = [vp, vp, vp, vp]
        L.orc_bvh_import.argtypes = [vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32]
        L.orc_bvh_validate.restype = C.c_int
        L.orc_bvh_validate.argtypes = [vp, C.c_char_p, C.c_size_t]
        L.orc_bvh_build_gpu_style.restype = C.c_int
        L.orc_bvh_build_gpu_style.argtypes = [vp, C.c_uint32]
        L.orc_bvh_sah_levels.restype = C.c_uint32
        L.orc_bvh_sah_levels.argtypes = [vp, vp, C.c_uint32]
        L.orc_bvh_same_tree.restype = C.c_int
        L.orc_bvh_same_tree.argtypes = [vp, vp, C.c_char_p, C.c_size_t]
        L.orc_trace.argtypes = [vp, vp, C.c_uint32, vp, C.c_int, C.POINTER(OrcTraversalStats), C.c_int]
        L.orc_light_dist_export.argtypes = [vp, vp, vp, C.POINTER(C.c_float)]
        L.orc_present.argtypes = [vp, C.c_uint32, C.c_uint32, C.POINTER(abi.GfxPresentParams), vp]
        L.orc_frame_create.restype = vp
        L.orc_frame_create.argtypes = [vp, C.c_uint32, C.c_uint32]
        L.orc_frame_destroy.argtypes = [vp]
        L.orc_rng_seed.argtypes = [vp, C.c_uint64]
        L.orc_restir_setup_neighbor_table.argtypes = [vp]
        L.orc_buffer_ptr.restype = vp
        L.orc_buffer_ptr.argtypes = [vp, C.c_int, C.c_uint32, C.POINTER(C.c_size_t)]
        L.orc_gbuffer.argtypes = [vp, C.POINTER(abi.GfxFrameParams), C.c_int]
        L.orc_restir.argtypes = [vp, C.POINTER(abi.GfxFrameParams), C.c_int, C.c_int]
        L.orc_pathtrace.argtypes = [vp, C.POINTER(abi.GfxFrameParams), C.c_int, C.c_int]
        L.orc_pathtrace.restype = C.c_uint64
        L.orc_restir_rearch.argtypes = [vp, C.POINTER(abi.GfxFrameParams), C.c_int, C.c_int]
        L.orc_restir_rearch.restype = C.c_uint64
        L.orc_regir_build_cells.argtypes = [vp, C.POINTER(abi.GfxFrameParams), C.c_uint32, C.c_int, C.c_int]
        L.orc_regir_update_access.argtypes = [vp, C.POINTER(abi.GfxFrameParams), C.c_uint32]
        L.orc_nrc_preprocess.argtypes = [vp, C.POINTER(abi.GfxFrameParams), C.c_uint32, C.c_uint32, C.c_int]
        L.orc_nrc_set_shard.argtypes = [vp, C.c_int, C.c_int, NRC_EXCHANGE_FN, NRC_SUM_FN, vp]
        for name in ("orc_nrc_accumulate", "orc_nrc_propagate", "orc_nrc_shuffle"):
            getattr(L, name).argtypes = [vp, C.POINTER(abi.GfxFrameParams)]
        L.orc_generate_primary_rays.argtypes = [C.POINTER(abi.GfxFrameParams), C.c_uint32, C.c_uint32, vp]
        L.orc_svgf_create.restype = vp
        L.orc_svgf_create.argtypes = [vp, C.c_uint32, C.c_uint32]
        L.orc_svgf_destroy.argtypes = [vp]
        L.orc_svgf_buffer_ptr.restype = vp
        L.orc_svgf_buffer_ptr.argtypes = [vp, C.c_int, C.c_uint32, C.POINTER(C.c_size_t)]
        L.orc_svgf_pass.restype = C.c_int
        L.orc_svgf_pass.argtypes = [vp, C.POINTER(abi.GfxFrameParams), C.c_int, C.c_uint32, C.c_int]
        L.orc_env_query.restype = C.c_int
        L.orc_env_query.argtypes = [vp, C.c_int, vp, C.c_uint32, vp]
        L.orc_light_sample_debug.restype = C.c_int
        L.orc_light_sample_debug.argtypes = [vp, C.c_int, vp, vp, C.c_uint32, vp]
        L.orc_rays_traced.restype = C.c_ulonglong
        L.orc_rays_traced.argtypes = [C.c_int]
        L.orc_nrc_create.restype = vp
        L.orc_nrc_create.argtypes = [C.c_uint32, C.c_float]
        L.orc_nrc_destroy.argtypes = [vp]
        L.orc_nrc_num_params.restype = C.c_uint32
        L.orc_nrc_num_params.argtypes = [vp]
        L.orc_nrc_num_matrix_weights.restype = C.c_uint32
        L.orc_nrc_num_matrix_weights.argtypes = [vp]
        L.orc_nrc_set_params.argtypes = [vp, vp]
        L.orc_nrc_get_params.argtypes = [vp, vp, C.c_int]
        L.orc_nrc_encode.argtypes = [vp, vp, C.c_uint32, vp, C.c_int]
        L.orc_nrc_infer.argtypes = [vp, vp, vp, C.c_uint32]
        L.orc_nrc_set_accumulate_half.argtypes = [vp, C.c_int]
        L.orc_nrc_init_master.argtypes = [vp, vp]
        L.orc_nrc_get_master.argtypes = [vp, vp]
        L.orc_nrc_get_gradients.argtypes = [vp, vp]
        L.orc_nrc_get_gradients.restype = C.c_int
        L.orc_nrc_train.restype = C.c_float
        L.orc_nrc_train.argtypes = [vp, vp, vp, C.c_uint32]
        _lib = L
    return _lib


def present(rgba: np.ndarray, mode: int = 0, flags: int = 3, brightness_scale: float = 1.0, alpha_override: float = 1.0) -> np.ndarray:
    """the reference's output side on a float4 image [H, W, 4] -> packed RGBA8 [H, W] uint32 (oracle/present.cpp)"""
    src = np.ascontiguousarray(rgba, dtype=np.float32)
    h, w = src.shape[:2]
    out = np.empty((h, w), dtype=np.uint32)
    pp = abi.GfxPresentParams(0, 0, mode, flags, brightness_scale, alpha_override)
    lib().orc_present(src.ctypes.data_as(C.c_void_p), w, h, C.byref(pp), out.ctypes.data_as(C.c_void_p))
    return out


class OracleScene:
    def __init__(self, scene, cfg: OrcBuildConfig | None = None, build_bvh: bool = True):
        """build_bvh=False skips the (single-threaded) SBVH build: import_bvh() must follow before anything traces"""
        self.arrays = abi.SceneArrays(scene)
        self.cfg = cfg or reference_build_config()
        self.h = lib().orc_scene_create(C.byref(self.arrays.desc), C.byref(self.cfg), 0 if build_bvh else -1)
        if not self.h:
            raise ValueError("orc_scene_create refused the scene (an environment map with a NaN texel)")

    def close(self):
        if self.h:
            lib().orc_scene_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def env_query(self, op: int, pairs: np.ndarray) -> np.ndarray:
        """environment light hooks: op 0 sample(u0, u1) -> (u, v, uvPDF), 1 evaluatePDF(u, v), 2 fetch(u, v) -> rgb"""
        a = np.ascontiguousarray(pairs, dtype=np.float32).reshape(-1, 2)
        out = np.zeros((a.shape[0], 3), dtype=np.float32)
        rc = lib().orc_env_query(self.h, op, a.ctypes.data_as(C.c_void_p), a.shape[0], out.ctypes.data_as(C.c_void_p))
        assert rc == 0, "scene has no environment map"
        return out

    def light_sample_debug(self, op: int, records: np.ndarray, env_rotation: float = 0.0, env_power: float = 1.0,
                           enable_env: bool = False) -> np.ndarray:
        """the oracle's side of gfx_light_sample_debug, ops 0 and 3-7: records [n, <= 16] float32 -> [n, 16] float32"""
        a = np.zeros((records.shape[0], 16), dtype=np.float32)
        a[:, :records.shape[1]] = records
        out = np.zeros_like(a)
        params = (C.c_float * 3)(env_rotation, env_power, 1.0 if enable_env else 0.0)
        rc = lib().orc_light_sample_debug(self.h, op, params, a.ctypes.data_as(C.c_void_p), a.shape[0],
                                          out.ctypes.data_as(C.c_void_p))
        assert rc == 0, f"orc_light_sample_debug({op}) = {rc}"
        return out

    def update_instances(self, instance_descs):
        """new instance transforms: rebuilds the world-space SBVH and the light distributions"""
        rc = lib().orc_scene_update_instances(self.h, instance_descs, len(instance_descs))
        assert rc == 0, rc

    @property
    def build_seconds(self) -> float:
        return lib().orc_scene_build_seconds(self.h)

    def info(self) -> abi.GfxBvhInfo:
        info = abi.GfxBvhInfo()
        lib().orc_bvh_info(self.h, C.byref(info))
        return info

    def export_bvh(self):
        info = self.info()
        nodes = np.zeros(info.numNodes, dtype=abi.NODE_DTYPE)
        refs = np.zeros(info.numPrimRefs, dtype=np.uint32)
        tris = np.zeros(info.numTriangles, dtype=abi.TRI_DTYPE)
        lib().orc_bvh_export(self.h, nodes.ctypes.data, refs.ctypes.data, tris.ctypes.data)
        return nodes, refs, tris

    def import_bvh(self, nodes, refs, tris):
        nodes = np.ascontiguousarray(nodes)
        refs = np.ascontiguousarray(refs)
        tris = np.ascontiguousarray(tris)
        lib().orc_bvh_import(self.h, nodes.ctypes.data, nodes.shape[0], refs.ctypes.data, refs.shape[0],
                             tris.ctypes.data, tris.shape[0])

    def validate(self) -> str:
        buf = C.create_string_buffer(512)
        rc = lib().orc_bvh_validate(self.h, buf, 512)
        return "" if rc == 0 else f"[{rc}] {buf.value.decode()}"

    def build_gpu_style(self, flags: int = 0) -> np.ndarray:
        """replace the BVH by the CPU restatement of the tree gfx_bvh_build(flags) builds (oracle/gpu_bvh.cpp: binned SAH,
        or LBVH with GFX_BVH_BUILD_FAST); returns the {small, big, huge} node counts of every SAH level as [levels, 3]"""
        assert lib().orc_bvh_build_gpu_style(self.h, flags) == 0, "PLOC has no restatement"
        num = lib().orc_bvh_sah_levels(self.h, None, 0)
        levels = np.zeros((num, 3), dtype=np.uint32)
        lib().orc_bvh_sah_levels(self.h, levels.ctypes.data, num)
        return levels

    def same_tree(self, other: "OracleScene") -> str:
        """"" if this BVH and other's are the same tree (every node field but the two base indices, every leaf's reference
        words), else the first difference as a slot path from the root"""
        buf = C.create_string_buffer(512)
        rc = lib().orc_bvh_same_tree(self.h, other.h, buf, 512)
        return "" if rc == 0 else buf.value.decode()

    def trace(self, rays: np.ndarray, mode: int = TRACE_CANONICAL, want_stats: bool = False, threads: int = 0):
        rays = np.ascontiguousarray(rays)
        assert rays.dtype == abi.RAY_DTYPE
        hits = np.zeros(rays.shape[0], dtype=abi.HIT_DTYPE)
        stats = OrcTraversalStats()
        lib().orc_trace(self.h, rays.ctypes.data, rays.shape[0], hits.ctypes.data, mode,
                        C.byref(stats) if want_stats else None, threads)
        return (hits, stats) if want_stats else hits

    def light_dist(self):
        n = len(self.arrays.scene.instances)
        w = np.zeros(n, dtype=np.float32)
        cdf = np.zeros(n, dtype=np.float32)
        integ = C.c_float()
        lib().orc_light_dist_export(self.h, w.ctypes.data, cdf.ctypes.data, C.byref(integ))
        return w, cdf, integ.value


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

    def buffer(self, buffer_id: int, index: int = 0, copy: bool = True) -> np.ndarray:
        """copy=False returns a writable view of the oracle's memory"""
        nbytes = C.c_size_t()
        ptr = lib().orc_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        dtype, comps, planes = abi.BUFFER_LAYOUT[buffer_id]
        raw = (C.c_uint8 * nbytes.value).from_address(ptr)
        arr = np.frombuffer(raw, dtype=dtype)
        arr = arr.copy() if copy else arr
        if planes > 1:
            return arr.reshape(planes, self.H, self.W, comps)
        return arr.reshape(self.H, self.W, comps) if comps > 1 else arr.reshape(self.H, self.W)

    def gbuffer(self, params, threads: int = 0):
        lib().orc_gbuffer(self.h, C.byref(params), threads)

    def restir(self, params, pass_id: int, threads: int = 0):
        lib().orc_restir(self.h, C.byref(params), pass_id, threads)

    def pathtrace(self, params, variant: int = 0, threads: int = 0) -> int:
        """one sample per pixel of the path tracer; returns the number of rays traced"""
        rays = int(lib().orc_pathtrace(self.h, C.byref(params), variant, threads))
        if rays == ORC_NOT_READY:
            raise RuntimeError("orc_pathtrace(GFX_PT_REGIR): call regir_build_cells first")
        return rays


    # -- NRC frame (nrc_setup_kernels.cu) -----------------------------------------------------------
    def linear_buffer(self, buffer_id: int, index: int = 0, copy: bool = True, params=None) -> np.ndarray:
        """NRC / ReGIR buffers (GFX_BUF_NRC_*, GFX_BUF_REGIR_*) as [rows, cols]; copy=False returns a writable view of
        the oracle's memory"""
        nbytes = C.c_size_t()
        ptr = lib().orc_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        dtype, cols, rows = abi.linear_buffer_layout(buffer_id, self.W, self.H, params)
        assert nbytes.value == rows * cols * np.dtype(dtype).itemsize, (buffer_id, nbytes.value, rows, cols)
        raw = (C.c_uint8 * nbytes.value).from_address(ptr)
        arr = np.frombuffer(raw, dtype=dtype).reshape(rows, cols)
        return arr.copy() if copy else arr

    def restir_rearch(self, params, pass_id: int, threads: int = 0) -> int:
        """rearchitected ReSTIR passes (RESTIR_PRESAMPLE_LIGHTS .. RESTIR_SHADE_AND_RESAMPLE); returns shadow rays traced"""
        return int(lib().orc_restir_rearch(self.h, C.byref(params), pass_id, threads))

    def regir_build_cells(self, params, frame_index: int, temporal: bool, threads: int = 0):
        lib().orc_regir_build_cells(self.h, C.byref(params), frame_index & 0xFFFFFFFF, 1 if temporal else 0, threads)

    def regir_update_access(self, params, frame_index: int):
        lib().orc_regir_update_access(self.h, C.byref(params), frame_index & 0xFFFFFFFF)

    def nrc_shard(self, rank: int, world: int):
        """the oracle's gfx_nrc_shard: the two collectives go through the default torch.distributed group (gloo in the CPU tests)"""
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
        self._shard_callbacks = (NRC_EXCHANGE_FN(exchange), NRC_SUM_FN(total))  # keep the thunks alive
        lib().orc_nrc_set_shard(self.h, rank, world, self._shard_callbacks[0], self._shard_callbacks[1], None)

    def nrc_preprocess(self, params, offset_unbiased_tile: int, offset_training_path: int, new_sequence: bool):
        lib().orc_nrc_preprocess(self.h, C.byref(params), offset_unbiased_tile, offset_training_path, 1 if new_sequence else 0)

    def nrc_accumulate(self, params):
        lib().orc_nrc_accumulate(self.h, C.byref(params))

    def nrc_propagate(self, params):
        lib().orc_nrc_propagate(self.h, C.byref(params))

    def nrc_shuffle(self, params):
        lib().orc_nrc_shuffle(self.h, C.byref(params))


class OracleSvgf:
    def __init__(self, oframe: OracleFrame):
        self.oframe = oframe
        self.W, self.H = oframe.W, oframe.H
        self.h = lib().orc_svgf_create(oframe.h, oframe.W, oframe.H)

    def close(self):
        if self.h:
            lib().orc_svgf_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def run(self, params, pass_id: int, stage: int = 0, threads: int = 0) -> int:
        """GFX_OK, or GFX_ERR_INVALID_ARGUMENT (-1) for the variance and a-trous passes on a frame under 2x2 pixels"""
        return lib().orc_svgf_pass(self.h, C.byref(params), pass_id, stage, threads)

    def buffer(self, buffer_id: int, index: int = 0, copy: bool = True) -> np.ndarray:
        """copy=False returns a writable view of the oracle's memory"""
        nbytes = C.c_size_t()
        ptr = lib().orc_svgf_buffer_ptr(self.h, buffer_id, index, C.byref(nbytes))
        dtype, comps, planes = abi.BUFFER_LAYOUT[buffer_id]
        raw = (C.c_uint8 * nbytes.value).from_address(ptr)
        arr = np.frombuffer(raw, dtype=dtype)
        arr = arr.copy() if copy else arr
        return arr.reshape(self.H, self.W, comps) if comps > 1 else arr.reshape(self.H, self.W)


class OracleNrc:
    """CPU restatement of NeuralRadianceCache (network_interface.cu) — see oracle/nrc.cpp."""

    def __init__(self, num_hidden_layers: int = 2, learning_rate: float = 1e-2):
        self.h = lib().orc_nrc_create(num_hidden_layers, learning_rate)
        self.num_params = lib().orc_nrc_num_params(self.h)
        self.num_matrix_weights = lib().orc_nrc_num_matrix_weights(self.h)

    def close(self):
        if self.h:
            lib().orc_nrc_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def set_params(self, params_f16: np.ndarray):
        p = np.ascontiguousarray(params_f16, dtype=np.float16)
        assert p.shape[0] == self.num_params
        lib().orc_nrc_set_params(self.h, p.ctypes.data)

    def get_params(self, ema: bool = True) -> np.ndarray:
        out = np.empty(self.num_params, dtype=np.float16)
        lib().orc_nrc_get_params(self.h, out.ctypes.data, 1 if ema else 0)
        return out

    def set_accumulate_half(self, on: bool):
        """fully-connected layers with tiny-cuda-nn's half accumulator fragments (oracle/nrc.cpp header) instead of fp32"""
        lib().orc_nrc_set_accumulate_half(self.h, 1 if on else 0)

    def init_master(self, master_f32: np.ndarray):
        """the state of a fresh tcnn::Trainer: fp32 master weights, their halves as training weights, zero EMA weights"""
        m = np.ascontiguousarray(master_f32, dtype=np.float32)
        assert m.shape[0] == self.num_params
        lib().orc_nrc_init_master(self.h, m.ctypes.data)

    def get_master(self) -> np.ndarray:
        out = np.empty(self.num_params, dtype=np.float32)
        lib().orc_nrc_get_master(self.h, out.ctypes.data)
        return out

    def get_gradients(self) -> np.ndarray:
        out = np.empty(self.num_params, dtype=np.float32)
        assert lib().orc_nrc_get_gradients(self.h, out.ctypes.data) == 0, "no training step yet"
        return out

    def encode(self, queries: np.ndarray, ema: bool = True) -> np.ndarray:
        q = np.ascontiguousarray(queries, dtype=np.float32)
        out = np.empty((q.shape[0], 64), dtype=np.float16)
        lib().orc_nrc_encode(self.h, q.ctypes.data, q.shape[0], out.ctypes.data, 1 if ema else 0)
        return out

    def infer(self, queries: np.ndarray) -> np.ndarray:
        q = np.ascontiguousarray(queries, dtype=np.float32)
        out = np.empty((q.shape[0], 3), dtype=np.float32)
        lib().orc_nrc_infer(self.h, q.ctypes.data, out.ctypes.data, q.shape[0])
        return out

    def train(self, queries: np.ndarray, targets: np.ndarray) -> float:
        q = np.ascontiguousarray(queries, dtype=np.float32)
        t = np.ascontiguousarray(targets, dtype=np.float32)
        return float(lib().orc_nrc_train(self.h, q.ctypes.data, t.ctypes.data, q.shape[0]))


def rays_traced(reset: bool = True) -> int:
    """rays the oracle's renderer entry points traced since the last reset"""
    return int(lib().orc_rays_traced(1 if reset else 0))


def primary_rays(params, width: int, height: int) -> np.ndarray:
    rays = np.zeros(width * height, dtype=abi.RAY_DTYPE)
    lib().orc_generate_primary_rays(C.byref(params), width, height, rays.ctypes.data)
    return rays
