"""Golden fixtures (tests/golden/golden_r01.*, written by tests/golden/make_golden.py from the CPU oracle when GPU
parity was established).  CPU: the oracle still reproduces them bit for bit (guards the checker against drift).
GPU: the CUDA path reproduces them without consulting the oracle at run time.  The nrc_contribution digest of golden_r01 is
the one regenerated after the NRC path tracer stopped rendering the training continuation of a path that had ended in the
cache (DESIGN.md); no other digest moved with that change."""
import hashlib
import os

import numpy as np
import pytest

from gfxexp_b200 import abi, scenes
from tests.golden import make_golden as G

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load():
    digests = {}
    with open(os.path.join(GOLDEN_DIR, "golden_r01.sha256")) as f:
        for line in f:
            h, name = line.split()[:2]
            digests[name] = h
    arrays = dict(np.load(os.path.join(GOLDEN_DIR, "golden_r01.npz")))
    return digests, arrays


def _check(res, digests, arrays):
    assert set(res) == set(digests)
    for name, arr in res.items():
        if name in arrays:
            a, b = np.ascontiguousarray(arr), arrays[name]
            assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{name} differs from the golden image"
        assert hashlib.sha256(np.ascontiguousarray(arr).tobytes()).hexdigest() == digests[name], f"{name} differs from its golden digest"


def test_oracle_reproduces_golden_frames(oracle):
    digests, arrays = _load()
    _check(G.run_all(G.OracleBackend(scenes.tiny_city_scene())), digests, arrays)


def test_oracle_reproduces_extra_golden(oracle):
    """output side + instance animation (SURVEY.md §8f-4, §8f-2): CPU-only digests, see make_golden_extra.py"""
    from tests.golden import make_golden_extra as GX
    want = {}
    with open(os.path.join(GOLDEN_DIR, "golden_r01_extra.sha256")) as f:
        for line in f:
            h, name = line.split()[:2]
            want[name] = h
    got = GX.run_all()
    assert set(got) == set(want)
    for name, arr in got.items():
        assert GX.digest(arr) == want[name], f"{name} differs from its golden digest"


def test_oracle_reproduces_r02_golden(oracle):
    """environment light, image textures, ingestion (round 2): CPU-only digests, see make_golden_r02.py"""
    from tests.golden import make_golden_r02 as G2
    want = {}
    with open(os.path.join(GOLDEN_DIR, "golden_r02.sha256")) as f:
        for line in f:
            h, name = line.split()[:2]
            want[name] = h
    got = G2.run_all()
    assert set(got) == set(want)
    for name, arr in got.items():
        assert G2.digest(arr) == want[name], f"{name} differs from its golden digest"


class _GpuBackend:
    def __init__(self, ctx, scene):
        self.ctx, self.scene = ctx, scene
        ctx.upload_scene(scene)
        ctx.build_bvh()
        self.reset()

    def reset(self): self.ctx.create_frame(G.W, G.H)
    def light_dist(self, i): self.ctx.build_light_distributions(i)
    def gbuffer(self, p): self.ctx.gbuffer(p)
    def restir(self, p, pass_id): self.ctx.restir(p, pass_id)
    def pathtrace(self, p, variant): self.ctx.pathtrace(p, variant)
    def regir_build(self, p, f, t): self.ctx.regir_build_cells(p, f, t)
    def regir_update(self, p, f): self.ctx.regir_update_access(p, f)
    def nrc_preprocess(self, p, a, b, new): self.ctx.nrc_preprocess(p, a, b, new)
    def buffer(self, buf, idx=0): return self.ctx.download(buf, idx)
    def linear(self, buf, idx=0, params=None): return self.ctx.download_linear(buf, idx, params=params)


@pytest.mark.gpu
def test_gpu_reproduces_golden_frames(gfx_ctx):
    digests, arrays = _load()
    _check(G.run_all(_GpuBackend(gfx_ctx, scenes.tiny_city_scene())), digests, arrays)
