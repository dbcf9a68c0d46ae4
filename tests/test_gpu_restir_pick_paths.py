"""GPU parity of the ReSTIR DI passes, bit-exact against the CPU oracle, on pick-guide buckets the city scenes do not have: pure
buckets whose light must never be culled by its bounding sphere (radius < 0: the area density is not a positive finite number,
gfxexp_b200/csrc/lighting.cuh classifyLight), next to the impure buckets that test_gpu_restir.py's scenes already cover."""
import numpy as np
import pytest
import torch

from gfxexp_b200 import abi, engine, scenes
from tests.test_gpu_restir import _compare_all, _setup

pytestmark = pytest.mark.gpu


def _bucket_keys(ctx):
    """the flattened pick's key at the first and at the last float of every pick-guide bucket (2^17 buckets)"""
    j = np.arange(1 << 17, dtype=np.uint32)
    first = (j.astype(np.float32) / np.float32(1 << 17)).view(np.uint32)
    last = np.append(first[1:] - 1, np.uint32(0x3F7FFFFF))
    ul = torch.from_numpy(np.concatenate([first, last]).view(np.float32)).cuda()
    flat = torch.empty(ul.numel(), dtype=torch.int32, device="cuda")
    chain = torch.empty_like(flat)
    ctx._check(ctx.lib.gfx_light_pick_debug(ctx.h, None, ul.data_ptr(), ul.numel(), flat.data_ptr(), chain.data_ptr()),
               "gfx_light_pick_debug")
    torch.cuda.synchronize()
    keys = flat.cpu().numpy().view(np.uint32)
    return keys[: 1 << 17], keys[1 << 17:]


@pytest.mark.parametrize("unbiased", [False, True])
def test_restir_uncullable_light_bit_exact(gfx_ctx, oracle, unbiased):
    scene = scenes.tiny_city_scene_degenerate_light()
    scene_name = scene.name
    w, h = 192, 108
    oscene, oframe = _setup(gfx_ctx, oracle, scene, w, h)
    p = abi.default_frame_params(scene, w, h)
    for frame in range(3):
        gfx_ctx.build_light_distributions(frame % 2)
        if frame == 0:
            first, last = _bucket_keys(gfx_ctx)
            pure = first == last
            # the quad far away is the last instance, so its two triangles hold the two largest light keys
            n = scene.num_emissive_triangles
            far = (first >= np.uint32(n - 2)) & (first < np.uint32(n))
            assert np.count_nonzero(pure & far) > 1000, "the degenerate light should own whole buckets"
            assert np.count_nonzero(~pure) > 100, "the scene should have impure buckets"
        for kind, pass_id in engine.restir_frame_passes(p, frame, num_spatial_passes=1, temporal=True, unbiased=unbiased):
            if kind == "gbuffer":
                gfx_ctx.gbuffer(p)
                oframe.gbuffer(p)
            else:
                gfx_ctx.restir(p, pass_id)
                oframe.restir(p, pass_id)
        gfx_ctx.synchronize()
        _compare_all(gfx_ctx, oframe, f"{scene_name} frame {frame} unbiased={unbiased}")
