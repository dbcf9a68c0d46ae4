"""BASELINE.json's full size (config 2: 2.87 M triangles, 1106 instances, 1920x1080), where the CPU oracle is too slow to
be the checker: size-independent properties of the CUDA path instead.
  * the three GPU-built BVHs (SAH, PLOC, LBVH) pass the oracle's structural validation (every triangle referenced, boxes
    contain subtrees), and the SAH and LBVH trees equal their CPU restatement node for node (oracle/gpu_bvh.cpp);
  * closest hits do not depend on the BVH: SAH tree == PLOC tree == LBVH tree, bit for bit, on primary + random rays (the
    canonical tie-break makes the answer a function of the triangles alone);
  * any-hit answers agree between the three trees;
  * a ReSTIR frame sequence is deterministic and equals the same sequence rendered as three row strips;
  * a sample of pixels of the first frame equals the oracle evaluated on just those rows (80-row strip), and so do three
    accumulated frames with temporal + spatial reuse (160-row strip, the 40 rows whose history stays inside it)."""
import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
BVH_BUILD_FAST = 0x100


def _render(ctx, scene, frames, strips=None):
    ctx.create_frame(W, H)
    p = abi.default_frame_params(scene, W, H)
    for f in range(frames):
        p.numAccumFrames = f
        ctx.build_light_distributions(f % 2)
        for kind, pid in engine.restir_frame_passes(p, f, 1, True, False):
            for y0, rows in (strips or [(0, 0)]):
                p.tileOriginY, p.tileRows = y0, rows
                ctx.gbuffer(p) if kind == "gbuffer" else ctx.restir(p, pid)
        p.tileOriginY, p.tileRows = 0, 0
    return ctx.download(abi.BUF_BEAUTY_ACCUM), ctx.download(abi.BUF_RNG)


def test_config2_full_size_properties(gfx_ctx, oracle):
    scene = scenes.bistro_class_scene()
    gfx_ctx.upload_scene(scene)
    p = abi.default_frame_params(scene, W, H)
    rng = np.random.default_rng(11)
    rays = oracle.primary_rays(p, W, H)[::5].copy()
    lo, hi = np.array(p.sceneAabbMin[:]), np.array(p.sceneAabbMax[:])
    extra = np.zeros(300000, dtype=abi.RAY_DTYPE)
    extra["org"] = (lo + (hi - lo) * rng.uniform(0, 1, size=(len(extra), 3))).astype(np.float32)
    d = rng.normal(size=(len(extra), 3))
    extra["dir"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    extra["tmax"] = np.float32(3.402823466e+38)
    rays = np.concatenate([rays, extra])

    results = {}
    exported = {}
    for tag, flags in (("sah", 0), ("ploc", 0x200), ("lbvh", BVH_BUILD_FAST)):
        gfx_ctx.build_bvh(flags)
        info = gfx_ctx.bvh_info()
        assert info.numTriangles == scene.num_triangles == info.numPrimRefs
        results[tag] = (gfx_ctx.trace(rays, abi.TRACE_CLOSEST), gfx_ctx.trace(rays, abi.TRACE_ANY))
        exported[tag] = gfx_ctx.export_bvh()
    a = results["ploc"][0]
    for tag in ("sah", "lbvh"):
        b = results[tag][0]
        for field in ("dist", "primIndex", "geomIndex", "instIndex", "bcB", "bcC"):
            assert np.array_equal(a[field].view(np.uint32), b[field].view(np.uint32)), f"closest hits differ between PLOC and {tag} in {field}"
        assert np.array_equal(results["ploc"][1]["dist"].view(np.uint32), results[tag][1]["dist"].view(np.uint32)), f"visibility differs ({tag})"
    assert 0.5 < float((a["primIndex"] != 0xFFFFFFFF).mean()) <= 1.0

    # structural validation of all three trees by the oracle's checker (no oracle SBVH build: import only), and the SAH (its
    # huge nodes take the multi-block split) and LBVH trees node for node against their CPU restatement (oracle/gpu_bvh.cpp)
    restated = oracle.OracleScene(scene, build_bvh=False)
    for tag, flags in (("sah", 0), ("lbvh", BVH_BUILD_FAST), ("ploc", 0x200)):
        checker = oracle.OracleScene(scene, build_bvh=False)
        checker.import_bvh(*exported[tag])
        assert checker.validate() == "", tag
        if tag != "ploc":
            levels = restated.build_gpu_style(flags)
            assert tag == "lbvh" or levels[:, 2].max() >= 2, levels[:6]
            diff = restated.same_tree(checker)
            assert diff == "", f"GPU {tag} tree differs from the restatement at {diff}"
    nodes, refs, tris = exported["ploc"]
    gfx_ctx.build_bvh(0)
    # and the restated CPU traverser walking the GPU tree agrees with the GPU traverser on a sample of the rays
    sample = rays[::97].copy()
    cpu_hits = checker.trace(sample, oracle.TRACE_CANONICAL)
    gpu_hits = a[::97]
    for field in ("dist", "primIndex", "geomIndex", "bcB", "bcC"):
        assert np.array_equal(cpu_hits[field].view(np.uint32), gpu_hits[field].view(np.uint32)), f"CPU walk of the GPU BVH differs in {field}"

    # the oracle on a strip of the full-size frame (it walks the imported GPU tree: hits do not depend on the tree):
    # frame 0 = G-buffer, initial RIS, spatial reuse, shading on rows 500..579; compared on the inner rows 530..549,
    # whose 20-pixel spatial neighbourhood lies inside the strip
    beauty0, _ = _render(gfx_ctx, scene, 1)
    oframe = oracle.OracleFrame(checker, W, H)
    po = abi.default_frame_params(scene, W, H)
    po.tileOriginY, po.tileRows = 500, 80
    for kind, pid in engine.restir_frame_passes(po, 0, 1, True, False):
        oframe.gbuffer(po) if kind == "gbuffer" else oframe.restir(po, pid)
    want = oframe.buffer(abi.BUF_BEAUTY_ACCUM)[530:550]
    assert np.array_equal(beauty0[530:550].view(np.uint32), want.view(np.uint32)), "full-size frame differs from the oracle strip"

    # the same for the temporal frames: three accumulated frames (initial; temporal + spatial; temporal + spatial) against the
    # oracle on rows 460..619.  Every frame's spatial gather reaches 20 rows, so the rows whose whole history lies inside the
    # strip shrink by 20 per frame: 520..559 after frame 2 (static camera: temporal reuse stays on the pixel).
    beauty012, _ = _render(gfx_ctx, scene, 3)
    oframe3 = oracle.OracleFrame(checker, W, H)
    po = abi.default_frame_params(scene, W, H)
    for f in range(3):
        po.numAccumFrames = f
        for kind, pid in engine.restir_frame_passes(po, f, 1, True, False):
            po.tileOriginY, po.tileRows = 460, 160
            oframe3.gbuffer(po) if kind == "gbuffer" else oframe3.restir(po, pid)
    want3 = oframe3.buffer(abi.BUF_BEAUTY_ACCUM)[520:560]
    assert np.array_equal(beauty012[520:560].view(np.uint32), want3.view(np.uint32)), "full-size temporal frames differ from the oracle strip"

    # determinism + strip sharding at full resolution (3 frames: initial, temporal, temporal)
    beauty1, rng1 = _render(gfx_ctx, scene, 3)
    beauty2, rng2 = _render(gfx_ctx, scene, 3)
    assert np.array_equal(beauty1.view(np.uint32), beauty2.view(np.uint32)) and np.array_equal(rng1, rng2), "frame sequence is not deterministic"
    beauty3, rng3 = _render(gfx_ctx, scene, 3, strips=[(0, 400), (400, 400), (800, 280)])
    assert np.array_equal(beauty1.view(np.uint32), beauty3.view(np.uint32)) and np.array_equal(rng1, rng3), "strips differ from the full frame"
    assert np.isfinite(beauty1).all() and beauty1[..., :3].mean() > 1e-3
