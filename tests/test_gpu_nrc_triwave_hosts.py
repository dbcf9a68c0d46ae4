"""The triangle-wave NRC network through the hosts: the headless C++ host's `-position-encoding tri` frames equal the Python host's
bit for bit, and (with two GPUs; skipped otherwise) the ReSTIR DI + NRC strip frames with a triangle-wave net equal one GPU's."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gfxexp_b200", "gfx_headless")
TRI = abi.NRC_POSITION_ENCODING_TRIANGLE_WAVE


def _tri_params():
    return engine.random_nrc_params(64 * 64 * 2 + 16 * 64, 64 * 64 * 2 + 16 * 64, seed=77)


def test_cpp_host_triangle_wave_frames_match_python_host(gfx_ctx, tmp_path):
    W, H, FRAMES = 96, 64, 3
    scene = scenes.tiny_city_scene()
    scene_path, out_path, params_path = (str(tmp_path / n) for n in ("scene.bin", "out.raw", "nrc.f16"))
    scenes.save_scene_bin(scene, scene_path, W, H)
    _tri_params().tofile(params_path)
    res = subprocess.run([HOST, scene_path, "nrc", str(W), str(H), str(FRAMES), out_path, params_path, "-position-encoding", "tri"],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    assert json.loads(res.stdout.strip().splitlines()[-1])["renderer"] == "nrc"
    got = np.fromfile(out_path, dtype=np.float32).reshape(H, W, 4)

    gfx_ctx.upload_scene(scene)
    gfx_ctx.build_bvh()
    gfx_ctx.create_frame(W, H)
    p = abi.default_frame_params(scene, W, H)
    net = engine.NeuralRadianceCache(gfx_ctx, 2, 1e-2, position_encoding=TRI)
    net.set_params(_tri_params())
    rs = np.random.RandomState(72139121)  # std::mt19937 perFrameRng(72139121)
    for f in range(FRAMES):
        p.numAccumFrames = f
        gfx_ctx.build_light_distributions(f % 2)
        gfx_ctx.nrc_frame(net, p, f, [int(v) for v in rs.randint(0, 2 ** 32, size=2, dtype=np.uint64)], train=True)
    want = gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)
    net.close()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "C++ host image differs from the Python host image"
    assert np.isfinite(got).all() and got[..., :3].mean() > 1e-4

    # a parameter file of the hash-grid network's size is refused by the triangle-wave host
    np.zeros(64 * 64 * 2 + 16 * 64 + 991232, dtype=np.float16).tofile(params_path)
    res = subprocess.run([HOST, scene_path, "nrc", str(W), str(H), "1", out_path, params_path, "-position-encoding", "tri"],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode != 0 and "9216 halves" in res.stderr, res.stderr


W2, H2, NRC_FRAMES = 320, 192, 4


def _offsets(f):
    rng = np.random.default_rng(1000 + f)
    return [int(rng.integers(0, 2 ** 32)) for _ in range(2)]


def _worker_restir_nrc_tri(rank, world, port, result_path):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from gfxexp_b200 import multigpu
    scene = scenes.small_city_scene()
    ctx = engine.Context(rank)
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(W2, H2)
    p = abi.default_frame_params(scene, W2, H2)
    p.maxPathLength = 5
    net = engine.NeuralRadianceCache(ctx, 2, 1e-2, position_encoding=TRI)
    driver = multigpu.StripDriver(ctx, p, W2, H2, rank, world)
    driver.enable_nrc(net)
    outs = []
    for f in range(NRC_FRAMES):
        p.numAccumFrames = f
        driver.render_restir_nrc_frame(f, _offsets(f))
        torch.cuda.synchronize()
        outs.append(driver.composited.cpu().numpy().copy())
    np.save(result_path + f".weights.{rank}.npy", net.read(abi.NRC_READ_MASTER))
    if rank == 0:
        np.save(result_path + ".frames.npy", np.stack(outs))
    dist.barrier()
    net.close()
    driver.comm.close()
    dist.destroy_process_group()
    ctx.close()


def test_restir_nrc_strips_with_triangle_wave_net_equal_single_gpu(tmp_path, gfx_ctx):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    result = str(tmp_path / "restir_nrc_tri")
    mp.spawn(_worker_restir_nrc_tri, args=(2, port, result), nprocs=2, join=True)
    got = np.load(result + ".frames.npy")
    scene = scenes.small_city_scene()
    ctx = gfx_ctx
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(W2, H2)
    p = abi.default_frame_params(scene, W2, H2)
    p.maxPathLength = 5
    net = engine.NeuralRadianceCache(ctx, 2, 1e-2, position_encoding=TRI)
    for f in range(NRC_FRAMES):
        p.numAccumFrames = f
        ctx.build_light_distributions(f % 2)
        for kind, pass_id in engine.restir_frame_passes(p, f, 1):
            ctx.gbuffer(p) if kind == "gbuffer" else ctx.restir(p, pass_id)
        off = _offsets(f)
        ctx.nrc_preprocess(p, off[0], off[1], f == 0)
        ctx.pathtrace(p, abi.PT_NRC)
        ctx.nrc_frame_infer(net)
        ctx.nrc_accumulate(p)
        ctx.nrc_propagate(p)
        ctx.nrc_shuffle(p)
        ctx.nrc_frame_train(net)
        ctx.synchronize()
        want = ctx.download(abi.BUF_BEAUTY_ACCUM).reshape(-1)
        assert np.array_equal(got[f].view(np.uint32), want.view(np.uint32)), f"frame {f}: sharded DI + NRC frame differs"
    want_weights = net.read(abi.NRC_READ_MASTER)
    net.close()
    for rank in range(2):
        w = np.load(result + f".weights.{rank}.npy")
        assert np.array_equal(w.view(np.uint32), want_weights.view(np.uint32)), f"rank {rank}: trained weights differ"
