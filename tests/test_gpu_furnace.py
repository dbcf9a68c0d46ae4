"""End to end against the integral: a plane under a uniform environment of radiance L (a furnace).  With one bounce, a pixel
that sees the plane at cos(theta_o) shows envLightPowerCoeff x L x albedo(cos(theta_o)), where albedo is the float64
quadrature of tests/shading_ref.py.  Unlike the oracle parity tests, this holds a rendered GPU value to an independently
computed number, at materials no test scene has: smoothness 0 to the 0.999 clamp, black, and a SimplePBR metal.

  the path tracer at maxPathLength 2 (NEE to the environment + the BSDF-sampled bounce's implicit hit, MIS): every material
  ReSTIR DI, initial RIS only, and the rearchitected ReSTIR with the unbiased estimator: smoothness <= 0.5, because their
  uniform-in-the-importance-map candidates cannot find a mirror lobe

The camera sees the plane from below, from two poses, so that the pixels cover cos(theta_o) from 1 down to about 0.05; each
pixel's cos(theta_o) comes in float64 from the camera model of the G-buffer pass (jitter off).  The residual
(image - expected) / expected is averaged in bins of cos(theta_o), and each bin's bar is derived from the spread of the
residual within it.  The same scene also runs 2 frames of each renderer against the CPU oracle, bit for bit."""
import math

import numpy as np
import pytest
from scipy.interpolate import CubicSpline

from gfxexp_b200 import abi, engine, scenes
from tests import shading_ref as R

pytestmark = pytest.mark.gpu

L_ENV, POWER = 2.0, 1.5
POSES = {"below": -90.0, "tilted": -28.0}      # rot_x pitch: the view direction's elevation above the horizontal, in degrees
W, H = 128, 96
COS_EDGES = np.array([0.05, 0.1, 0.2, 0.35, 0.5, 0.65, 0.8, 0.9, 1.0])


def _furnace_scene(mat, pitch):
    """a 4000-wide quad in the xz-plane facing -y, 100 below it the camera, and a uniform environment (restated from
    test_oracle_envlight.py's furnace)"""
    mats = np.zeros(1, dtype=scenes.MATERIAL_DTYPE)
    mats[0]["bsdfType"] = mat[0]
    mats[0]["p0"] = mat[1]
    mats[0]["p1"] = mat[2]
    mats[0]["p2"] = mat[3]
    plane = scenes.make_quad_light(4000.0, 0)
    scene = scenes.Scene([plane], mats, [scenes.make_instance([0])], np.array([0.0, -100.0, 0.0], dtype=np.float32),
                         scenes.rot_x(pitch).astype(np.float32), math.radians(50.0), "furnace")
    env = np.ones((16, 32, 4), dtype=np.float32)
    env[..., :3] = L_ENV
    scene.env_map = env
    return scene


def _cos_theta_o(p):
    """cos(theta_o) of every pixel centre in float64: direction = orientation (vw (0.5 - fx), vh (0.5 - fy), 1) as the
    G-buffer pass builds it, vh = 2 tan(fovY / 2); the plane's normal is -y, so cos(theta_o) = dot(-direction, n) = dir.y"""
    cam = p.camera
    o = np.array(cam.orientation[:], dtype=np.float64).reshape(3, 3)
    vh = 2 * math.tan(cam.fovY * 0.5)
    vw = cam.aspect * vh
    fx = (np.arange(W) + 0.5) / W
    fy = (np.arange(H) + 0.5) / H
    gx, gy = np.meshgrid(fx, fy)
    d = np.stack([vw * (0.5 - gx), vh * (0.5 - gy), np.ones_like(gx)], -1) @ o.T
    return d[..., 1] / np.linalg.norm(d, axis=-1)


def _albedo_curve(mat):
    b = R.setup(*mat)
    nodes = np.concatenate([np.linspace(0.04, 0.2, 17), np.linspace(0.21, 1.0, 40)])
    vals = np.array([R.albedo(b, c) for c in nodes])
    return CubicSpline(nodes, vals, axis=0)


def _render(ctx, scene, renderer, frames, oframe=None):
    ctx.upload_scene(scene)
    ctx.build_bvh()
    ctx.create_frame(W if oframe is None else oframe[1], H if oframe is None else oframe[2])
    p = abi.default_frame_params(scene, W if oframe is None else oframe[1], H if oframe is None else oframe[2])
    p.envLightPowerCoeff = POWER
    p.maxPathLength = 2
    fr = oframe[0] if oframe is not None else None
    for f in range(frames):
        p.numAccumFrames = f
        ctx.build_light_distributions(f % 2)
        if renderer == "pathtrace":
            p.frameIndex, p.bufferIndex = f, f % 2
            passes = [("gbuffer", -1), ("pathtrace", -1)]
        elif renderer == "restir":
            passes = list(engine.restir_frame_passes(p, f, 0, temporal=False))
        else:
            passes = list(engine.restir_rearch_frame_passes(p, f, temporal=False, spatial=False, unbiased=True))
        for kind, pid in passes:
            if kind == "gbuffer":
                ctx.gbuffer(p)
                fr is not None and fr.gbuffer(p)
            elif kind == "pathtrace":
                ctx.pathtrace(p)
                fr is not None and fr.pathtrace(p)
            else:
                ctx.restir(p, pid)
                if fr is not None:
                    fr.restir(p, pid) if renderer == "restir" else fr.restir_rearch(p, pid)
    ctx.synchronize()
    return p


# (bsdfType, p0, p1, p2) — SimplePBR: p1 = (occlusion, roughness, metallic)
COLOUR, F0 = (0.5, 0.4, 0.3), (0.04, 0.04, 0.04)
PT_MATERIALS = {
    "lambert": (0, COLOUR, (0, 0, 0), 0.0),
    "ds-s0": (1, COLOUR, F0, 0.0),
    "ds-s0.5": (1, COLOUR, F0, 0.5),
    "ds-s0.9": (1, COLOUR, F0, 0.9),
    "ds-s0.99": (1, COLOUR, F0, 0.99),
    "ds-s0.999": (1, COLOUR, F0, 0.999),
    "ds-white-s0.78": (1, (1, 1, 1), (1, 1, 1), 0.78),
    "ds-black-s0.5": (1, (0, 0, 0), (0, 0, 0), 0.5),
    "pbr-grey-metal-s1.0": (2, (0.5, 0.5, 0.5), (1.0, 0.0, 1.0), 0.0),
}
LIGHT_MATERIALS = ("lambert", "ds-s0", "ds-s0.5")


def _residual_bins(img, expected, cos_o, hit):
    """per bin of cos(theta_o): (n, mean, standard error) of the channel-averaged residual (image - expected) / expected"""
    r = ((img.astype(np.float64) - expected) / expected).mean(-1)
    out = []
    for lo, hi in zip(COS_EDGES[:-1], COS_EDGES[1:]):
        sel = hit & (cos_o >= lo) & (cos_o < hi)
        if sel.sum() >= 30:
            v = r[sel]
            out.append((lo, hi, int(sel.sum()), float(v.mean()), float(v.std(ddof=1) / math.sqrt(sel.sum()))))
    return out


@pytest.mark.parametrize("renderer,name", [("pathtrace", m) for m in PT_MATERIALS]
                         + [(r, m) for r in ("restir", "rearch") for m in LIGHT_MATERIALS])
def test_furnace_against_the_albedo(gfx_ctx, renderer, name):
    """Each bin's mean residual is within 5 standard errors of 0 (pixels are independent: no reuse across pixels or
    frames), plus 2e-4 for the float32 sampler and the 64 float32 accumulation steps; a bias that shows in the bins is a
    wrong BSDF, pdf or light-sampling weight."""
    mat = PT_MATERIALS[name]
    curve = _albedo_curve(mat)
    frames = 64
    covered = []
    for pose, pitch in POSES.items():
        scene = _furnace_scene(mat, pitch)
        p = _render(gfx_ctx, scene, renderer, frames)
        cos_o = _cos_theta_o(p)
        hit = gfx_ctx.download(abi.BUF_GBUFFER0, p.bufferIndex)[..., 0] != 0xFFFFFFFF
        hit &= cos_o > 0.045
        img = gfx_ctx.download(abi.BUF_BEAUTY_ACCUM)[..., :3]
        assert np.isfinite(img[hit]).all()
        expected = POWER * L_ENV * curve(np.clip(cos_o, 0.04, 1.0))
        for lo, hi, n, mean, se in _residual_bins(img, expected, cos_o, hit):
            covered.append((lo, hi))
            assert abs(mean) <= 5 * se + 2e-4, f"{pose} cos [{lo}, {hi}): mean residual {mean:.2e}, se {se:.2e}, n {n}"
    assert min(lo for lo, _ in covered) <= 0.05 and max(hi for _, hi in covered) >= 1.0


PARITY_MATERIALS = ("ds-s0", "ds-s0.999", "ds-black-s0.5", "pbr-grey-metal-s1.0", "lambert")


@pytest.mark.parametrize("renderer", ["pathtrace", "restir", "rearch"])
def test_furnace_gpu_equals_oracle(gfx_ctx, oracle, renderer):
    """2 frames of each renderer on the furnace scene, at fully rough, near-mirror, black and metal materials, from the
    tilted pose (cos(theta_o) down to 0.05): beauty and RNG state equal the oracle's bit for bit"""
    w, h = 64, 48
    for name in PARITY_MATERIALS:
        scene = _furnace_scene(PT_MATERIALS[name], POSES["tilted"])
        oscene = oracle.OracleScene(scene)
        oframe = oracle.OracleFrame(oscene, w, h)
        _render(gfx_ctx, scene, renderer, 2, (oframe, w, h))
        for buf in (abi.BUF_BEAUTY_ACCUM, abi.BUF_RNG):
            got, want = gfx_ctx.download(buf), oframe.buffer(buf)
            g = got.view(np.uint32) if got.dtype != np.uint64 else got
            wv = want.view(np.uint32) if want.dtype != np.uint64 else want
            assert np.array_equal(g, wv), f"{name} buffer {buf}: {int(np.count_nonzero(g != wv))} elements differ"
