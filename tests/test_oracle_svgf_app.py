"""CPU checks of the oracle's SVGF-app path tracer (GFX_PT_SVGF, oracle/svgf_app.cpp) that do not lean on the reference:
a white furnace through the path tracer and the temporal pass, what specular mollification may and may not change, and the
first vertex's albedo against a numpy restatement of evaluateDHReflectanceEstimate in the makeCoordinateSystem frame."""
import math

import numpy as np

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_svgf_app as OA


def _furnace_scene(radiance, albedo):
    mats = np.zeros(1, dtype=scenes.MATERIAL_DTYPE)
    mats[0]["p0"] = np.float32(albedo)
    mats[0]["bsdfType"] = scenes.BSDF_LAMBERT
    plane = scenes.make_quad_light(4000.0, 0)                         # a quad in the xz-plane facing -y, not emissive here
    ori = scenes.rot_x(-90.0).astype(np.float32)                      # the camera looks along +y, up at the quad
    scene = scenes.Scene([plane], mats, [scenes.make_instance([0])], np.array([0.0, -100.0, 0.0], dtype=np.float32), ori,
                         math.radians(50.0), "furnace")
    env = np.ones((16, 32, 4), dtype=np.float32)
    env[..., :3] = radiance
    scene.env_map = env
    return scene


def _frame(fr, sv, p, frame_index, after_temporal=None, **kw):
    for kind, pid, stage in engine.svgf_app_frame_passes(p, frame_index, **kw):
        if kind == "gbuffer":
            fr.gbuffer(p)
        elif kind == "pathtrace":
            fr.pathtrace(p, pid)
        elif kind == "svgf" and sv is not None:
            sv.run(p, pid, stage)
            if pid == abi.SVGF_TEMPORAL_ACCUMULATE and after_temporal is not None:
                after_temporal()


def test_white_furnace():
    """a Lambert plane of albedo rho under a uniform environment L: the beauty averages rho L, the demodulated lighting L"""
    L, rho, coeff = 2.0, 0.5, 1.5
    scene = _furnace_scene(L, rho)
    w = h = 24
    fr = OA.Frame(scene, w, h)
    sv = OA.Svgf(fr)
    p = abi.default_frame_params(scene, w, h)
    p.envLightPowerCoeff = coeff
    p.maxPathLength = 5
    beauty, lighting = [], []
    for f in range(16):
        _frame(fr, sv, p, f, after_temporal=lambda: lighting.append(sv.buffer(abi.BUF_SVGF_LIGHTING_VARIANCE, 0)[..., :3]))
        beauty.append(fr.buffer(abi.BUF_BEAUTY_ACCUM)[..., :3])
    assert (fr.buffer(abi.BUF_GBUFFER0, p.bufferIndex)[..., 0] != 0xFFFFFFFF).all(), "the camera must see the plane only"
    albedo = fr.buffer(abi.BUF_ALBEDO_ACCUM)
    assert np.all(albedo[..., :3] == np.float32(rho)), "Lambert: the DH reflectance is the albedo"
    assert abs(np.mean(beauty) / (rho * L * coeff) - 1) < 0.02, np.mean(beauty)
    assert abs(np.mean(lighting) / (L * coeff) - 1) < 0.02, np.mean(lighting)


def test_white_furnace_feedback_pass():
    """SVGF off, temporal accumulation on: feedbackNoisyLighting hands the temporal pass's lighting to the next frame, and
    the final image is that lighting times the albedo (stage 0's plane)"""
    L, rho, coeff = 2.0, 0.5, 1.5
    scene = _furnace_scene(L, rho)
    w = h = 24
    fr = OA.Frame(scene, w, h)
    sv = OA.Svgf(fr)
    p = abi.default_frame_params(scene, w, h)
    p.envLightPowerCoeff = coeff
    p.svgfFlags &= ~abi.SVGF_ENABLE_TAA
    for f in range(8):
        _frame(fr, sv, p, f, enable_svgf=False)
        lighting = sv.buffer(abi.BUF_SVGF_LIGHTING_VARIANCE, 0)
        assert np.array_equal(sv.buffer(abi.BUF_SVGF_PREV_LIGHTING).view(np.uint32), lighting.view(np.uint32))
        final = sv.buffer(abi.BUF_SVGF_FINAL, p.bufferIndex)[..., :3]
        assert np.array_equal(final, lighting[..., :3] * np.float32(rho))
    assert abs(float(lighting[..., :3].mean()) / (L * coeff) - 1) < 0.05


def _render(scene, w, h, max_path_length, mollify, frames=1):
    fr = OA.Frame(scene, w, h)
    p = abi.default_frame_params(scene, w, h)
    p.maxPathLength = max_path_length
    out = []
    for f in range(frames):
        _frame(fr, None, p, f, mollify=mollify)
        out.append(fr.buffer(abi.BUF_BEAUTY_ACCUM).copy())
    return np.stack(out), fr.buffer(abi.BUF_RNG), fr


def test_mollification_changes_bounces_only():
    """no bounce sets up a BSDF at maxPathLength 2: mollification cannot change a bit; at 5, on a glossy scene, it does"""
    scene = scenes.tiny_city_scene()
    w, h = 64, 40
    on2, rng_on2, _ = _render(scene, w, h, 2, True, 2)
    off2, rng_off2, _ = _render(scene, w, h, 2, False, 2)
    assert np.array_equal(on2.view(np.uint32), off2.view(np.uint32)) and np.array_equal(rng_on2, rng_off2)
    on5, _, _ = _render(scene, w, h, 5, True)
    off5, _, _ = _render(scene, w, h, 5, False)
    assert not np.array_equal(on5.view(np.uint32), off5.view(np.uint32))
    assert np.isfinite(on5).all() and np.isfinite(off5).all()


def _f32(x):
    return np.float32(x)


def _make_coordinate_system(n):
    sign = _f32(1.0) if n[2] >= 0 else _f32(-1.0)
    a = _f32(-1.0) / (sign + n[2])
    b = n[0] * n[1] * a
    t = np.array([1 + sign * n[0] * n[0] * a, sign * b, -sign * n[0]], dtype=np.float32)
    bt = np.array([b, sign + n[1] * n[1] * a, -n[1]], dtype=np.float32)
    return t, bt


def _dh_reflectance(mat, v_local):
    """evaluateDHReflectanceEstimate (common_device.cuh:372-374, 736-764) after BSDF::setup of a constant material"""
    p0, p1, p2 = (np.asarray(mat["p0"], np.float64), np.asarray(mat["p1"], np.float64), float(mat["p2"]))
    if mat["bsdfType"] == scenes.BSDF_LAMBERT:
        return p0
    if mat["bsdfType"] == 1:
        diffuse, f0, roughness = p0, p1, 1 - min(p2, 0.999)
    else:
        metallic = p1[2]
        diffuse = p0 * (1 - metallic)
        f0 = 0.16 * 0.25 * (1 - metallic) + p0 * metallic
        roughness = 1 - min(1 - p1[1], 0.999)
    cos_v = abs(v_local[2])
    f_d90 = 0.5 * roughness + 2 * roughness * cos_v ** 2
    diff_f = 1 + (f_d90 - 1) * (1 - cos_v) ** 5
    diffuse_dhr = diffuse * diff_f * (1 + (1 / 1.51 - 1) * roughness)
    spec_dhr = f0 + (1 - f0) * ((1 - cos_v) ** 5 * (1 - roughness))
    return np.minimum(diffuse_dhr + spec_dhr, 1.0)


def test_albedo_is_dh_reflectance_in_the_normal_frame():
    scene = scenes.tiny_city_scene()
    w, h = 64, 40
    fr = OA.Frame(scene, w, h)
    p = abi.default_frame_params(scene, w, h)
    _frame(fr, None, p, 0)
    gb0 = fr.buffer(abi.BUF_GBUFFER0, 0)
    albedo = fr.buffer(abi.BUF_ALBEDO_ACCUM)
    cam = np.asarray(p.camera.position[:], dtype=np.float32)
    hits = np.argwhere(gb0[..., 0] != 0xFFFFFFFF)
    assert len(hits) > 100
    rs = np.random.default_rng(5)
    checked = 0
    for y, x in hits[rs.choice(len(hits), 12, replace=False)]:
        inst_slot, mesh_slot, prim, qbc = (int(v) for v in gb0[y, x])
        inst, mesh = scene.instances[inst_slot], scene.meshes[mesh_slot]
        bc_b, bc_c = np.float32((qbc & 0xFFFF) / 65535.0), np.float32((qbc >> 16) / 65535.0)
        bc_a = 1 - (bc_b + bc_c)
        tri = mesh.triangles[prim]
        n_obj = bc_a * mesh.normals[tri[0]] + bc_b * mesh.normals[tri[1]] + bc_c * mesh.normals[tri[2]]
        pos_obj = bc_a * mesh.positions[tri[0]] + bc_b * mesh.positions[tri[1]] + bc_c * mesh.positions[tri[2]]
        n = np.asarray(inst.normal_matrix, np.float32).reshape(3, 3) @ n_obj
        n = (n / np.linalg.norm(n)).astype(np.float32)
        xf = np.asarray(inst.transform, np.float32).reshape(3, 4)
        pos = xf[:, :3] @ pos_obj + xf[:, 3]
        v_out = cam - pos
        v_out /= np.linalg.norm(v_out)
        t, bt = _make_coordinate_system(n)
        v_local = np.array([t @ v_out, bt @ v_out, n @ v_out])
        want = _dh_reflectance(scene.materials[mesh.material], v_local)
        assert np.allclose(albedo[y, x, :3], want, rtol=2e-4, atol=2e-5), (y, x, albedo[y, x], want)
        checked += 1
    assert checked == 12
    assert np.all(albedo[gb0[..., 0] == 0xFFFFFFFF] == 0)
