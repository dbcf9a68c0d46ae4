"""Seeded scenes for the G-buffer pass's float64 restatement (tests/gbuffer_ref.py) - TEST INFRASTRUCTURE for
tests/test_oracle_gbuffer_ref.py and tests/test_gpu_gbuffer_ref.py.

About 1900 triangles, so that a brute-force closest hit over every triangle stays cheap, built to reach the G-buffer's edges:
  * boxes instanced with yaw, pitch and uniform scale (make_instance), and one box under a non-uniform scale with shear, built
    directly as an Instance: the only instance whose normal matrix is not its normalised rotation.  It carries no emitter;
  * a smooth UV sphere (interpolated normals and tangents);
  * a quad seen from behind: its geometric normal points away from the camera and stays so;
  * a textured quad whose texture coordinates run outside [0, 1], negative ones included, with tangents tilted out of the
    surface (the Gram-Schmidt step moves them);
  * a quad whose vertex normals are zero (the (0, 0, 1) fallback) and one whose vertex tangents are parallel to its normals
    (a NaN tangent under a finite normal: the fallback tests only the normal);
  * an emitter, and sky over the top of the view;
  * frame 1 moves three instances (scenes.move_instance) and translates and turns the camera.
"""
from __future__ import annotations

import numpy as np

from gfxexp_b200 import abi, scenes

F32 = np.float32
NO_TEX = 0xFFFFFFFF
# materials
M_GROUND, M_BOX, M_SPHERE, M_BACK, M_TEXTURED, M_ZERO_N, M_PARALLEL_T, M_LIGHT, M_LAMBERT, M_PBR = range(10)
# instance slots (the order of scene.instances)
I_GROUND, I_BOX_YAW, I_BOX_PITCH, I_BOX_SCALED, I_SHEAR, I_SPHERE, I_BACK, I_TEXTURED, I_ZERO_N, I_PARALLEL_T, I_LIGHT = range(11)
MOVED = (I_BOX_YAW, I_SPHERE, I_SHEAR)


def _quad(corners, normal, tangent, uv, material) -> scenes.Mesh:
    """two triangles over corners a, b, c, d (counter-clockwise), one normal / tangent per vertex or shared"""
    n = np.broadcast_to(np.asarray(normal, np.float64), (4, 3))
    t = np.broadcast_to(np.asarray(tangent, np.float64), (4, 3))
    return scenes.Mesh(np.asarray(corners, F32), np.ascontiguousarray(n, F32), np.ascontiguousarray(t, F32), np.asarray(uv, F32),
                       np.array([[0, 1, 2], [0, 2, 3]], np.uint32), material)


def _materials():
    rng = np.random.default_rng(41)
    m = np.zeros(10, dtype=scenes.MATERIAL_DTYPE)
    m["bsdfType"] = scenes.BSDF_DIFFUSE_AND_SPECULAR
    m["p0"] = rng.uniform(0.1, 0.8, (10, 3)).astype(F32)
    m["p1"] = F32(0.04)
    m["p2"] = rng.uniform(0.1, 0.9, 10).astype(F32)
    m[M_LAMBERT]["bsdfType"] = scenes.BSDF_LAMBERT
    m[M_PBR]["bsdfType"] = scenes.BSDF_SIMPLE_PBR
    m[M_PBR]["p1"] = (1.0, 0.35, 0.6)
    m[M_LIGHT]["hasEmittance"] = 1
    m[M_LIGHT]["emittance"] = (12.0, 10.0, 8.0)
    return m


def _shear_instance(mesh_slots, translate) -> scenes.Instance:
    """a non-uniform scale with shear: transform, its normal matrix transpose(inverse(upper 3x3)) and curToPrev = identity"""
    upper = np.array([[1.4, 0.5, 0.0], [0.0, 0.6, 0.3], [0.35, 0.0, 1.1]]) @ scenes.rot_y(25.0)
    xf = np.concatenate([upper, np.asarray(translate, np.float64)[:, None]], 1).astype(F32)
    nm = np.linalg.inv(xf[:, :3].astype(np.float64)).T.astype(F32)
    ident = np.zeros((3, 4), F32)
    ident[0, 0] = ident[1, 1] = ident[2, 2] = 1
    return scenes.Instance(xf, ident, nm, 1.0, list(mesh_slots))


def scene(bump: bool = False) -> scenes.Scene:
    """bump: normal and height maps on some materials (GfxSceneDesc::bumpMaps), the default texel on the rest"""
    rng = np.random.default_rng(43)
    meshes = [
        scenes.make_plane(8, 40.0, M_GROUND),                                   # 0: 128 triangles
        scenes.make_box(3, (2.0, 3.0, 2.0), M_BOX, rng, 0.05),                  # 1: 108
        scenes.make_sphere(32, 16, 1.6, M_SPHERE),                              # 2: 960
        _quad([(-1.5, 0, 0), (1.5, 0, 0), (1.5, 2.5, 0), (-1.5, 2.5, 0)], (0, 0, 1), (1, 0, 0),
              [(0, 0), (1, 0), (1, 1), (0, 1)], M_BACK),                        # 3: faces +z, seen from -z
        _quad([(-1.5, 0, 0), (1.5, 0, 0), (1.5, 2.5, 0), (-1.5, 2.5, 0)], [(0, 0, 1), (0.2, 0, 1), (0, 0.3, 1), (-0.1, 0, 1)],
              [(1, 0, 0.6), (1, 0.2, -0.4), (0.8, -0.3, 0.5), (1, 0, 0)],
              [(-2.3, -1.7), (3.1, -1.2), (2.6, 2.9), (-1.4, 1.8)], M_TEXTURED),
        _quad([(-1, 0, 0), (1, 0, 0), (1, 2, 0), (-1, 2, 0)], (0, 0, 0), (1, 0, 0),
              [(0, 0), (1, 0), (1, 1), (0, 1)], M_ZERO_N),
        _quad([(-1, 0, 0), (1, 0, 0), (1, 2, 0), (-1, 2, 0)], (0, 0, 1), (0, 0, 1),
              [(0, 0), (1, 0), (1, 1), (0, 1)], M_PARALLEL_T),
        scenes.make_quad_light(2.0, M_LIGHT),
        scenes.make_box(2, (1.0, 1.0, 1.0), M_PBR),                             # 8: 48, under the shear
        scenes.make_box(2, (1.5, 1.5, 1.5), M_LAMBERT),                         # 9: 48
    ]
    mk = scenes.make_instance
    instances = [
        mk([0], (0, 0, 0)),
        mk([1], (-4.0, 0, -2.0), yaw_deg=33.0),
        mk([9], (4.5, 0.4, -3.0), yaw_deg=-20.0, pitch_deg=17.0),
        mk([1], (1.2, 0, -7.0), yaw_deg=70.0, scale=1.6, pitch_deg=-8.0),
        _shear_instance([8], (-1.3, 0.6, 2.5)),
        mk([2], (1.8, 1.6, 0.5), yaw_deg=40.0),
        mk([3], (-6.2, 0.0, 3.0), yaw_deg=180.0 - 25.0),          # its +z face turned away from the camera
        mk([4], (5.0, 0.2, 3.0), yaw_deg=-30.0),
        mk([5], (-2.4, 0.1, 6.0), yaw_deg=10.0),
        # unrotated, so that t - (n . t) n is exactly 0 in float32 as in float64.  With the bump on, a NaN tangent makes the
        # whole bump frame NaN: the quad then stands behind the camera
        mk([6], (2.6, 0.1, 30.0 if bump else 6.5)),
        mk([7], (0.0, 5.5, -1.0)),
    ]
    eye = np.array([0.3, 3.2, 14.0])
    sc = scenes.Scene(meshes, _materials(), instances, eye.astype(F32), scenes.look_at_orientation(eye, (0.0, 2.4, 0.0)),
                      0.9, name="gbuffer")
    sc.textures = [scenes.checker_texture(24, 40, 6, seed=5), scenes.checker_texture(7, 5, 3, seed=9)]
    mt = np.full((10, 4), NO_TEX, np.uint32)
    mt[M_TEXTURED, 0] = 0
    mt[M_BOX, 0] = 1
    sc.material_textures = mt
    if bump:
        base = len(sc.textures)
        sc.textures = sc.textures + [scenes.sine_normal_map(48, 32), scenes.noise_height_map(37, 23)]
        bm = np.full((10, 2), NO_TEX, np.uint32)
        bm[:, 1] = 0
        bm[M_GROUND] = (base + 1, abi.BUMP_HEIGHT_MAP)
        bm[M_SPHERE] = (base, abi.BUMP_NORMAL_MAP)
        bm[M_TEXTURED] = (base, abi.BUMP_NORMAL_MAP)
        bm[M_BOX] = (base + 1, abi.BUMP_HEIGHT_MAP)
        sc.bump_maps = bm
    return sc


def moved_instances(sc: scenes.Scene, k: float = 1.0):
    """frame 1's instances: MOVED translated, turned and rescaled through scenes.move_instance (the sheared box is moved by its
    own translation and keeps curToPrev as prev * inverse(cur))"""
    out = list(sc.instances)
    out[I_BOX_YAW] = scenes.move_instance(sc.instances[I_BOX_YAW], (-4.0 + 0.4 * k, 0.0, -2.0 + 0.3 * k), yaw_deg=33.0 + 9 * k)
    out[I_SPHERE] = scenes.move_instance(sc.instances[I_SPHERE], (1.8 - 0.3 * k, 1.6 + 0.2 * k, 0.5), yaw_deg=40.0 - 14 * k,
                                         scale=1.0 + 0.08 * k, pitch_deg=6 * k)
    prev = sc.instances[I_SHEAR]
    cur = _shear_instance(prev.mesh_slots, (-1.3 + 0.25 * k, 0.6, 2.5 - 0.2 * k))
    to44 = lambda m: np.vstack([np.asarray(m, np.float64), [0, 0, 0, 1]])
    cur.cur_to_prev = (to44(prev.transform) @ np.linalg.inv(to44(cur.transform)))[:3].astype(F32)
    out[I_SHEAR] = cur
    return out


def moved_camera(sc: scenes.Scene, W: int, H: int, k: float = 1.0):
    """frame 1's camera: translated by (0.6, -0.2, -0.9) k and turned toward a target 1.5 k to the right"""
    eye = np.asarray(sc.camera_position, np.float64) + k * np.array([0.6, -0.2, -0.9])
    cam = abi.make_camera(sc, W, H)
    cam.position = (abi.c_f * 3)(*eye.astype(F32))
    cam.orientation = (abi.c_f * 9)(*scenes.look_at_orientation(eye, (1.5 * k, 2.4, 0.0)).reshape(-1))
    return cam
