"""Light sampling restated in float64 from a scenes.Scene alone - TEST INFRASTRUCTURE.

What sampleLight (restir_di_shared.h:320-516) and the environment light (loadEnvironmentalTexture, common_host.cpp:2658-2711;
RegularConstantContinuousDistribution2D, common_shared.h:283-386) compute, written from their definitions instead of from the
library's or the oracle's tables:
  * emitters: triangle t of mesh m in instance i is picked with P_t = s_i^2 lum(E_m) A_obj,t / sum over all triangles of the same,
    and sampled uniformly over its world-space area, so its area density is P_t / A_world,t;
  * the environment: texels clamped to [0, 65504], importance lum x sin(theta of the texel centre), the texel pdf normalised so
    that its integral over [0, 1]^2 is 1, and the solid-angle density pdf / (2 pi^2 sin theta);
  * squareToTriangle and fromPolarYUp (with the rotation wrap of sampleEnvLight).
Emitters are listed in the order of the library's light records (instance, geometry in the instance, triangle), so row k belongs
to the light whose pick key is k.
"""
from __future__ import annotations

import dataclasses

import numpy as np

LUM = np.array([0.2126729, 0.7151522, 0.0721750])  # sRGB_calcLuminance (basic_types.h)


@dataclasses.dataclass
class Emitters:
    prob: np.ndarray          # P_t
    area_obj: np.ndarray      # A_obj,t
    area_world: np.ndarray    # A_world,t (instance transform applied)
    density: np.ndarray       # P_t / A_world,t
    inst: np.ndarray          # instance slot
    geom: np.ndarray          # geometry index in the instance
    prim: np.ndarray          # triangle index in the mesh
    emittance: np.ndarray     # [n, 3]
    world: np.ndarray         # [n, 3, 3] world-space vertices
    normals: np.ndarray       # [n, 3, 3] object-space vertex normals
    normal_matrix: np.ndarray  # [n, 3, 3]
    weight: np.ndarray        # s_i^2 lum(E) A_obj,t (unnormalised)


def emitters(scene) -> Emitters:
    cols = {k: [] for k in ("w", "aobj", "aw", "inst", "geom", "prim", "e", "world", "nrm", "nm")}
    for i, inst in enumerate(scene.instances):
        xf = np.asarray(inst.transform, dtype=np.float64)
        for k, slot in enumerate(inst.mesh_slots):
            mesh = scene.meshes[slot]
            mat = scene.materials[mesh.material]
            if not mat["hasEmittance"]:
                continue
            e = np.asarray(mat["emittance"], dtype=np.float64)
            p = mesh.positions.astype(np.float64)[mesh.triangles.astype(np.int64)]       # [T, 3, 3]
            aobj = 0.5 * np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1)
            wp = p @ xf[:, :3].T + xf[:, 3]
            aw = 0.5 * np.linalg.norm(np.cross(wp[:, 1] - wp[:, 0], wp[:, 2] - wp[:, 0]), axis=1)
            n = mesh.triangles.shape[0]
            cols["w"].append(float(inst.uniform_scale) ** 2 * float(LUM @ e) * aobj)
            cols["aobj"].append(aobj)
            cols["aw"].append(aw)
            cols["inst"].append(np.full(n, i))
            cols["geom"].append(np.full(n, k))
            cols["prim"].append(np.arange(n))
            cols["e"].append(np.broadcast_to(e, (n, 3)))
            cols["world"].append(wp)
            cols["nrm"].append(mesh.normals.astype(np.float64)[mesh.triangles.astype(np.int64)])
            cols["nm"].append(np.broadcast_to(np.asarray(inst.normal_matrix, dtype=np.float64), (n, 3, 3)))
    c = {k: np.concatenate(v) for k, v in cols.items()}
    total = c["w"].sum()
    prob = c["w"] / total if total > 0 else np.zeros_like(c["w"])
    with np.errstate(divide="ignore", invalid="ignore"):
        density = prob / c["aw"]
    return Emitters(prob, c["aobj"], c["aw"], density, c["inst"], c["geom"], c["prim"], c["e"], c["world"], c["nrm"], c["nm"], c["w"])


def square_to_triangle(u0, u1):
    """A Low-Distortion Map Between Triangle and Square (restir_di_shared.h:485-498) -> barycentrics (a, b, c)"""
    a = 0.5 * np.asarray(u0, dtype=np.float64)
    b = 0.5 * np.asarray(u1, dtype=np.float64)
    offset = b - a
    b = np.where(offset > 0, b + offset, b)
    a = np.where(offset > 0, a, a - offset)
    return a, b, 1 - (a + b)


def env_texels(env_map: np.ndarray) -> np.ndarray:
    """the clamp of loadEnvironmentalTexture: rgb in [0, 65504] (+inf -> 65504, negative -> 0)"""
    return np.clip(env_map[..., :3].astype(np.float64), 0.0, 65504.0)


def env_importance(env_map: np.ndarray) -> np.ndarray:
    h = env_map.shape[0]
    sin_centre = np.sin(np.pi * (np.arange(h) + 0.5) / h)
    return (env_texels(env_map) @ LUM) * sin_centre[:, None]


def env_pdf(env_map: np.ndarray) -> np.ndarray:
    """texel pdf over (u, v) in [0, 1]^2: sum(pdf) / (W H) = 1; all 0 for a black map"""
    imp = env_importance(env_map)
    total = imp.mean()
    return imp / total if total > 0 else np.zeros_like(imp)


def env_solid_angle_density(pdf_uv, v):
    """density with respect to solid angle (= the 'area density' at infinity) of a direction with texture coordinate v"""
    return pdf_uv / (2 * np.pi ** 2 * np.sin(np.pi * np.asarray(v, dtype=np.float64)))


def from_polar_y_up(phi, theta):
    phi = np.asarray(phi, dtype=np.float64)
    theta = np.asarray(theta, dtype=np.float64)
    return np.stack([-np.sin(phi) * np.sin(theta), np.cos(theta), np.cos(phi) * np.sin(theta)], axis=-1)


def env_direction(u, v, rotation: float):
    """sampleEnvLight's direction of texture coordinate (u, v): phi = 2 pi u - rotation wrapped into [0, 2 pi)"""
    phi = np.mod(2 * np.pi * np.asarray(u, dtype=np.float64) - rotation, 2 * np.pi)
    return from_polar_y_up(phi, np.pi * np.asarray(v, dtype=np.float64))
