"""Emitter layouts and environment maps that no renderer test scene has - TEST INFRASTRUCTURE for the light-sampling tests.

Emitter scenes (name -> builder): a single emissive triangle; an instance whose last geometry has zero emittance (trailing zero
weights at the geometry level); one mesh of 100 k triangles whose weights spread over 1e-8 .. 1, so that the smallest lie below
ulp(primIntegral) of the float32 scan; meshes of 1, 128, 129 and 1000 triangles around the primitive guide size kPrimGuideSize =
128; instances with uniformScale 0, 0.5 and 3 and one with a non-uniform transform, which the reference weights by uniformScale^2
regardless; and N instances of one triangle each (6 145 is the first count whose k_instanceDist scan needs more than 48 KB of
shared memory, 28 000 the largest count the library accepts).
"""
from __future__ import annotations

import numpy as np

from gfxexp_b200 import scenes

F32 = np.float32
EMITTER, DIFFUSE, DARK_EMITTER = 0, 1, 2


def _materials() -> np.ndarray:
    m = np.zeros(3, dtype=scenes.MATERIAL_DTYPE)
    m["p0"] = 0.5
    m["p1"] = 0.04
    m["p2"] = 0.3
    m["bsdfType"] = scenes.BSDF_DIFFUSE_AND_SPECULAR
    m["emittance"][EMITTER] = (10.0, 8.0, 6.0)
    m["hasEmittance"][EMITTER] = 1
    m["hasEmittance"][DARK_EMITTER] = 1  # an emitter of emittance 0: light records with weight 0
    return m


def tri_mesh(tris: np.ndarray, material: int) -> scenes.Mesh:
    """a mesh of separate triangles [T, 3, 3] with flat vertex normals"""
    tris = np.asarray(tris, dtype=np.float64)
    t = tris.shape[0]
    n = np.cross(tris[:, 1] - tris[:, 0], tris[:, 2] - tris[:, 0])
    n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-300)
    e = tris[:, 1] - tris[:, 0]
    e /= np.maximum(np.linalg.norm(e, axis=1, keepdims=True), 1e-300)
    return scenes.Mesh(tris.reshape(-1, 3).astype(F32), np.repeat(n, 3, axis=0).astype(F32), np.repeat(e, 3, axis=0).astype(F32),
                       np.zeros((3 * t, 2), dtype=F32), np.arange(3 * t, dtype=np.uint32).reshape(t, 3), material)


def _random_tris(rng, t: int, size: float = 1.0) -> np.ndarray:
    centre = rng.uniform(-4, 4, size=(t, 1, 3))
    return centre + size * rng.uniform(-0.5, 0.5, size=(t, 3, 3))


def _scene(meshes, instances, name) -> scenes.Scene:
    return scenes.Scene(meshes, _materials(), instances, np.array([0.0, 2.0, 12.0], dtype=F32),
                        scenes.look_at_orientation((0.0, 2.0, 12.0), (0.0, 0.0, 0.0)).astype(F32), 0.8, name=name)


def single_triangle() -> scenes.Scene:
    mesh = tri_mesh([[[0.0, 0.0, 0.0], [1.5, 0.2, 0.0], [0.3, 0.1, 1.1]]], EMITTER)
    return _scene([mesh], [scenes.make_instance([0], (0.5, 1.0, -0.5), yaw_deg=30.0, scale=2.0, pitch_deg=20.0)], "single_triangle")


def trailing_zero_geometry() -> scenes.Scene:
    rng = np.random.default_rng(1)
    meshes = [tri_mesh(_random_tris(rng, 6), EMITTER), tri_mesh(_random_tris(rng, 4), DIFFUSE),
              tri_mesh(_random_tris(rng, 5), EMITTER), tri_mesh(_random_tris(rng, 3), DARK_EMITTER)]
    return _scene(meshes, [scenes.make_instance([0, 1, 2, 3]), scenes.make_instance([2, 3], (1.0, 0.0, 0.0))], "trailing_zero_geometry")


def spread_weights(t: int = 100_000) -> scenes.Scene:
    rng = np.random.default_rng(2)
    area = 10.0 ** rng.uniform(-8.0, 0.0, size=t)  # weight of each triangle: 1e-8 .. 1 x lum(E)
    side = np.sqrt(2 * area)
    origin = np.stack([rng.uniform(-5, 5, t), np.zeros(t), rng.uniform(-5, 5, t)], axis=1)
    tris = np.stack([origin, origin + side[:, None] * [1.0, 0.0, 0.0], origin + side[:, None] * [0.0, 0.0, 1.0]], axis=1)
    return _scene([tri_mesh(tris, EMITTER)], [scenes.make_instance([0])], "spread_weights")


def guide_sizes() -> scenes.Scene:
    rng = np.random.default_rng(3)
    meshes = [tri_mesh(_random_tris(rng, t), EMITTER) for t in (1, 128, 129, 1000)]
    return _scene(meshes, [scenes.make_instance([k], (3.0 * k, 0.0, 0.0)) for k in range(4)], "guide_sizes")


def scaled_instances() -> scenes.Scene:
    rng = np.random.default_rng(4)
    mesh = tri_mesh(_random_tris(rng, 20), EMITTER)
    insts = [scenes.make_instance([0], (3.0 * k, 0.0, 0.0), scale=s) for k, s in enumerate((1.0, 1.0, 0.5, 3.0))]
    insts[1].transform[:, :3] = 0.0  # scale 0 (its normal matrix, the inverse of nothing, stays the identity's)
    insts[1].uniform_scale = 0.0
    skew = scenes.make_instance([0], (5.0, 0.0, 0.0), yaw_deg=15.0)  # non-uniform: diag(1, 2, 0.5), uniformScale stays 1
    skew.transform[:, :3] = (skew.transform[:, :3].astype(np.float64) @ np.diag([1.0, 2.0, 0.5])).astype(F32)
    skew.normal_matrix = np.linalg.inv(skew.transform[:, :3].astype(np.float64)).T.astype(F32)
    return _scene([mesh], insts + [skew], "scaled_instances")


def many_instances(n: int) -> scenes.Scene:
    rng = np.random.default_rng(5)
    mesh = tri_mesh(_random_tris(rng, 1, 0.3), EMITTER)
    pos = rng.uniform(-50, 50, size=(n, 3))
    scale = rng.uniform(0.5, 2.0, size=n)
    return _scene([mesh], [scenes.make_instance([0], tuple(pos[i]), scale=float(scale[i])) for i in range(n)], f"instances_{n}")


EMITTER_SCENES = {
    "single_triangle": single_triangle,
    "trailing_zero_geometry": trailing_zero_geometry,
    "spread_weights": spread_weights,
    "guide_sizes": guide_sizes,
    "scaled_instances": scaled_instances,
    "degenerate_light": scenes.tiny_city_scene_degenerate_light,
    "instances_6145": lambda: many_instances(6145),
}


# ---- environment maps: float32 [H, W, 4] ------------------------------------------------------------------------------------
def env_map(kind: str) -> np.ndarray:
    """kind: "1x1", "1xH", "Wx1", "37x19", "bright_texel" (1e4 against 1e-3), "black_rows" (the ground of a sky), "black_columns",
    "black_poles" (rows 0 and H - 1), "huge" (texels above 65504, +inf and negative), "black" (everywhere)"""
    sizes = {"1x1": (1, 1), "1xH": (1, 16), "Wx1": (24, 1)}
    w, h = sizes.get(kind, (37, 19))
    img = scenes.procedural_sky(w, h, sun_power=20.0, seed=9) if h > 1 else np.random.default_rng(6).uniform(0.1, 2.0, (h, w, 4)).astype(F32)
    img[..., 3] = 1.0
    if kind == "bright_texel":
        img[..., :3] = 1e-3
        img[5, 11, :3] = 1e4
    elif kind == "black_rows":
        img[h - 5:, :, :3] = 0.0
    elif kind == "black_columns":
        img[:, 3:9, :3] = 0.0
        img[:, w - 2:, :3] = 0.0
    elif kind == "black_poles":
        img[[0, h - 1], :, :3] = 0.0
    elif kind == "huge":
        img[2, 4, 0] = 1e6
        img[7, 7, :3] = np.inf
        img[9, 30, 1] = -5.0
        img[12, 1, :3] = -1.0
    elif kind == "black":
        img[..., :3] = 0.0
    return np.ascontiguousarray(img, dtype=F32)


ENV_KINDS = ["1x1", "1xH", "Wx1", "37x19", "bright_texel", "black_rows", "black_columns", "black_poles", "huge", "black"]


def sky_with_black_ground() -> scenes.Scene:
    """tiny_city_scene under procedural_sky(32, 16) whose rows 12-15 (the ground) are black"""
    scene = scenes.tiny_city_scene()
    scene.env_map = scenes.procedural_sky(32, 16)
    scene.env_map[12:, :, :3] = 0.0
    scene.name = "tiny_city_black_ground"
    return scene
