"""Deterministic synthetic scenes for the hot path (SURVEY.md §8d "Synthetic inputs").

The reference ships no Bistro/Zero-Day assets (restir_di/restir_di_main.cpp:1-26 asks the user
to download them), so configs 2-5 use a procedural "city block" with the same gross statistics
as Bistro exterior: ~2.8 M triangles in ~1 000 instances of ~50 meshes, 100 materials with 1x1
textures, ~20 000 emissive triangles in ~200 light instances.  Everything is generated with
numpy from a fixed seed; the same arrays feed the CUDA library and the CPU oracle.

Conventions mirrored from the reference host code:
  * materials are DiffuseAndSpecular with constant (1x1 texture) parameters; colour texels are
    UNORM8 + sRGB-decoded, scalar texels UNORM8 (common/common_host.cpp:1045-1088,1566-1585);
  * instance transforms are T * R * S(uniform) (common/common_host.cpp:2582-2656), normalMatrix =
    transpose(inverse(upper-left 3x3)) (:2635), curToPrevTransform = identity for static scenes
    (:2634).
"""
from __future__ import annotations

import dataclasses
import math
from typing import List, Optional

import numpy as np

F32 = np.float32


@dataclasses.dataclass
class Mesh:
    positions: np.ndarray  # [V,3] f32
    normals: np.ndarray    # [V,3] f32
    tangents: np.ndarray   # [V,3] f32
    texcoords: np.ndarray  # [V,2] f32
    triangles: np.ndarray  # [T,3] u32
    material: int


@dataclasses.dataclass
class Instance:
    transform: np.ndarray        # [3,4] f32
    cur_to_prev: np.ndarray      # [3,4] f32
    normal_matrix: np.ndarray    # [3,3] f32
    uniform_scale: float
    mesh_slots: List[int]


@dataclasses.dataclass
class Scene:
    meshes: List[Mesh]
    materials: np.ndarray        # structured array, see MATERIAL_DTYPE
    instances: List[Instance]
    camera_position: np.ndarray  # [3]
    camera_orientation: np.ndarray  # [3,3] row-major
    fov_y: float
    name: str = "scene"
    env_map: Optional[np.ndarray] = None  # float32 [H, W, 4] equirectangular environment map (GfxSceneDesc::envTexels) or None
    textures: Optional[List[np.ndarray]] = None       # float32 [H, W, 4] images, linear (after sRGB decode)
    material_textures: Optional[np.ndarray] = None    # uint32 [numMaterials, 4]: texture of p0, p1, p2, emittance or 0xFFFFFFFF
    bump_maps: Optional[np.ndarray] = None            # uint32 [numMaterials, 2]: bump-map texture or 0xFFFFFFFF, GfxBumpMapType

    @property
    def num_triangles(self) -> int:
        return sum(self.meshes[m].triangles.shape[0] for inst in self.instances for m in inst.mesh_slots)

    @property
    def num_emissive_triangles(self) -> int:
        n = 0
        for inst in self.instances:
            for m in inst.mesh_slots:
                if self.materials[self.meshes[m].material]["hasEmittance"]:
                    n += self.meshes[m].triangles.shape[0]
        return n


def procedural_sky(width: int = 64, height: int = 32, sun_power: float = 40.0, seed: int = 7) -> np.ndarray:
    """A small HDR equirectangular map in the layout loadEnvironmentalTexture expects (common/common_host.cpp:2658-2711; row 0 at
    theta = 0, i.e. +y): a horizon-brightened blue gradient, a warm ground, a sun blob of a few texels and a little per-texel
    noise so that no two importance values are equal.  Stands in for the -env-texture .exr the reference loads."""
    rng = np.random.default_rng(seed)
    v = (np.arange(height, dtype=np.float32) + 0.5) / height          # theta / pi
    u = (np.arange(width, dtype=np.float32) + 0.5) / width            # phi / 2 pi
    up = np.cos(np.pi * v)[:, None]                                    # +1 at the zenith
    sky = np.stack([0.25 + 0.35 * (1 - np.abs(up)), 0.45 + 0.35 * (1 - np.abs(up)), 0.9 - 0.2 * (1 - np.abs(up))], axis=-1)
    ground = np.array([0.18, 0.15, 0.12], dtype=np.float32)
    img = np.where(up[..., None] >= 0, sky, ground[None, None, :]).astype(np.float32)
    img = np.broadcast_to(img, (height, width, 3)).copy()
    du = np.minimum(np.abs(u - 0.3), 1 - np.abs(u - 0.3))[None, :]
    dv = (v - 0.28)[:, None]
    sun = sun_power * np.exp(-((du * 2) ** 2 + dv ** 2) / (2 * 0.03 ** 2))
    img += sun[..., None] * np.array([1.0, 0.9, 0.7], dtype=np.float32)
    img *= (1 + 0.05 * rng.random((height, width, 1), dtype=np.float32))
    out = np.ones((height, width, 4), dtype=np.float32)
    out[..., :3] = img
    return out


MATERIAL_DTYPE = np.dtype([
    ("p0", F32, 3), ("p2", F32), ("p1", F32, 3), ("bsdfType", np.uint32),
    ("emittance", F32, 3), ("hasEmittance", np.uint32)])

BSDF_LAMBERT, BSDF_DIFFUSE_AND_SPECULAR, BSDF_SIMPLE_PBR = 0, 1, 2


def srgb_unorm8_to_linear(q: np.ndarray) -> np.ndarray:
    """Texture-unit decode of an sRGB UNORM8 texel (IEC 61966-2-1 EOTF), float32 result."""
    c = q.astype(np.float64) / 255.0
    lin = np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)
    return lin.astype(F32)


# --------------------------------------------------------------------------------------
# mesh primitives
# --------------------------------------------------------------------------------------
def _grid_face(n: int, origin, du, dv, normal, rng: np.random.Generator | None, bump: float):
    """(n+1)^2 vertices spanning origin + s*du + t*dv, s,t in [0,1]; 2 n^2 triangles (CCW about `normal`)."""
    s, t = np.meshgrid(np.linspace(0.0, 1.0, n + 1), np.linspace(0.0, 1.0, n + 1), indexing="xy")
    s = s.reshape(-1, 1)
    t = t.reshape(-1, 1)
    origin = np.asarray(origin, dtype=np.float64)
    du = np.asarray(du, dtype=np.float64)
    dv = np.asarray(dv, dtype=np.float64)
    normal = np.asarray(normal, dtype=np.float64)
    pos = origin + s * du + t * dv
    if rng is not None and bump > 0.0:
        # displace interior vertices along the normal so faces are not exactly planar
        h = rng.uniform(-bump, bump, size=(pos.shape[0], 1))
        interior = ((s > 0) & (s < 1) & (t > 0) & (t < 1)).astype(np.float64)
        pos = pos + h * interior * normal
    nrm = np.broadcast_to(normal, pos.shape).copy()
    tan = np.broadcast_to(du / np.linalg.norm(du), pos.shape).copy()
    uv = np.concatenate([s, t], axis=1)
    idx = np.arange((n + 1) * (n + 1)).reshape(n + 1, n + 1)
    a = idx[:-1, :-1].reshape(-1)
    b = idx[:-1, 1:].reshape(-1)
    c = idx[1:, 1:].reshape(-1)
    d = idx[1:, :-1].reshape(-1)
    tris = np.concatenate([np.stack([a, b, c], 1), np.stack([a, c, d], 1)], 0)
    return pos, nrm, tan, uv, tris


def _merge(parts, material: int) -> Mesh:
    pos, nrm, tan, uv, tris = [], [], [], [], []
    base = 0
    for p, n_, t_, u, tr in parts:
        pos.append(p)
        nrm.append(n_)
        tan.append(t_)
        uv.append(u)
        tris.append(tr + base)
        base += p.shape[0]
    return Mesh(np.ascontiguousarray(np.concatenate(pos), dtype=F32),
                np.ascontiguousarray(np.concatenate(nrm), dtype=F32),
                np.ascontiguousarray(np.concatenate(tan), dtype=F32),
                np.ascontiguousarray(np.concatenate(uv), dtype=F32),
                np.ascontiguousarray(np.concatenate(tris), dtype=np.uint32), material)


def make_box(n: int, size, material: int, rng=None, bump: float = 0.0) -> Mesh:
    """Axis-aligned box centred at the origin in x/z, sitting on y=0; each face n x n quads (12 n^2 triangles)."""
    sx, sy, sz = size
    hx, hz = sx * 0.5, sz * 0.5
    faces = [
        ((-hx, 0, hz), (sx, 0, 0), (0, sy, 0), (0, 0, 1)),     # +z
        ((hx, 0, -hz), (-sx, 0, 0), (0, sy, 0), (0, 0, -1)),   # -z
        ((hx, 0, hz), (0, 0, -sz), (0, sy, 0), (1, 0, 0)),     # +x
        ((-hx, 0, -hz), (0, 0, sz), (0, sy, 0), (-1, 0, 0)),   # -x
        ((-hx, sy, hz), (sx, 0, 0), (0, 0, -sz), (0, 1, 0)),   # +y
        ((-hx, 0, -hz), (sx, 0, 0), (0, 0, sz), (0, -1, 0)),   # -y
    ]
    return _merge([_grid_face(n, o, du, dv, nn, rng, bump) for o, du, dv, nn in faces], material)


def make_plane(n: int, size: float, material: int, rng=None, bump: float = 0.0) -> Mesh:
    h = size * 0.5
    return _merge([_grid_face(n, (-h, 0, h), (size, 0, 0), (0, 0, -size), (0, 1, 0), rng, bump)], material)


def make_quad_light(size: float, material: int) -> Mesh:
    """createRectangleLight (common/common_host.cpp:2431-2476): a quad in the xz-plane facing -y."""
    h = size * 0.5
    return _merge([_grid_face(1, (-h, 0, -h), (size, 0, 0), (0, 0, size), (0, -1, 0), None, 0.0)], material)


def make_sphere(nu: int, nv: int, radius: float, material: int) -> Mesh:
    """UV sphere, 2*nu*(nv-1) triangles."""
    pos, nrm, tan, uv = [], [], [], []
    for j in range(nv + 1):
        theta = math.pi * j / nv
        for i in range(nu + 1):
            phi = 2.0 * math.pi * i / nu
            d = np.array([math.sin(theta) * math.cos(phi), math.cos(theta), math.sin(theta) * math.sin(phi)])
            pos.append(radius * d)
            nrm.append(d)
            tan.append(np.array([-math.sin(phi), 0.0, math.cos(phi)]))
            uv.append((i / nu, j / nv))
    tris = []
    for j in range(nv):
        for i in range(nu):
            a = j * (nu + 1) + i
            b = a + 1
            c = a + nu + 1
            d = c + 1
            if j != 0:
                tris.append((a, b, c))
            if j != nv - 1:
                tris.append((b, d, c))
    return Mesh(np.asarray(pos, dtype=F32), np.asarray(nrm, dtype=F32), np.asarray(tan, dtype=F32),
                np.asarray(uv, dtype=F32), np.asarray(tris, dtype=np.uint32), material)


# --------------------------------------------------------------------------------------
# transforms
# --------------------------------------------------------------------------------------
def rot_y(deg: float) -> np.ndarray:
    a = math.radians(deg)
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=np.float64)


def rot_x(deg: float) -> np.ndarray:
    a = math.radians(deg)
    c, s = math.cos(a), math.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]], dtype=np.float64)


def make_instance(mesh_slots, translate=(0, 0, 0), yaw_deg=0.0, scale=1.0, pitch_deg=0.0) -> Instance:
    r = rot_y(yaw_deg) @ rot_x(pitch_deg)
    m = np.zeros((3, 4), dtype=np.float64)
    m[:, :3] = r * scale
    m[:, 3] = translate
    m32 = m.astype(F32)
    # normalMatrix = transpose(inverse(upper-left)), evaluated in float like the reference host
    upper = m32[:, :3].astype(np.float64)
    nm = np.linalg.inv(upper).T.astype(F32)
    ident = np.zeros((3, 4), dtype=F32)
    ident[0, 0] = ident[1, 1] = ident[2, 2] = 1.0
    return Instance(m32, ident, nm, float(F32(scale)), list(mesh_slots))


def move_instance(prev: Instance, translate=(0, 0, 0), yaw_deg=0.0, scale=1.0, pitch_deg=0.0) -> Instance:
    """The instance one animation step later (InstanceController::update, common/common_host.h:798-856): a new T * R * S
    and curToPrevTransform = prevTransform * inverse(curTransform), which the G-buffer pass uses for motion vectors."""
    cur = make_instance(prev.mesh_slots, translate, yaw_deg, scale, pitch_deg)

    def to44(m34):
        m = np.eye(4, dtype=np.float64)
        m[:3, :] = np.asarray(m34, dtype=np.float64)
        return m
    cur_to_prev = (to44(prev.transform) @ np.linalg.inv(to44(cur.transform)))[:3, :].astype(F32)
    return Instance(cur.transform, cur_to_prev, cur.normal_matrix, cur.uniform_scale, list(prev.mesh_slots))


def _random_materials(rng: np.random.Generator, count: int) -> np.ndarray:
    mats = np.zeros(count, dtype=MATERIAL_DTYPE)
    q_diffuse = rng.integers(30, 230, size=(count, 3), dtype=np.int64)
    q_spec = rng.integers(5, 60, size=(count, 1), dtype=np.int64).repeat(3, axis=1)
    q_smooth = rng.integers(20, 200, size=count, dtype=np.int64)
    mats["p0"] = srgb_unorm8_to_linear(q_diffuse)
    mats["p1"] = srgb_unorm8_to_linear(q_spec)
    mats["p2"] = (q_smooth.astype(np.float64) / 255.0).astype(F32)
    mats["bsdfType"] = BSDF_DIFFUSE_AND_SPECULAR
    return mats


def look_at_orientation(eye, target) -> np.ndarray:
    """Row-major 3x3 whose columns are (right, up, forward); rays are orientation * (vw(.5-x), vh(.5-y), 1)
    (optix_gbuffer_kernels.cu:21-27)."""
    eye = np.asarray(eye, dtype=np.float64)
    fwd = np.asarray(target, dtype=np.float64) - eye
    fwd /= np.linalg.norm(fwd)
    up = np.array([0.0, 1.0, 0.0])
    right = np.cross(up, fwd)
    right /= np.linalg.norm(right)
    up2 = np.cross(fwd, right)
    return np.stack([right, up2, fwd], axis=1).astype(F32)


# --------------------------------------------------------------------------------------
# scenes
# --------------------------------------------------------------------------------------
def city_scene(num_buildings: int = 700, building_tess=(12, 20), ground_tess: int = 256, num_lamps: int = 200,
               num_props: int = 100, lamp_tess=(8, 6), num_building_meshes: int = 30, num_materials: int = 100,
               seed: int = 0xB157, name: str = "city") -> Scene:
    """Procedural city block ("Bistro-exterior-class", SURVEY.md §8d config 2)."""
    rng = np.random.default_rng(seed)
    materials = _random_materials(rng, num_materials)
    # the last 8 materials are emitters: warm/cool street lights and coloured signs
    num_emitters = 8
    for k in range(num_emitters):
        m = materials[num_materials - 1 - k]
        m["hasEmittance"] = 1
        tint = np.array([[1.0, 0.85, 0.6], [0.7, 0.85, 1.0], [1.0, 0.3, 0.2], [0.2, 1.0, 0.4],
                         [0.3, 0.4, 1.0], [1.0, 1.0, 1.0], [1.0, 0.6, 0.1], [0.8, 0.2, 1.0]][k], dtype=F32)
        m["emittance"] = tint * F32(40.0 + 10.0 * k)
        m["p0"] = F32(0.8)   # lamp glass: bright diffuse body so demodulated lighting stays finite (SVGF)
        m["p1"] = F32(0.04)
        m["p2"] = F32(0.3)
    meshes: List[Mesh] = []
    instances: List[Instance] = []

    extent = 24.0 * math.sqrt(max(num_buildings, 1) / 64.0)  # half-size of the block
    # ground
    meshes.append(make_plane(ground_tess, 2.2 * extent, int(rng.integers(0, num_materials - num_emitters)), rng, 0.01))
    instances.append(make_instance([0]))

    # building meshes: unit-ish boxes with bumpy facades
    building_slots = []
    for _ in range(num_building_meshes):
        n = int(rng.integers(building_tess[0], building_tess[1] + 1))
        size = (float(rng.uniform(3.0, 6.0)), float(rng.uniform(4.0, 14.0)), float(rng.uniform(3.0, 6.0)))
        mat = int(rng.integers(0, num_materials - num_emitters))
        building_slots.append(len(meshes))
        meshes.append(make_box(n, size, mat, rng, 0.03))
    # street grid: buildings on a jittered lattice, leaving an avenue along z through x = 0
    side = int(math.ceil(math.sqrt(num_buildings)))
    pitch = 2.0 * extent / side
    placed = 0
    for iz in range(side):
        for ix in range(side):
            if placed >= num_buildings:
                break
            cx = -extent + (ix + 0.5) * pitch + float(rng.uniform(-0.15, 0.15)) * pitch
            cz = -extent + (iz + 0.5) * pitch + float(rng.uniform(-0.15, 0.15)) * pitch
            if abs(cx) < 3.5:  # the avenue
                cx = math.copysign(3.5 + abs(cx), cx if cx != 0 else 1.0)
            slot = building_slots[int(rng.integers(0, len(building_slots)))]
            instances.append(make_instance([slot], (cx, 0.0, cz), float(rng.uniform(0.0, 360.0)),
                                           float(rng.uniform(0.7, 1.3))))
            placed += 1

    # lamps: pole (box) + emissive head (sphere) share one instance -> 2 mesh slots per instance
    lamp_variants = []
    for k in range(4):
        pole = len(meshes)
        meshes.append(make_box(1, (0.12, 3.0, 0.12), int(rng.integers(0, num_materials - num_emitters))))
        head = len(meshes)
        hm = make_sphere(lamp_tess[0], lamp_tess[1], 0.22, num_materials - 1 - (k % 2))
        hm.positions[:, 1] += F32(3.15)
        meshes.append(hm)
        lamp_variants.append([pole, head])
    for k in range(num_lamps):
        side_sign = -1.0 if (k % 2) else 1.0
        z = -extent + 2.0 * extent * (k + 0.5) / max(num_lamps, 1)
        x = side_sign * (2.6 + float(rng.uniform(0.0, 0.4)))
        if k % 5 == 4:  # every fifth lamp sits in a side street
            x = float(rng.uniform(-extent, extent))
        instances.append(make_instance(lamp_variants[k % 4], (x, 0.0, z), float(rng.uniform(0, 360)), 1.0))

    # emissive signs: small quads hung over the avenue, coloured emitters
    sign_slots = []
    for k in range(6):
        sign_slots.append(len(meshes))
        meshes.append(make_quad_light(0.8, num_materials - 3 - k))
    for k in range(max(num_lamps // 8, 1)):
        z = -extent + 2.0 * extent * (k + 0.5) / max(num_lamps // 8, 1)
        instances.append(make_instance([sign_slots[k % 6]], (float(rng.uniform(-2.0, 2.0)), 4.5, z),
                                       float(rng.uniform(0, 360)), float(rng.uniform(0.8, 1.5))))

    # props: spheres and crates on the pavement
    prop_slots = []
    for k in range(6):
        prop_slots.append(len(meshes))
        if k % 2 == 0:
            meshes.append(make_sphere(32, 16, 0.5, int(rng.integers(0, num_materials - num_emitters))))
        else:
            meshes.append(make_box(6, (0.9, 0.9, 0.9), int(rng.integers(0, num_materials - num_emitters)), rng, 0.02))
    for k in range(num_props):
        x = float(rng.uniform(-3.2, 3.2))
        z = float(rng.uniform(-extent, extent))
        slot = prop_slots[int(rng.integers(0, 6))]
        y = 0.5 if slot in prop_slots[0::2] else 0.0
        instances.append(make_instance([slot], (x, y, z), float(rng.uniform(0, 360)), float(rng.uniform(0.5, 1.2))))

    eye = np.array([0.4, 1.7, -extent * 0.85])
    target = np.array([0.0, 2.2, 0.0])
    return Scene(meshes, materials, instances, eye.astype(F32), look_at_orientation(eye, target),
                 math.radians(50.0), name)


def interior_scene(hall=(60.0, 9.0, 40.0), wall_tess: int = 200, num_columns: int = 80, column_tess: int = 30,
                   num_props: int = 300, prop_tess: int = 24, num_emitters: int = 5000, num_materials: int = 64,
                   seed: int = 0x2D47, name: str = "interior") -> Scene:
    """Procedural interior ("Zero-Day-class", SURVEY.md 8d config 3): a closed hall (floor, ceiling, four walls, all facing
    inwards) with rows of columns, props on the floor and MANY SMALL EMITTERS - panel lights of two triangles each hung
    under the ceiling and on the walls - lit with SimplePBR materials (baseColor / smoothness / metallic,
    common/common_device.cuh:767-776, 806-826), which the city scenes do not use."""
    rng = np.random.default_rng(seed)
    mats = np.zeros(num_materials, dtype=MATERIAL_DTYPE)
    q_base = rng.integers(40, 235, size=(num_materials, 3), dtype=np.int64)
    mats["p0"] = srgb_unorm8_to_linear(q_base)
    mats["p1"][:, 1] = (rng.integers(40, 230, size=num_materials) / 255.0).astype(F32)   # 1 - smoothness
    mats["p1"][:, 2] = np.where(rng.random(num_materials) < 0.25, 1.0, 0.0).astype(F32) * \
        (rng.integers(128, 256, size=num_materials) / 255.0).astype(F32)                  # metallic
    mats["bsdfType"] = BSDF_SIMPLE_PBR
    num_emitter_mats = 6
    tints = np.array([[1.0, 0.9, 0.75], [0.75, 0.85, 1.0], [1.0, 0.45, 0.3], [0.4, 1.0, 0.6], [0.5, 0.55, 1.0], [1.0, 1.0, 1.0]], dtype=F32)
    for k in range(num_emitter_mats):
        m = mats[num_materials - 1 - k]
        m["hasEmittance"] = 1
        m["emittance"] = tints[k] * F32(25.0 + 5.0 * k)
        m["p0"] = F32(0.8)
        m["p1"] = (0.0, 0.6, 0.0)
    body = num_materials - num_emitter_mats
    meshes: List[Mesh] = []
    instances: List[Instance] = []
    hx, hy, hz = hall[0] * 0.5, hall[1], hall[2] * 0.5
    # the shell, facing inwards
    shell = [((-hx, 0, hz), (hall[0], 0, 0), (0, 0, -hall[2]), (0, 1, 0)),        # floor
             ((-hx, hy, -hz), (hall[0], 0, 0), (0, 0, hall[2]), (0, -1, 0)),      # ceiling
             ((-hx, 0, -hz), (hall[0], 0, 0), (0, hy, 0), (0, 0, 1)),             # back wall (z = -hz), facing +z
             ((hx, 0, hz), (-hall[0], 0, 0), (0, hy, 0), (0, 0, -1)),             # front wall
             ((-hx, 0, hz), (0, 0, -hall[2]), (0, hy, 0), (1, 0, 0)),             # left wall, facing +x
             ((hx, 0, -hz), (0, 0, hall[2]), (0, hy, 0), (-1, 0, 0))]             # right wall
    for k, (o, du, dv, nn) in enumerate(shell):
        meshes.append(_merge([_grid_face(wall_tess, o, du, dv, nn, rng, 0.004)], int(rng.integers(0, body))))
        instances.append(make_instance([len(meshes) - 1]))
    # columns in two rows along x
    column_slots = []
    for _ in range(4):
        column_slots.append(len(meshes))
        meshes.append(make_box(column_tess, (0.9, hy, 0.9), int(rng.integers(0, body)), rng, 0.01))
    for k in range(num_columns):
        row = -1.0 if (k % 2) else 1.0
        x = -hx + hall[0] * (k // 2 + 0.5) / max(num_columns // 2, 1)
        instances.append(make_instance([column_slots[k % 4]], (x, 0.0, row * hz * 0.45), float(rng.uniform(0, 90)), 1.0))
    # props on the floor
    prop_slots = []
    for k in range(8):
        prop_slots.append(len(meshes))
        if k % 2 == 0:
            meshes.append(make_sphere(2 * prop_tess, prop_tess, 0.5, int(rng.integers(0, body))))
        else:
            meshes.append(make_box(prop_tess // 2, (1.0, 1.0, 1.0), int(rng.integers(0, body)), rng, 0.02))
    for k in range(num_props):
        slot = prop_slots[int(rng.integers(0, 8))]
        y = 0.5 if slot in prop_slots[0::2] else 0.0
        instances.append(make_instance([slot], (float(rng.uniform(-hx * 0.9, hx * 0.9)), y, float(rng.uniform(-hz * 0.9, hz * 0.9))),
                                       float(rng.uniform(0, 360)), float(rng.uniform(0.5, 1.6))))
    # many tiny emitters: 2-triangle panels under the ceiling (facing down) and a few per wall
    panel_slots = []
    for k in range(num_emitter_mats):
        panel_slots.append(len(meshes))
        meshes.append(make_quad_light(0.12, num_materials - 1 - k))
    for k in range(num_emitters):
        slot = panel_slots[int(rng.integers(0, num_emitter_mats))]
        x, z = float(rng.uniform(-hx * 0.95, hx * 0.95)), float(rng.uniform(-hz * 0.95, hz * 0.95))
        if k % 9 == 8:   # on a column-height ledge, tilted
            instances.append(make_instance([slot], (x, float(rng.uniform(2.0, hy - 1.0)), z), float(rng.uniform(0, 360)),
                                           float(rng.uniform(0.8, 2.0)), pitch_deg=float(rng.uniform(20, 70))))
        else:
            instances.append(make_instance([slot], (x, hy - 0.05, z), float(rng.uniform(0, 360)), float(rng.uniform(0.8, 2.0))))
    eye = np.array([-hx * 0.8, 1.7, hz * 0.1])
    target = np.array([hx * 0.6, 2.5, -hz * 0.2])
    return Scene(meshes, mats, instances, eye.astype(F32), look_at_orientation(eye, target), math.radians(50.0), name)


def zero_day_class_scene() -> Scene:
    """Config 3 scene: ~5 M triangles, ~5 400 instances, 10 000 small emissive triangles, SimplePBR materials."""
    return interior_scene(wall_tess=360, num_columns=80, column_tess=36, num_props=300, prop_tess=40, num_emitters=5000,
                          name="zero_day_class")


def small_interior_scene() -> Scene:
    """~30 k triangles with 96 two-triangle emitters and SimplePBR materials: oracle-speed parity of config 3's ingredients."""
    return interior_scene(hall=(16.0, 5.0, 12.0), wall_tess=24, num_columns=8, column_tess=6, num_props=16, prop_tess=8,
                          num_emitters=96, num_materials=24, name="small_interior")


def bistro_class_scene() -> Scene:
    """Config 2/4/5 scene: ~2.8 M triangles, ~1 000 instances, ~50 meshes, ~20 k emissive triangles."""
    return city_scene(num_buildings=760, building_tess=(14, 20), ground_tess=300, num_lamps=200, num_props=120,
                      lamp_tess=(10, 6), num_building_meshes=30, name="bistro_class")


def small_city_scene() -> Scene:
    """~60 k triangles: full-resolution GPU-vs-oracle parity in seconds."""
    return city_scene(num_buildings=36, building_tess=(5, 8), ground_tess=32, num_lamps=24, num_props=12,
                      lamp_tess=(8, 6), num_building_meshes=8, name="small_city")


def small_city_scene_env() -> Scene:
    """small_city_scene under an environment light (procedural_sky): emitters and the environment are both sampled."""
    scene = small_city_scene()
    scene.env_map = procedural_sky(64, 32)
    scene.name = "small_city_env"
    return scene


def checker_texture(width: int = 32, height: int = 16, cells: int = 4, lo=(0.08, 0.1, 0.3), hi=(0.8, 0.7, 0.5), seed: int = 3) -> np.ndarray:
    """float32 [H, W, 4] (linear, as GfxTextureDesc wants it): a checker with per-texel noise, no two texels alike"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:height, 0:width]
    mask = (((x * cells) // width + (y * cells) // height) % 2).astype(bool)
    img = np.where(mask[..., None], np.asarray(hi, dtype=F32), np.asarray(lo, dtype=F32)).astype(F32)
    img = img * (F32(0.85) + F32(0.15) * rng.random((height, width, 1), dtype=F32))
    out = np.ones((height, width, 4), dtype=F32)
    out[..., :3] = img
    return out


def small_city_scene_textured() -> Scene:
    """small_city_scene with image textures on most materials: albedo / diffuse / baseColor maps (p0), specular or
    occlusion-roughness-metallic maps (p1) and smoothness maps (p2), non-power-of-two sizes included; texture coordinates run
    beyond [0, 1) on the tessellated faces, so the repeat addressing is exercised.  Emitters keep constant emittance."""
    scene = small_city_scene()
    rng = np.random.default_rng(17)
    scene.textures = [checker_texture(32, 16, 4), checker_texture(24, 40, 6, (0.02, 0.02, 0.02), (0.3, 0.25, 0.2), 5),
                      checker_texture(7, 5, 3, (0.1, 0.1, 0.1), (0.6, 0.6, 0.6), 9), checker_texture(64, 64, 8, (0.2, 0.5, 0.2), (0.9, 0.9, 0.8), 11)]
    n = scene.materials.shape[0]
    mt = np.full((n, 4), 0xFFFFFFFF, dtype=np.uint32)
    for m in range(n):
        if scene.materials[m]["hasEmittance"]:
            continue
        pick = rng.integers(0, 5)
        if pick >= 1:
            mt[m, 0] = [0, 3, 0, 3][pick - 1]
        if pick >= 3 and scene.materials[m]["bsdfType"] != BSDF_LAMBERT:
            mt[m, 1] = 1
            mt[m, 2] = 2
    scene.material_textures = mt
    for mesh in scene.meshes:  # [0, 1] per face in the generator: stretch past the unit square, negative values included
        mesh.texcoords = (mesh.texcoords * F32(3.7) - F32(1.2)).astype(F32)
    scene.name = "small_city_textured"
    return scene


def unorm8(x: np.ndarray) -> np.ndarray:
    """float32 texels as the texture unit reads a UNORM8 texture: round(255 x) / 255 (no sRGB decode)"""
    return (np.round(np.clip(x, 0.0, 1.0) * 255.0).astype(F32) / F32(255.0)).astype(F32)


def sine_normal_map(width: int, height: int, freq=(3, 2), amplitude: float = 0.6, seed: int = 21) -> np.ndarray:
    """float32 [H, W, 4] normal map of the height field a sin(2 pi fx x / W) cos(2 pi fy y / H), stored as the reference reads
    it: rgb = (n + 1) / 2 with y in the DirectX convention (readModifiedNormal flips it back), quantised to UNORM8.  One texel in
    eight is shortened (x 0.6 .. 0.9) before quantisation, so that some decoded normals are far from unit length."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:height, 0:width].astype(np.float64)
    px, py = 2 * np.pi * freq[0] / width, 2 * np.pi * freq[1] / height
    dhdx = amplitude * px * width / 8 * np.cos(px * x) * np.cos(py * y)
    dhdy = -amplitude * py * height / 8 * np.sin(px * x) * np.sin(py * y)
    n = np.stack([-dhdx, -dhdy, np.ones_like(x)], axis=-1)
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    n *= np.where(rng.random((height, width, 1)) < 0.125, rng.uniform(0.6, 0.9, (height, width, 1)), 1.0)
    n[..., 1] = -n[..., 1]
    out = np.ones((height, width, 4), dtype=F32)
    out[..., :3] = unorm8((n + 1.0) * 0.5)
    return out


def noise_height_map(width: int, height: int, seed: int = 23) -> np.ndarray:
    """float32 [H, W, 4] of a one-channel height map as stbi_load(..., 4) expands a grey PNG: (g, g, g, 1), g a smooth bump
    pattern plus noise, quantised to UNORM8"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:height, 0:width].astype(np.float64)
    g = 0.5 + 0.3 * np.sin(2 * np.pi * 2 * x / width) * np.sin(2 * np.pi * 3 * y / height) + 0.15 * rng.random((height, width))
    out = np.ones((height, width, 4), dtype=F32)
    out[..., :3] = unorm8(g)[..., None]
    return out


def small_city_scene_bumped() -> Scene:
    """small_city_scene_textured with bump maps (GfxSceneDesc::bumpMaps): a sinusoidal normal map with some texels of non-unit
    length, a small non-square normal map, and one-channel height maps of non-power-of-two sizes, seeded.  Emitters and about a
    quarter of the other materials have no map (the reference's default 1x1 texel)."""
    scene = small_city_scene_textured()
    base = len(scene.textures)
    scene.textures = scene.textures + [sine_normal_map(48, 32), sine_normal_map(5, 3, (1, 1), 0.9, 29),
                                       noise_height_map(37, 23), noise_height_map(6, 10, 31)]
    maps = [(base, 0), (base + 1, 0), (base + 2, 1), (base + 3, 1)]  # (texture, GfxBumpMapType)
    rng = np.random.default_rng(19)
    n = scene.materials.shape[0]
    bm = np.zeros((n, 2), dtype=np.uint32)
    bm[:, 0] = 0xFFFFFFFF
    for m in range(n):
        pick = int(rng.integers(0, 5))
        if scene.materials[m]["hasEmittance"] or pick == 4:
            continue
        bm[m] = maps[pick]
    scene.bump_maps = bm
    scene.name = "small_city_bumped"
    return scene


def env_only_scene() -> Scene:
    """tiny_city_scene with every emitter switched off, lit by the environment alone: lightInstDist.integral() == 0, so every
    light sample is an environment sample (optix_restir_di_kernels.cu:87-89)."""
    scene = tiny_city_scene()
    scene.materials["hasEmittance"] = 0
    scene.materials["emittance"] = 0
    scene.env_map = procedural_sky(48, 24, sun_power=25.0, seed=11)
    scene.name = "env_only"
    return scene


def tiny_city_scene() -> Scene:
    """~4 k triangles: brute-force-checkable on the CPU."""
    return city_scene(num_buildings=9, building_tess=(2, 3), ground_tess=8, num_lamps=6, num_props=4,
                      lamp_tess=(6, 4), num_building_meshes=4, name="tiny_city")


def tiny_city_scene_degenerate_light() -> Scene:
    """tiny_city_scene plus a 0.5 x 0.5 quad light 10^7 units away: its object-space area gives it a few percent of the light
    selection probability (whole buckets of the pick guide), but in world space its corners round to one line (the float
    spacing there is 1), so its area density is infinite and its bounding sphere must never cull."""
    scene = tiny_city_scene()
    emitter = int(np.flatnonzero(scene.materials["hasEmittance"])[0])
    scene.meshes.append(make_quad_light(0.5, emitter))
    scene.instances.append(make_instance([len(scene.meshes) - 1], (1.0e7, 4.5, 0.0)))
    scene.name = "tiny_city_degenerate_light"
    return scene


def load_obj(path: str):
    """Minimal OBJ reader (v / f only, fan triangulation) for data/teapot.obj-style files, plain or gzip-compressed (.gz)."""
    import gzip
    verts, faces = [], []
    with (gzip.open(path, "rt") if path.endswith(".gz") else open(path, "r")) as fh:
        for line in fh:
            if line.startswith("v "):
                verts.append([float(v) for v in line.split()[1:4]])
            elif line.startswith("f "):
                idx = [int(tok.split("/")[0]) for tok in line.split()[1:]]
                idx = [i - 1 if i > 0 else len(verts) + i for i in idx]
                for k in range(1, len(idx) - 1):
                    faces.append((idx[0], idx[k], idx[k + 1]))
    return np.asarray(verts, dtype=F32), np.asarray(faces, dtype=np.uint32)


def mesh_from_triangles(verts: np.ndarray, faces: np.ndarray, material: int) -> Mesh:
    """Area-weighted vertex normals (assimp GenNormals-like) and makeCoordinateSystem-style tangents."""
    v = verts.astype(np.float64)
    fn = np.cross(v[faces[:, 1]] - v[faces[:, 0]], v[faces[:, 2]] - v[faces[:, 0]])
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, faces[:, k], fn)
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    n = np.where(ln > 0, n / np.maximum(ln, 1e-30), np.array([0.0, 1.0, 0.0]))
    sign = np.where(n[:, 2] >= 0, 1.0, -1.0)
    a = -1.0 / (sign + n[:, 2])
    b = n[:, 0] * n[:, 1] * a
    t = np.stack([1 + sign * n[:, 0] * n[:, 0] * a, sign * b, -sign * n[:, 0]], axis=1)
    uv = np.zeros((v.shape[0], 2))
    return Mesh(np.ascontiguousarray(v, dtype=F32), np.ascontiguousarray(n, dtype=F32),
                np.ascontiguousarray(t, dtype=F32), np.ascontiguousarray(uv, dtype=F32),
                np.ascontiguousarray(faces, dtype=np.uint32), material)


def teapot_like_scene(obj_path: str | None = None) -> Scene:
    """Config 1 (path_tracing on data/teapot.obj + one rectangle light).  Without an OBJ path a sphere of
    similar size stands in."""
    mats = np.zeros(2, dtype=MATERIAL_DTYPE)
    mats[0]["p0"] = F32(1.0)                       # Kd 1
    mats[0]["p1"] = F32(0.2)                       # Ks .2
    mats[0]["p2"] = F32(math.sqrt(10.0) / 11.0)    # smoothness = sqrt(Ns)/11 (common_host.cpp:2271-2274)
    mats[0]["bsdfType"] = BSDF_DIFFUSE_AND_SPECULAR
    mats[1]["bsdfType"] = BSDF_DIFFUSE_AND_SPECULAR
    mats[1]["hasEmittance"] = 1
    mats[1]["emittance"] = F32(50.0)
    mats[1]["p2"] = F32(0.3)
    if obj_path is not None:
        verts, faces = load_obj(obj_path)
        body = mesh_from_triangles(verts, faces, 0)
    else:
        body = make_sphere(96, 48, 60.0, 0)
        body.positions[:, 1] += F32(60.0)
    light = make_quad_light(100.0, 1)
    meshes = [body, light]
    instances = [make_instance([0]), make_instance([1], (0.0, 200.0, 0.0))]
    # camera: translate(0,133.3,200) * rotY(180) * rotX(25)  (nrtdsm/nrtdsm_sandbox.cpp:3137-3146)
    ori = (rot_y(180.0) @ rot_x(25.0)).astype(F32)
    return Scene(meshes, mats, instances, np.array([0.0, 133.3, 200.0], dtype=F32), ori, math.radians(50.0), "teapot")


def save_scene_bin(scene: Scene, path: str, width: int = 64, height: int = 64) -> None:
    """Flat binary scene file for the headless C++ host (host/gfx_headless.cpp): 'GFXS', counts, per-mesh arrays, the
    material / instance tables in the layouts of include/gfxb200.h, and the default GfxFrameParams of this scene."""
    import ctypes as C

    from . import abi
    sa = abi.SceneArrays(scene)
    params = abi.default_frame_params(scene, width, height)
    with open(path, "wb") as f:
        f.write(b"GFXS")
        f.write(np.asarray([len(scene.meshes), scene.materials.shape[0], len(scene.instances), sa.slots.shape[0],
                            C.sizeof(abi.GfxFrameParams)], dtype=np.uint32).tobytes())
        for m in scene.meshes:
            f.write(np.asarray([m.positions.shape[0], m.triangles.shape[0], m.material], dtype=np.uint32).tobytes())
            for a, dt in ((m.positions, np.float32), (m.normals, np.float32), (m.tangents, np.float32), (m.texcoords, np.float32),
                          (m.triangles, np.uint32)):
                f.write(np.ascontiguousarray(a, dtype=dt).tobytes())
        f.write(np.ascontiguousarray(scene.materials).tobytes())
        f.write(bytes(sa.instances))
        f.write(sa.slots.tobytes())
        f.write(bytes(params))
