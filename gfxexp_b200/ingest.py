"""Scene ingestion: Wavefront OBJ + MTL + PNG textures -> scenes.Scene, following what the reference asks of assimp
(createTriangleMeshes, common/common_host.cpp:2178-2429):

  aiProcess_Triangulate          faces are fan-triangulated
  aiProcess_JoinIdenticalVertices one vertex per distinct (position, texcoord, normal) triple of a material group
  aiProcess_GenNormals           per-face normals when the file has no `vn` (the face's vertices are then not shared)
  aiProcess_CalcTangentSpace     tangent = d(position)/du from the triangle's texcoords, accumulated per vertex; without usable
                                 texcoords the reference falls back to makeCoordinateSystem(normal) (:2347-2358)
  aiProcess_FlipUVs              v -> 1 - v
  one aiMesh per material        -> one scenes.Mesh per `usemtl` group

Materials (MaterialConvention::Traditional, :2219-2318): DiffuseAndSpecular with Kd / map_Kd, Ks / map_Ks, smoothness =
sqrt(Ns) / 11 (:2271-2274), emittance = Ke (map_Ke is refused: textured emitters are not supported by the light sampler).
Bump maps (:2280-2284, loadNormalTexture :1344-1356): `map_Bump` / `bump` (assimp's HEIGHT slot) before `norm` (NORMALS), UNORM
texels without sRGB decode; a PNG with more than one channel is a normal map, a one-channel PNG (and spnza_bricks_a_bump.png) a
height map -> Scene.bump_maps.
Image textures are decoded the way the reference's samplers present them to the filter (sampler_sRGB: UNORM8 -> sRGB -> linear
float, common_host.cpp:1462-1467) and handed over as fp32 RGBA (include/gfxb200.h GfxTextureDesc); PNG (8-bit, non-interlaced) is
read here with zlib - the reference reads its images through stb_image / DDS loaders, which are file-format code outside the path.
"""
from __future__ import annotations

import math
import os
import struct
import zlib
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import scenes

F32 = np.float32
NO_TEXTURE = 0xFFFFFFFF
BUMP_NORMAL_MAP, BUMP_HEIGHT_MAP = 0, 1  # GfxBumpMapType


# ---- PNG ---------------------------------------------------------------------------------------------------------------
def decode_png(data: bytes) -> np.ndarray:
    """8-bit non-interlaced PNG (grey, grey+alpha, RGB, RGBA, palette) -> uint8 [H, W, C]"""
    if data[:8] != b"\x89PNG\r\n\x1a\n":
        raise ValueError("not a PNG file")
    pos, idat, palette, trns = 8, [], None, None
    width = height = depth = ctype = interlace = None
    while pos < len(data):
        length, kind = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + length]
        pos += 12 + length
        if kind == b"IHDR":
            width, height, depth, ctype, _, _, interlace = struct.unpack(">IIBBBBB", body)
        elif kind == b"PLTE":
            palette = np.frombuffer(body, dtype=np.uint8).reshape(-1, 3)
        elif kind == b"tRNS":
            trns = np.frombuffer(body, dtype=np.uint8)
        elif kind == b"IDAT":
            idat.append(body)
        elif kind == b"IEND":
            break
    if depth != 8 or interlace != 0:
        raise ValueError("only 8-bit non-interlaced PNGs are supported")
    channels = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
    raw = zlib.decompress(b"".join(idat))
    stride = width * channels
    out = np.zeros((height, stride), dtype=np.uint8)
    prev = np.zeros(stride, dtype=np.int32)
    p = 0
    for y in range(height):
        f = raw[p]
        line = np.frombuffer(raw, dtype=np.uint8, count=stride, offset=p + 1).astype(np.int32)
        p += 1 + stride
        if f == 0:
            cur = line
        elif f == 2:
            cur = (line + prev) & 255
        else:  # 1 Sub, 3 Average, 4 Paeth: each byte depends on the byte `channels` to its left
            cur = np.zeros(stride, dtype=np.int32)
            for i in range(stride):
                a = cur[i - channels] if i >= channels else 0
                b = prev[i]
                c = prev[i - channels] if i >= channels else 0
                if f == 1:
                    pred = a
                elif f == 3:
                    pred = (a + b) >> 1
                else:
                    pa, pb, pc = abs(b - c), abs(a - c), abs(a + b - 2 * c)
                    pred = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
                cur[i] = (line[i] + pred) & 255
        out[y] = cur
        prev = cur
    img = out.reshape(height, width, channels)
    if ctype == 3:
        rgb = palette[img[..., 0]]
        if trns is not None:
            alpha = np.full(256, 255, dtype=np.uint8)
            alpha[:len(trns)] = trns
            return np.concatenate([rgb, alpha[img[..., 0]][..., None]], axis=-1)
        return rgb
    return img


def encode_png(img: np.ndarray) -> bytes:
    """uint8 [H, W, 3 or 4] -> PNG bytes (filter 0; for tests and tools)"""
    h, w, c = img.shape
    raw = b"".join(b"\x00" + np.ascontiguousarray(img[y]).tobytes() for y in range(h))

    def chunk(kind, body):
        return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body) & 0xFFFFFFFF)
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, {3: 2, 4: 6}[c], 0, 0, 0)) +
            chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def srgb_to_linear(u8: np.ndarray) -> np.ndarray:
    """the texture unit's sRGB read mode: UNORM8 -> [0, 1] -> linear (IEC 61966-2-1), fp32"""
    c = u8.astype(np.float64) / 255.0
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4).astype(F32)


def image_to_texture(u8: np.ndarray, srgb: bool = True) -> np.ndarray:
    """uint8 [H, W, C] -> float32 [H, W, 4] as the filter sees it: colour channels sRGB-decoded (or UNORM), alpha UNORM, 1 if absent"""
    if u8.ndim == 2:
        u8 = u8[..., None]
    h, w, c = u8.shape
    out = np.ones((h, w, 4), dtype=F32)
    colour = u8[..., :3] if c >= 3 else np.repeat(u8[..., :1], 3, axis=-1)
    out[..., :3] = srgb_to_linear(colour) if srgb else colour.astype(F32) / F32(255.0)
    if c in (2, 4):
        out[..., 3] = u8[..., -1].astype(F32) / F32(255.0)
    return out


# ---- MTL ---------------------------------------------------------------------------------------------------------------
def parse_mtl(path: str) -> Dict[str, dict]:
    mats: Dict[str, dict] = {}
    cur = None
    with open(path, "r") as fh:
        for line in fh:
            tok = line.split("#", 1)[0].split()
            if not tok:
                continue
            key = tok[0]
            if key == "newmtl":
                cur = mats.setdefault(" ".join(tok[1:]), {})
            elif cur is None:
                continue
            elif key in ("Kd", "Ks", "Ke"):
                cur[key] = [float(v) for v in tok[1:4]]
            elif key == "Ns":
                cur["Ns"] = float(tok[1])
            elif key in ("map_Kd", "map_Ks", "map_Ke"):
                cur[key] = tok[-1]  # options (-s, -o ...) are not interpreted
            elif key in ("map_Bump", "map_bump", "bump"):  # assimp's HEIGHT slot
                cur["bump"] = tok[-1]  # options (-bm ...) are not interpreted either
            elif key == "norm":  # assimp's NORMALS slot
                cur["norm"] = tok[-1]
    return mats


# ---- OBJ ---------------------------------------------------------------------------------------------------------------
def _index(tok: str, n: int) -> int:
    i = int(tok)
    return i - 1 if i > 0 else n + i


def load_obj_scene(path: str, camera_position=(0.0, 1.0, 5.0), camera_orientation=None, fov_y_deg: float = 50.0,
                   texture_loader=None) -> scenes.Scene:
    """OBJ (+ mtllib, + PNG maps) -> Scene with one mesh per material group and one identity instance"""
    base = os.path.dirname(os.path.abspath(path))
    pos: List[List[float]] = []
    tcs: List[List[float]] = []
    nrm: List[List[float]] = []
    groups: Dict[str, List[List[Tuple[int, int, int]]]] = {}
    order: List[str] = []
    mtl: Dict[str, dict] = {}
    cur = "__default__"
    with open(path, "r") as fh:
        for line in fh:
            tok = line.split("#", 1)[0].split()
            if not tok:
                continue
            key = tok[0]
            if key == "v":
                pos.append([float(v) for v in tok[1:4]])
            elif key == "vt":
                tcs.append([float(tok[1]), float(tok[2]) if len(tok) > 2 else 0.0])
            elif key == "vn":
                nrm.append([float(v) for v in tok[1:4]])
            elif key == "mtllib":
                mtl.update(parse_mtl(os.path.join(base, " ".join(tok[1:]))))
            elif key == "usemtl":
                cur = " ".join(tok[1:])
            elif key == "f":
                corners = []
                for t in tok[1:]:
                    parts = t.split("/")
                    v = _index(parts[0], len(pos))
                    vt = _index(parts[1], len(tcs)) if len(parts) > 1 and parts[1] else -1
                    vn = _index(parts[2], len(nrm)) if len(parts) > 2 and parts[2] else -1
                    corners.append((v, vt, vn))
                if cur not in groups:
                    groups[cur] = []
                    order.append(cur)
                for k in range(1, len(corners) - 1):  # aiProcess_Triangulate: fan
                    groups[cur].append([corners[0], corners[k], corners[k + 1]])
    P = np.asarray(pos, dtype=np.float64).reshape(-1, 3)
    T = np.asarray(tcs, dtype=np.float64).reshape(-1, 2)
    N = np.asarray(nrm, dtype=np.float64).reshape(-1, 3)

    materials = np.zeros(len(order), dtype=scenes.MATERIAL_DTYPE)
    material_textures = np.full((len(order), 4), NO_TEXTURE, dtype=np.uint32)
    bump_maps = np.zeros((len(order), 2), dtype=np.uint32)
    bump_maps[:, 0] = NO_TEXTURE
    textures: List[np.ndarray] = []
    texture_index: Dict[Tuple[str, bool], Tuple[int, int]] = {}

    def texture_and_channels(name: str, srgb: bool) -> Tuple[int, int]:
        key = (name, srgb)
        if key not in texture_index:
            file = os.path.join(base, name)
            if texture_loader is not None:
                img = texture_loader(file)
            else:
                with open(file, "rb") as fh:
                    img = decode_png(fh.read())
            texture_index[key] = (len(textures), 1 if img.ndim == 2 else img.shape[2])
            textures.append(image_to_texture(img, srgb))
        return texture_index[key]

    def texture(name: str, srgb: bool) -> int:
        return texture_and_channels(name, srgb)[0]

    meshes: List[scenes.Mesh] = []
    for mi, name in enumerate(order):
        m = mtl.get(name, {})
        materials[mi]["bsdfType"] = scenes.BSDF_DIFFUSE_AND_SPECULAR
        materials[mi]["p0"] = np.asarray(m.get("Kd", [0.0, 0.0, 0.0]), dtype=F32)      # :2248-2252 (black when absent)
        materials[mi]["p1"] = np.asarray(m.get("Ks", [0.0, 0.0, 0.0]), dtype=F32)
        materials[mi]["p2"] = F32(math.sqrt(m.get("Ns", 0.0)) / 11.0)                   # :2271-2274
        ke = m.get("Ke", [0.0, 0.0, 0.0])
        if "map_Ke" in m:
            raise ValueError(f"material {name}: map_Ke (textured emitter) is not supported")
        if any(v > 0 for v in ke):
            materials[mi]["emittance"] = np.asarray(ke, dtype=F32)
            materials[mi]["hasEmittance"] = 1
        if "map_Kd" in m:
            material_textures[mi, 0] = texture(m["map_Kd"], True)
        if "map_Ks" in m:
            material_textures[mi, 1] = texture(m["map_Ks"], True)
        bump = m.get("bump", m.get("norm"))  # the HEIGHT slot first, then NORMALS (common_host.cpp:2280-2284)
        if bump is not None:
            # loadNormalTexture (common_host.cpp:1344-1356): UNORM texels (no sRGB decode); more than one channel = normal map,
            # except the file the reference special-cases for Crytek Sponza
            tex, channels = texture_and_channels(bump, False)
            normal_map = channels > 1 and os.path.basename(bump) != "spnza_bricks_a_bump.png"
            bump_maps[mi] = (tex, BUMP_NORMAL_MAP if normal_map else BUMP_HEIGHT_MAP)

        # aiProcess_JoinIdenticalVertices within the material group; GenNormals gives every face its own vertices
        tris = groups[name]
        vert_of: Dict[Tuple, int] = {}
        vp, vt, vn, faces = [], [], [], []
        for fi, tri in enumerate(tris):
            face_n = None
            if any(c[2] < 0 for c in tri):
                a, b, c3 = (P[c[0]] for c in tri)
                face_n = np.cross(b - a, c3 - a)
                ln = np.linalg.norm(face_n)
                face_n = face_n / ln if ln > 0 else np.array([0.0, 1.0, 0.0])
            idx = []
            for c in tri:
                key = (c[0], c[1], c[2]) if face_n is None else (c[0], c[1], ("face", fi))
                if key not in vert_of:
                    vert_of[key] = len(vp)
                    vp.append(P[c[0]])
                    uv = T[c[1]] if c[1] >= 0 else np.zeros(2)
                    vt.append([uv[0], 1.0 - uv[1]] if c[1] >= 0 else [0.0, 0.0])     # aiProcess_FlipUVs
                    n = N[c[2]] if face_n is None else face_n
                    ln = np.linalg.norm(n)
                    vn.append(n / ln if ln > 0 else np.array([0.0, 1.0, 0.0]))
                idx.append(vert_of[key])
            faces.append(idx)
        vp, vt, vn = np.asarray(vp), np.asarray(vt), np.asarray(vn)
        faces = np.asarray(faces, dtype=np.int64)
        # aiProcess_CalcTangentSpace: dP/du per triangle, accumulated per vertex
        tan = np.zeros_like(vp)
        e1, e2 = vp[faces[:, 1]] - vp[faces[:, 0]], vp[faces[:, 2]] - vp[faces[:, 0]]
        d1, d2 = vt[faces[:, 1]] - vt[faces[:, 0]], vt[faces[:, 2]] - vt[faces[:, 0]]
        det = d1[:, 0] * d2[:, 1] - d2[:, 0] * d1[:, 1]
        ok = np.abs(det) > 1e-20
        ft = np.zeros_like(e1)
        ft[ok] = (e1[ok] * d2[ok, 1:2] - e2[ok] * d1[ok, 1:2]) / det[ok, None]
        for k in range(3):
            np.add.at(tan, faces[:, k], ft)
        ln = np.linalg.norm(tan, axis=1)
        bad = ~(ln > 1e-20)
        tan[~bad] /= ln[~bad, None]
        if bad.any():  # the reference's fallback (:2347-2358): makeCoordinateSystem(normal)
            n = vn[bad]
            sign = np.where(n[:, 2] >= 0, 1.0, -1.0)
            a = -1.0 / (sign + n[:, 2])
            b = n[:, 0] * n[:, 1] * a
            tan[bad] = np.stack([1 + sign * n[:, 0] * n[:, 0] * a, sign * b, -sign * n[:, 0]], axis=1)
        meshes.append(scenes.Mesh(np.ascontiguousarray(vp, dtype=F32), np.ascontiguousarray(vn, dtype=F32),
                                  np.ascontiguousarray(tan, dtype=F32), np.ascontiguousarray(vt, dtype=F32),
                                  np.ascontiguousarray(faces, dtype=np.uint32), mi))
    if camera_orientation is None:
        camera_orientation = scenes.rot_y(180.0).astype(F32)
    scene = scenes.Scene(meshes, materials, [scenes.make_instance(list(range(len(meshes))))],
                         np.asarray(camera_position, dtype=F32), np.asarray(camera_orientation, dtype=F32),
                         math.radians(fov_y_deg), os.path.splitext(os.path.basename(path))[0])
    if textures:
        scene.textures = textures
        if (material_textures != NO_TEXTURE).any():  # otherwise every texture is a bump map
            scene.material_textures = material_textures
    if (bump_maps[:, 0] != NO_TEXTURE).any():
        scene.bump_maps = bump_maps
    return scene
