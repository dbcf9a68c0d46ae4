"""Bump mapping on the CPU (perFramePlp.enableBumpMapping): detmath's dm_atan against libm, the oracle's applyBumpMapping,
readModifiedNormal and height-map gather against float64 / float32 numpy restatements of common_device.cuh:176-240, the
switch's effect on the oracle's G-buffer, and the importer's bump-map keys."""
import os

import numpy as np
import pytest

from gfxexp_b200 import abi, ingest, scenes
from tests import oracle_bump, texture_ref

F32 = np.float32


def _query(oscene, op, mat, inp, width):
    return oscene.bump_query(op, mat, inp, width)


@pytest.fixture(scope="module")
def bumped():
    scene = scenes.small_city_scene_bumped()
    return scene, oracle_bump.OracleScene(scene, build_bvh=False)


def test_atan_against_libm():
    x = np.concatenate([np.linspace(-60.0, 60.0, 400001), np.geomspace(1e-6, 1e7, 100001), -np.geomspace(1e-6, 1e7, 100001)])
    x = x.astype(F32)
    y = oracle_bump.dm_atan(x)
    assert np.max(np.abs(y - np.arctan(x.astype(np.float64)))) < 6e-7
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-40, -1e-40, 1e-45, 3.4e38, -3.4e38], dtype=F32)
    ys = oracle_bump.dm_atan(special)
    assert ys[0] == 0 and not np.signbit(ys[0]) and ys[1] == 0 and np.signbit(ys[1])
    assert ys[2] == F32(np.pi / 2) and ys[3] == -F32(np.pi / 2) and np.isnan(ys[4])
    assert ys[5] == special[5] and ys[6] == special[6] and ys[7] == special[7]  # atan(x) = x below the float epsilon
    assert abs(ys[8] - np.pi / 2) < 2e-7 and abs(ys[9] + np.pi / 2) < 2e-7


def _random_frames(rng, k):
    q, _ = np.linalg.qr(rng.normal(size=(k, 3, 3)))
    return q[:, :, 0], q[:, :, 1], q[:, :, 2]


def test_apply_bump_mapping_against_float64(bumped):
    _, oscene = bumped
    rng = np.random.default_rng(5)
    k = 20000
    t, b, nn = _random_frames(rng, k)
    n = rng.normal(size=(k, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    n[: k // 4, 2] = np.abs(n[: k // 4, 2])          # tilts of both signs, z > 0 and z <= 0
    n[k // 4: k // 4 + 50] = [0.0, 0.0, 1.0]          # no tilt at all
    n[k // 4 + 50: k // 4 + 100, :2] *= 1e-4          # projLength < 1e-3: the frame comes back unchanged
    inp = np.concatenate([n, t, b, nn], 1).astype(F32)
    got = _query(oscene, 1, 0, inp, 9).astype(np.float64)
    i64 = inp.astype(np.float64)
    want = texture_ref.apply_bump_mapping(i64[:, 0:3], i64[:, 3:6], i64[:, 6:9], i64[:, 9:12])
    assert np.abs(got - want).max() < 2e-5
    small = slice(k // 4, k // 4 + 100)
    assert np.array_equal(got[small], inp[small, 3:12].astype(np.float64))  # bit for bit: returned as it came
    # a unit modified normal turns an orthonormal frame into an orthonormal frame
    T, B, N = got[:, 0:3], got[:, 3:6], got[:, 6:9]
    for a, c in ((T, B), (B, N), (T, N)):
        assert np.abs(np.sum(a * c, 1)).max() < 1e-5
    for a in (T, B, N):
        assert np.abs(np.linalg.norm(a, axis=1) - 1).max() < 1e-5


def test_non_unit_normal_is_kept(bumped):
    _, oscene = bumped
    n = np.array([[0.3, -0.2, 0.5]], dtype=F32)  # |n| = 0.62: the frame normal keeps that length
    inp = np.concatenate([n, [[1, 0, 0, 0, 1, 0, 0, 0, 1]]], 1)
    got = _query(oscene, 1, 0, inp, 9)
    assert np.allclose(got[0, 6:9], n[0], atol=1e-7)


def test_default_texel_tilts_every_material(bumped):
    """createNormalTexture's 1x1 (127, 127, 255) texel: (-1/255, 1/255, 1) after the y flip, a tilt of atan(sqrt(2) / 255)"""
    scene, oscene = bumped
    m = int(np.flatnonzero(scene.bump_maps[:, 0] == abi.NO_BUMP_MAP)[0])
    uv = np.random.default_rng(1).uniform(-3, 3, (64, 2)).astype(F32)
    n = _query(oscene, 0, m, uv, 3)
    texel = np.array([[[F32(127) / F32(255), F32(127) / F32(255), 1, 1]]], dtype=F32)
    blend, _ = texture_ref.fetch_repeat(texel, uv[:, 0], uv[:, 1])  # the software filter's four taps of the one texel
    want = F32(2) * blend[:, :3] - F32(1)
    want[:, 1] = -want[:, 1]
    assert np.array_equal(n, want)
    assert np.abs(n - np.array([-1 / 255, 1 / 255, 1])).max() < 1e-6
    frame = _query(oscene, 1, 0, np.concatenate([n[:1], [[1, 0, 0, 0, 1, 0, 0, 0, 1]]], 1), 9)
    tilt = np.arccos(frame[0, 8] / np.linalg.norm(frame[0, 6:9]))
    assert abs(tilt - np.arctan(np.sqrt(2) / 255)) < 1e-5 and abs(np.sqrt(2) / 255 - 0.0055) < 1e-4


def test_normal_decode_and_height_gather_against_numpy(bumped):
    scene, oscene = bumped
    rng = np.random.default_rng(9)
    uv = rng.uniform(-2.5, 3.5, (4000, 2)).astype(F32)
    uv[:200] = (rng.integers(-8, 8, (200, 2)) / F32(8)).astype(F32)  # texel-boundary coordinates
    u, v = uv[:, 0], uv[:, 1]
    seen = set()
    for m in range(scene.materials.shape[0]):
        tex_index, kind = (int(x) for x in scene.bump_maps[m])
        if tex_index == abi.NO_BUMP_MAP or tex_index in seen:
            continue
        seen.add(tex_index)
        tex = scene.textures[tex_index]
        got_n = _query(oscene, 0, m, uv, 3)
        got_g = _query(oscene, 2, m, uv, 4)
        blend, _ = texture_ref.fetch_repeat(tex, u, v)
        x0, x1, y0, y1 = texture_ref.gather_indices(tex, u, v)
        want_g = np.stack([tex[y1, x0, 0], tex[y1, x1, 0], tex[y0, x1, 0], tex[y0, x0, 0]], 1)
        assert np.array_equal(got_g, want_g)
        if kind == abi.BUMP_NORMAL_MAP:
            want = F32(2) * blend[:, :3] - F32(1)
            want[:, 1] = -want[:, 1]
            assert np.array_equal(got_n, want)
        else:
            H, W = tex.shape[:2]
            coeff = F32(5.0 / 1024)
            dhdu = (coeff * F32(W)) * (want_g[:, 1] - want_g[:, 0])
            dhdv = (coeff * F32(H)) * (want_g[:, 0] - want_g[:, 3])
            n = np.stack([-dhdu, dhdv, np.ones_like(dhdu)], 1).astype(np.float64)
            assert np.abs(got_n - n / np.linalg.norm(n, axis=1, keepdims=True)).max() < 1e-6
            assert np.abs(np.linalg.norm(got_n, axis=1) - 1).max() < 1e-6
    assert len(seen) == 4  # both normal maps and both height maps were checked


def test_switch_changes_only_what_it_should(bumped):
    """the oracle G-buffer: off on the bumped scene = the same scene without a bump table; on differs"""
    scene, oscene = bumped
    plain = scenes.small_city_scene_bumped()
    plain.bump_maps = None
    oplain = oracle_bump.OracleScene(plain)
    oscene_bvh = oracle_bump.OracleScene(scene)
    W, H = 48, 32
    out = {}
    for key, osc, on in (("off", oscene_bvh, 0), ("plain", oplain, 0), ("on", oscene_bvh, 1)):
        f = oracle_bump.OracleFrame(osc, W, H)
        p = abi.default_frame_params(scene, W, H)
        p.enableBumpMapping = on
        f.gbuffer(p)
        out[key] = [f.buffer(b, 0).copy() for b in (abi.BUF_GBUFFER3, abi.BUF_ALBEDO_ACCUM, abi.BUF_NORMAL_ACCUM)]
    for a, b in zip(out["off"], out["plain"]):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert not np.array_equal(out["on"][0].view(np.uint32), out["off"][0].view(np.uint32))
    assert not np.array_equal(out["on"][2].view(np.uint32), out["off"][2].view(np.uint32))


def _write_obj(tmp_path, mtl_lines, images):
    for name, img in images.items():
        with open(os.path.join(tmp_path, name), "wb") as fh:
            fh.write(_png(img))
    with open(os.path.join(tmp_path, "m.mtl"), "w") as fh:
        fh.write("\n".join(mtl_lines) + "\n")
    lines = ["mtllib m.mtl", "v 0 0 0", "v 1 0 0", "v 0 1 0", "vt 0 0", "vt 1 0", "vt 0 1", "vn 0 0 1"]
    for k in range(len([ln for ln in mtl_lines if ln.startswith("newmtl")])):
        lines += [f"usemtl m{k}", "f 1/1/1 2/2/1 3/3/1"]
    path = os.path.join(tmp_path, "s.obj")
    with open(path, "w") as fh:
        fh.write("\n".join(lines) + "\n")
    return path


def _png(img):
    """grey (2-D) or RGB/RGBA uint8 -> PNG bytes"""
    import struct
    import zlib
    if img.ndim == 2:
        h, w = img.shape
        raw = b"".join(b"\x00" + img[y].tobytes() for y in range(h))

        def chunk(kind, body):
            return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body) & 0xFFFFFFFF)
        return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))
    return ingest.encode_png(img)


def test_ingest_bump_keys(tmp_path):
    rng = np.random.default_rng(3)
    grey = rng.integers(0, 256, (5, 7), dtype=np.uint8)
    rgb = rng.integers(0, 256, (4, 6, 3), dtype=np.uint8)
    sponza = rng.integers(0, 256, (3, 3, 3), dtype=np.uint8)
    mtl = ["newmtl m0", "Kd 0.5 0.5 0.5", "map_Bump -bm 0.3 h.png",    # one channel: height map
           "newmtl m1", "Kd 0.5 0.5 0.5", "bump n.png",                # RGB: normal map
           "newmtl m2", "Kd 0.5 0.5 0.5", "norm n.png",                # NORMALS slot
           "newmtl m3", "Kd 0.5 0.5 0.5", "map_Bump spnza_bricks_a_bump.png",  # the reference's Sponza exception
           "newmtl m4", "Kd 0.5 0.5 0.5", "norm h.png", "map_Bump n.png",     # HEIGHT before NORMALS
           "newmtl m5", "Kd 0.5 0.5 0.5"]                              # no map
    path = _write_obj(str(tmp_path), mtl, {"h.png": grey, "n.png": rgb, "spnza_bricks_a_bump.png": sponza})
    scene = ingest.load_obj_scene(path)
    bm = scene.bump_maps
    assert scene.material_textures is None  # no colour maps: the textures are all bump maps
    h, n = int(bm[0, 0]), int(bm[1, 0])
    assert bm[0, 1] == abi.BUMP_HEIGHT_MAP and bm[1, 1] == abi.BUMP_NORMAL_MAP
    assert tuple(bm[2]) == (n, abi.BUMP_NORMAL_MAP)
    assert bm[3, 1] == abi.BUMP_HEIGHT_MAP
    assert tuple(bm[4]) == (n, abi.BUMP_NORMAL_MAP)
    assert bm[5, 0] == abi.NO_BUMP_MAP
    # UNORM texels, no sRGB decode; a grey image is (g, g, g, 1) as stbi_load(..., 4) gives it
    assert np.array_equal(scene.textures[h][..., 0], grey.astype(F32) / F32(255))
    assert np.array_equal(scene.textures[h][..., 2], grey.astype(F32) / F32(255)) and (scene.textures[h][..., 3] == 1).all()
    assert np.array_equal(scene.textures[n][..., :3], rgb.astype(F32) / F32(255))
    desc = abi.SceneArrays(scene).desc  # and the C ABI carries the table
    assert bool(desc.bumpMaps) and desc.numTextures == len(scene.textures) and not bool(desc.materialTextures)


def test_ingest_keeps_map_ke_refusal(tmp_path):
    img = np.zeros((2, 2, 3), dtype=np.uint8)
    path = _write_obj(str(tmp_path), ["newmtl m0", "Ke 1 1 1", "map_Ke e.png", "map_Bump n.png"], {"e.png": img, "n.png": img})
    with pytest.raises(ValueError, match="map_Ke"):
        ingest.load_obj_scene(path)


@pytest.mark.parametrize("variant", [None, abi.PT_BASELINE, abi.PT_REGIR, abi.PT_NRC])
def test_switch_off_equals_the_oracle(variant):
    """the bump library's restated G-buffer pass and path tracers, switch off, give the oracle's buffers bit for bit (the
    restatement differs from render.cpp / pathtrace.inl / regir.inl / nrc_pathtrace.inl only at the frame sites)"""
    from tests import oracle_lib
    scene = scenes.small_city_scene_bumped()
    W, H = 40, 24
    frames = []
    for mod in (oracle_lib, oracle_bump):
        f = mod.OracleFrame(mod.OracleScene(scene), W, H)
        p = abi.default_frame_params(scene, W, H)
        p.maxPathLength = 4
        f.gbuffer(p)
        if variant == abi.PT_REGIR:
            f.regir_build_cells(p, 0, False)
        if variant == abi.PT_NRC:
            f.nrc_preprocess(p, 123, 456, True)
        if variant is not None:
            f.pathtrace(p, variant)
        bufs = [f.buffer(b, 0) for b in (abi.BUF_GBUFFER0, abi.BUF_GBUFFER2, abi.BUF_GBUFFER3, abi.BUF_NORMAL_ACCUM)]
        bufs += [f.buffer(abi.BUF_RNG), f.buffer(abi.BUF_BEAUTY_ACCUM)]
        if variant == abi.PT_NRC:
            bufs += [f.linear_buffer(abi.BUF_NRC_TERMINAL_INFO), f.linear_buffer(abi.BUF_NRC_TRAIN_VERTEX_INFO)]
        frames.append(bufs)
    for k, (a, b) in enumerate(zip(*frames)):
        assert np.array_equal(a.view(np.uint32) if a.dtype.itemsize == 4 else a, b.view(np.uint32) if b.dtype.itemsize == 4 else b), k
