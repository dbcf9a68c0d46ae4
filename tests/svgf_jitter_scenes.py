"""A scene for the TAA sub-pixel jitter tests (GFX_SVGF_SUBPIXEL_JITTER): one rectangle facing the camera whose edges fall at
chosen fractional pixel positions, so that which samples hit it, and how much of each pixel it covers, is known analytically."""
import math

import numpy as np

from gfxexp_b200 import scenes

W = H = 32
FOV_Y = math.radians(40.0)
DIST = 10.0
# Edges in top-down pixel coordinates.  The fractions stay at least 1/32 px from every ox = halton(2, i) (multiples of 1/16)
# and 1/54 px from every 1 - oy = 1 - halton(3, i) (multiples of 1/27) for i < 16.
LEFT, RIGHT = 8 + 11 / 32, 23 + 11 / 32
TOP, BOTTOM = 9 + 16.5 / 27, 22 + 7.5 / 27
EMITTANCE = 10.0
DIFFUSE = 0.01  # small, so that the rectangle's light on itself (next-event estimation at grazing angles) stays negligible


def rect_scene(emissive: bool = True) -> scenes.Scene:
    """The camera at (0, -DIST, 0) looks along +y (right = +x, up = -z); a primary ray through the pixel position (sx, sy)
    meets the plane y = 0 at x = DIST vw (0.5 - sx / W), z = -DIST vh (0.5 - sy / H)."""
    vh = 2 * math.tan(FOV_Y * 0.5)
    vw = vh * W / H
    x_of = lambda sx: DIST * vw * (0.5 - sx / W)  # noqa: E731
    z_of = lambda sy: -DIST * vh * (0.5 - sy / H)  # noqa: E731
    x0, x1 = x_of(RIGHT), x_of(LEFT)
    z0, z1 = z_of(TOP), z_of(BOTTOM)
    pos = np.array([[x0, 0, z0], [x1, 0, z0], [x1, 0, z1], [x0, 0, z1]], dtype=np.float32)
    nrm = np.tile(np.array([0, -1, 0], dtype=np.float32), (4, 1))
    tan = np.tile(np.array([1, 0, 0], dtype=np.float32), (4, 1))
    uv = np.array([[0, 0], [1, 0], [1, 1], [0, 1]], dtype=np.float32)
    tris = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.uint32)
    mats = np.zeros(1, dtype=scenes.MATERIAL_DTYPE)
    mats[0]["p0"] = np.float32(DIFFUSE)
    mats[0]["bsdfType"] = scenes.BSDF_LAMBERT
    if emissive:
        mats[0]["emittance"] = np.float32(EMITTANCE)
        mats[0]["hasEmittance"] = 1
    mesh = scenes.Mesh(pos, nrm, tan, uv, tris, 0)
    return scenes.Scene([mesh], mats, [scenes.make_instance([0])], np.array([0.0, -DIST, 0.0], dtype=np.float32),
                        scenes.rot_x(-90.0).astype(np.float32), FOV_Y, "jitter_rect")


def coverage() -> np.ndarray:
    """the fraction of each pixel the rectangle covers, [H, W]"""
    def overlap(lo, hi, n):
        c = np.arange(n, dtype=np.float64)
        return np.clip(np.minimum(c + 1, hi) - np.maximum(c, lo), 0.0, 1.0)
    return overlap(TOP, BOTTOM, H)[:, None] * overlap(LEFT, RIGHT, W)[None, :]
