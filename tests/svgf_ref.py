"""Float64 numpy restatement of the reference's SVGF passes, written from the reference (not from gfxexp_b200/csrc/svgf.cu or
oracle/denoise.cpp), with a per-pixel bar for every float output.  TEST INFRASTRUCTURE: tests/test_oracle_svgf_ref.py holds the
oracle against it, tests/test_gpu_svgf_passes.py the device.

  svgf/gpu_kernels/optix_pathtracing_kernels.cu:12-128   reprojectPreviousAccumulation (temporal accumulation)
                                                :325-378  demodulation, EMA 1/5, moments and sample info
  svgf/gpu_kernels/svgf.cu:6-26      depth, normal and luminance weights
                          :30-134    estimateVariance
                          :221-354   applyATrousFilter_box3x3
                          :356-374   feedbackNoisyLighting
                          :378-461   fillBackground (without the environment light: the 0.001 grey)
                          :465-611   reprojectPreviousAccumulation + applyAlbedoModulationAndTemporalAntiAliasing

The library reads its G-buffers where the reference reads rasterised ones (position GBuffer2 xyz, instance GBuffer0.x, material
GBuffer3.w, encoded shading normal GBuffer3.x, motion vector GBuffer1) and derives the reference's GL depth from the view-space z
with camera(aspect, fovY, 0.1, 1000).

Continuous values are float64.  Decisions are exact: integer and equality tests on the float32 inputs are exact anyway; the
reprojection (prevScreenPos, its pixel, the side of fDelta, the bilinear weights) and the sample-count rounding are evaluated in
float32 as the reference does, so the chosen neighbours, accept flags and counts are those of float32 code; the normal test runs in
float64 and records its smallest distance to 0.85 in `margins`, which callers hold away from float32's decoding error.

The bar of an output is first-order propagation of the float32 rounding of the code under test, per pixel: u = 2^-24 per
operation, with the three ill-conditioned places propagated explicitly -- the luminance weight's argument |dl| / (4 sigma + 1e-6),
which is huge when sigma ~ 0, the 128th power of the normal dot product (relative error x 128) and the depth weight's argument.
The weights' bars are the width of exp(-[a - da, a + da]), so they never exceed 1.

The object is stateful like the device: planes keep what an earlier pass or frame left in them where a pass does not write, so sky
pixels keep stale lighting, which the 3x3 variance blur of the a-trous stages reads without a depth test.  A window (y0, rows) of a
taller frame restates the rows of the window only; reads outside it clamp to the window, so callers compare rows one pass
footprint (the reprojection's motion, 3 + 1 rows for the variance, stepWidth + 1 for a-trous) away from its edges.
"""
from __future__ import annotations

import numpy as np

from gfxexp_b200 import abi
from tests import shading_ref

U = 2.0 ** -24
SKY = 0xFFFFFFFF
LUM = shading_ref.LUM
F32 = np.float32
DEC_ERR = 64 * U           # |float32 decodeVector dot float32 decodeVector - exact dot|: two polar decodes, sin / cos of 4 ulp
EXP_ERR = 8 * U            # relative error of the float32 exp (Cephes expf)
VARIANCE_KERNEL = np.array([0.00598, 0.060626, 0.241843, 0.383103, 0.241843, 0.060626, 0.00598])


def f32_fma(a, b, c):
    """float32 fmaf(a, b, c): the float64 product of two float32 is exact, one rounding of the sum to float32"""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def exp_bar(a, da):
    """exp(-a) and the width of exp(-[a - da, a + da]) plus the float32 exp's own error"""
    w = np.exp(-a)
    return w, np.exp(-np.maximum(a - da, 0.0)) - np.exp(-(a + da)) + EXP_ERR * w + 1e-37


def luminance(rgb):
    """sRGB_calcLuminance and its float32 bar"""
    rgb = np.asarray(rgb, np.float64)
    return rgb @ LUM, 6 * U * (np.abs(rgb) @ LUM)


def safe_divide(a, b):
    """RGB::safeDivide: a / b per channel, 0 where b is 0"""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(b != 0, a / np.where(b != 0, b, 1.0), 0.0)


def cam_vh_vw(cam):
    vh = 2 * np.tan(np.float64(cam.fovY) * 0.5)
    return vh, np.float64(cam.aspect) * vh


def depth_row():
    """the GL projection's depth row of camera(aspect, fovY, 0.1, 1000), in float32 as the host computes it"""
    near, far = F32(0.1), F32(1000.0)
    dz = far - near
    return float(-(near + far) / dz), float(F32(-2) * far * near / dz)


class SvgfRef:
    """the SVGF state of one frame size (or of a row window of it) and the six passes on it"""

    def __init__(self, W: int, H: int, y0: int = 0, rows: int | None = None):
        self.W, self.H, self.y0 = W, H, y0
        self.rows = H - y0 if rows is None else rows
        n = (self.rows, W)
        self.gb0 = [np.zeros(n + (4,), np.uint32) for _ in range(2)]
        self.gb1 = [np.zeros(n + (2,), F32) for _ in range(2)]
        self.gb2 = [np.zeros(n + (4,), F32) for _ in range(2)]
        self.gb3 = [np.zeros(n + (4,), np.uint32) for _ in range(2)]
        self.beauty = np.zeros(n + (4,), F32)
        self.albedo_accum = np.zeros(n + (4,), F32)
        self.lighting = [np.zeros(n + (4,)) for _ in range(2)]
        self.moments = [np.zeros(n + (2,)) for _ in range(2)]
        self.info = [np.zeros(n, np.uint32) for _ in range(2)]   # sample count (24 bits) | accept flags << 24
        self.prev_lighting = np.zeros(n + (4,))
        self.albedo = np.zeros(n + (4,))
        self.depth = [np.zeros(n) for _ in range(2)]
        self.final = [np.zeros(n + (4,)) for _ in range(2)]
        self.prev_screen_pos = np.zeros(n + (2,))
        self.psp_bar = np.zeros(n)
        self.margins = {"normal": np.inf}
        yy, xx = np.mgrid[0:self.rows, 0:W]
        self.Y, self.X = yy + y0, xx

    # ---- state ------------------------------------------------------------------------------------------------------------
    def load(self, buffer_id: int, index: int, arr: np.ndarray):
        """a plane of the library's layout (full frame or window rows) into the state"""
        a = np.asarray(arr)
        if a.shape[0] == self.H and self.rows != self.H:
            a = a[self.y0:self.y0 + self.rows]
        f = a.view(F32) if a.dtype == np.uint32 else a
        i = index & 1
        if buffer_id == abi.BUF_GBUFFER0:
            self.gb0[i] = a.view(np.uint32).copy()
        elif buffer_id == abi.BUF_GBUFFER1:
            self.gb1[i] = a.astype(F32)
        elif buffer_id == abi.BUF_GBUFFER2:
            self.gb2[i] = a.view(F32).copy()
        elif buffer_id == abi.BUF_GBUFFER3:
            self.gb3[i] = a.view(np.uint32).copy()
        elif buffer_id == abi.BUF_BEAUTY_ACCUM:
            self.beauty = a.astype(F32)
        elif buffer_id == abi.BUF_ALBEDO_ACCUM:
            self.albedo_accum = a.astype(F32)
        elif buffer_id == abi.BUF_SVGF_LIGHTING_VARIANCE:
            self.lighting[i] = f.astype(np.float64)
        elif buffer_id == abi.BUF_SVGF_MOMENTS:
            u = a.view(np.uint32)
            self.moments[i] = u[..., :2].view(F32).astype(np.float64)
            self.info[i] = u[..., 2].copy()
        elif buffer_id == abi.BUF_SVGF_PREV_LIGHTING:
            self.prev_lighting = f.astype(np.float64)
        elif buffer_id == abi.BUF_SVGF_ALBEDO:
            self.albedo = f.astype(np.float64)
        elif buffer_id == abi.BUF_SVGF_DEPTH:
            self.depth[i] = f.astype(np.float64)
        elif buffer_id == abi.BUF_SVGF_FINAL:
            self.final[i] = f.astype(np.float64)
        else:
            raise ValueError(buffer_id)

    def _at(self, plane, gy, gx):
        """plane at global rows gy, columns gx (in the frame); rows outside the window clamp to it"""
        return plane[np.clip(gy - self.y0, 0, self.rows - 1), gx]

    def _sky(self, cur):
        return self.gb0[cur][..., 0] == SKY

    # ---- temporal accumulation (optix_pathtracing_kernels.cu:12-128, :325-378) --------------------------------------------
    def temporal(self, p) -> dict:
        W, H = self.W, self.H
        cur = p.bufferIndex & 1
        prv = (cur + 1) % 2
        flags = p.svgfFlags
        sky = self._sky(cur)
        geo = ~sky
        inst, mat = self.gb0[cur][..., 0], self.gb3[cur][..., 3]
        pos = self.gb2[cur][..., :3].astype(np.float64)
        n = shading_ref.decode_vector(self.gb3[cur][..., 0].ravel()).reshape(pos.shape)
        out = {}

        # GL depth of the hit point; 1 (the cleared depth buffer) on sky pixels
        o = np.array(p.camera.orientation, np.float64).reshape(3, 3)
        cp = np.array(p.camera.position, np.float64)
        pv = (pos - cp) @ np.linalg.inv(o).T
        zv = -pv[..., 2]
        m22, m23 = depth_row()
        with np.errstate(divide="ignore", invalid="ignore"):
            ndc = (m22 * zv + m23) / (-zv)
            depth = 0.5 * ndc + 0.5
            dzv = 16 * U * (np.linalg.norm(pos, axis=-1) + np.linalg.norm(cp)) * np.abs(np.linalg.inv(o)).sum(1).max()
            depth_bar = 4 * U + 0.5 * abs(m23) / zv ** 2 * dzv + 2 * U * np.abs(ndc)
        self.depth[cur] = np.where(sky, 1.0, depth)
        out["depth"] = (self.depth[cur], np.where(sky, 0.0, depth_bar))

        # demodulation by the DH reflectance; tiny reflectance counts as zero (:325-336)
        dh = self.albedo_accum[..., :3].astype(np.float64)
        dh = np.where(self.albedo_accum[..., :3] < F32(0.001), 0.0, dh)
        self.albedo[geo] = np.concatenate([dh, np.zeros(dh.shape[:-1] + (1,))], -1)[geo]
        out["albedo"] = (self.albedo, np.zeros(self.albedo.shape))

        # prevScreenPos = (pixel centre - motion vector) / size, in float32 as the G-buffer pass stores it
        mv = self.gb1[cur]
        psx = (self.X.astype(F32) + F32(0.5) - mv[..., 0]) / F32(W)
        psy = (self.Y.astype(F32) + F32(0.5) - mv[..., 1]) / F32(H)
        self.prev_screen_pos[geo] = np.stack([psx, psy], -1).astype(np.float64)[geo]
        self.psp_bar[geo] = 0.0

        # reprojectPreviousAccumulation
        ta = bool(flags & abi.SVGF_ENABLE_TEMPORAL_ACCUMULATION)
        oos = (psx < 0) | (psy < 0) | (psx >= 1) | (psy >= 1)
        reproj = geo & ~oos & ta
        pvx, pvy = F32(W) * np.where(reproj, psx, F32(0)), F32(H) * np.where(reproj, psy, F32(0))
        ppx, ppy = pvx.astype(np.int64), pvy.astype(np.int64)
        fdx = pvx - (ppx.astype(F32) + F32(0.5))
        fdy = pvy - (ppy.astype(F32) + F32(0.5))
        dlx, dly = np.where(fdx < 0, -1, 1), np.where(fdy < 0, -1, 1)
        cx, cy = np.clip(ppx + dlx, 0, W - 1), np.clip(ppy + dly, 0, H - 1)
        nbs = [(ppx, ppy), (cx, ppy), (ppx, cy), (cx, cy)]
        s32, t32 = np.abs(fdx), np.abs(fdy)
        one = F32(1)
        w32 = [(one - s32) * (one - t32), s32 * (one - t32), (one - s32) * t32, s32 * t32]
        sum_w = np.zeros(sky.shape)
        acc_l = np.zeros(sky.shape + (3,))
        acc_m = np.zeros(sky.shape + (2,))
        acc_abs_l = np.zeros(sky.shape + (3,))
        acc_abs_m = np.zeros(sky.shape + (2,))
        cnt32, sw32 = np.zeros(sky.shape, F32), np.zeros(sky.shape, F32)
        accept = np.zeros(sky.shape, np.uint32)
        normal_margin = np.inf
        for i, (nx, ny) in enumerate(nbs):
            ok = reproj.copy()
            ok &= (self._at(self.gb0[prv][..., 0], ny, nx) == inst) & (self._at(self.gb3[prv][..., 3], ny, nx) == mat)
            nb_n = shading_ref.decode_vector(self._at(self.gb3[prv][..., 0], ny, nx).ravel()).reshape(n.shape)
            d = np.sum(nb_n * n, -1)
            if ok.any():
                normal_margin = min(normal_margin, float(np.min(np.abs(d[ok] - 0.85))))
            ok &= d > 0.85
            # (prev - cur).sqLength() > 0.1f, the sum as nested fmaf (nvcc contracts x*x + y*y + z*z)
            diff = self._at(self.gb2[prv][..., :3], ny, nx) - self.gb2[cur][..., :3]
            sq = f32_fma(diff[..., 2], diff[..., 2], f32_fma(diff[..., 1], diff[..., 1], diff[..., 0] * diff[..., 0]))
            ok &= ~(sq > F32(0.1))
            w = np.where(ok, w32[i].astype(np.float64), 0.0)
            nb_l = self._at(self.prev_lighting, ny, nx)[..., :3]
            nb_m = self._at(self.moments[prv], ny, nx)
            nb_c = self._at(self.info[prv], ny, nx) & 0xFFFFFF
            acc_l += w[..., None] * nb_l
            acc_m += w[..., None] * nb_m
            acc_abs_l += w[..., None] * np.abs(nb_l)
            acc_abs_m += w[..., None] * np.abs(nb_m)
            sum_w += w
            cnt32 = np.where(ok, cnt32 + w32[i] * nb_c.astype(F32), cnt32)
            sw32 = np.where(ok, sw32 + w32[i], sw32)
            accept |= np.where(ok, np.uint32(1 << i), np.uint32(0))
        self.margins["normal"] = min(self.margins["normal"], normal_margin)
        has = sum_w > 0
        with np.errstate(divide="ignore", invalid="ignore"):
            prev_l = np.where(has[..., None], acc_l / sum_w[..., None], 0.0)
            prev_m = np.where(has[..., None], acc_m / sum_w[..., None], 0.0)
            prev_l_bar = np.where(has[..., None], 10 * U * acc_abs_l / sum_w[..., None], 0.0)
            prev_m_bar = np.where(has[..., None], 10 * U * acc_abs_m / sum_w[..., None], 0.0)
            prev_count = np.where(has, np.floor((cnt32 / sw32).astype(np.float64) + 0.5), 0).astype(np.int64)  # roundf
        prev_flags = np.where(has, accept, 0)
        if (flags & abi.SVGF_IS_FIRST_FRAME) or not ta:
            prev_count[:] = 0
            prev_flags[:] = 0

        dem = safe_divide(self.beauty[..., :3].astype(np.float64), dh)
        dem_bar = U * np.abs(dem)
        lum, lum_bar = luminance(dem)
        lum_bar = lum_bar + dem_bar @ LUM
        sq, sq_bar = lum * lum, 2 * np.abs(lum) * lum_bar + U * lum * lum
        count = np.minimum(prev_count + 1, 65535)
        blend = (count > 1) & ta
        cw = np.where(count >= 5, 1 / 5, 1 / np.maximum(count, 1))   # EMA 1/5, cumulative average below 5 samples
        pw = 1 - cw

        def mix(prev, prev_bar, curv, cur_bar):
            b, c, q = (blend, cw, pw) if prev.ndim == 2 else (blend[..., None], cw[..., None], pw[..., None])
            v = q * prev + c * curv
            vb = q * prev_bar + c * cur_bar + 3 * U * (q * np.abs(prev) + c * np.abs(curv))
            return np.where(b, v, curv), np.where(b, vb, cur_bar)

        dem, dem_bar = mix(prev_l, prev_l_bar, dem, dem_bar)
        lum, lum_bar = mix(prev_m[..., 0], prev_m_bar[..., 0], lum, lum_bar)
        sq, sq_bar = mix(prev_m[..., 1], prev_m_bar[..., 1], sq, sq_bar)

        lighting0 = np.concatenate([dem, np.zeros(sky.shape + (1,))], -1)
        self.lighting[0] = np.where(sky[..., None], 0.0, lighting0)
        out["lighting0"] = (self.lighting[0], np.where(sky[..., None], 0.0, np.concatenate([dem_bar, np.zeros(sky.shape + (1,))], -1)))
        self.moments[cur] = np.where(geo[..., None], np.stack([lum, sq], -1), self.moments[cur])
        self.info[cur] = np.where(geo, (count.astype(np.uint32) & 0xFFFFFF) | (prev_flags.astype(np.uint32) << 24),
                                  self.info[cur])
        out["moments"] = (self.moments[cur], np.stack([lum_bar, sq_bar], -1), geo)
        out["info"] = (self.info[cur], geo)
        return out

    # ---- shared filter geometry (svgf.cu:6-26, 71-80, 264-272) ----------------------------------------------------------
    def _gradient(self, cur):
        W, H = self.W, self.H
        d = self.depth[cur]
        dx = np.where(self.X < W // 2, 1, -1)
        dy = np.where(self.Y < H // 2, 1, -1)
        hnb = self._at(d, self.Y, self.X + dx)
        vnb = self._at(d, self.Y + dy, self.X)
        return d, (hnb - d) * dx, (vnb - d) * dy, U * np.abs(hnb - d), U * np.abs(vnb - d)

    def _tap_weights(self, cur, ox, oy, n):
        """the depth and normal weights of the tap at offset (ox, oy) (arrays or ints), where it lies inside the frame and is not
        sky, with their bars; returns (valid, wz, dwz, wn, dwn, neighbour pixel (y, x))"""
        W, H = self.W, self.H
        d, dzdx, dzdy, ddzdx, ddzdy = self._grad
        nx, ny = self.X + ox, self.Y + oy
        inside = (nx >= 0) & (nx < W) & (ny >= 0) & (ny < H)
        cx, cy = np.clip(nx, 0, W - 1), np.clip(ny, 0, H - 1)
        nb_d = self._at(d, cy, cx)
        valid = inside & (nb_d != 1.0) & ~self._sky(cur)
        num = np.abs(nb_d - d)
        g = np.abs(dzdx * ox + dzdy * oy)
        den = g + 1e-6
        dden = 3 * U * (np.abs(dzdx * ox) + np.abs(dzdy * oy)) + np.abs(ox) * ddzdx + np.abs(oy) * ddzdy + U * den
        a = num / den
        wz, dwz = exp_bar(a, a * (3 * U + dden / den))
        nb_n = self._at(n, cy, cx)
        c = np.maximum(0.0, np.einsum("...k,...k->...", nb_n, n))
        wn = c ** 128
        dwn = np.minimum(c + DEC_ERR, 1.0) ** 128 - np.maximum(c - DEC_ERR, 0.0) ** 128 + 128 * U * wn
        return valid, wz, dwz, wn, dwn, (cy, cx)

    # ---- estimateVariance (svgf.cu:30-134) --------------------------------------------------------------------------------
    def variance(self, p) -> dict:
        cur = p.bufferIndex & 1
        geo = ~self._sky(cur)
        m1, m2 = self.moments[cur][..., 0], self.moments[cur][..., 1]
        count = self.info[cur] & 0xFFFFFF
        spatial = geo & (count < 4)
        self._grad = self._gradient(cur)
        n = shading_ref.decode_vector(self.gb3[cur][..., 0].ravel()).reshape(m1.shape + (3,))
        c = VARIANCE_KERNEL[3] ** 2
        taps = []
        for i in range(-3, 4):
            for j in range(-3, 4):
                if i == 0 and j == 0:
                    continue
                valid, wz, dwz, wn, dwn, nb = self._tap_weights(cur, j, i, n)
                h = VARIANCE_KERNEL[j + 3] * VARIANCE_KERNEL[i + 3]
                w = np.where(valid, h * wz * wn, 0.0)
                dw = np.where(valid, h * (dwz * wn + wz * dwn) + 4 * U * h * wz * wn, 0.0)
                taps.append((w, dw, self._at(self.moments[cur], *nb)))
        sw = c + sum(t[0] for t in taps)
        s1 = c * m1 + sum(t[0] * t[2][..., 0] for t in taps)
        s2 = c * m2 + sum(t[0] * t[2][..., 1] for t in taps)
        a1 = c * np.abs(m1) + sum(t[0] * np.abs(t[2][..., 0]) for t in taps)
        a2 = c * np.abs(m2) + sum(t[0] * np.abs(t[2][..., 1]) for t in taps)
        f1, f2 = s1 / sw, s2 / sw
        d1 = (sum(t[1] * np.abs(t[2][..., 0] - f1) for t in taps) + 52 * U * a1) / sw
        d2 = (sum(t[1] * np.abs(t[2][..., 1] - f2) for t in taps) + 52 * U * a2) / sw
        m1 = np.where(spatial, f1, m1)
        m2 = np.where(spatial, f2, m2)
        d1, d2 = np.where(spatial, d1, 0.0), np.where(spatial, d2, 0.0)
        var = np.maximum(m2 - m1 * m1, 0.0)
        bar = d2 + 2 * np.abs(m1) * d1 + 3 * U * (np.abs(m2) + m1 * m1)
        self.lighting[0][..., 3] = np.where(geo, var, self.lighting[0][..., 3])
        full_bar = np.zeros(self.lighting[0].shape)
        full_bar[..., 3] = np.where(geo, bar, 0.0)
        return {"lighting0": (self.lighting[0], full_bar)}

    # ---- applyATrousFilter_box3x3 (svgf.cu:221-354) -----------------------------------------------------------------------
    def atrous(self, p, stage: int) -> dict:
        assert 0 <= stage <= 4
        step = (1, 2, 4, 8, 16)[stage]
        cur = p.bufferIndex & 1
        geo = ~self._sky(cur)
        src = self.lighting[stage % 2]
        dst_i = (stage + 1) % 2
        feedback = bool(p.svgfFlags & abi.SVGF_FEEDBACK_1ST)
        if stage == 0 and not feedback:
            self.prev_lighting = np.where(geo[..., None], src, self.prev_lighting)
        lum, lum_bar = luminance(src[..., :3])
        self._grad = self._gradient(cur)
        n = shading_ref.decode_vector(self.gb3[cur][..., 0].ravel()).reshape(src.shape[:-1] + (3,))

        # 3x3 Gaussian of the variance, clamped at the border, no depth test (sky pixels' stale values included)
        gk = (0.25, 0.5, 0.25)
        local = np.zeros(lum.shape)
        for i in (-1, 0, 1):
            for j in (-1, 0, 1):
                ny, nx = np.clip(self.Y + i, 0, self.H - 1), np.clip(self.X + j, 0, self.W - 1)
                local += gk[i + 1] * gk[j + 1] * self._at(src[..., 3], ny, nx)
        sigma = np.sqrt(local)
        dsigma = 6 * U * sigma
        den_l = 4 * sigma + 1e-6
        dden_l = 4 * dsigma + 2 * U * den_l

        out_l = src[..., :3].copy()
        out_v = src[..., 3].copy()
        abs_l = np.abs(src[..., :3]).copy()
        sw = np.ones(lum.shape)
        taps = []
        for k in range(9):
            if k == 4:
                continue
            ox, oy = (k % 3 - 1) * step, (k // 3 - 1) * step
            valid, wz, dwz, wn, dwn, nb = self._tap_weights(cur, ox, oy, n)
            nb_lv = self._at(src, *nb)
            nb_lum, nb_lum_bar = luminance(nb_lv[..., :3])
            a = np.abs(nb_lum - lum) / den_l
            da = (nb_lum_bar + lum_bar + U * np.abs(nb_lum - lum)) / den_l + a * (dden_l / den_l + 2 * U)
            wl, dwl = exp_bar(a, da)
            w = np.where(valid, wz * wn * wl, 0.0)
            dw = np.where(valid, dwz * wn * wl + wz * dwn * wl + wz * wn * dwl + 3 * U * wz * wn * wl, 0.0)
            out_l += w[..., None] * nb_lv[..., :3]
            abs_l += w[..., None] * np.abs(nb_lv[..., :3])
            out_v += w * w * nb_lv[..., 3]
            sw += w
            taps.append((w, dw, nb_lv))
        res_l = out_l / sw[..., None]
        res_v = out_v / sw ** 2
        bar_l = (sum(t[1][..., None] * np.abs(t[2][..., :3] - res_l) for t in taps) + 12 * U * abs_l) / sw[..., None]
        dsw = sum(t[1] for t in taps)
        bar_v = sum(2 * t[0] * t[1] * t[2][..., 3] for t in taps) / sw ** 2 + 2 * res_v * dsw / sw + 16 * U * res_v
        res = np.concatenate([res_l, res_v[..., None]], -1)
        self.lighting[dst_i] = np.where(geo[..., None], res, self.lighting[dst_i])
        bar = np.where(geo[..., None], np.concatenate([bar_l, bar_v[..., None]], -1), 0.0)
        out = {f"lighting{dst_i}": (self.lighting[dst_i], bar)}
        if stage == 0 and feedback:
            self.prev_lighting = np.where(geo[..., None], res, self.prev_lighting)
            out["prev_lighting"] = (self.prev_lighting, bar)
        elif stage == 0:
            out["prev_lighting"] = (self.prev_lighting, np.zeros(bar.shape))
        return out

    # ---- feedbackNoisyLighting (svgf.cu:356-374) --------------------------------------------------------------------------
    def feedback_noisy_lighting(self) -> dict:
        self.prev_lighting = self.lighting[0].copy()
        return {"prev_lighting": (self.prev_lighting, np.zeros(self.prev_lighting.shape))}

    # ---- fillBackground (svgf.cu:378-461), environment light off ----------------------------------------------------------
    def background(self, p, num_filtering_stages: int) -> dict:
        cur = p.bufferIndex & 1
        sky = self._sky(cur)
        plane = num_filtering_stages % 2
        self.lighting[plane] = np.where(sky[..., None], np.array([0.001, 0.001, 0.001, 0.0]), self.lighting[plane])
        self.albedo = np.where(sky[..., None], np.array([1.0, 1.0, 1.0, 0.0]), self.albedo)
        vh, vw = cam_vh_vw(p.camera)
        fx, fy = (self.X + 0.5) / self.W, (self.Y + 0.5) / self.H
        o = np.array(p.camera.orientation, np.float64).reshape(3, 3)
        local = np.stack([vw * (0.5 - fx), vh * (0.5 - fy), np.ones(fx.shape)], -1)
        d = local @ o.T
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        po = np.array(p.prevCamera.orientation, np.float64).reshape(3, 3)
        d = d @ po
        d = d / d[..., 2:3]
        pvh, pvw = cam_vh_vw(p.prevCamera)
        psp = np.stack([0.5 - d[..., 0] / pvw, 0.5 - d[..., 1] / pvh], -1)
        self.prev_screen_pos = np.where(sky[..., None], psp, self.prev_screen_pos)
        self.psp_bar = np.where(sky, 64 * U * (1 + np.abs(d[..., 0]) / pvw + np.abs(d[..., 1]) / pvh), self.psp_bar)
        bar = np.zeros(self.lighting[plane].shape)
        bar[..., :3] = np.where(sky[..., None], U * 0.001, 0.0)
        return {f"lighting{plane}": (self.lighting[plane], bar), "albedo": (self.albedo, np.zeros(bar.shape))}

    # ---- albedo modulation + TAA (svgf.cu:465-611) ------------------------------------------------------------------------
    def modulate_taa(self, p, num_filtering_stages: int) -> dict:
        W, H = self.W, self.H
        cur = p.bufferIndex & 1
        prv = (cur + 1) % 2
        src = self.lighting[num_filtering_stages % 2][..., :3]
        modulate = bool(p.svgfFlags & abi.SVGF_MODULATE_ALBEDO)
        alb = self.albedo[..., :3] if modulate else np.ones(src.shape)
        fl = src * alb
        fl_bar = U * np.abs(fl)
        if (p.svgfFlags & abi.SVGF_ENABLE_TAA) and not (p.svgfFlags & abi.SVGF_IS_FIRST_FRAME):
            psp, dpsp = self.prev_screen_pos, self.psp_bar
            oos = (psp[..., 0] < 0) | (psp[..., 1] < 0) | (psp[..., 0] >= 1) | (psp[..., 1] >= 1)
            pvx, pvy = W * np.where(oos, 0.0, psp[..., 0]), H * np.where(oos, 0.0, psp[..., 1])
            ppx, ppy = np.floor(pvx).astype(np.int64), np.floor(pvy).astype(np.int64)
            fdx, fdy = pvx - (ppx + 0.5), pvy - (ppy + 0.5)
            cx = np.clip(ppx + np.where(fdx < 0, -1, 1), 0, W - 1)
            cy = np.clip(ppy + np.where(fdy < 0, -1, 1), 0, H - 1)
            s, t = np.abs(fdx), np.abs(fdy)
            pf = self.final[prv][..., :3]
            taps = [((1 - s) * (1 - t), ppx, ppy), (s * (1 - t), cx, ppy), ((1 - s) * t, ppx, cy), (s * t, cx, cy)]
            prev = sum(w[..., None] * self._at(pf, y, x) for w, x, y in taps)
            prev_abs = sum(w[..., None] * np.abs(self._at(pf, y, x)) for w, x, y in taps)
            # the bilinear lookup is continuous in prevScreenPos inside the screen: a position off by d moves it by at most
            # d times the spread of the 3x3 previous pixels around the base pixel
            lo, hi = np.full(prev.shape, np.inf), np.full(prev.shape, -np.inf)
            for i in (-1, 0, 1):
                for j in (-1, 0, 1):
                    v = self._at(pf, np.clip(ppy + i, 0, H - 1), np.clip(ppx + j, 0, W - 1))
                    lo, hi = np.minimum(lo, v), np.maximum(hi, v)
            dfd = (W + H) * dpsp + 4 * U * (np.abs(pvx) + np.abs(pvy) + 1)
            prev_bar = 12 * U * prev_abs + 2 * dfd[..., None] * (hi - lo)
            prev = np.where(oos[..., None], 0.0, prev)
            prev_bar = np.where(oos[..., None], 0.0, prev_bar)

            box_min, box_max, cross_min, cross_max = fl.copy(), fl.copy(), fl.copy(), fl.copy()
            mag = np.abs(fl).copy()
            for i in (-1, 0, 1):
                for j in (-1, 0, 1):
                    if i == 0 and j == 0:
                        continue
                    ny, nx = np.clip(self.Y + i, 0, H - 1), np.clip(self.X + j, 0, W - 1)
                    v = self._at(src, ny, nx) * self._at(alb, ny, nx)
                    mag = np.maximum(mag, np.abs(v))
                    box_min, box_max = np.minimum(box_min, v), np.maximum(box_max, v)
                    if i == 0 or j == 0:
                        cross_min, cross_max = np.minimum(cross_min, v), np.maximum(cross_max, v)
            nb_min, nb_max = 0.5 * (box_min + cross_min), 0.5 * (box_max + cross_max)
            clamp_bar = 3 * U * mag
            prev = np.minimum(np.maximum(prev, nb_min), nb_max)
            prev_bar = np.maximum(prev_bar, clamp_bar)
            cw = 1.0 / p.taaHistoryLength
            pw = 1.0 - cw
            fl_bar = pw * prev_bar + cw * fl_bar + 3 * U * (pw * np.abs(prev) + cw * np.abs(fl))
            fl = pw * prev + cw * fl
        self.final[cur] = np.concatenate([fl, np.ones(fl.shape[:-1] + (1,))], -1)
        bar = np.concatenate([fl_bar, np.zeros(fl.shape[:-1] + (1,))], -1)
        return {f"final{cur}": (self.final[cur], bar)}
