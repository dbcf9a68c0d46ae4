"""Seeded synthetic G-buffers and SVGF histories, and a driver that runs the SVGF passes one at a time on the oracle or the
device.  TEST INFRASTRUCTURE for tests/test_oracle_svgf_ref.py and tests/test_gpu_svgf_passes.py.

A frame holds several instances and materials, sky holes inside the image (discs and single pixels), creases where neighbouring
normals' dot product is 0.84 or 0.86 (either side of the reprojection's 0.85), depth steps between regions, and motion vectors for
a pan with a zoom, per-region motion and a patch pointing off screen.  Positions sit within 0.004 of a per-region anchor, so the
previous frame's neighbours pass the distance test (squared distance < 0.01) except in a patch moved by sqrt(0.2) on odd frames;
a patch moved by sqrt(0.05) passes it.  Beauty is HDR with 1e4 fireflies and exact zeros, albedo has channels below 0.001 and
exact zeros, and the history has sample counts 1 .. 65 535 with every accept-flag pattern.

Continuous inputs stay at least 1e-3 (relative) from the passes' branch thresholds: the normal test, the distance test,
`depth == 1` (geometry depth <= 0.998), the screen bounds and the pixel grid of the reprojected position.  With
`thresholds=True` patches sit on them instead: a position offset of (0.31622776f, 0, 0), whose float32 squared length is exactly
0.1f, and the next float above it; normals as close to 0.85 as the 16-bit polar codes get while float32 decoding still decides
the test (2e-6 .. 1e-4); motion vectors to exact pixel centres, to prevScreenPos 0, exactly 1.0 and the float just under 1.0; a
sample count of exactly 4 and 3 into the variance pass; geometry pixels at depth exactly 1.0 and the float just under it.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from gfxexp_b200 import abi
from tests import shading_ref

F32 = np.float32
SKY = 0xFFFFFFFF
FRAME_BUFFERS = (abi.BUF_GBUFFER0, abi.BUF_GBUFFER1, abi.BUF_GBUFFER2, abi.BUF_GBUFFER3, abi.BUF_BEAUTY_ACCUM,
                 abi.BUF_ALBEDO_ACCUM)
SVGF_PLANES = [(abi.BUF_SVGF_LIGHTING_VARIANCE, 2), (abi.BUF_SVGF_MOMENTS, 2), (abi.BUF_SVGF_PREV_LIGHTING, 1),
               (abi.BUF_SVGF_ALBEDO, 1), (abi.BUF_SVGF_DEPTH, 2), (abi.BUF_SVGF_FINAL, 2)]
ALL_PLANES = [(b, 2) for b in FRAME_BUFFERS[:4]] + [(abi.BUF_BEAUTY_ACCUM, 1), (abi.BUF_ALBEDO_ACCUM, 1)] + SVGF_PLANES
DIST_EXACT = F32(0.31622776)   # float32 squared length exactly 0.1f
TINY = 1e-30   # absolute slack for products of weights that underflow float32 (squared weights ~1e-20 times variances)


def encode(phi, theta):
    """the 16-bit polar code nearest to (phi, theta), the inverse of shading_ref.decode_vector"""
    qp = np.round(np.mod(phi, 2 * np.pi) / (2 * np.pi) * 65535).astype(np.uint32)
    qt = np.round(np.clip(theta, 0, np.pi) / np.pi * 65535).astype(np.uint32)
    return qp | (qt << 16)


def code_with_dot(q, target, lo=0.0, hi=np.inf, side=0):
    """a code whose decoded direction has a dot product with q's as close to target as the codes allow, with
    lo <= |dot - target| < hi, above target for side 1, below for side -1"""
    n = shading_ref.decode_vector(np.array([q]))[0]
    theta0 = float(np.arccos(np.clip(n[1], -1, 1)))
    best, best_err = None, np.inf
    for dt in np.linspace(-np.arccos(target) * 0.9, np.arccos(target) * 0.9, 400):
        qt = np.uint32(np.clip(round((theta0 + dt) / np.pi * 65535), 1, 65534))
        cand_theta = float(qt) / 65535 * np.pi
        # dot = cos t0 cos t + sin t0 sin t cos(dphi): solve for dphi, take the codes either side
        s = np.sin(theta0) * np.sin(cand_theta)
        if s < 1e-6:
            continue
        c = (target - np.cos(theta0) * np.cos(cand_theta)) / s
        if abs(c) > 1:
            continue
        phi0 = 2 * np.pi * float(q & 0xFFFF) / 65535
        for sgn in (1, -1):
            ph = phi0 + sgn * np.arccos(c)
            base = int(np.floor(np.mod(ph, 2 * np.pi) / (2 * np.pi) * 65535))
            codes = np.array([(base + k) % 65536 for k in (-1, 0, 1, 2)], np.uint32) | (np.uint32(qt) << 16)
            d = shading_ref.decode_vector(codes) @ n
            err = np.abs(d - target)
            ok = (err >= lo) & (err < hi) & (np.sign(d - target) * side >= 0)
            if ok.any():
                k = int(np.argmin(np.where(ok, err, np.inf)))
                if err[k] < best_err:
                    best, best_err = int(codes[k]), float(err[k])
    assert best is not None
    return np.uint32(best)


def rotation_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], np.float32)


def camera(W, H, yaw=0.0):
    cam = abi.GfxCamera()
    cam.aspect = float(F32(W) / F32(H))
    cam.fovY = float(F32(0.9))
    cam.position = (C.c_float * 3)(0.0, 0.0, 0.0)
    cam.orientation = (C.c_float * 9)(*rotation_y(yaw).reshape(-1))
    return cam


def frame_params(W, H, frame, flags, hist=16, yaw_step=0.004):
    """the parameters of frame `frame`: buffer index frame % 2, the first-frame flag on frame 0, a camera turning by yaw_step
    per frame (the previous camera is the last frame's), no environment light"""
    p = abi.GfxFrameParams()
    p.camera = camera(W, H, yaw_step * frame)
    p.prevCamera = camera(W, H, yaw_step * max(frame - 1, 0))
    p.frameIndex = frame
    p.bufferIndex = frame % 2
    p.tileOriginY = 0
    p.tileRows = 0
    p.svgfFlags = (flags & ~abi.SVGF_IS_FIRST_FRAME) | (abi.SVGF_IS_FIRST_FRAME if frame == 0 else 0)
    p.taaHistoryLength = hist
    p.enableEnvLight = 0
    return p


class SyntheticScene:
    def __init__(self, W: int, H: int, seed: int = 1, thresholds: bool = False):
        self.W, self.H, self.thresholds = W, H, thresholds
        self.seed = seed
        rng = np.random.default_rng(seed)
        self.R = 5
        self.rects = []   # (x0, y0, w, h, vx, vy) of regions 1..R-1 in pixels, moving by (vx, vy) per frame
        for _ in range(self.R - 1):
            w, h = max(1, int(W * rng.uniform(0.2, 0.5))), max(1, int(H * rng.uniform(0.2, 0.5)))
            self.rects.append((rng.uniform(-0.1, 0.9) * W, rng.uniform(-0.1, 0.9) * H, w, h, rng.uniform(-2, 2), rng.uniform(-2, 2)))
        self.codes = encode(rng.uniform(0, 2 * np.pi, self.R), rng.uniform(0.3, 2.8, self.R))
        self.crease = np.array([code_with_dot(q, 0.84 if r % 2 else 0.86, 0, 0.002) for r, q in enumerate(self.codes)])
        self.crease_x = rng.uniform(0.3, 0.7, self.R) * W
        self.anchors = np.stack([rng.uniform(-2, 2, self.R), rng.uniform(-1, 1, self.R), 4 + 3 * np.arange(self.R)], -1)
        self.region_mv = rng.uniform(-3, 3, (self.R, 2))
        self.sky_discs = [(rng.uniform(0, W), rng.uniform(0, H), max(W, H) * rng.uniform(0.05, 0.15)) for _ in range(2)]
        self.depth_slopes = rng.uniform(-1e-4, 1e-4, (self.R, 2))
        if thresholds:   # the closest codes either side of 0.85 that float32 decoding still puts on that side
            self.code_near = [code_with_dot(self.codes[0], 0.85, 2e-6, 1e-4, side) for side in (1, -1)]

    # ---- layout ------------------------------------------------------------------------------------------------------------
    def _patch(self, k, frac=0.2):
        """a seeded sub-rectangle number k as a boolean mask"""
        rng = np.random.default_rng(self.seed * 1000 + k)
        W, H = self.W, self.H
        x0, y0 = int(rng.uniform(0, 1 - frac) * W), int(rng.uniform(0, 1 - frac) * H)
        m = np.zeros((H, W), bool)
        m[y0:y0 + max(1, int(frac * H)), x0:x0 + max(1, int(frac * W))] = True
        return m

    def labels(self, frame):
        W, H = self.W, self.H
        yy, xx = np.mgrid[0:H, 0:W] + 0.5
        lab = np.zeros((H, W), np.int64)
        for r, (x0, y0, w, h, vx, vy) in enumerate(self.rects, 1):
            x0, y0 = x0 + vx * frame, y0 + vy * frame
            lab[(xx >= x0) & (xx < x0 + w) & (yy >= y0) & (yy < y0 + h)] = r
        sky = np.zeros((H, W), bool)
        for cx, cy, rad in self.sky_discs:
            sky |= (xx - cx - frame) ** 2 + (yy - cy) ** 2 < rad ** 2
        rng = np.random.default_rng(self.seed * 7919 + frame)
        sky |= rng.random((H, W)) < 0.01       # single sky pixels inside geometry
        return lab, sky

    # ---- G-buffers of one frame -------------------------------------------------------------------------------------------
    def gbuffers(self, frame) -> dict:
        W, H = self.W, self.H
        rng = np.random.default_rng(self.seed * 31 + frame + 1000)
        lab, sky = self.labels(frame)
        yy, xx = np.mgrid[0:H, 0:W]
        gb0 = np.zeros((H, W, 4), np.uint32)
        gb0[..., 0] = lab + 1
        gb0[..., 1] = np.arange(W * H, dtype=np.uint32).reshape(H, W)
        gb3 = np.zeros((H, W, 4), np.uint32)
        gb3[..., 0] = np.where(xx + 0.5 > self.crease_x[lab], self.crease[lab], self.codes[lab])
        gb3[..., 3] = 10 + lab % 3
        matflip = self._patch(1, 0.15) & (frame % 2 == 1)
        gb3[..., 3] = np.where(matflip, 20, gb3[..., 3])
        pos = self.anchors[lab] + rng.uniform(-0.004, 0.004, (H, W, 3))
        far = self._patch(2, 0.2) & (frame % 2 == 1)
        pos[far, 0] += np.sqrt(0.2)
        mid = self._patch(3, 0.2) & (frame % 2 == 1)
        pos[mid, 0] += np.sqrt(0.05)
        pos = pos.astype(F32)

        # motion: zoom + pan on the background, per-region motion, a patch pointing off screen
        c = np.stack([xx + 0.5 - W / 2, yy + 0.5 - H / 2], -1)
        mv = 0.03 * c + np.array([1.3, -0.7])
        mv = np.where((lab > 0)[..., None], self.region_mv[lab], mv)
        mv[self._patch(4, 0.15)] = (1.5 * W, 0.25 * H)
        mv = self._keep_off_thresholds(mv, xx, yy)

        if self.thresholds:
            t = self._patch(5, 0.5)                   # exact positions and the 0.1f distance test
            pos[t] = np.array([0.0, 0.5, 6.0], F32)
            half = t & (xx % 2 == 0)
            if frame % 2 == 1:
                pos[half, 0] = DIST_EXACT
                pos[t & ~half, 0] = np.nextafter(DIST_EXACT, F32(1))
            gb0[t, 0] = 1
            gb3[t, 3] = 10
            gb3[t, 0] = self.codes[0]
            if frame % 2 == 1:                        # normals on either side of 0.85 (decided by float32 decoding)
                gb3[t & ((xx + yy) % 3 == 1), 0] = self.code_near[0]
                gb3[t & ((xx + yy) % 3 == 2), 0] = self.code_near[1]
            cen = self._patch(7, 0.3)                 # exact pixel centres
            mv[cen] = np.round(mv[cen])
            mv[t] = 0.0
            mv[yy % 5 == 0] = (xx[yy % 5 == 0] + 0.5)[:, None] * np.array([1.0, 0.0])   # prevScreenPos.x = 0
            # the last column at prevScreenPos.x = 1.0 exactly and the float under it, likewise the last row in y
            under_x, under_y = self._under_one(W), self._under_one(H)
            mv[:, W - 1, 0] = np.where(yy[:, W - 1] % 2 == 0, -0.5, under_x)
            mv[H - 1, :, 1] = np.where(xx[H - 1] % 2 == 0, -0.5, under_y)
        sky_u = sky
        gb0[sky_u, 0] = SKY
        gb3[sky_u, 3] = SKY
        gb2 = np.zeros((H, W, 4), F32)
        gb2[..., :3] = pos
        return {abi.BUF_GBUFFER0: gb0, abi.BUF_GBUFFER1: mv.astype(F32), abi.BUF_GBUFFER2: gb2.view(np.uint32),
                abi.BUF_GBUFFER3: gb3}

    @staticmethod
    def _under_one(n):
        """a motion vector m with float32 (n - 1 + 0.5 - m) / n the largest float under 1 it can give (the float just under 1
        unless the division cannot land there)"""
        m = (F32(-0.5) + np.arange(1, 1 << 14, dtype=np.float64) * 2.0 ** -25).astype(F32)   # the floats above -0.5
        r = (F32(n - 1) + F32(0.5) - m) / F32(n)
        return m[np.argmax(np.where(r < 1, r, 0))]

    def _keep_off_thresholds(self, mv, xx, yy):
        """nudge motion vectors so that the reprojected position is >= 1e-3 from the screen bounds (relative to the screen),
        from pixel edges and from pixel centres (1e-3 of a pixel)"""
        W, H = self.W, self.H
        for k, (n, coord) in enumerate(((W, xx), (H, yy))):
            pv = coord + 0.5 - mv[..., k]
            for _ in range(4):
                ps = pv / n
                near_bound = (np.abs(ps) < 1e-3) | (np.abs(ps - 1) < 1e-3)
                pv = np.where(near_bound, pv + 3e-3 * n, pv)
                fr = pv - np.floor(pv)
                near_grid = (fr < 1e-3) | (fr > 1 - 1e-3) | (np.abs(fr - 0.5) < 1e-3)
                pv = np.where(near_grid, pv + 2.5e-3, pv)
            mv[..., k] = coord + 0.5 - pv
        return mv

    # ---- shading inputs and the history -----------------------------------------------------------------------------------
    def shading(self, frame) -> dict:
        W, H = self.W, self.H
        rng = np.random.default_rng(self.seed * 17 + frame + 5000)
        beauty = np.zeros((H, W, 4), F32)
        beauty[..., :3] = np.exp(rng.normal(-1, 1.2, (H, W, 3)))
        beauty[rng.random((H, W)) < 0.005, :3] = 1e4
        beauty[rng.random((H, W)) < 0.02, :3] = 0.0
        beauty[..., 1][rng.random((H, W)) < 0.02] = 0.0
        albedo = np.zeros((H, W, 4), F32)
        albedo[..., :3] = rng.uniform(0.05, 1.0, (H, W, 3))
        pick = rng.random((H, W, 3))
        albedo[..., :3][pick < 0.03] = 0.0005
        albedo[..., :3][(pick >= 0.03) & (pick < 0.04)] = 0.0
        albedo[..., :3][(pick >= 0.04) & (pick < 0.05)] = 0.002
        return {abi.BUF_BEAUTY_ACCUM: beauty, abi.BUF_ALBEDO_ACCUM: albedo}

    def history(self, first_frame: int = 0) -> list:
        """(buffer, index, plane) of everything frame first_frame reads from earlier frames: the G-buffers of the two frames before,
        stale lighting planes, moments with sample counts 1 .. 65 535 and every accept-flag pattern, previous lighting, the
        previous final frame"""
        W, H = self.W, self.H
        rng = np.random.default_rng(self.seed * 13 + 99)
        out = [(b, (first_frame + k) % 2, a) for k in (0, 1) for b, a in self.gbuffers(first_frame + k - 2).items()]
        for i in range(2):
            lv = np.zeros((H, W, 4), F32)
            lv[..., :3] = np.exp(rng.normal(-1, 1, (H, W, 3)))
            lv[..., 3] = np.where(rng.random((H, W)) < 0.2, 0.0, rng.uniform(0, 2, (H, W)))
            out.append((abi.BUF_SVGF_LIGHTING_VARIANCE, i, lv.view(np.float32)))
            m = np.zeros((H, W, 4), np.uint32)
            m1 = rng.uniform(0, 3, (H, W)).astype(F32)
            m2 = (m1 * m1 * rng.uniform(0.8, 3, (H, W))).astype(F32)
            counts = rng.choice(np.array([1, 2, 3, 3, 4, 5, 6, 9, 100, 65534, 65535], np.uint32), (H, W))
            flags = rng.integers(0, 16, (H, W)).astype(np.uint32)
            m[..., 0], m[..., 1] = m1.view(np.uint32), m2.view(np.uint32)
            m[..., 2] = counts | (flags << 24)
            out.append((abi.BUF_SVGF_MOMENTS, i, m))
            fin = np.ones((H, W, 4), F32)
            fin[..., :3] = np.exp(rng.normal(-1, 1, (H, W, 3)))
            out.append((abi.BUF_SVGF_FINAL, i, fin))
            out.append((abi.BUF_SVGF_DEPTH, i, rng.uniform(0.9, 0.99, (H, W)).astype(F32)))
        pl = np.zeros((H, W, 4), F32)
        pl[..., :3] = np.exp(rng.normal(-1, 1, (H, W, 3)))
        out.append((abi.BUF_SVGF_PREV_LIGHTING, 0, pl))
        out.append((abi.BUF_SVGF_ALBEDO, 0, rng.uniform(0, 1, (H, W, 4)).astype(F32)))
        return out

    def depth(self, frame) -> np.ndarray:
        """the depth plane the filters read: a slanted plane per region with steps between regions, 1.0 on sky pixels"""
        W, H = self.W, self.H
        lab, sky = self.labels(frame)
        yy, xx = np.mgrid[0:H, 0:W]
        d = 0.95 + 0.006 * lab + self.depth_slopes[lab, 0] * (xx - W / 2) + self.depth_slopes[lab, 1] * (yy - H / 2)
        d = np.clip(d, 0.5, 0.998).astype(F32)
        if self.thresholds:
            t = self._patch(8, 0.25)
            d[t & (xx % 3 == 0)] = 1.0
            d[t & (xx % 3 == 1)] = np.nextafter(F32(1), F32(0))
        d[sky | (self.gbuffers(frame)[abi.BUF_GBUFFER0][..., 0] == SKY)] = 1.0
        return d

    def variance_moments(self, frame, moments: np.ndarray) -> np.ndarray:
        """with thresholds, sample counts of exactly 4 and 3 in a patch of the moments plane the variance pass reads"""
        if not self.thresholds:
            return moments
        m = moments.copy()
        t = self._patch(9, 0.3)
        yy = np.mgrid[0:self.H, 0:self.W][0]
        m[..., 2] = np.where(t, np.where(yy % 2 == 0, 4, 3) | (m[..., 2] & 0xFF000000), m[..., 2])
        return m


# ---- the systems under test ----------------------------------------------------------------------------------------------
class OracleSide:
    def __init__(self, oracle, oscene, W, H):
        self.frame = oracle.OracleFrame(oscene, W, H)
        self.svgf = oracle.OracleSvgf(self.frame)

    def _view(self, buf, idx):
        return self.frame.buffer(buf, idx, copy=False) if buf in FRAME_BUFFERS else self.svgf.buffer(buf, idx, copy=False)

    def put(self, buf, idx, arr):
        v = self._view(buf, idx)
        v[...] = np.ascontiguousarray(arr).view(v.dtype).reshape(v.shape)

    def get(self, buf, idx):
        return self._view(buf, idx).copy()

    def run(self, p, pass_id, stage):
        return self.svgf.run(p, pass_id, stage)


class DeviceSide:
    def __init__(self, ctx, W, H):
        self.ctx = ctx
        ctx.create_frame(W, H)

    def put(self, buf, idx, arr):
        self.ctx.upload(buf, idx, np.ascontiguousarray(arr))

    def get(self, buf, idx):
        return self.ctx.download(buf, idx)

    def run(self, p, pass_id, stage):
        rc = self.ctx.lib.gfx_svgf_launch(self.ctx.h, None, C.byref(p), pass_id, stage)
        return rc


def frame_passes(num_filtering_stages):
    yield abi.SVGF_TEMPORAL_ACCUMULATE, 0
    yield abi.SVGF_ESTIMATE_VARIANCE, 0
    for s in range(num_filtering_stages):
        yield abi.SVGF_ATROUS, s
    yield abi.SVGF_FILL_BACKGROUND, num_filtering_stages
    yield abi.SVGF_MODULATE_TAA, num_filtering_stages


def run_frames(sides, scene: SyntheticScene, frames: int, flags: int, hist: int, stages: int, on_pass, first_frame: int = 0):
    """frames first_frame .. first_frame + frames - 1 of `scene` on every side, pass by pass: the frame's G-buffers, beauty and
    albedo go in first, the scene's depth plane (and threshold counts) before the variance pass; on_pass(p, pass_id, stage)
    runs the pass (on every side) and checks it.  The history goes in first: from first_frame 1 on the first frame reads it (its
    counts up to 65 535), frame 0 is the first frame, which resets the counts"""
    for buf, idx, arr in scene.history(first_frame):
        for s in sides:
            s.put(buf, idx, arr)
    for f in range(first_frame, first_frame + frames):
        p = frame_params(scene.W, scene.H, f, flags, hist)
        cur = f % 2
        planes = {**scene.gbuffers(f), **scene.shading(f)}
        for buf, arr in planes.items():
            for s in sides:
                s.put(buf, cur if buf in FRAME_BUFFERS[:4] else 0, arr)
        for pass_id, stage in frame_passes(stages):
            if pass_id == abi.SVGF_ESTIMATE_VARIANCE:
                depth = scene.depth(f)
                for s in sides:
                    s.put(abi.BUF_SVGF_DEPTH, cur, depth)
                    s.put(abi.BUF_SVGF_MOMENTS, cur, scene.variance_moments(f, s.get(abi.BUF_SVGF_MOMENTS, cur)))
            on_pass(p, pass_id, stage)


# ---- the restatement alongside a system under test -----------------------------------------------------------------------
def load_all(ref, side):
    """every plane of `side` into the restatement's state (the isolation of one pass: its float32 inputs are the side's)"""
    for buf, count in ALL_PLANES:
        for idx in range(count):
            ref.load(buf, idx, side.get(buf, idx))


def ref_pass(ref, p, pass_id, stage) -> dict:
    if pass_id == abi.SVGF_TEMPORAL_ACCUMULATE:
        return ref.temporal(p)
    if pass_id == abi.SVGF_ESTIMATE_VARIANCE:
        return ref.variance(p)
    if pass_id == abi.SVGF_ATROUS:
        return ref.atrous(p, stage)
    if pass_id == abi.SVGF_FILL_BACKGROUND:
        return ref.background(p, stage)
    if pass_id == abi.SVGF_MODULATE_TAA:
        return ref.modulate_taa(p, stage)
    if pass_id == abi.SVGF_FEEDBACK_NOISY_LIGHTING:
        return ref.feedback_noisy_lighting()
    raise ValueError(pass_id)


def compare_outputs(side, ref, outs: dict, cur: int, what: str, rows=None):
    """every output of a restated pass against the side's plane, within its per-pixel bar; sample counts and accept flags
    exactly.  rows = (lo, hi) compares frame rows lo .. hi - 1 of the restatement's window only."""
    lo, hi = (ref.y0, ref.y0 + ref.rows) if rows is None else rows
    sl = slice(lo - ref.y0, hi - ref.y0)
    for name, spec in outs.items():
        if name == "info":
            want, mask = spec
            got = side.get(abi.BUF_SVGF_MOMENTS, cur)[lo:hi, :, 2]
            bad = mask[sl] & (got != want[sl])
            assert not bad.any(), f"{what}: sample info differs at {np.argwhere(bad)[:5].tolist()} " \
                                  f"(got {got[bad][:5]}, want {want[sl][bad][:5]})"
            continue
        want, bar = spec[0][sl], spec[1][sl]
        mask = spec[2][sl] if len(spec) > 2 else np.ones(want.shape[:2], bool)
        if name == "moments":
            got = side.get(abi.BUF_SVGF_MOMENTS, cur)[lo:hi, :, :2].view(F32)
        else:
            buf, idx = {"lighting0": (abi.BUF_SVGF_LIGHTING_VARIANCE, 0), "lighting1": (abi.BUF_SVGF_LIGHTING_VARIANCE, 1),
                        "prev_lighting": (abi.BUF_SVGF_PREV_LIGHTING, 0), "albedo": (abi.BUF_SVGF_ALBEDO, 0),
                        "depth": (abi.BUF_SVGF_DEPTH, cur), "final0": (abi.BUF_SVGF_FINAL, 0),
                        "final1": (abi.BUF_SVGF_FINAL, 1)}[name]
            got = side.get(buf, idx)[lo:hi]
        got = got.astype(np.float64)
        err = np.abs(got - want)
        m = mask if err.ndim == 2 else mask[..., None]
        bad = m & ~(err <= bar + TINY)
        if bad.any():
            k = tuple(np.argwhere(bad)[np.argmax(((err - bar) / np.maximum(bar, 1e-300))[bad])])
            raise AssertionError(f"{what}: {name} off its bar at {int(bad.sum())} elements; worst at {k}: got {got[k]!r}, "
                                 f"restated {want[k]!r}, bar {bar[k]!r}")
