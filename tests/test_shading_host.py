"""The shading layer every renderer shares (gfxexp_b200/csrc/shading.cuh: BSDFs, sampling warps, encoders, frames), on the
CPU, at inputs no test scene reaches: smoothness 0 to the 0.999 clamp, black / grey / white materials, REGULARIZE, view
directions on and below the shading horizon.

  (a) shading.cuh built for the CPU (tests/cpp/shading_host.cpp) equals the oracle's restatement (oracle/shading.h) bit for bit
  (b) both are float32 code; tests/shading_ref.py restates the reference in float64 and bounds their error
  (c) sampleThroughput agrees with evaluate and evaluatePDF at the direction it returns
  (d) the mean of sampleThroughput is the float64 directional albedo (what every BSDF-sampled path relies on)
  (e) sampled directions follow evaluatePDF (chi-square)
  (f) evaluate is reciprocal
  (g) evaluateDHReflectanceEstimate is its own float64 formula
  (h) outputs are finite, and the two vGiven.z == 0 cases the reference leaves non-finite or inconsistent are pinned
  (i) encoders and frames: round trips, clamping, orthonormality, ray offsets
Parity alone cannot catch a slip that the device header and the oracle share; (b)-(i) can.
"""
import numpy as np
import pytest

from tests import shading_ops as S
from tests import shading_ref as R

F32 = np.float32


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return S.build_host(tmp_path_factory.mktemp("shading_host"))


@pytest.fixture(scope="module")
def orc(oracle):
    return S.oracle_runner(oracle)


def _rel(a, b, floor):
    return np.abs(np.asarray(a, np.float64) - b) / np.maximum(np.abs(b), floor)


def _jittered(n, seed):
    """n x n stratified u with a uniform jitter in every cell: an unbiased estimator, unlike cell centres"""
    rng = np.random.default_rng(seed)
    g0, g1 = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    top = F32(1 - 2.0 ** -24)
    u0 = np.minimum(((g0.ravel() + rng.random(n * n)) / n).astype(F32), top)
    u1 = np.minimum(((g1.ravel() + rng.random(n * n)) / n).astype(F32), top)
    return u0, u1


def _off_wedge_seams(u0, u1, eps=1e-5):
    """False where |2 u0 - 1| is within eps of |2 u1 - 1|: the concentric map's bottom wedge is mirrored (see
    test_concentric_disk_bottom_wedge_is_mirrored), so float32 and float64 may land on the two sides of a seam there"""
    sx, sy = 2 * np.asarray(u0, np.float64) - 1, 2 * np.asarray(u1, np.float64) - 1
    return np.abs(np.abs(sx) - np.abs(sy)) > eps


def _sample(host, mat, cos_o, u0, u1):
    v = np.repeat(S.view_dirs((cos_o,)), len(u0), axis=0)
    return v, host(S.SAMPLE, mat, S.records(v, u0, u1))


# materials of the float64 checks: Lambert, DiffuseAndSpecular coloured and white, SimplePBR grey half-metal
def _check_materials():
    out = []
    for reg in (False, True):
        out.append(("lambert", 0, (0.5, 0.4, 0.3), (0, 0, 0), 0.0, reg))
        for s in S.SMOOTHNESS:
            out.append((f"ds-{s}", 1, (0.5, 0.4, 0.3), (0.04, 0.04, 0.04), s, reg))
            out.append((f"ds-white-{s}", 1, (1, 1, 1), (1, 1, 1), s, reg))
            out.append((f"pbr-{s}", 2, (0.5, 0.5, 0.5), (1.0, 1 - s, 0.5), 0.0, reg))
    return out


CHECK = _check_materials()


def _pair(m):
    _, t, p0, p1, p2, reg = m
    return S.material(t, p0, p1, p2, reg), R.setup(t, p0, p1, p2, reg)


# ---- (a) -------------------------------------------------------------------------------------------------------------
def test_host_build_equals_oracle_bit_for_bit(host, orc):
    for name, mat in S.materials():
        for op, rec in S.bsdf_inputs(host, mat).items():
            a, b = host(op, mat, rec), orc(op, mat, rec)
            bad = np.flatnonzero((a.view(np.uint32) != b.view(np.uint32)).any(1))
            assert bad.size == 0, f"{name} op {op}: {bad.size} records differ, first {rec[bad[0]].tolist()}"
    mat = S.material(0, 0.0)
    for op, rec in S.helper_inputs().items():
        a, b = host(op, mat, rec), orc(op, mat, rec)
        bad = np.flatnonzero((a.view(np.uint32) != b.view(np.uint32)).any(1))
        assert bad.size == 0, f"op {op}: {bad.size} records differ, first {rec[bad[0]].tolist()}"


# ---- (b) -------------------------------------------------------------------------------------------------------------
WELL_CONDITIONED_COS = (1.0, 0.7, 0.2, 1e-3, -0.5)


@pytest.mark.parametrize("m", CHECK, ids=[f"{c[0]}{'-reg' if c[5] else ''}" for c in CHECK])
def test_bsdf_float32_against_float64(host, m):
    """Given the same u, the float32 BSDF stays within (measured maxima over this grid in brackets):
    evaluate and evaluatePDF 4e-6 relative (1.1e-6), the sampled pdf 5e-4 (2.6e-4), the throughput 1e-2 (6.4e-3: the sincos and
    sqrt chains of the VNDF sampler, amplified where 1 - P1^2 - P2^2 cancels), the sampled direction 5e-5 absolute (1.1e-5).  Below cos(theta_o) = 1e-3 the GGX
    tan^2 term (1 - z^2) / z^2 loses the digits of z (evaluate's error reaches 6e-5 at 1e-6); those cells are left to (h)."""
    mat, b = _pair(m)
    u0, u1 = S.stratified(48)
    for c in WELL_CONDITIONED_COS:
        v, o = _sample(host, mat, c, u0, u1)
        v64 = v.astype(np.float64)
        t64, l64, p64 = R.sample_throughput(b, v64, u0.astype(np.float64), u1.astype(np.float64))
        ok = (o[:, 6] > 0) & (p64 > 0) & _off_wedge_seams(u0, u1 if m[1] == 0 else np.full_like(u1, 0.3))
        assert ((o[:, 6] > 0) == (p64 > 0)).mean() > 0.99, c
        assert _rel(o[ok, 6], p64[ok], 0).max() < 5e-4, c
        assert _rel(o[ok, :3], t64[ok], 1e-3).max() < 1e-2, c
        assert np.abs(o[ok, 3:6] - l64[ok]).max() < 5e-5, c
        rec = S.records(v[ok], o[ok, 3:6])
        ev, pe = host(S.EVALUATE, mat, rec)[:, :3], host(S.EVALUATE_PDF, mat, rec)[:, 0]
        l32 = o[ok, 3:6].astype(np.float64)
        ev64, pe64 = R.evaluate(b, v64[ok], l32), R.evaluate_pdf(b, v64[ok], l32)
        fin = np.isfinite(ev64).all(1) & np.isfinite(pe64)
        assert fin.all(), c
        assert _rel(ev[fin], ev64[fin], 1e-6).max() < 4e-6, c
        assert _rel(pe[fin], pe64[fin], 1e-6).max() < 4e-6, c


def test_warps_float32_against_float64(host):
    mat = S.material(0, 0.0)
    u = S.u_pairs(4096)
    u = u[_off_wedge_seams(u[:, 0], u[:, 1])]
    d = host(S.CONCENTRIC_DISK, mat, S.records(u))
    x, y = R.concentric_sample_disk(u[:, 0].astype(np.float64), u[:, 1].astype(np.float64))
    assert np.abs(d[:, 0] - x).max() < 5e-7 and np.abs(d[:, 1] - y).max() < 5e-7     # measured 2.4e-7
    h = host(S.COSINE_HEMISPHERE, mat, S.records(u))
    h64 = R.cosine_sample_hemisphere(u[:, 0].astype(np.float64), u[:, 1].astype(np.float64))
    # z = sqrt(1 - r^2) amplifies the disk's error near the rim (r -> 1); elsewhere a few ulps
    assert np.abs(h[:, :3] - h64).max() < 1e-3
    inner = h64[:, 2] > 0.1
    assert np.abs(h[inner, :3] - h64[inner]).max() < 2e-6
    assert (h[:, 2] >= 0).all()


def test_concentric_disk_bottom_wedge_is_mirrored(host):
    """concentricSampleDisk's bottom wedge (sy < -|sx|) uses theta = 6 + sx / sy (common_device.cuh:306-309), where the
    Shirley-Chiu map has 6 - sx / sy: the wedge is mirrored left to right.  It still maps onto the same angular sector with
    the same area, so the density stays uniform (cosine-weighted after the lift) and no estimator is biased, but the map
    is discontinuous on the wedge's two seams: at sx = -sy > 0 the first wedge gives angle -pi/4, the bottom one 5 pi/4."""
    mat = S.material(0, 0.0)
    e = 2.0 ** -20
    u = np.array([[0.75, 0.25 + e], [0.75, 0.25 - e], [0.5, 0.1], [0.55, 0.1], [0.45, 0.1]], dtype=F32)
    d = host(S.CONCENTRIC_DISK, mat, S.records(u))[:, :2]
    assert d[0, 0] > 0.35 and d[0, 1] < -0.35          # first wedge, just above the seam: angle ~ -pi/4
    assert d[1, 0] < -0.35 and d[1, 1] < -0.35         # bottom wedge, just below it: angle ~ 5 pi/4
    assert abs(d[2, 0]) < 1e-7 and d[2, 1] < 0         # the wedge's centre line still maps to -y
    assert d[3, 0] < 0 < d[4, 0]                       # and sx > 0 lands at x < 0: mirrored
    # uniform density on the disk all the same: equal-area rings and sectors get equal counts
    rng = np.random.default_rng(2)
    uu = rng.random((200000, 2), dtype=np.float32)
    dd = host(S.CONCENTRIC_DISK, mat, S.records(uu))[:, :2].astype(np.float64)
    ring = np.minimum((np.sum(dd ** 2, 1) * 8).astype(int), 7)
    sector = np.minimum((np.mod(np.arctan2(dd[:, 1], dd[:, 0]), 2 * np.pi) / (2 * np.pi) * 8).astype(int), 7)
    hist = np.zeros((8, 8))
    np.add.at(hist, (ring, sector), 1)
    expect = len(uu) / 64
    assert ((hist - expect) ** 2 / expect).sum() / 64 < 1.5


# ---- (c) -------------------------------------------------------------------------------------------------------------
NEAR_MIRROR = (0.99, 0.999, 1.0)


@pytest.mark.parametrize("m", CHECK, ids=[f"{c[0]}{'-reg' if c[5] else ''}" for c in CHECK])
def test_sampling_consistency(host, m):
    """Throughput == evaluate cos / pdf, and the returned pdf == evaluatePDF at the returned direction, to 1e-4 relative.

    Near a mirror (smoothness >= 0.99 unregularised: alpha <= 1e-4) evaluatePDF rebuilds the half vector from the reflected
    direction, normalize(l + v), and in float32 that half vector is off by ~1e-7 rad: a fraction of a lobe alpha = 1e-4 wide
    in half-vector slope.  D(h) then differs from the D the sampler used; the pdfs disagree although both follow the
    reference's lines (common_device.cuh:586-589, 699-729).  The throughput is computed with the sampler's own D and pdf, so
    (d) shows it stays unbiased.  Those cells assert the measured disagreement instead of the tight bar."""
    mat, b = _pair(m)
    _, t, _, p1, s, reg = m
    smooth = (1 - p1[1]) if t == 2 else s
    mirror = t != 0 and not reg and smooth >= 0.99
    u0, u1 = S.stratified(64)
    for c in (1.0, 0.7, 0.2, 1e-3, -0.5):
        v, o = _sample(host, mat, c, u0, u1)
        ok = o[:, 6] > 0
        rec = S.records(v[ok], o[ok, 3:6])
        pe = host(S.EVALUATE_PDF, mat, rec)[:, 0]
        ev = host(S.EVALUATE, mat, rec)[:, :3]
        rel_pdf = _rel(pe, o[ok, 6], 0)
        thr = ev.astype(np.float64) * np.abs(o[ok, 5:6]) / o[ok, 6:7]
        rel_thr = _rel(thr, o[ok, :3], 1e-6)
        if not mirror and c == 1e-3 and t != 0:
            # grazing: the same half-vector rebuild, milder for wider lobes (measured 3.1e-2 at smoothness 0.9)
            assert rel_pdf.max() < 0.1 and rel_thr.max() < 0.1, (c, rel_pdf.max(), rel_thr.max())
        elif not mirror or c == 1.0:
            # at normal incidence the reflected half vector is the sampled one to the last bit for alpha this small
            assert rel_pdf.max() < 1e-4 and rel_thr.max() < 1e-4, (c, rel_pdf.max(), rel_thr.max())
        elif c in (0.7, 0.2, -0.5):
            frac = (rel_pdf > 1e-4).mean()
            assert 0.02 < frac < 0.95, (c, frac)          # measured 0.05 .. 0.70 over these cells
            assert rel_pdf.max() < 1.0, (c, rel_pdf.max())  # within a factor of 2 away from grazing
        else:  # cos 1e-3: grazing as well as near-mirror; nearly every sample disagrees, by orders of magnitude
            assert (rel_pdf > 1e-4).mean() > 0.9


def test_near_mirror_pdf_disagreement_counts(host):
    """The counts the float32 half-vector rebuild produces with diffuse (0.5, 0.4, 0.3), F0 0.04 and 256 x 256 cell-centred
    u (the regime of the test above, at full size)."""
    u0, u1 = S.stratified(256)
    counts = {}
    for s, c in ((0.99, 0.2), (0.99, 1e-3), (0.999, 0.2), (0.5, 0.2), (0.5, 0.7)):
        mat = S.material(1, (0.5, 0.4, 0.3), (0.04,) * 3, s)
        v, o = _sample(host, mat, c, u0, u1)
        ok = o[:, 6] > 0
        pe = host(S.EVALUATE_PDF, mat, S.records(v[ok], o[ok, 3:6]))[:, 0]
        r = _rel(pe, o[ok, 6], 0)
        counts[(s, c)] = (int((r > 1e-4).sum()), int((r > 0.1).sum()), int(ok.sum()))
    assert counts[(0.99, 0.2)][0] > 30000                              # of 65 536
    assert counts[(0.99, 1e-3)][1] > 20000                             # > 10 % off, of ~65 400 valid samples
    assert counts[(0.999, 0.2)][1] > 2000
    assert counts[(0.5, 0.2)][0] == 0 and counts[(0.5, 0.7)][0] == 0    # rough lobes: no sample off by 1e-4


# ---- (d) -------------------------------------------------------------------------------------------------------------
ALBEDO_COS = (1.0, 0.7, 0.2, 0.05, 1e-3)


@pytest.mark.parametrize("m", [c for c in CHECK if not c[5] or c[0].startswith("ds-0.999")],
                         ids=lambda c: f"{c[0]}{'-reg' if c[5] else ''}")
def test_sampling_is_unbiased(host, m):
    """mean(sampleThroughput) over 128 x 128 jittered-stratified u equals the float64 albedo within 5 standard errors
    (the i.i.d. estimate, which over-states a stratified estimator's error) plus 2e-4 relative for the float32 sampler."""
    mat, b = _pair(m)
    u0, u1 = _jittered(128, 7)
    for c in ALBEDO_COS:
        _, o = _sample(host, mat, c, u0, u1)
        t = o[:, :3].astype(np.float64)
        mean, se = t.mean(0), t.std(0) / np.sqrt(len(t))
        alb = R.albedo(b, float(F32(c)))
        if c == 1e-3 and b.roughness <= 0.01 + 1e-6:
            # grazing and near-mirror: the quadrature is converged here (doubling its panels moves it by < 1e-6), so the
            # gap is the float32 sampler's alone: the reflection 2 (v.m) m - v of a view 1e-3 above the horizon loses
            # the digits of l.z, and samples whose l.z rounds to <= 0 are dropped (measured 2.5 %)
            assert np.abs(R.albedo(b, float(F32(c)), n_xi=768, n_phi=768) - alb).max() < 1e-5
            assert (np.abs(mean - alb) <= 0.03 * alb).all(), (c, mean, alb)
            continue
        assert (np.abs(mean - alb) <= 5 * se + 2e-4 * alb + 1e-7).all(), (c, mean, alb, se)


def test_black_material_at_normal_incidence_takes_the_zero_weight_branch(host):
    """Diffuse and F0 both black: at cos(theta_o) = 1 both one-sample weights are 0 (common_device.cuh:565-568), so the
    sampler returns throughput 0 and pdf 0, although the Schlick term (1 - l.h)^5 leaves an albedo > 0.  The reference's
    estimator is biased there; the callers stop the path on the zero pdf (pathtrace.cuh sampleNextDirection)."""
    u0, u1 = _jittered(64, 3)
    for s in (0.0, 0.5, 0.9):
        mat = S.material(1, (0, 0, 0), (0, 0, 0), s)
        _, o = _sample(host, mat, 1.0, u0, u1)
        assert (o[:, :3] == 0).all() and (o[:, 6] == 0).all()
        assert (R.albedo(R.setup(1, (0, 0, 0), (0, 0, 0), s), 1.0) > 0).all()
        _, o = _sample(host, mat, 0.7, u0, u1)
        assert (o[:, 6] > 0).mean() > 0.5          # away from normal incidence the weights are > 0 again


# ---- (e) -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s,c,reg", [(0.0, 0.7, False), (0.5, 0.2, False), (0.5, 1.0, False), (0.9, 0.7, True)])
def test_sample_distribution_follows_evaluate_pdf(host, s, c, reg):
    """chi-square of 262 144 sampled directions in 24 x 24 bins of (cos^2 theta, phi) against evaluatePDF integrated over
    each bin (float64, 8 x 8 midpoints per bin), in the style of test_oracle_envlight.py"""
    mat = S.material(1, (0.5, 0.4, 0.3), (0.04,) * 3, s, reg)
    b = R.setup(1, (0.5, 0.4, 0.3), (0.04,) * 3, s, reg)
    rng = np.random.default_rng(11)
    u = rng.random((1 << 18, 2), dtype=np.float32)
    v, o = _sample(host, mat, c, u[:, 0], u[:, 1])
    ok = o[:, 6] > 0
    lz = o[ok, 5].astype(np.float64)
    ph = np.mod(np.arctan2(o[ok, 4], o[ok, 3]).astype(np.float64), 2 * np.pi)
    nb, k = 24, 8
    hist = np.zeros((nb, nb))
    np.add.at(hist, (np.minimum((lz ** 2 * nb).astype(int), nb - 1), np.minimum((ph / (2 * np.pi) * nb).astype(int), nb - 1)), 1)
    g = (np.arange(nb * k) + 0.5) / (nb * k)
    c2, pp = np.meshgrid(g, g * 2 * np.pi, indexing="ij")
    ct, st = np.sqrt(c2), np.sqrt(1 - c2)
    dirs = np.stack([st * np.cos(pp), st * np.sin(pp), ct], -1).reshape(-1, 3)
    vv = np.broadcast_to(v[0].astype(np.float64), dirs.shape)
    pdf = R.evaluate_pdf(b, vv, dirs).reshape(nb * k, nb * k)
    # d(omega) = d(cos theta) dphi = d(cos^2) dphi / (2 cos theta)
    cell = pdf / (2 * ct) * (1.0 / (nb * k)) * (2 * np.pi / (nb * k))
    expect = cell.reshape(nb, k, nb, k).sum((1, 3)) * len(u)
    assert abs(expect.sum() / ok.sum() - 1) < 0.01          # evaluatePDF integrates to the fraction of valid samples
    big = expect > 20
    chi2 = ((hist[big] - expect[big]) ** 2 / expect[big]).sum() / big.sum()
    assert 0.75 < chi2 < 1.3, chi2


# ---- (f) -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [c for c in CHECK if c[0] != "lambert"], ids=lambda c: f"{c[0]}{'-reg' if c[5] else ''}")
def test_evaluate_is_reciprocal(host, m):
    """f(v, l) == f(l, v): the half vector, D, the height-correlated G and Fresnel are symmetric, and so is the product of
    the two diffuse Fresnel factors; only the rounding order differs (measured <= 1.5e-6 relative)."""
    mat, _ = _pair(m)
    d = S.sphere_dirs(4096)
    d = d[np.abs(d[:, 2]) > 1e-3]
    v, l = d[: len(d) // 2], d[len(d) // 2: 2 * (len(d) // 2)]
    l = l * np.sign(l[:, 2:3]) * np.sign(v[:, 2:3])                 # same side
    a = host(S.EVALUATE, mat, S.records(v, l))[:, :3]
    b = host(S.EVALUATE, mat, S.records(l, v))[:, :3]
    assert _rel(a, b.astype(np.float64), 1e-6).max() < 4e-6


# ---- (g) -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", CHECK, ids=[f"{c[0]}{'-reg' if c[5] else ''}" for c in CHECK])
def test_dh_reflectance_estimate_formula(host, m):
    """evaluateDHReflectanceEstimate is the reference's ad-hoc estimate (common_device.cuh:736-764), held to its own
    float64 formula (measured <= 2.4e-7 relative), not to the albedo"""
    mat, b = _pair(m)
    v = S.view_dirs()
    got = host(S.DH_REFLECTANCE, mat, S.records(v))[:, :3]
    assert _rel(got, R.dh_reflectance_estimate(b, v.astype(np.float64)), 1e-6).max() < 1e-6


# ---- (h) -------------------------------------------------------------------------------------------------------------
def test_outputs_are_finite_off_the_horizon(host):
    """Every output over the grid is finite, or the sample is rejected with pdf 0, for every vGiven.z != 0"""
    for name, mat in S.materials():
        ins = S.bsdf_inputs(host, mat)
        s = ins[S.SAMPLE]
        o = host(S.SAMPLE, mat, s)
        off = s[:, 2] != 0
        good = np.isfinite(o).all(1) | (o[:, 6] == 0)
        assert good[off].all(), (name, s[off][~good[off]][:2].tolist())
        assert (o[off, 6] >= 0).all()
        rec = ins[S.EVALUATE]
        # l == -v has no half vector: evaluatePDF has no same-side guard (:691-734) and returns NaN there
        off = (rec[:, 2] != 0) & (rec[:, 5] != 0) & ~np.all(rec[:, 0:3] == -rec[:, 3:6], axis=1)
        assert np.isfinite(host(S.EVALUATE, mat, rec)[off]).all(), name
        assert np.isfinite(host(S.EVALUATE_PDF, mat, rec)[off]).all(), name
        assert np.isfinite(host(S.DH_REFLECTANCE, mat, ins[S.DH_REFLECTANCE])).all(), name


def test_view_on_the_horizon_is_the_reference_behaviour(host):
    """vGiven.z == 0 exactly (+0 or -0):
    - DiffuseAndSpecular: ggxEvaluatePDF divides G1 |v.m| D by |v.z| = 0 (common_device.cuh:506), and G1 is 0 there
      (its own guard, :454), so every diffuse-branch sample returns a NaN pdf and throughput; specular-branch samples are
      rejected with pdf 0 (:603-606).
    - Lambert: sampleThroughput flips every sample below the horizon with a pdf > 0 (:352-357), while evaluatePDF gives 0
      for that pair (:364-369).
    The path tracers contain both: sampleNextDirection stops the path unless 0 < pdf < inf (pathtrace.cuh), and the NRC
    training filter zeroes non-finite targets (nrc_pathtrace.cu)."""
    u = S.u_pairs(512)
    for z in (0.0, -0.0):
        v = np.repeat(np.array([[np.cos(0.3), np.sin(0.3), z]], dtype=F32), len(u), axis=0)
        rec = S.records(v, u)
        for s in (0.0, 0.5, 0.99):
            mat = S.material(1, (0.5, 0.4, 0.3), (0.04,) * 3, s)
            o = host(S.SAMPLE, mat, rec)
            nan = np.isnan(o[:, 6])
            assert nan.any() and np.isnan(o[nan, :3]).all()
            assert (o[~nan, 6] == 0).all()
            # either way the caller's test (dirPDensity > 0 && isfinite) rejects the sample
            assert not ((o[:, 6] > 0) & np.isfinite(o[:, 6])).any()
        mat = S.material(0, (0.5, 0.4, 0.3))
        o = host(S.SAMPLE, mat, rec)
        assert (o[:, 5] <= 0).all() and (o[:, 6] >= 0).all() and (o[:, 6] > 0).mean() > 0.95
        pe = host(S.EVALUATE_PDF, mat, S.records(v, o[:, 3:6]))[:, 0]
        assert (pe == 0).all()


# ---- (i) -------------------------------------------------------------------------------------------------------------
def test_polar_codes(host):
    """decode(encode(v)) is within one 16-bit step of v (theta: pi / 65535, phi: 2 pi / 65535 scaled by sin theta), and
    encode(decode(q)) drifts by at most one code step in each field.  The drift is truncation: the decoded angle rounds a
    hair below the code's exact value and static_cast<uint32_t> floors it (common_device.cuh:38-39)."""
    mat = S.material(0, 0.0)
    d = S.sphere_dirs(20000)
    q = host(S.ENCODE_VECTOR, mat, S.records(d))[:, 0].view(np.uint32)
    back = host(S.DECODE_VECTOR, mat, S.records(q))[:, :3]
    ang = np.arccos(np.clip(np.sum(back.astype(np.float64) * d, 1), -1, 1))
    mid = np.abs(d[:, 1]) < 0.99
    assert ang[mid].max() < 6 * 2 * np.pi / 65535                              # measured 5.2 phi steps
    assert ang.max() < 1e-3                                                      # acos at the poles
    rng = np.random.default_rng(4)
    codes = rng.integers(0, 2 ** 32, 50000, dtype=np.uint64).astype(np.uint32)
    codes = codes[((codes >> 16) > 64) & ((codes >> 16) < 65471)]              # acos loses the theta code near the poles
    again = host(S.ENCODE_VECTOR, mat, S.records(host(S.DECODE_VECTOR, mat, S.records(codes))[:, :3]))[:, 0].view(np.uint32)
    dphi = (again & 0xFFFF).astype(np.int64) - (codes & 0xFFFF)
    dphi = (dphi + 32768) % 65536 - 32768
    dth = (again >> 16).astype(np.int64) - (codes >> 16)
    assert np.abs(dth).max() <= 1 and np.abs(dphi).max() <= 1
    assert (dphi != 0).mean() > 0.15                                             # common, not a corner case (measured 23 %)
    # the example of a phi code stepping down: (theta 7, phi 52) -> (7, 51)
    c = np.array([(7 << 16) | 52], dtype=np.uint32)
    assert host(S.ENCODE_VECTOR, mat, S.records(host(S.DECODE_VECTOR, mat, S.records(c))[:, :3]))[0, 0].view(np.uint32) == (7 << 16) | 51
    # toPolarYUp / fromPolarYUp against float64: acos is ill-conditioned at the poles (|y| -> 1)
    ph, th = host(S.TO_POLAR, mat, S.records(d))[:, :2].T
    ph64, th64 = R.to_polar_y_up(d.astype(np.float64))
    mid = np.abs(d[:, 1]) < 0.99
    assert np.abs(th - th64)[mid].max() < 1e-6 and np.abs(th - th64).max() < 1e-3
    dp = np.abs(ph - ph64)
    dp = np.minimum(dp, 2 * np.pi - dp)
    assert dp[mid].max() < 2e-6
    assert (ph >= 0).all() and (ph < F32(2 * np.pi)).all()
    p = np.stack([ph64, th64], 1).astype(F32)
    fp = host(S.FROM_POLAR, mat, S.records(p))[:, :3]
    assert np.abs(fp - R.from_polar_y_up(p[:, 0].astype(np.float64), p[:, 1].astype(np.float64))).max() < 1e-6


def test_barycentric_and_texcoord_codes(host):
    mat = S.material(0, 0.0)
    bc = np.array([0, 1, -1e-8, 1 + 1e-7, 2, -3, np.nan, np.inf, -np.inf, 0.5, 1 / 65535, 0.99999], dtype=F32)
    q = host(S.ENCODE_BARYCENTRIC, mat, S.records(bc))[:, 0].view(np.uint32)
    assert q.tolist() == [0, 65535, 0, 65535, 65535, 0, 0, 65535, 0, 32767, 1, 65534]
    codes = np.arange(65536, dtype=np.uint32)
    dec = host(S.DECODE_BARYCENTRIC, mat, S.records(codes))[:, 0]
    assert np.abs(dec - codes / 65535.0).max() < 6e-8
    assert (host(S.ENCODE_BARYCENTRIC, mat, S.records(dec))[:, 0].view(np.uint32).astype(np.int64) >= codes.astype(np.int64) - 1).all()
    # texture coordinates wrap with tc - floor(tc); -1e-8 wraps to 1 - 1e-8, which the clamp holds at 65535; NaN -> 0
    tc = np.array([[0, 1], [-1e-8, 0.25], [np.nan, 2.5], [-0.0, -1.0], [3.75, -2.25], [1 - 2 ** -24, 0.5 / 65535]], dtype=F32)
    q = host(S.ENCODE_TEXCOORDS, mat, S.records(tc))[:, 0].view(np.uint32)
    lo, hi = (q & 0xFFFF).tolist(), (q >> 16).tolist()
    assert lo == [0, 65535, 0, 0, 49151, 65534] and hi == [0, 16383, 32767, 0, 49151, 0]
    back = host(S.DECODE_TEXCOORDS, mat, S.records(q))[:, :2]
    assert np.allclose(back, R.decode_tex_coords(q), atol=6e-8)


def test_make_coordinate_system(host):
    """orthonormal to 4e-7 for normals at and near +-z, and at z = -0 (where the sign switch picks -1)"""
    mat = S.material(0, 0.0)
    n = np.concatenate([S.near_pole_normals(), S.sphere_dirs(4000)])
    o = host(S.COORDINATE_SYSTEM, mat, S.records(n)).astype(np.float64)
    t, b, nn = o[:, :3], o[:, 3:6], n.astype(np.float64)
    for x, y in ((t, b), (t, nn), (b, nn)):
        assert np.abs(np.sum(x * y, 1)).max() < 4e-7
    assert np.abs(np.linalg.norm(t, axis=1) - 1).max() < 4e-7 and np.abs(np.linalg.norm(b, axis=1) - 1).max() < 4e-7
    # right-handed: t x b = n
    assert np.abs(np.cross(t, b) - nn).max() < 4e-7
    t64, b64 = R.make_coordinate_system(nn)
    assert np.abs(t - t64).max() < 4e-7 and np.abs(b - b64).max() < 4e-7
    # z = -0 compares >= 0, so it takes the upper branch: the same frame as z = +0
    zp = host(S.COORDINATE_SYSTEM, mat, S.records(np.array([[1, 0, 0.0], [1, 0, -0.0]], dtype=F32)))
    assert np.array_equal(zp[0, :6], zp[1, :6]) and zp[1, 4] == 1.0


def test_offset_ray_origin_moves_along_the_normal(host):
    """offsetRayOrigin (Ray Tracing Gems ch. 6) always moves p to the +n side: below |p| = 1/32 by n / 65536, above by
    256 n ulps of each coordinate; +-0 and denormals take the float branch"""
    mat = S.material(0, 0.0)
    p, n = S.offset_inputs()
    o = host(S.OFFSET_RAY_ORIGIN, mat, S.records(p, n))[:, :3]
    d = o.astype(np.float64) - p
    for k in range(3):
        moved = np.abs(n[:, k]) >= 1 / 256                 # dm_f2int(256 n) != 0: the int branch moves the coordinate
        small = np.abs(p[:, k]) < 1 / 32
        assert (np.sign(d[:, k]) == np.sign(n[:, k]))[moved | (small & (n[:, k] != 0))].all(), k
        assert (np.abs(d[small, k] - n[small, k].astype(np.float64) / 65536) <= np.spacing(np.abs(o[small, k])).astype(np.float64) + 1e-44).all()
        big = ~small
        ulp = np.spacing(np.abs(p[big, k]).astype(F32)).astype(np.float64)
        steps = np.trunc(256 * n[big, k].astype(F32)).astype(np.float64)
        assert (np.abs(d[big, k]) <= 2 * np.abs(steps) * ulp + 1e-30).all(), k
    assert np.isfinite(o).all()
