"""Light sampling against its own densities and a float64 restatement (tests/light_ref.py), on the CPU oracle (no GPU).

The oracle's sampleLight (oracle/render.cpp), evaluateEnvLightOnMiss and computeSurfacePointAtHit (oracle/pathtrace.inl) restate
the reference from the same reading as the library, and the GPU tests hold the two equal bit for bit
(test_gpu_light_sampling.py).  What is checked here is that those restatements sample what the estimators divide by:
  * every light is picked, over the 2^23 values of the PCG32 lattice k 2^-23, as often as both its float32 selection probability
    (the chain's lightProb = areaPDensity / recArea) and the float64 P_t = s_i^2 lum(E) A_obj,t / sum say;
  * the sampling side's area density equals the hit side's hypAreaPDensity, which the path tracers' MIS uses;
  * triangle samples are uniform over the triangle, at the float64 position, normal and emittance;
  * the environment map's pdf is the float64 one, its samples follow it, and the miss programs' density along a sampled direction
    is the sample's own;
  * the split between environment and emitter candidates gives the environment its share and keeps the remapped ul below 1.
"""
import math

import numpy as np
import pytest

from tests import light_ref as R
from tests import light_scenes as LS

N_LATTICE = 1 << 23
EPS32 = 2.0 ** -24  # unit roundoff of float32
KEY_NONE = 0x40000000


def lattice(lo: int = 0, hi: int = N_LATTICE) -> np.ndarray:
    return (np.arange(lo, hi, dtype=np.float64) * 2.0 ** -23).astype(np.float32)


def run(osc, op, rec, **kw):
    return osc.light_sample_debug(op, np.asarray(rec, dtype=np.float32), **kw)


def pick_lattice(osc, num_lights: int, chunk: int = 1 << 21):
    """counts per light key over the whole lattice, the number of kPickNone picks, and each light's lightProb / areaPDensity"""
    counts = np.zeros(num_lights, dtype=np.int64)
    light_prob = np.full(num_lights, np.nan, dtype=np.float32)
    density = np.full(num_lights, np.nan, dtype=np.float32)
    none = 0
    for lo in range(0, N_LATTICE, chunk):
        rec = np.zeros((chunk, 3), dtype=np.float32)
        rec[:, 0] = lattice(lo, lo + chunk)
        rec[:, 1:] = 0.5
        out = run(osc, 0, rec)
        keys = out[:, 0].view(np.uint32)
        is_none = (keys & KEY_NONE) != 0
        none += int(is_none.sum())
        k = keys[~is_none].astype(np.int64)
        counts += np.bincount(k, minlength=num_lights)
        light_prob[k] = out[~is_none, 11]
        density[k] = out[~is_none, 10]
    return counts, none, light_prob, density


def level_bar(scene, em: R.Emitters) -> np.ndarray:
    """Where a light's lattice frequency may differ from its probability, per light:
      * 4 lattice points: the piece of ul that picks a light has two ends, each rounded onto the lattice, and the remap
        (u - l) / (r - l) of the nested levels moves each end by at most one more point;
      * per level (instance, geometry, primitive) P_parent 2 ulp(I_level) / I_level: the float32 exclusive scan makes each CDF
        step differ from its weight by at most ulp(I_level) at either end, and the width of a piece at a level is scaled by the
        probability of its parent."""
    w = em.weight
    inst_w = np.zeros(len(scene.instances))
    np.add.at(inst_w, em.inst, w)
    geom_key = em.inst * 4096 + em.geom
    _, gidx = np.unique(geom_key, return_inverse=True)
    geom_w = np.bincount(gidx, weights=w)
    total = w.sum()
    rel = lambda x: np.spacing(np.float32(x)).astype(np.float64) / np.maximum(x, 1e-300)  # ulp(I) / I in float32
    p_inst = inst_w[em.inst] / total
    p_geom = np.divide(geom_w[gidx], inst_w[em.inst], out=np.zeros_like(p_inst), where=inst_w[em.inst] > 0)
    return 4 * 2.0 ** -23 + 2 * rel(total) + p_inst * 2 * rel(inst_w[em.inst]) + p_inst * p_geom * 2 * rel(geom_w[gidx])


@pytest.fixture(scope="module")
def oscenes(oracle):
    cache = {}

    def get(name):
        if name not in cache:
            scene = LS.EMITTER_SCENES[name]()
            cache[name] = (scene, oracle.OracleScene(scene, build_bvh=False), R.emitters(scene))
        return cache[name]
    return get


@pytest.mark.parametrize("name", list(LS.EMITTER_SCENES))
def test_pick_frequency_equals_the_density_divided_by(oscenes, name):
    scene, osc, em = oscenes(name)
    n = em.prob.size
    counts, none, light_prob, density = pick_lattice(osc, n)
    freq = counts / N_LATTICE
    bar = level_bar(scene, em)
    reached = counts > 0
    # (a) the chain's own float32 probability, which every estimator divides by (areaPDensity = lightProb * recArea)
    da = np.abs(freq[reached] - light_prob[reached].astype(np.float64))
    assert np.all(da <= bar[reached]), f"{name}: lattice frequency vs lightProb, worst {da.max():.3g} (bar {bar[reached][da.argmax()]:.3g})"
    # ... and recArea is the WORLD-space area: areaPDensity / lightProb = 1 / A_world.  Bar: the float32 world vertices are off by
    # an ulp of |P| each, which moves |cross| by (|e1| + |e2| + |e3|) 2 ulp(|P|) relative to 2 A; the products add a few ulps
    ok = reached & (em.area_world > 0) & np.isfinite(density) & (light_prob > 0)
    ratio = density[ok].astype(np.float64) / light_prob[ok] * em.area_world[ok]
    wv = em.world[ok]
    edges = sum(np.linalg.norm(wv[:, (k + 1) % 3] - wv[:, k], axis=1) for k in range(3))
    tol = 8 * EPS32 * (1 + np.abs(wv).max(axis=(1, 2)) * edges / (2 * em.area_world[ok]))
    assert np.all(np.abs(ratio - 1) <= tol), f"{name}: recArea is not 1 / world area: {ratio.min()} .. {ratio.max()}"
    # (b) the float64 P_t
    db = np.abs(freq - em.prob)
    below_floor = em.weight < np.spacing(np.float32(em.weight.sum())) * 0.5
    assert np.all(db[~below_floor] <= bar[~below_floor]), \
        f"{name}: lattice frequency vs float64 P_t, worst {db[~below_floor].max():.3g} at light {np.flatnonzero(~below_floor)[db[~below_floor].argmax()]}"
    # every light of probability >= 2^-20 is reached (it spans >= 8 lattice points)
    assert reached[em.prob >= 2.0 ** -20].all(), f"{name}: lights of P >= 2^-20 never picked"
    # no probability mass goes to sampleLight's early outs when every instance, geometry and triangle has a positive weight
    if name != "trailing_zero_geometry" and (em.prob > 0).all() and all(i.uniform_scale > 0 for i in scene.instances):
        assert none == 0, f"{name}: {none} lattice points picked no light"
    # total variation between the lattice frequencies and P_t: bounded by the per-light bars
    tv = float(db.sum())
    assert tv <= float(bar.sum()), f"{name}: total variation {tv:.3g} > {bar.sum():.3g}"


def test_lights_below_the_float32_scan_floor_are_the_references_quirk(oscenes):
    """A triangle whose weight is below half an ulp of its mesh's primIntegral adds nothing to the float32 running sum (or a whole
    ulp), so its CDF step is 0 or a multiple of ulp(primIntegral): it is never picked, or picked on a whole lattice point or more,
    while its lightProb (weight / integral) is its true small probability.  This is the reference's scan (compute_light_probs.cu,
    ext/cubd ExclusiveSum in float32), pinned here rather than hidden by a wider bar."""
    scene, osc, em = oscenes("spread_weights")
    counts, none, light_prob, _ = pick_lattice(osc, em.prob.size)
    floor = np.spacing(np.float32(em.weight.sum()))
    below = em.weight < 0.5 * floor
    assert below.sum() > 1000, "the scene no longer puts lights below the scan's floor"
    unreached = below & (counts == 0)
    assert unreached.sum() > 0.9 * below.sum(), f"only {unreached.sum()} of {below.sum()} sub-floor lights are never picked"
    # the estimators' bias is the unpicked lights' summed probability (2e-4 of the power in this scene): at most half an ulp of
    # the integral per sub-floor light, and not 0 - the quirk is real
    lost = em.prob[unreached].sum()
    assert 1e-5 < lost <= below.sum() * 0.5 * floor / em.weight.sum(), lost
    assert none == 0


@pytest.mark.parametrize("name", ["single_triangle", "scaled_instances"])
def test_triangle_samples(oscenes, name):
    """(u0, u1) on a 1024^2 lattice through squareToTriangle: position, normal and emittance against float64; the samples are
    uniform over 256 equal-area sub-triangles (chi-square)."""
    scene, osc, em = oscenes(name)
    light = int(np.flatnonzero(em.area_world > 0)[0])
    ul = np.float32(np.cumsum(em.prob)[light] - 0.5 * em.prob[light])  # inside the light's piece
    g = (np.arange(1024, dtype=np.float64) + 0.5) / 1024
    u0, u1 = [x.reshape(-1).astype(np.float32) for x in np.meshgrid(g, g, indexing="ij")]
    rec = np.stack([np.full_like(u0, ul), u0, u1], axis=1)
    out = run(osc, 0, rec)
    assert np.all(out[:, 0].view(np.uint32) == light)
    a, b, c = R.square_to_triangle(u0, u1)
    wv = em.world[light]
    pos64 = a[:, None] * wv[0] + b[:, None] * wv[1] + c[:, None] * wv[2]
    # barycentrics in float32 are exact to 2^-24 (a halving and one addition); positions: that, plus the float32 vertices and sum
    tol = 2.0 ** -24 * 3 * np.abs(wv).max() + 8 * EPS32 * np.abs(pos64).max(axis=1)
    assert np.all(np.abs(out[:, 1:4] - pos64).max(axis=1) <= tol)
    n64 = (a[:, None] * em.normals[light][0] + b[:, None] * em.normals[light][1] + c[:, None] * em.normals[light][2]) @ em.normal_matrix[light].T
    n64 /= np.linalg.norm(n64, axis=1, keepdims=True)
    assert np.abs(out[:, 4:7] - n64).max() <= 1e-6
    assert np.all(out[:, 7:10] == em.emittance[light].astype(np.float32))
    # uniformity: barycentric grid of 16 x 16 cells, each split into 2 triangles -> 256 equal-area sub-triangles
    fa, fb = a * 16, b * 16
    ia, ib = np.minimum(np.floor(fa), 15).astype(int), np.minimum(np.floor(fb), 15).astype(int)
    upper = (fa - ia) + (fb - ib) > 1
    valid = ia + ib < 16
    cell = (ia + ib * 16) * 2 + upper
    cnt = np.bincount(cell[valid], minlength=512)
    occupied = cnt[np.unique(cell[valid])]
    assert occupied.size == 256, occupied.size
    exp = u0.size / 256
    chi2 = float(((occupied - exp) ** 2 / exp).sum())
    assert chi2 < 255 + 5 * math.sqrt(2 * 255), chi2


@pytest.mark.parametrize("name", list(LS.EMITTER_SCENES))
def test_sampling_side_equals_hit_side(oscenes, name):
    """sampleLight's areaPDensity (op 0) against computeSurfacePointAtHit's hypAreaPDensity (op 5) for every light, and both
    against the float64 P_t / A_world,t.  Bars: the two float32 evaluations divide the same weights by the same integrals in a
    different order (a few ulps: 1e-5); the float64 bar adds the float32 scans' accumulated rounding, (number of summands) eps."""
    scene, osc, em = oscenes(name)
    # one lattice point of every light the lattice reaches
    pick = np.full(em.prob.size, np.nan, dtype=np.float32)
    for lo in range(0, N_LATTICE, 1 << 21):
        ul = lattice(lo, lo + (1 << 21))
        keys = run(osc, 0, ul[:, None])[:, 0].view(np.uint32)
        live = (keys & KEY_NONE) == 0
        k, first = np.unique(keys[live], return_index=True)
        pick[k] = ul[live][first]
    take = np.flatnonzero(np.isfinite(pick))
    take = take[np.linspace(0, take.size - 1, min(take.size, 20000)).astype(int)]
    rec = np.zeros((take.size, 3), dtype=np.float32)
    rec[:, 0] = pick[take]
    rec[:, 1:] = 0.25
    s_out = run(osc, 0, rec)
    assert np.all(s_out[:, 0].view(np.uint32) == take)
    h_rec = np.zeros((take.size, 5), dtype=np.float32)
    h_rec[:, 0] = em.inst[take].astype(np.uint32).view(np.float32)
    h_rec[:, 1] = em.geom[take].astype(np.uint32).view(np.float32)
    h_rec[:, 2] = em.prim[take].astype(np.uint32).view(np.float32)
    h_rec[:, 3:5] = 1.0 / 3.0
    h_out = run(osc, 5, h_rec)
    ds, dh = s_out[:, 10].astype(np.float64), h_out[:, 0].astype(np.float64)
    fin = np.isfinite(ds) & (ds > 0)
    assert np.array_equal(fin, np.isfinite(dh) & (dh > 0)), f"{name}: one side finite and positive, the other not"
    assert np.all(np.abs(ds[fin] / dh[fin] - 1) <= 1e-5), f"{name}: sampling vs hit side {np.abs(ds[fin] / dh[fin] - 1).max():.3g}"
    terms = len(scene.instances) + max(m.triangles.shape[0] for m in scene.meshes) + 8
    rel = np.abs(ds[fin] / em.density[take][fin] - 1)
    assert np.all(rel <= terms * EPS32 * 4 + 1e-5), f"{name}: vs float64 density {rel.max():.3g}"


def test_trailing_zero_geometry_is_never_picked(oscenes):
    scene, osc, em = oscenes("trailing_zero_geometry")
    counts, none, _, _ = pick_lattice(osc, em.prob.size)
    assert np.all(counts[em.prob == 0] == 0) and none == 0


# ---- environment map ------------------------------------------------------------------------------------------------------------
def _env_scene(oracle, kind):
    scene = LS.single_triangle()
    scene.env_map = LS.env_map(kind)
    return scene, oracle.OracleScene(scene, build_bvh=False)


@pytest.mark.parametrize("kind", LS.ENV_KINDS)
def test_env_pdf_equals_float64(oracle, kind):
    """evaluatePDF at every texel centre against the float64 texel pdf: float32 sums of W and H terms (Kahan-compensated) and two
    divisions: 1e-5 relative.  Black rows and a black map give 0, never NaN."""
    scene, osc = _env_scene(oracle, kind)
    h, w = scene.env_map.shape[:2]
    v, u = np.meshgrid((np.arange(h) + 0.5) / h, (np.arange(w) + 0.5) / w, indexing="ij")
    pdf = osc.env_query(1, np.stack([u.ravel(), v.ravel()], 1))[:, 0].reshape(h, w)
    want = R.env_pdf(scene.env_map)
    assert np.isfinite(pdf).all(), f"{kind}: non-finite pdf at {np.argwhere(~np.isfinite(pdf))[:4].tolist()}"
    np.testing.assert_allclose(pdf, want, rtol=1e-5, atol=1e-6 * max(want.max(), 1e-30))


def _env_samples(osc, n_side):
    """n_side^2 independent uniform (u0, u1): a grid would quantise each texel's count to whole grid lines"""
    u = np.random.default_rng(n_side).random((n_side * n_side, 2), dtype=np.float32)
    return u, osc.env_query(0, u)


@pytest.mark.parametrize("kind", [k for k in LS.ENV_KINDS if k != "black"])
def test_env_samples_follow_their_pdf(oracle, kind):
    """2048^2 random (u0, u1): each sample's uvPDF is evaluatePDF at the sample except on texel seams (where the float (u, v)
    rounds onto the next texel: pinned below 0.1 %), no sample lands on a texel of pdf 0 (black rows included), and the texel
    histogram passes a chi-square against the pdf."""
    scene, osc = _env_scene(oracle, kind)
    h, w = scene.env_map.shape[:2]
    u, smp = _env_samples(osc, 2048)
    assert np.isfinite(smp).all()
    assert np.all((smp[:, :2] >= 0) & (smp[:, :2] < 1))
    ev = osc.env_query(1, smp[:, :2])[:, 0]
    mismatch = ev != smp[:, 2]
    assert mismatch.mean() < 1e-3, f"{kind}: {mismatch.mean():.2%} of the samples' uvPDF differ from evaluatePDF"
    pdf = R.env_pdf(scene.env_map)
    tx = np.minimum((smp[:, 0] * w).astype(int), w - 1)
    ty = np.minimum((smp[:, 1] * h).astype(int), h - 1)
    assert np.all(smp[~mismatch, 2] > 0), f"{kind}: samples of pdf 0"
    cnt = np.bincount(ty * w + tx, minlength=w * h).astype(np.float64)
    exp = u.shape[0] * pdf.ravel() / (w * h)
    live = exp > 0
    assert cnt[~live].sum() <= mismatch.sum(), f"{kind}: {cnt[~live].sum()} samples on zero-pdf texels"
    if live.sum() > 1:
        dof = live.sum() - 1
        chi2 = float(((cnt[live] - exp[live]) ** 2 / np.maximum(exp[live], 1)).sum())
        assert chi2 < dof + 5 * math.sqrt(2 * dof) + 10, f"{kind}: chi-square {chi2:.1f}, dof {dof}"


@pytest.mark.parametrize("rotation", [0.0, 0.7, -3.0, float(np.float32(2 * np.pi) - np.float32(1e-6)), 10.0])
@pytest.mark.parametrize("kind", ["37x19", "black_rows"])
def test_env_direction_and_miss_density(oracle, kind, rotation):
    """sampleEnvLight's direction against float64 fromPolarYUp(2 pi u - rotation wrapped, pi v): float32 sin / cos of angles up
    to 2 pi (and the wrap of a rotation up to 10): 2e-5.  The miss programs' density along the sampled direction with
    probToSampleEnv = 1 (op 4) is the sample's areaPDensity: MIS weighs both strategies with the same density.  The round trip
    direction -> (u, v) lands on the neighbouring texel within float32 of a texel edge: those are counted and pinned."""
    scene, osc = _env_scene(oracle, kind)
    u, smp = _env_samples(osc, 256)
    out = run(osc, 3, u, env_rotation=rotation, enable_env=True)
    d = out[:, 0:3].astype(np.float64)
    want = R.env_direction(smp[:, 0], smp[:, 1], rotation)
    assert np.abs(d - want).max() <= 2e-5, f"direction vs float64: {np.abs(d - want).max():.3g}"
    dens = out[:, 3]
    live = dens > 0
    assert np.isfinite(dens).all() and live.mean() > 0.99
    np.testing.assert_allclose(dens[live], R.env_solid_angle_density(smp[live, 2], smp[live, 1]), rtol=1e-4)
    miss = run(osc, 4, np.concatenate([out[:, 0:3], np.ones((u.shape[0], 2), np.float32)], 1), env_rotation=rotation, enable_env=True)
    # a sample within float32 of a pole (v ~ 2e-5) has a positive density, but its direction rounds to (0, 1, 0), where the miss
    # side's sin(theta) is 0 and its density infinite: the reference's own quirk, pinned at below 1e-4 of the samples
    assert (~np.isfinite(miss[live, 0])).mean() < 1e-4
    same = np.abs(miss[live, 0] / dens[live] - 1) <= 1e-4
    assert same.mean() > 0.99, f"miss-side density differs from the sample's on {1 - same.mean():.2%} of the samples"


def test_black_rows_give_zero_density_and_mis_weight_one(oracle):
    """The defect the fix removes: with a black ground the miss program's density was 0 / 0 = NaN for every direction in those
    rows, and with it the MIS weight and the pixel.  Now the density is 0 and the MIS weight 1."""
    scene = LS.sky_with_black_ground()
    osc = oracle.OracleScene(scene, build_bvh=False)
    assert osc.env_query(1, np.array([[0.5, 0.9]], np.float32))[0, 0] == 0.0
    dirs = R.from_polar_y_up(np.linspace(0.1, 6.2, 64), np.full(64, 0.9 * np.pi)).astype(np.float32)
    rec = np.concatenate([dirs, np.full((64, 1), 0.3, np.float32), np.full((64, 1), 0.25, np.float32)], 1)
    out = run(osc, 4, rec, enable_env=True)
    assert np.all(out[:, 0] == 0.0) and np.all(out[:, 1] == 1.0), out[:4, :2]


def test_black_map_is_no_light(oracle):
    """A map that is black everywhere has nothing to sample: the environment counts as disabled, so no candidate or NEE sample
    is spent on it and no estimator divides by its density 0."""
    scene, osc = _env_scene(oracle, "black")
    rec = np.stack([np.zeros(4), np.full(4, 32), np.linspace(0, 0.9, 4)], 1).astype(np.float32)
    rec[:, :2] = rec[:, :2].astype(np.uint32).view(np.float32)
    assert np.all(run(osc, 6, rec, enable_env=True)[:, 0] == 0)
    assert np.all(run(osc, 7, rec[:, 2:], enable_env=True)[:, 0] == 0)
    h_rec = np.zeros((1, 5), np.float32)
    h_rec[:, 3:] = 1 / 3
    with_env = run(osc, 5, h_rec, enable_env=True)[0, 0]
    without = run(osc, 5, h_rec, enable_env=False)[0, 0]
    assert with_env == without > 0  # no (1 - probToSampleEnvLight) factor for a light nobody samples


def test_nan_texel_is_refused(oracle):
    scene = LS.single_triangle()
    scene.env_map = LS.env_map("37x19")
    scene.env_map[3, 4, 1] = np.nan
    with pytest.raises(ValueError):
        oracle.OracleScene(scene, build_bvh=False)


# ---- environment / emitter split ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [32, 30])
def test_candidate_split(oracle, n):
    """chooseEnvForCandidate over the lattice plus the 2^20 largest floats below 1: the remapped ul stays in [0, 1) (the flattened
    pick's domain ends at the largest float below 1; an ul of 1.0 would take the last guide bucket), and over the lattice the
    environment gets 0.25 n of the n candidates (n = 30: candidate 7 is split half and half).  The candidates whose split is
    fractional run on the whole lattice; the others (all or nothing, remapped by a division by 1) on every 64th lattice point."""
    scene, osc = _env_scene(oracle, "37x19")
    top = np.arange(0x3F800000 - (1 << 20), 0x3F800000, dtype=np.uint32).view(np.float32)
    env_total = 0.0
    for i in range(n):
        fractional = 0 < 0.25 * n - i < 1
        lat = lattice() if fractional else lattice()[::64]
        ul = np.concatenate([lat, top])
        rec = np.zeros((ul.size, 3), np.float32)
        rec[:, 0] = np.uint32(i).view(np.float32)
        rec[:, 1] = np.uint32(n).view(np.float32)
        rec[:, 2] = ul
        out = run(osc, 6, rec, enable_env=True)
        remapped = out[:, 1]
        assert np.all((remapped >= 0) & (remapped < 1)), f"candidate {i}: remapped ul {remapped.max()!r}"
        assert np.all(out[:, 2] == np.where(out[:, 0] > 0, 0.25, 0.75))
        env_total += float(out[:lat.size, 0].mean())
    assert abs(env_total - 0.25 * n) <= n * 2.0 ** -23, env_total


def test_nee_split(oracle):
    scene, osc = _env_scene(oracle, "37x19")
    top = np.arange(0x3F800000 - (1 << 20), 0x3F800000, dtype=np.uint32).view(np.float32)
    ul = np.concatenate([lattice(), top])
    out = run(osc, 7, ul[:, None], enable_env=True)
    assert np.all((out[:, 1] >= 0) & (out[:, 1] < 1)), out[:, 1].max()
    assert out[:N_LATTICE, 0].mean() == 0.25
