"""The oracle's G-buffer pass (oracle/render.cpp, and its copies in oracle/bump.cpp and oracle/svgf_taa_jitter.cpp) against
the float64 restatement of tests/gbuffer_ref.py, plane by plane, on the seeded scenes of tests/gbuffer_scenes.py: frame sizes
from 1x1, strips, every jitter, the bump, the textured city and two animated frames, with at most 1 % of pixels steered.  And
closed-form checks that need no restatement: hit points project back to their samples, a static frame's motion under
enableJittering is (0.5 - jx, 0.5 - jy), a miss pixel's motion under a translating camera, and the running means."""
import numpy as np
import pytest

from gfxexp_b200 import abi, scenes
from tests import gbuffer_ref as R, gbuffer_scenes as S, oracle_bump, oracle_lib, oracle_svgf_taa_jitter

PLANES = (abi.BUF_GBUFFER0, abi.BUF_GBUFFER1, abi.BUF_GBUFFER2, abi.BUF_GBUFFER3, abi.BUF_ALBEDO_ACCUM, abi.BUF_NORMAL_ACCUM,
          abi.BUF_RNG)
SIZES = [(1, 1), (7, 3), (13, 7), (67, 45)]
SENTINEL = 0xA5A5A5A5


def planes_of(frame):
    return {b: frame.buffer(b, 0) for b in PLANES}


def check(ref, planes, what, accum_prev=None, num_accum_frames=0, max_steered=0.01):
    bad = R.mismatches(ref, planes, accum_prev, num_accum_frames)
    assert not any(v.any() for v in bad.values()), f"{what}: {R.report(bad, ref)}"
    assert ref.steered.sum() <= max_steered * len(ref.pix), f"{what}: {int(ref.steered.sum())} of {len(ref.pix)} pixels steered"
    return int(ref.steered.sum())


def frame_params(sc, W, H, prev_k=-1.0):
    """frame 0 of the scene, its previous camera one step back along moved_camera"""
    p = abi.default_frame_params(sc, W, H)
    p.resetFlowBuffer = 0
    p.prevCamera = S.moved_camera(sc, W, H, prev_k)
    p.envLightRotation = 3.0   # the sky in view has phi in about [2.5, 3.8]: u = (phi + rotation) / 2 pi wraps inside it
    return p


@pytest.fixture(scope="module")
def plain():
    sc = S.scene()
    return sc, R.Scene64(sc), oracle_lib.OracleScene(sc)


@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_gbuffer_equals_restatement(plain, size):
    sc, s64, osc = plain
    W, H = size
    f = oracle_lib.OracleFrame(osc, W, H)
    p = frame_params(sc, W, H)
    f.gbuffer(p)
    ref = R.gbuffer(s64, p, W, H)
    check(ref, planes_of(f), f"{W}x{H}")
    if W * H > 1000:   # the scene's edge cases are all in view: sky, every instance, the NaN tangent, the fallback normal
        assert (~ref.hit).sum() > 0.1 * W * H
        assert set(np.unique(ref.ids[ref.hit, 0]).tolist()) == set(range(len(sc.instances)))
        assert (~np.isfinite(ref.tangent).all(1)).any()


@pytest.mark.parametrize("strip", [(3, 6), (11, 40), (0, 5), (22, 1)], ids=lambda s: f"{s[0]}+{s[1]}")
def test_strips_keep_other_rows(plain, strip):
    """tileOriginY not a multiple of 8 and tileRows past H: the strip equals the restatement, the other rows keep their bits"""
    sc, s64, osc = plain
    W, H = 29, 23
    f = oracle_lib.OracleFrame(osc, W, H)
    for b in PLANES:
        f.buffer(b, 0, copy=False).view(np.uint32)[...] = SENTINEL
    p = frame_params(sc, W, H)
    p.tileOriginY, p.tileRows = strip
    f.gbuffer(p)
    planes = planes_of(f)
    check(R.gbuffer(s64, p, W, H), planes, f"strip {strip}")
    y1 = min(H, strip[0] + strip[1])
    for b in PLANES:
        v = planes[b].view(np.uint32)
        assert (v[:strip[0]] == SENTINEL).all() and (v[y1:] == SENTINEL).all(), b


def test_enable_jittering(plain):
    """two PCG32 draws per pixel, the states written back; the motion vector still from the pixel centre"""
    sc, s64, osc = plain
    W, H = 31, 19
    f = oracle_lib.OracleFrame(osc, W, H, seed=12345)
    p = frame_params(sc, W, H)
    p.enableJittering = 1
    for frame in range(2):
        rng_in = f.buffer(abi.BUF_RNG, 0)
        f.gbuffer(p)
        ref = R.gbuffer(s64, p, W, H, rng_in=rng_in)
        check(ref, planes_of(f), f"jitter frame {frame}")


@pytest.mark.parametrize("history,frame_index", [(16, 5), (16, 16 + 11), (4, 6), (0, 3)])
def test_svgf_taa_jitter(history, frame_index):
    """GFX_SVGF_SUBPIXEL_JITTER: the ray through (halton(2, i), 1 - halton(3, i)), i = frameIndex % history (0 = 16), the motion
    vector from that sample"""
    sc = S.scene()
    W, H = 27, 17
    f = oracle_svgf_taa_jitter.Frame(sc, W, H)
    p = frame_params(sc, W, H)
    p.svgfFlags = abi.SVGF_ENABLE_TAA | abi.SVGF_SUBPIXEL_JITTER
    p.taaHistoryLength, p.frameIndex = history, frame_index
    f.gbuffer(p)
    ref = R.gbuffer(R.Scene64(sc), p, W, H)
    assert R.taa_sample(p) is not None
    check(ref, planes_of(f), f"TAA {history} {frame_index}")


def test_bump_mapping():
    sc = S.scene(bump=True)
    W, H = 53, 37
    f = oracle_bump.OracleFrame(oracle_bump.OracleScene(sc), W, H)
    p = frame_params(sc, W, H)
    p.enableBumpMapping = 1
    f.gbuffer(p)
    ref = R.gbuffer(R.Scene64(sc), p, W, H, bump=True)
    check(ref, planes_of(f), "bump")


def test_textured_city():
    sc = scenes.small_city_scene_textured()
    W, H = 24, 14
    f = oracle_lib.OracleFrame(oracle_lib.OracleScene(sc), W, H)
    p = abi.default_frame_params(sc, W, H)
    p.resetFlowBuffer = 0
    f.gbuffer(p)
    check(R.gbuffer(R.Scene64(sc), p, W, H), planes_of(f), "textured city")


def _animated(sc, osc, W, H, f):
    """frame 0, then frame 1 with moved instances (and a NaN curToPrev on the zero-normal quad) and a moved camera"""
    p0 = frame_params(sc, W, H)
    f.gbuffer(p0)
    moved = S.moved_instances(sc)
    moved[S.I_ZERO_N] = scenes.Instance(moved[S.I_ZERO_N].transform, np.full((3, 4), np.nan, np.float32),
                                        moved[S.I_ZERO_N].normal_matrix, 1.0, moved[S.I_ZERO_N].mesh_slots)
    osc.update_instances(abi.make_instance_descs(moved))
    sc1 = scenes.Scene(sc.meshes, sc.materials, moved, sc.camera_position, sc.camera_orientation, sc.fov_y)
    sc1.textures, sc1.material_textures = sc.textures, sc.material_textures
    p1 = abi.default_frame_params(sc, W, H)
    p1.resetFlowBuffer = 0
    p1.prevCamera = p0.camera
    p1.camera = S.moved_camera(sc, W, H)
    p1.frameIndex, p1.bufferIndex = 1, 1
    p1.envLightRotation = -3.5  # phi + rotation < 0 over part of the sky
    return sc1, moved, p1


def test_two_animated_frames():
    sc = S.scene()
    osc = oracle_lib.OracleScene(sc)
    W, H = 61, 41
    f = oracle_lib.OracleFrame(osc, W, H)
    sc1, moved, p1 = _animated(sc, osc, W, H, f)
    s64 = R.Scene64(sc1, prev_instances=sc.instances)
    f.gbuffer(p1)
    planes = {b: f.buffer(b, 1 if b < abi.BUF_RNG else 0) for b in PLANES}
    ref = R.gbuffer(s64, p1, W, H)
    check(ref, planes, "frame 1")
    # the moved instances are in view and move; the NaN previous position gives no motion
    for k in S.MOVED:
        sel = ref.hit & (ref.ids[:, 0] == k) & ~ref.steered
        assert sel.sum() > 5 and np.abs(ref.motion[sel] - ref.motion_obj[sel]).max() < 1e-3
    nanp = ref.hit & (ref.ids[:, 0] == S.I_ZERO_N)
    assert nanp.any() and (planes[abi.BUF_GBUFFER1].reshape(-1, 2)[ref.pix[nanp]] == 0).all()
    p1.resetFlowBuffer = 1
    f.gbuffer(p1)
    assert (f.buffer(abi.BUF_GBUFFER1, 1) == 0).all()


# ---- closed forms -----------------------------------------------------------------------------------------------------
def test_hit_points_project_to_their_samples(plain):
    """calcScreenPosition with the *current* camera returns each hit point's sample, jittered or not"""
    sc, s64, osc = plain
    W, H = 40, 30
    f = oracle_lib.OracleFrame(osc, W, H, seed=99)
    p = frame_params(sc, W, H)
    for jitter in (0, 1):
        p.enableJittering = jitter
        rng_in = f.buffer(abi.BUF_RNG, 0)
        f.gbuffer(p)
        ref = R.gbuffer(s64, p, W, H, rng_in=rng_in)
        gb2 = f.buffer(abi.BUF_GBUFFER2, 0).reshape(-1, 4)
        sel = ref.hit & ~ref.steered
        P = gb2[ref.pix[sel], :3].view(np.float32).astype(np.float64)
        cam = R.Camera64.of(p.camera)
        got = cam.screen_position(P) * [W, H]
        xs, ys = ref.pix[sel] % W, ref.pix[sel] // W
        if jitter:
            st = rng_in.reshape(-1)[ref.pix[sel]]
            st, jx = R.restir_ref.pcg_draw(st)
            _, jy = R.restir_ref.pcg_draw(st)
        else:
            jx = jy = 0.5
        want = np.stack([xs + jx, ys + jy], 1)
        bar = cam.screen_jacobian_bar(P, W, H, ref.bars["position"][sel])
        assert (np.abs(got - want).max(1) <= bar).all()


def test_static_jittered_motion_is_offset_from_centre(plain):
    """a static scene and camera under enableJittering: curRasterPos stays at the pixel centre, so motion = (0.5 - jx, 0.5 - jy)"""
    sc, s64, osc = plain
    W, H = 33, 21
    f = oracle_lib.OracleFrame(osc, W, H, seed=7)
    p = abi.default_frame_params(sc, W, H)
    p.resetFlowBuffer, p.enableJittering = 0, 1
    rng_in = f.buffer(abi.BUF_RNG, 0).reshape(-1)
    f.gbuffer(p)
    ref = R.gbuffer(s64, p, W, H, rng_in=rng_in)
    st, jx = R.restir_ref.pcg_draw(rng_in)
    _, jy = R.restir_ref.pcg_draw(st)
    mv = f.buffer(abi.BUF_GBUFFER1, 0).reshape(-1, 2).astype(np.float64)
    sel = ref.hit & ~ref.steered     # (a miss pixel's position is its direction: test_miss_motion_under_translating_camera)
    want = np.stack([0.5 - jx, 0.5 - jy], 1)
    assert (np.abs(mv - want)[sel].max(1) <= ref.bars["motion"][sel]).all()
    assert np.abs(want).max() > 0.4


def test_miss_motion_under_translating_camera(plain):
    """a miss pixel's position is its direction taken as a point: a translating camera gives it the motion of that point near the
    origin, W, H * (centre - calcScreenPosition(prev, d)), not the zero motion of a point at infinity"""
    sc, s64, osc = plain
    W, H = 36, 24
    f = oracle_lib.OracleFrame(osc, W, H)
    p = abi.default_frame_params(sc, W, H)
    p.resetFlowBuffer = 0
    p.prevCamera.position = (abi.c_f * 3)(*(np.array(p.camera.position[:]) + [0.5, 0.0, 0.0]).astype(np.float32))
    f.gbuffer(p)
    ref = R.gbuffer(s64, p, W, H)
    sky = ~ref.hit & ~ref.steered
    assert sky.sum() > 50
    d = R.Camera64.of(p.camera).direction((ref.pix[sky] % W + 0.5) / W, (ref.pix[sky] // W + 0.5) / H)
    prev = R.Camera64.of(p.prevCamera)
    want = np.stack([ref.pix[sky] % W + 0.5, ref.pix[sky] // W + 0.5], 1) - prev.screen_position(d) * [W, H]
    got = f.buffer(abi.BUF_GBUFFER1, 0).reshape(-1, 2)[ref.pix[sky]]
    assert np.abs(got - want).max() < 1e-3
    assert (np.abs(want).max(1) > 1.0).mean() > 0.9   # far from the zero motion of a point at infinity


def test_running_means(plain):
    """after N jittered frames the accumulated albedo and normal are the means of the frames' albedo and shading normal"""
    sc, s64, osc = plain
    W, H, N = 23, 15, 6
    f = oracle_lib.OracleFrame(osc, W, H, seed=3)
    p = abi.default_frame_params(sc, W, H)
    p.enableJittering = 1
    albedo, normal, steered = [], [], np.zeros(W * H, bool)
    for n in range(N):
        p.numAccumFrames = n
        prev = (f.buffer(abi.BUF_ALBEDO_ACCUM, 0), f.buffer(abi.BUF_NORMAL_ACCUM, 0))
        rng_in = f.buffer(abi.BUF_RNG, 0)
        f.gbuffer(p)
        ref = R.gbuffer(s64, p, W, H, rng_in=rng_in)
        check(ref, planes_of(f), f"accumulated frame {n}", prev, n)
        albedo.append(ref.albedo)
        normal.append(ref.shading_normal)
        steered |= ref.steered
    keep = ~steered
    a = f.buffer(abi.BUF_ALBEDO_ACCUM, 0).reshape(-1, 4)[:, :3]
    nn = f.buffer(abi.BUF_NORMAL_ACCUM, 0).reshape(-1, 4)[:, :3]
    assert np.abs(a - np.mean(albedo, 0))[keep].max() < 1e-3
    assert np.abs(nn - np.mean(normal, 0))[keep].max() < 1e-3
    assert np.abs(np.mean(normal, 0) - normal[0])[keep].max() > 0.01   # the jitter moved some pixels' normals
