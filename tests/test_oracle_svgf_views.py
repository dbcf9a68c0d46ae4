"""CPU checks of the SVGF app's debug views (gfx_svgf_debug_visualize): the oracle (oracle/svgf_views.cpp) against a numpy
transcription of debugVisualize (svgf/gpu_kernels/visualize.cu:27-83), on planes read back after oracle SVGF-app frames and on
planted planes, and the display rule of svgf_main.cpp:1907-1911."""
import numpy as np
import pytest

from gfxexp_b200 import abi, engine, scenes
from tests import oracle_svgf_views as OV

F32 = np.float32
VIEWS = list(range(7))
STAGES = 5  # the app's numFilteringStages, which it passes to every view launch (svgf_main.cpp:2127, 2143, 2184)


def np_views(lighting0, lighting1, albedo, normal, psp, moments, view, modulate=False, offset=0.5, scale=0.1, stages=5):
    """visualize.cu:27-83 in float32, pixel (x, y) of every plane to pixel (x, y) of the view"""
    h, w = albedo.shape[:2]
    out = np.zeros((h, w, 4), dtype=F32)
    out[..., 3] = 1
    with np.errstate(invalid="ignore", over="ignore"):
        if view == abi.SVGF_VIEW_NOISY_BEAUTY:
            rgb = lighting0[..., :3]
            out[..., :3] = rgb * albedo[..., :3] if modulate else rgb
        elif view == abi.SVGF_VIEW_VARIANCE:
            out[..., :3] = np.sqrt(lighting0[..., 3:4])
        elif view == abi.SVGF_VIEW_FILTERED_VARIANCE:
            out[..., :3] = np.sqrt((lighting0, lighting1)[stages % 2][..., 3:4])
        elif view == abi.SVGF_VIEW_ALBEDO:
            out[..., :3] = albedo[..., :3]
        elif view == abi.SVGF_VIEW_NORMAL:
            out[..., :3] = F32(0.5) * normal[..., :3] + F32(0.5)
        elif view == abi.SVGF_VIEW_MOTION_VECTOR:
            cur_x = (np.arange(w, dtype=F32) + F32(0.5)) / F32(w)
            cur_y = (np.arange(h, dtype=F32) + F32(0.5)) / F32(h)
            mv_x = F32(w) * (cur_x[None, :] - psp[..., 0])
            mv_y = F32(h) * (cur_y[:, None] - psp[..., 1])
            out[..., 0] = np.fmin(np.fmax(F32(scale) * mv_x + F32(offset), F32(0)), F32(1))
            out[..., 1] = np.fmin(np.fmax(F32(scale) * mv_y + F32(offset), F32(0)), F32(1))
            out[..., 2] = F32(offset)
        else:
            count = (moments[..., 2] & 0xFFFFFF).astype(F32)
            out[..., :3] = np.fmin(count / F32(255), F32(1))[..., None]
    return out


def _same(got, want):
    """bit for bit, except that any NaN equals any NaN"""
    g, w = got.view(np.uint32), want.view(np.uint32)
    both_nan = np.isnan(got) & np.isnan(want)
    return bool(np.all((g == w) | both_nan))


def _oracle_run(scene, w, h, frames, pan=0.0, env_rotation=0.0, modulate=False, check_orientation=False, svgf_off_from=None,
                **kw):
    """SVGF-app frames on the oracle; at each of the app's two launch points every view it launches there is compared with
    the numpy transcription of the planes read back.  svgf_off_from: SVGF is switched off from that frame on."""
    fr = OV.Frame(scene, w, h)
    sv = OV.Svgf(fr)
    p = abi.default_frame_params(scene, w, h)
    p.envLightRotation = env_rotation
    if modulate:
        p.svgfFlags |= abi.SVGF_MODULATE_ALBEDO
    else:
        p.svgfFlags &= ~abi.SVGF_MODULATE_ALBEDO
    checked = set()
    for frame in range(frames):
        cam = abi.make_camera(scene, w, h)
        cam.position[0] += pan * frame
        p.prevCamera = p.camera if frame > 0 else cam
        p.camera = cam
        if svgf_off_from is not None:
            kw["enable_svgf"] = frame < svgf_off_from
        for kind, pass_id, stage in engine.svgf_app_frame_passes(p, frame, view=abi.SVGF_VIEW_NOISY_BEAUTY, **kw):
            if kind == "gbuffer":
                fr.gbuffer(p)
            elif kind == "pathtrace":
                fr.pathtrace(p, pass_id)
            elif kind == "svgf":
                sv.run(p, pass_id, stage)
            elif kind == "svgf_view":
                # the first launch point: Noisy Beauty and Variance
                assert stage == STAGES
                for view in (abi.SVGF_VIEW_NOISY_BEAUTY, abi.SVGF_VIEW_VARIANCE):
                    _check_views(fr, sv, p, view, stage)
                    checked.add(view)
        for view in range(2, 7):  # the second launch point, after albedo modulation + TAA
            _check_views(fr, sv, p, view, STAGES)
            checked.add(view)
        if check_orientation:
            _check_orientation(fr, sv, p, STAGES)
    return checked, sv, p


def _check_views(fr, sv, p, view, stages):
    sv.debug_visualize(p, view, 0.5, 0.1, stages)
    got = sv.buffer(abi.BUF_SVGF_DEBUG_VISUALIZE)
    normal, psp = fr.view_inputs(p)
    want = np_views(sv.buffer(abi.BUF_SVGF_LIGHTING_VARIANCE, 0), sv.buffer(abi.BUF_SVGF_LIGHTING_VARIANCE, 1),
                    sv.buffer(abi.BUF_SVGF_ALBEDO), normal, psp, sv.buffer(abi.BUF_SVGF_MOMENTS, p.bufferIndex), view,
                    bool(p.svgfFlags & abi.SVGF_MODULATE_ALBEDO), 0.5, 0.1, stages)
    assert _same(got, want), f"view {view}: {np.count_nonzero(got != want)} elements differ"
    assert np.all(got[..., 3] == 1)


def _check_orientation(fr, sv, p, stages):
    """the view is written at the pixel whose planes it reads: background pixels (no instance in GBuffer0) show the albedo
    fillBackground writes, 1, and the normal n = 0 -> 0.5, exactly where GBuffer0 has them, and hits show neither.  This pins
    the library's own indexing (no flip between its planes and the view); that the app's view has the same orientation is read
    from the reference (visualize.cu reads its lighting at the launch index and writes at glPix, as svgf.cu:555, 610 do for the
    final image), not tested here."""
    sky = fr.buffer(abi.BUF_GBUFFER0, p.bufferIndex)[..., 0] == 0xFFFFFFFF
    h = sky.shape[0]
    assert sky[: h // 2].sum() > sky[h // 2:].sum(), "the scene's sky is expected in its upper half"
    sv.debug_visualize(p, abi.SVGF_VIEW_ALBEDO, 0.5, 0.1, stages)
    albedo = sv.buffer(abi.BUF_SVGF_DEBUG_VISUALIZE)
    sv.debug_visualize(p, abi.SVGF_VIEW_NORMAL, 0.5, 0.1, stages)
    normal = sv.buffer(abi.BUF_SVGF_DEBUG_VISUALIZE)
    assert np.all(albedo[sky][:, :3] == 1) and np.all(normal[sky][:, :3] == 0.5)
    unit_normal = np.abs(np.linalg.norm(2 * normal[..., :3].astype(np.float64) - 1, axis=-1) - 1) < 1e-3
    assert np.all(unit_normal[~sky])
    # the flipped assignment would not hold
    assert not np.array_equal(sky, sky[::-1])


ORACLE_CASES = {
    "city_static": (scenes.tiny_city_scene, 64, 40, 3, 0.0, {}),
    "city_pan": (scenes.tiny_city_scene, 64, 40, 3, 0.06, {}),
    "city_env_pan": (scenes.small_city_scene_env, 64, 40, 3, 0.04, {"env_rotation": 0.7, "check_orientation": True}),
    "city_modulate_albedo": (scenes.tiny_city_scene, 64, 40, 3, 0.04, {"modulate": True}),
    "city_env_modulate_albedo": (scenes.small_city_scene_env, 64, 40, 2, 0.04, {"env_rotation": 0.7, "modulate": True}),
    "taa_jitter": (scenes.tiny_city_scene, 64, 40, 3, 0.04, {"taa_jitter": True}),
}


@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_oracle_views_equal_numpy_on_svgf_app_frames(case):
    make, w, h, frames, pan, kw = ORACLE_CASES[case]
    assert _oracle_run(make(), w, h, frames, pan, **kw)[0] == set(VIEWS)


def test_oracle_views_with_svgf_off():
    """SVGF off: only the second launch point exists.  The app still passes numFilteringStages = 5, so Filtered Variance reads
    lighting plane 1, which no pass writes while SVGF is off"""
    checked, _, _ = _oracle_run(scenes.tiny_city_scene(), 64, 40, 3, 0.04, enable_svgf=False)
    assert checked == set(VIEWS[2:])


def test_oracle_views_after_svgf_is_switched_off():
    """SVGF on for two frames, then off: Filtered Variance keeps showing plane 1 as the last filtered frame left it"""
    checked, sv, p = _oracle_run(scenes.tiny_city_scene(), 64, 40, 4, 0.04, svgf_off_from=2)
    assert checked == set(VIEWS)
    frozen = sv.buffer(abi.BUF_SVGF_LIGHTING_VARIANCE, 1)[..., 3]
    assert np.count_nonzero(frozen) > 100
    sv.debug_visualize(p, abi.SVGF_VIEW_FILTERED_VARIANCE, 0.5, 0.1, STAGES)
    shown = sv.buffer(abi.BUF_SVGF_DEBUG_VISUALIZE)[..., 0]
    assert np.array_equal(shown, np.sqrt(frozen)) and np.count_nonzero(shown) > 100


def _planted(seed=7):
    h, w = 6, 12
    rng = np.random.default_rng(seed)
    lighting0 = rng.uniform(0, 4, (h, w, 4)).astype(F32)
    lighting1 = rng.uniform(0, 4, (h, w, 4)).astype(F32)
    albedo = rng.uniform(0, 1, (h, w, 4)).astype(F32)
    normal = rng.normal(size=(h, w, 4)).astype(F32)
    normal[..., :3] /= np.linalg.norm(normal[..., :3], axis=-1, keepdims=True)
    normal[0] = 0  # zero normals (background pixels)
    # variances: negative (NaN on both sides), zero, signed zero, tiny, infinite, NaN
    special = np.array([-1.0, -1e-30, 0.0, -0.0, 1e-38, 1e-30, 2.25, np.inf, np.nan, 1e30, 0.5, 7.0], dtype=F32)
    lighting0[1, :, 3] = special
    lighting1[2, :, 3] = special[::-1]
    # sample counts with the accept flags above bit 24
    counts = np.array([0, 1, 254, 255, 256, (1 << 24) - 1, 2, 127, 128, 253, 1000, 65535], dtype=np.uint32)
    flags = np.array([0, 0xF, 0x1, 0x8, 0xA, 0xF, 0x5, 0, 0x3, 0xC, 0x7, 0xF], dtype=np.uint32)
    moments = rng.integers(0, 2**32, (h, w, 4), dtype=np.uint64).astype(np.uint32)
    moments[..., 2] = (counts | (flags << 24))[None, :]
    # prevScreenPos: motion vectors from -2 W to +2 W in x and -2 H to +2 H in y, so that every scale clamps at both ends
    cur_x = (np.arange(w, dtype=F32) + F32(0.5)) / F32(w)
    cur_y = (np.arange(h, dtype=F32) + F32(0.5)) / F32(h)
    psp = np.zeros((h, w, 2), dtype=F32)
    psp[..., 0] = cur_x[None, :] - np.linspace(-2, 2, w, dtype=F32)[None, :] * np.float32(1.3)
    psp[..., 1] = cur_y[:, None] - np.linspace(-2, 2, h, dtype=F32)[:, None] * np.float32(0.7)
    psp[3, 3] = cur_x[3], cur_y[3]  # zero motion
    return lighting0, lighting1, albedo, normal, psp, moments


@pytest.mark.parametrize("view", VIEWS)
@pytest.mark.parametrize("modulate", [False, True])
def test_oracle_views_equal_numpy_on_planted_planes(view, modulate):
    planes = _planted()
    for scale, offset, stages in ((0.1, 0.5, 5), (0.0, 0.5, 4), (-0.3, 0.5, 5), (2.0, 0.25, 0), (-7.5, 1.5, 3)):
        got = OV.view_planes(*planes, view, modulate, offset, scale, stages)
        want = np_views(*planes, view, modulate, offset, scale, stages)
        assert _same(got, want), f"view {view} scale {scale}: {np.count_nonzero(got != want)} elements differ"


def test_planted_planes_cover_the_edges():
    """the planted inputs reach what the views have to get right"""
    lighting0, lighting1, albedo, normal, psp, moments = _planted()
    var = OV.view_planes(lighting0, lighting1, albedo, normal, psp, moments, abi.SVGF_VIEW_VARIANCE)
    assert np.isnan(var[1, 0, 0]) and var[1, 2, 0] == 0 and var[1, 6, 0] == 1.5
    count = OV.view_planes(lighting0, lighting1, albedo, normal, psp, moments, abi.SVGF_VIEW_SAMPLE_COUNT)[0, :6, 0]
    assert list(count) == [0, F32(1) / F32(255), F32(254) / F32(255), 1, 1, 1]
    for scale in (0.1, -0.3):
        mv = OV.view_planes(lighting0, lighting1, albedo, normal, psp, moments, abi.SVGF_VIEW_MOTION_VECTOR, scale=scale)
        assert mv[..., 0].min() == 0 and mv[..., 0].max() == 1 and mv[..., 1].min() == 0 and mv[..., 1].max() == 1
        assert mv[3, 3, 0] == 0.5 and mv[3, 3, 1] == 0.5 and np.all(mv[..., 2] == 0.5)
    mv0 = OV.view_planes(lighting0, lighting1, albedo, normal, psp, moments, abi.SVGF_VIEW_MOTION_VECTOR, scale=0.0)
    assert np.all(mv0[..., :3] == 0.5)
    nrm = OV.view_planes(lighting0, lighting1, albedo, normal, psp, moments, abi.SVGF_VIEW_NORMAL)
    assert np.all(nrm[0, :, :3] == 0.5)


def test_strip_writes_only_its_rows():
    planes = _planted()
    before = np.full((6, 12, 4), 3.0, dtype=F32)
    for view in VIEWS:
        got = OV.view_planes(*planes, view, out=before, rows=(2, 4))
        full = OV.view_planes(*planes, view)
        assert _same(got[2:4], full[2:4]) and np.all(got[:2] == 3) and np.all(got[4:] == 3)


def test_invalid_views_are_refused():
    planes = _planted()
    for view in (-1, 7, 8):
        with pytest.raises(ValueError):
            OV.view_planes(*planes, view)


def test_debug_buffer_before_the_first_view_is_refused():
    fr = OV.Frame(scenes.tiny_city_scene(), 16, 8)
    sv = OV.Svgf(fr)
    with pytest.raises(ValueError):
        sv.buffer(abi.BUF_SVGF_DEBUG_VISUALIZE)


def test_present_flags_follow_the_app():
    """svgf_main.cpp:1907-1911: tone map + sRGB gamma for Noisy Beauty, Variance, Filtered Variance (and Final Rendering),
    the raw values for the others"""
    tone = abi.PRESENT_TONE_MAP | abi.PRESENT_SRGB_GAMMA
    assert [engine.svgf_view_present_flags(v) for v in VIEWS] == [tone, tone, tone, 0, 0, 0, 0]


def test_frame_passes_launch_the_view_where_the_app_does():
    scene = scenes.tiny_city_scene()
    p = abi.default_frame_params(scene, 32, 16)
    for view in VIEWS:
        for enable_svgf in (True, False):
            kinds = [(k, pid) for k, pid, _ in engine.svgf_app_frame_passes(p, 1, enable_svgf=enable_svgf, view=view)]
            at = [i for i, (k, _) in enumerate(kinds) if k == "svgf_view"]
            if view <= abi.SVGF_VIEW_VARIANCE:
                if not enable_svgf:
                    assert at == []
                    continue
                assert kinds[at[0] - 1] == ("svgf", abi.SVGF_ESTIMATE_VARIANCE)
                assert kinds[at[0] + 1] == ("svgf", abi.SVGF_ATROUS)
            else:
                assert at == [len(kinds) - 1] and kinds[-2] == ("svgf", abi.SVGF_MODULATE_TAA)
            assert kinds[at[0]][1] == view
            stage = [st for k, _, st in engine.svgf_app_frame_passes(p, 1, enable_svgf=enable_svgf, view=view) if k == "svgf_view"]
            assert stage == [5]  # numFilteringStages, SVGF on or off
        # without a view the list is the one it was
        assert all(k != "svgf_view" for k, _, _ in engine.svgf_app_frame_passes(p, 1))
