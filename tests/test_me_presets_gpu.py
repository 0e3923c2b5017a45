"""GPU parity for motion estimation at the search windows of every preset (svtb200.me_params), bit-exact against the
CPU oracle: the chunked full-pel search, the full-pel shared-memory clamp, the chunked HME regime, the launcher's
CTA widths and the full-SAD search, each with a host-side check that the case really takes the path it is named
after.  test_oracle_me_presets.py pins the oracle against the reference on the same windows."""
import ctypes as C

import numpy as np
import pytest

import common as cm
import svtb200 as sb
from test_oracle_me_presets import make_periodic_case, structure

pytestmark = pytest.mark.gpu

# me.cu launcher constants
HME_FAST_SMEM = 64 * 1024
FP_SMEM_BYTES = 96 * 1024
FP_WARP_CANDIDATES = (4, 3, 6, 2, 8)


def scaled_dist(d):
    return d * 5 // 8 + (1 if d % 8 else 0)


def hme_pitch_words(saw, w, q):
    g = (saw + 4 * q - 1) // (4 * q)
    p = (q * g + w + 3) & ~3
    return p if p & 4 else p + 4


def fp_pitch_words(saw):
    w = 4 * ((saw + 15) >> 4) + 20
    return w if w & 4 else w + 4


def clamp_window(origin, pad, pic_size, ao, size):
    if origin + ao < -pad:
        ao = -pad - origin
    if origin + ao > pic_size - 1:
        ao = ao - ((origin + ao) - (pic_size - 1))
    if origin + ao + size > pic_size:
        size = max(1, size - ((origin + ao + size) - pic_size))
    return ao, size


def used_refs(p):
    return [(l, r) for l in range(p.num_lists) for r in range(p.num_refs[l])]


def launch_plan(p):
    """The kernel choices svt_b200_me_picture makes for `p`, with the launcher's own formulas: whether HME takes
    the chunked regime (hme_kernel_chunked), the full-pel kernel's shared memory (and whether it was clamped to
    FP_SMEM_BYTES) and its CTA width in warps."""
    maxd = max([1] + [scaled_dist(p.ref_dist[l][r]) for l, r in used_refs(p)])
    k = 2 if p.hme_search_method else 1

    def level_bytes(saw, sah, bw, bh):
        bhh = bh // 2 if k == 2 else bh
        wpw = max((saw - 1 + bw + 3) // 4 + 1, hme_pitch_words(saw, bw // 4, 2), hme_pitch_words(saw, bw // 4, 4))
        return 4 * wpw * 4 * (sah - 1 + (bhh - 1) * k + 1) + ((bw + 3) // 4) * 4 * bhh

    nrx, nry = p.number_hme_search_region_in_width, p.number_hme_search_region_in_height

    def amax(a, n):
        return max(a[0], a[1]) if n > 1 else a[0]

    w0 = min(amax(p.hme_level0_search_area_in_width_array, nrx) * maxd, amax(p.hme_level0_max_search_area_in_width_array, nrx))
    h0 = min(amax(p.hme_level0_search_area_in_height_array, nry) * maxd, amax(p.hme_level0_max_search_area_in_height_array, nry))
    hme_need = max(level_bytes((w0 + 15) & ~15, h0, 16, 16),
                   level_bytes((amax(p.hme_level1_search_area_in_width_array, nrx) + 7) & ~7,
                               amax(p.hme_level1_search_area_in_height_array, nry), 32, 32),
                   level_bytes((amax(p.hme_level2_search_area_in_width_array, nrx) + 7) & ~7,
                               amax(p.hme_level2_search_area_in_height_array, nry), 64, 64)) + 256
    saw = (min(p.search_area_width * maxd, p.max_me_search_width) + 7) & ~7
    sah = min(p.search_area_height * maxd, p.max_me_search_height)
    sub = p.me_search_method != 0
    fp_need = (32 if sub else 64) * 64 + fp_pitch_words(saw) * 4 * (sah - 1 + (63 if sub else 64)) + 64
    best = None
    for c in FP_WARP_CANDIDATES:
        cost = 0
        for l, r in used_refs(p):
            dd = scaled_dist(p.ref_dist[l][r])
            w = (min(p.search_area_width * dd, p.max_me_search_width) + 7) & ~7
            h = min(p.search_area_height * dd, p.max_me_search_height)
            tw = (h * 4 * ((w + 15) >> 4) + 31) // 32
            cost += (tw + c - 1) // c * c
        if best is None or cost < best[0]:
            best = (cost, c)
    return dict(hme_need=hme_need, hme_generic=hme_need > HME_FAST_SMEM, w0=w0, h0=h0,
                fp_smem=min(fp_need, FP_SMEM_BYTES), fp_smem_clamped=fp_need > FP_SMEM_BYTES, fp_warps=best[1])


def min_fullpel_chunks(p, hme):
    """Per searched (SB, list, reference): the fewest row chunks fullpel_kernel can split that search window into,
    from the HME results `hme` (the oracle's) with the kernel's own search-area reduction, picture-edge clamp and
    chunk formula.  The kernel re-centres on (0, 0) when that has the lower SAD (check_00_center); both centres
    are tried and the smaller count kept, so the kernel takes at least this many chunks.  0 = not searched."""
    plan = launch_plan(p)
    sub = p.me_search_method != 0
    nsrc, span = (32, 63) if sub else (64, 64)
    sbs_x, sbs_y = (p.full.width + 63) // 64, (p.full.height + 63) // 64
    out = np.zeros((sbs_x * sbs_y, 2, 4), np.int64)
    prune = p.enable_hme_flag and p.enable_hme_level2_flag
    for sb_i in range(sbs_x * sbs_y):
        ox, oy = (sb_i % sbs_x) * 64, (sb_i // sbs_x) * 64
        for l, r in used_refs(p):
            hr = hme[sb_i, l, r]
            if not hr["do_ref"]:
                continue
            dv = 1
            if prune and p.enable_me_sr_adjustment:
                th = p.reduce_me_sr_based_on_mv_length_th
                if abs(int(hr["sc_x"])) <= th and abs(int(hr["sc_y"])) <= th and hr["hme_sad"] < p.stationary_hme_sad_abs_th:
                    dv = p.stationary_me_sr_divisor
                elif hr["hme_sad"] < p.reduce_me_sr_based_on_hme_sad_abs_th:
                    dv = p.me_sr_divisor_for_low_hme_sad
            dd = scaled_dist(p.ref_dist[l][r])
            saw0 = ((min(p.search_area_width * dd, p.max_me_search_width) // dv) + 7) & ~7
            sah0 = max(1, min(p.search_area_height * dd, p.max_me_search_height) // dv)
            cx, cy = int(hr["sc_x"]), int(hr["sc_y"])
            centres = {(cx, cy)}
            if (cx or cy) and p.is_used_as_reference_flag:  # check_00_center's clamp of the HME centre, or (0, 0)
                cx = max(cx, -63 - ox)
                cx -= max(0, ox + cx - (p.full.width - 1))
                cy = max(cy, -63 - oy)
                cy -= max(0, oy + cy - (p.full.height - 1))
                centres = {(cx, cy), (0, 0)}
            counts = []
            for cx, cy in centres:
                xo, saw = clamp_window(ox, 63, p.full.width, cx - (saw0 >> 1), saw0)
                saw = saw if saw < 8 else saw & ~7
                _, sah = clamp_window(oy, 63, p.full.height, cy - (sah0 >> 1), sah0)
                budget_rows = (plan["fp_smem"] - nsrc * 64) // (fp_pitch_words(saw) * 4)
                chunk = max(1, min(sah, budget_rows - span + 1, 2048 // saw))
                counts.append(-(-sah // chunk))
            out[sb_i, l, r] = min(counts)
    return out


def gpu_vs_oracle(params, case, what):
    import gpu_runner as gr
    geos, src, refs = case
    want = cm.run_oracle_me(params, src, refs)
    got = gr.run_gpu_me(params, src, refs)
    cm.assert_me_equal(got, want, params, what)
    return want


PRESET_CASES = [(pr, w, h, s, motion) for pr in range(9) for (w, h, s) in ((320, 192, "ra"), (200, 136, "base_b16"))
                for motion in (True, False)]


@pytest.mark.parametrize("preset,w,h,struct,motion", PRESET_CASES)
def test_me_preset_windows_vs_oracle(preset, w, h, struct, motion):
    n0, n1, dist, tl = structure(preset, struct)
    params = sb.me_params(preset, w, h, n0, n1, dist, tl, 1)
    gpu_vs_oracle(params, cm.make_me_case(w, h, n0, n1, seed=60 + preset + w, motion=motion),
                  f"preset {preset} {w}x{h} {struct} motion={motion}")


def test_me_multi_chunk_fullpel_with_smem_clamp():
    """Preset 0, 256x256 windows: the full-pel request is clamped to FP_SMEM_BYTES, and the search runs in at least
    8 row chunks (2048 / 256 rows each) on random content."""
    w, h = 320, 192
    n0, n1, dist, tl = structure(0, "ra")
    params = sb.me_params(0, w, h, n0, n1, dist, tl, 1)
    plan = launch_plan(params)
    assert plan["fp_smem_clamped"] and plan["fp_smem"] == FP_SMEM_BYTES
    want = gpu_vs_oracle(params, cm.make_me_case(w, h, n0, n1, seed=70), "multi-chunk")
    assert min_fullpel_chunks(params, want.hme).max() >= 8


@pytest.mark.parametrize("preset,chunks", [(0, 8), (3, 2)])
def test_me_chunk_merge_keeps_first_tie(preset, chunks):
    """Periodic references: every period step is a tie for every PU, spread over several row chunks; the chunk
    merge must keep the first one in raster order, as the oracle (and the reference) does."""
    w, h = 200, 136
    n0, n1, dist, tl = structure(preset, "base_b16")
    params = sb.me_params(preset, w, h, n0, n1, dist, tl, 1)
    want = gpu_vs_oracle(params, make_periodic_case(w, h), f"periodic ties preset {preset}")
    assert min_fullpel_chunks(params, want.hme).max() >= chunks


@pytest.mark.parametrize("preset,dist,res_class,w,h", [
    (0, ((4, 1, 0, 0), (2, 0, 0, 0)), None, 320, 192),       # level-0 windows 60 * 3 = 180 per region
    (1, ((16, 2, 0, 0), (8, 0, 0, 0)), None, 200, 136),      # 60 * 10, capped at 240
    (1, ((1, 1, 0, 0), (1, 0, 0, 0)), sb.RES_4K, 320, 192),  # the 4K-class table: 120 per region at distance 1
])
def test_me_chunked_hme_kernel(preset, dist, res_class, w, h):
    """hme_kernel_chunked, the chunked HME regime: the staged regime's shared-memory need exceeds HME_FAST_SMEM."""
    params = sb.me_params(preset, w, h, 2, 1, dist, 1, 1, input_resolution_class=res_class)
    plan = launch_plan(params)
    assert plan["hme_generic"] and plan["hme_need"] > HME_FAST_SMEM
    assert plan["w0"] >= (120 if res_class is not None else 180)
    gpu_vs_oracle(params, cm.make_me_case(w, h, 2, 1, seed=80 + preset), f"chunked HME preset {preset}")


# (preset, reference distances, n_l0, n_l1, the full-pel CTA width in warps that the launcher picks for them)
CTA_CASES = [
    (4, ((1, 2, 3, 4), (1, 2, 3, 0)), 3, 3, 3),
    (8, ((1, 0, 0, 0), (1, 0, 0, 0)), 1, 1, 3),
    (8, ((2, 1, 3, 0), (2, 0, 0, 0)), 3, 1, 3),
    (0, ((1, 2, 0, 0), (1, 0, 0, 0)), 2, 1, 4),
    (3, ((16, 8, 4, 2), (16, 8, 4, 0)), 4, 3, 2),
]


def test_me_fullpel_cta_widths():
    """Three different full-pel CTA widths (2, 3 and 4 warps), each bit-exact against the oracle."""
    w, h = 200, 136
    for i, (preset, dist, n0, n1, warps) in enumerate(CTA_CASES):
        params = sb.me_params(preset, w, h, n0, n1, dist, 1, 1)
        assert launch_plan(params)["fp_warps"] == warps, i
        gpu_vs_oracle(params, cm.make_me_case(w, h, n0, n1, seed=90 + i), f"CTA case {i} ({warps} warps)")
    assert len({c[-1] for c in CTA_CASES}) >= 3


@pytest.mark.parametrize("preset", [0, 4])
def test_me_full_sad_search(preset):
    """hme_search_method = me_search_method = 0 (MRS's full-SAD search) on preset 0 and preset 4 windows."""
    w, h = 200, 136
    n0, n1, dist, tl = structure(preset, "ra")
    params = sb.me_params(preset, w, h, n0, n1, dist, tl, 1)
    params.hme_search_method = params.me_search_method = 0
    want = gpu_vs_oracle(params, cm.make_me_case(w, h, n0, n1, seed=100 + preset), f"full SAD preset {preset}")
    if preset == 0:
        assert launch_plan(params)["fp_smem_clamped"]
        assert min_fullpel_chunks(params, want.hme).max() >= 8


def test_me_preset1_720p_idempotent():
    """Preset 1 at 1280x720 (240 SBs), one reference per list at distance 1: 96x96 windows in 5 row chunks."""
    import gpu_runner as gr
    w, h = 1280, 720
    dist = ((1, 0, 0, 0), (1, 0, 0, 0))
    params = sb.me_params(1, w, h, 1, 1, dist, 1, 1)
    geos, src, refs = cm.make_me_case(w, h, 1, 1, seed=110)
    got = gr.run_gpu_me(params, src, refs)
    cm.assert_me_equal(got, gr.run_gpu_me(params, src, refs), params, "idempotence")
    want = cm.run_oracle_me(params, src, refs)
    cm.assert_me_equal(got, want, params, "720p preset 1 gpu-vs-oracle")
    assert min_fullpel_chunks(params, want.hme).max() >= 5


def _engine_me(lib, e, params, src, refs, n_sb):
    from test_engine_gpu import _host_pic
    hs = _host_pic(1, 1, src)
    hr = (sb.HostMePicture * 8)()
    for i in range(8):
        l, r = divmod(i, 4)
        if l < params.num_lists and r < params.num_refs[l]:
            hr[i] = _host_pic(10 + i, 10 + i, refs[i])
    got = cm.MeBuffers(n_sb)
    rc = lib.svt_b200_engine_me_picture(e, C.byref(params), C.byref(hs), hr, 1, cm.ptr(got.me_mv), cm.ptr(got.me_cand),
                                        cm.ptr(got.total_cand), cm.ptr(got.rc))
    return rc, got


def test_engine_me_picture_at_preset1_windows():
    """The engine's slot staging passes preset 1's windows (chunked HME, 192-wide full-pel windows) through: its
    outputs equal the direct entry's."""
    import gpu_runner as gr
    from test_engine_gpu import assert_me_result
    lib = sb.load()
    w, h = 320, 192
    n0, n1, dist, tl = structure(1, "ra")
    params = sb.me_params(1, w, h, n0, n1, dist, tl, 1)
    assert launch_plan(params)["hme_generic"]
    geos, src, refs = cm.make_me_case(w, h, n0, n1, seed=120)
    want = gr.run_gpu_me(params, src, refs)
    e = C.c_void_p()
    sb.check(lib.svt_b200_engine_create(0, C.byref(e)), lib)
    try:
        rc, got = _engine_me(lib, e, params, src, refs, want.n_sb)
        sb.check(rc, lib)
    finally:
        lib.svt_b200_engine_destroy(e)
    assert_me_result(got, want, want.n_sb, "engine vs direct, preset 1")


SVT_B200_ERR_UNSUPPORTED = -3
# screen-content search areas (set_me_hme_params_oq, sc_content_detected): M0-M3, M4-M5, M6+
SCREEN_CONTENT = [(0, 175, 750), (4, 125, 500), (8, 75, 350)]


@pytest.mark.parametrize("preset,area,max_area", SCREEN_CONTENT)
def test_me_screen_content_windows_refused(preset, area, max_area):
    """Screen-content windows are larger than the kernels are sized for: the direct entry and the engine refuse
    them with SVT_B200_ERR_UNSUPPORTED and an error message, and launch nothing."""
    import gpu_runner as gr
    lib = sb.load()
    w, h = 192, 128
    params = sb.me_params(preset, w, h, 1, 0, ((1, 0, 0, 0), (0, 0, 0, 0)), 1, 1)
    params.search_area_width = params.search_area_height = area * 3 // 2
    params.max_me_search_width = params.max_me_search_height = max_area
    geos, src, refs = cm.make_me_case(w, h, 1, 0, seed=130)
    before = lib.svt_b200_launch_count()
    with pytest.raises(RuntimeError, match=f"rc={SVT_B200_ERR_UNSUPPORTED}: .*larger than the kernels are sized for"):
        gr.run_gpu_me(params, src, refs)
    assert lib.svt_b200_launch_count() == before
    e = C.c_void_p()
    sb.check(lib.svt_b200_engine_create(0, C.byref(e)), lib)
    try:
        rc, _ = _engine_me(lib, e, params, src, refs, ((w + 63) // 64) * ((h + 63) // 64))
        assert rc == SVT_B200_ERR_UNSUPPORTED
        assert b"search area" in lib.svt_b200_last_error()
        assert lib.svt_b200_launch_count() == before
        # the engine still serves a supported call afterwards
        ok = sb.me_params(preset, w, h, 1, 0, ((1, 0, 0, 0), (0, 0, 0, 0)), 1, 1)
        rc, got = _engine_me(lib, e, ok, src, refs, ((w + 63) // 64) * ((h + 63) // 64))
        sb.check(rc, lib)
        np.testing.assert_array_equal(got.me_mv, cm.run_oracle_me(ok, src, refs).me_mv)
    finally:
        lib.svt_b200_engine_destroy(e)
