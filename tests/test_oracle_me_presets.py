"""Pins motion estimation at the search windows of every preset, not only preset 8's: the host-side preset table
(svtb200.me_params) against the reference's own parameter derivation, and the ME oracle (oracle/me_oracle.c)
against the reference's C search (oracle/_ref) at presets 0-7 and at MRS's full-SAD search.  The GPU parity
tests (test_me_presets_gpu.py) compare the CUDA path with the oracle on the same windows."""
import ctypes as C

import numpy as np
import pytest

import common as cm
import svtb200 as sb

needs_ref = pytest.mark.skipif(not cm.have_ref(), reason="oracle/_ref not built (no /root/reference here)")
# an oracle/_ref prebuilt from an older harness (and no reference tree to rebuild it from) lacks refh_me_params
needs_ref_params = pytest.mark.skipif(not (cm.have_ref() and hasattr(cm.refh(), "refh_me_params")),
                                      reason="oracle/_ref's harness has no refh_me_params: rebuild oracle/_ref from "
                                             "the reference tree")

# one picture size per input-resolution class (INPUT_SIZE_*_TH luma sample counts)
CLASS_SIZES = {sb.RES_240P: (320, 192), sb.RES_360P: (480, 360), sb.RES_480P: (720, 480), sb.RES_720P: (1280, 720),
               sb.RES_1080P: (1920, 1080), sb.RES_4K: (3840, 2160)}
PRESETS = list(range(sb.PRESET_MRS, 9))
# one-decimation HME (MR and MRS up to 720p): the reference derives it, the library does not implement it
ONE_DECIMATION = {(pr, cls) for pr in (sb.PRESET_MRS, sb.PRESET_MR) for cls in range(sb.RES_720P + 1)}

# reference structures that push the full-pel window to each preset's cap: (n_l0, n_l1, dist, temporal_layer).
# Presets 0-2 search up to 256x256 windows, so they get 2+1 references; presets 3-8 get 4+3.
STRUCT_WIDE = {
    "ra": (2, 1, ((1, 4, 0, 0), (2, 0, 0, 0)), 1),
    "base_b16": (2, 1, ((16, 2, 0, 0), (16, 0, 0, 0)), 0),   # base-layer B at distance 16: list1 HME skipped
}
STRUCT_NARROW = {
    "ra": (4, 3, ((1, 2, 4, 8), (1, 2, 4, 0)), 1),
    "base_b16": (4, 3, ((16, 8, 4, 2), (16, 8, 4, 0)), 0),
}


def structure(preset, name):
    return (STRUCT_WIDE if preset <= 2 else STRUCT_NARROW)[name]


def ref_me_params(preset, width, height, n_l0, n_l1, dist, temporal_layer=1, is_ref=1):
    """(return code, SvtB200MeParams) of the reference's signal_derivation_me_kernel_oq, without the search."""
    geos = sb.me_geometry(width, height)
    p = sb.MeParams()
    d = (C.c_int32 * 8)(*[dist[i // 4][i % 4] for i in range(8)])
    rc = cm.refh().refh_me_params(width, height, preset, n_l0, n_l1, d, temporal_layer, is_ref,
                                  C.byref(geos[0]), C.byref(geos[1]), C.byref(geos[2]), C.byref(p))
    return rc, p


def make_periodic_case(width, height, seed=9, period=8, noise=24):
    """References that repeat exactly every `period` samples in both directions, and a source that is the same
    pattern plus noise: every displacement by a multiple of the period gives every PU the same SAD, so the
    search's result is decided by its tie rule across the whole window (and across the full-pel search's row
    chunks).  The noise keeps the HME SAD high enough that the search area is not reduced."""
    geos = sb.me_geometry(width, height)
    rng = np.random.default_rng(seed)
    tile = rng.integers(40, 216, (period, period))
    pat = np.tile(tile, ((height + period - 1) // period, (width + period - 1) // period))[:height, :width]
    src = np.clip(pat + rng.integers(-noise, noise + 1, pat.shape), 0, 255).astype(np.uint8)
    ref = cm.me_planes(pat.astype(np.uint8), geos)
    return geos, cm.me_planes(src, geos), [ref] * 8


@needs_ref_params
@pytest.mark.parametrize("preset", PRESETS)
def test_me_params_table_matches_reference(preset):
    """svtb200.me_params == the reference's derivation, byte for byte, in every resolution class."""
    skipped = set()
    for cls, (w, h) in CLASS_SIZES.items():
        assert sb.input_resolution(w, h) == cls
        for n0, n1, dist, tl in (STRUCT_NARROW["ra"], (1, 0, ((1, 0, 0, 0), (0, 0, 0, 0)), 0)):
            rc, want = ref_me_params(preset, w, h, n0, n1, dist, tl)
            if rc == -3:
                skipped.add((preset, cls))
                with pytest.raises(ValueError):
                    sb.me_params(preset, w, h, n0, n1, dist, tl)
                continue
            assert rc == 0
            assert bytes(sb.me_params(preset, w, h, n0, n1, dist, tl)) == bytes(want), (preset, cls, n0, n1)
            # the class override carries a class's table to another picture size
            small = sb.me_params(preset, 320, 192, n0, n1, dist, tl, input_resolution_class=cls)
            big = sb.me_params(preset, w, h, n0, n1, dist, tl)
            small.full, small.quarter, small.sixteenth = big.full, big.quarter, big.sixteenth
            assert bytes(small) == bytes(big)
    assert skipped == {k for k in ONE_DECIMATION if k[0] == preset}


def test_preset8_table_is_me_params_8():
    for w, h in CLASS_SIZES.values():
        assert bytes(sb.preset8_me_params(w, h, 2, 1)) == bytes(sb.me_params(8, w, h, 2, 1))


def test_me_params_windows_per_preset():
    """The windows each preset sends the kernels (the table above checks them against the reference; this
    keeps the values that select kernel paths readable)."""
    p = {pr: sb.me_params(pr, 1920, 1080) for pr in range(9)}
    assert [(p[i].search_area_width, p[i].max_me_search_width, p[i].max_me_search_height) for i in range(9)] == [
        (96, 256, 256), (96, 192, 192), (96, 128, 128), (24, 64, 64), (24, 64, 64), (24, 64, 64), (24, 64, 32),
        (24, 64, 32), (24, 64, 32)]
    assert [p[i].hme_level0_search_area_in_width_array[0] for i in range(9)] == [60, 60] + [16] * 7
    assert [p[i].hme_level1_search_area_in_height_array[0] for i in range(9)] == [16] * 5 + [3] * 4
    assert [p[i].prune_ref_if_hme_sad_dev_bigger_than_th for i in range(9)] == [80] * 3 + [30] * 6
    assert sb.me_params(0, 3840, 2160).hme_level0_search_area_in_width_array[1] == 120
    mrs = sb.me_params(sb.PRESET_MRS, 1920, 1080)
    assert (mrs.hme_search_method, mrs.me_search_method, mrs.enable_me_hme_ref_pruning, mrs.enable_me_sr_adjustment) == (0, 0, 0, 0)
    assert mrs.prune_ref_if_hme_sad_dev_bigger_than_th == 0xFFFF


def oracle_vs_reference(preset, w, h, n0, n1, dist, tl, case):
    geos, src, refs = case
    params, want = cm.run_ref_me(w, h, preset, n0, n1, dist, tl, 1, geos, src, refs)
    assert bytes(params) == bytes(sb.me_params(preset, w, h, n0, n1, dist, tl, 1))
    got = cm.run_oracle_me(params, src, refs)
    cm.assert_me_equal(got, want, params, f"oracle-vs-reference preset {preset} {w}x{h}")
    return got


ORACLE_CASES = [(pr, w, h, s) for pr in range(8) for (w, h, s) in ((320, 192, "ra"), (200, 136, "base_b16"))]


@needs_ref
@pytest.mark.parametrize("preset,w,h,struct", ORACLE_CASES)
def test_me_oracle_matches_reference_at_preset(preset, w, h, struct):
    n0, n1, dist, tl = structure(preset, struct)
    oracle_vs_reference(preset, w, h, n0, n1, dist, tl, cm.make_me_case(w, h, n0, n1, seed=40 + preset + w))


@needs_ref
@pytest.mark.parametrize("preset", [1, 4])
def test_me_oracle_matches_reference_static_content(preset):
    n0, n1, dist, tl = structure(preset, "ra")
    oracle_vs_reference(preset, 320, 192, n0, n1, dist, tl, cm.make_me_case(320, 192, n0, n1, seed=6, motion=False))


@needs_ref
@pytest.mark.parametrize("preset", [0, 3])
def test_me_oracle_matches_reference_periodic_ties(preset):
    """Equal SADs at every period step across the whole window: first minimum in raster order wins."""
    n0, n1, dist, tl = structure(preset, "base_b16")
    got = oracle_vs_reference(preset, 200, 136, n0, n1, dist, tl, make_periodic_case(200, 136))
    assert (got.best_sad[:, 0, 0] > 0).all()  # the source noise keeps the SADs off zero


@needs_ref
def test_me_oracle_full_sad_matches_reference_at_mrs():
    """MRS: full-SAD HME and full-pel search (hme_search_method = me_search_method = 0), above the 720p class so
    the reference uses two-decimation HME; one list-0 reference at distance 1 (96x96 windows)."""
    w, h = 1280, 1200
    assert sb.input_resolution(w, h) == sb.RES_1080P
    dist = ((1, 0, 0, 0), (0, 0, 0, 0))
    got = oracle_vs_reference(sb.PRESET_MRS, w, h, 1, 0, dist, 1, cm.make_me_case(w, h, 1, 0, seed=12))
    assert got.total_cand.min() >= 1
