"""Pins the in-loop filter and ME parts of the oracle against the unmodified reference C path (oracle/_ref) on the content of
content_cases.py: flat, saturated, hard-edged and static pictures with all / none / filter-block skip maps.  The GPU tests
(test_filters_content_gpu.py) compare the CUDA kernels with the oracle on the same pictures, so every case here is one the
oracle is known to get right.  The first tests check, without the reference, that each content class reaches the branch it
exists for."""
import ctypes as C

import numpy as np
import pytest

import common as cm
import content_cases as cc
import svtb200 as sb
from test_dlf_gpu import flat_mi
from test_oracle_dlf import dlf_params, pick_params
from test_oracle_lr_frame import random_units, run_oracle_lr, run_ref_lr

needs_ref = pytest.mark.skipif(not cm.have_ref(), reason="oracle/_ref not built")

W, H = 200, 136  # neither a multiple of 64: partial filter blocks on the right and at the bottom
CASES = [(k, bd) for bd in cc.BIT_DEPTHS for k in cc.PAIR_KINDS]
CASE_IDS = [f"{k}-{bd}" for k, bd in CASES]
DLF_LEVELS = [(20, 24, 12, 9), (63, 63, 63, 63)]
PICK_MODES = [(0, 3), (0, 1), (1, 2), (0, 2), (1, 3)]  # (method, loop_filter_mode) as test_oracle_dlf.PICK_CASES
# the lambda finish_cdef_search derives (full lambda of the picture's base_q_idx and bit depth); the device decision takes it
# as an input, test_cdef_lambdas_are_the_references checks the values
CDEF_LAMBDA = {(172, 8): 257491, (172, 10): 257978, (128, 8): 71866, (128, 10): 71610}
APPLY_STRENGTHS = ((63, 61, 59, 62, 0, 17, 33, 3), (63, 0, 62, 1, 60, 33, 3, 47))
FLAT_STRENGTHS = ((63, 61, 59, 62, 1, 17, 33, 3), (63, 0, 62, 1, 60, 33, 3, 47))
DECIDE_CASES = [("flat_regions", 8), ("hard_edges", 10), ("static", 8), ("saturated", 10)]
# the picture-engine cases of test_filters_content_gpu.py: (kind, bit depth, width, height)
ENGINE_CASES = [("hard_edges", 8, 320, 200), ("saturated", 10, 320, 200), ("flat_regions", 8, 264, 136), ("static", 10, 200, 136),
                ("static_blocks", 8, 200, 136), ("flat_static", 10, 320, 200)]
ENGINE_IDS = [f"{k}-{bd}-{w}x{h}" for k, bd, w, h in ENGINE_CASES]
ENGINE_DLF = dict(levels=(36, 28, 20, 63), sharp=1, part_seed=8, pair_seed=9)
ENGINE_PICK_MODES = ((0, 3), (1, 2))
ENGINE_CHAINS = ((3, True), (1, False))  # (pick method, deblocking first)


def partition(mi_rows, mi_cols, seed=5):
    return cm.random_partition(mi_rows, mi_cols, seed)


def run_decide(pick, mi_rows, mi_cols, mse, skip, lam):
    p = sb.CdefDecideParams()
    cm.oracle().orc_cdef_decide_table(pick, C.byref(p))
    p.mi_rows, p.mi_cols, p.lambda_ = mi_rows, mi_cols, lam
    out, idx = sb.CdefDecision(), np.zeros(mse.shape[1], np.int8)
    cm.oracle().orc_cdef_decide(C.byref(p), cm.ptr(mse), cm.ptr(skip), skip.shape[1], C.byref(out), cm.ptr(idx))
    return out, idx


def oracle_cdef_search(pick, rec, src, skip, mi_rows, mi_cols, base_q=172):
    p = sb.CdefSearchParams()
    p.mi_rows, p.mi_cols, p.pri_damping = mi_rows, mi_cols, 3 + (base_q >> 6)
    cm.oracle().orc_cdef_strength_table(pick, C.byref(p))
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    got = np.zeros((2, nfb, 64), np.uint64)
    rs, ss = rec.struct(), src.struct()
    cm.oracle().orc_cdef_search(C.byref(p), C.byref(rs), C.byref(ss), cm.ptr(skip), skip.shape[1], cm.ptr(got))
    return p, got


def cdef_apply_params(mi_rows, mi_cols, damping, ys, uvs):
    p = sb.CdefApplyParams()
    p.mi_rows, p.mi_cols, p.damping = mi_rows, mi_cols, damping
    for i in range(8):
        p.y_strength[i], p.uv_strength[i] = ys[i], uvs[i]
    return p


def oracle_cdef_apply(p, rec, skip, idx):
    out = rec.copy()
    rs, os_ = rec.struct(), out.struct()
    cm.oracle().orc_cdef_apply(C.byref(p), C.byref(rs), C.byref(os_), cm.ptr(skip), skip.shape[1], cm.ptr(idx))
    return out


def assert_same(a, b, what=""):
    for i in range(3):
        np.testing.assert_array_equal(a.plane(i), b.plane(i), err_msg=f"{what} plane {i}")


# ---- each content class reaches its branch (no reference needed) ----------------------------------------------------
@pytest.mark.parametrize("bd", cc.BIT_DEPTHS)
def test_content_classes_reach_their_branches(bd):
    mx = cc.maxv(bd)
    # flat: every 8x8 block of a flat picture has zero CDEF variance, and so do many blocks of the flat-area picture
    for level in ("zero", "mid", "max"):
        f = cc.flat(W, H, bd, level)
        assert cc.cdef_zero_variance_blocks(f) == (W // 8) * (H // 8)
    # the flat-area pictures and the degraded flat pictures the CDEF tests filter have zero-variance blocks
    for seed in (4, 5, 10):
        for kind in ("flat_zero", "flat_mid", "flat_max", "flat_regions"):
            assert cc.cdef_zero_variance_blocks(cc.pair(kind, W, H, bd, seed)[1]) >= 5, (kind, seed)
    # saturated / flat areas / edges, as every test seeds them: large parts exactly on both rails, in every plane
    for seed in (2, 3, 4, 5, 7, 9, 10, 12):
        for make in (cc.saturated, cc.flat_regions, cc.hard_edges):
            f = make(W, H, bd, seed)
            for i in range(3):
                p = f.plane(i)
                assert (p == 0).mean() > 0.02 and (p == mx).mean() > 0.02, (make.__name__, seed, i)
        s = cc.saturated(W, H, bd, seed).plane(0).astype(np.int64)
        assert ((s > 0) & (s <= 3 << (bd - 8))).any() and ((s < mx) & (s >= mx - (3 << (bd - 8)))).any()  # noise at the rails
    # hard edges: steps on 16-, 8- and 4-sample boundaries and off them, in luma and chroma widths
    for n in (W, (W + 1) // 2, H // 2, 100):
        mods = {x % 16 for x in cc.edge_positions(n)}
        assert 0 in mods and 8 in mods and 4 in mods and mods - {0, 4, 8, 12}, (n, mods)
    # every 14-tap deblocking decision occurs on the 8-aligned and the 4-offset luma edges of the undegraded hard-edged
    # pictures the deblocking tests filter (the 'static' reconstructions), at the levels they use
    for w, h, seed in ((W, H, 2), (W, H, 3), (200, 136, ENGINE_DLF["pair_seed"]), (320, 200, ENGINE_DLF["pair_seed"])):
        e = cc.pair("static", w, h, bd, seed)[1].plane(0)
        for xs in (range(8, w, 8), range(4, w, 8)):
            for lv in (20, 63):
                d = cc.lpf_decisions(e, bd, lv, xs)
                assert min(d.values()) > 0, (w, seed, list(xs)[:2], lv, d)
    # static: the reconstruction equals the source / differs in a few blocks only
    s, r = cc.pair("static", W, H, bd)
    assert all((s.plane(i) == r.plane(i)).all() for i in range(3))
    s, r = cc.pair("static_blocks", W, H, bd)
    diff = s.plane(0) != r.plane(0)
    assert 0 < diff.sum() <= 4 * 64


@pytest.mark.parametrize("bd", cc.BIT_DEPTHS)
def test_level_search_sees_equal_sse(bd):
    """A flat static picture: deblocking at every level leaves it unchanged, so every trial of the level search returns the
    same SSE (0) and its comparisons are decided by their tie rule.  The static hard-edged picture has neighbouring levels
    with equal SSE."""
    mi_rows, mi_cols = H // 4, W // 4
    part = partition(mi_rows, mi_cols)
    s, r = cc.pair("flat_static", W, H, bd)
    sse = cc.dlf_level_sse(s, r, flat_mi, mi_rows, mi_cols, part, lambda lv: (lv, lv, lv, lv))
    assert (sse == 0).all()
    s, r = cc.pair("static", W, H, bd)
    sse = cc.dlf_level_sse(s, r, flat_mi, mi_rows, mi_cols, part, lambda lv: (lv, lv, lv, lv))
    assert sse[0, 0] == 0 and sse[63, 0] > 0 and (np.diff(sse[:, 0].astype(np.int64)) == 0).any()


def test_all_skip_map_gives_no_filter_block():
    """An all-skipped picture: the oracle's decision has sb_count == 0 and every filter block index -1; the mixed map
    skips whole filter blocks and keeps others."""
    for w, h in ((W, H), (320, 200), (1920, 1080)):
        mi_rows, mi_cols = cc.mi_dims(w, h)
        nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
        mse = np.random.default_rng(1).integers(0, 1 << 20, (2, nfb, 64)).astype(np.uint64)
        out, idx = run_decide(3, mi_rows, mi_cols, mse, cc.skip_map(mi_rows, mi_cols, "all"), 3500)
        assert out.sb_count == 0 and (idx == -1).all() and out.nb_cdef_strengths == 1
        mixed = cc.skip_map(mi_rows, mi_cols, "mixed", 2)
        fb_skip = cc.fb_all_skipped(mixed, mi_rows, mi_cols)
        assert fb_skip.any() and not fb_skip.all()
        out, idx = run_decide(3, mi_rows, mi_cols, mse, mixed, 3500)
        assert out.sb_count == (~fb_skip).sum() and ((idx == -1) == fb_skip).all()


# ---- deblocking ------------------------------------------------------------------------------------------------------
def run_ref_dlf(mi_rows, mi_cols, part, frame, levels, sharp):
    out = frame.copy()
    st = out.struct()
    flat = (sb.DlfMi * (mi_rows * mi_cols))()
    sbt, dep, inter, skip = (np.ascontiguousarray(x) for x in part)
    cm.refh().refh_dlf_frame(mi_rows, mi_cols, cm.ptr(sbt), cm.ptr(dep), cm.ptr(inter), cm.ptr(skip), (C.c_int32 * 4)(*levels), sharp,
                             C.byref(st), flat)
    return out, flat


@needs_ref
@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_dlf_frame_content_matches_reference(kind, bd):
    mi_rows, mi_cols = H // 4, W // 4
    part = partition(mi_rows, mi_cols)
    _, rec = cc.pair(kind, W, H, bd, 2)
    for levels, sharp in zip(DLF_LEVELS, (0, 3)):
        want, ref_flat = run_ref_dlf(mi_rows, mi_cols, part, rec, levels, sharp)
        assert bytes(ref_flat) == bytes(flat_mi(mi_rows, mi_cols, part, levels))
        got = rec.copy()
        gs = got.struct()
        cm.oracle().orc_dlf_frame(C.byref(dlf_params(mi_rows, mi_cols, levels, sharp)), C.byref(gs), ref_flat)
        assert_same(got, want, f"{kind} levels {levels}")
    if kind == "hard_edges":  # the strong levels filter some of the edges
        assert any((want.plane(i) != rec.plane(i)).any() for i in range(3))


@needs_ref
@pytest.mark.parametrize("bd", cc.BIT_DEPTHS)
@pytest.mark.parametrize("level", ["zero", "mid", "max"])
def test_dlf_leaves_flat_picture_unchanged_in_reference(level, bd):
    """Property the GPU tests assert too: a flat picture is a fixed point of deblocking at any level."""
    mi_rows, mi_cols = H // 4, W // 4
    part = partition(mi_rows, mi_cols)
    f = cc.flat(W, H, bd, level)
    for lv in (1, 20, 40, 63):
        out, _ = run_ref_dlf(mi_rows, mi_cols, part, f, (lv, lv, lv, lv), lv % 8)
        assert_same(out, f, f"level {lv}")


def check_pick(src, rec, part, method, mode, last):
    """The oracle's level search against the reference's; both leave the reconstruction as it was.  Returns the levels."""
    from test_oracle_dlf import run_ref_pick
    mi_rows, mi_cols = src.h // 4, src.w // 4
    want, ref_rec = run_ref_pick(mi_rows, mi_cols, part, src, rec, method, mode, last)
    assert_same(ref_rec, rec)
    p = pick_params(mi_rows, mi_cols, method, mode, last)
    r, t = rec.copy(), rec.copy()
    rs, ss, ts = r.struct(), src.struct(), t.struct()
    got = (C.c_int32 * 4)()
    cm.oracle().orc_pick_filter_level(C.byref(p), C.byref(rs), C.byref(ss), C.byref(ts), flat_mi(mi_rows, mi_cols, part, last), got)
    assert list(got) == want, (method, mode, list(got), want)
    assert_same(r, rec)
    return want


@needs_ref
@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_pick_filter_level_content_matches_reference(kind, bd):
    mi_rows, mi_cols = H // 4, W // 4
    part = partition(mi_rows, mi_cols, 6)
    src, rec = cc.pair(kind, W, H, bd, 3)
    for method, mode in PICK_MODES:
        check_pick(src, rec, part, method, mode, (20, 24, 12, 9) if mode != 1 else (8, 8, 4, 4))


@needs_ref
@pytest.mark.parametrize("bd", cc.BIT_DEPTHS)
@pytest.mark.parametrize("kind", ["static", "static_blocks"])
def test_pick_filter_level_chroma_after_luma_zero_matches_reference(kind, bd):
    """Static content drives the luma search to level 0.  The chroma trials then filter their plane alone
    (svt_av1_loop_filter_frame(plane, plane + 1)), whose frame_init fills that plane's level table although both luma
    levels are 0: the chroma levels are searched, not left at their previous values."""
    n_luma0 = n_chroma_moved = 0
    for pair_seed in range(4):
        src, rec = cc.pair(kind, W, H, bd, pair_seed)
        for part_seed in (4, 6, 8):
            part = partition(H // 4, W // 4, part_seed)
            for method, mode in ((0, 3), (1, 3)):
                lv = check_pick(src, rec, part, method, mode, (20, 24, 12, 9))
                n_luma0 += lv[0] == lv[1] == 0
                n_chroma_moved += lv[0] == lv[1] == 0 and (lv[2], lv[3]) != (12, 9)
    assert n_luma0 > 0 and n_chroma_moved > 0, (n_luma0, n_chroma_moved)


# ---- CDEF ------------------------------------------------------------------------------------------------------------
def ref_cdef_search(pick, rec, src, skip, mi_rows, mi_cols, base_q=172):
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    want = np.zeros((2, nfb, 64), np.uint64)
    rs, ss = rec.struct(), src.struct()
    cm.refh().refh_cdef_search(mi_rows, mi_cols, base_q, pick + 1, C.byref(rs), C.byref(ss), cm.ptr(skip), skip.shape[1], cm.ptr(want))
    return want


def ref_cdef_finish(pick, mse, skip, mi_rows, mi_cols, bd, base_q=172):
    bits, nb, lam = C.c_int32(), C.c_int32(), C.c_uint64()
    ys, uvs, fbs = (C.c_int32 * 8)(), (C.c_int32 * 8)(), np.zeros(mse.shape[1], np.int8)
    assert cm.refh().refh_cdef_finish(mi_rows, mi_cols, base_q, pick + 1, bd, cm.ptr(skip), skip.shape[1], cm.ptr(mse), C.byref(bits),
                                      C.byref(nb), ys, uvs, cm.ptr(fbs), C.byref(lam)) == 0
    return bits.value, nb.value, list(ys), list(uvs), fbs, lam.value


def ref_cdef_apply(rec, skip, idx, mi_rows, mi_cols, damping, ys, uvs):
    out = rec.copy()
    st = out.struct()
    cm.refh().refh_cdef_apply(mi_rows, mi_cols, damping, (C.c_int32 * 8)(*ys), (C.c_int32 * 8)(*uvs), C.byref(st), cm.ptr(skip),
                              skip.shape[1], cm.ptr(idx))
    return out


@needs_ref
@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_cdef_chain_content_matches_reference(kind, bd):
    """search (all four pick methods) -> finish_cdef_search on that search's output -> apply with the decision, each step of
    the oracle against the reference's, on the 'none' and 'mixed' skip maps."""
    mi_rows, mi_cols = cc.mi_dims(W, H)
    src, rec = cc.pair(kind, W, H, bd, 4)
    if kind.startswith("flat"):  # blocks where CDEF's adjust_strength returns 0
        assert cc.cdef_zero_variance_blocks(rec) > 0
    for pick in range(4):
        skip = cc.skip_map(mi_rows, mi_cols, ("none", "mixed")[pick % 2], pick)
        want = ref_cdef_search(pick, rec, src, skip, mi_rows, mi_cols)
        _, got = oracle_cdef_search(pick, rec, src, skip, mi_rows, mi_cols)
        np.testing.assert_array_equal(got, want, f"search pick {pick}")
        bits, nb, ys, uvs, fbs, lam = ref_cdef_finish(pick, want, skip, mi_rows, mi_cols, bd)
        assert lam == CDEF_LAMBDA[(172, bd)]
        out, idx = run_decide(pick, mi_rows, mi_cols, want, skip, lam)
        assert (out.cdef_bits, out.nb_cdef_strengths) == (bits, nb), pick
        assert list(out.y_strength)[:nb] == ys[:nb] and list(out.uv_strength)[:nb] == uvs[:nb], pick
        np.testing.assert_array_equal(idx, fbs)
        ref_out = ref_cdef_apply(rec, skip, fbs, mi_rows, mi_cols, 5, ys, uvs)
        orc_out = oracle_cdef_apply(cdef_apply_params(mi_rows, mi_cols, 5, ys, uvs), rec, skip, idx)
        assert_same(orc_out, ref_out, f"apply pick {pick}")


@needs_ref
@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_cdef_apply_content_fixed_strengths_matches_reference(kind, bd):
    """Apply with strong fixed strengths (primary up to 15, secondary 4) on every filter block: the [min, max] tap clamp and
    the output range on samples at the rails."""
    mi_rows, mi_cols = cc.mi_dims(W, H)
    _, rec = cc.pair(kind, W, H, bd, 5)
    skip = cc.skip_map(mi_rows, mi_cols, "none")
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    idx = (np.arange(nfb) % 8).astype(np.int8)
    ys, uvs = APPLY_STRENGTHS
    for damping in (3, 6):
        want = ref_cdef_apply(rec, skip, idx, mi_rows, mi_cols, damping, ys, uvs)
        got = oracle_cdef_apply(cdef_apply_params(mi_rows, mi_cols, damping, ys, uvs), rec, skip, idx)
        assert_same(got, want, f"damping {damping}")


@needs_ref
@pytest.mark.parametrize("bd", cc.BIT_DEPTHS)
def test_cdef_all_skipped_and_flat_in_reference(bd):
    """All-skip map: the reference's search leaves every table at 0 and its decision signals one strength with no block;
    the oracle agrees.  Flat pictures: the reference's CDEF at any strength leaves them unchanged (the GPU tests assert the
    same of the kernels)."""
    mi_rows, mi_cols = cc.mi_dims(W, H)
    src, rec = cc.pair("hard_edges", W, H, bd, 6)
    skip = cc.skip_map(mi_rows, mi_cols, "all")
    for pick in range(4):
        want = ref_cdef_search(pick, rec, src, skip, mi_rows, mi_cols)
        assert not want.any()
        bits, nb, ys, uvs, fbs, lam = ref_cdef_finish(pick, want, skip, mi_rows, mi_cols, bd)
        out, idx = run_decide(pick, mi_rows, mi_cols, want, skip, lam)
        assert out.sb_count == 0 and (bits, nb) == (out.cdef_bits, out.nb_cdef_strengths) == (0, 1)
        assert list(out.y_strength)[:1] == ys[:1] and list(out.uv_strength)[:1] == uvs[:1]
        assert (fbs == -1).all() and (idx == -1).all()
    skip = cc.skip_map(mi_rows, mi_cols, "none")
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    idx = (np.arange(nfb) % 8).astype(np.int8)
    ys, uvs = FLAT_STRENGTHS
    for level in ("zero", "mid", "max"):
        f = cc.flat(W, H, bd, level)
        for damping in (3, 5, 6):
            assert_same(ref_cdef_apply(f, skip, idx, mi_rows, mi_cols, damping, ys, uvs), f, f"{level} damping {damping}")


# ---- loop restoration ------------------------------------------------------------------------------------------------
LR_MODES = [(("wiener", "wiener", "wiener"), (1, 1, 1)), (("sgr", "sgr", "sgr"), (2, 2, 2)), (("mix", "mix", "mix"), (3, 3, 3))]


def lr_content(kind, bd, seed, modes, unit_sizes=(64, 32, 32), w=W, h=H):
    rng = np.random.default_rng(seed)
    src, rec = cc.pair(kind, w, h, bd, seed)
    dblk = cc.changed_blocks(rec, seed + 1, n=6)
    units = []
    for p in range(3):
        pw, ph = (w, h) if p == 0 else ((w + 1) // 2, (h + 1) // 2)
        n = max((pw + unit_sizes[p] // 2) // unit_sizes[p], 1) * max((ph + unit_sizes[p] // 2) // unit_sizes[p], 1)
        units.append(random_units(rng, n, modes[p]))
    return rec, dblk, units


@needs_ref
@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_lr_frame_content_matches_reference(kind, bd):
    for modes, ftypes in LR_MODES:
        cdef, dblk, units = lr_content(kind, bd, 7, modes)
        want = run_ref_lr(cdef, dblk, units, (64, 32, 32), ftypes, 0)
        got = run_oracle_lr(cdef, dblk, units, (64, 32, 32), ftypes, 0)
        assert_same(got, want, str(modes))
        for i in range(3):
            assert got.plane(i).max() <= cc.maxv(bd)


@needs_ref
@pytest.mark.parametrize("bd", cc.BIT_DEPTHS)
def test_lr_output_clips_reached_in_reference(bd):
    """On saturated and hard-edged content the reference's Wiener and self-guided outputs sit on both rails where the
    input did not (the output clips act): the GPU comparison on these pictures covers the clips."""
    for kind in ("saturated", "hard_edges"):
        for modes, ftypes in LR_MODES[:2]:
            cdef, dblk, units = lr_content(kind, bd, 7, modes)
            want = run_ref_lr(cdef, dblk, units, (64, 32, 32), ftypes, 0)
            y, c = want.plane(0), cdef.plane(0)
            assert ((y == cc.maxv(bd)) & (c < cc.maxv(bd))).any() and ((y == 0) & (c > 0)).any(), (kind, modes)


# ---- motion estimation -----------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("kind", ["flat", "black"])
@pytest.mark.parametrize("preset", [8, 5])
def test_me_flat_pictures_match_reference(kind, preset):
    """Constant pictures: every candidate of a reference has the same SAD, so HME, the full-pel search and the candidate
    lists are decided by tie rules alone."""
    from test_oracle_me_presets import structure
    w, h = 200, 136
    n0, n1, dist, tl = structure(preset, "ra")
    geos, src, refs = cc.me_flat_case(w, h, kind)
    params, want = cm.run_ref_me(w, h, preset, n0, n1, dist, tl, 1, geos, src, refs)
    got = cm.run_oracle_me(params, src, refs)
    cm.assert_me_equal(got, want, params, f"{kind} preset {preset}")
    if kind == "black":
        assert (want.best_sad[:, 0, 0] == 0).all()


# ---- the remaining inputs of the GPU tests, with the same parameters -------------------------------------------------
@needs_ref
def test_cdef_lambdas_are_the_references():
    mi_rows, mi_cols = cc.mi_dims(W, H)
    skip = cc.skip_map(mi_rows, mi_cols, "none")
    mse = np.ones((2, ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16), 64), np.uint64)
    for (base_q, bd), lam in CDEF_LAMBDA.items():
        assert ref_cdef_finish(3, mse, skip, mi_rows, mi_cols, bd, base_q)[-1] == lam


@needs_ref
@pytest.mark.parametrize("skip_kind", ["all", "none", "mixed"])
@pytest.mark.parametrize("kind,bd", DECIDE_CASES)
def test_cdef_decide_content_matches_reference(kind, bd, skip_kind):
    """The inputs of test_cdef_decide_content_vs_oracle: finish_cdef_search on the search output of the content."""
    mi_rows, mi_cols = cc.mi_dims(W, H)
    src, rec = cc.pair(kind, W, H, bd, 4)
    skip = cc.skip_map(mi_rows, mi_cols, skip_kind, 1)
    for pick in range(4):
        mse = ref_cdef_search(pick, rec, src, skip, mi_rows, mi_cols)
        bits, nb, ys, uvs, fbs, lam = ref_cdef_finish(pick, mse, skip, mi_rows, mi_cols, bd)
        out, idx = run_decide(pick, mi_rows, mi_cols, mse, skip, CDEF_LAMBDA[(172, bd)])
        assert (out.cdef_bits, out.nb_cdef_strengths) == (bits, nb), pick
        assert list(out.y_strength)[:nb] == ys[:nb] and list(out.uv_strength)[:nb] == uvs[:nb], pick
        np.testing.assert_array_equal(idx, fbs)
        if skip_kind == "all":
            assert out.sb_count == 0 and (fbs == -1).all()


@needs_ref
@pytest.mark.parametrize("kind,bd,w,h", ENGINE_CASES, ids=ENGINE_IDS)
def test_engine_dlf_and_pick_inputs_match_reference(kind, bd, w, h):
    """The inputs of test_engine_dlf_and_pick_content: deblocking at the engine levels, the level search, and the
    deblocking at the searched levels."""
    mi_rows, mi_cols = h // 4, w // 4
    part = partition(mi_rows, mi_cols, ENGINE_DLF["part_seed"])
    src, rec = cc.pair(kind, w, h, bd, ENGINE_DLF["pair_seed"])
    levels, sharp = ENGINE_DLF["levels"], ENGINE_DLF["sharp"]
    want, ref_flat = run_ref_dlf(mi_rows, mi_cols, part, rec, levels, sharp)
    got = rec.copy()
    gs = got.struct()
    cm.oracle().orc_dlf_frame(C.byref(dlf_params(mi_rows, mi_cols, levels, sharp)), C.byref(gs), ref_flat)
    assert_same(got, want, "dlf")
    for method, mode in ENGINE_PICK_MODES:
        lv = check_pick(src, rec, part, method, mode, (20, 24, 12, 9))
        want, ref_flat = run_ref_dlf(mi_rows, mi_cols, part, rec, tuple(lv), 0)
        got = rec.copy()
        gs = got.struct()
        cm.oracle().orc_dlf_frame(C.byref(dlf_params(mi_rows, mi_cols, tuple(lv), 0)), C.byref(gs), ref_flat)
        assert_same(got, want, f"pick {method},{mode}")


class ContentCdefChain:
    """The oracle's deblocking (optional, levels (20, 24, 12, 9), sharpness 1) -> strength search (base_q_idx 128) ->
    decision (the reference's lambda) -> apply (damping 5) on content_cases pictures and skip maps: what one
    svt_b200_engine_dlf_cdef_frame_dev call must produce.  ref_check() runs the reference's chain on the same inputs."""
    BASE_Q = 128

    def __init__(self, src, rec, skip_kind, pick, with_dlf, seed=0, levels=(20, 24, 12, 9)):
        orc = cm.oracle()
        self.src, self.rec, self.pick, self.levels = src, rec, pick, levels
        self.mi_rows, self.mi_cols = mi_rows, mi_cols = cc.mi_dims(src.w, src.h)
        self.skip = cc.skip_map(mi_rows, mi_cols, skip_kind, seed)
        pre = rec.copy()
        self.dp, self.flat, self.part = None, None, None
        if with_dlf:
            self.part = partition(mi_rows, mi_cols, seed + 5)
            self.flat = flat_mi(mi_rows, mi_cols, self.part, levels)
            self.dp = dlf_params(mi_rows, mi_cols, levels, 1)
            ps = pre.struct()
            orc.orc_dlf_frame(C.byref(self.dp), C.byref(ps), self.flat)
        self.sp, self.mse = oracle_cdef_search(pick, pre, src, self.skip, mi_rows, mi_cols, base_q=self.BASE_Q)
        self.lam = CDEF_LAMBDA[(self.BASE_Q, src.bd)]
        self.dcp = sb.CdefDecideParams()
        orc.orc_cdef_decide_table(pick, C.byref(self.dcp))
        self.dcp.mi_rows, self.dcp.mi_cols, self.dcp.lambda_ = mi_rows, mi_cols, self.lam
        self.nfb = self.mse.shape[1]
        self.want_dec, self.want_idx = run_decide(pick, mi_rows, mi_cols, self.mse, self.skip, self.lam)
        pa = cdef_apply_params(mi_rows, mi_cols, 5, list(self.want_dec.y_strength), list(self.want_dec.uv_strength))
        self.pre = pre
        self.want = oracle_cdef_apply(pa, pre, self.skip, self.want_idx)

    def ref_check(self):
        pre = self.rec
        if self.part is not None:
            pre, _ = run_ref_dlf(self.mi_rows, self.mi_cols, self.part, self.rec, self.levels, 1)
            assert_same(pre, self.pre, "deblocking")
        mse = ref_cdef_search(self.pick, pre, self.src, self.skip, self.mi_rows, self.mi_cols, self.BASE_Q)
        np.testing.assert_array_equal(self.mse, mse)
        bits, nb, ys, uvs, fbs, lam = ref_cdef_finish(self.pick, mse, self.skip, self.mi_rows, self.mi_cols, self.src.bd, self.BASE_Q)
        assert lam == self.lam
        d = self.want_dec
        assert (d.cdef_bits, d.nb_cdef_strengths) == (bits, nb)
        assert list(d.y_strength)[:nb] == ys[:nb] and list(d.uv_strength)[:nb] == uvs[:nb]
        np.testing.assert_array_equal(self.want_idx, fbs)
        assert_same(ref_cdef_apply(pre, self.skip, fbs, self.mi_rows, self.mi_cols, 5, ys, uvs), self.want, "apply")


@needs_ref
@pytest.mark.parametrize("skip_kind", ["all", "none", "mixed"])
@pytest.mark.parametrize("kind,bd,w,h", ENGINE_CASES, ids=ENGINE_IDS)
def test_engine_cdef_chain_inputs_match_reference(kind, bd, w, h, skip_kind):
    src, rec = cc.pair(kind, w, h, bd, 10)
    for pick, with_dlf in ENGINE_CHAINS:
        ContentCdefChain(src, rec, skip_kind, pick, with_dlf, seed=pick).ref_check()


@needs_ref
def test_engine_cdef_chain_1080p_inputs_match_reference():
    src, rec = cc.pair("hard_edges", 1920, 1080, 10, 11)
    ContentCdefChain(src, rec, "mixed", 3, True, seed=2).ref_check()


@needs_ref
@pytest.mark.parametrize("kind,bd,w,h", ENGINE_CASES, ids=ENGINE_IDS)
def test_engine_lr_inputs_match_reference(kind, bd, w, h):
    for modes, ftypes in LR_MODES:
        cdef, dblk, units = lr_content(kind, bd, 12, modes, w=w, h=h)
        want = run_ref_lr(cdef, dblk, units, (64, 32, 32), ftypes, 0)
        got = run_oracle_lr(cdef, dblk, units, (64, 32, 32), ftypes, 0)
        assert_same(got, want, str(modes))
