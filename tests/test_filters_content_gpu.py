"""GPU parity for the in-loop filters, the picture engine's filter chain and ME on the content of content_cases.py (flat,
saturated, hard-edged and static pictures; all / none / filter-block skip maps), bit-exact against the CPU oracle, which
test_oracle_filters_content.py pins to the reference on the same pictures.  Where a property is exact it is asserted as
well: a flat picture is a fixed point of deblocking at every level and of CDEF at every strength."""
import ctypes as C

import numpy as np
import pytest

import common as cm
import content_cases as cc
import svtb200 as sb
from test_dlf_gpu import flat_mi
from test_oracle_dlf import dlf_params, pick_params
from test_oracle_filters_content import (APPLY_STRENGTHS, CASE_IDS, CASES, CDEF_LAMBDA, DECIDE_CASES, DLF_LEVELS, ENGINE_CASES,
                                         ENGINE_CHAINS, ENGINE_DLF, ENGINE_IDS, ENGINE_PICK_MODES, FLAT_STRENGTHS, LR_MODES, PICK_MODES,
                                         ContentCdefChain, assert_same, cdef_apply_params, lr_content, oracle_cdef_apply,
                                         oracle_cdef_search, partition, run_decide)

pytestmark = pytest.mark.gpu

W, H = 200, 136


@pytest.fixture
def engine():
    lib = sb.load()
    e = C.c_void_p()
    sb.check(lib.svt_b200_engine_create(0, C.byref(e)), lib)
    yield e
    lib.svt_b200_engine_destroy(e)


def oracle_dlf(rec, mi_rows, mi_cols, part, levels, sharp):
    out = rec.copy()
    os_ = out.struct()
    cm.oracle().orc_dlf_frame(C.byref(dlf_params(mi_rows, mi_cols, levels, sharp)), C.byref(os_), flat_mi(mi_rows, mi_cols, part, levels))
    return out


def oracle_pick(p, src, rec, flat):
    r, t = rec.copy(), rec.copy()
    rs, ss, ts = r.struct(), src.struct(), t.struct()
    out = (C.c_int32 * 4)()
    cm.oracle().orc_pick_filter_level(C.byref(p), C.byref(rs), C.byref(ss), C.byref(ts), flat, out)
    return list(out)


# ---- direct entries --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_dlf_frame_content_vs_oracle(kind, bd):
    import gpu_runner as gr
    mi_rows, mi_cols = H // 4, W // 4
    part = partition(mi_rows, mi_cols)
    _, rec = cc.pair(kind, W, H, bd, 2)
    for levels, sharp in zip(DLF_LEVELS, (0, 3)):
        want = oracle_dlf(rec, mi_rows, mi_cols, part, levels, sharp)
        got = gr.run_gpu_dlf(dlf_params(mi_rows, mi_cols, levels, sharp), rec, flat_mi(mi_rows, mi_cols, part, levels))
        assert_same(got, want, f"levels {levels}")


@pytest.mark.parametrize("bd", cc.BIT_DEPTHS)
@pytest.mark.parametrize("level", ["zero", "mid", "max"])
def test_dlf_leaves_flat_picture_unchanged(level, bd):
    import gpu_runner as gr
    mi_rows, mi_cols = H // 4, W // 4
    part = partition(mi_rows, mi_cols)
    f = cc.flat(W, H, bd, level)
    for lv in (1, 20, 40, 63):
        levels = (lv, lv, lv, lv)
        got = gr.run_gpu_dlf(dlf_params(mi_rows, mi_cols, levels, lv % 8), f, flat_mi(mi_rows, mi_cols, part, levels))
        assert_same(got, f, f"level {lv}")


@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_pick_filter_level_content_vs_oracle(kind, bd):
    """The level search on flat / static content, where trial levels tie on SSE, with every method / mode pair."""
    mi_rows, mi_cols = H // 4, W // 4
    part = partition(mi_rows, mi_cols, 6)
    src, rec = cc.pair(kind, W, H, bd, 3)
    for method, mode in PICK_MODES:
        gpu_pick_vs_oracle(src, rec, part, method, mode, (20, 24, 12, 9) if mode != 1 else (8, 8, 4, 4))


def gpu_pick_vs_oracle(src, rec, part, method, mode, last):
    import gpu_runner as gr
    mi_rows, mi_cols = src.h // 4, src.w // 4
    flat = flat_mi(mi_rows, mi_cols, part, last)
    p = pick_params(mi_rows, mi_cols, method, mode, last)
    want = oracle_pick(p, src, rec, flat)
    got, after = gr.run_gpu_pick(p, rec, src, flat)
    assert got == want, (method, mode, got, want)
    assert_same(after, rec)
    return got


@pytest.mark.parametrize("bd", cc.BIT_DEPTHS)
@pytest.mark.parametrize("kind", ["static", "static_blocks"])
def test_pick_filter_level_chroma_after_luma_zero_vs_oracle(kind, bd):
    """Luma searched down to 0 on static content: the chroma trials still filter their plane at the trial level (the
    level table of a chroma-only pass is filled whatever the luma levels), as test_oracle_filters_content pins."""
    n_chroma_moved = 0
    for pair_seed in range(4):
        src, rec = cc.pair(kind, W, H, bd, pair_seed)
        for part_seed in (4, 6, 8):
            part = partition(H // 4, W // 4, part_seed)
            for method, mode in ((0, 3), (1, 3)):
                lv = gpu_pick_vs_oracle(src, rec, part, method, mode, (20, 24, 12, 9))
                n_chroma_moved += lv[0] == lv[1] == 0 and (lv[2], lv[3]) != (12, 9)
    assert n_chroma_moved > 0


@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_cdef_search_content_vs_oracle(kind, bd):
    import gpu_runner as gr
    mi_rows, mi_cols = cc.mi_dims(W, H)
    src, rec = cc.pair(kind, W, H, bd, 4)
    for pick in range(4):
        skip = cc.skip_map(mi_rows, mi_cols, ("none", "mixed")[pick % 2], pick)
        p, want = oracle_cdef_search(pick, rec, src, skip, mi_rows, mi_cols)
        got = gr.run_gpu_cdef_search(p, rec, src, skip)
        np.testing.assert_array_equal(got, want, f"pick {pick}")


def gpu_cdef_decide(pick, mi_rows, mi_cols, mse, skip, lam):
    import torch
    lib = sb.load()
    p = sb.CdefDecideParams()
    lib.svt_b200_cdef_decide_table(pick, C.byref(p))
    p.mi_rows, p.mi_cols, p.lambda_ = mi_rows, mi_cols, lam
    nfb = mse.shape[1]
    dm, dsk = torch.from_numpy(mse.view(np.int64)).cuda(), torch.from_numpy(np.ascontiguousarray(skip)).cuda()
    dout = torch.zeros(C.sizeof(sb.CdefDecision), dtype=torch.uint8, device="cuda")
    didx = torch.full((nfb,), 77, dtype=torch.int8, device="cuda")
    scr = torch.zeros(nfb * (16 + 16 * 64) + 64, dtype=torch.uint8, device="cuda")
    lib.svt_b200_cdef_decide.argtypes = [C.POINTER(sb.CdefDecideParams)] + [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                                                             C.c_void_p, C.c_void_p]
    sb.check(lib.svt_b200_cdef_decide(C.byref(p), dm.data_ptr(), dsk.data_ptr(), skip.shape[1], dout.data_ptr(), didx.data_ptr(),
                                      scr.data_ptr(), None), lib)
    torch.cuda.synchronize()
    return sb.CdefDecision.from_buffer_copy(dout.cpu().numpy().tobytes()), didx.cpu().numpy()


def assert_decision(got, want):
    assert (got.cdef_bits, got.nb_cdef_strengths, got.sb_count) == (want.cdef_bits, want.nb_cdef_strengths, want.sb_count)
    k = want.nb_cdef_strengths
    assert list(got.y_index)[:k] == list(want.y_index)[:k] and list(got.uv_index)[:k] == list(want.uv_index)[:k]
    assert list(got.y_strength)[:k] == list(want.y_strength)[:k] and list(got.uv_strength)[:k] == list(want.uv_strength)[:k]


@pytest.mark.parametrize("skip_kind", ["all", "none", "mixed"])
@pytest.mark.parametrize("kind,bd", DECIDE_CASES)
def test_cdef_decide_content_vs_oracle(kind, bd, skip_kind):
    """svt_b200_cdef_decide on the search output of this content (ties between strengths on flat / static pictures), with
    every block skipped (sb_count == 0: one strength signalled, no filter block), none, or whole filter blocks skipped."""
    mi_rows, mi_cols = cc.mi_dims(W, H)
    src, rec = cc.pair(kind, W, H, bd, 4)
    skip = cc.skip_map(mi_rows, mi_cols, skip_kind, 1)
    for pick in range(4):
        _, mse = oracle_cdef_search(pick, rec, src, skip, mi_rows, mi_cols)
        want, want_idx = run_decide(pick, mi_rows, mi_cols, mse, skip, CDEF_LAMBDA[(172, bd)])
        if skip_kind == "all":
            assert want.sb_count == 0 and want.nb_cdef_strengths == 1 and (want_idx == -1).all()
        got, idx = gpu_cdef_decide(pick, mi_rows, mi_cols, mse, skip, CDEF_LAMBDA[(172, bd)])
        assert_decision(got, want)
        np.testing.assert_array_equal(idx, want_idx)


@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_cdef_apply_content_vs_oracle(kind, bd):
    """Strong strengths on every filter block (the [min, max] tap clamp and rail samples), and the per-block strengths the
    decision picked on the mixed skip map."""
    import gpu_runner as gr
    mi_rows, mi_cols = cc.mi_dims(W, H)
    src, rec = cc.pair(kind, W, H, bd, 5)
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    skip = cc.skip_map(mi_rows, mi_cols, "none")
    idx = (np.arange(nfb) % 8).astype(np.int8)
    ys, uvs = APPLY_STRENGTHS
    for damping in (3, 6):
        p = cdef_apply_params(mi_rows, mi_cols, damping, ys, uvs)
        assert_same(gr.run_gpu_cdef_apply(p, rec, skip, idx), oracle_cdef_apply(p, rec, skip, idx), f"damping {damping}")
    # the decision test_cdef_chain_content_matches_reference pins for pick method 3
    src, rec = cc.pair(kind, W, H, bd, 4)
    skip = cc.skip_map(mi_rows, mi_cols, "mixed", 3)
    _, mse = oracle_cdef_search(3, rec, src, skip, mi_rows, mi_cols)
    dec, idx = run_decide(3, mi_rows, mi_cols, mse, skip, CDEF_LAMBDA[(172, bd)])
    p = cdef_apply_params(mi_rows, mi_cols, 5, list(dec.y_strength), list(dec.uv_strength))
    assert_same(gr.run_gpu_cdef_apply(p, rec, skip, idx), oracle_cdef_apply(p, rec, skip, idx), "decided")


@pytest.mark.parametrize("bd", cc.BIT_DEPTHS)
def test_cdef_leaves_flat_picture_unchanged(bd):
    import gpu_runner as gr
    mi_rows, mi_cols = cc.mi_dims(W, H)
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    skip = cc.skip_map(mi_rows, mi_cols, "none")
    idx = (np.arange(nfb) % 8).astype(np.int8)
    for level in ("zero", "mid", "max"):
        f = cc.flat(W, H, bd, level)
        for damping in (3, 6):
            p = cdef_apply_params(mi_rows, mi_cols, damping, *FLAT_STRENGTHS)
            assert_same(gr.run_gpu_cdef_apply(p, f, skip, idx), f, f"{level} damping {damping}")


@pytest.mark.parametrize("kind,bd", CASES, ids=CASE_IDS)
def test_lr_frame_content_vs_oracle(kind, bd):
    import gpu_runner as gr
    from test_oracle_lr_frame import run_oracle_lr
    for modes, ftypes in LR_MODES:
        cdef, dblk, units = lr_content(kind, bd, 7, modes)
        want = run_oracle_lr(cdef, dblk, units, (64, 32, 32), ftypes, 0)
        got = gr.run_gpu_lr(cdef, dblk, units, (64, 32, 32), ftypes, 0)
        assert_same(got, want, str(modes))


# ---- picture engine --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,bd,w,h", ENGINE_CASES, ids=ENGINE_IDS)
def test_engine_dlf_and_pick_content(engine, kind, bd, w, h):
    lib = sb.load()
    mi_rows, mi_cols = h // 4, w // 4
    part = partition(mi_rows, mi_cols, ENGINE_DLF["part_seed"])
    src, rec = cc.pair(kind, w, h, bd, ENGINE_DLF["pair_seed"])
    levels, sharp = ENGINE_DLF["levels"], ENGINE_DLF["sharp"]
    want = oracle_dlf(rec, mi_rows, mi_cols, part, levels, sharp)
    got = rec.copy()
    gs = got.struct()
    sb.check(lib.svt_b200_engine_dlf_frame(engine, C.byref(dlf_params(mi_rows, mi_cols, levels, sharp)), C.byref(gs),
                                           flat_mi(mi_rows, mi_cols, part, levels)), lib)
    assert_same(got, want, "dlf")
    for method, mode in ENGINE_PICK_MODES:
        last = (20, 24, 12, 9)
        flat = flat_mi(mi_rows, mi_cols, part, last)
        p = pick_params(mi_rows, mi_cols, method, mode, last)
        want_lv = oracle_pick(p, src, rec, flat)
        got = rec.copy()
        gs, ss = got.struct(), src.struct()
        lv = (C.c_int32 * 4)()
        sb.check(lib.svt_b200_engine_dlf_pick_frame(engine, C.byref(p), C.byref(gs), C.byref(ss), flat, lv), lib)
        assert list(lv) == want_lv, (method, mode)
        assert_same(got, oracle_dlf(rec, mi_rows, mi_cols, part, tuple(want_lv), 0), f"pick {method},{mode}")


class EngineCdefChain(ContentCdefChain):
    """ContentCdefChain (the oracle's chain, pinned to the reference) run as one svt_b200_engine_dlf_cdef_frame_dev call."""

    def run(self, lib, e, apply):
        got, dec, idx = self.rec.copy(), sb.CdefDecision(), np.full(self.nfb, 99, np.int8)
        gs, ss = got.struct(), self.src.struct()
        rc = lib.svt_b200_engine_dlf_cdef_frame_dev(e, C.byref(self.dp) if self.dp else None, self.flat, C.byref(self.sp), C.byref(self.dcp),
                                                    5, apply, C.byref(gs), C.byref(ss), cm.ptr(self.skip), self.skip.shape[1],
                                                    C.byref(dec), cm.ptr(idx))
        return rc, got, dec, idx

    def check(self, lib, e):
        tab = sb.CdefDecideParams()
        assert lib.svt_b200_cdef_decide_table(self.pick, C.byref(tab)) == self.sp.n_strengths
        assert list(tab.filter_strength) == list(self.dcp.filter_strength)
        rc, got, dec, idx = self.run(lib, e, 1)
        sb.check(rc, lib)
        assert_decision(dec, self.want_dec)
        np.testing.assert_array_equal(idx, self.want_idx)
        assert_same(got, self.want, "apply = 1")
        rc, again, dec, idx = self.run(lib, e, 0)  # decision only: the host picture untouched
        sb.check(rc, lib)
        assert_decision(dec, self.want_dec)
        np.testing.assert_array_equal(idx, self.want_idx)
        assert_same(again, self.rec, "apply = 0")


@pytest.mark.parametrize("skip_kind", ["all", "none", "mixed"])
@pytest.mark.parametrize("kind,bd,w,h", ENGINE_CASES, ids=ENGINE_IDS)
def test_engine_cdef_chain_content(engine, kind, bd, w, h, skip_kind):
    lib = sb.load()
    src, rec = cc.pair(kind, w, h, bd, 10)
    for pick, with_dlf in ENGINE_CHAINS:
        c = EngineCdefChain(src, rec, skip_kind, pick, with_dlf, seed=pick)
        if skip_kind == "all":
            assert c.want_dec.sb_count == 0 and (c.want_idx == -1).all()
            assert_same(c.want, c.pre, "all skipped: CDEF changes nothing")
        c.check(lib, engine)


def test_engine_cdef_chain_1080p_hard_edges(engine):
    """The bench geometry, 10-bit, hard-edged content: 1080 rows leave the last filter-block row partial (56 rows)."""
    lib = sb.load()
    src, rec = cc.pair("hard_edges", 1920, 1080, 10, 11)
    c = EngineCdefChain(src, rec, "mixed", 3, True, seed=2)
    assert 1080 % 64 and c.want_dec.sb_count > 0
    c.check(lib, engine)


@pytest.mark.parametrize("kind,bd,w,h", ENGINE_CASES, ids=ENGINE_IDS)
def test_engine_lr_frame_content(engine, kind, bd, w, h):
    from test_engine_gpu import lr_boundary_lines, lr_frame_params
    from test_oracle_lr_frame import run_oracle_lr
    lib = sb.load()
    for modes, ftypes in LR_MODES:
        cdef, dblk, units = lr_content(kind, bd, 12, modes, w=w, h=h)
        want = run_oracle_lr(cdef, dblk, units, (64, 32, 32), ftypes, 0)
        lines, keep = lr_boundary_lines(dblk)
        p, n_units = lr_frame_params(units, (64, 32, 32), ftypes)
        got = cdef.copy()
        gs = got.struct()
        sb.check(lib.svt_b200_engine_lr_frame(engine, C.byref(p), n_units, C.byref(gs), lines), lib)
        assert_same(got, want, str(modes))


# ---- motion estimation -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["flat", "black"])
@pytest.mark.parametrize("preset", [8, 5])
def test_me_flat_pictures_vs_oracle(engine, kind, preset):
    """Every candidate of a reference has the same SAD: the direct entry and the engine entry against the oracle."""
    import gpu_runner as gr
    from test_engine_gpu import assert_me_result
    from test_me_presets_gpu import _engine_me
    from test_oracle_me_presets import structure
    lib = sb.load()
    w, h = 200, 136
    n0, n1, dist, tl = structure(preset, "ra")
    params = sb.me_params(preset, w, h, n0, n1, dist, tl, 1)
    geos, src, refs = cc.me_flat_case(w, h, kind)
    want = cm.run_oracle_me(params, src, refs)
    cm.assert_me_equal(gr.run_gpu_me(params, src, refs), want, params, f"{kind} preset {preset}")
    n_sb = ((w + 63) // 64) * ((h + 63) // 64)
    rc, got = _engine_me(lib, engine, params, src, refs, n_sb)
    sb.check(rc, lib)
    assert_me_result(got, want, n_sb, f"engine {kind} preset {preset}")
