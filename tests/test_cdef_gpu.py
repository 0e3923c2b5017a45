"""GPU parity tests for CDEF (CUDA through the C ABI vs the CPU oracle), bit-exact incl. the double-precision
luma distortion (0 ULP)."""
import ctypes as C

import numpy as np
import pytest

import common as cm
import svtb200 as sb
from test_oracle_cdef import cdef_picture_case, filter_block_cases, rand_tile

pytestmark = pytest.mark.gpu


def test_filter_block_dropin():
    lib = sb.load()
    n = 0
    for bd, mode, bsize, pri, sec, d, damp, tile in filter_block_cases():
        n += 1
        if n % 3:
            continue  # one launch per call: keep the sweep short
        inp = tile.ctypes.data + (3 * 144 + 8) * 2
        outs = []
        for f in (lib.svt_cdef_filter_block_cuda, cm.oracle().orc_cdef_filter_block):
            d8, d16 = np.zeros((8, 8), np.uint8), np.zeros((8, 8), np.uint16)
            if bd == 8:
                f(cm.ptr(d8), None, 8, C.c_void_p(inp), pri, sec, d, damp, damp, bsize, bd - 8)
            else:
                f(None, cm.ptr(d16), 8, C.c_void_p(inp), pri, sec, d, damp, damp, bsize, bd - 8)
            outs.append((d8, d16))
        np.testing.assert_array_equal(outs[0][0], outs[1][0])
        np.testing.assert_array_equal(outs[0][1], outs[1][1])


def test_find_dir_dropin():
    lib = sb.load()
    rng = np.random.default_rng(2)
    for bd in (8, 10, 12):
        for mode in ("random", "smooth"):
            for _ in range(6):
                tile = rand_tile(rng, bd, mode)
                va, vb = C.c_int32(0), C.c_int32(0)
                a = lib.svt_cdef_find_dir_cuda(cm.ptr(tile), 144, C.byref(va), bd - 8)
                b = cm.oracle().orc_cdef_find_dir(cm.ptr(tile), 144, C.byref(vb), bd - 8)
                assert (a, va.value) == (b, vb.value)


@pytest.mark.parametrize("case", [(192, 136, 8, 3), (192, 136, 10, 3), (200, 72, 8, 0), (136, 128, 10, 1),
                                  (1920, 1080, 8, 3), (640, 360, 10, 2)])
def test_cdef_search_vs_oracle(case):
    import gpu_runner as gr
    w, h, bd, pick = case
    src, rec, mi_rows, mi_cols, skip = cdef_picture_case(w, h, bd)
    p = sb.CdefSearchParams()
    p.mi_rows, p.mi_cols, p.pri_damping = mi_rows, mi_cols, 3 + (172 >> 6)
    assert sb.load().svt_b200_cdef_strength_table(pick, C.byref(p)) == {0: 64, 1: 32, 2: 20, 3: 10}[pick]
    po = sb.CdefSearchParams()
    cm.oracle().orc_cdef_strength_table(pick, C.byref(po))
    assert list(p.pri_strength) == list(po.pri_strength) and list(p.sec_strength) == list(po.sec_strength)
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    want = np.zeros((2, nfb, 64), np.uint64)
    rs, ss = rec.struct(), src.struct()
    cm.oracle().orc_cdef_search(C.byref(p), C.byref(rs), C.byref(ss), cm.ptr(skip), skip.shape[1], cm.ptr(want))
    got = gr.run_gpu_cdef_search(p, rec, src, skip)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("case", [(192, 136, 8), (200, 72, 10), (640, 360, 10)])
def test_cdef_search_arbitrary_table(case):
    """A strength list that is NOT a pri x sec grid takes the list form of the search kernel (one pass per strength)."""
    import gpu_runner as gr
    w, h, bd = case
    src, rec, mi_rows, mi_cols, skip = cdef_picture_case(w, h, bd, seed=5)
    p = sb.CdefSearchParams()
    p.mi_rows, p.mi_cols, p.pri_damping = mi_rows, mi_cols, 5
    pris, secs = (0, 3, 3, 7, 15, 1, 0), (0, 1, 4, 2, 0, 4, 2)
    p.n_strengths = len(pris)
    for i, (a, b) in enumerate(zip(pris, secs)):
        p.pri_strength[i], p.sec_strength[i] = a, b
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    want = np.zeros((2, nfb, 64), np.uint64)
    rs, ss = rec.struct(), src.struct()
    cm.oracle().orc_cdef_search(C.byref(p), C.byref(rs), C.byref(ss), cm.ptr(skip), skip.shape[1], cm.ptr(want))
    got = gr.run_gpu_cdef_search(p, rec, src, skip)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("case", [(192, 136, 8), (192, 136, 10), (264, 72, 8), (1920, 1080, 8)])
def test_cdef_apply_vs_oracle(case):
    import gpu_runner as gr
    w, h, bd = case
    src, rec, mi_rows, mi_cols, skip = cdef_picture_case(w, h, bd, seed=21)
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    idx = np.random.default_rng(4).integers(-1, 8, nfb).astype(np.int8)
    p = sb.CdefApplyParams()
    p.mi_rows, p.mi_cols, p.damping = mi_rows, mi_cols, 5
    for i, (a, b) in enumerate(zip((0, 5, 17, 63, 40, 2, 12, 33), (0, 0, 9, 62, 4, 1, 60, 3))):
        p.y_strength[i], p.uv_strength[i] = a, b
    want = rec.copy()
    rs, ws = rec.struct(), want.struct()
    cm.oracle().orc_cdef_apply(C.byref(p), C.byref(rs), C.byref(ws), cm.ptr(skip), skip.shape[1], cm.ptr(idx))
    got = gr.run_gpu_cdef_apply(p, rec, skip, idx)
    for i in range(3):
        np.testing.assert_array_equal(got.plane(i), want.plane(i), err_msg=f"plane {i}")
    # idempotence property at full size: strength-0 everywhere leaves the picture untouched
    p0 = sb.CdefApplyParams()
    p0.mi_rows, p0.mi_cols, p0.damping = mi_rows, mi_cols, 5
    same = gr.run_gpu_cdef_apply(p0, rec, skip, np.zeros(nfb, np.int8))
    for i in range(3):
        np.testing.assert_array_equal(same.plane(i), rec.plane(i))


@pytest.mark.parametrize("case", [(0, 3, 68, 120, "smooth"), (1, 3, 68, 120, "rand"), (2, 2, 45, 80, "smooth"), (3, 1, 45, 80, "ties"),
                                  (4, 0, 34, 46, "smooth"), (5, 3, 16, 16, "rand"), (6, 3, 90, 160, "ties"), (7, 3, 270, 480, "smooth"),
                                  (8, 2, 540, 960, "rand")])
def test_cdef_decide_vs_oracle(case):
    """svt_b200_cdef_decide (finish_cdef_search on the device) on synthetic mse tables: all four strength tables (10 / 20 /
    32 / 64 entries: 100 to 4096 candidate pairs per search step), ties, skipped filter blocks, up to 2160p geometry."""
    import ctypes as C
    import torch
    from test_oracle_cdef_decide import decide_case
    seed, pick, mi_rows, mi_cols, kind = case
    lib, orc = sb.load(), cm.oracle()
    p = sb.CdefDecideParams()
    n = lib.svt_b200_cdef_decide_table(pick, C.byref(p))
    p.mi_rows, p.mi_cols, p.lambda_ = mi_rows, mi_cols, 1000 + 977 * seed
    skip, stride, mse = decide_case(seed, mi_rows, mi_cols, n, kind)
    nfb = mse.shape[1]
    want, want_idx = sb.CdefDecision(), np.zeros(nfb, np.int8)
    orc.orc_cdef_decide(C.byref(p), cm.ptr(mse), cm.ptr(skip), stride, C.byref(want), cm.ptr(want_idx))
    dm, dsk = torch.from_numpy(mse.view(np.int64)).cuda(), torch.from_numpy(skip).cuda()
    dout = torch.zeros(C.sizeof(sb.CdefDecision), dtype=torch.uint8, device="cuda")
    didx = torch.full((nfb,), 77, dtype=torch.int8, device="cuda")
    scr = torch.zeros(nfb * (16 + 16 * 64) + 64, dtype=torch.uint8, device="cuda")
    lib.svt_b200_cdef_decide.argtypes = [C.POINTER(sb.CdefDecideParams)] + [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    sb.check(lib.svt_b200_cdef_decide(C.byref(p), dm.data_ptr(), dsk.data_ptr(), stride, dout.data_ptr(), didx.data_ptr(), scr.data_ptr(), None), lib)
    torch.cuda.synchronize()
    got = sb.CdefDecision.from_buffer_copy(dout.cpu().numpy().tobytes())
    assert (got.cdef_bits, got.nb_cdef_strengths, got.sb_count) == (want.cdef_bits, want.nb_cdef_strengths, want.sb_count)
    k = want.nb_cdef_strengths
    assert list(got.y_index)[:k] == list(want.y_index)[:k] and list(got.uv_index)[:k] == list(want.uv_index)[:k]
    assert list(got.y_strength)[:k] == list(want.y_strength)[:k] and list(got.uv_strength)[:k] == list(want.uv_strength)[:k]
    np.testing.assert_array_equal(didx.cpu().numpy(), want_idx)
