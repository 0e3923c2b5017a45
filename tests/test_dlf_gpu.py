"""GPU parity tests for the deblocking filter (CUDA through the C ABI vs the CPU oracle), bit-exact."""
import ctypes as C

import numpy as np
import pytest

import common as cm
import svtb200 as sb
from test_oracle_dlf import DLF_CASES, dlf_case, dlf_params, edge_cases

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("length", [4, 6, 8, 14])
@pytest.mark.parametrize("direction", ["horizontal", "vertical"])
def test_lpf_dropins(length, direction):
    """test/DeblockTest.cc: all 16 svt_aom_[highbd_]lpf_* pointers."""
    lib, orc = sb.load(), cm.oracle()
    for bd, img, blimit, limit, thresh in edge_cases(length, n=24):
        hbd = bd > 8
        f = getattr(lib, f"svt_aom_{'highbd_' if hbd else ''}lpf_{direction}_{length}_cuda")
        a = img.astype(np.uint16 if hbd else np.uint8)
        b = a.copy()
        off = (16 * 32 + 16) * a.itemsize
        bl, li, th = (np.full(16, v, np.uint8) for v in (blimit & 255, limit, thresh))
        if hbd:
            f(C.c_void_p(a.ctypes.data + off), 32, cm.ptr(bl), cm.ptr(li), cm.ptr(th), bd)
        else:
            f(C.c_void_p(a.ctypes.data + off), 32, cm.ptr(bl), cm.ptr(li), cm.ptr(th))
        vert = direction == "vertical"
        orc.orc_lpf_edge(C.c_void_p(b.ctypes.data + off), int(hbd), 1 if vert else 32, 32 if vert else 1, length,
                         blimit & 255, limit, thresh, bd)
        np.testing.assert_array_equal(a, b)


def flat_mi(mi_rows, mi_cols, part, levels):
    """Flattened mi summary built in Python the same way the reference-side helper does (tests/test_oracle_dlf.py
    checks that helper against the reference when oracle/_ref is present)."""
    TXW = [4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64]
    TXH = [4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16]
    BW = {0: 4, 1: 4, 2: 8, 3: 8, 4: 8, 5: 16, 6: 16, 7: 16, 8: 32, 9: 32, 10: 32, 11: 64, 12: 64, 16: 4, 17: 16, 18: 8, 19: 32, 20: 16, 21: 64}
    BH = {0: 4, 1: 8, 2: 4, 3: 8, 4: 16, 5: 8, 6: 16, 7: 32, 8: 16, 9: 32, 10: 64, 11: 32, 12: 64, 16: 16, 17: 4, 18: 32, 19: 8, 20: 64, 21: 16}
    D = [[0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 11, 12, 4, 4, 4, 4, 13, 14, 15, 16, 17, 18],
         [0, 5, 6, 0, 1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4, 5, 6, 7, 8, 9, 10],
         [0, 5, 6, 1, 0, 0, 0, 1, 1, 1, 2, 2, 2, 4, 4, 4, 0, 0, 1, 1, 2, 2]]
    sbt, dep, inter, skip = part
    flat = (sb.DlfMi * (mi_rows * mi_cols))()
    for r in range(mi_rows):
        for c in range(mi_cols):
            f = flat[r * mi_cols + c]
            bs, d, it, sk = int(sbt[r, c]), int(dep[r, c]), int(inter[r, c]), int(skip[r, c])
            tx = D[0][bs] if it else D[d][bs]
            if it and not sk:
                tx = D[d][bs]
            cw, ch = max(BW[bs] // 2, 4), max(BH[bs] // 2, 4)
            f.tx_w[0], f.tx_h[0] = TXW[tx], TXH[tx]
            f.tx_w[1], f.tx_h[1] = min(cw, 32), min(ch, 32)   # largest chroma transform of the block (<= 32)
            # rectangular 4:1 chroma blocks use the 2:1-limited transform of av1_get_max_uv_txsize
            f.blk_w[0], f.blk_h[0], f.blk_w[1], f.blk_h[1] = BW[bs], BH[bs], cw, ch
            f.skip_inter = sk and it
            f.lvl_y[0], f.lvl_y[1], f.lvl_u, f.lvl_v = levels
            f.lvl_class = (1 * 2 + 1) if it else 0   # segment 0, LAST_FRAME / NEARESTMV-class or INTRA_FRAME
    return flat


@pytest.mark.parametrize("case", DLF_CASES + [(1920, 1080, 8, 9, (24, 20, 14, 10), 1), (640, 360, 10, 10, (40, 40, 30, 30), 0)])
def test_dlf_frame_vs_oracle(case):
    import gpu_runner as gr
    w, h, bd, seed, levels, sharp = case
    mi_rows, mi_cols, part, frame = dlf_case(w, h, bd, seed, levels, sharp)
    if cm.have_ref():
        from test_oracle_dlf import run_ref_dlf
        _, flat = run_ref_dlf(mi_rows, mi_cols, part, frame, levels, sharp)
        mine = flat_mi(mi_rows, mi_cols, part, levels)
        assert bytes(flat) == bytes(mine), "python mi summary differs from the reference-side helper"
    else:
        flat = flat_mi(mi_rows, mi_cols, part, levels)
    p = dlf_params(mi_rows, mi_cols, levels, sharp)
    want = frame.copy()
    st = want.struct()
    cm.oracle().orc_dlf_frame(C.byref(p), C.byref(st), flat)
    got = gr.run_gpu_dlf(p, frame, flat)
    for i in range(3):
        np.testing.assert_array_equal(got.plane(i), want.plane(i), err_msg=f"plane {i}")
    # property: deblocking never increases the range of the picture and a level-0 call is the identity
    p0 = dlf_params(mi_rows, mi_cols, (0, 0, 0, 0), sharp)
    same = gr.run_gpu_dlf(p0, frame, flat)
    for i in range(3):
        np.testing.assert_array_equal(same.plane(i), frame.plane(i))


@pytest.mark.parametrize("case", DLF_CASES[:2])
def test_dlf_frame_misaligned_planes_vs_oracle(case):
    """Planes whose base and stride are not multiples of 4 samples (pad 17) take the line-per-thread kernel."""
    import gpu_runner as gr
    w, h, bd, seed, levels, sharp = case
    mi_rows, mi_cols, part, aligned = dlf_case(w, h, bd, seed, levels, sharp)
    frame = cm.Yuv(w, h, bd, pad=17)
    for i in range(3):
        frame.plane(i)[...] = aligned.plane(i)
    st = frame.struct()
    assert st.stride_y % 4 and st.stride_c % 4
    flat = flat_mi(mi_rows, mi_cols, part, levels)
    p = dlf_params(mi_rows, mi_cols, levels, sharp)
    want = frame.copy()
    ws = want.struct()
    cm.oracle().orc_dlf_frame(C.byref(p), C.byref(ws), flat)
    got = gr.run_gpu_dlf(p, frame, flat)
    for i in range(3):
        np.testing.assert_array_equal(got.plane(i), want.plane(i), err_msg=f"plane {i}")


def test_frame_sse():
    import gpu_runner as gr
    for (w, h, bd) in ((192, 136, 8), (640, 360, 10), (1920, 1080, 8)):
        a = cm.synth_yuv(w, h, 1, 3, bd)
        b = cm.degrade(a, 4)
        want = np.zeros(3, np.uint64)
        sa, sbb = a.struct(), b.struct()
        cm.oracle().orc_frame_sse(C.byref(sa), C.byref(sbb), cm.ptr(want))
        np.testing.assert_array_equal(gr.run_gpu_sse(a, b), want)


@pytest.mark.parametrize("case", [(192, 136, 8, 1, 0, 3, (20, 24, 12, 9), 0, None), (192, 136, 8, 2, 0, 1, (8, 8, 4, 4), 0, None),
                                  (128, 128, 10, 3, 1, 3, (40, 40, 33, 20), 1, None), (264, 72, 8, 4, 0, 2, (0, 0, 0, 0), 0, None),
                                  (192, 136, 8, 5, 0, 3, (30, 30, 16, 16), 0, ((1, 0, 0, 0, -1, 0, -1, -1), (0, 0))),
                                  (1920, 1080, 8, 6, 0, 3, (24, 20, 14, 10), 0, None)])
def test_pick_filter_level_vs_oracle(case):
    """svt_av1_pick_filter_level: the searched levels equal the oracle's (itself pinned against the reference) and the
    reconstruction is left untouched, at small sizes and at the full 1080p geometry."""
    import gpu_runner as gr
    from test_oracle_dlf import pick_case, pick_params
    w, h, bd, seed, method, mode, last, only4, deltas = case
    mi_rows, mi_cols, part, src, rec = pick_case(w, h, bd, seed)
    flat = flat_mi(mi_rows, mi_cols, part, last)
    p = pick_params(mi_rows, mi_cols, method, mode, last, only4, deltas=deltas)
    r, t = rec.copy(), rec.copy()
    rs, ss, ts = r.struct(), src.struct(), t.struct()
    want = (C.c_int32 * 4)()
    cm.oracle().orc_pick_filter_level(C.byref(p), C.byref(rs), C.byref(ss), C.byref(ts), flat, want)
    got, after = gr.run_gpu_pick(p, rec, src, flat)
    assert got == list(want)
    for i in range(3):
        np.testing.assert_array_equal(after.plane(i), rec.plane(i))


@pytest.mark.parametrize("bd,key", [(8, 0), (8, 1), (10, 0), (10, 1), (12, 0), (12, 1)])
def test_pick_filter_level_from_q_and_minimal(bd, key):
    lib = sb.load()
    fr = sb.Frame(0, 0, 0, 0, 0, 64, 64, bd)
    for q in (4, 33, 120, 700, 1336, 5000, 21387):
        for method in (2, 3):
            p = sb.LpfPickParams()
            p.method, p.q_ac, p.key_frame = method, q, key
            for i in range(4):
                p.last_level[i] = 7 + i
            a, b = (C.c_int32 * 4)(), (C.c_int32 * 4)()
            sb.check(lib.svt_b200_pick_filter_level(C.byref(p), C.byref(fr), None, None, None, None, a, None), lib)
            cm.oracle().orc_pick_filter_level(C.byref(p), C.byref(fr), None, None, None, b)
            assert list(a) == list(b)
