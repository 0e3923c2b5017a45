"""The transform kernels at the edges of their range, bit-exact against the CPU oracle (tests/test_oracle_txfm_edges.py
pins it to the reference there): the fused per-unit entry with the reference's quantiser tables on full-range content,
partly filled CTAs, odd padding and odd chroma widths (unaligned samples), an in-place reconstruction, the drop-ins on
saturated residuals, in partial-frequency form and at 12 bits, and the open-loop intra search on flat, saturated,
hard-edged and odd-sized pictures.  Each case also checks, from the oracle's intermediates, that it reaches the clamp or
path it exists for (txfm_edge_cases.py)."""
import ctypes as C

import numpy as np
import pytest

import common as cm
import content_cases as cc
import svtb200 as sb
import txfm_edge_cases as ec
from test_oracle_txfm import TX_H, TX_W, allowed_types
from test_oracle_txfm_edges import INT16_CLAMP_SIZES, saturating_coeffs
from test_txfm_gpu import oracle_encode_tus, oracle_encode_tus_ex

pytestmark = pytest.mark.gpu

W, H = 192, 128


def cul_of(levels):
    """cul_level of av1_quantize_inv_quantize from the levels of each unit (see test_encode_tus_vs_oracle)."""
    return np.array([min(63, int(np.abs(q.astype(np.int64)).sum())) + (64 if q[0] < 0 else 128 if q[0] > 0 else 0)
                     for q in levels], np.int32)


def run_fused(p, src, pred, tus, slack=0, in_place=False):
    """svt_b200_encode_tus_cul with `slack` units of sentinels past the outputs (qcoeff 77, eob 0x7777, cul_level -7);
    in_place: the reconstruction is written into the prediction frame.  Returns recon, levels, eob, cul_level and the
    sentinel tails."""
    import torch
    import gpu_runner as gr
    lib = sb.load()
    n = min(TX_W[p.tx_size], 32) * min(TX_H[p.tx_size], 32)
    m = len(tus) + slack
    ds, dp = gr.DevYuv(src), gr.DevYuv(pred)
    dr = dp if in_place else gr.DevYuv(pred.copy())
    arr = (sb.Tu * len(tus))(*tus)
    dt = torch.from_numpy(np.frombuffer(arr, dtype=np.int32).copy()).cuda()
    q = torch.full((m * n,), 77, dtype=torch.int32, device="cuda")
    eob = torch.full((m,), 0x7777, dtype=torch.int16, device="cuda")
    cul = torch.full((m,), -7, dtype=torch.int32, device="cuda")
    ss, ps, rs = ds.struct(), dp.struct(), dr.struct()
    sb.check(lib.svt_b200_encode_tus_cul(C.byref(p), C.byref(ss), C.byref(ps), C.byref(rs), C.c_void_p(dt.data_ptr()), len(tus),
                                         C.c_void_p(q.data_ptr()), C.c_void_p(eob.data_ptr()), C.c_void_p(cul.data_ptr()), None), lib)
    torch.cuda.synchronize()
    qh, eh, ch = q.cpu().numpy(), eob.cpu().numpy().view(np.uint16), cul.cpu().numpy()
    k = len(tus)
    return dr.download(), qh[:k * n].reshape(k, n), eh[:k], ch[:k], (qh[k * n:], eh[k:], ch[k:])


def assert_fused_equal(got, want, what=""):
    got_rec, got_q, got_eob, got_cul = got[:4]
    want_rec, want_q, want_eob = want
    np.testing.assert_array_equal(got_eob, want_eob, err_msg=f"{what} eob")
    np.testing.assert_array_equal(got_q, want_q, err_msg=f"{what} levels")
    np.testing.assert_array_equal(got_cul, cul_of(want_q), err_msg=f"{what} cul_level")
    for i in range(3):
        np.testing.assert_array_equal(got_rec.plane(i), want_rec.plane(i), err_msg=f"{what} plane {i}")


@pytest.mark.parametrize("tx_size", range(19))
@pytest.mark.parametrize("bd,use_fp", [(8, 0), (8, 1), (10, 0), (10, 1)])
def test_fused_full_range_real_tables(tx_size, bd, use_fp):
    """Saturated, full-swing and hard-edged content against its complement at qindex 0 and 255: at 255 every size
    clips its reconstruction and the 8-bit sizes of INT16_CLAMP_SIZES have levels that the quantiser's int16 clamp
    changes."""
    reach = ec.Reach()
    for kind in ("full_swing", "saturated", "hard_edges"):
        src, pred = ec.pair(kind, W, H, bd, seed=tx_size)
        for qindex in (0, 255):
            p = ec.encode_params(tx_size, bd, qindex, use_fp)
            tus = ec.corner_tus(np.random.default_rng(tx_size), tx_size, W, H, limit=24)
            want = oracle_encode_tus(p, src, pred, tus, use_fp)
            got = run_fused(p, src, pred, tus)
            assert_fused_equal(got, want, f"{kind} qindex {qindex}")
            if qindex == 255:
                reach += ec.chain_reach(p, src, pred, tus, use_fp)
    assert reach.recon_clip > 0, reach
    assert (reach.int16_clamp > 0) == (bd == 8 and tx_size in INT16_CLAMP_SIZES[use_fp]), reach


@pytest.mark.parametrize("tx_size", range(19))
def test_fused_partly_filled_ctas(tx_size):
    """n_tus of 1, one short of a full CTA, one past it and one short of three: nothing is written past n_tus (sentinels
    stay), samples outside the listed units keep the prediction, and the listed units match the oracle."""
    bd = 8 if tx_size % 2 == 0 else 10
    k = ec.bpc(tx_size)
    src, pred = ec.pair("saturated", W, H, bd, seed=50 + tx_size)
    rng = np.random.default_rng(50 + tx_size)
    every = ec.corner_tus(rng, tx_size, W, H)
    every = [every[int(i)] for i in rng.permutation(len(every))]
    w, h = TX_W[tx_size], TX_H[tx_size]
    for n_tus in sorted({1, k - 1, k + 1, 3 * k - 1}):
        assert n_tus % k and n_tus <= len(every)  # the last CTA is partly filled
        tus = every[:n_tus]
        p = ec.encode_params(tx_size, bd, 128, tx_size % 3 == 0)
        want = oracle_encode_tus(p, src, pred, tus, p.use_fp)
        got = run_fused(p, src, pred, tus, slack=k + 1)
        assert_fused_equal(got, want, f"n_tus {n_tus}")
        tq, te, tc = got[4]
        assert (tq == 77).all() and (te == 0x7777).all() and (tc == -7).all(), f"n_tus {n_tus}: written past the last unit"
        for pl in range(3):
            outside = np.ones(pred.plane(pl).shape, bool)
            for t in tus:
                if t.plane == pl:
                    outside[t.y:t.y + h, t.x:t.x + w] = False
            np.testing.assert_array_equal(got[0].plane(pl)[outside], pred.plane(pl)[outside], err_msg=f"n_tus {n_tus} plane {pl}")


ODD_W, ODD_H, ODD_PAD = 198, 130, 13  # chroma 99x65, chroma stride 125: rows alternate in alignment


@pytest.mark.parametrize("bd", [8, 10])
def test_fused_odd_layout_and_in_place(bd):
    """Odd padding and odd chroma widths through svt_b200_encode_tus_cul for every size, units touching the right and
    bottom edge of every plane, most of them with a first sample that is not 4-byte aligned; one run per size writes the
    reconstruction into the prediction frame."""
    misaligned = 0
    for ts in range(19):
        src, pred = ec.pair("full_swing", ODD_W, ODD_H, bd, seed=70 + ts, pad=ODD_PAD)
        rng = np.random.default_rng(70 + ts)
        tus = ec.corner_tus(rng, ts, ODD_W, ODD_H, limit=16)
        assert ec.edge_planes(src, tus, ts) == {0, 1, 2}, ts
        misaligned += ec.misaligned_units(src, tus)
        p = ec.encode_params(ts, bd, 255 if ts % 2 else 128, ts % 3 == 1)
        want = oracle_encode_tus(p, src, pred, tus, p.use_fp)
        assert_fused_equal(run_fused(p, src, pred, tus), want, f"size {ts}")
        assert_fused_equal(run_fused(p, src, pred, tus, in_place=True), want, f"size {ts} in place")
    assert misaligned > 0


@pytest.mark.parametrize("bd,use_fp", [(8, 0), (10, 1)])
def test_fused_ex_odd_layout(bd, use_fp):
    """svt_b200_encode_tus_ex on the odd layout: mixed sizes, shapes and the reference's tables at qindex 0, 1, 128 and
    255 as four quantiser sets, in cells tiled from the bottom-right corner of every plane."""
    import gpu_runner as gr
    src, pred = ec.pair("saturated", ODD_W, ODD_H, bd, seed=90 + bd, pad=ODD_PAD)
    qsets = [[ec.quant_plane(bd, q) for _ in range(3)] for q in ec.QINDEXES]
    tus = ec.corner_mixed_tus(np.random.default_rng(90 + bd), ODD_W, ODD_H, len(qsets))
    assert ec.misaligned_units(src, tus) > 0
    corner = {t.plane for t in tus if (t.x + TX_W[t.tx_size], t.y + TX_H[t.tx_size]) == ec.plane_dims(ODD_W, ODD_H, t.plane)}
    assert corner == {0, 1, 2}
    want_rec, want_q, want_eob = oracle_encode_tus_ex(qsets, src, pred, tus, use_fp)
    got_rec, got_q, got_eob, got_cul, tail = gr.run_gpu_encode_tus_ex(qsets, use_fp, src, pred, tus)
    np.testing.assert_array_equal(got_eob, want_eob)
    for i, (g, wq) in enumerate(zip(got_q, want_q)):
        np.testing.assert_array_equal(g, wq, err_msg=f"unit {i}: size {tus[i].tx_size} shape {tus[i].pf_shape}")
    assert (tail == 77).all()
    np.testing.assert_array_equal(got_cul, cul_of(want_q))
    for i in range(3):
        np.testing.assert_array_equal(got_rec.plane(i), want_rec.plane(i), err_msg=f"plane {i}")


@pytest.mark.parametrize("qindex", ec.QINDEXES)
def test_quantizer_dropins_real_tables(qindex):
    """The quantiser drop-ins (the fused kernel's quant_one) with the reference's tables on coefficients at the forward
    transform's extremes and a little past them; at qindex 255 the int16 clamp of quantize_b and quantize_fp changes
    levels (the fused cases cannot reach that for quantize_b)."""
    lib, orc = sb.load(), cm.oracle()
    rng = np.random.default_rng(500 + qindex)
    variants = [("svt_aom_quantize_b_cuda", "b", 0, None), ("svt_aom_highbd_quantize_b_cuda", "b", 1, None),
                ("svt_av1_quantize_fp_cuda", "fp", 0, 0), ("svt_av1_quantize_fp_32x32_cuda", "fp", 0, 1),
                ("svt_av1_quantize_fp_64x64_cuda", "fp", 0, 2), ("svt_av1_highbd_quantize_fp_cuda", "fph", 1, None)]
    clamped = {"b": 0, "fp": 0, "hbd": 0}
    for name, kind, hbd, fixed_ls in variants:
        f = getattr(lib, name)
        bd = 10 if hbd else 8
        qa = ec.quant_arrays(bd, qindex)
        for n, ls in ((16, 0), (256, 0), (1024, 1), (1024, 2)):
            ls = ls if fixed_ls is None else fixed_ls
            coeff = saturating_coeffs(rng, n, bd)
            scan = rng.permutation(n).astype(np.int16)
            clamped["hbd" if hbd else kind] += ec.quant_reach(coeff, qa, ls, bd, kind != "b")
            rnd, quant = (qa["round"], qa["quant"]) if kind == "b" else (qa["round_fp"], qa["quant_fp"])
            q0, d0, e0 = np.full(n, 7, np.int32), np.full(n, 7, np.int32), C.c_uint16(9)
            q1, d1, e1 = np.full(n, 7, np.int32), np.full(n, 7, np.int32), C.c_uint16(9)
            base = [cm.ptr(coeff), C.c_ssize_t(n), cm.ptr(qa["zbin"]), cm.ptr(rnd), cm.ptr(quant), cm.ptr(qa["quant_shift"]),
                    cm.ptr(q0), cm.ptr(d0), cm.ptr(qa["dequant"]), C.byref(e0), cm.ptr(scan), cm.ptr(scan)]
            if kind == "b":
                f(*base, None, None, ls)
                orc.orc_quantize_b(cm.ptr(coeff), C.c_ssize_t(n), cm.ptr(qa["zbin"]), cm.ptr(rnd), cm.ptr(quant),
                                   cm.ptr(qa["quant_shift"]), cm.ptr(q1), cm.ptr(d1), cm.ptr(qa["dequant"]), C.byref(e1),
                                   cm.ptr(scan), None, None, ls, hbd)
            else:
                if kind == "fph":
                    f(*base, C.c_int16(ls))
                else:
                    f(*base)
                orc.orc_quantize_fp(cm.ptr(coeff), C.c_ssize_t(n), cm.ptr(rnd), cm.ptr(quant), cm.ptr(q1), cm.ptr(d1),
                                    cm.ptr(qa["dequant"]), C.byref(e1), cm.ptr(scan), ls, hbd)
            np.testing.assert_array_equal(q0, q1, err_msg=f"{name} n={n} ls={ls}")
            np.testing.assert_array_equal(d0, d1, err_msg=f"{name} n={n} ls={ls}")
            assert e0.value == e1.value, (name, n, ls)
    if qindex == 255:
        assert clamped["b"] > 0 and clamped["fp"] > 0, clamped


@pytest.mark.parametrize("tx_size", range(19))
def test_partial_frequency_dropins_every_type(tx_size):
    """N2 / N4 forward drop-ins for every allowed type at 8 and 10 bits, on random and saturated residuals."""
    lib, orc = sb.load(), cm.oracle()
    w, h = TX_W[tx_size], TX_H[tx_size]
    rng = np.random.default_rng(600 + tx_size)
    for shape, sh in (("N2", 1), ("N4", 2)):
        f = getattr(lib, f"svt_av1_fwd_txfm2d_{w}x{h}_{shape}_cuda")
        for bd in (8, 10):
            for tx_type in allowed_types(tx_size):
                kind = ec.RESIDUALS[tx_type % 4]
                for res in (rng.integers(-ec.maxv(bd), ec.maxv(bd) + 1, (h, w + 5)).astype(np.int16),
                            ec.residual(kind, w, h, bd, rng, stride=w + 5)):
                    want, got = np.zeros(w * h, np.int32), np.full(w * h, 3, np.int32)
                    orc.orc_fwd_txfm2d_pf(cm.ptr(res), cm.ptr(want), C.c_uint32(w + 5), tx_type, tx_size, bd, sh)
                    f(cm.ptr(res), cm.ptr(got), C.c_uint32(w + 5), tx_type, C.c_uint8(bd))
                    np.testing.assert_array_equal(got, want, err_msg=f"{shape} type {tx_type} bd {bd}")


@pytest.mark.parametrize("tx_size", range(19))
def test_fwd_dropins_saturated_every_type(tx_size):
    """The forward drop-ins on flat +-max, checkerboard and random-sign residuals for types 1-15 (DCT_DCT too at the
    sizes that allow only it), at 8, 10 and 12 bits."""
    lib, orc = sb.load(), cm.oracle()
    w, h = TX_W[tx_size], TX_H[tx_size]
    f = getattr(lib, f"svt_av1_fwd_txfm2d_{w}x{h}_cuda")
    rng = np.random.default_rng(700 + tx_size)
    for bd in (8, 10, 12):
        for tx_type in [t for t in allowed_types(tx_size) if t] or [0]:
            for kind in ec.RESIDUALS:
                res = ec.residual(kind, w, h, bd, rng, stride=w + 5)
                want, got = np.zeros(w * h, np.int32), np.zeros(w * h, np.int32)
                orc.orc_fwd_txfm2d(cm.ptr(res), cm.ptr(want), C.c_uint32(w + 5), tx_type, tx_size, bd)
                f(cm.ptr(res), cm.ptr(got), C.c_uint32(w + 5), tx_type, C.c_uint8(bd))
                np.testing.assert_array_equal(got, want, err_msg=f"type {tx_type} bd {bd} {kind}")


def call_inv_dropin(lib, tx_size, coeff, pred, stride_r, rec, stride_w, tx_type, bd):
    w, h = TX_W[tx_size], TX_H[tx_size]
    f = getattr(lib, f"svt_av1_inv_txfm2d_add_{w}x{h}_cuda")
    if w == h:
        f(cm.ptr(coeff), cm.ptr(pred), stride_r, cm.ptr(rec), stride_w, tx_type, bd)
    elif (w, h) in ((4, 8), (8, 4), (4, 16), (16, 4)):
        f(cm.ptr(coeff), cm.ptr(pred), stride_r, cm.ptr(rec), stride_w, tx_type, tx_size, bd)
    else:
        f(cm.ptr(coeff), cm.ptr(pred), stride_r, cm.ptr(rec), stride_w, tx_type, tx_size, w * h, bd)


@pytest.mark.parametrize("tx_size", range(19))
def test_inv_dropins_12bit(tx_size):
    """The inverse drop-ins at bit depth 12 (ranges 20 / 18): random coefficients past the 20-bit input clamp and the
    forward transform of saturated residuals, on a random prediction (the sum leaves [0, 4095])."""
    lib, orc = sb.load(), cm.oracle()
    w, h = TX_W[tx_size], TX_H[tx_size]
    iw, ih = min(w, 32), min(h, 32)
    rng = np.random.default_rng(800 + tx_size)
    bd = 12
    clamped = clipped = 0
    for tx_type in allowed_types(tx_size):
        for kind in ("big",) + ec.RESIDUALS:
            if kind == "big":
                coeff = rng.integers(-(1 << (bd + 9)), 1 << (bd + 9), iw * ih).astype(np.int32)
            else:
                full = np.zeros(w * h, np.int32)
                orc.orc_fwd_txfm2d(cm.ptr(ec.residual(kind, w, h, bd, rng)), cm.ptr(full), C.c_uint32(w), tx_type, tx_size, bd)
                coeff = np.ascontiguousarray(full.reshape(h, w)[:ih, :iw]).reshape(-1)
            clamped += ec.inv_input_reach(coeff, tx_size, bd)
            pred = rng.integers(0, 1 << bd, (h, w + 3)).astype(np.uint16)
            v = pred[:, :w].astype(np.int64) + ec.inverse_residual(coeff, tx_size, tx_type, bd)
            clipped += int(((v < 0) | (v > ec.maxv(bd))).sum())
            want, got = np.zeros((h, w + 7), np.uint16), np.zeros((h, w + 7), np.uint16)
            orc.orc_inv_txfm2d_add(cm.ptr(coeff), cm.ptr(pred), w + 3, cm.ptr(want), w + 7, tx_type, tx_size, bd)
            call_inv_dropin(lib, tx_size, coeff, pred, w + 3, got, w + 7, tx_type, bd)
            np.testing.assert_array_equal(got, want, err_msg=f"type {tx_type} {kind}")
    assert clamped > 0 and clipped > 0


# ---- open-loop intra search --------------------------------------------------------------------------------------
def ois_all(pic):
    """Costs of svt_b200_ois_dc_picture, svt_b200_ois_dc_picture_host and the oracle for one 8-bit picture."""
    import torch
    import gpu_runner as gr
    lib, orc = sb.load(), cm.oracle()
    w, h = pic.w, pic.h
    mbw, mbh = (w + 15) // 16, (h + 15) // 16
    pad = np.ascontiguousarray(np.pad(pic.plane(0), ((0, mbh * 16 - h + 16), (0, mbw * 16 - w + 16)), mode="edge"))
    want = np.zeros(mbw * mbh, np.int64)
    orc.orc_ois_dc_picture(cm.ptr(pad), pad.shape[1], w, h, cm.ptr(want))
    d = gr.DevYuv(pic)
    got = torch.full((mbw * mbh,), -5, dtype=torch.int64, device="cuda")
    st = d.struct()
    sb.check(lib.svt_b200_ois_dc_picture(C.byref(st), got.data_ptr(), None), lib)
    torch.cuda.synchronize()
    host = np.full(mbw * mbh, -5, np.int64)
    y = np.ascontiguousarray(pic.plane(0))
    sb.check(lib.svt_b200_ois_dc_picture_host(cm.ptr(y), y.shape[1], w, h, cm.ptr(host)), lib)
    return got.cpu().numpy().reshape(mbh, mbw), host.reshape(mbh, mbw), want.reshape(mbh, mbw)


def flat_dc_cost(v):
    """|DC| of the 16x16 forward DCT_DCT of a flat residual v (every other coefficient is 0): the columns (input << 2,
    cos_bit 13: the butterflies add exactly, so the DC is one half_btf of two sums of 8 samples) then >> 2 with rounding,
    then the rows (cos_bit 12)."""
    col = (5793 * 16 * (v << 2) + (1 << 12)) >> 13
    col = (col + 2) >> 2
    return abs((2896 * 16 * col + (1 << 11)) >> 12)


@pytest.mark.parametrize("level", ["zero", "mid", "max"])
@pytest.mark.parametrize("geom", [(64, 48), (160, 96)])
def test_ois_flat_closed_form(level, geom):
    """Flat pictures with sides that are multiples of 16: the top-left macroblock is predicted at 128, every other one
    from neighbours equal to itself, so a flat mid picture costs 0 everywhere and flat 0 / max pictures cost
    |DC(v - 128)| in the top-left macroblock only."""
    w, h = geom
    pic = cc.flat(w, h, 8, level)
    v = int(pic.plane(0)[0, 0])
    want = np.zeros((h // 16, w // 16), np.int64)
    want[0, 0] = flat_dc_cost(v - 128)
    assert (want[0, 0] == 0) == (level == "mid")
    for got in ois_all(pic):
        np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("kind", ["saturated", "hard_edges", "flat_max", "flat_zero"])
@pytest.mark.parametrize("geom", [(192, 128), (201, 119)])
def test_ois_content_and_odd_sizes(kind, geom):
    """Saturated and hard-edged pictures (the 16x16 DCT near its largest values) and flat ones, at a size with partial
    edge macroblocks (201x119: the reference's 127 / 129 fill there), through both entries, against the oracle."""
    w, h = geom
    pic = cc.PICTURES[kind](w, h, 8, 3)
    dev, host, want = ois_all(pic)
    np.testing.assert_array_equal(dev, want)
    np.testing.assert_array_equal(host, want)
    if kind in ("saturated", "hard_edges"):
        assert want.max() > flat_dc_cost(127)  # costlier than the largest flat block
