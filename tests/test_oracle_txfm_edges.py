"""Pins the transform / quantisation oracle against the unmodified reference C path (oracle/_ref) at the edges of its range:
saturated residuals at bit depths 8, 10 and 12, the 12-bit inverse transform, the quantisers on saturating coefficients
with the reference's own tables (tests/golden/quant_tables.json), and that fixture against svt_av1_build_quantizer.

test_dct_dct_matches_float_dct needs no reference: the oracle's DCT_DCT at every size against a float64 orthonormal 2-D
DCT, scaled as the integer transform scales it."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import scipy.fft

import common as cm
import txfm_edge_cases as ec
from test_oracle_txfm import TX_H, TX_W, allowed_types, call_ref_inv, fwd_ref_name

needs_ref = pytest.mark.skipif(not cm.have_ref(), reason="oracle/_ref not built")

# fwd_txfm_shift_ls (EbTransforms.h): the forward 2-D transform's shifts per size (positive: left)
FWD_SHIFT = [(2, 0, 0), (2, -1, 0), (2, -2, 0), (2, -4, 0), (0, -2, -2), (2, -1, 0), (2, -1, 0), (2, -2, 0), (2, -2, 0),
             (2, -4, 0), (2, -4, 0), (0, -2, -2), (2, -4, -2), (2, -1, 0), (2, -1, 0), (2, -2, 0), (2, -2, 0), (0, -2, 0),
             (2, -4, 0)]


def test_dct_dct_matches_float_dct():
    """An AV1 DCT of n points is sqrt(n/2) times the orthonormal DCT-II; the 2-D transform adds the three shifts and,
    for 2:1 rectangles, a factor sqrt(2).  The integer result stays within the rounding of its half_btf stages
    (0.5 each, log2(w) + log2(h) of them, plus the same count of 2^-11 relative for the quantised cosines): a wrong
    shift (x2), rectangle scale (x sqrt 2), flip or transposition is off by many tolerances.  The cosines' error
    scales with the intermediate values, which the block's largest coefficient bounds, so the relative term uses that."""
    orc = cm.oracle()
    rng = np.random.default_rng(11)
    for ts in range(19):
        w, h = TX_W[ts], TX_H[ts]
        stages = np.log2(w) + np.log2(h)
        rect = w == 2 * h or h == 2 * w
        scale = 2.0 ** sum(FWD_SHIFT[ts]) * np.sqrt(w / 2) * np.sqrt(h / 2) * (np.sqrt(2) if rect else 1.0)
        for bd in (8, 10, 12):
            blocks = [rng.integers(-ec.maxv(bd), ec.maxv(bd) + 1, (h, w)).astype(np.int16) for _ in range(3)]
            blocks += [ec.residual(k, w, h, bd, rng) for k in ec.RESIDUALS]
            for res in blocks:
                got = np.zeros(w * h, np.int32)
                orc.orc_fwd_txfm2d(cm.ptr(res), cm.ptr(got), C.c_uint32(w), 0, ts, bd)
                want = scipy.fft.dctn(res.astype(np.float64), type=2, norm="ortho") * scale
                tol = stages * (1 + np.abs(want).max() * 2.0 ** -11)
                err = np.abs(got.reshape(h, w) - want)
                assert err.max() <= tol, f"{w}x{h} bd {bd}: error {err.max():.2f} at {np.unravel_index(err.argmax(), err.shape)}"


@needs_ref
@pytest.mark.parametrize("tx_size", range(19))
def test_fwd_txfm2d_saturated_matches_reference(tx_size):
    ref, orc = cm.ref(), cm.oracle()
    w, h = TX_W[tx_size], TX_H[tx_size]
    rng = np.random.default_rng(200 + tx_size)
    f = getattr(ref, fwd_ref_name(tx_size))
    for bd in (8, 10, 12):
        for tx_type in allowed_types(tx_size):
            for kind in ec.RESIDUALS:
                res = ec.residual(kind, w, h, bd, rng, stride=w + 3)
                want, got = np.zeros(w * h, np.int32), np.zeros(w * h, np.int32)
                f(cm.ptr(res), cm.ptr(want), C.c_uint32(w + 3), tx_type, C.c_uint8(bd))
                orc.orc_fwd_txfm2d(cm.ptr(res), cm.ptr(got), C.c_uint32(w + 3), tx_type, tx_size, bd)
                np.testing.assert_array_equal(got, want, err_msg=f"{w}x{h} type {tx_type} bd {bd} {kind}")


@needs_ref
@pytest.mark.parametrize("tx_size", range(19))
def test_inv_txfm2d_12bit_matches_reference(tx_size):
    """bd 12: the row / column ranges 20 / 18 and the input clamp at 20 bits, on random coefficients past that clamp
    and on the forward transform of saturated residuals."""
    ref, orc = cm.ref(), cm.oracle()
    w, h = TX_W[tx_size], TX_H[tx_size]
    iw, ih = min(w, 32), min(h, 32)
    rng = np.random.default_rng(300 + tx_size)
    bd = 12
    clamped = 0
    for tx_type in allowed_types(tx_size):
        for kind in ("big", "big") + ec.RESIDUALS:
            if kind == "big":
                coeff = rng.integers(-(1 << (bd + 9)), 1 << (bd + 9), iw * ih).astype(np.int32)
            else:
                full = np.zeros(w * h, np.int32)
                orc.orc_fwd_txfm2d(cm.ptr(ec.residual(kind, w, h, bd, rng)), cm.ptr(full), C.c_uint32(w), tx_type, tx_size, bd)
                coeff = np.ascontiguousarray(full.reshape(h, w)[:ih, :iw]).reshape(-1)
            clamped += ec.inv_input_reach(coeff, tx_size, bd)
            pred = rng.integers(0, 1 << bd, (h, w + 3)).astype(np.uint16)
            want, got = np.zeros((h, w + 7), np.uint16), np.zeros((h, w + 7), np.uint16)
            call_ref_inv(ref, tx_size, coeff, pred, w + 3, want, w + 7, tx_type, bd)
            orc.orc_inv_txfm2d_add(cm.ptr(coeff), cm.ptr(pred), w + 3, cm.ptr(got), w + 7, tx_type, tx_size, bd)
            np.testing.assert_array_equal(got, want, err_msg=f"{w}x{h} type {tx_type} bd {bd} {kind}")
    assert clamped > 0  # the 20-bit input clamp changed coefficients


def saturating_coeffs(rng, n, bd):
    """n coefficients around the forward transform's extremes: +-(2^15 - 1 - k) (the int16 clamp's edge at 8 bits),
    +-4x that (10 bits), small ones, and zeros."""
    top = 32767 if bd == 8 else 4 * 32767
    c = rng.choice([-1, 1], n) * np.where(rng.random(n) < 0.5, top - rng.integers(0, 2000, n), rng.integers(0, 3000, n))
    c[rng.random(n) < 0.1] = 0
    return c.astype(np.int32)


@needs_ref
@pytest.mark.parametrize("qindex", ec.QINDEXES)
def test_quantizers_saturating_match_reference(qindex):
    """quantize_b and quantize_fp, low and high bit depth, at every log scale, with the reference's tables on
    coefficients at the transform's extremes; at qindex 255 the low-bit-depth int16 clamp changes levels of both."""
    ref, orc = cm.ref(), cm.oracle()
    rng = np.random.default_rng(400 + qindex)
    variants = [("svt_aom_quantize_b", "b", 0, None), ("svt_aom_highbd_quantize_b", "b", 1, None),
                ("svt_av1_quantize_fp", "fp", 0, 0), ("svt_av1_quantize_fp_32x32", "fp", 0, 1),
                ("svt_av1_quantize_fp_64x64", "fp", 0, 2), ("svt_av1_highbd_quantize_fp", "fp", 1, None)]
    clamped = {"b": 0, "fp": 0}
    for name, kind, hbd, fixed_ls in variants:
        f = C.cast(C.c_void_p.in_dll(ref, name).value, C.CFUNCTYPE(None))
        bd = 10 if hbd else 8
        qa = ec.quant_arrays(bd, qindex)
        for n, ls in ((16, 0), (256, 0), (1024, 1), (1024, 2)):
            ls = ls if fixed_ls is None else fixed_ls
            coeff = saturating_coeffs(rng, n, bd)
            scan = rng.permutation(n).astype(np.int16)
            clamped[kind] += ec.quant_reach(coeff, qa, ls, bd, kind == "fp")
            outs = []
            for which in (0, 1):
                q, d, eob = np.full(n, 77, np.int32), np.full(n, 77, np.int32), C.c_uint16(9)
                if kind == "b" and which == 0:
                    f(cm.ptr(coeff), C.c_ssize_t(n), cm.ptr(qa["zbin"]), cm.ptr(qa["round"]), cm.ptr(qa["quant"]),
                      cm.ptr(qa["quant_shift"]), cm.ptr(q), cm.ptr(d), cm.ptr(qa["dequant"]), C.byref(eob), cm.ptr(scan),
                      cm.ptr(scan), None, None, ls)
                elif kind == "b":
                    orc.orc_quantize_b(cm.ptr(coeff), C.c_ssize_t(n), cm.ptr(qa["zbin"]), cm.ptr(qa["round"]), cm.ptr(qa["quant"]),
                                       cm.ptr(qa["quant_shift"]), cm.ptr(q), cm.ptr(d), cm.ptr(qa["dequant"]), C.byref(eob),
                                       cm.ptr(scan), None, None, ls, hbd)
                elif which == 0:
                    args = [cm.ptr(coeff), C.c_ssize_t(n), cm.ptr(qa["zbin"]), cm.ptr(qa["round_fp"]), cm.ptr(qa["quant_fp"]),
                            cm.ptr(qa["quant_shift"]), cm.ptr(q), cm.ptr(d), cm.ptr(qa["dequant"]), C.byref(eob), cm.ptr(scan),
                            cm.ptr(scan)]
                    f(*(args + [C.c_int16(ls)] if hbd else args))
                else:
                    orc.orc_quantize_fp(cm.ptr(coeff), C.c_ssize_t(n), cm.ptr(qa["round_fp"]), cm.ptr(qa["quant_fp"]), cm.ptr(q),
                                        cm.ptr(d), cm.ptr(qa["dequant"]), C.byref(eob), cm.ptr(scan), ls, hbd)
                outs.append((q, d, eob.value))
            np.testing.assert_array_equal(outs[0][0], outs[1][0], err_msg=f"{name} n={n} ls={ls}")
            np.testing.assert_array_equal(outs[0][1], outs[1][1], err_msg=f"{name} n={n} ls={ls}")
            assert outs[0][2] == outs[1][2], (name, n, ls)
    if qindex == 255:
        assert clamped["b"] > 0 and clamped["fp"] > 0, clamped


@needs_ref
def test_quant_fixture_matches_build_quantizer():
    """tests/golden/quant_tables.json is what svt_av1_build_quantizer builds, for luma and both chroma planes (no
    delta-q), and its steps span the reference's range: 4 at qindex 0 up to 1336 / 1828 (8 bits) and 5347 / 7312
    (10 bits) at qindex 255."""
    spec = importlib.util.spec_from_file_location("make_quant_tables", os.path.join(cm.ROOT, "tests", "golden", "make_quant_tables.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    for bd in (8, 10):
        t = mk.build(bd)
        for q in ec.QINDEXES:
            want = ec.quant_arrays(bd, q)
            for pl in "yuv":
                got = {"quant": t[f"{pl}_quant"], "quant_shift": t[f"{pl}_quant_shift"], "zbin": t[f"{pl}_zbin"],
                       "round": t[f"{pl}_round"], "quant_fp": t[f"{pl}_quant_fp"], "round_fp": t[f"{pl}_round_fp"],
                       "dequant": t[f"{pl}_dequant_qtx"]}
                for k in ec.QKEYS:
                    np.testing.assert_array_equal(got[k][q, :2], want[k], err_msg=f"bd {bd} qindex {q} {pl} {k}")
    assert list(ec.quant_arrays(8, 0)["dequant"]) == [4, 4] and list(ec.quant_arrays(8, 255)["dequant"]) == [1336, 1828]
    assert list(ec.quant_arrays(10, 255)["dequant"]) == [5347, 7312]


# sizes whose 8-bit full-range cases at qindex 255 have a level that the quantiser's int16 clamp changes.  quantize_b
# has none: the forward transform's largest output (32648) plus its rounding never passes the next multiple of a step
# of the reference's qindex-255 tables above 32767, so its clamp is checked with the quantiser drop-ins instead.
INT16_CLAMP_SIZES = {0: (), 1: (3, 4, 17, 18)}  # use_fp -> tx sizes


@pytest.mark.parametrize("bd,use_fp", [(8, 0), (8, 1), (10, 0), (10, 1)])
def test_full_range_cases_reach_their_branches(bd, use_fp):
    """The fused-entry cases of test_txfm_edges_gpu.py, through the oracle alone: at qindex 255 every size clips its
    reconstruction, the 8-bit ones of INT16_CLAMP_SIZES (and no others) have a level the int16 clamp changes, and no case at 10 bits gets past the
    inverse transform's 18-bit input clamp with the reference's tables (that clamp is reached by the inverse drop-in
    cases instead)."""
    for ts in range(19):
        reach = ec.Reach()
        for kind in ("full_swing", "saturated", "hard_edges"):
            src, pred = ec.pair(kind, 192, 128, bd, seed=ts)
            tus = ec.corner_tus(np.random.default_rng(ts), ts, 192, 128, limit=24)
            reach += ec.chain_reach(ec.encode_params(ts, bd, 255, use_fp), src, pred, tus, use_fp)
        assert reach.recon_clip > 0, (ts, reach)
        assert (reach.int16_clamp > 0) == (bd == 8 and ts in INT16_CLAMP_SIZES[use_fp]), (ts, reach)
        assert reach.inv_clamp == 0, (ts, reach)
