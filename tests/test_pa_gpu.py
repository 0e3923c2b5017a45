"""svt_b200_picture_mean_variance against the oracle (pinned to the reference per SB in tests/test_oracle_pa.py); the
oracle reads an edge-replicated padded picture as the reference does, the GPU entry clamps its reads to the picture."""
import ctypes as C

import numpy as np
import pytest

import common as cm
import svtb200 as sb

pytestmark = pytest.mark.gpu


def _oracle(pic, w, h, full=0):
    """The oracle's per-SB y mean, variance, cb / cr means and average variance of `pic`."""
    orc = cm.oracle()
    orc.orc_picture_mean_variance.restype = C.c_uint16
    sbw, sbh = (w + 63) // 64, (h + 63) // 64
    n = sbw * sbh
    py = np.pad(pic.plane(0), ((0, sbh * 64 - h), (0, sbw * 64 - w)), mode="edge")
    pcb = np.pad(pic.plane(1), ((0, sbh * 32 - (h + 1) // 2), (0, sbw * 32 - (w + 1) // 2)), mode="edge")
    pcr = np.pad(pic.plane(2), ((0, sbh * 32 - (h + 1) // 2), (0, sbw * 32 - (w + 1) // 2)), mode="edge")
    w_ym, w_var = np.zeros((n, 85), np.uint8), np.zeros((n, 85), np.uint16)
    w_cb, w_cr = np.full((n, 21), 9, np.uint8), np.full((n, 21), 9, np.uint8)
    w_avg = orc.orc_picture_mean_variance(cm.ptr(py), py.shape[1], cm.ptr(pcb), cm.ptr(pcr), pcb.shape[1], w, h, full, cm.ptr(w_ym), cm.ptr(w_var),
                                          cm.ptr(w_cb), cm.ptr(w_cr))
    return n, w_ym, w_var, w_cb, w_cr, w_avg


@pytest.mark.parametrize("geom", [(1920, 1080, 0), (640, 360, 0), (352, 288, 0), (200, 120, 0), (3840, 2160, 0), (64, 64, 0)])
def test_picture_mean_variance_vs_oracle(geom):
    import torch
    import gpu_runner as gr
    w, h, full = geom
    lib = sb.load()
    pic = cm.synth_yuv(w, h, 2, 77, 8, noise=10)
    n, w_ym, w_var, w_cb, w_cr, w_avg = _oracle(pic, w, h, full)
    d = gr.DevYuv(pic)
    g_ym = torch.zeros(n * 85, dtype=torch.uint8, device="cuda")
    g_var = torch.zeros(n * 85, dtype=torch.int16, device="cuda")
    g_cb = torch.full((n * 21,), 7, dtype=torch.uint8, device="cuda")
    g_cr = torch.full((n * 21,), 7, dtype=torch.uint8, device="cuda")
    g_avg = torch.zeros(1, dtype=torch.int16, device="cuda")
    scratch = torch.zeros(1, dtype=torch.int64, device="cuda")
    st = d.struct()
    sb.check(lib.svt_b200_picture_mean_variance(C.byref(st), full, g_ym.data_ptr(), g_var.data_ptr(), g_cb.data_ptr(), g_cr.data_ptr(),
                                                g_avg.data_ptr(), scratch.data_ptr(), None), lib)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(g_ym.cpu().numpy().reshape(n, 85), w_ym)
    np.testing.assert_array_equal(g_var.cpu().numpy().view(np.uint16).reshape(n, 85), w_var)
    np.testing.assert_array_equal(g_cb.cpu().numpy().reshape(n, 21), w_cb)
    np.testing.assert_array_equal(g_cr.cpu().numpy().reshape(n, 21), w_cr)
    assert int(g_avg.cpu().numpy().view(np.uint16)[0]) == w_avg
    assert w_var.max() > 0
    assert lib.svt_b200_picture_mean_variance(C.byref(st), 1, g_ym.data_ptr(), g_var.data_ptr(), None, None, None, None, None) != 0
    # luma only (no chroma outputs, no average)
    g2 = torch.zeros(n * 85, dtype=torch.int16, device="cuda")
    sb.check(lib.svt_b200_picture_mean_variance(C.byref(st), full, g_ym.data_ptr(), g2.data_ptr(), None, None, None, None, None), lib)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(g2.cpu().numpy().view(np.uint16).reshape(n, 85), w_var)


@pytest.mark.parametrize("chroma", [1, 0], ids=["chroma", "luma"])
@pytest.mark.parametrize("avg", [1, 0], ids=["avg", "noavg"])
@pytest.mark.parametrize("geom", [(712, 392), (200, 136)])
def test_picture_mean_variance_host(geom, avg, chroma):
    """svt_b200_picture_mean_variance_host (host planes in, host arrays out) at ragged sizes, with and without the chroma
    means and the average variance: equal to the oracle the device entry is checked against above, and the outputs it
    was not asked for are left untouched."""
    w, h = geom
    lib = sb.load()
    pic = cm.synth_yuv(w, h, 2, 78, 8, noise=10)
    n, w_ym, w_var, w_cb, w_cr, w_avg = _oracle(pic, w, h)
    y, cb, cr = pic.plane(0), pic.plane(1), pic.plane(2)
    ym, var = np.full((n, 85), 5, np.uint8), np.full((n, 85), 5, np.uint16)
    cbm, crm = np.full((n, 21), 7, np.uint8), np.full((n, 21), 7, np.uint8)
    pav = np.full(1, 0xBEEF, np.uint16)
    sb.check(lib.svt_b200_picture_mean_variance_host(cm.ptr(y), y.strides[0], cm.ptr(cb) if chroma else None, cm.ptr(cr) if chroma else None,
                                                     cb.strides[0], w, h, cm.ptr(ym), cm.ptr(var), cm.ptr(cbm) if chroma else None,
                                                     cm.ptr(crm) if chroma else None, cm.ptr(pav) if avg else None), lib)
    np.testing.assert_array_equal(ym, w_ym)
    np.testing.assert_array_equal(var, w_var)
    if chroma:
        np.testing.assert_array_equal(cbm, w_cb)
        np.testing.assert_array_equal(crm, w_cr)
    else:
        assert (cbm == 7).all() and (crm == 7).all()
    assert int(pav[0]) == (w_avg if avg else 0xBEEF)
