"""The RTCD drop-ins and the `_host` entries from many threads at once, as the encoder's pipeline threads call them.

Every thread starts behind one barrier and runs its own seeded interleaving of host-pointer calls: at least one from each
source file that stages host data, and one `_host` call whose staging exceeds the 1 MB a thread's buffers start with,
placed between smaller calls so the thread's buffers grow in the middle of its sequence. Every expectation comes from
the CPU oracle, computed on the main thread before any thread starts; every result must be bit-exact."""
import ctypes as C
import threading

import numpy as np
import pytest

import common as cm
import misc_oracle as mo
import svtb200 as sb
import tf_cases as tc
from test_interp_gpu import kernel_table
from test_me_gpu import _call_sad_loop
from test_oracle_dlf import edge_cases
from test_oracle_lr import ConvolveParams, aligned_filter, lr_image, wiener_filter
from test_oracle_me import sad_case
from test_oracle_misc import _cdef_dist_case, _stats_case
from test_oracle_txfm import residual_block
from test_pa_gpu import _oracle as pa_oracle

pytestmark = pytest.mark.gpu

N_THREADS = 10


class Call:
    """One drop-in call with its own buffers: run() makes the call and returns what it produced, `want` is the oracle's."""

    def __init__(self, name, run, want):
        self.name, self.run, self.want = name, run, want


def sad_loop(lib, orc, rng):  # me.cu
    bw, bh, saw, sah = 32, 16, 48, 24
    src, ref, stride = sad_case(rng, bw, bh, saw, sah, "RANDOM")
    want = _call_sad_loop(orc.orc_sad_loop_kernel, src, ref, stride, bw, bh, saw, sah)
    return Call("svt_sad_loop_kernel_cuda", lambda: _call_sad_loop(lib.svt_sad_loop_kernel_cuda, src, ref, stride, bw, bh, saw, sah), want)


def nxm_sad(lib, orc, rng):  # misc.cu
    w, h = 24, 40
    a = rng.integers(0, 256, (h, w + 9), dtype=np.uint8)
    b = rng.integers(0, 256, (h, w + 5), dtype=np.uint8)
    lib.svt_nxm_sad_kernel_cuda.restype = C.c_uint32
    return Call("svt_nxm_sad_kernel_cuda",
                lambda: lib.svt_nxm_sad_kernel_cuda(cm.ptr(a), C.c_uint32(w + 9), cm.ptr(b), C.c_uint32(w + 5), C.c_uint32(h), C.c_uint32(w)),
                mo.sad(a[:, :w], b[:, :w]))


def subtract(lib, orc, rng):  # misc.cu
    w, h = 40, 24
    a = rng.integers(0, 256, (h, w + 5), dtype=np.uint8)
    b = rng.integers(0, 256, (h, w + 9), dtype=np.uint8)
    d = np.zeros((h, w + 1), np.int16)

    def run():
        lib.svt_aom_subtract_block_cuda(h, w, cm.ptr(d), C.c_ssize_t(w + 1), cm.ptr(a), C.c_ssize_t(w + 5), cm.ptr(b), C.c_ssize_t(w + 9))
        return d[:, :w].copy()
    return Call("svt_aom_subtract_block_cuda", run, mo.subtract(a[:, :w], b[:, :w]))


def fwd_txfm(lib, orc, rng):  # txfm.cu
    w = h = 16
    res = residual_block(rng, w, h, 10, "rand")
    want, got = np.zeros(w * h, np.int32), np.zeros(w * h, np.int32)
    orc.orc_fwd_txfm2d(cm.ptr(res), cm.ptr(want), C.c_uint32(w + 5), 0, 2, 10)

    def run():
        lib.svt_av1_fwd_txfm2d_16x16_cuda(cm.ptr(res), cm.ptr(got), C.c_uint32(w + 5), 0, C.c_uint8(10))
        return got.copy()
    return Call("svt_av1_fwd_txfm2d_16x16_cuda", run, want)


def cdef_dist(lib, orc, rng):  # cdef.cu
    bd, bsize, pli = 10, 3, 0
    fb, src, pick, dl = _cdef_dist_case(rng, bd, bsize, pli)
    src = np.ascontiguousarray(src)
    lib.svt_compute_cdef_dist_16bit_cuda.restype = C.c_uint64
    return Call("svt_compute_cdef_dist_16bit_cuda",
                lambda: lib.svt_compute_cdef_dist_16bit_cuda(cm.ptr(fb), 64, cm.ptr(src), cm.ptr(dl), len(pick), bsize, bd - 8, pli),
                mo.cdef_dist(fb, 64, src, pick, bsize, bd - 8, pli))


def lpf(lib, orc, rng):  # dlf.cu
    bd, img, blimit, limit, thresh = list(edge_cases(int(rng.integers(0, 1 << 16)), n=3))[1]
    a = img.astype(np.uint16)
    b = a.copy()
    off = (16 * 32 + 16) * a.itemsize
    bl, li, th = (np.full(16, v, np.uint8) for v in (blimit & 255, limit, thresh))
    orc.orc_lpf_edge(C.c_void_p(b.ctypes.data + off), 1, 1, 32, 8, blimit & 255, limit, thresh, bd)

    def run():
        lib.svt_aom_highbd_lpf_vertical_8_cuda(C.c_void_p(a.ctypes.data + off), 32, cm.ptr(bl), cm.ptr(li), cm.ptr(th), bd)
        return a.copy()
    return Call("svt_aom_highbd_lpf_vertical_8_cuda", run, b)


def wiener(lib, orc, rng):  # lr.cu
    w, h = 64, 32
    a = lr_image(rng, 8, "random").astype(np.uint8)
    stride = a.shape[1]
    p = a.ctypes.data + (8 * stride + 8)
    fx, fy = wiener_filter(rng), wiener_filter(rng)
    keep_x, px = aligned_filter(fx)
    keep_y, py = aligned_filter(fy)
    cp = ConvolveParams()
    cp.round_0, cp.round_1 = 3, 11
    d0, d1 = np.zeros((h, w + 5), np.uint8), np.zeros((h, w + 5), np.uint8)
    orc.orc_wiener_convolve_add_src(C.c_void_p(p), 0, C.c_ssize_t(stride), cm.ptr(d1), C.c_ssize_t(w + 5), cm.ptr(fx), cm.ptr(fy), w, h,
                                    cp.round_0, cp.round_1, 8)

    def run():
        _ = (a, keep_x, keep_y)  # the picture and the aligned filter tables live as long as the call
        lib.svt_av1_wiener_convolve_add_src_cuda(C.c_void_p(p), C.c_ssize_t(stride), cm.ptr(d0), C.c_ssize_t(w + 5), C.c_void_p(px),
                                                 C.c_void_p(py), w, h, C.byref(cp))
        return d0.copy()
    return Call("svt_av1_wiener_convolve_add_src_cuda", run, d1)


def stats(lib, orc, rng):  # lrpick.cu
    bd, win, w, h, hs, vs = 10, 7, 40, 24, 8, 8
    dgd, src = _stats_case(rng, bd, w, h, 1)
    n = win * win
    M, Hm = np.zeros(n, np.int64), np.zeros(n * n, np.int64)
    m2, h2 = mo.compute_stats(win, dgd, src, hs, hs + w, vs, vs + h, bd)

    def run():
        lib.svt_av1_compute_stats_highbd_cuda(win, C.c_void_p(dgd.ctypes.data >> 1), C.c_void_p(src.ctypes.data >> 1), hs, hs + w, vs, vs + h,
                                              dgd.shape[1], src.shape[1], cm.ptr(M), cm.ptr(Hm), bd)
        return np.concatenate([M, Hm])
    return Call("svt_av1_compute_stats_highbd_cuda", run, np.concatenate([m2, h2.reshape(-1)]))


def proj_error(lib, orc, rng):  # lrpick.cu
    w, h, r = 33, 17, (2, 1)
    src = rng.integers(0, 256, (h, w + 5)).astype(np.uint8)
    dat = np.clip(src.astype(np.int64) + rng.integers(-9, 10, src.shape), 0, 255).astype(np.uint8)
    f0 = ((dat.astype(np.int64) << 4) + rng.integers(-200, 201, dat.shape)).astype(np.int32)
    f1 = ((dat.astype(np.int64) << 4) + rng.integers(-200, 201, dat.shape)).astype(np.int32)
    xq = (C.c_int32 * 2)(int(rng.integers(-96, 32)), int(rng.integers(-32, 96)))
    params = (C.c_int32 * 4)(r[0], r[1], 0, 0)
    lib.svt_av1_lowbd_pixel_proj_error_cuda.restype = C.c_int64
    return Call("svt_av1_lowbd_pixel_proj_error_cuda",
                lambda: lib.svt_av1_lowbd_pixel_proj_error_cuda(cm.ptr(src), w, h, src.shape[1], cm.ptr(dat), dat.shape[1], cm.ptr(f0), f0.shape[1],
                                                                cm.ptr(f1), f1.shape[1], xq, params),
                mo.pixel_proj_error(src[:, :w], dat[:, :w], f0[:, :w], f1[:, :w], (xq[0], xq[1]), r, False))


def convolve8(lib, orc, rng):  # interp.cu
    w, h, step, vert = 32, 16, 16, int(rng.integers(0, 2))
    raw = np.zeros(16 * 8 + 256, np.int16)  # a 256-byte aligned [16][8] table, as get_filter_base requires
    off = (-raw.ctypes.data % 256) // 2
    table = raw[off:off + 128].reshape(16, 8)
    table[...] = kernel_table(lib, int(rng.integers(0, 4)), 8)
    q0 = int(rng.integers(0, 16))
    span = ((max(w, h) - 1) * step + q0 >> 4) + 16
    src = rng.integers(0, 256, (span + 16, span + 16)).astype(np.uint8)
    a, b = np.zeros((h, w), np.uint8), np.ones((h, w), np.uint8)
    s0 = C.c_void_p(src.ctypes.data + 8 * src.shape[1] + 8)
    orc.orc_convolve8(s0, C.c_ssize_t(src.shape[1]), cm.ptr(a), C.c_ssize_t(w), cm.ptr(table), q0, step, w, h, vert)
    f = C.c_void_p(table.ctypes.data + 16 * q0)
    fn = lib.svt_aom_convolve8_vert_cuda if vert else lib.svt_aom_convolve8_horiz_cuda

    def run():
        _ = raw
        fn(s0, C.c_ssize_t(src.shape[1]), cm.ptr(b), C.c_ssize_t(w), None if vert else f, 0 if vert else step, f if vert else None,
           step if vert else 0, w, h)
        return b.copy()
    return Call("svt_aom_convolve8_%s_cuda" % ("vert" if vert else "horiz"), run, a)


def tf_block(lib, orc, rng):  # tf.cu, a `_host` entry
    torc = cm.oracle()
    torc.orc_tf_normalize.restype = C.c_uint64
    c = tc.make_case(**tc.CASES[int(rng.integers(0, len(tc.CASES)))])
    want = tc.run_oracle(torc, c)
    den, be, df = tc.factors(torc, c)
    got = tc.fresh(c)

    def run():
        sb.check(lib.svt_b200_tf_planewise_block_host(c.bd, c.chroma, tc.ptr(c.y_src), c.ys, tc.ptr(c.y_pre), c.ps, tc.ptr(c.u_src),
                                                      tc.ptr(c.v_src), c.uvs, tc.ptr(c.u_pre), tc.ptr(c.v_pre), c.ups, c.bw, c.bh, den, be, df,
                                                      *[tc.ptr(a) for a in got]), lib)
        return np.concatenate([a.reshape(-1).astype(np.int64) for a in got])
    return Call("svt_b200_tf_planewise_block_host", run, np.concatenate([a.reshape(-1).astype(np.int64) for a in want]))


def pa_host(lib, orc, rng, w=1280, h=720):  # pa.cu: the large `_host` call (about 1.4 MB of staging)
    pic = cm.synth_yuv(w, h, 2, int(rng.integers(0, 1000)), 8, noise=10)
    n, w_ym, w_var, w_cb, w_cr, w_avg = pa_oracle(pic, w, h)
    y, cb, cr = pic.plane(0), pic.plane(1), pic.plane(2)
    ym, var = np.zeros((n, 85), np.uint8), np.zeros((n, 85), np.uint16)
    cbm, crm, pav = np.zeros((n, 21), np.uint8), np.zeros((n, 21), np.uint8), np.zeros(1, np.uint16)

    def run():
        sb.check(lib.svt_b200_picture_mean_variance_host(cm.ptr(y), y.strides[0], cm.ptr(cb), cm.ptr(cr), cb.strides[0], w, h, cm.ptr(ym),
                                                         cm.ptr(var), cm.ptr(cbm), cm.ptr(crm), cm.ptr(pav)), lib)
        return np.concatenate([ym.reshape(-1), var.reshape(-1), cbm.reshape(-1), crm.reshape(-1), pav])
    want = np.concatenate([w_ym.reshape(-1), w_var.reshape(-1), w_cb.reshape(-1), w_cr.reshape(-1), np.array([w_avg], np.uint16)])
    return Call(f"svt_b200_picture_mean_variance_host {w}x{h}", run, want)


SMALL = [sad_loop, nxm_sad, subtract, fwd_txfm, cdef_dist, lpf, wiener, stats, proj_error, convolve8, tf_block]


def test_dropins_from_many_threads():
    lib, orc = sb.load(), cm.oracle()
    plans = []
    for t in range(N_THREADS):
        rng = np.random.default_rng(5000 + t)
        small = [make(lib, orc, rng) for make in SMALL + [SMALL[int(i)] for i in rng.integers(0, len(SMALL), 5)]]
        rng.shuffle(small)
        mid = int(rng.integers(2, len(small) - 1))
        plans.append(small[:mid] + [pa_host(lib, orc, rng)] + small[mid:])
    barrier = threading.Barrier(N_THREADS)
    failures = []

    def worker(t):
        barrier.wait()
        for step, call in enumerate(plans[t]):
            try:
                got = call.run()
                if isinstance(call.want, np.ndarray):
                    np.testing.assert_array_equal(got, call.want)
                else:
                    assert got == call.want, (got, call.want)
            except Exception as e:  # noqa: BLE001  (reported with the thread, step and call below)
                failures.append(f"thread {t} step {step} {call.name}: {type(e).__name__}: {str(e)[:300]}")

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(N_THREADS)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not failures, "\n".join(failures)
    assert all(len(p) >= len(SMALL) + 1 for p in plans)
