#!/usr/bin/env python
"""Device time of the picture-level in-loop filter entries, one picture per launch sequence, at the two bench geometries
(1920x1080 8-bit = configs[1], 3840x2160 10-bit = configs[2]), against the measured HBM peak.

For every entry: a RING of distinct device pictures whose total size exceeds the 126 MB L2 (64 pictures at 1080p, 8 at
2160p); one timed pass = one call per ring picture, captured into a CUDA graph and replayed (so the figure is device
time, not host launch latency), CUDA events on the launch stream around the replay, 5 passes after a warm-up pass;
deblocking works in place, so the ring is restored from a pristine copy (untimed) before every pass.  Reported:
algorithmic bytes (DESIGN.md section 4) / time and - as the ceiling a launch of this SIZE can reach - a plain device
copy of the same pictures through the same ring (read + write of the same bytes).  One JSON object on stdout.

    python tools/kernel_bench.py > gpurun_out/kernel_bench.json
"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "svt-av1_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import common as cm  # noqa: E402
import gpu_runner as gr  # noqa: E402
import svtb200 as sb  # noqa: E402
from test_dlf_gpu import flat_mi  # noqa: E402
from test_oracle_dlf import dlf_case, dlf_params  # noqa: E402
from test_oracle_cdef import cdef_picture_case  # noqa: E402

lib = sb.load()
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    PEAK = 6650.0


STREAM = torch.cuda.Stream()
SP = C.c_void_p(STREAM.cuda_stream)


def ring_ms(fn, ring, restore=None, passes=5):
    """fn(i) issues the call on ring picture i on STREAM.  One pass over the ring is captured into a CUDA graph and
    replayed, so the figure is device time (no host launch latency between the calls).  Mean device time per call."""
    with torch.cuda.stream(STREAM):
        for i in range(ring):
            fn(i)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=STREAM):
            for i in range(ring):
                fn(i)
        tot = 0.0
        for _ in range(passes):
            if restore:
                restore()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(STREAM)
            g.replay()
            e1.record(STREAM)
            torch.cuda.synchronize()
            tot += e0.elapsed_time(e1)
    return tot / (passes * ring)


def row(name, ms, alg_bytes, copy_ms, note=""):
    return {"entry": name, "ms": round(ms, 5), "algorithmic_bytes": int(alg_bytes), "achieved_gbs": round(alg_bytes / ms / 1e6, 1),
            "frac_of_hbm_peak": round(alg_bytes / ms / 1e6 / PEAK, 4), "same_size_copy_ms": round(copy_ms, 5),
            "frac_of_same_size_copy": round(copy_ms / ms, 3), "note": note}


def geometry(w, h, bd):
    out = {"geometry": "%dx%d %d-bit 4:2:0" % (w, h, bd), "rows": []}
    bps = 2 if bd > 8 else 1
    samples = w * h * 3 // 2
    pic_bytes = samples * bps
    ring = max(4, -(-(160 << 20) // pic_bytes))  # ring of pictures > L2 (126 MB)
    out["ring_pictures"] = ring
    # the ceiling for a launch of this size: device copy of one picture (reads + writes pic_bytes)
    a = [torch.empty(pic_bytes, dtype=torch.uint8, device="cuda") for _ in range(ring)]
    b = [torch.empty(pic_bytes, dtype=torch.uint8, device="cuda") for _ in range(ring)]
    copy_ms = ring_ms(lambda i: b[i].copy_(a[i]), ring)
    out["same_size_copy"] = {"ms": round(copy_ms, 5), "gbs": round(2 * pic_bytes / copy_ms / 1e6, 1),
                             "frac_of_hbm_peak": round(2 * pic_bytes / copy_ms / 1e6 / PEAK, 4)}
    del a, b

    # ---- deblocking --------------------------------------------------------------------------------------------
    levels = (24, 20, 14, 10)
    mi_rows, mi_cols, part, frame = dlf_case(w, h, bd, 9, levels, 1)
    flat = flat_mi(mi_rows, mi_cols, part, levels)
    p = dlf_params(mi_rows, mi_cols, levels, 1)
    pristine = gr.DevYuv(frame.copy())
    dfs = [gr.DevYuv(frame) for _ in range(ring)]
    dmis = [torch.from_numpy(np.frombuffer(flat, dtype=np.uint8).copy()).cuda() for _ in range(ring)]
    sts = [d.struct() for d in dfs]

    def restore():
        for d in dfs:
            for t, t0 in zip(d.t, pristine.t):
                t.copy_(t0)
    call = lambda i: sb.check(lib.svt_b200_dlf_frame(C.byref(p), C.byref(sts[i]), C.c_void_p(dmis[i].data_ptr()), SP), lib)  # noqa: E731
    ms = ring_ms(call, ring, restore)
    alg = 2 * (2 * pic_bytes) + 2 * mi_rows * mi_cols * 16
    out["rows"].append(row("svt_b200_dlf_frame (2 launches: all vertical edges, all horizontal edges)", ms, alg, copy_ms,
                           "2 passes x (read + write) + the 16 B / 4x4 mode-info summary per pass"))
    del dfs, dmis, pristine

    # ---- CDEF --------------------------------------------------------------------------------------------------
    src, rec, mi_rows, mi_cols, skip = cdef_picture_case(w, h, bd)
    sp = sb.CdefSearchParams()
    sp.mi_rows, sp.mi_cols, sp.pri_damping = mi_rows, mi_cols, 5
    cm.oracle().orc_cdef_strength_table(3, C.byref(sp))
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    drs, dss, dos = [gr.DevYuv(rec) for _ in range(ring)], [gr.DevYuv(src) for _ in range(ring)], [gr.DevYuv(rec) for _ in range(ring)]
    dskip = torch.from_numpy(skip).cuda()
    dmse = torch.zeros(2 * nfb * 64, dtype=torch.int64, device="cuda")
    rss, sss, oss = [d.struct() for d in drs], [d.struct() for d in dss], [d.struct() for d in dos]
    ms = ring_ms(lambda i: sb.check(lib.svt_b200_cdef_search(C.byref(sp), C.byref(rss[i]), C.byref(sss[i]), C.c_void_p(dskip.data_ptr()),
                                                             skip.shape[1], C.c_void_p(dmse.data_ptr()), SP), lib), ring)
    out["rows"].append(row("svt_b200_cdef_search (10 strengths, preset 8 table)", ms, 2 * pic_bytes + nfb * 2 * 64 * 8, copy_ms,
                           "integer-ALU bound: 10 filter evaluations per sample"))
    pa = sb.CdefApplyParams()
    pa.mi_rows, pa.mi_cols, pa.damping = mi_rows, mi_cols, 5
    for k, (x, y) in enumerate(zip((0, 5, 17, 63, 40, 2, 12, 33), (0, 0, 9, 62, 4, 1, 60, 3))):
        pa.y_strength[k], pa.uv_strength[k] = x, y
    didx = torch.from_numpy((np.arange(nfb) % 8).astype(np.int8)).cuda()
    ms = ring_ms(lambda i: sb.check(lib.svt_b200_cdef_apply(C.byref(pa), C.byref(rss[i]), C.byref(oss[i]), C.c_void_p(dskip.data_ptr()),
                                                            skip.shape[1], C.c_void_p(didx.data_ptr()), SP), lib), ring)
    out["rows"].append(row("svt_b200_cdef_apply (8 strength pairs cycled over the filter blocks)", ms, 2 * pic_bytes, copy_ms))
    # the strength decision between the two (finish_cdef_search on the device): a single CTA, latency not bandwidth
    dcp = sb.CdefDecideParams()
    lib.svt_b200_cdef_decide_table(3, C.byref(dcp))
    dcp.mi_rows, dcp.mi_cols, dcp.lambda_ = mi_rows, mi_cols, 3500
    ddec = torch.zeros(C.sizeof(sb.CdefDecision), dtype=torch.uint8, device="cuda")
    didx2 = torch.zeros(nfb, dtype=torch.int8, device="cuda")
    dscr = torch.zeros(nfb * (16 + 16 * 64) + 64, dtype=torch.uint8, device="cuda")
    lib.svt_b200_cdef_decide.argtypes = [C.POINTER(sb.CdefDecideParams)] + [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    ms = ring_ms(lambda i: sb.check(lib.svt_b200_cdef_decide(C.byref(dcp), dmse.data_ptr(), dskip.data_ptr(), skip.shape[1], ddec.data_ptr(),
                                                             didx2.data_ptr(), dscr.data_ptr(), SP), lib), 8)
    out["rows"].append(row("svt_b200_cdef_decide (finish_cdef_search: 75 search steps over %d filter blocks x 100 strength pairs)" % nfb, ms,
                           nfb * 2 * 10 * 8, copy_ms, "one CTA: a latency chain of 75 dependent reductions, not a bandwidth kernel"))
    del drs, dss, dos

    # ---- pre-analysis entries (round 2): temporal filter, picture statistics, open-loop intra search ----------------
    if bd == 8 or True:
        n_acc = w * h * 3 // 2
        xs, ys = range(0, w - 31, 32), range(0, h - 31, 32)
        blocks = [(x, y) for y in ys for x in xs]
        arr = (sb.TfBlock * len(blocks))()
        rng = np.random.default_rng(7)
        for i, (x, y) in enumerate(blocks):
            arr[i].x, arr[i].y = x, y
            for q in range(4):
                arr[i].block_error[q], arr[i].d_factor[q] = float(rng.integers(0, 2000) / 256.0), 1.0 + float(rng.integers(0, 100)) / 100.0
        dblk = torch.from_numpy(np.frombuffer(arr, dtype=np.uint8).copy()).cuda()
        pred = cm.degrade(src, 32, amp=6)
        small = max(4, ring // 2)  # accumulators add 6 bytes per sample: a shorter ring still exceeds L2
        srcs, preds = [gr.DevYuv(src) for _ in range(small)], [gr.DevYuv(pred) for _ in range(small)]
        cw, ch = (w + 1) // 2, (h + 1) // 2
        accs = [[torch.zeros(h * w, dtype=torch.int32, device="cuda"), torch.zeros(ch * cw, dtype=torch.int32, device="cuda"),
                 torch.zeros(ch * cw, dtype=torch.int32, device="cuda")] for _ in range(small)]
        cnts = [[torch.zeros(h * w, dtype=torch.int16, device="cuda"), torch.zeros(ch * cw, dtype=torch.int16, device="cuda"),
                 torch.zeros(ch * cw, dtype=torch.int16, device="cuda")] for _ in range(small)]
        tas = []
        for a, c_ in zip(accs, cnts):
            ta = sb.TfAccum()
            for i in range(3):
                ta.accum[i], ta.count[i] = a[i].data_ptr(), c_[i].data_ptr()
            ta.stride_y, ta.stride_c = w, cw
            tas.append(ta)
        tp = sb.TfParams()
        for i in range(3):
            tp.den[i] = 2.0 * (4 * 1.9) ** 2
        tp.chroma, tp.block_w, tp.block_h = 1, 32, 32
        s_s, p_s = [d.struct() for d in srcs], [d.struct() for d in preds]
        ms_copy_small = copy_ms  # same-size copy measured above on the full ring
        ms = ring_ms(lambda i: sb.check(lib.svt_b200_tf_planewise(C.byref(tp), C.byref(s_s[i]), C.byref(p_s[i]), C.c_void_p(dblk.data_ptr()),
                                                                  len(blocks), C.byref(tas[i]), SP), lib), small)
        alg_tf = 2 * pic_bytes + 2 * n_acc * 6  # source + prediction read, accumulators (4 B) and counters (2 B) read + written
        out["rows"].append(row("svt_b200_tf_planewise (every 32x32 block of one reference picture, chroma on)", ms, alg_tf, ms_copy_small,
                               "double-precision weight chain per sample (IEEE div x3, expf restated)"))
        ms = ring_ms(lambda i: sb.check(lib.svt_b200_tf_central(C.byref(s_s[i]), C.byref(tas[i]), 1, SP), lib), small)
        out["rows"].append(row("svt_b200_tf_central", ms, pic_bytes + 2 * n_acc * 6, ms_copy_small))
        dsse = torch.zeros(2, dtype=torch.int64, device="cuda")
        ms = ring_ms(lambda i: sb.check(lib.svt_b200_tf_normalize(C.byref(s_s[i]), C.byref(tas[i]), 1, C.c_void_p(dsse.data_ptr()), SP), lib), small)
        out["rows"].append(row("svt_b200_tf_normalize", ms, 2 * pic_bytes + n_acc * 6, ms_copy_small))
        del accs, cnts, preds
        if bd == 8:
            n_sb = ((w + 63) // 64) * ((h + 63) // 64)
            o1 = torch.zeros(n_sb * 85, dtype=torch.uint8, device="cuda")
            o2 = torch.zeros(n_sb * 85, dtype=torch.int16, device="cuda")
            o3, o4 = torch.zeros(n_sb * 21, dtype=torch.uint8, device="cuda"), torch.zeros(n_sb * 21, dtype=torch.uint8, device="cuda")
            ms = ring_ms(lambda i: sb.check(lib.svt_b200_picture_mean_variance(C.byref(s_s[i]), 0, o1.data_ptr(), o2.data_ptr(), o3.data_ptr(),
                                                                                 o4.data_ptr(), None, None, SP), lib), small)
            out["rows"].append(row("svt_b200_picture_mean_variance (sub-sampled flavour: every other row)", ms, pic_bytes // 2, ms_copy_small,
                                   "reads half the rows; 32-byte sectors make the DRAM traffic ~ the whole picture"))
            mbn = ((w + 15) // 16) * ((h + 15) // 16)
            oc = torch.zeros(mbn, dtype=torch.int64, device="cuda")
            ms = ring_ms(lambda i: sb.check(lib.svt_b200_ois_dc_picture(C.byref(s_s[i]), oc.data_ptr(), SP), lib), small)
            out["rows"].append(row("svt_b200_ois_dc_picture (DC predictor + 16x16 DCT + SATD per macroblock)", ms, w * h + mbn * 8, ms_copy_small,
                                   "transform bound: 2 x 16-point DCT passes per macroblock on 16 threads"))
    return out


if __name__ == "__main__":
    res = {"hbm_peak_gbs": PEAK, "gpu": torch.cuda.get_device_name(0),
           "method": "ring of distinct pictures larger than L2, back-to-back calls, CUDA events around a pass, 5 passes after warm-up",
           "geometries": [geometry(1920, 1080, 8), geometry(3840, 2160, 10)]}
    print(json.dumps(res, indent=1))
