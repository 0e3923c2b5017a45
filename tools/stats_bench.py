#!/usr/bin/env python
"""svt_b200_lr_wiener_stats (all compute_stats calls of search_wiener for a luma plane, win 7; the INT8 tensor-core
kernel) at the two bench geometries.  Device time with CUDA events over 20 calls after 3 warm-up calls (the pictures,
3 MB / 25 MB, stay in L2: the kernel is arithmetic bound, see the MAC rates).  The checksum of each row is the XOR of
the returned statistics.

    python tools/stats_bench.py > gpurun_out/stats_bench.json
"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    for p in (os.path.join(ROOT, "svt-av1_b200"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import numpy as np
    import torch
    import common as cm
    import gpu_runner as gr
    import svtb200 as sb
    lib = sb.load()
    rows = []
    for (W, H, bd, unit) in ((1920, 1080, 8, 64), (1920, 1080, 8, 256), (3840, 2160, 10, 64), (3840, 2160, 10, 256)):
        src = cm.synth_yuv(W, H, 1, 21, bd)
        dgd = cm.degrade(src, 22, amp=8)
        dg, ds = gr.DevYuv(dgd), gr.DevYuv(src)
        rects = [(x, min(x + unit, W), y, min(y + unit, H)) for y in range(0, H, unit) for x in range(0, W, unit)]
        r = torch.tensor(rects, dtype=torch.int32, device="cuda")
        stats = torch.zeros(len(rects) * (49 + 49 * 49), dtype=torch.int64, device="cuda")
        scr = torch.zeros(len(rects), dtype=torch.int64, device="cuda")
        a, b = dg.struct(), ds.struct()
        fn = lambda: sb.check(lib.svt_b200_lr_wiener_stats(C.byref(a), C.byref(b), 0, 7, C.c_void_p(r.data_ptr()), len(rects), unit, unit,  # noqa: E731
                                                           C.c_void_p(stats.data_ptr()), C.c_void_p(scr.data_ptr()), None), lib)
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 20
        macs = W * H * (49 * 50 // 2 + 49)
        h = stats.cpu().numpy()
        rows.append({"geometry": "%dx%d %d-bit luma, %d units of %d" % (W, H, bd, len(rects), unit), "ms": round(ms, 4),
                     "useful_int_macs": macs, "useful_tmacs": round(macs / ms / 1e9, 2),
                     "checksum": int(np.bitwise_xor.reduce(h))})
    print(json.dumps({"device": torch.cuda.get_device_name(), "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
