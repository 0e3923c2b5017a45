#!/usr/bin/env python
"""Device time of one svt_b200_me_picture call (HME + full-pel search of one picture against all its references) at
1920x1080, in the two HME regimes: preset 1 with the random-access structure of test_oracle_me_presets.py takes the
chunked regime, preset 8 with its structure the staged one (launch_plan in tests/test_me_presets_gpu.py says which).
Synthetic content (common.make_me_case), device-resident planes; CUDA events on the launch stream around `--calls`
back-to-back calls after a warm-up, `--reps` times, median reported per case, with an md5 of the outputs so that two
builds can be checked for the same results.  SVTB200_LIB selects the library.  One JSON object on stdout.

    python tools/me_bench.py > me_bench.json
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "svt-av1_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402

import common as cm  # noqa: E402
import gpu_runner as gr  # noqa: E402
import svtb200 as sb  # noqa: E402
from test_me_presets_gpu import launch_plan  # noqa: E402
from test_oracle_me_presets import structure  # noqa: E402

W, H = 1920, 1080


def time_case(lib, preset, calls, reps):
    n0, n1, dist, tl = structure(preset, "ra")
    params = sb.me_params(preset, W, H, n0, n1, dist, tl, 1)
    _, src, refs = cm.make_me_case(W, H, n0, n1, seed=200 + preset)
    n_sb = ((W + 63) // 64) * ((H + 63) // 64)
    d_src = [gr.dev(x) for x in src]
    d_refs = [[gr.dev(x) for x in r] for r in refs]
    s = sb.MePlanes(*[t.data_ptr() for t in d_src])
    r = (sb.MePlanes * 8)(*[sb.MePlanes(*[t.data_ptr() for t in rr]) for rr in d_refs])
    fields = cm.MeBuffers(n_sb).fields()
    d_out = {k: torch.zeros(v.size * v.dtype.itemsize, dtype=torch.uint8, device="cuda") for k, v in fields.items()}
    o = sb.MeOutputs(*[d_out[k].data_ptr() for k in ("best_sad", "best_mv", "hme", "me_mv", "me_cand", "total_cand", "rc")])
    scratch = torch.zeros(lib.svt_b200_me_scratch_bytes(C.byref(params)), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream()

    def call():
        sb.check(lib.svt_b200_me_picture(C.byref(params), C.byref(s), r, C.byref(o), scratch.data_ptr(),
                                         C.c_void_p(stream.cuda_stream)), lib)

    for _ in range(5):
        call()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(calls):
            call()
        e1.record(stream)
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / calls)
    md5 = hashlib.md5()
    for k in sorted(d_out):
        md5.update(d_out[k].cpu().numpy().tobytes())
    plan = launch_plan(params)
    return {"preset": preset, "hme_regime": "chunked" if plan["hme_generic"] else "staged", "hme_need": plan["hme_need"],
            "refs": [n0, n1], "ms_per_picture": statistics.median(times), "ms_all": times, "outputs_md5": md5.hexdigest()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    lib = sb.load()
    cases = [time_case(lib, pr, a.calls, a.reps) for pr in (1, 8)]
    print(json.dumps({"device": torch.cuda.get_device_name(0), "size": [W, H], "lib": sb.LIB_PATH, "cases": cases}))


if __name__ == "__main__":
    main()
