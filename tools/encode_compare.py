"""Runs the reference's own EncApp in several builds / backend settings on one synthetic clip and compares the
bitstream and reconstruction md5 (SURVEY.md 8c(3): the encoder is deterministic, so the CUDA build must reproduce the
C-only build bit for bit), printing one JSON line per run.

    python tools/encode_compare.py --width 640 --height 360 --frames 30 --preset 8 --qp 50 [--bits 10] [--variants ...]

Variants: ref_c (oracle/_ref C-only), ref_simd (oracle/_ref/simd, AVX2/AVX-512 minus asm), cuda_c / cuda_simd (overlay
build with SVT_CUDA=1), and cuda_c:me / :dlf / :cdef (one stage on the GPU only).
"""
import argparse
import hashlib
import json
import os
import re
import resource
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_yuv  # noqa: E402

APPS = {
    "ref_c": os.path.join(ROOT, "oracle", "_ref", "app", "SvtAv1EncAppRef"),
    "ref_simd": os.path.join(ROOT, "oracle", "_ref", "app", "SvtAv1EncAppSimd"),
    "cuda_c": os.path.join(ROOT, "oracle", "_ref", "integration", "SvtAv1EncAppCudaC"),
    "cuda_simd": os.path.join(ROOT, "oracle", "_ref", "integration", "SvtAv1EncAppCudaSimd"),
}


def md5(path):
    h = hashlib.md5()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 22), b""):
            h.update(blk)
    return h.hexdigest()


def run_variant(variant, clip, width, height, frames, preset, qp, bits, workdir, extra_env=None, recon=True, timeout=3600,
                extra_args=()):
    base, _, stage = variant.partition(":")
    env = dict(os.environ)
    for k in list(env):
        if k.startswith("SVT_CUDA"):
            del env[k]
    if base.startswith("cuda"):
        env["SVT_CUDA"] = "1"
        if stage:
            for s in ("ME", "DLF", "CDEF"):
                env["SVT_CUDA_" + s] = "1" if s.lower() in stage.split("+") else "0"
    env.update(extra_env or {})
    tag = variant.replace(":", "_").replace("+", "_")
    ivf = os.path.join(workdir, tag + ".ivf")
    rec = os.path.join(workdir, tag + ".rec")
    cmd = [APPS[base], "-i", clip, "-w", str(width), "-h", str(height), "--fps", "30", "--preset", str(preset), "--rc", "0",
           "-q", str(qp), "-n", str(frames), "-b", ivf] + (["-o", rec] if recon else []) + \
          (["--input-depth", str(bits)] if bits != 8 else []) + list(extra_args)
    r0 = resource.getrusage(resource.RUSAGE_CHILDREN)
    t0 = time.time()
    p = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout)
    wall = time.time() - t0
    r1 = resource.getrusage(resource.RUSAGE_CHILDREN)
    out = p.stdout.decode(errors="replace")
    m = re.search(r"Average Speed:\s+([0-9.]+) fps", out)
    res = {"variant": variant, "rc": p.returncode, "fps": float(m.group(1)) if m else None, "wall_s": round(wall, 3),
           "cpu_s": round((r1.ru_utime - r0.ru_utime) + (r1.ru_stime - r0.ru_stime), 3),
           "ivf_md5": md5(ivf) if p.returncode == 0 and os.path.exists(ivf) else None,
           "rec_md5": md5(rec) if recon and p.returncode == 0 and os.path.exists(rec) else None}
    prof = [l for l in out.splitlines() if "CUDA profile" in l or "CUDA backend" in l]
    if prof:
        res["log"] = prof
    if p.returncode != 0:
        res["tail"] = out.splitlines()[-8:]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=640); ap.add_argument("--height", type=int, default=360)
    ap.add_argument("--frames", type=int, default=30); ap.add_argument("--preset", type=int, default=8)
    ap.add_argument("--qp", type=int, default=50); ap.add_argument("--bits", type=int, default=8)
    ap.add_argument("--variants", default="ref_c,cuda_c:me,cuda_c:dlf,cuda_c:cdef,cuda_c")
    ap.add_argument("--no-recon", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--workdir", default=None)
    ap.add_argument("--env", action="append", default=[], help="KEY=VALUE passed to the encoders (e.g. SVT_CUDA_ME_DS=1)")
    a = ap.parse_args()
    wd = a.workdir or tempfile.mkdtemp(prefix="svtenc_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    os.makedirs(wd, exist_ok=True)
    clip = os.path.join(wd, "clip_%dx%d_%d_%db.yuv" % (a.width, a.height, a.frames, a.bits))
    if not os.path.exists(clip):
        make_yuv.write_clip(clip, a.width, a.height, a.frames, a.bits)
    first = None
    for v in a.variants.split(","):
        r = run_variant(v, clip, a.width, a.height, a.frames, a.preset, a.qp, a.bits, wd, recon=not a.no_recon,
                        extra_env=dict([kv.split("=", 1) for kv in a.env], **({"SVT_CUDA_PROFILE": "1"} if a.profile else {})))
        if first is None:
            first = r
        r["same_as_first"] = (r["ivf_md5"] == first["ivf_md5"] and r["rec_md5"] == first["rec_md5"]) if r["ivf_md5"] else False
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
