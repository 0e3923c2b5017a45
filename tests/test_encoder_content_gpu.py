"""Encoder-level parity on hard content: the CUDA-backed encoder and the C-only reference encoder produce the same .ivf
and the same reconstruction on a clip of a fade from black, flat grey, saturated texture, hard-edged graphics, identical
static frames and a cut (content_cases.hard_clip_frames), and deblocking and CDEF ran on the GPU."""
import os
import re
import sys

import pytest

import content_cases as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import encode_compare as ec  # noqa: E402

pytestmark = pytest.mark.gpu

have = all(os.path.exists(ec.APPS[v]) for v in ("ref_c", "cuda_c"))


@pytest.mark.skipif(not have, reason="oracle/_ref/integration or oracle/_ref/app not built (python __graft_entry__.py)")
@pytest.mark.parametrize("preset,bits", [(8, 8), (6, 10)])
def test_hard_content_clip_bitstream_and_recon_md5(tmp_path, preset, bits):
    """640x360, CQP qp 50.  Screen-content detection is turned off (-scm 0): with it on, hard-edged pictures can be
    classified as screen content, whose ME search windows the GPU ME entry does not support; this test is about the
    filters on hard content, not about that path.

    CDEF runs on the GPU for every picture at both presets (cdef_level 4 on every picture above preset 3).  At preset 6
    (loop_filter_mode 3) every picture is deblocked on the GPU, with the level search.  At preset 8 the encoder deblocks
    reference pictures only (loop_filter_mode 1 for reference pictures, 0 otherwise): in the hierarchical mini-GOPs at
    least every second picture is a reference, and the top-layer pictures are not."""
    clip = str(tmp_path / ("hard_%d.yuv" % bits))
    n = cc.write_hard_clip(clip, 640, 360, bits)
    args = ("-scm", "0")
    ref = ec.run_variant("ref_c", clip, 640, 360, n, preset, 50, bits, str(tmp_path), extra_args=args)
    gpu = ec.run_variant("cuda_c", clip, 640, 360, n, preset, 50, bits, str(tmp_path), extra_args=args,
                         extra_env={"SVT_CUDA_PROFILE": "1"})
    assert ref["rc"] == 0 and gpu["rc"] == 0, (ref, gpu)
    assert ref["ivf_md5"] and ref["ivf_md5"] == gpu["ivf_md5"], (ref, gpu)
    assert ref["rec_md5"] and ref["rec_md5"] == gpu["rec_md5"], (ref, gpu)
    log = " ".join(gpu.get("log", []))
    m = re.search(r"engine: (\d+) ME pictures .*?, (\d+) dlf, (\d+) cdef", log)
    assert m, gpu.get("log")
    n_me, n_dlf, n_cdef = (int(x) for x in m.groups())
    assert n_me >= 1 and n_cdef == n, (n_me, n_dlf, n_cdef, n)
    if preset <= 6:
        assert n_dlf == n, (n_dlf, n)
    else:
        assert (n - 1) // 2 <= n_dlf < n, (n_dlf, n)
