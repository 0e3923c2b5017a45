"""Encoder-level parity (SURVEY.md 8c(3), VERDICT r1 item 1): the reference encoder with the CUDA backend bound in
(oracle/_ref/integration, SVT_CUDA=1) must produce the SAME .ivf bitstream and the SAME reconstruction as the plain C-only
reference encoder on the same synthetic YUV, through the reference's own application and API.  The encoder is
deterministic, so the comparison is an md5 equality.  Everything here runs the prebuilt binaries: no reference source is read at
run time."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import encode_compare as ec  # noqa: E402
import make_yuv  # noqa: E402

pytestmark = pytest.mark.gpu

need = [ec.APPS["ref_c"], ec.APPS["cuda_c"], ec.APPS["ref_simd"], ec.APPS["cuda_simd"]]
have = all(os.path.exists(p) for p in need)
skip_if_unbuilt = pytest.mark.skipif(not have, reason="oracle/_ref/integration or oracle/_ref/app not built (python __graft_entry__.py)")


def _clip(tmp_path, w, h, frames, bits):
    p = str(tmp_path / ("clip_%dx%d_%d_%d.yuv" % (w, h, frames, bits)))
    make_yuv.write_clip(p, w, h, frames, bits)
    return p


def _same(a, b):
    assert a["rc"] == 0 and b["rc"] == 0, (a, b)
    assert a["ivf_md5"] and a["ivf_md5"] == b["ivf_md5"], (a, b)
    assert a["rec_md5"] and a["rec_md5"] == b["rec_md5"], (a, b)


@skip_if_unbuilt
@pytest.mark.parametrize("stages", ["me", "dlf", "cdef", "me+dlf+cdef"])
def test_config1_360p_preset8_bitstream_and_recon_md5(tmp_path, stages):
    """BASELINE configs[0]: 640x360 8-bit, 30 frames, preset 8, CQP qp 50 - each GPU stage alone and all together."""
    clip = _clip(tmp_path, 640, 360, 30, 8)
    ref = ec.run_variant("ref_c", clip, 640, 360, 30, 8, 50, 8, str(tmp_path))
    gpu = ec.run_variant("cuda_c:" + stages, clip, 640, 360, 30, 8, 50, 8, str(tmp_path), extra_env={"SVT_CUDA_PROFILE": "1"})
    _same(ref, gpu)
    # the stage really ran on the GPU (the backend's profile line counts engine calls)
    log = " ".join(gpu.get("log", []))
    assert "ME pictures" in log
    import re
    m = re.search(r"engine: (\d+) ME pictures .*?, (\d+) dlf, (\d+) cdef", log)
    n_me, n_dlf, n_cdef = (int(x) for x in m.groups())
    assert (n_me > 0) == ("me" in stages) and (n_dlf > 0) == ("dlf" in stages) and (n_cdef > 0) == ("cdef" in stages), log


@skip_if_unbuilt
def test_360p_preset8_device_side_me_downsample(tmp_path):
    """SVT_CUDA_ME_DS=1: only the full-resolution luma is uploaded, the 1/4 and 1/16 HME planes are derived on the device
    (svt_b200_me_downsample) - the encode must not change."""
    clip = _clip(tmp_path, 640, 360, 20, 8)
    ref = ec.run_variant("ref_c", clip, 640, 360, 20, 8, 50, 8, str(tmp_path))
    gpu = ec.run_variant("cuda_c:me", clip, 640, 360, 20, 8, 50, 8, str(tmp_path), extra_env={"SVT_CUDA_ME_DS": "1"})
    _same(ref, gpu)


@skip_if_unbuilt
def test_10bit_preset6_bitstream_and_recon_md5(tmp_path):
    """A 10-bit preset-6 clip (the configs[2] stage set at a small size): 16-bit pipeline, loop_filter_mode 3 (level search +
    deblocking in dlf_kernel as one GPU call), CDEF on 16-bit planes, restoration search on the CPU and apply on the GPU."""
    clip = _clip(tmp_path, 640, 360, 24, 10)
    ref = ec.run_variant("ref_c", clip, 640, 360, 24, 6, 50, 10, str(tmp_path))
    gpu = ec.run_variant("cuda_c", clip, 640, 360, 24, 6, 50, 10, str(tmp_path), extra_env={"SVT_CUDA_PROFILE": "1"})
    _same(ref, gpu)
    import re
    m = re.search(r"engine: (\d+) ME pictures .*?, (\d+) dlf, (\d+) cdef, (\d+) lr", " ".join(gpu.get("log", [])))
    n_me, n_dlf, n_cdef, n_lr = (int(x) for x in m.groups())
    # every picture is deblocked (level search included) and CDEF-filtered on the GPU; the pictures whose restoration search
    # (CPU) picked Wiener / self-guided units are restored on the GPU from the saved boundary lines
    assert n_dlf == 24 and n_cdef == 24 and n_me >= 22 and n_lr >= 1, gpu.get("log")


@skip_if_unbuilt
def test_simd_build_with_cuda_backend_matches_simd_reference(tmp_path):
    """The speed build (reference AVX2/AVX-512 code + CUDA backend) against the reference's SIMD encoder, ragged size
    (not a multiple of 64), through the API driver the bench uses as well."""
    clip = _clip(tmp_path, 720, 400, 24, 8)
    ref = ec.run_variant("ref_simd", clip, 720, 400, 24, 8, 43, 8, str(tmp_path))
    gpu = ec.run_variant("cuda_simd", clip, 720, 400, 24, 8, 43, 8, str(tmp_path))
    _same(ref, gpu)


@skip_if_unbuilt
def test_gop_sharded_encode_matches_cpu_per_substream(tmp_path):
    """BASELINE configs[4] sharding (one stream, closed GOPs round-robin over encoder instances): every rank's CUDA-backed
    sub-stream is bit-identical to the CPU reference encode of the same sub-clip; the splice holds every packet once."""
    import json
    import subprocess
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "shard_encode.py"), "--width", "640", "--height", "360", "--frames", "96",
                        "--gop", "32", "--gpus", "2", "--sequential", "--variant", "cuda_simd", "--verify", "--decode", "--preset", "8", "--qp", "50",
                        "--workdir", str(tmp_path)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1800)
    assert r.returncode == 0, (r.stdout.decode()[-1500:], r.stderr.decode()[-1500:])
    d = json.loads(r.stdout.decode().strip().splitlines()[-1])
    assert d["parity"] is True and d["packets"] == 96
    assert d["decode_matches_recon"] is True  # the GOP-spliced stream decodes (reference decoder) to the spliced reconstructions


@skip_if_unbuilt
@pytest.mark.parametrize("switch,bits,preset", [("SVT_CUDA_TF", 8, 8), ("SVT_CUDA_TF", 10, 6), ("SVT_CUDA_PA", 8, 8), ("SVT_CUDA_OIS", 8, 8)])
def test_parity_switches_temporal_filter_picture_analysis_open_loop_intra(tmp_path, switch, bits, preset):
    """SVT_CUDA_OIS=1: the open-loop intra search of the TPL path (rank 3, presets >= 5: DC_PRED) for a whole picture in one GPU
    call.  The two rank-4 stages inside the real encoder (off by default: they are bit-exact but do not pay - one GPU round trip
    per 32x32 block / per picture): SVT_CUDA_TF=1 points the reference's temporal-filter RTCD pointers at the GPU drop-ins
    (every filtered sample of the key / base pictures goes through the reproduced double / expf chain), SVT_CUDA_PA=1 takes
    pcs->y_mean / variance / cb_mean / cr_mean / pic_avg_variance from svt_b200_picture_mean_variance.  The stream and the
    reconstruction must not change."""
    import re
    clip = _clip(tmp_path, 640, 360, 18, bits)
    ref = ec.run_variant("ref_c", clip, 640, 360, 18, preset, 50, bits, str(tmp_path))
    gpu = ec.run_variant("cuda_c", clip, 640, 360, 18, preset, 50, bits, str(tmp_path), extra_env={switch: "1", "SVT_CUDA_PROFILE": "1"})
    _same(ref, gpu)
    m = re.search(r"tf blocks on the GPU (\d+), picture-analysis pictures on the GPU (\d+), open-loop intra pictures on the GPU (\d+)",
                  " ".join(gpu.get("log", [])))
    assert m, gpu.get("log")
    n_tf, n_pa, n_ois = (int(x) for x in m.groups())
    if switch == "SVT_CUDA_TF":
        assert n_tf > 100 and n_pa == 0 and n_ois == 0, (n_tf, n_pa, n_ois)
    elif switch == "SVT_CUDA_PA":
        assert n_pa == 18 and n_tf == 0 and n_ois == 0, (n_tf, n_pa, n_ois)
    else:
        assert n_ois >= 1 and n_tf == 0 and n_pa == 0, (n_tf, n_pa, n_ois)


DEC = os.path.join(ROOT, "oracle", "_ref", "app", "SvtAv1DecApp")


@skip_if_unbuilt
@pytest.mark.skipif(not os.path.exists(DEC), reason="oracle/_ref/app/SvtAv1DecApp not built")
@pytest.mark.parametrize("bits,preset", [(8, 8), (10, 6)])
def test_conformance_decoder_output_equals_cuda_encoder_recon(tmp_path, bits, preset):
    """SURVEY 8c(3) conformance, independent of the C-only encoder: the bitstream of the CUDA-backed encoder, decoded by the
    reference's own AV1 decoder, equals the encoder's reconstruction (which the GPU deblocking / CDEF produced)."""
    import subprocess
    clip = _clip(tmp_path, 640, 360, 16, bits)
    gpu = ec.run_variant("cuda_c", clip, 640, 360, 16, preset, 50, bits, str(tmp_path))
    assert gpu["rc"] == 0 and gpu["rec_md5"]
    dec = str(tmp_path / "dec.yuv")
    p = subprocess.run([DEC, "-i", str(tmp_path / "cuda_c.ivf"), "-o", dec] + (["-bit-depth", str(bits)] if bits != 8 else []),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900)
    assert p.returncode == 0, p.stdout.decode(errors="replace")[-1500:]
    assert ec.md5(dec) == gpu["rec_md5"]
