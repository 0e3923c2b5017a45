#!/usr/bin/env python
"""Regenerates tests/golden/quant_tables.json from the unmodified reference (needs oracle/_ref):
python tests/golden/make_quant_tables.py

The luma quantiser tables that svt_av1_build_quantizer builds (no delta-q, so chroma is the same) at bit depths 8 and
10, for qindex 0, 1, 128 and 255: the dc / ac pairs of quant, quant_shift, zbin, round, quant_fp, round_fp and the
dequantiser in transform scale (dequant_qtx)."""
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.join(ROOT, "svt-av1_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import common as cm  # noqa: E402

QINDEX_RANGE = 256
QINDEXES = (0, 1, 128, 255)
# Quants (EbPictureControlSet.h): int16 [QINDEX_RANGE][8] arrays in this order; entry 0 is dc, 1 ac
QUANTS_FIELDS = ("y_quant", "y_quant_shift", "y_zbin", "y_round", "y_quant_fp", "u_quant_fp", "v_quant_fp", "y_round_fp",
                 "u_round_fp", "v_round_fp", "u_quant", "v_quant", "u_quant_shift", "v_quant_shift", "u_zbin", "v_zbin",
                 "u_round", "v_round")
DEQUANTS_FIELDS = ("y_dequant_qtx", "u_dequant_qtx", "v_dequant_qtx", "y_dequant_q3", "u_dequant_q3", "v_dequant_q3")
KEYS = ("quant", "quant_shift", "zbin", "round", "quant_fp", "round_fp", "dequant")


def build(bd):
    """{field: int16 [QINDEX_RANGE][8]} of svt_av1_build_quantizer(bd, no delta-q)."""
    quants = np.zeros((len(QUANTS_FIELDS), QINDEX_RANGE, 8), np.int16)
    deq = np.zeros((len(DEQUANTS_FIELDS), QINDEX_RANGE, 8), np.int16)
    cm.ref().svt_av1_build_quantizer(bd, 0, 0, 0, 0, 0, cm.ptr(quants), cm.ptr(deq))
    out = dict(zip(QUANTS_FIELDS, quants))
    out.update(zip(DEQUANTS_FIELDS, deq))
    return out


def luma_tables(bd):
    t = build(bd)
    src = {"quant": "y_quant", "quant_shift": "y_quant_shift", "zbin": "y_zbin", "round": "y_round",
           "quant_fp": "y_quant_fp", "round_fp": "y_round_fp", "dequant": "y_dequant_qtx"}
    return {str(q): {k: [int(v) for v in t[src[k]][q, :2]] for k in KEYS} for q in QINDEXES}


def main():
    assert cm.have_ref(), "build oracle/_ref first (make -C oracle)"
    out = {"source": "svt-av1 v0.8.6 svt_av1_build_quantizer (oracle/_ref), luma, no delta-q; [dc, ac] pairs per qindex",
           "tables": {str(bd): luma_tables(bd) for bd in (8, 10)}}
    with open(os.path.join(HERE, "quant_tables.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
