"""Inputs that drive the transform / quantisation kernels to the edges of their range, and the checks that they get there.

- residual blocks: flat +max and -max, the Nyquist checkerboard, random signs at full magnitude;
- source / prediction pairs: full-swing pictures (every residual is +max or -max, pred = max - src, in 64x64 cells of
  flat, checkerboard and random-sign patterns) and the content_cases pictures (saturated, hard-edged, flat) against
  their complement;
- the real quantiser tables of the reference (tests/golden/quant_tables.json) at qindex 0, 1, 128 and 255;
- frame layouts: odd padding, pictures with odd chroma widths, and transform units tiled from the bottom-right corner of
  every plane, so that units touch the right and bottom edge and most first samples are not 4-byte aligned.

Next to them, the host-side checks that a case reaches the branch it exists for, read from the oracle's intermediates
(chain_reach): a quantiser input past the int16 clamp of the low-bit-depth quantisers that changes its level, a dequantised coefficient past the
inverse transform's input clamp, pred + residual outside [0, max] before the reconstruction clip, a unit whose first
sample is not 4-byte aligned.  A case that stops reaching its branch fails instead of passing vacuously."""
import ctypes as C
import json
import os

import numpy as np

import common as cm
import content_cases as cc
import svtb200 as sb
from test_oracle_txfm import TX_H, TX_W, allowed_types

QUANT_JSON = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "quant_tables.json")
QINDEXES = (0, 1, 128, 255)
QKEYS = ("quant", "quant_shift", "zbin", "round", "quant_fp", "round_fp", "dequant")


def maxv(bd):
    return (1 << bd) - 1


def bpc(ts):
    """Transform units per CTA of the fused kernel (128 lanes, one per column / row of the longer side)."""
    return 128 // max(TX_W[ts], TX_H[ts])


def log_scale(ts):
    n = TX_W[ts] * TX_H[ts]
    return (n > 256) + (n > 1024)


# ---- quantiser tables --------------------------------------------------------------------------------------------
_tables = None


def quant_fixture():
    global _tables
    if _tables is None:
        with open(QUANT_JSON) as f:
            _tables = json.load(f)["tables"]
    return _tables


def quant_arrays(bd, qindex):
    """{key: int16 [dc, ac]} of the reference's luma tables."""
    t = quant_fixture()[str(bd)][str(qindex)]
    return {k: np.array(t[k], np.int16) for k in QKEYS}


def quant_plane(bd, qindex):
    a = quant_arrays(bd, qindex)
    q = sb.QuantPlane()
    for i in range(2):
        for k in QKEYS:
            getattr(q, k)[i] = int(a[k][i])
    return q


def encode_params(ts, bd, qindex, use_fp):
    p = sb.EncodeParams()
    p.tx_size, p.use_fp = ts, use_fp
    for i in range(3):
        p.q[i] = quant_plane(bd, qindex)
    return p


# ---- residual blocks ---------------------------------------------------------------------------------------------
RESIDUALS = ("flat_max", "flat_min", "checker", "signs")


def residual(kind, w, h, bd, rng, stride=None):
    """An int16 residual block (h x stride, stride >= w) at full magnitude: flat +max / -max, the Nyquist checkerboard
    (+max where row + column is even), or random signs."""
    mx = maxv(bd)
    stride = stride or w
    if kind == "flat_max":
        return np.full((h, stride), mx, np.int16)
    if kind == "flat_min":
        return np.full((h, stride), -mx, np.int16)
    if kind == "checker":
        y, x = np.mgrid[0:h, 0:stride]
        return np.where((x + y) % 2 == 0, mx, -mx).astype(np.int16)
    assert kind == "signs"
    return (rng.choice([-1, 1], (h, stride)) * mx).astype(np.int16)


# ---- pictures ----------------------------------------------------------------------------------------------------
def full_swing_picture(w, h, bd, seed=0, pad=16):
    """A picture of 0 and max only: per 64x64 cell of each plane, flat max, flat 0, a one-sample checkerboard or random
    rails.  Against its complement as prediction every residual is +max or -max."""
    rng = np.random.default_rng(seed)
    f = cm.Yuv(w, h, bd, pad)
    mx = maxv(bd)
    for i in range(3):
        p = f.plane(i)
        ph, pw = p.shape
        y, x = np.mgrid[0:ph, 0:pw]
        kind = ((y // 64) + (x // 64) + i) % 4
        checker = np.where((x + y) % 2 == 0, mx, 0)
        rails = rng.choice([0, mx], (ph, pw))
        p[...] = np.select([kind == 0, kind == 1, kind == 2], [mx, 0, checker], rails)
    return f


def complement(f):
    """max - f: as a prediction of f, the residual is 2 f - max."""
    o = f.copy()
    for i in range(3):
        o.plane(i)[...] = maxv(f.bd) - f.plane(i).astype(np.int64)
    return o


def with_pad(f, pad):
    o = cm.Yuv(f.w, f.h, f.bd, pad)
    for i in range(3):
        o.plane(i)[...] = f.plane(i)
    return o


def pair(kind, w, h, bd, seed=0, pad=16):
    """(source, prediction) at full range: the source against its complement."""
    if kind == "full_swing":
        src = full_swing_picture(w, h, bd, seed, pad)
    else:
        src = with_pad(cc.PICTURES[kind](w, h, bd, seed), pad)
    return src, complement(src)


# ---- unit layouts ------------------------------------------------------------------------------------------------
def plane_dims(w, h, pl):
    return (w, h) if pl == 0 else ((w + 1) // 2, (h + 1) // 2)


def corner_tus(rng, ts, w_pic, h_pic, planes=(0, 1, 2), limit=None):
    """Non-overlapping units of size ts tiled from the bottom-right corner of every plane: the last column of units
    touches the right edge and the last row the bottom edge.  `limit` keeps the corner unit of every plane, up to half
    the limit of other units on the right or bottom edge, and fills the rest at random."""
    w, h = TX_W[ts], TX_H[ts]
    types = allowed_types(ts)
    cand = []
    for pl in planes:
        pw, ph = plane_dims(w_pic, h_pic, pl)
        for y in range(ph - h, -1, -h):
            for x in range(pw - w, -1, -w):
                cand.append((x, y, pl, 2 if (x + w == pw and y + h == ph) else int(x + w == pw or y + h == ph)))
    if limit and len(cand) > limit:
        keep = {i for i, c in enumerate(cand) if c[3] == 2}
        edge = [i for i, c in enumerate(cand) if c[3] == 1]
        keep |= set(rng.choice(edge, min(len(edge), max(0, limit // 2 - len(keep))), replace=False).tolist())
        rest = [i for i in range(len(cand)) if i not in keep]
        keep |= set(rng.choice(rest, max(0, limit - len(keep)), replace=False).tolist())
        cand = [cand[i] for i in sorted(keep)]
    return [sb.Tu(x, y, pl, int(rng.choice(types))) for x, y, pl, _ in cand]


def corner_mixed_tus(rng, w_pic, h_pic, n_qsets, per_cell=6):
    """Units of mixed sizes, shapes and quantiser sets (sb.TuEx) for svt_b200_encode_tus_ex: 64x64 cells tiled from the
    bottom-right corner of every plane, each cell tiled with one random size, `per_cell` of its units kept (its
    bottom-right one always, so every plane has a unit in its bottom-right corner), the list shuffled."""
    tus = []
    for pl in range(3):
        pw, ph = plane_dims(w_pic, h_pic, pl)
        for cy in range(ph - 64, -1, -64):
            for cx in range(pw - 64, -1, -64):
                ts = int(rng.integers(0, 19))
                w, h = TX_W[ts], TX_H[ts]
                cell = [(cx + x, cy + y) for y in range(0, 64, h) for x in range(0, 64, w)]
                picks = [len(cell) - 1] + list(rng.choice(len(cell) - 1, min(len(cell) - 1, per_cell - 1), replace=False))
                for k in picks:
                    x, y = cell[int(k)]
                    tus.append(sb.TuEx(x, y, pl, int(rng.choice(allowed_types(ts))), ts, int(rng.integers(0, 4)),
                                       int(rng.integers(0, n_qsets)), 0))
    return [tus[int(i)] for i in rng.permutation(len(tus))]


def first_sample_offset(f, tu):
    """Byte offset of a unit's first sample from the start of its plane buffer (numpy and the device copies of
    gpu_runner.DevYuv allocate 4-byte aligned buffers, so this is its alignment)."""
    b = f.bufs[tu.plane]
    return ((f.pad + tu.y) * b.shape[1] + f.pad + tu.x) * b.itemsize


def misaligned_units(f, tus):
    return sum(first_sample_offset(f, t) % 4 != 0 for t in tus)


def edge_planes(f, tus, ts):
    """Planes in which some unit of size ts touches the right edge and some unit the bottom edge."""
    w, h = TX_W[ts], TX_H[ts]
    out = set()
    for pl in range(3):
        pw, ph = plane_dims(f.w, f.h, pl)
        mine = [t for t in tus if t.plane == pl]
        if any(t.x + w == pw for t in mine) and any(t.y + h == ph for t in mine):
            out.add(pl)
    return out


# ---- the oracle chain with its intermediates ---------------------------------------------------------------------
class Reach:
    """What one oracle run got to: counts of levels the int16 clamp changes (low bit depth), of inverse inputs
    past the clamp at bd + 8 bits, of samples where pred + residual left [0, max], and the largest |coefficient|."""

    def __init__(self):
        self.int16_clamp = 0
        self.inv_clamp = 0
        self.recon_clip = 0
        self.max_coeff = 0
        self.max_dequant = 0

    def __iadd__(self, o):
        for k in vars(self):
            setattr(self, k, max(getattr(self, k), getattr(o, k)) if k.startswith("max") else getattr(self, k) + getattr(o, k))
        return self

    def __repr__(self):
        return "Reach(" + ", ".join(f"{k}={v}" for k, v in vars(self).items()) + ")"


def rpot(v, n):
    return (v + (1 << (n - 1))) >> n if n else v


def quant_reach(coeff, qa, ls, bd, use_fp):
    """Coefficients (raster, n of them) whose level the int16 clamp of the low-bit-depth quantisers changes: kept by the
    zbin / dequant test, |c| + round past 32767, and a different level than the unclamped sum would give (0 at high
    bit depth, where there is no clamp)."""
    if bd > 8:
        return 0
    a = np.abs(coeff.astype(np.int64))
    ac = np.ones(a.size, bool)
    ac[0] = False

    def pick(k):
        return np.where(ac, int(qa[k][1]), int(qa[k][0]))

    if use_fp:
        tmp = a + np.where(ac, rpot(int(qa["round_fp"][1]), ls), rpot(int(qa["round_fp"][0]), ls))
        kept = (a << (1 + ls)) >= pick("dequant")

        def level(t):
            return (t * pick("quant_fp")) >> (16 - ls)
    else:
        tmp = a + np.where(ac, rpot(int(qa["round"][1]), ls), rpot(int(qa["round"][0]), ls))
        kept = a * 32 >= (np.where(ac, rpot(int(qa["zbin"][1]), ls), rpot(int(qa["zbin"][0]), ls)) << 5)

        def level(t):
            t = t * 32
            return ((((t * pick("quant")) >> 16) + t) * pick("quant_shift")) >> (16 - ls + 5)
    return int((kept & (tmp > 32767) & (level(np.minimum(tmp, 32767)) != level(tmp))).sum())


def inv_input_reach(dq, ts, bd):
    """Dequantised coefficients that the inverse transform's input clamp (bd + 8 bits, after the 1/sqrt(2) of 2:1
    rectangles) changes."""
    w, h = TX_W[ts], TX_H[ts]
    v = dq.astype(np.int64)
    if w == 2 * h or h == 2 * w:
        v = (v * 2896 + 2048) >> 12
    lim = (1 << (bd + 7)) - 1
    return int(((v > lim) | (v < -lim - 1)).sum())


def inverse_residual(dq, ts, tx_type, bd):
    """The inverse transform's residual, clamped to [-max, max], from two oracle runs on a prediction of 0 and of max
    (pred + this residual leaves [0, max] only where pred + the true residual does)."""
    w, h = TX_W[ts], TX_H[ts]
    orc = cm.oracle()
    mx = maxv(bd)
    lo, hi = np.zeros((h, w), np.uint16), np.zeros((h, w), np.uint16)
    p0, p1 = np.zeros((h, w), np.uint16), np.full((h, w), mx, np.uint16)
    orc.orc_inv_txfm2d_add(cm.ptr(dq), cm.ptr(p0), w, cm.ptr(lo), w, tx_type, ts, bd)
    orc.orc_inv_txfm2d_add(cm.ptr(dq), cm.ptr(p1), w, cm.ptr(hi), w, tx_type, ts, bd)
    return lo.astype(np.int64) - (mx - hi.astype(np.int64))


def chain_reach(params, src, pred, tus, use_fp):
    """The Reach of the per-unit chain of oracle_encode_tus (test_txfm_gpu.py): residual, forward transform, quantiser,
    inverse transform, with the same oracle calls; every plane quantises with params.q[0]."""
    orc = cm.oracle()
    ts = params.tx_size
    w, h = TX_W[ts], TX_H[ts]
    n = min(w, 32) * min(h, 32)
    bd = src.bd
    hbd = 1 if bd > 8 else 0
    ls = log_scale(ts)
    qp = params.q[0]
    qa = {k: np.array(getattr(qp, k)[:], np.int16) for k in QKEYS}
    reach = Reach()
    for tu in tus:
        sblk = np.ascontiguousarray(src.plane(tu.plane)[tu.y:tu.y + h, tu.x:tu.x + w])
        pblk = np.ascontiguousarray(pred.plane(tu.plane)[tu.y:tu.y + h, tu.x:tu.x + w])
        res = np.zeros((h, w), np.int16)
        orc.orc_residual(cm.ptr(sblk), C.c_uint32(w), cm.ptr(pblk), C.c_uint32(w), cm.ptr(res), C.c_uint32(w), C.c_uint32(w),
                         C.c_uint32(h), hbd)
        coeff = np.zeros(w * h, np.int32)
        orc.orc_fwd_txfm2d(cm.ptr(res), cm.ptr(coeff), C.c_uint32(w), tu.tx_type, ts, bd)
        if max(w, h) == 64:
            orc.orc_handle_transform64(cm.ptr(coeff), ts)
        scan = scan_of(ts, tu.tx_type)
        q, dq, eob = np.zeros(n, np.int32), np.zeros(n, np.int32), C.c_uint16(0)
        if use_fp:
            orc.orc_quantize_fp(cm.ptr(coeff), C.c_ssize_t(n), cm.ptr(qa["round_fp"]), cm.ptr(qa["quant_fp"]), cm.ptr(q), cm.ptr(dq),
                                cm.ptr(qa["dequant"]), C.byref(eob), cm.ptr(scan), ls, hbd)
        else:
            orc.orc_quantize_b(cm.ptr(coeff), C.c_ssize_t(n), cm.ptr(qa["zbin"]), cm.ptr(qa["round"]), cm.ptr(qa["quant"]),
                               cm.ptr(qa["quant_shift"]), cm.ptr(q), cm.ptr(dq), cm.ptr(qa["dequant"]), C.byref(eob), cm.ptr(scan),
                               None, None, ls, hbd)
        r = Reach()
        r.max_coeff = int(np.abs(coeff[:n].astype(np.int64)).max())
        r.max_dequant = int(np.abs(dq.astype(np.int64)).max())
        r.int16_clamp = quant_reach(coeff[:n], qa, ls, bd, use_fp)
        r.inv_clamp = inv_input_reach(dq, ts, bd)
        v = pblk.astype(np.int64) + inverse_residual(dq, ts, tu.tx_type, bd)
        r.recon_clip = int(((v < 0) | (v > maxv(bd))).sum())
        reach += r
    return reach


_scans = {}


def scan_of(ts, tx_type):
    """The scan order of (size, type) from the product's table; test_txfm_gpu checks it against the reference's."""
    key = (ts, tx_type)
    if key not in _scans:
        s = np.zeros(1024, np.int16)
        assert sb.load().svt_b200_get_scan(ts, tx_type, cm.ptr(s)) > 0
        _scans[key] = s
    return _scans[key]
