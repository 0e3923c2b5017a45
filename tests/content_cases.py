"""Seeded pictures for the in-loop filter and ME tests that the smooth synthetic texture (common.synth_yuv) never produces:
flat pictures and flat areas, texture clipped hard at 0 and at the maximum, ladders of step edges with a checkerboard and
glyph blocks, and reconstructions equal to (or differing in a few blocks from) their source; plus CDEF skip maps that skip
every 8x8 block, none, or whole 64x64 filter blocks.  Each luma / chroma plane is generated on its own.

Next to the generators are the host-side checks that a case reaches the branch it exists for (a CDEF block of zero variance,
equal level-search SSEs, every deblocking mask decision, samples on both rails), so a case that stops reaching it fails
instead of passing vacuously."""
import ctypes as C

import numpy as np

import common as cm
import svtb200 as sb

BIT_DEPTHS = (8, 10)


def maxv(bd):
    return (1 << bd) - 1


def plane_shapes(w, h):
    return [(h, w), ((h + 1) // 2, (w + 1) // 2), ((h + 1) // 2, (w + 1) // 2)]


def from_planes(w, h, bd, planes):
    f = cm.Yuv(w, h, bd)
    for i, p in enumerate(planes):
        f.plane(i)[...] = np.clip(p, 0, maxv(bd))
    return f


# ---- flat ------------------------------------------------------------------------------------------------------------
def flat(w, h, bd, level):
    """Every sample of every plane at `level` ('zero', 'mid', 'max' or a sample value)."""
    v = {"zero": 0, "mid": 1 << (bd - 1), "max": maxv(bd)}.get(level, level)
    return from_planes(w, h, bd, [np.full(s, v, np.int64) for s in plane_shapes(w, h)])


def flat_regions(w, h, bd, seed=0):
    """Flat rectangles at several levels (0 and the maximum among them) separated by sharp edges; the rectangle grid is
    drawn per plane, with edges on and off the 8-sample grid."""
    rng = np.random.default_rng(seed)
    mx = maxv(bd)
    planes = []
    for ph, pw in plane_shapes(w, h):
        levels = [0, mx, 1 << (bd - 1), mx // 4, 3 * mx // 4, 1, mx - 1]
        xs = np.unique(np.concatenate([[0], rng.integers(1, pw, 5), [16, 40, 47]]))
        ys = np.unique(np.concatenate([[0], rng.integers(1, ph, 4), [24, 33]]))
        xs, ys = xs[xs < pw], ys[ys < ph]
        p = np.zeros((ph, pw), np.int64)
        for i, y0 in enumerate(ys):
            for j, x0 in enumerate(xs):
                p[y0:, x0:] = levels[(i * len(xs) + j + int(rng.integers(0, 3))) % len(levels)]
        planes.append(p)
    return from_planes(w, h, bd, planes)


# ---- saturated -------------------------------------------------------------------------------------------------------
def saturated(w, h, bd, seed=0):
    """A texture of three times the sample range, clipped: large areas exactly 0 or exactly the maximum, and next to the
    rails a few codes of noise (also clipped)."""
    rng = np.random.default_rng(seed)
    mx = maxv(bd)
    sc = 1 << (bd - 8)
    planes = []
    for k, (ph, pw) in enumerate(plane_shapes(w, h)):
        y, x = np.mgrid[0:ph, 0:pw].astype(np.float64)
        t = np.sin(x / (9.0 + 4 * k) + 0.7 * k) + np.cos(y / (7.0 + 3 * k))
        v = (0.5 + 0.75 * t) * mx
        v = np.clip(np.rint(v), 0, mx)
        near = (v <= 4 * sc) | (v >= mx - 4 * sc)
        noise = rng.integers(-3 * sc, 3 * sc + 1, v.shape) * near * (rng.random(v.shape) < 0.5)
        planes.append(np.clip(v + noise, 0, mx).astype(np.int64))
    return from_planes(w, h, bd, planes)


# ---- hard edges ------------------------------------------------------------------------------------------------------
def _ladder(n, mx, edges, base):
    """1-d profile of n samples at `base` (0 or mx) with pulses away from it: the pulse k spans edges[2k]..edges[2k+1], so
    both of its edges have contrast c_k, and c_k rises from 1 code to the full range along the profile."""
    pos = [p for p in edges if 0 < p < n]
    pos = pos[:len(pos) // 2 * 2]
    contrasts = np.rint(np.geomspace(1, mx, max(1, len(pos) // 2))).astype(np.int64)
    prof = np.full(n, base, np.int64)
    for k in range(len(pos) // 2):
        prof[pos[2 * k]:pos[2 * k + 1]] = base + int(contrasts[k]) if base == 0 else base - int(contrasts[k])
    return prof


EDGE_OFFSETS = (8, 0, 4, 3, 13, 5)  # in consecutive 16-sample blocks: 8-aligned, 16-aligned, 4-aligned, off the grid


def edge_positions(n):
    """Step positions 16 * k + EDGE_OFFSETS[k % 6]: on 16-, 8- and 4-sample boundaries and off them, at least 8 apart."""
    return [16 * k + EDGE_OFFSETS[k % 6] for k in range(n // 16 + 1) if 0 < 16 * k + EDGE_OFFSETS[k % 6] < n]


def hard_edges(w, h, bd, seed=0):
    """Per plane: vertical step edges in the upper half (pulses up from 0) and horizontal ones in the lower half (pulses down
    from the maximum), a ladder of contrasts from 1 to the full range on and off 4 / 8 / 16-sample transform boundaries; a band with small noise near the edges (high
    edge variance), a checkerboard and binary 'glyph' blocks at offsets that are not multiples of 8."""
    rng = np.random.default_rng(seed)
    mx = maxv(bd)
    sc = 1 << (bd - 8)
    planes = []
    for k, (ph, pw) in enumerate(plane_shapes(w, h)):
        p = np.zeros((ph, pw), np.int64)
        top = ph // 2
        p[:top] = _ladder(pw, mx, edge_positions(pw), 0)[None, :]
        p[top:] = _ladder(ph - top, mx, edge_positions(ph - top), mx)[:, None]
        # rows with a few codes of noise: |p1 - p0| beyond the hev threshold on some edges, inside the mask on others
        band = slice(top // 3, top // 3 + max(4, top // 6))
        p[band] += rng.integers(-4 * sc, 4 * sc + 1, p[band].shape)
        # checkerboard of 3-sample cells
        cy, cx = 5 + 8 * (k % 2), 13
        ch, cw = min(24, ph - cy), min(30, pw - cx)
        if ch > 0 and cw > 0:
            yy, xx = np.mgrid[0:ch, 0:cw]
            p[cy:cy + ch, cx:cx + cw] = np.where(((yy // 3) + (xx // 3)) % 2, mx, 0)
        # 5x7 glyphs, 0 on the maximum and the maximum on 0, at odd offsets
        for g in range(6):
            gy, gx = int(rng.integers(0, max(1, ph - 9))) | 1, int(rng.integers(0, max(1, pw - 7))) | 1
            bits = rng.random((7, 5)) < 0.5
            blk = p[gy:gy + 7, gx:gx + 5]
            blk[...] = np.where(bits[:blk.shape[0], :blk.shape[1]], mx if g % 2 else 0, 0 if g % 2 else mx)
        planes.append(p)
    return from_planes(w, h, bd, planes)


# ---- static ----------------------------------------------------------------------------------------------------------
def changed_blocks(src, seed=0, n=4, amp=9):
    """`src` with `n` 8x8 luma blocks (and the 4x4 chroma blocks under them) moved by up to `amp` codes, clipped."""
    rng = np.random.default_rng(seed)
    out = src.copy()
    sc = 1 << (src.bd - 8)
    for _ in range(n):
        by, bx = int(rng.integers(0, src.h // 8)), int(rng.integers(0, src.w // 8))
        for i in range(3):
            s = 8 if i == 0 else 4
            blk = out.plane(i)[by * s:(by + 1) * s, bx * s:(bx + 1) * s]
            d = int(rng.integers(1, amp + 1)) * (1 if rng.random() < 0.5 else -1) * sc
            blk[...] = np.clip(blk.astype(np.int64) + d, 0, maxv(src.bd))
    return out


# name -> picture(w, h, bd, seed)
PICTURES = {
    "flat_zero": lambda w, h, bd, seed: flat(w, h, bd, "zero"),
    "flat_mid": lambda w, h, bd, seed: flat(w, h, bd, "mid"),
    "flat_max": lambda w, h, bd, seed: flat(w, h, bd, "max"),
    "flat_regions": flat_regions,
    "saturated": saturated,
    "hard_edges": hard_edges,
}


def pair(kind, w, h, bd, seed=0):
    """(source, reconstruction) of one content class:
    - 'flat_*', 'flat_regions', 'saturated', 'hard_edges': the picture and that picture degraded (block offsets + noise),
      so the filters have something to do on this content;
    - 'static': a hard-edged picture as its own reconstruction;
    - 'static_blocks': the same with a few blocks changed;
    - 'flat_static': a mid-grey picture as its own reconstruction."""
    if kind == "static":
        s = hard_edges(w, h, bd, seed)
        return s, s.copy()
    if kind == "static_blocks":
        s = hard_edges(w, h, bd, seed)
        return s, changed_blocks(s, seed + 1)
    if kind == "flat_static":
        s = flat(w, h, bd, "mid")
        return s, s.copy()
    s = PICTURES[kind](w, h, bd, seed)
    return s, cm.degrade(s, seed + 3, amp=6)


PAIR_KINDS = ["flat_zero", "flat_mid", "flat_max", "flat_regions", "saturated", "hard_edges", "static", "static_blocks",
              "flat_static"]


# ---- skip maps -------------------------------------------------------------------------------------------------------
def skip_map(mi_rows, mi_cols, kind, seed=0):
    """Per-8x8 skip flags, row stride = the encoder's ((mi_cols + 1) / 2 rounded up to 16):
    'all' (every block skipped: no filter block takes part), 'none', or 'mixed' (whole 64x64 filter blocks skipped in a
    checker pattern, the rest skipped at random)."""
    rows8, cols8 = (mi_rows + 1) // 2, (mi_cols + 1) // 2
    stride = (cols8 + 15) & ~15
    if kind == "all":
        return np.ones((rows8, stride), np.uint8)
    if kind == "none":
        return np.zeros((rows8, stride), np.uint8)
    rng = np.random.default_rng(seed)
    m = (rng.random((rows8, stride)) < 0.35).astype(np.uint8)
    for r in range(0, rows8, 8):
        for c in range(0, cols8, 8):
            if ((r // 8) + (c // 8)) % 2 == 0:
                m[r:r + 8, c:c + 8] = 1
    return m


def fb_all_skipped(skip, mi_rows, mi_cols):
    """Per 64x64 filter block: every 8x8 block inside the picture skipped."""
    rows8, cols8 = (mi_rows + 1) // 2, (mi_cols + 1) // 2
    nvfb, nhfb = (mi_rows + 15) // 16, (mi_cols + 15) // 16
    return np.array([[skip[8 * r:min(8 * r + 8, rows8), 8 * c:min(8 * c + 8, cols8)].all() for c in range(nhfb)]
                     for r in range(nvfb)]).reshape(-1)


def mi_dims(w, h):
    return 2 * ((h + 7) // 8), 2 * ((w + 7) // 8)


# ---- "reaches its branch" checks -------------------------------------------------------------------------------------
def cdef_zero_variance_blocks(f):
    """Number of 8x8 luma blocks for which cdef_find_dir (the oracle's) reports var == 0 (CDEF's adjust_strength then
    returns 0: the block gets no primary filtering)."""
    y = np.ascontiguousarray(f.plane(0).astype(np.uint16))
    n = 0
    var = C.c_int32()
    for by in range(0, f.h - 7, 8):
        for bx in range(0, f.w - 7, 8):
            cm.oracle().orc_cdef_find_dir(C.c_void_p(y.ctypes.data + (by * y.shape[1] + bx) * 2), y.shape[1], C.byref(var), f.bd - 8)
            n += var.value == 0
    return n


def dlf_level_sse(src, rec, flat_mi_fn, mi_rows, mi_cols, part, levels_of):
    """Luma / chroma SSE against `src` of `rec` deblocked (oracle) at each of the 64 levels: array [64, 3]."""
    from test_oracle_dlf import dlf_params
    out = np.zeros((64, 3), np.uint64)
    for lv in range(64):
        levels = levels_of(lv)
        p = dlf_params(mi_rows, mi_cols, levels, 0)
        f = rec.copy()
        fs = f.struct()
        cm.oracle().orc_dlf_frame(C.byref(p), C.byref(fs), flat_mi_fn(mi_rows, mi_cols, part, levels))
        ss, fs = src.struct(), f.struct()
        cm.oracle().orc_frame_sse(C.byref(ss), C.byref(fs), cm.ptr(out[lv]))
    return out


def lpf_decisions(plane, bd, level, x_edges):
    """numpy restatement of the 14-tap luma edge decisions (filter_mask, hev, flat, flat2 of the AV1 loop filter,
    sharpness 0) on the vertical edges at columns `x_edges`: counts of 'none', 'filter4' (mask, not flat), 'hev' (mask and
    high edge variance), 'flat' (8-tap: flat, not flat2) and 'flat2' (14-tap)."""
    sh = bd - 8
    lim = max(level, 1)
    blimit = (2 * (level + 2) + lim) << sh
    limit, thresh, one = lim << sh, (level >> 4) << sh, 1 << sh
    a = plane.astype(np.int64)
    counts = dict(none=0, filter4=0, hev=0, flat=0, flat2=0)
    for x in x_edges:
        if x < 7 or x + 7 > a.shape[1]:
            continue
        p = [a[:, x - 1 - i] for i in range(7)]
        q = [a[:, x + i] for i in range(7)]
        mask = (np.abs(p[3] - p[2]) <= limit) & (np.abs(p[2] - p[1]) <= limit) & (np.abs(p[1] - p[0]) <= limit) & \
               (np.abs(q[1] - q[0]) <= limit) & (np.abs(q[2] - q[1]) <= limit) & (np.abs(q[3] - q[2]) <= limit) & \
               (np.abs(p[0] - q[0]) * 2 + np.abs(p[1] - q[1]) // 2 <= blimit)
        fl = np.ones_like(mask)
        for i in (1, 2, 3):
            fl &= (np.abs(p[i] - p[0]) <= one) & (np.abs(q[i] - q[0]) <= one)
        fl2 = np.ones_like(mask)
        for i in (4, 5, 6):
            fl2 &= (np.abs(p[i] - p[0]) <= one) & (np.abs(q[i] - q[0]) <= one)
        hev = (np.abs(p[1] - p[0]) > thresh) | (np.abs(q[1] - q[0]) > thresh)
        counts["none"] += int((~mask).sum())
        counts["flat2"] += int((mask & fl & fl2).sum())
        counts["flat"] += int((mask & fl & ~fl2).sum())
        counts["hev"] += int((mask & ~fl & hev).sum())
        counts["filter4"] += int((mask & ~fl & ~hev).sum())
    return counts


def rail_fractions(f):
    """Fraction of samples exactly at 0 and exactly at the maximum, over all planes."""
    allv = np.concatenate([f.plane(i).reshape(-1) for i in range(3)]).astype(np.int64)
    return float((allv == 0).mean()), float((allv == maxv(f.bd)).mean())


# ---- ME pictures -----------------------------------------------------------------------------------------------------
def me_flat_case(w, h, kind):
    """Source and eight references of an ME case on constant luma: 'black' (every sample 0) or 'flat' (source at 128,
    references at 128 and at 120): every candidate of a reference has the same SAD."""
    geos = sb.me_geometry(w, h)
    if kind == "black":
        src_v, ref_v = 0, [0] * 8
    else:
        src_v, ref_v = 128, [128, 120, 128, 120, 120, 128, 120, 128]
    src = cm.me_planes(np.full((h, w), src_v, np.uint8), geos)
    refs = [cm.me_planes(np.full((h, w), v, np.uint8), geos) for v in ref_v]
    return geos, src, refs


# ---- an encoder clip -------------------------------------------------------------------------------------------------
def hard_clip_frames(w, h, bd, seed=0):
    """The frames of a clip in this order: a fade from black (into the hard-edged picture), flat mid-grey, saturated
    texture moving 3 samples a frame, hard-edged graphics moving 2 samples a frame, five identical (static) frames, and a
    cut to a picture of flat areas."""
    edges, sat, regions = hard_edges(w, h, bd, seed), saturated(w, h, bd, seed + 1), flat_regions(w, h, bd, seed + 2)
    grey = flat(w, h, bd, "mid")

    def planes(f, scale=1.0, shift=0):
        return [np.roll(np.rint(f.plane(i) * scale), -shift // (2 if i else 1), axis=1).astype(np.int64) for i in range(3)]

    frames = [planes(edges, k / 4) for k in range(4)]
    frames += [planes(grey)] * 2
    frames += [planes(sat, shift=3 * k) for k in range(3)]
    frames += [planes(edges, shift=2 * k) for k in range(3)]
    frames += [planes(edges, shift=6)] * 5
    frames += [planes(regions)] * 2
    return frames


def write_hard_clip(path, w, h, bd, seed=0):
    """hard_clip_frames as planar 4:2:0 (8-bit: uint8, else little-endian uint16); returns the number of frames."""
    frames = hard_clip_frames(w, h, bd, seed)
    with open(path, "wb") as f:
        for fr in frames:
            for p in fr:
                f.write(np.clip(p, 0, maxv(bd)).astype(np.uint8 if bd == 8 else "<u2").tobytes())
    return len(frames)
