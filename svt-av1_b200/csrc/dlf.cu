// dlf.cu — AV1 deblocking loop filter on sm_90a.
//
// Replaces (reference files under Source/Lib):
//   svt_aom_lpf_{horizontal,vertical}_{4,6,8,14}_c + svt_aom_highbd_lpf_*   Common/Codec/EbDeblockingCommon.c:251-924
//   set_lpf_parameters, svt_av1_filter_block_plane_vert/horz, loop_filter_sb,
//   svt_av1_loop_filter_frame                                              Encoder/Codec/EbDeblockingFilter.c:168-753
//   picture_sse_calculations (distortion of svt_av1_pick_filter_level)      Encoder/Codec/EbDeblockingFilter.c:830-964
//
// Design: the reference filters one 64x64 SB at a time on a single thread per picture (vertical edges of SB n,
// then horizontal edges of SB n-1).  AV1 guarantees that edges of one direction never read what another edge of
// the same direction writes and that no horizontal-edge filter touches a sample a later vertical-edge filter reads,
// so the whole picture is two launches: every vertical edge in parallel, then every horizontal edge — one thread
// per sample line of an edge, edge parameters (length, level) derived on the fly from a 16-byte-per-4x4 summary of
// the mode-info grid.  HBM traffic: the picture is read and written once per pass (2 B/sample + 1 B/edge, §8d).
#include <algorithm>

#include "common.cuh"

using namespace svtb200;

namespace {

__device__ __forceinline__ int sclamp(int v, int bd) {
    const int lo = -(128 << (bd - 8)), hi = (128 << (bd - 8)) - 1;
    return v < lo ? lo : (v > hi ? hi : v);
}

// One sample line of an edge. px: p6..p0 at [0..6], q0..q6 at [7..13]. Returns the number of taps per side that may
// have changed (0 = untouched).  Same decisions as filter4/6/8/14 and their masks (EbDeblockingCommon.c:148-924).
__device__ __forceinline__ int lpf_sample(int *px, int len, int blimit, int limit, int thresh, int bd) {
    const int sh = bd - 8;
#define P(i) px[6 - (i)]
#define Q(i) px[7 + (i)]
    const int lim = limit << sh, blim = blimit << sh, thr = thresh << sh, one = 1 << sh;
    bool mask = abs(P(1) - P(0)) <= lim && abs(Q(1) - Q(0)) <= lim && abs(P(0) - Q(0)) * 2 + abs(P(1) - Q(1)) / 2 <= blim;
    if (len >= 6) mask = mask && abs(P(2) - P(1)) <= lim && abs(Q(2) - Q(1)) <= lim;
    if (len >= 8) mask = mask && abs(P(3) - P(2)) <= lim && abs(Q(3) - Q(2)) <= lim;
    bool flat = false, flat2 = false;
    if (len >= 6) {
        flat = abs(P(1) - P(0)) <= one && abs(Q(1) - Q(0)) <= one && abs(P(2) - P(0)) <= one && abs(Q(2) - Q(0)) <= one;
        if (len >= 8) flat = flat && abs(P(3) - P(0)) <= one && abs(Q(3) - Q(0)) <= one;
    }
    if (len == 14)
        flat2 = abs(P(4) - P(0)) <= one && abs(Q(4) - Q(0)) <= one && abs(P(5) - P(0)) <= one && abs(Q(5) - Q(0)) <= one &&
            abs(P(6) - P(0)) <= one && abs(Q(6) - Q(0)) <= one;
    const int p0 = P(0), p1 = P(1), p2 = P(2), p3 = P(3), p4 = P(4), p5 = P(5), p6 = P(6);
    const int q0 = Q(0), q1 = Q(1), q2 = Q(2), q3 = Q(3), q4 = Q(4), q5 = Q(5), q6 = Q(6);
#define R(v, n) (((v) + (1 << ((n)-1))) >> (n))
    if (len == 14 && flat2 && flat && mask) {
        P(5) = R(p6 * 7 + p5 * 2 + p4 * 2 + p3 + p2 + p1 + p0 + q0, 4);
        P(4) = R(p6 * 5 + p5 * 2 + p4 * 2 + p3 * 2 + p2 + p1 + p0 + q0 + q1, 4);
        P(3) = R(p6 * 4 + p5 + p4 * 2 + p3 * 2 + p2 * 2 + p1 + p0 + q0 + q1 + q2, 4);
        P(2) = R(p6 * 3 + p5 + p4 + p3 * 2 + p2 * 2 + p1 * 2 + p0 + q0 + q1 + q2 + q3, 4);
        P(1) = R(p6 * 2 + p5 + p4 + p3 + p2 * 2 + p1 * 2 + p0 * 2 + q0 + q1 + q2 + q3 + q4, 4);
        P(0) = R(p6 + p5 + p4 + p3 + p2 + p1 * 2 + p0 * 2 + q0 * 2 + q1 + q2 + q3 + q4 + q5, 4);
        Q(0) = R(p5 + p4 + p3 + p2 + p1 + p0 * 2 + q0 * 2 + q1 * 2 + q2 + q3 + q4 + q5 + q6, 4);
        Q(1) = R(p4 + p3 + p2 + p1 + p0 + q0 * 2 + q1 * 2 + q2 * 2 + q3 + q4 + q5 + q6 * 2, 4);
        Q(2) = R(p3 + p2 + p1 + p0 + q0 + q1 * 2 + q2 * 2 + q3 * 2 + q4 + q5 + q6 * 3, 4);
        Q(3) = R(p2 + p1 + p0 + q0 + q1 + q2 * 2 + q3 * 2 + q4 * 2 + q5 + q6 * 4, 4);
        Q(4) = R(p1 + p0 + q0 + q1 + q2 + q3 * 2 + q4 * 2 + q5 * 2 + q6 * 5, 4);
        Q(5) = R(p0 + q0 + q1 + q2 + q3 + q4 * 2 + q5 * 2 + q6 * 7, 4);
        return 6;
    }
    if (len >= 8 && flat && mask) {
        P(2) = R(p3 + p3 + p3 + 2 * p2 + p1 + p0 + q0, 3);
        P(1) = R(p3 + p3 + p2 + 2 * p1 + p0 + q0 + q1, 3);
        P(0) = R(p3 + p2 + p1 + 2 * p0 + q0 + q1 + q2, 3);
        Q(0) = R(p2 + p1 + p0 + 2 * q0 + q1 + q2 + q3, 3);
        Q(1) = R(p1 + p0 + q0 + 2 * q1 + q2 + q3 + q3, 3);
        Q(2) = R(p0 + q0 + q1 + 2 * q2 + q3 + q3 + q3, 3);
        return 3;
    }
    if (len == 6 && flat && mask) {
        P(1) = R(p2 * 3 + p1 * 2 + p0 * 2 + q0, 3);
        P(0) = R(p2 + p1 * 2 + p0 * 2 + q0 * 2 + q1, 3);
        Q(0) = R(p1 + p0 * 2 + q0 * 2 + q1 * 2 + q2, 3);
        Q(1) = R(p0 + q0 * 2 + q1 * 2 + q2 * 3, 3);
        return 2;
    }
    if (!mask) return 0; // filter4 with mask = 0 is the identity
    const int off = 0x80 << sh;
    const int ps1 = p1 - off, ps0 = p0 - off, qs0 = q0 - off, qs1 = q1 - off;
    const bool hev = abs(p1 - p0) > thr || abs(q1 - q0) > thr;
    int f = hev ? sclamp(ps1 - qs1, bd) : 0;
    f = sclamp(f + 3 * (qs0 - ps0), bd);
    const int f1 = sclamp(f + 4, bd) >> 3, f2 = sclamp(f + 3, bd) >> 3;
    Q(0) = sclamp(qs0 - f1, bd) + off;
    P(0) = sclamp(ps0 + f2, bd) + off;
    const int f3 = hev ? 0 : ((f1 + 1) >> 1);
    Q(1) = sclamp(qs1 - f3, bd) + off;
    P(1) = sclamp(ps1 + f3, bd) + off;
    return 2;
#undef P
#undef Q
#undef R
}

__device__ __forceinline__ int taps_of(int len) { return len == 4 ? 2 : len == 6 ? 3 : len == 8 ? 4 : 7; }

struct DlfDev {
    SvtB200DlfParams p;
    void *plane[3];
    int stride[3];
    int bd;
    const SvtB200DlfMi *mi;
    const uint8_t *lut; // device [3][2][128] level table indexed by lvl_class, or null: per-mi levels
};

// set_lpf_parameters on the flattened summary
__device__ __forceinline__ int edge_params(const DlfDev &d, int plane, int vert, int x, int y, int &level) {
    const SvtB200DlfParams &p = d.p;
    const int ss = plane ? 1 : 0;
    const int mi_row = ss | ((y << ss) >> 2), mi_col = ss | ((x << ss) >> 2);
    const SvtB200DlfMi *cur = d.mi + (size_t)mi_row * p.mi_stride + mi_col;
    const int ts = vert ? cur->tx_w[ss] : cur->tx_h[ss];
    const int coord = vert ? x : y;
    if ((coord & (ts - 1)) || !coord) return 0;
    const SvtB200DlfMi *prev = vert ? cur - (1 << ss) : cur - (size_t)(1 << ss) * p.mi_stride;
    const int pv_ts = vert ? prev->tx_w[ss] : prev->tx_h[ss];
    int cl, pl;
    if (d.lut) { // get_filter_level: lfi_n->lvl[plane][segment][dir][ref][mode], dir 0 = vertical edges
        const uint8_t *t = d.lut + (plane * 2 + (vert ? 0 : 1)) * 128;
        cl = t[cur->lvl_class & 127];
        pl = t[prev->lvl_class & 127];
    } else {
        cl = plane == 0 ? cur->lvl_y[vert ? 0 : 1] : plane == 1 ? cur->lvl_u : cur->lvl_v;
        pl = plane == 0 ? prev->lvl_y[vert ? 0 : 1] : plane == 1 ? prev->lvl_u : prev->lvl_v;
    }
    const bool pu_edge = !(coord & ((vert ? cur->blk_w[ss] : cur->blk_h[ss]) - 1));
    if (!((cl || pl) && (!prev->skip_inter || !cur->skip_inter || pu_edge))) return 0;
    const int mn = min(ts, pv_ts);
    level = cl ? cl : pl;
    if (mn <= 4) return 4;
    if (mn == 8) return plane ? 6 : 8;
    return plane ? 6 : 14;
}
__device__ __forceinline__ void thresholds(int level, int sharpness, int &blimit, int &limit, int &thresh) {
    int lim = level >> ((sharpness > 0) + (sharpness > 4));
    if (sharpness > 0 && lim > 9 - sharpness) lim = 9 - sharpness;
    if (lim < 1) lim = 1;
    limit = lim;
    blimit = 2 * (level + 2) + lim;
    thresh = level >> 4;
}

// One thread per sample line of a 4x4 unit's leading edge.  vert = 1: thread = (row y, unit column ux);
// vert = 0: thread = (unit row uy, column x) so that a warp walks along a row of the picture (coalesced).
template <typename T>
__global__ void __launch_bounds__(256) dlf_pass_kernel(const __grid_constant__ DlfDev d, int planes, int vert) {
    const int plane = (planes >> (2 * blockIdx.z)) & 3; // the planes of one direction share a launch (grid.z)
    const int ss = plane ? 1 : 0;
    const int pw = (d.p.mi_cols * 4) >> ss, ph = (d.p.mi_rows * 4) >> ss;
    const int nx = vert ? pw / 4 : pw, ny = vert ? ph : ph / 4;
    const int gx = blockIdx.x * blockDim.x + threadIdx.x, gy = blockIdx.y;
    if (gx >= nx || gy >= ny) return;
    const int x = vert ? gx * 4 : gx, y = vert ? gy : gy * 4;
    int level = 0;
    const int len = edge_params(d, plane, vert, vert ? x : (x & ~3), vert ? (y & ~3) : y, level);
    if (!len) return;
    int bl, li, th;
    thresholds(level, d.p.sharpness, bl, li, th);
    T *s = reinterpret_cast<T *>(d.plane[plane]) + (size_t)y * d.stride[plane] + x;
    const ptrdiff_t across = vert ? 1 : d.stride[plane];
    const int n = taps_of(len);
    int px[14];
#pragma unroll
    for (int t = 0; t < 7; t++) {
        px[6 - t] = t < n ? (int)s[-(ptrdiff_t)(t + 1) * across] : 0;
        px[7 + t] = t < n ? (int)s[(ptrdiff_t)t * across] : 0;
    }
    const int changed = lpf_sample(px, len, bl, li, th, d.bd);
#pragma unroll
    for (int t = 0; t < 6; t++)
        if (t < changed) {
            s[-(ptrdiff_t)(t + 1) * across] = (T)px[6 - t];
            s[(ptrdiff_t)t * across] = (T)px[7 + t];
        }
}

// ---- block-edge kernels (the fast path) ----------------------------------------------------------------------------
// One thread per 4x4 unit's leading edge = its FOUR sample lines: the edge parameters are derived once per edge instead of
// once per line, and the samples move as 32/64-bit words.
//  * vertical edges : thread (unit column, unit row); per line one aligned 4-sample word either side of the edge (two
//    for the 14-tap filter).  Only the samples a filter may change are stored, in the widest aligned pieces that do not
//    touch a neighbouring edge's samples (a 4-tap edge 4 samples away owns x-4, x-3).
//  * horizontal edges: thread = the unit's 4 columns, one 4-sample word per row, 128 B per warp and row; the rows a
//    filter of this length may change are stored as whole words (no other edge of the pass writes them).
// Needs 4-sample-aligned planes (base and stride multiples of 4 samples): every picture the engine allocates, and the
// reference's EbPictureBufferDesc planes.  Anything else takes dlf_pass_kernel.
template <typename T> struct Word4; // four samples
template <> struct Word4<uint8_t> {
    using W = uint32_t;
    static __device__ __forceinline__ void unpack(W w, int *v) {
        v[0] = w & 0xff, v[1] = (w >> 8) & 0xff, v[2] = (w >> 16) & 0xff, v[3] = w >> 24;
    }
    static __device__ __forceinline__ W pack(const int *v) { return (W)v[0] | ((W)v[1] << 8) | ((W)v[2] << 16) | ((W)v[3] << 24); }
};
template <> struct Word4<uint16_t> {
    using W = uint2;
    static __device__ __forceinline__ void unpack(W w, int *v) {
        v[0] = w.x & 0xffff, v[1] = w.x >> 16, v[2] = w.y & 0xffff, v[3] = w.y >> 16;
    }
    static __device__ __forceinline__ W pack(const int *v) {
        return make_uint2((uint32_t)v[0] | ((uint32_t)v[1] << 16), (uint32_t)v[2] | ((uint32_t)v[3] << 16));
    }
};
template <typename T> __device__ __forceinline__ int lane_get(uint32_t w, int c) { return (w >> (8 * c)) & 0xff; }
template <typename T> __device__ __forceinline__ int lane_get(uint2 w, int c) { return ((c < 2 ? w.x : w.y) >> (16 * (c & 1))) & 0xffff; }
template <typename T> __device__ __forceinline__ void lane_set(uint32_t &w, int c, int v) {
    w = (w & ~(0xffu << (8 * c))) | ((uint32_t)v << (8 * c));
}
template <typename T> __device__ __forceinline__ void lane_set(uint2 &w, int c, int v) {
    uint32_t &h = c < 2 ? w.x : w.y;
    h = (h & ~(0xffffu << (16 * (c & 1)))) | ((uint32_t)v << (16 * (c & 1)));
}
// samples a filter of this length may change on each side (filter4 / filter6: 2, filter8: 3, filter14: 6)
__device__ __forceinline__ int mod_of(int len) { return len == 14 ? 6 : len == 8 ? 3 : 2; }

template <typename T>
__global__ void __launch_bounds__(256) dlf_vert_kernel(const __grid_constant__ DlfDev d, int planes) {
    using WT = typename Word4<T>::W;
    const int plane = (planes >> (2 * blockIdx.z)) & 3;
    const int ss = plane ? 1 : 0;
    const int pw = (d.p.mi_cols * 4) >> ss, ph = (d.p.mi_rows * 4) >> ss;
    const int ux = blockIdx.x * 32 + (threadIdx.x & 31), uy = blockIdx.y * 8 + (threadIdx.x >> 5);
    const int x = ux * 4, y = uy * 4;
    if (x >= pw || y >= ph || ux == 0) return;
    int level = 0;
    const int len = edge_params(d, plane, 1, x, y, level);
    if (!len) return;
    int bl, li, th;
    thresholds(level, d.p.sharpness, bl, li, th);
    T *row0 = reinterpret_cast<T *>(d.plane[plane]) + (size_t)y * d.stride[plane] + x;
    const int rows = min(4, ph - y);
    const bool wide = len == 14;
    // all loads of the edge's four lines are issued before the first line is filtered (one memory round trip, not four)
    WT w[4][4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const T *row = row0 + (size_t)min(r, rows - 1) * d.stride[plane];
        w[r][1] = *reinterpret_cast<const WT *>(row - 4);
        w[r][2] = *reinterpret_cast<const WT *>(row);
        if (wide) {
            w[r][0] = *reinterpret_cast<const WT *>(row - 8);
            w[r][3] = *reinterpret_cast<const WT *>(row + 4);
        } else {
            w[r][0] = w[r][3] = WT{};
        }
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
        if (r >= rows) break;
        T *row = row0 + (size_t)r * d.stride[plane];
        int px[16]; // samples x-8 .. x+7; lpf_sample works on px+1 (p6 = x-7 .. q6 = x+6)
        Word4<T>::unpack(w[r][0], px);
        Word4<T>::unpack(w[r][1], px + 4);
        Word4<T>::unpack(w[r][2], px + 8);
        Word4<T>::unpack(w[r][3], px + 12);
        const int changed = lpf_sample(px + 1, len, bl, li, th, d.bd);
        if (!changed) continue;
        if (changed == 6) { // x-6 .. x+5: two samples, two words, two samples
            row[-6] = (T)px[2], row[-5] = (T)px[3];
            *reinterpret_cast<WT *>(row - 4) = Word4<T>::pack(px + 4);
            *reinterpret_cast<WT *>(row) = Word4<T>::pack(px + 8);
            row[4] = (T)px[12], row[5] = (T)px[13];
        } else { // 2 or 3 samples each side: never the word's far samples (they may belong to the next edge)
            if (changed == 3) row[-3] = (T)px[5], row[2] = (T)px[10];
            row[-2] = (T)px[6], row[-1] = (T)px[7], row[0] = (T)px[8], row[1] = (T)px[9];
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256) dlf_horz_kernel(const __grid_constant__ DlfDev d, int planes) {
    using WT = typename Word4<T>::W;
    const int plane = (planes >> (2 * blockIdx.z)) & 3;
    const int ss = plane ? 1 : 0;
    const int pw = (d.p.mi_cols * 4) >> ss, ph = (d.p.mi_rows * 4) >> ss;
    const int ux = blockIdx.x * 32 + (threadIdx.x & 31), uy = blockIdx.y * 8 + (threadIdx.x >> 5);
    const int x = ux * 4, y = uy * 4;
    if (x >= pw || y >= ph || uy == 0) return;
    int level = 0;
    const int len = edge_params(d, plane, 0, x, y, level);
    if (!len) return;
    int bl, li, th;
    thresholds(level, d.p.sharpness, bl, li, th);
    const ptrdiff_t st = d.stride[plane];
    T *s = reinterpret_cast<T *>(d.plane[plane]) + (size_t)y * st + x;
    const int n = taps_of(len), m = mod_of(len);
    // the 14 rows stay packed (one word of 4 columns per row); a column is unpacked, filtered and its changed samples
    // merged back into the words - 28 live registers instead of a 4 x 14 sample array (occupancy)
    WT up[7], dn[7]; // up[t] = row y-1-t, dn[t] = row y+t
#pragma unroll
    for (int t = 0; t < 7; t++) {
        up[t] = t < n ? *reinterpret_cast<const WT *>(s - (ptrdiff_t)(t + 1) * st) : WT{};
        dn[t] = t < n ? *reinterpret_cast<const WT *>(s + (ptrdiff_t)t * st) : WT{};
    }
    int any = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
        int px[14];
#pragma unroll
        for (int t = 0; t < 7; t++) px[6 - t] = lane_get<T>(up[t], c), px[7 + t] = lane_get<T>(dn[t], c);
        const int changed = lpf_sample(px, len, bl, li, th, d.bd);
        any |= changed;
#pragma unroll
        for (int t = 0; t < 6; t++)
            if (t < changed) lane_set<T>(up[t], c, px[6 - t]), lane_set<T>(dn[t], c, px[7 + t]);
    }
    if (!any) return;
#pragma unroll
    for (int t = 0; t < 6; t++)
        if (t < m) {
            *reinterpret_cast<WT *>(s - (ptrdiff_t)(t + 1) * st) = up[t];
            *reinterpret_cast<WT *>(s + (ptrdiff_t)t * st) = dn[t];
        }
}

// drop-in: one 4-line edge segment staged as a 16 x 4 window (p7..q7 across, 4 lines)
__global__ void lpf_edge_kernel(uint16_t *win, int len, int blimit, int limit, int thresh, int bd) {
    const int i = threadIdx.x;
    if (i >= 4) return;
    int px[14];
    for (int t = 0; t < 7; t++) {
        px[6 - t] = win[i * 16 + 7 - t];
        px[7 + t] = win[i * 16 + 8 + t];
    }
    lpf_sample(px, len, blimit, limit, thresh, bd);
    for (int t = 0; t < 7; t++) {
        win[i * 16 + 7 - t] = (uint16_t)px[6 - t];
        win[i * 16 + 8 + t] = (uint16_t)px[7 + t];
    }
}

template <typename T>
__global__ void __launch_bounds__(256) sse_kernel(const T *a, int sa, const T *b, int sb, int w, int h, unsigned long long *out) {
    unsigned long long acc = 0;
    for (int y = blockIdx.x; y < h; y += gridDim.x)
        for (int x = threadIdx.x; x < w; x += blockDim.x) {
            const int dlt = (int)a[(size_t)y * sa + x] - (int)b[(size_t)y * sb + x];
            acc += (unsigned long long)(dlt * dlt);
        }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}

void lpf_dropin(void *s, int hbd, int pitch, int vert, int len, const uint8_t *blimit, const uint8_t *limit,
                const uint8_t *thresh, int bd) {
    Staging st({128}); // 4 lines of 16 samples across the edge
    SVTB_CUDA_FATAL(st.status());
    uint16_t *w = st.h<uint16_t>(0);
    const int n = len == 4 ? 2 : len == 6 ? 3 : len == 8 ? 4 : 7;
    const ptrdiff_t across = vert ? 1 : pitch, along = vert ? pitch : 1;
    memset(w, 0, 128);
    for (int i = 0; i < 4; i++)
        for (int t = 0; t < n; t++) {
            const ptrdiff_t op = i * along - (t + 1) * across, oq = i * along + t * across;
            w[i * 16 + 7 - t] = hbd ? ((uint16_t *)s)[op] : ((uint8_t *)s)[op];
            w[i * 16 + 8 + t] = hbd ? ((uint16_t *)s)[oq] : ((uint8_t *)s)[oq];
        }
    SVTB_CUDA_FATAL(st.upload(0, 0));
    SVTB_LAUNCH(lpf_edge_kernel, 1, 32, 0, st.stream(), st.d<uint16_t>(0), len, (int)*blimit, (int)*limit, (int)*thresh, bd);
    SVTB_CUDA_FATAL(st.download(0, 0));
    for (int i = 0; i < 4; i++)
        for (int t = 0; t < n; t++) {
            const ptrdiff_t op = i * along - (t + 1) * across, oq = i * along + t * across;
            if (hbd) {
                ((uint16_t *)s)[op] = w[i * 16 + 7 - t];
                ((uint16_t *)s)[oq] = w[i * 16 + 8 + t];
            } else {
                ((uint8_t *)s)[op] = (uint8_t)w[i * 16 + 7 - t];
                ((uint8_t *)s)[oq] = (uint8_t)w[i * 16 + 8 + t];
            }
        }
}

} // namespace

extern "C" {

#define LPF_DROPIN(DIR, VERT, N)                                                                                            \
    void svt_aom_lpf_##DIR##_##N##_cuda(uint8_t *s, int32_t pitch, const uint8_t *blimit, const uint8_t *limit,             \
                                        const uint8_t *thresh) {                                                            \
        lpf_dropin(s, 0, pitch, VERT, N, blimit, limit, thresh, 8);                                                         \
    }                                                                                                                       \
    void svt_aom_highbd_lpf_##DIR##_##N##_cuda(uint16_t *s, int32_t pitch, const uint8_t *blimit, const uint8_t *limit,     \
                                               const uint8_t *thresh, int32_t bd) {                                         \
        lpf_dropin(s, 1, pitch, VERT, N, blimit, limit, thresh, bd);                                                        \
    }
LPF_DROPIN(horizontal, 0, 4)
LPF_DROPIN(horizontal, 0, 6)
LPF_DROPIN(horizontal, 0, 8)
LPF_DROPIN(horizontal, 0, 14)
LPF_DROPIN(vertical, 1, 4)
LPF_DROPIN(vertical, 1, 6)
LPF_DROPIN(vertical, 1, 8)
LPF_DROPIN(vertical, 1, 14)

static int dlf_frame_impl(const SvtB200DlfParams *p, const SvtB200Frame *frame, const SvtB200DlfMi *mi, const uint8_t *lut,
                          void *stream) {
    if (!p || !frame || !mi || !frame->y || !frame->cb || !frame->cr || p->mi_rows <= 0 || p->mi_cols <= 0 ||
        p->mi_stride < p->mi_cols) {
        set_error("svt_b200_dlf_frame: bad argument");
        return SVT_B200_ERR_ARG;
    }
    DlfDev d;
    d.p = *p;
    d.plane[0] = frame->y;
    d.plane[1] = frame->cb;
    d.plane[2] = frame->cr;
    d.stride[0] = frame->stride_y;
    d.stride[1] = d.stride[2] = frame->stride_c;
    d.bd = frame->bit_depth;
    d.mi = mi;
    d.lut = lut;
    cudaStream_t st = (cudaStream_t)stream;
    const bool hbd = frame->bit_depth > 8;
    // all vertical edges of every plane first, then all horizontal edges (see the header comment)
    int planes = 0, n_planes = 0, max_w = 0, max_h = 0;
    for (int plane = p->plane_start; plane < p->plane_end; plane++) {
        if (plane == 0 && !p->filter_level[0] && !p->filter_level[1]) break; // loop_filter_sb :629-636
        if (plane == 1 && !p->filter_level_u) continue;
        if (plane == 2 && !p->filter_level_v) continue;
        const int ss = plane ? 1 : 0;
        planes |= plane << (2 * n_planes++);
        max_w = std::max(max_w, (p->mi_cols * 4) >> ss);
        max_h = std::max(max_h, (p->mi_rows * 4) >> ss);
    }
    // the block-edge kernels move 4-sample words: planes whose base / stride are 4-sample aligned (every EbPictureBufferDesc
    // and every engine picture); other layouts take the line-per-thread kernel
    const size_t wbytes = hbd ? 8 : 4;
    const bool aligned = ((uintptr_t)frame->y % wbytes) == 0 && ((uintptr_t)frame->cb % wbytes) == 0 &&
        ((uintptr_t)frame->cr % wbytes) == 0 && frame->stride_y % 4 == 0 && frame->stride_c % 4 == 0;
    for (int vert = 1; vert >= 0 && n_planes; vert--) {
        if (aligned) {
            dim3 grid((max_w / 4 + 31) / 32, (max_h / 4 + 7) / 8, n_planes); // CTA = 32 x 8 units = 128 x 32 samples
            if (vert) {
                if (hbd)
                    SVTB_LAUNCH(dlf_vert_kernel<uint16_t>, grid, 256, 0, st, d, planes);
                else
                    SVTB_LAUNCH(dlf_vert_kernel<uint8_t>, grid, 256, 0, st, d, planes);
            } else {
                if (hbd)
                    SVTB_LAUNCH(dlf_horz_kernel<uint16_t>, grid, 256, 0, st, d, planes);
                else
                    SVTB_LAUNCH(dlf_horz_kernel<uint8_t>, grid, 256, 0, st, d, planes);
            }
            continue;
        }
        const int nx = vert ? max_w / 4 : max_w, ny = vert ? max_h : max_h / 4;
        dim3 grid((nx + 255) / 256, ny, n_planes);
        if (hbd)
            SVTB_LAUNCH(dlf_pass_kernel<uint16_t>, grid, 256, 0, st, d, planes, vert);
        else
            SVTB_LAUNCH(dlf_pass_kernel<uint8_t>, grid, 256, 0, st, d, planes, vert);
    }
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

int svt_b200_dlf_frame(const SvtB200DlfParams *p, const SvtB200Frame *frame, const SvtB200DlfMi *mi, void *stream) {
    return dlf_frame_impl(p, frame, mi, nullptr, stream);
}
int svt_b200_dlf_frame_lut(const SvtB200DlfParams *p, const SvtB200Frame *frame, const SvtB200DlfMi *mi, const uint8_t *lut,
                           void *stream) {
    if (!lut) {
        set_error("svt_b200_dlf_frame_lut: null level table");
        return SVT_B200_ERR_ARG;
    }
    return dlf_frame_impl(p, frame, mi, lut, stream);
}

// svt_av1_loop_filter_frame_init (EbDeblockingCommon.c:78-145): lvl[plane][seg][dir][ref][mode] as lut[plane][dir][class].
// The planes from plane_start on, as frame_init's loop: a table started at a chroma plane is filled even when both luma
// levels are 0 (the chroma trials of the level search filter plane..plane+1 only).
static void lf_level_lut(const SvtB200LfFrameInit *init, const int32_t levels[4], int plane_start, uint8_t lut[3][2][128]) {
    static const int seg_lvl_lf_lut[3][2] = {{1, 2}, {3, 3}, {4, 4}}; // SEG_LVL_ALT_LF_Y_V, _Y_H, _U, _V
    const int filt[3] = {levels[0], levels[2], levels[3]}, filt_r[3] = {levels[1], levels[2], levels[3]};
    memset(lut, 0, 3 * 2 * 128);
    for (int plane = plane_start; plane < 3; plane++) {
        if (plane == 0 && !filt[0] && !filt_r[0]) break;
        if (plane && !filt[plane]) continue;
        for (int seg = 0; seg < 8; seg++)
            for (int dir = 0; dir < 2; dir++) {
                int lvl_seg = dir == 0 ? filt[plane] : filt_r[plane];
                const int f = seg_lvl_lf_lut[plane][dir];
                if (init->segmentation_enabled && ((init->seg_feature_mask[seg] >> f) & 1)) {
                    lvl_seg += init->seg_feature_data[seg][f];
                    lvl_seg = lvl_seg < 0 ? 0 : (lvl_seg > 63 ? 63 : lvl_seg);
                }
                for (int ref = 0; ref < 8; ref++)
                    for (int mode = 0; mode < 2; mode++) {
                        int v = lvl_seg;
                        if (init->mode_ref_delta_enabled) {
                            const int scale = 1 << (lvl_seg >> 5);
                            // INTRA_FRAME has a single entry ([0]); entry [1] is never read (mode_lf_lut of intra modes is 0)
                            v = ref == 0 ? lvl_seg + init->ref_deltas[0] * scale
                                         : lvl_seg + init->ref_deltas[ref] * scale + init->mode_deltas[mode] * scale;
                            v = v < 0 ? 0 : (v > 63 ? 63 : v);
                        }
                        lut[plane][dir][seg * 16 + ref * 2 + mode] = (uint8_t)v;
                    }
            }
    }
}
int svt_b200_lf_level_lut(const SvtB200LfFrameInit *init, const int32_t levels[4], uint8_t lut[3][2][128]) {
    if (!init || !levels || !lut) return SVT_B200_ERR_ARG;
    lf_level_lut(init, levels, 0, lut);
    return SVT_B200_OK;
}

namespace {
struct PickCtx {
    const SvtB200LpfPickParams *p;
    const SvtB200Frame *recon, *source, *temp;
    const SvtB200DlfMi *mi;
    uint8_t *d_lut; // device 768 B
    unsigned long long *d_sse; // device
    uint8_t *h_lut; // pinned staging of the calling thread: the level table, then the SSE read back
    unsigned long long *h_sse;
    cudaStream_t st;
    int32_t cur[4]; // frame levels as the search progresses (frm_hdr->loop_filter_params)
};
int plane_copy(const SvtB200Frame *src, const SvtB200Frame *dst, int plane, cudaStream_t st) {
    const int es = src->bit_depth > 8 ? 2 : 1;
    const int w = plane ? src->width >> 1 : src->width, h = plane ? src->height >> 1 : src->height;
    const void *s = plane == 0 ? src->y : plane == 1 ? src->cb : src->cr;
    void *d = plane == 0 ? dst->y : plane == 1 ? dst->cb : dst->cr;
    const size_t ss = (size_t)(plane ? src->stride_c : src->stride_y) * es, ds = (size_t)(plane ? dst->stride_c : dst->stride_y) * es;
    return cudaMemcpy2DAsync(d, ds, s, ss, (size_t)w * es, h, cudaMemcpyDeviceToDevice, st) == cudaSuccess ? 0 : -1;
}
// try_filter_frame (:966-1026): filter one plane of recon at the trial level, SSE against the source, restore the plane
int64_t try_filter(PickCtx &c, int level, int plane, int dir) {
    int32_t lv[4] = {c.cur[0], c.cur[1], c.cur[2], c.cur[3]};
    if (plane == 0) {
        if (dir != 1) lv[0] = level; // dir 0: only [0]; dir 2: both
        if (dir != 0) lv[1] = level;
    } else {
        lv[1 + plane] = level;
    }
    // the trial levels stay in the frame header (set base filters ... :1007-1014)
    for (int i = 0; i < 4; i++) c.cur[i] = lv[i];
    uint8_t(*lut)[2][128] = reinterpret_cast<uint8_t(*)[2][128]>(c.h_lut);
    lf_level_lut(&c.p->init, lv, plane, lut);
    SvtB200DlfParams dp = c.p->dlf;
    dp.sharpness = 0;
    dp.filter_level[0] = lv[0], dp.filter_level[1] = lv[1], dp.filter_level_u = lv[2], dp.filter_level_v = lv[3];
    dp.plane_start = plane, dp.plane_end = plane + 1;
    // the pinned staging buffer is reused by the next trial: the previous trial ended with a stream synchronise
    if (cudaMemcpyAsync(c.d_lut, c.h_lut, 768, cudaMemcpyHostToDevice, c.st) != cudaSuccess) return -1;
    if (dlf_frame_impl(&dp, c.recon, c.mi, c.d_lut, c.st) != SVT_B200_OK) return -1;
    if (cudaMemsetAsync(c.d_sse, 0, 8, c.st) != cudaSuccess) return -1;
    const int w = plane ? c.recon->width >> 1 : c.recon->width, h = plane ? c.recon->height >> 1 : c.recon->height;
    const void *a = plane == 0 ? c.source->y : plane == 1 ? c.source->cb : c.source->cr;
    const void *b = plane == 0 ? c.recon->y : plane == 1 ? c.recon->cb : c.recon->cr;
    const int sa = plane ? c.source->stride_c : c.source->stride_y, sb = plane ? c.recon->stride_c : c.recon->stride_y;
    const int grid = h < 592 ? h : 592;
    if (c.recon->bit_depth > 8)
        SVTB_LAUNCH(sse_kernel<uint16_t>, grid, 256, 0, c.st, (const uint16_t *)a, sa, (const uint16_t *)b, sb, w, h, c.d_sse);
    else
        SVTB_LAUNCH(sse_kernel<uint8_t>, grid, 256, 0, c.st, (const uint8_t *)a, sa, (const uint8_t *)b, sb, w, h, c.d_sse);
    if (plane_copy(c.temp, c.recon, plane, c.st)) return -1; // re-instate the unfiltered plane
    if (cudaMemcpyAsync(c.h_sse, c.d_sse, 8, cudaMemcpyDeviceToHost, c.st) != cudaSuccess) return -1;
    if (cudaStreamSynchronize(c.st) != cudaSuccess) return -1;
    return (int64_t)*c.h_sse;
}
// search_filter_level (:1027-1191)
int search_level(PickCtx &c, int plane, int dir, int *err) {
    const int lvl = plane == 0 ? c.p->last_level[dir == 2 ? 2 : dir] : plane == 1 ? c.p->last_level[2] : c.p->last_level[3];
    int filt_mid = lvl < 0 ? 0 : (lvl > 63 ? 63 : lvl);
    int filter_step = filt_mid < 16 ? 4 : filt_mid / 4;
    int filt_direction = 0;
    int64_t ss_err[64];
    for (int i = 0; i < 64; i++) ss_err[i] = -1;
    if (plane_copy(c.recon, c.temp, plane, c.st)) { *err = 1; return 0; }
    int64_t best_err = try_filter(c, filt_mid, plane, dir);
    if (best_err < 0) { *err = 1; return 0; }
    int filt_best = filt_mid;
    ss_err[filt_mid] = best_err;
    const bool one_step = c.p->loop_filter_mode <= 2;
    if (one_step) filter_step = 2;
    while (filter_step > 0) {
        const int filt_high = filt_mid + filter_step > 63 ? 63 : filt_mid + filter_step;
        const int filt_low = filt_mid - filter_step < 0 ? 0 : filt_mid - filter_step;
        int64_t bias = (best_err >> (15 - (filt_mid / 8))) * filter_step; // bias against raising the level
        if (!c.p->tx_mode_only_4x4) bias >>= 1;
        if (filt_direction <= 0 && filt_low != filt_mid) {
            if (ss_err[filt_low] < 0) {
                ss_err[filt_low] = try_filter(c, filt_low, plane, dir);
                if (ss_err[filt_low] < 0) { *err = 1; return 0; }
            }
            if (ss_err[filt_low] < best_err + bias) {
                if (ss_err[filt_low] < best_err) best_err = ss_err[filt_low];
                filt_best = filt_low;
            }
        }
        if (filt_direction >= 0 && filt_high != filt_mid) {
            if (ss_err[filt_high] < 0) {
                ss_err[filt_high] = try_filter(c, filt_high, plane, dir);
                if (ss_err[filt_high] < 0) { *err = 1; return 0; }
            }
            if (ss_err[filt_high] < best_err - bias) {
                if (!one_step) best_err = ss_err[filt_high]; // the <= 2 branch (:1117-1118) does not update best_err
                filt_best = filt_high;
            }
        }
        if (one_step) break;
        if (filt_best == filt_mid) {
            filter_step /= 2;
            filt_direction = 0;
        } else {
            filt_direction = filt_best < filt_mid ? -1 : 1;
            filt_mid = filt_best;
        }
    }
    return filt_best;
}
} // namespace

int svt_b200_pick_filter_level(const SvtB200LpfPickParams *p, const SvtB200Frame *recon, const SvtB200Frame *source,
                               const SvtB200Frame *temp, const SvtB200DlfMi *mi, void *scratch, int32_t *levels_out, void *stream) {
    if (!p || !levels_out || p->method < 0 || p->method > 3) {
        set_error("svt_b200_pick_filter_level: bad argument");
        return SVT_B200_ERR_ARG;
    }
    if (p->method == 3) { // LPF_PICK_MINIMAL_LPF: only the luma levels are touched
        levels_out[0] = levels_out[1] = 0;
        levels_out[2] = p->last_level[2];
        levels_out[3] = p->last_level[3];
        return SVT_B200_OK;
    }
    if (p->method == 2) { // LPF_PICK_FROM_Q (:1209-1249)
        const int bd = recon ? recon->bit_depth : 8, q = p->q_ac;
        auto rpo2 = [](long long v, int n) { return (int)((v + (1ll << (n - 1))) >> n); };
        int g = bd == 8 ? (p->key_frame ? rpo2((long long)q * 17563 - 421574, 18) : rpo2((long long)q * 6017 + 650707, 18))
                        : bd == 10 ? rpo2((long long)q * 20723 + 4060632, 20) : rpo2((long long)q * 20723 + 16242526, 22);
        if (bd != 8 && p->key_frame) g -= 4;
        g = g > 2 ? g - 2 : g > 1 ? g - 1 : g;
        const int gc = g > 1 ? g / 2 : g;
        auto cl = [](int v) { return v < 0 ? 0 : (v > 63 ? 63 : v); };
        levels_out[0] = levels_out[1] = cl(g);
        levels_out[2] = levels_out[3] = cl(gc);
        return SVT_B200_OK;
    }
    if (!recon || !source || !temp || !mi || !scratch || recon->bit_depth != source->bit_depth || recon->bit_depth != temp->bit_depth ||
        recon->width != source->width || recon->height != source->height) {
        set_error("svt_b200_pick_filter_level: bad argument");
        return SVT_B200_ERR_ARG;
    }
    PickCtx c;
    c.p = p, c.recon = recon, c.source = source, c.temp = temp, c.mi = mi;
    c.d_lut = (uint8_t *)scratch;
    c.d_sse = (unsigned long long *)((uint8_t *)scratch + 768);
    c.st = (cudaStream_t)stream;
    // pinned side only, on the caller's stream: reserved once for the whole search (nothing the search runs stages)
    Staging s({768, 8});
    SVTB_CUDA_TRY(s.status());
    c.h_lut = s.h(0);
    c.h_sse = s.h<unsigned long long>(1);
    for (int i = 0; i < 4; i++) c.cur[i] = p->last_level[i];
    int err = 0;
    const int y = search_level(c, 0, 2, &err);
    if (!err) {
        c.cur[0] = c.cur[1] = y;
        const int u = search_level(c, 1, 0, &err);
        if (!err) {
            c.cur[2] = u;
            const int v = search_level(c, 2, 0, &err);
            if (!err) c.cur[3] = v;
        }
    }
    if (err) {
        set_error("svt_b200_pick_filter_level: CUDA failure");
        return SVT_B200_ERR_CUDA;
    }
    for (int i = 0; i < 4; i++) levels_out[i] = c.cur[i];
    return SVT_B200_OK;
}

int svt_b200_frame_sse(const SvtB200Frame *a, const SvtB200Frame *b, uint64_t *sse, void *stream) {
    if (!a || !b || !sse || a->bit_depth != b->bit_depth || a->width != b->width || a->height != b->height) {
        set_error("svt_b200_frame_sse: bad argument");
        return SVT_B200_ERR_ARG;
    }
    cudaStream_t st = (cudaStream_t)stream;
    SVTB_CUDA_TRY(cudaMemsetAsync(sse, 0, 3 * sizeof(uint64_t), st));
    for (int pl = 0; pl < 3; pl++) {
        const int w = pl ? (a->width + 1) >> 1 : a->width, h = pl ? (a->height + 1) >> 1 : a->height;
        const void *pa = pl == 0 ? a->y : pl == 1 ? a->cb : a->cr, *pb = pl == 0 ? b->y : pl == 1 ? b->cb : b->cr;
        const int sa = pl ? a->stride_c : a->stride_y, sb = pl ? b->stride_c : b->stride_y;
        const int grid = h < 592 ? h : 592;
        if (a->bit_depth > 8)
            SVTB_LAUNCH(sse_kernel<uint16_t>, grid, 256, 0, st, (const uint16_t *)pa, sa, (const uint16_t *)pb, sb, w, h,
                        (unsigned long long *)(sse + pl));
        else
            SVTB_LAUNCH(sse_kernel<uint8_t>, grid, 256, 0, st, (const uint8_t *)pa, sa, (const uint8_t *)pb, sb, w, h,
                        (unsigned long long *)(sse + pl));
    }
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}
}
