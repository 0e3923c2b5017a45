// lr.cu — loop-restoration kernels on sm_90a: self-guided filter, its projection apply, separable Wiener.
//
// Replaces (reference files under Source/Lib/Common/Codec):
//   svt_av1_selfguided_restoration_c        EbRestoration.c:1012-1045 (internals :744-1010, boxsum :541-705)
//   svt_apply_selfguided_restoration_c      EbRestoration.c:1047-1084 (svt_decode_xq :707)
//   svt_av1_wiener_convolve_add_src_c / svt_av1_highbd_wiener_convolve_add_src_c   convolve.c:53-260
//
// Design: one CTA per processing unit (<= 64x64 + 3-sample rim).  The unit is staged once in shared memory;
// the box sums of the self-guided filter are evaluated directly from it ((2r+1)^2 taps per a/b sample — the rim
// makes every window complete, so no integral image and no edge cases), a/b for the (w+2)x(h+2) neighbourhood
// are kept in shared memory and both radii are produced from the same tile.  The Wiener filter keeps the
// horizontally filtered (h+7) x w intermediate in shared memory, so HBM traffic is 2 B/sample (8-bit) in both
// cases.  This round provides the RTCD drop-ins; the frame-level stripe loop is the next §8 row.
#include <algorithm>

#include "common.cuh"

using namespace svtb200;

namespace {

__constant__ int8_t c_sgr_r[16][2] = {{2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1},
                                      {2, 1}, {2, 1}, {0, 1}, {0, 1}, {0, 1}, {0, 1}, {2, 0}, {2, 0}};
__constant__ int16_t c_sgr_s[16][2] = {{140, 3236}, {112, 2158}, {93, 1618}, {80, 1438}, {70, 1295}, {58, 1177}, {47, 1079}, {37, 996},
                                       {30, 925},   {25, 863},   {-1, 2589}, {-1, 1618}, {-1, 1177}, {-1, 925},  {56, -1},   {22, -1}};
static const int8_t h_sgr_r[16][2] = {{2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1},
                                      {2, 1}, {2, 1}, {0, 1}, {0, 1}, {0, 1}, {0, 1}, {2, 0}, {2, 0}};

__device__ __forceinline__ int x_by_xplus1(int z) { // eb_x_by_xplus1: round(256 z/(z+1)), 0 -> 1, 255 -> 256
    if (z == 0) return 1;
    if (z >= 255) return 256;
    return (256 * z + (z + 1) / 2) / (z + 1);
}
__device__ __forceinline__ uint32_t rpot(uint32_t v, int n) { return n ? (v + (1u << (n - 1))) >> n : v; }

constexpr int SGR_NT = 256;

// tile: (h+6) x (w+6) uint16 samples (stride tw = w+6), origin at (3,3).  A/B: (h+2) x (w+2) int32.
__device__ void sgr_pass(const uint16_t *tile, int tw, int w, int h, int32_t *A, int32_t *B, int32_t *dst, int dst_stride,
                         int bd, int idx, int pass) {
    const int r = c_sgr_r[idx][pass], n = (2 * r + 1) * (2 * r + 1);
    const uint32_t s = (uint32_t)c_sgr_s[idx][pass];
    const uint32_t one_by_n = (4096 + n / 2) / n;
    const int bs = w + 2;
    const bool fast = pass == 0;
    const uint16_t *org = tile + 3 * tw + 3;
    __syncthreads();
    for (int t = threadIdx.x; t < (h + 2) * (w + 2); t += SGR_NT) {
        const int i = t / bs - 1, j = t % bs - 1;
        if (fast && ((i + 1) & 1)) continue; /* the fast pass evaluates rows -1, 1, 3, ... only */
        uint32_t sum = 0, sq = 0;
        for (int y = -r; y <= r; y++)
            for (int x = -r; x <= r; x++) {
                const uint32_t v = org[(i + y) * tw + j + x];
                sum += v;
                sq += v * v;
            }
        const uint32_t a = rpot(sq, 2 * (bd - 8)), b = rpot(sum, bd - 8);
        const uint32_t p = (a * n < b * b) ? 0 : a * n - b * b;
        const uint32_t z = rpot(p * s, 20);
        const int av = x_by_xplus1((int)min(z, 255u));
        A[t] = av;
        B[t] = (int32_t)rpot((uint32_t)(256 - av) * sum * one_by_n, 12);
    }
    __syncthreads();
#define AA(i, j) A[((i) + 1) * bs + (j) + 1]
#define BB(i, j) B[((i) + 1) * bs + (j) + 1]
    for (int t = threadIdx.x; t < h * w; t += SGR_NT) {
        const int i = t / w, j = t % w;
        int32_t a, b, nb;
        if (!fast) {
            nb = 5;
            a = (AA(i, j) + AA(i, j - 1) + AA(i, j + 1) + AA(i - 1, j) + AA(i + 1, j)) * 4 +
                (AA(i - 1, j - 1) + AA(i + 1, j - 1) + AA(i - 1, j + 1) + AA(i + 1, j + 1)) * 3;
            b = (BB(i, j) + BB(i, j - 1) + BB(i, j + 1) + BB(i - 1, j) + BB(i + 1, j)) * 4 +
                (BB(i - 1, j - 1) + BB(i + 1, j - 1) + BB(i - 1, j + 1) + BB(i + 1, j + 1)) * 3;
        } else if (!(i & 1)) {
            nb = 5;
            a = (AA(i - 1, j) + AA(i + 1, j)) * 6 + (AA(i - 1, j - 1) + AA(i + 1, j - 1) + AA(i - 1, j + 1) + AA(i + 1, j + 1)) * 5;
            b = (BB(i - 1, j) + BB(i + 1, j)) * 6 + (BB(i - 1, j - 1) + BB(i + 1, j - 1) + BB(i - 1, j + 1) + BB(i + 1, j + 1)) * 5;
        } else {
            nb = 4;
            a = AA(i, j) * 6 + (AA(i, j - 1) + AA(i, j + 1)) * 5;
            b = BB(i, j) * 6 + (BB(i, j - 1) + BB(i, j + 1)) * 5;
        }
        const int32_t v = a * (int32_t)org[i * tw + j] + b;
        const int sh = 8 + nb - 4;
        dst[i * dst_stride + j] = (v + (1 << (sh - 1))) >> sh;
    }
#undef AA
#undef BB
}

struct SgrArgs {
    const uint16_t *tile_in; // (h+6) x (w+6) packed samples
    int w, h, bd, idx;
    int32_t *flt0, *flt1; // w-strided outputs (device)
    // apply mode
    int apply, xq0, xq1;
    uint16_t *out; // w-strided
};
__global__ void __launch_bounds__(SGR_NT) sgr_kernel(const SgrArgs a) {
    extern __shared__ int32_t sm[];
    const int tw = a.w + 6, th = a.h + 6;
    int32_t *A = sm, *B = A + (a.w + 2) * (a.h + 2);
    uint16_t *tile = reinterpret_cast<uint16_t *>(B + (a.w + 2) * (a.h + 2));
    for (int i = threadIdx.x; i < tw * th; i += SGR_NT) tile[i] = a.tile_in[i];
    __syncthreads();
    const int r0 = c_sgr_r[a.idx][0], r1 = c_sgr_r[a.idx][1];
    if (r0 > 0) sgr_pass(tile, tw, a.w, a.h, A, B, a.flt0, a.w, a.bd, a.idx, 0);
    if (r1 > 0) sgr_pass(tile, tw, a.w, a.h, A, B, a.flt1, a.w, a.bd, a.idx, 1);
    if (!a.apply) return;
    __syncthreads();
    __threadfence_block();
    const int mx = (1 << a.bd) - 1;
    for (int t = threadIdx.x; t < a.w * a.h; t += SGR_NT) {
        const int i = t / a.w, j = t % a.w;
        const int32_t u = (int32_t)tile[(i + 3) * tw + j + 3] << 4;
        int32_t v = u << 7;
        if (r0 > 0) v += a.xq0 * (a.flt0[t] - u);
        if (r1 > 0) v += a.xq1 * (a.flt1[t] - u);
        const int16_t wv = (int16_t)((v + (1 << 10)) >> 11);
        a.out[t] = (uint16_t)(wv < 0 ? 0 : (wv > mx ? mx : wv));
    }
}

struct WienerArgs {
    const uint16_t *tile_in; // (h+7) x (w+7) packed samples, origin (3,3)
    int w, h, bd, round_0, round_1;
    int16_t fx[8], fy[8];
    uint16_t *out; // w-strided
};
__global__ void __launch_bounds__(256) wiener_kernel(const WienerArgs a) {
    extern __shared__ int32_t sm[];
    const int tw = a.w + 7, ih = a.h + 7;
    uint16_t *tile = reinterpret_cast<uint16_t *>(sm);
    uint16_t *tmp = tile + tw * ih;
    for (int i = threadIdx.x; i < tw * ih; i += blockDim.x) tile[i] = a.tile_in[i];
    __syncthreads();
    const int lim = (1 << (a.bd + 1 + 7 - a.round_0)) - 1;
    for (int t = threadIdx.x; t < ih * a.w; t += blockDim.x) {
        const int y = t / a.w, x = t % a.w;
        int32_t sum = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) sum += (int32_t)tile[y * tw + x + k] * a.fx[k];
        sum += ((int32_t)tile[y * tw + x + 3] << 7) + (1 << (a.bd + 7 - 1));
        const int32_t v = (sum + (1 << (a.round_0 - 1))) >> a.round_0;
        tmp[t] = (uint16_t)(v < 0 ? 0 : (v > lim ? lim : v));
    }
    __syncthreads();
    const int mx = (1 << a.bd) - 1;
    for (int t = threadIdx.x; t < a.h * a.w; t += blockDim.x) {
        const int y = t / a.w, x = t % a.w;
        int32_t sum = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) sum += (int32_t)tmp[(y + k) * a.w + x] * a.fy[k];
        sum += ((int32_t)tmp[(y + 3) * a.w + x] << 7) - (1 << (a.bd + a.round_1 - 1));
        int32_t v = (sum + (1 << (a.round_1 - 1))) >> a.round_1;
        a.out[t] = (uint16_t)(v < 0 ? 0 : (v > mx ? mx : v));
    }
}


// ---------------------------------------------------------------------------------------------------------------
// Frame-level loop restoration (svt_av1_loop_restoration_filter_frame).  Work item = one processing unit (64 luma /
// 32 chroma samples wide) of one stripe (64 / 32 rows, the first one 8 / 4 rows shorter).  Stripes and processing-unit
// columns are global partitions of the plane (restoration units are unions of them), so an item is (plane, stripe,
// column) in closed form and the unit it belongs to follows from its top-left sample.  The reference overwrites the 3
// rows above / below a stripe IN PLACE with saved boundary lines, filters, and restores them; that input is a pure
// function of (CDEF picture, deblocked picture): rows {-3,-2,-1} = deblocked rows {y0-2, y0-2, y0-1}, rows
// {h, h+1, h+2} = deblocked rows {y1, y1+1, y1+1} (clamped to the plane), columns clamped to the plane
// (extend_lines / svt_extend_frame); the first / last stripe of the picture keeps the CDEF rows (clamped).  The CTA
// composes that tile in shared memory and runs the same filter cores as the drop-ins.
// ---------------------------------------------------------------------------------------------------------------
struct LrPlaneDev {
    const void *cdef, *dblk;
    void *out;
    int stride_c, stride_d, stride_o;
    int w, h, ss; // plane size, 1 for chroma
    int rtype, unit_size, hunits, vunits;
    const SvtB200LrUnit *units;
    int n_stripes, n_cols, item0;
};
struct LrFrameDev {
    LrPlaneDev pl[3];
    int bd, optimized, n_items;
};
constexpr int LR_SMEM = (71 * 71 * 2 + 15) / 16 * 16 + 2 * 66 * 66 * 4 + 2 * 64 * 64 * 4; // tile + A/B + flt0/flt1

template <typename T>
__global__ void __launch_bounds__(SGR_NT) lr_frame_kernel(const __grid_constant__ LrFrameDev d) {
    extern __shared__ int32_t sm[];
    const int item = blockIdx.x;
    const int pi = item >= d.pl[2].item0 ? 2 : item >= d.pl[1].item0 ? 1 : 0;
    const LrPlaneDev &pl = d.pl[pi];
    const int li = item - pl.item0, s = li / pl.n_cols, c = li - s * pl.n_cols;
    const int SH = 64 >> pl.ss, off = 8 >> pl.ss, PW = 64 >> pl.ss;
    const int ys = max(0, s * SH - off), ye = min((s + 1) * SH - off, pl.h), h = ye - ys;
    const int xs = c * PW, w = min(PW, pl.w - xs);
    const T *cdef = reinterpret_cast<const T *>(pl.cdef);
    const T *dblk = reinterpret_cast<const T *>(pl.dblk);
    T *out = reinterpret_cast<T *>(pl.out);
    int type = 0;
    const SvtB200LrUnit *u = nullptr;
    if (pl.rtype) {
        const int ui = min((ys + (s ? off : 0)) / pl.unit_size, pl.vunits - 1), uj = min(xs / pl.unit_size, pl.hunits - 1);
        u = pl.units + ui * pl.hunits + uj;
        type = u->restoration_type;
    }
    if (type == 0) { // RESTORE_NONE: copy_tile
        for (int t = threadIdx.x; t < w * h; t += SGR_NT) {
            const int i = t / w, j = t - i * w;
            out[(size_t)(ys + i) * pl.stride_o + xs + j] = cdef[(size_t)(ys + i) * pl.stride_c + xs + j];
        }
        return;
    }
    // ---- compose the (h+7) x (w+7) input tile, origin (3,3) ----
    uint16_t *tile = reinterpret_cast<uint16_t *>(sm);
    const int tw = w + 7, th = h + 7;
    const bool copy_above = s > 0, copy_below = (s + 1) * SH - off < pl.h;
    for (int t = threadIdx.x; t < tw * th; t += SGR_NT) {
        const int r = t / tw - 3, cx = t - (t / tw) * tw - 3;
        const int x = min(max(xs + cx, 0), pl.w - 1);
        int yy = ys + r;
        bool from_dblk = false;
        if (r < 0 && copy_above) {
            if (!d.optimized) {
                yy = ys - 2 + max(r + 2, 0);
                from_dblk = true;
            } else if (r == -3) {
                yy = ys - 2;
            }
        } else if (r >= h && copy_below) {
            const int i = r - h;
            if (!d.optimized) {
                yy = ye + min(i, 1);
                from_dblk = true;
            } else if (i >= 2) {
                yy = ye + 1;
            }
        }
        yy = min(max(yy, 0), pl.h - 1);
        tile[t] = from_dblk ? (uint16_t)dblk[(size_t)yy * pl.stride_d + x] : (uint16_t)cdef[(size_t)yy * pl.stride_c + x];
    }
    __syncthreads();
    const int bd = d.bd, mx = (1 << bd) - 1;
    if (type == 1) { // RESTORE_WIENER: wiener_filter_stripe[_highbd] with get_conv_params_wiener(bd)
        int round_0 = 3, round_1 = 11;
        if (bd + 7 - round_0 + 2 > 16) {
            const int e = bd + 7 - round_0 + 2 - 16;
            round_0 += e;
            round_1 -= e;
        }
        uint16_t *tmp = tile + ((tw * th + 7) & ~7);
        const int lim = (1 << (bd + 1 + 7 - round_0)) - 1;
        for (int t = threadIdx.x; t < th * w; t += SGR_NT) {
            const int y = t / w, x = t - y * w;
            int32_t sum = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) sum += (int32_t)tile[y * tw + x + k] * u->hfilter[k];
            sum += ((int32_t)tile[y * tw + x + 3] << 7) + (1 << (bd + 7 - 1));
            const int32_t v = (sum + (1 << (round_0 - 1))) >> round_0;
            tmp[t] = (uint16_t)(v < 0 ? 0 : (v > lim ? lim : v));
        }
        __syncthreads();
        for (int t = threadIdx.x; t < h * w; t += SGR_NT) {
            const int y = t / w, x = t - y * w;
            int32_t sum = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) sum += (int32_t)tmp[(y + k) * w + x] * u->vfilter[k];
            sum += ((int32_t)tmp[(y + 3) * w + x] << 7) - (1 << (bd + round_1 - 1));
            const int32_t v = (sum + (1 << (round_1 - 1))) >> round_1;
            out[(size_t)(ys + y) * pl.stride_o + xs + x] = (T)(v < 0 ? 0 : (v > mx ? mx : v));
        }
        return;
    }
    // RESTORE_SGRPROJ: svt_apply_selfguided_restoration (the SGR cores read a (h+6) x (w+6) tile of pitch tw)
    int32_t *A = sm + ((71 * 71 * 2 + 15) / 16 * 16) / 4, *B = A + 66 * 66, *flt0 = B + 66 * 66, *flt1 = flt0 + 64 * 64;
    const int idx = u->sgr_ep;
    const int r0 = c_sgr_r[idx][0], r1 = c_sgr_r[idx][1];
    if (r0 > 0) sgr_pass(tile, tw, w, h, A, B, flt0, w, bd, idx, 0);
    if (r1 > 0) sgr_pass(tile, tw, w, h, A, B, flt1, w, bd, idx, 1);
    __syncthreads();
    int xq0, xq1; // svt_decode_xq
    if (r0 == 0) {
        xq0 = 0;
        xq1 = 128 - u->sgr_xqd[1];
    } else if (r1 == 0) {
        xq0 = u->sgr_xqd[0];
        xq1 = 0;
    } else {
        xq0 = u->sgr_xqd[0];
        xq1 = 128 - xq0 - u->sgr_xqd[1];
    }
    for (int t = threadIdx.x; t < w * h; t += SGR_NT) {
        const int i = t / w, j = t - i * w;
        const int32_t uu = (int32_t)tile[(i + 3) * tw + j + 3] << 4;
        int32_t v = uu << 7;
        if (r0 > 0) v += xq0 * (flt0[t] - uu);
        if (r1 > 0) v += xq1 * (flt1[t] - uu);
        const int16_t wv = (int16_t)((v + (1 << 10)) >> 11);
        out[(size_t)(ys + i) * pl.stride_o + xs + j] = (T)(wv < 0 ? 0 : (wv > mx ? mx : wv));
    }
}


// ---------------------------------------------------------------------------------------------------------------
// Self-guided SEARCH, device resident (search_selfguided_restoration, EbRestorationPick.c:583-661): for every
// restoration unit and every parameter set ep of a list, apply_sgr (:554-581: the filter per processing unit, tiled
// from the unit's origin) with both outputs kept in HBM (16 sets x 2 x 4 B x 3.1 M samples = 400 MB at 1080p: what
// 180 GB are for), plus the five sums of svt_get_proj_subspace per (unit, ep).  A second entry evaluates
// get_pixel_proj_error for one candidate xq per (unit, ep), so the host's hill climb (finer_search_pixel_proj_error)
// costs one launch + one small read-back per step for ALL units and parameter sets at once.
// ---------------------------------------------------------------------------------------------------------------
struct SgrSearchDev {
    const void *dgd, *src;
    int dgd_stride, src_stride, pw, ph, ss, bd;
    const int32_t *rects; // [n_units][4] h_start, h_end, v_start, v_end
    int eps[16], n_eps, tiles_x;
    int32_t *flt; // [n_eps][2][ph][pw]
    long long *sums; // [n_units][n_eps][5]: H00 H11 H01 C0 C1
    const int32_t *xq; // [n_units][n_eps][2]
    long long *err; // [n_units][n_eps]
};

template <typename T>
__global__ void __launch_bounds__(SGR_NT) sgr_search_filter_kernel(const __grid_constant__ SgrSearchDev d) {
    extern __shared__ int32_t sm[];
    const int unit = blockIdx.y, ei = blockIdx.z, idx = d.eps[ei];
    const int32_t *rc = d.rects + 4 * unit;
    const int PU = 64 >> d.ss;
    const int tx = blockIdx.x % d.tiles_x, ty = blockIdx.x / d.tiles_x;
    const int xs = rc[0] + tx * PU, ys = rc[2] + ty * PU;
    if (xs >= rc[1] || ys >= rc[3]) return;
    const int w = min(PU, rc[1] - xs), h = min(PU, rc[3] - ys);
    const T *dg = reinterpret_cast<const T *>(d.dgd);
    const T *sr = reinterpret_cast<const T *>(d.src);
    uint16_t *tile = reinterpret_cast<uint16_t *>(sm);
    const int tw = w + 6, th = h + 6;
    for (int t = threadIdx.x; t < tw * th; t += SGR_NT) { // the unit's surroundings, clamped = the extended picture
        const int r = t / tw, c = t - r * tw;
        const int yy = min(max(ys + r - 3, 0), d.ph - 1), xx = min(max(xs + c - 3, 0), d.pw - 1);
        tile[t] = (uint16_t)dg[(size_t)yy * d.dgd_stride + xx];
    }
    int32_t *A = sm + ((71 * 71 * 2 + 15) / 16 * 16) / 4, *B = A + 66 * 66, *flt0 = B + 66 * 66, *flt1 = flt0 + 64 * 64;
    const int r0 = c_sgr_r[idx][0], r1 = c_sgr_r[idx][1];
    if (r0 > 0) sgr_pass(tile, tw, w, h, A, B, flt0, w, d.bd, idx, 0);
    if (r1 > 0) sgr_pass(tile, tw, w, h, A, B, flt1, w, d.bd, idx, 1);
    __syncthreads();
    const size_t plane = (size_t)d.pw * d.ph;
    int32_t *g0 = d.flt + (size_t)ei * 2 * plane, *g1 = g0 + plane;
    long long v[5] = {0, 0, 0, 0, 0};
    for (int t = threadIdx.x; t < w * h; t += SGR_NT) {
        const int i = t / w, j = t - i * w;
        const size_t o = (size_t)(ys + i) * d.pw + xs + j;
        const long long u = (long long)tile[(i + 3) * tw + j + 3] << 4;
        const long long s = ((long long)sr[(size_t)(ys + i) * d.src_stride + xs + j] << 4) - u;
        long long f1 = 0, f2 = 0;
        if (r0 > 0) {
            g0[o] = flt0[t];
            f1 = flt0[t] - u;
        }
        if (r1 > 0) {
            g1[o] = flt1[t];
            f2 = flt1[t] - u;
        }
        v[0] += f1 * f1, v[1] += f2 * f2, v[2] += f1 * f2, v[3] += f1 * s, v[4] += f2 * s;
    }
    long long *out = d.sums + ((size_t)unit * d.n_eps + ei) * 5;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
        if ((threadIdx.x & 31) == 0 && v[k]) atomicAdd(reinterpret_cast<unsigned long long *>(out + k), (unsigned long long)v[k]);
    }
}

template <typename T>
__global__ void __launch_bounds__(256) sgr_search_error_kernel(const __grid_constant__ SgrSearchDev d) {
    const int unit = blockIdx.y, ei = blockIdx.z, idx = d.eps[ei];
    const int32_t *rc = d.rects + 4 * unit;
    const int w = rc[1] - rc[0], h = rc[3] - rc[2];
    const T *dg = reinterpret_cast<const T *>(d.dgd);
    const T *sr = reinterpret_cast<const T *>(d.src);
    const int r0 = c_sgr_r[idx][0], r1 = c_sgr_r[idx][1];
    const int xq0 = d.xq[((size_t)unit * d.n_eps + ei) * 2], xq1 = d.xq[((size_t)unit * d.n_eps + ei) * 2 + 1];
    const size_t plane = (size_t)d.pw * d.ph;
    const int32_t *g0 = d.flt + (size_t)ei * 2 * plane, *g1 = g0 + plane;
    const bool hbd = sizeof(T) == 2;
    long long acc = 0;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < w * h; t += gridDim.x * blockDim.x) {
        const int i = t / w, j = t - i * w;
        const int y = rc[2] + i, x = rc[0] + j;
        const int dv = dg[(size_t)y * d.dgd_stride + x], s = sr[(size_t)y * d.src_stride + x];
        int e;
        if (r0 > 0 || r1 > 0) { // svt_av1_{lowbd,highbd}_pixel_proj_error_c
            const int u = dv << 4;
            int v = hbd ? (1 << 10) : (u << 7);
            if (r0 > 0) v += xq0 * (g0[(size_t)y * d.pw + x] - u);
            if (r1 > 0) v += xq1 * (g1[(size_t)y * d.pw + x] - u);
            e = hbd ? (v >> 11) + dv - s : ((v + (1 << 10)) >> 11) - s;
        } else {
            e = dv - s;
        }
        acc += (long long)(e * e);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(reinterpret_cast<unsigned long long *>(d.err + (size_t)unit * d.n_eps + ei), (unsigned long long)acc);
}

static void lr_attrs() {
    static PerDeviceOnce once;
    once.run([] {
        SVTB_ATTR(sgr_kernel, 96 * 1024);
        SVTB_ATTR(wiener_kernel, 96 * 1024);
        SVTB_ATTR(lr_frame_kernel<uint8_t>, LR_SMEM);
        SVTB_ATTR(lr_frame_kernel<uint16_t>, LR_SMEM);
        SVTB_ATTR(sgr_search_filter_kernel<uint8_t>, LR_SMEM);
        SVTB_ATTR(sgr_search_filter_kernel<uint16_t>, LR_SMEM);
    });
}

// The reference passes high-bit-depth planes as CONVERT_TO_BYTEPTR(ptr) (= ptr >> 1): undo it like CONVERT_TO_SHORTPTR
static inline const uint16_t *short_ptr(const uint8_t *p) { return (const uint16_t *)(((uintptr_t)p) << 1); }

// gather a rim-extended rectangle into packed uint16
static void gather(uint16_t *dst, const uint8_t *src8, int highbd, ptrdiff_t stride, int x0, int y0, int w, int h) {
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const ptrdiff_t o = (ptrdiff_t)(y0 + y) * stride + x0 + x;
            dst[(size_t)y * w + x] = highbd ? short_ptr(src8)[o] : src8[o];
        }
}

static void sgr_run(const uint8_t *dat8, int width, int height, int stride, int eps, int bit_depth, int highbd, int32_t *flt0,
                    int32_t *flt1, int flt_stride, const int32_t *xqd, uint8_t *dst8, int dst_stride) {
    lr_attrs();
    if ((size_t)(width + 6) * (height + 6) > 7396 + 2000 || width <= 0 || height <= 0 || eps < 0 || eps > 15) {
        fprintf(stderr, "svt_av1_selfguided_restoration_cuda: unit %dx%d larger than a restoration processing unit\n", width, height);
        abort();
    }
    const size_t tile_b = (size_t)(width + 6) * (height + 6) * 2, fb = (size_t)width * height * 4;
    Staging s({tile_b, fb, fb, (size_t)width * height * 2});
    SVTB_CUDA_FATAL(s.status());
    gather(s.h<uint16_t>(0), dat8, highbd, stride, -3, -3, width + 6, height + 6);
    SVTB_CUDA_FATAL(s.upload(0, 0));
    SgrArgs a;
    a.tile_in = s.d<const uint16_t>(0);
    a.w = width;
    a.h = height;
    a.bd = bit_depth;
    a.idx = eps;
    a.flt0 = s.d<int32_t>(1);
    a.flt1 = s.d<int32_t>(2);
    a.apply = xqd != nullptr;
    a.xq0 = a.xq1 = 0;
    if (xqd) { // svt_decode_xq
        const int r0 = h_sgr_r[eps][0], r1 = h_sgr_r[eps][1];
        if (r0 == 0) {
            a.xq0 = 0;
            a.xq1 = 128 - xqd[1];
        } else if (r1 == 0) {
            a.xq0 = xqd[0];
            a.xq1 = 0;
        } else {
            a.xq0 = xqd[0];
            a.xq1 = 128 - a.xq0 - xqd[1];
        }
    }
    a.out = s.d<uint16_t>(3);
    const size_t smem = (size_t)2 * (width + 2) * (height + 2) * 4 + tile_b + 16;
    SVTB_LAUNCH(sgr_kernel, 1, SGR_NT, smem, s.stream(), a);
    SVTB_CUDA_FATAL(s.download(1, 3));
    if (!xqd) {
        if (h_sgr_r[eps][0] > 0) s.get_rows(1, flt0, flt_stride, 4, width, height);
        if (h_sgr_r[eps][1] > 0) s.get_rows(2, flt1, flt_stride, 4, width, height);
    } else {
        const uint16_t *ho = s.h<uint16_t>(3);
        for (int y = 0; y < height; y++)
            for (int x = 0; x < width; x++) {
                if (highbd)
                    ((uint16_t *)short_ptr(dst8))[(ptrdiff_t)y * dst_stride + x] = ho[(size_t)y * width + x];
                else
                    dst8[(ptrdiff_t)y * dst_stride + x] = (uint8_t)ho[(size_t)y * width + x];
            }
    }
}

static void wiener_run(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst, ptrdiff_t dst_stride, const int16_t *filter_x,
                       const int16_t *filter_y, int w, int h, int round_0, int round_1, int bd, int highbd) {
    lr_attrs();
    if (w <= 0 || h <= 0 || w > 128 || h > 128) {
        fprintf(stderr, "svt_av1_wiener_convolve_add_src_cuda: %dx%d out of range\n", w, h);
        abort();
    }
    const size_t tile_b = (size_t)(w + 7) * (h + 7) * 2;
    Staging s({tile_b, (size_t)w * h * 2});
    SVTB_CUDA_FATAL(s.status());
    gather(s.h<uint16_t>(0), src, highbd, src_stride, -3, -3, w + 7, h + 7);
    SVTB_CUDA_FATAL(s.upload(0, 0));
    WienerArgs a;
    a.tile_in = s.d<const uint16_t>(0);
    a.w = w;
    a.h = h;
    a.bd = bd;
    a.round_0 = round_0;
    a.round_1 = round_1;
    // the reference recovers kernel + offset from a 256-byte aligned table (get_filter_base / get_filter_offset,
    // convolve.c:49-57); with the x/y steps fixed at 16 that always resolves to the 8 taps pointed at
    memcpy(a.fx, filter_x, 16);
    memcpy(a.fy, filter_y, 16);
    a.out = s.d<uint16_t>(1);
    const size_t smem = tile_b + (size_t)(h + 7) * w * 2 + 16;
    SVTB_LAUNCH(wiener_kernel, 1, 256, smem, s.stream(), a);
    SVTB_CUDA_FATAL(s.download(1, 1));
    const uint16_t *ho = s.h<uint16_t>(1);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            if (highbd)
                ((uint16_t *)short_ptr(dst))[(ptrdiff_t)y * dst_stride + x] = ho[(size_t)y * w + x];
            else
                dst[(ptrdiff_t)y * dst_stride + x] = (uint8_t)ho[(size_t)y * w + x];
        }
}

} // namespace

extern "C" {

void svt_av1_selfguided_restoration_cuda(const uint8_t *dgd8, int32_t width, int32_t height, int32_t dgd_stride, int32_t *flt0,
                                         int32_t *flt1, int32_t flt_stride, int32_t sgr_params_idx, int32_t bit_depth,
                                         int32_t highbd) {
    sgr_run(dgd8, width, height, dgd_stride, sgr_params_idx, bit_depth, highbd, flt0, flt1, flt_stride, nullptr, nullptr, 0);
}
void svt_apply_selfguided_restoration_cuda(const uint8_t *dat, int32_t width, int32_t height, int32_t stride, int32_t eps,
                                           const int32_t *xqd, uint8_t *dst, int32_t dst_stride, int32_t *tmpbuf,
                                           int32_t bit_depth, int32_t highbd) {
    (void)tmpbuf;
    sgr_run(dat, width, height, stride, eps, bit_depth, highbd, nullptr, nullptr, 0, xqd, dst, dst_stride);
}
// conv_params: the reference's ConvolveParams; only round_0 / round_1 are read (offsets 20 and 24 of the struct,
// EbDefinitions.h:379-392) — passed as a pointer to keep the RTCD signature
struct ConvolveParamsView {
    int32_t ref, do_average;
    void *dst;
    int32_t dst_stride, round_0, round_1;
};
void svt_av1_wiener_convolve_add_src_cuda(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst, ptrdiff_t dst_stride,
                                          const int16_t *filter_x, const int16_t *filter_y, int32_t w, int32_t h,
                                          const void *conv_params) {
    const ConvolveParamsView *cp = (const ConvolveParamsView *)conv_params;
    wiener_run(src, src_stride, dst, dst_stride, filter_x, filter_y, w, h, cp->round_0, cp->round_1, 8, 0);
}
void svt_av1_highbd_wiener_convolve_add_src_cuda(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst, ptrdiff_t dst_stride,
                                                 const int16_t *filter_x, const int16_t *filter_y, int32_t w, int32_t h,
                                                 const void *conv_params, int32_t bd) {
    const ConvolveParamsView *cp = (const ConvolveParamsView *)conv_params;
    wiener_run(src, src_stride, dst, dst_stride, filter_x, filter_y, w, h, cp->round_0, cp->round_1, bd, 1);
}

int svt_b200_lr_frame(const SvtB200LrFrameParams *p, const SvtB200Frame *cdef, const SvtB200Frame *deblocked, const SvtB200Frame *out,
                      void *stream) {
    if (!p || !cdef || !deblocked || !out || cdef->bit_depth != deblocked->bit_depth || cdef->bit_depth != out->bit_depth ||
        cdef->width != out->width || cdef->height != out->height || out->y == cdef->y || out->y == deblocked->y) {
        set_error("svt_b200_lr_frame: bad argument (out must not alias the inputs)");
        return SVT_B200_ERR_ARG;
    }
    lr_attrs();
    LrFrameDev d;
    memset(&d, 0, sizeof(d));
    d.bd = cdef->bit_depth;
    d.optimized = p->optimized_lr != 0;
    int items = 0;
    for (int i = 0; i < 3; i++) {
        LrPlaneDev &pl = d.pl[i];
        const int ss = i ? 1 : 0;
        pl.cdef = i == 0 ? cdef->y : i == 1 ? cdef->cb : cdef->cr;
        pl.dblk = i == 0 ? deblocked->y : i == 1 ? deblocked->cb : deblocked->cr;
        pl.out = i == 0 ? out->y : i == 1 ? out->cb : out->cr;
        pl.stride_c = i ? cdef->stride_c : cdef->stride_y;
        pl.stride_d = i ? deblocked->stride_c : deblocked->stride_y;
        pl.stride_o = i ? out->stride_c : out->stride_y;
        pl.ss = ss;
        pl.w = (cdef->width + ss) >> ss; // ROUND_POWER_OF_TWO(frame size, ss): whole_frame_rect
        pl.h = (cdef->height + ss) >> ss;
        pl.rtype = p->plane[i].frame_restoration_type;
        pl.unit_size = p->plane[i].restoration_unit_size;
        if (pl.rtype) {
            if (!p->plane[i].units || pl.unit_size < (64 >> ss) || (pl.unit_size % (64 >> ss))) {
                set_error("svt_b200_lr_frame: bad restoration unit size / missing unit array");
                return SVT_B200_ERR_ARG;
            }
            pl.hunits = std::max((pl.w + (pl.unit_size >> 1)) / pl.unit_size, 1); // count_units_in_tile
            pl.vunits = std::max((pl.h + (pl.unit_size >> 1)) / pl.unit_size, 1);
            pl.units = p->plane[i].units;
        }
        const int SH = 64 >> ss, off = 8 >> ss;
        pl.n_stripes = (pl.h + off + SH - 1) / SH;
        pl.n_cols = (pl.w + SH - 1) / SH;
        pl.item0 = items;
        items += pl.n_stripes * pl.n_cols;
    }
    d.n_items = items;
    cudaStream_t st = (cudaStream_t)stream;
    if (d.bd > 8)
        SVTB_LAUNCH(lr_frame_kernel<uint16_t>, items, SGR_NT, LR_SMEM, st, d);
    else
        SVTB_LAUNCH(lr_frame_kernel<uint8_t>, items, SGR_NT, LR_SMEM, st, d);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

static int sgr_search_setup(SgrSearchDev &d, const SvtB200Frame *dgd, const SvtB200Frame *src, int plane, const int32_t *rects, int n_units,
                            const int32_t *eps, int n_eps, int32_t *flt) {
    if (!dgd || !src || !rects || !eps || !flt || plane < 0 || plane > 2 || n_units <= 0 || n_eps <= 0 || n_eps > 16 ||
        dgd->bit_depth != src->bit_depth)
        return -1;
    memset(&d, 0, sizeof(d));
    const int ss = plane ? 1 : 0;
    d.dgd = plane == 0 ? dgd->y : plane == 1 ? dgd->cb : dgd->cr;
    d.src = plane == 0 ? src->y : plane == 1 ? src->cb : src->cr;
    d.dgd_stride = plane ? dgd->stride_c : dgd->stride_y;
    d.src_stride = plane ? src->stride_c : src->stride_y;
    d.pw = (dgd->width + ss) >> ss;
    d.ph = (dgd->height + ss) >> ss;
    d.ss = ss;
    d.bd = dgd->bit_depth;
    d.rects = rects;
    d.n_eps = n_eps;
    for (int i = 0; i < n_eps; i++) {
        if (eps[i] < 0 || eps[i] > 15) return -1;
        d.eps[i] = eps[i];
    }
    d.flt = flt;
    return 0;
}

int svt_b200_lr_sgr_filter_sums(const SvtB200Frame *dgd, const SvtB200Frame *src, int32_t plane, const int32_t *rects, int32_t n_units,
                                int32_t max_unit_w, int32_t max_unit_h, const int32_t *eps, int32_t n_eps, int32_t *flt, int64_t *sums,
                                void *stream) {
    SgrSearchDev d;
    if (!sums || max_unit_w <= 0 || max_unit_h <= 0 || sgr_search_setup(d, dgd, src, plane, rects, n_units, eps, n_eps, flt)) {
        set_error("svt_b200_lr_sgr_filter_sums: bad argument");
        return SVT_B200_ERR_ARG;
    }
    lr_attrs();
    d.sums = (long long *)sums;
    const int PU = 64 >> d.ss;
    d.tiles_x = (max_unit_w + PU - 1) / PU;
    const int tiles_y = (max_unit_h + PU - 1) / PU;
    cudaStream_t st = (cudaStream_t)stream;
    SVTB_CUDA_TRY(cudaMemsetAsync(sums, 0, (size_t)n_units * n_eps * 5 * 8, st));
    const dim3 grid(d.tiles_x * tiles_y, n_units, n_eps);
    if (d.bd > 8)
        SVTB_LAUNCH(sgr_search_filter_kernel<uint16_t>, grid, SGR_NT, LR_SMEM, st, d);
    else
        SVTB_LAUNCH(sgr_search_filter_kernel<uint8_t>, grid, SGR_NT, LR_SMEM, st, d);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

int svt_b200_lr_sgr_proj_error(const SvtB200Frame *dgd, const SvtB200Frame *src, int32_t plane, const int32_t *rects, int32_t n_units,
                               int32_t max_unit_w, int32_t max_unit_h, const int32_t *eps, int32_t n_eps, const int32_t *flt,
                               const int32_t *xq, int64_t *err, void *stream) {
    SgrSearchDev d;
    if (!xq || !err || max_unit_w <= 0 || max_unit_h <= 0 ||
        sgr_search_setup(d, dgd, src, plane, rects, n_units, eps, n_eps, const_cast<int32_t *>(flt))) {
        set_error("svt_b200_lr_sgr_proj_error: bad argument");
        return SVT_B200_ERR_ARG;
    }
    d.xq = xq;
    d.err = (long long *)err;
    cudaStream_t st = (cudaStream_t)stream;
    SVTB_CUDA_TRY(cudaMemsetAsync(err, 0, (size_t)n_units * n_eps * 8, st));
    const dim3 grid(std::min(16, (max_unit_w * max_unit_h + 255) / 256), n_units, n_eps);
    if (d.bd > 8)
        SVTB_LAUNCH(sgr_search_error_kernel<uint16_t>, grid, 256, 0, st, d);
    else
        SVTB_LAUNCH(sgr_search_error_kernel<uint8_t>, grid, 256, 0, st, d);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}
}
