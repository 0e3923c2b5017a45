// cdef.cu — constrained directional enhancement filter on sm_90a.
//
// Replaces (reference files under Source/Lib):
//   svt_cdef_find_dir_c, svt_cdef_filter_block_c, svt_cdef_filter_fb   Common/Codec/EbCdef.c:132-388
//   cdef_seg_search / cdef_seg_search16bit                             Encoder/Codec/EbCdefProcess.c:80-475
//   compute_cdef_dist_c / _8bit_c (incl. the double-precision 8x8 distortion) Encoder/Codec/EbEncCdef.c:20-220
//   svt_av1_cdef_frame / av1_cdef_frame16bit                           Encoder/Codec/EbEncCdef.c:292-1030
//
// Design: the strength search runs two CTAs per 64x64 filter block, one for luma and one for both chroma planes (it
// stages the luma tile too, for the block directions).  Each plane of the deblocked reconstruction of the block (+2
// sample rim, frame exterior = CDEF_VERY_LARGE) is staged ONCE into shared memory as int16 and every strength of the
// search is evaluated from that tile, so HBM traffic is recon + source once per block (2 B/sample, SURVEY §8d) instead
// of once per strength.  One kernel body has two search forms: the separable form for the pri x sec grids that every
// encoder table is (plane_search_grid), and one pass per strength for any other list (plane_search_list).  The apply
// runs one CTA per filter block.  The 8x8 luma distortion keeps the reference's double formula with explicit
// round-to-nearest intrinsics (no FMA contraction) so it is bit-identical (0 ULP).
#include <algorithm>

#include "common.cuh"

using namespace svtb200;

namespace {

constexpr int VERY_LARGE = 16384; // CDEF_VERY_LARGE
constexpr int TS = 72; // tile row stride (int16): 64 + 2*2 rim, padded
constexpr int NT = 256;

__constant__ int8_t c_dir[8][2][2] = {{{-1, 1}, {-2, 2}}, {{0, 1}, {-1, 2}}, {{0, 1}, {0, 2}}, {{0, 1}, {1, 2}},
                                      {{1, 1}, {2, 2}},   {{1, 0}, {2, 1}},  {{1, 0}, {2, 0}}, {{1, 0}, {2, -1}}};

__device__ __forceinline__ int msb(uint32_t n) { return 31 - __clz((int)n); }

// constrain() of EbCdef.c:86-93 with the shift (max(0, damping - msb(threshold))) hoisted by the caller
// sign(diff) * min(|diff|, lim) == clamp(diff, -lim, lim) for lim >= 0; -lim = min(0, (|diff| >> shift) - threshold)
// is one VIADDMNMX (DPX add+min), so the whole function is IABS, SHF, VIADDMNMX, neg, VIMNMX, VIMNMX.
__device__ __forceinline__ int constrain_s(int diff, int threshold, int shift) {
    const int nlim = __viaddmin_s32(abs(diff) >> shift, -threshold, 0);
    return min(max(diff, nlim), -nlim);
}
__device__ __forceinline__ int adjust_strength(int strength, int var) {
    const int i = (var >> 6) ? min(msb((uint32_t)(var >> 6)), 12) : 0;
    return var ? (strength * (4 + i) + 8) >> 4 : 0;
}

// Tile offsets of the primary taps (direction dir) and the secondary taps (dir +/- 2) in a tile of row stride s
__device__ __forceinline__ void tap_offsets(int dir, int s, int (&po)[2], int (&o2)[2], int (&o6)[2]) {
#pragma unroll
    for (int k = 0; k < 2; k++) {
        po[k] = c_dir[dir][k][0] * s + c_dir[dir][k][1];
        o2[k] = c_dir[(dir + 2) & 7][k][0] * s + c_dir[(dir + 2) & 7][k][1];
        o6[k] = c_dir[(dir + 6) & 7][k][0] * s + c_dir[(dir + 6) & 7][k][1];
    }
}

// svt_cdef_filter_block_c for one sample, with everything that is constant over a block hoisted into CdefTaps by the
// caller: tap offsets for the block's direction, damping shifts, tap weights.  `in` points into an int16 tile of the row
// stride `s` given to make_taps.  kBorder = false is used for filter blocks that do not touch the frame edge (no
// CDEF_VERY_LARGE samples in the tile): the "!= VERY_LARGE" tests vanish.  For pri == sec == 0 the result is x, which
// lies inside [min, max].
struct CdefTaps {
    int po[2], o2[2], o6[2];
    int pt0, pt1, psh, ssh;
};
__device__ __forceinline__ CdefTaps make_taps(int pri, int sec, int dir, int pri_damping, int sec_damping, int coeff_shift, int s) {
    CdefTaps t;
    tap_offsets(dir, s, t.po, t.o2, t.o6);
    const int odd = (pri >> coeff_shift) & 1;
    t.pt0 = odd ? 3 : 4;
    t.pt1 = odd ? 3 : 2;
    t.psh = pri ? max(0, pri_damping - msb((uint32_t)pri)) : 0;
    t.ssh = sec ? max(0, sec_damping - msb((uint32_t)sec)) : 0;
    return t;
}
template <bool kBorder>
__device__ __forceinline__ int cdef_px(const int16_t *in, const CdefTaps &t, int pri, int sec) {
    const int x = in[0];
    int sum = 0, mx = x, mn = x;
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const int p0 = in[t.po[k]], p1 = in[-t.po[k]];
        const int s0 = in[t.o2[k]], s1 = in[-t.o2[k]], s2 = in[t.o6[k]], s3 = in[-t.o6[k]];
        if (pri) sum += (k ? t.pt1 : t.pt0) * (constrain_s(p0 - x, pri, t.psh) + constrain_s(p1 - x, pri, t.psh));
        if (sec)
            sum += (k ? 1 : 2) * (constrain_s(s0 - x, sec, t.ssh) + constrain_s(s1 - x, sec, t.ssh) + constrain_s(s2 - x, sec, t.ssh) +
                                  constrain_s(s3 - x, sec, t.ssh));
        mn = min(mn, min(min(p0, p1), min(min(s0, s1), min(s2, s3))));
        if (kBorder) {
            if (p0 != VERY_LARGE) mx = max(mx, p0);
            if (p1 != VERY_LARGE) mx = max(mx, p1);
            if (s0 != VERY_LARGE) mx = max(mx, s0);
            if (s1 != VERY_LARGE) mx = max(mx, s1);
            if (s2 != VERY_LARGE) mx = max(mx, s2);
            if (s3 != VERY_LARGE) mx = max(mx, s3);
        } else {
            mx = max(mx, max(max(p0, p1), max(max(s0, s1), max(s2, s3))));
        }
    }
    const int y = x + ((8 + sum - (sum < 0)) >> 4);
    return min(max(y, mn), mx);
}

// svt_cdef_find_dir_c (EbCdef.c:132-232) on an 8x8 block of an int16 tile, EIGHT lanes per block (L = lane & 7, the
// eight lanes are consecutive and all active).  Lane L holds row L and column L of the block.  A directional line sum
// ("partial") gathers one sample per row: with a rotate-by-(L -/+ j) shuffle of register j every lane collects the
// two lines whose index is L mod 8 — e.g. for direction 0 (bin = i + j) lane L gets x[i][j] from lane i = (L - j) & 7,
// which belongs to bin L when j <= L and to bin L + 8 otherwise.  Directions 1/3 use the row-pair sums, 5/7 are the
// same patterns on the transposed block.  Weights 840/k are the reference's div_table.  Costs are then summed over
// the eight lanes; every lane returns the direction and *var.
__device__ __forceinline__ int find_dir8(const int16_t *img, int stride, int *var, int coeff_shift) {
    const int lane = threadIdx.x & 31, L = lane & 7, base = lane & ~7;
    int x[8], t[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        x[j] = (img[L * stride + j] >> coeff_shift) - 128;
        t[j] = (img[j * stride + L] >> coeff_shift) - 128;
    }
    int c[8];
    { // directions 2 (bin = i) and 6 (bin = j)
        int sr = 0, sc = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            sr += x[j];
            sc += t[j];
        }
        c[2] = sr * sr * 105;
        c[6] = sc * sc * 105;
    }
    { // direction 0: bin = i + j;  direction 4: bin = 7 + i - j
        int a0 = 0, b0 = 0, a4 = 0, b4 = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int v0 = __shfl_sync(0xffffffffu, x[j], base + ((L - j) & 7));
            const int v4 = __shfl_sync(0xffffffffu, x[j], base + ((L + j) & 7));
            if (j <= L)
                a0 += v0; // bin L
            else
                b0 += v0; // bin L + 8
            if (L + j < 8)
                a4 += v4; // bin 7 + L
            else
                b4 += v4; // bin L - 1
        }
        c[0] = a0 * a0 * (840 / (L + 1)) + (L < 7 ? b0 * b0 * (840 / (7 - L)) : 0);
        c[4] = a4 * a4 * (840 / (8 - L)) + (L > 0 ? b4 * b4 * (840 / L) : 0);
    }
    // odd directions: bins 0..10, weight 105 for bins 3..7, 420/(b+1) for b < 3, 420/(11-b) for b > 7
    const int w_lo = L < 3 ? 420 / (L + 1) : 105; // bin L
    const int w_lo8 = L < 3 ? 420 / (3 - L) : 0; // bin L + 8 (exists for L <= 2)
    const int w_hi = L < 5 ? 105 : 420 / (8 - L); // bin 3 + L
    const int w_hi5 = L >= 5 ? 420 / (L - 4) : 0; // bin L - 5 (exists for L >= 5)
    int a1 = 0, b1 = 0, a3 = 0, b3 = 0, a7 = 0, b7 = 0, a5 = 0, b5 = 0;
#pragma unroll
    for (int s = 0; s < 4; s++) {
        const int pr = x[2 * s] + x[2 * s + 1]; // row L, column pair s
        const int pc = t[2 * s] + t[2 * s + 1]; // column L, row pair s
        const int v1 = __shfl_sync(0xffffffffu, pr, base + ((L - s) & 7)); // direction 1: bin = i + j/2
        const int v3 = __shfl_sync(0xffffffffu, pr, base + ((L + s) & 7)); // direction 3: bin = 3 + i - j/2
        const int v7 = __shfl_sync(0xffffffffu, pc, base + ((L - s) & 7)); // direction 7: bin = i/2 + j
        const int v5 = __shfl_sync(0xffffffffu, pc, base + ((L + s) & 7)); // direction 5: bin = 3 - i/2 + j
        if (s <= L) {
            a1 += v1;
            a7 += v7;
        } else {
            b1 += v1;
            b7 += v7;
        }
        if (L + s < 8) {
            a3 += v3;
            a5 += v5;
        } else {
            b3 += v3;
            b5 += v5;
        }
    }
    c[1] = a1 * a1 * w_lo + b1 * b1 * w_lo8;
    c[7] = a7 * a7 * w_lo + b7 * b7 * w_lo8;
    c[3] = a3 * a3 * w_hi + b3 * b3 * w_hi5;
    c[5] = a5 * a5 * w_hi + b5 * b5 * w_hi5;
#pragma unroll
    for (int d = 0; d < 8; d++)
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) c[d] += __shfl_xor_sync(0xffffffffu, c[d], o);
    int best_cost = 0, best_dir = 0;
#pragma unroll
    for (int d = 0; d < 8; d++)
        if (c[d] > best_cost) {
            best_cost = c[d];
            best_dir = d;
        }
    int orth = 0;
#pragma unroll
    for (int d = 0; d < 8; d++)
        if (d == ((best_dir + 4) & 7)) orth = c[d];
    *var = (best_cost - orth) >> 10;
    return best_dir;
}

// directions + variances of `count` listed blocks (by/bx in 8x8 units inside the tile), eight lanes per block
__device__ __forceinline__ void find_dirs(const int16_t *in, const uint8_t *s_by, const uint8_t *s_bx, int count, int cs, int8_t *s_dir,
                                          int *s_var) {
    const int tid = threadIdx.x;
    for (int b0 = 0; b0 < count; b0 += NT / 8) {
        const int b = b0 + (tid >> 3);
        const int bb = b < count ? b : 0;
        int v;
        const int dir = find_dir8(in + 8 * s_by[bb] * TS + 8 * s_bx[bb], TS, &v, cs);
        if (b < count && (tid & 7) == 0) {
            s_dir[b] = (int8_t)dir;
            s_var[b] = v;
        }
    }
}

struct FrameDev {
    const void *p[3];
    int stride[3];
    int hbd;
};

// Stage the filter block of plane `pli` (+2 rim; outside the frame = VERY_LARGE) into an int16 tile.  Work item = four
// horizontally adjacent samples starting at a frame x that is a multiple of 4 (tile columns 4g-2 .. 4g+1, written as
// two aligned 32-bit shared stores); interior groups are read with one or two 32-bit global loads, groups that
// touch the frame edge sample by sample.  Two items per thread are loaded before the first is stored (the staging is
// global-latency bound: ncu long_scoreboard on the store).
template <typename T>
__device__ __forceinline__ void load_group(const T *plane, int stride, int pw, int ph, int yy, int xx, int (&v)[4]) {
    if (yy < 0 || yy >= ph) {
        v[0] = v[1] = v[2] = v[3] = VERY_LARGE;
        return;
    }
    const T *p = plane + (size_t)yy * stride + xx;
    if (xx >= 0 && xx + 3 < pw) {
        if (sizeof(T) == 1) {
            const uintptr_t a = (uintptr_t)p;
            const uint32_t *g = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
            const uint32_t w = __funnelshift_r(g[0], (a & 3) ? g[1] : 0u, (int)(a & 3) * 8);
            v[0] = w & 0xff, v[1] = (w >> 8) & 0xff, v[2] = (w >> 16) & 0xff, v[3] = w >> 24;
            return;
        }
        if (((uintptr_t)p & 3) == 0) {
            const uint32_t w0 = reinterpret_cast<const uint32_t *>(p)[0], w1 = reinterpret_cast<const uint32_t *>(p)[1];
            v[0] = w0 & 0xffff, v[1] = w0 >> 16, v[2] = w1 & 0xffff, v[3] = w1 >> 16;
            return;
        }
    }
#pragma unroll
    for (int j = 0; j < 4; j++) v[j] = (xx + j >= 0 && xx + j < pw) ? (int)p[j] : VERY_LARGE;
}
template <typename T>
__device__ void load_tile(const void *plane_v, int stride, int pw, int ph, int y0, int x0, int bh, int bw, int16_t *tile) {
    const T *plane = reinterpret_cast<const T *>(plane_v);
    const int gpr = (bw + 9) >> 2, total = (bh + 4) * gpr; // groups per tile row (bw is even)
    for (int i = threadIdx.x; i < total; i += 2 * NT) {
        int v[2][4], r[2], g[2];
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const int ii = i + u * NT;
            r[u] = ii / gpr;
            g[u] = ii - r[u] * gpr;
            if (ii < total) load_group<T>(plane, stride, pw, ph, y0 + r[u] - 2, x0 - 4 + 4 * g[u], v[u]);
        }
#pragma unroll
        for (int u = 0; u < 2; u++) {
            if (i + u * NT >= total) continue;
            const int c0 = 4 * g[u] - 2; // tile column of the group's first sample
            uint32_t *row = reinterpret_cast<uint32_t *>(tile + r[u] * TS);
            if (c0 >= 0 && c0 + 1 < bw + 4) row[c0 >> 1] = (uint32_t)(uint16_t)v[u][0] | ((uint32_t)(uint16_t)v[u][1] << 16);
            if (c0 + 3 < bw + 4) row[(c0 + 2) >> 1] = (uint32_t)(uint16_t)v[u][2] | ((uint32_t)(uint16_t)v[u][3] << 16);
        }
    }
}

// 64x64 filter blocks (16x16 4x4 units) per picture column or row of `mi` 4x4 units
static int fb_count(int mi) { return (mi + 15) / 16; }

// One plane's part of a filter block, in samples of that plane
struct PlaneRect {
    int pw, ph; // plane size
    int bh, bw; // block size, clipped to the plane
    int y0, x0; // block origin
};
// The filter block of CTA x index `fb` (raster order, nhfb per row) in a picture of mi_rows x mi_cols 4x4 units
struct FilterBlock {
    int mi_rows, mi_cols;
    int fbr, fbc; // row and column in filter blocks
    int nvb, nhb; // size in 4x4 units, clipped to the picture
    int border; // nonzero when the +2 rim reaches outside the frame (CDEF_VERY_LARGE samples present); an int, as a bool
                // member costs cdef_apply_kernel 8 registers
    __device__ FilterBlock(int fb, int nhfb, int mi_rows_, int mi_cols_) : mi_rows(mi_rows_), mi_cols(mi_cols_) {
        fbr = fb / nhfb;
        fbc = fb - fbr * nhfb;
        nvb = min(16, mi_rows - 16 * fbr);
        nhb = min(16, mi_cols - 16 * fbc);
        border = fbr == 0 || fbc == 0 || 16 * (fbr + 1) >= mi_rows || 16 * (fbc + 1) >= mi_cols;
    }
    __device__ PlaneRect plane(int pli) const {
        const int sh = pli ? 1 : 0;
        return {(mi_cols * 4) >> sh, (mi_rows * 4) >> sh, (nvb * 4) >> sh, (nhb * 4) >> sh, (fbr * 64) >> sh, (fbc * 64) >> sh};
    }
};
// Stage plane `pli` of the filter block from `f` into `tile`, between two barriers: the first one waits until every
// thread is done with the previous plane's tile.
template <typename T>
__device__ __forceinline__ PlaneRect stage_plane(const FilterBlock &fb, const FrameDev &f, int pli, int16_t *tile) {
    const PlaneRect r = fb.plane(pli);
    __syncthreads();
    load_tile<T>(f.p[pli], f.stride[pli], r.pw, r.ph, r.y0, r.x0, r.bh, r.bw, tile);
    __syncthreads();
    return r;
}

// Strengths of the search's separable form (see plane_search_grid): entry gi = pi * NSEC + si is (pri[pi], sec[si])
struct CdefGrid {
    int npri;
    int pri[16], sec[4];
};
struct CdefSearchDev {
    SvtB200CdefSearchParams p;
    CdefGrid g; // read by the grid instances only
    FrameDev recon, source;
    const uint8_t *skip8;
    int skip_stride;
    uint64_t *mse;
    int nvfb, nhfb, coeff_shift;
};

// svt_sb_compute_cdef_list: raster list of the filter block's non-skip 8x8 blocks into s_by, s_bx (warp 0, two blocks per
// lane, ballots).  Ends with a barrier and returns the count to every thread.
__device__ __forceinline__ int block_list(const FilterBlock &fb, const uint8_t *skip8, int skip_stride, uint8_t *s_by, uint8_t *s_bx) {
    __shared__ int s_count;
    const int tid = threadIdx.x;
    if (tid < 32) {
        unsigned int m[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int b = tid + 32 * h, r = (b >> 3) * 2, c = (b & 7) * 2;
            const bool on = r < fb.nvb && c < fb.nhb && !skip8[(size_t)((16 * fb.fbr + r) >> 1) * skip_stride + ((16 * fb.fbc + c) >> 1)];
            m[h] = __ballot_sync(0xffffffffu, on);
        }
#pragma unroll
        for (int h = 0; h < 2; h++)
            if ((m[h] >> tid) & 1u) {
                const int n = (h ? __popc(m[0]) : 0) + __popc(m[h] & ((1u << tid) - 1u));
                s_by[n] = (uint8_t)((tid + 32 * h) >> 3);
                s_bx[n] = (uint8_t)(tid & 7);
            }
        if (tid == 0) s_count = __popc(m[0]) + __popc(m[1]);
    }
    __syncthreads();
    return s_count;
}

// Write plane `pli`'s 64 entries of this filter block's mse row from the sums in s_mse, and clear s_mse for the next plane.
// The two chroma planes share a row.  Entries past n_strengths, and every entry of an all-skip filter block (count 0,
// svt_sb_all_skip: not searched), are 0.
__device__ __forceinline__ void store_mse(const CdefSearchDev &d, int pli, int count, unsigned long long *s_mse) {
    uint64_t *out = d.mse + ((pli ? (size_t)d.nvfb * d.nhfb : 0) + blockIdx.x) * 64;
    for (int gi = threadIdx.x; gi < 64; gi += NT) {
        unsigned long long v = 0;
        if (count && gi < d.p.n_strengths) v = s_mse[gi] >> (2 * d.coeff_shift);
        s_mse[gi] = 0;
        if (pli == 2)
            out[gi] += v;
        else
            out[gi] = v;
    }
}

// dist_8x8_8bit_c / dist_8x8_16bit_c (EbEncCdef.c:20-33, 75-98): identical IEEE double operation sequence
__device__ __forceinline__ unsigned long long dist8x8_from_sums(unsigned long long sum_s, unsigned long long sum_d,
                                                                unsigned long long sum_s2, unsigned long long sum_d2,
                                                                unsigned long long sum_sd, int coeff_shift) {
    const unsigned long long svar = sum_s2 - ((sum_s * sum_s + 32) >> 6);
    const unsigned long long dvar = sum_d2 - ((sum_d * sum_d + 32) >> 6);
    const double a = __dmul_rn((double)(sum_d2 + sum_s2 - 2 * sum_sd), .5);
    const double b = __dmul_rn(a, (double)(svar + dvar + (unsigned long long)(400 << 2 * coeff_shift)));
    const double c = __dsqrt_rn(__dadd_rn((double)(20000 << 4 * coeff_shift), __dmul_rn((double)svar, (double)dvar)));
    return (unsigned long long)floor(__dadd_rn(.5, __ddiv_rn(b, c)));
}

// ---- search, list form --------------------------------------------------------------------------------------------
// Any strength list: one pass over the listed blocks per strength.  A thread owns one row of one 8x8 (or 4x4 chroma) block.
template <typename T>
__device__ __forceinline__ int ldpx(const void *p, size_t off) {
    return reinterpret_cast<const T *>(p)[off];
}
template <typename T>
__device__ __forceinline__ void plane_search_list(const CdefSearchDev &d, const int16_t *in, int count, const uint8_t *s_by,
                                                  const uint8_t *s_bx, const int8_t *s_dir, const int *s_var, unsigned long long *s_mse,
                                                  int pli, int y0, int x0, int damping, bool border) {
    const int tid = threadIdx.x, bs = pli ? 4 : 8, cs = d.coeff_shift;
    const SvtB200CdefSearchParams &p = d.p;
    const int rows_per_blk = bs; // threads per block = rows
    const int blk_per_pass = NT / rows_per_blk;
    const void *sp = d.source.p[pli];
    const int sstride = d.source.stride[pli];
    for (int gi = 0; gi < p.n_strengths; gi++) {
        const int pri = p.pri_strength[gi] << cs, sec = p.sec_strength[gi] << cs;
        unsigned long long acc = 0;
        for (int b0 = 0; b0 < count; b0 += blk_per_pass) {
            const int b = b0 + tid / rows_per_blk, row = tid % rows_per_blk;
            const bool live = b < count;
            unsigned int ss = 0, sd = 0, ss2 = 0, sd2 = 0, ssd = 0, se = 0;
            if (live) {
                const int by = s_by[b], bx = s_bx[b];
                const int t = pli ? pri : adjust_strength(pri, s_var[b]);
                const int dir = pri ? s_dir[b] : 0;
                const int16_t *q = in + (by * bs + row) * TS + bx * bs;
                const size_t so = (size_t)(y0 + by * bs + row) * sstride + x0 + bx * bs;
                const bool ident = t == 0 && sec == 0;
                const CdefTaps taps = make_taps(t, sec, dir, damping, damping, cs, TS);
                for (int j = 0; j < bs; j++) {
                    const int f = ident ? (int)q[j] : (border ? cdef_px<true>(q + j, taps, t, sec) : cdef_px<false>(q + j, taps, t, sec));
                    const int o = ldpx<T>(sp, so + j);
                    if (pli == 0) {
                        ss += f;
                        sd += o;
                        ss2 += f * f;
                        sd2 += o * o;
                        ssd += f * o;
                    } else {
                        se += (o - f) * (o - f);
                    }
                }
            }
            if (pli == 0) { // 8 lanes = one 8x8 block
#pragma unroll
                for (int o = 1; o < 8; o <<= 1) {
                    ss += __shfl_xor_sync(0xffffffffu, ss, o);
                    sd += __shfl_xor_sync(0xffffffffu, sd, o);
                    ss2 += __shfl_xor_sync(0xffffffffu, ss2, o);
                    sd2 += __shfl_xor_sync(0xffffffffu, sd2, o);
                    ssd += __shfl_xor_sync(0xffffffffu, ssd, o);
                }
                if (live && row == 0) acc += dist8x8_from_sums(ss, sd, ss2, sd2, ssd, cs);
            } else {
                acc += se;
            }
        }
        // CTA-wide sum of this strength
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if ((tid & 31) == 0 && acc) atomicAdd(&s_mse[gi], acc);
    }
}

// ---- search, separable form ---------------------------------------------------------------------------------------
// Every strength table the encoder uses (get_cdef_filter_strengths) is a GRID: gi = pi * nsec + si.  The filter sum
// of cdef_filter_block is P(pri) + S(sec) with P over the 4 primary taps and S over the 8 secondary taps, and the
// clamp range [min, max] depends on the tap set only, so per pixel the search needs S and min/max once per
// direction set (direction 0 for the pri == 0 entries — `t ? dir : 0` in svt_cdef_filter_fb — and the block's
// direction for the rest) and P once per primary strength: for the 5x2 table of preset 8 that is 32 constrain()
// evaluations per pixel instead of 72, 24 tile loads instead of 108.
constexpr int CDEF_COMPACT_NG = 20; // strength tables up to this size park the per-block sums for a compact distortion pass
// Not inlined, and the grid instances of the search kernel are built for 4 resident CTAs per SM: a force-inlined
// plane_search_grid and (256,3) / (256,2) launch bounds remove most of the stack frame but were slower when measured - the
// kernel lives on 4 resident CTAs per SM hiding the constrain() ALU chains.
template <typename T, int BS, int NSEC, bool LUMA, bool kBorder>
__device__ __noinline__ void plane_search_grid(const CdefSearchDev &d, const CdefGrid &g, const int16_t *in, int count,
                                               const uint8_t *s_by, const uint8_t *s_bx, const int8_t *s_dir, const int *s_var,
                                               unsigned long long *s_mse, uint32_t *s_sums, int pli, int y0, int x0, int damping) {
    const int tid = threadIdx.x, lane = tid & 31;
    const int ng = g.npri * NSEC;
    // The 8x8 luma distortion is ~100 double-precision instructions evaluated by ONE lane per block: inside the strength
    // loop it is issued for 2 active lanes per warp.  With a small table the three sums per (block, strength) are parked
    // in shared memory and evaluated afterwards with all lanes busy (one (strength, block) pair per thread).
    const bool compact = LUMA && ng <= CDEF_COMPACT_NG;
    const int cs = d.coeff_shift;
    const T *sp = reinterpret_cast<const T *>(d.source.p[pli]);
    const int sstride = d.source.stride[pli];
    constexpr int PX = 4; // samples per thread: a quarter (chroma: a whole) block row
    constexpr int TPB = BS * BS / PX; // threads per block: 16 (luma 8x8) or 4 (chroma 4x4)
    constexpr int BPP = NT / TPB; // blocks per pass
    for (int b0 = 0; b0 < count; b0 += BPP) {
        if (b0 + (tid & ~31) / TPB >= count) continue; // whole warp idle (shuffles below are per warp)
        const int b = b0 + tid / TPB, sub = tid % TPB;
        const int row = sub / (BS / PX), col = (sub % (BS / PX)) * PX;
        const bool live = b < count;
        const int bb = live ? b : 0;
        const int by = s_by[bb], bx = s_bx[bb];
        const int16_t *q = in + (by * BS + row) * TS + bx * BS + col;
        const T *so = sp + (size_t)(y0 + by * BS + row) * sstride + x0 + bx * BS + col;
        const int bdir = s_dir[bb], var = s_var[bb];
        int x[PX], o[PX], mn[PX], mx[PX], S[PX][NSEC];
        unsigned int sd = 0, sd2 = 0;
#pragma unroll
        for (int j = 0; j < PX; j++) {
            x[j] = q[j];
            o[j] = (int)so[j];
            if (LUMA) {
                sd += o[j];
                sd2 += o[j] * o[j];
            }
        }
        if (LUMA) {
#pragma unroll
            for (int s = 1; s < TPB; s <<= 1) {
                sd += __shfl_xor_sync(0xffffffffu, sd, s);
                sd2 += __shfl_xor_sync(0xffffffffu, sd2, s);
            }
        }
        int have = -1; // direction set S/mn/mx currently hold: 0 = direction 0, 1 = block direction
        for (int pi = 0; pi < g.npri; pi++) {
            const int pri = g.pri[pi] << cs;
            const int want = pri ? 1 : 0;
            const int dir = pri ? bdir : 0;
            if (want != have) { // uniform over the CTA
                have = want;
                int o2[2], o6[2], po[2];
                tap_offsets(dir, TS, po, o2, o6);
#pragma unroll
                for (int j = 0; j < PX; j++) {
                    int tp[12];
#pragma unroll
                    for (int k = 0; k < 2; k++) {
                        tp[4 * k + 0] = q[j + o2[k]], tp[4 * k + 1] = q[j - o2[k]];
                        tp[4 * k + 2] = q[j + o6[k]], tp[4 * k + 3] = q[j - o6[k]];
                        tp[8 + 2 * k] = q[j + po[k]], tp[9 + 2 * k] = q[j - po[k]];
                    }
                    int lo = x[j], hi = x[j];
#pragma unroll
                    for (int i = 0; i < 12; i++) {
                        lo = min(lo, tp[i]);
                        hi = (kBorder && tp[i] == VERY_LARGE) ? hi : max(hi, tp[i]);
                    }
                    mn[j] = lo;
                    mx[j] = hi;
#pragma unroll
                    for (int si = 0; si < NSEC; si++) {
                        const int sec = g.sec[si] << cs;
                        int acc = 0;
                        if (sec) {
                            const int ssh = max(0, damping - msb((uint32_t)sec));
#pragma unroll
                            for (int k = 0; k < 2; k++) {
                                const int w = k ? 1 : 2;
                                acc += w * (constrain_s(tp[4 * k] - x[j], sec, ssh) + constrain_s(tp[4 * k + 1] - x[j], sec, ssh) +
                                            constrain_s(tp[4 * k + 2] - x[j], sec, ssh) + constrain_s(tp[4 * k + 3] - x[j], sec, ssh));
                            }
                        }
                        S[j][si] = acc;
                    }
                }
            }
            const int t = LUMA ? adjust_strength(pri, var) : pri;
            const int odd = (t >> cs) & 1;
            const int pt0 = odd ? 3 : 4, pt1 = odd ? 3 : 2;
            const int psh = t ? max(0, damping - msb((uint32_t)t)) : 0;
            const int po0 = c_dir[dir][0][0] * TS + c_dir[dir][0][1], po1 = c_dir[dir][1][0] * TS + c_dir[dir][1][1];
            unsigned int ss[NSEC], ss2[NSEC], ssd[NSEC];
#pragma unroll
            for (int si = 0; si < NSEC; si++) ss[si] = ss2[si] = ssd[si] = 0;
#pragma unroll
            for (int j = 0; j < PX; j++) {
                int P = 0;
                if (t) {
                    P = pt0 * (constrain_s(q[j + po0] - x[j], t, psh) + constrain_s(q[j - po0] - x[j], t, psh)) +
                        pt1 * (constrain_s(q[j + po1] - x[j], t, psh) + constrain_s(q[j - po1] - x[j], t, psh));
                }
#pragma unroll
                for (int si = 0; si < NSEC; si++) {
                    const int sum = P + S[j][si];
                    const int y = x[j] + ((8 + sum - (sum < 0)) >> 4);
                    const int f = min(max(y, mn[j]), mx[j]);
                    if (LUMA) {
                        ss[si] += f;
                        ss2[si] += f * f;
                        ssd[si] += f * o[j];
                    } else {
                        ss[si] += (o[j] - f) * (o[j] - f);
                    }
                }
            }
#pragma unroll
            for (int si = 0; si < NSEC; si++) {
                unsigned long long v;
                if (LUMA) { // 16 lanes = one 8x8 block
#pragma unroll
                    for (int s = 1; s < TPB; s <<= 1) {
                        ss[si] += __shfl_xor_sync(0xffffffffu, ss[si], s);
                        ss2[si] += __shfl_xor_sync(0xffffffffu, ss2[si], s);
                        ssd[si] += __shfl_xor_sync(0xffffffffu, ssd[si], s);
                    }
                    if (compact) {
                        if (live && sub == 0) {
                            uint32_t *e = s_sums + (b * CDEF_COMPACT_NG + pi * NSEC + si) * 3;
                            e[0] = ss[si], e[1] = ss2[si], e[2] = ssd[si];
                            if (pi == 0 && si == 0) {
                                s_sums[64 * CDEF_COMPACT_NG * 3 + 2 * b] = sd;
                                s_sums[64 * CDEF_COMPACT_NG * 3 + 2 * b + 1] = sd2;
                            }
                        }
                        continue;
                    }
                    v = (live && sub == 0) ? dist8x8_from_sums(ss[si], sd, ss2[si], sd2, ssd[si], cs) : 0ull;
                    v += __shfl_xor_sync(0xffffffffu, v, 16);
                } else {
                    v = live ? ss[si] : 0u;
#pragma unroll
                    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
                }
                if (lane == 0 && v) atomicAdd(&s_mse[pi * NSEC + si], v);
            }
        }
    }
    if (compact) { // item = strength * 64 + block: a warp works for one strength
        __syncthreads();
        for (int it = tid; it < ng * 64; it += NT) {
            const int gi = it >> 6, b = it & 63;
            unsigned long long v = 0;
            if (b < count) {
                const uint32_t *e = s_sums + (b * CDEF_COMPACT_NG + gi) * 3;
                v = dist8x8_from_sums(e[0], s_sums[64 * CDEF_COMPACT_NG * 3 + 2 * b], e[1], s_sums[64 * CDEF_COMPACT_NG * 3 + 2 * b + 1], e[2], cs);
            }
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
            if (lane == 0 && v) atomicAdd(&s_mse[gi], v);
        }
    }
}

// NSEC = 2, 4: a grid table (plane_search_grid); NSEC = 0: any strength list (plane_search_list).
// grid.y = 2: CTA (fb, 0) searches the luma plane, CTA (fb, 1) both chroma planes (it stages the luma tile once more for
// the block directions).  One CTA per filter block was 510 CTAs = 0.86 waves at 1080p (ncu launch__waves_per_multiprocessor)
// with every CTA a serial chain over three planes; split, the grid is 1020 CTAs of 2/3 and 1/3 of that chain.
template <typename T, int NSEC>
__global__ void __launch_bounds__(NT, 4) cdef_search_kernel(const __grid_constant__ CdefSearchDev d) {
    __shared__ int16_t tile[68 * TS];
    __shared__ uint8_t s_by[64], s_bx[64];
    __shared__ int8_t s_dir[64];
    __shared__ int s_var[64];
    __shared__ unsigned long long s_mse[64];
    __shared__ uint32_t s_sums[NSEC ? 64 * CDEF_COMPACT_NG * 3 + 128 : 1]; // parked (sum f, sum f^2, sum f*o) per (block, strength) + (sum o, sum o^2)
    const FilterBlock fb(blockIdx.x, d.nhfb, d.p.mi_rows, d.p.mi_cols);
    const bool chroma_cta = blockIdx.y != 0;
    const int cs = d.coeff_shift;
    for (int i = threadIdx.x; i < 64; i += NT) s_mse[i] = 0;
    const int count = block_list(fb, d.skip8, d.skip_stride, s_by, s_bx);
    if (count == 0) {
        store_mse(d, chroma_cta ? 1 : 0, 0, s_mse);
        return;
    }
    for (int pli = 0; pli < (chroma_cta ? 3 : 1); pli++) {
        const PlaneRect r = stage_plane<T>(fb, d.recon, pli, tile);
        const int16_t *in = tile + 2 * TS + 2;
        if (pli == 0) {
            find_dirs(in, s_by, s_bx, count, cs, s_dir, s_var);
            __syncthreads();
            if (chroma_cta) continue; // directions only
        }
        const int damping = d.p.pri_damping + cs - (pli != 0);
        if constexpr (NSEC == 0) {
            plane_search_list<T>(d, in, count, s_by, s_bx, s_dir, s_var, s_mse, pli, r.y0, r.x0, damping, fb.border);
        } else if (pli == 0) {
            if (fb.border)
                plane_search_grid<T, 8, NSEC, true, true>(d, d.g, in, count, s_by, s_bx, s_dir, s_var, s_mse, s_sums, pli, r.y0, r.x0, damping);
            else
                plane_search_grid<T, 8, NSEC, true, false>(d, d.g, in, count, s_by, s_bx, s_dir, s_var, s_mse, s_sums, pli, r.y0, r.x0, damping);
        } else {
            if (fb.border)
                plane_search_grid<T, 4, NSEC, false, true>(d, d.g, in, count, s_by, s_bx, s_dir, s_var, s_mse, s_sums, pli, r.y0, r.x0, damping);
            else
                plane_search_grid<T, 4, NSEC, false, false>(d, d.g, in, count, s_by, s_bx, s_dir, s_var, s_mse, s_sums, pli, r.y0, r.x0, damping);
        }
        __syncthreads();
        store_mse(d, pli, count, s_mse);
    }
}

struct CdefApplyDev {
    const SvtB200CdefDecision *dec; // null: strengths from p (host); else from the device decision of cdef_decide_kernel
    SvtB200CdefApplyParams p;
    FrameDev recon, out;
    const uint8_t *skip8;
    int skip_stride;
    const int8_t *fb_idx;
    int nvfb, nhfb, coeff_shift;
};

// A signalled strength, pri * 4 + sec with sec 3 standing for 4, as the filter's (pri, sec)
__device__ __forceinline__ int2 decode_strength(int s) {
    const int sec = s % 4;
    return make_int2(s / 4, sec + (sec == 3));
}

// Tried: one CTA per 32x32 QUADRANT of the filter block (4x the CTAs, a quarter of the serial chain each): bit-exact but
// slower at 1080p and at 2160p 10-bit: the rim samples and the per-quadrant set-up cost more than the shorter chain saves - the kernel is throughput
// bound (12 taps x constrain() per sample), not latency bound.  One CTA per filter block kept.
template <typename T>
__global__ void __launch_bounds__(NT) cdef_apply_kernel(const __grid_constant__ CdefApplyDev d) {
    __shared__ int16_t tile[68 * TS];
    __shared__ uint8_t s_skip[64];
    __shared__ int8_t s_dir[64];
    __shared__ int s_var[64];
    __shared__ int s_any;
    const int tid = threadIdx.x;
    const SvtB200CdefApplyParams &p = d.p;
    const FilterBlock fb(blockIdx.x, d.nhfb, p.mi_rows, p.mi_cols);
    const int cs = d.coeff_shift;
    const bool border = fb.border; // read once here: read from fb in the sample loop, the kernel takes 8 more registers
    const int idx = d.fb_idx[blockIdx.x];
    int2 y = make_int2(0, 0), uv = make_int2(0, 0); // (primary, secondary) strength of luma and of chroma
    if (idx >= 0) {
        y = decode_strength(d.dec ? d.dec->y_strength[idx] : p.y_strength[idx]);
        uv = decode_strength(d.dec ? d.dec->uv_strength[idx] : p.uv_strength[idx]);
    }
    const bool fb_on = idx >= 0 && !(y.x == 0 && y.y == 0 && uv.x == 0 && uv.y == 0);
    if (tid == 0) s_any = 0;
    __syncthreads();
    if (tid < 64) {
        const int by = tid >> 3, bx = tid & 7;
        int sk = 1;
        if (fb_on && 2 * by < fb.nvb && 2 * bx < fb.nhb)
            sk = d.skip8[(size_t)((16 * fb.fbr + 2 * by) >> 1) * d.skip_stride + ((16 * fb.fbc + 2 * bx) >> 1)];
        s_skip[tid] = (uint8_t)sk;
        if (!sk) s_any = 1;
    }
    __syncthreads();
    const bool filt = fb_on && s_any;
    for (int pli = 0; pli < 3; pli++) {
        const int sh = pli ? 1 : 0;
        const PlaneRect rect = stage_plane<T>(fb, d.recon, pli, tile);
        const int16_t *in = tile + 2 * TS + 2;
        if (pli == 0 && filt) {
            for (int b0 = 0; b0 < 64; b0 += NT / 8) { // eight lanes per block; skipped blocks are computed and dropped
                const int b = b0 + (tid >> 3);
                int v;
                const int dir = find_dir8(in + 8 * (b >> 3) * TS + 8 * (b & 7), TS, &v, cs);
                if (!s_skip[b] && (tid & 7) == 0) {
                    s_dir[b] = (int8_t)dir;
                    s_var[b] = v;
                }
            }
            __syncthreads();
        }
        const int pri = (pli ? uv.x : y.x) << cs, s2 = (pli ? uv.y : y.y) << cs;
        const int damping = p.damping + cs - (pli != 0);
        T *op = reinterpret_cast<T *>(const_cast<void *>(d.out.p[pli]));
        const int ostride = d.out.stride[pli];
        // four samples of one block row per thread: direction, strengths, tap offsets and shifts are per-block values
        const int q4 = rect.bw >> 2;
        for (int i = tid; i < rect.bh * q4; i += NT) {
            const int r = i / q4, c = (i - r * q4) << 2;
            const int b = (r >> (3 - sh)) * 8 + (c >> (3 - sh));
            const int16_t *q = in + r * TS + c;
            int o[4] = {q[0], q[1], q[2], q[3]};
            if (filt && !s_skip[b]) {
                const int t = pli ? pri : adjust_strength(pri, s_var[b]);
                if (t | s2) {
                    const CdefTaps taps = make_taps(t, s2, pri ? s_dir[b] : 0, damping, damping, cs, TS);
#pragma unroll
                    for (int j = 0; j < 4; j++) o[j] = border ? cdef_px<true>(q + j, taps, t, s2) : cdef_px<false>(q + j, taps, t, s2);
                }
            }
            T *dst = op + (size_t)(rect.y0 + r) * ostride + rect.x0 + c;
            if (sizeof(T) == 1 && ((uintptr_t)dst & 3) == 0)
                *reinterpret_cast<uint32_t *>(dst) = (uint32_t)o[0] | ((uint32_t)o[1] << 8) | ((uint32_t)o[2] << 16) | ((uint32_t)o[3] << 24);
            else if (sizeof(T) == 2 && ((uintptr_t)dst & 7) == 0)
                *reinterpret_cast<uint2 *>(dst) = make_uint2((uint32_t)o[0] | ((uint32_t)o[1] << 16), (uint32_t)o[2] | ((uint32_t)o[3] << 16));
            else {
#pragma unroll
                for (int j = 0; j < 4; j++) dst[j] = (T)o[j];
            }
        }
    }
}

// drop-in kernels ----------------------------------------------------------------------------------------
__global__ void find_dir_kernel(const uint16_t *img, int stride, int coeff_shift, int *out) {
    __shared__ int16_t t[64];
    for (int i = threadIdx.x; i < 64; i += blockDim.x) t[i] = (int16_t)img[(i >> 3) * stride + (i & 7)];
    __syncthreads();
    int v;
    const int dir = find_dir8(t, 8, &v, coeff_shift); // one warp = four redundant groups of eight lanes
    if (threadIdx.x == 0) {
        out[0] = dir;
        out[1] = v;
    }
}
// in: 12x12 uint16 window (2 rim) of the block, out: 8x8 ints
__global__ void filter_block_kernel(const uint16_t *win, int pri, int sec, int dir, int pd, int sd, int rows, int cols,
                                    int coeff_shift, uint16_t *out) {
    __shared__ int16_t t[12 * 12];
    for (int i = threadIdx.x; i < 144; i += blockDim.x) t[i] = (int16_t)win[i];
    __syncthreads();
    const int i = threadIdx.x >> 3, j = threadIdx.x & 7;
    if (i < rows && j < cols) {
        const CdefTaps taps = make_taps(pri, sec, dir, pd, sd, coeff_shift, 12);
        out[i * 8 + j] = (uint16_t)cdef_px<true>(t + (i + 2) * 12 + j + 2, taps, pri, sec);
    }
}

static int frame_dev(const SvtB200Frame *f, FrameDev *o) {
    if (!f || !f->y || !f->cb || !f->cr || (f->bit_depth != 8 && f->bit_depth != 10 && f->bit_depth != 12)) return -1;
    o->p[0] = f->y;
    o->p[1] = f->cb;
    o->p[2] = f->cr;
    o->stride[0] = f->stride_y;
    o->stride[1] = o->stride[2] = f->stride_c;
    o->hbd = f->bit_depth > 8;
    return 0;
}

// compute_cdef_dist_c / compute_cdef_dist_8bit_c (EbEncCdef.c:134-220) on packed blocks: thread = one block
__global__ void cdef_dist_kernel(const uint16_t *dst, const uint16_t *src, int count, int bw, int bh, int luma8x8, int coeff_shift,
                                 unsigned long long *out) {
    unsigned long long acc = 0;
    for (int b = threadIdx.x; b < count; b += blockDim.x) {
        const uint16_t *d = dst + b * bw * bh, *s = src + b * bw * bh;
        if (luma8x8) {
            unsigned long long ss = 0, sd = 0, ss2 = 0, sd2 = 0, ssd = 0;
            for (int i = 0; i < 64; i++) {
                const unsigned long long sv = s[i], dv = d[i];
                ss += sv, sd += dv, ss2 += sv * sv, sd2 += dv * dv, ssd += sv * dv;
            }
            acc += dist8x8_from_sums(ss, sd, ss2, sd2, ssd, coeff_shift);
        } else {
            for (int i = 0; i < bw * bh; i++) {
                const int e = (int)d[i] - (int)s[i];
                acc += (unsigned long long)(e * e);
            }
        }
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}

struct CdefListView { // CdefList (Common/Codec/EbCdef.h): uint8_t by, bx, skip
    uint8_t by, bx, skip;
};
uint64_t cdef_dist_dropin(const void *dst, int hbd, int dstride, const void *src, const void *dlist_v, int count, int bsize,
                          int coeff_shift, int pli) {
    if (count <= 0) return 0;
    const CdefListView *dl = (const CdefListView *)dlist_v;
    // BlockSize: BLOCK_4X4 0, BLOCK_4X8 1, BLOCK_8X4 2, BLOCK_8X8 3
    const int bw = (bsize == 3 || bsize == 2) ? 8 : 4, bh = (bsize == 3 || bsize == 1) ? 8 : 4, n = bw * bh;
    Staging s({(size_t)count * n * 2, (size_t)count * n * 2, 8});
    SVTB_CUDA_FATAL(s.status());
    uint16_t *hd = s.h<uint16_t>(0), *hs = s.h<uint16_t>(1);
    for (int b = 0; b < count; b++) {
        const int y0 = dl[b].by * bh, x0 = dl[b].bx * bw;
        for (int i = 0; i < bh; i++)
            for (int j = 0; j < bw; j++) {
                const size_t o = (size_t)(y0 + i) * dstride + x0 + j;
                hd[b * n + i * bw + j] = hbd ? ((const uint16_t *)dst)[o] : ((const uint8_t *)dst)[o];
                hs[b * n + i * bw + j] = hbd ? ((const uint16_t *)src)[b * n + i * bw + j] : ((const uint8_t *)src)[b * n + i * bw + j];
            }
    }
    SVTB_CUDA_FATAL(s.upload(0, 1));
    SVTB_CUDA_FATAL(cudaMemsetAsync(s.d(2), 0, 8, s.stream()));
    SVTB_LAUNCH(cdef_dist_kernel, 1, 64, 0, s.stream(), s.d<const uint16_t>(0), s.d<const uint16_t>(1), count, bw, bh,
                (int)(bsize == 3 && pli == 0), coeff_shift, s.d<unsigned long long>(2));
    SVTB_CUDA_FATAL(s.download(2, 2));
    return *s.h<unsigned long long>(2) >> (2 * coeff_shift);
}

__global__ void copy_rect8_kernel(uint16_t *dst, const uint8_t *src, int n) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = src[i];
}
} // namespace

// ---- the strength decision on the device: finish_cdef_search (EbEncCdef.c:1167-1340) --------------------------------
// One CTA of 1024 threads.  svt_search_one_dual_c adds, to the nb already chosen (luma, chroma) pairs, the pair (j, k) that
// minimises the sum over filter blocks of min(best so far, mse0[j] + mse1[k]); the n x n candidate pairs are the threads
// (pairs x block slices when n^2 < 1024), the per-block "best so far" is one pass over the blocks, the argmin is the first
// minimum in (j outer, k inner) order = the smallest (sum, j * n + k).  joint_strength_search_dual calls it 5 n times per
// number of sets n = 1, 2, 4, 8.  uint64 sums only: exact whatever the order.
struct DecideDev {
    SvtB200CdefDecideParams p;
    const unsigned long long *mse0, *mse1;
    const uint8_t *skip8;
    int skip_stride, nvfb, nhfb, rows8, cols8;
    SvtB200CdefDecision *out;
    int8_t *fb_idx;
    int *sb_list;               // [nfb]
    unsigned long long *best_sb; // [nfb]
    unsigned long long *c0, *c1; // [sb_count][n]: the searched strengths of the participating blocks, dense (L1-resident at 1080p)
};

__device__ __forceinline__ void lex_min(unsigned long long &v, int &i, unsigned long long ov, int oi) {
    if (ov < v || (ov == v && oi < i)) v = ov, i = oi;
}

__global__ void __launch_bounds__(1024) cdef_decide_kernel(const DecideDev d) {
    __shared__ int s_count, s_lev0[8], s_lev1[8], s_best_idx;
    __shared__ unsigned long long s_part[1024], s_best_val, s_rv[32];
    __shared__ int s_ri[32];
    const int tid = threadIdx.x, nfb = d.nvfb * d.nhfb, n = d.p.n_strengths, P = n * n;
    if (tid == 0) s_count = 0;
    __syncthreads();
    for (int fb = tid; fb < nfb; fb += 1024) {
        const int fbr = fb / d.nhfb, fbc = fb - fbr * d.nhfb;
        int all_skip = 1;
        for (int r = 8 * fbr; r < min(8 * fbr + 8, d.rows8) && all_skip; r++)
            for (int c = 8 * fbc; c < min(8 * fbc + 8, d.cols8); c++)
                if (!d.skip8[(size_t)r * d.skip_stride + c]) {
                    all_skip = 0;
                    break;
                }
        d.fb_idx[fb] = -1;
        if (!all_skip) d.sb_list[atomicAdd(&s_count, 1)] = fb;
    }
    __syncthreads();
    const int sb_count = s_count;
    // the 64-entry rows of the search output hold n <= 64 used entries: copy them densely once (the 75 search steps below
    // re-read the table; 82 KB instead of 522 KB at 1080p with the 10-strength table)
    for (int idx = tid; idx < sb_count * n; idx += 1024) {
        const int i = idx / n, st = idx - i * n;
        d.c0[idx] = d.mse0[(size_t)d.sb_list[i] * 64 + st];
        d.c1[idx] = d.mse1[(size_t)d.sb_list[i] * 64 + st];
    }
    __syncthreads();
    // pairs per pass and block slices: PP pair slots (a multiple of 32), G = 1024 / PP slices of the block list
    const int PP = min(1024, (P + 31) & ~31), G = 1024 / PP;
    const int slot = tid % PP, slice = tid / PP;

    auto search_one = [&](int nb) -> unsigned long long {
        for (int i = tid; i < sb_count; i += 1024) {
            const unsigned long long *m0 = d.c0 + (size_t)i * n, *m1 = d.c1 + (size_t)i * n;
            unsigned long long best = 1ull << 63;
            for (int g = 0; g < nb; g++) best = min(best, m0[s_lev0[g]] + m1[s_lev1[g]]);
            d.best_sb[i] = best;
        }
        __syncthreads();
        unsigned long long bv = ~0ull;
        int bi = 0x7fffffff;
        for (int p0 = 0; p0 < P; p0 += PP) { // one pass unless n^2 > 1024 (the 64-entry table)
            const int pr = p0 + slot;
            unsigned long long acc = 0;
            if (pr < P && slice < G) {
                const int j = pr / n, k = pr - j * n;
                const unsigned long long *q0 = d.c0 + j, *q1 = d.c1 + k;
                int i = slice;
                unsigned long long a0 = 0, a1 = 0, a2 = 0, a3 = 0; // four independent chains: the loop is latency bound
                for (; i + 3 * G < sb_count; i += 4 * G) {
                    const size_t o0 = (size_t)i * n, o1 = (size_t)(i + G) * n, o2 = (size_t)(i + 2 * G) * n, o3 = (size_t)(i + 3 * G) * n;
                    a0 += min(d.best_sb[i], q0[o0] + q1[o0]);
                    a1 += min(d.best_sb[i + G], q0[o1] + q1[o1]);
                    a2 += min(d.best_sb[i + 2 * G], q0[o2] + q1[o2]);
                    a3 += min(d.best_sb[i + 3 * G], q0[o3] + q1[o3]);
                }
                for (; i < sb_count; i += G) a0 += min(d.best_sb[i], q0[(size_t)i * n] + q1[(size_t)i * n]);
                acc = a0 + a1 + a2 + a3;
            }
            s_part[tid] = acc;
            __syncthreads();
            if (tid < PP && p0 + tid < P) {
                unsigned long long t = 0;
                for (int g = 0; g < G; g++) t += s_part[g * PP + tid];
                lex_min(bv, bi, t, p0 + tid);
            }
            __syncthreads();
        }
        for (int o = 16; o > 0; o >>= 1) lex_min(bv, bi, __shfl_xor_sync(0xffffffffu, bv, o), __shfl_xor_sync(0xffffffffu, bi, o));
        if ((tid & 31) == 0) s_rv[tid >> 5] = bv, s_ri[tid >> 5] = bi;
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < 32; w++) lex_min(bv, bi, s_rv[w], s_ri[w]);
            s_lev0[nb] = bi / n;
            s_lev1[nb] = bi - (bi / n) * n;
            s_best_val = bv;
            s_best_idx = bi;
        }
        __syncthreads();
        return s_best_val;
    };

    unsigned long long best_cost = 1ull << 63;
    for (int bits = 0; bits <= 3; bits++) {
        const int ns = 1 << bits;
        unsigned long long tot = 1ull << 63;
        for (int i = 0; i < ns; i++) tot = search_one(i);
        for (int i = 0; i < 4 * ns; i++) {
            if (tid == 0)
                for (int j = 0; j < ns - 1; j++) s_lev0[j] = s_lev0[j + 1], s_lev1[j] = s_lev1[j + 1];
            __syncthreads();
            tot = search_one(ns - 1);
        }
        const long long total_bits = (long long)sb_count * bits + ns * 6 * 2; // CDEF_STRENGTH_BITS = 6
        const unsigned long long rate = (unsigned long long)(total_bits * 512), dist = tot * 16; // av1_cost_literal
        const unsigned long long cost = ((rate * d.p.lambda + 256) >> 9) + dist * 128;          // RDCOST
        if (cost < best_cost) { // the same value in every thread
            best_cost = cost;
            if (tid == 0) {
                d.out->cdef_bits = bits;
                for (int j = 0; j < ns; j++) d.out->y_index[j] = s_lev0[j], d.out->uv_index[j] = s_lev1[j];
            }
        }
        __syncthreads();
    }
    __threadfence_block();
    __syncthreads();
    const int nb = 1 << d.out->cdef_bits;
    for (int i = tid; i < sb_count; i += 1024) {
        const size_t o = (size_t)i * n;
        unsigned long long best = 1ull << 63;
        int bg = 0;
        for (int g = 0; g < nb; g++) {
            const unsigned long long c = d.c0[o + d.out->y_index[g]] + d.c1[o + d.out->uv_index[g]];
            if (c < best) best = c, bg = g;
        }
        d.fb_idx[d.sb_list[i]] = (int8_t)bg;
    }
    if (tid == 0) {
        d.out->nb_cdef_strengths = nb;
        d.out->sb_count = sb_count;
        d.out->reserved = 0;
        for (int j = 0; j < 8; j++) {
            if (j >= nb) d.out->y_index[j] = d.out->uv_index[j] = 0;
            d.out->y_strength[j] = j < nb ? d.p.filter_strength[d.out->y_index[j]] : 0;
            d.out->uv_strength[j] = j < nb ? d.p.filter_strength[d.out->uv_index[j]] : 0;
        }
    }
}

// Every table of get_cdef_filter_strengths is a grid, gi = pi * nsec + si with nsec 2 or 4 and at most 16 primary
// strengths: returns nsec and fills g, or 0 for any other strength list (g zeroed).
static int strength_grid(const SvtB200CdefSearchParams &p, CdefGrid &g) {
    memset(&g, 0, sizeof(g));
    int nsec = 1;
    while (nsec < p.n_strengths && p.pri_strength[nsec] == p.pri_strength[0]) nsec++;
    bool grid = (nsec == 2 || nsec == 4) && p.n_strengths % nsec == 0 && p.n_strengths / nsec <= 16;
    for (int gi = 0; grid && gi < p.n_strengths; gi++)
        grid = p.pri_strength[gi] == p.pri_strength[gi / nsec * nsec] && p.sec_strength[gi] == p.sec_strength[gi % nsec];
    if (!grid) return 0;
    g.npri = p.n_strengths / nsec;
    for (int i = 0; i < g.npri; i++) g.pri[i] = p.pri_strength[i * nsec];
    for (int i = 0; i < nsec; i++) g.sec[i] = p.sec_strength[i];
    return nsec;
}
template <typename T>
static void launch_search(int nsec, const CdefSearchDev &d, cudaStream_t st) {
    const dim3 grid(d.nvfb * d.nhfb, 2);
    if (nsec == 4)
        SVTB_LAUNCH((cdef_search_kernel<T, 4>), grid, NT, 0, st, d);
    else if (nsec == 2)
        SVTB_LAUNCH((cdef_search_kernel<T, 2>), grid, NT, 0, st, d);
    else
        SVTB_LAUNCH((cdef_search_kernel<T, 0>), grid, NT, 0, st, d);
}

// The two apply entries once d holds the strengths (host params, or the device decision): the argument checks, the
// filter-block grid and the launch.  `strengths` is false when the entry was given none.
static int apply_launch(const char *entry, CdefApplyDev &d, bool strengths, const SvtB200Frame *recon, const SvtB200Frame *out,
                        const uint8_t *skip8, int32_t skip_stride, const int8_t *fb_strength_idx, void *stream) {
    if (!strengths || !skip8 || !fb_strength_idx || frame_dev(recon, &d.recon) || frame_dev(out, &d.out) ||
        recon->bit_depth != out->bit_depth || recon->y == out->y) {
        set_error("%s: bad argument (out must not alias recon)", entry);
        return SVT_B200_ERR_ARG;
    }
    d.skip8 = skip8;
    d.skip_stride = skip_stride;
    d.fb_idx = fb_strength_idx;
    d.nvfb = fb_count(d.p.mi_rows);
    d.nhfb = fb_count(d.p.mi_cols);
    d.coeff_shift = recon->bit_depth - 8;
    cudaStream_t st = (cudaStream_t)stream;
    if (d.recon.hbd)
        SVTB_LAUNCH(cdef_apply_kernel<uint16_t>, d.nvfb * d.nhfb, NT, 0, st, d);
    else
        SVTB_LAUNCH(cdef_apply_kernel<uint8_t>, d.nvfb * d.nhfb, NT, 0, st, d);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

extern "C" {

int svt_b200_cdef_strength_table(int pick_method, SvtB200CdefSearchParams *p) {
    // get_cdef_filter_strengths (EbDefinitions.h:1696-1722) + `sec_strength + (sec_strength == 3)` of the callers
    static const int n[4] = {64, 32, 20, 10};
    static const int pri1[8] = {0, 1, 2, 3, 5, 7, 10, 13}, pri2[5] = {0, 2, 4, 8, 14}, sec3[2] = {0, 2};
    if (!p || pick_method < 0 || pick_method > 3) return SVT_B200_ERR_ARG;
    const int tot_sec = pick_method == 3 ? 2 : 4;
    p->n_strengths = n[pick_method];
    for (int gi = 0; gi < p->n_strengths; gi++) {
        const int pi = gi / tot_sec, si = gi % tot_sec;
        const int pri = pick_method == 0 ? pi : pick_method == 1 ? pri1[pi] : pri2[pi];
        const int sec = pick_method == 3 ? sec3[si] : si;
        p->pri_strength[gi] = pri;
        p->sec_strength[gi] = sec + (sec == 3);
    }
    return p->n_strengths;
}

int svt_b200_cdef_search(const SvtB200CdefSearchParams *p, const SvtB200Frame *recon, const SvtB200Frame *source,
                         const uint8_t *skip8, int32_t skip_stride, uint64_t *mse, void *stream) {
    CdefSearchDev d;
    if (!p || !skip8 || !mse || frame_dev(recon, &d.recon) || frame_dev(source, &d.source) ||
        recon->bit_depth != source->bit_depth || p->n_strengths < 1 || p->n_strengths > 64) {
        set_error("svt_b200_cdef_search: bad argument");
        return SVT_B200_ERR_ARG;
    }
    d.p = *p;
    d.skip8 = skip8;
    d.skip_stride = skip_stride;
    d.mse = mse;
    d.nvfb = fb_count(p->mi_rows);
    d.nhfb = fb_count(p->mi_cols);
    d.coeff_shift = recon->bit_depth - 8;
    const int nsec = strength_grid(*p, d.g);
    if (d.recon.hbd)
        launch_search<uint16_t>(nsec, d, (cudaStream_t)stream);
    else
        launch_search<uint8_t>(nsec, d, (cudaStream_t)stream);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

int svt_b200_cdef_apply(const SvtB200CdefApplyParams *p, const SvtB200Frame *recon, const SvtB200Frame *out,
                        const uint8_t *skip8, int32_t skip_stride, const int8_t *fb_strength_idx, void *stream) {
    CdefApplyDev d{};
    if (p) d.p = *p;
    return apply_launch("svt_b200_cdef_apply", d, p != nullptr, recon, out, skip8, skip_stride, fb_strength_idx, stream);
}

int svt_b200_cdef_decide_table(int pick_method, SvtB200CdefDecideParams *p) {
    SvtB200CdefSearchParams sp;
    if (!p) return SVT_B200_ERR_ARG;
    const int n = svt_b200_cdef_strength_table(pick_method, &sp);
    if (n <= 0) return n;
    p->n_strengths = n;
    for (int g = 0; g < n; g++) {
        // STORE_CDEF_FILTER_STRENGTH (EbEncCdef.c:1165): pri * CDEF_SEC_STRENGTHS + sec; the search table stores sec + (sec == 3)
        const int sec = sp.sec_strength[g] == 4 ? 3 : sp.sec_strength[g];
        p->filter_strength[g] = pick_method == 0 ? g : sp.pri_strength[g] * 4 + sec;
    }
    return n;
}

int svt_b200_cdef_decide(const SvtB200CdefDecideParams *p, const uint64_t *mse, const uint8_t *skip8, int32_t skip_stride,
                         SvtB200CdefDecision *out, int8_t *fb_strength_idx, void *scratch, void *stream) {
    if (!p || !mse || !skip8 || !out || !fb_strength_idx || !scratch || p->n_strengths < 1 || p->n_strengths > 64 || p->mi_rows <= 0 ||
        p->mi_cols <= 0) {
        set_error("svt_b200_cdef_decide: bad argument");
        return SVT_B200_ERR_ARG;
    }
    DecideDev d;
    d.p = *p;
    d.nvfb = fb_count(p->mi_rows);
    d.nhfb = fb_count(p->mi_cols);
    const size_t nfb = (size_t)d.nvfb * d.nhfb;
    d.mse0 = reinterpret_cast<const unsigned long long *>(mse);
    d.mse1 = d.mse0 + nfb * 64;
    d.skip8 = skip8;
    d.skip_stride = skip_stride;
    d.rows8 = (p->mi_rows + 1) / 2;
    d.cols8 = (p->mi_cols + 1) / 2;
    d.out = out;
    d.fb_idx = fb_strength_idx;
    d.best_sb = reinterpret_cast<unsigned long long *>(scratch);
    d.c0 = d.best_sb + nfb;
    d.c1 = d.c0 + nfb * p->n_strengths;
    d.sb_list = reinterpret_cast<int *>(d.c1 + nfb * p->n_strengths);
    SVTB_LAUNCH(cdef_decide_kernel, 1, 1024, 0, (cudaStream_t)stream, d);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

int svt_b200_cdef_apply_dev(int32_t mi_rows, int32_t mi_cols, int32_t damping, const SvtB200CdefDecision *decision,
                            const SvtB200Frame *recon, const SvtB200Frame *out, const uint8_t *skip8, int32_t skip_stride,
                            const int8_t *fb_strength_idx, void *stream) {
    CdefApplyDev d{};
    d.p.mi_rows = mi_rows, d.p.mi_cols = mi_cols, d.p.damping = damping;
    d.dec = decision;
    return apply_launch("svt_b200_cdef_apply_dev", d, decision != nullptr, recon, out, skip8, skip_stride, fb_strength_idx, stream);
}

int32_t svt_cdef_find_dir_cuda(const uint16_t *img, int32_t stride, int32_t *var, int32_t coeff_shift) {
    Staging s({128, 8});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, img, stride, 2, 8, 8);
    SVTB_CUDA_FATAL(s.upload(0, 0));
    SVTB_LAUNCH(find_dir_kernel, 1, 32, 0, s.stream(), s.d<const uint16_t>(0), 8, coeff_shift, s.d<int>(1));
    SVTB_CUDA_FATAL(s.download(1, 1));
    *var = s.h<int>(1)[1];
    return s.h<int>(1)[0];
}

void svt_cdef_filter_block_cuda(uint8_t *dst8, uint16_t *dst16, int32_t dstride, const uint16_t *in,
                                int32_t pri_strength, int32_t sec_strength, int32_t dir, int32_t pri_damping,
                                int32_t sec_damping, int32_t bsize, int32_t coeff_shift) {
    const int rows = 4 << (bsize == 3 || bsize == 1), cols = 4 << (bsize == 3 || bsize == 2);
    Staging s({288, 128}); // the 12x12 window around the block, the 8x8 output
    SVTB_CUDA_FATAL(s.status());
    uint16_t *h = s.h<uint16_t>(0);
    for (int i = 0; i < 12; i++)
        for (int j = 0; j < 12; j++) h[i * 12 + j] = (i < rows + 4 && j < cols + 4) ? in[(i - 2) * 144 + (j - 2)] : 0;
    SVTB_CUDA_FATAL(s.upload(0, 0));
    SVTB_LAUNCH(filter_block_kernel, 1, 64, 0, s.stream(), s.d<const uint16_t>(0), pri_strength, sec_strength, dir, pri_damping,
                sec_damping, rows, cols, coeff_shift, s.d<uint16_t>(1));
    SVTB_CUDA_FATAL(s.download(1, 1));
    const uint16_t *o = s.h<uint16_t>(1);
    for (int i = 0; i < rows; i++)
        for (int j = 0; j < cols; j++) {
            if (dst8)
                dst8[i * dstride + j] = (uint8_t)o[i * 8 + j];
            else
                dst16[i * dstride + j] = o[i * 8 + j];
        }
}

uint64_t svt_compute_cdef_dist_16bit_cuda(const uint16_t *dst, int32_t dstride, const uint16_t *src, const void *dlist,
                                          int32_t cdef_count, int32_t bsize, int32_t coeff_shift, int32_t pli) {
    return cdef_dist_dropin(dst, 1, dstride, src, dlist, cdef_count, bsize, coeff_shift, pli);
}
uint64_t svt_compute_cdef_dist_8bit_cuda(const uint8_t *dst8, int32_t dstride, const uint8_t *src8, const void *dlist,
                                         int32_t cdef_count, int32_t bsize, int32_t coeff_shift, int32_t pli) {
    return cdef_dist_dropin(dst8, 0, dstride, src8, dlist, cdef_count, bsize, coeff_shift, pli);
}

void svt_copy_rect8_8bit_to_16bit_cuda(uint16_t *dst, int32_t dstride, const uint8_t *src, int32_t sstride, int32_t v, int32_t h) {
    if (v <= 0 || h <= 0) return;
    const size_t n = (size_t)v * h;
    Staging s({n, 2 * n});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, src, sstride, 1, h, v);
    SVTB_CUDA_FATAL(s.upload(0, 0));
    SVTB_LAUNCH(copy_rect8_kernel, (int)std::min<size_t>(64, (n + 255) / 256), 256, 0, s.stream(), s.d<uint16_t>(1), s.d<const uint8_t>(0), (int)n);
    SVTB_CUDA_FATAL(s.download(1, 1));
    s.get_rows(1, dst, dstride, 2, h, v);
}
}
