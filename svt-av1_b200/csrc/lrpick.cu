// lrpick.cu — the reductions of the loop-restoration SEARCH on sm_90a.
//
// Replaces (reference files under Source/Lib/Encoder/Codec):
//   svt_av1_compute_stats_c / svt_av1_compute_stats_highbd_c   EbRestorationPick.c:704-790 (find_average EbRestorationPick.h:24-44)
//   svt_av1_lowbd_pixel_proj_error_c / svt_av1_highbd_pixel_proj_error_c   EbRestorationPick.c:174-315
//
// compute_stats builds the Wiener normal equations of one restoration unit: with y = the win x win window of the
// degraded picture around a sample (minus the unit average, column-major: idx = (dx+hw)*win + (dy+hw)) and x = the
// source sample (minus the average), M[k] = sum y[k] x and H[k][l] = sum y[k] y[l] over the unit (int64, exact).
// Three kernels: stats_sum_kernel (the unit averages), stats_mma_kernel (M and H on the INT8 tensor cores, exact: see
// its comment) and stats_finish_kernel (high-bit-depth divider, mirror of H).  The linear solves of the search stay on
// the host (double precision, tiny), as in SURVEY.md §8(a).
#include <algorithm>

#include "common.cuh"

using namespace svtb200;

namespace {

struct StatsUnit { // one restoration unit of a plane
    int h_start, h_end, v_start, v_end;
};
struct StatsDev {
    const void *dgd, *src; // planes (device), sample (0,0)
    int dgd_stride, src_stride, pw, ph; // reads of dgd outside [0,pw)x[0,ph) are clamped (= the replicated border)
    int clamp; // 0: the caller guarantees a halo of win/2 valid samples around every unit (drop-in staging)
    const StatsUnit *units;
    int n_units;
    unsigned long long *sum; // [n_units] sample sums for the average
    long long *out; // [n_units][win2 + win2*win2]: M then H (upper triangle filled; mirrored by finish_kernel)
    int divider; // 1 / 4 / 16 (high bit depth 8/10/12)
};

template <typename T>
__global__ void __launch_bounds__(256) stats_sum_kernel(const StatsDev d) {
    const StatsUnit u = d.units[blockIdx.y];
    const int w = u.h_end - u.h_start, h = u.v_end - u.v_start;
    const T *p = reinterpret_cast<const T *>(d.dgd);
    unsigned long long acc = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < w * h; i += gridDim.x * blockDim.x) {
        const int y = i / w, x = i - y * w;
        acc += p[(size_t)(u.v_start + y) * d.dgd_stride + u.h_start + x];
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(&d.sum[blockIdx.y], acc);
}

// ---- the normal equations on the INT8 tensor cores ------------------------------------------------------------
// H and M together are the Gram matrix of z = [the win2 window differences, the source difference] over the samples of
// a unit: G = Z^T Z (upper triangle; column win2 is M).  The differences need 9 (8-bit) to 13 (12-bit) bits, the tensor
// cores multiply int8, so every difference is split once, at staging, into balanced limbs  v = 128 * hi + lo,
// lo in [-64, 63], |hi| <= 32, and THREE int8 Gram matrices are accumulated, of hi, of lo and of (hi + lo) (which
// still fits: |hi + lo| <= 96):   v_k v_l = 16256 * hi_k hi_l + 128 * (hi + lo)_k (hi + lo)_l - 127 * lo_k lo_l.
// Every product sum is an exact int32 (4096 samples * 96^2 < 2^31) and the combination is done in int64, so the result
// is the reference's integer sum bit for bit (EbRestorationPick.c:704-790), whatever the order.
//
// mma.sync.m16n8k32.s8: the K dimension are 32 samples of one tile row, the M / N dimensions rows of Z^T / columns of Z.
// Both operands are the same data: lane (g, tig) holds, for row m = g + 8 j of Z^T, the 8 samples 8 tig .. 8 tig + 7 of
// the K step as two registers, which are at once rows g / g + 8 of the A fragments of row tile j / 2 and column g of the B
// fragment of column tile j (the K index -> sample map is ours to choose as long as A and B agree).  A register is 4
// consecutive bytes of a staged int8 plane at an arbitrary byte offset (window column kc): three aligned LDS.32 and two
// PRMT per row.  A CTA owns a 64x64 sample tile of one unit; warp = (limb, quarter of the tile rows); 16 (win 7) or 6
// (win 5) accumulator tiles per warp stay in registers for the whole tile, are merged through int32 shared atomics,
// combined to int64 and sent to the unit's M / H with one 64-bit global atomic per entry and CTA.
// row pitch of the staged window planes: 37 words - the 7 window rows a quarter-warp group reads in one LDS land 5 banks
// apart (bank = 5 kr + 2 tig: conflict-free but for one pair), against 2-way conflicts on most banks with the dense 18-word
// pitch (ncu: 42 % of the shared wavefronts were conflicts) - which changed the run time by nothing measurable (0.107 ms
// either way): the kernel is bound by its 12 warps / SM (116 registers), not by the shared-memory pipe; the source planes
// (one reader per group) stay dense
constexpr int TC_TW = 64, TC_TH = 64, TC_NT = 384, TC_PITCH = 148, TC_XPITCH = 72, TC_SLICES = 4;

__device__ __forceinline__ void mma_s8(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// One resident CTA per SM: a register cap for two (80 registers) spills the accumulators and runs slower.
template <typename T, int WIN>
__global__ void __launch_bounds__(TC_NT, 1) stats_mma_kernel(const StatsDev d, int tiles_x_max) {
    constexpr int HW = WIN / 2, WIN2 = WIN * WIN, NROW = WIN2 + 1, NJ = (NROW + 7) / 8, MT = (NJ + 1) / 2;
    constexpr int RH = TC_TH + 2 * HW, YB = RH * TC_PITCH, XB = TC_TH * TC_XPITCH, SW = TC_XPITCH / 4; // SW: staged words per row
    constexpr int NTILE = MT * NJ - MT * (MT - 1); // sum over mt of (NJ - 2 mt): column tiles nt >= 2 mt
    static_assert(3 * NTILE * 128 * 4 <= 3 * (YB + XB), "the merge buffer aliases the staged planes");
    static_assert(TC_TW + 2 * HW <= TC_XPITCH - 2 && TC_XPITCH <= TC_PITCH, "a row read ends inside the staged words");
    __shared__ __align__(16) uint8_t s_raw[3 * (YB + XB)]; // [limb] window planes, then [limb] source planes
    const StatsUnit u = d.units[blockIdx.y];
    const int uw = u.h_end - u.h_start, uh = u.v_end - u.v_start;
    const int tx = blockIdx.x % tiles_x_max, ty = blockIdx.x / tiles_x_max;
    const int x0 = u.h_start + tx * TC_TW, y0 = u.v_start + ty * TC_TH;
    if (x0 >= u.h_end || y0 >= u.v_end) return;
    const int tw = min(TC_TW, u.h_end - x0), th = min(TC_TH, u.v_end - y0);
    const int avg = (int)(d.sum[blockIdx.y] / (unsigned long long)(uw * uh)); // find_average: truncating division
    const T *dg = reinterpret_cast<const T *>(d.dgd);
    const T *sr = reinterpret_cast<const T *>(d.src);
    const int tid = threadIdx.x;
    // staging: 4 samples -> one word of each limb plane
    for (int i = tid; i < (RH + TC_TH) * SW; i += TC_NT) {
        const int r = i / SW, wc = i - r * SW;
        const bool win_row = r < RH;
        const int rr = win_row ? r : r - RH;
        uint32_t ph = 0, pl = 0, ps = 0;
#pragma unroll
        for (int b = 0; b < 4; b++) {
            const int c = wc * 4 + b;
            int v = 0;
            if (win_row) {
                if (rr < th + 2 * HW && c < tw + 2 * HW) {
                    int yy = y0 + rr - HW, xx = x0 + c - HW;
                    if (d.clamp) {
                        yy = min(max(yy, 0), d.ph - 1);
                        xx = min(max(xx, 0), d.pw - 1);
                    }
                    v = (int)dg[(size_t)yy * d.dgd_stride + xx] - avg;
                }
            } else if (rr < th && c < tw) {
                v = (int)sr[(size_t)(y0 + rr) * d.src_stride + x0 + c] - avg;
            }
            const int lo = ((v + 64) & 127) - 64, hi = (v - lo) >> 7;
            ph |= (uint32_t)(uint8_t)hi << (8 * b);
            pl |= (uint32_t)(uint8_t)lo << (8 * b);
            ps |= (uint32_t)(uint8_t)(hi + lo) << (8 * b);
        }
        const int o = (win_row ? rr * TC_PITCH : 3 * YB + rr * TC_XPITCH) + wc * 4, lstride = win_row ? YB : XB;
        *reinterpret_cast<uint32_t *>(s_raw + o) = ph;
        *reinterpret_cast<uint32_t *>(s_raw + o + lstride) = pl;
        *reinterpret_cast<uint32_t *>(s_raw + o + 2 * lstride) = ps;
    }
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, tig = lane & 3;
    const int limb = warp % 3, slice = warp / 3;
    // byte offset of row m = g + 8 j of Z^T at tile sample (0, 0): window element (kc, kr) -> kr rows down, kc bytes right
    int off[NJ];
#pragma unroll
    for (int j = 0; j < NJ; j++) {
        const int m = g + 8 * j;
        if (m < WIN2) {
            const int kc = m / WIN, kr = m - kc * WIN;
            off[j] = limb * YB + kr * TC_PITCH + kc;
        } else {
            off[j] = 3 * YB + limb * XB; // the source row (m == WIN2); rows beyond it are masked to zero below
        }
    }
    const int last_pitch = (g + 8 * (NJ - 1) >= WIN2) ? TC_XPITCH : TC_PITCH; // only row group NJ - 1 can be the source row
    const uint32_t last_mask = (g + 8 * (NJ - 1) <= WIN2) ? 0xffffffffu : 0u;
    int acc[NTILE][4];
#pragma unroll
    for (int t = 0; t < NTILE; t++)
#pragma unroll
        for (int q = 0; q < 4; q++) acc[t][q] = 0;
    for (int pi = slice; pi < th; pi += TC_SLICES) {
        for (int pj0 = 0; pj0 < tw; pj0 += 32) {
            const int colb = pi * TC_PITCH + pj0 + 8 * tig, colb_last = pi * last_pitch + pj0 + 8 * tig;
            uint32_t f[2 * MT][2];
#pragma unroll
            for (int j = 0; j < NJ; j++) {
                const int a = off[j] + (j == NJ - 1 ? colb_last : colb);
                const uint32_t *wp = reinterpret_cast<const uint32_t *>(s_raw + (a & ~3));
                const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2], sel = 0x3210u + 0x1111u * (uint32_t)(a & 3);
                f[j][0] = __byte_perm(w0, w1, sel);
                f[j][1] = __byte_perm(w1, w2, sel);
            }
            f[NJ - 1][0] &= last_mask;
            f[NJ - 1][1] &= last_mask;
            if (2 * MT > NJ) f[2 * MT - 1][0] = f[2 * MT - 1][1] = 0;
            if (pj0 + 32 > tw) { // ragged right edge: samples outside the unit contribute a zero vector
                const int nv = min(max(tw - (pj0 + 8 * tig), 0), 8);
                const uint32_t m0 = nv >= 4 ? 0xffffffffu : (1u << (8 * nv)) - 1u;
                const uint32_t m1 = nv >= 8 ? 0xffffffffu : nv <= 4 ? 0u : (1u << (8 * (nv - 4))) - 1u;
#pragma unroll
                for (int j = 0; j < NJ; j++) {
                    f[j][0] &= m0;
                    f[j][1] &= m1;
                }
            }
            int t = 0;
#pragma unroll
            for (int mt = 0; mt < MT; mt++)
#pragma unroll
                for (int nt = 2 * mt; nt < NJ; nt++, t++)
                    mma_s8(acc[t], f[2 * mt][0], f[2 * mt + 1][0], f[2 * mt][1], f[2 * mt + 1][1], f[nt][0], f[nt][1]);
        }
    }
    __syncthreads(); // every warp is done with the planes: reuse them as the merge buffer
    int *s_g = reinterpret_cast<int *>(s_raw);
    for (int i = tid; i < 3 * NTILE * 128; i += TC_NT) s_g[i] = 0;
    __syncthreads();
#pragma unroll
    for (int t = 0; t < NTILE; t++)
#pragma unroll
        for (int q = 0; q < 4; q++)
            if (acc[t][q]) atomicAdd(&s_g[(limb * NTILE + t) * 128 + q * 32 + lane], acc[t][q]);
    __syncthreads();
    long long *out = d.out + (size_t)blockIdx.y * (WIN2 + WIN2 * WIN2);
    for (int i = tid; i < NTILE * 128; i += TC_NT) {
        const int t = i >> 7, q = (i >> 5) & 3, ln = i & 31;
        int mt = 0, rem = t; // tile index -> (mt, nt)
        while (rem >= NJ - 2 * mt) {
            rem -= NJ - 2 * mt;
            mt++;
        }
        const int nt = 2 * mt + rem;
        const int k = 16 * mt + (ln >> 2) + 8 * (q >> 1), l = 8 * nt + 2 * (ln & 3) + (q & 1);
        if (k > l || l > WIN2 || k >= WIN2) continue;
        const long long v = 16256ll * s_g[i] + 128ll * s_g[2 * NTILE * 128 + i] - 127ll * s_g[NTILE * 128 + i];
        if (v) atomicAdd(reinterpret_cast<unsigned long long *>(out + (l == WIN2 ? k : WIN2 + k * WIN2 + l)), (unsigned long long)v);
    }
}

// high-bit-depth divider (truncating, as C's `/=`) and the mirror of the upper triangle
__global__ void stats_finish_kernel(long long *out, int n_units, int win2, int divider) {
    long long *o = out + (size_t)blockIdx.x * (win2 + win2 * win2);
    for (int i = threadIdx.x; i < win2 + win2 * win2; i += blockDim.x) {
        if (i >= win2) {
            const int k = (i - win2) / win2, l = (i - win2) - k * win2;
            if (l < k) continue;
        }
        if (divider > 1) o[i] /= divider;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < win2 * win2; i += blockDim.x) {
        const int k = i / win2, l = i - k * win2;
        if (l < k) o[win2 + i] = o[win2 + l * win2 + k];
    }
}

int stats_launch(StatsDev &d, int win, int hbd, int max_uw, int max_uh, cudaStream_t st) {
    const int win2 = win * win;
    if (cudaMemsetAsync(d.sum, 0, (size_t)d.n_units * 8, st) != cudaSuccess) return -1;
    if (cudaMemsetAsync(d.out, 0, (size_t)d.n_units * (win2 + win2 * win2) * 8, st) != cudaSuccess) return -1;
    const dim3 gs(std::min(64, (max_uw * max_uh + 255) / 256), d.n_units);
    const int tiles_x = (max_uw + TC_TW - 1) / TC_TW, tiles_y = (max_uh + TC_TH - 1) / TC_TH;
    const dim3 gt(tiles_x * tiles_y, d.n_units);
    if (hbd) {
        SVTB_LAUNCH(stats_sum_kernel<uint16_t>, gs, 256, 0, st, d);
        if (win == 7)
            SVTB_LAUNCH((stats_mma_kernel<uint16_t, 7>), gt, TC_NT, 0, st, d, tiles_x);
        else
            SVTB_LAUNCH((stats_mma_kernel<uint16_t, 5>), gt, TC_NT, 0, st, d, tiles_x);
    } else {
        SVTB_LAUNCH(stats_sum_kernel<uint8_t>, gs, 256, 0, st, d);
        if (win == 7)
            SVTB_LAUNCH((stats_mma_kernel<uint8_t, 7>), gt, TC_NT, 0, st, d, tiles_x);
        else
            SVTB_LAUNCH((stats_mma_kernel<uint8_t, 5>), gt, TC_NT, 0, st, d, tiles_x);
    }
    SVTB_LAUNCH(stats_finish_kernel, d.n_units, 256, 0, st, d.out, d.n_units, win2, d.divider);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// ---- RTCD drop-in (host pointers): stage the unit + halo, run, copy M and H back -------------------------------
void stats_dropin(int win, const void *dgd, const void *src, int hbd, int h_start, int h_end, int v_start, int v_end, int dgd_stride,
                  int src_stride, int64_t *M, int64_t *H, int bit_depth) {
    const int hw = win / 2, win2 = win * win;
    const int uw = h_end - h_start, uh = v_end - v_start;
    if ((win != 7 && win != 5) || uw <= 0 || uh <= 0) {
        fprintf(stderr, "svt_av1_compute_stats_cuda: unsupported window %d / empty unit\n", win);
        abort();
    }
    const int es = hbd ? 2 : 1, dw = uw + 2 * hw, dh = uh + 2 * hw;
    // the unit + halo, the unit's source, then io: StatsUnit at 0, the sum word at 32, M and H from 64
    Staging s({(size_t)dw * dh * es, (size_t)uw * uh * es, 64 + (size_t)(win2 + win2 * win2) * 8});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, (const uint8_t *)dgd + ((ptrdiff_t)(v_start - hw) * dgd_stride + h_start - hw) * es, dgd_stride, es, dw, dh);
    s.put_rows(1, (const uint8_t *)src + ((ptrdiff_t)v_start * src_stride + h_start) * es, src_stride, es, uw, uh);
    *s.h<StatsUnit>(2) = StatsUnit{hw, hw + uw, hw, hw + uh};
    SVTB_CUDA_FATAL(s.upload(0, 2, sizeof(StatsUnit)));
    StatsDev d;
    d.dgd = s.d(0);
    d.src = s.d(1) - ((size_t)hw * uw + hw) * es; // so that (hw, hw) addresses the first staged source sample
    d.dgd_stride = dw;
    d.src_stride = uw;
    d.pw = dw;
    d.ph = dh;
    d.clamp = 0;
    d.units = s.d<const StatsUnit>(2);
    d.n_units = 1;
    d.sum = (unsigned long long *)(s.d(2) + 32);
    d.out = (long long *)(s.d(2) + 64);
    d.divider = !hbd ? 1 : bit_depth == 12 ? 16 : bit_depth == 10 ? 4 : 1;
    if (stats_launch(d, win, hbd, uw, uh, s.stream())) fatal("svt_av1_compute_stats_cuda", cudaGetLastError());
    SVTB_CUDA_FATAL(s.download(2, 2));
    memcpy(M, s.h(2) + 64, (size_t)win2 * 8);
    memcpy(H, s.h(2) + 64 + (size_t)win2 * 8, (size_t)win2 * win2 * 8);
}

// ---- pixel projection error -----------------------------------------------------------------------------------
struct ProjArgs {
    const void *src, *dat;
    const int32_t *flt0, *flt1;
    int w, h, src_stride, dat_stride, f0s, f1s, xq0, xq1, r0, r1, hbd;
    unsigned long long *out;
};
__global__ void __launch_bounds__(256) proj_error_kernel(const ProjArgs a) {
    long long acc = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.w * a.h; i += gridDim.x * blockDim.x) {
        const int y = i / a.w, x = i - y * a.w;
        const int s = a.hbd ? ((const uint16_t *)a.src)[(size_t)y * a.src_stride + x] : ((const uint8_t *)a.src)[(size_t)y * a.src_stride + x];
        const int dv = a.hbd ? ((const uint16_t *)a.dat)[(size_t)y * a.dat_stride + x] : ((const uint8_t *)a.dat)[(size_t)y * a.dat_stride + x];
        int e;
        if (a.r0 > 0 || a.r1 > 0) {
            const int u = dv << 4; // SGRPROJ_RST_BITS
            int v = a.hbd ? (1 << 10) : (u << 7); // highbd: half; lowbd: u << SGRPROJ_PRJ_BITS (rounded below)
            if (a.r0 > 0) v += a.xq0 * (a.flt0[(size_t)y * a.f0s + x] - u);
            if (a.r1 > 0) v += a.xq1 * (a.flt1[(size_t)y * a.f1s + x] - u);
            e = a.hbd ? (v >> 11) + dv - s : ((v + (1 << 10)) >> 11) - s;
        } else {
            e = dv - s;
        }
        acc += (long long)(e * e);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(a.out, (unsigned long long)acc);
}

// the staging of both projection drop-ins: src, dat and the filtered planes the parameters use packed and uploaded,
// then region 4 (= a.out): n_out 64-bit sums, zeroed on the device
Staging proj_stage(ProjArgs &a, const void *src, int width, int height, int src_stride, const void *dat, int dat_stride,
                   const int32_t *flt0, int f0s, const int32_t *flt1, int f1s, const int32_t *params, int hbd, int n_out) {
    const int es = hbd ? 2 : 1, r0 = params[0], r1 = params[1];
    const size_t pb = (size_t)width * height * es, fb = (size_t)width * height * 4;
    Staging s({pb, pb, fb, fb, (size_t)n_out * 8});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, src, src_stride, es, width, height);
    s.put_rows(1, dat, dat_stride, es, width, height);
    if (r0 > 0) s.put_rows(2, flt0, f0s, 4, width, height);
    if (r1 > 0) s.put_rows(3, flt1, f1s, 4, width, height);
    SVTB_CUDA_FATAL(s.upload(0, 3));
    a.src = s.d(0);
    a.dat = s.d(1);
    a.flt0 = s.d<const int32_t>(2);
    a.flt1 = s.d<const int32_t>(3);
    a.w = width, a.h = height, a.src_stride = a.dat_stride = a.f0s = a.f1s = width;
    a.xq0 = a.xq1 = 0, a.r0 = r0, a.r1 = r1, a.hbd = hbd;
    a.out = s.d<unsigned long long>(4);
    SVTB_CUDA_FATAL(cudaMemsetAsync(a.out, 0, (size_t)n_out * 8, s.stream()));
    return s;
}

int64_t proj_dropin(const void *src, int width, int height, int src_stride, const void *dat, int dat_stride, const int32_t *flt0,
                    int f0s, const int32_t *flt1, int f1s, const int32_t *xq, const int32_t *params /* SgrParamsType: r[2], s[2] */,
                    int hbd) {
    if (width <= 0 || height <= 0) return 0;
    ProjArgs a;
    Staging s = proj_stage(a, src, width, height, src_stride, dat, dat_stride, flt0, f0s, flt1, f1s, params, hbd, 1);
    a.xq0 = xq[0], a.xq1 = xq[1];
    SVTB_LAUNCH(proj_error_kernel, std::min(64, (width * height + 255) / 256), 256, 0, s.stream(), a);
    SVTB_CUDA_FATAL(s.download(4, 4));
    return *s.h<int64_t>(4);
}

// svt_get_proj_subspace_c (EbRestorationPick.c:337-440): the five sums over the unit.  The reference accumulates them
// in double, but every term is an integer (u, s, f1, f2 are integers) and every partial sum stays below 2^53, so the
// double sums are exact and equal these 64-bit integer sums; the 2x2 solve below repeats the reference's expressions.
__global__ void __launch_bounds__(256) proj_sums_kernel(const ProjArgs a, long long *out /*[5]: H00 H11 H01 C0 C1*/) {
    long long h00 = 0, h11 = 0, h01 = 0, c0 = 0, c1 = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.w * a.h; i += gridDim.x * blockDim.x) {
        const int y = i / a.w, x = i - y * a.w;
        const int sv = a.hbd ? ((const uint16_t *)a.src)[(size_t)y * a.src_stride + x] : ((const uint8_t *)a.src)[(size_t)y * a.src_stride + x];
        const int dv = a.hbd ? ((const uint16_t *)a.dat)[(size_t)y * a.dat_stride + x] : ((const uint8_t *)a.dat)[(size_t)y * a.dat_stride + x];
        const long long u = dv << 4, s = (long long)(sv << 4) - u;
        const long long f1 = a.r0 > 0 ? (long long)a.flt0[(size_t)y * a.f0s + x] - u : 0;
        const long long f2 = a.r1 > 0 ? (long long)a.flt1[(size_t)y * a.f1s + x] - u : 0;
        h00 += f1 * f1, h11 += f2 * f2, h01 += f1 * f2, c0 += f1 * s, c1 += f2 * s;
    }
    long long v[5] = {h00, h11, h01, c0, c1};
#pragma unroll
    for (int k = 0; k < 5; k++) {
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
        if ((threadIdx.x & 31) == 0 && v[k]) atomicAdd(reinterpret_cast<unsigned long long *>(out + k), (unsigned long long)v[k]);
    }
}

void proj_subspace_dropin(const void *src, int width, int height, int src_stride, const void *dat, int dat_stride, int hbd,
                          const int32_t *flt0, int f0s, const int32_t *flt1, int f1s, int *xq, const int32_t *params) {
    xq[0] = xq[1] = 0;
    if (width <= 0 || height <= 0) return;
    const int r0 = params[0], r1 = params[1];
    ProjArgs a;
    Staging s = proj_stage(a, src, width, height, src_stride, dat, dat_stride, flt0, f0s, flt1, f1s, params, hbd, 5);
    SVTB_LAUNCH(proj_sums_kernel, std::min(64, (width * height + 255) / 256), 256, 0, s.stream(), a, s.d<long long>(4));
    SVTB_CUDA_FATAL(s.download(4, 4));
    long long v[5];
    memcpy(v, s.h(4), 40);
    const int size = width * height;
    double H[2][2], C[2], det, x[2];
    H[0][0] = (double)v[0], H[1][1] = (double)v[1], H[0][1] = (double)v[2], C[0] = (double)v[3], C[1] = (double)v[4];
    H[0][0] /= size;
    H[0][1] /= size;
    H[1][1] /= size;
    H[1][0] = H[0][1];
    C[0] /= size;
    C[1] /= size;
    if (r0 == 0) {
        det = H[1][1];
        if (det < 1e-8) return; // ill-posed, default values
        x[1] = C[1] / det;
        xq[1] = (int)rint(x[1] * (1 << 7));
    } else if (r1 == 0) {
        det = H[0][0];
        if (det < 1e-8) return;
        x[0] = C[0] / det;
        xq[0] = (int)rint(x[0] * (1 << 7));
    } else {
        det = (H[0][0] * H[1][1] - H[0][1] * H[1][0]);
        if (det < 1e-8) return;
        x[0] = (H[1][1] * C[0] - H[0][1] * C[1]) / det;
        x[1] = (H[0][0] * C[1] - H[1][0] * C[0]) / det;
        xq[0] = (int)rint(x[0] * (1 << 7));
        xq[1] = (int)rint(x[1] * (1 << 7));
    }
}

static inline const void *short_ptr(const uint8_t *p) { return (const void *)(((uintptr_t)p) << 1); } // CONVERT_TO_SHORTPTR

} // namespace

extern "C" {

void svt_av1_compute_stats_cuda(int32_t wiener_win, const uint8_t *dgd8, const uint8_t *src8, int32_t h_start, int32_t h_end,
                                int32_t v_start, int32_t v_end, int32_t dgd_stride, int32_t src_stride, int64_t *M, int64_t *H) {
    stats_dropin(wiener_win, dgd8, src8, 0, h_start, h_end, v_start, v_end, dgd_stride, src_stride, M, H, 8);
}
void svt_av1_compute_stats_highbd_cuda(int32_t wiener_win, const uint8_t *dgd8, const uint8_t *src8, int32_t h_start, int32_t h_end,
                                       int32_t v_start, int32_t v_end, int32_t dgd_stride, int32_t src_stride, int64_t *M, int64_t *H,
                                       int32_t bit_depth) {
    stats_dropin(wiener_win, short_ptr(dgd8), short_ptr(src8), 1, h_start, h_end, v_start, v_end, dgd_stride, src_stride, M, H, bit_depth);
}
int64_t svt_av1_lowbd_pixel_proj_error_cuda(const uint8_t *src8, int32_t width, int32_t height, int32_t src_stride, const uint8_t *dat8,
                                            int32_t dat_stride, int32_t *flt0, int32_t flt0_stride, int32_t *flt1, int32_t flt1_stride,
                                            int32_t xq[2], const void *params) {
    return proj_dropin(src8, width, height, src_stride, dat8, dat_stride, flt0, flt0_stride, flt1, flt1_stride, xq,
                       (const int32_t *)params, 0);
}
int64_t svt_av1_highbd_pixel_proj_error_cuda(const uint8_t *src8, int32_t width, int32_t height, int32_t src_stride, const uint8_t *dat8,
                                             int32_t dat_stride, int32_t *flt0, int32_t flt0_stride, int32_t *flt1, int32_t flt1_stride,
                                             int32_t xq[2], const void *params) {
    return proj_dropin(short_ptr(src8), width, height, src_stride, short_ptr(dat8), dat_stride, flt0, flt0_stride, flt1, flt1_stride,
                       xq, (const int32_t *)params, 1);
}

void svt_get_proj_subspace_cuda(const uint8_t *src8, int32_t width, int32_t height, int32_t src_stride, const uint8_t *dat8,
                                int32_t dat_stride, int32_t use_highbitdepth, int32_t *flt0, int32_t flt0_stride, int32_t *flt1,
                                int32_t flt1_stride, int32_t *xq, const void *params) {
    proj_subspace_dropin(use_highbitdepth ? short_ptr(src8) : (const void *)src8, width, height, src_stride,
                         use_highbitdepth ? short_ptr(dat8) : (const void *)dat8, dat_stride, use_highbitdepth != 0, flt0, flt0_stride, flt1,
                         flt1_stride, xq, (const int32_t *)params);
}

// Wiener statistics of every restoration unit of one plane, device resident (the batched form of the search's
// compute_stats calls: search_wiener, EbRestorationPick.c).  rects: DEVICE array of n_units {h_start, h_end, v_start,
// v_end}; out: DEVICE int64 [n_units][win2 + win2*win2] (M then H); scratch: >= 8 * n_units bytes (device).
int svt_b200_lr_wiener_stats(const SvtB200Frame *dgd, const SvtB200Frame *src, int32_t plane, int32_t wiener_win,
                             const int32_t *rects, int32_t n_units, int32_t max_unit_w, int32_t max_unit_h, int64_t *out,
                             void *scratch, void *stream) {
    if (!dgd || !src || !rects || !out || !scratch || plane < 0 || plane > 2 || (wiener_win != 7 && wiener_win != 5) || n_units <= 0 ||
        dgd->bit_depth != src->bit_depth || max_unit_w <= 0 || max_unit_h <= 0) {
        set_error("svt_b200_lr_wiener_stats: bad argument");
        return SVT_B200_ERR_ARG;
    }
    const int ss = plane ? 1 : 0;
    StatsDev d;
    d.dgd = plane == 0 ? dgd->y : plane == 1 ? dgd->cb : dgd->cr;
    d.src = plane == 0 ? src->y : plane == 1 ? src->cb : src->cr;
    d.dgd_stride = plane ? dgd->stride_c : dgd->stride_y;
    d.src_stride = plane ? src->stride_c : src->stride_y;
    d.pw = (dgd->width + ss) >> ss;
    d.ph = (dgd->height + ss) >> ss;
    d.clamp = 1;
    d.units = reinterpret_cast<const StatsUnit *>(rects);
    d.n_units = n_units;
    d.sum = (unsigned long long *)scratch;
    d.out = (long long *)out;
    d.divider = dgd->bit_depth == 12 ? 16 : dgd->bit_depth == 10 ? 4 : 1;
    if (stats_launch(d, wiener_win, dgd->bit_depth > 8, max_unit_w, max_unit_h, (cudaStream_t)stream)) {
        set_error("svt_b200_lr_wiener_stats: launch failed");
        return SVT_B200_ERR_CUDA;
    }
    return SVT_B200_OK;
}
}
