// txfm.cuh — device-side integer transforms of AV1 as SVT-AV1 v0.8.6 computes them (bit-exact).
//
// Replaces the hand-unrolled stage lists of Source/Lib/Encoder/Codec/EbTransforms.c:75-2271 and
// Source/Lib/Common/Codec/EbInvTransforms.c:75-2358.  The butterfly networks are generated from their
// recursive structure (DCT-n = butterfly ; DCT-n/2 ; ODD(n/2) ; bit reversal) instead of being spelled out;
// every layer acts on disjoint pairs.  Two forms of the same structure functions: fully unrolled templates on a
// register array (n <= 32: one thread loads a row/column, transforms it in registers, stores it) and an in-place
// strided shared-memory form (n = 64).  Only half_btf() rounds; additions are exact, so evaluation order of
// independent sub-networks cannot change a bit (DESIGN.md §Transforms).
#pragma once
#include <cmath>
#include <cstdint>

#include "common.cuh"

namespace svtb200 {

// per-translation-unit copies (no relocatable device code): every .cu that includes this header uploads them with
// txfm_upload_tables() once per device before launching a kernel that uses them
static __constant__ int32_t c_cospi[4][64]; // cos_bit 10..13
static __constant__ int32_t c_sinpi[4][5];

// host: fills the constant tables on the current device
static void txfm_upload_tables() {
    int32_t cospi[4][64];
    // eb_av1_cospi_arr_data: round(cos(i*pi/128) * 2^bit).  eb_av1_sinpi_arr_data is hand-adjusted in the reference
    // (sinpi[1] + sinpi[2] == sinpi[4]) and therefore kept as data.
    static const int32_t sinpi[4][5] = {{0, 330, 621, 836, 951}, {0, 660, 1241, 1672, 1901},
                                        {0, 1321, 2482, 3344, 3803}, {0, 2642, 4964, 6689, 7606}};
    for (int b = 10; b <= 13; b++)
        for (int i = 0; i < 64; i++) cospi[b - 10][i] = (int32_t)floor(cos(M_PI * i / 128.0) * (double)(1 << b) + 0.5);
    SVTB_CUDA_FATAL(cudaMemcpyToSymbol(c_cospi, cospi, sizeof(cospi)));
    SVTB_CUDA_FATAL(cudaMemcpyToSymbol(c_sinpi, sinpi, sizeof(sinpi)));
}

// Common/Codec/EbInvTransforms.h:285-312: 32-bit wrapping products, 64-bit sum, rounding shift
__device__ __forceinline__ int32_t half_btf(int32_t w0, int32_t in0, int32_t w1, int32_t in1, int bit) {
    const long long r = (long long)(int32_t)((uint32_t)w0 * (uint32_t)in0) + (long long)(int32_t)((uint32_t)w1 * (uint32_t)in1);
    return (int32_t)((r + (1ll << (bit - 1))) >> bit);
}
__device__ __forceinline__ int32_t round_shift64(long long v, int bit) { return (int32_t)((v + (1ll << (bit - 1))) >> bit); }
__device__ __forceinline__ int32_t wadd(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
__device__ __forceinline__ int32_t wsub(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }
__device__ __forceinline__ int32_t clampv(int32_t v, int bit) { // clamp_value, EbInvTransforms.c:67
    if (bit <= 0) return v;
    const int32_t mx = (int32_t)((1ll << (bit - 1)) - 1), mn = (int32_t)(-(1ll << (bit - 1)));
    return v < mn ? mn : (v > mx ? mx : v);
}
__device__ __forceinline__ int brev(int v, int bits) { return (int)(__brev((unsigned)v) >> (32 - bits)); }
__device__ __forceinline__ int ilog2(int n) { return 31 - __clz(n); }
__host__ __device__ constexpr int clog2(int n) { return n <= 1 ? 0 : 1 + clog2(n / 2); }

#define TX(i) x[(i) * s]

__device__ inline void odd_butterflies(int32_t *x, int s, int m, int S, int clamp_bit) {
    for (int base = 0; base < m; base += S) {
        const bool mirrored = (base / S) & 1;
        for (int i = 0; i < S / 2; i++) {
            const int lo = base + i, hi = base + S - 1 - i;
            const int32_t a = TX(lo), b = TX(hi);
            const int32_t sum = clampv(wadd(a, b), clamp_bit), dif = clampv(mirrored ? wsub(b, a) : wsub(a, b), clamp_bit);
            TX(mirrored ? hi : lo) = sum;
            TX(mirrored ? lo : hi) = dif;
        }
    }
}
__device__ inline void odd_rotations(int32_t *x, int s, int m, int j, const int32_t *c, int bit) {
    const int G = m >> j;
    for (int t = 0; t < m / 2; t++) {
        const int u = t & (G - 1), p = m - 1 - t;
        if (u < G / 4 || u >= 3 * G / 4) continue;
        const int k = (32 >> j) * brev((1 << j) + t / G, j + 1);
        const int32_t a = TX(t), b = TX(p);
        if (u < G / 2) {
            TX(t) = half_btf(-c[k], a, c[64 - k], b, bit);
            TX(p) = half_btf(c[k], b, c[64 - k], a, bit);
        } else {
            TX(t) = half_btf(-c[64 - k], a, -c[k], b, bit);
            TX(p) = half_btf(c[64 - k], b, -c[k], a, bit);
        }
    }
}
__device__ inline void odd_final_rotation(int32_t *x, int s, int m, const int32_t *c, int bit, bool inverse) {
    const int n = 2 * m, L = ilog2(n);
    for (int t = 0; t < m / 2; t++) {
        const int p = m - 1 - t, k = (64 / n) * brev(m + t, L);
        const int32_t a = TX(t), b = TX(p);
        if (!inverse) {
            TX(t) = half_btf(c[64 - k], a, c[k], b, bit);
            TX(p) = half_btf(c[64 - k], b, -c[k], a, bit);
        } else {
            TX(t) = half_btf(c[64 - k], a, -c[k], b, bit);
            TX(p) = half_btf(c[k], a, c[64 - k], b, bit);
        }
    }
}
__device__ inline void bit_reverse_permute(int32_t *x, int s, int n) {
    const int L = ilog2(n);
    for (int j = 0; j < n; j++) {
        const int r = brev(j, L);
        if (r > j) {
            const int32_t t = TX(j);
            TX(j) = TX(r);
            TX(r) = t;
        }
    }
}
__device__ inline void fdct(int32_t *x, int s, int n_total, int bit) {
    const int32_t *c = c_cospi[bit - 10];
    for (int n = n_total; n >= 4; n >>= 1) {
        const int m = n / 2, L = ilog2(n);
        for (int i = 0; i < m; i++) {
            const int32_t a = TX(i), b = TX(n - 1 - i);
            TX(i) = wadd(a, b);
            TX(n - 1 - i) = wsub(a, b);
        }
        int32_t *y = x + m * s;
        for (int j = 0; j <= L - 3; j++) {
            odd_rotations(y, s, m, j, c, bit);
            odd_butterflies(y, s, m, m >> (j + 1), 0);
        }
        odd_final_rotation(y, s, m, c, bit, false);
    }
    const int32_t a = TX(0), b = TX(1);
    TX(0) = half_btf(c[32], a, c[32], b, bit);
    TX(1) = half_btf(-c[32], b, c[32], a, bit);
    bit_reverse_permute(x, s, n_total);
}
__device__ inline void idct(int32_t *x, int s, int n_total, int bit, int clamp_bit) {
    const int32_t *c = c_cospi[bit - 10];
    bit_reverse_permute(x, s, n_total);
    {
        const int32_t a = TX(0), b = TX(1);
        TX(0) = half_btf(c[32], a, c[32], b, bit);
        TX(1) = half_btf(c[32], a, -c[32], b, bit);
    }
    for (int n = 4; n <= n_total; n <<= 1) {
        const int m = n / 2, L = ilog2(n);
        int32_t *y = x + m * s;
        odd_final_rotation(y, s, m, c, bit, true);
        for (int j = L - 3; j >= 0; j--) {
            odd_butterflies(y, s, m, m >> (j + 1), clamp_bit);
            odd_rotations(y, s, m, j, c, bit);
        }
        for (int i = 0; i < m; i++) {
            const int32_t a = TX(i), b = TX(n - 1 - i);
            TX(i) = clampv(wadd(a, b), clamp_bit);
            TX(n - 1 - i) = clampv(wsub(a, b), clamp_bit);
        }
    }
}

// ---- ADST (EbTransforms.c:1445-1826, EbInvTransforms.c:707-1105) ----
__device__ inline void fadst4(int32_t *x, int s, int bit) {
    const int32_t *sp = c_sinpi[bit - 10];
    const int32_t x0 = TX(0), x1 = TX(1), x2 = TX(2), x3 = TX(3);
    if (!(x0 | x1 | x2 | x3)) return; // all zero stays zero
    auto M = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); };
    const int32_t s0 = M(sp[1], x0), s1 = M(sp[4], x0), s2 = M(sp[2], x1), s3 = M(sp[1], x1), s4 = M(sp[3], x2),
                  s5 = M(sp[4], x3), s6 = M(sp[2], x3), s7 = wsub(wadd(x0, x1), x3);
    const int32_t y0 = wadd(wadd(s0, s2), s5), y1 = M(sp[3], s7), y2 = wadd(wsub(s1, s3), s6), y3 = s4;
    TX(0) = round_shift64((long long)wadd(y0, y3), bit);
    TX(1) = round_shift64((long long)y1, bit);
    TX(2) = round_shift64((long long)wsub(y2, y3), bit);
    TX(3) = round_shift64((long long)wadd(wsub(y2, y0), y3), bit);
}
__device__ inline void iadst4(int32_t *x, int s, int bit) {
    const int32_t *sp = c_sinpi[bit - 10];
    const int32_t x0 = TX(0), x1 = TX(1), x2 = TX(2), x3 = TX(3);
    if (!(x0 | x1 | x2 | x3)) return;
    auto M = [](int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); };
    int32_t s0 = M(sp[1], x0), s1 = M(sp[2], x0), s2 = M(sp[3], x1), s3 = M(sp[4], x2), s4 = M(sp[1], x2),
            s5 = M(sp[2], x3), s6 = M(sp[4], x3), s7 = wadd(wsub(x0, x2), x3);
    s0 = wadd(wadd(s0, s3), s5);
    s1 = wsub(wsub(s1, s4), s6);
    s3 = s2;
    s2 = M(sp[3], s7);
    TX(0) = round_shift64((long long)wadd(s0, s3), bit);
    TX(1) = round_shift64((long long)wadd(s1, s3), bit);
    TX(2) = round_shift64((long long)s2, bit);
    TX(3) = round_shift64((long long)wsub(wadd(s0, s1), s3), bit);
}

// identity (forward and inverse scale identically: EbTransforms.c:2239-2278, EbInvTransforms.c:2321-2358)
__device__ inline void identity_scale(int32_t *x, int s, int n) {
    for (int i = 0; i < n; i++) {
        const int32_t v = TX(i);
        int32_t o;
        if (n == 4) o = round_shift64((long long)v * 5793, 12);
        else if (n == 8) o = (int32_t)((uint32_t)v * 2u);
        else if (n == 16) o = round_shift64((long long)v * 2 * 5793, 12);
        else if (n == 32) o = (int32_t)((uint32_t)v * 4u);
        else o = round_shift64((long long)v * 4 * 5793, 12);
        TX(i) = o;
    }
}
#undef TX

// kind: 0 DCT, 1 ADST, 2 FLIPADST, 3 IDTX

// ---------------------------------------------------------------------------------------------------------------
// Register-resident, fully unrolled versions of the same networks (n <= 32).  The structure functions above are
// re-stated as templates so that after unrolling every index and every cospi subscript is a compile-time constant:
// a 1-D transform is then N strided LDS, the butterflies in registers, N STS — no index arithmetic, no in-place
// shared-memory traffic between layers.  Bit-exactness is by construction (same layers, same half_btf); the
// in-place versions remain for n = 64 and as the structural reference the tests cross-check.
// ---------------------------------------------------------------------------------------------------------------
template <int M, int S>
__device__ __forceinline__ void r_odd_butterflies(int32_t *x, int clamp_bit) {
#pragma unroll
    for (int base = 0; base < M; base += S) {
        const bool mirrored = (base / S) & 1;
#pragma unroll
        for (int i = 0; i < S / 2; i++) {
            const int lo = base + i, hi = base + S - 1 - i;
            const int32_t a = x[lo], b = x[hi];
            const int32_t sum = clampv(wadd(a, b), clamp_bit), dif = clampv(mirrored ? wsub(b, a) : wsub(a, b), clamp_bit);
            x[mirrored ? hi : lo] = sum;
            x[mirrored ? lo : hi] = dif;
        }
    }
}
template <int M, int J>
__device__ __forceinline__ void r_odd_rotations(int32_t *x, const int32_t *c, int bit) {
    constexpr int G = M >> J;
#pragma unroll
    for (int t = 0; t < M / 2; t++) {
        const int u = t & (G - 1), p = M - 1 - t;
        if (u < G / 4 || u >= 3 * G / 4) continue;
        const int k = (32 >> J) * brev((1 << J) + t / G, J + 1);
        const int32_t a = x[t], b = x[p];
        if (u < G / 2) {
            x[t] = half_btf(-c[k], a, c[64 - k], b, bit);
            x[p] = half_btf(c[k], b, c[64 - k], a, bit);
        } else {
            x[t] = half_btf(-c[64 - k], a, -c[k], b, bit);
            x[p] = half_btf(c[64 - k], b, -c[k], a, bit);
        }
    }
}
template <int M, bool INV>
__device__ __forceinline__ void r_odd_final(int32_t *x, const int32_t *c, int bit) {
    constexpr int N = 2 * M;
#pragma unroll
    for (int t = 0; t < M / 2; t++) {
        const int p = M - 1 - t, k = (64 / N) * brev(M + t, clog2(N));
        const int32_t a = x[t], b = x[p];
        if (!INV) {
            x[t] = half_btf(c[64 - k], a, c[k], b, bit);
            x[p] = half_btf(c[64 - k], b, -c[k], a, bit);
        } else {
            x[t] = half_btf(c[64 - k], a, -c[k], b, bit);
            x[p] = half_btf(c[k], a, c[64 - k], b, bit);
        }
    }
}
// odd half of a DCT-2M: layers j = 0 .. log2(2M) - 3
template <int M, int J>
__device__ __forceinline__ void r_odd_fwd_layers(int32_t *y, const int32_t *c, int bit) {
    if constexpr (J <= clog2(2 * M) - 3) {
        r_odd_rotations<M, J>(y, c, bit);
        r_odd_butterflies<M, (M >> (J + 1))>(y, 0);
        r_odd_fwd_layers<M, J + 1>(y, c, bit);
    }
}
template <int M, int J>
__device__ __forceinline__ void r_odd_inv_layers(int32_t *y, const int32_t *c, int bit, int clamp_bit) {
    if constexpr (J >= 0) {
        r_odd_butterflies<M, (M >> (J + 1))>(y, clamp_bit);
        r_odd_rotations<M, J>(y, c, bit);
        r_odd_inv_layers<M, J - 1>(y, c, bit, clamp_bit);
    }
}
template <int N>
__device__ __forceinline__ void r_fdct_rec(int32_t *x, const int32_t *c, int bit) {
    if constexpr (N >= 4) {
        constexpr int M = N / 2;
#pragma unroll
        for (int i = 0; i < M; i++) {
            const int32_t a = x[i], b = x[N - 1 - i];
            x[i] = wadd(a, b);
            x[N - 1 - i] = wsub(a, b);
        }
        r_odd_fwd_layers<M, 0>(x + M, c, bit);
        r_odd_final<M, false>(x + M, c, bit);
        r_fdct_rec<N / 2>(x, c, bit);
    } else {
        const int32_t a = x[0], b = x[1];
        x[0] = half_btf(c[32], a, c[32], b, bit);
        x[1] = half_btf(-c[32], b, c[32], a, bit);
    }
}
template <int N, int NT>
__device__ __forceinline__ void r_idct_rec(int32_t *x, const int32_t *c, int bit, int clamp_bit) {
    if constexpr (N == 2) {
        const int32_t a = x[0], b = x[1];
        x[0] = half_btf(c[32], a, c[32], b, bit);
        x[1] = half_btf(c[32], a, -c[32], b, bit);
    } else {
        constexpr int M = N / 2;
        r_idct_rec<N / 2, NT>(x, c, bit, clamp_bit);
        r_odd_final<M, true>(x + M, c, bit);
        r_odd_inv_layers<M, (clog2(N)) - 3>(x + M, c, bit, clamp_bit);
#pragma unroll
        for (int i = 0; i < M; i++) {
            const int32_t a = x[i], b = x[N - 1 - i];
            x[i] = clampv(wadd(a, b), clamp_bit);
            x[N - 1 - i] = clampv(wsub(a, b), clamp_bit);
        }
    }
}
template <int N>
__device__ __forceinline__ void r_bit_reverse(int32_t *x) {
#pragma unroll
    for (int j = 0; j < N; j++) {
        const int r = brev(j, clog2(N));
        if (r > j) {
            const int32_t t = x[j];
            x[j] = x[r];
            x[r] = t;
        }
    }
}
template <int N>
__device__ __forceinline__ void r_fdct(int32_t *x, int bit) {
    const int32_t *c = c_cospi[bit - 10];
    r_fdct_rec<N>(x, c, bit);
    r_bit_reverse<N>(x);
}
template <int N>
__device__ __forceinline__ void r_idct(int32_t *x, int bit, int clamp_bit) {
    const int32_t *c = c_cospi[bit - 10];
    r_bit_reverse<N>(x);
    r_idct_rec<N, N>(x, c, bit, clamp_bit);
}

// ADST-8/16 in registers
template <int N, int H>
__device__ __forceinline__ void r_adst_rotations(int32_t *v, const int32_t *c, int bit) {
    constexpr int NP = H / 2;
#pragma unroll
    for (int g = 0; g < N; g += 2 * H)
#pragma unroll
        for (int i = 0; i < NP; i++) {
            const int a0 = g + H + 2 * i, a1 = a0 + 1;
            const int32_t a = v[a0], b = v[a1];
            if (H == 2) {
                v[a0] = half_btf(c[32], a, c[32], b, bit);
                v[a1] = half_btf(c[32], a, -c[32], b, bit);
            } else {
                constexpr int half = NP / 2 > 0 ? NP / 2 : 1;
                const int q = i % half;
                const int k = (64 / H) * (H >= 8 ? 4 * q + 1 : 1);
                if (i < half) {
                    v[a0] = half_btf(c[k], a, c[64 - k], b, bit);
                    v[a1] = half_btf(c[64 - k], a, -c[k], b, bit);
                } else {
                    v[a0] = half_btf(-c[64 - k], a, c[k], b, bit);
                    v[a1] = half_btf(c[k], a, c[64 - k], b, bit);
                }
            }
        }
}
template <int N, int H>
__device__ __forceinline__ void r_adst_addsub(int32_t *v, int clamp_bit) {
#pragma unroll
    for (int g = 0; g < N; g += 2 * H)
#pragma unroll
        for (int i = 0; i < H; i++) {
            const int32_t a = v[g + i], b = v[g + H + i];
            v[g + i] = clampv(wadd(a, b), clamp_bit);
            v[g + H + i] = clampv(wsub(a, b), clamp_bit);
        }
}
template <int N>
__device__ __forceinline__ void r_adst_final(int32_t *v, const int32_t *c, int bit) {
#pragma unroll
    for (int i = 0; i < N / 2; i++) {
        const int k = (32 + 128 * i) / N;
        const int32_t a = v[2 * i], b = v[2 * i + 1];
        v[2 * i] = half_btf(c[k], a, c[64 - k], b, bit);
        v[2 * i + 1] = half_btf(c[64 - k], a, -c[k], b, bit);
    }
}
template <int N, int H>
__device__ __forceinline__ void r_fadst_layers(int32_t *v, const int32_t *c, int bit) {
    if constexpr (H < N) {
        r_adst_rotations<N, H>(v, c, bit);
        r_adst_addsub<N, H>(v, 0);
        r_fadst_layers<N, 2 * H>(v, c, bit);
    }
}
template <int N, int H>
__device__ __forceinline__ void r_iadst_layers(int32_t *v, const int32_t *c, int bit, int clamp_bit) {
    if constexpr (H >= 2) {
        r_adst_addsub<N, H>(v, clamp_bit);
        r_adst_rotations<N, H>(v, c, bit);
        r_iadst_layers<N, H / 2>(v, c, bit, clamp_bit);
    }
}
// the signed input / output permutations of ADST-8/16 as ternary chains: they fold to constants once the loops
// over i are unrolled (a table lookup would keep v[] in local memory)
__host__ __device__ constexpr int adst_in_perm(int n, int i) {
    return n == 8 ? (i == 0 ? 0 : i == 1 ? -7 : i == 2 ? -3 : i == 3 ? 4 : i == 4 ? -1 : i == 5 ? 6 : i == 6 ? 2 : -5) : (i == 0 ? 0 : i == 1 ? -15 : i == 2 ? -7 : i == 3 ? 8 : i == 4 ? -3 : i == 5 ? 12 : i == 6 ? 4 : i == 7 ? -11 : i == 8 ? -1 : i == 9 ? 14 : i == 10 ? 6 : i == 11 ? -9 : i == 12 ? 2 : i == 13 ? -13 : i == 14 ? -5 : 10);
}
__host__ __device__ constexpr int adst_out_perm(int n, int i) {
    return n == 8 ? (i == 0 ? 1 : i == 1 ? 6 : i == 2 ? 3 : i == 3 ? 4 : i == 4 ? 5 : i == 5 ? 2 : i == 6 ? 7 : 0) : (i == 0 ? 1 : i == 1 ? 14 : i == 2 ? 3 : i == 3 ? 12 : i == 4 ? 5 : i == 5 ? 10 : i == 6 ? 7 : i == 7 ? 8 : i == 8 ? 9 : i == 9 ? 6 : i == 10 ? 11 : i == 11 ? 4 : i == 12 ? 13 : i == 13 ? 2 : i == 14 ? 15 : 0);
}
template <int N>
__device__ __forceinline__ void r_fadst(int32_t *x, int bit) {
    if constexpr (N == 4) {
        fadst4(x, 1, bit);
    } else {
        const int32_t *c = c_cospi[bit - 10];
        int32_t v[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
            const int p = adst_in_perm(N, i);
            v[i] = p < 0 ? wsub(0, x[-p]) : x[p];
        }
        r_fadst_layers<N, 2>(v, c, bit);
        r_adst_final<N>(v, c, bit);
#pragma unroll
        for (int i = 0; i < N; i++) x[i] = v[adst_out_perm(N, i)];
    }
}
template <int N>
__device__ __forceinline__ void r_iadst(int32_t *x, int bit, int clamp_bit) {
    if constexpr (N == 4) {
        iadst4(x, 1, bit);
    } else {
        const int32_t *c = c_cospi[bit - 10];
        int32_t v[N];
#pragma unroll
        for (int i = 0; i < N; i++) v[adst_out_perm(N, i)] = x[i];
        r_adst_final<N>(v, c, bit);
        r_iadst_layers<N, N / 2>(v, c, bit, clamp_bit);
#pragma unroll
        for (int i = 0; i < N; i++) {
            const int p = adst_in_perm(N, i);
            x[p < 0 ? -p : p] = p < 0 ? wsub(0, v[i]) : v[i];
        }
    }
}
template <int N>
__device__ __forceinline__ void r_identity(int32_t *x) {
#pragma unroll
    for (int i = 0; i < N; i++) {
        const int32_t v = x[i];
        if (N == 4) x[i] = round_shift64((long long)v * 5793, 12);
        else if (N == 8) x[i] = (int32_t)((uint32_t)v * 2u);
        else if (N == 16) x[i] = round_shift64((long long)v * 2 * 5793, 12);
        else x[i] = (int32_t)((uint32_t)v * 4u);
    }
}

// One 1-D pass over a strided line: load (pre), transform in registers, (post) store.
template <int N, bool INV, typename Pre, typename Post>
__device__ __forceinline__ void r_pass(int32_t *p, int s, int kind, int bit, int clamp_bit, Pre pre, Post post) {
    int32_t v[N];
#pragma unroll
    for (int i = 0; i < N; i++) v[i] = pre(p[i * s]);
    if (kind == 0) {
        if (INV) r_idct<N>(v, bit, clamp_bit);
        else r_fdct<N>(v, bit);
    } else if (kind == 3) {
        r_identity<N>(v);
    } else {
        if constexpr (N <= 16) {
            if (INV) r_iadst<N>(v, bit, clamp_bit);
            else r_fadst<N>(v, bit);
        }
    }
#pragma unroll
    for (int i = 0; i < N; i++) p[i * s] = post(v[i]);
}
template <typename Pre, typename Post>
__device__ __forceinline__ void fwd_1d_pass(int32_t *p, int s, int n, int kind, int bit, Pre pre, Post post) {
    switch (n) {
    case 4: r_pass<4, false>(p, s, kind, bit, 0, pre, post); break;
    case 8: r_pass<8, false>(p, s, kind, bit, 0, pre, post); break;
    case 16: r_pass<16, false>(p, s, kind, bit, 0, pre, post); break;
    case 32: r_pass<32, false>(p, s, kind, bit, 0, pre, post); break;
    default:
        for (int i = 0; i < n; i++) p[i * s] = pre(p[i * s]); // n == 64: DCT or identity only, in place
        if (kind == 0) fdct(p, s, n, bit);
        else identity_scale(p, s, n);
        for (int i = 0; i < n; i++) p[i * s] = post(p[i * s]);
    }
}
template <typename Pre, typename Post>
__device__ __forceinline__ void inv_1d_pass(int32_t *p, int s, int n, int kind, int bit, int clamp_bit, Pre pre, Post post) {
    switch (n) {
    case 4: r_pass<4, true>(p, s, kind, bit, clamp_bit, pre, post); break;
    case 8: r_pass<8, true>(p, s, kind, bit, clamp_bit, pre, post); break;
    case 16: r_pass<16, true>(p, s, kind, bit, clamp_bit, pre, post); break;
    case 32: r_pass<32, true>(p, s, kind, bit, clamp_bit, pre, post); break;
    default:
        for (int i = 0; i < n; i++) p[i * s] = pre(p[i * s]);
        if (kind == 0) idct(p, s, n, bit, clamp_bit);
        else identity_scale(p, s, n);
        for (int i = 0; i < n; i++) p[i * s] = post(p[i * s]);
    }
}

// ---- 2-D configuration (av1_transform_config / svt_av1_get_inv_txfm_cfg) -------------------------------------
struct TxCfg {
    int w, h; // transform size
    int vk, hk; // 1-D kinds for columns / rows
    int ud, lr; // flips
    int fs0, fs1, fs2; // forward shifts (EbTransforms.h:26-44)
    int is0, is1; // inverse shifts (EbInvTransforms.h:51-69)
    int cbc, cbr; // forward cos_bit for columns / rows
    int rect; // |log2(w/h)| == 1
};

// ---- 2-D transforms in place on a block in shared memory (w x h int32, row pitch `pitch`) -------------------
// Lane li of the block's T lanes takes the columns and the rows li, li + T, ...  Each body holds the barrier between
// its two passes, so every thread of the CTA calls it; `live` keeps the lanes of a missing block out of the passes.
// The size comes from t: where make_txcfg<TS> fixed it at compile time, the loop bounds and the 1-D sizes fold.

// av1_transform_two_d_* without the input flips (the caller applies them as it loads the block): the column pass
// with shifts 0 and 1, then the row pass with shift 2 and the 1/sqrt(2) scaling of 2:1 rectangles.
__device__ __forceinline__ void fwd_txfm2d(int32_t *buf, int pitch, const TxCfg &t, int li, int T, bool live) {
    if (live)
        for (int c = li; c < t.w; c += T) {
            const int fs0 = t.fs0, fs1 = t.fs1;
            fwd_1d_pass(buf + c, pitch, t.h, t.vk, t.cbc, [=](int32_t v) { return (int32_t)((uint32_t)v << fs0); },
                        [=](int32_t v) { return fs1 ? round_shift64((long long)v, -fs1) : v; });
        }
    __syncthreads();
    if (live)
        for (int r = li; r < t.h; r += T) {
            const int fs2 = t.fs2, rect = t.rect;
            fwd_1d_pass(buf + r * pitch, 1, t.w, t.hk, t.cbr, [](int32_t v) { return v; }, [=](int32_t v) {
                if (fs2) v = round_shift64((long long)v, -fs2);
                if (rect) v = round_shift64((long long)v * 5793, 12);
                return v;
            });
        }
}

// svt_av1_inv_txfm2d_add_* without the output flips and the prediction add (the caller's store): the row pass with
// the rectangular scaling and shift 0, then the column pass with shift 1; bd sets the reference's clamps.  A live lane
// runs first() before its rows: the fused kernel publishes a unit's eob there, inside the same live branch.
template <typename First>
__device__ __forceinline__ void inv_txfm2d(int32_t *buf, int pitch, const TxCfg &t, int bd, int li, int T, bool live, First first) {
    const int range_row = bd == 8 ? 16 : bd == 10 ? 18 : 20, range_col = bd == 8 ? 16 : bd == 10 ? 16 : 18;
    if (live) {
        first();
        for (int r = li; r < t.h; r += T) {
            const int rect = t.rect, is0 = t.is0;
            inv_1d_pass(buf + r * pitch, 1, t.w, t.hk, 12, range_row, [=](int32_t v) {
                if (rect) v = round_shift64((long long)v * 2896, 12);
                return clampv(v, bd + 8);
            }, [=](int32_t v) { return is0 ? round_shift64((long long)v, -is0) : v; });
        }
    }
    __syncthreads();
    if (live) {
        const int col_clamp = max(bd + 6, 16);
        for (int c = li; c < t.w; c += T) {
            inv_1d_pass(buf + c, pitch, t.h, t.vk, 12, range_col, [=](int32_t v) { return clampv(v, col_clamp); },
                        [](int32_t v) { return round_shift64((long long)v, 4); });
        }
    }
}

} // namespace svtb200
