// me.cu — open-loop motion estimation on sm_90a.
//
// Replaces (reference files under Source/Lib/Encoder):
//   svt_sad_loop_kernel_c                      C_DEFAULT/EbComputeSAD_C.c:57-96
//   svt_ext_all_sad_calculation_8x8_16x16_c    Codec/EbMotionEstimation.c:230-390
//   svt_ext_eight_sad_calculation_32x32_64x64_c Codec/EbMotionEstimation.c:396-455
//   svt_ext_sad_calculation_8x8_16x16_c / _32x32_64x64_c  :122-225
//   motion_estimate_sb and everything below it (:852-3041) for a whole picture.
//
// Design (not a port of the AVX2 mpsadbw code):
//   * one picture is two launches and no host sync, each with one CTA per (super-block, reference picture):
//     - the three HME levels (one body, hme_sb), in one of two regimes chosen per picture by me_launch_plan.
//       hme_kernel_staged: every search region's window of a level and the source block are in shared memory at once
//       and the regions are searched concurrently.  hme_kernel_chunked, when a level's staged need exceeds HME_FAST_SMEM
//       (presets 0-1 at reference distances above one, or with the 4K-class table): block_search runs the
//       regions one after another, each window chunked through HME_SMEM_BYTES;
//     - fullpel_kernel<SUB>, the integer full-pel search; the SB's last CTA also runs the SB epilogue;
//   * SAD arithmetic uses the native VABSDIFF4.U8.ACC (4 abs-diffs + accumulate per lane-op); a task is Q
//     search positions of one row with the same byte alignment, so one funnel-shifted (SHF) copy of a window
//     row feeds all Q positions (DESIGN.md §4);
//   * "first minimum in raster order" (the reference's strict `<` running best) is an argmin over the key
//     (sad << 32 | raster_index): REDUX.MIN warp reductions + one shared-memory atomicMin per warp;
//   * the data-dependent glue between the stages (search-centre choice, reference pruning, search-region
//     shrinking, candidate list) runs on-device, in the CTA that completes an SB in each kernel.
#include "common.cuh"

using namespace svtb200;

namespace {

constexpr int kMaxSadValue = 128 * 128 * 255; // MAX_SAD_VALUE, Codec/EbMotionEstimation.h:93
constexpr int NT_SEARCH = 256;

__constant__ uint8_t c_tab16[16] = {0, 1, 4, 5, 2, 3, 6, 7, 8, 9, 12, 13, 10, 11, 14, 15};
__constant__ uint8_t c_inv16[16] = {0, 1, 4, 5, 2, 3, 6, 7, 8, 9, 12, 13, 10, 11, 14, 15}; // self-inverse
__constant__ uint8_t c_tab8[64] = {0,  1,  4,  5,  16, 17, 20, 21, 2,  3,  6,  7,  18, 19, 22, 23,
                                   8,  9,  12, 13, 24, 25, 28, 29, 10, 11, 14, 15, 26, 27, 30, 31,
                                   32, 33, 36, 37, 48, 49, 52, 53, 34, 35, 38, 39, 50, 51, 54, 55,
                                   40, 41, 44, 45, 56, 57, 60, 61, 42, 43, 46, 47, 58, 59, 62, 63};

// The reference's search-window clamp, statement for statement (e.g. EbMotionEstimation.c:927-975): the
// left/top clamp moves the origin and then re-tests the corrected origin (never true), so only the
// right/bottom clamp shrinks the size.
__host__ __device__ __forceinline__ void clamp_window(int origin, int pad, int pic_size, int &ao, int &size) {
    if (origin + ao < -pad) ao = -pad - origin;
    if (origin + ao > pic_size - 1) ao = ao - ((origin + ao) - (pic_size - 1));
    if (origin + ao + size > pic_size) size = max(1, size - ((origin + ao + size) - pic_size));
}
__host__ __device__ __forceinline__ int scaled_dist(int dist) { return ((dist * 5) / 8) + ((dist % 8) == 0 ? 0 : 1); }

// The search window of HME region (rx, ry) at `level` (0: 1/16, 1: 1/4, 2: full resolution), hme_level_0/1/2
// (:852-1318): offset (xo, yo) from the block and size, at the level's resolution.  Level 0 is centred on the block and
// scaled by the reference's distance multiplier `mult` (scaled_dist * 100); levels 1 and 2 are centred on the previous
// level's result (cx, cy), like (ox, oy) the block origin, in full-resolution samples.
struct HmeWindow {
    int xo, yo, saw, sah;
};
__host__ __device__ __forceinline__ HmeWindow hme_window(const SvtB200MeParams &p, int level, int rx, int ry, int mult, int cx, int cy,
                                                         int ox, int oy) {
    const SvtB200Plane &pl = level == 0 ? p.sixteenth : level == 1 ? p.quarter : p.full;
    const int shf = 2 - level, o_x = ox >> shf, o_y = oy >> shf;
    HmeWindow w;
    if (level == 0) {
        w.saw = min((int)(int16_t)((((p.hme_level0_search_area_in_width_array[rx] * mult) / 100) + 15) & ~0x0F),
                    (int)(int16_t)((p.hme_level0_max_search_area_in_width_array[rx] + 15) & ~0x0F));
        w.sah = min((int)(int16_t)((p.hme_level0_search_area_in_height_array[ry] * mult) / 100),
                    (int)(int16_t)p.hme_level0_max_search_area_in_height_array[ry]);
        int xdist = 0, ydist = 0;
        for (int i = 0; i < rx; i++)
            xdist += min((int)(int16_t)((p.hme_level0_search_area_in_width_array[i] * mult) / 100),
                         (int)(int16_t)p.hme_level0_max_search_area_in_width_array[i]);
        for (int i = 0; i < ry; i++)
            ydist += min((int)(int16_t)((p.hme_level0_search_area_in_height_array[i] * mult) / 100),
                         (int)(int16_t)p.hme_level0_max_search_area_in_height_array[i]);
        w.xo = -(int)(int16_t)(min((p.hme_level0_total_search_area_width * mult) / 100, p.hme_level0_max_total_search_area_width) >> 1) +
               xdist;
        w.yo = -(int)(int16_t)(min((p.hme_level0_total_search_area_height * mult) / 100, p.hme_level0_max_total_search_area_height) >> 1) +
               ydist;
        clamp_window(o_x, pl.origin_x - 1, pl.width, w.xo, w.saw);
        w.saw = w.saw < 16 ? w.saw : w.saw & ~0x0F;
        clamp_window(o_y, pl.origin_y - 1, pl.height, w.yo, w.sah);
    } else {
        const int aw = level == 1 ? p.hme_level1_search_area_in_width_array[rx] : p.hme_level2_search_area_in_width_array[rx];
        const int ah = level == 1 ? p.hme_level1_search_area_in_height_array[ry] : p.hme_level2_search_area_in_height_array[ry];
        w.saw = (int16_t)((aw + 7) & ~0x07);
        w.sah = ah;
        w.xo = -(w.saw >> 1) + (cx >> shf);
        w.yo = -(w.sah >> 1) + (cy >> shf);
        clamp_window(o_x, level == 1 ? pl.origin_x - 1 : 63, pl.width, w.xo, w.saw);
        w.saw = w.saw < 8 ? w.saw : w.saw & ~0x07;
        clamp_window(o_y, level == 1 ? pl.origin_y - 1 : 63, pl.height, w.yo, w.sah);
    }
    return w;
}

// integer_search_sb's search area of a reference at scaled distance `dist`, before HME's search-area divisor, and the
// window width it becomes (rounded up to a multiple of 8) once divided
__host__ __device__ __forceinline__ int2 fp_search_area(const SvtB200MeParams &p, int dist) {
    return make_int2(min(p.search_area_width * dist, p.max_me_search_width), min(p.search_area_height * dist, p.max_me_search_height));
}
__host__ __device__ __forceinline__ int fp_window_width(int w) { return (w + 7) & ~0x07; }

// Stage `rows` rows of `nbytes` bytes (arbitrary alignment, global) into shared-memory words of pitch `wpw`:
// one warp per row, one lane per 32-bit word, aligned LDG + funnel shift instead of byte loads.  Only the aligned
// words that overlap [src, src + nbytes) are read (at most 3 bytes of over-read, inside the padded planes).
__device__ __forceinline__ void stage_rows_n(uint32_t *dst, int wpw, const uint8_t *__restrict__ src, ptrdiff_t stride, int rows,
                                             int nbytes, int nwarps) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int row = warp; row < rows; row += nwarps) {
        const uintptr_t a = (uintptr_t)(src + (ptrdiff_t)row * stride);
        const uint32_t *ga = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
        const int sh = (int)(a & 3) * 8;
        const int need = (nbytes + (int)(a & 3) + 3) >> 2; // aligned words covering the row
        for (int wd = lane; wd < wpw; wd += 32) {
            const uint32_t lo = wd < need ? ga[wd] : 0u, hi = (wd + 1) < need ? ga[wd + 1] : 0u;
            dst[row * wpw + wd] = __funnelshift_r(lo, hi, sh);
        }
    }
}

// -----------------------------------------------------------------------------------------------------
// Block-cooperative exhaustive search of one bw x bh block over a saw x sah window (svt_sad_loop_kernel).
// `ref` points at search position (0,0); reference row of block row r at search row ys is
// ys*raw_stride + r*k*raw_stride.  Returns (sad << 32 | ys*saw + xs) of the first minimum, or ~0 if no
// position exists.  smem: `smem_bytes` of scratch (uint32 aligned); s_red: NT/32 uint64.
// -----------------------------------------------------------------------------------------------------
template <int NT>
__device__ uint64_t block_search(const uint8_t *__restrict__ src, int src_stride, const uint8_t *__restrict__ ref,
                                 int raw_stride, int k, int bw, int bh, int saw, int sah, uint32_t *smem,
                                 int smem_bytes, uint64_t *s_red) {
    const int tid = threadIdx.x;
    const int spw = (bw + 3) >> 2; // source words per row
    const int wpw = ((saw - 1 + bw + 3) >> 2) + 1; // window words per row (+1: funnel reads one past)
    const int wbytes = saw - 1 + bw;
    uint32_t *s_src = smem;
    uint32_t *s_win = smem + spw * bh;
    const int budget_rows = (smem_bytes - spw * bh * 4) / (wpw * 4);
    const int span = (bh - 1) * k + 1;
    int chunk = budget_rows - span + 1; // search rows per pass
    if (chunk > sah) chunk = sah;
    if (chunk < 1) chunk = 1; // caller guarantees enough smem for one row
    const uint32_t tail_mask = (bw & 3) ? ((1u << (8 * (bw & 3))) - 1u) : 0xffffffffu;

    __syncthreads(); // previous users of smem are done
    { // stage the source block (bytewise: arbitrary alignment)
        uint8_t *sb = reinterpret_cast<uint8_t *>(s_src);
        for (int i = tid; i < bh * spw * 4; i += NT) {
            int r = i / (spw * 4), c = i - r * (spw * 4);
            sb[i] = c < bw ? src[(size_t)r * src_stride + c] : 0;
        }
    }
    uint64_t best = ~0ull;
    for (int y0 = 0; y0 < sah; y0 += chunk) {
        const int cr = min(chunk, sah - y0);
        const int rows = cr - 1 + span;
        __syncthreads();
        {
            uint8_t *wb = reinterpret_cast<uint8_t *>(s_win);
            const int rb = wpw * 4;
            for (int i = tid; i < rows * rb; i += NT) {
                int r = i / rb, c = i - r * rb;
                wb[i] = c < wbytes ? ref[(size_t)(y0 + r) * raw_stride + c] : 0;
            }
        }
        __syncthreads();
        for (int p = tid; p < cr * saw; p += NT) {
            const int ysl = p / saw, xs = p - ysl * saw;
            const int a = xs >> 2, sh = (xs & 3) * 8;
            uint32_t sad = 0;
            for (int r = 0; r < bh; r++) {
                const uint32_t *wr = s_win + (ysl + r * k) * wpw + a;
                const uint32_t *sr = s_src + r * spw;
                uint32_t lo = wr[0];
                for (int w = 0; w < spw; w++) {
                    uint32_t hi = wr[w + 1];
                    uint32_t v = __funnelshift_r(lo, hi, sh);
                    uint32_t s = sr[w];
                    if (w == spw - 1) {
                        v &= tail_mask;
                        s &= tail_mask;
                    }
                    sad = sad4(s, v, sad);
                    lo = hi;
                }
            }
            uint64_t key = ((uint64_t)sad << 32) | (uint32_t)((y0 + ysl) * saw + xs);
            best = key < best ? key : best;
        }
    }
    best = warp_min_u64(best);
    __syncthreads();
    if ((tid & 31) == 0) s_red[tid >> 5] = best;
    __syncthreads();
    uint64_t r = s_red[0];
#pragma unroll
    for (int i = 1; i < NT / 32; i++) r = s_red[i] < r ? s_red[i] : r;
    return r;
}

// -----------------------------------------------------------------------------------------------------
// Picture-level state passed by value to the kernels
// -----------------------------------------------------------------------------------------------------
struct RawHme { // one (sb, list, ref): result of the last enabled HME level, before cross-ref logic
    int16_t x, y;
    uint32_t valid;
    uint64_t sad;
};

struct HmeState;
struct MeDev {
    SvtB200MeParams p;
    SvtB200MePlanes src;
    SvtB200MePlanes refs[2][4];
    SvtB200MeOutputs out;
    RawHme *raw; // [n_sb][2][4]
    HmeState *hstate; // [n_sb]: search centres / pruning / search-area divisors, written by the SB's last HME CTA
    unsigned int *hme_done; // [n_sb]: HME CTAs of the SB that have published their result
    unsigned int *fp_done; // [n_sb]: full-pel CTAs of the SB that have stored their results
    int sbs_x, sbs_y;
    int slot_l[8], slot_r[8], n_slots;
    int fp_smem_bytes; // dynamic shared memory given to fullpel_kernel
};

struct HmeState {
    int16_t sc_x[2][4], sc_y[2][4];
    uint64_t sad[2][4];
    uint32_t do_ref[2][4];
    uint32_t divisor[2][4];
};

// set_final_seach_centre_sb's cross-reference carry (EbMotionEstimation.c:2575-2740) +
// hme_prune_ref_and_adjust_sr (:2779-2823). Serial, tiny; run by one thread.
__device__ void derive_hme_state(const SvtB200MeParams &p, const RawHme *raw /*[2][4]*/, HmeState &h) {
    for (int l = 0; l < 2; l++)
        for (int r = 0; r < 4; r++) {
            h.sc_x[l][r] = h.sc_y[l][r] = 0;
            h.sad[l][r] = 0xFFFFFFFFull;
            h.do_ref[l][r] = 1;
            h.divisor[l][r] = 1;
        }
    uint64_t carry_sad = 0;
    for (int l = 0; l < p.num_lists; l++)
        for (int r = 0; r < p.num_refs[l]; r++) {
            const RawHme &w = raw[l * 4 + r];
            int16_t scx = 0, scy = 0;
            if (w.valid) {
                scx = w.x;
                scy = w.y;
                carry_sad = w.sad;
            }
            h.sc_x[l][r] = scx;
            h.sc_y[l][r] = scy;
            h.sad[l][r] = carry_sad;
        }
    const bool prune_ref = p.enable_hme_flag && p.enable_hme_level2_flag;
    if (prune_ref && (p.enable_me_sr_adjustment || p.enable_me_hme_ref_pruning)) {
        uint64_t best = h.sad[0][0];
        for (int l = 0; l < 2; l++)
            for (int r = 0; r < 4; r++) best = h.sad[l][r] < best ? h.sad[l][r] : best;
        const uint32_t th = (uint32_t)p.prune_ref_if_hme_sad_dev_bigger_than_th & 0xFFFFu;
        for (int l = 0; l < 2; l++)
            for (int r = 0; r < 4; r++) {
                if (p.enable_me_hme_ref_pruning && th != 0xFFFFu && (h.sad[l][r] - best) * 100 > (uint64_t)th * best)
                    h.do_ref[l][r] = 0;
                if (p.enable_me_sr_adjustment) {
                    if (abs((int)h.sc_x[l][r]) <= p.reduce_me_sr_based_on_mv_length_th &&
                        abs((int)h.sc_y[l][r]) <= p.reduce_me_sr_based_on_mv_length_th &&
                        h.sad[l][r] < (uint64_t)p.stationary_hme_sad_abs_th)
                        h.divisor[l][r] = p.stationary_me_sr_divisor;
                    else if (h.sad[l][r] < (uint64_t)p.reduce_me_sr_based_on_hme_sad_abs_th)
                        h.divisor[l][r] = p.me_sr_divisor_for_low_hme_sad;
                }
            }
    }
}

// Tail of the HME kernel (thread 0): publish this (SB, reference) result; the CTA that completes the SB derives the
// cross-reference state ONCE for the full-pel and finalize kernels (it was a serial prologue in each of their CTAs).
__device__ void hme_publish(const MeDev &d, int sb, RawHme *out, const RawHme &w) {
    *out = w;
    __threadfence();
    const unsigned int prev = atomicAdd(&d.hme_done[sb], 1u);
    if (prev + 1 == (unsigned int)d.n_slots) {
        __threadfence();
        RawHme raw[8];
        const ulonglong2 *g = reinterpret_cast<const ulonglong2 *>(d.raw + (size_t)sb * 8);
        for (int i = 0; i < 8; i++) { // L2 reads: the other CTAs' results were written by other SMs
            const ulonglong2 v = __ldcg(g + i);
            memcpy(&raw[i], &v, sizeof(RawHme));
        }
        HmeState h;
        derive_hme_state(d.p, raw, h);
        d.hstate[sb] = h;
    }
}

// ---- HME, staged regime: all (up to 2x2) search regions of a level are searched concurrently ------------------
// Per level: every region's window + the (shared) source block are staged once.  Full-width blocks (sbw == 64) use
// the aligned-task scheme of the full-pel kernel: a task is Q positions of one search row with the same byte
// alignment, x = 4Q*m + c + 4k, so that one shifted copy of the window row (W + Q - 1 SHF) feeds W*Q VABSDIFF4 and
// all loads are 8/16-byte LDS.  The rows of a task are split over `tpp` threads so that the tiny level-1/2 areas
// (8x3) still fill the CTA; every warp works for ONE region, so the per-region argmin is a warp reduction plus one
// shared 64-bit atomicMin.  Ragged blocks (picture width not a multiple of 64) take hme_level_search below.
constexpr int HME_FAST_SMEM = 64 * 1024; // the most dynamic shared memory the staged regime is launched with
constexpr int HME_SMEM_BYTES = 40 * 1024; // the chunked regime's block_search budget
struct HmeJob {
    const uint8_t *ref; // search position (0,0)
    int xo, yo, saw, sah;
    int woff, wpw; // window offset (words) in smem, words per row
    int q, gpr, t0, nt; // positions per task (2|4), task groups per row, first (padded) task id, padded task count
    uint32_t magic; // ceil(2^32 / (4 * gpr)): task id -> search row by one IMAD.HI
};

__host__ __device__ __forceinline__ int hme_pitch_words(int saw, int w, int q) {
    const int g = (saw + 4 * q - 1) / (4 * q);
    int p = (q * g + w + 3) & ~3;
    return (p & 4) ? p : p + 4;
}

template <int W, int Q>
__device__ __forceinline__ void hme_task_rows(const uint32_t *__restrict__ s_src, const uint32_t *__restrict__ wbase, int wpw, int k,
                                              int sh, int r0, int rstep, int bh, uint32_t (&acc)[Q]) {
    uint32_t a[Q][2];
#pragma unroll
    for (int q = 0; q < Q; q++) a[q][0] = a[q][1] = 0;
#pragma unroll 1
    for (int r = r0; r < bh; r += rstep) {
        uint32_t s[W], w[W + Q], f[W + Q - 1];
        const uint32_t *sp = s_src + r * W;
        const uint32_t *wp = wbase + r * k * wpw;
#pragma unroll
        for (int i = 0; i < W / 4; i++) {
            const uint4 v = reinterpret_cast<const uint4 *>(sp)[i];
            s[4 * i] = v.x, s[4 * i + 1] = v.y, s[4 * i + 2] = v.z, s[4 * i + 3] = v.w;
        }
        if (Q == 4) {
#pragma unroll
            for (int i = 0; i < (W + Q) / 4; i++) {
                const uint4 v = reinterpret_cast<const uint4 *>(wp)[i];
                w[4 * i] = v.x, w[4 * i + 1] = v.y, w[4 * i + 2] = v.z, w[4 * i + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int i = 0; i < (W + Q) / 2; i++) {
                const uint2 v = reinterpret_cast<const uint2 *>(wp)[i];
                w[2 * i] = v.x, w[2 * i + 1] = v.y;
            }
        }
#pragma unroll
        for (int i = 0; i < W + Q - 1; i++) f[i] = __funnelshift_r(w[i], w[i + 1], sh);
#pragma unroll
        for (int i = 0; i < W; i++)
#pragma unroll
            for (int q = 0; q < Q; q++) a[q][i & 1] = sad4(s[i], f[i + q], a[q][i & 1]);
    }
#pragma unroll
    for (int q = 0; q < Q; q++) acc[q] = a[q][0] + a[q][1];
}

// one task round of a warp: decode, search, reduce.  Returns this lane's best key (~0 if none): packed 32-bit
// (sad << kshift | index) when the level's SAD and index ranges fit (kshift != 0), else the index in the low word of a
// 64-bit key; the caller reduces accordingly.
template <int W, int Q>
__device__ __forceinline__ unsigned long long hme_task(const HmeJob &jb, const uint32_t *s_src, const uint32_t *smem, int u, bool live,
                                                       int k, int bh, int tpp, int sub, int kshift) {
    const int tpr = 4 * jb.gpr;
    const int ys = live ? (int)__umulhi((uint32_t)u, jb.magic) : 0; // u / tpr (u < 2^16, tpr <= 2^8: exact)
    const int rem = live ? u - ys * tpr : 0;
    const int m = rem >> 2, c = rem & 3;
    uint32_t acc[Q];
    hme_task_rows<W, Q>(s_src, smem + jb.woff + ys * jb.wpw + m * Q, jb.wpw, k, c * 8, sub, tpp, bh, acc);
    for (int o = 1; o < tpp; o <<= 1)
#pragma unroll
        for (int q = 0; q < Q; q++) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
    unsigned long long best = ~0ull;
    if (live && sub == 0) {
        const int x0 = 4 * Q * m + c;
        const uint32_t i0 = (uint32_t)(ys * jb.saw + x0);
        if (kshift) {
            uint32_t b32 = 0xffffffffu;
#pragma unroll
            for (int q = 0; q < Q; q++) b32 = min(b32, (x0 + 4 * q < jb.saw) ? (acc[q] << kshift) + i0 + 4 * q : 0xffffffffu);
            best = b32;
        } else {
#pragma unroll
            for (int q = 0; q < Q; q++) {
                const unsigned long long key = ((unsigned long long)acc[q] << 32) | (i0 + 4 * q);
                if (x0 + 4 * q < jb.saw && key < best) best = key;
            }
        }
    }
    return best;
}

// Stage `rows` rows of `nbytes` bytes (arbitrary alignment, global) into shared-memory words of pitch `wpw`; element
// i = row * wpw + word is handled by thread i mod nt.  Four independent elements per thread are loaded before the
// first is stored, so four global-load latencies overlap (the staging phases are latency-bound: ncu long_scoreboard).
__device__ __forceinline__ void stage_flat(uint32_t *dst, int wpw, const uint8_t *__restrict__ src, ptrdiff_t stride, int rows,
                                           int nbytes, int nt) {
    const int total = rows * wpw;
    int i = threadIdx.x;
    int row = i / wpw, wd = i - row * wpw;
    const int dr = nt / wpw, dw = nt - dr * wpw; // advance of (row, word) per step of nt elements: no division in the loop
    while (i < total) {
        uint32_t lo[4], hi[4];
        int sh[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            lo[u] = hi[u] = 0;
            sh[u] = 0;
            if (i + u * nt < total) {
                const uintptr_t a = (uintptr_t)(src + (ptrdiff_t)row * stride);
                const uint32_t *ga = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
                const int need = (nbytes + (int)(a & 3) + 3) >> 2; // aligned words covering the row
                if (wd < need) lo[u] = ga[wd];
                if (wd + 1 < need) hi[u] = ga[wd + 1];
                sh[u] = (int)(a & 3) * 8;
            }
            row += dr;
            wd += dw;
            if (wd >= wpw) {
                wd -= wpw;
                row++;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; u++)
            if (i + u * nt < total) dst[i + u * nt] = __funnelshift_r(lo[u], hi[u], sh[u]);
        i += 4 * nt;
    }
}

// Stage `rows` rows into shared memory with a GROUP of `gsize` (power of two) threads, `t` = index inside the group:
// a row is covered by lw = min(pow2 >= wpw, gsize) lanes, gsize / lw rows per pass, so that row and word come from
// shifts (the generic flat mapping costs two integer divisions per call, which dominated the small HME windows).
// Four rows are in flight per thread.
__device__ __forceinline__ void stage_group(uint32_t *dst, int wpw, const uint8_t *__restrict__ src, ptrdiff_t stride, int rows,
                                            int nbytes, int t, int gsize) {
    int lg = 32 - __clz(wpw - 1); // log2(pow2 >= wpw), wpw >= 2
    const int lgs = 31 - __clz(gsize);
    if (lg > lgs) lg = lgs;
    const int lw = 1 << lg, rpp = gsize >> lg, wd0 = t & (lw - 1);
    for (int row0 = t >> lg; row0 < rows; row0 += 4 * rpp) {
        for (int wd = wd0; wd < wpw; wd += lw) {
            uint32_t lo[4], hi[4];
            int sh[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int row = row0 + u * rpp;
                lo[u] = hi[u] = 0;
                sh[u] = 0;
                if (row < rows) {
                    const uintptr_t a = (uintptr_t)(src + (ptrdiff_t)row * stride);
                    const uint32_t *ga = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
                    const int need = (nbytes + (int)(a & 3) + 3) >> 2;
                    if (wd < need) lo[u] = ga[wd];
                    if (wd + 1 < need) hi[u] = ga[wd + 1];
                    sh[u] = (int)(a & 3) * 8;
                }
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int row = row0 + u * rpp;
                if (row < rows) dst[row * wpw + wd] = __funnelshift_r(lo[u], hi[u], sh[u]);
            }
        }
    }
}

template <int NT, int W>
__device__ void hme_level_search_aligned(const uint8_t *__restrict__ src, int src_stride, int raw_stride, int k, int bh,
                                         const HmeJob *jobs, int njobs, int tpp, int ntasks, int kshift, uint32_t *smem,
                                         unsigned long long *s_key) {
    const int tid = threadIdx.x;
    stage_group(smem, W, src, src_stride, bh, 4 * W, tid, NT); // the source block: all threads
    const int span = (bh - 1) * k + 1;
    { // the windows: one quarter of the CTA per search region, concurrently
        constexpr int GS = NT / 4;
        for (int j = tid / GS; j < njobs; j += 4) {
            const HmeJob jb = jobs[j];
            stage_group(smem + jb.woff, jb.wpw, jb.ref, raw_stride, jb.sah - 1 + span, jb.saw - 1 + 4 * W, tid % GS, GS);
        }
    }
    __syncthreads();
    const int ltpp = 31 - __clz(tpp); // tpp is a power of two: shifts instead of divisions
    const int sub = tid & (tpp - 1), gpt = NT >> ltpp;
    for (int g0 = 0; g0 < ntasks; g0 += gpt) {
        if (g0 + ((tid & ~31) >> ltpp) >= ntasks) continue; // warp-uniform
        const int t = g0 + (tid >> ltpp);
        int j = 0;
        while (j + 1 < njobs && t >= jobs[j + 1].t0) j++; // warp-uniform: task ranges are padded to whole warps
        const HmeJob jb = jobs[j];
        const int u = t - jb.t0;
        const bool live = u < jb.sah * 4 * jb.gpr;
        unsigned long long best = jb.q == 4 ? hme_task<W, 4>(jb, smem, smem, u, live, k, bh, tpp, sub, kshift)
                                            : hme_task<W, 2>(jb, smem, smem, u, live, k, bh, tpp, sub, kshift);
        if (kshift) {
            const uint32_t m32 = __reduce_min_sync(0xffffffffu, (uint32_t)best);
            best = m32 == 0xffffffffu ? ~0ull : ((unsigned long long)(m32 >> kshift) << 32) | (m32 & ((1u << kshift) - 1u));
        } else {
            best = warp_min_u64(best);
        }
        if ((tid & 31) == 0 && best != ~0ull) atomicMin(&s_key[j], best);
    }
    __syncthreads();
}

// ragged-width fallback: one job after the other, word-granular loads, tail mask
template <int NT>
__device__ void hme_level_search(const uint8_t *__restrict__ src, int src_stride, int raw_stride, int k, int bw, int bh,
                                 const HmeJob *jobs, int njobs, uint32_t *smem, unsigned long long *s_key) {
    const int tid = threadIdx.x;
    const int spw = (bw + 3) >> 2;
    uint32_t *s_src = smem;
    const uint32_t tail_mask = (bw & 3) ? ((1u << (8 * (bw & 3))) - 1u) : 0xffffffffu;
    stage_rows_n(s_src, spw, src, src_stride, bh, bw, NT / 32); // the source block, once for all jobs
    const int span = (bh - 1) * k + 1;
    for (int j = 0; j < njobs; j++) {
        const HmeJob jb = jobs[j];
        stage_rows_n(smem + jb.woff, jb.wpw, jb.ref, raw_stride, jb.sah - 1 + span, jb.saw - 1 + bw, NT / 32);
    }
    __syncthreads();
    for (int j = 0; j < njobs; j++) {
        const HmeJob jb = jobs[j];
        const int P = jb.saw * jb.sah;
        int tpp = 1;
        while (tpp * 2 * P <= NT && tpp * 2 <= 32 && tpp * 2 <= bh) tpp *= 2;
        const int sub = tid & (tpp - 1), gpt = NT / tpp;
        const uint32_t *s_win = smem + jb.woff;
        unsigned long long best = ~0ull;
        for (int g0 = 0; g0 < P; g0 += gpt) { // uniform trip count: all lanes join the shuffles
            const int g = g0 + tid / tpp;
            const bool live = g < P;
            uint32_t sad = 0;
            int ys = 0, xs = 0;
            if (live) {
                ys = g / jb.saw;
                xs = g - ys * jb.saw;
                const int a = xs >> 2, sh = (xs & 3) * 8;
                for (int r = sub; r < bh; r += tpp) {
                    const uint32_t *wr = s_win + (ys + r * k) * jb.wpw + a;
                    const uint32_t *sr = s_src + r * spw;
                    uint32_t lo = wr[0];
                    for (int w = 0; w < spw; w++) {
                        const uint32_t hi = wr[w + 1];
                        uint32_t v = __funnelshift_r(lo, hi, sh), sv = sr[w];
                        if (w == spw - 1) {
                            v &= tail_mask;
                            sv &= tail_mask;
                        }
                        sad = sad4(sv, v, sad);
                        lo = hi;
                    }
                }
            }
            for (int o = 1; o < tpp; o <<= 1) sad += __shfl_xor_sync(0xffffffffu, sad, o);
            if (live && sub == 0) {
                const unsigned long long key = ((unsigned long long)sad << 32) | (uint32_t)g;
                best = key < best ? key : best;
            }
        }
        best = warp_min_u64(best);
        if ((tid & 31) == 0 && best != ~0ull) atomicMin(&s_key[j], best);
    }
    __syncthreads();
}

// Staged regime, lanes 0..3 (one per search region; `jl`: the region exists) after the region's window is in `jb`:
// window pitch and offset (words) after the source block, task ranges padded to whole warps, rows-per-task split and
// key packing.  Prefix sums / maxima over the four lanes by shuffles (no serial section, one barrier).
__device__ __forceinline__ void hme_task_layout(HmeJob &jb, bool jl, int bw, int bh, int k, bool aligned, int &s_tpp, int &s_ntasks,
                                                int &s_kshift) {
    const int tid = threadIdx.x;
    if (jl) {
        jb.q = (jb.saw & 15) ? 2 : 4;
        jb.gpr = (jb.saw + 4 * jb.q - 1) / (4 * jb.q);
        jb.magic = (uint32_t)((0x100000000ull + 4 * jb.gpr - 1) / (4 * jb.gpr));
        jb.wpw = aligned ? hme_pitch_words(jb.saw, bw >> 2, jb.q) : ((jb.saw - 1 + bw + 3) >> 2) + 1;
    }
    const unsigned m4 = 0xfu;
    const int wsz = jl ? jb.wpw * (jb.sah - 1 + (bh - 1) * k + 1) : 0;
    int inc = wsz, v = __shfl_up_sync(m4, inc, 1);
    if (tid >= 1) inc += v;
    v = __shfl_up_sync(m4, inc, 2);
    if (tid >= 2) inc += v;
    jb.woff = ((bw + 3) >> 2) * bh + inc - wsz;
    const int T = jl ? jb.sah * 4 * jb.gpr : 0;
    int tpp = 32, tot = 0;
    for (;; tpp >>= 1) {
        const int pad = 32 / tpp;
        jb.nt = (T + pad - 1) & ~(pad - 1);
        inc = jb.nt;
        v = __shfl_up_sync(m4, inc, 1);
        if (tid >= 1) inc += v;
        v = __shfl_up_sync(m4, inc, 2);
        if (tid >= 2) inc += v;
        tot = __shfl_sync(m4, inc, 3);
        jb.t0 = inc - jb.nt;
        if (tpp == 1 || (tpp <= bh && tot * tpp <= NT_SEARCH)) break; // same decision in all four lanes
    }
    int maxp = jl ? jb.saw * jb.sah : 1;
    maxp = max(maxp, __shfl_xor_sync(m4, maxp, 1));
    maxp = max(maxp, __shfl_xor_sync(m4, maxp, 2));
    if (tid == 0) {
        s_tpp = tpp;
        s_ntasks = tot;
        // packed 32-bit keys when (largest SAD of the level, largest position index) fit together
        const int ibits = 32 - __clz(maxp - 1 > 0 ? maxp - 1 : 1);
        const int sbits = 32 - __clz(255 * bw * bh);
        s_kshift = (ibits + sbits <= 31) ? ibits : 0;
    }
}

// Kernel A: hierarchical ME, one CTA per (SB, reference).  hme_level_0/1/2 (:852-1318) for the search regions, then the
// region choice of set_final_seach_centre_sb.  Per level, lanes 0..3 place one region's window each (hme_window), the
// CTA searches every region, and lanes 0..3 turn each region's key into its centre.  Only the search differs between the
// regimes (me_launch_plan picks one per picture):
//   STAGED:  every region's window is in shared memory at once: hme_level_search_aligned<W>, or hme_level_search for
//            ragged picture widths;
//   chunked: block_search runs the regions one after another, each window chunked through HME_SMEM_BYTES.
// One body, two kernels, because the regimes need different launch bounds: the chunked kernel gives no minimum of CTAs
// per SM (with one, even of 1, its call took 9 % longer at 1920x1080 preset 1 on an H100 SXM at 700 W).
template <bool STAGED>
__device__ __forceinline__ void hme_sb(const MeDev &d) {
    extern __shared__ uint4 smem4[];
    uint32_t *smem = reinterpret_cast<uint32_t *>(smem4);
    __shared__ HmeJob s_jobs[4];
    __shared__ int s_tpp, s_ntasks, s_kshift;
    __shared__ unsigned long long s_key[4];
    __shared__ int s_cx[4], s_cy[4];
    __shared__ unsigned long long s_csad[4];
    const SvtB200MeParams &p = d.p;
    const int tid = threadIdx.x;
    const int sb = blockIdx.x, slot = blockIdx.y;
    const int l = d.slot_l[slot], r = d.slot_r[slot];
    RawHme *out = d.raw + (size_t)sb * 8 + l * 4 + r;
    const bool active = (p.temporal_layer_index > 0 || l == 0) && p.enable_hme_flag &&
                        (p.enable_hme_level0_flag || p.enable_hme_level1_flag || p.enable_hme_level2_flag);
    if (!active) {
        if (tid == 0) {
            RawHme z = {0, 0, 0, 0};
            hme_publish(d, sb, out, z);
        }
        return;
    }
    const int sx = sb % d.sbs_x, sy = sb / d.sbs_x;
    const int ox = sx * 64, oy = sy * 64;
    const int sbw = min(p.full.width - ox, 64), sbh = min(p.full.height - oy, 64);
    const int sub = p.hme_search_method != 0;
    const bool aligned = sbw == 64; // block rows are whole 16-byte groups at every level
    const int mult = scaled_dist(p.ref_dist[l][r]) * 100;
    const int nrw = p.number_hme_search_region_in_width, nrh = p.number_hme_search_region_in_height;
    const int njobs = nrw * nrh;
    const SvtB200MePlanes &rp = d.refs[l][r];
    if (tid < 4) {
        s_cx[tid] = s_cy[tid] = 0;
        s_csad[tid] = 0;
    }
    for (int level = 0; level < 3; level++) {
        const bool on = level == 0 ? p.enable_hme_level0_flag : level == 1 ? p.enable_hme_level1_flag : p.enable_hme_level2_flag;
        if (!on) continue;
        const SvtB200Plane &pl = level == 0 ? p.sixteenth : level == 1 ? p.quarter : p.full;
        const int shf = 2 - level;
        const int o_x = ox >> shf, o_y = oy >> shf, bw = sbw >> shf, bh0 = sbh >> shf;
        const int bh = sub ? bh0 >> 1 : bh0, k = sub ? 2 : 1;
        const uint8_t *srcp = level == 0 ? d.src.sixteenth : level == 1 ? d.src.quarter : d.src.full;
        const uint8_t *refp = level == 0 ? rp.sixteenth : level == 1 ? rp.quarter : rp.full;
        __syncthreads(); // previous level's results (s_cx/s_cy) are final; smem free
        if (tid < 4) { // one lane per search region, in (ry outer, rx inner) order
            const bool jl = tid < njobs;
            HmeJob jb;
            memset(&jb, 0, sizeof(jb));
            if (jl) {
                const HmeWindow w = hme_window(p, level, tid % nrw, tid / nrw, mult, s_cx[tid], s_cy[tid], ox, oy);
                jb.ref = refp + (size_t)(pl.origin_y + o_y + w.yo) * pl.stride + pl.origin_x + o_x + w.xo;
                jb.xo = w.xo;
                jb.yo = w.yo;
                jb.saw = w.saw;
                jb.sah = w.sah;
            }
            if (STAGED) hme_task_layout(jb, jl, bw, bh, k, aligned, s_tpp, s_ntasks, s_kshift);
            if (jl) {
                s_jobs[tid] = jb;
                s_key[tid] = ~0ull;
            }
        }
        __syncthreads();
        const uint8_t *s = srcp + (size_t)(pl.origin_y + o_y) * pl.stride + pl.origin_x + o_x;
        const int sstr = sub ? pl.stride * 2 : pl.stride;
        if constexpr (STAGED) {
            if (!aligned)
                hme_level_search<NT_SEARCH>(s, sstr, pl.stride, k, bw, bh, s_jobs, njobs, smem, s_key);
            else if (level == 0)
                hme_level_search_aligned<NT_SEARCH, 4>(s, sstr, pl.stride, k, bh, s_jobs, njobs, s_tpp, s_ntasks, s_kshift, smem, s_key);
            else if (level == 1)
                hme_level_search_aligned<NT_SEARCH, 8>(s, sstr, pl.stride, k, bh, s_jobs, njobs, s_tpp, s_ntasks, s_kshift, smem, s_key);
            else
                hme_level_search_aligned<NT_SEARCH, 16>(s, sstr, pl.stride, k, bh, s_jobs, njobs, s_tpp, s_ntasks, s_kshift, smem, s_key);
        } else {
            __shared__ uint64_t s_red[NT_SEARCH / 32];
            for (int j = 0; j < njobs; j++) {
                const uint64_t key = block_search<NT_SEARCH>(s, sstr, s_jobs[j].ref, pl.stride, k, bw, bh, s_jobs[j].saw, s_jobs[j].sah,
                                                             smem, HME_SMEM_BYTES, s_red);
                if (tid == 0) s_key[j] = key;
            }
            __syncthreads();
        }
        if (tid < njobs) {
            const unsigned long long key = s_key[tid];
            const uint32_t sad = (uint32_t)(key >> 32), idx = (uint32_t)key;
            int kx = 0, ky = 0;
            unsigned long long lsad = 0xffffff; // svt_sad_loop_kernel_c start value; centre untouched if never beaten
            if (sad < 0xffffffu) {
                lsad = sad;
                kx = idx % s_jobs[tid].saw;
                ky = idx / s_jobs[tid].saw;
            }
            const int scale = level == 0 ? 4 : level == 1 ? 2 : 1;
            s_csad[tid] = sub ? lsad * 2 : lsad;
            s_cx[tid] = (int16_t)((kx + s_jobs[tid].xo) * scale);
            s_cy[tid] = (int16_t)((ky + s_jobs[tid].yo) * scale);
        }
    }
    __syncthreads();
    if (tid == 0) { // set_final_seach_centre_sb: region (0,0) first, then strict `<` in (ry outer, rx inner) order
        unsigned long long bs = s_csad[0];
        int bx = s_cx[0], by = s_cy[0];
        for (int j = 1; j < njobs; j++)
            if (s_csad[j] < bs) {
                bs = s_csad[j];
                bx = s_cx[j];
                by = s_cy[j];
            }
        RawHme w;
        w.x = (int16_t)bx;
        w.y = (int16_t)by;
        w.valid = 1;
        w.sad = bs;
        hme_publish(d, sb, out, w);
    }
}
__global__ void __launch_bounds__(NT_SEARCH, 6) hme_kernel_staged(const __grid_constant__ MeDev d) { hme_sb<true>(d); }
__global__ void __launch_bounds__(NT_SEARCH) hme_kernel_chunked(const __grid_constant__ MeDev d) { hme_sb<false>(d); }

// -----------------------------------------------------------------------------------------------------
// SB epilogue: me_prune_ref (:2145-2199), construct_me_candidate_array (:2825-2905), MeSbResults (:2964-3040).
// Run by the LAST full-pel CTA of the SB (all blockDim.x threads; `sm` = >= 640 bytes of free shared memory).
// Results of the other references were written by other SMs in this same launch: read them through L2 (__ldcg).
// -----------------------------------------------------------------------------------------------------
__device__ void finalize_sb(const MeDev &d, int sb, uint32_t *sm) {
    HmeState &s_h = *reinterpret_cast<HmeState *>(sm); // 160 B
    uint32_t *s_first = sm + 40; // [85]
    uint32_t *s_refsad = sm + 128; // [8]: sum of the 64 8x8 SADs per reference (< 2^26)
    const SvtB200MeParams &p = d.p;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31;
    const uint32_t *bsad = d.out.best_sad + (size_t)sb * 2 * 4 * 85;
    const uint32_t *bmv = d.out.best_mv + (size_t)sb * 2 * 4 * 85;
    if (tid == 0) s_h = d.hstate[sb];
    if (tid < 8) s_refsad[tid] = 0;
    __syncthreads();
    const bool prune = p.enable_hme_flag && p.enable_hme_level2_flag && p.enable_me_hme_ref_pruning;
    if (prune) {
        for (int i = tid; i < 8 * 64; i += nt) { // warp-uniform slot: 64 consecutive items per reference
            const int slot = i >> 6, l = slot >> 2, r = slot & 3;
            uint32_t v = 0;
            if (l < p.num_lists && r < p.num_refs[l] && s_h.do_ref[l][r]) v = __ldcg(bsad + slot * 85 + 21 + (i & 63));
            v = __reduce_add_sync(0xffffffffu, v);
            if (lane == 0 && v) atomicAdd(&s_refsad[slot], v);
        }
        __syncthreads();
    }
    if (tid == 0) {
        if (prune) {
            for (int l = 0; l < p.num_lists; l++)
                for (int r = 0; r < p.num_refs[l]; r++)
                    s_h.sad[l][r] = s_h.do_ref[l][r] ? (uint64_t)s_refsad[l * 4 + r] : (uint64_t)kMaxSadValue * 64;
            uint64_t best = s_h.sad[0][0];
            for (int l = 0; l < 2; l++)
                for (int r = 0; r < 4; r++) best = s_h.sad[l][r] < best ? s_h.sad[l][r] : best;
            const uint32_t th = (uint32_t)p.prune_ref_if_me_sad_dev_bigger_than_th & 0xFFFFu;
            for (int l = 0; l < 2; l++)
                for (int r = 0; r < 4; r++)
                    if (th != 0xFFFFu && (s_h.sad[l][r] - best) * 100 > (uint64_t)th * best) s_h.do_ref[l][r] = 0;
        }
        for (int l = 0; l < 2; l++)
            for (int r = 0; r < 4; r++) {
                SvtB200HmeResult o;
                o.sc_x = s_h.sc_x[l][r];
                o.sc_y = s_h.sc_y[l][r];
                o.do_ref = s_h.do_ref[l][r];
                o.hme_sad = s_h.sad[l][r];
                d.out.hme[(size_t)sb * 8 + l * 4 + r] = o;
            }
    }
    __syncthreads();
    for (int pu = tid; pu < 85; pu += nt) {
        uint8_t *cand = d.out.me_cand + ((size_t)sb * 85 + pu) * 23;
        int16_t *mv = d.out.me_mv + ((size_t)sb * 85 + pu) * 7 * 2;
        for (int i = 0; i < 23; i++) cand[i] = 0;
        for (int i = 0; i < 14; i++) mv[i] = 0;
        uint32_t first = 0;
        int n = 0;
        if (pu < p.max_number_of_pus_per_sb) {
            const int n_idx = pu > 20 ? c_tab8[pu - 21] + 21 : pu > 4 ? c_tab16[pu - 5] + 5 : pu;
            for (int l = 0; l < p.num_lists; l++)
                for (int r = 0; r < p.num_refs[l]; r++) {
                    if (!s_h.do_ref[l][r]) continue;
                    if (n == 0) first = __ldcg(bsad + (l * 4 + r) * 85 + n_idx);
                    if (n < 23) cand[n] = (uint8_t)(l | (l == 0 ? (r << 2) : (r << 4)) | (l == 1 ? 0x80 : 0));
                    n++;
                }
            if (p.num_lists > 1) {
                for (int a = 0; a < p.num_refs[0]; a++)
                    for (int b = 0; b < p.num_refs[1]; b++)
                        if (s_h.do_ref[0][a] && s_h.do_ref[1][b]) {
                            if (n < 23) cand[n] = (uint8_t)(2 | (a << 2) | (b << 4) | 0x80);
                            n++;
                        }
                for (int a = 1; a < p.num_refs[0]; a++)
                    if (s_h.do_ref[0][0] && s_h.do_ref[0][a]) {
                        if (n < 23) cand[n] = (uint8_t)(2 | (a << 4));
                        n++;
                    }
                if (p.num_refs[1] == 3 && s_h.do_ref[1][0] && s_h.do_ref[1][2]) {
                    if (n < 23) cand[n] = (uint8_t)(2 | (2 << 4) | 0x40 | 0x80);
                    n++;
                }
            }
            for (int l = 0; l < p.num_lists; l++)
                for (int r = 0; r < p.num_refs[l]; r++) {
                    const uint32_t v = __ldcg(bmv + (l * 4 + r) * 85 + n_idx);
                    const int s = (l ? 4 : 0) + r;
                    mv[2 * s] = (int16_t)(v & 0xffff);
                    mv[2 * s + 1] = (int16_t)(v >> 16);
                }
        }
        d.out.total_cand[(size_t)sb * 85 + pu] = (uint8_t)min(n, 23);
        s_first[pu] = first;
    }
    __syncthreads();
    if (tid < 32) { // rc_me_distortion: sum of the first candidate's 8x8 (or 16x16) SADs
        uint32_t rc = 0;
        if (p.rc_dist_from_8x8)
            rc = s_first[21 + tid] + s_first[21 + 32 + tid];
        else if (tid < 16)
            rc = s_first[5 + tid];
        rc = __reduce_add_sync(0xffffffffu, rc);
        if (tid == 0) d.out.rc_me_distortion[sb] = rc;
    }
}

// -----------------------------------------------------------------------------------------------------
// Kernel B: integer full-pel search (integer_search_sb :1868-2139 + open_loop_me_fullpel_search_sblock)
//
// Work decomposition.  A "task" is FOUR search positions of one search row that share their byte alignment:
// x = 16m + c + 4k (k = 0..3).  Per 64-pixel source row the task loads the 16 source words (4 LDS.128) and the 20
// window words starting at word 4m (5 LDS.128, 16-byte aligned), forms the 19 words of the window shifted by c bytes
// (one SHF each) and feeds them to 64 VABSDIFF4: the shifted stream is shared by the four positions, so the inner
// loop is 1.44 issue slots per VABSDIFF4.  The 8x8 SADs of a band of eight blocks live in 32 accumulators; 16x16,
// 32x32 and 64x64 SADs are their sums (ext_all_sad_calculation_8x8_16x16 / ext_eight_sad_calculation_32x32_64x64).
// Positions that do not exist (x >= saw, dead lanes) start their 8x8 accumulators at BIAS = one more than the
// largest 8x8 SAD, so at every level (4x, 16x, 64x BIAS) they lose against any real position without a select.
// First-minimum-in-raster-order = argmin of the packed key (sad << SH) + index: REDUX.MIN per PU, then the lane
// that owns the PU keeps the running minimum in a register; one shared atomicMin per lane per task round.
// -----------------------------------------------------------------------------------------------------
constexpr int FP_SMEM_BYTES = 96 * 1024;

__host__ __device__ __forceinline__ int fp_pitch_words(int saw) {
    const int w = 4 * ((saw + 15) >> 4) + 20;
    return (w & 4) ? w : w + 4; // odd number of 16-byte units: consecutive rows start in different banks
}

template <bool SUB>
__global__ void __launch_bounds__(NT_SEARCH, 2) fullpel_kernel(const __grid_constant__ MeDev d) {
    extern __shared__ uint4 smem4[];
    uint32_t *smem = reinterpret_cast<uint32_t *>(smem4);
    __shared__ unsigned long long s_best[85]; // (sad << 32 | raster index) over the whole window
    __shared__ unsigned int s_cbest[85]; // (sad << SH | index inside the current chunk)
    __shared__ uint32_t s_sad2[2];
    constexpr int SH = SUB ? 12 : 11; // SUB keeps the un-doubled SAD (19 bits) in the key
    constexpr uint32_t BIAS = SUB ? 8192u : 16384u;
    constexpr int NR = SUB ? 4 : 8, KR = SUB ? 2 : 1; // rows summed per 8x8, window rows per summed row
    constexpr int NSRC = SUB ? 32 : 64;
    const SvtB200MeParams &p = d.p;
    const int tid = threadIdx.x, lane = tid & 31, nt = blockDim.x; // nt: 64..256, chosen by the host (load balance)
    const int sb = blockIdx.x, slot = blockIdx.y;
    const int l = d.slot_l[slot], r = d.slot_r[slot];
    uint32_t *o_sad = d.out.best_sad + ((size_t)(sb * 2 + l) * 4 + r) * 85;
    uint32_t *o_mv = d.out.best_mv + ((size_t)(sb * 2 + l) * 4 + r) * 85;

    const HmeState &hs = d.hstate[sb]; // derived once per SB by the last HME CTA (hme_publish)
    if (!hs.do_ref[l][r]) { // pruned by HME: the reference skips the search; slots are defined as 0
        for (int i = tid; i < 85; i += nt) {
            o_sad[i] = 0;
            o_mv[i] = 0;
        }
    } else {
    const int sx = sb % d.sbs_x, sy = sb / d.sbs_x;
    const int ox = sx * 64, oy = sy * 64;
    const SvtB200Plane &fp = p.full;
    const int pic_w = fp.width, pic_h = fp.height;
    const int sbw = min(pic_w - ox, 64), sbh = min(pic_h - oy, 64);
    const uint8_t *srcb = d.src.full + (size_t)(fp.origin_y + oy) * fp.stride + fp.origin_x + ox;
    const uint8_t *refb = d.refs[l][r].full + (size_t)(fp.origin_y + oy) * fp.stride + fp.origin_x + ox;

    int xsc = hs.sc_x[l][r], ysc = hs.sc_y[l][r];
    const int2 area = fp_search_area(p, scaled_dist(p.ref_dist[l][r]));
    const int dv = (int)hs.divisor[l][r];
    int saw = (int16_t)fp_window_width((int16_t)area.x / dv);
    int sah = (int16_t)max(1, (int16_t)area.y / dv);

    // ---- stage the source rows that take part in the SAD (even rows only with sub-sampling) ----
    uint32_t *s_src = smem; // [NSRC][16 words]
    uint32_t *s_win = smem + NSRC * 16;
    if (tid == 0) s_sad2[0] = s_sad2[1] = 0;
    for (int i = tid; i < 85; i += nt) s_best[i] = ((unsigned long long)kMaxSadValue << 32) | 0xffffffffull;
    stage_flat(s_src, 16, srcb, (ptrdiff_t)KR * fp.stride, NSRC, 64, nt);
    __syncthreads();

    if ((xsc != 0 || ysc != 0) && p.is_used_as_reference_flag) { // check_00_center :1348-1421 (even rows, SAD << 1)
        int cx = xsc, cy = ysc;
        if (ox + cx < -63) cx = -63 - ox;
        if (ox + cx > fp.width - 1) cx = cx - ((ox + cx) - (fp.width - 1));
        if (oy + cy < -63) cy = -63 - oy;
        if (oy + cy > fp.height - 1) cy = cy - ((oy + cy) - (fp.height - 1));
        const uint8_t *rh = refb + (ptrdiff_t)cy * fp.stride + cx;
        uint32_t z = 0, h = 0;
        const int rows = sbh >> 1, nw = (sbw + 3) >> 2;
        for (int i = tid; i < rows * nw; i += nt) { // one source word (4 samples) against both candidates
            const int rr = i / nw, wq = i - rr * nw;
            const uint32_t mask = (4 * wq + 4 > sbw) ? (1u << (8 * (sbw - 4 * wq))) - 1u : 0xffffffffu;
            const uint32_t sv = s_src[(SUB ? rr : 2 * rr) * 16 + wq] & mask;
            const uintptr_t a0 = (uintptr_t)(refb + (ptrdiff_t)rr * 2 * fp.stride + 4 * wq);
            const uintptr_t a1 = (uintptr_t)(rh + (ptrdiff_t)rr * 2 * fp.stride + 4 * wq);
            const uint32_t *g0 = reinterpret_cast<const uint32_t *>(a0 & ~(uintptr_t)3);
            const uint32_t *g1 = reinterpret_cast<const uint32_t *>(a1 & ~(uintptr_t)3);
            const uint32_t v0 = __funnelshift_r(g0[0], (a0 & 3) ? g0[1] : 0u, (int)(a0 & 3) * 8);
            const uint32_t v1 = __funnelshift_r(g1[0], (a1 & 3) ? g1[1] : 0u, (int)(a1 & 3) * 8);
            z = sad4(sv, v0 & mask, z);
            h = sad4(sv, v1 & mask, h);
        }
        z = __reduce_add_sync(0xffffffffu, z);
        h = __reduce_add_sync(0xffffffffu, h);
        if (lane == 0) {
            atomicAdd(&s_sad2[0], z);
            atomicAdd(&s_sad2[1], h);
        }
        __syncthreads();
        if (s_sad2[0] <= s_sad2[1]) cx = cy = 0; // (sad<<1) on both sides, zero wins ties
        xsc = cx;
        ysc = cy;
    }
    int xo = xsc - (saw >> 1), yo = ysc - (sah >> 1);
    clamp_window(ox, 63, pic_w, xo, saw);
    saw = saw < 8 ? saw : saw & ~0x07;
    clamp_window(oy, 63, pic_h, yo, sah);

    const int span = SUB ? 63 : 64;
    const int wbytes = saw + 63;
    const int wpw = fp_pitch_words(saw);
    const int budget_rows = (d.fp_smem_bytes - NSRC * 64) / (wpw * 4);
    int chunk = min(sah, budget_rows - span + 1);
    chunk = min(chunk, 2048 / saw); // chunk-local position index must fit 11 bits
    if (chunk < 1) chunk = 1;
    const int tpr = 4 * ((saw + 15) >> 4); // tasks per search row

    // which PU this lane owns in the lane-resident running minima
    int pu8[2], puh = -1;
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int by8 = 4 * h + (lane >> 3), bx8 = lane & 7;
        pu8[h] = 21 + 4 * c_tab16[(by8 >> 1) * 4 + (bx8 >> 1)] + (by8 & 1) * 2 + (bx8 & 1);
    }
    if (lane < 16)
        puh = 5 + c_tab16[lane];
    else if (lane < 20)
        puh = 1 + (lane - 16);
    else if (lane == 20)
        puh = 0;

    for (int y0 = 0; y0 < sah; y0 += chunk) {
        const int cr = min(chunk, sah - y0);
        const int rows = cr - 1 + span;
        __syncthreads();
        stage_flat(s_win, wpw, refb + (ptrdiff_t)(yo + y0) * fp.stride + xo, fp.stride, rows, wbytes, nt);
        for (int i = tid; i < 85; i += nt) s_cbest[i] = 0xffffffffu;
        __syncthreads();
        const int ntasks = cr * tpr;
        for (int qb = 0; qb < ntasks; qb += nt) {
            if (qb + (tid & ~31) >= ntasks) continue; // whole warp has no task: reductions are per warp
            const int t = qb + tid;
            const bool live = t < ntasks;
            const int ysl = live ? t / tpr : 0;
            const int rem = live ? t - ysl * tpr : 0;
            const int x0 = (rem >> 2) * 16 + (rem & 3);
            const int sh = (rem & 3) * 8;
            uint32_t idx[4], bias[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                idx[k] = (uint32_t)(ysl * saw + x0 + 4 * k); // index inside the chunk (< 2048 when valid)
                bias[k] = (live && x0 + 4 * k < saw) ? 0u : BIAS;
            }
            const uint32_t *wbase = s_win + ysl * wpw + (rem >> 2) * 4;
            uint32_t best8 = 0xffffffffu, besth = 0xffffffffu;
            uint32_t a64[4] = {0, 0, 0, 0}, a32[4][2] = {{0, 0}, {0, 0}, {0, 0}, {0, 0}};
            for (int bp = 0; bp < 4; bp++) { // pairs of 8-row bands = rows of 16x16 blocks
                uint32_t a16[4][4];
#pragma unroll
                for (int k = 0; k < 4; k++)
#pragma unroll
                    for (int j = 0; j < 4; j++) a16[k][j] = 0;
#pragma unroll
                for (int bb = 0; bb < 2; bb++) {
                    const int band = 2 * bp + bb;
                    uint32_t a8[4][8];
#pragma unroll
                    for (int k = 0; k < 4; k++)
#pragma unroll
                        for (int j = 0; j < 8; j++) a8[k][j] = bias[k];
                    const uint32_t *srow = s_src + band * NR * 16;
                    const uint32_t *wrow = wbase + band * 8 * wpw;
#pragma unroll
                    for (int rr = 0; rr < NR; rr++) {
                        const uint4 *sp = reinterpret_cast<const uint4 *>(srow + rr * 16);
                        const uint4 *wp = reinterpret_cast<const uint4 *>(wrow + rr * KR * wpw);
                        uint32_t s[16], w[20], f[19];
#pragma unroll
                        for (int i = 0; i < 4; i++) {
                            const uint4 v = sp[i];
                            s[4 * i] = v.x, s[4 * i + 1] = v.y, s[4 * i + 2] = v.z, s[4 * i + 3] = v.w;
                        }
#pragma unroll
                        for (int i = 0; i < 5; i++) {
                            const uint4 v = wp[i];
                            w[4 * i] = v.x, w[4 * i + 1] = v.y, w[4 * i + 2] = v.z, w[4 * i + 3] = v.w;
                        }
#pragma unroll
                        for (int i = 0; i < 19; i++) f[i] = __funnelshift_r(w[i], w[i + 1], sh);
#pragma unroll
                        for (int i = 0; i < 16; i++)
#pragma unroll
                            for (int k = 0; k < 4; k++) a8[k][i >> 1] = sad4(s[i], f[i + k], a8[k][i >> 1]);
                    }
                    const int lrel = lane - ((band & 3) << 3);
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        uint32_t bk = min(min((a8[0][j] << SH) + idx[0], (a8[1][j] << SH) + idx[1]),
                                          min((a8[2][j] << SH) + idx[2], (a8[3][j] << SH) + idx[3]));
                        const uint32_t m = __reduce_min_sync(0xffffffffu, bk);
                        if (lrel == j) best8 = min(best8, m);
#pragma unroll
                        for (int k = 0; k < 4; k++) a16[k][j >> 1] += a8[k][j];
                    }
                    if (band & 3) {
                        if ((band & 3) == 3) { // a half of the SB is complete: hand its 32 8x8 minima over
                            atomicMin(&s_cbest[pu8[band >> 2]], best8);
                            best8 = 0xffffffffu;
                        }
                    }
                }
                const int lrel16 = lane - 4 * bp;
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    uint32_t bk = min(min((a16[0][j] << SH) + idx[0], (a16[1][j] << SH) + idx[1]),
                                      min((a16[2][j] << SH) + idx[2], (a16[3][j] << SH) + idx[3]));
                    const uint32_t m = __reduce_min_sync(0xffffffffu, bk);
                    if (lrel16 == j) besth = min(besth, m);
#pragma unroll
                    for (int k = 0; k < 4; k++) a32[k][j >> 1] += a16[k][j];
                }
                if (bp & 1) {
                    const int lrel32 = lane - 16 - (bp >> 1) * 2;
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        uint32_t bk = min(min((a32[0][j] << SH) + idx[0], (a32[1][j] << SH) + idx[1]),
                                          min((a32[2][j] << SH) + idx[2], (a32[3][j] << SH) + idx[3]));
                        const uint32_t m = __reduce_min_sync(0xffffffffu, bk);
                        if (lrel32 == j) besth = min(besth, m);
#pragma unroll
                        for (int k = 0; k < 4; k++) {
                            a64[k] += a32[k][j];
                            a32[k][j] = 0;
                        }
                    }
                }
            }
            {
                uint32_t bk = min(min((a64[0] << SH) + idx[0], (a64[1] << SH) + idx[1]),
                                  min((a64[2] << SH) + idx[2], (a64[3] << SH) + idx[3]));
                const uint32_t m = __reduce_min_sync(0xffffffffu, bk);
                if (lane == 20) besth = min(besth, m);
            }
            if (puh >= 0) atomicMin(&s_cbest[puh], besth);
        }
        __syncthreads();
        // merge the chunk into the running best: chunks advance in raster order, so strict `<` on the SAD keeps
        // the first minimum
        for (int i = tid; i < 85; i += nt) {
            const unsigned int c = s_cbest[i];
            if (c != 0xffffffffu) {
                const unsigned long long sadc = SUB ? (unsigned long long)(c >> SH) << 1 : (unsigned long long)(c >> SH);
                if (sadc < (s_best[i] >> 32)) s_best[i] = (sadc << 32) | (unsigned int)(y0 * saw + (c & 2047u));
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < 85; i += nt) {
        const unsigned long long key = s_best[i];
        const uint32_t sad = (uint32_t)(key >> 32), idx = (uint32_t)key;
        uint32_t mv = 0;
        if (idx != 0xffffffffu) {
            const int ys = idx / saw, xs = idx - ys * saw;
            // (y<<18)|(uint16)(x<<2) and the 8-point variant both equal this packing (see DESIGN.md §ME)
            mv = ((uint32_t)(uint16_t)((yo + ys) * 4) << 16) | (uint16_t)((xo + xs) * 4);
        }
        o_sad[i] = sad;
        o_mv[i] = mv;
    }
    } // searched reference
    // the SB's last full-pel CTA runs the SB epilogue (was a separate, latency-bound launch)
    __threadfence();
    __syncthreads();
    if (tid == 0) s_sad2[0] = (atomicAdd(&d.fp_done[sb], 1u) + 1u == (unsigned int)d.n_slots);
    __syncthreads();
    if (s_sad2[0]) {
        __threadfence();
        finalize_sb(d, sb, smem);
    }
}


// -----------------------------------------------------------------------------------------------------
// Small kernels behind the RTCD drop-ins (single block worth of work each; fidelity, not throughput)
// -----------------------------------------------------------------------------------------------------
struct SadLoopArgs {
    const uint8_t *src, *ref;
    int src_stride, raw_stride, k, bw, bh, saw, sah;
    uint64_t *out; // [0] key
    int smem_bytes;
};
__global__ void __launch_bounds__(NT_SEARCH) sad_loop_kernel(const SadLoopArgs a) {
    extern __shared__ uint32_t smem[];
    __shared__ uint64_t s_red[NT_SEARCH / 32];
    uint64_t key = block_search<NT_SEARCH>(a.src, a.src_stride, a.ref, a.raw_stride, a.k, a.bw, a.bh, a.saw, a.sah,
                                           smem, a.smem_bytes, s_red);
    if (threadIdx.x == 0) a.out[0] = key;
}

// 8 search points x 16 16x16 blocks: thread = (block, point). Layout of io (uint32 words):
//   [0..63] best_sad_8x8  [64..79] best_sad_16x16  [80..143] best_mv8x8  [144..159] best_mv16x16
//   [160..287] eight_sad16x16[16][8]  [288..799] eight_sad8x8[64][8]
__global__ void __launch_bounds__(128) ext_all_sad_kernel(const uint8_t *src, int ss, const uint8_t *ref, int rs,
                                                          uint32_t mv, int sub, uint32_t *io) {
    __shared__ uint32_t s8[64][8], s16[16][8];
    const int t = threadIdx.x, i = t & 7, ras = t >> 3;
    const int by = ras >> 2, bx = ras & 3, b = c_tab16[ras];
    uint32_t sum = 0;
    for (int q = 0; q < 4; q++) {
        const uint8_t *s = src + (size_t)(16 * by + (q >> 1) * 8) * ss + 16 * bx + (q & 1) * 8;
        const uint8_t *r = ref + (size_t)(16 * by + (q >> 1) * 8) * rs + 16 * bx + (q & 1) * 8 + i;
        uint32_t v = 0;
        if (sub) {
            for (int y = 0; y < 4; y++)
                for (int x = 0; x < 8; x++) v += abs((int)s[(size_t)2 * y * ss + x] - (int)r[(size_t)2 * y * rs + x]);
            v <<= 1;
        } else {
            for (int y = 0; y < 8; y++)
                for (int x = 0; x < 8; x++) v += abs((int)s[(size_t)y * ss + x] - (int)r[(size_t)y * rs + x]);
        }
        s8[4 * b + q][i] = v;
        sum += v;
    }
    s16[b][i] = sum;
    __syncthreads();
    const int16_t mx = (int16_t)(mv & 0xffff), my = (int16_t)(mv >> 16);
    if (t < 80) { // one thread per PU walks the 8 points in order (strict <)
        const bool is16 = t >= 64;
        const int pu = is16 ? t - 64 : t;
        uint32_t *bs = io + (is16 ? 64 + pu : pu), *bm = io + (is16 ? 144 + pu : 80 + pu);
        uint32_t cur = *bs, cmv = *bm;
        for (int j = 0; j < 8; j++) {
            uint32_t v = is16 ? s16[pu][j] : s8[pu][j];
            if (v < cur) {
                cur = v;
                cmv = ((uint32_t)(uint16_t)my << 16) | (uint16_t)(int16_t)(mx + 4 * j);
            }
        }
        *bs = cur;
        *bm = cmv;
    }
    for (int j = t; j < 128; j += 128) io[160 + j] = s16[j >> 3][j & 7];
    for (int j = t; j < 512; j += 128) io[288 + j] = s8[j >> 3][j & 7];
}

// io: [0..127] sad16x16[16][8] (in)  [128..131] best32 [132] best64 [133..136] mv32 [137] mv64 [138..169] sad32[4][8]
__global__ void ext_eight_32_64_kernel(uint32_t mv, uint32_t *io) {
    if (threadIdx.x != 0) return;
    const int16_t mx = (int16_t)(mv & 0xffff), my = (int16_t)(mv >> 16);
    for (int i = 0; i < 8; i++) {
        uint32_t s64 = 0;
        const uint32_t pm = ((uint32_t)(uint16_t)my << 16) | (uint16_t)(int16_t)(mx + 4 * i);
        for (int q = 0; q < 4; q++) {
            uint32_t s = io[(4 * q) * 8 + i] + io[(4 * q + 1) * 8 + i] + io[(4 * q + 2) * 8 + i] + io[(4 * q + 3) * 8 + i];
            io[138 + q * 8 + i] = s;
            if (s < io[128 + q]) {
                io[128 + q] = s;
                io[133 + q] = pm;
            }
            s64 += s;
        }
        if (s64 < io[132]) {
            io[132] = s64;
            io[137] = pm;
        }
    }
}

// single-point variants. io16: [0..3] best8 [4] best16 [5..8] mv8 [9] mv16 [10] sad16 [11..14] sad8
__global__ void ext_sad_8_16_kernel(const uint8_t *src, int ss, const uint8_t *ref, int rs, uint32_t mv, int sub,
                                    uint32_t *io) {
    __shared__ uint32_t s8[4];
    const int q = threadIdx.x;
    if (q < 4) {
        const uint8_t *s = src + (size_t)(q >> 1) * 8 * ss + (q & 1) * 8;
        const uint8_t *r = ref + (size_t)(q >> 1) * 8 * rs + (q & 1) * 8;
        uint32_t v = 0;
        if (sub) {
            for (int y = 0; y < 4; y++)
                for (int x = 0; x < 8; x++) v += abs((int)s[(size_t)2 * y * ss + x] - (int)r[(size_t)2 * y * rs + x]);
            v <<= 1;
        } else {
            for (int y = 0; y < 8; y++)
                for (int x = 0; x < 8; x++) v += abs((int)s[(size_t)y * ss + x] - (int)r[(size_t)y * rs + x]);
        }
        s8[q] = v;
        io[11 + q] = v;
        if (v < io[q]) {
            io[q] = v;
            io[5 + q] = mv;
        }
    }
    __syncthreads();
    if (q == 0) {
        uint32_t s = s8[0] + s8[1] + s8[2] + s8[3];
        if (s < io[4]) {
            io[4] = s;
            io[9] = mv;
        }
        io[10] = s;
    }
}
// io: [0..15] sad16 (in) [16..19] best32 [20] best64 [21..24] mv32 [25] mv64 [26..29] sad32
__global__ void ext_sad_32_64_kernel(uint32_t mv, uint32_t *io) {
    if (threadIdx.x != 0) return;
    uint32_t s64 = 0;
    for (int q = 0; q < 4; q++) {
        uint32_t s = io[4 * q] + io[4 * q + 1] + io[4 * q + 2] + io[4 * q + 3];
        io[26 + q] = s;
        if (s < io[16 + q]) {
            io[16 + q] = s;
            io[21 + q] = mv;
        }
        s64 += s;
    }
    if (s64 < io[20]) {
        io[20] = s64;
        io[25] = mv;
    }
}

__global__ void fill32_kernel(uint32_t *p, int n, uint32_t v) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

static void set_attrs() {
    static PerDeviceOnce once;
    once.run([] {
        SVTB_ATTR(hme_kernel_chunked, HME_SMEM_BYTES);
        SVTB_ATTR(hme_kernel_staged, HME_FAST_SMEM);
        SVTB_ATTR(fullpel_kernel<true>, FP_SMEM_BYTES);
        SVTB_ATTR(fullpel_kernel<false>, FP_SMEM_BYTES);
        SVTB_ATTR(sad_loop_kernel, 200 * 1024);
    });
}

// The per-picture scratch: byte offsets of MeDev's raw[n_sb][2][4], hstate[n_sb], hme_done[n_sb] and fp_done[n_sb], and
// the total.
struct MeScratch {
    size_t raw, hstate, hme_done, fp_done, bytes;
};
MeScratch me_scratch(const SvtB200MeParams &p) {
    const size_t n_sb = (size_t)((p.full.width + 63) / 64) * ((p.full.height + 63) / 64);
    MeScratch s;
    s.raw = 0;
    s.hstate = s.raw + n_sb * 8 * sizeof(RawHme);
    s.hme_done = s.hstate + n_sb * sizeof(HmeState);
    s.fp_done = s.hme_done + n_sb * sizeof(unsigned int);
    s.bytes = s.fp_done + n_sb * sizeof(unsigned int);
    return s;
}

// What svt_b200_me_picture launches for a picture with parameters `p` (validated): the HME regime, the dynamic shared
// memory of the HME and full-pel kernels, and the full-pel CTA width.  Host arithmetic only.
struct MeLaunchPlan {
    bool hme_staged;
    int hme_smem, fp_smem, fp_threads;
};
MeLaunchPlan me_launch_plan(const SvtB200MeParams &p) {
    // per reference: the full-pel warp-tasks (32 tasks of 4 positions) of its whole search window
    int maxd = 1, n = 0, warp_tasks[SVT_B200_ME_LISTS * SVT_B200_ME_MAX_REFS];
    for (int l = 0; l < p.num_lists; l++)
        for (int r = 0; r < p.num_refs[l]; r++) {
            const int dd = scaled_dist(p.ref_dist[l][r]);
            maxd = std::max(maxd, dd);
            const int2 a = fp_search_area(p, dd);
            warp_tasks[n++] = (a.y * 4 * ((fp_window_width(a.x) + 15) >> 4) + 31) / 32;
        }
    MeLaunchPlan plan;
    { // worst-case shared memory of one HME level in the staged regime (4 windows + the source block)
        const int k = p.hme_search_method ? 2 : 1;
        auto level_bytes = [&](int saw, int sah, int bw, int bh) {
            const int bhh = k == 2 ? bh / 2 : bh;
            int wpw = ((saw - 1 + bw + 3) / 4) + 1;
            wpw = std::max(wpw, std::max(hme_pitch_words(saw, bw / 4, 2), hme_pitch_words(saw, bw / 4, 4)));
            const size_t win = (size_t)wpw * 4 * (sah - 1 + (bhh - 1) * k + 1);
            return 4 * win + (size_t)((bw + 3) / 4) * 4 * bhh;
        };
        // the kernel indexes the per-region arrays with [rx] / [ry]: size for the largest region that is used, at the
        // largest distance
        const int nrx = p.number_hme_search_region_in_width, nry = p.number_hme_search_region_in_height;
        auto amax = [](const int32_t *a, int n) { return n > 1 ? std::max(a[0], a[1]) : a[0]; };
        int w0 = amax(p.hme_level0_search_area_in_width_array, nrx) * maxd, h0 = amax(p.hme_level0_search_area_in_height_array, nry) * maxd;
        const int w0m = amax(p.hme_level0_max_search_area_in_width_array, nrx), h0m = amax(p.hme_level0_max_search_area_in_height_array, nry);
        if (w0 > w0m) w0 = w0m;
        if (h0 > h0m) h0 = h0m;
        size_t a = level_bytes((w0 + 15) & ~15, h0, 16, 16);
        size_t b = level_bytes((amax(p.hme_level1_search_area_in_width_array, nrx) + 7) & ~7, amax(p.hme_level1_search_area_in_height_array, nry), 32, 32);
        size_t c = level_bytes((amax(p.hme_level2_search_area_in_width_array, nrx) + 7) & ~7, amax(p.hme_level2_search_area_in_height_array, nry), 64, 64);
        size_t hme_need = a > b ? a : b;
        hme_need = hme_need > c ? hme_need : c;
        hme_need += 256;
        plan.hme_staged = hme_need <= (size_t)HME_FAST_SMEM;
        plan.hme_smem = plan.hme_staged ? (int)hme_need : HME_SMEM_BYTES;
    }
    { // the full-pel search: source rows + the largest window (whole if it fits)
        const int2 a = fp_search_area(p, maxd);
        const int saw = fp_window_width(a.x), sah = a.y;
        const int sub = p.me_search_method != 0;
        size_t need = (size_t)(sub ? 32 : 64) * 64 + (size_t)fp_pitch_words(saw) * 4 * (sah - 1 + (sub ? 63 : 64)) + 64;
        if (need > (size_t)FP_SMEM_BYTES) need = FP_SMEM_BYTES;
        plan.fp_smem = (int)need;
    }
    // full-pel CTA size: pick the warp count that divides the per-reference warp-task counts best (idle warps only hold
    // registers until the CTA's last round ends)
    static const int cand[5] = {4, 3, 6, 2, 8};
    long best_cost = -1;
    for (int ci = 0; ci < 5; ci++) {
        long cost = 0;
        for (int i = 0; i < n; i++) cost += (long)((warp_tasks[i] + cand[ci] - 1) / cand[ci]) * cand[ci];
        if (best_cost < 0 || cost < best_cost) {
            best_cost = cost;
            plan.fp_threads = cand[ci] * 32;
        }
    }
    return plan;
}

} // namespace

extern "C" {

size_t svt_b200_me_scratch_bytes(const SvtB200MeParams *p) {
    if (!p) return 0;
    return me_scratch(*p).bytes;
}

int svt_b200_me_picture(const SvtB200MeParams *p, const SvtB200MePlanes *src,
                        const SvtB200MePlanes refs[SVT_B200_ME_LISTS][SVT_B200_ME_MAX_REFS],
                        const SvtB200MeOutputs *out, void *scratch, void *stream) {
    if (!p || !src || !refs || !out || !scratch) {
        set_error("svt_b200_me_picture: null argument");
        return SVT_B200_ERR_ARG;
    }
    if (p->num_lists < 1 || p->num_lists > 2 || p->num_refs[0] < 1 || p->num_refs[0] > 4 || p->num_refs[1] < 0 ||
        p->num_refs[1] > 4 || p->number_hme_search_region_in_width > 2 || p->number_hme_search_region_in_height > 2 ||
        p->number_hme_search_region_in_width < 1 || p->number_hme_search_region_in_height < 1) {
        set_error("svt_b200_me_picture: reference structure / HME regions out of range");
        return SVT_B200_ERR_ARG;
    }
    // window sizes the staging budget was sized for (every preset of v0.8.6 at non-screen content fits)
    if (p->max_me_search_width > 256 || p->max_me_search_height > 256 ||
        std::max(p->hme_level0_max_search_area_in_width_array[0], p->hme_level0_max_search_area_in_width_array[1]) > 240 ||
        std::max(p->hme_level0_max_search_area_in_height_array[0], p->hme_level0_max_search_area_in_height_array[1]) > 240) {
        set_error("svt_b200_me_picture: search area larger than the kernels are sized for");
        return SVT_B200_ERR_UNSUPPORTED;
    }
    set_attrs();
    const MeLaunchPlan plan = me_launch_plan(*p);
    const MeScratch sc = me_scratch(*p);
    MeDev d;
    memset(&d, 0, sizeof(d));
    d.p = *p;
    d.src = *src;
    memcpy(d.refs, refs, sizeof(d.refs));
    d.out = *out;
    d.raw = (RawHme *)((char *)scratch + sc.raw);
    d.hstate = (HmeState *)((char *)scratch + sc.hstate);
    d.hme_done = (unsigned int *)((char *)scratch + sc.hme_done);
    d.fp_done = (unsigned int *)((char *)scratch + sc.fp_done);
    d.sbs_x = (p->full.width + 63) / 64;
    d.sbs_y = (p->full.height + 63) / 64;
    int n = 0;
    for (int l = 0; l < p->num_lists; l++)
        for (int r = 0; r < p->num_refs[l]; r++) {
            d.slot_l[n] = l;
            d.slot_r[n] = r;
            n++;
        }
    d.n_slots = n;
    d.fp_smem_bytes = plan.fp_smem;
    const int n_sb = d.sbs_x * d.sbs_y;
    cudaStream_t st = (cudaStream_t)stream;
    // slots of unused references are defined as zero
    SVTB_CUDA_TRY(cudaMemsetAsync(out->best_sad, 0, (size_t)n_sb * 8 * 85 * 4, st));
    SVTB_CUDA_TRY(cudaMemsetAsync(out->best_mv, 0, (size_t)n_sb * 8 * 85 * 4, st));
    SVTB_CUDA_TRY(cudaMemsetAsync(scratch, 0, sc.bytes, st));
    if (plan.hme_staged)
        SVTB_LAUNCH(hme_kernel_staged, dim3(n_sb, n), NT_SEARCH, plan.hme_smem, st, d);
    else
        SVTB_LAUNCH(hme_kernel_chunked, dim3(n_sb, n), NT_SEARCH, plan.hme_smem, st, d);
    if (p->me_search_method != 0)
        SVTB_LAUNCH(fullpel_kernel<true>, dim3(n_sb, n), plan.fp_threads, plan.fp_smem, st, d);
    else
        SVTB_LAUNCH(fullpel_kernel<false>, dim3(n_sb, n), plan.fp_threads, plan.fp_smem, st, d);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

// ---------------------------------------------------------------------------------------------------
// RTCD drop-ins (host pointers)
// ---------------------------------------------------------------------------------------------------
void svt_sad_loop_kernel_cuda(uint8_t *src, uint32_t src_stride, uint8_t *ref, uint32_t ref_stride,
                              uint32_t block_height, uint32_t block_width, uint64_t *best_sad,
                              int16_t *x_search_center, int16_t *y_search_center, uint32_t src_stride_raw,
                              int16_t search_area_width, int16_t search_area_height) {
    *best_sad = 0xffffff;
    if (search_area_width <= 0 || search_area_height <= 0 || block_width == 0 || block_height == 0) return;
    if (src_stride_raw == 0 || ref_stride % src_stride_raw != 0) {
        fprintf(stderr, "svt_sad_loop_kernel_cuda: ref_stride must be a multiple of src_stride_raw\n");
        abort();
    }
    set_attrs();
    const int k = ref_stride / src_stride_raw;
    const int bw = block_width, bh = block_height, saw = search_area_width, sah = search_area_height;
    const int ww = saw - 1 + bw, wh = (sah - 1) + (bh - 1) * k + 1;
    Staging s({(size_t)bw * bh, (size_t)ww * wh, 8});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, src, src_stride, 1, bw, bh);
    s.put_rows(1, ref, src_stride_raw, 1, ww, wh);
    SVTB_CUDA_FATAL(s.upload(0, 1));
    SadLoopArgs a;
    a.src = s.d(0);
    a.ref = s.d(1);
    a.src_stride = bw;
    a.raw_stride = ww;
    a.k = k;
    a.bw = bw;
    a.bh = bh;
    a.saw = saw;
    a.sah = sah;
    a.out = s.d<uint64_t>(2);
    // enough shared memory for the source block + at least one search row, up to 200 KB
    const size_t spw = (bw + 3) / 4, wpw = (ww + 3) / 4 + 1;
    size_t need = spw * bh * 4 + wpw * 4 * (size_t)wh;
    size_t min_need = spw * bh * 4 + wpw * 4 * (size_t)((bh - 1) * k + 1);
    if (min_need > 200 * 1024) {
        fprintf(stderr, "svt_sad_loop_kernel_cuda: block too large for shared memory\n");
        abort();
    }
    if (need > 200 * 1024) need = 200 * 1024;
    a.smem_bytes = (int)need;
    SVTB_LAUNCH(sad_loop_kernel, 1, NT_SEARCH, need, s.stream(), a);
    SVTB_CUDA_FATAL(s.download(2, 2));
    const uint64_t key = *s.h<uint64_t>(2);
    const uint32_t sad = (uint32_t)(key >> 32), idx = (uint32_t)key;
    if (sad < 0xffffffu) { // strict < against the 0xffffff start value
        *best_sad = sad;
        *x_search_center = (int16_t)(idx % saw);
        *y_search_center = (int16_t)(idx / saw);
    }
}

void svt_ext_all_sad_calculation_8x8_16x16_cuda(uint8_t *src, uint32_t src_stride, uint8_t *ref,
                                                uint32_t ref_stride, uint32_t mv, uint32_t *p_best_sad_8x8,
                                                uint32_t *p_best_sad_16x16, uint32_t *p_best_mv8x8,
                                                uint32_t *p_best_mv16x16, uint32_t p_eight_sad16x16[16][8],
                                                uint32_t p_eight_sad8x8[64][8], uint8_t sub_sad) {
    Staging s({64 * 64, 71 * 64, 800 * 4});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, src, src_stride, 1, 64, 64);
    s.put_rows(1, ref, ref_stride, 1, 71, 64);
    uint32_t *io = s.h<uint32_t>(2);
    memcpy(io, p_best_sad_8x8, 64 * 4);
    memcpy(io + 64, p_best_sad_16x16, 16 * 4);
    memcpy(io + 80, p_best_mv8x8, 64 * 4);
    memcpy(io + 144, p_best_mv16x16, 16 * 4);
    SVTB_CUDA_FATAL(s.upload(0, 2, 160 * 4));
    SVTB_LAUNCH(ext_all_sad_kernel, 1, 128, 0, s.stream(), s.d(0), 64, s.d(1), 71, mv, (int)sub_sad, s.d<uint32_t>(2));
    SVTB_CUDA_FATAL(s.download(2, 2));
    memcpy(p_best_sad_8x8, io, 64 * 4);
    memcpy(p_best_sad_16x16, io + 64, 16 * 4);
    memcpy(p_best_mv8x8, io + 80, 64 * 4);
    memcpy(p_best_mv16x16, io + 144, 16 * 4);
    memcpy(p_eight_sad16x16, io + 160, 128 * 4);
    memcpy(p_eight_sad8x8, io + 288, 512 * 4);
}

void svt_ext_eight_sad_calculation_32x32_64x64_cuda(uint32_t p_sad16x16[16][8], uint32_t *p_best_sad_32x32,
                                                    uint32_t *p_best_sad_64x64, uint32_t *p_best_mv32x32,
                                                    uint32_t *p_best_mv64x64, uint32_t mv,
                                                    uint32_t p_sad32x32[4][8]) {
    Staging s({170 * 4});
    SVTB_CUDA_FATAL(s.status());
    uint32_t *io = s.h<uint32_t>(0);
    memcpy(io, p_sad16x16, 128 * 4);
    memcpy(io + 128, p_best_sad_32x32, 16);
    io[132] = *p_best_sad_64x64;
    memcpy(io + 133, p_best_mv32x32, 16);
    io[137] = *p_best_mv64x64;
    SVTB_CUDA_FATAL(s.upload(0, 0, 138 * 4));
    SVTB_LAUNCH(ext_eight_32_64_kernel, 1, 32, 0, s.stream(), mv, s.d<uint32_t>(0));
    SVTB_CUDA_FATAL(s.download(0, 0));
    memcpy(p_best_sad_32x32, io + 128, 16);
    *p_best_sad_64x64 = io[132];
    memcpy(p_best_mv32x32, io + 133, 16);
    *p_best_mv64x64 = io[137];
    memcpy(p_sad32x32, io + 138, 32 * 4);
}

void svt_ext_sad_calculation_8x8_16x16_cuda(uint8_t *src, uint32_t src_stride, uint8_t *ref, uint32_t ref_stride,
                                            uint32_t *p_best_sad_8x8, uint32_t *p_best_sad_16x16,
                                            uint32_t *p_best_mv8x8, uint32_t *p_best_mv16x16, uint32_t mv,
                                            uint32_t *p_sad16x16, uint32_t *p_sad8x8, uint8_t sub_sad) {
    Staging s({256, 256, 15 * 4});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, src, src_stride, 1, 16, 16);
    s.put_rows(1, ref, ref_stride, 1, 16, 16);
    uint32_t *io = s.h<uint32_t>(2);
    memcpy(io, p_best_sad_8x8, 16);
    io[4] = *p_best_sad_16x16;
    memcpy(io + 5, p_best_mv8x8, 16);
    io[9] = *p_best_mv16x16;
    SVTB_CUDA_FATAL(s.upload(0, 2, 10 * 4));
    SVTB_LAUNCH(ext_sad_8_16_kernel, 1, 32, 0, s.stream(), s.d(0), 16, s.d(1), 16, mv, (int)sub_sad, s.d<uint32_t>(2));
    SVTB_CUDA_FATAL(s.download(2, 2));
    memcpy(p_best_sad_8x8, io, 16);
    *p_best_sad_16x16 = io[4];
    memcpy(p_best_mv8x8, io + 5, 16);
    *p_best_mv16x16 = io[9];
    *p_sad16x16 = io[10];
    memcpy(p_sad8x8, io + 11, 16);
}

void svt_ext_sad_calculation_32x32_64x64_cuda(uint32_t *p_sad16x16, uint32_t *p_best_sad_32x32,
                                              uint32_t *p_best_sad_64x64, uint32_t *p_best_mv32x32,
                                              uint32_t *p_best_mv64x64, uint32_t mv, uint32_t *p_sad32x32) {
    Staging s({30 * 4});
    SVTB_CUDA_FATAL(s.status());
    uint32_t *io = s.h<uint32_t>(0);
    memcpy(io, p_sad16x16, 64);
    memcpy(io + 16, p_best_sad_32x32, 16);
    io[20] = *p_best_sad_64x64;
    memcpy(io + 21, p_best_mv32x32, 16);
    io[25] = *p_best_mv64x64;
    SVTB_CUDA_FATAL(s.upload(0, 0, 26 * 4));
    SVTB_LAUNCH(ext_sad_32_64_kernel, 1, 32, 0, s.stream(), mv, s.d<uint32_t>(0));
    SVTB_CUDA_FATAL(s.download(0, 0));
    memcpy(p_best_sad_32x32, io + 16, 16);
    *p_best_sad_64x64 = io[20];
    memcpy(p_best_mv32x32, io + 21, 16);
    *p_best_mv64x64 = io[25];
    memcpy(p_sad32x32, io + 26, 16);
}

void svt_initialize_buffer_32bits_cuda(uint32_t *pointer, uint32_t count128, uint32_t count32, uint32_t value) {
    const int n = (int)(count128 * 4 + count32);
    if (n <= 0) return;
    Staging s({(size_t)n * 4});
    SVTB_CUDA_FATAL(s.status());
    SVTB_LAUNCH(fill32_kernel, (n + 255) / 256, 256, 0, s.stream(), s.d<uint32_t>(0), n, value);
    SVTB_CUDA_FATAL(s.download(0, 0));
    memcpy(pointer, s.h(0), (size_t)n * 4);
}
}
