// interp.cu — translational inter prediction: the AV1 sub-pel interpolation filters (SURVEY 8(f) rank 1).
//
// Replaces, in svt-av1 v0.8.6 (Source/Lib/Common/Codec/EbInterPrediction.c unless noted):
//   svt_av1_convolve_{2d_sr,x_sr,y_sr,2d_copy_sr}_c :349-470, svt_av1_jnt_convolve_{2d,x,y,2d_copy}_c :552-745 and the
//   highbd forms :747-1145 (RTCD drop-ins, host pointers); svt_aom_convolve8_{horiz,vert}_c (convolve.c:249-308);
//   and, batched per picture, the enc_make_inter_predictor calls of av1_inter_prediction
//   (Encoder/Codec/EbEncInterPrediction.c:3591-3762, :4040-4930): MV clamp (clamp_mv_to_umv_border_sb :24-45), split
//   into whole-sample position + 1/16 phase, dispatch on (phase_x != 0, phase_y != 0, compound), and for compound blocks
//   the second reference averaged (plain or distance weighted) into the first without the CONV_BUF round trip.
//
// Work decomposition: a HALF warp filters one tile of <= 16x8 output samples (two unrelated tiles per warp). Lane r reads
// row r of the (th+7)x(tw+7) source window into registers (aligned 32-bit loads + funnel shifts) and runs the horizontal
// pass there (dp4a / dp2a on the AV1 kernels halved into int8), leaving the int16 intermediate the reference keeps in
// im_block in shared memory; then each lane slides the vertical 8 taps down a column strip of <= 8 rows. The sixteen
// reference functions differ only in which pass runs and in the rounding, so all of them are one device routine
// (conv_tile) + one finishing step. Bound: instruction issue (per-tile set-up is comparable to the filtering for small
// blocks); HBM traffic is ~(1 + n_refs) B per predicted sample.
#include <algorithm>
#include <mutex>

#include "common.cuh"

namespace svtb200 {
namespace {

// AV1 interpolation kernels, half coefficients (every tap is even; spec 7.11.3.4 Subpel_Filters): regular, smooth, sharp,
// and the 4-tap regular / smooth used when the block is <= 4 wide (av1_get_interp_filter_params_with_block_size :1251-1262).
// BILINEAR is computed. tests/test_interp_gpu.py pins svt_b200_get_interp_kernel against the reference's tables.
#define K_ROW(a, b, c, d, e, f, g, h) {a, b, c, d, e, f, g, h}
const int8_t h_half_taps[5][16][8] = {
    {K_ROW(0, 0, 0, 64, 0, 0, 0, 0), K_ROW(0, 1, -3, 63, 4, -1, 0, 0), K_ROW(0, 1, -5, 61, 9, -2, 0, 0), K_ROW(0, 1, -6, 58, 14, -4, 1, 0),
     K_ROW(0, 1, -7, 55, 19, -5, 1, 0), K_ROW(0, 1, -7, 51, 24, -6, 1, 0), K_ROW(0, 1, -8, 47, 29, -6, 1, 0),
     K_ROW(0, 1, -7, 42, 33, -6, 1, 0), K_ROW(0, 1, -7, 38, 38, -7, 1, 0), K_ROW(0, 1, -6, 33, 42, -7, 1, 0),
     K_ROW(0, 1, -6, 29, 47, -8, 1, 0), K_ROW(0, 1, -6, 24, 51, -7, 1, 0), K_ROW(0, 1, -5, 19, 55, -7, 1, 0),
     K_ROW(0, 1, -4, 14, 58, -6, 1, 0), K_ROW(0, 0, -2, 9, 61, -5, 1, 0), K_ROW(0, 0, -1, 4, 63, -3, 1, 0)},
    {K_ROW(0, 0, 0, 64, 0, 0, 0, 0), K_ROW(0, 1, 14, 31, 17, 1, 0, 0), K_ROW(0, 0, 13, 31, 18, 2, 0, 0), K_ROW(0, 0, 11, 31, 20, 2, 0, 0),
     K_ROW(0, 0, 10, 30, 21, 3, 0, 0), K_ROW(0, 0, 9, 29, 22, 4, 0, 0), K_ROW(0, 0, 8, 28, 23, 5, 0, 0), K_ROW(0, -1, 8, 27, 24, 6, 0, 0),
     K_ROW(0, -1, 7, 26, 26, 7, -1, 0), K_ROW(0, 0, 6, 24, 27, 8, -1, 0), K_ROW(0, 0, 5, 23, 28, 8, 0, 0), K_ROW(0, 0, 4, 22, 29, 9, 0, 0),
     K_ROW(0, 0, 3, 21, 30, 10, 0, 0), K_ROW(0, 0, 2, 20, 31, 11, 0, 0), K_ROW(0, 0, 2, 18, 31, 13, 0, 0), K_ROW(0, 0, 1, 17, 31, 14, 1, 0)},
    {K_ROW(0, 0, 0, 64, 0, 0, 0, 0), K_ROW(-1, 1, -3, 63, 4, -1, 1, 0), K_ROW(-1, 3, -6, 62, 8, -3, 2, -1),
     K_ROW(-1, 4, -9, 60, 13, -5, 3, -1), K_ROW(-2, 5, -11, 58, 19, -7, 3, -1), K_ROW(-2, 5, -11, 54, 24, -9, 4, -1),
     K_ROW(-2, 5, -12, 50, 30, -10, 4, -1), K_ROW(-2, 5, -12, 45, 35, -11, 5, -1), K_ROW(-2, 6, -12, 40, 40, -12, 6, -2),
     K_ROW(-1, 5, -11, 35, 45, -12, 5, -2), K_ROW(-1, 4, -10, 30, 50, -12, 5, -2), K_ROW(-1, 4, -9, 24, 54, -11, 5, -2),
     K_ROW(-1, 3, -7, 19, 58, -11, 5, -2), K_ROW(-1, 3, -5, 13, 60, -9, 4, -1), K_ROW(-1, 2, -3, 8, 62, -6, 3, -1),
     K_ROW(0, 1, -1, 4, 63, -3, 1, -1)},
    {K_ROW(0, 0, 0, 64, 0, 0, 0, 0), K_ROW(0, 0, -2, 63, 4, -1, 0, 0), K_ROW(0, 0, -4, 61, 9, -2, 0, 0), K_ROW(0, 0, -5, 58, 14, -3, 0, 0),
     K_ROW(0, 0, -6, 55, 19, -4, 0, 0), K_ROW(0, 0, -6, 51, 24, -5, 0, 0), K_ROW(0, 0, -7, 47, 29, -5, 0, 0),
     K_ROW(0, 0, -6, 42, 33, -5, 0, 0), K_ROW(0, 0, -6, 38, 38, -6, 0, 0), K_ROW(0, 0, -5, 33, 42, -6, 0, 0),
     K_ROW(0, 0, -5, 29, 47, -7, 0, 0), K_ROW(0, 0, -5, 24, 51, -6, 0, 0), K_ROW(0, 0, -4, 19, 55, -6, 0, 0),
     K_ROW(0, 0, -3, 14, 58, -5, 0, 0), K_ROW(0, 0, -2, 9, 61, -4, 0, 0), K_ROW(0, 0, -1, 4, 63, -2, 0, 0)},
    {K_ROW(0, 0, 0, 64, 0, 0, 0, 0), K_ROW(0, 0, 15, 31, 17, 1, 0, 0), K_ROW(0, 0, 13, 31, 18, 2, 0, 0), K_ROW(0, 0, 11, 31, 20, 2, 0, 0),
     K_ROW(0, 0, 10, 30, 21, 3, 0, 0), K_ROW(0, 0, 9, 29, 22, 4, 0, 0), K_ROW(0, 0, 8, 28, 23, 5, 0, 0), K_ROW(0, 0, 7, 27, 24, 6, 0, 0),
     K_ROW(0, 0, 6, 26, 26, 6, 0, 0), K_ROW(0, 0, 6, 24, 27, 7, 0, 0), K_ROW(0, 0, 5, 23, 28, 8, 0, 0), K_ROW(0, 0, 4, 22, 29, 9, 0, 0),
     K_ROW(0, 0, 3, 21, 30, 10, 0, 0), K_ROW(0, 0, 2, 20, 31, 11, 0, 0), K_ROW(0, 0, 2, 18, 31, 13, 0, 0), K_ROW(0, 0, 1, 17, 31, 15, 0, 0)}};
__constant__ int8_t c_half_taps[5][16][8];

int upload_tables() { // once per device
    static std::mutex mu;
    static bool done[64] = {};
    int dev = 0;
    SVTB_CUDA_TRY(cudaGetDevice(&dev));
    if (dev >= 64) return SVT_B200_ERR_ARG;
    std::lock_guard<std::mutex> lk(mu);
    if (!done[dev]) {
        SVTB_CUDA_TRY(cudaMemcpyToSymbol(c_half_taps, h_half_taps, sizeof(h_half_taps)));
        done[dev] = true;
    }
    return SVT_B200_OK;
}

// which table a filter id resolves to for a block `w` wide: -1 = bilinear
__host__ __device__ inline int table_of(int filter, int w) {
    if (filter == 3) return -1;
    if (w <= 4) return filter == 1 ? 4 : 3; // sharp -> the regular 4-tap kernel
    return filter;
}
// the 8 half taps of a kernel row, packed one per byte (taps 0..3, taps 4..7)
__device__ __forceinline__ uint2 load_half_taps(int filter, int w, int subpel) {
    const int t = table_of(filter, w);
    if (t < 0) return make_uint2((uint32_t)(64 - 4 * subpel) << 24, (uint32_t)(4 * subpel)); // bilinear: taps 3 and 4
    const int2 v = *reinterpret_cast<const int2 *>(c_half_taps[t][subpel]);
    return make_uint2((uint32_t)v.x, (uint32_t)v.y);
}
__device__ __forceinline__ void unpack_taps(uint2 p, int (&f)[8]) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
        f[k] = (int)(int8_t)(p.x >> (8 * k));
        f[4 + k] = (int)(int8_t)(p.y >> (8 * k));
    }
}
__device__ __forceinline__ int dp4a_us(uint32_t a, uint32_t b, int c) { // 4 x (u8 * s8) + c
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ int dp2a_lo_us(uint32_t a, uint32_t b, int c) { // 2 x (u16 * s8 (bytes 0, 1 of b)) + c
    int d;
    asm("dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ int dp2a_hi_us(uint32_t a, uint32_t b, int c) { // ... bytes 2, 3 of b
    int d;
    asm("dp2a.hi.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// A tile is <= 16 x 8 predicted samples and belongs to one HALF warp (16 lanes): its window has <= 15 rows, one per lane.
constexpr int TILE_W = 16, TILE_H = 8, WIN = TILE_H + 7, IM_P = 18; // IM_P: int16 pitch of an intermediate row (9 words)
struct HalfSmem {
    int16_t im[WIN * IM_P];           // the horizontal pass (im_block), or the samples themselves when it does not run
    uint16_t first[TILE_W * TILE_H];  // CONV_BUF of the tile (compound), lane-private slots
    uint32_t pad;
};

__device__ __forceinline__ int rshift_round(int v, int n) { return (v + ((1 << n) >> 1)) >> n; } // ROUND_POWER_OF_TWO
__device__ __forceinline__ int clip_bd(int v, int bd) { return min(max(v, 0), (1 << bd) - 1); }
// i / d for i < 1024, d <= 32 (inv = ceil(2^16 / d))
__device__ __forceinline__ int div_small(int i, int inv) { return (i * inv) >> 16; }
// ceil(2^16 / d), d = 1..32 without a division: exact for these d in fp32
__device__ __forceinline__ int inv_small(int d) { return (int)ceilf(__fdividef(65536.0f, (float)d) - 0.01f); }
// ROUND_POWER_OF_TWO(sum + off, n) of a sum whose taps were divided by 2^H (all taps and offsets are multiples of 2^H)
template <int H>
__device__ __forceinline__ int rr(int s, int off, int n) {
    return (s + (off >> H) + (1 << (n - 1 - H))) >> (n - H);
}

struct Rounds {
    int r0, r1, bd;
};
// get_conv_params_no_round (convolve.h:44-71)
__host__ __device__ inline Rounds conv_rounds(int bd, bool compound) {
    Rounds r{3, compound ? 7 : 11, bd};
    const int over = bd + 7 - r.r0 + 2 - 16;
    if (over > 0) {
        r.r0 += over;
        if (!compound) r.r1 -= over;
    }
    return r;
}

// One row of the source window (<= 23 samples) in registers, read with aligned 32-bit loads and realigned.
template <typename T>
struct Row;
template <>
struct Row<uint8_t> {
    uint32_t W[6];
    __device__ __forceinline__ void load(const uint8_t *rp, int n) {
        const int mis = (int)((uintptr_t)rp & 3);
        const uint32_t *p = (const uint32_t *)(rp - mis);
        const int nw = (mis + n + 3) >> 2;
        uint32_t w[7];
#pragma unroll
        for (int i = 0; i < 7; i++) w[i] = i < nw ? __ldg(p + i) : 0u;
#pragma unroll
        for (int i = 0; i < 6; i++) W[i] = __funnelshift_r(w[i], w[i + 1], 8 * mis);
    }
    __device__ __forceinline__ int sample(int k) const { return (int)((W[k >> 2] >> (8 * (k & 3))) & 0xffu); }
    __device__ __forceinline__ uint32_t quad(int x) const { return (x & 3) ? __funnelshift_r(W[x >> 2], W[(x >> 2) + 1], 8 * (x & 3)) : W[x >> 2]; }
    // sum over the 8 half taps of samples x .. x + 7
    __device__ __forceinline__ int hsum_half(int x, uint2 t) const { return dp4a_us(quad(x + 4), t.y, dp4a_us(quad(x), t.x, 0)); }
};
template <>
struct Row<uint16_t> {
    uint32_t W[12];
    __device__ __forceinline__ void load(const uint16_t *rp, int n) {
        const int mis = (int)((uintptr_t)rp & 3);
        const uint32_t *p = (const uint32_t *)((const uint8_t *)rp - mis);
        const int nw = (mis + 2 * n + 3) >> 2;
        uint32_t w[13];
#pragma unroll
        for (int i = 0; i < 13; i++) w[i] = i < nw ? __ldg(p + i) : 0u;
#pragma unroll
        for (int i = 0; i < 12; i++) W[i] = __funnelshift_r(w[i], w[i + 1], 8 * mis);
    }
    __device__ __forceinline__ int sample(int k) const { return (int)((W[k >> 1] >> (16 * (k & 1))) & 0xffffu); }
    __device__ __forceinline__ uint32_t pair(int x) const { return (x & 1) ? __funnelshift_r(W[x >> 1], W[(x >> 1) + 1], 16) : W[x >> 1]; }
    __device__ __forceinline__ int hsum_half(int x, uint2 t) const {
        return dp2a_hi_us(pair(x + 6), t.y, dp2a_lo_us(pair(x + 4), t.y, dp2a_hi_us(pair(x + 2), t.x, dp2a_lo_us(pair(x), t.x, 0))));
    }
};

// One reference's filtering of a tile by a half warp (`sub` = lane & 15): src addresses the tile's sample (0,0) in the
// reference plane. The two halves of a warp work on unrelated tiles; everything below is per half except the two
// __syncwarp(), which every lane reaches (a half with nothing to do passes th = 0 and an empty strip).
//   phase A  lane r owns row r of the (th + 7) x (tw + 7) window: it reads the row into registers, runs the horizontal
//            filter for the 16 columns and leaves the int16 row (im_block of the reference) in shared memory;
//   phase B  lane (x, g) owns a column strip of <= 8 rows: sliding 8-tap window down the column.
// H = 1: taps are the AV1 kernels halved (hx packed per byte for dp4a / dp2a, fy[] = halves); H = 0: fx[] / fy[] hold
// arbitrary int16 taps (the drop-ins, whose caller owns the table).
// On return val[j] belongs to output (yb + j, x) of the tile (see strip_of): without `compound` the prediction sample,
// with it this reference's intermediate (what the jnt forms store to / combine with CONV_BUF).
struct Strip {
    int x, yb, rows; // rows = 0: idle lane
    int rpg;         // rows per strip (uniform in the half): rows <= rpg <= 8
};
__device__ __forceinline__ Strip strip_of(int tw, int th, int sub) {
    const int inv_tw = inv_small(max(tw, 1));
    const int ng = div_small(16, inv_tw), g = div_small(sub, inv_tw);
    const int rpg = div_small(th + ng - 1, inv_small(ng));
    Strip s;
    s.x = sub - g * tw;
    s.yb = g * rpg;
    s.rows = g < ng ? max(0, min(rpg, th - s.yb)) : 0;
    s.rpg = rpg;
    return s;
}

template <typename T, int H>
__device__ __forceinline__ void conv_tile(const T *__restrict__ src, int stride, int tw, int th, bool sx, bool sy, uint2 hx,
                                          const int (&fx)[8], const int (&fy)[8], Rounds rd, bool compound, HalfSmem &s, int sub,
                                          Strip st, int (&val)[8]) {
    const int wh = th ? th + (sy ? 7 : 0) : 0;
    const int offset_bits = rd.bd + 14 - rd.r0;
    const int round_offset = (1 << (offset_bits - rd.r1)) + (1 << (offset_bits - rd.r1 - 1));
    const int bits2 = 14 - rd.r0 - rd.r1;
    __syncwarp(); // the previous readers of im are done
    if (sub < wh) {
        Row<T> row;
        row.load(src + (ptrdiff_t)(sub - (sy ? 3 : 0)) * stride - (sx ? 3 : 0), tw + (sx ? 7 : 0));
        uint32_t *out = reinterpret_cast<uint32_t *>(s.im + sub * IM_P);
        if (sx) {
            const int off = sy ? 1 << (rd.bd + 6) : 0; // the 2-D forms offset the first pass
#pragma unroll
            for (int x = 0; x < TILE_W; x += 2) {
                if (x == TILE_W / 2 && tw <= TILE_W / 2) break; // narrow tile: the upper columns are not needed
                int v[2];
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    int sum;
                    if (H) {
                        sum = row.hsum_half(x + e, hx);
                    } else {
                        sum = 0;
#pragma unroll
                        for (int k = 0; k < 8; k++) sum += fx[k] * row.sample(x + e + k);
                    }
                    v[e] = rr<H>(sum, off, rd.r0);
                }
                out[x >> 1] = (uint32_t)(v[0] & 0xffff) | (uint32_t)v[1] << 16;
            }
        } else {
#pragma unroll
            for (int x = 0; x < TILE_W; x += 2) {
                if (x == TILE_W / 2 && tw <= TILE_W / 2) break;
                out[x >> 1] = (uint32_t)row.sample(x) | (uint32_t)row.sample(x + 1) << 16;
            }
        }
    }
    __syncwarp();
    int v[15];
#pragma unroll
    for (int k = 0; k < 15; k++) {
        if (k >= st.rpg + (sy ? 7 : 0) || !st.rpg) break;
        v[k] = (k < st.rows + (sy ? 7 : 0)) ? (int)s.im[(st.yb + k) * IM_P + st.x] : 0;
    }
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (j >= st.rpg) break;
        int res;
        if (sy) {
            int sum = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) sum += fy[k] * v[j + k];
            if (sx) { // 2-D
                res = rr<H>(sum, 1 << offset_bits, rd.r1);
                res = compound ? (int)(uint16_t)res : clip_bd(rshift_round((int)(int16_t)(uint16_t)(res - round_offset), bits2), rd.bd);
            } else {
                res = compound ? rr<H>(sum << (7 - rd.r0), 0, rd.r1) + round_offset : clip_bd(rr<H>(sum, 0, 7), rd.bd);
            }
        } else if (sx) {
            res = compound ? (1 << (7 - rd.r1)) * v[j] + round_offset : clip_bd(rshift_round(v[j], 7 - rd.r0), rd.bd);
        } else {
            res = compound ? (int)(uint16_t)((uint16_t)(v[j] << bits2) + (uint16_t)round_offset) : v[j];
        }
        val[j] = res;
    }
}

// the do_average branch of the jnt forms
__device__ __forceinline__ int jnt_average(int first, int res, bool use_jnt, int fwd, int bck, Rounds rd) {
    const int offset_bits = rd.bd + 14 - rd.r0;
    const int round_offset = (1 << (offset_bits - rd.r1)) + (1 << (offset_bits - rd.r1 - 1));
    int tmp = use_jnt ? (first * fwd + res * bck) >> 4 : (first + res) >> 1;
    tmp -= round_offset;
    return clip_bd(rshift_round(tmp, 14 - rd.r0 - rd.r1), rd.bd);
}

// ---------------------------------------------------------------------------------------------------------------------
// Picture-level entry. The unit of work is one 16x16 tile of one job (both references of a compound block):
//   inter_expand_kernel  one thread per job reserves its tiles in an item list (warp scan + one atomic per warp),
//   inter_tiles_kernel   persistent warps stride over the items.
// A job whose tiles do not fit the caller's scratch (or that has more than 64 tiles) is filtered by the expanding warp
// itself, so the result never depends on the scratch size.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int MAX_REF_FRAMES = 8;
struct InterDev {
    const void *ref[MAX_REF_FRAMES][3];
    int ref_stride[MAX_REF_FRAMES][2];
    void *pred[3];
    int pred_stride[2];
    const SvtB200InterJob *jobs;
    int n_jobs, bd;
    uint32_t *count; // items reserved so far (zeroed before the expansion)
    uint32_t *items; // job << ITEM_TILE_BITS | tile, or ITEM_HOLE
    int cap;
};
constexpr int INTER_NT = 128;
constexpr uint32_t ITEM_HOLE = 0xFFFFFFFFu;
constexpr int ITEM_TILE_BITS = 7; // <= 128 tiles of 16 x 8 per job (128 x 128)

__device__ __forceinline__ int job_tiles(const SvtB200InterJob &b) {
    return ((b.bw + TILE_W - 1) / TILE_W) * ((b.bh + TILE_H - 1) / TILE_H);
}

// One tile per half warp: `valid` halves predict tile t of job b, the others only keep the warp's barriers company.
template <typename T>
__device__ __forceinline__ void predict_tile(const InterDev &d, const SvtB200InterJob &b, int t, bool valid, HalfSmem &sm, int sub) {
    const int pl = b.plane, ss = pl != 0, compound = valid && b.n_refs == 2;
    const int bw = b.bw, bh = b.bh;
    const Rounds rd = conv_rounds(d.bd, compound);
    const int ntx = (bw + TILE_W - 1) / TILE_W;
    const int ty = div_small(t, inv_small(max(ntx, 1))), tx = t - ty * ntx;
    const int tw = valid ? min(TILE_W, bw - tx * TILE_W) : 0, th = valid ? min(TILE_H, bh - ty * TILE_H) : 0;
    const Strip st = strip_of(tw, th, sub);
    const Strip idle{0, 0, 0, 0};
    // clamp_mv_to_umv_border_sb: the MV in 1/16 sample of this plane, kept within (bw + 4) samples of the picture
    const int sc = 1 << (1 - ss);
    const int spel_left = (4 + bw) << 4, spel_top = (4 + bh) << 4;
    const int passes = __any_sync(0xffffffffu, compound) ? 2 : 1;
    int val[8];
#pragma unroll 1
    for (int r = 0; r < passes; r++) {
        const bool act = valid && r <= compound;
        int col = (int16_t)((r ? b.mv_col[1] : b.mv_col[0]) * sc), row = (int16_t)((r ? b.mv_row[1] : b.mv_row[0]) * sc);
        col = (int16_t)clampi(col, b.mb_to_left_edge * sc - spel_left, b.mb_to_right_edge * sc + spel_left - 16);
        row = (int16_t)clampi(row, b.mb_to_top_edge * sc - spel_top, b.mb_to_bottom_edge * sc + spel_top - 16);
        const int spx = col & 15, spy = row & 15;
        const int px = ((b.pre_x << 4) + col) >> 4, py = ((b.pre_y << 4) + row) >> 4;
        const uint2 hx = load_half_taps(b.filter_x & 3, bw, spx);
        int fy[8];
        unpack_taps(load_half_taps(b.filter_y & 3, bh, spy), fy);
        const int rf = (r ? b.ref[1] : b.ref[0]) & (MAX_REF_FRAMES - 1);
        const T *src = (const T *)d.ref[rf][pl] + (ptrdiff_t)(py + ty * TILE_H) * d.ref_stride[rf][ss] + px + tx * TILE_W;
        conv_tile<T, 1>(src, d.ref_stride[rf][ss], tw, act ? th : 0, spx != 0, spy != 0, hx, fy, fy, rd, compound, sm, sub,
                        act ? st : idle, val);
        if (compound && r == 0) {
#pragma unroll
            for (int j = 0; j < 8; j++) sm.first[j * 16 + sub] = (uint16_t)val[j]; // through CONV_BUF (uint16), lane-private
        }
    }
    if (!valid) return;
    T *dst = (T *)d.pred[pl] + (ptrdiff_t)(b.dst_y + ty * TILE_H + st.yb) * d.pred_stride[ss] + b.dst_x + tx * TILE_W + st.x;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (j >= st.rows) break;
        const int v = compound ? jnt_average(sm.first[j * 16 + sub], val[j], b.use_jnt_comp_avg, b.fwd_offset, b.bck_offset, rd) : val[j];
        dst[(ptrdiff_t)j * d.pred_stride[ss]] = (T)v;
    }
}

template <typename T>
__global__ void __launch_bounds__(INTER_NT) inter_expand_kernel(const __grid_constant__ InterDev d) {
    __shared__ HalfSmem sm[INTER_NT / 16];
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * INTER_NT + threadIdx.x;
    const int nt = j < d.n_jobs ? job_tiles(d.jobs[j]) : 0;
    int incl = nt; // inclusive scan over the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    uint32_t base = 0;
    if (lane == 0 && total) base = atomicAdd(d.count, (uint32_t)total);
    base = __shfl_sync(0xffffffffu, base, 0) + incl - nt;
    const bool fits = nt <= (1 << ITEM_TILE_BITS) && base + nt <= (uint32_t)d.cap;
    for (int t = 0; t < nt; t++)
        if (base + t < (uint32_t)d.cap) d.items[base + t] = fits ? ((uint32_t)j << ITEM_TILE_BITS | t) : ITEM_HOLE;
    uint32_t inl = __ballot_sync(0xffffffffu, nt && !fits); // rare: filtered here, one job after the other
    while (inl) {
        const int src_lane = __ffs(inl) - 1;
        inl &= inl - 1;
        const int jj = __shfl_sync(0xffffffffu, j, src_lane);
        const SvtB200InterJob b = d.jobs[jj];
        const int n = job_tiles(b);
        for (int t = 0; t < n; t += 2) {
            const int tt = t + (lane >> 4);
            predict_tile<T>(d, b, tt, tt < n, sm[threadIdx.x >> 4], lane & 15);
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(INTER_NT, 6) inter_tiles_kernel(const __grid_constant__ InterDev d) {
    __shared__ HalfSmem sm[INTER_NT / 16];
    const int half = threadIdx.x >> 4, sub = threadIdx.x & 15; // half warps, each with its own item
    const uint32_t n = min(*d.count, (uint32_t)d.cap);
    const uint32_t n_pairs = (n + 1) >> 1, step = gridDim.x * (INTER_NT / 32);
    for (uint32_t i = blockIdx.x * (INTER_NT / 32) + (threadIdx.x >> 5); i < n_pairs; i += step) {
        const uint32_t k = 2 * i + (half & 1);
        const uint32_t item = k < n ? d.items[k] : ITEM_HOLE;
        const bool valid = item != ITEM_HOLE;
        const SvtB200InterJob b = d.jobs[valid ? item >> ITEM_TILE_BITS : 0];
        predict_tile<T>(d, b, (int)(item & ((1u << ITEM_TILE_BITS) - 1)), valid, sm[half], sub);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// RTCD drop-ins: one block through staging
// ---------------------------------------------------------------------------------------------------------------------
struct ConvArgs {
    const void *win; // staged (w + 7) x (h + 7) source window, sample (0,0) of the block at (3,3)
    uint16_t *conv;  // CONV_BUF, w x h
    void *out;       // w x h
    int w, h, r0, r1, bd;
    int sx, sy, compound, do_average, use_jnt, fwd, bck;
    int16_t fx[8], fy[8];
};

template <typename T>
__global__ void __launch_bounds__(32) convolve_dropin_kernel(const __grid_constant__ ConvArgs a) {
    __shared__ HalfSmem s[2];
    const int half = threadIdx.x >> 4, sub = threadIdx.x & 15;
    const int tx = blockIdx.x, ty = blockIdx.y * 2 + half; // the two halves take vertically adjacent tiles
    const bool valid = ty * TILE_H < a.h;
    const int tw = valid ? min(TILE_W, a.w - tx * TILE_W) : 0, th = valid ? min(TILE_H, a.h - ty * TILE_H) : 0;
    const int stride = a.w + 7;
    const Strip st = strip_of(tw, th, sub);
    int fx[8], fy[8], val[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        fx[k] = a.fx[k];
        fy[k] = a.fy[k];
    }
    const Rounds rd{a.r0, a.r1, a.bd};
    const T *src = (const T *)a.win + (ptrdiff_t)(3 + ty * TILE_H) * stride + 3 + tx * TILE_W;
    conv_tile<T, 0>(src, stride, tw, th, a.sx != 0, a.sy != 0, make_uint2(0, 0), fx, fy, rd, a.compound != 0, s[half], sub, st, val);
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (j >= st.rows) break;
        const size_t o = (size_t)(ty * TILE_H + st.yb + j) * a.w + tx * TILE_W + st.x;
        if (!a.compound)
            ((T *)a.out)[o] = (T)val[j];
        else if (!a.do_average)
            a.conv[o] = (uint16_t)val[j];
        else
            ((T *)a.out)[o] = (T)jnt_average(a.conv[o], val[j], a.use_jnt != 0, a.fwd, a.bck, rd);
    }
}

// `form` = sx * 4 + sy * 2 + compound: which of convolve[sx][sy][is_compound] (:1162-1175) this call is
template <typename T>
void convolve_run(const char *name, int form, const T *src, int src_stride, T *dst, int dst_stride, int w, int h,
                  const SvtB200InterpFilterParams *fpx, const SvtB200InterpFilterParams *fpy, int spx, int spy,
                  const SvtB200ConvolveParams *cp, int bd) {
    const int sx = form >> 2 & 1, sy = form >> 1 & 1, compound = form & 1;
    if (w <= 0 || h <= 0 || w > 128 || h > 128 || !src || !cp || (sx && (!fpx || fpx->taps != 8)) || (sy && (!fpy || fpy->taps != 8)) ||
        (compound && !cp->dst) || (!(compound && !cp->do_average) && !dst)) {
        fprintf(stderr, "%s_cuda: bad argument (w %d h %d; 8-tap kernels only)\n", name, w, h);
        abort();
    }
    const int ww = w + 7, wh = h + 7;
    Staging s({sizeof(T) * ww * wh, (size_t)2 * w * h, sizeof(T) * w * h}); // window, conv (compound), out
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, src - 3 * (ptrdiff_t)src_stride - 3, src_stride, sizeof(T), ww, wh);
    const bool avg = compound && cp->do_average;
    if (avg) s.put_rows(1, cp->dst, cp->dst_stride, 2, w, h);
    SVTB_CUDA_FATAL(s.upload(0, avg ? 1 : 0));
    ConvArgs a;
    memset(&a, 0, sizeof(a));
    a.win = s.d(0);
    a.conv = s.d<uint16_t>(1);
    a.out = s.d(2);
    a.w = w, a.h = h, a.r0 = cp->round_0, a.r1 = cp->round_1, a.bd = bd;
    a.sx = sx, a.sy = sy, a.compound = compound, a.do_average = cp->do_average;
    a.use_jnt = cp->use_jnt_comp_avg, a.fwd = cp->fwd_offset, a.bck = cp->bck_offset;
    if (sx) memcpy(a.fx, fpx->filter_ptr + 8 * (spx & 15), 16); // av1_get_interp_filter_subpel_kernel
    if (sy) memcpy(a.fy, fpy->filter_ptr + 8 * (spy & 15), 16);
    SVTB_LAUNCH(convolve_dropin_kernel<T>, dim3((w + TILE_W - 1) / TILE_W, (h + 2 * TILE_H - 1) / (2 * TILE_H)), 32, 0, s.stream(), a);
    const bool to_conv = compound && !cp->do_average;
    SVTB_CUDA_FATAL(s.download(to_conv ? 1 : 2, to_conv ? 1 : 2));
    if (to_conv)
        s.get_rows(1, cp->dst, cp->dst_stride, 2, w, h);
    else
        s.get_rows(2, dst, dst_stride, sizeof(T), w, h);
}

// svt_aom_convolve8_horiz / vert: position q0 + i * step sixteenths along the filtered axis
struct Conv8Args {
    const uint8_t *win; // staged window; the sample the first output is centred on sits at (3,3) along the filtered axis
    uint8_t *out;
    int w, h, stride, q0, step, vert;
    int16_t table[16][8];
};
__global__ void convolve8_kernel(const __grid_constant__ Conv8Args a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.w * a.h) return;
    const int y = i / a.w, x = i - y * a.w;
    const int q = a.q0 + (a.vert ? y : x) * a.step;
    const int16_t *f = a.table[q & 15];
    const uint8_t *p = a.vert ? a.win + (size_t)(q >> 4) * a.stride + x : a.win + (size_t)y * a.stride + (q >> 4);
    const int inc = a.vert ? a.stride : 1;
    int sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) sum += f[k] * p[k * inc];
    a.out[i] = (uint8_t)clip_bd(rshift_round(sum, 7), 8);
}

void convolve8_run(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst, ptrdiff_t dst_stride, const int16_t *filter, int step,
                   int w, int h, int vert) {
    if (w <= 0 || h <= 0 || w > 128 || h > 136 || step <= 0 || step > 64 || !filter || !src || !dst) {
        fprintf(stderr, "svt_aom_convolve8_%s_cuda: bad argument\n", vert ? "vert" : "horiz");
        abort();
    }
    // get_filter_base / get_filter_offset (convolve.c:49-57): the pointer addresses one row of a 256-byte aligned table
    const int16_t *base = (const int16_t *)((uintptr_t)filter & ~(uintptr_t)0xFF);
    Conv8Args a;
    memcpy(a.table, base, sizeof(a.table));
    a.q0 = (int)((filter - base) / 8);
    a.step = step, a.w = w, a.h = h, a.vert = vert;
    const int span = ((((vert ? h : w) - 1) * step + a.q0) >> 4) + 8; // samples touched along the filtered axis
    const int ww = vert ? w : span, wh = vert ? span : h;
    a.stride = ww;
    Staging s({(size_t)ww * wh, (size_t)w * h});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, vert ? src - 3 * src_stride : src - 3, src_stride, 1, ww, wh);
    SVTB_CUDA_FATAL(s.upload(0, 0));
    a.win = s.d(0);
    a.out = s.d(1);
    SVTB_LAUNCH(convolve8_kernel, (w * h + 127) / 128, 128, 0, s.stream(), a);
    SVTB_CUDA_FATAL(s.download(1, 1));
    s.get_rows(1, dst, dst_stride, 1, w, h);
}

} // namespace
} // namespace svtb200

using namespace svtb200;

extern "C" {

#define SVTB_CONVOLVE_DEF(NAME, FORM)                                                                                            \
    void NAME##_cuda(const uint8_t *src, int32_t src_stride, uint8_t *dst, int32_t dst_stride, int32_t w, int32_t h,             \
                     SvtB200InterpFilterParams *fpx, SvtB200InterpFilterParams *fpy, const int32_t spx, const int32_t spy,       \
                     SvtB200ConvolveParams *cp) {                                                                                \
        convolve_run<uint8_t>(#NAME, FORM, src, src_stride, dst, dst_stride, w, h, fpx, fpy, spx, spy, cp, 8);                   \
    }
#define SVTB_HBD_CONVOLVE_DEF(NAME, FORM)                                                                                        \
    void NAME##_cuda(const uint16_t *src, int32_t src_stride, uint16_t *dst, int32_t dst_stride, int32_t w, int32_t h,           \
                     const SvtB200InterpFilterParams *fpx, const SvtB200InterpFilterParams *fpy, const int32_t spx,              \
                     const int32_t spy, SvtB200ConvolveParams *cp, int32_t bd) {                                                 \
        convolve_run<uint16_t>(#NAME, FORM, src, src_stride, dst, dst_stride, w, h, fpx, fpy, spx, spy, cp, bd);                 \
    }
SVTB_CONVOLVE_DEF(svt_av1_convolve_2d_copy_sr, 0)
SVTB_CONVOLVE_DEF(svt_av1_jnt_convolve_2d_copy, 1)
SVTB_CONVOLVE_DEF(svt_av1_convolve_y_sr, 2)
SVTB_CONVOLVE_DEF(svt_av1_jnt_convolve_y, 3)
SVTB_CONVOLVE_DEF(svt_av1_convolve_x_sr, 4)
SVTB_CONVOLVE_DEF(svt_av1_jnt_convolve_x, 5)
SVTB_CONVOLVE_DEF(svt_av1_convolve_2d_sr, 6)
SVTB_CONVOLVE_DEF(svt_av1_jnt_convolve_2d, 7)
SVTB_HBD_CONVOLVE_DEF(svt_av1_highbd_convolve_2d_copy_sr, 0)
SVTB_HBD_CONVOLVE_DEF(svt_av1_highbd_jnt_convolve_2d_copy, 1)
SVTB_HBD_CONVOLVE_DEF(svt_av1_highbd_convolve_y_sr, 2)
SVTB_HBD_CONVOLVE_DEF(svt_av1_highbd_jnt_convolve_y, 3)
SVTB_HBD_CONVOLVE_DEF(svt_av1_highbd_convolve_x_sr, 4)
SVTB_HBD_CONVOLVE_DEF(svt_av1_highbd_jnt_convolve_x, 5)
SVTB_HBD_CONVOLVE_DEF(svt_av1_highbd_convolve_2d_sr, 6)
SVTB_HBD_CONVOLVE_DEF(svt_av1_highbd_jnt_convolve_2d, 7)

void svt_aom_convolve8_horiz_cuda(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst, ptrdiff_t dst_stride, const int16_t *filter_x,
                                  int x_step_q4, const int16_t *filter_y, int y_step_q4, int w, int h) {
    (void)filter_y, (void)y_step_q4;
    convolve8_run(src, src_stride, dst, dst_stride, filter_x, x_step_q4, w, h, 0);
}
void svt_aom_convolve8_vert_cuda(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst, ptrdiff_t dst_stride, const int16_t *filter_x,
                                 int x_step_q4, const int16_t *filter_y, int y_step_q4, int w, int h) {
    (void)filter_x, (void)x_step_q4;
    convolve8_run(src, src_stride, dst, dst_stride, filter_y, y_step_q4, w, h, 1);
}

void svt_aom_upsampled_pred_cuda(void *xd, const void *cm, int mi_row, int mi_col, const void *mv, uint8_t *comp_pred, int width,
                                 int height, int subpel_x_q3, int subpel_y_q3, const uint8_t *ref, int ref_stride, int subpel_search) {
    (void)xd, (void)cm, (void)mi_row, (void)mi_col, (void)mv;
    if (subpel_search < 1 || subpel_search > 3 || width <= 0 || height <= 0 || width > 128 || height > 128 || !comp_pred || !ref) {
        fprintf(stderr, "svt_aom_upsampled_pred_cuda: bad argument\n");
        abort();
    }
    if (!subpel_x_q3 && !subpel_y_q3) {
        for (int i = 0; i < height; i++) memcpy(comp_pred + (size_t)i * width, ref + (ptrdiff_t)i * ref_stride, (size_t)width);
        return;
    }
    // av1_get_filter (variance.c:200-210): bilinear / the regular 4-tap / the regular 8-tap kernels, as a 256-byte aligned
    // [16][8] table the way svt_aom_convolve8_* locate it (get_filter_base)
    alignas(256) int16_t table[16][8];
    for (int sp = 0; sp < 16; sp++) svt_b200_get_interp_kernel(subpel_search == 1 ? 3 : 0, subpel_search == 3 ? 8 : 4, sp, table[sp]);
    if (!subpel_y_q3) {
        convolve8_run(ref, ref_stride, comp_pred, width, table[subpel_x_q3 << 1], 16, width, height, 0);
    } else if (!subpel_x_q3) {
        convolve8_run(ref, ref_stride, comp_pred, width, table[subpel_y_q3 << 1], 16, width, height, 1);
    } else { // both: the first pass over height + 7 rows is rounded to 8 bits before the second
        static thread_local uint8_t temp[(128 + 8) * 128];
        const int ih = height + 7;
        convolve8_run(ref - 3 * (ptrdiff_t)ref_stride, ref_stride, temp, width, table[subpel_x_q3 << 1], 16, width, ih, 0);
        convolve8_run(temp + 3 * width, width, comp_pred, width, table[subpel_y_q3 << 1], 16, width, height, 1);
    }
}

int svt_b200_get_interp_kernel(int32_t interp_filter, int32_t w, int32_t subpel, int16_t out[8]) {
    if (interp_filter < 0 || interp_filter > 3 || w <= 0 || subpel < 0 || subpel > 15 || !out) {
        set_error("svt_b200_get_interp_kernel: bad argument");
        return SVT_B200_ERR_ARG;
    }
    const int t = table_of(interp_filter, w);
    for (int k = 0; k < 8; k++) out[k] = t < 0 ? 0 : (int16_t)(2 * h_half_taps[t][subpel][k]);
    if (t < 0) {
        out[3] = (int16_t)(128 - 8 * subpel);
        out[4] = (int16_t)(8 * subpel);
    }
    return SVT_B200_OK;
}

size_t svt_b200_inter_predict_scratch_bytes(int32_t n_jobs, int32_t width, int32_t height) {
    if (n_jobs < 0 || width <= 0 || height <= 0) return 0;
    // one item per 16x8 tile: a block of AV1 shape has at most 1 + area / 64 of them, and non-overlapping jobs cover at most
    // the three planes of the (64-aligned) picture
    const size_t area = (size_t)(width + 64) * (height + 64) * 3 / 2;
    return 256 + 4 * ((size_t)n_jobs + area / 64);
}

int svt_b200_inter_predict(const SvtB200Frame *refs, int32_t n_ref_frames, const SvtB200Frame *pred, const SvtB200InterJob *jobs,
                           int32_t n_jobs, void *scratch, size_t scratch_bytes, void *stream) {
    if (!refs || !pred || n_ref_frames < 1 || n_ref_frames > MAX_REF_FRAMES || n_jobs < 0 || n_jobs >= (1 << (32 - ITEM_TILE_BITS)) || (n_jobs && !jobs) ||
        !scratch || scratch_bytes < 256 || (pred->bit_depth != 8 && pred->bit_depth != 10 && pred->bit_depth != 12)) {
        set_error("svt_b200_inter_predict: bad argument (1..%d reference pictures, scratch >= 256 bytes)", MAX_REF_FRAMES);
        return SVT_B200_ERR_ARG;
    }
    if (n_jobs == 0) return SVT_B200_OK;
    if (int rc = upload_tables()) return rc;
    InterDev d;
    memset(&d, 0, sizeof(d));
    for (int i = 0; i < n_ref_frames; i++) {
        if (refs[i].bit_depth != pred->bit_depth) {
            set_error("svt_b200_inter_predict: reference %d has another bit depth", i);
            return SVT_B200_ERR_ARG;
        }
        d.ref[i][0] = refs[i].y, d.ref[i][1] = refs[i].cb, d.ref[i][2] = refs[i].cr;
        d.ref_stride[i][0] = refs[i].stride_y, d.ref_stride[i][1] = refs[i].stride_c;
    }
    d.pred[0] = pred->y, d.pred[1] = pred->cb, d.pred[2] = pred->cr;
    d.pred_stride[0] = pred->stride_y, d.pred_stride[1] = pred->stride_c;
    d.jobs = jobs, d.n_jobs = n_jobs, d.bd = pred->bit_depth;
    d.count = (uint32_t *)scratch;
    d.items = (uint32_t *)scratch + 64;
    d.cap = (int)std::min<size_t>((scratch_bytes - 256) / 4, (size_t)1 << 30);
    cudaStream_t st = (cudaStream_t)stream;
    // SM count and occupancy are per device (a process may drive several GPUs): cached per device ordinal
    int dev = 0;
    SVTB_CUDA_TRY(cudaGetDevice(&dev));
    dev &= 63;
    static std::atomic<int> n_sm_dev[64], occ_dev[64][2];
    int n_sm = n_sm_dev[dev].load();
    if (!n_sm) {
        SVTB_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
        n_sm_dev[dev].store(n_sm);
    }
    SVTB_CUDA_TRY(cudaMemsetAsync(d.count, 0, 4, st));
    const int hb = d.bd > 8;
    int occ = occ_dev[dev][hb].load(); // resident CTAs per SM of the persistent kernel
    if (!occ) {
        if (hb)
            SVTB_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, inter_tiles_kernel<uint16_t>, INTER_NT, 0));
        else
            SVTB_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, inter_tiles_kernel<uint8_t>, INTER_NT, 0));
        occ_dev[dev][hb].store(occ);
    }
    const int g1 = (n_jobs + INTER_NT - 1) / INTER_NT, g2 = n_sm * std::max(occ, 1);
    if (d.bd == 8) {
        SVTB_LAUNCH(inter_expand_kernel<uint8_t>, g1, INTER_NT, 0, st, d);
        SVTB_LAUNCH(inter_tiles_kernel<uint8_t>, g2, INTER_NT, 0, st, d);
    } else {
        SVTB_LAUNCH(inter_expand_kernel<uint16_t>, g1, INTER_NT, 0, st, d);
        SVTB_LAUNCH(inter_tiles_kernel<uint16_t>, g2, INTER_NT, 0, st, d);
    }
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

} // extern "C"
