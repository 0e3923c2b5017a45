// txfm.cu — residual, forward/inverse 2-D transforms and quantisation on sm_90a.
//
// Replaces (reference files under Source/Lib):
//   svt_residual_kernel8bit/16bit                    Common/Codec/EbPictureOperators.c:106-150
//   svt_av1_fwd_txfm2d_* / svt_av1_transform_two_d_* Encoder/Codec/EbTransforms.c:2301-3053 (19 sizes x 16 types)
//   svt_handle_transform64x64/64x32/32x64/64x16/16x64 Encoder/Codec/EbTransforms.c:2763-2931
//   svt_av1_inv_txfm2d_add_*                         Common/Codec/EbInvTransforms.c:2455-2752
//   svt_aom_quantize_b / svt_aom_highbd_quantize_b   Encoder/Codec/EbFullLoop.c:37-93, 171-225
//   svt_av1_quantize_fp[_32x32/_64x64], svt_av1_highbd_quantize_fp  Encoder/Codec/EbFullLoop.c:314-600
//   the per-TU body of av1_encode_loop (EbCodingLoop.c:290-...) as ONE fused kernel:
//       residual -> forward txfm -> quantise/dequantise -> inverse txfm -> reconstruct
//
// Design: a transform block lives in shared memory for its whole life (w x h int32, odd pitch); one thread
// owns a column in the column pass and a row in the row pass, so a 64x64 block is 64 lanes and small blocks
// are packed several per CTA.  In the fused kernel HBM sees only src + pred in and qcoeff + recon out
// (7 B/px for 8-bit, SURVEY §8d) — the int32 coefficient planes of the reference's five separate calls never
// leave the SM.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "txfm.cuh"

#include <cmath>
#include <mutex>

namespace svtb200 {

__constant__ uint8_t c_txw[19] = {4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64};
__constant__ uint8_t c_txh[19] = {4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16};
__constant__ int8_t c_fwd_shift[19][3] = {{2, 0, 0},  {2, -1, 0}, {2, -2, 0}, {2, -4, 0}, {0, -2, -2}, {2, -1, 0}, {2, -1, 0},
                                          {2, -2, 0}, {2, -2, 0}, {2, -4, 0}, {2, -4, 0}, {0, -2, -2}, {2, -4, -2}, {2, -1, 0},
                                          {2, -1, 0}, {2, -2, 0}, {2, -2, 0}, {0, -2, 0}, {2, -4, 0}};
__constant__ int8_t c_inv_shift0[19] = {0, -1, -2, -2, -2, 0, 0, -1, -1, -1, -1, -1, -1, -1, -1, -2, -2, -2, -2};
__constant__ int8_t c_fwd_cos_col[5][5] = {{13, 13, 13, 0, 0}, {13, 13, 13, 12, 0}, {13, 13, 13, 12, 13}, {0, 13, 13, 12, 13}, {0, 0, 13, 12, 13}};
__constant__ int8_t c_fwd_cos_row[5][5] = {{13, 13, 12, 0, 0}, {13, 13, 13, 12, 0}, {13, 13, 12, 13, 12}, {0, 12, 13, 12, 11}, {0, 0, 12, 11, 10}};
__constant__ uint8_t c_vtx[16] = {0, 1, 0, 1, 2, 0, 2, 1, 2, 3, 0, 3, 1, 3, 2, 3};
__constant__ uint8_t c_htx[16] = {0, 0, 1, 1, 0, 2, 2, 2, 1, 3, 3, 0, 3, 1, 3, 2};

static const uint8_t h_txw[19] = {4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64};
static const uint8_t h_txh[19] = {4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16};

__device__ TxCfg make_txcfg(int tx_size, int tx_type) {
    TxCfg t;
    t.w = c_txw[tx_size];
    t.h = c_txh[tx_size];
    t.vk = c_vtx[tx_type];
    t.hk = c_htx[tx_type];
    t.ud = t.vk == 2;
    t.lr = t.hk == 2;
    t.fs0 = c_fwd_shift[tx_size][0];
    t.fs1 = c_fwd_shift[tx_size][1];
    t.fs2 = c_fwd_shift[tx_size][2];
    t.is0 = c_inv_shift0[tx_size];
    t.is1 = -4;
    const int wi = ilog2(t.w) - 2, hi = ilog2(t.h) - 2;
    t.cbc = c_fwd_cos_col[wi][hi];
    t.cbr = c_fwd_cos_row[wi][hi];
    t.rect = (t.w == 2 * t.h) || (t.h == 2 * t.w);
    return t;
}

} // namespace svtb200

using namespace svtb200;

namespace {

constexpr int TX_NT = 128; // threads per CTA of the transform kernels
__host__ __device__ inline int tx_pitch(int w) { return w | 1; } // odd pitch: conflict-free row pass

// One descriptor per transform unit of a batched launch.
struct TuDev {
    int32_t x, y; // top-left sample inside the plane
    int32_t plane; // 0 Y, 1 Cb, 2 Cr
    int32_t tx_type;
};

// ---------------------------------------------------------------------------------------------------------------
// forward: residual (int16, strided) -> coefficients (int32, contiguous w x h; 64-wide sizes optionally re-packed)
// ---------------------------------------------------------------------------------------------------------------
struct FwdArgs {
    const int16_t *in; // block b at in + b * in_block_stride
    size_t in_block_stride;
    int in_stride;
    int32_t *out; // block b at out + b * w*h
    const int32_t *tx_types; // per block (device) or null -> tx_type
    int tx_type, tx_size, n_blocks;
    int pf_shift; // 0 full, 1 N2, 2 N4: keep only the top-left (w>>s) x (h>>s) coefficients (EbTransforms.c:5401,7007)
    int repack64; // 1: svt_handle_transform* semantics (zero the dropped area, pack 32-wide, energy -> energy[b])
    uint64_t *energy;
};
__global__ void __launch_bounds__(TX_NT) fwd_txfm_kernel(const FwdArgs a) {
    extern __shared__ int32_t sm[];
    const int w = c_txw[a.tx_size], h = c_txh[a.tx_size];
    const int T = max(w, h), bpc = TX_NT / T, pitch = tx_pitch(w);
    const int lb = threadIdx.x / T, li = threadIdx.x % T;
    const int b = blockIdx.x * bpc + lb;
    const bool live = b < a.n_blocks && lb < bpc;
    int32_t *buf = sm + lb * (pitch * h);
    TxCfg t = make_txcfg(a.tx_size, live && a.tx_types ? a.tx_types[b] : a.tx_type);
    if (live) {
        const int16_t *src = a.in + (size_t)b * a.in_block_stride;
        for (int i = li; i < w * h; i += T) {
            const int r = i / w, c = i - r * w;
            buf[r * pitch + c] = src[(size_t)(t.ud ? h - 1 - r : r) * a.in_stride + (t.lr ? w - 1 - c : c)];
        }
    }
    __syncthreads();
    if (live) {
        for (int c = li; c < t.w; c += T) { /* column pass */
            const int fs0 = t.fs0, fs1 = t.fs1;
            fwd_1d_pass(buf + c, pitch, t.h, t.vk, t.cbc, [=](int32_t v) { return (int32_t)((uint32_t)v << fs0); },
                        [=](int32_t v) { return fs1 ? round_shift64((long long)v, -fs1) : v; });
        }
    }
    __syncthreads();
    if (live) {
        for (int r = li; r < t.h; r += T) { /* row pass */
            const int fs2 = t.fs2, rect = t.rect;
            fwd_1d_pass(buf + r * pitch, 1, t.w, t.hk, t.cbr, [](int32_t v) { return v; }, [=](int32_t v) {
                if (fs2) v = round_shift64((long long)v, -fs2);
                if (rect) v = round_shift64((long long)v * 5793, 12);
                return v;
            });
        }
    }
    __syncthreads();
    __shared__ unsigned long long s_e2[TX_NT];
    unsigned long long e = 0;
    if (live) {
        int32_t *dst = a.out + (size_t)b * w * h;
        if (!a.repack64) {
            const int kw2 = w >> a.pf_shift, kh2 = h >> a.pf_shift;
            for (int i = li; i < w * h; i += T) dst[i] = ((i % w) < kw2 && (i / w) < kh2) ? buf[(i / w) * pitch + (i % w)] : 0;
        } else {
            // svt_handle_transform* (EbTransforms.c:2763-2931): energy of the dropped area, zero it, then re-pack the
            // kept 32-wide rows to the front.  Entries behind the packed block keep what the in-place C code leaves.
            const int kw = min(w, 32), kh = min(h, 32);
            for (int i = li; i < w * h; i += T) {
                const int r = i / w, c = i - r * w;
                const int32_t v = buf[r * pitch + c];
                const bool dropped = r >= kh || c >= kw;
                if (dropped) e += (unsigned long long)((long long)v * (long long)v);
                dst[i] = (kw != w && i < kw * kh) ? buf[(i / kw) * pitch + (i % kw)] : (dropped ? 0 : v);
            }
        }
    }
    if (a.repack64) { // uniform branch: CTA-wide barrier is safe
        s_e2[threadIdx.x] = e;
        __syncthreads();
        if (live && li == 0 && a.energy) {
            unsigned long long tot = 0;
            for (int i = 0; i < T; i++) tot += s_e2[lb * T + i];
            a.energy[b] = tot;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// inverse: coefficients -> residual added to the prediction, clipped (svt_av1_inv_txfm2d_add_*)
// ---------------------------------------------------------------------------------------------------------------
struct InvArgs {
    const int32_t *in; // block b at in + b * iw*ih (64-wide sizes: 32-wide packed input)
    const uint16_t *pred;
    uint16_t *recon; // block b at + b * block_stride
    size_t pred_block_stride, recon_block_stride;
    int stride_r, stride_w;
    int tx_type, tx_size, n_blocks, bd;
};
__global__ void __launch_bounds__(TX_NT) inv_txfm_kernel(const InvArgs a) {
    extern __shared__ int32_t sm[];
    const int w = c_txw[a.tx_size], h = c_txh[a.tx_size];
    const int iw = min(w, 32), ih = min(h, 32);
    const int T = max(w, h), bpc = TX_NT / T, pitch = tx_pitch(w);
    const int lb = threadIdx.x / T, li = threadIdx.x % T;
    const int b = blockIdx.x * bpc + lb;
    const bool live = b < a.n_blocks && lb < bpc;
    int32_t *buf = sm + lb * (pitch * h);
    TxCfg t = make_txcfg(a.tx_size, a.tx_type);
    if (live) {
        const int32_t *src = a.in + (size_t)b * iw * ih;
        for (int i = li; i < w * h; i += T) {
            const int r = i / w, c = i - r * w;
            buf[r * pitch + c] = (r < ih && c < iw) ? src[r * iw + c] : 0;
        }
    }
    __syncthreads();
    const int bd = a.bd;
    const int range_row = bd == 8 ? 16 : bd == 10 ? 18 : 20, range_col = bd == 8 ? 16 : bd == 10 ? 16 : 18;
    if (live) {
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
    __syncthreads();
    if (live) {
        const uint16_t *pr = a.pred + (size_t)b * a.pred_block_stride;
        uint16_t *rc = a.recon + (size_t)b * a.recon_block_stride;
        const int mx = (1 << bd) - 1;
        for (int i = li; i < w * h; i += T) {
            const int r = i / w, c = i - r * w;
            // lr flip: output column c is the transform of buffer column w-1-c; ud flip: output row r = result row h-1-r
            const int32_t res = buf[(t.ud ? h - 1 - r : r) * pitch + (t.lr ? w - 1 - c : c)];
            const long long v = (long long)pr[(size_t)r * a.stride_r + c] + res;
            rc[(size_t)r * a.stride_w + c] = (uint16_t)(v < 0 ? 0 : (v > mx ? mx : v));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// quantisers (one CTA per coefficient block; thread i handles scan position i, i+blockDim, ...)
// ---------------------------------------------------------------------------------------------------------------
struct QuantTab { // dc/ac pairs, as the reference's zbin_ptr/round_ptr/quant_ptr/quant_shift_ptr/dequant_ptr
    int16_t zbin[2], round[2], quant[2], quant_shift[2], dequant[2];
};
__device__ __forceinline__ int rpot(int v, int n) { return n ? (v + (1 << (n - 1))) >> n : v; }

// mode: 0 quantize_b lowbd, 1 quantize_b highbd, 2 quantize_fp lowbd, 3 quantize_fp highbd
__device__ __forceinline__ void quant_one(int mode, int c, int ac, const QuantTab &q, int log_scale, int wt, int iwt,
                                          int32_t &qc, int32_t &dqc) {
    const int sign = c < 0 ? -1 : 0;
    const int abs_c = (c ^ sign) - sign;
    qc = 0;
    dqc = 0;
    if (mode <= 1) {
        const int zb = rpot(q.zbin[ac], log_scale);
        bool keep;
        if (mode == 1) {
            const int cw = c * wt;
            keep = cw >= zb * 32 || cw <= -zb * 32;
        } else {
            keep = abs_c * wt >= (zb << 5);
        }
        if (!keep) return;
        long long tmp = (long long)abs_c + rpot(q.round[ac], log_scale);
        if (mode == 0) tmp = tmp < -32768 ? -32768 : (tmp > 32767 ? 32767 : tmp);
        tmp *= wt;
        const int32_t v = (int32_t)(((((tmp * q.quant[ac]) >> 16) + tmp) * q.quant_shift[ac]) >> (16 - log_scale + 5));
        qc = (v ^ sign) - sign;
        const int dq = (q.dequant[ac] * iwt + 16) >> 5;
        const int32_t adq = (int32_t)((uint32_t)v * (uint32_t)dq) >> log_scale;
        dqc = (adq ^ sign) - sign;
    } else {
        const int rounding = rpot(q.round[ac], log_scale);
        if (mode == 3) {
            if ((abs_c << (1 + log_scale)) >= q.dequant[ac]) {
                const int v = (int)((((long long)abs_c + rounding) * q.quant[ac]) >> (16 - log_scale));
                qc = (v ^ sign) - sign;
                const int32_t adq = (int32_t)((uint32_t)v * (uint32_t)q.dequant[ac]) >> log_scale;
                dqc = (adq ^ sign) - sign;
            }
        } else if (((long long)abs_c << (1 + log_scale)) >= (int)q.dequant[ac]) {
            long long a = (long long)abs_c + rounding;
            a = a < -32768 ? -32768 : (a > 32767 ? 32767 : a);
            const int v = (int)((a * q.quant[ac]) >> (16 - log_scale));
            if (v) {
                qc = (v ^ sign) - sign;
                const int32_t adq = (int32_t)((uint32_t)v * (uint32_t)q.dequant[ac]) >> log_scale;
                dqc = (adq ^ sign) - sign;
            }
        }
    }
}

struct QuantArgs {
    const int32_t *coeff;
    int32_t *qcoeff, *dqcoeff;
    uint16_t *eob;
    const int16_t *scan;
    const uint8_t *qm, *iqm;
    QuantTab q;
    int n, log_scale, mode;
};
__global__ void __launch_bounds__(256) quant_kernel(const QuantArgs a) {
    __shared__ int s_eob;
    if (threadIdx.x == 0) s_eob = 0;
    __syncthreads();
    int eob = 0;
    for (int i = threadIdx.x; i < a.n; i += blockDim.x) {
        const int rc = a.scan[i];
        int32_t qc, dqc;
        quant_one(a.mode, a.coeff[rc], rc != 0, a.q, a.log_scale, a.qm ? a.qm[rc] : 32, a.iqm ? a.iqm[rc] : 32, qc, dqc);
        a.qcoeff[rc] = qc;
        a.dqcoeff[rc] = dqc;
        if (qc) eob = max(eob, i + 1);
    }
    eob = __reduce_max_sync(0xffffffffu, eob);
    if ((threadIdx.x & 31) == 0) atomicMax(&s_eob, eob);
    __syncthreads();
    if (threadIdx.x == 0) *a.eob = (uint16_t)s_eob;
}

template <typename T>
__global__ void residual_kernel(const T *src, int ss, const T *pred, int ps, int16_t *res, int rs, int w, int h) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < w * h; i += gridDim.x * blockDim.x) {
        const int y = i / w, x = i - y * w;
        res[(size_t)y * rs + x] = (int16_t)((int)src[(size_t)y * ss + x] - (int)pred[(size_t)y * ps + x]);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// fused per-TU encode: residual -> fwd txfm -> quant/dequant -> inverse txfm -> recon (av1_encode_loop body)
// ---------------------------------------------------------------------------------------------------------------
struct EncodeDev {
    const void *src[3], *pred[3];
    void *recon[3];
    int src_stride[3], pred_stride[3], recon_stride[3];
    int hbd, bd;
    const TuDev *tus;
    int n_tus, tx_size;
    const int16_t *iscan[3]; // device INVERSE scan tables (raster position -> scan index): default / mrow (V_*) / mcol (H_*)
    QuantTab q[3]; // per plane
    int quant_mode; // 0 quantize_b, 2 quantize_fp (the highbd variants are chosen from hbd)
    int32_t *qcoeff; // [n_tus][iw*ih]
    uint16_t *eob; // [n_tus]
    int32_t *cul_level; // [n_tus] or null: av1_quantize_inv_quantize's return value (EbFullLoop.c:1596-1608)
    int pf_shape; // EB_TRANS_COEFF_SHAPE of av1_estimate_transform: 0 default, 1 N2, 2 N4, 3 ONLY_DC (EbTransforms.c:3613-3670)
    const long long *qoff; // null: TU b writes qcoeff + b * n, eob[b]; else qcoeff + qoff[b] and eob / cul_level [out_idx[b]]
    const int32_t *out_idx;
};
// four horizontally adjacent samples at p (any alignment): aligned 32-bit loads + funnel shift for bytes
template <typename T>
__device__ __forceinline__ void load4(const T *p, int (&v)[4]) {
    if (sizeof(T) == 1) {
        const uintptr_t a = (uintptr_t)p;
        const uint32_t *g = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
        const uint32_t w = __funnelshift_r(g[0], (a & 3) ? g[1] : 0u, (int)(a & 3) * 8);
        v[0] = w & 0xff, v[1] = (w >> 8) & 0xff, v[2] = (w >> 16) & 0xff, v[3] = w >> 24;
    } else if (((uintptr_t)p & 3) == 0) {
        const uint32_t w0 = reinterpret_cast<const uint32_t *>(p)[0], w1 = reinterpret_cast<const uint32_t *>(p)[1];
        v[0] = w0 & 0xffff, v[1] = w0 >> 16, v[2] = w1 & 0xffff, v[3] = w1 >> 16;
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] = (int)p[j];
    }
}
template <typename T>
__device__ __forceinline__ void store4(T *p, const int (&v)[4]) {
    if (sizeof(T) == 1 && ((uintptr_t)p & 3) == 0) {
        *reinterpret_cast<uint32_t *>(p) = (uint32_t)v[0] | ((uint32_t)v[1] << 8) | ((uint32_t)v[2] << 16) | ((uint32_t)v[3] << 24);
    } else if (sizeof(T) == 2 && ((uintptr_t)p & 3) == 0) {
        reinterpret_cast<uint32_t *>(p)[0] = (uint32_t)v[0] | ((uint32_t)v[1] << 16);
        reinterpret_cast<uint32_t *>(p)[1] = (uint32_t)v[2] | ((uint32_t)v[3] << 16);
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++) p[j] = (T)v[j];
    }
}

// TS >= 0: kernel specialised for that tx_size (TX_4X4..TX_32X32: every loop bound, the 1-D sizes and the dispatch
// inside fwd/inv_1d_pass are compile-time, which also keeps the straight-line transform code of the other sizes out of
// the instruction cache); TS = -1: any size.
template <typename T, int TS>
__global__ void __launch_bounds__(TX_NT) encode_tu_kernel(const __grid_constant__ EncodeDev d) {
    extern __shared__ int32_t sm[];
    const int w = TS >= 0 ? (4 << TS) : c_txw[d.tx_size], h = TS >= 0 ? (4 << TS) : c_txh[d.tx_size];
    const int iw = min(w, 32), ih = min(h, 32), n = iw * ih;
    const int lw = 31 - __clz(w), liw = 31 - __clz(iw);
    const int Tn = max(w, h), bpc = TX_NT / Tn, pitch = tx_pitch(w);
    const int lb = threadIdx.x / Tn, li = threadIdx.x % Tn;
    const int b = blockIdx.x * bpc + lb;
    const bool live = b < d.n_tus && lb < bpc;
    int32_t *buf = sm + lb * (pitch * h);
    __shared__ int s_eob[TX_NT / 4], s_cul[TX_NT / 4];
    TuDev tu = {0, 0, 0, 0};
    if (live) tu = d.tus[b];
    TxCfg t = make_txcfg(TS >= 0 ? TS : d.tx_size, tu.tx_type);
    if (TS >= 0) t.w = t.h = 4 << TS;
    const int pl = tu.plane;
    int dc_sign = 0; // set_dc_sign: 1 negative, 2 positive DC level (held by the thread that quantises position 0)
    if (live) { // residual, four samples per step
        const T *sp = reinterpret_cast<const T *>(d.src[pl]) + (size_t)tu.y * d.src_stride[pl] + tu.x;
        const T *pp = reinterpret_cast<const T *>(d.pred[pl]) + (size_t)tu.y * d.pred_stride[pl] + tu.x;
        for (int i = li; i < (w * h) >> 2; i += Tn) {
            const int r = i >> (lw - 2), c = (i & ((w >> 2) - 1)) << 2;
            const int rr = t.ud ? h - 1 - r : r, cc = t.lr ? w - 4 - c : c;
            int sv[4], pv[4];
            load4<T>(sp + (size_t)rr * d.src_stride[pl] + cc, sv);
            load4<T>(pp + (size_t)rr * d.pred_stride[pl] + cc, pv);
#pragma unroll
            for (int j = 0; j < 4; j++) buf[r * pitch + c + j] = sv[t.lr ? 3 - j : j] - pv[t.lr ? 3 - j : j];
        }
        if (li == 0) s_eob[lb] = s_cul[lb] = 0;
    }
    __syncthreads();
    if (live)
        for (int c = li; c < t.w; c += Tn) {
            const int fs0 = t.fs0, fs1 = t.fs1;
            fwd_1d_pass(buf + c, pitch, t.h, t.vk, t.cbc, [=](int32_t v) { return (int32_t)((uint32_t)v << fs0); },
                        [=](int32_t v) { return fs1 ? round_shift64((long long)v, -fs1) : v; });
        }
    __syncthreads();
    if (live)
        for (int r = li; r < t.h; r += Tn) {
            const int fs2 = t.fs2, rect = t.rect;
            fwd_1d_pass(buf + r * pitch, 1, t.w, t.hk, t.cbr, [](int32_t v) { return v; }, [=](int32_t v) {
                if (fs2) v = round_shift64((long long)v, -fs2);
                if (rect) v = round_shift64((long long)v * 5793, 12);
                return v;
            });
        }
    __syncthreads();
    // quantise + dequantise in place, in raster order (every coefficient is quantised independently; the scan order
    // only defines eob = 1 + the largest scan index of a non-zero level, looked up for the non-zero levels only).
    // Coefficients outside the kept 32x32 of 64-wide sizes are dropped = 0.
    if (live) {
        const int log_scale = (w * h > 256) + (w * h > 1024); // av1_get_tx_scale
        const int mode = d.quant_mode + (d.hbd ? 1 : 0);
        const int16_t *iscan = d.iscan[(t.vk != 3 && t.hk == 3) ? 1 : (t.vk == 3 && t.hk != 3) ? 2 : 0];
        int32_t *qout = d.qoff ? d.qcoeff + d.qoff[b] : d.qcoeff + (size_t)b * n;
        // partial-frequency shapes: the N2 / N4 transforms produce the top-left half / quarter (per dimension) of the
        // default transform's coefficients and zeros elsewhere; ONLY_DC keeps coefficient 0 alone
        const int kw = d.pf_shape == 3 ? 1 : min(iw, w >> d.pf_shape), kh = d.pf_shape == 3 ? 1 : min(ih, h >> d.pf_shape);
        int eob = 0, lvl = 0;
        for (int i = li; i < n; i += Tn) {
            const int r = i >> liw, c = i & (iw - 1);
            int32_t qc, dqc;
            const int32_t coef = (r < kh && c < kw) ? buf[r * pitch + c] : 0;
            quant_one(mode, coef, i != 0, d.q[pl], log_scale, 32, 32, qc, dqc);
            qout[i] = qc;
            buf[r * pitch + c] = dqc;
            if (qc) {
                eob = max(eob, (int)iscan[i] + 1);
                lvl += min(abs(qc), 64); // cul_level saturates at COEFF_CONTEXT_MASK = 63: 64 per term is enough
                if (i == 0) dc_sign = qc < 0 ? 1 : 2;
            }
        }
        if (eob) {
            atomicMax(&s_eob[lb], eob);
            atomicAdd(&s_cul[lb], lvl);
        }
        if (w > 32 || h > 32)
            for (int i = li; i < w * h; i += Tn) { // zero the dropped high-frequency area of 64-wide transforms
                const int r = i >> lw, c = i & (w - 1);
                if (r >= ih || c >= iw) buf[r * pitch + c] = 0;
            }
    }
    __syncthreads();
    const int bd = d.bd;
    const int range_row = bd == 8 ? 16 : bd == 10 ? 18 : 20, range_col = bd == 8 ? 16 : bd == 10 ? 16 : 18;
    if (live) {
        if (li == 0) {
            const int ob = d.out_idx ? d.out_idx[b] : b;
            d.eob[ob] = (uint16_t)s_eob[lb];
            if (d.cul_level) d.cul_level[ob] = min(63, s_cul[lb]) + (dc_sign == 1 ? 64 : dc_sign == 2 ? 128 : 0);
        }
        for (int r = li; r < t.h; r += Tn) {
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
        for (int c = li; c < t.w; c += Tn) {
            inv_1d_pass(buf + c, pitch, t.h, t.vk, 12, range_col, [=](int32_t v) { return clampv(v, col_clamp); },
                        [](int32_t v) { return round_shift64((long long)v, 4); });
        }
    }
    __syncthreads();
    if (live) { // reconstruction, four samples per step
        const T *pp = reinterpret_cast<const T *>(d.pred[pl]) + (size_t)tu.y * d.pred_stride[pl] + tu.x;
        T *rp = reinterpret_cast<T *>(d.recon[pl]) + (size_t)tu.y * d.recon_stride[pl] + tu.x;
        const int mx = (1 << bd) - 1;
        for (int i = li; i < (w * h) >> 2; i += Tn) {
            const int r = i >> (lw - 2), c = (i & ((w >> 2) - 1)) << 2;
            int pv[4], o[4];
            load4<T>(pp + (size_t)r * d.pred_stride[pl] + c, pv);
            const int32_t *br = buf + (t.ud ? h - 1 - r : r) * pitch;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int v = pv[j] + br[t.lr ? w - 1 - (c + j) : c + j];
                o[j] = v < 0 ? 0 : (v > mx ? mx : v);
            }
            store4<T>(rp + (size_t)r * d.recon_stride[pl] + c, o);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Level packing for the device -> host hand-over: the entropy coder reads a TU's levels in scan order up to eob, and
// after quantisation most of a TU is zero, so the D2H stream is "eob levels per TU in scan order" + offsets instead
// of n int32 per TU (at qindex ~170 that is > 10x fewer bytes; D2H of the raster int32 blocks bounded the end-to-end
// rate).  Two launches: exclusive scan of eob (one CTA; <= 32 K TUs per call is far above a 4K frame's count per
// transform size), then the gather.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) eob_scan_kernel(const uint16_t *eob, int n, uint32_t *offsets /*[n+1]*/, uint32_t *total,
                                                        const uint32_t *base /* device: first offset, or null = 0 */) {
    __shared__ uint32_t s_part[1024];
    const int per = (n + 1023) / 1024, t = threadIdx.x;
    uint32_t sum = 0;
    for (int i = t * per; i < min(n, (t + 1) * per); i++) sum += eob[i];
    s_part[t] = sum;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) { // Hillis-Steele inclusive scan of the 1024 partial sums
        const uint32_t v = t >= o ? s_part[t - o] : 0;
        __syncthreads();
        s_part[t] += v;
        __syncthreads();
    }
    const uint32_t b0 = base ? *base : 0u;
    uint32_t run = b0 + (t ? s_part[t - 1] : 0);
    for (int i = t * per; i < min(n, (t + 1) * per); i++) {
        offsets[i] = run;
        run += eob[i];
    }
    if (t == 1023) {
        offsets[n] = b0 + s_part[1023];
        *total = b0 + s_part[1023];
    }
}
__global__ void __launch_bounds__(256) pack_levels_kernel(const int32_t *qcoeff, const uint16_t *eob, const uint32_t *offsets,
                                                          const int16_t *scan, int n_tus, int n, int32_t *out) {
    const int b = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31; // one warp per TU
    if (b >= n_tus) return;
    const int e = eob[b];
    const int32_t *q = qcoeff + (size_t)b * n;
    int32_t *o = out + offsets[b];
    for (int i = lane; i < e; i += 32) o[i] = q[scan[i]];
}

static size_t tx_smem_bytes(int tx_size) {
    const int w = h_txw[tx_size], h = h_txh[tx_size];
    const int T = w > h ? w : h, bpc = TX_NT / T;
    return (size_t)bpc * tx_pitch(w) * h * 4;
}
static int tx_grid(int tx_size, int n) {
    const int w = h_txw[tx_size], h = h_txh[tx_size];
    const int T = w > h ? w : h, bpc = TX_NT / T;
    return (n + bpc - 1) / bpc;
}
static void tx_attrs() {
    static PerDeviceOnce once;
    once.run([] {
        SVTB_ATTR(fwd_txfm_kernel, 64 * 1024);
        SVTB_ATTR(inv_txfm_kernel, 64 * 1024);
        SVTB_ATTR((encode_tu_kernel<uint8_t, -1>), 64 * 1024);
        SVTB_ATTR((encode_tu_kernel<uint16_t, -1>), 64 * 1024);
    });
}

// ---- host side of the drop-ins --------------------------------------------------------------------------------
static void fwd_dropin(int16_t *input, int32_t *output, uint32_t stride, int tx_type, int tx_size, int repack,
                       uint64_t *energy_out, int pf_shift = 0) {
    txfm_tables_init();
    tx_attrs();
    const int w = h_txw[tx_size], h = h_txh[tx_size];
    Staging s({(size_t)w * h * 2, (size_t)w * h * 4, 8});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, input, stride, 2, w, h);
    SVTB_CUDA_FATAL(s.upload(0, 0));
    FwdArgs a;
    a.in = s.d<const int16_t>(0);
    a.in_block_stride = 0;
    a.in_stride = w;
    a.out = s.d<int32_t>(1);
    a.tx_types = nullptr;
    a.tx_type = tx_type;
    a.tx_size = tx_size;
    a.n_blocks = 1;
    a.repack64 = repack;
    a.pf_shift = pf_shift;
    a.energy = s.d<uint64_t>(2);
    SVTB_LAUNCH(fwd_txfm_kernel, 1, TX_NT, tx_smem_bytes(tx_size), s.stream(), a);
    SVTB_CUDA_FATAL(s.download(1, 2));
    memcpy(output, s.h(1), (size_t)w * h * 4);
    if (energy_out) memcpy(energy_out, s.h(2), 8);
}

static void inv_dropin(const int32_t *input, uint16_t *output_r, int32_t stride_r, uint16_t *output_w, int32_t stride_w,
                       int tx_type, int tx_size, int bd) {
    txfm_tables_init();
    tx_attrs();
    const int w = h_txw[tx_size], h = h_txh[tx_size];
    const int iw = w > 32 ? 32 : w, ih = h > 32 ? 32 : h;
    Staging s({(size_t)iw * ih * 4, (size_t)w * h * 2, (size_t)w * h * 2});
    SVTB_CUDA_FATAL(s.status());
    memcpy(s.h(0), input, (size_t)iw * ih * 4);
    s.put_rows(1, output_r, stride_r, 2, w, h);
    SVTB_CUDA_FATAL(s.upload(0, 1));
    InvArgs a;
    a.in = s.d<const int32_t>(0);
    a.pred = s.d<const uint16_t>(1);
    a.recon = s.d<uint16_t>(2);
    a.pred_block_stride = a.recon_block_stride = 0;
    a.stride_r = a.stride_w = w;
    a.tx_type = tx_type;
    a.tx_size = tx_size;
    a.n_blocks = 1;
    a.bd = bd;
    SVTB_LAUNCH(inv_txfm_kernel, 1, TX_NT, tx_smem_bytes(tx_size), s.stream(), a);
    SVTB_CUDA_FATAL(s.download(2, 2));
    s.get_rows(2, output_w, stride_w, 2, w, h);
}

static void quant_dropin(int mode, const int32_t *coeff, intptr_t n, const int16_t *zbin, const int16_t *round,
                         const int16_t *quant, const int16_t *quant_shift, int32_t *qcoeff, int32_t *dqcoeff,
                         const int16_t *dequant, uint16_t *eob, const int16_t *scan, const uint8_t *qm, const uint8_t *iqm,
                         int log_scale) {
    // coeff | scan | qm | iqm in, qcoeff | dqcoeff | eob out
    const size_t cb = (size_t)n * 4;
    Staging s({cb, (size_t)n * 2, (size_t)n, (size_t)n, cb, cb, 2});
    SVTB_CUDA_FATAL(s.status());
    memcpy(s.h(0), coeff, cb);
    memcpy(s.h(1), scan, (size_t)n * 2);
    if (qm) memcpy(s.h(2), qm, n);
    if (iqm) memcpy(s.h(3), iqm, n);
    SVTB_CUDA_FATAL(s.upload(0, 3));
    QuantArgs a;
    a.coeff = s.d<const int32_t>(0);
    a.scan = s.d<const int16_t>(1);
    a.qm = qm ? s.d(2) : nullptr;
    a.iqm = iqm ? s.d(3) : nullptr;
    a.qcoeff = s.d<int32_t>(4);
    a.dqcoeff = s.d<int32_t>(5);
    a.eob = s.d<uint16_t>(6);
    for (int i = 0; i < 2; i++) {
        a.q.zbin[i] = zbin ? zbin[i] : 0;
        a.q.round[i] = round[i];
        a.q.quant[i] = quant[i];
        a.q.quant_shift[i] = quant_shift ? quant_shift[i] : 0;
        a.q.dequant[i] = dequant[i];
    }
    a.n = (int)n;
    a.log_scale = log_scale;
    a.mode = mode;
    SVTB_LAUNCH(quant_kernel, 1, 256, 0, s.stream(), a);
    SVTB_CUDA_FATAL(s.download(4, 6));
    memcpy(qcoeff, s.h(4), cb);
    memcpy(dqcoeff, s.h(5), cb);
    memcpy(eob, s.h(6), 2);
}

} // namespace

extern "C" {

// --- forward transforms: one exported symbol per RTCD pointer (aom_dsp_rtcd.h:105-216) ---
#define FWD_DROPIN(W, H, TXS)                                                                                     \
    void svt_av1_fwd_txfm2d_##W##x##H##_cuda(int16_t *input, int32_t *output, uint32_t input_stride, uint8_t tx_type, \
                                             uint8_t bit_depth) {                                                 \
        (void)bit_depth;                                                                                          \
        fwd_dropin(input, output, input_stride, tx_type, TXS, 0, nullptr);                                        \
    }                                                                                                             \
    void svt_av1_fwd_txfm2d_##W##x##H##_N2_cuda(int16_t *input, int32_t *output, uint32_t input_stride,           \
                                                uint8_t tx_type, uint8_t bit_depth) {                             \
        (void)bit_depth;                                                                                          \
        fwd_dropin(input, output, input_stride, tx_type, TXS, 0, nullptr, 1);                                     \
    }                                                                                                             \
    void svt_av1_fwd_txfm2d_##W##x##H##_N4_cuda(int16_t *input, int32_t *output, uint32_t input_stride,           \
                                                uint8_t tx_type, uint8_t bit_depth) {                             \
        (void)bit_depth;                                                                                          \
        fwd_dropin(input, output, input_stride, tx_type, TXS, 0, nullptr, 2);                                     \
    }
FWD_DROPIN(4, 4, 0)
FWD_DROPIN(8, 8, 1)
FWD_DROPIN(16, 16, 2)
FWD_DROPIN(32, 32, 3)
FWD_DROPIN(64, 64, 4)
FWD_DROPIN(4, 8, 5)
FWD_DROPIN(8, 4, 6)
FWD_DROPIN(8, 16, 7)
FWD_DROPIN(16, 8, 8)
FWD_DROPIN(16, 32, 9)
FWD_DROPIN(32, 16, 10)
FWD_DROPIN(32, 64, 11)
FWD_DROPIN(64, 32, 12)
FWD_DROPIN(4, 16, 13)
FWD_DROPIN(16, 4, 14)
FWD_DROPIN(8, 32, 15)
FWD_DROPIN(32, 8, 16)
FWD_DROPIN(16, 64, 17)
FWD_DROPIN(64, 16, 18)

// --- inverse transforms (common_dsp_rtcd.h:105-156); rectangular ones carry tx_size (+eob) like the reference ---
#define INV_SQ(W, TXS)                                                                                            \
    void svt_av1_inv_txfm2d_add_##W##x##W##_cuda(const int32_t *input, uint16_t *output_r, int32_t stride_r,      \
                                                 uint16_t *output_w, int32_t stride_w, uint8_t tx_type, int32_t bd) { \
        inv_dropin(input, output_r, stride_r, output_w, stride_w, tx_type, TXS, bd);                              \
    }
#define INV_RECT(W, H, TXS)                                                                                       \
    void svt_av1_inv_txfm2d_add_##W##x##H##_cuda(const int32_t *input, uint16_t *output_r, int32_t stride_r,      \
                                                 uint16_t *output_w, int32_t stride_w, uint8_t tx_type,           \
                                                 uint8_t tx_size, int32_t eob, int32_t bd) {                      \
        (void)tx_size;                                                                                            \
        (void)eob;                                                                                                \
        inv_dropin(input, output_r, stride_r, output_w, stride_w, tx_type, TXS, bd);                              \
    }
#define INV_RECT_NOEOB(W, H, TXS)                                                                                 \
    void svt_av1_inv_txfm2d_add_##W##x##H##_cuda(const int32_t *input, uint16_t *output_r, int32_t stride_r,      \
                                                 uint16_t *output_w, int32_t stride_w, uint8_t tx_type,           \
                                                 uint8_t tx_size, int32_t bd) {                                   \
        (void)tx_size;                                                                                            \
        inv_dropin(input, output_r, stride_r, output_w, stride_w, tx_type, TXS, bd);                              \
    }
INV_SQ(4, 0)
INV_SQ(8, 1)
INV_SQ(16, 2)
INV_SQ(32, 3)
INV_SQ(64, 4)
INV_RECT_NOEOB(4, 8, 5)
INV_RECT_NOEOB(8, 4, 6)
INV_RECT(8, 16, 7)
INV_RECT(16, 8, 8)
INV_RECT(16, 32, 9)
INV_RECT(32, 16, 10)
INV_RECT(32, 64, 11)
INV_RECT(64, 32, 12)
INV_RECT_NOEOB(4, 16, 13)
INV_RECT_NOEOB(16, 4, 14)
INV_RECT(8, 32, 15)
INV_RECT(32, 8, 16)
INV_RECT(16, 64, 17)
INV_RECT(64, 16, 18)

// svt_handle_transform64x64 & co. (aom_dsp_rtcd.h:222-245): operate in place on the w x h coefficient array
#define HANDLE64(W, H, TXS)                                                                    \
    uint64_t svt_handle_transform##W##x##H##_cuda(int32_t *output) {                           \
        /* identity "transform" of the already transformed block is not available: run the */ \
        /* zero-out / re-pack on the device through a plain copy kernel                      */ \
        return svt_b200_handle_transform64(output, TXS);                                       \
    }
uint64_t svt_b200_handle_transform64(int32_t *output, int tx_size);
HANDLE64(64, 64, 4)
HANDLE64(32, 64, 11)
HANDLE64(64, 32, 12)
HANDLE64(16, 64, 17)
HANDLE64(64, 16, 18)

void svt_aom_quantize_b_cuda(const int32_t *coeff_ptr, intptr_t n_coeffs, const int16_t *zbin_ptr, const int16_t *round_ptr,
                             const int16_t *quant_ptr, const int16_t *quant_shift_ptr, int32_t *qcoeff_ptr,
                             int32_t *dqcoeff_ptr, const int16_t *dequant_ptr, uint16_t *eob_ptr, const int16_t *scan,
                             const int16_t *iscan, const uint8_t *qm_ptr, const uint8_t *iqm_ptr, const int32_t log_scale) {
    (void)iscan;
    quant_dropin(0, coeff_ptr, n_coeffs, zbin_ptr, round_ptr, quant_ptr, quant_shift_ptr, qcoeff_ptr, dqcoeff_ptr, dequant_ptr,
                 eob_ptr, scan, qm_ptr, iqm_ptr, log_scale);
}
void svt_aom_highbd_quantize_b_cuda(const int32_t *coeff_ptr, intptr_t n_coeffs, const int16_t *zbin_ptr,
                                    const int16_t *round_ptr, const int16_t *quant_ptr, const int16_t *quant_shift_ptr,
                                    int32_t *qcoeff_ptr, int32_t *dqcoeff_ptr, const int16_t *dequant_ptr, uint16_t *eob_ptr,
                                    const int16_t *scan, const int16_t *iscan, const uint8_t *qm_ptr, const uint8_t *iqm_ptr,
                                    const int32_t log_scale) {
    (void)iscan;
    quant_dropin(1, coeff_ptr, n_coeffs, zbin_ptr, round_ptr, quant_ptr, quant_shift_ptr, qcoeff_ptr, dqcoeff_ptr, dequant_ptr,
                 eob_ptr, scan, qm_ptr, iqm_ptr, log_scale);
}
#define QFP(NAME, LS)                                                                                                   \
    void NAME(const int32_t *coeff_ptr, intptr_t n_coeffs, const int16_t *zbin_ptr, const int16_t *round_ptr,           \
              const int16_t *quant_ptr, const int16_t *quant_shift_ptr, int32_t *qcoeff_ptr, int32_t *dqcoeff_ptr,      \
              const int16_t *dequant_ptr, uint16_t *eob_ptr, const int16_t *scan, const int16_t *iscan) {               \
        (void)iscan;                                                                                                    \
        quant_dropin(2, coeff_ptr, n_coeffs, zbin_ptr, round_ptr, quant_ptr, quant_shift_ptr, qcoeff_ptr, dqcoeff_ptr,  \
                     dequant_ptr, eob_ptr, scan, nullptr, nullptr, LS);                                                 \
    }
QFP(svt_av1_quantize_fp_cuda, 0)
QFP(svt_av1_quantize_fp_32x32_cuda, 1)
QFP(svt_av1_quantize_fp_64x64_cuda, 2)
void svt_av1_highbd_quantize_fp_cuda(const int32_t *coeff_ptr, intptr_t n_coeffs, const int16_t *zbin_ptr,
                                     const int16_t *round_ptr, const int16_t *quant_ptr, const int16_t *quant_shift_ptr,
                                     int32_t *qcoeff_ptr, int32_t *dqcoeff_ptr, const int16_t *dequant_ptr, uint16_t *eob_ptr,
                                     const int16_t *scan, const int16_t *iscan, int16_t log_scale) {
    (void)iscan;
    quant_dropin(3, coeff_ptr, n_coeffs, zbin_ptr, round_ptr, quant_ptr, quant_shift_ptr, qcoeff_ptr, dqcoeff_ptr, dequant_ptr,
                 eob_ptr, scan, nullptr, nullptr, log_scale);
}

static void residual_dropin(const void *src, uint32_t ss, const void *pred, uint32_t ps, int16_t *res, uint32_t rs, uint32_t w,
                            uint32_t h, int hbd) {
    const size_t e = hbd ? 2 : 1, pb = (size_t)w * h * e;
    Staging s({pb, pb, (size_t)w * h * 2});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, src, ss, e, w, h);
    s.put_rows(1, pred, ps, e, w, h);
    SVTB_CUDA_FATAL(s.upload(0, 1));
    if (hbd)
        SVTB_LAUNCH(residual_kernel<uint16_t>, 4, 256, 0, s.stream(), s.d<const uint16_t>(0), (int)w, s.d<const uint16_t>(1), (int)w,
                    s.d<int16_t>(2), (int)w, (int)w, (int)h);
    else
        SVTB_LAUNCH(residual_kernel<uint8_t>, 4, 256, 0, s.stream(), s.d<const uint8_t>(0), (int)w, s.d<const uint8_t>(1), (int)w,
                    s.d<int16_t>(2), (int)w, (int)w, (int)h);
    SVTB_CUDA_FATAL(s.download(2, 2));
    s.get_rows(2, res, rs, 2, w, h);
}
void svt_residual_kernel8bit_cuda(uint8_t *input, uint32_t input_stride, uint8_t *pred, uint32_t pred_stride, int16_t *residual,
                                  uint32_t residual_stride, uint32_t area_width, uint32_t area_height) {
    residual_dropin(input, input_stride, pred, pred_stride, residual, residual_stride, area_width, area_height, 0);
}
void svt_residual_kernel16bit_cuda(uint16_t *input, uint32_t input_stride, uint16_t *pred, uint32_t pred_stride,
                                   int16_t *residual, uint32_t residual_stride, uint32_t area_width, uint32_t area_height) {
    residual_dropin(input, input_stride, pred, pred_stride, residual, residual_stride, area_width, area_height, 1);
}
}

// ---- zero-out / re-pack of 64-wide coefficient blocks on the device ----
namespace {
__global__ void handle64_kernel(int32_t *io, int w, int h, unsigned long long *energy) {
    extern __shared__ int32_t sm[];
    const int kw = min(w, 32), kh = min(h, 32);
    unsigned long long e = 0;
    for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
        const int r = i / w, c = i - r * w;
        const int32_t v = io[i];
        sm[i] = v;
        if (r >= kh || c >= kw) e += (unsigned long long)((long long)v * (long long)v);
    }
    __shared__ unsigned long long s_e;
    if (threadIdx.x == 0) s_e = 0;
    __syncthreads();
    for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&s_e, e);
    __syncthreads();
    for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
        const int r = i / w, c = i - r * w;
        io[i] = (kw != w && i < kw * kh) ? sm[(i / kw) * w + (i % kw)] : ((r >= kh || c >= kw) ? 0 : sm[i]);
    }
    if (threadIdx.x == 0) *energy = s_e;
}
} // namespace

extern "C" uint64_t svt_b200_handle_transform64(int32_t *output, int tx_size) {
    const int w = h_txw[tx_size], h = h_txh[tx_size];
    const size_t nb = (size_t)w * h * 4;
    Staging s({nb, 8});
    SVTB_CUDA_FATAL(s.status());
    memcpy(s.h(0), output, nb);
    SVTB_CUDA_FATAL(s.upload(0, 0));
    SVTB_LAUNCH(handle64_kernel, 1, 256, nb, s.stream(), s.d<int32_t>(0), w, h, s.d<unsigned long long>(1));
    SVTB_CUDA_FATAL(s.download(0, 1));
    memcpy(output, s.h(0), nb);
    return *s.h<uint64_t>(1);
}

// ---------------------------------------------------------------------------------------------------------------
// batched / picture-level entries
// ---------------------------------------------------------------------------------------------------------------
extern "C" {

// svt_av1_inv_txfm_add_c (EbInvTransforms.c:3302-3323): the low-bit-depth wrapper — widen the prediction to 16 bit, run
// the (high-bit-depth) inverse transform at bd = 8, narrow the result.  TxfmParam (EbDefinitions.h:779-791) is read
// through a layout view: packed 1-byte enums tx_type / tx_size, then int32 lossless, bd, is_hbd, tx_set_type, eob.
struct TxfmParamView {
    uint8_t tx_type, tx_size;
    int32_t lossless, bd, is_hbd;
    uint8_t tx_set_type;
    int32_t eob;
};
void svt_av1_inv_txfm_add_cuda(const int32_t *dqcoeff, uint8_t *dst_r, int32_t stride_r, uint8_t *dst_w, int32_t stride_w,
                               const void *txfm_param) {
    const TxfmParamView *tp = (const TxfmParamView *)txfm_param;
    const int tx_size = tp->tx_size, tx_type = tp->tx_type;
    if (tx_size > 18 || tx_type > 15 || tp->lossless) {
        fprintf(stderr, "svt_av1_inv_txfm_add_cuda: tx_size %d / tx_type %d / lossless %d is not supported\n", tx_size, tx_type, tp->lossless);
        abort();
    }
    const int w = h_txw[tx_size], h = h_txh[tx_size];
    uint16_t tmp[64 * 64];
    for (int r = 0; r < h; r++)
        for (int c = 0; c < w; c++) tmp[r * 64 + c] = dst_r[(size_t)r * stride_r + c];
    inv_dropin(dqcoeff, tmp, 64, tmp, 64, tx_type, tx_size, tp->bd);
    for (int r = 0; r < h; r++)
        for (int c = 0; c < w; c++) dst_w[(size_t)r * stride_w + c] = (uint8_t)tmp[r * 64 + c];
}

int svt_b200_get_scan(int tx_size, int tx_type, int16_t *scan_out) {
    // get_scan (Common/Codec/EbCoefficients.c / av1_scan_orders): 64-wide sizes scan as their 32-wide packing;
    // 2-D types: zig-zag (diagonals alternate for squares, fixed direction for rectangles); V_* (row-identity):
    // row scan; H_*: column scan; IDTX: default.
    if (tx_size < 0 || tx_size > 18 || tx_type < 0 || tx_type > 15 || !scan_out) return SVT_B200_ERR_ARG;
    int w = h_txw[tx_size], h = h_txh[tx_size];
    if (w > 32) w = 32;
    if (h > 32) h = 32;
    static const uint8_t vtx[16] = {0, 1, 0, 1, 2, 0, 2, 1, 2, 3, 0, 3, 1, 3, 2, 3};
    static const uint8_t htx[16] = {0, 0, 1, 1, 0, 2, 2, 2, 1, 3, 3, 0, 3, 1, 3, 2};
    const int vk = vtx[tx_type], hk = htx[tx_type];
    int n = 0;
    if (vk != 3 && hk == 3) { // V_DCT / V_ADST / V_FLIPADST: mrow_scan (raster)
        for (int i = 0; i < w * h; i++) scan_out[n++] = (int16_t)i;
    } else if (vk == 3 && hk != 3) { // H_*: mcol_scan
        for (int c = 0; c < w; c++)
            for (int r = 0; r < h; r++) scan_out[n++] = (int16_t)(r * w + c);
    } else {
        for (int d = 0; d < w + h - 1; d++) {
            // direction of travel along anti-diagonal d
            bool down_left; // true: start at the top-right end and walk towards bottom-left
            if (w == h) down_left = (d & 1) != 0;
            else down_left = h > w;
            if (down_left) {
                for (int r = 0; r < h; r++) {
                    const int c = d - r;
                    if (c >= 0 && c < w) scan_out[n++] = (int16_t)(r * w + c);
                }
            } else {
                for (int r = h - 1; r >= 0; r--) {
                    const int c = d - r;
                    if (c >= 0 && c < w) scan_out[n++] = (int16_t)(r * w + c);
                }
            }
        }
    }
    return n;
}


} // extern "C"
namespace {
const int16_t *scan_tables(int tx_size);
}
extern "C" {
// see include/svt_av1_b200.h
int svt_b200_pack_levels(int32_t tx_size, int32_t tx_class, const int32_t *qcoeff, const uint16_t *eob, int32_t n_tus, int32_t *packed,
                         uint32_t *offsets, uint32_t *total, void *stream) {
    return svt_b200_pack_levels_at(tx_size, tx_class, qcoeff, eob, n_tus, packed, offsets, total, nullptr, stream);
}

int svt_b200_pack_levels_at(int32_t tx_size, int32_t tx_class, const int32_t *qcoeff, const uint16_t *eob, int32_t n_tus, int32_t *packed,
                            uint32_t *offsets, uint32_t *total, const uint32_t *base, void *stream) {
    if (tx_size < 0 || tx_size > 18 || tx_class < 0 || tx_class > 2 || !qcoeff || !eob || !packed || !offsets || !total || n_tus < 0 ||
        n_tus > (1 << 20)) {
        set_error("svt_b200_pack_levels: bad argument");
        return SVT_B200_ERR_ARG;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (n_tus == 0) {
        if (base) {
            SVTB_CUDA_TRY(cudaMemcpyAsync(total, base, 4, cudaMemcpyDeviceToDevice, st));
            SVTB_CUDA_TRY(cudaMemcpyAsync(offsets, base, 4, cudaMemcpyDeviceToDevice, st));
        } else {
            SVTB_CUDA_TRY(cudaMemsetAsync(total, 0, 4, st));
            SVTB_CUDA_TRY(cudaMemsetAsync(offsets, 0, 4, st));
        }
        return SVT_B200_OK;
    }
    const int16_t *tab = scan_tables(tx_size);
    if (!tab) return SVT_B200_ERR_CUDA;
    const int n = (h_txw[tx_size] > 32 ? 32 : h_txw[tx_size]) * (h_txh[tx_size] > 32 ? 32 : h_txh[tx_size]);
    SVTB_LAUNCH(eob_scan_kernel, 1, 1024, 0, st, eob, n_tus, offsets, total, base);
    SVTB_LAUNCH(pack_levels_kernel, (n_tus + 7) / 8, 256, 0, st, qcoeff, eob, offsets, tab + 3072 + tx_class * 1024, n_tus, n, packed);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

} // extern "C"
namespace {
// device-resident inverse scan tables: [device][tx_size] -> 3 x 1024 int16
const int16_t *scan_tables(int tx_size) { // [3][1024] inverse scans, then [3][1024] forward scans
    static std::mutex mu;
    static int16_t *tabs[64][19] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev >= 64) return nullptr;
    std::lock_guard<std::mutex> lk(mu);
    if (tabs[dev][tx_size]) return tabs[dev][tx_size];
    static int16_t hs[1024], hi[6][1024];
    const int types[3] = {0, 10, 11}; // DCT_DCT (default scan), V_DCT (mrow), H_DCT (mcol)
    const int n = (h_txw[tx_size] > 32 ? 32 : h_txw[tx_size]) * (h_txh[tx_size] > 32 ? 32 : h_txh[tx_size]);
    for (int k = 0; k < 3; k++) {
        svt_b200_get_scan(tx_size, types[k], hs);
        for (int i = 0; i < 1024; i++) hi[k][i] = hi[3 + k][i] = 0;
        for (int i = 0; i < n; i++) {
            hi[k][hs[i]] = (int16_t)i;
            hi[3 + k][i] = hs[i];
        }
    }
    int16_t *dp = nullptr;
    if (cudaMalloc(&dp, sizeof(hi)) != cudaSuccess) return nullptr;
    if (cudaMemcpy(dp, hi, sizeof(hi), cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
    tabs[dev][tx_size] = dp;
    return dp;
}
} // namespace
extern "C" {

int svt_b200_encode_tus(const SvtB200EncodeParams *p, const SvtB200Frame *src, const SvtB200Frame *pred,
                        const SvtB200Frame *recon, const SvtB200Tu *tus, int32_t n_tus, int32_t *qcoeff, uint16_t *eob,
                        void *scratch, void *stream) {
    (void)scratch; // kept for ABI stability: the scan tables are resident per device since round 1
    return svt_b200_encode_tus_cul(p, src, pred, recon, tus, n_tus, qcoeff, eob, nullptr, stream);
}

static int encode_launch(const SvtB200EncodeParams *p, int pf_shape, const long long *qoff, const int32_t *out_idx,
                         const SvtB200Frame *src, const SvtB200Frame *pred, const SvtB200Frame *recon, const SvtB200Tu *tus,
                         int32_t n_tus, int32_t *qcoeff, uint16_t *eob, int32_t *cul_level, void *stream);

int svt_b200_encode_tus_cul(const SvtB200EncodeParams *p, const SvtB200Frame *src, const SvtB200Frame *pred,
                            const SvtB200Frame *recon, const SvtB200Tu *tus, int32_t n_tus, int32_t *qcoeff, uint16_t *eob,
                            int32_t *cul_level, void *stream) {
    return encode_launch(p, 0, nullptr, nullptr, src, pred, recon, tus, n_tus, qcoeff, eob, cul_level, stream);
}

static int encode_launch(const SvtB200EncodeParams *p, int pf_shape, const long long *qoff, const int32_t *out_idx,
                         const SvtB200Frame *src, const SvtB200Frame *pred, const SvtB200Frame *recon, const SvtB200Tu *tus,
                         int32_t n_tus, int32_t *qcoeff, uint16_t *eob, int32_t *cul_level, void *stream) {
    if (!p || !src || !pred || !recon || !tus || !qcoeff || !eob || n_tus < 0 || p->tx_size < 0 || p->tx_size > 18 ||
        src->bit_depth != pred->bit_depth || src->bit_depth != recon->bit_depth) {
        set_error("svt_b200_encode_tus: bad argument");
        return SVT_B200_ERR_ARG;
    }
    if (n_tus == 0) return SVT_B200_OK;
    txfm_tables_init();
    tx_attrs();
    static_assert(sizeof(SvtB200Tu) == sizeof(TuDev), "descriptor layout");
    EncodeDev d;
    const SvtB200Frame *fr[3] = {src, pred, recon};
    for (int i = 0; i < 3; i++) {
        d.src[i] = i == 0 ? fr[0]->y : i == 1 ? fr[0]->cb : fr[0]->cr;
        d.pred[i] = i == 0 ? fr[1]->y : i == 1 ? fr[1]->cb : fr[1]->cr;
        d.recon[i] = i == 0 ? fr[2]->y : i == 1 ? fr[2]->cb : fr[2]->cr;
        d.src_stride[i] = i == 0 ? fr[0]->stride_y : fr[0]->stride_c;
        d.pred_stride[i] = i == 0 ? fr[1]->stride_y : fr[1]->stride_c;
        d.recon_stride[i] = i == 0 ? fr[2]->stride_y : fr[2]->stride_c;
        for (int k = 0; k < 2; k++) {
            d.q[i].zbin[k] = p->q[i].zbin[k];
            d.q[i].round[k] = p->use_fp ? p->q[i].round_fp[k] : p->q[i].round[k];
            d.q[i].quant[k] = p->use_fp ? p->q[i].quant_fp[k] : p->q[i].quant[k];
            d.q[i].quant_shift[k] = p->q[i].quant_shift[k];
            d.q[i].dequant[k] = p->q[i].dequant[k];
        }
    }
    d.bd = src->bit_depth;
    d.hbd = src->bit_depth > 8;
    d.tus = reinterpret_cast<const TuDev *>(tus);
    d.n_tus = n_tus;
    d.tx_size = p->tx_size;
    d.quant_mode = p->use_fp ? 2 : 0;
    d.qcoeff = qcoeff;
    d.eob = eob;
    d.cul_level = cul_level;
    d.pf_shape = pf_shape;
    d.qoff = qoff;
    d.out_idx = out_idx;
    // inverse scan tables of this size: built once per (device, tx_size) and kept resident (`scratch` is unused since
    // then; the parameter stays for ABI stability)
    const int16_t *tab = scan_tables(p->tx_size);
    if (!tab) return SVT_B200_ERR_CUDA;
    for (int i = 0; i < 3; i++) d.iscan[i] = tab + i * 1024;
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = tx_grid(p->tx_size, n_tus);
    const size_t smem = tx_smem_bytes(p->tx_size);
#define SVTB_ENC(TSV)                                                                          \
    do {                                                                                       \
        if (d.hbd)                                                                             \
            SVTB_LAUNCH((encode_tu_kernel<uint16_t, TSV>), grid, TX_NT, smem, st, d);          \
        else                                                                                   \
            SVTB_LAUNCH((encode_tu_kernel<uint8_t, TSV>), grid, TX_NT, smem, st, d);           \
    } while (0)
    switch (p->tx_size) {
    case 0: SVTB_ENC(0); break;
    case 1: SVTB_ENC(1); break;
    case 2: SVTB_ENC(2); break;
    case 3: SVTB_ENC(3); break;
    default: SVTB_ENC(-1); break;
    }
#undef SVTB_ENC
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

// av1_estimate_transform's dispatcher generality for the fused path (VERDICT r1 a11): a HOST list of transform units of MIXED
// transform sizes, partial-frequency shapes and quantiser sets (per-block qindex / segment delta-q: av1_quantize_inv_quantize
// picks the table by q_index, EbFullLoop.c:1400-1470).  The list is bucketed by (tx_size, pf_shape, qset) on the host, every
// bucket is one launch of the size-specialised kernel, and the outputs land in INPUT order: eob[i] / cul_level[i], and the
// levels of unit i at qcoeff + qcoeff_offsets[i] (min(w,32) * min(h,32) entries; offsets returned to the caller).
int svt_b200_encode_tus_ex(const SvtB200EncodeParamsEx *p, const SvtB200Frame *src, const SvtB200Frame *pred,
                           const SvtB200Frame *recon, const SvtB200TuEx *tus, int32_t n_tus, int32_t *qcoeff,
                           int64_t *qcoeff_offsets, uint16_t *eob, int32_t *cul_level, void *scratch, size_t scratch_bytes,
                           void *stream) {
    if (!p || !tus || !qcoeff || !qcoeff_offsets || !eob || n_tus < 0 || !p->qsets || p->n_qsets < 1 || !scratch) {
        set_error("svt_b200_encode_tus_ex: bad argument");
        return SVT_B200_ERR_ARG;
    }
    const size_t per_tu = sizeof(TuDev) + sizeof(long long) + sizeof(int32_t);
    if (scratch_bytes < (size_t)n_tus * per_tu + 256) {
        set_error("svt_b200_encode_tus_ex: scratch too small (%zu bytes per unit + 256)", per_tu);
        return SVT_B200_ERR_ARG;
    }
    // offsets in input order
    long long off = 0;
    for (int i = 0; i < n_tus; i++) {
        const SvtB200TuEx &t = tus[i];
        if (t.tx_size > 18 || t.pf_shape > 3 || t.plane > 2 || t.qset >= p->n_qsets) {
            set_error("svt_b200_encode_tus_ex: unit %d out of range", i);
            return SVT_B200_ERR_ARG;
        }
        qcoeff_offsets[i] = off;
        off += (long long)std::min<int>(h_txw[t.tx_size], 32) * std::min<int>(h_txh[t.tx_size], 32);
    }
    qcoeff_offsets[n_tus] = off;
    if (n_tus == 0) return SVT_B200_OK;
    // bucket: stable sort of the indices by key
    std::vector<int32_t> order(n_tus);
    for (int i = 0; i < n_tus; i++) order[i] = i;
    auto key = [&](int i) { return ((uint32_t)tus[i].tx_size << 24) | ((uint32_t)tus[i].pf_shape << 16) | tus[i].qset; };
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return key(a) < key(b); });
    // pinned staging of the calling thread: TuDev[n], then qoff[n] | out_idx[n] as one region, so that the upload
    // (at most n * per_tu + 255 bytes) fits the caller's scratch
    Staging s({(size_t)n_tus * sizeof(TuDev), (size_t)n_tus * (sizeof(long long) + sizeof(int32_t))});
    SVTB_CUDA_TRY(s.status());
    TuDev *h_tu = s.h<TuDev>(0);
    long long *h_qoff = s.h<long long>(1);
    int32_t *h_idx = reinterpret_cast<int32_t *>(h_qoff + n_tus);
    for (int k = 0; k < n_tus; k++) {
        const SvtB200TuEx &t = tus[order[k]];
        h_tu[k] = TuDev{t.x, t.y, t.plane, t.tx_type};
        h_qoff[k] = qcoeff_offsets[order[k]];
        h_idx[k] = order[k];
    }
    uint8_t *dsc = reinterpret_cast<uint8_t *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    SVTB_CUDA_TRY(cudaMemcpyAsync(dsc, h_tu, s.span(0, 1), cudaMemcpyHostToDevice, st));
    const TuDev *d_tu = reinterpret_cast<const TuDev *>(dsc);
    const long long *d_qoff = reinterpret_cast<const long long *>(dsc + s.off(1));
    const int32_t *d_idx = reinterpret_cast<const int32_t *>(d_qoff + n_tus);
    int rc = SVT_B200_OK;
    for (int k0 = 0; k0 < n_tus && rc == SVT_B200_OK;) {
        int k1 = k0;
        while (k1 < n_tus && key(order[k1]) == key(order[k0])) k1++;
        const SvtB200TuEx &t = tus[order[k0]];
        SvtB200EncodeParams bp;
        bp.tx_size = t.tx_size;
        bp.use_fp = p->use_fp;
        for (int pl = 0; pl < 3; pl++) bp.q[pl] = p->qsets[t.qset][pl];
        rc = encode_launch(&bp, t.pf_shape, d_qoff + k0, d_idx + k0, src, pred, recon, reinterpret_cast<const SvtB200Tu *>(d_tu + k0),
                           k1 - k0, qcoeff, eob, cul_level, stream);
        k0 = k1;
    }
    // the pinned staging of this thread is reused by its next call
    SVTB_CUDA_TRY(cudaStreamSynchronize(st));
    return rc;
}
} // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Open-loop intra search of the TPL path, the flavour of presets >= 5 (tpl_opt_flag: DC_PRED only):
// open_loop_intra_search_mb (EbMotionEstimation.c:3043-3155) for every 16x16 macroblock of a picture in one launch.
// 16 threads per macroblock (one row / one column of the 16x16 DCT each), 8 macroblocks per CTA.  Neighbours come from
// the source picture (update_neighbor_samples_array_open_loop_mb, EbEncIntraPrediction.c:1201: above = at most
// min(32, width - x) samples of the row over the block, the rest 127; left = at most min(32, height - y) samples, the rest
// 129), the predictor is dc_pred[x > 0][y > 0][TX_16X16], the cost svt_aom_satd of svt_av1_fwd_txfm2d_16x16(DCT_DCT) of the
// residual.  Samples right of / below the picture are read as the replicated edge (the reference reads its padded input
// picture there).
// ---------------------------------------------------------------------------------------------------------------
namespace {
struct OisDev {
    const uint8_t *y;
    int stride, w, h, mbw, n_mb;
    long long *cost;
};
__global__ void __launch_bounds__(TX_NT) ois_dc_kernel(const OisDev d) {
    extern __shared__ int32_t sm[];
    constexpr int W = 16, T = 16, BPC = TX_NT / T;
    const int pitch = tx_pitch(W);
    const int lb = threadIdx.x / T, li = threadIdx.x % T;
    const int mb = blockIdx.x * BPC + lb;
    const bool live = mb < d.n_mb;
    int32_t *buf = sm + lb * (pitch * W);
    const TxCfg t = make_txcfg(2 /* TX_16X16 */, 0 /* DCT_DCT */);
    const int mx = live ? mb % d.mbw : 0, my = live ? mb / d.mbw : 0, x = mx * 16, y = my * 16;
    // DC: lane li holds above[li] and left[li]; the 16 lanes of a macroblock are one half-warp
    int a = 0, l = 0;
    if (y > 0) a = li < min(32, d.w - x) ? d.y[(size_t)(y - 1) * d.stride + x + li] : 127;
    if (x > 0) l = li < min(32, d.h - y) ? d.y[(size_t)(y + li) * d.stride + x - 1] : 129;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        l += __shfl_xor_sync(0xffffffffu, l, o);
    }
    const int dc = (x > 0 && y > 0) ? (a + l + 16) >> 5 : y > 0 ? (a + 8) >> 4 : x > 0 ? (l + 8) >> 4 : 128;
    if (live) {
        const uint8_t *row = d.y + (size_t)min(y + li, d.h - 1) * d.stride;
#pragma unroll
        for (int c = 0; c < W; c++) buf[li * pitch + c] = (int)row[min(x + c, d.w - 1)] - dc;
    }
    __syncthreads();
    if (live) {
        const int fs0 = t.fs0, fs1 = t.fs1;
        fwd_1d_pass(buf + li, pitch, t.h, t.vk, t.cbc, [=](int32_t v) { return (int32_t)((uint32_t)v << fs0); },
                    [=](int32_t v) { return fs1 ? round_shift64((long long)v, -fs1) : v; });
    }
    __syncthreads();
    long long s = 0;
    if (live) {
        const int fs2 = t.fs2;
        fwd_1d_pass(buf + li * pitch, 1, t.w, t.hk, t.cbr, [](int32_t v) { return v; },
                    [=](int32_t v) { return fs2 ? round_shift64((long long)v, -fs2) : v; });
#pragma unroll
        for (int c = 0; c < W; c++) s += abs(buf[li * pitch + c]);
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (live && li == 0) d.cost[mb] = s;
}
} // namespace

extern "C" {

// pic: 8-bit picture (the luma plane is read); cost: DEVICE int64 [mb rows][mb cols], mb cols = (width + 15) / 16 =
// the reference's mb_stride; every entry is OisMbResults::intra_cost of that macroblock, its intra_mode is DC_PRED.
int svt_b200_ois_dc_picture(const SvtB200Frame *pic, int64_t *cost, void *stream) {
    if (!pic || !pic->y || pic->bit_depth != 8 || !cost || pic->width <= 0 || pic->height <= 0) {
        set_error("svt_b200_ois_dc_picture: bad argument (8-bit pictures)");
        return SVT_B200_ERR_ARG;
    }
    txfm_tables_init();
    OisDev d;
    d.y = (const uint8_t *)pic->y, d.stride = pic->stride_y, d.w = pic->width, d.h = pic->height;
    d.mbw = (pic->width + 15) / 16;
    d.n_mb = d.mbw * ((pic->height + 15) / 16);
    d.cost = (long long *)cost;
    const int bpc = TX_NT / 16;
    SVTB_LAUNCH(ois_dc_kernel, (d.n_mb + bpc - 1) / bpc, TX_NT, (size_t)bpc * tx_pitch(16) * 16 * sizeof(int32_t), (cudaStream_t)stream, d);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

// the same with a HOST luma plane in and a host cost array out (the encoder binding: integration/svt_cuda_backend.c)
int svt_b200_ois_dc_picture_host(const uint8_t *y, int32_t stride, int32_t width, int32_t height, int64_t *cost) {
    if (!y || !cost || width <= 0 || height <= 0) {
        set_error("svt_b200_ois_dc_picture_host: bad argument");
        return SVT_B200_ERR_ARG;
    }
    const int n_mb = ((width + 15) / 16) * ((height + 15) / 16);
    Staging s({(size_t)width * height, (size_t)n_mb * 8});
    SVTB_CUDA_TRY(s.status());
    s.put_rows(0, y, stride, 1, width, height);
    SVTB_CUDA_TRY(s.upload(0, 0));
    SvtB200Frame f = {s.d(0), nullptr, nullptr, width, 0, width, height, 8};
    const int rc = svt_b200_ois_dc_picture(&f, s.d<int64_t>(1), s.stream());
    if (rc) return rc;
    SVTB_CUDA_TRY(s.download(1, 1));
    memcpy(cost, s.h(1), (size_t)n_mb * 8);
    return SVT_B200_OK;
}
}
