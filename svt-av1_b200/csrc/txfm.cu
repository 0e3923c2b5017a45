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
//   open_loop_intra_search_mb of the TPL path (DC_PRED, 16x16 DCT cost) for a whole picture
//
// Design: a transform block lives in shared memory for its whole life (w x h int32, odd pitch); one thread
// owns a column in the column pass and a row in the row pass, so a 64x64 block is 64 lanes and small blocks
// are packed several per CTA.  The 2-D transforms are written once, fwd_txfm2d and inv_txfm2d (txfm.cuh), and every
// kernel runs them: the forward and inverse drop-ins (one block), the fused kernel (specialised per square size
// through make_txcfg<TS>) and the open-loop intra search (16x16 DCT).  In the fused kernel HBM sees only src + pred in
// and qcoeff + recon out (7 B/px for 8-bit, SURVEY §8d) — the int32 coefficient planes of the reference's five
// separate calls never leave the SM.
//
// Layout: tables and kernels, then the host helpers, then every exported entry in one extern "C" block.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "txfm.cuh"

#include <cmath>
#include <mutex>

namespace svtb200 {

// Width and height per TxSize (TX_4X4 .. TX_64X16) and the 1-D kinds of the columns (vtx) and rows (htx) per TxType
// (0 DCT, 1 ADST, 2 FLIPADST, 3 IDTX).  The host reads these; tx_setup() uploads them to the __constant__ copies below
// for the kernels, and a kernel specialised for one size reads them at compile time (tx_w_dev).
constexpr uint8_t k_txw[19] = {4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64};
constexpr uint8_t k_txh[19] = {4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16};
constexpr uint8_t k_vtx[16] = {0, 1, 0, 1, 2, 0, 2, 1, 2, 3, 0, 3, 1, 3, 2, 3};
constexpr uint8_t k_htx[16] = {0, 0, 1, 1, 0, 2, 2, 2, 1, 3, 3, 0, 3, 1, 3, 2};
// the coded part of a side: 64-wide transforms keep their top-left 32 x 32 coefficients
__host__ __device__ constexpr int tx_coded(int n) { return n < 32 ? n : 32; }
// scan of a transform type (get_scan): 1 row scan for V_* (identity rows), 2 column scan for H_*, 0 the default scan
__host__ __device__ constexpr int scan_class(int vk, int hk) { return (vk != 3 && hk == 3) ? 1 : (vk == 3 && hk != 3) ? 2 : 0; }

__constant__ uint8_t c_txw[19];
__constant__ uint8_t c_txh[19];
__constant__ int8_t c_fwd_shift[19][3] = {{2, 0, 0},  {2, -1, 0}, {2, -2, 0}, {2, -4, 0}, {0, -2, -2}, {2, -1, 0}, {2, -1, 0},
                                          {2, -2, 0}, {2, -2, 0}, {2, -4, 0}, {2, -4, 0}, {0, -2, -2}, {2, -4, -2}, {2, -1, 0},
                                          {2, -1, 0}, {2, -2, 0}, {2, -2, 0}, {0, -2, 0}, {2, -4, 0}};
__constant__ int8_t c_inv_shift0[19] = {0, -1, -2, -2, -2, 0, 0, -1, -1, -1, -1, -1, -1, -1, -1, -2, -2, -2, -2};
__constant__ int8_t c_fwd_cos_col[5][5] = {{13, 13, 13, 0, 0}, {13, 13, 13, 12, 0}, {13, 13, 13, 12, 13}, {0, 13, 13, 12, 13}, {0, 0, 13, 12, 13}};
__constant__ int8_t c_fwd_cos_row[5][5] = {{13, 13, 12, 0, 0}, {13, 13, 13, 12, 0}, {13, 13, 12, 13, 12}, {0, 12, 13, 12, 11}, {0, 0, 12, 11, 10}};
__constant__ uint8_t c_vtx[16];
__constant__ uint8_t c_htx[16];

// Width / height of a transform in device code: a compile-time constant in a kernel specialised for size TS >= 0, so
// that its loop bounds and 1-D sizes fold; the __constant__ table for TS = -1 (any size).
template <int TS>
__device__ __forceinline__ int tx_w_dev(int tx_size) {
    if constexpr (TS >= 0) {
        constexpr int w = k_txw[TS];
        return w;
    } else {
        return c_txw[tx_size];
    }
}
template <int TS>
__device__ __forceinline__ int tx_h_dev(int tx_size) {
    if constexpr (TS >= 0) {
        constexpr int h = k_txh[TS];
        return h;
    } else {
        return c_txh[tx_size];
    }
}

// av1_transform_config / svt_av1_get_inv_txfm_cfg of (tx_size, tx_type).  TS >= 0 fixes the size: the fields derived
// from it are read from the tables as for any size, then w and h become compile-time constants, so that the passes
// over t (fwd_txfm2d, inv_txfm2d) get compile-time loop bounds and 1-D sizes.
template <int TS = -1>
__device__ TxCfg make_txcfg(int tx_size, int tx_type) {
    if (TS >= 0) tx_size = TS;
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
    t.w = tx_w_dev<TS>(tx_size);
    t.h = tx_h_dev<TS>(tx_size);
    return t;
}

} // namespace svtb200

using namespace svtb200;

namespace {

constexpr int TX_NT = 128; // threads per CTA of the transform kernels
__host__ __device__ constexpr int tx_pitch(int w) { return w | 1; } // odd pitch: conflict-free row pass
// blocks of a w x h transform per CTA: one lane per column / row of the longer side
__host__ __device__ constexpr int tx_bpc(int w, int h) { return TX_NT / (w > h ? w : h); }

// One descriptor per transform unit of a batched launch.
struct TuDev {
    int32_t x, y; // top-left sample inside the plane
    int32_t plane; // 0 Y, 1 Cb, 2 Cr
    int32_t tx_type;
};

// ---------------------------------------------------------------------------------------------------------------
// forward drop-in: one residual block (int16, w x h) -> coefficients (int32, contiguous w x h)
// ---------------------------------------------------------------------------------------------------------------
struct FwdArgs {
    const int16_t *in;
    int32_t *out;
    int tx_type, tx_size;
    int pf_shift; // 0 full, 1 N2, 2 N4: keep only the top-left (w>>s) x (h>>s) coefficients (EbTransforms.c:5401,7007)
};
__global__ void __launch_bounds__(TX_NT) fwd_txfm_kernel(const FwdArgs a) {
    extern __shared__ int32_t sm[];
    const TxCfg t = make_txcfg(a.tx_size, a.tx_type);
    const int w = t.w, h = t.h, T = max(w, h), pitch = tx_pitch(w), li = threadIdx.x;
    const bool live = li < T; // one block: the lanes past its longer side idle
    if (live)
        for (int i = li; i < w * h; i += T) {
            const int r = i / w, c = i - r * w;
            sm[r * pitch + c] = a.in[(t.ud ? h - 1 - r : r) * w + (t.lr ? w - 1 - c : c)];
        }
    __syncthreads();
    fwd_txfm2d(sm, pitch, t, li, T, live);
    __syncthreads();
    if (live) {
        const int kw = w >> a.pf_shift, kh = h >> a.pf_shift;
        for (int i = li; i < w * h; i += T) a.out[i] = ((i % w) < kw && (i / w) < kh) ? sm[(i / w) * pitch + (i % w)] : 0;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// inverse drop-in: one block of coefficients (64-wide sizes: the 32-wide packed input) -> residual added to the
// prediction, clipped (svt_av1_inv_txfm2d_add_*); prediction and reconstruction are w x h
// ---------------------------------------------------------------------------------------------------------------
struct InvArgs {
    const int32_t *in;
    const uint16_t *pred;
    uint16_t *recon;
    int tx_type, tx_size, bd;
};
__global__ void __launch_bounds__(TX_NT) inv_txfm_kernel(const InvArgs a) {
    extern __shared__ int32_t sm[];
    const TxCfg t = make_txcfg(a.tx_size, a.tx_type);
    const int w = t.w, h = t.h, iw = tx_coded(w), ih = tx_coded(h);
    const int T = max(w, h), pitch = tx_pitch(w), li = threadIdx.x;
    const bool live = li < T; // one block: the lanes past its longer side idle
    if (live)
        for (int i = li; i < w * h; i += T) {
            const int r = i / w, c = i - r * w;
            sm[r * pitch + c] = (r < ih && c < iw) ? a.in[r * iw + c] : 0;
        }
    __syncthreads();
    inv_txfm2d(sm, pitch, t, a.bd, li, T, live, [] {});
    __syncthreads();
    if (live) {
        const int mx = (1 << a.bd) - 1;
        for (int i = li; i < w * h; i += T) {
            const int r = i / w, c = i - r * w;
            // lr flip: output column c is the transform of buffer column w-1-c; ud flip: output row r = result row h-1-r
            const int32_t res = sm[(t.ud ? h - 1 - r : r) * pitch + (t.lr ? w - 1 - c : c)];
            const long long v = (long long)a.pred[i] + res;
            a.recon[i] = (uint16_t)(v < 0 ? 0 : (v > mx ? mx : v));
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
    const int w = tx_w_dev<TS>(d.tx_size), h = tx_h_dev<TS>(d.tx_size);
    const int iw = tx_coded(w), ih = tx_coded(h), n = iw * ih;
    const int lw = 31 - __clz(w), liw = 31 - __clz(iw);
    const int Tn = max(w, h), bpc = tx_bpc(w, h), pitch = tx_pitch(w);
    const int lb = threadIdx.x / Tn, li = threadIdx.x % Tn;
    const int b = blockIdx.x * bpc + lb;
    const bool live = b < d.n_tus && lb < bpc;
    int32_t *buf = sm + lb * (pitch * h);
    __shared__ int s_eob[TX_NT / 4], s_cul[TX_NT / 4];
    TuDev tu = {0, 0, 0, 0};
    if (live) tu = d.tus[b];
    const TxCfg t = make_txcfg<TS>(d.tx_size, tu.tx_type);
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
    fwd_txfm2d(buf, pitch, t, li, Tn, live);
    __syncthreads();
    // quantise + dequantise in place, in raster order (every coefficient is quantised independently; the scan order
    // only defines eob = 1 + the largest scan index of a non-zero level, looked up for the non-zero levels only).
    // Coefficients outside the kept 32x32 of 64-wide sizes are dropped = 0.
    if (live) {
        const int log_scale = (w * h > 256) + (w * h > 1024); // av1_get_tx_scale
        const int mode = d.quant_mode + (d.hbd ? 1 : 0);
        const int16_t *iscan = d.iscan[scan_class(t.vk, t.hk)];
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
    // the unit's eob and cul_level (complete in s_eob / s_cul after the barrier), published by its first lane
    inv_txfm2d(buf, pitch, t, bd, li, Tn, live, [=, &d] {
        if (li == 0) {
            const int ob = d.out_idx ? d.out_idx[b] : b;
            d.eob[ob] = (uint16_t)s_eob[lb];
            if (d.cul_level) d.cul_level[ob] = min(63, s_cul[lb]) + (dc_sign == 1 ? 64 : dc_sign == 2 ? 128 : 0);
        }
    });
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

// zero-out / re-pack of a 64-wide coefficient block, in place, with the energy of the dropped area
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
struct OisDev {
    const uint8_t *y;
    int stride, w, h, mbw, n_mb;
    long long *cost;
};
__global__ void __launch_bounds__(TX_NT) ois_dc_kernel(const OisDev d) {
    extern __shared__ int32_t sm[];
    constexpr int W = 16, BPC = tx_bpc(W, W), pitch = tx_pitch(W);
    const int lb = threadIdx.x / W, li = threadIdx.x % W;
    const int mb = blockIdx.x * BPC + lb;
    const bool live = mb < d.n_mb;
    int32_t *buf = sm + lb * (pitch * W);
    const TxCfg t = make_txcfg<2 /* TX_16X16 */>(2, 0 /* DCT_DCT */);
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
    fwd_txfm2d(buf, pitch, t, li, W, live);
    long long s = 0; // lane li sums the row it transformed last
    if (live)
#pragma unroll
        for (int c = 0; c < W; c++) s += abs(buf[li * pitch + c]);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (live && li == 0) d.cost[mb] = s;
}

// ---------------------------------------------------------------------------------------------------------------
// host helpers
// ---------------------------------------------------------------------------------------------------------------
static int coded_count(int tx_size) { return tx_coded(k_txw[tx_size]) * tx_coded(k_txh[tx_size]); }

// Launch of n transform blocks of w x h: CTAs of TX_NT threads holding tx_bpc(w, h) blocks, each block in its own
// odd-pitch int32 buffer in shared memory.
struct TxLaunch {
    int grid;
    size_t smem;
};
static TxLaunch tx_launch(int w, int h, int n) {
    const int bpc = tx_bpc(w, h);
    return {(n + bpc - 1) / bpc, (size_t)bpc * tx_pitch(w) * h * sizeof(int32_t)};
}

// What every transform kernel needs on the current device, once per device: the constant tables and the kernels'
// dynamic shared-memory limit.  Failures are fatal.
static void tx_setup() {
    static PerDeviceOnce once;
    once.run([] {
        txfm_upload_tables();
        SVTB_CUDA_FATAL(cudaMemcpyToSymbol(c_txw, k_txw, sizeof(k_txw)));
        SVTB_CUDA_FATAL(cudaMemcpyToSymbol(c_txh, k_txh, sizeof(k_txh)));
        SVTB_CUDA_FATAL(cudaMemcpyToSymbol(c_vtx, k_vtx, sizeof(k_vtx)));
        SVTB_CUDA_FATAL(cudaMemcpyToSymbol(c_htx, k_htx, sizeof(k_htx)));
        SVTB_ATTR(fwd_txfm_kernel, 64 * 1024);
        SVTB_ATTR(inv_txfm_kernel, 64 * 1024);
        SVTB_ATTR((encode_tu_kernel<uint8_t, -1>), 64 * 1024);
        SVTB_ATTR((encode_tu_kernel<uint16_t, -1>), 64 * 1024);
    });
}

// dc/ac pairs; the quantize_fp family passes no zbin / quant_shift, which read as zeros
static QuantTab quant_tab(const int16_t *zbin, const int16_t *round, const int16_t *quant, const int16_t *quant_shift,
                          const int16_t *dequant) {
    QuantTab q;
    for (int i = 0; i < 2; i++) {
        q.zbin[i] = zbin ? zbin[i] : 0;
        q.round[i] = round[i];
        q.quant[i] = quant[i];
        q.quant_shift[i] = quant_shift ? quant_shift[i] : 0;
        q.dequant[i] = dequant[i];
    }
    return q;
}

// plane pl (0 Y, 1 Cb, 2 Cr) of a frame and its stride in samples
struct FramePlane {
    void *ptr;
    int stride;
};
static FramePlane frame_plane(const SvtB200Frame *f, int pl) {
    return {pl == 0 ? f->y : pl == 1 ? f->cb : f->cr, pl == 0 ? f->stride_y : f->stride_c};
}

// ---- host side of the drop-ins --------------------------------------------------------------------------------
static void fwd_dropin(int16_t *input, int32_t *output, uint32_t stride, int tx_type, int tx_size, int pf_shift) {
    tx_setup();
    const int w = k_txw[tx_size], h = k_txh[tx_size];
    Staging s({(size_t)w * h * 2, (size_t)w * h * 4});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, input, stride, 2, w, h);
    SVTB_CUDA_FATAL(s.upload(0, 0));
    FwdArgs a;
    a.in = s.d<const int16_t>(0);
    a.out = s.d<int32_t>(1);
    a.tx_type = tx_type;
    a.tx_size = tx_size;
    a.pf_shift = pf_shift;
    SVTB_LAUNCH(fwd_txfm_kernel, 1, TX_NT, tx_launch(w, h, 1).smem, s.stream(), a);
    SVTB_CUDA_FATAL(s.download(1, 1));
    memcpy(output, s.h(1), (size_t)w * h * 4);
}

static void inv_dropin(const int32_t *input, uint16_t *output_r, int32_t stride_r, uint16_t *output_w, int32_t stride_w,
                       int tx_type, int tx_size, int bd) {
    tx_setup();
    const int w = k_txw[tx_size], h = k_txh[tx_size];
    const size_t nb = (size_t)coded_count(tx_size) * 4;
    Staging s({nb, (size_t)w * h * 2, (size_t)w * h * 2});
    SVTB_CUDA_FATAL(s.status());
    memcpy(s.h(0), input, nb);
    s.put_rows(1, output_r, stride_r, 2, w, h);
    SVTB_CUDA_FATAL(s.upload(0, 1));
    InvArgs a;
    a.in = s.d<const int32_t>(0);
    a.pred = s.d<const uint16_t>(1);
    a.recon = s.d<uint16_t>(2);
    a.tx_type = tx_type;
    a.tx_size = tx_size;
    a.bd = bd;
    SVTB_LAUNCH(inv_txfm_kernel, 1, TX_NT, tx_launch(w, h, 1).smem, s.stream(), a);
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
    a.q = quant_tab(zbin, round, quant, quant_shift, dequant);
    a.n = (int)n;
    a.log_scale = log_scale;
    a.mode = mode;
    SVTB_LAUNCH(quant_kernel, 1, 256, 0, s.stream(), a);
    SVTB_CUDA_FATAL(s.download(4, 6));
    memcpy(qcoeff, s.h(4), cb);
    memcpy(dqcoeff, s.h(5), cb);
    memcpy(eob, s.h(6), 2);
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

// ---- batched / picture-level entries ----------------------------------------------------------------------------
// device-resident scan tables of one size, built on first use per device: [3][1024] inverse scans (raster position ->
// scan index), then [3][1024] forward scans, each in scan_class order (default, row, column).  nullptr on a CUDA failure.
const int16_t *scan_tables(int tx_size) {
    static std::mutex mu;
    static int16_t *tabs[64][19] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev >= 64) return nullptr;
    std::lock_guard<std::mutex> lk(mu);
    if (tabs[dev][tx_size]) return tabs[dev][tx_size];
    static int16_t hs[1024], hi[6][1024];
    const int types[3] = {0, 10, 11}; // DCT_DCT (default scan), V_DCT (mrow), H_DCT (mcol)
    const int n = coded_count(tx_size);
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

template <int TS>
void encode_kernel_launch(const EncodeDev &d, const TxLaunch &l, cudaStream_t st) {
    if (d.hbd) SVTB_LAUNCH((encode_tu_kernel<uint16_t, TS>), l.grid, TX_NT, l.smem, st, d);
    else SVTB_LAUNCH((encode_tu_kernel<uint8_t, TS>), l.grid, TX_NT, l.smem, st, d);
}

int encode_launch(const SvtB200EncodeParams *p, int pf_shape, const long long *qoff, const int32_t *out_idx,
                  const SvtB200Frame *src, const SvtB200Frame *pred, const SvtB200Frame *recon, const SvtB200Tu *tus,
                  int32_t n_tus, int32_t *qcoeff, uint16_t *eob, int32_t *cul_level, void *stream) {
    if (!p || !src || !pred || !recon || !tus || !qcoeff || !eob || n_tus < 0 || p->tx_size < 0 || p->tx_size > 18 ||
        src->bit_depth != pred->bit_depth || src->bit_depth != recon->bit_depth) {
        set_error("svt_b200_encode_tus: bad argument");
        return SVT_B200_ERR_ARG;
    }
    if (n_tus == 0) return SVT_B200_OK;
    tx_setup();
    static_assert(sizeof(SvtB200Tu) == sizeof(TuDev), "descriptor layout");
    EncodeDev d;
    for (int i = 0; i < 3; i++) {
        const FramePlane s = frame_plane(src, i), pr = frame_plane(pred, i), rc = frame_plane(recon, i);
        d.src[i] = s.ptr, d.src_stride[i] = s.stride;
        d.pred[i] = pr.ptr, d.pred_stride[i] = pr.stride;
        d.recon[i] = rc.ptr, d.recon_stride[i] = rc.stride;
        const SvtB200QuantPlane &q = p->q[i];
        d.q[i] = quant_tab(q.zbin, p->use_fp ? q.round_fp : q.round, p->use_fp ? q.quant_fp : q.quant, q.quant_shift, q.dequant);
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
    const int16_t *tab = scan_tables(p->tx_size);
    if (!tab) return SVT_B200_ERR_CUDA;
    for (int i = 0; i < 3; i++) d.iscan[i] = tab + i * 1024;
    cudaStream_t st = (cudaStream_t)stream;
    const TxLaunch l = tx_launch(k_txw[p->tx_size], k_txh[p->tx_size], n_tus);
    switch (p->tx_size) {
    case 0: encode_kernel_launch<0>(d, l, st); break;
    case 1: encode_kernel_launch<1>(d, l, st); break;
    case 2: encode_kernel_launch<2>(d, l, st); break;
    case 3: encode_kernel_launch<3>(d, l, st); break;
    default: encode_kernel_launch<-1>(d, l, st); break;
    }
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

} // namespace

extern "C" {

// --- forward transforms: one exported symbol per RTCD pointer (aom_dsp_rtcd.h:105-216) ---
#define FWD_DROPIN(W, H, TXS)                                                                                     \
    void svt_av1_fwd_txfm2d_##W##x##H##_cuda(int16_t *input, int32_t *output, uint32_t input_stride, uint8_t tx_type, \
                                             uint8_t bit_depth) {                                                 \
        (void)bit_depth;                                                                                          \
        fwd_dropin(input, output, input_stride, tx_type, TXS, 0);                                                 \
    }                                                                                                             \
    void svt_av1_fwd_txfm2d_##W##x##H##_N2_cuda(int16_t *input, int32_t *output, uint32_t input_stride,           \
                                                uint8_t tx_type, uint8_t bit_depth) {                             \
        (void)bit_depth;                                                                                          \
        fwd_dropin(input, output, input_stride, tx_type, TXS, 1);                                                 \
    }                                                                                                             \
    void svt_av1_fwd_txfm2d_##W##x##H##_N4_cuda(int16_t *input, int32_t *output, uint32_t input_stride,           \
                                                uint8_t tx_type, uint8_t bit_depth) {                             \
        (void)bit_depth;                                                                                          \
        fwd_dropin(input, output, input_stride, tx_type, TXS, 2);                                                 \
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
uint64_t svt_b200_handle_transform64(int32_t *output, int tx_size) {
    const int w = k_txw[tx_size], h = k_txh[tx_size];
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
#define HANDLE64(W, H, TXS) \
    uint64_t svt_handle_transform##W##x##H##_cuda(int32_t *output) { return svt_b200_handle_transform64(output, TXS); }
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

void svt_residual_kernel8bit_cuda(uint8_t *input, uint32_t input_stride, uint8_t *pred, uint32_t pred_stride, int16_t *residual,
                                  uint32_t residual_stride, uint32_t area_width, uint32_t area_height) {
    residual_dropin(input, input_stride, pred, pred_stride, residual, residual_stride, area_width, area_height, 0);
}
void svt_residual_kernel16bit_cuda(uint16_t *input, uint32_t input_stride, uint16_t *pred, uint32_t pred_stride,
                                   int16_t *residual, uint32_t residual_stride, uint32_t area_width, uint32_t area_height) {
    residual_dropin(input, input_stride, pred, pred_stride, residual, residual_stride, area_width, area_height, 1);
}

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
    const int w = k_txw[tx_size], h = k_txh[tx_size];
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
    const int w = tx_coded(k_txw[tx_size]), h = tx_coded(k_txh[tx_size]), cls = scan_class(k_vtx[tx_type], k_htx[tx_type]);
    int n = 0;
    if (cls == 1) { // V_DCT / V_ADST / V_FLIPADST: mrow_scan (raster)
        for (int i = 0; i < w * h; i++) scan_out[n++] = (int16_t)i;
    } else if (cls == 2) { // H_*: mcol_scan
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
    const int n = coded_count(tx_size);
    SVTB_LAUNCH(eob_scan_kernel, 1, 1024, 0, st, eob, n_tus, offsets, total, base);
    SVTB_LAUNCH(pack_levels_kernel, (n_tus + 7) / 8, 256, 0, st, qcoeff, eob, offsets, tab + 3072 + tx_class * 1024, n_tus, n, packed);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

int svt_b200_encode_tus(const SvtB200EncodeParams *p, const SvtB200Frame *src, const SvtB200Frame *pred,
                        const SvtB200Frame *recon, const SvtB200Tu *tus, int32_t n_tus, int32_t *qcoeff, uint16_t *eob,
                        void *scratch, void *stream) {
    (void)scratch; // kept for ABI stability: the scan tables are resident per device since round 1
    return svt_b200_encode_tus_cul(p, src, pred, recon, tus, n_tus, qcoeff, eob, nullptr, stream);
}

int svt_b200_encode_tus_cul(const SvtB200EncodeParams *p, const SvtB200Frame *src, const SvtB200Frame *pred,
                            const SvtB200Frame *recon, const SvtB200Tu *tus, int32_t n_tus, int32_t *qcoeff, uint16_t *eob,
                            int32_t *cul_level, void *stream) {
    return encode_launch(p, 0, nullptr, nullptr, src, pred, recon, tus, n_tus, qcoeff, eob, cul_level, stream);
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
        off += coded_count(t.tx_size);
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

// pic: 8-bit picture (the luma plane is read); cost: DEVICE int64 [mb rows][mb cols], mb cols = (width + 15) / 16 =
// the reference's mb_stride; every entry is OisMbResults::intra_cost of that macroblock, its intra_mode is DC_PRED.
int svt_b200_ois_dc_picture(const SvtB200Frame *pic, int64_t *cost, void *stream) {
    if (!pic || !pic->y || pic->bit_depth != 8 || !cost || pic->width <= 0 || pic->height <= 0) {
        set_error("svt_b200_ois_dc_picture: bad argument (8-bit pictures)");
        return SVT_B200_ERR_ARG;
    }
    tx_setup();
    OisDev d;
    d.y = (const uint8_t *)pic->y, d.stride = pic->stride_y, d.w = pic->width, d.h = pic->height;
    d.mbw = (pic->width + 15) / 16;
    d.n_mb = d.mbw * ((pic->height + 15) / 16);
    d.cost = (long long *)cost;
    const TxLaunch l = tx_launch(16, 16, d.n_mb);
    SVTB_LAUNCH(ois_dc_kernel, l.grid, TX_NT, l.smem, (cudaStream_t)stream, d);
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
