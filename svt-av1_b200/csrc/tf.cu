// tf.cu — the temporal filter's planewise weighting on sm_90a (SURVEY.md 8(f) rank 4).
//
// Replaces (reference: Source/Lib/Encoder/Codec/EbTemporalFiltering.c):
//   svt_av1_apply_temporal_filter_planewise_c      :643-811   (aom_dsp_rtcd.c:365)
//   svt_av1_apply_temporal_filter_planewise_hbd_c  :829-1017  (aom_dsp_rtcd.c:366)
//   apply_filtering_central[_highbd]               :551-621
//   get_final_filtered_pixels                      :1943-2050
//
// Per sample of a 32x32 block the reference sums the squared prediction error over a 5x5 window clamped to the block
// (chroma: 5x5 chroma window + the co-located 2x2 luma errors), then turns it into a weight through a short chain of
// double operations and one expf:  w = (int)(expf((float)-min((5 * sum / n + block_error) / 6 * d_factor / den, 7)) * 1000).
// IEEE double +, *, / are the same on every machine when they are not fused or reordered - the chain is written with
// the round-to-nearest intrinsics.  expf is the algorithm glibc (>= 2.27) uses, restated with the same discipline; the
// oracle's copy is compared with the host libm on all 1.09e9 floats of [-8, -0] (tests/test_oracle_tf.py) and this
// kernel's copy with the oracle's on the same set (tests/test_tf_gpu.py), so the weights are the reference's, not close to.
//
// Mapping: one CTA per 32x32 block (up to 64x64), 256 threads; squared errors of the block's three planes are staged
// in shared memory once; a thread produces the luma weights of its samples and, for even (row, col), the two chroma
// weights.  The block-level terms (block_error and d_factor per 16x16 quadrant: tf_16x16/32x32_block_error and MVs of
// MeContext, sqrtf / powf) and the per-plane denominator 2 n_decay^2 (log1p of the noise level) are computed by the
// caller on the host exactly as the reference does and arrive as doubles.
#include "common.cuh"

using namespace svtb200;

namespace {

__constant__ unsigned long long c_exp2f_tab[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull, 0x3fef72b83c7d517bull,
    0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull, 0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull,
    0x3feedea64c123422ull, 0x3feece086061892dull, 0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull,
    0x3feea47eb03a5585ull, 0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull, 0x3feee89f995ad3adull,
    0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull, 0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full,
    0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull};

// glibc's expf (sysdeps/ieee754/flt-32/e_expf.c) for |x| < 87: N = 32 table, degree-3 polynomial, all in double
__device__ __forceinline__ float expf_exact(float x) {
    const double inv_ln2_n = 0x1.71547652b82fep+0 * 32, shift = 0x1.8p52;
    const double c0 = 0x1.c6af84b912394p-5 / 32 / 32 / 32, c1 = 0x1.ebfce50fac4f3p-3 / 32 / 32, c2 = 0x1.62e42ff0c52d6p-1 / 32;
    const double z = __dmul_rn(inv_ln2_n, (double)x);
    double kd = __dadd_rn(z, shift);
    const unsigned long long ki = (unsigned long long)__double_as_longlong(kd);
    kd = __dsub_rn(kd, shift);
    const double r = __dsub_rn(z, kd);
    const double s = __longlong_as_double((long long)(c_exp2f_tab[ki & 31] + (ki << 47)));
    const double zz = __dadd_rn(__dmul_rn(c0, r), c1);
    const double r2 = __dmul_rn(r, r);
    double y = __dadd_rn(__dmul_rn(c2, r), 1.0);
    y = __dadd_rn(__dmul_rn(zz, r2), y);
    y = __dmul_rn(y, s);
    return __double2float_rn(y);
}

__device__ __forceinline__ int tf_weight(unsigned long long sum, int n, double block_error, double d_factor, double den) {
    const double window_error = __ddiv_rn(__ull2double_rn(sum), (double)n);
    const double combined = __ddiv_rn(__dadd_rn(__dmul_rn(5.0, window_error), block_error), 6.0);
    const double b = __ddiv_rn(__dmul_rn(combined, d_factor), den);
    const double scaled = b < 7.0 ? b : 7.0;
    return (int)__fmul_rn(expf_exact(__double2float_rn(-scaled)), 1000.0f);
}

struct TfBlockDev { // == SvtB200TfBlock
    int32_t x, y;
    double block_error[4], d_factor[4];
};
struct TfDev {
    const void *src[3], *pre[3];
    int src_stride[2], pre_stride[2]; // luma, chroma (samples)
    uint32_t *accum[3];
    uint16_t *count[3];
    int acc_stride[2];
    double den[3];
    int bw, bh, chroma, shift; // shift = 2 * (bit_depth - 8)
    const TfBlockDev *blocks;
};

template <typename T>
__global__ void __launch_bounds__(256) tf_planewise_kernel(const TfDev d) {
    __shared__ uint32_t s_y[64 * 64];
    __shared__ uint32_t s_u[32 * 32], s_v[32 * 32];
    const TfBlockDev b = d.blocks[blockIdx.x];
    const int bw = d.bw, bh = d.bh, uw = bw >> 1, uh = bh >> 1, tid = threadIdx.x;
    const T *ys = reinterpret_cast<const T *>(d.src[0]) + (size_t)b.y * d.src_stride[0] + b.x;
    const T *yp = reinterpret_cast<const T *>(d.pre[0]) + (size_t)b.y * d.pre_stride[0] + b.x;
    for (int i = tid; i < bw * bh; i += 256) {
        const int r = i / bw, c = i - r * bw;
        const int df = (int)ys[(size_t)r * d.src_stride[0] + c] - (int)yp[(size_t)r * d.pre_stride[0] + c];
        s_y[i] = (uint32_t)(df * df);
    }
    const size_t co_s = (size_t)(b.y >> 1) * d.src_stride[1] + (b.x >> 1), co_p = (size_t)(b.y >> 1) * d.pre_stride[1] + (b.x >> 1);
    const T *up = reinterpret_cast<const T *>(d.pre[1]) + co_p, *vp = reinterpret_cast<const T *>(d.pre[2]) + co_p;
    if (d.chroma) {
        const T *us = reinterpret_cast<const T *>(d.src[1]) + co_s, *vs = reinterpret_cast<const T *>(d.src[2]) + co_s;
        for (int i = tid; i < uw * uh; i += 256) {
            const int r = i / uw, c = i - r * uw;
            const int du = (int)us[(size_t)r * d.src_stride[1] + c] - (int)up[(size_t)r * d.pre_stride[1] + c];
            const int dv = (int)vs[(size_t)r * d.src_stride[1] + c] - (int)vp[(size_t)r * d.pre_stride[1] + c];
            s_u[i] = (uint32_t)(du * du);
            s_v[i] = (uint32_t)(dv * dv);
        }
    }
    __syncthreads();
    uint32_t *ya = d.accum[0] + (size_t)b.y * d.acc_stride[0] + b.x;
    uint16_t *yc = d.count[0] + (size_t)b.y * d.acc_stride[0] + b.x;
    for (int i = tid; i < bw * bh; i += 256) {
        const int r = i / bw, c = i - r * bw;
        unsigned long long sum = 0;
#pragma unroll
        for (int dy = -2; dy <= 2; dy++) {
            const int rr = min(max(r + dy, 0), bh - 1);
#pragma unroll
            for (int dx = -2; dx <= 2; dx++) sum += s_y[rr * bw + min(max(c + dx, 0), bw - 1)];
        }
        const int q = (r >= bh / 2) * 2 + (c >= bw / 2);
        const int w = tf_weight(sum >> d.shift, 25, b.block_error[q], b.d_factor[q], d.den[0]);
        const size_t k = (size_t)r * d.acc_stride[0] + c;
        yc[k] = (uint16_t)(yc[k] + w);
        ya[k] += (uint32_t)(w * (int)yp[(size_t)r * d.pre_stride[0] + c]);
    }
    if (!d.chroma) return;
    const size_t co_a = (size_t)(b.y >> 1) * d.acc_stride[1] + (b.x >> 1);
    for (int i = tid; i < uw * uh; i += 256) {
        const int ur = i / uw, uc = i - ur * uw, r = ur * 2, c = uc * 2;
        unsigned long long su = (unsigned long long)s_y[r * bw + c] + s_y[r * bw + c + 1] + s_y[(r + 1) * bw + c] + s_y[(r + 1) * bw + c + 1];
        unsigned long long sv = su;
#pragma unroll
        for (int dy = -2; dy <= 2; dy++) {
            const int rr = min(max(ur + dy, 0), uh - 1);
#pragma unroll
            for (int dx = -2; dx <= 2; dx++) {
                const int cc = min(max(uc + dx, 0), uw - 1);
                su += s_u[rr * uw + cc];
                sv += s_v[rr * uw + cc];
            }
        }
        const int q = (r >= bh / 2) * 2 + (c >= bw / 2);
        const size_t m = co_a + (size_t)ur * d.acc_stride[1] + uc;
        int w = tf_weight(su >> d.shift, 29, b.block_error[q], b.d_factor[q], d.den[1]);
        d.count[1][m] = (uint16_t)(d.count[1][m] + w);
        d.accum[1][m] += (uint32_t)(w * (int)up[(size_t)ur * d.pre_stride[1] + uc]);
        w = tf_weight(sv >> d.shift, 29, b.block_error[q], b.d_factor[q], d.den[2]);
        d.count[2][m] = (uint16_t)(d.count[2][m] + w);
        d.accum[2][m] += (uint32_t)(w * (int)vp[(size_t)ur * d.pre_stride[1] + uc]);
    }
}

// the centre frame (weight 1000 everywhere) and the final normalisation, picture-wide: plane p of grid.y
struct TfPlaneDev {
    void *pix[3];
    int pix_stride[2], acc_stride[2], w[2], h[2];
    uint32_t *accum[3];
    uint16_t *count[3];
    unsigned long long *sse; // [2]: luma, chroma
    int n_planes;
};
template <typename T>
__global__ void __launch_bounds__(256) tf_central_kernel(const TfPlaneDev d) {
    const int p = blockIdx.y, c = p ? 1 : 0, w = d.w[c], h = d.h[c];
    const T *px = reinterpret_cast<const T *>(d.pix[p]);
    for (int i = blockIdx.x * 256 + threadIdx.x; i < w * h; i += gridDim.x * 256) {
        const int r = i / w, x = i - r * w;
        const size_t k = (size_t)r * d.acc_stride[c] + x;
        d.accum[p][k] += 1000u * (uint32_t)px[(size_t)r * d.pix_stride[c] + x];
        d.count[p][k] = (uint16_t)(d.count[p][k] + 1000);
    }
}
template <typename T>
__global__ void __launch_bounds__(256) tf_normalize_kernel(const TfPlaneDev d) {
    const int p = blockIdx.y, c = p ? 1 : 0, w = d.w[c], h = d.h[c];
    T *px = reinterpret_cast<T *>(d.pix[p]);
    unsigned long long sse = 0;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < w * h; i += gridDim.x * 256) {
        const int r = i / w, x = i - r * w;
        const size_t k = (size_t)r * d.acc_stride[c] + x;
        const uint32_t cnt = d.count[p][k], v = (d.accum[p][k] + (cnt >> 1)) / cnt;
        const int df = (int)px[(size_t)r * d.pix_stride[c] + x] - (int)v;
        sse += (unsigned long long)((long long)df * df);
        px[(size_t)r * d.pix_stride[c] + x] = (T)v;
    }
    for (int o = 16; o > 0; o >>= 1) sse += __shfl_xor_sync(0xffffffffu, sse, o);
    if ((threadIdx.x & 31) == 0 && sse && d.sse) atomicAdd(&d.sse[c], sse);
}

__global__ void expf_checksum_kernel(uint32_t lo, uint32_t hi, unsigned long long *out) {
    unsigned long long acc = 0;
    for (unsigned long long u = (unsigned long long)lo + blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; u <= hi;
         u += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t v = (uint32_t)u;
        const uint32_t o = __float_as_uint(expf_exact(__uint_as_float(v)));
        acc += (unsigned long long)o * (unsigned long long)(2 * (v & 0xffff) + 1);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}

bool frames_ok(const SvtB200Frame *a, const SvtB200Frame *b) {
    return a && b && a->y && b->y && a->bit_depth == b->bit_depth && (a->bit_depth == 8 || a->bit_depth == 10 || a->bit_depth == 12);
}

} // namespace

extern "C" {

int svt_b200_tf_planewise(const SvtB200TfParams *p, const SvtB200Frame *src, const SvtB200Frame *pred, const SvtB200TfBlock *blocks,
                          int32_t n_blocks, const SvtB200TfAccum *acc, void *stream) {
    static_assert(sizeof(TfBlockDev) == sizeof(SvtB200TfBlock), "SvtB200TfBlock layout");
    if (!p || !frames_ok(src, pred) || !blocks || !acc || n_blocks < 0 || p->block_w < 2 || p->block_h < 2 || p->block_w > 64 ||
        p->block_h > 64 || (p->block_w & 1) || (p->block_h & 1) || !acc->accum[0] || !acc->count[0] ||
        (p->chroma && (!src->cb || !src->cr || !pred->cb || !pred->cr || !acc->accum[1] || !acc->accum[2] || !acc->count[1] || !acc->count[2]))) {
        set_error("svt_b200_tf_planewise: bad argument");
        return SVT_B200_ERR_ARG;
    }
    if (n_blocks == 0) return SVT_B200_OK;
    TfDev d;
    d.src[0] = src->y, d.src[1] = src->cb, d.src[2] = src->cr;
    d.pre[0] = pred->y, d.pre[1] = pred->cb, d.pre[2] = pred->cr;
    d.src_stride[0] = src->stride_y, d.src_stride[1] = src->stride_c;
    d.pre_stride[0] = pred->stride_y, d.pre_stride[1] = pred->stride_c;
    for (int i = 0; i < 3; i++) d.accum[i] = acc->accum[i], d.count[i] = acc->count[i], d.den[i] = p->den[i];
    d.acc_stride[0] = acc->stride_y, d.acc_stride[1] = acc->stride_c;
    d.bw = p->block_w, d.bh = p->block_h, d.chroma = p->chroma, d.shift = 2 * (src->bit_depth - 8);
    d.blocks = reinterpret_cast<const TfBlockDev *>(blocks);
    cudaStream_t st = (cudaStream_t)stream;
    if (src->bit_depth > 8)
        SVTB_LAUNCH(tf_planewise_kernel<uint16_t>, n_blocks, 256, 0, st, d);
    else
        SVTB_LAUNCH(tf_planewise_kernel<uint8_t>, n_blocks, 256, 0, st, d);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

static int plane_pass(int normalize, const SvtB200Frame *f, const SvtB200TfAccum *acc, int32_t chroma, unsigned long long *sse, void *stream) {
    if (!f || !f->y || !acc || !acc->accum[0] || !acc->count[0] || (chroma && (!f->cb || !f->cr || !acc->accum[1] || !acc->accum[2]))) {
        set_error("svt_b200_tf_central / _normalize: bad argument");
        return SVT_B200_ERR_ARG;
    }
    TfPlaneDev d;
    d.pix[0] = f->y, d.pix[1] = f->cb, d.pix[2] = f->cr;
    d.pix_stride[0] = f->stride_y, d.pix_stride[1] = f->stride_c;
    d.acc_stride[0] = acc->stride_y, d.acc_stride[1] = acc->stride_c;
    d.w[0] = f->width, d.h[0] = f->height, d.w[1] = (f->width + 1) >> 1, d.h[1] = (f->height + 1) >> 1;
    for (int i = 0; i < 3; i++) d.accum[i] = acc->accum[i], d.count[i] = acc->count[i];
    d.sse = sse;
    d.n_planes = chroma ? 3 : 1;
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 g(std::min(1184, (f->width * f->height + 255) / 256), d.n_planes);
    if (normalize) {
        if (sse) SVTB_CUDA_TRY(cudaMemsetAsync(sse, 0, 16, st));
        if (f->bit_depth > 8)
            SVTB_LAUNCH(tf_normalize_kernel<uint16_t>, g, 256, 0, st, d);
        else
            SVTB_LAUNCH(tf_normalize_kernel<uint8_t>, g, 256, 0, st, d);
    } else {
        if (f->bit_depth > 8)
            SVTB_LAUNCH(tf_central_kernel<uint16_t>, g, 256, 0, st, d);
        else
            SVTB_LAUNCH(tf_central_kernel<uint8_t>, g, 256, 0, st, d);
    }
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

int svt_b200_tf_central(const SvtB200Frame *center, const SvtB200TfAccum *acc, int32_t chroma, void *stream) {
    return plane_pass(0, center, acc, chroma, nullptr, stream);
}

int svt_b200_tf_normalize(const SvtB200Frame *dst, const SvtB200TfAccum *acc, int32_t chroma, uint64_t *sse2, void *stream) {
    return plane_pass(1, dst, acc, chroma, reinterpret_cast<unsigned long long *>(sse2), stream);
}

// checksum of this library's expf over the floats with bit patterns lo..hi (test hook: compared with the oracle's)
int svt_b200_tf_expf_checksum(uint32_t lo_bits, uint32_t hi_bits, uint64_t *out_host) {
    Staging s({8});
    SVTB_CUDA_TRY(s.status());
    SVTB_CUDA_TRY(cudaMemsetAsync(s.d(0), 0, 8, s.stream()));
    SVTB_LAUNCH(expf_checksum_kernel, 132 * 8, 256, 0, s.stream(), lo_bits, hi_bits, s.d<unsigned long long>(0));
    SVTB_CUDA_TRY(cudaGetLastError());
    SVTB_CUDA_TRY(s.download(0, 0));
    memcpy(out_host, s.h(0), 8);
    return SVT_B200_OK;
}

// One block with HOST pointers in the reference's layout (the body of the RTCD drop-ins for
// svt_av1_apply_temporal_filter_planewise / _hbd: oracle/rtcd_install.c reads the MeContext fields, computes den /
// block_error / d_factor as the reference does, and calls this).  accum / count use the prediction's strides.
int svt_b200_tf_planewise_block_host(int32_t bit_depth, int32_t chroma, const void *y_src, int32_t y_src_stride, const void *y_pre,
                                     int32_t y_pre_stride, const void *u_src, const void *v_src, int32_t uv_src_stride,
                                     const void *u_pre, const void *v_pre, int32_t uv_pre_stride, uint32_t bw, uint32_t bh,
                                     const double *den3, const double *block_error4, const double *d_factor4, uint32_t *y_accum,
                                     uint16_t *y_count, uint32_t *u_accum, uint16_t *u_count, uint32_t *v_accum, uint16_t *v_count) {
    if (bw > 64 || bh > 64 || bw < 2 || bh < 2 || ((bw | bh) & 1)) {
        set_error("svt_b200_tf_planewise_block_host: block %ux%u", bw, bh);
        return SVT_B200_ERR_ARG;
    }
    const int es = bit_depth > 8 ? 2 : 1, uw = bw / 2, uh = bh / 2;
    // [src y | src u | src v | pre y | pre u | pre v] samples, then accum x3 (u32), count x3 (u16), block
    const size_t ny = (size_t)bw * bh, nc = (size_t)uw * uh;
    Staging s({ny * es, nc * es, nc * es, ny * es, nc * es, nc * es, ny * 4, nc * 4, nc * 4, ny * 2, nc * 2, nc * 2, sizeof(TfBlockDev)});
    SVTB_CUDA_TRY(s.status());
    s.put_rows(0, y_src, y_src_stride, es, bw, bh);
    s.put_rows(3, y_pre, y_pre_stride, es, bw, bh);
    s.put_rows(6, y_accum, y_pre_stride, 4, bw, bh);
    s.put_rows(9, y_count, y_pre_stride, 2, bw, bh);
    if (chroma) {
        s.put_rows(1, u_src, uv_src_stride, es, uw, uh);
        s.put_rows(2, v_src, uv_src_stride, es, uw, uh);
        s.put_rows(4, u_pre, uv_pre_stride, es, uw, uh);
        s.put_rows(5, v_pre, uv_pre_stride, es, uw, uh);
        s.put_rows(7, u_accum, uv_pre_stride, 4, uw, uh);
        s.put_rows(8, v_accum, uv_pre_stride, 4, uw, uh);
        s.put_rows(10, u_count, uv_pre_stride, 2, uw, uh);
        s.put_rows(11, v_count, uv_pre_stride, 2, uw, uh);
    }
    TfBlockDev *blk = s.h<TfBlockDev>(12);
    blk->x = blk->y = 0;
    for (int i = 0; i < 4; i++) blk->block_error[i] = block_error4[i], blk->d_factor[i] = d_factor4[i];
    SVTB_CUDA_TRY(s.upload(0, 12));
    SvtB200Frame fs = {s.d(0), s.d(1), s.d(2), (int32_t)bw, (int32_t)uw, (int32_t)bw, (int32_t)bh, bit_depth};
    SvtB200Frame fp = {s.d(3), s.d(4), s.d(5), (int32_t)bw, (int32_t)uw, (int32_t)bw, (int32_t)bh, bit_depth};
    SvtB200TfAccum acc;
    for (int i = 0; i < 3; i++) acc.accum[i] = s.d<uint32_t>(6 + i), acc.count[i] = s.d<uint16_t>(9 + i);
    acc.stride_y = bw, acc.stride_c = uw;
    SvtB200TfParams p;
    for (int i = 0; i < 3; i++) p.den[i] = den3[i];
    p.chroma = chroma, p.block_w = bw, p.block_h = bh;
    const int rc = svt_b200_tf_planewise(&p, &fs, &fp, s.d<const SvtB200TfBlock>(12), 1, &acc, s.stream());
    if (rc) return rc;
    SVTB_CUDA_TRY(s.download(6, 11));
    s.get_rows(6, y_accum, y_pre_stride, 4, bw, bh);
    s.get_rows(9, y_count, y_pre_stride, 2, bw, bh);
    if (chroma) {
        s.get_rows(7, u_accum, uv_pre_stride, 4, uw, uh);
        s.get_rows(8, v_accum, uv_pre_stride, 4, uw, uh);
        s.get_rows(10, u_count, uv_pre_stride, 2, uw, uh);
        s.get_rows(11, v_count, uv_pre_stride, 2, uw, uh);
    }
    return SVT_B200_OK;
}
}
