// misc.cu — the small reductions that sit next to the transform chain and the single-position SAD family, as RTCD
// drop-ins (host pointers).  Replaces (reference files under Source/Lib):
//   svt_aom_subtract_block / svt_aom_highbd_subtract_block          Common/Codec/EbInterPrediction.c:65
//   svt_full_distortion_kernel32_bits / _cbf_zero32_bits            Common/Codec/EbPictureOperators.c:156-231
//   svt_spatial_full_distortion_kernel / svt_full_distortion_kernel16_bits  Common/C_DEFAULT/EbPictureOperators_C.c:65, EbPictureOperators.c:182
//   svt_aom_satd, svt_av1_block_error                               Common/Codec/common_dsp_rtcd.c:47-69
//   svt_aom_sadMxN, svt_aom_sadMxNx4d (22 sizes), svt_nxm_sad_kernel(_sub_sampled), sad_16b_kernel
//                                                                   Encoder/C_DEFAULT/sad_av1.c, EbComputeSAD_C.c:39-56
// One block-wide reduction kernel serves all of them (mode selects the per-element term); these calls are tiny, so
// the wrappers exist for pointer-table completeness and parity tests, not for throughput.
#include "common.cuh"

using namespace svtb200;

namespace {

enum { M_SAD8 = 0, M_SAD16, M_SSE8, M_SSE16, M_DIST32, M_SQ32, M_SATD, M_BLKERR, M_VAR8 };

// a, b: packed w x h arrays (element size by mode). out[0], out[1]: 64-bit results.
__global__ void __launch_bounds__(256) reduce2_kernel(const void *a, const void *b, int n, int mode, unsigned long long *out) {
    unsigned long long r0 = 0, r1 = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        switch (mode) {
        case M_SAD8: r0 += (unsigned)abs((int)((const uint8_t *)a)[i] - (int)((const uint8_t *)b)[i]); break;
        case M_SAD16: r0 += (unsigned)abs((int)((const uint16_t *)a)[i] - (int)((const uint16_t *)b)[i]); break;
        case M_SSE8: {
            const long long d = (long long)((const uint8_t *)a)[i] - ((const uint8_t *)b)[i];
            r0 += (unsigned long long)(d * d);
            break;
        }
        case M_SSE16: {
            const long long d = (long long)((const uint16_t *)a)[i] - ((const uint16_t *)b)[i];
            r0 += (unsigned long long)(d * d);
            break;
        }
        case M_DIST32: {
            const long long c = ((const int32_t *)a)[i], d = c - (long long)((const int32_t *)b)[i];
            r0 += (unsigned long long)(d * d);
            r1 += (unsigned long long)(c * c);
            break;
        }
        case M_SQ32: {
            const long long c = ((const int32_t *)a)[i];
            r0 += (unsigned long long)(c * c);
            break;
        }
        case M_SATD: r0 += (unsigned long long)(long long)abs(((const int32_t *)a)[i]); break;
        case M_VAR8: { // variance_c: sum of differences (two's complement in r0) and of their squares
            const long long d = (long long)((const uint8_t *)a)[i] - ((const uint8_t *)b)[i];
            r0 += (unsigned long long)d;
            r1 += (unsigned long long)(d * d);
            break;
        }
        default: { // svt_av1_block_error_c: int products (32-bit), 64-bit sums
            const int c = ((const int32_t *)a)[i], d = c - ((const int32_t *)b)[i];
            r0 += (unsigned long long)(long long)(int)((unsigned)d * (unsigned)d);
            r1 += (unsigned long long)(long long)(int)((unsigned)c * (unsigned)c);
            break;
        }
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        r0 += __shfl_xor_sync(0xffffffffu, r0, o);
        r1 += __shfl_xor_sync(0xffffffffu, r1, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&out[0], r0);
        atomicAdd(&out[1], r1);
    }
}
template <typename T>
__global__ void subtract_kernel(const T *src, const T *pred, int16_t *diff, int n) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) diff[i] = (int16_t)((int)src[i] - (int)pred[i]);
}

// returns {r0, r1}
static void reduce2(const void *a, size_t sa, const void *b, size_t sb, int w, int h, int esz, int mode, uint64_t res[2]) {
    const size_t nb = (size_t)w * h * esz;
    Staging s({nb, nb, 16});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, a, sa, esz, w, h);
    if (b) s.put_rows(1, b, sb, esz, w, h);
    memset(s.h(2), 0, 16);
    SVTB_CUDA_FATAL(s.upload(0, 2));
    SVTB_LAUNCH(reduce2_kernel, 1, 256, 0, s.stream(), (const void *)s.d(0), (const void *)s.d(1), w * h, mode,
                s.d<unsigned long long>(2));
    SVTB_CUDA_FATAL(s.download(2, 2));
    memcpy(res, s.h(2), 16);
}

static void subtract(int rows, int cols, int16_t *diff, ptrdiff_t ds, const void *src, ptrdiff_t ss, const void *pred, ptrdiff_t ps,
                     int esz) {
    const size_t nb = (size_t)rows * cols * esz;
    Staging s({nb, nb, (size_t)rows * cols * 2});
    SVTB_CUDA_FATAL(s.status());
    s.put_rows(0, src, ss, esz, cols, rows);
    s.put_rows(1, pred, ps, esz, cols, rows);
    SVTB_CUDA_FATAL(s.upload(0, 1));
    if (esz == 2)
        SVTB_LAUNCH(subtract_kernel<uint16_t>, 4, 256, 0, s.stream(), s.d<const uint16_t>(0), s.d<const uint16_t>(1), s.d<int16_t>(2),
                    rows * cols);
    else
        SVTB_LAUNCH(subtract_kernel<uint8_t>, 4, 256, 0, s.stream(), s.d<const uint8_t>(0), s.d<const uint8_t>(1), s.d<int16_t>(2),
                    rows * cols);
    SVTB_CUDA_FATAL(s.download(2, 2));
    s.get_rows(2, diff, ds, 2, cols, rows);
}

} // namespace

extern "C" {

void svt_aom_subtract_block_cuda(int rows, int cols, int16_t *diff_ptr, ptrdiff_t diff_stride, const uint8_t *src_ptr,
                                 ptrdiff_t src_stride, const uint8_t *pred_ptr, ptrdiff_t pred_stride) {
    subtract(rows, cols, diff_ptr, diff_stride, src_ptr, src_stride, pred_ptr, pred_stride, 1);
}
void svt_aom_highbd_subtract_block_cuda(int rows, int cols, int16_t *diff_ptr, ptrdiff_t diff_stride, const uint8_t *src_ptr,
                                        ptrdiff_t src_stride, const uint8_t *pred_ptr, ptrdiff_t pred_stride, int bd) {
    (void)bd; // CONVERT_TO_SHORTPTR convention of the reference
    subtract(rows, cols, diff_ptr, diff_stride, (const void *)(((uintptr_t)src_ptr) << 1), src_stride,
             (const void *)(((uintptr_t)pred_ptr) << 1), pred_stride, 2);
}
void svt_full_distortion_kernel32_bits_cuda(int32_t *coeff, uint32_t coeff_stride, int32_t *recon_coeff, uint32_t recon_coeff_stride,
                                            uint64_t distortion_result[2], uint32_t area_width, uint32_t area_height) {
    reduce2(coeff, coeff_stride, recon_coeff, recon_coeff_stride, area_width, area_height, 4, M_DIST32, distortion_result);
}
void svt_full_distortion_kernel_cbf_zero32_bits_cuda(int32_t *coeff, uint32_t coeff_stride, uint64_t distortion_result[2],
                                                     uint32_t area_width, uint32_t area_height) {
    uint64_t r[2];
    reduce2(coeff, coeff_stride, nullptr, 0, area_width, area_height, 4, M_SQ32, r);
    distortion_result[0] = distortion_result[1] = r[0];
}
uint64_t svt_spatial_full_distortion_kernel_cuda(uint8_t *input, uint32_t input_offset, uint32_t input_stride, uint8_t *recon,
                                                 int32_t recon_offset, uint32_t recon_stride, uint32_t area_width,
                                                 uint32_t area_height) {
    uint64_t r[2];
    reduce2(input + input_offset, input_stride, recon + recon_offset, recon_stride, area_width, area_height, 1, M_SSE8, r);
    return r[0];
}
uint64_t svt_full_distortion_kernel16_bits_cuda(uint8_t *input, uint32_t input_offset, uint32_t input_stride, uint8_t *recon,
                                                int32_t recon_offset, uint32_t recon_stride, uint32_t area_width,
                                                uint32_t area_height) {
    uint64_t r[2];
    reduce2((uint16_t *)input + input_offset, input_stride, (uint16_t *)recon + recon_offset, recon_stride, area_width, area_height, 2,
            M_SSE16, r);
    return r[0];
}
int svt_aom_satd_cuda(const int32_t *coeff, int length) {
    uint64_t r[2];
    reduce2(coeff, length, nullptr, 0, length, 1, 4, M_SATD, r);
    return (int)r[0];
}
int64_t svt_av1_block_error_cuda(const int32_t *coeff, const int32_t *dqcoeff, intptr_t block_size, int64_t *ssz) {
    uint64_t r[2];
    reduce2(coeff, block_size, dqcoeff, block_size, (int)block_size, 1, 4, M_BLKERR, r);
    *ssz = (int64_t)r[1];
    return (int64_t)r[0];
}
uint32_t svt_nxm_sad_kernel_cuda(const uint8_t *src, uint32_t src_stride, const uint8_t *ref, uint32_t ref_stride, uint32_t height,
                                 uint32_t width) {
    if (!height || !width) return 0;
    uint64_t r[2];
    reduce2(src, src_stride, ref, ref_stride, width, height, 1, M_SAD8, r);
    return (uint32_t)r[0];
}
uint32_t svt_nxm_sad_kernel_sub_sampled_cuda(const uint8_t *src, uint32_t src_stride, const uint8_t *ref, uint32_t ref_stride,
                                             uint32_t height, uint32_t width) {
    uint64_t r[2]; // the C table entry is svt_nxm_sad_kernel_helper_c (aom_dsp_rtcd.c:372): a plain N x M SAD
    reduce2(src, src_stride, ref, ref_stride, width, height, 1, M_SAD8, r);
    return (uint32_t)r[0];
}
uint32_t sad_16b_kernel_cuda(uint16_t *src, uint32_t src_stride, uint16_t *ref, uint32_t ref_stride, uint32_t height, uint32_t width) {
    uint64_t r[2];
    reduce2(src, src_stride, ref, ref_stride, width, height, 2, M_SAD16, r);
    return (uint32_t)r[0];
}

#define SAD_MXN(W, H)                                                                                                   \
    uint32_t svt_aom_sad##W##x##H##_cuda(const uint8_t *src_ptr, int src_stride, const uint8_t *ref_ptr, int ref_stride) { \
        uint64_t r[2];                                                                                                  \
        reduce2(src_ptr, src_stride, ref_ptr, ref_stride, W, H, 1, M_SAD8, r);                                          \
        return (uint32_t)r[0];                                                                                          \
    }                                                                                                                   \
    void svt_aom_sad##W##x##H##x4d_cuda(const uint8_t *src_ptr, int src_stride, const uint8_t *const ref_ptr[],          \
                                        int ref_stride, uint32_t *sad_array) {                                          \
        for (int i = 0; i < 4; i++) sad_array[i] = svt_aom_sad##W##x##H##_cuda(src_ptr, src_stride, ref_ptr[i], ref_stride); \
    }
SAD_MXN(128, 128) SAD_MXN(128, 64) SAD_MXN(64, 128) SAD_MXN(64, 64) SAD_MXN(64, 32) SAD_MXN(64, 16) SAD_MXN(32, 64)
SAD_MXN(32, 32) SAD_MXN(32, 16) SAD_MXN(32, 8) SAD_MXN(16, 64) SAD_MXN(16, 32) SAD_MXN(16, 16) SAD_MXN(16, 8)
SAD_MXN(16, 4) SAD_MXN(8, 32) SAD_MXN(8, 16) SAD_MXN(8, 8) SAD_MXN(8, 4) SAD_MXN(4, 16) SAD_MXN(4, 8) SAD_MXN(4, 4)

// svt_aom_varianceWxH (aom_dsp_rtcd.h:488-530; C impl Encoder/C_DEFAULT/EbComputeVariance_C.c:14-61) and svt_aom_mse16x16
// (:249; Encoder/Codec/EbPsnr.c:84-89 — despite its name it also returns sse - sum^2 / 256): the reference's 32-bit wrap kept
static uint32_t variance_run(const void *a, int sa, const void *b, int sb, int w, int h, uint32_t *sse) {
    uint64_t r[2];
    reduce2(a, (size_t)sa, b, (size_t)sb, w, h, 1, M_VAR8, r);
    const int64_t sum = (int64_t)r[0];
    *sse = (uint32_t)r[1];
    return *sse - (uint32_t)((sum * sum) / (w * h));
}
#define VAR_WXH(W, H)                                                                                                          \
    unsigned int svt_aom_variance##W##x##H##_cuda(const uint8_t *a, int a_stride, const uint8_t *b, int b_stride, unsigned int *sse) { \
        return variance_run(a, a_stride, b, b_stride, W, H, sse);                                                        \
    }
VAR_WXH(4, 4) VAR_WXH(4, 8) VAR_WXH(4, 16) VAR_WXH(8, 4) VAR_WXH(8, 8) VAR_WXH(8, 16) VAR_WXH(8, 32) VAR_WXH(16, 4) VAR_WXH(16, 8)
VAR_WXH(16, 16) VAR_WXH(16, 32) VAR_WXH(16, 64) VAR_WXH(32, 8) VAR_WXH(32, 16) VAR_WXH(32, 32) VAR_WXH(32, 64) VAR_WXH(64, 16)
VAR_WXH(64, 32) VAR_WXH(64, 64) VAR_WXH(64, 128) VAR_WXH(128, 64) VAR_WXH(128, 128)
uint32_t svt_aom_mse16x16_cuda(const uint8_t *src_ptr, int32_t source_stride, const uint8_t *ref_ptr, int32_t recon_stride, uint32_t *sse) {
    return variance_run(src_ptr, source_stride, ref_ptr, recon_stride, 16, 16, sse);
}
}

// ---------------------------------------------------------------------------------------------------------------------
// svt_b200_me_downsample: the 1/4 and 1/16 HME planes on the device, padding included (SURVEY 8(f) rank 4).
// Replication padding = the shrink evaluated at the output coordinate clamped into the plane, so one launch per level
// writes the whole padded buffer: 4 output samples (one 32-bit store) per thread. Streaming, HBM/L2 bound and tiny
// (2.1 MB read, 0.8 MB written at 1080p).
// ---------------------------------------------------------------------------------------------------------------------
namespace {
struct ShrinkArgs {
    const uint8_t *in; // sample (0,0) of the input picture
    uint8_t *out;      // element (0,0) of the padded output buffer
    int in_stride, in_w, in_h;
    int out_stride, out_w, out_h, pad_x, pad_y;
    int step, filtered;
};
__global__ void __launch_bounds__(256) shrink_kernel(const __grid_constant__ ShrinkArgs a) {
    const int gx = (blockIdx.x * blockDim.x + threadIdx.x) * 4, gy = blockIdx.y; // in the padded buffer
    if (gx >= a.out_stride) return;
    const int cy = clampi(gy - a.pad_y, 0, a.out_h - 1);
    const int half = a.step >> 1;
    uint32_t word = 0;
#pragma unroll
    for (int e = 0; e < 4; e++) {
        const int cx = clampi(gx + e - a.pad_x, 0, a.out_w - 1);
        int v;
        if (a.filtered) { // downsample_2d: the 2x2 samples left/above position (half + step * c)
            const int y = min(half + a.step * cy, a.in_h - 1), x = min(half + a.step * cx, a.in_w - 1);
            const uint8_t *p = a.in + (size_t)(y - 1) * a.in_stride + x - 1;
            v = (__ldg(p) + __ldg(p + 1) + __ldg(p + a.in_stride) + __ldg(p + a.in_stride + 1) + 2) >> 2;
        } else { // decimation_2d
            v = __ldg(a.in + (size_t)min(a.step * cy, a.in_h - 1) * a.in_stride + min(a.step * cx, a.in_w - 1));
        }
        word |= (uint32_t)v << (8 * e);
    }
    uint8_t *o = a.out + (size_t)gy * a.out_stride + gx;
    if (gx + 4 <= a.out_stride && (((uintptr_t)o) & 3) == 0)
        *reinterpret_cast<uint32_t *>(o) = word;
    else
        for (int e = 0; e < 4 && gx + e < a.out_stride; e++) o[e] = (uint8_t)(word >> (8 * e));
}
int shrink_launch(const uint8_t *in, const SvtB200Plane &gi, uint8_t *out, const SvtB200Plane &go, int step, int filtered,
                  cudaStream_t st) {
    ShrinkArgs a;
    a.in = in + (size_t)gi.origin_y * gi.stride + gi.origin_x;
    a.out = out;
    a.in_stride = gi.stride, a.in_w = gi.width, a.in_h = gi.height;
    a.out_stride = go.stride, a.out_w = go.width, a.out_h = go.height, a.pad_x = go.origin_x, a.pad_y = go.origin_y;
    a.step = step, a.filtered = filtered;
    const int rows = go.height + 2 * go.origin_y;
    SVTB_LAUNCH(shrink_kernel, dim3((go.stride + 1023) / 1024, rows), 256, 0, st, a);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}
} // namespace

extern "C" int svt_b200_me_downsample(const SvtB200Plane *full, const SvtB200Plane *quarter, const SvtB200Plane *sixteenth,
                                      const SvtB200MePlanes *planes, int32_t filtered, void *stream) {
    if (!full || !quarter || !sixteenth || !planes || !planes->full || !planes->quarter || !planes->sixteenth || full->width < 8 ||
        full->height < 8 || quarter->width != full->width >> 1 || quarter->height != full->height >> 1 ||
        sixteenth->width != full->width >> 2 || sixteenth->height != full->height >> 2 ||
        quarter->stride < quarter->width + 2 * quarter->origin_x || sixteenth->stride < sixteenth->width + 2 * sixteenth->origin_x) {
        set_error("svt_b200_me_downsample: bad argument (quarter = full / 2, sixteenth = full / 4)");
        return SVT_B200_ERR_ARG;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = shrink_launch(planes->full, *full, (uint8_t *)planes->quarter, *quarter, 2, filtered != 0, st)) return rc;
    if (filtered) // sixteenth from the quarter plane just written
        return shrink_launch(planes->quarter, *quarter, (uint8_t *)planes->sixteenth, *sixteenth, 2, 1, st);
    return shrink_launch(planes->full, *full, (uint8_t *)planes->sixteenth, *sixteenth, 4, 0, st);
}
