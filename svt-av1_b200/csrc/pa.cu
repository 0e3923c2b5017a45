// pa.cu — picture-analysis block statistics on sm_90a (SURVEY.md 8(f) rank 4, the "variance" half).
//
// Replaces (reference: Source/Lib/Encoder/Codec/EbPictureAnalysisProcess.c):
//   compute_block_mean_compute_variance :1005-2575 with svt_compute_interm_var_four8x8 / svt_compute_sub_mean_8x8 /
//   svt_compute_mean_square_values_8x8 / compute_mean_8x8 (aom_dsp_rtcd.c:374-376, C :287-378),
//   compute_chroma_block_mean :493-1003, zero_out_chroma_block_mean :432-487 and the pic_avg_variance of
//   compute_picture_spatial_statistics :2929-2974 - for every SB of a picture in one launch.
// One CTA per 64x64 SB, 256 threads: four threads share an 8x8 block (one or two of its rows each), shuffle-reduce
// the sum and the sum of squares, the levels above are (a + b + c + d) >> 2 in shared memory.  The reference reads the
// SBs of the right / bottom edge from its padded input picture, which holds replicated edge samples
// (pad_picture_to_multiple_of_min_blk_size_dimensions :3164, generate_padding): reads are clamped to the picture.
#include "common.cuh"

using namespace svtb200;

namespace {

struct PaDev {
    const uint8_t *y, *cb, *cr;
    int stride_y, stride_c, width, height, sbw, full;
    uint8_t *y_mean, *cb_mean, *cr_mean;
    uint16_t *variance;
    unsigned long long *total;
};

__device__ __forceinline__ void level_up(const unsigned long long *in, int n_in, unsigned long long *out, int i) {
    const int n = n_in / 2, r = i / n, c = i - r * n;
    out[i] = (in[(2 * r) * n_in + 2 * c] + in[(2 * r) * n_in + 2 * c + 1] + in[(2 * r + 1) * n_in + 2 * c] + in[(2 * r + 1) * n_in + 2 * c + 1]) >> 2;
}

__global__ void __launch_bounds__(256) pa_sb_kernel(const PaDev d) {
    __shared__ unsigned long long m8[64], s8[64], m16[16], s16[16], m32[4], s32[4], m64[1], s64[1], c16[2][16], c32[2][4];
    const int sb = blockIdx.x, sx = sb % d.sbw, sy = sb / d.sbw, tid = threadIdx.x;
    const int b = tid >> 2, part = tid & 3, bx = sx * 64 + (b & 7) * 8, by = sy * 64 + (b >> 3) * 8;
    // rows of this thread: sub-sampled -> row 2 * part; full -> rows 2 * part and 2 * part + 1
    unsigned sum = 0, sq = 0;
    for (int k = 0; k < (d.full ? 2 : 1); k++) {
        const int yy = min(by + 2 * part + k, d.height - 1);
        const uint8_t *row = d.y + (size_t)yy * d.stride_y;
#pragma unroll
        for (int c = 0; c < 8; c++) {
            const unsigned v = row[min(bx + c, d.width - 1)];
            sum += v;
            sq += v * v;
        }
    }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1), sq += __shfl_xor_sync(0xffffffffu, sq, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2), sq += __shfl_xor_sync(0xffffffffu, sq, 2);
    if (part == 0) {
        m8[b] = d.full ? ((unsigned long long)sum << 8) / 64 : (unsigned long long)sum << 3;
        s8[b] = d.full ? ((unsigned long long)sq << 16) / 64 : (unsigned long long)sq << 11;
    }
    // chroma of complete SBs: 16 blocks of 8x8 per plane, threads 0..127 = (plane, block, part)
    const bool complete = sx * 64 + 64 <= d.width && sy * 64 + 64 <= d.height, chroma = d.cb_mean != nullptr;
    if (chroma && complete && tid < 128) {
        const int pl = tid >> 6, cbk = (tid >> 2) & 15;
        const uint8_t *p = (pl ? d.cr : d.cb) + (size_t)(sy * 32 + (cbk >> 2) * 8) * d.stride_c + sx * 32 + (cbk & 3) * 8;
        unsigned cs = 0;
        for (int k = 0; k < (d.full ? 2 : 1); k++)
#pragma unroll
            for (int c = 0; c < 8; c++) cs += p[(size_t)(2 * part + k) * d.stride_c + c];
        cs += __shfl_xor_sync(0xffffffffu, cs, 1);
        cs += __shfl_xor_sync(0xffffffffu, cs, 2);
        if (part == 0) c16[pl][cbk] = d.full ? ((unsigned long long)cs << 8) / 64 : (unsigned long long)cs << 3;
    }
    __syncthreads();
    if (tid < 16) level_up(m8, 8, m16, tid), level_up(s8, 8, s16, tid);
    if (tid >= 32 && tid < 40 && chroma && complete) level_up(c16[(tid - 32) >> 2], 4, c32[(tid - 32) >> 2], (tid - 32) & 3);
    __syncthreads();
    if (tid < 4) level_up(m16, 4, m32, tid), level_up(s16, 4, s32, tid);
    __syncthreads();
    if (tid == 0) level_up(m32, 2, m64, 0), level_up(s32, 2, s64, 0);
    __syncthreads();
    uint8_t *ym = d.y_mean + (size_t)sb * 85;
    uint16_t *vr = d.variance + (size_t)sb * 85;
    if (tid < 85) {
        unsigned long long m, s;
        if (tid == 0) m = m64[0], s = s64[0];
        else if (tid < 5) m = m32[tid - 1], s = s32[tid - 1];
        else if (tid < 21) m = m16[tid - 5], s = s16[tid - 5];
        else m = m8[tid - 21], s = s8[tid - 21];
        ym[tid] = (uint8_t)(m >> 8);
        const uint16_t v = (uint16_t)((s - m * m) >> 16);
        vr[tid] = v;
        if (tid == 0 && d.total) atomicAdd(d.total, (unsigned long long)v);
    }
    if (chroma && tid >= 128 && tid < 128 + 42) {
        const int pl = (tid - 128) / 21, i = (tid - 128) % 21;
        uint8_t *o = (pl ? d.cr_mean : d.cb_mean) + (size_t)sb * 21;
        unsigned long long m = 0;
        if (complete) {
            if (i == 0) m = (c32[pl][0] + c32[pl][1] + c32[pl][3] + c32[pl][3]) >> 2; // the reference's expression (:900-905)
            else if (i < 5) m = c32[pl][i - 1];
            else m = c16[pl][i - 5];
        }
        o[i] = (uint8_t)(m >> 8);
    }
}

__global__ void pa_finish_kernel(const unsigned long long *total, int n_sb, uint16_t *avg) { *avg = (uint16_t)(*total / (unsigned long long)n_sb); }

} // namespace

extern "C" {

int svt_b200_picture_mean_variance(const SvtB200Frame *pic, int32_t full_precision, uint8_t *y_mean, uint16_t *variance, uint8_t *cb_mean,
                                   uint8_t *cr_mean, uint16_t *pic_avg_variance, void *scratch, void *stream) {
    if (full_precision) {
        // BLOCK_MEAN_PREC_FULL cannot run in the reference either: its compute_mean_8x8 RTCD pointer is never assigned
        // (aom_dsp_rtcd.h:646, no SET_* line in aom_dsp_rtcd.c), so there is nothing to be bit-exact with
        set_error("svt_b200_picture_mean_variance: only the sub-sampled flavour (BLOCK_MEAN_PREC_SUB, the sequence default) exists");
        return SVT_B200_ERR_ARG;
    }
    if (!pic || !pic->y || pic->bit_depth != 8 || !y_mean || !variance || pic->width <= 0 || pic->height <= 0 || (!cb_mean != !cr_mean) ||
        (cb_mean && (!pic->cb || !pic->cr)) || (pic_avg_variance && !scratch)) {
        set_error("svt_b200_picture_mean_variance: bad argument (8-bit pictures: picture analysis runs on the 8-bit input)");
        return SVT_B200_ERR_ARG;
    }
    PaDev d;
    d.y = (const uint8_t *)pic->y, d.cb = (const uint8_t *)pic->cb, d.cr = (const uint8_t *)pic->cr;
    d.stride_y = pic->stride_y, d.stride_c = pic->stride_c, d.width = pic->width, d.height = pic->height;
    d.sbw = (pic->width + 63) / 64;
    const int n_sb = d.sbw * ((pic->height + 63) / 64);
    d.full = full_precision ? 1 : 0;
    d.y_mean = y_mean, d.variance = variance, d.cb_mean = cb_mean, d.cr_mean = cr_mean;
    d.total = pic_avg_variance ? (unsigned long long *)scratch : nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    if (d.total) SVTB_CUDA_TRY(cudaMemsetAsync(d.total, 0, 8, st));
    SVTB_LAUNCH(pa_sb_kernel, n_sb, 256, 0, st, d);
    if (d.total) SVTB_LAUNCH(pa_finish_kernel, 1, 1, 0, st, d.total, n_sb, pic_avg_variance);
    SVTB_CUDA_TRY(cudaGetLastError());
    return SVT_B200_OK;
}

// The same with HOST planes in / host arrays out (the form the encoder binding uses: integration/svt_cuda_backend.c
// svt_cuda_pa_statistics): the planes are packed into the calling thread's pinned staging, one upload, one download.
int svt_b200_picture_mean_variance_host(const uint8_t *y, int32_t stride_y, const uint8_t *cb, const uint8_t *cr, int32_t stride_c,
                                        int32_t width, int32_t height, uint8_t *y_mean, uint16_t *variance, uint8_t *cb_mean,
                                        uint8_t *cr_mean, uint16_t *pic_avg_variance) {
    if (!y || !y_mean || !variance || width <= 0 || height <= 0 || (!cb != !cr) || (!cb_mean != !cr_mean) || (cb_mean && !cb)) {
        set_error("svt_b200_picture_mean_variance_host: bad argument");
        return SVT_B200_ERR_ARG;
    }
    const int cw = (width + 1) >> 1, ch = (height + 1) >> 1, n_sb = ((width + 63) / 64) * ((height + 63) / 64);
    // y | cb | cr in; y mean | variance | cb mean | cr mean | (average variance, its 8-byte sum at 64) out
    Staging s({(size_t)width * height, (size_t)cw * ch, (size_t)cw * ch, (size_t)n_sb * 85, (size_t)n_sb * 170, (size_t)n_sb * 21,
               (size_t)n_sb * 21, 72});
    SVTB_CUDA_TRY(s.status());
    s.put_rows(0, y, stride_y, 1, width, height);
    if (cb_mean) {
        s.put_rows(1, cb, stride_c, 1, cw, ch);
        s.put_rows(2, cr, stride_c, 1, cw, ch);
    }
    SVTB_CUDA_TRY(s.upload(0, cb_mean ? 2 : 0));
    SvtB200Frame f = {s.d(0), cb_mean ? s.d(1) : nullptr, cb_mean ? s.d(2) : nullptr, width, cw, width, height, 8};
    const int rc = svt_b200_picture_mean_variance(&f, 0, s.d(3), s.d<uint16_t>(4), cb_mean ? s.d(5) : nullptr, cb_mean ? s.d(6) : nullptr,
                                                  s.d<uint16_t>(7), s.d(7) + 64, s.stream());
    if (rc) return rc;
    SVTB_CUDA_TRY(s.download(3, 7));
    memcpy(y_mean, s.h(3), (size_t)n_sb * 85);
    memcpy(variance, s.h(4), (size_t)n_sb * 170);
    if (cb_mean) {
        memcpy(cb_mean, s.h(5), (size_t)n_sb * 21);
        memcpy(cr_mean, s.h(6), (size_t)n_sb * 21);
    }
    if (pic_avg_variance) memcpy(pic_avg_variance, s.h(7), 2);
    return SVT_B200_OK;
}
}
