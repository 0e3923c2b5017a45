/*
 * svt_av1_b200.h — C ABI of the H100 (sm_90a) hot-path library `libsvtav1_b200.so`.
 *
 * Scope (SURVEY.md §8): open-loop motion estimation (HME + full-pel SAD search), residual +
 * forward/inverse transform + quantisation, and the in-loop filters (deblock, CDEF, restoration)
 * of SVT-AV1 v0.8.6.  Two families of entry points:
 *
 *  (1) `*_cuda` drop-ins with EXACTLY the signature of the reference's RTCD function pointers
 *      (Source/Lib/Encoder/Codec/aom_dsp_rtcd.h, Source/Lib/Common/Codec/common_dsp_rtcd.h).
 *      They take HOST pointers, stage through a thread-local pinned buffer + stream, run the sm_90a
 *      kernel and copy the result back.  They exist for API fidelity and parity tests; a launch per
 *      8x8 block can never be fast.  The installer that assigns them to the reference's pointers is compiled next
 *      to the reference's headers (oracle/rtcd_install.c: svt_cuda_install_rtcd(), 225 pointers, type-checked at compile
 *      time; INTEGRATION.md section 1 shows the setup_rtcd_internal hook).
 *
 *  (2) `svt_b200_*` picture-level ("batched") entries, which are where throughput comes from.  They
 *      replace the L2 segment loops of the reference (motion_estimation_kernel, EncDec final pass,
 *      dlf_kernel, cdef_kernel, rest_kernel).  All pointers are DEVICE pointers unless the name ends
 *      in `_host`; `stream` is a `cudaStream_t` passed as `void*` (NULL = default stream).
 *
 *  (3) `svt_b200_engine_*`: the picture engine - HOST pictures in, host results out, synchronous and re-entrant -
 *      which is what the reference's process loops call (integration/svt_cuda_backend.c).
 *
 * No torch / C++ types cross this boundary.  Every function returns 0 on success or a negative
 * SvtB200Status; there is NO CPU fallback — a missing GPU is an error.
 */
#ifndef SVT_AV1_B200_H
#define SVT_AV1_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SVT_B200_API __attribute__((visibility("default")))

typedef enum SvtB200Status {
    SVT_B200_OK = 0,
    SVT_B200_ERR_CUDA = -1, /* a CUDA runtime call failed (message via svt_b200_last_error) */
    SVT_B200_ERR_ARG = -2, /* bad argument */
    SVT_B200_ERR_UNSUPPORTED = -3 /* configuration outside what the kernels implement */
} SvtB200Status;

/* ---- library / device management -------------------------------------------------------------- */
SVT_B200_API int svt_b200_version(void);
SVT_B200_API int svt_b200_device_count(void); /* <0 on error, 0 if no GPU */
SVT_B200_API int svt_b200_set_device(int device);
SVT_B200_API const char *svt_b200_last_error(void); /* thread-local text of the last failure */
/* Number of kernel launches issued by this library since load (all threads); bench.py reports it. */
SVT_B200_API uint64_t svt_b200_launch_count(void);
SVT_B200_API void *svt_b200_malloc(size_t bytes); /* cudaMalloc */
SVT_B200_API void svt_b200_free(void *dptr);
SVT_B200_API void *svt_b200_malloc_host(size_t bytes); /* pinned host memory */
SVT_B200_API void svt_b200_free_host(void *hptr);
SVT_B200_API int svt_b200_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream);
SVT_B200_API int svt_b200_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream);
SVT_B200_API int svt_b200_stream_sync(void *stream);

/* =============================================================================================== */
/* (1) RTCD drop-ins: motion estimation                                                            */
/* =============================================================================================== */

/* replaces svt_sad_loop_kernel  (aom_dsp_rtcd.h:597; C impl Encoder/C_DEFAULT/EbComputeSAD_C.c:57) */
SVT_B200_API void svt_sad_loop_kernel_cuda(uint8_t *src, uint32_t src_stride, uint8_t *ref,
                                           uint32_t ref_stride, uint32_t block_height,
                                           uint32_t block_width, uint64_t *best_sad,
                                           int16_t *x_search_center, int16_t *y_search_center,
                                           uint32_t src_stride_raw, int16_t search_area_width,
                                           int16_t search_area_height);

/* replaces svt_ext_all_sad_calculation_8x8_16x16 (aom_dsp_rtcd.h:640; EbMotionEstimation.c:362) */
SVT_B200_API void svt_ext_all_sad_calculation_8x8_16x16_cuda(
    uint8_t *src, uint32_t src_stride, uint8_t *ref, uint32_t ref_stride, uint32_t mv,
    uint32_t *p_best_sad_8x8, uint32_t *p_best_sad_16x16, uint32_t *p_best_mv8x8,
    uint32_t *p_best_mv16x16, uint32_t p_eight_sad16x16[16][8], uint32_t p_eight_sad8x8[64][8],
    uint8_t sub_sad);

/* replaces svt_ext_eight_sad_calculation_32x32_64x64 (aom_dsp_rtcd.h:641; EbMotionEstimation.c:396) */
SVT_B200_API void svt_ext_eight_sad_calculation_32x32_64x64_cuda(
    uint32_t p_sad16x16[16][8], uint32_t *p_best_sad_32x32, uint32_t *p_best_sad_64x64,
    uint32_t *p_best_mv32x32, uint32_t *p_best_mv64x64, uint32_t mv, uint32_t p_sad32x32[4][8]);

/* replaces svt_ext_sad_calculation_8x8_16x16 (aom_dsp_rtcd.h:630; EbMotionEstimation.c:122) */
SVT_B200_API void svt_ext_sad_calculation_8x8_16x16_cuda(
    uint8_t *src, uint32_t src_stride, uint8_t *ref, uint32_t ref_stride, uint32_t *p_best_sad_8x8,
    uint32_t *p_best_sad_16x16, uint32_t *p_best_mv8x8, uint32_t *p_best_mv16x16, uint32_t mv,
    uint32_t *p_sad16x16, uint32_t *p_sad8x8, uint8_t sub_sad);

/* replaces svt_ext_sad_calculation_32x32_64x64 (aom_dsp_rtcd.h:636; EbMotionEstimation.c:191) */
SVT_B200_API void svt_ext_sad_calculation_32x32_64x64_cuda(
    uint32_t *p_sad16x16, uint32_t *p_best_sad_32x32, uint32_t *p_best_sad_64x64,
    uint32_t *p_best_mv32x32, uint32_t *p_best_mv64x64, uint32_t mv, uint32_t *p_sad32x32);

/* replaces svt_nxm_sad_kernel (aom_dsp_rtcd.h:644; Encoder/C_DEFAULT/EbComputeSAD_C.c helper) */
SVT_B200_API uint32_t svt_nxm_sad_kernel_cuda(const uint8_t *src, uint32_t src_stride,
                                              const uint8_t *ref, uint32_t ref_stride,
                                              uint32_t height, uint32_t width);

/* replaces svt_initialize_buffer_32bits (aom_dsp_rtcd.h:642): fills count128*4+count32 words */
SVT_B200_API void svt_initialize_buffer_32bits_cuda(uint32_t *pointer, uint32_t count128,
                                                    uint32_t count32, uint32_t value);

/* =============================================================================================== */
/* (2) Picture-level open-loop ME: replaces the SB loop of motion_estimation_kernel               */
/*     (EbMotionEstimationProcess.c:831-965) -> motion_estimate_sb (EbMotionEstimation.c:2912).    */
/* =============================================================================================== */

#define SVT_B200_ME_MAX_REFS 4 /* REF_LIST_MAX_DEPTH (EbDefinitions.h) */
#define SVT_B200_ME_LISTS 2 /* MAX_NUM_OF_REF_PIC_LIST */
#define SVT_B200_ME_PU 85 /* SQUARE_PU_COUNT: 1x64^2 + 4x32^2 + 16x16^2 + 64x8^2 */
#define SVT_B200_ME_MAX_MV 7 /* MAX_PA_ME_MV   (EbMotionEstimationLcuResults.h:23) */
#define SVT_B200_ME_MAX_CAND 23 /* MAX_PA_ME_CAND (EbMotionEstimationLcuResults.h:24) */

/* Geometry of one padded 8-bit luma plane (EbPictureBufferDesc: stride_y, origin_x/y, width/height). */
typedef struct SvtB200Plane {
    int32_t stride;
    int32_t origin_x;
    int32_t origin_y;
    int32_t width;
    int32_t height;
} SvtB200Plane;

/* Mirror of the MeContext search parameters (EbMotionEstimationContext.h:325-400) that
 * signal_derivation_me_kernel_oq / set_me_hme_params_oq (EbMotionEstimationProcess.c:113-420) fill,
 * plus the per-picture fields motion_estimation_kernel copies from the PCS (:914-940). */
typedef struct SvtB200MeParams {
    /* geometry (source and every reference share it) */
    SvtB200Plane full; /* input_padded_picture_ptr */
    SvtB200Plane quarter; /* quarter_{decimated,filtered}_picture_ptr */
    SvtB200Plane sixteenth; /* sixteenth_{decimated,filtered}_picture_ptr */
    /* reference structure */
    int32_t num_lists; /* num_of_list_to_search + 1: 1 (P) or 2 (B) */
    int32_t num_refs[SVT_B200_ME_LISTS]; /* num_of_ref_pic_to_search[] (<=4, list1 <=3) */
    int32_t ref_dist[SVT_B200_ME_LISTS][SVT_B200_ME_MAX_REFS]; /* |poc - ref poc| (get_me_reference) */
    int32_t temporal_layer_index;
    int32_t is_used_as_reference_flag;
    /* HME */
    int32_t enable_hme_flag, enable_hme_level0_flag, enable_hme_level1_flag, enable_hme_level2_flag;
    int32_t hme_search_method; /* 0 = FULL_SAD_SEARCH, 1 = SUB_SAD_SEARCH */
    int32_t me_search_method; /* idem for the full-pel search */
    int32_t number_hme_search_region_in_width, number_hme_search_region_in_height; /* <=2 each */
    int32_t hme_level0_total_search_area_width, hme_level0_total_search_area_height;
    int32_t hme_level0_max_total_search_area_width, hme_level0_max_total_search_area_height;
    int32_t hme_level0_search_area_in_width_array[2], hme_level0_search_area_in_height_array[2];
    int32_t hme_level0_max_search_area_in_width_array[2], hme_level0_max_search_area_in_height_array[2];
    int32_t hme_level1_search_area_in_width_array[2], hme_level1_search_area_in_height_array[2];
    int32_t hme_level2_search_area_in_width_array[2], hme_level2_search_area_in_height_array[2];
    /* full-pel ME */
    int32_t search_area_width, search_area_height, max_me_search_width, max_me_search_height;
    /* pruning / search-region adjustment (MeHmeRefPruneCtrls, MeSrCtrls) */
    int32_t enable_me_hme_ref_pruning;
    int32_t prune_ref_if_hme_sad_dev_bigger_than_th; /* 0xFFFF = off */
    int32_t prune_ref_if_me_sad_dev_bigger_than_th; /* 0xFFFF = off */
    int32_t enable_me_sr_adjustment;
    int32_t reduce_me_sr_based_on_mv_length_th, stationary_hme_sad_abs_th, stationary_me_sr_divisor;
    int32_t reduce_me_sr_based_on_hme_sad_abs_th, me_sr_divisor_for_low_hme_sad;
    /* result shaping */
    int32_t max_number_of_pus_per_sb; /* pcs->max_number_of_pus_per_sb: 85 (or 21 / 5) */
    int32_t rc_dist_from_8x8; /* 1 if input_resolution <= 480p (EbMotionEstimation.c:3025) */
} SvtB200MeParams;

/* Device-side planes of one picture: the padded full-res luma and its two decimations. Pointers
 * address element (0,0) of the PADDED buffer (EbPictureBufferDesc::buffer_y). */
typedef struct SvtB200MePlanes {
    const uint8_t *full;
    const uint8_t *quarter;
    const uint8_t *sixteenth;
} SvtB200MePlanes;

/* Per-picture outputs, all device pointers, n_sb = ceil(w/64)*ceil(h/64) superblocks in raster order.
 *  best_sad / best_mv : [n_sb][2][4][85] — MeContext::p_sb_best_sad / p_sb_best_mv after
 *                       integer_search_sb; index order is the reference's internal PU order
 *                       (64x64, 4x 32x32, 16x 16x16 z-order, 64x 8x8 z-order).  MVs are packed
 *                       (y<<16)|(x&0xffff) in quarter-pel units, as the reference stores them.
 *  hme                : [n_sb][2][4] {int16 sc_x, int16 sc_y, uint32 do_ref, uint64 hme_sad}
 *  me_mv              : [n_sb][85*7] {int16 x, int16 y}          (MeSbResults::me_mv_array)
 *  me_cand            : [n_sb][85*23] uint8 bit-field             (MeSbResults::me_candidate_array;
 *                       bits 0-1 direction, 2-3 ref_idx_l0, 4-5 ref_idx_l1, 6 ref0_list, 7 ref1_list;
 *                       the index of the list a uni-pred candidate does NOT use is written as 0 —
 *                       the reference leaves a stale value there that nothing reads)
 *  total_cand         : [n_sb][85] uint8                          (total_me_candidate_index)
 *  rc_me_distortion   : [n_sb] uint32                             (pcs->rc_me_distortion) */
typedef struct SvtB200HmeResult {
    int16_t sc_x, sc_y;
    uint32_t do_ref;
    uint64_t hme_sad;
} SvtB200HmeResult;

typedef struct SvtB200MeOutputs {
    uint32_t *best_sad;
    uint32_t *best_mv;
    SvtB200HmeResult *hme;
    int16_t *me_mv;
    uint8_t *me_cand;
    uint8_t *total_cand;
    uint32_t *rc_me_distortion;
} SvtB200MeOutputs;

/* Bytes of device scratch svt_b200_me_picture needs for a picture of this geometry. */
SVT_B200_API size_t svt_b200_me_scratch_bytes(const SvtB200MeParams *p);

/* Open-loop ME of one whole picture against up to 2x4 references, all resident in HBM.
 * refs[list][idx] are only read for idx < num_refs[list]. Asynchronous on `stream`. */
SVT_B200_API int svt_b200_me_picture(const SvtB200MeParams *p, const SvtB200MePlanes *src,
                                     const SvtB200MePlanes refs[SVT_B200_ME_LISTS][SVT_B200_ME_MAX_REFS],
                                     const SvtB200MeOutputs *out, void *scratch, void *stream);

/* The 1/4 and 1/16 planes of one picture from its full-resolution luma, padding included (SURVEY 8(f) rank 4):
 * filtered != 0 replaces downsample_filtering_input_picture[_ime] (EbPictureAnalysisProcess.c:3606-3720; downsample_2d
 * :223-256: 2x2 average, quarter from full, sixteenth from quarter — every preset <= M9), filtered == 0
 * downsample_decimation_input_picture[_ime] (:3312-3360; decimation_2d :193-216: top-left sample, both from full), each
 * followed by generate_padding (EbMcp.c:112-164).  planes: DEVICE buffers, `full` read (its padding is not needed),
 * `quarter` / `sixteenth` written in full.  With this the HME planes need not be uploaded.  Requires
 * quarter = full / 2 and sixteenth = full / 4 in both dimensions (rounded down).  Asynchronous on `stream`. */
SVT_B200_API int svt_b200_me_downsample(const SvtB200Plane *full, const SvtB200Plane *quarter, const SvtB200Plane *sixteenth,
                                        const SvtB200MePlanes *planes, int32_t filtered, void *stream);

/* =============================================================================================== */
/* Pictures for the EncDec / in-loop-filter entries                                                */
/* =============================================================================================== */

/* A 4:2:0 picture in HBM (or host memory for the *_host variants). Pointers address sample (0,0) of
 * each plane (i.e. EbPictureBufferDesc::buffer_* + origin offsets); strides are in SAMPLES.
 * bit_depth 8 -> uint8_t samples, 10 -> uint16_t samples (the reference's is_16bit pipeline). */
typedef struct SvtB200Frame {
    void *y, *cb, *cr;
    int32_t stride_y, stride_c;
    int32_t width, height; /* luma size; chroma is (width+1)>>1 x (height+1)>>1 */
    int32_t bit_depth;
} SvtB200Frame;

/* =============================================================================================== */
/* CDEF                                                                                            */
/* =============================================================================================== */

/* replaces svt_cdef_find_dir (common_dsp_rtcd.h:1032; C impl Common/Codec/EbCdef.c:132-197) */
SVT_B200_API int32_t svt_cdef_find_dir_cuda(const uint16_t *img, int32_t stride, int32_t *var,
                                            int32_t coeff_shift);
/* replaces svt_cdef_filter_block (common_dsp_rtcd.h:1034; EbCdef.c:202-257). `in` points inside a
 * CDEF_BSTRIDE(144)-strided uint16 tile with >=2 valid rows/columns around the block; bsize is the
 * reference's BlockSize enum value (BLOCK_4X4=0, BLOCK_4X8=1, BLOCK_8X4=2, BLOCK_8X8=3). */
SVT_B200_API void svt_cdef_filter_block_cuda(uint8_t *dst8, uint16_t *dst16, int32_t dstride,
                                             const uint16_t *in, int32_t pri_strength,
                                             int32_t sec_strength, int32_t dir, int32_t pri_damping,
                                             int32_t sec_damping, int32_t bsize, int32_t coeff_shift);

/* replace svt_copy_rect8_8bit_to_16bit (common_dsp_rtcd.h:1036-1037; EbCdef.c:118-123): widening rectangle copy */
SVT_B200_API void svt_copy_rect8_8bit_to_16bit_cuda(uint16_t *dst, int32_t dstride, const uint8_t *src, int32_t sstride,
                                                    int32_t v, int32_t h);
/* replace svt_compute_cdef_dist_16bit / _8bit (aom_dsp_rtcd.h:67-70; compute_cdef_dist_c / _8bit_c, EbEncCdef.c:134-220):
 * distortion of the filtered blocks of one filter block against the packed source blocks (luma 8x8: the perceptual
 * double-precision measure; otherwise SSE), >> 2*coeff_shift.  dlist: the reference's CdefList array {by, bx, skip}.
 * bsize: BlockSize (BLOCK_4X4 0, 4X8 1, 8X4 2, 8X8 3). */
SVT_B200_API uint64_t svt_compute_cdef_dist_16bit_cuda(const uint16_t *dst, int32_t dstride, const uint16_t *src,
                                                       const void *dlist, int32_t cdef_count, int32_t bsize,
                                                       int32_t coeff_shift, int32_t pli);
SVT_B200_API uint64_t svt_compute_cdef_dist_8bit_cuda(const uint8_t *dst8, int32_t dstride, const uint8_t *src8,
                                                      const void *dlist, int32_t cdef_count, int32_t bsize,
                                                      int32_t coeff_shift, int32_t pli);


#define SVT_B200_CDEF_MAX_STRENGTHS 64 /* TOTAL_STRENGTHS (EbDefinitions.h:1675-1690) */

/* Strength search of cdef_kernel: replaces cdef_seg_search / cdef_seg_search16bit
 * (Encoder/Codec/EbCdefProcess.c:80-277, 281-475) for a whole picture. */
typedef struct SvtB200CdefSearchParams {
    int32_t mi_rows, mi_cols; /* Av1Common::mi_rows / mi_cols (4x4 units) */
    int32_t pri_damping; /* 3 + (base_q_idx >> 6); sec_damping is the same */
    int32_t n_strengths; /* nb_cdef_strengths[pick_method] */
    /* per strength index gi: (threshold, sec_strength + (sec_strength == 3)) exactly as passed to
     * svt_cdef_filter_fb (EbCdefProcess.c:236-252); fill with svt_b200_cdef_strength_table(). */
    int32_t pri_strength[SVT_B200_CDEF_MAX_STRENGTHS];
    int32_t sec_strength[SVT_B200_CDEF_MAX_STRENGTHS];
} SvtB200CdefSearchParams;

/* Host helper mirroring get_cdef_filter_strengths (EbDefinitions.h:1696-1722).
 * pick_method: 0 full(64), 1 lvl1(32), 2 lvl2(20), 3 lvl3(10 — preset 8). Returns n_strengths. */
SVT_B200_API int svt_b200_cdef_strength_table(int pick_method, SvtB200CdefSearchParams *p);

/* recon  : deblocked reconstruction (pcs->src[] in the reference), read only
 * source : the input picture (pcs->ref_coeff[])
 * skip8  : device uint8 [ceil(mi_rows/2)][skip_stride]: 1 where every 4x4 of the 8x8 is `skip`
 *          (is_8x8_block_skip, EbEncCdef.c:238); this flattens the ModeInfo grid
 * mse    : device uint64 [2][nvfb*nhfb][64] = pcs->mse_seg (plane 0 = Y, 1 = Cb+Cr); entries of filter
 *          blocks the reference skips (all-skip) are written as 0. */
SVT_B200_API int svt_b200_cdef_search(const SvtB200CdefSearchParams *p, const SvtB200Frame *recon,
                                      const SvtB200Frame *source, const uint8_t *skip8,
                                      int32_t skip_stride, uint64_t *mse, void *stream);

/* Frame apply: replaces svt_av1_cdef_frame / av1_cdef_frame16bit (EbEncCdef.c:292-660, 663-1030).
 * fb_strength_idx : device int8 [nvfb*nhfb], mbmi.cdef_strength of each 64x64 filter block (-1: skip)
 * y_strength/uv_strength : frm_hdr->cdef_params.cdef_y_strength / cdef_uv_strength (host arrays of 8)
 * Reads `recon` (pre-CDEF) and writes `out` (may not alias recon: the GPU version is out-of-place,
 * which is what the reference's line/column buffers emulate). Blocks that are not filtered are copied. */
typedef struct SvtB200CdefApplyParams {
    int32_t mi_rows, mi_cols;
    int32_t damping; /* frm_hdr->cdef_params.cdef_damping */
    int32_t y_strength[8], uv_strength[8];
} SvtB200CdefApplyParams;
SVT_B200_API int svt_b200_cdef_apply(const SvtB200CdefApplyParams *p, const SvtB200Frame *recon,
                                     const SvtB200Frame *out, const uint8_t *skip8, int32_t skip_stride,
                                     const int8_t *fb_strength_idx, void *stream);

/* The strength decision of the CDEF search on the device: replaces finish_cdef_search (EbEncCdef.c:1167-1340;
 * joint_strength_search_dual :1136, svt_search_one_dual_c :1070) between svt_b200_cdef_search and svt_b200_cdef_apply, so
 * the picture does not visit the host in between.  All integer (uint64 sums, RDCOST with the picture's lambda): exact.
 * lambda: full_lambda of av1_lambda_assignment_function_table[pred_structure](pcs, ..., bit_depth, base_q_idx, EB_FALSE)
 * (:1209); filter_strength[gi]: what STORE_CDEF_FILTER_STRENGTH writes for index gi (:1165; pri * CDEF_SEC_STRENGTHS + sec of
 * get_cdef_filter_strengths, the identity for the full 64-entry table) - svt_b200_cdef_decide_table() fills it.
 * mse / skip8: DEVICE, as svt_b200_cdef_search wrote / read them.  out: DEVICE SvtB200CdefDecision; fb_strength_idx: DEVICE
 * int8 [nvfb*nhfb] (mbmi.cdef_strength of each filter block, -1 for the all-skip ones): the input of
 * svt_b200_cdef_apply_dev.  scratch: DEVICE, >= (16 + 16 * n_strengths) bytes per filter block + 64. */
typedef struct SvtB200CdefDecideParams {
    int32_t mi_rows, mi_cols;
    int32_t n_strengths; /* nb_cdef_strengths[pick_method] (start_gi = 0) */
    int32_t reserved;
    uint64_t lambda;
    int32_t filter_strength[SVT_B200_CDEF_MAX_STRENGTHS];
} SvtB200CdefDecideParams;
typedef struct SvtB200CdefDecision {
    int32_t cdef_bits;                      /* frm_hdr->cdef_params.cdef_bits */
    int32_t nb_cdef_strengths;              /* ppcs->nb_cdef_strengths = 1 << cdef_bits */
    int32_t y_strength[8], uv_strength[8];  /* frm_hdr->cdef_params.cdef_y_strength / cdef_uv_strength (after STORE_...) */
    int32_t y_index[8], uv_index[8];        /* the same as indices into the searched strength table */
    int32_t sb_count;                       /* filter blocks that took part */
    int32_t reserved;
} SvtB200CdefDecision;
SVT_B200_API int svt_b200_cdef_decide_table(int pick_method, SvtB200CdefDecideParams *p); /* n_strengths + filter_strength */
SVT_B200_API int svt_b200_cdef_decide(const SvtB200CdefDecideParams *p, const uint64_t *mse, const uint8_t *skip8,
                                      int32_t skip_stride, SvtB200CdefDecision *out, int8_t *fb_strength_idx, void *scratch,
                                      void *stream);
/* svt_b200_cdef_apply with the strengths taken from a DEVICE SvtB200CdefDecision (the output of svt_b200_cdef_decide) */
SVT_B200_API int svt_b200_cdef_apply_dev(int32_t mi_rows, int32_t mi_cols, int32_t damping, const SvtB200CdefDecision *decision,
                                         const SvtB200Frame *recon, const SvtB200Frame *out, const uint8_t *skip8,
                                         int32_t skip_stride, const int8_t *fb_strength_idx, void *stream);

/* =============================================================================================== */
/* Residual / forward + inverse transform / quantisation                                           */
/* =============================================================================================== */

/* replaces svt_residual_kernel8bit / 16bit (common_dsp_rtcd.h:169,180; EbPictureOperators.c:130,106) */
SVT_B200_API void svt_residual_kernel8bit_cuda(uint8_t *input, uint32_t input_stride, uint8_t *pred,
                                               uint32_t pred_stride, int16_t *residual,
                                               uint32_t residual_stride, uint32_t area_width,
                                               uint32_t area_height);
SVT_B200_API void svt_residual_kernel16bit_cuda(uint16_t *input, uint32_t input_stride, uint16_t *pred,
                                                uint32_t pred_stride, int16_t *residual,
                                                uint32_t residual_stride, uint32_t area_width,
                                                uint32_t area_height);

/* replace svt_av1_fwd_txfm2d_{WxH} (aom_dsp_rtcd.h:105-216; C impl EbTransforms.c:2301-3053).
 * tx_type is the reference's TxType (a 1-byte packed enum, DCT_DCT=0 ... H_FLIPADST=15): uint8_t keeps the by-value
 * argument ABI identical; likewise TxSize below. */
#define SVT_B200_DECL_FWD(W, H)                                                                      \
    SVT_B200_API void svt_av1_fwd_txfm2d_##W##x##H##_cuda(int16_t *input, int32_t *output,           \
                                                          uint32_t input_stride, uint8_t tx_type,    \
                                                          uint8_t bit_depth);                        \
    /* partial-frequency shapes svt_av1_fwd_txfm2d_WxH_N2 / _N4 (aom_dsp_rtcd.h:150-216) */           \
    SVT_B200_API void svt_av1_fwd_txfm2d_##W##x##H##_N2_cuda(int16_t *input, int32_t *output,        \
                                                             uint32_t input_stride, uint8_t tx_type, \
                                                             uint8_t bit_depth);                     \
    SVT_B200_API void svt_av1_fwd_txfm2d_##W##x##H##_N4_cuda(int16_t *input, int32_t *output,        \
                                                             uint32_t input_stride, uint8_t tx_type, \
                                                             uint8_t bit_depth);
SVT_B200_DECL_FWD(4, 4) SVT_B200_DECL_FWD(8, 8) SVT_B200_DECL_FWD(16, 16) SVT_B200_DECL_FWD(32, 32)
SVT_B200_DECL_FWD(64, 64) SVT_B200_DECL_FWD(4, 8) SVT_B200_DECL_FWD(8, 4) SVT_B200_DECL_FWD(8, 16)
SVT_B200_DECL_FWD(16, 8) SVT_B200_DECL_FWD(16, 32) SVT_B200_DECL_FWD(32, 16) SVT_B200_DECL_FWD(32, 64)
SVT_B200_DECL_FWD(64, 32) SVT_B200_DECL_FWD(4, 16) SVT_B200_DECL_FWD(16, 4) SVT_B200_DECL_FWD(8, 32)
SVT_B200_DECL_FWD(32, 8) SVT_B200_DECL_FWD(16, 64) SVT_B200_DECL_FWD(64, 16)

/* replace svt_handle_transform64x64 / 64x32 / 32x64 / 64x16 / 16x64 (aom_dsp_rtcd.h:222-245;
 * EbTransforms.c:2763-2931): in place on the w x h coefficient array, returns the dropped energy */
SVT_B200_API uint64_t svt_handle_transform64x64_cuda(int32_t *output);
SVT_B200_API uint64_t svt_handle_transform64x32_cuda(int32_t *output);
SVT_B200_API uint64_t svt_handle_transform32x64_cuda(int32_t *output);
SVT_B200_API uint64_t svt_handle_transform64x16_cuda(int32_t *output);
SVT_B200_API uint64_t svt_handle_transform16x64_cuda(int32_t *output);
SVT_B200_API uint64_t svt_b200_handle_transform64(int32_t *output, int tx_size);

/* replace svt_av1_inv_txfm2d_add_{WxH} (common_dsp_rtcd.h:105-156; EbInvTransforms.c:2455-2752) */
#define SVT_B200_DECL_INV_SQ(W)                                                                        \
    SVT_B200_API void svt_av1_inv_txfm2d_add_##W##x##W##_cuda(                                         \
        const int32_t *input, uint16_t *output_r, int32_t stride_r, uint16_t *output_w, int32_t stride_w, \
        uint8_t tx_type, int32_t bd);
#define SVT_B200_DECL_INV_RECT(W, H)                                                                   \
    SVT_B200_API void svt_av1_inv_txfm2d_add_##W##x##H##_cuda(                                         \
        const int32_t *input, uint16_t *output_r, int32_t stride_r, uint16_t *output_w, int32_t stride_w, \
        uint8_t tx_type, uint8_t tx_size, int32_t eob, int32_t bd);
#define SVT_B200_DECL_INV_RECT_NOEOB(W, H)                                                             \
    SVT_B200_API void svt_av1_inv_txfm2d_add_##W##x##H##_cuda(                                         \
        const int32_t *input, uint16_t *output_r, int32_t stride_r, uint16_t *output_w, int32_t stride_w, \
        uint8_t tx_type, uint8_t tx_size, int32_t bd);
SVT_B200_DECL_INV_SQ(4) SVT_B200_DECL_INV_SQ(8) SVT_B200_DECL_INV_SQ(16) SVT_B200_DECL_INV_SQ(32)
SVT_B200_DECL_INV_SQ(64) SVT_B200_DECL_INV_RECT_NOEOB(4, 8) SVT_B200_DECL_INV_RECT_NOEOB(8, 4)
SVT_B200_DECL_INV_RECT(8, 16) SVT_B200_DECL_INV_RECT(16, 8) SVT_B200_DECL_INV_RECT(16, 32)
SVT_B200_DECL_INV_RECT(32, 16) SVT_B200_DECL_INV_RECT(32, 64) SVT_B200_DECL_INV_RECT(64, 32)
SVT_B200_DECL_INV_RECT_NOEOB(4, 16) SVT_B200_DECL_INV_RECT_NOEOB(16, 4) SVT_B200_DECL_INV_RECT(8, 32)
SVT_B200_DECL_INV_RECT(32, 8) SVT_B200_DECL_INV_RECT(16, 64) SVT_B200_DECL_INV_RECT(64, 16)

/* replace svt_av1_inv_txfm_add (common_dsp_rtcd.h:155-156; EbInvTransforms.c:3302-3323): the 8-bit entry — prediction
 * and reconstruction are uint8 planes, txfm_param is the reference's TxfmParam (tx_type, tx_size, bd, eob are read; lossless
 * is not supported). */
SVT_B200_API void svt_av1_inv_txfm_add_cuda(const int32_t *dqcoeff, uint8_t *dst_r, int32_t stride_r, uint8_t *dst_w,
                                            int32_t stride_w, const void *txfm_param);

/* replace svt_aom_quantize_b / svt_aom_highbd_quantize_b (aom_dsp_rtcd.h:252,254; EbFullLoop.c:37,171) and
 * svt_av1_quantize_fp[_32x32/_64x64] / svt_av1_highbd_quantize_fp (aom_dsp_rtcd.h:256-262; :314-600).
 * QmVal is uint8_t in the reference. */
SVT_B200_API void svt_aom_quantize_b_cuda(const int32_t *coeff_ptr, intptr_t n_coeffs, const int16_t *zbin_ptr,
                                          const int16_t *round_ptr, const int16_t *quant_ptr,
                                          const int16_t *quant_shift_ptr, int32_t *qcoeff_ptr,
                                          int32_t *dqcoeff_ptr, const int16_t *dequant_ptr, uint16_t *eob_ptr,
                                          const int16_t *scan, const int16_t *iscan, const uint8_t *qm_ptr,
                                          const uint8_t *iqm_ptr, const int32_t log_scale);
SVT_B200_API void svt_aom_highbd_quantize_b_cuda(const int32_t *coeff_ptr, intptr_t n_coeffs,
                                                 const int16_t *zbin_ptr, const int16_t *round_ptr,
                                                 const int16_t *quant_ptr, const int16_t *quant_shift_ptr,
                                                 int32_t *qcoeff_ptr, int32_t *dqcoeff_ptr,
                                                 const int16_t *dequant_ptr, uint16_t *eob_ptr,
                                                 const int16_t *scan, const int16_t *iscan,
                                                 const uint8_t *qm_ptr, const uint8_t *iqm_ptr,
                                                 const int32_t log_scale);
#define SVT_B200_DECL_QFP(NAME)                                                                          \
    SVT_B200_API void NAME(const int32_t *coeff_ptr, intptr_t n_coeffs, const int16_t *zbin_ptr,         \
                           const int16_t *round_ptr, const int16_t *quant_ptr,                           \
                           const int16_t *quant_shift_ptr, int32_t *qcoeff_ptr, int32_t *dqcoeff_ptr,    \
                           const int16_t *dequant_ptr, uint16_t *eob_ptr, const int16_t *scan,           \
                           const int16_t *iscan);
SVT_B200_DECL_QFP(svt_av1_quantize_fp_cuda)
SVT_B200_DECL_QFP(svt_av1_quantize_fp_32x32_cuda)
SVT_B200_DECL_QFP(svt_av1_quantize_fp_64x64_cuda)
SVT_B200_API void svt_av1_highbd_quantize_fp_cuda(const int32_t *coeff_ptr, intptr_t n_coeffs,
                                                  const int16_t *zbin_ptr, const int16_t *round_ptr,
                                                  const int16_t *quant_ptr, const int16_t *quant_shift_ptr,
                                                  int32_t *qcoeff_ptr, int32_t *dqcoeff_ptr,
                                                  const int16_t *dequant_ptr, uint16_t *eob_ptr,
                                                  const int16_t *scan, const int16_t *iscan, int16_t log_scale);

/* Scan order of a transform (get_scan / av1_scan_orders[tx_size][tx_type], Common/Codec/EbCoefficients.h):
 * writes the positions in scan order (64-wide sizes scan as their 32-wide packing); returns the count. */
SVT_B200_API int svt_b200_get_scan(int tx_size, int tx_type, int16_t *scan_out);

/* Fused per-transform-unit encode, the body of av1_encode_loop (Encoder/Codec/EbCodingLoop.c:290-...):
 *   residual = src - pred  ->  forward transform  ->  quantise + dequantise  ->  inverse transform  ->
 *   recon = clip(pred + residual').   One launch handles n_tus units of ONE transform size. */
typedef struct SvtB200Tu { /* one transform unit */
    int32_t x, y; /* top-left sample inside its plane */
    int32_t plane; /* 0 Y, 1 Cb, 2 Cr */
    int32_t tx_type; /* TxType enum value */
} SvtB200Tu;
typedef struct SvtB200QuantPlane { /* dc/ac pairs of Quants/Dequants (EbPictureControlSet.h:98-136) at this qindex */
    int16_t zbin[2], round[2], quant[2], quant_shift[2], dequant[2];
    int16_t round_fp[2], quant_fp[2];
} SvtB200QuantPlane;
typedef struct SvtB200EncodeParams {
    int32_t tx_size; /* TxSize enum value (TX_4X4=0 ... TX_64X16=18) */
    int32_t use_fp; /* 0: svt_aom_[highbd_]quantize_b, 1: svt_av1_[highbd_]quantize_fp (EbFullLoop.c:1527) */
    SvtB200QuantPlane q[3];
} SvtB200EncodeParams;
/* tus: device array; qcoeff: device int32 [n_tus][min(w,32)*min(h,32)]; eob: device uint16 [n_tus];
 * scratch: >= 8 KB of device memory. pred and recon may be the same frame. */
SVT_B200_API int svt_b200_encode_tus(const SvtB200EncodeParams *p, const SvtB200Frame *src,
                                     const SvtB200Frame *pred, const SvtB200Frame *recon,
                                     const SvtB200Tu *tus, int32_t n_tus, int32_t *qcoeff, uint16_t *eob,
                                     void *scratch, void *stream);
/* The dispatcher generality of av1_estimate_transform / av1_quantize_inv_quantize for the fused path (EbTransforms.c:3613-3670
 * trans_coeff_shape; EbFullLoop.c:1400-1470 table set by q_index): transform units of MIXED sizes, partial-frequency shapes
 * and quantiser sets in one call.  tus: HOST array, bucketed by (tx_size, pf_shape, qset) inside - one launch of the
 * size-specialised kernel per bucket.  Outputs in INPUT order: eob[i], cul_level[i] (device; cul_level may be NULL) and the
 * levels of unit i at qcoeff + qcoeff_offsets[i] (device; min(w,32)*min(h,32) int32 each); qcoeff_offsets: HOST array of
 * n_tus + 1 entries filled by the call (qcoeff must hold qcoeff_offsets[n_tus] entries: <= 1024 per unit).
 * scratch: device memory, >= 28 bytes per unit + 256.  Synchronous on `stream` (returns when the results are complete). */
typedef struct SvtB200TuEx {
    int32_t x, y;     /* top-left sample inside its plane */
    uint8_t plane;    /* 0 Y, 1 Cb, 2 Cr */
    uint8_t tx_type;  /* TxType */
    uint8_t tx_size;  /* TxSize, TX_4X4 = 0 ... TX_64X16 = 18 */
    uint8_t pf_shape; /* EB_TRANS_COEFF_SHAPE: 0 DEFAULT_SHAPE, 1 N2_SHAPE, 2 N4_SHAPE, 3 ONLY_DC_SHAPE (EbDefinitions.h:2611-2614) */
    uint16_t qset;    /* index into SvtB200EncodeParamsEx::qsets (one per distinct q_index in the picture) */
    uint16_t reserved;
} SvtB200TuEx;
typedef struct SvtB200EncodeParamsEx {
    int32_t use_fp;                      /* as SvtB200EncodeParams::use_fp */
    int32_t n_qsets;
    const SvtB200QuantPlane (*qsets)[3]; /* HOST array [n_qsets][3 planes] */
} SvtB200EncodeParamsEx;
SVT_B200_API int svt_b200_encode_tus_ex(const SvtB200EncodeParamsEx *p, const SvtB200Frame *src, const SvtB200Frame *pred,
                                        const SvtB200Frame *recon, const SvtB200TuEx *tus, int32_t n_tus, int32_t *qcoeff,
                                        int64_t *qcoeff_offsets, uint16_t *eob, int32_t *cul_level, void *scratch,
                                        size_t scratch_bytes, void *stream);

/* Device -> host hand-over of the levels: the entropy coder reads a TU's levels in scan order up to eob
 * (av1_write_coeffs_txb_1d), so instead of n int32 per TU the host can fetch `packed` = the eob[b] levels of TU b in scan
 * order at packed[offsets[b] .. offsets[b+1]) (offsets: exclusive prefix sum of eob, n_tus + 1 entries; *total = the
 * sum).  tx_class selects the scan: 0 default, 1 mrow (V_* types), 2 mcol (H_* types) — a call covers TUs of one class.
 * All pointers are device pointers; packed must hold n_tus * min(w,32) * min(h,32) entries in the worst case. */
SVT_B200_API int svt_b200_pack_levels(int32_t tx_size, int32_t tx_class, const int32_t *qcoeff, const uint16_t *eob,
                                      int32_t n_tus, int32_t *packed, uint32_t *offsets, uint32_t *total, void *stream);
/* Same, appending to a stream that already holds *base entries (base: DEVICE uint32, e.g. the `total` of the previous
 * call): offsets start at *base and *total = *base + sum(eob).  Lets the calls of one picture (one per transform size)
 * build ONE packed stream, fetched with one copy. */
SVT_B200_API int svt_b200_pack_levels_at(int32_t tx_size, int32_t tx_class, const int32_t *qcoeff, const uint16_t *eob,
                                         int32_t n_tus, int32_t *packed, uint32_t *offsets, uint32_t *total,
                                         const uint32_t *base, void *stream);
/* Same, plus cul_level[n_tus] (device int32, may be NULL): the value av1_quantize_inv_quantize returns
 * (EbFullLoop.c:1596-1608): min(63, sum |qcoeff|) with set_dc_sign of the DC level (bit 6 negative, +128 positive). */
SVT_B200_API int svt_b200_encode_tus_cul(const SvtB200EncodeParams *p, const SvtB200Frame *src,
                                         const SvtB200Frame *pred, const SvtB200Frame *recon,
                                         const SvtB200Tu *tus, int32_t n_tus, int32_t *qcoeff, uint16_t *eob,
                                         int32_t *cul_level, void *stream);

/* =============================================================================================== */
/* Deblocking loop filter                                                                          */
/* =============================================================================================== */

/* replace svt_aom_lpf_{horizontal,vertical}_{4,6,8,14} and svt_aom_highbd_lpf_* (common_dsp_rtcd.h:1039-1069;
 * C impl Common/Codec/EbDeblockingCommon.c:251-924): one 4-sample edge segment, in place. */
#define SVT_B200_DECL_LPF(DIR, N)                                                                          \
    SVT_B200_API void svt_aom_lpf_##DIR##_##N##_cuda(uint8_t *s, int32_t pitch, const uint8_t *blimit,     \
                                                     const uint8_t *limit, const uint8_t *thresh);         \
    SVT_B200_API void svt_aom_highbd_lpf_##DIR##_##N##_cuda(uint16_t *s, int32_t pitch,                    \
                                                            const uint8_t *blimit, const uint8_t *limit,   \
                                                            const uint8_t *thresh, int32_t bd);
SVT_B200_DECL_LPF(horizontal, 4) SVT_B200_DECL_LPF(horizontal, 6) SVT_B200_DECL_LPF(horizontal, 8)
SVT_B200_DECL_LPF(horizontal, 14) SVT_B200_DECL_LPF(vertical, 4) SVT_B200_DECL_LPF(vertical, 6)
SVT_B200_DECL_LPF(vertical, 8) SVT_B200_DECL_LPF(vertical, 14)

/* Per-4x4 (luma mi unit) summary of the ModeInfo grid that set_lpf_parameters (EbDeblockingFilter.c:168-319)
 * looks at.  The integration overlay fills it with the reference's own helpers (get_transform_size :134,
 * get_plane_block_size, lfi_n->lvl[][][][][] or get_filter_level_delta_lf) — see INTEGRATION.md; index [0] is
 * luma, [1] chroma (chroma reads the entry at the odd mi row/column of its 8x8, as the reference does). */
typedef struct SvtB200DlfMi {
    uint8_t tx_w[2], tx_h[2]; /* transform width / height in samples of that plane (4..64) */
    uint8_t blk_w[2], blk_h[2]; /* prediction block width / height in samples of that plane */
    uint8_t skip_inter; /* block_mi.skip && is_inter_block */
    uint8_t lvl_y[2]; /* filter level for luma vertical edges [0] / horizontal edges [1] */
    uint8_t lvl_u, lvl_v;
    uint8_t lvl_class; /* segment_id * 16 + ref_frame[0] * 2 + mode_lf_lut[mode]: the only block properties the level
                          table lfi_n->lvl[plane][seg][dir][ref][mode] is indexed by (EbDeblockingCommon.c:42-73); read
                          instead of lvl_* by the entries that take a level table (svt_b200_pick_filter_level) */
    uint8_t pad[2];
} SvtB200DlfMi;

typedef struct SvtB200DlfParams {
    int32_t mi_rows, mi_cols; /* picture size in 4x4 luma units */
    int32_t mi_stride; /* entries per row of the SvtB200DlfMi array */
    int32_t sharpness; /* frm_hdr->loop_filter_params.sharpness_level */
    int32_t filter_level[2], filter_level_u, filter_level_v; /* frame levels: planes with level 0 are skipped
                                                                exactly like loop_filter_sb (:629-636) */
    int32_t plane_start, plane_end; /* [start, end) as svt_av1_loop_filter_frame's arguments */
} SvtB200DlfParams;

/* svt_av1_loop_filter_frame (EbDeblockingFilter.c:711-753): deblocks `frame` in place. mi: device array
 * [mi_rows][mi_stride]. Two launches per call (all vertical edges, then all horizontal edges). */
SVT_B200_API int svt_b200_dlf_frame(const SvtB200DlfParams *p, const SvtB200Frame *frame,
                                    const SvtB200DlfMi *mi, void *stream);

/* The same with the block levels taken from a level table instead of the lvl_* fields of the summary:
 * lut = DEVICE uint8 [3][2][128] as svt_b200_lf_level_lut fills it (lfi_n->lvl[plane][seg][dir][ref][mode] indexed by lvl_class). */
SVT_B200_API int svt_b200_dlf_frame_lut(const SvtB200DlfParams *p, const SvtB200Frame *frame, const SvtB200DlfMi *mi,
                                        const uint8_t *lut, void *stream);

/* What svt_av1_loop_filter_frame_init (EbDeblockingCommon.c:78-145) reads besides the four frame levels. */
typedef struct SvtB200LfFrameInit {
    int32_t mode_ref_delta_enabled; /* lf->mode_ref_delta_enabled */
    int8_t ref_deltas[8], mode_deltas[2]; /* lf->ref_deltas[REF_FRAMES], lf->mode_deltas[MAX_MODE_LF_DELTAS] */
    int32_t segmentation_enabled; /* frm_hdr->segmentation_params.segmentation_enabled */
    uint8_t seg_feature_mask[8]; /* bit f: feature f active for the segment (features 1..4 = ALT_LF_Y_V, Y_H, U, V) */
    int16_t seg_feature_data[8][8]; /* segmentation_params.feature_data[segment][feature] */
} SvtB200LfFrameInit;

/* The level table of svt_av1_loop_filter_frame_init for frame levels {y vertical, y horizontal, u, v}:
 * lut[plane][dir][lvl_class]. Host function (no GPU work). */
SVT_B200_API int svt_b200_lf_level_lut(const SvtB200LfFrameInit *init, const int32_t levels[4], uint8_t lut[3][2][128]);

/* svt_av1_pick_filter_level (EbDeblockingFilter.c:1193-1297) with search_filter_level / try_filter_frame /
 * picture_sse_calculations (:1027-1191, :966-1026, :830-964).  method: LpfPickMethod (0 full image, 1 sub-image,
 * 2 from q, 3 minimal).  For methods 0/1 every trial is one device deblocking pass of one plane of `recon` + one SSE
 * against `source` + a plane copy back from `temp`; the bisection itself runs on the host (one 8-byte D2H per trial).
 * recon is unchanged on return.  Blocks take their level from the table of svt_b200_lf_level_lut via lvl_class
 * (delta_lf_present pictures are not searched by the reference's callers either). */
typedef struct SvtB200LpfPickParams {
    SvtB200DlfParams dlf; /* geometry; the levels / sharpness fields are ignored (sharpness is forced to 0, :1202) */
    SvtB200LfFrameInit init;
    int32_t method; /* LPF_PICK_FROM_FULL_IMAGE 0, LPF_PICK_FROM_SUBIMAGE 1, LPF_PICK_FROM_Q 2, LPF_PICK_MINIMAL_LPF 3 */
    int32_t loop_filter_mode; /* pcs->parent_pcs_ptr->loop_filter_mode (<= 2: one +-2 refinement, else bisection) */
    int32_t tx_mode_only_4x4; /* frm_hdr->tx_mode == ONLY_4X4 */
    int32_t q_ac; /* svt_av1_ac_quant_q3(base_q_idx, 0, bit_depth), method 2 only */
    int32_t key_frame; /* frm_hdr->frame_type == KEY_FRAME, method 2 only */
    int32_t last_level[4]; /* lf->filter_level[0], [1], filter_level_u, filter_level_v on entry */
} SvtB200LpfPickParams;
/* scratch: >= 1 KB of device memory.  levels_out: host int32[4] = {filter_level[0], [1], u, v}. temp: a frame of the same
 * geometry as recon (contents are overwritten). */
SVT_B200_API int svt_b200_pick_filter_level(const SvtB200LpfPickParams *p, const SvtB200Frame *recon,
                                            const SvtB200Frame *source, const SvtB200Frame *temp,
                                            const SvtB200DlfMi *mi, void *scratch, int32_t *levels_out, void *stream);

/* Sum of squared differences of two pictures per plane (picture_sse_calculations,
 * EbDeblockingFilter.c:830-964), the distortion measure of svt_av1_pick_filter_level. sse: device uint64[3]. */
SVT_B200_API int svt_b200_frame_sse(const SvtB200Frame *a, const SvtB200Frame *b, uint64_t *sse, void *stream);

/* =============================================================================================== */
/* Loop restoration: RTCD drop-ins of the filters + the frame-level filter                         */
/* =============================================================================================== */

/* replace svt_av1_selfguided_restoration / svt_apply_selfguided_restoration (common_dsp_rtcd.h:187-191;
 * EbRestoration.c:1012-1084).  High-bit-depth planes are passed as CONVERT_TO_BYTEPTR(ptr), as in the reference. */
SVT_B200_API void svt_av1_selfguided_restoration_cuda(const uint8_t *dgd8, int32_t width, int32_t height,
                                                      int32_t dgd_stride, int32_t *flt0, int32_t *flt1,
                                                      int32_t flt_stride, int32_t sgr_params_idx,
                                                      int32_t bit_depth, int32_t highbd);
SVT_B200_API void svt_apply_selfguided_restoration_cuda(const uint8_t *dat, int32_t width, int32_t height,
                                                        int32_t stride, int32_t eps, const int32_t *xqd,
                                                        uint8_t *dst, int32_t dst_stride, int32_t *tmpbuf,
                                                        int32_t bit_depth, int32_t highbd);
/* replace svt_av1_wiener_convolve_add_src / svt_av1_highbd_wiener_convolve_add_src (common_dsp_rtcd.h:183,185;
 * convolve.c:105-260). conv_params points at the reference's ConvolveParams (only round_0/round_1 are read). */
SVT_B200_API void svt_av1_wiener_convolve_add_src_cuda(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst,
                                                       ptrdiff_t dst_stride, const int16_t *filter_x,
                                                       const int16_t *filter_y, int32_t w, int32_t h,
                                                       const void *conv_params);
SVT_B200_API void svt_av1_highbd_wiener_convolve_add_src_cuda(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst,
                                                              ptrdiff_t dst_stride, const int16_t *filter_x,
                                                              const int16_t *filter_y, int32_t w, int32_t h,
                                                              const void *conv_params, int32_t bd);

/* =============================================================================================== */
/* Small reductions around the transform chain + the single-position SAD family (RTCD drop-ins)    */
/* =============================================================================================== */
/* replace svt_aom_subtract_block / svt_aom_highbd_subtract_block (common_dsp_rtcd.h:241,243) */
SVT_B200_API void svt_aom_subtract_block_cuda(int rows, int cols, int16_t *diff_ptr, ptrdiff_t diff_stride,
                                              const uint8_t *src_ptr, ptrdiff_t src_stride, const uint8_t *pred_ptr,
                                              ptrdiff_t pred_stride);
SVT_B200_API void svt_aom_highbd_subtract_block_cuda(int rows, int cols, int16_t *diff_ptr, ptrdiff_t diff_stride,
                                                     const uint8_t *src_ptr, ptrdiff_t src_stride,
                                                     const uint8_t *pred_ptr, ptrdiff_t pred_stride, int bd);
/* replace svt_full_distortion_kernel32_bits / _cbf_zero32_bits / svt_spatial_full_distortion_kernel /
 * svt_full_distortion_kernel16_bits (common_dsp_rtcd.h:172-179) */
SVT_B200_API void svt_full_distortion_kernel32_bits_cuda(int32_t *coeff, uint32_t coeff_stride, int32_t *recon_coeff,
                                                         uint32_t recon_coeff_stride, uint64_t distortion_result[2],
                                                         uint32_t area_width, uint32_t area_height);
SVT_B200_API void svt_full_distortion_kernel_cbf_zero32_bits_cuda(int32_t *coeff, uint32_t coeff_stride,
                                                                  uint64_t distortion_result[2], uint32_t area_width,
                                                                  uint32_t area_height);
SVT_B200_API uint64_t svt_spatial_full_distortion_kernel_cuda(uint8_t *input, uint32_t input_offset,
                                                              uint32_t input_stride, uint8_t *recon,
                                                              int32_t recon_offset, uint32_t recon_stride,
                                                              uint32_t area_width, uint32_t area_height);
SVT_B200_API uint64_t svt_full_distortion_kernel16_bits_cuda(uint8_t *input, uint32_t input_offset,
                                                             uint32_t input_stride, uint8_t *recon,
                                                             int32_t recon_offset, uint32_t recon_stride,
                                                             uint32_t area_width, uint32_t area_height);
/* replace svt_aom_satd / svt_av1_block_error (aom_dsp_rtcd.h:215,217) */
SVT_B200_API int svt_aom_satd_cuda(const int32_t *coeff, int length);
SVT_B200_API int64_t svt_av1_block_error_cuda(const int32_t *coeff, const int32_t *dqcoeff, intptr_t block_size,
                                              int64_t *ssz);
/* replace svt_nxm_sad_kernel_sub_sampled / sad_16b_kernel (aom_dsp_rtcd.h:643,651) */
SVT_B200_API uint32_t svt_nxm_sad_kernel_sub_sampled_cuda(const uint8_t *src, uint32_t src_stride, const uint8_t *ref,
                                                          uint32_t ref_stride, uint32_t height, uint32_t width);
SVT_B200_API uint32_t sad_16b_kernel_cuda(uint16_t *src, uint32_t src_stride, uint16_t *ref, uint32_t ref_stride,
                                          uint32_t height, uint32_t width);
/* replace svt_aom_sadMxN / svt_aom_sadMxNx4d (aom_dsp_rtcd.h:264-388) */
#define SVT_B200_DECL_SAD(W, H)                                                                           \
    SVT_B200_API uint32_t svt_aom_sad##W##x##H##_cuda(const uint8_t *src_ptr, int src_stride,             \
                                                      const uint8_t *ref_ptr, int ref_stride);            \
    SVT_B200_API void svt_aom_sad##W##x##H##x4d_cuda(const uint8_t *src_ptr, int src_stride,              \
                                                     const uint8_t *const ref_ptr[], int ref_stride,      \
                                                     uint32_t *sad_array);
SVT_B200_DECL_SAD(128, 128) SVT_B200_DECL_SAD(128, 64) SVT_B200_DECL_SAD(64, 128) SVT_B200_DECL_SAD(64, 64)
SVT_B200_DECL_SAD(64, 32) SVT_B200_DECL_SAD(64, 16) SVT_B200_DECL_SAD(32, 64) SVT_B200_DECL_SAD(32, 32)
SVT_B200_DECL_SAD(32, 16) SVT_B200_DECL_SAD(32, 8) SVT_B200_DECL_SAD(16, 64) SVT_B200_DECL_SAD(16, 32)
SVT_B200_DECL_SAD(16, 16) SVT_B200_DECL_SAD(16, 8) SVT_B200_DECL_SAD(16, 4) SVT_B200_DECL_SAD(8, 32)
SVT_B200_DECL_SAD(8, 16) SVT_B200_DECL_SAD(8, 8) SVT_B200_DECL_SAD(8, 4) SVT_B200_DECL_SAD(4, 16)
SVT_B200_DECL_SAD(4, 8) SVT_B200_DECL_SAD(4, 4)

/* RestorationUnitInfo (Common/Codec/EbRestoration.h): what svt_av1_loop_restoration_filter_unit reads per unit. */
typedef struct SvtB200LrUnit {
    int32_t restoration_type; /* RESTORE_NONE 0, RESTORE_WIENER 1, RESTORE_SGRPROJ 2 */
    int16_t vfilter[8], hfilter[8]; /* wiener_info.vfilter / hfilter (InterpKernel; tap [7] is 0) */
    int32_t sgr_ep, sgr_xqd[2]; /* sgrproj_info.ep, .xqd */
} SvtB200LrUnit;
typedef struct SvtB200LrPlane {
    int32_t frame_restoration_type; /* rsi->frame_restoration_type: 0 = plane passes through unchanged */
    int32_t restoration_unit_size; /* rsi->restoration_unit_size (multiple of 64; chroma: of 32) */
    const SvtB200LrUnit *units; /* DEVICE array [vert_units][horz_units], unit counts as count_units_in_tile
                                   (EbRestoration.c:175) derives them from the plane size */
} SvtB200LrPlane;
typedef struct SvtB200LrFrameParams {
    SvtB200LrPlane plane[3];
    int32_t optimized_lr; /* rsi->optimized_lr: stripe context of 1 replicated CDEF row instead of deblocked rows */
} SvtB200LrFrameParams;

/* svt_av1_loop_restoration_filter_frame (Common/Codec/EbRestoration.c:1293-1364) with the stripe protocol of
 * svt_av1_loop_restoration_filter_unit (:1162-1261), setup/restore_processing_stripe_boundary (:353-507) and the
 * boundary lines of svt_av1_loop_restoration_save_boundary_lines (:1645-1868), single tile, no super-resolution.
 * cdef: the picture after CDEF (filter input); deblocked: the picture after deblocking, before CDEF (its rows are
 * the 2-row stripe context the reference saves with after_cdef = 0); out: the restored picture (must not alias).
 * One launch; every 64x64 (chroma 32x32) processing unit of every stripe is one CTA. */
SVT_B200_API int svt_b200_lr_frame(const SvtB200LrFrameParams *p, const SvtB200Frame *cdef, const SvtB200Frame *deblocked,
                                   const SvtB200Frame *out, void *stream);

/* =============================================================================================== */
/* Loop restoration search: the reductions (the double-precision solves stay on the host)          */
/* =============================================================================================== */

/* replace svt_av1_compute_stats / svt_av1_compute_stats_highbd (aom_dsp_rtcd.h:71-74; EbRestorationPick.c:704-790):
 * Wiener normal equations M[win^2], H[win^2 x win^2] (int64, exact) of one restoration unit. High-bit-depth planes are
 * passed as CONVERT_TO_BYTEPTR pointers, as in the reference. */
SVT_B200_API void svt_av1_compute_stats_cuda(int32_t wiener_win, const uint8_t *dgd8, const uint8_t *src8,
                                             int32_t h_start, int32_t h_end, int32_t v_start, int32_t v_end,
                                             int32_t dgd_stride, int32_t src_stride, int64_t *M, int64_t *H);
SVT_B200_API void svt_av1_compute_stats_highbd_cuda(int32_t wiener_win, const uint8_t *dgd8, const uint8_t *src8,
                                                    int32_t h_start, int32_t h_end, int32_t v_start, int32_t v_end,
                                                    int32_t dgd_stride, int32_t src_stride, int64_t *M, int64_t *H,
                                                    int32_t bit_depth);
/* replace svt_av1_lowbd_pixel_proj_error / svt_av1_highbd_pixel_proj_error (aom_dsp_rtcd.h:84-87;
 * EbRestorationPick.c:174-315). params: the reference's SgrParamsType {r[2], s[2]}. */
SVT_B200_API int64_t svt_av1_lowbd_pixel_proj_error_cuda(const uint8_t *src8, int32_t width, int32_t height,
                                                         int32_t src_stride, const uint8_t *dat8, int32_t dat_stride,
                                                         int32_t *flt0, int32_t flt0_stride, int32_t *flt1,
                                                         int32_t flt1_stride, int32_t xq[2], const void *params);
SVT_B200_API int64_t svt_av1_highbd_pixel_proj_error_cuda(const uint8_t *src8, int32_t width, int32_t height,
                                                          int32_t src_stride, const uint8_t *dat8, int32_t dat_stride,
                                                          int32_t *flt0, int32_t flt0_stride, int32_t *flt1,
                                                          int32_t flt1_stride, int32_t xq[2], const void *params);
/* replace svt_get_proj_subspace (aom_dsp_rtcd.h:219-220; EbRestorationPick.c:337-440): the projection coefficients xq[2]
 * of the self-guided filter.  The five sums are exact 64-bit integer reductions on the device (the reference's double
 * accumulations are exact too: integer terms, partial sums < 2^53); the 2x2 solve repeats the reference's double
 * expressions on the host. */
SVT_B200_API void svt_get_proj_subspace_cuda(const uint8_t *src8, int32_t width, int32_t height, int32_t src_stride,
                                             const uint8_t *dat8, int32_t dat_stride, int32_t use_highbitdepth,
                                             int32_t *flt0, int32_t flt0_stride, int32_t *flt1, int32_t flt1_stride,
                                             int32_t *xq, const void *params);
/* The compute_stats calls of search_wiener for every restoration unit of one plane in three launches, pictures resident
 * on the device.  rects: DEVICE int32 [n_units][4] = {h_start, h_end, v_start, v_end} (RestorationTileLimits); reads of
 * dgd outside the plane are clamped (= the 3-sample replicated border the reference extends the picture by);
 * out: DEVICE int64 [n_units][win^2 + win^4] (M, then H); scratch: DEVICE, >= 8 * n_units bytes. */
SVT_B200_API int svt_b200_lr_wiener_stats(const SvtB200Frame *dgd, const SvtB200Frame *src, int32_t plane,
                                          int32_t wiener_win, const int32_t *rects, int32_t n_units,
                                          int32_t max_unit_w, int32_t max_unit_h, int64_t *out, void *scratch,
                                          void *stream);

/* The self-guided side of the search (search_selfguided_restoration, EbRestorationPick.c:583-661) for every restoration
 * unit of one plane and every parameter set of eps[] (host array, values 0..15) at once, pictures resident on the device:
 *  - svt_b200_lr_sgr_filter_sums: apply_sgr (:554-581; the filter per 64x64 / 32x32 processing unit tiled from the unit's
 *    origin, reads outside the plane clamped) with both outputs kept in flt = DEVICE int32 [n_eps][2][plane_h][plane_w], and
 *    the five sums of svt_get_proj_subspace in sums = DEVICE int64 [n_units][n_eps][5] = {H00, H11, H01, C0, C1} (before the
 *    division by the unit size; the 2x2 solve stays on the host);
 *  - svt_b200_lr_sgr_proj_error: get_pixel_proj_error (:316-360) for one decoded xq pair per (unit, ep): xq = DEVICE int32
 *    [n_units][n_eps][2], err = DEVICE int64 [n_units][n_eps]; one call per step of finer_search_pixel_proj_error.
 * rects: DEVICE int32 [n_units][4] = {h_start, h_end, v_start, v_end}. */
SVT_B200_API int svt_b200_lr_sgr_filter_sums(const SvtB200Frame *dgd, const SvtB200Frame *src, int32_t plane,
                                             const int32_t *rects, int32_t n_units, int32_t max_unit_w, int32_t max_unit_h,
                                             const int32_t *eps, int32_t n_eps, int32_t *flt, int64_t *sums, void *stream);
SVT_B200_API int svt_b200_lr_sgr_proj_error(const SvtB200Frame *dgd, const SvtB200Frame *src, int32_t plane,
                                            const int32_t *rects, int32_t n_units, int32_t max_unit_w, int32_t max_unit_h,
                                            const int32_t *eps, int32_t n_eps, const int32_t *flt, const int32_t *xq,
                                            int64_t *err, void *stream);

/* =============================================================================================== */
/* Inter prediction (translational, SURVEY 8(f) rank 1): the sub-pel interpolation filters          */
/* =============================================================================================== */

/* Layout-compatible mirrors of the two reference structs the convolve pointers take
 * (InterpFilterParams EbDefinitions.h:493-498, ConvolveParams EbDefinitions.h:379-392). */
typedef struct SvtB200InterpFilterParams {
    const int16_t *filter_ptr; /* [subpel_shifts][taps] */
    uint16_t taps, subpel_shifts;
    int32_t interp_filter; /* InterpFilter enum (unused here) */
} SvtB200InterpFilterParams;
typedef struct SvtB200ConvolveParams {
    int32_t ref, do_average;
    uint16_t *dst; /* CONV_BUF of the compound path */
    int32_t dst_stride, round_0, round_1, plane, is_compound, use_jnt_comp_avg, fwd_offset, bck_offset,
        use_dist_wtd_comp_avg;
} SvtB200ConvolveParams;

/* replace svt_av1_convolve_{2d_sr,x_sr,y_sr,2d_copy_sr} and svt_av1_jnt_convolve_{2d,x,y,2d_copy}
 * (common_dsp_rtcd.h:194-211; C impl EbInterPrediction.c:349-480, :552-745) and their highbd forms (:212-229; C impl
 * :747-1145).  Host pointers, same argument meaning; taps are always 8 (the reference's 4-tap kernels are zero padded).
 * The jnt forms read (do_average) or write conv_params->dst exactly as the C code does. */
#define SVT_B200_CONVOLVE_DECL(NAME)                                                                                  \
    SVT_B200_API void NAME##_cuda(const uint8_t *src, int32_t src_stride, uint8_t *dst, int32_t dst_stride, int32_t w, \
                                  int32_t h, SvtB200InterpFilterParams *filter_params_x,                               \
                                  SvtB200InterpFilterParams *filter_params_y, const int32_t subpel_x_q4,               \
                                  const int32_t subpel_y_q4, SvtB200ConvolveParams *conv_params);
#define SVT_B200_HBD_CONVOLVE_DECL(NAME)                                                                               \
    SVT_B200_API void NAME##_cuda(const uint16_t *src, int32_t src_stride, uint16_t *dst, int32_t dst_stride,          \
                                  int32_t w, int32_t h, const SvtB200InterpFilterParams *filter_params_x,              \
                                  const SvtB200InterpFilterParams *filter_params_y, const int32_t subpel_x_q4,         \
                                  const int32_t subpel_y_q4, SvtB200ConvolveParams *conv_params, int32_t bd);
SVT_B200_CONVOLVE_DECL(svt_av1_convolve_2d_copy_sr)
SVT_B200_CONVOLVE_DECL(svt_av1_convolve_2d_sr)
SVT_B200_CONVOLVE_DECL(svt_av1_convolve_x_sr)
SVT_B200_CONVOLVE_DECL(svt_av1_convolve_y_sr)
SVT_B200_CONVOLVE_DECL(svt_av1_jnt_convolve_2d_copy)
SVT_B200_CONVOLVE_DECL(svt_av1_jnt_convolve_2d)
SVT_B200_CONVOLVE_DECL(svt_av1_jnt_convolve_x)
SVT_B200_CONVOLVE_DECL(svt_av1_jnt_convolve_y)
SVT_B200_HBD_CONVOLVE_DECL(svt_av1_highbd_convolve_2d_copy_sr)
SVT_B200_HBD_CONVOLVE_DECL(svt_av1_highbd_convolve_2d_sr)
SVT_B200_HBD_CONVOLVE_DECL(svt_av1_highbd_convolve_x_sr)
SVT_B200_HBD_CONVOLVE_DECL(svt_av1_highbd_convolve_y_sr)
SVT_B200_HBD_CONVOLVE_DECL(svt_av1_highbd_jnt_convolve_2d_copy)
SVT_B200_HBD_CONVOLVE_DECL(svt_av1_highbd_jnt_convolve_2d)
SVT_B200_HBD_CONVOLVE_DECL(svt_av1_highbd_jnt_convolve_x)
SVT_B200_HBD_CONVOLVE_DECL(svt_av1_highbd_jnt_convolve_y)

/* replace svt_aom_convolve8_horiz / svt_aom_convolve8_vert (common_dsp_rtcd.h:230-233; convolve.c:249-308): filter_x /
 * filter_y point INTO a 256-byte aligned [16][8] kernel table (get_filter_base / get_filter_offset, convolve.c), the
 * position steps by x_step_q4 / y_step_q4 sixteenths per output sample. */
SVT_B200_API void svt_aom_convolve8_horiz_cuda(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst, ptrdiff_t dst_stride,
                                               const int16_t *filter_x, int x_step_q4, const int16_t *filter_y,
                                               int y_step_q4, int w, int h);
SVT_B200_API void svt_aom_convolve8_vert_cuda(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst, ptrdiff_t dst_stride,
                                              const int16_t *filter_x, int x_step_q4, const int16_t *filter_y,
                                              int y_step_q4, int w, int h);

/* The interpolation kernel av1_get_interp_filter_params_with_block_size(filter, w) selects (EbInterPrediction.c:1251-1262:
 * the 4-tap tables when w <= 4), row `subpel` (0..15), as this library holds it. Returns 0, or <0 on a bad argument. */
SVT_B200_API int svt_b200_get_interp_kernel(int32_t interp_filter, int32_t w, int32_t subpel, int16_t out[8]);

/* One enc_make_inter_predictor call (EbEncInterPrediction.c:3663-3762; unscaled references, no masked compound / OBMC /
 * warp / intra-BC), or the List0 + List1 pair of calls of a BI_PRED block merged (n_refs == 2: what av1_inter_prediction
 * :4330-4930 issues with do_average 0 then 1; the CONV_BUF intermediate stays on chip).  All positions in samples of
 * `plane`; the host decomposes a block into its per-plane jobs exactly as av1_inter_prediction does (including the
 * sub8x8 chroma case, :4150-4330, where each job carries the neighbour's MV / reference and the b4 size). */
typedef struct SvtB200InterJob {
    uint8_t plane;  /* 0 Y, 1 Cb, 2 Cr (ss_x = ss_y = plane != 0) */
    uint8_t n_refs; /* 1, or 2 = compound */
    uint8_t bw, bh; /* blk_width, blk_height (also select the 4-tap kernels when <= 4) */
    uint8_t ref[2]; /* index into refs[] */
    uint8_t filter_x, filter_y; /* av1_extract_interp_filter(interp_filters, 1 / 0): 0 regular, 1 smooth, 2 sharp, 3 bilinear */
    uint8_t use_jnt_comp_avg, fwd_offset, bck_offset, reserved; /* svt_av1_dist_wtd_comp_weight_assign (:310-347) */
    int16_t dst_x, dst_y; /* where the block lands in the prediction plane */
    int16_t pre_x, pre_y; /* pu_origin_{x,y}[_chroma] */
    int16_t mv_row[2], mv_col[2]; /* MvUnit mv[list].y / .x, 1/8 luma sample */
    int32_t mb_to_left_edge, mb_to_right_edge, mb_to_top_edge, mb_to_bottom_edge; /* blk_ptr->av1xd */
} SvtB200InterJob;

/* Every job of a picture: refs[] = the n_ref_frames reference pictures (recon, padded at least as far as
 * clamp_mv_to_umv_border_sb lets a block reach: bw + 4 + 4 samples beyond the picture, as EbPictureBufferDesc pads
 * them), pred = the prediction picture, jobs = DEVICE array.  8-bit -> uint8_t planes, 10/12-bit -> uint16_t planes
 * (av1_inter_prediction with is16bit).  Jobs must not overlap in pred.  scratch: DEVICE memory holding the list of
 * 16x8 tiles the jobs expand to; svt_b200_inter_predict_scratch_bytes() sizes it for non-overlapping jobs of a
 * width x height picture.  A smaller scratch (>= 256 bytes) only costs speed, never correctness.  Asynchronous on
 * `stream` (two launches). */
SVT_B200_API size_t svt_b200_inter_predict_scratch_bytes(int32_t n_jobs, int32_t width, int32_t height);
SVT_B200_API int svt_b200_inter_predict(const SvtB200Frame *refs, int32_t n_ref_frames, const SvtB200Frame *pred,
                                        const SvtB200InterJob *jobs, int32_t n_jobs, void *scratch, size_t scratch_bytes,
                                        void *stream);

/* =============================================================================================== */
/* Sub-pel motion refinement (SURVEY 8(f) rank 2)                                                  */
/* =============================================================================================== */

/* replace svt_aom_varianceWxH (22 sizes, aom_dsp_rtcd.h:488-530; EbComputeVariance_C.c:14-61) and svt_aom_mse16x16 (:249;
 * EbPsnr.c:84-89, which returns the variance too) */
#define SVT_B200_VAR_DECL(W, H)                                                                                      \
    SVT_B200_API unsigned int svt_aom_variance##W##x##H##_cuda(const uint8_t *src_ptr, int source_stride,             \
                                                               const uint8_t *ref_ptr, int ref_stride, unsigned int *sse);
SVT_B200_VAR_DECL(4, 4) SVT_B200_VAR_DECL(4, 8) SVT_B200_VAR_DECL(4, 16) SVT_B200_VAR_DECL(8, 4) SVT_B200_VAR_DECL(8, 8)
SVT_B200_VAR_DECL(8, 16) SVT_B200_VAR_DECL(8, 32) SVT_B200_VAR_DECL(16, 4) SVT_B200_VAR_DECL(16, 8) SVT_B200_VAR_DECL(16, 16)
SVT_B200_VAR_DECL(16, 32) SVT_B200_VAR_DECL(16, 64) SVT_B200_VAR_DECL(32, 8) SVT_B200_VAR_DECL(32, 16) SVT_B200_VAR_DECL(32, 32)
SVT_B200_VAR_DECL(32, 64) SVT_B200_VAR_DECL(64, 16) SVT_B200_VAR_DECL(64, 32) SVT_B200_VAR_DECL(64, 64) SVT_B200_VAR_DECL(64, 128)
SVT_B200_VAR_DECL(128, 64) SVT_B200_VAR_DECL(128, 128)
SVT_B200_API uint32_t svt_aom_mse16x16_cuda(const uint8_t *src_ptr, int32_t source_stride, const uint8_t *ref_ptr,
                                            int32_t recon_stride, uint32_t *sse);
/* replaces svt_aom_upsampled_pred (aom_dsp_rtcd.h:354; Encoder/C_DEFAULT/variance.c:212-269). xd, cm, mi_row, mi_col, mv are
 * unused by the C code as well; subpel_search: 1 USE_2_TAPS, 2 USE_4_TAPS, 3 USE_8_TAPS. */
SVT_B200_API void svt_aom_upsampled_pred_cuda(void *xd, const void *cm, int mi_row, int mi_col, const void *mv, uint8_t *comp_pred,
                                              int width, int height, int subpel_x_q3, int subpel_y_q3, const uint8_t *ref,
                                              int ref_stride, int subpel_search);

/* svt_av1_find_best_sub_pixel_tree (Encoder/Codec/mcomp.c:350-418) as md_subpel_search sets it up
 * (EbProductCodingLoop.c:2063-2155: 8-bit luma, no second predictor / mask / OBMC, last_mv_search_list == NULL), for a
 * batch of independent (block, reference) searches.  The search is the reference's: centre error, then per round
 * (1/2, 1/4, 1/8 sample) left / right / up / down, the diagonal they point to, and with iters_per_step > 1 the
 * second-level check; an evaluation = svt_aom_upsampled_pred (Encoder/C_DEFAULT/variance.c:212-269: 8-tap / 4-tap /
 * bilinear kernels, two passes each rounded to 8 bits) + svt_aom_varianceWxH (EbComputeVariance_C.c:14-61) +
 * svt_mv_err_cost (mcomp.c:44-64). */
typedef struct SvtB200SubpelJob {
    int16_t blk_x, blk_y; /* context_ptr->blk_origin_x / _y */
    uint8_t bw, bh;       /* block_size_wide / _high [bsize] */
    uint8_t ref;          /* index into refs[] */
    uint8_t reserved;
    int16_t start_mv_row, start_mv_col; /* subpel_start_mv: the full-pel MV in 1/8 sample (multiples of 8; anything else is
                                           rejected with besterr = -1, like a block that does not fit or ref >= n_ref_frames).
                                           The reference's last_mv_search_list early-out (mcomp.c) is not modelled: pass jobs
                                           as md_subpel_search does, with last_mv_search_list == NULL */
    int16_t ref_mv_row, ref_mv_col;     /* context_ptr->ref_mv (the MV the rate is measured from) */
    int16_t col_min, col_max, row_min, row_max; /* ms_params->mv_limits (svt_av1_set_subpel_mv_search_range, mcomp.h:124-138) */
} SvtB200SubpelJob;
typedef struct SvtB200SubpelParams {
    int32_t allow_hp;           /* eight_pel_search_enabled && frm_hdr.allow_high_precision_mv */
    int32_t forced_stop;        /* SUBPEL_FORCE_STOP: 0 EIGHTH_PEL .. 3 FULL_PEL */
    int32_t iters_per_step;     /* md_subpel_ctrls.subpel_iters_per_step */
    int32_t subpel_search_type; /* SUBPEL_SEARCH_TYPE: 1 USE_2_TAPS, 2 USE_4_TAPS, 3 USE_8_TAPS */
    int32_t mv_cost_type;       /* MV_COST_TYPE: 0 ENTROPY, 1 L1_LOWRES, 2 L1_MIDRES, 3 L1_HDRES, 4 NONE */
    int32_t error_per_bit;      /* AOMMAX(rdmult >> RD_EPB_SHIFT, 1) */
    int32_t mvjcost[4];         /* md_rate_estimation_ptr->nmv_vec_cost */
    int32_t max_block_w, max_block_h; /* largest bw / bh among the jobs (sizes the shared-memory window and the CTA); 0 = 128.
                                       * A job that exceeds it is not searched: besterr = distortion = -1, mv = start_mv */
    const int32_t *mvcost[2];   /* DEVICE, nmvcoststack[0 / 1]: centred tables, indices -16383 .. 16383 (MV_COST_ENTROPY only) */
} SvtB200SubpelParams;
typedef struct SvtB200SubpelResult {
    int16_t mv_row, mv_col; /* *bestmv */
    int32_t besterr;        /* the return value */
    int32_t distortion;     /* *distortion */
    uint32_t sse;           /* *sse1 */
} SvtB200SubpelResult;
/* src: the source picture, refs[]: the reference pictures (8-bit; only the luma planes are read; references padded as
 * the reference pads them: the limits keep a block within AOM_INTERP_EXTEND of the picture and 4 taps reach beyond);
 * jobs / results: DEVICE arrays.  Asynchronous on `stream`. */
SVT_B200_API int svt_b200_subpel_search(const SvtB200SubpelParams *p, const SvtB200Frame *src, const SvtB200Frame *refs,
                                        int32_t n_ref_frames, const SvtB200SubpelJob *jobs, int32_t n_jobs,
                                        SvtB200SubpelResult *results, void *stream);

/* =============================================================================================== */
/* (3) Picture engine: the picture-level entries with HOST buffers, as the reference's process     */
/*     loops own them (SURVEY.md 8b "Batched entry", "Memory ownership", "Threading").             */
/*     One engine per encoder handle and GPU.  Every call is synchronous for its caller and        */
/*     re-entrant: the reference calls from N pipeline threads for N pictures at once.             */
/* =============================================================================================== */
typedef struct SvtB200Engine SvtB200Engine;

typedef struct SvtB200EngineStats {
    uint64_t me_pictures, dlf_frames, cdef_frames, lr_frames;
    uint64_t me_plane_uploads, me_plane_hits; /* ME plane residency cache: pictures uploaded / found resident */
    uint64_t h2d_bytes, d2h_bytes, pinned_bytes;
    /* wall time summed over calling threads: waiting for a slot, waiting for another thread's upload of a shared
     * reference, issuing copies + launches, waiting for the GPU, copying between host pictures and pinned staging */
    uint64_t ns_slot_wait, ns_plane_wait, ns_issue, ns_sync, ns_host_copy;
} SvtB200EngineStats;

/* device: CUDA ordinal (the integration reads SVT_CUDA_DEVICE).  Fails (no CPU fallback) when it does not exist.
 * The engine copies host pictures through its own pinned staging: the caller's buffers stay pageable, and the engine
 * reads or writes them only during a call. */
SVT_B200_API int svt_b200_engine_create(int device, SvtB200Engine **out);
SVT_B200_API void svt_b200_engine_destroy(SvtB200Engine *e);
SVT_B200_API int svt_b200_engine_get_stats(SvtB200Engine *e, SvtB200EngineStats *out);

/* The three padded 8-bit luma planes of one picture in HOST memory (EbPaReferenceObject: input_padded_picture_ptr,
 * quarter_/sixteenth_{filtered,decimated}_picture_ptr; pointers address element (0,0) of the padded buffer_y).
 * (key, tag) identify the content - the integration passes the EbPaReferenceObject pointer and the picture number -
 * so a picture uploaded once (as ME source) is found resident when later pictures use it as reference.
 * quarter / sixteenth may be NULL: they are then derived on the device (svt_b200_me_downsample). */
typedef struct SvtB200HostMePicture {
    const void *key;
    uint64_t tag;
    const uint8_t *full, *quarter, *sixteenth;
} SvtB200HostMePicture;

/* Replaces the SB loop of motion_estimation_kernel (EbMotionEstimationProcess.c:831-965) for one picture with host
 * planes and host results: me_mv [n_sb][85*7][2] int16, me_cand [n_sb][85*23], total_cand [n_sb][85],
 * rc_me_distortion [n_sb] (layouts of SvtB200MeOutputs).  filtered_downsample: only read when a picture carries no
 * quarter / sixteenth planes (scs->down_sampling_method_me_search == ME_FILTERED_DOWNSAMPLED). */
SVT_B200_API int svt_b200_engine_me_picture(SvtB200Engine *e, const SvtB200MeParams *p, const SvtB200HostMePicture *src,
                                            const SvtB200HostMePicture refs[SVT_B200_ME_LISTS][SVT_B200_ME_MAX_REFS],
                                            int32_t filtered_downsample, int16_t *me_mv, uint8_t *me_cand,
                                            uint8_t *total_cand, uint32_t *rc_me_distortion);

/* svt_av1_loop_filter_frame (EbDeblockingFilter.c:711) on a HOST picture, in place; mi: host array. */
SVT_B200_API int svt_b200_engine_dlf_frame(SvtB200Engine *e, const SvtB200DlfParams *p, const SvtB200Frame *frame,
                                           const SvtB200DlfMi *mi);

/* dlf_kernel for loop_filter_mode >= 2 (presets <= 6; EbDlfProcess.c:186-216): svt_av1_pick_filter_level(FROM_FULL_IMAGE)
 * followed by svt_av1_loop_filter_frame with the picked levels, on a HOST picture in place.  recon / source are uploaded
 * once, every trial of the level search (one plane pass + SSE + plane restore) runs on the device, then the frame is
 * deblocked with the result and read back.  levels_out: {filter_level[0], [1], u, v} for the frame header.
 * mi: host array [mi_rows][mi_cols] (lvl_class is what is read).  pp->dlf.sharpness is ignored (the reference forces 0). */
SVT_B200_API int svt_b200_engine_dlf_pick_frame(SvtB200Engine *e, const SvtB200LpfPickParams *pp, const SvtB200Frame *recon,
                                                const SvtB200Frame *source, const SvtB200DlfMi *mi, int32_t levels_out[4]);

/* svt_av1_loop_restoration_filter_frame of rest_kernel (EbRestProcess.c:530-534; presets <= 6) on a HOST picture in place.
 * frame: the picture after CDEF (cm->frame_to_show).  The stripe context comes from the boundary lines the reference saved
 * with svt_av1_loop_restoration_save_boundary_lines(after_cdef = 0) - RestorationStripeBoundaries of each plane: `above` /
 * `below` address sample 0 of line 0 of stripe 0 (stripe_boundary_above/below + RESTORATION_EXTRA_HORZ), two lines per
 * stripe, `stride` samples apart.  p->plane[i].units are HOST arrays here (n_units[i] entries); planes whose
 * frame_restoration_type is 0 are left untouched. */
typedef struct SvtB200HostLrLines {
    const void *above, *below;
    int32_t stride;
} SvtB200HostLrLines;
SVT_B200_API int svt_b200_engine_lr_frame(SvtB200Engine *e, const SvtB200LrFrameParams *p, const int32_t n_units[3],
                                          const SvtB200Frame *frame, const SvtB200HostLrLines lines[3]);

/* The CDEF stage of cdef_kernel (EbCdefProcess.c:510-534) for one HOST picture, preceded by the deblocking of the
 * picture when dlf != NULL (mi: host array [mi_rows][mi_cols]): the reconstruction is uploaded ONCE, deblocked on the
 * device and handed to the CDEF stages there - for pictures whose deblocked version nobody needs on the host (no loop
 * restoration: svt_av1_loop_restoration_save_boundary_lines would read it).  Strength search of every 64x64 filter
 * block, the strength decision (svt_b200_cdef_decide: finish_cdef_search, EbEncCdef.c:1167), frame apply written back
 * into `recon` (host) in place when apply != 0, one download, ONE synchronisation.  With apply = 0 the host
 * reconstruction is left as it was: the reference does not filter a picture nobody reads.  decision / fb_strength_idx:
 * HOST outputs (frame header fields and mbmi.cdef_strength per filter block, -1 = all-skip block).  skip_stride up to
 * ((mi_cols + 1) / 2 + 15) & ~15 fits the engine's staging of the skip map; a larger stride may return SVT_B200_ERR_ARG. */
SVT_B200_API int svt_b200_engine_dlf_cdef_frame_dev(SvtB200Engine *e, const SvtB200DlfParams *dlf, const SvtB200DlfMi *mi,
                                                    const SvtB200CdefSearchParams *sp, const SvtB200CdefDecideParams *dp,
                                                    int32_t damping, int32_t apply, const SvtB200Frame *recon,
                                                    const SvtB200Frame *source, const uint8_t *skip8, int32_t skip_stride,
                                                    SvtB200CdefDecision *decision, int8_t *fb_strength_idx);

/* =============================================================================================== */
/* Temporal filtering (SURVEY.md 8(f) rank 4)                                                      */
/* =============================================================================================== */

/* The planewise weighting of the temporal filter for many blocks of one (centre picture, motion-compensated reference)
 * pair: replaces the per-32x32 calls of svt_av1_apply_temporal_filter_planewise[_hbd] (aom_dsp_rtcd.c:365-366; C
 * EbTemporalFiltering.c:643-811, 829-1017) made by apply_filtering_block_plane_wise (:1025-1131).  Bit-exact, floating
 * point chain included (see csrc/tf.cu).  src: the picture being filtered; pred: its motion-compensated prediction from
 * one reference picture, same geometry; accum / count: picture-sized accumulators (device), same coordinates as pred.
 * blocks: DEVICE array; x / y: luma position of the block (even); block_error[q] / d_factor[q] for the four quadrants
 * q = (row >= h/2) * 2 + (col >= w/2), computed as the reference does (:696-734):
 *   block_error = split ? tf_16x16_block_error[idx*4+q] / 256 : tf_32x32_block_error[idx] / 1024   (errors >> 4 at 10 bit)
 *   d_factor    = max(sqrtf(powf(mv.row,2) + powf(mv.col,2)) / max(min_frame_size * 0.1, 1), 1)
 * den[p] = 2 * n_decay^2, n_decay = decay_control * (0.7 + log1p(noise_levels[p])) (:712). */
typedef struct SvtB200TfBlock {
    int32_t x, y;
    double block_error[4], d_factor[4];
} SvtB200TfBlock;
typedef struct SvtB200TfParams {
    double den[3];
    int32_t chroma;           /* MeContext::tf_chroma */
    int32_t block_w, block_h; /* 32 x 32 in the reference (BW >> 1); even, <= 64 */
} SvtB200TfParams;
typedef struct SvtB200TfAccum {
    uint32_t *accum[3];
    uint16_t *count[3];
    int32_t stride_y, stride_c; /* entries */
} SvtB200TfAccum;
SVT_B200_API int svt_b200_tf_planewise(const SvtB200TfParams *p, const SvtB200Frame *src, const SvtB200Frame *pred,
                                       const SvtB200TfBlock *blocks, int32_t n_blocks, const SvtB200TfAccum *acc, void *stream);
/* apply_filtering_central[_highbd] (:551-621) for the whole picture: accum += 1000 * sample, count += 1000 */
SVT_B200_API int svt_b200_tf_central(const SvtB200Frame *center, const SvtB200TfAccum *acc, int32_t chroma, void *stream);
/* get_final_filtered_pixels (:1943-2050) for the whole picture: dst = (accum + count / 2) / count in place;
 * sse2: DEVICE uint64[2] or NULL: sum of (old - new)^2 for luma and for both chroma planes (filtered_sse / filtered_sse_uv) */
SVT_B200_API int svt_b200_tf_normalize(const SvtB200Frame *dst, const SvtB200TfAccum *acc, int32_t chroma, uint64_t *sse2,
                                       void *stream);
/* One block, HOST pointers in the reference's layout: the body of the drop-ins for the two RTCD pointers (the
 * MeContext-reading shim lives next to the reference's headers: oracle/rtcd_install.c, integration/). */
SVT_B200_API int svt_b200_tf_planewise_block_host(int32_t bit_depth, int32_t chroma, const void *y_src, int32_t y_src_stride,
                                                  const void *y_pre, int32_t y_pre_stride, const void *u_src, const void *v_src,
                                                  int32_t uv_src_stride, const void *u_pre, const void *v_pre,
                                                  int32_t uv_pre_stride, uint32_t bw, uint32_t bh, const double *den3,
                                                  const double *block_error4, const double *d_factor4, uint32_t *y_accum,
                                                  uint16_t *y_count, uint32_t *u_accum, uint16_t *u_count, uint32_t *v_accum,
                                                  uint16_t *v_count);
/* Picture-analysis block statistics of a whole 8-bit picture: per 64x64 SB (raster order) the 85 luma means and
 * variances of compute_block_mean_compute_variance (EbPictureAnalysisProcess.c:1005-2575; entries in EbMeTierZeroPu order,
 * EbMotionEstimationContext.h:51-137 = pcs->y_mean[sb][] / pcs->variance[sb][]), the 21 chroma means per plane of
 * compute_chroma_block_mean (:493-1003; entries 0..20 of pcs->cb_mean[sb][] / cr_mean[sb][]; zero for incomplete SBs as
 * zero_out_chroma_block_mean :432) and pcs->pic_avg_variance (:2929-2974).  full_precision must be 0: the sub-sampled flavour
 * (BLOCK_MEAN_PREC_SUB, EbSequenceControlSet.c:192) is the only one the reference can run - its FULL flavour calls the
 * compute_mean_8x8 RTCD pointer, which no SET_* line of aom_dsp_rtcd.c assigns.  Samples right of / below the picture read as
 * the replicated edge, which is what the reference's padded input picture holds there.  All outputs DEVICE:
 * y_mean [n_sb][85] uint8, variance [n_sb][85] uint16, cb_mean / cr_mean [n_sb][21] uint8 or both NULL, pic_avg_variance
 * one uint16 or NULL (then scratch, 8 bytes of device memory, may be NULL too). */
SVT_B200_API int svt_b200_picture_mean_variance(const SvtB200Frame *pic, int32_t full_precision, uint8_t *y_mean, uint16_t *variance,
                                                uint8_t *cb_mean, uint8_t *cr_mean, uint16_t *pic_avg_variance, void *scratch,
                                                void *stream);
/* the same with HOST planes (sample (0,0) pointers, strides in bytes) and host output arrays; synchronous */
SVT_B200_API int svt_b200_picture_mean_variance_host(const uint8_t *y, int32_t stride_y, const uint8_t *cb, const uint8_t *cr,
                                                     int32_t stride_c, int32_t width, int32_t height, uint8_t *y_mean,
                                                     uint16_t *variance, uint8_t *cb_mean, uint8_t *cr_mean,
                                                     uint16_t *pic_avg_variance);
/* Open-loop intra search of the TPL path (SURVEY.md 8(f) rank 3) for every 16x16 macroblock of an 8-bit picture: replaces
 * the open_loop_intra_search_mb calls of the ME process (EbMotionEstimationProcess.c:965-975; C EbMotionEstimation.c:3043-3155)
 * for the TPL controls of presets >= 5 (tpl_ctrls.tpl_opt_flag = 1, EbPictureDecisionProcess.c:3899-3935), where the mode loop
 * is DC_PRED only.  cost: DEVICE int64 [mb rows][mb cols] with mb cols = (width + 15) / 16 (the reference's mb_stride):
 * OisMbResults::intra_cost; intra_mode is DC_PRED (0) for every macroblock.  The multi-mode search of presets < 5
 * (directional / smooth / Paeth predictors) is not built. */
SVT_B200_API int svt_b200_ois_dc_picture(const SvtB200Frame *pic, int64_t *cost, void *stream);
SVT_B200_API int svt_b200_ois_dc_picture_host(const uint8_t *y, int32_t stride, int32_t width, int32_t height, int64_t *cost);
/* test hook: checksum of the library's expf over the floats with bit patterns lo..hi (see oracle orc_expf_checksum) */
SVT_B200_API int svt_b200_tf_expf_checksum(uint32_t lo_bits, uint32_t hi_bits, uint64_t *out_host);

#ifdef __cplusplus
}
#endif
#endif /* SVT_AV1_B200_H */
