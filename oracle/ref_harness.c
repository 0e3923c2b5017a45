/*
 * ref_harness.c — thin C driver around the UNMODIFIED reference (svt-av1 v0.8.6) compiled into
 * oracle/_ref/libSvtAv1EncRef.so.  TEST INFRASTRUCTURE: it lets the Python tests and bench.py call the
 * reference's own SB-level / frame-level C routines (which take the encoder's internal structs) with plain
 * pointers.  It includes the reference headers from /root/reference at build time (never copied) and is
 * built by Makefile.ref into oracle/_ref/librefharness.so.
 *
 * Every entry sets up exactly the fields the reference routine reads, citing where the encoder itself
 * sets them.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "EbDefinitions.h"
#include "EbSequenceControlSet.h"
#include "EbPictureControlSet.h"
#include "EbPictureBufferDesc.h"
#include "EbMotionEstimationProcess.h"
#include "EbMotionEstimation.h"
#include "EbMotionEstimationContext.h"
#include "EbMotionEstimationLcuResults.h"
#include "EbSystemResourceManager.h"
#include "aom_dsp_rtcd.h"
#include "common_dsp_rtcd.h"

#include "../include/svt_av1_b200.h"

#define REFH_API __attribute__((visibility("default")))

static int g_rtcd_done = 0;
REFH_API void refh_init(void) {
    if (!g_rtcd_done) {
        setup_common_rtcd_internal(0); /* CPU_FLAGS = 0 -> every pointer = the _c function */
        setup_rtcd_internal(0);
        g_rtcd_done = 1;
    }
}

static void plane_desc(EbPictureBufferDesc *d, const SvtB200Plane *g, const uint8_t *buf) {
    memset(d, 0, sizeof(*d));
    d->buffer_y = (uint8_t *)buf;
    d->stride_y = (uint16_t)g->stride;
    d->origin_x = (uint16_t)g->origin_x;
    d->origin_y = (uint16_t)g->origin_y;
    d->width = (uint16_t)g->width;
    d->height = (uint16_t)g->height;
    d->max_width = (uint16_t)g->width;
    d->max_height = (uint16_t)g->height;
    d->bit_depth = EB_8BIT;
}

/* Picture-level state of one ME call: what motion_estimation_kernel's caller sets up before
 * signal_derivation_me_kernel_oq (EbMotionEstimationProcess.c:344) derives the preset's ME/HME parameters. */
typedef struct {
    SequenceControlSet *scs;
    PictureParentControlSet *pcs;
    EbObjectWrapper scs_wrap;
    MotionEstimationContext_t mectx;
    MeContext *me;
} MeSetup;

static MeSetup *me_setup_new(int width, int height, int enc_mode, int n_l0, int n_l1, int temporal_layer, int is_ref) {
    refh_init();
    MeSetup *s = calloc(1, sizeof(*s));
    SequenceControlSet *scs = s->scs = calloc(1, sizeof(*scs));
    PictureParentControlSet *pcs = s->pcs = calloc(1, sizeof(*pcs));
    s->scs_wrap.object_ptr = scs;
    pcs->scs_wrapper_ptr = &s->scs_wrap;

    /* sequence-level fields read by ME (EbEncHandle.c set_param_based_on_input / copy_api_from_app) */
    scs->static_config.use_default_me_hme = EB_TRUE;
    scs->static_config.frame_rate = 30 << 16;
    scs->static_config.enable_global_motion = EB_TRUE;
    scs->static_config.unrestricted_motion_vector = EB_TRUE;
    scs->sb_sz = 64;
    /* derive_input_resolution (EbUtility / EbEncHandle.c) on the luma sample count */
    {
        uint32_t n = (uint32_t)width * (uint32_t)height;
        scs->input_resolution = n < INPUT_SIZE_240p_TH   ? INPUT_SIZE_240p_RANGE
            : n < INPUT_SIZE_360p_TH                     ? INPUT_SIZE_360p_RANGE
            : n < INPUT_SIZE_480p_TH                     ? INPUT_SIZE_480p_RANGE
            : n < INPUT_SIZE_720p_TH                     ? INPUT_SIZE_720p_RANGE
            : n < INPUT_SIZE_1080p_TH                    ? INPUT_SIZE_1080p_RANGE
            : n < INPUT_SIZE_4K_TH                       ? INPUT_SIZE_4K_RANGE
                                                         : INPUT_SIZE_8K_RANGE;
    }
    pcs->enc_mode = (EbEncMode)enc_mode;
    pcs->sc_content_detected = 0;
    pcs->enable_hme_flag = 1; /* EbPictureDecisionProcess.c: hme flags on for all presets by default */
    pcs->enable_hme_level0_flag = 1;
    pcs->enable_hme_level1_flag = 1;
    pcs->enable_hme_level2_flag = 1;
    pcs->is_used_as_reference_flag = (EbBool)is_ref;
    pcs->temporal_layer_index = (uint8_t)temporal_layer;
    pcs->slice_type = n_l1 > 0 ? B_SLICE : P_SLICE;
    pcs->aligned_width = (uint16_t)width;
    pcs->aligned_height = (uint16_t)height;
    pcs->max_number_of_pus_per_sb = SQUARE_PU_COUNT;
    pcs->ref_list0_count_try = (uint8_t)n_l0;
    pcs->ref_list1_count_try = (uint8_t)n_l1;
    pcs->picture_number = 100;

    s->me = calloc(1, sizeof(*s->me));
    me_context_ctor(s->me);
    s->mectx.me_context_ptr = s->me;
    signal_derivation_me_kernel_oq(scs, pcs, &s->mectx);
    return s;
}

static void me_setup_free(MeSetup *s) {
    s->me->dctor(s->me);
    free(s->me);
    free(s->pcs);
    free(s->scs);
    free(s);
}

/* The derived parameters in the C-ABI's plain struct; -3 when the preset uses an HME decimation the ABI
 * does not describe (ONE_DECIMATION_HME: MR / MRS at <= 720p). */
static int me_export_params(const MeSetup *s, int n_l0, int n_l1, const int32_t *ref_dist /*[8]*/, int temporal_layer,
                            int is_ref, const SvtB200Plane *gfull, const SvtB200Plane *gquarter,
                            const SvtB200Plane *gsixteenth, SvtB200MeParams *p) {
    const MeContext *me = s->me;
    memset(p, 0, sizeof(*p));
    p->full = *gfull;
    p->quarter = *gquarter;
    p->sixteenth = *gsixteenth;
    p->num_lists = n_l1 > 0 ? 2 : 1;
    p->num_refs[0] = n_l0;
    p->num_refs[1] = n_l1;
    for (int i = 0; i < 8; i++) p->ref_dist[i / 4][i % 4] = ref_dist[i];
    p->temporal_layer_index = temporal_layer;
    p->is_used_as_reference_flag = is_ref;
    p->enable_hme_flag = me->enable_hme_flag;
    p->enable_hme_level0_flag = me->enable_hme_level0_flag;
    p->enable_hme_level1_flag = me->enable_hme_level1_flag;
    p->enable_hme_level2_flag = me->enable_hme_level2_flag;
    p->hme_search_method = me->hme_search_method == SUB_SAD_SEARCH;
    p->me_search_method = me->me_search_method == SUB_SAD_SEARCH;
    p->number_hme_search_region_in_width = me->number_hme_search_region_in_width;
    p->number_hme_search_region_in_height = me->number_hme_search_region_in_height;
    p->hme_level0_total_search_area_width = me->hme_level0_total_search_area_width;
    p->hme_level0_total_search_area_height = me->hme_level0_total_search_area_height;
    p->hme_level0_max_total_search_area_width = me->hme_level0_max_total_search_area_width;
    p->hme_level0_max_total_search_area_height = me->hme_level0_max_total_search_area_height;
    for (int i = 0; i < 2; i++) {
        p->hme_level0_search_area_in_width_array[i] = me->hme_level0_search_area_in_width_array[i];
        p->hme_level0_search_area_in_height_array[i] = me->hme_level0_search_area_in_height_array[i];
        p->hme_level0_max_search_area_in_width_array[i] = me->hme_level0_max_search_area_in_width_array[i];
        p->hme_level0_max_search_area_in_height_array[i] = me->hme_level0_max_search_area_in_height_array[i];
        p->hme_level1_search_area_in_width_array[i] = me->hme_level1_search_area_in_width_array[i];
        p->hme_level1_search_area_in_height_array[i] = me->hme_level1_search_area_in_height_array[i];
        p->hme_level2_search_area_in_width_array[i] = me->hme_level2_search_area_in_width_array[i];
        p->hme_level2_search_area_in_height_array[i] = me->hme_level2_search_area_in_height_array[i];
    }
    p->search_area_width = me->search_area_width;
    p->search_area_height = me->search_area_height;
    p->max_me_search_width = me->max_me_search_width;
    p->max_me_search_height = me->max_me_search_height;
    p->enable_me_hme_ref_pruning = me->me_hme_prune_ctrls.enable_me_hme_ref_pruning;
    p->prune_ref_if_hme_sad_dev_bigger_than_th = me->me_hme_prune_ctrls.prune_ref_if_hme_sad_dev_bigger_than_th;
    p->prune_ref_if_me_sad_dev_bigger_than_th = me->me_hme_prune_ctrls.prune_ref_if_me_sad_dev_bigger_than_th;
    p->enable_me_sr_adjustment = me->me_sr_adjustment_ctrls.enable_me_sr_adjustment;
    p->reduce_me_sr_based_on_mv_length_th = me->me_sr_adjustment_ctrls.reduce_me_sr_based_on_mv_length_th;
    p->stationary_hme_sad_abs_th = me->me_sr_adjustment_ctrls.stationary_hme_sad_abs_th;
    p->stationary_me_sr_divisor = me->me_sr_adjustment_ctrls.stationary_me_sr_divisor;
    p->reduce_me_sr_based_on_hme_sad_abs_th = me->me_sr_adjustment_ctrls.reduce_me_sr_based_on_hme_sad_abs_th;
    p->me_sr_divisor_for_low_hme_sad = me->me_sr_adjustment_ctrls.me_sr_divisor_for_low_hme_sad;
    p->max_number_of_pus_per_sb = s->pcs->max_number_of_pus_per_sb;
    p->rc_dist_from_8x8 = s->scs->input_resolution <= INPUT_SIZE_480p_RANGE;
    return me->hme_decimation != TWO_DECIMATION_HME ? -3 : 0;
}

/* The preset's ME/HME parameters only, exactly as refh_me_picture derives and exports them, without the search. */
REFH_API int refh_me_params(int width, int height, int enc_mode, int n_l0, int n_l1, const int32_t *ref_dist /*[8]*/,
                            int temporal_layer, int is_ref, const SvtB200Plane *gfull, const SvtB200Plane *gquarter,
                            const SvtB200Plane *gsixteenth, SvtB200MeParams *params_out) {
    MeSetup *s = me_setup_new(width, height, enc_mode, n_l0, n_l1, temporal_layer, is_ref);
    const int rc = me_export_params(s, n_l0, n_l1, ref_dist, temporal_layer, is_ref, gfull, gquarter, gsixteenth, params_out);
    me_setup_free(s);
    return rc;
}

/* Derive the preset's ME/HME parameters (me_setup_new) and run motion_estimate_sb (EbMotionEstimation.c:2912)
 * over every SB of one picture, with the per-SB set-up of motion_estimation_kernel
 * (EbMotionEstimationProcess.c:831-940).  planes: src, then refs[list*4+idx]. */
REFH_API int refh_me_picture(int width, int height, int enc_mode, int n_l0, int n_l1,
                             const int32_t *ref_dist /*[8]*/, int temporal_layer, int is_ref,
                             const SvtB200Plane *gfull, const SvtB200Plane *gquarter,
                             const SvtB200Plane *gsixteenth, const SvtB200MePlanes *src,
                             const SvtB200MePlanes *refs /*[8]*/, SvtB200MeParams *params_out,
                             uint32_t *best_sad, uint32_t *best_mv, SvtB200HmeResult *hme, int16_t *me_mv,
                             uint8_t *me_cand, uint8_t *total_cand, uint32_t *rc_me_distortion) {
    MeSetup *s = me_setup_new(width, height, enc_mode, n_l0, n_l1, temporal_layer, is_ref);
    PictureParentControlSet *pcs = s->pcs;
    MeContext *me = s->me;
    if (params_out) {
        const int rc = me_export_params(s, n_l0, n_l1, ref_dist, temporal_layer, is_ref, gfull, gquarter, gsixteenth,
                                        params_out);
        if (rc) {
            me_setup_free(s);
            return rc;
        }
    }

    const int sbs_x = (width + 63) / 64, sbs_y = (height + 63) / 64, n_sb = sbs_x * sbs_y;
    pcs->sb_total_count = (uint16_t)n_sb;
    pcs->rc_me_distortion = calloc(n_sb, sizeof(uint32_t));
    MotionEstimationData med;
    memset(&med, 0, sizeof(med));
    med.me_results = calloc(n_sb, sizeof(MeSbResults *));
    pcs->pa_me_data = &med;
    for (int i = 0; i < n_sb; i++) {
        med.me_results[i] = calloc(1, sizeof(MeSbResults));
        me_sb_results_ctor(med.me_results[i]);
        /* the ctor mallocs; slots of references that are not searched are never written -> define them */
        memset(med.me_results[i]->me_mv_array, 0, sizeof(MvCandidate) * SQUARE_PU_COUNT * MAX_PA_ME_MV);
        memset(med.me_results[i]->total_me_candidate_index, 0, SQUARE_PU_COUNT);
    }

    EbPictureBufferDesc in_full, in_q, in_s, rf[8], rq[8], rs[8];
    plane_desc(&in_full, gfull, src->full);
    plane_desc(&in_q, gquarter, src->quarter);
    plane_desc(&in_s, gsixteenth, src->sixteenth);
    for (int i = 0; i < 8; i++) {
        plane_desc(&rf[i], gfull, refs[i].full);
        plane_desc(&rq[i], gquarter, refs[i].quarter);
        plane_desc(&rs[i], gsixteenth, refs[i].sixteenth);
    }

    for (int sy = 0; sy < sbs_y; sy++)
        for (int sx = 0; sx < sbs_x; sx++) {
            const int sb = sy * sbs_x + sx;
            const uint32_t ox = sx * 64, oy = sy * 64;
            const uint32_t sb_width = (uint32_t)(width - ox) < 64 ? (uint32_t)(width - ox) : 64;
            /* EbMotionEstimationProcess.c:847-908: load SB + decimated SBs into the context */
            uint32_t bi = (in_full.origin_y + oy) * in_full.stride_y + in_full.origin_x + ox;
            for (unsigned r = 0; r < 64; r++)
                memcpy(&me->sb_buffer[r * 64], &in_full.buffer_y[bi + r * in_full.stride_y], 64);
            me->sb_src_ptr = &in_full.buffer_y[bi];
            me->sb_src_stride = in_full.stride_y;
            bi = (in_q.origin_y + (oy >> 1)) * in_q.stride_y + in_q.origin_x + (ox >> 1);
            for (unsigned r = 0; r < 32; r++)
                memcpy(&me->quarter_sb_buffer[r * me->quarter_sb_buffer_stride],
                       &in_q.buffer_y[bi + r * in_q.stride_y], sb_width >> 1);
            bi = (in_s.origin_y + (oy >> 2)) * in_s.stride_y + in_s.origin_x + (ox >> 2);
            {
                uint8_t *fp = &in_s.buffer_y[bi], *lp = me->sixteenth_sb_buffer;
                const int full = me->hme_search_method == FULL_SAD_SEARCH;
                for (unsigned r = 0; r < 16; r += full ? 1 : 2) {
                    memcpy(lp, fp, sb_width >> 2);
                    lp += 16;
                    fp += in_s.stride_y << (full ? 0 : 1);
                }
            }
            /* :910-940 */
            me->me_type = ME_OPEN_LOOP;
            me->num_of_list_to_search = (pcs->slice_type == P_SLICE) ? REF_LIST_0 : REF_LIST_1;
            me->num_of_ref_pic_to_search[0] = pcs->ref_list0_count_try;
            me->num_of_ref_pic_to_search[1] = pcs->slice_type == B_SLICE ? pcs->ref_list1_count_try : 0;
            me->temporal_layer_index = pcs->temporal_layer_index;
            me->is_used_as_reference_flag = pcs->is_used_as_reference_flag;
            for (int l = 0; l < 2; l++)
                for (int r = 0; r < 4; r++) {
                    me->me_ds_ref_array[l][r].picture_ptr = &rf[l * 4 + r];
                    me->me_ds_ref_array[l][r].quarter_picture_ptr = &rq[l * 4 + r];
                    me->me_ds_ref_array[l][r].sixteenth_picture_ptr = &rs[l * 4 + r];
                    me->me_ds_ref_array[l][r].picture_number = pcs->picture_number - (uint64_t)ref_dist[l * 4 + r];
                }
            memset(me->p_sb_best_sad, 0, sizeof(me->p_sb_best_sad)); /* defined value for unsearched slots */
            motion_estimate_sb(pcs, sb, ox, oy, me, &in_full);

            for (int l = 0; l < 2; l++)
                for (int r = 0; r < 4; r++) {
                    memcpy(best_sad + ((size_t)(sb * 2 + l) * 4 + r) * 85, me->p_sb_best_sad[l][r], 85 * 4);
                    memcpy(best_mv + ((size_t)(sb * 2 + l) * 4 + r) * 85, me->p_sb_best_mv[l][r], 85 * 4);
                    SvtB200HmeResult *h = &hme[(size_t)(sb * 2 + l) * 4 + r];
                    memset(h, 0, sizeof(*h));
                    h->sc_x = me->hme_results[l][r].hme_sc_x;
                    h->sc_y = me->hme_results[l][r].hme_sc_y;
                    h->do_ref = me->hme_results[l][r].do_ref;
                    h->hme_sad = me->hme_results[l][r].hme_sad;
                }
            MeSbResults *res = med.me_results[sb];
            for (int pu = 0; pu < 85; pu++) {
                total_cand[(size_t)sb * 85 + pu] = res->total_me_candidate_index[pu];
                for (int c = 0; c < 23; c++) {
                    uint8_t v = 0;
                    if (c < res->total_me_candidate_index[pu]) {
                        MeCandidate mc = res->me_candidate_array[pu * MAX_PA_ME_CAND + c];
                        /* the index of the list a uni-pred candidate does not use is stale in the reference
                         * (construct_me_candidate_array writes only ref_index[list]); nothing reads it */
                        uint8_t i0 = mc.direction == 1 ? 0 : mc.ref_idx_l0;
                        uint8_t i1 = mc.direction == 0 ? 0 : mc.ref_idx_l1;
                        v = (uint8_t)(mc.direction | (i0 << 2) | (i1 << 4) | (mc.ref0_list << 6) | (mc.ref1_list << 7));
                    }
                    me_cand[((size_t)sb * 85 + pu) * 23 + c] = v;
                }
                for (int m = 0; m < 7; m++) {
                    me_mv[(((size_t)sb * 85 + pu) * 7 + m) * 2] = res->me_mv_array[pu * MAX_PA_ME_MV + m].x_mv;
                    me_mv[(((size_t)sb * 85 + pu) * 7 + m) * 2 + 1] = res->me_mv_array[pu * MAX_PA_ME_MV + m].y_mv;
                }
            }
            rc_me_distortion[sb] = pcs->rc_me_distortion[sb];
        }
    for (int i = 0; i < n_sb; i++) {
        med.me_results[i]->dctor(med.me_results[i]);
        free(med.me_results[i]);
    }
    free(med.me_results);
    free(pcs->rc_me_distortion);
    me_setup_free(s);
    return 0;
}

/* ====================================================================================================
 * CDEF: cdef_seg_search[16bit] (EbCdefProcess.c:80,281) and svt_av1_cdef_frame / av1_cdef_frame16bit
 * (EbEncCdef.c:292,663) on a picture described by plain pointers.
 * ================================================================================================== */
#include "EbCdefProcess.h"
#include "EbEncCdef.h"
#include "EbReferenceObject.h"

void cdef_seg_search(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr, uint32_t segment_index);
void cdef_seg_search16bit(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr, uint32_t segment_index);
void svt_av1_cdef_frame(void *context_ptr, SequenceControlSet *scs_ptr, PictureControlSet *pCs);
void av1_cdef_frame16bit(void *context_ptr, SequenceControlSet *scs_ptr, PictureControlSet *pCs);

typedef struct {
    SequenceControlSet *scs;
    PictureControlSet *pcs;
    PictureParentControlSet *ppcs;
    Av1Common *cm;
    ModeInfo *mi;
    ModeInfo **grid;
    EbPictureBufferDesc recon, input;
    EbObjectWrapper scs_wrap;
} FiltCtx;

/* Picture state shared by the in-loop filter entries. skip8: [ceil(mi_rows/2)][skip_stride]. */
static FiltCtx *filt_ctx_new(int mi_rows, int mi_cols, int bit_depth, const SvtB200Frame *recon,
                             const SvtB200Frame *input, const uint8_t *skip8, int skip_stride,
                             const int8_t *fb_strength_idx) {
    refh_init();
    FiltCtx *c = calloc(1, sizeof(*c));
    c->scs = calloc(1, sizeof(SequenceControlSet));
    c->pcs = calloc(1, sizeof(PictureControlSet));
    c->ppcs = calloc(1, sizeof(PictureParentControlSet));
    c->cm = calloc(1, sizeof(Av1Common));
    c->scs_wrap.object_ptr = c->scs;
    c->pcs->scs_wrapper_ptr = &c->scs_wrap;
    c->pcs->parent_pcs_ptr = c->ppcs;
    c->ppcs->scs_wrapper_ptr = &c->scs_wrap;
    c->ppcs->av1_cm = c->cm;
    c->scs->static_config.encoder_bit_depth = bit_depth;
    c->scs->seq_header.color_config.mono_chrome = 0;
    c->cm->mi_rows = mi_rows;
    c->cm->mi_cols = mi_cols;
    c->cm->mi_stride = mi_cols;
    c->pcs->mi_stride = mi_cols;
    c->ppcs->aligned_width = (uint16_t)(mi_cols * 4);
    c->ppcs->aligned_height = (uint16_t)(mi_rows * 4);
    c->ppcs->is_used_as_reference_flag = EB_FALSE;
    c->mi = calloc((size_t)mi_rows * mi_cols, sizeof(ModeInfo));
    c->grid = calloc((size_t)mi_rows * mi_cols, sizeof(ModeInfo *));
    const int nhfb = (mi_cols + 15) / 16;
    for (int r = 0; r < mi_rows; r++)
        for (int q = 0; q < mi_cols; q++) {
            ModeInfo *m = &c->mi[(size_t)r * mi_cols + q];
            c->grid[(size_t)r * mi_cols + q] = m;
            m->mbmi.block_mi.sb_type = BLOCK_8X8;
            m->mbmi.block_mi.skip = skip8 ? skip8[(r >> 1) * skip_stride + (q >> 1)] : 0;
            m->mbmi.cdef_strength = fb_strength_idx ? fb_strength_idx[(r >> 4) * nhfb + (q >> 4)] : 0;
        }
    c->pcs->mi_grid_base = c->grid;
    const int hbd = bit_depth > 8;
    EbPictureBufferDesc *d[2] = {&c->recon, &c->input};
    const SvtB200Frame *f[2] = {recon, input};
    for (int i = 0; i < 2; i++) {
        if (!f[i]) continue;
        d[i]->buffer_y = f[i]->y;
        d[i]->buffer_cb = f[i]->cb;
        d[i]->buffer_cr = f[i]->cr;
        d[i]->stride_y = (uint16_t)f[i]->stride_y;
        d[i]->stride_cb = d[i]->stride_cr = (uint16_t)f[i]->stride_c;
        d[i]->origin_x = d[i]->origin_y = 0;
        d[i]->width = (uint16_t)(mi_cols * 4);
        d[i]->height = (uint16_t)(mi_rows * 4);
        d[i]->bit_depth = hbd ? EB_10BIT : EB_8BIT;
    }
    c->pcs->recon_picture_ptr = &c->recon;
    c->pcs->recon_picture16bit_ptr = &c->recon;
    c->pcs->input_frame16bit = &c->input;
    c->ppcs->enhanced_picture_ptr = &c->input;
    return c;
}
static void filt_ctx_free(FiltCtx *c) {
    free(c->mi);
    free(c->grid);
    free(c->cm);
    free(c->ppcs);
    free(c->pcs);
    free(c->scs);
    free(c);
}

REFH_API int refh_cdef_search(int mi_rows, int mi_cols, int base_q_idx, int cdef_level, const SvtB200Frame *recon,
                              const SvtB200Frame *source, const uint8_t *skip8, int skip_stride,
                              uint64_t *mse /*[2][nfb][64]*/) {
    FiltCtx *c = filt_ctx_new(mi_rows, mi_cols, recon->bit_depth, recon, source, skip8, skip_stride, NULL);
    const int nfb = ((mi_rows + 15) / 16) * ((mi_cols + 15) / 16);
    c->ppcs->frm_hdr.quantization_params.base_q_idx = (uint8_t)base_q_idx;
    c->ppcs->cdef_level = (int8_t)cdef_level;
    c->pcs->cdef_segments_column_count = 1;
    c->pcs->cdef_segments_row_count = 1;
    c->pcs->cdef_segments_total_count = 1;
    memset(mse, 0, sizeof(uint64_t) * 2 * nfb * 64);
    c->pcs->mse_seg[0] = (uint64_t(*)[TOTAL_STRENGTHS])mse;
    c->pcs->mse_seg[1] = (uint64_t(*)[TOTAL_STRENGTHS])(mse + (size_t)nfb * 64);
    c->pcs->src[0] = recon->y;
    c->pcs->src[1] = recon->cb;
    c->pcs->src[2] = recon->cr;
    c->pcs->ref_coeff[0] = source->y;
    c->pcs->ref_coeff[1] = source->cb;
    c->pcs->ref_coeff[2] = source->cr;
    if (recon->bit_depth > 8)
        cdef_seg_search16bit(c->pcs, c->scs, 0);
    else
        cdef_seg_search(c->pcs, c->scs, 0);
    filt_ctx_free(c);
    return 0;
}

/* in place on `recon` (the reference's behaviour) */
/* finish_cdef_search (EbEncCdef.c:1167) on a given mse table: frame header fields, per-filter-block choice, and the lambda the
 * reference derived for the picture (the oracle takes it as an input). */
#include "EbEncDecProcess.h"
#include "EbModeDecisionProcess.h"
void finish_cdef_search(EncDecContext *context_ptr, PictureControlSet *pcs_ptr, int32_t selected_strength_cnt[64]);
REFH_API int refh_cdef_finish(int mi_rows, int mi_cols, int base_q_idx, int cdef_level, int bit_depth, const uint8_t *skip8,
                              int skip_stride, const uint64_t *mse, int32_t *cdef_bits, int32_t *nb_strengths, int32_t *y_strength8,
                              int32_t *uv_strength8, int8_t *fb_strength, uint64_t *lambda_out) {
    SvtB200Frame dummy;
    memset(&dummy, 0, sizeof(dummy));
    dummy.bit_depth = bit_depth;
    FiltCtx *c = filt_ctx_new(mi_rows, mi_cols, bit_depth, &dummy, &dummy, skip8, skip_stride, NULL);
    const int nfb = ((mi_rows + 15) / 16) * ((mi_cols + 15) / 16), nhfb = (mi_cols + 15) / 16;
    c->ppcs->frm_hdr.quantization_params.base_q_idx = (uint8_t)base_q_idx;
    c->ppcs->cdef_level = (int8_t)cdef_level;
    c->ppcs->pred_structure = 0;
    uint64_t *copy = (uint64_t *)malloc(sizeof(uint64_t) * 2 * nfb * 64);
    memcpy(copy, mse, sizeof(uint64_t) * 2 * nfb * 64);
    c->pcs->mse_seg[0] = (uint64_t(*)[TOTAL_STRENGTHS])copy;
    c->pcs->mse_seg[1] = (uint64_t(*)[TOTAL_STRENGTHS])(copy + (size_t)nfb * 64);
    for (int i = 0; i < mi_rows * mi_cols; i++) c->mi[i].mbmi.cdef_strength = -1;
    uint32_t fast_lambda = 0, full_lambda = 0;
    (*av1_lambda_assignment_function_table[0])(c->pcs, &fast_lambda, &full_lambda, (uint8_t)c->input.bit_depth, (uint16_t)(uint8_t)base_q_idx, EB_FALSE);
    *lambda_out = full_lambda;
    int32_t cnt[64] = {0};
    finish_cdef_search(0, c->pcs, cnt);
    *cdef_bits = c->ppcs->frm_hdr.cdef_params.cdef_bits;
    *nb_strengths = c->ppcs->nb_cdef_strengths;
    for (int i = 0; i < 8; i++) {
        y_strength8[i] = c->ppcs->frm_hdr.cdef_params.cdef_y_strength[i];
        uv_strength8[i] = c->ppcs->frm_hdr.cdef_params.cdef_uv_strength[i];
    }
    for (int fb = 0; fb < nfb; fb++) fb_strength[fb] = c->mi[(size_t)(16 * (fb / nhfb)) * mi_cols + 16 * (fb % nhfb)].mbmi.cdef_strength;
    free(copy);
    filt_ctx_free(c);
    return 0;
}

REFH_API int refh_cdef_apply(int mi_rows, int mi_cols, int damping, const int32_t *y_strength,
                             const int32_t *uv_strength, SvtB200Frame *recon, const uint8_t *skip8, int skip_stride,
                             const int8_t *fb_strength_idx) {
    FiltCtx *c = filt_ctx_new(mi_rows, mi_cols, recon->bit_depth, recon, NULL, skip8, skip_stride, fb_strength_idx);
    c->ppcs->frm_hdr.cdef_params.cdef_damping = (uint8_t)damping;
    for (int i = 0; i < 8; i++) {
        c->ppcs->frm_hdr.cdef_params.cdef_y_strength[i] = y_strength[i];
        c->ppcs->frm_hdr.cdef_params.cdef_uv_strength[i] = uv_strength[i];
    }
    if (recon->bit_depth > 8)
        av1_cdef_frame16bit(NULL, c->scs, c->pcs);
    else
        svt_av1_cdef_frame(NULL, c->scs, c->pcs);
    filt_ctx_free(c);
    return 0;
}

/* ====================================================================================================
 * scan orders: av1_scan_orders[tx_size][tx_type] is a static table in a header (Common/Codec/EbCoefficients.h:2563)
 * ================================================================================================== */
#include "EbCoefficients.h"
REFH_API int refh_get_scan(int tx_size, int tx_type, int16_t *out) {
    const ScanOrder *so = &av1_scan_orders[tx_size][tx_type];
    int w = tx_size_wide[tx_size], h = tx_size_high[tx_size];
    if (w > 32) w = 32;
    if (h > 32) h = 32;
    memcpy(out, so->scan, sizeof(int16_t) * w * h);
    return w * h;
}

/* ====================================================================================================
 * Deblocking: svt_av1_loop_filter_frame (EbDeblockingFilter.c:711) on a picture whose ModeInfo grid is built
 * from per-mi arrays (sb_type, tx_depth, is_inter, skip).  Also emits the flattened SvtB200DlfMi summary with
 * the reference's own tables/inline helpers — what the integration overlay computes inside the reference.
 * ================================================================================================== */
#include "EbDeblockingFilter.h"
#include "EbUtility.h"
void svt_av1_loop_filter_init(PictureControlSet *pcs_ptr);

static FiltCtx *dlf_ctx(int mi_rows, int mi_cols, const uint8_t *sb_type, const uint8_t *tx_depth, const uint8_t *is_inter,
                        const uint8_t *skip, const int32_t *levels /*y0,y1,u,v*/, int sharpness, SvtB200Frame *frame,
                        const SvtB200Frame *source, SvtB200DlfMi *flat /*[mi_rows][mi_cols]*/) {
    FiltCtx *c = filt_ctx_new(mi_rows, mi_cols, frame->bit_depth, frame, source, NULL, 0, NULL);
    c->ppcs->scs_ptr = c->scs;
    c->scs->seq_header.sb_size = BLOCK_64X64;
    c->scs->sb_size_pix = 64;
    c->scs->max_input_luma_width = (uint16_t)(mi_cols * 4);
    c->scs->max_input_luma_height = (uint16_t)(mi_rows * 4);
    c->scs->max_input_pad_right = 0;
    c->scs->max_input_pad_bottom = 0;
    c->scs->subsampling_x = c->scs->subsampling_y = 1;
    struct LoopFilter *lf = &c->ppcs->frm_hdr.loop_filter_params;
    lf->filter_level[0] = levels[0];
    lf->filter_level[1] = levels[1];
    lf->filter_level_u = levels[2];
    lf->filter_level_v = levels[3];
    lf->sharpness_level = sharpness;
    lf->mode_ref_delta_enabled = 0;
    c->ppcs->frm_hdr.delta_lf_params.delta_lf_present = 0;
    for (int r = 0; r < mi_rows; r++)
        for (int q = 0; q < mi_cols; q++) {
            const size_t i = (size_t)r * mi_cols + q;
            ModeInfo *m = &c->mi[i];
            m->mbmi.block_mi.sb_type = (BlockSize)sb_type[i];
            m->mbmi.tx_depth = tx_depth[i];
            m->mbmi.block_mi.ref_frame[0] = is_inter[i] ? LAST_FRAME : INTRA_FRAME;
            m->mbmi.block_mi.skip = skip[i];
            m->mbmi.block_mi.mode = is_inter[i] ? NEARESTMV : DC_PRED;
            if (flat) {
                SvtB200DlfMi *f = &flat[i];
                memset(f, 0, sizeof(*f));
                const BlockSize bs = (BlockSize)sb_type[i];
                TxSize tx = is_inter[i] ? tx_depth_to_tx_size[0][bs] : tx_depth_to_tx_size[tx_depth[i]][bs];
                if (is_inter[i] && !skip[i]) tx = tx_depth_to_tx_size[tx_depth[i]][bs];
                const TxSize uv = av1_get_max_uv_txsize(bs, 1, 1);
                f->tx_w[0] = (uint8_t)tx_size_wide[txsize_horz_map[tx]];
                f->tx_h[0] = (uint8_t)tx_size_high[txsize_vert_map[tx]];
                f->tx_w[1] = (uint8_t)tx_size_wide[txsize_horz_map[uv]];
                f->tx_h[1] = (uint8_t)tx_size_high[txsize_vert_map[uv]];
                const BlockSize cb = get_plane_block_size(bs, 1, 1);
                f->blk_w[0] = block_size_wide[bs];
                f->blk_h[0] = block_size_high[bs];
                f->blk_w[1] = block_size_wide[cb];
                f->blk_h[1] = block_size_high[cb];
                f->skip_inter = skip[i] && is_inter[i];
                f->lvl_y[0] = (uint8_t)levels[0]; /* lfi_n->lvl[..]: no ref/mode deltas, no segmentation */
                f->lvl_y[1] = (uint8_t)levels[1];
                f->lvl_u = (uint8_t)levels[2];
                f->lvl_v = (uint8_t)levels[3];
                /* segment 0, ref_frame[0], mode_lf_lut[mode] (NEARESTMV -> 1, DC_PRED -> 0) */
                f->lvl_class = (uint8_t)((is_inter[i] ? LAST_FRAME : INTRA_FRAME) * 2 + (is_inter[i] ? 1 : 0));
            }
        }
    svt_av1_loop_filter_init(c->pcs);
    c->recon.bit_depth = frame->bit_depth > 8 ? EB_10BIT : EB_8BIT;
    c->recon.width = (uint16_t)(mi_cols * 4);
    c->recon.height = (uint16_t)(mi_rows * 4);
    return c;
}

REFH_API int refh_dlf_frame(int mi_rows, int mi_cols, const uint8_t *sb_type, const uint8_t *tx_depth,
                            const uint8_t *is_inter, const uint8_t *skip, const int32_t *levels /*y0,y1,u,v*/,
                            int sharpness, SvtB200Frame *frame, SvtB200DlfMi *flat /*[mi_rows][mi_cols]*/) {
    FiltCtx *c = dlf_ctx(mi_rows, mi_cols, sb_type, tx_depth, is_inter, skip, levels, sharpness, frame, NULL, flat);
    svt_av1_loop_filter_frame(&c->recon, c->pcs, 0, 3);
    filt_ctx_free(c);
    return 0;
}

/* svt_av1_pick_filter_level (EbDeblockingFilter.c:1193) on the same picture description; `temp` is the DlfContext's
 * temp_lf_recon_picture; mode_ref_delta (ref_deltas / mode_deltas) optional. */
#include "EbDlfProcess.h"
REFH_API int refh_pick_filter_level(int mi_rows, int mi_cols, const uint8_t *sb_type, const uint8_t *tx_depth,
                                    const uint8_t *is_inter, const uint8_t *skip, const int32_t *last_levels, int method,
                                    int loop_filter_mode, int tx_mode_only_4x4, int base_q_idx, int key_frame,
                                    const int8_t *ref_deltas /*8 or NULL*/, const int8_t *mode_deltas /*2*/,
                                    SvtB200Frame *recon, const SvtB200Frame *source, SvtB200Frame *temp, int32_t *levels_out) {
    FiltCtx *c = dlf_ctx(mi_rows, mi_cols, sb_type, tx_depth, is_inter, skip, last_levels, 0, recon, source, NULL);
    FrameHeader *fh = &c->ppcs->frm_hdr;
    c->ppcs->loop_filter_mode = (uint8_t)loop_filter_mode;
    fh->tx_mode = tx_mode_only_4x4 ? ONLY_4X4 : TX_MODE_SELECT;
    fh->quantization_params.base_q_idx = (uint8_t)base_q_idx;
    fh->frame_type = key_frame ? KEY_FRAME : INTER_FRAME;
    if (ref_deltas) {
        fh->loop_filter_params.mode_ref_delta_enabled = 1;
        for (int i = 0; i < 8; i++) fh->loop_filter_params.ref_deltas[i] = ref_deltas[i];
        for (int i = 0; i < 2; i++) fh->loop_filter_params.mode_deltas[i] = mode_deltas[i];
    }
    DlfContext ctx;
    memset(&ctx, 0, sizeof(ctx));
    EbPictureBufferDesc tdesc = c->recon;
    tdesc.buffer_y = temp->y;
    tdesc.buffer_cb = temp->cb;
    tdesc.buffer_cr = temp->cr;
    tdesc.stride_y = (uint16_t)temp->stride_y;
    tdesc.stride_cb = tdesc.stride_cr = (uint16_t)temp->stride_c;
    ctx.temp_lf_recon_picture_ptr = &tdesc;
    ctx.temp_lf_recon_picture16bit_ptr = &tdesc;
    svt_av1_pick_filter_level(&ctx, &c->input, c->pcs, (LpfPickMethod)method);
    levels_out[0] = fh->loop_filter_params.filter_level[0];
    levels_out[1] = fh->loop_filter_params.filter_level[1];
    levels_out[2] = fh->loop_filter_params.filter_level_u;
    levels_out[3] = fh->loop_filter_params.filter_level_v;
    filt_ctx_free(c);
    return 0;
}

/* ====================================================================================================
 * Loop restoration, frame level: svt_av1_loop_restoration_save_boundary_lines (after deblocking and after CDEF) +
 * svt_av1_loop_restoration_filter_frame, on Yv12BufferConfig views of our frames (which must carry a border of at
 * least 8 samples: the reference extends / overwrites it in place).  `cdef` is filtered in place.
 * ================================================================================================== */
#include "EbRestoration.h"
static void yv12_view(Yv12BufferConfig *y, const SvtB200Frame *f, int hbd) {
    memset(y, 0, sizeof(*y));
    const int w = f->width, h = f->height;
    y->y_width = (w + 7) & ~7;
    y->y_height = (h + 7) & ~7;
    y->uv_width = y->y_width >> 1;
    y->uv_height = y->y_height >> 1;
    y->y_crop_width = w;
    y->y_crop_height = h;
    y->uv_crop_width = (w + 1) >> 1;
    y->uv_crop_height = (h + 1) >> 1;
    y->y_stride = f->stride_y;
    y->uv_stride = f->stride_c;
    y->y_buffer = hbd ? CONVERT_TO_BYTEPTR(f->y) : (uint8_t *)f->y;
    y->u_buffer = hbd ? CONVERT_TO_BYTEPTR(f->cb) : (uint8_t *)f->cb;
    y->v_buffer = hbd ? CONVERT_TO_BYTEPTR(f->cr) : (uint8_t *)f->cr;
    y->subsampling_x = y->subsampling_y = 1;
    y->bit_depth = (uint32_t)f->bit_depth;
    y->flags = hbd ? YV12_FLAG_HIGHBITDEPTH : 0;
    y->border = 8;
}
REFH_API int refh_lr_frame(SvtB200Frame *cdef, const SvtB200Frame *dblk, const int32_t *frame_types, const int32_t *unit_sizes,
                           const SvtB200LrUnit *const *units /*[3] host arrays*/, int optimized_lr) {
    refh_init();
    const int hbd = cdef->bit_depth > 8;
    Av1Common *cm = calloc(1, sizeof(Av1Common));
    cm->use_highbitdepth = hbd;
    cm->bit_depth = cdef->bit_depth;
    cm->subsampling_x = cm->subsampling_y = 1;
    cm->mi_rows = (cdef->height + 3) >> 2;
    cm->mi_cols = (cdef->width + 3) >> 2;
    cm->frm_size.frame_width = cm->frm_size.superres_upscaled_width = (uint16_t)cdef->width;
    cm->frm_size.frame_height = cm->frm_size.superres_upscaled_height = (uint16_t)cdef->height;
    cm->frm_size.superres_denominator = 8;
    for (int p = 0; p < 3; p++) {
        cm->rst_info[p].frame_restoration_type = (RestorationType)frame_types[p];
        cm->rst_info[p].restoration_unit_size = unit_sizes[p];
    }
    if (svt_av1_alloc_restoration_buffers(cm) != EB_ErrorNone) return -1;
    cm->rst_tmpbuf = (int32_t *)svt_aom_memalign(16, RESTORATION_TMPBUF_SIZE);
    for (int p = 0; p < 3; p++) {
        RestorationInfo *rsi = &cm->rst_info[p];
        for (int i = 0; i < rsi->units_per_tile; i++) {
            RestorationUnitInfo *ri = &rsi->unit_info[i];
            const SvtB200LrUnit *u = &units[p][i];
            ri->restoration_type = (RestorationType)u->restoration_type;
            for (int k = 0; k < 8; k++) {
                ri->wiener_info.vfilter[k] = u->vfilter[k];
                ri->wiener_info.hfilter[k] = u->hfilter[k];
            }
            ri->sgrproj_info.ep = u->sgr_ep;
            ri->sgrproj_info.xqd[0] = u->sgr_xqd[0];
            ri->sgrproj_info.xqd[1] = u->sgr_xqd[1];
        }
    }
    Yv12BufferConfig fc, fd;
    yv12_view(&fc, cdef, hbd);
    yv12_view(&fd, dblk, hbd);
    svt_av1_loop_restoration_save_boundary_lines(&fd, cm, 0);
    svt_av1_loop_restoration_save_boundary_lines(&fc, cm, 1);
    svt_av1_loop_restoration_filter_frame(&fc, cm, optimized_lr);
    for (int p = 0; p < 3; p++) {
        free(cm->rst_info[p].unit_info);
        free(cm->rst_info[p].boundaries.stripe_boundary_above);
        free(cm->rst_info[p].boundaries.stripe_boundary_below);
    }
    svt_aom_free(cm->rst_tmpbuf);
    free(cm);
    return 0;
}
REFH_API int refh_lr_units(int width, int height, int plane, int unit_size, int *hunits, int *vunits) {
    Av1Common cm;
    memset(&cm, 0, sizeof(cm));
    cm.subsampling_x = cm.subsampling_y = 1;
    cm.frm_size.frame_width = cm.frm_size.superres_upscaled_width = (uint16_t)width;
    cm.frm_size.frame_height = cm.frm_size.superres_upscaled_height = (uint16_t)height;
    RestorationInfo rsi;
    memset(&rsi, 0, sizeof(rsi));
    rsi.restoration_unit_size = unit_size;
    if (svt_av1_alloc_restoration_struct(&cm, &rsi, plane > 0) != EB_ErrorNone) return -1;
    *hunits = rsi.horz_units_per_tile;
    *vunits = rsi.vert_units_per_tile;
    free(rsi.unit_info);
    return rsi.units_per_tile;
}

/* ====================================================================================================
 * EncDec per-TU chain with the reference's own kernels, through its RTCD pointers (C paths):
 *   svt_residual_kernel8bit/16bit -> svt_av1_fwd_txfm2d_* (+ svt_handle_transform*) -> svt_aom_[highbd_]quantize_b or
 *   svt_av1_[highbd_]quantize_fp -> svt_av1_inv_txfm2d_add_*   (the body of av1_encode_loop, EbCodingLoop.c:290-...)
 * ================================================================================================== */
static void ref_fwd(int tx_size, int16_t *res, int32_t *coeff, uint32_t stride, TxType tt, uint8_t bd) {
    switch (tx_size) {
    case TX_4X4: svt_av1_fwd_txfm2d_4x4(res, coeff, stride, tt, bd); break;
    case TX_8X8: svt_av1_fwd_txfm2d_8x8(res, coeff, stride, tt, bd); break;
    case TX_16X16: svt_av1_fwd_txfm2d_16x16(res, coeff, stride, tt, bd); break;
    case TX_32X32: svt_av1_fwd_txfm2d_32x32(res, coeff, stride, tt, bd); break;
    case TX_64X64: svt_av1_fwd_txfm2d_64x64(res, coeff, stride, tt, bd); svt_handle_transform64x64(coeff); break;
    case TX_4X8: svt_av1_fwd_txfm2d_4x8(res, coeff, stride, tt, bd); break;
    case TX_8X4: svt_av1_fwd_txfm2d_8x4(res, coeff, stride, tt, bd); break;
    case TX_8X16: svt_av1_fwd_txfm2d_8x16(res, coeff, stride, tt, bd); break;
    case TX_16X8: svt_av1_fwd_txfm2d_16x8(res, coeff, stride, tt, bd); break;
    case TX_16X32: svt_av1_fwd_txfm2d_16x32(res, coeff, stride, tt, bd); break;
    case TX_32X16: svt_av1_fwd_txfm2d_32x16(res, coeff, stride, tt, bd); break;
    case TX_32X64: svt_av1_fwd_txfm2d_32x64(res, coeff, stride, tt, bd); svt_handle_transform32x64(coeff); break;
    case TX_64X32: svt_av1_fwd_txfm2d_64x32(res, coeff, stride, tt, bd); svt_handle_transform64x32(coeff); break;
    case TX_4X16: svt_av1_fwd_txfm2d_4x16(res, coeff, stride, tt, bd); break;
    case TX_16X4: svt_av1_fwd_txfm2d_16x4(res, coeff, stride, tt, bd); break;
    case TX_8X32: svt_av1_fwd_txfm2d_8x32(res, coeff, stride, tt, bd); break;
    case TX_32X8: svt_av1_fwd_txfm2d_32x8(res, coeff, stride, tt, bd); break;
    case TX_16X64: svt_av1_fwd_txfm2d_16x64(res, coeff, stride, tt, bd); svt_handle_transform16x64(coeff); break;
    default: svt_av1_fwd_txfm2d_64x16(res, coeff, stride, tt, bd); svt_handle_transform64x16(coeff); break;
    }
}
static void ref_inv(int tx_size, const int32_t *dq, uint16_t *pr, int sr, uint16_t *rc, int sw, TxType tt, int eob, int bd) {
    switch (tx_size) {
    case TX_4X4: svt_av1_inv_txfm2d_add_4x4(dq, pr, sr, rc, sw, tt, bd); break;
    case TX_8X8: svt_av1_inv_txfm2d_add_8x8(dq, pr, sr, rc, sw, tt, bd); break;
    case TX_16X16: svt_av1_inv_txfm2d_add_16x16(dq, pr, sr, rc, sw, tt, bd); break;
    case TX_32X32: svt_av1_inv_txfm2d_add_32x32(dq, pr, sr, rc, sw, tt, bd); break;
    case TX_64X64: svt_av1_inv_txfm2d_add_64x64(dq, pr, sr, rc, sw, tt, bd); break;
    case TX_4X8: svt_av1_inv_txfm2d_add_4x8(dq, pr, sr, rc, sw, tt, TX_4X8, bd); break;
    case TX_8X4: svt_av1_inv_txfm2d_add_8x4(dq, pr, sr, rc, sw, tt, TX_8X4, bd); break;
    case TX_8X16: svt_av1_inv_txfm2d_add_8x16(dq, pr, sr, rc, sw, tt, TX_8X16, eob, bd); break;
    case TX_16X8: svt_av1_inv_txfm2d_add_16x8(dq, pr, sr, rc, sw, tt, TX_16X8, eob, bd); break;
    case TX_16X32: svt_av1_inv_txfm2d_add_16x32(dq, pr, sr, rc, sw, tt, TX_16X32, eob, bd); break;
    case TX_32X16: svt_av1_inv_txfm2d_add_32x16(dq, pr, sr, rc, sw, tt, TX_32X16, eob, bd); break;
    case TX_32X64: svt_av1_inv_txfm2d_add_32x64(dq, pr, sr, rc, sw, tt, TX_32X64, eob, bd); break;
    case TX_64X32: svt_av1_inv_txfm2d_add_64x32(dq, pr, sr, rc, sw, tt, TX_64X32, eob, bd); break;
    case TX_4X16: svt_av1_inv_txfm2d_add_4x16(dq, pr, sr, rc, sw, tt, TX_4X16, bd); break;
    case TX_16X4: svt_av1_inv_txfm2d_add_16x4(dq, pr, sr, rc, sw, tt, TX_16X4, bd); break;
    case TX_8X32: svt_av1_inv_txfm2d_add_8x32(dq, pr, sr, rc, sw, tt, TX_8X32, eob, bd); break;
    case TX_32X8: svt_av1_inv_txfm2d_add_32x8(dq, pr, sr, rc, sw, tt, TX_32X8, eob, bd); break;
    case TX_16X64: svt_av1_inv_txfm2d_add_16x64(dq, pr, sr, rc, sw, tt, TX_16X64, eob, bd); break;
    default: svt_av1_inv_txfm2d_add_64x16(dq, pr, sr, rc, sw, tt, TX_64X16, eob, bd); break;
    }
}

/* The reference's own dispatcher (EbTransforms.c:3613): every shape, every size, through its RTCD pointers. */
#include "EbTransforms.h"
REFH_API uint64_t refh_estimate_transform(int16_t *res, uint32_t stride, int32_t *coeff, int tx_size, int bit_depth, int tx_type,
                                          int shape) {
    refh_init();
    uint64_t energy = 0;
    av1_estimate_transform(res, stride, coeff, 0, (TxSize)tx_size, &energy, (uint32_t)bit_depth, (TxType)tx_type, PLANE_TYPE_Y,
                           (EB_TRANS_COEFF_SHAPE)shape);
    return energy;
}

REFH_API int refh_encode_tus(const SvtB200EncodeParams *p, const SvtB200Frame *src, const SvtB200Frame *pred,
                             const SvtB200Frame *recon, const SvtB200Tu *tus, int n_tus, int32_t *qcoeff, uint16_t *eobs) {
    refh_init();
    const int ts = p->tx_size, w = tx_size_wide[ts], h = tx_size_high[ts];
    const int iw = w > 32 ? 32 : w, ih = h > 32 ? 32 : h, n = iw * ih;
    const int bd = src->bit_depth, hbd = bd > 8;
    const int log_scale = (w * h > 256) + (w * h > 1024);
    int16_t res[64 * 64];
    int32_t coeff[64 * 64], dq[32 * 32];
    uint16_t p16[64 * 64], r16[64 * 64];
    for (int i = 0; i < n_tus; i++) {
        const SvtB200Tu *t = &tus[i];
        const int pl = t->plane;
        const int ss = pl ? src->stride_c : src->stride_y, ps = pl ? pred->stride_c : pred->stride_y,
                  rs = pl ? recon->stride_c : recon->stride_y;
        const void *sp = pl == 0 ? src->y : pl == 1 ? src->cb : src->cr;
        const void *pp = pl == 0 ? pred->y : pl == 1 ? pred->cb : pred->cr;
        void *rp = pl == 0 ? recon->y : pl == 1 ? recon->cb : recon->cr;
        if (hbd)
            svt_residual_kernel16bit((uint16_t *)sp + (size_t)t->y * ss + t->x, ss, (uint16_t *)pp + (size_t)t->y * ps + t->x, ps,
                                     res, w, w, h);
        else
            svt_residual_kernel8bit((uint8_t *)sp + (size_t)t->y * ss + t->x, ss, (uint8_t *)pp + (size_t)t->y * ps + t->x, ps, res,
                                    w, w, h);
        ref_fwd(ts, res, coeff, w, (TxType)t->tx_type, (uint8_t)bd);
        const ScanOrder *so = &av1_scan_orders[ts][t->tx_type];
        const SvtB200QuantPlane *q = &p->q[pl];
        int32_t *qc = qcoeff + (size_t)i * n;
        uint16_t eob = 0;
        if (p->use_fp) {
            if (hbd)
                svt_av1_highbd_quantize_fp(coeff, n, q->zbin, q->round_fp, q->quant_fp, q->quant_shift, qc, dq, q->dequant, &eob,
                                           so->scan, so->iscan, (int16_t)log_scale);
            else if (log_scale == 0)
                svt_av1_quantize_fp(coeff, n, q->zbin, q->round_fp, q->quant_fp, q->quant_shift, qc, dq, q->dequant, &eob, so->scan, so->iscan);
            else if (log_scale == 1)
                svt_av1_quantize_fp_32x32(coeff, n, q->zbin, q->round_fp, q->quant_fp, q->quant_shift, qc, dq, q->dequant, &eob, so->scan, so->iscan);
            else
                svt_av1_quantize_fp_64x64(coeff, n, q->zbin, q->round_fp, q->quant_fp, q->quant_shift, qc, dq, q->dequant, &eob, so->scan, so->iscan);
        } else if (hbd) {
            svt_aom_highbd_quantize_b(coeff, n, q->zbin, q->round, q->quant, q->quant_shift, qc, dq, q->dequant, &eob, so->scan,
                                      so->iscan, NULL, NULL, log_scale);
        } else {
            svt_aom_quantize_b(coeff, n, q->zbin, q->round, q->quant, q->quant_shift, qc, dq, q->dequant, &eob, so->scan, so->iscan,
                               NULL, NULL, log_scale);
        }
        eobs[i] = eob;
        /* inverse + reconstruction through the 16-bit kernels (the lowbd wrapper svt_av1_inv_txfm_add_c copies the
         * 8-bit prediction into a 16-bit scratch the same way, EbInvTransforms.c:3302-3330) */
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++)
                p16[y * w + x] = hbd ? ((uint16_t *)pp)[(size_t)(t->y + y) * ps + t->x + x] : ((uint8_t *)pp)[(size_t)(t->y + y) * ps + t->x + x];
        ref_inv(ts, dq, p16, w, r16, w, (TxType)t->tx_type, eob, bd);
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                if (hbd)
                    ((uint16_t *)rp)[(size_t)(t->y + y) * rs + t->x + x] = r16[y * w + x];
                else
                    ((uint8_t *)rp)[(size_t)(t->y + y) * rs + t->x + x] = (uint8_t)r16[y * w + x];
            }
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------------------------------ */
/* Inter prediction: the reference's sixteen convolve functions by index, its kernel tables, and                      */
/* enc_make_inter_predictor per job of svt_b200_inter_predict.                                                        */
/* ------------------------------------------------------------------------------------------------------------------ */
#include "EbInterPrediction.h"
#include "EbCodingUnit.h"
#include "convolve.h"

void enc_make_inter_predictor(uint8_t *src_ptr, uint8_t *dst_ptr, int16_t pre_y, int16_t pre_x, MV mv,
                              const struct ScaleFactors *const sf, ConvolveParams *conv_params, InterpFilters interp_filters,
                              InterInterCompoundData *interinter_comp, uint16_t frame_width, uint16_t frame_height,
                              uint8_t blk_width, uint8_t blk_height, BlockSize bsize, MacroBlockD *av1xd, int32_t src_stride,
                              int32_t dst_stride, uint8_t plane, const uint32_t ss_y, const uint32_t ss_x, uint8_t bit_depth,
                              uint8_t use_intrabc, uint8_t is_masked_compound, uint8_t is16bit); /* EbEncInterPrediction.c:3663 */
void asm_set_convolve_asm_table(void);
void asm_set_convolve_hbd_asm_table(void);

REFH_API void refh_interp_kernel(int filter, int w, int subpel, int16_t out[8]) {
    InterpFilterParams p = av1_get_interp_filter_params_with_block_size((InterpFilter)filter, w);
    memcpy(out, p.filter_ptr + 8 * (subpel & 15), 16);
}

/* which = sx * 4 + sy * 2 + compound, the index order of convolve[sx][sy][is_compound] (EbInterPrediction.c:1162-1175) */
REFH_API void refh_convolve(int which, int hbd, const void *src, int src_stride, void *dst, int dst_stride, int w, int h,
                            int filter_x, int filter_y, int subpel_x, int subpel_y, int round_0, int round_1, int do_average,
                            int use_jnt, int fwd_offset, int bck_offset, uint16_t *conv_dst, int conv_stride, int bd) {
    static const AomConvolveFn lo[8] = {svt_av1_convolve_2d_copy_sr_c, svt_av1_jnt_convolve_2d_copy_c, svt_av1_convolve_y_sr_c,
                                        svt_av1_jnt_convolve_y_c,      svt_av1_convolve_x_sr_c,        svt_av1_jnt_convolve_x_c,
                                        svt_av1_convolve_2d_sr_c,      svt_av1_jnt_convolve_2d_c};
    static const aom_highbd_convolve_fn_t hi[8] = {
        svt_av1_highbd_convolve_2d_copy_sr_c, svt_av1_highbd_jnt_convolve_2d_copy_c, svt_av1_highbd_convolve_y_sr_c,
        svt_av1_highbd_jnt_convolve_y_c,      svt_av1_highbd_convolve_x_sr_c,        svt_av1_highbd_jnt_convolve_x_c,
        svt_av1_highbd_convolve_2d_sr_c,      svt_av1_highbd_jnt_convolve_2d_c};
    InterpFilterParams px = av1_get_interp_filter_params_with_block_size((InterpFilter)filter_x, w);
    InterpFilterParams py = av1_get_interp_filter_params_with_block_size((InterpFilter)filter_y, h);
    ConvolveParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.do_average = do_average;
    cp.dst = conv_dst;
    cp.dst_stride = conv_stride;
    cp.round_0 = round_0;
    cp.round_1 = round_1;
    cp.is_compound = which & 1;
    cp.use_jnt_comp_avg = cp.use_dist_wtd_comp_avg = use_jnt;
    cp.fwd_offset = fwd_offset;
    cp.bck_offset = bck_offset;
    if (hbd)
        hi[which]((const uint16_t *)src, src_stride, (uint16_t *)dst, dst_stride, w, h, &px, &py, subpel_x, subpel_y, &cp, bd);
    else
        lo[which]((const uint8_t *)src, src_stride, (uint8_t *)dst, dst_stride, w, h, &px, &py, subpel_x, subpel_y, &cp);
}

REFH_API void refh_convolve8(const uint8_t *src, ptrdiff_t src_stride, uint8_t *dst, ptrdiff_t dst_stride, int filter, int q0,
                             int step, int w, int h, int vert) {
    InterpFilterParams p = av1_get_interp_filter_params_with_block_size((InterpFilter)filter, 8);
    const int16_t *f = p.filter_ptr + 8 * q0; /* the tables are 256-byte aligned (EbInterPrediction.c:258) */
    if (vert)
        svt_aom_convolve8_vert_c(src, src_stride, dst, dst_stride, NULL, 0, f, step, w, h);
    else
        svt_aom_convolve8_horiz_c(src, src_stride, dst, dst_stride, f, step, NULL, 0, w, h);
}

/* The jobs through enc_make_inter_predictor, set up as av1_inter_prediction does (EbEncInterPrediction.c:4330-4930):
 * identity scale factors, get_conv_params_no_round(0, do_average, 0, tmp_dst, 128 / 64, is_compound, bit_depth), the
 * jnt weights copied into the second call's ConvolveParams. */
REFH_API void refh_inter_predict(const SvtB200Frame *refs, int n_ref_frames, const SvtB200Frame *pred, const SvtB200InterJob *jobs,
                                 int n_jobs) {
    refh_init();
    asm_set_convolve_asm_table();
    asm_set_convolve_hbd_asm_table();
    const int bd = pred->bit_depth, hbd = bd > 8;
    static uint16_t tmp_dst[128 * 128];
    (void)n_ref_frames;
    for (int j = 0; j < n_jobs; j++) {
        const SvtB200InterJob *b = &jobs[j];
        const int ss = b->plane != 0, compound = b->n_refs == 2;
        const int dstride = b->plane ? pred->stride_c : pred->stride_y;
        uint8_t *dplane = (uint8_t *)(b->plane == 0 ? pred->y : b->plane == 1 ? pred->cb : pred->cr);
        uint8_t *dst = dplane + (((ptrdiff_t)b->dst_y * dstride + b->dst_x) << hbd);
        MacroBlockD xd;
        memset(&xd, 0, sizeof(xd));
        xd.mb_to_left_edge = b->mb_to_left_edge;
        xd.mb_to_right_edge = b->mb_to_right_edge;
        xd.mb_to_top_edge = b->mb_to_top_edge;
        xd.mb_to_bottom_edge = b->mb_to_bottom_edge;
        for (int r = 0; r < b->n_refs; r++) {
            const SvtB200Frame *rf = &refs[b->ref[r]];
            const int sstride = b->plane ? rf->stride_c : rf->stride_y;
            uint8_t *splane = (uint8_t *)(b->plane == 0 ? rf->y : b->plane == 1 ? rf->cb : rf->cr);
            ScaleFactors sf;
            svt_av1_setup_scale_factors_for_frame(&sf, rf->width, rf->height, rf->width, rf->height);
            ConvolveParams cp = get_conv_params_no_round(0, r, 0, tmp_dst, b->plane ? 64 : 128, compound, bd);
            if (r == 1) {
                cp.use_jnt_comp_avg = cp.use_dist_wtd_comp_avg = b->use_jnt_comp_avg;
                cp.fwd_offset = b->fwd_offset;
                cp.bck_offset = b->bck_offset;
            }
            MV mv;
            mv.row = b->mv_row[r];
            mv.col = b->mv_col[r];
            enc_make_inter_predictor(splane, dst, b->pre_y, b->pre_x, mv, &sf, &cp, av1_make_interp_filters(b->filter_y, b->filter_x),
                                     NULL, (uint16_t)rf->width, (uint16_t)rf->height, b->bw, b->bh, BLOCK_8X8, &xd, sstride, dstride,
                                     b->plane, ss, ss, (uint8_t)bd, 0, 0, (uint8_t)hbd);
        }
    }
}

/* downsample_filtering_input_picture_ime / downsample_decimation_input_picture_ime (EbPictureAnalysisProcess.c:3667-3720,
 * :3362-3410) on plain buffers */
void downsample_filtering_input_picture_ime(EbPictureBufferDesc *input_padded_picture_ptr, EbPictureBufferDesc *quarter_picture_ptr,
                                            EbPictureBufferDesc *sixteenth_picture_ptr);
void downsample_decimation_input_picture_ime(EbPictureBufferDesc *input_padded_picture_ptr,
                                             EbPictureBufferDesc *quarter_decimated_picture_ptr,
                                             EbPictureBufferDesc *sixteenth_decimated_picture_ptr);
REFH_API void refh_me_downsample(const SvtB200Plane *full, const SvtB200Plane *quarter, const SvtB200Plane *sixteenth,
                                 const SvtB200MePlanes *planes, int filtered) {
    EbPictureBufferDesc f, q, s;
    plane_desc(&f, full, planes->full);
    plane_desc(&q, quarter, planes->quarter);
    plane_desc(&s, sixteenth, planes->sixteenth);
    if (filtered)
        downsample_filtering_input_picture_ime(&f, &q, &s);
    else
        downsample_decimation_input_picture_ime(&f, &q, &s);
}

/* ------------------------------------------------------------------------------------------------------------------ */
/* Sub-pel refinement: svt_av1_find_best_sub_pixel_tree per job, parameters set as md_subpel_search does               */
/* (EbProductCodingLoop.c:2063-2155).                                                                                 */
/* ------------------------------------------------------------------------------------------------------------------ */
#include "mcomp.h"
#include "av1me.h"
void init_fn_ptr(void);
extern AomVarianceFnPtr mefn_ptr[BlockSizeS_ALL];

REFH_API int refh_subpel_search(const SvtB200SubpelParams *p, const int32_t *mvcost0, const int32_t *mvcost1, const SvtB200Frame *src,
                                const SvtB200Frame *refs, int n_ref_frames, const SvtB200SubpelJob *jobs, int n_jobs,
                                SvtB200SubpelResult *results) {
    refh_init();
    init_fn_ptr();
    (void)n_ref_frames;
    for (int i = 0; i < n_jobs; i++) {
        const SvtB200SubpelJob *j = &jobs[i];
        int bsize = -1;
        for (int b = 0; b < BlockSizeS_ALL; b++)
            if (block_size_wide[b] == j->bw && block_size_high[b] == j->bh) bsize = b;
        if (bsize < 0) return -1;
        MacroBlockD xd;
        memset(&xd, 0, sizeof(xd));
        xd.mi_row = j->blk_y >> 2;
        xd.mi_col = j->blk_x >> 2;
        MV ref_mv = {j->ref_mv_row, j->ref_mv_col};
        SUBPEL_MOTION_SEARCH_PARAMS ms;
        memset(&ms, 0, sizeof(ms));
        ms.allow_hp = p->allow_hp;
        ms.forced_stop = (SUBPEL_FORCE_STOP)p->forced_stop;
        ms.iters_per_step = p->iters_per_step;
        ms.mv_limits.col_min = j->col_min, ms.mv_limits.col_max = j->col_max;
        ms.mv_limits.row_min = j->row_min, ms.mv_limits.row_max = j->row_max;
        ms.mv_cost_params.ref_mv = &ref_mv;
        ms.mv_cost_params.mv_cost_type = (MV_COST_TYPE)p->mv_cost_type;
        ms.mv_cost_params.error_per_bit = p->error_per_bit;
        ms.mv_cost_params.mvjcost = p->mvjcost;
        ms.mv_cost_params.mvcost[0] = mvcost0;
        ms.mv_cost_params.mvcost[1] = mvcost1;
        ms.var_params.vfp = &mefn_ptr[bsize];
        ms.var_params.subpel_search_type = (SUBPEL_SEARCH_TYPE)p->subpel_search_type;
        ms.var_params.w = j->bw;
        ms.var_params.h = j->bh;
        const SvtB200Frame *rf = &refs[j->ref];
        struct svt_buf_2d rb, sb2;
        memset(&rb, 0, sizeof(rb));
        memset(&sb2, 0, sizeof(sb2));
        rb.buf = (uint8_t *)rf->y + (ptrdiff_t)j->blk_y * rf->stride_y + j->blk_x;
        rb.stride = rf->stride_y, rb.width = rf->width, rb.height = rf->height;
        sb2.buf = (uint8_t *)src->y + (ptrdiff_t)j->blk_y * src->stride_y + j->blk_x;
        sb2.stride = src->stride_y, sb2.width = src->width, sb2.height = src->height;
        ms.var_params.ms_buffers.ref = &rb;
        ms.var_params.ms_buffers.src = &sb2;
        MV start = {j->start_mv_row, j->start_mv_col}, best;
        int dist = 0;
        unsigned int sse = 0;
        const int err = svt_av1_find_best_sub_pixel_tree(&xd, NULL, &ms, start, &best, &dist, &sse, NULL);
        results[i].mv_row = best.row, results[i].mv_col = best.col;
        results[i].besterr = err, results[i].distortion = dist, results[i].sse = sse;
    }
    return 0;
}

/* the limits md_subpel_search derives for a block (EbProductCodingLoop.c:2090-2101) */
REFH_API void refh_subpel_limits(int mi_rows, int mi_cols, int blk_x, int blk_y, int bw, int bh, int ref_mv_row, int ref_mv_col,
                                 int16_t out[4]) {
    MV ref_mv = {(int16_t)ref_mv_row, (int16_t)ref_mv_col};
    MvLimits lim;
    const int mi_row = blk_y >> 2, mi_col = blk_x >> 2;
    lim.row_min = -(((mi_row + (bh >> 2)) * MI_SIZE) + AOM_INTERP_EXTEND);
    lim.col_min = -(((mi_col + (bw >> 2)) * MI_SIZE) + AOM_INTERP_EXTEND);
    lim.row_max = (mi_rows - mi_row) * MI_SIZE + AOM_INTERP_EXTEND;
    lim.col_max = (mi_cols - mi_col) * MI_SIZE + AOM_INTERP_EXTEND;
    svt_av1_set_mv_search_range(&lim, &ref_mv);
    SubpelMvLimits sl;
    svt_av1_set_subpel_mv_search_range(&sl, (FullMvLimits *)&lim, &ref_mv);
    out[0] = (int16_t)sl.col_min, out[1] = (int16_t)sl.col_max, out[2] = (int16_t)sl.row_min, out[3] = (int16_t)sl.row_max;
}

/* ====================================================================================================
 * Temporal filter: the reference's svt_av1_apply_temporal_filter_planewise[_hbd] on one block, with the MeContext fields
 * it reads (EbMotionEstimationContext.h:443-458) filled from plain arguments.  via_rtcd: 0 calls the _c functions, 1 the
 * RTCD pointers (whatever is installed there).
 * ================================================================================================== */
#include "EbTemporalFiltering.h"
REFH_API int refh_tf_planewise(int via_rtcd, int bit_depth, int chroma, int block_row, int block_col, const int32_t *split_flag4,
                               const uint64_t *err16_16, const uint64_t *err32_4, const int16_t *mvx16_16, const int16_t *mvy16_16,
                               const int16_t *mvx32_4, const int16_t *mvy32_4, int min_frame_size, const void *y_src,
                               int y_src_stride, const void *y_pre, int y_pre_stride, const void *u_src, const void *v_src,
                               int uv_src_stride, const void *u_pre, const void *v_pre, int uv_pre_stride, unsigned bw, unsigned bh,
                               int ss_x, int ss_y, const double *noise_levels, int decay_control, uint32_t *y_accum,
                               uint16_t *y_count, uint32_t *u_accum, uint16_t *u_count, uint32_t *v_accum, uint16_t *v_count) {
    refh_init();
    MeContext *c = (MeContext *)calloc(1, sizeof(MeContext));
    if (!c) return -1;
    c->tf_chroma = (uint8_t)chroma;
    c->tf_block_row = block_row;
    c->tf_block_col = block_col;
    c->min_frame_size = (uint16_t)min_frame_size;
    for (int i = 0; i < 4; i++) {
        c->tf_32x32_block_split_flag[i] = split_flag4[i];
        c->tf_32x32_block_error[i] = err32_4[i];
        c->tf_32x32_mv_x[i] = mvx32_4[i];
        c->tf_32x32_mv_y[i] = mvy32_4[i];
    }
    for (int i = 0; i < 16; i++) {
        c->tf_16x16_block_error[i] = err16_16[i];
        c->tf_16x16_mv_x[i] = mvx16_16[i];
        c->tf_16x16_mv_y[i] = mvy16_16[i];
    }
    if (bit_depth == 8)
        (via_rtcd ? svt_av1_apply_temporal_filter_planewise : svt_av1_apply_temporal_filter_planewise_c)(
            c, y_src, y_src_stride, y_pre, y_pre_stride, u_src, v_src, uv_src_stride, u_pre, v_pre, uv_pre_stride, bw, bh, ss_x, ss_y,
            noise_levels, decay_control, y_accum, y_count, u_accum, u_count, v_accum, v_count);
    else
        (via_rtcd ? svt_av1_apply_temporal_filter_planewise_hbd : svt_av1_apply_temporal_filter_planewise_hbd_c)(
            c, y_src, y_src_stride, y_pre, y_pre_stride, u_src, v_src, uv_src_stride, u_pre, v_pre, uv_pre_stride, bw, bh, ss_x, ss_y,
            noise_levels, decay_control, y_accum, y_count, u_accum, u_count, v_accum, v_count, (uint32_t)bit_depth);
    free(c);
    return 0;
}

/* ====================================================================================================
 * Picture analysis: the reference's compute_block_mean_compute_variance / compute_chroma_block_mean on one SB
 * (EbPictureAnalysisProcess.c:1005, :493) with the minimal control sets they touch.
 * ================================================================================================== */
EbErrorType compute_block_mean_compute_variance(SequenceControlSet *scs_ptr, PictureParentControlSet *pcs_ptr,
                                                EbPictureBufferDesc *input_padded_picture_ptr, uint32_t sb_index,
                                                uint32_t input_luma_origin_index);
EbErrorType compute_chroma_block_mean(SequenceControlSet *scs_ptr, PictureParentControlSet *pcs_ptr,
                                      EbPictureBufferDesc *input_padded_picture_ptr, uint32_t sb_coding_order,
                                      uint32_t input_cb_origin_index, uint32_t input_cr_origin_index);
REFH_API int refh_sb_mean_variance(uint8_t *y, int stride_y, uint32_t luma_index, uint8_t *cb, uint8_t *cr, int stride_c,
                                   uint32_t chroma_index, int full_precision, uint8_t *y_mean85, uint16_t *var85, uint8_t *cb_mean85,
                                   uint8_t *cr_mean85) {
    refh_init();
    SequenceControlSet *scs = (SequenceControlSet *)calloc(1, sizeof(SequenceControlSet));
    PictureParentControlSet *pcs = (PictureParentControlSet *)calloc(1, sizeof(PictureParentControlSet));
    EbPictureBufferDesc pic;
    memset(&pic, 0, sizeof(pic));
    if (!scs || !pcs) return -1;
    scs->block_mean_calc_prec = full_precision ? BLOCK_MEAN_PREC_FULL : BLOCK_MEAN_PREC_SUB;
    uint8_t *ym = y_mean85, *cbm = cb_mean85, *crm = cr_mean85;
    uint16_t *vr = var85;
    pcs->y_mean = &ym;
    pcs->cb_mean = &cbm;
    pcs->cr_mean = &crm;
    pcs->variance = &vr;
    pic.buffer_y = y, pic.buffer_cb = cb, pic.buffer_cr = cr;
    pic.stride_y = (uint16_t)stride_y, pic.stride_cb = pic.stride_cr = (uint16_t)stride_c;
    compute_block_mean_compute_variance(scs, pcs, &pic, 0, luma_index);
    if (cb && cr) compute_chroma_block_mean(scs, pcs, &pic, 0, chroma_index, chroma_index);
    free(scs);
    free(pcs);
    return 0;
}

/* ====================================================================================================
 * Open-loop intra search: the reference's open_loop_intra_search_mb (EbMotionEstimation.c:3043) over every SB of a
 * picture with the TPL controls of `tpl_level` (set_tpl_controls: >= 5 -> DC_PRED only).  buf: padded luma buffer,
 * (origin_x, origin_y) its first picture sample.  cost / mode: [mb rows][mb cols].
 * ================================================================================================== */
EbErrorType open_loop_intra_search_mb(PictureParentControlSet *pcs_ptr, uint32_t sb_index, EbPictureBufferDesc *input_ptr);
EbErrorType sb_params_init(SequenceControlSet *scs_ptr);
void set_tpl_controls(PictureParentControlSet *pcs_ptr, uint8_t tpl_level);
void init_intra_dc_predictors_c_internal(void);
void init_intra_predictors_internal(void);
REFH_API int refh_ois_picture(uint8_t *buf, int stride, int origin_x, int origin_y, int width, int height, int tpl_level,
                              int64_t *cost, int32_t *mode) {
    refh_init();
    static int intra_tables = 0;
    if (!intra_tables) { /* as svt_av1_enc_init does (EbEncHandle.c:1149-1153) */
        init_intra_dc_predictors_c_internal();
        init_intra_predictors_internal();
        intra_tables = 1;
    }
    SequenceControlSet *scs = (SequenceControlSet *)calloc(1, sizeof(SequenceControlSet));
    PictureParentControlSet *pcs = (PictureParentControlSet *)calloc(1, sizeof(PictureParentControlSet));
    EbObjectWrapper wrap;
    EbPictureBufferDesc pic;
    memset(&wrap, 0, sizeof(wrap));
    memset(&pic, 0, sizeof(pic));
    if (!scs || !pcs) return -1;
    wrap.object_ptr = scs;
    pcs->scs_wrapper_ptr = &wrap;
    pcs->scs_ptr = scs;
    scs->sb_sz = 64;
    scs->seq_header.max_frame_width = (uint16_t)width;
    scs->seq_header.max_frame_height = (uint16_t)height;
    scs->static_config.enable_paeth = DEFAULT;
    scs->static_config.enable_smooth = DEFAULT;
    if (sb_params_init(scs) != EB_ErrorNone) return -2;
    pic.buffer_y = buf, pic.stride_y = (uint16_t)stride, pic.origin_x = (uint16_t)origin_x, pic.origin_y = (uint16_t)origin_y;
    pic.width = (uint16_t)width, pic.height = (uint16_t)height;
    pcs->enhanced_picture_ptr = &pic;
    set_tpl_controls(pcs, (uint8_t)tpl_level);
    const int mbw = (width + 15) / 16, mbh = (height + 15) / 16;
    OisMbResults *res = (OisMbResults *)calloc((size_t)mbw * mbh, sizeof(OisMbResults));
    OisMbResults **ptrs = (OisMbResults **)calloc((size_t)mbw * mbh, sizeof(OisMbResults *));
    for (int i = 0; i < mbw * mbh; i++) {
        ptrs[i] = &res[i];
        res[i].intra_cost = -1, res[i].intra_mode = -1;
    }
    pcs->ois_mb_results = ptrs;
    for (uint32_t sb = 0; sb < scs->sb_total_count; sb++) open_loop_intra_search_mb(pcs, sb, &pic);
    for (int i = 0; i < mbw * mbh; i++) cost[i] = res[i].intra_cost, mode[i] = res[i].intra_mode;
    free(res), free(ptrs), free(scs), free(pcs); /* sb_params_array belongs to the reference's allocation tracker */
    return 0;
}
