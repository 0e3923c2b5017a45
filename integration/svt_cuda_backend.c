/*
 * svt_cuda_backend.c - the reference-side binding of libsvtav1_b200.so (INTEGRATION.md section 2).
 *
 * Compiled INTO the overlay build of the reference encoder (integration/Makefile) against the reference's own
 * headers, exactly like a file a maintainer would add under Source/Lib/Encoder/Codec/.  It translates the encoder's
 * structs (PictureParentControlSet, MeContext, EbPaReferenceObject, the ModeInfo grid, FrameHeader) into the plain
 * C ABI of include/svt_av1_b200.h and back.  The hooks that call it are inserted into copies of six reference files
 * by integration/overlay.py; the mounted reference stays untouched and nothing of it is copied into this repository.
 *
 * Switches (environment, read once):
 *   SVT_CUDA=1            turn the CUDA backend on (default: off -> the build behaves exactly like the reference)
 *   SVT_CUDA_DEVICE=n     CUDA ordinal (default 0)
 *   SVT_CUDA_ME / SVT_CUDA_DLF / SVT_CUDA_CDEF / SVT_CUDA_LR = 0 to leave one stage on the CPU (default 1 when SVT_CUDA=1)
 *   SVT_CUDA_ME_DS=1      derive the 1/4 and 1/16 ME planes on the device instead of uploading the host's
 *   SVT_CUDA_PROFILE=1    print per-stage wall time / call counts at deinit (also for the CPU path, for comparison)
 * There is NO CPU fallback once a stage is on: a failing GPU call prints the library's message and aborts.
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "EbDefinitions.h"
#include "EbSequenceControlSet.h"
#include "EbPictureControlSet.h"
#include "EbPictureBufferDesc.h"
#include "EbReferenceObject.h"
#include "EbMotionEstimationProcess.h"
#include "EbMotionEstimation.h"
#include "EbMotionEstimationContext.h"
#include "EbMotionEstimationLcuResults.h"
#include "EbGlobalMotionEstimation.h"
#include "EbDeblockingFilter.h"
#include "EbDeblockingCommon.h"
#include "EbEncCdef.h"
#include "EbCdef.h"
#include "EbUtility.h"
#include "EbLog.h"

#include "svt_av1_b200.h"
#include "svt_cuda_backend.h"
#include "aom_dsp_rtcd.h"
static volatile long long g_tf_calls = 0;
#define SVT_CUDA_TF_COUNT() __sync_fetch_and_add(&g_tf_calls, 1)
#include "svt_cuda_tf_shim.h"
static void (*g_tf_saved[2])(void);

static int            g_on = -1, g_me = 0, g_dlf = 0, g_cdef = 0, g_lr = 0, g_me_ds = 0, g_prof = 0, g_tf = 0, g_pa = 0, g_ois = 0;
static volatile long long g_pa_calls = 0, g_ois_calls = 0;
/* SVT_CUDA_PROFILE: host-side pieces of the deblocking / CDEF hooks (thread-ns): mode-info flattening, skip8 map, the
 * engine call as a whole */
static volatile long long g_ns_flatten = 0, g_ns_skip8 = 0, g_ns_engine_cdef = 0;
#define PROF_ADD(var, t_start) do { if (g_prof) __sync_fetch_and_add(&(var), now_ns() - (t_start)); } while (0)
static SvtB200Engine *g_engine = NULL;
static int            g_users  = 0;

enum { ST_ME, ST_DLF, ST_CDEF, ST_LR, ST_N };
static struct { volatile int64_t ns, calls; } g_stat[2][ST_N]; /* [gpu?][stage] */
static const char *g_stage_name[ST_N] = {"me", "dlf", "cdef", "lr"};

static int64_t now_ns(void) {
    struct timespec t;
    clock_gettime(CLOCK_MONOTONIC, &t);
    return (int64_t)t.tv_sec * 1000000000ll + t.tv_nsec;
}
static void stat_add(int gpu, int stage, int64_t t0) {
    __sync_fetch_and_add(&g_stat[gpu][stage].ns, now_ns() - t0);
    __sync_fetch_and_add(&g_stat[gpu][stage].calls, 1);
}
int64_t svt_cuda_prof_begin(void) { return g_prof ? now_ns() : 0; }
void    svt_cuda_prof_end_cpu(int stage, int64_t t0) {
    if (g_prof) stat_add(0, stage, t0);
}

static int env_flag(const char *name, int dflt) {
    const char *v = getenv(name);
    return v ? atoi(v) != 0 : dflt;
}

static void die(const char *what, int rc) {
    fprintf(stderr, "SVT [CUDA backend]: %s failed (%d): %s - no CPU fallback, aborting\n", what, rc, svt_b200_last_error());
    abort();
}

/* EbEncHandle.c svt_av1_enc_init hook (after setup_rtcd_internal, :1144-1145) */
void svt_cuda_backend_init(void) {
    if (g_on < 0) {
        g_on   = env_flag("SVT_CUDA", 0);
        g_prof = env_flag("SVT_CUDA_PROFILE", 0);
        if (g_on) {
            g_me    = env_flag("SVT_CUDA_ME", 1);
            g_dlf   = env_flag("SVT_CUDA_DLF", 1);
            g_cdef  = env_flag("SVT_CUDA_CDEF", 1);
            g_lr    = env_flag("SVT_CUDA_LR", 1);
            g_me_ds = env_flag("SVT_CUDA_ME_DS", 0);
            /* parity switches, off by default: bit-exact, but per-block / per-picture round trips that do not pay */
            g_tf = env_flag("SVT_CUDA_TF", 0);
            g_pa = env_flag("SVT_CUDA_PA", 0);
            g_ois = env_flag("SVT_CUDA_OIS", 0);
        }
    }
    if (!g_on) return;
    if (g_users++ == 0) {
        const char *d  = getenv("SVT_CUDA_DEVICE");
        int         rc = svt_b200_engine_create(d ? atoi(d) : 0, &g_engine);
        if (rc) die("svt_b200_engine_create", rc);
        SVT_LOG("SVT [CUDA backend]: libsvtav1_b200 v%d on device %d (me %d, dlf %d, cdef %d, lr %d, tf %d, pa %d)\n", svt_b200_version(),
                d ? atoi(d) : 0, g_me, g_dlf, g_cdef, g_lr, g_tf, g_pa);
        if (g_tf) { /* the temporal filter's weighting through the GPU drop-ins (svt_cuda_tf_shim.h) */
            g_tf_saved[0] = (void (*)(void))svt_av1_apply_temporal_filter_planewise;
            g_tf_saved[1] = (void (*)(void))svt_av1_apply_temporal_filter_planewise_hbd;
            svt_av1_apply_temporal_filter_planewise     = svt_av1_apply_temporal_filter_planewise_cuda;
            svt_av1_apply_temporal_filter_planewise_hbd = svt_av1_apply_temporal_filter_planewise_hbd_cuda;
        }
    }
}

/* svt_av1_enc_deinit hook: prints the profile and releases the engine */
void svt_cuda_backend_deinit(void) {
    if (g_prof) {
        for (int gpu = 0; gpu < 2; gpu++)
            for (int s = 0; s < ST_N; s++)
                if (g_stat[gpu][s].calls)
                    fprintf(stderr, "SVT [CUDA profile]: %-4s %s: %lld calls, %.3f ms total wall in stage threads, %.3f ms/call\n",
                            g_stage_name[s], gpu ? "gpu" : "cpu", (long long)g_stat[gpu][s].calls, g_stat[gpu][s].ns / 1e6,
                            g_stat[gpu][s].ns / 1e6 / g_stat[gpu][s].calls);
    }
    if (!g_on || !g_engine) return;
    if (--g_users == 0) {
        if (g_prof) {
            SvtB200EngineStats st;
            svt_b200_engine_get_stats(g_engine, &st);
            fprintf(stderr,
                    "SVT [CUDA profile]: engine: %llu ME pictures (%llu plane uploads, %llu resident hits), %llu dlf, %llu cdef, %llu lr, "
                    "H2D %.1f MB, D2H %.1f MB, pinned %.1f MB, %llu kernel launches; thread-ms: slot wait %.1f, issue %.1f "
                    "(of which wait for another thread's upload %.1f), wait for GPU %.1f, host staging copies %.1f\n",
                    (unsigned long long)st.me_pictures, (unsigned long long)st.me_plane_uploads,
                    (unsigned long long)st.me_plane_hits, (unsigned long long)st.dlf_frames, (unsigned long long)st.cdef_frames,
                    (unsigned long long)st.lr_frames, st.h2d_bytes / 1e6, st.d2h_bytes / 1e6, st.pinned_bytes / 1e6, (unsigned long long)svt_b200_launch_count(),
                    st.ns_slot_wait / 1e6, st.ns_issue / 1e6, st.ns_plane_wait / 1e6, st.ns_sync / 1e6, st.ns_host_copy / 1e6);
        }
        if (g_prof)
            fprintf(stderr, "SVT [CUDA profile]: host side of the filter hooks, thread-ms: flatten mode info %.1f, skip8 map %.1f, CDEF engine calls %.1f\n",
                    g_ns_flatten / 1e6, g_ns_skip8 / 1e6, g_ns_engine_cdef / 1e6);
        if (g_prof && (g_tf || g_pa || g_ois))
            fprintf(stderr, "SVT [CUDA profile]: tf blocks on the GPU %lld, picture-analysis pictures on the GPU %lld, open-loop intra pictures on the GPU %lld\n",
                    (long long)g_tf_calls, (long long)g_pa_calls, (long long)g_ois_calls);
        if (g_tf && g_tf_saved[0]) {
            svt_av1_apply_temporal_filter_planewise     = (__typeof__(svt_av1_apply_temporal_filter_planewise))g_tf_saved[0];
            svt_av1_apply_temporal_filter_planewise_hbd = (__typeof__(svt_av1_apply_temporal_filter_planewise_hbd))g_tf_saved[1];
        }
        svt_b200_engine_destroy(g_engine);
        g_engine = NULL;
    }
}

int svt_cuda_me_active(void) { return g_on > 0 && g_me; }

/* 8-bit content carried in 16-bit containers (is_16bit_pipeline) keeps the C path: the kernels read bit_depth from the
 * container type */
static int containers_ok(const SequenceControlSet *scs_ptr) {
    return !(scs_ptr->static_config.is_16bit_pipeline && scs_ptr->static_config.encoder_bit_depth == EB_8BIT);
}
int svt_cuda_dlf_applies(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr) {
    PictureParentControlSet *ppcs = pcs_ptr->parent_pcs_ptr;
    return g_on > 0 && g_dlf && containers_ok(scs_ptr) && !ppcs->frm_hdr.delta_lf_params.delta_lf_present &&
        ppcs->av1_cm->tiles_info.tile_cols * ppcs->av1_cm->tiles_info.tile_rows == 1;
}
int svt_cuda_lr_applies(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr) {
    PictureParentControlSet *ppcs = pcs_ptr->parent_pcs_ptr;
    return g_on > 0 && g_lr && containers_ok(scs_ptr) && av1_superres_unscaled(&ppcs->av1_cm->frm_size) &&
        ppcs->av1_cm->tiles_info.tile_cols * ppcs->av1_cm->tiles_info.tile_rows == 1;
}
int svt_cuda_cdef_applies(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr) {
    (void)pcs_ptr;
    return g_on > 0 && g_cdef && containers_ok(scs_ptr) && scs_ptr->seq_header.sb_size != BLOCK_128X128;
}

/* ===================================================================================================================
 * Motion estimation: the SB loop of motion_estimation_kernel (EbMotionEstimationProcess.c:831-965)
 * ================================================================================================================= */
static void plane_geom(SvtB200Plane *g, const EbPictureBufferDesc *d) {
    g->stride   = d->stride_y;
    g->origin_x = d->origin_x;
    g->origin_y = d->origin_y;
    g->width    = d->width;
    g->height   = d->height;
}

static void host_pic(SvtB200HostMePicture *h, EbPaReferenceObject *o, int filtered) {
    h->key  = o;
    h->tag  = o->picture_number;
    h->full = o->input_padded_picture_ptr->buffer_y;
    if (g_me_ds) {
        h->quarter = h->sixteenth = NULL;
    } else {
        h->quarter   = (filtered ? o->quarter_filtered_picture_ptr : o->quarter_decimated_picture_ptr)->buffer_y;
        h->sixteenth = (filtered ? o->sixteenth_filtered_picture_ptr : o->sixteenth_decimated_picture_ptr)->buffer_y;
    }
}

/* MeContext (as signal_derivation_me_kernel_oq left it) + the per-picture fields motion_estimation_kernel copies from
 * the PCS (:914-940) -> SvtB200MeParams.  Returns 0 when the configuration is outside what the GPU path implements. */
static int me_params(SvtB200MeParams *p, const MeContext *me, const PictureParentControlSet *pcs, const SequenceControlSet *scs,
                     const EbPictureBufferDesc *full, const EbPictureBufferDesc *quarter, const EbPictureBufferDesc *sixteenth) {
    memset(p, 0, sizeof(*p));
    if (me->hme_decimation != TWO_DECIMATION_HME || !me->enable_hme_flag || !me->enable_hme_level0_flag ||
        !me->enable_hme_level1_flag || !me->enable_hme_level2_flag)
        return 0;
    plane_geom(&p->full, full);
    plane_geom(&p->quarter, quarter);
    plane_geom(&p->sixteenth, sixteenth);
    p->num_lists   = pcs->slice_type == P_SLICE ? 1 : 2;
    p->num_refs[0] = pcs->ref_list0_count_try;
    p->num_refs[1] = pcs->slice_type == B_SLICE ? pcs->ref_list1_count_try : 0;
    for (int l = 0; l < p->num_lists; l++)
        for (int r = 0; r < p->num_refs[l]; r++) {
            const EbPaReferenceObject *ro = (EbPaReferenceObject *)pcs->ref_pa_pic_ptr_array[l][r]->object_ptr;
            /* get_me_reference: ABS((int16_t)(picture_number - ref picture_number)), EbMotionEstimation.c:1861 */
            p->ref_dist[l][r] = ABS((int16_t)(pcs->picture_number - ro->picture_number));
        }
    p->temporal_layer_index      = pcs->temporal_layer_index;
    p->is_used_as_reference_flag = pcs->is_used_as_reference_flag;
    p->enable_hme_flag           = me->enable_hme_flag;
    p->enable_hme_level0_flag    = me->enable_hme_level0_flag;
    p->enable_hme_level1_flag    = me->enable_hme_level1_flag;
    p->enable_hme_level2_flag    = me->enable_hme_level2_flag;
    p->hme_search_method         = me->hme_search_method == SUB_SAD_SEARCH;
    p->me_search_method          = me->me_search_method == SUB_SAD_SEARCH;
    p->number_hme_search_region_in_width       = me->number_hme_search_region_in_width;
    p->number_hme_search_region_in_height      = me->number_hme_search_region_in_height;
    p->hme_level0_total_search_area_width      = me->hme_level0_total_search_area_width;
    p->hme_level0_total_search_area_height     = me->hme_level0_total_search_area_height;
    p->hme_level0_max_total_search_area_width  = me->hme_level0_max_total_search_area_width;
    p->hme_level0_max_total_search_area_height = me->hme_level0_max_total_search_area_height;
    for (int i = 0; i < 2; i++) {
        p->hme_level0_search_area_in_width_array[i]      = me->hme_level0_search_area_in_width_array[i];
        p->hme_level0_search_area_in_height_array[i]     = me->hme_level0_search_area_in_height_array[i];
        p->hme_level0_max_search_area_in_width_array[i]  = me->hme_level0_max_search_area_in_width_array[i];
        p->hme_level0_max_search_area_in_height_array[i] = me->hme_level0_max_search_area_in_height_array[i];
        p->hme_level1_search_area_in_width_array[i]      = me->hme_level1_search_area_in_width_array[i];
        p->hme_level1_search_area_in_height_array[i]     = me->hme_level1_search_area_in_height_array[i];
        p->hme_level2_search_area_in_width_array[i]      = me->hme_level2_search_area_in_width_array[i];
        p->hme_level2_search_area_in_height_array[i]     = me->hme_level2_search_area_in_height_array[i];
    }
    p->search_area_width    = me->search_area_width;
    p->search_area_height   = me->search_area_height;
    p->max_me_search_width  = me->max_me_search_width;
    p->max_me_search_height = me->max_me_search_height;
    p->enable_me_hme_ref_pruning               = me->me_hme_prune_ctrls.enable_me_hme_ref_pruning;
    p->prune_ref_if_hme_sad_dev_bigger_than_th = me->me_hme_prune_ctrls.prune_ref_if_hme_sad_dev_bigger_than_th;
    p->prune_ref_if_me_sad_dev_bigger_than_th  = me->me_hme_prune_ctrls.prune_ref_if_me_sad_dev_bigger_than_th;
    p->enable_me_sr_adjustment                 = me->me_sr_adjustment_ctrls.enable_me_sr_adjustment;
    p->reduce_me_sr_based_on_mv_length_th      = me->me_sr_adjustment_ctrls.reduce_me_sr_based_on_mv_length_th;
    p->stationary_hme_sad_abs_th               = me->me_sr_adjustment_ctrls.stationary_hme_sad_abs_th;
    p->stationary_me_sr_divisor                = me->me_sr_adjustment_ctrls.stationary_me_sr_divisor;
    p->reduce_me_sr_based_on_hme_sad_abs_th    = me->me_sr_adjustment_ctrls.reduce_me_sr_based_on_hme_sad_abs_th;
    p->me_sr_divisor_for_low_hme_sad           = me->me_sr_adjustment_ctrls.me_sr_divisor_for_low_hme_sad;
    p->max_number_of_pus_per_sb                = pcs->max_number_of_pus_per_sb;
    p->rc_dist_from_8x8                        = scs->input_resolution <= INPUT_SIZE_480p_RANGE;
    return 1;
}

/* Called once per ME segment in place of the SB loop.  Segment 0 of a picture runs the whole picture on the GPU; every
 * segment then does the reference's own accounting (me_processed_sb_count, the global-motion tail :949-962), so the
 * downstream stage still sees one result per segment and starts only when all SBs are done.  Returns 0 when the GPU
 * path does not apply to this picture (the caller then runs the reference's loop). */
int svt_cuda_me_segment(MotionEstimationContext_t *context_ptr, PictureParentControlSet *pcs_ptr, SequenceControlSet *scs_ptr,
                        EbPaReferenceObject *pa_ref_obj, EbPictureBufferDesc *input_padded_picture_ptr,
                        EbPictureBufferDesc *quarter_picture_ptr, EbPictureBufferDesc *sixteenth_picture_ptr,
                        EbPictureBufferDesc *input_picture_ptr, uint32_t segment_index, uint32_t x_sb_start_index,
                        uint32_t x_sb_end_index, uint32_t y_sb_start_index, uint32_t y_sb_end_index) {
    if (!svt_cuda_me_active()) return 0;
    MeContext *me = context_ptr->me_context_ptr;
    /* scaled references (super-res / resize) keep the C path: the planes are not the PA object's */
    if (input_padded_picture_ptr != pa_ref_obj->input_padded_picture_ptr) return 0;
    const int       filtered = scs_ptr->down_sampling_method_me_search == ME_FILTERED_DOWNSAMPLED;
    SvtB200MeParams p;
    if (!me_params(&p, me, pcs_ptr, scs_ptr, input_padded_picture_ptr, quarter_picture_ptr, sixteenth_picture_ptr)) return 0;

    if (segment_index == 0) {
        const int64_t        t0   = g_prof ? now_ns() : 0;
        const uint32_t       n_sb = pcs_ptr->sb_total_count;
        SvtB200HostMePicture src, refs[SVT_B200_ME_LISTS][SVT_B200_ME_MAX_REFS];
        memset(refs, 0, sizeof(refs));
        host_pic(&src, pa_ref_obj, filtered);
        for (int l = 0; l < p.num_lists; l++)
            for (int r = 0; r < p.num_refs[l]; r++)
                host_pic(&refs[l][r], (EbPaReferenceObject *)pcs_ptr->ref_pa_pic_ptr_array[l][r]->object_ptr, filtered);
        const size_t b_mv = (size_t)n_sb * SQUARE_PU_COUNT * MAX_PA_ME_MV * sizeof(MvCandidate);
        const size_t b_cd = (size_t)n_sb * SQUARE_PU_COUNT * MAX_PA_ME_CAND, b_tc = (size_t)n_sb * SQUARE_PU_COUNT;
        uint8_t *    buf  = (uint8_t *)malloc(b_mv + b_cd + b_tc);
        if (!buf) die("malloc", -1);
        int rc = svt_b200_engine_me_picture(g_engine, &p, &src, refs, filtered, (int16_t *)buf, buf + b_mv, buf + b_mv + b_cd,
                                            pcs_ptr->rc_me_distortion);
        if (rc) die("svt_b200_engine_me_picture", rc);
        for (uint32_t sb = 0; sb < n_sb; sb++) {
            MeSbResults *r = pcs_ptr->pa_me_data->me_results[sb];
            memcpy(r->me_mv_array, buf + (size_t)sb * SQUARE_PU_COUNT * MAX_PA_ME_MV * sizeof(MvCandidate),
                   SQUARE_PU_COUNT * MAX_PA_ME_MV * sizeof(MvCandidate));
            memcpy(r->me_candidate_array, buf + b_mv + (size_t)sb * SQUARE_PU_COUNT * MAX_PA_ME_CAND, SQUARE_PU_COUNT * MAX_PA_ME_CAND);
            memcpy(r->total_me_candidate_index, buf + b_mv + b_cd + (size_t)sb * SQUARE_PU_COUNT, SQUARE_PU_COUNT);
        }
        free(buf);
        if (g_prof) stat_add(1, ST_ME, t0);
    }
    svt_block_on_mutex(pcs_ptr->me_processed_sb_mutex);
    pcs_ptr->me_processed_sb_count += (x_sb_end_index - x_sb_start_index) * (y_sb_end_index - y_sb_start_index);
    if (pcs_ptr->me_processed_sb_count == pcs_ptr->sb_total_count) {
        if (pcs_ptr->gm_ctrls.enabled)
            global_motion_estimation(pcs_ptr, input_picture_ptr);
        else
            memset(pcs_ptr->is_global_motion, EB_FALSE, MAX_NUM_OF_REF_PIC_LIST * REF_LIST_MAX_DEPTH);
    }
    svt_release_mutex(pcs_ptr->me_processed_sb_mutex);
    return 1;
}

/* ===================================================================================================================
 * Deblocking: svt_av1_loop_filter_frame (EbDeblockingFilter.c:711) for the picture of dlf_kernel
 * ================================================================================================================= */
static __thread SvtB200DlfMi *t_mi     = NULL;
static __thread size_t        t_mi_cap = 0;

static void host_frame(SvtB200Frame *f, const EbPictureBufferDesc *d, int is_16bit, int width, int height) {
    const int bps = is_16bit ? 2 : 1;
    f->y          = d->buffer_y + ((size_t)d->origin_x + (size_t)d->origin_y * d->stride_y) * bps;
    f->cb         = d->buffer_cb + ((size_t)(d->origin_x >> 1) + (size_t)(d->origin_y >> 1) * d->stride_cb) * bps;
    f->cr         = d->buffer_cr + ((size_t)(d->origin_x >> 1) + (size_t)(d->origin_y >> 1) * d->stride_cr) * bps;
    f->stride_y   = d->stride_y;
    f->stride_c   = d->stride_cb;
    f->width      = width;
    f->height     = height;
    f->bit_depth  = is_16bit ? 10 : 8;
}

/* One SvtB200DlfMi per 4x4: exactly the quantities set_lpf_parameters / get_transform_size (EbDeblockingFilter.c:134-320)
 * derive from a ModeInfo, computed with the reference's own tables. */
static void flatten_mi(SvtB200DlfMi *f, const MbModeInfo *mbmi, const LoopFilterInfoN *lfi_n) {
    const BlockSize bs    = mbmi->block_mi.sb_type;
    const int       inter = is_inter_block_no_intrabc(mbmi->block_mi.ref_frame[0]);
    TxSize          tx    = inter ? tx_depth_to_tx_size[0][bs] : tx_depth_to_tx_size[mbmi->tx_depth][bs];
    if (inter && !mbmi->block_mi.skip) tx = tx_depth_to_tx_size[mbmi->tx_depth][bs];
    const TxSize    uv = av1_get_max_uv_txsize(bs, 1, 1);
    const BlockSize cb = get_plane_block_size(bs, 1, 1);
    f->tx_w[0]         = (uint8_t)tx_size_wide[txsize_horz_map[tx]];
    f->tx_h[0]         = (uint8_t)tx_size_high[txsize_vert_map[tx]];
    f->tx_w[1]         = (uint8_t)tx_size_wide[txsize_horz_map[uv]];
    f->tx_h[1]         = (uint8_t)tx_size_high[txsize_vert_map[uv]];
    f->blk_w[0]        = block_size_wide[bs];
    f->blk_h[0]        = block_size_high[bs];
    f->blk_w[1]        = block_size_wide[cb];
    f->blk_h[1]        = block_size_high[cb];
    f->skip_inter      = mbmi->block_mi.skip && inter;
    const PredictionMode mode = (mbmi->block_mi.mode == INTRA_MODE_4x4) ? DC_PRED : mbmi->block_mi.mode;
    const int            rf = mbmi->block_mi.ref_frame[0], ml = mode_lf_lut[mode];
    f->lvl_y[0]  = lfi_n->lvl[0][0][0][rf][ml];
    f->lvl_y[1]  = lfi_n->lvl[0][0][1][rf][ml];
    f->lvl_u     = lfi_n->lvl[1][0][0][rf][ml];
    f->lvl_v     = lfi_n->lvl[2][0][0][rf][ml];
    f->lvl_class = (uint8_t)(rf * 2 + ml);
    f->pad[0] = f->pad[1] = 0;
}

static SvtB200DlfMi *flatten_picture_into(PictureControlSet *pcs_ptr, SvtB200DlfMi *dst);
static SvtB200DlfMi *flatten_picture(PictureControlSet *pcs_ptr) {
    PictureParentControlSet *ppcs = pcs_ptr->parent_pcs_ptr;
    const size_t             n    = (size_t)ppcs->av1_cm->mi_rows * ppcs->av1_cm->mi_cols;
    if (t_mi_cap < n) {
        free(t_mi);
        t_mi     = (SvtB200DlfMi *)malloc(n * sizeof(SvtB200DlfMi));
        t_mi_cap = n;
        if (!t_mi) die("malloc", -1);
    }
    return flatten_picture_into(pcs_ptr, t_mi);
}
static SvtB200DlfMi *flatten_picture_into(PictureControlSet *pcs_ptr, SvtB200DlfMi *t_mi) {
    PictureParentControlSet *ppcs    = pcs_ptr->parent_pcs_ptr;
    const int                mi_rows = ppcs->av1_cm->mi_rows, mi_cols = ppcs->av1_cm->mi_cols;
    const LoopFilterInfoN *lfi_n = &ppcs->lf_info;
    /* Every 4x4 cell owns a ModeInfo (EbAdaptiveMotionVectorPrediction.c update_mi_map fills all cells of a block alike), and
     * dereferencing each one is a cache miss: 518k of them at 2160p.  A block's entry is computed at its first cell of a
     * row and replicated over the block's width; rows below the block's first row copy the row above (same block: the
     * cell's sb_type says how many rows the block spans and AV1 blocks are aligned to their size). */
    for (int r = 0; r < mi_rows; r++) {
        ModeInfo **   row = pcs_ptr->mi_grid_base + (size_t)r * pcs_ptr->mi_stride;
        SvtB200DlfMi *out = t_mi + (size_t)r * mi_cols;
        for (int c = 0; c < mi_cols;) {
            const MbModeInfo *m   = &row[c]->mbmi;
            const int         bw4 = mi_size_wide[m->block_mi.sb_type], bh4 = mi_size_high[m->block_mi.sb_type];
            const int         n   = AOMMIN(bw4 - (c & (bw4 - 1)), mi_cols - c);
            if ((r & (bh4 - 1)) && r > 0)
                memcpy(&out[c], &out[c - mi_cols], (size_t)n * sizeof(SvtB200DlfMi)); /* not the block's first row */
            else {
                flatten_mi(&out[c], m, lfi_n);
                for (int k = 1; k < n; k++) out[c + k] = out[c];
            }
            c += n;
        }
    }
    return t_mi;
}

static EbPictureBufferDesc *recon_of(PictureControlSet *pcs_ptr, int is_16bit) { /* the selection of dlf_kernel (EbDlfProcess.c:180-193) */
    PictureParentControlSet *ppcs = pcs_ptr->parent_pcs_ptr;
    if (ppcs->is_used_as_reference_flag == EB_TRUE)
        return is_16bit ? ((EbReferenceObject *)ppcs->reference_picture_wrapper_ptr->object_ptr)->reference_picture16bit
                        : ((EbReferenceObject *)ppcs->reference_picture_wrapper_ptr->object_ptr)->reference_picture;
    return is_16bit ? pcs_ptr->recon_picture16bit_ptr : pcs_ptr->recon_picture_ptr;
}

static __thread const PictureControlSet *t_filtered = NULL; /* svt_cuda_dlf_pick_frame already deblocked this picture */

/* Deblocking deferred into the CDEF stage's GPU call (svt_b200_engine_dlf_cdef_frame_dev): the DLF stage only derives the
 * parameters; the reconstruction is then uploaded once for both filters.  Only when nobody needs the deblocked picture on the
 * host: no loop restoration (its boundary lines are saved from the deblocked host picture in dlf_kernel), no statistics. */
#include <pthread.h>
typedef struct PendingDlf {
    const PictureControlSet *pcs;
    SvtB200DlfParams         p;
    SvtB200DlfMi *           mi;
    size_t                   cap;
    int                      used;
} PendingDlf;
#define N_PENDING 64
static PendingDlf      g_pend[N_PENDING];
static pthread_mutex_t g_pend_mu = PTHREAD_MUTEX_INITIALIZER;

static int fuse_ok(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr) {
    return svt_cuda_cdef_applies(pcs_ptr, scs_ptr) && scs_ptr->seq_header.cdef_level && pcs_ptr->parent_pcs_ptr->cdef_level &&
        !scs_ptr->seq_header.enable_restoration && !scs_ptr->static_config.stat_report;
}
static PendingDlf *pending_take(const PictureControlSet *pcs_ptr, int create) {
    PendingDlf *e = NULL;
    pthread_mutex_lock(&g_pend_mu);
    for (int i = 0; i < N_PENDING && !e; i++)
        if (g_pend[i].used && g_pend[i].pcs == pcs_ptr) e = &g_pend[i];
    if (!e && create)
        for (int i = 0; i < N_PENDING && !e; i++)
            if (!g_pend[i].used) {
                e       = &g_pend[i];
                e->used = 1;
                e->pcs  = pcs_ptr;
            }
    pthread_mutex_unlock(&g_pend_mu);
    return e;
}
static void pending_release(PendingDlf *e) {
    pthread_mutex_lock(&g_pend_mu);
    e->used = 0;
    e->pcs  = NULL;
    pthread_mutex_unlock(&g_pend_mu);
}

/* Deblocks the reconstruction of pcs in place on the GPU (only called when svt_cuda_dlf_applies).  The caller has run
 * svt_av1_loop_filter_init, svt_av1_pick_filter_level and - as svt_av1_loop_filter_frame does first (:724) -
 * svt_av1_loop_filter_frame_init(frm_hdr, lf_info, 0, 3) is run here. */
void svt_cuda_dlf_frame(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr, EbPictureBufferDesc *recon_buffer) {
    PictureParentControlSet *ppcs    = pcs_ptr->parent_pcs_ptr;
    FrameHeader *            frm_hdr = &ppcs->frm_hdr;
    const int is_16bit = scs_ptr->static_config.encoder_bit_depth > EB_8BIT || scs_ptr->static_config.is_16bit_pipeline;
    if (t_filtered == pcs_ptr) { /* level search and filtering were one GPU call */
        t_filtered = NULL;
        return;
    }
    if (!frm_hdr->loop_filter_params.filter_level[0] && !frm_hdr->loop_filter_params.filter_level[1]) return;
    if (!recon_buffer) recon_buffer = recon_of(pcs_ptr, is_16bit);
    svt_av1_loop_filter_frame_init(frm_hdr, &ppcs->lf_info, 0, 3);
    const int64_t t0      = g_prof ? now_ns() : 0;
    const int     mi_rows = ppcs->av1_cm->mi_rows, mi_cols = ppcs->av1_cm->mi_cols;
    PendingDlf *  pend    = fuse_ok(pcs_ptr, scs_ptr) ? pending_take(pcs_ptr, 1) : NULL;
    SvtB200DlfMi *mi;
    if (pend) {
        const size_t n = (size_t)mi_rows * mi_cols;
        if (pend->cap < n) {
            free(pend->mi);
            pend->mi  = (SvtB200DlfMi *)malloc(n * sizeof(SvtB200DlfMi));
            pend->cap = n;
            if (!pend->mi) die("malloc", -1);
        }
        mi = flatten_picture_into(pcs_ptr, pend->mi);
    } else
        { const int64_t tf0 = g_prof ? now_ns() : 0; mi = flatten_picture(pcs_ptr); PROF_ADD(g_ns_flatten, tf0); }
    SvtB200DlfParams p;
    memset(&p, 0, sizeof(p));
    p.mi_rows         = mi_rows;
    p.mi_cols         = mi_cols;
    p.mi_stride       = mi_cols;
    p.sharpness       = frm_hdr->loop_filter_params.sharpness_level;
    p.filter_level[0] = frm_hdr->loop_filter_params.filter_level[0];
    p.filter_level[1] = frm_hdr->loop_filter_params.filter_level[1];
    p.filter_level_u  = frm_hdr->loop_filter_params.filter_level_u;
    p.filter_level_v  = frm_hdr->loop_filter_params.filter_level_v;
    p.plane_start     = 0;
    p.plane_end       = 3;
    if (pend) { /* the CDEF stage's call deblocks first (svt_cuda_cdef_picture) */
        pend->p = p;
        if (g_prof) stat_add(1, ST_DLF, t0);
        return;
    }
    SvtB200Frame f;
    host_frame(&f, recon_buffer, is_16bit, mi_cols * 4, mi_rows * 4);
    int rc = svt_b200_engine_dlf_frame(g_engine, &p, &f, mi);
    if (rc) die("svt_b200_engine_dlf_frame", rc);
    if (g_prof) stat_add(1, ST_DLF, t0);
}

/* svt_av1_pick_filter_level(LPF_PICK_FROM_FULL_IMAGE) + svt_av1_loop_filter_frame of dlf_kernel (loop_filter_mode >= 2,
 * EbDlfProcess.c:186-216) as ONE GPU call: the level search (search_filter_level x3: luma, U, V; every trial = filter a
 * plane + SSE against the source + restore) and the final deblocking share one upload of the picture.  Returns 0 when the
 * C path has to run (picture size not a multiple of 8: the SSE and the filter then cover different areas). */
int svt_cuda_dlf_pick_frame(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr, EbPictureBufferDesc *recon_buffer) {
    PictureParentControlSet *ppcs    = pcs_ptr->parent_pcs_ptr;
    FrameHeader *            frm_hdr = &ppcs->frm_hdr;
    struct LoopFilter *      lf      = &frm_hdr->loop_filter_params;
    const int is_16bit = scs_ptr->static_config.encoder_bit_depth > EB_8BIT || scs_ptr->static_config.is_16bit_pipeline;
    const int mi_rows = ppcs->av1_cm->mi_rows, mi_cols = ppcs->av1_cm->mi_cols;
    EbPictureBufferDesc *input = is_16bit ? pcs_ptr->input_frame16bit : (EbPictureBufferDesc *)ppcs->enhanced_picture_ptr;
    if (input->width != mi_cols * 4 || input->height != mi_rows * 4) return 0;
    const int64_t t0 = g_prof ? now_ns() : 0;
    if (!recon_buffer) recon_buffer = recon_of(pcs_ptr, is_16bit);
    lf->sharpness_level = 0; /* :1202 */
    SvtB200LpfPickParams pp;
    memset(&pp, 0, sizeof(pp));
    pp.dlf.mi_rows = mi_rows, pp.dlf.mi_cols = mi_cols, pp.dlf.mi_stride = mi_cols;
    pp.dlf.plane_start = 0, pp.dlf.plane_end = 3;
    pp.init.mode_ref_delta_enabled = lf->mode_ref_delta_enabled;
    for (int i = 0; i < 8; i++) pp.init.ref_deltas[i] = lf->ref_deltas[i];
    for (int i = 0; i < 2; i++) pp.init.mode_deltas[i] = lf->mode_deltas[i];
    pp.init.segmentation_enabled = frm_hdr->segmentation_params.segmentation_enabled;
    for (int sg = 0; sg < 8; sg++) {
        pp.init.seg_feature_mask[sg] = 0;
        for (int f = 0; f < 8; f++) {
            if (frm_hdr->segmentation_params.feature_enabled[sg][f]) pp.init.seg_feature_mask[sg] |= (uint8_t)(1u << f);
            pp.init.seg_feature_data[sg][f] = frm_hdr->segmentation_params.feature_data[sg][f];
        }
    }
    pp.method           = 0; /* LPF_PICK_FROM_FULL_IMAGE */
    pp.loop_filter_mode = ppcs->loop_filter_mode;
    pp.tx_mode_only_4x4 = frm_hdr->tx_mode == ONLY_4X4;
    pp.last_level[0] = lf->filter_level[0], pp.last_level[1] = lf->filter_level[1];
    pp.last_level[2] = lf->filter_level_u, pp.last_level[3] = lf->filter_level_v;
    SvtB200DlfMi *mi = flatten_picture(pcs_ptr); /* only lvl_class is read on this path */
    SvtB200Frame  rec, src;
    host_frame(&rec, recon_buffer, is_16bit, mi_cols * 4, mi_rows * 4);
    host_frame(&src, input, is_16bit, mi_cols * 4, mi_rows * 4);
    int32_t lv[4];
    int     rc = svt_b200_engine_dlf_pick_frame(g_engine, &pp, &rec, &src, mi, lv);
    if (rc) die("svt_b200_engine_dlf_pick_frame", rc);
    lf->filter_level[0] = lv[0], lf->filter_level[1] = lv[1], lf->filter_level_u = lv[2], lf->filter_level_v = lv[3];
    svt_av1_loop_filter_frame_init(frm_hdr, &ppcs->lf_info, 0, 3); /* what svt_av1_loop_filter_frame leaves behind */
    t_filtered = pcs_ptr;
    if (g_prof) stat_add(1, ST_DLF, t0);
    return 1;
}

/* ===================================================================================================================
 * CDEF: cdef_seg_search[16bit] of every segment + finish_cdef_search + svt_av1_cdef_frame / av1_cdef_frame16bit
 * (cdef_kernel, EbCdefProcess.c:510-534) for one picture
 * ================================================================================================================= */
static __thread uint8_t * t_skip     = NULL;
static __thread size_t    t_skip_cap = 0;

/* Runs the whole CDEF stage of the picture (search of every filter block, finish_cdef_search, frame apply); called by
 * the thread that completes the last CDEF segment, in place of finish_cdef_search + svt_av1_cdef_frame (only when
 * svt_cuda_cdef_applies; the per-segment cdef_seg_search calls are skipped by the hook). */
void svt_cuda_cdef_picture(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr) {
    const int64_t            t0   = g_prof ? now_ns() : 0;
    PictureParentControlSet *ppcs = pcs_ptr->parent_pcs_ptr;
    const Av1Common *        cm   = ppcs->av1_cm;
    const int is_16bit = scs_ptr->static_config.encoder_bit_depth > EB_8BIT || scs_ptr->static_config.is_16bit_pipeline;
    const int mi_rows = cm->mi_rows, mi_cols = cm->mi_cols;
    const int nvfb = (mi_rows + MI_SIZE_64X64 - 1) / MI_SIZE_64X64, nhfb = (mi_cols + MI_SIZE_64X64 - 1) / MI_SIZE_64X64;

    SvtB200CdefSearchParams sp;
    memset(&sp, 0, sizeof(sp));
    const int pick_method = ppcs->cdef_level == 2 ? 1 : ppcs->cdef_level == 3 ? 2 : ppcs->cdef_level == 4 ? 3 : 0;
    svt_b200_cdef_strength_table(pick_method, &sp);
    sp.mi_rows     = mi_rows;
    sp.mi_cols     = mi_cols;
    sp.pri_damping = 3 + (ppcs->frm_hdr.quantization_params.base_q_idx >> 6);

    /* skip8[r8][c8] = is_8x8_block_skip (EbEncCdef.c:241) */
    const int    rows8 = (mi_rows + 1) / 2, skip_stride = ((mi_cols + 1) / 2 + 15) & ~15;
    const size_t b_skip = (size_t)rows8 * skip_stride;
    if (t_skip_cap < b_skip) {
        free(t_skip);
        t_skip     = (uint8_t *)malloc(b_skip);
        t_skip_cap = b_skip;
    }
    if (!t_skip) die("malloc", -1);
    const int64_t ts0 = g_prof ? now_ns() : 0;
    memset(t_skip, 1, b_skip);
    ModeInfo **grid = pcs_ptr->mi_grid_base;
    const int  ms   = pcs_ptr->mi_stride;
    /* is_8x8_block_skip = AND of the four cells' skip flags; a block of 8x8 or more has one flag for all its cells, so one
     * dereference serves the block's whole width (only sub-8x8 partitions need all four cells) */
    for (int r = 0; r < mi_rows; r += 2) {
        uint8_t *out = t_skip + (size_t)(r >> 1) * skip_stride;
        for (int c = 0; c < mi_cols;) {
            const MbModeInfo *m   = &grid[r * ms + c]->mbmi;
            const int         bw4 = mi_size_wide[m->block_mi.sb_type], bh4 = mi_size_high[m->block_mi.sb_type];
            if (bw4 >= 2 && bh4 >= 2) {
                const int n = AOMMIN(bw4 - (c & (bw4 - 1)), mi_cols - c);
                memset(out + (c >> 1), m->block_mi.skip ? 1 : 0, (size_t)(n + 1) >> 1);
                c += n;
            } else {
                int sk = 1;
                for (int dr = 0; dr < 2; dr++)
                    for (int dc = 0; dc < 2; dc++)
                        if (r + dr < mi_rows && c + dc < mi_cols) sk &= (int)grid[(r + dr) * ms + c + dc]->mbmi.block_mi.skip;
                out[c >> 1] = (uint8_t)sk;
                c += 2;
            }
        }
    }

    PROF_ADD(g_ns_skip8, ts0);
    /* pcs->src[] / ref_coeff[] were set by dlf_kernel's pre-cdef prep (EbDlfProcess.c:254-300): sample (0,0) of each plane */
    EbPictureBufferDesc *recon_desc;
    if (ppcs->is_used_as_reference_flag == EB_TRUE)
        recon_desc = is_16bit ? ((EbReferenceObject *)ppcs->reference_picture_wrapper_ptr->object_ptr)->reference_picture16bit
                              : ((EbReferenceObject *)ppcs->reference_picture_wrapper_ptr->object_ptr)->reference_picture;
    else
        recon_desc = is_16bit ? pcs_ptr->recon_picture16bit_ptr : pcs_ptr->recon_picture_ptr;
    EbPictureBufferDesc *input_desc = is_16bit ? pcs_ptr->input_frame16bit : (EbPictureBufferDesc *)ppcs->enhanced_picture_ptr;
    SvtB200Frame recon, source;
    memset(&recon, 0, sizeof(recon));
    memset(&source, 0, sizeof(source));
    recon.y = pcs_ptr->src[0];
    recon.cb = pcs_ptr->src[1];
    recon.cr = pcs_ptr->src[2];
    recon.stride_y = recon_desc->stride_y;
    recon.stride_c = recon_desc->stride_cb;
    source.y = pcs_ptr->ref_coeff[0];
    source.cb = pcs_ptr->ref_coeff[1];
    source.cr = pcs_ptr->ref_coeff[2];
    source.stride_y = input_desc->stride_y;
    source.stride_c = input_desc->stride_cb;
    recon.width = source.width = mi_cols * 4;
    recon.height = source.height = mi_rows * 4;
    recon.bit_depth = source.bit_depth = is_16bit ? 10 : 8;

    PendingDlf *pend = pending_take(pcs_ptr, 0); /* deblocking deferred by the DLF stage: same upload, deblock, then CDEF */
    const int64_t te0 = g_prof ? now_ns() : 0;
    /* finish_cdef_search on the device (svt_b200_cdef_decide): the picture makes one round trip.  Inputs the reference
     * derives on the host: the picture's lambda (EbEncCdef.c:1209) and the strength table of the pick method */
    SvtB200CdefDecideParams dp;
    memset(&dp, 0, sizeof(dp));
    svt_b200_cdef_decide_table(pick_method, &dp);
    dp.mi_rows = mi_rows;
    dp.mi_cols = mi_cols;
    uint32_t fast_lambda = 0, full_lambda = 0;
    (*av1_lambda_assignment_function_table[ppcs->pred_structure])(pcs_ptr, &fast_lambda, &full_lambda,
                                                                 (uint8_t)ppcs->enhanced_picture_ptr->bit_depth,
                                                                 (uint16_t)(uint8_t)ppcs->frm_hdr.quantization_params.base_q_idx, EB_FALSE);
    dp.lambda = full_lambda;
    /* EbCdefProcess.c:527-529: the frame is not filtered when nobody reads it */
    const int apply = scs_ptr->seq_header.enable_restoration != 0 || ppcs->is_used_as_reference_flag || scs_ptr->static_config.recon_enabled;
    SvtB200CdefDecision dec;
    int8_t *            fb_idx = (int8_t *)malloc((size_t)nvfb * nhfb);
    if (!fb_idx) die("malloc", -1);
    int rc = svt_b200_engine_dlf_cdef_frame_dev(g_engine, pend ? &pend->p : NULL, pend ? pend->mi : NULL, &sp, &dp, sp.pri_damping, apply,
                                                &recon, &source, t_skip, skip_stride, &dec, fb_idx);
    PROF_ADD(g_ns_engine_cdef, te0);
    if (pend) pending_release(pend);
    if (rc) die("svt_b200_engine_dlf_cdef_frame_dev", rc);
    /* what finish_cdef_search leaves behind (EbEncCdef.c:1276-1336) */
    FrameHeader *fh            = &ppcs->frm_hdr;
    fh->cdef_params.cdef_bits  = (uint8_t)dec.cdef_bits;
    ppcs->nb_cdef_strengths    = dec.nb_cdef_strengths;
    for (int j = 0; j < dec.nb_cdef_strengths; j++) {
        fh->cdef_params.cdef_y_strength[j]  = dec.y_strength[j];
        fh->cdef_params.cdef_uv_strength[j] = dec.uv_strength[j];
    }
    fh->cdef_params.cdef_damping = sp.pri_damping;
    for (int fbr = 0; fbr < nvfb; fbr++)
        for (int fbc = 0; fbc < nhfb; fbc++) {
            const int8_t v = fb_idx[fbr * nhfb + fbc];
            if (v >= 0) pcs_ptr->mi_grid_base[MI_SIZE_64X64 * fbr * pcs_ptr->mi_stride + MI_SIZE_64X64 * fbc]->mbmi.cdef_strength = v;
        }
    free(fb_idx);
    if (g_prof) stat_add(1, ST_CDEF, t0);
}

/* ===================================================================================================================
 * Loop restoration, apply side: svt_av1_loop_restoration_filter_frame(cm->frame_to_show, cm, 0) of rest_kernel
 * (EbRestProcess.c:530-534).  The search (restoration_seg_search, rest_finish_search) stays the reference's.
 * ================================================================================================================= */
#include "EbRestoration.h"
static __thread SvtB200LrUnit *t_units[3]     = {NULL, NULL, NULL};
static __thread int            t_units_cap[3] = {0, 0, 0};

void svt_cuda_lr_frame(PictureControlSet *pcs_ptr, SequenceControlSet *scs_ptr) {
    (void)scs_ptr;
    const int64_t     t0    = g_prof ? now_ns() : 0;
    Av1Common *       cm    = pcs_ptr->parent_pcs_ptr->av1_cm;
    Yv12BufferConfig *frame = cm->frame_to_show;
    const int         hbd   = cm->use_highbitdepth;
    SvtB200LrFrameParams p;
    SvtB200HostLrLines   lines[3];
    int32_t              n_units[3];
    memset(&p, 0, sizeof(p));
    p.optimized_lr = 0;
    for (int pl = 0; pl < 3; pl++) {
        RestorationInfo *rsi = &cm->rst_info[pl];
        rsi->optimized_lr    = 0; /* what svt_av1_loop_restoration_filter_frame(frame, cm, 0) sets (:1324) */
        p.plane[pl].frame_restoration_type = rsi->frame_restoration_type;
        p.plane[pl].restoration_unit_size  = rsi->restoration_unit_size;
        const int n = rsi->units_per_tile;
        if (t_units_cap[pl] < n) {
            free(t_units[pl]);
            t_units[pl]     = (SvtB200LrUnit *)malloc((size_t)n * sizeof(SvtB200LrUnit));
            t_units_cap[pl] = n;
            if (!t_units[pl]) die("malloc", -1);
        }
        for (int u = 0; u < n; u++) {
            const RestorationUnitInfo *ri = &rsi->unit_info[u];
            SvtB200LrUnit *            o  = &t_units[pl][u];
            o->restoration_type = ri->restoration_type;
            memcpy(o->vfilter, ri->wiener_info.vfilter, sizeof(o->vfilter));
            memcpy(o->hfilter, ri->wiener_info.hfilter, sizeof(o->hfilter));
            o->sgr_ep     = ri->sgrproj_info.ep;
            o->sgr_xqd[0] = ri->sgrproj_info.xqd[0];
            o->sgr_xqd[1] = ri->sgrproj_info.xqd[1];
        }
        n_units[pl]        = n;
        p.plane[pl].units  = t_units[pl];
        lines[pl].above    = rsi->boundaries.stripe_boundary_above + (RESTORATION_EXTRA_HORZ << hbd);
        lines[pl].below    = rsi->boundaries.stripe_boundary_below + (RESTORATION_EXTRA_HORZ << hbd);
        lines[pl].stride   = rsi->boundaries.stripe_boundary_stride;
    }
    SvtB200Frame f;
    memset(&f, 0, sizeof(f));
    f.y         = REAL_PTR(hbd, frame->buffers[0]);
    f.cb        = REAL_PTR(hbd, frame->buffers[1]);
    f.cr        = REAL_PTR(hbd, frame->buffers[2]);
    f.stride_y  = frame->strides[0];
    f.stride_c  = frame->strides[1];
    f.width     = frame->crop_widths[0];
    f.height    = frame->crop_heights[0];
    f.bit_depth = hbd ? (int)cm->bit_depth : 8;
    int rc      = svt_b200_engine_lr_frame(g_engine, &p, n_units, &f, lines);
    if (rc) die("svt_b200_engine_lr_frame", rc);
    if (g_prof) stat_add(1, ST_LR, t0);
}

/* compute_picture_spatial_statistics (EbPictureAnalysisProcess.c:2929-2974): SVT_CUDA_PA=1 computes pcs->y_mean / variance /
 * cb_mean / cr_mean of every SB and pic_avg_variance in one GPU call.  Returns 0 when the C loop must run. */
int svt_cuda_pa_statistics(PictureParentControlSet *pcs_ptr, EbPictureBufferDesc *input_picture_ptr,
                           EbPictureBufferDesc *input_padded_picture_ptr, uint32_t sb_total_count) {
    if (g_on <= 0 || !g_pa || input_picture_ptr->bit_depth != EB_8BIT) return 0;
    const int w = input_picture_ptr->width, h = input_picture_ptr->height;
    const int sbw = (w + 63) / 64, sbh = (h + 63) / 64;
    if ((uint32_t)(sbw * sbh) != sb_total_count || sb_total_count != pcs_ptr->sb_total_count) return 0;
    /* the SBs must be in raster order (sb_params_array is), checked on the last one */
    if (pcs_ptr->sb_params_array[sb_total_count - 1].origin_x != (sbw - 1) * 64 || pcs_ptr->sb_params_array[sb_total_count - 1].origin_y != (sbh - 1) * 64)
        return 0;
    const size_t n  = sb_total_count;
    uint8_t *    ym = (uint8_t *)malloc(n * (85 + 21 + 21) + n * 85 * 2 + 2);
    if (!ym) return 0;
    uint16_t *vr = (uint16_t *)(ym + n * (85 + 21 + 21) + ((n * (85 + 21 + 21)) & 1)) ;
    uint8_t * cbm = ym + n * 85, *crm = cbm + n * 21;
    uint16_t  avg = 0;
    /* luma from the padded picture (same samples inside the picture), chroma from the input picture, as the reference */
    const uint8_t *y  = input_padded_picture_ptr->buffer_y + input_padded_picture_ptr->origin_y * input_padded_picture_ptr->stride_y + input_padded_picture_ptr->origin_x;
    const uint8_t *cb = input_picture_ptr->buffer_cb + (input_picture_ptr->origin_y >> 1) * input_picture_ptr->stride_cb + (input_picture_ptr->origin_x >> 1);
    const uint8_t *cr = input_picture_ptr->buffer_cr + (input_picture_ptr->origin_y >> 1) * input_picture_ptr->stride_cr + (input_picture_ptr->origin_x >> 1);
    int rc = svt_b200_picture_mean_variance_host(y, input_padded_picture_ptr->stride_y, cb, cr, input_picture_ptr->stride_cb, w, h, ym, vr, cbm, crm, &avg);
    if (rc) die("svt_b200_picture_mean_variance_host", rc);
    for (uint32_t sb = 0; sb < sb_total_count; sb++) {
        memcpy(pcs_ptr->y_mean[sb], ym + (size_t)sb * 85, 85);
        memcpy(pcs_ptr->variance[sb], vr + (size_t)sb * 85, 85 * sizeof(uint16_t));
        memcpy(pcs_ptr->cb_mean[sb], cbm + (size_t)sb * 21, 21); /* the reference writes entries 0..20 only */
        memcpy(pcs_ptr->cr_mean[sb], crm + (size_t)sb * 21, 21);
    }
    pcs_ptr->pic_avg_variance = avg;
    free(ym);
    __sync_fetch_and_add(&g_pa_calls, 1);
    return 1;
}

/* The open-loop intra search loop of the ME process (EbMotionEstimationProcess.c:965-975): SVT_CUDA_OIS=1 and the TPL
 * controls of presets >= 5 (DC_PRED only) -> the thread that owns segment 0 searches every macroblock of the picture in one
 * GPU call and fills pcs->ois_mb_results; the other segments' threads skip their loop.  Returns 0 when the C loop must run. */
int svt_cuda_ois_segment(PictureParentControlSet *pcs_ptr, SequenceControlSet *scs_ptr, EbPictureBufferDesc *input_picture_ptr,
                         uint32_t segment_index) {
    if (g_on <= 0 || !g_ois) return 0;
    EbPictureBufferDesc *enh = pcs_ptr->enhanced_picture_ptr;
    if (!pcs_ptr->tpl_data.tpl_ctrls.tpl_opt_flag || input_picture_ptr->bit_depth != EB_8BIT || !enh) return 0;
    const int w = enh->width, h = enh->height;
    if (w != scs_ptr->seq_header.max_frame_width || h != scs_ptr->seq_header.max_frame_height || (w & 7) || (h & 7)) return 0;
    if (segment_index != 0) return 1;
    const int mbw = (w + 15) / 16, mbh = (h + 15) / 16;
    int64_t * cost = (int64_t *)malloc((size_t)mbw * mbh * sizeof(int64_t));
    if (!cost) die("svt_cuda_ois_segment: out of memory", -1);
    const uint8_t *y = input_picture_ptr->buffer_y + enh->origin_x + (size_t)enh->origin_y * input_picture_ptr->stride_y;
    int rc = svt_b200_ois_dc_picture_host(y, input_picture_ptr->stride_y, w, h, cost);
    if (rc) die("svt_b200_ois_dc_picture_host", rc);
    for (int i = 0; i < mbw * mbh; i++) {
        OisMbResults *r = pcs_ptr->ois_mb_results[i];
        memset(r, 0, sizeof(*r));
        r->intra_mode = DC_PRED;
        r->intra_cost = cost[i];
    }
    free(cost);
    __sync_fetch_and_add(&g_ois_calls, 1);
    return 1;
}
