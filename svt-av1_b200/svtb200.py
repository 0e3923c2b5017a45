"""ctypes binding of libsvtav1_b200.so (include/svt_av1_b200.h) — host-side convenience for tests and bench.py.

The product is the C-ABI library; this module only mirrors its structs and loads it.  There is no CPU
fallback: if the shared library is missing, `load()` raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SVTB200_LIB: an experimental build of the same library (kernel variants for tools/kernel_bench.py); default = the product
LIB_PATH = os.environ.get("SVTB200_LIB") or os.path.join(_HERE, "libsvtav1_b200.so")

ME_MAX_REFS, ME_LISTS, ME_PU, ME_MAX_MV, ME_MAX_CAND = 4, 2, 85, 7, 23


class Plane(C.Structure):
    _fields_ = [("stride", C.c_int32), ("origin_x", C.c_int32), ("origin_y", C.c_int32),
                ("width", C.c_int32), ("height", C.c_int32)]


class MeParams(C.Structure):
    _fields_ = [
        ("full", Plane), ("quarter", Plane), ("sixteenth", Plane),
        ("num_lists", C.c_int32), ("num_refs", C.c_int32 * 2), ("ref_dist", (C.c_int32 * 4) * 2),
        ("temporal_layer_index", C.c_int32), ("is_used_as_reference_flag", C.c_int32),
        ("enable_hme_flag", C.c_int32), ("enable_hme_level0_flag", C.c_int32),
        ("enable_hme_level1_flag", C.c_int32), ("enable_hme_level2_flag", C.c_int32),
        ("hme_search_method", C.c_int32), ("me_search_method", C.c_int32),
        ("number_hme_search_region_in_width", C.c_int32), ("number_hme_search_region_in_height", C.c_int32),
        ("hme_level0_total_search_area_width", C.c_int32), ("hme_level0_total_search_area_height", C.c_int32),
        ("hme_level0_max_total_search_area_width", C.c_int32),
        ("hme_level0_max_total_search_area_height", C.c_int32),
        ("hme_level0_search_area_in_width_array", C.c_int32 * 2),
        ("hme_level0_search_area_in_height_array", C.c_int32 * 2),
        ("hme_level0_max_search_area_in_width_array", C.c_int32 * 2),
        ("hme_level0_max_search_area_in_height_array", C.c_int32 * 2),
        ("hme_level1_search_area_in_width_array", C.c_int32 * 2),
        ("hme_level1_search_area_in_height_array", C.c_int32 * 2),
        ("hme_level2_search_area_in_width_array", C.c_int32 * 2),
        ("hme_level2_search_area_in_height_array", C.c_int32 * 2),
        ("search_area_width", C.c_int32), ("search_area_height", C.c_int32),
        ("max_me_search_width", C.c_int32), ("max_me_search_height", C.c_int32),
        ("enable_me_hme_ref_pruning", C.c_int32),
        ("prune_ref_if_hme_sad_dev_bigger_than_th", C.c_int32),
        ("prune_ref_if_me_sad_dev_bigger_than_th", C.c_int32),
        ("enable_me_sr_adjustment", C.c_int32),
        ("reduce_me_sr_based_on_mv_length_th", C.c_int32), ("stationary_hme_sad_abs_th", C.c_int32),
        ("stationary_me_sr_divisor", C.c_int32), ("reduce_me_sr_based_on_hme_sad_abs_th", C.c_int32),
        ("me_sr_divisor_for_low_hme_sad", C.c_int32),
        ("max_number_of_pus_per_sb", C.c_int32), ("rc_dist_from_8x8", C.c_int32),
    ]


class MePlanes(C.Structure):
    _fields_ = [("full", C.c_void_p), ("quarter", C.c_void_p), ("sixteenth", C.c_void_p)]


class HmeResult(C.Structure):
    _fields_ = [("sc_x", C.c_int16), ("sc_y", C.c_int16), ("do_ref", C.c_uint32), ("hme_sad", C.c_uint64)]


class MeOutputs(C.Structure):
    _fields_ = [("best_sad", C.c_void_p), ("best_mv", C.c_void_p), ("hme", C.c_void_p),
                ("me_mv", C.c_void_p), ("me_cand", C.c_void_p), ("total_cand", C.c_void_p),
                ("rc_me_distortion", C.c_void_p)]


class Frame(C.Structure):
    _fields_ = [("y", C.c_void_p), ("cb", C.c_void_p), ("cr", C.c_void_p), ("stride_y", C.c_int32),
                ("stride_c", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("bit_depth", C.c_int32)]


class CdefSearchParams(C.Structure):
    _fields_ = [("mi_rows", C.c_int32), ("mi_cols", C.c_int32), ("pri_damping", C.c_int32),
                ("n_strengths", C.c_int32), ("pri_strength", C.c_int32 * 64), ("sec_strength", C.c_int32 * 64)]


class CdefApplyParams(C.Structure):
    _fields_ = [("mi_rows", C.c_int32), ("mi_cols", C.c_int32), ("damping", C.c_int32),
                ("y_strength", C.c_int32 * 8), ("uv_strength", C.c_int32 * 8)]


class Tu(C.Structure):
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("plane", C.c_int32), ("tx_type", C.c_int32)]


class QuantPlane(C.Structure):
    _fields_ = [("zbin", C.c_int16 * 2), ("round", C.c_int16 * 2), ("quant", C.c_int16 * 2),
                ("quant_shift", C.c_int16 * 2), ("dequant", C.c_int16 * 2), ("round_fp", C.c_int16 * 2),
                ("quant_fp", C.c_int16 * 2)]


class EncodeParams(C.Structure):
    _fields_ = [("tx_size", C.c_int32), ("use_fp", C.c_int32), ("q", QuantPlane * 3)]


class CdefDecideParams(C.Structure):
    _fields_ = [("mi_rows", C.c_int32), ("mi_cols", C.c_int32), ("n_strengths", C.c_int32), ("reserved", C.c_int32), ("lambda_", C.c_uint64),
                ("filter_strength", C.c_int32 * 64)]


class CdefDecision(C.Structure):
    _fields_ = [("cdef_bits", C.c_int32), ("nb_cdef_strengths", C.c_int32), ("y_strength", C.c_int32 * 8), ("uv_strength", C.c_int32 * 8),
                ("y_index", C.c_int32 * 8), ("uv_index", C.c_int32 * 8), ("sb_count", C.c_int32), ("reserved", C.c_int32)]


class TfBlock(C.Structure):
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("block_error", C.c_double * 4), ("d_factor", C.c_double * 4)]


class TfParams(C.Structure):
    _fields_ = [("den", C.c_double * 3), ("chroma", C.c_int32), ("block_w", C.c_int32), ("block_h", C.c_int32)]


class TfAccum(C.Structure):
    _fields_ = [("accum", C.c_void_p * 3), ("count", C.c_void_p * 3), ("stride_y", C.c_int32), ("stride_c", C.c_int32)]


class TuEx(C.Structure):
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("plane", C.c_uint8), ("tx_type", C.c_uint8), ("tx_size", C.c_uint8),
                ("pf_shape", C.c_uint8), ("qset", C.c_uint16), ("reserved", C.c_uint16)]


class EncodeParamsEx(C.Structure):
    _fields_ = [("use_fp", C.c_int32), ("n_qsets", C.c_int32), ("qsets", C.POINTER(QuantPlane * 3))]


TX_W = [4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64]
TX_H = [4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16]


class DlfMi(C.Structure):
    _fields_ = [("tx_w", C.c_uint8 * 2), ("tx_h", C.c_uint8 * 2), ("blk_w", C.c_uint8 * 2), ("blk_h", C.c_uint8 * 2),
                ("skip_inter", C.c_uint8), ("lvl_y", C.c_uint8 * 2), ("lvl_u", C.c_uint8), ("lvl_v", C.c_uint8),
                ("lvl_class", C.c_uint8), ("pad", C.c_uint8 * 2)]


class DlfParams(C.Structure):
    _fields_ = [("mi_rows", C.c_int32), ("mi_cols", C.c_int32), ("mi_stride", C.c_int32), ("sharpness", C.c_int32),
                ("filter_level", C.c_int32 * 2), ("filter_level_u", C.c_int32), ("filter_level_v", C.c_int32),
                ("plane_start", C.c_int32), ("plane_end", C.c_int32)]


class LfFrameInit(C.Structure):
    _fields_ = [("mode_ref_delta_enabled", C.c_int32), ("ref_deltas", C.c_int8 * 8), ("mode_deltas", C.c_int8 * 2),
                ("segmentation_enabled", C.c_int32), ("seg_feature_mask", C.c_uint8 * 8),
                ("seg_feature_data", (C.c_int16 * 8) * 8)]


class LpfPickParams(C.Structure):
    _fields_ = [("dlf", DlfParams), ("init", LfFrameInit), ("method", C.c_int32), ("loop_filter_mode", C.c_int32),
                ("tx_mode_only_4x4", C.c_int32), ("q_ac", C.c_int32), ("key_frame", C.c_int32), ("last_level", C.c_int32 * 4)]


class LrUnit(C.Structure):
    _fields_ = [("restoration_type", C.c_int32), ("vfilter", C.c_int16 * 8), ("hfilter", C.c_int16 * 8), ("sgr_ep", C.c_int32),
                ("sgr_xqd", C.c_int32 * 2)]


class LrPlane(C.Structure):
    _fields_ = [("frame_restoration_type", C.c_int32), ("restoration_unit_size", C.c_int32), ("units", C.c_void_p)]


class LrFrameParams(C.Structure):
    _fields_ = [("plane", LrPlane * 3), ("optimized_lr", C.c_int32)]


class InterpFilterParams(C.Structure):  # EbDefinitions.h:493-498
    _fields_ = [("filter_ptr", C.c_void_p), ("taps", C.c_uint16), ("subpel_shifts", C.c_uint16), ("interp_filter", C.c_int32)]


class ConvolveParams(C.Structure):  # EbDefinitions.h:379-392
    _fields_ = [("ref", C.c_int32), ("do_average", C.c_int32), ("dst", C.c_void_p), ("dst_stride", C.c_int32),
                ("round_0", C.c_int32), ("round_1", C.c_int32), ("plane", C.c_int32), ("is_compound", C.c_int32),
                ("use_jnt_comp_avg", C.c_int32), ("fwd_offset", C.c_int32), ("bck_offset", C.c_int32),
                ("use_dist_wtd_comp_avg", C.c_int32)]


class InterJob(C.Structure):
    _fields_ = [("plane", C.c_uint8), ("n_refs", C.c_uint8), ("bw", C.c_uint8), ("bh", C.c_uint8), ("ref", C.c_uint8 * 2),
                ("filter_x", C.c_uint8), ("filter_y", C.c_uint8), ("use_jnt_comp_avg", C.c_uint8), ("fwd_offset", C.c_uint8),
                ("bck_offset", C.c_uint8), ("reserved", C.c_uint8), ("dst_x", C.c_int16), ("dst_y", C.c_int16),
                ("pre_x", C.c_int16), ("pre_y", C.c_int16), ("mv_row", C.c_int16 * 2), ("mv_col", C.c_int16 * 2),
                ("mb_to_left_edge", C.c_int32), ("mb_to_right_edge", C.c_int32), ("mb_to_top_edge", C.c_int32),
                ("mb_to_bottom_edge", C.c_int32)]


INTER_JOB_DTYPE = [("plane", "u1"), ("n_refs", "u1"), ("bw", "u1"), ("bh", "u1"), ("ref", "u1", 2), ("filter_x", "u1"),
                   ("filter_y", "u1"), ("use_jnt_comp_avg", "u1"), ("fwd_offset", "u1"), ("bck_offset", "u1"), ("reserved", "u1"),
                   ("dst_x", "<i2"), ("dst_y", "<i2"), ("pre_x", "<i2"), ("pre_y", "<i2"), ("mv_row", "<i2", 2),
                   ("mv_col", "<i2", 2), ("mb_to_left_edge", "<i4"), ("mb_to_right_edge", "<i4"), ("mb_to_top_edge", "<i4"),
                   ("mb_to_bottom_edge", "<i4")]


class SubpelParams(C.Structure):
    _fields_ = [("allow_hp", C.c_int32), ("forced_stop", C.c_int32), ("iters_per_step", C.c_int32), ("subpel_search_type", C.c_int32),
                ("mv_cost_type", C.c_int32), ("error_per_bit", C.c_int32), ("mvjcost", C.c_int32 * 4), ("max_block_w", C.c_int32),
                ("max_block_h", C.c_int32), ("mvcost", C.c_void_p * 2)]


SUBPEL_JOB_DTYPE = [("blk_x", "<i2"), ("blk_y", "<i2"), ("bw", "u1"), ("bh", "u1"), ("ref", "u1"), ("reserved", "u1"),
                    ("start_mv_row", "<i2"), ("start_mv_col", "<i2"), ("ref_mv_row", "<i2"), ("ref_mv_col", "<i2"),
                    ("col_min", "<i2"), ("col_max", "<i2"), ("row_min", "<i2"), ("row_max", "<i2")]
SUBPEL_RESULT_DTYPE = [("mv_row", "<i2"), ("mv_col", "<i2"), ("besterr", "<i4"), ("distortion", "<i4"), ("sse", "<u4")]


class HostMePicture(C.Structure):  # SvtB200HostMePicture
    _fields_ = [("key", C.c_void_p), ("tag", C.c_uint64), ("full", C.c_void_p), ("quarter", C.c_void_p), ("sixteenth", C.c_void_p)]


class HostLrLines(C.Structure):  # SvtB200HostLrLines
    _fields_ = [("above", C.c_void_p), ("below", C.c_void_p), ("stride", C.c_int32)]


class EngineStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("me_pictures", "dlf_frames", "cdef_frames", "lr_frames", "me_plane_uploads", "me_plane_hits",
                                          "h2d_bytes", "d2h_bytes", "pinned_bytes", "ns_slot_wait", "ns_plane_wait", "ns_issue",
                                          "ns_sync", "ns_host_copy")]


# input-resolution classes (EbDefinitions.h ResolutionRange) and the luma sample counts that bound them
RES_240P, RES_360P, RES_480P, RES_720P, RES_1080P, RES_4K, RES_8K = range(7)
_RES_TH = (0x28500, 0x4CE00, 0xA1400, 0x16DA00, 0x535200, 0x140A000)
PRESET_MRS, PRESET_MR = -2, -1


def input_resolution(width, height):
    """derive_input_resolution: the resolution class of a width x height picture."""
    n = width * height
    return next((i for i, th in enumerate(_RES_TH) if n < th), RES_8K)


def me_params(preset, width, height, n_l0=1, n_l1=1, dist=((1, 2, 3, 4), (1, 2, 3, 4)), temporal_layer=1, is_ref=1,
              input_resolution_class=None):
    """ME parameters of `preset` (-2 = MRS .. 8) for non-screen content, default ME/HME, 30 fps, single pass, as
    signal_derivation_me_kernel_oq derives them (EbMotionEstimationProcess.c:113-420: set_me_hme_params_oq,
    set_me_hme_ref_prune_ctrls, set_me_sr_adjustment_ctrls).  `input_resolution_class` (RES_*) overrides the class
    derived from width x height, so that a small picture can carry a larger class's table.  Raises ValueError where
    the preset uses one-decimation HME (MR / MRS at <= 720p), which the library does not implement.  Tests check
    this table against the reference's own derivation (oracle/_ref) when it is available."""
    if not PRESET_MRS <= preset <= 8:
        raise ValueError(f"preset {preset} out of range")
    res = input_resolution(width, height) if input_resolution_class is None else input_resolution_class
    if preset <= PRESET_MR and res <= RES_720P:
        raise ValueError(f"preset {preset} at resolution class {res} uses one-decimation HME")
    p = MeParams()
    geo = me_geometry(width, height)
    p.full, p.quarter, p.sixteenth = geo
    p.num_lists = 2 if n_l1 > 0 else 1
    p.num_refs[0], p.num_refs[1] = n_l0, n_l1
    for l in range(2):
        for r in range(4):
            p.ref_dist[l][r] = dist[l][r]
    p.temporal_layer_index, p.is_used_as_reference_flag = temporal_layer, is_ref
    p.enable_hme_flag = p.enable_hme_level0_flag = p.enable_hme_level1_flag = p.enable_hme_level2_flag = 1
    p.hme_search_method = p.me_search_method = 0 if preset <= PRESET_MRS else 1  # full SAD at MRS, else sub-sampled
    p.number_hme_search_region_in_width = p.number_hme_search_region_in_height = 2
    # full-pel search area (scaled by 3/2 below: 30 fps is a low frame rate) and its cap
    if preset <= 2:
        sa = 64
        max_w = max_h = {0: 256, 1: 192, 2: 128}[max(preset, 0)]
    elif preset <= 5:
        sa, max_w, max_h = 16, 64, 64
    else:
        sa, max_w, max_h = 16, 64, 32
    p.search_area_width = p.search_area_height = sa * 3 // 2
    p.max_me_search_width, p.max_me_search_height = max_w, max_h
    # HME level 0: total area over the 2x2 regions, each region gets half of it in each direction
    if preset <= 1:
        total, max_total = (120 if res <= RES_1080P else 240), 480
    else:
        total, max_total = 32, 164
    p.hme_level0_total_search_area_width = p.hme_level0_total_search_area_height = total
    p.hme_level0_max_total_search_area_width = p.hme_level0_max_total_search_area_height = max_total
    l12_w, l12_h = (16, 16) if preset <= 4 else (8, 3)
    for i in range(2):
        p.hme_level0_search_area_in_width_array[i] = p.hme_level0_search_area_in_height_array[i] = total // 2
        p.hme_level0_max_search_area_in_width_array[i] = p.hme_level0_max_search_area_in_height_array[i] = max_total // 2
        p.hme_level1_search_area_in_width_array[i] = p.hme_level2_search_area_in_width_array[i] = l12_w
        p.hme_level1_search_area_in_height_array[i] = p.hme_level2_search_area_in_height_array[i] = l12_h
    # HME / ME reference pruning: off at MR and MRS, level 2 at M0-M2, level 4 above
    if preset <= PRESET_MR:
        p.enable_me_hme_ref_pruning = 0
        p.prune_ref_if_hme_sad_dev_bigger_than_th = p.prune_ref_if_me_sad_dev_bigger_than_th = 0xFFFF
    else:
        p.enable_me_hme_ref_pruning = 1
        p.prune_ref_if_hme_sad_dev_bigger_than_th = 80 if preset <= 2 else 30
        p.prune_ref_if_me_sad_dev_bigger_than_th = 60
    # HME-based search-area adjustment: off at MRS (level 0 leaves the thresholds at zero), level 2 above
    if preset > PRESET_MRS:
        p.enable_me_sr_adjustment = 1
        p.reduce_me_sr_based_on_mv_length_th = 4
        p.stationary_hme_sad_abs_th = 12000
        p.stationary_me_sr_divisor = 8
        p.reduce_me_sr_based_on_hme_sad_abs_th = 6000
        p.me_sr_divisor_for_low_hme_sad = 8
    p.max_number_of_pus_per_sb = 85
    p.rc_dist_from_8x8 = 1 if res <= RES_480P else 0
    return p


def preset8_me_params(width, height, n_l0=1, n_l1=1, dist=((1, 2, 3, 4), (1, 2, 3, 4)), temporal_layer=1,
                      is_ref=1):
    """ME parameters of preset 8 (ENC_M8), 30 fps: me_params(8, ...)."""
    return me_params(8, width, height, n_l0, n_l1, dist, temporal_layer, is_ref)


def me_geometry(width, height):
    """Plane geometry the reference allocates for ME: full-res padded by sb_sz+ME_FILTER_TAP = 68, the 1/4 and
    1/16 planes by sb_sz>>1 and sb_sz>>2 (EbEncHandle.c:971-988, 1030-1053)."""
    def mk(w, h, pad):
        return Plane(w + 2 * pad, pad, pad, w, h)
    return mk(width, height, 68), mk(width >> 1, height >> 1, 32), mk(width >> 2, height >> 2, 16)


_lib = None


def load():
    """Load the CUDA C-ABI library. Raises (never falls back) if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} missing: run __graft_entry__.build() (nvcc sm_90a); there is no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    lib.svt_b200_last_error.restype = C.c_char_p
    lib.svt_b200_launch_count.restype = C.c_uint64
    lib.svt_b200_malloc.restype = C.c_void_p
    lib.svt_b200_malloc.argtypes = [C.c_size_t]
    lib.svt_b200_free.argtypes = [C.c_void_p]
    lib.svt_b200_malloc_host.restype = C.c_void_p
    lib.svt_b200_malloc_host.argtypes = [C.c_size_t]
    lib.svt_b200_free_host.argtypes = [C.c_void_p]
    lib.svt_b200_memcpy_h2d.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.svt_b200_memcpy_d2h.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.svt_b200_stream_sync.argtypes = [C.c_void_p]
    lib.svt_b200_me_scratch_bytes.restype = C.c_size_t
    lib.svt_b200_me_scratch_bytes.argtypes = [C.POINTER(MeParams)]
    lib.svt_b200_me_picture.argtypes = [C.POINTER(MeParams), C.POINTER(MePlanes), C.POINTER(MePlanes),
                                        C.POINTER(MeOutputs), C.c_void_p, C.c_void_p]
    lib.svt_nxm_sad_kernel_cuda.restype = C.c_uint32
    lib.svt_b200_handle_transform64.restype = C.c_uint64
    lib.svt_b200_dlf_frame.argtypes = [C.POINTER(DlfParams), C.POINTER(Frame), C.c_void_p, C.c_void_p]
    lib.svt_b200_frame_sse.argtypes = [C.POINTER(Frame), C.POINTER(Frame), C.c_void_p, C.c_void_p]
    for n in ("64x64", "64x32", "32x64", "64x16", "16x64"):
        getattr(lib, f"svt_handle_transform{n}_cuda").restype = C.c_uint64
    lib.svt_b200_encode_tus.argtypes = [C.POINTER(EncodeParams), C.POINTER(Frame), C.POINTER(Frame), C.POINTER(Frame),
                                        C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.svt_b200_picture_mean_variance.argtypes = [C.POINTER(Frame), C.c_int32] + [C.c_void_p] * 7
    lib.svt_b200_cdef_decide_table.argtypes = [C.c_int, C.POINTER(CdefDecideParams)]
    lib.svt_b200_engine_dlf_cdef_frame_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(CdefSearchParams), C.POINTER(CdefDecideParams),
                                                       C.c_int32, C.c_int32, C.POINTER(Frame), C.POINTER(Frame), C.c_void_p, C.c_int32,
                                                       C.POINTER(CdefDecision), C.c_void_p]
    lib.svt_b200_ois_dc_picture.argtypes = [C.POINTER(Frame), C.c_void_p, C.c_void_p]
    lib.svt_b200_ois_dc_picture_host.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.svt_b200_tf_planewise.argtypes = [C.POINTER(TfParams), C.POINTER(Frame), C.POINTER(Frame), C.c_void_p, C.c_int32,
                                          C.POINTER(TfAccum), C.c_void_p]
    lib.svt_b200_tf_central.argtypes = [C.POINTER(Frame), C.POINTER(TfAccum), C.c_int32, C.c_void_p]
    lib.svt_b200_tf_normalize.argtypes = [C.POINTER(Frame), C.POINTER(TfAccum), C.c_int32, C.c_void_p, C.c_void_p]
    lib.svt_b200_tf_expf_checksum.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64)]
    lib.svt_b200_tf_planewise_block_host.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                                     C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_uint32, C.c_uint32,
                                                     C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)] + [C.c_void_p] * 6
    lib.svt_b200_encode_tus_ex.argtypes = [C.POINTER(EncodeParamsEx), C.POINTER(Frame), C.POINTER(Frame), C.POINTER(Frame),
                                           C.POINTER(TuEx), C.c_int32, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_size_t, C.c_void_p]
    lib.svt_b200_cdef_search.argtypes = [C.POINTER(CdefSearchParams), C.POINTER(Frame), C.POINTER(Frame), C.c_void_p,
                                         C.c_int32, C.c_void_p, C.c_void_p]
    lib.svt_b200_cdef_apply.argtypes = [C.POINTER(CdefApplyParams), C.POINTER(Frame), C.POINTER(Frame), C.c_void_p,
                                        C.c_int32, C.c_void_p, C.c_void_p]
    _lib = lib
    return lib


def check(rc, lib=None):
    if rc != 0:
        lib = lib or load()
        raise RuntimeError(f"svt_b200 call failed rc={rc}: {lib.svt_b200_last_error().decode()}")
