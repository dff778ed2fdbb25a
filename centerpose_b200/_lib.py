"""ctypes binding of libcenterpose_b200.so (include/centerpose_b200.h).

The product path has NO fallback: if the shared library is missing or a call
fails, a RuntimeError is raised.  (`python -m centerpose_b200.build` or
`__graft_entry__.build()` produces the library in-tree.)
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CP_LIB_PATH") or os.path.join(HERE, "libcenterpose_b200.so")      # CP_LIB_PATH: A/B another build

CP_MAX_HEADS = 16
CP_POSE_RECORD = 192
CP_DETS_RECORD = 128
CP_META_DOUBLES = 16
CP_MAX_K = 128
CP_MAX_MODELS = 16

CP_ARCH_DLA34 = 0
CP_ARCH_DLAV1_34 = 1
CP_ARCH_RES_18, CP_ARCH_RES_34, CP_ARCH_RES_50, CP_ARCH_RES_101, CP_ARCH_RES_152 = 2, 3, 4, 5, 6
CP_PREC_FP32 = 0
CP_PREC_TF32X3 = 1
CP_PREC_BF16 = 2
CP_PREC_TF32 = 3
PRECISIONS = {"fp32": CP_PREC_FP32, "tf32x3": CP_PREC_TF32X3, "bf16": CP_PREC_BF16, "tf32": CP_PREC_TF32}

# cp_pose_field
P_SCORE, P_CLS, P_STATUS, P_NPTS, P_BBOX, P_CT, P_KPS = 0, 1, 2, 3, 4, 8, 10
P_KPS_DISP_MEAN, P_KPS_HM_MEAN, P_KPS_HM_STD, P_KPS_HM_HEIGHT, P_KPS_DISP_STD = 26, 42, 58, 74, 82
P_OBJ_SCALE, P_OBJ_SCALE_UNC, P_TRACKING, P_TRACKING_HP = 98, 101, 104, 106
P_LOCATION, P_QUAT, P_REPROJ, P_PROJ_CUBOID, P_KPS_3D_CAM, P_KPS_PNP, P_SRC_INDEX = 122, 125, 129, 130, 146, 173, 191
# cp_dets_field
D_BBOX, D_SCORE, D_CLS, D_KPS, D_OBJ_SCALE, D_OBJ_SCALE_UNC, D_TRACKING, D_TRACKING_HP = 0, 4, 5, 6, 22, 25, 28, 30
D_KPS_DISP_MEAN, D_KPS_DISP_STD, D_KPS_HM_MEAN, D_KPS_HM_STD, D_KPS_HM_HEIGHT, D_IND = 46, 62, 78, 94, 110, 118
# cp_track_field
CP_TRACK_RECORD = 320
T_ID, T_AGE, T_ACTIVE, T_IN_BOXES, T_PNP2_STATUS, T_CONF_AVG = 192, 193, 194, 195, 196, 197
T_KPS_FUSION_MEAN, T_KPS_FUSION_STD, T_KPS_MEAN_KF, T_KPS_STD_KF = 200, 216, 232, 248
T_OBJ_SCALE_KF, T_OBJ_SCALE_UNC_KF, T_KPS_PNP_KF, T_KPS_3D_CAM_KF = 264, 267, 270, 288
# cp_seed_field
CP_SEED_RECORD = 264
S_KPS_FUSION_MEAN, S_KPS_FUSION_STD, S_KPS_GT, S_HAS_CT, S_HAS_KPS_GT, S_KPS_PNP_KF, S_HAS_KPS_PNP_KF = 192, 208, 224, 242, 243, 244, 262
# cp_render_mode
RENDER_TRACKS, RENDER_GT, RENDER_EMPTY = 0, 1, 2
# cp_pnp_status
PNP_NOT_RUN, PNP_OK, PNP_INVISIBLE, PNP_BEHIND, PNP_FEW_POINTS, PNP_SOLVER_FAIL = 0, 1, 2, 3, 4, 5

EXPORTS = [
    "cp_version", "cp_last_error", "cp_plan_create", "cp_plan_destroy", "cp_plan_load_weights",
    "cp_forward", "cp_plan_bytes", "cp_plan_forward_launches", "cp_decode_workspace_bytes",
    "cp_decode_pnp", "cp_infer", "cp_dcn_v2_forward", "cp_preprocess", "cp_plan_num_ops", "cp_plan_profile",
    "cp_dcn_v2_forward_ex", "cp_conv2d", "cp_dcn_v2_backward",
    "cp_preprocess_affine", "cp_tracker_create", "cp_tracker_destroy", "cp_tracker_reset", "cp_tracker_step", "cp_tracker_render",
    "cp_tracker_render_ex", "cp_tracker_seed", "cp_plan_op_desc", "cp_plan_arena", "cp_plan_run_ops",
    "cp_preprocess_ragged", "cp_tracker_step_ex", "cp_tracker_render_ex2", "cp_tracker_seed_ex",
    "cp_plan_create_multi", "cp_plan_load_weights_model", "cp_plan_num_models", "cp_plan_op_desc_model", "cp_infer_multi",
    "cp_plan_create_multi_track", "cp_infer_multi_track", "cp_tracker_create_multi",
    "cp_plan_create_ex", "cp_plan_memory", "cp_plan_allocations", "cp_preprocess_yuv420",
    "cp_preprocess_slots_dev", "cp_tracker_reset_dev", "cp_tracker_render_dev",
    "cp_preprocess_frame_table_bytes", "cp_preprocess_frame_table", "cp_preprocess_slots_ragged_dev",
    "cp_preprocess_slots_rows_dev", "cp_gather_rows_dev", "cp_tracker_render_dev2", "cp_tracker_step_dev",
    "cp_preprocess_formats", "cp_preprocess_frame_table_formats", "cp_plan_op_ksegments", "cp_plan_ksegments",
    "cp_preprocess_remap", "cp_preprocess_frame_table_maps", "cp_preprocess_resize_affine",
    "cp_jpeg_parse", "cp_jpeg_workspace_bytes", "cp_jpeg_decode", "cp_jpeg_last_rounds",
    "cp_jpeg_slots_workspace_bytes", "cp_jpeg_slots_block_bytes", "cp_jpeg_slots_prepare", "cp_jpeg_decode_slots_dev",
    "cp_jpeg_mask_counts_dev",
]

# cp_pixel_format; "bgr" is the interleaved uint8 [H,W,3] input of every other pre-process entry point.  The camera
# formats carry ffmpeg's pix_fmt names; CP_PIX_PER_FRAME launches a frame table of per-frame formats, and CP_PIX_REMAP
# OR-ed into either launches a table with coordinate maps (cp_preprocess_frame_table_maps).
CP_PIX_NV12, CP_PIX_I420, CP_PIX_BGR = 0, 1, 2
CP_PIX_RGB24, CP_PIX_RGBA, CP_PIX_BGRA, CP_PIX_YUYV422, CP_PIX_UYVY422 = 16, 17, 18, 32, 33
CP_PIX_GRAY, CP_PIX_BAYER_RGGB8, CP_PIX_BAYER_BGGR8, CP_PIX_BAYER_GBRG8, CP_PIX_BAYER_GRBG8 = 48, 49, 50, 51, 52
CP_PIX_PER_FRAME = 64
CP_PIX_REMAP = 128
# the colour formats, and the sensor formats: one uint8 [H,W] plane per frame, mono or a Bayer mosaic named after its
# pixels (0,0) (0,1) / (1,0) (1,1) as ffmpeg, V4L2 and ROS name it
PIXEL_FORMATS = ("bgr", "nv12", "i420", "rgb24", "rgba", "bgra", "yuyv422", "uyvy422")
SENSOR_FORMATS = ("gray", "bayer_rggb8", "bayer_bggr8", "bayer_gbrg8", "bayer_grbg8")
PIXEL_FORMAT_CODES = {"bgr": CP_PIX_BGR, "nv12": CP_PIX_NV12, "i420": CP_PIX_I420, "rgb24": CP_PIX_RGB24,
                      "rgba": CP_PIX_RGBA, "bgra": CP_PIX_BGRA, "yuyv422": CP_PIX_YUYV422, "uyvy422": CP_PIX_UYVY422,
                      "gray": CP_PIX_GRAY, "bayer_rggb8": CP_PIX_BAYER_RGGB8, "bayer_bggr8": CP_PIX_BAYER_BGGR8,
                      "bayer_gbrg8": CP_PIX_BAYER_GBRG8, "bayer_grbg8": CP_PIX_BAYER_GRBG8}

# cp_jpeg_refusal: why cp_jpeg_parse refuses a file; cp_jpeg_error: the bits of a frame's error word after cp_jpeg_decode
JPEG_REFUSALS = {0: "ok", 1: "not a JPEG file", 2: "truncated header", 3: "progressive JPEG", 4: "lossless JPEG",
                 5: "arithmetic coding", 6: "samples other than 8 bits", 7: "not 1 or 3 components",
                 8: "more than one scan", 9: "height set by a DNL marker", 10: "unsupported chroma sampling",
                 11: "RGB-coded JPEG", 12: "missing or malformed DQT / DHT", 13: "malformed header",
                 14: "more than 2^30 pixels"}
JPEG_ERR_CODE, JPEG_ERR_RUN, JPEG_ERR_SHORT, JPEG_ERR_RESTART, JPEG_ERR_SYNC = 1, 2, 4, 8, 16
JPEG_ERRORS = {JPEG_ERR_CODE: "invalid Huffman code", JPEG_ERR_RUN: "AC run past coefficient 63",
               JPEG_ERR_SHORT: "restart segment ends early", JPEG_ERR_RESTART: "missing or misnumbered RST marker",
               JPEG_ERR_SYNC: "Huffman synchronisation timed out"}

# cp_plan_create_ex / cp_plan_memory flags
CP_PLAN_REUSE_ACTIVATIONS = 1
CP_PLAN_MULTI_TRACK = 2
CP_PLAN_BATCH_INVARIANT = 32

# cp_kpath: how a conv_tma / dcn_tma launch summed its K segments (cp_plan_op_ksegments)
KPATH_NONE, KPATH_ONE, KPATH_SPLIT, KPATH_FOLD = 0, 1, 2, 3

# cp_op_family
FAM_NONE, FAM_IGEMM_FP32, FAM_STEM, FAM_CONV3_C16, FAM_IGEMM_UMMA, FAM_CONV_TMA, FAM_DCN_TMA = 0, 1, 2, 3, 4, 5, 6
FAM_MAXPOOL, FAM_UPADD, FAM_GN_RELU, FAM_GRU = 7, 8, 9, 10
FAMILY_NAMES = {FAM_NONE: "fused", FAM_IGEMM_FP32: "igemm_fp32", FAM_STEM: "stem", FAM_CONV3_C16: "conv3_c16",
                FAM_IGEMM_UMMA: "igemm_umma", FAM_CONV_TMA: "conv_tma", FAM_DCN_TMA: "dcn_tma", FAM_MAXPOOL: "maxpool",
                FAM_UPADD: "upadd", FAM_GN_RELU: "gn_relu", FAM_GRU: "gru"}


class CpJpegHuff(ctypes.Structure):
    _fields_ = [("look", ctypes.c_uint16 * 512), ("maxcode", ctypes.c_int32 * 18), ("valoffset", ctypes.c_int32 * 18),
                ("vals", ctypes.c_uint8 * 256)]


class CpJpegHeader(ctypes.Structure):
    _fields_ = ([(n, ctypes.c_int32) for n in ("status", "width", "height", "out_h", "out_w", "orientation", "ncomp",
                                                "hmax", "vmax", "mcux", "mcuy", "blocks_per_mcu", "restart_interval")] +
                [("scan_begin", ctypes.c_int64), ("scan_end", ctypes.c_int64), ("comp_h", ctypes.c_int32 * 3),
                 ("comp_v", ctypes.c_int32 * 3), ("quant", (ctypes.c_int16 * 64) * 3), ("dc", CpJpegHuff * 3),
                 ("ac", CpJpegHuff * 3)])


class CpOpStat(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 96), ("kind", ctypes.c_int32), ("ms", ctypes.c_float),
                ("flops", ctypes.c_double), ("bytes", ctypes.c_double)]


class CpActDesc(ctypes.Structure):
    _fields_ = [("off", ctypes.c_int64), ("ext", ctypes.c_int32), ("C", ctypes.c_int32), ("H", ctypes.c_int32),
                ("W", ctypes.c_int32), ("stride", ctypes.c_int32)]


class CpOpDesc(ctypes.Structure):
    _fields_ = ([("name", ctypes.c_char * 96)] +
                [(n, ctypes.c_int32) for n in ("kind", "family", "x3", "nsrc")] +
                [("src", CpActDesc * 4), ("out", CpActDesc), ("out_head", ctypes.c_int32)] +
                [(n, ctypes.c_int32) for n in ("kh", "stride", "pad", "Cin", "Cout", "CoutPad", "Kpad")] +
                [("w", ctypes.c_void_p), ("w_ld", ctypes.c_int32), ("bias", ctypes.c_void_p)] +
                [(n, ctypes.c_int32) for n in ("relu", "has_res", "res_after_relu")] +
                [("res", CpActDesc), ("om", CpActDesc), ("up_w", ctypes.c_void_p), ("f", ctypes.c_int32),
                 ("has_skip", ctypes.c_int32), ("skip", CpActDesc), ("gamma", ctypes.c_void_p),
                 ("beta", ctypes.c_void_p), ("groups", ctypes.c_int32), ("gx", CpActDesc), ("gh", CpActDesc),
                 ("gprev", CpActDesc), ("first_step", ctypes.c_int32)] +
                [(n, ctypes.c_int32) for n in ("fuse_heads", "fused_away", "parent", "n_children")] +
                [("children", ctypes.c_int32 * CP_MAX_HEADS)])


class CpOpLaunch(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("family", "BN", "ksplit", "grid")]


class CpMemoryInfo(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int64) for n in ("activation_bytes", "weight_bytes", "tile_bytes", "workspace_bytes")]


class CpActAlloc(ctypes.Structure):
    _fields_ = [("floats", ctypes.c_int64), ("off", ctypes.c_int64), ("first", ctypes.c_int32), ("last", ctypes.c_int32)]


class CpConfig(ctypes.Structure):
    _fields_ = [
        ("arch", ctypes.c_int32), ("tracking", ctypes.c_int32), ("tracking_task_gru", ctypes.c_int32),
        ("max_batch", ctypes.c_int32), ("height", ctypes.c_int32), ("width", ctypes.c_int32),
        ("precision", ctypes.c_int32), ("device", ctypes.c_int32), ("head_conv", ctypes.c_int32),
        ("num_heads", ctypes.c_int32),
        ("head_names", ctypes.c_char_p * CP_MAX_HEADS),
        ("head_channels", ctypes.c_int32 * CP_MAX_HEADS),
    ]


class CpHeads(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in (
        "hm", "wh", "hps", "reg", "hm_hp", "hp_offset", "scale", "hps_uncertainty",
        "scale_uncertainty", "tracking", "tracking_hp")]


class CpDecodeParams(ctypes.Structure):
    _fields_ = [
        ("batch", ctypes.c_int32), ("out_h", ctypes.c_int32), ("out_w", ctypes.c_int32),
        ("num_classes", ctypes.c_int32), ("num_joints", ctypes.c_int32), ("K", ctypes.c_int32),
        ("rep_mode", ctypes.c_int32), ("use_moments", ctypes.c_int32), ("nms", ctypes.c_int32),
        ("visible_thresh", ctypes.c_int32), ("opencv_return", ctypes.c_int32),
        ("apply_sigmoid", ctypes.c_int32), ("use_pnp", ctypes.c_int32),
        ("vis_thresh", ctypes.c_float), ("balance", ctypes.c_float), ("modern_bool_semantics", ctypes.c_int32),
        ("test_scale", ctypes.c_float), ("num_scales", ctypes.c_int32),
    ]


class CpTrackerConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in (
        "streams", "max_tracks", "kalman", "scale_pool", "use_pnp", "hps_uncertainty", "max_age", "visible_thresh",
        "opencv_return", "render_hm_mode", "render_hmhp_mode", "device")] + [
        (n, ctypes.c_float) for n in ("new_thresh", "pre_thresh", "R", "conf_lo", "conf_hi")] + [
        ("hungarian", ctypes.c_int32)]


_lib = None


def lib_available():
    return os.path.exists(LIB_PATH)


def load():
    """Load the shared library (once).  Raises RuntimeError when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "centerpose_b200: %s not found -- run `python -m centerpose_b200.build` "
            "(there is no CPU / PyTorch fallback for the hot path)" % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
    L.cp_version.restype = ctypes.c_int
    L.cp_last_error.restype = ctypes.c_char_p
    L.cp_plan_create.argtypes = [ctypes.POINTER(CpConfig), ctypes.POINTER(vp)]
    L.cp_plan_destroy.argtypes = [vp]
    L.cp_plan_load_weights.argtypes = [vp, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(vp),
                                       ctypes.POINTER(i64), i32, vp]
    L.cp_forward.argtypes = [vp, i32, vp, vp, vp, vp, ctypes.POINTER(vp), vp]
    L.cp_plan_num_ops.argtypes = [vp]
    L.cp_plan_profile.argtypes = [vp, i32, vp, vp, vp, vp, ctypes.POINTER(vp), vp, ctypes.POINTER(CpOpStat), i32,
                                  ctypes.POINTER(i32)]
    L.cp_plan_op_desc.argtypes = [vp, i32, ctypes.POINTER(CpOpDesc)]
    L.cp_plan_arena.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(i64)]
    L.cp_plan_run_ops.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp, ctypes.POINTER(vp), vp, ctypes.POINTER(CpOpLaunch)]
    L.cp_plan_bytes.argtypes = [vp]
    L.cp_plan_bytes.restype = i64
    L.cp_plan_forward_launches.argtypes = [vp]
    L.cp_plan_forward_launches.restype = i32
    L.cp_decode_workspace_bytes.argtypes = [ctypes.POINTER(CpDecodeParams)]
    L.cp_decode_workspace_bytes.restype = ctypes.c_size_t
    L.cp_decode_pnp.argtypes = [ctypes.POINTER(CpDecodeParams), ctypes.POINTER(CpHeads), vp, vp, vp, vp, vp,
                                ctypes.c_size_t, vp]
    L.cp_infer.argtypes = [vp, i32, vp, vp, vp, vp, ctypes.POINTER(CpDecodeParams), vp,
                           ctypes.POINTER(vp), vp, vp, vp, vp]
    L.cp_dcn_v2_forward.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp]
    L.cp_dcn_v2_forward_ex.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    L.cp_dcn_v2_backward.argtypes = [vp] * 10 + [i32] * 6 + [vp]
    L.cp_conv2d.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp]
    L.cp_preprocess.argtypes = [vp, vp, i32, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_float),
                                ctypes.POINTER(ctypes.c_float), vp]
    L.cp_preprocess_affine.argtypes = [vp, vp, i32, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_double),
                                       ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), vp]
    L.cp_preprocess_resize_affine.argtypes = [vp, vp, i32, i32, i32, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_double),
                                              ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), vp]
    L.cp_preprocess_ragged.argtypes = [vp, i64, ctypes.POINTER(i64), ctypes.POINTER(i32), vp, i32, i32, i32,
                                       ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_float),
                                       ctypes.POINTER(ctypes.c_float), vp]
    L.cp_preprocess_yuv420.argtypes = [vp, i64, ctypes.POINTER(i64), ctypes.POINTER(i32), i32, vp, i32, i32, i32,
                                       ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_float),
                                       ctypes.POINTER(ctypes.c_float), vp]
    L.cp_preprocess_slots_dev.argtypes = [vp, i32, i32, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_double),
                                          ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), vp, vp, vp, vp]
    L.cp_preprocess_frame_table_bytes.argtypes = [i32]
    L.cp_preprocess_frame_table_bytes.restype = i64
    L.cp_preprocess_frame_table.argtypes = [i64, ctypes.POINTER(i64), ctypes.POINTER(i32), i32, i32, i32, i32,
                                            ctypes.POINTER(ctypes.c_double), vp, vp]
    L.cp_preprocess_slots_ragged_dev.argtypes = [vp, vp, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_float),
                                                 ctypes.POINTER(ctypes.c_float), vp, vp, vp, vp]
    L.cp_preprocess_slots_rows_dev.argtypes = [vp, vp, i32, vp, i32, i32, i32, ctypes.POINTER(ctypes.c_float),
                                               ctypes.POINTER(ctypes.c_float), vp, vp, vp, vp, vp]
    L.cp_gather_rows_dev.argtypes = [vp, vp, i64, i32, vp, vp]
    L.cp_preprocess_formats.argtypes = [vp, i64, ctypes.POINTER(i64), ctypes.POINTER(i32), ctypes.POINTER(i32), vp, i32,
                                        i32, i32, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_float),
                                        ctypes.POINTER(ctypes.c_float), vp]
    L.cp_preprocess_frame_table_formats.argtypes = [i64, ctypes.POINTER(i64), ctypes.POINTER(i32), ctypes.POINTER(i32),
                                                    i32, i32, i32, ctypes.POINTER(ctypes.c_double), vp, vp]
    L.cp_preprocess_remap.argtypes = [vp, i64, ctypes.POINTER(i64), ctypes.POINTER(i32), ctypes.POINTER(i32),
                                      ctypes.POINTER(vp), vp, i32, i32, i32, ctypes.POINTER(ctypes.c_double),
                                      ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), vp]
    L.cp_preprocess_frame_table_maps.argtypes = [i64, ctypes.POINTER(i64), ctypes.POINTER(i32), i32, ctypes.POINTER(i32),
                                                 ctypes.POINTER(vp), i32, i32, i32, ctypes.POINTER(ctypes.c_double), vp, vp]
    L.cp_tracker_create.argtypes = [ctypes.POINTER(CpTrackerConfig), ctypes.POINTER(vp)]
    L.cp_tracker_destroy.argtypes = [vp]
    L.cp_tracker_reset.argtypes = [vp, i32, vp]
    L.cp_tracker_step.argtypes = [vp, i32, vp, vp, i32, vp, vp, vp, vp]
    L.cp_tracker_render.argtypes = [vp, i32, vp, vp, i32, i32, vp, vp, vp]
    L.cp_tracker_render_ex.argtypes = [vp, i32, vp, vp, i32, i32, ctypes.POINTER(i32), vp, vp, vp]
    L.cp_tracker_seed.argtypes = [vp, i32, vp, vp, i32, vp]
    L.cp_tracker_step_ex.argtypes = [vp, i32, ctypes.POINTER(i32), vp, vp, i32, vp, vp, vp, vp]
    L.cp_tracker_render_ex2.argtypes = [vp, i32, ctypes.POINTER(i32), vp, vp, i32, i32, ctypes.POINTER(i32), vp, vp, vp]
    L.cp_tracker_seed_ex.argtypes = [vp, i32, ctypes.POINTER(i32), vp, vp, i32, vp]
    L.cp_tracker_reset_dev.argtypes = [vp, i32, vp, vp]
    L.cp_tracker_render_dev.argtypes = [vp, i32, vp, vp, i32, i32, vp, vp, vp, vp]
    L.cp_tracker_render_dev2.argtypes = [vp, i32, vp, vp, vp, i32, i32, vp, vp, vp, vp]
    L.cp_tracker_step_dev.argtypes = [vp, i32, vp, vp, vp, i32, vp, vp, vp, vp]
    L.cp_plan_create_multi.argtypes = [ctypes.POINTER(CpConfig), i32, ctypes.POINTER(vp)]
    L.cp_plan_load_weights_model.argtypes = [vp, i32, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(vp),
                                             ctypes.POINTER(i64), i32, vp]
    L.cp_plan_num_models.argtypes = [vp]
    L.cp_plan_op_desc_model.argtypes = [vp, i32, i32, ctypes.POINTER(CpOpDesc)]
    L.cp_infer_multi.argtypes = [vp, i32, vp, ctypes.POINTER(CpDecodeParams), vp, ctypes.POINTER(vp), vp, vp, vp, vp]
    L.cp_plan_create_multi_track.argtypes = [ctypes.POINTER(CpConfig), i32, ctypes.POINTER(vp)]
    L.cp_infer_multi_track.argtypes = [vp, i32, vp, vp, vp, vp, ctypes.POINTER(CpDecodeParams), vp, ctypes.POINTER(vp), vp,
                                       vp, vp, vp]
    L.cp_tracker_create_multi.argtypes = [ctypes.POINTER(CpTrackerConfig), i32, ctypes.POINTER(vp)]
    L.cp_plan_create_ex.argtypes = [ctypes.POINTER(CpConfig), i32, ctypes.c_uint32, ctypes.POINTER(vp)]
    L.cp_plan_memory.argtypes = [ctypes.POINTER(CpConfig), i32, ctypes.c_uint32, ctypes.POINTER(CpMemoryInfo)]
    L.cp_plan_allocations.argtypes = [ctypes.POINTER(CpConfig), i32, ctypes.c_uint32, ctypes.POINTER(CpActAlloc), i32,
                                      ctypes.POINTER(i32)]
    L.cp_plan_op_ksegments.argtypes = [vp, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), ctypes.POINTER(i32)]
    L.cp_plan_ksegments.argtypes = [ctypes.POINTER(CpConfig), i32, ctypes.c_uint32, ctypes.POINTER(i32), i32,
                                    ctypes.POINTER(i32)]
    L.cp_jpeg_parse.argtypes = [vp, i64, ctypes.POINTER(CpJpegHeader)]
    L.cp_jpeg_workspace_bytes.argtypes = [ctypes.POINTER(CpJpegHeader), i32]
    L.cp_jpeg_workspace_bytes.restype = ctypes.c_size_t
    L.cp_jpeg_decode.argtypes = [ctypes.POINTER(CpJpegHeader), i32, vp, vp, vp, vp, vp, ctypes.c_size_t, vp, i32, vp]
    L.cp_jpeg_last_rounds.argtypes = []
    L.cp_jpeg_slots_workspace_bytes.argtypes = [i32, ctypes.POINTER(i32), ctypes.POINTER(i64), i32]
    L.cp_jpeg_slots_workspace_bytes.restype = ctypes.c_size_t
    L.cp_jpeg_slots_block_bytes.argtypes = [i32]
    L.cp_jpeg_slots_block_bytes.restype = ctypes.c_size_t
    L.cp_jpeg_slots_prepare.argtypes = [i32, ctypes.POINTER(i32), ctypes.POINTER(i64), i32, ctypes.POINTER(CpJpegHeader),
                                        ctypes.POINTER(i64), ctypes.POINTER(i64), vp]
    L.cp_jpeg_decode_slots_dev.argtypes = [vp, i32, ctypes.POINTER(i32), ctypes.POINTER(i64), i32, vp, vp, vp,
                                           ctypes.c_size_t, vp, vp]
    L.cp_jpeg_mask_counts_dev.argtypes = [vp, vp, i32, i32, vp, vp]
    for name in EXPORTS:
        fn = getattr(L, name)
        if name not in ("cp_version", "cp_last_error", "cp_plan_bytes", "cp_plan_forward_launches",
                        "cp_decode_workspace_bytes", "cp_preprocess_frame_table_bytes", "cp_jpeg_workspace_bytes",
                        "cp_jpeg_slots_workspace_bytes", "cp_jpeg_slots_block_bytes"):
            fn.restype = ctypes.c_int
    _lib = L
    return L


def check(rc, what=""):
    if rc != 0:
        msg = load().cp_last_error()
        raise RuntimeError("centerpose_b200 %s failed (%d): %s" % (what, rc, msg.decode() if msg else "?"))
