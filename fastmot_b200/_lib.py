"""ctypes binding of libfastmot_b200.so (include/fastmot_b200.h).

There is no CPU fallback: if the shared library is missing or the device is not an H100 the product
classes raise.  Loading the library (dlopen + symbol lookup) needs no GPU; running any op does.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfastmot_b200.so")

c_p = C.c_void_p
c_i = C.c_int
c_d = C.c_double
c_f = C.c_float
c_ll = C.c_longlong


class FmKalmanParams(C.Structure):
    _fields_ = [("trans_mat", c_d * 64), ("acc_cov", c_d * 64),
                ("std_factor_acc", c_d), ("std_offset_acc", c_d),
                ("std_factor_det", c_d * 2), ("std_factor_klt", c_d * 2),
                ("min_std_det", c_d * 2), ("min_std_klt", c_d * 2),
                ("init_pos_weight", c_d), ("init_vel_weight", c_d)]


class FmPyramid(C.Structure):
    _fields_ = [("n_levels", c_i), ("w", c_i * 8), ("h", c_i * 8), ("img", c_p * 8), ("deriv", c_p * 8)]


class FmTrackJob(C.Structure):
    _fields_ = [("slot", c_i), ("x0", c_i), ("y0", c_i), ("cw", c_i), ("ch", c_i), ("area", c_i), ("n_keep", c_i),
                ("redetect", c_i), ("min_dist", c_i), ("scratch_off", c_i), ("eig_max", c_f), ("pad", c_i)]


class FmFlowPlan(C.Structure):
    """include/fastmot_b200.h: FmFlowPlan (field order and types must match)."""
    _fields_ = [("frame_w", c_i), ("frame_h", c_i), ("gray", c_p * 2), ("pyr", FmPyramid * 2),
                ("tlbr_pool", c_p), ("slots", c_p), ("owner", c_p), ("kp_pool", c_p), ("kp_prev_pool", c_p),
                ("kp_count", c_p), ("max_kp", c_i),
                ("feat_density", c_d), ("feat_dist_factor", c_d), ("quality", c_d), ("max_corners", c_i),
                ("jobs", c_p), ("scratch", c_p), ("scratch_cap", c_i), ("flags", c_p),
                ("bg", c_p), ("bg_mask", c_p), ("bg_score", c_p), ("bg_w", c_i), ("bg_h", c_i), ("bg_thresh", c_i),
                ("unscale_x", c_f), ("unscale_y", c_f), ("bg_pts", c_p), ("bg_count", c_p), ("max_bg", c_i),
                ("all_prev", c_p), ("all_cur", c_p), ("status", c_p), ("err", c_p), ("trk_begin", c_p), ("meta", c_p),
                ("max_points", c_i), ("pt_scale_x", c_f), ("pt_scale_y", c_f), ("win_w", c_i), ("win_h", c_i),
                ("lk_max_count", c_i), ("lk_epsilon", c_f), ("lk_min_eig", c_f), ("max_error", c_f),
                ("ransac_max_iter", c_i), ("ransac_conf", c_d), ("ransac_thresh", c_d), ("inlier_thresh", c_i),
                ("refine_iters", c_i), ("good_idx", c_p), ("inl_idx", c_p), ("bg_kp", c_p), ("bg_kp_prev", c_p),
                ("bg_kp_count", c_p), ("est_boxes", c_p), ("sig", c_p), ("klt_tlbr", c_p), ("klt_ok", c_p),
                ("klt_ok_bytes", c_ll), ("inlier_ratio", c_p), ("rounds_ahead", c_i),
                ("block_size", c_i), ("gradient_size", c_i), ("use_harris", c_i), ("harris_k", c_d)]


class FmConvDesc(C.Structure):
    _fields_ = [(k, c_i) for k in ("n", "hi", "wi", "cin", "cin_stride", "cin_offset", "ho", "wo", "cout",
                                   "cout_stride", "cout_offset", "kh", "kw", "stride", "pad", "act", "res_stride",
                                   "res_offset")] + [("ws", c_p), ("ws_bytes", c_ll)]


class FmOsbStreams(C.Structure):
    _fields_ = [("x", c_p), ("n", c_i), ("h", c_i), ("w", c_i), ("cin", c_i), ("mid", c_i), ("w1", c_p), ("b1", c_p),
                ("pw", c_p), ("dw", c_p), ("tails", c_p * 4), ("gap_part", c_p)]


class FmOsbMerge(C.Structure):
    _fields_ = [("n", c_i), ("hw", c_i), ("cin", c_i), ("cout", c_i), ("mid", c_i), ("cr", c_i), ("strips", c_i),
                ("tails", c_p * 4), ("gap_part", c_p), ("gw1", c_p), ("gb1", c_p), ("gw2", c_p), ("gb2", c_p),
                ("wimg", c_p), ("bias", c_p), ("x", c_p), ("res", c_p), ("out", c_p), ("gate_scratch", c_p)]


class FmCascadeDesc(C.Structure):
    _fields_ = [(k, c_i) for k in ("n_det", "n_conf", "n_groups", "n_unconf", "n_hist", "cap")] + \
               [(k, c_p) for k in ("goff", "conf_active", "feat_cost", "iou_cost", "reid_cost", "det_conf",
                                   "det_occluded", "sub", "out")] + [("conf_thresh", c_d), ("max_reid_cost", c_d)]


class FmYoloHead(C.Structure):
    _fields_ = [("anchors", c_f * 12), ("scale_x_y", c_f)]


class FmFrame(C.Structure):
    _fields_ = [("y", c_p), ("uv", c_p), ("w", c_i), ("h", c_i), ("pitch", c_i), ("uv_pitch", c_i), ("format", c_i),
                ("v", c_p)]


class FmFrameGeom(C.Structure):
    _fields_ = [("frame", FmFrame), ("roi_x", c_i), ("roi_y", c_i), ("roi_w", c_i), ("roi_h", c_i),
                ("size_w", c_f), ("size_h", c_f), ("off_x", c_f), ("off_y", c_f)]


FM_PIX_BGR, FM_PIX_NV12, FM_PIX_I420, FM_PIX_YUY2, FM_PIX_BGRX = 0, 1, 2, 3, 4


# name -> (restype, argtypes); kept in one table so tests can check it against the header
SIGNATURES = {
    "fm_last_error": (C.c_char_p, []),
    "fm_version": (c_i, []),
    "fm_device_ok": (c_i, []),
    "fm_memcpy_async": (c_i, [c_p, c_p, c_ll, c_p]),
    "fm_host_is_pinned": (c_i, [c_p]),
    "fm_launch_count": (c_ll, []),
    "fm_kalman_step_batched": (c_i, [c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_p, c_p, c_p,
                                      C.POINTER(FmKalmanParams), c_d, c_d, c_p, c_p, c_p]),
    "fm_kalman_create_batched": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_i, C.POINTER(FmKalmanParams), c_p]),
    "fm_motion_distance": (c_i, [c_p, c_p, c_p, c_i, c_p, c_i, C.POINTER(FmKalmanParams), c_p, c_p]),
    "fm_matching_cost": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i,
                               c_d, c_d, c_d, C.POINTER(FmKalmanParams), c_p, c_p]),
    "fm_feature_update": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p]),
    "fm_iou_cost": (c_i, [c_p, c_p, c_p, c_i, c_p, c_p, c_p, c_i, c_d, c_p, c_p]),
    "fm_find_occluded": (c_i, [c_p, c_i, c_d, c_p, c_p]),
    "fm_lsa_workspace_bytes": (c_ll, [c_i, c_i]),
    "fm_lsa": (c_i, [c_p, c_i, c_i, c_p, c_p, c_p, c_p]),
    "fm_greedy_match": (c_i, [c_p, c_i, c_i, c_d, c_p, c_p, c_p]),
    "fm_assoc_cascade": (c_i, [C.POINTER(FmCascadeDesc), c_p]),
    "fm_assoc_cascade_out_ints": (c_ll, [c_i]),
    "fm_letterbox_preproc": (c_i, [C.POINTER(FmFrame), c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_p, c_p]),
    "fm_roi_resize_norm": (c_i, [C.POINTER(FmFrame), c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_p]),
    "fm_letterbox_preproc_geom": (c_i, [c_p, c_i, c_i, c_i, c_p, c_p]),
    "fm_roi_resize_norm_geom": (c_i, [c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_p, c_p]),
    "fm_frame_resize": (c_i, [C.POINTER(FmFrame), c_p, c_i, c_i, c_p]),
    "fm_yolo_decode_filter_geom": (c_i, [c_p, c_i, c_ll, c_i, c_i, c_i, c_i, c_i, C.POINTER(FmYoloHead), c_i, c_i,
                                          c_i, c_i, c_i, c_i, c_p, c_d, c_p, c_p, c_p, c_p, c_i, c_p]),
    "fm_diou_nms_filter_batch": (c_i, [c_i, c_p, c_p, c_i, c_p, c_i, c_d, c_d, c_d, c_p, c_i, c_p, c_p, c_p, c_p, c_p,
                                        c_p]),
    "fm_yolo_decode_filter": (c_i, [c_p, c_i, c_i, c_i, c_i, c_i, C.POINTER(FmYoloHead), c_i, c_i, c_i, c_i, c_i, c_p,
                                     c_d, c_f, c_f, c_f, c_f, c_p, c_p, c_p, c_i, c_p]),
    "fm_gray_half": (c_i, [C.POINTER(FmFrame), c_p, c_p, c_p]),
    "fm_gray_resize": (c_i, [C.POINTER(FmFrame), c_p, c_p, c_i, c_i, c_p]),
    "fm_pyr_level": (c_i, [c_p, c_i, c_i, c_p, c_p]),
    "fm_scharr": (c_i, [c_p, c_i, c_i, c_p, c_p]),
    "fm_bg_small": (c_i, [c_p, c_p, c_i, c_i, c_p, c_p, c_i, c_i, c_p]),
    "fm_flow_keypoints": (c_i, [c_p, c_i, c_i, c_p, c_p, c_i, c_p, c_p, c_p, c_i, c_d, c_d, c_d, c_i, c_p, c_p, c_i,
                                 c_p, c_p, c_p]),
    "fm_flow_keypoints_cfg": (c_i, [c_p, c_i, c_i, c_p, c_p, c_i, c_p, c_p, c_p, c_i, c_d, c_d, c_d, c_i, c_i, c_i, c_i,
                                     c_d, c_p, c_p, c_i, c_p, c_p, c_p]),
    "fm_fast_detect": (c_i, [c_p, c_p, c_i, c_i, c_i, c_f, c_f, c_p, c_p, c_p, c_i, c_p]),
    "fm_gather_points": (c_i, [c_p, c_p, c_i, c_p, c_i, c_p, c_p, c_p, c_p, c_p, c_i, c_p]),
    "fm_lk_track": (c_i, [c_p, c_p, c_p, c_p, c_f, c_f, c_i, c_i, c_i, c_f, c_f, c_f, c_p, c_p, c_p, c_p]),
    "fm_ransac_homography": (c_i, [c_p, c_p, c_p, c_p, c_i, c_d, c_d, c_i, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_i,
                                    c_p]),
    "fm_ransac_affine_partial_batch": (c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_p, c_p, c_p,
                                              c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_d, c_d, c_i, c_i, c_i, c_p]),
    "fm_flow_plan_create": (c_p, [C.POINTER(FmFlowPlan)]),
    "fm_flow_plan_destroy": (None, [c_p]),
    "fm_flow_predict": (c_i, [c_p, C.POINTER(FmFrame), c_i, c_i, c_p, c_p, c_p, c_p]),
    "fm_conv2d_simt": (c_i, [C.POINTER(FmConvDesc), c_p, c_p, c_p, c_p, c_p, c_p]),
    "fm_maxpool": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_p]),
    "fm_maxpool_pad": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_p]),
    "fm_avgpool2": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_p]),
    "fm_upsample_copy": (c_i, [c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_p]),
    "fm_add_act": (c_i, [c_p, c_p, c_p, c_ll, c_i, c_p]),
    "fm_add_act_strided": (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_p, c_i, c_i, c_ll, c_i, c_i, c_p]),
    "fm_conv2d_tc": (c_i, [C.POINTER(FmConvDesc), c_p, c_p, c_p, c_p, c_p, c_p]),
    "fm_conv2d_tc_supported": (c_i, [C.POINTER(FmConvDesc)]),
    "fm_conv2d_tma": (c_i, [C.POINTER(FmConvDesc), c_p, c_p, c_p, c_p, c_p, c_p]),
    "fm_conv2d_tma_supported": (c_i, [C.POINTER(FmConvDesc)]),
    "fm_dwconv3": (c_i, [c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p]),
    "fm_global_avgpool": (c_i, [c_p, c_p, c_i, c_i, c_i, c_p]),
    "fm_channel_gate": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p]),
    "fm_fc_norm": (c_i, [c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_p]),
    "fm_channel_gate4": (c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_p]),
    "fm_probe_umma": (c_i, [c_p, c_i, c_i, c_p, c_p, c_i, c_i, c_p, c_p, c_p]),
    "fm_osb_streams": (c_i, [C.POINTER(FmOsbStreams), c_p]),
    "fm_osb_streams_strips": (c_i, [c_i, c_i, c_i]),
    "fm_osb_merge": (c_i, [C.POINTER(FmOsbMerge), c_p]),
    "fm_osb_merge_ncta": (c_i, [c_i, c_i]),
    "fm_osnet_stem": (c_i, [c_p, c_i, c_p, c_p, c_p, c_p]),
    "fm_channel_gate4_pooled": (c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i,
                                      c_p]),
    "fm_nms_mask_bytes": (c_ll, [c_i]),
    "fm_diou_nms_filter": (c_i, [c_p, c_p, c_p, c_i, c_d, c_d, c_d, c_p, c_i, c_p, c_p, c_p, c_p, c_p, c_p]),
}


class FastMOTLibError(RuntimeError):
    pass


_lib = None


def load():
    """dlopen the library and bind every symbol of the header. Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FastMOTLibError(
            f"{LIB_PATH} not found: build it with `python -m fastmot_b200.build` "
            "(there is no CPU fallback for the fastmot_b200 hot path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise FastMOTLibError(f"symbol {name} missing from {LIB_PATH}") from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().fm_last_error().decode(errors="replace")
        raise FastMOTLibError(f"{what} failed (code {rc}): {msg}")


def require_device():
    """Raise unless an H100-class (sm_90) device is usable (called by every product class constructor)."""
    lib = load()
    if not lib.fm_device_ok():
        raise FastMOTLibError("fastmot_b200 needs an sm_90 (H100) CUDA device: "
                              + lib.fm_last_error().decode(errors="replace"))
    return lib


_graph_kernels = 0


def count_graph_kernels(n):
    """Kernels executed through CUDA-graph replays never pass the C-ABI launch sites; account for them here."""
    global _graph_kernels
    _graph_kernels += n


def launch_count():
    """Number of fastmot_b200 kernels launched so far in this process (bench.py `gpu_launches`)."""
    return int(load().fm_launch_count()) + _graph_kernels
