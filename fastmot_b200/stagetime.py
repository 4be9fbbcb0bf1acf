"""Per-stage GPU timing of the hot path for bench.py's `roofline_stages`.

`enable()` wraps every C-ABI entry point of the loaded library with a pair of CUDA events recorded on the current
stream (the callers launch on torch's current stream), keyed by the stage the entry point belongs to; `collect()`
synchronises and returns {stage: (total_ms, calls)}.  Off by default: the wrappers add two event records per call, so
the benchmark runs its timed passes without them and a separate pass with them.  The conv stacks are CUDA-graph
replays and are timed by fastmot_b200.engine's own profiler.
"""
import torch

from . import _lib

STAGE_OF = {
    "fm_letterbox_preproc": "preproc",
    "fm_yolo_decode_filter": "decode+nms", "fm_diou_nms_filter": "decode+nms",
    "fm_roi_resize_norm": "crops",
    "fm_gray_half": "klt-image", "fm_pyr_level": "klt-image", "fm_scharr": "klt-image", "fm_bg_small": "klt-image",
    "fm_gray_resize": "klt-image",
    "fm_flow_keypoints": "keypoints", "fm_fast_detect": "keypoints", "fm_gather_points": "keypoints",
    "fm_flow_keypoints_cfg": "keypoints",
    "fm_lk_track": "lk",
    "fm_ransac_homography": "ransac", "fm_ransac_affine_partial_batch": "ransac",
    "fm_kalman_step_batched": "kalman", "fm_kalman_create_batched": "kalman",
    "fm_matching_cost": "cost", "fm_iou_cost": "cost", "fm_find_occluded": "cost", "fm_motion_distance": "cost",
    "fm_assoc_cascade": "cost+lsa",
    "fm_lsa": "lsa", "fm_greedy_match": "lsa",
    "fm_feature_update": "feature-update",
}

_records = {}
_saved = {}


def enable():
    lib = _lib.load()
    if _saved:
        return
    for name, stage in STAGE_OF.items():
        fn = getattr(lib, name, None)
        if fn is None:
            continue
        _saved[name] = fn

        def wrapper(*args, _fn=fn, _stage=stage):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = _fn(*args)
            e1.record()
            _records.setdefault(_stage, []).append((e0, e1))
            return rc
        setattr(lib, name, wrapper)


def active():
    """True while the per-entry-point wrappers are installed (Flow then keeps its call-by-call sequence)."""
    return bool(_saved)


def disable():
    lib = _lib.load()
    for name, fn in _saved.items():
        setattr(lib, name, fn)
    _saved.clear()


def collect():
    torch.cuda.synchronize()
    out = {}
    for stage, evs in _records.items():
        out[stage] = (sum(e0.elapsed_time(e1) for e0, e1 in evs), len(evs))
    _records.clear()
    return out
