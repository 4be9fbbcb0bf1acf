"""KLT optical-flow stage on the GPU with the reference's constructor / attributes (fastmot/flow.py:16-264).

`predict_device` enqueues the whole of `Flow.predict` — gray + optical-flow image (any frame size and scale) and its
pyramid with Scharr derivatives, occlusion ("owner") map, per-track keypoint filtering and Shi-Tomasi / Harris
re-detection (every cv2.goodFeaturesToTrack setting), FAST background corners, pyramidal LK on
all points at once, RANSAC homography, per-track RANSAC partial-affine with box prediction — as ~15 kernel
launches with no OpenCV and no host round trip except one 16-byte status read.  Results stay on the device:
predicted boxes / flags / inlier ratios in the track pool, the homography in a 9-double buffer that the batched
Kalman kernel reads directly.
"""
import ctypes as C
import logging

import numpy as np
import torch

from . import _lib
from .devmem import ptr, stream_ptr, device_frame, UploadSlot, FrameUploader

LOGGER = logging.getLogger(__name__)

# candidate corners the selection kernel sorts in shared memory (csrc/klt_feat.cu GFTT_MAX_CAND); a box with more
# selects them in global memory from scratch_floats.  Also the keypoint rows a track has when maxCorners is <= 0 or
# above 4096: more kept corners raise at run time
GFTT_MAX_CAND = 4096
# keyword arguments of cv2.goodFeaturesToTrack that obj_feat_params may set (minDistance and mask come from the track)
_GFTT_KEYS = {"maxCorners", "qualityLevel", "blockSize", "useHarrisDetector", "k", "gradientSize"}


def fast_corner_bound(w, h):
    """Most corners FAST with non-max suppression can keep in a w x h image: the interior is (w-6) x (h-6) and no two
    kept corners are 8-neighbours."""
    return -(-max(w - 6, 0) // 2) * -(-max(h - 6, 0) // 2)


def _depth_key(track):
    """Sort key equivalent to Track.__lt__ (fastmot/track.py:160-162): bottom edge, then younger first."""
    return (float(track.bboxes[-1][3]), -track.age)


class Flow:
    def __init__(self, size,
                 bg_feat_scale_factor=(0.1, 0.1),
                 opt_flow_scale_factor=(0.5, 0.5),
                 feat_density=0.005,
                 feat_dist_factor=0.06,
                 ransac_max_iter=500,
                 ransac_conf=0.99,
                 max_error=100,
                 inlier_thresh=4,
                 bg_feat_thresh=10,
                 obj_feat_params=None,
                 opt_flow_params=None,
                 max_points=1 << 18,
                 max_bg_points=1 << 16,
                 max_tracks=2048,
                 scratch_floats=1 << 24):
        self.size = size
        assert 0 < bg_feat_scale_factor[0] <= 1 and 0 < bg_feat_scale_factor[1] <= 1
        self.bg_feat_scale_factor = bg_feat_scale_factor
        assert 0 < opt_flow_scale_factor[0] <= 1 and 0 < opt_flow_scale_factor[1] <= 1
        self.opt_flow_scale_factor = opt_flow_scale_factor
        assert 0 <= feat_density <= 1
        self.feat_density = feat_density
        assert feat_dist_factor >= 0
        self.feat_dist_factor = feat_dist_factor
        assert ransac_max_iter >= 0
        self.ransac_max_iter = ransac_max_iter
        assert 0 <= ransac_conf <= 1
        self.ransac_conf = ransac_conf
        assert 0 <= max_error <= 255
        self.max_error = max_error
        assert inlier_thresh >= 1
        self.inlier_thresh = inlier_thresh
        assert bg_feat_thresh >= 0
        if bg_feat_thresh > 255:
            # cv2's FAST tests most columns with the threshold cut to 8 bits and the last few with it clamped to 255,
            # so above 255 its corners depend on where they lie in the image: no result to be exact against
            raise ValueError(f"bg_feat_thresh must be at most 255 (the largest pixel contrast), got {bg_feat_thresh}")
        self.bg_feat_thresh = bg_feat_thresh

        self.obj_feat_params = {"maxCorners": 1000, "qualityLevel": 0.06, "blockSize": 3}
        # the reference ignores the configured opt_flow_params (inverted `is None`, flow.py:92-93) and always
        # runs with these values; accept the argument, keep the reference's effective behaviour
        self.opt_flow_params = {"winSize": (5, 5), "maxLevel": 5, "criteria": (3, 10, 0.03)}
        if obj_feat_params is not None:
            self.obj_feat_params.update(vars(obj_feat_params))
        unknown = set(self.obj_feat_params) - _GFTT_KEYS
        if unknown:
            raise TypeError(f"obj_feat_params: cv2.goodFeaturesToTrack takes no argument {sorted(unknown)}")
        mk = self.obj_feat_params
        self.block_size = int(mk["blockSize"])
        self.gradient_size = int(mk.get("gradientSize", 3))
        self.use_harris = bool(mk.get("useHarrisDetector", False))
        self.harris_k = float(mk.get("k", 0.04))
        if self.block_size < 1:
            raise ValueError(f"obj_feat_params.blockSize must be >= 1, got {mk['blockSize']}")
        if self.gradient_size not in (1, 3, 5, 7):
            raise ValueError(f"obj_feat_params.gradientSize must be 1, 3, 5 or 7, got {mk.get('gradientSize')}")
        # the default goodFeaturesToTrack setting runs the original kernels (csrc/klt_feat.cu)
        self._default_feat = (self.block_size == 3 and self.gradient_size == 3 and not self.use_harris
                              and 0 < int(mk["maxCorners"]) <= 1024)
        # keypoint rows per track (TrackPool.max_kp): 1024 up to maxCorners 1024, else maxCorners bounded by the
        # candidate cap (maxCorners <= 0 is no limit)
        mc = int(mk["maxCorners"])
        self.max_kp = 1024 if 0 < mc <= 1024 else min(mc if mc > 0 else GFTT_MAX_CAND, GFTT_MAX_CAND)

        W, H = size
        # Python's round (half to even), as the reference sizes its buffers (flow.py:102-105)
        self.opt_flow_sz = (round(opt_flow_scale_factor[0] * W), round(opt_flow_scale_factor[1] * H))
        self.bg_feat_sz = (round(bg_feat_scale_factor[0] * W), round(bg_feat_scale_factor[1] * H))
        if min(self.opt_flow_sz) < 1:
            raise ValueError(f"opt_flow_scale_factor {tuple(opt_flow_scale_factor)} gives an empty optical-flow image "
                             f"{self.opt_flow_sz} for frame size {tuple(size)}")
        if min(self.bg_feat_sz) < 1:
            raise ValueError(f"bg_feat_scale_factor {tuple(bg_feat_scale_factor)} gives an empty background image "
                             f"{self.bg_feat_sz} for frame size {tuple(size)}")
        # exactly half the frame both ways: cv2.resize's 2x2 mean (fm_gray_half); otherwise INTER_LINEAR (fm_gray_resize)
        self._half = 2 * self.opt_flow_sz[0] == W and 2 * self.opt_flow_sz[1] == H

        self._lib = _lib.require_device()
        dev = torch.device("cuda")
        u8, i32, f32 = torch.uint8, torch.int32, torch.float32
        win_w, win_h = self.opt_flow_params["winSize"]
        # pyramid geometry of cv::buildOpticalFlowPyramid
        sizes = [self.opt_flow_sz]
        for _ in range(self.opt_flow_params["maxLevel"]):
            w, h = (sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2
            if w <= win_w or h <= win_h:
                break
            sizes.append((w, h))
        self.level_sizes = sizes
        self.gray = [torch.zeros(H, W, dtype=u8, device=dev) for _ in range(2)]
        self.pyr = [[torch.zeros(h, w, dtype=u8, device=dev) for (w, h) in sizes] for _ in range(2)]
        self.deriv = [[torch.zeros(h, w, 2, dtype=torch.int16, device=dev) for (w, h) in sizes] for _ in range(2)]
        self.pyr_desc = []
        for k in range(2):
            d = _lib.FmPyramid()
            d.n_levels = len(sizes)
            for i, (w, h) in enumerate(sizes):
                d.w[i], d.h[i] = w, h
                d.img[i] = self.pyr[k][i].data_ptr()
                d.deriv[i] = self.deriv[k][i].data_ptr()
            self.pyr_desc.append(d)
        self.prev = 0
        self.owner = torch.zeros(H, W, dtype=i32, device=dev)
        bw, bh = self.bg_feat_sz
        self.bg = torch.zeros(bh, bw, dtype=u8, device=dev)
        self.bg_mask = torch.zeros(bh, bw, dtype=u8, device=dev)
        self.bg_score = torch.zeros(bh, bw, dtype=u8, device=dev)
        # FAST's non-max suppression keeps no two touching corners, so the background buffers are sized to hold every
        # corner the image can have and the point list is never cut short
        max_bg_points = max(max_bg_points, fast_corner_bound(bw, bh))
        self.max_points, self.max_bg, self.max_tracks = max_points, max_bg_points, max_tracks
        self.bg_pts = torch.zeros(max_bg_points, 2, dtype=f32, device=dev)
        self.bg_count = torch.zeros(1, dtype=i32, device=dev)
        self.all_prev = torch.zeros(max_points, 2, dtype=f32, device=dev)
        self.all_cur = torch.zeros(max_points, 2, dtype=f32, device=dev)
        self.status = torch.zeros(max_points, dtype=u8, device=dev)
        self.err = torch.zeros(max_points, dtype=f32, device=dev)
        self.trk_begin = torch.zeros(max_tracks + 1, dtype=i32, device=dev)
        self.slots_dev = torch.zeros(max_tracks, dtype=i32, device=dev)
        self.jobs = torch.zeros(max_tracks * C.sizeof(_lib.FmTrackJob), dtype=u8, device=dev)
        self.scratch = torch.zeros(scratch_floats, dtype=f32, device=dev)
        self.scratch_cap = scratch_floats
        # [0] scratch counter, [1] kp status, [8:24] round flags, [24:28] gather meta (read back with the flags)
        self.flags = torch.zeros(32, dtype=i32, device=dev)
        self.meta = self.flags[24:28]
        self.good_idx = torch.zeros(max_bg_points, dtype=i32, device=dev)
        self.inl_idx = torch.zeros(max_bg_points, dtype=i32, device=dev)
        self.bg_kp = torch.zeros(max_bg_points, 2, dtype=f32, device=dev)
        self.bg_kp_prev = torch.zeros(max_bg_points, 2, dtype=f32, device=dev)
        self.bg_kp_count = torch.zeros(1, dtype=i32, device=dev)
        self.est_boxes = torch.zeros(2 * max_tracks * 5, dtype=i32, device=dev)
        self.sig = torch.zeros(max_tracks, dtype=torch.int64, device=dev)
        self._h_flags = torch.zeros(32, dtype=i32).pin_memory()
        # True (set by MultiTracker): predict_device returns without any host sync; the caller checks the round flags
        # together with its own read-back (check_flags / finish_rounds)
        self.defer_sync = False
        self.rounds_last = 0
        self._affine_args = (0, size[0], size[1])
        self._h_slots = torch.zeros(max_tracks, dtype=i32).pin_memory()
        self._upload = UploadSlot(FrameUploader(size))
        self._side = torch.cuda.Stream()
        self._ev_lk = torch.cuda.Event()
        self._ev_h = torch.cuda.Event()
        self.pool = None
        self._runner = None
        self._order = []
        self._bg_cache = None
        self.rounds_last = 0

    def bind_pool(self, pool):
        if pool.max_kp < self.max_kp:
            raise ValueError(f"TrackPool.max_kp {pool.max_kp} < {self.max_kp} keypoints per track that maxCorners "
                             f"{self.obj_feat_params['maxCorners']} allows")
        if getattr(self, "_runner", None) is not None:
            self._lib.fm_flow_plan_destroy(self._runner)
        self.pool = pool
        self._runner = None

    # ------------------------------------------------------------------ one-call runner (csrc/flow_runner.cu)
    def _plan(self):
        """Freezes every fixed buffer address and parameter of predict_device into an FmFlowPlan; the per-frame
        enqueue is then a single C-ABI call (fm_flow_predict).  An active stagetime pass (which times the individual
        entry points) keeps the call-by-call sequence below."""
        pool = self.pool
        P = _lib.FmFlowPlan()
        W, H = self.size
        P.frame_w, P.frame_h = W, H
        for k in range(2):
            P.gray[k] = self.gray[k].data_ptr()
            C.memmove(C.byref(P.pyr[k]), C.byref(self.pyr_desc[k]), C.sizeof(_lib.FmPyramid))
        P.tlbr_pool, P.slots, P.owner = pool.tlbr.data_ptr(), self.slots_dev.data_ptr(), self.owner.data_ptr()
        P.kp_pool, P.kp_prev_pool, P.kp_count, P.max_kp = (pool.kp.data_ptr(), pool.kp_prev.data_ptr(),
                                                          pool.kp_count.data_ptr(), pool.max_kp)
        mk = self.obj_feat_params
        P.feat_density, P.feat_dist_factor = float(self.feat_density), float(self.feat_dist_factor)
        P.quality, P.max_corners = float(mk["qualityLevel"]), int(mk["maxCorners"])
        P.jobs, P.scratch, P.scratch_cap, P.flags = (self.jobs.data_ptr(), self.scratch.data_ptr(), self.scratch_cap,
                                                     self.flags.data_ptr())
        bw, bh = self.bg_feat_sz
        P.bg, P.bg_mask, P.bg_score = self.bg.data_ptr(), self.bg_mask.data_ptr(), self.bg_score.data_ptr()
        P.bg_w, P.bg_h, P.bg_thresh = bw, bh, int(self.bg_feat_thresh)
        P.unscale_x = float(np.float32(1) / np.float32(self.bg_feat_scale_factor[0]))
        P.unscale_y = float(np.float32(1) / np.float32(self.bg_feat_scale_factor[1]))
        P.bg_pts, P.bg_count, P.max_bg = self.bg_pts.data_ptr(), self.bg_count.data_ptr(), self.max_bg
        P.all_prev, P.all_cur, P.status, P.err = (self.all_prev.data_ptr(), self.all_cur.data_ptr(),
                                                  self.status.data_ptr(), self.err.data_ptr())
        P.trk_begin, P.meta, P.max_points = self.trk_begin.data_ptr(), self.meta.data_ptr(), self.max_points
        win, crit = self.opt_flow_params["winSize"], self.opt_flow_params["criteria"]
        P.pt_scale_x, P.pt_scale_y = float(self.opt_flow_scale_factor[0]), float(self.opt_flow_scale_factor[1])
        P.win_w, P.win_h, P.lk_max_count = int(win[0]), int(win[1]), int(crit[1])
        P.lk_epsilon, P.lk_min_eig, P.max_error = float(crit[2]), 1e-4, float(self.max_error)
        P.ransac_max_iter, P.ransac_conf, P.ransac_thresh = int(self.ransac_max_iter), float(self.ransac_conf), 3.0
        P.inlier_thresh, P.refine_iters = int(self.inlier_thresh), 10
        P.good_idx, P.inl_idx = self.good_idx.data_ptr(), self.inl_idx.data_ptr()
        P.bg_kp, P.bg_kp_prev, P.bg_kp_count = (self.bg_kp.data_ptr(), self.bg_kp_prev.data_ptr(),
                                                self.bg_kp_count.data_ptr())
        P.est_boxes, P.sig = self.est_boxes.data_ptr(), self.sig.data_ptr()
        P.klt_tlbr, P.klt_ok = pool.klt_tlbr.data_ptr(), pool.klt_ok.data_ptr()
        P.klt_ok_bytes = pool.klt_ok.numel() * pool.klt_ok.element_size()
        P.inlier_ratio = pool.inlier_ratio.data_ptr()
        P.rounds_ahead = self.ROUNDS_AHEAD
        P.block_size, P.gradient_size = self.block_size, self.gradient_size
        P.use_harris, P.harris_k = int(self.use_harris), self.harris_k
        return P

    def _get_runner(self):
        if not self.USE_RUNNER or self.pool is None:
            return None
        from . import stagetime
        if stagetime.active():
            return None
        if self._runner is None:
            h = self._lib.fm_flow_plan_create(C.byref(self._plan()))
            if not h:
                raise _lib.FastMOTLibError("fm_flow_plan_create: " + self._lib.fm_last_error().decode(errors="replace"))
            self._runner = C.c_void_p(h)
        return self._runner

    def __del__(self):
        h = getattr(self, "_runner", None)
        if h is not None:
            try:
                self._lib.fm_flow_plan_destroy(h)
            except Exception:
                pass

    USE_RUNNER = True       # False keeps the call-by-call sequence (tests compare the two)

    # ------------------------------------------------------------------ lazily fetched attributes
    def _fetch_bg(self):
        if self._bg_cache is None:
            n = int(self.bg_kp_count.item())
            self._bg_cache = (self.bg_kp_prev[:n].cpu().numpy().copy(), self.bg_kp[:n].cpu().numpy().copy())
        return self._bg_cache

    @property
    def bg_keypoints(self):
        return self._fetch_bg()[1]

    @property
    def prev_bg_keypoints(self):
        return self._fetch_bg()[0]

    # ------------------------------------------------------------------
    def _to_device(self, frame):
        """The device Frame of a frame of this stage's size (BGR, or a Frame of any pixel format); host frames are
        uploaded."""
        return device_frame(frame, self._upload, size=self.size)

    def _preprocess(self, frame_dev, k):
        """cvtColor + resize (flow.py:153-154) and the LK pyramid with derivatives for buffer k (frame_dev: a device
        Frame or an HxWx3 u8 cuda tensor of this stage's size)."""
        s = stream_ptr()
        lib = self._lib
        frame_dev = device_frame(frame_dev, size=self.size)
        fm = C.byref(frame_dev.fm())
        if self._half:
            _lib.check(lib.fm_gray_half(fm, ptr(self.gray[k]), ptr(self.pyr[k][0]), s), "fm_gray_half")
        else:
            sw, sh = self.opt_flow_sz
            _lib.check(lib.fm_gray_resize(fm, ptr(self.gray[k]), ptr(self.pyr[k][0]), sw, sh, s), "fm_gray_resize")
        for i, (w, h) in enumerate(self.level_sizes):
            if i + 1 < len(self.level_sizes):
                _lib.check(lib.fm_pyr_level(ptr(self.pyr[k][i]), w, h, ptr(self.pyr[k][i + 1]), s), "fm_pyr_level")
            _lib.check(lib.fm_scharr(ptr(self.pyr[k][i]), w, h, ptr(self.deriv[k][i]), s), "fm_scharr")

    def init(self, frame):
        """flow.py:121-133"""
        if frame is None:
            return
        self._preprocess(self._to_device(frame), self.prev)
        self.bg_kp_count.zero_()
        self._bg_cache = None

    def predict_device(self, frame, tracks, h_dev, h_ok_dev):
        """Enqueue flow.py:135-264 for `tracks` (active Track objects); returns the nearest-first order
        [(trk_id, slot)].  Homography -> h_dev (9 f64), success flag -> h_ok_dev (i32)."""
        lib, pool = self._lib, self.pool
        W, H = self.size
        s = stream_ptr()
        cur = 1 - self.prev
        frame_dev = self._to_device(frame)
        # order tracks from closest to farthest (flow.py:157; Python's stable sort on Track.__lt__)
        # Track.__lt__ compares (tlbr[-1], -age); sorting on that key gives the identical (stable) order without a
        # Python-level __lt__ call per comparison (0.45 ms per frame at 200 tracks)
        tracks.sort(key=_depth_key, reverse=True)
        n = len(tracks)
        if n > self.max_tracks:
            raise MemoryError("more active tracks than Flow.max_tracks")
        self._order = [(t.trk_id, t.slot) for t in tracks]
        if n:
            self._h_slots[:n] = torch.as_tensor(np.fromiter((t.slot for t in tracks), np.int32, n))
            self.slots_dev[:n].copy_(self._h_slots[:n], non_blocking=True)
        runner = self._get_runner()
        if runner is not None:
            main = torch.cuda.current_stream()
            _lib.check(lib.fm_flow_predict(runner, C.byref(frame_dev.fm()), self.prev, n, ptr(h_dev), ptr(h_ok_dev),
                                           C.c_void_p(main.cuda_stream), C.c_void_p(self._side.cuda_stream)),
                       "fm_flow_predict")
            self.prev = cur                      # flow.py:212-213
            self._bg_cache = None
            self._affine_args = (n, W, H)
            self.rounds_last = self.ROUNDS_AHEAD
            if not self.defer_sync:
                self.finish_rounds(self.ROUNDS_AHEAD)
            return self._order
        self._preprocess(frame_dev, cur)
        pool.klt_ok.zero_()
        fl = self.flags.data_ptr()
        mk = self.obj_feat_params
        if self._default_feat:
            _lib.check(lib.fm_flow_keypoints(ptr(self.gray[self.prev]), W, H, ptr(pool.tlbr), ptr(self.slots_dev), n,
                                             ptr(self.owner), ptr(pool.kp), ptr(pool.kp_count), pool.max_kp,
                                             float(self.feat_density), float(self.feat_dist_factor),
                                             float(mk["qualityLevel"]), int(mk["maxCorners"]), ptr(self.jobs),
                                             ptr(self.scratch), self.scratch_cap, C.c_void_p(fl), C.c_void_p(fl + 4),
                                             s), "fm_flow_keypoints")
        else:
            _lib.check(lib.fm_flow_keypoints_cfg(
                ptr(self.gray[self.prev]), W, H, ptr(pool.tlbr), ptr(self.slots_dev), n, ptr(self.owner), ptr(pool.kp),
                ptr(pool.kp_count), pool.max_kp, float(self.feat_density), float(self.feat_dist_factor),
                float(mk["qualityLevel"]), int(mk["maxCorners"]), self.block_size, self.gradient_size,
                int(self.use_harris), self.harris_k, ptr(self.jobs), ptr(self.scratch), self.scratch_cap,
                C.c_void_p(fl), C.c_void_p(fl + 4), s), "fm_flow_keypoints_cfg")
        bw, bh = self.bg_feat_sz
        _lib.check(lib.fm_bg_small(ptr(self.gray[self.prev]), ptr(self.owner), W, H, ptr(self.bg), ptr(self.bg_mask),
                                   bw, bh, s), "fm_bg_small")
        ux = float(np.float32(1) / np.float32(self.bg_feat_scale_factor[0]))
        uy = float(np.float32(1) / np.float32(self.bg_feat_scale_factor[1]))
        _lib.check(lib.fm_fast_detect(ptr(self.bg), ptr(self.bg_mask), bw, bh, int(self.bg_feat_thresh), ux, uy,
                                      ptr(self.bg_score), ptr(self.bg_pts), ptr(self.bg_count), self.max_bg, s),
                   "fm_fast_detect")
        _lib.check(lib.fm_gather_points(ptr(pool.kp), ptr(pool.kp_count), pool.max_kp, ptr(self.slots_dev), n,
                                        ptr(self.bg_pts), ptr(self.bg_count), ptr(self.all_prev),
                                        ptr(self.trk_begin), ptr(self.meta), self.max_points, s), "fm_gather_points")
        win = self.opt_flow_params["winSize"]
        crit = self.opt_flow_params["criteria"]
        _lib.check(lib.fm_lk_track(C.byref(self.pyr_desc[self.prev]), C.byref(self.pyr_desc[cur]), ptr(self.all_prev),
                                   ptr(self.meta), float(self.opt_flow_scale_factor[0]),
                                   float(self.opt_flow_scale_factor[1]), int(win[0]), int(win[1]), int(crit[1]),
                                   float(crit[2]), 1e-4, float(self.max_error), ptr(self.all_cur), ptr(self.status),
                                   ptr(self.err), s), "fm_lk_track")
        self.prev = cur   # flow.py:212-213
        # camera-motion RANSAC (one CTA, latency bound) runs on a side stream next to the per-track affine rounds:
        # they only share read-only LK outputs.  The affine kernels no longer gate on h_ok -- when the homography
        # fails the caller drops every KLT box anyway (flow.py:227-229, tracker.py:152-156).
        main = torch.cuda.current_stream()
        self._ev_lk.record(main)
        self._side.wait_event(self._ev_lk)
        s_h = C.c_void_p(self._side.cuda_stream)
        _lib.check(lib.fm_ransac_homography(ptr(self.all_prev), ptr(self.all_cur), ptr(self.status), ptr(self.meta),
                                            int(self.ransac_max_iter), float(self.ransac_conf), 3.0,
                                            int(self.inlier_thresh), ptr(self.good_idx), ptr(self.inl_idx),
                                            ptr(h_dev), ptr(h_ok_dev), ptr(self.bg_kp), ptr(self.bg_kp_prev),
                                            ptr(self.bg_kp_count), self.max_bg, s_h), "fm_ransac_homography")
        self._ev_h.record(self._side)
        self._bg_cache = None
        # The serial "paint the predicted box, filter the next track" dependency is resolved by rounds (rounds past
        # the fixed point exit at once on the device).  ROUNDS_AHEAD rounds are enqueued without reading anything
        # back; the flags travel with the Kalman results (MultiTracker.apply_kalman) and `finish_rounds` runs more
        # rounds only in the rare case the fixed point was not reached (the Kalman launch is held by the same flag).
        self._affine_args = (n, W, H)
        rounds = 0
        for _ in range(self.ROUNDS_AHEAD // 4):
            rounds = self._enqueue_rounds(rounds, 4)
        if not self.defer_sync:
            rounds = self.finish_rounds(rounds)
        main.wait_event(self._ev_h)          # H / h_ok are consumed by the Kalman step that follows
        return self._order

    ROUNDS_AHEAD = 8

    def _enqueue_rounds(self, rounds, step):
        lib, pool = self._lib, self.pool
        n, W, H = self._affine_args
        fl = self.flags.data_ptr()
        _lib.check(lib.fm_ransac_affine_partial_batch(
            ptr(self.all_prev), ptr(self.all_cur), ptr(self.status), ptr(self.trk_begin), ptr(self.slots_dev), n,
            step, C.c_void_p(fl + 32), None, ptr(self.est_boxes), ptr(self.sig), ptr(pool.tlbr),
            ptr(pool.klt_tlbr), ptr(pool.klt_ok), ptr(pool.inlier_ratio), ptr(pool.kp), ptr(pool.kp_prev),
            ptr(pool.kp_count), pool.max_kp, W, H, int(self.ransac_max_iter), float(self.ransac_conf), 3.0,
            int(self.inlier_thresh), 10, rounds, stream_ptr()), "fm_ransac_affine_partial_batch")
        self.rounds_last = rounds + step
        return rounds + step

    def hold_flag_ptr(self):
        """Device address of the 'something changed' flag of the last enqueued round (0 = fixed point reached)."""
        return C.c_void_p(self.flags.data_ptr() + 32 + 4 * ((self.rounds_last - 1) & 15))

    def check_flags(self, hf):
        """hf: the 32 status ints copied back.  Raises on overflow; returns True when the rounds converged."""
        n = self._affine_args[0]
        if hf[1] == 2:
            raise MemoryError("Flow scratch overflow (code 2): the corner re-detection of this frame's boxes needs more "
                              f"than scratch_floats={self.scratch_cap} floats; raise scratch_floats")
        if hf[1] == 4:
            raise MemoryError(f"Flow keypoint overflow (code 4): a track kept more corners than its {self.max_kp} "
                              f"keypoint rows (maxCorners={self.obj_feat_params['maxCorners']}; at most "
                              f"{GFTT_MAX_CAND} rows per track); set maxCorners between 1 and {GFTT_MAX_CAND}")
        if hf[1] != 0:
            raise MemoryError(f"Flow keypoint status code {int(hf[1])}")
        if hf[27] != 0:
            raise MemoryError("Flow point overflow: the track keypoints and background corners of this frame are more "
                              f"than max_points={self.max_points}; raise max_points")
        return n == 0 or hf[8 + ((self.rounds_last - 1) & 15)] == 0 or self.rounds_last >= 2 * max(n, 1) + 2

    def finish_rounds(self, rounds=None):
        """Blocking tail of the rounds loop: read the flags, run four more rounds while something still changes."""
        lib = self._lib
        rounds = self.rounds_last if rounds is None else rounds
        fl = self.flags.data_ptr()
        while True:
            s = stream_ptr()
            lib.fm_memcpy_async(C.c_void_p(self._h_flags.data_ptr()), C.c_void_p(fl), 128, s)
            torch.cuda.current_stream().synchronize()
            if self.check_flags(self._h_flags.numpy()):
                break
            rounds = self._enqueue_rounds(rounds, 4)
        return rounds

    def fetch_klt_bboxes(self, order=None):
        """dict trk_id -> tlbr (f64) of the tracks whose box was predicted by the last predict_device."""
        order = self._order if order is None else order
        if not order:
            return {}
        slots = torch.as_tensor([s for _, s in order], device=self.pool.klt_ok.device)
        ok = self.pool.klt_ok[slots].cpu().numpy()
        boxes = self.pool.klt_tlbr[slots].cpu().numpy()
        return {tid: boxes[i].copy() for i, (tid, _) in enumerate(order) if ok[i]}

    def predict(self, frame, tracks):
        """Drop-in `Flow.predict` (flow.py:135-264): returns (dict trk_id -> tlbr, 3x3 homography or None)."""
        dev = self.pool.klt_ok.device
        h = torch.zeros(9, dtype=torch.float64, device=dev)
        ok = torch.zeros(1, dtype=torch.int32, device=dev)
        order = self.predict_device(frame, tracks, h, ok)
        if int(ok.item()) == 0:
            LOGGER.warning('Camera motion estimation failed')
            return {}, None
        return self.fetch_klt_bboxes(order), h.cpu().numpy().reshape(3, 3)
