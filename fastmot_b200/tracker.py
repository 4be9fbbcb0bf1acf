"""MultiTracker: same constructor, methods and public attributes as fastmot/tracker.py:18-401, with the
numeric work moved to batched sm_90a kernels (csrc/kalman.cu, csrc/assoc.cu, csrc/klt_*.cu).

Host side keeps only what is inherently bookkeeping in the reference: the `tracks` dict, the `hist_tracks`
OrderedDict, the cascade's id lists/sets (their Python container orders are part of the observable
behaviour — SURVEY.md Appendix A) and logging.  Per frame there is one small H2D block (`Uplink`), a handful
of kernel launches and one D2H block (`Downlink`).
"""
from types import SimpleNamespace
from collections import OrderedDict
import ctypes as C
import itertools
import logging
import os

import numpy as np
import torch

from . import _lib
from .devmem import Uplink, Downlink, ptr, stream_ptr
from .pool import TrackPool
from .track import Track
from .kalman_filter import (KalmanFilter, FM_KF_WARP, FM_KF_PREDICT, FM_KF_UPDATE, FM_KF_MEAS_DET,
                            FM_KF_MEAS_BY_SLOT)
from .utils.numba_compat import set_difference_order

LOGGER = logging.getLogger(__name__)

_METRICS = {'EUCLIDEAN': 0, 'COSINE': 1}


class DeviceEmbeddings:
    """(N, dim) float32 embeddings resident on the GPU; converts to numpy on demand."""

    def __init__(self, tensor):
        self.tensor = tensor

    def __len__(self):
        return self.tensor.shape[0]

    @property
    def shape(self):
        return tuple(self.tensor.shape)

    def __array__(self, dtype=None, copy=None):
        a = self.tensor.detach().cpu().numpy()
        return a.astype(dtype) if dtype is not None else a


class MultiTracker:
    def __init__(self, size, metric,
                 max_age=6,
                 age_penalty=2,
                 motion_weight=0.2,
                 max_assoc_cost=0.9,
                 max_reid_cost=0.45,
                 iou_thresh=0.4,
                 duplicate_thresh=0.8,
                 occlusion_thresh=0.7,
                 conf_thresh=0.5,
                 confirm_hits=1,
                 history_size=50,
                 kalman_filter_cfg=None,
                 flow_cfg=None,
                 pool_capacity=2048,
                 feat_dim=512):
        self.size = size
        self.metric_name = metric.upper()
        if self.metric_name not in _METRICS:
            raise KeyError(metric)
        self.metric = _METRICS[self.metric_name]
        assert max_age >= 1
        self.max_age = max_age
        assert age_penalty >= 1
        self.age_penalty = age_penalty
        assert 0 <= motion_weight <= 1
        self.motion_weight = motion_weight
        assert 0 <= max_assoc_cost <= 2
        self.max_assoc_cost = max_assoc_cost
        assert 0 <= max_reid_cost <= 2
        self.max_reid_cost = max_reid_cost
        assert 0 <= iou_thresh <= 1
        self.iou_thresh = iou_thresh
        assert 0 <= duplicate_thresh <= 1
        self.duplicate_thresh = duplicate_thresh
        assert 0 <= occlusion_thresh <= 1
        self.occlusion_thresh = occlusion_thresh
        assert 0 <= conf_thresh <= 1
        self.conf_thresh = conf_thresh
        assert confirm_hits >= 1
        self.confirm_hits = confirm_hits
        assert history_size >= 0
        self.history_size = history_size

        if kalman_filter_cfg is None:
            kalman_filter_cfg = SimpleNamespace()
        if flow_cfg is None:
            flow_cfg = SimpleNamespace()

        self._lib = _lib.require_device()
        self.tracks = {}
        self.hist_tracks = OrderedDict()
        self._last_id = 0           # track ids are per tracker: several trackers in one process never share them
        self.kf = KalmanFilter(**vars(kalman_filter_cfg))
        from .flow import Flow
        self.flow = Flow(self.size, **vars(flow_cfg))
        # keypoint rows sized by obj_feat_params.maxCorners (1024 for the default 1000)
        self.pool = TrackPool(pool_capacity, feat_dim, max_kp=self.flow.max_kp)
        self.flow.bind_pool(self.pool)
        self.frame_rect = np.array([0., 0., size[0] - 1., size[1] - 1.])

        self.up = Uplink(1 << 20, depth=8)        # per-stage id lists (many flushes per update)
        self.up_det = Uplink(4 << 20, depth=2)    # detections of the current update (one flush per update)
        self.down = Downlink(1 << 20)
        dev = torch.device("cuda")
        self._cost = torch.empty(1 << 20, dtype=torch.float64, device=dev)   # up to 1024x1024
        self._lsa_ws = torch.empty(1 << 18, dtype=torch.uint8, device=dev)
        self._homography_dev = torch.zeros(9, dtype=torch.float64, device=dev)
        self._h_ok_dev = torch.zeros(1, dtype=torch.int32, device=dev)

        # FM_FUSE_CASCADE=0: one cost + assignment launch and one D2H per cascade stage (the r01 path, also taken for
        # frames with more than 256 detections / tracks per list and for single-stage frames); 2: fused whenever it fits
        self.fuse_cascade = {"0": 0, "2": 2}.get(os.environ.get("FM_FUSE_CASCADE", "1"), 1)   # 2 = always
        self._klt_bboxes = {}
        self._klt_stale = False
        self._klt_order = None
        self.homography = None

    # ------------------------------------------------------------------------------------------------
    @property
    def klt_bboxes(self):
        """dict trk_id -> tlbr of the last compute_flow (lazy D2H)."""
        if self._klt_stale:
            self._klt_bboxes = self.flow.fetch_klt_bboxes(self._klt_order)
            self._klt_stale = False
        return self._klt_bboxes

    @klt_bboxes.setter
    def klt_bboxes(self, value):
        self._klt_bboxes = value
        self._klt_stale = False

    def reset(self, dt):
        """tracker.py:109-119"""
        self.kf.reset_dt(dt)
        for trk in self.hist_tracks.values():
            self.pool.release(trk.slot)
        self.hist_tracks.clear()
        self._last_id = 0

    def _clear_tracks(self):
        for trk in self.tracks.values():
            self.pool.release(trk.slot)
        self.tracks.clear()

    def _new_tracks(self, frame_id, det_tlbr_host, det_labels_host, det_ids, det_tlbr_dev):
        """Spawn tracks for detections `det_ids` in that order (tracker.py:131-137, 288-293)."""
        n = len(det_ids)
        if n == 0:
            return
        new = []
        for det_id in det_ids:
            self._last_id += 1
            trk = Track(self._last_id, frame_id, det_tlbr_host[det_id].copy(), self.pool, int(det_labels_host[det_id]),
                        self.confirm_hits)
            self.tracks[trk.trk_id] = trk
            new.append(trk)
            LOGGER.debug(f"{'Detected:':<14}{trk}")
        slots = np.fromiter((t.slot for t in new), np.int32, n)
        self.pool.reset_slots(slots)
        p_slots = self.up.put(slots)
        p_idx = self.up.put(np.asarray(det_ids, np.int32))
        self.up.flush()
        self.kf.create_batched(self.pool.mean, self.pool.cov, self.pool.tlbr, p_slots, det_tlbr_dev, p_idx, n)

    def init(self, frame, detections):
        """tracker.py:121-137"""
        self._clear_tracks()
        self.flow.init(frame)
        det_tlbr = np.ascontiguousarray(detections.tlbr, np.float64).reshape(-1, 4)
        labels = np.asarray(detections.label).reshape(-1)
        if len(det_tlbr) == 0:
            return
        p_tlbr = self.up.put(det_tlbr)
        self._new_tracks(0, det_tlbr, labels, list(range(len(det_tlbr))), p_tlbr)

    def track(self, frame):
        """tracker.py:139-148"""
        self.compute_flow(frame)
        self.apply_kalman()

    # ------------------------------------------------------------------------------------------------
    def inject_flow(self, klt_bboxes, homography, inlier_ratios=None):
        """Test/diagnostic hook: bypass KLT with externally supplied results (e.g. the oracle's) so the
        Kalman/association stages can be checked in isolation (SURVEY.md §8c, tier T3 'KLT bypassed')."""
        self._injected = (dict(klt_bboxes), None if homography is None else np.asarray(homography, np.float64),
                          dict(inlier_ratios or {}))

    def compute_flow(self, frame):
        """tracker.py:150-162"""
        injected = getattr(self, '_injected', None)
        if injected is not None:
            self._injected = None
            klt, H, ratios = injected
            self.klt_bboxes, self.homography = klt, H
            if H is None:
                self._clear_tracks()
                return
            ids = [k for k in klt if k in self.tracks]
            self.pool.klt_ok.zero_()
            if ids:
                slots = torch.as_tensor(np.fromiter((self.tracks[k].slot for k in ids), np.int64, len(ids)),
                                        device=self.pool.klt_ok.device)
                boxes = torch.as_tensor(np.array([klt[k] for k in ids], np.float64).reshape(-1, 4),
                                        device=self.pool.klt_ok.device)
                self.pool.klt_tlbr[slots] = boxes
                self.pool.klt_ok[slots] = 1
                rat = torch.as_tensor(np.array([ratios.get(k, 1.0) for k in ids], np.float64),
                                      device=self.pool.klt_ok.device)
                self.pool.inlier_ratio[slots] = rat
            self._homography_dev.copy_(torch.as_tensor(H.reshape(9)))
            self._h_ok_dev.fill_(1)
            self._flow_pending = False
            return
        active_tracks = [track for track in self.tracks.values() if track.active]
        # the flow kernels leave klt boxes / flags in the pool and H / ok flag on the device; nothing is
        # synchronised here — apply_kalman consumes them and reports failure with its own D2H block.
        self.flow.defer_sync = True
        self._klt_order = self.flow.predict_device(frame, active_tracks, self._homography_dev, self._h_ok_dev)
        self._klt_stale = True
        self._flow_pending = True

    def apply_kalman(self):
        """tracker.py:164-183 as one launch + one D2H (which also carries the flow status and the KLT round flags)."""
        n = len(self.tracks)
        items = list(self.tracks.items())
        pending = getattr(self, '_flow_pending', False)

        def launch(hold):
            self.down.reset()
            p_hok, _ = self.down.alloc((1,), np.int32)
            p_H, _ = self.down.alloc((9,), np.float64)
            p_fl, _ = self.down.alloc((32,), np.int32)
            if n:
                slots = np.fromiter((t.slot for _, t in items), np.int32, n)
                mult = np.fromiter((max(self.age_penalty * t.age, 1) for _, t in items), np.float64, n)
                p_slots = self.up.put(slots)
                p_mult = self.up.put(mult)
                self.up.flush()
                p_tlbr, _ = self.down.alloc((n, 4), np.float64)
                p_lost, _ = self.down.alloc((n,), np.uint8)
                self.kf.step_batched(self.pool.mean, self.pool.cov, self.pool.tlbr, p_slots, n,
                                     FM_KF_WARP | FM_KF_PREDICT | FM_KF_UPDATE | FM_KF_MEAS_BY_SLOT,
                                     homography=ptr(self._homography_dev), h_ok=ptr(self._h_ok_dev),
                                     meas=ptr(self.pool.klt_tlbr), has_meas=ptr(self.pool.klt_ok),
                                     mult_num=p_mult, mult_den_pool=ptr(self.pool.inlier_ratio),
                                     frame_size=self.size, out_tlbr=p_tlbr, out_lost=p_lost, hold=hold)
            # piggy-back the flow status and the round flags on the same D2H
            self._copy_status(p_hok, p_H)
            self._lib.fm_memcpy_async(p_fl, ptr(self.flow.flags), 128, stream_ptr())
            return self.down.fetch()

        res = launch(self.flow.hold_flag_ptr() if pending else None)
        if pending and not self.flow.check_flags(res[2]):
            # rare: the KLT box rounds enqueued ahead did not converge; the Kalman launch was held on the device
            self.flow.finish_rounds()
            res = launch(None)
        res = [res[0], res[1]] + list(res[3:])
        h_ok = int(res[0][0])
        if getattr(self, '_flow_pending', False):
            self._flow_pending = False
            if not h_ok:
                self.homography = None
                self._klt_bboxes, self._klt_stale = {}, False
                LOGGER.warning('Camera motion estimation failed')
                self._clear_tracks()
                return
            self.homography = res[1].reshape(3, 3).copy()
        if not n:
            return
        tlbrs = res[2].copy()
        for (_, track), tlbr in zip(items, tlbrs):      # Track.update (track.py:108): the predicted box joins the history
            track.bboxes.append(tlbr)
        for k in np.nonzero(res[3])[0].tolist():        # tracks that left the frame (tracker.py:176-181), in dict order
            trk_id, track = items[k]
            if track.confirmed:
                LOGGER.info(f"{'Out:':<14}{track}")
            self._mark_lost(trk_id)

    def _copy_status(self, p_hok, p_H):
        s = stream_ptr()
        self._lib.fm_memcpy_async(p_hok, ptr(self._h_ok_dev), 4, s)
        self._lib.fm_memcpy_async(p_H, ptr(self._homography_dev), 72, s)

    # ------------------------------------------------------------------------------------------------
    def _split(self, c4r, nr, nc, row_ids, col_ids):
        """matching.py:57-70 on the kernel's col4row encoding."""
        assigned = c4r != -1
        cols = np.where(c4r >= 0, c4r, -2 - c4r)
        good = np.nonzero(c4r >= 0)[0]
        demoted = np.nonzero(c4r <= -2)[0]
        matches = [(row_ids[r], col_ids[cols[r]]) for r in good.tolist()]
        u_rows = [row_ids[r] for r in set_difference_order(nr, np.nonzero(assigned)[0])]
        u_cols = [col_ids[c] for c in set_difference_order(nc, cols[assigned])]
        for r in demoted.tolist():
            u_rows.append(row_ids[r])
            u_cols.append(col_ids[cols[r]])
        return matches, u_rows, u_cols

    def _solve(self, kind, trk_ids, det_ids, ctx, hist=False, greedy_max=None):
        """cost kernel + assignment kernel + D2H for one cascade stage.
        kind: 'feat' (tracker.py:314-341), 'iou' (343-353), 'reid' (355-366)."""
        nr, nc = len(trk_ids), len(det_ids)
        if nr == 0 or nc == 0:
            return [], list(trk_ids), list(det_ids)
        src = self.hist_tracks if hist else self.tracks
        trks = [src[t] for t in trk_ids]
        slots = np.fromiter((t.slot for t in trks), np.int32, nr)
        if kind == 'reid':
            # reference quirk (tracker.py:364): labels are taken from the FIRST n_hist history tracks
            labels = np.fromiter(itertools.islice((t.label for t in self.hist_tracks.values()), nr), np.int64, nr)
        else:
            labels = np.fromiter((t.label for t in trks), np.int64, nr)
        p_slots = self.up.put(slots)
        p_labels = self.up.put(labels)
        p_sel = self.up.put(np.asarray(det_ids, np.int32))
        self.up.flush()
        if nr * nc > self._cost.numel():
            self._cost = torch.empty(nr * nc, dtype=torch.float64, device=self._cost.device)
        s = stream_ptr()
        lib = self._lib
        if kind == 'feat':
            fill = min(self.max_assoc_cost + 0.1, 1.)
            rc = lib.fm_matching_cost(ptr(self.pool.feat_avg), ptr(self.pool.feat_valid), ptr(self.pool.mean),
                                      ptr(self.pool.cov), p_slots, p_labels, nr, ctx['emb'], ctx['tlbr'],
                                      ctx['labels'], ctx['occ'], p_sel, nc, ctx['dim'], self.metric, fill,
                                      self.motion_weight, self.max_assoc_cost, self.kf.params, ptr(self._cost), s)
        elif kind == 'reid':
            rc = lib.fm_matching_cost(ptr(self.pool.feat_avg), None, ptr(self.pool.mean), ptr(self.pool.cov),
                                      p_slots, p_labels, nr, ctx['emb'], ctx['tlbr'], ctx['labels'], None, p_sel,
                                      nc, ctx['dim'], self.metric, 1.0, -1.0, -1.0, self.kf.params,
                                      ptr(self._cost), s)
        else:
            rc = lib.fm_iou_cost(ptr(self.pool.tlbr), p_slots, p_labels, nr, ctx['tlbr'], ctx['labels'], p_sel, nc,
                                 1. - self.iou_thresh, ptr(self._cost), s)
        _lib.check(rc, "cost kernel")
        self.down.reset()
        p_c4r, _ = self.down.alloc((nr,), np.int32)
        if greedy_max is None:
            p_st, _ = self.down.alloc((1,), np.int32)
            need = lib.fm_lsa_workspace_bytes(nr, nc)
            if need > self._lsa_ws.numel():
                self._lsa_ws = torch.empty(int(need), dtype=torch.uint8, device=self._cost.device)
            _lib.check(lib.fm_lsa(ptr(self._cost), nr, nc, p_c4r, p_st, ptr(self._lsa_ws), s), "fm_lsa")
            res = self.down.fetch()
            if int(res[1][0]) != 0:
                raise ValueError('cost matrix is infeasible')
            return self._split(res[0], nr, nc, list(trk_ids), list(det_ids))
        p_ord, _ = self.down.alloc((nr,), np.int32)
        _lib.check(lib.fm_greedy_match(ptr(self._cost), nr, nc, float(greedy_max), p_c4r, p_ord, s),
                   "fm_greedy_match")
        res = self.down.fetch()
        return self._split_greedy(res[0], res[1], nr, nc, list(trk_ids), list(det_ids))

    @staticmethod
    def _split_greedy(c4r, order, nr, nc, row_ids, col_ids):
        """matching.py:73-97: matches in discovery order, leftovers in index order."""
        rows = np.nonzero(c4r >= 0)[0]
        rows = rows[np.argsort(order[rows], kind='stable')]
        matches = [(row_ids[r], col_ids[c4r[r]]) for r in rows.tolist()]
        taken = np.zeros(nc, bool)
        taken[c4r[rows]] = True
        u_rows = [row_ids[r] for r in np.nonzero(c4r < 0)[0].tolist()]
        u_cols = [col_ids[c] for c in np.nonzero(~taken)[0].tolist()]
        return matches, u_rows, u_cols

    def update(self, frame_id, detections, embeddings):
        """tracker.py:185-293"""
        det_tlbr = np.ascontiguousarray(detections.tlbr, np.float64).reshape(-1, 4)
        det_label = np.ascontiguousarray(detections.label, np.int64).reshape(-1)
        det_conf = np.asarray(detections.conf, np.float64).reshape(-1)
        n_det = len(det_tlbr)
        dev = self._cost.device

        # ---- stage the detections once
        if isinstance(embeddings, DeviceEmbeddings):
            emb_t = embeddings.tensor
        elif torch.is_tensor(embeddings):
            emb_t = embeddings
        else:
            emb_np = np.ascontiguousarray(embeddings, np.float32)
            emb_t = torch.as_tensor(emb_np).to(dev, non_blocking=False) if emb_np.size else \
                torch.zeros(0, self.pool.feat_dim, dtype=torch.float32, device=dev)
        emb_t = emb_t.contiguous()
        if emb_t.dtype != torch.float32:
            emb_t = emb_t.float()
        dim = emb_t.shape[1] if emb_t.ndim == 2 and emb_t.shape[0] else self.pool.feat_dim
        if dim != self.pool.feat_dim:
            raise ValueError(f"embedding dim {dim} != pool feat_dim {self.pool.feat_dim}")
        self._emb_keepalive = emb_t
        p_tlbr = self.up_det.put(det_tlbr)
        p_labels = self.up_det.put(det_label)
        self.up_det.flush()
        self.down.reset()
        occluded_det_mask = np.zeros(n_det, bool)
        occ_dev = torch.empty(max(n_det, 1), dtype=torch.uint8, device=dev)
        if n_det:
            _lib.check(self._lib.fm_find_occluded(p_tlbr, n_det, float(self.occlusion_thresh), ptr(occ_dev),
                                                  stream_ptr()), "fm_find_occluded")
        ctx = dict(emb=ptr(emb_t), tlbr=p_tlbr, labels=p_labels, occ=ptr(occ_dev), dim=dim)
        occ_fetched = False

        confirmed_by_depth, unconfirmed = self._group_tracks_by_depth()
        hist_ids = [trk_id for trk_id, track in self.hist_tracks.items() if track.avg_feat.count >= 2]

        fused = None
        # stages that will certainly run (the IoU stage of the still-active leftovers is only known on the device)
        n_stages = sum(1 for g in confirmed_by_depth if g) + bool(unconfirmed) + bool(hist_ids)
        if (self.fuse_cascade == 2 or (self.fuse_cascade and n_stages >= 2)) and 0 < n_det <= 256 and \
                len(unconfirmed) <= 256 and len(hist_ids) <= 256 and sum(len(g) for g in confirmed_by_depth) <= 256:
            # every stage in one launch, one D2H (csrc/assoc_cascade.cu).  With a single stage the per-stage path is
            # already one launch pair + one D2H and skips the full IoU / re-id matrices, so it stays.
            fused = self._cascade_fused(ctx, n_det, det_conf, confirmed_by_depth, unconfirmed, hist_ids, occ_dev)
        if fused is not None:
            (matches1, u_trk_ids1, matches2, u_trk_ids2, matches3, u_trk_ids3, reid_matches, invalid_u_det_ids,
             reid_u_det_ids, occluded_det_mask) = fused
        else:
            # 1st association: appearance + motion, young tracks first
            matches1 = []
            u_trk_ids1 = []
            u_det_ids = list(range(n_det))
            for depth, trk_ids in enumerate(confirmed_by_depth):
                if len(u_det_ids) == 0:
                    u_trk_ids1.extend(itertools.chain.from_iterable(confirmed_by_depth[depth:]))
                    break
                if len(trk_ids) == 0:
                    continue
                matches, u_trk_ids, u_det_ids = self._solve('feat', trk_ids, u_det_ids, ctx)
                matches1 += matches
                u_trk_ids1 += u_trk_ids

            # 2nd association: IoU with still-active tracks
            active = [trk_id for trk_id in u_trk_ids1 if self.tracks[trk_id].active]
            u_trk_ids1 = [trk_id for trk_id in u_trk_ids1 if not self.tracks[trk_id].active]
            matches2, u_trk_ids2, u_det_ids = self._solve('iou', active, u_det_ids, ctx)

            # 3rd association: unconfirmed tracks
            matches3, u_trk_ids3, u_det_ids = self._solve('iou', unconfirmed, u_det_ids, ctx)

            # re-identification against the lost-track history
            if n_det:
                occluded_det_mask = occ_dev[:n_det].cpu().numpy().astype(bool)
            u_det_ids = [det_id for det_id in u_det_ids if det_conf[det_id] >= self.conf_thresh]
            valid_u_det_ids = [det_id for det_id in u_det_ids if not occluded_det_mask[det_id]]
            invalid_u_det_ids = [det_id for det_id in u_det_ids if occluded_det_mask[det_id]]
            reid_matches, _, reid_u_det_ids = self._solve('reid', hist_ids, valid_u_det_ids, ctx, hist=True,
                                                          greedy_max=self.max_reid_cost)

        matches = itertools.chain(matches1, matches2, matches3)
        u_trk_ids = itertools.chain(u_trk_ids1, u_trk_ids2, u_trk_ids3)

        # rectify matches that may cause duplicate tracks
        matches, u_trk_ids = self._rectify_matches(matches, u_trk_ids, ctx)

        # reinstate re-identified tracks (tracker.py:250-256)
        if reid_matches:
            feat_slots, feat_idx, feat_cnt = [], [], []
            for trk_id, det_id in reid_matches:
                track = self.hist_tracks.pop(trk_id)
                LOGGER.info(f"{'Reidentified:':<14}{track}")
                track.reinstate(frame_id, det_tlbr[det_id].copy())
                self.tracks[trk_id] = track
                feat_slots.append(track.slot)
                feat_idx.append(det_id)
                feat_cnt.append(track.avg_feat.count)
            n = len(feat_slots)
            p_s = self.up.put(np.asarray(feat_slots, np.int32))
            p_i = self.up.put(np.asarray(feat_idx, np.int32))
            p_c = self.up.put(np.asarray(feat_cnt, np.int32))
            self.up.flush()
            self.kf.create_batched(self.pool.mean, self.pool.cov, self.pool.tlbr, p_s, p_tlbr, p_i, n)
            self.pool.kp_count[torch.as_tensor(feat_slots, device=dev)] = 0
            self._feature_update(p_s, p_i, p_c, n, ctx)

        # update matched tracks (tracker.py:258-274): one batched Kalman update, then host bookkeeping
        match_list = list(matches)
        if match_list:
            n = len(match_list)
            slots = np.fromiter((self.tracks[t].slot for t, _ in match_list), np.int32, n)
            meas = det_tlbr[[d for _, d in match_list]]
            p_s = self.up.put(slots)
            p_m = self.up.put(meas)
            self.up.flush()
            self.down.reset()
            p_out, _ = self.down.alloc((n, 4), np.float64)
            p_lost, _ = self.down.alloc((n,), np.uint8)
            self.kf.step_batched(self.pool.mean, self.pool.cov, self.pool.tlbr, p_s, n,
                                 FM_KF_UPDATE | FM_KF_MEAS_DET, meas=p_m, frame_size=self.size,
                                 out_tlbr=p_out, out_lost=p_lost)
            res = self.down.fetch()
            out_tlbr, out_lost = res[0].copy(), res[1].copy()
            feat_slots, feat_idx, feat_cnt = [], [], []
            for k, (trk_id, det_id) in enumerate(match_list):
                track = self.tracks[trk_id]
                is_valid = not occluded_det_mask[det_id]
                if track.hits == self.confirm_hits - 1:
                    LOGGER.info(f"{'Found:':<14}{track}")
                if out_lost[k]:
                    is_valid = False
                    if track.confirmed:
                        LOGGER.info(f"{'Out:':<14}{track}")
                    self._mark_lost(trk_id)
                track.add_detection(frame_id, out_tlbr[k], is_valid)
                if is_valid:
                    feat_slots.append(track.slot)
                    feat_idx.append(det_id)
                    feat_cnt.append(track.avg_feat.count)
            if feat_slots:
                p_s = self.up.put(np.asarray(feat_slots, np.int32))
                p_i = self.up.put(np.asarray(feat_idx, np.int32))
                p_c = self.up.put(np.asarray(feat_cnt, np.int32))
                self.up.flush()
                self._feature_update(p_s, p_i, p_c, len(feat_slots), ctx)

        # clean up lost tracks (tracker.py:276-285)
        for trk_id in u_trk_ids:
            track = self.tracks[trk_id]
            track.mark_missed()
            if not track.confirmed:
                LOGGER.debug(f"{'Unconfirmed:':<14}{track}")
                self.pool.release(track.slot)
                del self.tracks[trk_id]
                continue
            if track.age > self.max_age:
                LOGGER.info(f"{'Lost:':<14}{track}")
                self._mark_lost(trk_id)

        # start new tracks (tracker.py:287-293)
        new_det_ids = list(itertools.chain(invalid_u_det_ids, reid_u_det_ids))
        self._new_tracks(frame_id, det_tlbr, det_label, new_det_ids, p_tlbr)

    def _cascade_fused(self, ctx, n_det, det_conf, confirmed_by_depth, unconfirmed, hist_ids, occ_dev):
        """tracker.py:199-233 as three cost launches over ALL rows x ALL detections + one fm_assoc_cascade launch + one
        D2H.  Returns the lists `update` continues with (same contents and orders as the per-stage path)."""
        lib = self._lib
        conf_ids = list(itertools.chain.from_iterable(confirmed_by_depth))
        n_conf, n_unconf, n_hist = len(conf_ids), len(unconfirmed), len(hist_ids)
        row_ids = conf_ids + list(unconfirmed)
        n_rows = n_conf + n_unconf
        if n_rows + n_hist == 0:
            return None
        goff = np.zeros(len(confirmed_by_depth) + 1, np.int32)
        goff[1:] = np.cumsum([len(g) for g in confirmed_by_depth])
        trks = [self.tracks[t] for t in row_ids]
        slots = np.fromiter((t.slot for t in trks), np.int32, n_rows)
        labels = np.fromiter((t.label for t in trks), np.int64, n_rows)
        active = np.fromiter((t.active for t in trks[:n_conf]), np.uint8, n_conf)
        h_slots = np.fromiter((self.hist_tracks[t].slot for t in hist_ids), np.int32, n_hist)
        # reference quirk (tracker.py:364): labels are taken from the FIRST n_hist history tracks
        h_labels = np.fromiter(itertools.islice((t.label for t in self.hist_tracks.values()), n_hist), np.int64, n_hist)
        up = self.up
        p_slots, p_labels, p_goff = up.put(slots), up.put(labels), up.put(goff)
        p_active = up.put(active)
        p_hslots, p_hlabels = up.put(h_slots), up.put(h_labels)
        p_conf = up.put(np.ascontiguousarray(det_conf, np.float64))
        up.flush()
        need = (n_conf + n_rows + n_hist) * n_det + 256 * 256
        if need > self._cost.numel():
            self._cost = torch.empty(need, dtype=torch.float64, device=self._cost.device)
        base = self._cost.data_ptr()
        p_feat = C.c_void_p(base)
        p_iou = C.c_void_p(base + 8 * n_conf * n_det)
        p_reid = C.c_void_p(base + 8 * (n_conf + n_rows) * n_det)
        p_sub = C.c_void_p(base + 8 * (n_conf + n_rows + n_hist) * n_det)
        s = stream_ptr()
        if n_conf:
            fill = min(self.max_assoc_cost + 0.1, 1.)
            _lib.check(lib.fm_matching_cost(ptr(self.pool.feat_avg), ptr(self.pool.feat_valid), ptr(self.pool.mean),
                                            ptr(self.pool.cov), p_slots, p_labels, n_conf, ctx['emb'], ctx['tlbr'],
                                            ctx['labels'], ctx['occ'], None, n_det, ctx['dim'], self.metric, fill,
                                            self.motion_weight, self.max_assoc_cost, self.kf.params, p_feat, s),
                       "fm_matching_cost")
        if n_rows:
            _lib.check(lib.fm_iou_cost(ptr(self.pool.tlbr), p_slots, p_labels, n_rows, ctx['tlbr'], ctx['labels'], None,
                                       n_det, 1. - self.iou_thresh, p_iou, s), "fm_iou_cost")
        if n_hist:
            _lib.check(lib.fm_matching_cost(ptr(self.pool.feat_avg), None, ptr(self.pool.mean), ptr(self.pool.cov),
                                            p_hslots, p_hlabels, n_hist, ctx['emb'], ctx['tlbr'], ctx['labels'], None,
                                            None, n_det, ctx['dim'], self.metric, 1.0, -1.0, -1.0, self.kf.params,
                                            p_reid, s), "fm_matching_cost")
        cap = max(n_rows, n_det, n_hist, 1)
        n_out = int(lib.fm_assoc_cascade_out_ints(cap))
        self.down.reset()
        p_out, _ = self.down.alloc((n_out,), np.int32)
        d = _lib.FmCascadeDesc()
        d.n_det, d.n_conf, d.n_groups, d.n_unconf, d.n_hist, d.cap = n_det, n_conf, len(confirmed_by_depth), n_unconf, \
            n_hist, cap
        d.goff, d.conf_active = p_goff, p_active
        d.feat_cost, d.iou_cost, d.reid_cost = p_feat, p_iou, p_reid
        d.det_conf, d.det_occluded = p_conf, ptr(occ_dev)
        d.sub, d.out = p_sub, p_out
        d.conf_thresh, d.max_reid_cost = float(self.conf_thresh), float(self.max_reid_cost)
        _lib.check(lib.fm_assoc_cascade(C.byref(d), s), "fm_assoc_cascade")
        o = self.down.fetch()[0]
        hdr = o[:16]
        if int(hdr[0]) != 0:
            raise ValueError('cost matrix is infeasible')
        arr = [o[16 + k * cap: 16 + (k + 1) * cap] for k in range(14)]

        def pairs(rows, dets, n, ids):
            return [(ids[r], int(c)) for r, c in zip(rows[:n].tolist(), dets[:n].tolist())]

        def rows_of(a, n):
            return [row_ids[r] for r in a[:n].tolist()]

        n_m1, n_m2, n_m3, n_u1, n_u2, n_u3, n_reid, n_inv, n_ru = (int(v) for v in hdr[1:10])
        matches1 = pairs(arr[0], arr[1], n_m1, row_ids)
        matches2 = pairs(arr[2], arr[3], n_m2, row_ids)
        matches3 = pairs(arr[4], arr[5], n_m3, row_ids)
        u1, u2, u3 = rows_of(arr[6], n_u1), rows_of(arr[7], n_u2), rows_of(arr[8], n_u3)
        reid_matches = pairs(arr[9], arr[10], n_reid, hist_ids)
        invalid = arr[11][:n_inv].tolist()
        reid_u = arr[12][:n_ru].tolist()
        occ = arr[13][:n_det].astype(bool)
        return matches1, u1, matches2, u2, matches3, u3, reid_matches, invalid, reid_u, occ

    def _feature_update(self, p_slots, p_idx, p_cnt, n, ctx):
        rc = self._lib.fm_feature_update(ptr(self.pool.feat_sum), ptr(self.pool.feat_avg), ptr(self.pool.feat_last),
                                         ptr(self.pool.feat_valid), p_slots, ctx['emb'], p_idx, p_cnt, n,
                                         ctx['dim'], stream_ptr())
        _lib.check(rc, "fm_feature_update")

    def _mark_lost(self, trk_id):
        """tracker.py:295-300"""
        track = self.tracks.pop(trk_id)
        if track.confirmed:
            self.hist_tracks[trk_id] = track
            if len(self.hist_tracks) > self.history_size:
                _, old = self.hist_tracks.popitem(last=False)
                self.pool.release(old.slot)
        else:
            self.pool.release(track.slot)

    def _group_tracks_by_depth(self, group_size=2):
        """tracker.py:302-312"""
        n_depth = (self.max_age + group_size) // group_size
        confirmed_by_depth = [[] for _ in range(n_depth)]
        unconfirmed = []
        for trk_id, track in self.tracks.items():
            if track.confirmed:
                depth = track.age // group_size
                confirmed_by_depth[depth].append(trk_id)
            else:
                unconfirmed.append(trk_id)
        return confirmed_by_depth, unconfirmed

    def _rectify_matches(self, matches, u_trk_ids, ctx):
        """tracker.py:368-401"""
        matches, u_trk_ids = set(matches), set(u_trk_ids)
        inactive_matches = [match for match in matches if not self.tracks[match[0]].active]
        u_active = [trk_id for trk_id in u_trk_ids
                    if self.tracks[trk_id].confirmed and self.tracks[trk_id].active]

        n_inactive_matches = len(inactive_matches)
        if n_inactive_matches == 0 or len(u_active) == 0:
            return matches, u_trk_ids

        m_inactive, det_ids = zip(*inactive_matches)
        # IoU distance between unmatched active tracks and the detections claimed by inactive tracks
        nr, nc = len(u_active), n_inactive_matches
        slots = np.fromiter((self.tracks[t].slot for t in u_active), np.int32, nr)
        p_slots = self.up.put(slots)
        p_sel = self.up.put(np.asarray(det_ids, np.int32))
        self.up.flush()
        s = stream_ptr()
        _lib.check(self._lib.fm_iou_cost(ptr(self.pool.tlbr), p_slots, None, nr, ctx['tlbr'], None, p_sel, nc,
                                         -1.0, ptr(self._cost), s), "fm_iou_cost")
        self.down.reset()
        p_c4r, _ = self.down.alloc((nr,), np.int32)
        p_ord, _ = self.down.alloc((nr,), np.int32)
        _lib.check(self._lib.fm_greedy_match(ptr(self._cost), nr, nc, 1. - self.duplicate_thresh, p_c4r, p_ord, s),
                   "fm_greedy_match")
        res = self.down.fetch()
        dup_matches, _, _ = self._split_greedy(res[0], res[1], nr, nc, list(u_active), list(range(nc)))

        for u_trk_id, col in dup_matches:
            m_trk_id, det_id = m_inactive[col], det_ids[col]
            t_u_active, t_m_inactive = self.tracks[u_trk_id], self.tracks[m_trk_id]
            if t_m_inactive.end_frame < t_u_active.start_frame:
                LOGGER.debug(f"{'Merged:':<14}{u_trk_id} -> {m_trk_id}")
                self._merge_continuation(t_m_inactive, t_u_active)
                u_trk_ids.remove(u_trk_id)
                self.pool.release(t_u_active.slot)
                del self.tracks[u_trk_id]
            else:
                LOGGER.debug(f"{'Duplicate:':<14}{m_trk_id} -> {u_trk_id}")
                u_trk_ids.remove(u_trk_id)
                u_trk_ids.add(m_trk_id)
                matches.remove((m_trk_id, det_id))
                matches.add((u_trk_id, det_id))
        return matches, u_trk_ids

    def _merge_continuation(self, dst, other):
        """Track.merge_continuation (track.py:206-219) on pool slots (rare path)."""
        dst.frame_ids.extend(other.frame_ids)
        dst.bboxes.extend(other.bboxes)
        dst.age = other.age
        dst.hits += other.hits
        self.pool.copy_slot(dst.slot, other.slot, ['mean', 'cov', 'tlbr', 'kp', 'kp_prev', 'kp_count',
                                                   'inlier_ratio'])
        if other.avg_feat.count:
            self.pool.copy_slot(dst.slot, other.slot, ['feat_last'])
        # AverageFeature.merge (track.py:109-117)
        dst.avg_feat.count += other.avg_feat.count
        if dst.avg_feat.count == other.avg_feat.count:      # dst had no feature yet
            if other.avg_feat.count:
                self.pool.copy_slot(dst.slot, other.slot, ['feat_sum', 'feat_avg', 'feat_valid'])
        elif other.avg_feat.count:
            p_s = self.up.put(np.asarray([dst.slot], np.int32))
            p_i = self.up.put(np.asarray([other.slot], np.int32))
            p_c = self.up.put(np.asarray([dst.avg_feat.count], np.int32))
            self.up.flush()
            rc = self._lib.fm_feature_update(ptr(self.pool.feat_sum), ptr(self.pool.feat_avg), None,
                                             ptr(self.pool.feat_valid), p_s, ptr(self.pool.feat_sum), p_i, p_c, 1,
                                             self.pool.feat_dim, stream_ptr())
            _lib.check(rc, "fm_feature_update")
