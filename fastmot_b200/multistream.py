"""MultiStreamMOT: several camera streams of one frame size tracked in one process, with the surface of `MOT`.

All streams share one detector cadence, so a detector frame falls on the same step for every stream.  That is what
lets the streams share the networks: on a detector frame the N frames go through ONE batched YOLO forward
(YOLODetector(batch=N)), and the crops of all N streams through ONE OSNet forward (FeatureExtractor.
extract_multi_async).  Tracking stays per stream: one MultiTracker each, stepped exactly as MOT steps its own, so
every stream's tracks (ids included) are those a separate MOT would produce on that stream alone.
"""
from types import SimpleNamespace
import logging

import numpy as np
import torch

from .detector import YOLODetector
from .feature_extractor import FeatureExtractor
from .tracker import MultiTracker
from .devmem import FrameUploader
from .mot import DetectorType
from .utils import Profiler

LOGGER = logging.getLogger(__name__)


class MultiStreamMOT:
    def __init__(self, size, num_streams,
                 detector_type='YOLO',
                 detector_frame_skip=5,
                 class_ids=(1,),
                 ssd_detector_cfg=None,
                 yolo_detector_cfg=None,
                 public_detector_cfg=None,
                 feature_extractor_cfgs=None,
                 tracker_cfg=None,
                 visualizer_cfg=None,
                 draw=False,
                 detections_override=None,
                 embeddings_override=None):
        """size: (width, height) shared by every stream.  The keyword arguments are MOT's, so the reference's
        `mot_cfg` (cfg/mot.json) passes unchanged; ssd_detector_cfg, public_detector_cfg and visualizer_cfg are
        accepted and unused, since only the YOLO detector runs several streams.  detections_override(stream,
        frame_id) and embeddings_override(stream, frame_id, detections) replace the networks' OUTPUT after both ran,
        as MOT's hooks do."""
        if not (isinstance(size, (tuple, list)) and len(size) == 2 and all(np.isscalar(v) for v in size)):
            raise ValueError("MultiStreamMOT takes one frame size (width, height) shared by every stream; "
                             "streams of different sizes need separate trackers")
        self.size = tuple(int(v) for v in size)
        if num_streams < 1:
            raise ValueError("num_streams must be >= 1")
        self.num_streams = num_streams
        self.detector_type = DetectorType[detector_type.upper()]
        if self.detector_type != DetectorType.YOLO:
            raise NotImplementedError(f"detector_type {detector_type!r}: several streams are tracked with the batched "
                                      "YOLO detector only")
        assert detector_frame_skip >= 1
        self.detector_frame_skip = detector_frame_skip
        self.class_ids = tuple(np.unique(class_ids))
        self.draw = draw
        if draw:
            LOGGER.warning("draw=True: fastmot_b200 has no visualizer (out of scope); frames are left untouched. "
                           "Use visible_tracks(stream) to draw with your own code.")
        if yolo_detector_cfg is None:
            yolo_detector_cfg = SimpleNamespace()
        if feature_extractor_cfgs is None:
            feature_extractor_cfgs = (SimpleNamespace(),)
        if tracker_cfg is None:
            tracker_cfg = SimpleNamespace()
        if len(feature_extractor_cfgs) != len(class_ids):
            raise ValueError('Number of feature extractors must match length of class IDs')

        self.detector = YOLODetector(self.size, self.class_ids, batch=num_streams, **vars(yolo_detector_cfg))
        # one extractor per class as in MOT; its crop capacity holds every stream's crops
        self.extractors = []
        for cfg in feature_extractor_cfgs:
            kw = dict(vars(cfg))
            kw['max_crops'] = kw.get('max_crops', 512) * num_streams
            self.extractors.append(FeatureExtractor(size=self.size, **kw))
        self.trackers = [MultiTracker(self.size, self.extractors[0].metric, **vars(tracker_cfg),
                                      feat_dim=self.extractors[0].feature_dim) for _ in range(num_streams)]
        self.frame_count = 0
        self._uploaders = [FrameUploader(self.size, depth=3) for _ in range(num_streams)]
        self._det_stream = torch.cuda.Stream()
        self._main_ready = torch.cuda.Event()
        self._reid_stream = torch.cuda.Stream()
        self._reid_done = torch.cuda.Event()
        self.detections_override = detections_override
        self.embeddings_override = embeddings_override

    def visible_tracks(self, stream):
        """Confirmed and active tracks of one stream."""
        return (track for track in self.trackers[stream].tracks.values() if track.confirmed and track.active)

    def reset(self, cap_dt):
        self.frame_count = 0
        for trk in self.trackers:
            trk.reset(cap_dt)

    def prefetch(self, frames):
        """Starts the uploads of the frames a later `step` call will receive (host arrays only)."""
        self._check_frames(frames)
        for up, f in zip(self._uploaders, frames):
            if not torch.is_tensor(f):
                up.prefetch(f)

    def _check_frames(self, frames):
        if len(frames) != self.num_streams:
            raise ValueError(f"expected {self.num_streams} frames, got {len(frames)}")

    def _detect_async(self, frames_dev):
        self._main_ready.record()
        with torch.cuda.stream(self._det_stream):
            self._det_stream.wait_event(self._main_ready)   # frame uploads happened on the main stream
            self.detector.detect_batch_async(frames_dev)

    def _detections(self):
        dets = self.detector.postprocess_batch()
        if self.detections_override is not None:
            dets = [self.detections_override(s, self.frame_count) for s in range(self.num_streams)]
        return dets

    def step(self, frames):
        """One step of every stream: frames[s] is stream s's next HxWx3 u8 frame (host array or cuda tensor)."""
        self._check_frames(frames)
        frames_dev = [f if torch.is_tensor(f) else up.upload(f) for f, up in zip(frames, self._uploaders)]
        if self.frame_count == 0:
            self._detect_async(frames_dev)
            detections = self._detections()
            for trk, f, d in zip(self.trackers, frames_dev, detections):
                trk.init(f, d)
        elif self.frame_count % self.detector_frame_skip == 0:
            with Profiler('preproc'):
                self._detect_async(frames_dev)
            with Profiler('detect'):
                with Profiler('track'):
                    for trk, f in zip(self.trackers, frames_dev):
                        trk.compute_flow(f)
                detections = self._detections()
            with Profiler('extract'):
                # [class][stream] boxes, split by class as MOT does
                cls_bboxes = [[d.tlbr[np.asarray(d.label) == cls_id] for d in detections] for cls_id in self.class_ids]
                main = torch.cuda.current_stream()
                with torch.cuda.stream(self._reid_stream):
                    self._reid_stream.wait_event(self._main_ready)
                    for extractor, bboxes in zip(self.extractors, cls_bboxes):
                        extractor.extract_multi_async(frames_dev, bboxes)
                    self._reid_done.record(self._reid_stream)
                with Profiler('track', aggregate=True):
                    for trk in self.trackers:
                        trk.apply_kalman()
                main.wait_event(self._reid_done)
                per_cls = [extractor.postprocess() for extractor in self.extractors]
                embeddings = []
                for s in range(self.num_streams):
                    if len(per_cls) > 1:
                        embeddings.append(np.concatenate([np.asarray(e[s]) for e in per_cls]))
                    else:
                        embeddings.append(per_cls[0][s])
                if self.embeddings_override is not None:
                    embeddings = [self.embeddings_override(s, self.frame_count, detections[s])
                                  for s in range(self.num_streams)]
            with Profiler('assoc'):
                for trk, d, e in zip(self.trackers, detections, embeddings):
                    trk.update(self.frame_count, d, e)
        else:
            with Profiler('track'):
                for trk, f in zip(self.trackers, frames_dev):
                    trk.track(f)
        self.frame_count += 1
