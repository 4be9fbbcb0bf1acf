"""MultiCameraMOT: a group of cameras tracked in one process, each with its own frame size and its own timeline.

Every camera keeps MOT's schedule on its own frames: its local frame 0 initialises its tracker and every
detector_frame_skip-th local frame after it is a detector frame.  A camera that has no frame on a step (not started
yet, dropped, ended) passes None and does nothing; its frame count does not advance.  On each step the cameras on a
detector frame (init included) share the networks: their frames go through ONE letterbox launch and ONE YOLO forward
at batch k = their number (YOLODetector(batch=N) runs a batch-k engine that shares the batch-N engine's memory), and
the crops of the non-init ones through ONE OSNet forward.  The other present cameras track.  Tracking stays per
camera: one MultiTracker each, stepped exactly as MOT steps its own, so each camera's tracks (ids included) are those
a separate MOT of its size would produce on that camera's frames alone.

Starting the cameras on different steps staggers their detector frames, so each step carries about k = N / K cameras'
detector work instead of all N every K-th step.
"""
from types import SimpleNamespace
import logging

import numpy as np
import torch

from .detector import YOLODetector
from .feature_extractor import FeatureExtractor
from .tracker import MultiTracker
from .devmem import FrameResizer, FrameUploader, check_capture_size, check_pixel_format, device_frame, prefetch_frame
from .mot import DetectorType
from .utils import Profiler

LOGGER = logging.getLogger(__name__)


def plan_step(frame_counts, present, detector_frame_skip):
    """What each camera does on one step, from its local frame count and whether it has a frame: returns the camera
    indices that (init, detect, track), each ascending.  Absent cameras are in none of the three."""
    init, detect, track = [], [], []
    for s, (n, p) in enumerate(zip(frame_counts, present)):
        if not p:
            continue
        if n == 0:
            init.append(s)
        elif n % detector_frame_skip == 0:
            detect.append(s)
        else:
            track.append(s)
    return init, detect, track


class MultiCameraMOT:
    def __init__(self, sizes,
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
                 embeddings_override=None,
                 pixel_format=None,
                 capture_size=None,
                 capture_sizes=None,
                 pixel_formats=None):
        """sizes: one (width, height) tracking size per camera.  pixel_formats: one pixel format per camera (any of
        MOT's: 'BGR', 'NV12', 'I420', 'YUY2', 'BGRX'), e.g. a USB camera (YUY2), an RTSP camera (I420) and a CSI
        camera (NV12) in one group; pixel_format: one format for every camera (MOT's keyword); give at most one of the
        two (neither: 'BGR').  The keyword arguments are MOT's, so the reference's `mot_cfg`
        (cfg/mot.json) passes unchanged; ssd_detector_cfg, public_detector_cfg and visualizer_cfg are accepted and
        unused, since only the YOLO detector runs several cameras.  detections_override(camera, frame_id) and
        embeddings_override(camera, frame_id, detections) replace the networks' OUTPUT after both ran, as MOT's hooks
        do; frame_id is the camera's local frame count.

        capture_sizes: one entry per camera, the (width, height) its frames arrive at, or None for a camera whose
        frames come at its tracking size; a scaled camera's frames are resized on the GPU as MOT(capture_size=...)
        resizes them.  capture_size: one capture size for every camera (MOT's keyword); give at most one of the two."""
        if len(sizes) < 1:
            raise ValueError("MultiCameraMOT needs at least one camera")
        self.sizes = []
        for wh in sizes:
            if not (isinstance(wh, (tuple, list)) and len(wh) == 2 and all(np.isscalar(v) for v in wh)):
                raise ValueError(f"every camera size must be (width, height), got {wh!r}")
            self.sizes.append(tuple(int(v) for v in wh))
        self.num_cameras = N = len(self.sizes)
        if pixel_format is not None and pixel_formats is not None:
            raise ValueError("give pixel_format (every camera) or pixel_formats (one per camera), not both")
        if pixel_formats is None:
            pixel_formats = [pixel_format or 'BGR'] * N
        if len(pixel_formats) != N:
            raise ValueError(f"pixel_formats: expected {N} entries (one per camera), got {len(pixel_formats)}")
        self.pixel_formats = []
        for s, fmt in enumerate(pixel_formats):
            try:
                self.pixel_formats.append(check_pixel_format(fmt))
            except ValueError as e:
                raise ValueError(f"camera {s}: {e}") from None
        # the group's one format, None for a group of several
        self.pixel_format = self.pixel_formats[0] if len(set(self.pixel_formats)) == 1 else None
        if capture_size is not None and capture_sizes is not None:
            raise ValueError("give capture_size (every camera) or capture_sizes (one per camera), not both")
        if capture_sizes is None:
            capture_sizes = [capture_size] * N
        if len(capture_sizes) != N:
            raise ValueError(f"capture_sizes: expected {N} entries (one per camera), got {len(capture_sizes)}")
        self.capture_sizes = []
        for s, (cs, wh, fmt) in enumerate(zip(capture_sizes, self.sizes, self.pixel_formats)):
            try:
                self.capture_sizes.append(check_capture_size(cs, wh, fmt))
            except ValueError as e:
                raise ValueError(f"camera {s}: {e}") from None
        self.detector_type = DetectorType[detector_type.upper()]
        if self.detector_type != DetectorType.YOLO:
            raise NotImplementedError(f"detector_type {detector_type!r}: several cameras are tracked with the batched "
                                      "YOLO detector only")
        assert detector_frame_skip >= 1
        self.detector_frame_skip = detector_frame_skip
        self.class_ids = tuple(np.unique(class_ids))
        self.draw = draw
        if draw:
            LOGGER.warning("draw=True: fastmot_b200 has no visualizer (out of scope); frames are left untouched. "
                           "Use visible_tracks(camera) to draw with your own code.")
        if yolo_detector_cfg is None:
            yolo_detector_cfg = SimpleNamespace()
        if feature_extractor_cfgs is None:
            feature_extractor_cfgs = (SimpleNamespace(),)
        if tracker_cfg is None:
            tracker_cfg = SimpleNamespace()
        if len(feature_extractor_cfgs) != len(class_ids):
            raise ValueError('Number of feature extractors must match length of class IDs')

        # a detector call over k cameras' frames runs the batch-k engine (the batch-N one at k = N), each frame with the
        # geometry of its own size
        self.detector = YOLODetector(self.sizes[0], self.class_ids, batch=N, **vars(yolo_detector_cfg))
        # one extractor per class as in MOT; its crop capacity holds every camera's crops
        self.extractors = []
        for cfg in feature_extractor_cfgs:
            kw = dict(vars(cfg))
            kw['max_crops'] = kw.get('max_crops', 512) * N
            self.extractors.append(FeatureExtractor(size=self.sizes[0], **kw))
        self.trackers = [MultiTracker(wh, self.extractors[0].metric, **vars(tracker_cfg),
                                      feat_dim=self.extractors[0].feature_dim) for wh in self.sizes]
        self.frame_counts = [0] * N
        self._uploaders = [FrameUploader(wh, depth=3, pixel_format=fmt)
                           for wh, fmt in zip(self.capture_sizes, self.pixel_formats)]
        self._resizers = [None if cs == wh else FrameResizer(wh) for cs, wh in zip(self.capture_sizes, self.sizes)]
        self._det_stream = torch.cuda.Stream()
        self._main_ready = torch.cuda.Event()
        self._reid_stream = torch.cuda.Stream()
        self._reid_done = torch.cuda.Event()
        self.detections_override = detections_override
        self.embeddings_override = embeddings_override

    def visible_tracks(self, camera):
        """Confirmed and active tracks of one camera."""
        return (track for track in self.trackers[camera].tracks.values() if track.confirmed and track.active)

    def reset(self, cap_dt):
        """Every camera starts over: its next frame is its local frame 0."""
        self.frame_counts = [0] * self.num_cameras
        for trk in self.trackers:
            trk.reset(cap_dt)

    def reset_stream(self, camera, cap_dt):
        """One camera starts over (a reconnect): its next frame is its local frame 0, its track ids restart at 1."""
        self.frame_counts[camera] = 0
        self.trackers[camera].reset(cap_dt)

    def prefetch(self, frames):
        """Starts the uploads of the frames a later `step` call will receive (host arrays only; None is skipped)."""
        self._each_frame(prefetch_frame, frames)

    def _each_frame(self, fn, frames):
        """[fn(frame, camera's uploader, camera's pixel format, camera's capture size) or None] over the cameras' frames
        (None: no frame); a frame of the wrong size or form raises ValueError naming its camera."""
        if len(frames) != self.num_cameras:
            raise ValueError(f"expected {self.num_cameras} frames, got {len(frames)}")
        out = []
        for s, (f, up, fmt, wh) in enumerate(zip(frames, self._uploaders, self.pixel_formats, self.capture_sizes)):
            try:
                out.append(None if f is None else fn(f, up, fmt, wh))
            except ValueError as e:
                raise ValueError(f"camera {s}: {e}") from None
        return out

    def _detect_async(self, frames_dev):
        self._main_ready.record()
        with torch.cuda.stream(self._det_stream):
            self._det_stream.wait_event(self._main_ready)   # frame uploads happened on the main stream
            self.detector.detect_batch_async(frames_dev)

    def _detections(self, cams):
        dets = self.detector.postprocess_batch(names=[f"camera {s}" for s in cams])
        if self.detections_override is not None:
            dets = [self.detections_override(s, self.frame_counts[s]) for s in cams]
        return dict(zip(cams, dets))

    def step(self, frames):
        """One step of the group: frames[s] is camera s's next frame in its pixel format, in any form MOT takes for
        that format (HxWx3 u8 host array or cuda tensor for BGR), or None when camera s has no frame on this step."""
        frames_dev = self._each_frame(device_frame, frames)
        # scaled cameras: resized on the main stream, before _main_ready is recorded (devmem.FrameResizer)
        frames_dev = [f if f is None or r is None else r.resize(f) for f, r in zip(frames_dev, self._resizers)]
        init, detect, track = plan_step(self.frame_counts, [f is not None for f in frames], self.detector_frame_skip)
        cams = sorted(init + detect)                 # the detector batch, in camera order
        if not cams:
            with Profiler('track'):
                for s in track:
                    self.trackers[s].track(frames_dev[s])
        else:
            with Profiler('preproc'):
                self._detect_async([frames_dev[s] for s in cams])
            with Profiler('detect'):
                # the other cameras' tracking steps run on the main stream under the detector forward
                with Profiler('track'):
                    for s in detect:
                        self.trackers[s].compute_flow(frames_dev[s])
                    for s in track:
                        self.trackers[s].track(frames_dev[s])
                detections = self._detections(cams)
            for s in init:
                self.trackers[s].init(frames_dev[s], detections[s])
        if detect:
            with Profiler('extract'):
                # [class][camera] boxes, split by class as MOT does
                cls_bboxes = [[detections[s].tlbr[np.asarray(detections[s].label) == cls_id] for s in detect]
                              for cls_id in self.class_ids]
                main = torch.cuda.current_stream()
                with torch.cuda.stream(self._reid_stream):
                    self._reid_stream.wait_event(self._main_ready)
                    for extractor, bboxes in zip(self.extractors, cls_bboxes):
                        extractor.extract_multi_async([frames_dev[s] for s in detect], bboxes)
                    self._reid_done.record(self._reid_stream)
                with Profiler('track', aggregate=True):
                    for s in detect:
                        self.trackers[s].apply_kalman()
                main.wait_event(self._reid_done)
                per_cls = [extractor.postprocess() for extractor in self.extractors]
                embeddings = {}
                for i, s in enumerate(detect):
                    if len(per_cls) > 1:
                        embeddings[s] = np.concatenate([np.asarray(e[i]) for e in per_cls])
                    else:
                        embeddings[s] = per_cls[0][i]
                if self.embeddings_override is not None:
                    embeddings = {s: self.embeddings_override(s, self.frame_counts[s], detections[s]) for s in detect}
            with Profiler('assoc'):
                for s in detect:
                    self.trackers[s].update(self.frame_counts[s], detections[s], embeddings[s])
        for s in init + detect + track:
            self.frame_counts[s] += 1
