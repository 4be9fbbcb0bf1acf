"""MOT: the per-frame scheduler with the reference's surface (fastmot/mot.py:25-196): `MOT(size, ...)`,
`reset(cap_dt)`, `step(frame)`, `visible_tracks()`, `frame_count`, `print_timing_info()`.

The frame is uploaded once per step and shared by the detector, the KLT stage and the ReID crops.  Detection
(letterbox + conv stack + decode + NMS) runs on its own CUDA stream concurrently with the KLT kernels, the ReID
batch concurrently with the batched Kalman step — the GPU-side analogue of the reference's GPU-inference /
CPU-tracking overlap (mot.py:138-158).
"""
from types import SimpleNamespace
from enum import Enum
import logging

import numpy as np
import torch

from .detector import YOLODetector, PublicDetector
from .feature_extractor import FeatureExtractor
from .tracker import MultiTracker
from .devmem import FrameResizer, FrameUploader, check_capture_size, check_pixel_format, device_frame, prefetch_frame
from .utils import Profiler

LOGGER = logging.getLogger(__name__)


class DetectorType(Enum):
    SSD = 0
    YOLO = 1
    PUBLIC = 2


class MOT:
    def __init__(self, size,
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
                 embeddings_tap=None,
                 pixel_format='BGR',
                 capture_size=None):
        """pixel_format: the layout every frame arrives in, in any form devmem.pixel_frame accepts for it:
          'BGR'  -- HxWx3 u8 (host array or cuda tensor);
          'NV12' -- as hardware video decoders and CSI cameras emit it (host (3H/2, W) array, pitched cuda tensor, or a
                    (Y, UV) pair of cuda planes);
          'I420' -- as software decoders (and PyAV / FFmpeg yuv420p) emit it (host (3H/2, W) array, tight cuda tensor,
                    or a (Y, U, V) triple of cuda planes);
          'YUY2' -- as USB cameras emit it (host or pitched cuda (H, W, 2));
          'BGRX' -- as nvvidconv emits it (host or pitched cuda (H, W, 4)).
        Raw frames are read in place by the letterbox, crop and KLT kernels; tracks, detections and embeddings are
        those of the BGR path on cv2.cvtColor(frame, code), code = COLOR_YUV2BGR_NV12, _I420, _YUY2 or
        COLOR_BGRA2BGR.

        size is the tracking size (the reference's resize_to).  capture_size: the (width, height) of the frames `step`
        and `prefetch` receive (the reference's stream_cfg.resolution; even for NV12 and I420, an even width for
        YUY2), when it differs from `size`.  Each frame is uploaded at that size and scaled to `size` on the GPU, bit
        for bit cv2.resize(frame, size) with INTER_LINEAR (of the cv2 decode for the raw formats); tracks and boxes are
        in tracking-size coordinates, as in the reference.  None, or capture_size == size, tracks the frames as they
        come."""
        self.size = size
        self.pixel_format = check_pixel_format(pixel_format)
        self.capture_size = check_capture_size(capture_size, size, self.pixel_format)
        self.detector_type = DetectorType[detector_type.upper()]
        assert detector_frame_skip >= 1
        self.detector_frame_skip = detector_frame_skip
        self.class_ids = tuple(np.unique(class_ids))
        self.draw = draw
        if draw:
            # mot.py:166-167,191-196 draw on the host frame with OpenCV; visualisation is outside the GPU hot path
            # (SURVEY.md §2.1 row 12).  Say so instead of silently ignoring the flag.
            LOGGER.warning("draw=True: fastmot_b200 has no visualizer (out of scope); frames are left untouched. "
                           "Use visible_tracks() to draw with your own code.")
        if self.detector_type == DetectorType.SSD:
            raise NotImplementedError("the SSD detector is not on the H100 hot path (SURVEY.md §2.1 row 2)")
        if yolo_detector_cfg is None:
            yolo_detector_cfg = SimpleNamespace()
        if feature_extractor_cfgs is None:
            feature_extractor_cfgs = (SimpleNamespace(),)
        if tracker_cfg is None:
            tracker_cfg = SimpleNamespace()
        if len(feature_extractor_cfgs) != len(class_ids):
            raise ValueError('Number of feature extractors must match length of class IDs')

        LOGGER.info('Loading detector model...')
        if self.detector_type == DetectorType.PUBLIC:
            if public_detector_cfg is None:
                raise ValueError("detector_type 'PUBLIC' needs public_detector_cfg (sequence_path, conf_thresh, max_area)")
            # mot.py:75-77: MOT Challenge public detections instead of the conv stack
            self.detector = PublicDetector(self.size, self.class_ids, self.detector_frame_skip,
                                           **vars(public_detector_cfg))
        else:
            self.detector = YOLODetector(self.size, self.class_ids, **vars(yolo_detector_cfg))
        LOGGER.info('Loading feature extractor models...')
        self.extractors = [FeatureExtractor(size=self.size, **vars(cfg)) for cfg in feature_extractor_cfgs]
        self.tracker = MultiTracker(self.size, self.extractors[0].metric, **vars(tracker_cfg),
                                    feat_dim=self.extractors[0].feature_dim)
        self.frame_count = 0
        self._uploader = FrameUploader(self.capture_size, depth=3, pixel_format=self.pixel_format)
        self._resizer = None if self.capture_size == tuple(size) else FrameResizer(size)
        self._det_stream = torch.cuda.Stream()
        self._main_ready = torch.cuda.Event()
        # ReID crops + OSNet run on their own stream so that the batched Kalman step, its read-back and the host side
        # of the association set-up proceed under the OSNet forward (mot.py:147-156: the reference overlaps the
        # extractor's GPU work with apply_kalman on the CPU the same way)
        self._reid_stream = torch.cuda.Stream()
        self._reid_done = torch.cuda.Event()
        # Optional callable frame_id -> recarray[DET_DTYPE]: replaces the detector's OUTPUT after the full
        # detector pipeline has run (synthetic-weight benchmarking: random weights cannot detect).
        self.detections_override = detections_override
        # Optional callable (frame_id, detections) -> (N, dim) embeddings replacing the ReID OUTPUT (parity rigs).
        self.embeddings_override = embeddings_override
        # Optional observer (frame_id, detections, embeddings): sees what the association stage is fed (parity rigs).
        self.embeddings_tap = embeddings_tap

    def visible_tracks(self):
        """Confirmed and active tracks (mot.py:103-112)."""
        return (track for track in self.tracker.tracks.values()
                if track.confirmed and track.active)

    def reset(self, cap_dt):
        """mot.py:114-123"""
        self.frame_count = 0
        self.tracker.reset(cap_dt)

    def _detect_async(self, frame_dev):
        self._main_ready.record()
        with torch.cuda.stream(self._det_stream):
            self._det_stream.wait_event(self._main_ready)   # frame upload happened on the main stream
            self.detector.detect_async(frame_dev)

    def _detections(self):
        dets = self.detector.postprocess()
        if self.detections_override is not None:
            dets = self.detections_override(self.frame_count)
        return dets

    def prefetch(self, frame):
        """Optional read-ahead: starts the host-to-device copy of the NEXT frame (the ndarray a later `step` call will
        receive) on an upload stream, so it overlaps the current step's kernels (role of the reference's VideoIO
        frame queue, fastmot/videoio.py:125-142)."""
        prefetch_frame(frame, self._uploader, self.pixel_format, self.capture_size)

    def step(self, frame):
        """mot.py:125-168"""
        frame_dev = device_frame(frame, self._uploader, self.pixel_format, self.capture_size)
        if self._resizer is not None:
            frame_dev = self._resizer.resize(frame_dev)    # on the main stream, before _main_ready is recorded
        detections = []
        if self.frame_count == 0:
            self._detect_async(frame_dev)
            detections = self._detections()
            self.tracker.init(frame_dev, detections)
        elif self.frame_count % self.detector_frame_skip == 0:
            with Profiler('preproc'):
                self._detect_async(frame_dev)
            with Profiler('detect'):
                with Profiler('track'):
                    self.tracker.compute_flow(frame_dev)
                detections = self._detections()
            with Profiler('extract'):
                cls_bboxes = self._split_bboxes_by_cls(detections.tlbr, detections.label, self.class_ids)
                main = torch.cuda.current_stream()
                with torch.cuda.stream(self._reid_stream):
                    # _main_ready (recorded by _detect_async on the main stream at the top of this step) orders the
                    # crops after the frame upload and after everything the previous update read from the engines
                    self._reid_stream.wait_event(self._main_ready)
                    for extractor, bboxes in zip(self.extractors, cls_bboxes):
                        extractor.extract_async(frame_dev, bboxes)
                    self._reid_done.record(self._reid_stream)
                with Profiler('track', aggregate=True):
                    self.tracker.apply_kalman()
                main.wait_event(self._reid_done)         # embeddings feed the association kernels on the main stream
                embeddings = [extractor.postprocess() for extractor in self.extractors]
                if len(embeddings) > 1:
                    embeddings = np.concatenate([np.asarray(e) for e in embeddings])
                else:
                    embeddings = embeddings[0]
                if self.embeddings_override is not None:
                    embeddings = self.embeddings_override(self.frame_count, detections)
                if self.embeddings_tap is not None:
                    self.embeddings_tap(self.frame_count, detections, embeddings)
            with Profiler('assoc'):
                self.tracker.update(self.frame_count, detections, embeddings)
        else:
            with Profiler('track'):
                self.tracker.track(frame_dev)
        self.frame_count += 1

    @staticmethod
    def print_timing_info():
        LOGGER.debug('=================Timing Stats=================')
        LOGGER.debug(f"{'track time:':<37}{Profiler.get_avg_millis('track'):>6.3f} ms")
        LOGGER.debug(f"{'preprocess time:':<37}{Profiler.get_avg_millis('preproc'):>6.3f} ms")
        LOGGER.debug(f"{'detect/flow time:':<37}{Profiler.get_avg_millis('detect'):>6.3f} ms")
        LOGGER.debug(f"{'feature extract/kalman filter time:':<37}"
                     f"{Profiler.get_avg_millis('extract'):>6.3f} ms")
        LOGGER.debug(f"{'association time:':<37}{Profiler.get_avg_millis('assoc'):>6.3f} ms")

    @staticmethod
    def _split_bboxes_by_cls(bboxes, labels, class_ids):
        """mot.py:180-189 for sorted labels; unlike the reference's bisect (SURVEY.md §8 a6) this also works for
        more than one class."""
        labels = np.asarray(labels)
        return [bboxes[labels == cls_id] for cls_id in class_ids]
