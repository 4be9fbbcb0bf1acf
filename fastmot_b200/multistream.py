"""MultiStreamMOT: several camera streams of one frame size tracked in one process, with the surface of `MOT`.

It is the MultiCameraMOT of N equal-size cameras that all deliver a frame on every step.  They share one detector
cadence, so a detector frame falls on the same step for every stream: the N frames go through ONE batched YOLO forward
(YOLODetector(batch=N), always at batch N), and the crops of all N streams through ONE OSNet forward.  Tracking stays
per stream: one MultiTracker each, stepped exactly as MOT steps its own, so every stream's tracks (ids included) are
those a separate MOT would produce on that stream alone.
"""
import numpy as np

from .multicamera import MultiCameraMOT


class MultiStreamMOT(MultiCameraMOT):
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
                 embeddings_override=None,
                 pixel_format='BGR',
                 capture_size=None):
        """size: (width, height) shared by every stream; pixel_format (any of MOT's: 'BGR', 'NV12', 'I420', 'YUY2',
        'BGRX') applies to every stream.  The keyword arguments are MOT's, so the reference's
        `mot_cfg` (cfg/mot.json) passes unchanged; ssd_detector_cfg, public_detector_cfg and visualizer_cfg are
        accepted and unused, since only the YOLO detector runs several streams.  detections_override(stream,
        frame_id) and embeddings_override(stream, frame_id, detections) replace the networks' OUTPUT after both ran,
        as MOT's hooks do.  capture_size: the (width, height) every stream's frames arrive at when it differs from
        `size`, as in MOT; each frame is resized to `size` on the GPU."""
        if not (isinstance(size, (tuple, list)) and len(size) == 2 and all(np.isscalar(v) for v in size)):
            raise ValueError("MultiStreamMOT takes one frame size (width, height) shared by every stream; "
                             "streams of different sizes need MultiCameraMOT")
        self.size = tuple(int(v) for v in size)
        if num_streams < 1:
            raise ValueError("num_streams must be >= 1")
        self.num_streams = num_streams
        super().__init__([self.size] * num_streams, detector_type=detector_type,
                         detector_frame_skip=detector_frame_skip, class_ids=class_ids,
                         ssd_detector_cfg=ssd_detector_cfg, yolo_detector_cfg=yolo_detector_cfg,
                         public_detector_cfg=public_detector_cfg, feature_extractor_cfgs=feature_extractor_cfgs,
                         tracker_cfg=tracker_cfg, visualizer_cfg=visualizer_cfg, draw=draw,
                         detections_override=detections_override, embeddings_override=embeddings_override,
                         pixel_format=pixel_format, capture_size=capture_size)

    @property
    def frame_count(self):
        """Frames each stream has been stepped since the last reset."""
        return self.frame_counts[0]

    def step(self, frames):
        """One step of every stream: frames[s] is stream s's next frame, in any form MOT takes for the pixel format
        (HxWx3 u8 host array or cuda tensor for BGR)."""
        if any(f is None for f in frames):
            raise ValueError("every stream delivers a frame on every step; cameras that skip steps need "
                             "MultiCameraMOT")
        super().step(frames)
