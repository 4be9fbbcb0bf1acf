"""Detector front-end with the reference's API (fastmot/detector.py:18-42, 220-365): `Detector` ABC,
`YOLODetector(size, class_ids, model, conf_thresh, nms_thresh, max_area, min_aspect_ratio)` with
`__call__ / detect_async / postprocess`, returning `np.recarray[DET_DTYPE]` sorted by class.

Everything between the uploaded frame and the final D rows runs on the GPU: letterbox pre-processing,
the conv stack (fastmot_b200.engine), head decode fused with the score filter, DIoU-NMS.
SSDDetector / PublicDetector are out of scope (SURVEY.md §2.1 row 2).
"""
import abc
import ctypes as C

import numpy as np
import torch

from . import _lib, models
from .devmem import ptr, stream_ptr, device_frame, FrameUploader, UploadSlot
from .models.yolo import check_heads

DET_DTYPE = np.dtype(
    [('tlbr', float, 4),
     ('label', int),
     ('conf', float)],
    align=True
)


class Detector(abc.ABC):
    @abc.abstractmethod
    def __init__(self, size):
        self.size = size

    def __call__(self, frame):
        """Detect objects synchronously."""
        self.detect_async(frame)
        return self.postprocess()

    @abc.abstractmethod
    def detect_async(self, frame):
        raise NotImplementedError

    @abc.abstractmethod
    def postprocess(self):
        raise NotImplementedError


def letterbox_geometry(src_wh, dst_wh, letterbox):
    """fastmot/detector.py:302-320 -> roi (x, y, w, h) in the network input, upscaled_sz, bbox_offset."""
    src = np.array(src_wh)
    dst = np.array(dst_wh)
    if letterbox:
        scale_factor = min(dst / src)
        scaled_size = np.rint(src * scale_factor).astype(int)
        img_offset = (dst - scaled_size) / 2
        roi = (int(img_offset[0]), int(img_offset[1]), int(scaled_size[0]), int(scaled_size[1]))
        upscaled_sz = np.rint(dst / scale_factor).astype(int)
        bbox_offset = (upscaled_sz - src) / 2
    else:
        roi = (0, 0, int(dst[0]), int(dst[1]))
        upscaled_sz = src
        bbox_offset = np.zeros(2)
    return roi, upscaled_sz, bbox_offset


class YOLODetector(Detector):
    def __init__(self, size,
                 class_ids,
                 model='YOLOv4',
                 conf_thresh=0.25,
                 nms_thresh=0.5,
                 max_area=800000,
                 min_aspect_ratio=1.2,
                 max_dets=4096,
                 key_cap=16384,
                 engine=None,
                 batch=1):
        """batch = B > 1: the detector runs up to B frames per forward (detect_batch_async / postprocess_batch);
        key_cap and max_dets then hold per image.  k frames of any sizes run the engine of batch k (at k < B it shares
        the batch-B engine's weights and buffers), each frame with the letterbox and box geometry of its own size."""
        super().__init__(size)
        self._lib = _lib.require_device()
        self.model = models.YOLO.get_model(model)
        check_heads(self.model)
        assert 0 <= conf_thresh <= 1
        self.conf_thresh = conf_thresh
        assert 0 <= nms_thresh <= 1
        self.nms_thresh = nms_thresh
        assert max_area >= 0
        self.max_area = max_area
        assert min_aspect_ratio >= 0
        self.min_aspect_ratio = min_aspect_ratio

        self.label_mask = np.zeros(self.model.NUM_CLASSES, dtype=np.bool_)
        try:
            self.label_mask[tuple(class_ids),] = True
        except IndexError as err:
            raise ValueError('Unsupported class IDs') from err

        c, in_h, in_w = self.model.INPUT_SHAPE
        self.input_wh = (in_w, in_h)
        self.roi, self.upscaled_sz, self.bbox_offset = letterbox_geometry(size, self.input_wh, self.model.LETTERBOX)

        dev = torch.device("cuda")
        assert batch >= 1
        B = self.batch = batch
        self.max_dets, self.key_cap = max_dets, key_cap
        self.heads = []
        k0 = 0
        for factor, anchors, scale in zip(self.model.LAYER_FACTORS, self.model.ANCHORS, self.model.SCALES):
            h = _lib.FmYoloHead()
            for i, a in enumerate(anchors):
                h.anchors[i] = float(a)
            h.scale_x_y = float(scale)
            na = len(anchors) // 2
            self.heads.append(dict(head=h, w=in_w // factor, h=in_h // factor, na=na, base=k0))
            k0 += na * (in_w // factor) * (in_h // factor)
        self.num_candidates = k0
        self._label_mask_dev = torch.as_tensor(self.label_mask.astype(np.uint8)).to(dev)
        # image b owns rows [b k0, (b + 1) k0) of the candidate table, keys [b key_cap, (b + 1) key_cap), one mask
        # segment and output rows [b max_dets, (b + 1) max_dets)
        self._dense = torch.zeros(B * k0, 8, dtype=torch.float32, device=dev)
        self._keys = torch.zeros(B * key_cap, dtype=torch.int64, device=dev)
        self._counter = torch.zeros(B, dtype=torch.int32, device=dev)
        self._mask = torch.zeros(B * int(self._lib.fm_nms_mask_bytes(key_cap)), dtype=torch.uint8, device=dev)
        # outputs packed in one block -> one D2H
        self._out_tlbr = torch.zeros(B * max_dets, 4, dtype=torch.float64, device=dev)
        self._out_label = torch.zeros(B * max_dets, dtype=torch.int64, device=dev)
        self._out_conf = torch.zeros(B * max_dets, dtype=torch.float64, device=dev)
        # [count, status, n_candidates, -] (batch: [count[B], status[B], n_candidates[B]])
        self._out_meta = torch.zeros(max(4, 3 * B), dtype=torch.int32, device=dev)
        self._h_tlbr = torch.zeros(B * max_dets, 4, dtype=torch.float64).pin_memory()
        self._h_label = torch.zeros(B * max_dets, dtype=torch.int64).pin_memory()
        self._h_conf = torch.zeros(B * max_dets, dtype=torch.float64).pin_memory()
        self._h_meta = torch.zeros(max(4, 3 * B), dtype=torch.int32).pin_memory()
        lead = () if B == 1 else (B,)
        self.inp = torch.zeros(lead + (in_h, in_w, 8), dtype=torch.float16, device=dev)   # NHWC8
        # host frames of image b go through slot b
        self._uploads = [UploadSlot(FrameUploader(size))] + [UploadSlot() for _ in range(B - 1)]
        # per-frame geometry of detect_batch_async (one FmFrameGeom row per image)
        self._geom_bytes = C.sizeof(_lib.FmFrameGeom)
        self._geom_h = torch.zeros(B * self._geom_bytes, dtype=torch.uint8).pin_memory()
        self._geom = torch.zeros(B * self._geom_bytes, dtype=torch.uint8, device=dev)
        self._geom_ev = None
        self._geometry = {tuple(size): (self.roi, self.upscaled_sz, self.bbox_offset)}
        self._k = B                 # images of the last detect_batch_async
        self.frame_dev = None
        self._done = torch.cuda.Event()
        if engine is None:
            from .engine import build_yolo_engine
            engine = build_yolo_engine(self.model, batch=B)
        if getattr(engine, 'batch', 1) != B:
            raise ValueError(f"the engine runs {getattr(engine, 'batch', 1)} images per forward, the detector {B}")
        if getattr(engine, 'head_shapes', None) is not None:
            check_heads(self.model, engine.head_shapes)
        self.backend = engine
        self._engines = {B: engine}     # batch k -> engine; k < B share the batch-B engine's resources

    # ------------------------------------------------------------------
    def preprocess(self, frame_dev):
        """fastmot/detector.py:289-300 on the device (frame_dev: HxWx3 u8 cuda tensor, or a device Frame of this
        detector's size: a frame of any pixel format is read in place)."""
        f = device_frame(frame_dev, size=self.size)
        rx, ry, rw, rh = self.roi
        rc = self._lib.fm_letterbox_preproc(C.byref(f.fm()), self.input_wh[0], self.input_wh[1], rx, ry, rw, rh, 1,
                                            ptr(self.inp), stream_ptr())
        _lib.check(rc, "fm_letterbox_preproc")

    def detect_async(self, frame):
        """Upload (if `frame` is a host array or a host Frame), pre-process, run the conv stack and the whole
        post-processing asynchronously; `postprocess` waits for the D result rows."""
        self.frame_dev = device_frame(frame, self._uploads[0])
        self.preprocess(self.frame_dev)
        heads = self.backend.forward(self.inp)
        self.postprocess_heads_async(heads)

    def postprocess_heads_async(self, head_tensors):
        """Decode + filter + NMS for raw head tensors [(5+C)*A, H, W] (fp16 or fp32)."""
        s = stream_ptr()
        self._counter.zero_()
        lib = self._lib
        for hd, t in zip(self.heads, head_tensors):
            assert t.is_contiguous()
            nhwc = 1 if getattr(self.backend, "heads_nhwc", False) else 0
            rc = lib.fm_yolo_decode_filter(ptr(t), 1 if t.dtype == torch.float16 else 0, nhwc, hd['w'], hd['h'],
                                           hd['na'],
                                           C.byref(hd['head']), self.model.NUM_CLASSES, self.input_wh[0],
                                           self.input_wh[1], 1 if self.model.NEW_COORDS else 0, hd['base'],
                                           ptr(self._label_mask_dev), float(self.conf_thresh),
                                           float(self.upscaled_sz[0]), float(self.upscaled_sz[1]),
                                           float(self.bbox_offset[0]), float(self.bbox_offset[1]),
                                           ptr(self._dense), ptr(self._keys), ptr(self._counter), self.key_cap, s)
            _lib.check(rc, "fm_yolo_decode_filter")
        meta = self._out_meta
        rc = lib.fm_diou_nms_filter(ptr(self._keys), ptr(self._dense), ptr(self._counter), self.key_cap,
                                    float(self.nms_thresh), float(self.max_area), float(self.min_aspect_ratio),
                                    ptr(self._mask), self.max_dets, ptr(self._out_tlbr), ptr(self._out_label),
                                    ptr(self._out_conf), C.c_void_p(meta.data_ptr()),
                                    C.c_void_p(meta.data_ptr() + 4), s)
        _lib.check(rc, "fm_diou_nms_filter")
        lib.fm_memcpy_async(C.c_void_p(meta.data_ptr() + 8), ptr(self._counter), 4, s)
        self._h_meta.copy_(meta, non_blocking=True)
        self._h_tlbr.copy_(self._out_tlbr, non_blocking=True)
        self._h_label.copy_(self._out_label, non_blocking=True)
        self._h_conf.copy_(self._out_conf, non_blocking=True)
        self._done.record()

    def postprocess(self):
        """Waits for the async pipeline and returns np.recarray[DET_DTYPE] (class asc, objectness desc)."""
        self._done.synchronize()
        n, status, n_cand = (int(v) for v in self._h_meta[:3])
        dets = self._image_dets(n, status, n_cand, 0)
        self.last_num_candidates = n_cand
        return dets

    def _image_dets(self, n, status, n_cand, row0, name=None):
        """One image's n detections, rows [row0, row0 + n) of the host outputs, as np.recarray[DET_DTYPE].  Its NMS
        status raises on an overflow; the message starts with `name` when one is given."""
        prefix = "" if name is None else f"{name}: "
        if status == 2:
            raise RuntimeError(f"{prefix}more than max_dets = {self.max_dets} boxes survived NMS and the area / aspect "
                               "filters; raise max_dets (no silent truncation)")
        if status != 0:
            raise RuntimeError(f"{prefix}{n_cand} candidates passed conf_thresh but key_cap is {self.key_cap}; "
                               "raise key_cap (no silent truncation)")
        dets = np.zeros(n, DET_DTYPE)
        dets['tlbr'] = self._h_tlbr.numpy()[row0:row0 + n]
        dets['label'] = self._h_label.numpy()[row0:row0 + n]
        dets['conf'] = self._h_conf.numpy()[row0:row0 + n]
        return dets.view(np.recarray)

    # ------------------------------------------------------------------ batch > 1
    def detect_batch_async(self, frames):
        """detect_async for 1..B frames (HxWx3 u8 of any sizes, or Frames of any sizes and formats) at once: one
        letterbox launch, one forward of the batch-k engine, one decode launch per head and one batched NMS;
        `postprocess_batch` waits for the results.  Each frame gets the letterbox and box geometry of its own size."""
        k = len(frames)
        if not 1 <= k <= self.batch:
            raise ValueError(f"expected 1 to {self.batch} frames, got {k}")
        self.frames_dev = [device_frame(f, up) for f, up in zip(frames, self._uploads)]
        geom = self.preprocess_frames(self.frames_dev)
        # a batch-1 input has no image dimension, in this detector and in its batch-1 engine
        inp = self.inp if self.batch == 1 else self.inp[:k] if k > 1 else self.inp[0]
        heads = self.engine(k).forward(inp)
        self.postprocess_heads_batch_async(heads, k, geom)

    def engine(self, k):
        """The conv stack at batch k (1 <= k <= B); k < B is built on first use and shares the batch-B engine's
        weights, workspace and buffers (YoloEngine.with_batch)."""
        if k not in self._engines:
            if not 1 <= k < self.batch:
                raise ValueError(f"batch {k} is outside 1..{self.batch}")
            self._engines[k] = self.backend.with_batch(k)
        return self._engines[k]

    def build_engines(self):
        """Builds the engines of every batch 1..B now rather than on first use."""
        for k in range(1, self.batch + 1):
            self.engine(k)

    def geometry(self, wh):
        """(roi, upscaled_sz, bbox_offset) of frames of size wh = (width, height) in this detector's input."""
        wh = tuple(int(v) for v in wh)
        if wh not in self._geometry:
            self._geometry[wh] = letterbox_geometry(wh, self.input_wh, self.model.LETTERBOX)
        return self._geometry[wh]

    def _upload_geom(self, sizes, frames=None):
        """Fills one FmFrameGeom row per image, of frame size sizes[b] = (width, height) and device Frame frames[b]
        (no frame fields when frames is None: only the head decode reads the rows), and uploads the rows to
        self._geom in one copy from the pinned block; returns self._geom."""
        rows = (_lib.FmFrameGeom * len(sizes))()
        for b, (r, (w, h)) in enumerate(zip(rows, sizes)):
            (rx, ry, rw, rh), up, off = self.geometry((w, h))
            if frames is not None:
                r.frame = frames[b].fm()
            r.roi_x, r.roi_y, r.roi_w, r.roi_h = rx, ry, rw, rh
            r.size_w, r.size_h, r.off_x, r.off_y = float(up[0]), float(up[1]), float(off[0]), float(off[1])
        if self._geom_ev is not None:
            self._geom_ev.synchronize()          # the previous table upload has left the pinned block
        nb = len(sizes) * self._geom_bytes
        C.memmove(self._geom_h.data_ptr(), C.addressof(rows), nb)
        self._geom[:nb].copy_(self._geom_h[:nb], non_blocking=True)
        self._geom_ev = torch.cuda.Event()
        self._geom_ev.record()
        return self._geom

    def preprocess_frames(self, frames_dev):
        """Letterbox of k frames of any sizes (HxWx3 u8 cuda tensors, or device Frames of either format) into
        self.inp[:k], one launch.  Uploads their FmFrameGeom table and returns it: the head decode reads it too."""
        k = len(frames_dev)
        if not 1 <= k <= self.batch:
            raise ValueError(f"expected 1 to {self.batch} frames, got {k}")
        frames = [device_frame(f) for f in frames_dev]
        geom = self._upload_geom([f.size for f in frames], frames)
        rc = self._lib.fm_letterbox_preproc_geom(ptr(geom), k, self.input_wh[0], self.input_wh[1], ptr(self.inp),
                                                 stream_ptr())
        _lib.check(rc, "fm_letterbox_preproc_geom")
        return geom

    def postprocess_heads_batch_async(self, head_tensors, k=None, geom=None):
        """Decode + filter + NMS of k (default B) images' fp16 NHWC heads [k][H][W][(5+C)*A] ([H][W][(5+C)*A] at
        k = 1).  geom: the device FmFrameGeom table of preprocess_frames (each image's own box geometry); without it
        every image has this detector's size, and k rows of that size are uploaded."""
        s = stream_ptr()
        B, k0 = self.batch, self.num_candidates
        k = B if k is None else k
        if geom is None:
            geom = self._upload_geom([self.size] * k)
        self._k = k
        self._counter.zero_()
        lib = self._lib
        for hd, t in zip(self.heads, head_tensors):
            assert t.is_contiguous() and t.dtype == torch.float16 and t.numel() % k == 0
            rc = lib.fm_yolo_decode_filter_geom(ptr(t), k, t.numel() // k, 1, 1, hd['w'], hd['h'], hd['na'],
                                                C.byref(hd['head']), self.model.NUM_CLASSES, self.input_wh[0],
                                                self.input_wh[1], 1 if self.model.NEW_COORDS else 0, hd['base'], k0,
                                                ptr(self._label_mask_dev), float(self.conf_thresh), ptr(geom),
                                                ptr(self._dense), ptr(self._keys), ptr(self._counter), self.key_cap, s)
            _lib.check(rc, "fm_yolo_decode_filter_geom")
        meta = self._out_meta
        rc = lib.fm_diou_nms_filter_batch(k, ptr(self._keys), ptr(self._dense), k0, ptr(self._counter), self.key_cap,
                                          float(self.nms_thresh), float(self.max_area), float(self.min_aspect_ratio),
                                          ptr(self._mask), self.max_dets, ptr(self._out_tlbr), ptr(self._out_label),
                                          ptr(self._out_conf), ptr(meta[:k]), ptr(meta[B:B + k]), s)
        _lib.check(rc, "fm_diou_nms_filter_batch")
        lib.fm_memcpy_async(ptr(meta[2 * B:2 * B + k]), ptr(self._counter), 4 * k, s)
        self._h_meta.copy_(meta, non_blocking=True)
        self._h_tlbr.copy_(self._out_tlbr, non_blocking=True)
        self._h_label.copy_(self._out_label, non_blocking=True)
        self._h_conf.copy_(self._out_conf, non_blocking=True)
        self._done.record()

    def postprocess_batch(self, names=None):
        """Waits for detect_batch_async; returns a list of k np.recarray[DET_DTYPE], one per frame, each ordered as
        `postprocess` orders one frame's detections.  An overflow raises and names image b as names[b] (default
        'image b')."""
        self._done.synchronize()
        B, k = self.batch, self._k
        count, status, n_cand = (self._h_meta.numpy()[i * B:i * B + k].tolist() for i in range(3))
        out = [self._image_dets(count[b], status[b], n_cand[b], b * self.max_dets,
                                f"image {b}" if names is None else names[b]) for b in range(k)]
        self.last_num_candidates = n_cand
        return out


class PublicDetector(Detector):
    """MOT Challenge public detections (`det/det.txt` of a sequence directory) served at the detector cadence —
    the reference's `PublicDetector` (fastmot/detector.py:368-431).  A file reader, not a kernel: it runs on the
    host exactly as in the reference; everything downstream of it (ReID crops, OSNet, tracker) is the GPU path.

    Row format: frame (1-based), id, left, top, width, height, conf, ... .  Each box is rounded with `to_tlbr`
    (half-to-even on x, y, x+w-1, y+h-1), scaled from the sequence resolution (`seqinfo.ini`) to `size`, rounded
    again, and kept if `area <= max_area`; confidences are forced to 1.0 and labels to 1 (person), as in the
    reference.  `sequence_path` may be absolute or relative to the working directory (the reference resolves it
    against its repository root).
    """

    def __init__(self, size, class_ids, frame_skip, sequence_path=None, conf_thresh=0.5, max_area=800000):
        super().__init__(size)
        import configparser
        from collections import defaultdict
        from pathlib import Path
        assert tuple(class_ids) == (1,)
        self.frame_skip = frame_skip
        assert sequence_path is not None
        self.seq_root = Path(sequence_path)
        assert 0 <= conf_thresh <= 1
        self.conf_thresh = conf_thresh
        assert max_area >= 0
        self.max_area = max_area
        assert self.seq_root.exists()
        seqinfo = configparser.ConfigParser()
        seqinfo.read(self.seq_root / 'seqinfo.ini')
        self.seq_size = (int(seqinfo['Sequence']['imWidth']), int(seqinfo['Sequence']['imHeight']))
        self.detections = defaultdict(list)
        self.frame_id = 0
        rows = np.atleast_2d(np.loadtxt(self.seq_root / 'det' / 'det.txt', delimiter=','))
        seq_wh = np.asarray(self.seq_size, np.float64)
        dst_wh = np.asarray(self.size, np.float64)
        for row in rows:
            if row.size < 6:
                continue
            frame_id = int(row[0]) - 1
            x, y, w, h = row[2:6]
            tlbr = np.rint(np.array([x, y, x + w - 1., y + h - 1.]))       # to_tlbr, rect.py:48-57
            tlbr[:2] = tlbr[:2] / seq_wh * dst_wh
            tlbr[2:] = tlbr[2:] / seq_wh * dst_wh
            tlbr = np.rint(tlbr)
            bw, bh = tlbr[2] - tlbr[0] + 1., tlbr[3] - tlbr[1] + 1.
            box_area = 0. if bw <= 0 or bh <= 0 else bw * bh                 # rect.py:27-32
            conf, label = 1.0, 1
            if conf >= self.conf_thresh and box_area <= self.max_area:
                self.detections[frame_id].append((tlbr, label, conf))

    def detect_async(self, frame):
        pass

    def postprocess(self):
        detections = np.array(self.detections[self.frame_id], DET_DTYPE).view(np.recarray)
        self.frame_id += self.frame_skip
        return detections
