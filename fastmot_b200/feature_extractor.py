"""ReID feature extractor with the reference's API (fastmot/feature_extractor.py:11-98):
`FeatureExtractor(model, batch_size)`, `extract_async(frame, tlbrs)`, `postprocess() -> (N, 512)` unit-norm rows,
`__call__`, `metric`, `null_embeddings`.

All crops of a frame are pre-processed by one kernel launch straight from the device-resident frame (the reference
crops + cv2.resize's on CPU threads and uploads 16 crops at a time) and run through the OSNet engine in one batch;
the embeddings stay on the GPU (`DeviceEmbeddings`) and feed the association kernels directly.  The reference's
aliasing defect for > batch_size crops (SURVEY.md Appendix A) is not reproduced.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, models
from .devmem import ptr, stream_ptr, device_frame, UploadSlot
from .tracker import DeviceEmbeddings


class FeatureExtractor:
    def __init__(self, model='OSNet025', batch_size=16, max_crops=512, size=(1920, 1080), use_tc=True,
                 use_graph=True):
        self._lib = _lib.require_device()
        self.model = models.ReID.get_model(model)
        assert batch_size >= 1
        self.batch_size = batch_size
        self.feature_dim = self.model.OUTPUT_LAYOUT
        self.max_crops = max_crops
        self.size = size
        self._use_tc, self._use_graph = use_tc, use_graph
        self._engines = {}
        dev = torch.device("cuda")
        self._tlbr_dev = torch.zeros(max_crops, 4, dtype=torch.float64, device=dev)
        self._tlbr_host = torch.zeros(max_crops, 4, dtype=torch.float64).pin_memory()
        self._upload = UploadSlot()
        self.last_num_features = 0
        self._out = None
        self._splits = None         # per-stream crop offsets of the last extract_multi_async
        self._frame_idx_host = torch.zeros(max_crops, dtype=torch.int32).pin_memory()
        self._frame_idx_dev = torch.zeros(max_crops, dtype=torch.int32, device=dev)
        self._geom_host = self._geom_dev = None     # FmFrameGeom rows of extract_multi_async's frames
        self._geom_ev = None

    def _engine(self, n):
        """Engines are planned per batch bucket (multiples of 8 crops): a frame pays for its own crops, not for
        max_crops."""
        from .engine import build_reid_engine
        b = max(8, -(-n // 8) * 8)
        if b not in self._engines:
            self._engines[b] = build_reid_engine(self.model, max_batch=b, use_tc=self._use_tc,
                                                 use_graph=self._use_graph)
        return self._engines[b]

    def __call__(self, frame, tlbrs):
        self.extract_async(frame, tlbrs)
        return self.postprocess()

    @property
    def metric(self):
        return self.model.METRIC

    def extract_async(self, frame, tlbrs):
        """frame: HxWx3 u8 host array or cuda tensor, or a Frame (of any pixel format, read in place); tlbrs: (N,4)."""
        tlbrs = np.ascontiguousarray(tlbrs, np.float64).reshape(-1, 4)
        n = len(tlbrs)
        self.last_num_features = n
        self._out = None
        self._splits = None
        if n == 0:
            return
        if n > self.max_crops:
            raise MemoryError(f"{n} crops > max_crops {self.max_crops}")
        frame_dev = device_frame(frame, self._upload)
        eng = self._engine(n)
        self._tlbr_host[:n] = torch.as_tensor(tlbrs)
        self._tlbr_dev[:n].copy_(self._tlbr_host[:n], non_blocking=True)
        c, ih, iw = self.model.INPUT_SHAPE
        rc = self._lib.fm_roi_resize_norm(C.byref(frame_dev.fm()), ptr(self._tlbr_dev), None, n, iw, ih, eng.inp_layout,
                                          ptr(eng.inp), stream_ptr())
        _lib.check(rc, "fm_roi_resize_norm")
        self._out = eng.forward(n)

    def extract_multi_async(self, frames, tlbrs_per_stream):
        """extract_async over several streams at once: frames[s] (HxWx3 u8 cuda tensors or device Frames of either
        format, each of its own size) with
        its boxes tlbrs_per_stream[s].  All crops are cut in one launch, each clamped to its own frame, and run through
        one OSNet forward (the batch buckets of extract_async hold the sum over streams); `postprocess` then returns
        one slice per stream."""
        if len(frames) != len(tlbrs_per_stream):
            raise ValueError("one box array per frame")
        tl = [np.ascontiguousarray(t, np.float64).reshape(-1, 4) for t in tlbrs_per_stream]
        counts = [len(t) for t in tl]
        n = sum(counts)
        self.last_num_features = n
        self._out = None
        self._splits = np.concatenate([[0], np.cumsum(counts)]).astype(int)
        if n == 0:
            return
        if n > self.max_crops:
            raise MemoryError(f"{n} crops > max_crops {self.max_crops}")
        rows = (_lib.FmFrameGeom * len(frames))()
        for r, f in zip(rows, frames):
            r.frame = device_frame(f).fm()
        nb = C.sizeof(rows)
        if self._geom_host is None or self._geom_host.numel() < nb:
            if self._geom_ev is not None:
                self._geom_ev.synchronize()
            self._geom_host = torch.zeros(nb, dtype=torch.uint8).pin_memory()
            self._geom_dev = torch.zeros(nb, dtype=torch.uint8, device=self._frame_idx_dev.device)
            self._geom_ev = None
        eng = self._engine(n)
        self._tlbr_host[:n] = torch.as_tensor(np.concatenate(tl))
        self._tlbr_dev[:n].copy_(self._tlbr_host[:n], non_blocking=True)
        self._frame_idx_host[:n] = torch.as_tensor(np.repeat(np.arange(len(frames), dtype=np.int32), counts))
        self._frame_idx_dev[:n].copy_(self._frame_idx_host[:n], non_blocking=True)
        if self._geom_ev is not None:
            self._geom_ev.synchronize()          # the previous table upload has left the pinned block
        C.memmove(self._geom_host.data_ptr(), C.addressof(rows), nb)
        self._geom_dev[:nb].copy_(self._geom_host[:nb], non_blocking=True)
        self._geom_ev = torch.cuda.Event()
        self._geom_ev.record()
        c, ih, iw = self.model.INPUT_SHAPE
        rc = self._lib.fm_roi_resize_norm_geom(ptr(self._geom_dev), ptr(self._frame_idx_dev), ptr(self._tlbr_dev), n,
                                               iw, ih, eng.inp_layout, ptr(eng.inp), stream_ptr())
        _lib.check(rc, "fm_roi_resize_norm_geom")
        self._out = eng.forward(n)

    def postprocess(self):
        """Returns DeviceEmbeddings (N, feature_dim) — numpy-convertible, rows L2-normalised.  After
        extract_multi_async: a list with one entry per stream, each a view of that stream's rows of the shared
        output (no copy)."""
        if self._splits is not None:
            sp = self._splits
            return [DeviceEmbeddings(self._out[a:b]) if b > a else np.empty((0, self.feature_dim))
                    for a, b in zip(sp[:-1], sp[1:])]
        if self.last_num_features == 0:
            return np.empty((0, self.feature_dim))
        return DeviceEmbeddings(self._out)

    def null_embeddings(self, detections):
        embeddings = np.ones((len(detections), self.feature_dim))
        embeddings /= np.linalg.norm(embeddings, axis=1, keepdims=True)
        return embeddings
