"""GPU parity: detector pre/post-processing kernels (csrc/preproc.cu, csrc/detect.cu) vs the reference golden
and the oracle.  Box/label lists bit-exact for new_coords heads and for the NMS stage; old-coords heads use
__expf so boxes may move by <= 1 px at rounding boundaries."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu


class _NoEngine:
    def forward(self, x):
        raise RuntimeError("no conv engine in this test")


def _make_heads(model, rng, obj_bias):
    """Synthetic raw head tensors [(5+C)*A, H, W] fp32 with sparse objectness."""
    c, H, W = model.INPUT_SHAPE
    heads = []
    for factor, anchors in zip(model.LAYER_FACTORS, model.ANCHORS):
        A = len(anchors) // 2
        h, w = H // factor, W // factor
        t = rng.normal(0, 1, (A, 5 + model.NUM_CLASSES, h, w)).astype(np.float32)
        if model.NEW_COORDS:
            t = 1 / (1 + np.exp(-t))                       # logistic-activated conv outputs
            t[:, 4] = 1 / (1 + np.exp(-(rng.normal(0, 1.5, (A, h, w)) + obj_bias)))
            t[:, 2:4] *= 1.2
        else:
            t[:, 4] = rng.normal(0, 1.5, (A, h, w)) + obj_bias
            t[:, 2:4] *= 0.4
        heads.append(np.ascontiguousarray(t.reshape(A * (5 + model.NUM_CLASSES), h, w).astype(np.float32)))
    return heads


@pytest.mark.parametrize("name,obj_bias", [("YOLOv4CSP", -3.0), ("YOLOv4Tiny", -2.0), ("YOLOv4P5", -4.0),
                                            ("YOLOv4", -3.0)])
def test_decode_filter_nms_vs_oracle(name, obj_bias):
    from fastmot_b200.detector import YOLODetector
    from fastmot_b200 import models
    from oracle import detect
    model = models.YOLO.get_model(name)
    class_ids = (0,) if model.NUM_CLASSES == 1 else (0, 1)
    det = YOLODetector((1920, 1080), class_ids, name, min_aspect_ratio=0.3, engine=_NoEngine())
    rng = np.random.default_rng(4)
    heads = _make_heads(model, rng, obj_bias)
    dec = [detect.yolo_decode(h, a, s, det.input_wh, model.NUM_CLASSES, model.NEW_COORDS)
           for h, a, s in zip(heads, model.ANCHORS, model.SCALES)]
    want = detect.filter_dets(np.concatenate(dec), det.upscaled_sz, det.bbox_offset, det.label_mask, 0.25, 0.5,
                              800000, 0.3)
    for dtype in (torch.float32,):
        dev_heads = [torch.as_tensor(h).to("cuda").to(dtype).contiguous() for h in heads]
        det.postprocess_heads_async(dev_heads)
        got = det.postprocess()
        assert 50 < len(want[0]) < 4000, len(want[0])
        if model.NEW_COORDS:
            assert len(got) == len(want[0])
            assert np.array_equal(got.tlbr, want[0])
            assert np.array_equal(got.label, want[1])
            np.testing.assert_allclose(got.conf, want[2], atol=1e-7)
        else:
            assert abs(len(got) - len(want[0])) <= max(2, len(want[0]) // 200)
            if len(got) == len(want[0]):
                assert np.abs(got.tlbr - want[0]).max() <= 1.0
                np.testing.assert_allclose(got.conf, want[2], atol=1e-4)


def test_nms_stage_against_reference_golden():
    """sort + DIoU-NMS + rounding + filters fed with the golden's decoded candidates (bit-exact)."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.load()
    g = np.load(os.path.join(GOLDEN, "detect_filter.npz"))
    for k in range(int(g['n'])):
        det = g[f'det_{k}']
        size, off, lm = g[f'size_{k}'].astype(np.float64), g[f'off_{k}'], g[f'lm_{k}']
        score = (det[:, 4] * det[:, 6]).astype(np.float32)
        keep = np.nonzero(lm[det[:, 5].astype(int)] & (score.astype(np.float64) >= 0.25))[0]
        d = det.copy()
        d[:, :4] = (d[:, :4].astype(np.float64) * np.concatenate([size, size])).astype(np.float32)
        d[:, :2] = (d[:, :2].astype(np.float64) - off).astype(np.float32)
        dense = np.zeros((len(det), 8), np.float32)
        dense[:, :7] = d
        bits = (~d[keep, 4].view(np.uint32)).astype(np.uint64)
        keys = (d[keep, 5].astype(np.uint64) << np.uint64(56)) | (bits << np.uint64(24)) | keep.astype(np.uint64)
        cap = 16384
        keys_d = torch.zeros(cap, dtype=torch.int64, device="cuda")
        keys_d[:len(keys)] = torch.as_tensor(keys.view(np.int64)).to("cuda")
        dense_d = torch.as_tensor(dense).to("cuda")
        counter = torch.tensor([len(keys)], dtype=torch.int32, device="cuda")
        mask = torch.zeros(int(lib.fm_nms_mask_bytes(cap)), dtype=torch.uint8, device="cuda")
        o_t = torch.zeros(4096, 4, dtype=torch.float64, device="cuda")
        o_l = torch.zeros(4096, dtype=torch.int64, device="cuda")
        o_c = torch.zeros(4096, dtype=torch.float64, device="cuda")
        meta = torch.zeros(2, dtype=torch.int32, device="cuda")
        import ctypes as C
        rc = lib.fm_diou_nms_filter(ptr(keys_d), ptr(dense_d), ptr(counter), cap, 0.5, 800000.0, 1.2, ptr(mask), 4096,
                                    ptr(o_t), ptr(o_l), ptr(o_c), C.c_void_p(meta.data_ptr()),
                                    C.c_void_p(meta.data_ptr() + 4), stream_ptr())
        _lib.check(rc, "nms")
        torch.cuda.synchronize()
        n, st = meta.cpu().numpy().tolist()
        assert st == 0
        assert n == len(g[f'tlbr_{k}'])
        assert np.array_equal(o_t.cpu().numpy()[:n], g[f'tlbr_{k}'])
        assert np.array_equal(o_l.cpu().numpy()[:n], g[f'label_{k}'])
        np.testing.assert_allclose(o_c.cpu().numpy()[:n], g[f'conf_{k}'], atol=1e-7)


def test_key_overflow_is_reported():
    from fastmot_b200.detector import YOLODetector
    from fastmot_b200 import models
    model = models.YOLO.get_model("YOLOv4CSP")
    det = YOLODetector((1920, 1080), (0,), "YOLOv4CSP", engine=_NoEngine(), key_cap=256)
    heads = _make_heads(model, np.random.default_rng(0), 2.0)
    det.postprocess_heads_async([torch.as_tensor(h).to("cuda") for h in heads])
    with pytest.raises(RuntimeError):
        det.postprocess()


def test_empty_detections():
    from fastmot_b200.detector import YOLODetector
    from fastmot_b200 import models
    model = models.YOLO.get_model("YOLOv4CSP")
    det = YOLODetector((1920, 1080), (0,), "YOLOv4CSP", engine=_NoEngine())
    heads = [np.zeros_like(h) for h in _make_heads(model, np.random.default_rng(0), 0.0)]
    det.postprocess_heads_async([torch.as_tensor(h).to("cuda") for h in heads])
    out = det.postprocess()
    assert len(out) == 0 and out.tlbr.shape == (0, 4)


@pytest.mark.parametrize("model_name", ["YOLOv4CSP", "YOLOv4Tiny"])
def test_letterbox_preproc_fmframe(model_name):
    from fastmot_b200 import _lib, models
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    from fastmot_b200.synth import SyntheticScene
    from oracle import detect
    lib = _lib.load()
    model = models.YOLO.get_model(model_name)
    _, H, W = model.INPUT_SHAPE
    frame = SyntheticScene(30, seed=2).frame(1)
    roi, _, _ = detect.letterbox_geometry((1920, 1080), (W, H), model.LETTERBOX)
    want = detect.letterbox(frame, (W, H), roi)
    fr = Frame.bgr(torch.as_tensor(frame).to("cuda"))
    fd = C.byref(fr.fm())
    out32 = torch.zeros(3, H, W, dtype=torch.float32, device="cuda")
    _lib.check(lib.fm_letterbox_preproc(fd, W, H, *roi, 0, ptr(out32), stream_ptr()), "lb")
    got = out32.cpu().numpy()
    diff = np.abs(got - want) * 255
    assert diff.max() <= 1.0 + 1e-3            # reference semantics pinned only to +-1 LSB (CuPy absent)
    assert (diff < 1e-3).mean() > 0.999
    out16 = torch.zeros(H, W, 8, dtype=torch.float16, device="cuda")
    _lib.check(lib.fm_letterbox_preproc(fd, W, H, *roi, 1, ptr(out16), stream_ptr()), "lb")
    g16 = out16.cpu().float().numpy()
    assert np.abs(g16[..., :3].transpose(2, 0, 1) - got).max() <= 1e-3
    assert np.all(g16[..., 3:] == 0)


def test_roi_resize_norm_fmframe():
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    from fastmot_b200.synth import SyntheticScene
    from oracle import detect
    lib = _lib.load()
    sc = SyntheticScene(60, seed=1)
    frame = sc.frame(0)
    tl = sc.detections(0)[0]
    tl = np.concatenate([tl, [[-5.5, 10.2, 40.7, 90.9], [1890, 1000, 1950, 1100], [100, 100, 400, 700]]])
    want = detect.roi_preprocess(frame, tl)                  # cv2.resize path of the reference
    fr = Frame.bgr(torch.as_tensor(frame).to("cuda"))
    fd = C.byref(fr.fm())
    td = torch.as_tensor(np.ascontiguousarray(tl, np.float64)).to("cuda")
    n = len(tl)
    out = torch.zeros(n, 3, 256, 128, dtype=torch.float32, device="cuda")
    ncnt = torch.tensor([n], dtype=torch.int32, device="cuda")
    _lib.check(lib.fm_roi_resize_norm(fd, ptr(td), ptr(ncnt), n + 5, 128, 256, 0, ptr(out), stream_ptr()), "roi")
    got = out.cpu().numpy()
    std = np.array([0.229, 0.224, 0.225])[None, :, None, None]
    lsb = np.abs(got - want) * 255 * std
    assert lsb.max() <= 1.0 + 1e-2
    assert (lsb < 1e-2).mean() > 0.99
    exact = detect.roi_preprocess_fixedpoint(frame, tl)      # the formula the kernel implements
    np.testing.assert_allclose(got, exact, atol=2e-6)
    out16 = torch.zeros(n, 256, 128, 8, dtype=torch.float16, device="cuda")
    _lib.check(lib.fm_roi_resize_norm(fd, ptr(td), None, n, 128, 256, 1, ptr(out16), stream_ptr()), "roi")
    g16 = out16.cpu().float().numpy()[..., :3].transpose(0, 3, 1, 2)
    assert np.abs(g16 - got).max() <= 2e-3
