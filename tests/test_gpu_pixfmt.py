"""GPU: I420, YUY2 and BGRx frames read in place by the letterbox, crop, KLT gray and frame-resize kernels, and tracked
end to end.

Frames are SyntheticScene frames encoded with cv2 (oracle/pixfmt.py; BGRx with a fourth byte that is not zero).  The
reference is always the BGR path fed the cv2 decode (cv2.cvtColor with COLOR_YUV2BGR_I420, _YUY2 or COLOR_BGRA2BGR);
every comparison is bit for bit.  Each kernel check runs on two device forms of the same frame: tight, and pitched
(I420: three planes in padded surfaces, filled with 255 outside the frame; YUY2 and BGRx: rows of W + 64 pixels).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from test_gpu_multistream import _boxes
from test_gpu_nv12 import SIZES, _bits_equal, _dets_fn, _geom_table, _nets_kw, _scene_bgr, _synth_env
from test_gpu_nv12 import _device_form as _nv12_device_form

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

FMTS = ["I420", "YUY2", "BGRX"]
FORMS = {"I420": ["tight", "planes"], "YUY2": ["tight", "pitched"], "BGRX": ["tight", "pitched"]}
CASES = [(f, form) for f in FMTS for form in FORMS[f]]
CASE_IDS = [f"{f}-{form}" for f, form in CASES]


def _encode(bgr, fmt):
    from oracle import pixfmt
    from oracle.nv12 import bgr_to_nv12
    if fmt == "BGR":
        return bgr
    if fmt == "NV12":
        return bgr_to_nv12(bgr)
    if fmt == "BGRX":
        return pixfmt.bgr_to_bgrx(bgr, x=173)
    return pixfmt.DECODES[fmt][2](bgr)


def _raw_pair(fmt, size, seed=3, t=2):
    """(raw host frame in fmt, its cv2 BGR decode)."""
    from oracle.pixfmt import cv2_decode
    raw = _encode(_scene_bgr(size, seed, t), fmt)
    return raw, cv2_decode(raw, fmt)


def _device_form(raw, fmt, form):
    """The host frame `raw` of format fmt on the device in one of FORMS[fmt] (what devmem.pixel_frame accepts)."""
    t = torch.as_tensor(raw)
    if fmt == "NV12":
        return _nv12_device_form(raw, form)
    if fmt == "BGR" or form == "tight":
        return t.cuda()
    if fmt == "I420":
        h, w = raw.shape[0] * 2 // 3, raw.shape[1]
        q = h * w // 4
        c = t[h:].reshape(-1)
        ys = torch.full((h + 16, w + 64), 255, dtype=torch.uint8, device="cuda")
        cs = torch.full((2, h // 2 + 8, w // 2 + 32), 255, dtype=torch.uint8, device="cuda")
        ys[:h, :w] = t[:h].cuda()
        cs[0, :h // 2, :w // 2] = c[:q].view(h // 2, w // 2).cuda()
        cs[1, :h // 2, :w // 2] = c[q:].view(h // 2, w // 2).cuda()
        return ys[:h, :w], cs[0, :h // 2, :w // 2], cs[1, :h // 2, :w // 2]
    h, w, ch = raw.shape
    surf = torch.full((h, w + 64, ch), 255, dtype=torch.uint8, device="cuda")
    surf[:, :w] = t.cuda()
    return surf[:, :w]


def _frame(raw, fmt, form):
    from fastmot_b200.devmem import pixel_frame
    return pixel_frame(_device_form(raw, fmt, form), fmt)


def _bgr_frame(bgr):
    from fastmot_b200.devmem import Frame
    return Frame.bgr(torch.as_tensor(bgr).cuda())


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("fmt, form", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("model", ["YOLOv4Tiny", "YOLOv4CSP"])
def test_letterbox_equals_bgr_on_cv2_decode(model, layout, fmt, form):
    """Stretched (YOLOv4-tiny 416) and letterboxed (YOLOv4-csp 640) one-frame letterbox, fp32 CHW and fp16 NHWC8."""
    from fastmot_b200 import _lib, models
    from fastmot_b200.detector import letterbox_geometry
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    m = models.YOLO.get_model(model)
    _, in_h, in_w = m.INPUT_SHAPE
    raw, bgr = _raw_pair(fmt, SIZES[0])
    (rx, ry, rw, rh), _, _ = letterbox_geometry(SIZES[0], (in_w, in_h), m.LETTERBOX)
    if layout == 0:
        want, got = (torch.full((3, in_h, in_w), -1.0, device="cuda") for _ in range(2))
    else:
        want, got = (torch.full((in_h, in_w, 8), -1.0, dtype=torch.float16, device="cuda") for _ in range(2))
    b = _bgr_frame(bgr)
    _lib.check(lib.fm_letterbox_preproc(C.byref(b.fm()), in_w, in_h, rx, ry, rw, rh, layout, ptr(want),
                                        stream_ptr()), "fm_letterbox_preproc BGR")
    f = _frame(raw, fmt, form)
    _lib.check(lib.fm_letterbox_preproc(C.byref(f.fm()), in_w, in_h, rx, ry, rw, rh, layout, ptr(got), stream_ptr()),
               f"fm_letterbox_preproc {fmt}")
    assert _bits_equal(got, want)
    assert float(want.float().std()) > 0.05          # a real picture, not a constant


@pytest.mark.parametrize("fmt, form", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("layout", [1, 2])
def test_crops_equal_bgr_on_cv2_decode(layout, fmt, form):
    """One-frame crops, boxes partly outside the frame included (the ReID layouts 1 and 2)."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    raw, bgr = _raw_pair(fmt, SIZES[0], seed=5)
    tl = _boxes(67, 21)
    tl[:3] = [[-40.7, -15.2, 60.3, 200.9], [1850.4, 1000.6, 2010.1, 1200.0], [-5.0, 900.0, 1930.0, 1100.0]]
    tl_dev = torch.as_tensor(tl).cuda()
    n, ow, oh = len(tl), 128, 256
    shape = {1: (n, oh, ow, 8), 2: (n, oh + 8, ow + 8, 4)}[layout]
    want, got = (torch.zeros(shape, dtype=torch.float16, device="cuda") for _ in range(2))
    b = _bgr_frame(bgr)
    _lib.check(lib.fm_roi_resize_norm(C.byref(b.fm()), ptr(tl_dev), None, n, ow, oh, layout, ptr(want),
                                      stream_ptr()), "fm_roi_resize_norm BGR")
    f = _frame(raw, fmt, form)
    assert f.size == SIZES[0]
    _lib.check(lib.fm_roi_resize_norm(C.byref(f.fm()), ptr(tl_dev), None, n, ow, oh, layout, ptr(got), stream_ptr()),
               f"fm_roi_resize_norm {fmt}")
    assert _bits_equal(got, want)


@pytest.mark.parametrize("fmt, form", CASES, ids=CASE_IDS)
def test_gray_half_and_gray_resize_equal_bgr(fmt, form):
    """gray_half at 1080p (the per-format 2x2 block loads) and gray_resize at optical-flow scale 0.6 x 0.45."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    W, H = SIZES[0]
    raw, bgr = _raw_pair(fmt, SIZES[0], seed=9)
    b = _bgr_frame(bgr)
    f = _frame(raw, fmt, form)
    bgr_fm, raw_fm = C.byref(b.fm()), C.byref(f.fm())
    for sw, sh in ((W // 2, H // 2), (round(0.6 * W), round(0.45 * H))):
        g_want, g_got = (torch.zeros(H, W, dtype=torch.uint8, device="cuda") for _ in range(2))
        s_want, s_got = (torch.zeros(sh, sw, dtype=torch.uint8, device="cuda") for _ in range(2))
        if 2 * sw == W:
            _lib.check(lib.fm_gray_half(bgr_fm, ptr(g_want), ptr(s_want), stream_ptr()), "gray_half BGR")
            _lib.check(lib.fm_gray_half(raw_fm, ptr(g_got), ptr(s_got), stream_ptr()), f"gray_half {fmt}")
        else:
            _lib.check(lib.fm_gray_resize(bgr_fm, ptr(g_want), ptr(s_want), sw, sh, stream_ptr()), "gray_resize BGR")
            _lib.check(lib.fm_gray_resize(raw_fm, ptr(g_got), ptr(s_got), sw, sh, stream_ptr()), f"gray_resize {fmt}")
        assert _bits_equal(g_got, g_want), (sw, sh)
        assert _bits_equal(s_got, s_want), (sw, sh)
        assert np.array_equal(g_want.cpu().numpy(), cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY))


@pytest.mark.parametrize("fmt, form", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("dst", [(960, 540), (1280, 720)], ids=["2x", "generic"])
def test_frame_resize_equals_cv2_resize_of_cv2_decode(dst, fmt, form):
    """fm_frame_resize from 1080p on the exact-2x area path and the generic path."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    raw, bgr = _raw_pair(fmt, SIZES[0], seed=11)
    f = _frame(raw, fmt, form)
    w, h = dst
    out = torch.full((h, w, 3), 77, dtype=torch.uint8, device="cuda")
    _lib.check(lib.fm_frame_resize(C.byref(f.fm()), ptr(out), w, h, stream_ptr()), "fm_frame_resize")
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), cv2.resize(bgr, dst))


@pytest.mark.parametrize("form", ["tight", "pitched"])
def test_geometry_table_mixes_five_formats_three_sizes(form):
    """fm_letterbox_preproc_geom (YOLOv4-csp 640) and fm_roi_resize_norm_geom (layout 2) over a table of six rows of
    1920x1080, 1280x720 and 1024x768 whose rows are BGR, NV12, I420, YUY2 and BGRx frames: the all-BGR table's output
    on the cv2 decodes.  form: every raw row tight, or pitched (NV12 two planes, I420 three planes)."""
    from fastmot_b200 import _lib, models
    from fastmot_b200.detector import letterbox_geometry
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    m = models.YOLO.get_model("YOLOv4CSP")
    _, in_h, in_w = m.INPUT_SHAPE
    fmts = ["YUY2", "I420", "NV12", "BGRX", "BGR", "I420"]
    sizes = [SIZES[i % 3] for i in range(len(fmts))]
    rows = len(fmts)
    pairs = [_raw_pair(fmt, wh, seed=7 + i) for i, (fmt, wh) in enumerate(zip(fmts, sizes))]
    pitched = {"NV12": "planes", "I420": "planes", "YUY2": "pitched", "BGRX": "pitched", "BGR": "tight"}
    raw_frames = [_frame(raw, fmt, "tight" if form == "tight" else pitched[fmt]) for (raw, _), fmt in zip(pairs, fmts)]
    bgr_frames = [_bgr_frame(b) for _, b in pairs]
    rois = [letterbox_geometry(wh, (in_w, in_h), m.LETTERBOX)[0] for wh in sizes]
    per = 23
    tl = np.concatenate([_boxes(per, 11 + i) * np.tile([wh[0] / 1920, wh[1] / 1080], 2) for i, wh in enumerate(sizes)])
    tl_dev = torch.as_tensor(tl).cuda()
    idx = torch.as_tensor(np.repeat(np.arange(rows, dtype=np.int32), per)).cuda()
    n = len(tl)
    out = {}
    for name, frames in (("bgr", bgr_frames), ("mixed", raw_frames)):
        g = _geom_table(frames, rois)
        lb = torch.full((rows, in_h, in_w, 8), -1.0, dtype=torch.float16, device="cuda")
        _lib.check(lib.fm_letterbox_preproc_geom(ptr(g), rows, in_w, in_h, ptr(lb), stream_ptr()), "letterbox_geom")
        cr = torch.zeros(n, 264, 136, 4, dtype=torch.float16, device="cuda")
        _lib.check(lib.fm_roi_resize_norm_geom(ptr(g), ptr(idx), ptr(tl_dev), n, 128, 256, 2, ptr(cr), stream_ptr()),
                   "roi_geom")
        torch.cuda.synchronize()
        out[name] = (lb, cr, g)
    assert _bits_equal(out["mixed"][0], out["bgr"][0])
    assert _bits_equal(out["mixed"][1], out["bgr"][1])


def test_frame_descriptor_rejects_bad_new_formats():
    """I420 without a V plane, of an odd size or with a short pitch; YUY2 of an odd width or with a short pitch; BGRx
    with a short pitch; an unknown format: every entry refuses them and says why."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    I420, YUY2, BGRX = _lib.FM_PIX_I420, _lib.FM_PIX_YUY2, _lib.FM_PIX_BGRX

    def fm(w, h, pitch, uv_pitch, fmt, uv=p, v=p):
        return C.byref(_lib.FmFrame(p, uv, w, h, pitch, uv_pitch, fmt, v))
    bad = [fm(32, 16, 0, 0, I420, v=None), fm(32, 16, 0, 0, I420, uv=None), fm(30, 15, 0, 0, I420),
           fm(32, 16, 31, 0, I420), fm(32, 16, 0, 15, I420), fm(31, 16, 0, 0, YUY2), fm(32, 16, 63, 0, YUY2),
           fm(32, 16, 127, 0, BGRX), fm(32, 16, 0, 0, 5)]
    good = [fm(32, 16, 0, 0, I420), fm(32, 16, 40, 16, I420), fm(32, 15, 64, 0, YUY2), fm(31, 15, 124, 0, BGRX)]
    for f in bad:
        assert lib.fm_letterbox_preproc(f, 8, 8, 0, 0, 8, 8, 1, ptr(out), stream_ptr()) != 0
        assert "fm_letterbox_preproc" in lib.fm_last_error().decode()
        assert lib.fm_roi_resize_norm(f, ptr(out), None, 1, 8, 8, 1, ptr(out), stream_ptr()) != 0
        assert lib.fm_gray_resize(f, ptr(out), ptr(out), 8, 4, stream_ptr()) != 0
        assert lib.fm_frame_resize(f, ptr(out), 8, 8, stream_ptr()) != 0
        assert "I420" in lib.fm_last_error().decode()
    for f in good:
        assert lib.fm_letterbox_preproc(f, 8, 8, 0, 0, 8, 8, 1, ptr(out), stream_ptr()) == 0
        assert lib.fm_frame_resize(f, ptr(out), 8, 8, stream_ptr()) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ end to end
def _input(raw, fmt, t):
    """Step t's frame in one of the forms MOT takes, in turn: host array (read ahead), tight, pitched."""
    forms = [None] + FORMS[fmt]
    k = t % 3
    return raw if k == 0 else _device_form(raw, fmt, forms[k])


def _assert_same_tracks(va, vb, where):
    assert set(va) == set(vb), (where, set(va) ^ set(vb))
    for i in va:
        assert np.array_equal(va[i], vb[i]), (where, i)


def _run_pair(fmt, size, capture, monkeypatch, T=12):
    """MOT(size, pixel_format=fmt, capture_size=capture) on raw frames against MOT(size) on the cv2 decodes (resized
    to size with cv2.resize when capture differs): detector input, KLT gray images and pyramids, embeddings and visible
    tracks equal at every step."""
    from fastmot_b200 import MOT
    from fastmot_b200.synth import SyntheticScene
    from oracle.pixfmt import cv2_decode
    from test_gpu_frame_resize import _scaled_dets_fn
    _synth_env(monkeypatch, "YOLOv4Tiny")
    cap = capture or size
    scene = SyntheticScene(64, size=cap, seed=4, label=0)
    dets = _scaled_dets_fn(scene, (size[0] / cap[0], size[1] / cap[1])) if capture else _dets_fn(scene)
    raw = [_encode(scene.frame(t), fmt) for t in range(T)]
    want = [cv2_decode(f, fmt) for f in raw]
    if capture:
        want = [cv2.resize(f, size) for f in want]
    taps = {"ref": [], "raw": []}

    def tap(name):
        return lambda i, d, e: taps[name].append((i, np.array(np.asarray(e), np.float32)))
    ref = MOT(size, detections_override=dets, embeddings_tap=tap("ref"), **_nets_kw("YOLOv4Tiny"))
    mot = MOT(size, detections_override=dets, embeddings_tap=tap("raw"), pixel_format=fmt.lower(),
              capture_size=capture, **_nets_kw("YOLOv4Tiny"))
    for m in (ref, mot):
        m.reset(1 / 30)
    n_vis = 0
    for t in range(T):
        ref.step(want[t])
        if t + 1 < T and (t + 1) % 3 == 0:
            mot.prefetch(raw[t + 1])                  # read-ahead of the next host frame
        mot.step(_input(raw[t], fmt, t))
        torch.cuda.synchronize()
        if t % 5 == 0:
            assert torch.equal(ref.detector.inp, mot.detector.inp), t
        fa, fb = ref.tracker.flow, mot.tracker.flow
        for k in range(2):
            assert torch.equal(fa.gray[k], fb.gray[k]), (t, k)
            for la, lb in zip(fa.pyr[k], fb.pyr[k]):
                assert torch.equal(la, lb), (t, k)
        va = {trk.trk_id: trk.tlbr.copy() for trk in ref.visible_tracks()}
        vb = {trk.trk_id: trk.tlbr.copy() for trk in mot.visible_tracks()}
        _assert_same_tracks(va, vb, t)
        n_vis = len(va)
    assert n_vis > 10
    assert [i for i, _ in taps["raw"]] == [i for i, _ in taps["ref"]] == [5, 10]
    for (_, ea), (_, eb) in zip(taps["ref"], taps["raw"]):
        assert ea.shape == eb.shape and len(ea) > 10
        assert np.array_equal(ea.view(np.uint32), eb.view(np.uint32))
    return mot


@pytest.mark.parametrize("fmt", FMTS)
def test_mot_equals_mot_bgr_on_cv2_decode(fmt, monkeypatch):
    """MOT(pixel_format=fmt) against MOT on the cv2 decodes: KLT on, real OSNet embeddings, three detector frames;
    frames arrive as host arrays (with read-ahead) and in both device forms."""
    from fastmot_b200.synth import SyntheticScene
    _run_pair(fmt, SyntheticScene(64, seed=4, label=0).size, None, monkeypatch)


def test_mot_capture_size_i420(monkeypatch):
    """I420 frames captured at 1080p and tracked at 720p against MOT(720p) on cv2.resize of the cv2 decodes."""
    mot = _run_pair("I420", (1280, 720), (1920, 1080), monkeypatch)
    assert mot._resizer is not None and mot.capture_size == (1920, 1080)


def test_multicamera_mixed_formats_equal_bgr():
    """MultiCameraMOT(pixel_formats=['YUY2', 'I420', 'NV12']) over three frame sizes under
    test_multicamera_cpu.schedule (batches of 1, 2 and 3 cameras, a reconnect, dropped and ended cameras) against an
    all-BGR group on the cv2 decodes: the same tracks per camera at every step, with real OSNet embeddings."""
    from fastmot_b200 import MultiCameraMOT
    from fastmot_b200.synth import SyntheticScene
    from oracle.pixfmt import cv2_decode
    from test_multicamera_cpu import schedule
    plans = schedule()
    T = len(plans)
    fmts = ["YUY2", "I420", "NV12"]
    scenes = [SyntheticScene(48, size=wh, seed=13 + 7 * s, label=0) for s, wh in enumerate(SIZES)]
    dets = [_dets_fn(sc) for sc in scenes]
    local, inputs = [0, 0, 0], []
    for t in range(T):
        if t == 14:
            local[1] = 0
        row = []
        for s in range(3):
            if s in sum(plans[t], []):
                row.append(_encode(scenes[s].frame(local[s]), fmts[s]))
                local[s] += 1
            else:
                row.append(None)
        inputs.append(row)
    kw = _nets_kw('YOLOv4Tiny')
    groups = {"BGR": MultiCameraMOT(SIZES, detections_override=lambda s, i: dets[s](i), **kw),
              "raw": MultiCameraMOT(SIZES, detections_override=lambda s, i: dets[s](i), pixel_formats=fmts, **kw)}
    assert groups["raw"].pixel_formats == fmts and groups["raw"].pixel_format is None
    assert [u.pixel_format for u in groups["raw"]._uploaders] == fmts
    for g in groups.values():
        g.reset(1 / 30)
    seen = 0
    for t in range(T):
        if t == 14:
            for g in groups.values():
                g.reset_stream(1, 1 / 30)
        groups["BGR"].step([None if f is None else cv2_decode(f, fmts[s]) for s, f in enumerate(inputs[t])])
        groups["raw"].step([None if f is None else
                            (f if (t + s) % 2 == 0 else _device_form(f, fmts[s], "tight" if fmts[s] != "NV12" else
                                                                      "planes"))
                            for s, f in enumerate(inputs[t])])
        for s in range(3):
            va = {trk.trk_id: trk.tlbr.copy() for trk in groups["BGR"].visible_tracks(s)}
            vb = {trk.trk_id: trk.tlbr.copy() for trk in groups["raw"].visible_tracks(s)}
            _assert_same_tracks(va, vb, (t, s))
            seen += len(va)
    assert seen > 0


@pytest.mark.parametrize("pinned", [True, False])
@pytest.mark.parametrize("fmt, per_pixel", [("I420", 1.5), ("YUY2", 2), ("BGRX", 4)])
def test_uploader_read_ahead_copies_each_frame_once(fmt, per_pixel, pinned):
    """prefetch(frame t + 1) issued before upload(frame t): upload(frame t) takes frame t's read-ahead (right
    contents, one copy of W * H * bytes-per-pixel per frame), and a frame that was never prefetched is copied on
    upload.  The uploaded tensor parses as a device frame of the format."""
    from fastmot_b200.devmem import FrameUploader, Frame
    rng = np.random.default_rng(17)
    size = (64, 48)
    up = FrameUploader(size, depth=3, pixel_format=fmt)
    assert up.nbytes == int(64 * 48 * per_pixel)
    frames = [rng.integers(0, 256, up.shape, dtype=np.uint8) for _ in range(7)]
    if pinned:
        frames = [torch.as_tensor(f).pin_memory().numpy() for f in frames]
    up.prefetch(frames[0])
    for t in range(6):
        up.prefetch(frames[t + 1])
        d = up.upload(frames[t])
        torch.cuda.synchronize()
        assert np.array_equal(d.cpu().numpy(), frames[t]), t
        assert up.bytes_copied == (t + 2) * up.nbytes, t
    f = up.upload_frame(Frame(fmt, *size, frames[6]))
    extra = rng.integers(0, 256, up.shape, dtype=np.uint8)
    d2 = up.upload(extra)
    torch.cuda.synchronize()
    assert (f.format, f.size, f.on_device) == (fmt, size, True)
    assert np.array_equal(f.y.cpu().numpy(), frames[6][:48] if fmt == "I420" else frames[6])
    assert np.array_equal(d2.cpu().numpy(), extra)
    assert up.bytes_copied == 8 * up.nbytes
