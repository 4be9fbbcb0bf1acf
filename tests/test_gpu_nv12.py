"""GPU: NV12 frames read in place by the letterbox, crop and KLT gray kernels, and tracked end to end.

Frames are SyntheticScene frames taken to NV12 (cv2 BGR -> I420, U and V interleaved: oracle/nv12.py).  The reference
is always the BGR path fed cv2.cvtColor(nv12, cv2.COLOR_YUV2BGR_NV12); every comparison is bit for bit.  Each kernel
check runs on three device layouts of the same NV12 frame: tight (3H/2, W), pitched (row stride W + 64), and two planes
in a padded-height decoder surface (Y in a surface of 1088 rows for 1080p, UV after it; padding filled with 255).
"""
import ctypes as C
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from test_gpu_multistream import _boxes
from test_gpu_yolo_ops import CASES

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

SIZES = [(1920, 1080), (1280, 720), (1024, 768)]
FORMS = ["tight", "pitched", "planes"]


def _scene_bgr(size, seed=3, t=2):
    from fastmot_b200.synth import SyntheticScene
    return SyntheticScene(64, size=size, seed=seed, label=0).frame(t)


def _nv12_pair(size, seed=3, t=2):
    """(NV12 host frame, its cv2 BGR decode)."""
    from oracle.nv12 import bgr_to_nv12
    nv = bgr_to_nv12(_scene_bgr(size, seed, t))
    return nv, cv2.cvtColor(nv, cv2.COLOR_YUV2BGR_NV12)


def _device_form(nv, form):
    """The NV12 host frame `nv` on the device in one of FORMS (what devmem.nv12_frame accepts)."""
    h, w = nv.shape[0] * 2 // 3, nv.shape[1]
    t = torch.as_tensor(nv)
    if form == "tight":
        return t.cuda()
    if form == "pitched":
        surf = torch.full((3 * h // 2, w + 64), 255, dtype=torch.uint8, device="cuda")
        surf[:, :w] = t.cuda()
        return surf[:, :w]
    hp = (h + 15) // 16 * 16
    hp = hp + 16 if hp == h else hp
    surf = torch.full((hp + hp // 2, w + 32), 255, dtype=torch.uint8, device="cuda")
    surf[:h, :w] = t[:h].cuda()
    surf[hp:hp + h // 2, :w] = t[h:].cuda()
    return surf[:h, :w], surf[hp:hp + h // 2, :w]


def _frame(nv, form):
    from fastmot_b200.devmem import nv12_frame
    return nv12_frame(_device_form(nv, form))


def _bits_equal(a, b):
    torch.cuda.synchronize()
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _geom_table(frames, rois):
    """Device FmFrameGeom rows of `frames` (devmem.Frame) with letterbox ROIs `rois`."""
    from fastmot_b200 import _lib
    rows = (_lib.FmFrameGeom * len(frames))()
    for r, f, roi in zip(rows, frames, rois):
        r.frame = f.fm()
        r.roi_x, r.roi_y, r.roi_w, r.roi_h = roi
    return torch.frombuffer(bytearray(bytes(rows)), dtype=torch.uint8).cuda()


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("model", ["YOLOv4Tiny", "YOLOv4CSP"])
def test_letterbox_nv12_fmframe_equals_bgr_on_cv2_decode(model, layout, form):
    """Stretched (YOLOv4-tiny 416) and letterboxed (YOLOv4-csp 640) one-frame letterbox, fp32 CHW and fp16 NHWC8."""
    from fastmot_b200 import _lib, models
    from fastmot_b200.detector import letterbox_geometry
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    lib = _lib.require_device()
    m = models.YOLO.get_model(model)
    _, in_h, in_w = m.INPUT_SHAPE
    W, H = SIZES[0]
    nv, bgr = _nv12_pair(SIZES[0])
    (rx, ry, rw, rh), _, _ = letterbox_geometry((W, H), (in_w, in_h), m.LETTERBOX)
    if layout == 0:
        want, got = (torch.full((3, in_h, in_w), -1.0, device="cuda") for _ in range(2))
    else:
        want, got = (torch.full((in_h, in_w, 8), -1.0, dtype=torch.float16, device="cuda") for _ in range(2))
    bgr_dev = Frame.bgr(torch.as_tensor(bgr).cuda())
    _lib.check(lib.fm_letterbox_preproc(C.byref(bgr_dev.fm()), in_w, in_h, rx, ry, rw, rh, layout, ptr(want),
                                        stream_ptr()), "fm_letterbox_preproc BGR")
    f = _frame(nv, form)
    _lib.check(lib.fm_letterbox_preproc(C.byref(f.fm()), in_w, in_h, rx, ry, rw, rh, layout, ptr(got), stream_ptr()),
               "fm_letterbox_preproc NV12")
    assert _bits_equal(got, want)
    assert float(want.float().std()) > 0.05          # a real picture, not a constant


@pytest.mark.parametrize("form", FORMS)
def test_geometry_table_fmframe_rows_three_sizes(form):
    """fm_letterbox_preproc_geom (YOLOv4-csp 640, each size its own ROI) and fm_roi_resize_norm_geom (layout 2) over
    1920x1080, 1280x720 and 1024x768 at once: an all-NV12 table and a mixed NV12 / BGR table give the all-BGR table's
    output on the cv2 decodes."""
    from fastmot_b200 import _lib, models
    from fastmot_b200.detector import letterbox_geometry
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    lib = _lib.require_device()
    m = models.YOLO.get_model("YOLOv4CSP")
    _, in_h, in_w = m.INPUT_SHAPE
    pairs = [_nv12_pair(wh, seed=7 + i) for i, wh in enumerate(SIZES)]
    rois = [letterbox_geometry(wh, (in_w, in_h), m.LETTERBOX)[0] for wh in SIZES]
    bgr_frames = [Frame.bgr(torch.as_tensor(b).cuda()) for _, b in pairs]
    nv_frames = [_frame(nv, form) for nv, _ in pairs]
    tables = {"bgr": bgr_frames, "nv12": nv_frames, "mixed": [nv_frames[0], bgr_frames[1], nv_frames[2]]}
    per = 29
    tl = np.concatenate([_boxes(per, 11 + i) * np.tile([wh[0] / 1920, wh[1] / 1080], 2)
                         for i, wh in enumerate(SIZES)])
    tl_dev = torch.as_tensor(tl).cuda()
    idx = torch.as_tensor(np.repeat(np.arange(3, dtype=np.int32), per)).cuda()
    n = len(tl)
    out = {}
    for name, frames in tables.items():
        g = _geom_table(frames, rois)
        lb = torch.full((3, in_h, in_w, 8), -1.0, dtype=torch.float16, device="cuda")
        _lib.check(lib.fm_letterbox_preproc_geom(ptr(g), 3, in_w, in_h, ptr(lb), stream_ptr()), "letterbox_geom")
        cr = torch.zeros(n, 264, 136, 4, dtype=torch.float16, device="cuda")
        _lib.check(lib.fm_roi_resize_norm_geom(ptr(g), ptr(idx), ptr(tl_dev), n, 128, 256, 2, ptr(cr), stream_ptr()),
                   "roi_geom")
        torch.cuda.synchronize()
        out[name] = (lb, cr, g)
    for name in ("nv12", "mixed"):
        assert _bits_equal(out[name][0], out["bgr"][0]), name
        assert _bits_equal(out[name][1], out["bgr"][1]), name


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("layout", [0, 1, 2])
def test_crops_nv12_fmframe_equal_bgr_on_cv2_decode(layout, form):
    """One-frame crops, boxes partly outside the frame included, at every output layout."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    lib = _lib.require_device()
    W, H = SIZES[0]
    nv, bgr = _nv12_pair(SIZES[0], seed=5)
    tl = _boxes(67, 21)
    tl[:3] = [[-40.7, -15.2, 60.3, 200.9], [1850.4, 1000.6, 2010.1, 1200.0], [-5.0, 900.0, 1930.0, 1100.0]]
    tl_dev = torch.as_tensor(tl).cuda()
    n, ow, oh = len(tl), 128, 256
    shape = {0: (n, 3, oh, ow), 1: (n, oh, ow, 8), 2: (n, oh + 8, ow + 8, 4)}[layout]
    dt = torch.float32 if layout == 0 else torch.float16
    want, got = (torch.zeros(shape, dtype=dt, device="cuda") for _ in range(2))
    bgr_dev = Frame.bgr(torch.as_tensor(bgr).cuda())
    _lib.check(lib.fm_roi_resize_norm(C.byref(bgr_dev.fm()), ptr(tl_dev), None, n, ow, oh, layout, ptr(want),
                                      stream_ptr()), "fm_roi_resize_norm BGR")
    f = _frame(nv, form)
    assert f.size == (W, H)
    _lib.check(lib.fm_roi_resize_norm(C.byref(f.fm()), ptr(tl_dev), None, n, ow, oh, layout, ptr(got), stream_ptr()),
               "fm_roi_resize_norm NV12")
    assert _bits_equal(got, want)


@pytest.mark.parametrize("form", FORMS)
def test_gray_half_and_gray_resize_nv12_fmframe(form):
    """gray_half at 1080p (2x2 block = one chroma sample) and gray_resize at optical-flow scale 0.6 x 0.45."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    lib = _lib.require_device()
    W, H = SIZES[0]
    nv, bgr = _nv12_pair(SIZES[0], seed=9)
    bgr_dev = Frame.bgr(torch.as_tensor(bgr).cuda())
    bgr_fm = C.byref(bgr_dev.fm())
    f = _frame(nv, form)
    assert f.size == (W, H)
    nv_fm = C.byref(f.fm())
    for sw, sh in ((W // 2, H // 2), (round(0.6 * W), round(0.45 * H))):
        g_want, g_got = (torch.zeros(H, W, dtype=torch.uint8, device="cuda") for _ in range(2))
        s_want, s_got = (torch.zeros(sh, sw, dtype=torch.uint8, device="cuda") for _ in range(2))
        if 2 * sw == W:
            _lib.check(lib.fm_gray_half(bgr_fm, ptr(g_want), ptr(s_want), stream_ptr()), "gray_half BGR")
            _lib.check(lib.fm_gray_half(nv_fm, ptr(g_got), ptr(s_got), stream_ptr()), "gray_half NV12")
        else:
            _lib.check(lib.fm_gray_resize(bgr_fm, ptr(g_want), ptr(s_want), sw, sh, stream_ptr()), "gray_resize BGR")
            _lib.check(lib.fm_gray_resize(nv_fm, ptr(g_got), ptr(s_got), sw, sh, stream_ptr()), "gray_resize NV12")
        assert _bits_equal(g_got, g_want), (sw, sh)
        assert _bits_equal(s_got, s_want), (sw, sh)
        want = cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)
        assert np.array_equal(g_want.cpu().numpy(), want)


def test_frame_descriptor_rejects_bad_nv12_and_null_bgr():
    """NV12 frames with an odd size, a short pitch or no UV plane, and a BGR frame without pixels, are rejected."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    out = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()

    def fm(y, uv, w, h, pitch, uv_pitch, fmt=_lib.FM_PIX_NV12):
        return C.byref(_lib.FmFrame(y, uv, w, h, pitch, uv_pitch, fmt))
    assert lib.fm_gray_half(fm(p, p, 31, 16, 32, 32), ptr(out), ptr(out), stream_ptr()) != 0
    assert lib.fm_gray_resize(fm(p, p, 32, 15, 32, 32), ptr(out), ptr(out), 16, 8, stream_ptr()) != 0
    assert lib.fm_gray_half(fm(p, p, 32, 16, 30, 32), ptr(out), ptr(out), stream_ptr()) != 0
    assert lib.fm_letterbox_preproc(fm(p, None, 32, 16, 32, 32), 8, 8, 0, 0, 8, 8, 1, ptr(out), stream_ptr()) != 0
    assert lib.fm_letterbox_preproc(fm(None, None, 32, 16, 0, 0, _lib.FM_PIX_BGR), 8, 8, 0, 0, 8, 8, 1, ptr(out),
                                    stream_ptr()) != 0


# ------------------------------------------------------------------------------------------------ end to end
def _synth_env(monkeypatch, name):
    bias, gain, _ = CASES[name]
    monkeypatch.setenv("FM_SYNTH_OBJ_BIAS", str(bias))
    monkeypatch.setenv("FM_SYNTH_HEAD_GAIN", str(gain))


def _nets_kw(name):
    from oracle.run import default_tracker_cfg
    return dict(detector_frame_skip=5, class_ids=(0,), yolo_detector_cfg=NS(model=name),
                feature_extractor_cfgs=(NS(model='OSNet025'),), tracker_cfg=NS(**default_tracker_cfg()))


def _dets_fn(scene):
    from fastmot_b200 import DET_DTYPE

    def dets(t):
        tl, lb, cf, _ = scene.detections(t)
        d = np.zeros(len(tl), DET_DTYPE)
        d['tlbr'], d['label'], d['conf'] = tl, lb, cf
        return d.view(np.recarray)
    return dets


def _nv12_input(nv, t):
    """Step t's NV12 frame in one of the forms MOT takes, in turn: host array, tight, pitched, two-plane surface."""
    k = t % 4
    return nv if k == 0 else _device_form(nv, FORMS[k - 1])


@pytest.mark.parametrize("model", ["YOLOv4Tiny", "YOLOv4CSP"])
def test_mot_nv12_equals_mot_bgr_on_cv2_decode(model, monkeypatch):
    """MOT(pixel_format='NV12') against MOT on the cv2 decodes: KLT on, real OSNet embeddings (bit for bit through
    embeddings_tap), three detector frames; detector input, KLT gray images and visible track ids / boxes equal at
    every step.  NV12 frames arrive as host arrays (with read-ahead), tight, pitched and two-plane device frames."""
    from fastmot_b200 import MOT
    from fastmot_b200.synth import SyntheticScene
    from oracle.nv12 import bgr_to_nv12
    _synth_env(monkeypatch, model)
    scene = SyntheticScene(64, seed=4, label=0)
    dets = _dets_fn(scene)
    T = 12
    nv = [bgr_to_nv12(scene.frame(t)) for t in range(T)]
    bgr = [cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) for f in nv]
    taps = {"bgr": [], "nv12": []}

    def tap(name):
        return lambda i, d, e: taps[name].append((i, np.array(np.asarray(e), np.float32)))

    mots = {name: MOT(scene.size, detections_override=dets, embeddings_tap=tap(name),
                      pixel_format=name.upper(), **_nets_kw(model)) for name in taps}
    for m in mots.values():
        m.reset(1 / 30)
    n_vis = 0
    for t in range(T):
        mots["bgr"].step(bgr[t])
        x = _nv12_input(nv[t], t)
        if t + 1 < T and (t + 1) % 4 == 0:
            mots["nv12"].prefetch(nv[t + 1])
        mots["nv12"].step(x)
        torch.cuda.synchronize()
        a, b = mots["bgr"], mots["nv12"]
        if t % 5 == 0:
            assert torch.equal(a.detector.inp, b.detector.inp), t
        fa, fb = a.tracker.flow, b.tracker.flow
        for k in range(2):
            assert torch.equal(fa.gray[k], fb.gray[k]), (t, k)
            for la, lb in zip(fa.pyr[k], fb.pyr[k]):
                assert torch.equal(la, lb), (t, k)
        va = {trk.trk_id: trk.tlbr.copy() for trk in a.visible_tracks()}
        vb = {trk.trk_id: trk.tlbr.copy() for trk in b.visible_tracks()}
        assert set(va) == set(vb), (t, set(va) ^ set(vb))
        for i in va:
            assert np.array_equal(va[i], vb[i]), (t, i)
        n_vis = len(va)
    assert n_vis > 10
    assert [i for i, _ in taps["nv12"]] == [i for i, _ in taps["bgr"]] == [5, 10]
    for (_, ea), (_, eb) in zip(taps["bgr"], taps["nv12"]):
        assert ea.shape == eb.shape and len(ea) > 10
        assert np.array_equal(ea.view(np.uint32), eb.view(np.uint32))


def test_multicamera_nv12_equals_bgr():
    """MultiCameraMOT over three frame sizes under test_multicamera_cpu.schedule (batches of 1, 2 and 3 cameras, a
    reconnect, dropped and ended cameras), pixel_format='NV12' against 'BGR' on the cv2 decodes: the same tracks per
    camera at every step, with real OSNet embeddings."""
    from fastmot_b200 import MultiCameraMOT
    from fastmot_b200.synth import SyntheticScene
    from oracle.nv12 import bgr_to_nv12
    from test_multicamera_cpu import schedule
    plans = schedule()
    T = len(plans)
    scenes = [SyntheticScene(48, size=wh, seed=13 + 7 * s, label=0) for s, wh in enumerate(SIZES)]
    dets = [_dets_fn(sc) for sc in scenes]
    # camera s's frame on step t is its local frame (restarting after camera 1's reconnect at step 14)
    local, inputs = [0, 0, 0], []
    for t in range(T):
        if t == 14:
            local[1] = 0
        row = []
        for s in range(3):
            if s in sum(plans[t], []):
                row.append(bgr_to_nv12(scenes[s].frame(local[s])))
                local[s] += 1
            else:
                row.append(None)
        inputs.append(row)
    groups = {fmt: MultiCameraMOT(SIZES, detections_override=lambda s, i: dets[s](i), pixel_format=fmt,
                                  **_nets_kw('YOLOv4Tiny')) for fmt in ("BGR", "NV12")}
    for g in groups.values():
        g.reset(1 / 30)
    seen = 0
    for t in range(T):
        if t == 14:
            for g in groups.values():
                g.reset_stream(1, 1 / 30)
        groups["BGR"].step([None if f is None else cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) for f in inputs[t]])
        groups["NV12"].step([None if f is None else _nv12_input(f, t + s) for s, f in enumerate(inputs[t])])
        for s in range(3):
            va = {trk.trk_id: trk.tlbr.copy() for trk in groups["BGR"].visible_tracks(s)}
            vb = {trk.trk_id: trk.tlbr.copy() for trk in groups["NV12"].visible_tracks(s)}
            assert set(va) == set(vb), (t, s, set(va) ^ set(vb))
            for i in va:
                assert np.array_equal(va[i], vb[i]), (t, s, i)
            seen += len(va)
    assert seen > 0


@pytest.mark.parametrize("pinned", [True, False])
@pytest.mark.parametrize("fmt", ["BGR", "NV12"])
def test_uploader_read_ahead_copies_each_frame_once(fmt, pinned):
    """prefetch(frame t + 1) issued before upload(frame t), as bench.py's e2e pass does: upload(frame t) takes frame t's
    read-ahead (right contents, one copy per frame), and a frame that was never prefetched is copied on upload."""
    from fastmot_b200.devmem import FrameUploader
    rng = np.random.default_rng(17)
    size = (64, 48)
    up = FrameUploader(size, depth=3, pixel_format=fmt)
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
    d = up.upload(frames[6])
    extra = rng.integers(0, 256, up.shape, dtype=np.uint8)
    d2 = up.upload(extra)
    torch.cuda.synchronize()
    assert np.array_equal(d.cpu().numpy(), frames[6]) and np.array_equal(d2.cpu().numpy(), extra)
    assert up.bytes_copied == 8 * up.nbytes
