"""GPU: frames captured at another size than the tracking size.

fm_frame_resize against cv2.resize (INTER_LINEAR) bit for bit, on BGR frames and on NV12 frames in the three device
layouts of test_gpu_nv12 (the reference is cv2.resize of the cv2 decode), and MOT / MultiCameraMOT with capture sizes
against the same trackers fed frames resized on the host with cv2.resize.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from test_frame_resize_cpu import IDS, PAIRS
from test_gpu_nv12 import FORMS, _device_form, _nets_kw, _synth_env

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")


def _noise(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def _resize_dev(f, size):
    """fm_frame_resize of the device Frame f to size = (w, h), as a host array."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    w, h = size
    out = torch.full((h, w, 3), 77, dtype=torch.uint8, device="cuda")
    _lib.check(lib.fm_frame_resize(C.byref(f.fm()), ptr(out), w, h, stream_ptr()), "fm_frame_resize")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _ndiff(a, b):
    assert a.shape == b.shape
    return int((a != b).sum())


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("src, dst", PAIRS, ids=IDS)
def test_frame_resize_bgr_equals_cv2(src, dst):
    from fastmot_b200.devmem import Frame
    img = _noise((src[1], src[0], 3), src[0] * 7919 + src[1])
    got = _resize_dev(Frame.bgr(torch.as_tensor(img).cuda()), dst)
    assert _ndiff(got, cv2.resize(img, dst)) == 0


EVEN = [(s, d, i) for (s, d), i in zip(PAIRS, IDS) if s[0] % 2 == 0 and s[1] % 2 == 0]


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("src, dst", [e[:2] for e in EVEN], ids=[e[2] for e in EVEN])
def test_frame_resize_nv12_equals_cv2_on_cv2_decode(src, dst, form):
    from fastmot_b200.devmem import nv12_frame
    w, h = src
    nv = _noise((3 * h // 2, w), w * 31 + h)
    got = _resize_dev(nv12_frame(_device_form(nv, form)), dst)
    assert _ndiff(got, cv2.resize(cv2.cvtColor(nv, cv2.COLOR_YUV2BGR_NV12), dst)) == 0


def test_frame_resize_rejects_bad_inputs():
    """A NULL frame, an empty output size, a NULL output and an odd NV12 frame return an error and say why."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    bgr = _lib.FmFrame(p, None, 64, 32, 0, 0, _lib.FM_PIX_BGR)

    def err():
        return lib.fm_last_error().decode()
    assert lib.fm_frame_resize(None, ptr(out), 16, 8, stream_ptr()) != 0
    assert "fm_frame_resize" in err() and "frame" in err()
    assert lib.fm_frame_resize(C.byref(bgr), ptr(out), 0, 8, stream_ptr()) != 0
    assert "output size" in err()
    assert lib.fm_frame_resize(C.byref(bgr), ptr(out), 16, -1, stream_ptr()) != 0
    assert "output size" in err()
    assert lib.fm_frame_resize(C.byref(bgr), None, 16, 8, stream_ptr()) != 0
    assert "dst" in err()
    odd = _lib.FmFrame(p, p, 63, 32, 64, 64, _lib.FM_PIX_NV12)
    assert lib.fm_frame_resize(C.byref(odd), ptr(out), 16, 8, stream_ptr()) != 0
    assert "even" in err()
    assert lib.fm_frame_resize(C.byref(bgr), ptr(out), 16, 8, stream_ptr()) == 0


# ------------------------------------------------------------------------------------------------ end to end
def _scaled_dets_fn(scene, k):
    """The scene's scripted boxes scaled by k = tracking size / capture size."""
    from fastmot_b200 import DET_DTYPE
    kx, ky = k

    def dets(t):
        tl, lb, cf, _ = scene.detections(t)
        d = np.zeros(len(tl), DET_DTYPE)
        d['tlbr'], d['label'], d['conf'] = tl * np.array([kx, ky, kx, ky]), lb, cf
        return d.view(np.recarray)
    return dets


def _bgr_input(f, t):
    """Step t's BGR frame: a host array (steps 0, 2, ...) or a cuda tensor."""
    return f if t % 2 == 0 else torch.as_tensor(f).cuda()


def _nv12_input(nv, t):
    """Step t's NV12 frame, in turn: host array, tight, pitched, two-plane surface."""
    k = t % 4
    return nv if k == 0 else _device_form(nv, FORMS[k - 1])


@pytest.mark.parametrize("fmt", ["BGR", "NV12"])
@pytest.mark.parametrize("capture, size", [((1920, 1080), (1280, 720)), ((1280, 720), (1920, 1080))],
                         ids=["1080p-to-720p", "720p-to-1080p"])
def test_mot_capture_size_equals_mot_on_cv2_resize(capture, size, fmt, monkeypatch):
    """MOT(size, capture_size=capture) on capture-size frames against MOT(size) fed cv2.resize(frame, size) (of the cv2
    decode for NV12): KLT on, real OSNet embeddings (bit for bit through embeddings_tap), three detector frames; the
    detector input, the KLT gray images and pyramids and the visible track ids / boxes are equal at every step.  Host
    frames are read ahead with prefetch."""
    from fastmot_b200 import MOT
    from fastmot_b200.synth import SyntheticScene
    from oracle.nv12 import bgr_to_nv12
    _synth_env(monkeypatch, "YOLOv4Tiny")
    scene = SyntheticScene(64, size=capture, seed=4, label=0)
    dets = _scaled_dets_fn(scene, (size[0] / capture[0], size[1] / capture[1]))
    T = 12
    raw = [scene.frame(t) for t in range(T)]
    if fmt == "NV12":
        raw = [bgr_to_nv12(f) for f in raw]
        want = [cv2.resize(cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12), size) for f in raw]
        inputs = [_nv12_input(f, t) for t, f in enumerate(raw)]
    else:
        want = [cv2.resize(f, size) for f in raw]
        inputs = [_bgr_input(f, t) for t, f in enumerate(raw)]
    taps = {"ref": [], "scaled": []}

    def tap(name):
        return lambda i, d, e: taps[name].append((i, np.array(np.asarray(e), np.float32)))

    ref = MOT(size, detections_override=dets, embeddings_tap=tap("ref"), **_nets_kw("YOLOv4Tiny"))
    mot = MOT(size, detections_override=dets, embeddings_tap=tap("scaled"), pixel_format=fmt, capture_size=capture,
              **_nets_kw("YOLOv4Tiny"))
    assert mot._resizer is not None and mot.capture_size == capture
    for m in (ref, mot):
        m.reset(1 / 30)
    n_vis = 0
    for t in range(T):
        ref.step(want[t])
        if t + 1 < T and isinstance(inputs[t + 1], np.ndarray):
            mot.prefetch(inputs[t + 1])             # read-ahead of the next host frame, at the capture size
        mot.step(inputs[t])
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
        assert set(va) == set(vb), (t, set(va) ^ set(vb))
        for i in va:
            assert np.array_equal(va[i], vb[i]), (t, i)
        n_vis = len(va)
    assert n_vis > 10
    assert [i for i, _ in taps["scaled"]] == [i for i, _ in taps["ref"]] == [5, 10]
    for (_, ea), (_, eb) in zip(taps["ref"], taps["scaled"]):
        assert ea.shape == eb.shape and len(ea) > 10
        assert np.array_equal(ea.view(np.uint32), eb.view(np.uint32))


def test_mot_rejects_frames_of_another_size_and_odd_nv12_capture():
    from fastmot_b200 import MOT
    mot = MOT((640, 360), capture_size=(1280, 720), **_nets_kw("YOLOv4Tiny"))
    mot.reset(1 / 30)
    with pytest.raises(ValueError, match=r"\(640, 360\).*\(1280, 720\)"):
        mot.step(np.zeros((360, 640, 3), np.uint8))
    with pytest.raises(ValueError, match="even"):
        MOT((640, 360), capture_size=(1279, 720), pixel_format="NV12", **_nets_kw("YOLOv4Tiny"))


def _step_launches(mot, frames):
    """Library launches of each step over `frames`."""
    from fastmot_b200 import _lib
    out = []
    for f in frames:
        n0 = _lib.launch_count()
        mot.step(f)
        torch.cuda.synchronize()
        out.append(_lib.launch_count() - n0)
    return out


def test_unscaled_mot_launches_no_resize(monkeypatch):
    """capture_size=None and capture_size == size build no resizer and launch what MOT(size) launches; a scaled MOT
    launches exactly one kernel more per step (the resize)."""
    from fastmot_b200 import MOT
    from fastmot_b200.synth import SyntheticScene
    _synth_env(monkeypatch, "YOLOv4Tiny")
    size, capture = (1280, 720), (1920, 1080)
    scene = SyntheticScene(64, size=capture, seed=4, label=0)
    dets = _scaled_dets_fn(scene, (2 / 3, 2 / 3))
    raw = [scene.frame(t) for t in range(6)]
    small = [cv2.resize(f, size) for f in raw]
    counts = {}
    for name, cap in (("none", None), ("equal", size), ("scaled", capture)):
        m = MOT(size, detections_override=dets, capture_size=cap, **_nets_kw("YOLOv4Tiny"))
        assert (m._resizer is None) == (name != "scaled")
        m.reset(1 / 30)
        counts[name] = _step_launches(m, raw if name == "scaled" else small)
    assert counts["equal"] == counts["none"]
    assert counts["scaled"] == [n + 1 for n in counts["none"]], counts


def test_multicamera_capture_sizes_equal_host_resized_group():
    """MultiCameraMOT under test_multicamera_cpu.schedule (batches of 1, 2 and 3 cameras, a reconnect, dropped and
    ended cameras) with camera 0 captured at 1080p and tracked at 720p, camera 1 captured at 4K and tracked at 1080p
    (the exact-2x path) and camera 2 unscaled, against a group fed cv2.resize'd host frames: equal tracks per camera at
    every step, with real OSNet embeddings."""
    from fastmot_b200 import MultiCameraMOT
    from fastmot_b200.synth import SyntheticScene
    from test_multicamera_cpu import schedule
    plans = schedule()
    T = len(plans)
    sizes = [(1280, 720), (1920, 1080), (1024, 768)]
    captures = [(1920, 1080), (3840, 2160), None]
    scenes = [SyntheticScene(48, size=cap or wh, seed=13 + 7 * s, label=0)
              for s, (cap, wh) in enumerate(zip(captures, sizes))]
    dets = [_scaled_dets_fn(sc, (wh[0] / sc.size[0], wh[1] / sc.size[1])) for sc, wh in zip(scenes, sizes)]
    groups = {name: MultiCameraMOT(sizes, detections_override=lambda s, i: dets[s](i),
                                   capture_sizes=captures if name == "scaled" else None, **_nets_kw('YOLOv4Tiny'))
              for name in ("ref", "scaled")}
    assert [r is None for r in groups["scaled"]._resizers] == [False, False, True]
    for g in groups.values():
        g.reset(1 / 30)
    local, seen = [0, 0, 0], 0
    for t in range(T):
        if t == 14:
            local[1] = 0
            for g in groups.values():
                g.reset_stream(1, 1 / 30)
        raw = []
        for s in range(3):
            if s in sum(plans[t], []):
                raw.append(scenes[s].frame(local[s]))
                local[s] += 1
            else:
                raw.append(None)
        groups["ref"].step([None if f is None else cv2.resize(f, wh) for f, wh in zip(raw, sizes)])
        groups["scaled"].step([None if f is None else _bgr_input(f, t + s) for s, f in enumerate(raw)])
        for s in range(3):
            va = {trk.trk_id: trk.tlbr.copy() for trk in groups["ref"].visible_tracks(s)}
            vb = {trk.trk_id: trk.tlbr.copy() for trk in groups["scaled"].visible_tracks(s)}
            assert set(va) == set(vb), (t, s, set(va) ^ set(vb))
            for i in va:
                assert np.array_equal(va[i], vb[i]), (t, s, i)
            seen += len(va)
    assert seen > 0


def test_multistream_capture_size_is_passed_to_every_stream():
    from fastmot_b200 import MultiStreamMOT
    ms = MultiStreamMOT((1280, 720), 2, capture_size=(1920, 1080), **_nets_kw('YOLOv4Tiny'))
    assert ms.capture_sizes == [(1920, 1080)] * 2 and all(r is not None for r in ms._resizers)
    with pytest.raises(ValueError, match="camera 1"):
        ms.step([np.zeros((1080, 1920, 3), np.uint8), np.zeros((720, 1280, 3), np.uint8)])
