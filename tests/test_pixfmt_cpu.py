"""CPU: the I420, YUY2 and BGRx -> BGR restatements (oracle/pixfmt.py) against cv2.cvtColor, and the frame descriptor's
parsing of the three formats (fastmot_b200.devmem): every accepted form and the rejected ones."""
import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import pixfmt as opf
from fastmot_b200 import devmem

from test_nv12_cpu import _all_triples_frame


def _triples_i420():
    """The 512 x 32768 frame of test_nv12_cpu holding every (Y, U, V) once, as I420 (U and V de-interleaved)."""
    nv = _all_triples_frame()
    h, w = nv.shape[0] * 2 // 3, nv.shape[1]
    uv = nv[h:].reshape(-1)
    return np.concatenate([nv[:h].reshape(-1), uv[0::2], uv[1::2]]).reshape(3 * h // 2, w)


def _triples_yuy2():
    """A 256 x 65536 YUY2 frame holding every (Y, U, V) once: row i has U = i, pixel pairs 128 j .. 128 j + 127 have
    V = j and carry Y = 0..255 (two per pair)."""
    H, W = 256, 256 * 256
    pairs = np.empty((H, W // 2, 4), np.uint8)
    yv = np.tile(np.arange(256, dtype=np.uint8).reshape(128, 2), (256, 1))
    pairs[..., 0], pairs[..., 2] = yv[None, :, 0], yv[None, :, 1]
    pairs[..., 1] = np.arange(256, dtype=np.uint8)[:, None]
    pairs[..., 3] = np.repeat(np.arange(256, dtype=np.uint8), 128)[None, :]
    return pairs.reshape(H, W, 2)


def _keys(Y, U, V):
    return (Y.astype(np.int64) << 16) | (U.astype(np.int64) << 8) | V


def test_i420_oracle_equals_cv2_on_all_yuv_triples():
    yuv = _triples_i420()
    h, w = yuv.shape[0] * 2 // 3, yuv.shape[1]
    q = h * w // 4
    c = yuv[h:].reshape(-1)
    up = lambda p: np.repeat(np.repeat(p.reshape(h // 2, w // 2), 2, 0), 2, 1)
    assert np.unique(_keys(yuv[:h], up(c[:q]), up(c[q:]))).size == 1 << 24
    want = cv2.cvtColor(yuv, cv2.COLOR_YUV2BGR_I420)
    got = opf.i420_to_bgr(yuv)
    assert got.shape == want.shape and got.dtype == np.uint8
    assert int((got != want).sum()) == 0


def test_yuy2_oracle_equals_cv2_on_all_yuv_triples():
    yuy2 = _triples_yuy2()
    p = yuy2.reshape(yuy2.shape[0], -1, 4)
    assert np.unique(_keys(yuy2[..., 0], np.repeat(p[..., 1], 2, 1), np.repeat(p[..., 3], 2, 1))).size == 1 << 24
    want = cv2.cvtColor(yuy2, cv2.COLOR_YUV2BGR_YUY2)
    got = opf.yuy2_to_bgr(yuy2)
    assert got.shape == want.shape and got.dtype == np.uint8
    assert int((got != want).sum()) == 0


@pytest.mark.parametrize("shape", [(1080, 1920), (37, 51)])
def test_bgrx_oracle_equals_cv2_on_random_frames(shape):
    bgrx = np.random.default_rng(shape[1]).integers(0, 256, shape + (4,), dtype=np.uint8)
    want = cv2.cvtColor(bgrx, cv2.COLOR_BGRA2BGR)
    assert np.array_equal(opf.bgrx_to_bgr(bgrx), want)


@pytest.mark.parametrize("fmt", ["I420", "YUY2", "BGRX"])
def test_encoders_round_trip_through_cv2_decode(fmt):
    """The cv2 encoders give frames of the host layout devmem expects, and their cv2 decode is the restatement's."""
    bgr = np.random.default_rng(3).integers(0, 256, (48, 64, 3), dtype=np.uint8)
    _, restate, encode = opf.DECODES[fmt]
    raw = encode(bgr)
    assert raw.shape == devmem.FrameUploader.frame_shape((64, 48), fmt)
    assert np.array_equal(restate(raw), opf.cv2_decode(raw, fmt))


# ---------------------------------------------------------------------------------------------------- descriptors
@pytest.mark.parametrize("fmt, shape", [("I420", (1620, 1920)), ("YUY2", (1080, 1920, 2)), ("BGRX", (1080, 1920, 4))])
def test_descriptor_host_array(fmt, shape):
    f = devmem.pixel_frame(np.zeros(shape, np.uint8), fmt.lower())
    assert (f.format, f.size, f.on_device) == (fmt, (1920, 1080), False)
    assert devmem.FrameUploader.frame_shape((1920, 1080), fmt) == shape


def test_descriptor_i420_tight_tensor_layout():
    """A tight (3H/2, W) tensor: U follows the Y plane, V follows U, both with row pitch W/2 (CPU tensor: the layout
    check does not look at the device)."""
    t = torch.zeros(1620, 1920, dtype=torch.uint8)
    f = devmem.frame_layout(t, "I420")
    assert (f.size, f.y_pitch, f.uv_pitch) == ((1920, 1080), 1920, 960)
    assert f.uv.data_ptr() == t.data_ptr() + 1080 * 1920
    assert f.v.data_ptr() == t.data_ptr() + 1080 * 1920 + 540 * 960
    with pytest.raises(ValueError, match="cuda"):
        devmem.pixel_frame(t, "I420")


def test_descriptor_i420_three_planes_layout():
    """Pitched planes of a decoder surface: Y with row stride 2048, U and V with row stride 1024."""
    ys = torch.zeros(1088, 2048, dtype=torch.uint8)
    cs = torch.zeros(2, 544, 1024, dtype=torch.uint8)
    f = devmem.frame_layout((ys[:1080, :1920], cs[0, :540, :960], cs[1, :540, :960]), "I420")
    assert (f.size, f.y_pitch, f.uv_pitch) == ((1920, 1080), 2048, 1024)
    assert f.v.data_ptr() == cs.data_ptr() + 544 * 1024
    fm = f.fm()
    assert (fm.format, fm.pitch, fm.uv_pitch, fm.v) == (2, 2048, 1024, f.v.data_ptr())


@pytest.mark.parametrize("fmt, ch", [("YUY2", 2), ("BGRX", 4)])
def test_descriptor_packed_pitched_tensor_layout(fmt, ch):
    surf = torch.zeros(1080, 1920 + 64, ch, dtype=torch.uint8)
    f = devmem.frame_layout(surf[:, :1920], fmt)
    assert (f.size, f.y_pitch) == ((1920, 1080), (1920 + 64) * ch)
    assert f.fm().format == {"YUY2": 3, "BGRX": 4}[fmt]
    with pytest.raises(ValueError, match="cuda"):
        devmem.pixel_frame(surf[:, :1920], fmt)


@pytest.mark.parametrize("fmt, bad, what", [
    ("I420", np.zeros((1620, 1920), np.uint16), "uint8"),
    ("I420", np.zeros((1080, 1920, 3), np.uint8), r"\(3H/2, W\)"),
    ("I420", np.zeros((1621, 1920), np.uint8), r"\(3H/2, W\)"),
    ("I420", np.zeros((1620, 1919), np.uint8), "even"),
    ("I420", torch.zeros(1620, 1920, 2, dtype=torch.uint8), r"\(3H/2, W\)"),
    ("I420", torch.zeros(1620, 1984, dtype=torch.uint8)[:, :1920], "tight"),
    ("I420", (torch.zeros(1080, 1920, dtype=torch.uint8), torch.zeros(540, 960, dtype=torch.uint8)), "triple"),
    ("I420", (torch.zeros(1080, 1920, dtype=torch.uint8), torch.zeros(540, 960, dtype=torch.uint8),
              torch.zeros(540, 958, dtype=torch.uint8)), r"V plane: expected shape \(540, 960\)"),
    ("I420", (torch.zeros(1080, 1920, dtype=torch.uint8), torch.zeros(540, 1024, dtype=torch.uint8)[:, :960],
              torch.zeros(540, 960, dtype=torch.uint8)), "equal row strides"),
    ("I420", (torch.zeros(1080, 1920, dtype=torch.uint8), torch.zeros(540, 1920, dtype=torch.uint8)[:, ::2],
              torch.zeros(540, 1920, dtype=torch.uint8)[:, ::2]), "stride"),
    ("I420", (torch.zeros(1081, 1920, dtype=torch.uint8), torch.zeros(540, 960, dtype=torch.uint8),
              torch.zeros(540, 960, dtype=torch.uint8)), "even"),
    ("I420", (torch.zeros(1080, 1920, dtype=torch.uint8), torch.zeros(540, 960, dtype=torch.int16),
              torch.zeros(540, 960, dtype=torch.uint8)), "uint8"),
    ("YUY2", np.zeros((1080, 1920, 3), np.uint8), r"\(H, W, 2\)"),
    ("YUY2", np.zeros((1080, 1919, 2), np.uint8), "even width"),
    ("YUY2", np.zeros((1080, 1920, 2), np.int8), "uint8"),
    ("YUY2", torch.zeros(1080, 1920, 2, dtype=torch.uint8).transpose(0, 1), "strides"),
    ("YUY2", torch.zeros(1080 * 3840, dtype=torch.uint8).as_strided((1080, 1920, 2), (3800, 2, 1)), "strides"),
    ("YUY2", torch.zeros(1080, 1920, 4, dtype=torch.uint8)[..., :2], "strides"),
    ("BGRX", np.zeros((1080, 1920, 3), np.uint8), r"\(H, W, 4\)"),
    ("BGRX", np.zeros((0, 1920, 4), np.uint8), "non-empty"),
    ("BGRX", torch.zeros(1080, 1920, 4, dtype=torch.float32), "uint8"),
    ("BGRX", torch.zeros(1080, 1920, 8, dtype=torch.uint8)[..., ::2], "strides"),
    ("BGRX", torch.zeros(1080 * 7680, dtype=torch.uint8).as_strided((1080, 1920, 4), (7676, 4, 1)), "strides"),
    ("BGRX", "frame.raw", "ndarray or cuda tensor"),
    ("YUY2", [np.zeros((4, 4, 2), np.uint8)], "ndarray or cuda tensor"),
])
def test_descriptor_rejects(fmt, bad, what):
    with pytest.raises(ValueError, match=what):
        devmem.frame_layout(bad, fmt)


def test_descriptor_rejects_frame_of_another_format_and_unknown_format():
    f = devmem.frame_layout(np.zeros((8, 8, 2), np.uint8), "YUY2")
    with pytest.raises(ValueError, match="I420"):
        devmem.frame_layout(f, "I420")
    with pytest.raises(ValueError, match="pixel_format"):
        devmem.frame_layout(np.zeros((8, 8, 2), np.uint8), "UYVY")


@pytest.mark.parametrize("fmt, size, ok", [
    ("I420", (1279, 720), False), ("I420", (1280, 721), False), ("I420", (1280, 720), True),
    ("YUY2", (1279, 720), False), ("YUY2", (1280, 721), True),
    ("BGRX", (1279, 721), True), ("BGR", (1279, 721), True), ("NV12", (1280, 721), False),
])
def test_capture_size_evenness_per_format(fmt, size, ok):
    if ok:
        assert devmem.check_capture_size(size, (640, 360), fmt) == size
    else:
        with pytest.raises(ValueError, match="even"):
            devmem.check_capture_size(size, (640, 360), fmt)


def test_as_frame_checks_size_for_every_format():
    frames = {"I420": np.zeros((540, 640), np.uint8), "YUY2": np.zeros((360, 640, 2), np.uint8),
              "BGRX": np.zeros((360, 640, 4), np.uint8)}
    for fmt, a in frames.items():
        assert devmem.as_frame(a, fmt, (640, 360)).size == (640, 360)
        with pytest.raises(ValueError, match=r"\(640, 360\).*\(1280, 720\)"):
            devmem.as_frame(a, fmt, (1280, 720))


@pytest.mark.parametrize("kw, what", [
    (dict(pixel_format="NV12", pixel_formats=["NV12"] * 3), "not both"),
    (dict(pixel_formats=["YUY2", "I420"]), "expected 3 entries"),
    (dict(pixel_formats=["YUY2", "UYVY", "NV12"]), "camera 1: pixel_format"),
    (dict(pixel_formats=["YUY2", "I420", "NV12"], capture_sizes=[None, (1279, 720), None]), "camera 1: .*even"),
    (dict(pixel_formats=["YUY2", "BGRX", "NV12"], capture_sizes=[(1919, 1080), None, None]), "camera 0: .*even"),
])
def test_multicamera_rejects_bad_pixel_formats(kw, what):
    """MultiCameraMOT checks its per-camera formats (and each camera's capture size against its own format) before it
    builds anything."""
    from fastmot_b200 import MultiCameraMOT
    with pytest.raises(ValueError, match=what):
        MultiCameraMOT([(1280, 720), (640, 360), (1024, 768)], **kw)
