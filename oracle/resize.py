"""cv2.resize(frame, (dw, dh)) with the default INTER_LINEAR for u8 frames, as OpenCV 4.13 computes it, restated in NumPy
(what fm_frame_resize computes on the GPU: fastmot_b200/csrc/frame_resize.cu, cv_linear.cuh).

Exactly 2x smaller in both axes (sw == 2 dw, sh == 2 dh): OpenCV's 2x2 area path, (a + b + c + d + 2) >> 2 per channel.
Every other size pair (an exact 3x included) takes the generic path, 11-bit fixed point.  Per axis, for output index d:
    scale = 1 / (dsize / ssize)                  (double)
    f = float32((d + 0.5) * scale - 0.5),  i = floor(f),  f -= i
    weights rint((1 - f) * 2048), rint(f * 2048)  (float32, half to even)
Columns: a tap with i < 0 or i >= sw - 1 takes the edge column alone (index clamped AND f = 0).
Rows: only the row indices i and i + 1 are clamped to [0, sh - 1]; f is kept.
Horizontal sum h = p[i] * a0 + p[i + 1] * a1 (int); vertical ((b0 (h0 >> 4)) >> 16) + ((b1 (h1 >> 4)) >> 16) + 2) >> 2.
An NV12 frame is resized after its cv2.cvtColor(COLOR_YUV2BGR_NV12) decode (oracle/nv12.py).
"""
import numpy as np

from .nv12 import nv12_to_bgr


def _split(dsize, ssize):
    """Source index (int64) and float32 fraction of every output index along one axis."""
    scale = 1.0 / (dsize / ssize)
    f = ((np.arange(dsize) + 0.5) * scale - 0.5).astype(np.float32)
    i = np.floor(f).astype(np.int64)
    return i, f - i.astype(np.float32)


def _weights(f):
    one, q = np.float32(1.0), np.float32(2048.0)
    return np.rint((one - f) * q).astype(np.int64), np.rint(f * q).astype(np.int64)


def taps(dsize, ssize, axis):
    """(i0, i1, w0, w1) int64 arrays over the dsize output indices; axis 'col' or 'row' picks the edge rule."""
    i, f = _split(dsize, ssize)
    if axis == "col":
        edge = (i < 0) | (i >= ssize - 1)
        f = np.where(edge, np.float32(0.0), f)
        i = np.clip(i, 0, ssize - 1)
        i0, i1 = i, np.minimum(i + 1, ssize - 1)
    else:
        i0, i1 = np.clip(i, 0, ssize - 1), np.clip(i + 1, 0, ssize - 1)
    w0, w1 = _weights(f)
    return i0, i1, w0, w1


def resize_bgr(img, size):
    """(sh, sw, C) uint8 -> (dh, dw, C) uint8 of size = (dw, dh)."""
    img = np.asarray(img)
    dw, dh = size
    sh, sw = img.shape[:2]
    src = img.astype(np.int64)
    if sw == 2 * dw and sh == 2 * dh:
        s = src[0::2, 0::2] + src[0::2, 1::2] + src[1::2, 0::2] + src[1::2, 1::2]
        return ((s + 2) >> 2).astype(np.uint8)
    x0, x1, a0, a1 = taps(dw, sw, "col")
    y0, y1, b0, b1 = taps(dh, sh, "row")
    h = src[:, x0] * a0[:, None] + src[:, x1] * a1[:, None]          # (sh, dw, C)
    b0, b1 = b0[:, None, None], b1[:, None, None]
    out = (((b0 * (h[y0] >> 4)) >> 16) + ((b1 * (h[y1] >> 4)) >> 16) + 2) >> 2
    return out.astype(np.uint8)


def resize_nv12(yuv, size):
    """(3H/2, W) uint8 NV12 -> cv2.resize(cv2.cvtColor(yuv, COLOR_YUV2BGR_NV12), size) as (dh, dw, 3) uint8."""
    return resize_bgr(nv12_to_bgr(yuv), size)
