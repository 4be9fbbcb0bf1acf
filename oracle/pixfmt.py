"""I420, YUY2 and BGRx -> BGR as OpenCV 4.13's cv2.cvtColor computes them, restated in NumPy, and the cv2 encoders the
tests build such frames with.

I420 and YUY2 use the BT.601 limited-range integer formula of oracle/nv12.py (yuv_to_bgr); only the sampling differs:
  I420 (COLOR_YUV2BGR_I420): (3H/2, W) -- H rows of Y, then the U plane and the V plane, each H/2 x W/2 stored as H/4
       rows of W bytes; the chroma of the pixel's 2x2 block (nearest neighbour), as NV12.
  YUY2 (COLOR_YUV2BGR_YUY2): (H, W, 2) -- each row is Y0 U Y1 V per pixel pair; pixels 2i and 2i + 1 share U and V.
  BGRx (COLOR_BGRA2BGR): (H, W, 4) -- the fourth byte is dropped.
The GPU kernels read the same layouts in place (fastmot_b200/csrc/pixel_src.cuh).
"""
import numpy as np

from .nv12 import yuv_to_bgr


def _bgr(Y, U, V):
    return np.stack(yuv_to_bgr(Y, U, V), -1).astype(np.uint8)


def i420_to_bgr(yuv):
    """(3H/2, W) uint8 I420 frame -> (H, W, 3) uint8 BGR."""
    yuv = np.asarray(yuv)
    h, w = yuv.shape[0] * 2 // 3, yuv.shape[1]
    q = h * w // 4
    chroma = yuv[h:].reshape(-1)
    U = chroma[:q].reshape(h // 2, w // 2)
    V = chroma[q:].reshape(h // 2, w // 2)
    up = lambda c: np.repeat(np.repeat(c, 2, 0), 2, 1)
    return _bgr(yuv[:h], up(U), up(V))


def yuy2_to_bgr(yuy2):
    """(H, W, 2) uint8 YUY2 frame -> (H, W, 3) uint8 BGR."""
    yuy2 = np.asarray(yuy2)
    pairs = yuy2.reshape(yuy2.shape[0], -1, 4)          # Y0 U Y1 V
    U = np.repeat(pairs[..., 1], 2, 1)
    V = np.repeat(pairs[..., 3], 2, 1)
    return _bgr(yuy2[..., 0], U, V)


def bgrx_to_bgr(bgrx):
    """(H, W, 4) uint8 BGRx frame -> (H, W, 3) uint8 BGR."""
    return np.ascontiguousarray(np.asarray(bgrx)[..., :3])


def bgr_to_i420(bgr):
    """(H, W, 3) uint8 BGR (H, W even) -> (3H/2, W) uint8 I420 (cv2.COLOR_BGR2YUV_I420)."""
    import cv2
    return cv2.cvtColor(np.ascontiguousarray(bgr), cv2.COLOR_BGR2YUV_I420)


def bgr_to_yuy2(bgr):
    """(H, W, 3) uint8 BGR (W even) -> (H, W, 2) uint8 YUY2 (cv2.COLOR_BGR2YUV_YUY2)."""
    import cv2
    return cv2.cvtColor(np.ascontiguousarray(bgr), cv2.COLOR_BGR2YUV_YUY2)


def bgr_to_bgrx(bgr, x=0):
    """(H, W, 3) uint8 BGR -> (H, W, 4) uint8 BGRx (cv2.COLOR_BGR2BGRA) with the fourth byte set to x."""
    import cv2
    out = cv2.cvtColor(np.ascontiguousarray(bgr), cv2.COLOR_BGR2BGRA)
    out[..., 3] = x
    return out


# format -> (cv2 decode code name, NumPy restatement, cv2-based encoder)
DECODES = {"I420": ("COLOR_YUV2BGR_I420", i420_to_bgr, bgr_to_i420),
           "YUY2": ("COLOR_YUV2BGR_YUY2", yuy2_to_bgr, bgr_to_yuy2),
           "BGRX": ("COLOR_BGRA2BGR", bgrx_to_bgr, bgr_to_bgrx)}


def cv2_decode(frame, fmt):
    """cv2.cvtColor(frame, code) with the decode code of `fmt` (also 'NV12'; 'BGR' passes through)."""
    import cv2
    if fmt == "BGR":
        return frame
    code = "COLOR_YUV2BGR_NV12" if fmt == "NV12" else DECODES[fmt][0]
    return cv2.cvtColor(frame, getattr(cv2, code))
