"""NV12 -> BGR as OpenCV 4.13's cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_NV12) computes it, restated in NumPy.

Per pixel, with the chroma (U, V) of the pixel's 2x2 block (nearest neighbour), u = U - 128, v = V - 128 and
y = max(Y - 16, 0) * 1220542 + 2^19 (BT.601 limited range, 20 fractional bits):
    B = clamp((y + 2116026 u) >> 20)   G = clamp((y - 852492 v - 409993 u) >> 20)   R = clamp((y + 1673527 v) >> 20)
The GPU kernels convert inline with the same integers (fastmot_b200/csrc/pixel_src.cuh).
"""
import numpy as np


def yuv_to_bgr(Y, U, V):
    """Elementwise (Y, U, V) -> (B, G, R) int32 arrays in [0, 255]."""
    Y, U, V = (np.asarray(a, np.int32) for a in (Y, U, V))
    u, v = U - 128, V - 128
    y = np.maximum(Y - 16, 0) * 1220542 + (1 << 19)
    return tuple(np.clip(c >> 20, 0, 255) for c in (y + 2116026 * u, y - 852492 * v - 409993 * u, y + 1673527 * v))


def nv12_to_bgr(yuv):
    """(3H/2, W) uint8 NV12 frame -> (H, W, 3) uint8 BGR."""
    yuv = np.asarray(yuv)
    h = yuv.shape[0] * 2 // 3
    uv = yuv[h:].reshape(h // 2, -1, 2)
    U = np.repeat(np.repeat(uv[..., 0], 2, 0), 2, 1)
    V = np.repeat(np.repeat(uv[..., 1], 2, 0), 2, 1)
    return np.stack(yuv_to_bgr(yuv[:h], U, V), -1).astype(np.uint8)


def bgr_to_nv12(bgr):
    """(H, W, 3) uint8 BGR (H, W even) -> (3H/2, W) uint8 NV12: cv2's BGR -> I420 with U and V interleaved."""
    import cv2
    h, w = bgr.shape[:2]
    i420 = cv2.cvtColor(np.ascontiguousarray(bgr), cv2.COLOR_BGR2YUV_I420)
    out = np.empty((h * 3 // 2, w), np.uint8)
    out[:h] = i420[:h]
    q = h // 4
    out[h:].reshape(-1)[0::2] = i420[h:h + q].reshape(-1)
    out[h:].reshape(-1)[1::2] = i420[h + q:].reshape(-1)
    return out
