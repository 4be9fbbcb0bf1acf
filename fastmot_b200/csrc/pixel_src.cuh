// Pixel sources of the kernels that read camera frames (letterbox, ReID crops, KLT gray image).  Each source hands
// out one pixel as B, G, R ints:
//   BgrSrc  : u8 HWC BGR, tight rows (w * 3 bytes);
//   Nv12Src : NV12 -- a Y plane and a half-resolution interleaved UV plane, each with its own row pitch in bytes.  The
//             pixel is converted inline exactly as OpenCV 4.13's cvtColor(COLOR_YUV2BGR_NV12) does: fixed point with
//             20 fractional bits, chroma of the pixel's 2x2 block (nearest neighbour).  Pinned against cv2 on all
//             2^24 (Y, U, V) triples by tests/test_nv12_cpu.py through the restatement in oracle/nv12.py.
#pragma once
#include "../../include/fastmot_b200.h"

__device__ __forceinline__ int fm_clamp_u8(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

__device__ __forceinline__ void fm_yuv_to_bgr(int Y, int U, int V, int v[3]) {
    const int u = U - 128, w = V - 128;
    const int y = (Y > 16 ? Y - 16 : 0) * 1220542 + (1 << 19);
    v[0] = fm_clamp_u8((y + 2116026 * u) >> 20);
    v[1] = fm_clamp_u8((y - 852492 * w - 409993 * u) >> 20);
    v[2] = fm_clamp_u8((y + 1673527 * w) >> 20);
}

struct BgrSrc {
    const unsigned char* p;
    int w;
    __device__ __forceinline__ void px(int x, int y, int v[3]) const {
        const unsigned char* q = p + ((size_t)y * w + x) * 3;
        v[0] = q[0]; v[1] = q[1]; v[2] = q[2];
    }
};

struct Nv12Src {
    const unsigned char* y;
    const unsigned char* uv;
    int y_pitch, uv_pitch;
    __device__ __forceinline__ void px(int x, int r, int v[3]) const {
        const unsigned char* c = uv + (size_t)(r >> 1) * uv_pitch + (x & ~1);
        fm_yuv_to_bgr(y[(size_t)r * y_pitch + x], c[0], c[1], v);
    }
};

// The pixel source of an FmFrame: returns f(BgrSrc{...}) or f(Nv12Src{...}) (an NV12 pitch of 0 means w).
template <class F>
__host__ __device__ __forceinline__ auto fm_visit_src(const FmFrame& fr, F&& f) {
    if (fr.format == FM_PIX_NV12)
        return f(Nv12Src{fr.y, fr.uv, fr.pitch ? fr.pitch : fr.w, fr.uv_pitch ? fr.uv_pitch : fr.w});
    return f(BgrSrc{fr.y, fr.w});
}

// what every one-frame entry point requires of its frame (include/fastmot_b200.h: FmFrame)
static inline bool fm_frame_ok(const FmFrame& f) {
    if (!f.y || f.w <= 0 || f.h <= 0) return false;
    if (f.format == FM_PIX_BGR) return true;
    return f.format == FM_PIX_NV12 && f.uv && f.w % 2 == 0 && f.h % 2 == 0 && (f.pitch == 0 || f.pitch >= f.w) &&
           (f.uv_pitch == 0 || f.uv_pitch >= f.w);
}
#define FM_FRAME_RULES "a BGR frame needs y and w, h > 0; an NV12 frame both planes, even w, h > 0 and pitches >= w"
