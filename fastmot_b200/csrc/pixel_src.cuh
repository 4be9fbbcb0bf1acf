// Pixel sources of the kernels that read camera frames (letterbox, ReID crops, KLT gray image, frame resize).  Each
// source hands out one pixel as B, G, R ints:
//   BgrSrc     : u8 HWC BGR, tight rows (w * 3 bytes);
//   Yuv420Src  : 4:2:0 -- a Y plane and half-resolution chroma, each with its own row pitch in bytes.  Nv12Src reads
//                one interleaved UV plane (V is the byte after U), I420Src a U and a V plane of one pitch;
//   Yuy2Src    : packed 4:2:2 -- Y0 U Y1 V per pixel pair, with a row pitch in bytes;
//   BgrxSrc    : packed B G R x, 4 bytes per pixel, with a row pitch in bytes.
// A YUV pixel is converted inline exactly as OpenCV 4.13's cvtColor(COLOR_YUV2BGR_NV12 / _I420 / _YUY2) does: fixed
// point with 20 fractional bits, the chroma of the pixel's 2x2 block (4:2:0) or pixel pair (4:2:2), nearest
// neighbour.  Pinned against cv2 on all 2^24 (Y, U, V) triples by tests/test_nv12_cpu.py and tests/test_pixfmt_cpu.py
// through the restatements in oracle/nv12.py and oracle/pixfmt.py.
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

// CSTEP: bytes from one chroma sample to the next in a chroma row -- 2 for NV12 (U at uv[2i], V at uv[2i + 1]), 1 for
// I420 (U at uv[i], V at v[i], both planes with pitch uv_pitch).  v is not read for NV12.
template <int CSTEP>
struct Yuv420Src {
    const unsigned char* y;
    const unsigned char* uv;
    int y_pitch, uv_pitch;
    const unsigned char* v;
    // offset of the chroma sample of the 2x2 block holding pixel (x, r)
    __device__ __forceinline__ size_t chroma(int x, int r) const {
        return (size_t)(r >> 1) * uv_pitch + (CSTEP == 2 ? (x & ~1) : (x >> 1));
    }
    __device__ __forceinline__ int U(size_t c) const { return uv[c]; }
    __device__ __forceinline__ int V(size_t c) const { return CSTEP == 2 ? uv[c + 1] : v[c]; }
    __device__ __forceinline__ void px(int x, int r, int o[3]) const {
        const size_t c = chroma(x, r);
        fm_yuv_to_bgr(y[(size_t)r * y_pitch + x], U(c), V(c), o);
    }
};
using Nv12Src = Yuv420Src<2>;
using I420Src = Yuv420Src<1>;

struct Yuy2Src {
    const unsigned char* p;
    int pitch;
    __device__ __forceinline__ void px(int x, int r, int v[3]) const {
        const unsigned char* q = p + (size_t)r * pitch + (x & ~1) * 2;   // Y0 U Y1 V of the pixel pair
        fm_yuv_to_bgr(q[(x & 1) * 2], q[1], q[3], v);
    }
};

struct BgrxSrc {
    const unsigned char* p;
    int pitch;
    __device__ __forceinline__ void px(int x, int r, int v[3]) const {
        const unsigned char* q = p + (size_t)r * pitch + x * 4;
        v[0] = q[0]; v[1] = q[1]; v[2] = q[2];
    }
};

// The pixel source of an FmFrame: returns f(src) for the source of its format (a pitch of 0 is the tight pitch:
// w for the Y plane of NV12 / I420, w for NV12's UV plane, w / 2 for I420's U and V planes, 2w for YUY2, 4w for BGRx).
template <class F>
__host__ __device__ __forceinline__ auto fm_visit_src(const FmFrame& fr, F&& f) {
    switch (fr.format) {
    case FM_PIX_NV12:
        return f(Nv12Src{fr.y, fr.uv, fr.pitch ? fr.pitch : fr.w, fr.uv_pitch ? fr.uv_pitch : fr.w, nullptr});
    case FM_PIX_I420:
        return f(I420Src{fr.y, fr.uv, fr.pitch ? fr.pitch : fr.w, fr.uv_pitch ? fr.uv_pitch : fr.w / 2, fr.v});
    case FM_PIX_YUY2:
        return f(Yuy2Src{fr.y, fr.pitch ? fr.pitch : 2 * fr.w});
    case FM_PIX_BGRX:
        return f(BgrxSrc{fr.y, fr.pitch ? fr.pitch : 4 * fr.w});
    default:
        return f(BgrSrc{fr.y, fr.w});
    }
}

// what every one-frame entry point requires of its frame (include/fastmot_b200.h: FmFrame)
static inline bool fm_frame_ok(const FmFrame& f) {
    if (!f.y || f.w <= 0 || f.h <= 0) return false;
    const bool even = f.w % 2 == 0 && f.h % 2 == 0;
    switch (f.format) {
    case FM_PIX_BGR:
        return true;
    case FM_PIX_NV12:
        return f.uv && even && (f.pitch == 0 || f.pitch >= f.w) && (f.uv_pitch == 0 || f.uv_pitch >= f.w);
    case FM_PIX_I420:
        return f.uv && f.v && even && (f.pitch == 0 || f.pitch >= f.w) && (f.uv_pitch == 0 || f.uv_pitch >= f.w / 2);
    case FM_PIX_YUY2:
        return f.w % 2 == 0 && (f.pitch == 0 || f.pitch >= 2 * f.w);
    case FM_PIX_BGRX:
        return f.pitch == 0 || f.pitch >= 4 * f.w;
    default:
        return false;
    }
}
#define FM_FRAME_RULES                                                                                                 \
    "a frame needs y and w, h > 0; NV12 both planes, even w and h, pitches >= w; I420 the Y, U and V planes, even w "  \
    "and h, pitch >= w, uv_pitch >= w / 2; YUY2 an even w, pitch >= 2w; BGRx pitch >= 4w"
