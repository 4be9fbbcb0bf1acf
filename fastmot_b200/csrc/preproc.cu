// Image pre-processing kernels (HBM-bound, one pass each):
//   fm_letterbox_preproc : BGR u8 HWC frame -> bilinear resize (half-pixel centres, edge replicate, rounded to u8)
//                          -> RGB, x/255, letterbox pad 0.5   (fastmot/detector.py:289-320)
//   fm_roi_resize_norm   : per-detection crop + OpenCV-style fixed-point bilinear resize to 128x256 + ImageNet
//                          normalisation, all crops in one launch (fastmot/feature_extractor.py:48-60, 84-98;
//                          fastmot/utils/rect.py:92-97)
// Both read a frame of any pixel format (FmFrame) in place; a YUV bilinear tap is converted to BGR before it is
// interpolated (pixel_src.cuh).  The *_geom entries read each frame (and, for the letterbox, its ROI) from a device
// FmFrameGeom table (one grid slice per frame, or one frame index per crop), so one launch covers several frames of
// any sizes and formats; every pixel is computed by the same body as in the one-frame entries.
// Outputs are either fp32 planar CHW (the reference's TensorRT input layout; used for parity tests) or fp16
// NHWC with C padded to 8 (one 16-byte chunk per pixel; what the conv engine consumes).
#include "common.cuh"
#include "../../include/fastmot_b200.h"
#include "pixel_src.cuh"

namespace {

template <int LAYOUT>  // 0: fp32 CHW, 1: fp16 NHWC8, 2: fp16 NHWC4 inside a 4-pixel zero border ([H + 8][W + 8][4])
__device__ __forceinline__ void store_px(void* out, int H, int W, int y, int x, float r, float g, float b) {
    if (LAYOUT == 2) {
        // 8 bytes per pixel; the border (never written here, zeroed once by the owner of the buffer) is the zero
        // padding of the 7x7 stem, so its TMA tiles need no bounds handling (csrc/osnet_stem.cu)
        __align__(8) __half2 v[2];
        v[0] = __floats2half2_rn(r, g);
        v[1] = __floats2half2_rn(b, 0.0f);
        *reinterpret_cast<int2*>((__half*)out + ((size_t)(y + 4) * (W + 8) + x + 4) * 4) = *reinterpret_cast<const int2*>(v);
    } else if (LAYOUT == 0) {
        float* o = (float*)out;
        size_t plane = (size_t)H * W, p = (size_t)y * W + x;
        o[p] = r; o[plane + p] = g; o[2 * plane + p] = b;
    } else {
        // 8 channels = one 16-byte chunk per pixel: the tensor-core conv gathers operands in 16-byte units
        __align__(16) __half2 v[4];
        v[0] = __floats2half2_rn(r, g);
        v[1] = __floats2half2_rn(b, 0.0f);
        v[2] = __floats2half2_rn(0.0f, 0.0f);
        v[3] = v[2];
        *reinterpret_cast<int4*>((__half*)out + ((size_t)y * W + x) * 8) = *reinterpret_cast<const int4*>(v);
    }
}

// One output pixel (x, y) of the letterbox of a src_w x src_h frame read through `src`.
template <int LAYOUT, class Src>
__device__ __forceinline__ void letterbox_px(const Src& src, int src_w, int src_h, int dst_w, int dst_h, int roi_x,
                                             int roi_y, int roi_w, int roi_h, void* out, int x, int y) {
    const int rx = x - roi_x, ry = y - roi_y;
    if (rx < 0 || ry < 0 || rx >= roi_w || ry >= roi_h) {
        store_px<LAYOUT>(out, dst_h, dst_w, y, x, 0.5f, 0.5f, 0.5f);  // detector.py:318
        return;
    }
    // zoom(order=1, mode='opencv', grid_mode=True): half-pixel centres, clamp, linear in double, rint -> u8
    const double zx = (double)src_w / roi_w, zy = (double)src_h / roi_h;
    double sx = (rx + 0.5) * zx - 0.5, sy = (ry + 0.5) * zy - 0.5;
    sx = fmin(fmax(sx, 0.0), (double)(src_w - 1));
    sy = fmin(fmax(sy, 0.0), (double)(src_h - 1));
    const int x0 = (int)floor(sx), y0 = (int)floor(sy);
    const int x1 = min(x0 + 1, src_w - 1), y1 = min(y0 + 1, src_h - 1);
    const double fx = sx - x0, fy = sy - y0;
    // each tap is a BGR pixel before interpolation (a YUV tap is converted with its own chroma)
    int p00[3], p01[3], p10[3], p11[3];
    src.px(x0, y0, p00);
    src.px(x1, y0, p01);
    src.px(x0, y1, p10);
    src.px(x1, y1, p11);
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        double top = p00[c] * (1.0 - fx) + p01[c] * fx;
        double bot = p10[c] * (1.0 - fx) + p11[c] * fx;
        double val = rint(top * (1.0 - fy) + bot * fy);           // stays uint8 in the reference
        v[c] = (float)(val * (1.0 / 255.0));                      // cp.multiply(u8, 1/255.) -> f32
    }
    store_px<LAYOUT>(out, dst_h, dst_w, y, x, v[2], v[1], v[0]);  // BGR -> RGB
}

template <int LAYOUT, class Src>
__global__ void __launch_bounds__(256) letterbox_kernel(Src src, int src_w, int src_h, int dst_w, int dst_h, int roi_x,
                                                         int roi_y, int roi_w, int roi_h, void* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= dst_w) return;
    letterbox_px<LAYOUT>(src, src_w, src_h, dst_w, dst_h, roi_x, roi_y, roi_w, roi_h, out, x, blockIdx.y);
}

// image blockIdx.z takes its frame (any pixel format), size and ROI from geom[blockIdx.z] and writes the blockIdx.z-th
// NHWC8 image of out
__global__ void __launch_bounds__(256) letterbox_geom_kernel(const FmFrameGeom* __restrict__ geom, int dst_w,
                                                              int dst_h, void* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= dst_w) return;
    const FmFrameGeom& g = geom[blockIdx.z];
    out = (__half*)out + (size_t)blockIdx.z * dst_h * dst_w * 8;
    fm_visit_src(g.frame, [&](const auto& src) {
        letterbox_px<1>(src, g.frame.w, g.frame.h, dst_w, dst_h, g.roi_x, g.roi_y, g.roi_w, g.roi_h, out, x,
                        blockIdx.y);
    });
}

// OpenCV INTER_LINEAR for 8-bit: 11-bit fixed-point coefficients, horizontal pass in int, vertical pass
// ((b0*(S0>>4))>>16 + (b1*(S1>>4))>>16 + 2) >> 2.
__device__ __forceinline__ void cv_coef(int d, double scale, int ssize, int& s, int& a0, int& a1) {
    float f = (float)((d + 0.5) * scale - 0.5);
    int si = (int)floorf(f);
    f -= si;
    if (si < 0) { f = 0.f; si = 0; }
    if (si >= ssize - 1) { f = 0.f; si = ssize - 1; }
    s = si;
    a0 = (int)rintf((1.f - f) * 2048.f);
    a1 = (int)rintf(f * 2048.f);
}

// Crop `crop` of a src_w x src_h frame read through `src`, output pixel (x, y).
template <int LAYOUT, class Src>
__device__ __forceinline__ void roi_px(const Src& src, int src_w, int src_h, const double* __restrict__ tlbrs, int crop,
                                       int out_w, int out_h, void* __restrict__ out, int x, int y) {
    // multi_crop (rect.py:92-97): truncate toward zero, clamp lower bound to 0; numpy slicing clamps the upper
    const double* b = tlbrs + (size_t)crop * 4;
    int cx0 = max((int)b[0], 0), cy0 = max((int)b[1], 0);
    int cx1 = min(max((int)b[2], 0), src_w - 1), cy1 = min(max((int)b[3], 0), src_h - 1);
    cx0 = min(cx0, src_w - 1); cy0 = min(cy0, src_h - 1);
    const int cw = max(cx1 - cx0 + 1, 1), ch = max(cy1 - cy0 + 1, 1);
    int sx, sy, a0, a1, b0, b1;
    cv_coef(x, (double)cw / out_w, cw, sx, a0, a1);
    cv_coef(y, (double)ch / out_h, ch, sy, b0, b1);
    const int sx1 = min(sx + 1, cw - 1), sy1 = min(sy + 1, ch - 1);
    // each tap is a BGR pixel before interpolation (a YUV tap is converted with its own chroma)
    int p00[3], p01[3], p10[3], p11[3];
    src.px(cx0 + sx, cy0 + sy, p00);
    src.px(cx0 + sx1, cy0 + sy, p01);
    src.px(cx0 + sx, cy0 + sy1, p10);
    src.px(cx0 + sx1, cy0 + sy1, p11);
    float v[3];
    const float mean[3] = {0.406f, 0.456f, 0.485f};   // indexed by BGR channel
    const float stdv[3] = {0.225f, 0.224f, 0.229f};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        int h0 = p00[c] * a0 + p01[c] * a1;
        int h1 = p10[c] * a0 + p11[c] * a1;
        int px = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
        px = min(max(px, 0), 255);
        v[c] = (float)(((double)px / 255.0 - (double)mean[c]) / (double)stdv[c]);
    }
    void* o = LAYOUT == 0 ? (void*)((float*)out + (size_t)crop * 3 * out_h * out_w)
              : LAYOUT == 1 ? (void*)((__half*)out + (size_t)crop * 8 * out_h * out_w)
                            : (void*)((__half*)out + (size_t)crop * 4 * (out_h + 8) * (out_w + 8));
    store_px<LAYOUT>(o, out_h, out_w, y, x, v[2], v[1], v[0]);
}

template <int LAYOUT, class Src>
__global__ void __launch_bounds__(128) roi_resize_norm_kernel(Src src, int src_w, int src_h,
                                                               const double* __restrict__ tlbrs,
                                                               const int* __restrict__ n_ptr, int n_max, int out_w,
                                                               int out_h, void* __restrict__ out) {
    const int crop = blockIdx.z;
    const int n = n_ptr ? min(*n_ptr, n_max) : n_max;
    if (crop >= n) return;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= out_w) return;
    roi_px<LAYOUT>(src, src_w, src_h, tlbrs, crop, out_w, out_h, out, x, blockIdx.y);
}

// crop i is cut from geom[frame_idx[i]]'s frame (any pixel format), with that frame's own width and height
template <int LAYOUT>
__global__ void __launch_bounds__(128) roi_resize_norm_geom_kernel(const FmFrameGeom* __restrict__ geom,
                                                                    const int* __restrict__ frame_idx,
                                                                    const double* __restrict__ tlbrs, int n, int out_w,
                                                                    int out_h, void* __restrict__ out) {
    const int crop = blockIdx.z;
    if (crop >= n) return;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= out_w) return;
    const FmFrame& f = geom[frame_idx[crop]].frame;
    fm_visit_src(f, [&](const auto& src) {
        roi_px<LAYOUT>(src, f.w, f.h, tlbrs, crop, out_w, out_h, out, x, blockIdx.y);
    });
}

}  // namespace

extern "C" int fm_letterbox_preproc(const FmFrame* frame, int dst_w, int dst_h, int roi_x, int roi_y, int roi_w,
                                    int roi_h, int layout, void* out, void* stream) {
    FM_REQUIRE(frame && fm_frame_ok(*frame), "fm_letterbox_preproc: " FM_FRAME_RULES);
    FM_REQUIRE(layout == 0 || layout == 1, "fm_letterbox_preproc: layout must be 0 (f32 CHW) or 1 (f16 NHWC8)");
    FM_REQUIRE(roi_w > 0 && roi_h > 0, "fm_letterbox_preproc: empty ROI");
    const dim3 grid(fm_cdiv(dst_w, 256), dst_h);
    const int w = frame->w, h = frame->h;
    fm_visit_src(*frame, [&](auto src) {
        if (layout == 0)
            letterbox_kernel<0><<<grid, 256, 0, (cudaStream_t)stream>>>(src, w, h, dst_w, dst_h, roi_x, roi_y, roi_w,
                                                                        roi_h, out);
        else
            letterbox_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(src, w, h, dst_w, dst_h, roi_x, roi_y, roi_w,
                                                                        roi_h, out);
    });
    FM_CHECK_LAUNCH("fm_letterbox_preproc");
    return FM_OK;
}

extern "C" int fm_roi_resize_norm(const FmFrame* frame, const double* tlbrs, const int* n_dev, int n_max, int out_w,
                                  int out_h, int layout, void* out, void* stream) {
    FM_REQUIRE(frame && fm_frame_ok(*frame), "fm_roi_resize_norm: " FM_FRAME_RULES);
    FM_REQUIRE(layout >= 0 && layout <= 2, "fm_roi_resize_norm: layout must be 0 (f32 CHW), 1 (f16 NHWC8) or 2 (f16 NHWC4, padded)");
    if (n_max <= 0) return FM_OK;
    FM_REQUIRE(n_max <= 65535, "fm_roi_resize_norm: more than 65535 crops");
    const dim3 grid(fm_cdiv(out_w, 128), out_h, n_max);
    const int w = frame->w, h = frame->h;
    fm_visit_src(*frame, [&](auto src) {
        if (layout == 0)
            roi_resize_norm_kernel<0><<<grid, 128, 0, (cudaStream_t)stream>>>(src, w, h, tlbrs, n_dev, n_max, out_w,
                                                                              out_h, out);
        else if (layout == 1)
            roi_resize_norm_kernel<1><<<grid, 128, 0, (cudaStream_t)stream>>>(src, w, h, tlbrs, n_dev, n_max, out_w,
                                                                              out_h, out);
        else
            roi_resize_norm_kernel<2><<<grid, 128, 0, (cudaStream_t)stream>>>(src, w, h, tlbrs, n_dev, n_max, out_w,
                                                                              out_h, out);
    });
    FM_CHECK_LAUNCH("fm_roi_resize_norm");
    return FM_OK;
}

extern "C" int fm_letterbox_preproc_geom(const FmFrameGeom* geom, int batch, int dst_w, int dst_h, void* out,
                                         void* stream) {
    FM_REQUIRE(geom != nullptr, "fm_letterbox_preproc_geom: geometry table is NULL");
    FM_REQUIRE(batch > 0 && batch <= 65535, "fm_letterbox_preproc_geom: batch must be in [1, 65535]");
    dim3 grid(fm_cdiv(dst_w, 256), dst_h, batch);
    letterbox_geom_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(geom, dst_w, dst_h, out);
    FM_CHECK_LAUNCH("fm_letterbox_preproc_geom");
    return FM_OK;
}

extern "C" int fm_roi_resize_norm_geom(const FmFrameGeom* geom, const int* frame_idx, const double* tlbrs, int n,
                                       int out_w, int out_h, int layout, void* out, void* stream) {
    FM_REQUIRE(layout >= 0 && layout <= 2, "fm_roi_resize_norm_geom: layout must be 0 (f32 CHW), 1 (f16 NHWC8) or 2 (f16 NHWC4, padded)");
    if (n <= 0) return FM_OK;
    FM_REQUIRE(geom != nullptr && frame_idx != nullptr, "fm_roi_resize_norm_geom: geometry table or index is NULL");
    FM_REQUIRE(n <= 65535, "fm_roi_resize_norm_geom: more than 65535 crops");
    dim3 grid(fm_cdiv(out_w, 128), out_h, n);
    if (layout == 0)
        roi_resize_norm_geom_kernel<0><<<grid, 128, 0, (cudaStream_t)stream>>>(geom, frame_idx, tlbrs, n, out_w, out_h,
                                                                               out);
    else if (layout == 1)
        roi_resize_norm_geom_kernel<1><<<grid, 128, 0, (cudaStream_t)stream>>>(geom, frame_idx, tlbrs, n, out_w, out_h,
                                                                               out);
    else
        roi_resize_norm_geom_kernel<2><<<grid, 128, 0, (cudaStream_t)stream>>>(geom, frame_idx, tlbrs, n, out_w, out_h,
                                                                               out);
    FM_CHECK_LAUNCH("fm_roi_resize_norm_geom");
    return FM_OK;
}
