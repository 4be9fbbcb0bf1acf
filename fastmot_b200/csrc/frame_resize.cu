// Frame resize (HBM-bound, one pass): cv2.resize(frame, (dw, dh)) with the default INTER_LINEAR into a tight BGR u8
// frame, for cameras that capture at another size than the one they are tracked at.  A frame of any pixel format
// (FmFrame) is read in place; each YUV tap is converted to BGR before it is interpolated (pixel_src.cuh), so the result
// is cv2.resize of the frame's cv2.cvtColor decode.
//   * exactly 2x smaller in both axes: OpenCV takes its 2x2 area path, (a + b + c + d + 2) >> 2 per channel;
//   * any other size pair: the generic 11-bit fixed-point path of cv_linear.cuh (an exact 3x is NOT special-cased).
// One thread per output pixel; the three bytes of consecutive pixels are consecutive, so a warp stores 96 contiguous
// bytes per row segment.
#include "common.cuh"
#include "../../include/fastmot_b200.h"
#include "pixel_src.cuh"
#include "cv_linear.cuh"

namespace {

template <class Src>
__global__ void __launch_bounds__(256) frame_resize_linear_kernel(Src src, int sw, int sh,
                                                                   unsigned char* __restrict__ dst, int dw, int dh,
                                                                   double scale_x, double scale_y) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= dw) return;
    const FmLinearTap c = fm_linear_col(x, scale_x, sw), r = fm_linear_row(y, scale_y, sh);
    int p00[3], p01[3], p10[3], p11[3];
    src.px(c.i0, r.i0, p00);
    src.px(c.i1, r.i0, p01);
    src.px(c.i0, r.i1, p10);
    src.px(c.i1, r.i1, p11);
    unsigned char* o = dst + ((size_t)y * dw + x) * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k)
        o[k] = fm_linear_v(r, p00[k] * c.w0 + p01[k] * c.w1, p10[k] * c.w0 + p11[k] * c.w1);
}

// sw == 2 * dw and sh == 2 * dh: output pixel (x, y) is the rounded mean of the 2x2 block at (2x, 2y)
template <class Src>
__global__ void __launch_bounds__(256) frame_resize_half_kernel(Src src, unsigned char* __restrict__ dst, int dw,
                                                                 int dh) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= dw) return;
    int a[3], b[3], c[3], d[3];
    src.px(2 * x, 2 * y, a);
    src.px(2 * x + 1, 2 * y, b);
    src.px(2 * x, 2 * y + 1, c);
    src.px(2 * x + 1, 2 * y + 1, d);
    unsigned char* o = dst + ((size_t)y * dw + x) * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) o[k] = (a[k] + b[k] + c[k] + d[k] + 2) >> 2;
}

}  // namespace

extern "C" int fm_frame_resize(const FmFrame* src, unsigned char* dst, int dw, int dh, void* stream) {
    FM_REQUIRE(src && fm_frame_ok(*src), "fm_frame_resize: " FM_FRAME_RULES);
    FM_REQUIRE(dst != nullptr, "fm_frame_resize: dst is NULL");
    FM_REQUIRE(dw > 0 && dh > 0 && dh <= 65535, "fm_frame_resize: the output size must be dw > 0, 0 < dh <= 65535");
    const int sw = src->w, sh = src->h;
    const dim3 grid(fm_cdiv(dw, 256), dh);
    const cudaStream_t s = (cudaStream_t)stream;
    const bool half = sw == 2 * dw && sh == 2 * dh;
    const double scale_x = 1.0 / ((double)dw / sw), scale_y = 1.0 / ((double)dh / sh);
    fm_visit_src(*src, [&](auto px) {
        if (half)
            frame_resize_half_kernel<<<grid, 256, 0, s>>>(px, dst, dw, dh);
        else
            frame_resize_linear_kernel<<<grid, 256, 0, s>>>(px, sw, sh, dst, dw, dh, scale_x, scale_y);
    });
    FM_CHECK_LAUNCH("fm_frame_resize");
    return FM_OK;
}
