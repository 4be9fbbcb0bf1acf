// KLT image pyramid kernels (byte work, HBM/L2-bound): BGR->gray + 0.5x box mean in one pass, BGR->gray + an
// INTER_LINEAR resize to any optical-flow size (both also reading YUV and BGRx frames in place, pixel_src.cuh),
// 5-tap Gaussian pyrDown, int16 Scharr derivatives, background-scale image + mask.
//
// Reference: fastmot/flow.py:121-133, 153-154, 187-189 (cv2.cvtColor / cv2.resize) and the pyramid that
// cv2.calcOpticalFlowPyrLK builds internally (flow.py:203-207; OpenCV lkpyramid.cpp: buildOpticalFlowPyramid,
// calcScharrDeriv).  Fixed-point formulas restated in SURVEY.md Appendix C.
#include "common.cuh"
#include "../../include/fastmot_b200.h"
#include "pixel_src.cuh"
#include "cv_linear.cuh"

namespace {

__device__ __forceinline__ int gray_of(const int p[3]) {
    // OpenCV 4.13 BGR2GRAY, 15-bit fixed point (pinned against cv2.cvtColor: 0 mismatches on 1M random pixels;
    // the 14-bit constants 1868/9617/4899 quoted in SURVEY.md Appendix C differ on 0.2 % of pixels)
    return (p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + 16384) >> 15;
}

// The four pixels of the 2x2 block at (x0, y0) (x1 = x0 + 1, y1 = y0 + 1 inside the frame; w and h are even).
template <class Src>
__device__ __forceinline__ void block_bgr(const Src& s, int x0, int y0, int x1, int y1, int a[3], int b[3], int c[3],
                                          int d[3]) {
    s.px(x0, y0, a); s.px(x1, y0, b); s.px(x0, y1, c); s.px(x1, y1, d);
}

// A 4:2:0 2x2 block at even (x0, y0) is exactly one chroma sample: one U and one V load for the four pixels.
template <int CSTEP>
__device__ __forceinline__ void block_bgr(const Yuv420Src<CSTEP>& s, int x0, int y0, int x1, int y1, int a[3],
                                          int b[3], int c[3], int d[3]) {
    const size_t q = s.chroma(x0, y0);
    const int U = s.U(q), V = s.V(q);
    const unsigned char* r0 = s.y + (size_t)y0 * s.y_pitch;
    const unsigned char* r1 = s.y + (size_t)y1 * s.y_pitch;
    fm_yuv_to_bgr(r0[x0], U, V, a); fm_yuv_to_bgr(r0[x1], U, V, b);
    fm_yuv_to_bgr(r1[x0], U, V, c); fm_yuv_to_bgr(r1[x1], U, V, d);
}

// A YUY2 2x2 block at even (x0, y0) is one pixel pair per row: one Y0 U Y1 V group each.
__device__ __forceinline__ void block_bgr(const Yuy2Src& s, int x0, int y0, int x1, int y1, int a[3], int b[3],
                                          int c[3], int d[3]) {
    const unsigned char* q0 = s.p + (size_t)y0 * s.pitch + x0 * 2;
    const unsigned char* q1 = s.p + (size_t)y1 * s.pitch + x0 * 2;
    fm_yuv_to_bgr(q0[0], q0[1], q0[3], a); fm_yuv_to_bgr(q0[2], q0[1], q0[3], b);
    fm_yuv_to_bgr(q1[0], q1[1], q1[3], c); fm_yuv_to_bgr(q1[2], q1[1], q1[3], d);
}

// One thread per 2x2 block of the full-resolution frame.
template <class Src>
__global__ void __launch_bounds__(256) gray_half_kernel(Src src, int w, int h, unsigned char* __restrict__ gray,
                                                         unsigned char* __restrict__ small, int sw, int sh) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;  // small coords
    const int y = blockIdx.y;
    if (x >= sw || y >= sh) return;
    const int x0 = 2 * x, y0 = 2 * y;
    const int x1 = min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1);
    int pa[3], pb[3], pc[3], pd[3];
    block_bgr(src, x0, y0, x1, y1, pa, pb, pc, pd);
    const int a = gray_of(pa), b = gray_of(pb);
    const int c = gray_of(pc), d = gray_of(pd);
    gray[(size_t)y0 * w + x0] = a;
    gray[(size_t)y0 * w + x1] = b;
    gray[(size_t)y1 * w + x0] = c;
    gray[(size_t)y1 * w + x1] = d;
    small[(size_t)y * sw + x] = (a + b + c + d + 2) >> 2;  // cv2.resize INTER_LINEAR at exactly 0.5x
}

template <class Src>
__global__ void __launch_bounds__(256) gray_kernel(Src src, int w, int h, unsigned char* __restrict__ gray) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= w || y >= h) return;
    int p[3];
    src.px(x, y, p);
    gray[(size_t)y * w + x] = gray_of(p);
}

// cv2.resize(src, (dw, dh)) INTER_LINEAR for u8 at a downscale (dw <= sw, dh <= sh): OpenCV's generic resize with
// 11-bit coefficients (cv_linear.cuh, shared with fm_frame_resize).
__global__ void __launch_bounds__(256) resize_linear_kernel(const unsigned char* __restrict__ src, int sw, int sh,
                                                             unsigned char* __restrict__ dst, int dw, int dh,
                                                             double scale_x, double scale_y) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= dw || y >= dh) return;
    const FmLinearTap c = fm_linear_col(x, scale_x, sw), r = fm_linear_row(y, scale_y, sh);
    const unsigned char* r0 = src + (size_t)r.i0 * sw;
    const unsigned char* r1 = src + (size_t)r.i1 * sw;
    const int h0 = r0[c.i0] * c.w0 + r0[c.i1] * c.w1, h1 = r1[c.i0] * c.w0 + r1[c.i1] * c.w1;
    dst[(size_t)y * dw + x] = fm_linear_v(r, h0, h1);
}

__device__ __forceinline__ int reflect101(int p, int n) {
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = p < 0 ? -p : 2 * n - 2 - p;
    return p;
}

// pyrDown: dst(x,y) = (sum_{i,j} g[i] g[j] src(2x+i-2, 2y+j-2) + 128) >> 8, g = [1 4 6 4 1], BORDER_REFLECT_101
__global__ void __launch_bounds__(256) pyr_down_kernel(const unsigned char* __restrict__ src, int sw, int sh,
                                                        unsigned char* __restrict__ dst, int dw, int dh) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= dw || y >= dh) return;
    const int g[5] = {1, 4, 6, 4, 1};
    int acc = 0;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const unsigned char* row = src + (size_t)reflect101(2 * y + j - 2, sh) * sw;
        int racc = 0;
#pragma unroll
        for (int i = 0; i < 5; ++i) racc += g[i] * row[reflect101(2 * x + i - 2, sw)];
        acc += g[j] * racc;
    }
    dst[(size_t)y * dw + x] = (acc + 128) >> 8;
}

// calcScharrDeriv: vertical [3 10 3] smoothing / [-1 0 1] diff first, then horizontal; reflect-101 borders.
__global__ void __launch_bounds__(256) scharr_kernel(const unsigned char* __restrict__ src, int w, int h,
                                                      short2* __restrict__ deriv) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= w || y >= h) return;
    const unsigned char* r0 = src + (size_t)reflect101(y - 1, h) * w;
    const unsigned char* r1 = src + (size_t)y * w;
    const unsigned char* r2 = src + (size_t)reflect101(y + 1, h) * w;
    const int xm = reflect101(x - 1, w), xp = reflect101(x + 1, w);
    const int s_m = (r0[xm] + r2[xm]) * 3 + r1[xm] * 10, s_p = (r0[xp] + r2[xp]) * 3 + r1[xp] * 10;
    const int d_m = r2[xm] - r0[xm], d_c = r2[x] - r0[x], d_p = r2[xp] - r0[xp];
    deriv[(size_t)y * w + x] = make_short2((short)(s_p - s_m), (short)((d_p + d_m) * 3 + d_c * 10));
}

// Background image (cv2.resize INTER_LINEAR, cv_linear.cuh) and its mask, cv2.resize INTER_NEAREST of the owner map
// (FM_NO_OWNER is background, 255).  scale_x / scale_y are OpenCV's 1 / (dsize / ssize); INTER_NEAREST samples source
// index floor(d * scale), which differs from floor(d * ssize / dsize) wherever the exact product is an integer.
__global__ void bg_small_kernel(const unsigned char* __restrict__ gray, const int* __restrict__ owner, int w, int h,
                                unsigned char* __restrict__ bg, unsigned char* __restrict__ bg_mask, int bw, int bh,
                                double scale_x, double scale_y) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= bw || y >= bh) return;
    const FmLinearTap c = fm_linear_col(x, scale_x, w), r = fm_linear_row(y, scale_y, h);
    const unsigned char* r0 = gray + (size_t)r.i0 * w;
    const unsigned char* r1 = gray + (size_t)r.i1 * w;
    const int h0 = r0[c.i0] * c.w0 + r0[c.i1] * c.w1, h1 = r1[c.i0] * c.w0 + r1[c.i1] * c.w1;
    bg[(size_t)y * bw + x] = fm_linear_v(r, h0, h1);
    // clamps as selects (VIMNMX3, cv_linear.cuh)
    const int nx0 = (int)floor(x * scale_x), ny0 = (int)floor(y * scale_y);
    const int nx = nx0 < w - 1 ? nx0 : w - 1, ny = ny0 < h - 1 ? ny0 : h - 1;
    bg_mask[(size_t)y * bw + x] = owner[(size_t)ny * w + nx] == FM_NO_OWNER ? 255 : 0;
}

}  // namespace

extern "C" int fm_gray_half(const FmFrame* frame, unsigned char* gray, unsigned char* small, void* stream) {
    FM_REQUIRE(frame && fm_frame_ok(*frame), "fm_gray_half: " FM_FRAME_RULES);
    const int w = frame->w, h = frame->h;
    const int sw = (w + 1) / 2, sh = (h + 1) / 2;
    FM_REQUIRE(w % 2 == 0 && h % 2 == 0, "fm_gray_half: frame size must be even (0.5x resize = 2x2 mean)");
    const dim3 grid(fm_cdiv(sw, 256), sh);
    fm_visit_src(*frame, [&](auto src) {
        gray_half_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, w, h, gray, small, sw, sh);
    });
    FM_CHECK_LAUNCH("fm_gray_half");
    return FM_OK;
}

extern "C" int fm_gray_resize(const FmFrame* frame, unsigned char* gray, unsigned char* small, int sw, int sh,
                              void* stream) {
    FM_REQUIRE(frame && fm_frame_ok(*frame), "fm_gray_resize: " FM_FRAME_RULES);
    const int w = frame->w, h = frame->h;
    FM_REQUIRE(sw > 0 && sh > 0 && sw <= w && sh <= h,
               "fm_gray_resize: the optical-flow image must be non-empty and no larger than the frame");
    fm_visit_src(*frame, [&](auto src) {
        gray_kernel<<<dim3(fm_cdiv(w, 256), h), 256, 0, (cudaStream_t)stream>>>(src, w, h, gray);
    });
    resize_linear_kernel<<<dim3(fm_cdiv(sw, 256), sh), 256, 0, (cudaStream_t)stream>>>(
        gray, w, h, small, sw, sh, 1.0 / ((double)sw / w), 1.0 / ((double)sh / h));
    fm_count_launches(1);
    FM_CHECK_LAUNCH("fm_gray_resize");
    return FM_OK;
}

extern "C" int fm_pyr_level(const unsigned char* src, int sw, int sh, unsigned char* dst, void* stream) {
    const int dw = (sw + 1) / 2, dh = (sh + 1) / 2;
    dim3 grid(fm_cdiv(dw, 256), dh);
    pyr_down_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, sw, sh, dst, dw, dh);
    FM_CHECK_LAUNCH("fm_pyr_level");
    return FM_OK;
}

extern "C" int fm_scharr(const unsigned char* src, int w, int h, short* deriv, void* stream) {
    dim3 grid(fm_cdiv(w, 256), h);
    scharr_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, w, h, (short2*)deriv);
    FM_CHECK_LAUNCH("fm_scharr");
    return FM_OK;
}

extern "C" int fm_bg_small(const unsigned char* gray, const int* owner, int w, int h, unsigned char* bg,
                           unsigned char* bg_mask, int bw, int bh, void* stream) {
    dim3 grid(fm_cdiv(bw, 128), bh);
    bg_small_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(gray, owner, w, h, bg, bg_mask, bw, bh,
                                                            1.0 / ((double)bw / w), 1.0 / ((double)bh / h));
    FM_CHECK_LAUNCH("fm_bg_small");
    return FM_OK;
}
