// cv2.resize(..., INTER_LINEAR) of 8-bit images as OpenCV 4.13 computes it on its generic path (resize.cpp): per axis
// scale = 1 / (dsize / ssize) in double, source coordinate f = (float)((d + 0.5) * scale - 0.5), i = floor(f),
// 11-bit coefficients rint((1 - frac) * 2048) and rint(frac * 2048), a horizontal pass in int and the vertical pass of
// VResizeLinearVec_32s8u.  Columns and rows are clamped differently at the image edges (fm_linear_col, fm_linear_row);
// both rules are pinned against cv2.resize by tests/test_frame_resize_cpu.py through oracle/resize.py.
#pragma once

// The two source indices and 11-bit weights of one output coordinate along one axis.
struct FmLinearTap {
    int i0, i1, w0, w1;
};

// Columns: a tap before the first source column or on / after the last one takes that edge column alone (the index is
// clamped and the fraction set to 0).  Clamps are selects: ptxas 12.9 fuses chained integer min / max into VIMNMX3,
// which returns wrong results on sm_90 (see fast_score_kernel in klt_feat.cu).
__device__ __forceinline__ FmLinearTap fm_linear_col(int d, double scale, int ssize) {
    float f = (float)((d + 0.5) * scale - 0.5);
    int i = (int)floorf(f);
    f -= i;
    if (i < 0) { f = 0.f; i = 0; }
    if (i >= ssize - 1) { f = 0.f; i = ssize - 1; }
    const int i1 = i + 1 < ssize ? i + 1 : ssize - 1;
    return {i, i1, (int)rintf((1.f - f) * 2048.f), (int)rintf(f * 2048.f)};
}

// Rows: only the two source row indices are clamped, the fraction is kept.  The first and last rows of an upscale
// therefore blend one source row with itself, each weight truncated on its own in fm_linear_v (1-LSB differences
// against a zeroed fraction).  For a downscale i stays in [0, ssize - 1), or the fraction is 0, so both rules agree.
__device__ __forceinline__ FmLinearTap fm_linear_row(int d, double scale, int ssize) {
    float f = (float)((d + 0.5) * scale - 0.5);
    const int i = (int)floorf(f);
    f -= i;
    const int i0 = i < 0 ? 0 : i > ssize - 1 ? ssize - 1 : i;
    const int i1 = i + 1 < 0 ? 0 : i + 1 > ssize - 1 ? ssize - 1 : i + 1;
    return {i0, i1, (int)rintf((1.f - f) * 2048.f), (int)rintf(f * 2048.f)};
}

// Vertical pass: h0, h1 are the horizontal sums (p[i0] * w0 + p[i1] * w1 of a column tap) on rows r.i0 and r.i1.
__device__ __forceinline__ int fm_linear_v(const FmLinearTap& r, int h0, int h1) {
    return (((r.w0 * (h0 >> 4)) >> 16) + ((r.w1 * (h1 >> 4)) >> 16) + 2) >> 2;
}
