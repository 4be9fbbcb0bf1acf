// KLT keypoint maintenance: occlusion ("owner") map, per-track keypoint filtering, Shi-Tomasi / Harris re-detection
// (cv2.goodFeaturesToTrack semantics) inside the visible part of each box, FAST-9/16 background corners,
// and the gather that builds the flat point list for the LK kernel.
//
// goodFeaturesToTrack's default settings (blockSize 3, gradientSize 3, minimum eigenvalue, 0 < maxCorners <= 1024)
// run gftt_eig_kernel and gftt_select_kernel<false>; every other setting runs gftt_response_kernel and
// gftt_select_kernel<true>.
//
// Reference: fastmot/flow.py:156-200 (+ helpers :266-306, 335-344), fastmot/utils/rect.py:60-89,
// fastmot/utils/numba.py:32-39.  OpenCV routines restated: goodFeaturesToTrack / cornerMinEigenVal
// (featureselect.cpp, corner.cpp) and FAST_t<16> + cornerScore<16> (fast.cpp, fast_score.cpp).
//
// The reference paints boxes into `fg_mask` one track at a time (nearest first) and reads the mask while it
// goes.  Equivalent order-free form used here: owner[p] = smallest rank k of a track whose clipped box covers p;
// track k sees pixel p as foreground  <=>  owner[p] == k.
#include "common.cuh"
#include "../../include/fastmot_b200.h"

#include <float.h>
#include <limits.h>

namespace {

struct Box {
    int x0, y0, x1, y1;  // clipped inclusive integer crop, valid if x1 >= x0 && y1 >= y0
    bool valid;
};

// intersection(track.tlbr, frame_rect) then crop(): int truncation, lower clamp (rect.py:60-89)
__device__ __forceinline__ Box clip_box(const double* t, int w, int h) {
    Box b;
    double x0 = fmax(t[0], 0.0), y0 = fmax(t[1], 0.0), x1 = fmin(t[2], (double)(w - 1)), y1 = fmin(t[3], (double)(h - 1));
    b.valid = !(x1 < x0 || y1 < y0);
    b.x0 = max((int)x0, 0); b.y0 = max((int)y0, 0);
    b.x1 = min(max((int)x1, 0), w - 1); b.y1 = min(max((int)y1, 0), h - 1);
    return b;
}

__global__ void owner_clear_kernel(int* __restrict__ owner, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) owner[i] = FM_NO_OWNER;
}

// One CTA per track (rank = blockIdx.x in nearest-first order).
__global__ void __launch_bounds__(256) owner_paint_kernel(const double* __restrict__ tlbr_pool,
                                                           const int* __restrict__ slots, int n_trk, int w, int h,
                                                           int* __restrict__ owner) {
    const int k = blockIdx.x;
    if (k >= n_trk) return;
    Box b = clip_box(tlbr_pool + (size_t)slots[k] * 4, w, h);
    if (!b.valid) return;
    const int bw = b.x1 - b.x0 + 1, bh = b.y1 - b.y0 + 1;
    for (int i = threadIdx.x; i < bw * bh; i += blockDim.x) {
        int y = b.y0 + i / bw, x = b.x0 + i % bw;
        atomicMin(owner + (size_t)y * w + x, k);
    }
}

// Same, for arbitrary rounded boxes painted with crop() semantics (second pass of flow.py:237-263).
// ---------------------------------------------------------------------------------------------------------
// Per-track: visible area, filter propagated keypoints (_rect_filter, flow.py:283-294), decide re-detection.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) kp_prepare_kernel(const double* __restrict__ tlbr_pool,
                                                          const int* __restrict__ slots, int n_trk, int w, int h,
                                                          const int* __restrict__ owner, float* __restrict__ kp_pool,
                                                          int* __restrict__ kp_count, int max_kp, double feat_density,
                                                          double feat_dist_factor, FmTrackJob* __restrict__ jobs,
                                                          int* __restrict__ scratch_counter, int scratch_cap,
                                                          int scratch_per_px) {
    __shared__ int s_cnt[8];
    __shared__ int s_area, s_base, s_total;
    const int k = blockIdx.x;
    if (k >= n_trk) return;
    const int slot = slots[k];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const double* t = tlbr_pool + (size_t)slot * 4;
    Box b = clip_box(t, w, h);
    FmTrackJob job;
    job.slot = slot;
    job.x0 = b.x0; job.y0 = b.y0;
    job.cw = b.valid ? b.x1 - b.x0 + 1 : 0;
    job.ch = b.valid ? b.y1 - b.y0 + 1 : 0;
    // visible area = mask_area(crop(fg_mask, inside_tlbr))
    int cnt = 0;
    for (int i = tid; i < job.cw * job.ch; i += blockDim.x) {
        int y = b.y0 + i / job.cw, x = b.x0 + i % job.cw;
        cnt += owner[(size_t)y * w + x] == k;
    }
    cnt = warp_sum(cnt);
    if (lane == 0) s_cnt[wid] = cnt;
    __syncthreads();
    if (tid == 0) {
        int a = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) a += s_cnt[i];
        s_area = a;
        s_base = 0;
    }
    __syncthreads();
    const int area = s_area;
    // stable in-place compaction of the propagated keypoints
    float* kp = kp_pool + (size_t)slot * max_kp * 2;
    const int n_old = min(kp_count[slot], max_kp);
    // inside test uses the *unclipped-to-int* intersection box (doubles), like `pts2i >= tlbr[:2]`
    const double ix0 = fmax(t[0], 0.0), iy0 = fmax(t[1], 0.0), ix1 = fmin(t[2], (double)(w - 1)), iy1 = fmin(t[3], (double)(h - 1));
    for (int base = 0; base < n_old; base += blockDim.x) {
        const int i = base + tid;
        float px = 0, py = 0;
        bool keep = false;
        if (i < n_old && b.valid) {
            px = kp[2 * i]; py = kp[2 * i + 1];
            const int xi = (int)rintf(px), yi = (int)rintf(py);
            keep = xi >= ix0 && xi <= ix1 && yi >= iy0 && yi <= iy1;
            if (keep) keep = xi >= 0 && yi >= 0 && xi < w && yi < h && owner[(size_t)yi * w + xi] == k;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_cnt[wid] = __popc(bal);
        __syncthreads();
        int off = s_base;
        for (int i2 = 0; i2 < wid; ++i2) off += s_cnt[i2];
        off += __popc(bal & ((1u << lane) - 1));
        __syncthreads();  // all reads of kp[base..] done before any write lands (writes go to indices <= i)
        if (keep) { kp[2 * off] = px; kp[2 * off + 1] = py; }
        if (tid == 0) {
            int tot = 0;
            for (int i2 = 0; i2 < (int)(blockDim.x >> 5); ++i2) tot += s_cnt[i2];
            s_total = tot;
        }
        __syncthreads();
        if (tid == 0) s_base += s_total;
        __syncthreads();
    }
    if (tid == 0) {
        const int n_keep = s_base;
        job.area = area;
        job.n_keep = n_keep;
        job.redetect = b.valid && ((double)n_keep < feat_density * (double)area) ? 1 : 0;
        if (!b.valid) { job.n_keep = 0; }
        // minDistance = max(round(sqrt(area) * factor), 1)   (flow.py:268-270; round half even)
        double md = rint(sqrt((double)area) * feat_dist_factor);
        job.min_dist = md < 1.0 ? 1 : (int)md;
        job.scratch_off = -1;
        job.eig_max = 0.f;
        if (job.redetect) {
            int need = job.cw * job.ch * scratch_per_px;
            int off = atomicAdd(scratch_counter, need);
            if (off + need <= scratch_cap) job.scratch_off = off;
            else job.redetect = 2;  // overflow flag, surfaced to the host
            kp_count[slot] = 0;
        } else {
            kp_count[slot] = job.n_keep;
        }
        jobs[k] = job;
    }
}

// ---------------------------------------------------------------------------------------------------------
// The default setting: cornerMinEigenVal(blockSize 3, Sobel 3) on the crop of the previous gray frame; reflect-101 on
// the crop.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int refl(int p, int n) {
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = p < 0 ? -p : 2 * n - 2 - p;
    return p;
}

__global__ void __launch_bounds__(256) gftt_eig_kernel(const unsigned char* __restrict__ gray, int w, int h,
                                                        const int* __restrict__ owner, FmTrackJob* __restrict__ jobs,
                                                        int n_trk, float* __restrict__ scratch) {
    __shared__ float s_max[8];
    const int k = blockIdx.x;
    if (k >= n_trk) return;
    FmTrackJob job = jobs[k];
    if (job.redetect != 1) return;
    const int cw = job.cw, ch = job.ch;
    const float scale = (float)(1.0 / (4.0 * 3.0 * 255.0));
    float* eig = scratch + job.scratch_off;
    float vmax = 0.f;
    for (int i = threadIdx.x; i < cw * ch; i += blockDim.x) {
        const int y = i / cw, x = i - y * cw;
        float sxx = 0.f, sxy = 0.f, syy = 0.f;
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int yy = refl(y + dy, ch), xx = refl(x + dx, cw);
                // Sobel at (xx, yy) of the crop with reflect-101 borders
                const int ym = refl(yy - 1, ch), yp = refl(yy + 1, ch), xm = refl(xx - 1, cw), xp = refl(xx + 1, cw);
                const unsigned char* r0 = gray + (size_t)(job.y0 + ym) * w + job.x0;
                const unsigned char* r1 = gray + (size_t)(job.y0 + yy) * w + job.x0;
                const unsigned char* r2 = gray + (size_t)(job.y0 + yp) * w + job.x0;
                const int gx = (r0[xp] - r0[xm]) + 2 * (r1[xp] - r1[xm]) + (r2[xp] - r2[xm]);
                const int gy = (r2[xm] - r0[xm]) + 2 * (r2[xx] - r0[xx]) + (r2[xp] - r0[xp]);
                const float fx = gx * scale, fy = gy * scale;
                sxx += fx * fx; sxy += fx * fy; syy += fy * fy;
            }
        }
        const float a = sxx * 0.5f, b = sxy, c = syy * 0.5f;
        const float v = (a + c) - sqrtf((a - c) * (a - c) + b * b);
        eig[i] = v;
        if (owner[(size_t)(job.y0 + y) * w + job.x0 + x] == k) vmax = fmaxf(vmax, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = vmax;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, s_max[i]);
        jobs[k].eig_max = m;
    }
}

// ---------------------------------------------------------------------------------------------------------
// cornerMinEigenVal / cornerHarris (corner.cpp: cornerEigenValsVecs) for any blockSize >= 1 and Sobel aperture
// 1 / 3 / 5 / 7 on the crop of the previous gray frame; reflect-101 on the crop for the Sobel and the box filter.
// Pass 1 writes the scaled gradient products (Dx^2, Dx*Dy, Dy^2) of every crop pixel to three scratch planes after
// the response map, pass 2 sums them over the unnormalised blockSize x blockSize window anchored at blockSize / 2
// (even sizes reach one pixel further up / left) and forms the response.  The selection only needs the corners it
// picks to be OpenCV's, not the response bits: the float sums run in a different order than OpenCV's filters.
// ---------------------------------------------------------------------------------------------------------
// Sobel taps of aperture 1 / 3 / 5 / 7 centred in 7 entries: smoothing (binomial) and first derivative.
// Aperture 1 is the 3-tap [-1 0 1] derivative with no smoothing (getSobelKernels).
__constant__ int c_sobel_smooth[4][7] = {{0, 0, 0, 1, 0, 0, 0}, {0, 0, 1, 2, 1, 0, 0}, {0, 1, 4, 6, 4, 1, 0},
                                         {1, 6, 15, 20, 15, 6, 1}};
__constant__ int c_sobel_deriv[4][7] = {{0, 0, -1, 0, 1, 0, 0}, {0, 0, -1, 0, 1, 0, 0}, {0, -1, -2, 0, 2, 1, 0},
                                        {-1, -4, -5, 0, 5, 4, 1}};

__global__ void __launch_bounds__(256) gftt_response_kernel(const unsigned char* __restrict__ gray, int w, int h,
                                                             const int* __restrict__ owner,
                                                             FmTrackJob* __restrict__ jobs, int n_trk,
                                                             float* __restrict__ scratch, int block_size,
                                                             int gradient_size, int use_harris, float harris_k) {
    __shared__ float s_max[8];
    const int k = blockIdx.x;
    if (k >= n_trk) return;
    const FmTrackJob job = jobs[k];
    if (job.redetect != 1) return;
    const int cw = job.cw, ch = job.ch, n = cw * ch;
    const int t = gradient_size >> 1, r = gradient_size == 1 ? 1 : t;   // table row, tap radius
    const float scale = (float)(1.0 / ((double)(1 << (gradient_size - 1)) * block_size * 255.0));
    float* eig = scratch + job.scratch_off;
    float* cxx = eig + n;
    float* cxy = cxx + n;
    float* cyy = cxy + n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int y = i / cw, x = i - y * cw;
        int cols[7];
        for (int q = -r; q <= r; ++q) cols[q + 3] = job.x0 + refl(x + q, cw);
        int gx = 0, gy = 0;
        for (int p = -r; p <= r; ++p) {
            const unsigned char* row = gray + (size_t)(job.y0 + refl(y + p, ch)) * w;
            int dxr = 0, sxr = 0;
            for (int q = -r; q <= r; ++q) {
                const int v = row[cols[q + 3]];
                dxr += c_sobel_deriv[t][q + 3] * v;
                sxr += c_sobel_smooth[t][q + 3] * v;
            }
            gx += c_sobel_smooth[t][p + 3] * dxr;
            gy += c_sobel_deriv[t][p + 3] * sxr;
        }
        const float fx = gx * scale, fy = gy * scale;
        cxx[i] = fx * fx; cxy[i] = fx * fy; cyy[i] = fy * fy;
    }
    __syncthreads();
    const int anchor = block_size >> 1;
    float vmax = -FLT_MAX;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int y = i / cw, x = i - y * cw;
        float a = 0.f, b = 0.f, c = 0.f;
        for (int p = 0; p < block_size; ++p) {
            const int ro = refl(y - anchor + p, ch) * cw;
            for (int q = 0; q < block_size; ++q) {
                const int j = ro + refl(x - anchor + q, cw);
                a += cxx[j]; b += cxy[j]; c += cyy[j];
            }
        }
        float v;
        if (use_harris) {
            v = a * c - b * b - harris_k * (a + c) * (a + c);
        } else {
            a *= 0.5f; c *= 0.5f;
            v = (a + c) - sqrtf((a - c) * (a - c) + b * b);
        }
        eig[i] = v;
        if (owner[(size_t)(job.y0 + y) * w + job.x0 + x] == k) vmax = fmaxf(vmax, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = vmax;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = -FLT_MAX;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, s_max[i]);
        jobs[k].eig_max = m == -FLT_MAX ? 0.f : m;      // minMaxLoc over an empty mask gives 0
    }
}

// Ascending order of the key == descending order of v, for either sign (the Harris response can be negative).
__device__ __forceinline__ unsigned desc_key(float v) {
    const unsigned u = __float_as_uint(v);
    return (u & 0x80000000u) ? u : ~(u | 0x80000000u);
}

// threshold + 3x3 local maximum + sort (value desc, address desc) + greedy min-distance + ellipse filter.
// kGeneral = false: the default settings (response > 0, at most 1024 corners kept in shared memory).  kGeneral = true:
// any response sign (THRESH_TOZERO is applied to the neighbours before the local-maximum test, as OpenCV's dilate
// sees them), maxCorners <= 0 means no limit, and the accepted corners go to acc_list (two ints per corner, in the
// gradient planes of this track's scratch, free once the response is final).
#define GFTT_MAX_CAND 4096
template <bool kGeneral>
__global__ void __launch_bounds__(256) gftt_select_kernel(const int* __restrict__ owner, int w, int h,
                                                           const double* __restrict__ tlbr_pool,
                                                           FmTrackJob* __restrict__ jobs, int n_trk,
                                                           const float* __restrict__ scratch, double quality,
                                                           int max_corners, float* __restrict__ kp_pool,
                                                           int* __restrict__ kp_count, int max_kp,
                                                           int* __restrict__ status, float* __restrict__ acc_scratch) {
    __shared__ unsigned long long s_key[GFTT_MAX_CAND];
    __shared__ unsigned char s_dead[GFTT_MAX_CAND];
    __shared__ int s_n, s_nacc, s_cur;
    __shared__ short s_accx[kGeneral ? 1 : 1024], s_accy[kGeneral ? 1 : 1024];
    const int k = blockIdx.x;
    if (k >= n_trk) return;
    const FmTrackJob job = jobs[k];
    if (job.redetect == 2 && threadIdx.x == 0) status[0] = 2;
    if (job.redetect != 1) return;
    const int cw = job.cw, ch = job.ch, tid = threadIdx.x;
    const float* eig = scratch + job.scratch_off;
    int* acc_list = kGeneral ? (int*)(acc_scratch + job.scratch_off + cw * ch) : nullptr;
    const float thr = (float)((double)job.eig_max * quality);
    if (tid == 0) { s_n = 0; s_nacc = 0; }
    __syncthreads();
    for (int i = tid; i < cw * ch; i += blockDim.x) {
        const int y = i / cw, x = i - y * cw;
        if (y < 1 || x < 1 || y >= ch - 1 || x >= cw - 1) continue;
        const float v = eig[i];
        if (!(v > thr)) continue;  // THRESH_TOZERO then `val != 0`
        if (kGeneral && v == 0.f) continue;
        if (owner[(size_t)(job.y0 + y) * w + job.x0 + x] != k) continue;
        bool ismax = true;
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                float nb = eig[(y + dy) * cw + (x + dx)];
                if (kGeneral && !(nb > thr)) nb = 0.f;
                ismax = ismax && (v >= nb);
            }
        if (!ismax) continue;
        const int pos = atomicAdd(&s_n, 1);
        if (pos < GFTT_MAX_CAND) {
            // ascending u64 sort == value desc (v > 0), then pixel index desc
            const unsigned vk = kGeneral ? desc_key(v) : ~__float_as_uint(v);
            s_key[pos] = ((unsigned long long)vk << 32) | (unsigned)(0x7fffffff - i);
        }
    }
    __syncthreads();
    int n = s_n;
    if (n > GFTT_MAX_CAND) {
        if (tid == 0) status[0] = 3;  // candidate overflow, surfaced to the host
        n = GFTT_MAX_CAND;
    }
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    for (int i = n + tid; i < np2; i += blockDim.x) s_key[i] = ~0ull;
    __syncthreads();
    for (int kk = 2; kk <= np2; kk <<= 1)
        for (int j = kk >> 1; j > 0; j >>= 1) {
            for (int t = tid; t < (np2 >> 1); t += blockDim.x) {
                const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1)), hi = lo | j;
                const bool asc = (lo & kk) == 0;
                const unsigned long long a = s_key[lo], b = s_key[hi];
                if ((a > b) == asc) { s_key[lo] = b; s_key[hi] = a; }
            }
            __syncthreads();
        }
    for (int i = tid; i < n; i += blockDim.x) s_dead[i] = 0;
    __syncthreads();
    // greedy min-distance: one barrier pair per ACCEPTED corner
    const int md2 = job.min_dist * job.min_dist;
    int cur = 0;
    const int cap = kGeneral ? (max_corners > 0 ? max_corners : INT_MAX) : min(max_corners, 1024);
    while (true) {
        if (tid == 0) {
            int c = cur;
            while (c < n && s_dead[c]) ++c;
            s_cur = (s_nacc < cap) ? c : n;
        }
        __syncthreads();
        cur = s_cur;
        if (cur >= n) break;
        const int idx = 0x7fffffff - (int)(s_key[cur] & 0xffffffffu);
        const int cy = idx / cw, cx = idx - cy * cw;
        if (tid == 0) {
            if (kGeneral) { acc_list[2 * s_nacc] = cx; acc_list[2 * s_nacc + 1] = cy; }
            else { s_accx[s_nacc] = cx; s_accy[s_nacc] = cy; }
            s_nacc = s_nacc + 1;
        }
        for (int j = cur + 1 + tid; j < n; j += blockDim.x) {
            if (s_dead[j]) continue;
            const int ji = 0x7fffffff - (int)(s_key[j] & 0xffffffffu);
            const int jy = ji / cw, jx = ji - jy * cw;
            const int dx = jx - cx, dy = jy - cy;
            if (dx * dx + dy * dy < md2) s_dead[j] = 1;
        }
        ++cur;
        __syncthreads();
    }
    __syncthreads();
    // _ellipse_filter (flow.py:298-306): pts + offset (f32), inside the ellipse inscribed in the FULL box
    if (tid == 0) {
        const double* t = tlbr_pool + (size_t)job.slot * 4;
        const double ccx = (t[0] + t[2]) / 2, ccy = (t[1] + t[3]) / 2;
        const double ax = (t[2] - t[0] + 1) * 0.5, ay = (t[3] - t[1] + 1) * 0.5;
        float* kp = kp_pool + (size_t)job.slot * max_kp * 2;
        int m = 0;
        for (int i = 0; i < s_nacc && m < max_kp; ++i) {
            const int ax_i = kGeneral ? acc_list[2 * i] : s_accx[i], ay_i = kGeneral ? acc_list[2 * i + 1] : s_accy[i];
            const float px = (float)ax_i + (float)job.x0, py = (float)ay_i + (float)job.y0;
            const double ux = ((double)px - ccx) / ax, uy = ((double)py - ccy) / ay;
            if (ux * ux + uy * uy <= 1.0) { kp[2 * m] = px; kp[2 * m + 1] = py; ++m; }
        }
        kp_count[job.slot] = m;
    }
}

// ---------------------------------------------------------------------------------------------------------
// FAST-9/16 with non-max suppression on the small background image.
// ---------------------------------------------------------------------------------------------------------
__global__ void fast_score_kernel(const unsigned char* __restrict__ img, int w, int h, int threshold,
                                  unsigned char* __restrict__ score) {
    // Bresenham circle of radius 3 (the loops below are unrolled: the offsets become immediates)
    constexpr int kDx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    constexpr int kDy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= w || y >= h) return;
    int sc = 0;
    if (x >= 3 && y >= 3 && x < w - 3 && y < h - 3) {
        // The differences are small integers, exact in fp32.  Integer min / max chains are avoided on purpose: ptxas
        // 12.9 fuses them into three-input VIMNMX3 instructions that return wrong minima / maxima on sm_90.
        const int v = img[y * w + x];
        float d[25];
#pragma unroll
        for (int k = 0; k < 16; ++k) d[k] = (float)(v - (int)img[(y + kDy[k]) * w + x + kDx[k]]);
#pragma unroll
        for (int k = 16; k < 25; ++k) d[k] = d[k - 16];
        // A = max over the 16 arcs of min(d) (darker), B = max over arcs of min(-d) (brighter)
        float A = -256.f, B = -256.f;
#pragma unroll
        for (int s = 0; s < 16; ++s) {
            float mn = d[s], mx = d[s];
#pragma unroll
            for (int k = 1; k < 9; ++k) { mn = fminf(mn, d[s + k]); mx = fmaxf(mx, d[s + k]); }
            A = fmaxf(A, mn);
            B = fmaxf(B, -mx);
        }
        const int best = (int)fmaxf(A, B);
        if (best > threshold) sc = best - 1;  // corner; cornerScore = max(threshold, A, B) - 1
    }
    score[y * w + x] = (unsigned char)sc;
}

// NMS (strictly greater than the 8 neighbours), pixel mask, row-major ordered compaction; single CTA.
// Pixels are cut into 32-pixel words; warp w takes words w, w + 32, ... (lanes read consecutive pixels, four words'
// scores are in flight at once), the keep decision of every pixel is taken once and kept as a ballot word in shared
// memory; a block scan over the word popcounts gives every word its output offset, the scatter only replays bits.
#define FAST_NMS_MAX_WORDS 4096      // 131 072 pixels at the background scale (1920x1080 x 0.1^2 = 20 736)
__global__ void __launch_bounds__(1024) fast_nms_kernel(const unsigned char* __restrict__ score,
                                                         const unsigned char* __restrict__ mask, int w, int h,
                                                         float unscale_x, float unscale_y, float* __restrict__ out_pts,
                                                         int* __restrict__ out_count, int max_pts) {
    __shared__ unsigned s_bits[FAST_NMS_MAX_WORDS];
    __shared__ int s_pref[FAST_NMS_MAX_WORDS];
    __shared__ int s_warp[32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int n = w * h;
    const int words = (n + 31) >> 5;
    for (int base = wid; base < words; base += 32 * 4) {
        int sc[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int wd = base + 32 * u;
            const int i = (wd << 5) + lane;
            sc[u] = (wd < words && i < n) ? (int)score[i] : 0;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int wd = base + 32 * u;              // warp-uniform
            if (wd >= words) break;
            const int i = (wd << 5) + lane;
            bool ok = false;
            if (sc[u] != 0) {
                // a non-zero score is an interior pixel; neighbours outside [3, w-3) x [3, h-3) have score 0
                const int v = sc[u];
                ok = v > score[i - 1] && v > score[i + 1] && v > score[i - w - 1] && v > score[i - w] &&
                     v > score[i - w + 1] && v > score[i + w - 1] && v > score[i + w] && v > score[i + w + 1] &&
                     mask[i] != 0;
            }
            const unsigned bal = __ballot_sync(0xffffffffu, ok);
            if (lane == 0) s_bits[wd] = bal;
        }
    }
    __syncthreads();
    // exclusive prefix of the word popcounts: thread t owns words 4t .. 4t+3
    int c[4], tot = 0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int wd = 4 * tid + u;
        c[u] = wd < words ? __popc(s_bits[wd]) : 0;
        tot += c[u];
    }
    int v = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    if (lane == 31) s_warp[wid] = v;
    __syncthreads();
    if (wid == 0) {
        int t = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += u;
        }
        s_warp[lane] = t;
        if (lane == 31) *out_count = min(t, max_pts);
    }
    __syncthreads();
    int run = v - tot + (wid ? s_warp[wid - 1] : 0);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int wd = 4 * tid + u;
        if (wd < words) s_pref[wd] = run;
        run += c[u];
    }
    __syncthreads();
    for (int wd = wid; wd < words; wd += 32) {
        const unsigned bal = s_bits[wd];
        if ((bal >> lane) & 1u) {
            const int pos = s_pref[wd] + __popc(bal & ((1u << lane) - 1u));
            if (pos < max_pts) {
                const int i = (wd << 5) + lane;
                const int y = i / w, x = i - y * w;
                out_pts[2 * pos] = (float)x * unscale_x;      // _unscale_pts (flow.py:335-344)
                out_pts[2 * pos + 1] = (float)y * unscale_y;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// Gather: all_prev_pts = concat(track keypoints in rank order) ++ background points; begin/end per track.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) gather_points_kernel(const float* __restrict__ kp_pool,
                                                              const int* __restrict__ kp_count, int max_kp,
                                                              const int* __restrict__ slots, int n_trk,
                                                              const float* __restrict__ bg_pts,
                                                              const int* __restrict__ bg_count,
                                                              float* __restrict__ all_pts, int* __restrict__ trk_begin,
                                                              int* __restrict__ meta, int max_pts) {
    __shared__ int s_off[1025];
    __shared__ int s_cnt[2048];
    const int tid = threadIdx.x;
    // counts are fetched in parallel (the dependent slot -> count loads are the slow part), prefix by thread 0
    for (int k = tid; k < n_trk && k < 2048; k += blockDim.x) s_cnt[k] = min(kp_count[slots[k]], max_kp);
    __syncthreads();
    if (tid == 0) {
        int acc = 0;
        for (int k = 0; k < n_trk; ++k) {
            trk_begin[k] = acc;
            acc += k < 2048 ? s_cnt[k] : min(kp_count[slots[k]], max_kp);
        }
        trk_begin[n_trk] = acc;
        int nb = *bg_count;
        if (acc + nb > max_pts) { meta[3] = 1; nb = max(0, max_pts - acc); acc = min(acc, max_pts); }
        meta[0] = acc;        // bg_begin = number of object points
        meta[1] = acc + nb;   // total points P
        meta[2] = nb;
        s_off[0] = acc;
    }
    __syncthreads();
    const int n_obj = s_off[0];
    // one warp per track (32 warps in flight) instead of a serial walk over the tracks
    const int lane = tid & 31, wid = tid >> 5, nwarp = blockDim.x >> 5;
    for (int k = wid; k < n_trk; k += nwarp) {
        const int b = trk_begin[k], e = min(trk_begin[k + 1], max_pts);
        const float* src = kp_pool + (size_t)slots[k] * max_kp * 2;
        for (int i = lane; i < (e - b) * 2; i += 32) all_pts[2 * (size_t)b + i] = src[i];
    }
    const int nb = meta[2];
    for (int i = tid; i < nb * 2; i += blockDim.x) all_pts[2 * (size_t)n_obj + i] = bg_pts[i];
}

}  // namespace

extern "C" int fm_flow_keypoints(const unsigned char* prev_gray, int w, int h, const double* tlbr_pool,
                                 const int* slots, int n_trk, int* owner, float* kp_pool, int* kp_count, int max_kp,
                                 double feat_density, double feat_dist_factor, double quality, int max_corners,
                                 FmTrackJob* jobs, float* scratch, int scratch_cap, int* scratch_counter, int* status,
                                 void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    owner_clear_kernel<<<FM_NUM_SMS * 4, 256, 0, s>>>(owner, (size_t)w * h);
    cudaMemsetAsync(scratch_counter, 0, sizeof(int), s);
    cudaMemsetAsync(status, 0, sizeof(int), s);
    if (n_trk > 0) {
        owner_paint_kernel<<<n_trk, 256, 0, s>>>(tlbr_pool, slots, n_trk, w, h, owner);
        kp_prepare_kernel<<<n_trk, 256, 0, s>>>(tlbr_pool, slots, n_trk, w, h, owner, kp_pool, kp_count, max_kp,
                                                feat_density, feat_dist_factor, jobs, scratch_counter, scratch_cap, 1);
        gftt_eig_kernel<<<n_trk, 256, 0, s>>>(prev_gray, w, h, owner, jobs, n_trk, scratch);
        gftt_select_kernel<false><<<n_trk, 256, 0, s>>>(owner, w, h, tlbr_pool, jobs, n_trk, scratch, quality,
                                                        max_corners, kp_pool, kp_count, max_kp, status, nullptr);
    }
    FM_CHECK_LAUNCH("fm_flow_keypoints");
    return FM_OK;
}

extern "C" int fm_flow_keypoints_cfg(const unsigned char* prev_gray, int w, int h, const double* tlbr_pool,
                                     const int* slots, int n_trk, int* owner, float* kp_pool, int* kp_count,
                                     int max_kp, double feat_density, double feat_dist_factor, double quality,
                                     int max_corners, int block_size, int gradient_size, int use_harris,
                                     double harris_k, FmTrackJob* jobs, float* scratch, int scratch_cap,
                                     int* scratch_counter, int* status, void* stream) {
    if (block_size == 3 && gradient_size == 3 && !use_harris && max_corners > 0 && max_corners <= 1024)
        return fm_flow_keypoints(prev_gray, w, h, tlbr_pool, slots, n_trk, owner, kp_pool, kp_count, max_kp,
                                 feat_density, feat_dist_factor, quality, max_corners, jobs, scratch, scratch_cap,
                                 scratch_counter, status, stream);
    FM_REQUIRE(block_size >= 1, "fm_flow_keypoints_cfg: blockSize must be >= 1");
    FM_REQUIRE(gradient_size == 1 || gradient_size == 3 || gradient_size == 5 || gradient_size == 7,
               "fm_flow_keypoints_cfg: gradientSize must be 1, 3, 5 or 7");
    FM_REQUIRE(max_kp >= (max_corners > 0 ? min(max_corners, GFTT_MAX_CAND) : GFTT_MAX_CAND),
               "fm_flow_keypoints_cfg: max_kp is smaller than the corners one track may keep");
    cudaStream_t s = (cudaStream_t)stream;
    owner_clear_kernel<<<FM_NUM_SMS * 4, 256, 0, s>>>(owner, (size_t)w * h);
    cudaMemsetAsync(scratch_counter, 0, sizeof(int), s);
    cudaMemsetAsync(status, 0, sizeof(int), s);
    if (n_trk > 0) {
        owner_paint_kernel<<<n_trk, 256, 0, s>>>(tlbr_pool, slots, n_trk, w, h, owner);
        // four floats per crop pixel: the response map and the three gradient-product planes
        kp_prepare_kernel<<<n_trk, 256, 0, s>>>(tlbr_pool, slots, n_trk, w, h, owner, kp_pool, kp_count, max_kp,
                                                feat_density, feat_dist_factor, jobs, scratch_counter, scratch_cap, 4);
        gftt_response_kernel<<<n_trk, 256, 0, s>>>(prev_gray, w, h, owner, jobs, n_trk, scratch, block_size,
                                                   gradient_size, use_harris, (float)harris_k);
        gftt_select_kernel<true><<<n_trk, 256, 0, s>>>(owner, w, h, tlbr_pool, jobs, n_trk, scratch, quality,
                                                       max_corners, kp_pool, kp_count, max_kp, status, scratch);
    }
    FM_CHECK_LAUNCH("fm_flow_keypoints_cfg");
    return FM_OK;
}

extern "C" int fm_fast_detect(const unsigned char* img, const unsigned char* mask, int w, int h, int threshold,
                              float unscale_x, float unscale_y, unsigned char* score, float* out_pts, int* out_count,
                              int max_pts, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid(fm_cdiv(w, 128), h);
    FM_REQUIRE((long long)w * h <= 32ll * FAST_NMS_MAX_WORDS, "fm_fast_detect: image larger than 131072 pixels");
    fast_score_kernel<<<grid, 128, 0, s>>>(img, w, h, threshold, score);
    fast_nms_kernel<<<1, 1024, 0, s>>>(score, mask, w, h, unscale_x, unscale_y, out_pts, out_count, max_pts);
    FM_CHECK_LAUNCH("fm_fast_detect");
    return FM_OK;
}

extern "C" int fm_gather_points(const float* kp_pool, const int* kp_count, int max_kp, const int* slots, int n_trk,
                                const float* bg_pts, const int* bg_count, float* all_pts, int* trk_begin, int* meta,
                                int max_pts, void* stream) {
    cudaMemsetAsync(meta, 0, 4 * sizeof(int), (cudaStream_t)stream);
    gather_points_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(kp_pool, kp_count, max_kp, slots, n_trk, bg_pts,
                                                               bg_count, all_pts, trk_begin, meta, max_pts);
    FM_CHECK_LAUNCH("fm_gather_points");
    return FM_OK;
}
