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

// Candidate test of the selection: interior pixel of the crop, response above the quality threshold, seen by track k,
// 3x3 local maximum.  On success `key` is the sort key: ascending u64 == value desc, then crop pixel index desc
// (OpenCV's greaterThanPtr order).
template <bool kGeneral>
__device__ __forceinline__ bool gftt_candidate(const float* __restrict__ eig, const int* __restrict__ owner, int w,
                                               const FmTrackJob& job, int k, float thr, int i,
                                               unsigned long long& key) {
    const int cw = job.cw, ch = job.ch;
    const int y = i / cw, x = i - y * cw;
    if (y < 1 || x < 1 || y >= ch - 1 || x >= cw - 1) return false;
    const float v = eig[i];
    if (!(v > thr)) return false;  // THRESH_TOZERO then `val != 0`
    if (kGeneral && v == 0.f) return false;
    if (owner[(size_t)(job.y0 + y) * w + job.x0 + x] != k) return false;
    bool ismax = true;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            float nb = eig[(y + dy) * cw + (x + dx)];
            if (kGeneral && !(nb > thr)) nb = 0.f;
            ismax = ismax && (v >= nb);
        }
    if (!ismax) return false;
    // value desc (the default setting's responses are > 0, so the inverted bits order them), then pixel index desc
    const unsigned vk = kGeneral ? desc_key(v) : ~__float_as_uint(v);
    key = ((unsigned long long)vk << 32) | (unsigned)(0x7fffffff - i);
    return true;
}

__device__ __forceinline__ void bitonic_sort_smem(unsigned long long* s_key, int np2, int tid) {
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
}

// One pass of the block-wide merge sort: the sorted runs [2r*q, 2r*q + r) and [2r*q + r, 2r*(q+1)) of src are merged
// into dst.  Each thread writes GFTT_MERGE_ITEMS consecutive outputs of one pair (the count divides 2r) after a
// merge-path search for how many of them come from the first run.  The keys are unique and never ~0.
#define GFTT_MERGE_ITEMS 32
__device__ __forceinline__ void merge_pass(const unsigned long long* src, unsigned long long* dst, int n, int run,
                                           int tid) {
    for (int o = tid * GFTT_MERGE_ITEMS; o < n; o += blockDim.x * GFTT_MERGE_ITEMS) {
        const int base = o - o % (2 * run);
        const int na = min(run, n - base);
        const int nb = min(run, n - base - na);
        const unsigned long long* A = src + base;
        const unsigned long long* B = A + na;
        const int d = o - base;
        int lo = d > nb ? d - nb : 0, hi = d < na ? d : na;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (A[mid] < B[d - 1 - mid]) lo = mid + 1;
            else hi = mid;
        }
        int ai = lo, bi = d - lo;
        unsigned long long ka = ai < na ? A[ai] : ~0ull, kb = bi < nb ? B[bi] : ~0ull;
        const int end = d + GFTT_MERGE_ITEMS < na + nb ? d + GFTT_MERGE_ITEMS : na + nb;
        for (int q = d; q < end; ++q) {
            if (ka < kb) { dst[base + q] = ka; ++ai; ka = ai < na ? A[ai] : ~0ull; }
            else { dst[base + q] = kb; ++bi; kb = bi < nb ? B[bi] : ~0ull; }
        }
    }
}

// threshold + 3x3 local maximum + sort (value desc, address desc) + greedy min-distance + ellipse filter.
// kGeneral = false: the default settings (response > 0, at most 1024 corners kept in shared memory).  kGeneral = true:
// any response sign (THRESH_TOZERO is applied to the neighbours before the local-maximum test, as OpenCV's dilate
// sees them), maxCorners <= 0 means no limit, and the accepted corners go to acc_list (two ints per corner, in the
// gradient planes of this track's scratch, free once the response is final).
//
// A box of at most GFTT_MAX_CAND candidates sorts its keys in shared memory and runs the greedy loop there (one barrier
// pair per accepted corner, each scanning the remaining candidates).  A box with more claims its candidate storage from
// `work` through the per-frame scratch counter (status 2 when it does not fit) and runs the same selection in global
// memory: keys re-collected, sorted as GFTT_MAX_CAND-key shared-memory chunks merged pass by pass, then the greedy loop
// over chunks of 256 sorted candidates against a grid of minDistance cells holding the accepted corners (OpenCV's own
// structure): every thread tests one candidate against the 3x3 cells around it, then warp 0 settles the chunk's
// survivors in order.  Both paths accept exactly the corners of the sequential greedy.  Kept corners beyond max_kp
// set status 4.
#define GFTT_MAX_CAND 4096
constexpr int kSelectThreads = 256;
template <bool kGeneral>
__global__ void __launch_bounds__(kSelectThreads) gftt_select_kernel(const int* __restrict__ owner, int w, int h,
                                                                      const double* __restrict__ tlbr_pool,
                                                                      FmTrackJob* __restrict__ jobs, int n_trk,
                                                                      const float* __restrict__ scratch,
                                                                      double quality, int max_corners,
                                                                      float* __restrict__ kp_pool,
                                                                      int* __restrict__ kp_count, int max_kp,
                                                                      int* __restrict__ status,
                                                                      float* __restrict__ work,
                                                                      int* __restrict__ scratch_counter,
                                                                      int scratch_cap) {
    __shared__ unsigned long long s_key[GFTT_MAX_CAND];
    __shared__ unsigned char s_dead[GFTT_MAX_CAND];
    __shared__ int s_n, s_nacc, s_cur, s_off;
    __shared__ short s_accx[kGeneral ? 1 : 1024], s_accy[kGeneral ? 1 : 1024];
    __shared__ int s_cidx[kSelectThreads];
    const int k = blockIdx.x;
    if (k >= n_trk) return;
    const FmTrackJob job = jobs[k];
    if (job.redetect == 2 && threadIdx.x == 0) status[0] = 2;
    if (job.redetect != 1) return;
    const int cw = job.cw, ch = job.ch, tid = threadIdx.x;
    const float* eig = scratch + job.scratch_off;
    int* acc_list = kGeneral ? (int*)(work + job.scratch_off + cw * ch) : nullptr;
    const float thr = (float)((double)job.eig_max * quality);
    if (tid == 0) { s_n = 0; s_nacc = 0; }
    __syncthreads();
    for (int i = tid; i < cw * ch; i += blockDim.x) {
        unsigned long long key;
        if (!gftt_candidate<kGeneral>(eig, owner, w, job, k, thr, i, key)) continue;
        const int pos = atomicAdd(&s_n, 1);
        if (pos < GFTT_MAX_CAND) s_key[pos] = key;
    }
    __syncthreads();
    const int n = s_n;
    const int md2 = job.min_dist * job.min_dist;
    const int cap = kGeneral ? (max_corners > 0 ? max_corners : INT_MAX) : min(max_corners, 1024);
    if (n <= GFTT_MAX_CAND) {
        int np2 = 1;
        while (np2 < n) np2 <<= 1;
        for (int i = n + tid; i < np2; i += blockDim.x) s_key[i] = ~0ull;
        __syncthreads();
        bitonic_sort_smem(s_key, np2, tid);
        for (int i = tid; i < n; i += blockDim.x) s_dead[i] = 0;
        __syncthreads();
        // greedy min-distance: one barrier pair per ACCEPTED corner
        int cur = 0;
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
    } else {
        // ---- global-memory path.  Layout from an 8-byte aligned start: keys[n], sort buffer[n] (u64), accepted-corner
        // nodes {crop index, next} [min(n, cap)] (int2), grid cell heads [gw * gh] (int, -1 = empty).
        const int md = job.min_dist;
        const int gw = (cw + md - 1) / md, gh = (ch + md - 1) / md;
        // the default setting's cap (at most 1024) is below n; min(n, cap) there would chain onto cap's own min,
        // which ptxas fuses into a VIMNMX3 (DESIGN section 4)
        const int n_node = !kGeneral ? cap : (n < cap ? n : cap);
        const long long need = 4ll * n + 2ll * n_node + (long long)gw * gh + 1;
        if (tid == 0) {
            int off = -1;
            if (need <= (long long)scratch_cap) {
                const int o = atomicAdd(scratch_counter, (int)need);
                if (o >= 0 && (long long)o + need <= (long long)scratch_cap) off = o;
            }
            if (off < 0) status[0] = 2;  // raise scratch_floats
            s_off = off;
            s_cur = 0;
        }
        __syncthreads();
        if (s_off < 0) return;
        unsigned long long* keys = (unsigned long long*)(work + ((s_off + 1) & ~1));
        unsigned long long* tmp = keys + n;
        int2* nodes = (int2*)(tmp + n);
        int* heads = (int*)(nodes + n_node);
        const int lane = tid & 31, wid = tid >> 5;
        for (int i = tid; i < gw * gh; i += blockDim.x) heads[i] = -1;
        __syncthreads();
        // re-collect the keys, one shared-memory atomic per warp
        for (int base = 0; base < cw * ch; base += blockDim.x) {
            const int i = base + tid;
            unsigned long long key = 0;
            const bool c = i < cw * ch && gftt_candidate<kGeneral>(eig, owner, w, job, k, thr, i, key);
            const unsigned bal = __ballot_sync(0xffffffffu, c);
            int wpos = 0;
            if (lane == 0 && bal) wpos = atomicAdd(&s_cur, __popc(bal));
            wpos = __shfl_sync(0xffffffffu, wpos, 0);
            if (c) keys[wpos + __popc(bal & ((1u << lane) - 1u))] = key;
        }
        __syncthreads();
        // sort: shared-memory bitonic chunks of GFTT_MAX_CAND keys, then merge passes (keys <-> tmp)
        for (int c0 = 0; c0 < n; c0 += GFTT_MAX_CAND) {
            for (int i = tid; i < GFTT_MAX_CAND; i += blockDim.x) s_key[i] = c0 + i < n ? keys[c0 + i] : ~0ull;
            __syncthreads();
            bitonic_sort_smem(s_key, GFTT_MAX_CAND, tid);
            for (int i = tid; i < GFTT_MAX_CAND && c0 + i < n; i += blockDim.x) keys[c0 + i] = s_key[i];
            __syncthreads();
        }
        unsigned long long* src = keys;
        unsigned long long* dst = tmp;
        for (int run = GFTT_MAX_CAND; run < n; run <<= 1) {
            merge_pass(src, dst, n, run, tid);
            __syncthreads();
            unsigned long long* t = src; src = dst; dst = t;
        }
        // greedy min-distance over chunks of kSelectThreads sorted candidates
        for (int c0 = 0; c0 < n; c0 += kSelectThreads) {
            const int j = c0 + tid;
            int idx = 0;
            bool alive = false;
            if (j < n) {
                idx = 0x7fffffff - (int)(src[j] & 0xffffffffu);
                const int cy = idx / cw, cx = idx - cy * cw, gx = cx / md, gy = cy / md;
                alive = true;
                for (int yy = gy - 1; yy <= gy + 1; ++yy) {
                    if (yy < 0 || yy >= gh) continue;
                    for (int xx = gx - 1; xx <= gx + 1; ++xx) {
                        if (xx < 0 || xx >= gw) continue;
                        for (int a = heads[yy * gw + xx]; a >= 0 && alive; ) {
                            const int2 nd = nodes[a];
                            const int ay = nd.x / cw, ax = nd.x - ay * cw;
                            const int dx = ax - cx, dy = ay - cy;
                            alive = dx * dx + dy * dy >= md2;
                            a = nd.y;
                        }
                    }
                }
            }
            s_cidx[tid] = idx;
            s_dead[tid] = alive;
            __syncthreads();
            if (wid == 0) {
                // lane l holds candidates l, l + 32, ... of the chunk; live[g] has a bit per candidate still to settle
                int px[kSelectThreads / 32], py[kSelectThreads / 32];
                unsigned live[kSelectThreads / 32];
#pragma unroll
                for (int g = 0; g < kSelectThreads / 32; ++g) {
                    const int id = s_cidx[32 * g + lane];
                    py[g] = id / cw; px[g] = id - py[g] * cw;
                    live[g] = __ballot_sync(0xffffffffu, s_dead[32 * g + lane] != 0);
                }
                int nacc = s_nacc;
#pragma unroll
                for (int g = 0; g < kSelectThreads / 32; ++g) {
                    while (live[g] != 0u && nacc < cap) {
                        // the first live candidate is accepted; it kills every later one closer than minDistance
                        const int f = __ffs(live[g]) - 1;
                        const int fx = __shfl_sync(0xffffffffu, px[g], f), fy = __shfl_sync(0xffffffffu, py[g], f);
                        if (lane == 0) {
                            if (kGeneral) { acc_list[2 * nacc] = fx; acc_list[2 * nacc + 1] = fy; }
                            else { s_accx[nacc] = fx; s_accy[nacc] = fy; }
                            const int cell = (fy / md) * gw + fx / md;
                            nodes[nacc] = make_int2(fy * cw + fx, heads[cell]);
                            heads[cell] = nacc;
                        }
                        ++nacc;
#pragma unroll
                        for (int g2 = g; g2 < kSelectThreads / 32; ++g2) {
                            const int dx = px[g2] - fx, dy = py[g2] - fy;
                            live[g2] &= ~__ballot_sync(0xffffffffu, dx * dx + dy * dy < md2);
                        }
                    }
                }
                if (lane == 0) s_nacc = nacc;
            }
            __syncthreads();
            if (s_nacc >= cap) break;
        }
    }
    __syncthreads();
    // _ellipse_filter (flow.py:298-306): pts + offset (f32), inside the ellipse inscribed in the FULL box
    if (tid == 0) {
        const double* t = tlbr_pool + (size_t)job.slot * 4;
        const double ccx = (t[0] + t[2]) / 2, ccy = (t[1] + t[3]) / 2;
        const double ax = (t[2] - t[0] + 1) * 0.5, ay = (t[3] - t[1] + 1) * 0.5;
        float* kp = kp_pool + (size_t)job.slot * max_kp * 2;
        int m = 0;
        for (int i = 0; i < s_nacc; ++i) {
            const int ax_i = kGeneral ? acc_list[2 * i] : s_accx[i], ay_i = kGeneral ? acc_list[2 * i + 1] : s_accy[i];
            const float px = (float)ax_i + (float)job.x0, py = (float)ay_i + (float)job.y0;
            const double ux = ((double)px - ccx) / ax, uy = ((double)py - ccy) / ay;
            if (ux * ux + uy * uy <= 1.0) {
                if (m == max_kp) { status[0] = 4; break; }  // more kept corners than keypoint rows
                kp[2 * m] = px; kp[2 * m + 1] = py; ++m;
            }
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
// Images of more than FAST_NMS_MAX_WORDS words are walked in chunks of that many words, the output offset carried from
// one chunk to the next (the default 1920x1080 x 0.1 background, 20 736 pixels, is one chunk).
#define FAST_NMS_MAX_WORDS 4096
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
    int carry = 0;                                     // points of the chunks before this one
    for (int c0 = 0; c0 < words; c0 += FAST_NMS_MAX_WORDS) {
        const int cw = min(words - c0, FAST_NMS_MAX_WORDS);   // words of this chunk; s_* are indexed chunk-local
        for (int base = wid; base < cw; base += 32 * 4) {
            int sc[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int lw = base + 32 * u;
                const int i = ((c0 + lw) << 5) + lane;
                sc[u] = (lw < cw && i < n) ? (int)score[i] : 0;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int lw = base + 32 * u;              // warp-uniform
                if (lw >= cw) break;
                const int i = ((c0 + lw) << 5) + lane;
                bool ok = false;
                if (sc[u] != 0) {
                    // a non-zero score is an interior pixel; neighbours outside [3, w-3) x [3, h-3) have score 0
                    const int v = sc[u];
                    ok = v > score[i - 1] && v > score[i + 1] && v > score[i - w - 1] && v > score[i - w] &&
                         v > score[i - w + 1] && v > score[i + w - 1] && v > score[i + w] && v > score[i + w + 1] &&
                         mask[i] != 0;
                }
                const unsigned bal = __ballot_sync(0xffffffffu, ok);
                if (lane == 0) s_bits[lw] = bal;
            }
        }
        __syncthreads();
        // exclusive prefix of the word popcounts: thread t owns words 4t .. 4t+3
        int c[4], tot = 0;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int lw = 4 * tid + u;
            c[u] = lw < cw ? __popc(s_bits[lw]) : 0;
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
        }
        __syncthreads();
        int run = carry + v - tot + (wid ? s_warp[wid - 1] : 0);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int lw = 4 * tid + u;
            if (lw < cw) s_pref[lw] = run;
            run += c[u];
        }
        carry += s_warp[31];
        __syncthreads();
        for (int lw = wid; lw < cw; lw += 32) {
            const unsigned bal = s_bits[lw];
            if ((bal >> lane) & 1u) {
                const int pos = s_pref[lw] + __popc(bal & ((1u << lane) - 1u));
                if (pos < max_pts) {
                    const int i = ((c0 + lw) << 5) + lane;
                    const int y = i / w, x = i - y * w;
                    out_pts[2 * pos] = (float)x * unscale_x;      // _unscale_pts (flow.py:335-344)
                    out_pts[2 * pos + 1] = (float)y * unscale_y;
                }
            }
        }
        __syncthreads();                               // the next chunk rewrites s_bits, s_pref and s_warp
    }
    if (tid == 0) *out_count = min(carry, max_pts);
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
        // begins are clamped to max_pts so that an overflowing frame (meta[3]) never makes the per-track kernels read
        // past all_pts
        for (int k = 0; k < n_trk; ++k) {
            trk_begin[k] = min(acc, max_pts);
            acc += k < 2048 ? s_cnt[k] : min(kp_count[slots[k]], max_kp);
        }
        trk_begin[n_trk] = min(acc, max_pts);
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
        gftt_select_kernel<false><<<n_trk, kSelectThreads, 0, s>>>(owner, w, h, tlbr_pool, jobs, n_trk, scratch,
                                                                   quality, max_corners, kp_pool, kp_count, max_kp,
                                                                   status, scratch, scratch_counter, scratch_cap);
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
        gftt_select_kernel<true><<<n_trk, kSelectThreads, 0, s>>>(owner, w, h, tlbr_pool, jobs, n_trk, scratch,
                                                                  quality, max_corners, kp_pool, kp_count, max_kp,
                                                                  status, scratch, scratch_counter, scratch_cap);
    }
    FM_CHECK_LAUNCH("fm_flow_keypoints_cfg");
    return FM_OK;
}

extern "C" int fm_fast_detect(const unsigned char* img, const unsigned char* mask, int w, int h, int threshold,
                              float unscale_x, float unscale_y, unsigned char* score, float* out_pts, int* out_count,
                              int max_pts, void* stream) {
    FM_REQUIRE(threshold >= 0 && threshold <= 255, "fm_fast_detect: threshold must be in [0, 255]");
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid(fm_cdiv(w, 128), h);
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
