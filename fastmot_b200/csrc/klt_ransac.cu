// Robust motion models for the KLT stage, one CTA per model:
//   fm_ransac_homography          — camera motion from background matches  (fastmot/flow.py:215-232)
//   fm_ransac_affine_partial_batch — 4-dof similarity per track + box prediction + mask bookkeeping
//                                    (fastmot/flow.py:234-264, 274-279, 310-323)
//
// Both restate OpenCV's RANSACPointSetRegistrator (calib3d ptsetreg.cpp): RNG seeded with (uint64)-1,
// getSubset's rejection sampling, checkSubset, adaptive iteration count (RANSACUpdateNumIters), "first strictly
// better wins", followed by the Levenberg-Marquardt refinement of calib3d levmarq.cpp (lambda schedule
// Rlo/Rhi = 0.25/0.75, <= 10 iterations).  Hypotheses are evaluated in parallel batches and then scanned in
// OpenCV's sequential order, so the accepted model and iteration count are the ones the serial loop produces.
// The serial painting of predicted boxes into fg_mask is replaced by a fixed-point iteration over rounds
// (see fm_ransac_affine_partial_batch).
#include "common.cuh"
#include "../../include/fastmot_b200.h"
#include <float.h>

namespace {

// ------------------------------------------------------------------------------------------------ RNG
struct CvRng {
    unsigned long long state;
    __device__ unsigned next() {
        state = (unsigned long long)(unsigned)state * 4164903690ULL + (unsigned)(state >> 32);
        return (unsigned)state;
    }
    __device__ int uniform(int a, int b) { return a == b ? a : (int)(next() % (unsigned)(b - a) + a); }
};

__device__ int ransac_update_num_iters(double p, double ep, int model_points, int max_iters) {
    p = fmax(p, 0.); p = fmin(p, 1.);
    ep = fmax(ep, 0.); ep = fmin(ep, 1.);
    double num = fmax(1. - p, DBL_MIN);
    double denom = 1. - pow(1. - ep, (double)model_points);
    if (denom < DBL_MIN) return 0;
    num = log(num);
    denom = log(denom);
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : (int)rint(num / denom);
}

// ------------------------------------------------------------------------------------------------ block reduce
template <int N>
__device__ __forceinline__ void block_reduce(double* vals, double* s_red /* [nwarps][N] */, double* s_out /* [N] */) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < N; ++k) {
        double v = warp_sum(vals[k]);
        if (lane == 0) s_red[wid * N + k] = v;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < N; k += blockDim.x) {
        double a = 0.0;
        for (int w = 0; w < nw; ++w) a += s_red[w * N + k];
        s_out[k] = a;
    }
    __syncthreads();
}

// Gaussian elimination with partial pivoting, n <= 8, A is n x n row-major (destroyed), b -> x. Returns false if singular.
__device__ bool solve_dense(double* A, double* b, int n) {
    for (int c = 0; c < n; ++c) {
        int piv = c;
        double best = fabs(A[c * n + c]);
        for (int r = c + 1; r < n; ++r)
            if (fabs(A[r * n + c]) > best) { best = fabs(A[r * n + c]); piv = r; }
        if (!(best > 0.0)) return false;
        if (piv != c) {
            for (int k = 0; k < n; ++k) { double t = A[c * n + k]; A[c * n + k] = A[piv * n + k]; A[piv * n + k] = t; }
            double t = b[c]; b[c] = b[piv]; b[piv] = t;
        }
        const double inv = 1.0 / A[c * n + c];
        for (int r = c + 1; r < n; ++r) {
            const double f = A[r * n + c] * inv;
            if (f == 0.0) continue;
            for (int k = c; k < n; ++k) A[r * n + k] -= f * A[c * n + k];
            b[r] -= f * b[c];
        }
    }
    for (int r = n - 1; r >= 0; --r) {
        double v = b[r];
        for (int k = r + 1; k < n; ++k) v -= A[r * n + k] * b[k];
        b[r] = v / A[r * n + r];
    }
    return true;
}

// The same elimination run by one warp: lane k owns column k of the system (lane N the right-hand side), the pivot
// search and the row factors are computed redundantly from broadcast shared-memory reads, so every element sees the
// operations of solve_dense in the same order (bit-identical result) while a column step costs one dependent
// shared-memory round instead of ~N^2.  Call with all 32 lanes; A / b in shared memory.
template <int N>
__device__ __forceinline__ bool solve_dense_warp(double* A, double* b) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int c = 0; c < N; ++c) {
        int piv = c;
        double best = fabs(A[c * N + c]);
#pragma unroll
        for (int r = c + 1; r < N; ++r) {
            const double v = fabs(A[r * N + c]);
            if (v > best) { best = v; piv = r; }
        }
        if (!(best > 0.0)) return false;                 // warp-uniform
        __syncwarp();
        if (piv != c) {
            if (lane < N) { const double t = A[c * N + lane]; A[c * N + lane] = A[piv * N + lane]; A[piv * N + lane] = t; }
            else if (lane == N) { const double t = b[c]; b[c] = b[piv]; b[piv] = t; }
        }
        __syncwarp();
        const double inv = 1.0 / A[c * N + c];
        double f[N];
#pragma unroll
        for (int r = c + 1; r < N; ++r) f[r] = A[r * N + c] * inv;
        __syncwarp();                                    // every lane holds the factors before column c changes
        if (lane >= c && lane < N) {
            const double acl = A[c * N + lane];
#pragma unroll
            for (int r = c + 1; r < N; ++r)
                if (f[r] != 0.0) A[r * N + lane] -= f[r] * acl;
        } else if (lane == N) {
            const double bc = b[c];
#pragma unroll
            for (int r = c + 1; r < N; ++r)
                if (f[r] != 0.0) b[r] -= f[r] * bc;
        }
        __syncwarp();
    }
    if (lane == 0) {
        for (int r = N - 1; r >= 0; --r) {
            double v = b[r];
            for (int k = r + 1; k < N; ++k) v -= A[r * N + k] * b[k];
            b[r] = v / A[r * N + r];
        }
    }
    __syncwarp();
    return true;
}

// ------------------------------------------------------------------------------------------------ LM (levmarq.cpp)
// Problem concept: static const int NP; void accumulate(const double* x, bool need_jac, double* acc) where
// acc = [S, v[NP], A upper-triangular row-major NP(NP+1)/2]; block-parallel, result reduced into s_acc.
// The scalar bookkeeping between the block-wide passes (normal-equation solve, gain ratio, lambda schedule) is run
// by warp 0 cooperatively; it used to be one thread walking shared memory and was most of each iteration.
template <class Problem>
__device__ __forceinline__ void lm_refine(Problem& prob, double* x /* shared [NP] */, int max_iters, double* s_red,
                                          double* s_acc, double* s_work /* >= 3*NP*NP + 6*NP doubles */) {
    constexpr int NP = Problem::NP;
    constexpr int NA = 1 + NP + NP * (NP + 1) / 2;
    double* A = s_work;                 // NP*NP
    double* Ap = A + NP * NP;           // NP*NP
    double* v = Ap + NP * NP;           // NP
    double* d = v + NP;                 // NP
    double* xd = d + NP;                // NP
    double* Dg = xd + NP;               // NP
    double* tmp = Dg + NP;              // NP*NP + NP scratch
    __shared__ double s_S, s_lambda, s_lc;
    __shared__ int s_proceed;
    const int lane = threadIdx.x & 31;
    const bool w0 = threadIdx.x < 32;
    // unpack the reduced [S, v, upper(A)] into the symmetric matrix (warp 0; index map computed per element)
    auto unpack = [&]() {
        if (lane == 0) s_S = s_acc[0];
        if (lane < NP) v[lane] = s_acc[1 + lane];
        for (int e = lane; e < NP * NP; e += 32) {
            const int i = e / NP, j = e - i * NP;
            const int lo = i < j ? i : j, hi = i < j ? j : i;
            A[e] = s_acc[1 + NP + lo * NP - lo * (lo - 1) / 2 + (hi - lo)];
        }
    };
    double acc[NA];
    prob.accumulate(x, true, acc);
    block_reduce<NA>(acc, s_red, s_acc);
    if (w0) {
        unpack();
        __syncwarp();
        if (lane < NP) Dg[lane] = A[lane * NP + lane];
        if (lane == 0) { s_lambda = 1.0; s_lc = 0.75; s_proceed = 1; }
    }
    __syncthreads();
    for (int iter = 0; iter < max_iters; ++iter) {
        if (w0) {
            const double lambda = s_lambda;
            for (int e = lane; e < NP * NP; e += 32) {
                const int i = e / NP, j = e - i * NP;
                Ap[e] = A[e] + (i == j ? Dg[i] * lambda : 0.0);
            }
            if (lane < NP) d[lane] = v[lane];
            __syncwarp();
            const bool ok = solve_dense_warp<NP>(Ap, d);
            if (lane < NP) {
                if (!ok) d[lane] = 0.0;
                xd[lane] = x[lane] - d[lane];
            }
        }
        __syncthreads();
        prob.accumulate(xd, false, acc);
        block_reduce<1>(acc, s_red, s_acc);      // only the residual norm is needed for the trial step
        const bool improved = s_acc[0] < s_S;
        if (w0) {
            const double Sd = s_acc[0], S = s_S;
            // dS = sum_i d_i (2 v_i - (A d)_i), dv = d.v, dinf = max |d_i|: lane i forms its term, lane 0 adds them
            // in index order (the order of the scalar loop)
            double term_s = 0.0, term_v = 0.0, term_i = 0.0;
            if (lane < NP) {
                double Ad = 0.0;
                for (int j = 0; j < NP; ++j) Ad += A[lane * NP + j] * d[j];
                term_s = d[lane] * (2.0 * v[lane] - Ad);
                term_v = d[lane] * v[lane];
                term_i = fabs(d[lane]);
            }
            double dS = 0.0, dv = 0.0, dinf = 0.0;
#pragma unroll
            for (int i = 0; i < NP; ++i) {
                dS += __shfl_sync(0xffffffffu, term_s, i);
                dv += __shfl_sync(0xffffffffu, term_v, i);
                dinf = fmax(dinf, __shfl_sync(0xffffffffu, term_i, i));
            }
            const double R = (S - Sd) / (fabs(dS) > DBL_EPSILON ? dS : 1.0);
            double lambda = s_lambda, lc = s_lc;       // every lane tracks the schedule; lane 0 publishes it
            if (R > 0.75) {
                lambda *= 0.5;
                if (lambda < lc) lambda = 0.0;
            } else if (R < 0.25) {
                double nu = (Sd - S) / (fabs(dv) > DBL_EPSILON ? dv : 1.0) + 2.0;
                nu = fmin(fmax(nu, 2.0), 10.0);
                if (lambda == 0.0) {
                    // lambda = lc = 1 / max |diag(A^-1)|
                    double maxval = DBL_EPSILON;
                    for (int c = 0; c < NP; ++c) {
                        __syncwarp();
                        for (int e = lane; e < NP * NP; e += 32) tmp[e] = A[e];
                        double* ev = tmp + NP * NP;
                        if (lane < NP) ev[lane] = (lane == c) ? 1.0 : 0.0;
                        __syncwarp();
                        if (solve_dense_warp<NP>(tmp, ev)) maxval = fmax(maxval, fabs(ev[c]));
                    }
                    lambda = lc = 1.0 / maxval;
                    nu *= 0.5;
                }
                lambda *= nu;
            }
            __syncwarp();
            if (lane == 0) { s_lambda = lambda; s_lc = lc; tmp[0] = dinf; }
        }
        __syncthreads();
        if (improved) {
            if (threadIdx.x < NP) x[threadIdx.x] = xd[threadIdx.x];
            __syncthreads();
            prob.accumulate(x, true, acc);
            block_reduce<NA>(acc, s_red, s_acc);
            if (w0) unpack();
        }
        if (threadIdx.x == 0) {
            // proceed = iter+1 < maxIters && |d|_inf >= eps && |r|_inf >= eps (r_inf approximated by sqrt(S)).
            // OpenCV uses eps = FLT_EPSILON on |d|_inf, which in practice runs all 10 iterations; the step norm
            // shrinks quadratically, so we stop once a step is below 1e-9 (parameter change invisible at 1e-9).
            s_proceed = (tmp[0] >= 1e-9) && (sqrt(s_S) >= FLT_EPSILON);
        }
        __syncthreads();
        if (!s_proceed) break;
    }
}

// ------------------------------------------------------------------------------------------------ affine partial
struct AffineProblem {
    static const int NP = 4;
    const float* src;
    const float* dst;
    const int* idx;  // inlier index list
    int n;
    __device__ __forceinline__ void accumulate(const double* h, bool need_jac, double* acc) const {
        constexpr int NA = 1 + 4 + 10;
#pragma unroll
        for (int k = 0; k < NA; ++k) acc[k] = 0.0;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int p = idx[i];
            const double Mx = src[2 * p], My = src[2 * p + 1];
            const double ex = h[0] * Mx - h[1] * My + h[2] - dst[2 * p];
            const double ey = h[1] * Mx + h[0] * My + h[3] - dst[2 * p + 1];
            acc[0] += ex * ex + ey * ey;
            if (need_jac) {
                const double J0[4] = {Mx, -My, 1.0, 0.0}, J1[4] = {My, Mx, 0.0, 1.0};
                int q = 5;
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    acc[1 + a] += J0[a] * ex + J1[a] * ey;
#pragma unroll
                    for (int b = a; b < 4; ++b) acc[q++] += J0[a] * J0[b] + J1[a] * J1[b];
                }
            }
        }
    }
};

struct HomographyProblem {
    static const int NP = 8;
    const float* src;
    const float* dst;
    const int* idx;
    int n;
    const float4* cache;   // optional shared-memory copy of the n inlier pairs (src.x, src.y, dst.x, dst.y)
    __device__ __forceinline__ void accumulate(const double* h, bool need_jac, double* acc) const {
        constexpr int NA = 1 + 8 + 36;
#pragma unroll
        for (int k = 0; k < NA; ++k) acc[k] = 0.0;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            // every LM pass re-reads all pairs: from the cache when they fit (two dependent L2 round trips per pass
            // were ~60 % of the kernel's stall samples)
            float4 pr;
            if (cache) pr = cache[i];
            else { const int p = idx[i]; pr = make_float4(src[2 * p], src[2 * p + 1], dst[2 * p], dst[2 * p + 1]); }
            const double Mx = pr.x, My = pr.y;
            double ww = h[6] * Mx + h[7] * My + 1.0;
            ww = fabs(ww) > DBL_EPSILON ? 1.0 / ww : 0.0;
            const double xi = (h[0] * Mx + h[1] * My + h[2]) * ww, yi = (h[3] * Mx + h[4] * My + h[5]) * ww;
            const double ex = xi - pr.z, ey = yi - pr.w;
            acc[0] += ex * ex + ey * ey;
            if (need_jac) {
                const double J0[8] = {Mx * ww, My * ww, ww, 0, 0, 0, -Mx * ww * xi, -My * ww * xi};
                const double J1[8] = {0, 0, 0, Mx * ww, My * ww, ww, -Mx * ww * yi, -My * ww * yi};
                int q = 9;
#pragma unroll
                for (int a = 0; a < 8; ++a) {
                    acc[1 + a] += J0[a] * ex + J1[a] * ey;
#pragma unroll
                    for (int b = a; b < 8; ++b) acc[q++] += J0[a] * J0[b] + J1[a] * J1[b];
                }
            }
        }
    }
};

// 2-point similarity (AffinePartial2DEstimatorCallback::runKernel)
__device__ void affine_partial_from2(const float* f0, const float* f1, const float* t0, const float* t1, double* M) {
    const double x1 = f0[0], y1 = f0[1], x2 = f1[0], y2 = f1[1];
    const double X1 = t0[0], Y1 = t0[1], X2 = t1[0], Y2 = t1[1];
    const double d = 1. / ((x1 - x2) * (x1 - x2) + (y1 - y2) * (y1 - y2));
    const double S0 = d * ((X1 - X2) * (x1 - x2) + (Y1 - Y2) * (y1 - y2));
    const double S1 = d * ((Y1 - Y2) * (x1 - x2) - (X1 - X2) * (y1 - y2));
    const double S2 = d * ((Y1 - Y2) * (x1 * y2 - x2 * y1) - (X1 * y2 - X2 * y1) * (y1 - y2) - (X1 * x2 - X2 * x1) * (x1 - x2));
    const double S3 = d * (-(X1 - X2) * (x1 * y2 - x2 * y1) - (Y1 * x2 - Y2 * x1) * (x1 - x2) - (Y1 * y2 - Y2 * y1) * (y1 - y2));
    M[0] = S0; M[1] = -S1; M[2] = S2;
    M[3] = S1; M[4] = S0; M[5] = S3;
}

// Affine2DEstimatorCallback::computeError: the model rounded to float and the residual formed in float, each operation
// rounded on its own (no FMA contraction), so a point within rounding of the threshold falls on OpenCV's side of it
__device__ __forceinline__ bool affine_inlier(const double* F, const float* f, const float* t, double thr2) {
    const float a = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn((float)F[0], f[0]), __fmul_rn((float)F[1], f[1])),
                                        (float)F[2]), t[0]);
    const float b = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn((float)F[3], f[0]), __fmul_rn((float)F[4], f[1])),
                                        (float)F[5]), t[1]);
    const float e = __fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b));
    return (double)e <= thr2;
}

#define AFF_MAX_PTS 1024
#define AFF_BATCH 32

// One CTA (128 threads) per track per round.  kMaxPts bounds the points of one track: AFF_MAX_PTS when a track keeps
// at most 1024 keypoints (goodFeaturesToTrack's default settings), AFF_MAX_PTS_LARGE when maxCorners allows more.
#define AFF_MAX_PTS_LARGE 4096
template <int kMaxPts>
__global__ void __launch_bounds__(128) affine_partial_kernel(
    const float* __restrict__ all_prev, const float* __restrict__ all_cur, const unsigned char* __restrict__ status,
    const int* __restrict__ trk_begin, const int* __restrict__ slots, int n_trk, int round,
    const int* __restrict__ round_changed_prev, int* __restrict__ round_changed, const int* __restrict__ h_ok,
    const int* __restrict__ est_prev /* [n_trk][5] x0,y0,x1,y1,valid */, int* __restrict__ est_cur,
    unsigned long long* __restrict__ sig, double* __restrict__ tlbr_pool, double* __restrict__ klt_tlbr,
    unsigned char* __restrict__ klt_ok, double* __restrict__ inlier_ratio, float* __restrict__ kp_pool,
    float* __restrict__ kp_prev_pool, int* __restrict__ kp_count, int max_kp, int frame_w, int frame_h, int max_iters,
    double confidence, double thresh, int inlier_thresh, int refine_iters) {
    __shared__ int s_idx[kMaxPts];
    __shared__ int s_inl[kMaxPts];
    __shared__ int s_sub[AFF_BATCH][2];
    __shared__ double s_model[AFF_BATCH][6];
    __shared__ int s_cnt[AFF_BATCH];
    __shared__ double s_best[6], s_x[4];
    __shared__ double s_red[4 * 15], s_acc[15], s_work[3 * 16 + 6 * 4 + 4];
    __shared__ int s_n, s_ninl, s_done, s_niters, s_maxgood, s_iter, s_warpcnt[4];
    __shared__ unsigned long long s_hash;
    const int k = blockIdx.x;
    if (k >= n_trk) return;
    if (h_ok && *h_ok == 0) return;                          // camera motion failed: nothing is predicted
    if (round > 0 && round_changed_prev[0] == 0) return;     // fixed point already reached
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int slot = slots[k];
    const int beg = trk_begin[k], end = trk_begin[k + 1];
    // ---- _get_good_match + _fg_filter (ordered compaction) ----
    if (tid == 0) { s_n = 0; s_hash = 1469598103934665603ULL; }
    __syncthreads();
    for (int base = beg; base < end; base += blockDim.x) {
        const int i = base + tid;
        bool keep = false;
        if (i < end && status[i]) {
            const int xi = (int)rintf(all_cur[2 * i]), yi = (int)rintf(all_cur[2 * i + 1]);
            keep = xi >= 0 && yi >= 0 && xi < frame_w && yi < frame_h;
            for (int j = 0; keep && j < k; ++j) {
                const int* e = est_prev + j * 5;
                if (e[4] && xi >= e[0] && xi <= e[2] && yi >= e[1] && yi <= e[3]) keep = false;
            }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warpcnt[wid] = __popc(bal);
        __syncthreads();
        int off = s_n;
        for (int w = 0; w < wid; ++w) off += s_warpcnt[w];
        off += __popc(bal & ((1u << lane) - 1));
        if (keep && off < kMaxPts) s_idx[off] = i;
        __syncthreads();
        if (tid == 0) s_n = min(s_n + s_warpcnt[0] + s_warpcnt[1] + s_warpcnt[2] + s_warpcnt[3], kMaxPts);
        __syncthreads();
    }
    const int m = s_n;
    // signature of the filtered set: FNV over indices (thread 0; m is small)
    if (tid == 0) {
        unsigned long long hsh = s_hash;
        for (int i = 0; i < m; ++i) { hsh ^= (unsigned long long)(s_idx[i] - beg + 1); hsh *= 1099511628211ULL; }
        hsh ^= (unsigned long long)m << 48;
        s_hash = hsh | 1ULL;
    }
    __syncthreads();
    int* ecur = est_cur + k * 5;
    if (round > 0 && sig[k] == s_hash) {
        if (tid < 5) ecur[tid] = est_prev[k * 5 + tid];      // result stands
        return;
    }
    if (tid == 0) { sig[k] = s_hash; atomicExch(round_changed, 1); }
    // ---- failure defaults ----
    auto fail = [&]() {
        if (tid == 0) {
            kp_count[slot] = 0;
            klt_ok[slot] = 0;
            ecur[0] = ecur[1] = ecur[2] = ecur[3] = 0; ecur[4] = 0;
        }
    };
    if (m < 3) { fail(); return; }
    // ---- RANSAC ----
    const double thr2 = thresh * thresh;
    __shared__ CvRng s_rng;
    if (tid == 0) { s_rng.state = 0xffffffffffffffffULL; s_niters = max(max_iters, 1); s_maxgood = 0; s_iter = 0; s_done = 0; }
    __syncthreads();
    while (true) {
        if (tid == 0) {
            for (int h = 0; h < AFF_BATCH; ++h) {   // getSubset: two distinct indices, no degeneracy test for 2 points
                int i0 = s_rng.uniform(0, m), i1;
                for (i1 = s_rng.uniform(0, m); i1 == i0; i1 = s_rng.uniform(0, m)) {}
                s_sub[h][0] = i0; s_sub[h][1] = i1;
            }
        }
        __syncthreads();
        if (tid < AFF_BATCH) {
            const int a = s_idx[s_sub[tid][0]], b = s_idx[s_sub[tid][1]];
            affine_partial_from2(all_prev + 2 * a, all_prev + 2 * b, all_cur + 2 * a, all_cur + 2 * b, s_model[tid]);
        }
        __syncthreads();
        {
            const int h = tid >> 2, part = tid & 3;
            int c = 0;
            for (int i = part; i < m; i += 4) {
                const int p = s_idx[i];
                c += affine_inlier(s_model[h], all_prev + 2 * p, all_cur + 2 * p, thr2);
            }
            c += __shfl_xor_sync(0xffffffffu, c, 1);
            c += __shfl_xor_sync(0xffffffffu, c, 2);
            if (part == 0) s_cnt[h] = c;
        }
        __syncthreads();
        if (tid == 0) {
            // replay of the sequential loop over this batch; the RNG draws of the unused tail are discarded,
            // exactly as if the serial loop had stopped
            for (int h = 0; h < AFF_BATCH; ++h) {
                if (s_iter >= s_niters) { s_done = 1; break; }
                const int good = s_cnt[h];
                if (good > max(s_maxgood, 1)) {
                    for (int q = 0; q < 6; ++q) s_best[q] = s_model[h][q];
                    s_maxgood = good;
                    s_niters = ransac_update_num_iters(confidence, (double)(m - good) / m, 2, s_niters);
                }
                ++s_iter;
            }
            if (s_iter >= s_niters) s_done = 1;
        }
        __syncthreads();
        if (s_done) break;
    }
    if (s_maxgood == 0) { fail(); return; }
    // ---- inlier set of the best model, ordered ----
    if (tid == 0) s_ninl = 0;
    __syncthreads();
    for (int base = 0; base < m; base += blockDim.x) {
        const int i = base + tid;
        bool in = false;
        if (i < m) { const int p = s_idx[i]; in = affine_inlier(s_best, all_prev + 2 * p, all_cur + 2 * p, thr2); }
        const unsigned bal = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_warpcnt[wid] = __popc(bal);
        __syncthreads();
        int off = s_ninl;
        for (int w = 0; w < wid; ++w) off += s_warpcnt[w];
        off += __popc(bal & ((1u << lane) - 1));
        if (in) s_inl[off] = s_idx[i];
        __syncthreads();
        if (tid == 0) s_ninl += s_warpcnt[0] + s_warpcnt[1] + s_warpcnt[2] + s_warpcnt[3];
        __syncthreads();
    }
    const int n_in = s_ninl;
    // ---- LM refinement of (a, b, tx, ty) on the inliers ----
    if (tid == 0) { s_x[0] = s_best[0]; s_x[1] = s_best[3]; s_x[2] = s_best[2]; s_x[3] = s_best[5]; }
    __syncthreads();
    if (refine_iters > 0) {
        AffineProblem prob{all_prev, all_cur, s_inl, n_in};
        lm_refine(prob, s_x, refine_iters, s_red, s_acc, s_work);
    }
    __syncthreads();
    // ---- _estimate_bbox (flow.py:274-279) + acceptance tests (flow.py:251-256) ----
    __shared__ int s_ok;
    __shared__ double s_box[4];
    if (tid == 0) {
        const double a = s_x[0], b = s_x[1], tx = s_x[2], ty = s_x[3];
        const double* t = tlbr_pool + (size_t)slot * 4;
        const double nx = a * t[0] - b * t[1] + tx, ny = b * t[0] + a * t[1] + ty;
        double scale = sqrt(a * a + b * b);
        if (scale < 0.9 || scale > 1.1) scale = 1.0;
        const double w = t[2] - t[0] + 1.0, h = t[3] - t[1] + 1.0;
        const double x1 = rint(nx), y1 = rint(ny), x2 = rint(nx + w * scale - 1.0), y2 = rint(ny + h * scale - 1.0);
        const bool isect = !(fmin(x2, frame_w - 1.0) < fmax(x1, 0.0) || fmin(y2, frame_h - 1.0) < fmax(y1, 0.0));
        const bool ok = isect && n_in >= inlier_thresh && !(isnan(x1) || isnan(y1) || isnan(x2) || isnan(y2));
        s_ok = ok;
        s_box[0] = x1; s_box[1] = y1; s_box[2] = x2; s_box[3] = y2;
        if (ok) {
            klt_tlbr[(size_t)slot * 4 + 0] = x1; klt_tlbr[(size_t)slot * 4 + 1] = y1;
            klt_tlbr[(size_t)slot * 4 + 2] = x2; klt_tlbr[(size_t)slot * 4 + 3] = y2;
            klt_ok[slot] = 1;
            inlier_ratio[slot] = (double)n_in / (double)m;
            // crop(fg_mask, est_tlbr)[:] = 0  (rect.py:82-89): int truncation, lower clamp; numpy clamps the upper
            ecur[0] = max((int)x1, 0); ecur[1] = max((int)y1, 0); ecur[2] = max((int)x2, 0); ecur[3] = max((int)y2, 0);
            ecur[4] = 1;
            kp_count[slot] = min(n_in, max_kp);
        }
    }
    __syncthreads();
    if (!s_ok) {
        // note: the reference assigns prev_keypoints/keypoints before this test; keypoints end up empty
        fail();
        return;
    }
    float* kp = kp_pool + (size_t)slot * max_kp * 2;
    float* kpp = kp_prev_pool + (size_t)slot * max_kp * 2;
    for (int i = tid; i < min(n_in, max_kp); i += blockDim.x) {
        const int p = s_inl[i];
        kp[2 * i] = all_cur[2 * p]; kp[2 * i + 1] = all_cur[2 * p + 1];
        kpp[2 * i] = all_prev[2 * p]; kpp[2 * i + 1] = all_prev[2 * p + 1];
    }
}

// ------------------------------------------------------------------------------------------------ homography
__device__ bool have_collinear(const float* pts /* 4 x 2 */, int count) {
    const int i = count - 1;
    for (int j = 0; j < i; ++j) {
        const double dx1 = pts[2 * j] - pts[2 * i], dy1 = pts[2 * j + 1] - pts[2 * i + 1];
        for (int kk = 0; kk < j; ++kk) {
            const double dx2 = pts[2 * kk] - pts[2 * i], dy2 = pts[2 * kk + 1] - pts[2 * i + 1];
            if (fabs(dx2 * dy1 - dy2 * dx1) <= FLT_EPSILON * (fabs(dx1) + fabs(dy1) + fabs(dx2) + fabs(dy2))) return true;
        }
    }
    return false;
}

__device__ double det3(const float* a, const float* b, const float* c) {
    // rows (x, y, 1)
    return (double)a[0] * ((double)b[1] - (double)c[1]) - (double)a[1] * ((double)b[0] - (double)c[0]) +
           ((double)b[0] * (double)c[1] - (double)b[1] * (double)c[0]);
}

__device__ bool homography_check_subset(const float* s, const float* d) {
    if (have_collinear(s, 4) || have_collinear(d, 4)) return false;
    const int tt[4][3] = {{0, 1, 2}, {1, 2, 3}, {0, 2, 3}, {0, 1, 3}};
    int negative = 0;
    for (int i = 0; i < 4; ++i) {
        const int* t = tt[i];
        const double A = det3(s + 2 * t[0], s + 2 * t[1], s + 2 * t[2]);
        const double B = det3(d + 2 * t[0], d + 2 * t[1], d + 2 * t[2]);
        negative += A * B < 0;
    }
    return negative == 0 || negative == 4;
}

// Normalised DLT for n >= 4 correspondences given the 9x9 normal matrix LtL: smallest eigenvector by Jacobi rotations.
// One warp, round-robin ("chess tournament") ordering: each of the 9 rounds of a sweep applies 4 rotations on disjoint
// index pairs at once -- lanes 0..3 derive the angles, then 36 (rotation, row) tasks update the columns of A and V and
// 36 more the rows of A.  A sweep is 9 dependent steps instead of 36; every rotation is the textbook one
// (t = sgn(theta) / (|theta| + sqrt(theta^2 + 1))), only their order differs from a cyclic-by-row sweep, which changes
// the result at rounding level (H is refined by LM afterwards).  The serial sweep on one thread was far slower.
__device__ void jacobi_smallest_eigvec9_warp(double* Amat /* 81, destroyed */, double* Vmat /* 81 */,
                                             double* out9 /* shared */) {
    constexpr int n = 9;
    __shared__ double s_cs[4][2];
    __shared__ int s_pq[4][2];
    const int lane = threadIdx.x & 31;
    for (int i = lane; i < n * n; i += 32) Vmat[i] = (i / n == i % n) ? 1.0 : 0.0;
    __syncwarp();
    for (int sweep = 0; sweep < 30; ++sweep) {
        bool rotated = false;
        for (int round = 0; round < n; ++round) {
            bool act = false;
            if (lane < 4) {
                int p = (round + lane + 1) % n, q = (round - (lane + 1) + n) % n;
                if (p > q) { const int t = p; p = q; q = t; }
                const double apq = Amat[p * n + q], app = Amat[p * n + p], aqq = Amat[q * n + q];
                double c = 1.0, sn = 0.0;
                // off-diagonal already below double rounding of the diagonal pair: nothing left to annihilate
                if (fabs(apq) > 1e-17 * (fabs(app) + fabs(aqq))) {
                    act = true;
                    const double theta = (aqq - app) / (2.0 * apq);
                    const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                    c = 1.0 / sqrt(t * t + 1.0);
                    sn = t * c;
                }
                s_cs[lane][0] = c; s_cs[lane][1] = sn;
                s_pq[lane][0] = p; s_pq[lane][1] = act ? q : -1;
            }
            const unsigned any = __ballot_sync(0xffffffffu, act);
            if (!any) continue;                               // warp-uniform
            rotated = true;
            __syncwarp();
            for (int idx = lane; idx < 4 * n; idx += 32) {     // columns p, q of A and V, row r
                const int k = idx / n, r = idx - k * n;
                const int p = s_pq[k][0], q = s_pq[k][1];
                if (q < 0) continue;
                const double c = s_cs[k][0], sn = s_cs[k][1];
                const double arp = Amat[r * n + p], arq = Amat[r * n + q];
                Amat[r * n + p] = c * arp - sn * arq;
                Amat[r * n + q] = sn * arp + c * arq;
                const double vrp = Vmat[r * n + p], vrq = Vmat[r * n + q];
                Vmat[r * n + p] = c * vrp - sn * vrq;
                Vmat[r * n + q] = sn * vrp + c * vrq;
            }
            __syncwarp();
            for (int idx = lane; idx < 4 * n; idx += 32) {     // rows p, q of A, column r
                const int k = idx / n, r = idx - k * n;
                const int p = s_pq[k][0], q = s_pq[k][1];
                if (q < 0) continue;
                const double c = s_cs[k][0], sn = s_cs[k][1];
                const double apr = Amat[p * n + r], aqr = Amat[q * n + r];
                Amat[p * n + r] = c * apr - sn * aqr;
                Amat[q * n + r] = sn * apr + c * aqr;
            }
            __syncwarp();
        }
        if (!rotated) break;
    }
    if (lane == 0) {
        int best = 0;
        for (int i = 1; i < n; ++i)
            if (Amat[i * n + i] < Amat[best * n + best]) best = i;
        for (int r = 0; r < n; ++r) out9[r] = Vmat[r * n + best];
    }
    __syncwarp();
}

__device__ void denormalise_h(const double* H0, const double* cm, const double* sm, const double* cM, const double* sM,
                              double* H) {
    // H = invHnorm * H0 * Hnorm2 ; invHnorm = [1/sm.x 0 cm.x; 0 1/sm.y cm.y; 0 0 1], Hnorm2 = [sM.x 0 -cM.x sM.x; ...]
    double T[9];
    for (int c = 0; c < 3; ++c) {
        T[0 * 3 + c] = H0[0 * 3 + c] / sm[0] + cm[0] * H0[2 * 3 + c];
        T[1 * 3 + c] = H0[1 * 3 + c] / sm[1] + cm[1] * H0[2 * 3 + c];
        T[2 * 3 + c] = H0[2 * 3 + c];
    }
    for (int r = 0; r < 3; ++r) {
        H[r * 3 + 0] = T[r * 3 + 0] * sM[0];
        H[r * 3 + 1] = T[r * 3 + 1] * sM[1];
        H[r * 3 + 2] = -T[r * 3 + 0] * cM[0] * sM[0] - T[r * 3 + 1] * cM[1] * sM[1] + T[r * 3 + 2];
    }
    const double inv = 1.0 / H[8];
    for (int i = 0; i < 9; ++i) H[i] *= inv;
}

// 4-point homography: same normalisation as OpenCV, exact 8x8 solve instead of the 9x9 eigen problem.
__device__ bool homography_from4(const float* M /* src 4x2 */, const float* mm /* dst 4x2 */, double* H) {
    double cM[2] = {0, 0}, cm[2] = {0, 0}, sM[2] = {0, 0}, sm[2] = {0, 0};
    for (int i = 0; i < 4; ++i) { cm[0] += mm[2 * i]; cm[1] += mm[2 * i + 1]; cM[0] += M[2 * i]; cM[1] += M[2 * i + 1]; }
    for (int c = 0; c < 2; ++c) { cm[c] /= 4; cM[c] /= 4; }
    for (int i = 0; i < 4; ++i) {
        sm[0] += fabs(mm[2 * i] - cm[0]); sm[1] += fabs(mm[2 * i + 1] - cm[1]);
        sM[0] += fabs(M[2 * i] - cM[0]); sM[1] += fabs(M[2 * i + 1] - cM[1]);
    }
    if (fabs(sm[0]) < DBL_EPSILON || fabs(sm[1]) < DBL_EPSILON || fabs(sM[0]) < DBL_EPSILON || fabs(sM[1]) < DBL_EPSILON)
        return false;
    for (int c = 0; c < 2; ++c) { sm[c] = 4 / sm[c]; sM[c] = 4 / sM[c]; }
    double A[64], b[8];
    for (int i = 0; i < 4; ++i) {
        const double x = (mm[2 * i] - cm[0]) * sm[0], y = (mm[2 * i + 1] - cm[1]) * sm[1];
        const double X = (M[2 * i] - cM[0]) * sM[0], Y = (M[2 * i + 1] - cM[1]) * sM[1];
        double* r0 = A + (2 * i) * 8;
        double* r1 = A + (2 * i + 1) * 8;
        r0[0] = X; r0[1] = Y; r0[2] = 1; r0[3] = 0; r0[4] = 0; r0[5] = 0; r0[6] = -x * X; r0[7] = -x * Y; b[2 * i] = x;
        r1[0] = 0; r1[1] = 0; r1[2] = 0; r1[3] = X; r1[4] = Y; r1[5] = 1; r1[6] = -y * X; r1[7] = -y * Y; b[2 * i + 1] = y;
    }
    if (!solve_dense(A, b, 8)) return false;
    double H0[9] = {b[0], b[1], b[2], b[3], b[4], b[5], b[6], b[7], 1.0};
    denormalise_h(H0, cm, sm, cM, sM, H);
    return true;
}

// HomographyEstimatorCallback::computeError in float, each operation rounded on its own (no FMA contraction)
__device__ __forceinline__ bool homography_inlier(const float* Hf, const float* M, const float* m, double thr2) {
    const float ww = __fdiv_rn(1.f, __fadd_rn(__fadd_rn(__fmul_rn(Hf[6], M[0]), __fmul_rn(Hf[7], M[1])), 1.f));
    const float dx = __fsub_rn(__fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(Hf[0], M[0]), __fmul_rn(Hf[1], M[1])), Hf[2]), ww),
                               m[0]);
    const float dy = __fsub_rn(__fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(Hf[3], M[0]), __fmul_rn(Hf[4], M[1])), Hf[5]), ww),
                               m[1]);
    const float e = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
    return (double)e <= thr2;
}

#define HOM_BATCH 8
// optional phase timestamps of the homography kernel (scripts/profile_flow.py; not part of the public ABI)
__device__ unsigned long long* g_hom_dbg = nullptr;
#define HOM_STAMP(k)                                                               \
    do {                                                                           \
        if (g_hom_dbg && threadIdx.x == 0) {                                       \
            unsigned long long t_;                                                 \
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));                  \
            g_hom_dbg[(k)] = t_;                                                   \
        }                                                                          \
    } while (0)
#define HOM_CACHE 1536   // inlier pairs kept in shared memory for the LM passes (24 KB)
__global__ void __launch_bounds__(256) homography_kernel(const float* __restrict__ all_prev,
                                                          const float* __restrict__ all_cur,
                                                          const unsigned char* __restrict__ status,
                                                          const int* __restrict__ meta, int max_iters,
                                                          double confidence, double thresh, int inlier_thresh,
                                                          int* __restrict__ good_idx /* scratch >= max bg */,
                                                          int* __restrict__ inl_idx, double* __restrict__ H_out,
                                                          int* __restrict__ h_ok, float* __restrict__ bg_kp,
                                                          float* __restrict__ bg_kp_prev, int* __restrict__ bg_kp_count,
                                                          int max_bg) {
    __shared__ int s_n, s_warpcnt[8], s_sub[HOM_BATCH][4], s_subok[HOM_BATCH], s_cnt[HOM_BATCH];
    __shared__ double s_H[HOM_BATCH][9], s_best[9], s_x[8];
    __shared__ float s_Hf[HOM_BATCH][8];
    __shared__ int s_done, s_niters, s_maxgood, s_iter, s_fail, s_ninl;
    __shared__ double s_red[8 * 45], s_acc[45], s_work[3 * 64 + 6 * 8 + 8];
    __shared__ double s_LtL[81], s_V[81], s_nrm[8], s_h9[9];
    __shared__ CvRng s_rng;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    HOM_STAMP(0);
    const int bg_begin = meta[0];
    const int bg_end = meta[1] - 1;  // `_get_good_match(..., bg_begin, -1)` drops the last point (flow.py:216-217)
    if (tid == 0) { s_n = 0; s_fail = 0; }
    __syncthreads();
    for (int base = bg_begin; base < bg_end; base += blockDim.x) {
        const int i = base + tid;
        const bool keep = i < bg_end && status[i];
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warpcnt[wid] = __popc(bal);
        __syncthreads();
        int off = s_n;
        for (int w = 0; w < wid; ++w) off += s_warpcnt[w];
        off += __popc(bal & ((1u << lane) - 1));
        if (keep && off < max_bg) good_idx[off] = i;
        __syncthreads();
        if (tid == 0) {
            int t = 0;
            for (int w = 0; w < 8; ++w) t += s_warpcnt[w];
            s_n = min(s_n + t, max_bg);
        }
        __syncthreads();
    }
    const int n = s_n;
    auto fail_out = [&]() {
        if (tid == 0) { *h_ok = 0; *bg_kp_count = 0; }
    };
    if (n < 4) { fail_out(); return; }
    const double thr2 = thresh * thresh;
    if (n == 4) {
        // method 0: plain least squares on the four matches, every point is an inlier, no LM
        if (tid == 0) {
            float M[8], mm[8];
            for (int i = 0; i < 4; ++i) {
                const int p = good_idx[i];
                M[2 * i] = all_prev[2 * p]; M[2 * i + 1] = all_prev[2 * p + 1];
                mm[2 * i] = all_cur[2 * p]; mm[2 * i + 1] = all_cur[2 * p + 1];
            }
            double H[9];
            if (!homography_from4(M, mm, H)) s_fail = 1;
            else {
                for (int i = 0; i < 9; ++i) H_out[i] = H[i];
                for (int i = 0; i < 4; ++i) {
                    bg_kp[2 * i] = mm[2 * i]; bg_kp[2 * i + 1] = mm[2 * i + 1];
                    bg_kp_prev[2 * i] = M[2 * i]; bg_kp_prev[2 * i + 1] = M[2 * i + 1];
                }
                *bg_kp_count = 4;
                *h_ok = 4 >= inlier_thresh ? 1 : 0;
                if (4 < inlier_thresh) *bg_kp_count = 0;
            }
        }
        __syncthreads();
        if (s_fail) fail_out();
        return;
    }
    HOM_STAMP(1);
    // niters = MAX(maxIters, 1): one hypothesis is drawn even when maxIters is 0
    if (tid == 0) { s_rng.state = 0xffffffffffffffffULL; s_niters = max(max_iters, 1); s_maxgood = 0; s_iter = 0; s_done = 0; }
    __syncthreads();
    while (true) {
        if (tid == 0) {
            for (int h = 0; h < HOM_BATCH; ++h) {
                bool found = false;
                for (int attempt = 0; attempt < 10000 && !found; ++attempt) {
                    int idx[4];
                    float S[8], D[8];
                    for (int i = 0; i < 4; ++i) {
                        int v;
                        while (true) {
                            v = s_rng.uniform(0, n);
                            bool dup = false;
                            for (int q = 0; q < i; ++q) dup = dup || idx[q] == v;
                            if (!dup) break;
                        }
                        idx[i] = v;
                        const int p = good_idx[v];
                        S[2 * i] = all_prev[2 * p]; S[2 * i + 1] = all_prev[2 * p + 1];
                        D[2 * i] = all_cur[2 * p]; D[2 * i + 1] = all_cur[2 * p + 1];
                    }
                    if (homography_check_subset(S, D)) {
                        found = true;
                        for (int i = 0; i < 4; ++i) s_sub[h][i] = idx[i];
                    }
                }
                s_subok[h] = found;
            }
        }
        __syncthreads();
        if (tid < HOM_BATCH) {
            bool ok = s_subok[tid];
            if (ok) {
                float S[8], D[8];
                for (int i = 0; i < 4; ++i) {
                    const int p = good_idx[s_sub[tid][i]];
                    S[2 * i] = all_prev[2 * p]; S[2 * i + 1] = all_prev[2 * p + 1];
                    D[2 * i] = all_cur[2 * p]; D[2 * i + 1] = all_cur[2 * p + 1];
                }
                ok = homography_from4(S, D, s_H[tid]);
            }
            s_cnt[tid] = ok ? 0 : -1;      // -1: runKernel produced no model
            for (int q = 0; q < 8; ++q) s_Hf[tid][q] = ok ? (float)s_H[tid][q] : 0.f;
        }
        __syncthreads();
        {   // warp `wid` counts inliers of hypothesis `wid`
            int c = 0;
            if (s_cnt[wid] == 0) {
                for (int i = lane; i < n; i += 32) {
                    const int p = good_idx[i];
                    c += homography_inlier(s_Hf[wid], all_prev + 2 * p, all_cur + 2 * p, thr2);
                }
                c = warp_sum(c);
            }
            __syncthreads();
            if (lane == 0 && s_cnt[wid] == 0) s_cnt[wid] = c;
        }
        __syncthreads();
        if (tid == 0) {
            for (int h = 0; h < HOM_BATCH; ++h) {
                if (s_iter >= s_niters) { s_done = 1; break; }
                if (!s_subok[h]) {             // getSubset failed: `if (iter == 0) return false; break;`
                    if (s_iter == 0) s_fail = 1;
                    s_done = 1;
                    break;
                }
                const int good = s_cnt[h];
                if (good > max(s_maxgood, 3)) {
                    for (int q = 0; q < 9; ++q) s_best[q] = s_H[h][q];
                    s_maxgood = good;
                    s_niters = ransac_update_num_iters(confidence, (double)(n - good) / n, 4, s_niters);
                }
                ++s_iter;
            }
            if (s_iter >= s_niters) s_done = 1;
        }
        __syncthreads();
        if (s_done) break;
    }
    HOM_STAMP(2);
    if (g_hom_dbg && tid == 0) { g_hom_dbg[8] = (unsigned long long)s_iter; g_hom_dbg[9] = (unsigned long long)n; }
    if (s_fail || s_maxgood == 0) { fail_out(); return; }
    // ---- inliers of the best model (ordered) ----
    __shared__ float s_bestf[8];
    if (tid < 8) s_bestf[tid] = (float)s_best[tid];
    if (tid == 0) s_ninl = 0;
    __syncthreads();
    for (int base = 0; base < n; base += blockDim.x) {
        const int i = base + tid;
        bool in = false;
        if (i < n) { const int p = good_idx[i]; in = homography_inlier(s_bestf, all_prev + 2 * p, all_cur + 2 * p, thr2); }
        const unsigned bal = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_warpcnt[wid] = __popc(bal);
        __syncthreads();
        int off = s_ninl;
        for (int w = 0; w < wid; ++w) off += s_warpcnt[w];
        off += __popc(bal & ((1u << lane) - 1));
        if (in) inl_idx[off] = good_idx[i];
        __syncthreads();
        if (tid == 0) {
            int t = 0;
            for (int w = 0; w < 8; ++w) t += s_warpcnt[w];
            s_ninl += t;
        }
        __syncthreads();
    }
    const int n_in = s_ninl;
    HOM_STAMP(3);
    // ---- runKernel on all inliers: normalised DLT (HomographyEstimatorCallback::runKernel) ----
    double acc[45];
    {
        double a4[4] = {0, 0, 0, 0};  // cm.x cm.y cM.x cM.y
        for (int i = tid; i < n_in; i += blockDim.x) {
            const int p = inl_idx[i];
            a4[0] += all_cur[2 * p]; a4[1] += all_cur[2 * p + 1]; a4[2] += all_prev[2 * p]; a4[3] += all_prev[2 * p + 1];
        }
        block_reduce<4>(a4, s_red, s_acc);
        if (tid < 4) s_nrm[tid] = s_acc[tid] / n_in;
        __syncthreads();
        for (int q = 0; q < 4; ++q) a4[q] = 0;
        for (int i = tid; i < n_in; i += blockDim.x) {
            const int p = inl_idx[i];
            a4[0] += fabs(all_cur[2 * p] - s_nrm[0]); a4[1] += fabs(all_cur[2 * p + 1] - s_nrm[1]);
            a4[2] += fabs(all_prev[2 * p] - s_nrm[2]); a4[3] += fabs(all_prev[2 * p + 1] - s_nrm[3]);
        }
        block_reduce<4>(a4, s_red, s_acc);
        if (tid < 4) s_nrm[4 + tid] = s_acc[tid];
        __syncthreads();
    }
    bool degenerate = false;
    for (int q = 0; q < 4; ++q) degenerate = degenerate || fabs(s_nrm[4 + q]) < DBL_EPSILON;
    if (!degenerate) {
        const double cm[2] = {s_nrm[0], s_nrm[1]}, cM[2] = {s_nrm[2], s_nrm[3]};
        const double sm[2] = {n_in / s_nrm[4], n_in / s_nrm[5]}, sM[2] = {n_in / s_nrm[6], n_in / s_nrm[7]};
        for (int q = 0; q < 45; ++q) acc[q] = 0.0;
        for (int i = tid; i < n_in; i += blockDim.x) {
            const int p = inl_idx[i];
            const double x = (all_cur[2 * p] - cm[0]) * sm[0], y = (all_cur[2 * p + 1] - cm[1]) * sm[1];
            const double X = (all_prev[2 * p] - cM[0]) * sM[0], Y = (all_prev[2 * p + 1] - cM[1]) * sM[1];
            const double Lx[9] = {X, Y, 1, 0, 0, 0, -x * X, -x * Y, -x};
            const double Ly[9] = {0, 0, 0, X, Y, 1, -y * X, -y * Y, -y};
            int q = 0;
#pragma unroll
            for (int a = 0; a < 9; ++a)
#pragma unroll
                for (int b = a; b < 9; ++b) acc[q++] += Lx[a] * Lx[b] + Ly[a] * Ly[b];
        }
        block_reduce<45>(acc, s_red, s_acc);
        if (tid == 0) {
            int q = 0;
            for (int a = 0; a < 9; ++a)
                for (int b = a; b < 9; ++b) { s_LtL[a * 9 + b] = s_acc[q]; s_LtL[b * 9 + a] = s_acc[q]; ++q; }
        }
        __syncthreads();
        HOM_STAMP(4);
        if (wid == 0) jacobi_smallest_eigvec9_warp(s_LtL, s_V, s_h9);
        __syncthreads();
        if (tid == 0) {
            double H[9];
            denormalise_h(s_h9, cm, sm, cM, sM, H);
            for (int i = 0; i < 8; ++i) s_x[i] = H[i];
        }
    } else if (tid == 0) {
        for (int i = 0; i < 8; ++i) s_x[i] = s_best[i];   // runKernel returned 0: H keeps the RANSAC model
    }
    __syncthreads();
    HOM_STAMP(5);
    // ---- LM refinement (HomographyRefineCallback, 10 iterations) ----
    {
        __shared__ float4 s_pairs[HOM_CACHE];
        const bool cached = n_in <= HOM_CACHE;
        if (cached) {
            for (int i = tid; i < n_in; i += blockDim.x) {
                const int p = inl_idx[i];
                s_pairs[i] = make_float4(all_prev[2 * p], all_prev[2 * p + 1], all_cur[2 * p], all_cur[2 * p + 1]);
            }
        }
        __syncthreads();
        HomographyProblem prob{all_prev, all_cur, inl_idx, n_in, cached ? s_pairs : nullptr};
        lm_refine(prob, s_x, 10, s_red, s_acc, s_work);
    }
    __syncthreads();
    HOM_STAMP(6);
    // ---- the mask findHomography returns: every match whose error under the refined model is within the threshold ----
    if (tid < 8) s_bestf[tid] = (float)s_x[tid];
    if (tid == 0) s_ninl = 0;
    __syncthreads();
    for (int base = 0; base < n; base += blockDim.x) {
        const int i = base + tid;
        bool in = false;
        if (i < n) { const int p = good_idx[i]; in = homography_inlier(s_bestf, all_prev + 2 * p, all_cur + 2 * p, thr2); }
        const unsigned bal = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_warpcnt[wid] = __popc(bal);
        __syncthreads();
        int off = s_ninl;
        for (int w = 0; w < wid; ++w) off += s_warpcnt[w];
        off += __popc(bal & ((1u << lane) - 1));
        if (in) inl_idx[off] = good_idx[i];
        __syncthreads();
        if (tid == 0) {
            int t = 0;
            for (int w = 0; w < 8; ++w) t += s_warpcnt[w];
            s_ninl += t;
        }
        __syncthreads();
    }
    const int n_fin = s_ninl;
    if (g_hom_dbg && tid == 0) g_hom_dbg[10] = (unsigned long long)n_in;
    if (tid == 0) {
        for (int i = 0; i < 8; ++i) H_out[i] = s_x[i];
        H_out[8] = 1.0;
        const bool ok = n_fin >= inlier_thresh;
        *h_ok = ok ? 1 : 0;
        *bg_kp_count = ok ? min(n_fin, max_bg) : 0;
    }
    for (int i = tid; i < min(n_fin, max_bg); i += blockDim.x) {
        const int p = inl_idx[i];
        bg_kp[2 * i] = all_cur[2 * p]; bg_kp[2 * i + 1] = all_cur[2 * p + 1];
        bg_kp_prev[2 * i] = all_prev[2 * p]; bg_kp_prev[2 * i + 1] = all_prev[2 * p + 1];
    }
}

}  // namespace

extern "C" int fm_klt_set_debug(void* dbg) {
    unsigned long long* p = (unsigned long long*)dbg;
    cudaMemcpyToSymbol(g_hom_dbg, &p, sizeof(p));
    return FM_OK;
}

extern "C" int fm_ransac_homography(const float* all_prev, const float* all_cur, const unsigned char* status,
                                    const int* meta, int max_iters, double confidence, double thresh,
                                    int inlier_thresh, int* good_idx, int* inl_idx, double* H_out, int* h_ok,
                                    float* bg_kp, float* bg_kp_prev, int* bg_kp_count, int max_bg, void* stream) {
    homography_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(all_prev, all_cur, status, meta, max_iters, confidence,
                                                           thresh, inlier_thresh, good_idx, inl_idx, H_out, h_ok, bg_kp,
                                                           bg_kp_prev, bg_kp_count, max_bg);
    FM_CHECK_LAUNCH("fm_ransac_homography");
    return FM_OK;
}

extern "C" int fm_ransac_affine_partial_batch(const float* all_prev, const float* all_cur, const unsigned char* status,
                                              const int* trk_begin, const int* slots, int n_trk, int n_rounds,
                                              int* round_flags, const int* h_ok, int* est_boxes,
                                              unsigned long long* sig, double* tlbr_pool, double* klt_tlbr,
                                              unsigned char* klt_ok, double* inlier_ratio, float* kp_pool,
                                              float* kp_prev_pool, int* kp_count, int max_kp, int frame_w, int frame_h,
                                              int max_iters, double confidence, double thresh, int inlier_thresh,
                                              int refine_iters, int first_round, void* stream) {
    if (n_trk <= 0) return FM_OK;
    FM_REQUIRE(max_kp <= AFF_MAX_PTS_LARGE, "fm_ransac_affine_partial_batch: max_kp above 4096");
    cudaStream_t s = (cudaStream_t)stream;
    auto kernel = max_kp <= AFF_MAX_PTS ? affine_partial_kernel<AFF_MAX_PTS> : affine_partial_kernel<AFF_MAX_PTS_LARGE>;
    for (int r = first_round; r < first_round + n_rounds; ++r) {
        const int* prev_flag = r > 0 ? round_flags + ((r - 1) & 15) : nullptr;
        int* cur_flag = round_flags + (r & 15);
        cudaMemsetAsync(cur_flag, 0, sizeof(int), s);
        const int* est_prev = est_boxes + ((r + 1) & 1) * n_trk * 5;
        int* est_cur = est_boxes + (r & 1) * n_trk * 5;
        if (r == 0) cudaMemsetAsync(est_boxes, 0, sizeof(int) * 2 * n_trk * 5, s);
        kernel<<<n_trk, 128, 0, s>>>(all_prev, all_cur, status, trk_begin, slots, n_trk, r, prev_flag, cur_flag, h_ok,
                                     est_prev, est_cur, sig, tlbr_pool, klt_tlbr, klt_ok, inlier_ratio, kp_pool,
                                     kp_prev_pool, kp_count, max_kp, frame_w, frame_h, max_iters, confidence, thresh,
                                     inlier_thresh, refine_iters);
    }
    FM_CHECK_LAUNCH("fm_ransac_affine_partial_batch");
    return FM_OK;
}
