// Association block: fused appearance+motion cost matrix, IoU cost, occlusion flags,
// rectangular linear sum assignment (bit-exact SciPy replay) and greedy matching.
//
// Reference call sites: fastmot/tracker.py:185-247, 314-366; fastmot/utils/distance.py:16-108;
// fastmot/utils/matching.py:10-116; fastmot/utils/rect.py:142-157; fastmot/kalman_filter.py:206-225.
#include "common.cuh"
#include "../../include/fastmot_b200.h"
#include <float.h>

int fm_launch_lsa_block(const double* cost, int nr, int nc, int* col4row, int* status, unsigned char* ws, int use_smem,
                        size_t smem_bytes, cudaStream_t s);   // assoc_lsa_block.cu

namespace {

// ----------------------------------------------------------------------------------------------------------
// matching cost: one CTA per track row, one warp per (row, detection) pair, lanes across the feature dim.
// ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) matching_cost_kernel(
    const float* __restrict__ feat_pool, const unsigned char* __restrict__ feat_valid_pool,
    const double* __restrict__ mean_pool, const double* __restrict__ cov_pool, const int* __restrict__ trk_slots,
    const long long* __restrict__ trk_labels, int n_trk, const float* __restrict__ det_emb,
    const double* __restrict__ det_tlbr, const long long* __restrict__ det_labels,
    const unsigned char* __restrict__ det_occluded, const int* __restrict__ det_sel, int n_det, int dim, int metric,
    double fill_val, double motion_weight, double max_cost, FmKalmanParams prm, double* __restrict__ cost) {
    extern __shared__ float s_feat[];  // dim floats
    __shared__ double s_L[16], s_pm[4], s_anorm;
    __shared__ int s_valid;
    const int i = blockIdx.x;
    const int slot = trk_slots[i];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const bool use_motion = motion_weight >= 0.0;
    if (tid == 0) s_valid = feat_valid_pool ? feat_valid_pool[slot] : 1;
    for (int k = tid; k < dim; k += blockDim.x) s_feat[k] = feat_pool[(size_t)slot * dim + k];
    if (tid == 32 && use_motion) {
        // project(mean, cov, DETECTOR) then Cholesky (kalman_filter.py:321-336, 347-353)
        const double* x = mean_pool + (size_t)slot * 8;
        const double* P = cov_pool + (size_t)slot * 64;
        double w = x[2] - x[0] + 1.0, h = x[3] - x[1] + 1.0;
        double S[16];
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) S[r * 4 + c] = P[r * 8 + c];
        for (int r = 0; r < 4; ++r) {
            double sd = fmax(prm.std_factor_det[r & 1] * ((r & 1) ? h : w), prm.min_std_det[r & 1]);
            S[r * 4 + r] += sd * sd;
            s_pm[r] = x[r];
        }
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) s_L[r * 4 + c] = 0.0;
        for (int c = 0; c < 4; ++c) {
            double d = S[c * 4 + c];
            for (int k = 0; k < c; ++k) d -= s_L[c * 4 + k] * s_L[c * 4 + k];
            d = sqrt(d);
            s_L[c * 4 + c] = d;
            for (int r = c + 1; r < 4; ++r) {
                double v = S[r * 4 + c];
                for (int k = 0; k < c; ++k) v -= s_L[r * 4 + k] * s_L[c * 4 + k];
                s_L[r * 4 + c] = v / d;
            }
        }
    }
    __syncthreads();
    if (wid == 0) {
        double a = 0.0;
        for (int k = lane; k < dim; k += 32) a += (double)s_feat[k] * (double)s_feat[k];
        a = warp_sum(a);
        if (lane == 0) s_anorm = sqrt(a);
    }
    __syncthreads();
    const long long tl = trk_labels ? trk_labels[i] : 0;
    for (int j = wid; j < n_det; j += (blockDim.x >> 5)) {
        const int dj = det_sel ? det_sel[j] : j;
        const float* e = det_emb + (size_t)dj * dim;
        double c;
        const bool empty = (!s_valid) || (det_occluded && det_occluded[dj]);
        if (empty) {
            c = fill_val;
        } else if (metric == FM_METRIC_COSINE) {
            double dot = 0.0, nb = 0.0;
            for (int k = lane; k < dim; k += 32) {
                double b = (double)e[k];
                dot += (double)s_feat[k] * b;
                nb += b * b;
            }
            dot = warp_sum(dot);
            nb = warp_sum(nb);
            c = 1.0 - dot / (s_anorm * sqrt(nb));
        } else {
            double d2 = 0.0;
            for (int k = lane; k < dim; k += 32) {
                double d = (double)s_feat[k] - (double)e[k];
                d2 += d * d;
            }
            c = sqrt(warp_sum(d2));
        }
        if (lane == 0) {
            if (use_motion) {
                const double* z = det_tlbr + (size_t)dj * 4;
                double y[4];
                for (int r = 0; r < 4; ++r) {
                    double v = z[r] - s_pm[r];
                    for (int k = 0; k < r; ++k) v -= s_L[r * 4 + k] * y[k];
                    y[r] = v / s_L[r * 4 + r];
                }
                double m = y[0] * y[0] + y[1] * y[1] + y[2] * y[2] + y[3] * y[3];
                c = (1.0 - motion_weight) * c + motion_weight * (1.0 / FM_CHI_SQ_INV_95) * m;
                if (m > FM_CHI_SQ_INV_95) c = FM_INF_COST;
            }
            // label gate only when both sides have labels, as in iou_cost_kernel
            if ((trk_labels && det_labels && tl != det_labels[dj]) || (max_cost >= 0.0 && c > max_cost))
                c = FM_INF_COST;
            cost[(size_t)i * n_det + j] = c;
        }
    }
}

__global__ void iou_cost_kernel(const double* __restrict__ pool, const int* __restrict__ trk_slots,
                                const long long* __restrict__ trk_labels, int n_trk,
                                const double* __restrict__ det_tlbr, const long long* __restrict__ det_labels,
                                const int* __restrict__ det_sel, int n_det, double max_cost,
                                double* __restrict__ cost) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_trk * n_det) return;
    int i = idx / n_det, j = idx - i * n_det;
    const double* a = pool + (size_t)(trk_slots ? trk_slots[i] : i) * 4;
    int dj = det_sel ? det_sel[j] : j;
    const double* b = det_tlbr + (size_t)dj * 4;
    double aw = a[2] - a[0] + 1.0, ah = a[3] - a[1] + 1.0;
    double bw = b[2] - b[0] + 1.0, bh = b[3] - b[1] + 1.0;
    double area1 = (aw <= 0 || ah <= 0) ? 0.0 : aw * ah;
    double area2 = (bw <= 0 || bh <= 0) ? 0.0 : bw * bh;
    double iw = fmin(a[2], b[2]) - fmax(a[0], b[0]) + 1.0;
    double ih = fmin(a[3], b[3]) - fmax(a[1], b[1]) + 1.0;
    double c = 1.0;
    if (iw > 0 && ih > 0) {
        double inter = iw * ih;
        c = 1.0 - inter / (area1 + area2 - inter);
    }
    if ((trk_labels && det_labels && trk_labels[i] != det_labels[dj]) || (max_cost >= 0.0 && c > max_cost))
        c = FM_INF_COST;
    cost[idx] = c;
}

__global__ void find_occluded_kernel(const double* __restrict__ tlbr, int n, double thresh,
                                     unsigned char* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* a = tlbr + (size_t)i * 4;
    double aw = a[2] - a[0] + 1.0, ah = a[3] - a[1] + 1.0;
    double area = (aw <= 0 || ah <= 0) ? 0.0 : aw * ah;
    unsigned char occ = 0;
    for (int j = 0; j < n; ++j) {
        if (j == i) continue;
        const double* b = tlbr + (size_t)j * 4;
        double iw = fmin(a[2], b[2]) - fmax(a[0], b[0]) + 1.0;
        double ih = fmin(a[3], b[3]) - fmax(a[1], b[1]) + 1.0;
        if (iw > 0 && ih > 0 && iw * ih / area >= thresh) { occ = 1; break; }
    }
    out[i] = occ;
}

// Solver state of lsa_block_kernel (the layout carve() in assoc_lsa_block.cu cuts), 16-byte rounded: it decides
// between shared memory and the caller's workspace.
inline size_t lsa_bytes(int nr, int nc) {
    size_t s = sizeof(double) * ((size_t)nr + 2 * (size_t)nc) + sizeof(int) * ((size_t)nr + 3 * (size_t)nc) +
               (size_t)nr + (size_t)nc;
    return (s + 15) & ~(size_t)15;
}

// ----------------------------------------------------------------------------------------------------------
// Greedy matching, one CTA.
// ----------------------------------------------------------------------------------------------------------
#define GREEDY_MAX 4096
__global__ void __launch_bounds__(1024) greedy_kernel(const double* __restrict__ cost, int nr, int nc,
                                                       double max_cost, int* __restrict__ col4row,
                                                       int* __restrict__ match_order) {
    __shared__ unsigned char rdead[GREEDY_MAX], cdead[GREEDY_MAX];
    __shared__ double s_val[32];
    __shared__ int s_idx[32];
    __shared__ int s_stop;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int k = tid; k < nr; k += blockDim.x) { rdead[k] = 0; col4row[k] = -1; match_order[k] = -1; }
    for (int k = tid; k < nc; k += blockDim.x) cdead[k] = 0;
    if (tid == 0) s_stop = 0;
    __syncthreads();
    const int total = nr * nc;
    const int max_iter = nr < nc ? nr : nc;
    for (int iter = 0; iter < max_iter; ++iter) {
        double best = INFINITY;
        int bidx = 0x7fffffff;
        for (int e = tid; e < total; e += blockDim.x) {
            int r = e / nc, c = e - r * nc;
            if (rdead[r] || cdead[c]) continue;
            double v = cost[e];
            if (v < best || (v == best && e < bidx)) { best = v; bidx = e; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            double ov = __shfl_xor_sync(0xffffffffu, best, o);
            int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
            if (ov < best || (ov == best && oi < bidx)) { best = ov; bidx = oi; }
        }
        if (lane == 0) { s_val[wid] = best; s_idx[wid] = bidx; }
        __syncthreads();
        if (wid == 0) {
            int nw = blockDim.x >> 5;
            best = lane < nw ? s_val[lane] : INFINITY;
            bidx = lane < nw ? s_idx[lane] : 0x7fffffff;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                double ov = __shfl_xor_sync(0xffffffffu, best, o);
                int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
                if (ov < best || (ov == best && oi < bidx)) { best = ov; bidx = oi; }
            }
            if (lane == 0) {
                if (bidx != 0x7fffffff && best <= max_cost) {
                    int r = bidx / nc, c = bidx - r * nc;
                    rdead[r] = 1; cdead[c] = 1;
                    col4row[r] = c; match_order[r] = iter;
                } else {
                    s_stop = 1;
                }
            }
        }
        __syncthreads();
        if (s_stop) break;
    }
}

__global__ void __launch_bounds__(128) feature_update_kernel(float* __restrict__ sum_pool, float* __restrict__ avg_pool,
                                                              float* __restrict__ last_pool,
                                                              unsigned char* __restrict__ valid_pool,
                                                              const int* __restrict__ slots, const float* __restrict__ vec,
                                                              const int* __restrict__ vec_idx,
                                                              const int* __restrict__ counts, int n, int dim) {
    __shared__ double s_part[4];
    const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int slot = slots[i];
    const float* v = vec + (size_t)(vec_idx ? vec_idx[i] : i) * dim;
    float* sum = sum_pool + (size_t)slot * dim;
    float* avg = avg_pool + (size_t)slot * dim;
    const int cnt = counts[i];
    if (last_pool)
        for (int k = tid; k < dim; k += blockDim.x) last_pool[(size_t)slot * dim + k] = v[k];
    if (cnt <= 1) {
        for (int k = tid; k < dim; k += blockDim.x) { float x = v[k]; sum[k] = x; avg[k] = x; }
    } else {
        const double div = 1.0 / (double)cnt;
        double part = 0.0;
        for (int k = tid; k < dim; k += blockDim.x) {
            float s = sum[k] + v[k];
            sum[k] = s;
            float a = (float)((double)s * div);
            avg[k] = a;
            part += (double)a * (double)a;
        }
        part = warp_sum(part);
        if (lane == 0) s_part[wid] = part;
        __syncthreads();
        float nrm = (float)sqrt(s_part[0] + s_part[1] + s_part[2] + s_part[3]);
        const double inv = 1.0 / (double)nrm;
        for (int k = tid; k < dim; k += blockDim.x) avg[k] = (float)((double)avg[k] * inv);
    }
    if (tid == 0) valid_pool[slot] = 1;
}

}  // namespace

extern "C" int fm_feature_update(float* sum_pool, float* avg_pool, float* last_pool, unsigned char* valid_pool,
                                 const int* slots,
                                 const float* vec, const int* vec_idx, const int* counts, int n, int dim,
                                 void* stream) {
    if (n <= 0) return FM_OK;
    feature_update_kernel<<<n, 128, 0, (cudaStream_t)stream>>>(sum_pool, avg_pool, last_pool, valid_pool, slots, vec,
                                                               vec_idx, counts, n, dim);
    FM_CHECK_LAUNCH("fm_feature_update");
    return FM_OK;
}

extern "C" int fm_matching_cost(const float* feat_pool, const unsigned char* feat_valid_pool, const double* mean_pool,
                                const double* cov_pool, const int* trk_slots, const long long* trk_labels, int n_trk,
                                const float* det_emb, const double* det_tlbr, const long long* det_labels,
                                const unsigned char* det_occluded, const int* det_sel, int n_det, int dim, int metric,
                                double fill_val, double motion_weight, double max_cost, const FmKalmanParams* params,
                                double* cost, void* stream) {
    FM_REQUIRE(params != nullptr, "fm_matching_cost: params is NULL");
    FM_REQUIRE(dim > 0 && dim <= 8192, "fm_matching_cost: dim out of range");
    if (n_trk <= 0 || n_det <= 0) return FM_OK;
    matching_cost_kernel<<<n_trk, 256, dim * sizeof(float), (cudaStream_t)stream>>>(
        feat_pool, feat_valid_pool, mean_pool, cov_pool, trk_slots, trk_labels, n_trk, det_emb, det_tlbr, det_labels,
        det_occluded, det_sel, n_det, dim, metric, fill_val, motion_weight, max_cost, *params, cost);
    FM_CHECK_LAUNCH("fm_matching_cost");
    return FM_OK;
}

extern "C" int fm_iou_cost(const double* trk_tlbr_pool, const int* trk_slots, const long long* trk_labels, int n_trk,
                           const double* det_tlbr, const long long* det_labels, const int* det_sel, int n_det,
                           double max_cost, double* cost, void* stream) {
    if (n_trk <= 0 || n_det <= 0) return FM_OK;
    int total = n_trk * n_det;
    iou_cost_kernel<<<fm_cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(
        trk_tlbr_pool, trk_slots, trk_labels, n_trk, det_tlbr, det_labels, det_sel, n_det, max_cost, cost);
    FM_CHECK_LAUNCH("fm_iou_cost");
    return FM_OK;
}

extern "C" int fm_find_occluded(const double* tlbr, int n, double thresh, unsigned char* out, void* stream) {
    if (n <= 0) return FM_OK;
    find_occluded_kernel<<<fm_cdiv(n, 128), 128, 0, (cudaStream_t)stream>>>(tlbr, n, thresh, out);
    FM_CHECK_LAUNCH("fm_find_occluded");
    return FM_OK;
}

extern "C" long long fm_lsa_workspace_bytes(int nr, int nc) {
    int a = nr < nc ? nr : nc, b = nr < nc ? nc : nr;
    return (long long)lsa_bytes(a, b);
}

extern "C" int fm_lsa(const double* cost, int nr, int nc, int* col4row, int* status, void* workspace, void* stream) {
    FM_REQUIRE(nr >= 0 && nc >= 0, "fm_lsa: negative shape");
    if (nr == 0) return FM_OK;
    if (nc == 0) {
        // SciPy returns empty assignment; every row is unassigned.
        cudaMemsetAsync(col4row, 0xff, sizeof(int) * nr, (cudaStream_t)stream);
        cudaMemsetAsync(status, 0, sizeof(int), (cudaStream_t)stream);
        return FM_OK;
    }
    int a = nr < nc ? nr : nc, b = nr < nc ? nc : nr;
    size_t bytes = lsa_bytes(a, b);
    int use_smem = bytes <= 46 * 1024;
    FM_REQUIRE(use_smem || workspace, "fm_lsa: workspace required for this size");
    fm_launch_lsa_block(cost, nr, nc, col4row, status, (unsigned char*)workspace, use_smem, bytes,
                        (cudaStream_t)stream);
    FM_CHECK_LAUNCH("fm_lsa");
    return FM_OK;
}

extern "C" int fm_greedy_match(const double* cost, int nr, int nc, double max_cost, int* col4row, int* match_order,
                               void* stream) {
    FM_REQUIRE(nr <= GREEDY_MAX && nc <= GREEDY_MAX, "fm_greedy_match: shape exceeds 4096");
    if (nr <= 0) return FM_OK;
    if (nc <= 0) {
        cudaMemsetAsync(col4row, 0xff, sizeof(int) * nr, (cudaStream_t)stream);
        cudaMemsetAsync(match_order, 0xff, sizeof(int) * nr, (cudaStream_t)stream);
        return FM_OK;
    }
    greedy_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(cost, nr, nc, max_cost, col4row, match_order);
    FM_CHECK_LAUNCH("fm_greedy_match");
    return FM_OK;
}
