// Blocked greedy NMS scan (one CTA) + final detection filters with ordered, parallel output compaction.
// Replaces the serial candidate-by-candidate loop: 64 candidates per step are resolved by warp 0 from the diagonal
// mask words, then all 32 warps OR the mask rows of the survivors into the tail of the removed-bitmap (one
// independent coalesced row load per warp task, shared-memory atomicOr).  Semantics identical to
// fastmot/utils/rect.py:198-244 + fastmot/detector.py:357-365.
#include "common.cuh"
#include "../../include/fastmot_b200.h"

namespace {

constexpr int NMS_THREADS = 1024;

struct NmsOut {
    bool ok;
    double x1, y1, x2, y2, conf;
    long long label;
};

__device__ __forceinline__ NmsOut nms_final_filter(const unsigned long long* __restrict__ keys,
                                                   const float* __restrict__ dense, int i, double max_area,
                                                   double min_ar) {
    NmsOut o;
    const float* d = dense + (size_t)(keys[i] & 0xffffff) * 8;
    o.x1 = rint((double)d[0]); o.y1 = rint((double)d[1]);
    // to_tlbr under Numba: x + w is an f32 add, the `- 1.` literal promotes to f64 (oracle/detect.py)
    o.x2 = rint((double)(d[0] + d[2]) - 1.0); o.y2 = rint((double)(d[1] + d[3]) - 1.0);
    const double w = o.x2 - o.x1 + 1.0, h = o.y2 - o.y1 + 1.0;
    const double area = (w <= 0 || h <= 0) ? 0.0 : w * h;
    const double ar = w > 0 ? h / w : 0.0;
    o.ok = area > 0 && area <= max_area && ar >= min_ar;
    o.label = (long long)d[5];
    o.conf = (double)__fmul_rn(d[4], d[6]);
    return o;
}

// one CTA per image (blockIdx.x): the image's segments of keys, dense rows, mask and outputs (detect.cu)
__global__ void __launch_bounds__(NMS_THREADS) nms_scan_blocked_kernel(const unsigned long long* __restrict__ keys,
                                                                        const float* __restrict__ dense, int cand_stride,
                                                                        const int* __restrict__ counter, int key_cap,
                                                                        const unsigned long long* __restrict__ mask,
                                                                        int mask_words, double max_area, double min_ar,
                                                                        int max_out, double* __restrict__ out_tlbr,
                                                                        long long* __restrict__ out_label,
                                                                        double* __restrict__ out_conf,
                                                                        int* __restrict__ out_count, int* __restrict__ status) {
    extern __shared__ unsigned long long sm[];   // removed[nw] | keep[nw] | okbits (u32 x 2nw) | prefix (i32 x 2nw)
    __shared__ unsigned long long s_kept;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int img = blockIdx.x;
    keys += (size_t)img * key_cap;
    dense += (size_t)img * cand_stride * 8;
    counter += img;
    mask += (size_t)img * key_cap * mask_words;
    out_tlbr += (size_t)img * max_out * 4;
    out_label += (size_t)img * max_out;
    out_conf += (size_t)img * max_out;
    out_count += img;
    status += img;
    const int n = min(*counter, key_cap);
    const int nw = (n + 63) >> 6;
    unsigned long long* removed = sm;
    unsigned long long* keep = sm + nw;
    unsigned* okbits = reinterpret_cast<unsigned*>(sm + 2 * nw);
    int* prefix = reinterpret_cast<int*>(okbits + 2 * nw);
    for (int w = tid; w < nw; w += NMS_THREADS) { removed[w] = 0; keep[w] = 0; }
    __syncthreads();
    for (int blk = 0; blk < nw; ++blk) {
        const int base = blk << 6;
        if (warp == 0) {
            // diagonal words of the 64 rows of this block (bit b of row r set => r suppresses base+b, b > r)
            const int r0 = base + lane, r1 = base + 32 + lane;
            const unsigned long long d0 = r0 < n ? mask[(size_t)r0 * mask_words + blk] : 0ull;
            const unsigned long long d1 = r1 < n ? mask[(size_t)r1 * mask_words + blk] : 0ull;
            unsigned long long rem = removed[blk];
            unsigned long long kept = 0;
            const int lim = min(64, n - base);
            for (int b = 0; b < lim; ++b) {
                const unsigned long long row = __shfl_sync(0xffffffffu, b < 32 ? d0 : d1, b & 31);
                if (!((rem >> b) & 1ull)) { kept |= 1ull << b; rem |= row; }
            }
            if (lane == 0) { keep[blk] = kept; s_kept = kept; }
        }
        __syncthreads();
        // survivors of this block suppress later blocks: task = (survivor, chunk of 32 consecutive words)
        const unsigned long long kept = s_kept;
        const unsigned lo = (unsigned)kept, hi = (unsigned)(kept >> 32);
        const int nlo = __popc(lo), nk = nlo + __popc(hi);
        const int tail = nw - (blk + 1);
        const int nchunks = (tail + 31) >> 5;
        const int ntasks = nk * nchunks;
        for (int task = warp; task < ntasks; task += NMS_THREADS / 32) {
            const int r = task / nchunks, c = task - r * nchunks;
            const int bit = r < nlo ? (int)__fns(lo, 0, r + 1) : 32 + (int)__fns(hi, 0, r - nlo + 1);
            const int w = blk + 1 + (c << 5) + lane;
            if (w < nw) {
                const unsigned long long v = mask[(size_t)(base + bit) * mask_words + w];
                if (v) atomicOr(&removed[w], v);
            }
        }
        __syncthreads();
    }
    // final filters + ordered compaction (detector.py:357-365): flag pass, block prefix over 32-candidate words,
    // then the ordered scatter
    const int nw32 = (n + 31) >> 5;
    for (int i0 = warp << 5; i0 < n; i0 += NMS_THREADS) {
        const int i = i0 + lane;
        bool ok = false;
        if (i < n && ((keep[i >> 6] >> (i & 63)) & 1ull)) ok = nms_final_filter(keys, dense, i, max_area, min_ar).ok;
        const unsigned bal = __ballot_sync(0xffffffffu, ok);
        if (lane == 0) okbits[i0 >> 5] = bal;
    }
    __syncthreads();
    if (warp == 0) {                 // exclusive prefix of popcounts, 32 words per round
        int run = 0;
        for (int w0 = 0; w0 < nw32; w0 += 32) {
            const int w = w0 + lane;
            const int cnt = w < nw32 ? __popc(okbits[w]) : 0;
            int inc = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            if (w < nw32) prefix[w] = run + inc - cnt;
            run += __shfl_sync(0xffffffffu, inc, 31);
        }
        if (lane == 0) {
            *out_count = min(run, max_out);
            if (run > max_out && status[0] == 0) status[0] = 2;   // more survivors than max_out rows: host raises (no silent drop)
        }
    }
    __syncthreads();
    for (int i0 = warp << 5; i0 < n; i0 += NMS_THREADS) {
        const int i = i0 + lane;
        const unsigned bal = okbits[i0 >> 5];
        if (i < n && ((bal >> lane) & 1u)) {
            const int pos = prefix[i0 >> 5] + __popc(bal & ((1u << lane) - 1));
            if (pos < max_out) {
                const NmsOut o = nms_final_filter(keys, dense, i, max_area, min_ar);
                out_tlbr[pos * 4 + 0] = o.x1; out_tlbr[pos * 4 + 1] = o.y1;
                out_tlbr[pos * 4 + 2] = o.x2; out_tlbr[pos * 4 + 3] = o.y2;
                out_label[pos] = o.label;
                out_conf[pos] = o.conf;
            }
        }
    }
}

}  // namespace

int fm_launch_nms_scan(int batch, const unsigned long long* keys, const float* dense, int cand_stride,
                       const int* counter, int key_cap, const unsigned long long* mask, int words, double max_area,
                       double min_ar, int max_out, double* out_tlbr, long long* out_label, double* out_conf,
                       int* out_count, int* status, cudaStream_t s) {
    nms_scan_blocked_kernel<<<batch, NMS_THREADS, (size_t)(4 * words + 4) * 8, s>>>(keys, dense, cand_stride, counter,
                                                                     key_cap, mask, words,
                                                                     max_area, min_ar, max_out, out_tlbr, out_label,
                                                                     out_conf, out_count, status);
    return 0;
}
