// Warp-specialised, TMA-fed wgmma convolution for sm_90a with the split-K reduction done inside a thread-block
// cluster (distributed shared memory) -- the batch-1 detector layers of the YOLO stack (role of the TensorRT conv
// tactics behind fastmot/utils/inference.py:106-117; layer semantics of scripts/yolo2onnx.py:558-700).
//
//   D[128 output pixels, BN filters] = sum over K slices of  A_slice[128 x 64] * W_slice[BN x 64]^T
//
// Supported layers: 1x1 (stride 1) and 3x3 (stride 1 or 2), "same" padding, cin % 64 == 0, 8-channel aligned input
// views (everything else stays on conv_tc.cu).  A K slice is (filter tap, 64 input channels).
//   * A operand: one TMA box per slice.  The 128 tile rows are a TW x TH rectangle of output pixels; for tap (r, s)
//     the box is the same rectangle shifted by (r - pad, s - pad) in a [C, W, H] tensor map, so the zero padding is the
//     TMA out-of-bounds fill and no thread ever computes an im2col address.  1x1 layers use the flattened
//     [C, N*H*W, 1] view (128 consecutive pixels).  Stride-2 layers read a 5-D parity view of the input,
//     [C, w & 1, w / 2, h & 1, h / 2]: tap (r, s) of output (y, x) is element (parity, index) = ((s + 1) & 1,
//     x + (s - 1 >> 1)) of that view, again one rectangular box per slice.
//   * B operand: one TMA box [64 x BN] of the K-major weight matrix [cout][kh*kw*cin].
//   * both land 128-byte swizzled in an NS-stage mbarrier ring filled by one producer warp; two consumer warpgroups
//     (64 tile rows each) issue four wgmma (64 x BN x 16) per slice, accumulators in registers.  Weight boxes of the
//     first stages are requested before griddepcontrol.wait (they do not depend on the previous layer) and the CTA's
//     remaining weight boxes are prefetched into L2 at the same point, so the previous layer's tail hides the HBM
//     latency of this layer's weights.
//   * split K: gridDim.z = S CTAs of one cluster share an output tile, each owns nk / S slices.  Tile row r is finished
//     by cluster rank r % S: every CTA pushes its fp32 partial of that row into a slot of the owner's shared memory
//     (st.shared::cluster, asynchronous); after one cluster barrier the owner sums its S slots from local memory and
//     finishes the row (bias, activation, residual, fp16 NHWC store, lanes along the channels).  No fp32 workspace in
//     HBM, no second kernel, no remote load on the critical path.
//   * S == 1: the tile goes registers -> fp16 staging -> coalesced rows like conv_tc.cu.
#include "tc_common.cuh"
#include "conv_act.cuh"
#include <stdlib.h>
#include <string.h>

namespace {

using namespace tc;

struct ConvTmaArgs {
    int W, H, TW, TH, tiles_w;      // output plane, tile rectangle, tiles per plane row
    int kc, kw, pad, s2;            // cin / 64, filter width, padding, stride-2 flag (5-D parity view of the input)
    int vec_ok;                     // output / residual views are 8-channel aligned (16-byte stores)
    int nk, sps;                    // K slices in total / per cluster rank
    int cout, cout_stride, cout_offset, res_stride, res_offset, act;
    const float* bias;
    const __half* residual;
    __half* out;
};

// optional timeline stamps (scripts/yolo_phases.py): CTA (0,0,0) of every launch records %globaltimer at entry, after
// griddepcontrol.wait, when its accumulator is complete, and at exit, in launch order
__device__ unsigned long long* g_tma_dbg = nullptr;
__device__ unsigned int g_tma_dbg_n = 0;
__device__ __forceinline__ unsigned long long gtimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ void cl_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
// no memory ordering (compiles without the MEMBAR.ALL.GPU of the release form): only "every peer got here"
__device__ __forceinline__ void cl_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cl_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t cl_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void st_cluster_v2(uint32_t local_saddr, uint32_t rank, float x, float y) {
    uint32_t raddr;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(local_saddr), "r"(rank));
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(raddr), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void bar_sync_epi() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Code size matters here: every CTA runs its epilogue exactly once, so the epilogue executes out of a cold instruction
// cache.  A first version (rows unrolled four-fold, one activation switch per unrolled row and per residual order, one
// instantiation per ring depth: ~10 000 SASS instructions = 160 KB per kernel) spent microseconds per CTA in the row loop;
// this one keeps a single rolled row loop with one activation site and takes the ring depth at run time.
struct RowOut {
    size_t pix;
    bool ok;
};

__device__ __forceinline__ RowOut row_out(const ConvTmaArgs& a, int rr, int rows_used, int w0, int h0, float inv_tw) {
    const int hl = (int)(((float)rr + 0.5f) * inv_tw);       // rr / TW (rr < 128: the half keeps it exact)
    const int wl = rr - hl * a.TW;
    const int h = h0 + hl, w = w0 + wl;
    RowOut r;
    r.ok = rr < rows_used && h < a.H && w < a.W;
    r.pix = (size_t)h * a.W + w;
    return r;
}

// two consumer warpgroups (warps 0-7, tile rows 64 g ..) and one producer warp (TMA)
constexpr int kEpiWarps = 8, kEpiThreads = kEpiWarps * 32, kThreads = kEpiThreads + 32;
constexpr int kMaxStages = 8;

template <int BN>
__global__ void __launch_bounds__(kThreads, 1) conv_tma_kernel(const __grid_constant__ CUtensorMap map_a,
                                                             const __grid_constant__ CUtensorMap map_b, ConvTmaArgs a,
                                                             int NS) {
    constexpr int A_BYTES = 16384, B_BYTES = BN * 128, STAGE = A_BYTES + B_BYTES;
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ uint64_t full[kMaxStages], empty[kMaxStages];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    fm_pdl_trigger();
    unsigned long long* dbg = nullptr;
    if (g_tma_dbg && tid == 0 && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
        const unsigned int slot = atomicAdd(&g_tma_dbg_n, 1u);
        if (slot < 512) {
            dbg = g_tma_dbg + (size_t)slot * 8;
            dbg[0] = gtimer_ns();
            dbg[4] = ((unsigned long long)gridDim.x << 40) | ((unsigned long long)gridDim.y << 24) |
                     ((unsigned long long)gridDim.z << 16) | (unsigned long long)a.nk;
            dbg[5] = ((unsigned long long)BN << 32) | (unsigned long long)NS;
        }
    }
    const int S = (int)gridDim.z;
    const int z = S > 1 ? (int)cl_rank() : 0;
    const int th = (int)blockIdx.x / a.tiles_w, tw = (int)blockIdx.x - th * a.tiles_w;
    const int w0 = tw * a.TW, h0 = th * a.TH;
    const int n0 = (int)blockIdx.y * BN;
    const int rows_used = a.TW * a.TH;
    const int k0 = z * a.sps;
    // only the last rank can own fewer than sps slices.  A select, not min(): ptxas 12.9 fuses min(NS, min(..)) below
    // into a three-input VIMNMX3, which computes wrong results on sm_90 (see fast_score_kernel in klt_feat.cu)
    const int iters = z == S - 1 ? a.nk - k0 : a.sps;

    if (tid == 0) {
        if (smem_u32(smem) & 1023u) __trap();
        for (int i = 0; i < NS; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kEpiWarps); }
        mbar_fence_init();
    }
    if (warp == kEpiWarps && lane == 0) { tma_prefetch_desc(&map_a); tma_prefetch_desc(&map_b); }
    __syncthreads();
    // cluster phase 0: "this CTA is running" (waited for before the first remote store into a peer's shared memory)
    if (S > 1) cl_arrive_relaxed();

    // epilogue geometry: a thread finishes 8 channels (chunk ch) of rows r0, r0 + RPP, ...
    constexpr int CPR = BN / 8;                       // 16-byte output chunks per row
    constexpr int RPP = kEpiThreads / CPR;            // rows per pass
    constexpr int PITCH16 = BN * 2 + 16, PITCH32 = BN * 4 + 16;
    const int ch = tid % CPR, r0 = tid / CPR;
    const int n = n0 + ch * 8;
    const int rmax = (128 + S - 1) / S;               // rows a cluster rank finishes (slot pitch of the fp32 partials)
    // fp32 partial rows pushed by the cluster peers land BEHIND the ring: a peer that finishes its K range early writes
    // here while this CTA's TMA / wgmma pipeline is still using the ring
    uint8_t* slots = smem + (size_t)NS * STAGE;
    const int nrows = S == 1 ? 128 : (128 - z + S - 1) / S;
    const float inv_tw = 1.0f / (float)a.TW;
    const bool vec = a.vec_ok != 0;
    const bool has_res = a.residual != nullptr && vec;
    float b8[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) b8[e] = 0.f;
    RowOut ro_next;
    ro_next.ok = false; ro_next.pix = 0;
    uint4 rv_next = make_uint4(0u, 0u, 0u, 0u);

    if (warp == kEpiWarps) {
        // ------------------------------------------- producer warp -------------------------------------------
        if (lane == 0) {
            const uint32_t tx = (uint32_t)rows_used * 128u + (uint32_t)B_BYTES;
            // slice i lives in ring stage i % NS
            auto load_b = [&](int i, int st) {
                mbar_expect_tx(&full[st], tx);
                tma_load_3d(smem + (size_t)st * STAGE + A_BYTES, &map_b, &full[st], (k0 + i) * 64, n0, 0);
            };
            auto load_a = [&](int i, int st) {
                const int g = k0 + i;
                const int tap = g / a.kc, c = g - tap * a.kc;
                const int fr = tap / a.kw, fs = tap - fr * a.kw;
                if (a.s2)
                    tma_load_5d(smem + (size_t)st * STAGE, &map_a, &full[st], c * 64, (fs + 1) & 1, w0 + ((fs - 1) >> 1),
                                (fr + 1) & 1, h0 + ((fr - 1) >> 1));
                else
                    tma_load_3d(smem + (size_t)st * STAGE, &map_a, &full[st], c * 64, w0 + fs - a.pad, h0 + fr - a.pad);
            };
            const int pre = min(NS, iters);
            for (int i = 0; i < pre; ++i) load_b(i, i);        // weights: independent of the previous layer
            for (int i = pre; i < iters; ++i) tma_prefetch_l2_3d(&map_b, (k0 + i) * 64, n0, 0);
            fm_pdl_wait();
            for (int i = 0; i < pre; ++i) load_a(i, i);
#pragma unroll 1
            for (int i = pre; i < iters; ++i) {
                const int st = i % NS;
                mbar_wait(&empty[st], (uint32_t)((i / NS - 1) & 1));     // the wgmma of slice i - NS retired
                load_b(i, st);
                load_a(i, st);
            }
        } else {
            fm_pdl_wait();
        }
        __syncwarp();
        if (S > 1) cl_wait();
    } else {
        // ------------------------------------------- consumer warpgroups -------------------------------------
        // Everything that does not need the accumulator is fetched while the main loop runs: the bias of this thread's
        // 8 channels (a constant: even before griddepcontrol.wait) and the residual of its first row.
        if (vec && a.bias && n < a.cout) {
            const float4 ba = __ldg(reinterpret_cast<const float4*>(a.bias + n));
            const float4 bb = __ldg(reinterpret_cast<const float4*>(a.bias + n + 4));
            b8[0] = ba.x; b8[1] = ba.y; b8[2] = ba.z; b8[3] = ba.w;
            b8[4] = bb.x; b8[5] = bb.y; b8[6] = bb.z; b8[7] = bb.w;
        }
        fm_pdl_wait();
        if (dbg) dbg[1] = gtimer_ns();
        if (r0 < nrows) {
            ro_next = row_out(a, S == 1 ? r0 : z + r0 * S, rows_used, w0, h0, inv_tw);
            if (ro_next.ok && has_res && n < a.cout)
                rv_next = *reinterpret_cast<const uint4*>(a.residual + ro_next.pix * a.res_stride + a.res_offset + n);
        }
        const int g = warp >> 2, wq = warp & 3;
        float acc[BN / 2];
#pragma unroll
        for (int e = 0; e < BN / 2; ++e) acc[e] = 0.f;
#pragma unroll 1
        for (int i = 0; i < iters; ++i) {
            const int st = i % NS;
            mbar_wait(&full[st], (uint32_t)((i / NS) & 1));
            const uint32_t sa = smem_u32(smem + (size_t)st * STAGE) + g * 64 * 128, sb = smem_u32(smem + (size_t)st * STAGE) + A_BYTES;
            wg_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) mma_m64<BN>(acc, smem_desc_sw128(sa + k * 32), smem_desc_sw128(sb + k * 32), 1);
            wg_commit();
            wg_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
        }
        if (dbg) dbg[2] = gtimer_ns();
        if (S == 1) {
            bar_sync_epi();                               // both warpgroups are done with the ring: it becomes staging
#pragma unroll
            for (int i = 0; i < BN / 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int row = g * 64 + wq * 16 + (lane >> 2) + e * 8, col = i * 8 + (lane & 3) * 2;
                    *reinterpret_cast<uint32_t*>(smem + row * PITCH16 + col * 2) = pack_h2(acc[i * 4 + e * 2], acc[i * 4 + e * 2 + 1]);
                }
        } else {
            // push: tile row `row` is finished by cluster rank row % S; this CTA's fp32 partial of it goes straight
            // into slot [z][row / S] of THAT CTA's shared memory (asynchronous remote stores: no round trip)
            cl_wait();                                    // phase 0: every peer has started
#pragma unroll
            for (int i = 0; i < BN / 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int row = g * 64 + wq * 16 + (lane >> 2) + e * 8, col = i * 8 + (lane & 3) * 2;
                    const uint32_t dst = smem_u32(slots) + (uint32_t)((z * rmax + row / S) * PITCH32 + col * 4);
                    st_cluster_v2(dst, (uint32_t)(row % S), acc[i * 4 + e * 2], acc[i * 4 + e * 2 + 1]);
                }
        }
        if (S == 1) bar_sync_epi();
    }
    if (S > 1) {            // every thread of every CTA of the cluster: all partial rows have been pushed to their owners
        cl_arrive();
        cl_wait();
    }
    if (dbg) dbg[6] = gtimer_ns();
    if (warp < kEpiWarps && n < a.cout) {
        // finish rows: S == 1 all 128 rows of the own fp16 tile; S > 1 rows z, z + S, ... summed over the S fp32 slots.
        // A thread keeps its 8 channels for every row; ONE rolled loop, ONE activation site; the next row's residual is
        // requested before the current row is finished.
        const int act = a.act & 0xff;
        const bool res_first = (a.act & FM_ACT_AFTER_RESIDUAL) != 0;
#pragma unroll 1
        for (int ri = r0; ri < nrows; ri += RPP) {
            const RowOut ro = ro_next;
            const uint4 rv = rv_next;
            const int rr = S == 1 ? ri : z + ri * S;
            if (ri + RPP < nrows) {
                ro_next = row_out(a, S == 1 ? ri + RPP : z + (ri + RPP) * S, rows_used, w0, h0, inv_tw);
                rv_next = make_uint4(0u, 0u, 0u, 0u);
                if (ro_next.ok && has_res)
                    rv_next = *reinterpret_cast<const uint4*>(a.residual + ro_next.pix * a.res_stride + a.res_offset + n);
            }
            if (!ro.ok) continue;
            float x[8];
            if (S == 1) {
                const uint4 pk = *reinterpret_cast<const uint4*>(smem + rr * PITCH16 + ch * 16);
                const __half2* ph = reinterpret_cast<const __half2*>(&pk);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(ph[e]);
                    x[2 * e] = f.x;
                    x[2 * e + 1] = f.y;
                }
            } else {
                const uint8_t* src = slots + ri * PITCH32 + ch * 32;
#pragma unroll
                for (int e = 0; e < 8; ++e) x[e] = 0.f;
#pragma unroll 1
                for (int pz = 0; pz < S; ++pz) {
                    const float4 v0 = *reinterpret_cast<const float4*>(src + (size_t)pz * rmax * PITCH32);
                    const float4 v1 = *reinterpret_cast<const float4*>(src + (size_t)pz * rmax * PITCH32 + 16);
                    x[0] += v0.x; x[1] += v0.y; x[2] += v0.z; x[3] += v0.w;
                    x[4] += v1.x; x[5] += v1.y; x[6] += v1.z; x[7] += v1.w;
                }
            }
            if (vec) {
                // out = act(x + b [+ res if res_first]) [+ res otherwise]
                float rf[8];
                const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(rh[e]);
                    rf[2 * e] = f.x;
                    rf[2 * e + 1] = f.y;
                }
#pragma unroll
                for (int e = 0; e < 8; ++e) x[e] += b8[e] + (res_first ? rf[e] : 0.f);
                tc_act8(x, act);
#pragma unroll
                for (int e = 0; e < 8; ++e) x[e] += res_first ? 0.f : rf[e];
                *reinterpret_cast<uint4*>(a.out + ro.pix * a.cout_stride + a.cout_offset + n) =
                    make_uint4(pack_h2(x[0], x[1]), pack_h2(x[2], x[3]), pack_h2(x[4], x[5]), pack_h2(x[6], x[7]));
            } else {
                // ragged views (detection heads: 18 channels, 36-byte pixel pitch): element-wise
#pragma unroll 1
                for (int e = 0; e < 8; ++e) {
                    if (n + e >= a.cout) break;
                    float xe = 0.f;
#pragma unroll
                    for (int k = 0; k < 8; ++k) xe = k == e ? x[k] : xe;      // register select, no local memory
                    const float res = a.residual ? __half2float(a.residual[ro.pix * a.res_stride + a.res_offset + n + e]) : 0.f;
                    float v = xe + (a.bias ? __ldg(a.bias + n + e) : 0.f) + (res_first ? res : 0.f);
                    v = tc_act(v, act) + (res_first ? 0.f : res);
                    a.out[ro.pix * a.cout_stride + a.cout_offset + n + e] = __float2half(v);
                }
            }
        }
    }
    if (dbg) dbg[7] = gtimer_ns();
    if (S > 1) {            // nobody leaves while a peer may still read its tile (its loads have returned: their
        cl_arrive_relaxed();    // values fed the stores above), nothing to publish
        cl_wait();
    }
    if (dbg) dbg[3] = gtimer_ns();
}

struct Plan {
    int W, H, TW, TH, tiles_w, tiles;
};

Plan plan_tiles(const FmConvDesc* d) {
    Plan p;
    if (d->kh == 1) {
        p.W = d->n * d->ho * d->wo; p.H = 1; p.TW = 128; p.TH = 1;
        p.tiles_w = fm_cdiv(p.W, 128); p.tiles = p.tiles_w;
        return p;
    }
    p.W = d->wo; p.H = d->ho;
    int best = 1 << 30, btw = 8;
    for (int tw = 4; tw <= 128 && tw <= p.W; ++tw) {
        const int th = 128 / tw;
        if (th < 1) break;
        const int t = fm_cdiv(p.W, tw) * fm_cdiv(p.H, th);
        // fewer tiles first; then the wider rectangle (longer contiguous runs for the TMA box and the stores)
        if (t < best || (t == best && tw > btw)) { best = t; btw = tw; }
    }
    p.TW = btw; p.TH = 128 / btw;
    p.tiles_w = fm_cdiv(p.W, p.TW);
    p.tiles = best;
    return p;
}

constexpr int kSlotRows = 136;        // S * ceil(128 / S) <= 135 rows of fp32 partials

// dynamic shared memory: ring + (clusters only) the slots the peers push their partial rows into
template <int BN>
constexpr int smem_bytes(int ns, bool split) { return ns * (16384 + BN * 128) + (split ? kSlotRows * (BN * 4 + 16) : 0); }

template <int BN>
void set_attrs() {
    static bool done = false;
    if (done) return;
    cudaFuncSetAttribute(conv_tma_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 2048);
    cudaFuncSetAttribute(conv_tma_kernel<BN>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    done = true;
}

// how many clusters of s CTAs (ring depth ns) can be resident at once
template <int BN>
int max_clusters(int s) {
    static int cache[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (cache[s]) return cache[s];
    set_attrs<BN>();
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(1, 1, s);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem_bytes<BN>(BN == 128 ? 4 : 7, true);
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = s;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, conv_tma_kernel<BN>, &cfg) != cudaSuccess || n <= 0) {
        cudaGetLastError();
        n = s == 1 ? FM_NUM_SMS : -1;
    }
    cache[s] = n;
    return n;
}

int split_limit() {
    static int v = -1;                   // FM_CONV_TMA_SPLIT=<n>: upper bound of the cluster size (1 = never split K)
    if (v < 0) { const char* e = getenv("FM_CONV_TMA_SPLIT"); v = e ? atoi(e) : 8; if (v < 1) v = 1; if (v > 8) v = 8; }
    return v;
}

// cluster size for `tiles` output tiles of nk slices each: the deepest split that still runs as ONE wave of
// co-scheduled clusters and leaves every CTA at least two slices
template <int BN>
int pick_split(int tiles, int nk) {
    if (tiles > 100) return 1;
    int smax = nk / 2 < split_limit() ? nk / 2 : split_limit();
    for (int s = smax; s >= 2; --s)
        if (max_clusters<BN>(s) >= tiles) return s;
    return 1;
}

template <int BN>
int launch_tma(const FmConvDesc* d, const Plan& p, int S, const void* in, const void* wgt, const float* bias,
               const void* residual, void* out, cudaStream_t st) {
    const int kc = d->cin / 64, taps = d->kh * d->kw, nk = taps * kc;
    const int ncol = fm_cdiv(d->cout, BN);
    set_attrs<BN>();
    int sps = fm_cdiv(nk, S);
    S = fm_cdiv(nk, sps);
    // ring depth: as deep as one CTA per SM allows next to the slots of a cluster
    const int ns = S > 1 ? (BN == 128 ? 4 : 7) : (BN == 128 ? 6 : 8);
    const int smem_total = smem_bytes<BN>(ns, S > 1);
    ConvTmaArgs a;
    a.W = p.W; a.H = p.H; a.TW = p.TW; a.TH = p.TH; a.tiles_w = p.tiles_w;
    a.kc = kc; a.kw = d->kw; a.pad = d->pad; a.s2 = d->stride == 2; a.nk = nk; a.sps = sps;
    a.cout = d->cout; a.cout_stride = d->cout_stride; a.cout_offset = d->cout_offset;
    a.res_stride = d->res_stride; a.res_offset = d->res_offset; a.act = d->act;
    a.vec_ok = ((d->cout | d->cout_stride | d->cout_offset) & 7) == 0 &&
               (residual == nullptr || ((d->res_stride | d->res_offset) & 7) == 0);
    a.bias = bias; a.residual = (const __half*)residual; a.out = (__half*)out;
    CUtensorMap map_a, map_b;
    const __half* base = (const __half*)in + d->cin_offset;
    const uint64_t cs = (uint64_t)d->cin_stride;
    int rc;
    if (d->kh == 1) {
        rc = fm_make_tmap_f16_3d(&map_a, base, (uint64_t)d->cin, (uint64_t)p.W, 1, cs, (uint64_t)p.W * cs, 64, 128, 1);
    } else if (d->stride == 1) {
        rc = fm_make_tmap_f16_3d(&map_a, base, (uint64_t)d->cin, (uint64_t)p.W, (uint64_t)p.H, cs, (uint64_t)p.W * cs, 64,
                                 (uint32_t)p.TW, (uint32_t)p.TH);
    } else {
        // [C, w & 1, w / 2, h & 1, h / 2] view of the [hi][wi][C] input
        const uint64_t dims[5] = {(uint64_t)d->cin, 2, (uint64_t)d->wi / 2, 2, (uint64_t)d->hi / 2};
        const uint64_t strides[4] = {cs, 2 * cs, (uint64_t)d->wi * cs, 2 * (uint64_t)d->wi * cs};
        const uint32_t box[5] = {64, 1, (uint32_t)p.TW, 1, (uint32_t)p.TH};
        rc = fm_make_tmap_f16_nd(&map_a, base, 5, dims, strides, box);
    }
    if (rc) return rc;
    const uint64_t ktot = (uint64_t)taps * d->cin;
    rc = fm_make_tmap_f16_3d(&map_b, wgt, ktot, (uint64_t)d->cout, 1, ktot, ktot * d->cout, 64, BN, 1);
    if (rc) return rc;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.tiles, ncol, S);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem_total;
    cfg.stream = st;
    cudaLaunchAttribute attrs[2];
    attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[0].val.programmaticStreamSerializationAllowed = 1;
    if (S > 1) {
        attrs[1].id = cudaLaunchAttributeClusterDimension;
        attrs[1].val.clusterDim.x = 1; attrs[1].val.clusterDim.y = 1; attrs[1].val.clusterDim.z = S;
    }
    cfg.attrs = attrs;
    cfg.numAttrs = S > 1 ? 2 : 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, conv_tma_kernel<BN>, map_a, map_b, a, ns);
    if (e != cudaSuccess) { fm_set_last_error(cudaGetErrorString(e)); return FM_ERR_CUDA; }
    return FM_OK;
}

}  // namespace

extern "C" int fm_conv_tma_set_debug(void* buf) {     // debugging aid, not part of the public header
    unsigned long long* p = (unsigned long long*)buf;
    unsigned int zero = 0;
    cudaMemcpyToSymbol(g_tma_dbg, &p, sizeof(p));
    cudaMemcpyToSymbol(g_tma_dbg_n, &zero, sizeof(zero));
    return FM_OK;
}

extern "C" int fm_conv2d_tma_supported(const FmConvDesc* d) {
    if (!d) return 0;
    if (d->kh != d->kw || (d->kh != 1 && d->kh != 3)) return 0;
    if (d->pad != d->kh / 2) return 0;
    if (d->stride == 1) {
        if (d->hi != d->ho || d->wi != d->wo) return 0;
    } else if (d->stride == 2) {
        if (d->kh != 3 || (d->hi & 1) || (d->wi & 1) || d->ho != d->hi / 2 || d->wo != d->wi / 2) return 0;
    } else {
        return 0;
    }
    if (d->cin < 64 || d->cin % 64 || d->cin_stride % 8 || d->cin_offset % 8) return 0;
    if (d->cout < 8) return 0;
    if (d->kh == 3 && (d->n != 1 || d->wo < 4)) return 0;       // one image per [C, W, H] tensor map
    if ((long long)d->n * d->ho * d->wo <= 0) return 0;
    return 1;
}

extern "C" int fm_conv2d_tma(const FmConvDesc* d, const void* in, const void* wgt, const float* bias, const void* residual,
                             void* out, void* stream) {
    FM_REQUIRE(d != nullptr, "fm_conv2d_tma: desc is NULL");
    FM_REQUIRE(fm_conv2d_tma_supported(d), "fm_conv2d_tma: layer not supported by the TMA path (1x1 s1 / 3x3 s1|s2, same "
                                           "padding, cin % 64 == 0, 8-channel aligned input view)");
    FM_REQUIRE((((uintptr_t)in | (uintptr_t)wgt) & 15) == 0, "fm_conv2d_tma: input / weights must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const Plan p = plan_tiles(d);
    const int nk = d->kh * d->kw * (d->cin / 64);
    // 64-wide filter tiles when 128-wide ones (with the deepest K split the layer allows) would leave half the GPU idle
    int bn = d->cout >= 128 ? 128 : 64;
    if (bn == 128) {
        const int smax = nk / 2 < 8 ? (nk / 2 < 1 ? 1 : nk / 2) : 8;
        if ((long long)p.tiles * fm_cdiv(d->cout, 128) * smax <= FM_NUM_SMS / 2) bn = 64;
    }
    const int tiles = p.tiles * fm_cdiv(d->cout, bn);
    int rc;
    const int S = bn == 128 ? pick_split<128>(tiles, nk) : pick_split<64>(tiles, nk);
    rc = bn == 128 ? launch_tma<128>(d, p, S, in, wgt, bias, residual, out, st)
                   : launch_tma<64>(d, p, S, in, wgt, bias, residual, out, st);
    if (rc) return rc;
    FM_CHECK_LAUNCH("fm_conv2d_tma");
    return FM_OK;
}
