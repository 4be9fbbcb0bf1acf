// Fused OSNet OSBlock kernels for sm_90a (replace the per-layer launches of the ReID stack; role of the TensorRT
// OSNet engine behind fastmot/utils/inference.py:106-117 + fastmot/feature_extractor.py:48-74).
//
// osb_streams_kernel<W, MID, T, NS, CL>  ("kernel S")
//   One CTA owns a strip of T x 128 pixels of one crop (all W columns, SR = 128 T / W rows) and computes, without
//   leaving the SM,   x1 = relu(conv1x1(x) + b1)   and the four Lite-3x3 streams of the block
//       stream s:  (1x1 linear conv -> depthwise 3x3 + bias + ReLU)  x (s + 1)
//   writing only the four stream outputs ("tails", fp16 NHWC) and their per-channel sums (for the channel gate).
//   * conv1: A tiles arrive by TMA (one box per image row, 128-byte swizzle, zero fill outside the image), weight
//     slices by cp.async.bulk, through an NS-stage mbarrier ring filled by one producer warp.
//   * two consumer warpgroups (tile rows 64 g ..) run every 1x1 conv as wgmma with the accumulators in registers.  The
//     conv1 result (x1) and the running stream activation stay in shared memory as fp16 wgmma A tiles (128 pixels x
//     MID, K-major, 128-byte swizzle), written by the threads that compute them.
//   * tile t holds the image rows y = t (mod T) of the strip, so the T pixels a thread owns in the depthwise step (one
//     row in every tile) are vertically adjacent: the depthwise 3x3 loads (T + 2) x 3 neighbours for T outputs.  Its
//     input (the pointwise output, fp16) is chunk-planar [8 channels][row][x], with a zero row above and below.
//   * strips of stage 1 carry a 4-row halo that is recomputed (4 = the deepest stream); rows outside the image are
//     forced to zero after every pointwise conv (= the zero padding of the depthwise conv).
//   Depthwise roles: compute warp w covers pixel quarter w & 3 (one pixel per lane and tile) and channel half w >> 2.
//
// Layouts: activations NHWC fp16; weight images are packed on the host (fastmot_b200/packing.py).
#include "tc_common.cuh"
#include "../../include/fastmot_b200.h"
#include <string.h>

namespace {

using namespace tc;


// optional phase stamps (scripts/osb_phases.py): clock64 of one CTA at the phase boundaries of every level
__device__ long long* g_osb_dbg = nullptr;
#define OSB_STAMP(slot)                                                                        \
    do {                                                                                       \
        if (g_osb_dbg && blockIdx.x == gridDim.x / 2) g_osb_dbg[(slot)] = clock64();           \
    } while (0)

struct OsbStreamsArgs {
    int H, n_crops, cin, R, halo, strips;
    const uint8_t* w1;      // conv1 weight image: cin/64 slices of [MID x 128 B]
    const float* b1;        // [MID]
    const uint8_t* pw;      // 10 pointwise images, each PW_BYTES
    const uint8_t* dw;      // 10 blobs, each DW_BYTES: [9][MID] fp16 | pw bias f32[MID] | dw bias f32[MID]
    __half* tails[4];       // chunk-planar [n][MID / 8][H][W][8] each
    float* gap_part;        // [n][strips][4][MID]
};

// ---- thread-block cluster helpers (DSMEM halo exchange between the strips of one crop) ----
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ void st_cluster_b32(uint32_t local_saddr, uint32_t rank, uint32_t v) {
    uint32_t raddr;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(local_saddr), "r"(rank));
    asm volatile("st.shared::cluster.b32 [%0], %1;" ::"r"(raddr), "r"(v) : "memory");
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// level -> (stream, depth in stream)
__device__ __forceinline__ void level_sj(int lvl, int& s, int& j) {
    if (lvl < 1) { s = 0; j = lvl; }
    else if (lvl < 3) { s = 1; j = lvl - 1; }
    else if (lvl < 6) { s = 2; j = lvl - 3; }
    else { s = 3; j = lvl - 6; }
}

// byte offset of (row, channel pair col) in an fp16 A tile of NSL 64-channel slices (K-major, 128-byte swizzle)
__device__ __forceinline__ uint32_t a_tile_off(int row, int col) {
    return (uint32_t)((col >> 6) * 16384) + sw128_off(row, (col & 63) >> 3) + (uint32_t)((col & 7) * 2);
}

template <int W, int MID, int T, int NS>
struct SCfg {
    static constexpr int NW = 8;                            // compute warps = two consumer warpgroups
    static constexpr int kThreads = NW * 32 + 32;
    static constexpr int SR = 128 * T / W;                  // strip rows
    static constexpr int RQ = 32 / W;                       // image rows per pixel quarter and tile
    static constexpr int TROWS = 128 / W;                   // image rows per tile
    static constexpr int CW = MID / (NW / 4);               // channels per compute warp (depthwise)
    static constexpr int NCH = MID / 8;                     // 16-byte chunks per pixel
    static constexpr int NSL = (MID + 63) / 64;             // K slices of the pointwise weights / activation tiles
    static constexpr int PW_BYTES = NSL * MID * 128;
    static constexpr int DW_BYTES = 9 * MID * 2 + 2 * MID * 4;
    static constexpr int PLANE = (SR + 2) * W * 16;         // bytes of one chunk plane of P
    static constexpr int P_BYTES = NCH * PLANE;
    static constexpr int STAGE = 16384 + MID * 128;
    static constexpr int RING = NS * STAGE;
    static constexpr int REGION = ((P_BYTES > RING ? P_BYTES : RING) + 1023) / 1024 * 1024;
    static constexpr int TILE = NSL * 16384;                // one 128-pixel activation tile (wgmma A operand)
    static constexpr int DWB = (DW_BYTES + 127) / 128 * 128;  // one depthwise / bias blob
    static constexpr int DW_AREA = (2 * DWB + 1023) / 1024 * 1024;   // keeps the swizzled region 1024-byte aligned
    static constexpr int SMEM = PW_BYTES + DW_AREA + REGION + 2 * T * TILE + 4 * NW * CW;
    static_assert(W == 8 || W == 16 || W == 32, "W");
    static_assert(MID % 32 == 0 && MID <= 128, "MID");
    static_assert(SMEM <= 227 * 1024, "shared memory budget");
};

// CL > 1: the CL strips of a crop form a thread-block cluster; nothing is recomputed: after every pointwise conv the
// first / last row of a strip is also stored into the neighbour strip's halo row through distributed shared memory.
// Cluster barrier protocol (every thread of the cluster alternates arrive / wait):
//   arrive (conv1 ring dead)  |  per level:  wait -> pointwise epilogue (local + remote rows) -> arrive, wait ->
//   depthwise -> arrive  |  final wait.
template <int W, int MID, int T, int NS, int CL>
__global__ void __launch_bounds__(8 * 32 + 32, 1)
osb_streams_kernel(const __grid_constant__ CUtensorMap map_x, OsbStreamsArgs a) {
    using C = SCfg<W, MID, T, NS>;
    constexpr int kComputeWarps = C::NW, kComputeThreads = C::NW * 32;
    // 1024-byte alignment comes from the declaration: rounding the pointer through an integer makes the compiler lose
    // the shared address space and emit generic LD/ST
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* s_pw = smem;                                               // pointwise weight image (one level)
    uint8_t* s_dw0 = s_pw + C::PW_BYTES;                                // two depthwise / bias blobs
    constexpr int DWB = C::DWB;
    uint8_t* s_region = s_dw0 + C::DW_AREA;                             // conv1 ring (1024-aligned), later the P planes
    uint8_t* s_x1 = s_region + C::REGION;                               // T tiles of x1
    uint8_t* s_act = s_x1 + T * C::TILE;                                // T tiles of the running stream activation
    float* s_gap = reinterpret_cast<float*>(s_act + T * C::TILE);       // [NW warps][CW]
    __shared__ uint64_t ring_full[NS], ring_empty[NS];
    __shared__ uint64_t pw_full, pw_empty, dw_full[2];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    fm_pdl_trigger();
    const int crop = blockIdx.x / a.strips, strip = blockIdx.x - crop * a.strips;   // CL > 1: strip == cluster rank
    const int y0 = strip * a.R - a.halo;                                // image row of strip row 0
    const int nsl1 = a.cin >> 6;

    if (tid == 0) {
        if (smem_u32(smem) & 1023u) __trap();                           // swizzled tiles need the alignment
        for (int i = 0; i < NS; ++i) { mbar_init(&ring_full[i], 1); mbar_init(&ring_empty[i], kComputeWarps); }
        mbar_init(&pw_full, 1); mbar_init(&pw_empty, kComputeWarps);
        mbar_init(&dw_full[0], 1); mbar_init(&dw_full[1], 1);
        mbar_fence_init();
    }
    if (warp == kComputeWarps && lane == 0) tma_prefetch_desc(&map_x);
    __syncthreads();
    fm_pdl_wait();
    if (tid == 0) OSB_STAMP(0);

    if (warp == kComputeWarps) {
        // =========================================== producer warp =============================================
        if (lane == 0) {
            // weights of level 0
            mbar_expect_tx(&pw_full, C::PW_BYTES);
            bulk_load(s_pw, a.pw, C::PW_BYTES, &pw_full);
            mbar_expect_tx(&dw_full[0], C::DW_BYTES);
            bulk_load(s_dw0, a.dw, C::DW_BYTES, &dw_full[0]);
            // conv1: ring of (A tile slice by TMA, weight slice by bulk copy)
            const int iters = T * nsl1;
            for (int i = 0; i < iters; ++i) {
                const int s = i % NS, t = i / nsl1, ks = i - t * nsl1;
                if (i >= NS) mbar_wait(&ring_empty[s], (uint32_t)((i / NS - 1) & 1));
                uint8_t* sa = s_region + (size_t)s * C::STAGE;
                mbar_expect_tx(&ring_full[s], C::STAGE);
#pragma unroll
                for (int rr = 0; rr < C::TROWS; ++rr) {
                    const int y = y0 + rr * T + t;
                    tma_load_3d(sa + rr * W * 128, &map_x, &ring_full[s], ks * 64, y * W, crop);
                }
                bulk_load(sa + 16384, a.w1 + (size_t)ks * MID * 128, MID * 128, &ring_full[s]);
            }
            OSB_STAMP(1);
        }
        __syncwarp();
        if (CL > 1) cluster_arrive();
        for (int lvl = 0; lvl < 10; ++lvl) {
            if (lvl + 1 < 10 && lane == 0) {
                // every consumer warp's wgmma of this level retired: s_pw is free, and so is the depthwise blob of
                // level lvl - 1 (its depthwise finished before this level's wgmma started)
                mbar_wait(&pw_empty, (uint32_t)(lvl & 1));
                OSB_STAMP(16 + lvl * 16 + 3);
                uint8_t* sd = s_dw0 + ((lvl + 1) & 1) * DWB;
                mbar_expect_tx(&dw_full[(lvl + 1) & 1], C::DW_BYTES);
                bulk_load(sd, a.dw + (size_t)(lvl + 1) * C::DW_BYTES, C::DW_BYTES, &dw_full[(lvl + 1) & 1]);
                mbar_expect_tx(&pw_full, C::PW_BYTES);
                bulk_load(s_pw, a.pw + (size_t)(lvl + 1) * C::PW_BYTES, C::PW_BYTES, &pw_full);
            }
            __syncwarp();
            if (CL > 1) { cluster_wait(); cluster_arrive(); cluster_wait(); cluster_arrive(); }
        }
        if (CL > 1) cluster_wait();
    } else {
        // =========================================== compute warps ============================================
        const int q = warp & 3, g = warp >> 2;
        // depthwise ownership: pixel row q * 32 + lane of every tile, channels c0 .. c0 + CW
        const int yl = lane / W, x = lane % W;
        const int run = q * C::RQ + yl;                                 // vertical run of T rows owned by this thread
        const int c0 = g * C::CW;                                       // first channel of this warp
        // wgmma fragment ownership: tile rows frow + 8 e, channels 8 i + fcol + {0, 1}
        const int frow = g * 64 + q * 16 + (lane >> 2), fcol = (lane & 3) * 2;
        // ---- conv1 (+ relu(acc + b1) -> fp16 -> x1 tiles) ----
        {
            float b[MID / 4];
#pragma unroll
            for (int i = 0; i < MID / 8; ++i) {
                b[2 * i] = __ldg(a.b1 + i * 8 + fcol);
                b[2 * i + 1] = __ldg(a.b1 + i * 8 + fcol + 1);
            }
            for (int t = 0; t < T; ++t) {
                float acc[MID / 2];
#pragma unroll
                for (int e = 0; e < MID / 2; ++e) acc[e] = 0.f;
                for (int ks = 0; ks < nsl1; ++ks) {
                    const int i = t * nsl1 + ks, s = i % NS;
                    mbar_wait(&ring_full[s], (uint32_t)((i / NS) & 1));
                    const uint32_t sa = smem_u32(s_region + (size_t)s * C::STAGE);
                    wg_fence();
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        mma_m64<MID>(acc, smem_desc_sw128(sa + g * 8192 + k * 32), smem_desc_sw128(sa + 16384 + k * 32), 1);
                    wg_commit();
                    wg_wait<0>();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&ring_empty[s]);
                }
#pragma unroll
                for (int i = 0; i < MID / 8; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        *reinterpret_cast<uint32_t*>(s_x1 + t * C::TILE + a_tile_off(frow + 8 * e, i * 8 + fcol)) =
                            pack_h2(fmaxf(acc[i * 4 + 2 * e] + b[2 * i], 0.f), fmaxf(acc[i * 4 + 2 * e + 1] + b[2 * i + 1], 0.f));
            }
            fence_async_smem();                   // x1 (generic stores) -> visible to wgmma
            named_bar_sync(1, kComputeThreads);   // every conv1 wgmma retired: the ring is dead
            // zero the border rows of P
            for (int i = tid; i < C::NCH * 2 * W; i += kComputeThreads) {
                const int ch = i / (2 * W), rem = i - ch * 2 * W, top = rem / W, xx = rem - top * W;
                // in a cluster the inner halo rows belong to the neighbour strips (they write them every level)
                if (CL > 1 && (top ? strip != CL - 1 : strip != 0)) continue;
                *reinterpret_cast<uint4*>(s_region + (size_t)ch * C::PLANE + ((top ? C::SR + 1 : 0) * W + xx) * 16) =
                    make_uint4(0u, 0u, 0u, 0u);
            }
            if (CL > 1) cluster_arrive();         // this CTA's conv1 ring (= the P planes) may now be written remotely
        }
        // ---- levels ----
        for (int lvl = 0; lvl < 10; ++lvl) {
            int s, j;
            level_sj(lvl, s, j);
            const bool tail = j == s;
            const uint8_t* sd = s_dw0 + (lvl & 1) * DWB;
            const __half* dww = reinterpret_cast<const __half*>(sd);                    // [9][MID]
            const float* bpw = reinterpret_cast<const float*>(sd + 9 * MID * 2);        // [MID]
            const float* bdw = bpw + MID;                                               // [MID]
            __half* tail_base = s == 0 ? a.tails[0] : s == 1 ? a.tails[1] : s == 2 ? a.tails[2] : a.tails[3];
            mbar_wait(&pw_full, (uint32_t)(lvl & 1));
            mbar_wait_sleep(&dw_full[lvl & 1], (uint32_t)((lvl >> 1) & 1));
            if (tid == 0) OSB_STAMP(16 + lvl * 16 + 4);
            if (CL > 1) cluster_wait();        // every strip of the crop is done reading its planes (previous level)
            // pointwise conv of tile t (A = x1 or the running activation, B = s_pw) and its epilogue:
            // acc + bias -> fp16 (zero outside the image) -> P planes
            const uint8_t* a_base = j == 0 ? s_x1 : s_act;
            for (int t = 0; t < T; ++t) {
                float acc[MID / 2];
#pragma unroll
                for (int e = 0; e < MID / 2; ++e) acc[e] = 0.f;
                const uint32_t sa = smem_u32(a_base + t * C::TILE) + g * 8192, sb = smem_u32(s_pw);
                wg_fence();
#pragma unroll
                for (int k = 0; k < MID / 16; ++k)
                    mma_m64<MID>(acc, smem_desc_sw128(sa + (k >> 2) * 16384 + (k & 3) * 32),
                                 smem_desc_sw128(sb + (k >> 2) * MID * 128 + (k & 3) * 32), 1);
                wg_commit();
                wg_wait<0>();
                if (t == T - 1) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&pw_empty);
                }
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int row = frow + 8 * e;
                    const int rr = row / W, xx = row - rr * W;
                    const int yloc = rr * T + t, y = y0 + yloc;
                    const bool inside = y >= 0 && y < a.H;
#pragma unroll
                    for (int i = 0; i < MID / 8; ++i) {
                        const int col = i * 8 + fcol;
                        const uint32_t pv = inside ? pack_h2(acc[i * 4 + 2 * e] + bpw[col], acc[i * 4 + 2 * e + 1] + bpw[col + 1]) : 0u;
                        uint8_t* dst = s_region + (size_t)(col >> 3) * C::PLANE + ((yloc + 1) * W + xx) * 16 + (col & 7) * 2;
                        *reinterpret_cast<uint32_t*>(dst) = pv;
                        if (CL > 1) {
                            // first / last row of the strip -> halo row of the strip above / below
                            if (yloc == 0 && strip > 0)
                                st_cluster_b32(smem_u32(dst) + (uint32_t)(C::SR * W * 16), (uint32_t)(strip - 1), pv);
                            if (yloc == C::SR - 1 && strip < CL - 1)
                                st_cluster_b32(smem_u32(dst) - (uint32_t)(C::SR * W * 16), (uint32_t)(strip + 1), pv);
                        }
                    }
                }
            }
            if (tid == 0) OSB_STAMP(16 + lvl * 16 + 6);
            if (CL > 1) { cluster_arrive(); cluster_wait(); }      // all rows (own and halo) of the crop are in place
            else named_bar_sync(1, kComputeThreads);
            if (tid == 0) OSB_STAMP(16 + lvl * 16 + 7);
            // depthwise 3x3 + bias + ReLU over the vertical run of this thread
            float gsum[8];
#pragma unroll
            for (int i = 0; i < C::CW / 8; ++i) {
                const int c8 = c0 / 8 + i;
                const uint8_t* plane = s_region + (size_t)c8 * C::PLANE + (size_t)(run * T) * W * 16;
                __half2 wv[9][4];
#pragma unroll
                for (int k = 0; k < 9; ++k) {
                    const uint4 u = *reinterpret_cast<const uint4*>(dww + k * MID + c8 * 8);
                    wv[k][0] = *reinterpret_cast<const __half2*>(&u.x); wv[k][1] = *reinterpret_cast<const __half2*>(&u.y);
                    wv[k][2] = *reinterpret_cast<const __half2*>(&u.z); wv[k][3] = *reinterpret_cast<const __half2*>(&u.w);
                }
                __half2 bias2[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) bias2[e] = __floats2half2_rn(bdw[c8 * 8 + 2 * e], bdw[c8 * 8 + 2 * e + 1]);
                if (tail) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) gsum[e] = 0.f;
                }
                uint4 win[4][3];
                auto load_row = [&](int r, uint4 (&dst)[3]) {
                    const uint8_t* rp = plane + (size_t)r * W * 16;
                    dst[1] = *reinterpret_cast<const uint4*>(rp + x * 16);
                    dst[0] = x > 0 ? *reinterpret_cast<const uint4*>(rp + (x - 1) * 16) : make_uint4(0u, 0u, 0u, 0u);
                    dst[2] = x < W - 1 ? *reinterpret_cast<const uint4*>(rp + (x + 1) * 16) : make_uint4(0u, 0u, 0u, 0u);
                };
                load_row(0, win[0]);
                load_row(1, win[1]);
                load_row(2, win[2]);
#pragma unroll
                for (int t = 0; t < T; ++t) {
                    if (t + 1 < T) load_row(t + 3, win[(t + 3) & 3]);      // next output's new row, before the math
                    __half2 o[4] = {bias2[0], bias2[1], bias2[2], bias2[3]};
#pragma unroll
                    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                        for (int dx = 0; dx < 3; ++dx) {
                            const uint4& v = win[(t + dy) & 3][dx];
                            o[0] = __hfma2(wv[dy * 3 + dx][0], *reinterpret_cast<const __half2*>(&v.x), o[0]);
                            o[1] = __hfma2(wv[dy * 3 + dx][1], *reinterpret_cast<const __half2*>(&v.y), o[1]);
                            o[2] = __hfma2(wv[dy * 3 + dx][2], *reinterpret_cast<const __half2*>(&v.z), o[2]);
                            o[3] = __hfma2(wv[dy * 3 + dx][3], *reinterpret_cast<const __half2*>(&v.w), o[3]);
                        }
                    const __half2 z = __float2half2_rn(0.f);
                    uint32_t p[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        o[e] = __hmax2(o[e], z);
                        p[e] = *reinterpret_cast<const uint32_t*>(&o[e]);
                    }
                    if (!tail) {
                        // A operand of the next level: tile t, row q * 32 + lane, one 16-byte chunk
                        const int m = q * 32 + lane;
                        *reinterpret_cast<uint4*>(s_act + t * C::TILE + (c8 >> 3) * 16384 + sw128_off(m, c8 & 7)) =
                            make_uint4(p[0], p[1], p[2], p[3]);
                    } else {
                        const int yloc = run * T + t, y = y0 + yloc;
                        if (yloc >= a.halo && yloc < a.halo + a.R && y < a.H) {
                            // chunk-planar tail [crop][chunk][y][x][8]: a warp writes whole 16-byte-per-pixel rows
                            *reinterpret_cast<uint4*>(tail_base + ((((size_t)crop * C::NCH + c8) * a.H + y) * W + x) * 8) =
                                make_uint4(p[0], p[1], p[2], p[3]);
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const float2 f = __half22float2(o[e]);
                                gsum[2 * e] += f.x;
                                gsum[2 * e + 1] += f.y;
                            }
                        }
                    }
                }
                if (tail) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        const float v = warp_sum(gsum[e]);
                        if (lane == 0) s_gap[warp * C::CW + i * 8 + e] = v;
                    }
                }
            }
            if (tail) {
                named_bar_sync(1, kComputeThreads);
                if (tid < MID) {
                    // channel tid belongs to channel half g2; sum its four pixel quarters in a fixed order
                    const int g2 = tid / C::CW, cc = tid - g2 * C::CW;
                    float v = 0.f;
#pragma unroll
                    for (int q2 = 0; q2 < 4; ++q2) v += s_gap[(g2 * 4 + q2) * C::CW + cc];
                    a.gap_part[(((size_t)crop * a.strips + strip) * 4 + s) * MID + tid] = v;
                }
            } else {
                fence_async_smem();               // the activation tiles (generic stores) -> visible to wgmma
            }
            if (tid == 0) OSB_STAMP(16 + lvl * 16 + 8);
            if (CL > 1) cluster_arrive();
            else named_bar_sync(1, kComputeThreads);
        }
        if (CL > 1) cluster_wait();
    }
}

template <int W, int MID, int T, int NS, int CL>
int launch_streams(const FmOsbStreams* d, cudaStream_t st) {
    using C = SCfg<W, MID, T, NS>;
    OsbStreamsArgs a;
    a.H = d->h; a.n_crops = d->n; a.cin = d->cin;
    if (CL > 1) { a.R = C::SR; a.halo = 0; a.strips = CL; }
    else if (d->h == C::SR) { a.R = C::SR; a.halo = 0; a.strips = 1; }
    else { a.halo = 4; a.R = C::SR - 8; a.strips = d->h / a.R; }
    if (a.R <= 0 || a.strips * a.R != d->h) { fm_set_last_error("fm_osb_streams: strip plan"); return FM_ERR_ARG; }
    a.w1 = (const uint8_t*)d->w1; a.b1 = d->b1; a.pw = (const uint8_t*)d->pw; a.dw = (const uint8_t*)d->dw;
    for (int i = 0; i < 4; ++i) a.tails[i] = (__half*)d->tails[i];
    a.gap_part = d->gap_part;
    CUtensorMap map;
    int rc = fm_make_tmap_f16_3d(&map, d->x, (uint64_t)d->cin, (uint64_t)d->h * W, (uint64_t)d->n, (uint64_t)d->cin,
                                 (uint64_t)d->h * W * d->cin, 64, W, 1);
    if (rc) return rc;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(osb_streams_kernel<W, MID, T, NS, CL>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM);
        attr = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(d->n * a.strips);
    cfg.blockDim = dim3(C::kThreads);
    cfg.dynamicSmemBytes = C::SMEM;
    cfg.stream = st;
    cudaLaunchAttribute attrs[2];
    attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[0].val.programmaticStreamSerializationAllowed = 1;
    if (CL > 1) {
        attrs[1].id = cudaLaunchAttributeClusterDimension;
        attrs[1].val.clusterDim.x = CL; attrs[1].val.clusterDim.y = 1; attrs[1].val.clusterDim.z = 1;
    }
    cfg.attrs = attrs;
    cfg.numAttrs = CL > 1 ? 2 : 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, osb_streams_kernel<W, MID, T, NS, CL>, map, a);
    if (e != cudaSuccess) { fm_set_last_error(cudaGetErrorString(e)); return FM_ERR_CUDA; }
    return FM_OK;
}

// =====================================================================================================================
// osb_merge_kernel<MID, NCTA>  ("kernel G"): the second half of an OSBlock in one launch
//     g_s   = sigmoid(W2 relu(W1 mean(tail_s) + b1) + b2)               (unified aggregation gate, s = 0..3)
//     u     = sum_s g_s * tail_s                                        (fp16, never leaves the SM)
//     out   = relu(conv3(u) + b3 + identity)        identity = x (cin == cout)  or  downsample(x) (1x1, cin != cout)
// One CTA = 128 consecutive pixels of one crop x NCTA output channels.  The downsample conv is folded into the same
// accumulation as extra K slices: x tiles arrive by TMA while the two consumer warpgroups build u in shared memory
// (tails are chunk-planar, so lanes run along the pixels and land swizzled rows without bank conflicts); weight slices
// of [W_down | W_3] stream through the same ring by cp.async.bulk (one producer warp).  wgmma 64 x NCTA x 16 per
// warpgroup, accumulators in registers.  Epilogue: registers -> fp16 staging tile -> coalesced rows (+ identity rows
// read coalesced) -> ReLU -> NHWC.
// =====================================================================================================================
}  // namespace
int fm_gate_fc4_part(const float* gap_part, int strips, int n, int hw, const float* w1, const float* b1, const float* w2,
                     const float* b2, float* gate, int c, int cr, cudaStream_t s);    // nn_vec.cu
namespace {

struct OsbMergeArgs {
    int n, hw, cin, cout, strips, has_down, cr;
    const __half* tails[4];      // chunk-planar [n][MID / 8][hw][8]
    const float* gap_part;       // [n][strips][4][MID]
    const float* gates;          // [4][n][MID] sigmoid gates (gate_fc4_part_kernel)
    const uint8_t* wimg;         // per N range: (cin / 64 if has_down) + NSLU slices of [NCTA x 128 B]
    const float* bias;           // [cout] = b3 (+ b_down)
    const __half* res;           // identity [n][hw][cout] or NULL
    __half* out;                 // [n][hw][cout]
};

template <int MID, int NCTA>
struct GCfg {
    static constexpr int NSLU = (MID + 63) / 64;
    static constexpr int NS = 2;
    static constexpr int BSL = NCTA * 128;                  // one weight slice
    static constexpr int STAGE = 16384 + BSL;
    static constexpr int RING = NS * STAGE;
    static constexpr int PITCH = NCTA * 2 + 16;             // staging row
    static constexpr int STG = 128 * PITCH;
    static constexpr int REGION = ((RING > STG ? RING : STG) + 1023) / 1024 * 1024;
    static constexpr int U_BYTES = NSLU * 16384;            // u: NSLU swizzled K slices of [128 pixels x 64]
    static constexpr int SMEM = REGION + U_BYTES + 4 * MID * 4;
    static constexpr int kThreads = 8 * 32 + 32;
};

template <int MID, int NCTA>
__global__ void __launch_bounds__(288, 2)
osb_merge_kernel(const __grid_constant__ CUtensorMap map_x, OsbMergeArgs a) {
    using C = GCfg<MID, NCTA>;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* s_region = smem;                                    // ring (A slice | weight slice), later the staging tile
    uint8_t* s_u = smem + C::REGION;                             // u tile (wgmma A operand)
    float* s_gate = reinterpret_cast<float*>(s_u + C::U_BYTES);  // [4][MID]
    __shared__ uint64_t ring_full[C::NS], ring_empty[C::NS];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    fm_pdl_trigger();
    const int tiles_per = a.hw >> 7;
    const int crop = blockIdx.x / tiles_per, p0 = (blockIdx.x - crop * tiles_per) << 7;
    const int n0 = blockIdx.y * NCTA;
    const int nslx = a.has_down ? (a.cin >> 6) : 0;
    const int iters = nslx + C::NSLU;
    if (tid == 0) {
        if (smem_u32(smem) & 1023u) __trap();
        for (int i = 0; i < C::NS; ++i) { mbar_init(&ring_full[i], 1); mbar_init(&ring_empty[i], 8); }
        mbar_fence_init();
    }
    if (warp == 8 && lane == 0 && a.has_down) tma_prefetch_desc(&map_x);
    __syncthreads();
    fm_pdl_wait();

    if (warp == 8) {
        // ------------------------------------------- producer warp -------------------------------------------
        if (lane == 0) {
            const uint8_t* wimg = a.wimg + (size_t)blockIdx.y * iters * C::BSL;
            for (int i = 0; i < iters; ++i) {
                const int st = i % C::NS;
                if (i >= C::NS) mbar_wait(&ring_empty[st], (uint32_t)((i / C::NS - 1) & 1));
                uint8_t* sa = s_region + (size_t)st * C::STAGE;
                const bool isx = i < nslx;
                mbar_expect_tx(&ring_full[st], (isx ? 16384u : 0u) + (uint32_t)C::BSL);
                if (isx) tma_load_3d(sa, &map_x, &ring_full[st], i * 64, p0, crop);
                bulk_load(sa + 16384, wimg + (size_t)i * C::BSL, C::BSL, &ring_full[st]);
            }
        }
    } else {
        // ------------------------------------------- consumer warpgroups -------------------------------------
        constexpr int NCH = MID / 8;
        // gates of this crop (computed once per crop by the small FC kernel launched before this one)
        for (int i = tid; i < 4 * MID; i += 256) {
            const int st = i / MID, c = i - st * MID;
            s_gate[i] = a.gates[((size_t)st * a.n + crop) * MID + c];
        }
        named_bar_sync(1, 256);
        // u tile: item = (chunk, pixel); lanes run along the pixels (coalesced planar reads, conflict-free swizzled
        // writes)
        for (int i = tid; i < NCH * 128; i += 256) {
            const int c8 = i >> 7, px = i & 127;
            const size_t off = (((size_t)crop * NCH + c8) * a.hw + p0 + px) * 8;
            float o[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) o[q] = 0.f;
#pragma unroll
            for (int st = 0; st < 4; ++st) {
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(a.tails[st] + off));
                const __half2* h = reinterpret_cast<const __half2*>(&v);
                const float* g = s_gate + st * MID + c8 * 8;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float2 f = __half22float2(h[q]);
                    o[2 * q] += f.x * g[2 * q];
                    o[2 * q + 1] += f.y * g[2 * q + 1];
                }
            }
            *reinterpret_cast<uint4*>(s_u + (c8 >> 3) * 16384 + sw128_off(px, c8 & 7)) =
                make_uint4(pack_h2(o[0], o[1]), pack_h2(o[2], o[3]), pack_h2(o[4], o[5]), pack_h2(o[6], o[7]));
        }
        fence_async_smem();            // generic-proxy writes -> visible to the tensor core
        named_bar_sync(1, 256);
        const int g = warp >> 2, wq = warp & 3;
        float acc[NCTA / 2];
#pragma unroll
        for (int e = 0; e < NCTA / 2; ++e) acc[e] = 0.f;
        for (int i = 0; i < iters; ++i) {
            const int st = i % C::NS;
            mbar_wait(&ring_full[st], (uint32_t)((i / C::NS) & 1));
            const bool isx = i < nslx;
            const uint32_t sb = smem_u32(s_region + (size_t)st * C::STAGE) + 16384;
            const uint32_t sa = (isx ? smem_u32(s_region + (size_t)st * C::STAGE) : smem_u32(s_u + (i - nslx) * 16384)) +
                                g * 64 * 128;
            const int ksteps = isx ? 4 : min(4, (MID - (i - nslx) * 64) / 16);
            wg_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (k < ksteps) mma_m64<NCTA>(acc, smem_desc_sw128(sa + k * 32), smem_desc_sw128(sb + k * 32), 1);
            wg_commit();
            wg_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&ring_empty[st]);
        }
        named_bar_sync(1, 256);        // the ring is idle: it becomes the staging tile
#pragma unroll
        for (int i = 0; i < NCTA / 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int row = g * 64 + wq * 16 + (lane >> 2) + e * 8, col = i * 8 + (lane & 3) * 2;
                *reinterpret_cast<uint32_t*>(s_region + row * C::PITCH + col * 2) = pack_h2(acc[i * 4 + e * 2], acc[i * 4 + e * 2 + 1]);
            }
        named_bar_sync(1, 256);
        // coalesced pass: lanes along the channels
        constexpr int CPR = NCTA / 8;                       // 16-byte chunks per row
        for (int i = tid; i < 128 * CPR; i += 256) {
            const int rr = i / CPR, ch = i - rr * CPR;
            const int n = n0 + ch * 8;
            const uint4 pk = *reinterpret_cast<const uint4*>(s_region + rr * C::PITCH + ch * 16);
            const __half2* ph = reinterpret_cast<const __half2*>(&pk);
            const size_t gofs = ((size_t)crop * a.hw + p0 + rr) * a.cout + n;
            const float4 ba = __ldg(reinterpret_cast<const float4*>(a.bias + n));
            const float4 bb = __ldg(reinterpret_cast<const float4*>(a.bias + n + 4));
            float xv[8];
            { const float2 f = __half22float2(ph[0]); xv[0] = f.x + ba.x; xv[1] = f.y + ba.y; }
            { const float2 f = __half22float2(ph[1]); xv[2] = f.x + ba.z; xv[3] = f.y + ba.w; }
            { const float2 f = __half22float2(ph[2]); xv[4] = f.x + bb.x; xv[5] = f.y + bb.y; }
            { const float2 f = __half22float2(ph[3]); xv[6] = f.x + bb.z; xv[7] = f.y + bb.w; }
            if (a.res) {
                const uint4 rv = __ldg(reinterpret_cast<const uint4*>(a.res + gofs));
                const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(rh[e]);
                    xv[2 * e] += f.x;
                    xv[2 * e + 1] += f.y;
                }
            }
            *reinterpret_cast<uint4*>(a.out + gofs) =
                make_uint4(pack_h2(fmaxf(xv[0], 0.f), fmaxf(xv[1], 0.f)), pack_h2(fmaxf(xv[2], 0.f), fmaxf(xv[3], 0.f)),
                           pack_h2(fmaxf(xv[4], 0.f), fmaxf(xv[5], 0.f)), pack_h2(fmaxf(xv[6], 0.f), fmaxf(xv[7], 0.f)));
        }
    }
}

template <int MID, int NCTA>
int launch_merge(const FmOsbMerge* d, cudaStream_t st) {
    using C = GCfg<MID, NCTA>;
    OsbMergeArgs a;
    a.n = d->n; a.hw = d->hw; a.cin = d->cin; a.cout = d->cout; a.strips = d->strips; a.cr = d->cr;
    a.has_down = d->x != nullptr;
    for (int i = 0; i < 4; ++i) a.tails[i] = (const __half*)d->tails[i];
    a.gap_part = d->gap_part;
    a.gates = d->gate_scratch;
    a.wimg = (const uint8_t*)d->wimg; a.bias = d->bias; a.res = (const __half*)d->res; a.out = (__half*)d->out;
    CUtensorMap map;
    memset(&map, 0, sizeof map);
    if (a.has_down) {
        int rc = fm_make_tmap_f16_3d(&map, d->x, (uint64_t)d->cin, (uint64_t)d->hw, (uint64_t)d->n, (uint64_t)d->cin,
                                     (uint64_t)d->hw * d->cin, 64, 128, 1);
        if (rc) return rc;
    }
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(osb_merge_kernel<MID, NCTA>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM);
        attr = true;
    }
    dim3 grid(d->n * (d->hw >> 7), d->cout / NCTA);
    cudaError_t e = fm_launch_pdl(osb_merge_kernel<MID, NCTA>, grid, dim3(C::kThreads), (size_t)C::SMEM, st, map, a);
    if (e != cudaSuccess) { fm_set_last_error(cudaGetErrorString(e)); return FM_ERR_CUDA; }
    return FM_OK;
}

}  // namespace

// output channels per CTA: 64 / 48 accumulators per thread keep two CTAs on an SM
extern "C" int fm_osb_merge_ncta(int mid, int cout) {
    if (mid == 64 && cout % 128 == 0) return 128;
    if (mid == 96 && cout % 96 == 0) return 96;
    if (mid == 128 && cout % 128 == 0) return 128;
    return 0;
}

extern "C" int fm_osb_merge(const FmOsbMerge* d, void* stream) {
    FM_REQUIRE(d != nullptr, "fm_osb_merge: desc is NULL");
    FM_REQUIRE(fm_osb_merge_ncta(d->mid, d->cout) > 0, "fm_osb_merge: unsupported (mid, cout)");
    FM_REQUIRE(d->hw % 128 == 0 && d->cr >= 1 && d->cr <= 8 && d->strips >= 1, "fm_osb_merge: hw / cr / strips");
    FM_REQUIRE((d->x != nullptr) != (d->res != nullptr), "fm_osb_merge: exactly one of x (downsample) and res (identity)");
    FM_REQUIRE(d->x == nullptr || (d->cin % 64 == 0 && d->cin >= 64), "fm_osb_merge: cin must be a multiple of 64");
    FM_REQUIRE(d->gate_scratch != nullptr, "fm_osb_merge: gate_scratch (4 * n * mid floats) is NULL");
    if (d->n <= 0) return FM_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = fm_gate_fc4_part(d->gap_part, d->strips, d->n, d->hw, d->gw1, d->gb1, d->gw2, d->gb2, d->gate_scratch, d->mid,
                              d->cr, st);
    if (rc) return rc;
    if (d->mid == 64) rc = launch_merge<64, 128>(d, st);
    else if (d->mid == 96) rc = launch_merge<96, 96>(d, st);
    else rc = launch_merge<128, 128>(d, st);
    if (rc) return rc;
    FM_CHECK_LAUNCH("fm_osb_merge");
    return FM_OK;
}

namespace {
}  // namespace

extern "C" int fm_osb_set_debug(void* dbg) {     // debugging aid, not part of the public header
    long long* p = (long long*)dbg;
    cudaMemcpyToSymbol(g_osb_dbg, &p, sizeof(p));
    return FM_OK;
}

extern "C" int fm_osb_streams_strips(int h, int w, int mid) {
    if (w == 32 && mid == 64 && h == 64) return 4;  // one 4-CTA cluster per crop
    if (w == 32 && mid == 64) return h == 16 ? 1 : (h % 8 == 0 && h > 16 ? h / 8 : 0);   // 16 rows = one strip, no halo
    if (w == 16 && mid == 96 && h == 32) return 2;  // two-CTA cluster per crop
    if (w == 8 && mid == 128) return h == 16 ? 1 : 0;
    return 0;
}

extern "C" int fm_osb_streams(const FmOsbStreams* d, void* stream) {
    FM_REQUIRE(d != nullptr, "fm_osb_streams: desc is NULL");
    FM_REQUIRE(fm_osb_streams_strips(d->h, d->w, d->mid) > 0, "fm_osb_streams: unsupported stage geometry");
    FM_REQUIRE(d->cin % 64 == 0 && d->cin >= 64, "fm_osb_streams: cin must be a multiple of 64");
    if (d->n <= 0) return FM_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    // stage 1 (w 32): a 4-CTA cluster per 64-row crop, other heights as strips (fm_osb_streams_strips)
    if (d->w == 32 && d->h == 64) rc = launch_streams<32, 64, 4, 3, 4>(d, st);
    else if (d->w == 32) rc = launch_streams<32, 64, 4, 3, 1>(d, st);
    else if (d->w == 16) rc = launch_streams<16, 96, 2, 2, 2>(d, st);       // two 16-row strips per crop
    else rc = launch_streams<8, 128, 1, 2, 1>(d, st);
    if (rc) return rc;
    FM_CHECK_LAUNCH("fm_osb_streams");
    return FM_OK;
}
