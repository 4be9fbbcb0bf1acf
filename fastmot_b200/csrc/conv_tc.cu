// wgmma implicit-GEMM convolution for sm_90a (the dense contraction of the detector and ReID stacks).
//
//   D[M = N*Ho*Wo pixels, Cout] = im2col(X)[M, K = kh*kw*Cin] * W^T[K, Cout],  fp16 operands, fp32 accumulate.
//
// conv_tc_kernel<BN, STAGES, SPLITK>: one CTA (one warpgroup) computes a 128 x BN output tile as two m64 halves.  The
// K loop walks 64-element slices: all 128 threads gather the A slice (128 pixels x 64 reduction elements, zero-filled
// at the image border; 1x1 / stride-1 layers skip the im2col index arithmetic) and the B slice (BN filters x 64) with
// 16-byte cp.async (LDGSTS) copies straight into the 128-byte-swizzled K-major layout wgmma reads; the warpgroup then
// issues 2 x 4 wgmma.mma_async (64 x BN x 16) per slice, accumulators in registers.  The smem ring is STAGES deep with
// STAGES-1 slices of copies in flight; a stage is refilled only after the wgmma that read it retired.  STAGES is chosen
// against the wave capacity of the layer (launch code at the bottom): deep rings for one-wave layers, shallow rings
// (more resident CTAs) for many-wave ones.
// Epilogue: the accumulator fragments are staged in the now idle ring buffers and written out with lanes running
// along the channels (row-coalesced 16-byte stores), fusing bias + activation (+ residual, + channel-slice offsets, so
// route/concat layers need no copy).
// Under-filled grids split K over blockIdx.z (as many splits as fit in ONE wave of resident CTAs); the partial
// tiles go through the same smem transpose to an fp32 workspace and splitk_reduce_kernel finishes the layer.
// All launches are programmatic-dependent-launch chains (common.cuh).
//
// The split-K scratch belongs to the caller (FmConvDesc.ws): one per engine / stream, no library-global state.
//
// Replaces the TensorRT conv tactics behind fastmot/utils/inference.py:106-117.
#include "tc_common.cuh"
#include "../../include/fastmot_b200.h"
#include "conv_act.cuh"

namespace {

using tc::smem_u32;

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;           // fp16 elements per K slice = one 128-byte swizzle row

__device__ unsigned long long* g_dbg_dev = nullptr;   // optional per-CTA phase timestamps (scripts/bench_conv.py)

__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
#define DBG_STAMP(k)                                                                             \
    do {                                                                                         \
        if (g_dbg_dev && tid == 0) {                                                             \
            const int cta = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);      \
            if (cta < 4096) g_dbg_dev[cta * 8 + (k)] = gtimer();                                 \
        }                                                                                        \
    } while (0)

// Epilogue for 32 consecutive output channels of one pixel row: bias + activation (+ residual) and fp16 NHWC store.
// A thread writes one full 32-byte sector (two back-to-back 16-byte stores) whenever the slice is 32-byte aligned:
// single 16-byte stores to rows that are hundreds of bytes apart are partial-sector writes.
__device__ __forceinline__ void epilogue_store32(float (&v32)[32], size_t m, int n_base, const FmConvDesc& d,
                                                 const float* __restrict__ bias, const __half* __restrict__ residual,
                                                 __half* __restrict__ out, int act, bool res_first) {
    // every index into v32 is a compile-time constant after unrolling: the accumulators must stay in registers
    // (a first version indexed them dynamically and the epilogue ran out of local memory)
    const bool al16 = ((d.cout_stride | d.cout_offset) & 15) == 0;
    const bool res16 = residual != nullptr && ((d.res_stride | d.res_offset) & 15) == 0;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int n = n_base + hh * 16;
        if (n < d.cout) {
            const bool full = n + 16 <= d.cout;
            float v[16];
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const float x = v32[hh * 16 + q] + ((bias && (full || n + q < d.cout)) ? bias[n + q] : 0.f);
                v[q] = res_first ? x : tc_act(x, act);
            }
            __half* op = out + m * d.cout_stride + d.cout_offset + n;
            if (full && al16) {
                if (residual) {
                    const __half* rp = residual + m * d.res_stride + d.res_offset + n;
                    if (res16) {
                        const uint4 r0 = *reinterpret_cast<const uint4*>(rp);
                        const uint4 r1 = *reinterpret_cast<const uint4*>(rp + 8);
                        const uint32_t r[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&r[q]));
                            v[2 * q] += f.x; v[2 * q + 1] += f.y;
                        }
                    } else {
#pragma unroll
                        for (int q = 0; q < 16; ++q) v[q] += __half2float(rp[q]);
                    }
                }
                uint32_t w[8];
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float a = res_first ? tc_act(v[2 * q], act) : v[2 * q];
                    const float b = res_first ? tc_act(v[2 * q + 1], act) : v[2 * q + 1];
                    const __half2 h = __floats2half2_rn(a, b);
                    w[q] = *reinterpret_cast<const uint32_t*>(&h);
                }
                *reinterpret_cast<uint4*>(op) = make_uint4(w[0], w[1], w[2], w[3]);
                *reinterpret_cast<uint4*>(op + 8) = make_uint4(w[4], w[5], w[6], w[7]);
            } else {
#pragma unroll
                for (int q = 0; q < 16; ++q) {
                    if (n + q < d.cout) {
                        float x = v[q];
                        if (residual) x += __half2float(residual[m * d.res_stride + d.res_offset + n + q]);
                        op[q] = __float2half(res_first ? tc_act(x, act) : x);
                    }
                }
            }
        }
    }
}


// Staged epilogue of one warp's 32 x BN slab of the fp16 tile in shared memory (row pitch BN * 2 + 16 bytes):
// written back with lanes running along the channels, so each store instruction covers whole rows; a lane keeps the
// same 8 channels for every row and so loads its bias once.  Needs 8-channel alignment of the output / residual views.
template <int BN>
__device__ __forceinline__ void epilogue_staged(const uint8_t* stg, int lane, int m_warp0, int n0, int M,
                                                const FmConvDesc& d, const float* __restrict__ bias,
                                                const __half* __restrict__ residual, __half* __restrict__ out,
                                                int act, bool res_first) {
    constexpr int PITCH = BN * 2 + 16;           // bytes; +16 keeps the per-row 16-byte accesses conflict-free
    constexpr int CPR = BN / 8;                  // 16-byte chunks per row
    constexpr int RPI = 32 / CPR;                // rows per store instruction
    const int chunk = lane % CPR, rsub = lane / CPR;
    const int n = n0 + chunk * 8;
    if (n < d.cout) {                            // cout % 8 == 0 (staged_ok): the whole chunk is in range
        float b8[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) b8[q] = bias ? bias[n + q] : 0.f;
        const __half* rp = residual ? residual + d.res_offset + n : nullptr;
        __half* op = out + d.cout_offset + n;
#pragma unroll 2
        for (int r0 = 0; r0 < 32; r0 += RPI) {
            const int row = r0 + rsub;
            const int mm = m_warp0 + row;
            if (mm >= M) break;
            const uint4 pk = *reinterpret_cast<const uint4*>(stg + row * PITCH + chunk * 16);
            const __half2* ph = reinterpret_cast<const __half2*>(&pk);
            float x[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 f = __half22float2(ph[q]);
                x[2 * q] = f.x + b8[2 * q];
                x[2 * q + 1] = f.y + b8[2 * q + 1];
            }
            if (!res_first) tc_act8(x, act);
            if (rp) {
                const uint4 rv = *reinterpret_cast<const uint4*>(rp + (size_t)mm * d.res_stride);
                const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float2 f = __half22float2(rh[q]);
                    x[2 * q] += f.x;
                    x[2 * q + 1] += f.y;
                }
            }
            if (res_first) tc_act8(x, act);
            uint32_t w[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const __half2 h = __floats2half2_rn(x[2 * q], x[2 * q + 1]);
                w[q] = *reinterpret_cast<const uint32_t*>(&h);
            }
            *reinterpret_cast<uint4*>(op + (size_t)mm * d.cout_stride) = make_uint4(w[0], w[1], w[2], w[3]);
        }
    }
    __syncwarp();
}

__device__ __forceinline__ bool staged_ok(const FmConvDesc& d, const void* residual) {
    return ((d.cout_stride | d.cout_offset | d.cout) & 7) == 0 &&
           (residual == nullptr || ((d.res_stride | d.res_offset) & 7) == 0);
}

// The accumulators of both m64 halves live in registers (BN floats per thread); SPLITK instantiations also carry the
// partial-sum path.
template <int BN, int STAGES, bool SPLITK>
__global__ void __launch_bounds__(128) conv_tc_kernel(FmConvDesc d, const __half* __restrict__ in,
                                                       const __half* __restrict__ wgt, const float* __restrict__ bias,
                                                       const __half* __restrict__ residual, __half* __restrict__ out,
                                                       float* ws, int slices_per_split) {
    // 1024-byte alignment for the 128B swizzle atoms, by declaration (rounding the pointer through an integer makes the
    // compiler fall back to generic LD / ST for the staged epilogue)
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr int A_BYTES = TC_BM * 128, B_BYTES = BN * 128, STAGE_BYTES = A_BYTES + B_BYTES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    fm_pdl_trigger();
    DBG_STAMP(0);
    const int m0 = blockIdx.x * TC_BM, n0 = blockIdx.y * BN;
    const int M = d.n * d.ho * d.wo;
    const int Ktot = d.kh * d.kw * d.cin;
    const int nk_total = (Ktot + TC_BK - 1) / TC_BK;
    // split-K: blockIdx.z owns K slices [kb0, kb0 + nk); partial sums go to the fp32 workspace
    const int kb0 = blockIdx.z * slices_per_split;
    const int nk = min(nk_total - kb0, slices_per_split);
    DBG_STAMP(1);

    // ---- per-thread gather plan: chunk column c (16 B = 8 channels), rows (tid>>3) + 16*i ----
    const int c = tid & 7;
    const int rbase = tid >> 3;
    int pn[8], ph[8], pw[8];
    // 1x1 / stride 1 / no padding: input pixel == output pixel, no index arithmetic at all
    const bool pointwise = d.kh == 1 && d.kw == 1 && d.stride == 1 && d.pad == 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + rbase + 16 * i;
        if (pointwise) {
            pn[i] = m < M ? 0 : -1; ph[i] = 0; pw[i] = 0;
        } else if (m < M) {
            const int wo = m % d.wo, t = m / d.wo, ho = t % d.ho;
            pn[i] = t / d.ho;
            ph[i] = ho * d.stride - d.pad;
            pw[i] = wo * d.stride - d.pad;
        } else {
            pn[i] = -1; ph[i] = 0; pw[i] = 0;
        }
    }

    // cp.async (LDGSTS) gather of K-slice `kb` into ring stage `st`; out-of-image / out-of-range chunks are
    // zero-filled by passing src-size 0.
    auto issue_loads = [&](int kb, int st) {
        uint8_t* sA = smem + (size_t)st * STAGE_BYTES;
        uint8_t* sB = sA + A_BYTES;
        const int kelem = (kb0 + kb) * TC_BK + c * 8;
        const bool kvalid = kelem < Ktot;
        if (pointwise) {
            const __half* base = in + d.cin_offset + (kvalid ? kelem : 0);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int r = rbase + 16 * i;
                const bool ok = kvalid && pn[i] >= 0;
                const __half* src = ok ? base + (size_t)(m0 + r) * d.cin_stride : in;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(sA + r * 128 + ((c ^ (r & 7)) << 4))),
                             "l"(src), "r"(ok ? 16u : 0u));
            }
        } else {
        const int tap = kvalid ? kelem / d.cin : 0;
        const int cch = kvalid ? kelem - tap * d.cin : 0;
        const int fr = tap / d.kw, fs = tap - fr * d.kw;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = rbase + 16 * i;
            const __half* src = in;
            uint32_t bytes = 0;
            if (kvalid && pn[i] >= 0) {
                const int hi = ph[i] + fr, wi = pw[i] + fs;
                if (hi >= 0 && hi < d.hi && wi >= 0 && wi < d.wi) {
                    src = in + (((size_t)pn[i] * d.hi + hi) * d.wi + wi) * d.cin_stride + d.cin_offset + cch;
                    bytes = 16;
                }
            }
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(sA + r * 128 + ((c ^ (r & 7)) << 4))),
                         "l"(src), "r"(bytes));
        }
        }
#pragma unroll
        for (int i = 0; i < BN / 16; ++i) {
            const int r = rbase + 16 * i;
            const int n = n0 + r;
            const bool ok = kvalid && n < d.cout;
            const __half* src = ok ? wgt + (size_t)n * Ktot + kelem : wgt;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(sB + r * 128 + ((c ^ (r & 7)) << 4))),
                         "l"(src), "r"(ok ? 16u : 0u));
        }
    };

    // everything above is independent of other kernels' output; the activations (and the split-K workspace /
    // output buffers, which an earlier kernel may still be reading) are not
    fm_pdl_wait();
    float acc[2][BN / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
#pragma unroll
    for (int p = 0; p < STAGES - 1; ++p) {
        if (p < nk) issue_loads(p, p);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    DBG_STAMP(2);
    for (int kb = 0; kb < nk; ++kb) {
        const int s = kb % STAGES;
        if (STAGES == 1) {
            issue_loads(kb, 0);
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        asm volatile("cp.async.wait_group %0;" ::"n"(STAGES > 1 ? STAGES - 2 : 0) : "memory");   // slice kb landed
        tc::fence_async_smem();  // make the smem writes visible to the tensor-core (async) proxy
        // every thread is here: slice kb is complete, and the wgmma of slice kb - 1 has retired in every warp
        __syncthreads();
        if (STAGES > 1) {
            const int kn = kb + STAGES - 1;        // refills the stage of slice kb - 1
            if (kn < nk) issue_loads(kn, kn % STAGES);
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        const uint32_t a_addr = smem_u32(smem + (size_t)s * STAGE_BYTES), b_addr = a_addr + A_BYTES;
        tc::wg_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) {
            // advance 16 elements (32 bytes) along K inside the swizzle atom
            const uint64_t bdesc = tc::smem_desc_sw128(b_addr + k * 32);
#pragma unroll
            for (int h = 0; h < 2; ++h)
                tc::mma_m64<BN>(acc[h], tc::smem_desc_sw128(a_addr + h * 64 * 128 + k * 32), bdesc, 1);
        }
        tc::wg_commit();
        tc::wg_wait<0>();
        if (STAGES == 1) __syncthreads();
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    DBG_STAMP(3);
    __syncthreads();                              // the ring is idle: it becomes the staging tile
    DBG_STAMP(4);

    // ---- epilogue ----
    const int m = m0 + tid;
    const int act = d.act & 0xff;
    const bool res_first = (d.act & FM_ACT_AFTER_RESIDUAL) != 0;
    const bool staged = !SPLITK && staged_ok(d, residual);
    constexpr int PITCH16 = BN * 2 + 16, PITCH32 = BN * 4 + 16;
    // fragments -> smem rows: fp16 for the staged epilogue, raw fp32 otherwise
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < BN / 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int row = h * 64 + warp * 16 + (lane >> 2) + e * 8, col = i * 8 + (lane & 3) * 2;
                const float x0 = acc[h][i * 4 + e * 2], x1 = acc[h][i * 4 + e * 2 + 1];
                if (staged)
                    *reinterpret_cast<uint32_t*>(smem + row * PITCH16 + col * 2) = tc::pack_h2(x0, x1);
                else
                    *reinterpret_cast<float2*>(smem + row * PITCH32 + col * 4) = make_float2(x0, x1);
            }
    __syncthreads();
    if (staged) {
        epilogue_staged<BN>(smem + (size_t)warp * 32 * PITCH16, lane, m0 + warp * 32, n0, M, d, bias, residual, out,
                            act, res_first);
    } else if (SPLITK && (d.cout & 3) == 0) {
        // raw fp32 partials, whole rows per store instruction
        const uint8_t* stg = smem + (size_t)warp * 32 * PITCH32;
        constexpr int LPR = BN / 4, RPI = 32 / LPR;
        const int n = n0 + (lane % LPR) * 4;
        float* wz = ws + (size_t)blockIdx.z * M * d.cout;
#pragma unroll 4
        for (int r0 = 0; r0 < 32; r0 += RPI) {
            const int row = r0 + lane / LPR;
            const int mm = m0 + warp * 32 + row;
            if (mm < M && n < d.cout)
                *reinterpret_cast<float4*>(wz + (size_t)mm * d.cout + n) =
                    *reinterpret_cast<const float4*>(stg + row * PITCH32 + (lane % LPR) * 16);
        }
    } else {
        // one output row per thread, 32 channels at a time
#pragma unroll 1
        for (int j0 = 0; j0 < BN; j0 += 32) {
            float v32[32];
#pragma unroll
            for (int q = 0; q < 32; q += 4) {
                const float4 f = *reinterpret_cast<const float4*>(smem + tid * PITCH32 + (j0 + q) * 4);
                v32[q] = f.x; v32[q + 1] = f.y; v32[q + 2] = f.z; v32[q + 3] = f.w;
            }
            if (j0 == 0) DBG_STAMP(7);
            if (m >= M) continue;
            if (SPLITK) {                     // raw fp32 partials; bias / activation happen in splitk_reduce_kernel
                float* wp = ws + ((size_t)blockIdx.z * M + m) * d.cout + n0 + j0;
#pragma unroll
                for (int q = 0; q < 32; ++q)
                    if (n0 + j0 + q < d.cout) wp[q] = v32[q];
                continue;
            }
            epilogue_store32(v32, (size_t)m, n0 + j0, d, bias, residual, out, act, res_first);
        }
    }
    DBG_STAMP(5);
    DBG_STAMP(6);
}

__global__ void __launch_bounds__(256) splitk_reduce_kernel(FmConvDesc d, const float* __restrict__ ws, int splits,
                                                             const float* __restrict__ bias,
                                                             const __half* __restrict__ residual,
                                                             __half* __restrict__ out) {
    fm_pdl_trigger();
    fm_pdl_wait();
    const int M = d.n * d.ho * d.wo;
    const size_t total = (size_t)M * d.cout;
    const int act = d.act & 0xff;
    const bool res_first = (d.act & FM_ACT_AFTER_RESIDUAL) != 0;
    if (staged_ok(d, residual)) {
        // 8 channels per thread: two 128-bit partial-sum loads per split, one 128-bit store
        const int cg = d.cout >> 3;
        const size_t total8 = (size_t)M * cg;
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total8;
             i += (size_t)gridDim.x * blockDim.x) {
            const size_t m = i / cg;
            const int n = (int)(i - m * cg) * 8;
            float x[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) x[q] = bias ? bias[n + q] : 0.f;
            const float* wp = ws + m * d.cout + n;
            for (int z = 0; z < splits; ++z) {
                const float4 a = *reinterpret_cast<const float4*>(wp + (size_t)z * total);
                const float4 b2 = *reinterpret_cast<const float4*>(wp + (size_t)z * total + 4);
                x[0] += a.x; x[1] += a.y; x[2] += a.z; x[3] += a.w;
                x[4] += b2.x; x[5] += b2.y; x[6] += b2.z; x[7] += b2.w;
            }
            if (!res_first) tc_act8(x, act);
            if (residual) {
                const uint4 rv = *reinterpret_cast<const uint4*>(residual + m * d.res_stride + d.res_offset + n);
                const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float2 f = __half22float2(rh[q]);
                    x[2 * q] += f.x;
                    x[2 * q + 1] += f.y;
                }
            }
            if (res_first) tc_act8(x, act);
            uint32_t w[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const __half2 h = __floats2half2_rn(x[2 * q], x[2 * q + 1]);
                w[q] = *reinterpret_cast<const uint32_t*>(&h);
            }
            *reinterpret_cast<uint4*>(out + m * d.cout_stride + d.cout_offset + n) = make_uint4(w[0], w[1], w[2], w[3]);
        }
        return;
    }
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t m = i / d.cout;
        const int n = (int)(i - m * d.cout);
        float acc = 0.f;
        for (int z = 0; z < splits; ++z) acc += ws[(size_t)z * total + i];
        float v = acc + (bias ? bias[n] : 0.f);
        if (!res_first) v = tc_act(v, act);
        if (residual) v += __half2float(residual[m * d.res_stride + d.res_offset + n]);
        if (res_first) v = tc_act(v, act);
        out[m * d.cout_stride + d.cout_offset + n] = __float2half(v);
    }
}

template <int BN, int STAGES>
int launch_tc(const FmConvDesc* d, const void* in, const void* wgt, const float* bias, const void* residual, void* out,
              cudaStream_t s) {
    // the ring doubles as the epilogue's staging tile (128 rows x (BN*4+16) bytes at most)
    constexpr int ring = STAGES * (TC_BM * 128 + BN * 128), stg32 = TC_BM * (BN * 4 + 16);
    constexpr int smem = (ring > stg32 ? ring : stg32) + 1024;
    constexpr int smem_split = smem;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(conv_tc_kernel<BN, STAGES, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(conv_tc_kernel<BN, STAGES, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_split);
        attr = true;
    }
    const int M = d->n * d->ho * d->wo;
    const int nk = (d->kh * d->kw * d->cin + TC_BK - 1) / TC_BK;
    dim3 grid(fm_cdiv(M, TC_BM), fm_cdiv(d->cout, BN), 1);
    int sps = nk;
    // split-K when the output tiling alone cannot fill the SMs (batch-1 deep layers)
    const int tiles = grid.x * grid.y;
    float* ws = (float*)d->ws;
    if (ws && tiles <= FM_NUM_SMS / 2 && nk >= 8) {
        // as many K splits as still fit in ONE wave of resident CTAs: one CTA more than the SMs hold runs after the
        // others and doubles the layer time
        constexpr int per_sm = (227 * 1024) / (smem_split + 1024) > 0 ? (227 * 1024) / (smem_split + 1024) : 1;
        int want = FM_NUM_SMS * per_sm / tiles;
        if (want > nk / 4) want = nk / 4;
        if (want > 1) {
            sps = (nk + want - 1) / want;
            const int splits = (nk + sps - 1) / sps;
            if ((long long)splits * M * d->cout * 4 <= d->ws_bytes) grid.z = splits; else sps = nk;
        }
    }
    if (grid.z > 1)
        fm_launch_pdl(conv_tc_kernel<BN, STAGES, true>, grid, dim3(128), (size_t)smem_split, s, *d, (const __half*)in,
                      (const __half*)wgt, bias, (const __half*)residual, (__half*)out, ws, sps);
    else
        fm_launch_pdl(conv_tc_kernel<BN, STAGES, false>, grid, dim3(128), (size_t)smem, s, *d, (const __half*)in,
                      (const __half*)wgt, bias, (const __half*)residual, (__half*)out, ws, sps);
    if (grid.z > 1) {
        const size_t total = (size_t)M * d->cout;
        const int blocks = (int)((total + 255) / 256 < (size_t)FM_NUM_SMS * 8 ? (total + 255) / 256 : FM_NUM_SMS * 8);
        fm_launch_pdl(splitk_reduce_kernel, dim3(blocks), dim3(256), (size_t)0, s, *d, (const float*)ws, (int)grid.z,
                      bias, (const __half*)residual, (__half*)out);
        fm_count_launches(1);
    }
    return 0;
}

}  // namespace

extern "C" int fm_conv_set_debug(void* dbg) {
    unsigned long long* p = (unsigned long long*)dbg;
    cudaMemcpyToSymbol(g_dbg_dev, &p, sizeof(p));
    return FM_OK;
}

extern "C" int fm_conv2d_tc_supported(const FmConvDesc* d) {
    if (!d) return 0;
    if (d->cin % 8 || d->cin_stride % 8 || d->cin_offset % 8) return 0;   // 16-byte operand chunks
    if ((long long)d->kh * d->kw * d->cin < 32) return 0;                  // not worth a tensor-core tile
    if (d->n * d->ho * d->wo <= 0 || d->cout <= 0) return 0;
    return 1;
}

extern "C" int fm_conv2d_tc(const FmConvDesc* d, const void* in, const void* wgt, const float* bias,
                            const void* residual, void* out, void* stream) {
    FM_REQUIRE(d != nullptr, "fm_conv2d_tc: desc is NULL");
    FM_REQUIRE(fm_conv2d_tc_supported(d), "fm_conv2d_tc: shape not supported by the wgmma path");
    cudaStream_t s = (cudaStream_t)stream;
    const int nk = (d->kh * d->kw * d->cin + TC_BK - 1) / TC_BK;
    const int m_tiles_all = (d->n * d->ho * d->wo + TC_BM - 1) / TC_BM;
    // ring depth follows the K extent: short reductions (OSNet 1x1) want many co-resident CTAs, long ones (3x3 on
    // wide layers) want many slices of copies in flight
    int bn = d->cout <= 32 ? 32 : d->cout <= 64 ? 64 : 128;
    if (bn == 128) {
        // between half a wave and two waves of 128-wide tiles, 64-wide tiles fill the SMs better (e.g.
        // 128->128 @ 224x16x8 and the 80x80 YOLO 3x3); fewer tiles than that go to split-K instead
        const int tiles128 = m_tiles_all * ((d->cout + 127) / 128);
        if (tiles128 > FM_NUM_SMS / 2 && tiles128 < 2 * FM_NUM_SMS) bn = 64;
    }
    // Ring depth: deep rings hide the gather latency of a long K loop, but they cost residency (6 x 32 KB = one CTA
    // per SM).  What decides is how the tile count sits against one wave of resident CTAs:
    //   * the layer fits in one wave at the deep setting          -> deep ring (and split-K fills the idle SMs),
    //   * it fits in one wave only with a shallower ring          -> that ring (a second, mostly empty wave doubles
    //                                                                the layer time),
    //   * many waves either way (OSNet stem, first YOLO layers)   -> shallow ring, residency hides the latency.
    const int tiles = m_tiles_all * ((d->cout + bn - 1) / bn);
    if (bn == 32) {
        if (nk == 1) launch_tc<32, 1>(d, in, wgt, bias, residual, out, s);
        else if (nk <= 2 || tiles > 5 * FM_NUM_SMS) launch_tc<32, 2>(d, in, wgt, bias, residual, out, s);
        else launch_tc<32, 4>(d, in, wgt, bias, residual, out, s);
    } else if (bn == 64) {
        // 64-wide: 4 stages = 96 KB (2 CTAs / SM), 2 stages = 48 KB (4 / SM)
        if (nk == 1) launch_tc<64, 1>(d, in, wgt, bias, residual, out, s);
        else if (nk <= 2 || tiles > 2 * FM_NUM_SMS)
            launch_tc<64, 2>(d, in, wgt, bias, residual, out, s);   // e.g. the OSNet 7x7 stem
        else launch_tc<64, 4>(d, in, wgt, bias, residual, out, s);
    } else {
        // 128-wide: 6 stages = 192 KB (1 CTA / SM), 3 stages = 96 KB (2 / SM), 2 stages = 64 KB (3 / SM)
        if (nk == 1) launch_tc<128, 1>(d, in, wgt, bias, residual, out, s);
        else if (nk <= 2 || tiles > 2 * FM_NUM_SMS) launch_tc<128, 2>(d, in, wgt, bias, residual, out, s);
        else if (nk < 6 || tiles > FM_NUM_SMS) launch_tc<128, 3>(d, in, wgt, bias, residual, out, s);
        else launch_tc<128, 6>(d, in, wgt, bias, residual, out, s);
    }
    FM_CHECK_LAUNCH("fm_conv2d_tc");
    return FM_OK;
}
