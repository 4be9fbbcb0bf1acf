// 16-byte vectorised versions of the bandwidth-bound NHWC fp16 layers (8 channels per thread).  Each `fm_vec_*`
// returns 1 if it handled the call (all channel counts / strides / offsets multiples of 8), 0 otherwise — the
// scalar kernels in nn.cu remain the general path.
#include "common.cuh"
#include "../../include/fastmot_b200.h"

namespace {

// 8 halves moved as ONE 128-bit access.  (A struct of four __half2 is copied member-wise by nvcc -- four 32-bit
// LDG/STG per vector -- so the payload is a uint4 and the half2 view is taken only for arithmetic.)
struct H8 { uint4 u; };
static_assert(sizeof(H8) == 16, "H8 must be 16 bytes");

__device__ __forceinline__ H8 ld8(const __half* p) { H8 h; h.u = *reinterpret_cast<const uint4*>(p); return h; }
__device__ __forceinline__ void st8(__half* p, const H8& v) { *reinterpret_cast<uint4*>(p) = v.u; }
__device__ __forceinline__ float2 h2f(uint32_t w) {
    return __half22float2(*reinterpret_cast<const __half2*>(&w));
}
__device__ __forceinline__ uint32_t f2h(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ void to_f(const H8& h, float* f) {
    float2 t;
    t = h2f(h.u.x); f[0] = t.x; f[1] = t.y;
    t = h2f(h.u.y); f[2] = t.x; f[3] = t.y;
    t = h2f(h.u.z); f[4] = t.x; f[5] = t.y;
    t = h2f(h.u.w); f[6] = t.x; f[7] = t.y;
}
__device__ __forceinline__ H8 to_h(const float* f) {
    H8 h;
    h.u = make_uint4(f2h(f[0], f[1]), f2h(f[2], f[3]), f2h(f[4], f[5]), f2h(f[6], f[7]));
    return h;
}

__device__ __forceinline__ float act_f(float v, int act) {
    switch (act) {
        case FM_ACT_LEAKY: return v > 0.f ? v : 0.1f * v;
        case FM_ACT_RELU: return v > 0.f ? v : 0.f;
        case FM_ACT_MISH: { float sp = v > 20.f ? v : log1pf(__expf(v)); return v * tanhf(sp); }
        case FM_ACT_SWISH: return v / (1.f + __expf(-v));
        case FM_ACT_LOGISTIC: return 1.f / (1.f + __expf(-v));
        default: return v;
    }
}

// depthwise 3x3 s1 p1 + bias + act; thread = (pixel, 8-channel group)
__global__ void __launch_bounds__(256) dwconv3_vec(const __half* __restrict__ in, const __half* __restrict__ w,
                                                    const float* __restrict__ bias, __half* __restrict__ out, int n,
                                                    int h, int wd, int c, int act) {
    const int cg = c >> 3;
    const size_t total = (size_t)n * h * wd * cg;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int g = idx % cg;
        size_t t = idx / cg;
        const int x = t % wd; t /= wd;
        const int y = t % h;
        const int b = t / h;
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = bias ? bias[g * 8 + q] : 0.f;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int yy = y + r - 1;
            if (yy < 0 || yy >= h) continue;
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                const int xx = x + s - 1;
                if (xx < 0 || xx >= wd) continue;
                float a[8], ww[8];
                to_f(ld8(in + (((size_t)b * h + yy) * wd + xx) * c + g * 8), a);
                to_f(ld8(w + (size_t)(r * 3 + s) * c + g * 8), ww);
#pragma unroll
                for (int q = 0; q < 8; ++q) acc[q] += a[q] * ww[q];
            }
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = act_f(acc[q], act);
        st8(out + idx * 8, to_h(acc));
    }
}

// depthwise 3x3: 4 horizontally adjacent pixels x 8 channels per thread (weights and the 3x6 input window are loaded
// once per thread: 18 + 9 vector loads for 4 outputs instead of 4 x 18).  Border taps read a clamped (valid) address
// and are zeroed afterwards, so the six loads of a row carry no control dependence and issue back to back; the
// earlier `continue`-guarded version exposed one DRAM latency per load.
__global__ void __launch_bounds__(256) dwconv3_vec4(const __half* __restrict__ in, const __half* __restrict__ w,
                                                     const float* __restrict__ bias, __half* __restrict__ out, int n,
                                                     int h, int wd, int c, int act) {
    const int cg = c >> 3, xg = wd >> 2;
    const size_t total = (size_t)n * h * xg * cg;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int g = idx % cg;
        size_t t = idx / cg;
        const int x0 = (int)(t % xg) * 4; t /= xg;
        const int y = t % h;
        const int b = t / h;
        // all 18 window loads first (clamped addresses), weights next, math last
        H8 raw[3][6];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int yy = min(max(y + r - 1, 0), h - 1);
            const __half* row = in + (((size_t)b * h + yy) * wd) * c + g * 8;
#pragma unroll
            for (int cx = 0; cx < 6; ++cx) {
                const int xx = min(max(x0 + cx - 1, 0), wd - 1);
                raw[r][cx] = ld8(row + (size_t)xx * c);
            }
        }
        float acc[4][8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float bq = bias ? bias[g * 8 + q] : 0.f;
#pragma unroll
            for (int p = 0; p < 4; ++p) acc[p][q] = bq;
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int yy = y + r - 1;
            const bool rok = yy >= 0 && yy < h;
            float ww[3][8];
#pragma unroll
            for (int k = 0; k < 3; ++k) to_f(ld8(w + (size_t)(r * 3 + k) * c + g * 8), ww[k]);
#pragma unroll
            for (int cx = 0; cx < 6; ++cx) {
                const int xx = x0 + cx - 1;
                const bool ok = rok && xx >= 0 && xx < wd;
                H8 v = raw[r][cx];
                if (!ok) v.u = make_uint4(0u, 0u, 0u, 0u);
                float a[8];
                to_f(v, a);
#pragma unroll
                for (int p = 0; p < 4; ++p) {
                    const int s = cx - p;          // tap column for output pixel p
                    if (s < 0 || s > 2) continue;
#pragma unroll
                    for (int q = 0; q < 8; ++q) acc[p][q] += a[q] * ww[s][q];
                }
            }
        }
#pragma unroll
        for (int p = 0; p < 4; ++p) {
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[p][q] = act_f(acc[p][q], act);
            st8(out + ((((size_t)b * h + y) * wd) + x0 + p) * c + g * 8, to_h(acc[p]));
        }
    }
}

// depthwise 3x3, shared-memory tiled: one CTA owns DW_R output rows of one image (all columns, all channels), stages
// the DW_R + 2 input rows once with cp.async (zero-filled above / below the image) and computes from shared memory.
// The untiled kernel above re-fetches every input pixel ~4.5x through L1/L2 (3 rows x 1.5 column overlap), which is
// what bounded it at ~2 TB/s of useful traffic; here HBM sees (DW_R + 2) / DW_R reads + 1 write.
constexpr int DW_R = 8;

__global__ void __launch_bounds__(256, 3) dwconv3_tile(const __half* __restrict__ in, const __half* __restrict__ w,
                                                     const float* __restrict__ bias, __half* __restrict__ out, int h,
                                                     int wd, int c, int act) {
    extern __shared__ __align__(16) unsigned char dw_smem[];
    __half* tile = reinterpret_cast<__half*>(dw_smem);                       // [(DW_R+2)][wd][c]
    __half* sw = tile + (size_t)(DW_R + 2) * wd * c;                         // [9][c]
    fm_pdl_trigger();
    const int cg = c >> 3, xg = wd >> 2;
    const int b = blockIdx.y, y0 = blockIdx.x * DW_R;
    const int rows_in = DW_R + 2;
    for (int i = threadIdx.x; i < 9 * cg; i += blockDim.x) {       // weights do not depend on the previous kernel
        const unsigned dst = (unsigned)__cvta_generic_to_shared(sw + (size_t)i * 8);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, 16;" ::"r"(dst), "l"(w + (size_t)i * 8));
    }
    fm_pdl_wait();
    const __half* img = in + (size_t)b * h * wd * c;
    // ---- stage rows y0-1 .. y0+DW_R: they are one contiguous run of 16-byte chunks in the image (full-width rows), so
    // chunk i of the tile is chunk first + i of the image; chunks before / after the image are zero-filled ----
    const int row_chunks = wd * cg;
    const int first = (y0 - 1) * row_chunks, img_chunks = h * row_chunks;
    for (int i = threadIdx.x; i < rows_in * row_chunks; i += blockDim.x) {
        const int gi = first + i;
        const bool ok = gi >= 0 && gi < img_chunks;
        const __half* src = img + (size_t)(ok ? gi : 0) * 8;
        const unsigned dst = (unsigned)__cvta_generic_to_shared(tile + (size_t)i * 8);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16u : 0u));
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    // ---- compute: item = (row, 4-pixel group, 8-channel group) ----
    const int items = DW_R * xg * cg;
    for (int it = threadIdx.x; it < items; it += blockDim.x) {
        const int g = it % cg;
        int t = it / cg;
        const int x0 = (t % xg) * 4;
        const int ry = t / xg;
        const int y = y0 + ry;
        if (y >= h) break;                       // items are row-major: everything after is out of range too
        float acc[4][8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float bq = bias ? bias[g * 8 + q] : 0.f;
#pragma unroll
            for (int p = 0; p < 4; ++p) acc[p][q] = bq;
        }
        // One window row at a time: the three taps of a row are combined in packed fp16 (HMUL2 + 2 HFMA2 per channel
        // pair, no conversions), the three row sums and the bias are accumulated in fp32.  The all-fp32 version spent
        // ~45 % of its instructions on FFMA + half->float conversions and was issue bound (ncu: 68 % issue active,
        // 1126 instructions per 4-pixel item); the row sums carry two fp16 roundings each, the same order as the
        // final fp16 store.
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const __half* row = tile + ((size_t)(ry + r) * wd) * c + g * 8;
            __half2 wv[3][4], av[6][4];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const uint4 u = ld8(sw + (size_t)(r * 3 + k) * c + g * 8).u;
                wv[k][0] = *reinterpret_cast<const __half2*>(&u.x); wv[k][1] = *reinterpret_cast<const __half2*>(&u.y);
                wv[k][2] = *reinterpret_cast<const __half2*>(&u.z); wv[k][3] = *reinterpret_cast<const __half2*>(&u.w);
            }
#pragma unroll
            for (int cx = 0; cx < 6; ++cx) {
                const int xx = x0 + cx - 1;
                uint4 u = make_uint4(0u, 0u, 0u, 0u);
                if (xx >= 0 && xx < wd) u = ld8(row + (size_t)xx * c).u;
                av[cx][0] = *reinterpret_cast<const __half2*>(&u.x); av[cx][1] = *reinterpret_cast<const __half2*>(&u.y);
                av[cx][2] = *reinterpret_cast<const __half2*>(&u.z); av[cx][3] = *reinterpret_cast<const __half2*>(&u.w);
            }
#pragma unroll
            for (int p = 0; p < 4; ++p)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    __half2 sm = __hmul2(wv[0][j], av[p][j]);
                    sm = __hfma2(wv[1][j], av[p + 1][j], sm);
                    sm = __hfma2(wv[2][j], av[p + 2][j], sm);
                    const float2 f = __half22float2(sm);
                    acc[p][2 * j] += f.x;
                    acc[p][2 * j + 1] += f.y;
                }
        }
        __half* orow = out + (((size_t)b * h + y) * wd + x0) * c + g * 8;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[p][q] = act_f(acc[p][q], act);
            st8(orow + (size_t)p * c, to_h(acc[p]));
        }
    }
}

// out = act(a + b), contiguous
__global__ void __launch_bounds__(256) add_act_vec(const __half* __restrict__ a, const __half* __restrict__ b,
                                                    __half* __restrict__ out, size_t n8, int act) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
        float x[8], y[8];
        to_f(ld8(a + i * 8), x);
        to_f(ld8(b + i * 8), y);
#pragma unroll
        for (int q = 0; q < 8; ++q) x[q] = act_f(x[q] + y[q], act);
        st8(out + i * 8, to_h(x));
    }
}

__global__ void __launch_bounds__(256) add_act_strided_vec(const __half* __restrict__ a, int as, int ao,
                                                            const __half* __restrict__ b, int bs, int bo,
                                                            __half* __restrict__ out, int os, int oo, size_t pixels,
                                                            int c, int act) {
    const int cg = c >> 3;
    const size_t total = pixels * cg;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t p = i / cg;
        const int g = (int)(i - p * cg) * 8;
        float x[8], y[8];
        to_f(ld8(a + p * as + ao + g), x);
        to_f(ld8(b + p * bs + bo + g), y);
#pragma unroll
        for (int q = 0; q < 8; ++q) x[q] = act_f(x[q] + y[q], act);
        st8(out + p * os + oo + g, to_h(x));
    }
}

__global__ void __launch_bounds__(256) avgpool2_vec(const __half* __restrict__ in, __half* __restrict__ out, int n,
                                                     int hi, int wi, int c) {
    const int ho = hi / 2, wo = wi / 2, cg = c >> 3;
    const size_t total = (size_t)n * ho * wo * cg;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int g = idx % cg;
        size_t t = idx / cg;
        const int x = t % wo; t /= wo;
        const int y = t % ho;
        const int b = t / ho;
        const __half* p = in + (((size_t)b * hi + 2 * y) * wi + 2 * x) * c + g * 8;
        float a0[8], a1[8], a2[8], a3[8];
        to_f(ld8(p), a0); to_f(ld8(p + c), a1); to_f(ld8(p + (size_t)wi * c), a2); to_f(ld8(p + (size_t)wi * c + c), a3);
#pragma unroll
        for (int q = 0; q < 8; ++q) a0[q] = 0.25f * (a0[q] + a1[q] + a2[q] + a3[q]);
        st8(out + idx * 8, to_h(a0));
    }
}

__global__ void __launch_bounds__(256) maxpool_vec(const __half* __restrict__ in, __half* __restrict__ out, int n,
                                                    int hi, int wi, int c, int cis, int cio, int ho, int wo, int cos,
                                                    int coo, int k, int stride, int plh, int plw) {
    const int cg = c >> 3;
    const size_t total = (size_t)n * ho * wo * cg;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int g = idx % cg;
        size_t t = idx / cg;
        const int x = t % wo; t /= wo;
        const int y = t % ho;
        const int b = t / ho;
        float best[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) best[q] = -INFINITY;
        for (int r = 0; r < k; ++r) {
            const int yy = y * stride - plh + r;
            if (yy < 0 || yy >= hi) continue;
            for (int s = 0; s < k; ++s) {
                const int xx = x * stride - plw + s;
                if (xx < 0 || xx >= wi) continue;
                float a[8];
                to_f(ld8(in + (((size_t)b * hi + yy) * wi + xx) * cis + cio + g * 8), a);
#pragma unroll
                for (int q = 0; q < 8; ++q) best[q] = fmaxf(best[q], a[q]);
            }
        }
        st8(out + (((size_t)b * ho + y) * wo + x) * cos + coo + g * 8, to_h(best));
    }
}

__global__ void __launch_bounds__(256) upsample_copy_vec(const __half* __restrict__ in, __half* __restrict__ out, int n,
                                                          int hi, int wi, int c, int cis, int cio, int s, int cos,
                                                          int coo) {
    const int ho = hi * s, wo = wi * s, cg = c >> 3;
    const size_t total = (size_t)n * ho * wo * cg;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int g = idx % cg;
        size_t t = idx / cg;
        const int x = t % wo; t /= wo;
        const int y = t % ho;
        const int b = t / ho;
        st8(out + (((size_t)b * ho + y) * wo + x) * cos + coo + g * 8,
            ld8(in + (((size_t)b * hi + y / s) * wi + x / s) * cis + cio + g * 8));
    }
}

// global average pool: one CTA per (sample, 64-channel slab); lanes over channel groups, warps over pixels
__global__ void __launch_bounds__(256) gap_vec(const __half* __restrict__ in, float* __restrict__ out, int hw, int c) {
    __shared__ float s_acc[32][65];
    const int b = blockIdx.x, slab = blockIdx.y;
    const int c0 = slab * 64;
    const int cgs = min(64, c - c0) >> 3;          // channel groups in this slab (<= 8)
    const int tid = threadIdx.x;
    const int g = tid % 8, prow = tid / 8;         // 32 pixel rows
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    if (g < cgs) {
        const __half* p = in + (size_t)b * hw * c + c0 + g * 8;
        for (int i = prow; i < hw; i += 32) {
            float a[8];
            to_f(ld8(p + (size_t)i * c), a);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += a[q];
        }
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) s_acc[prow][g * 8 + q] = acc[q];
    __syncthreads();
    if (tid < 64 && c0 + tid < c) {
        float a = 0.f;
        for (int r = 0; r < 32; ++r) a += s_acc[r][tid];
        out[(size_t)b * c + c0 + tid] = a / hw;
    }
}

__global__ void __launch_bounds__(256) gate_apply_vec(const __half* __restrict__ x, const float* __restrict__ gate,
                                                       __half* __restrict__ acc, size_t per_sample, int c, size_t total8,
                                                       int accumulate) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total8; i += (size_t)gridDim.x * blockDim.x) {
        const size_t e = i * 8;
        const int ch = e % c;
        const size_t b = e / per_sample;
        float v[8], a[8];
        to_f(ld8(x + e), v);
        const float* gp = gate + b * c + ch;
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] *= gp[q];
        if (accumulate) {
            to_f(ld8(acc + e), a);
#pragma unroll
            for (int q = 0; q < 8; ++q) v[q] += a[q];
        }
        st8(acc + e, to_h(v));
    }
}

inline int vgrid(size_t total, int block = 256) {
    size_t g = (total + block - 1) / block;
    size_t cap = (size_t)FM_NUM_SMS * 32;
    return (int)(g < cap ? (g ? g : 1) : cap);
}
inline bool al8(int v) { return (v & 7) == 0; }

}  // namespace

int fm_vec_dwconv3(const void* in, const void* w, const float* bias, void* out, int n, int h, int wd, int c, int act,
                   cudaStream_t s) {
    if (!al8(c)) return 0;
    if ((wd & 3) == 0) {
        const size_t tile_bytes = ((size_t)(DW_R + 2) * wd + 9) * c * sizeof(__half);
        if (tile_bytes <= 96 * 1024 && h >= DW_R) {
            static size_t attr_bytes = 0;
            if (tile_bytes > attr_bytes) {
                cudaFuncSetAttribute(dwconv3_tile, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(96 * 1024));
                attr_bytes = 96 * 1024;
            }
            dim3 grid((h + DW_R - 1) / DW_R, n);
            fm_launch_pdl(dwconv3_tile, grid, dim3(256), tile_bytes, s, (const __half*)in, (const __half*)w, bias,
                          (__half*)out, h, wd, c, act);
            return 1;
        }
        const size_t total4 = (size_t)n * h * (wd >> 2) * (c >> 3);
        dwconv3_vec4<<<vgrid(total4), 256, 0, s>>>((const __half*)in, (const __half*)w, bias, (__half*)out, n, h, wd, c,
                                                   act);
        return 1;
    }
    const size_t total = (size_t)n * h * wd * (c >> 3);
    dwconv3_vec<<<vgrid(total), 256, 0, s>>>((const __half*)in, (const __half*)w, bias, (__half*)out, n, h, wd, c, act);
    return 1;
}
int fm_vec_add_act(const void* a, const void* b, void* out, long long n, int act, cudaStream_t s) {
    if (n & 7) return 0;
    add_act_vec<<<vgrid((size_t)n >> 3), 256, 0, s>>>((const __half*)a, (const __half*)b, (__half*)out, (size_t)n >> 3, act);
    return 1;
}
int fm_vec_add_act_strided(const void* a, int as, int ao, const void* b, int bs, int bo, void* out, int os, int oo,
                           long long pixels, int c, int act, cudaStream_t s) {
    if (!(al8(as) && al8(ao) && al8(bs) && al8(bo) && al8(os) && al8(oo) && al8(c))) return 0;
    add_act_strided_vec<<<vgrid((size_t)pixels * (c >> 3)), 256, 0, s>>>((const __half*)a, as, ao, (const __half*)b, bs,
                                                                        bo, (__half*)out, os, oo, (size_t)pixels, c, act);
    return 1;
}
int fm_vec_avgpool2(const void* in, void* out, int n, int hi, int wi, int c, cudaStream_t s) {
    if (!al8(c)) return 0;
    avgpool2_vec<<<vgrid((size_t)n * (hi / 2) * (wi / 2) * (c >> 3)), 256, 0, s>>>((const __half*)in, (__half*)out, n, hi,
                                                                                  wi, c);
    return 1;
}
int fm_vec_maxpool(const void* in, void* out, int n, int hi, int wi, int c, int cis, int cio, int ho, int wo, int cos,
                   int coo, int k, int stride, int plh, int plw, cudaStream_t s) {
    if (!(al8(c) && al8(cis) && al8(cio) && al8(cos) && al8(coo))) return 0;
    maxpool_vec<<<vgrid((size_t)n * ho * wo * (c >> 3)), 256, 0, s>>>((const __half*)in, (__half*)out, n, hi, wi, c, cis,
                                                                     cio, ho, wo, cos, coo, k, stride, plh, plw);
    return 1;
}
int fm_vec_upsample_copy(const void* in, void* out, int n, int hi, int wi, int c, int cis, int cio, int sc, int cos,
                         int coo, cudaStream_t s) {
    if (!(al8(c) && al8(cis) && al8(cio) && al8(cos) && al8(coo))) return 0;
    upsample_copy_vec<<<vgrid((size_t)n * hi * sc * wi * sc * (c >> 3)), 256, 0, s>>>(
        (const __half*)in, (__half*)out, n, hi, wi, c, cis, cio, sc, cos, coo);
    return 1;
}
int fm_vec_gap(const void* in, float* out, int n, int hw, int c, cudaStream_t s) {
    if (!al8(c)) return 0;
    dim3 grid(n, (c + 63) / 64);
    gap_vec<<<grid, 256, 0, s>>>((const __half*)in, out, hw, c);
    return 1;
}
int fm_vec_gate_apply(const void* x, const float* gate, void* acc, size_t per_sample, int c, size_t total, int accumulate,
                      cudaStream_t s) {
    if (!al8(c)) return 0;
    gate_apply_vec<<<vgrid(total >> 3), 256, 0, s>>>((const __half*)x, gate, (__half*)acc, per_sample, c, total >> 3,
                                                     accumulate);
    return 1;
}

// ---------------------------------------------------------------------------------------------------------
// OSNet unified aggregation gate for the four streams of a block (shared gate weights):
//   acc = sum_s x_s * sigmoid(W2 relu(W1 GAP(x_s) + b1) + b2)
// three launches (pool all streams, tiny FCs, one fused apply) instead of 4 x (pool, FC, read-modify-write).
// ---------------------------------------------------------------------------------------------------------
namespace {

struct Ptr4 { const __half* p[4]; };

__global__ void __launch_bounds__(256) gap4_vec(Ptr4 x, float* __restrict__ pooled /* [4][n][c] */, int n, int hw, int c) {
    __shared__ float s_acc[32][65];
    const int b = blockIdx.x, slab = blockIdx.y, st = blockIdx.z;
    const int c0 = slab * 64;
    const int cgs = min(64, c - c0) >> 3;
    const int tid = threadIdx.x, g = tid % 8, prow = tid / 8;
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    if (g < cgs) {
        const __half* p = x.p[st] + (size_t)b * hw * c + c0 + g * 8;
        for (int i = prow; i < hw; i += 32) {
            float a[8];
            to_f(ld8(p + (size_t)i * c), a);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += a[q];
        }
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) s_acc[prow][g * 8 + q] = acc[q];
    __syncthreads();
    if (tid < 64 && c0 + tid < c) {
        float a = 0.f;
        for (int r = 0; r < 32; ++r) a += s_acc[r][tid];
        pooled[((size_t)st * n + b) * c + c0 + tid] = a / hw;
    }
}

__global__ void __launch_bounds__(128) gate_fc4_kernel(const float* __restrict__ pooled, const float* __restrict__ w1,
                                                        const float* __restrict__ b1, const float* __restrict__ w2,
                                                        const float* __restrict__ b2, float* __restrict__ gate, int c,
                                                        int cr) {
    extern __shared__ float sh[];
    float* sp = sh;
    float* sh1 = sh + c;
    const size_t row = blockIdx.x;          // st * n + b
    for (int i = threadIdx.x; i < c; i += blockDim.x) sp[i] = pooled[row * c + i];
    __syncthreads();
    for (int j = threadIdx.x; j < cr; j += blockDim.x) {
        float a = b1[j];
        for (int i = 0; i < c; ++i) a += w1[(size_t)j * c + i] * sp[i];
        sh1[j] = a > 0.f ? a : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        float a = b2[i];
        for (int j = 0; j < cr; ++j) a += w2[(size_t)i * cr + j] * sh1[j];
        gate[row * c + i] = 1.f / (1.f + __expf(-a));
    }
}

__global__ void __launch_bounds__(256) gate_apply4_vec(Ptr4 x, const float* __restrict__ gate /* [4][n][c] */,
                                                        __half* __restrict__ acc, size_t per_sample, int n, int c,
                                                        size_t total8) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total8; i += (size_t)gridDim.x * blockDim.x) {
        const size_t e = i * 8;
        const int ch = e % c;
        const size_t b = e / per_sample;
        float out[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) out[q] = 0.f;
#pragma unroll
        for (int st = 0; st < 4; ++st) {
            float v[8];
            to_f(ld8(x.p[st] + e), v);
            const float* gp = gate + ((size_t)st * n + b) * c + ch;
#pragma unroll
            for (int q = 0; q < 8; ++q) out[q] += v[q] * gp[q];
        }
        st8(acc + e, to_h(out));
    }
}

}  // namespace

namespace {
// gate FCs fed by the per-strip channel sums fm_osb_streams leaves behind (no separate pooling pass)
__global__ void __launch_bounds__(128) gate_fc4_part_kernel(const float* __restrict__ gap_part, int strips, int n, int hw,
                                                             const float* __restrict__ w1, const float* __restrict__ b1,
                                                             const float* __restrict__ w2, const float* __restrict__ b2,
                                                             float* __restrict__ gate, int c, int cr) {
    extern __shared__ float sh[];
    float* sp = sh;
    float* sh1 = sh + c;
    const int st = blockIdx.x / n, b = blockIdx.x - st * n;
    const float inv = 1.f / (float)hw;
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        float a = 0.f;
        for (int k = 0; k < strips; ++k) a += gap_part[(((size_t)b * strips + k) * 4 + st) * c + i];
        sp[i] = a * inv;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < cr; j += blockDim.x) {
        float a = b1[j];
        for (int i = 0; i < c; ++i) a += w1[(size_t)j * c + i] * sp[i];
        sh1[j] = a > 0.f ? a : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        float a = b2[i];
        for (int j = 0; j < cr; ++j) a += w2[(size_t)i * cr + j] * sh1[j];
        gate[(size_t)blockIdx.x * c + i] = 1.f / (1.f + __expf(-a));
    }
}
}  // namespace

namespace {
// acc[b][p][c] = sum_s gate[s][b][c] * tail_s[b][c / 8][p][c % 8]: the tails come chunk-planar from fm_osb_streams (lanes
// along the pixels on the read side), the sum leaves NHWC (lanes along the channels on the write side); 64 pixels per
// block go through shared memory in between.
__global__ void __launch_bounds__(256) gate_apply4_planar(Ptr4 x, const float* __restrict__ gate /* [4][n][c] */,
                                                           __half* __restrict__ acc, int n, int hw, int c) {
    extern __shared__ uint8_t sh_t[];
    const int nch = c >> 3, pitch = c * 2 + 16;
    const int blocks_per = hw >> 6;
    const int b = blockIdx.x / blocks_per, p0 = (blockIdx.x - b * blocks_per) << 6;
    for (int i = threadIdx.x; i < nch * 64; i += blockDim.x) {
        const int chunk = i >> 6, px = i & 63;
        float out[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) out[q] = 0.f;
        const size_t off = (((size_t)b * nch + chunk) * hw + p0 + px) * 8;
#pragma unroll
        for (int st = 0; st < 4; ++st) {
            float v[8];
            to_f(ld8(x.p[st] + off), v);
            const float* gp = gate + ((size_t)st * n + b) * c + chunk * 8;
#pragma unroll
            for (int q = 0; q < 8; ++q) out[q] += v[q] * gp[q];
        }
        *reinterpret_cast<H8*>(sh_t + px * pitch + chunk * 16) = to_h(out);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nch * 64; i += blockDim.x) {
        const int px = i / nch, chunk = i - px * nch;
        st8(acc + ((size_t)b * hw + p0 + px) * c + chunk * 8, *reinterpret_cast<const H8*>(sh_t + px * pitch + chunk * 16));
    }
}
}  // namespace

// gate FCs of one OSBlock from the strip sums (shared with fm_osb_merge): gate[4][n][c]
int fm_gate_fc4_part(const float* gap_part, int strips, int n, int hw, const float* w1, const float* b1, const float* w2,
                     const float* b2, float* gate, int c, int cr, cudaStream_t s) {
    gate_fc4_part_kernel<<<4 * n, 128, (c + cr) * sizeof(float), s>>>(gap_part, strips, n, hw, w1, b1, w2, b2, gate, c, cr);
    fm_count_launches(1);
    return FM_OK;
}

// tails chunk-planar [n][c / 8][hw][8] (fm_osb_streams output), acc NHWC; hw must be a multiple of 64
extern "C" int fm_channel_gate4_pooled(const void* x0, const void* x1, const void* x2, const void* x3,
                                       const float* gap_part, int strips, float* gate, const float* w1, const float* b1,
                                       const float* w2, const float* b2, void* acc, int n, int hw, int c, int cr,
                                       void* stream) {
    if (n <= 0) return FM_OK;
    if ((c & 7) || (hw & 63)) {
        fm_set_last_error("fm_channel_gate4_pooled: c must be a multiple of 8 and hw a multiple of 64");
        return FM_ERR_ARG;
    }
    cudaStream_t s = (cudaStream_t)stream;
    Ptr4 p;
    p.p[0] = (const __half*)x0; p.p[1] = (const __half*)x1; p.p[2] = (const __half*)x2; p.p[3] = (const __half*)x3;
    gate_fc4_part_kernel<<<4 * n, 128, (c + cr) * sizeof(float), s>>>(gap_part, strips, n, hw, w1, b1, w2, b2, gate, c, cr);
    gate_apply4_planar<<<n * (hw >> 6), 256, 64 * (c * 2 + 16), s>>>(p, gate, (__half*)acc, n, hw, c);
    fm_count_launches(1);
    FM_CHECK_LAUNCH("fm_channel_gate4_pooled");
    return FM_OK;
}

extern "C" int fm_channel_gate4(const void* x0, const void* x1, const void* x2, const void* x3, float* pooled,
                                float* gate, const float* w1, const float* b1, const float* w2, const float* b2,
                                void* acc, int n, int hw, int c, int cr, void* stream) {
    if (n <= 0) return FM_OK;
    if (c & 7) {
        fm_set_last_error("fm_channel_gate4: channel count must be a multiple of 8");
        return FM_ERR_ARG;
    }
    cudaStream_t s = (cudaStream_t)stream;
    Ptr4 p;
    p.p[0] = (const __half*)x0; p.p[1] = (const __half*)x1; p.p[2] = (const __half*)x2; p.p[3] = (const __half*)x3;
    dim3 g1(n, (c + 63) / 64, 4);
    gap4_vec<<<g1, 256, 0, s>>>(p, pooled, n, hw, c);
    gate_fc4_kernel<<<4 * n, 128, (c + cr) * sizeof(float), s>>>(pooled, w1, b1, w2, b2, gate, c, cr);
    const size_t total = (size_t)n * hw * c;
    gate_apply4_vec<<<vgrid(total >> 3), 256, 0, s>>>(p, gate, (__half*)acc, (size_t)hw * c, n, c, total >> 3);
    fm_count_launches(2);
    FM_CHECK_LAUNCH("fm_channel_gate4");
    return FM_OK;
}
