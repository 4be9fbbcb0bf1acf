// Rectangular LSA with a whole CTA (one thread per remaining column): a replay of SciPy's shortest-augmenting-path
// solver (`remaining` is filled in reverse and compacted by swap-with-last; among equal minima the LAST unassigned
// column in scan order wins, otherwise the FIRST minimum; doubles are combined in SciPy's order
// ((minVal + c) - u) - v), with the per-step scan, the dual update and the resets spread over up to 1024 threads.
// Bit-exact by construction: every floating-point expression is evaluated by exactly one thread in SciPy's order;
// only the (associative) min / index selection is parallel.
#include "common.cuh"
#include "../../include/fastmot_b200.h"
#include "assoc_lsa.cuh"

namespace {

struct Bufs {
    double *u, *v, *spc;
    int *path, *col4row, *row4col, *remaining;
    unsigned char *SR, *SC;
};

__device__ __forceinline__ Bufs carve(unsigned char* base, int nr, int nc) {
    Bufs b;
    size_t off = 0;
    b.u = (double*)(base + off); off += sizeof(double) * nr;
    b.v = (double*)(base + off); off += sizeof(double) * nc;
    b.spc = (double*)(base + off); off += sizeof(double) * nc;
    b.path = (int*)(base + off); off += sizeof(int) * nc;
    b.col4row = (int*)(base + off); off += sizeof(int) * nr;
    b.row4col = (int*)(base + off); off += sizeof(int) * nc;
    b.remaining = (int*)(base + off); off += sizeof(int) * nc;
    b.SR = base + off; off += nr;
    b.SC = base + off;
    return b;
}

__global__ void __launch_bounds__(1024) lsa_block_kernel(const double* __restrict__ cost, int nr0, int nc0,
                                                          int* __restrict__ out_col4row, int* __restrict__ status,
                                                          unsigned char* gws, int use_smem) {
    extern __shared__ __align__(16) unsigned char s_ws[];
    __shared__ double s_wmin[32];
    __shared__ int s_wfirst[32], s_wlast[32];
    __shared__ double s_minval;
    __shared__ int s_i, s_sink, s_numrem, s_infeasible;
    const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, wid = tid >> 5, nwarps = T >> 5;
    const bool transpose = nc0 < nr0;
    const int nr = transpose ? nc0 : nr0;
    const int nc = transpose ? nr0 : nc0;
    Bufs B = carve(use_smem ? s_ws : gws, nr, nc);
#define COST(i, j) (transpose ? cost[(size_t)(j) * nc0 + (i)] : cost[(size_t)(i) * nc0 + (j)])
    for (int k = tid; k < nr; k += T) { B.u[k] = 0.0; B.col4row[k] = -1; }
    for (int k = tid; k < nc; k += T) { B.v[k] = 0.0; B.row4col[k] = -1; B.path[k] = -1; }
    if (tid == 0) { status[0] = 0; s_infeasible = 0; }
    __syncthreads();
    for (int curRow = 0; curRow < nr; ++curRow) {
        for (int k = tid; k < nc; k += T) { B.remaining[k] = nc - k - 1; B.SC[k] = 0; B.spc[k] = INFINITY; }
        for (int k = tid; k < nr; k += T) B.SR[k] = 0;
        if (tid == 0) { s_minval = 0.0; s_i = curRow; s_sink = -1; s_numrem = nc; }
        __syncthreads();
        while (true) {
            const int i = s_i;
            const int num_remaining = s_numrem;
            const double minVal = s_minval;
            const double ui = B.u[i];
            double l_min = INFINITY;
            int l_first = 0x7fffffff, l_lastU = -1;
            for (int it = tid; it < num_remaining; it += T) {
                const int j = B.remaining[it];
                const double r = __dsub_rn(__dsub_rn(__dadd_rn(minVal, COST(i, j)), ui), B.v[j]);
                double s = B.spc[j];
                if (r < s) { B.path[j] = i; B.spc[j] = r; s = r; }
                const bool un = B.row4col[j] == -1;
                if (s < l_min) { l_min = s; l_first = it; l_lastU = un ? it : -1; }
                else if (s == l_min) { if (l_first == 0x7fffffff) l_first = it; if (un) l_lastU = it; }
            }
            // warp level
            double m = l_min;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmin(m, __shfl_xor_sync(0xffffffffu, m, o));
            int cf = (l_min == m) ? l_first : 0x7fffffff;
            int cl = (l_min == m) ? l_lastU : -1;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                cf = min(cf, __shfl_xor_sync(0xffffffffu, cf, o));
                cl = max(cl, __shfl_xor_sync(0xffffffffu, cl, o));
            }
            if (lane == 0) { s_wmin[wid] = m; s_wfirst[wid] = cf; s_wlast[wid] = cl; }
            __syncthreads();
            if (tid == 0) {
                if (i == curRow || true) B.SR[i] = 1;
                double gm = INFINITY;
                for (int w = 0; w < nwarps; ++w) gm = fmin(gm, s_wmin[w]);
                int gf = 0x7fffffff, gl = -1;
                for (int w = 0; w < nwarps; ++w)
                    if (s_wmin[w] == gm) { gf = min(gf, s_wfirst[w]); gl = max(gl, s_wlast[w]); }
                if (gm == INFINITY) {
                    s_infeasible = 1;
                } else {
                    s_minval = gm;
                    const int index = (gl >= 0) ? gl : gf;
                    const int j = B.remaining[index];
                    const int r4c = B.row4col[j];
                    if (r4c == -1) s_sink = j; else s_i = r4c;
                    B.SC[j] = 1;
                    B.remaining[index] = B.remaining[num_remaining - 1];
                    s_numrem = num_remaining - 1;
                }
            }
            __syncthreads();
            if (s_infeasible || s_sink != -1) break;
        }
        if (s_infeasible) break;
        const double minVal = s_minval;
        const int sink = s_sink;
        if (tid == 0) B.u[curRow] = __dadd_rn(B.u[curRow], minVal);
        for (int k = tid; k < nr; k += T)
            if (B.SR[k] && k != curRow) B.u[k] = __dadd_rn(B.u[k], __dsub_rn(minVal, B.spc[B.col4row[k]]));
        for (int k = tid; k < nc; k += T)
            if (B.SC[k]) B.v[k] = __dsub_rn(B.v[k], __dsub_rn(minVal, B.spc[k]));
        __syncthreads();
        if (tid == 0) {
            int j = sink;
            while (true) {
                const int ii = B.path[j];
                B.row4col[j] = ii;
                const int tmp = B.col4row[ii];
                B.col4row[ii] = j;
                j = tmp;
                if (ii == curRow) break;
            }
        }
        __syncthreads();
    }
    if (s_infeasible) {
        if (tid == 0) status[0] = 1;
        for (int k = tid; k < nr0; k += T) out_col4row[k] = -1;
        return;
    }
    for (int k = tid; k < nr0; k += T) {
        int c = transpose ? B.row4col[k] : B.col4row[k];
        if (c >= 0 && cost[(size_t)k * nc0 + c] >= FM_INF_COST) c = -2 - c;
        out_col4row[k] = c;
    }
#undef COST
}


// -----------------------------------------------------------------------------------------------------------------
// Version 2 (columns <= 1024): one column per thread with all per-column state in registers (reduced cost spc,
// dual v, path, row4col, position in SciPy's `remaining` array), ONE barrier per inner step and no serial section:
// every warp publishes its (minimum, last unassigned tie, first tie) and all threads reduce the <= 32 entries
// redundantly.  The cost row of the next `curRow` is prefetched while the current row is solved, the visited rows'
// dual updates use u[r] += minVal - (minVal at the step that reached r) -- the same value SciPy reads back as
// shortestPathCosts[col4row[r]] -- and only the augmenting-path walk (a few links) is done by one thread.
// Same replay of scipy/optimize/rectangular_lsap/rectangular_lsap.cpp as above: scan order of `remaining`
// (positions), swap-with-last compaction, "last unassigned among equal minima, else first minimum", fp64 operation
// order -> bit-exact assignments, also with ties.
// -----------------------------------------------------------------------------------------------------------------
using lsa::dkey;

struct WarpEntry { unsigned long long key; int posU, posF, colU, colF, r4cF, pad; };

__global__ void __launch_bounds__(1024) lsa_v2_kernel(const double* __restrict__ cost, int nr0, int nc0,
                                                       int* __restrict__ out_col4row, int* __restrict__ status) {
    __shared__ double s_u[1024], s_vmv[1024];
    __shared__ int s_col4row[1024], s_path[1024], s_r4c[1024], s_vrow[1024];
    __shared__ WarpEntry s_ent[2][32];
    const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, wid = tid >> 5, nwarps = T >> 5;
    const bool transpose = nc0 < nr0;
    const int nr = transpose ? nc0 : nr0;
    const int nc = transpose ? nr0 : nc0;
    const int j = tid;
    const bool mine = j < nc;
    const size_t sj = transpose ? (size_t)j * nc0 : (size_t)j, si = transpose ? (size_t)1 : (size_t)nc0;
#define COST2(i) (cost[sj + (size_t)(i) * si])
    for (int k = tid; k < nr; k += T) { s_u[k] = 0.0; s_col4row[k] = -1; }
    double v = 0.0;
    int r4c = -1, path = -1;
    double nxt = mine ? COST2(0) : 0.0;
    const unsigned long long KINF = dkey(INFINITY);
    bool infeasible = false;
    __syncthreads();
    for (int cur = 0; cur < nr; ++cur) {
        double spc = INFINITY;
        int pos = mine ? nc - 1 - j : -1;
        bool sc = false;
        int num = nc, i = cur, sink = -1, nvis = 0, par = 0;
        double minVal = 0.0;
        double c_i = nxt;
        if (mine && cur + 1 < nr) nxt = COST2(cur + 1);
        while (true) {
            if (tid == 0) { s_vrow[nvis] = i; s_vmv[nvis] = minVal; }
            ++nvis;
            const double ui = s_u[i];
            unsigned long long key = KINF;
            if (pos >= 0) {
                const double r = __dsub_rn(__dsub_rn(__dadd_rn(minVal, c_i), ui), v);
                if (r < spc) { spc = r; path = i; }
                key = dkey(spc + 0.0);          // -0.0 and +0.0 compare equal in SciPy's '<'; give them one key
            }
            // warp minimum of the 64-bit order-preserving keys
            const unsigned hi = (unsigned)(key >> 32);
            const unsigned mhi = __reduce_min_sync(0xffffffffu, hi);
            const unsigned lo = hi == mhi ? (unsigned)key : 0xffffffffu;
            const unsigned mlo = __reduce_min_sync(0xffffffffu, lo);
            const unsigned long long wkey = ((unsigned long long)mhi << 32) | mlo;
            const bool tie = pos >= 0 && key == wkey;
            const int posU = __reduce_max_sync(0xffffffffu, (tie && r4c == -1) ? pos : -1);
            const int posF = __reduce_min_sync(0xffffffffu, tie ? pos : 0x7fffffff);
            WarpEntry& e = s_ent[par][wid];
            if (lane == 0) { e.key = wkey; e.posU = posU; e.posF = posF; }
            if (tie && pos == posU) e.colU = j;
            if (tie && pos == posF) { e.colF = j; e.r4cF = r4c; }
            __syncthreads();
            unsigned long long gkey = KINF;
            for (int w = 0; w < nwarps; ++w) gkey = min(gkey, s_ent[par][w].key);
            if (gkey == KINF) { infeasible = true; break; }
            int bestU = -1, colU = -1, bestF = 0x7fffffff, colF = -1, r4cF = -1;
            for (int w = 0; w < nwarps; ++w) {
                const WarpEntry& q = s_ent[par][w];
                if (q.key != gkey) continue;
                if (q.posU > bestU) { bestU = q.posU; colU = q.colU; }
                if (q.posF < bestF) { bestF = q.posF; colF = q.colF; r4cF = q.r4cF; }
            }
            const int idx = bestU >= 0 ? bestU : bestF;
            const int jsel = bestU >= 0 ? colU : colF;
            const int rsel = bestU >= 0 ? -1 : r4cF;
            // minVal = the winning spc (decode the key back to the double)
            minVal = __longlong_as_double((long long)((gkey >> 63) ? (gkey & 0x7fffffffffffffffull) : ~gkey));
            if (j == jsel) { sc = true; pos = -1; }
            else if (pos == num - 1) pos = idx;
            --num;
            if (rsel == -1) { sink = jsel; break; }
            i = rsel;
            if (pos >= 0) c_i = COST2(i);
            par ^= 1;
        }
        if (infeasible) break;
        // dual updates (SciPy: u[cur] += minVal; u[r] += minVal - spc[col4row[r]] for visited r; v[j] -= minVal - spc[j])
        if (tid == 0) s_u[cur] = __dadd_rn(s_u[cur], minVal);
        if (tid >= 1 && tid < nvis) {
            const int r = s_vrow[tid];
            s_u[r] = __dadd_rn(s_u[r], __dsub_rn(minVal, s_vmv[tid]));
        }
        if (sc) v = __dsub_rn(v, __dsub_rn(minVal, spc));
        if (mine) { s_path[j] = path; s_r4c[j] = r4c; }
        __syncthreads();
        if (tid == 0) {
            int jj = sink;
            while (true) {
                const int ii = s_path[jj];
                s_r4c[jj] = ii;
                const int tmp = s_col4row[ii];
                s_col4row[ii] = jj;
                jj = tmp;
                if (ii == cur) break;
            }
        }
        __syncthreads();
        if (mine) r4c = s_r4c[j];
    }
    if (infeasible) {
        if (tid == 0) status[0] = 1;
        for (int k = tid; k < nr0; k += T) out_col4row[k] = -1;
        return;
    }
    if (tid == 0) status[0] = 0;
    __syncthreads();
    for (int k = tid; k < nr0; k += T) {
        int c = transpose ? s_r4c[k] : s_col4row[k];
        if (c >= 0 && cost[(size_t)k * nc0 + c] >= FM_INF_COST) c = -2 - c;
        out_col4row[k] = c;
    }
#undef COST2
}


// -----------------------------------------------------------------------------------------------------------------
// Version 3 (columns <= 256): ONE warp, K columns per lane, every per-column quantity in registers, no barrier at
// all: a step is K reduced-cost updates per lane, two redux.sync for the 64-bit minimum, two for the tie positions,
// a ballot to find the owner of the selected column.  Same SciPy replay as above (positions in `remaining`,
// swap-with-last, tie rule, fp64 operation order) -> bit-exact.  The walk along the augmenting path is done by
// lane 0 from the (column, path) pairs recorded at every selection.
// -----------------------------------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(32) lsa_warp_kernel(const double* __restrict__ cost, int nr0, int nc0,
                                                       int* __restrict__ out_col4row, int* __restrict__ status) {
    __shared__ lsa::LsaWarpSmem sm;
    lsa::lsa_warp_solve<K>(cost, nr0, nc0, out_col4row, status, sm);
}

}  // namespace

int fm_launch_lsa_block(const double* cost, int nr, int nc, int* col4row, int* status, unsigned char* ws, int use_smem,
                        size_t smem_bytes, cudaStream_t s) {
    const int big = nr > nc ? nr : nc;
    if (big <= 256) {
        if (big <= 32) lsa_warp_kernel<1><<<1, 32, 0, s>>>(cost, nr, nc, col4row, status);
        else if (big <= 64) lsa_warp_kernel<2><<<1, 32, 0, s>>>(cost, nr, nc, col4row, status);
        else if (big <= 128) lsa_warp_kernel<4><<<1, 32, 0, s>>>(cost, nr, nc, col4row, status);
        else lsa_warp_kernel<8><<<1, 32, 0, s>>>(cost, nr, nc, col4row, status);
        return 0;
    }
    if (big <= 1024) {
        int t2 = 64;
        while (t2 < big) t2 <<= 1;
        lsa_v2_kernel<<<1, t2, 0, s>>>(cost, nr, nc, col4row, status);
        return 0;
    }
    int threads = 64;
    while (threads < big && threads < 1024) threads <<= 1;
    lsa_block_kernel<<<1, threads, use_smem ? smem_bytes : 0, s>>>(cost, nr, nc, col4row, status, ws, use_smem);
    return 0;
}
