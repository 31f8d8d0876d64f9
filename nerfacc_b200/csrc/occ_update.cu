// occ_update.cu -- occupancy-grid maintenance (SURVEY 8 row f4): the step on the producer side of the path.
//
// Reference: OccGridEstimator._update (/root/reference/nerfacc/estimators/occ_grid.py:367-404)
//     occs[ids]  = maximum(occs[ids] * ema_decay, occ)                         (:395-398)
//     thre       = clamp(occs[occs >= 0].mean(), max=occ_thre)                 (:400-402)
//     binaries   = (occs > thre).view(levels, rx, ry, rz)                      (:403-404)
// there: a gather, a multiply, a maximum, an index_put, a boolean mask-select (which synchronises), a mean, a
// clamp, a compare -- and then, on the next sampling() call, a re-pack of the bool grid.  Here:
//
//   occ_ema_gather_kernel / occ_ema_scatter_kernel   the EMA-max at the sampled cells.  Two passes because the
//                     cell list may name a cell twice (uniform + occupied draws): every draw must see the OLD
//                     value, then the largest result wins (one of the outcomes index_put may produce, and the
//                     only deterministic one).
//   occ_mean_kernel   sum (f64) and count of the visible cells (occs >= 0), fixed-order two-level reduction; the
//                     last CTA folds the partials and writes the threshold -- no host round trip.
//   occ_threshold_pack_kernel   one pass over occs: writes the bool grid the estimator keeps (state_dict
//                     compatibility) AND the traversal's brick words, class mip and occupied-brick bounds, so the
//                     next sampling() finds its derived cache ready (no nfa_occ_pack).
//
// HBM-bound byte work: 4 B/cell read + 1 B/cell written (+ 1/8 B of brick words); no tensor cores.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/nerfacc_b200.h"
#include "sm_count.cuh"
#include "occ_pack.cuh"

namespace nfa {

constexpr int kUpdThreads = 256;

// torch.maximum: NaN if either operand is NaN
__device__ __forceinline__ float max_nan(float a, float b) { return (a != a || b != b) ? NAN : fmaxf(a, b); }

__global__ void __launch_bounds__(kUpdThreads) occ_ema_gather_kernel(int64_t n, const int64_t* __restrict__ ids,
                                                                     const float* __restrict__ occ, float decay,
                                                                     const float* __restrict__ occs,
                                                                     float* __restrict__ fresh)
{
    for (int64_t i = (int64_t)blockIdx.x * kUpdThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kUpdThreads)
        fresh[i] = max_nan(__fmul_rn(occs[ids[i]], decay), occ[i]);
}

// float max through integer atomics: floats with a clear sign bit order like signed ints, those with the sign bit
// set like reversed unsigned ints.  The path is chosen by the sign bit, not by `v >= 0`: -0.0 compares equal to
// +0.0 but its bits are INT_MIN, which the signed max would never prefer to the -INFINITY the reset left.  So the
// draws reduce in the total order -inf < ... < -0.0 < +0.0 < ... < +inf.  A NaN is stored as is (and stays: the
// integer compare below never replaces it by a number that is not also the result of some draw).
__device__ __forceinline__ void atomic_max_float(float* addr, float v)
{
    if (v != v) {
        *addr = v;
        return;
    }
    if (__float_as_int(v) >= 0) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

__global__ void __launch_bounds__(kUpdThreads) occ_ema_reset_kernel(int64_t n, const int64_t* __restrict__ ids,
                                                                    float* __restrict__ occs)
{
    // every draw of a cell resets it to the smallest float so that the max below sees only fresh values
    for (int64_t i = (int64_t)blockIdx.x * kUpdThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kUpdThreads)
        occs[ids[i]] = -INFINITY;
}

__global__ void __launch_bounds__(kUpdThreads) occ_ema_scatter_kernel(int64_t n, const int64_t* __restrict__ ids,
                                                                      const float* __restrict__ fresh,
                                                                      float* __restrict__ occs)
{
    for (int64_t i = (int64_t)blockIdx.x * kUpdThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kUpdThreads)
        atomic_max_float(occs + ids[i], fresh[i]);
}

struct MeanPartial {
    double sum;
    unsigned long long count;
};

// workspace: [0,16) u32 done counter (+pad), [16,32) f32 threshold (+pad), then MeanPartial[grid]
__global__ void __launch_bounds__(kUpdThreads) occ_mean_kernel(int64_t n_cells, const float* __restrict__ occs,
                                                               float occ_thre, unsigned int* __restrict__ done,
                                                               float* __restrict__ thre, MeanPartial* __restrict__ part)
{
    __shared__ double s_sum[kUpdThreads / 32];
    __shared__ unsigned long long s_cnt[kUpdThreads / 32];
    __shared__ bool s_last;
    double sum = 0.0;
    unsigned long long cnt = 0;
    // fixed assignment of cells to threads and a fixed combination order => the same bits on every run
    const int64_t n4 = n_cells >> 2;
    const float4* v4 = reinterpret_cast<const float4*>(occs);
    const bool aligned = (((uintptr_t)occs) & 15u) == 0;
    if (aligned) {
        for (int64_t i = (int64_t)blockIdx.x * kUpdThreads + threadIdx.x; i < n4; i += (int64_t)gridDim.x * kUpdThreads) {
            const float4 v = v4[i];
            if (v.x >= 0.f) { sum += v.x; ++cnt; }
            if (v.y >= 0.f) { sum += v.y; ++cnt; }
            if (v.z >= 0.f) { sum += v.z; ++cnt; }
            if (v.w >= 0.f) { sum += v.w; ++cnt; }
        }
    }
    for (int64_t i = (aligned ? n4 * 4 : 0) + (int64_t)blockIdx.x * kUpdThreads + threadIdx.x; i < n_cells;
         i += (int64_t)gridDim.x * kUpdThreads) {
        const float v = occs[i];
        if (v >= 0.f) { sum += v; ++cnt; }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, s);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, s);
    }
    if ((threadIdx.x & 31) == 0) {
        s_sum[threadIdx.x >> 5] = sum;
        s_cnt[threadIdx.x >> 5] = cnt;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        MeanPartial p = {0.0, 0ull};
        for (int k = 0; k < kUpdThreads / 32; ++k) {
            p.sum += s_sum[k];
            p.count += s_cnt[k];
        }
        part[blockIdx.x] = p;
        __threadfence();
        s_last = atomicAdd(done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last && threadIdx.x == 0) {
        __threadfence();
        double tot = 0.0;
        unsigned long long c = 0;
        for (unsigned int k = 0; k < gridDim.x; ++k) {
            const volatile MeanPartial* q = part + k;
            tot += q->sum;
            c += q->count;
        }
        // mean of an empty selection is NaN in torch, and clamp(NaN, max=..) stays NaN: nothing is occupied then
        const float mean = c ? (float)(tot / (double)c) : NAN;
        *thre = (mean != mean) ? mean : fminf(mean, occ_thre);
        *done = 0u;  // reusable
    }
}

// One CTA per (level, brick x, brick y): 16 rows (4 x-planes * 4 y-rows) of rz floats each, thread z owns column z.
// Four consecutive threads hold the four z cells of a brick; their row bits are OR-ed with two shuffles.
__global__ void __launch_bounds__(kUpdThreads) occ_threshold_pack_kernel(OccGeom g, const float* __restrict__ occs,
                                                                         const float* __restrict__ thre_p,
                                                                         uint8_t* __restrict__ binaries,
                                                                         uint64_t* __restrict__ words,
                                                                         uint32_t* __restrict__ coarse,
                                                                         int32_t* __restrict__ bounds)
{
    const float thre = *thre_p;
    const int level = blockIdx.z, bx = blockIdx.x, by = blockIdx.y;
    const int64_t cells = (int64_t)g.res[0] * g.res[1] * g.res[2];
    const float* lo = occs + level * cells;
    uint8_t* lb = binaries + level * cells;
    const int nzq = (g.res[2] + 3) & ~3;  // columns incl. the padding of the last brick
    for (int zb = 0; zb < nzq; zb += kUpdThreads) {  // every thread takes every turn: the shuffles need whole warps
        const int z = zb + threadIdx.x;
        uint64_t w = 0;
        if (z < g.res[2]) {
#pragma unroll
            for (int dx = 0; dx < 4; ++dx) {
                const int x = bx * 4 + dx;
                if (x >= g.res[0]) break;
#pragma unroll
                for (int dy = 0; dy < 4; ++dy) {
                    const int y = by * 4 + dy;
                    if (y >= g.res[1]) break;
                    const int64_t c = ((int64_t)x * g.res[1] + y) * g.res[2] + z;
                    const bool on = lo[c] > thre;  // NaN threshold / NaN occupancy: false, as in torch
                    lb[c] = on ? 1 : 0;
                    if (on) w |= 1ull << ((dx << 4) | (dy << 2) | (z & 3));
                }
            }
        }
        w |= __shfl_xor_sync(0xffffffffu, w, 1);  // the four z cells of a brick sit in four consecutive lanes
        w |= __shfl_xor_sync(0xffffffffu, w, 2);
        if ((z & 3) == 0 && z < nzq) {
            const int bz = z >> 2;
            const int b = (bx * g.nb[1] + by) * g.nb[2] + bz + level * g.wpl;
            words[b] = w;
            if (w != 0) {
                atomicOr(coarse + (b >> 4), (w == ~0ull ? kBrickFull : kBrickMixed) << ((b & 15) << 1));
                int32_t* bb = bounds + 6 * level;
                atomicMin(bb + 0, bx); atomicMin(bb + 1, by); atomicMin(bb + 2, bz);
                atomicMax(bb + 3, bx); atomicMax(bb + 4, by); atomicMax(bb + 5, bz);
            }
        }
    }
}

__global__ void occ_pack_clear_kernel(uint32_t* coarse, int64_t n_coarse, int32_t* bounds, int n_grids)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_coarse) coarse[i] = 0u;
    if (i < 6 * n_grids) bounds[i] = (i % 6) < 3 ? kBoundsMinInit : kBoundsMaxInit;
}

}  // namespace nfa

using namespace nfa;

static inline int32_t launch_status_u()
{
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? NFA_OK : (int32_t)e;
}

static inline int grid_for(int64_t n, int per_thread)
{
    const int64_t b = (n + (int64_t)kUpdThreads * per_thread - 1) / ((int64_t)kUpdThreads * per_thread);
    return (int)(b < 1 ? 1 : (b < kNumSMs * 8 ? b : kNumSMs * 8));
}

extern "C" {

int32_t nfa_occ_ema_update(int64_t n, const int64_t* cell_ids, const float* occ, float ema_decay, float* occs,
                           float* scratch, nfa_stream_t stream)
{
    if (n < 0) return NFA_ERR_ARG;
    if (n == 0) return NFA_OK;
    if (!cell_ids || !occ || !occs || !scratch) return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    const int blocks = grid_for(n, 4);
    occ_ema_gather_kernel<<<blocks, kUpdThreads, 0, s>>>(n, cell_ids, occ, ema_decay, occs, scratch);
    occ_ema_reset_kernel<<<blocks, kUpdThreads, 0, s>>>(n, cell_ids, occs);
    occ_ema_scatter_kernel<<<blocks, kUpdThreads, 0, s>>>(n, cell_ids, scratch, occs);
    return launch_status_u();
}

static inline int mean_grid(int64_t n_cells) { return grid_for(n_cells, 16); }

int64_t nfa_occ_threshold_workspace_bytes(int64_t n_cells)
{
    return n_cells < 0 ? 0 : 32 + (int64_t)mean_grid(n_cells) * (int64_t)sizeof(MeanPartial);
}

int32_t nfa_occ_threshold_pack(int32_t n_grids, int32_t rx, int32_t ry, int32_t rz, const float* occs, float occ_thre,
                               uint8_t* binaries, uint64_t* words, uint32_t* coarse, int32_t* bounds, void* workspace,
                               nfa_stream_t stream)
{
    if (n_grids <= 0 || rx <= 0 || ry <= 0 || rz <= 0) return NFA_ERR_ARG;
    if (!occs || !binaries || !words || !coarse || !bounds || !workspace) return NFA_ERR_ARG;
    if ((((uintptr_t)workspace) & 15u) != 0) return NFA_ERR_ARG;
    const OccGeom g = occ_geom(n_grids, rx, ry, rz);
    if ((int64_t)n_grids * g.wpl > (int64_t)INT32_MAX || g.nb[1] > 65535 || n_grids > 65535) return NFA_ERR_UNSUPPORTED;
    const int64_t n_cells = (int64_t)n_grids * rx * ry * rz;
    cudaStream_t s = (cudaStream_t)stream;
    unsigned int* done = (unsigned int*)workspace;
    float* thre = (float*)((char*)workspace + 16);
    MeanPartial* part = (MeanPartial*)((char*)workspace + 32);
    const int64_t n_coarse = occ_coarse_words(g);
    const int64_t clr = n_coarse > 6 * n_grids ? n_coarse : 6 * n_grids;
    cudaMemsetAsync(done, 0, 4, s);
    occ_pack_clear_kernel<<<(int)((clr + 255) / 256), 256, 0, s>>>(coarse, n_coarse, bounds, n_grids);
    occ_mean_kernel<<<mean_grid(n_cells), kUpdThreads, 0, s>>>(n_cells, occs, occ_thre, done, thre, part);
    occ_threshold_pack_kernel<<<dim3(g.nb[0], g.nb[1], n_grids), kUpdThreads, 0, s>>>(g, occs, thre, binaries, words,
                                                                                      coarse, bounds);
    return launch_status_u();
}

}  // extern "C"
