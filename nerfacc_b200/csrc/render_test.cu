// render_test.cu -- early-terminated test-time rendering (OccGridEstimator.render_test).
//
// The test-mode loop of nerfacc's examples (examples/utils.py:267-439) marches every live ray a few samples at a
// time, shades those samples, composites them onto the running per-ray result with prefix_trans = 1 - opacity and
// retires a ray once it is opaque or has left the grid.  One round here is:
//
//   rt_march_kernel      1 thread / live ray (ray order), the walk of march_generic.cuh with the step limit of the
//                        round into fixed-stride sample slots (SampleSink); n_samples of the round computed on the
//                        device from the previous round's n_alive; each ray's terminate plane becomes its next near
//                        plane; every slot's sample offset inside its tile and, in the last CTA, the tile bases and
//                        {n_alive, n_samples, samples, kept samples so far} to a pinned slot: the round's one host wait
//   rt_expand_kernel     fixed-stride slots -> packed (ray_indices, t_starts, t_ends) in ray order, the arrays the
//                        field closure gets
//   rt_composite_kernel  a warp per live ray, a lane per 4 consecutive samples (the layout and arithmetic of
//                        composite.cu): T = (1 - opacity) exp(-prefix), alpha, w, the alpha_thre mask, the colour /
//                        opacity / depth sums added into the running outputs (no atomics), the ray's live flag, its
//                        rank among the CTA's live rays and, in the last CTA, the CTA bases and the next n_alive
//   rt_scatter_kernel    the live rays -> the next round's ray list (ray order kept)
//
// plus rt_init_kernel before the first round and rt_finish_kernel (background blend, depth normalisation) after the
// last.  See DESIGN.md section 4.11.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/nerfacc_b200.h"
#include "march_generic.cuh"
#include "occ_pack.cuh"
#include "sm_count.cuh"

namespace nfa {

namespace {

constexpr int kMarchTile = 128;     // live-ray slots per march CTA
constexpr int kCompWarps = 8;       // warps per composite CTA ...
constexpr int kCompRays = 32;       // ... each compositing this many live rays in turn
constexpr int kCompTile = kCompWarps * kCompRays;
constexpr int kMaxSamplesPerRound = 64;  // examples/utils.py:352
constexpr unsigned kFull = 0xffffffffu;
constexpr float kEpsF32 = 1.1920929e-07f;  // torch.finfo(float32).eps (examples/utils.py:432)

// Workspace layout (offsets 16-byte aligned), for R rays and at most min_samples * R samples per round:
//   header (64 B): u32 march_done, u32 comp_done, i32 n_alive (of the next march), u32 pad, u64 kept samples
//   lists [2][R] i32      live rays of the even / odd rounds, ascending
//   near [R] f32          every ray's near plane (the previous round's terminate plane)
//   cnt [R] u32           samples of live slot i in this round
//   loc [R] u32           samples of the earlier slots of its march tile
//   rank [R] i32          rank of slot i among the live rays of its composite CTA after this round, -1: retired
//   tile_sum [T] u32, tile_base [T] u64      march tiles (T = ceil(R / kMarchTile))
//   comp_sum [C] u32, comp_base [C] u64      composite CTAs (C = ceil(R / kCompTile))
//   slot_ts [cap] f32, slot_te [cap] f32     fixed-stride samples, cap = min_samples * R
struct RtWs {
    uint32_t* march_done;
    uint32_t* comp_done;
    int32_t* n_alive;
    unsigned long long* kept;
    int32_t* lists;
    float* near;
    uint32_t* cnt;
    uint32_t* loc;
    int32_t* rank;
    uint32_t* tile_sum;
    unsigned long long* tile_base;
    uint32_t* comp_sum;
    unsigned long long* comp_base;
    float* slot_ts;
    float* slot_te;
    int32_t n_rays;
};

inline int64_t align16(int64_t x) { return (x + 15) & ~(int64_t)15; }

inline int64_t rt_ws_bytes(int32_t R, int32_t min_samples, RtWs* w, char* base)
{
    const int64_t T = (R + kMarchTile - 1) / kMarchTile, C = (R + kCompTile - 1) / kCompTile;
    const int64_t cap = (int64_t)min_samples * R;
    int64_t at = 64;
    auto take = [&](int64_t bytes) {
        char* p = base ? base + at : nullptr;
        at += align16(bytes);
        return p;
    };
    char* lists = take(8 * (int64_t)R);
    char* near = take(4 * (int64_t)R);
    char* cnt = take(4 * (int64_t)R);
    char* loc = take(4 * (int64_t)R);
    char* rank = take(4 * (int64_t)R);
    char* tile_sum = take(4 * T);
    char* tile_base = take(8 * T);
    char* comp_sum = take(4 * C);
    char* comp_base = take(8 * C);
    char* slot_ts = take(4 * cap);
    char* slot_te = take(4 * cap);
    if (w) {
        w->march_done = (uint32_t*)base;
        w->comp_done = (uint32_t*)(base + 4);
        w->n_alive = (int32_t*)(base + 8);
        w->kept = (unsigned long long*)(base + 16);
        w->lists = (int32_t*)lists;
        w->near = (float*)near;
        w->cnt = (uint32_t*)cnt;
        w->loc = (uint32_t*)loc;
        w->rank = (int32_t*)rank;
        w->tile_sum = (uint32_t*)tile_sum;
        w->tile_base = (unsigned long long*)tile_base;
        w->comp_sum = (uint32_t*)comp_sum;
        w->comp_base = (unsigned long long*)comp_base;
        w->slot_ts = (float*)slot_ts;
        w->slot_te = (float*)slot_te;
        w->n_rays = R;
    }
    return at;
}

inline RtWs rt_ws_view(void* base, int32_t R, int32_t min_samples)
{
    RtWs w;
    rt_ws_bytes(R, min_samples, &w, (char*)base);
    return w;
}

// n_samples of a round (examples/utils.py:352): max(min(R // n_alive, 64), min_samples)
__device__ __forceinline__ int32_t round_samples(int32_t R, int32_t n_alive, int32_t min_samples)
{
    return n_alive > 0 ? max(min(R / n_alive, kMaxSamplesPerRound), min_samples) : 0;
}

// ---------------------------------------------------------------------------
// two-level scan: a CTA-wide exclusive scan, the CTA sums, and the exclusive scan of the sums in the last CTA
// ---------------------------------------------------------------------------
// Exclusive prefix of v over the CTA's threads (in thread order); `total` gets the CTA's sum in every thread.
__device__ __forceinline__ uint32_t cta_exclusive_scan(uint32_t v, uint32_t& total)
{
    __shared__ uint32_t s_warp[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        const uint32_t y = __shfl_up_sync(kFull, x, s);
        if (lane >= s) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t before = x - v;
    total = 0;
    for (int k = 0; k < n_warps; ++k) {
        const uint32_t s = s_warp[k];
        if (k < warp) before += s;
        total += s;
    }
    __syncthreads();  // s_warp is free again
    return before;
}

// Store this CTA's sum; true in every thread of the last CTA to get here (it then runs tile_bases).
__device__ __forceinline__ bool tile_arrive(uint32_t sum, uint32_t* sums, uint32_t* done)
{
    __shared__ bool s_last;
    if (threadIdx.x == 0) {
        sums[blockIdx.x] = sum;
        __threadfence();
        s_last = atomicAdd(done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    return s_last;
}

// Last CTA only: bases[i] = sums[0] + ... + sums[i - 1] for the n tiles (a contiguous chunk per thread); returns the
// grand total in every thread and leaves *done zero for the next launch.
__device__ __forceinline__ unsigned long long tile_bases(const uint32_t* sums, unsigned long long* bases, int n,
                                                         uint32_t* done)
{
    __shared__ unsigned long long s_warp[32];
    __threadfence();
    const int T = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = T >> 5;
    const int chunk = (n + T - 1) / T;
    const int i0 = min(tid * chunk, n), i1 = min(i0 + chunk, n);
    unsigned long long a = 0;
    for (int i = i0; i < i1; ++i) a += *(const volatile uint32_t*)&sums[i];
    unsigned long long x = a;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        const unsigned long long y = __shfl_up_sync(kFull, x, s);
        if (lane >= s) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    unsigned long long base = x - a, total = 0;
    for (int k = 0; k < n_warps; ++k) {
        if (k < warp) base += s_warp[k];
        total += s_warp[k];
    }
    for (int i = i0; i < i1; ++i) {
        bases[i] = base;
        base += *(const volatile uint32_t*)&sums[i];
    }
    if (tid == 0) *done = 0u;
    return total;
}

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rt_init_kernel(RtWs ws, float near_plane)
{
    const int R = ws.n_rays;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < R; r += gridDim.x * blockDim.x) {
        ws.lists[r] = r;  // round 0: every ray, in order
        ws.near[r] = near_plane;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        *ws.n_alive = R;
        *ws.kept = 0ull;
    }
}

struct RtMarchParams {
    RtWs ws;
    int32_t round;
    const float* rays_o;
    const float* rays_d;
    float far_plane;
    OccGeom g;
    const uint64_t* words;
    const uint32_t* coarse;
    const float* aabbs;
    const float* t_sorted;
    const int64_t* t_indices;
    const uint8_t* hits;
    float step_size, cone_angle;
    int32_t min_samples;
    int64_t* status_host;  // pinned [4]
};

// Grid: every slot a ray can have (R), so that the launch does not depend on n_alive, which only the device knows.
__global__ void __launch_bounds__(kMarchTile) rt_march_kernel(const RtMarchParams p)
{
    const RtWs& ws = p.ws;
    const int R = ws.n_rays;
    const int32_t n_alive = *(const volatile int32_t*)ws.n_alive;
    const int32_t ns = round_samples(R, n_alive, p.min_samples);
    const int i = blockIdx.x * kMarchTile + threadIdx.x;
    uint32_t n = 0;
    if (i < n_alive) {
        const int r = ws.lists[(int64_t)(p.round & 1) * R + i];
        OccView occ;
        occ.words = p.words;
        occ.coarse = p.coarse;
        occ.bounds = nullptr;
        occ.g = p.g;
        SampleSink out;
        out.t_starts = ws.slot_ts;
        out.t_ends = ws.slot_te;
        out.base = (int64_t)i * ns;
        out.n_samples = 0;
        const int G = p.g.n_grids;
        const SortedBoxes boxes{p.aabbs, G, p.t_sorted + (int64_t)r * 2 * G, p.t_indices + (int64_t)r * 2 * G,
                                p.hits + (int64_t)r * G};
        const float o[3] = {p.rays_o[3 * (int64_t)r], p.rays_o[3 * (int64_t)r + 1], p.rays_o[3 * (int64_t)r + 2]};
        const float d[3] = {p.rays_d[3 * (int64_t)r], p.rays_d[3 * (int64_t)r + 1], p.rays_d[3 * (int64_t)r + 2]};
        ws.near[r] = generic_march_ray(boxes, occ, o, d, ws.near[r], p.far_plane, p.step_size, p.cone_angle, ns, out);
        n = (uint32_t)out.n_samples;
        ws.cnt[i] = n;
    }
    uint32_t tile_total;
    const uint32_t before = cta_exclusive_scan(n, tile_total);
    if (i < n_alive) ws.loc[i] = before;
    if (!tile_arrive(tile_total, ws.tile_sum, ws.march_done)) return;
    const unsigned long long total = tile_bases(ws.tile_sum, ws.tile_base, gridDim.x, ws.march_done);
    if (threadIdx.x == 0) {
        // read by the host after it has waited for this kernel
        p.status_host[0] = n_alive;
        p.status_host[1] = ns;
        p.status_host[2] = (int64_t)total;
        p.status_host[3] = (int64_t)*(const volatile unsigned long long*)ws.kept;
    }
}

__device__ __forceinline__ int64_t slot_start(const RtWs& ws, int i)
{
    return (int64_t)ws.tile_base[i / kMarchTile] + ws.loc[i];
}

// Thread per fixed-stride slot element (coalesced reads); slot i's samples land at its packed offset.
__global__ void __launch_bounds__(256) rt_expand_kernel(RtWs ws, int32_t round, int32_t n_alive, int32_t ns,
                                                        int64_t* __restrict__ ray_indices, float* __restrict__ t_starts,
                                                        float* __restrict__ t_ends)
{
    const int64_t n_slots = (int64_t)n_alive * ns;
    const int32_t* list = ws.lists + (int64_t)(round & 1) * ws.n_rays;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_slots;
         e += (int64_t)gridDim.x * blockDim.x) {
        const int i = (int)(e / ns);
        const uint32_t j = (uint32_t)(e - (int64_t)i * ns);
        if (j >= ws.cnt[i]) continue;
        const int64_t k = slot_start(ws, i) + j;
        ray_indices[k] = list[i];
        t_starts[k] = ws.slot_ts[e];
        t_ends[k] = ws.slot_te[e];
    }
}

struct RtCompositeParams {
    RtWs ws;
    int32_t round, n_alive, ns;
    int64_t n_total;
    const float* t_starts;
    const float* t_ends;
    const float* rgbs;    // [n_total, 3]
    const float* sigmas;  // [n_total]
    float alpha_thre;
    float opc_thre;       // a ray stays alive while its opacity <= this (1 - early_stop_eps)
    float* colors;        // [R, 3], running
    float* opacities;     // [R], running
    float* depths;        // [R], running (un-normalised)
};

__device__ __forceinline__ float exp_neg(float x) { return __expf(-x); }  // as composite.cu

// CTA b composites live slots [b * kCompTile, (b + 1) * kCompTile): warp w the kCompRays slots from
// b * kCompTile + w * kCompRays, one after the other.  A ray has at most 64 samples in a round, so one pass of 32
// lanes x 4 samples covers it; the 4-sample groups are aligned to the packed array, as composite.cu aligns them,
// so that T, alpha and w carry the same bits as render_weight_from_density(prefix_trans=...) on the same samples.
__global__ void __launch_bounds__(kCompWarps * 32) rt_composite_kernel(const RtCompositeParams p)
{
    const RtWs& ws = p.ws;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int R = ws.n_rays;
    const int32_t* list = ws.lists + (int64_t)(p.round & 1) * R;
    const int slot0 = blockIdx.x * kCompTile + warp * kCompRays;
    uint32_t my_live = 0;  // lane j: slot slot0 + j stays alive
    unsigned long long kept = 0;
    for (int j = 0; j < kCompRays; ++j) {
        const int i = slot0 + j;
        if (i >= p.n_alive) break;
        const int r = list[i];
        const int64_t start = slot_start(ws, i);
        const uint32_t cnt = ws.cnt[i];
        const int64_t end = start + cnt;
        const float op0 = p.opacities[r];
        const float pt = 1.0f - op0;  // prefix_trans (examples/utils.py:390)
        float op1 = op0, aD = 0.f, aC0 = 0.f, aC1 = 0.f, aC2 = 0.f;
        uint32_t n_kept = 0;
        if (cnt > 0) {
            const int64_t g = (start >> 2) + lane;  // this lane's group: samples 4g .. 4g + 3
            float ts[4], te[4], sg[4], c[12], x[4], incl[4];
            bool ok[4];
            float run = 0.f;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int64_t k = 4 * g + e;
                ok[e] = k >= start && k < end;
                ts[e] = te[e] = sg[e] = 0.f;
                c[3 * e] = c[3 * e + 1] = c[3 * e + 2] = 0.f;
                if (ok[e]) {
                    ts[e] = __ldg(p.t_starts + k);
                    te[e] = __ldg(p.t_ends + k);
                    sg[e] = __ldg(p.sigmas + k);
                    c[3 * e] = __ldg(p.rgbs + 3 * k);
                    c[3 * e + 1] = __ldg(p.rgbs + 3 * k + 1);
                    c[3 * e + 2] = __ldg(p.rgbs + 3 * k + 2);
                }
                // reference volrend.py:271-277 (render_weight_from_density)
                x[e] = ok[e] ? sg[e] * (te[e] - ts[e]) : 0.f;
                run += x[e];
                incl[e] = run;
            }
            float tot = run;
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const float y = __shfl_up_sync(kFull, tot, s);
                if (lane >= s) tot += y;
            }
            const float off = 0.0f + (tot - run);
            float wks[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float T = exp_neg(off + (incl[e] - x[e])) * pt;
                const float a = 1.0f - exp_neg(x[e]);
                const float w = T * a;
                // alpha_thre drops samples from the sums only, not from the transmittance (examples/utils.py:392-400)
                const bool keep = ok[e] && (!(p.alpha_thre > 0.0f) || a >= p.alpha_thre);
                const float wk = keep ? w : 0.f;
                wks[e] = wk;
                n_kept += keep ? 1u : 0u;
                aD += wk * ((ts[e] + te[e]) * 0.5f);
                aC0 += wk * c[3 * e];
                aC1 += wk * c[3 * e + 1];
                aC2 += wk * c[3 * e + 2];
            }
            // The opacity decides whether the ray stays live, so it is summed as accumulate_along_rays_ adds into it:
            // one weight after the other onto the running value, in sample order (lane by lane, 4 samples each).
            const int n_lanes = (int)(((end - 1) >> 2) - (start >> 2)) + 1;
            for (int l = 0; l < n_lanes; ++l) {
#pragma unroll
                for (int e = 0; e < 4; ++e) op1 = op1 + __shfl_sync(kFull, wks[e], l);
            }
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) {
                aD += __shfl_xor_sync(kFull, aD, s);
                aC0 += __shfl_xor_sync(kFull, aC0, s);
                aC1 += __shfl_xor_sync(kFull, aC1, s);
                aC2 += __shfl_xor_sync(kFull, aC2, s);
                n_kept += __shfl_xor_sync(kFull, n_kept, s);
            }
        }
        if (lane == 0 && cnt > 0) {
            p.opacities[r] = op1;
            p.depths[r] += aD;
            p.colors[3 * (int64_t)r] += aC0;
            p.colors[3 * (int64_t)r + 1] += aC1;
            p.colors[3 * (int64_t)r + 2] += aC2;
        }
        kept += n_kept;
        // examples/utils.py:423-428: not opaque yet, and the round's step limit was what stopped the ray
        if (lane == j && op1 <= p.opc_thre && cnt == (uint32_t)p.ns) my_live = 1u;
    }
    if (lane == 0 && kept) atomicAdd(ws.kept, kept);
    uint32_t cta_live;
    const uint32_t before = cta_exclusive_scan(my_live, cta_live);
    const int i = slot0 + lane;
    if (i < p.n_alive) ws.rank[i] = my_live ? (int32_t)before : -1;
    if (!tile_arrive(cta_live, ws.comp_sum, ws.comp_done)) return;
    const unsigned long long n_next = tile_bases(ws.comp_sum, ws.comp_base, gridDim.x, ws.comp_done);
    if (threadIdx.x == 0) *ws.n_alive = (int32_t)n_next;
}

// Live slot i of this round -> slot comp_base[CTA] + rank of the next round's list.
__global__ void __launch_bounds__(256) rt_scatter_kernel(RtWs ws, int32_t round, int32_t n_alive)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_alive) return;
    const int32_t k = ws.rank[i];
    if (k < 0) return;
    const int64_t R = ws.n_rays;
    ws.lists[(int64_t)((round + 1) & 1) * R + (int64_t)ws.comp_base[i / kCompTile] + k] =
        ws.lists[(int64_t)(round & 1) * R + i];
}

// examples/utils.py:431-432
__global__ void __launch_bounds__(256) rt_finish_kernel(RtWs ws, const float* bkgd, float* colors,
                                                        const float* opacities, float* depths, int64_t* status_host)
{
    const int R = ws.n_rays;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < R; r += gridDim.x * blockDim.x) {
        const float op = opacities[r];
        if (bkgd) {
            const float k = 1.0f - op;
            colors[3 * (int64_t)r] += bkgd[0] * k;
            colors[3 * (int64_t)r + 1] += bkgd[1] * k;
            colors[3 * (int64_t)r + 2] += bkgd[2] * k;
        }
        depths[r] = depths[r] / fmaxf(op, kEpsF32);
    }
    if (status_host && blockIdx.x == 0 && threadIdx.x == 0) status_host[3] = (int64_t)*ws.kept;
}

inline int grid_for(int64_t threads, int threads_per_cta)
{
    const int64_t ctas = (threads + threads_per_cta - 1) / threads_per_cta;
    const int64_t cap = (int64_t)kNumSMs * 8;
    return (int)(ctas < 1 ? 1 : (ctas < cap ? ctas : cap));
}

inline int32_t launch_status()
{
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? NFA_OK : (int32_t)e;
}

}  // namespace

}  // namespace nfa

using namespace nfa;

extern "C" {

int64_t nfa_render_test_workspace_bytes(int32_t n_rays, int32_t min_samples)
{
    if (n_rays < 0 || min_samples < 1) return 0;
    return rt_ws_bytes(n_rays, min_samples, nullptr, nullptr);
}

int32_t nfa_render_test_begin(int32_t n_rays, int32_t min_samples, float near_plane, void* workspace,
                              nfa_stream_t stream)
{
    if (n_rays < 0 || min_samples < 1) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!workspace || (((uintptr_t)workspace) & 15u) != 0) return NFA_ERR_ARG;
    rt_init_kernel<<<grid_for(n_rays, 256), 256, 0, (cudaStream_t)stream>>>(
        rt_ws_view(workspace, n_rays, min_samples), near_plane);
    return launch_status();
}

int32_t nfa_render_test_march(int32_t n_rays, int32_t min_samples, int32_t round, const float* rays_o,
                              const float* rays_d, float far_plane, int32_t n_grids, int32_t rx, int32_t ry, int32_t rz,
                              const uint64_t* words, const uint32_t* coarse, const float* aabbs, const float* t_sorted,
                              const int64_t* t_indices, const uint8_t* hits, float step_size, float cone_angle,
                              void* workspace, int64_t* status_host, nfa_stream_t stream)
{
    // !(cone_angle >= 0): negative or NaN
    if (n_rays <= 0 || min_samples < 1 || round < 0 || n_grids <= 0 || rx <= 0 || ry <= 0 || rz <= 0 ||
        !(cone_angle >= 0.0f))
        return NFA_ERR_ARG;
    if (!(step_size > 0.0f)) return NFA_ERR_UNSUPPORTED;  // one sample per cell: no step limit per round fits
    if (!rays_o || !rays_d || !words || !coarse || !aabbs || !t_sorted || !t_indices || !hits || !workspace ||
        !status_host || (((uintptr_t)workspace) & 15u) != 0)
        return NFA_ERR_ARG;
    RtMarchParams p;
    p.ws = rt_ws_view(workspace, n_rays, min_samples);
    p.round = round;
    p.rays_o = rays_o;
    p.rays_d = rays_d;
    p.far_plane = far_plane;
    p.g = occ_geom(n_grids, rx, ry, rz);
    p.words = words;
    p.coarse = coarse;
    p.aabbs = aabbs;
    p.t_sorted = t_sorted;
    p.t_indices = t_indices;
    p.hits = hits;
    p.step_size = step_size;
    p.cone_angle = cone_angle;
    p.min_samples = min_samples;
    p.status_host = status_host;
    rt_march_kernel<<<(n_rays + kMarchTile - 1) / kMarchTile, kMarchTile, 0, (cudaStream_t)stream>>>(p);
    return launch_status();
}

int32_t nfa_render_test_expand(int32_t n_rays, int32_t min_samples, int32_t round, int32_t n_alive, int32_t n_samples,
                               const void* workspace, int64_t* ray_indices, float* t_starts, float* t_ends,
                               nfa_stream_t stream)
{
    if (n_rays <= 0 || min_samples < 1 || round < 0 || n_alive < 0 || n_alive > n_rays || n_samples < 0 ||
        (int64_t)n_alive * n_samples > (int64_t)min_samples * n_rays)
        return NFA_ERR_ARG;
    if (!workspace) return NFA_ERR_ARG;
    const int64_t n_slots = (int64_t)n_alive * n_samples;
    if (n_slots == 0) return NFA_OK;
    if (!ray_indices || !t_starts || !t_ends) return NFA_ERR_ARG;
    rt_expand_kernel<<<grid_for(n_slots, 256), 256, 0, (cudaStream_t)stream>>>(
        rt_ws_view(const_cast<void*>(workspace), n_rays, min_samples), round, n_alive, n_samples, ray_indices,
        t_starts, t_ends);
    return launch_status();
}

int32_t nfa_render_test_composite(int32_t n_rays, int32_t min_samples, int32_t round, int32_t n_alive,
                                  int32_t n_samples, int64_t n_total, void* workspace, const float* t_starts,
                                  const float* t_ends, const float* rgbs, const float* sigmas, float alpha_thre,
                                  float opacity_thre, float* colors, float* opacities, float* depths,
                                  nfa_stream_t stream)
{
    if (n_rays <= 0 || min_samples < 1 || round < 0 || n_alive <= 0 || n_alive > n_rays || n_samples < 1 ||
        n_samples > kMaxSamplesPerRound || n_total < 0 || n_total > (int64_t)n_alive * n_samples)
        return NFA_ERR_ARG;
    if (!workspace || !colors || !opacities || !depths) return NFA_ERR_ARG;
    if (n_total > 0 && (!t_starts || !t_ends || !rgbs || !sigmas)) return NFA_ERR_ARG;
    RtCompositeParams p;
    p.ws = rt_ws_view(workspace, n_rays, min_samples);
    p.round = round;
    p.n_alive = n_alive;
    p.ns = n_samples;
    p.n_total = n_total;
    p.t_starts = t_starts;
    p.t_ends = t_ends;
    p.rgbs = rgbs;
    p.sigmas = sigmas;
    p.alpha_thre = alpha_thre;
    p.opc_thre = opacity_thre;
    p.colors = colors;
    p.opacities = opacities;
    p.depths = depths;
    const cudaStream_t s = (cudaStream_t)stream;
    rt_composite_kernel<<<(n_alive + kCompTile - 1) / kCompTile, kCompWarps * 32, 0, s>>>(p);
    rt_scatter_kernel<<<(n_alive + 255) / 256, 256, 0, s>>>(p.ws, round, n_alive);
    return launch_status();
}

int32_t nfa_render_test_finish(int32_t n_rays, int32_t min_samples, const void* workspace, const float* bkgd,
                               float* colors, const float* opacities, float* depths, int64_t* status_host,
                               nfa_stream_t stream)
{
    if (n_rays < 0 || min_samples < 1) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!workspace || !colors || !opacities || !depths) return NFA_ERR_ARG;
    rt_finish_kernel<<<grid_for(n_rays, 256), 256, 0, (cudaStream_t)stream>>>(
        rt_ws_view(const_cast<void*>(workspace), n_rays, min_samples), bkgd, colors, opacities, depths, status_host);
    return launch_status();
}

}  // extern "C"
