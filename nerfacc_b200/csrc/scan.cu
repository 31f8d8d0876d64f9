// scan.cu -- segmented scans over the packed layout, pack_info.
//
// replaces (paths relative to /root/reference):
//   nerfacc/cuda/csrc/scan.cu:9-304 + include/utils_scan.cuh:21-263
//       (packed_info flavour: {in,ex}clusive_{sum,prod}, forward and the
//        reverse-iterator backward launches)
//   nerfacc/cuda/csrc/scan_cub.cu:59-287 (ray-index flavour, CUB DeviceScan::*ByKey)
//   nerfacc/pack.py:38-46 (pack_info = index_add_ + cumsum)
//
// Packed flavour: one warp per ray, shuffle scan per 32-element tile with a
// running carry; no shared memory and no block barriers (the reference's
// Blelloch-in-smem kernel syncs under divergent control flow).
// Key flavour: single pass, tile-local segmented scan + decoupled look-back for
// the value carried into each tile (one tile deep in practice).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/nerfacc_b200.h"
#include "sm_count.cuh"
#include "vis_block.cuh"

namespace nfa {

constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kScanWarps = 8;

template <bool kProd>
__device__ __forceinline__ float op_apply(float a, float b) { return kProd ? a * b : a + b; }
template <bool kProd>
__device__ __forceinline__ float op_identity() { return kProd ? 1.0f : 0.0f; }

// ---------------------------------------------------------------------------
// packed_info flavour
// ---------------------------------------------------------------------------
template <bool kProd, bool kInclusive, bool kReverse>
__global__ void __launch_bounds__(kScanWarps * 32) scan_packed_kernel(int32_t n_rays,
                                                                      const int64_t* __restrict__ packed_info,
                                                                      const float* __restrict__ in,
                                                                      float* __restrict__ out, int32_t normalize)
{
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * kScanWarps + (threadIdx.x >> 5);
    if (r >= n_rays) return;
    const longlong2 pi = *reinterpret_cast<const longlong2*>(packed_info + 2 * (int64_t)r);
    const int64_t start = pi.x, n = pi.y;
    float carry = op_identity<kProd>();
    for (int64_t base = 0; base < n; base += 32) {
        const int64_t j = base + lane;
        const bool valid = j < n;
        const int64_t k = kReverse ? start + n - 1 - j : start + j;
        const float x = valid ? __ldg(in + k) : op_identity<kProd>();
        float incl = x;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            const float y = __shfl_up_sync(kFullMask, incl, s);
            if (lane >= s) incl = op_apply<kProd>(y, incl);
        }
        float res;
        if (kInclusive) {
            res = op_apply<kProd>(carry, incl);
        } else {
            float excl = __shfl_up_sync(kFullMask, incl, 1);
            if (lane == 0) excl = op_identity<kProd>();
            res = op_apply<kProd>(carry, excl);
        }
        if (valid) out[k] = res;
        carry = op_apply<kProd>(carry, __shfl_sync(kFullMask, incl, 31));
    }
    if (normalize) {  // reference utils_scan.cuh:102-109 (forward inclusive sum only)
        const float tot = fmaxf(carry, 1e-10f);
        __syncwarp();
        for (int64_t j = lane; j < n; j += 32) out[start + j] = out[start + j] / tot;
    }
}

// ---------------------------------------------------------------------------
// key (ray index) flavour: a segment is a maximal run of equal consecutive keys.
// ONE pass over the data (the reference: cub::DeviceScan::*ByKey, scan_cub.cu:18-56): every CTA scans a tile of
// 2048 elements and gets the value carried into it by decoupled look-back.  Tiles are claimed through an atomic
// ticket (so a tile's predecessors are always running or done), publish the aggregate of their trailing open
// segment as one 64-bit word (value | has-a-head | status), and look back only until a tile that contains a
// segment head -- with ~130 samples per ray that is the tile right before, so nothing ever waits on a chain.
// ---------------------------------------------------------------------------
constexpr int kKeyThreads = 256;
#ifndef NFA_KEY_ITEMS
#define NFA_KEY_ITEMS 8
#endif
constexpr int kKeyItems = NFA_KEY_ITEMS;  // 4 or 8 consecutive elements per thread
constexpr int kKeyTile = kKeyThreads * kKeyItems;

// tile descriptor: bits 0-31 value, bit 32 "the tile contains a segment head", bits 62-63 status
constexpr unsigned long long kStAggregate = 1ull << 62;  // value = this tile alone (no head in it): keep looking back
constexpr unsigned long long kStPrefix = 2ull << 62;     // value = everything a successor needs: stop here
constexpr unsigned long long kStMask = 3ull << 62;

template <bool kProd>
struct SegPair {
    float v;
    int f;
};
template <bool kProd>
__device__ __forceinline__ SegPair<kProd> seg_combine(SegPair<kProd> a, SegPair<kProd> b)
{
    SegPair<kProd> r;
    r.v = b.f ? b.v : op_apply<kProd>(a.v, b.v);
    r.f = a.f | b.f;
    return r;
}

__device__ __forceinline__ unsigned long long tile_word(float v, int has_head, unsigned long long status)
{
    return (unsigned long long)__float_as_uint(v) | ((unsigned long long)(has_head ? 1 : 0) << 32) | status;
}

// workspace: [0,8) ticket counter, [16, 16 + 8 n_tiles) tile descriptors; zeroed by the launcher
template <bool kProd, bool kInclusive, bool kReverse, bool kVec>
__global__ void __launch_bounds__(kKeyThreads) scan_bykey_kernel(int64_t n, const int64_t* __restrict__ keys,
                                                                 const float* __restrict__ in, float* __restrict__ out,
                                                                 unsigned int* __restrict__ ticket,
                                                                 unsigned long long* __restrict__ desc)
{
    __shared__ float s_v[kKeyThreads / 32];
    __shared__ int s_f[kKeyThreads / 32];
    __shared__ long long s_last_key[kKeyThreads / 32];
    __shared__ int s_first_head;
    __shared__ unsigned int s_tile;
    __shared__ float s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        s_tile = atomicAdd(ticket, 1u);
        s_first_head = kKeyTile;
    }
    __syncthreads();
    const unsigned int tile = s_tile;
    const int64_t tile0 = (int64_t)tile * kKeyTile;
    const int64_t j0 = tile0 + (int64_t)tid * kKeyItems;  // logical index of this thread's first element

    // ---- load 8 consecutive (logical) elements per thread
    float x[kKeyItems];
    long long key[kKeyItems];
    if (kVec && j0 + kKeyItems <= n) {  // forward, 16-byte aligned arrays: two float4 + four longlong2 per thread
#pragma unroll
        for (int q = 0; q < kKeyItems / 4; ++q) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(in + j0) + q);
            x[4 * q] = a.x; x[4 * q + 1] = a.y; x[4 * q + 2] = a.z; x[4 * q + 3] = a.w;
        }
#pragma unroll
        for (int q = 0; q < kKeyItems / 2; ++q) {
            const longlong2 kk = __ldg(reinterpret_cast<const longlong2*>(keys + j0) + q);
            key[2 * q] = kk.x;
            key[2 * q + 1] = kk.y;
        }
    } else {
#pragma unroll
        for (int e = 0; e < kKeyItems; ++e) {
            const int64_t j = j0 + e;
            const int64_t k = kReverse ? n - 1 - j : j;
            x[e] = j < n ? __ldg(in + k) : op_identity<kProd>();
            key[e] = j < n ? __ldg(keys + k) : (long long)0x7fffffffffffffffll;
        }
    }
    // key of the element before this thread's first one: previous lane, previous warp (shared), previous tile (global)
    long long prev = __shfl_up_sync(kFullMask, key[kKeyItems - 1], 1);
    if (lane == 31) s_last_key[warp] = key[kKeyItems - 1];
    __syncthreads();
    if (lane == 0) {
        if (warp > 0) prev = s_last_key[warp - 1];
        else if (tile0 > 0) prev = __ldg(keys + (kReverse ? n - 1 - (tile0 - 1) : tile0 - 1));
    }
    // ---- thread-local segmented inclusive scan
    int head[kKeyItems];
    float res[kKeyItems];
    SegPair<kProd> acc;
    acc.v = op_identity<kProd>();
    acc.f = 0;
    int first_head_local = kKeyTile;
#pragma unroll
    for (int e = 0; e < kKeyItems; ++e) {
        const int64_t j = j0 + e;
        head[e] = (j < n && (j == 0 || key[e] != (e ? key[e - 1] : prev))) ? 1 : 0;
        if (head[e] && first_head_local == kKeyTile) first_head_local = tid * kKeyItems + e;
        if (head[e]) {
            acc.v = x[e];
            acc.f = 1;
        } else {
            acc.v = op_apply<kProd>(acc.v, x[e]);
        }
        res[e] = acc.v;
    }
    // ---- block-level segmented scan of the per-thread aggregates
    SegPair<kProd> incl = acc;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        SegPair<kProd> y;
        y.v = __shfl_up_sync(kFullMask, incl.v, s);
        y.f = __shfl_up_sync(kFullMask, incl.f, s);
        if (lane >= s) incl = seg_combine<kProd>(y, incl);
    }
    if (lane == 31) {
        s_v[warp] = incl.v;
        s_f[warp] = incl.f;
    }
    if (first_head_local != kKeyTile) atomicMin(&s_first_head, first_head_local);
    __syncthreads();
    SegPair<kProd> pre;  // exclusive prefix over the threads of the tile
    pre.v = op_identity<kProd>();
    pre.f = 0;
    for (int w = 0; w < warp; ++w) {
        SegPair<kProd> y;
        y.v = s_v[w];
        y.f = s_f[w];
        pre = seg_combine<kProd>(pre, y);
    }
    {
        SegPair<kProd> y;
        y.v = __shfl_up_sync(kFullMask, incl.v, 1);
        y.f = __shfl_up_sync(kFullMask, incl.f, 1);
        if (lane > 0) pre = seg_combine<kProd>(pre, y);
    }
    // ---- publish this tile, look back for the value carried in (one thread; the chain is one tile deep in practice)
    if (tid == kKeyThreads - 1) {
        const SegPair<kProd> tot = seg_combine<kProd>(pre, acc);
        float carry = op_identity<kProd>();
        volatile unsigned long long* d = desc;
        if (tile == 0 || tot.f) {
            d[tile] = tile_word(tot.v, tot.f, kStPrefix);  // a head inside (or nothing before): complete for successors
        } else {
            d[tile] = tile_word(tot.v, 0, kStAggregate);
        }
        if (tile > 0) {
            for (long long t = (long long)tile - 1; t >= 0; --t) {
                unsigned long long w;
                do {
                    w = d[t];
                } while ((w & kStMask) == 0ull);
                carry = op_apply<kProd>(__uint_as_float((unsigned int)w), carry);
                if ((w & kStMask) == kStPrefix) break;
            }
            if (!tot.f) {
                __threadfence();
                d[tile] = tile_word(op_apply<kProd>(carry, tot.v), 0, kStPrefix);
            }
        }
        s_carry = carry;
    }
    __syncthreads();
    const float carry = s_carry;
    const int lead = s_first_head;  // elements of the tile before its first head continue the previous tile's segment
    // ---- results: elements before the thread's first head continue `pre`; those before the tile's first head also `carry`
    float o[kKeyItems];
    bool open = true;
    // inclusive value of the element just before this thread's first one (pre.v is the identity for thread 0)
    float run_prev = pre.f ? pre.v : op_apply<kProd>(carry, pre.v);
#pragma unroll
    for (int e = 0; e < kKeyItems; ++e) {
        if (head[e]) open = false;
        float incl_v = open ? op_apply<kProd>(pre.v, res[e]) : res[e];
        if (tid * kKeyItems + e < lead) incl_v = op_apply<kProd>(carry, incl_v);
        o[e] = kInclusive ? incl_v : (head[e] ? op_identity<kProd>() : run_prev);
        run_prev = incl_v;
    }
    if (kVec && j0 + kKeyItems <= n) {
#pragma unroll
        for (int q = 0; q < kKeyItems / 4; ++q)
            reinterpret_cast<float4*>(out + j0)[q] = make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
    } else {
#pragma unroll
        for (int e = 0; e < kKeyItems; ++e) {
            const int64_t j = j0 + e;
            if (j < n) out[kReverse ? n - 1 - j : j] = o[e];
        }
    }
}

// ---------------------------------------------------------------------------
// pack_info
// ---------------------------------------------------------------------------
constexpr int kPackTile = 1024;

__global__ void __launch_bounds__(256) pack_count_kernel(int64_t n, const int64_t* __restrict__ ray_indices,
                                                         int32_t n_rays, unsigned long long* __restrict__ counts)
{
    // warp-aggregated histogram: one atomic per run of equal keys inside a warp
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t n_up = (n + 31) & ~(int64_t)31;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_up; i += stride) {
        const bool valid = i < n;
        const long long key = valid ? ray_indices[i] : -1;
        const long long prev = __shfl_up_sync(kFullMask, key, 1);
        const bool head = valid && (lane == 0 || prev != key);
        const unsigned heads = __ballot_sync(kFullMask, head);
        const unsigned valids = __ballot_sync(kFullMask, valid);
        if (head && key >= 0 && key < n_rays) {
            const unsigned later = heads & ~((2u << lane) - 1u);  // heads strictly after this lane
            const int end = later ? __ffs(later) - 1 : (32 - __clz(valids));
            atomicAdd(counts + key, (unsigned long long)(end - lane));
        }
    }
}

__global__ void __launch_bounds__(kPackTile) pack_tilesum_kernel(int32_t n_rays,
                                                                const unsigned long long* __restrict__ counts,
                                                                unsigned long long* __restrict__ tile_sums)
{
    __shared__ unsigned long long s[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int r = blockIdx.x * kPackTile + tid;
    unsigned long long v = r < n_rays ? counts[r] : 0ull;
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) v += __shfl_xor_sync(kFullMask, v, sft);
    if (lane == 0) s[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = s[lane];
#pragma unroll
        for (int sft = 16; sft > 0; sft >>= 1) v += __shfl_xor_sync(kFullMask, v, sft);
        if (lane == 0) tile_sums[blockIdx.x] = v;
    }
}

__global__ void __launch_bounds__(kPackTile) pack_scan_kernel(int32_t n_rays,
                                                             const unsigned long long* __restrict__ counts,
                                                             const unsigned long long* __restrict__ tile_sums,
                                                             int64_t* __restrict__ packed_info,
                                                             int64_t* __restrict__ total_dev,
                                                             int64_t* __restrict__ total_host)
{
    __shared__ unsigned long long s[32];
    __shared__ unsigned long long s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned long long b = 0;
    for (int i = tid; i < (int)blockIdx.x; i += kPackTile) b += tile_sums[i];
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) b += __shfl_xor_sync(kFullMask, b, sft);
    if (lane == 0) s[warp] = b;
    __syncthreads();
    if (tid == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < 32; ++w) t += s[w];
        s_base = t;
    }
    __syncthreads();
    const int r = blockIdx.x * kPackTile + tid;
    const unsigned long long c = r < n_rays ? counts[r] : 0ull;
    unsigned long long x = c;
#pragma unroll
    for (int sft = 1; sft < 32; sft <<= 1) {
        const unsigned long long y = __shfl_up_sync(kFullMask, x, sft);
        if (lane >= sft) x += y;
    }
    __syncthreads();
    if (lane == 31) s[warp] = x;
    __syncthreads();
    unsigned long long pre = s_base;
    for (int w = 0; w < warp; ++w) pre += s[w];
    if (r < n_rays) {
        longlong2 v;
        v.x = (long long)(pre + x - c);
        v.y = (long long)c;
        *reinterpret_cast<longlong2*>(packed_info + 2 * (int64_t)r) = v;
        if (r == n_rays - 1) {  // grand total, optionally straight into pinned host memory
            if (total_dev) *total_dev = v.x + v.y;
            if (total_host) {
                *total_host = v.x + v.y;
                __threadfence_system();
            }
        }
    }
}

// ---------------------------------------------------------------------------
// Visibility filter + stream compaction (the sigma_fn / alpha_fn branch of
// OccGridEstimator.sampling, reference estimators/occ_grid.py:180-220 +
// volrend.py:379-494): keep sample i iff T_i >= early_stop_eps and (alpha_thre <= 0 or
// alpha_i >= alpha_thre).  The reference runs a scan kernel, ~6 elementwise ops and three
// synchronising boolean mask-selects; here: mask + per-ray counts, the two-level scan of
// pack_info, and a ballot compaction that writes the kept samples and their packed_info.
// ---------------------------------------------------------------------------
template <bool kAlpha>
__global__ void __launch_bounds__(kScanWarps * 32) vis_mask_kernel(int32_t n_rays,
                                                                   const int64_t* __restrict__ packed_info,
                                                                   const float* __restrict__ t_starts,
                                                                   const float* __restrict__ t_ends,
                                                                   const float* __restrict__ dens, float early_stop_eps,
                                                                   float alpha_thre, uint8_t* __restrict__ mask,
                                                                   unsigned long long* __restrict__ counts)
{
    const int lane = threadIdx.x & 31;
    for (int r = blockIdx.x * kScanWarps + (threadIdx.x >> 5); r < n_rays; r += gridDim.x * kScanWarps) {
        const longlong2 pi = *reinterpret_cast<const longlong2*>(packed_info + 2 * (int64_t)r);
        const int64_t start = pi.x, n = pi.y;
        float carry = kAlpha ? 1.0f : 0.0f;  // `init` of the reference kernel; then the previous blocks' total
        const unsigned kept =
            vis_blocks<kAlpha>(t_starts, t_ends, dens, start, n, lane, carry, early_stop_eps, alpha_thre, mask, 0);
        if (lane == 0) counts[r] = kept;
    }
}

__global__ void __launch_bounds__(kScanWarps * 32) vis_compact_kernel(int32_t n_rays,
                                                                      const int64_t* __restrict__ packed_info,
                                                                      const int64_t* __restrict__ new_packed_info,
                                                                      const uint8_t* __restrict__ mask,
                                                                      const float* __restrict__ t_starts,
                                                                      const float* __restrict__ t_ends,
                                                                      int64_t* __restrict__ out_ray,
                                                                      float* __restrict__ out_ts, float* __restrict__ out_te)
{
    const int lane = threadIdx.x & 31;
    for (int r = blockIdx.x * kScanWarps + (threadIdx.x >> 5); r < n_rays; r += gridDim.x * kScanWarps) {
        const longlong2 pi = *reinterpret_cast<const longlong2*>(packed_info + 2 * (int64_t)r);
        const longlong2 po = *reinterpret_cast<const longlong2*>(new_packed_info + 2 * (int64_t)r);
        if (po.y == 0) continue;
        int64_t dst = po.x;
        for (int64_t base = 0; base < pi.y; base += 32) {
            const int64_t i = pi.x + base + lane;
            const bool keep = (base + lane < pi.y) && mask[i];
            const unsigned b = __ballot_sync(kFullMask, keep);
            if (keep) {
                const int64_t k = dst + __popc(b & ((1u << lane) - 1u));
                out_ray[k] = r;
                out_ts[k] = __ldg(t_starts + i);
                out_te[k] = __ldg(t_ends + i);
            }
            dst += __popc(b);
        }
    }
}

// ---------------------------------------------------------------------------
// Visibility filter in rounds (OccGridEstimator.sampling_until_opaque): the field closure runs on each live ray's
// next k samples only, and a ray stops being live once the transmittance its next sample would get fails
// T >= early_stop_eps.  Each round advances a ray by whole 32-sample blocks from its first sample (k is a multiple
// of 32) and carries the block total across rounds, so every T, alpha and keep bit is the one-shot filter's
// (vis_blocks, vis_block.cuh).  Per round: a gather of the closure's inputs, the closure, the step (mask bytes,
// kept counts, carry, live flag), the exclusive scan of the live flags (pack_tilesum / pack_scan), a scatter of the
// next live list with each slot's sample count, and the scan of those counts, whose total goes to a pinned status
// slot with the next round's n_alive, k and the running kept total.  The finish is vis_compact_kernel over the
// kept counts' scan; mask bytes of samples that were never evaluated stay 0 from the zeroing at the start.
// See DESIGN.md section 4.12.
// ---------------------------------------------------------------------------
constexpr int kRoundBlock = 32;      // samples per scan block: a round evaluates whole blocks of every live ray
constexpr int kRoundMaxBlocks = 8;   // k_r = 32 clamp(rays with samples / n_alive, 1, 8)

// Workspace (offsets 16-byte aligned) for R rays and N samples:
//   header (64 B): i64 live rays after the current step (scan total), u64 kept samples so far
//   lists [2][R] i32     live rays of the even / odd rounds, ascending
//   carry [R] f32        per ray: total of its evaluated blocks
//   done [R] i64         per ray: samples evaluated
//   counts [R] u64       per ray: samples kept (what pack_scan turns into the new packed_info)
//   live [R] u64         per slot of the current round: stays live (0 / 1)
//   live_pi [R][2] i64   exclusive scan of `live` (slot's rank among the live slots, flag)
//   cnt [R] u64          per slot of the next round: its sample count
//   plan [R][2] i64      exclusive scan of `cnt`: (offset into the closure's inputs, count)
//   tile_sums [T] u64    T = ceil(R / kPackTile)
//   mask [N] u8          keep byte of every sample
struct VisRoundsWs {
    int64_t* n_next;
    unsigned long long* kept;
    int32_t* lists;
    float* carry;
    int64_t* done;
    unsigned long long* counts;
    unsigned long long* live;
    int64_t* live_pi;
    unsigned long long* cnt;
    int64_t* plan;
    unsigned long long* tile_sums;
    uint8_t* mask;
    int32_t n_rays;
};

static int64_t vis_rounds_bytes(int32_t R, int64_t N, VisRoundsWs* w, char* base)
{
    const int64_t T = (R + kPackTile - 1) / kPackTile;
    int64_t at = 64;
    auto take = [&](int64_t bytes) {
        char* p = base ? base + at : nullptr;
        at += (bytes + 15) & ~(int64_t)15;
        return p;
    };
    char* lists = take(8 * (int64_t)R);
    char* carry = take(4 * (int64_t)R);
    char* done = take(8 * (int64_t)R);
    char* counts = take(8 * (int64_t)R);
    char* live = take(8 * (int64_t)R);
    char* live_pi = take(16 * (int64_t)R);
    char* cnt = take(8 * (int64_t)R);
    char* plan = take(16 * (int64_t)R);
    char* tile_sums = take(8 * T);
    char* mask = take(N);
    if (w) {
        w->n_next = (int64_t*)base;
        w->kept = (unsigned long long*)(base + 8);
        w->lists = (int32_t*)lists;
        w->carry = (float*)carry;
        w->done = (int64_t*)done;
        w->counts = (unsigned long long*)counts;
        w->live = (unsigned long long*)live;
        w->live_pi = (int64_t*)live_pi;
        w->cnt = (unsigned long long*)cnt;
        w->plan = (int64_t*)plan;
        w->tile_sums = (unsigned long long*)tile_sums;
        w->mask = (uint8_t*)mask;
        w->n_rays = R;
    }
    return at;
}

static VisRoundsWs vis_rounds_view(void* base, int32_t R, int64_t N)
{
    VisRoundsWs w;
    vis_rounds_bytes(R, N, &w, (char*)base);
    return w;
}

// Every ray: nothing evaluated or kept, the initial carry; slot r of the "round before round 0" is ray r, live when
// it has samples.
__global__ void __launch_bounds__(256) vis_rounds_init_kernel(VisRoundsWs ws, const int64_t* __restrict__ packed_info,
                                                              float carry0)
{
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < ws.n_rays; r += gridDim.x * blockDim.x) {
        ws.carry[r] = carry0;
        ws.done[r] = 0;
        ws.counts[r] = 0ull;
        ws.live[r] = packed_info[2 * (int64_t)r + 1] > 0 ? 1ull : 0ull;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *ws.kept = 0ull;
}

// Warp per live slot: the slot's next plan[i].y samples (from the ray's first unevaluated one) -> the closure's
// inputs at offset plan[i].x.
__global__ void __launch_bounds__(kScanWarps * 32) vis_rounds_gather_kernel(VisRoundsWs ws, int32_t round,
                                                                            int32_t n_alive,
                                                                            const int64_t* __restrict__ packed_info,
                                                                            const float* __restrict__ t_starts,
                                                                            const float* __restrict__ t_ends,
                                                                            int64_t* __restrict__ out_ray,
                                                                            float* __restrict__ out_ts,
                                                                            float* __restrict__ out_te)
{
    const int lane = threadIdx.x & 31;
    const int32_t* list = ws.lists + (int64_t)(round & 1) * ws.n_rays;
    for (int i = blockIdx.x * kScanWarps + (threadIdx.x >> 5); i < n_alive; i += gridDim.x * kScanWarps) {
        const int r = list[i];
        const longlong2 pl = *reinterpret_cast<const longlong2*>(ws.plan + 2 * (int64_t)i);
        const int64_t src = packed_info[2 * (int64_t)r] + ws.done[r];
        for (int64_t j = lane; j < pl.y; j += 32) {
            out_ray[pl.x + j] = r;
            out_ts[pl.x + j] = __ldg(t_starts + src + j);
            out_te[pl.x + j] = __ldg(t_ends + src + j);
        }
    }
}

// Warp per live slot: the filter over the slot's samples of this round (the closure's inputs and outputs at offset
// plan[i].x), their mask bytes at the ray's sample positions, the kept count, the carry, and whether the ray stays
// live: samples left, and its next sample's T passes.
template <bool kAlpha>
__global__ void __launch_bounds__(kScanWarps * 32) vis_rounds_step_kernel(VisRoundsWs ws, int32_t round,
                                                                          int32_t n_alive,
                                                                          const int64_t* __restrict__ packed_info,
                                                                          const float* __restrict__ t_starts,
                                                                          const float* __restrict__ t_ends,
                                                                          const float* __restrict__ dens,
                                                                          float early_stop_eps, float alpha_thre)
{
    const int lane = threadIdx.x & 31;
    const int32_t* list = ws.lists + (int64_t)(round & 1) * ws.n_rays;
    unsigned long long kept_warp = 0;
    for (int i = blockIdx.x * kScanWarps + (threadIdx.x >> 5); i < n_alive; i += gridDim.x * kScanWarps) {
        const int r = list[i];
        const longlong2 pl = *reinterpret_cast<const longlong2*>(ws.plan + 2 * (int64_t)i);
        const longlong2 pi = *reinterpret_cast<const longlong2*>(packed_info + 2 * (int64_t)r);
        const int64_t d0 = ws.done[r];
        float carry = ws.carry[r];
        const unsigned kept = vis_blocks<kAlpha>(t_starts, t_ends, dens, pl.x, pl.y, lane, carry, early_stop_eps,
                                                 alpha_thre, ws.mask, pi.x + d0 - pl.x);
        kept_warp += kept;
        if (lane == 0) {
            const int64_t d1 = d0 + pl.y;
            ws.counts[r] += kept;
            ws.done[r] = d1;
            ws.carry[r] = carry;
            ws.live[i] = (d1 < pi.y && vis_next_passes<kAlpha>(carry, early_stop_eps)) ? 1ull : 0ull;
        }
    }
    if (lane == 0 && kept_warp) atomicAdd(ws.kept, kept_warp);
}

// Thread per slot of the round just stepped (`first`: the rays themselves, before round 0): a live slot moves to its
// rank in the next round's list and gets min(k, samples left) samples; the others zero the tail of `cnt`, so that
// the scan over all n_cur entries totals the next round's samples.  Slot 0 also publishes the next round's
// {n_alive, k, -, kept samples so far}; the scan of `cnt` fills in the sample count.
__global__ void __launch_bounds__(256) vis_rounds_scatter_kernel(VisRoundsWs ws, int32_t round, int32_t n_cur,
                                                                 int32_t first, int32_t n_with_samples,
                                                                 const int64_t* __restrict__ packed_info,
                                                                 int64_t* status_host)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cur) return;
    const int64_t n_next = *ws.n_next;
    const int64_t q = n_next > 0 ? n_with_samples / n_next : 1;
    const int64_t k = first ? kRoundBlock : kRoundBlock * (q < 1 ? 1 : (q > kRoundMaxBlocks ? kRoundMaxBlocks : q));
    const longlong2 lb = *reinterpret_cast<const longlong2*>(ws.live_pi + 2 * (int64_t)i);
    if (lb.y) {
        const int r = first ? i : ws.lists[(int64_t)(round & 1) * ws.n_rays + i];
        ws.lists[(int64_t)(first ? 0 : (round + 1) & 1) * ws.n_rays + lb.x] = r;
        const int64_t left = packed_info[2 * (int64_t)r + 1] - ws.done[r];
        ws.cnt[lb.x] = (unsigned long long)(left < k ? left : k);
    } else {
        ws.cnt[n_next + i - lb.x] = 0ull;
    }
    if (i == 0) {  // read by the host after it has waited for the scan behind this kernel
        status_host[0] = n_next;
        status_host[1] = n_next > 0 ? k : 0;
        status_host[3] = (int64_t)*ws.kept;
    }
}

}  // namespace nfa

using namespace nfa;

static inline int32_t launch_status_s()
{
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? NFA_OK : (int32_t)e;
}

template <bool kProd, bool kInclusive>
static void launch_packed(bool reverse, int32_t n_rays, const int64_t* pi, const float* in, float* out,
                          int32_t normalize, cudaStream_t s)
{
    const int blocks = (n_rays + kScanWarps - 1) / kScanWarps;
    if (reverse) scan_packed_kernel<kProd, kInclusive, true><<<blocks, kScanWarps * 32, 0, s>>>(n_rays, pi, in, out, normalize);
    else scan_packed_kernel<kProd, kInclusive, false><<<blocks, kScanWarps * 32, 0, s>>>(n_rays, pi, in, out, normalize);
}

template <bool kProd, bool kInclusive, bool kReverse>
static void launch_bykey(int64_t n, const int64_t* keys, const float* in, float* out, void* workspace, cudaStream_t s)
{
    const int n_tiles = (int)((n + kKeyTile - 1) / kKeyTile);
    unsigned int* ticket = (unsigned int*)workspace;
    unsigned long long* desc = (unsigned long long*)((char*)workspace + 16);
    cudaMemsetAsync(workspace, 0, 16 + (size_t)n_tiles * 8, s);
    const bool vec = !kReverse && ((((uintptr_t)keys) | ((uintptr_t)in) | ((uintptr_t)out)) & 15u) == 0;
    if (vec) scan_bykey_kernel<kProd, kInclusive, kReverse, true><<<n_tiles, kKeyThreads, 0, s>>>(n, keys, in, out, ticket, desc);
    else scan_bykey_kernel<kProd, kInclusive, kReverse, false><<<n_tiles, kKeyThreads, 0, s>>>(n, keys, in, out, ticket, desc);
}

extern "C" {

int32_t nfa_scan_packed(int32_t n_rays, const int64_t* packed_info, const float* in, float* out, int32_t op_prod,
                        int32_t inclusive, int32_t reverse, int32_t normalize, nfa_stream_t stream)
{
    if (n_rays < 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!packed_info || !in || !out) return NFA_ERR_ARG;
    if ((((uintptr_t)packed_info) & 15u) != 0) return NFA_ERR_ARG;
    if (normalize && (op_prod || !inclusive || reverse)) return NFA_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    if (op_prod) {
        if (inclusive) launch_packed<true, true>(reverse, n_rays, packed_info, in, out, normalize, s);
        else launch_packed<true, false>(reverse, n_rays, packed_info, in, out, normalize, s);
    } else {
        if (inclusive) launch_packed<false, true>(reverse, n_rays, packed_info, in, out, normalize, s);
        else launch_packed<false, false>(reverse, n_rays, packed_info, in, out, normalize, s);
    }
    return launch_status_s();
}

int64_t nfa_scan_by_key_workspace_bytes(int64_t n)
{
    if (n <= 0) return 16;
    const int64_t n_tiles = (n + kKeyTile - 1) / kKeyTile;
    return 16 + ((n_tiles * 8 + 15) & ~(int64_t)15);
}

int32_t nfa_scan_by_key(int64_t n, const int64_t* keys, const float* in, float* out, int32_t op_prod,
                        int32_t inclusive, int32_t reverse, void* workspace, nfa_stream_t stream)
{
    if (n < 0) return NFA_ERR_ARG;
    if (n == 0) return NFA_OK;
    if (!keys || !in || !out || !workspace) return NFA_ERR_ARG;
    if (n > (int64_t)kKeyTile * INT32_MAX) return NFA_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
#define NFA_BYKEY(P, I, R) launch_bykey<P, I, R>(n, keys, in, out, workspace, s)
    if (op_prod) {
        if (inclusive) { if (reverse) NFA_BYKEY(true, true, true); else NFA_BYKEY(true, true, false); }
        else { if (reverse) NFA_BYKEY(true, false, true); else NFA_BYKEY(true, false, false); }
    } else {
        if (inclusive) { if (reverse) NFA_BYKEY(false, true, true); else NFA_BYKEY(false, true, false); }
        else { if (reverse) NFA_BYKEY(false, false, true); else NFA_BYKEY(false, false, false); }
    }
#undef NFA_BYKEY
    return launch_status_s();
}

int64_t nfa_pack_info_workspace_bytes(int32_t n_rays)
{
    if (n_rays <= 0) return 16;
    const int64_t tiles = (n_rays + kPackTile - 1) / kPackTile;
    return (int64_t)n_rays * 8 + tiles * 8 + 16;
}

int32_t nfa_counts_to_packed_info(int32_t n_rays, const int64_t* counts, int64_t* packed_info, void* workspace,
                                  nfa_stream_t stream)
{
    if (n_rays < 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!counts || !packed_info || !workspace) return NFA_ERR_ARG;
    if ((((uintptr_t)packed_info) & 15u) != 0) return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    const int tiles = (n_rays + kPackTile - 1) / kPackTile;
    unsigned long long* tile_sums = (unsigned long long*)workspace;
    const unsigned long long* c = reinterpret_cast<const unsigned long long*>(counts);
    pack_tilesum_kernel<<<tiles, kPackTile, 0, s>>>(n_rays, c, tile_sums);
    pack_scan_kernel<<<tiles, kPackTile, 0, s>>>(n_rays, c, tile_sums, packed_info, nullptr, nullptr);
    return launch_status_s();
}

int32_t nfa_pack_info(int64_t n, const int64_t* ray_indices, int32_t n_rays, int64_t* packed_info, void* workspace,
                      nfa_stream_t stream)
{
    if (n < 0 || n_rays < 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!packed_info || !workspace || (n > 0 && !ray_indices)) return NFA_ERR_ARG;
    if ((((uintptr_t)packed_info) & 15u) != 0) return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long* counts = (unsigned long long*)workspace;
    const int tiles = (n_rays + kPackTile - 1) / kPackTile;
    unsigned long long* tile_sums = counts + n_rays;
    cudaError_t e = cudaMemsetAsync(counts, 0, (size_t)n_rays * 8, s);
    if (e != cudaSuccess) return (int32_t)e;
    if (n > 0) {
        const int64_t warps = (n + 31) / 32;
        const int blocks = (int)((warps + 7) / 8 < kNumSMs * 16 ? (warps + 7) / 8 : kNumSMs * 16);
        pack_count_kernel<<<blocks, 256, 0, s>>>(n, ray_indices, n_rays, counts);
    }
    pack_tilesum_kernel<<<tiles, kPackTile, 0, s>>>(n_rays, counts, tile_sums);
    pack_scan_kernel<<<tiles, kPackTile, 0, s>>>(n_rays, counts, tile_sums, packed_info, nullptr, nullptr);
    return launch_status_s();
}

int64_t nfa_visibility_workspace_bytes(int32_t n_rays, int64_t n_samples)
{
    if (n_rays <= 0 || n_samples < 0) return 16;
    const int64_t tiles = (n_rays + kPackTile - 1) / kPackTile;
    return ((n_samples + 15) & ~(int64_t)15) + (int64_t)n_rays * 8 + tiles * 8 + 16;
}

int32_t nfa_visibility_compact(int32_t n_rays, int64_t n_samples, const int64_t* packed_info, const float* t_starts,
                               const float* t_ends, const float* sigmas_or_alphas, int32_t from_alpha,
                               float early_stop_eps, float alpha_thre, void* workspace, int64_t* new_packed_info,
                               int64_t* out_ray_indices, float* out_t_starts, float* out_t_ends, int64_t* total_dev,
                               int64_t* total_host, nfa_stream_t stream)
{
    if (n_rays < 0 || n_samples < 0) return NFA_ERR_ARG;
    if (total_host) *total_host = 0;
    if (n_rays == 0) return NFA_OK;
    if (!packed_info || !new_packed_info || !workspace) return NFA_ERR_ARG;
    if (n_samples > 0 && (!t_starts || !t_ends || !sigmas_or_alphas || !out_ray_indices || !out_t_starts || !out_t_ends))
        return NFA_ERR_ARG;
    if (((((uintptr_t)packed_info) | ((uintptr_t)new_packed_info)) & 15u) != 0) return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    uint8_t* mask = (uint8_t*)workspace;
    unsigned long long* counts = (unsigned long long*)((char*)workspace + ((n_samples + 15) & ~(int64_t)15));
    const int tiles = (n_rays + kPackTile - 1) / kPackTile;
    unsigned long long* tile_sums = counts + n_rays;
    const int need = (n_rays + kScanWarps - 1) / kScanWarps;
    const int blocks = need < kNumSMs * 8 ? need : kNumSMs * 8;
    if (from_alpha)
        vis_mask_kernel<true><<<blocks, kScanWarps * 32, 0, s>>>(n_rays, packed_info, t_starts, t_ends, sigmas_or_alphas,
                                                                 early_stop_eps, alpha_thre, mask, counts);
    else
        vis_mask_kernel<false><<<blocks, kScanWarps * 32, 0, s>>>(n_rays, packed_info, t_starts, t_ends, sigmas_or_alphas,
                                                                  early_stop_eps, alpha_thre, mask, counts);
    pack_tilesum_kernel<<<tiles, kPackTile, 0, s>>>(n_rays, counts, tile_sums);
    pack_scan_kernel<<<tiles, kPackTile, 0, s>>>(n_rays, counts, tile_sums, new_packed_info, total_dev, total_host);
    if (n_samples > 0)
        vis_compact_kernel<<<blocks, kScanWarps * 32, 0, s>>>(n_rays, packed_info, new_packed_info, mask, t_starts, t_ends,
                                                              out_ray_indices, out_t_starts, out_t_ends);
    return launch_status_s();
}


int64_t nfa_vis_rounds_workspace_bytes(int32_t n_rays, int64_t n_samples)
{
    if (n_rays < 1 || n_samples < 0) return 0;
    return vis_rounds_bytes(n_rays, n_samples, nullptr, nullptr);
}

static void vis_rounds_plan(const VisRoundsWs& w, int32_t round, int32_t n_cur, int32_t first, int32_t n_with_samples,
                            const int64_t* packed_info, int64_t* status_host, cudaStream_t s)
{
    const int tiles = (n_cur + kPackTile - 1) / kPackTile;
    pack_tilesum_kernel<<<tiles, kPackTile, 0, s>>>(n_cur, w.live, w.tile_sums);
    pack_scan_kernel<<<tiles, kPackTile, 0, s>>>(n_cur, w.live, w.tile_sums, w.live_pi, w.n_next, nullptr);
    vis_rounds_scatter_kernel<<<(n_cur + 255) / 256, 256, 0, s>>>(w, round, n_cur, first, n_with_samples, packed_info,
                                                                  status_host);
    pack_tilesum_kernel<<<tiles, kPackTile, 0, s>>>(n_cur, w.cnt, w.tile_sums);
    pack_scan_kernel<<<tiles, kPackTile, 0, s>>>(n_cur, w.cnt, w.tile_sums, w.plan, nullptr, status_host + 2);
}

static inline bool aligned16(const void* p) { return (((uintptr_t)p) & 15u) == 0; }

int32_t nfa_vis_rounds_begin(int32_t n_rays, int64_t n_samples, const int64_t* packed_info, int32_t from_alpha,
                             void* workspace, int64_t* status_host, nfa_stream_t stream)
{
    if (n_rays < 1 || n_samples < 0) return NFA_ERR_ARG;
    if (!packed_info || !workspace || !status_host || !aligned16(packed_info) || !aligned16(workspace))
        return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    const VisRoundsWs w = vis_rounds_view(workspace, n_rays, n_samples);
    if (n_samples > 0) {
        const cudaError_t e = cudaMemsetAsync(w.mask, 0, (size_t)n_samples, s);
        if (e != cudaSuccess) return (int32_t)e;
    }
    const int need = (n_rays + 255) / 256;
    vis_rounds_init_kernel<<<need < kNumSMs * 8 ? need : kNumSMs * 8, 256, 0, s>>>(w, packed_info,
                                                                                  from_alpha ? 1.0f : 0.0f);
    vis_rounds_plan(w, 0, n_rays, 1, 0, packed_info, status_host, s);
    return launch_status_s();
}

static bool vis_rounds_round_ok(int32_t n_rays, int64_t n_samples, int32_t round, int32_t n_alive)
{
    return n_rays >= 1 && n_samples >= 0 && round >= 0 && n_alive >= 1 && n_alive <= n_rays;
}

int32_t nfa_vis_rounds_gather(int32_t n_rays, int64_t n_samples, int32_t round, int32_t n_alive,
                              const int64_t* packed_info, const float* t_starts, const float* t_ends,
                              const void* workspace, int64_t* out_ray_indices, float* out_t_starts, float* out_t_ends,
                              nfa_stream_t stream)
{
    if (!vis_rounds_round_ok(n_rays, n_samples, round, n_alive)) return NFA_ERR_ARG;
    if (!packed_info || !t_starts || !t_ends || !workspace || !out_ray_indices || !out_t_starts || !out_t_ends ||
        !aligned16(workspace))
        return NFA_ERR_ARG;
    const int need = (n_alive + kScanWarps - 1) / kScanWarps;
    vis_rounds_gather_kernel<<<need < kNumSMs * 8 ? need : kNumSMs * 8, kScanWarps * 32, 0, (cudaStream_t)stream>>>(
        vis_rounds_view(const_cast<void*>(workspace), n_rays, n_samples), round, n_alive, packed_info, t_starts,
        t_ends, out_ray_indices, out_t_starts, out_t_ends);
    return launch_status_s();
}

int32_t nfa_vis_rounds_step(int32_t n_rays, int64_t n_samples, int32_t round, int32_t n_alive,
                            int32_t n_with_samples, const int64_t* packed_info, const float* t_starts,
                            const float* t_ends, const float* sigmas_or_alphas, int32_t from_alpha,
                            float early_stop_eps, float alpha_thre, void* workspace, int64_t* status_host,
                            nfa_stream_t stream)
{
    if (!vis_rounds_round_ok(n_rays, n_samples, round, n_alive) || n_with_samples < n_alive ||
        n_with_samples > n_rays)
        return NFA_ERR_ARG;
    if (!packed_info || !t_starts || !t_ends || !sigmas_or_alphas || !workspace || !status_host ||
        !aligned16(workspace))
        return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    const VisRoundsWs w = vis_rounds_view(workspace, n_rays, n_samples);
    const int need = (n_alive + kScanWarps - 1) / kScanWarps;
    const int blocks = need < kNumSMs * 8 ? need : kNumSMs * 8;
    if (from_alpha)
        vis_rounds_step_kernel<true><<<blocks, kScanWarps * 32, 0, s>>>(w, round, n_alive, packed_info, t_starts,
                                                                        t_ends, sigmas_or_alphas, early_stop_eps,
                                                                        alpha_thre);
    else
        vis_rounds_step_kernel<false><<<blocks, kScanWarps * 32, 0, s>>>(w, round, n_alive, packed_info, t_starts,
                                                                         t_ends, sigmas_or_alphas, early_stop_eps,
                                                                         alpha_thre);
    vis_rounds_plan(w, round, n_alive, 0, n_with_samples, packed_info, status_host, s);
    return launch_status_s();
}

int32_t nfa_vis_rounds_finish(int32_t n_rays, int64_t n_samples, const int64_t* packed_info, const float* t_starts,
                              const float* t_ends, const void* workspace, int64_t* new_packed_info,
                              int64_t* out_ray_indices, float* out_t_starts, float* out_t_ends, nfa_stream_t stream)
{
    if (n_rays < 1 || n_samples < 0) return NFA_ERR_ARG;
    if (!packed_info || !workspace || !new_packed_info || !aligned16(workspace) || !aligned16(packed_info) ||
        !aligned16(new_packed_info))
        return NFA_ERR_ARG;
    if (n_samples > 0 && (!t_starts || !t_ends || !out_ray_indices || !out_t_starts || !out_t_ends))
        return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    const VisRoundsWs w = vis_rounds_view(const_cast<void*>(workspace), n_rays, n_samples);
    const int tiles = (n_rays + kPackTile - 1) / kPackTile;
    pack_tilesum_kernel<<<tiles, kPackTile, 0, s>>>(n_rays, w.counts, w.tile_sums);
    pack_scan_kernel<<<tiles, kPackTile, 0, s>>>(n_rays, w.counts, w.tile_sums, new_packed_info, nullptr, nullptr);
    if (n_samples > 0) {
        const int need = (n_rays + kScanWarps - 1) / kScanWarps;
        vis_compact_kernel<<<need < kNumSMs * 8 ? need : kNumSMs * 8, kScanWarps * 32, 0, s>>>(
            n_rays, packed_info, new_packed_info, w.mask, t_starts, t_ends, out_ray_indices, out_t_starts,
            out_t_ends);
    }
    return launch_status_s();
}

}  // extern "C"
