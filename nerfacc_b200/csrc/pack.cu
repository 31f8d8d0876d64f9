// pack.cu -- moving per-sample data between the packed layout and the padded per-ray layout.
//
// packed: (N, row) rows, ray r owning rows [start_r, start_r + count_r) (packed_info = (start, count));
// padded: (n_rays, S, row) rows, ray r owning row block r.
//
// The kernels move bytes and do no arithmetic: every entry point takes the size of one row in bytes, and copies in
// units of 16, 8, 4, 2 or 1 bytes -- the largest that divides the row size and every pointer -- so any dtype comes
// out bit-exact.  A warp owns a ray (or a mask row); its rows are contiguous on at least one side, so the lanes
// walk consecutive units and each warp-wide load / store covers 32 consecutive units.
//
// Packed outputs that must be defined everywhere (unpack_info's -1 at positions no chunk covers, pack_rows' zeros)
// are written in one pass when the chunks are in order -- start_r >= end_{r-1} for every r, as for every packed_info
// this library returns -- by letting each ray also write the gap behind its chunk.  chunk_order_kernel checks that
// order on the device (16 B of packed_info per ray), and only when it fails does fill_if_unordered_kernel pre-fill the
// output before the chunks are scattered; no host synchronisation either way.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/nerfacc_b200.h"
#include "sm_count.cuh"

namespace nfa {

constexpr int kPkWarps = 8;
constexpr int kPkThreads = kPkWarps * 32;
constexpr int kCheckBlocks = kNumSMs;  // chunk_order_kernel's grid: one flag word per CTA
constexpr unsigned kPkFull = 0xffffffffu;

template <int U> struct UnitOf;
template <> struct UnitOf<16> { using T = uint4; };
template <> struct UnitOf<8> { using T = unsigned long long; };
template <> struct UnitOf<4> { using T = uint32_t; };
template <> struct UnitOf<2> { using T = uint16_t; };
template <> struct UnitOf<1> { using T = uint8_t; };

__device__ __forceinline__ int64_t clamp64(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : (v > hi ? hi : v); }

template <class T>
__device__ __forceinline__ void warp_fill(T* __restrict__ dst, int64_t n, T v, int lane)
{
    for (int64_t k = lane; k < n; k += 32) dst[k] = v;
}

template <class T>
__device__ __forceinline__ void warp_copy(T* __restrict__ dst, const T* __restrict__ src, int64_t n, int lane)
{
    for (int64_t k = lane; k < n; k += 32) dst[k] = src[k];
}

// Every CTA of a kernel that follows chunk_order_kernel reads all flag words (L2-resident) before it starts.
__device__ __forceinline__ bool chunks_unordered(const uint32_t* __restrict__ flags)
{
    uint32_t f = 0;
    for (int i = threadIdx.x; i < kCheckBlocks; i += blockDim.x) f |= flags[i];
    return __syncthreads_or(f != 0) != 0;
}

__device__ __forceinline__ void load_chunk(const int64_t* __restrict__ pi, int64_t r, int64_t& s, int64_t& e)
{
    s = pi[2 * r];
    const int64_t c = pi[2 * r + 1];
    e = s + (c > 0 ? c : 0);
}

// flags[blockIdx.x] = 1 iff some ray of this CTA's share starts before the previous ray's chunk ends.
__global__ void __launch_bounds__(kPkThreads) chunk_order_kernel(int32_t n_rays, const int64_t* __restrict__ pi,
                                                                 uint32_t* __restrict__ flags)
{
    bool bad = false;
    for (int64_t r = 1 + (int64_t)blockIdx.x * kPkThreads + threadIdx.x; r < n_rays;
         r += (int64_t)gridDim.x * kPkThreads) {
        int64_t ps, pe, s, e;
        load_chunk(pi, r - 1, ps, pe);
        load_chunk(pi, r, s, e);
        bad |= s < pe;
    }
    const int any = __syncthreads_or(bad);
    if (threadIdx.x == 0) flags[blockIdx.x] = any ? 1u : 0u;
}

template <class T>
__global__ void __launch_bounds__(kPkThreads) fill_if_unordered_kernel(T* __restrict__ dst, int64_t n, T v,
                                                                       const uint32_t* __restrict__ flags)
{
    if (!chunks_unordered(flags)) return;
    for (int64_t k = (int64_t)blockIdx.x * kPkThreads + threadIdx.x; k < n; k += (int64_t)gridDim.x * kPkThreads)
        dst[k] = v;
}

// The range of packed positions [lo, hi) ray r writes: its chunk, clipped to [0, n), plus -- when the chunks are in
// order -- the gap up to the next chunk (and, for ray 0, the gap in front of it).
__device__ __forceinline__ void ray_span(const int64_t* __restrict__ pi, int32_t n_rays, int64_t n, int64_t r,
                                         bool ordered, int64_t s, int64_t e, int64_t& lo, int64_t& hi)
{
    if (ordered) {
        lo = r == 0 ? 0 : clamp64(s, 0, n);
        const int64_t next = r + 1 < n_rays ? pi[2 * (r + 1)] : n;
        hi = clamp64(next, lo, n);
    } else {
        lo = clamp64(s, 0, n);
        hi = clamp64(e, lo, n);
    }
}

__global__ void __launch_bounds__(kPkThreads) unpack_info_kernel(int32_t n_rays, const int64_t* __restrict__ pi,
                                                                 int64_t n, long long* __restrict__ ray_indices,
                                                                 const uint32_t* __restrict__ flags)
{
    const bool ordered = !chunks_unordered(flags);
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kPkWarps + (threadIdx.x >> 5); r < n_rays;
         r += (int64_t)gridDim.x * kPkWarps) {
        int64_t s, e, lo, hi;
        load_chunk(pi, r, s, e);
        ray_span(pi, n_rays, n, r, ordered, s, e, lo, hi);
        const int64_t a = clamp64(s, lo, hi), b = clamp64(e, a, hi);
        warp_fill(ray_indices + lo, a - lo, -1ll, lane);
        warp_fill(ray_indices + a, b - a, (long long)r, lane);
        warp_fill(ray_indices + b, hi - b, -1ll, lane);
    }
}

// padded (n_rays, S, upr units) -> packed (n, upr units); truncated rows (j >= S) and uncovered rows get zeros.
template <class T>
__global__ void __launch_bounds__(kPkThreads) pack_rows_kernel(int32_t n_rays, const int64_t* __restrict__ pi,
                                                               int64_t n, int64_t S, int64_t upr,
                                                               const T* __restrict__ padded, T* __restrict__ packed,
                                                               const uint32_t* __restrict__ flags)
{
    const bool ordered = !chunks_unordered(flags);
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kPkWarps + (threadIdx.x >> 5); r < n_rays;
         r += (int64_t)gridDim.x * kPkWarps) {
        int64_t s, e, lo, hi;
        load_chunk(pi, r, s, e);
        ray_span(pi, n_rays, n, r, ordered, s, e, lo, hi);
        const int64_t a = clamp64(s, lo, hi), b = clamp64(e, a, hi), m = clamp64(s + S, a, b);
        warp_fill(packed + lo * upr, (a - lo) * upr, T{}, lane);
        warp_copy(packed + a * upr, padded + (r * S + (a - s)) * upr, (m - a) * upr, lane);
        warp_fill(packed + m * upr, (hi - m) * upr, T{}, lane);
    }
}

// packed (n, upr units) -> padded (n_rays, S, upr units); every padded row is written, pad_row where no data lands.
template <class T>
__global__ void __launch_bounds__(kPkThreads) unpack_rows_kernel(int32_t n_rays, const int64_t* __restrict__ pi,
                                                                 int64_t n, int64_t S, int64_t upr,
                                                                 const T* __restrict__ packed,
                                                                 const T* __restrict__ pad_row,
                                                                 T* __restrict__ padded)
{
    const int lane = threadIdx.x & 31;
    const uint32_t u = (uint32_t)upr, step = 32u % u;
    const int64_t row_units = S * upr;
    for (int64_t r = (int64_t)blockIdx.x * kPkWarps + (threadIdx.x >> 5); r < n_rays;
         r += (int64_t)gridDim.x * kPkWarps) {
        int64_t s, e;
        load_chunk(pi, r, s, e);
        // rows j of this ray that have data: 0 <= j < min(count, S) and 0 <= s + j < n
        const int64_t j0 = clamp64(-s, 0, S);
        const int64_t j1 = clamp64(e - s < n - s ? e - s : n - s, j0, S);
        const int64_t k0 = j0 * upr, k1 = j1 * upr;
        T* __restrict__ dst = padded + r * row_units;
        const T* __restrict__ src = packed + s * upr;  // only dereferenced for k in [k0, k1)
        uint32_t w = (uint32_t)lane % u;                // k mod upr, kept incrementally
        for (int64_t k = lane; k < row_units; k += 32) {
            dst[k] = (k >= k0 && k < k1) ? src[k] : pad_row[w];
            w += step;
            if (w >= u) w -= u;
        }
    }
}

// Mask-addressed rows: row j of ray r is kept iff mask[r, j]; the kept rows of ray r go, in order, to packed rows
// start_r, start_r + 1, ...  kPack: padded -> packed.  !kPack: packed -> padded, zeros where the mask is false.
template <class T, bool kPack>
__global__ void __launch_bounds__(kPkThreads) masked_rows_kernel(int32_t n_rays, int64_t S, int64_t upr,
                                                                 const uint8_t* __restrict__ mask,
                                                                 const int64_t* __restrict__ pi,
                                                                 const T* __restrict__ in, T* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const unsigned below = (1u << lane) - 1u;
    for (int64_t r = (int64_t)blockIdx.x * kPkWarps + (threadIdx.x >> 5); r < n_rays;
         r += (int64_t)gridDim.x * kPkWarps) {
        int64_t q = pi[2 * r];
        for (int64_t j0 = 0; j0 < S; j0 += 32) {
            const int64_t j = j0 + lane;
            const bool keep = j < S && mask[r * S + j] != 0;
            const unsigned bits = __ballot_sync(kPkFull, keep);
            const int64_t packed_row = (q + __popc(bits & below)) * upr, padded_row = (r * S + j) * upr;
            if (kPack) {
                if (keep) {
                    const T* __restrict__ src = in + padded_row;
                    T* __restrict__ dst = out + packed_row;
#pragma unroll 1
                    for (int64_t w = 0; w < upr; ++w) dst[w] = src[w];
                }
            } else if (j < S) {
                T* __restrict__ dst = out + padded_row;
                if (keep) {
                    const T* __restrict__ src = in + packed_row;
#pragma unroll 1
                    for (int64_t w = 0; w < upr; ++w) dst[w] = src[w];
                } else {
#pragma unroll 1
                    for (int64_t w = 0; w < upr; ++w) dst[w] = T{};
                }
            }
            q += __popc(bits);
        }
    }
}

__global__ void __launch_bounds__(kPkThreads) mask_counts_kernel(int32_t n_rays, int64_t S,
                                                                 const uint8_t* __restrict__ mask,
                                                                 long long* __restrict__ counts)
{
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kPkWarps + (threadIdx.x >> 5); r < n_rays;
         r += (int64_t)gridDim.x * kPkWarps) {
        long long c = 0;
        for (int64_t j = lane; j - lane < S; j += 32)
            c += __popc(__ballot_sync(kPkFull, j < S && mask[r * S + j] != 0));
        if (lane == 0) counts[r] = c;
    }
}

}  // namespace nfa

using namespace nfa;

static inline int32_t launch_status_p()
{
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? NFA_OK : (int32_t)e;
}

// warp-per-ray grid: at most one wave of 8-warp CTAs (8 resident per SM at 256 threads)
static inline int ray_grid(int32_t n_rays)
{
    const int need = (n_rays + kPkWarps - 1) / kPkWarps;
    return need < kNumSMs * 8 ? need : kNumSMs * 8;
}

static inline int fill_grid(int64_t n)
{
    const int64_t need = (n + kPkThreads - 1) / kPkThreads;
    return (int)(need < kNumSMs * 8 ? need : kNumSMs * 8);
}

// largest copy unit (16, 8, 4, 2 or 1 bytes) dividing the row size and every pointer
static inline int unit_bytes(int64_t row_bytes, const void* a, const void* b, const void* c)
{
    const uintptr_t m = (uintptr_t)row_bytes | (uintptr_t)a | (uintptr_t)b | (uintptr_t)c;
    for (int u = 16; u > 1; u >>= 1)
        if ((m & (uintptr_t)(u - 1)) == 0) return u;
    return 1;
}

#define NFA_BY_UNIT(U, CALL)                                   \
    switch (U) {                                               \
    case 16: { using T = UnitOf<16>::T; CALL; } break;         \
    case 8: { using T = UnitOf<8>::T; CALL; } break;           \
    case 4: { using T = UnitOf<4>::T; CALL; } break;           \
    case 2: { using T = UnitOf<2>::T; CALL; } break;           \
    default: { using T = UnitOf<1>::T; CALL; } break;          \
    }

extern "C" {

int64_t nfa_chunk_order_workspace_bytes(void) { return (int64_t)kCheckBlocks * 4; }

int32_t nfa_unpack_info(int32_t n_rays, const int64_t* packed_info, int64_t n_samples, int64_t* ray_indices,
                        void* workspace, nfa_stream_t stream)
{
    if (n_rays < 0 || n_samples < 0) return NFA_ERR_ARG;
    if (n_rays == 0 || n_samples == 0) return NFA_OK;
    if (!packed_info || !ray_indices || !workspace) return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    uint32_t* flags = (uint32_t*)workspace;
    long long* out = reinterpret_cast<long long*>(ray_indices);
    chunk_order_kernel<<<kCheckBlocks, kPkThreads, 0, s>>>(n_rays, packed_info, flags);
    fill_if_unordered_kernel<long long><<<fill_grid(n_samples), kPkThreads, 0, s>>>(out, n_samples, -1ll, flags);
    unpack_info_kernel<<<ray_grid(n_rays), kPkThreads, 0, s>>>(n_rays, packed_info, n_samples, out, flags);
    return launch_status_p();
}

int32_t nfa_unpack_rows(int32_t n_rays, const int64_t* packed_info, int64_t n_packed, int64_t n_per_ray,
                        int64_t row_bytes, const void* packed, const void* pad_row, void* padded, nfa_stream_t stream)
{
    if (n_rays < 0 || n_packed < 0 || n_per_ray < 0 || row_bytes < 0) return NFA_ERR_ARG;
    if (n_rays == 0 || n_per_ray == 0 || row_bytes == 0) return NFA_OK;
    if (!packed_info || !pad_row || !padded || (n_packed > 0 && !packed)) return NFA_ERR_ARG;
    const int u = unit_bytes(row_bytes, packed, pad_row, padded);
    const int64_t upr = row_bytes / u;
    if (upr > INT32_MAX) return NFA_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    NFA_BY_UNIT(u, (unpack_rows_kernel<T><<<ray_grid(n_rays), kPkThreads, 0, s>>>(
                       n_rays, packed_info, n_packed, n_per_ray, upr, (const T*)packed, (const T*)pad_row,
                       (T*)padded)));
    return launch_status_p();
}

int32_t nfa_pack_rows(int32_t n_rays, const int64_t* packed_info, int64_t n_packed, int64_t n_per_ray,
                      int64_t row_bytes, const void* padded, void* packed, void* workspace, nfa_stream_t stream)
{
    if (n_rays < 0 || n_packed < 0 || n_per_ray < 0 || row_bytes < 0) return NFA_ERR_ARG;
    if (n_packed == 0 || row_bytes == 0) return NFA_OK;
    if (!packed || !workspace || (n_rays > 0 && !packed_info) || (n_rays > 0 && n_per_ray > 0 && !padded))
        return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    if (n_rays == 0) {  // no chunk covers anything
        const cudaError_t e = cudaMemsetAsync(packed, 0, (size_t)(n_packed * row_bytes), s);
        return e == cudaSuccess ? NFA_OK : (int32_t)e;
    }
    const int u = unit_bytes(row_bytes, padded, packed, nullptr);
    const int64_t upr = row_bytes / u;
    uint32_t* flags = (uint32_t*)workspace;
    chunk_order_kernel<<<kCheckBlocks, kPkThreads, 0, s>>>(n_rays, packed_info, flags);
    NFA_BY_UNIT(u, (fill_if_unordered_kernel<T><<<fill_grid(n_packed * upr), kPkThreads, 0, s>>>(
                       (T*)packed, n_packed * upr, T{}, flags),
                    pack_rows_kernel<T><<<ray_grid(n_rays), kPkThreads, 0, s>>>(
                       n_rays, packed_info, n_packed, n_per_ray, upr, (const T*)padded, (T*)packed, flags)));
    return launch_status_p();
}

int32_t nfa_mask_counts(int32_t n_rays, int64_t n_per_ray, const uint8_t* mask, int64_t* counts, nfa_stream_t stream)
{
    if (n_rays < 0 || n_per_ray < 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!counts || (n_per_ray > 0 && !mask)) return NFA_ERR_ARG;
    mask_counts_kernel<<<ray_grid(n_rays), kPkThreads, 0, (cudaStream_t)stream>>>(
        n_rays, n_per_ray, mask, reinterpret_cast<long long*>(counts));
    return launch_status_p();
}

static int32_t masked_rows(bool to_packed, int32_t n_rays, int64_t n_per_ray, int64_t row_bytes, const uint8_t* mask,
                           const int64_t* packed_info, const void* in, void* out, cudaStream_t s)
{
    if (n_rays < 0 || n_per_ray < 0 || row_bytes < 0) return NFA_ERR_ARG;
    if (n_rays == 0 || n_per_ray == 0 || row_bytes == 0) return NFA_OK;
    if (!mask || !packed_info || !out || (to_packed && !in)) return NFA_ERR_ARG;  // no packed rows: `in` may be NULL
    const int u = unit_bytes(row_bytes, in, out, nullptr);
    const int64_t upr = row_bytes / u;
    if (to_packed) {
        NFA_BY_UNIT(u, (masked_rows_kernel<T, true><<<ray_grid(n_rays), kPkThreads, 0, s>>>(
                           n_rays, n_per_ray, upr, mask, packed_info, (const T*)in, (T*)out)));
    } else {
        NFA_BY_UNIT(u, (masked_rows_kernel<T, false><<<ray_grid(n_rays), kPkThreads, 0, s>>>(
                           n_rays, n_per_ray, upr, mask, packed_info, (const T*)in, (T*)out)));
    }
    return launch_status_p();
}

int32_t nfa_pack_masked(int32_t n_rays, int64_t n_per_ray, int64_t row_bytes, const uint8_t* mask,
                        const int64_t* packed_info, const void* padded, void* packed, nfa_stream_t stream)
{
    return masked_rows(true, n_rays, n_per_ray, row_bytes, mask, packed_info, padded, packed, (cudaStream_t)stream);
}

int32_t nfa_unpack_masked(int32_t n_rays, int64_t n_per_ray, int64_t row_bytes, const uint8_t* mask,
                          const int64_t* packed_info, const void* packed, void* padded, nfa_stream_t stream)
{
    return masked_rows(false, n_rays, n_per_ray, row_bytes, mask, packed_info, packed, padded, (cudaStream_t)stream);
}

}  // extern "C"
