// composite.cu -- fused volume-rendering accumulation over the packed layout.
//
// One kernel computes what the reference does with ~25 ATen launches
// (/root/reference/nerfacc/volrend.py:79-164): sigma*dt, alpha, the per-ray
// exclusive scan, transmittance, weights, and the three accumulate_along_rays
// reductions (colour, opacity, depth) plus expected-depth normalisation and
// background blend; a second kernel is the matching backward.
//
// Mapping: a ray's samples are contiguous in the packed arrays, so a warp owns a
// ray and a lane owns a group of 4 consecutive samples (global index 4g .. 4g+3):
// the warp covers 128 samples per step, each lane scans its group in registers and
// one shuffle scan joins the lanes; per-lane partial sums are reduced once per ray.
// Groups are aligned to the ARRAY, not to the ray: the first / last group of a ray
// may hold samples of its neighbours, which are masked (and written element-wise).
// No atomics (deterministic, unlike the reference's index_add_), no tensor
// cores (no contraction here); the kernels are HBM-bound: 44 B/sample forward,
// 48 B/sample backward (SURVEY.md section 8d).
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/nerfacc_b200.h"
#include "sm_count.cuh"

namespace nfa {

constexpr int kWarpsPerCta = 8;
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(kFull, v, s);
    return v;
}

// inclusive scan within the warp (sum)
__device__ __forceinline__ float warp_scan_sum(float v, int lane)
{
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        const float y = __shfl_up_sync(kFull, v, s);
        if (lane >= s) v += y;
    }
    return v;
}
__device__ __forceinline__ float warp_scan_prod(float v, int lane)
{
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        const float y = __shfl_up_sync(kFull, v, s);
        if (lane >= s) v *= y;
    }
    return v;
}

struct CompositeParams {
    int32_t n_rays;
    const int64_t* packed_info;  // [R,2]
    const float* t_starts;       // density route (also depth accumulation)
    const float* t_ends;
    const float* dens;           // sigmas (density route) or alphas (alpha route)
    const float* rgbs;           // [N,3] or null
    const float* prefix_trans;   // [N] or null
    const float* bkgd;           // [3] or null
    int32_t expected_depths;
    // forward outputs (nullable)
    float* weights;
    float* trans;
    float* alphas;
    float* colors;   // [R,3]
    float* opac;     // [R]
    float* depths;   // [R]
    float* raw;      // [R,5] raw (colour, opacity, depth) sums kept for the backward
    // backward inputs (nullable)
    const float* gC;
    const float* gO;
    const float* gD;
    const float* gW;
    const float* gT;
    const float* gA;
    // backward outputs
    float* g_dens;   // [N]
    float* g_rgbs;   // [N,3] or null
};

// exp(-x) for x >= 0 through MUFU.EX2 (ex2.approx): the outputs are in [0, 1] and the absolute
// error stays ~1e-6 for the |x| <= 15 that still give a non-negligible result -- inside the 1e-5
// parity tolerance -- while the accurate expf costs ~5x the instructions in an issue-bound kernel.
__device__ __forceinline__ float exp_neg(float x) { return __expf(-x); }

constexpr float kEpsF32 = 1.1920929e-07f;  // torch.finfo(float32).eps, reference volrend.py:158

// Compile-time specialisation of the forward and backward kernels.
//   kAlpha: the alpha route (`dens` holds alphas) instead of the density route.
//   kVec:   every per-sample pointer is 16-byte aligned, so a group that lies inside the array moves as one float4
//           per array (the 12 colour floats as three).  Otherwise every group is loaded and stored element-wise, as
//           the array's last partial group always is.  The arithmetic is the same either way, so results do not
//           depend on where the inputs sit in memory.
//   kHot:   the training step: density route with colours, no prefix_trans, every forward output; in the backward,
//           upstream gradients on colours / opacities / depths only; fewer than 2^31 - 8 samples.  Every test of an
//           optional pointer folds to a constant and indices are 32-bit: these kernels are as much issue-bound as
//           HBM-bound, so instructions per sample matter.
template <bool kAlpha_, bool kVec_, bool kHot_ = false>
struct Cfg {
    static constexpr bool kAlpha = kAlpha_, kVec = kVec_, kHot = kHot_;
    using Index = std::conditional_t<kHot, int, int64_t>;
    // `has`: a pointer every hot call passes; `extra`: one no hot call passes
    static __device__ __forceinline__ bool has(const void* q) { return kHot || q != nullptr; }
    static __device__ __forceinline__ bool extra(const void* q) { return !kHot && q != nullptr; }
};
using HotCfg = Cfg<false, true, true>;

// Group g (samples 4g .. 4g+3) of a ray [start, end): the samples lo <= e < hi belong to the ray.
template <class C>
struct Span {
    using I = typename C::Index;
    I g, n_total;
    int lo, hi;
    bool valid;  // the group overlaps the ray

    __device__ __forceinline__ Span(I g_, I g_last, I start, I end, I n_total_) : g(g_), n_total(n_total_)
    {
        valid = g <= g_last;
        if constexpr (sizeof(I) == 4) {
            lo = start - 4 * g;
            hi = end - 4 * g;
        } else {  // only how the bounds compare with 0 .. 4 matters: clamp before narrowing
            lo = (int)max((I)-8, start - 4 * g);
            hi = (int)min((I)8, end - 4 * g);
        }
        if (!valid) lo = 4;
    }
    __device__ __forceinline__ bool ok(int e) const { return e >= lo && e < hi; }
    // The group lies inside the array and moves as float4.  Evaluated where it is used: computed up front, it
    // leads the compiler to keep one pointer per array live across the loop (10 more registers on the hot path).
    __device__ __forceinline__ bool full() const { return C::kVec && 4 * g + 3 < n_total; }
    __device__ __forceinline__ bool all() const { return lo <= 0 && hi >= 4 && full(); }
};

// the g-th float4 of `base`
template <class I>
__device__ __forceinline__ void ldg4(const float* base, I g, float x[4])
{
    const float4 v = __ldg(reinterpret_cast<const float4*>(base) + g);
    x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
}

template <class C>
__device__ __forceinline__ void load4(const float* base, const Span<C>& s, float x[4])
{
    if (s.full()) {
        ldg4(base, s.g, x);
    } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) x[e] = (4 * s.g + e < s.n_total) ? __ldg(base + 4 * s.g + e) : 0.f;
    }
}

template <class C>
__device__ __forceinline__ void store4(float* base, const Span<C>& s, const float x[4])
{
    if (s.all()) {
        *(reinterpret_cast<float4*>(base) + s.g) = make_float4(x[0], x[1], x[2], x[3]);
    } else {
#pragma unroll
        for (int e = 0; e < 4; ++e)
            if (s.ok(e)) base[4 * s.g + e] = x[e];
    }
}

// the inputs of one group; what is absent stays 0 (prefix_trans: 1)
struct Group {
    float ts[4], te[4], v[4], pt[4], c[12];
};

template <class C>
__device__ __forceinline__ void load_group(const CompositeParams& p, const Span<C>& s, bool colours, Group& h)
{
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        h.ts[e] = h.te[e] = h.v[e] = 0.f;
        h.pt[e] = 1.f;
    }
#pragma unroll
    for (int k = 0; k < 12; ++k) h.c[k] = 0.f;
    if (!s.valid) return;
    const bool dt = C::has(p.t_starts), pt = C::extra(p.prefix_trans);
    if (s.full()) {
        ldg4(p.dens, s.g, h.v);
        if (dt) {
            ldg4(p.t_starts, s.g, h.ts);
            ldg4(p.t_ends, s.g, h.te);
        }
        if (pt) ldg4(p.prefix_trans, s.g, h.pt);
        if (colours) {
            ldg4(p.rgbs, 3 * s.g, h.c);
            ldg4(p.rgbs, 3 * s.g + 1, h.c + 4);
            ldg4(p.rgbs, 3 * s.g + 2, h.c + 8);
        }
    } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const auto i = 4 * s.g + e;
            if (i >= s.n_total) continue;
            h.v[e] = __ldg(p.dens + i);
            if (dt) {
                h.ts[e] = __ldg(p.t_starts + i);
                h.te[e] = __ldg(p.t_ends + i);
            }
            if (pt) h.pt[e] = __ldg(p.prefix_trans + i);
            if (colours) {
                h.c[3 * e] = __ldg(p.rgbs + 3 * i);
                h.c[3 * e + 1] = __ldg(p.rgbs + 3 * i + 1);
                h.c[3 * e + 2] = __ldg(p.rgbs + 3 * i + 2);
            }
        }
    }
}

// upstream gradients on the per-sample outputs (0 where absent); unused ones are never loaded
template <class C>
__device__ __forceinline__ void load_sample_grads(const CompositeParams& p, const Span<C>& s, float gw[4],
                                                  float gt[4], float ga[4])
{
#pragma unroll
    for (int e = 0; e < 4; ++e) gw[e] = gt[e] = ga[e] = 0.f;
    if (!s.valid) return;
    if (C::extra(p.gW)) load4(p.gW, s, gw);
    if (C::extra(p.gT)) load4(p.gT, s, gt);
    if (C::extra(p.gA)) load4(p.gA, s, ga);
}

// transmittance, alpha and weight of a group's samples; `carry` is what the ray's earlier groups pass on
struct GroupFwd {
    float T[4], a[4], w[4], x[4];  // x: sigma*dt (density route) or 1-alpha (alpha route)
};

template <class C>
__device__ __forceinline__ void group_forward(const Group& h, const Span<C>& s, int lane, float& carry,
                                              GroupFwd& q)
{
    if constexpr (!C::kAlpha) {
        // reference volrend.py:271-275
        float run = 0.f, incl[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            q.x[e] = s.ok(e) ? h.v[e] * (h.te[e] - h.ts[e]) : 0.f;
            run += q.x[e];
            incl[e] = run;
        }
        const float tot = warp_scan_sum(run, lane);  // inclusive over lanes
        const float off = carry + (tot - run);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            q.T[e] = exp_neg(off + (incl[e] - q.x[e])) * h.pt[e];
            q.a[e] = 1.0f - exp_neg(q.x[e]);
            q.w[e] = q.T[e] * q.a[e];
        }
        carry += __shfl_sync(kFull, tot, 31);
    } else {
        // reference volrend.py:211-213
        float run = 1.f, excl[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            q.x[e] = s.ok(e) ? 1.0f - h.v[e] : 1.0f;
            excl[e] = run;
            run *= q.x[e];
        }
        const float tot = warp_scan_prod(run, lane);
        float off = __shfl_up_sync(kFull, tot, 1);
        if (lane == 0) off = 1.0f;
        off *= carry;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            q.T[e] = off * excl[e] * h.pt[e];
            q.a[e] = h.v[e];
            q.w[e] = q.T[e] * q.a[e];
        }
        carry *= __shfl_sync(kFull, tot, 31);
    }
}

template <class C>
__global__ void __launch_bounds__(kWarpsPerCta * 32) composite_fwd_kernel(const CompositeParams p,
                                                                           typename C::Index n_total)
{
    using I = typename C::Index;
    const int lane = threadIdx.x & 31;
    const bool accumulate = C::has(p.opac) || C::has(p.colors) || C::has(p.depths) || C::has(p.raw);
    // persistent warps: ray = global warp id, then stride by the number of warps in the grid
    for (int r = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5); r < p.n_rays; r += gridDim.x * kWarpsPerCta) {
        const longlong2 pi = *reinterpret_cast<const longlong2*>(p.packed_info + 2 * (int64_t)r);
        const I start = (I)pi.x, end = (I)(pi.x + pi.y);
        float carry = C::kAlpha ? 1.0f : 0.0f;
        float aO = 0.f, aD = 0.f, aC0 = 0.f, aC1 = 0.f, aC2 = 0.f;
        if (end > start) {
            const I g_last = (end - 1) >> 2;
            for (I gb = start >> 2; gb <= g_last; gb += 32) {
                const Span<C> s(gb + lane, g_last, start, end, n_total);
                Group h;
                load_group(p, s, C::has(p.rgbs), h);
                GroupFwd q;
                group_forward(h, s, lane, carry, q);
                if (!s.valid) continue;
                if (C::has(p.weights)) store4(p.weights, s, q.w);
                if (C::has(p.trans)) store4(p.trans, s, q.T);
                if (C::has(p.alphas)) store4(p.alphas, s, q.a);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float w = s.ok(e) ? q.w[e] : 0.f;
                    aO += w;
                    aD += w * ((h.ts[e] + h.te[e]) * 0.5f);
                    aC0 += w * h.c[3 * e];
                    aC1 += w * h.c[3 * e + 1];
                    aC2 += w * h.c[3 * e + 2];
                }
            }
        }
        if (!accumulate) continue;
        aO = warp_sum(aO);
        aD = warp_sum(aD);
        aC0 = warp_sum(aC0);
        aC1 = warp_sum(aC1);
        aC2 = warp_sum(aC2);
        if (lane == 0) {
            if (C::has(p.raw)) {
                float* w = p.raw + 5 * (int64_t)r;
                w[0] = aC0; w[1] = aC1; w[2] = aC2; w[3] = aO; w[4] = aD;
            }
            if (C::has(p.opac)) p.opac[r] = aO;
            if (C::has(p.depths)) p.depths[r] = p.expected_depths ? aD / fmaxf(aO, kEpsF32) : aD;
            if (C::has(p.colors)) {
                float b0 = 0.f, b1 = 0.f, b2 = 0.f;
                if (p.bkgd) {
                    const float k = 1.0f - aO;
                    b0 = p.bkgd[0] * k; b1 = p.bkgd[1] * k; b2 = p.bkgd[2] * k;
                }
                p.colors[3 * (int64_t)r + 0] = aC0 + b0;
                p.colors[3 * (int64_t)r + 1] = aC1 + b1;
                p.colors[3 * (int64_t)r + 2] = aC2 + b2;
            }
        }
    }
}

// Backward.  With g_i = dL/dw_i = gC'.c_i + gO' + gD'.m_i + gW_i  (primes: after
// undoing background blend / depth normalisation) the reference's autograd graph
// (volrend.py:271-277,375; scan.py:419-424) reduces to
//   density: dL/dsigma_i = d_i [ (g_i T_i + gA_i)(1-a_i) - S_i ]
//   alpha  : dL/dalpha_i = g_i T_i + gA_i - S_i / max(1-a_i, 1e-10)      (scan.cu:299)
//   S_i = sum_{k>i} (g_k w_k + gT_k T_k),     dL/dc_i = w_i gC'
// S_i is taken as Total - inclusive prefix, so the ray is walked once, forwards,
// re-computing T/w from the inputs instead of re-reading saved tensors.
template <class C>
__global__ void __launch_bounds__(kWarpsPerCta * 32) composite_bwd_kernel(const CompositeParams p,
                                                                           typename C::Index n_total)
{
    using I = typename C::Index;
    const int lane = threadIdx.x & 31;
    for (int r = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5); r < p.n_rays; r += gridDim.x * kWarpsPerCta) {
        const longlong2 pi = *reinterpret_cast<const longlong2*>(p.packed_info + 2 * (int64_t)r);
        const I start = (I)pi.x, end = (I)(pi.x + pi.y);
        if (end <= start) continue;

        // upstream per-ray gradients, moved back to the raw sums
        float gc0 = 0.f, gc1 = 0.f, gc2 = 0.f, go = 0.f, gd = 0.f;
        if (p.gC) {
            gc0 = p.gC[3 * (int64_t)r]; gc1 = p.gC[3 * (int64_t)r + 1]; gc2 = p.gC[3 * (int64_t)r + 2];
        }
        if (p.gO) go = p.gO[r];
        if (p.gD) gd = p.gD[r];
        float rC0 = 0.f, rC1 = 0.f, rC2 = 0.f, rO = 0.f, rD = 0.f;
        if (C::has(p.raw)) {
            const float* w = p.raw + 5 * (int64_t)r;
            rC0 = w[0]; rC1 = w[1]; rC2 = w[2]; rO = w[3]; rD = w[4];
        }
        if (p.bkgd) go -= gc0 * p.bkgd[0] + gc1 * p.bkgd[1] + gc2 * p.bkgd[2];
        if (p.expected_depths && p.gD) {
            if (rO > kEpsF32) {
                go -= gd * rD / (rO * rO);
                gd = gd / rO;
            } else {
                gd = gd / kEpsF32;
            }
        }
        // the hot path loads colours even without gC: they are multiplied by zero
        const bool have_rgb = C::kHot || (p.rgbs != nullptr && p.gC != nullptr);
        const I g_first = start >> 2, g_last = (end - 1) >> 2;

        // Total = sum_k (g_k w_k + gT_k T_k): from the saved sums, or with gradients on weights / trans a first pass
        float total;
        if (C::has(p.raw) && !C::extra(p.gW) && !C::extra(p.gT)) {
            total = gc0 * rC0 + gc1 * rC1 + gc2 * rC2 + go * rO + gd * rD;
        } else {
            float carry = C::kAlpha ? 1.0f : 0.0f;
            float acc = 0.f;
            for (I gb = g_first; gb <= g_last; gb += 32) {
                const Span<C> s(gb + lane, g_last, start, end, n_total);
                Group h;
                load_group(p, s, false, h);  // colours per sample below: as a group they cost 7 more registers
                GroupFwd q;
                group_forward(h, s, lane, carry, q);
                float gw[4], gt[4], ga[4];
                load_sample_grads(p, s, gw, gt, ga);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (!s.ok(e)) continue;
                    const I i = 4 * s.g + e;
                    float gg = go + gd * ((h.ts[e] + h.te[e]) * 0.5f);
                    if (have_rgb)
                        gg += gc0 * __ldg(p.rgbs + 3 * i) + gc1 * __ldg(p.rgbs + 3 * i + 1) +
                              gc2 * __ldg(p.rgbs + 3 * i + 2);
                    if (C::extra(p.gW)) gg += gw[e];
                    float t = gg * q.w[e];
                    if (C::extra(p.gT)) t += gt[e] * q.T[e];
                    acc += t;
                }
            }
            total = warp_sum(acc);
        }

        float carry = C::kAlpha ? 1.0f : 0.0f;
        float pcarry = 0.f;
        for (I gb = g_first; gb <= g_last; gb += 32) {
            const Span<C> s(gb + lane, g_last, start, end, n_total);
            Group h;
            load_group(p, s, have_rgb, h);
            float gw[4], gt[4], ga[4];
            load_sample_grads(p, s, gw, gt, ga);
            GroupFwd q;
            group_forward(h, s, lane, carry, q);
            // outside the hot path the per-sample gradients are added whether given or not (0 when absent)
            float gg[4], incl[4];
            float run = 0.f;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                gg[e] = go + gd * ((h.ts[e] + h.te[e]) * 0.5f) + gc0 * h.c[3 * e] + gc1 * h.c[3 * e + 1] +
                        gc2 * h.c[3 * e + 2];
                if (!C::kHot) gg[e] += gw[e];
                float term = gg[e] * q.w[e];
                if (!C::kHot) term += gt[e] * q.T[e];
                run += s.ok(e) ? term : 0.f;
                incl[e] = run;
            }
            const float tot = warp_scan_sum(run, lane);
            const float off = pcarry + (tot - run);
            pcarry += __shfl_sync(kFull, tot, 31);
            if (!s.valid) continue;
            float gi[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float suffix = total - (off + incl[e]);
                if constexpr (!C::kAlpha) {
                    float gT = gg[e] * q.T[e];
                    if (!C::kHot) gT += ga[e];
                    gi[e] = (h.te[e] - h.ts[e]) * (gT * (1.0f - q.a[e]) - suffix);
                } else {
                    gi[e] = gg[e] * q.T[e] + ga[e] - suffix / fmaxf(q.x[e], 1e-10f);
                }
            }
            store4(p.g_dens, s, gi);
            if (!C::has(p.g_rgbs)) continue;
            if (s.all()) {
                float4* dst = reinterpret_cast<float4*>(p.g_rgbs) + 3 * s.g;
                dst[0] = make_float4(q.w[0] * gc0, q.w[0] * gc1, q.w[0] * gc2, q.w[1] * gc0);
                dst[1] = make_float4(q.w[1] * gc1, q.w[1] * gc2, q.w[2] * gc0, q.w[2] * gc1);
                dst[2] = make_float4(q.w[2] * gc2, q.w[3] * gc0, q.w[3] * gc1, q.w[3] * gc2);
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (!s.ok(e)) continue;
                    const I i = 4 * s.g + e;
                    p.g_rgbs[3 * i + 0] = q.w[e] * gc0;
                    p.g_rgbs[3 * i + 1] = q.w[e] * gc1;
                    p.g_rgbs[3 * i + 2] = q.w[e] * gc2;
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------
// accumulate_along_rays (reference volrend.py:497-561), packed segments
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kWarpsPerCta * 32) accumulate_fwd_kernel(
    int32_t n_rays, const int64_t* __restrict__ packed_info, const float* __restrict__ weights,
    const float* __restrict__ values, int32_t dim, float* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    if (r >= n_rays) return;
    const longlong2 pi = *reinterpret_cast<const longlong2*>(packed_info + 2 * (int64_t)r);
    const int64_t start = pi.x, n = pi.y;
    if (values == nullptr) {
        float acc = 0.f;
        for (int64_t j = lane; j < n; j += 32) acc += __ldg(weights + start + j);
        acc = warp_sum(acc);
        if (lane == 0) out[r] = acc;
        return;
    }
    // one pass per channel: lanes stride over the ray's samples (weights stay in L1)
    for (int c = 0; c < dim; ++c) {
        float acc = 0.f;
        for (int64_t j = lane; j < n; j += 32) acc += __ldg(weights + start + j) * __ldg(values + (start + j) * dim + c);
        acc = warp_sum(acc);
        if (lane == 0) out[(int64_t)r * dim + c] = acc;
    }
}

// generic fallback for ungrouped ray_indices: float atomics like index_add_
__global__ void __launch_bounds__(256) accumulate_atomic_kernel(
    int64_t n, const int64_t* __restrict__ ray_indices, const float* __restrict__ weights,
    const float* __restrict__ values, int32_t dim, float* __restrict__ out)
{
    const int64_t total = n * dim;
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total; f += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = f / dim;
        const int c = (int)(f - i * dim);
        const float v = values ? weights[i] * values[f] : weights[i];
        atomicAdd(out + ray_indices[i] * dim + c, v);
    }
}

// backward of accumulate: g_w[i] = sum_c gout[ray, c] * v[i, c];  g_v[i, c] = w[i] * gout[ray, c]
__global__ void __launch_bounds__(256) accumulate_bwd_kernel(
    int64_t n, const int64_t* __restrict__ ray_indices, const float* __restrict__ weights,
    const float* __restrict__ values, int32_t dim, const float* __restrict__ gout, float* __restrict__ g_w,
    float* __restrict__ g_v)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = ray_indices[i];
        const float w = weights[i];
        float acc = 0.f;
        for (int c = 0; c < dim; ++c) {
            const float g = gout[r * dim + c];
            if (values) {
                acc += g * values[i * dim + c];
                if (g_v) g_v[i * dim + c] = w * g;
            } else {
                acc += g;
            }
        }
        if (g_w) g_w[i] = acc;
    }
}

}  // namespace nfa

using namespace nfa;

// persistent grid: as many CTAs as are resident at once (occupancy x SM count), never more than one warp per ray
template <class Kernel>
static inline int persistent_grid(Kernel k, int32_t n_rays)
{
    int per_sm = 0, dev = 0, sms = kNumSMs;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kWarpsPerCta * 32, 0) != cudaSuccess || per_sm < 1)
        per_sm = 2;
    const int need = (n_rays + kWarpsPerCta - 1) / kWarpsPerCta;
    const int cap = per_sm * sms;
    return need < cap ? need : cap;
}

static inline int32_t launch_status_c()
{
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? NFA_OK : (int32_t)e;
}

template <class I>
static inline void launch(void (*kernel)(CompositeParams, I), const CompositeParams& p, int32_t n_rays,
                          int64_t n_samples, cudaStream_t s)
{
    kernel<<<persistent_grid(kernel, n_rays), kWarpsPerCta * 32, 0, s>>>(p, (I)n_samples);
}

extern "C" {

int32_t nfa_composite_fwd(int32_t n_rays, int64_t n_samples, const int64_t* packed_info, const float* t_starts,
                          const float* t_ends,
                          const float* sigmas_or_alphas, int32_t from_alpha, const float* rgbs,
                          const float* prefix_trans, const float* bkgd, int32_t expected_depths, float* weights,
                          float* trans, float* alphas, float* colors, float* opacities, float* depths, float* raw,
                          nfa_stream_t stream)
{
    if (n_rays < 0 || n_samples < 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!packed_info || !sigmas_or_alphas) return NFA_ERR_ARG;
    if (!from_alpha && (!t_starts || !t_ends)) return NFA_ERR_ARG;
    if ((t_starts == nullptr) != (t_ends == nullptr)) return NFA_ERR_ARG;
    if ((((uintptr_t)packed_info) & 15u) != 0) return NFA_ERR_ARG;
    CompositeParams p = {};
    p.n_rays = n_rays;
    p.packed_info = packed_info;
    p.t_starts = t_starts;
    p.t_ends = t_ends;
    p.dens = sigmas_or_alphas;
    p.rgbs = rgbs;
    p.prefix_trans = prefix_trans;
    p.bkgd = bkgd;
    p.expected_depths = expected_depths;
    p.weights = weights;
    p.trans = trans;
    p.alphas = alphas;
    p.colors = colors;
    p.opac = opacities;
    p.depths = depths;
    p.raw = raw;
    const uintptr_t al = (uintptr_t)t_starts | (uintptr_t)t_ends | (uintptr_t)sigmas_or_alphas | (uintptr_t)rgbs |
                         (uintptr_t)prefix_trans | (uintptr_t)weights | (uintptr_t)trans | (uintptr_t)alphas;
    const cudaStream_t s = (cudaStream_t)stream;
    const bool aligned = (al & 15u) == 0 && n_samples > 0;
    const bool hot = aligned && !from_alpha && rgbs && !prefix_trans && weights && trans && alphas && colors &&
                     opacities && depths && raw && n_samples < (int64_t)0x7fffffff - 8;
    if (hot) launch(composite_fwd_kernel<HotCfg>, p, n_rays, n_samples, s);
    else if (aligned && from_alpha) launch(composite_fwd_kernel<Cfg<true, true>>, p, n_rays, n_samples, s);
    else if (aligned) launch(composite_fwd_kernel<Cfg<false, true>>, p, n_rays, n_samples, s);
    else if (from_alpha) launch(composite_fwd_kernel<Cfg<true, false>>, p, n_rays, n_samples, s);
    else launch(composite_fwd_kernel<Cfg<false, false>>, p, n_rays, n_samples, s);
    return launch_status_c();
}

int32_t nfa_composite_bwd(int32_t n_rays, int64_t n_samples, const int64_t* packed_info, const float* t_starts,
                          const float* t_ends,
                          const float* sigmas_or_alphas, int32_t from_alpha, const float* rgbs,
                          const float* prefix_trans, const float* bkgd, int32_t expected_depths, const float* raw,
                          const float* g_colors, const float* g_opacities, const float* g_depths,
                          const float* g_weights, const float* g_trans, const float* g_alphas, float* g_in,
                          float* g_rgbs, nfa_stream_t stream)
{
    if (n_rays < 0 || n_samples < 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!packed_info || !sigmas_or_alphas || !g_in) return NFA_ERR_ARG;
    if (!from_alpha && (!t_starts || !t_ends)) return NFA_ERR_ARG;
    if ((t_starts == nullptr) != (t_ends == nullptr)) return NFA_ERR_ARG;
    if ((g_colors || g_opacities || g_depths) && !raw) return NFA_ERR_ARG;
    if ((((uintptr_t)packed_info) & 15u) != 0) return NFA_ERR_ARG;
    CompositeParams p = {};
    p.n_rays = n_rays;
    p.packed_info = packed_info;
    p.t_starts = t_starts;
    p.t_ends = t_ends;
    p.dens = sigmas_or_alphas;
    p.rgbs = rgbs;
    p.prefix_trans = prefix_trans;
    p.bkgd = bkgd;
    p.expected_depths = expected_depths;
    p.raw = const_cast<float*>(raw);
    p.gC = g_colors;
    p.gO = g_opacities;
    p.gD = g_depths;
    p.gW = g_weights;
    p.gT = g_trans;
    p.gA = g_alphas;
    p.g_dens = g_in;
    p.g_rgbs = g_rgbs;
    const uintptr_t al = (uintptr_t)t_starts | (uintptr_t)t_ends | (uintptr_t)sigmas_or_alphas | (uintptr_t)rgbs |
                         (uintptr_t)prefix_trans | (uintptr_t)g_weights | (uintptr_t)g_trans | (uintptr_t)g_alphas |
                         (uintptr_t)g_in | (uintptr_t)g_rgbs;
    const cudaStream_t s = (cudaStream_t)stream;
    const bool aligned = (al & 15u) == 0 && n_samples > 0;
    const bool hot = aligned && !from_alpha && rgbs && g_rgbs && raw && !prefix_trans && !g_weights && !g_trans &&
                     !g_alphas && n_samples < (int64_t)0x7fffffff - 8;
    if (hot) launch(composite_bwd_kernel<HotCfg>, p, n_rays, n_samples, s);
    else if (aligned && from_alpha) launch(composite_bwd_kernel<Cfg<true, true>>, p, n_rays, n_samples, s);
    else if (aligned) launch(composite_bwd_kernel<Cfg<false, true>>, p, n_rays, n_samples, s);
    else if (from_alpha) launch(composite_bwd_kernel<Cfg<true, false>>, p, n_rays, n_samples, s);
    else launch(composite_bwd_kernel<Cfg<false, false>>, p, n_rays, n_samples, s);
    return launch_status_c();
}

int32_t nfa_accumulate_fwd(int32_t n_rays, const int64_t* packed_info, const float* weights, const float* values,
                           int32_t dim, float* out, nfa_stream_t stream)
{
    if (n_rays < 0 || dim <= 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!packed_info || !weights || !out) return NFA_ERR_ARG;
    if (values == nullptr && dim != 1) return NFA_ERR_ARG;
    if ((((uintptr_t)packed_info) & 15u) != 0) return NFA_ERR_ARG;
    const int blocks = (n_rays + kWarpsPerCta - 1) / kWarpsPerCta;
    accumulate_fwd_kernel<<<blocks, kWarpsPerCta * 32, 0, (cudaStream_t)stream>>>(n_rays, packed_info, weights, values,
                                                                                 dim, out);
    return launch_status_c();
}

int32_t nfa_accumulate_atomic(int64_t n, const int64_t* ray_indices, const float* weights, const float* values,
                              int32_t dim, float* out, nfa_stream_t stream)
{
    if (n < 0 || dim <= 0) return NFA_ERR_ARG;
    if (n == 0) return NFA_OK;
    if (!ray_indices || !weights || !out) return NFA_ERR_ARG;
    if (values == nullptr && dim != 1) return NFA_ERR_ARG;
    const int64_t total = n * dim;
    const int blocks = (int)((total + 255) / 256 < kNumSMs * 16 ? (total + 255) / 256 : kNumSMs * 16);
    accumulate_atomic_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(n, ray_indices, weights, values, dim, out);
    return launch_status_c();
}

int32_t nfa_accumulate_bwd(int64_t n, const int64_t* ray_indices, const float* weights, const float* values,
                           int32_t dim, const float* g_out, float* g_weights, float* g_values, nfa_stream_t stream)
{
    if (n < 0 || dim <= 0) return NFA_ERR_ARG;
    if (n == 0) return NFA_OK;
    if (!ray_indices || !weights || !g_out) return NFA_ERR_ARG;
    if (values == nullptr && (dim != 1 || g_values)) return NFA_ERR_ARG;
    const int blocks = (int)((n + 255) / 256 < kNumSMs * 16 ? (n + 255) / 256 : kNumSMs * 16);
    accumulate_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(n, ray_indices, weights, values, dim, g_out,
                                                                    g_weights, g_values);
    return launch_status_c();
}

}  // extern "C"
