// vis_block.cuh -- one 32-sample block of the visibility filter's transmittance scan.
//
// Shared by vis_mask_kernel (the one-shot filter of OccGridEstimator.sampling) and vis_rounds_step_kernel
// (OccGridEstimator.sampling_until_opaque), so that both compute every T, alpha and keep bit with the same
// arithmetic in the same order.  A ray's samples are scanned in blocks of 32 aligned to its first sample, with the
// previous blocks' total carried from one block to the next (`carry`).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace nfa {

// exp as the reference evaluates it: ATen's exp kernel calls the CUDA math library's expf (not the ex2.approx
// shortcut): the keep / drop decision compares T and alpha with thresholds, so the last bit matters.
__device__ __forceinline__ float vis_exp_neg(float x) { return expf(-x); }

// Inclusive scan of one 32-element block in the summation ORDER of the reference's packed scan kernel
// (include/utils_scan.cuh:146-263, launched 16 x 32 => blocks of 2 x 16 = 32 elements): the running total of the
// previous blocks is folded into element 0, then a Brent-Kung up-sweep / down-sweep.  Float addition is not
// associative, and `sampling(sigma_fn=...)` thresholds the result, so the tree is reproduced step by step
// (9 shuffles instead of the 5 of a Kogge-Stone scan; the filter is memory-bound).
template <bool kProd>
__device__ __forceinline__ float ref_block_scan(float x, float carry, int lane)
{
    if (lane == 0) x = kProd ? x * carry : x + carry;  // utils_scan.cuh:196-198
#pragma unroll
    for (int d = 1; d <= 16; d <<= 1) {  // up-sweep, :203-209
        const float y = __shfl_up_sync(0xffffffffu, x, d);
        if (((lane + 1) & (2 * d - 1)) == 0) x = kProd ? y * x : y + x;
    }
#pragma unroll
    for (int d = 8; d >= 1; d >>= 1) {  // down-sweep, :212-218
        const float y = __shfl_up_sync(0xffffffffu, x, d);
        if (((lane + 1) & (2 * d - 1)) == d && lane + 1 > d) x = kProd ? y * x : y + x;
    }
    return x;
}

// The blocks of `n` consecutive samples of one ray, called by all 32 lanes of a warp: sample s (0 <= s < n) has
// the interval t_starts[start + s] .. t_ends[start + s] and the density (or alpha) dens[start + s], and its keep bit
// goes to mask[start + s + mask_shift].  The blocks are aligned to sample 0.  `carry` is the total of the ray's
// blocks before these (0 for densities, 1 for alphas before the ray's first block) and leaves as the total including
// them.  Returns the number of samples kept: T >= early_stop_eps and (alpha_thre <= 0 or alpha >= alpha_thre).
//
// Once the carry fails `T >= early_stop_eps` (T = exp(-carry) for densities, carry for alphas), every later sample of
// the ray fails it too as long as densities are >= 0 (alphas in [0, 1]): each later exclusive value is a rounded sum
// (product) that includes the carry and terms >= 0 (factors in [0, 1]), so it is >= (<=) the carry, and
// vis_exp_neg does not increase (tests/test_gpu_vis_rounds.py pins that for every float).
//
// The order of the statements, and of the three pointers below, decides how nvcc schedules vis_mask_kernel's loads;
// compare its SASS (cuobjdump -sass) before and after an edit.
template <bool kAlpha>
__device__ __forceinline__ unsigned vis_blocks(const float* t_starts, const float* t_ends, const float* dens,
                                               int64_t start, int64_t n, int lane, float& carry, float early_stop_eps,
                                               float alpha_thre, uint8_t* mask, int64_t mask_shift)
{
    unsigned kept = 0;
    for (int64_t base = 0; base < n; base += 32) {
        const int64_t i = start + base + lane;
        const bool valid = base + lane < n;
        float T, a;
        if (!kAlpha) {
            // volrend.py:271-275: sigmas_dt = sigmas * (t_ends - t_starts); alphas = 1 - exp(-sigmas_dt);
            // trans = exp(-exclusive_sum(sigmas_dt))
            const float *ps = t_starts + i, *pe = t_ends + i, *pd = dens + i;
            const float sd = valid ? __fmul_rn(__ldg(pd), __fsub_rn(__ldg(pe), __ldg(ps))) : 0.f;
            const float incl = ref_block_scan<false>(sd, carry, lane);
            float excl = __shfl_up_sync(0xffffffffu, incl, 1);
            if (lane == 0) excl = carry;
            T = vis_exp_neg(excl);
            a = __fsub_rn(1.0f, vis_exp_neg(sd));
            carry = __shfl_sync(0xffffffffu, incl, 31);
        } else {
            // volrend.py:208-210: trans = exclusive_prod(1 - alphas)
            a = valid ? __ldg(dens + i) : 0.f;
            const float incl = ref_block_scan<true>(valid ? __fsub_rn(1.0f, a) : 1.0f, carry, lane);
            float excl = __shfl_up_sync(0xffffffffu, incl, 1);
            if (lane == 0) excl = carry;
            T = excl;
            carry = __shfl_sync(0xffffffffu, incl, 31);
        }
        const bool keep = valid && (T >= early_stop_eps) && (!(alpha_thre > 0.0f) || a >= alpha_thre);
        if (valid) mask[i + mask_shift] = keep ? 1 : 0;
        kept += __popc(__ballot_sync(0xffffffffu, keep));
    }
    return kept;
}

// Would the ray's next sample, after blocks totalling `carry`, pass T >= early_stop_eps?
template <bool kAlpha>
__device__ __forceinline__ bool vis_next_passes(float carry, float early_stop_eps)
{
    return (kAlpha ? carry : vis_exp_neg(carry)) >= early_stop_eps;
}

}  // namespace nfa
