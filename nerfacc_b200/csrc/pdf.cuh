// pdf.cuh -- per-sample arithmetic of inverse-transform ("importance") sampling, searchsorted and the proposal loss.
//
// Behaviour follows /root/reference/nerfacc/cuda/csrc/pdf.cu:22-63 (bound searches), :97-166
// (one sample from a piecewise-linear CDF), :168-243 (edges between neighbouring samples) and the
// cuRAND Philox4x32-10 stream the reference draws its per-ray jitter from (curand_init(seed,
// ray, offset) + curand_uniform, pdf.cu:139-145).  Floating-point contraction is written out the
// way nvcc/ptxas fuse the reference (read from its SASS): `u` and `t` are one FMA each,
// everything else is a plain rounded op.  Host+device so tests/host_sim can run it on the CPU.
#pragma once

#include <stdint.h>

#include "nfa_math.cuh"

namespace nfa {

// first index in [start, end) whose value is > v (end if none); same probe order as pdf.cu:43-63
template <class Index>
NFA_HD Index upper_bound_f(const float* a, Index start, Index end, float v)
{
    while (start < end) {
        const Index mid = start + ((end - start) >> 1);
        if (!(a[mid] > v)) start = mid + 1;
        else end = mid;
    }
    return start;
}

// searchsorted's pair for one query value against key edges [base, last]: key[left] <= v < key[right], both
// clipped to the range (pdf.cu:247-287)
template <class Index>
NFA_HD void search_ids(const float* a, Index base, Index last, float v, Index& left, Index& right)
{
    const Index pos = upper_bound_f<Index>(a, base, last, v);
    left = pos - 1 < last ? pos - 1 : last;
    if (left < base) left = base;
    right = pos < last ? pos : last;
    if (right < base) right = base;
}

// Proposal loss of one query interval (estimators/prop_net.py `_pdf_loss_torch`, the reference's prop_net.py:232-256):
// w = cq[j+1] - cq[j], wo = ck[R_j] - ck[L_j], loss = clip(w - wo, min=0) ** 2 / (w + eps), every op rounded as ATen
// rounds it.  clip keeps a NaN (`d < 0` is false for it); `eps` is the Python scalar rounded to float, as ATen does.
NFA_HD float pdf_loss_term(float w, float wo, float eps)
{
    const float d = f_sub(w, wo);
    const float c = d < 0.f ? 0.f : d;
    return f_div(f_mul(c, c), f_add(w, eps));
}

// d loss / d wo for the upstream gradient g, in the order ATen's autograd chain evaluates it (div, pow 2, clip, sub):
// where(d >= 0, -((g / (w + eps)) * (2 * c)), 0).  Key edge R_j receives this, key edge L_j its negation.
NFA_HD float pdf_loss_grad_wo(float w, float wo, float eps, float g)
{
    const float d = f_sub(w, wo);
    if (!(d >= 0.f)) return 0.f;
    return -f_mul(f_div(g, f_add(w, eps)), f_mul(2.f, d));  // c == d here
}

// Sum of the terms of the intervals j with ids[j] == k, in ascending j from +0: one key edge's share of one of the two
// scatter_adds of ATen's gather backward.  `sorted`: ids do not decrease along j, so those intervals are the run that
// starts at the first ids[j] >= k.
NFA_HD float pdf_loss_fold(const int32_t* ids, const float* t, int32_t n, int32_t k, bool sorted, bool negate)
{
    int32_t j = 0;
    if (sorted) {
        int32_t hi = n;
        while (j < hi) {
            const int32_t mid = j + ((hi - j) >> 1);
            if (ids[mid] < k) j = mid + 1;
            else hi = mid;
        }
    }
    float s = 0.f;
    for (; j < n; ++j) {
        const int32_t id = ids[j];
        if (id == k) s = f_add(s, negate ? -t[j] : t[j]);
        else if (sorted && id > k) break;
    }
    return s;
}

// number of chunk starts <= item (pdf.cu:65-80); the owning chunk is this minus one
NFA_HD int32_t chunk_upper_bound(const int64_t* packed_info, int32_t n_chunks, int64_t item)
{
    int32_t start = 0, end = n_chunks;
    while (start < end) {
        const int32_t mid = start + ((end - start) >> 1);
        if (!(packed_info[2 * (int64_t)mid] > item)) start = mid + 1;
        else end = mid;
    }
    return start;
}

NFA_HD uint32_t mul_hi_u32(uint32_t a, uint32_t b)
{
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}

// Philox4x32-10 (Salmon et al., SC'11) with cuRAND's state layout: key = seed, counter =
// (offset/4 as 64 bits, subsequence as 64 bits); returns output word (offset & 3).  For offsets that
// are multiples of 4 (torch's generator hands those out) this is what
// curand_init(seed, subsequence, offset) followed by one curand() call yields.
NFA_HD uint32_t philox_word(uint64_t seed, uint64_t subsequence, uint64_t offset)
{
    uint32_t c0 = (uint32_t)(offset >> 2), c1 = (uint32_t)(offset >> 34);
    uint32_t c2 = (uint32_t)subsequence, c3 = (uint32_t)(subsequence >> 32);
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = mul_hi_u32(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = mul_hi_u32(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    const uint32_t w = (uint32_t)(offset & 3u);
    return w == 0 ? c0 : (w == 1 ? c1 : (w == 2 ? c2 : c3));
}

// curand_uniform: (0, 1]
NFA_HD float philox_uniform(uint64_t seed, uint64_t subsequence, uint64_t offset)
{
    return f_fma((float)philox_word(seed, subsequence, offset), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
}

// Position of sample `sid` on the CDF axis (pdf.cu:135-146).
template <class Index>
NFA_HD float is_u(float u_floor, float u_step, Index sid, float bias)
{
    return f_fma(f_add((float)sid, bias), u_step, u_floor);
}

// Invert the piecewise-linear CDF at u over edges [base, last] (pdf.cu:148-165).
template <class Index>
NFA_HD float is_invert(const float* cdfs, const float* vals, Index base, Index last, float u)
{
    const Index p = upper_bound_f<Index>(cdfs, base, last, u);
    Index p0 = p - 1 < last ? p - 1 : last;
    if (p0 < base) p0 = base;
    Index p1 = p < last ? p : last;
    if (p1 < base) p1 = base;
    const float u_lower = cdfs[p0], u_upper = cdfs[p1];
    const float t_lower = vals[p0], t_upper = vals[p1];
    const float du = f_sub(u_upper, u_lower);
    if (du < 1e-10f) return f_mul(f_add(t_lower, t_upper), 0.5f);
    const float scaling = f_div(f_sub(t_upper, t_lower), du);
    return f_fma(f_sub(u, u_lower), scaling, t_lower);
}

// Edge k (0..n) between the n sample centres ts[0..n) of one ray (pdf.cu:203-241).  n == 1 is
// undefined in the reference (it reads the next ray's first sample and never writes the right edge);
// here a single sample spans the whole input range.
template <class Index>
NFA_HD float is_edge(const float* ts, Index n, Index k, float t_min, float t_max)
{
    if (n == 1) return k == 0 ? t_min : t_max;
    if (k == 0) {
        const float t = ts[0];
        return f_max(f_sub(t, f_mul(f_sub(ts[1], t), 0.5f)), t_min);
    }
    if (k == n) {
        const float t = ts[n - 1];
        return f_min(f_add(t, f_mul(f_sub(t, ts[n - 2]), 0.5f)), t_max);
    }
    return f_mul(f_add(ts[k], ts[k - 1]), 0.5f);
}

// s in [0,1] -> t (estimators/prop_net.py:215-229 `_transform_stot`, evaluated the way ATen does:
// every op rounded separately).  lindisp: 1 / (s * (1/far) + (1 - s) * (1/near)).
NFA_HD float stot(float s, float s_min, float s_max, bool lindisp)
{
    const float x = f_add(f_mul(s, s_max), f_mul(f_sub(1.0f, s), s_min));
    return lindisp ? f_div(1.0f, x) : x;
}

}  // namespace nfa
