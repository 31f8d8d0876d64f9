// pdf.cu -- importance (inverse-transform) sampling along rays and per-ray searchsorted.
//
// replaces (paths relative to /root/reference):
//   nerfacc/cuda/csrc/pdf.cu:97-166   importance_sampling_kernel   (one thread per output sample)
//   nerfacc/cuda/csrc/pdf.cu:168-243  compute_intervels_kernel     (second launch over the samples)
//   nerfacc/cuda/csrc/pdf.cu:247-287  searchsorted_kernel
//   nerfacc/cuda/csrc/pdf.cu:293-456  host wrappers (both importance_sampling overloads, searchsorted)
//   nerfacc/estimators/prop_net.py:232-256  _pdf_loss and its autograd graph (ATen ops; no kernel in the reference)
//
// A ray is resampled by one warp (short rays: the proposal-network shapes) or one CTA (long rays): its
// CDF and edge positions are staged in shared memory once, every thread inverts the CDF for its samples
// with the bound search running out of shared memory, the sample centres stay in shared memory, and the
// same threads then write the edges between neighbouring centres -- one launch and one pass over the
// inputs instead of two launches whose threads each binary-search global memory.  Optionally the same launch also maps the edges from the normalised
// axis to ray distance (t_starts / t_ends of the proposal estimator), which otherwise costs six
// elementwise ATen launches per proposal level.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/nerfacc_b200.h"
#include "sm_count.cuh"
#include "pdf.cuh"

namespace nfa {

constexpr int kIsThreads = 128;
constexpr int kSearchThreads = 256;
constexpr int64_t kIsSmemFloats = 50 * 1024;  // 200 KB of the 227 KB a CTA may opt in to
constexpr int64_t kWarpRayFloats = 1024;       // rays whose tables fit 4 KB take the warp-per-ray kernel

struct IsParams {
    int32_t n_rays;
    const float* vals;
    const float* cdfs;
    const int64_t* in_packed;   // null: batched input, in_edges per ray
    int64_t in_edges;
    const int64_t* out_packed;  // null: batched output, n_out samples per ray; else samples' (start, count)
    const int64_t* iv_packed;   // intervals' (start, count) when out_packed is given
    int64_t n_out;
    int32_t stratified;
    uint64_t seed, offset;
    float* sample_vals;
    int64_t* sample_ray;
    float* iv_vals;
    int64_t* iv_ray;
    uint8_t* iv_left;
    uint8_t* iv_right;
    // optional s -> t mapping of the edges (batched output only)
    float* t_starts;
    float* t_ends;
    float s_min, s_max;
    int32_t lindisp;
};

// One ray, resampled by `kLanes` cooperating threads (a whole CTA or one warp) whose rank is `tid`.
// kStage: `stage` holds room for this ray's CDF, edge positions and sample centres.  Per-ray counts and
// positions are 32-bit (a ray with 2^31 edges does not exist); only the array offsets are 64-bit.
template <bool kStage, int kLanes, bool kCta>
NFA_D void resample_ray(const IsParams& p, int32_t ray, int tid, float* stage, float bias)
{
    int64_t base;
    int32_t n_in;
    if (p.in_packed) {
        base = p.in_packed[2 * (int64_t)ray];
        n_in = (int32_t)p.in_packed[2 * (int64_t)ray + 1];
    } else {
        base = (int64_t)ray * p.in_edges;
        n_in = (int32_t)p.in_edges;
    }
    int64_t s_base, e_base;
    int32_t n;
    if (p.out_packed) {
        s_base = p.out_packed[2 * (int64_t)ray];
        n = (int32_t)p.out_packed[2 * (int64_t)ray + 1];
        e_base = p.iv_packed[2 * (int64_t)ray];
    } else {
        n = (int32_t)p.n_out;
        s_base = (int64_t)ray * n;
        e_base = s_base + ray;
    }
    if (n <= 0) return;  // uniform over the cooperating threads

    const float* cdf = p.cdfs + base;
    const float* val = p.vals + base;
    float* const out_s = p.sample_vals + s_base;
    float* ts = out_s;
    if (kStage) {
        float* s_cdf = stage;
        float* s_val = stage + n_in;
        for (int32_t i = tid; i < n_in; i += kLanes) {
            s_cdf[i] = __ldg(cdf + i);
            s_val[i] = __ldg(val + i);
        }
        cdf = s_cdf;
        val = s_val;
        ts = stage + 2 * n_in;
        if (kCta) __syncthreads(); else __syncwarp();
    }

    const float quiet_nan = __int_as_float(0x7fc00000);
    const float t_min = n_in > 0 ? val[0] : quiet_nan;
    const float t_max = n_in > 0 ? val[n_in - 1] : quiet_nan;
    const float u_floor = n_in > 0 ? cdf[0] : quiet_nan;
    const float u_ceil = n_in > 0 ? cdf[n_in - 1] : quiet_nan;
    const float u_step = f_div(f_sub(u_ceil, u_floor), (float)n);

    for (int32_t sid = tid; sid < n; sid += kLanes) {
        const float t = n_in > 0 ? is_invert<int32_t>(cdf, val, 0, n_in - 1, is_u<int32_t>(u_floor, u_step, sid, bias))
                                 : quiet_nan;
        ts[sid] = t;
        if (kStage) out_s[sid] = t;
        if (p.sample_ray) p.sample_ray[s_base + sid] = ray;
    }
    // centres visible to the cooperating threads (shared memory, or this CTA's own global writes)
    if (kCta) __syncthreads(); else __syncwarp();

    // edges 0 .. n-1 by the thread of the same index; the thread holding the last one adds the closing edge n
    // (a separate pass over k = n would cost a whole extra loop trip when n is a multiple of the group size)
    float* const out_e = p.iv_vals + e_base;
    for (int32_t k = tid; k < n; k += kLanes) {
        const float e = is_edge<int32_t>(ts, n, k, t_min, t_max);
        out_e[k] = e;
        float e_close = 0.f;
        const bool closes = k == n - 1;
        if (closes) {
            e_close = is_edge<int32_t>(ts, n, n, t_min, t_max);
            out_e[n] = e_close;
        }
        if (p.out_packed) {
            p.iv_ray[e_base + k] = ray;
            p.iv_left[e_base + k] = 1;
            p.iv_right[e_base + k] = k > 0;
            if (closes) {
                p.iv_ray[e_base + n] = ray;
                p.iv_left[e_base + n] = 0;
                p.iv_right[e_base + n] = 1;
            }
        } else if (p.t_starts) {
            const float t = stot(e, p.s_min, p.s_max, p.lindisp != 0);
            p.t_starts[s_base + k] = t;
            if (k > 0) p.t_ends[s_base + k - 1] = t;
            if (closes) p.t_ends[s_base + k] = stot(e_close, p.s_min, p.s_max, p.lindisp != 0);
        }
    }
    if (kStage) {  // before the next ray overwrites the staging area
        if (kCta) __syncthreads(); else __syncwarp();
    }
}

// CTA per ray: long rays (hundreds of edges / samples).  kStage = false searches global memory (rays whose
// tables exceed shared memory).
template <bool kStage>
__global__ void __launch_bounds__(kIsThreads) importance_sampling_kernel(IsParams p)
{
    extern __shared__ float smem[];
    for (int32_t ray = blockIdx.x; ray < p.n_rays; ray += gridDim.x) {
        const float bias = p.stratified ? philox_uniform(p.seed, (uint64_t)(int64_t)ray, p.offset) : 0.5f;
        resample_ray<kStage, kIsThreads, true>(p, ray, threadIdx.x, smem, bias);
    }
}

// Warp per ray, kIsWarps rays in flight per CTA: the proposal-network shapes (tens of edges and samples per
// ray, 10^5..10^6 rays), where a CTA per ray would leave most of its threads idle between two barriers.
constexpr int kIsWarps = 8;
// Stratified: a warp takes `chunk` consecutive rays per turn, lane l draws the jitter of ray l (one Philox4x32-10
// block is ~100 instructions; drawn per ray by all 32 lanes it was a quarter of the kernel), then the rays are
// resampled one after the other with the jitter handed over by shuffle.
template <bool kStratified>
__global__ void __launch_bounds__(kIsWarps * 32) importance_sampling_warp_kernel(IsParams p, int32_t floats_per_ray,
                                                                                 int32_t chunk /* rays per turn, <= 32 */)
{
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* stage = smem + (size_t)warp * floats_per_ray;
    if constexpr (!kStratified) {  // one ray per turn, neighbouring rays on neighbouring warps
        for (int64_t ray = (int64_t)blockIdx.x * kIsWarps + warp; ray < p.n_rays; ray += (int64_t)gridDim.x * kIsWarps)
            resample_ray<true, 32, false>(p, (int32_t)ray, lane, stage, 0.5f);
    } else
    for (int64_t ray0 = ((int64_t)blockIdx.x * kIsWarps + warp) * chunk; ray0 < p.n_rays;
         ray0 += (int64_t)gridDim.x * kIsWarps * chunk) {
        const int n = (int)min((int64_t)chunk, p.n_rays - ray0);
        float jitter = 0.5f;
        if (lane < n) jitter = philox_uniform(p.seed, (uint64_t)(ray0 + lane), p.offset);
        for (int i = 0; i < n; ++i)
            resample_ray<true, 32, false>(p, (int32_t)(ray0 + i), lane, stage, __shfl_sync(0xffffffffu, jitter, i));
    }
}

// ---------------------------------------------------------------------------
// Batched input AND output (the proposal-network shapes, BASELINE config 4: [n_rays, 65] -> 32 samples): the hot
// flavour.  Same arithmetic as resample_ray (pdf.cuh), but
//   * a warp takes `chunk` consecutive rays and keeps TWO staging buffers: the CDF / edge rows of ray i+1 are copied
//     global -> shared with cp.async (LDGSTS, no register round trip, no scoreboard wait) while ray i is resampled;
//   * every per-ray quantity that the generic kernel derives from the packed / batched switch is a pointer that
//     advances by a constant.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void cp_async_f32(float* dst_smem, const float* src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void cp_async_wait()
{
    asm volatile("cp.async.wait_group %0;" ::"n"(kPending) : "memory");
}

template <bool kStratified, bool kMapT>
__global__ void __launch_bounds__(kIsWarps * 32) importance_sampling_batched_kernel(IsParams p, int32_t n_in, int32_t n,
                                                                                   int32_t chunk)
{
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // per warp: stage[2][2 * n_in] (cdf row, then edge-position row) and the n sample centres
    float* const base = smem + (size_t)warp * (4 * n_in + n);
    float* const ts = base + 4 * n_in;
    const float quiet_nan = __int_as_float(0x7fc00000);

    auto stage_ray = [&](int64_t ray, int buf) {  // asynchronous: completes at the next wait
        const float* c = p.cdfs + ray * n_in;
        const float* v = p.vals + ray * n_in;
        float* d = base + buf * 2 * n_in;
        for (int i = lane; i < n_in; i += 32) {
            cp_async_f32(d + i, c + i);
            cp_async_f32(d + n_in + i, v + i);
        }
        cp_async_commit();
    };

    for (int64_t ray0 = ((int64_t)blockIdx.x * kIsWarps + warp) * chunk; ray0 < p.n_rays;
         ray0 += (int64_t)gridDim.x * kIsWarps * chunk) {
        const int cnt = (int)min((int64_t)chunk, p.n_rays - ray0);
        float jitter = 0.5f;
        if (kStratified && lane < cnt) jitter = philox_uniform(p.seed, (uint64_t)(ray0 + lane), p.offset);
        stage_ray(ray0, 0);
        float* out_s = p.sample_vals + ray0 * n;
        float* out_e = p.iv_vals + ray0 * (n + 1);
        float* out_a = kMapT ? p.t_starts + ray0 * n : nullptr;
        float* out_b = kMapT ? p.t_ends + ray0 * n : nullptr;
        for (int i = 0; i < cnt; ++i) {
            const int buf = i & 1;
            if (i + 1 < cnt) {
                stage_ray(ray0 + i + 1, buf ^ 1);
                cp_async_wait<1>();
            } else {
                cp_async_wait<0>();
            }
            __syncwarp();
            const float* cdf = base + buf * 2 * n_in;
            const float* val = cdf + n_in;
            const float bias = kStratified ? __shfl_sync(0xffffffffu, jitter, i) : 0.5f;
            const float t_min = val[0], t_max = val[n_in - 1];
            const float u_floor = cdf[0], u_ceil = cdf[n_in - 1];
            const float u_step = f_div(f_sub(u_ceil, u_floor), (float)n);
            for (int sid = lane; sid < n; sid += 32) {
                const float t = is_invert<int32_t>(cdf, val, 0, n_in - 1, is_u<int32_t>(u_floor, u_step, sid, bias));
                ts[sid] = t;
                out_s[sid] = t;
                if (p.sample_ray) p.sample_ray[(ray0 + i) * n + sid] = ray0 + i;
            }
            __syncwarp();
            for (int k = lane; k < n; k += 32) {
                const float e = is_edge<int32_t>(ts, n, k, t_min, t_max);
                out_e[k] = e;
                const bool closes = k == n - 1;
                float e_close = 0.f;
                if (closes) {
                    e_close = is_edge<int32_t>(ts, n, n, t_min, t_max);
                    out_e[n] = e_close;
                }
                if (kMapT) {
                    const float t = stot(e, p.s_min, p.s_max, p.lindisp != 0);
                    out_a[k] = t;
                    if (k > 0) out_b[k - 1] = t;
                    if (closes) out_b[k] = stot(e_close, p.s_min, p.s_max, p.lindisp != 0);
                }
            }
            __syncwarp();  // `ts` and this stage are free again
            out_s += n;
            out_e += n + 1;
            if (kMapT) {
                out_a += n;
                out_b += n;
            }
        }
    }
    (void)quiet_nan;
}

struct SearchParams {
    int64_t n_query;
    const float* q_vals;
    const int64_t* q_packed;  // null: batched query, q_edges per ray
    const int64_t* q_ray;     // optional ray id per query item (flattened query)
    int32_t n_rays;
    int64_t q_edges;
    const float* k_vals;
    const int64_t* k_packed;  // null: batched key, k_edges per ray
    int64_t k_edges;
    int64_t* ids_left;
    int64_t* ids_right;
};

__global__ void __launch_bounds__(kSearchThreads) searchsorted_kernel(SearchParams p)
{
    for (int64_t i = (int64_t)blockIdx.x * kSearchThreads + threadIdx.x; i < p.n_query;
         i += (int64_t)gridDim.x * kSearchThreads) {
        int64_t ray;
        if (!p.q_packed) ray = i / p.q_edges;
        else if (p.q_ray) ray = p.q_ray[i];
        else ray = chunk_upper_bound(p.q_packed, p.n_rays, i) - 1;
        int64_t base, last;
        if (p.k_packed) {
            base = p.k_packed[2 * ray];
            last = base + p.k_packed[2 * ray + 1] - 1;
        } else {
            base = ray * p.k_edges;
            last = base + p.k_edges - 1;
        }
        int64_t l, r;
        search_ids<int64_t>(p.k_vals, base, last, __ldg(p.q_vals + i), l, r);
        const int64_t rel = p.q_packed ? 0 : base;  // batched queries get per-ray positions
        p.ids_left[i] = l - rel;
        p.ids_right[i] = r - rel;
    }
}

// ---------------------------------------------------------------------------
// Proposal loss (PropNetEstimator.compute_loss, prop_net.py `_pdf_loss`) over batched rows: query edges / cdfs
// (n_rays, Eq), key edges / cdfs (n_rays, Ek).  Interval j of a ray spans query edges j and j+1; L_j is searchsorted's
// left id of edge j, R_j its right id of edge j+1.  A warp per ray; key rows of up to kLossStageEdges edges are staged
// in the warp's shared memory, longer ones are searched where they lie.
// ---------------------------------------------------------------------------
constexpr int kLossWarps = 8;
constexpr int kLossCtasPerSm = 6;                             // one wave: registers allow 6 CTAs per SM
constexpr int32_t kLossStageEdges = 512;                      // 4 KB of edges + cdfs per warp
constexpr int64_t kLossMaxIntervals = NFA_PDF_LOSS_MAX_INTERVALS;  // the backward's per-interval rows: 12 B each
constexpr int kLossMaxSmem = 227 * 1024;

struct PdfLossParams {
    int64_t n_rays;
    int32_t q_edges, k_edges;
    const float* q_vals;
    const float* q_cdfs;
    const float* k_vals;
    const float* k_cdfs;
    float eps;
    float* loss;             // forward: (n_rays, Eq - 1)
    const float* grad_loss;  // backward: (n_rays, Eq - 1)
    float* grad_k_cdfs;      // backward: (n_rays, Ek)
};

// The key row of `ray`: copied into `stage` (2 * Ek floats) or read in place.
template <bool kStage>
NFA_D void loss_key_row(const PdfLossParams& p, int64_t ray, int lane, float* stage, const float*& kv, const float*& kc)
{
    kv = p.k_vals + ray * p.k_edges;
    kc = p.k_cdfs + ray * p.k_edges;
    if (kStage) {
        for (int32_t i = lane; i < p.k_edges; i += 32) {
            stage[i] = __ldg(kv + i);
            stage[p.k_edges + i] = __ldg(kc + i);
        }
        __syncwarp();
        kv = stage;
        kc = stage + p.k_edges;
    }
}

// L_j, R_j and w = cq[j+1] - cq[j], wo = ck[R_j] - ck[L_j] of interval j
NFA_D void loss_interval(const PdfLossParams& p, const float* qv, const float* qc, const float* kv, const float* kc,
                         int32_t j, int32_t& left, int32_t& right, float& w, float& wo)
{
    int32_t unused;
    search_ids<int32_t>(kv, 0, p.k_edges - 1, __ldg(qv + j), left, unused);
    search_ids<int32_t>(kv, 0, p.k_edges - 1, __ldg(qv + j + 1), unused, right);
    w = f_sub(__ldg(qc + j + 1), __ldg(qc + j));
    wo = f_sub(kc[right], kc[left]);
}

template <bool kStage>
__global__ void __launch_bounds__(kLossWarps * 32, kLossCtasPerSm) pdf_loss_fwd_kernel(PdfLossParams p)
{
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* const stage = smem + (size_t)warp * 2 * p.k_edges;
    const int32_t n = p.q_edges - 1;
    for (int64_t ray = (int64_t)blockIdx.x * kLossWarps + warp; ray < p.n_rays;
         ray += (int64_t)gridDim.x * kLossWarps) {
        const float *kv, *kc;
        loss_key_row<kStage>(p, ray, lane, stage, kv, kc);
        const float* qv = p.q_vals + ray * p.q_edges;
        const float* qc = p.q_cdfs + ray * p.q_edges;
        for (int32_t j = lane; j < n; j += 32) {
            int32_t l, r;
            float w, wo;
            loss_interval(p, qv, qc, kv, kc, j, l, r, w, wo);
            p.loss[ray * n + j] = pdf_loss_term(w, wo, p.eps);
        }
        if (kStage) __syncwarp();  // before the next ray overwrites the stage
    }
}

// Dense gradient of the key cdfs.  Per warp: [staged key row: 2 * Ek floats] R_j, L_j, t_j (n each).  Key edge k gets
// (R-side sum) + (L-side sum), each summed in ascending j by pdf_loss_fold (pdf.cuh): no atomics, so the bits depend on
// neither the launch nor the run.  Rows whose ids both do not decrease (sorted rows) search for their run; others scan
// every j.
template <bool kStage>
__global__ void __launch_bounds__(kLossWarps * 32, kLossCtasPerSm) pdf_loss_bwd_kernel(PdfLossParams p,
                                                                                       int32_t floats_per_warp)
{
    extern __shared__ float smem[];
    const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* const stage = smem + (size_t)warp * floats_per_warp;
    const int32_t n = p.q_edges - 1;
    int32_t* const s_right = reinterpret_cast<int32_t*>(stage + (kStage ? 2 * p.k_edges : 0));
    int32_t* const s_left = s_right + n;
    float* const s_term = reinterpret_cast<float*>(s_left + n);
    for (int64_t ray = (int64_t)blockIdx.x * warps + warp; ray < p.n_rays; ray += (int64_t)gridDim.x * warps) {
        const float *kv, *kc;
        loss_key_row<kStage>(p, ray, lane, stage, kv, kc);
        const float* qv = p.q_vals + ray * p.q_edges;
        const float* qc = p.q_cdfs + ray * p.q_edges;
        for (int32_t j = lane; j < n; j += 32) {
            int32_t l, r;
            float w, wo;
            loss_interval(p, qv, qc, kv, kc, j, l, r, w, wo);
            s_right[j] = r;
            s_left[j] = l;
            s_term[j] = pdf_loss_grad_wo(w, wo, p.eps, __ldg(p.grad_loss + ray * n + j));
        }
        __syncwarp();
        bool sorted = true;
        for (int32_t j = lane + 1; j < n; j += 32)
            sorted = sorted && s_right[j] >= s_right[j - 1] && s_left[j] >= s_left[j - 1];
        sorted = __all_sync(0xffffffffu, sorted);
        float* const gk = p.grad_k_cdfs + ray * p.k_edges;
        for (int32_t k = lane; k < p.k_edges; k += 32)
            gk[k] = f_add(pdf_loss_fold(s_right, s_term, n, k, sorted, false),
                          pdf_loss_fold(s_left, s_term, n, k, sorted, true));
        __syncwarp();  // before the next ray overwrites the rows
    }
}

}  // namespace nfa

using namespace nfa;

extern "C" {

int32_t nfa_importance_sampling(int32_t n_rays, const float* vals, const float* cdfs, const int64_t* in_packed_info,
                                int64_t in_edges, int64_t max_in_edges, const int64_t* out_packed_info,
                                const int64_t* iv_packed_info, int64_t n_out, int64_t max_out, int32_t stratified,
                                uint64_t seed, uint64_t offset, float* sample_vals, int64_t* sample_ray_indices,
                                float* iv_vals, int64_t* iv_ray_indices, uint8_t* iv_left, uint8_t* iv_right,
                                float* t_starts, float* t_ends, float s_min, float s_max, int32_t lindisp,
                                nfa_stream_t stream)
{
    if (n_rays < 0 || in_edges < 0 || n_out < 0 || max_in_edges < 0 || max_out < 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!sample_vals || !iv_vals) return NFA_ERR_ARG;
    if (max_in_edges > 0 && (!vals || !cdfs)) return NFA_ERR_ARG;
    if (out_packed_info && (!iv_packed_info || !iv_ray_indices || !iv_left || !iv_right)) return NFA_ERR_ARG;
    if ((t_starts != nullptr) != (t_ends != nullptr)) return NFA_ERR_ARG;
    if (t_starts && out_packed_info) return NFA_ERR_UNSUPPORTED;
    if (!out_packed_info && n_out == 0) return NFA_OK;

    IsParams p;
    p.n_rays = n_rays;
    p.vals = vals;
    p.cdfs = cdfs;
    p.in_packed = in_packed_info;
    p.in_edges = in_edges;
    p.out_packed = out_packed_info;
    p.iv_packed = iv_packed_info;
    p.n_out = n_out;
    p.stratified = stratified;
    p.seed = seed;
    p.offset = offset;
    p.sample_vals = sample_vals;
    p.sample_ray = sample_ray_indices;
    p.iv_vals = iv_vals;
    p.iv_ray = iv_ray_indices;
    p.iv_left = iv_left;
    p.iv_right = iv_right;
    p.t_starts = t_starts;
    p.t_ends = t_ends;
    p.s_min = s_min;
    p.s_max = s_max;
    p.lindisp = lindisp;

    const int64_t in_cap = in_packed_info ? max_in_edges : in_edges;
    const int64_t out_cap = out_packed_info ? max_out : n_out;
    const int64_t floats = 2 * in_cap + out_cap;
    cudaStream_t s = (cudaStream_t)stream;
    if (!in_packed_info && !out_packed_info && in_edges >= 2 && n_out >= 1 && 4 * in_edges + n_out <= kWarpRayFloats) {
        // batched rows in, batched rows out (proposal-network shapes): double-buffered warp-per-ray kernel.  A warp
        // walks `chunk` consecutive rays (the next ray's rows are in flight while this one is resampled)
        const int64_t fl = 4 * in_edges + n_out;
        const size_t bytes = (size_t)fl * kIsWarps * sizeof(float);
        int64_t chunk = (int64_t)n_rays / (kNumSMs * 8 * kIsWarps);
        chunk = chunk < 1 ? 1 : (chunk > 32 ? 32 : chunk);
        const int64_t want = ((int64_t)n_rays + chunk * kIsWarps - 1) / (chunk * kIsWarps);
        const unsigned grid = (unsigned)(want < (1 << 20) ? want : (1 << 20));
#define NFA_IS_BATCHED(S, M) importance_sampling_batched_kernel<S, M><<<grid, kIsWarps * 32, bytes, s>>>(p, (int32_t)in_edges, (int32_t)n_out, (int32_t)chunk)
        if (stratified) { if (t_starts) NFA_IS_BATCHED(true, true); else NFA_IS_BATCHED(true, false); }
        else { if (t_starts) NFA_IS_BATCHED(false, true); else NFA_IS_BATCHED(false, false); }
#undef NFA_IS_BATCHED
        return (int32_t)cudaGetLastError();
    }
    if (floats <= kWarpRayFloats) {
        // short rays: a warp each; persistent CTAs sized to fill the machine
        const size_t bytes = (size_t)floats * kIsWarps * sizeof(float);
        // stratified: 8 rays per turn, so one Philox block serves 8 rays (32 rays per turn left a partial last
        // wave as long as a whole CTA).  Plain: one ray per turn, neighbouring rays on neighbouring warps (measured
        // faster than turns of 8).
        int64_t chunk = stratified ? (int64_t)n_rays / (kNumSMs * 64) : 1;
        chunk = chunk < 1 ? 1 : (chunk > 8 ? 8 : chunk);
        const int64_t want = ((int64_t)n_rays + chunk * kIsWarps - 1) / (chunk * kIsWarps);
        const int64_t cap = kNumSMs * 8 * 4;
        const unsigned grid = (unsigned)(want < cap ? want : cap);
        if (stratified)
            importance_sampling_warp_kernel<true><<<grid, kIsWarps * 32, bytes, s>>>(p, (int32_t)floats, (int32_t)chunk);
        else
            importance_sampling_warp_kernel<false><<<grid, kIsWarps * 32, bytes, s>>>(p, (int32_t)floats, (int32_t)chunk);
        return (int32_t)cudaGetLastError();
    }
    const unsigned grid = (unsigned)(n_rays < (1 << 20) ? n_rays : (1 << 20));
    if (floats <= kIsSmemFloats) {
        const size_t bytes = (size_t)floats * sizeof(float);
        if (bytes > 48 * 1024) {
            cudaError_t e = cudaFuncSetAttribute(importance_sampling_kernel<true>,
                                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
            if (e != cudaSuccess) return (int32_t)e;
        }
        importance_sampling_kernel<true><<<grid, kIsThreads, bytes, s>>>(p);
    } else {
        importance_sampling_kernel<false><<<grid, kIsThreads, 0, s>>>(p);
    }
    return (int32_t)cudaGetLastError();
}

int32_t nfa_searchsorted(int64_t n_query, const float* query_vals, const int64_t* query_packed_info,
                         const int64_t* query_ray_indices, int32_t n_rays, int64_t query_edges,
                         const float* key_vals, const int64_t* key_packed_info, int64_t key_edges,
                         int64_t* ids_left, int64_t* ids_right, nfa_stream_t stream)
{
    if (n_query < 0 || n_rays < 0 || query_edges < 0 || key_edges < 0) return NFA_ERR_ARG;
    if (n_query == 0) return NFA_OK;
    if (!query_vals || !key_vals || !ids_left || !ids_right) return NFA_ERR_ARG;
    if (!query_packed_info && query_edges == 0) return NFA_ERR_ARG;
    SearchParams p;
    p.n_query = n_query;
    p.q_vals = query_vals;
    p.q_packed = query_packed_info;
    p.q_ray = query_ray_indices;
    p.n_rays = n_rays;
    p.q_edges = query_edges;
    p.k_vals = key_vals;
    p.k_packed = key_packed_info;
    p.k_edges = key_edges;
    p.ids_left = ids_left;
    p.ids_right = ids_right;
    const int64_t blocks = (n_query + kSearchThreads - 1) / kSearchThreads;
    const unsigned grid = (unsigned)(blocks < kNumSMs * 64 ? blocks : kNumSMs * 64);
    searchsorted_kernel<<<grid, kSearchThreads, 0, (cudaStream_t)stream>>>(p);
    return (int32_t)cudaGetLastError();
}

static int32_t pdf_loss_params(int64_t n_rays, int64_t q_edges, const float* q_vals, const float* q_cdfs,
                               int64_t k_edges, const float* k_vals, const float* k_cdfs, float eps, PdfLossParams& p)
{
    if (n_rays < 0 || q_edges < 1 || k_edges < 1 || q_edges > INT32_MAX || k_edges > INT32_MAX) return NFA_ERR_ARG;
    p.n_rays = n_rays;
    p.q_edges = (int32_t)q_edges;
    p.k_edges = (int32_t)k_edges;
    p.q_vals = q_vals;
    p.q_cdfs = q_cdfs;
    p.k_vals = k_vals;
    p.k_cdfs = k_cdfs;
    p.eps = eps;
    p.loss = nullptr;
    p.grad_loss = nullptr;
    p.grad_k_cdfs = nullptr;
    return NFA_OK;
}

int32_t nfa_pdf_loss_fwd(int64_t n_rays, int64_t q_edges, const float* q_vals, const float* q_cdfs, int64_t k_edges,
                         const float* k_vals, const float* k_cdfs, float eps, float* loss, nfa_stream_t stream)
{
    PdfLossParams p;
    const int32_t rc = pdf_loss_params(n_rays, q_edges, q_vals, q_cdfs, k_edges, k_vals, k_cdfs, eps, p);
    if (rc != NFA_OK) return rc;
    if (n_rays == 0 || q_edges == 1) return NFA_OK;
    if (!q_vals || !q_cdfs || !k_vals || !k_cdfs || !loss) return NFA_ERR_ARG;
    p.loss = loss;
    const int64_t want = (n_rays + kLossWarps - 1) / kLossWarps;
    const unsigned grid = (unsigned)(want < kNumSMs * kLossCtasPerSm ? want : kNumSMs * kLossCtasPerSm);
    cudaStream_t s = (cudaStream_t)stream;
    if (k_edges <= kLossStageEdges)
        pdf_loss_fwd_kernel<true><<<grid, kLossWarps * 32, (size_t)kLossWarps * 2 * k_edges * sizeof(float), s>>>(p);
    else
        pdf_loss_fwd_kernel<false><<<grid, kLossWarps * 32, 0, s>>>(p);
    return (int32_t)cudaGetLastError();
}

int32_t nfa_pdf_loss_bwd(int64_t n_rays, int64_t q_edges, const float* q_vals, const float* q_cdfs, int64_t k_edges,
                         const float* k_vals, const float* k_cdfs, float eps, const float* grad_loss,
                         float* grad_k_cdfs, nfa_stream_t stream)
{
    PdfLossParams p;
    const int32_t rc = pdf_loss_params(n_rays, q_edges, q_vals, q_cdfs, k_edges, k_vals, k_cdfs, eps, p);
    if (rc != NFA_OK) return rc;
    if (q_edges - 1 > kLossMaxIntervals) return NFA_ERR_UNSUPPORTED;
    if (n_rays == 0) return NFA_OK;
    if (!q_vals || !q_cdfs || !k_vals || !k_cdfs || !grad_k_cdfs || (q_edges > 1 && !grad_loss)) return NFA_ERR_ARG;
    p.grad_loss = grad_loss;
    p.grad_k_cdfs = grad_k_cdfs;
    const bool stage = k_edges <= kLossStageEdges;
    const int32_t floats = (int32_t)((stage ? 2 * k_edges : 0) + 3 * (q_edges - 1));
    const size_t per_warp = (size_t)floats * sizeof(float);
    int warps = per_warp > 0 ? (int)(kLossMaxSmem / per_warp) : kLossWarps;
    warps = warps < kLossWarps ? warps : kLossWarps;
    const size_t bytes = per_warp * warps;
    // one wave: as many CTAs as fit an SM by threads and by shared memory
    int per_sm = kLossCtasPerSm * kLossWarps / warps;
    if (bytes > 0 && (size_t)per_sm * bytes > (size_t)kLossMaxSmem) per_sm = (int)(kLossMaxSmem / bytes);
    const int64_t want = (n_rays + warps - 1) / warps;
    const unsigned grid = (unsigned)(want < (int64_t)kNumSMs * per_sm ? want : (int64_t)kNumSMs * per_sm);
    cudaStream_t s = (cudaStream_t)stream;
#define NFA_LOSS_BWD(S)                                                                                               \
    do {                                                                                                              \
        if (bytes > 48 * 1024) {                                                                                      \
            const cudaError_t e = cudaFuncSetAttribute(pdf_loss_bwd_kernel<S>,                                        \
                                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);      \
            if (e != cudaSuccess) return (int32_t)e;                                                                  \
        }                                                                                                             \
        pdf_loss_bwd_kernel<S><<<grid, warps * 32, bytes, s>>>(p, floats);                                            \
    } while (0)
    if (stage) NFA_LOSS_BWD(true);
    else NFA_LOSS_BWD(false);
#undef NFA_LOSS_BWD
    return (int32_t)cudaGetLastError();
}

}  // extern "C"
