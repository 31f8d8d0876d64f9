// CPU build of the proposal-loss arithmetic of pdf.cuh, in the order pdf_loss_fwd_kernel / pdf_loss_bwd_kernel (pdf.cu)
// apply it: per ray, L_j / R_j by searchsorted's search and clipping, the per-interval term, and for the backward the
// per-key sums of pdf_loss_fold.  The device runs a warp per ray; here the rays are serialised.  Compiled by
// tests/test_prop_loss_cpu.py with -ffp-contract=off.
#include <cstdint>
#include <vector>

#include "../../nerfacc_b200/csrc/pdf.cuh"

using namespace nfa;

namespace {

void interval(const float* qv, const float* qc, const float* kv, const float* kc, int32_t ek, int32_t j, int32_t& left,
              int32_t& right, float& w, float& wo)
{
    int32_t unused;
    search_ids<int32_t>(kv, 0, ek - 1, qv[j], left, unused);
    search_ids<int32_t>(kv, 0, ek - 1, qv[j + 1], unused, right);
    w = f_sub(qc[j + 1], qc[j]);
    wo = f_sub(kc[right], kc[left]);
}

}  // namespace

extern "C" {

// loss [n_rays, eq - 1]; ids_left / ids_right [n_rays, eq - 1] (L_j, R_j) when given
void sim_pdf_loss_fwd(int64_t n_rays, int32_t eq, const float* q_vals, const float* q_cdfs, int32_t ek,
                      const float* k_vals, const float* k_cdfs, float eps, float* loss, int64_t* ids_left,
                      int64_t* ids_right)
{
    const int32_t n = eq - 1;
    for (int64_t r = 0; r < n_rays; ++r) {
        for (int32_t j = 0; j < n; ++j) {
            int32_t l, rt;
            float w, wo;
            interval(q_vals + r * eq, q_cdfs + r * eq, k_vals + r * ek, k_cdfs + r * ek, ek, j, l, rt, w, wo);
            loss[r * n + j] = pdf_loss_term(w, wo, eps);
            if (ids_left) ids_left[r * n + j] = l;
            if (ids_right) ids_right[r * n + j] = rt;
        }
    }
}

// grad_k_cdfs [n_rays, ek] from grad_loss [n_rays, eq - 1]
void sim_pdf_loss_bwd(int64_t n_rays, int32_t eq, const float* q_vals, const float* q_cdfs, int32_t ek,
                      const float* k_vals, const float* k_cdfs, float eps, const float* grad_loss, float* grad_k_cdfs)
{
    const int32_t n = eq - 1;
    std::vector<int32_t> right(n > 0 ? n : 1), left(n > 0 ? n : 1);
    std::vector<float> term(n > 0 ? n : 1);
    for (int64_t r = 0; r < n_rays; ++r) {
        bool sorted = true;
        for (int32_t j = 0; j < n; ++j) {
            float w, wo;
            interval(q_vals + r * eq, q_cdfs + r * eq, k_vals + r * ek, k_cdfs + r * ek, ek, j, left[j], right[j], w,
                     wo);
            term[j] = pdf_loss_grad_wo(w, wo, eps, grad_loss[r * n + j]);
            if (j > 0) sorted = sorted && right[j] >= right[j - 1] && left[j] >= left[j - 1];
        }
        for (int32_t k = 0; k < ek; ++k)
            grad_k_cdfs[r * ek + k] = f_add(pdf_loss_fold(right.data(), term.data(), n, k, sorted, false),
                                            pdf_loss_fold(left.data(), term.data(), n, k, sorted, true));
    }
}

// the per-interval terms alone: loss and d loss / d wo of (w, wo, g) element by element
void sim_pdf_loss_terms(int64_t n, const float* w, const float* wo, const float* g, float eps, float* loss,
                        float* grad_wo)
{
    for (int64_t i = 0; i < n; ++i) {
        loss[i] = pdf_loss_term(w[i], wo[i], eps);
        grad_wo[i] = pdf_loss_grad_wo(w[i], wo[i], eps, g[i]);
    }
}

}  // extern "C"
