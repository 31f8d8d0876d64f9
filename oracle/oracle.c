/*
 * oracle.c -- CPU restatement of nerfacc's sampling + compositing hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under nerfacc_b200/ may import, link or
 * call this file; only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference leg use it, and only as the checker or as
 * the timed CPU baseline -- never as the product path.
 *
 * Every function restates one piece of the reference (paths relative to
 * /root/reference) in scalar IEEE binary32 arithmetic.  The reference kernels
 * are compiled by nvcc with its default FMA contraction; the contraction
 * pattern that nvcc 12.9 / ptxas actually emits was read off the
 * SASS of nerfacc/cuda/csrc/grid.cu (see DESIGN.md "Arithmetic contract") and
 * is reproduced here with explicit fmaf() calls.  This file must be built with
 * -ffp-contract=off so the compiler adds no contractions of its own.
 *
 * Parity status: pinned.  tests/golden/ holds vectors produced by the
 * reference CUDA build on a GPU (oracle/gen_golden_gpu.py for traversal,
 * compositing and scans, oracle/gen_golden_pdf_gpu.py for importance sampling,
 * searchsorted and PropNetEstimator) and the reference's own test / docstring
 * known-answer vectors; tests/test_oracle_*.py and tests/test_pdf_cpu.py check
 * this file against all of them.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------ */
/* small helpers                                                       */
/* ------------------------------------------------------------------ */

/* nerfacc/cuda/csrc/include/utils_math.cuh:1167-1174 -- clamp(f,a,b) is
 * fmaxf(a, fminf(f, b)) for floats and max(a, min(f, b)) for ints. */
static inline float clampf(float f, float lo, float hi) { return fmaxf(lo, fminf(f, hi)); }
static inline int clampi(int v, int lo, int hi) { int m = v < hi ? v : hi; return lo > m ? lo : m; }

/* nerfacc/cuda/csrc/grid.cu:23-28 -- marching step length at distance t. */
static inline float step_len(float t, float cone_angle, float dt_min, float dt_max)
{
    return clampf(t * cone_angle, dt_min, dt_max);
}

/* float -> int conversion as the device does it (cvt.rzi.s32.f32: truncate,
 * saturate, NaN -> 0); utils_math.cuh:177-180 make_int3(float3). */
static inline int trunc_to_int(float f)
{
    if (f != f) return 0;
    if (f >= 2147483648.0f) return INT32_MAX;
    if (f <= -2147483648.0f) return INT32_MIN;
    return (int)f;
}

/* ------------------------------------------------------------------ */
/* ray / box slab test                                                 */
/* ------------------------------------------------------------------ */

/* nerfacc/cuda/csrc/include/utils_grid.cuh:10-55.  Returns hit flag; on a
 * hit tmin/tmax are clamped to [near, far].  inv = 1/dir, IEEE division
 * (data_spec_packed.cuh:49). */
static int slab_test(const float o[3], const float inv[3], const float box[6],
                     float near, float far, float *tmin_out, float *tmax_out)
{
    float lo, hi;
    for (int a = 0; a < 3; ++a) {
        float t_lo, t_hi;
        if (inv[a] >= 0.0f) {
            t_lo = (box[a] - o[a]) * inv[a];
            t_hi = (box[3 + a] - o[a]) * inv[a];
        } else {
            t_lo = (box[3 + a] - o[a]) * inv[a];
            t_hi = (box[a] - o[a]) * inv[a];
        }
        if (a == 0) {
            lo = t_lo;
            hi = t_hi;
        } else {
            if (lo > t_hi || t_lo > hi) return 0;
            if (t_lo > lo) lo = t_lo;
            if (t_hi < hi) hi = t_hi;
        }
    }
    if (hi <= 0.0f) return 0;
    *tmin_out = fmaxf(lo, near);
    *tmax_out = fminf(hi, far);
    return 1;
}

/* nerfacc/cuda/csrc/grid.cu:284-313 (kernel) + nerfacc/grid.py:13-51. */
ORC_API void orc_ray_aabb_intersect(
    int32_t n_rays, const float *rays_o, const float *rays_d,
    int32_t n_aabbs, const float *aabbs,
    float near_plane, float far_plane, float miss_value,
    float *t_mins, float *t_maxs, uint8_t *hits)
{
#pragma omp parallel for schedule(static)
    for (int32_t r = 0; r < n_rays; ++r) {
        const float *o = rays_o + 3 * r, *d = rays_d + 3 * r;
        float inv[3] = {1.0f / d[0], 1.0f / d[1], 1.0f / d[2]};
        for (int32_t g = 0; g < n_aabbs; ++g) {
            float a = miss_value, b = miss_value;
            int hit = slab_test(o, inv, aabbs + 6 * g, near_plane, far_plane, &a, &b);
            if (!hit) { a = miss_value; b = miss_value; }
            t_mins[(int64_t)r * n_aabbs + g] = a;
            t_maxs[(int64_t)r * n_aabbs + g] = b;
            hits[(int64_t)r * n_aabbs + g] = (uint8_t)hit;
        }
    }
}

/* nerfacc/grid.py:158-162 -- sort(cat([t_mins, t_maxs], -1), -1): ascending,
 * value + position in the concatenation.  Ties keep concatenation order (only
 * missed boxes tie, at +inf, and those entries are never used). */
ORC_API void orc_sort_intersections(
    int32_t n_rays, int32_t n_aabbs, const float *t_mins, const float *t_maxs,
    float *t_sorted, int64_t *t_indices)
{
    const int32_t m = 2 * n_aabbs;
#pragma omp parallel for schedule(static)
    for (int32_t r = 0; r < n_rays; ++r) {
        float *v = t_sorted + (int64_t)r * m;
        int64_t *ix = t_indices + (int64_t)r * m;
        for (int32_t j = 0; j < m; ++j) {
            float x = j < n_aabbs ? t_mins[(int64_t)r * n_aabbs + j]
                                  : t_maxs[(int64_t)r * n_aabbs + (j - n_aabbs)];
            int32_t k = j;
            while (k > 0 && v[k - 1] > x) { v[k] = v[k - 1]; ix[k] = ix[k - 1]; --k; }
            v[k] = x;
            ix[k] = j;
        }
    }
}

/* ------------------------------------------------------------------ */
/* grid traversal                                                      */
/* ------------------------------------------------------------------ */

typedef struct {
    /* rays */
    int32_t n_rays;
    const float *rays_o, *rays_d;
    const uint8_t *rays_mask; /* NULL = all rays */
    /* grids */
    int32_t n_grids;
    int32_t res[3];
    const uint8_t *binaries; /* [n_grids, rx, ry, rz] */
    const float *aabbs;      /* [n_grids, 6] */
    /* sorted box crossings */
    const uint8_t *hits;      /* [n_rays, n_grids] */
    const float *t_sorted;    /* [n_rays, 2 n_grids] */
    const int64_t *t_indices; /* [n_rays, 2 n_grids] */
    /* options */
    const float *near_planes, *far_planes;
    float step_size, cone_angle;
    int32_t steps_limit; /* <= 0: unlimited */
    /* edge ("intervals") outputs */
    int64_t *iv_starts, *iv_cnts; /* [n_rays] */
    float *iv_vals;
    int64_t *iv_ray;
    uint8_t *iv_left, *iv_right;
    /* sample outputs */
    int64_t *sm_starts, *sm_cnts; /* [n_rays] */
    float *sm_vals;
    int64_t *sm_ray;
    uint8_t *sm_valid;
    float *terminate_planes; /* [n_rays] or NULL */
} orc_traverse_t;

/* DDA set-up for one (ray, level, [tmin,tmax]) segment:
 * nerfacc/cuda/csrc/include/utils_grid.cuh:58-114.  fmaf() marks the three
 * places where the SASS of the reference holds an FFMA. */
typedef struct {
    float tdist[3], delta[3];
    int cur[3], step[3], overflow[3];
} dda_t;

static void dda_begin(dda_t *s, const float o[3], const float d[3], const float inv[3],
                      float tmin, float tmax, float eps, const float box[6], const int res[3])
{
    const float t_in = tmin + eps, t_out = tmax + (-eps);
    for (int a = 0; a < 3; ++a) {
        const float resf = (float)res[a];
        const float extent = box[3 + a] - box[a];
        const float voxel = extent / resf;
        const float p_in = fmaf(d[a], t_in, o[a]);
        const float p_out = fmaf(d[a], t_out, o[a]);
        /* utils_contraction.cuh:19-24 roi_to_unit, then * res, truncate, clamp */
        int first = clampi(trunc_to_int(((p_in - box[a]) / extent) * resf), 0, res[a] - 1);
        int last = clampi(trunc_to_int(((p_out - box[a]) / extent) * resf), 0, res[a] - 1);
        const int ahead = d[a] > 0.0f ? 1 : 0;
        const float face = (float)(uint32_t)(first + ahead);
        const float cross = fmaf(inv[a], box[a] + fmaf(face, voxel, -p_in), tmin);
        const float sgn = d[a] > 0.0f ? 1.0f : -1.0f;
        if (d[a] == 0.0f) {
            s->tdist[a] = tmax;
            s->delta[a] = tmax;
            s->step[a] = 0;
        } else {
            s->tdist[a] = cross;
            s->delta[a] = sgn * (inv[a] * voxel);
            s->step[a] = d[a] > 0.0f ? 1 : -1;
        }
        s->cur[a] = first;
        s->overflow[a] = last + s->step[a];
    }
}

/* utils_grid.cuh:116-142: advance to the next cell; 0 when the index on the
 * stepped axis reaches the overflow index.  Axis choice: x only if strictly
 * smaller than both, else y if strictly smaller than z, else z. */
static int dda_next(dda_t *s)
{
    int a;
    if (s->tdist[0] < s->tdist[1] && s->tdist[0] < s->tdist[2]) a = 0;
    else if (s->tdist[1] < s->tdist[2]) a = 1;
    else a = 2;
    s->cur[a] += s->step[a];
    s->tdist[a] += s->delta[a];
    return s->cur[a] != s->overflow[a];
}

/* One ray of nerfacc/cuda/csrc/grid.cu:68-282.  `fill` == 0 counts only
 * (first pass), != 0 writes at the ray's chunk offsets (second pass /
 * over-allocate pass). */
static void traverse_one(const orc_traverse_t *c, int32_t r, int fill)
{
    const float eps = 1e-6f; /* grid.cu:95 */
    const int G = c->n_grids;
    const int want_iv = c->iv_cnts != NULL, want_sm = c->sm_cnts != NULL;

    if (c->rays_mask && !c->rays_mask[r]) return; /* grid.cu:100 */
    if (fill) {                                    /* grid.cu:103-106 */
        if (want_iv && c->iv_cnts[r] == 0) return;
        if (want_sm && c->sm_cnts[r] == 0) return;
    }
    const int64_t iv_base = (fill && want_iv) ? c->iv_starts[r] : 0;
    const int64_t sm_base = (fill && want_sm) ? c->sm_starts[r] : 0;

    const float near = c->near_planes[r], far = c->far_planes[r];
    const float *o = c->rays_o + 3 * (int64_t)r, *d = c->rays_d + 3 * (int64_t)r;
    const float inv[3] = {1.0f / d[0], 1.0f / d[1], 1.0f / d[2]};
    const uint8_t *hit = c->hits + (int64_t)r * G;
    const float *ts = c->t_sorted + (int64_t)r * 2 * G;
    const int64_t *ti = c->t_indices + (int64_t)r * 2 * G;
    const int64_t cells_per_level = (int64_t)c->res[0] * c->res[1] * c->res[2];
    const float step = c->step_size, cone = c->cone_angle;
    const int limit = c->steps_limit;

    int64_t n_edges = 0, n_samples = 0;
    float t_last = near;
    int continuous = 0;

    for (int i = 0; i < 2 * G - 1; ++i) { /* grid.cu:129 */
        int entering = ti[i] < G;
        int64_t level = ti[i] % G;
        if (!hit[level]) continue;
        if (!entering) { /* grid.cu:138-146 */
            if (ti[i + 1] < G) continue;
            level = ti[i + 1] % G;
            if (!hit[level]) continue;
        }
        const float seg_lo = fmaxf(ts[i], near);
        const float seg_hi = fminf(ts[i + 1], far);
        if (seg_lo >= seg_hi) continue;

        if (!continuous) { /* grid.cu:153-163 */
            if (step <= 0.0f) {
                t_last = seg_lo;
            } else {
                const float dt = step_len(t_last, cone, step, 1e10f);
                while (!(t_last + dt * 0.5f >= seg_lo)) t_last += dt;
            }
        }

        dda_t s;
        dda_begin(&s, o, d, inv, seg_lo, seg_hi, eps, c->aabbs + 6 * level, c->res);

        while (limit <= 0 || n_samples < limit) { /* grid.cu:184 */
            float t_cell = fminf(s.tdist[0], fminf(s.tdist[1], s.tdist[2]));
            t_cell = fminf(t_cell, seg_hi);
            const int64_t cell = (int64_t)s.cur[0] * c->res[1] * c->res[2] +
                                 (int64_t)s.cur[1] * c->res[2] + s.cur[2] + level * cells_per_level;
            if (!c->binaries[cell]) { /* grid.cu:194-205 */
                if (step <= 0.0f) {
                    t_last = t_cell;
                } else {
                    const float dt = step_len(t_last, cone, step, 1e10f);
                    while (!(t_last + dt * 0.5f >= t_cell)) t_last += dt;
                }
                continuous = 0;
            } else { /* grid.cu:206-262 */
                while (limit <= 0 || n_samples < limit) {
                    float t_next;
                    if (step <= 0.0f) {
                        t_next = t_cell;
                    } else {
                        const float dt = step_len(t_last, cone, step, 1e10f);
                        if (t_last + dt * 0.5f >= t_cell) break;
                        t_next = t_last + dt;
                    }
                    if (want_iv) { /* grid.cu:219-245 */
                        if (!continuous) {
                            if (fill) {
                                int64_t k = iv_base + n_edges;
                                c->iv_vals[k] = t_last; c->iv_ray[k] = r; c->iv_left[k] = 1;
                                c->iv_vals[k + 1] = t_next; c->iv_ray[k + 1] = r; c->iv_right[k + 1] = 1;
                            }
                            n_edges += 2;
                        } else {
                            if (fill) {
                                int64_t k = iv_base + n_edges;
                                c->iv_vals[k] = t_next; c->iv_ray[k] = r;
                                c->iv_left[k - 1] = 1; c->iv_right[k] = 1;
                            }
                            n_edges += 1;
                        }
                    }
                    if (want_sm && fill) { /* grid.cu:248-255 */
                        int64_t k = sm_base + n_samples;
                        c->sm_vals[k] = (t_next + t_last) * 0.5f;
                        c->sm_ray[k] = r;
                        c->sm_valid[k] = 1;
                    }
                    n_samples += 1;
                    continuous = 1;
                    t_last = t_next;
                    if (t_next >= t_cell) break;
                }
            }
            if (!dda_next(&s)) break;
        }
    }
    if (c->terminate_planes) c->terminate_planes[r] = t_last;
    if (want_iv) c->iv_cnts[r] = n_edges;
    if (want_sm) c->sm_cnts[r] = n_samples;
}

/* Pass driver: pass 0 = count (writes *_cnts), pass 1 = fill.  The caller does
 * the exclusive scan + allocation in between, as data_spec.hpp:86-96 does. */
ORC_API void orc_traverse_pass(const orc_traverse_t *ctx, int32_t fill)
{
#pragma omp parallel for schedule(dynamic, 64)
    for (int32_t r = 0; r < ctx->n_rays; ++r) traverse_one(ctx, r, fill);
}

ORC_API int32_t orc_traverse_ctx_size(void) { return (int32_t)sizeof(orc_traverse_t); }

/* ------------------------------------------------------------------ */
/* packed segmented scans (nerfacc/scan.py, csrc/scan.cu, scan_cub.cu) */
/* ------------------------------------------------------------------ */

/* op: 0 = sum, 1 = product.  inclusive: 0/1.  reverse: scan each chunk from
 * its last element to its first (what the reverse-iterator backward launches
 * do, scan.cu:44-52).  Sequential f32 accumulation per chunk. */
ORC_API void orc_scan_packed(
    int32_t n_rays, const int64_t *starts, const int64_t *cnts,
    const float *in, float *out, int32_t op, int32_t inclusive, int32_t reverse, int32_t normalize)
{
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t r = 0; r < n_rays; ++r) {
        const int64_t s = starts[r], n = cnts[r];
        float acc = op ? 1.0f : 0.0f;
        for (int64_t j = 0; j < n; ++j) {
            const int64_t k = reverse ? s + n - 1 - j : s + j;
            const float x = in[k];
            if (inclusive) { acc = op ? acc * x : acc + x; out[k] = acc; }
            else { out[k] = acc; acc = op ? acc * x : acc + x; }
        }
        if (normalize && inclusive && !op) { /* utils_scan.cuh:102-109 */
            const float tot = fmaxf(acc, 1e-10f);
            for (int64_t j = 0; j < n; ++j) out[s + j] /= tot;
        }
    }
}

/* Key-segmented flavour (scan_cub.cu:18-56): a segment is a maximal run of
 * equal consecutive keys. */
ORC_API void orc_scan_by_key(
    int64_t n, const int64_t *keys, const float *in, float *out,
    int32_t op, int32_t inclusive, int32_t reverse)
{
    float acc = op ? 1.0f : 0.0f;
    for (int64_t j = 0; j < n; ++j) {
        const int64_t k = reverse ? n - 1 - j : j;
        const int64_t prev = reverse ? k + 1 : k - 1;
        if (j == 0 || keys[k] != keys[prev]) acc = op ? 1.0f : 0.0f;
        const float x = in[k];
        if (inclusive) { acc = op ? acc * x : acc + x; out[k] = acc; }
        else { out[k] = acc; acc = op ? acc * x : acc + x; }
    }
}

/* nerfacc/pack.py:38-46: counts by index_add, starts by exclusive cumsum. */
ORC_API void orc_pack_info(int64_t n, const int64_t *ray_indices, int32_t n_rays, int64_t *packed /* [n_rays,2] */)
{
    for (int32_t r = 0; r < n_rays; ++r) { packed[2 * r] = 0; packed[2 * r + 1] = 0; }
    for (int64_t i = 0; i < n; ++i) packed[2 * ray_indices[i] + 1] += 1;
    int64_t run = 0;
    for (int32_t r = 0; r < n_rays; ++r) { packed[2 * r] = run; run += packed[2 * r + 1]; }
}

/* ------------------------------------------------------------------ */
/* packed compositing (nerfacc/volrend.py)                             */
/* ------------------------------------------------------------------ */

/* Forward of rendering() for packed samples, density route:
 * volrend.py:271-277 (sigma*dt, alpha, trans), :375 (weights), :145-162
 * (colour / opacity / depth accumulation, expected depth, background).
 * f32 arithmetic, sequential accumulation in ray order.  Any of the
 * per-ray outputs may be NULL.  rgbs may be NULL (then colors must be). */
ORC_API void orc_composite_fwd(
    int32_t n_rays, const int64_t *starts, const int64_t *cnts,
    const float *t_starts, const float *t_ends, const float *sigmas, const float *rgbs,
    const float *prefix_trans, const float *bkgd, int32_t expected_depths,
    float *weights, float *trans, float *alphas,
    float *colors, float *opac, float *depths)
{
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t r = 0; r < n_rays; ++r) {
        const int64_t s = starts[r], n = cnts[r];
        float acc = 0.0f, C[3] = {0, 0, 0}, O = 0.0f, D = 0.0f;
        for (int64_t k = s; k < s + n; ++k) {
            const float sd = sigmas[k] * (t_ends[k] - t_starts[k]);
            const float a = 1.0f - expf(-sd);
            float T = expf(-acc);
            if (prefix_trans) T = T * prefix_trans[k];
            const float w = T * a;
            acc += sd;
            if (alphas) alphas[k] = a;
            if (trans) trans[k] = T;
            if (weights) weights[k] = w;
            if (rgbs) for (int c = 0; c < 3; ++c) C[c] += w * rgbs[3 * k + c];
            O += w;
            D += w * ((t_starts[k] + t_ends[k]) / 2.0f);
        }
        if (expected_depths) D = D / fmaxf(O, 1.1920929e-07f);
        if (bkgd) for (int c = 0; c < 3; ++c) C[c] = C[c] + bkgd[c] * (1.0f - O);
        if (colors) for (int c = 0; c < 3; ++c) colors[3 * r + c] = C[c];
        if (opac) opac[r] = O;
        if (depths) depths[r] = D;
    }
}

/* Same, alpha route (volrend.py:211-215, :322). */
ORC_API void orc_composite_alpha_fwd(
    int32_t n_rays, const int64_t *starts, const int64_t *cnts,
    const float *alphas, const float *prefix_trans, float *weights, float *trans)
{
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t r = 0; r < n_rays; ++r) {
        const int64_t s = starts[r], n = cnts[r];
        float T = 1.0f;
        for (int64_t k = s; k < s + n; ++k) {
            float Tk = T;
            if (prefix_trans) Tk = Tk * prefix_trans[k];
            if (trans) trans[k] = Tk;
            if (weights) weights[k] = Tk * alphas[k];
            T = T * (1.0f - alphas[k]);
        }
    }
}

/* Gradient of a scalar loss through orc_composite_fwd, in double precision.
 * Upstream grads: gC [R,3], gO [R], gD [R] on the *returned* colors /
 * opacities / depths (i.e. after expected-depth normalisation and background
 * blend), plus optional per-sample gW, gT, gA on extras.  Derived from the
 * op list at volrend.py:145-162,271-277,375 (SURVEY.md section 8a):
 *   g_i   = gC'.c_i + gO' + gD'.m_i + gW_i
 *   dL/ds_i = d_i [ (g_i T_i + gA_i)(1-a_i) - sum_{k>i} (g_k w_k + gT_k T_k) ]
 *   dL/dc_i = w_i gC'
 */
ORC_API void orc_composite_bwd(
    int32_t n_rays, const int64_t *starts, const int64_t *cnts,
    const float *t_starts, const float *t_ends, const float *sigmas, const float *rgbs,
    const float *prefix_trans, const float *bkgd, int32_t expected_depths,
    const float *gC, const float *gO, const float *gD,
    const float *gW, const float *gT, const float *gA,
    double *g_sigmas, double *g_rgbs)
{
#pragma omp parallel for schedule(dynamic, 256)
    for (int32_t r = 0; r < n_rays; ++r) {
        const int64_t s = starts[r], n = cnts[r];
        if (n == 0) continue;
        /* forward in double to get O, D_acc */
        double acc = 0, O = 0, Dacc = 0;
        for (int64_t k = s; k < s + n; ++k) {
            double dl = (double)t_ends[k] - (double)t_starts[k];
            double sd = (double)sigmas[k] * dl;
            double T = exp(-acc) * (prefix_trans ? (double)prefix_trans[k] : 1.0);
            double w = T * (1.0 - exp(-sd));
            O += w;
            Dacc += w * (((double)t_starts[k] + (double)t_ends[k]) / 2.0);
            acc += sd;
        }
        double gc[3] = {0, 0, 0}, go = gO ? gO[r] : 0.0, gd = gD ? gD[r] : 0.0;
        if (gC) for (int c = 0; c < 3; ++c) gc[c] = gC[3 * r + c];
        if (bkgd) for (int c = 0; c < 3; ++c) go -= gc[c] * (double)bkgd[c];
        if (expected_depths) {
            const double eps = 1.1920928955078125e-07;
            if (O > eps) { go -= gd * Dacc / (O * O); gd = gd / O; }
            else { gd = gd / eps; }
        }
        /* reverse sweep with suffix sum */
        double suffix = 0;
        double tot = acc;
        for (int64_t k = s + n - 1; k >= s; --k) {
            double dl = (double)t_ends[k] - (double)t_starts[k];
            double sd = (double)sigmas[k] * dl;
            tot -= sd;
            double T = exp(-tot) * (prefix_trans ? (double)prefix_trans[k] : 1.0);
            double a = 1.0 - exp(-sd);
            double w = T * a;
            double m = ((double)t_starts[k] + (double)t_ends[k]) / 2.0;
            double g = go + gd * m + (gW ? (double)gW[k] : 0.0);
            if (rgbs) for (int c = 0; c < 3; ++c) g += gc[c] * (double)rgbs[3 * k + c];
            double ga = gA ? (double)gA[k] : 0.0;
            g_sigmas[k] = dl * ((g * T + ga) * (1.0 - a) - suffix);
            if (g_rgbs) for (int c = 0; c < 3; ++c) g_rgbs[3 * k + c] = w * gc[c];
            suffix += g * w + (gT ? (double)gT[k] * T : 0.0);
        }
    }
}

/* nerfacc/volrend.py:546-561 with grouped indices. */
ORC_API void orc_accumulate(
    int32_t n_rays, int64_t n, const int64_t *ray_indices,
    const float *weights, const float *values, int32_t dim, float *out /* [n_rays, dim] zero-filled here */)
{
    memset(out, 0, sizeof(float) * (size_t)n_rays * (size_t)dim);
    for (int64_t i = 0; i < n; ++i)
        for (int32_t c = 0; c < dim; ++c)
            out[ray_indices[i] * dim + c] += values ? weights[i] * values[i * dim + c] : weights[i];
}

ORC_API void orc_set_num_threads(int32_t n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

ORC_API int32_t orc_num_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ------------------------------------------------------------------ */
/* PDF: importance sampling, searchsorted                              */
/* ------------------------------------------------------------------ */

/* nerfacc/cuda/csrc/pdf.cu:43-63 upper_bound (data_sort == nullptr) */
static int64_t pdf_upper_bound(const float *data, int64_t start, int64_t end, float val)
{
    while (start < end) {
        const int64_t mid = start + ((end - start) >> 1);
        const float mid_val = data[mid];
        if (!(mid_val > val)) start = mid + 1;
        else end = mid;
    }
    return start;
}

/* nerfacc/cuda/csrc/pdf.cu:65-80 binary_search_chunk_id */
static int32_t pdf_chunk_id(int64_t item, int32_t n_chunks, const int64_t *starts /* stride 2 */)
{
    int32_t start = 0, end = n_chunks;
    while (start < end) {
        const int32_t mid = start + ((end - start) >> 1);
        if (!(starts[2 * (int64_t)mid] > item)) start = mid + 1;
        else end = mid;
    }
    return start;
}

static inline int64_t clamp_i64(int64_t v, int64_t lo, int64_t hi) { int64_t m = v < hi ? v : hi; return m > lo ? m : lo; }

/* cuRAND Philox4x32-10 (curand_philox4x32_x.h of the CUDA toolkit the reference links; algorithm of
 * Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC'11).
 * curand_init(seed, subsequence, offset): key = (seed lo, seed hi); counter = 0; the subsequence is added
 * to the upper 64 counter bits, offset / 4 to the lower 64, offset % 4 selects the output word.
 * curand_uniform(): x * 2^-32 + 2^-33 as one FMA (SASS of pdf.cu:144). */
ORC_API uint32_t orc_philox_word(uint64_t seed, uint64_t subsequence, uint64_t offset)
{
    uint32_t ctr[4] = {(uint32_t)(offset >> 2), (uint32_t)(offset >> 34), (uint32_t)subsequence, (uint32_t)(subsequence >> 32)};
    uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    for (int round = 0; round < 10; ++round) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * ctr[0];
        const uint64_t p1 = (uint64_t)0xCD9E8D57u * ctr[2];
        const uint32_t out[4] = {(uint32_t)(p1 >> 32) ^ ctr[1] ^ key[0], (uint32_t)p1,
                                 (uint32_t)(p0 >> 32) ^ ctr[3] ^ key[1], (uint32_t)p0};
        memcpy(ctr, out, sizeof(out));
        key[0] += 0x9E3779B9u;
        key[1] += 0xBB67AE85u;
    }
    return ctr[offset & 3u];
}

ORC_API float orc_philox_uniform(uint64_t seed, uint64_t subsequence, uint64_t offset)
{
    return fmaf((float)orc_philox_word(seed, subsequence, offset), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
}

/* nerfacc/cuda/csrc/pdf.cu:97-166 importance_sampling_kernel followed by :168-243 compute_intervels_kernel,
 * one loop iteration per device thread.  in_packed / out_packed NULL = batched.  For flattened output the
 * edges' (start, count) come in iv_packed (count = n + 1 for n > 0, else 0; pdf.cu:341-344).
 * A ray resampled to a single sample reads samples.vals[tid + 1] in the reference ("FIXME: out of bounds?",
 * pdf.cu:208) and never writes its right edge: undefined there, [t_min, t_max] here. */
ORC_API void orc_importance_sampling(
    int32_t n_rays, const float *vals, const float *cdfs, const int64_t *in_packed, int64_t in_edges,
    const int64_t *out_packed, const int64_t *iv_packed, int64_t n_out, int32_t stratified, uint64_t seed,
    uint64_t offset, float *sample_vals, int64_t *sample_ray, float *iv_vals, int64_t *iv_ray, uint8_t *iv_left,
    uint8_t *iv_right)
{
    for (int32_t ray_id = 0; ray_id < n_rays; ++ray_id) {
        const int64_t n_samples = out_packed ? out_packed[2 * (int64_t)ray_id + 1] : n_out;
        const int64_t sbase = out_packed ? out_packed[2 * (int64_t)ray_id] : (int64_t)ray_id * n_out;
        const int64_t base = in_packed ? in_packed[2 * (int64_t)ray_id] : (int64_t)ray_id * in_edges;
        const int64_t last = base + (in_packed ? in_packed[2 * (int64_t)ray_id + 1] : in_edges) - 1;
        const int64_t base_out = out_packed ? iv_packed[2 * (int64_t)ray_id] : (int64_t)ray_id * (n_out + 1);
        if (n_samples <= 0) continue;
        /* --- samples --- */
        for (int64_t sid = 0; sid < n_samples; ++sid) {
            const int64_t tid = sbase + sid;
            if (out_packed && sample_ray) sample_ray[tid] = ray_id;
            const float u_floor = cdfs[base];
            const float u_ceil = cdfs[last];
            const float u_step = (u_ceil - u_floor) / (float)n_samples;
            float bias = 0.5f;
            if (stratified) bias = orc_philox_uniform(seed, (uint64_t)ray_id, offset);
            const float u = fmaf((float)sid + bias, u_step, u_floor);
            const int64_t p = pdf_upper_bound(cdfs, base, last, u);
            const int64_t p0 = clamp_i64(p - 1, base, last);
            const int64_t p1 = clamp_i64(p, base, last);
            const float u_lower = cdfs[p0], u_upper = cdfs[p1];
            const float t_lower = vals[p0], t_upper = vals[p1];
            float t;
            if (u_upper - u_lower < 1e-10f) {
                t = (t_lower + t_upper) * 0.5f;
            } else {
                const float scaling = (t_upper - t_lower) / (u_upper - u_lower);
                t = fmaf(u - u_lower, scaling, t_lower);
            }
            sample_vals[tid] = t;
        }
        /* --- edges --- */
        const float t_min = vals[base], t_max = vals[last];
        if (n_samples == 1) {
            iv_vals[base_out] = t_min;
            iv_vals[base_out + 1] = t_max;
        }
        for (int64_t sid = 0; sid < n_samples && n_samples > 1; ++sid) {
            const int64_t tid = sbase + sid;
            if (sid == 0) {
                const float t = sample_vals[tid], t_next = sample_vals[tid + 1];
                const float half_width = (t_next - t) * 0.5f;
                iv_vals[base_out] = fmaxf(t - half_width, t_min);
            } else {
                const float t = sample_vals[tid], t_prev = sample_vals[tid - 1];
                iv_vals[base_out + sid] = (t + t_prev) * 0.5f;
                if (sid == n_samples - 1) {
                    const float half_width = (t - t_prev) * 0.5f;
                    iv_vals[base_out + sid + 1] = fminf(t + half_width, t_max);
                }
            }
        }
        if (out_packed)
            for (int64_t k = 0; k <= n_samples; ++k) {
                iv_ray[base_out + k] = ray_id;
                iv_left[base_out + k] = k < n_samples;
                iv_right[base_out + k] = k > 0;
            }
    }
}

/* nerfacc/cuda/csrc/pdf.cu:247-287 searchsorted_kernel */
ORC_API void orc_searchsorted(
    int64_t n_query, const float *q_vals, const int64_t *q_packed, const int64_t *q_ray, int32_t n_rays,
    int64_t q_edges, const float *k_vals, const int64_t *k_packed, int64_t k_edges, int64_t *ids_left,
    int64_t *ids_right)
{
    for (int64_t tid = 0; tid < n_query; ++tid) {
        int64_t ray_id;
        if (!q_packed) ray_id = tid / q_edges;
        else if (!q_ray) ray_id = pdf_chunk_id(tid, n_rays, q_packed) - 1;
        else ray_id = q_ray[tid];
        const int64_t base = k_packed ? k_packed[2 * ray_id] : ray_id * k_edges;
        const int64_t last = base + (k_packed ? k_packed[2 * ray_id + 1] : k_edges) - 1;
        const int64_t p = pdf_upper_bound(k_vals, base, last, q_vals[tid]);
        const int64_t rel = q_packed ? 0 : base;
        ids_left[tid] = clamp_i64(p - 1, base, last) - rel;
        ids_right[tid] = clamp_i64(p, base, last) - rel;
    }
}

/* ------------------------------------------------------------------------- */
/* grid maintenance: OccGridEstimator._update                                 */
/* (nerfacc/estimators/occ_grid.py:367-404); pinned by tests/golden/ref_occ_update.npz */
/* ------------------------------------------------------------------------- */

/* occ_grid.py:395-398  occs[ids] = maximum(occs[ids] * ema_decay, occ).  The right-hand side is evaluated on the
 * OLD values for every draw before anything is written (index_put_); when `ids` names a cell more than once
 * torch keeps one of the candidates (the last one on the CPU, an arbitrary one on CUDA) -- this restatement
 * keeps the largest, the only rule that does not depend on the order of the writes: largest in the total order
 * -inf < ... < -0.0 < +0.0 < ... < +inf, NaN if any candidate is NaN.  `fresh`: n floats. */
ORC_API void orc_occ_ema_update(int64_t n, const int64_t* ids, const float* occ, float ema_decay, float* occs,
                                float* fresh)
{
    for (int64_t i = 0; i < n; ++i) {
        const float a = occs[ids[i]] * ema_decay, b = occ[i];
        fresh[i] = (a != a || b != b) ? NAN : (a > b ? a : b); /* torch.maximum propagates NaN */
    }
    for (int64_t i = 0; i < n; ++i) occs[ids[i]] = -INFINITY;
    for (int64_t i = 0; i < n; ++i) {
        float* dst = occs + ids[i];
        if (fresh[i] != fresh[i] || *dst != *dst) *dst = NAN;
        else if (fresh[i] > *dst || (fresh[i] == *dst && signbit(*dst) && !signbit(fresh[i]))) *dst = fresh[i];
    }
}

/* occ_grid.py:400-404  thre = clamp(occs[occs >= 0].mean(), max=occ_thre); binaries = occs > thre.
 * The mean is accumulated in double (torch reduces in float32 in an order of its own; the two agree to the last
 * bit or two of the mean, which only matters for a cell whose occupancy sits on the threshold).  Returns thre. */
ORC_API float orc_occ_threshold(int64_t n_cells, const float* occs, float occ_thre, uint8_t* binaries)
{
    double sum = 0.0;
    int64_t cnt = 0;
    for (int64_t i = 0; i < n_cells; ++i)
        if (occs[i] >= 0.0f) { sum += occs[i]; ++cnt; }
    const float mean = cnt ? (float)(sum / (double)cnt) : NAN;
    const float thre = (mean != mean) ? mean : (mean < occ_thre ? mean : occ_thre);
    for (int64_t i = 0; i < n_cells; ++i) binaries[i] = occs[i] > thre ? 1 : 0;
    return thre;
}
