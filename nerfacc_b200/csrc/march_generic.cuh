// march_generic.cuh -- every traverse_grids mode the closed-form fast path does not cover.
//
// cone_angle > 0 (the step grows with t, so there is no single lattice), step_size <= 0
// (one sample per occupied cell), traverse_steps_limit, over_allocate and rays_mask
// (/root/reference/nerfacc/cuda/csrc/grid.cu:68-282, launches :364-470).  One thread marches one
// ray sample by sample, in the reference's order of operations; a first pass counts, a second
// fills at the scanned offsets (or one pass into fixed-stride slots when over-allocating).
// The same walk with a run sink (RunSink) feeds nfa_march / nfa_expand_samples with cone_angle > 0, the
// growing-step sampling path: runs instead of samples, one pass, replayed by the expand kernel.
// With a sample sink (SampleSink) it is the round march of render_test.cu: fixed-stride samples of the live rays.
// Reuses the DDA set-up, slab test, occupancy words and crossing iterators of march.cuh.
// Host+device so that tests/host_sim can check it against the oracle on the CPU.
#pragma once

#include "march.cuh"

namespace nfa {

NFA_HD uint32_t occ_class(const uint32_t* mip, int brick)
{
    return (mip[brick >> 4] >> ((brick & 15) << 1)) & 3u;
}

// the 64 cell bits of a brick: only mixed bricks are read from memory
NFA_HD uint64_t occ_brick_bits(const OccView& occ, int brick)
{
    const uint32_t c = occ_class(occ.coarse, brick);
    return c == kBrickMixed ? occ.words[brick] : (c == kBrickFull ? ~0ull : 0ull);
}

NFA_HD bool occ_test(const OccView& v, int level, int ix, int iy, int iz)
{
    const int b = ((ix >> 2) * v.g.nb[1] + (iy >> 2)) * v.g.nb[2] + (iz >> 2) + level * v.g.wpl;
    return (occ_brick_bits(v, b) >> (((ix & 3) << 4) | ((iy & 3) << 2) | (iz & 3))) & 1ull;
}

// reference grid.cu:23-28
NFA_HD float step_length(float t, float cone_angle, float dt_min)
{
    return f_max(dt_min, f_min(f_mul(t, cone_angle), 1e10f));
}

// Output sink: counts always; writes when `fill`.
struct GenericOut {
    bool fill;
    int64_t ray;
    // interval edges
    bool want_iv;
    int64_t iv_base;
    float* iv_vals;
    int64_t* iv_ray;
    uint8_t* iv_left;
    uint8_t* iv_right;
    // samples
    bool want_sm;
    int64_t sm_base;
    float* sm_vals;
    int64_t* sm_ray;
    uint8_t* sm_valid;
    // counters
    int64_t n_edges, n_samples;
};

// reference grid.cu:219-257: record one sample [t_last, t_next]
NFA_HD void generic_emit(GenericOut& o, float t_last, float t_next, bool continuous)
{
    if (o.want_iv) {
        if (!continuous) {
            if (o.fill) {
                const int64_t k = o.iv_base + o.n_edges;
                o.iv_vals[k] = t_last; o.iv_ray[k] = o.ray; o.iv_left[k] = 1;
                o.iv_vals[k + 1] = t_next; o.iv_ray[k + 1] = o.ray; o.iv_right[k + 1] = 1;
            }
            o.n_edges += 2;
        } else {
            if (o.fill) {
                const int64_t k = o.iv_base + o.n_edges;
                o.iv_vals[k] = t_next; o.iv_ray[k] = o.ray;
                o.iv_left[k - 1] = 1; o.iv_right[k] = 1;
            }
            o.n_edges += 1;
        }
    }
    if (o.want_sm && o.fill) {
        const int64_t k = o.sm_base + o.n_samples;
        o.sm_vals[k] = f_mul(f_add(t_next, t_last), 0.5f);
        o.sm_ray[k] = o.ray;
        o.sm_valid[k] = 1;
    }
    o.n_samples += 1;
}

// Run sink (march_cone_kernel): the samples of a ray as runs -- maximal chains of samples emitted with `continuous`
// set, each sample starting where the previous one ended.  An emission with `continuous == false` opens a run and
// the continuous ones that follow extend it; `continuous` is not reset between grid levels, so a run can span
// levels.  Inside a run every sample is [t, cone_next(t)] of the previous sample's end (the emission loop below
// computes t_next = t_last + step_length(t_last) and nothing else moves t_last between two such emissions), so a run
// is fully described by (t_first, n) and cone_expand_run() replays it bit for bit.  Closed runs go to
// `pool.put(sample_off, n, t_first, run_idx)`.
template <class Pool>
struct RunSink {
    Pool pool;
    int64_t n_samples;   // samples of the ray so far (generic_march_ray's step limit reads it)
    uint32_t n_runs;     // runs closed so far
    uint32_t run_off;    // samples of the ray before the open run
    uint32_t run_n;      // samples in the open run; 0: none open
    float run_first;     // start of the open run's first sample
};

template <class Pool>
NFA_HD void run_sink_init(RunSink<Pool>& o)
{
    o.n_samples = 0;
    o.n_runs = 0;
    o.run_off = 0;
    o.run_n = 0;
    o.run_first = 0.f;
}

// hand the open run (if any) to the pool; called by the next opening emission and once at the end of the ray
template <class Pool>
NFA_HD void run_sink_close(RunSink<Pool>& o)
{
    if (o.run_n == 0u) return;
    o.pool.put(o.run_off, o.run_n, o.run_first, o.n_runs);
    o.n_runs += 1;
    o.run_n = 0;
}

template <class Pool>
NFA_HD void generic_emit(RunSink<Pool>& o, float t_last, float t_next, bool continuous)
{
    (void)t_next;  // implied by t_last: see RunSink
    if (!continuous) {
        run_sink_close(o);
        o.run_off = (uint32_t)o.n_samples;
        o.run_first = t_last;
    }
    o.run_n += 1;
    o.n_samples += 1;
}

// Sample sink (render_test.cu, OccGridEstimator.render_test): sample j of the ray as (t_starts, t_ends) at slot
// base + j of two fixed-stride arrays.  t_start is t_last: an emission with `continuous` set starts where the previous
// one ended, so this is the interval form's vals[is_left] / vals[is_right] pair without the edges.  The caller's
// step limit bounds j.
struct SampleSink {
    float* t_starts;
    float* t_ends;
    int64_t base;
    int64_t n_samples;  // samples of the ray so far (generic_march_ray's step limit reads it)
};

NFA_HD void generic_emit(SampleSink& o, float t_last, float t_next, bool continuous)
{
    (void)continuous;
    o.t_starts[o.base + o.n_samples] = t_last;
    o.t_ends[o.base + o.n_samples] = t_next;
    o.n_samples += 1;
}

// The end of a sample that starts at t inside a run (reference grid.cu:215,259 with step_size > 0).
NFA_HD float cone_next(float t, float cone, float step) { return f_add(t, step_length(t, cone, step)); }

// The start of the sample j places after the one that starts at t, inside a run.
NFA_HD float cone_advance(float t, uint32_t j, float cone, float step)
{
    for (uint32_t s = 0; s < j; ++s) t = cone_next(t, cone, step);
    return t;
}

// Replay the run (t_first, n) into samples k0 .. k0 + n - 1 of the output arrays, none at or past `capacity`, in
// the order expand_cone_kernel uses: pieces of kExpandLanes samples, sample j of a piece computed by `lane` j from
// the piece's start, the next piece starting at the end of the last sample.
constexpr uint32_t kExpandLanes = 32;

NFA_HD void cone_expand_run(float t_first, uint32_t n, float cone, float step, int64_t ray, int64_t k0,
                            int64_t capacity, int64_t* ray_indices, float* t_starts, float* t_ends)
{
    float t = t_first;
    for (uint32_t base = 0; base < n; base += kExpandLanes) {
        const uint32_t m = n - base < kExpandLanes ? n - base : kExpandLanes;
        float last = t;
        for (uint32_t lane = 0; lane < m; ++lane) {
            const float ts = cone_advance(t, lane, cone, step);
            const float te = cone_next(ts, cone, step);
            const int64_t k = k0 + base + lane;
            if (k < capacity) {
                ray_indices[k] = ray;
                t_starts[k] = ts;
                t_ends[k] = te;
            }
            last = te;
        }
        t = last;
    }
}

// March one ray into the sink `out` (GenericOut, RunSink or SampleSink).  Returns the terminate plane (reference
// grid.cu:274-275).
template <class Boxes, class Out>
NFA_HD float generic_march_ray(const Boxes& boxes, const OccView& occ, const float o[3], const float d[3],
                               float near, float far, float step, float cone, int32_t limit, Out& out)
{
    Walk w;  // only the ray fields + segment iterator are used here
    walk_init(w, o, d, near, far);
    float t_last = near;
    bool continuous = false;
    int level;
    float lo, hi;
    while (boxes.next(w, w.seg_i, level, lo, hi)) {
        if (!continuous) {  // grid.cu:153-163
            if (step <= 0.0f) {
                t_last = lo;
            } else {
                const float dt = step_length(t_last, cone, step);
                const float half = f_mul(dt, 0.5f);
                for (int g = 0; g < (1 << 30) && !(f_add(t_last, half) >= lo); ++g) {
                    const float tn = f_add(t_last, dt);
                    if (!(tn > t_last)) break;  // stuck: the reference would spin forever
                    t_last = tn;
                }
            }
        }
        Dda s;
        dda_begin(s, w.o, w.d, w.inv, lo, hi, boxes.aabb(level), occ.g.res);
        for (int guard = 0; guard < (1 << 22) && (limit <= 0 || out.n_samples < limit); ++guard) {  // grid.cu:184
            if ((unsigned)s.cur[0] >= (unsigned)occ.g.res[0] || (unsigned)s.cur[1] >= (unsigned)occ.g.res[1] ||
                (unsigned)s.cur[2] >= (unsigned)occ.g.res[2])
                break;  // the reference reads out of bounds here
            const float tt = f_min(f_min(s.td[0], f_min(s.td[1], s.td[2])), hi);
            if (!occ_test(occ, level, s.cur[0], s.cur[1], s.cur[2])) {  // grid.cu:194-205
                if (step <= 0.0f) {
                    t_last = tt;
                } else {
                    const float dt = step_length(t_last, cone, step);
                    const float half = f_mul(dt, 0.5f);
                    for (int g = 0; g < (1 << 30) && !(f_add(t_last, half) >= tt); ++g) {
                        const float tn = f_add(t_last, dt);
                        if (!(tn > t_last)) break;
                        t_last = tn;
                    }
                }
                continuous = false;
            } else {  // grid.cu:206-262
                while (limit <= 0 || out.n_samples < limit) {
                    float t_next;
                    if (step <= 0.0f) {
                        t_next = tt;
                    } else {
                        const float dt = step_length(t_last, cone, step);
                        if (f_add(t_last, f_mul(dt, 0.5f)) >= tt) break;
                        t_next = f_add(t_last, dt);
                    }
                    generic_emit(out, t_last, t_next, continuous);
                    continuous = true;
                    const bool stuck = !(t_next > t_last) && step > 0.0f;
                    t_last = t_next;
                    if (t_next >= tt || stuck) break;
                }
            }
            // utils_grid.cuh:116-142
            int a;
            if (s.td[0] < s.td[1] && s.td[0] < s.td[2]) a = 0;
            else if (s.td[1] < s.td[2]) a = 1;
            else a = 2;
            bool leave;
            if (a == 0) { s.cur[0] += s.st[0]; s.td[0] = f_add(s.td[0], s.dl[0]); leave = s.cur[0] == s.ov[0]; }
            else if (a == 1) { s.cur[1] += s.st[1]; s.td[1] = f_add(s.td[1], s.dl[1]); leave = s.cur[1] == s.ov[1]; }
            else { s.cur[2] += s.st[2]; s.td[2] = f_add(s.td[2], s.dl[2]); leave = s.cur[2] == s.ov[2]; }
            if (leave) break;
        }
    }
    return t_last;
}

}  // namespace nfa
