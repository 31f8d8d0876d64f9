// march_generic.cuh -- every traverse_grids mode the closed-form fast path does not cover.
//
// cone_angle > 0 (the step grows with t, so there is no single lattice), step_size <= 0
// (one sample per occupied cell), traverse_steps_limit, over_allocate and rays_mask
// (/root/reference/nerfacc/cuda/csrc/grid.cu:68-282, launches :364-470).  One thread marches one
// ray sample by sample, in the reference's order of operations; a first pass counts, a second
// fills at the scanned offsets (or one pass into fixed-stride slots when over-allocating).
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

// March one ray.  Returns the terminate plane (reference grid.cu:274-275).
template <class Boxes>
NFA_HD float generic_march_ray(const Boxes& boxes, const OccView& occ, const float o[3], const float d[3],
                               float near, float far, float step, float cone, int32_t limit, GenericOut& out)
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
