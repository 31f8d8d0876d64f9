// march.cuh -- per-ray occupancy-grid traversal, constant-step fast path.
//
// Restates the semantics of the reference's traverse_grids_kernel
// (/root/reference/nerfacc/cuda/csrc/grid.cu:68-282 with the helpers in
// include/utils_grid.cuh:10-142) for cone_angle == 0 and step_size > 0, split
// into two phases so that a warp of unrelated rays stays convergent:
//
//  phase 1 (walk_*)  the DDA walks cells exactly like the reference (same f32
//                    evaluation order and FMA contraction as the reference's
//                    SASS, see DESIGN.md) but does no marching at all:
//                    it only records *stretches* -- maximal chains of occupied
//                    cells -- as (pend, open) pairs in the time domain:
//                    `pend` = where the reference's skip loops would have moved
//                    t_last before the stretch, `open` = exit time of its last cell.
//  phase 2 (lat_*)   turns stretches into runs (t_first, n) of consecutive lattice
//                    samples with two closed-form seeks each (lattice.cuh).  All
//                    lanes do this at the same time, so the expensive integer
//                    code is not serialised by divergence; on one grid level the
//                    stretches of a warp's rays are independent and are dealt out
//                    to the lanes (lat_anchor / lat_stretch / lat_take), nested
//                    levels take a ray's stretches in order (lat_consume).
//
// The per-sample arrays are produced later by the expand kernel from the runs.
// The code is host+device so that tests/host_sim can run the very same logic on
// the CPU against the oracle (oracle/oracle.c) without a GPU.
#pragma once

#include "lattice.cuh"

namespace nfa {

// ---------------------------------------------------------------------------
// Bit-packed occupancy: 4x4x4-cell bricks, one uint64 per brick, plus a
// 2-bit-per-brick class mip (bit 0: some cell occupied, bit 1: all 64 cells
// occupied; so 0 = empty, 1 = mixed, 3 = full) that the generic traversal reads
// (march_generic.cuh).  Derived cache of the estimator's bool `binaries`
// (reference estimators/occ_grid.py:73-76).
// ---------------------------------------------------------------------------
struct OccGeom {
    int res[3];   // cells per axis
    int nb[3];    // bricks per axis = ceil(res/4)
    int wpl;      // words (bricks) per level
    int n_grids;
};

NFA_HD OccGeom occ_geom(int n_grids, int rx, int ry, int rz)
{
    OccGeom g;
    g.res[0] = rx; g.res[1] = ry; g.res[2] = rz;
    g.nb[0] = (rx + 3) >> 2; g.nb[1] = (ry + 3) >> 2; g.nb[2] = (rz + 3) >> 2;
    g.wpl = g.nb[0] * g.nb[1] * g.nb[2];
    g.n_grids = n_grids;
    return g;
}

struct OccView {
    const uint64_t* words;   // [n_grids * wpl]
    const uint32_t* coarse;  // class mip, 16 bricks per word: [(n_grids * wpl + 15) / 16]
    const int32_t* bounds;   // [n_grids][6] bounding box of the non-empty bricks (brick units,
                             // min xyz then max xyz, inclusive; min > max: level empty), or null
    OccGeom g;
};

enum : uint32_t { kBrickEmpty = 0u, kBrickMixed = 1u, kBrickFull = 3u };

// ---------------------------------------------------------------------------
// Ray / box slab test: reference utils_grid.cuh:10-55.
// ---------------------------------------------------------------------------
NFA_HD bool slab_test(const float o[3], const float inv[3], const float* box,
                      float near, float far, float& tmin, float& tmax)
{
    float lo = 0.f, hi = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        float t_lo, t_hi;
        if (inv[a] >= 0.0f) {
            t_lo = f_mul(f_sub(box[a], o[a]), inv[a]);
            t_hi = f_mul(f_sub(box[3 + a], o[a]), inv[a]);
        } else {
            t_lo = f_mul(f_sub(box[3 + a], o[a]), inv[a]);
            t_hi = f_mul(f_sub(box[a], o[a]), inv[a]);
        }
        if (a == 0) {
            lo = t_lo;
            hi = t_hi;
        } else {
            if (lo > t_hi || t_lo > hi) return false;
            if (t_lo > lo) lo = t_lo;
            if (t_hi < hi) hi = t_hi;
        }
    }
    if (hi <= 0.0f) return false;
    tmin = f_max(lo, near);
    tmax = f_min(hi, far);
    return true;
}

// ---------------------------------------------------------------------------
// DDA over one (ray, level, [seg_lo, seg_hi]) segment.
// Set-up: reference utils_grid.cuh:58-114; step: utils_grid.cuh:116-142.
// ---------------------------------------------------------------------------
struct Dda {
    float td[3], dl[3];
    int cur[3], st[3], ov[3];
};

NFA_HD void dda_begin(Dda& s, const float o[3], const float d[3], const float inv[3],
                      float tmin, float tmax, const float* box, const int res[3])
{
    const float eps = 1e-6f;  // reference grid.cu:95
    const float t_in = f_add(tmin, eps);
    const float t_out = f_add(tmax, -eps);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float resf = (float)res[a];
        const float extent = f_sub(box[3 + a], box[a]);
        const float voxel = f_div(extent, resf);
        const float p_in = f_fma(d[a], t_in, o[a]);
        const float p_out = f_fma(d[a], t_out, o[a]);
        const int first = i_clamp(f_trunc_i32(f_mul(f_div(f_sub(p_in, box[a]), extent), resf)), 0, res[a] - 1);
        const int last = i_clamp(f_trunc_i32(f_mul(f_div(f_sub(p_out, box[a]), extent), resf)), 0, res[a] - 1);
        const int ahead = d[a] > 0.0f ? 1 : 0;
        const float face = (float)(uint32_t)(first + ahead);
        const float cross = f_fma(inv[a], f_add(box[a], f_fma(face, voxel, -p_in)), tmin);
        if (d[a] == 0.0f) {
            s.td[a] = tmax;
            s.dl[a] = tmax;
            s.st[a] = 0;
        } else {
            s.td[a] = cross;
            const float m = f_mul(inv[a], voxel);
            s.dl[a] = d[a] > 0.0f ? m : -m;
            s.st[a] = d[a] > 0.0f ? 1 : -1;
        }
        s.cur[a] = first;
        s.ov[a] = last + s.st[a];
    }
}

// ---------------------------------------------------------------------------
// Phase 1: the walk.  Events of the reference kernel, per ray:
//   SEG(lo)   segment start: `if (!continuous)` skip to lo        grid.cu:153-163
//   EMPTY(tt) empty cell: skip past its exit tt, continuous=false grid.cu:194-205
//   OCC(tt)   occupied cell: emit samples while mid < tt          grid.cu:206-262
// A stretch is a maximal event sequence without EMPTY.  `continuous` is false at
// its start and turns true at its first emitted sample, so inside a stretch a
// later SEG only skips if nothing was emitted yet: such a SEG splits the stretch
// into a second, `joined` descriptor whose pend is applied conditionally.
// ---------------------------------------------------------------------------
struct Walk {
    // ray
    float o[3], d[3], inv[3];
    float near, far;
    // segment iteration
    int seg_i;       // next crossing index to look at
    int level;
    float seg_hi;
    // DDA of the current segment, kept in scalars (reference utils_grid.cuh:58-142)
    float tdx, tdy, tdz;   // next crossing time per axis
    float dlx, dly, dlz;   // crossing-time increment per axis
    int remx, remy, remz;  // steps left on the axis before the walk ends (overflow index or grid edge)
    // occupancy cursor: current brick word + bit of the current cell inside it, and what one step along an
    // axis adds to them (0 for an axis the ray does not move along)
    int dbx, dby, dbz;     // to `bit`: +-16, +-4, +-1
    int sbx, sby, sbz;     // to `brick` when the step leaves the brick: +-nb[1]*nb[2], +-nb[2], +-1
    int brick;
    int bit;               // (x&3)<<4 | (y&3)<<2 | (z&3)
    uint64_t word;
    // state flags (ints, not bools: the compiler would byte-pack bools and shuffle them around)
    int in_seg;
    int open;        // inside a stretch (no EMPTY since it began)
    int joined;      // the current descriptor continues the previous one (SEG inside a stretch)
    int done;
    // empty-space acceleration (single level, no terminate plane wanted): see walk_open_segment
    int accel;
    float t_stop;
    // stretch under construction.  `pend` is the skip target: while no stretch is open it
    // accumulates (max) the exits of empty cells / segment starts; once a stretch opens it is
    // frozen and becomes that stretch's pend.  `d_open` is the exit of the stretch's last occupied
    // cell, -inf while the current descriptor has not seen one.
    float pend, d_open;
};

NFA_HD void walk_init(Walk& w, const float o[3], const float d[3], float near, float far)
{
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        w.o[a] = o[a];
        w.d[a] = d[a];
        w.inv[a] = f_rcp(d[a]);
    }
    w.near = near;
    w.far = far;
    w.seg_i = 0;
    w.level = 0;
    w.seg_hi = 0.f;
    w.tdx = w.tdy = w.tdz = 0.f;
    w.dlx = w.dly = w.dlz = 0.f;
    w.remx = w.remy = w.remz = 0;
    w.dbx = w.dby = w.dbz = 0;
    w.sbx = w.sby = w.sbz = 0;
    w.brick = 0;
    w.bit = 0;
    w.word = 0;
    w.in_seg = 0;
    w.open = 0;
    w.joined = 0;
    w.done = 0;
    w.accel = 0;
    w.t_stop = INFINITY;
    w.pend = -INFINITY;
    w.d_open = -INFINITY;
}

NFA_HD void walk_load_brick(Walk& w, const OccView& occ)
{
    w.word = occ.words[w.brick];
}

// Steps left on one axis: until the index reaches the overflow index (reference
// utils_grid.cuh:121-139, `current == overflow` ends the walk) or leaves the grid
// (where the reference itself would read out of bounds).
NFA_HD int walk_steps_left(int first, int last, int st, int res)
{
    const int big = 0x7fffffff;
    if (st == 0) return first == last ? 1 : big;
    const int to_ov = (last - first) * st + 1;
    const int to_edge = st > 0 ? res - first : first + 1;
    return (to_ov >= 1 && to_ov < to_edge) ? to_ov : to_edge;
}

NFA_HD void walk_open_segment(Walk& w, const OccView& occ, int level, float lo, float hi, const float* box)
{
    Dda s;
    dda_begin(s, w.o, w.d, w.inv, lo, hi, box, occ.g.res);
    w.level = level;
    w.seg_hi = hi;
    w.t_stop = INFINITY;
    int remx = walk_steps_left(s.cur[0], s.ov[0] - s.st[0], s.st[0], occ.g.res[0]);
    int remy = walk_steps_left(s.cur[1], s.ov[1] - s.st[1], s.st[1], occ.g.res[1]);
    int remz = walk_steps_left(s.cur[2], s.ov[2] - s.st[2], s.st[2], occ.g.res[2]);

    // Empty-space acceleration.  Everything outside the bounding box of the non-empty bricks is
    // empty, and walking empty cells only moves the skip target forward.  So (a) jump the DDA to
    // where the ray enters that box -- the crossing times are chains td (+) dl (+) dl ..., i.e.
    // lattices, and "how many crossings lie before T" / "what is the chain value there" are the
    // closed-form seeks of lattice.cuh, so the state after the jump is bit-identical to having
    // stepped -- and (b) stop once the ray has left the box.  Used when nothing after the last
    // occupied cell is observable: one level, no terminate plane.  The box is grown by one cell,
    // far more than the rounding of this (inexact) slab test, and the first cell after the jump
    // is still outside the true box, so it re-establishes the skip target exactly.
    if (w.accel && occ.bounds != nullptr && !w.open) {
        const int32_t* bb = occ.bounds + 6 * level;
        bool dead = bb[0] > bb[3];
        float t_in = lo, t_out = hi;
        if (!dead) {
            float glo[3], ghi[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                const float voxel = (box[3 + a] - box[a]) / (float)occ.g.res[a];
                glo[a] = box[a] + (float)(4 * bb[a] - 1) * voxel;
                ghi[a] = box[a] + (float)(4 * bb[3 + a] + 5) * voxel;
            }
            const float gbox[6] = {glo[0], glo[1], glo[2], ghi[0], ghi[1], ghi[2]};
            float a0, a1;
            if (slab_test(w.o, w.inv, gbox, lo, hi, a0, a1)) {
                t_in = a0;
                t_out = a1;
            } else {
                dead = true;
            }
        }
        if (!dead && t_in > lo) {
            float t[3] = {s.td[0], s.td[1], s.td[2]};
            uint32_t n[3] = {0u, 0u, 0u};
            bool ok = true;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                Lattice La = lat_make(s.dl[a]);
                La.half = 0.0f;  // plain "first chain value >= target"
                ok = ok && lat_seek(La, t[a], t_in, n[a]);
            }
            if (ok) {
                if (n[0] >= (uint32_t)remx || n[1] >= (uint32_t)remy || n[2] >= (uint32_t)remz) {
                    dead = true;  // the walk ends before it reaches the occupied region
                } else {
                    s.td[0] = t[0]; s.td[1] = t[1]; s.td[2] = t[2];
                    remx -= (int)n[0]; remy -= (int)n[1]; remz -= (int)n[2];
                    s.cur[0] += s.st[0] * (int)n[0];
                    s.cur[1] += s.st[1] * (int)n[1];
                    s.cur[2] += s.st[2] * (int)n[2];
                }
            }
        }
        if (dead) {  // nothing occupied on this segment
            w.in_seg = 0;
            return;
        }
        w.t_stop = t_out;
    }
    w.tdx = s.td[0]; w.tdy = s.td[1]; w.tdz = s.td[2];
    w.dlx = s.dl[0]; w.dly = s.dl[1]; w.dlz = s.dl[2];
    w.dbx = s.st[0] * 16; w.dby = s.st[1] * 4; w.dbz = s.st[2];
    w.sbx = s.st[0] * occ.g.nb[1] * occ.g.nb[2]; w.sby = s.st[1] * occ.g.nb[2]; w.sbz = s.st[2];
    w.remx = remx; w.remy = remy; w.remz = remz;
    w.brick = ((s.cur[0] >> 2) * occ.g.nb[1] + (s.cur[1] >> 2)) * occ.g.nb[2] + (s.cur[2] >> 2) + level * occ.g.wpl;
    w.bit = ((s.cur[0] & 3) << 4) | ((s.cur[1] & 3) << 2) | (s.cur[2] & 3);
    walk_load_brick(w, occ);
    w.in_seg = 1;
}

// Crossing source for a single grid level: what ray_aabb_intersect + torch.sort
// produce for n_grids == 1 (reference grid.py:156-162), computed in place.
struct SingleBox {
    const float* box;
    NFA_HD const float* aabb(int) const { return box; }
    // next valid segment at or after index i (i is advanced past it); false when exhausted
    NFA_HD bool next(const Walk& w, int& i, int& level, float& lo, float& hi) const
    {
        if (i > 0) return false;
        i = 1;
        float tmin, tmax;
        if (!slab_test(w.o, w.inv, box, -INFINITY, INFINITY, tmin, tmax)) return false;
        lo = f_max(tmin, w.near);
        hi = f_min(tmax, w.far);
        level = 0;
        return !(lo >= hi);
    }
};

// Crossings given sorted (reference grid.cu:129-150).
struct SortedBoxes {
    const float* aabbs;
    int G;
    const float* t_sorted;     // this ray's [2G]
    const int64_t* t_indices;  // this ray's [2G]
    const uint8_t* hits;       // this ray's [G]
    NFA_HD const float* aabb(int level) const { return aabbs + 6 * level; }
    NFA_HD bool next(const Walk& w, int& i, int& level, float& lo, float& hi) const
    {
        for (; i < 2 * G - 1; ++i) {
            const int64_t id = t_indices[i];
            int lv = (int)(id % G);
            if (!hits[lv]) continue;
            if (!(id < G)) {  // leaving this box: go on only if still inside the next one
                const int64_t nx = t_indices[i + 1];
                if (nx < G) continue;
                lv = (int)(nx % G);
                if (!hits[lv]) continue;
            }
            lo = f_max(t_sorted[i], w.near);
            hi = f_min(t_sorted[i + 1], w.far);
            if (lo >= hi) continue;
            level = lv;
            ++i;
            return true;
        }
        return false;
    }
};

// Walk until the ray is finished or `cap` descriptors are buffered.  Descriptors are
// appended through `buf.put(j, pend, open, joined)`; the caller flushes the buffer
// (phase 2) and calls again to resume.  A descriptor without occupied cells (open =
// -inf) still carries its conditional skip.
template <class Boxes, class Buf>
NFA_HD void walk_run(Walk& w, const Boxes& boxes, const OccView& occ, Buf& buf, int& n_desc, int cap)
{
    while (!w.done && n_desc < cap) {
        if (!w.in_seg) {
            int level;
            float lo, hi;
            if (!boxes.next(w, w.seg_i, level, lo, hi)) {
                if (w.open) buf.put(n_desc++, w.pend, w.d_open, w.joined != 0);
                w.done = 1;
                return;
            }
            // SEG(lo)
            if (w.open) {
                buf.put(n_desc++, w.pend, w.d_open, w.joined != 0);
                w.pend = lo;
                w.joined = 1;
                w.d_open = -INFINITY;
            } else {
                w.pend = f_max(w.pend, lo);
            }
            walk_open_segment(w, occ, level, lo, hi, boxes.aabb(level));
            continue;
        }
        // Cells of the current segment, on local scalars: one pass = one cell of the reference's loop
        // (grid.cu:184-271).  The lanes of a warp follow unrelated rays, so the pass has no branch but the rare
        // stretch boundary: the axis choice, the counters and the occupancy cursor are selects.
        float tdx = w.tdx, tdy = w.tdy, tdz = w.tdz;
        int remx = w.remx, remy = w.remy, remz = w.remz;
        int bit = w.bit, brick = w.brick;
        uint64_t word = w.word;
        int open = w.open, joined = w.joined;
        float pend = w.pend, d_open = w.d_open;
        const float dlx = w.dlx, dly = w.dly, dlz = w.dlz, seg_hi = w.seg_hi, t_stop = w.t_stop;
        const int dbx = w.dbx, dby = w.dby, dbz = w.dbz, sbx = w.sbx, sby = w.sby, sbz = w.sbz;
        int in_seg = 1;
        while (in_seg && n_desc < cap) {
            const float tt = f_min(f_min(tdx, f_min(tdy, tdz)), seg_hi);  // grid.cu:185-186
            // --- the DDA step first (utils_grid.cuh:116-142: x only if strictly smallest, else y if strictly
            // below z, else z).  It does not depend on the occupancy, and the brick word that the previous pass
            // may have requested has these ~30 instructions to arrive before the bit test below reads it.
            // The occupancy cursor moves along the stepped axis: add inside the axis' 2-bit field of `bit`; a
            // carry / borrow out of the field means the step left the brick.
            const bool mx = tdx < tdy && tdx < tdz;
            const bool my = !mx && (tdy < tdz);
            const bool mz = !mx && !my;
            tdx = mx ? f_add(tdx, dlx) : tdx;
            tdy = my ? f_add(tdy, dly) : tdy;
            tdz = mz ? f_add(tdz, dlz) : tdz;
            remx -= mx ? 1 : 0;
            remy -= my ? 1 : 0;
            remz -= mz ? 1 : 0;
            const int db = mx ? dbx : (my ? dby : dbz);
            const int mk = mx ? 0x30 : (my ? 0x0c : 0x03);
            const int sb = mx ? sbx : (my ? sby : sbz);
            const int nb = bit + db;
            const bool crossed = ((nb ^ bit) & ~mk) != 0;
            const int bit_next = (bit & ~mk) | (nb & mk);
            // only the stepped counter changed and all three were positive: one of them is 0 <=> that one is
            const int rem_min = remx < remy ? (remx < remz ? remx : remz) : (remy < remz ? remy : remz);
            const bool stop = rem_min == 0 || tt >= t_stop;  // overflow index / grid edge, or past the occupied box

            // --- the cell just left: OCC(tt) / EMPTY(tt)
            const int occd = (int)((uint32_t)(word >> bit) & 1u);
            if (occd != open) {  // a stretch opens (its pend is frozen from here on) or closes
                if (open) {      // EMPTY(tt) closes the stretch
                    buf.put(n_desc++, pend, d_open, joined != 0);
                    pend = -INFINITY;
                } else {
                    joined = 0;
                }
                open = occd;
            }
            if (occd) d_open = tt;             // the stretch grows
            else pend = f_max(pend, tt);       // the skip target moves on

            // --- commit the step
            bit = bit_next;
#ifdef __CUDA_ARCH__
            in_seg = stop ? 0 : 1;
            brick += crossed ? sb : 0;
            {   // predicated load: a branch here costs more than the load it skips
                const uint64_t* src = occ.words + brick;
                asm volatile("{\n.reg .pred p;\nsetp.ne.s32 p, %2, 0;\n@p ld.global.nc.u64 %0, [%1];\n}"
                             : "+l"(word) : "l"(src), "r"((int)(crossed && !stop)));
            }
#else
            if (stop) {
                in_seg = 0;
            } else if (crossed) {
                brick += sb;
                word = occ.words[brick];
            }
#endif
        }
        w.tdx = tdx; w.tdy = tdy; w.tdz = tdz;
        w.remx = remx; w.remy = remy; w.remz = remz;
        w.bit = bit; w.brick = brick; w.word = word;
        w.open = open; w.joined = joined;
        w.pend = pend; w.d_open = d_open;
        w.in_seg = in_seg;
    }
}

// Skip target still pending at the end of the ray (for the terminate plane, grid.cu:274-275).
NFA_HD float walk_tail_pend(const Walk& w)
{
    return w.open ? -INFINITY : w.pend;
}

// ---------------------------------------------------------------------------
// Phase 2: stretches -> runs on the lattice.  A run is a maximal chain of
// consecutive lattice samples, exactly the reference's `continuous` chains
// (grid.cu:219-245,258-259), so runs also delimit traverse_grids()' interval edges.
// ---------------------------------------------------------------------------
struct LatState {
    Lattice L;
    float t;          // lattice anchor (the reference's t_last once pending skips are applied)
    float run_first;
    uint32_t run_n;   // samples in the open run (> 0 <=> the reference's `continuous`)
    uint32_t n_samples, n_runs;
    bool ok;          // false once the lattice got stuck (the reference would not terminate)
};

struct RunOut {
    bool valid;
    float t_first;
    uint32_t n;
    uint32_t sample_off;  // samples of this ray before the run
    uint32_t run_idx;     // runs of this ray before the run
};

NFA_HD void lat_init(LatState& m, const Lattice& L, float near)
{
    m.L = L;
    m.t = near;
    m.run_first = 0.f;
    m.run_n = 0;
    m.n_samples = 0;
    m.n_runs = 0;
    m.ok = true;
}

NFA_HD void lat_close(LatState& m, RunOut& out)
{
    out.valid = m.run_n > 0;
    if (out.valid) {
        out.t_first = m.run_first;
        out.n = m.run_n;
        out.sample_off = m.n_samples;
        out.run_idx = m.n_runs;
        m.n_samples += m.run_n;
        m.n_runs += 1;
        m.run_n = 0;
    }
}

// Consume one descriptor; `out` reports the run that this descriptor closed, if any.
NFA_HD void lat_consume(LatState& m, float pend, float open, bool joined, RunOut& out)
{
    out.valid = false;
    if (!joined) lat_close(m, out);  // an EMPTY cell separated this stretch from the previous one
    if (!m.ok) return;
    uint32_t k = 0;
    if (m.run_n == 0) {
        m.ok = lat_seek(m.L, m.t, pend, k);
        if (!m.ok) return;
        m.run_first = m.t;
    }
    k = 0;
    m.ok = lat_seek(m.L, m.t, open, k);
    m.run_n += k;
}

// Phase 2 by stretch (one grid level).  There every stretch follows an EMPTY cell, so it is its own run, and the run's
// first sample and length depend only on the ray's lattice and the stretch's two times: the first lattice point with
// t + dt/2 >= target is the same whichever earlier lattice point the search starts from, and targets only grow along
// a ray.  So a ray's stretches need not be taken one after the other: lat_anchor() climbs to the first one (the long
// seek from `near`), lat_stretch() handles any stretch from that anchor (any lane may do it), and lat_take() adds the
// results up in order.  Same runs as lat_consume() on the same descriptors (tests/test_host_sim.py).
constexpr uint32_t kStretchFailed = 0xffffffffu;

NFA_HD void lat_anchor(LatState& m, const LatTable& table, float pend0)
{
    if (!m.ok) return;
    lat_table_jump(table, pend0, m.t);
    uint32_t k = 0;
    m.ok = lat_seek(m.L, m.t, pend0, k);
}

NFA_HD void lat_stretch(const Lattice& L, float anchor, bool ok, float pend, float open, float& first, uint32_t& n,
                        float& after)
{
    float t = anchor;
    uint32_t k = 0;
    ok = ok && lat_seek(L, t, pend, k);
    first = t;
    k = 0;
    ok = ok && lat_seek(L, t, open, k);
    n = ok ? k : kStretchFailed;
    after = t;
}

NFA_HD void lat_take(LatState& m, float first, uint32_t n, RunOut& out)
{
    out.valid = false;
    if (!m.ok) return;
    if (n == kStretchFailed) {
        m.ok = false;
        return;
    }
    if (n == 0u) return;
    out.valid = true;
    out.t_first = first;
    out.n = n;
    out.sample_off = m.n_samples;
    out.run_idx = m.n_runs;
    m.n_samples += n;
    m.n_runs += 1;
}

// End of ray: close the open run and (optionally) apply the trailing skip.
NFA_HD float lat_finish(LatState& m, float tail_pend, bool want_terminate, RunOut& out)
{
    lat_close(m, out);
    if (want_terminate && m.ok && tail_pend > -INFINITY) {
        uint32_t k = 0;
        m.ok = lat_seek(m.L, m.t, tail_pend, k);
    }
    return m.t;
}

}  // namespace nfa
