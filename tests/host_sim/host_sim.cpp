// host_sim.cpp -- CPU build of the product's host+device traversal logic
// (nerfacc_b200/csrc/{lattice,march,expand,occ_pack}.cuh), for tests only.
//
// The kernels in nerfacc_b200/csrc/traverse.cu are thin thread/warp mappings
// around these headers; running the same headers on the CPU lets the
// `-m "not gpu"` suite check the closed-form lattice and the lazy march against
// the oracle's serial restatement of the reference.  This library is never
// loaded by the nerfacc_b200 package (there is no CPU fallback in the product).
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../nerfacc_b200/csrc/occ_pack.cuh"
#include "../../nerfacc_b200/csrc/expand.cuh"
#include "../../nerfacc_b200/csrc/march_generic.cuh"
#include "../../nerfacc_b200/csrc/pdf.cuh"

using namespace nfa;

extern "C" {

// serial reference chain: k steps of t += dt
float sim_chain(float t, float dt, uint32_t k)
{
    for (uint32_t i = 0; i < k; ++i) t = t + dt;
    return t;
}

// closed-form seek; returns ok flag
int sim_seek(float t0, float dt, float target, float* t_out, uint32_t* k_out)
{
    Lattice L = lat_make(dt);
    float t = t0;
    uint32_t k = 0;
    bool ok = lat_seek(L, t, target, k);
    *t_out = t;
    *k_out = k;
    return ok ? 1 : 0;
}

// first lattice point with t + dt/2 >= target, from `near`: plainly, and through the binade table (lattice.cuh)
int sim_seek_with_table(float dt, float near, float target, float* t_plain, float* t_table)
{
    const Lattice L = lat_make(dt);
    LatTable T;
    lat_table_build(L, near, T);
    float a = near, b = near;
    uint32_t ka = 0, kb = 0;
    const bool oka = lat_seek(L, a, target, ka);
    lat_table_jump(T, target, b);
    const bool okb = lat_seek(L, b, target, kb);
    *t_plain = a;
    *t_table = b;
    return (oka ? 1 : 0) | (okb ? 2 : 0) | (T.n << 2);
}

// expand one run into starts/ends
void sim_expand_run(float t_first, float dt, uint32_t n, float* starts, float* ends)
{
    Lattice L = lat_make(dt);
    RunIter it{t_first, n};
    uint32_t w = 0;
    while (it.left > 0) {
        LatPiece p;
        uint32_t c = run_next_piece(L, it, p);
        for (uint32_t j = 0; j < c; ++j) {
            starts[w] = piece_start(p, j);
            ends[w] = starts[w] + dt;
            ++w;
        }
    }
}

int64_t sim_occ_words(int n_grids, int rx, int ry, int rz) { return (int64_t)n_grids * occ_geom(n_grids, rx, ry, rz).wpl; }
int64_t sim_occ_coarse_words(int n_grids, int rx, int ry, int rz) { return occ_coarse_words(occ_geom(n_grids, rx, ry, rz)); }

void sim_occ_pack(int n_grids, int rx, int ry, int rz, const uint8_t* binaries, uint64_t* words, uint32_t* coarse,
                  int32_t* bounds)
{
    OccGeom g = occ_geom(n_grids, rx, ry, rz);
    memset(coarse, 0, sizeof(uint32_t) * occ_coarse_words(g));
    for (int l = 0; l < n_grids; ++l)
        for (int a = 0; a < 3; ++a) { bounds[6 * l + a] = kBoundsMinInit; bounds[6 * l + 3 + a] = kBoundsMaxInit; }
    const int64_t cells = (int64_t)rx * ry * rz;
    for (int l = 0; l < n_grids; ++l)
        for (int bx = 0; bx < g.nb[0]; ++bx)
            for (int by = 0; by < g.nb[1]; ++by)
                for (int bz = 0; bz < g.nb[2]; ++bz) {
                    const int b = (bx * g.nb[1] + by) * g.nb[2] + bz + l * g.wpl;
                    const uint64_t w = occ_brick_word(binaries + l * cells, g, bx, by, bz);
                    words[b] = w;
                    if (w) {
                        coarse[b >> 4] |= (w == ~0ull ? kBrickFull : kBrickMixed) << ((b & 15) << 1);
                        const int bc[3] = {bx, by, bz};
                        for (int a = 0; a < 3; ++a) {
                            if (bc[a] < bounds[6 * l + a]) bounds[6 * l + a] = bc[a];
                            if (bc[a] > bounds[6 * l + 3 + a]) bounds[6 * l + 3 + a] = bc[a];
                        }
                    }
                }
}

}  // extern "C"

static long g_by_stretch_rounds, g_tables;

// descriptor buffer with the capacity of the device kernel's per-ray slots (march_kernel: 8, or 16 when wide)
template <int kSlots>
struct HostBuf {
    enum { K = kSlots };
    float pend[K], open[K];
    bool joined[K];
    void put(int j, float p, float o, bool jn) { pend[j] = p; open[j] = o; joined[j] = jn; }
};

template <int kSlots, class Boxes>
static float march_one(const Boxes& boxes, const OccView& occ, const float* o, const float* d, float near, float far,
                       const Lattice& L, LatState& m, std::vector<float>& vt, std::vector<uint32_t>& vn, int accel)
{
    Walk w;
    walk_init(w, o, d, near, far);
    w.accel = accel;
    lat_init(m, L, near);
    HostBuf<kSlots> buf;
    int n_desc = 0;
    RunOut out;
    // same chunked structure as the kernel: walk until the buffer is full, then flush it
    for (long guard = 0; guard < (1L << 26); ++guard) {
        walk_run(w, boxes, occ, buf, n_desc, kSlots);
        for (int j = 0; j < n_desc; ++j) {
            lat_consume(m, buf.pend[j], buf.open[j], buf.joined[j], out);
            if (out.valid) { vt.push_back(out.t_first); vn.push_back(out.n); }
        }
        n_desc = 0;
        if (w.done) break;
    }
    const float term = lat_finish(m, walk_tail_pend(w), accel == 0, out);
    if (out.valid) { vt.push_back(out.t_first); vn.push_back(out.n); }
    return term;
}

// The kernel's phase 2 for one grid level: a round's stretches handled independently from one anchor
// (march.cuh: lat_anchor / lat_stretch / lat_take), the way march_kernel deals them out to the lanes of a warp.
template <int kSlots>
static float march_one_by_stretch(const OccView& occ, const float* box, const float* o, const float* d, float near,
                                  float far, const Lattice& L, LatState& m, std::vector<float>& vt,
                                  std::vector<uint32_t>& vn)
{
    SingleBox boxes{box};
    Walk w;
    walk_init(w, o, d, near, far);
    w.accel = 1;
    lat_init(m, L, near);
    LatTable table;  // (the kernel gets it from the host, for a uniform near plane; here every ray builds its own)
    lat_table_build(L, near, table);
    if (table.n > 0) ++g_tables;
    HostBuf<kSlots> buf;
    int n_desc = 0;
    RunOut out;
    for (long guard = 0; guard < (1L << 26); ++guard) {
        walk_run(w, boxes, occ, buf, n_desc, kSlots);
        bool any_joined = false;
        for (int j = 0; j < n_desc; ++j) any_joined = any_joined || buf.joined[j];
        if (any_joined) {
            for (int j = 0; j < n_desc; ++j) {
                lat_consume(m, buf.pend[j], buf.open[j], buf.joined[j], out);
                if (out.valid) { vt.push_back(out.t_first); vn.push_back(out.n); }
            }
        } else {
            ++g_by_stretch_rounds;
            if (m.run_n > 0) {
                lat_close(m, out);
                if (out.valid) { vt.push_back(out.t_first); vn.push_back(out.n); }
            }
            if (n_desc > 0) lat_anchor(m, table, buf.pend[0]);
            const float anchor = m.t;
            const bool ok = m.ok;
            float first[kSlots], after[kSlots];
            uint32_t cnt[kSlots];
            for (int j = n_desc - 1; j >= 0; --j)  // any order: here the last one first
                lat_stretch(L, anchor, ok, buf.pend[j], buf.open[j], first[j], cnt[j], after[j]);
            for (int j = 0; j < n_desc; ++j) {
                lat_take(m, first[j], cnt[j], out);
                if (out.valid) { vt.push_back(out.t_first); vn.push_back(out.n); }
            }
            if (n_desc > 0 && m.ok) m.t = after[n_desc - 1];
        }
        n_desc = 0;
        if (w.done) break;
    }
    const float term = lat_finish(m, walk_tail_pend(w), false, out);
    if (out.valid) { vt.push_back(out.t_first); vn.push_back(out.n); }
    return term;
}

// March all rays with a descriptor buffer of kSlots stretches; see sim_march.
template <int kSlots>
static int64_t march_all(int32_t n_rays, const float* rays_o, const float* rays_d, const float* near_planes,
                         const float* far_planes, int n_grids, int rx, int ry, int rz, const uint64_t* words,
                         const uint32_t* coarse, const int32_t* bounds, int accel, const float* aabbs,
                         const float* t_sorted, const int64_t* t_indices, const uint8_t* hits, float step_size,
                         int64_t* n_samples, int64_t* n_runs, float* terminate, int32_t* ok_flags, float* run_t,
                         uint32_t* run_n, int64_t run_capacity)
{
    OccView occ;
    occ.words = words;
    occ.coarse = coarse;
    occ.bounds = bounds;
    occ.g = occ_geom(n_grids, rx, ry, rz);
    const Lattice L = lat_make(step_size);
    int64_t total = 0;
    std::vector<float> vt;
    std::vector<uint32_t> vn;
    for (int32_t r = 0; r < n_rays; ++r) {
        vt.clear();
        vn.clear();
        LatState m;
        float term;
        if (t_sorted == nullptr && accel == 2) {  // accel == 2: phase 2 by stretch, as march_kernel does it for one level
            term = march_one_by_stretch<kSlots>(occ, aabbs, rays_o + 3 * r, rays_d + 3 * r, near_planes[r],
                                                far_planes[r], L, m, vt, vn);
        } else if (t_sorted == nullptr) {
            SingleBox b{aabbs};
            term = march_one<kSlots>(b, occ, rays_o + 3 * r, rays_d + 3 * r, near_planes[r], far_planes[r], L, m, vt,
                                     vn, accel);
        } else {
            SortedBoxes b{aabbs, n_grids, t_sorted + (int64_t)r * 2 * n_grids, t_indices + (int64_t)r * 2 * n_grids,
                          hits + (int64_t)r * n_grids};
            term = march_one<kSlots>(b, occ, rays_o + 3 * r, rays_d + 3 * r, near_planes[r], far_planes[r], L, m, vt,
                                     vn, 0);
        }
        n_samples[r] = m.n_samples;
        n_runs[r] = m.n_runs;
        terminate[r] = term;
        ok_flags[r] = m.ok ? 1 : 0;
        if (total + (int64_t)vt.size() > run_capacity) return -1;
        for (size_t q = 0; q < vt.size(); ++q) { run_t[total] = vt[q]; run_n[total] = vn[q]; ++total; }
    }
    return total;
}

extern "C" {

void sim_by_stretch_counts(long* out, int reset)
{
    out[0] = g_by_stretch_rounds;
    out[1] = g_tables;
    if (reset) g_by_stretch_rounds = g_tables = 0;
}

// March all rays; per ray: n_samples, n_runs, terminate plane; runs appended to
// flat arrays (caller passes capacity; returns total runs or -1 on overflow).
// `slots` stretch descriptors are buffered per ray between the two phases: 8 or 16, as the two widths of
// march_kernel (traverse.cu: kDescSlots / kDescSlotsWide); any other value returns -2.
int64_t sim_march_slots(int32_t n_rays, const float* rays_o, const float* rays_d,
                        const float* near_planes, const float* far_planes,
                        int n_grids, int rx, int ry, int rz, const uint64_t* words, const uint32_t* coarse,
                        const int32_t* bounds, int accel, const float* aabbs,
                        const float* t_sorted, const int64_t* t_indices, const uint8_t* hits,  // NULL => single level inline
                        float step_size,
                        int64_t* n_samples, int64_t* n_runs, float* terminate, int32_t* ok_flags,
                        float* run_t, uint32_t* run_n, int64_t run_capacity, int slots)
{
    if (slots == 8)
        return march_all<8>(n_rays, rays_o, rays_d, near_planes, far_planes, n_grids, rx, ry, rz, words, coarse, bounds,
                            accel, aabbs, t_sorted, t_indices, hits, step_size, n_samples, n_runs, terminate, ok_flags,
                            run_t, run_n, run_capacity);
    if (slots == 16)
        return march_all<16>(n_rays, rays_o, rays_d, near_planes, far_planes, n_grids, rx, ry, rz, words, coarse,
                             bounds, accel, aabbs, t_sorted, t_indices, hits, step_size, n_samples, n_runs, terminate,
                             ok_flags, run_t, run_n, run_capacity);
    return -2;
}

// the 8-slot march (march_kernel's narrow width)
int64_t sim_march(int32_t n_rays, const float* rays_o, const float* rays_d,
                  const float* near_planes, const float* far_planes,
                  int n_grids, int rx, int ry, int rz, const uint64_t* words, const uint32_t* coarse,
                  const int32_t* bounds, int accel, const float* aabbs,
                  const float* t_sorted, const int64_t* t_indices, const uint8_t* hits,
                  float step_size,
                  int64_t* n_samples, int64_t* n_runs, float* terminate, int32_t* ok_flags,
                  float* run_t, uint32_t* run_n, int64_t run_capacity)
{
    return sim_march_slots(n_rays, rays_o, rays_d, near_planes, far_planes, n_grids, rx, ry, rz, words, coarse, bounds,
                           accel, aabbs, t_sorted, t_indices, hits, step_size, n_samples, n_runs, terminate, ok_flags,
                           run_t, run_n, run_capacity, 8);
}


// Generic traversal (cone angle, per-cell sampling, step limits, masks): one pass over all rays.
// fill == 0: counts only (iv_cnts / sm_cnts written); fill == 1: arrays written at iv_starts / sm_starts.
void sim_generic_pass(int32_t n_rays, const float* rays_o, const float* rays_d, const uint8_t* rays_mask,
                      const float* near_planes, const float* far_planes,
                      int n_grids, int rx, int ry, int rz, const uint64_t* words, const uint32_t* coarse,
                      const float* aabbs, const float* t_sorted, const int64_t* t_indices, const uint8_t* hits,
                      float step_size, float cone_angle, int32_t limit, int32_t fill,
                      const int64_t* iv_starts, int64_t* iv_cnts, float* iv_vals, int64_t* iv_ray, uint8_t* iv_left,
                      uint8_t* iv_right, const int64_t* sm_starts, int64_t* sm_cnts, float* sm_vals, int64_t* sm_ray,
                      uint8_t* sm_valid, float* terminate)
{
    OccView occ;
    occ.words = words;
    occ.coarse = coarse;
    occ.bounds = nullptr;
    occ.g = occ_geom(n_grids, rx, ry, rz);
    for (int32_t r = 0; r < n_rays; ++r) {
        if (rays_mask && !rays_mask[r]) continue;                      // reference grid.cu:100
        if (fill && (iv_cnts[r] == 0 || sm_cnts[r] == 0)) continue;    // grid.cu:103-106
        GenericOut out;
        out.fill = fill != 0;
        out.ray = r;
        out.want_iv = true;
        out.want_sm = true;
        out.iv_base = fill ? iv_starts[r] : 0;
        out.sm_base = fill ? sm_starts[r] : 0;
        out.iv_vals = iv_vals; out.iv_ray = iv_ray; out.iv_left = iv_left; out.iv_right = iv_right;
        out.sm_vals = sm_vals; out.sm_ray = sm_ray; out.sm_valid = sm_valid;
        out.n_edges = 0;
        out.n_samples = 0;
        SortedBoxes b{aabbs, n_grids, t_sorted + (int64_t)r * 2 * n_grids, t_indices + (int64_t)r * 2 * n_grids,
                      hits + (int64_t)r * n_grids};
        const float term = generic_march_ray(b, occ, rays_o + 3 * r, rays_d + 3 * r, near_planes[r], far_planes[r],
                                             step_size, cone_angle, limit, out);
        if (terminate) terminate[r] = term;
        iv_cnts[r] = out.n_edges;
        sm_cnts[r] = out.n_samples;
    }
}

// ---- pdf.cuh: the per-ray body of importance_sampling_kernel (pdf.cu), threads serialised
float sim_philox_uniform(uint64_t seed, uint64_t subsequence, uint64_t offset)
{
    return philox_uniform(seed, subsequence, offset);
}

void sim_importance_sampling(int32_t n_rays, const float* vals, const float* cdfs, const int64_t* in_packed,
                             int64_t in_edges, const int64_t* out_packed, const int64_t* iv_packed, int64_t n_out,
                             int32_t stratified, uint64_t seed, uint64_t offset, float* sample_vals,
                             int64_t* sample_ray, float* iv_vals, int64_t* iv_ray, uint8_t* iv_left, uint8_t* iv_right,
                             float* t_starts, float* t_ends, float s_min, float s_max, int32_t lindisp)
{
    for (int32_t ray = 0; ray < n_rays; ++ray) {
        const int64_t base = in_packed ? in_packed[2 * (int64_t)ray] : (int64_t)ray * in_edges;
        const int64_t n_in = in_packed ? in_packed[2 * (int64_t)ray + 1] : in_edges;
        const int64_t n = out_packed ? out_packed[2 * (int64_t)ray + 1] : n_out;
        const int64_t s_base = out_packed ? out_packed[2 * (int64_t)ray] : (int64_t)ray * n;
        const int64_t e_base = out_packed ? iv_packed[2 * (int64_t)ray] : (int64_t)ray * (n + 1);
        if (n <= 0 || n_in <= 0) continue;
        const float* cdf = cdfs + base;
        const float* val = vals + base;
        float* ts = sample_vals + s_base;
        const float u_floor = cdf[0], u_ceil = cdf[n_in - 1];
        const float u_step = f_div(f_sub(u_ceil, u_floor), (float)n);
        const float bias = stratified ? philox_uniform(seed, (uint64_t)(int64_t)ray, offset) : 0.5f;
        for (int64_t sid = 0; sid < n; ++sid) {
            ts[sid] = is_invert<int64_t>(cdf, val, 0, n_in - 1, is_u<int64_t>(u_floor, u_step, sid, bias));
            if (sample_ray) sample_ray[s_base + sid] = ray;
        }
        for (int64_t k = 0; k <= n; ++k) {
            const float e = is_edge<int64_t>(ts, n, k, val[0], val[n_in - 1]);
            iv_vals[e_base + k] = e;
            if (out_packed) {
                iv_ray[e_base + k] = ray;
                iv_left[e_base + k] = k < n;
                iv_right[e_base + k] = k > 0;
            } else if (t_starts) {
                const float t = stot(e, s_min, s_max, lindisp != 0);
                if (k < n) t_starts[s_base + k] = t;
                if (k > 0) t_ends[s_base + k - 1] = t;
            }
        }
    }
}

void sim_searchsorted(int64_t n_query, const float* q_vals, const int64_t* q_packed, const int64_t* q_ray,
                      int32_t n_rays, int64_t q_edges, const float* k_vals, const int64_t* k_packed, int64_t k_edges,
                      int64_t* ids_left, int64_t* ids_right)
{
    for (int64_t i = 0; i < n_query; ++i) {
        int64_t ray;
        if (!q_packed) ray = i / q_edges;
        else if (q_ray) ray = q_ray[i];
        else ray = chunk_upper_bound(q_packed, n_rays, i) - 1;
        const int64_t base = k_packed ? k_packed[2 * ray] : ray * k_edges;
        const int64_t last = base + (k_packed ? k_packed[2 * ray + 1] : k_edges) - 1;
        const int64_t pos = upper_bound_f<int64_t>(k_vals, base, last, q_vals[i]);
        int64_t l = pos - 1 < last ? pos - 1 : last;
        if (l < base) l = base;
        int64_t r = pos < last ? pos : last;
        if (r < base) r = base;
        const int64_t rel = q_packed ? 0 : base;
        ids_left[i] = l - rel;
        ids_right[i] = r - rel;
    }
}

}  // extern "C"
