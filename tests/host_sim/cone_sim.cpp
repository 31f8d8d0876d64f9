// CPU build of the growing-step sampling path (cone_angle > 0): the walk of march_generic.cuh with the run sink that
// march_cone_kernel uses, then every run replayed by cone_expand_run as expand_cone_kernel does it.  The device-only
// parts (pool slots by atomics, the tile-wise scan) are replaced by their serial equivalents: runs in walk order,
// packed_info by an exclusive scan over the rays.  Compiled by tests/test_cone_host_sim.py with -ffp-contract=off.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../nerfacc_b200/csrc/occ_pack.cuh"
#include "../../nerfacc_b200/csrc/march_generic.cuh"

using namespace nfa;

namespace {

struct Run {
    uint32_t ray, sample_off, n;
    float t_first;
    uint32_t run_idx;
};

struct VecPool {
    std::vector<Run>* runs;
    uint32_t ray;
    void put(uint32_t sample_off, uint32_t n, float t_first, uint32_t run_idx)
    {
        runs->push_back(Run{ray, sample_off, n, t_first, run_idx});
    }
};

}  // namespace

extern "C" {

// Growing-step sampling of n_rays rays.  near_planes / far_planes: per ray, or both null for the scalars.
// t_sorted / t_indices / hits: the sorted box crossings, or null (one level: crossings computed per ray).
// Writes packed_info [n_rays, 2] and run_counts [n_rays]; writes the samples below `capacity`; returns their number.
int64_t sim_cone_sampling(int32_t n_rays, const float* rays_o, const float* rays_d, const float* near_planes,
                          const float* far_planes, float near_plane, float far_plane, int n_grids, int rx, int ry,
                          int rz, const uint8_t* binaries, const float* aabbs, const float* t_sorted,
                          const int64_t* t_indices, const uint8_t* hits, float step_size, float cone_angle,
                          int64_t* packed_info, int64_t* run_counts, int64_t capacity, int64_t* ray_indices,
                          float* t_starts, float* t_ends)
{
    const OccGeom g = occ_geom(n_grids, rx, ry, rz);
    std::vector<uint64_t> words((size_t)n_grids * g.wpl);
    std::vector<uint32_t> coarse((size_t)occ_coarse_words(g), 0u);
    const int64_t cells = (int64_t)rx * ry * rz;
    for (int l = 0; l < n_grids; ++l)
        for (int bx = 0; bx < g.nb[0]; ++bx)
            for (int by = 0; by < g.nb[1]; ++by)
                for (int bz = 0; bz < g.nb[2]; ++bz) {
                    const int b = (bx * g.nb[1] + by) * g.nb[2] + bz + l * g.wpl;
                    const uint64_t w = occ_brick_word(binaries + l * cells, g, bx, by, bz);
                    words[b] = w;
                    if (w) coarse[b >> 4] |= (w == ~0ull ? kBrickFull : kBrickMixed) << ((b & 15) << 1);
                }
    OccView occ;
    occ.words = words.data();
    occ.coarse = coarse.data();
    occ.bounds = nullptr;
    occ.g = g;

    std::vector<Run> runs;
    int64_t total = 0;
    for (int32_t r = 0; r < n_rays; ++r) {
        RunSink<VecPool> out;
        run_sink_init(out);
        out.pool.runs = &runs;
        out.pool.ray = (uint32_t)r;
        const float near = near_planes ? near_planes[r] : near_plane;
        const float far = far_planes ? far_planes[r] : far_plane;
        if (t_sorted == nullptr) {
            const SingleBox boxes{aabbs};
            generic_march_ray(boxes, occ, rays_o + 3 * r, rays_d + 3 * r, near, far, step_size, cone_angle, -1, out);
        } else {
            const SortedBoxes boxes{aabbs, n_grids, t_sorted + (int64_t)r * 2 * n_grids,
                                    t_indices + (int64_t)r * 2 * n_grids, hits + (int64_t)r * n_grids};
            generic_march_ray(boxes, occ, rays_o + 3 * r, rays_d + 3 * r, near, far, step_size, cone_angle, -1, out);
        }
        run_sink_close(out);
        packed_info[2 * r] = total;
        packed_info[2 * r + 1] = out.n_samples;
        run_counts[r] = out.n_runs;
        total += out.n_samples;
    }
    for (const Run& q : runs)
        cone_expand_run(q.t_first, q.n, cone_angle, step_size, q.ray, packed_info[2 * q.ray] + q.sample_off, capacity,
                        ray_indices, t_starts, t_ends);
    return total;
}

}  // extern "C"
