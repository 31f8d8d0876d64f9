// CPU build of the round march of render_test.cu: the walk of march_generic.cuh into a SampleSink, the live rays
// (rays_mask) in ray order, ray k of them writing its samples to fixed-stride slots k * limit ...  The device kernel
// runs one thread per live ray; here the rays are serialised.  Compiled by tests/test_render_test_cpu.py with
// -ffp-contract=off.
#include <cstdint>

#include "../../nerfacc_b200/csrc/march_generic.cuh"

using namespace nfa;

extern "C" {

// words / coarse: the packed grid (host_sim's sim_occ_pack).  Writes counts [n_live], terminate [n_rays] (live rays
// only) and slot_ts / slot_te [n_live * limit]; returns the number of live rays.
int32_t sim_sample_sink_round(int32_t n_rays, const float* rays_o, const float* rays_d, const uint8_t* rays_mask,
                              const float* near_planes, float far_plane, int n_grids, int rx, int ry, int rz,
                              const uint64_t* words, const uint32_t* coarse, const float* aabbs, const float* t_sorted,
                              const int64_t* t_indices, const uint8_t* hits, float step_size, float cone_angle,
                              int32_t limit, int64_t* counts, float* terminate, float* slot_ts, float* slot_te)
{
    OccView occ;
    occ.words = words;
    occ.coarse = coarse;
    occ.bounds = nullptr;
    occ.g = occ_geom(n_grids, rx, ry, rz);
    int32_t k = 0;
    for (int32_t r = 0; r < n_rays; ++r) {
        if (rays_mask && !rays_mask[r]) continue;
        SampleSink out;
        out.t_starts = slot_ts;
        out.t_ends = slot_te;
        out.base = (int64_t)k * limit;
        out.n_samples = 0;
        const SortedBoxes b{aabbs, n_grids, t_sorted + (int64_t)r * 2 * n_grids, t_indices + (int64_t)r * 2 * n_grids,
                            hits + (int64_t)r * n_grids};
        terminate[r] = generic_march_ray(b, occ, rays_o + 3 * r, rays_d + 3 * r, near_planes[r], far_plane, step_size,
                                         cone_angle, limit, out);
        counts[k] = out.n_samples;
        ++k;
    }
    return k;
}

}  // extern "C"
