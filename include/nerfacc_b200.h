/*
 * nerfacc_b200.h -- C ABI of libnerfacc_b200.so (hand-written sm_90a CUDA).
 *
 * This is the drop-in boundary for nerfacc's sampling + compositing hot path.
 * Each entry point replaces one function of the reference's pybind11 module
 * `nerfacc.csrc` / `nerfacc_cuda` (/root/reference/nerfacc/cuda/csrc/nerfacc.cpp:126-163)
 * or one ATen composition in the reference's Python layer; the replaced
 * interface is cited above every declaration (paths relative to /root/reference).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the parameter says "host-visible";
 *   - the library never allocates, frees or synchronises: the caller (PyTorch)
 *     owns all inputs, outputs and workspaces and passes the stream to launch on;
 *   - return value: 0 ok, < 0 argument error (NFA_ERR_*), > 0 a cudaError_t from
 *     the launch.  Nothing is thrown or printed across the ABI;
 *   - all index outputs are int64 (the reference's public dtype), floats are IEEE binary32.
 */
#ifndef NERFACC_B200_H_
#define NERFACC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NFA_OK 0
#define NFA_ERR_ARG (-1)         /* null pointer / negative size / inconsistent sizes */
#define NFA_ERR_UNSUPPORTED (-2) /* valid request outside what this build implements */

#define NFA_ABI_VERSION 15

typedef void* nfa_stream_t; /* cudaStream_t */

int32_t nfa_version(void);
const char* nfa_error_string(int32_t code);

/* ----------------------------------------------------------------------- */
/* Ray / box intersection                                                   */
/* ----------------------------------------------------------------------- */

/* replaces: ray_aabb_intersect(rays_o, rays_d, aabbs, near, far, miss)
 *   nerfacc/cuda/csrc/nerfacc.cpp:68-74, grid.cu:477-519 (kernel :284-313).
 * t_mins, t_maxs: [n_rays, n_aabbs] f32; hits: [n_rays, n_aabbs] bool bytes. */
int32_t nfa_ray_aabb_intersect(int32_t n_rays, const float* rays_o, const float* rays_d,
                               int32_t n_aabbs, const float* aabbs,
                               float near_plane, float far_plane, float miss_value,
                               float* t_mins, float* t_maxs, uint8_t* hits, nfa_stream_t stream);

/* replaces: the ray_aabb_intersect + torch.cat + torch.sort sequence of
 *   nerfacc/grid.py:156-162 in one pass.  t_sorted: [n_rays, 2*n_aabbs] f32
 *   ascending, t_indices: [n_rays, 2*n_aabbs] i64 (position in cat([t_mins, t_maxs])),
 *   hits: [n_rays, n_aabbs].  n_aabbs <= 32. */
int32_t nfa_intersect_sorted(int32_t n_rays, const float* rays_o, const float* rays_d,
                             int32_t n_aabbs, const float* aabbs,
                             float* t_sorted, int64_t* t_indices, uint8_t* hits, nfa_stream_t stream);

/* ----------------------------------------------------------------------- */
/* Occupancy grid: bool bytes -> 4x4x4 brick words                          */
/* ----------------------------------------------------------------------- */

/* Derived cache of OccGridEstimator.binaries (nerfacc/estimators/occ_grid.py:73-76):
 * words  [nfa_occ_words()]        uint64, one per 4x4x4-cell brick,
 * coarse [nfa_occ_coarse_words()] uint32, two bits per brick, 16 bricks per word: bit 0 "some cell set",
 *                                 bit 1 "all 64 cells set" (0 empty, 1 mixed, 3 full); read by
 *                                 nfa_traverse_generic and the growing-step nfa_march,
 * bounds [n_grids * 6]            int32, per level min xyz / max xyz (inclusive, brick units) of the
 *                                 non-empty bricks; min > max when the level is empty. */
int64_t nfa_occ_words(int32_t n_grids, int32_t rx, int32_t ry, int32_t rz);
int64_t nfa_occ_coarse_words(int32_t n_grids, int32_t rx, int32_t ry, int32_t rz);
int32_t nfa_occ_pack(int32_t n_grids, int32_t rx, int32_t ry, int32_t rz, const uint8_t* binaries,
                     uint64_t* words, uint32_t* coarse, int32_t* bounds, nfa_stream_t stream);

/* Grid maintenance (OccGridEstimator._update, nerfacc/estimators/occ_grid.py:367-404).
 * nfa_occ_ema_update: occs[cell_ids[i]] = max(occs[cell_ids[i]] * ema_decay, occ[i]) (:395-398); a cell named more
 *   than once gets the largest of its results in the order -inf < ... < -0.0 < +0.0 < ... < +inf, NaN if any
 *   result is NaN.  scratch: n floats.
 * nfa_occ_threshold_pack: thre = min(mean(occs[occs >= 0]), occ_thre) (:400-402), binaries = occs > thre (:403-404)
 *   written as bool bytes AND as the derived cache nfa_occ_pack would build from them (words / coarse / bounds),
 *   one pass, no host synchronisation.  workspace: nfa_occ_threshold_workspace_bytes(n_cells) bytes, 16-byte
 *   aligned, n_cells = n_grids*rx*ry*rz. */
int32_t nfa_occ_ema_update(int64_t n, const int64_t* cell_ids, const float* occ, float ema_decay, float* occs,
                           float* scratch, nfa_stream_t stream);
int64_t nfa_occ_threshold_workspace_bytes(int64_t n_cells);
int32_t nfa_occ_threshold_pack(int32_t n_grids, int32_t rx, int32_t ry, int32_t rz, const float* occs, float occ_thre,
                               uint8_t* binaries, uint64_t* words, uint32_t* coarse, int32_t* bounds, void* workspace,
                               nfa_stream_t stream);

/* packed_info = [exclusive cumsum(counts), counts] for int64 per-ray counts (the chunk_starts / chunk_cnts pair of
 * data_spec.hpp:86-96 after a one-pass traversal).  workspace: nfa_pack_info_workspace_bytes(n_rays) bytes. */
int32_t nfa_counts_to_packed_info(int32_t n_rays, const int64_t* counts, int64_t* packed_info, void* workspace,
                                  nfa_stream_t stream);

/* Measurement aid (scripts/march_trace.py), not used by the product path: per-warp time stamps of the following
 * constant-step (cone_angle == 0) nfa_march launches are written to `buffer` (8 x uint64 per warp, n_tiles x 16
 * warps); null switches it off.  Growing-step launches write none. */
void nfa_debug_set_march_trace(void* buffer);

/* ----------------------------------------------------------------------- */
/* Grid traversal by runs (step_size > 0)                                   */
/* ----------------------------------------------------------------------- */

/* replaces: traverse_grids(...) nerfacc/cuda/csrc/nerfacc.cpp:75-96, grid.cu:320-474
 *   (kernel :68-282) for the two-pass (exact allocation) mode; with the expand calls below, also the
 *   `vals[is_left]`, `vals[is_right]` of nerfacc/estimators/occ_grid.py:174-177.
 *
 * nfa_march: one pass per ray.  Appends every run (t_first, n) of consecutive
 *   samples to a pool inside `workspace` (capacity `run_capacity` runs) and writes per-ray
 *   sample / run counts there; the totals
 *     totals[0] = n_samples, [1] = n_runs, [2] = run_capacity used, [3] = rays whose
 *     marching variable stopped advancing (the reference would not terminate)
 *   go to `totals` (4 x int64, device memory) and, if given, to `totals_host` (host-visible
 *   pinned memory written by the kernel itself, so no separate copy has to be queued).
 *   near_planes / far_planes: per-ray [n_rays], or both NULL to use the scalars near_plane /
 *   far_plane for every ray (reference occ_grid.py:154-155 builds those tensors with full_like).  If totals[1] > run_capacity the pool
 *   overflowed: call again with a larger pool (counts and totals are still exact).
 *   t_sorted / t_indices / hits may be NULL when n_grids == 1 (crossings are then
 *   computed in the kernel).  `words`, `coarse` and `bounds` come from nfa_occ_pack.
 *   workspace: nfa_march_workspace_bytes(n_rays, run_capacity) bytes whose first 64
 *   bytes are zero on first use (the kernels leave it reusable).
 *   cone_angle (>= 0) selects the walk:
 *   == 0  constant step, one DDA pass.  `coarse` is not read; `bounds` (nullable) lets single-level calls
 *         without terminate planes jump over / stop after empty space; terminate_planes [n_rays] may be NULL.
 *   >  0  growing step (unbounded scenes), dt = clamp(t * cone_angle, step_size, 1e10), sample by sample in the
 *         reference's order of operations.  `coarse` is required, `bounds` is not read, terminate_planes must be
 *         NULL.  A ray whose marching variable stops advancing (t + dt == t) ends there without an error, as in
 *         nfa_traverse_generic: totals[3] is always 0. */
int64_t nfa_march_workspace_bytes(int32_t n_rays, int64_t run_capacity);
int32_t nfa_march(int32_t n_rays, const float* rays_o, const float* rays_d,
                  const float* near_planes, const float* far_planes, float near_plane, float far_plane,
                  int32_t n_grids, int32_t rx, int32_t ry, int32_t rz,
                  const uint64_t* words, const uint32_t* coarse, const int32_t* bounds, const float* aabbs,
                  const float* t_sorted, const int64_t* t_indices, const uint8_t* hits,
                  float step_size, float cone_angle, int64_t run_capacity, void* workspace, int64_t* totals,
                  int64_t* totals_host, float* terminate_planes, nfa_stream_t stream);

/* nfa_expand_samples: runs -> packed (ray_indices, t_starts, t_ends) + packed_info.
 *   replaces the fill pass plus `vals[is_left]`, `vals[is_right]` of
 *   nerfacc/estimators/occ_grid.py:174-177.  `totals` is the device array nfa_march
 *   filled; step_size and cone_angle must be the march's.  Elements at index >= capacity are not written (the
 *   caller re-runs with a larger buffer).  packed_info: [n_rays, 2] = (chunk_start, chunk_cnt), 16-byte aligned,
 *   always written by this call (in the one kernel it launches, also when capacity or run_capacity is 0).
 *   cone_angle == 0: every run computed from the lattice closed form.  cone_angle > 0: every run replayed as
 *   t_{j+1} = t_j + dt(t_j) from its t_first (the same float operations as the march, so the same bits). */
int32_t nfa_expand_samples(int32_t n_rays, int64_t run_capacity, const void* workspace,
                           const int64_t* totals, float step_size, float cone_angle, int64_t capacity,
                           int64_t* packed_info, int64_t* ray_indices, float* t_starts, float* t_ends,
                           nfa_stream_t stream);

/* nfa_expand_intervals: runs of a constant-step nfa_march -> the RaySegmentsSpec pair traverse_grids returns
 *   (nerfacc/cuda/csrc/include/data_spec.hpp:6-16, nerfacc/data_specs.py:12-180):
 *   intervals {vals, ray_indices, is_left, is_right, packed_info} with n_samples + n_runs
 *   edges, samples {vals = midpoints, ray_indices, is_valid, packed_info}. */
int32_t nfa_expand_intervals(int32_t n_rays, int64_t run_capacity, const void* workspace,
                             const int64_t* totals, float step_size,
                             int64_t edge_capacity, int64_t sample_capacity,
                             int64_t* iv_packed_info, float* iv_vals, int64_t* iv_ray_indices,
                             uint8_t* iv_is_left, uint8_t* iv_is_right,
                             int64_t* sm_packed_info, float* sm_vals, int64_t* sm_ray_indices,
                             uint8_t* sm_is_valid, nfa_stream_t stream);

/* nfa_traverse_generic: the remaining modes of traverse_grids (nerfacc.cpp:75-96, grid.cu:320-474) --
 *   cone_angle > 0, step_size <= 0 (one sample per occupied cell), traverse_steps_limit, over_allocate
 *   and rays_mask -- marched sample by sample, one thread per ray, in the reference's order.
 *   fill == 0: count pass, writes iv_cnts / sm_cnts [n_rays] (edges / samples per ray).
 *   fill != 0: writes the arrays at iv_starts / sm_starts (exclusive scans of the counts, or the
 *   fixed strides of over_allocate), skipping rays whose count is 0, then stores the actual counts.
 *   Flag / value arrays must be zero-filled by the caller, as data_spec.hpp:62-84 does.
 *   rays_mask (bool bytes) may be NULL; the crossings t_sorted / t_indices / hits are required. */
/* `slots` (nullable; needs fill != 0 and traverse_steps_limit > 0): over-allocation in one pass (grid.cu:364-404).
 * slots[r] = number of unmasked rays before ray r; ray r writes its edges at slots[r] * 2 * limit and its samples at
 * slots[r] * limit, `iv_starts` / `sm_starts` are not read, and iv_cnts / sm_cnts receive the counts of every ray
 * (0 for masked rays). */
int32_t nfa_traverse_generic(int32_t n_rays, const float* rays_o, const float* rays_d, const uint8_t* rays_mask,
                             const float* near_planes, const float* far_planes,
                             int32_t n_grids, int32_t rx, int32_t ry, int32_t rz,
                             const uint64_t* words, const uint32_t* coarse, const float* aabbs,
                             const float* t_sorted, const int64_t* t_indices, const uint8_t* hits,
                             float step_size, float cone_angle, int32_t traverse_steps_limit, int32_t fill,
                             const int64_t* slots,
                             const int64_t* iv_starts, int64_t* iv_cnts, float* iv_vals, int64_t* iv_ray_indices,
                             uint8_t* iv_is_left, uint8_t* iv_is_right,
                             const int64_t* sm_starts, int64_t* sm_cnts, float* sm_vals, int64_t* sm_ray_indices,
                             uint8_t* sm_is_valid, float* terminate_planes, nfa_stream_t stream);

/* ----------------------------------------------------------------------- */
/* Volume rendering over the packed layout                                  */
/* ----------------------------------------------------------------------- */

/* replaces: the ATen composition of nerfacc/volrend.py:79-164 --
 *   render_weight_from_density (:326-376 -> :219-278 -> exclusive_sum, scan.py:80-145,
 *   native exclusive_sum / exclusive_sum_cub, nerfacc.cpp:15-21,49-53) or
 *   render_weight_from_alpha (:281-323 -> exclusive_prod*, nerfacc.cpp:30-39,62-65),
 *   followed by accumulate_along_rays x3 (:145-156,497-561), expected-depth
 *   normalisation (:157-158) and background blend (:161-162).
 * from_alpha == 0: `sigmas_or_alphas` holds sigmas and t_starts/t_ends are required;
 * from_alpha != 0: it holds alphas (t_starts/t_ends only needed for depths).
 * n_samples = length N of the per-sample arrays (segments in packed_info index into them).
 * Nullable: rgbs, prefix_trans, bkgd[3], every output.  Per-sample outputs [N]
 * (weights, trans, alphas), per-ray outputs colors [R,3], opacities [R], depths [R];
 * raw [R,5] keeps the un-normalised (colour, opacity, depth) sums for the backward. */
int32_t nfa_composite_fwd(int32_t n_rays, int64_t n_samples, const int64_t* packed_info,
                          const float* t_starts, const float* t_ends,
                          const float* sigmas_or_alphas, int32_t from_alpha,
                          const float* rgbs, const float* prefix_trans, const float* bkgd,
                          int32_t expected_depths,
                          float* weights, float* trans, float* alphas,
                          float* colors, float* opacities, float* depths, float* raw,
                          nfa_stream_t stream);

/* replaces: the autograd graph of the above -- index_add_ backward (gather), mul
 *   backward, _ExclusiveSumCUB.backward / _ExclusiveSum.backward (nerfacc/scan.py:307-337,
 *   403-424; native exclusive_sum[_cub](..., backward=true)), the product-scan backwards
 *   (nerfacc.cpp:26-39,57-65; scan.cu:167-304), exp/mul backward.
 * Upstream gradients (all nullable): g_colors [R,3], g_opacities [R], g_depths [R] on the
 * values nfa_composite_fwd returned (needs `raw`), g_weights / g_trans / g_alphas [N] on
 * the per-sample outputs.  Outputs: g_in [N] (d/dsigma or d/dalpha), g_rgbs [N,3] (nullable). */
int32_t nfa_composite_bwd(int32_t n_rays, int64_t n_samples, const int64_t* packed_info,
                          const float* t_starts, const float* t_ends,
                          const float* sigmas_or_alphas, int32_t from_alpha,
                          const float* rgbs, const float* prefix_trans, const float* bkgd,
                          int32_t expected_depths, const float* raw,
                          const float* g_colors, const float* g_opacities, const float* g_depths,
                          const float* g_weights, const float* g_trans, const float* g_alphas,
                          float* g_in, float* g_rgbs, nfa_stream_t stream);

/* replaces: accumulate_along_rays (nerfacc/volrend.py:497-561): out[r, :] = sum_i w_i v_i.
 *   _fwd: segmented (grouped samples, packed_info), deterministic, out fully written.
 *   _atomic: any ray_indices order, float atomics into a zero-filled (or, for the
 *            in-place variant volrend.py:564-587, pre-filled) `out`.
 *   _bwd: g_weights [N] and g_values [N,dim] (nullable) from g_out [R,dim].
 * values == NULL means accumulate the weights themselves (dim must be 1). */
int32_t nfa_accumulate_fwd(int32_t n_rays, const int64_t* packed_info, const float* weights,
                           const float* values, int32_t dim, float* out, nfa_stream_t stream);
int32_t nfa_accumulate_atomic(int64_t n, const int64_t* ray_indices, const float* weights,
                              const float* values, int32_t dim, float* out, nfa_stream_t stream);
int32_t nfa_accumulate_bwd(int64_t n, const int64_t* ray_indices, const float* weights,
                           const float* values, int32_t dim, const float* g_out,
                           float* g_weights, float* g_values, nfa_stream_t stream);

/* ----------------------------------------------------------------------- */
/* Segmented scans and pack_info                                            */
/* ----------------------------------------------------------------------- */

/* replaces: inclusive_sum / exclusive_sum (chunk_starts, chunk_cnts, inputs, normalize, backward)
 *   and {in,ex}clusive_prod_forward  -- nerfacc/cuda/csrc/nerfacc.cpp:8-39, scan.cu:9-304.
 *   reverse != 0 scans every chunk from its last element (what `backward=true` does).
 *   The product backwards are composed in Python from a reverse sum scan, as scan.cu:199-210 does. */
int32_t nfa_scan_packed(int32_t n_rays, const int64_t* packed_info, const float* in, float* out,
                        int32_t op_prod, int32_t inclusive, int32_t reverse, int32_t normalize,
                        nfa_stream_t stream);

/* replaces: {in,ex}clusive_sum_cub(indices, inputs, backward), {in,ex}clusive_prod_cub_forward
 *   -- nerfacc.cpp:41-65, scan_cub.cu:59-287 (cub::DeviceScan::*ByKey).  A segment is a
 *   maximal run of equal consecutive keys.  workspace: nfa_scan_by_key_workspace_bytes(n). */
int64_t nfa_scan_by_key_workspace_bytes(int64_t n);
int32_t nfa_scan_by_key(int64_t n, const int64_t* keys, const float* in, float* out,
                        int32_t op_prod, int32_t inclusive, int32_t reverse, void* workspace,
                        nfa_stream_t stream);

/* replaces: pack_info (nerfacc/pack.py:38-46: zeros + index_add_ + cumsum + stack).
 *   packed_info [n_rays, 2] = (chunk_start, chunk_cnt).  workspace:
 *   nfa_pack_info_workspace_bytes(n_rays).  Indices outside [0, n_rays) are ignored. */
int64_t nfa_pack_info_workspace_bytes(int32_t n_rays);
int32_t nfa_pack_info(int64_t n, const int64_t* ray_indices, int32_t n_rays, int64_t* packed_info,
                      void* workspace, nfa_stream_t stream);

/* ----------------------------------------------------------------------- */
/* Packed <-> padded per-ray layout (nerfacc 0.3's unpack_info / unpack_data / pack_data, removed in 0.5.0,     */
/* CHANGELOG.md:38; in 0.5 code the `data[mask]` / index-arithmetic ATen compositions written in their place)   */
/* ----------------------------------------------------------------------- */

/* Byte movers: a row is `row_bytes` bytes (element size x elements per sample), copied in the largest of
 * 16 / 8 / 4 / 2 / 1-byte units that divides row_bytes and every data pointer, so any dtype is bit-exact.
 * packed rows [n_packed]; padded rows [n_rays, n_per_ray]; packed_info [n_rays, 2] = (start, count), counts < 0
 * read as 0.  Packed positions outside [0, n_packed) are neither read nor written.
 * "In order" below means start_r >= start_{r-1} + count_{r-1} for every r (every packed_info this library returns);
 * the library checks it on the device.  workspace: nfa_chunk_order_workspace_bytes() bytes, no initial value. */
int64_t nfa_chunk_order_workspace_bytes(void);

/* replaces: unpack_info(packed_info, n_samples) (0.3) / torch.repeat_interleave(arange(n_rays), counts).
 *   ray_indices [n_samples] int64: r on chunk r, -1 where no chunk lands.  Chunks in order: one store pass
 *   (each ray also writes the gap behind its chunk); otherwise a -1 fill pass first.  Chunks must not overlap. */
int32_t nfa_unpack_info(int32_t n_rays, const int64_t* packed_info, int64_t n_samples, int64_t* ray_indices,
                        void* workspace, nfa_stream_t stream);

/* replaces: unpack_data(packed_info, data, n_samples, pad_value) (0.3) / torch.full + masked index assignment.
 *   padded[r, j] = packed[start_r + j] for j < min(count_r, n_per_ray) (and inside [0, n_packed)), else the
 *   row at `pad_row` (device memory, row_bytes bytes).  Every padded row is written by the one kernel.
 *   packed may be NULL when n_packed == 0. */
int32_t nfa_unpack_rows(int32_t n_rays, const int64_t* packed_info, int64_t n_packed, int64_t n_per_ray,
                        int64_t row_bytes, const void* packed, const void* pad_row, void* padded, nfa_stream_t stream);

/* replaces: the backward of the above (a scatter of the padded gradient into zeros).
 *   packed[start_r + j] = padded[r, j] for j < min(count_r, n_per_ray); every other packed row (truncated, or in
 *   no chunk) is zero.  Chunks in order: one pass; otherwise a zero fill pass first. */
int32_t nfa_pack_rows(int32_t n_rays, const int64_t* packed_info, int64_t n_packed, int64_t n_per_ray,
                      int64_t row_bytes, const void* padded, void* packed, void* workspace, nfa_stream_t stream);

/* replaces: mask.sum(-1) of pack_data (0.3).  counts [n_rays] int64 = number of nonzero bytes in each row of
 *   mask [n_rays, n_per_ray] (bool bytes); nfa_counts_to_packed_info turns them into packed_info. */
int32_t nfa_mask_counts(int32_t n_rays, int64_t n_per_ray, const uint8_t* mask, int64_t* counts, nfa_stream_t stream);

/* replaces: data[mask] of pack_data (0.3) and its backward (a masked scatter into zeros).
 *   Row j of ray r is kept iff mask[r, j]; the kept rows of ray r are packed rows start_r, start_r + 1, ... in j
 *   order (packed_info from nfa_counts_to_packed_info of nfa_mask_counts).
 *   nfa_pack_masked:   padded -> packed (only kept rows written).
 *   nfa_unpack_masked: packed -> padded, every padded row written (zero where the mask is false); packed may be
 *                      NULL when no mask byte is set. */
int32_t nfa_pack_masked(int32_t n_rays, int64_t n_per_ray, int64_t row_bytes, const uint8_t* mask,
                        const int64_t* packed_info, const void* padded, void* packed, nfa_stream_t stream);
int32_t nfa_unpack_masked(int32_t n_rays, int64_t n_per_ray, int64_t row_bytes, const uint8_t* mask,
                          const int64_t* packed_info, const void* packed, void* padded, nfa_stream_t stream);

/* replaces: the visibility branch of OccGridEstimator.sampling (nerfacc/estimators/occ_grid.py:180-220):
 *   render_visibility_from_density / _from_alpha (volrend.py:379-494; native exclusive_sum / exclusive_prod on
 *   packed_info) followed by three boolean mask-selects.  Keeps sample i iff T_i >= early_stop_eps and
 *   (alpha_thre <= 0 or alpha_i >= alpha_thre); writes the kept (ray_indices, t_starts, t_ends) compacted in
 *   ray order, their packed_info, and the kept total (device and/or pinned host memory).  The outputs need room
 *   for n_samples elements (the caller narrows after one sync).  workspace: nfa_visibility_workspace_bytes(). */
int64_t nfa_visibility_workspace_bytes(int32_t n_rays, int64_t n_samples);
int32_t nfa_visibility_compact(int32_t n_rays, int64_t n_samples, const int64_t* packed_info,
                               const float* t_starts, const float* t_ends, const float* sigmas_or_alphas,
                               int32_t from_alpha, float early_stop_eps, float alpha_thre, void* workspace,
                               int64_t* new_packed_info, int64_t* out_ray_indices, float* out_t_starts,
                               float* out_t_ends, int64_t* total_dev, int64_t* total_host, nfa_stream_t stream);

/* The same filter in rounds (OccGridEstimator.sampling_until_opaque): the field runs on each live ray's next k
 *   samples only (k a multiple of 32), and a ray stops being live once its next sample's transmittance fails
 *   T >= early_stop_eps.  Every T, alpha and keep bit is nfa_visibility_compact's when densities are >= 0 (alphas in
 *   [0, 1]).  The workspace (nfa_vis_rounds_workspace_bytes; 16-byte aligned, no state carried between calls) holds the live-ray lists, the per-ray carries and counts and the mask; it is owned by one stream.
 *   status_host (pinned, [4]) = {n_alive, k, samples of the round, kept samples so far}, written for the next round
 *   by begin and every step; n_alive == 0 ends the loop.  n_alive / round / n_with_samples come from it.
 *   begin   every ray with samples live (in ray order, round 0, k = 32), mask zeroed.  n_with_samples = its n_alive.
 *   gather  the round's closure inputs, in ray order: each live ray's next min(k, left) samples.
 *   step    the closure's float32 outputs for those samples: mask bytes, kept counts and carries; the next round's
 *           live list, k = 32 clamp(n_with_samples / n_alive, 1, 8) and sample count.
 *   finish  the kept (ray_indices, t_starts, t_ends) compacted in ray order and their packed_info. */
int64_t nfa_vis_rounds_workspace_bytes(int32_t n_rays, int64_t n_samples);
int32_t nfa_vis_rounds_begin(int32_t n_rays, int64_t n_samples, const int64_t* packed_info, int32_t from_alpha,
                             void* workspace, int64_t* status_host, nfa_stream_t stream);
int32_t nfa_vis_rounds_gather(int32_t n_rays, int64_t n_samples, int32_t round, int32_t n_alive,
                              const int64_t* packed_info, const float* t_starts, const float* t_ends,
                              const void* workspace, int64_t* out_ray_indices, float* out_t_starts, float* out_t_ends,
                              nfa_stream_t stream);
int32_t nfa_vis_rounds_step(int32_t n_rays, int64_t n_samples, int32_t round, int32_t n_alive,
                            int32_t n_with_samples, const int64_t* packed_info, const float* t_starts,
                            const float* t_ends, const float* sigmas_or_alphas, int32_t from_alpha,
                            float early_stop_eps, float alpha_thre, void* workspace, int64_t* status_host,
                            nfa_stream_t stream);
int32_t nfa_vis_rounds_finish(int32_t n_rays, int64_t n_samples, const int64_t* packed_info, const float* t_starts,
                              const float* t_ends, const void* workspace, int64_t* new_packed_info,
                              int64_t* out_ray_indices, float* out_t_starts, float* out_t_ends, nfa_stream_t stream);

/* ----------------------------------------------------------------------- */
/* Early-terminated test-time rendering (OccGridEstimator.render_test)      */
/* ----------------------------------------------------------------------- */

/* replaces: the test-mode rendering loop of nerfacc's examples (examples/utils.py:267-439): per round
 *   traverse_grids(traverse_steps_limit, over_allocate, rays_mask, t_sorted, t_indices, hits), three boolean
 *   mask-selects, render_weight_from_density(prefix_trans = 1 - opacity), the optional alpha_thre compaction, three
 *   accumulate_along_rays_ and the new ray mask; then the background blend and depth normalisation.
 * The workspace (nfa_render_test_workspace_bytes; 16-byte aligned, zeroed once when allocated, left reusable by every
 *   call) holds the live-ray lists, every ray's near plane, the round's fixed-stride samples and the scans; it is
 *   owned by one stream.  min_samples: 1 (cone_angle == 0) or 4.  Per call:
 *   begin      every ray live, near planes = near_plane, kept-sample count 0.
 *   march      round `round` (0, 1, ...): n_alive from the device (R, or what the previous composite left),
 *              n_samples = max(min(R / n_alive, 64), min_samples), every live ray marched with that step limit
 *              (t_sorted / t_indices / hits: nfa_intersect_sorted), its terminate plane kept as its next near plane;
 *              status_host (pinned, [4]) = {n_alive, n_samples, samples of the round, kept samples of the earlier
 *              rounds}, written when the kernel ends.  n_alive == 0: nothing was marched, the loop is over.
 *              step_size <= 0 is NFA_ERR_UNSUPPORTED.
 *   expand     the round's samples in ray order (the field's inputs); n_alive / n_samples from status_host.
 *   composite  the field's float32 rgbs [n_total, 3] and sigmas [n_total] onto the running colors [R, 3], opacities
 *              [R] and depths [R] (zero before round 0): weights from all the round's samples, alpha_thre > 0 drops
 *              samples with alpha < alpha_thre from the sums only; a ray stays live while opacity <= opacity_thre
 *              (1 - early_stop_eps) and it got n_samples samples.  Deterministic: no atomics on the outputs.
 *   finish     colors += bkgd (1 - opacity) when bkgd [3] is given, depths /= max(opacity, FLT_EPSILON); with
 *              status_host, status_host[3] = kept samples of all rounds. */
int64_t nfa_render_test_workspace_bytes(int32_t n_rays, int32_t min_samples);
int32_t nfa_render_test_begin(int32_t n_rays, int32_t min_samples, float near_plane, void* workspace,
                              nfa_stream_t stream);
int32_t nfa_render_test_march(int32_t n_rays, int32_t min_samples, int32_t round, const float* rays_o,
                              const float* rays_d, float far_plane, int32_t n_grids, int32_t rx, int32_t ry, int32_t rz,
                              const uint64_t* words, const uint32_t* coarse, const float* aabbs, const float* t_sorted,
                              const int64_t* t_indices, const uint8_t* hits, float step_size, float cone_angle,
                              void* workspace, int64_t* status_host, nfa_stream_t stream);
int32_t nfa_render_test_expand(int32_t n_rays, int32_t min_samples, int32_t round, int32_t n_alive, int32_t n_samples,
                               const void* workspace, int64_t* ray_indices, float* t_starts, float* t_ends,
                               nfa_stream_t stream);
int32_t nfa_render_test_composite(int32_t n_rays, int32_t min_samples, int32_t round, int32_t n_alive,
                                  int32_t n_samples, int64_t n_total, void* workspace, const float* t_starts,
                                  const float* t_ends, const float* rgbs, const float* sigmas, float alpha_thre,
                                  float opacity_thre, float* colors, float* opacities, float* depths,
                                  nfa_stream_t stream);
int32_t nfa_render_test_finish(int32_t n_rays, int32_t min_samples, const void* workspace, const float* bkgd,
                               float* colors, const float* opacities, float* depths, int64_t* status_host,
                               nfa_stream_t stream);

/* ----------------------------------------------------------------------- */
/* PDF: importance sampling and per-ray searchsorted                        */
/* ----------------------------------------------------------------------- */

/* replaces: importance_sampling(RaySegmentsSpec, cdfs, n_intervals_per_ray [int | Tensor], stratified)
 *   -- nerfacc.cpp:97-112, pdf.cu:293-426 (kernels :97-243).  Resamples every ray's piecewise-linear CDF
 *   (edges `vals`, values `cdfs`) to n sample centres and the n+1 edges between them, in one launch.
 *   input:  batched (in_packed_info NULL, in_edges per ray) or flattened (in_packed_info [n_rays,2] =
 *           (start, count); max_in_edges >= every count, used to size shared memory);
 *   output: batched (out_packed_info NULL): sample_vals [n_rays, n_out], iv_vals [n_rays, n_out+1];
 *           flattened: out_packed_info / iv_packed_info [n_rays,2] give every ray's slice of the samples
 *           and of the edges (count+1 edges for count > 0, else 0), max_out >= every sample count;
 *           sample_ray_indices (optional), iv_ray_indices, iv_left, iv_right are then filled too.
 *   stratified: one jitter per ray = first cuRAND Philox4x32-10 uniform of (seed, subsequence = ray,
 *           offset) -- pdf.cu:139-145 with the (seed, offset) pair of torch's CUDA generator.
 *   t_starts / t_ends (optional, batched output): the edges mapped s -> t as PropNetEstimator does
 *           (estimators/prop_net.py:215-229): t = s*s_max + (1-s)*s_min, or its reciprocal when `lindisp`
 *           (then s_min = 1/near, s_max = 1/far). */
int32_t nfa_importance_sampling(int32_t n_rays, const float* vals, const float* cdfs, const int64_t* in_packed_info,
                                int64_t in_edges, int64_t max_in_edges, const int64_t* out_packed_info,
                                const int64_t* iv_packed_info, int64_t n_out, int64_t max_out, int32_t stratified,
                                uint64_t seed, uint64_t offset, float* sample_vals, int64_t* sample_ray_indices,
                                float* iv_vals, int64_t* iv_ray_indices, uint8_t* iv_left, uint8_t* iv_right,
                                float* t_starts, float* t_ends, float s_min, float s_max, int32_t lindisp,
                                nfa_stream_t stream);

/* replaces: searchsorted(query RaySegmentsSpec, key RaySegmentsSpec) -> (ids_left, ids_right)
 *   -- nerfacc.cpp:113-116, pdf.cu:429-456 (kernel :247-287).  For every query value the pair of key edges of
 *   the same ray with key[left] <= q < key[right], clipped to the ray's edge range.  Batched operands pass a
 *   NULL packed_info and their per-ray edge count; a batched query gets positions relative to its ray's keys,
 *   a flattened one absolute positions.  query_ray_indices is optional (else found from query_packed_info). */
int32_t nfa_searchsorted(int64_t n_query, const float* query_vals, const int64_t* query_packed_info,
                         const int64_t* query_ray_indices, int32_t n_rays, int64_t query_edges,
                         const float* key_vals, const int64_t* key_packed_info, int64_t key_edges,
                         int64_t* ids_left, int64_t* ids_right, nfa_stream_t stream);

/* replaces: the ATen composition of the proposal loss, estimators/prop_net.py:232-256 `_pdf_loss` (searchsorted, a
 *   diff, two gathers, clip, ** 2, a division); the reference has no kernel for it.  Batched rows only: query edges /
 *   cdfs [n_rays, q_edges], key edges / cdfs [n_rays, k_edges].  Interval j of a ray spans query edges j and j+1;
 *   L_j = searchsorted's left id of query edge j, R_j its right id of query edge j+1 (nfa_searchsorted's search and
 *   clipping), and loss [n_rays, q_edges-1] = clip(w - wo, min=0)^2 / (w + eps) with w = cq[j+1] - cq[j],
 *   wo = ck[R_j] - ck[L_j], every op rounded as ATen rounds it, so the values are ATen's bit for bit.
 *   eps: the Python scalar rounded to float.  q_edges >= 1 and k_edges >= 1; q_edges == 1 writes nothing. */
int32_t nfa_pdf_loss_fwd(int64_t n_rays, int64_t q_edges, const float* q_vals, const float* q_cdfs, int64_t k_edges,
                         const float* k_vals, const float* k_cdfs, float eps, float* loss, nfa_stream_t stream);

/* replaces: the autograd graph of the above for the key cdfs (estimators/prop_net.py:232-256; ATen: the chain's
 *   backwards and two gather backwards, each zeros + a float-atomic scatter_add_).  grad_loss [n_rays, q_edges-1]
 *   (may be NULL when q_edges == 1) -> grad_k_cdfs [n_rays, k_edges], every element written (zeros included).  The
 *   per-interval term is ATen's: where(d >= 0, -((g / (w + eps)) * (2 * c)), 0), d = w - wo, c = clip(d, min=0); key
 *   edge k gets the sum over R_j == k in ascending j, plus the sum over L_j == k (of the negated terms) in ascending j.
 *   No atomics: the result does not change from run to run.  q_edges - 1 > NFA_PDF_LOSS_MAX_INTERVALS is
 *   NFA_ERR_UNSUPPORTED (a ray's ids and terms are staged in shared memory). */
#define NFA_PDF_LOSS_MAX_INTERVALS 16384
int32_t nfa_pdf_loss_bwd(int64_t n_rays, int64_t q_edges, const float* q_vals, const float* q_cdfs, int64_t k_edges,
                         const float* k_vals, const float* k_cdfs, float eps, const float* grad_loss,
                         float* grad_k_cdfs, nfa_stream_t stream);

/* ----------------------------------------------------------------------- */
/* Data-parallel exchange: sum of per-rank scalars over NVLink peer memory  */
/* ----------------------------------------------------------------------- */

/* No counterpart in the reference (it is single-GPU; SURVEY.md section 8(e) gives the ray-sharded path exactly one
 * exchange, the all-reduce of the scalar training loss).  Every rank owns a mailbox of `turns` x `world` 8-byte words
 * in its own device memory.  The four calls below are the only ones in this library that allocate / map memory:
 * CUDA IPC can export plain cudaMalloc allocations only, not memory of the caller's pool.
 *   create:  allocate + zero the mailbox, return it and its 64-byte CUDA IPC handle (exchanged by the host side);
 *   open:    map a peer's mailbox from its handle (same node; peer access is enabled lazily);  close / destroy. */
int32_t nfa_mailbox_create(int32_t world, int32_t turns, void** box, unsigned char* handle64);
int32_t nfa_mailbox_open(const unsigned char* handle64, void** peer_box);
int32_t nfa_mailbox_close(void* peer_box);
int32_t nfa_mailbox_destroy(void* box);

/* post: store (value, tag) as one 8-byte word into slot [turn][rank] of every mailbox listed in `boxes` (device
 *   array of `world` mailbox pointers, entry `rank` being the caller's own) -- st.global over NVLink, no handshake.
 * sum:  out[0] = scale * sum of the `world` values of `turn` in the caller's own mailbox, in rank order, once all
 *   carry `tag`; waits for stragglers with a bounded spin (then out = NaN and *status = 1).  `tag` must change from
 *   one use of a turn to the next (the step number does). */
int32_t nfa_mailbox_post(const float* value, const void* boxes, int32_t world, int32_t rank, int32_t turn, uint32_t tag,
                         nfa_stream_t stream);
int32_t nfa_mailbox_sum(const void* box, int32_t world, int32_t turn, uint32_t tag, float scale, float* out,
                        int32_t* status, nfa_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* NERFACC_B200_H_ */
