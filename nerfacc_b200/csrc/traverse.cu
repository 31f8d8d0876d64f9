// traverse.cu -- occupancy-grid traversal kernels for sm_90a and their C ABI.
//
// Pipeline for one OccGridEstimator.sampling() call (reference
// nerfacc/estimators/occ_grid.py:154-177 -> nerfacc/grid.py:93-192 ->
// nerfacc/cuda/csrc/grid.cu:320-474):
//
//   occ_pack_kernel   bool grid -> 4x4x4 brick words + 2-bit/brick class mip (cached per grid version)
//   march_kernel      1 thread / ray, march_tile_rays() rays / CTA.  Ray tile staged
//                     into shared memory with cp.async.bulk (TMA 1-D) + mbarrier; the
//                     tile's rays are ordered by expected walk length so that the lanes
//                     of a warp finish together.  Phase 1: pure DDA walk recording
//                     occupied stretches (divergent but cheap); phase 2: closed-form
//                     lattice seeks, a warp's stretches dealt out to its lanes (march.cuh).  Runs go to a pool
//                     (one atomic per warp and round); per-ray counts, each ray's sample offset inside its tile,
//                     per-tile sums and (last CTA) the tile bases + grand totals are left in the workspace.
//   offsets_kernel    1 CTA / tile: tile base from the tile sums + block scan -> packed_info (ray-ordered
//                     offsets, so ray_indices stay sorted).  Interval form and the scalar fallback only: the
//                     vectorised samples kernel writes packed_info itself from (tile base, offset in tile).
//   expand_runs_vec_kernel / expand_runs_kernel
//                     one warp per run: lanes compute their samples from the lattice
//                     closed form (expand.cuh) and store them coalesced, 128-bit stores
//                     when the outputs are 16-byte aligned; the <true> flavour writes the
//                     interval-edge form traverse_grids() returns.
//   generic_traverse_kernel  every other traverse_grids mode (march_generic.cuh).
//   ray_aabb_kernel / intersect_sorted_kernel  slab tests (+ sorted crossings of nested boxes).
//
// No tensor cores: the path has no dense contraction; it is bound by dependent
// f32 chains (march) and by HBM stores (expand).  See DESIGN.md.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/nerfacc_b200.h"
#include "sm_count.cuh"
#include "expand.cuh"
#include "march.cuh"
#include "march_generic.cuh"
#include "occ_pack.cuh"

namespace nfa {

constexpr int kMaxTileRays = 512;   // rays per CTA in the march / offsets kernels: march_tile_rays(), <= this
constexpr int kDescSlots = 8;       // stretch descriptors buffered per ray between the two march phases ...
constexpr int kDescSlotsWide = 16;  // ... and when one wave holds every ray (shared memory to spare): no second round
constexpr int kSortBuckets = 256;   // counting sort of a tile's rays by expected walk length

// Rays per march CTA (= threads).  All CTAs of a batch this size are resident at once, so the kernel takes as
// long as the SM with the most rays: pick the tile that spreads the rays most evenly over the kNumSMs SMs
// (65 536 rays on 132 SMs: 128 tiles of 512 rays, one per SM, instead of 512 tiles of 128 = 4 on some SMs
// and 3 on others); ties go to the larger tile, whose rays sort into more uniform warps.  Large batches
// (several waves) use 256.
inline int march_tile_rays(int32_t n_rays)
{
    const int kSMs = kNumSMs;
    if (n_rays <= 32) return 32;
    if ((int64_t)n_rays > (int64_t)kSMs * 2048) return 256;
    int best = 128;
    int64_t best_cost = INT64_MAX;
    for (int t = 64; t <= kMaxTileRays; t += 32) {
        const int64_t tiles = (n_rays + t - 1) / t;
        const int64_t per_sm = (tiles + kSMs - 1) / kSMs;
        if (per_sm * t > 2048) continue;  // would not be resident together
        const int64_t cost = per_sm * t;
        if (cost <= best_cost) {
            best_cost = cost;
            best = t;
        }
    }
    return best;
}
constexpr int kExpandThreads = 256;

// One run of consecutive lattice samples, as written by the march kernel (32 bytes, two 16-byte stores).
struct RunRec {
    uint32_t ray;         // ray id (tile-global)
    uint32_t sample_off;  // samples of the ray before this run
    uint32_t n;           // samples in the run
    uint32_t t_first;     // bit pattern of the first sample's start
    uint32_t run_idx;     // runs of the ray before this run (interval edges: +1 edge per run)
    uint32_t tile;        // march tile of the ray (its sample offsets are relative to the tile's base)
    uint32_t pad[2];
};

struct TileSum {
    unsigned long long samples;
    uint32_t runs;
    uint32_t stuck;  // rays whose lattice stopped advancing
};

// Workspace layout (all offsets 16-byte aligned):
//   [0, 64)                 header: u32 done_counter, u32 pool_cursor
//   tile_sums [n_tiles]     TileSum
//   cnt_samples [R] u32, cnt_runs [R] u32
//   loc_samples [R] u32     samples of the earlier rays of the same tile
//   tile_base [n_tiles] u64 samples of the earlier tiles
//   pool [run_capacity]     RunRec
struct Workspace {
    uint32_t* done;
    uint32_t* cursor;
    TileSum* tiles;
    uint32_t* cnt_samples;
    uint32_t* cnt_runs;
    uint32_t* loc_samples;
    unsigned long long* tile_base;
    RunRec* pool;
    int n_tiles;
    int tile_rays;
    int64_t run_capacity;
};

__host__ __device__ inline int64_t align16(int64_t x) { return (x + 15) & ~(int64_t)15; }

inline int64_t ws_bytes(int32_t n_rays, int64_t run_capacity)
{
    const int tile = march_tile_rays(n_rays);
    const int64_t nt = (n_rays + tile - 1) / tile;
    return 64 + align16(nt * (int64_t)sizeof(TileSum)) + align16((int64_t)n_rays * 4) * 3 + align16(nt * 8) +
           run_capacity * (int64_t)sizeof(RunRec);
}

inline Workspace ws_view(void* base, int32_t n_rays, int64_t run_capacity)
{
    Workspace w;
    char* p = (char*)base;
    w.tile_rays = march_tile_rays(n_rays);
    w.n_tiles = (n_rays + w.tile_rays - 1) / w.tile_rays;
    w.run_capacity = run_capacity;
    w.done = (uint32_t*)p;
    w.cursor = (uint32_t*)(p + 4);
    p += 64;
    w.tiles = (TileSum*)p;
    p += align16(w.n_tiles * (int64_t)sizeof(TileSum));
    w.cnt_samples = (uint32_t*)p;
    p += align16((int64_t)n_rays * 4);
    w.cnt_runs = (uint32_t*)p;
    p += align16((int64_t)n_rays * 4);
    w.loc_samples = (uint32_t*)p;
    p += align16((int64_t)n_rays * 4);
    w.tile_base = (unsigned long long*)p;
    p += align16((int64_t)w.n_tiles * 8);
    w.pool = (RunRec*)p;
    return w;
}

// ---------------------------------------------------------------------------
// small PTX wrappers: mbarrier + 1-D bulk async copy (TMA) global -> shared
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    // bounded: a lost completion must fault, not hang the GPU
    for (int spin = 0; spin < (1 << 22); ++spin) {
        uint32_t ok;
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (ok) return;
    }
    __trap();
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---------------------------------------------------------------------------
// occupancy packing
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) occ_pack_kernel(OccGeom g, const uint8_t* __restrict__ binaries,
                                                       uint64_t* __restrict__ words, uint32_t* __restrict__ coarse,
                                                       int32_t* __restrict__ bounds, int64_t n_words, int64_t n_coarse)
{
    const int64_t cells = (int64_t)g.res[0] * g.res[1] * g.res[2];
    // one thread per brick; a half-warp's 16 bricks share one word of the class mip
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < n_coarse * 16;
         b += (int64_t)gridDim.x * blockDim.x) {
        uint64_t w = 0;
        if (b < n_words) {
            const int level = (int)(b / g.wpl);
            int rem = (int)(b - (int64_t)level * g.wpl);
            const int bz = rem % g.nb[2];
            rem /= g.nb[2];
            const int by = rem % g.nb[1];
            const int bx = rem / g.nb[1];
            w = occ_brick_word(binaries + level * cells, g, bx, by, bz);
            words[b] = w;
            if (w != 0) {  // bounding box of the non-empty bricks (few atomics: occupied bricks only)
                int32_t* bb = bounds + 6 * level;
                atomicMin(bb + 0, bx); atomicMin(bb + 1, by); atomicMin(bb + 2, bz);
                atomicMax(bb + 3, bx); atomicMax(bb + 4, by); atomicMax(bb + 5, bz);
            }
        }
        // bit 0: some cell set, bit 1: all 64 set (march.cuh occ_class)
        uint32_t v = (w == 0 ? kBrickEmpty : (w == ~0ull ? kBrickFull : kBrickMixed)) << ((threadIdx.x & 15) << 1);
#pragma unroll
        for (int s = 8; s > 0; s >>= 1) v |= __shfl_xor_sync(0xffffffffu, v, s);
        if ((threadIdx.x & 15) == 0) coarse[b >> 4] = v;
    }
}

__global__ void occ_bounds_init_kernel(int32_t* bounds, int n_grids)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 6 * n_grids) bounds[i] = (i % 6) < 3 ? kBoundsMinInit : kBoundsMaxInit;
}

// ---------------------------------------------------------------------------
// march
// ---------------------------------------------------------------------------
struct MarchParams {
    int32_t n_rays;
    const float* rays_o;
    const float* rays_d;
    const float* near_planes;  // per ray, or null: near_plane for every ray
    const float* far_planes;
    float near_plane, far_plane;
    OccGeom g;
    const uint64_t* words;
    const int32_t* bounds;  // occupied-brick bounding boxes (nullable)
    const float* aabbs;
    const float* t_sorted;
    const int64_t* t_indices;
    const uint8_t* hits;
    float step_size;
    LatTable lat_table;   // lattice points at the binade starts, from the uniform near plane (n = 0: none)
    unsigned long long* trace;  // measurement aid (nfa_debug_set_march_trace): 8 x u64 per warp, or null
    Workspace ws;
    int64_t* totals;
    int64_t* totals_host;  // optional host-visible mirror (pinned memory), saves a D2H copy node
    float* terminate;
};

// descriptor buffer: one shared-memory column per thread, joined flags in a register
struct SmemBuf {
    float* pend;   // [slots][tile]
    float* open;
    uint32_t joined_mask;
    int tid, tile;
    __device__ __forceinline__ void put(int j, float p, float o, bool jn)
    {
        pend[j * tile + tid] = p;
        open[j * tile + tid] = o;
        joined_mask |= (jn ? 1u : 0u) << j;
    }
};

// append the runs the lanes of a warp closed in this step: one atomic per warp
__device__ __forceinline__ void emit_runs(const RunOut& out, uint32_t ray, uint32_t tile, const Workspace& ws, int lane)
{
    const unsigned mask = __ballot_sync(0xffffffffu, out.valid);
    if (mask == 0u) return;
    const int leader = __ffs(mask) - 1;
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(ws.cursor, (uint32_t)__popc(mask));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (out.valid) {
        const uint32_t slot = base + (uint32_t)__popc(mask & ((1u << lane) - 1u));
        if ((int64_t)slot < ws.run_capacity) {
            uint4* dst = reinterpret_cast<uint4*>(ws.pool + slot);
            dst[0] = make_uint4(ray, out.sample_off, out.n, __float_as_uint(out.t_first));
            dst[1] = make_uint4(out.run_idx, tile, 0u, 0u);
        }
    }
}

// dynamic shared memory of the march kernel (tile = blockDim.x rays):
//   [o: 3 tile f32] [d: 3 tile f32] [pend: slots tile] [open: slots tile] [order: tile u32]
__host__ __device__ inline size_t march_smem_bytes(int tile, int slots)
{
    return (size_t)tile * 4 * (3 + 3 + 2 * slots + 1);
}

template <bool kSingle, int kSlots>
__global__ void __launch_bounds__(kMaxTileRays) march_kernel(const MarchParams p)
{
    extern __shared__ __align__(16) uint32_t s_dyn[];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ unsigned long long s_red_samples[kMaxTileRays / 32];
    __shared__ uint32_t s_red_runs[kMaxTileRays / 32], s_red_flags[kMaxTileRays / 32], s_wsum[kMaxTileRays / 32];
    __shared__ bool s_last;
    __shared__ uint32_t s_hist[kSortBuckets];

    const int T = blockDim.x;            // threads = rays of a (full) tile
    const int tid = threadIdx.x, lane = tid & 31;
    unsigned long long tr_t0 = 0, tr_c0 = 0, tr_c1 = 0, tr_c2 = 0, tr_c3 = 0, tr_w = 0;
    int tr_first = 1, tr_loops = 0;
    if (p.trace) {
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tr_t0));
        tr_c0 = clock64();
    }
    const int tile = blockIdx.x;
    const int r0 = tile * T;
    const int nr = min(T, p.n_rays - r0);
    float* s_o = reinterpret_cast<float*>(s_dyn);
    float* s_d = s_o + 3 * T;
    float* s_pend = s_d + 3 * T;
    constexpr int S = kSlots;  // stretch descriptors buffered per ray
    float* s_open = s_pend + S * T;
    uint32_t* s_sort = reinterpret_cast<uint32_t*>(s_open + S * T);
    float* s_tail = reinterpret_cast<float*>(s_sort);  // lattice point after a ray's last stretch: each thread has read
                                                       // its s_sort slot long before a lane of its warp writes here

    // ---- stage the ray tile into shared memory: TMA bulk copies + mbarrier
    const float* g_o = p.rays_o + (int64_t)r0 * 3;
    const float* g_d = p.rays_d + (int64_t)r0 * 3;
    const uint32_t ray_bytes = (uint32_t)nr * 12u;
    const bool bulk_rays = ((ray_bytes & 15u) == 0u) && ((((uintptr_t)g_o) | ((uintptr_t)g_d)) & 15u) == 0u;
    if (tid == 0) mbar_init(&s_bar, 1);
    if (kSingle && tid < kSortBuckets) s_hist[tid] = 0u;
    if (kSingle && T < kSortBuckets) {
        for (int i = tid + T; i < kSortBuckets; i += T) s_hist[i] = 0u;
    }
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(&s_bar, bulk_rays ? 2u * ray_bytes : 0u);
        if (bulk_rays) {
            bulk_g2s(s_o, g_o, ray_bytes, &s_bar);
            bulk_g2s(s_d, g_d, ray_bytes, &s_bar);
        }
    }
    if (!bulk_rays) {
        for (int i = tid; i < nr * 3; i += T) {
            s_o[i] = g_o[i];
            s_d[i] = g_d[i];
        }
    }
    mbar_wait(&s_bar, 0);
    __syncthreads();

    // ---- order the tile's rays by expected walk length, so the 32 lanes of a warp finish together.
    // A warp runs as long as its longest ray; with rays in input order a third of the lanes of the cell loop idle.
    // The estimate (cells crossed between the slab hits of the box the walk is confined to) only decides which
    // thread takes which ray -- every output is indexed by ray id.  Counting sort: bucket histogram with shared
    // atomics (the order inside a bucket is arbitrary and irrelevant), one warp scans the buckets.
    int rt = tid;
    if (kSingle) {
        uint32_t bucket = 0;
        if (tid < nr) {
            const float* box = p.aabbs;
            const bool have_bb = p.bounds != nullptr && p.terminate == nullptr && p.bounds[0] <= p.bounds[3];
            float tn = p.near_planes ? p.near_planes[r0 + tid] : p.near_plane;
            float tf = p.far_planes ? p.far_planes[r0 + tid] : p.far_plane;
            float cells = 0.f, span = 0.f;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                const float voxel = (box[3 + a] - box[a]) / (float)p.g.res[a];
                const float lo = have_bb ? box[a] + (float)(4 * p.bounds[a] - 1) * voxel : box[a];
                const float hi = have_bb ? box[a] + (float)(4 * p.bounds[3 + a] + 5) * voxel : box[3 + a];
                const float oa = s_o[tid * 3 + a], da = s_d[tid * 3 + a];
                const float inv = __fdividef(1.0f, da);
                const float t0 = (lo - oa) * inv, t1 = (hi - oa) * inv;
                tn = fmaxf(tn, fminf(t0, t1));
                tf = fminf(tf, fmaxf(t0, t1));
                cells += __fdividef(fabsf(da), voxel);
                span += __fdividef(hi - lo, voxel);  // a walk crosses at most this many cells (all three axes)
            }
            // real rays take buckets 1 .. 255 (NaN / miss -> 1); bucket 0 is left to the threads without a ray, so
            // that those sort in front of every ray
            const float est = cells * (tf - tn) * __fdividef((float)(kSortBuckets - 2), span);
            bucket = 1u;
            if (est > 0.f) bucket = 1u + (est < (float)(kSortBuckets - 2) ? (uint32_t)est : (uint32_t)(kSortBuckets - 2));
        }
        const uint32_t pos = atomicAdd(&s_hist[bucket], 1u);
        __syncthreads();
        if (tid < 32) {  // exclusive scan of the 256 bucket counts: 8 per lane + a shuffle scan
            uint32_t c[kSortBuckets / 32], sum = 0;
#pragma unroll
            for (int i = 0; i < kSortBuckets / 32; ++i) {
                c[i] = s_hist[tid * (kSortBuckets / 32) + i];
                sum += c[i];
            }
            uint32_t incl = sum;
#pragma unroll
            for (int sft = 1; sft < 32; sft <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, incl, sft);
                if (lane >= sft) incl += y;
            }
            uint32_t run = incl - sum;
#pragma unroll
            for (int i = 0; i < kSortBuckets / 32; ++i) {
                s_hist[tid * (kSortBuckets / 32) + i] = run;
                run += c[i];
            }
        }
        __syncthreads();
        s_sort[s_hist[bucket] + pos] = (uint32_t)tid;
        __syncthreads();
        rt = (int)s_sort[tid];
    }
    const int r = r0 + rt;
    bool active = rt < nr;
    float near = 0.f, far = 0.f;
    if (active) {
        near = p.near_planes ? p.near_planes[r] : p.near_plane;
        far = p.far_planes ? p.far_planes[r] : p.far_plane;
    }

    if (p.trace) tr_c1 = clock64();  // staging + sort done
    // ---- two-phase march (march.cuh) ---------------------------------------
    OccView occ;
    occ.words = p.words;
    occ.coarse = nullptr;  // the march reads brick words only
    occ.bounds = p.bounds;
    occ.g = p.g;
    const Lattice L = lat_make(p.step_size);
    const float o[3] = {active ? s_o[rt * 3 + 0] : 0.f, active ? s_o[rt * 3 + 1] : 0.f, active ? s_o[rt * 3 + 2] : 0.f};
    const float d[3] = {active ? s_d[rt * 3 + 0] : 1.f, active ? s_d[rt * 3 + 1] : 1.f, active ? s_d[rt * 3 + 2] : 1.f};
    Walk w;
    LatState m;
    walk_init(w, o, d, near, far);
    lat_init(m, L, near);
    w.done = active ? 0 : 1;
    // nothing after the last occupied cell is observable without a terminate plane on one level
    w.accel = (kSingle && p.terminate == nullptr) ? 1 : 0;
    SmemBuf buf;
    buf.pend = s_pend;
    buf.open = s_open;
    buf.joined_mask = 0u;
    buf.tid = tid;
    buf.tile = T;
    int n_desc = 0;
    const int G = p.g.n_grids;
    const int64_t rr = active ? r : 0;
    const SingleBox single{p.aabbs};
    const SortedBoxes sorted{p.aabbs, G, kSingle ? nullptr : p.t_sorted + rr * 2 * G,
                             kSingle ? nullptr : p.t_indices + rr * 2 * G, kSingle ? nullptr : p.hits + rr * G};
    for (;;) {
        // phase 1: DDA only (divergent, cheap)
        if (kSingle) walk_run(w, single, occ, buf, n_desc, S);
        else walk_run(w, sorted, occ, buf, n_desc, S);
        if (p.trace) {
            if (tr_first) tr_w = clock64();  // first walk pass of this warp done
            tr_first = 0;
            ++tr_loops;
        }
        // phase 2: lattice seeks, all lanes in step
        const int maxd = __reduce_max_sync(0xffffffffu, n_desc);
        if (kSingle && !__any_sync(0xffffffffu, buf.joined_mask != 0u)) {
            // One level: the stretches of the warp's 32 rays are independent (march.cuh, lat_stretch), so they are
            // dealt out to the lanes -- most rays have one, a ray that grazes the surface up to 8, and a lane that
            // took its ray's stretches one after the other made the warp with the grazing rays the tile's slowest.
            if (__any_sync(0xffffffffu, m.run_n > 0u)) {  // (only after a round that went the other way)
                RunOut out;
                lat_close(m, out);
                emit_runs(out, (uint32_t)r, (uint32_t)tile, p.ws, lane);
            }
            if (n_desc > 0) lat_anchor(m, p.lat_table, s_pend[tid]);
            const float anchor = m.t;
            __syncwarp();  // the first stretch's slot is rewritten below, possibly by another lane
            int incl = n_desc;
#pragma unroll
            for (int sft = 1; sft < 32; sft <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, incl, sft);
                if (lane >= sft) incl += y;
            }
            const int total = __shfl_sync(0xffffffffu, incl, 31);
            const int excl = incl - n_desc;
            for (int base = 0; base < total; base += 32) {
                const int i = min(base + lane, total - 1);
                int o = 0;  // owner of stretch i: the first lane whose inclusive count exceeds i
#pragma unroll
                for (int sft = 16; sft > 0; sft >>= 1) {
                    const int v = __shfl_sync(0xffffffffu, incl, o + sft - 1);
                    if (v <= i) o += sft;
                }
                const int j = i - __shfl_sync(0xffffffffu, excl, o);
                const float a_o = __shfl_sync(0xffffffffu, anchor, o);
                const int ok_o = __shfl_sync(0xffffffffu, m.ok ? 1 : 0, o);
                const int nd_o = __shfl_sync(0xffffffffu, n_desc, o);
                if (base + lane < total) {
                    const int col = tid - lane + o;
                    float first, after;
                    uint32_t n;
                    lat_stretch(L, a_o, ok_o != 0, s_pend[j * T + col], s_open[j * T + col], first, n, after);
                    s_pend[j * T + col] = first;
                    s_open[j * T + col] = __uint_as_float(n);
                    if (j == nd_o - 1) s_tail[col] = after;
                }
            }
            __syncwarp();
            // back to one lane per ray: count the ray's runs (stretches that hold a sample), take the pool slots of the
            // whole warp with ONE atomic (its round trip to L2 per stretch index was a fifth of this phase), then
            // add up the offsets and write the records -- plain per-lane loops, no warp-wide step inside
            uint32_t mine = 0;
            {
                bool still_ok = m.ok;
                for (int j = 0; j < n_desc; ++j) {
                    const uint32_t n = __float_as_uint(s_open[j * T + tid]);
                    if (n == kStretchFailed) still_ok = false;
                    mine += (still_ok && n != 0u) ? 1u : 0u;
                }
            }
            uint32_t upto = mine;
#pragma unroll
            for (int sft = 1; sft < 32; sft <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, upto, sft);
                if (lane >= sft) upto += y;
            }
            const uint32_t all = __shfl_sync(0xffffffffu, upto, 31);
            if (all != 0u) {
                uint32_t slot = 0;
                if (lane == 0) slot = atomicAdd(p.ws.cursor, all);
                slot = __shfl_sync(0xffffffffu, slot, 0) + upto - mine;
                for (int j = 0; j < n_desc; ++j) {
                    RunOut out;
                    lat_take(m, s_pend[j * T + tid], __float_as_uint(s_open[j * T + tid]), out);
                    if (out.valid) {
                        if ((int64_t)slot < p.ws.run_capacity) {
                            uint4* dst = reinterpret_cast<uint4*>(p.ws.pool + slot);
                            dst[0] = make_uint4((uint32_t)r, out.sample_off, out.n, __float_as_uint(out.t_first));
                            dst[1] = make_uint4(out.run_idx, (uint32_t)tile, 0u, 0u);
                        }
                        ++slot;
                    }
                }
            } else {
                for (int j = 0; j < n_desc; ++j) {  // nothing to write; a failed seek still has to be noted
                    RunOut out;
                    lat_take(m, s_pend[j * T + tid], __float_as_uint(s_open[j * T + tid]), out);
                }
            }
            if (n_desc > 0 && m.ok) m.t = s_tail[tid];
        } else {
            for (int j = 0; j < maxd; ++j) {
                RunOut out;
                out.valid = false;
                if (j < n_desc)
                    lat_consume(m, s_pend[j * T + tid], s_open[j * T + tid], (buf.joined_mask >> j) & 1u, out);
                emit_runs(out, (uint32_t)r, (uint32_t)tile, p.ws, lane);
            }
        }
        n_desc = 0;
        buf.joined_mask = 0u;
        if (__all_sync(0xffffffffu, w.done != 0)) break;
    }
    {
        RunOut out;
        out.valid = false;
        float term = 0.f;
        if (active) term = lat_finish(m, walk_tail_pend(w), p.terminate != nullptr, out);
        emit_runs(out, (uint32_t)r, (uint32_t)tile, p.ws, lane);
        if (active) {
            p.ws.cnt_samples[r] = m.n_samples;
            p.ws.cnt_runs[r] = m.n_runs;
            if (p.terminate) p.terminate[r] = term;
        }
    }

    if (p.trace) {
        tr_c2 = clock64();  // this warp's rays done
    }
    // ---- tile sums, and grand totals by the last CTA to finish ------------
    const int n_warps = T >> 5;
    unsigned long long vs = active ? m.n_samples : 0u;
    uint32_t vr = active ? m.n_runs : 0u, vf = (active && !m.ok) ? 1u : 0u;
#pragma unroll
    for (int sft = 16; sft > 0; sft >>= 1) {
        vs += __shfl_xor_sync(0xffffffffu, vs, sft);
        vr += __shfl_xor_sync(0xffffffffu, vr, sft);
        vf += __shfl_xor_sync(0xffffffffu, vf, sft);
    }
    if (lane == 0) {
        s_red_samples[tid >> 5] = vs;
        s_red_runs[tid >> 5] = vr;
        s_red_flags[tid >> 5] = vf;
    }
    __syncthreads();
    if (tid == 0) {
        TileSum ts;
        ts.samples = 0;
        ts.runs = 0;
        ts.stuck = 0;
        for (int k = 0; k < n_warps; ++k) {
            ts.samples += s_red_samples[k];
            ts.runs += s_red_runs[k];
            ts.stuck += s_red_flags[k];
        }
        p.ws.tiles[tile] = ts;
        __threadfence();
        const uint32_t prev = atomicAdd(p.ws.done, 1u);
        s_last = (prev == (uint32_t)(gridDim.x - 1));
    }
    // Samples of the earlier rays of this tile, in RAY order (the threads hold the rays in sorted order): with the
    // tile bases below this is every ray's packed_info start, so that no separate offsets pass has to run before the
    // samples are expanded.  The descriptor buffers are free by now (barrier above): counts go through them.
    uint32_t* s_cnt = reinterpret_cast<uint32_t*>(s_pend);
    if (active) s_cnt[rt] = m.n_samples;
    __syncthreads();
    {
        const uint32_t cs = tid < nr ? s_cnt[tid] : 0u;
        uint32_t xs = cs;
#pragma unroll
        for (int sft = 1; sft < 32; sft <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, xs, sft);
            if (lane >= sft) xs += y;
        }
        if (lane == 31) s_wsum[tid >> 5] = xs;
        __syncthreads();
        uint32_t before = xs - cs;
        for (int k = 0; k < (tid >> 5); ++k) before += s_wsum[k];
        if (tid < nr) p.ws.loc_samples[r0 + tid] = before;
    }
    if (p.trace && lane == 0) {
        tr_c3 = clock64();  // past the tile's last barrier
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        unsigned int smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        unsigned long long* q = p.trace + 8 * ((size_t)blockIdx.x * (kMaxTileRays / 32) + (tid >> 5));
        q[0] = tr_t0; q[1] = t1; q[2] = tr_c1 - tr_c0; q[3] = tr_c2 - tr_c0; q[4] = tr_c3 - tr_c0; q[5] = smid;
        q[6] = ((unsigned long long)tr_loops << 48) | ((tr_w - tr_c0) & 0xffffffffffffull); q[7] = 1;
    }
    if (s_last) {
        __threadfence();
        // tile bases (exclusive scan of the tile sums: a contiguous chunk of tiles per thread) and the grand totals
        const int n_tiles = p.ws.n_tiles;
        const int chunk = (n_tiles + T - 1) / T;
        const int i0 = min(tid * chunk, n_tiles), i1 = min(i0 + chunk, n_tiles);
        unsigned long long a = 0, b = 0, c = 0;
        for (int i = i0; i < i1; ++i) {
            const volatile unsigned long long* q = (const volatile unsigned long long*)&p.ws.tiles[i];
            const unsigned long long w0 = q[0], w1 = q[1];  // {samples}, {runs | stuck << 32}
            a += w0;
            b += (uint32_t)w1;
            c += w1 >> 32;
        }
        unsigned long long xa = a;
#pragma unroll
        for (int sft = 1; sft < 32; sft <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, xa, sft);
            if (lane >= sft) xa += y;
        }
#pragma unroll
        for (int sft = 16; sft > 0; sft >>= 1) {
            b += __shfl_xor_sync(0xffffffffu, b, sft);
            c += __shfl_xor_sync(0xffffffffu, c, sft);
        }
        __shared__ unsigned long long s_tot[3][kMaxTileRays / 32];
        if (lane == 31) s_tot[0][tid >> 5] = xa;
        if (lane == 0) {
            s_tot[1][tid >> 5] = b;
            s_tot[2][tid >> 5] = c;
        }
        __syncthreads();
        {
            unsigned long long base = xa - a;
            for (int k = 0; k < (tid >> 5); ++k) base += s_tot[0][k];
            for (int i = i0; i < i1; ++i) {
                p.ws.tile_base[i] = base;
                base += *(const volatile unsigned long long*)&p.ws.tiles[i];
            }
        }
        if (tid < 3) {
            unsigned long long v = 0;
            for (int k = 0; k < n_warps; ++k) v += s_tot[tid][k];
            // totals: [0] samples, [1] runs, [2] run-pool capacity used for this call, [3] stuck rays
            p.totals[tid == 2 ? 3 : tid] = (int64_t)v;
            if (p.totals_host) p.totals_host[tid == 2 ? 3 : tid] = (int64_t)v;
        }
        if (tid == 3) {
            p.totals[2] = p.ws.run_capacity;
            if (p.totals_host) p.totals_host[2] = p.ws.run_capacity;
        }
        // (no system-scope fence: the host reads the pinned totals after it has waited for this kernel)
        if (tid == 0) {  // leave the workspace reusable
            *p.ws.done = 0u;
            *p.ws.cursor = 0u;
        }
    }
}

// ---------------------------------------------------------------------------
// offsets: per-ray packed_info from the counts (tile base from the tile sums + block scan)
// ---------------------------------------------------------------------------
template <bool kIntervals>
__global__ void __launch_bounds__(kMaxTileRays) offsets_kernel(int32_t n_rays, Workspace ws, int64_t* sm_packed_info,
                                                              int64_t* iv_packed_info)
{
    __shared__ unsigned long long s_red[2][kMaxTileRays / 32];
    __shared__ unsigned long long s_base[2];
    __shared__ uint32_t s_wsum[2][kMaxTileRays / 32];
    const int T = blockDim.x;  // == ws.tile_rays
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = T >> 5;
    const int tile = blockIdx.x;
    const int r0 = tile * T;
    const int nr = min(T, n_rays - r0);

    unsigned long long a = 0, b = 0;
    for (int i = tid; i < tile; i += T) {
        const TileSum ts = ws.tiles[i];
        a += ts.samples;
        b += ts.runs;
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, s);
        b += __shfl_xor_sync(0xffffffffu, b, s);
    }
    if (lane == 0) {
        s_red[0][warp] = a;
        s_red[1][warp] = b;
    }
    uint32_t cs = 0, cr = 0;
    if (tid < nr) {
        cs = ws.cnt_samples[r0 + tid];
        cr = ws.cnt_runs[r0 + tid];
    }
    uint32_t xs = cs, xr = cr;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        const uint32_t ys = __shfl_up_sync(0xffffffffu, xs, s);
        const uint32_t yr = __shfl_up_sync(0xffffffffu, xr, s);
        if (lane >= s) {
            xs += ys;
            xr += yr;
        }
    }
    if (lane == 31) {
        s_wsum[0][warp] = xs;
        s_wsum[1][warp] = xr;
    }
    __syncthreads();
    if (tid == 0) {
        unsigned long long ta = 0, tb = 0;
        for (int k = 0; k < n_warps; ++k) {
            ta += s_red[0][k];
            tb += s_red[1][k];
        }
        s_base[0] = ta;
        s_base[1] = tb;
    }
    __syncthreads();
    unsigned long long wsum = 0, wrun = 0;
    for (int k = 0; k < warp; ++k) {
        wsum += s_wsum[0][k];
        wrun += s_wsum[1][k];
    }
    if (tid < nr) {
        const unsigned long long off = s_base[0] + wsum + (xs - cs);
        // packed_info = [chunk_start, chunk_cnt]  (reference data_specs.py:68-69)
        longlong2 v;
        v.x = (long long)off;
        v.y = (long long)cs;
        *reinterpret_cast<longlong2*>(sm_packed_info + 2 * (int64_t)(r0 + tid)) = v;
        if (kIntervals) {
            longlong2 e;  // a run of n samples has n + 1 edges
            e.x = (long long)(off + s_base[1] + wrun + (xr - cr));
            e.y = (long long)cs + (long long)cr;
            *reinterpret_cast<longlong2*>(iv_packed_info + 2 * (int64_t)(r0 + tid)) = e;
        }
    }
}

// ---------------------------------------------------------------------------
// expand: runs -> per-sample arrays, one warp per run, coalesced stores
// ---------------------------------------------------------------------------
struct ExpandParams {
    Workspace ws;
    int32_t n_rays;
    const int64_t* totals;  // device copy of the march totals ([1] = number of runs)
    float step_size;
    int64_t sample_capacity;
    const int64_t* sm_packed_info;
    int64_t* packed_out;  // samples-only vectorised kernel: packed_info is written here, not read
    int64_t* ray_indices;
    float* t_starts;
    float* t_ends;
    // interval mode
    int64_t edge_capacity;
    const int64_t* iv_packed_info;
    float* iv_vals;
    int64_t* iv_ray_indices;
    uint8_t* iv_is_left;
    uint8_t* iv_is_right;
    float* sm_vals;
    uint8_t* sm_is_valid;
};

template <bool kIntervals>
__global__ void __launch_bounds__(kExpandThreads) expand_runs_kernel(const ExpandParams p)
{
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * kExpandThreads + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * kExpandThreads) >> 5;
    int64_t n_runs = p.totals[1];
    if (n_runs > p.ws.run_capacity) n_runs = p.ws.run_capacity;  // the host re-runs with a larger pool
    const Lattice L = lat_make(p.step_size);
    for (int64_t q = warp0; q < n_runs; q += n_warps) {
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(p.ws.pool + q));
        const int64_t ray = a.x;
        int64_t off = p.sm_packed_info[2 * ray] + a.y;
        int64_t eoff = 0;
        if (kIntervals) {
            const uint4 b = __ldg(reinterpret_cast<const uint4*>(p.ws.pool + q) + 1);
            eoff = p.iv_packed_info[2 * ray] + a.y + b.x;
        }
        RunIter it;
        it.t = __uint_as_float(a.w);
        it.left = a.z;
        bool first_piece = true;
        while (it.left > 0) {
            LatPiece pc;
            const uint32_t c = run_next_piece(L, it, pc);
            for (uint32_t j = lane; j < c; j += 32) {
                const float ts = piece_start(pc, j);
                const float te = f_add(ts, L.dt);
                const int64_t k = off + j;
                if (!kIntervals) {
                    if (k < p.sample_capacity) {
                        p.ray_indices[k] = ray;
                        p.t_starts[k] = ts;
                        p.t_ends[k] = te;
                    }
                } else {
                    if (k < p.sample_capacity) {
                        p.ray_indices[k] = ray;                     // samples.ray_indices
                        p.sm_vals[k] = f_mul(f_add(te, ts), 0.5f);  // reference grid.cu:251
                        p.sm_is_valid[k] = 1;
                    }
                    const int64_t e = eoff + j;
                    if (e < p.edge_capacity) {  // left edge of sample j (reference grid.cu:219-245)
                        p.iv_vals[e] = ts;
                        p.iv_ray_indices[e] = ray;
                        p.iv_is_left[e] = 1;
                        p.iv_is_right[e] = (first_piece && j == 0) ? 0 : 1;
                    }
                    if (it.left == 0 && j == c - 1 && e + 1 < p.edge_capacity) {  // closing edge of the run
                        p.iv_vals[e + 1] = te;
                        p.iv_ray_indices[e + 1] = ray;
                        p.iv_is_left[e + 1] = 0;
                        p.iv_is_right[e + 1] = 1;
                    }
                }
            }
            off += c;
            eoff += c;
            first_piece = false;
        }
    }
}

// Samples-only expansion with 128-bit stores: a piece (lattice.cuh) of a run is written as an
// unaligned head (< 4 samples), a body of output groups [4G, 4G+3] -- one lane per group: a float4 of
// starts, a float4 of ends, two longlong2 of ray ids -- and a tail.  Same values as the scalar kernel.
// (32-bit sample offsets and one division less per run were measured: no change -- the store stream bounds it.)
__global__ void __launch_bounds__(kExpandThreads) expand_runs_vec_kernel(const ExpandParams p)
{
    using Idx = int64_t;
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * kExpandThreads + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * kExpandThreads) >> 5;
    int64_t n_runs = p.totals[1];
    if (n_runs > p.ws.run_capacity) n_runs = p.ws.run_capacity;
    const Lattice L = lat_make(p.step_size);
    // packed_info of every ray = [base of the ray's march tile + samples of the tile's earlier rays, count]: the march
    // kernel left both parts in the workspace, so no offsets pass runs in front of this kernel.  The runs below take
    // their offsets from the same two arrays, not from packed_info (another CTA may not have written it yet).
    for (int64_t r = (int64_t)blockIdx.x * kExpandThreads + threadIdx.x; r < p.n_rays;
         r += (int64_t)gridDim.x * kExpandThreads) {
        longlong2 v;
        v.x = (long long)(p.ws.tile_base[r / p.ws.tile_rays] + p.ws.loc_samples[r]);
        v.y = (long long)p.ws.cnt_samples[r];
        *reinterpret_cast<longlong2*>(p.packed_out + 2 * r) = v;
    }
    for (int64_t q = warp0; q < n_runs; q += n_warps) {
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(p.ws.pool + q));
        const uint32_t run_tile = __ldg(&p.ws.pool[q].tile);
        const long long ray = a.x;
        const int64_t off64 = (int64_t)(p.ws.tile_base[run_tile] + p.ws.loc_samples[ray]) + a.y;
        RunIter it;
        it.t = __uint_as_float(a.w);
        it.left = a.z;
        if (off64 >= p.sample_capacity) it.left = 0;
        else if (off64 + it.left > p.sample_capacity) it.left = (uint32_t)(p.sample_capacity - off64);
        Idx off = (Idx)off64;
        while (it.left > 0) {
            LatPiece pc;
            const Idx c = (Idx)run_next_piece(L, it, pc);
            // head: bring `off` to a multiple of 4 (also covers short pieces entirely)
            const int head = (int)min((Idx)((4 - (off & 3)) & 3), c);
            const Idx body_groups = (c - head) >> 2;
            const int tail = (int)(c - head - 4 * body_groups);
            if (lane < head) {
                const float ts = piece_start(pc, (uint32_t)lane);
                p.ray_indices[off + lane] = ray;
                p.t_starts[off + lane] = ts;
                p.t_ends[off + lane] = f_add(ts, L.dt);
            }
            const Idx g0 = (off + head) >> 2;
            for (Idx gi = lane; gi < body_groups; gi += 32) {
                const uint32_t j = (uint32_t)(head + 4 * gi);
                float4 s4, e4;
                s4.x = piece_start(pc, j);     e4.x = f_add(s4.x, L.dt);
                s4.y = piece_start(pc, j + 1); e4.y = f_add(s4.y, L.dt);
                s4.z = piece_start(pc, j + 2); e4.z = f_add(s4.z, L.dt);
                s4.w = piece_start(pc, j + 3); e4.w = f_add(s4.w, L.dt);
                reinterpret_cast<float4*>(p.t_starts)[g0 + gi] = s4;
                reinterpret_cast<float4*>(p.t_ends)[g0 + gi] = e4;
                const longlong2 rr = make_longlong2(ray, ray);
                reinterpret_cast<longlong2*>(p.ray_indices)[2 * (g0 + gi)] = rr;
                reinterpret_cast<longlong2*>(p.ray_indices)[2 * (g0 + gi) + 1] = rr;
            }
            if (lane < tail) {
                const Idx k = off + head + 4 * body_groups + lane;
                const float ts = piece_start(pc, (uint32_t)(head + 4 * body_groups + lane));
                p.ray_indices[k] = ray;
                p.t_starts[k] = ts;
                p.t_ends[k] = f_add(ts, L.dt);
            }
            off += c;
        }
    }
}

// ---------------------------------------------------------------------------
// generic traversal (march_generic.cuh): cone angle, per-cell sampling, step limit, masks
// ---------------------------------------------------------------------------
struct GenericParams {
    int32_t n_rays;
    const float* rays_o;
    const float* rays_d;
    const uint8_t* rays_mask;  // nullable
    const float* near_planes;
    const float* far_planes;
    OccGeom g;
    const uint64_t* words;
    const uint32_t* coarse;
    const float* aabbs;
    const float* t_sorted;
    const int64_t* t_indices;
    const uint8_t* hits;
    float step_size, cone_angle;
    int32_t limit;
    int32_t fill;
    const int64_t* slots;  // over-allocation: index of the ray among the unmasked ones (its fixed-stride slot), or null
    const int64_t* iv_starts;
    int64_t* iv_cnts;
    float* iv_vals;
    int64_t* iv_ray;
    uint8_t* iv_left;
    uint8_t* iv_right;
    const int64_t* sm_starts;
    int64_t* sm_cnts;
    float* sm_vals;
    int64_t* sm_ray;
    uint8_t* sm_valid;
    float* terminate;
};

__global__ void __launch_bounds__(128) generic_traverse_kernel(const GenericParams p)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= p.n_rays) return;
    if (p.rays_mask && !p.rays_mask[r]) {  // reference grid.cu:100
        if (p.slots) p.iv_cnts[r] = p.sm_cnts[r] = 0;
        return;
    }
    if (p.fill && !p.slots && (p.iv_cnts[r] == 0 || p.sm_cnts[r] == 0)) return;  // grid.cu:103-106
    OccView occ;
    occ.words = p.words;
    occ.coarse = p.coarse;
    occ.bounds = nullptr;
    occ.g = p.g;
    GenericOut out;
    out.fill = p.fill != 0;
    out.ray = r;
    out.want_iv = true;
    out.want_sm = true;
    // fixed-stride slots (over_allocate, grid.cu:364-404): 2 * limit edges and limit samples per unmasked ray
    out.iv_base = p.slots ? p.slots[r] * 2 * p.limit : (p.fill ? p.iv_starts[r] : 0);
    out.sm_base = p.slots ? p.slots[r] * p.limit : (p.fill ? p.sm_starts[r] : 0);
    out.iv_vals = p.iv_vals; out.iv_ray = p.iv_ray; out.iv_left = p.iv_left; out.iv_right = p.iv_right;
    out.sm_vals = p.sm_vals; out.sm_ray = p.sm_ray; out.sm_valid = p.sm_valid;
    out.n_edges = 0;
    out.n_samples = 0;
    const int G = p.g.n_grids;
    const SortedBoxes boxes{p.aabbs, G, p.t_sorted + (int64_t)r * 2 * G, p.t_indices + (int64_t)r * 2 * G,
                            p.hits + (int64_t)r * G};
    const float o[3] = {p.rays_o[3 * (int64_t)r], p.rays_o[3 * (int64_t)r + 1], p.rays_o[3 * (int64_t)r + 2]};
    const float d[3] = {p.rays_d[3 * (int64_t)r], p.rays_d[3 * (int64_t)r + 1], p.rays_d[3 * (int64_t)r + 2]};
    const float term = generic_march_ray(boxes, occ, o, d, p.near_planes[r], p.far_planes[r], p.step_size, p.cone_angle,
                                         p.limit, out);
    if (p.terminate) p.terminate[r] = term;
    p.iv_cnts[r] = out.n_edges;
    p.sm_cnts[r] = out.n_samples;
}

// ---------------------------------------------------------------------------
// ray / box kernels (reference grid.cu:284-313; grid.py:156-162)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ray_aabb_kernel(int32_t n_rays, const float* __restrict__ rays_o,
                                                       const float* __restrict__ rays_d, int32_t n_aabbs,
                                                       const float* __restrict__ aabbs, float near, float far,
                                                       float miss, float* __restrict__ t_mins,
                                                       float* __restrict__ t_maxs, uint8_t* __restrict__ hits)
{
    const int64_t total = (int64_t)n_rays * n_aabbs;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / n_aabbs;
        const int g = (int)(i - r * n_aabbs);
        const float o[3] = {rays_o[3 * r], rays_o[3 * r + 1], rays_o[3 * r + 2]};
        const float inv[3] = {f_rcp(rays_d[3 * r]), f_rcp(rays_d[3 * r + 1]), f_rcp(rays_d[3 * r + 2])};
        float a = miss, b = miss;
        const bool hit = slab_test(o, inv, aabbs + 6 * g, near, far, a, b);
        t_mins[i] = hit ? a : miss;
        t_maxs[i] = hit ? b : miss;
        hits[i] = hit ? 1 : 0;
    }
}

constexpr int kMaxSortBoxes = 32;

__global__ void __launch_bounds__(128) intersect_sorted_kernel(int32_t n_rays, const float* __restrict__ rays_o,
                                                               const float* __restrict__ rays_d, int32_t n_aabbs,
                                                               const float* __restrict__ aabbs,
                                                               float* __restrict__ t_sorted,
                                                               int64_t* __restrict__ t_indices,
                                                               uint8_t* __restrict__ hits)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rays) return;
    const float o[3] = {rays_o[3 * (int64_t)r], rays_o[3 * (int64_t)r + 1], rays_o[3 * (int64_t)r + 2]};
    const float inv[3] = {f_rcp(rays_d[3 * (int64_t)r]), f_rcp(rays_d[3 * (int64_t)r + 1]),
                          f_rcp(rays_d[3 * (int64_t)r + 2])};
    float v[2 * kMaxSortBoxes];
    int ix[2 * kMaxSortBoxes];
    const int m = 2 * n_aabbs;
    for (int g = 0; g < n_aabbs; ++g) {
        float a = INFINITY, b = INFINITY;
        const bool hit = slab_test(o, inv, aabbs + 6 * g, -INFINITY, INFINITY, a, b);
        v[g] = hit ? a : INFINITY;
        v[n_aabbs + g] = hit ? b : INFINITY;
        hits[(int64_t)r * n_aabbs + g] = hit ? 1 : 0;
    }
    // stable insertion sort of (value, position in cat([t_mins, t_maxs]))
    for (int j = 0; j < m; ++j) {
        const float x = v[j];
        int k = j;
        while (k > 0 && v[k - 1] > x) {
            v[k] = v[k - 1];
            ix[k] = ix[k - 1];
            --k;
        }
        v[k] = x;
        ix[k] = j;
    }
    for (int j = 0; j < m; ++j) {
        t_sorted[(int64_t)r * m + j] = v[j];
        t_indices[(int64_t)r * m + j] = ix[j];
    }
}

}  // namespace nfa

// ===========================================================================
// C ABI
// ===========================================================================
using namespace nfa;

static inline int32_t launch_status()
{
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? NFA_OK : (int32_t)e;
}

static unsigned long long* g_march_trace = nullptr;

// One march launch; the dynamic shared memory limit is raised above the 48 KiB default once per instantiation and
// device.
template <bool kSingle, int kSlots>
static void launch_march(const MarchParams& p, int tiles, int threads, cudaStream_t s)
{
    const size_t dyn = march_smem_bytes(threads, kSlots);
    static bool raised[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dyn > 40 * 1024 && !raised[dev & 63]) {
        cudaFuncSetAttribute(march_kernel<kSingle, kSlots>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        raised[dev & 63] = true;
    }
    march_kernel<kSingle, kSlots><<<tiles, threads, dyn, s>>>(p);
}

extern "C" {

// measurement aid, not part of the product path: per-warp time stamps of the next nfa_march launches go to
// `buffer` (8 x u64 per warp, n_tiles x 16 warps); null switches it off
void nfa_debug_set_march_trace(void* buffer) { g_march_trace = (unsigned long long*)buffer; }

int32_t nfa_version(void) { return NFA_ABI_VERSION; }

const char* nfa_error_string(int32_t code)
{
    if (code == NFA_OK) return "ok";
    if (code == NFA_ERR_ARG) return "invalid argument";
    if (code == NFA_ERR_UNSUPPORTED) return "unsupported configuration";
    if (code > 0) return cudaGetErrorString((cudaError_t)code);
    return "unknown error";
}

int32_t nfa_ray_aabb_intersect(int32_t n_rays, const float* rays_o, const float* rays_d, int32_t n_aabbs,
                               const float* aabbs, float near_plane, float far_plane, float miss_value,
                               float* t_mins, float* t_maxs, uint8_t* hits, nfa_stream_t stream)
{
    if (n_rays < 0 || n_aabbs < 0) return NFA_ERR_ARG;
    const int64_t total = (int64_t)n_rays * n_aabbs;
    if (total == 0) return NFA_OK;
    if (!rays_o || !rays_d || !aabbs || !t_mins || !t_maxs || !hits) return NFA_ERR_ARG;
    const int blocks = (int)((total + 255) / 256 < kNumSMs * 32 ? (total + 255) / 256 : kNumSMs * 32);
    ray_aabb_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(n_rays, rays_o, rays_d, n_aabbs, aabbs, near_plane,
                                                               far_plane, miss_value, t_mins, t_maxs, hits);
    return launch_status();
}

int32_t nfa_intersect_sorted(int32_t n_rays, const float* rays_o, const float* rays_d, int32_t n_aabbs,
                             const float* aabbs, float* t_sorted, int64_t* t_indices, uint8_t* hits,
                             nfa_stream_t stream)
{
    if (n_rays < 0 || n_aabbs <= 0) return NFA_ERR_ARG;
    if (n_aabbs > kMaxSortBoxes) return NFA_ERR_UNSUPPORTED;
    if (n_rays == 0) return NFA_OK;
    if (!rays_o || !rays_d || !aabbs || !t_sorted || !t_indices || !hits) return NFA_ERR_ARG;
    intersect_sorted_kernel<<<(n_rays + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n_rays, rays_o, rays_d, n_aabbs,
                                                                                    aabbs, t_sorted, t_indices, hits);
    return launch_status();
}

int64_t nfa_occ_words(int32_t n_grids, int32_t rx, int32_t ry, int32_t rz)
{
    if (n_grids <= 0 || rx <= 0 || ry <= 0 || rz <= 0) return 0;
    return (int64_t)n_grids * occ_geom(n_grids, rx, ry, rz).wpl;
}

int64_t nfa_occ_coarse_words(int32_t n_grids, int32_t rx, int32_t ry, int32_t rz)
{
    if (n_grids <= 0 || rx <= 0 || ry <= 0 || rz <= 0) return 0;
    return occ_coarse_words(occ_geom(n_grids, rx, ry, rz));
}

int32_t nfa_occ_pack(int32_t n_grids, int32_t rx, int32_t ry, int32_t rz, const uint8_t* binaries, uint64_t* words,
                     uint32_t* coarse, int32_t* bounds, nfa_stream_t stream)
{
    if (n_grids <= 0 || rx <= 0 || ry <= 0 || rz <= 0 || !binaries || !words || !coarse || !bounds) return NFA_ERR_ARG;
    const OccGeom g = occ_geom(n_grids, rx, ry, rz);
    const int64_t n_words = (int64_t)n_grids * g.wpl;
    if (n_words > (int64_t)INT32_MAX) return NFA_ERR_UNSUPPORTED;
    const int64_t n_coarse = occ_coarse_words(g);
    const int64_t threads = n_coarse * 16;
    const int blocks = (int)((threads + 255) / 256 < kNumSMs * 16 ? (threads + 255) / 256 : kNumSMs * 16);
    occ_bounds_init_kernel<<<(6 * n_grids + 127) / 128, 128, 0, (cudaStream_t)stream>>>(bounds, n_grids);
    occ_pack_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(g, binaries, words, coarse, bounds, n_words, n_coarse);
    return launch_status();
}

int64_t nfa_march_workspace_bytes(int32_t n_rays, int64_t run_capacity)
{
    return (n_rays < 0 || run_capacity < 0) ? 0 : ws_bytes(n_rays, run_capacity);
}

int32_t nfa_march(int32_t n_rays, const float* rays_o, const float* rays_d, const float* near_planes,
                  const float* far_planes, float near_plane, float far_plane, int32_t n_grids, int32_t rx,
                  int32_t ry, int32_t rz,
                  const uint64_t* words, const int32_t* bounds, const float* aabbs,
                  const float* t_sorted, const int64_t* t_indices, const uint8_t* hits, float step_size,
                  int64_t run_capacity, void* workspace, int64_t* totals, int64_t* totals_host,
                  float* terminate_planes, nfa_stream_t stream)
{
    if (n_rays < 0 || n_grids <= 0 || rx <= 0 || ry <= 0 || rz <= 0 || run_capacity < 0) return NFA_ERR_ARG;
    if (run_capacity > (int64_t)UINT32_MAX) return NFA_ERR_UNSUPPORTED;
    if (!(step_size > 0.0f)) return NFA_ERR_UNSUPPORTED;
    if (!totals) return NFA_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    if ((near_planes == nullptr) != (far_planes == nullptr)) return NFA_ERR_ARG;
    if (n_rays == 0) {
        if (totals_host) totals_host[0] = totals_host[1] = totals_host[2] = totals_host[3] = 0;
        return (int32_t)cudaMemsetAsync(totals, 0, 4 * sizeof(int64_t), s);
    }
    if (!rays_o || !rays_d || !words || !aabbs || !workspace)
        return NFA_ERR_ARG;
    const bool have_sorted = t_sorted && t_indices && hits;
    if (!have_sorted && n_grids != 1) return NFA_ERR_ARG;
    MarchParams p;
    p.n_rays = n_rays;
    p.rays_o = rays_o;
    p.rays_d = rays_d;
    p.near_planes = near_planes;
    p.far_planes = far_planes;
    p.near_plane = near_plane;
    p.far_plane = far_plane;
    p.g = occ_geom(n_grids, rx, ry, rz);
    p.words = words;
    p.bounds = bounds;
    p.aabbs = aabbs;
    p.t_sorted = have_sorted ? t_sorted : nullptr;
    p.t_indices = have_sorted ? t_indices : nullptr;
    p.hits = have_sorted ? hits : nullptr;
    p.step_size = step_size;
    p.trace = g_march_trace;
    p.lat_table.n = 0;
    p.lat_table.e0 = 0;
    if (near_planes == nullptr && step_size > 0.f) {  // the climb from the near plane, once per (step, near plane)
        static thread_local LatTable cached;
        static thread_local float cached_dt = 0.f, cached_near = 0.f;
        static thread_local bool cached_valid = false;
        if (!cached_valid || cached_dt != step_size || cached_near != near_plane) {
            lat_table_build(lat_make(step_size), near_plane, cached);
            cached_dt = step_size;
            cached_near = near_plane;
            cached_valid = true;
        }
        p.lat_table = cached;
    }
    p.ws = ws_view(workspace, n_rays, run_capacity);
    p.totals = totals;
    p.totals_host = totals_host;
    p.terminate = terminate_planes;
    const int tiles = p.ws.n_tiles, threads = p.ws.tile_rays;
    // one wave (every tile resident at once, at most two per SM): room for twice the descriptor slots
    const bool wide = tiles <= 2 * kNumSMs && threads >= 224;
    if (!have_sorted) {
        if (wide) launch_march<true, kDescSlotsWide>(p, tiles, threads, s);
        else launch_march<true, kDescSlots>(p, tiles, threads, s);
    } else {
        if (wide) launch_march<false, kDescSlotsWide>(p, tiles, threads, s);
        else launch_march<false, kDescSlots>(p, tiles, threads, s);
    }
    return launch_status();
}

static inline int expand_grid(int64_t run_capacity)
{
    const int64_t ctas = (run_capacity * 32 + kExpandThreads - 1) / kExpandThreads;
    const int64_t cap = kNumSMs * 8;  // 8 resident CTAs of 256 threads per SM
    return (int)(ctas < 1 ? 1 : (ctas < cap ? ctas : cap));
}

int32_t nfa_expand_samples(int32_t n_rays, int64_t run_capacity, const void* workspace, const int64_t* totals,
                           float step_size, int64_t capacity, int64_t* packed_info, int64_t* ray_indices,
                           float* t_starts, float* t_ends, nfa_stream_t stream)
{
    if (n_rays < 0 || capacity < 0 || run_capacity < 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!workspace || !packed_info || !totals) return NFA_ERR_ARG;
    if (capacity > 0 && (!ray_indices || !t_starts || !t_ends)) return NFA_ERR_ARG;
    if ((((uintptr_t)packed_info) & 15u) != 0) return NFA_ERR_ARG;
    const Workspace ws = ws_view(const_cast<void*>(workspace), n_rays, run_capacity);
    cudaStream_t s = (cudaStream_t)stream;
    const uintptr_t al = (uintptr_t)ray_indices | (uintptr_t)t_starts | (uintptr_t)t_ends;
    const bool expand = capacity > 0 && run_capacity > 0;
    // the vectorised kernel writes packed_info itself (from what the march left in the workspace); the offsets pass
    // only runs in front of the scalar fallback (unaligned outputs) or when there is nothing to expand
    if (!expand || (al & 15u) != 0) offsets_kernel<false><<<ws.n_tiles, ws.tile_rays, 0, s>>>(n_rays, ws, packed_info, nullptr);
    if (expand) {
        ExpandParams p = {};
        p.ws = ws;
        p.n_rays = n_rays;
        p.totals = totals;
        p.step_size = step_size;
        p.sample_capacity = capacity;
        p.sm_packed_info = packed_info;
        p.packed_out = packed_info;
        p.ray_indices = ray_indices;
        p.t_starts = t_starts;
        p.t_ends = t_ends;
        if ((al & 15u) != 0) expand_runs_kernel<false><<<expand_grid(run_capacity), kExpandThreads, 0, s>>>(p);
        else expand_runs_vec_kernel<<<expand_grid(run_capacity), kExpandThreads, 0, s>>>(p);
    }
    return launch_status();
}

int32_t nfa_expand_intervals(int32_t n_rays, int64_t run_capacity, const void* workspace, const int64_t* totals,
                             float step_size, int64_t edge_capacity, int64_t sample_capacity,
                             int64_t* iv_packed_info, float* iv_vals, int64_t* iv_ray_indices, uint8_t* iv_is_left,
                             uint8_t* iv_is_right, int64_t* sm_packed_info, float* sm_vals, int64_t* sm_ray_indices,
                             uint8_t* sm_is_valid, nfa_stream_t stream)
{
    if (n_rays < 0 || edge_capacity < 0 || sample_capacity < 0 || run_capacity < 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!workspace || !iv_packed_info || !sm_packed_info || !totals) return NFA_ERR_ARG;
    if (edge_capacity > 0 && (!iv_vals || !iv_ray_indices || !iv_is_left || !iv_is_right)) return NFA_ERR_ARG;
    if (sample_capacity > 0 && (!sm_vals || !sm_ray_indices || !sm_is_valid)) return NFA_ERR_ARG;
    if (((((uintptr_t)iv_packed_info) | ((uintptr_t)sm_packed_info)) & 15u) != 0) return NFA_ERR_ARG;
    const Workspace ws = ws_view(const_cast<void*>(workspace), n_rays, run_capacity);
    cudaStream_t s = (cudaStream_t)stream;
    offsets_kernel<true><<<ws.n_tiles, ws.tile_rays, 0, s>>>(n_rays, ws, sm_packed_info, iv_packed_info);
    if (edge_capacity > 0 && run_capacity > 0) {
        ExpandParams p = {};
        p.ws = ws;
        p.totals = totals;
        p.step_size = step_size;
        p.sample_capacity = sample_capacity;
        p.sm_packed_info = sm_packed_info;
        p.ray_indices = sm_ray_indices;
        p.edge_capacity = edge_capacity;
        p.iv_packed_info = iv_packed_info;
        p.iv_vals = iv_vals;
        p.iv_ray_indices = iv_ray_indices;
        p.iv_is_left = iv_is_left;
        p.iv_is_right = iv_is_right;
        p.sm_vals = sm_vals;
        p.sm_is_valid = sm_is_valid;
        expand_runs_kernel<true><<<expand_grid(run_capacity), kExpandThreads, 0, s>>>(p);
    }
    return launch_status();
}

int32_t nfa_traverse_generic(int32_t n_rays, const float* rays_o, const float* rays_d, const uint8_t* rays_mask,
                             const float* near_planes, const float* far_planes, int32_t n_grids, int32_t rx, int32_t ry,
                             int32_t rz, const uint64_t* words, const uint32_t* coarse, const float* aabbs,
                             const float* t_sorted, const int64_t* t_indices, const uint8_t* hits, float step_size,
                             float cone_angle, int32_t traverse_steps_limit, int32_t fill, const int64_t* slots,
                             const int64_t* iv_starts, int64_t* iv_cnts, float* iv_vals, int64_t* iv_ray_indices, uint8_t* iv_is_left,
                             uint8_t* iv_is_right, const int64_t* sm_starts, int64_t* sm_cnts, float* sm_vals,
                             int64_t* sm_ray_indices, uint8_t* sm_is_valid, float* terminate_planes, nfa_stream_t stream)
{
    if (n_rays < 0 || n_grids <= 0 || rx <= 0 || ry <= 0 || rz <= 0) return NFA_ERR_ARG;
    if (n_rays == 0) return NFA_OK;
    if (!rays_o || !rays_d || !near_planes || !far_planes || !words || !coarse || !aabbs || !t_sorted || !t_indices ||
        !hits || !iv_cnts || !sm_cnts)
        return NFA_ERR_ARG;
    if (fill && !slots && (!iv_starts || !sm_starts)) return NFA_ERR_ARG;
    if (slots && !(fill && traverse_steps_limit > 0)) return NFA_ERR_ARG;
    GenericParams p;
    p.n_rays = n_rays;
    p.rays_o = rays_o;
    p.rays_d = rays_d;
    p.rays_mask = rays_mask;
    p.near_planes = near_planes;
    p.far_planes = far_planes;
    p.g = occ_geom(n_grids, rx, ry, rz);
    p.words = words;
    p.coarse = coarse;
    p.aabbs = aabbs;
    p.t_sorted = t_sorted;
    p.t_indices = t_indices;
    p.hits = hits;
    p.step_size = step_size;
    p.cone_angle = cone_angle;
    p.limit = traverse_steps_limit;
    p.fill = fill;
    p.slots = slots;
    p.iv_starts = iv_starts; p.iv_cnts = iv_cnts; p.iv_vals = iv_vals; p.iv_ray = iv_ray_indices;
    p.iv_left = iv_is_left; p.iv_right = iv_is_right;
    p.sm_starts = sm_starts; p.sm_cnts = sm_cnts; p.sm_vals = sm_vals; p.sm_ray = sm_ray_indices;
    p.sm_valid = sm_is_valid;
    p.terminate = terminate_planes;
    generic_traverse_kernel<<<(n_rays + 127) / 128, 128, 0, (cudaStream_t)stream>>>(p);
    return launch_status();
}

}  // extern "C"
