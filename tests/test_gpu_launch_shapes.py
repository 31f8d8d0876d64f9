"""The march / expand / compositing kernels at every launch shape they dispatch to.

`nfa_march` picks its tile (rays per CTA) and one of four `march_kernel<kSingle, kSlots>` instantiations from the
batch size alone (traverse.cu: march_tile_rays and the `wide` rule).  Small test batches only ever reach a few of
them, so this file chooses its ray counts from a Python mirror of that rule (pinned against the library on the CPU)
and runs every instantiation, the 32- and 256-ray tiles, rays whose stretch counts sit on both sides of the 8- and
16-slot boundaries, the run-pool re-march, clipped and unaligned expands through the C ABI, and the compositing
kernels with more rays than resident warps -- bit-exact against the CPU oracle (float outputs at the compositing
bars).  The CPU tests pin the mirror and run the host simulation of the walk at both slot widths."""
import ctypes as C

import numpy as np
import pytest
import torch

from nerfacc_b200 import scenes

dev = "cuda:0"

# ---------------------------------------------------------------- the launch rule, mirrored

NUM_SMS = 132        # sm_count.cuh: kNumSMs (H100 SXM)
SLOTS, SLOTS_WIDE = 8, 16


def march_tile_rays(n_rays):
    """traverse.cu march_tile_rays: rays per march CTA (the tile that spreads the rays most evenly over the SMs
    with every CTA resident, ties to the larger tile).  Element-wise on an int64 array."""
    r = np.asarray(n_rays, np.int64)
    best, best_cost = np.full(r.shape, 128), np.full(r.shape, np.iinfo(np.int64).max)
    for t in range(64, 513, 32):
        cost = -(-(-(-r // t)) // NUM_SMS) * t          # ceil(tiles / SMs) tiles of t rays on the busiest SM
        ok = (cost <= 2048) & (cost <= best_cost)
        best, best_cost = np.where(ok, t, best), np.where(ok, cost, best_cost)
    return np.where(r <= 32, 32, np.where(r > NUM_SMS * 2048, 256, best))


def march_shape(n_rays: int, levels: int):
    """(one level?, descriptor slots, tile): which march_kernel instantiation nfa_march launches, and its tile."""
    t = int(march_tile_rays(n_rays))
    wide = -(-n_rays // t) <= 2 * NUM_SMS and t >= 224
    return levels == 1, SLOTS_WIDE if wide else SLOTS, t


def _workspace_bytes(n_rays, tile):
    """nfa_march_workspace_bytes(n_rays, 0) for a given tile: header, tile sums, three per-ray u32 arrays, tile
    bases (traverse.cu ws_bytes); strictly increasing in the tile count."""
    a16 = lambda x: (x + 15) // 16 * 16
    nt = -(-n_rays // tile)
    return 64 + a16(16 * nt) + 3 * a16(4 * n_rays) + a16(8 * nt)


# Ray counts of the sampling matrix (levels, rays), and what each one launches.
R_TILE32 = 29          # <= 32 rays: one 32-ray tile
R_WIDE1 = 30_000       # wide: 118 tiles of 256, one per SM
R_WIDE2 = 100_000      # wide: 261 tiles of 384, two per SM
R_GAP = 86_000         # inside the wide range's size, but 384 tiles of 224: narrow
R_NARROW = 140_000     # narrow, 64-ray tiles
R_T256 = 300_000       # beyond 132 x 2048: 256-ray tiles
MATRIX_R = (R_TILE32, R_WIDE1, R_WIDE2, R_GAP, R_NARROW, R_T256)
# stretch counts of the comb rays: both sides of the 8- and 16-slot boundaries, and three rounds of 16
COMB_K = (1, 7, 8, 9, 15, 16, 17, 33)


def test_tile_mirror_reproduces_the_library_workspace_size():
    """The mirror's tile count gives the library's workspace size for every batch up to 2^20 rays: the rule that
    picks the tile cannot change without this test (and the coverage claim below) noticing."""
    from nerfacc_b200 import _lib
    lib = _lib.load()
    rs = np.arange(1, (1 << 20) + 1, dtype=np.int64)
    want = _workspace_bytes(rs, march_tile_rays(rs))
    fn = lib.nfa_march_workspace_bytes
    got = np.fromiter((fn(int(r), 0) for r in rs), np.int64, count=rs.size)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"mirror disagrees with the library at n_rays = {rs[bad[:10]].tolist()}"
    # the edges of the rule: one 32-ray tile, the start and end of the first wide range, 256-ray tiles
    assert [march_shape(r, 1)[1:] for r in (32, 33, 25_344, 25_345, 84_480, 84_481, 270_336, 270_337)] == \
        [(8, 32), (8, 64), (8, 192), (16, 224), (16, 320), (8, 224), (8, 512), (8, 256)]


def test_chosen_ray_counts_cover_every_launch_shape():
    """The sampling matrix below runs all four march instantiations, the 32- and 256-ray tiles, and both widths with
    rays of 7 to 33 stretches (comb scene, one and four levels)."""
    shapes = {march_shape(r, lv) for r in MATRIX_R for lv in (1, 4)}
    assert {(s, k) for s, k, _ in shapes} == {(True, 8), (True, 16), (False, 8), (False, 16)}
    assert {t for _, _, t in shapes} >= {32, 256}
    assert march_shape(R_WIDE1, 1)[1:] == (16, 256) and march_shape(R_WIDE2, 1)[1:] == (16, 384)
    assert march_shape(R_GAP, 1)[1] == 8 and march_shape(R_NARROW, 1)[1] == 8 and march_shape(R_T256, 1)[2] == 256
    assert -(-R_WIDE1 // 256) <= NUM_SMS < -(-R_WIDE2 // 384) <= 2 * NUM_SMS   # one, then two tiles per SM
    # a 33-stretch ray takes three rounds of the wide buffer and five of the narrow one
    assert max(COMB_K) > 2 * SLOTS_WIDE and any(SLOTS < k <= SLOTS_WIDE for k in COMB_K)
    # the run-pool and expand cases
    assert march_shape(POOL_R[0], 1)[1] == 8 and march_shape(POOL_R[1], 1)[1] == 16
    assert COMPOSITE_R > NUM_SMS * 64


# ---------------------------------------------------------------- scenes with a known stretch count

def comb_grid(levels: int) -> np.ndarray:
    """[levels, 128, 8, 8]: along x, occupied one-cell slabs separated by empty cells.  The (y, z) column of row
    (y, z) holds k = COMB_K[(y + 3z) % 8] slabs; outer levels are empty."""
    g = np.zeros((levels, 128, 8, 8), bool)
    for y in range(8):
        for z in range(8):
            g[0, 1:2 * COMB_K[(y + 3 * z) % 8]:2, y, z] = True
    return g


def comb_rays(per_row: int, levels: int, seed: int = 0):
    """Rays along +x / -x through the comb rows: the first of each row along x at the cell centre, the others
    offset and tilted by less than the half cell they would need to leave the row.  Returns (o, d, k)."""
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(64), per_row)
    yz = np.stack([rows // 8, rows % 8], 1)
    centre = -1.0 + (yz + 0.5) * 0.25
    first = np.arange(rows.size) % per_row == 0
    sign = np.where(first | (rng.random(rows.size) < 0.5), 1.0, -1.0)
    start = 1.5 if levels == 1 else 8.5                      # outside the outermost box
    off = np.where(first[:, None], 0.0, rng.uniform(-0.04, 0.04, (rows.size, 2)))
    tilt = np.where(first[:, None], 0.0, rng.uniform(-0.06, 0.06, (rows.size, 2)) / (start + 1.0))
    o = np.concatenate([(-sign * start)[:, None], centre + off], 1)
    d = np.concatenate([sign[:, None], tilt], 1)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    k = np.array([COMB_K[(y + 3 * z) % 8] for y, z in yz])
    return o.astype(np.float32), d.astype(np.float32), k


COMB_STEP = 0.0117   # 3/4 of a cell: every slab holds a sample and every gap breaks the run, so runs == stretches


def frag_scene(levels: int):
    """Fragmented grids with many stretches per ray: the ball with half its cells dropped (one level), or a random
    half-full 4-level grid with rays from all directions.  Returns (bins, aabbs, o, d, step, far plane)."""
    rng = np.random.default_rng(7 if levels == 1 else 11)
    if levels == 1:
        bins = scenes.ball_grid(128) & (rng.random((1, 128, 128, 128)) > 0.5)
        o, d = scenes.ball_rays(4096, seed=5)
        return bins, scenes.nested_aabbs(1), o, d, 1.3e-2, 1e10
    bins = rng.random((4, 32, 32, 32)) > 0.5
    o = rng.standard_normal((4096, 3)).astype(np.float32)
    d = rng.standard_normal((4096, 3)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return bins, scenes.nested_aabbs(4), o, d, 0.08, 5.0


def scene(name: str):
    kind, levels = name[:-1], int(name[-1])
    if kind == "comb":
        o, d, _ = comb_rays(64, levels)
        return comb_grid(levels), scenes.nested_aabbs(levels), o, d, COMB_STEP, 1e10
    return frag_scene(levels)


SCENES = ("comb1", "comb4", "frag1", "frag4")


# ---------------------------------------------------------------- host simulation at both slot widths (CPU)

F = C.POINTER(C.c_float)
U32 = C.POINTER(C.c_uint32)
I64 = C.POINTER(C.c_int64)
U8 = C.POINTER(C.c_uint8)
U64 = C.POINTER(C.c_uint64)
I32 = C.POINTER(C.c_int32)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _sim_slots(sim, ro, rd, bins, aabbs, step, slots, multi, accel):
    """March every ray in the host simulation with `slots` descriptor slots, expand the runs; as the kernels do."""
    sim.sim_march_slots.restype = C.c_int64
    sim.sim_march_slots.argtypes = [C.c_int32, F, F, F, F, C.c_int, C.c_int, C.c_int, C.c_int, U64, U32, I32, C.c_int, F,
                                    F, I64, U8, C.c_float, I64, I64, F, I32, F, U32, C.c_int64, C.c_int]
    G, rx, ry, rz = bins.shape
    R = ro.shape[0]
    words = np.zeros(sim.sim_occ_words(G, rx, ry, rz), np.uint64)
    coarse = np.zeros(sim.sim_occ_coarse_words(G, rx, ry, rz), np.uint32)
    bounds = np.zeros(6 * G, np.int32)
    b8 = np.ascontiguousarray(bins.astype(np.uint8))
    sim.sim_occ_pack(G, rx, ry, rz, _p(b8, U8), _p(words, U64), _p(coarse, U32), _p(bounds, I32))
    near, far = np.zeros(R, np.float32), np.full(R, 1e10, np.float32)
    ns, nr = np.zeros(R, np.int64), np.zeros(R, np.int64)
    term, ok = np.zeros(R, np.float32), np.zeros(R, np.int32)
    cap = 64 * R + 1024
    rt, rn = np.zeros(cap, np.float32), np.zeros(cap, np.uint32)
    ts_, ti_, h_ = multi if multi is not None else (None, None, None)
    tot = sim.sim_march_slots(R, _p(ro, F), _p(rd, F), _p(near, F), _p(far, F), G, rx, ry, rz, _p(words, U64),
                              _p(coarse, U32), _p(bounds, I32), accel, _p(aabbs, F), _p(ts_, F), _p(ti_, I64), _p(h_, U8),
                              step, _p(ns, I64), _p(nr, I64), _p(term, F), _p(ok, I32), _p(rt, F), _p(rn, U32), cap, slots)
    assert tot >= 0 and ok.all()
    N = int(ns.sum())
    s, e = np.empty(N, np.float32), np.empty(N, np.float32)
    w = 0
    for q in range(int(tot)):
        n = int(rn[q])
        sim.sim_expand_run(float(rt[q]), step, n, s[w:].ctypes.data_as(F), e[w:].ctypes.data_as(F))
        w += n
    assert w == N
    return ns, nr, s, e, term


@pytest.mark.parametrize("name", SCENES)
def test_host_sim_walk_at_8_and_16_slots(host_sim, orc, name):
    """The shared walk / lattice logic with the narrow and the wide descriptor buffer, against the oracle: comb rays
    of 1 to 33 stretches (one and three rounds of 16), fragmented scenes; one level (inline walk, empty-space jump,
    phase 2 by stretch) and nested."""
    bins, aabbs, ro, rd, step, far = scene(name)
    ro, rd = ro[::4].copy(), rd[::4].copy()      # 1024 rays
    R = ro.shape[0]
    iv, sm, o_term = orc.traverse_grids(ro, rd, bins, aabbs, near_planes=np.zeros(R, np.float32),
                                        far_planes=np.full(R, 1e10, np.float32), step_size=step)
    runs = iv["packed_info"][:, 1] - sm["packed_info"][:, 1]
    if name.startswith("comb"):
        np.testing.assert_array_equal(runs, comb_rays(64, bins.shape[0])[2][::4])   # runs == stretches == k
    assert runs.max() > 2 * SLOTS_WIDE if name.startswith("comb") else runs.max() > SLOTS_WIDE
    multi = None
    if bins.shape[0] > 1:
        tm, tM, h = orc.ray_aabb_intersect(ro, rd, aabbs)
        tsrt, tidx = orc.sort_intersections(tm, tM)
        multi = (tsrt, tidx, np.ascontiguousarray(h.astype(np.uint8)))
    accels = (0, 1, 2) if multi is None else (0,)
    for slots in (SLOTS, SLOTS_WIDE):
        for accel in accels:
            ns, nr, s, e, term = _sim_slots(host_sim, ro, rd, bins, aabbs, step, slots, multi, accel)
            msg = f"{name} slots={slots} accel={accel}"
            np.testing.assert_array_equal(ns, sm["packed_info"][:, 1], err_msg=msg)
            np.testing.assert_array_equal(nr, runs, err_msg=msg)
            np.testing.assert_array_equal(s, iv["vals"][iv["is_left"]], err_msg=msg)
            np.testing.assert_array_equal(e, iv["vals"][iv["is_right"]], err_msg=msg)
            if accel == 0:
                d = ~np.isnan(o_term)
                np.testing.assert_array_equal(term[d], o_term[d], err_msg=msg)
    assert host_sim.sim_march_slots(0, *([None] * 4), 1, 1, 1, 1, *([None] * 3), 0, *([None] * 4), 0.01,
                                    *([None] * 6), 0, 12) == -2   # only the two kernel widths exist


# ---------------------------------------------------------------- GPU helpers

def T(a, **kw):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev, **kw)


def N(t):
    return t.detach().cpu().numpy()


def _estimator(bins, aabbs):
    import nerfacc_b200 as nfa
    est = nfa.OccGridEstimator(torch.from_numpy(aabbs[0]), resolution=list(bins.shape[1:]), levels=bins.shape[0]).to(dev)
    est.binaries = T(bins)
    return est


def _batch(n_distinct: int, n_rays: int, seed: int):
    """Indices of a batch of `n_rays` rays drawn from `n_distinct`: every distinct ray as evenly as possible,
    shuffled so that each warp sees a mix."""
    idx = np.resize(np.arange(n_distinct), n_rays)
    np.random.default_rng(seed).shuffle(idx)
    return idx


def _gather(pi, idx):
    """Per-ray segments `pi` of the distinct rays -> (packed_info of the batch, source position of every element,
    ray id of every element)."""
    cnt = pi[idx, 1]
    start = np.cumsum(cnt) - cnt
    src = np.repeat(pi[idx, 0] - start, cnt) + np.arange(int(cnt.sum()))
    return np.stack([start, cnt], -1), src, np.repeat(np.arange(len(idx)), cnt)


_oracle_cache = {}


def _oracle(orc, name):
    """The oracle's traversal of a scene's distinct rays (computed once per scene)."""
    if name not in _oracle_cache:
        bins, aabbs, ro, rd, step, far = scene(name)
        R = ro.shape[0]
        _oracle_cache[name] = orc.traverse_grids(ro, rd, bins, aabbs, near_planes=np.zeros(R, np.float32),
                                                 far_planes=np.full(R, far, np.float32), step_size=step)
    return _oracle_cache[name]


# ---------------------------------------------------------------- sampling matrix

@pytest.mark.gpu
@pytest.mark.parametrize("n_rays", MATRIX_R)
@pytest.mark.parametrize("name", SCENES)
def test_sampling_at_every_launch_shape(orc, name, n_rays):
    """est.sampling on batches of repeated, shuffled rays vs the oracle on the distinct rays: ray_indices, t_starts,
    t_ends and packed_info bit-exact."""
    import nerfacc_b200 as nfa
    bins, aabbs, ro, rd, step, far = scene(name)
    iv, sm, _ = _oracle(orc, name)
    idx = _batch(ro.shape[0], n_rays, seed=n_rays)
    pi, src, ray = _gather(sm["packed_info"], idx)
    assert len(src) <= 10_500_000
    o_ts, o_te = iv["vals"][iv["is_left"]], iv["vals"][iv["is_right"]]
    est = _estimator(bins, aabbs)
    ri, ts, te = est.sampling(T(ro[idx]), T(rd[idx]), render_step_size=step, far_plane=far)
    np.testing.assert_array_equal(N(ri), ray)
    np.testing.assert_array_equal(N(ts), o_ts[src])
    np.testing.assert_array_equal(N(te), o_te[src])
    np.testing.assert_array_equal(N(nfa.pack_info(ri, n_rays)), pi)


@pytest.mark.gpu
@pytest.mark.parametrize("name,n_rays", [("comb1", R_WIDE2), ("comb4", R_WIDE1), ("frag1", R_T256),
                                         ("frag4", R_GAP), ("comb4", R_TILE32)])
def test_traverse_grids_at_launch_shapes(orc, name, n_rays):
    """traverse_grids (march with terminate planes + nfa_expand_intervals) vs the oracle: every interval and sample
    field, both packed_info arrays and the terminate planes."""
    import nerfacc_b200 as nfa
    bins, aabbs, ro, rd, step, far = scene(name)
    o_iv, o_sm, o_term = _oracle(orc, name)
    idx = _batch(ro.shape[0], n_rays, seed=n_rays + 1)
    iv, sm, term = nfa.traverse_grids(T(ro[idx]), T(rd[idx]), T(bins), T(aabbs),
                                      far_planes=torch.full((n_rays,), far, device=dev), step_size=step)
    ipi, isrc, iray = _gather(o_iv["packed_info"], idx)
    spi, ssrc, sray = _gather(o_sm["packed_info"], idx)
    np.testing.assert_array_equal(N(iv.packed_info), ipi)
    np.testing.assert_array_equal(N(iv.vals), o_iv["vals"][isrc])
    np.testing.assert_array_equal(N(iv.is_left), o_iv["is_left"][isrc])
    np.testing.assert_array_equal(N(iv.is_right), o_iv["is_right"][isrc])
    np.testing.assert_array_equal(N(iv.ray_indices), iray)
    np.testing.assert_array_equal(N(sm.packed_info), spi)
    np.testing.assert_array_equal(N(sm.vals), o_sm["vals"][ssrc])
    np.testing.assert_array_equal(N(sm.ray_indices), sray)
    assert bool(sm.is_valid.all())
    want = o_term[idx]
    d = ~np.isnan(want)
    np.testing.assert_array_equal(N(term)[d], want[d])


@pytest.mark.gpu
def test_every_march_instantiation_and_tile_ran():
    """The march kernels the profiler saw at the matrix's ray counts: all four instantiations, each launch the one
    the mirror predicts (so the tiles the mirror gives these counts, 32 and 256 among them, are the ones that ran)."""
    import re
    from torch.profiler import ProfilerActivity, profile

    def instantiation(kernel_name):   # demangled ("march_kernel<true, 16>") or mangled ("march_kernelILb1ELi16E")
        m = re.search(r"march_kernel<(true|false), ?(\d+)>", kernel_name)
        if m:
            return f"march_kernel<{m[1]}, {m[2]}>"
        m = re.search(r"march_kernelILb([01])ELi(\d+)E", kernel_name)
        return None if m is None else f"march_kernel<{'true' if m[1] == '1' else 'false'}, {m[2]}>"

    seen = set()
    for name in ("comb1", "comb4"):
        bins, aabbs, ro, rd, step, far = scene(name)
        est = _estimator(bins, aabbs)
        for n_rays in MATRIX_R:
            idx = _batch(ro.shape[0], n_rays, seed=3)
            o, d = T(ro[idx]), T(rd[idx])
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                est.sampling(o, d, render_step_size=step, far_plane=far)
                torch.cuda.synchronize()
            launched = {instantiation(ev.name) for ev in prof.events()} - {None}
            assert len(launched) == 1, (name, n_rays, launched)
            seen.add((launched.pop(), n_rays, bins.shape[0]))
    inst = {s[0] for s in seen}
    assert inst == {"march_kernel<true, 8>", "march_kernel<true, 16>", "march_kernel<false, 8>",
                    "march_kernel<false, 16>"}, inst
    for kname, n_rays, levels in seen:   # each launch is the one the mirror predicts
        single, slots, _ = march_shape(n_rays, levels)
        assert kname == f"march_kernel<{'true' if single else 'false'}, {slots}>", (kname, n_rays, levels)


# ---------------------------------------------------------------- run-pool overflow

POOL_R = (20_000, 60_000)   # narrow (160-ray tiles) and wide (480-ray tiles)


@pytest.mark.gpu
@pytest.mark.parametrize("n_rays", POOL_R)
def test_run_pool_overflow_remarches(orc, n_rays):
    """A new stream gets its own scratch whose run pool holds 2R + 1024 runs; the fragmented ball has ~14 runs per
    ray, so the first march overflows it.  The pool must have grown (only the re-march grows it) and the samples
    must still be the oracle's."""
    from nerfacc_b200 import _lib, grid as _grid
    bins, aabbs, ro, rd, step, far = scene("frag1")
    iv, sm, _ = _oracle(orc, "frag1")
    idx = _batch(ro.shape[0], n_rays, seed=n_rays + 2)
    pi, src, ray = _gather(sm["packed_info"], idx)
    runs = int((iv["packed_info"][idx, 1] - sm["packed_info"][idx, 1]).sum())
    assert runs > 2 * n_rays + 1024
    est = _estimator(bins, aabbs)
    o, d = T(ro[idx]), T(rd[idx])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        key = (torch.device(dev), _lib.stream_ptr(torch.device(dev)))
        _grid._scratch_cache.pop(key, None)     # the stream may be one a previous test used: start from a new scratch
        ri, ts, te = est.sampling(o, d, render_step_size=step)
        scratch = _grid._scratch_cache[key]
    torch.cuda.synchronize()
    assert len(scratch) == 1 and scratch[0].run_capacity >= runs > 2 * n_rays + 1024
    np.testing.assert_array_equal(N(ri), ray)
    np.testing.assert_array_equal(N(ts), iv["vals"][iv["is_left"]][src])
    np.testing.assert_array_equal(N(te), iv["vals"][iv["is_right"]][src])


# ---------------------------------------------------------------- expand through the C ABI

GUARD = 256
F_SENT, I_SENT, B_SENT = -1234.5, -7, 0xAB


def _march_abi(name):
    """One nfa_march of a scene's distinct rays into a workspace of our own; returns what the expand calls need."""
    from nerfacc_b200 import _lib, grid as _grid
    lib = _lib.load()
    bins, aabbs, ro, rd, step, far = scene(name)
    R = ro.shape[0]
    G, rx, ry, rz = bins.shape
    device = torch.device(dev)
    occ = _grid._OccPack(T(bins))
    o, d, a = T(ro), T(rd), T(aabbs)
    tsrt = tidx = hits = None
    if G > 1:
        tsrt = torch.empty((R, 2 * G), dtype=torch.float32, device=dev)
        tidx = torch.empty((R, 2 * G), dtype=torch.int64, device=dev)
        hits = torch.empty((R, G), dtype=torch.bool, device=dev)
        _lib.call("nfa_intersect_sorted", device, R, o.data_ptr(), d.data_ptr(), G, a.data_ptr(), tsrt.data_ptr(),
                  tidx.data_ptr(), hits.data_ptr())
    cap = 64 * R + 1024
    ws = torch.zeros(lib.nfa_march_workspace_bytes(R, cap), dtype=torch.uint8, device=dev)
    tot = torch.zeros(4, dtype=torch.int64, device=dev)
    _lib.call("nfa_march", device, R, o.data_ptr(), d.data_ptr(), None, None, 0.0, far, G, rx, ry, rz,
              occ.words.data_ptr(), occ.bounds.data_ptr(), a.data_ptr(), _lib.ptr(tsrt), _lib.ptr(tidx), _lib.ptr(hits),
              step, cap, ws.data_ptr(), tot.data_ptr(), None, None)
    n, runs, _, stuck = (int(v) for v in N(tot))
    assert stuck == 0 and 0 < runs <= cap
    return dict(R=R, cap=cap, ws=ws, tot=tot, step=step, n=n, runs=runs, keep=(occ, o, d, a, tsrt, tidx, hits))


def _expand_samples(m, capacity, offsets=(0, 0)):
    """nfa_expand_samples into sentinel-filled allocations of n + GUARD (+ offset) elements; the views start
    `offsets` = (float elements, int64 elements) into them.  Returns (packed_info, the three allocations, views)."""
    from nerfacc_b200 import _lib
    n, fo, io = m["n"], offsets[0], offsets[1]
    ts_buf = torch.full((n + GUARD + fo,), F_SENT, device=dev)
    te_buf = torch.full((n + GUARD + fo,), F_SENT, device=dev)
    ri_buf = torch.full((n + GUARD + io,), I_SENT, dtype=torch.int64, device=dev)
    pi = torch.full((m["R"], 2), I_SENT, dtype=torch.int64, device=dev)
    ts, te, ri = ts_buf[fo:], te_buf[fo:], ri_buf[io:]
    _lib.call("nfa_expand_samples", torch.device(dev), m["R"], m["cap"], m["ws"].data_ptr(), m["tot"].data_ptr(),
              m["step"], capacity, pi.data_ptr(), ri.data_ptr(), ts.data_ptr(), te.data_ptr())
    torch.cuda.synchronize()
    return N(pi), (N(ri_buf), N(ts_buf), N(te_buf)), (N(ri), N(ts), N(te))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["frag1", "comb4"])
def test_expand_samples_clipped_and_unaligned(orc, name):
    """nfa_expand_samples with capacity n - k (the speculative call whose batch outgrew the hint): the first
    `capacity` elements are the full result, nothing at or past `capacity` is written, packed_info is complete.
    With outputs 4 / 8 bytes off 16-byte alignment (scalar kernel + offsets pass) the result is byte-identical."""
    bins, aabbs, ro, rd, step, far = scene(name)
    m = _march_abi(name)
    n = m["n"]
    o_ri, o_ts, o_te, o_pi = orc.occgrid_sampling(ro, rd, bins, aabbs, render_step_size=step, far_plane=far)
    pi, _, (ri, ts, te) = _expand_samples(m, n)
    ri, ts, te = ri[:n], ts[:n], te[:n]
    np.testing.assert_array_equal(pi, o_pi)
    np.testing.assert_array_equal(ri, o_ri)
    np.testing.assert_array_equal(ts, o_ts)
    np.testing.assert_array_equal(te, o_te)
    full = (ri, ts, te)
    for offsets in ((0, 0), (1, 1), (2, 1), (1, 0)):        # 4- / 8-byte offsets: the scalar kernel
        for k in (0, 1, 3, 4, 5, n // 2):
            cap = n - k
            pk, bufs, views = _expand_samples(m, cap, offsets)
            msg = f"offsets={offsets} capacity=n-{k}"
            np.testing.assert_array_equal(pk, pi, err_msg=msg)
            for got, want, buf, off, sent in zip(views, full, bufs, (offsets[1], offsets[0], offsets[0]),
                                                 (I_SENT, F_SENT, F_SENT)):
                assert got[:cap].tobytes() == want[:cap].tobytes(), msg
                assert (got[cap:] == sent).all(), f"{msg}: written at or past the capacity"
                assert (buf[:off] == sent).all(), f"{msg}: written before the output"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["frag1", "comb4"])
def test_expand_intervals_clipped(orc, name):
    """nfa_expand_intervals with edge_capacity / sample_capacity below the totals: the kept prefix of every array is
    the full result, nothing past a capacity is written, both packed_info arrays are complete; the full result is
    the oracle's traverse_grids."""
    from nerfacc_b200 import _lib
    m = _march_abi(name)
    bins, aabbs, ro, rd, step, far = scene(name)
    R, n, runs = m["R"], m["n"], m["runs"]
    e = n + runs

    def run(ecap, scap):
        fl = lambda k: torch.full((k + GUARD,), F_SENT, device=dev)
        il = lambda k: torch.full((k + GUARD,), I_SENT, dtype=torch.int64, device=dev)
        bl = lambda k: torch.full((k + GUARD,), B_SENT, dtype=torch.uint8, device=dev)
        out = dict(iv_pi=torch.full((R, 2), I_SENT, dtype=torch.int64, device=dev), iv_vals=fl(e), iv_ray=il(e),
                   iv_left=bl(e), iv_right=bl(e), sm_pi=torch.full((R, 2), I_SENT, dtype=torch.int64, device=dev),
                   sm_vals=fl(n), sm_ray=il(n), sm_valid=bl(n))
        _lib.call("nfa_expand_intervals", torch.device(dev), R, m["cap"], m["ws"].data_ptr(), m["tot"].data_ptr(), step,
                  ecap, scap, *[out[k].data_ptr() for k in ("iv_pi", "iv_vals", "iv_ray", "iv_left", "iv_right",
                                                            "sm_pi", "sm_vals", "sm_ray", "sm_valid")])
        torch.cuda.synchronize()
        return {k: N(v) for k, v in out.items()}

    full = run(e, n)
    o_iv, o_sm, _ = orc.traverse_grids(ro, rd, bins, aabbs, near_planes=np.zeros(R, np.float32),
                                       far_planes=np.full(R, far, np.float32), step_size=step)
    np.testing.assert_array_equal(full["iv_pi"], o_iv["packed_info"])
    np.testing.assert_array_equal(full["iv_vals"][:e], o_iv["vals"])
    np.testing.assert_array_equal(full["iv_ray"][:e], o_iv["ray_indices"])
    np.testing.assert_array_equal(full["iv_left"][:e], o_iv["is_left"])
    np.testing.assert_array_equal(full["iv_right"][:e], o_iv["is_right"])
    np.testing.assert_array_equal(full["sm_pi"], o_sm["packed_info"])
    np.testing.assert_array_equal(full["sm_vals"][:n], o_sm["vals"])
    np.testing.assert_array_equal(full["sm_ray"][:n], o_sm["ray_indices"])
    assert (full["sm_valid"][:n] == 1).all()
    for k in (1, 3, 4, 5, n // 2):
        got = run(e - k, n - k)
        for key in ("iv_pi", "sm_pi"):
            np.testing.assert_array_equal(got[key], full[key], err_msg=f"{key} k={k}")
        for key, cap, sent in (("iv_vals", e - k, F_SENT), ("iv_ray", e - k, I_SENT), ("iv_left", e - k, B_SENT),
                               ("iv_right", e - k, B_SENT), ("sm_vals", n - k, F_SENT), ("sm_ray", n - k, I_SENT),
                               ("sm_valid", n - k, B_SENT)):
            assert got[key][:cap].tobytes() == full[key][:cap].tobytes(), f"{key} k={k}"
            assert (got[key][cap:] == sent).all(), f"{key} k={k}: written at or past the capacity"


@pytest.mark.gpu
def test_speculative_expand_outgrown_and_oversized_hint(orc):
    """sampling() queues the expand before its one sync, sized by the previous call: a batch with more than twice
    the samples (hint < n: the clipped expand is discarded and redone), then a tiny one (hint >> n: the buffers are
    shrunk in place).  Each is the oracle's."""
    bins, aabbs, ro, rd, step, far = scene("frag1")
    est = _estimator(bins, aabbs)
    iv, sm, _ = _oracle(orc, "frag1")
    o_ts, o_te = iv["vals"][iv["is_left"]], iv["vals"][iv["is_right"]]
    for i, idx in enumerate((np.arange(1500), _batch(ro.shape[0], 9000, seed=4), np.arange(100, 140))):
        pi, src, ray = _gather(sm["packed_info"], idx)
        hint = est._capacity_hint
        if i == 1:
            assert 0 < hint < len(src) // 2
        if i == 2:
            assert hint > 100 * len(src)
        ri, ts, te = est.sampling(T(ro[idx]), T(rd[idx]), render_step_size=step)
        np.testing.assert_array_equal(N(ri), ray)
        np.testing.assert_array_equal(N(ts), o_ts[src])
        np.testing.assert_array_equal(N(te), o_te[src])


# ---------------------------------------------------------------- compositing past the resident-warp count

COMPOSITE_R = 32_768


def _ragged(R, seed):
    rng = np.random.default_rng(seed)
    cnts = rng.integers(0, 80, R)
    special = np.array([0, 1, 3, 4, 5, 31, 32, 33, 127, 128, 129, 250])
    cnts[rng.choice(R, 4 * special.size, replace=False)] = np.tile(special, 4)
    return torch.from_numpy(cnts.astype(np.int64))


def _alpha_grad_f64(alphas, pi, rgb, mids, gC, gO, gD, gW):
    """float64 torch autograd of the alpha route's loss, all rays at once on a zero-padded [R, max count] matrix
    (the formulation of test_vector_and_scalar_kernels_agree)."""
    starts, cnts = pi[:, 0], pi[:, 1]
    R, S = cnts.shape[0], int(cnts.max())
    col = torch.arange(S, device=dev)[None, :]
    valid = col < cnts[:, None]
    src = (starts[:, None] + col).clamp(max=alphas.shape[0] - 1)
    a64 = alphas.detach().double().requires_grad_(True)
    a = torch.where(valid, a64[src], 0.0)
    Tm = torch.cumprod(torch.cat([a.new_ones(R, 1), 1 - a[:, :-1]], 1), 1)
    w = Tm * a
    g = lambda x: torch.where(valid, x.double()[src], 0.0)
    O = w.sum(1)
    loss = (w[..., None] * torch.where(valid[..., None], rgb.detach().double()[src], 0.0) * gC.double()[:, None, :]).sum() \
        + (O * gO[:, 0].double()).sum() + ((w * g(mids)).sum(1) / O.clamp_min(1.1920929e-07) * gD[:, 0].double()).sum() \
        + (w * g(gW)).sum()
    loss.backward()
    return a64.grad


@pytest.mark.gpu
def test_compositing_tiers_past_resident_warps(orc):
    """One warp per ray in a persistent grid capped at the resident CTAs: with more rays than 64 warps per SM, every
    warp takes a second ray.  Each kernel tier at that size -- hot (density, every output), vec (alpha route, density
    with prefix_trans, gradients on weights / trans / alphas), scalar (4-byte-offset views, both routes) -- vs the
    float64 oracle at the bars of the small-batch tests."""
    import nerfacc_b200 as nfa
    from nerfacc_b200 import _lib
    R = COMPOSITE_R
    assert R > torch.cuda.get_device_properties(0).multi_processor_count * 64
    cnts = _ragged(R, 12)
    starts = torch.cumsum(cnts, 0) - cnts
    pi = torch.stack([starts, cnts], -1).to(dev)
    n = int(cnts.sum())
    g = torch.Generator().manual_seed(13)
    ri = torch.repeat_interleave(torch.arange(R), cnts).to(dev)
    gC, gO, gD = (torch.rand(sh, generator=g).to(dev) for sh in [(R, 3), (R, 1), (R, 1)])
    gW, gT, gA = (torch.rand(n, generator=g).to(dev) for _ in range(3))
    ts0 = torch.rand(n, generator=g).to(dev) * 0.5
    te0 = ts0 + 0.01 + torch.rand(n, generator=g).to(dev) * 0.02
    sig0 = 8 * torch.rand(n, generator=g).to(dev)
    rgb0 = torch.rand(n, 3, generator=g).to(dev)
    pt0 = 0.5 + 0.5 * torch.rand(n, generator=g).to(dev)
    npi = N(pi)

    def place(t, off):  # a copy whose storage starts `off` float32 elements into its buffer
        buf = torch.empty((t.shape[0] + off,) + tuple(t.shape[1:]), device=dev)
        buf[off:].copy_(t)
        return buf[off:]

    launches = _lib.launches
    # hot: density route, every output; gradients on colours / opacities / depths only
    sig, rgb = sig0.clone().requires_grad_(True), rgb0.clone().requires_grad_(True)
    col, op, dep, ex = nfa.rendering(ts0, te0, ri, n_rays=R, rgb_sigma_fn=lambda a, b, c: (rgb, sig))
    ((col * gC).sum() + (op * gO).sum() + (dep * gD).sum()).backward()
    o = orc.composite(N(ts0), N(te0), N(sig0), N(rgb0), packed_info=npi)
    for got, key in [(ex["weights"], "weights"), (ex["trans"], "trans"), (ex["alphas"], "alphas"), (col, "colors"),
                     (op, "opacities"), (dep, "depths")]:
        np.testing.assert_allclose(N(got), o[key], atol=1e-5, rtol=0, err_msg=f"hot {key}")
    gs, gr = orc.composite_backward(N(ts0), N(te0), N(sig0), N(rgb0), npi, gC=N(gC), gO=N(gO).ravel(), gD=N(gD).ravel())
    np.testing.assert_allclose(N(sig.grad), gs, atol=1e-5, rtol=1e-4, err_msg="hot g_sigmas")
    np.testing.assert_allclose(N(rgb.grad), gr, atol=1e-5, rtol=1e-4, err_msg="hot g_rgbs")

    # vec: density with prefix_trans, gradients on weights / trans / alphas
    sig = sig0.clone().requires_grad_(True)
    w, tr, a = nfa.render_weight_from_density(ts0, te0, sig, packed_info=pi, prefix_trans=pt0)
    o = orc.composite(N(ts0), N(te0), N(sig0), None, packed_info=npi, prefix_trans=N(pt0))
    for got, key in [(w, "weights"), (tr, "trans"), (a, "alphas")]:
        np.testing.assert_allclose(N(got), o[key], atol=1e-5, rtol=0, err_msg=f"vec prefix_trans {key}")
    ((w * gW).sum() + (tr * gT).sum() + (a * gA).sum()).backward()
    gs, _ = orc.composite_backward(N(ts0), N(te0), N(sig0), None, npi, gW=N(gW), gT=N(gT), gA=N(gA), prefix_trans=N(pt0))
    np.testing.assert_allclose(N(sig.grad), gs, atol=1e-5, rtol=1e-4, err_msg="vec prefix_trans g_sigmas")

    # vec and scalar: the alpha route (and the density route on unaligned views), gradients on the extras too
    for off in (0, 1):
        ts, te = place(ts0, off), place(te0, off)
        assert (ts.data_ptr() % 16 != 0) == bool(off)
        for use_alpha in (True, False) if off else (True,):
            base = sig0 / 10.0 if use_alpha else sig0
            dens, rgb = place(base, off).requires_grad_(True), place(rgb0, off).requires_grad_(True)
            fn = lambda a_, b_, c_: (rgb, dens)
            col, op, dep, ex = nfa.rendering(ts, te, ri, n_rays=R, **({"rgb_alpha_fn": fn} if use_alpha else
                                                                       {"rgb_sigma_fn": fn}))
            ((col * gC).sum() + (op * gO).sum() + (dep * gD).sum() + (ex["weights"] * gW).sum()).backward()
            tag = f"{'alpha' if use_alpha else 'density'} off={off}"
            if use_alpha:
                ow, oT = orc.render_weight_from_alpha(N(base), packed_info=npi)
                np.testing.assert_allclose(N(ex["weights"]), ow, atol=1e-5, rtol=0, err_msg=tag)
                np.testing.assert_allclose(N(ex["trans"]), oT, atol=1e-5, rtol=0, err_msg=tag)
                want = _alpha_grad_f64(base, pi, rgb0, (ts0 + te0) / 2, gC, gO, gD, gW)
                np.testing.assert_allclose(N(dens.grad), N(want), atol=5e-5, rtol=1e-3, err_msg=tag)
            else:
                o = orc.composite(N(ts0), N(te0), N(base), N(rgb0), packed_info=npi)
                for got, key in [(ex["weights"], "weights"), (ex["trans"], "trans"), (col, "colors"),
                                 (op, "opacities"), (dep, "depths")]:
                    np.testing.assert_allclose(N(got), o[key], atol=1e-5, rtol=0, err_msg=f"{tag} {key}")
                gs, gr = orc.composite_backward(N(ts0), N(te0), N(base), N(rgb0), npi, gC=N(gC), gO=N(gO).ravel(),
                                                gD=N(gD).ravel(), gW=N(gW))
                np.testing.assert_allclose(N(dens.grad), gs, atol=2e-5, rtol=1e-4, err_msg=tag)
                np.testing.assert_allclose(N(rgb.grad), gr, atol=1e-5, rtol=1e-4, err_msg=tag)
    assert _lib.launches - launches >= 10   # every route above went through the native kernels
