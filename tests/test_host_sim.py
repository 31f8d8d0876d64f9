"""CPU checks of the product's host+device traversal headers (lattice.cuh / march.cuh /
expand.cuh / occ_pack.cuh, compiled for the host by tests/host_sim) against
(a) serial float chains and (b) the oracle's restatement of the reference kernel."""
import ctypes as C

import numpy as np
import pytest

from nerfacc_b200 import scenes

F = C.POINTER(C.c_float)
U32 = C.POINTER(C.c_uint32)
I64 = C.POINTER(C.c_int64)
U8 = C.POINTER(C.c_uint8)
U64 = C.POINTER(C.c_uint64)
I32 = C.POINTER(C.c_int32)

STEPS = [1e-3, 5e-3, 5.2e-3, 0.01, 2 ** -8, 3 * 2 ** -10, 1.5 * 2 ** -7, 0.0123456, 1e-2 / 3, 0.25, 0.7]


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _seek_serial(t0, dt, target):
    t, dt, target = np.float32(t0), np.float32(dt), np.float32(target)
    h = np.float32(dt * np.float32(0.5))
    k = 0
    while not (np.float32(t + h) >= target):
        t = np.float32(t + dt)
        k += 1
    return float(t), k


@pytest.mark.parametrize("dt", STEPS)
def test_lattice_seek_matches_serial_chain(host_sim, dt):
    rng = np.random.default_rng(int(dt * 1e7))
    for _ in range(200):
        t0 = float(np.float32(rng.choice([0.0, rng.random() * dt * 4, rng.random() * 0.1, rng.random() * 5,
                                          rng.random() * 40, -rng.random() * 0.05])))
        target = float(np.float32(t0 + rng.random() * rng.choice([0.01, 0.1, 1, 6])))
        t, k = C.c_float(), C.c_uint32()
        ok = host_sim.sim_seek(t0, dt, target, C.byref(t), C.byref(k))
        ts, ks = _seek_serial(t0, dt, target)
        assert ok == 1 and np.float32(t.value) == np.float32(ts) and k.value == ks, (dt, t0, target)


@pytest.mark.parametrize("dt", STEPS)
def test_run_expansion_matches_serial_chain(host_sim, dt):
    rng = np.random.default_rng(int(dt * 1e7) + 1)
    for _ in range(40):
        t0 = float(np.float32(rng.choice([0.0, rng.random() * dt * 4, rng.random() * 5, rng.random() * 40,
                                          1.99, 3.999, 7.9995])))
        n = int(rng.integers(1, 700))
        s, e = np.empty(n, np.float32), np.empty(n, np.float32)
        host_sim.sim_expand_run(t0, dt, n, _p(s, F), _p(e, F))
        t, d = np.float32(t0), np.float32(dt)
        ref = np.empty(n, np.float32)
        for i in range(n):
            ref[i] = t
            t = np.float32(t + d)
        np.testing.assert_array_equal(s, ref)
        np.testing.assert_array_equal(e[:-1], s[1:])
        assert e[-1] == t


def test_stuck_lattice_is_reported(host_sim):
    # dt far below ulp(t)/2: the reference would spin forever; we report it
    t, k = C.c_float(), C.c_uint32()
    assert host_sim.sim_seek(1.0e6, 1e-3, 2.0e6, C.byref(t), C.byref(k)) == 0


def _sim_sampling(sim, ro, rd, bins, aabbs, near, far, step, multi=None, accel=0):
    G, rx, ry, rz = bins.shape
    R = ro.shape[0]
    words = np.zeros(sim.sim_occ_words(G, rx, ry, rz), np.uint64)
    coarse = np.zeros(sim.sim_occ_coarse_words(G, rx, ry, rz), np.uint32)
    b8 = np.ascontiguousarray(bins.astype(np.uint8))
    bounds = np.zeros(6 * G, np.int32)
    sim.sim_occ_pack(G, rx, ry, rz, _p(b8, U8), _p(words, U64), _p(coarse, U32), _p(bounds, I32))
    ns, nr = np.zeros(R, np.int64), np.zeros(R, np.int64)
    term, ok = np.zeros(R, np.float32), np.zeros(R, np.int32)
    cap = 2_000_000
    rt, rn = np.zeros(cap, np.float32), np.zeros(cap, np.uint32)
    ts_, ti_, hits_ = (None, None, None) if multi is None else multi
    tot = sim.sim_march(R, _p(ro, F), _p(rd, F), _p(near, F), _p(far, F), G, rx, ry, rz, _p(words, U64), _p(coarse, U32),
                        _p(bounds, I32), C.c_int(accel), _p(aabbs, F), _p(ts_, F), _p(ti_, I64), _p(hits_, U8), C.c_float(step), _p(ns, I64), _p(nr, I64),
                        _p(term, F), _p(ok, I32), _p(rt, F), _p(rn, U32), C.c_int64(cap))
    assert tot >= 0
    N = int(ns.sum())
    s, e, ri = np.empty(N, np.float32), np.empty(N, np.float32), np.empty(N, np.int64)
    w = q = 0
    for r in range(R):
        for _ in range(nr[r]):
            n = int(rn[q])
            sim.sim_expand_run(float(rt[q]), step, n, s[w:].ctypes.data_as(F), e[w:].ctypes.data_as(F))
            ri[w:w + n] = r
            w += n
            q += 1
    assert w == N
    return ri, s, e, ns, nr, term, ok


def _compare(sim, orc, ro, rd, bins, aabbs, near, far, step, multi=False, accel=0):
    iv, sm, term_o = orc.traverse_grids(ro, rd, bins, aabbs, near_planes=near, far_planes=far, step_size=step)
    m = None
    if multi:
        tm, tM, h = orc.ray_aabb_intersect(ro, rd, aabbs)
        tsrt, tidx = orc.sort_intersections(tm, tM)
        m = (tsrt, tidx, np.ascontiguousarray(h.astype(np.uint8)))
    ri, s, e, ns, nr, term, ok = _sim_sampling(sim, ro, rd, bins, aabbs, near, far, step, m, accel)
    assert ok.all()
    np.testing.assert_array_equal(ns, sm["packed_info"][:, 1])
    np.testing.assert_array_equal(nr, iv["packed_info"][:, 1] - sm["packed_info"][:, 1])  # runs = edges - samples
    np.testing.assert_array_equal(ri, sm["ray_indices"])
    np.testing.assert_array_equal(s, iv["vals"][iv["is_left"]])
    np.testing.assert_array_equal(e, iv["vals"][iv["is_right"]])
    if not accel:  # the accelerated walk stops early: terminate planes are not produced
        d = ~np.isnan(term_o)
        np.testing.assert_array_equal(term[d], term_o[d])
    return len(ri)


def test_march_ball_scene(host_sim, orc):
    R = 2048
    ro, rd = scenes.ball_rays(R)
    bins, aabbs = scenes.ball_grid(128), scenes.nested_aabbs(1)
    near, far = np.zeros(R, np.float32), np.full(R, 1e10, np.float32)
    n = _compare(host_sim, orc, ro, rd, bins, aabbs, near, far, scenes.BALL_STEP)
    assert 122 <= n / R <= 134  # SURVEY 8d calibration window
    rng = np.random.default_rng(7)
    _compare(host_sim, orc, ro, rd, bins, aabbs, (rng.random(R) * scenes.BALL_STEP).astype(np.float32), far, scenes.BALL_STEP)
    _compare(host_sim, orc, ro[:256], rd[:256], bins, aabbs, near[:256], far[:256], 1e-3)
    frag = bins & (rng.random(bins.shape) > 0.5)
    _compare(host_sim, orc, ro[:512], rd[:512], frag, aabbs, near[:512], far[:512], scenes.BALL_STEP)
    # empty-space acceleration (jump to / stop at the bounding box of the occupied bricks)
    _compare(host_sim, orc, ro, rd, bins, aabbs, near, far, scenes.BALL_STEP, accel=1)
    _compare(host_sim, orc, ro[:512], rd[:512], frag, aabbs, near[:512], far[:512], scenes.BALL_STEP, accel=1)
    off_centre = np.zeros((1, 128, 128, 128), bool)
    off_centre[0, 90:120, 5:9, 60:61] = True
    off_centre[0, 97, 100, 3] = True
    _compare(host_sim, orc, ro, rd, off_centre, aabbs, near, far, 3e-3, accel=1)
    _compare(host_sim, orc, ro, rd, off_centre, aabbs, (rng.random(R) * 4).astype(np.float32),
             (3 + rng.random(R) * 3).astype(np.float32), 3e-3, accel=1)


def test_march_nested_random_grids(host_sim, orc):
    rng = np.random.default_rng(11)
    R = 200
    ro = rng.standard_normal((R, 3)).astype(np.float32)
    rd = rng.standard_normal((R, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    bins4 = rng.random((4, 32, 32, 32)) > 0.5
    a4 = scenes.nested_aabbs(4)
    zero, inf = np.zeros(R, np.float32), np.full(R, np.inf, np.float32)
    _compare(host_sim, orc, ro, rd, bins4, a4, zero, inf, 2e-3, multi=True)
    _compare(host_sim, orc, ro, rd, bins4, a4, rng.random(R).astype(np.float32), (1 + rng.random(R) * 3).astype(np.float32),
             1e-2, multi=True)
    # single level: crossings computed inline vs supplied sorted arrays
    _compare(host_sim, orc, ro, rd, bins4[:1], a4[:1], zero, inf, 3e-3)
    _compare(host_sim, orc, ro, rd, bins4[:1], a4[:1], zero, inf, 3e-3, accel=1)
    _compare(host_sim, orc, ro, rd, odd_single := (rng.random((1, 30, 17, 5)) > 0.7), a4[:1], zero, inf, 4e-3, accel=1)
    _compare(host_sim, orc, ro, rd, bins4[:1], a4[:1], zero, inf, 3e-3, multi=True)
    # resolution not a multiple of the brick size, non-cubic
    odd = rng.random((2, 30, 17, 5)) > 0.3
    _compare(host_sim, orc, ro, rd, odd, a4[:2], zero, inf, 4e-3, multi=True)


def test_march_degenerate_rays(host_sim, orc):
    rng = np.random.default_rng(3)
    bins4 = rng.random((4, 32, 32, 32)) > 0.5
    a4 = scenes.nested_aabbs(4)
    ro = np.array([[-2, 0.1, 0.2], [0.3, -3, 0.1], [0.01, 0.02, 5], [0, 0, 0], [9, 9, 9], [0.5, 0.5, 0.5]], np.float32)
    rd = np.array([[1, 0, 0], [0, 1, 0], [0, 0, -1], [0, 0, 1], [1, 0, 0], [-0.6, 0.8, 0]], np.float32)
    R = len(ro)
    _compare(host_sim, orc, ro, rd, bins4, a4, np.zeros(R, np.float32), np.full(R, np.inf, np.float32), 1e-2, multi=True)
    # 1x1x1 grid, near/far inside the box (reference tests/test_grid.py:135-159)
    d = np.array([[1.0, 0.01, 0.01]])
    d = (d / np.linalg.norm(d)).astype(np.float32)
    _compare(host_sim, orc, np.array([[-1.0, 0, 0]], np.float32), d, np.ones((1, 1, 1, 1), bool),
             np.array([[0, 0, 0, 1, 1, 1]], np.float32), np.array([1.2], np.float32), np.array([1.5], np.float32), 0.05)
    # empty grid and empty ray batch
    e = np.zeros((1, 8, 8, 8), bool)
    assert _compare(host_sim, orc, ro, rd, e, a4[:1], np.zeros(R, np.float32), np.full(R, np.inf, np.float32), 1e-2) == 0
    assert _compare(host_sim, orc, ro, rd, e, a4[:1], np.zeros(R, np.float32), np.full(R, np.inf, np.float32), 1e-2, accel=1) == 0
    _compare(host_sim, orc, ro, rd, bins4[:1], a4[:1], np.zeros(R, np.float32), np.full(R, np.inf, np.float32), 1e-2, accel=1)


def test_march_matches_reference_cuda_goldens(host_sim):
    from conftest import golden_bins, load_golden
    for name in ["ref_sampling_ball", "ref_sampling_frag"]:
        z = load_golden(name)
        R = z["rays_o"].shape[0]
        step = float(z["kw_vals"][0])
        ri, s, e, ns, nr, term, ok = _sim_sampling(host_sim, z["rays_o"], z["rays_d"], golden_bins(z), z["aabbs"],
                                                   np.zeros(R, np.float32), np.full(R, 1e10, np.float32), step, accel=1)
        np.testing.assert_array_equal(ns, z["packed_info"][:, 1])
        np.testing.assert_array_equal(s, z["t_starts"])
        np.testing.assert_array_equal(e, z["t_ends"])


# ---------------------------------------------------------------- generic marcher (march_generic.cuh)

def _sim_generic(sim, ro, rd, bins, aabbs, near, far, step, cone, limit=-1, over_allocate=False, mask=None, orc=None):
    G, rx, ry, rz = bins.shape
    R = ro.shape[0]
    words = np.zeros(sim.sim_occ_words(G, rx, ry, rz), np.uint64)
    coarse = np.zeros(sim.sim_occ_coarse_words(G, rx, ry, rz), np.uint32)
    bounds = np.zeros(6 * G, np.int32)
    b8 = np.ascontiguousarray(bins.astype(np.uint8))
    sim.sim_occ_pack(G, rx, ry, rz, _p(b8, U8), _p(words, U64), _p(coarse, U32), _p(bounds, I32))
    tm, tM, h = orc.ray_aabb_intersect(ro, rd, aabbs)
    tsrt, tidx = orc.sort_intersections(tm, tM)
    hits = np.ascontiguousarray(h.astype(np.uint8))
    iv_cnts, sm_cnts = np.zeros(R, np.int64), np.zeros(R, np.int64)
    term = np.full(R, np.nan, np.float32)
    m8 = None if mask is None else np.ascontiguousarray(mask.astype(np.uint8))

    def run(fill, use_mask, iv_s, sm_s, arrs):
        sim.sim_generic_pass(R, _p(ro, F), _p(rd, F), _p(m8 if use_mask else None, U8), _p(near, F), _p(far, F), G, rx, ry, rz,
                             _p(words, U64), _p(coarse, U32), _p(aabbs, F), _p(tsrt, F), _p(tidx, I64), _p(hits, U8),
                             C.c_float(step), C.c_float(cone), C.c_int32(limit), C.c_int32(fill),
                             _p(iv_s, I64), _p(iv_cnts, I64), *[_p(a, t) for a, t in arrs[:4]],
                             _p(sm_s, I64), _p(sm_cnts, I64), *[_p(a, t) for a, t in arrs[4:]], _p(term if fill else None, F))

    if over_allocate:
        mm = np.ones(R, np.int64) if mask is None else mask.astype(np.int64)
        iv_cnts[:] = 2 * limit * mm
        sm_cnts[:] = limit * mm
    else:
        run(0, False, None, None, [(None, F), (None, I64), (None, U8), (None, U8), (None, F), (None, I64), (None, U8)])
    iv_s = (np.cumsum(iv_cnts) - iv_cnts).astype(np.int64)
    sm_s = (np.cumsum(sm_cnts) - sm_cnts).astype(np.int64)
    ne, ns = int(iv_cnts.sum()), int(sm_cnts.sum())
    iv_vals, iv_ray = np.zeros(ne, np.float32), np.zeros(ne, np.int64)
    iv_l, iv_r = np.zeros(ne, np.uint8), np.zeros(ne, np.uint8)
    sm_vals, sm_ray, sm_valid = np.zeros(ns, np.float32), np.zeros(ns, np.int64), np.zeros(ns, np.uint8)
    run(1, over_allocate, iv_s, sm_s, [(iv_vals, F), (iv_ray, I64), (iv_l, U8), (iv_r, U8), (sm_vals, F), (sm_ray, I64), (sm_valid, U8)])
    return dict(iv_vals=iv_vals, iv_ray=iv_ray, iv_left=iv_l.astype(bool), iv_right=iv_r.astype(bool), iv_cnts=iv_cnts.copy(),
                sm_vals=sm_vals, sm_ray=sm_ray, sm_valid=sm_valid.astype(bool), sm_cnts=sm_cnts.copy(), term=term)


def _check_generic(sim, orc, ro, rd, bins, aabbs, near, far, step, cone, **kw):
    mine = _sim_generic(sim, ro, rd, bins, aabbs, near, far, step, cone, orc=orc, **kw)
    iv, sm, term = orc.traverse_grids(ro, rd, bins, aabbs, near_planes=near, far_planes=far, step_size=step, cone_angle=cone,
                                      traverse_steps_limit=kw.get("limit", -1) if kw.get("limit", -1) > 0 else None,
                                      over_allocate=kw.get("over_allocate", False), rays_mask=kw.get("mask"))
    np.testing.assert_array_equal(mine["iv_cnts"], iv["packed_info"][:, 1])
    np.testing.assert_array_equal(mine["sm_cnts"], sm["packed_info"][:, 1])
    np.testing.assert_array_equal(mine["iv_vals"], iv["vals"])
    np.testing.assert_array_equal(mine["iv_left"], iv["is_left"])
    np.testing.assert_array_equal(mine["iv_right"], iv["is_right"])
    np.testing.assert_array_equal(mine["iv_ray"], iv["ray_indices"])
    np.testing.assert_array_equal(mine["sm_vals"], sm["vals"])
    np.testing.assert_array_equal(mine["sm_valid"], sm["is_valid"])
    np.testing.assert_array_equal(mine["sm_ray"], sm["ray_indices"])
    d = ~np.isnan(term)
    np.testing.assert_array_equal(mine["term"][d], term[d])
    return int(mine["sm_cnts"].sum())


def test_generic_marcher_modes(host_sim, orc):
    rng = np.random.default_rng(21)
    R = 120
    ro = rng.standard_normal((R, 3)).astype(np.float32)
    rd = rng.standard_normal((R, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    bins4 = rng.random((4, 32, 32, 32)) > 0.5
    a4 = scenes.nested_aabbs(4)
    zero, inf = np.zeros(R, np.float32), np.full(R, np.inf, np.float32)
    assert _check_generic(host_sim, orc, ro, rd, bins4, a4, zero, inf, 1e-2, 0.0) > 0          # same as the fast path
    assert _check_generic(host_sim, orc, ro, rd, bins4, a4, zero, inf, 5e-3, 0.01) > 0         # cone angle
    assert _check_generic(host_sim, orc, ro, rd, bins4, a4, (rng.random(R)).astype(np.float32),
                          (2 + rng.random(R)).astype(np.float32), 1e-2, 0.004) > 0
    assert _check_generic(host_sim, orc, ro, rd, bins4, a4, zero, inf, 0.0, 0.0) > 0           # one sample per cell
    assert _check_generic(host_sim, orc, ro, rd, bins4[:1], a4[:1], zero, inf, -1.0, 0.0) > 0
    # bounded marching into fixed-stride slots, with a ray mask (reference examples/utils.py:356-375)
    mask = rng.random(R) > 0.3
    assert _check_generic(host_sim, orc, ro, rd, bins4, a4, zero, inf, 1e-2, 0.0, limit=37, over_allocate=True, mask=mask) > 0
    assert _check_generic(host_sim, orc, ro, rd, bins4, a4, zero, inf, 1e-2, 0.003, limit=5, over_allocate=True) > 0
    # a limit without over-allocation (two-pass; the mask is ignored there, reference grid.cu:418,450)
    assert _check_generic(host_sim, orc, ro, rd, bins4, a4, zero, inf, 1e-2, 0.0, limit=50, mask=mask) > 0


# ---------------------------------------------------------------- grids of whole bricks, full grids

def test_march_brick_aligned_and_uniform_grids(host_sim, orc):
    """The walk against the oracle on the ball scene (with and without the empty-space jump), on grids made of whole
    4x4x4 bricks (all empty / all occupied) alone and mixed with random cells, on a non-cubic grid and on a grid with
    every cell occupied; one level and nested."""
    sim = host_sim
    R = 1024
    ro, rd = scenes.ball_rays(R)
    bins, aabbs = scenes.ball_grid(128), scenes.nested_aabbs(1)
    near, far = np.zeros(R, np.float32), np.full(R, 1e10, np.float32)
    _compare(sim, orc, ro, rd, bins, aabbs, near, far, scenes.BALL_STEP, accel=1)
    rng = np.random.default_rng(7)
    _compare(sim, orc, ro, rd, bins, aabbs, near, far, scenes.BALL_STEP)
    frag = bins & (rng.random(bins.shape) > 0.5)
    _compare(sim, orc, ro[:512], rd[:512], frag, aabbs, near[:512], far[:512], scenes.BALL_STEP, accel=1)
    ro2 = rng.standard_normal((200, 3)).astype(np.float32)
    rd2 = rng.standard_normal((200, 3)).astype(np.float32)
    rd2 /= np.linalg.norm(rd2, axis=1, keepdims=True)
    bins4 = rng.random((4, 32, 32, 32)) > 0.5
    blocks = np.kron(rng.random((4, 8, 8, 8)) > 0.5, np.ones((1, 4, 4, 4), bool))   # whole bricks on / off
    a4 = scenes.nested_aabbs(4)
    zero, inf = np.zeros(200, np.float32), np.full(200, np.inf, np.float32)
    for grid in (bins4, blocks, blocks & bins4):
        _compare(sim, orc, ro2, rd2, grid, a4, zero, inf, 2e-3, multi=True)
        _compare(sim, orc, ro2, rd2, grid[:1], a4[:1], zero, inf, 3e-3, accel=1)
    _compare(sim, orc, ro2, rd2, rng.random((2, 30, 17, 5)) > 0.3, a4[:2], zero, inf, 4e-3, multi=True)
    full = np.ones((1, 16, 16, 16), bool)
    _compare(sim, orc, ro2, rd2, full, a4[:1], zero, inf, 1e-2, accel=1)
    _compare(sim, orc, ro2, rd2, full, a4[:1], rng.random(200).astype(np.float32), (1 + rng.random(200) * 3).astype(np.float32), 1e-2)


def test_binade_table_seek_is_the_plain_seek(host_sim):
    """The march kernel starts a ray's first seek from a host-built table of lattice points at the binade starts
    (lattice.cuh: LatTable).  The point it arrives at must be the one the plain climb from `near` arrives at."""
    import ctypes as C
    sim = host_sim
    sim.sim_seek_with_table.argtypes = [C.c_float, C.c_float, C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    sim.sim_seek_with_table.restype = C.c_int
    rng = np.random.default_rng(5)
    a, b = C.c_float(), C.c_float()
    used = 0
    for _ in range(4000):
        dt = np.float32(10.0 ** rng.uniform(-4, 0.5))
        near = np.float32(0.0 if rng.random() < 0.5 else 10.0 ** rng.uniform(-3, 1))
        kind = rng.random()
        if kind < 0.6:
            target = np.float32(near + dt * rng.uniform(0, 3000))
        elif kind < 0.8:   # exactly at / next to a power of two
            e = int(rng.integers(-6, 8))
            target = np.nextafter(np.float32(2.0 ** e), np.float32(rng.choice([-1e9, 1e9]))) if rng.random() < 0.7 else np.float32(2.0 ** e)
        else:
            target = np.float32(10.0 ** rng.uniform(-5, 3))
        if target / dt > 3e5:
            continue   # keeps the plain climb short
        r = sim.sim_seek_with_table(dt, near, target, C.byref(a), C.byref(b))
        assert (r & 1) == ((r >> 1) & 1)
        if r & 1:
            assert np.float32(a.value).tobytes() == np.float32(b.value).tobytes(), (dt, near, target, a.value, b.value)
        used += (r >> 2) > 0
    assert used > 1000


# ---------------------------------------------------------------- phase 2 by stretch (one level)

def test_lattice_by_stretch_matches(host_sim, orc):
    """march_kernel deals the stretches of a warp's rays out to the lanes: each is turned into its run from the ray's
    anchor, independently of the ray's other stretches (march.cuh: lat_anchor / lat_stretch / lat_take).  accel=2 in
    the simulation takes that path (last stretch first) and the result must be the oracle's, bit for bit -- also over
    several buffer rounds, with per-ray near planes, and at step sizes where stretches hold no sample at all."""
    import ctypes as C
    sim = host_sim
    rng = np.random.default_rng(17)
    R = 2048
    ro, rd = scenes.ball_rays(R)
    bins, aabbs = scenes.ball_grid(128), scenes.nested_aabbs(1)
    near, far = np.zeros(R, np.float32), np.full(R, 1e10, np.float32)
    cnt = (C.c_long * 2)()
    sim.sim_by_stretch_counts(cnt, 1)
    _compare(sim, orc, ro, rd, bins, aabbs, near, far, scenes.BALL_STEP, accel=2)
    sim.sim_by_stretch_counts(cnt, 1)
    assert cnt[0] >= R and cnt[1] == R        # every ray took the by-stretch path, with a binade table
    _compare(sim, orc, ro, rd, bins, aabbs, (rng.random(R) * scenes.BALL_STEP).astype(np.float32), far, scenes.BALL_STEP, accel=2)
    frag = bins & (rng.random(bins.shape) > 0.5)  # many stretches: several rounds of the 8-slot buffer
    _compare(sim, orc, ro[:512], rd[:512], frag, aabbs, near[:512], far[:512], scenes.BALL_STEP, accel=2)
    _compare(sim, orc, ro[:512], rd[:512], frag, aabbs, near[:512], far[:512], 0.05, accel=2)   # step > cell: empty runs
    _compare(sim, orc, ro[:512], rd[:512], frag, aabbs, near[:512], far[:512], 0.3, accel=2)
    frag2 = bins & (rng.random(bins.shape) > 0.03)
    _compare(sim, orc, ro[:1024], rd[:1024], frag2, aabbs, near[:1024], far[:1024], scenes.BALL_STEP, accel=2)
    _compare(sim, orc, ro[:1024], rd[:1024], frag2, aabbs, near[:1024], far[:1024], 7e-4, accel=2)
    off_centre = np.zeros((1, 128, 128, 128), bool)
    off_centre[0, 90:120, 5:9, 60:61] = True
    off_centre[0, 97, 100, 3] = True
    _compare(sim, orc, ro, rd, off_centre, aabbs, near, far, 3e-3, accel=2)
    _compare(sim, orc, ro, rd, off_centre, aabbs, (rng.random(R) * 4).astype(np.float32),
             (3 + rng.random(R) * 3).astype(np.float32), 3e-3, accel=2)
    ro2 = rng.standard_normal((300, 3)).astype(np.float32)
    rd2 = rng.standard_normal((300, 3)).astype(np.float32)
    rd2 /= np.linalg.norm(rd2, axis=1, keepdims=True)
    zero, inf = np.zeros(300, np.float32), np.full(300, np.inf, np.float32)
    a1 = scenes.nested_aabbs(1)
    for grid in (rng.random((1, 32, 32, 32)) > 0.5, rng.random((1, 30, 17, 5)) > 0.7, np.ones((1, 16, 16, 16), bool),
                 np.kron(rng.random((1, 8, 8, 8)) > 0.5, np.ones((1, 4, 4, 4), bool))):
        _compare(sim, orc, ro2, rd2, grid, a1, zero, inf, 3e-3, accel=2)
        _compare(sim, orc, ro2, rd2, grid, a1, rng.random(300).astype(np.float32), (1 + rng.random(300) * 3).astype(np.float32), 1e-2, accel=2)
    # axis-aligned and other degenerate rays
    ro3 = np.array([[-2, 0.1, 0.2], [0.3, -3, 0.1], [0.01, 0.02, 5], [0, 0, 0], [9, 9, 9], [0.5, 0.5, 0.5]], np.float32)
    rd3 = np.array([[1, 0, 0], [0, 1, 0], [0, 0, -1], [0, 0, 1], [1, 0, 0], [-0.6, 0.8, 0]], np.float32)
    _compare(sim, orc, ro3, rd3, rng.random((1, 32, 32, 32)) > 0.5, a1, np.zeros(6, np.float32), np.full(6, np.inf, np.float32), 1e-2, accel=2)
