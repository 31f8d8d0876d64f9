"""CPU checks of the growing-step sampling path (cone_angle > 0: march_generic.cuh's walk into a run sink, then
cone_expand_run replaying every run), compiled for the host by tests/host_sim/cone_sim.cpp, against the oracle's
restatement of the reference (occgrid_sampling: traverse_grids + vals[is_left] / vals[is_right]), bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from nerfacc_b200 import scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = C.POINTER(C.c_float)
I64 = C.POINTER(C.c_int64)
U8 = C.POINTER(C.c_uint8)


@pytest.fixture(scope="session")
def cone_sim(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "host_sim", "cone_sim.cpp")
    so = str(tmp_path_factory.mktemp("cone_sim") / "libcone_sim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                           "-Wno-unknown-pragmas", "-o", so, src])
    lib = C.CDLL(so)
    lib.sim_cone_sampling.restype = C.c_int64
    return lib


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _sim(sim, orc, ro, rd, bins, aabbs, near, far, near_s, far_s, step, cone, sorted_crossings):
    ro, rd = np.ascontiguousarray(ro, np.float32), np.ascontiguousarray(rd, np.float32)
    G, rx, ry, rz = bins.shape
    R = ro.shape[0]
    b8 = np.ascontiguousarray(bins.astype(np.uint8))
    aabbs = np.ascontiguousarray(aabbs, np.float32)
    ts_ = ti_ = h_ = None
    if sorted_crossings:
        tm, tM, h = orc.ray_aabb_intersect(ro, rd, aabbs)
        ts_, ti_ = orc.sort_intersections(tm, tM)
        h_ = np.ascontiguousarray(h.astype(np.uint8))
    pi, runs = np.zeros((R, 2), np.int64), np.zeros(R, np.int64)

    def call(cap, ri, s, e):
        return sim.sim_cone_sampling(R, _p(ro, F), _p(rd, F), _p(near, F), _p(far, F), C.c_float(near_s),
                                     C.c_float(far_s), G, rx, ry, rz, _p(b8, U8), _p(aabbs, F), _p(ts_, F), _p(ti_, I64),
                                     _p(h_, U8), C.c_float(step), C.c_float(cone), _p(pi, I64), _p(runs, I64),
                                     C.c_int64(cap), _p(ri, I64), _p(s, F), _p(e, F))

    n = call(0, None, None, None)
    ri, s, e = np.full(n, -1, np.int64), np.full(n, np.nan, np.float32), np.full(n, np.nan, np.float32)
    assert call(n, ri, s, e) == n
    return ri, s, e, pi, runs


def _check(sim, orc, ro, rd, bins, aabbs, step, cone, near_plane=0.0, far_plane=1e10, t_min=None, t_max=None,
           sorted_crossings=None):
    """sim vs oracle; per-ray planes when t_min / t_max are given, the two scalars otherwise.  Returns the sample
    count."""
    R = ro.shape[0]
    if sorted_crossings is None:
        sorted_crossings = bins.shape[0] > 1
    o_ri, o_ts, o_te, o_pi = orc.occgrid_sampling(ro, rd, bins, aabbs, near_plane=near_plane, far_plane=far_plane,
                                                  t_min=t_min, t_max=t_max, render_step_size=step, cone_angle=cone)
    near = far = None
    if t_min is not None or t_max is not None:
        near = np.full(R, near_plane, np.float32) if t_min is None else np.maximum(np.float32(near_plane), t_min)
        far = np.full(R, far_plane, np.float32) if t_max is None else np.minimum(np.float32(far_plane), t_max)
        near, far = near.astype(np.float32), far.astype(np.float32)
    ri, s, e, pi, runs = _sim(sim, orc, ro, rd, bins, aabbs, near, far, near_plane, far_plane, step, cone,
                              sorted_crossings)
    np.testing.assert_array_equal(pi, o_pi)
    np.testing.assert_array_equal(ri, o_ri)
    assert s.tobytes() == o_ts.tobytes() and e.tobytes() == o_te.tobytes()
    # runs = the reference's chains of continuous samples: edges - samples of traverse_grids' interval form
    near_a = np.full(R, near_plane, np.float32) if near is None else near
    far_a = np.full(R, far_plane, np.float32) if far is None else far
    iv, sm, _ = orc.traverse_grids(ro, rd, bins, aabbs, near_planes=near_a, far_planes=far_a, step_size=step,
                                   cone_angle=cone)
    np.testing.assert_array_equal(runs, iv["packed_info"][:, 1] - sm["packed_info"][:, 1])
    return len(ri)


def _random_rays(rng, R, scale=1.0):
    ro = (rng.standard_normal((R, 3)) * scale).astype(np.float32)
    rd = rng.standard_normal((R, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    return ro, rd


def _fragments(rng, levels, res, keep=0.5):
    """ref_runner.grid_for's layout: a ball at level 0, random fragments of shells further out."""
    out = [scenes.ball_grid(res)[0]]
    for _ in range(1, levels):
        shell = scenes.ball_grid(res, radius=0.8)[0] & ~scenes.ball_grid(res, radius=0.3)[0]
        out.append(shell & (rng.random((res, res, res)) > keep))
    return np.stack(out)


def test_cone_ball_one_level(cone_sim, orc):
    R = 1024
    ro, rd = scenes.ball_rays(R)
    bins, a1 = scenes.ball_grid(128), scenes.nested_aabbs(1)
    n = _check(cone_sim, orc, ro, rd, bins, a1, scenes.BALL_STEP, 0.01)
    assert n > 10 * R
    _check(cone_sim, orc, ro, rd, bins, a1, scenes.BALL_STEP, 0.01, sorted_crossings=True)  # crossings supplied
    frag = bins & (np.random.default_rng(1).random(bins.shape) > 0.5)  # many runs per ray
    _check(cone_sim, orc, ro[:256], rd[:256], frag, a1, 1e-3, 0.004, near_plane=0.2)


@pytest.mark.parametrize("res", [32, 128])
def test_cone_four_nested_levels_of_fragments(cone_sim, orc, res):
    """nerfacc's unbounded-scene setting (levels=4, step 1e-3, cone 0.004, near 0.2), origins inside the boxes."""
    rng = np.random.default_rng(res)
    bins, a4 = _fragments(rng, 4, res), scenes.nested_aabbs(4)
    R = 256 if res == 32 else 64
    ro, rd = scenes.ball_rays(R, seed=res)           # origins at distance 4: inside levels 2 and 3
    n = _check(cone_sim, orc, ro, rd, bins, a4, 1e-3, 0.004, near_plane=0.2)
    assert n > 0
    ro2, rd2 = _random_rays(rng, R, 1.5)             # anywhere, mostly inside level 1..3
    _check(cone_sim, orc, ro2, rd2, bins, a4, 1e-3, 0.004, near_plane=0.2)
    _check(cone_sim, orc, ro2, rd2, rng.random(bins.shape) > 0.5, a4, 1e-3, 0.004, near_plane=0.2)


def test_cone_per_ray_planes(cone_sim, orc):
    rng = np.random.default_rng(5)
    bins, a4 = rng.random((4, 32, 32, 32)) > 0.5, scenes.nested_aabbs(4)
    R = 200
    ro, rd = _random_rays(rng, R)
    t_min = rng.random(R).astype(np.float32)
    t_max = (t_min + 3 * rng.random(R)).astype(np.float32)
    assert _check(cone_sim, orc, ro, rd, bins, a4, 1e-2, 0.004, near_plane=0.15, far_plane=3.4, t_min=t_min,
                  t_max=t_max) > 0
    jitter = (0.2 + rng.random(R) * 1e-3).astype(np.float32)   # stratified near planes
    assert _check(cone_sim, orc, ro, rd, bins, a4, 1e-3, 0.004, t_min=jitter) > 0
    bins1, a1 = bins[:1], a4[:1]
    assert _check(cone_sim, orc, ro, rd, bins1, a1, 5e-3, 0.01, t_min=jitter, t_max=t_max) > 0


def test_cone_misses_empty_grid_and_degenerate_rays(cone_sim, orc):
    rng = np.random.default_rng(9)
    bins, a4 = rng.random((4, 32, 32, 32)) > 0.5, scenes.nested_aabbs(4)
    # rays that miss every box (from far away, pointing away), axis-aligned rays, a ray from the centre
    ro = np.array([[20, 20, 20], [-30, 0, 0], [-2, 0.1, 0.2], [0.3, -3, 0.1], [0.01, 0.02, 5], [0, 0, 0],
                   [9, 9, 9], [0.5, 0.5, 0.5]], np.float32)
    rd = np.array([[1, 0, 0], [-1, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, -1], [0, 0, 1], [1, 0, 0], [-0.6, 0.8, 0]],
                  np.float32)
    assert _check(cone_sim, orc, ro, rd, bins, a4, 1e-2, 0.004) > 0
    misses = _check(cone_sim, orc, ro[:2], rd[:2], bins, a4, 1e-2, 0.004)
    assert misses == 0
    empty = np.zeros((4, 32, 32, 32), bool)
    ro2, rd2 = _random_rays(rng, 100)
    assert _check(cone_sim, orc, ro2, rd2, empty, a4, 1e-3, 0.004, near_plane=0.2) == 0
    assert _check(cone_sim, orc, ro2, rd2, empty[:1], a4[:1], 1e-3, 0.004) == 0


def test_cone_constant_dt_region_and_its_end(cone_sim, orc):
    """dt = max(step, t * cone): rays that stay below t = step / cone march with the constant step, rays that cross it
    switch to the growing step inside a run."""
    step, cone = 1e-2, 0.004           # t = 2.5 is where the step starts to grow
    rng = np.random.default_rng(13)
    full, a4 = np.ones((4, 16, 16, 16), bool), scenes.nested_aabbs(4)
    R = 100
    ro, rd = _random_rays(rng, R, 0.3)
    below = np.full(R, 2.4, np.float32)
    assert _check(cone_sim, orc, ro, rd, full, a4, step, cone, far_plane=2.4) > 200 * R   # ~240 steps of 1e-2 each
    _check(cone_sim, orc, ro, rd, full, a4, step, cone, t_max=below)
    n_cross = _check(cone_sim, orc, ro, rd, full, a4, step, cone, near_plane=2.0, far_plane=6.0)
    assert n_cross > 0
    # the same with holes, so that runs end and start on both sides of t = 2.5
    holes = rng.random((4, 16, 16, 16)) > 0.3
    _check(cone_sim, orc, ro, rd, holes, a4, step, cone, near_plane=2.0, far_plane=6.0)
    _check(cone_sim, orc, ro, rd, holes[:1], a4[:1], step, cone, near_plane=0.5, far_plane=4.0)
