"""OccGridEstimator.render_test without a GPU: argument errors, the render_test entry points of the C ABI, and the
round march's sample sink (march_generic.cuh SampleSink, compiled for the host by tests/host_sim/sample_sink_sim.cpp)
against the fixed-stride interval sink of traverse_grids' test mode (tests/host_sim/host_sim.cpp), bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import nerfacc_b200 as nfa
from nerfacc_b200 import scenes
from test_host_sim import _sim_generic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = C.POINTER(C.c_float)
I64 = C.POINTER(C.c_int64)
U8 = C.POINTER(C.c_uint8)
U32 = C.POINTER(C.c_uint32)
U64 = C.POINTER(C.c_uint64)
I32 = C.POINTER(C.c_int32)

ENTRY_POINTS = ("nfa_render_test_workspace_bytes", "nfa_render_test_begin", "nfa_render_test_march",
                "nfa_render_test_expand", "nfa_render_test_composite", "nfa_render_test_finish")


def test_cpu_tensors_are_not_implemented():
    est = nfa.OccGridEstimator([-1.0, -1.0, -1.0, 1.0, 1.0, 1.0], resolution=16)
    fn = lambda ts, te, ri: (torch.zeros(ts.shape[0], 3), torch.zeros(ts.shape[0]))  # noqa: E731
    for step in (1e-2, 0.0):  # the native route and the loop over the public functions
        with pytest.raises(NotImplementedError):
            est.render_test(torch.zeros(4, 3), torch.ones(4, 3), fn, max_samples=16, render_step_size=step)
    assert "render_test" not in dir(nfa)  # a method of the estimator only: nothing new at the package level


def test_entry_points_and_argument_errors():
    from nerfacc_b200 import _lib
    lib = _lib.load()
    assert _lib.ABI_VERSION == 15 and lib.nfa_version() == 15
    for name in ENTRY_POINTS:
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    ws = lib.nfa_render_test_workspace_bytes
    assert ws(-1, 1) == 0 and ws(10, 0) == 0
    for R in (1, 33, 5000, 1 << 20):
        # lists, near planes, counts, offsets, ranks and min_samples x R fixed-stride sample pairs
        assert ws(R, 1) >= 6 * 4 * R + 8 * R and ws(R, 4) - ws(R, 1) >= 2 * 4 * 3 * R - 32
    # rejected before any pointer is read: every other pointer may be a dummy (non-null, 16-byte aligned) address
    P = 1 << 20

    def march(R=64, ms=1, rnd=0, step=1e-2, cone=0.0, words=P, status=P):
        return lib.nfa_render_test_march(R, ms, rnd, P, P, 1e10, 1, 32, 32, 32, words, P, P, P, P, P, step, cone, P,
                                         status, None)

    assert march(step=0.0) == -2 and march(step=-1.0) == -2  # one sample per cell: the public-function loop
    for bad in (dict(R=0), dict(ms=0), dict(rnd=-1), dict(cone=-0.1), dict(cone=float("nan")), dict(words=None),
                dict(status=None)):
        assert march(**bad) == -1, bad
    assert lib.nfa_render_test_begin(-1, 1, 0.0, P, None) == -1
    assert lib.nfa_render_test_begin(8, 1, 0.0, P + 4, None) == -1  # misaligned workspace
    assert lib.nfa_render_test_expand(8, 1, 0, 9, 1, P, P, P, P, None) == -1    # more live rays than rays
    assert lib.nfa_render_test_expand(8, 1, 0, 8, 2, P, P, P, P, None) == -1    # more slots than the workspace has
    assert lib.nfa_render_test_composite(8, 1, 0, 4, 65, 0, P, P, P, P, P, 0.0, 0.9999, P, P, P, None) == -1
    assert lib.nfa_render_test_composite(8, 1, 0, 4, 2, 9, P, P, P, P, P, 0.0, 0.9999, P, P, P, None) == -1
    assert lib.nfa_render_test_composite(8, 1, 0, 4, 2, 8, P, P, P, None, P, 0.0, 0.9999, P, P, P, None) == -1
    assert lib.nfa_render_test_finish(8, 1, None, None, P, P, P, None, None) == -1


@pytest.fixture(scope="module")
def sink_sim(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "host_sim", "sample_sink_sim.cpp")
    so = str(tmp_path_factory.mktemp("sample_sink_sim") / "libsample_sink_sim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                           "-Wno-unknown-pragmas", "-o", so, src])
    return C.CDLL(so)


def _sink_round(sim, host_sim, orc, ro, rd, bins, aabbs, near, step, cone, limit, mask):
    G, rx, ry, rz = bins.shape
    R = ro.shape[0]
    words = np.zeros(host_sim.sim_occ_words(G, rx, ry, rz), np.uint64)
    coarse = np.zeros(host_sim.sim_occ_coarse_words(G, rx, ry, rz), np.uint32)
    bounds = np.zeros(6 * G, np.int32)
    b8 = np.ascontiguousarray(bins.astype(np.uint8))
    host_sim.sim_occ_pack(G, rx, ry, rz, b8.ctypes.data_as(U8), words.ctypes.data_as(U64), coarse.ctypes.data_as(U32),
                          bounds.ctypes.data_as(I32))
    tm, tM, h = orc.ray_aabb_intersect(ro, rd, aabbs)
    tsrt, tidx = orc.sort_intersections(tm, tM)
    hits = np.ascontiguousarray(h.astype(np.uint8))
    m8 = np.ascontiguousarray(mask.astype(np.uint8))
    n_live = int(mask.sum())
    counts = np.zeros(n_live, np.int64)
    term = np.full(R, np.nan, np.float32)
    slot_ts = np.full(n_live * limit, np.nan, np.float32)
    slot_te = np.full(n_live * limit, np.nan, np.float32)
    p = lambda a, t: a.ctypes.data_as(t)  # noqa: E731
    k = sim.sim_sample_sink_round(R, p(ro, F), p(rd, F), p(m8, U8), p(near, F), C.c_float(np.inf), G, rx, ry, rz,
                                  p(words, U64), p(coarse, U32), p(aabbs, F), p(tsrt, F), p(tidx, I64), p(hits, U8),
                                  C.c_float(step), C.c_float(cone), C.c_int32(limit), p(counts, I64), p(term, F),
                                  p(slot_ts, F), p(slot_te, F))
    assert k == n_live
    keep = (np.arange(limit)[None, :] < counts[:, None]).reshape(-1)  # slot k's first counts[k] samples, in ray order
    ray_of_slot = np.repeat(np.flatnonzero(mask), limit)
    return counts, term, slot_ts[keep], slot_te[keep], ray_of_slot[keep]


def test_sample_sink_matches_the_fixed_stride_sink(host_sim, orc, sink_sim):
    """The host-sim scenes of test_host_sim.test_generic_marcher_modes (random 4-level grids, per-ray near planes,
    masks, step limits, cone angles) and the ball scene: the same counts, terminate planes and samples as
    traverse_grids(traverse_steps_limit, over_allocate=True, rays_mask) followed by vals[is_left] / vals[is_right] /
    ray_indices[is_valid]."""
    rng = np.random.default_rng(21)
    R = 120
    ro = rng.standard_normal((R, 3)).astype(np.float32)
    rd = rng.standard_normal((R, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    bins4 = rng.random((4, 32, 32, 32)) > 0.5
    a4 = scenes.nested_aabbs(4)
    zero = np.zeros(R, np.float32)
    bro, brd = scenes.ball_rays(R, seed=9)
    ball = scenes.ball_grid(64)
    cases = [
        (ro, rd, bins4, a4, zero, 1e-2, 0.0, 37, rng.random(R) > 0.3),
        (ro, rd, bins4, a4, zero, 1e-2, 0.003, 5, np.ones(R, bool)),
        (ro, rd, bins4, a4, rng.random(R).astype(np.float32), 1e-2, 0.004, 4, rng.random(R) > 0.5),
        (ro, rd, bins4[:1], a4[:1], zero, 5e-3, 0.0, 64, np.ones(R, bool)),
        (bro, brd, ball, scenes.nested_aabbs(1), zero, 5.2e-3, 0.0, 1, rng.random(R) > 0.2),
        (bro, brd, ball, scenes.nested_aabbs(1), np.full(R, 3.8, np.float32), 5.2e-3, 0.0, 17, np.ones(R, bool)),
    ]
    inf = np.full(R, np.inf, np.float32)
    n_total = 0
    for o, d, bins, aabbs, near, step, cone, limit, mask in cases:
        counts, term, ts, te, ri = _sink_round(sink_sim, host_sim, orc, o, d, bins, aabbs, near, step, cone, limit,
                                               mask)
        ref = _sim_generic(host_sim, o, d, bins, aabbs, near, inf, step, cone, limit=limit, over_allocate=True,
                           mask=mask, orc=orc)
        np.testing.assert_array_equal(counts, ref["sm_cnts"][mask])
        np.testing.assert_array_equal(term[mask], ref["term"][mask])
        np.testing.assert_array_equal(ts, ref["iv_vals"][ref["iv_left"]])
        np.testing.assert_array_equal(te, ref["iv_vals"][ref["iv_right"]])
        np.testing.assert_array_equal(ri, ref["sm_ray"][ref["sm_valid"]])
        n_total += len(ts)
        assert (counts == limit).any() or limit > 30  # the step limit is what stops some rays
    assert n_total > 1000
