"""OccGridEstimator.sampling with growing steps (cone_angle > 0) on the GPU: nfa_march + nfa_expand_samples with
cone_angle > 0 (march_cone_kernel, expand_cone_kernel) behind sampling_begin / sampling_end.  Bit-exact against the
CPU oracle, against the traverse_grids route this path replaced (edge/flag form + mask-selects), and against the
reference CUDA build (tests/golden/ref_live_cone360.npz, oracle/gen_golden_cone_gpu.py)."""
import numpy as np
import pytest
import torch

import nerfacc_b200 as nfa
from nerfacc_b200 import scenes
from nerfacc_b200.grid import traverse_grids
from conftest import load_golden
from oracle.gen_golden_cone_gpu import CONE360, run_cone360
import ref_runner as rr

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def N(t):
    return t.detach().cpu().numpy()


def _estimator(bins, aabbs, occ_mean=0.3):
    est = nfa.OccGridEstimator(torch.from_numpy(aabbs[0]), resolution=list(bins.shape[1:]), levels=bins.shape[0]).to(dev)
    est.binaries = T(bins)
    est.occs.fill_(occ_mean)
    return est


def _old_route(est, rays_o, rays_d, sigma_fn=None, alpha_fn=None, near_plane=0.0, far_plane=1e10, t_min=None,
               t_max=None, render_step_size=1e-3, early_stop_eps=1e-4, alpha_thre=0.0, stratified=False,
               cone_angle=0.0):
    """What sampling(cone_angle > 0) ran before: traverse_grids' edge/flag form, two mask-selects, the filter."""
    near_planes, far_planes = est._ray_planes(rays_o, near_plane, far_plane, t_min, t_max, stratified,
                                              render_step_size, always=True)
    intervals, samples, _ = traverse_grids(rays_o, rays_d, est.binaries, est.aabbs, near_planes=near_planes,
                                           far_planes=far_planes, step_size=render_step_size, cone_angle=cone_angle)
    return est._drop_invisible(samples.ray_indices, intervals.vals[intervals.is_left],
                               intervals.vals[intervals.is_right], samples.packed_info, sigma_fn, alpha_fn,
                               early_stop_eps, alpha_thre)


def _same(got, want):
    for a, b in zip(got, want):
        assert a.dtype == b.dtype and a.shape == b.shape
        assert torch.equal(a, b)


def _fragments(rng, levels, res):
    out = [scenes.ball_grid(res)[0]]
    for _ in range(1, levels):
        shell = scenes.ball_grid(res, radius=0.8)[0] & ~scenes.ball_grid(res, radius=0.3)[0]
        out.append(shell & (rng.random((res, res, res)) > 0.5))
    return np.stack(out)


def _random_rays(rng, R, scale=1.0):
    ro = (rng.standard_normal((R, 3)) * scale).astype(np.float32)
    rd = rng.standard_normal((R, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    return ro, rd


def _scene(name):
    """(rays_o, rays_d, binaries, aabbs, sampling kwargs) of the oracle-parity scenes."""
    rng = np.random.default_rng(len(name))
    if name == "ball":
        ro, rd = scenes.ball_rays(4096)
        return ro, rd, scenes.ball_grid(128), scenes.nested_aabbs(1), dict(render_step_size=scenes.BALL_STEP,
                                                                            cone_angle=0.01)
    if name in ("lvl4_32", "lvl4_128"):
        res = 32 if name == "lvl4_32" else 128
        ro, rd = scenes.ball_rays(2048 if res == 32 else 256, seed=res)
        return ro, rd, _fragments(rng, 4, res), scenes.nested_aabbs(4), dict(render_step_size=1e-3, cone_angle=0.004,
                                                                              near_plane=0.2)
    if name == "inside":                       # origins anywhere inside the nested boxes
        ro, rd = _random_rays(rng, 1024, 1.5)
        return ro, rd, _fragments(rng, 4, 32), scenes.nested_aabbs(4), dict(render_step_size=1e-3, cone_angle=0.004,
                                                                             near_plane=0.2)
    if name == "planes":                       # per-ray near / far planes
        ro, rd = _random_rays(rng, 512)
        t_min = rng.random(512).astype(np.float32)
        t_max = (t_min + 3 * rng.random(512)).astype(np.float32)
        return ro, rd, rng.random((4, 32, 32, 32)) > 0.5, scenes.nested_aabbs(4), dict(
            render_step_size=1e-2, cone_angle=0.004, near_plane=0.15, far_plane=3.4, t_min=t_min, t_max=t_max)
    if name == "misses":                       # from far away, pointing away from every box
        ro = np.tile(np.array([[20, 20, 20], [-30, 0, 0]], np.float32), (64, 1))
        rd = np.tile(np.array([[1, 0, 0], [-1, 0, 0]], np.float32), (64, 1))
        return ro, rd, rng.random((4, 32, 32, 32)) > 0.5, scenes.nested_aabbs(4), dict(render_step_size=1e-2,
                                                                                         cone_angle=0.004)
    if name == "empty":
        ro, rd = _random_rays(rng, 512)
        return ro, rd, np.zeros((4, 32, 32, 32), bool), scenes.nested_aabbs(4), dict(render_step_size=1e-3,
                                                                                       cone_angle=0.004)
    if name == "const_dt":                     # below / across t = step / cone = 2.5
        ro, rd = _random_rays(rng, 512, 0.3)
        far = np.where(np.arange(512) % 2 == 0, 2.4, 6.0).astype(np.float32)
        return ro, rd, rng.random((4, 16, 16, 16)) > 0.3, scenes.nested_aabbs(4), dict(
            render_step_size=1e-2, cone_angle=0.004, t_max=far)
    raise KeyError(name)


SCENES = ["ball", "lvl4_32", "lvl4_128", "inside", "planes", "misses", "empty", "const_dt"]


@pytest.mark.parametrize("name", SCENES)
def test_cone_sampling_matches_oracle(orc, name):
    ro, rd, bins, aabbs, kw = _scene(name)
    est = _estimator(bins, aabbs)
    tkw = {k: (T(v) if isinstance(v, np.ndarray) else v) for k, v in kw.items()}
    ri, ts, te = est.sampling(T(ro), T(rd), **tkw)
    o_ri, o_ts, o_te, o_pi = orc.occgrid_sampling(ro, rd, bins, aabbs, **kw)
    np.testing.assert_array_equal(N(ri), o_ri)
    assert N(ts).tobytes() == o_ts.tobytes() and N(te).tobytes() == o_te.tobytes()
    R = ro.shape[0]
    pi = ri._nfa_packed[0]                                    # what the expand kernel wrote
    np.testing.assert_array_equal(N(pi), o_pi)
    np.testing.assert_array_equal(N(pi), orc.pack_info(o_ri, R))
    if name in ("misses", "empty"):
        assert ri.numel() == 0
    else:
        assert ri.numel() > 0


def test_cone_sampling_same_bits_as_traverse_grids_route_360():
    """65 536 rays, 4 x 128^3 levels, step 1e-3, cone 0.004, near 0.2, stratified with the same seed: the full arrays
    of the new route equal those of traverse_grids + vals[is_left] / vals[is_right]."""
    c = CONE360
    ro, rd = scenes.ball_rays(c["rays"], seed=42)
    est = _estimator(rr.grid_for(c), scenes.nested_aabbs(c["levels"]))
    kw = dict(near_plane=c["near"], render_step_size=c["step"], cone_angle=c["cone"], stratified=True)
    o, d = T(ro), T(rd)
    for seed in (0, 1):
        torch.manual_seed(seed)
        got = est.sampling(o, d, **kw)
        torch.manual_seed(seed)
        want = _old_route(est, o, d, **kw)
        _same(got, want)
        assert got[0].numel() > 10 * c["rays"]
        torch.testing.assert_close(nfa.pack_info(got[0], c["rays"]), nfa.pack_info(want[0].clone(), c["rays"]),
                                   rtol=0, atol=0)


def test_cone_sampling_matches_reference_cuda_build():
    ref = dict(load_golden("ref_live_cone360"))
    got = run_cone360(nfa, dev)
    assert sorted(got) == sorted(ref)
    for k, v in ref.items():
        assert str(got[k]) == str(v), k
    assert 0 < int(ref["vis_n"]) < int(ref["n"])


def test_cone_visibility_filter_keeps_the_same_samples():
    rng = np.random.default_rng(3)
    ro, rd = scenes.ball_rays(8192, seed=3)
    est = _estimator(_fragments(rng, 4, 64), scenes.nested_aabbs(4))
    o, d = T(ro), T(rd)
    base = dict(near_plane=0.2, render_step_size=1e-3, cone_angle=0.004)
    for kw in (dict(sigma_fn=rr.field_sigma, alpha_thre=1e-2), dict(sigma_fn=rr.field_sigma, early_stop_eps=1e-2),
               dict(alpha_fn=rr.field_alpha, alpha_thre=2e-2, early_stop_eps=1e-2)):
        got, want = est.sampling(o, d, **base, **kw), _old_route(est, o, d, **base, **kw)
        _same(got, want)
        assert 0 < got[0].numel() < est.sampling(o, d, **base)[0].numel()


def test_cone_zero_rays_and_all_miss_batches():
    rng = np.random.default_rng(4)
    est = _estimator(rng.random((4, 32, 32, 32)) > 0.5, scenes.nested_aabbs(4))
    empty = torch.empty((0, 3), device=dev)
    for kw in ({}, dict(sigma_fn=rr.field_sigma, alpha_thre=1e-2)):
        ri, ts, te = est.sampling(empty, empty, render_step_size=1e-3, cone_angle=0.004, **kw)
        assert ri.numel() == ts.numel() == te.numel() == 0 and ri.dtype == torch.int64
    ro = T(np.tile(np.array([[20, 20, 20]], np.float32), (1000, 1)))
    rd = T(np.tile(np.array([[1, 0, 0]], np.float32), (1000, 1)))
    for kw in ({}, dict(sigma_fn=rr.field_sigma, alpha_thre=1e-2)):
        got = est.sampling(ro, rd, render_step_size=1e-3, cone_angle=0.004, **kw)
        _same(got, _old_route(est, ro, rd, render_step_size=1e-3, cone_angle=0.004, **kw))
        assert got[0].numel() == 0
        assert torch.equal(nfa.pack_info(got[0], 1000), torch.zeros((1000, 2), dtype=torch.int64, device=dev))


def test_cone_split_matches_sampling():
    """sampling_end(sampling_begin(..., cone_angle=c)) == sampling(..., cone_angle=c): plain, two tickets in flight,
    a capacity hint that is too small (re-expand) and one that is too large (views shrunk)."""
    rng = np.random.default_rng(6)
    ro, rd = scenes.ball_rays(6000, seed=6)
    est = _estimator(_fragments(rng, 4, 64), scenes.nested_aabbs(4))
    o, d = T(ro), T(rd)
    kw = dict(near_plane=0.2, render_step_size=1e-3, cone_angle=0.004)
    want = est.sampling(o, d, **kw)
    n = want[0].numel()
    _same(est.sampling_end(est.sampling_begin(o, d, **kw)), want)
    mid = est.sampling(o[:1000], d[:1000], **kw)
    t1 = est.sampling_begin(o, d, **kw)
    t2 = est.sampling_begin(o[:1000], d[:1000], **kw)       # second workspace while the first is in flight
    got2, got1 = est.sampling_end(t2), est.sampling_end(t1)
    _same(got1, want)
    _same(got2, mid)
    for hint in (100, n - 1, 4 * n):
        est._capacity_hint = hint
        _same(est.sampling_end(est.sampling_begin(o, d, **kw)), want)
    est._capacity_hint = 4 * n
    f_want = _old_route(est, o, d, sigma_fn=rr.field_sigma, alpha_thre=1e-2, **kw)
    _same(est.sampling_end(est.sampling_begin(o, d, **kw), sigma_fn=rr.field_sigma, alpha_thre=1e-2), f_want)
    with pytest.raises(ValueError):
        est.sampling_begin(o, d, render_step_size=1e-3, cone_angle=-0.1)
    with pytest.raises(ValueError):
        est.sampling_begin(o.cpu(), d.cpu(), cone_angle=0.004)


def test_cone_run_pool_overflow_re_marches():
    """A fragmented grid gives far more runs than the first run pool of a fresh workspace holds (2 R + 1024): the
    march runs again with a larger pool and the result is unchanged."""
    rng = np.random.default_rng(8)
    R = 300
    ro, rd = _random_rays(rng, R, 1.5)
    bins = rng.random((4, 128, 128, 128)) > 0.5
    est = _estimator(bins, scenes.nested_aabbs(4))
    o, d = T(ro), T(rd)
    kw = dict(near_plane=0.2, render_step_size=1e-3, cone_angle=0.004)
    want = _old_route(est, o, d, **kw)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()                                # a stream no workspace has been made for yet
    with torch.cuda.stream(s):
        ticket = est.sampling_begin(o, d, **kw)
        cap0 = ticket.sc.run_capacity
        res = ticket.finish()
    torch.cuda.synchronize()
    assert cap0 == 2 * R + 1024 and res.n_runs > cap0
    _same((res.ray_indices, res.t_starts, res.t_ends), want)
    assert torch.equal(res.packed_info, nfa.pack_info(want[0], R))


def test_cone_two_streams_and_sampling_begin_does_not_sync():
    rng = np.random.default_rng(9)
    est = _estimator(_fragments(rng, 4, 64), scenes.nested_aabbs(4))
    A = tuple(T(x) for x in scenes.ball_rays(20000, seed=1))
    B = tuple(T(x) for x in scenes.ball_rays(31000, seed=2))
    kw = dict(near_plane=0.2, render_step_size=1e-3, cone_angle=0.004)
    want_a, want_b = est.sampling(*A, **kw), est.sampling(*B, **kw)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for _ in range(3):
        with torch.cuda.stream(s1):
            ta = est.sampling_begin(*A, **kw)
        with torch.cuda.stream(s2):
            tb = est.sampling_begin(*B, **kw)
        with torch.cuda.stream(s1):
            got_a = est.sampling_end(ta)
        with torch.cuda.stream(s2):
            got_b = est.sampling_end(tb)
        torch.cuda.synchronize()
        _same(got_a, want_a)
        _same(got_b, want_b)
    # after one warm-up call (workspace, pinned totals slot), queueing the traversal never waits for the GPU
    for skw in (dict(), dict(stratified=True), dict(t_min=torch.full_like(A[0][:, 0], 0.3))):
        est.sampling_end(est.sampling_begin(*A, **kw, **skw))
        torch.cuda.set_sync_debug_mode("error")
        try:
            ticket = est.sampling_begin(*A, **kw, **skw)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        got = est.sampling_end(ticket)
        if not skw:
            _same(got, want_a)
