"""GPU parity tests: the native sm_90a path (through the C ABI) vs the CPU oracle,
vs golden vectors of the reference CUDA build, and the reference's own test cases
(/root/reference/tests/test_{grid,rendering,pack,scan}.py) restated.

Bars (BASELINE.json north_star): bit-exact ray_indices / packed_info / t_starts / t_ends;
1e-5 abs on weights / colours (tolerances are written next to each assert)."""
import hashlib
import os

import numpy as np
import pytest
import torch

import nerfacc_b200 as nfa
from nerfacc_b200 import _lib, scenes
from conftest import golden_bins, load_golden

pytestmark = pytest.mark.gpu
dev = "cuda:0"


def T(a, **kw):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev, **kw)


def N(t):
    return t.detach().cpu().numpy()


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _estimator(bins, aabbs):
    est = nfa.OccGridEstimator(torch.from_numpy(aabbs[0]), resolution=list(bins.shape[1:]), levels=bins.shape[0]).to(dev)
    est.binaries = T(bins)
    return est


def test_native_library_is_loaded():
    lib = _lib.load()
    assert lib.nfa_version() == _lib.ABI_VERSION
    before = _lib.launches
    nfa.pack_info(torch.tensor([0, 0, 1], device=dev), 2)
    assert _lib.launches > before  # the call went through the C ABI, not a torch fallback


# ---------------------------------------------------------------- sampling vs oracle

def _check_sampling(orc, ro, rd, bins, aabbs, **kw):
    est = _estimator(bins, aabbs)
    tk = {k: (T(v) if isinstance(v, np.ndarray) else v) for k, v in kw.items()}
    out = []
    for _ in range(2):  # second call takes the capacity-hint (expand-before-sync) path
        ri, ts, te = est.sampling(T(ro), T(rd), **tk)
        out.append((ri, ts, te))
    o_ri, o_ts, o_te, o_pi = orc.occgrid_sampling(ro, rd, bins, aabbs, **kw)
    for ri, ts, te in out:
        assert ri.dtype == torch.int64 and ts.dtype == torch.float32
        np.testing.assert_array_equal(N(ri), o_ri)   # bit-exact
        np.testing.assert_array_equal(N(ts), o_ts)   # bit-exact
        np.testing.assert_array_equal(N(te), o_te)   # bit-exact
        np.testing.assert_array_equal(N(nfa.pack_info(ri, ro.shape[0])), o_pi)
    return len(o_ri)


def test_sampling_ball_scene(orc):
    ro, rd = scenes.ball_rays(4096)
    n = _check_sampling(orc, ro, rd, scenes.ball_grid(128), scenes.nested_aabbs(1), render_step_size=scenes.BALL_STEP)
    assert 122 <= n / 4096 <= 134


def test_sampling_many_runs_per_ray(orc):
    """Many runs per ray: exercises the descriptor-buffer flush loop and the run-pool re-march."""
    ro, rd = scenes.ball_rays(1024)
    rng = np.random.default_rng(7)
    frag = scenes.ball_grid(128) & (rng.random((1, 128, 128, 128)) > 0.5)
    _check_sampling(orc, ro, rd, frag, scenes.nested_aabbs(1), render_step_size=scenes.BALL_STEP)


def test_sampling_nested_levels_and_planes(orc):
    rng = np.random.default_rng(11)
    R = 300
    ro = rng.standard_normal((R, 3)).astype(np.float32)
    rd = rng.standard_normal((R, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    bins4 = rng.random((4, 32, 32, 32)) > 0.5
    a4 = scenes.nested_aabbs(4)
    _check_sampling(orc, ro, rd, bins4, a4, render_step_size=1e-2)
    _check_sampling(orc, ro, rd, bins4, a4, render_step_size=1e-2, near_plane=0.15, far_plane=3.4,
                    t_min=rng.random(R).astype(np.float32), t_max=(1 + 3 * rng.random(R)).astype(np.float32))
    _check_sampling(orc, ro, rd, rng.random((2, 30, 17, 5)) > 0.3, a4[:2], render_step_size=4e-3)
    # stratified jitter stand-in: per-ray near planes inside one step
    _check_sampling(orc, ro, rd, bins4[:1], a4[:1], render_step_size=5e-3, t_min=(rng.random(R) * 5e-3).astype(np.float32))


@pytest.mark.parametrize("seed", range(10))
def test_sampling_random_scenes(orc, seed):
    """Randomised scenes: odd grid shapes, 1-3 levels, sparse to dense occupancy, rays from inside and outside,
    random step sizes and clipping planes -- bit-exact against the oracle every time."""
    rng = np.random.default_rng(1000 + seed)
    R = int(rng.integers(130, 400))  # not a multiple of the 128-ray tile
    levels = int(rng.integers(1, 4))
    shape = tuple(int(v) for v in rng.integers(5, 41, 3))
    density = float(rng.choice([0.02, 0.2, 0.5, 0.9]))
    bins = rng.random((levels,) + shape) < density
    if seed % 3 == 0:  # a compact blob, so the occupied-brick bounding box is much smaller than the grid
        blob = np.zeros(shape, bool)
        c = [s // 2 for s in shape]
        blob[max(c[0] - 3, 0):c[0] + 3, max(c[1] - 2, 0):c[1] + 2, max(c[2] - 3, 0):c[2] + 4] = True
        bins[0] = blob
    aabbs = scenes.nested_aabbs(levels)
    inside = rng.random(R) < 0.4
    ro = np.where(inside[:, None], rng.uniform(-1, 1, (R, 3)), rng.standard_normal((R, 3)) * 3).astype(np.float32)
    rd = rng.standard_normal((R, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    if seed % 4 == 1:
        rd[::7] = np.array([0.0, 1.0, 0.0], np.float32)  # axis-aligned rays (infinite crossing times)
    step = float(rng.choice([2e-3, 5e-3, 1.3e-2, 3e-2]))
    kw = dict(render_step_size=step)
    if seed % 2 == 0:
        kw.update(near_plane=float(rng.uniform(0, 0.5)), far_plane=float(rng.uniform(2, 8)))
    if seed % 5 == 3:
        kw.update(t_min=rng.uniform(0, 1, R).astype(np.float32), t_max=rng.uniform(1, 6, R).astype(np.float32))
    _check_sampling(orc, ro, rd, bins, aabbs, **kw)


def test_sampling_edge_cases(orc):
    a1 = scenes.nested_aabbs(1)
    est = _estimator(np.zeros((1, 8, 8, 8), bool), a1)
    ro, rd = scenes.ball_rays(100)
    ri, ts, te = est.sampling(T(ro), T(rd), render_step_size=1e-2)  # empty grid
    assert ri.numel() == ts.numel() == te.numel() == 0 and ri.dtype == torch.int64
    ri, ts, te = est.sampling(T(ro[:0]), T(rd[:0]), render_step_size=1e-2)  # empty ray batch
    assert ri.numel() == 0
    full = _estimator(np.ones((1, 4, 4, 4), bool), a1)
    away = T(ro) * 0 + torch.tensor([5.0, 5.0, 5.0], device=dev)
    ri, _, _ = full.sampling(away, T(np.tile(np.array([[1, 0, 0]], np.float32), (100, 1))), render_step_size=1e-2)
    assert ri.numel() == 0  # all rays miss
    # axis-aligned directions (zero components)
    ro2 = np.array([[-2, 0.1, 0.2], [0.3, -3, 0.1], [0.01, 0.02, 5], [0, 0, 0]], np.float32)
    rd2 = np.array([[1, 0, 0], [0, 1, 0], [0, 0, -1], [0, 0, 1]], np.float32)
    rng = np.random.default_rng(3)
    _check_sampling(orc, ro2, rd2, rng.random((4, 32, 32, 32)) > 0.5, scenes.nested_aabbs(4), render_step_size=1e-2)
    # step far below the float32 resolution of t: the reference would never terminate, we raise
    huge = nfa.OccGridEstimator([-1e6, -1e6, -1e6, 1e6, 1e6, 1e6], resolution=4).to(dev)
    huge.binaries = torch.ones_like(huge.binaries)
    with pytest.raises(RuntimeError, match="cannot advance"):
        huge.sampling(T(ro2[:1] * 0), T(rd2[:1]), near_plane=3.0e5, far_plane=1e10, render_step_size=1e-3)


def test_grid_mutation_invalidates_pack(orc):
    ro, rd = scenes.ball_rays(256)
    a1 = scenes.nested_aabbs(1)
    est = _estimator(scenes.ball_grid(32), a1)
    n0 = est.sampling(T(ro), T(rd), render_step_size=1e-2)[0].numel()
    est.binaries[0, :16] = False  # in-place edit
    o = orc.occgrid_sampling(ro, rd, N(est.binaries), a1, render_step_size=1e-2)
    assert est.sampling(T(ro), T(rd), render_step_size=1e-2)[0].numel() == len(o[0]) < n0
    est.binaries = T(scenes.ball_grid(32, radius=0.3))  # reassignment (reference occ_grid.py:404)
    o = orc.occgrid_sampling(ro, rd, scenes.ball_grid(32, radius=0.3), a1, render_step_size=1e-2)
    np.testing.assert_array_equal(N(est.sampling(T(ro), T(rd), render_step_size=1e-2)[1]), o[1])


# ---------------------------------------------------------------- vs reference-CUDA goldens

@pytest.mark.parametrize("name", ["ref_sampling_ball", "ref_sampling_frag", "ref_sampling_lvl4",
                                  "ref_sampling_lvl4_tminmax"])
def test_sampling_matches_reference_cuda(name):
    z = load_golden(name)
    kw = dict(zip([str(s) for s in z["kw_names"]], [float(v) for v in z["kw_vals"]]))
    if "in_t_min" in z:
        kw["t_min"], kw["t_max"] = T(z["in_t_min"]), T(z["in_t_max"])
    est = _estimator(golden_bins(z), z["aabbs"])
    ri, ts, te = est.sampling(T(z["rays_o"]), T(z["rays_d"]), **kw)
    assert ri.numel() == int(z["n_samples"])
    assert _sha(N(ri)) == str(z["ray_indices_sha"])                                   # bit-exact
    np.testing.assert_array_equal(N(nfa.pack_info(ri, z["rays_o"].shape[0])), z["packed_info"])  # bit-exact
    np.testing.assert_array_equal(N(ts), z["t_starts"])
    np.testing.assert_array_equal(N(te), z["t_ends"])


def test_traverse_grids_matches_reference_cuda(orc):
    z = load_golden("ref_traverse_lvl4")
    iv, sm, term = nfa.traverse_grids(T(z["rays_o"]), T(z["rays_d"]), T(golden_bins(z)), T(z["aabbs"]),
                                      step_size=float(z["step_size"]))
    np.testing.assert_array_equal(N(iv.vals), z["iv_vals"])
    np.testing.assert_array_equal(np.packbits(N(iv.is_left)), z["iv_left"])
    np.testing.assert_array_equal(np.packbits(N(iv.is_right)), z["iv_right"])
    np.testing.assert_array_equal(N(iv.packed_info), z["iv_packed_info"])
    assert _sha(N(iv.ray_indices)) == str(z["iv_ray_sha"])
    np.testing.assert_array_equal(N(sm.vals), z["sm_vals"])
    np.testing.assert_array_equal(N(sm.packed_info), z["sm_packed_info"])
    assert _sha(N(sm.ray_indices)) == str(z["sm_ray_sha"]) and bool(sm.is_valid.all())
    _, _, o_term = orc.traverse_grids(z["rays_o"], z["rays_d"], golden_bins(z), z["aabbs"], step_size=float(z["step_size"]))
    d = ~np.isnan(o_term)
    np.testing.assert_array_equal(N(term)[d], z["terminate"][d])
    # pre-computed crossings (reference examples/utils.py:332-342) give the same result
    tm, tM, hits = nfa.ray_aabb_intersect(T(z["rays_o"]), T(z["rays_d"]), T(z["aabbs"]))
    tsrt, tidx = torch.sort(torch.cat([tm, tM], -1), -1)
    iv2, _, _ = nfa.traverse_grids(T(z["rays_o"]), T(z["rays_d"]), T(golden_bins(z)), T(z["aabbs"]),
                                   step_size=float(z["step_size"]), t_sorted=tsrt, t_indices=tidx, hits=hits)
    np.testing.assert_array_equal(N(iv2.vals), z["iv_vals"])


def test_ray_aabb_matches_reference_cuda():
    z = load_golden("ref_ray_aabb")
    tm, tM, h = nfa.ray_aabb_intersect(T(z["rays_o"]), T(z["rays_d"]), T(z["aabbs"]))
    np.testing.assert_array_equal(N(tm), z["t_mins"])
    np.testing.assert_array_equal(N(tM), z["t_maxs"])
    np.testing.assert_array_equal(N(h), z["hits"])
    # reference tests/test_grid.py:8-35: agrees with the plain-torch version
    _tm, _tM, _h = nfa.grid._ray_aabb_intersect(T(z["rays_o"]), T(z["rays_d"]), T(z["aabbs"]))
    assert torch.allclose(tm, _tm) and torch.allclose(tM, _tM) and (h == _h).all()


def test_rendering_matches_reference_cuda():
    z = load_golden("ref_render_ball")
    R = int(z["n_rays"])
    ri = T(np.repeat(np.arange(R), z["packed_info"][:, 1]))
    sig, rgb = T(z["sigmas"]).requires_grad_(True), T(z["rgbs"]).requires_grad_(True)
    col, op, dep, ex = nfa.rendering(T(z["t_starts"]), T(z["t_ends"]), ri, n_rays=R,
                                     rgb_sigma_fn=lambda a, b, c: (rgb, sig), render_bkgd=T(z["bkgd"]))
    for got, key in [(ex["weights"], "weights"), (ex["trans"], "trans"), (ex["alphas"], "alphas"), (col, "colors"),
                     (op, "opacities"), (dep, "depths")]:
        np.testing.assert_allclose(N(got), z[key], atol=1e-5, rtol=0, err_msg=key)   # north_star tolerance
    ((col * T(z["gC"])).sum() + (op * T(z["gO"])).sum() + (dep * T(z["gD"])).sum()).backward()
    np.testing.assert_allclose(N(sig.grad), z["g_sigmas"], atol=1e-5, rtol=1e-4)
    np.testing.assert_allclose(N(rgb.grad), z["g_rgbs"], atol=1e-5, rtol=1e-4)
    x = load_golden("ref_render_extras")
    al = T(x["alphas_in"]).requires_grad_(True)
    w, tr = nfa.render_weight_from_alpha(al, ray_indices=ri, n_rays=R)
    np.testing.assert_allclose(N(w), x["weights_a"], atol=1e-5, rtol=0)
    np.testing.assert_allclose(N(tr), x["trans_a"], atol=1e-5, rtol=0)
    ((w * T(x["gW"])).sum() + (tr * T(x["gT"])).sum()).backward()
    np.testing.assert_allclose(N(al.grad), x["g_alphas"], atol=2e-5, rtol=1e-4)
    sig.grad = None
    w2, t2, a2 = nfa.render_weight_from_density(T(z["t_starts"]), T(z["t_ends"]), sig, ray_indices=ri, n_rays=R)
    ((w2 * T(x["gW"])).sum() + (t2 * T(x["gT"])).sum() + (a2 * T(x["gA"])).sum()).backward()
    np.testing.assert_allclose(N(sig.grad), x["g_sigmas"], atol=1e-5, rtol=1e-4)


def test_scans_match_reference_cuda():
    s = load_golden("ref_scans")
    pi = T(s["packed_info"])
    idx = T(np.repeat(np.arange(len(s["packed_info"])), s["packed_info"][:, 1]))
    gy = T((np.arange(len(s["x"])) % 7 + 1).astype(np.float32))
    for nm in ["inclusive_sum", "exclusive_sum", "inclusive_prod", "exclusive_prod"]:
        for mode in ["packed", "key"]:
            x = T(s["x"]).requires_grad_(True)
            y = getattr(nfa, nm)(x, packed_info=pi) if mode == "packed" else getattr(nfa, nm)(x, indices=idx)
            np.testing.assert_allclose(N(y), s[f"{nm}_{mode}"], rtol=2e-5, atol=1e-6, err_msg=f"{nm}/{mode}")
            (y * gy).sum().backward()
            np.testing.assert_allclose(N(x.grad), s[f"{nm}_{mode}_grad"], rtol=5e-5, atol=1e-5, err_msg=f"{nm}/{mode}/grad")


# ---------------------------------------------------------------- fused compositing vs the f64 oracle

def _ball_samples(R=2048):
    ro, rd = scenes.ball_rays(R)
    est = _estimator(scenes.ball_grid(128), scenes.nested_aabbs(1))
    ri, ts, te = est.sampling(T(ro), T(rd), render_step_size=scenes.BALL_STEP)
    return ri, ts, te, N(nfa.pack_info(ri, R))


@pytest.mark.parametrize("expected_depths,bkgd", [(True, True), (False, False)])
def test_fused_rendering_vs_oracle(orc, expected_depths, bkgd):
    R = 2048
    ri, ts, te, pi = _ball_samples(R)
    n = ri.numel()
    g = torch.Generator().manual_seed(43)
    sig = (5 * torch.rand(n, generator=g)).to(dev).requires_grad_(True)
    rgb = torch.rand(n, 3, generator=g).to(dev).requires_grad_(True)
    bk = torch.tensor([0.2, 0.5, 0.9], device=dev) if bkgd else None
    col, op, dep, ex = nfa.rendering(ts, te, ri, n_rays=R, rgb_sigma_fn=lambda a, b, c: (rgb, sig), render_bkgd=bk,
                                     expected_depths=expected_depths)
    assert col.shape == (R, 3) and op.shape == (R, 1) and dep.shape == (R, 1)
    o = orc.composite(N(ts), N(te), N(sig), N(rgb), packed_info=pi, render_bkgd=None if bk is None else N(bk),
                      expected_depths=expected_depths)
    for got, key in [(ex["weights"], "weights"), (ex["trans"], "trans"), (ex["alphas"], "alphas"), (col, "colors"),
                     (op, "opacities"), (dep, "depths")]:
        np.testing.assert_allclose(N(got), o[key], atol=1e-5, rtol=0, err_msg=key)
    gC, gO, gD = (torch.rand(s, generator=g).to(dev) for s in [(R, 3), (R, 1), (R, 1)])
    ((col * gC).sum() + (op * gO).sum() + (dep * gD).sum()).backward()
    gs, gr = orc.composite_backward(N(ts), N(te), N(sig), N(rgb), pi, gC=N(gC), gO=N(gO).ravel(), gD=N(gD).ravel(),
                                    render_bkgd=None if bk is None else N(bk), expected_depths=expected_depths)
    np.testing.assert_allclose(N(sig.grad), gs, atol=1e-5, rtol=1e-4)
    np.testing.assert_allclose(N(rgb.grad), gr, atol=1e-5, rtol=1e-4)
    # weights sum to the opacity; colours are linear in rgbs
    np.testing.assert_allclose(N(nfa.accumulate_along_rays(ex["weights"], None, ri, R)), N(op), atol=1e-5)
    col2, _, _, _ = nfa.rendering(ts, te, ri, n_rays=R, rgb_sigma_fn=lambda a, b, c: (2 * rgb.detach(), sig.detach()))
    col1, _, _, _ = nfa.rendering(ts, te, ri, n_rays=R, rgb_sigma_fn=lambda a, b, c: (rgb.detach(), sig.detach()))
    np.testing.assert_allclose(N(col2), 2 * N(col1), atol=1e-5)


def test_vector_and_scalar_kernels_agree(orc):
    """16-byte aligned inputs take the 128-bit kernels, anything else the element-wise ones; both must match the
    oracle.  Also ragged rays: empty rays, 1-sample rays, rays that start / end mid-group."""
    g = torch.Generator().manual_seed(9)
    cnts = torch.tensor([0, 1, 3, 4, 5, 0, 127, 128, 129, 2, 0, 0, 33, 64, 1, 7, 250, 0, 31], dtype=torch.int64)
    starts = torch.cumsum(cnts, 0) - cnts
    pi = torch.stack([starts, cnts], -1).to(dev)
    n, R = int(cnts.sum()), len(cnts)
    for off in (0, 1):  # off=1: views with a 4-byte offset -> element-wise kernels
        def place(t):  # copy into a view whose storage offset is `off` elements (4 bytes): not 16-byte aligned
            buf = torch.empty((t.shape[0] + off,) + tuple(t.shape[1:]), device=dev)
            v = buf[off:]
            v.copy_(t)
            return v
        ts = place(torch.rand(n, generator=g).to(dev) * 0.5)
        te = place(ts + 0.01 + torch.rand(n, generator=g).to(dev) * 0.02)
        sig = place(8 * torch.rand(n, generator=g).to(dev)).requires_grad_(True)
        rgb = place(torch.rand(n, 3, generator=g).to(dev)).requires_grad_(True)
        assert (ts.data_ptr() % 16 != 0) == bool(off)
        sig_l, rgb_l = sig.detach().clone().requires_grad_(True), rgb.detach().clone().requires_grad_(True)
        ri = torch.repeat_interleave(torch.arange(R), cnts).to(dev)
        for use_alpha in (False, True):
            sig_l.grad = rgb_l.grad = None
            dens = sig_l if not use_alpha else (sig_l / 10.0)
            d_in = dens if off == 0 else torch.cat([dens.new_zeros(1), dens])[1:]
            c_in = rgb_l if off == 0 else torch.cat([rgb_l.new_zeros(1, 3), rgb_l])[1:]
            fn = (lambda a, b, c: (c_in, d_in))
            kw = dict(rgb_alpha_fn=fn) if use_alpha else dict(rgb_sigma_fn=fn)
            col, op, dep, ex = nfa.rendering(ts, te, ri, n_rays=R, **kw)
            gC, gO, gD = (torch.rand(sh, generator=g).to(dev) for sh in [(R, 3), (R, 1), (R, 1)])
            gW = torch.rand(n, generator=g).to(dev)
            ((col * gC).sum() + (op * gO).sum() + (dep * gD).sum() + (ex["weights"] * gW).sum()).backward()
            if not use_alpha:
                o = orc.composite(N(ts), N(te), N(dens), N(rgb_l), packed_info=N(pi))
                gs, gr = orc.composite_backward(N(ts), N(te), N(dens), N(rgb_l), N(pi), gC=N(gC), gO=N(gO).ravel(),
                                                gD=N(gD).ravel(), gW=N(gW))
                for got, key in [(ex["weights"], "weights"), (ex["trans"], "trans"), (col, "colors"), (op, "opacities"),
                                 (dep, "depths")]:
                    np.testing.assert_allclose(N(got), o[key], atol=1e-5, rtol=0, err_msg=f"{key} off={off}")
                np.testing.assert_allclose(N(sig_l.grad), gs, atol=2e-5, rtol=1e-4)
                np.testing.assert_allclose(N(rgb_l.grad), gr, atol=1e-5, rtol=1e-4)
            else:
                ow, oT = orc.render_weight_from_alpha(N(dens), packed_info=N(pi))
                np.testing.assert_allclose(N(ex["weights"]), ow, atol=1e-5, rtol=0)
                np.testing.assert_allclose(N(ex["trans"]), oT, atol=1e-5, rtol=0)
                # gradient vs torch autograd on the batched formulation, ray by ray
                ref = torch.zeros_like(dens)
                d64 = dens.detach().double().requires_grad_(True)
                tot = 0
                for r in range(R):
                    s0, c0 = int(starts[r]), int(cnts[r])
                    if c0 == 0:
                        continue
                    a = d64[s0:s0 + c0]
                    T = torch.cumprod(torch.cat([a.new_ones(1), 1 - a[:-1]]), 0)
                    w = T * a
                    m = ((ts + te) / 2)[s0:s0 + c0].double()
                    O = w.sum()
                    tot = tot + (w[:, None] * rgb_l.detach()[s0:s0 + c0].double() * gC[r].double()).sum() + O * gO[r, 0].double() \
                        + (w * m).sum() / O.clamp_min(1.1920929e-07) * gD[r, 0].double() + (w * gW[s0:s0 + c0].double()).sum()
                tot.backward()
                got = sig_l.grad * 10.0  # d/d(alpha) = 10 * d/d(sig_l)
                np.testing.assert_allclose(N(got), N(d64.grad), atol=5e-5, rtol=1e-3)


def test_general_gradients_prefix_trans_and_alpha_route(orc):
    R = 512
    ri, ts, te, pi = _ball_samples(R)
    n = ri.numel()
    g = torch.Generator().manual_seed(5)
    sig = (5 * torch.rand(n, generator=g)).to(dev).requires_grad_(True)
    pt = (0.5 + 0.5 * torch.rand(n, generator=g)).to(dev)
    gW, gT, gA = (torch.rand(n, generator=g).to(dev) for _ in range(3))
    for kwargs in [dict(ray_indices=ri, n_rays=R), dict(packed_info=T(pi))]:
        sig.grad = None
        w, tr, a = nfa.render_weight_from_density(ts, te, sig, prefix_trans=pt, **kwargs)
        o = orc.composite(N(ts), N(te), N(sig), None, packed_info=pi, prefix_trans=N(pt))
        np.testing.assert_allclose(N(w), o["weights"], atol=1e-5)
        np.testing.assert_allclose(N(tr), o["trans"], atol=1e-5)
        ((w * gW).sum() + (tr * gT).sum() + (a * gA).sum()).backward()
        gs, _ = orc.composite_backward(N(ts), N(te), N(sig), None, pi, gW=N(gW), gT=N(gT), gA=N(gA), prefix_trans=N(pt))
        np.testing.assert_allclose(N(sig.grad), gs, atol=1e-5, rtol=1e-4)
    # background colour that requires grad goes through autograd
    bk = torch.tensor([0.2, 0.5, 0.9], device=dev, requires_grad=True)
    rgb = torch.rand(n, 3, generator=g).to(dev)
    col, op, _, _ = nfa.rendering(ts, te, ri, n_rays=R, rgb_sigma_fn=lambda a, b, c: (rgb, sig.detach()), render_bkgd=bk)
    col.sum().backward()
    np.testing.assert_allclose(N(bk.grad), np.full(3, float((1 - op).sum())), rtol=1e-5)
    # transmittance / visibility entry points
    tr2, a2 = nfa.render_transmittance_from_density(ts, te, sig.detach(), ray_indices=ri, n_rays=R)
    o = orc.composite(N(ts), N(te), N(sig), None, packed_info=pi)
    np.testing.assert_allclose(N(tr2), o["trans"], atol=1e-5)
    vis = nfa.render_visibility_from_density(ts, te, sig.detach(), ray_indices=ri, n_rays=R, early_stop_eps=0.3, alpha_thre=0.01)
    exp = (o["trans"] >= 0.3) & (o["alphas"] >= 0.01)
    assert (N(vis) != exp).mean() < 1e-4  # thresholds on values that differ by ~1e-7


# ---------------------------------------------------------------- the reference's own test cases

def test_reference_rendering_cases():
    ri = torch.tensor([0, 2, 2, 2, 2], dtype=torch.int64, device=dev)
    al = torch.tensor([0.4, 0.3, 0.8, 0.8, 0.5], device=dev)
    # tests/test_rendering.py:8-34
    vis = nfa.render_visibility_from_alpha(al, ray_indices=ri, early_stop_eps=0.03, alpha_thre=0.0)
    assert vis.tolist() == [True, True, True, True, False]
    vis = nfa.render_visibility_from_alpha(al, ray_indices=ri, early_stop_eps=0.05, alpha_thre=0.35)
    assert vis.tolist() == [True, False, True, True, False]
    # :38-57
    w, _ = nfa.render_weight_from_alpha(al, ray_indices=ri, n_rays=3)
    assert torch.allclose(w, torch.tensor([0.4, 0.3, 0.7 * 0.8, 0.14 * 0.8, 0.028 * 0.5], device=dev))
    # :61-83 density == alpha
    sig = torch.rand(5, device=dev)
    ts = torch.rand_like(sig)
    te = torch.rand_like(sig) + 1.0
    w1, _, _ = nfa.render_weight_from_density(ts, te, sig, ray_indices=ri, n_rays=3)
    w2, _ = nfa.render_weight_from_alpha(1.0 - torch.exp(-sig * (te - ts)), ray_indices=ri, n_rays=3)
    assert torch.allclose(w1, w2)
    # :87-106 accumulate, ray 1 empty
    vals = torch.rand(5, 2, device=dev)
    acc = nfa.accumulate_along_rays(al, values=vals, ray_indices=ri, n_rays=3)
    assert acc.shape == (3, 2) and torch.allclose(acc[0], al[0] * vals[0]) and (acc[1] == 0).all()
    assert torch.allclose(acc[2], (al[1:, None] * vals[1:]).sum(0))
    out = torch.ones(3, 2, device=dev)
    nfa.accumulate_along_rays_(al, values=vals, ray_indices=ri, outputs=out)
    assert torch.allclose(out, acc + 1)
    # :197-218 smoke
    nfa.rendering(ts, te, ray_indices=ri, n_rays=3, rgb_sigma_fn=lambda a, b, c: (torch.stack([a] * 3, -1), a))
    c, o, d, _ = nfa.rendering(ts[:0], te[:0], ray_indices=ri[:0], n_rays=3, rgb_sigma_fn=lambda a, b, c: (torch.stack([a] * 3, -1), a))
    assert c.shape == (3, 3) and (c == 0).all() and (o == 0).all()


def test_reference_grad_goldens_all_routes():
    # tests/test_rendering.py:110-193
    ri = torch.tensor([0, 2, 2, 2, 2], dtype=torch.int64, device=dev)
    pi = torch.tensor([[0, 1], [1, 0], [1, 4]], dtype=torch.long, device=dev)
    sig = torch.tensor([0.4, 0.8, 0.1, 0.8, 0.1], device=dev, requires_grad=True)
    ts = torch.rand_like(sig)
    te = ts + 1.0
    w_ref = torch.tensor([0.3297, 0.5507, 0.0428, 0.2239, 0.0174], device=dev)
    g_ref = torch.tensor([0.6703, 0.1653, 0.1653, 0.1653, 0.1653], device=dev)

    def routes():
        tr, _ = nfa.render_transmittance_from_density(ts, te, sig, ray_indices=ri, n_rays=3)
        yield tr * (1.0 - torch.exp(-sig * (te - ts)))
        tr, _ = nfa.render_transmittance_from_density(ts, te, sig, packed_info=pi, n_rays=3)
        yield tr * (1.0 - torch.exp(-sig * (te - ts)))
        yield nfa.render_weight_from_density(ts, te, sig, ray_indices=ri, n_rays=3)[0]
        yield nfa.render_weight_from_density(ts, te, sig, packed_info=pi, n_rays=3)[0]
        yield nfa.render_weight_from_alpha(1.0 - torch.exp(-sig * (te - ts)), ray_indices=ri, n_rays=3)[0]
        yield nfa.render_weight_from_alpha(1.0 - torch.exp(-sig * (te - ts)), packed_info=pi, n_rays=3)[0]

    for w in routes():
        sig.grad = None
        w.sum().backward()
        assert torch.allclose(w_ref, w, atol=1e-4) and torch.allclose(g_ref, sig.grad, atol=1e-4)


def test_reference_pack_and_scan_cases():
    # tests/test_pack.py:8-18 (int64 result compared with an int32 golden)
    ri = torch.tensor([0, 2, 2, 2, 2], dtype=torch.int64, device=dev)
    gold = torch.tensor([[0, 1], [1, 0], [1, 4]], dtype=torch.int32, device=dev)
    assert (nfa.pack_info(ri, n_rays=3) == gold).all()
    assert nfa.pack_info(ri).shape == (3, 2) and nfa.pack_info(ri.int(), 3).dtype == torch.int32
    # tests/test_scan.py:8-172: batched vs packed vs by-key, values and gradients
    torch.manual_seed(42)
    for fn, tol in [(nfa.inclusive_sum, 1e-5), (nfa.exclusive_sum, 3e-4), (nfa.inclusive_prod, 1e-5), (nfa.exclusive_prod, 1e-5)]:
        data = torch.rand((5, 1000), device=dev, requires_grad=True)
        o1 = fn(data).flatten()
        o1.sum().backward()
        g1 = data.grad.clone()
        data.grad = None
        starts = torch.arange(0, data.numel(), data.shape[1], device=dev, dtype=torch.long)
        pi = torch.stack([starts, torch.full((5,), 1000, dtype=torch.long, device=dev)], -1)
        o2 = fn(data.flatten(), packed_info=pi)
        o2.sum().backward()
        g2 = data.grad.clone()
        data.grad = None
        idx = torch.arange(5, device=dev, dtype=torch.long).repeat_interleave(1000)
        o3 = fn(data.flatten(), indices=idx)
        o3.sum().backward()
        g3 = data.grad.clone()
        assert torch.allclose(o1, o2, atol=tol) and torch.allclose(o1, o3, atol=tol)
        assert torch.allclose(g1, g2, rtol=1e-3, atol=1e-4) and torch.allclose(g1, g3, rtol=1e-3, atol=1e-4)


def test_reference_grid_cases():
    from nerfacc_b200.grid import _enlarge_aabb, _query
    torch.manual_seed(42)
    # tests/test_grid.py:39-68
    ro = torch.randn((10, 3), device=dev)
    rd = torch.randn((10, 3), device=dev)
    rd = rd / rd.norm(dim=-1, keepdim=True)
    base = torch.tensor([-1.0, -1.0, -1.0, 1.0, 1.0, 1.0], device=dev)
    aabbs = torch.stack([_enlarge_aabb(base, 2 ** i) for i in range(4)])
    binaries = torch.rand((4, 32, 32, 32), device=dev) > 0.5
    iv, sm, _ = nfa.traverse_grids(ro, rd, binaries, aabbs)
    ts, te = iv.vals[iv.is_left], iv.vals[iv.is_right]
    pos = ro[sm.ray_indices] + rd[sm.ray_indices] * (ts + te)[:, None] / 2.0
    occs, sel = _query(pos, binaries, base)
    assert occs.all() and sel.all() and ts.numel() > 0
    # :135-159
    d = torch.tensor([[1.0, 0.01, 0.01]], device=dev)
    iv, _, _ = nfa.traverse_grids(torch.tensor([[-1.0, 0.0, 0.0]], device=dev), d / d.norm(),
                                  torch.ones((1, 1, 1, 1), dtype=torch.bool, device=dev),
                                  torch.tensor([[0.0, 0.0, 0.0, 1.0, 1.0, 1.0]], device=dev), step_size=0.05,
                                  near_planes=torch.tensor([1.2], device=dev), far_planes=torch.tensor([1.5], device=dev))
    assert iv.vals.numel() > 0 and (iv.vals >= 1.2 - 0.025).all() and (iv.vals <= 1.5 + 0.025).all()
    # :163-203
    n_rays = 64
    ro = torch.rand((n_rays, 3), device=dev) * 2 - 1.0
    rd = torch.rand((n_rays, 3), device=dev)
    rd = rd / rd.norm(dim=-1, keepdim=True)
    t_min = torch.rand((n_rays,), device=dev)
    t_max = t_min + torch.rand((n_rays,), device=dev)
    est = nfa.OccGridEstimator(roi_aabb=base, resolution=32, levels=4)
    est.binaries = binaries
    ri, ts, te = est.sampling(rays_o=ro, rays_d=rd, near_plane=0.15, far_plane=0.85, t_min=t_min, t_max=t_max,
                              render_step_size=0.01)
    assert (ts >= (t_min[ri] - 0.005)).all() and (te <= (t_max[ri] + 0.005)).all()
    # :207-233
    est = nfa.OccGridEstimator(roi_aabb=base, resolution=32, levels=4).to(dev)
    K = torch.tensor([[[100.0, 0, 50.0], [0, 100.0, 50.0], [0, 0, 1]]], device=dev)
    pose = torch.tensor([[[-1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, -1.0, 2.5]]], device=dev)
    est.mark_invisible_cells(K, pose, 100, 100)
    assert (est.occs == -1).sum() == 77660 and (est.occs == 0).sum() == 53412


def test_sampling_with_sigma_fn_filters_like_reference_semantics(orc):
    R = 512
    ro, rd = scenes.ball_rays(R)
    est = _estimator(scenes.ball_grid(64), scenes.nested_aabbs(1))
    est.occs.fill_(1.0)
    sigma_fn = lambda ts, te, ri: 40.0 * torch.ones_like(ts)
    ri, ts, te = est.sampling(T(ro), T(rd), sigma_fn=sigma_fn, render_step_size=1e-2, early_stop_eps=1e-2, alpha_thre=0.0)
    o_ri, o_ts, o_te, o_pi = orc.occgrid_sampling(ro, rd, scenes.ball_grid(64), scenes.nested_aabbs(1), render_step_size=1e-2)
    o = orc.composite(o_ts, o_te, np.full(len(o_ts), 40.0, np.float32), None, packed_info=o_pi)
    keep = o["trans"] >= 1e-2
    assert abs(int(keep.sum()) - ri.numel()) <= 2 and 0 < ri.numel() < len(o_ri)


# ---------------------------------------------------------------- full-size properties (config 2 of BASELINE.json)

def test_full_size_properties():
    R = 65536
    ro, rd = scenes.ball_rays(R)
    bins = scenes.ball_grid(128)
    est = _estimator(bins, scenes.nested_aabbs(1))
    tro, trd = T(ro), T(rd)
    ri, ts, te = est.sampling(tro, trd, render_step_size=scenes.BALL_STEP)
    ri2, ts2, te2 = est.sampling(tro, trd, render_step_size=scenes.BALL_STEP)  # hinted path, deterministic
    assert torch.equal(ri, ri2) and torch.equal(ts, ts2) and torch.equal(te, te2)
    n = ri.numel()
    assert 122 <= n / R <= 134
    assert (ri[1:] >= ri[:-1]).all()                       # sorted / grouped
    pi = nfa.pack_info(ri, R)
    assert int(pi[:, 1].sum()) == n and (pi[:, 0] == torch.cumsum(pi[:, 1], 0) - pi[:, 1]).all()
    cnt = torch.bincount(ri, minlength=R)
    assert torch.equal(cnt, pi[:, 1])
    assert (te > ts).all()
    same_ray = ri[1:] == ri[:-1]
    contiguous = te[:-1] == ts[1:]
    gap = ts[1:] - te[:-1]
    assert (gap[same_ray] >= 0).all() and contiguous[same_ray].float().mean() > 0.95  # runs share edges bit-exactly
    # every midpoint sits in an occupied cell (reference tests/test_grid.py:59-68)
    pos = tro[ri] + trd[ri] * ((ts + te) / 2.0)[:, None]
    occ, sel = nfa.grid._query(pos, T(bins), torch.from_numpy(scenes.ROI_AABB).to(dev))
    # positions are re-computed here in float32, so a few midpoints land a rounding error outside their cell
    assert sel.all() and occ.float().mean() > 0.9999
    # compositing at full size: weights sum to opacity, checksum of the per-ray reduction
    sig = 5 * torch.rand(n, device=dev)
    rgb = torch.rand(n, 3, device=dev)
    col, op, dep, ex = nfa.rendering(ts, te, ri, n_rays=R, rgb_sigma_fn=lambda a, b, c: (rgb, sig))
    w64 = torch.zeros(R, dtype=torch.float64, device=dev).index_add_(0, ri, ex["weights"].double())
    assert (w64 - op[:, 0].double()).abs().max() < 1e-5
    c64 = torch.zeros(R, 3, dtype=torch.float64, device=dev).index_add_(0, ri, (ex["weights"][:, None] * rgb).double())
    assert (c64 - col.double()).abs().max() < 1e-5
    assert (ex["trans"] <= 1).all() and (ex["trans"] >= 0).all() and (op <= 1 + 1e-5).all()
    first = pi[pi[:, 1] > 0, 0]
    assert (ex["trans"][first] == 1).all()


def test_abi_direct_call_with_raw_pointers():
    """Call the library the way a foreign host would: plain pointers and sizes."""
    lib = _lib.load()
    ri = torch.tensor([0, 0, 0, 2, 2, 5], dtype=torch.int64, device=dev)
    out = torch.empty((6, 2), dtype=torch.int64, device=dev)
    ws = torch.empty(lib.nfa_pack_info_workspace_bytes(6), dtype=torch.uint8, device=dev)
    rc = lib.nfa_pack_info(6, ri.data_ptr(), 6, out.data_ptr(), ws.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert out.tolist() == [[0, 3], [3, 0], [3, 2], [5, 0], [5, 0], [5, 1]]
    assert lib.nfa_pack_info(6, ri.data_ptr(), 6, out.data_ptr() + 8, ws.data_ptr(), None) == -1  # misaligned output


# ---------------------------------------------------------------- the other traverse_grids modes (generic kernel)

def _cmp_traverse(orc, ro, rd, bins, aabbs, **kw):
    tkw = {k: (T(v) if isinstance(v, np.ndarray) else v) for k, v in kw.items()}
    iv, sm, term = nfa.traverse_grids(T(ro), T(rd), T(bins), T(aabbs), **tkw)
    o_iv, o_sm, o_term = orc.traverse_grids(ro, rd, bins, aabbs, **kw)
    np.testing.assert_array_equal(N(iv.packed_info), o_iv["packed_info"])
    np.testing.assert_array_equal(N(sm.packed_info), o_sm["packed_info"])
    np.testing.assert_array_equal(N(iv.vals), o_iv["vals"])
    np.testing.assert_array_equal(N(iv.is_left), o_iv["is_left"])
    np.testing.assert_array_equal(N(iv.is_right), o_iv["is_right"])
    np.testing.assert_array_equal(N(iv.ray_indices), o_iv["ray_indices"])
    np.testing.assert_array_equal(N(sm.vals), o_sm["vals"])
    np.testing.assert_array_equal(N(sm.is_valid), o_sm["is_valid"])
    np.testing.assert_array_equal(N(sm.ray_indices), o_sm["ray_indices"])
    d = ~np.isnan(o_term)
    np.testing.assert_array_equal(N(term)[d], o_term[d])
    return int(o_sm["packed_info"][:, 1].sum())


def test_traverse_grids_generic_modes(orc):
    rng = np.random.default_rng(21)
    R = 200
    ro = rng.standard_normal((R, 3)).astype(np.float32)
    rd = rng.standard_normal((R, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    bins4 = rng.random((4, 32, 32, 32)) > 0.5
    a4 = scenes.nested_aabbs(4)
    assert _cmp_traverse(orc, ro, rd, bins4, a4, step_size=5e-3, cone_angle=0.01) > 0
    assert _cmp_traverse(orc, ro, rd, bins4, a4, step_size=1e-2, cone_angle=0.004, near_planes=rng.random(R).astype(np.float32),
                         far_planes=(2 + rng.random(R)).astype(np.float32)) > 0
    assert _cmp_traverse(orc, ro, rd, bins4, a4, step_size=0.0) > 0       # one sample per occupied cell
    assert _cmp_traverse(orc, ro, rd, bins4[:1], a4[:1], step_size=-1.0) > 0
    mask = rng.random(R) > 0.3
    assert _cmp_traverse(orc, ro, rd, bins4, a4, step_size=1e-2, traverse_steps_limit=37, over_allocate=True, rays_mask=mask) > 0
    assert _cmp_traverse(orc, ro, rd, bins4, a4, step_size=1e-2, cone_angle=0.003, traverse_steps_limit=5, over_allocate=True) > 0
    assert _cmp_traverse(orc, ro, rd, bins4, a4, step_size=1e-2, traverse_steps_limit=50, rays_mask=mask) > 0
    # sampling() with a cone angle goes through the same kernel
    est = _estimator(bins4, a4)
    ri, ts, te = est.sampling(T(ro), T(rd), render_step_size=5e-3, cone_angle=0.01)
    o_ri, o_ts, o_te, _ = orc.occgrid_sampling(ro, rd, bins4, a4, render_step_size=5e-3, cone_angle=0.01)
    np.testing.assert_array_equal(N(ri), o_ri)
    np.testing.assert_array_equal(N(ts), o_ts)
    np.testing.assert_array_equal(N(te), o_te)


def test_reference_test_mode_marching():
    """reference tests/test_grid.py:72-131: two bounded rounds reproduce the one-shot traversal."""
    from nerfacc_b200.grid import _enlarge_aabb
    torch.manual_seed(42)
    n_rays = 10
    ro = torch.randn((n_rays, 3), device=dev)
    rd = torch.randn((n_rays, 3), device=dev)
    rd = rd / rd.norm(dim=-1, keepdim=True)
    base = torch.tensor([-1.0, -1.0, -1.0, 1.0, 1.0, 1.0], device=dev)
    aabbs = torch.stack([_enlarge_aabb(base, 2 ** i) for i in range(4)])
    binaries = torch.rand((4, 32, 32, 32), device=dev) > 0.5
    iv, sm, _ = nfa.traverse_grids(ro, rd, binaries, aabbs)
    ts, te = iv.vals[iv.is_left], iv.vals[iv.is_right]
    acc_s = nfa.accumulate_along_rays(ts, None, sm.ray_indices, n_rays)
    acc_e = nfa.accumulate_along_rays(te, None, sm.ray_indices, n_rays)
    _acc_s = _acc_e = 0.0
    term, mask = None, None
    for _ in range(2):
        _iv, _sm, term = nfa.traverse_grids(ro, rd, binaries, aabbs, near_planes=term, traverse_steps_limit=4000,
                                            over_allocate=True, rays_mask=mask)
        mask = _sm.packed_info[:, 1] == 4000
        _ri = _sm.ray_indices[_sm.is_valid]
        _acc_s = _acc_s + nfa.accumulate_along_rays(_iv.vals[_iv.is_left], None, _ri, n_rays)
        _acc_e = _acc_e + nfa.accumulate_along_rays(_iv.vals[_iv.is_right], None, _ri, n_rays)
    assert (~mask).all()
    assert torch.allclose(_acc_s, acc_s, atol=1e-1) and torch.allclose(acc_e, _acc_e, atol=1e-1)


def test_fused_visibility_compaction(orc):
    """sampling(sigma_fn=...) / (alpha_fn=...): fused mask + compaction vs masking the oracle's samples."""
    R = 2048
    ro, rd = scenes.ball_rays(R)
    bins, a1 = scenes.ball_grid(64), scenes.nested_aabbs(1)
    est = _estimator(bins, a1)
    est.occs.fill_(0.3)
    o_ri, o_ts, o_te, o_pi = orc.occgrid_sampling(ro, rd, bins, a1, render_step_size=1e-2)
    g = torch.Generator().manual_seed(2)
    sig_all = (30 * torch.rand(len(o_ri), generator=g)).to(dev)
    calls = []

    def sigma_fn(ts, te, ri):
        calls.append(ts.shape[0])
        return sig_all
    for eps, thre in [(1e-2, 0.0), (1e-3, 0.05), (0.0, 0.1)]:
        ri, ts, te = est.sampling(T(ro), T(rd), sigma_fn=sigma_fn, render_step_size=1e-2, early_stop_eps=eps, alpha_thre=thre)
        o = orc.composite(o_ts, o_te, N(sig_all), None, packed_info=o_pi)
        thre_eff = min(thre, 0.3) if thre > 0 else 0.0
        keep = o["trans"] >= eps
        if thre_eff > 0:
            keep &= o["alphas"] >= thre_eff
        # samples whose T / alpha sit within float noise of a threshold may flip
        border = (np.abs(o["trans"] - eps) < 2e-6) | ((thre_eff > 0) & (np.abs(o["alphas"] - thre_eff) < 2e-6))
        got = np.zeros(len(o_ri), bool)
        # map the kept samples back to positions through (ray, t_start), which is unique
        key_all = {(int(r), float(t)): i for i, (r, t) in enumerate(zip(o_ri, o_ts))}
        idx = np.array([key_all[(int(r), float(t))] for r, t in zip(N(ri), N(ts))], dtype=np.int64)
        got[idx] = True
        assert (got != keep)[~border].sum() == 0
        assert (np.diff(idx) > 0).all()                                   # order preserved, grouped by ray
        np.testing.assert_array_equal(N(te), o_te[idx])
        pk = N(nfa.pack_info(ri, R))
        np.testing.assert_array_equal(pk[:, 1], np.bincount(N(ri), minlength=R))
        np.testing.assert_array_equal(pk[:, 0], np.cumsum(pk[:, 1]) - pk[:, 1])
    assert calls and all(c == len(o_ri) for c in calls)
    # alpha_fn route
    al_all = (0.5 * torch.rand(len(o_ri), generator=g)).to(dev)
    ri, ts, te = est.sampling(T(ro), T(rd), alpha_fn=lambda a, b, c: al_all, render_step_size=1e-2, early_stop_eps=1e-2)
    _, oT = orc.render_weight_from_alpha(N(al_all), packed_info=o_pi)
    keep = oT >= 1e-2
    assert abs(int(keep.sum()) - ri.numel()) <= 3 and ri.numel() < len(o_ri)


def test_distortion_loss_matches_pairwise_definition():
    """nerfacc.distortion (losses.py:7-41) against the O(n^2) definition of the mip-NeRF 360 regulariser."""
    torch.manual_seed(0)
    cnts = torch.tensor([5, 0, 17, 1, 40], device=dev)
    ri = torch.repeat_interleave(torch.arange(5, device=dev), cnts)
    n = int(cnts.sum())
    edges = torch.rand(n, device=dev)
    ts = edges
    te = edges + 0.05 + 0.1 * torch.rand(n, device=dev)
    w = torch.rand(n, device=dev, requires_grad=True)
    loss = nfa.distortion(w, ts, te, ri, 5)
    assert loss.shape == (5, 1)
    loss.sum().backward()
    want = torch.zeros(5, dtype=torch.float64)
    wd, sd, ed = w.detach().double().cpu(), ts.double().cpu(), te.double().cpu()
    start = 0
    for r, c in enumerate(cnts.tolist()):
        ww, m = wd[start:start + c], 0.5 * (sd[start:start + c] + ed[start:start + c])
        pair = (ww[:, None] * ww[None, :] * (m[:, None] - m[None, :]).abs()).sum()
        want[r] = pair + ((ww ** 2) * (ed[start:start + c] - sd[start:start + c])).sum() / 3
        start += c
    # intervals of one ray are not ordered here, so only the ordered-midpoint identity the loss relies on is
    # checked on the sorted ray; the others are checked through the closed form below
    mids = 0.5 * (ts + te)
    closed = torch.zeros(5, dtype=torch.float64)
    start = 0
    for r, c in enumerate(cnts.tolist()):
        ww, m = wd[start:start + c], mids.double().cpu()[start:start + c]
        W = torch.cumsum(ww, 0) - ww
        M = torch.cumsum(ww * m, 0) - ww * m
        closed[r] = (2 * (ww * m * W - ww * M)).sum() + ((ww ** 2) * (ed[start:start + c] - sd[start:start + c])).sum() / 3
        start += c
    np.testing.assert_allclose(N(loss)[:, 0], closed.numpy(), rtol=1e-5, atol=1e-6)
    assert w.grad is not None and torch.isfinite(w.grad).all()
    # with midpoints sorted along the ray the closed form IS the pairwise definition
    order = torch.argsort(mids[:5])
    l2 = nfa.distortion(w.detach()[:5][order], ts[:5][order], te[:5][order], ri[:5], 1)
    np.testing.assert_allclose(N(l2)[0, 0], want[0].item(), rtol=1e-5, atol=1e-6)


def test_peer_mailbox_single_rank_roundtrip():
    """csrc/peer.cu on one rank: CUDA IPC export, post / sum kernels, ring wrap-around, status flag."""
    import torch.distributed as dist
    from nerfacc_b200 import parallel
    created = not dist.is_initialized()
    if created:
        import tempfile
        store = os.path.join(tempfile.mkdtemp(), "store")
        try:
            dist.init_process_group("nccl", init_method=f"file://{store}", world_size=1, rank=0,
                                    device_id=torch.device(dev))
        except Exception as exc:  # no usable NCCL in this environment: the mailbox needs a process group
            pytest.skip(f"cannot create a single-rank NCCL group: {exc}")
    try:
        mb = parallel.PeerMailbox.get(torch.device(dev))
        assert mb is not None, "CUDA IPC mailbox could not be created"
        tickets = []
        for k in range(3 * parallel.PeerMailbox.TURNS + 1):   # laps around the ring of turns
            v = torch.tensor(float(k) + 0.25, device=dev)
            tickets.append((mb.post(v), float(k) + 0.25))
            if len(tickets) > 2:                               # read two steps late
                t, want = tickets.pop(0)
                assert float(mb.collect(t, 2.0)) == 2.0 * want
        mb.check()
        # a turn whose tag never arrives: bounded wait, NaN and the status flag (kept short: own mailbox only)
    finally:
        parallel.PeerMailbox.shutdown()
        if created:
            dist.destroy_process_group()


def test_sampling_begin_end_matches_sampling():
    """The split call returns what sampling() returns, also with two traversals in flight and a filter at the end."""
    ro, rd = scenes.ball_rays(3000)
    est = _estimator(scenes.ball_grid(128), scenes.nested_aabbs(1))
    o, d = T(ro), T(rd)
    want = est.sampling(o, d, render_step_size=scenes.BALL_STEP)
    t1 = est.sampling_begin(o, d, render_step_size=scenes.BALL_STEP)
    t2 = est.sampling_begin(o[:1000], d[:1000], render_step_size=scenes.BALL_STEP, near_plane=3.6)
    t3 = est.sampling_begin(o, d, render_step_size=scenes.BALL_STEP)           # same shape as t1: second workspace
    mid = est.sampling(o[:1000], d[:1000], render_step_size=scenes.BALL_STEP, near_plane=3.6)  # a plain call in between
    got1, got3, got2 = est.sampling_end(t1), est.sampling_end(t3), est.sampling_end(t2)
    for a, b in zip(want, got1):
        assert torch.equal(a, b)
    for a, b in zip(want, got3):
        assert torch.equal(a, b)
    for a, b in zip(mid, got2):
        assert torch.equal(a, b)
    sig = lambda ts, te, ri: 20.0 + 0.0 * ts  # opaque after ~0.23 units: most of every ray is dropped
    f_want = est.sampling(o, d, sigma_fn=sig, render_step_size=scenes.BALL_STEP, early_stop_eps=1e-2)
    f_got = est.sampling_end(est.sampling_begin(o, d, render_step_size=scenes.BALL_STEP), sigma_fn=sig, early_stop_eps=1e-2)
    for a, b in zip(f_want, f_got):
        assert torch.equal(a, b)
    assert f_got[0].numel() < want[0].numel()
    with pytest.raises(ValueError):
        est.sampling_begin(o.cpu(), d.cpu())


# ---------------------------------------------------------------- round 2: advisor findings

def test_gradients_flow_through_t_and_prefix_trans():
    """render_*_from_density are differentiable in t_starts / t_ends / prefix_trans in the reference
    (volrend.py:271-277); the fused kernels treat them as constants, so such calls must take the ATen route."""
    torch.manual_seed(3)
    cnts = torch.tensor([7, 0, 33, 1, 64], device=dev)
    ri = torch.repeat_interleave(torch.arange(5, device=dev), cnts)
    n = int(cnts.sum())
    pi = nfa.pack_info(ri, 5)
    ts0 = torch.rand(n, device=dev)
    te0 = ts0 + 0.01 + 0.05 * torch.rand(n, device=dev)
    sig0 = 3 * torch.rand(n, device=dev)
    pre0 = 0.5 + 0.5 * torch.rand(n, device=dev)

    def plain(ts, te, sig, pre):  # per-ray loops, plain torch, float64
        w = []
        for r in range(5):
            s, c = int(pi[r, 0]), int(pi[r, 1])
            sd = (sig[s:s + c] * (te[s:s + c] - ts[s:s + c])).double()
            T = torch.exp(-(torch.cumsum(sd, 0) - sd)) * pre[s:s + c].double()
            w.append(T * (1 - torch.exp(-sd)))
        return torch.cat(w)

    for kw in (dict(packed_info=pi), dict(ray_indices=ri, n_rays=5)):
        leaves = [x.clone().requires_grad_(True) for x in (ts0, te0, sig0, pre0)]
        w, T, a = nfa.render_weight_from_density(leaves[0], leaves[1], leaves[2], prefix_trans=leaves[3], **kw)
        (w * torch.arange(n, device=dev)).sum().backward()
        ref_leaves = [x.clone().requires_grad_(True) for x in (ts0, te0, sig0, pre0)]
        (plain(*ref_leaves) * torch.arange(n, device=dev)).sum().backward()
        for got, want, name in zip(leaves, ref_leaves, ("t_starts", "t_ends", "sigmas", "prefix_trans")):
            assert got.grad is not None, name
            torch.testing.assert_close(got.grad, want.grad, atol=2e-4, rtol=2e-4, msg=name)
    # only t requires grad: the result must still carry a graph (the fused early-out must not swallow it)
    ts = ts0.clone().requires_grad_(True)
    T, a = nfa.render_transmittance_from_density(ts, te0, sig0, packed_info=pi)
    assert T.requires_grad and a.requires_grad
    col, op, dep, _ = nfa.rendering(ts, te0, ri, n_rays=5, rgb_sigma_fn=lambda a_, b_, c_: (torch.ones(n, 3, device=dev), sig0))
    assert col.requires_grad


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_sampling_on_a_device_that_is_not_current():
    """The totals event must be recorded on the stream of the tensors' device (advisor finding, grid.py)."""
    other = torch.device("cuda:1")
    ro, rd = scenes.ball_rays(2048)
    bins = scenes.ball_grid(64)
    with torch.cuda.device(0):
        est = nfa.OccGridEstimator(torch.from_numpy(scenes.ROI_AABB), resolution=64).to(other)
        est.binaries = torch.from_numpy(bins).to(other)
        a = est.sampling(torch.from_numpy(ro).to(other), torch.from_numpy(rd).to(other), render_step_size=1e-2)
        b = est.sampling(torch.from_numpy(ro[:1000]).to(other), torch.from_numpy(rd[:1000]).to(other), render_step_size=1e-2)
    with torch.cuda.device(1):
        c = est.sampling(torch.from_numpy(ro).to(other), torch.from_numpy(rd).to(other), render_step_size=1e-2)
    assert a[0].numel() > 0 and torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
    assert b[0].numel() > 0 and int(b[0].max()) < 1000


def test_two_streams_sampling_concurrently_do_not_share_scratch():
    """Workspaces and pinned count slots are per (device, stream): two streams sampling at once stay correct."""
    from nerfacc_b200 import grid as _grid
    bins = scenes.ball_grid(128)
    est = _estimator(bins, scenes.nested_aabbs(1))
    ro_a, rd_a = scenes.ball_rays(20000, seed=1)
    ro_b, rd_b = scenes.ball_rays(31000, seed=2)
    A, B = (T(ro_a), T(rd_a)), (T(ro_b), T(rd_b))
    want_a = est.sampling(*A, render_step_size=scenes.BALL_STEP)
    want_b = est.sampling(*B, render_step_size=scenes.BALL_STEP)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for _ in range(3):
        with torch.cuda.stream(s1):
            ta = est.sampling_begin(*A, render_step_size=scenes.BALL_STEP)
        with torch.cuda.stream(s2):
            tb = est.sampling_begin(*B, render_step_size=scenes.BALL_STEP)
        with torch.cuda.stream(s1):
            got_a = est.sampling_end(ta)
        with torch.cuda.stream(s2):
            got_b = est.sampling_end(tb)
        torch.cuda.synchronize()
        for g, w in zip(got_a + got_b, want_a + want_b):
            assert torch.equal(g, w)
    keys = {k for k in _grid._scratch_cache if k[0] == torch.device(dev)}
    assert len({k[1] for k in keys}) >= 3  # default stream + the two side streams each own a scratch


# ---------------------------------------------------------------- f4: grid maintenance kernels (csrc/occ_update.cu)

@pytest.mark.parametrize("case", ["warm", "sampled", "sampled_hi"])
def test_grid_update_kernels_match_oracle_and_reference_golden(orc, case):
    from nerfacc_b200.grid import _OccPack
    z = load_golden("ref_occ_update")
    before, ids, occ = z[case + "_occs_before"], z[case + "_ids"], z[case + "_occ"]
    occ_thre, decay = (float(v) for v in z[case + "_args"])
    lib = _lib.load()
    occs = T(before).clone()
    scratch = torch.empty(len(ids), dtype=torch.float32, device=dev)
    t_ids, t_occ = T(ids), T(occ)
    _lib.call("nfa_occ_ema_update", occs.device, len(ids), _lib.ptr(t_ids), _lib.ptr(t_occ), decay, _lib.ptr(occs),
              _lib.ptr(scratch))
    want = orc.occ_ema_update(before, ids, occ, decay)
    np.testing.assert_array_equal(N(occs), want)                     # bit-exact, duplicates included (largest wins)
    shape = z[case + "_binaries"].shape
    bins = torch.empty(shape, dtype=torch.bool, device=dev)
    pack = _OccPack(None, shape=shape, device=torch.device(dev))
    ws = torch.empty(lib.nfa_occ_threshold_workspace_bytes(occs.numel()), dtype=torch.uint8, device=dev)
    for _ in range(2):  # the workspace is reusable
        _lib.call("nfa_occ_threshold_pack", occs.device, *shape, _lib.ptr(occs), occ_thre, _lib.ptr(bins),
                  _lib.ptr(pack.words), _lib.ptr(pack.coarse), _lib.ptr(pack.bounds), _lib.ptr(ws))
    o_bins, o_thre = orc.occ_threshold(want, occ_thre)
    np.testing.assert_array_equal(N(bins).reshape(-1), o_bins.reshape(-1))
    assert np.float32(N(ws[16:20].view(torch.float32))[0]) == np.float32(o_thre)
    fresh = _OccPack(bins)                                            # what nfa_occ_pack builds from the bool grid
    assert torch.equal(pack.words, fresh.words) and torch.equal(pack.coarse, fresh.coarse)
    assert torch.equal(pack.bounds, fresh.bounds)
    # and on the reference's own `occs` the bool grid is the reference's
    occs2 = T(z[case + "_occs_after"])
    _lib.call("nfa_occ_threshold_pack", occs2.device, *shape, _lib.ptr(occs2), occ_thre, _lib.ptr(bins),
              _lib.ptr(pack.words), _lib.ptr(pack.coarse), _lib.ptr(pack.bounds), _lib.ptr(ws))
    np.testing.assert_array_equal(N(bins), z[case + "_binaries"])


def test_estimator_update_native_path_feeds_sampling():
    """_update on the GPU: same result as the reference's torch formulation on the same draws, and the packed grid
    it leaves behind is what sampling() would have built."""
    torch.manual_seed(11)
    est = nfa.OccGridEstimator(torch.from_numpy(scenes.ROI_AABB), resolution=32, levels=2).to(dev)
    est.train()

    def occ_eval_fn(x):
        return torch.exp(-6.0 * (x * x).sum(-1, keepdim=True)) * 0.05

    for step in (0, 300):
        before, bins_before = est.occs.clone(), est.binaries
        state = torch.cuda.get_rng_state()
        est._update(step=step, occ_eval_fn=occ_eval_fn, occ_thre=0.01, ema_decay=0.95, warmup_steps=256)
        got_occs, got_bins = est.occs.clone(), est.binaries.clone()
        assert getattr(est.binaries, "_nfa_occ", None) is not None    # derived cache attached by the kernel
        # replay with the reference's op sequence (occ_grid.py:367-404) on the same random draws
        torch.cuda.set_rng_state(state)
        est.occs.copy_(before)
        kernel_bins, est.binaries = est.binaries, bins_before          # the cell draw looks at the OLD grid
        per_level = est._get_all_cells() if step < 256 else est._sample_uniform_and_occupied_cells(est.cells_per_lvl // 4)
        est.binaries = kernel_bins
        for lvl, indices in enumerate(per_level):
            coords = est.grid_coords[indices]
            x = (coords + torch.rand_like(coords, dtype=torch.float32)) / est.resolution
            x = est.aabbs[lvl, :3] + x * (est.aabbs[lvl, 3:] - est.aabbs[lvl, :3])
            occ = occ_eval_fn(x).squeeze(-1)
            cell_ids = lvl * est.cells_per_lvl + indices
            new = torch.maximum(est.occs[cell_ids] * 0.95, occ)
            ref_occs = est.occs.clone()
            ref_occs.scatter_reduce_(0, cell_ids, torch.full_like(new, -float("inf")), "amin", include_self=True)
            ref_occs.scatter_reduce_(0, cell_ids, new, "amax", include_self=True)
            est.occs.copy_(ref_occs)
        assert torch.equal(est.occs, got_occs)
        thre = torch.clamp(est.occs[est.occs >= 0].double().mean().float(), max=0.01)
        assert torch.equal((est.occs > thre).view(got_bins.shape), got_bins)
    assert getattr(est.binaries, "_nfa_occ", None) is not None        # still the kernel-made pack
    ro, rd = scenes.ball_rays(4096)
    a = est.sampling(T(ro), T(rd), render_step_size=1e-2)
    est2 = nfa.OccGridEstimator(torch.from_numpy(scenes.ROI_AABB), resolution=32, levels=2).to(dev)
    est2.binaries = got_bins.clone()
    b = est2.sampling(T(ro), T(rd), render_step_size=1e-2)
    assert a[0].numel() > 0 and all(torch.equal(x, y) for x, y in zip(a, b))


def test_by_key_scan_single_pass_many_tiles():
    """The key-addressed scans run one tile of 2048 elements per CTA with decoupled look-back: segments that cross
    tile boundaries, segments longer than several tiles (the look-back chain), unaligned views (scalar loads), the
    reverse direction (autograd of the sum scans) -- against float64 cumulative sums / products per segment."""
    torch.manual_seed(5)
    cnts = torch.cat([torch.randint(0, 300, (400,)), torch.tensor([5000, 1, 0, 9000, 2047, 2048, 2049, 3]),
                      torch.randint(0, 64, (300,))]).to(dev)
    keys = torch.repeat_interleave(torch.arange(len(cnts), device=dev), cnts)
    n = keys.numel()
    assert n > 40 * 2048
    xs = torch.rand(n + 3, device=dev) * 0.2 + 0.9           # around 1: products stay in range
    starts = torch.cumsum(cnts, 0) - cnts
    for off in (0, 1):                                       # off = 1: 4-byte aligned views -> scalar path
        x = xs[off:off + n]
        k = keys.clone() if off == 0 else torch.cat([keys.new_zeros(1), keys])[1:]
        xd = x.double()
        cs = torch.cumsum(xd, 0)
        base = torch.where(starts > 0, cs[(starts - 1).clamp(min=0)], torch.zeros_like(cs[:1]))
        incl_sum = cs - torch.repeat_interleave(base, cnts)
        lg = torch.cumsum(torch.log(xd), 0)
        lbase = torch.where(starts > 0, lg[(starts - 1).clamp(min=0)], torch.zeros_like(lg[:1]))
        incl_prod = torch.exp(lg - torch.repeat_interleave(lbase, cnts))
        first = torch.zeros(n, dtype=torch.bool, device=dev)
        first[starts[cnts > 0]] = True
        excl_sum = torch.where(first, torch.zeros_like(incl_sum), torch.roll(incl_sum, 1))
        excl_prod = torch.where(first, torch.ones_like(incl_prod), torch.roll(incl_prod, 1))
        for name, want, tol in (("inclusive_sum", incl_sum, 2e-5), ("exclusive_sum", excl_sum, 2e-5),
                                ("inclusive_prod", incl_prod, 5e-4), ("exclusive_prod", excl_prod, 5e-4)):
            got = getattr(nfa, name)(x, indices=k)
            torch.testing.assert_close(got.double(), want, rtol=tol, atol=tol * 50, msg=f"{name} off={off}")
        # reverse direction through autograd: d/dx of sum(inclusive_sum * g) is the reverse inclusive sum of g
        xg = x.clone().requires_grad_(True)
        g = torch.rand(n, device=dev)
        (nfa.inclusive_sum(xg, indices=k) * g).sum().backward()
        gd = g.double()
        rcs = torch.flip(torch.cumsum(torch.flip(gd, [0]), 0), [0])
        ends = starts + cnts
        rbase = torch.where(ends < n, rcs[ends.clamp(max=n - 1)], torch.zeros_like(rcs[:1]))
        want_grad = rcs - torch.repeat_interleave(rbase, cnts)
        torch.testing.assert_close(xg.grad.double(), want_grad, rtol=2e-5, atol=1e-3)
