"""Golden digests of the test-mode rendering loop (nerfacc examples/utils.py:267-439) from the UNMODIFIED reference
CUDA build.

Run on a GPU box from the repo root, after `build()` made oracle/_ref:

    python oracle/gen_golden_testmode_gpu.py OUT_DIR      # writes OUT_DIR/ref_live_testmode.npz

`run_testmode_loop` restates that loop over a package's public functions (ray_aabb_intersect, traverse_grids in test
mode, render_weight_from_density with prefix_trans, accumulate_along_rays_); it runs unchanged on the reference and on
this package, and tests/test_gpu_render_test.py uses it as the fixture that OccGridEstimator.render_test is checked
against.  The stored cases are the 128^3 ball scene (one level, cone 0) and the ref_live_cone360 scene (four levels,
cone 0.004, near 0.2) with the analytic field `ball_field`: per round the number of samples per ray, the sample
count and SHA-256 digests of the closure's (ray_indices, t_starts, t_ends) (tests/ref_runner.py `sha`), then the
sample total and the colours, opacities and depths of every ray.  Nothing of nerfacc_b200 is imported when this runs as
a script.
"""
import os
import sys
from importlib import import_module

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ref_runner as rr  # noqa: E402

# rendering options of each golden case (render_test's keyword arguments)
GOLDEN = {
    "ball": dict(scene=dict(res=128, levels=1, rays=4000), max_samples=1024, render_step_size=5e-3,
                 render_bkgd=(0.2, 0.4, 0.6), alpha_thre=0.0),
    "cone360": dict(scene=dict(res=128, levels=4, rays=2000), max_samples=1024, render_step_size=1e-3,
                    near_plane=0.2, cone_angle=0.004, alpha_thre=1e-2),
}


def scene(nf, dev, res, levels, rays, seed=42):
    """(estimator, rays_o, rays_d): tests/ref_runner.py `grid_for` (a ball at level 0, fragments of shells outside)
    and the ball scene's rays."""
    ro, rd = rr.scenes.ball_rays(rays, seed=seed)
    case = dict(res=res, levels=levels)
    est = nf.OccGridEstimator(torch.from_numpy(rr.scenes.nested_aabbs(levels)[0]), resolution=res,
                              levels=levels).to(dev)
    est.binaries = torch.from_numpy(rr.grid_for(case)).to(dev)
    return est, torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)


def ball_field(rays_o, rays_d, scale=2000.0, radius=0.45):
    """Deterministic analytic field: density `scale * max(radius - |x|, 0)`, colour 0.5 + 0.5 sin(5 x + 1) at the
    sample's midpoint x.  The same torch ops on both packages give the same bits."""
    def fn(t_starts, t_ends, ray_indices):
        tm = ((t_starts + t_ends) * 0.5)[:, None]
        x = rays_o[ray_indices] + rays_d[ray_indices] * tm
        r = (x * x).sum(-1).sqrt()
        return 0.5 + 0.5 * torch.sin(5.0 * x + 1.0), scale * torch.clamp(radius - r, min=0.0)
    return fn


def recording(fn, log):
    """`fn`, logging a copy of every call's (ray_indices, t_starts, t_ends)."""
    def g(t_starts, t_ends, ray_indices):
        log.append((ray_indices.clone(), t_starts.clone(), t_ends.clone()))
        return fn(t_starts, t_ends, ray_indices)
    return g


@torch.no_grad()
def run_testmode_loop(nf, est, rays_o, rays_d, rgb_sigma_fn, max_samples, near_plane=0.0, far_plane=1e10,
                  render_step_size=1e-3, render_bkgd=None, cone_angle=0.0, alpha_thre=0.0, early_stop_eps=1e-4):
    """The test-mode loop over package `nf`'s public functions.  Returns (colors, opacities, depths, total_samples,
    n_samples of every round, live rays when the loop stopped)."""
    accumulate_along_rays_ = import_module(nf.__name__ + ".volrend").accumulate_along_rays_  # not exported
    R = rays_o.shape[0]
    dev = rays_o.device
    opacity = torch.zeros(R, 1, device=dev)
    depth = torch.zeros(R, 1, device=dev)
    rgb = torch.zeros(R, 3, device=dev)
    alive = torch.ones(R, device=dev, dtype=torch.bool)
    min_samples = 1 if cone_angle == 0 else 4
    spent, total, rounds = 0, 0, []
    near = torch.full_like(rays_o[:, 0], near_plane)
    far = torch.full_like(rays_o[:, 0], far_plane)
    t_mins, t_maxs, hits = nf.ray_aabb_intersect(rays_o, rays_d, est.aabbs)
    G = est.binaries.shape[0]
    if G > 1:
        t_sorted, t_indices = torch.sort(torch.cat([t_mins, t_maxs], -1), -1)
    else:
        t_sorted = torch.cat([t_mins, t_maxs], -1)
        t_indices = torch.arange(2 * G, device=dev, dtype=torch.int64).expand(R, 2 * G)
    n_alive = R
    while spent < max_samples:
        n_alive = int(alive.sum().item())
        if n_alive == 0:
            break
        n_samples = max(min(R // n_alive, 64), min_samples)
        spent += n_samples
        rounds.append(n_samples)
        iv, sm, term = nf.traverse_grids(rays_o, rays_d, est.binaries, est.aabbs, near, far, render_step_size,
                                         cone_angle, n_samples, True, alive, t_sorted, t_indices, hits)
        ts, te = iv.vals[iv.is_left], iv.vals[iv.is_right]
        ri = sm.ray_indices[sm.is_valid]
        rgbs, sigmas = rgb_sigma_fn(ts, te, ri)
        w, _, a = nf.render_weight_from_density(ts, te, sigmas, ray_indices=ri, n_rays=R,
                                                prefix_trans=1 - opacity[ri].squeeze(-1))
        if alpha_thre > 0:
            keep = a >= alpha_thre
            ri, rgbs, w, ts, te = ri[keep], rgbs[keep], w[keep], ts[keep], te[keep]
        accumulate_along_rays_(w, values=rgbs, ray_indices=ri, outputs=rgb)
        accumulate_along_rays_(w, values=None, ray_indices=ri, outputs=opacity)
        accumulate_along_rays_(w, values=(ts + te)[..., None] / 2.0, ray_indices=ri, outputs=depth)
        near = term
        alive = (opacity.view(-1) <= 1 - early_stop_eps) & (sm.packed_info[:, 1] == n_samples)
        total += ri.shape[0]
        n_alive = int(alive.sum().item())
    if render_bkgd is not None:
        rgb = rgb + render_bkgd * (1.0 - opacity)
    depth = depth / opacity.clamp_min(torch.finfo(torch.float32).eps)
    return rgb, opacity, depth, total, rounds, n_alive


def golden_case(nf, name, dev, run=None) -> dict:
    """Case `name` of GOLDEN through `run(est, rays_o, rays_d, fn, **options) -> (colors, opacities, depths, total)`
    (default: run_testmode_loop over `nf`), reduced to what the golden file keeps."""
    opts = dict(GOLDEN[name])
    est, ro, rd = scene(nf, dev, **opts.pop("scene"))
    if opts.get("render_bkgd") is not None:
        opts["render_bkgd"] = torch.tensor(opts["render_bkgd"], device=dev)
    log = []
    fn = recording(ball_field(ro, rd), log)
    if run is None:
        run = lambda *a, **k: run_testmode_loop(nf, *a, **k)[:4]  # noqa: E731
    col, op, dep, total = run(est, ro, rd, fn, **opts)
    N = lambda t: t.detach().cpu().numpy()  # noqa: E731
    return {
        "counts": np.asarray([len(ri) for ri, _, _ in log], dtype=np.int64),
        "sha_rounds": np.asarray([rr.sha(ri) + rr.sha(ts) + rr.sha(te) for ri, ts, te in log]),
        "total": np.int64(total),
        "colors": N(col), "opacities": N(op), "depths": N(dep),
    }


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit("usage: python oracle/gen_golden_testmode_gpu.py OUT_DIR")
    out_dir = sys.argv[1]
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import nerfacc as ref
    assert "oracle/_ref" in ref.__file__.replace("\\", "/"), ref.__file__
    os.makedirs(out_dir, exist_ok=True)
    res = {}
    for name in GOLDEN:
        for k, v in golden_case(ref, name, torch.device("cuda:0")).items():
            res[f"{name}_{k}"] = v
        print("ok", name, "rounds", len(res[f"{name}_counts"]), "samples", res[f"{name}_counts"].sum(),
              "total", int(res[f"{name}_total"]), flush=True)
    np.savez_compressed(os.path.join(out_dir, "ref_live_testmode.npz"), **res)
