"""Time an evaluation image three ways on one GPU (DESIGN.md section 9):

  render_test   OccGridEstimator.render_test (csrc/render_test.cu: one host wait per round)
  loop          the same test-mode loop over the public functions (traverse_grids test mode, mask-selects,
                render_weight_from_density, accumulate_along_rays_: examples/utils.py:267-439)
  occgrid       render_image_with_occgrid (examples/utils.py:54-167): sampling(sigma_fn=...) then rendering, in
                chunks of 8192 rays

on two workloads: an 800 x 800 pinhole image of the 128^3 ball scene, and BASELINE config 3 (256^3 ball grid,
1 048 576 rays of scenes.ball_rays).  The field is oracle/gen_golden_testmode_gpu.py's analytic ball, step 5.2e-3.
Each route: warm-up, then the median of --runs runs, each timed with CUDA events after a 256 MiB write that flushes
the L2; the number of samples handed to the field (field evaluations) is counted per route.

    python scripts/render_test_probe.py [--runs 20] [--out FILE.json]   # the report is printed; --out also saves it
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import nerfacc_b200 as nfa  # noqa: E402
from nerfacc_b200 import scenes  # noqa: E402
from nerfacc_b200.estimators.occ_grid import _render_test_public  # noqa: E402
from oracle.gen_golden_testmode_gpu import ball_field  # noqa: E402

STEP = scenes.BALL_STEP


def camera_rays(width, height, dist=4.0, focal=1.6):
    """Pinhole camera on the +z axis looking at the origin: one ray per pixel centre."""
    j, i = torch.meshgrid(torch.arange(height, dtype=torch.float32), torch.arange(width, dtype=torch.float32),
                          indexing="ij")
    x = (i + 0.5 - width / 2) / (width / 2)
    y = (j + 0.5 - height / 2) / (height / 2)
    d = torch.stack([x, y, torch.full_like(x, -focal)], -1).reshape(-1, 3)
    d = d / d.norm(dim=-1, keepdim=True)
    o = torch.tensor([0.0, 0.0, dist]).expand_as(d).contiguous()
    return o, d


def counted(fn, n):
    def g(t_starts, t_ends, ray_indices):
        n[0] += t_starts.shape[0]
        return fn(t_starts, t_ends, ray_indices)
    return g


def route_render_test(est, ro, rd, field, n):
    return est.render_test(ro, rd, counted(field, n), max_samples=1024, render_step_size=STEP)[:3]


def route_loop(est, ro, rd, field, n):
    return _render_test_public(est, ro, rd, counted(field, n), 1024, 0.0, 1e10, STEP, None, 0.0, 0.0, 1e-4)[:3]


def route_occgrid(est, ro, rd, field, n, chunk=8192):
    out = []
    for i in range(0, ro.shape[0], chunk):
        o, d = ro[i:i + chunk], rd[i:i + chunk]
        f = counted(ball_field(o, d), n)
        ri, ts, te = est.sampling(o, d, sigma_fn=lambda a, b, c: f(a, b, c)[1], render_step_size=STEP)
        col, op, dep, _ = nfa.rendering(ts, te, ri, n_rays=o.shape[0], rgb_sigma_fn=f)
        out.append((col, op, dep))
    return [torch.cat(x, 0) for x in zip(*out)]


ROUTES = {"render_test": route_render_test, "loop": route_loop, "occgrid": route_occgrid}


def workload(name, dev):
    if name == "image800":
        res, (ro, rd) = 128, camera_rays(800, 800)
    else:  # config 3
        res = 256
        ro, rd = (torch.from_numpy(a) for a in scenes.ball_rays(1 << 20, seed=42))
    est = nfa.OccGridEstimator(torch.from_numpy(scenes.ROI_AABB), resolution=res).to(dev)
    est.binaries = torch.from_numpy(scenes.ball_grid(res)).to(dev)
    return est, ro.to(dev), rd.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON report to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_test_probe: needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    report = {"gpu": gpu, "runs": args.runs, "step": STEP, "workloads": {}}
    for wl in ("image800", "config3"):
        est, ro, rd = workload(wl, dev)
        field = ball_field(ro, rd)
        res, outs = {}, {}
        for name, route in ROUTES.items():
            n = [0]
            outs[name] = route(est, ro, rd, field, n)  # warm-up
            evals = n[0]
            times = []
            for _ in range(args.runs):
                flush.fill_(1)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                route(est, ro, rd, field, [0])
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b))
            res[name] = {"median_ms": float(np.median(times)), "min_ms": float(np.min(times)),
                         "max_ms": float(np.max(times)), "field_evals": int(evals)}
            print(wl, name, res[name], flush=True)
        # the two test-mode routes compute the same image
        res["max_abs_diff_render_test_vs_loop"] = max(float((x - y).abs().max()) for x, y in
                                                     zip(outs["render_test"], outs["loop"]))
        res["max_abs_diff_opacity_render_test_vs_occgrid"] = float((outs["render_test"][1] - outs["occgrid"][1])
                                                                   .abs().max())
        res["n_rays"] = int(ro.shape[0])
        report["workloads"][wl] = res
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
