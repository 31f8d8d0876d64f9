"""Growing-step sampling (cone_angle > 0) on one GPU: the route through nfa_march / nfa_expand_samples with
cone_angle > 0 against the traverse_grids route it replaced, and against the reference CUDA build, on the 360-like
case of oracle/gen_golden_cone_gpu.py (65 536 rays, 4 x 128^3 levels, step 1e-3, cone 0.004, near 0.2).

    python scripts/cone_probe.py [--iters N] [--out FILE]   # prints JSON; --out: the result also as a JSON file

- sampling() per call: host clock around the call + a device synchronise, old and new route alternated in one
  process after warm-up, without and with the visibility filter (sigma_fn, alpha_thre 1e-2); median and spread.
- the reference CUDA build (oracle/_ref) on the same inputs, in a child process (its `nerfacc` package and this
  repository's must not meet in one interpreter).
- walk and expand kernel times from CUDA events over repeated launches through the sampling job's own launch
  methods (_MarchJob._launch_march / _expand_samples, the calls sampling() makes), the sample count N, and the expand's
  16 B/sample (int64 ray index + two float32) over its time next to a fill_ of the same number of bytes.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _inputs(dev):
    import ref_runner as rr
    from oracle.gen_golden_cone_gpu import CONE360 as c
    ro, rd = rr.scenes.ball_rays(c["rays"], seed=42)
    return c, rr, torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev), rr.grid_for(c), \
        rr.scenes.nested_aabbs(c["levels"])


def _time_calls(fns, iters):
    """{name: [seconds per call]}, the callables alternated call by call."""
    out = {k: [] for k in fns}
    for _ in range(iters):
        for k, f in fns.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            out[k].append(time.perf_counter() - t0)
    return out


def _summary(ts):
    a = np.array(ts) * 1e3
    return dict(median_ms=float(np.median(a)), p10_ms=float(np.percentile(a, 10)), p90_ms=float(np.percentile(a, 90)))


def _events(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters  # ms


def reference(iters):
    """Child process: the reference CUDA build on the same inputs."""
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import nerfacc as ref
    assert "oracle/_ref" in ref.__file__.replace("\\", "/"), ref.__file__
    dev = torch.device("cuda:0")
    c, rr, o, d, bins, aabbs = _inputs(dev)
    est = ref.OccGridEstimator(torch.from_numpy(aabbs[0]), resolution=c["res"], levels=c["levels"]).to(dev)
    est.binaries = torch.from_numpy(bins).to(dev)
    est.occs.fill_(c["occ_mean"])
    kw = dict(near_plane=c["near"], render_step_size=c["step"], cone_angle=c["cone"])
    fns = {"ref": lambda: est.sampling(o, d, **kw),
           "ref_filter": lambda: est.sampling(o, d, sigma_fn=rr.field_sigma, alpha_thre=c["thre"], **kw)}
    _time_calls(fns, 3)
    res = {k: _summary(v) for k, v in _time_calls(fns, iters).items()}
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", help="also write the result to this JSON file")
    ap.add_argument("--reference", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cone_probe: needs a CUDA device")
    if args.reference:
        return reference(args.iters)
    import nerfacc_b200 as nfa
    from nerfacc_b200.grid import _MarchJob, traverse_grids
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    card = q.stdout.strip()
    print(json.dumps(dict(card=card)), flush=True)

    c, rr, o, d, bins, aabbs = _inputs(dev)
    est = nfa.OccGridEstimator(torch.from_numpy(aabbs[0]), resolution=c["res"], levels=c["levels"]).to(dev)
    est.binaries = torch.from_numpy(bins).to(dev)
    est.occs.fill_(c["occ_mean"])
    kw = dict(near_plane=c["near"], render_step_size=c["step"], cone_angle=c["cone"])
    filt = dict(sigma_fn=rr.field_sigma, alpha_thre=c["thre"])

    def old(**extra):  # sampling(cone_angle > 0) before: traverse_grids + two mask-selects + the filter
        npl, fpl = est._ray_planes(o, c["near"], 1e10, None, None, False, c["step"], always=True)
        iv, sm, _ = traverse_grids(o, d, est.binaries, est.aabbs, near_planes=npl, far_planes=fpl,
                                   step_size=c["step"], cone_angle=c["cone"])
        return est._drop_invisible(sm.ray_indices, iv.vals[iv.is_left], iv.vals[iv.is_right], sm.packed_info,
                                   extra.get("sigma_fn"), None, 1e-4, extra.get("alpha_thre", 0.0))

    fns = {"old": lambda: old(), "new": lambda: est.sampling(o, d, **kw),
           "old_filter": lambda: old(**filt), "new_filter": lambda: est.sampling(o, d, **kw, **filt)}
    for a, b in (("old", "new"), ("old_filter", "new_filter")):  # same bits, at the timed size
        for x, y in zip(fns[a](), fns[b]()):
            assert torch.equal(x, y), (a, b)
    _time_calls(fns, 3)
    calls = {k: _summary(v) for k, v in _time_calls(fns, args.iters).items()}
    n = int(est.sampling(o, d, **kw)[0].numel())
    n_kept = int(est.sampling(o, d, **kw, **filt)[0].numel())

    # kernels alone, launched the way sampling() launches them (as bench.py times the constant-step ones)
    job = _MarchJob(o, d, est.binaries, est.aabbs, None, None, c["step"], None, None, None, want_intervals=False,
                    want_terminate=False, near_plane=c["near"], far_plane=1e10, cone_angle=c["cone"])
    job._launch_march()
    n_k, runs = job._read_totals()
    if runs > job.sc.run_capacity:  # run pool too small: march again with room for every run
        job.sc.reserve(o.shape[0], runs + 1024)
        job._launch_march()
        n_k, runs = job._read_totals()
    assert n_k == n, (n_k, n)

    fill_buf = torch.empty(16 * n, dtype=torch.uint8, device=dev)
    it = 200
    t_walk, t_expand = _events(job._launch_march, it), _events(lambda: job._expand_samples(n), it)
    job.sc.busy = False
    job.sc = None
    t_fill = _events(lambda: fill_buf.fill_(1), it)
    kernels = dict(n_samples=n, n_runs=runs, samples_per_run=n / max(runs, 1), walk_ms=t_walk, expand_ms=t_expand,
                   expand_GBps=16 * n / (t_expand * 1e-3) / 1e9, fill_same_bytes_ms=t_fill,
                   fill_GBps=16 * n / (t_fill * 1e-3) / 1e9)

    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--reference", "--iters", str(args.iters)],
                       capture_output=True, text=True)
    ref = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else dict(error=r.stderr[-2000:])

    res = dict(card=card, case=dict(c, kept_after_filter=n_kept), sampling_call=calls, reference_cuda=ref,
               kernels=kernels)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
