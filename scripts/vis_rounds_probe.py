"""Time the visibility filter two ways on one GPU (DESIGN.md sections 4.12 and 9):

  sampling         OccGridEstimator.sampling(sigma_fn=...): the field on every marched sample, then the one-shot filter
  until_opaque     OccGridEstimator.sampling_until_opaque(sigma_fn=...): the field in rounds, rays retired once opaque

on the config-2 scene (65 536 rays of scenes.ball_rays, tests/ref_runner.py's 128^3 ball grid, step 5.2e-3), with
three fields:

  soft     tests/ref_runner.py `field_sigma` (density 1..7 everywhere): almost no ray becomes opaque
  opaque   the density of the analytic ball of oracle/gen_golden_testmode_gpu.py (scale 2000), elementwise
  mlp      a fixed-seed MLP (positional encoding, 3 x 64 ReLU, softplus density) standing in for a field of realistic
           cost; cuBLAS may pick different kernels for different batch sizes, so its kept set may differ

Per route and field: the median / min / max time per call over --runs calls (host clock around the call plus a device
synchronise, after a warm-up), the samples handed to the field, its calls (rounds) and the host waits; and whether the
two routes keep the same samples.  Also: the field's own time summed over the rounds (replayed on the recorded inputs),
the march alone, and what is left per round of sampling_until_opaque (gather, step, scans, one host wait), and the
time of zeroing the N-byte mask.

    python scripts/vis_rounds_probe.py [--runs 20] [--out FILE.json]   # the report is printed; --out also saves it
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

import nerfacc_b200 as nfa  # noqa: E402
import ref_runner as rr  # noqa: E402
from nerfacc_b200 import scenes  # noqa: E402

STEP = scenes.BALL_STEP


def opaque_field(ro, rd, scale=2000.0, radius=0.45):
    def fn(t_starts, t_ends, ray_indices):
        tm = (t_starts + t_ends) * 0.5
        o, d = ro[ray_indices], rd[ray_indices]
        x, y, z = o[:, 0] + d[:, 0] * tm, o[:, 1] + d[:, 1] * tm, o[:, 2] + d[:, 2] * tm
        return scale * torch.clamp(radius - torch.sqrt(x * x + y * y + z * z), min=0.0)
    return fn


def mlp_field(ro, rd, dev, width=64, n_freq=6):
    g = torch.Generator(device="cpu").manual_seed(0)
    dims = [3 + 6 * n_freq, width, width, width, 1]
    layers = [(torch.randn(a, b, generator=g) * (2.0 / a) ** 0.5, torch.zeros(b)) for a, b in zip(dims[:-1], dims[1:])]
    layers = [(w.to(dev), b.to(dev)) for w, b in layers]
    freqs = (2.0 ** torch.arange(n_freq, dtype=torch.float32)).to(dev)

    def fn(t_starts, t_ends, ray_indices):
        tm = ((t_starts + t_ends) * 0.5)[:, None]
        x = ro[ray_indices] + rd[ray_indices] * tm
        xf = (x[:, :, None] * freqs).reshape(x.shape[0], -1)
        h = torch.cat([x, torch.sin(xf), torch.cos(xf)], -1)
        for i, (w, b) in enumerate(layers):
            h = h @ w + b
            if i < len(layers) - 1:
                h = torch.relu(h)
        return torch.nn.functional.softplus(h[:, 0] - 1.0) * 50.0
    return fn


class Counter:
    def __init__(self, fn):
        self.fn, self.samples, self.calls, self.inputs = fn, 0, 0, None

    def __call__(self, t_starts, t_ends, ray_indices):
        self.samples += t_starts.shape[0]
        self.calls += 1
        if self.inputs is not None:
            self.inputs.append((t_starts.clone(), t_ends.clone(), ray_indices.clone()))
        return self.fn(t_starts, t_ends, ray_indices)


def timed(fn, runs):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": float(np.median(out)), "min_ms": float(np.min(out)), "max_ms": float(np.max(out))}


def count_waits(fn):
    waits = [0]
    real = torch.cuda.Event.synchronize

    def counting(self):
        waits[0] += 1
        return real(self)
    torch.cuda.Event.synchronize = counting
    try:
        res = fn()
    finally:
        torch.cuda.Event.synchronize = real
    return res, waits[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON report to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vis_rounds_probe: needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    case = rr.CASES["config2"]
    ro, rd, bins, aabbs = rr.make_inputs(case)
    est = nfa.OccGridEstimator(torch.from_numpy(aabbs[0]), resolution=case["res"], levels=case["levels"]).to(dev)
    est.binaries = torch.from_numpy(bins).to(dev)
    ro, rd = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    n_marched = est.sampling(ro, rd, render_step_size=STEP)[0].numel()
    report = {"gpu": gpu, "torch_gpu": torch.cuda.get_device_name(dev), "runs": args.runs, "n_rays": int(ro.shape[0]),
              "n_marched": int(n_marched), "fields": {}}
    report["march_only"] = timed(lambda: est.sampling(ro, rd, render_step_size=STEP), args.runs)
    mask = torch.empty(n_marched, dtype=torch.uint8, device=dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    mask.zero_()
    a.record()
    for _ in range(100):
        mask.zero_()
    b.record()
    b.synchronize()
    report["mask_zero_us"] = a.elapsed_time(b) * 10.0
    fields = {"soft": rr.field_sigma, "opaque": opaque_field(ro, rd), "mlp": mlp_field(ro, rd, dev)}
    for name, field in fields.items():
        res = {}
        outs = {}
        for route, method in (("sampling", est.sampling), ("until_opaque", est.sampling_until_opaque)):
            c = Counter(field)
            call = lambda: method(ro, rd, sigma_fn=c, render_step_size=STEP)  # noqa: E731
            outs[route], waits = count_waits(call)
            samples, calls = c.samples, c.calls
            res[route] = dict(timed(call, args.runs), field_samples=samples, rounds=calls, host_waits=waits)
            # the field alone on the same inputs, round by round
            c.inputs, c.samples, c.calls = [], 0, 0
            call()
            inputs = c.inputs
            res[route]["field_ms"] = timed(lambda: [field(*x) for x in inputs], args.runs)["median_ms"]
            print(name, route, res[route], flush=True)
        u = res["until_opaque"]
        u["per_round_ms"] = (u["median_ms"] - u["field_ms"] - report["march_only"]["median_ms"]) / max(u["rounds"], 1)
        res["identical"] = all(torch.equal(x, y) for x, y in zip(outs["sampling"], outs["until_opaque"]))
        if name == "mlp" and not res["identical"]:
            res["note"] = "cuBLAS results depend on the batch, so the kept sets may legitimately differ"
        res["field_samples_ratio"] = res["until_opaque"]["field_samples"] / max(res["sampling"]["field_samples"], 1)
        report["fields"][name] = res
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
