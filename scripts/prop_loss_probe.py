"""Timing of PropNetEstimator.compute_loss + backward with the native proposal loss and with the ATen formulation it
replaces (`_pdf_loss_torch`), alternated in one process: config 4 (262 144 rays, one 64-sample proposal level, 32 final
samples) and the mip-NeRF 360 example's two levels (256 and 96 proposal samples, 48 final ones, 4 096 rays).

Per route and workload the median of RUNS CUDA-event times with the L2 flushed before each (min and max beside it),
after a warm-up.  `--profile` instead counts the kernels of one call per route with torch.profiler and sums their
device time.  Prints one JSON line per row; the card's name, power limit and max SM clock come from nvidia-smi in the
same run.

    python scripts/prop_loss_probe.py [--runs 20] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerfacc_b200.estimators.prop_net as pn  # noqa: E402
from nerfacc_b200.data_specs import RayIntervals  # noqa: E402

dev = torch.device("cuda:0")
# name -> (rays, final samples, proposal samples per level)
WORKLOADS = {"config4": (262144, 32, [64]), "example_two_levels": (4096, 48, [256, 96])}
ROUTES = {"native": pn._pdf_loss, "aten": pn._pdf_loss_torch}


def level_bytes(R, eq, ek):
    """Algorithmic bytes of one level: forward reads both rows of edges and cdfs and writes the losses; the backward
    also reads the upstream gradient and writes the key cdfs' gradient."""
    fwd = R * (2 * eq + 2 * ek) * 4 + R * (eq - 1) * 4
    return {"fwd": fwd, "bwd": fwd + R * (eq - 1) * 4 + R * ek * 4}


def make(R, n, levels):
    g = torch.Generator(device=dev).manual_seed(0)

    def rows(e):
        return torch.sort(torch.rand(R, e, device=dev, generator=g), -1)[0]

    keys = [(rows(m + 1), rows(m + 1).requires_grad_(True)) for m in levels]
    query = rows(n + 1)
    trans = 1.0 - rows(n)
    return keys, query, trans


def step(est, keys, query, trans):
    for k, ck in keys:
        ck.grad = None
        est.prop_cache.append((RayIntervals(k), ck))
    est.prop_cache.append((RayIntervals(query), None))
    est.compute_loss(trans, loss_scaler=1024.0).backward()


def with_route(route, fn):
    saved = pn._pdf_loss
    pn._pdf_loss = route
    try:
        return fn()
    finally:
        pn._pdf_loss = saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          "0"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": torch.cuda.get_device_name(dev), "nvidia_smi": smi, "runs": args.runs}))
    est = pn.PropNetEstimator().to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for name, (R, n, levels) in WORKLOADS.items():
        keys, query, trans = make(R, n, levels)
        shapes = [level_bytes(R, n + 1, m + 1) for m in levels]
        if args.profile:
            row = {"workload": name}
            for route, fn in ROUTES.items():
                with_route(fn, lambda: step(est, keys, query, trans))  # warm-up outside the trace
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    with_route(fn, lambda: step(est, keys, query, trans))
                    torch.cuda.synchronize()
                kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                           and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
                row[f"{route}_kernels"] = len(kernels)
                row[f"{route}_kernel_us"] = round(sum(e.device_time_total for e in kernels), 1)
                row[f"{route}_kernel_names"] = sorted({e.name[:60] for e in kernels})
                loss_us = {}
                for e in kernels:
                    if "pdf_loss" in e.name:
                        loss_us[e.name[:40]] = round(loss_us.get(e.name[:40], 0.0) + e.device_time_total, 1)
                row[f"{route}_loss_kernels_us"] = loss_us
            print(json.dumps(row))
            continue
        times = {route: [] for route in ROUTES}
        for route, fn in ROUTES.items():
            for _ in range(3):
                with_route(fn, lambda: step(est, keys, query, trans))
        for _ in range(args.runs):
            for route, fn in ROUTES.items():  # alternated
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                with_route(fn, lambda: step(est, keys, query, trans))
                b.record()
                b.synchronize()
                times[route].append(a.elapsed_time(b))
        row = {"workload": name, "n_rays": R, "query_edges": n + 1, "key_edges": [m + 1 for m in levels],
               "bytes_per_level": shapes}
        for route, t in times.items():
            t.sort()
            row[f"{route}_ms"] = {"median": round(t[len(t) // 2], 4), "min": round(t[0], 4), "max": round(t[-1], 4)}
        total = sum(s["fwd"] + s["bwd"] for s in shapes)
        row["native_GBps_of_algorithmic_bytes"] = round(total / row["native_ms"]["median"] / 1e6, 1)
        print(json.dumps(row))


if __name__ == "__main__":
    main()
