"""Kernel-level timing of the two fused compositing kernels on config 2 (8.5 M samples, 65536 rays), CUDA events,
L2 flushed between launches: the launches bench.py's roofline section makes, on their own.

    python scripts/composite_probe.py [REPS] [--offset K]

--offset K (1..3) stores every per-sample input and output K float32 elements past a 16-byte boundary, which
takes the element-wise kernels instead of the hot ones."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerfacc_b200 as nfa  # noqa: E402
from nerfacc_b200 import _lib, scenes  # noqa: E402

dev = torch.device("cuda:0")
ap = argparse.ArgumentParser()
ap.add_argument("reps", nargs="?", type=int, default=20)
ap.add_argument("--offset", type=int, default=0, choices=range(4))
args = ap.parse_args()
reps = args.reps
R = 65536
ro, rd = scenes.ball_rays(R)
est = nfa.OccGridEstimator(torch.from_numpy(scenes.ROI_AABB), resolution=128).to(dev)
est.binaries = torch.from_numpy(scenes.ball_grid(128)).to(dev)
ri, ts, te = est.sampling(torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev), render_step_size=scenes.BALL_STEP)
N = ri.numel()
pi = nfa.pack_info(ri, R)
f32 = dict(dtype=torch.float32, device=dev)


def place(t):  # a copy of t starting args.offset elements into its buffer
    buf = torch.empty(t.numel() + args.offset, **f32)
    v = buf[args.offset:].view(t.shape)
    v.copy_(t)
    return v


sg, cl, gcol = 5 * torch.rand(N, **f32), torch.rand(N, 3, **f32), torch.rand(R, 3, **f32)
ts, te, sg, cl = place(ts), place(te), place(sg), place(cl)
w_o, t_o, a_o = place(torch.empty(N, **f32)), place(torch.empty(N, **f32)), place(torch.empty(N, **f32))
c_o, o_o, d_o, raw = torch.empty((R, 3), **f32), torch.empty((R, 1), **f32), torch.empty((R, 1), **f32), torch.empty((R, 5), **f32)
g_sg, g_cl = place(torch.empty(N, **f32)), place(torch.empty((N, 3), **f32))
P = _lib.ptr
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def k_fwd():
    _lib.call("nfa_composite_fwd", dev, R, N, P(pi), P(ts), P(te), P(sg), 0, P(cl), None, None, 1, P(w_o), P(t_o), P(a_o),
              P(c_o), P(o_o), P(d_o), P(raw))


def k_bwd():
    _lib.call("nfa_composite_bwd", dev, R, N, P(pi), P(ts), P(te), P(sg), 0, P(cl), None, None, 1, P(raw), P(gcol), None,
              None, None, None, None, P(g_sg), P(g_cl))


def timed(fn):
    fn()
    tot = []
    for _ in range(reps):
        flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        tot.append(a.elapsed_time(b) * 1e3)
    tot.sort()
    return {"median_us": round(tot[len(tot) // 2], 1), "min_us": round(tot[0], 1)}


print(json.dumps({"n_samples": N, "offset": args.offset, "composite_fwd": timed(k_fwd), "composite_bwd": timed(k_bwd),
                  "checksum": [float(c_o.double().sum()), float(g_sg.double().sum())]}))
