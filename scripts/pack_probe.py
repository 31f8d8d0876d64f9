"""Call-level timing of unpack_info / unpack_data / pack_data (and the two backwards) on the config-2 layout of
bench.py (ball scene, 65 536 rays, ~8.5 M samples, per-sample rows of 3 float32), next to the plain-torch formulation
of each and a fill_ of the same output bytes (bench.py's write-only yardstick).  Median of CUDA-event times over REPS
calls, L2 flushed before each call; GB/s from the algorithmic bytes.  Prints one JSON line per row.

    python scripts/pack_probe.py [REPS]
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerfacc_b200 as nfa  # noqa: E402
from nerfacc_b200 import pack, scenes  # noqa: E402

dev = torch.device("cuda:0")
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 50
R = 65536
ro, rd = scenes.ball_rays(R)
est = nfa.OccGridEstimator(torch.from_numpy(scenes.ROI_AABB), resolution=128, levels=1).to(dev)
est.binaries = torch.from_numpy(scenes.ball_grid(128)).to(dev)
ri, ts, te = est.sampling(torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev), render_step_size=scenes.BALL_STEP)
N = ri.numel()
pi = nfa.pack_info(ri, R)
S = int(pi[:, 1].max())
x = torch.rand(N, 3, device=dev)
padded = nfa.unpack_data(pi, x, S)
mask = torch.arange(S, device=dev) < pi[:, 1:]  # the prefix mask: pack_data(unpack_data(x)) == x
K = int(mask.sum())
g_padded = torch.rand(R, S, 3, device=dev)
g_packed = torch.rand(K, 3, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
ROW = 12


def torch_unpack_info():
    out = torch.full((N,), -1, dtype=torch.int64, device=dev)
    out[:] = torch.repeat_interleave(torch.arange(R, device=dev), pi[:, 1], output_size=N)
    return out


def torch_unpack_data():
    out = torch.zeros((R, S, 3), device=dev)
    valid = torch.arange(S, device=dev) < pi[:, 1:]
    out[valid] = x[(pi[:, :1] + torch.arange(S, device=dev))[valid]]
    return out


def torch_pack_data():
    counts = mask.sum(-1)
    return padded[mask], torch.stack([torch.cumsum(counts, 0) - counts, counts], -1)


def torch_pack_rows():  # unpack_data's backward as torch would run it (index_put's backward)
    valid = torch.arange(S, device=dev) < pi[:, 1:]
    out = torch.zeros((N, 3), device=dev)
    out.index_put_(((pi[:, :1] + torch.arange(S, device=dev))[valid],), g_padded[valid], accumulate=True)
    return out


def torch_unpack_masked():  # pack_data's backward as torch would run it (masked scatter into zeros)
    out = torch.zeros((R, S, 3), device=dev)
    out[mask] = g_packed
    return out


def fill(nbytes):
    buf = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    return lambda: buf.fill_(1)


# name -> (native, torch formulation, algorithmic bytes, output bytes)
ROWS = {
    "unpack_info": (lambda: nfa.unpack_info(pi, N), torch_unpack_info, 8 * N + 16 * R, 8 * N),
    "unpack_data": (lambda: nfa.unpack_data(pi, x, S), torch_unpack_data, ROW * N + ROW * R * S + 16 * R,
                    ROW * R * S),
    "pack_data": (lambda: nfa.pack_data(padded, mask), torch_pack_data, R * S + 2 * ROW * K + 16 * R, ROW * K + 16 * R),
    "unpack_data.backward": (lambda: pack._PackRows.apply(g_padded, pi, N), torch_pack_rows,
                             ROW * N + ROW * N + 16 * R, ROW * N),
    "pack_data.backward": (lambda: pack._UnpackMasked.apply(g_packed, mask, pi, S), torch_unpack_masked,
                           R * S + ROW * K + ROW * R * S + 16 * R, ROW * R * S),
}


def median_ms(fn):
    for _ in range(3):
        fn()
    times = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": torch.cuda.get_device_name(dev), "nvidia_smi": smi, "n_rays": R, "n_samples": N,
                      "max_count": S, "row_bytes": ROW, "reps": reps}))
    for name, (native, ref, nbytes, out_bytes) in ROWS.items():
        t_n, t_t, t_f = median_ms(native), median_ms(ref), median_ms(fill(out_bytes))
        print(json.dumps({"call": name, "bytes": nbytes, "native_ms": round(t_n, 4),
                          "native_GBps": round(nbytes / t_n / 1e6, 1), "torch_ms": round(t_t, 4),
                          "torch_GBps": round(nbytes / t_t / 1e6, 1), "fill_ms": round(t_f, 4),
                          "fill_GBps": round(out_bytes / t_f / 1e6, 1), "speedup_vs_torch": round(t_t / t_n, 2)}))


if __name__ == "__main__":
    main()
