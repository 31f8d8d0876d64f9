"""Golden digests of growing-step sampling (cone_angle > 0) from the UNMODIFIED reference CUDA build.

Run on a GPU box from the repo root, after `build()` made oracle/_ref:

    python oracle/gen_golden_cone_gpu.py OUT_DIR      # writes OUT_DIR/ref_live_cone360.npz

The case is nerfacc's unbounded-scene setting (examples/train_ngp_nerf_occ.py: 4 levels, render_step_size 1e-3,
cone_angle 0.004, near_plane 0.2) at 65 536 rays over four 128^3 levels (tests/ref_runner.py `grid_for`, the ball
scene's rays, whose origins lie inside levels 2 and 3): plain sampling, and sampling with a density field and
alpha_thre 1e-2.  Only SHA-256 digests, shapes and counts are stored (tests/ref_runner.py `sha`);
tests/test_gpu_cone_sampling.py runs `run_cone360` on the product and compares.  Nothing of nerfacc_b200 is imported
when this runs as a script.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ref_runner as rr  # noqa: E402

CONE360 = dict(res=128, levels=4, rays=65536, step=1e-3, cone=0.004, near=0.2, thre=1e-2, occ_mean=0.3)


def run_cone360(nf, dev) -> dict:
    """Both sampling calls of the case through package `nf` (reference or product: same public API)."""
    c = CONE360
    ro, rd = rr.scenes.ball_rays(c["rays"], seed=42)
    bins, aabbs = rr.grid_for(c), rr.scenes.nested_aabbs(c["levels"])
    est = nf.OccGridEstimator(torch.from_numpy(aabbs[0]), resolution=c["res"], levels=c["levels"]).to(dev)
    est.binaries = torch.from_numpy(bins).to(dev)
    est.occs.fill_(c["occ_mean"])
    tro, trd = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    kw = dict(near_plane=c["near"], render_step_size=c["step"], cone_angle=c["cone"])
    out = {}
    for tag, extra in (("", {}), ("vis_", dict(sigma_fn=rr.field_sigma, alpha_thre=c["thre"]))):
        ri, ts, te = est.sampling(tro, trd, **kw, **extra)
        pi = nf.pack_info(ri, c["rays"])
        out[tag + "n"] = np.int64(ri.numel())
        for k, v in (("ri", ri), ("ts", ts), ("te", te), ("packed_info", pi)):
            out[f"sha_{tag}{k}"] = np.asarray(rr.sha(v))
    return out


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit("usage: python oracle/gen_golden_cone_gpu.py OUT_DIR")
    out_dir = sys.argv[1]
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import nerfacc as ref
    assert "oracle/_ref" in ref.__file__.replace("\\", "/"), ref.__file__
    os.makedirs(out_dir, exist_ok=True)
    res = run_cone360(ref, torch.device("cuda:0"))
    np.savez_compressed(os.path.join(out_dir, "ref_live_cone360.npz"), **res)
    print("ok cone360", {k: (str(v) if v.ndim == 0 and v.dtype.kind == "i" else "sha") for k, v in res.items()})
