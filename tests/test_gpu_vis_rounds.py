"""OccGridEstimator.sampling_until_opaque (csrc/scan.cu, nfa_vis_rounds_*): the visibility filter with the field run in
rounds must keep exactly what `sampling(sigma_fn | alpha_fn, ...)` keeps -- bit for bit, with the same packed_info --
while handing the field each sample at most once, grouped by ray, in whole 32-sample blocks from the ray's first
sample; and the kept sets of the unmodified reference build (tests/golden/ref_live_vis_*.npz)."""
import os
import subprocess

import numpy as np
import pytest
import torch

import nerfacc_b200 as nfa
import ref_runner as rr
from conftest import ROOT, load_golden
from nerfacc_b200 import scenes
from nerfacc_b200.pack import _stashed_packed_info

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


def scene(res=128, levels=1, rays=65536, seed=42, flip_every=0):
    """ref_runner's grid (a ball at level 0, shell fragments outside) and the ball scene's rays; with `flip_every`,
    every flip_every-th ray points away and gets no samples."""
    ro, rd = scenes.ball_rays(rays, seed=seed)
    if flip_every:
        rd[::flip_every] *= -1.0
    est = nfa.OccGridEstimator(torch.from_numpy(scenes.nested_aabbs(levels)[0]), resolution=res, levels=levels).to(dev)
    est.binaries = torch.from_numpy(rr.grid_for(dict(res=res, levels=levels))).to(dev)
    return est, torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)


def opaque_field(ro, rd, scale=2000.0, radius=0.45):
    """The density of oracle/gen_golden_testmode_gpu.py `ball_field`, elementwise (no reduction over the axes)."""
    def fn(t_starts, t_ends, ray_indices):
        tm = (t_starts + t_ends) * 0.5
        o, d = ro[ray_indices], rd[ray_indices]
        x, y, z = o[:, 0] + d[:, 0] * tm, o[:, 1] + d[:, 1] * tm, o[:, 2] + d[:, 2] * tm
        return scale * torch.clamp(radius - torch.sqrt(x * x + y * y + z * z), min=0.0)
    return fn


def alpha_of(sigma_fn):
    def fn(t_starts, t_ends, ray_indices):
        return 1.0 - torch.exp(-sigma_fn(t_starts, t_ends, ray_indices) * (t_ends - t_starts))
    return fn


def recording(fn, log):
    def g(t_starts, t_ends, ray_indices):
        log.append((ray_indices.clone(), t_starts.clone(), t_ends.clone()))
        return fn(t_starts, t_ends, ray_indices)
    return g


class SampleIndex:
    """Position of every (ray, t_start) among the unfiltered samples of `sampling()`."""

    def __init__(self, est, ro, rd, **kw):
        self.ri, self.ts, self.te = est.sampling(ro, rd, **kw)
        self.pi = nfa.pack_info(self.ri, ro.shape[0])
        self.key = self._key(self.ri, self.ts)
        assert bool((self.key[1:] > self.key[:-1]).all())

    @staticmethod
    def _key(ri, ts):
        return ri.double() * 64.0 + ts.double()  # ts < 64 in these scenes: ray-major order, exact in float64

    def find(self, ri, ts):
        idx = torch.searchsorted(self.key, self._key(ri, ts))
        return idx.clamp(max=self.key.numel() - 1)

    def position(self, ri, ts):
        """Index of each sample within its ray."""
        return self.find(ri, ts) - self.pi[ri, 0]


def check_same(est, ro, rd, fn, alpha=False, reseed=None, **kw):
    """sampling() and sampling_until_opaque() on the same inputs: the same bits in all three outputs and in the
    stashed packed_info.  Returns (kept, what the closure got in each round)."""
    key = "alpha_fn" if alpha else "sigma_fn"
    if reseed is not None:
        torch.manual_seed(reseed)
    want = est.sampling(ro, rd, **{key: fn}, **kw)
    log = []
    if reseed is not None:
        torch.manual_seed(reseed)
    got = est.sampling_until_opaque(ro, rd, **{key: recording(fn, log)}, **kw)
    for a, b in zip(got, want):
        assert a.dtype == b.dtype and torch.equal(a, b)
    R = ro.shape[0]
    pw, pg = _stashed_packed_info(want[0], R), _stashed_packed_info(got[0], R)
    assert pw is not None and pg is not None and torch.equal(pg, pw)
    assert all(len(ri) > 0 for ri, _, _ in log)  # never called with zero samples
    return want, log


def check_handed_over(idx: SampleIndex, log):
    """Every call grouped by ray in ascending order; every sample one of sampling()'s, handed over at most once; per
    ray, the samples handed over are a prefix of whole 32-blocks (or all of the ray).  Returns the samples handed
    over in all."""
    seen = []
    for ri, ts, te in log:
        assert bool((ri[1:] >= ri[:-1]).all())
        k = idx.find(ri, ts)
        assert torch.equal(idx.ri[k], ri) and torch.equal(idx.ts[k], ts) and torch.equal(idx.te[k], te)
        assert bool((k[1:] > k[:-1]).all())  # each ray's samples in order
        seen.append(k)
    k = torch.cat(seen) if seen else torch.zeros(0, dtype=torch.int64, device=dev)
    assert torch.unique(k).numel() == k.numel()  # at most once
    R = idx.pi.shape[0]
    ray = idx.ri[k]
    got = torch.zeros(R, dtype=torch.int64, device=dev).index_add_(0, ray, torch.ones_like(ray))
    last = torch.full((R,), -1, dtype=torch.int64, device=dev).scatter_reduce_(0, ray, k - idx.pi[ray, 0], "amax")
    assert torch.equal(last + 1, got)  # a prefix of the ray
    n = idx.pi[:, 1]
    assert bool(((got % 32 == 0) | (got == n)).all())  # whole blocks, except where the ray ends
    return k.numel()


# ---------------------------------------------------------------------------------------------------------------
def test_reference_build_golden():
    """tests/ref_runner.py's vis cases through sampling_until_opaque: the reference build's kept set (SHA-256)."""
    for name in ("vis_ball", "vis_lvl4", "vis_alpha"):
        case, ref = rr.CASES[name], load_golden("ref_live_" + name)
        ro, rd, bins, aabbs = rr.make_inputs(case)
        est = nfa.OccGridEstimator(torch.from_numpy(aabbs[0]), resolution=case["res"], levels=case["levels"]).to(dev)
        est.binaries = torch.from_numpy(bins).to(dev)
        est.occs.fill_(case["occ_mean"])
        kw = dict(alpha_fn=rr.field_alpha) if case.get("alpha") else dict(sigma_fn=rr.field_sigma)
        ri, ts, te = est.sampling_until_opaque(torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev),
                                               render_step_size=case["step"], early_stop_eps=case["eps"],
                                               alpha_thre=case["thre"], **kw)
        got = {"ri": ri.cpu().numpy().astype(np.int32), "ts": ts.cpu().numpy(), "te": te.cpu().numpy()}
        for k, v in got.items():
            assert rr.sha(v) == str(ref["sha_" + k]), (name, k)


def test_config2_opaque_field_hands_over_under_half_of_the_samples():
    est, ro, rd = scene()
    idx = SampleIndex(est, ro, rd, render_step_size=scenes.BALL_STEP)
    want, log = check_same(est, ro, rd, opaque_field(ro, rd), render_step_size=scenes.BALL_STEP)
    handed = check_handed_over(idx, log)
    n = idx.ri.numel()
    # 8 513 610 marched samples; on an H100 the field saw 3 797 761 of them (0.446), in 3 rounds
    print(f"config 2, opaque field: {handed} of {n} samples ({handed / n:.3f}) in {len(log)} rounds, "
          f"{want[0].numel()} kept")
    assert handed < n // 2 and len(log) >= 2
    assert len(log[0][0]) == int(torch.clamp(idx.pi[:, 1], max=32).sum())  # round 0: every ray's first block


def test_config2_soft_field():
    est, ro, rd = scene()
    idx = SampleIndex(est, ro, rd, render_step_size=scenes.BALL_STEP)
    _, log = check_same(est, ro, rd, rr.field_sigma, render_step_size=scenes.BALL_STEP)
    handed = check_handed_over(idx, log)
    assert handed > 0.9 * idx.ri.numel()  # almost no ray retires


@pytest.mark.parametrize("alpha_thre", [0.0, 1e-2])
def test_four_levels_cone(alpha_thre):
    est, ro, rd = scene(res=64, levels=4, rays=8192)
    est.occs.fill_(0.3)
    kw = dict(render_step_size=1e-3, near_plane=0.2, cone_angle=0.004, alpha_thre=alpha_thre)
    idx = SampleIndex(est, ro, rd, render_step_size=1e-3, near_plane=0.2, cone_angle=0.004)
    for fn in (opaque_field(ro, rd), rr.field_sigma):
        _, log = check_same(est, ro, rd, fn, **kw)
        check_handed_over(idx, log)


@pytest.mark.parametrize("alpha_thre", [0.0, 1e-2])
def test_alpha_route(alpha_thre):
    est, ro, rd = scene(rays=16384)
    est.occs.fill_(0.5)
    idx = SampleIndex(est, ro, rd, render_step_size=scenes.BALL_STEP)
    for fn, eps in ((rr.field_alpha, 1e-2), (alpha_of(opaque_field(ro, rd)), 1e-4)):
        _, log = check_same(est, ro, rd, fn, alpha=True, render_step_size=scenes.BALL_STEP, early_stop_eps=eps,
                            alpha_thre=alpha_thre)
        check_handed_over(idx, log)


def test_alpha_thre_with_densities():
    est, ro, rd = scene(rays=16384)
    est.occs.fill_(0.3)
    for fn in (opaque_field(ro, rd), rr.field_sigma):
        check_same(est, ro, rd, fn, render_step_size=scenes.BALL_STEP, alpha_thre=1e-2, early_stop_eps=1e-3)


def test_t_min_t_max_and_stratified():
    est, ro, rd = scene(rays=16384)
    g = torch.Generator(device="cpu").manual_seed(5)
    t_min = (3.4 + torch.rand(ro.shape[0], generator=g)).to(dev)
    t_max = t_min + 0.2 + torch.rand(ro.shape[0], generator=g).to(dev)
    fn = opaque_field(ro, rd)
    check_same(est, ro, rd, fn, render_step_size=scenes.BALL_STEP, t_min=t_min, t_max=t_max)
    for seed in (0, 1):
        check_same(est, ro, rd, fn, reseed=seed, render_step_size=scenes.BALL_STEP, stratified=True)
        check_same(est, ro, rd, fn, reseed=seed, render_step_size=scenes.BALL_STEP, stratified=True, t_min=t_min,
                   t_max=t_max)


@pytest.mark.parametrize("R", [1, 33])
def test_small_batches_and_rays_without_samples(R):
    for flip in (0, 3):
        est, ro, rd = scene(rays=R, seed=3, flip_every=flip)
        for fn in (opaque_field(ro, rd), rr.field_sigma):
            check_same(est, ro, rd, fn, render_step_size=scenes.BALL_STEP)
    est, ro, rd = scene(rays=5000, flip_every=3)
    idx = SampleIndex(est, ro, rd, render_step_size=scenes.BALL_STEP)
    assert int((idx.pi[:, 1] == 0).sum()) >= 5000 // 3
    _, log = check_same(est, ro, rd, opaque_field(ro, rd), render_step_size=scenes.BALL_STEP)
    check_handed_over(idx, log)


@pytest.mark.parametrize("first_fail", [31, 32, 33])
def test_transmittance_first_fails_at_a_block_edge(first_fail):
    """A density spike at sample first_fail - 1 of every ray, zero elsewhere: T first fails at sample first_fail."""
    est, ro, rd = scene(rays=4096)
    idx = SampleIndex(est, ro, rd, render_step_size=scenes.BALL_STEP)

    def spike(t_starts, t_ends, ray_indices):
        j = idx.position(ray_indices, t_starts)
        return torch.where(j == first_fail - 1, 1e5, 0.0).float()

    _, log = check_same(est, ro, rd, spike, render_step_size=scenes.BALL_STEP)
    check_handed_over(idx, log)
    long_rays = idx.pi[:, 1] > first_fail
    first_round = torch.zeros(ro.shape[0], dtype=torch.int64, device=dev).index_add_(
        0, log[0][0], torch.ones_like(log[0][0]))
    assert bool((first_round[long_rays] == 32).all())
    later = torch.cat([ri for ri, _, _ in log[1:]]) if len(log) > 1 else log[0][0][:0]
    live_after_0 = torch.zeros(ro.shape[0], dtype=torch.bool, device=dev)
    live_after_0[later] = True
    # a spike at sample 30 or 31 ends the ray in round 0; at sample 32 it is only seen in round 1
    assert bool((live_after_0[long_rays] == (first_fail == 33)).all())


def test_nan_densities_and_an_all_zero_field():
    est, ro, rd = scene(rays=16384)
    base = opaque_field(ro, rd, scale=50.0)

    def with_nan(t_starts, t_ends, ray_indices):
        s = base(t_starts, t_ends, ray_indices)
        return torch.where((ray_indices % 7 == 3) & (t_starts > 3.7), float("nan"), s)

    check_same(est, ro, rd, with_nan, render_step_size=scenes.BALL_STEP)
    idx = SampleIndex(est, ro, rd, render_step_size=scenes.BALL_STEP)
    _, log = check_same(est, ro, rd, lambda ts, te, ri: torch.zeros_like(ts), render_step_size=scenes.BALL_STEP)
    assert check_handed_over(idx, log) == idx.ri.numel()  # nothing retires: the field sees every sample


def test_one_host_wait_per_round_and_no_other_sync(monkeypatch):
    est, ro, rd = scene()
    fn = opaque_field(ro, rd)
    est.sampling_until_opaque(ro, rd, sigma_fn=fn, render_step_size=scenes.BALL_STEP)  # workspaces exist now
    waits, calls = [], []
    real = torch.cuda.Event.synchronize
    monkeypatch.setattr(torch.cuda.Event, "synchronize", lambda self: (waits.append(1), real(self))[1])
    torch.cuda.set_sync_debug_mode("error")
    try:
        est.sampling_until_opaque(ro, rd, sigma_fn=recording(fn, calls), render_step_size=scenes.BALL_STEP,
                                  alpha_thre=0.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(calls) >= 2 and len(waits) == len(calls) + 2  # the march, one per round, one after the last


def test_two_streams_and_repeated_runs_are_bit_identical():
    est, ro, rd = scene(rays=32768)
    est2, ro2, rd2 = scene(res=64, levels=4, rays=8192, seed=5)
    kw = dict(sigma_fn=opaque_field(ro, rd), render_step_size=scenes.BALL_STEP)
    kw2 = dict(alpha_fn=rr.field_alpha, render_step_size=1e-3, near_plane=0.2, cone_angle=0.004, early_stop_eps=1e-2)
    want = est.sampling_until_opaque(ro, rd, **kw)
    want2 = est2.sampling_until_opaque(ro2, rd2, **kw2)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        got = est.sampling_until_opaque(ro, rd, **kw)
    with torch.cuda.stream(s2):
        got2 = est2.sampling_until_opaque(ro2, rd2, **kw2)
    torch.cuda.synchronize()
    again = est.sampling_until_opaque(ro, rd, **kw)
    for a, b in ((got, want), (got2, want2), (again, want)):
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def test_closure_outputs_must_be_float32():
    est, ro, rd = scene(res=64, rays=256)
    fn = opaque_field(ro, rd)
    for cast in (torch.Tensor.half, torch.Tensor.double):
        with pytest.raises(RuntimeError, match="float32"):
            est.sampling_until_opaque(ro, rd, sigma_fn=lambda *a: cast(fn(*a)), render_step_size=scenes.BALL_STEP)
    with pytest.raises(AssertionError, match="sigmas must have shape"):
        est.sampling_until_opaque(ro, rd, sigma_fn=lambda *a: fn(*a)[:, None], render_step_size=scenes.BALL_STEP)
    check_same(est, ro, rd, fn, render_step_size=scenes.BALL_STEP)  # still usable


def test_routes_that_are_sampling_itself():
    est, ro, rd = scene(rays=2048)
    fn = opaque_field(ro, rd)
    for kw in (dict(), dict(sigma_fn=fn, early_stop_eps=0.0, alpha_thre=1e-2), dict(sigma_fn=fn, render_step_size=0.0)):
        calls = []
        if "sigma_fn" in kw:
            kw["sigma_fn"] = recording(fn, calls)
        kw.setdefault("render_step_size", scenes.BALL_STEP)
        want = est.sampling(ro, rd, **kw)
        got = est.sampling_until_opaque(ro, rd, **kw)
        for a, b in zip(got, want):
            assert torch.equal(a, b)
        assert len(calls) in (0, 2)  # one closure call each


_EXP_CHECK = r"""
#include <cstdio>
#include <cstdint>
#include "vis_block.cuh"
__global__ void check(unsigned long long* bad)
{
    // every pair of consecutive non-negative floats x0 < x1 up to +inf: exp(-x1) <= exp(-x0), and 0 above 104
    const uint32_t n = 0x7f800000u;
    for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < n; b += gridDim.x * blockDim.x) {
        const float x0 = __uint_as_float(b), x1 = __uint_as_float(b + 1);
        const float y0 = nfa::vis_exp_neg(x0), y1 = nfa::vis_exp_neg(x1);
        if (!(y1 <= y0)) atomicAdd(bad, 1ull);
        if (x1 > 104.0f && y1 != 0.0f) atomicAdd(bad + 1, 1ull);
    }
}
int main()
{
    unsigned long long* d;
    unsigned long long h[2];
    cudaMalloc(&d, sizeof(h));
    cudaMemset(d, 0, sizeof(h));
    check<<<132 * 16, 256>>>(d);
    cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost);
    const cudaError_t e = cudaGetLastError();
    printf("%d %llu %llu\n", (int)e, h[0], h[1]);
    cudaFree(d);
    return e != cudaSuccess;
}
"""


def test_filter_exp_never_increases(tmp_path):
    """The density route retires a ray once exp(-carry) < early_stop_eps; that every later sample fails too rests on
    vis_exp_neg (the filter's expf, as compiled into the library) never increasing.  Checked for every float."""
    src = tmp_path / "exp_check.cu"
    src.write_text(_EXP_CHECK)
    exe = tmp_path / "exp_check"
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I",
                           os.path.join(ROOT, "nerfacc_b200", "csrc"), "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    err, increases, nonzero_above = (int(v) for v in out)
    assert err == 0 and increases == 0 and nonzero_above == 0
