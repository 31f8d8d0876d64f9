"""The fused compositing kernels give the same bits whichever instantiation a call reaches: the hot one (density
route, every output), the general 16-byte-aligned one, and the element-wise one that inputs 4, 8 or 12 bytes off
alignment take.  Ragged rays put ray boundaries at every position inside a 4-sample group."""
import numpy as np
import pytest
import torch

from nerfacc_b200 import _lib

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
P = _lib.ptr
SPECIAL = [0, 1, 3, 4, 5, 31, 32, 33, 127, 128, 129, 250]


def _inputs(seed=21):
    rng = np.random.default_rng(seed)
    cnts = np.concatenate([np.tile(SPECIAL, 3), rng.integers(0, 80, 60)])
    rng.shuffle(cnts)
    cnts = torch.from_numpy(cnts.astype(np.int64))
    R, n = len(cnts), int(cnts.sum())
    g = torch.Generator().manual_seed(seed)
    rand = lambda *sh: torch.rand(*sh, generator=g).to(dev)  # noqa: E731
    ts = rand(n) * 0.5
    x = dict(pi=torch.stack([torch.cumsum(cnts, 0) - cnts, cnts], -1).to(dev), R=R, n=n, ts=ts,
             te=ts + 0.01 + rand(n) * 0.02, sig=8 * rand(n), alpha=0.3 * rand(n), rgb=rand(n, 3),
             bkgd=torch.tensor([0.2, 0.5, 0.9], device=dev), gC=rand(R, 3), gO=rand(R), gD=rand(R), gW=rand(n),
             gT=rand(n), gA=rand(n))
    return x


def _place(t, off):
    """A copy of `t` starting `off` float32 elements into its buffer (never an empty one: no null pointers)."""
    buf = torch.empty(t.numel() + off + 4, device=dev)
    v = buf[off:off + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _fwd(x, off, alpha_route, alphas_out=True):
    n, R = x["n"], x["R"]
    dens = _place(x["alpha"] if alpha_route else x["sig"], off)
    ts, te, rgb = _place(x["ts"], off), _place(x["te"], off), _place(x["rgb"], off)
    out = {k: _place(torch.full((n,), float("nan"), device=dev), off) for k in ("weights", "trans", "alphas")}
    out.update(colors=torch.empty(R, 3, device=dev), opac=torch.empty(R, device=dev),
               depths=torch.empty(R, device=dev), raw=torch.empty(R, 5, device=dev))
    if alpha_route or not alphas_out:
        out.pop("alphas")
    _lib.call("nfa_composite_fwd", dev, R, n, P(x["pi"]), P(ts), P(te), P(dens), int(alpha_route), P(rgb), None,
              P(x["bkgd"]), 1, P(out["weights"]), P(out["trans"]), P(out.get("alphas")), P(out["colors"]),
              P(out["opac"]), P(out["depths"]), P(out["raw"]))
    return {k: v.clone() for k, v in out.items()}


def _bwd(x, raw, off, alpha_route, extras, g_rgbs=True):
    n, R = x["n"], x["R"]
    dens = _place(x["alpha"] if alpha_route else x["sig"], off)
    ts, te, rgb = _place(x["ts"], off), _place(x["te"], off), _place(x["rgb"], off)
    gW, gT, gA = ((_place(x[k], off) for k in ("gW", "gT", "gA")) if extras else (None, None, None))
    g_in = _place(torch.full((n,), float("nan"), device=dev), off)
    g_rgb = _place(torch.full((n, 3), float("nan"), device=dev), off) if g_rgbs else None
    _lib.call("nfa_composite_bwd", dev, R, n, P(x["pi"]), P(ts), P(te), P(dens), int(alpha_route), P(rgb), None,
              P(x["bkgd"]), 1, P(raw), P(x["gC"]), P(x["gO"]), P(x["gD"]), P(gW), P(gT), P(gA), P(g_in), P(g_rgb))
    return {"g_in": g_in.clone()} if g_rgb is None else {"g_in": g_in.clone(), "g_rgbs": g_rgb.clone()}


def _assert_equal(a, b, what):
    for k in a:
        if k in b:
            assert torch.equal(a[k], b[k]), f"{what}: {k} differs, max |d| = {(a[k] - b[k]).abs().max().item()}"


@pytest.mark.parametrize("alpha_route", [False, True])
def test_compositing_bits_do_not_depend_on_route_or_alignment(alpha_route):
    x = _inputs()
    # forward: hot (density, every output) or vec (alpha route) at off = 0; the general aligned kernel without `alphas`
    ref = _fwd(x, 0, alpha_route)
    assert not any(v.isnan().any() for v in ref.values())
    if not alpha_route:
        _assert_equal(ref, _fwd(x, 0, alpha_route, alphas_out=False), "general aligned forward")
    for off in (1, 2, 3):  # 4 / 8 / 12 bytes off alignment: the element-wise kernel
        _assert_equal(ref, _fwd(x, off, alpha_route), f"forward, {4 * off}-byte offset")
    # backward, from the same saved sums: without and with gradients on weights / trans / alphas
    raw = ref["raw"]
    for extras in (False, True):
        want = _bwd(x, raw, 0, alpha_route, extras)
        assert not any(v.isnan().any() for v in want.values())
        if not alpha_route and not extras:
            # The element-wise kernel is the general one, so its g_in is compared with the general aligned kernel's
            # (reached by leaving out g_rgbs).  The hot kernel rounds g_in differently from that (by up to 3.5e-9
            # here, as it did before the kernels were merged); its g_rgbs must match exactly.
            gen = _bwd(x, raw, 0, alpha_route, extras, g_rgbs=False)
            torch.testing.assert_close(want["g_in"], gen["g_in"], rtol=1e-5, atol=1e-7)
            want["g_in"] = gen["g_in"]
        for off in (1, 2, 3):
            _assert_equal(want, _bwd(x, raw, off, alpha_route, extras), f"backward extras={extras}, {4 * off}-byte off")


@pytest.mark.parametrize("alpha_route", [False, True])
def test_compositing_rays_without_samples(alpha_route):
    """n_rays > 0 with n_samples == 0: zero opacity and depth, the background colour, a backward that succeeds, and
    nothing read or written per sample."""
    R = 37
    pi = torch.zeros(R, 2, dtype=torch.int64, device=dev)
    z = torch.zeros(16, device=dev)  # stands in for every per-sample array
    bk = torch.tensor([0.2, 0.5, 0.9], device=dev)
    c, op, dp, raw = (torch.full(sh, float("nan"), device=dev) for sh in [(R, 3), (R,), (R,), (R, 5)])
    _lib.call("nfa_composite_fwd", dev, R, 0, P(pi), P(z), P(z), P(z), int(alpha_route), P(z), None, P(bk), 1, P(z),
              P(z), None, P(c), P(op), P(dp), P(raw))
    assert torch.equal(op, torch.zeros(R, device=dev))
    assert torch.equal(dp, torch.zeros(R, device=dev))
    assert torch.equal(c, bk.expand(R, 3))
    assert torch.equal(raw, torch.zeros(R, 5, device=dev))
    gC, gO, gD = torch.rand(R, 3, device=dev), torch.rand(R, device=dev), torch.rand(R, device=dev)
    _lib.call("nfa_composite_bwd", dev, R, 0, P(pi), P(z), P(z), P(z), int(alpha_route), P(z), None, P(bk), 1, P(raw),
              P(gC), P(gO), P(gD), P(z), P(z), P(z), P(z), P(z))
    assert torch.equal(z, torch.zeros(16, device=dev))
