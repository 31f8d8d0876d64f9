"""The proposal loss on the GPU: `_pdf_loss` on batched float32 CUDA rows runs nfa_pdf_loss_fwd / nfa_pdf_loss_bwd.

Bars: the per-interval loss is `_pdf_loss_torch`'s bit for bit (NaN at the same positions); the key cdfs' gradient is
ATen's bit for bit at every key edge with at most one contribution per side, and elsewhere within the error of float32
summation of a float64 evaluation of the same sums; two backward passes give the same bits; PropNetEstimator's
training step returns the loss it returned with the ATen formulation, bit for bit."""
import numpy as np
import pytest
import torch

import nerfacc_b200.estimators.prop_net as pn
from nerfacc_b200 import _lib
from nerfacc_b200.data_specs import RayIntervals
from nerfacc_b200.estimators.prop_net import PropNetEstimator
from nerfacc_b200.pdf import importance_sampling, searchsorted
from test_prop_loss_cpu import loss_cases

pytestmark = pytest.mark.gpu
dev = "cuda:0"
EPS = 1e-7


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def same_or_nan(a, b):
    """NaN at the same positions; torch.equal on the rest."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return a.shape == b.shape and torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def _args(qv, qc, kv, kc, lead=None):
    t = [T(x) for x in (qv, qc, kv, kc)]
    if lead is not None:
        t = [x.reshape(lead + (x.shape[-1],)) for x in t]
    return RayIntervals(t[0]), t[1], RayIntervals(t[2]), t[3]


@pytest.mark.parametrize("eq", [2, 33, 49, 257])
@pytest.mark.parametrize("ek", [1, 2, 65, 97, 257, 3000])
def test_forward_matches_aten(eq, ek):
    rng = np.random.default_rng(eq * 10000 + ek)
    for R in (1, 31, 4097):
        for name, case in loss_cases(rng, R, eq, ek).items():
            args = _args(*case)
            n0 = _lib.launches
            got = pn._pdf_loss(*args)
            assert _lib.launches - n0 == 1, (R, name)
            assert same_or_nan(got, pn._pdf_loss_torch(*args)), (R, name)
    for name, case in loss_cases(rng, 6, eq, ek).items():  # any leading shape, flattened like pdf._layout does
        args = _args(*case, lead=(2, 3))
        got = pn._pdf_loss(*args)
        assert got.shape == (2, 3, eq - 1) and same_or_nan(got, pn._pdf_loss_torch(*args)), name


def _contributions(q, k, t):
    """Per key edge: the number of contributions of each side, the largest |term| and sum |term| over both sides, and
    the float64 sum (R side + L side) of the float32 terms t (d loss / d wo of each interval)."""
    left, right = searchsorted(k, q)
    left, right = left[..., :-1], right[..., 1:]
    shape = k.vals.shape
    z = lambda dt: torch.zeros(shape, dtype=dt, device=dev)  # noqa: E731
    n_r = z(torch.int64).scatter_add_(-1, right, torch.ones_like(right))
    n_l = z(torch.int64).scatter_add_(-1, left, torch.ones_like(left))
    a = t.abs().double()
    big = z(torch.float64).scatter_reduce_(-1, right, a, "amax").scatter_reduce_(-1, left, a, "amax")
    total_abs = z(torch.float64).scatter_add_(-1, right, a).scatter_add_(-1, left, a)
    exact = z(torch.float64).scatter_add_(-1, right, t.double()).scatter_add_(-1, left, -t.double())
    return n_r, n_l, big, total_abs, exact


@pytest.mark.parametrize("eq,ek", [(33, 65), (49, 97), (49, 257), (257, 65), (33, 3000), (2, 1), (257, 2)])
def test_key_gradient_matches_aten_autograd(eq, ek):
    rng = np.random.default_rng(eq + 7 * ek)
    torch.manual_seed(eq + 7 * ek)
    R = 4097
    for name, case in loss_cases(rng, R, eq, ek).items():
        q, cq, k, ck = _args(*case)
        g = torch.randn(R, eq - 1, device=dev)
        ck_n, ck_t = ck.clone().requires_grad_(True), ck.clone().requires_grad_(True)
        loss = pn._pdf_loss(q, cq, k, ck_n)
        n0 = _lib.launches
        loss.backward(g)
        assert _lib.launches - n0 == 1, name
        loss_t = pn._pdf_loss_torch(q, cq, k, ck_t)
        loss_t.backward(g)
        assert same_or_nan(loss.detach(), loss_t.detach()), name
        # the per-interval terms, as ATen's chain computes them
        left, right = searchsorted(k, q)
        wo = (ck.gather(-1, right[..., 1:]) - ck.gather(-1, left[..., :-1])).requires_grad_(True)
        w = cq[..., 1:] - cq[..., :-1]
        (torch.clip(w - wo, min=0) ** 2 / (w + EPS)).backward(g)
        n_r, n_l, big, total_abs, exact = _contributions(q, k, wo.grad)
        single = (n_r <= 1) & (n_l <= 1)
        assert single.any() or ek <= 2, name  # two key edges take every interval's contributions
        assert same_or_nan(ck_n.grad[single], ck_t.grad[single]), name
        # elsewhere: 1e-6 of the edge's largest contribution, or the worst-case error of m float32 additions when
        # that is larger (the R-side and L-side sums can cancel, so no bound relative to the result)
        m = (n_r + n_l).double()
        tol = torch.maximum(1e-6 * big, m * 2.0 ** -24 * total_abs)
        fin = torch.isfinite(exact)
        for got in (ck_n.grad, ck_t.grad):
            assert torch.equal(torch.isnan(got), ~fin), name
            assert torch.all((got.double() - exact).abs()[fin] <= tol[fin]), name


def _sorted_rows(R, e, gen):
    return torch.sort(torch.rand(R, e, device=dev, generator=gen), -1)[0]


@pytest.mark.parametrize("R,eq,eks", [(262144, 33, [65]), (8192, 49, [257, 97])])
def test_gradient_is_the_same_every_run_and_launch(R, eq, eks):
    """config 4 (262 144 rays, 32 samples from a 64-bin proposal) and the mip-NeRF 360 example's two levels: two
    backward passes, and a third over the first third of the rays alone (a smaller grid), give the same bits."""
    gen = torch.Generator(device=dev).manual_seed(eq)
    q, cq = _sorted_rows(R, eq, gen), _sorted_rows(R, eq, gen)
    g = torch.rand(R, eq - 1, device=dev, generator=gen)
    for ek in eks:
        k, ck = _sorted_rows(R, ek, gen), _sorted_rows(R, ek, gen)

        def grad(rows):
            leaf = ck[rows].clone().requires_grad_(True)
            pn._pdf_loss(RayIntervals(q[rows]), cq[rows], RayIntervals(k[rows]), leaf).backward(g[rows])
            return leaf.grad

        first, second, third = grad(slice(None)), grad(slice(None)), grad(slice(0, R // 3))
        assert torch.equal(first, second)
        assert torch.equal(third, first[: R // 3])
        assert (first != 0).any()


def _flattened(R, eq, k, ck, gen):
    """Flattened query intervals (per-ray counts: packed_info, is_left / is_right) with their cdfs, and the batched key
    rows `k`, `ck` as flattened ones (the branch the reference marks "not tested")."""
    iv = RayIntervals(vals=_sorted_rows(R, 9, gen))
    cnts = torch.randint(1, eq, (R,), device=dev, generator=gen)
    fq, _ = importance_sampling(iv, _sorted_rows(R, 9, gen), cnts)
    ek = k.shape[-1]
    starts = torch.arange(R, device=dev, dtype=torch.int64) * ek
    fk = RayIntervals(vals=k.reshape(-1), packed_info=torch.stack([starts, torch.full_like(starts, ek)], -1))
    return fq, torch.rand(fq.vals.shape, device=dev, generator=gen), fk, ck.reshape(-1)


def test_other_inputs_take_the_aten_formulation(monkeypatch):
    gen = torch.Generator(device=dev).manual_seed(1)
    R, eq, ek = 64, 17, 33
    q, cq, k, ck = (_sorted_rows(R, eq, gen), _sorted_rows(R, eq, gen), _sorted_rows(R, ek, gen),
                    _sorted_rows(R, ek, gen))
    fq, fcq, fk, fck = _flattened(R, eq, k, ck, gen)
    cases = {
        "cpu": (RayIntervals(q.cpu()), cq.cpu(), RayIntervals(k.cpu()), ck.cpu()),
        "float64": (RayIntervals(q.double()), cq.double(), RayIntervals(k.double()), ck.double()),
        "flattened query": (fq, fcq, fk, fck),
        "query cdfs need a gradient": (RayIntervals(q), cq.clone().requires_grad_(True), RayIntervals(k), ck),
    }
    torch_route = pn._pdf_loss_torch
    seen = []
    monkeypatch.setattr(pn, "_pdf_loss_torch", lambda *a: seen.append(1) or torch_route(*a))
    for name, args in cases.items():
        if name == "cpu":  # the native searchsorted is CUDA only; the ATen body says so as it always did
            with pytest.raises(NotImplementedError):
                pn._pdf_loss(*args)
            assert len(seen) == 1
            continue
        n0, before = _lib.launches, len(seen)
        got = pn._pdf_loss(*args)
        assert len(seen) == before + 1, name
        assert _lib.launches - n0 == 1, name  # its searchsorted
        assert torch.equal(got.detach(), torch_route(*args).detach()), name
    # the query-gradient case still differentiates both sides
    q_args = cases["query cdfs need a gradient"]
    pn._pdf_loss(*q_args).sum().backward()
    assert q_args[1].grad is not None
    # no gradient wanted: the native forward without an autograd node
    ckg = ck.clone().requires_grad_(True)
    with torch.no_grad():
        assert pn._pdf_loss(RayIntervals(q), cq, RayIntervals(k), ckg).grad_fn is None
    assert pn._pdf_loss(RayIntervals(q), cq, RayIntervals(k), ck).grad_fn is None
    assert pn._pdf_loss(RayIntervals(q), cq, RayIntervals(k), ckg).grad_fn is not None


def test_empty_inputs():
    gen = torch.Generator(device=dev).manual_seed(2)
    n0 = _lib.launches
    e = torch.empty(0, 5, device=dev)
    out = pn._pdf_loss(RayIntervals(e), e, RayIntervals(torch.empty(0, 9, device=dev)), torch.empty(0, 9, device=dev))
    assert out.shape == (0, 4) and _lib.launches == n0
    q1 = _sorted_rows(7, 1, gen)
    k, ck = _sorted_rows(7, 9, gen), _sorted_rows(7, 9, gen).requires_grad_(True)
    out = pn._pdf_loss(RayIntervals(q1), q1, RayIntervals(k), ck)
    assert out.shape == (7, 0) and _lib.launches == n0
    out.sum().backward()
    assert torch.equal(ck.grad, torch.zeros_like(ck))  # the backward writes the zeros ATen's gather backward gives


def _mlp_field(seed, width=32):
    g = torch.Generator().manual_seed(seed)
    params = [torch.nn.Parameter((torch.randn(1, width, generator=g) * 0.5).to(dev)),
              torch.nn.Parameter((torch.randn(width, generator=g) * 0.1 + 0.5).to(dev)),
              torch.nn.Parameter((torch.randn(width, 1, generator=g) * 0.5).to(dev))]

    def fn(t_starts, t_ends):
        mid = ((t_starts + t_ends) * 0.5).unsqueeze(-1)
        return torch.nn.functional.softplus(torch.relu(mid @ params[0] + params[1]) @ params[2]).squeeze(-1) * 4.0
    return params, fn


def _training_step(route, n_rays=4096):
    """One proposal update of the mip-NeRF 360 example's shapes (proposals of 256 and 96 samples, 48 final ones,
    loss_scaler 1024), from fixed parameters and a fixed seed."""
    torch.manual_seed(5)
    (p1, f1), (p2, f2) = _mlp_field(1), _mlp_field(2)
    opt = torch.optim.SGD(p1 + p2, lr=1e-5)
    est = PropNetEstimator(optimizer=opt).to(dev)
    ts, te = est.sampling([f1, f2], [256, 96], 48, n_rays=n_rays, near_plane=0.2, far_plane=1e3,
                          sampling_type="lindisp", stratified=True, requires_grad=True)
    mid = (ts + te) * 0.5
    sig = 3.0 * torch.exp(-((torch.log(mid) - 1.0) / 0.5) ** 2)
    trans = torch.exp(-torch.cumsum(torch.cat([torch.zeros_like(sig[:, :1]), (sig * (te - ts))[:, :-1]], -1), -1))
    saved = pn._pdf_loss
    pn._pdf_loss = route
    try:
        loss = est.update_every_n_steps(trans, requires_grad=True, loss_scaler=1024)
    finally:
        pn._pdf_loss = saved
    return loss, [p.detach().clone() for p in p1 + p2]


def _training_start():
    return [p.detach().clone() for p in _mlp_field(1)[0] + _mlp_field(2)[0]]


def test_propnet_step_matches_the_aten_step():
    loss_n, params_n = _training_step(pn._pdf_loss)
    loss_n2, params_n2 = _training_step(pn._pdf_loss)
    loss_t, params_t = _training_step(pn._pdf_loss_torch)
    assert loss_n > 0 and loss_n == loss_t  # the same float, bit for bit
    assert loss_n2 == loss_n
    moved = False
    for a, b, c, p0 in zip(params_n, params_n2, params_t, _training_start()):
        assert torch.equal(a, b)  # reproducible from run to run
        assert (a - c).abs().max() <= 1e-6 * c.abs().max()  # ATen's gradient adds with atomics in no fixed order
        moved = moved or not torch.equal(a, p0)
    assert moved


def test_peak_memory_below_the_aten_route():
    gen = torch.Generator(device=dev).manual_seed(4)
    R, eq, ek = 262144, 33, 65
    q, cq, k = _sorted_rows(R, eq, gen), _sorted_rows(R, eq, gen), _sorted_rows(R, ek, gen)
    ck0 = _sorted_rows(R, ek, gen)

    def peak(route):
        ck = ck0.clone().requires_grad_(True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        route(RayIntervals(q), cq, RayIntervals(k), ck).mean().backward()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    native, aten = peak(pn._pdf_loss), peak(pn._pdf_loss_torch)
    assert native < aten, (native, aten)
