"""CPU checks of the proposal loss (PropNetEstimator.compute_loss's `_pdf_loss`): the arithmetic of csrc/pdf.cuh,
compiled for the host by tests/host_sim/pdf_loss_sim.cpp in the order the two kernels of pdf.cu apply it, bit-exact
against the ATen formulation (`_pdf_loss_torch`, with the oracle's searchsorted) and its CPU autograd; and the C ABI's
argument errors of nfa_pdf_loss_fwd / nfa_pdf_loss_bwd."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import nerfacc_b200.estimators.prop_net as pn
from nerfacc_b200 import _lib
from nerfacc_b200.data_specs import RayIntervals

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = C.POINTER(C.c_float)
I64 = C.POINTER(C.c_int64)
P = 1 << 20  # a dummy, 16-byte aligned, non-null address
EPS = 1e-7


def loss_cases(rng, R, eq, ek):
    """name -> (query edges, query cdfs, key edges, key cdfs), float32 (R, eq) / (R, ek): the input families the CPU
    and GPU tests share."""
    def rows(n, e, lo=0.0, hi=1.0):
        return np.sort(rng.uniform(lo, hi, (n, e)), -1).astype(np.float32)

    cases = {"sorted": (rows(R, eq), rows(R, eq), rows(R, ek), rows(R, ek))}
    # query edges past both ends of the key range: clipped ids
    cases["outside"] = (rows(R, eq, -0.5, 1.5), rows(R, eq), rows(R, ek, 0.2, 0.8), rows(R, ek))
    # flat query cdfs (w = 0, so 0 / eps) and key cdfs with plateaus
    qc = np.repeat(rng.uniform(0, 1, (R, 1)).astype(np.float32), eq, -1)
    kc = rows(R, ek)
    kc[:, ek // 3: 2 * ek // 3] = kc[:, ek // 3: ek // 3 + 1]
    cases["flat"] = (rows(R, eq), qc, rows(R, ek), kc)
    # d exactly 0: dyadic key cdfs, query cdfs built from the envelope so that w == wo (every sum exact)
    qv, kv = rows(R, eq), rows(R, ek)
    kc = np.sort(rng.integers(0, 65, (R, ek)), -1).astype(np.float32) / 64
    pos = np.stack([np.searchsorted(kv[r, :ek - 1], qv[r], side="right") for r in range(R)])
    left, right = np.clip(pos - 1, 0, ek - 1), np.clip(pos, 0, ek - 1)
    wo = np.take_along_axis(kc, right[:, 1:], -1) - np.take_along_axis(kc, left[:, :-1], -1)
    qc = np.concatenate([np.zeros((R, 1)), np.cumsum(wo, -1)], -1).astype(np.float32)
    qc[::2, 1:] += np.float32(1 / 128)  # every other ray: w > wo in its first interval, d == 0 in the others
    cases["d_zero"] = (qv, qc, kv, kc)
    # NaN anywhere
    nan = [rows(R, eq), rows(R, eq), rows(R, ek), rows(R, ek)]
    for a in nan:
        a[rng.random(a.shape) < 0.03] = np.nan
    cases["nan"] = tuple(nan)
    # unsorted keys (edges and cdfs): ids follow the search's probe order
    cases["unsorted_keys"] = (rows(R, eq), rows(R, eq), rng.uniform(0, 1, (R, ek)).astype(np.float32),
                              rng.uniform(0, 1, (R, ek)).astype(np.float32))
    return cases


def same_bits_or_nan(a, b):
    """NaN at the same positions, every other element equal (a signed zero equals zero, as in torch.equal)."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)],
                                                                                            b[~np.isnan(b)])


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "host_sim", "pdf_loss_sim.cpp")
    so = str(tmp_path_factory.mktemp("pdf_loss_sim") / "libpdf_loss_sim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                           "-Wno-unknown-pragmas", "-o", so, src])
    return C.CDLL(so)


@pytest.fixture
def oracle_searchsorted(orc, monkeypatch):
    """`_pdf_loss_torch` on CPU tensors, its searchsorted answered by the oracle."""
    def cpu_searchsorted(key, query):
        left, right = orc.searchsorted(np.ascontiguousarray(key.vals.numpy()),
                                       np.ascontiguousarray(query.vals.numpy()))
        return torch.from_numpy(left), torch.from_numpy(right)

    monkeypatch.setattr(pn, "searchsorted", cpu_searchsorted)


def _p(a, t):
    return a.ctypes.data_as(t)


def sim_fwd(sim, qv, qc, kv, kc):
    R, eq, ek = qv.shape[0], qv.shape[1], kv.shape[1]
    loss = np.zeros((R, eq - 1), np.float32)
    left, right = np.zeros((R, eq - 1), np.int64), np.zeros((R, eq - 1), np.int64)
    sim.sim_pdf_loss_fwd(C.c_int64(R), eq, _p(qv, F), _p(qc, F), ek, _p(kv, F), _p(kc, F), C.c_float(EPS),
                         _p(loss, F), _p(left, I64), _p(right, I64))
    return loss, left, right


def sim_bwd(sim, qv, qc, kv, kc, g):
    R, eq, ek = qv.shape[0], qv.shape[1], kv.shape[1]
    gk = np.full((R, ek), np.nan, np.float32)
    sim.sim_pdf_loss_bwd(C.c_int64(R), eq, _p(qv, F), _p(qc, F), ek, _p(kv, F), _p(kc, F), C.c_float(EPS),
                         _p(np.ascontiguousarray(g, np.float32), F), _p(gk, F))
    return gk


def torch_loss_and_grad(qv, qc, kv, kc, g):
    ck = torch.from_numpy(kc.copy()).requires_grad_(True)
    loss = pn._pdf_loss_torch(RayIntervals(torch.from_numpy(qv)), torch.from_numpy(qc),
                              RayIntervals(torch.from_numpy(kv)), ck, EPS)
    loss.backward(torch.from_numpy(g))
    return loss.detach().numpy(), ck.grad.numpy()


SHAPES = [(2, 2), (2, 1), (33, 65), (49, 97), (49, 257), (9, 3), (65, 17)]


@pytest.mark.parametrize("eq,ek", SHAPES)
def test_forward_and_gradient_match_aten_on_cpu(sim, oracle_searchsorted, eq, ek):
    rng = np.random.default_rng(eq * 1000 + ek)
    for name, (qv, qc, kv, kc) in loss_cases(rng, 24, eq, ek).items():
        g = rng.standard_normal((24, eq - 1)).astype(np.float32)
        g[:, ::5] = 0.0
        want, want_gk = torch_loss_and_grad(qv, qc, kv, kc, g)
        got, left, right = sim_fwd(sim, qv, qc, kv, kc)
        assert same_bits_or_nan(got, want), name
        gk = sim_bwd(sim, qv, qc, kv, kc, g)
        # edges with at most one contribution per side: the same bits as ATen, whatever order it sums in
        single = np.ones((24, ek), bool)
        for r in range(24):
            for ids in (left[r], right[r]):
                single[r, np.bincount(ids, minlength=ek) > 1] = False
        assert single.any(), name
        assert same_bits_or_nan(gk[single], want_gk[single]), name
        # ATen's CPU scatter_add also adds in ascending j, so on the CPU every edge matches
        assert same_bits_or_nan(gk, want_gk), name


def test_cases_cover_what_they_name(sim):
    rng = np.random.default_rng(3)
    cases = loss_cases(rng, 16, 33, 65)
    qv, qc, kv, kc = cases["outside"]
    _, left, right = sim_fwd(sim, qv, qc, kv, kc)
    assert (left == 0).any() and (right == 64).any()
    qv, qc, kv, kc = cases["d_zero"]
    w = qc[:, 1:] - qc[:, :-1]
    loss, left, right = sim_fwd(sim, qv, qc, kv, kc)
    wo = np.take_along_axis(kc, right, -1) - np.take_along_axis(kc, left, -1)
    assert ((w == wo) & (w > 0)).sum() > 100 and (w > wo).any()
    assert np.all(loss[w == wo] == 0)
    qv, qc, kv, kc = cases["flat"]
    loss, _, _ = sim_fwd(sim, qv, qc, kv, kc)
    assert np.all(loss == 0)
    assert np.isnan(sim_fwd(sim, *cases["nan"])[0]).any()


def test_gradient_term_matches_autograd_elementwise(sim):
    """d loss / d wo of pdf.cuh against torch's CPU autograd of clip(w - wo, min=0) ** 2 / (w + eps), element by
    element, over random values, w = 0, d = 0, d < 0, NaN and a zero upstream gradient."""
    rng = np.random.default_rng(11)
    n = 200_000
    w = rng.uniform(0, 1, n).astype(np.float32)
    wo = (rng.uniform(-0.3, 1, n)).astype(np.float32)
    g = (rng.standard_normal(n) * 3).astype(np.float32)
    w[:500] = 0
    wo[500:1000] = w[500:1000]
    g[1000:1500] = 0
    w[1500:1600] = np.nan
    wo[1600:1700] = np.nan
    g[1700:1800] = np.nan
    loss, gwo = np.zeros(n, np.float32), np.zeros(n, np.float32)
    sim.sim_pdf_loss_terms(C.c_int64(n), _p(w, F), _p(wo, F), _p(g, F), C.c_float(EPS), _p(loss, F), _p(gwo, F))
    tw, two = torch.from_numpy(w), torch.from_numpy(wo).requires_grad_(True)
    want = torch.clip(tw - two, min=0) ** 2 / (tw + EPS)
    want.backward(torch.from_numpy(g))
    assert same_bits_or_nan(loss, want.detach().numpy())
    assert same_bits_or_nan(gwo, two.grad.numpy())


def test_abi_entry_points_and_argument_errors():
    lib = _lib.load()
    for name in ("nfa_pdf_loss_fwd", "nfa_pdf_loss_bwd"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    header = open(os.path.join(ROOT, "include", "nerfacc_b200.h")).read()
    assert int(re.search(r"#define NFA_PDF_LOSS_MAX_INTERVALS (\d+)", header).group(1)) == _lib.PDF_LOSS_MAX_INTERVALS

    def fwd(R=4, eq=9, ek=5, qv=P, qc=P, kv=P, kc=P, out=P):
        return lib.nfa_pdf_loss_fwd(R, eq, qv, qc, ek, kv, kc, EPS, out, None)

    def bwd(R=4, eq=9, ek=5, qv=P, qc=P, kv=P, kc=P, g=P, out=P):
        return lib.nfa_pdf_loss_bwd(R, eq, qv, qc, ek, kv, kc, EPS, g, out, None)

    for call in (fwd, bwd):
        for bad in (dict(R=-1), dict(eq=0), dict(eq=-3), dict(ek=0), dict(ek=-1), dict(qv=None), dict(qc=None),
                    dict(kv=None), dict(kc=None), dict(out=None)):
            assert call(**bad) == -1, (call.__name__, bad)
        assert call(R=0) == 0  # nothing to do, nothing read
    assert bwd(g=None) == -1
    assert fwd(eq=1) == 0  # no intervals: the forward writes nothing
    assert bwd(eq=_lib.PDF_LOSS_MAX_INTERVALS + 2) == -2
    assert bwd(R=0, eq=_lib.PDF_LOSS_MAX_INTERVALS + 2) == -2


def test_cpu_and_float64_take_the_aten_formulation(oracle_searchsorted, monkeypatch):
    rng = np.random.default_rng(2)
    qv, qc, kv, kc = loss_cases(rng, 6, 9, 17)["sorted"]
    calls = []
    monkeypatch.setattr(_lib, "call", lambda *a: calls.append(a))
    for dt in (torch.float32, torch.float64):
        args = (RayIntervals(torch.from_numpy(qv).to(dt)), torch.from_numpy(qc).to(dt),
                RayIntervals(torch.from_numpy(kv).to(dt)), torch.from_numpy(kc).to(dt))
        assert torch.equal(pn._pdf_loss(*args), pn._pdf_loss_torch(*args))
    assert calls == []
