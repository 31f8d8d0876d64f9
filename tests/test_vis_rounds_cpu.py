"""OccGridEstimator.sampling_until_opaque without a GPU: the nfa_vis_rounds_* entry points of the C ABI, their argument
errors and workspace sizes (on dummy pointers: every error is returned before a pointer is read), and the method's
CPU-tensor error."""
import pytest
import torch

import nerfacc_b200 as nfa
from nerfacc_b200 import _lib

ENTRY_POINTS = ("nfa_vis_rounds_workspace_bytes", "nfa_vis_rounds_begin", "nfa_vis_rounds_gather",
                "nfa_vis_rounds_step", "nfa_vis_rounds_finish")
P = 1 << 20  # a dummy, 16-byte aligned, non-null address


def test_entry_points_and_workspace_bytes():
    lib = _lib.load()
    assert _lib.ABI_VERSION == 15 and lib.nfa_version() == 15  # entry points added, nothing changed
    for name in ENTRY_POINTS:
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    ws = lib.nfa_vis_rounds_workspace_bytes
    assert ws(0, 10) == 0 and ws(-1, 10) == 0 and ws(10, -1) == 0
    for R, N in ((1, 0), (33, 1000), (65536, 8_513_610)):
        # two live lists, carry, done, counts, live flags, two (rank | offset, count) scans, per-slot counts, the mask
        per_ray = 2 * 4 + 4 + 8 + 8 + 8 + 16 + 8 + 16
        assert ws(R, N) >= per_ray * R + N
        assert ws(R, N) % 16 == 0
        assert ws(R, N + 16) - ws(R, N) == 16  # the mask is the only per-sample part


def test_argument_errors_do_not_need_a_gpu():
    lib = _lib.load()
    begin, gather, step, finish = (lib.nfa_vis_rounds_begin, lib.nfa_vis_rounds_gather, lib.nfa_vis_rounds_step,
                                   lib.nfa_vis_rounds_finish)
    assert begin(0, 10, P, 0, P, P, None) == -1        # no rays
    assert begin(8, -1, P, 0, P, P, None) == -1        # negative sample count
    assert begin(8, 10, None, 0, P, P, None) == -1
    assert begin(8, 10, P, 0, P + 4, P, None) == -1    # misaligned workspace
    assert begin(8, 10, P + 8, 0, P, P, None) == -1    # misaligned packed_info
    assert begin(8, 10, P, 0, P, None, None) == -1     # no status slot

    def g(R=8, N=10, rnd=0, alive=4, ws=P, out=P):
        return gather(R, N, rnd, alive, P, P, P, ws, out, P, P, None)

    for bad in (dict(R=0), dict(N=-1), dict(rnd=-1), dict(alive=0), dict(alive=9), dict(ws=None), dict(ws=P + 4),
                dict(out=None)):
        assert g(**bad) == -1, bad

    def s(R=8, N=10, rnd=0, alive=4, with_samples=6, dens=P, status=P):
        return step(R, N, rnd, alive, with_samples, P, P, P, dens, 0, 1e-4, 0.0, P, status, None)

    for bad in (dict(alive=0), dict(alive=9), dict(with_samples=3), dict(with_samples=9), dict(rnd=-1),
                dict(dens=None), dict(status=None)):
        assert s(**bad) == -1, bad
    assert finish(0, 10, P, P, P, P, P, P, P, P, None) == -1
    assert finish(8, 10, P, P, P, P, P + 8, P, P, P, None) == -1  # misaligned new packed_info
    assert finish(8, 10, P, P, P, P, P, None, P, P, None) == -1   # samples but no outputs


def test_cpu_tensors_are_not_implemented():
    est = nfa.OccGridEstimator([-1.0, -1.0, -1.0, 1.0, 1.0, 1.0], resolution=16)
    fn = lambda ts, te, ri: torch.zeros_like(ts)  # noqa: E731
    for kw in (dict(sigma_fn=fn), dict(alpha_fn=fn), dict(sigma_fn=fn, render_step_size=0.0), {}):
        with pytest.raises(NotImplementedError):
            est.sampling_until_opaque(torch.zeros(4, 3), torch.ones(4, 3), **kw)
    assert "sampling_until_opaque" not in dir(nfa)  # a method of the estimator only: nothing new at the package level
