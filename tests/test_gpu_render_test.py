"""OccGridEstimator.render_test (csrc/render_test.cu) against the test-mode loop of nerfacc's examples restated over
this package's public functions (oracle/gen_golden_testmode_gpu.py `run_testmode_loop`), and against the same loop run by
the unmodified reference build (tests/golden/ref_live_testmode.npz).

Per call: the same rounds with the same n_samples, the same samples handed to the field in every round (bit for bit),
the same sample total, and colours / opacities / depths within 1e-5.  The samples stay bit-exact only while no ray
ends a round with an opacity within rounding distance of 1 - early_stop_eps (DESIGN.md section 4.11): the field is
dense enough (`ball_field`, 2 000 per unit depth at the centre) that opacities jump past the threshold."""
import numpy as np
import pytest
import torch

import nerfacc_b200 as nfa
from conftest import load_golden
from nerfacc_b200.estimators import occ_grid
from oracle.gen_golden_testmode_gpu import GOLDEN, ball_field, golden_case, recording, scene, run_testmode_loop

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

SCENES = {
    "lvl1": dict(scene=dict(res=128, levels=1, rays=5000), render_step_size=5e-3),
    "cone4": dict(scene=dict(res=128, levels=4, rays=5000), render_step_size=1e-3, near_plane=0.2, cone_angle=0.004),
}


def _round_samples(log):
    """Like `recording`, but logs n_samples of the round too: render_test's pinned status slot holds it while the
    field runs."""
    def wrap(fn):
        def g(t_starts, t_ends, ray_indices):
            sc = occ_grid._rt_scratch[(dev, nfa._lib.stream_ptr(dev))]
            log.append(int(sc.status_np[1]))
            return fn(t_starts, t_ends, ray_indices)
        return g
    return wrap


def check(est, ro, rd, field, **opts):
    """render_test and the fixture on the same inputs; returns the fixture's (rounds, live rays at the end, log)."""
    want_log, got_log, got_ns = [], [], []
    want = run_testmode_loop(nfa, est, ro, rd, recording(field, want_log), **opts)
    got = est.render_test(ro, rd, _round_samples(got_ns)(recording(field, got_log)), **opts)
    col, op, dep, total, rounds, n_alive = want
    assert got_ns == rounds[:len(got_log)] and len(got_log) == len(rounds) == len(want_log)
    for k, ((a_ri, a_ts, a_te), (b_ri, b_ts, b_te)) in enumerate(zip(got_log, want_log)):
        assert torch.equal(a_ri, b_ri) and torch.equal(a_ts, b_ts) and torch.equal(a_te, b_te), f"round {k}"
    assert got[3] == total
    for g, w in zip(got[:3], (col, op, dep)):
        assert g.shape == w.shape and g.dtype == torch.float32
        assert (g - w).abs().max().item() <= 1e-5
    return rounds, n_alive, want_log, got


@pytest.mark.parametrize("bkgd", [None, (0.2, 0.4, 0.6)])
@pytest.mark.parametrize("alpha_thre", [0.0, 1e-2])
@pytest.mark.parametrize("name", list(SCENES))
def test_matches_the_public_function_loop(name, alpha_thre, bkgd):
    opts = dict(SCENES[name])
    est, ro, rd = scene(nfa, dev, **opts.pop("scene"))
    if bkgd is not None:
        opts["render_bkgd"] = torch.tensor(bkgd, device=dev)
    rounds, n_alive, log, got = check(est, ro, rd, ball_field(ro, rd), max_samples=1024, alpha_thre=alpha_thre,
                                      **opts)
    assert len(rounds) >= 3
    assert got[1].max().item() > 0.9999 and got[1].min().item() < 0.5  # some rays opaque, some left the grid


def test_sample_budget_stops_the_loop_with_rays_alive():
    est, ro, rd = scene(nfa, dev, res=128, levels=1, rays=5000)
    rounds, n_alive, _, _ = check(est, ro, rd, ball_field(ro, rd), max_samples=3, render_step_size=5e-3,
                                  render_bkgd=torch.ones(3, device=dev))
    assert sum(rounds) >= 3 and n_alive > 0


def test_missed_rays_and_every_ray_retired_after_round_one():
    est, ro, rd = scene(nfa, dev, res=128, levels=1, rays=3001)
    rd = torch.where((torch.arange(3001, device=dev) % 3 == 0)[:, None], -rd, rd)  # a third point away: no hit
    rounds, n_alive, log, got = check(est, ro, rd, ball_field(ro, rd, scale=1e6, radius=2.0), max_samples=1024,
                                      render_step_size=5e-3)
    assert rounds == [1] and n_alive == 0
    assert (got[1][::3] == 0).all() and len(log[0][0]) == 2000


def test_round_without_samples():
    # a step longer than the ball, whose second midpoint (t = 4) lies in it: at most one sample per ray, then every
    # live ray marches on past the ball and gets none
    est, ro, rd = scene(nfa, dev, res=128, levels=1, rays=2000)
    rounds, n_alive, log, _ = check(est, ro, rd, ball_field(ro, rd, scale=1e-2), max_samples=1024,
                                    render_step_size=8.0 / 3.0)
    assert len(log[0][0]) > 0 and any(len(ri) == 0 for ri, _, _ in log) and n_alive == 0


@pytest.mark.parametrize("R", [1, 33])
def test_small_batches(R):
    est, ro, rd = scene(nfa, dev, res=128, levels=1, rays=R, seed=3)
    for opts in (dict(render_step_size=2e-2), dict(render_step_size=5e-3, cone_angle=0.01)):
        rounds, _, _, _ = check(est, ro, rd, ball_field(ro, rd), max_samples=96, **opts)
        assert len(rounds) >= 2


def test_two_streams_and_repeated_runs_are_bit_identical():
    est, ro, rd = scene(nfa, dev, res=128, levels=4, rays=5000)
    est2, ro2, rd2 = scene(nfa, dev, res=128, levels=1, rays=4000, seed=5)
    kw = dict(max_samples=1024, render_step_size=1e-3, near_plane=0.2, cone_angle=0.004, alpha_thre=1e-2)
    kw2 = dict(max_samples=1024, render_step_size=5e-3, render_bkgd=torch.rand(3, device=dev))
    want = est.render_test(ro, rd, ball_field(ro, rd), **kw)
    want2 = est2.render_test(ro2, rd2, ball_field(ro2, rd2), **kw2)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        got = est.render_test(ro, rd, ball_field(ro, rd), **kw)
    with torch.cuda.stream(s2):
        got2 = est2.render_test(ro2, rd2, ball_field(ro2, rd2), **kw2)
    torch.cuda.synchronize()
    for a, b in ((got, want), (got2, want2)):
        assert a[3] == b[3]
        for x, y in zip(a[:3], b[:3]):
            assert torch.equal(x, y)  # no atomics: the same bits every time, on any stream
    check(est, ro, rd, ball_field(ro, rd), **kw)


def test_one_host_wait_per_round(monkeypatch):
    est, ro, rd = scene(nfa, dev, res=128, levels=1, rays=5000)
    field = ball_field(ro, rd)
    est.render_test(ro, rd, field, max_samples=1024, render_step_size=5e-3)  # workspace and pinned slot exist now
    _, _, _, _, rounds, _ = run_testmode_loop(nfa, est, ro, rd, field, max_samples=1024, render_step_size=5e-3)
    waits = []
    real = torch.cuda.Event.synchronize
    monkeypatch.setattr(torch.cuda.Event, "synchronize", lambda self: (waits.append(1), real(self))[1])
    for max_samples, extra in ((1024, 1), (3, 1)):
        # every ray retired: one more march finds none alive; budget spent: one wait for the sample total
        waits.clear()
        n_rounds = sum(1 for s in np.cumsum([0] + rounds)[:-1] if s < max_samples)
        torch.cuda.set_sync_debug_mode("error")
        try:
            est.render_test(ro, rd, field, max_samples=max_samples, render_step_size=5e-3)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert len(waits) == n_rounds + extra, (max_samples, len(waits), n_rounds)


def test_field_outputs_must_be_float32():
    est, ro, rd = scene(nfa, dev, res=64, levels=1, rays=256)
    field = ball_field(ro, rd)
    for cast in (lambda c, s: (c.half(), s), lambda c, s: (c, s.double())):
        with pytest.raises(RuntimeError, match="float32"):
            est.render_test(ro, rd, lambda *a: cast(*field(*a)), max_samples=64, render_step_size=5e-3)
    col, op, dep, total = est.render_test(ro, rd, field, max_samples=64, render_step_size=5e-3)  # still usable
    assert total > 0


def test_reference_build_golden():
    """The loop as the unmodified reference build runs it: the same samples per round (SHA-256), colours,
    opacities and depths within 1e-5."""
    ref = load_golden("ref_live_testmode")
    for name in GOLDEN:
        got = golden_case(nfa, name, dev, run=lambda est, *a, **k: est.render_test(*a, **k))
        np.testing.assert_array_equal(got["counts"], ref[f"{name}_counts"], err_msg=name)
        np.testing.assert_array_equal(got["sha_rounds"], ref[f"{name}_sha_rounds"], err_msg=name)
        assert int(got["total"]) == int(ref[f"{name}_total"]), name
        for k in ("colors", "opacities", "depths"):
            np.testing.assert_allclose(got[k], ref[f"{name}_{k}"], atol=1e-5, rtol=0, err_msg=f"{name} {k}")
