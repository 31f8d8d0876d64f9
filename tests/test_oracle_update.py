"""Grid maintenance (SURVEY 8 row f4): the oracle's restatement of OccGridEstimator._update against golden vectors
of the reference itself (tests/golden/ref_occ_update.npz, made by oracle/gen_golden_update_cpu.py on the CPU)."""
import numpy as np
import pytest

from conftest import load_golden


@pytest.mark.parametrize("case", ["warm", "sampled", "sampled_hi"])
def test_oracle_update_matches_reference(orc, case):
    z = load_golden("ref_occ_update")
    before, ids, occ = z[case + "_occs_before"], z[case + "_ids"], z[case + "_occ"]
    want, want_bin = z[case + "_occs_after"], z[case + "_binaries"]
    occ_thre, decay = (float(v) for v in z[case + "_args"])
    got = orc.occ_ema_update(before, ids, occ, decay)
    uniq, cnt = np.unique(ids, return_counts=True)
    once = np.zeros(len(before), bool)
    once[uniq[cnt == 1]] = True
    dup = np.zeros(len(before), bool)
    dup[uniq[cnt > 1]] = True
    untouched = ~(once | dup)
    np.testing.assert_array_equal(got[untouched], before[untouched])
    np.testing.assert_array_equal(got[once], want[once])           # bit-exact where the cell was drawn once
    # drawn twice: the reference keeps one candidate (the last write), we keep the largest
    cand_max = np.full(len(before), -np.inf, np.float32)
    np.maximum.at(cand_max, ids, np.maximum(before[ids] * np.float32(decay), occ))
    np.testing.assert_array_equal(got[dup], cand_max[dup])
    assert (want[dup] <= got[dup]).all()
    if case == "warm":
        assert not dup.any() and once.sum() == len(ids)
    else:
        assert dup.any()
    # threshold on the reference's own occs: binaries identical
    bins, thre = orc.occ_threshold(want, occ_thre)
    assert thre <= occ_thre
    np.testing.assert_array_equal(bins.reshape(want_bin.shape), want_bin)
    assert (~bins[want < 0]).all()                                  # invisible cells stay empty


def test_oracle_update_keeps_the_largest_in_the_total_order(orc):
    """A cell drawn more than once keeps its largest result in the order -0.0 < +0.0, whichever draw comes first, a
    -0.0 result is not lost to the -inf a drawn cell starts from, and NaN wins."""
    draws = [(0.0, -0.0), (-0.0, 0.0), (-0.0,), (-0.0, -0.5), (-0.5, -0.0), (np.nan, 1.0), (1.0, np.nan)]
    ids = np.array([c for c, d in enumerate(draws) for _ in d], np.int64)
    occ = np.array([v for d in draws for v in d], np.float32)
    before = np.full(len(draws), -np.inf, np.float32)  # -inf * 1.0 = -inf: every result is the draw itself
    got = orc.occ_ema_update(before, ids, occ, 1.0)
    want = np.array([0.0, 0.0, -0.0, -0.0, -0.0, np.nan, np.nan], np.float32)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    np.testing.assert_array_equal(got[ok].view(np.uint32), want[ok].view(np.uint32))
