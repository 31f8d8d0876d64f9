"""Occupancy-grid maintenance (csrc/occ_update.cu) against references written here from the documented semantics.

- nfa_occ_ema_update: occs[ids] = maximum(occs[ids] * ema_decay, occ) (reference occ_grid.py:395-398).  A cell drawn
  once gets exactly torch.maximum's result on the device.  A cell drawn more than once gets the largest of its
  draws' results in the total order -inf < ... < -0.0 < +0.0 < ... < +inf, NaN if any result is NaN.
- nfa_occ_threshold_pack: thre = min(mean(occs[occs >= 0]), occ_thre) (:400-402) and binaries = occs > thre
  (:403-404), plus the march's packed form of the bool grid (march.cuh OccView): 64-bit brick words, the 2-bit class
  mip and the per-level brick bounds.  The layout is restated in numpy below, not read from the product headers.
- OccGridEstimator._update end to end, replayed in float64 on the same random draws.

Nothing here uses the product headers or the CPU oracle for the expected values."""
import itertools
import math

import numpy as np
import pytest
import torch

import nerfacc_b200 as nfa
from nerfacc_b200 import _lib, scenes

pytestmark = pytest.mark.gpu
dev = "cuda:0"


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def N(t):
    return t.detach().cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_same_floats(got, want, what):
    """Bit for bit, except that any NaN matches any NaN (the kernel writes the canonical NaN, torch passes on an
    operand's NaN bits)."""
    got, want = np.asarray(got, np.float32).reshape(-1), np.asarray(want, np.float32).reshape(-1)
    bad = (_bits(got) != _bits(want)) & ~(np.isnan(got) & np.isnan(want))
    if bad.any():
        i = np.flatnonzero(bad)[:8]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} differ, e.g. at {i.tolist()}: got "
                             f"{got[i].tolist()} (0x{' 0x'.join(f'{b:08x}' for b in _bits(got[i]))}), want "
                             f"{want[i].tolist()} (0x{' 0x'.join(f'{b:08x}' for b in _bits(want[i]))})")


# ---------------------------------------------------------------------------------------------------- EMA-max

# draw values and prior occupancies: signed zeros, subnormals, infinities, NaNs of both signs, -1 (invisible)
POOL = np.array([0.0, -0.0, 0.5, -0.5, 1.0, -1.0, 3.0e38, -3.0e38, 1e-45, -1e-45, 1.5e-39, -1.5e-39, np.inf, -np.inf,
                 np.nan, 0.0], np.float32)
POOL[-1] = np.uint32(0xFFC00000).view(np.float32)  # NaN with the sign bit set


def _mixed(rng, n, invisible=0.0):
    """Signed values over many binades, a tenth of them from POOL, `invisible` of them -1."""
    v = (rng.standard_normal(n) * 10.0 ** rng.uniform(-6, 3, n)).astype(np.float32)
    sp = rng.random(n) < 0.1
    v[sp] = POOL[rng.integers(0, len(POOL), int(sp.sum()))]
    v[rng.random(n) < invisible] = -1.0
    return v


def _draw_list(rng, n_draws, n_cells):
    """(prior occs, cell ids, draw values).  Every cell starts drawn once; then
    - every (prior, draw) pairing of POOL on cells drawn once;
    - every (prior, draw, draw) triple of POOL on cells drawn twice in adjacent slots (one warp), and again with the
      two draws half the list apart (different CTAs, and in a long list different grid-stride turns);
    - cells drawn 2-32 times inside one warp, and 2-32 times inside one 256-draw window (one CTA);
    - a few cells drawn hundreds of times all over the list."""
    P = len(POOL)
    ids = rng.permutation(n_cells)[:n_draws].astype(np.int64)
    vals = _mixed(rng, n_draws)
    prior = _mixed(rng, n_cells, invisible=0.1)
    used = np.zeros(n_draws, bool)

    s = np.arange(P * P)
    prior[ids[s]], vals[s] = POOL[s // P], POOL[s % P]
    used[s] = True
    trip = np.array(list(itertools.product(range(P), repeat=3)))
    a = -(-P * P // 32) * 32 + 2 * np.arange(len(trip))  # even slots: both draws of a pair in one warp
    d0 = a[-1] + 2 + np.arange(len(trip))
    d1 = d0 + n_draws // 2
    for x, y in ((a, a + 1), (d0, d1)):
        ids[y] = ids[x]
        prior[ids[x]], vals[x], vals[y] = POOL[trip[:, 0]], POOL[trip[:, 1]], POOL[trip[:, 2]]
        used[x] = used[y] = True

    for width, groups in ((256, 64), (32, 256)):
        free = np.flatnonzero(~used[: n_draws // width * width].reshape(-1, width).any(1))
        for w in rng.choice(free, groups, replace=False):
            slots = w * width + rng.choice(width, int(rng.integers(2, 33)), replace=False)
            ids[slots] = ids[slots[0]]
            used[w * width:(w + 1) * width] = True
    for _ in range(6):
        slots = rng.choice(np.flatnonzero(~used), int(rng.integers(200, 700)), replace=False)
        ids[slots] = ids[slots[0]]
        used[slots] = True
    return prior, ids, vals


def _ema_expected(prior, ids, vals, decay):
    """(expected occs, torch.maximum(old * decay, occ) per draw as torch computes it on the device)."""
    old = prior[ids]
    # the float32 product, rounded once (exact in float64 first): pins the rounding of `decay` to float32
    with np.errstate(invalid="ignore"):  # inf * 0
        prod = (old.astype(np.float64) * np.float64(np.float32(decay))).astype(np.float32)
    torch_prod = T(old) * decay
    assert_same_floats(N(torch_prod), prod, "old * decay")
    fresh = N(torch.maximum(torch_prod, T(vals)))
    # largest fresh value per cell in the total order: map the bits onto integers that order the same way
    b = _bits(fresh).astype(np.int64)
    key = np.where(b >= 2 ** 31, (2 ** 31 - 1) - b, b)  # sign bit set: -0.0 -> -1, -tiny -> -2, ..., -inf lowest
    best = np.full(len(prior), np.iinfo(np.int64).min)
    np.maximum.at(best, ids, key)
    want = prior.copy()
    drawn = np.unique(ids)
    k = best[drawn]
    want[drawn] = np.where(k >= 0, k, (2 ** 31 - 1) - k).astype(np.uint32).view(np.float32)
    want[ids[np.isnan(fresh)]] = np.nan
    return want, fresh


def _ema_update(prior, ids, vals, decay):
    occs = T(prior)
    scratch = torch.empty(len(ids), dtype=torch.float32, device=dev)
    t_ids, t_vals = T(ids), T(vals)
    _lib.call("nfa_occ_ema_update", occs.device, len(ids), _lib.ptr(t_ids), _lib.ptr(t_vals), float(decay),
              _lib.ptr(occs), _lib.ptr(scratch))
    return N(occs)


@pytest.mark.parametrize("decay", [0.0, 0.95, 1.0])
@pytest.mark.parametrize("n_draws", [1 << 16, 1_200_000])  # 1.2M: past the grid cap of the three kernels
def test_ema_update_matches_reference(decay, n_draws):
    rng = np.random.default_rng(n_draws + int(decay * 100))
    prior, ids, vals = _draw_list(rng, n_draws, n_draws + n_draws // 4)
    counts = np.bincount(ids, minlength=len(prior))
    assert counts.max() >= 200 and (counts == 1).sum() > n_draws // 4
    want, fresh = _ema_expected(prior, ids, vals, decay)
    got = _ema_update(prior, ids, vals, decay)

    assert np.array_equal(_bits(got[counts == 0]), _bits(prior[counts == 0])), "a cell that was not drawn changed"
    once = np.flatnonzero(counts == 1)
    slot = np.zeros(len(prior), np.int64)
    slot[ids] = np.arange(len(ids))
    assert_same_floats(got[once], fresh[slot[once]], "cells drawn once vs torch.maximum")
    assert_same_floats(got, want, "every cell vs the total-order maximum of its draws")
    # the signed zeros: a -0.0 result must read back as -0.0 (the reset value -inf must not survive)
    neg_zero = (want == 0) & np.signbit(want)
    assert neg_zero[counts > 1].any() and neg_zero[counts == 1].any()
    assert not np.isinf(got[neg_zero]).any(), "a -0.0 result was left at -inf"
    assert np.array_equal(_bits(_ema_update(prior, ids, vals, decay)), _bits(got)), "two runs differ"


# ---------------------------------------------------------------------------------------------------- threshold + pack

def _pack_reference(bins):
    """The march's packed form of a (G, rx, ry, rz) bool grid (march.cuh OccView):
    - one uint64 per 4x4x4 brick, bit (dx << 4) | (dy << 2) | dz, brick (bx * nb1 + by) * nb2 + bz + level * wpl,
      cells past the grid edge empty;
    - classes empty 0 / mixed 1 / full 3 (all 64 bits), 2 bits each, 16 bricks per uint32, word count padded to a
      multiple of 4;
    - per level the inclusive min and max brick x, y, z of the non-empty bricks; an empty level keeps
      0x7f7f7f7f / 0x80808080."""
    G, rx, ry, rz = bins.shape
    nb = [(r + 3) // 4 for r in (rx, ry, rz)]
    pad = np.zeros((G, nb[0] * 4, nb[1] * 4, nb[2] * 4), bool)
    pad[:, :rx, :ry, :rz] = bins
    cells = pad.reshape(G, nb[0], 4, nb[1], 4, nb[2], 4).transpose(0, 1, 3, 5, 2, 4, 6).reshape(-1, 64)
    words = np.packbits(cells, axis=-1, bitorder="little").view("<u8").reshape(-1)
    cls = np.where(words == 0, 0, np.where(words == np.uint64(2 ** 64 - 1), 3, 1)).astype(np.uint64)
    n_coarse = ((len(words) + 15) // 16 + 3) // 4 * 4
    cls = np.concatenate([cls, np.zeros(n_coarse * 16 - len(cls), np.uint64)]).reshape(n_coarse, 16)
    coarse = (cls << (2 * np.arange(16, dtype=np.uint64))).sum(1).astype(np.uint32)
    bounds = np.tile(np.array([0x7F7F7F7F] * 3 + [-0x7F7F7F80] * 3, np.int32), (G, 1))
    occupied = words.reshape(G, *nb) != 0
    for lvl in range(G):
        bxyz = np.argwhere(occupied[lvl])
        if len(bxyz):
            bounds[lvl] = np.concatenate([bxyz.min(0), bxyz.max(0)])
    return words, coarse, bounds.reshape(-1)


def _threshold_reference(occs, occ_thre):
    vis = occs[occs >= 0].astype(np.float64)
    mean = np.float32(math.fsum(vis.tolist()) / len(vis)) if len(vis) else np.float32(np.nan)
    return mean if np.isnan(mean) else np.minimum(mean, np.float32(occ_thre))


def _lattice(rng, n, hi):
    """Uniform on [0, hi) in steps of 2**-24: float32 cells whose float64 sum is exact in any order (up to 2**29
    cells below 1), so the mean has one right answer."""
    return (rng.integers(0, int(hi * 2 ** 24), n) / 2 ** 24).astype(np.float32)


def _ball(rng, shape):
    """Cells of each level: inside a ball >= 0.5 (full bricks), outside below 2**-6 (mixed bricks), a lattice of
    invisible (-1) cells and some -0.0 outside; all on the 2**-24 lattice."""
    G, rx, ry, rz = shape
    x, y, z = np.meshgrid(*[(np.arange(r) + 0.5) / r - 0.5 for r in (rx, ry, rz)], indexing="ij")
    inside = np.broadcast_to(x * x + y * y + z * z < (0.3 + 0.05 * np.arange(G)[:, None, None, None]) ** 2, shape)
    inside = inside.reshape(-1)
    occs = np.where(inside, 0.5 + _lattice(rng, inside.size, 0.5), _lattice(rng, inside.size, 2 ** -6))
    out = ~inside
    occs[out & (np.arange(occs.size) % 7 == 3)] = -1.0
    occs[out & (np.arange(occs.size) % 11 == 5)] = -0.0
    return occs.astype(np.float32)


def _contents(kind, shape, rng):
    n = int(np.prod(shape))
    if kind == "invisible":  # no visible cell: the mean and the threshold are NaN, the grid empty
        return np.full(n, -1.0, np.float32), 0.01
    if kind == "at_mean":  # pairs m - d, m + d and cells at m: the mean is m, and a cell at m stays false
        m = 2.0 ** -5
        n_inv = n // 9  # invisible cells do not count
        n_vis = n - n_inv
        d = _lattice(rng, n_vis // 2, m)
        d[: n_vis // 10] = 0.0
        occs = np.concatenate([m - d, m + d, np.full(n_vis % 2, m, np.float32), np.full(n_inv, -1.0, np.float32)])
        return rng.permutation(occs).astype(np.float32), 0.5
    occs = _ball(rng, shape)
    if kind == "ball_below":  # occ_thre below the mean: the threshold is occ_thre
        return occs, 2.0 ** -8
    if kind == "ball_above":  # occ_thre above the mean: the threshold is the mean
        return occs, 0.9
    if kind == "at_thre":  # cells exactly at the threshold stay false (strict >)
        occs[rng.random(n) < 0.2] = 2.0 ** -8
        return occs, 2.0 ** -8
    if kind == "inf":  # the mean is +inf, the threshold occ_thre; -inf is not visible
        occs[n // 2] = np.inf
        if n > 2:
            occs[n // 3] = -np.inf
        return occs, 0.75
    if kind == "nan":  # NaN cells neither count towards the mean nor pass the threshold
        occs[rng.random(n) < 0.1] = np.nan
        occs[0] = np.nan
        return occs, 0.9
    raise ValueError(kind)


SHAPES = [(1, 1, 1, 1), (1, 5, 7, 9), (3, 17, 13, 21), (1, 3, 5, 257), (2, 6, 9, 300), (3, 12, 20, 8),
          (4, 128, 128, 128)]
CONTENTS = ["ball_below", "ball_above", "at_mean", "at_thre", "invisible", "inf", "nan"]
# offset 1: `occs` starts one float past a 16-byte boundary, so the mean reads it with scalar loads only
CASES = [(s, c, 0) for s in SHAPES for c in CONTENTS] + [(s, "ball_below", 1) for s in SHAPES]


def _threshold_pack(occs, shape, occ_thre, ws):
    from nerfacc_b200.grid import _OccPack
    bins = torch.ones(shape, dtype=torch.bool, device=dev)  # poisoned: every output must be written
    pack = _OccPack(None, shape=shape, device=torch.device(dev))
    pack.words.fill_(0x5A5A5A5A5A5A5A5A)
    pack.coarse.fill_(-1)
    pack.bounds.fill_(12345)
    _lib.call("nfa_occ_threshold_pack", occs.device, *shape, _lib.ptr(occs), float(occ_thre), _lib.ptr(bins),
              _lib.ptr(pack.words), _lib.ptr(pack.coarse), _lib.ptr(pack.bounds), _lib.ptr(ws))
    thre = N(ws[16:20].view(torch.float32))[0]
    return thre, bins, pack


@pytest.mark.parametrize("shape,kind,offset", CASES, ids=[f"{'x'.join(map(str, s))}-{c}-off{o}" for s, c, o in CASES])
def test_threshold_pack_matches_reference(shape, kind, offset):
    from nerfacc_b200.grid import _OccPack
    rng = np.random.default_rng(sum(shape) * 31 + len(kind) + offset)
    occs_np, occ_thre = _contents(kind, shape, rng)
    n = occs_np.size
    base = torch.empty(n + 4, dtype=torch.float32, device=dev)
    occs = base[offset:offset + n]
    occs.copy_(T(occs_np))
    assert (occs.data_ptr() % 16 == 0) == (offset == 0)
    lib = _lib.load()
    ws = torch.full((lib.nfa_occ_threshold_workspace_bytes(n),), 0xFF, dtype=torch.uint8, device=dev)

    want_thre = _threshold_reference(occs_np, occ_thre)
    want_bins = (occs_np > want_thre).reshape(shape)
    want_words, want_coarse, want_bounds = _pack_reference(want_bins)
    if kind == "at_mean":
        assert want_thre == np.float32(2.0 ** -5)
    if kind in ("at_thre", "inf"):
        assert want_thre == np.float32(occ_thre)

    runs = [_threshold_pack(occs, shape, occ_thre, ws) for _ in range(2)]  # the workspace is reusable
    for thre, bins, pack in runs:
        assert_same_floats(thre, want_thre, "threshold")
        np.testing.assert_array_equal(N(bins), want_bins)
        np.testing.assert_array_equal(N(pack.words).view(np.uint64), want_words)
        np.testing.assert_array_equal(N(pack.coarse).view(np.uint32), want_coarse)
        np.testing.assert_array_equal(N(pack.bounds), want_bounds)
        fresh = _OccPack(bins)  # the other writer of the packed form, from the bool grid
        assert torch.equal(pack.words, fresh.words) and torch.equal(pack.coarse, fresh.coarse)
        assert torch.equal(pack.bounds, fresh.bounds)
    assert N(occs).tobytes() == occs_np.tobytes()  # the input is read only


# ---------------------------------------------------------------------------------------------------- estimator

def _field(scale):
    """Occupancy falling off from the origin; exactly -0.0 where x < -0.5."""
    def occ_eval_fn(x):
        v = scale * torch.exp(-0.05 * (x * x).sum(-1, keepdim=True))
        return torch.where(x[:, :1] < -0.5, -torch.zeros_like(v), v)
    return occ_eval_fn


def _sigma_fn(t_starts, t_ends, ray_indices):
    """Alphas spread over [0, 1) so that the alpha test depends on the value of occs.mean()."""
    u = torch.frac(ray_indices.float() * 0.6180339887 + t_starts * 7.3) * 0.999
    return -torch.log1p(-u) / (t_ends - t_starts)


def _replay(est, occs, bins, step, occ_eval_fn, occ_thre, ema_decay, warmup_steps):
    """OccGridEstimator._update as the reference writes it (occ_grid.py:367-404), on `occs` / `bins` before the
    update, in float64 where it computes: the same random draws in the same order, then per draw the float32 product
    rounded once and torch.maximum, the largest result per cell in the total order, the float64 mean."""
    cells, levels = est.cells_per_lvl, est.levels
    idx = torch.arange(cells, device=dev)
    per_level = []
    for lvl in range(levels):
        lvl_occs = occs[lvl * cells:(lvl + 1) * cells]
        if step < warmup_steps:
            per_level.append(idx[lvl_occs >= 0.0])
        else:
            n = cells // 4
            uniform = torch.randint(cells, (n,), device=dev)
            uniform = uniform[lvl_occs[uniform] >= 0.0]
            occupied = torch.nonzero(bins[lvl].flatten())[:, 0]
            if n < len(occupied):
                occupied = occupied[torch.randint(len(occupied), (n,), device=dev)]
            per_level.append(torch.cat([uniform, occupied], dim=0))
    ids, vals = [], []
    for lvl, indices in enumerate(per_level):
        coords = est.grid_coords[indices]
        x = (coords + torch.rand_like(coords, dtype=torch.float32)) / est.resolution
        x = est.aabbs[lvl, :3] + x * (est.aabbs[lvl, 3:] - est.aabbs[lvl, :3])
        vals.append(N(occ_eval_fn(x).squeeze(-1)))
        ids.append(N(lvl * cells + indices))
    want, _ = _ema_expected(N(occs), np.concatenate(ids), np.concatenate(vals), ema_decay)
    thre = _threshold_reference(want, occ_thre)
    return want, (want > thre).reshape(tuple(bins.shape))


def _sampling(est, rays, **kw):
    return est.sampling(*rays, render_step_size=1e-2, **kw)


@pytest.mark.parametrize("resolution,levels", [([17, 13, 21], 3), ([6, 5, 260], 2)], ids=["17x13x21", "rz260"])
def test_estimator_update_matches_float64_replay(resolution, levels):
    """_update across the warm-up / sampled-draws boundary on a grid with invisible cells and a region whose
    occupancy is -0.0: occs and binaries as the replay, -0.0 never turned into -inf, and sampling() reads the packed
    grid and the mean the update left behind."""
    torch.manual_seed(3)
    roi = torch.from_numpy(scenes.ROI_AABB)
    est = nfa.OccGridEstimator(roi, resolution=resolution, levels=levels).to(dev)
    est.train()
    K = torch.tensor([[[32.0, 0.0, 32.0], [0.0, 32.0, 32.0], [0.0, 0.0, 1.0]]], device=dev)
    c2w = torch.tensor([[[1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, -3.0]]], device=dev)
    est.mark_invisible_cells(K, c2w, 64, 64)
    invisible = est.occs < 0
    assert 0 < int(invisible.sum()) < est.occs.numel() // 4
    # a grid trained or loaded on the CPU can hold -0.0 where the field is -0.0: there torch.maximum(+0.0, -0.0) is
    # -0.0 on the vectorised path
    centres = est.aabbs[:, None, :3] + (est.grid_coords[None].float() + 0.5) / est.resolution * (
        est.aabbs[:, None, 3:] - est.aabbs[:, None, :3])
    neg_region = (centres[..., 0] < -0.6).reshape(-1) & ~invisible
    est.occs[neg_region] = -0.0
    rays = tuple(T(a) for a in scenes.ball_rays(2048, seed=7))
    est2 = nfa.OccGridEstimator(roi, resolution=resolution, levels=levels).to(dev)

    for step, scale in ((0, 0.9), (128, 0.4), (255, 0.7), (256, 0.3), (300, 0.8), (512, 0.5)):
        occ_eval_fn = _field(scale)
        _sampling(est, rays, sigma_fn=_sigma_fn, alpha_thre=0.99, early_stop_eps=0.0)  # caches occs.mean()
        mean_before = est._occs_mean()
        before, bins_before = est.occs.clone(), est.binaries.clone()
        state = torch.cuda.get_rng_state()
        est._update(step=step, occ_eval_fn=occ_eval_fn, occ_thre=0.01, ema_decay=0.95, warmup_steps=256)
        got_occs, got_bins = N(est.occs), N(est.binaries)
        assert getattr(est.binaries, "_nfa_occ", None) is not None  # the packed form came with the update

        torch.cuda.set_rng_state(state)
        want_occs, want_bins = _replay(est, before, bins_before, step, occ_eval_fn, 0.01, 0.95, 256)
        assert_same_floats(got_occs, want_occs, f"occs after step {step}")
        np.testing.assert_array_equal(got_bins, want_bins)
        neg_zero = (want_occs == 0) & np.signbit(want_occs)
        assert neg_zero.any() and not np.isinf(got_occs[neg_zero]).any(), "a -0.0 cell was left at -inf"
        assert (got_occs[N(invisible)] == -1.0).all()
        assert got_bins.any() and not got_bins.all()

        # sampling() on the packed grid the update wrote, and on the occs.mean() after the update
        mean_after = float(est.occs.mean())
        assert mean_after != mean_before and est._occs_mean() == mean_after
        est2.binaries = est.binaries.clone()
        est2.occs = est.occs.clone()
        for kw in ({}, dict(sigma_fn=_sigma_fn, alpha_thre=0.99, early_stop_eps=0.0)):
            a, b = _sampling(est, rays, **kw), _sampling(est2, rays, **kw)
            assert a[0].numel() > 0
            for x, y in zip(a, b):
                assert torch.equal(x, y)
