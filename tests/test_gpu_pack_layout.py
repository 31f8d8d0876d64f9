"""unpack_info / unpack_data / pack_data on the GPU, bit for bit against their plain-torch formulations
(repeat_interleave for unpack_info, full + masked index assignment for unpack_data, data[mask] + cumsum for
pack_data), over ragged rays whose boundaries fall at every offset inside a 16-byte group, every dtype, tails of
every row size class, inputs 1-3 elements off 16-byte alignment, gaps, unordered chunks and empty inputs."""
import numpy as np
import pytest
import torch

import nerfacc_b200 as nfa
from nerfacc_b200 import _lib, scenes

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
SPECIAL = [0, 1, 31, 32, 33, 127, 128, 129, 250]
DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.float64, torch.int64, torch.bool, torch.uint8]
TAILS = [(), (1,), (3,), (4,), (5,), (16,), (2, 3)]
BITS = {2: torch.int16, 4: torch.int32, 8: torch.int64}


# ---------------------------------------------------------------------------------------------- torch formulation
def ref_unpack_info(pi, n):
    pi = pi.to(torch.int64)
    starts, counts = pi[:, 0], pi[:, 1].clamp_min(0)
    out = torch.full((n,), -1, dtype=torch.int64, device=pi.device)
    rays = torch.repeat_interleave(torch.arange(len(pi), device=pi.device), counts)
    first = torch.repeat_interleave(torch.cumsum(counts, 0) - counts, counts)
    pos = torch.repeat_interleave(starts, counts) + torch.arange(rays.numel(), device=pi.device) - first
    keep = (pos >= 0) & (pos < n)
    out[pos[keep]] = rays[keep]
    return out


def pad_tensor(pad, dtype):
    return torch.tensor(pad).to(dtype)


def ref_unpack_data(pi, data, S, pad=0):
    pi = pi.to(torch.int64)
    starts, counts = pi[:, :1], pi[:, 1:]
    out = pad_tensor(pad, data.dtype).to(data.device).expand((len(pi), S) + tuple(data.shape[1:])).clone()
    pos = starts + torch.arange(S, device=data.device)
    valid = (torch.arange(S, device=data.device) < counts) & (pos >= 0) & (pos < data.shape[0])
    out[valid] = data[pos[valid]]
    return out


def ref_pack_data(data, mask):
    counts = mask.sum(-1)
    return data[mask], torch.stack([torch.cumsum(counts, 0) - counts, counts], -1)


# ---------------------------------------------------------------------------------------------- helpers
def bits(t):
    return t.view(BITS[t.element_size()]) if t.is_floating_point() else t


def assert_bits_equal(a, b, what=""):
    assert a.dtype == b.dtype and a.shape == b.shape, f"{what}: {a.dtype}{tuple(a.shape)} vs {b.dtype}{tuple(b.shape)}"
    assert torch.equal(bits(a), bits(b)), what


def ragged_counts(seed, extra=40, hi=80):
    rng = np.random.default_rng(seed)
    c = np.concatenate([np.tile(SPECIAL, 2), rng.integers(0, hi, extra)])
    rng.shuffle(c)
    return torch.from_numpy(c.astype(np.int64)).to(dev)


def packed_info_of(counts):
    return torch.stack([torch.cumsum(counts, 0) - counts, counts], -1)


def random_data(shape, dtype, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    n = int(np.prod(shape)) if len(shape) else 1
    if dtype == torch.bool:
        return (torch.rand(shape, generator=g) > 0.5).to(dev)
    size = torch.empty((), dtype=dtype).element_size()
    raw = torch.randint(0, 256, (n * size,), dtype=torch.uint8, generator=g)
    return raw.view(dtype).view(shape).to(dev)  # every bit pattern, NaN payloads included


def place(t, off):
    """A copy of `t` whose storage starts `off` elements past a 16-byte boundary."""
    buf = torch.empty(t.numel() + off + 16, dtype=t.dtype, device=dev)
    v = buf[off:off + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def pads_for(dtype):
    return [0, -1, float("inf"), float("nan")] if dtype.is_floating_point else [0, -1]


# ---------------------------------------------------------------------------------------------- unpack_info
def test_unpack_info_inverts_contiguous_packed_info():
    for seed in range(3):
        counts = ragged_counts(seed)
        pi = packed_info_of(counts)
        n = int(counts.sum())
        ri = nfa.unpack_info(pi, n)
        assert ri.dtype == torch.int64 and ri.shape == (n,)
        assert torch.equal(ri, torch.repeat_interleave(torch.arange(len(counts), device=dev), counts))
        assert torch.equal(nfa.unpack_info(pi.to(torch.int32), n), ri)
        assert torch.equal(nfa.pack_info(ri, len(counts)), pi)


def test_unpack_info_gaps_overruns_and_unordered_chunks():
    counts = ragged_counts(7)
    R = len(counts)
    stride = 260
    strided = torch.stack([torch.arange(R, device=dev) * stride, counts], -1)  # fixed stride: gaps behind every ray
    n_full = R * stride
    for n in (n_full, n_full - 200, n_full - 3000, n_full + 77, 1, 5000):  # chunks cut by n, or a tail gap
        assert torch.equal(nfa.unpack_info(strided, n), ref_unpack_info(strided, n)), n
    pi = packed_info_of(counts)
    total = int(counts.sum())
    for n in (total - 1, total - 250, total + 300):
        assert torch.equal(nfa.unpack_info(pi, n), ref_unpack_info(pi, n)), n
    # unordered chunks (rows permuted), and zero-count rays whose start points anywhere: the fill path
    perm = torch.randperm(R, generator=torch.Generator().manual_seed(3)).to(dev)
    for q in (strided[perm], pi[perm]):
        assert torch.equal(nfa.unpack_info(q, n_full), ref_unpack_info(q, n_full))
    odd = pi.clone()
    odd[counts == 0, 0] = 0
    assert torch.equal(nfa.unpack_info(odd, total), ref_unpack_info(odd, total))
    # leading gap in front of ray 0, negative starts
    shifted = pi + torch.tensor([40, 0], device=dev)
    assert torch.equal(nfa.unpack_info(shifted, total + 40), ref_unpack_info(shifted, total + 40))
    neg = pi - torch.tensor([50, 0], device=dev)
    assert torch.equal(nfa.unpack_info(neg, total), ref_unpack_info(neg, total))


def test_unpack_info_empty_inputs():
    pi = packed_info_of(ragged_counts(1))
    assert nfa.unpack_info(pi, 0).shape == (0,)
    empty = torch.empty((0, 2), dtype=torch.int64, device=dev)
    assert torch.equal(nfa.unpack_info(empty, 9), torch.full((9,), -1, device=dev))
    assert nfa.unpack_info(empty, 0).shape == (0,)
    zeros = torch.zeros((5, 2), dtype=torch.int64, device=dev)
    assert torch.equal(nfa.unpack_info(zeros, 4), torch.full((4,), -1, device=dev))


# ---------------------------------------------------------------------------------------------- unpack_data
@pytest.mark.parametrize("tail", TAILS, ids=str)
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_unpack_data_bits(dtype, tail):
    counts = ragged_counts(11)
    pi = packed_info_of(counts)
    n, mx = int(counts.sum()), int(counts.max())
    x = random_data((n,) + tail, dtype, seed=5)
    for off in (0, 1, 2, 3):
        xo = place(x, off)
        for S in (None, mx - 7, mx, mx + 5):
            for pad in pads_for(dtype) if S == mx + 5 else [0]:
                got = nfa.unpack_data(pi, xo, S, pad) if S is not None else nfa.unpack_data(pi, xo)
                assert_bits_equal(got, ref_unpack_data(pi, x, S or mx, pad), f"off {off} S {S} pad {pad}")
    # gaps (fixed stride) and chunks that run past the data
    stride = mx + 3
    strided = torch.stack([torch.arange(len(counts), device=dev) * stride, counts], -1)
    y = random_data((len(counts) * stride - 100,) + tail, dtype, seed=6)
    for pad in pads_for(dtype):
        assert_bits_equal(nfa.unpack_data(strided, place(y, 1), mx, pad), ref_unpack_data(strided, y, mx, pad), "gaps")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bool], ids=str)
def test_unpack_data_empty_and_noncontiguous(dtype):
    counts = ragged_counts(2)
    pi = packed_info_of(counts)
    n = int(counts.sum())
    empty_pi = torch.empty((0, 2), dtype=torch.int64, device=dev)
    x = random_data((n, 3), dtype, seed=1)
    assert nfa.unpack_data(empty_pi, x).shape == (0, 0, 3)
    assert nfa.unpack_data(empty_pi, x, 6).shape == (0, 6, 3)
    assert nfa.unpack_data(pi, x, 0).shape == (len(counts), 0, 3)
    zero_pi = torch.zeros((4, 2), dtype=torch.int64, device=dev)
    none = x[:0]
    assert_bits_equal(nfa.unpack_data(zero_pi, none, 3, -1), ref_unpack_data(zero_pi, none, 3, -1), "N = 0")
    assert nfa.unpack_data(zero_pi, none).shape == (4, 0, 3)
    xt = random_data((3, n), dtype, seed=2).t()  # non-contiguous
    assert_bits_equal(nfa.unpack_data(pi, xt, 40), ref_unpack_data(pi, xt.contiguous(), 40), "non-contiguous")


# ---------------------------------------------------------------------------------------------- pack_data
def ragged_mask(seed, R=60, S=263):
    rng = np.random.default_rng(seed)
    m = rng.random((R, S)) < rng.random((R, 1))
    lens = np.concatenate([np.tile(SPECIAL, 3), rng.integers(0, S, R)])[:R]
    prefix = np.arange(S)[None, :] < lens[:, None]
    m[: R // 2] = prefix[: R // 2]  # half the rows: prefix masks of every SPECIAL length
    m[5] = False
    return torch.from_numpy(m).to(dev)


@pytest.mark.parametrize("tail", TAILS, ids=str)
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_pack_data_bits(dtype, tail):
    mask = ragged_mask(3)
    x = random_data(tuple(mask.shape) + tail, dtype, seed=8)
    ref_x, ref_pi = ref_pack_data(x, mask)
    for off in (0, 1, 2, 3):
        got_x, got_pi = nfa.pack_data(place(x, off), mask)
        assert_bits_equal(got_x, ref_x, f"off {off}")
        assert got_pi.dtype == torch.int64 and torch.equal(got_pi, ref_pi)


@pytest.mark.parametrize("dtype", [torch.float32, torch.uint8], ids=str)
def test_pack_data_empty_and_noncontiguous(dtype):
    mask = ragged_mask(4)
    R, S = mask.shape
    x = random_data((R, S, 2), dtype, seed=3)
    px, ppi = nfa.pack_data(x, torch.zeros_like(mask))
    assert px.shape == (0, 2) and torch.equal(ppi, torch.zeros((R, 2), dtype=torch.int64, device=dev))
    px, ppi = nfa.pack_data(x[:0], mask[:0])
    assert px.shape == (0, 2) and ppi.shape == (0, 2)
    px, ppi = nfa.pack_data(x[:, :0], mask[:, :0])
    assert px.shape == (0, 2) and torch.equal(ppi, torch.zeros((R, 2), dtype=torch.int64, device=dev))
    xt = random_data((S, R), dtype, seed=4).t()  # (R, S), non-contiguous, no tail
    mt = ragged_mask(5, R=S, S=R).t()
    got_x, got_pi = nfa.pack_data(xt, mt)
    ref_x, ref_pi = ref_pack_data(xt, mt)
    assert_bits_equal(got_x, ref_x, "non-contiguous")
    assert torch.equal(got_pi, ref_pi)


# ---------------------------------------------------------------------------------------------- round trips
def ball_sampling(n_rays, res=128):
    ro, rd = scenes.ball_rays(n_rays)
    est = nfa.OccGridEstimator(torch.from_numpy(scenes.ROI_AABB), resolution=res, levels=1).to(dev)
    est.binaries = torch.from_numpy(scenes.ball_grid(res)).to(dev)
    ri, ts, te = est.sampling(torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev),
                              render_step_size=scenes.BALL_STEP)
    return ri, ts, te


def test_round_trips_on_the_ball_scene():
    R = 4096
    ri, ts, te = ball_sampling(R)
    n = ri.numel()
    pi = nfa.pack_info(ri, R)
    assert torch.equal(nfa.unpack_info(pi, n), ri)
    assert torch.equal(nfa.pack_info(nfa.unpack_info(pi, n).clone(), R), pi)
    x = torch.stack([ts, te, ts * te], -1)
    padded = nfa.unpack_data(pi, x)
    prefix = torch.arange(padded.shape[1], device=dev) < pi[:, 1:]
    back, back_pi = nfa.pack_data(padded, prefix)
    assert_bits_equal(back, x, "pack_data(unpack_data(x))")
    assert torch.equal(back_pi, pi)


def test_config2_sized_layout():
    """The ball scene of bench.py: ~8.5 M samples over 65 536 rays, tail (3,) float32."""
    R = 65536
    ri, ts, te = ball_sampling(R)
    n = ri.numel()
    assert n > 5_000_000
    pi = nfa.pack_info(ri, R)
    assert torch.equal(nfa.unpack_info(pi, n), ri)
    assert torch.equal(nfa.unpack_info(pi, n), ref_unpack_info(pi, n))
    x = random_data((n, 3), torch.float32, seed=9)
    padded = nfa.unpack_data(pi, x)
    ref = ref_unpack_data(pi, x, int(pi[:, 1].max()))
    assert_bits_equal(padded, ref, "unpack_data")
    mask = torch.arange(padded.shape[1], device=dev) < pi[:, 1:]
    mask &= torch.rand(mask.shape, generator=torch.Generator(device=dev).manual_seed(1), device=dev) < 0.7
    got_x, got_pi = nfa.pack_data(padded, mask)
    ref_x, ref_pi = ref_pack_data(padded, mask)
    assert_bits_equal(got_x, ref_x, "pack_data")
    assert torch.equal(got_pi, ref_pi)


# ---------------------------------------------------------------------------------------------- gradients
def test_gradients_match_the_torch_formulation_bit_for_bit():
    counts = ragged_counts(13)
    pi = packed_info_of(counts)
    n, mx = int(counts.sum()), int(counts.max())
    R = len(counts)
    stride = mx + 3
    strided = torch.stack([torch.arange(R, device=dev) * stride, counts], -1)
    perm = torch.randperm(R, generator=torch.Generator().manual_seed(4)).to(dev)
    for q, N, S in ((pi, n, mx), (pi, n, mx - 40), (strided, R * stride - 50, mx), (strided[perm], R * stride, mx - 3)):
        x = torch.randn(N, 5, device=dev)
        w = torch.randn(R, S, 5, device=dev)
        a = x.clone().requires_grad_(True)
        b = x.clone().requires_grad_(True)
        (nfa.unpack_data(q, a, S, 1.5) * w).sum().backward()
        (ref_unpack_data(q, b, S, 1.5) * w).sum().backward()
        assert_bits_equal(a.grad, b.grad, f"unpack_data grad S {S}")
    mask = ragged_mask(6)
    x = torch.randn(tuple(mask.shape) + (3,), device=dev)
    w = torch.randn(int(mask.sum()), 3, device=dev)
    a = x.clone().requires_grad_(True)
    b = x.clone().requires_grad_(True)
    (nfa.pack_data(a, mask)[0] * w).sum().backward()
    (ref_pack_data(b, mask)[0] * w).sum().backward()
    assert_bits_equal(a.grad, b.grad, "pack_data grad")


def test_gradcheck_and_gradgradcheck_float64():
    counts = torch.tensor([3, 0, 5, 1, 4], device=dev)
    pi = packed_info_of(counts)
    gaps = torch.tensor([[0, 2], [4, 3], [9, 0], [10, 4]], device=dev)  # gaps, and a chunk running past N
    for q, n, S in ((pi, 13, 4), (pi, 13, 6), (gaps, 12, 3)):
        x = torch.randn(n, 2, dtype=torch.float64, device=dev, requires_grad=True)
        f = lambda t: nfa.unpack_data(q, t, S, -2.0)  # noqa: E731
        assert torch.autograd.gradcheck(f, (x,))
        assert torch.autograd.gradgradcheck(f, (x,))
    mask = torch.rand(5, 7, generator=torch.Generator().manual_seed(2)).to(dev) < 0.5
    y = torch.randn(5, 7, dtype=torch.float64, device=dev, requires_grad=True)
    g = lambda t: nfa.pack_data(t, mask)[0]  # noqa: E731
    assert torch.autograd.gradcheck(g, (y,))
    assert torch.autograd.gradgradcheck(g, (y,))


def test_native_kernels_ran():
    counts = ragged_counts(0)
    pi = packed_info_of(counts)
    x = torch.rand(int(counts.sum()), device=dev)
    before = _lib.launches
    nfa.unpack_info(pi, x.numel())
    nfa.unpack_data(pi, x)
    nfa.pack_data(x[:10].view(2, 5), torch.ones(2, 5, dtype=torch.bool, device=dev))
    assert _lib.launches - before == 5  # unpack_info, unpack_rows, mask_counts, counts_to_packed_info, pack_masked
