"""pack_info: per-sample ray indices -> per-ray (start, count); unpack_info, unpack_data, pack_data: conversions
between the packed layout ((all_samples, ...) + packed_info) and the padded per-ray layout ((n_rays, n_samples, ...)).

pack_info mirrors /root/reference/nerfacc/pack.py:10-49 (same name, arguments, dtype rule and error behaviour); the
histogram + scan run in ``nfa_pack_info`` instead of ``index_add_`` + ``cumsum``.  unpack_info / unpack_data /
pack_data are nerfacc 0.3's functions (removed in 0.5.0, reference CHANGELOG.md:38) with 0.3's names, argument order
and defaults; per-sample data may be flattened ``(N,)`` as well as ``(N, D)``.  They move bytes in
``csrc/pack.cu`` (``nfa_unpack_info``, ``nfa_unpack_rows`` / ``nfa_pack_rows``, ``nfa_mask_counts`` +
``nfa_pack_masked`` / ``nfa_unpack_masked``), so any dtype comes out bit-exact.
"""
import math
from typing import Optional, Tuple

import torch
from torch import Tensor

from . import _lib


def _stash_packed_info(ray_indices: Tensor, packed_info: Tensor, n_rays: int) -> None:
    """Remember the packed_info a traversal produced together with `ray_indices`.

    Both come out of the same kernel, so consumers that are handed exactly this
    tensor object (unmodified) need not rebuild the segments from 8 B/sample of indices.
    """
    ray_indices._nfa_packed = (packed_info, int(n_rays), ray_indices._version)


def _stashed_packed_info(ray_indices: Tensor, n_rays: Optional[int]) -> Optional[Tensor]:
    st = getattr(ray_indices, "_nfa_packed", None)
    if st is None:
        return None
    packed_info, n, version = st
    if version != ray_indices._version or (n_rays is not None and int(n_rays) != n):
        return None
    return packed_info


@torch.no_grad()
def pack_info(ray_indices: Tensor, n_rays: Optional[int] = None) -> Tensor:
    """(n_rays, 2) tensor of (chunk_start, chunk_cnt) for grouped `ray_indices`.

    Same contract as the reference: CUDA only (``NotImplementedError`` otherwise),
    output dtype follows the input dtype, ``n_rays=None`` infers ``max + 1``.
    """
    assert ray_indices.dim() == 1, "ray_indices must be a 1D tensor with shape (n_samples)."
    if not ray_indices.is_cuda:
        raise NotImplementedError("Only support cuda inputs.")
    # (with n_rays=None the reference returns max + 1 rows, which the stash -- one row per ray -- need not have)
    cached = _stashed_packed_info(ray_indices, n_rays) if n_rays is not None else None
    if cached is not None:
        return cached if cached.dtype == ray_indices.dtype else cached.to(ray_indices.dtype)
    if n_rays is None:
        n_rays = int(ray_indices.max().item()) + 1 if ray_indices.numel() > 0 else 0
    n_rays = int(n_rays)
    device = ray_indices.device
    idx = ray_indices.contiguous()
    if idx.dtype != torch.int64:
        idx = idx.to(torch.int64)
    lib = _lib.load()
    out = torch.empty((n_rays, 2), dtype=torch.int64, device=device)
    if n_rays > 0:
        ws = torch.empty(lib.nfa_pack_info_workspace_bytes(n_rays), dtype=torch.uint8, device=device)
        _lib.call("nfa_pack_info", device, idx.numel(), _lib.ptr(idx), n_rays, _lib.ptr(out), _lib.ptr(ws))
    return out if ray_indices.dtype == torch.int64 else out.to(ray_indices.dtype)


def _check_packed_info(packed_info: Tensor) -> Tensor:
    assert packed_info.dim() == 2 and packed_info.shape[-1] == 2, "packed_info must be a 2D tensor with shape (n_rays, 2)."
    _lib.require_cuda(packed_info, "packed_info")
    return packed_info.to(torch.int64).contiguous()


def _row_bytes(t: Tensor, lead: int) -> int:
    return t.element_size() * math.prod(t.shape[lead:])


def _order_workspace(device) -> Tensor:
    return torch.empty(_lib.load().nfa_chunk_order_workspace_bytes(), dtype=torch.uint8, device=device)


@torch.no_grad()
def unpack_info(packed_info: Tensor, n_samples: int) -> Tensor:
    """(n_samples,) int64 ray indices of the packed layout `packed_info` describes: ``r`` on ray r's chunk
    ``[start_r, start_r + count_r)``, ``-1`` where no chunk lands; chunk elements at or beyond `n_samples` are
    dropped.  Chunks must not overlap.  The inverse of :func:`pack_info`."""
    pi = _check_packed_info(packed_info)
    n, n_rays, device = int(n_samples), pi.shape[0], pi.device
    out = torch.empty((n,), dtype=torch.int64, device=device)
    if n == 0:
        return out
    if n_rays == 0:
        return out.fill_(-1)
    _lib.call("nfa_unpack_info", device, n_rays, _lib.ptr(pi), n, _lib.ptr(out), _lib.ptr(_order_workspace(device)))
    return out


def _pad_row(pad_value, like: Tensor, tail) -> Tensor:
    # pad_value cast to the data's dtype the way Tensor.to casts (e.g. -1 -> 255 for uint8)
    src = torch.tensor(pad_value, dtype=torch.float64 if isinstance(pad_value, float) else None)
    return torch.full(tail, src.to(like.dtype).item(), dtype=like.dtype, device=like.device)


class _UnpackRows(torch.autograd.Function):
    """packed (N, *tail) -> padded (n_rays, S, *tail); the backward is _PackRows."""

    @staticmethod
    def forward(ctx, data: Tensor, pi: Tensor, n_per_ray: int, pad_value):
        data = data.contiguous()
        n, tail, n_rays = data.shape[0], tuple(data.shape[1:]), pi.shape[0]
        out = data.new_empty((n_rays, n_per_ray) + tail)
        ctx.save_for_backward(pi)
        ctx.n = n
        if out.numel() > 0:
            pad = _pad_row(pad_value, data, tail)
            _lib.call("nfa_unpack_rows", data.device, n_rays, _lib.ptr(pi), n, n_per_ray, _row_bytes(data, 1),
                      _lib.ptr(data) if n > 0 else None, _lib.ptr(pad), _lib.ptr(out))
        return out

    @staticmethod
    def backward(ctx, grad: Tensor):
        (pi,) = ctx.saved_tensors
        return _PackRows.apply(grad, pi, ctx.n), None, None, None


class _PackRows(torch.autograd.Function):
    """padded (n_rays, S, *tail) -> packed (N, *tail), zero where no chunk row lands; the backward is _UnpackRows."""

    @staticmethod
    def forward(ctx, padded: Tensor, pi: Tensor, n: int):
        padded = padded.contiguous()
        n_rays, n_per_ray, tail = padded.shape[0], padded.shape[1], tuple(padded.shape[2:])
        out = padded.new_empty((n,) + tail)
        ctx.save_for_backward(pi)
        ctx.n_per_ray = n_per_ray
        if out.numel() > 0:
            _lib.call("nfa_pack_rows", padded.device, n_rays, _lib.ptr(pi), n, n_per_ray, _row_bytes(padded, 2),
                      _lib.ptr(padded) if padded.numel() > 0 else None, _lib.ptr(out),
                      _lib.ptr(_order_workspace(padded.device)))
        return out

    @staticmethod
    def backward(ctx, grad: Tensor):
        (pi,) = ctx.saved_tensors
        return _UnpackRows.apply(grad, pi, ctx.n_per_ray, 0), None, None


def unpack_data(packed_info: Tensor, data: Tensor, n_samples: Optional[int] = None, pad_value=0) -> Tensor:
    """Packed per-sample `data` (N, *tail) -> padded (n_rays, n_samples, *tail).

    ``out[r, j] = data[start_r + j]`` for ``j < min(count_r, n_samples)``; every other position is `pad_value`, cast
    to ``data.dtype``.  ``n_samples=None`` takes the longest ray (one host sync); longer rays are truncated.
    Differentiable with respect to floating `data` (truncated or uncovered samples get a zero gradient)."""
    pi = _check_packed_info(packed_info)
    assert data.dim() >= 1, "data must have a leading sample dimension (N, ...)."
    _lib.require_cuda(data, "data")
    if n_samples is None:
        n_samples = max(int(pi[:, 1].max().item()), 0) if pi.shape[0] > 0 else 0
    return _UnpackRows.apply(data, pi, int(n_samples), pad_value)


class _PackMasked(torch.autograd.Function):
    """padded (R, S, *tail) -> data[mask]; the backward is _UnpackMasked."""

    @staticmethod
    def forward(ctx, data: Tensor, mask: Tensor, pi: Tensor, n: int):
        data = data.contiguous()
        n_rays, n_per_ray, tail = data.shape[0], data.shape[1], tuple(data.shape[2:])
        out = data.new_empty((n,) + tail)
        ctx.save_for_backward(mask, pi)
        ctx.n_per_ray = n_per_ray
        if out.numel() > 0:
            _lib.call("nfa_pack_masked", data.device, n_rays, n_per_ray, _row_bytes(data, 2), _lib.ptr(mask),
                      _lib.ptr(pi), _lib.ptr(data), _lib.ptr(out))
        return out

    @staticmethod
    def backward(ctx, grad: Tensor):
        mask, pi = ctx.saved_tensors
        return _UnpackMasked.apply(grad, mask, pi, ctx.n_per_ray), None, None, None


class _UnpackMasked(torch.autograd.Function):
    """packed (N, *tail) -> padded (R, S, *tail) at the mask positions, zeros elsewhere; the backward is _PackMasked."""

    @staticmethod
    def forward(ctx, packed: Tensor, mask: Tensor, pi: Tensor, n_per_ray: int):
        packed = packed.contiguous()
        n, tail, n_rays = packed.shape[0], tuple(packed.shape[1:]), mask.shape[0]
        out = packed.new_empty((n_rays, n_per_ray) + tail)
        ctx.save_for_backward(mask, pi)
        ctx.n = n
        if out.numel() > 0:
            _lib.call("nfa_unpack_masked", packed.device, n_rays, n_per_ray, _row_bytes(packed, 1), _lib.ptr(mask),
                      _lib.ptr(pi), _lib.ptr(packed) if n > 0 else None, _lib.ptr(out))
        return out

    @staticmethod
    def backward(ctx, grad: Tensor):
        mask, pi = ctx.saved_tensors
        return _PackMasked.apply(grad, mask, pi, ctx.n), None, None, None


def pack_data(data: Tensor, mask: Tensor) -> Tuple[Tensor, Tensor]:
    """Padded `data` (R, S, *tail) -> (``data[mask]``, packed_info) for a (R, S) bool `mask`.

    ``packed_info`` is int64 ``[cumsum(counts) - counts, counts]`` with ``counts = mask.sum(-1)``.  One host sync,
    to size the output.  Differentiable with respect to `data` (zeros where the mask is false)."""
    assert mask.dtype == torch.bool, "mask must be a bool tensor."
    assert mask.dim() == 2, "mask must be a 2D tensor with shape (n_rays, n_samples)."
    assert data.dim() >= 2 and tuple(data.shape[:2]) == tuple(mask.shape), \
        "data must have shape (n_rays, n_samples, ...) matching mask."
    _lib.require_cuda(data, "data")
    _lib.require_cuda(mask, "mask")
    mask = mask.contiguous()
    n_rays, n_per_ray = mask.shape
    device = data.device
    pi = torch.empty((n_rays, 2), dtype=torch.int64, device=device)
    if n_rays == 0 or n_per_ray == 0:
        pi.zero_()
        n = 0
    else:
        counts = torch.empty((n_rays,), dtype=torch.int64, device=device)
        _lib.call("nfa_mask_counts", device, n_rays, n_per_ray, _lib.ptr(mask), _lib.ptr(counts))
        ws = torch.empty(_lib.load().nfa_pack_info_workspace_bytes(n_rays), dtype=torch.uint8, device=device)
        _lib.call("nfa_counts_to_packed_info", device, n_rays, _lib.ptr(counts), _lib.ptr(pi), _lib.ptr(ws))
        start, count = pi[-1].tolist()  # the one host sync
        n = start + count
    return _PackMasked.apply(data, mask, pi, n), pi
