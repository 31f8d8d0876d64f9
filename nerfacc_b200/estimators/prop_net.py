"""Proposal-network transmittance estimator (mip-NeRF 360 style resampling).

Same class, methods, arguments and caching protocol as /root/reference/nerfacc/estimators/prop_net.py:17-313.
Each proposal level is one fused native launch (`nfa_importance_sampling`: sample centres, the edges
between them and, when no gradient is needed through the edges, their s -> t mapping) plus the fused
transmittance kernel; the reference spends two launches and ~10 ATen ops per level on the same work.  The training
loss of each level (`_pdf_loss`) is one native launch forward and one backward, with a gradient that does not change
from run to run.
"""
from typing import Callable, List, Optional, Tuple

try:
    from typing import Literal
except ImportError:  # pragma: no cover
    from typing_extensions import Literal

import torch
from torch import Tensor
from torch.autograd.function import once_differentiable

from .. import _lib
from ..data_specs import RayIntervals
from ..pdf import _importance_sampling, searchsorted
from ..volrend import _grad_through, render_transmittance_from_density
from .base import AbstractEstimator


class PropNetEstimator(AbstractEstimator):
    """Proposal network transmittance estimator.

    Args:
        optimizer: optimizer of the proposal networks (stepped by :meth:`update_every_n_steps`).
        scheduler: optional learning-rate scheduler of the proposal networks.
    """

    def __init__(
        self,
        optimizer: Optional[torch.optim.Optimizer] = None,
        scheduler: Optional[torch.optim.lr_scheduler._LRScheduler] = None,
    ) -> None:
        super().__init__()
        self.optimizer = optimizer
        self.scheduler = scheduler
        self.prop_cache: List = []

    @torch.no_grad()
    def sampling(
        self,
        prop_sigma_fns: List[Callable],
        prop_samples: List[int],
        num_samples: int,
        # rendering options
        n_rays: int,
        near_plane: float,
        far_plane: float,
        sampling_type: Literal["uniform", "lindisp"] = "lindisp",
        # training options
        stratified: bool = False,
        requires_grad: bool = False,
    ) -> Tuple[Tensor, Tensor]:
        """Sample with the CDFs of the proposal networks (reference prop_net.py:37-129).

        ``prop_sigma_fns[i](t_starts, t_ends) -> sigmas`` (all ``(n_rays, prop_samples[i])``).  With
        ``requires_grad`` the proposal outputs are cached for :meth:`update_every_n_steps`.
        Returns ``t_starts, t_ends`` of shape ``(n_rays, num_samples)``.
        """
        assert len(prop_sigma_fns) == len(prop_samples), (
            "The number of proposal networks and the number of samples should be the same."
        )
        if sampling_type not in ("uniform", "lindisp"):
            raise ValueError(f"Unknown transform_type: {sampling_type}")
        stot = _stot_constants(sampling_type, near_plane, far_plane)
        device = self.device
        cdfs = torch.cat([torch.zeros((n_rays, 1), device=device), torch.ones((n_rays, 1), device=device)], dim=-1)
        intervals = RayIntervals(vals=cdfs)

        for level_fn, level_samples in zip(prop_sigma_fns, prop_samples):
            intervals, _, t_starts, t_ends = _importance_sampling(intervals, cdfs, level_samples, stratified, stot)
            with torch.set_grad_enabled(requires_grad):
                sigmas = level_fn(t_starts, t_ends)
                assert sigmas.shape == t_starts.shape
                trans, _ = render_transmittance_from_density(t_starts, t_ends, sigmas)
                cdfs = 1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], dim=-1)
                if requires_grad:
                    self.prop_cache.append((intervals, cdfs))

        intervals, _, t_starts, t_ends = _importance_sampling(intervals, cdfs, num_samples, stratified, stot)
        if requires_grad:
            self.prop_cache.append((intervals, None))
        return t_starts, t_ends

    @torch.enable_grad()
    def compute_loss(self, trans: Tensor, loss_scaler: float = 1.0) -> Tensor:
        """Proposal loss against the final transmittance ``(n_rays, num_samples)`` (reference prop_net.py:131-154)."""
        if len(self.prop_cache) == 0:
            return torch.zeros((), device=self.device)
        intervals, _ = self.prop_cache.pop()
        cdfs = (1.0 - torch.cat([trans, torch.zeros_like(trans[:, :1])], dim=-1)).detach()
        loss = 0.0
        while self.prop_cache:
            prop_intervals, prop_cdfs = self.prop_cache.pop()
            loss = loss + _pdf_loss(intervals, cdfs, prop_intervals, prop_cdfs).mean()
        return loss * loss_scaler

    @torch.enable_grad()
    def update_every_n_steps(self, trans: Tensor, requires_grad: bool = False, loss_scaler: float = 1.0) -> float:
        """Train the proposal networks when ``requires_grad``; always advance the scheduler
        (reference prop_net.py:156-193).  Returns the proposal loss as a float."""
        if requires_grad:
            return self._update(trans=trans, loss_scaler=loss_scaler)
        if self.scheduler is not None:
            self.scheduler.step()
        return 0.0

    @torch.enable_grad()
    def _update(self, trans: Tensor, loss_scaler: float = 1.0) -> float:
        assert len(self.prop_cache) > 0
        assert self.optimizer is not None, "No optimizer is provided."
        loss = self.compute_loss(trans, loss_scaler)
        self.optimizer.zero_grad()
        loss.backward()
        self.optimizer.step()
        if self.scheduler is not None:
            self.scheduler.step()
        return loss.item()


def get_proposal_requires_grad_fn(target: float = 5.0, num_steps: int = 1000) -> Callable:
    """Schedule of how often the proposal networks train: every step at first, every ``target`` steps
    after ``num_steps`` (reference prop_net.py:196-212)."""
    since_last = 0

    def proposal_requires_grad_fn(step: int) -> bool:
        nonlocal since_last
        wanted = min(step / num_steps, 1.0) * target
        fire = since_last > wanted
        if fire:
            since_last = 0
        since_last += 1
        return fire

    return proposal_requires_grad_fn


def _stot_constants(transform_type: str, t_min: float, t_max: float) -> Tuple[float, float, bool]:
    if transform_type == "uniform":
        return float(t_min), float(t_max), False
    if transform_type == "lindisp":
        return 1 / t_min, 1 / t_max, True
    raise ValueError(f"Unknown transform_type: {transform_type}")


def _transform_stot(
    transform_type: Literal["uniform", "lindisp"],
    s_vals: torch.Tensor,
    t_min: torch.Tensor,
    t_max: torch.Tensor,
) -> torch.Tensor:
    """Normalised s in [0, 1] -> ray distance t (reference prop_net.py:215-229)."""
    if transform_type == "uniform":
        return s_vals * t_max + (1 - s_vals) * t_min
    if transform_type == "lindisp":
        return 1 / (s_vals * (1 / t_max) + (1 - s_vals) * (1 / t_min))
    raise ValueError(f"Unknown transform_type: {transform_type}")


def _pdf_loss(
    segments_query: RayIntervals,
    cdfs_query: torch.Tensor,
    segments_key: RayIntervals,
    cdfs_key: torch.Tensor,
    eps: float = 1e-7,
) -> torch.Tensor:
    """How much the query histogram exceeds the key histogram's envelope (reference prop_net.py:232-256).

    Batched float32 CUDA rows with the same leading shape run ``nfa_pdf_loss_fwd`` (and ``nfa_pdf_loss_bwd`` for the
    key cdfs' gradient): the values are :func:`_pdf_loss_torch`'s bit for bit, and the gradient is summed in a fixed
    order, so it is the same from run to run.  Everything else -- CPU tensors, flattened queries, other dtypes, a
    query cdf that needs a gradient (the kernels give none to the query side) -- runs :func:`_pdf_loss_torch`."""
    q, k = segments_query.vals, segments_key.vals
    native = (
        q.dim() > 1 and k.dim() > 1 and q.shape[:-1] == k.shape[:-1]
        and cdfs_query.shape == q.shape and cdfs_key.shape == k.shape
        and q.shape[-1] >= 1 and k.shape[-1] >= 1 and q.shape[-1] - 1 <= _lib.PDF_LOSS_MAX_INTERVALS
        and all(t.is_cuda and t.dtype == torch.float32 for t in (q, cdfs_query, k, cdfs_key))
        and not _grad_through(cdfs_query)
    )
    if not native:
        return _pdf_loss_torch(segments_query, cdfs_query, segments_key, cdfs_key, eps)
    if _grad_through(cdfs_key):
        return _PdfLoss.apply(q, cdfs_query, k, cdfs_key, eps)
    return _pdf_loss_fwd(q, cdfs_query, k, cdfs_key, eps)


def _loss_rows(q: Tensor, cq: Tensor, k: Tensor, ck: Tensor):
    """(R, Eq) and (R, Ek) contiguous rows of the batched operands."""
    eq, ek = q.shape[-1], k.shape[-1]
    return (q.reshape(-1, eq).contiguous(), cq.reshape(-1, eq).contiguous(), k.reshape(-1, ek).contiguous(),
            ck.reshape(-1, ek).contiguous())


def _pdf_loss_fwd(q: Tensor, cq: Tensor, k: Tensor, ck: Tensor, eps: float) -> Tensor:
    rq, rcq, rk, rck = _loss_rows(q, cq, k, ck)
    n_rays, eq, ek = rq.shape[0], rq.shape[1], rk.shape[1]
    loss = torch.empty(q.shape[:-1] + (eq - 1,), dtype=torch.float32, device=q.device)
    if loss.numel() > 0:
        _lib.call("nfa_pdf_loss_fwd", q.device, n_rays, eq, rq.data_ptr(), rcq.data_ptr(), ek, rk.data_ptr(),
                  rck.data_ptr(), eps, loss.data_ptr())
    return loss


class _PdfLoss(torch.autograd.Function):
    """Per-interval proposal loss; the gradient flows to the key cdfs only (``_pdf_loss`` routes the other cases)."""

    @staticmethod
    def forward(ctx, q: Tensor, cq: Tensor, k: Tensor, ck: Tensor, eps: float):
        ctx.save_for_backward(q, cq, k, ck)
        ctx.eps = eps
        return _pdf_loss_fwd(q, cq, k, ck, eps)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad: Tensor):
        q, cq, k, ck = ctx.saved_tensors
        rq, rcq, rk, rck = _loss_rows(q, cq, k, ck)
        n_rays, eq, ek = rq.shape[0], rq.shape[1], rk.shape[1]
        grad_ck = torch.empty(ck.shape, dtype=torch.float32, device=ck.device)
        if n_rays > 0:
            g = grad.reshape(n_rays, eq - 1).contiguous()
            _lib.call("nfa_pdf_loss_bwd", q.device, n_rays, eq, rq.data_ptr(), rcq.data_ptr(), ek, rk.data_ptr(),
                      rck.data_ptr(), ctx.eps, _lib.ptr(g) if g.numel() > 0 else None, grad_ck.data_ptr())
        return None, None, None, grad_ck, None


def _pdf_loss_torch(
    segments_query: RayIntervals,
    cdfs_query: torch.Tensor,
    segments_key: RayIntervals,
    cdfs_key: torch.Tensor,
    eps: float = 1e-7,
) -> torch.Tensor:
    """``_pdf_loss`` as ATen ops, the reference's formulation (prop_net.py:232-256)."""
    ids_left, ids_right = searchsorted(segments_key, segments_query)
    if segments_query.vals.dim() > 1:
        w = cdfs_query[..., 1:] - cdfs_query[..., :-1]
        ids_left, ids_right = ids_left[..., :-1], ids_right[..., 1:]
    else:
        assert segments_query.is_left is not None and segments_query.is_right is not None
        w = cdfs_query[segments_query.is_right] - cdfs_query[segments_query.is_left]
        ids_left, ids_right = ids_left[segments_query.is_left], ids_right[segments_query.is_right]
    w_outer = cdfs_key.gather(-1, ids_right) - cdfs_key.gather(-1, ids_left)
    return torch.clip(w - w_outer, min=0) ** 2 / (w + eps)


def _outer(t0_starts: Tensor, t0_ends: Tensor, t1_starts: Tensor, t1_ends: Tensor, y1: Tensor) -> Tensor:
    """Upper bound of histogram (t1, y1) over the bins of t0 (reference prop_net.py:259-293)."""
    cy1 = torch.cat([torch.zeros_like(y1[..., :1]), torch.cumsum(y1, dim=-1)], dim=-1)
    top = y1.shape[-1] - 1
    idx_lo = torch.searchsorted(t1_starts.contiguous(), t0_starts.contiguous(), side="right") - 1
    idx_hi = torch.searchsorted(t1_ends.contiguous(), t0_ends.contiguous(), side="right")
    idx_lo, idx_hi = idx_lo.clamp(0, top), idx_hi.clamp(0, top)
    return torch.take_along_dim(cy1[..., 1:], idx_hi, dim=-1) - torch.take_along_dim(cy1[..., :-1], idx_lo, dim=-1)


def _lossfun_outer(t: Tensor, w: Tensor, t_env: Tensor, w_env: Tensor) -> Tensor:
    """mip-NeRF 360 proposal loss on batched histograms (reference prop_net.py:296-313)."""
    eps = torch.finfo(t.dtype).eps
    w_outer = _outer(t[..., :-1], t[..., 1:], t_env[..., :-1], t_env[..., 1:], w_env)
    return torch.clip(w - w_outer, min=0) ** 2 / (w + eps)
