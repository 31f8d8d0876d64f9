"""Occupancy-grid estimator (Instant-NGP style empty-space skipping).

Mirrors /root/reference/nerfacc/estimators/occ_grid.py: same constructor,
buffers (so state_dicts interchange), `sampling` signature/returns (:85-221) and
grid-maintenance entry points (:224-404).  `sampling` runs on the native
traversal pipeline (grid._march); the occupancy bit-pack it consumes is a derived
cache keyed on the `binaries` tensor version, so assigning or mutating
`estimator.binaries` (reference :404, tests/test_grid.py:190) just works.
"""
from typing import Callable, List, Optional, Tuple, Union

import torch
from torch import Tensor

from ..grid import _enlarge_aabb, _MarchJob, traverse_grids
from .. import _lib
from ..pack import _stash_packed_info
from ..volrend import render_visibility_from_alpha, render_visibility_from_density
from .base import AbstractEstimator


class OccGridEstimator(AbstractEstimator):
    """Multi-level binary occupancy grid used to skip empty space while marching.

    Args:
        roi_aabb: region of interest {xmin, ymin, zmin, xmax, ymax, zmax}; level i covers it scaled by 2**i.
        resolution: cells per axis (int, or 3 ints).  Default 128.
        levels: number of nested levels.  Default 1.
    """

    DIM: int = 3

    def __init__(
        self,
        roi_aabb: Union[List[int], Tensor],
        resolution: Union[int, List[int], Tensor] = 128,
        levels: int = 1,
        **kwargs,
    ) -> None:
        super().__init__()
        if "contraction_type" in kwargs:
            raise ValueError("`contraction_type` is not supported anymore for nerfacc >= 0.4.0.")

        if isinstance(resolution, int):
            resolution = [resolution] * self.DIM
        if isinstance(resolution, (list, tuple)):
            resolution = torch.tensor(resolution, dtype=torch.int32)
        assert isinstance(resolution, Tensor), f"Invalid type: {resolution}!"
        assert resolution.shape[0] == self.DIM, f"Invalid shape: {resolution}!"

        if isinstance(roi_aabb, (list, tuple)):
            roi_aabb = torch.tensor(roi_aabb, dtype=torch.float32)
        assert isinstance(roi_aabb, Tensor), f"Invalid type: {roi_aabb}!"
        assert roi_aabb.shape[0] == self.DIM * 2, f"Invalid shape: {roi_aabb}!"

        aabbs = torch.stack([_enlarge_aabb(roi_aabb, 2**i) for i in range(levels)], dim=0)

        self.cells_per_lvl = int(resolution.prod().item())
        self.levels = levels

        # persistent state: names / shapes / dtypes as in the reference (occ_grid.py:67-76)
        self.register_buffer("resolution", resolution)  # [3]
        self.register_buffer("aabbs", aabbs)  # [levels, 6]
        self.register_buffer("occs", torch.zeros(self.levels * self.cells_per_lvl))
        self.register_buffer("binaries", torch.zeros([levels] + resolution.tolist(), dtype=torch.bool))

        # derived helpers (occ_grid.py:79-83)
        grid_coords = _meshgrid3d(resolution).reshape(self.cells_per_lvl, self.DIM)
        self.register_buffer("grid_coords", grid_coords, persistent=False)
        self.register_buffer("grid_indices", torch.arange(self.cells_per_lvl), persistent=False)

        # size of the previous sample batch: lets `sampling` launch the expand kernel
        # before the (single) host sync instead of after it
        self._capacity_hint = 0
        # ray-sharded data parallelism: all-reduce(max) `occs` in `_update` so that every replica thresholds the
        # same grid (the ranks evaluate `occ_eval_fn` at different random points).  Off by default.
        self.sync_across_ranks = False

    @torch.no_grad()
    def sampling(
        self,
        rays_o: Tensor,  # [n_rays, 3]
        rays_d: Tensor,  # [n_rays, 3]
        sigma_fn: Optional[Callable] = None,
        alpha_fn: Optional[Callable] = None,
        near_plane: float = 0.0,
        far_plane: float = 1e10,
        t_min: Optional[Tensor] = None,  # [n_rays]
        t_max: Optional[Tensor] = None,  # [n_rays]
        render_step_size: float = 1e-3,
        early_stop_eps: float = 1e-4,
        alpha_thre: float = 0.0,
        stratified: bool = False,
        cone_angle: float = 0.0,
    ) -> Tuple[Tensor, Tensor, Tensor]:
        """Place samples in occupied cells along each ray.

        Returns (ray_indices [N] int64, t_starts [N], t_ends [N]), grouped by ray in
        ascending order.  With `sigma_fn` / `alpha_fn`, samples that are occluded
        (transmittance < early_stop_eps) or transparent (alpha < alpha_thre) are dropped.
        Not differentiable.  Semantics: reference occ_grid.py:85-221.
        """
        fast = cone_angle >= 0.0 and render_step_size > 0.0 and rays_o.is_cuda
        if fast:
            ticket = self.sampling_begin(rays_o, rays_d, near_plane=near_plane, far_plane=far_plane, t_min=t_min,
                                         t_max=t_max, render_step_size=render_step_size, stratified=stratified,
                                         cone_angle=cone_angle)
            return self.sampling_end(ticket, sigma_fn=sigma_fn, alpha_fn=alpha_fn, early_stop_eps=early_stop_eps,
                                     alpha_thre=alpha_thre)
        near_planes, far_planes = self._ray_planes(rays_o, near_plane, far_plane, t_min, t_max, stratified,
                                                   render_step_size, always=True)
        intervals, samples, _ = traverse_grids(
            rays_o, rays_d, self.binaries, self.aabbs, near_planes=near_planes, far_planes=far_planes,
            step_size=render_step_size, cone_angle=cone_angle)
        t_starts = intervals.vals[intervals.is_left]
        t_ends = intervals.vals[intervals.is_right]
        return self._drop_invisible(samples.ray_indices, t_starts, t_ends, samples.packed_info, sigma_fn, alpha_fn,
                                    early_stop_eps, alpha_thre)

    @torch.no_grad()
    def sampling_begin(
        self,
        rays_o: Tensor,
        rays_d: Tensor,
        near_plane: float = 0.0,
        far_plane: float = 1e10,
        t_min: Optional[Tensor] = None,
        t_max: Optional[Tensor] = None,
        render_step_size: float = 1e-3,
        stratified: bool = False,
        cone_angle: float = 0.0,
    ):
        """First half of :meth:`sampling` (CUDA, render_step_size > 0, cone_angle >= 0): queue the traversal and
        return a ticket at once.

        The size of a batch is only known once the traversal has run, so ``sampling()`` has to wait for the GPU
        once per call -- on a training step that is host-bound that wait (and the kernel itself) sits on the
        critical path.  A loop that knows its next rays early can call ``sampling_begin`` for batch k+1 before
        ``loss.backward()`` of batch k and ``sampling_end`` at the top of step k+1: the traversal then runs behind
        the backward kernels while the host is busy, and ``sampling_end`` returns without waiting.  The occupancy
        grid is read when the traversal runs; call ``sampling_end`` before changing it.  With ``cone_angle > 0``
        (unbounded scenes: the step grows with the distance) the same split applies.  Not part of nerfacc's API.
        """
        if not (rays_o.is_cuda and render_step_size > 0.0 and cone_angle >= 0.0):
            raise ValueError("sampling_begin: only CUDA rays with render_step_size > 0 and cone_angle >= 0 can be "
                             "split; use sampling().")
        near_planes, far_planes = self._ray_planes(rays_o, near_plane, far_plane, t_min, t_max, stratified,
                                                   render_step_size, always=False)
        return _MarchJob(rays_o.contiguous().float(), rays_d.contiguous().float(), self.binaries,
                         self.aabbs.contiguous().float(), near_planes, far_planes, float(render_step_size), None, None,
                         None, want_intervals=False, want_terminate=False, capacity_hint=self._capacity_hint,
                         near_plane=float(near_plane), far_plane=float(far_plane),
                         cone_angle=float(cone_angle)).begin()

    @torch.no_grad()
    def sampling_end(
        self,
        ticket,
        sigma_fn: Optional[Callable] = None,
        alpha_fn: Optional[Callable] = None,
        early_stop_eps: float = 1e-4,
        alpha_thre: float = 0.0,
    ) -> Tuple[Tensor, Tensor, Tensor]:
        """Second half of :meth:`sampling`: wait for the traversal's sample count, return the samples (after the
        optional visibility filter)."""
        res = self._finish_march(ticket)
        return self._drop_invisible(res.ray_indices, res.t_starts, res.t_ends, res.packed_info, sigma_fn, alpha_fn,
                                    early_stop_eps, alpha_thre)

    def _finish_march(self, ticket):
        res = ticket.finish()
        # ~6% head-room over the last batch; re-measured every call
        self._capacity_hint = res.n_samples + (res.n_samples >> 4) + 1024
        return res

    @torch.no_grad()
    def sampling_until_opaque(
        self,
        rays_o: Tensor,  # [n_rays, 3]
        rays_d: Tensor,  # [n_rays, 3]
        sigma_fn: Optional[Callable] = None,
        alpha_fn: Optional[Callable] = None,
        near_plane: float = 0.0,
        far_plane: float = 1e10,
        t_min: Optional[Tensor] = None,  # [n_rays]
        t_max: Optional[Tensor] = None,  # [n_rays]
        render_step_size: float = 1e-3,
        early_stop_eps: float = 1e-4,
        alpha_thre: float = 0.0,
        stratified: bool = False,
        cone_angle: float = 0.0,
    ) -> Tuple[Tensor, Tensor, Tensor]:
        """:meth:`sampling` with the visibility filter's field evaluated in rounds: each round hands the closure the
        next k samples of every ray that is still live (k a multiple of 32, from 32 up to 256 as rays retire), and a
        ray retires once the transmittance its next sample would get fails T >= early_stop_eps.  Behind an opaque
        surface the field is no longer evaluated, where :meth:`sampling` evaluates it on every marched sample and
        then drops those samples.  Same arguments, defaults and return value as :meth:`sampling`:
        (ray_indices, t_starts, t_ends), grouped by ray, with their packed_info attached.  Not part of nerfacc's API.

        The results are bit-identical to ``sampling(...)`` with the same arguments (and the same RNG state when
        `stratified`) when
          - the closure is batch-invariant: each sample's output does not depend on which other samples share the
            call.  Elementwise torch ops are; a cuBLAS MLP may not be;
          - densities are >= 0 and alphas lie in [0, 1], as every activation of nerfacc's examples gives.
        The samples are those of :meth:`sampling`'s march.  Each round advances a ray by whole 32-sample blocks from
        its first sample and carries the transmittance scan across rounds, so every T, alpha and keep bit is the
        one-shot filter's; once T fails the threshold it fails for every later sample of the ray too.

        The closure is called once per round, never with zero samples.  Its inputs are grouped by ray in ascending
        order, each ray's samples in order, with indices into `rays_o`; each sample is handed over at most once.  It
        must return float32 (anything else raises RuntimeError) of shape (N,).  The host waits for the GPU once for
        the march, once per round and once after the last round.

        Without a closure, with early_stop_eps <= 0 (no ray can retire) or render_step_size <= 0 this is
        :meth:`sampling` itself (one closure call)."""
        _lib.require_cuda(rays_o, "sampling_until_opaque")
        kw = dict(near_plane=near_plane, far_plane=far_plane, t_min=t_min, t_max=t_max,
                  render_step_size=render_step_size, stratified=stratified, cone_angle=cone_angle)
        if (sigma_fn is None and alpha_fn is None) or not (early_stop_eps > 0.0) or not (render_step_size > 0.0) \
                or not (cone_angle >= 0.0):
            return self.sampling(rays_o, rays_d, sigma_fn=sigma_fn, alpha_fn=alpha_fn, early_stop_eps=early_stop_eps,
                                 alpha_thre=alpha_thre, **kw)
        res = self._finish_march(self.sampling_begin(rays_o, rays_d, **kw))
        if res.t_starts.shape[0] == 0 or res.packed_info.shape[0] == 0:  # nothing to evaluate: sampling's own path
            return self._drop_invisible(res.ray_indices, res.t_starts, res.t_ends, res.packed_info, sigma_fn,
                                        alpha_fn, early_stop_eps, alpha_thre)
        if alpha_thre > 0.0:
            alpha_thre = min(alpha_thre, self._occs_mean())
        use_sigma = sigma_fn is not None
        return _visibility_rounds(res.t_starts, res.t_ends, res.packed_info, sigma_fn if use_sigma else alpha_fn,
                                  not use_sigma, float(early_stop_eps), float(alpha_thre))

    @staticmethod
    def _ray_planes(rays_o, near_plane, far_plane, t_min, t_max, stratified, render_step_size, always: bool):
        """Per-ray near / far planes (reference occ_grid.py:152-163), or (None, None) when the two scalars do."""
        if not (always or t_min is not None or t_max is not None or stratified):
            return None, None  # the kernel takes the two scalars directly
        near_planes = torch.full_like(rays_o[..., 0], fill_value=near_plane)
        far_planes = torch.full_like(rays_o[..., 0], fill_value=far_plane)
        if t_min is not None:
            near_planes = torch.clamp(near_planes, min=t_min)
        if t_max is not None:
            far_planes = torch.clamp(far_planes, max=t_max)
        if stratified:
            near_planes += torch.rand_like(near_planes) * render_step_size
        return near_planes.contiguous().float(), far_planes.contiguous().float()

    def _drop_invisible(self, ray_indices, t_starts, t_ends, packed_info, sigma_fn, alpha_fn, early_stop_eps,
                        alpha_thre):
        """The visibility filter of `sampling` (occ_grid.py:180-220)."""
        if not ((alpha_thre > 0.0 or early_stop_eps > 0.0) and (sigma_fn is not None or alpha_fn is not None)):
            return ray_indices, t_starts, t_ends
        if alpha_thre > 0.0:  # min(0, mean) can never enable the alpha test, so the mean is only needed here
            alpha_thre = min(alpha_thre, self._occs_mean())
        use_sigma = sigma_fn is not None
        if t_starts.shape[0] != 0:
            dens = (sigma_fn if use_sigma else alpha_fn)(t_starts, t_ends, ray_indices)
        else:
            dens = torch.empty((0,), device=t_starts.device)
        assert dens.shape == t_starts.shape, "{} must have shape of (N,)! Got {}".format(
            "sigmas" if use_sigma else "alphas", dens.shape)
        if t_starts.is_cuda and dens.dtype == torch.float32:
            return _visibility_compact(t_starts, t_ends, dens.detach(), packed_info, from_alpha=not use_sigma,
                                       early_stop_eps=float(early_stop_eps), alpha_thre=float(alpha_thre))
        if use_sigma:
            masks = render_visibility_from_density(t_starts=t_starts, t_ends=t_ends, sigmas=dens,
                                                   packed_info=packed_info, early_stop_eps=early_stop_eps,
                                                   alpha_thre=alpha_thre)
        else:
            masks = render_visibility_from_alpha(alphas=dens, packed_info=packed_info,
                                                 early_stop_eps=early_stop_eps, alpha_thre=alpha_thre)
        return ray_indices[masks], t_starts[masks], t_ends[masks]

    @torch.no_grad()
    def render_test(
        self,
        rays_o: Tensor,  # [n_rays, 3]
        rays_d: Tensor,  # [n_rays, 3]
        rgb_sigma_fn: Callable,
        max_samples: int,
        near_plane: float = 0.0,
        far_plane: float = 1e10,
        render_step_size: float = 1e-3,
        render_bkgd: Optional[Tensor] = None,
        cone_angle: float = 0.0,
        alpha_thre: float = 0.0,
        early_stop_eps: float = 1e-4,
    ) -> Tuple[Tensor, Tensor, Tensor, int]:
        """Render an evaluation image with early ray termination: march every live ray a few samples at a time,
        shade only those samples, composite them onto the running result and retire a ray once it is opaque
        (opacity > 1 - early_stop_eps) or has left the grid, until no ray is live or `max_samples` samples per ray
        have been asked for.  Field work stops where the surfaces are, and a round needs memory for at most
        n_alive x n_samples samples.  Not part of nerfacc's API.

        Its results are those of the test-mode loop of nerfacc's examples (examples/utils.py:267-439,
        `render_image_with_occgrid_test`): the same rounds, the same samples handed to the field in each round,
        and colours, opacities and depths of the same arithmetic, summed without atomics (so two runs give the same
        image).  `rgb_sigma_fn(t_starts, t_ends, ray_indices) -> (rgbs (N, 3), sigmas (N,))` is `rendering`'s closure,
        with ray indices into `rays_o`; it must return float32.  Returns (colors (R, 3), opacities (R, 1), depths (R, 1),
        total_samples): depths are normalised by the opacity, `render_bkgd` is blended in where given, and
        total_samples counts the samples that passed `alpha_thre`.

        Each round waits for the GPU once, for its sample count (plus one wait at the end when `max_samples` stops
        the loop, for the sample total).  `render_step_size <= 0` (one sample per cell) runs the loop over the public
        functions instead.  Inference only."""
        _lib.require_cuda(rays_o, "render_test")
        if render_step_size > 0.0:
            return _render_test_native(self, rays_o, rays_d, rgb_sigma_fn, int(max_samples), float(near_plane),
                                       float(far_plane), float(render_step_size), render_bkgd, float(cone_angle),
                                       float(alpha_thre), float(early_stop_eps))
        return _render_test_public(self, rays_o, rays_d, rgb_sigma_fn, int(max_samples), near_plane, far_plane,
                                   render_step_size, render_bkgd, cone_angle, alpha_thre, early_stop_eps)

    def _occs_mean(self) -> float:
        """`occs.mean()` (reference occ_grid.py:183), cached per version of the buffer: the reference pays a
        2M-element reduction and a host sync for it on every sampling call."""
        key = (self.occs.data_ptr(), self.occs._version)
        if getattr(self, "_occs_mean_key", None) != key:
            self._occs_mean_val = float(self.occs.mean().item())
            self._occs_mean_key = key
        return self._occs_mean_val

    # ------------------------------------------------------------------
    # grid maintenance (occ_grid.py:224-404)
    # ------------------------------------------------------------------
    @torch.no_grad()
    def update_every_n_steps(
        self,
        step: int,
        occ_eval_fn: Callable,
        occ_thre: float = 1e-2,
        ema_decay: float = 0.95,
        warmup_steps: int = 256,
        n: int = 16,
    ) -> None:
        """Refresh the grid every `n` training steps by evaluating `occ_eval_fn` at cell samples."""
        if not self.training:
            raise RuntimeError(
                "You should only call this function only during training. "
                "Please call _update() directly if you want to update the "
                "field during inference."
            )
        if step % n == 0 and self.training:
            self._update(step=step, occ_eval_fn=occ_eval_fn, occ_thre=occ_thre, ema_decay=ema_decay,
                         warmup_steps=warmup_steps)

    @torch.no_grad()
    def mark_invisible_cells(
        self,
        K: Tensor,
        c2w: Tensor,
        width: int,
        height: int,
        near_plane: float = 0.0,
        chunk: int = 32**3,
    ) -> None:
        """Give cells no camera covers an occupancy of -1 so they are never sampled.

        K: (N, 3, 3) or (1, 3, 3) intrinsics; c2w: (N, 3, 4) or (N, 4, 4) poses.
        A cell stays valid (0) when at least one camera sees it in front of
        `near_plane` and no camera has it inside the image but closer than `near_plane`.
        """
        assert K.dim() == 3 and K.shape[1:] == (3, 3)
        assert c2w.dim() == 3 and (c2w.shape[1:] == (3, 4) or c2w.shape[1:] == (4, 4))
        assert K.shape[0] == c2w.shape[0] or K.shape[0] == 1

        n_cams = c2w.shape[0]
        rot_w2c = c2w[:, :3, :3].transpose(2, 1)  # (n_cams, 3, 3)
        trans_w2c = -rot_w2c @ c2w[:, :3, 3:]  # (n_cams, 3, 1)

        for lvl, indices in enumerate(self._get_all_cells()):
            coords = self.grid_coords[indices]
            lo, extent = self.aabbs[lvl, :3], self.aabbs[lvl, 3:] - self.aabbs[lvl, :3]
            for i in range(0, len(indices), chunk):
                ids = indices[i : i + chunk]
                unit = coords[i : i + chunk] / (self.resolution - 1)
                pts_w = (lo + unit * extent).T  # (3, chunk)
                uvd = K @ (rot_w2c @ pts_w + trans_w2c)  # (n_cams, 3, chunk)
                depth = uvd[:, 2]
                uv = uvd[:, :2] / uvd[:, 2:]
                in_image = (depth >= 0) & (uv[:, 0] >= 0) & (uv[:, 0] < width) & (uv[:, 1] >= 0) & (uv[:, 1] < height)
                seen = ((depth >= near_plane) & in_image).sum(0) / n_cams > 0
                too_close = ((depth < near_plane) & in_image).any(0)
                keep = seen & ~too_close
                self.occs[lvl * self.cells_per_lvl + ids] = torch.where(keep, 0.0, -1.0)

    @torch.no_grad()
    def _get_all_cells(self) -> List[Tensor]:
        """Per level: every cell not marked invisible (occupancy >= 0)."""
        out = []
        for lvl in range(self.levels):
            occ = self.occs[lvl * self.cells_per_lvl + self.grid_indices]
            out.append(self.grid_indices[occ >= 0.0])
        return out

    @torch.no_grad()
    def _sample_uniform_and_occupied_cells(self, n: int) -> List[Tensor]:
        """Per level: `n` uniformly drawn cells plus up to `n` currently occupied ones."""
        out = []
        for lvl in range(self.levels):
            uniform = torch.randint(self.cells_per_lvl, (n,), device=self.device)
            uniform = uniform[self.occs[lvl * self.cells_per_lvl + uniform] >= 0.0]
            occupied = torch.nonzero(self.binaries[lvl].flatten())[:, 0]
            if n < len(occupied):
                pick = torch.randint(len(occupied), (n,), device=self.device)
                occupied = occupied[pick]
            out.append(torch.cat([uniform, occupied], dim=0))
        return out

    @torch.no_grad()
    def _update(
        self,
        step: int,
        occ_eval_fn: Callable,
        occ_thre: float = 0.01,
        ema_decay: float = 0.95,
        warmup_steps: int = 256,
    ) -> None:
        """EMA-max update of `occs` at sampled cells, then re-threshold into `binaries` (reference :367-404).

        On the GPU the arithmetic runs in csrc/occ_update.cu: the EMA-max at the sampled cells, then ONE pass that
        takes the mean of the visible cells, thresholds, and writes both the bool grid and the traversal's packed
        form of it -- no host synchronisation, and the next `sampling()` finds its derived cache ready.  Cell
        sampling and the user's `occ_eval_fn` stay in torch (same random streams as the reference)."""
        if step < warmup_steps:
            per_level = self._get_all_cells()
        else:
            per_level = self._sample_uniform_and_occupied_cells(self.cells_per_lvl // 4)

        native = self.occs.is_cuda and self.occs.dtype == torch.float32 and self.occs.is_contiguous()
        for lvl, indices in enumerate(per_level):
            coords = self.grid_coords[indices]
            unit = (coords + torch.rand_like(coords, dtype=torch.float32)) / self.resolution
            pts = self.aabbs[lvl, :3] + unit * (self.aabbs[lvl, 3:] - self.aabbs[lvl, :3])
            occ = occ_eval_fn(pts).squeeze(-1)
            cell_ids = lvl * self.cells_per_lvl + indices
            if native and occ.is_cuda:
                n = cell_ids.shape[0]
                if n:
                    ids, val = cell_ids.contiguous(), occ.detach().to(torch.float32).contiguous()
                    scratch = torch.empty(n, dtype=torch.float32, device=self.occs.device)
                    _lib.call("nfa_occ_ema_update", self.occs.device, n, _lib.ptr(ids), _lib.ptr(val), float(ema_decay),
                              _lib.ptr(self.occs), _lib.ptr(scratch))
            else:
                self.occs[cell_ids] = torch.maximum(self.occs[cell_ids] * ema_decay, occ)
        if self.sync_across_ranks:  # keep the replicas of a ray-sharded job on one grid (SURVEY 8e)
            from ..parallel import all_reduce_max_
            all_reduce_max_(self.occs)
        if native:
            self._threshold_native(float(occ_thre))
        else:
            thre = torch.clamp(self.occs[self.occs >= 0].mean(), max=occ_thre)
            self.binaries = (self.occs > thre).view(self.binaries.shape)

    def _threshold_native(self, occ_thre: float) -> None:
        """binaries = occs > min(mean(occs[occs >= 0]), occ_thre), written together with its packed form."""
        from ..grid import _OccPack
        lib = _lib.load()
        device, shape = self.occs.device, tuple(int(v) for v in self.binaries.shape)
        binaries = torch.empty(shape, dtype=torch.bool, device=device)
        pack = _OccPack(None, shape=shape, device=device)
        ws = torch.empty(lib.nfa_occ_threshold_workspace_bytes(self.occs.numel()), dtype=torch.uint8, device=device)
        _lib.call("nfa_occ_threshold_pack", device, shape[0], shape[1], shape[2], shape[3], _lib.ptr(self.occs), occ_thre,
                  _lib.ptr(binaries), _lib.ptr(pack.words), _lib.ptr(pack.coarse), _lib.ptr(pack.bounds), _lib.ptr(ws))
        self.binaries = binaries
        binaries._nfa_occ = (binaries._version, pack)  # grid._packed_grid: the derived cache is already there
        self._occs_mean_key = None  # occs changed behind torch's version counter


_vis_scratch = {}


def _visibility_compact(t_starts: Tensor, t_ends: Tensor, dens: Tensor, packed_info: Tensor, from_alpha: bool,
                        early_stop_eps: float, alpha_thre: float):
    """Fused visibility test + compaction (nfa_visibility_compact): returns the kept
    (ray_indices, t_starts, t_ends), grouped by ray, with their packed_info attached."""
    device = t_starts.device
    n, n_rays = t_starts.shape[0], packed_info.shape[0]
    lib = _lib.load()
    pi = packed_info.contiguous()
    if pi.dtype != torch.int64:
        pi = pi.to(torch.int64)
    key = (device, _lib.stream_ptr(device))  # per stream: the pinned count slot is protected by stream order only
    sc = _vis_scratch.get(key)
    if sc is None:
        if len(_vis_scratch) >= 16:
            _vis_scratch.clear()
        sc = _vis_scratch[key] = (torch.zeros(1, dtype=torch.int64).pin_memory(), torch.cuda.Event())
    total_host, event = sc
    ws = torch.empty(lib.nfa_visibility_workspace_bytes(n_rays, n), dtype=torch.uint8, device=device)
    new_pi = torch.empty((n_rays, 2), dtype=torch.int64, device=device)
    out_ri = torch.empty(n, dtype=torch.int64, device=device)
    out_ts = torch.empty(n, dtype=torch.float32, device=device)
    out_te = torch.empty(n, dtype=torch.float32, device=device)
    if n_rays == 0:
        return out_ri, out_ts, out_te
    _lib.call("nfa_visibility_compact", device, n_rays, n, _lib.ptr(pi), _lib.ptr(t_starts.contiguous()),
              _lib.ptr(t_ends.contiguous()), _lib.ptr(dens.contiguous()), int(from_alpha), early_stop_eps, alpha_thre,
              _lib.ptr(ws), _lib.ptr(new_pi), _lib.ptr(out_ri), _lib.ptr(out_ts), _lib.ptr(out_te), None,
              _lib.ptr(total_host))
    event.record(torch.cuda.current_stream(device))
    event.synchronize()  # the one sync of this stage: the kept count
    kept = int(total_host.item())
    out_ri, out_ts, out_te = out_ri[:kept], out_ts[:kept], out_te[:kept]
    _stash_packed_info(out_ri, new_pi, n_rays)
    return out_ri, out_ts, out_te


def _visibility_rounds(t_starts: Tensor, t_ends: Tensor, packed_info: Tensor, fn: Callable, from_alpha: bool,
                       early_stop_eps: float, alpha_thre: float):
    """The visibility filter in rounds (csrc/scan.cu, nfa_vis_rounds_*): per round one host wait (for the round's
    live rays and sample count, computed on the device), the gather of the closure's inputs, the closure, the step.
    Returns the kept (ray_indices, t_starts, t_ends) with their packed_info attached."""
    from ..volrend import _f32c
    device = t_starts.device
    n, n_rays = t_starts.shape[0], packed_info.shape[0]
    pi = packed_info.contiguous()
    if pi.dtype != torch.int64:
        pi = pi.to(torch.int64)
    ts, te = t_starts.contiguous(), t_ends.contiguous()
    sc = _stream_scratch(_vr_scratch, device)
    sc.reserve(_lib.load().nfa_vis_rounds_workspace_bytes(n_rays, n))
    ws, status = _lib.ptr(sc.workspace), sc.status_np
    stream = torch.cuda.current_stream(device)
    _lib.call("nfa_vis_rounds_begin", device, n_rays, n, _lib.ptr(pi), int(from_alpha), ws, _lib.ptr(sc.status))
    rnd, n_with_samples = 0, -1
    while True:
        sc.event.record(stream)
        sc.event.synchronize()  # the round's one wait: its live rays, sample count and the kept total so far
        n_alive, m = int(status[0]), int(status[2])
        if rnd == 0:
            n_with_samples = n_alive
        if n_alive == 0:
            kept = int(status[3])
            break
        ray_indices = torch.empty(m, dtype=torch.int64, device=device)
        r_starts = torch.empty(m, dtype=torch.float32, device=device)
        r_ends = torch.empty(m, dtype=torch.float32, device=device)
        _lib.call("nfa_vis_rounds_gather", device, n_rays, n, rnd, n_alive, _lib.ptr(pi), _lib.ptr(ts), _lib.ptr(te),
                  ws, _lib.ptr(ray_indices), _lib.ptr(r_starts), _lib.ptr(r_ends))
        dens = fn(r_starts, r_ends, ray_indices)
        assert dens.shape == r_starts.shape, "{} must have shape of (N,)! Got {}".format(
            "alphas" if from_alpha else "sigmas", dens.shape)
        dens = _f32c(dens.detach())
        _lib.call("nfa_vis_rounds_step", device, n_rays, n, rnd, n_alive, n_with_samples, _lib.ptr(pi),
                  _lib.ptr(r_starts), _lib.ptr(r_ends), _lib.ptr(dens), int(from_alpha), early_stop_eps, alpha_thre,
                  ws, _lib.ptr(sc.status))
        rnd += 1
    new_pi = torch.empty((n_rays, 2), dtype=torch.int64, device=device)
    out_ri = torch.empty(max(kept, 1), dtype=torch.int64, device=device)
    out_ts = torch.empty(max(kept, 1), dtype=torch.float32, device=device)
    out_te = torch.empty(max(kept, 1), dtype=torch.float32, device=device)
    _lib.call("nfa_vis_rounds_finish", device, n_rays, n, _lib.ptr(pi), _lib.ptr(ts), _lib.ptr(te), ws,
              _lib.ptr(new_pi), _lib.ptr(out_ri), _lib.ptr(out_ts), _lib.ptr(out_te))
    out_ri, out_ts, out_te = out_ri[:kept], out_ts[:kept], out_te[:kept]
    _stash_packed_info(out_ri, new_pi, n_rays)
    return out_ri, out_ts, out_te


class _StreamScratch:
    """Workspace, pinned status slot and event of a loop in rounds (render_test, sampling_until_opaque) for one
    (device, stream); the workspace only grows."""

    def __init__(self, device):
        self.device = device
        self.workspace = None
        self.status = torch.zeros(4, dtype=torch.int64).pin_memory()
        self.status_np = self.status.numpy()  # same pinned memory
        self.event = torch.cuda.Event()

    def reserve(self, need: int) -> None:
        if self.workspace is None or self.workspace.numel() < need:
            # zeroed: render_test's kernels expect (and leave behind) zero arrival counters
            self.workspace = torch.zeros(need, dtype=torch.uint8, device=self.device)


def _stream_scratch(table: dict, device) -> _StreamScratch:
    key = (device, _lib.stream_ptr(device))  # per stream: stream order is what protects the workspace
    sc = table.get(key)
    if sc is None:
        if len(table) >= 16:
            table.clear()
        sc = table[key] = _StreamScratch(device)
    return sc


_rt_scratch: dict = {}
_vr_scratch: dict = {}


def _render_test_scratch(device, n_rays: int, min_samples: int) -> _StreamScratch:
    sc = _stream_scratch(_rt_scratch, device)
    sc.reserve(_lib.load().nfa_render_test_workspace_bytes(n_rays, min_samples))
    return sc


def _render_test_native(est, rays_o, rays_d, rgb_sigma_fn, max_samples: int, near_plane: float, far_plane: float,
                        step_size: float, render_bkgd, cone_angle: float, alpha_thre: float, early_stop_eps: float):
    """OccGridEstimator.render_test on csrc/render_test.cu: per round march (one host wait, for the round's
    n_alive / n_samples / sample count, all computed on the device), expand, the field, composite."""
    from ..grid import _packed_grid, _sorted_crossings
    from ..volrend import _f32c
    device = rays_o.device
    rays_o, rays_d = rays_o.contiguous().float(), rays_d.contiguous().float()
    aabbs = est.aabbs.contiguous().float()
    R = rays_o.shape[0]
    colors = torch.zeros((R, 3), dtype=torch.float32, device=device)
    opacities = torch.zeros((R, 1), dtype=torch.float32, device=device)
    depths = torch.zeros((R, 1), dtype=torch.float32, device=device)
    if R == 0:
        return colors, opacities, depths, 0
    bkgd = None if render_bkgd is None else render_bkgd.to(device=device, dtype=torch.float32).reshape(3).contiguous()
    G, rx, ry, rz = (int(s) for s in est.binaries.shape)
    occ = _packed_grid(est.binaries)
    t_sorted, t_indices, hits = _sorted_crossings(rays_o, rays_d, aabbs, G)
    min_samples = 1 if cone_angle == 0 else 4  # examples/utils.py:322
    # `opacity <= 1 - early_stop_eps` compares in float32 (examples/utils.py:425): round the threshold once, here
    opacity_thre = float(torch.tensor(1.0 - early_stop_eps, dtype=torch.float32))
    sc = _render_test_scratch(device, R, min_samples)
    ws, status = _lib.ptr(sc.workspace), sc.status_np
    stream = torch.cuda.current_stream(device)
    _lib.call("nfa_render_test_begin", device, R, min_samples, near_plane, ws)
    iter_samples, k, total = 0, 0, None
    while iter_samples < max_samples:
        _lib.call("nfa_render_test_march", device, R, min_samples, k, _lib.ptr(rays_o), _lib.ptr(rays_d), far_plane, G,
                  rx, ry, rz, _lib.ptr(occ.words), _lib.ptr(occ.coarse), _lib.ptr(aabbs), _lib.ptr(t_sorted),
                  _lib.ptr(t_indices), _lib.ptr(hits), step_size, cone_angle, ws, _lib.ptr(sc.status))
        sc.event.record(stream)
        sc.event.synchronize()  # the round's one wait
        n_alive, n_samples, n = int(status[0]), int(status[1]), int(status[2])
        if n_alive == 0:
            total = int(status[3])  # every composite has run: the kept total is complete
            break
        iter_samples += n_samples
        ray_indices = torch.empty(n, dtype=torch.int64, device=device)
        t_starts = torch.empty(n, dtype=torch.float32, device=device)
        t_ends = torch.empty(n, dtype=torch.float32, device=device)
        if n:
            _lib.call("nfa_render_test_expand", device, R, min_samples, k, n_alive, n_samples, ws,
                      _lib.ptr(ray_indices), _lib.ptr(t_starts), _lib.ptr(t_ends))
        rgbs, sigmas = rgb_sigma_fn(t_starts, t_ends, ray_indices)
        assert rgbs.shape == (n, 3), "rgbs must have shape (N, 3), got {}".format(tuple(rgbs.shape))
        assert sigmas.shape == (n,), "sigmas must have shape (N,), got {}".format(tuple(sigmas.shape))
        rgbs, sigmas = _f32c(rgbs.detach()), _f32c(sigmas.detach())
        _lib.call("nfa_render_test_composite", device, R, min_samples, k, n_alive, n_samples, n, ws,
                  _lib.ptr(t_starts), _lib.ptr(t_ends), _lib.ptr(rgbs), _lib.ptr(sigmas), alpha_thre, opacity_thre,
                  _lib.ptr(colors), _lib.ptr(opacities), _lib.ptr(depths))
        k += 1
    _lib.call("nfa_render_test_finish", device, R, min_samples, ws, _lib.ptr(bkgd), _lib.ptr(colors),
              _lib.ptr(opacities), _lib.ptr(depths), None if (total is not None or k == 0) else _lib.ptr(sc.status))
    if total is None:
        if k > 0:  # the sample budget ended the loop: the last composite's kept samples are still on the device
            sc.event.record(stream)
            sc.event.synchronize()
            total = int(status[3])
        else:
            total = 0
    return colors, opacities, depths, total


def _render_test_public(est, rays_o, rays_d, rgb_sigma_fn, max_samples: int, near_plane, far_plane, step_size,
                        render_bkgd, cone_angle, alpha_thre, early_stop_eps):
    """render_test as the reference's loop over the public functions (examples/utils.py:314-439)."""
    from ..grid import ray_aabb_intersect
    from ..volrend import accumulate_along_rays_, render_weight_from_density
    device, R = rays_o.device, rays_o.shape[0]
    opacity = torch.zeros(R, 1, device=device)
    depth = torch.zeros(R, 1, device=device)
    rgb = torch.zeros(R, 3, device=device)
    ray_mask = torch.ones(R, device=device).bool()
    min_samples = 1 if cone_angle == 0 else 4
    iter_samples = total_samples = 0
    near_planes = torch.full_like(rays_o[..., 0], fill_value=near_plane)
    far_planes = torch.full_like(rays_o[..., 0], fill_value=far_plane)
    t_mins, t_maxs, hits = ray_aabb_intersect(rays_o, rays_d, est.aabbs)
    n_grids = est.binaries.size(0)
    if n_grids > 1:
        t_sorted, t_indices = torch.sort(torch.cat([t_mins, t_maxs], -1), -1)
    else:
        t_sorted = torch.cat([t_mins, t_maxs], -1)
        t_indices = torch.arange(0, n_grids * 2, device=device, dtype=torch.int64).expand(R, n_grids * 2)
    opc_thre = 1 - early_stop_eps
    while iter_samples < max_samples:
        n_alive = int(ray_mask.sum().item())
        if n_alive == 0:
            break
        n_samples = max(min(R // n_alive, 64), min_samples)
        iter_samples += n_samples
        intervals, samples, termination_planes = traverse_grids(
            rays_o, rays_d, est.binaries, est.aabbs, near_planes, far_planes, step_size, cone_angle, n_samples, True,
            ray_mask, t_sorted, t_indices, hits)
        t_starts = intervals.vals[intervals.is_left]
        t_ends = intervals.vals[intervals.is_right]
        ray_indices = samples.ray_indices[samples.is_valid]
        packed_info = samples.packed_info
        rgbs, sigmas = rgb_sigma_fn(t_starts, t_ends, ray_indices)
        weights, _, alphas = render_weight_from_density(t_starts, t_ends, sigmas, ray_indices=ray_indices, n_rays=R,
                                                        prefix_trans=1 - opacity[ray_indices].squeeze(-1))
        if alpha_thre > 0:
            vis = alphas >= alpha_thre
            ray_indices, rgbs, weights, t_starts, t_ends = (ray_indices[vis], rgbs[vis], weights[vis], t_starts[vis],
                                                            t_ends[vis])
        accumulate_along_rays_(weights, values=rgbs, ray_indices=ray_indices, outputs=rgb)
        accumulate_along_rays_(weights, values=None, ray_indices=ray_indices, outputs=opacity)
        accumulate_along_rays_(weights, values=(t_starts + t_ends)[..., None] / 2.0, ray_indices=ray_indices,
                               outputs=depth)
        near_planes = termination_planes
        ray_mask = torch.logical_and(opacity.view(-1) <= opc_thre, packed_info[:, 1] == n_samples)
        total_samples += ray_indices.shape[0]
    if render_bkgd is not None:
        rgb = rgb + render_bkgd * (1.0 - opacity)
    depth = depth / opacity.clamp_min(torch.finfo(torch.float32).eps)
    return rgb, opacity, depth, total_samples


def _meshgrid3d(res: Tensor, device: Union[torch.device, str] = "cpu") -> Tensor:
    """(rx, ry, rz, 3) integer cell coordinates."""
    assert len(res) == 3
    rx, ry, rz = res.tolist()
    axes = [torch.arange(n, dtype=torch.long) for n in (rx, ry, rz)]
    return torch.stack(torch.meshgrid(axes, indexing="ij"), dim=-1).to(device)
