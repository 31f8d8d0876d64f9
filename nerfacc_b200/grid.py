"""Ray/box intersection and occupancy-grid traversal.

Public names, arguments and return types mirror /root/reference/nerfacc/grid.py
(ray_aabb_intersect :13-51, traverse_grids :93-192, helpers :54-90,195-237).

`traverse_grids` drives the native pipeline of csrc/traverse.cu:
pack the bool grid to brick words (cached) -> march (one DDA pass, runs) ->
expand (coalesced per-sample arrays).  One host synchronisation per call, to
learn the output size -- the reference needs two (data_spec.hpp:90-91) plus
those of the boolean-mask selects in its callers.
"""
from typing import Dict, Optional, Tuple

import torch
from torch import Tensor

from . import _lib
from .data_specs import RayIntervals, RaySamples
from .pack import _stash_packed_info


@torch.no_grad()
def ray_aabb_intersect(
    rays_o: Tensor,
    rays_d: Tensor,
    aabbs: Tensor,
    near_plane: float = -float("inf"),
    far_plane: float = float("inf"),
    miss_value: float = float("inf"),
) -> Tuple[Tensor, Tensor, Tensor]:
    """Slab test of every ray against every box.

    Returns (t_mins, t_maxs, hits), each (n_rays, m); misses hold `miss_value`
    (reference grid.py:13-51 -> csrc/grid.cu:284-313).
    """
    assert rays_o.ndim == 2 and rays_o.shape[-1] == 3
    assert rays_d.ndim == 2 and rays_d.shape[-1] == 3
    assert aabbs.ndim == 2 and aabbs.shape[-1] == 6
    _lib.require_cuda(rays_o, "ray_aabb_intersect")
    rays_o, rays_d, aabbs = rays_o.contiguous().float(), rays_d.contiguous().float(), aabbs.contiguous().float()
    n_rays, m = rays_o.shape[0], aabbs.shape[0]
    device = rays_o.device
    t_mins = torch.empty((n_rays, m), dtype=torch.float32, device=device)
    t_maxs = torch.empty((n_rays, m), dtype=torch.float32, device=device)
    hits = torch.empty((n_rays, m), dtype=torch.bool, device=device)
    if n_rays * m > 0:
        _lib.call("nfa_ray_aabb_intersect", device, n_rays, _lib.ptr(rays_o), _lib.ptr(rays_d), m, _lib.ptr(aabbs),
                  float(near_plane), float(far_plane), float(miss_value), _lib.ptr(t_mins), _lib.ptr(t_maxs),
                  _lib.ptr(hits))
    return t_mins, t_maxs, hits


def _ray_aabb_intersect(
    rays_o: Tensor,
    rays_d: Tensor,
    aabbs: Tensor,
    near_plane: float = -float("inf"),
    far_plane: float = float("inf"),
    miss_value: float = float("inf"),
) -> Tuple[Tensor, Tensor, Tensor]:
    """Plain-torch slab test with the same outputs as :func:`ray_aabb_intersect` (test helper)."""
    lo, hi = aabbs[None, :, :3], aabbs[None, :, 3:]
    o, d = rays_o[:, None, :], rays_d[:, None, :]
    ta, tb = (lo - o) / d, (hi - o) / d
    t_mins = torch.minimum(ta, tb).amax(dim=-1)
    t_maxs = torch.maximum(ta, tb).amin(dim=-1)
    hits = (t_maxs > t_mins) & (t_maxs > 0)
    t_mins = torch.where(hits, t_mins.clamp(near_plane, far_plane), torch.full_like(t_mins, miss_value))
    t_maxs = torch.where(hits, t_maxs.clamp(near_plane, far_plane), torch.full_like(t_maxs, miss_value))
    return t_mins, t_maxs, hits


# --------------------------------------------------------------------------
# native traversal plumbing
# --------------------------------------------------------------------------

class _OccPack:
    """Brick-packed copy of a bool grid; derived, never persisted (SURVEY section 5)."""

    __slots__ = ("words", "coarse", "bounds", "shape")

    def __init__(self, binaries: Optional[Tensor], shape=None, device=None):
        """Pack `binaries`; or, with `binaries=None`, only allocate for `shape` on `device` (the grid-update
        kernel then fills bool grid and pack in one pass, estimators/occ_grid.py `_update`)."""
        lib = _lib.load()
        if binaries is not None:
            shape, device = binaries.shape, binaries.device
        g, rx, ry, rz = (int(s) for s in shape)
        self.shape = (g, rx, ry, rz)
        self.words = torch.empty(lib.nfa_occ_words(g, rx, ry, rz), dtype=torch.int64, device=device)
        self.coarse = torch.empty(lib.nfa_occ_coarse_words(g, rx, ry, rz), dtype=torch.int32, device=device)
        self.bounds = torch.empty(6 * g, dtype=torch.int32, device=device)
        if binaries is not None:
            b = binaries.contiguous()
            if b.dtype != torch.bool:
                b = b != 0
            _lib.call("nfa_occ_pack", device, g, rx, ry, rz, _lib.ptr(b), _lib.ptr(self.words), _lib.ptr(self.coarse),
                      _lib.ptr(self.bounds))


def _packed_grid(binaries: Tensor) -> _OccPack:
    """Brick-pack `binaries`, cached ON the tensor object and keyed by its version counter.

    The cache dies with the tensor and is invalidated by any in-place write, so
    `estimator.binaries = new` / `estimator.binaries[...] = x` are both picked up
    (a pointer-keyed cache is not safe: the allocator recycles addresses).
    """
    hit = getattr(binaries, "_nfa_occ", None)
    if hit is not None and hit[0] == binaries._version and hit[1].shape == tuple(int(s) for s in binaries.shape):
        return hit[1]
    pack = _OccPack(binaries)
    binaries._nfa_occ = (binaries._version, pack)
    return pack


class _MarchScratch:
    """Reusable march workspace (counts, tile sums, run pool) + pinned read-back slot of one (device, stream).

    It is sized for the largest batch seen and only ever grows: training loops that resize their ray batch every
    step (the reference's own NGP loop does, to hit a target sample count) would otherwise allocate a new pinned
    buffer -- a synchronising cudaHostAlloc -- on nearly every call."""

    def __init__(self, device):
        self.device = device
        self.run_capacity = 0
        self.workspace = None
        self.totals_dev = torch.zeros(4, dtype=torch.int64, device=device)
        self.totals_host = torch.zeros(4, dtype=torch.int64).pin_memory()
        self.totals_np = self.totals_host.numpy()  # same pinned memory: reading it costs no dispatcher call
        self.event = torch.cuda.Event()
        self.busy = False

    def reserve(self, n_rays: int, run_capacity: int = 0) -> None:
        """Room for `n_rays` rays and max(run_capacity, what was seen so far, 2 n_rays + 1024) runs.  The layout inside
        the buffer is recomputed per call by the library; a fresh buffer is zeroed because the kernel expects (and
        leaves behind) a zero header."""
        lib = _lib.load()
        self.run_capacity = max(self.run_capacity, int(run_capacity), 2 * n_rays + 1024)
        need = lib.nfa_march_workspace_bytes(n_rays, self.run_capacity)
        if self.workspace is None or self.workspace.numel() < need:
            self.workspace = torch.zeros(need + (need >> 2), dtype=torch.uint8, device=self.device)


_scratch_cache: Dict[tuple, list] = {}


def _scratch_acquire(device, n_rays: int) -> _MarchScratch:
    """A workspace nobody is marching into, for the CURRENT stream of `device`: two streams sampling at the same
    time must not share a run pool or a pinned totals slot (stream order is what protects them).  One scratch per
    (device, stream) in the usual one-call-at-a-time use; a second one is made when a march is still in flight
    (sampling_begin without its sampling_end yet)."""
    key = (device, _lib.stream_ptr(device))
    pool = _scratch_cache.get(key)
    if pool is None:
        if len(_scratch_cache) >= 16:
            _scratch_cache.clear()
        pool = _scratch_cache[key] = []
    for sc in pool:
        if not sc.busy:
            break
    else:
        sc = _MarchScratch(device)
        pool.append(sc)
    sc.busy = True
    sc.reserve(n_rays)
    return sc


class _MarchResult:
    __slots__ = ("n_samples", "n_runs", "ray_indices", "t_starts", "t_ends", "packed_info",
                 "intervals", "samples", "terminate_planes")


class _MarchJob:
    """Constant-step traversal: march -> expand, with ONE host synchronisation, in two halves.

    `begin()` queues the march and, given a `capacity_hint` (size of the previous batch plus head-room), the
    expand kernels behind it; `finish()` waits for the totals, re-runs the cheap tail only if the batch outgrew
    the hint (or the run pool) and returns the result.  `near_planes` / `far_planes` may both be None: every ray
    then uses the scalars.  The job keeps its inputs alive and owns its workspace until `finish()`.
    """

    def __init__(self, rays_o: Tensor, rays_d: Tensor, binaries: Tensor, aabbs: Tensor, near_planes: Optional[Tensor],
                 far_planes: Optional[Tensor], step_size: float, t_sorted: Optional[Tensor],
                 t_indices: Optional[Tensor], hits: Optional[Tensor], want_intervals: bool, want_terminate: bool,
                 capacity_hint: int = 0, near_plane: float = 0.0, far_plane: float = float("inf")):
        self.device = device = rays_o.device
        self.n_rays = n_rays = rays_o.shape[0]
        self.shape = tuple(int(s) for s in binaries.shape)
        n_grids = self.shape[0]
        self.occ = _packed_grid(binaries)
        if n_grids > 1 and t_sorted is None:
            t_sorted = torch.empty((n_rays, 2 * n_grids), dtype=torch.float32, device=device)
            t_indices = torch.empty((n_rays, 2 * n_grids), dtype=torch.int64, device=device)
            hits = torch.empty((n_rays, n_grids), dtype=torch.bool, device=device)
            if n_rays > 0:
                _lib.call("nfa_intersect_sorted", device, n_rays, _lib.ptr(rays_o), _lib.ptr(rays_d), n_grids,
                          _lib.ptr(aabbs), _lib.ptr(t_sorted), _lib.ptr(t_indices), _lib.ptr(hits))
        self.inputs = (rays_o, rays_d, aabbs, near_planes, far_planes, t_sorted, t_indices, hits)
        self.planes = (float(near_plane), float(far_plane))
        self.step_size = float(step_size)
        self.want_intervals, self.capacity_hint = want_intervals, int(capacity_hint)
        self.term = torch.empty(n_rays, dtype=torch.float32, device=device) if want_terminate else None
        self.packed_info = torch.empty((n_rays, 2), dtype=torch.int64, device=device)
        self.sc = _scratch_acquire(device, n_rays)
        self.bufs, self.cap = None, 0

    def __del__(self):
        sc = getattr(self, "sc", None)
        if sc is not None:
            sc.busy = False  # a ticket that was dropped without sampling_end()

    def _launch_march(self) -> None:
        rays_o, rays_d, aabbs, near_planes, far_planes, t_sorted, t_indices, hits = self.inputs
        n_grids, rx, ry, rz = self.shape
        sc, occ = self.sc, self.occ
        _lib.call("nfa_march", self.device, self.n_rays, _lib.ptr(rays_o), _lib.ptr(rays_d), _lib.ptr(near_planes),
                  _lib.ptr(far_planes), self.planes[0], self.planes[1], n_grids, rx, ry, rz, _lib.ptr(occ.words),
                  _lib.ptr(occ.bounds), _lib.ptr(aabbs), _lib.ptr(t_sorted), _lib.ptr(t_indices),
                  _lib.ptr(hits), self.step_size, sc.run_capacity, _lib.ptr(sc.workspace), _lib.ptr(sc.totals_dev),
                  _lib.ptr(sc.totals_host), _lib.ptr(self.term))
        # on the stream (of THIS device) the march was launched on: the default `record()` would use the current
        # device's stream and the totals could be read before they are written
        sc.event.record(torch.cuda.current_stream(self.device))

    def _read_totals(self):
        # wait for the totals only: kernels queued behind the march (the speculative expand) keep running while
        # the host prepares the next launches
        if _lib.idle_tasks:
            _lib.run_idle_tasks()  # deferred host work fills the wait for the march
        self.sc.event.synchronize()
        tot = self.sc.totals_np
        n, runs, stuck = int(tot[0]), int(tot[1]), int(tot[3])
        if stuck:
            raise RuntimeError(
                f"traverse_grids: step_size={self.step_size} is below the float32 resolution of the marching "
                f"distance on {stuck} ray(s); the march cannot advance (the reference would not terminate).")
        return n, runs

    def _expand_samples(self, cap: int):
        device, sc = self.device, self.sc
        ri = torch.empty(cap, dtype=torch.int64, device=device)
        ts = torch.empty(cap, dtype=torch.float32, device=device)
        te = torch.empty(cap, dtype=torch.float32, device=device)
        _lib.call("nfa_expand_samples", device, self.n_rays, sc.run_capacity, _lib.ptr(sc.workspace),
                  _lib.ptr(sc.totals_dev), self.step_size, cap, _lib.ptr(self.packed_info), _lib.ptr(ri), _lib.ptr(ts),
                  _lib.ptr(te))
        return ri, ts, te

    def begin(self) -> "_MarchJob":
        self._launch_march()
        if not self.want_intervals and self.capacity_hint > 0:
            self.cap = self.capacity_hint
            self.bufs = self._expand_samples(self.cap)  # speculative: queued before the sync
        return self

    def finish(self) -> _MarchResult:
        device, n_rays, sc, packed_info = self.device, self.n_rays, self.sc, self.packed_info
        res = _MarchResult()
        res.terminate_planes = self.term
        res.intervals = res.samples = None
        try:
            n, runs = self._read_totals()
            if runs > sc.run_capacity:  # run pool overflow: rare (very fragmented grids); re-march with room
                sc.reserve(n_rays, runs + (runs >> 2) + 1024)
                self._launch_march()
                n, runs = self._read_totals()
                self.bufs = None
            if not self.want_intervals:
                if self.bufs is None or n > self.cap:
                    self.bufs = self._expand_samples(n)
                ri, ts, te = self.bufs
                if ri.shape[0] != n:  # the speculative buffers are longer: shrink the views in place (no new tensors)
                    ri.resize_(n)
                    ts.resize_(n)
                    te.resize_(n)
                res.ray_indices, res.t_starts, res.t_ends = ri, ts, te
            else:
                e = n + runs
                iv_pi = torch.empty((n_rays, 2), dtype=torch.int64, device=device)
                iv_vals = torch.empty(e, dtype=torch.float32, device=device)
                iv_ray = torch.empty(e, dtype=torch.int64, device=device)
                iv_left = torch.empty(e, dtype=torch.bool, device=device)
                iv_right = torch.empty(e, dtype=torch.bool, device=device)
                sm_vals = torch.empty(n, dtype=torch.float32, device=device)
                sm_ray = torch.empty(n, dtype=torch.int64, device=device)
                sm_valid = torch.empty(n, dtype=torch.bool, device=device)
                _lib.call("nfa_expand_intervals", device, n_rays, sc.run_capacity, _lib.ptr(sc.workspace),
                          _lib.ptr(sc.totals_dev), self.step_size, e, n, _lib.ptr(iv_pi), _lib.ptr(iv_vals),
                          _lib.ptr(iv_ray), _lib.ptr(iv_left), _lib.ptr(iv_right), _lib.ptr(packed_info),
                          _lib.ptr(sm_vals), _lib.ptr(sm_ray), _lib.ptr(sm_valid))
                res.intervals = RayIntervals(vals=iv_vals, packed_info=iv_pi, ray_indices=iv_ray, is_left=iv_left,
                                             is_right=iv_right)
                res.samples = RaySamples(vals=sm_vals, packed_info=packed_info, ray_indices=sm_ray, is_valid=sm_valid)
                res.ray_indices = sm_ray
        finally:
            # stream order protects the workspace: whatever marches into it next is queued behind this expand
            sc.busy = False
            self.sc = None
        res.n_samples, res.n_runs, res.packed_info = n, runs, packed_info
        _stash_packed_info(res.ray_indices, packed_info, n_rays)
        return res


def _march(*args, **kwargs) -> _MarchResult:
    """One synchronous pass: see :class:`_MarchJob`."""
    return _MarchJob(*args, **kwargs).begin().finish()


@torch.no_grad()
def traverse_grids(
    rays_o: Tensor,  # [n_rays, 3]
    rays_d: Tensor,  # [n_rays, 3]
    binaries: Tensor,  # [m, resx, resy, resz]
    aabbs: Tensor,  # [m, 6]
    near_planes: Optional[Tensor] = None,  # [n_rays]
    far_planes: Optional[Tensor] = None,  # [n_rays]
    step_size: Optional[float] = 1e-3,
    cone_angle: Optional[float] = 0.0,
    traverse_steps_limit: Optional[int] = None,
    over_allocate: Optional[bool] = False,
    rays_mask: Optional[Tensor] = None,  # [n_rays]
    t_sorted: Optional[Tensor] = None,  # [n_rays, m * 2]
    t_indices: Optional[Tensor] = None,  # [n_rays, m * 2]
    hits: Optional[Tensor] = None,  # [n_rays, m]
) -> Tuple[RayIntervals, RaySamples, Tensor]:
    """March rays through one or more nested binary grids.

    Same arguments, defaults and return triple (RayIntervals, RaySamples,
    termination planes) as the reference (grid.py:93-192).  Not differentiable.
    """
    _lib.require_cuda(rays_o, "traverse_grids")
    device = rays_o.device
    rays_o, rays_d = rays_o.contiguous().float(), rays_d.contiguous().float()
    aabbs = aabbs.contiguous().float()
    if near_planes is None:
        near_planes = torch.zeros_like(rays_o[:, 0])
    if far_planes is None:
        far_planes = torch.full_like(rays_o[:, 0], float("inf"))
    near_planes, far_planes = near_planes.contiguous().float(), far_planes.contiguous().float()
    if traverse_steps_limit is None:
        traverse_steps_limit = -1
    if over_allocate:
        assert traverse_steps_limit > 0, "traverse_steps_limit must be set if over_allocate is True."
    have_sorted = t_sorted is not None and t_indices is not None and hits is not None
    if have_sorted:
        t_sorted, t_indices, hits = t_sorted.contiguous().float(), t_indices.contiguous(), hits.contiguous()
    else:
        t_sorted = t_indices = hits = None

    fast = (cone_angle == 0.0 and step_size is not None and step_size > 0.0 and traverse_steps_limit <= 0
            and not over_allocate)
    if fast:
        # rays_mask is ignored in exact-allocation mode by the reference too (grid.cu:418,450)
        res = _march(rays_o, rays_d, binaries, aabbs, near_planes, far_planes, float(step_size), t_sorted, t_indices,
                     hits, want_intervals=True, want_terminate=True)
        return res.intervals, res.samples, res.terminate_planes
    return _traverse_generic(rays_o, rays_d, binaries, aabbs, near_planes, far_planes, float(step_size),
                             float(cone_angle), int(traverse_steps_limit), bool(over_allocate), rays_mask, t_sorted,
                             t_indices, hits)


def _traverse_generic(rays_o, rays_d, binaries, aabbs, near_planes, far_planes, step_size, cone_angle, limit,
                      over_allocate, rays_mask, t_sorted, t_indices, hits):
    """cone_angle > 0, step_size <= 0, step limits, over-allocation, masks: count pass -> scan -> fill pass
    (one pass into fixed-stride slots when over-allocating), reference grid.cu:364-470."""
    device = rays_o.device
    n_rays = rays_o.shape[0]
    n_grids, rx, ry, rz = (int(s) for s in binaries.shape)
    occ = _packed_grid(binaries)
    if t_sorted is None:
        t_sorted = torch.empty((n_rays, 2 * n_grids), dtype=torch.float32, device=device)
        t_indices = torch.empty((n_rays, 2 * n_grids), dtype=torch.int64, device=device)
        hits = torch.empty((n_rays, n_grids), dtype=torch.bool, device=device)
        if n_rays > 0:
            _lib.call("nfa_intersect_sorted", device, n_rays, _lib.ptr(rays_o), _lib.ptr(rays_d), n_grids,
                      _lib.ptr(aabbs), _lib.ptr(t_sorted), _lib.ptr(t_indices), _lib.ptr(hits))
    if t_indices.dtype != torch.int64:
        t_indices = t_indices.to(torch.int64)
    if hits.dtype != torch.bool:
        hits = hits != 0
    mask = None
    if rays_mask is not None:
        mask = rays_mask.contiguous()
        if mask.dtype != torch.bool:
            mask = mask != 0
    term = torch.empty(n_rays, dtype=torch.float32, device=device)

    def run(fill, use_mask, iv_s, iv_c, sm_s, sm_c, arrays, slots=None):
        if n_rays == 0:
            return
        _lib.call("nfa_traverse_generic", device, n_rays, _lib.ptr(rays_o), _lib.ptr(rays_d),
                  _lib.ptr(mask) if use_mask else None, _lib.ptr(near_planes), _lib.ptr(far_planes), n_grids, rx, ry, rz,
                  _lib.ptr(occ.words), _lib.ptr(occ.coarse), _lib.ptr(aabbs), _lib.ptr(t_sorted), _lib.ptr(t_indices),
                  _lib.ptr(hits), step_size, cone_angle, limit, int(fill), _lib.ptr(slots), _lib.ptr(iv_s), _lib.ptr(iv_c),
                  *[_lib.ptr(a) for a in arrays[:4]], _lib.ptr(sm_s), _lib.ptr(sm_c),
                  *[_lib.ptr(a) for a in arrays[4:]], _lib.ptr(term) if fill else None)

    if over_allocate:
        return _traverse_bounded(run, device, n_rays, limit, mask, term)
    iv_cnts = torch.zeros(n_rays, dtype=torch.int64, device=device)
    sm_cnts = torch.zeros(n_rays, dtype=torch.int64, device=device)
    run(False, False, None, iv_cnts, None, sm_cnts, [None] * 7)
    iv_starts = torch.cumsum(iv_cnts, 0) - iv_cnts
    sm_starts = torch.cumsum(sm_cnts, 0) - sm_cnts
    n_edges = int(iv_cnts.sum().item()) if n_rays else 0
    n_samples = int(sm_cnts.sum().item()) if n_rays else 0
    iv_vals = torch.zeros(n_edges, dtype=torch.float32, device=device)
    iv_ray = torch.zeros(n_edges, dtype=torch.int64, device=device)
    iv_left = torch.zeros(n_edges, dtype=torch.bool, device=device)
    iv_right = torch.zeros(n_edges, dtype=torch.bool, device=device)
    sm_vals = torch.zeros(n_samples, dtype=torch.float32, device=device)
    sm_ray = torch.zeros(n_samples, dtype=torch.int64, device=device)
    sm_valid = torch.zeros(n_samples, dtype=torch.bool, device=device)
    run(True, False, iv_starts, iv_cnts, sm_starts, sm_cnts,
        [iv_vals, iv_ray, iv_left, iv_right, sm_vals, sm_ray, sm_valid])
    intervals = RayIntervals(vals=iv_vals, packed_info=torch.stack([iv_starts, iv_cnts], -1), ray_indices=iv_ray,
                             is_left=iv_left, is_right=iv_right)
    samples = RaySamples(vals=sm_vals, packed_info=torch.stack([sm_starts, sm_cnts], -1), ray_indices=sm_ray,
                         is_valid=sm_valid)
    return intervals, samples, term


def _traverse_bounded(run, device, n_rays: int, limit: int, mask: Optional[Tensor], term: Tensor):
    """`traverse_steps_limit` + `over_allocate` (+ `rays_mask`): one pass into fixed-stride slots (reference
    grid.cu:364-404) -- the call the test-mode rendering loop makes once per round (examples/utils.py:340-375), so
    its cost is host work: one zero-filled arena carved into the seven output arrays (one memset instead of seven),
    one synchronisation (the number of unmasked rays; none without a mask), the slot offsets computed in the
    kernel from the rays' rank among the unmasked ones, packed_info of the actual counts by a native scan."""
    lib = _lib.load()
    if mask is None:
        n_alive = n_rays
        slots = torch.arange(n_rays, dtype=torch.int64, device=device)
    else:
        csum = torch.cumsum(mask, 0, dtype=torch.int64)
        n_alive = int(csum[-1].item()) if n_rays else 0
        slots = csum - mask.to(torch.int64)
    n_edges, n_samples = 2 * limit * n_alive, limit * n_alive
    # arena: int64 arrays first (8-byte aligned), then float32, then the three flag arrays
    sizes = (8 * n_edges, 8 * n_samples, 4 * n_edges, 4 * n_samples, n_edges, n_edges, n_samples)
    arena = torch.zeros(sum(sizes), dtype=torch.uint8, device=device)
    parts, at = [], 0
    for nbytes in sizes:
        parts.append(arena[at:at + nbytes])
        at += nbytes
    iv_ray, sm_ray = parts[0].view(torch.int64), parts[1].view(torch.int64)
    iv_vals, sm_vals = parts[2].view(torch.float32), parts[3].view(torch.float32)
    iv_left, iv_right, sm_valid = parts[4].view(torch.bool), parts[5].view(torch.bool), parts[6].view(torch.bool)
    cnts = torch.empty((2, n_rays), dtype=torch.int64, device=device)
    run(True, mask is not None, None, cnts[0], None, cnts[1],
        [iv_vals, iv_ray, iv_left, iv_right, sm_vals, sm_ray, sm_valid], slots=slots)
    # reference grid.cu:402-404: starts recomputed from the actual counts
    packed = torch.empty((2, n_rays, 2), dtype=torch.int64, device=device)
    if n_rays:
        ws = torch.empty(lib.nfa_pack_info_workspace_bytes(n_rays), dtype=torch.uint8, device=device)
        for k in (0, 1):
            _lib.call("nfa_counts_to_packed_info", device, n_rays, _lib.ptr(cnts[k]), _lib.ptr(packed[k]), _lib.ptr(ws))
    intervals = RayIntervals(vals=iv_vals, packed_info=packed[0], ray_indices=iv_ray, is_left=iv_left, is_right=iv_right)
    samples = RaySamples(vals=sm_vals, packed_info=packed[1], ray_indices=sm_ray, is_valid=sm_valid)
    return intervals, samples, term


def _enlarge_aabb(aabb, factor: float) -> Tensor:
    """Scale a box about its centre (reference grid.py:195-198)."""
    lo, hi = aabb[:3], aabb[3:]
    mid, half = (lo + hi) * 0.5, (hi - lo) * 0.5
    return torch.cat([mid - half * factor, mid + half * factor])


def _query(x: Tensor, data: Tensor, base_aabb: Tensor) -> Tensor:
    """Look up `data` (m, rx, ry, rz) at points `x`, picking the mip level of nested 2x boxes.

    Test helper with the reference's semantics (grid.py:201-237): returns (values * selector, selector).
    """
    lo, hi = base_aabb[:3], base_aabb[3:]
    u = (x - lo) / (hi - lo) - 0.5  # base box -> [-0.5, 0.5]^3
    reach = u.abs().amax(dim=-1).clamp(min=0.1)  # keep frexp away from 0
    level = (torch.frexp(reach)[1].long() + 1).clamp(min=0)
    inside = level < data.shape[0]
    u = u / (2.0 ** level)[:, None] + 0.5
    res = torch.tensor(data.shape[1:], device=x.device)
    cell = torch.minimum((u * res).long(), res - 1)
    level = level.clamp(max=data.shape[0] - 1)
    return data[level, cell[:, 0], cell[:, 1], cell[:, 2]] * inside, inside
