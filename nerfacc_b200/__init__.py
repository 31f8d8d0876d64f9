"""nerfacc_b200 -- hand-written CUDA sampling + volume-rendering hot path with nerfacc's API.

The public names are the subset of /root/reference/nerfacc/__init__.py that lies on the hot path
(SURVEY.md section 8) plus ``defer_until_wait``; ``import nerfacc`` resolves to this package through
the alias package at the repository root.
"""
from . import data_specs, grid, losses, pack, parallel, pdf, scan, volrend
from ._lib import defer_until_wait
from .estimators import occ_grid as _occ_grid
from .estimators import prop_net as _prop_net
from .version import __version__

_EXPORTS = {
    scan: ("inclusive_prod", "exclusive_prod", "inclusive_sum", "exclusive_sum"),
    pack: ("pack_info", "unpack_info", "pack_data", "unpack_data"),
    volrend: ("render_visibility_from_alpha", "render_visibility_from_density", "render_weight_from_alpha",
              "render_weight_from_density", "render_transmittance_from_alpha", "render_transmittance_from_density",
              "accumulate_along_rays", "accumulate_along_rays_", "rendering"),
    data_specs: ("RayIntervals", "RaySamples"),
    grid: ("ray_aabb_intersect", "traverse_grids"),
    _occ_grid: ("OccGridEstimator",),
    _prop_net: ("PropNetEstimator",),
    pdf: ("importance_sampling", "searchsorted"),
    losses: ("distortion",),
}

__all__ = ["__version__", "defer_until_wait"]
for _module, _names in _EXPORTS.items():
    for _name in _names:
        globals()[_name] = getattr(_module, _name)
        __all__.append(_name)
del _module, _names, _name
