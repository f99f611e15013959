"""gsplat 0.1.11-compatible surface used by the reference (ca_code/utils/render_gsplat.py:10-11):
`project_gaussians` and `rasterize_gaussians`, backed by hand-written sm_90a kernels.

gsplat is a third-party dependency that is not part of the reference tree; signatures and semantics are
those of its 0.1.11 release as restated in SURVEY.md Appendix A.
"""
from .project import project_gaussians  # noqa: F401
from .rasterize import rasterize_gaussians  # noqa: F401
from .utils import (  # noqa: F401
    bin_and_sort_gaussians,
    compute_cumulative_intersects,
    get_tile_bin_edges,
    map_gaussian_to_intersects,
)

__version__ = "0.1.11+goliath_b200"
