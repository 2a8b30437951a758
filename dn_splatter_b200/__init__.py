"""dn_splatter_b200 — H100-native (sm_90a) depth+normal Gaussian rasterizer behind the dn-splatter
plugin surface.  The arithmetic lives in libdnr_b200.so (C ABI: include/dnr.h); see DESIGN.md."""
from .rasterize import RasterOutput, RasterSettings, dn_rasterize, get_viewmat  # noqa: F401
from .mesh import (TSDFVolume, TriangleMesh, export_marching_cubes_mesh, export_tsdf_mesh, filter_small_clusters,  # noqa: F401
                   marching_cubes, write_ply)
from .poisson import (export_dn_poisson_mesh, export_gaussians_poisson_mesh, export_level_set_poisson_mesh,  # noqa: F401
                      filter_smooth_laplacian, poisson_reconstruct, remove_statistical_outlier, trim_low_density,
                      voxel_down_sample, write_point_cloud_ply)

__version__ = "0.1.0"
