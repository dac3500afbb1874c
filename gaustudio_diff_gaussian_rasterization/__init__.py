"""Drop-in module under the reference's real import name (gaustudio/renderers/base.py:7,
$RAST/setup.py:18-22): `from gaustudio_diff_gaussian_rasterization import GaussianRasterizationSettings,
GaussianRasterizer` resolves to the H100-native implementation."""
from gaustudio_b200 import _C  # noqa: F401  (same attribute name as the reference's pybind module)
from gaustudio_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, _RasterizeGaussians,  # noqa: F401
                                       cpu_deep_copy_tuple, rasterize_gaussians)
