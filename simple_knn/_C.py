"""Drop-in module under the import name of simple_knn's extension (`from simple_knn._C import distCUDA2`, what
graphdeco's, 2DGS's and Mip-Splatting's train.py and gaustudio's VanillaPointCloud use): resolves to the exact
neighbour search of gaustudio_b200 (initializers.dist2)."""
from gaustudio_b200.initializers import dist2 as distCUDA2  # noqa: F401
