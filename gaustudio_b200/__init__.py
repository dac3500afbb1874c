"""gaustudio_b200: H100-native (sm_90a) differentiable 3D Gaussian Splatting tile rasterizer behind the
gaustudio renderer-plugin surface.  Product path = hand-written CUDA in libgsr_b200.so (C ABI: include/gsr.h);
Python here only mirrors the reference's operator interface.  No CPU fallback."""
__version__ = "0.1.0"
