"""Drop-in for the reference's un-vendored dependency `diff_gaussian_rasterization`
(requirements.txt:17; imported at src/model/decoder/cuda_splatting.py:5-8).  With this
directory on sys.path the reference's own `render_cuda` runs unmodified on these CUDA kernels."""
from pixelsplat_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer"]
