"""pixelsplat_b200 -- native H100 (sm_90a) render hot path of pixelSplat.

Sub-modules that touch the GPU (`rasterizer`, `decoder`, `encoder`) load the CUDA library through
`_lib` and raise if it is not built; there is no CPU fallback.  `synthetic` is pure host code.
"""
__version__ = "0.1.0"
