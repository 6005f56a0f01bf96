from .cuda_splatting import (DepthRenderingMode, get_projection_matrix, render_cuda,
                             render_cuda_orthographic, render_depth_cuda, render_views, render_views_mse,
                             render_views_mse_with_depth, render_views_with_depth)
from .decoder_splatting_cuda import (DECODERS, DecoderOutput, DecoderSplattingCUDA,
                                     DecoderSplattingCUDACfg, Gaussians, get_decoder)
