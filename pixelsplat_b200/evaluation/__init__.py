"""Evaluation on the RE10k / ACID test split: the reference's test step and metric computer on the GPU.

The reference scores 8-bit frames: its test step writes each render as a PNG (prep_image truncates
clip(x, 0, 1) * 255 to uint8) and its metric computer reads the PNGs back.  Here the quantisation, the dequantised
planes and the squared error are one pass of csrc/eval_images.cu, so every metric equals the PNG round trip's and
no float image goes to the host.

- `Evaluator(encoder, decoder, output_path).run(loader)`: ModelWrapper.test_step over a split, with PSNR / SSIM /
  LPIPS per scene and their mean over scenes; `load_checkpoint` reads a pixelSplat `.ckpt` into the encoder.
- `compute_metrics(methods, loader)`: MetricComputer over saved frame directories.
- `frame_metrics`, `frame_pass` and the image_io drop-ins `prep_image`, `save_image`, `load_image`.
- `python -m pixelsplat_b200.evaluation --help`: both as a command line.
"""
from .checkpoint import load_checkpoint
from .evaluator import Benchmarker, EvaluationResult, Evaluator, SceneResult, mean_over_scenes
from .frames import FramePass, frame_pass, psnr_from_sse
from .image_io import load_frames, load_image, prep_image, quantise, read_frame, save_frame, save_image
from .metric_computer import Method, MetricsResult, compute_metrics, preview_table, scene_frame_paths
from .metrics import frame_metrics, frame_metrics_chunked

__all__ = ["load_checkpoint", "Benchmarker", "EvaluationResult", "Evaluator", "SceneResult", "mean_over_scenes",
           "FramePass", "frame_pass", "psnr_from_sse", "load_frames", "load_image", "prep_image", "quantise",
           "read_frame", "save_frame", "save_image", "Method", "MetricsResult", "compute_metrics", "preview_table",
           "scene_frame_paths", "frame_metrics", "frame_metrics_chunked"]
