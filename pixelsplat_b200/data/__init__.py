"""Data loading: the reference's RE10k / ACID dataset and view samplers, with its crop shim on the GPU
(csrc/image_resample.cu).  A loop reads `DatasetRE10k` through a DataLoader and calls `device_shim` on each
batch; the result is the batch the reference's loader gives."""
from .crop_shim import (apply_crop_shim, center_crop, device_shim, resample_table, rescale, rescale_and_crop,
                        rescale_and_crop_u8)
from .dataset_re10k import DatasetCfgCommon, DatasetRE10k, DatasetRE10kCfg
from .view_sampler import (StepTracker, ViewSamplerBounded, ViewSamplerBoundedCfg, ViewSamplerEvaluation,
                           ViewSamplerEvaluationCfg, get_view_sampler)

__all__ = ["apply_crop_shim", "center_crop", "device_shim", "resample_table", "rescale", "rescale_and_crop",
           "rescale_and_crop_u8", "DatasetCfgCommon", "DatasetRE10k", "DatasetRE10kCfg", "StepTracker",
           "ViewSamplerBounded", "ViewSamplerBoundedCfg", "ViewSamplerEvaluation", "ViewSamplerEvaluationCfg",
           "get_view_sampler"]
