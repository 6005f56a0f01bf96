"""Training on RE10k / ACID: the reference's training step and optimiser without Lightning.

- `Trainer(encoder, decoder, losses).fit(loader, max_steps, output)`: ModelWrapper.training_step over a DataLoader of
  `DatasetRE10k`, with `optim.ClipAdam` (csrc/optimizer.cu) as the optimiser end; checkpoints in Lightning's layout,
  which `evaluation.load_checkpoint` reads, and `Trainer.resume`.
- `Trainer.validation_step` and `fit(..., validation=loader, val_every=250)`: ModelWrapper.validation_step on a
  scene of the test split (`presets.make_val_dataset`), with its own seeded generators.
- `presets`: the reference's re10k / acid / re10k_depth_loss training configurations.
- `python -m pixelsplat_b200.training --help`: the command line.
"""
from .presets import (PRESETS, TRAIN_PRESETS, TrainPreset, dataset_cfg, make_losses, make_train_dataset,
                      make_val_dataset, train_preset)
from .trainer import Trainer

__all__ = ["PRESETS", "TRAIN_PRESETS", "TrainPreset", "dataset_cfg", "make_losses", "make_train_dataset",
           "make_val_dataset", "train_preset", "Trainer"]
