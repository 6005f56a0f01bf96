"""LightningModule as far as EvaluationIndexGenerator uses it: an nn.Module whose `device` is the CPU."""
import torch


class LightningModule(torch.nn.Module):
    @property
    def device(self) -> torch.device:
        return torch.device("cpu")
