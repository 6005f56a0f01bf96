"""Loading a pixelSplat Lightning checkpoint (`re10k.ckpt`, `acid.ckpt`) into this package's `EncoderEpipolar`."""
from __future__ import annotations

from pathlib import Path
from typing import Union

import torch
from torch import nn

PREFIX = "encoder."


def load_checkpoint(path: Union[Path, str], encoder: nn.Module) -> int:
    """Loads the `encoder.*` entries of the checkpoint's `state_dict` into `encoder` with strict=True and returns
    the checkpoint's `global_step` (0 when absent), for information.

    The file is read with `torch.load(weights_only=True)`: no pickled code runs.  Every state-dict key must start
    with `encoder.`: the reference's decoder and LPIPS loss hold only non-persistent tensors, so a pixelSplat
    checkpoint has no other key, and one that does is not a checkpoint of this model (ValueError).  A missing or
    unexpected encoder key raises as `load_state_dict(strict=True)` does."""
    ckpt = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(ckpt, dict) or "state_dict" not in ckpt:
        raise ValueError(f"load_checkpoint: {path} is not a Lightning checkpoint (no 'state_dict')")
    state = ckpt["state_dict"]
    other = sorted(k for k in state if not k.startswith(PREFIX))
    if other:
        raise ValueError(f"load_checkpoint: {path} holds {len(other)} keys outside '{PREFIX}*' (e.g. {other[:3]}); "
                         "a pixelSplat checkpoint holds encoder weights only")
    encoder.load_state_dict({k[len(PREFIX):]: v for k, v in state.items()}, strict=True)
    return int(ckpt.get("global_step", 0))
