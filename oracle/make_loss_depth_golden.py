"""Generates tests/golden/loss_depth.npz by running the REFERENCE's LossDepth (src/loss/loss_depth.py) on the CPU in
float64 and float32.  Authoring container only:

    python oracle/make_loss_depth_golden.py

TEST INFRASTRUCTURE.  Inputs are regenerated from tests/test_depth_cpu.loss_depth_case on both sides; only the
reference's loss values and depth gradients are stored, for sigma_image None / 12 and use_second_derivative
off / on.
"""
from __future__ import annotations

import sys
import types
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import epipolar_ref  # noqa: E402
from tests.test_depth_cpu import loss_depth_case  # noqa: E402

OUT = ROOT / "tests" / "golden" / "loss_depth.npz"


def load_loss_depth():
    epipolar_ref.load(2)          # sys.path, stubs, bare packages
    for name in ("src.loss", "src.model.decoder"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__path__ = [str(epipolar_ref.REFERENCE / name.replace(".", "/"))]
            sys.modules[name] = m
    # loss_depth.py imports DecoderOutput for its annotations only; the reference's decoder module pulls in the
    # dataset configuration, so a stand-in module provides the name
    if "src.model.decoder.decoder" not in sys.modules:
        dec = types.ModuleType("src.model.decoder.decoder")
        dec.DecoderOutput = object
        sys.modules["src.model.decoder.decoder"] = dec
    from src.loss import loss_depth
    return loss_depth


def main() -> None:
    ld = load_loss_depth()
    out = {}
    for dtype, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
        c = loss_depth_case(dtype)
        for sigma in (None, 12.0):
            for second in (False, True):
                depth = c["depth"].clone().requires_grad_(True)
                loss = ld.LossDepth(ld.LossDepthCfgWrapper(ld.LossDepthCfg(0.25, sigma, second)))
                pred = types.SimpleNamespace(depth=depth)
                batch = {"target": {"near": c["near"], "far": c["far"], "image": c["image"]}}
                value = loss.forward(pred, batch, None, 0)
                value.backward()
                key = f"{tag}_{'none' if sigma is None else int(sigma)}_{int(second)}"
                out[key + "_loss"] = value.detach().numpy()
                out[key + "_grad"] = depth.grad.numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, sorted(out))


if __name__ == "__main__":
    main()
