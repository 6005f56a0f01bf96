"""The dataset fixtures of oracle/make_dataset_golden.py: the tiny RE10k-format dataset (tests/golden/re10k_tiny)
and what the reference's DatasetRE10k yields on it (tests/golden/dataset_re10k_v1.npz), with this package's
DatasetRE10k built on the same configuration."""
from __future__ import annotations

import hashlib
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"
DATA = GOLDEN / "re10k_tiny"
SHAPES = {"test": (180, 320), "train": (256, 256)}


def fixture() -> dict:
    return dict(np.load(GOLDEN / "dataset_re10k_v1.npz"))


def expected(stage: str) -> list[dict]:
    """The reference's examples of `stage`: scene, flip and per view set the recorded arrays.  A view's image u
    (uint8 [3, h, w], the reference's float image times 255) is stored as `image_sha256` (one digest per view) and
    `image_sub` (every 8th row and column, to locate a mismatch)."""
    g = fixture()
    out = []
    for i in range(int(g[f"{stage}/count"])):
        ex = {"scene": str(g[f"{stage}/scene"][i]), "flip": bool(g[f"{stage}/flip"][i])}
        for v in ("context", "target"):
            ex[v] = {k: g[f"{stage}/{i}/{v}/{k}"] for k in ("extrinsics", "intrinsics", "near", "far", "index",
                                                         "image_sha256", "image_sub")}
        out.append(ex)
    return out


def image_digest(u: np.ndarray) -> str:
    """SHA-256 of one view's uint8 [3, h, w] image in C order, as the fixture stores it."""
    return hashlib.sha256(np.ascontiguousarray(u, dtype=np.uint8).tobytes()).hexdigest()


def assert_images_equal(u: np.ndarray, want: dict, what) -> None:
    """uint8 [v, 3, h, w] against a view set's recorded images, bit for bit."""
    assert u.dtype == np.uint8 and u.shape[0] == len(want["image_sha256"]), what
    assert np.array_equal(u[:, :, ::8, ::8], want["image_sub"]), what
    assert [image_digest(x) for x in u] == list(want["image_sha256"]), what


def dataset(stage: str):
    """This package's DatasetRE10k on re10k_tiny with the configuration the fixture was made with."""
    from pixelsplat_b200.data import (DatasetRE10k, DatasetRE10kCfg, ViewSamplerBoundedCfg,
                                      ViewSamplerEvaluationCfg, get_view_sampler)
    if stage == "test":
        vs = ViewSamplerEvaluationCfg("evaluation", DATA / "evaluation_index.json", 2)
    else:
        vs = ViewSamplerBoundedCfg("bounded", 2, 1, 2, 6, 0, 0, 2, 6)
    cfg = DatasetRE10kCfg(image_shape=list(SHAPES[stage]), background_color=[0.0, 0.0, 0.0],
                          cameras_are_circular=False, overfit_to_scene=None, view_sampler=vs, name="re10k",
                          roots=[DATA], baseline_epsilon=1e-3, max_fov=100.0, make_baseline_1=True, augment=True)
    return DatasetRE10k(cfg, stage, get_view_sampler(vs, stage, False, False, None))


def examples(stage: str) -> list[dict]:
    """This package's examples of `stage`, seeded as the fixture's run of the reference was."""
    torch.manual_seed(int(fixture()["train_seed"]) if stage == "train" else 0)
    return list(dataset(stage))
