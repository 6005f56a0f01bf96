"""The reference's DatasetRE10k (src/dataset/dataset_re10k.py) over its `.torch` chunks, without the host resize.

It reads the same chunks, skips the same examples and draws from torch's RNG in the same order (chunk and example
shuffles, the view sampler, the augmentation coin), so a seeded single-process loader yields the reference's
examples.  What it yields differs in one way: each view's image is the decoded uint8 [360, 640, 3] (PIL, as in the
reference), uncropped, and a "flip" flag records the augmentation coin; the extrinsics are already reflected.
`pixelsplat_b200.data.device_shim` then flips, resizes and crops the batch on the GPU, which gives the images
and intrinsics the reference's loader gives, bit for bit.

With `cameras_only=True` (the evaluation-index generator, which reads scenes through the reference's `all` view
sampler) it decodes no frame: each example is every frame's cameras, the scene key and the frame count, after the
same skips, with the image shape read from each JPEG header.
"""
from __future__ import annotations

import json
import logging
from dataclasses import dataclass
from functools import cached_property
from io import BytesIO
from pathlib import Path
from typing import Literal

import numpy as np
import torch
from PIL import Image
from torch import Tensor
from torch.utils.data import IterableDataset

from .view_sampler import Stage, ViewSampler, ViewSamplerCfg

log = logging.getLogger(__name__)

IMAGE_SHAPE = (360, 640, 3)   # the shape the reference keeps; other decoded shapes skip the example


@dataclass
class DatasetCfgCommon:
    image_shape: list[int]
    background_color: list[float]
    cameras_are_circular: bool
    overfit_to_scene: str | None
    view_sampler: ViewSamplerCfg


@dataclass
class DatasetRE10kCfg(DatasetCfgCommon):
    name: Literal["re10k"]
    roots: list[Path]
    baseline_epsilon: float
    max_fov: float
    make_baseline_1: bool
    augment: bool


def get_fov(intrinsics: Tensor) -> Tensor:
    """[b, 3, 3] normalised intrinsics -> [b, 2] (fov_x, fov_y) in radians, as the reference computes it."""
    intrinsics_inv = intrinsics.inverse()

    def process_vector(vector):
        vector = torch.tensor(vector, dtype=torch.float32, device=intrinsics.device)
        vector = torch.einsum("bij,j->bi", intrinsics_inv, vector)
        return vector / vector.norm(dim=-1, keepdim=True)

    left, right = process_vector([0, 0.5, 1]), process_vector([1, 0.5, 1])
    top, bottom = process_vector([0.5, 0, 1]), process_vector([0.5, 1, 1])
    fov_x = (left * right).sum(dim=-1).acos()
    fov_y = (top * bottom).sum(dim=-1).acos()
    return torch.stack((fov_x, fov_y), dim=-1)


def reflect_extrinsics(extrinsics: Tensor) -> Tensor:
    reflect = torch.eye(4, dtype=torch.float32, device=extrinsics.device)
    reflect[0, 0] = -1
    return reflect @ extrinsics @ reflect


def decode_images(images: list[Tensor]) -> list[np.ndarray]:
    """JPEG bytes (uint8 tensors) -> decoded uint8 arrays, HWC for RGB."""
    return [np.array(Image.open(BytesIO(image.numpy().tobytes()))) for image in images]


class DatasetRE10k(IterableDataset):
    near: float = 0.1
    far: float = 1000.0

    def __init__(self, cfg: DatasetRE10kCfg, stage: Stage, view_sampler: ViewSampler | None,
                 cameras_only: bool = False) -> None:
        super().__init__()
        self.cfg = cfg
        self.stage = stage
        self.view_sampler = view_sampler
        self.cameras_only = cameras_only
        self.chunks = []
        for root in cfg.roots:
            root = Path(root) / self.data_stage
            self.chunks.extend(sorted(path for path in root.iterdir() if path.suffix == ".torch"))
        if cfg.overfit_to_scene is not None:
            chunk_path = self.index[cfg.overfit_to_scene]
            self.chunks = [chunk_path] * len(self.chunks)

    def shuffle(self, lst: list) -> list:
        indices = torch.randperm(len(lst))
        return [lst[x] for x in indices]

    def __iter__(self):
        if self.stage in ("train", "val"):
            self.chunks = self.shuffle(self.chunks)
        worker_info = torch.utils.data.get_worker_info()
        if self.stage == "test" and worker_info is not None:
            self.chunks = [chunk for i, chunk in enumerate(self.chunks) if i % worker_info.num_workers == worker_info.id]

        for chunk_path in self.chunks:
            chunk = torch.load(chunk_path, weights_only=True)
            if self.cfg.overfit_to_scene is not None:
                item = [x for x in chunk if x["key"] == self.cfg.overfit_to_scene]
                assert len(item) == 1
                chunk = item * len(chunk)
            if self.stage in ("train", "val"):
                chunk = self.shuffle(chunk)

            for example in chunk:
                out = self.convert_example(example)
                if out is not None:
                    yield out

    def convert_example(self, example: dict) -> dict | None:
        """One chunk entry -> the yielded example, or None where the reference skips it."""
        if self.cameras_only:
            return self.convert_cameras(example)
        extrinsics, intrinsics = self.convert_poses(example["cameras"])
        scene = example["key"]
        try:
            context_indices, target_indices = self.view_sampler.sample(scene, extrinsics, intrinsics)
        except ValueError:
            return None                                       # not enough frames
        if (get_fov(intrinsics).rad2deg() > self.cfg.max_fov).any():
            return None
        try:
            context_images = decode_images([example["images"][i.item()] for i in context_indices])
            target_images = decode_images([example["images"][i.item()] for i in target_indices])
        except IndexError:
            return None
        if any(im.shape != IMAGE_SHAPE for im in context_images + target_images):
            log.info("Skipped bad example %s: an image is not %s.", scene, IMAGE_SHAPE)
            return None

        context_extrinsics = extrinsics[context_indices]
        if context_extrinsics.shape[0] == 2 and self.cfg.make_baseline_1:
            a, b = context_extrinsics[:, :3, 3]
            scale = (a - b).norm()
            if scale < self.cfg.baseline_epsilon:
                log.info("Skipped %s because of insufficient baseline %.6f", scene, float(scale))
                return None
            extrinsics[:, :3, 3] /= scale
        else:
            scale = 1

        def views(indices: Tensor, images: list[np.ndarray]) -> dict:
            return {"extrinsics": extrinsics[indices], "intrinsics": intrinsics[indices],
                    "image": torch.from_numpy(np.stack(images)),
                    "near": self.get_bound("near", len(indices)) / scale,
                    "far": self.get_bound("far", len(indices)) / scale, "index": indices}

        out = {"context": views(context_indices, context_images), "target": views(target_indices, target_images),
               "scene": scene, "flip": torch.tensor(False)}
        # The reference's augmentation shim: one coin per example, drawn after the sampler; the images are
        # flipped on the device (device_shim), the extrinsics here.
        if self.stage == "train" and self.cfg.augment and not torch.rand(tuple()) < 0.5:
            for v in ("context", "target"):
                out[v]["extrinsics"] = reflect_extrinsics(out[v]["extrinsics"])
            out["flip"] = torch.tensor(True)
        return out

    def convert_cameras(self, example: dict) -> dict | None:
        """The `all` sampler's example without its images: {"extrinsics" [v, 4, 4], "intrinsics" [v, 3, 3] (as
        stored, before the crop shim), "scene", "num_frames"}, or None where the reference skips it: a field of view
        over max_fov, fewer images than cameras (its IndexError), a frame that would not decode to IMAGE_SHAPE, or
        with exactly two frames, an insufficient baseline (the two-view rescale then applies)."""
        extrinsics, intrinsics = self.convert_poses(example["cameras"])
        scene, v = example["key"], extrinsics.shape[0]
        if (get_fov(intrinsics).rad2deg() > self.cfg.max_fov).any() or len(example["images"]) < v:
            return None
        for i in range(v):
            image = Image.open(BytesIO(example["images"][i].numpy().tobytes()))   # reads the header only
            if (image.size[1], image.size[0], len(image.getbands())) != IMAGE_SHAPE:
                log.info("Skipped bad example %s: an image is not %s.", scene, IMAGE_SHAPE)
                return None
        if v == 2 and self.cfg.make_baseline_1:
            a, b = extrinsics[:, :3, 3]
            scale = (a - b).norm()
            if scale < self.cfg.baseline_epsilon:
                log.info("Skipped %s because of insufficient baseline %.6f", scene, float(scale))
                return None
            extrinsics[:, :3, 3] /= scale
        return {"extrinsics": extrinsics, "intrinsics": intrinsics, "scene": scene, "num_frames": v}

    def convert_poses(self, poses: Tensor) -> tuple[Tensor, Tensor]:
        """[b, 18] RE10k cameras -> (camera-to-world [b, 4, 4], normalised intrinsics [b, 3, 3])."""
        b, _ = poses.shape
        intrinsics = torch.eye(3, dtype=torch.float32).repeat(b, 1, 1)
        fx, fy, cx, cy = poses[:, :4].T
        intrinsics[:, 0, 0] = fx
        intrinsics[:, 1, 1] = fy
        intrinsics[:, 0, 2] = cx
        intrinsics[:, 1, 2] = cy
        w2c = torch.eye(4, dtype=torch.float32).repeat(b, 1, 1)
        w2c[:, :3] = poses[:, 6:].reshape(b, 3, 4)
        return w2c.inverse(), intrinsics

    def get_bound(self, bound: Literal["near", "far"], num_views: int) -> Tensor:
        value = torch.tensor(getattr(self, bound), dtype=torch.float32)
        return value.expand(num_views).clone()

    @property
    def data_stage(self) -> Stage:
        if self.cfg.overfit_to_scene is not None:
            return "test"
        if self.stage == "val":
            return "test"
        return self.stage

    @cached_property
    def index(self) -> dict[str, Path]:
        merged_index = {}
        data_stages = [self.data_stage]
        if self.cfg.overfit_to_scene is not None:
            data_stages = ("test", "train")
        for data_stage in data_stages:
            for root in self.cfg.roots:
                with (Path(root) / data_stage / "index.json").open("r") as f:
                    index = json.load(f)
                index = {k: Path(root) / data_stage / v for k, v in index.items()}
                assert not (set(merged_index.keys()) & set(index.keys()))
                merged_index = {**merged_index, **index}
        return merged_index

    def __len__(self) -> int:
        return len(self.index.keys())
