"""Generates the dataset fixtures under tests/golden/: a tiny synthetic RE10k-format dataset (re10k_tiny/) and what
the REFERENCE's own DatasetRE10k yields on it (dataset_re10k_v1.npz).  It needs a checkout of the
reference at REFERENCE (below):

    python oracle/make_dataset_golden.py

TEST INFRASTRUCTURE.  The dataset has a "test" and a "train" chunk of 360 x 640 JPEGs (smooth seeded content,
made with PIL) and random poses.  Besides the scenes that load, the test chunk holds one scene each that the
reference skips for a field of view over max_fov, for an image that is not 360 x 640, for a context baseline under
baseline_epsilon and for having no evaluation-index entry; the train chunk holds one with too few frames.

The reference runs (a) in test stage with ViewSamplerEvaluation on evaluation_index.json at image_shape 180 x 320
and (b) in train stage with ViewSamplerBounded, augmentation on, torch.manual_seed(train_seed), at 256 x 256
(train_seed, stored in the fixture, is the first seed that gives both a flipped and an unflipped example).  Every yielded example is recorded: scene,
per view set the extrinsics, intrinsics, near, far and indices, plus the augmentation coin, read by wrapping the
reference's apply_augmentation_shim.  The reference's float images are u / 255 in float32 exactly (checked here), so
each view's image is pinned by u: the SHA-256 of u's bytes (uint8 [3, h, w], C order) and, to locate a mismatch,
every 8th row and column of u.  Storing u whole would make the fixture about 1.3 MB.

The reference's view_sampler package imports dacite (oracle/_stubs/dacite) and, for the IndexEntry dataclass,
src/evaluation/evaluation_index_generator.py, whose own imports (lightning, matplotlib) are absent offline; that
module is pre-registered with an IndexEntry of the same two fields.
"""
from __future__ import annotations

import dataclasses
import hashlib
import io
import json
import shutil
import sys
import types
from pathlib import Path

import numpy as np
import torch
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]
REFERENCE = Path("/root/reference")
OUT = ROOT / "tests" / "golden"
DATA = OUT / "re10k_tiny"
TEST_SHAPE = (180, 320)
TRAIN_SHAPE = (256, 256)
TRAIN_NUM_TARGET_VIEWS = 1


def _jpeg(rng: np.random.Generator, h: int = 360, w: int = 640) -> torch.Tensor:
    """A smooth seeded RGB image with some texture, JPEG-encoded (quality 85), as the chunks store frames."""
    yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
    f = rng.uniform(1, 6, (3, 2))
    p = rng.uniform(0, 2 * np.pi, (3, 2))
    img = np.stack([0.5 + 0.25 * np.sin(f[c, 0] * 2 * np.pi * xx + p[c, 0]) * np.cos(f[c, 1] * 2 * np.pi * yy + p[c, 1])
                    for c in range(3)], -1)
    for _ in range(4):                                           # a few sharp-edged discs
        cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(10, 60)
        img[(yy * h - cy) ** 2 + (xx * w - cx) ** 2 < r * r] = rng.uniform(0, 1, 3)
    img = np.clip(img * 255, 0, 255).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, format="JPEG", quality=85)
    return torch.frombuffer(bytearray(buf.getvalue()), dtype=torch.uint8)


def _cameras(rng: np.random.Generator, n: int, fx: float = 0.9, static: bool = False) -> torch.Tensor:
    """[n, 18] RE10k cameras: fx fy cx cy (normalised), two unused entries, w2c [3, 4] row-major."""
    out = np.zeros((n, 18), np.float32)
    for i in range(n):
        a = rng.normal(0, 0.1, 3)
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        R = np.eye(3) + np.sin(0.5) * K + (1 - np.cos(0.5)) * K @ K
        u, _, vt = np.linalg.svd(R)
        R = u @ vt
        t = np.array([0.0, 0.0, 0.0]) if static else np.array([0.3 * i, 0.05 * i, 0.02 * i]) + rng.normal(0, 0.01, 3)
        out[i, :4] = (fx, fx * 16 / 9, 0.5, 0.5)
        out[i, 6:] = np.concatenate([R, t[:, None]], 1).reshape(-1)
    return torch.from_numpy(out)


def write_dataset() -> None:
    rng = np.random.default_rng(20261016)
    frames = [_jpeg(rng) for _ in range(14)]
    small = _jpeg(rng, 240, 320)

    def scene(key, n, images, **kw):
        return {"key": key, "url": f"https://example.invalid/{key}", "timestamps": torch.arange(n) * 33_333,
                "cameras": _cameras(rng, n, **kw), "images": images}

    test = [scene("aaa", 6, frames[0:6]), scene("bbb", 6, frames[6:12]),
            scene("ccc", 6, frames[0:6], fx=0.25),                       # field of view over max_fov
            scene("ddd", 6, [small] * 6),                                # not 360 x 640
            scene("eee", 6, frames[0:6], static=True),                   # zero baseline
            scene("fff", 6, frames[6:12])]                               # no evaluation-index entry
    train = [scene("ggg", 8, frames[6:14]), scene("hhh", 8, frames[0:8]),
             scene("iii", 2, frames[0:2])]                               # too few frames for the bounded sampler
    if DATA.exists():
        shutil.rmtree(DATA)
    for stage, chunk in (("test", test), ("train", train)):
        (DATA / stage).mkdir(parents=True)
        torch.save(chunk, DATA / stage / "000000.torch")
        (DATA / stage / "index.json").write_text(json.dumps({s["key"]: "000000.torch" for s in chunk}))
    index = {"aaa": {"context": [0, 4], "target": [1, 3]}, "bbb": {"context": [1, 5], "target": [2]},
             "ccc": {"context": [0, 2], "target": [1]}, "ddd": {"context": [0, 2], "target": [1]},
             "eee": {"context": [0, 4], "target": [2]}, "fff": None}
    (DATA / "evaluation_index.json").write_text(json.dumps(index))


def load_reference():
    for p in (str(ROOT / "oracle" / "_stubs"), str(REFERENCE)):
        if p not in sys.path:
            sys.path.insert(0, p)
    pkg = types.ModuleType("src.dataset")
    pkg.__path__ = [str(REFERENCE / "src" / "dataset")]
    sys.modules.setdefault("src.dataset", pkg)

    @dataclasses.dataclass
    class IndexEntry:
        context: tuple[int, int]
        target: tuple[int, ...]

    gen = types.ModuleType("src.evaluation.evaluation_index_generator")
    gen.IndexEntry = IndexEntry
    sys.modules.setdefault("src.evaluation.evaluation_index_generator", gen)
    from omegaconf import DictConfig
    from src.global_cfg import set_cfg
    set_cfg(DictConfig({"dataset": {"view_sampler": {"num_context_views": 2}}}))
    from src.dataset import dataset_re10k
    from src.dataset import view_sampler
    return dataset_re10k, view_sampler


def dataset_cfgs(ds_mod, vs_mod, stage: str):
    """(dataset cfg, view sampler cfg) of the reference's re10k config for `stage` on re10k_tiny."""
    if stage == "test":
        vs = vs_mod.ViewSamplerEvaluationCfg("evaluation", DATA / "evaluation_index.json", 2)
        shape = TEST_SHAPE
    else:
        vs = vs_mod.ViewSamplerBoundedCfg("bounded", 2, TRAIN_NUM_TARGET_VIEWS, 2, 6, 0, 0, 2, 6)
        shape = TRAIN_SHAPE
    cfg = ds_mod.DatasetRE10kCfg(image_shape=list(shape), background_color=[0.0, 0.0, 0.0],
                                 cameras_are_circular=False, overfit_to_scene=None, view_sampler=vs,
                                 name="re10k", roots=[DATA], baseline_epsilon=1e-3, max_fov=100.0,
                                 make_baseline_1=True, augment=True)
    return cfg, vs


def run_reference(ds_mod, vs_mod, stage: str, seed: int) -> list[dict]:
    cfg, vs = dataset_cfgs(ds_mod, vs_mod, stage)
    sampler = vs_mod.get_view_sampler(vs, stage, False, False, None)
    flips = []
    original = ds_mod.apply_augmentation_shim

    def recording(example, generator=None):
        out = original(example, generator)
        flips.append(out is not example)
        return out

    ds_mod.apply_augmentation_shim = recording
    try:
        torch.manual_seed(seed)
        examples = list(ds_mod.DatasetRE10k(cfg, stage, sampler))
    finally:
        ds_mod.apply_augmentation_shim = original
    if stage != "train":
        flips = [False] * len(examples)
    for ex, f in zip(examples, flips):
        ex["flip"] = f
    return examples


def image_digest(u: np.ndarray) -> str:
    """SHA-256 of one view's uint8 [3, h, w] image in C order (tests/dataset_golden.py computes the same)."""
    return hashlib.sha256(np.ascontiguousarray(u, dtype=np.uint8).tobytes()).hexdigest()


def record(examples: list[dict], stage: str) -> dict:
    out = {f"{stage}/count": np.array(len(examples)),
           f"{stage}/scene": np.array([e["scene"] for e in examples]),
           f"{stage}/flip": np.array([e["flip"] for e in examples])}
    for i, e in enumerate(examples):
        for v in ("context", "target"):
            for k in ("extrinsics", "intrinsics", "near", "far", "index"):
                out[f"{stage}/{i}/{v}/{k}"] = e[v][k].numpy()
            x = e[v]["image"]
            u = (x.double() * 255).round().to(torch.uint8)
            assert torch.equal(torch.tensor(u.numpy() / 255, dtype=torch.float32), x), "image is not u / 255"
            out[f"{stage}/{i}/{v}/image_sha256"] = np.array([image_digest(a) for a in u.numpy()])
            out[f"{stage}/{i}/{v}/image_sub"] = u.numpy()[:, :, ::8, ::8]
    return out


def main() -> None:
    write_dataset()
    ds_mod, vs_mod = load_reference()
    test = run_reference(ds_mod, vs_mod, "test", 0)
    assert [e["scene"] for e in test] == ["aaa", "bbb"], [e["scene"] for e in test]
    for seed in range(100):
        train = run_reference(ds_mod, vs_mod, "train", seed)
        if len(set(e["flip"] for e in train)) == 2:
            break
    assert sorted(e["scene"] for e in train) == ["ggg", "hhh"]
    fixture = {**record(test, "test"), **record(train, "train"), "train_seed": np.array(seed)}
    np.savez_compressed(OUT / "dataset_re10k_v1.npz", **fixture)
    size = sum(p.stat().st_size for p in DATA.rglob("*") if p.is_file())
    print(f"train seed {seed}, flips {[e['flip'] for e in train]}; dataset {size / 1e3:.0f} kB, fixture "
          f"{(OUT / 'dataset_re10k_v1.npz').stat().st_size / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
