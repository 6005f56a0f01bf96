"""Generates tests/golden/evaluation_index_v1.npz by running the REFERENCE's EvaluationIndexGenerator.test_step
(src/evaluation/evaluation_index_generator.py) on the CPU.  Authoring container only:

    python oracle/make_index_golden.py

TEST INFRASTRUCTURE.  lightning is absent offline: oracle/_stubs/lightning gives test_step a LightningModule whose
device is the CPU.  The preview helpers it imports (image_io, annotation, layout) are replaced by empty modules,
because previews are off.  Everything else is the reference's own code.  For each configuration of
tests/index_util.CONFIGS, one generator runs test_step over the trajectories of tests/index_util.FAMILIES in that
order (so the random stream runs across scenes, as in the reference).  The image only gives test_step its shape: a
zero-stride expanded tensor.

project_rays is wrapped to record every overlap the walk evaluates.  test_step calls it twice per candidate k:
first with the context rays and camera k (overlap_b), then with k's rays and the context camera (overlap_a).  The
camera a call receives is a view of the scene's extrinsics, so its frame is read from its offset.  The fixture
stores, per configuration and family:
  cam/<family>/extrinsics, cam/<family>/intrinsics   the float32 cameras
  <config>/<family>/pairs    int64 [n, 4] (context, k, count_a, count_b) in evaluation order, where count is the
                             number of rays whose overlaps_image is set (the mean the reference thresholds is
                             float32(count) / float32(h * w), asserted here)
  entries                    JSON {config: {family: null | {"context": [a, b], "target": [...]}}}
  configs                    JSON {config: {"h", "w", "cfg": the generator's fields}}
  re10k_tiny                 JSON: the index the reference's generator makes of tests/golden/re10k_tiny's test split
                             in the "small" configuration, read by the reference's DatasetRE10k with the `all` view
                             sampler at 256 x 256 through a DataLoader with 8 workers, as generate_evaluation_index
                             reads it (its JSON layout, with the key order it writes)
"""
from __future__ import annotations

import json
import os
import sys
import types
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
REFERENCE = Path("/root/reference")
sys.path.insert(0, str(ROOT))
from tests import index_util  # noqa: E402

OUT = ROOT / "tests" / "golden" / "evaluation_index_v1.npz"
TINY = ROOT / "tests" / "golden" / "re10k_tiny"
DEFAULTS = dict(num_target_views=3, min_distance=45, max_distance=135, min_overlap=0.6, max_overlap=1.0, seed=123)


def load_generator():
    os.environ.setdefault("TQDM_DISABLE", "1")
    for p in (str(ROOT / "oracle" / "_stubs"), str(REFERENCE)):
        if p not in sys.path:
            sys.path.insert(0, p)
    for name, attrs in (("src.misc.image_io", ("save_image",)), ("src.visualization.annotation", ("add_label",)),
                        ("src.visualization.layout", ("add_border", "hcat"))):
        m = types.ModuleType(name)
        for a in attrs:
            setattr(m, a, None)
        sys.modules[name] = m
    import src.evaluation.evaluation_index_generator as gen
    return gen


def reference_tiny_index(gen, fields: dict) -> str:
    import json as _json
    import tempfile

    import torch
    from src.dataset.dataset_re10k import DatasetRE10k, DatasetRE10kCfg
    from src.dataset.view_sampler.view_sampler_all import ViewSamplerAll, ViewSamplerAllCfg
    cfg = DatasetRE10kCfg(image_shape=[256, 256], background_color=[0.0, 0.0, 0.0], cameras_are_circular=False,
                          overfit_to_scene=None, view_sampler=ViewSamplerAllCfg("all"), name="re10k", roots=[TINY],
                          baseline_epsilon=1e-3, max_fov=100.0, make_baseline_1=True, augment=True)
    dataset = DatasetRE10k(cfg, "test", ViewSamplerAll(cfg.view_sampler, "test", False, False, None))
    loader = torch.utils.data.DataLoader(dataset, batch_size=1, num_workers=8)
    with tempfile.TemporaryDirectory() as tmp:
        module = gen.EvaluationIndexGenerator(gen.EvaluationIndexGeneratorCfg(output_path=Path(tmp),
                                                                            save_previews=False, **fields))
        for i, batch in enumerate(loader):
            module.test_step(batch, i)
        module.save_index()
        text = (Path(tmp) / "evaluation_index.json").read_text()
    print(f"re10k_tiny: {_json.loads(text)}")
    return text


def main() -> None:
    import torch
    gen = load_generator()
    calls: list[tuple[int, int, float]] = []
    base = {"ptr": 0}
    project_rays = gen.project_rays

    def recording_project_rays(origins, directions, extrinsics, intrinsics, *args, **kwargs):
        out = project_rays(origins, directions, extrinsics, intrinsics, *args, **kwargs)
        frame = (extrinsics.data_ptr() - base["ptr"]) // (16 * extrinsics.element_size())
        mask = out["overlaps_image"]
        calls.append((frame, int(mask.sum()), float(mask.float().mean())))
        return out

    gen.project_rays = recording_project_rays
    configs_by_name = dict((n, o) for n, _, _, o in index_util.CONFIGS)
    out: dict[str, np.ndarray] = {}
    entries: dict[str, dict] = {}
    configs: dict[str, dict] = {}
    for family in index_util.FAMILIES:
        E, K = index_util.trajectory(family)
        out[f"cam/{family}/extrinsics"], out[f"cam/{family}/intrinsics"] = E, K
    for name, h, w, overrides in index_util.CONFIGS:
        fields = {**DEFAULTS, **overrides}
        cfg = gen.EvaluationIndexGeneratorCfg(output_path=Path("unused"), save_previews=False, **fields)
        module = gen.EvaluationIndexGenerator(cfg)
        entries[name] = {}
        configs[name] = {"h": h, "w": w, "cfg": fields}
        for family in index_util.FAMILIES:
            E = torch.from_numpy(out[f"cam/{family}/extrinsics"])[None]
            K = torch.from_numpy(out[f"cam/{family}/intrinsics"])[None]
            v = E.shape[1]
            base["ptr"] = E.data_ptr()
            image = torch.zeros(()).expand(1, v, 3, h, w)
            calls.clear()
            module.test_step({"target": {"image": image, "extrinsics": E, "intrinsics": K}, "scene": [family]}, 0)
            assert len(calls) % 2 == 0
            pairs = []
            for (k, count_b, mean_b), (c, count_a, mean_a) in zip(calls[0::2], calls[1::2]):
                for count, mean in ((count_a, mean_a), (count_b, mean_b)):
                    assert mean == float(np.float32(count) / np.float32(h * w)), (count, mean)
                pairs.append((c, k, count_a, count_b))
            out[f"{name}/{family}/pairs"] = np.array(pairs, dtype=np.int64).reshape(-1, 4)
            e = module.index[family]
            entries[name][family] = None if e is None else {"context": list(e.context), "target": list(e.target)}
            print(f"{name} {family}: {len(pairs)} pairs, entry {entries[name][family]}", flush=True)
    out["re10k_tiny"] = np.array(reference_tiny_index(gen, {**DEFAULTS, **configs_by_name["small"]}))
    out["entries"] = np.array(json.dumps(entries))
    out["configs"] = np.array(json.dumps(configs))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
