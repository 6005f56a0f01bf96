"""CPU tests of the training's validation: the comparison image's layout, the stage-"val" dataset on the tiny RE10k
dataset (tests/dataset_golden.py) and its seeded generators, and the `--val-every` command-line option."""
from dataclasses import replace

import pytest
import torch

from pixelsplat_b200.data import ViewSamplerBoundedCfg
from pixelsplat_b200.training import presets as tp
from pixelsplat_b200.training.trainer import comparison_layout, validation_rng
from tests import dataset_golden as dg

# re10k_tiny's scenes have 2 to 8 frames: the presets' context gap of 25 to 45 frames would skip them all
TINY_SAMPLER = ViewSamplerBoundedCfg("bounded", 2, 4, 2, 6, 0, 0, 2, 6)


def test_comparison_layout_places_each_view_and_fills_the_rest_with_white():
    g = torch.Generator().manual_seed(0)
    ctx, gt, prob, det = (torch.rand(n, 3, 8, 8, generator=g) * 0.5 for n in (2, 4, 4, 4))
    out = comparison_layout(ctx, gt, prob, det)
    # 4 targets of 8 rows with 3 gaps of 8, 4 columns of 8 with 3 gaps of 8, a border of 8 around
    assert out.shape == (3, 4 * 8 + 3 * 8 + 16, 4 * 8 + 3 * 8 + 16) and out.dtype == torch.float32
    covered = torch.zeros(out.shape[1:], dtype=torch.bool)
    for col, views in enumerate((ctx, gt, prob, det)):
        x = 8 + col * 16
        for i, view in enumerate(views):
            y = 8 + i * 16                                    # aligned to the top: the context column starts there too
            assert torch.equal(out[:, y:y + 8, x:x + 8], view), (col, i)
            covered[y:y + 8, x:x + 8] = True
    assert (out[:, ~covered] == 1.0).all()                  # gaps, the context column's padding and the border


def val_cfg():
    return tp.dataset_cfg(replace(tp.train_preset("re10k"), view_sampler=TINY_SAMPLER), dg.DATA)


def draw(seed: int, n: int) -> list[dict]:
    torch.manual_seed(seed)
    it = iter(tp.make_val_dataset(val_cfg(), None))
    return [next(it) for _ in range(n)]


def list_all(seed: int) -> list[dict]:
    torch.manual_seed(seed)
    return list(tp.make_val_dataset(val_cfg(), None))


def test_val_dataset_reads_the_test_split_with_four_targets_and_no_flip():
    cfg = val_cfg()
    assert cfg.augment                                      # the training's augmentation is on; stage "val" skips it
    test_scenes = set(dg.dataset("test").index)
    for seed in range(4):
        examples = list_all(seed)
        # ccc (field of view), ddd (image shape) and eee (baseline) are the fixture's skipped scenes
        assert sorted(e["scene"] for e in examples) == ["aaa", "bbb", "fff"] and {"aaa", "bbb", "fff"} <= test_scenes
        for e in examples:
            assert e["context"]["index"].shape == (2,) and e["target"]["index"].shape == (4,)
            assert not bool(e["flip"])


def test_val_dataset_is_reproducible_from_its_seed_and_the_fork_hides_its_draws():
    a, b = draw(3, 3), draw(3, 3)
    for x, y in zip(a, b):
        assert x["scene"] == y["scene"]
        for v in ("context", "target"):
            assert torch.equal(x[v]["index"], y[v]["index"]) and torch.equal(x[v]["image"], y[v]["image"])
    orders = {tuple(e["scene"] for e in list_all(s)) for s in range(4)}
    assert len(orders) > 1                                  # the shuffle does draw from the generator

    torch.manual_seed(11)
    before = torch.get_rng_state()
    it = iter(tp.make_val_dataset(val_cfg(), None))
    with validation_rng(0, 250):
        first = next(it)
    assert torch.equal(torch.get_rng_state(), before)
    with validation_rng(0, 250):
        torch.manual_seed(0)                                # what the fork saw is not what it restores
    assert torch.equal(torch.get_rng_state(), before)
    # the same (rank, step) gives the same example; another step another draw of the sampler
    with validation_rng(0, 250):
        again = next(iter(tp.make_val_dataset(val_cfg(), None)))
    assert again["scene"] == first["scene"] and torch.equal(again["target"]["index"], first["target"]["index"])


def test_command_line_val_every_defaults_to_zero_and_rejects_negative_values(capsys):
    from pixelsplat_b200.training.__main__ import parse
    common = ["--dataset-root", str(dg.DATA), "--output", "out"]
    assert parse(common).val_every == 0
    assert parse(common + ["--val-every", "250"]).val_every == 250
    with pytest.raises(SystemExit):
        parse(common + ["--val-every", "-1"])
    assert "--val-every" in capsys.readouterr().err


def test_command_line_without_a_test_split_stops_before_the_first_step(tmp_path):
    from pixelsplat_b200.training.__main__ import main
    root = tmp_path / "data"
    (root / "train").mkdir(parents=True)
    with pytest.raises(SystemExit) as e:
        main(["--dataset-root", str(root), "--output", str(tmp_path / "out"), "--val-every", "1"])
    assert "test" in str(e.value) and "--val-every 0" in str(e.value)
    assert not (tmp_path / "out").exists()
