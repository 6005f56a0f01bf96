"""CPU tests of pixelsplat_b200.data.DatasetRE10k against what the reference's DatasetRE10k yields on the same
tiny dataset (tests/dataset_golden.py): scene order, skips, indices, extrinsics (reflections included),
intrinsics before the crop, near / far and flip decisions exactly, and the crop shim restated on the host
(oracle/resample_oracle.py) on the yielded uint8 views equals the reference's images bit for bit."""
import numpy as np
import pytest
import torch

from oracle import resample_oracle as ro
from pixelsplat_b200.data.crop_shim import scaled_shape
from pixelsplat_b200.data.view_sampler import (StepTracker, ViewSamplerBounded, ViewSamplerBoundedCfg,
                                               ViewSamplerEvaluation, ViewSamplerEvaluationCfg)
from tests import dataset_golden as dg


@pytest.mark.parametrize("stage", ["test", "train"])
def test_dataset_matches_the_reference(stage):
    want, got = dg.expected(stage), dg.examples(stage)
    assert [e["scene"] for e in got] == [e["scene"] for e in want]
    assert [bool(e["flip"]) for e in got] == [e["flip"] for e in want]
    if stage == "train":
        assert {e["flip"] for e in want} == {False, True}
    h_out, w_out = dg.SHAPES[stage]
    for g, w in zip(got, want):
        for v in ("context", "target"):
            gv, wv = g[v], w[v]
            assert np.array_equal(gv["index"].numpy(), wv["index"])
            assert np.array_equal(gv["extrinsics"].numpy(), wv["extrinsics"])
            for k in ("near", "far"):
                assert np.array_equal(gv[k].numpy(), wv[k])
            assert gv["image"].dtype == torch.uint8 and gv["image"].shape[1:] == (360, 640, 3)
            # the crop shim on the host: intrinsics as center_crop updates them, images bit for bit
            h_s, w_s = scaled_shape(360, 640, (h_out, w_out))
            K = gv["intrinsics"].clone()
            K[..., 0, 0] *= w_s / w_out
            K[..., 1, 1] *= h_s / h_out
            assert np.array_equal(K.numpy(), wv["intrinsics"])
            crop = ((h_s - h_out) // 2, (w_s - w_out) // 2, h_out, w_out)
            out = np.stack([ro.resample_and_crop(img, (h_s, w_s), crop, bool(g["flip"])).transpose(2, 0, 1)
                            for img in gv["image"].numpy()])
            dg.assert_images_equal(out, wv, (g["scene"], v))


def test_test_stage_splits_chunks_per_worker():
    loader = torch.utils.data.DataLoader(dg.dataset("test"), batch_size=None, num_workers=2)
    scenes = [e["scene"] for e in loader]
    assert sorted(scenes) == ["aaa", "bbb"]           # one chunk: worker 0 yields it, worker 1 nothing


def test_bounded_sampler_warm_up_reads_the_shared_step():
    cfg = ViewSamplerBoundedCfg("bounded", 2, 1, 20, 40, 0, 100, 2, 6)
    tracker = StepTracker()
    s = ViewSamplerBounded(cfg, "train", False, False, tracker)
    ext = torch.eye(4).expand(100, 4, 4)
    torch.manual_seed(0)
    gaps = [int(c[1] - c[0]) for c, _ in (s.sample("x", ext, ext[:, :3, :3]) for _ in range(20))]
    assert max(gaps) <= 6 and min(gaps) >= 2
    tracker.set_step(100)
    gaps = [int(c[1] - c[0]) for c, _ in (s.sample("x", ext, ext[:, :3, :3]) for _ in range(20))]
    assert min(gaps) >= 20 and max(gaps) <= 40
    with pytest.raises(ValueError):
        s.sample("x", ext[:10], ext[:10, :3, :3])


def test_evaluation_sampler_adds_a_third_context_index():
    cfg = ViewSamplerEvaluationCfg("evaluation", dg.DATA / "evaluation_index.json", 3)
    s = ViewSamplerEvaluation(cfg, "test", False, False, None)
    c, t = s.sample("aaa", torch.eye(4).expand(6, 4, 4), torch.eye(3).expand(6, 3, 3))
    assert c.tolist() == [0, 2, 4] and t.tolist() == [1, 3]
    with pytest.raises(ValueError):
        s.sample("fff", torch.eye(4).expand(6, 4, 4), torch.eye(3).expand(6, 3, 3))
