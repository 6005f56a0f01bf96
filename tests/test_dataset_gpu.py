"""GPU tests of the data pipeline end to end: DatasetRE10k through a DataLoader and device_shim equals what the
reference's DatasetRE10k (with its host crop shim) yields on the tiny dataset of tests/dataset_golden.py, images
bit for bit and cameras exactly; the batch then feeds EncoderEpipolar's data shim and forward."""
import numpy as np
import pytest
import torch

from pixelsplat_b200.data import device_shim
from tests import dataset_golden as dg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _batches(stage: str, batch_size: int):
    torch.manual_seed(int(dg.fixture()["train_seed"]) if stage == "train" else 0)
    # the loader's own seed comes from a generator of its own, so the dataset draws from torch's RNG as the
    # reference's run did
    loader = torch.utils.data.DataLoader(dg.dataset(stage), batch_size=batch_size, num_workers=0,
                                         pin_memory=True, generator=torch.Generator().manual_seed(0))
    return [device_shim(b, dg.SHAPES[stage]) for b in loader]


@pytest.mark.parametrize("stage,batch_size", [("test", 1), ("train", 2)])
def test_dataset_and_device_shim_equal_the_reference(stage, batch_size):
    want = dg.expected(stage)
    got = []
    for b in _batches(stage, batch_size):
        for i in range(len(b["scene"])):
            got.append({"scene": b["scene"][i], **{v: {k: x[i] for k, x in b[v].items()}
                                                   for v in ("context", "target")}})
    assert [g["scene"] for g in got] == [w["scene"] for w in want]
    for g, w in zip(got, want):
        for v in ("context", "target"):
            img = g[v]["image"]
            assert img.is_cuda and img.dtype == torch.float32 and img.shape[-2:] == dg.SHAPES[stage]
            u = (img.double() * 255).round()
            assert torch.equal(img, (u / 255).float())
            dg.assert_images_equal(u.to(torch.uint8).cpu().numpy(), w[v], (g["scene"], v))
            for k in ("intrinsics", "extrinsics", "near", "far", "index"):
                assert np.array_equal(g[v][k].cpu().numpy(), w[v][k]), (g["scene"], v, k)


def test_batch_feeds_the_encoder():
    from pixelsplat_b200.encoder.encoder_epipolar import EncoderEpipolar
    from tests.test_backbone_cpu import _re10k_encoder_cfg
    batch = _batches("train", 2)[0]
    torch.manual_seed(0)
    enc = EncoderEpipolar(_re10k_encoder_cfg(), num_context_views=2).to(DEV)
    batch = enc.get_data_shim()(batch)
    with torch.no_grad():
        gs = enc(batch["context"], global_step=0)
    torch.cuda.synchronize()
    assert gs.means.shape == (2, 2 * 256 * 256 * 3, 3) and torch.isfinite(gs.means).all()
