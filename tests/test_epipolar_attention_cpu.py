"""The float64 restatement of the fused epipolar attention (tests/epipolar_attention_f64.py), checked without a GPU:

  1. its sample positions and bilinear features against the REFERENCE sampler's own float64 run
     (tests/golden/epipolar_geometry.npz, written by oracle/make_epipolar_golden.py on the seeded 4-channel images);
  2. its positional encoding against pixelsplat_b200/encoder/positional_encoding.py evaluated in float64;
  3. the soft-max invariants: mass sums to 1 over the other views, lse is the log-sum-exp of the scores, every z row
     is a convex combination of that row's samples; and autograd's gradients against central differences.

The GPU tests (test_epipolar_attention_gpu.py) hold the kernels to this restatement.
"""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import epipolar_attention_f64 as ref
from tests import golden_util as gu

GOLD = Path(__file__).resolve().parent / "golden"
# (tag, b, v, grid) of the float64 reference runs in the fixture
GEOMETRY = [("generic", 2, 2, (8, 8)), ("parallel", 1, 3, (8, 8)), ("diverging", 1, 2, (8, 8)),
            ("generic3", 1, 3, (6, 10))]


@pytest.mark.parametrize("tag,b,v,grid", GEOMETRY)
def test_samples_match_the_reference_sampler(tag, b, v, grid):
    gold = np.load(GOLD / "epipolar_geometry.npz")
    g = lambda k: torch.from_numpy(gold[f"{tag}_f64_{k}"])
    seg, valid = g("segments"), g("valid")
    S = gold[f"{tag}_f64_rel_disparity"].shape[-1]
    # positions: the reference forms xy_min + u (xy_max - xy_min) from the same segment ends (1 ulp apart at most)
    xy = ref.sample_positions(seg, S)
    d_xy = float((xy - g("xy_sample")).abs().max())
    assert d_xy < 1e-12, d_xy
    # features: the fixture stores the reference's float64 samples rounded to float32, so the bar is half an ulp
    images = gu.seeded_like("sampler.images", (b, v, 4, *grid), 1.0, torch.float64)
    f = ref.sample_features(images.permute(0, 1, 3, 4, 2), seg, valid, S)
    gold_f = g("features").double()
    assert f.shape == gold_f.shape == (b, v, v - 1, grid[0] * grid[1], S, 4)
    assert not f[~valid].any()
    d_f = (f - gold_f).abs()
    assert bool((d_f <= 2.0 ** -24 * gold_f.abs() + 1e-12).all()), float(d_f.max())
    assert (float(f.abs().max()) > 0.5) == bool(valid.any())      # the diverging rig leaves no valid ray
    # and grid_sample, the reference's own sampler, agrees to float64 round-off on the unrounded values
    gs = []
    for vi, row in enumerate(ref.other_views(v)):
        per = []
        for o, src in enumerate(row):
            grid_ = (2 * xy[:, vi, o] - 1).reshape(b, -1, 1, 2)
            smp = torch.nn.functional.grid_sample(images[:, src], grid_, mode="bilinear", padding_mode="zeros",
                                                  align_corners=False)
            per.append(smp[..., 0].permute(0, 2, 1).reshape(b, grid[0] * grid[1], S, 4))
        gs.append(torch.stack(per, 1))
    gs = torch.stack(gs, 1) * valid.double()[..., None, None]
    assert float((f - gs).abs().max()) < 1e-12


@pytest.mark.parametrize("octaves", [1, 10, 16])
def test_positional_encoding_matches_the_module(octaves):
    """PositionalEncoding evaluated in float64 keeps its float32 buffers' values: frequencies float32(2 pi) 2^k (what
    the restatement uses) and the phase float32(pi / 2), which is 4.4e-8 above pi / 2.  The cosine half therefore
    differs by up to that phase error; the sine half agrees to float64 round-off of the phase (rd 2 pi 2^15 ~ 2e5)."""
    from pixelsplat_b200.encoder.positional_encoding import PositionalEncoding
    g = torch.Generator().manual_seed(octaves)
    rd = torch.cat([torch.rand(4096, generator=g, dtype=torch.float64), torch.tensor([0.0, 1.0, 0.5, 1e-7],
                                                                                   dtype=torch.float64)])
    mod = PositionalEncoding(octaves).double()(rd[:, None])
    ours = ref.positional_encoding(rd, 2 * octaves)
    assert ours.shape == mod.shape == (rd.numel(), 2 * octaves)
    phase_err = float(np.float32(np.pi / 2)) - np.pi / 2
    assert float((ours[:, 0::2] - mod[:, 0::2]).abs().max()) < 1e-10
    assert float((ours[:, 1::2] - mod[:, 1::2]).abs().max()) < 1.01 * phase_err + 1e-10
    assert torch.equal(ours[-4, 0::2], torch.zeros(octaves)) and torch.equal(ours[-4, 1::2], torch.ones(octaves))


def _case(b=2, v=3, grid=(3, 4), S=5, heads=2, npe=4, C=4, bias=True, seed=0):
    """Small random inputs: segments partly off the map, a few invalid rays, view 0's first query all invalid."""
    g = torch.Generator().manual_seed(seed)
    h, w = grid
    ov, R = v - 1, h * w
    n = b * v * R
    seg = torch.rand(b, v, ov, R, 4, generator=g, dtype=torch.float64) * 1.4 - 0.2
    valid = torch.rand(b, v, ov, R, generator=g) > 0.2
    valid[0, 0, :, 0] = False
    rd = torch.rand(b, v, ov, R, S, generator=g, dtype=torch.float64)
    r = lambda *s: torch.randn(s, generator=g, dtype=torch.float64)
    return dict(feat_cl=r(b, v, h, w, C), segments=seg, valid=valid, rel_disparity=rd, qt=r(n, heads, C),
                pq=0.5 * r(n, heads, npe), bias=r(n, heads, ov) if bias else None, heads=heads), \
        dict(dz=r(n, heads, C), de=r(n, heads, npe), dmass=r(n, heads, ov))


@pytest.mark.parametrize("bias", [False, True])
def test_softmax_invariants(bias):
    x, _ = _case(bias=bias)
    out = ref.forward(**x)
    n, H, ov = out["mass"].shape
    S = x["rel_disparity"].shape[-1]
    assert torch.allclose(out["mass"].sum(-1), torch.ones(n, H, dtype=torch.float64), rtol=0, atol=1e-14)
    # lse against the scores restated directly from the samples and the PE
    f, pe = out["samples"], out["pe"]
    score = torch.einsum("nhc,nosc->nhos", x["qt"], f) + torch.einsum("nhj,nosj->nhos", x["pq"], pe)
    if bias:
        score = score + x["bias"][..., None]
    smax = score.reshape(n, H, -1).max(-1).values
    lse = smax + torch.log(torch.exp(score.reshape(n, H, -1) - smax[..., None]).sum(-1))
    assert float((out["lse"] - lse).abs().max()) < 1e-12
    # z is a convex combination of the row's samples: the weights a = exp(score - lse) are >= 0 and sum to 1
    a = torch.exp(score - out["lse"][..., None, None])
    assert bool((a >= 0).all()) and torch.allclose(a.sum((-1, -2)), torch.ones(n, H, dtype=torch.float64), atol=1e-14)
    assert float((out["z"] - torch.einsum("nhos,nosc->nhc", a, f)).abs().max()) < 1e-12
    lo, hi = f.amin((1, 2))[:, None], f.amax((1, 2))[:, None]              # per row and channel
    assert bool(((out["z"] >= lo - 1e-12) & (out["z"] <= hi + 1e-12)).all())
    # a query whose rays are all invalid sees only zero samples: z = 0, but the PE and the bias still spread mass
    first = out["z"][0]
    assert torch.equal(first, torch.zeros_like(first)) and bool((out["mass"][0] > 0).all())
    assert bool((out["e"][0].abs() > 0).any())
    assert S == f.shape[2]


@pytest.mark.parametrize("bias", [False, True])
def test_gradients_match_central_differences(bias):
    """autograd of <z, dz> + <e, de> + <mass, dmass> against central differences of the same scalar (a few entries of
    each input), with and without a bias: the mass cotangent reaches dqt, dpq and dfeat either way."""
    x, cot = _case(b=1, v=3, grid=(2, 3), S=3, heads=2, npe=4, bias=bias, seed=3)
    got = ref.forward_backward(**x, **cot)

    def loss(**over):
        o = ref.forward(**{**x, **over})
        return float((o["z"] * cot["dz"]).sum() + (o["e"] * cot["de"]).sum() + (o["mass"] * cot["dmass"]).sum())

    g = torch.Generator().manual_seed(9)
    names = [("qt", "dqt"), ("pq", "dpq"), ("feat_cl", "dfeat")] + ([("bias", "dbias")] if bias else [])
    for name, gname in names:
        t = x[name]
        for i in torch.randint(0, t.numel(), (6,), generator=g).tolist():
            eps = 1e-6
            tp, tm = t.clone(), t.clone()
            tp.view(-1)[i] += eps
            tm.view(-1)[i] -= eps
            fd = (loss(**{name: tp}) - loss(**{name: tm})) / (2 * eps)
            an = float(got[gname].reshape(-1)[i])
            assert abs(fd - an) <= 1e-6 * (1 + abs(fd)), (name, i, fd, an)
    # without the mass cotangent the gradients change: it is not dropped
    no_mass = ref.forward_backward(**x, dz=cot["dz"], de=cot["de"])
    assert float((no_mass["dqt"] - got["dqt"]).abs().max()) > 1e-3
