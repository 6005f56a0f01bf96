"""CPU tests of LPIPS: the float64 restatement of the lpips package's LPIPS(net="vgg") (oracle/lpips_oracle.py) and its
gradient, exact properties, the dropout hash, the module's state-dict keys and weight loading (never a download),
LossLpips' empty state dict, and the C ABI's and the Python layer's argument checks (which reject before anything
reaches a device)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import lpips_oracle as lo


def _features(seed, n=2, shapes=((6, 5, 7), (9, 3, 4))):
    g = torch.Generator().manual_seed(seed)
    # away from zero: at an all-zero column the norm has a kink, and finite differences straddle it
    relu = lambda s: torch.randn((n, *s), generator=g, dtype=torch.float64).abs() + 0.05
    return [relu(s) for s in shapes], [relu(s) for s in shapes], [torch.rand(s[0], generator=g, dtype=torch.float64)
                                                                   for s in shapes]


def test_oracle_head_gradcheck():
    f0, f1, w = _features(0)
    f0 = [t.requires_grad_(True) for t in f0]
    f1 = [t.requires_grad_(True) for t in f1]
    fn = lambda a0, a1, b0, b1: lo.head([a0, a1], [b0, b1], w)
    assert torch.autograd.gradcheck(fn, (*f0, *f1), eps=1e-6, atol=1e-8)
    masks = [torch.from_numpy(lo.dropout_mask(7, l, tuple(t.shape))) for l, t in enumerate(f0)]
    fn = lambda a0, a1, b0, b1: lo.head([a0, a1], [b0, b1], w, masks)
    assert torch.autograd.gradcheck(fn, (*f0, *f1), eps=1e-6, atol=1e-8)


def test_oracle_whole_gradcheck_at_16x16():
    sd = {k: v.double() for k, v in lo.random_state_dict(1).items()}
    g = torch.Generator().manual_seed(2)
    a = torch.rand((1, 3, 16, 16), generator=g, dtype=torch.float64).requires_grad_(True)
    b = torch.rand((1, 3, 16, 16), generator=g, dtype=torch.float64)
    assert torch.autograd.gradcheck(lambda x: lo.lpips(x, b, sd, normalize=True), (a,), eps=1e-6, atol=1e-7,
                                    nondet_tol=0.0, fast_mode=True)


def test_identical_inputs_give_zero_and_the_distance_is_symmetric():
    sd = {k: v.double() for k, v in lo.random_state_dict(3).items()}
    g = torch.Generator().manual_seed(4)
    a = torch.rand((2, 3, 32, 24), generator=g, dtype=torch.float64)
    b = torch.rand((2, 3, 32, 24), generator=g, dtype=torch.float64)
    assert lo.lpips(a, a, sd, normalize=True).shape == (2, 1, 1, 1)
    assert float(lo.lpips(a, a, sd, normalize=True).abs().max()) == 0.0
    d_ab, d_ba = lo.lpips(a, b, sd, normalize=True), lo.lpips(b, a, sd, normalize=True)
    assert float((d_ab - d_ba).abs().max()) <= 1e-15 * float(d_ab.abs().max()) and float(d_ab.min()) > 0
    # an all-zero feature column normalises to zero (no NaN in the forward)
    f = [torch.zeros(1, 4, 2, 2, dtype=torch.float64)]
    assert float(lo.head(f, [torch.ones_like(f[0])], [torch.ones(4, dtype=torch.float64)])) == pytest.approx(1.0)


def test_dropout_hash_keep_rate_and_independence():
    shape = (3, 64, 32, 32)
    m0 = lo.dropout_mask(12345, 0, shape)
    assert set(np.unique(m0)) == {0.0, 2.0}
    n = m0.size
    rate = float((m0 == 2).mean())
    assert abs(rate - 0.5) <= 4 * 0.5 / n ** 0.5, rate          # Bernoulli(1/2): within 4 sigma
    assert abs(m0.mean() - 1.0) <= 8 / n ** 0.5                  # E[m] = 1
    others = (lo.dropout_mask(12346, 0, shape), lo.dropout_mask(12345, 1, shape), lo.dropout_mask(-12345, 0, shape))
    for other in others:
        agree = float((other == m0).mean())
        assert abs(agree - 0.5) <= 4 * 0.5 / n ** 0.5, agree    # unrelated streams
    # neighbouring elements are not correlated
    flat = (m0.reshape(-1) == 2).astype(np.float64)
    corr = np.corrcoef(flat[:-1], flat[1:])[0, 1]
    assert abs(corr) < 4 / n ** 0.5
    # a negative seed is its uint64 two's complement
    assert np.array_equal(lo.dropout_mask(-1, 2, (5,)), lo.dropout_mask(2 ** 64 - 1, 2, (5,)))
    assert np.array_equal(lo.dropout_mask(99, 4, (2, 3)), lo.dropout_mask(99, 4, (6,)).reshape(2, 3))


def _expected_keys():
    keys = {"scaling_layer.shift", "scaling_layer.scale"}
    for i in lo.CONVS:
        keys |= {f"net.slice{lo.slice_of(i)}.{i}.weight", f"net.slice{lo.slice_of(i)}.{i}.bias"}
    return keys | {f"lin{k}.model.1.weight" for k in range(5)}


def test_state_dict_keys_and_shapes():
    from pixelsplat_b200.lpips import Lpips
    m = Lpips()
    sd = m.state_dict()
    assert set(sd) == _expected_keys() == set(lo.random_state_dict(0))
    ref = lo.random_state_dict(0)
    assert all(sd[k].shape == ref[k].shape for k in sd)
    assert not any(p.requires_grad for p in m.parameters())
    np.testing.assert_allclose(sd["scaling_layer.shift"].reshape(-1).numpy(), lo.SHIFT, rtol=1e-7)
    np.testing.assert_allclose(sd["scaling_layer.scale"].reshape(-1).numpy(), lo.SCALE, rtol=1e-7)
    # the package's duplicate `lins.{k}` keys are accepted and dropped
    dup = dict(ref) | {f"lins.{k}.model.1.weight": ref[f"lin{k}.model.1.weight"] + 1 for k in range(5)}
    m.load_state_dict(dup)
    assert all(torch.equal(m.state_dict()[k], ref[k]) for k in ref)


def _write_weight_files(tmp_path, seed):
    ref = lo.random_state_dict(seed)
    vgg = {}
    for i in lo.CONVS:
        for p in ("weight", "bias"):
            vgg[f"features.{i}.{p}"] = ref[f"net.slice{lo.slice_of(i)}.{i}.{p}"]
    vgg["classifier.0.weight"] = torch.zeros(4, 2)                 # torchvision's file has the classifier too
    vgg["classifier.0.bias"] = torch.zeros(4)
    lin = {f"lin{k}.model.1.weight": ref[f"lin{k}.model.1.weight"] for k in range(5)}
    torch.save(vgg, tmp_path / "vgg16-397923af.pth")
    (tmp_path / "lpips" / "weights" / "v0.1").mkdir(parents=True)
    torch.save(lin, tmp_path / "lpips" / "weights" / "v0.1" / "vgg.pth")
    return ref


def test_from_files_maps_torchvision_and_package_keys(tmp_path):
    from pixelsplat_b200.lpips import Lpips
    ref = _write_weight_files(tmp_path, 5)
    m = Lpips.from_files(tmp_path / "vgg16-397923af.pth", tmp_path / "lpips" / "weights" / "v0.1" / "vgg.pth")
    sd = m.state_dict()
    assert set(sd) == set(ref) and all(torch.equal(sd[k], ref[k]) for k in ref)


def test_from_files_default_locations(tmp_path, monkeypatch):
    import importlib.machinery
    import importlib.util

    from pixelsplat_b200 import lpips as lp
    ref = _write_weight_files(tmp_path, 6)
    (tmp_path / "hub" / "checkpoints").mkdir(parents=True)
    (tmp_path / "vgg16-397923af.pth").rename(tmp_path / "hub" / "checkpoints" / "vgg16-397923af.pth")
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    spec = importlib.machinery.ModuleSpec("lpips", None, is_package=True)
    spec.submodule_search_locations = [str(tmp_path / "lpips")]
    monkeypatch.setattr(importlib.util, "find_spec", lambda name, *a: spec if name == "lpips" else None)
    sd = lp.Lpips.from_files().state_dict()
    assert all(torch.equal(sd[k], ref[k]) for k in ref)


def test_missing_files_raise_and_never_download(tmp_path, monkeypatch):
    import importlib.util

    from pixelsplat_b200 import lpips as lp

    def no_download(*a, **k):
        raise AssertionError("a download was attempted")

    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_download)
    monkeypatch.setattr(torch.hub, "download_url_to_file", no_download)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "empty_hub"))
    with pytest.raises(FileNotFoundError, match="vgg16-397923af.pth"):
        lp.Lpips.from_files()
    _write_weight_files(tmp_path, 7)
    with pytest.raises(FileNotFoundError, match="vgg.pth"):
        lp.Lpips.from_files(tmp_path / "vgg16-397923af.pth", tmp_path / "nowhere" / "vgg.pth")
    monkeypatch.setattr(importlib.util, "find_spec", lambda name, *a: None)
    with pytest.raises(FileNotFoundError, match="no lpips package"):
        lp.Lpips.from_files(tmp_path / "vgg16-397923af.pth")


def test_loss_lpips_adds_no_state_dict_keys():
    from pixelsplat_b200.loss import (LossLpips, LossLpipsCfg, LossLpipsCfgWrapper, LossMse, LossMseCfg,
                                      LossMseCfgWrapper)
    from pixelsplat_b200.lpips import Lpips
    loss = LossLpips(LossLpipsCfgWrapper(LossLpipsCfg(0.05, 150_000)), lpips=Lpips())
    assert loss.name == "lpips" and loss.cfg.weight == 0.05 and loss.cfg.apply_after_step == 150_000
    assert loss.state_dict() == {} and list(loss.parameters()) == []
    assert len(list(loss.buffers())) == len(_expected_keys())
    losses = torch.nn.ModuleList([LossMse(LossMseCfgWrapper(LossMseCfg(1.0))), loss])
    assert losses.state_dict() == {}
    # before apply_after_step: a float32 zero on the image's device
    batch = {"target": {"image": torch.rand(1, 2, 3, 16, 16)}}
    z = loss(type("P", (), {"color": torch.rand(1, 2, 3, 16, 16)})(), batch, None, 149_999)
    assert z.dtype == torch.float32 and z.device == batch["target"]["image"].device and float(z) == 0.0


def _desc(n_layers=2, N=2, shapes=((64, 8, 8), (128, 4, 4)), seed=None):
    from pixelsplat_b200 import _lib
    buf = ctypes.create_string_buffer(16)
    p = ctypes.addressof(buf)
    d = _lib.LpipsDesc()
    d.n_layers, d.N = n_layers, N
    for l, (c, h, w) in enumerate(shapes[:n_layers]):
        d.layers[l] = _lib.LpipsLayer(p, p, p, c, h, w)
    d.dropout_seed = seed
    return d, p, buf


def test_abi_rejects_invalid_arguments():
    from pixelsplat_b200 import _lib
    lib = _lib.lib
    size = ctypes.c_size_t()
    d, p, _keep = _desc()
    assert lib.ps_lpips_workspace_bytes(ctypes.byref(d), ctypes.byref(size)) == 0
    # C = 64: 128-pixel tiles (one per image), C = 128: 64-pixel tiles -> one partial per (layer, image)
    assert size.value % 256 == 0 and size.value >= 4 * 4
    assert lib.ps_lpips_workspace_bytes(ctypes.byref(d), None) == 1
    assert lib.ps_lpips_workspace_bytes(None, ctypes.byref(size)) == 1
    ws_bytes = size.value
    bad = []
    for n_layers, N in ((0, 2), (6, 2), (2, 0), (-1, 2)):
        x, _, _k = _desc(min(max(n_layers, 0), 5), N)
        x.n_layers = n_layers
        bad.append(x)
    for shape in ((0, 8, 8), (8193, 1, 1), (64, 0, 8), (64, 8, -1), (512, 2048, 2048)):
        x, _, _k = _desc(2, 2, ((64, 8, 8), shape))
        bad.append(x)
    bufs = [ctypes.create_string_buffer(16) for _ in range(3)]
    q = [ctypes.addressof(b) for b in bufs]
    for x in bad:
        assert lib.ps_lpips_workspace_bytes(ctypes.byref(x), ctypes.byref(size)) == 1
        assert b"bad shape" in lib.ps_last_error()
        assert lib.ps_lpips_forward(ctypes.byref(x), q[0], q[1], ws_bytes, None) == 1
        g = _lib.LpipsGrads()
        g.d_x0[0] = g.d_x0[1] = q[2]
        assert lib.ps_lpips_backward(ctypes.byref(x), q[0], ctypes.byref(g), None) == 1
    # NULL pointers, one at a time
    for field in ("x0", "x1", "weight"):
        x, _, _k = _desc()
        setattr(x.layers[1], field, None)
        assert lib.ps_lpips_forward(ctypes.byref(x), q[0], q[1], ws_bytes, None) == 1 and b"NULL" in lib.ps_last_error()
        g = _lib.LpipsGrads()
        g.d_x0[0] = g.d_x0[1] = q[2]
        assert lib.ps_lpips_backward(ctypes.byref(x), q[0], ctypes.byref(g), None) == 1
        assert b"NULL" in lib.ps_last_error()
    assert lib.ps_lpips_forward(ctypes.byref(d), None, q[1], ws_bytes, None) == 1 and b"NULL" in lib.ps_last_error()
    assert lib.ps_lpips_forward(ctypes.byref(d), q[0], None, ws_bytes, None) == 1 and b"NULL" in lib.ps_last_error()
    assert lib.ps_lpips_forward(ctypes.byref(d), q[0], q[1], ws_bytes - 1, None) == 1
    assert b"workspace" in lib.ps_last_error()
    g = _lib.LpipsGrads()
    g.d_x1[0] = q[2]                                      # layer 1 has neither side
    assert lib.ps_lpips_backward(ctypes.byref(d), q[0], ctypes.byref(g), None) == 1
    assert b"neither" in lib.ps_last_error()
    g.d_x0[1] = q[2]
    assert lib.ps_lpips_backward(ctypes.byref(d), None, ctypes.byref(g), None) == 1
    assert lib.ps_lpips_backward(ctypes.byref(d), q[0], None, None) == 1


def test_python_layer_rejects_invalid_inputs():
    from pixelsplat_b200.lpips import Lpips, lpips_head
    m = Lpips()
    a = torch.rand(2, 3, 32, 32)
    with pytest.raises(ValueError, match="no CPU path"):
        m(a, a.clone())
    with pytest.raises(ValueError, match="float32"):
        m(a.double(), a.double())
    with pytest.raises(ValueError, match="one shape"):
        m(a, a[:, :, :31])
    with pytest.raises(ValueError, match=r"\[N, 3, H, W\]"):
        m(a[:, :2], a[:, :2])
    with pytest.raises(ValueError, match="one shape"):
        m(a[0], a[0])
    with pytest.raises(ValueError, match="at least 16"):
        m(torch.rand(1, 3, 15, 40), torch.rand(1, 3, 15, 40))
    f = [torch.rand(2, 8, 4, 4)]
    w = [torch.rand(8)]
    with pytest.raises(ValueError, match="no CPU path"):
        lpips_head(f, [f[0].clone()], w)
    with pytest.raises(ValueError, match="1 to 5 layers"):
        lpips_head(f * 6, f * 6, w * 6)
    with pytest.raises(ValueError, match="one shape"):
        lpips_head(f, [torch.rand(2, 8, 4, 3)], w)
    with pytest.raises(ValueError, match=r"\[C\]"):
        lpips_head(f, [f[0].clone()], [torch.rand(7)])
    with pytest.raises(ValueError, match="float32"):
        lpips_head([f[0].double()], [f[0].double()], w)
