"""CPU tests of the optimiser's host side: the float64 oracle against torch, the segment table, ClipAdam's state
layout, the trainer's checkpoint saver and the training presets."""
import numpy as np
import pytest
import torch

from oracle import adam_oracle as ao
from pixelsplat_b200 import _lib, optim
from pixelsplat_b200.evaluation.checkpoint import load_checkpoint, read_checkpoint, save_checkpoint
from pixelsplat_b200.parallel import GradientReducer


def _tensors(seed=0, shapes=((3, 5), (7,), (1,), (2, 2, 2))):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g, dtype=torch.float64) for s in shapes]


@pytest.mark.parametrize("W", [1, 3, 2000])
def test_oracle_lr_factors_equal_linear_lr(W):
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.Adam([p], lr=1.5e-4)
    sched = torch.optim.lr_scheduler.LinearLR(opt, 1 / W, 1, total_iters=W)
    for t in range(min(W, 40) + 4):
        assert ao.warm_up_factor(t, W) * 1.5e-4 == pytest.approx(sched.get_last_lr()[0], rel=1e-12)
        assert optim.warm_up_factor(t, W) == ao.warm_up_factor(t, W)
        opt.step()
        sched.step()
    assert ao.warm_up_factor(W + 3, W) == 1.0


@pytest.mark.parametrize("scale", [10.0, 0.01])        # clipping active / inactive
def test_oracle_equals_torch_clip_adam_linear_lr_in_float64(scale):
    params = [torch.nn.Parameter(t.clone()) for t in _tensors()]
    opt = torch.optim.Adam(params, lr=1e-2)
    sched = torch.optim.lr_scheduler.LinearLR(opt, 1 / 3, 1, total_iters=3)
    oracle = ao.AdamOracle([p.detach().numpy() for p in params], lr=1e-2, warm_up_steps=3, max_norm=0.5)
    for step in range(10):
        grads = [scale * g for g in _tensors(seed=step + 1)]
        for p, g in zip(params, grads):
            p.grad = g.clone()
        norm = torch.nn.utils.clip_grad_norm_(params, 0.5)
        opt.step()
        sched.step()
        assert oracle.step([g.numpy() for g in grads]) == pytest.approx(float(norm), rel=1e-12)
        for p, q, m in zip(params, oracle.params, oracle.exp_avg):
            np.testing.assert_allclose(p.detach().numpy(), q, rtol=1e-11, atol=1e-14)
            np.testing.assert_allclose(opt.state[p]["exp_avg"].numpy(), m, rtol=1e-11, atol=1e-16)


def test_segment_table_offsets_alignment_and_empty_tensors():
    C = _lib.CLIP_ADAM_CHUNK
    base = 1 << 20
    rows = [(base, base + 4096, base + 8192, base + 12288, 1),          # one element, aligned
            (base, base + 4, base + 4, base + 4, 0),                    # empty: dropped
            (base + 16, base + 4100, base + 8196, base + 12292, C),      # gradient one element past a boundary
            (base + 32, base + 4096 + 12, base, base, 2 * C - 3),        # skew 3: fills two chunks exactly
            (base + 32, base + 4096 + 12, base, base, 2 * C - 2)]        # one more element: a third chunk
    table, chunks = optim.segment_table(rows)
    assert table.dtype == np.int64 and table.shape == (4, 6)
    assert table[:, 4].tolist() == [1, C, 2 * C - 3, 2 * C - 2]
    assert table[:, 5].tolist() == [0, 1, 3, 5] and chunks == 8
    assert [optim.vectorised(r) for r in table] == [True, False, False, False]
    assert optim.vectorised((base + 4, base + 20, base + 36, base + 52, 9, 0))
    with pytest.raises(ValueError, match="4-byte aligned"):
        optim.segment_table([(base + 2, base, base, base, 4)])
    assert _lib.lib.ps_clip_adam_segment_chunks(base + 12, 1) == 1
    assert _lib.lib.ps_clip_adam_segment_chunks(base + 12, C - 2) == 2


def _model():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(5, 7), torch.nn.ReLU(), torch.nn.Linear(7, 3))


def test_state_dict_round_trips_through_torch_adam():
    model = _model()
    adam = torch.optim.Adam(model.parameters(), lr=1.5e-4)
    sched = torch.optim.lr_scheduler.LinearLR(adam, 1 / 2000, 1, total_iters=2000)
    for _ in range(3):
        adam.zero_grad()
        model(torch.randn(4, 5)).square().sum().backward()
        adam.step()
        sched.step()
    params = list(model.parameters())
    ours = optim.ClipAdam(params, GradientReducer(params))
    ours.load_state_dict(adam.state_dict())              # lr is the scheduled one, initial_lr the base one
    assert ours.base_lr == 1.5e-4 and ours.steps == 3 and int(ours.step_counter) == 3
    assert ours.lr() == pytest.approx(sched.get_last_lr()[0], rel=1e-12)
    sd = ours.state_dict()
    assert sd["param_groups"][0]["lr"] == pytest.approx(sched.get_last_lr()[0], rel=1e-12)
    back = torch.optim.Adam(model.parameters(), lr=1.0)
    back.load_state_dict(sd)
    for p in params:
        assert back.state[p]["step"] == 3
        assert torch.equal(back.state[p]["exp_avg"], adam.state[p]["exp_avg"])
        assert torch.equal(back.state[p]["exp_avg_sq"], adam.state[p]["exp_avg_sq"])
    assert back.param_groups[0]["initial_lr"] == 1.5e-4 and back.param_groups[0]["betas"] == (0.9, 0.999)
    sch = ours.scheduler_state_dict()
    assert sch["last_epoch"] == 3 and sch["_last_lr"][0] == pytest.approx(sched.state_dict()["_last_lr"][0], rel=1e-12)

    # torch keeps no entry for a parameter that never had a gradient: zero moments here
    sd2 = adam.state_dict()
    del sd2["state"][0]
    ours.load_state_dict(sd2)
    assert not ours.moments(0)[0].any() and ours.moments(1)[0].any()

    sd["state"][1]["step"] = torch.tensor(5.0)
    with pytest.raises(ValueError, match="different steps"):
        ours.load_state_dict(sd)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ours.step()


def test_parameter_outside_the_reducer_is_rejected():
    model = _model()
    params = list(model.parameters())
    with pytest.raises(ValueError, match="not in the GradientReducer"):
        optim.ClipAdam(params, GradientReducer(params[:2]))


def test_saved_checkpoint_is_read_by_load_checkpoint(tmp_path):
    model = _model()
    params = list(model.parameters())
    opt = optim.ClipAdam(params, GradientReducer(params))
    path = save_checkpoint(tmp_path / "checkpoints" / "epoch=0-step=0.ckpt", model, 0, 0, opt.state_dict(),
                           opt.scheduler_state_dict(), {"torch": torch.get_rng_state()})
    assert [p.name for p in path.parent.iterdir()] == [path.name]        # the temporary name is gone
    other = _model()
    with torch.no_grad():
        for p in other.parameters():
            p.zero_()
    assert load_checkpoint(path, other) == 0
    assert all(torch.equal(a, b) for a, b in zip(model.parameters(), other.parameters()))
    ckpt = read_checkpoint(path)
    assert set(ckpt) == {"epoch", "global_step", "state_dict", "optimizer_states", "lr_schedulers", "rng_state"}
    opt.load_state_dict(ckpt["optimizer_states"][0])
    ckpt["state_dict"]["decoder.x"] = torch.zeros(1)
    torch.save(ckpt, tmp_path / "foreign.ckpt")
    with pytest.raises(ValueError, match="outside 'encoder"):
        load_checkpoint(tmp_path / "foreign.ckpt", other)


def test_presets_hold_the_reference_values():
    from pixelsplat_b200.training import presets as tp
    for name in ("re10k", "acid"):
        p = tp.train_preset(name)
        # config/experiment/{re10k,acid}.yaml
        assert (p.batch_size, p.max_steps, p.losses) == (7, 300_001, ("mse", "lpips")) and p.depth_mode is None
        # config/main.yaml
        assert (p.num_workers, p.checkpoint_every, p.lr, p.warm_up_steps, p.max_norm) == (16, 5000, 1.5e-4, 2000, 0.5)
        # config/loss/mse.yaml, lpips.yaml
        assert (p.mse_weight, p.lpips_weight, p.lpips_apply_after_step) == (1.0, 0.05, 150_000)
        # config/dataset/view_sampler/bounded.yaml + view_sampler_dataset_specific_config/bounded_re10k.yaml
        vs = p.view_sampler
        assert (vs.num_context_views, vs.num_target_views) == (2, 4)
        assert (vs.min_distance_between_context_views, vs.max_distance_between_context_views) == (45, 45)
        assert (vs.initial_min_distance_between_context_views, vs.initial_max_distance_between_context_views) == (25, 25)
        assert (vs.min_distance_to_context_views, vs.warm_up_steps) == (0, 150_000)
    # config/main.yaml: seed, data_loader.train.seed
    assert (tp.SEED, tp.LOADER_SEED) == (111123, 1234)
    d = tp.train_preset("re10k_depth_loss")
    # config/experiment/re10k_depth_loss.yaml, config/loss/depth.yaml
    assert (d.max_steps, d.losses, d.depth_mode) == (350_001, ("mse", "lpips", "depth"), "depth")
    assert (d.depth_weight, d.depth_sigma_image, d.depth_use_second_derivative) == (0.25, 12.0, True)
    cfg = tp.dataset_cfg(tp.train_preset("re10k"), "datasets/re10k", overfit_to_scene="abc")
    assert cfg.view_sampler is tp.train_preset("re10k").view_sampler and cfg.overfit_to_scene == "abc"
    assert cfg.image_shape == [256, 256] and cfg.make_baseline_1 and cfg.augment
    losses = tp.make_losses(d, lpips=torch.nn.Identity())
    assert [l.name for l in losses] == ["mse", "lpips", "depth"] and losses[1].cfg.apply_after_step == 150_000
    with pytest.raises(ValueError, match="unknown preset"):
        tp.train_preset("kitti")


def test_command_line_parses():
    from pixelsplat_b200.training.__main__ import parse
    a = parse(["--dataset-root", "d", "--output", "o", "--preset", "acid", "--max-steps", "5", "--deterministic",
               "--backbone-weights", "v.pth", "r.pth", "--overfit-to-scene", "s"])
    assert a.preset == "acid" and a.max_steps == 5 and a.deterministic and len(a.backbone_weights) == 2
    assert a.batch_size is None and a.resume is None and a.overfit_to_scene == "s"
