"""GPU tests of csrc/optimizer.cu behind optim.ClipAdam: against the float64 oracle (oracle/adam_oracle.py) with
torch's own float32 clip_grad_norm_ + Adam + LinearLR as the error yardstick, and the properties the training step
relies on: untouched gradients, frozen all-zero tensors, bit-reproducibility, CUDA-graph replay, NaN propagation."""
import numpy as np
import pytest
import torch

from oracle import adam_oracle as ao
from pixelsplat_b200 import _lib, optim
from pixelsplat_b200.parallel import GradientReducer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = _lib.CLIP_ADAM_CHUNK
W = 3                                        # warm-up steps: steps 1 and 2 lie inside, 5 and 50 after
LR = 1e-3

SETS = {
    # hundreds of tiny tensors: every chunk is heads and tails
    "tiny": [1 + (i * 7) % 33 for i in range(300)],
    # sizes around the vector width and the chunk size, at whatever bucket offsets the odd ones before them leave
    "straddle": [1, 2, 3, 4, 5, 7, 8, 9, C - 1, C, C + 1, 2 * C - 1, 2 * C, 2 * C + 1, 1023, 1024, 1025, 3 * C + 2],
    # multiples of four in storage of their own: every tensor takes the float4 route
    "aligned": [3 * C, 64, 2 * C + 4, 4, 5 * C + 256],
    "big": [5, 2 ** 24 + 3, 2],
}


def build(sizes, seed=0, views=False, bucket_bytes=1 << 20):
    """Parameters (each its own storage, or views at odd offsets of one buffer), their reducer and ClipAdam."""
    g = torch.Generator().manual_seed(seed)
    init = [torch.randn(n, generator=g) for n in sizes]
    if views:
        flat = torch.empty(sum(sizes) + 1, device=DEV)
        params, off = [], 1
        for t in init:
            params.append(torch.nn.Parameter(flat[off:off + t.numel()].copy_(t.to(DEV))))
            off += t.numel()
    else:
        params = [torch.nn.Parameter(t.to(DEV)) for t in init]
    reducer = GradientReducer(params, bucket_bytes=bucket_bytes)
    opt = optim.ClipAdam(params, reducer, lr=LR, warm_up_steps=W, max_norm=0.5)
    return init, params, reducer, opt


def grads_for(sizes, step, scale, seed=100):
    g = torch.Generator().manual_seed(seed + step)
    return [scale * torch.randn(n, generator=g) for n in sizes]


def set_grads(params, grads):
    for p, g in zip(params, grads):
        p.grad.copy_(g.to(DEV))


def scale_for(sizes, regime):
    n = float(sum(sizes))
    return {"clipping": 1.0, "inactive": 0.1 / n ** 0.5, "edge": 0.5 / n ** 0.5}[regime]


def rel(xs, refs):
    """Largest absolute difference over all tensors over the largest reference magnitude."""
    diff = max(float(np.abs(x.detach().double().cpu().numpy() - r).max()) for x, r in zip(xs, refs))
    return diff / max(float(np.abs(r).max()) for r in refs)


def check_against_oracle(name, regime, checkpoints, views=False):
    sizes = SETS[name]
    scale = scale_for(sizes, regime)
    # one bucket for the 16M-element tensor and its neighbours: its gradient then starts two elements in
    init, params, reducer, opt = build(sizes, views=views, bucket_bytes=(1 << 28) if name == "big" else (1 << 20))
    oracle = ao.AdamOracle([t.numpy() for t in init], lr=LR, warm_up_steps=W, max_norm=0.5)
    t_params = [torch.nn.Parameter(t.to(DEV)) for t in init]
    adam = torch.optim.Adam(t_params, lr=LR)
    sched = torch.optim.lr_scheduler.LinearLR(adam, 1 / W, 1, total_iters=W)
    routes = [optim.vectorised(r) for r in _table(opt, params)]
    assert all(routes) if name == "aligned" else not all(routes)        # which sets reach the scalar route
    for step in range(1, max(checkpoints) + 1):
        grads = grads_for(sizes, step, scale)
        reducer.zero_grad()
        set_grads(params, grads)
        before = [b["flat"].clone() for b in reducer.buckets]
        assert opt.lr() == pytest.approx(oracle.lr_now(), rel=1e-12)
        opt.step()
        assert all(torch.equal(a, b["flat"]) for a, b in zip(before, reducer.buckets))     # .grad is only read
        for p, g in zip(t_params, grads):
            p.grad = g.to(DEV)
        t_norm = torch.nn.utils.clip_grad_norm_(t_params, 0.5)
        adam.step()
        sched.step()
        o_norm = oracle.step([g.numpy() for g in grads])
        if step not in checkpoints:
            continue
        e_norm = abs(float(opt.grad_norm) - o_norm) / o_norm
        assert e_norm <= 4 * abs(float(t_norm) - o_norm) / o_norm + 1e-6, (step, e_norm)
        ours = (params, [opt.moments(i)[0] for i in range(len(params))],
                [opt.moments(i)[1] for i in range(len(params))])
        theirs = (t_params, [adam.state[p]["exp_avg"] for p in t_params], [adam.state[p]["exp_avg_sq"] for p in t_params])
        for what, a, b, r in zip(("param", "exp_avg", "exp_avg_sq"), ours, theirs,
                                 (oracle.params, oracle.exp_avg, oracle.exp_avg_sq)):
            e, e_t = rel(a, r), rel(b, r)
            assert e <= 4 * e_t + 2e-7, (name, regime, step, what, e, e_t)
        assert int(opt.step_counter) == step
    if regime == "clipping":
        assert float(opt.grad_norm) > 5.0
    elif regime == "inactive":
        assert float(opt.grad_norm) < 0.5
    else:
        assert 0.45 < float(opt.grad_norm) < 0.55


def _table(opt, params):
    return [(p.data_ptr(), p.grad.data_ptr(), *(m.data_ptr() for m in opt.moments(i)), p.numel(), 0)
            for i, p in enumerate(params)]


@pytest.mark.parametrize("regime", ["clipping", "inactive", "edge"])
@pytest.mark.parametrize("name", ["tiny", "straddle", "aligned"])
def test_kernel_matches_the_float64_oracle(name, regime):
    check_against_oracle(name, regime, (1, 2, 5, 50))


def test_parameters_that_are_views_at_odd_offsets():
    check_against_oracle("straddle", "clipping", (1, 2, 5), views=True)


def test_one_tensor_of_16m_elements():
    check_against_oracle("big", "clipping", (1, 2, 5))      # 50 steps of the float64 oracle on 2^24 elements take long


def test_zero_gradient_tensor_stays_bit_unchanged_while_neighbours_move():
    sizes = [C + 3, 37, 2 * C]
    init, params, reducer, opt = build(sizes)
    for step in range(1, 6):
        reducer.zero_grad()
        grads = grads_for(sizes, step, 1.0)
        grads[1].zero_()
        set_grads(params, grads)
        opt.step()
    assert torch.equal(params[1].detach().cpu(), init[1])
    assert not opt.moments(1)[0].any() and not opt.moments(1)[1].any()
    assert not torch.equal(params[0].detach().cpu(), init[0]) and not torch.equal(params[2].detach().cpu(), init[2])


def run_steps(sizes, n, graph_after=None):
    init, params, reducer, opt = build(sizes)
    graph = None
    for step in range(1, n + 1):
        set_grads(params, grads_for(sizes, step, 0.02))
        if graph_after is not None and step == graph_after + 1:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                opt.step()
        if graph is not None:
            graph.replay()
        else:
            opt.step()
    torch.cuda.synchronize()
    return ([p.detach().clone() for p in params], [opt.moments(i)[1].clone() for i in range(len(params))],
            opt.grad_norm.clone(), int(opt.step_counter))


def test_two_runs_give_identical_bits_and_a_graph_replays_the_schedule():
    sizes = SETS["straddle"] + SETS["tiny"][:40]
    a, b = run_steps(sizes, 7), run_steps(sizes, 7)
    g = run_steps(sizes, 7, graph_after=3)                  # 3 eager steps, capture, 4 replays with fresh gradients
    for other in (b, g):
        assert other[3] == 7 and torch.equal(a[2], other[2])
        assert all(torch.equal(x, y) for x, y in zip(a[0], other[0]))
        assert all(torch.equal(x, y) for x, y in zip(a[1], other[1]))


def test_nan_gradient_gives_nan_parameters_as_torch_does():
    sizes = [C + 1, 9]
    init, params, reducer, opt = build(sizes)
    grads = grads_for(sizes, 1, 1.0)
    grads[0][17] = float("nan")
    set_grads(params, grads)
    opt.step()
    t_params = [torch.nn.Parameter(t.to(DEV)) for t in init]
    for p, g in zip(t_params, grads):
        p.grad = g.to(DEV)
    torch.nn.utils.clip_grad_norm_(t_params, 0.5)
    torch.optim.Adam(t_params, lr=LR).step()
    assert torch.isnan(opt.grad_norm)
    for p, t in zip(params, t_params):
        assert torch.isnan(t).all() and torch.isnan(p).all()


def test_bad_arguments_are_rejected_before_a_launch():
    import ctypes
    d = _lib.ClipAdamDesc(n_segments=0, n_chunks=0, warm_up_steps=3, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8,
                          max_norm=0.5)
    out = ctypes.c_size_t()
    with pytest.raises(ValueError, match="at least one segment"):
        _lib.check(_lib.lib.ps_clip_adam_workspace_bytes(ctypes.byref(d), ctypes.byref(out)), "workspace")
    d.n_segments, d.n_chunks, d.beta1 = 1, 1, 1.0
    with pytest.raises(ValueError, match="bad scalars"):
        _lib.check(_lib.lib.ps_clip_adam_workspace_bytes(ctypes.byref(d), ctypes.byref(out)), "workspace")
