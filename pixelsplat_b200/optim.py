"""`ClipAdam`: the optimiser end of the reference's training step (Lightning's gradient_clip_val 0.5,
`optim.Adam(lr=1.5e-4)` and the `LinearLR` warm-up of model_wrapper.py's configure_optimizers) as one call of
csrc/optimizer.cu: two launches over the `GradientReducer`'s gradient buckets, no host synchronisation, the step
counter on the device (so a captured CUDA graph replays the schedule), bit-reproducible.

One step counter serves every parameter, where torch keeps one per parameter and skips a parameter whose `.grad` is
None.  The two agree for this model: an unused parameter's bucket view holds zeros, and with exp_avg = exp_avg_sq = 0
a zero gradient gives an update of exactly 0, so the parameter and its moments stay bit-unchanged until its first
non-zero gradient -- but its bias corrections then start from the global step rather than from 1.  A state whose
entries carry different steps therefore cannot be loaded (`load_state_dict` raises).
"""
from __future__ import annotations

import ctypes
from typing import Iterable, Sequence

import numpy as np
import torch

from . import _lib
from .parallel import GradientReducer


def segment_table(rows: Sequence[tuple[int, int, int, int, int]]) -> tuple[np.ndarray, int]:
    """The kernel's segment table from (param, grad, exp_avg, exp_avg_sq addresses, element count) per tensor, empty
    tensors dropped: int64 [n, 6] rows of `_lib.CLIP_ADAM_SEGMENT_FIELDS`, and the total number of chunks."""
    table, chunks = [], 0
    for p, g, m, v, count in rows:
        if count == 0:
            continue
        if (p | g | m | v) & 3:
            raise ValueError("ClipAdam: a float32 tensor is not 4-byte aligned")
        table.append((p, g, m, v, count, chunks))
        chunks += _lib.lib.ps_clip_adam_segment_chunks(g, count)
    return np.array(table, dtype=np.int64).reshape(-1, len(_lib.CLIP_ADAM_SEGMENT_FIELDS)), chunks


def vectorised(row: Sequence[int]) -> bool:
    """Whether the update kernel walks this table row in float4 units: all four tensors sit at the same offset from
    a 16-byte boundary (the norm pass always does, it reads the gradient alone)."""
    p, g, m, v = (int(x) for x in row[:4])
    return ((p ^ g) | (m ^ g) | (v ^ g)) & 15 == 0


def warm_up_factor(steps_taken: int, warm_up_steps: int) -> float:
    if warm_up_steps <= 0:
        return 1.0
    start = 1.0 / warm_up_steps
    return start + (1.0 - start) * min(steps_taken, warm_up_steps) / warm_up_steps


class ClipAdam:
    """Clip-by-global-norm + Adam + linear warm-up over `params`, whose gradients live in `reducer`'s buckets.

    `params` is the model's parameter list (index = position, as in torch's optimiser state); every one of them must
    be float32 and be held by `reducer`.  The moments live in two flat buffers per bucket, laid out like the bucket.
    Call `step()` after `reducer.finish()`; `.grad` is left as backward produced it.  `grad_norm` (float32 scalar on
    the device) is the last step's norm before clipping."""

    LAUNCHES_PER_STEP = 2

    def __init__(self, params: Iterable[torch.nn.Parameter], reducer: GradientReducer, lr: float = 1.5e-4,
                 warm_up_steps: int = 2000, max_norm: float = 0.5, betas: tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-8) -> None:
        self.params = list(params)
        if not self.params:
            raise ValueError("ClipAdam: no parameters")
        self.reducer = reducer
        self.base_lr, self.warm_up_steps, self.max_norm = float(lr), int(warm_up_steps), float(max_norm)
        self.betas, self.eps = (float(betas[0]), float(betas[1])), float(eps)
        where = {}
        for bi, b in enumerate(reducer.buckets):
            off = 0
            for p in b["params"]:
                where[id(p)] = (bi, off)
                off += p.numel()
        self.device = self.params[0].device
        for i, p in enumerate(self.params):
            if id(p) not in where:
                raise ValueError(f"ClipAdam: parameter {i} is not in the GradientReducer (requires_grad is "
                                 f"{p.requires_grad})")
            if p.dtype != torch.float32 or p.device != self.device or not p.is_contiguous():
                raise ValueError(f"ClipAdam: parameter {i} must be a contiguous float32 tensor on {self.device}")
        self._where = [where[id(p)] for p in self.params]
        self._exp_avg = [torch.zeros_like(b["flat"]) for b in reducer.buckets]
        self._exp_avg_sq = [torch.zeros_like(b["flat"]) for b in reducer.buckets]
        self.step_counter = torch.zeros((), dtype=torch.int64, device=self.device)
        self.grad_norm = torch.zeros((), dtype=torch.float32, device=self.device)
        self.steps = 0                       # host mirror of step_counter: one per step() call
        self.table = None                    # the device segment table [n, 6] int64, built by the first step()
        self.n_chunks = 0

    # ---- state -----------------------------------------------------------------------------------------------
    def moments(self, i: int) -> tuple[torch.Tensor, torch.Tensor]:
        """Parameter i's exp_avg and exp_avg_sq: views of the flat moment buffers, shaped like the parameter."""
        (bi, off), p = self._where[i], self.params[i]
        return (self._exp_avg[bi][off:off + p.numel()].view_as(p), self._exp_avg_sq[bi][off:off + p.numel()].view_as(p))

    def lr(self) -> float:
        """The learning rate of the next step, from the host mirror of the step (no device read)."""
        return self.base_lr * warm_up_factor(self.steps, self.warm_up_steps)

    def state_dict(self) -> dict:
        """torch.optim.Adam's layout; `lr` is the scheduled value and `initial_lr` the base one, as a LinearLR-driven
        Adam saves them.  Reads the device counter (a synchronisation: checkpoint time only)."""
        steps = int(self.step_counter.item())
        state = {}
        for i in range(len(self.params)):
            m, v = self.moments(i)
            state[i] = {"step": torch.tensor(float(steps)), "exp_avg": m.detach().clone(),
                        "exp_avg_sq": v.detach().clone()}
        group = {"lr": self.base_lr * warm_up_factor(steps, self.warm_up_steps), "betas": self.betas, "eps": self.eps,
                 "weight_decay": 0, "amsgrad": False, "maximize": False, "foreach": None, "capturable": False,
                 "differentiable": False, "fused": None, "decoupled_weight_decay": False, "initial_lr": self.base_lr,
                 "params": list(range(len(self.params)))}
        return {"state": state, "param_groups": [group]}

    def scheduler_state_dict(self) -> dict:
        """The `LinearLR` state a Lightning checkpoint keeps in `lr_schedulers[0]` at this step."""
        steps = int(self.step_counter.item())
        return {"start_factor": 1.0 / max(self.warm_up_steps, 1), "end_factor": 1.0,
                "total_iters": self.warm_up_steps, "base_lrs": [self.base_lr], "last_epoch": steps,
                "_step_count": steps + 1, "_get_lr_called_within_step": False,
                "_last_lr": [self.base_lr * warm_up_factor(steps, self.warm_up_steps)]}

    def load_state_dict(self, sd: dict) -> None:
        """Takes moments and the step from a torch.optim.Adam state (or `optimizer_states[0]` of a Lightning
        checkpoint) and the base learning rate, betas and eps from its single parameter group.  Parameters without
        an entry (torch keeps none for a parameter that never had a gradient) get zero moments."""
        groups = sd["param_groups"]
        if len(groups) != 1 or len(groups[0]["params"]) != len(self.params):
            raise ValueError(f"ClipAdam: expected one parameter group of {len(self.params)} parameters")
        g = groups[0]
        if g.get("weight_decay", 0) or g.get("amsgrad", False) or g.get("maximize", False):
            raise ValueError("ClipAdam: weight decay, amsgrad and maximize are not supported")
        steps = {int(e["step"]) for e in sd["state"].values()}
        if len(steps) > 1:
            raise ValueError(f"ClipAdam: the state's entries carry different steps ({sorted(steps)[:4]}...); one "
                             "global step counter cannot represent it")
        order = {pid: i for i, pid in enumerate(g["params"])}
        for b in (*self._exp_avg, *self._exp_avg_sq):
            b.zero_()
        for pid, e in sd["state"].items():
            m, v = self.moments(order[pid])
            m.copy_(e["exp_avg"])
            v.copy_(e["exp_avg_sq"])
        self.base_lr = float(g.get("initial_lr", g["lr"]))
        self.betas, self.eps = (float(g["betas"][0]), float(g["betas"][1])), float(g["eps"])
        self.steps = steps.pop() if steps else 0
        self.step_counter.fill_(self.steps)
        self.table = None                   # the descriptor carries lr, betas and eps

    # ---- the step ---------------------------------------------------------------------------------------------
    def _build(self) -> None:
        if self.device.type != "cuda":
            raise RuntimeError("ClipAdam.step: the parameters are not on a CUDA device; there is no CPU path")
        rows = []
        for i, p in enumerate(self.params):
            (bi, off), (m, v) = self._where[i], self.moments(i)
            flat = self.reducer.buckets[bi]["flat"]
            want = flat.data_ptr() + off * flat.element_size()
            if p.grad is None or p.grad.data_ptr() != want:
                raise RuntimeError(f"ClipAdam.step: parameter {i}'s .grad is not its GradientReducer bucket view "
                                   "(call reducer.zero_grad() at the start of the step)")
            rows.append((p.data_ptr(), want, m.data_ptr(), v.data_ptr(), p.numel()))
        table, chunks = segment_table(rows)
        if not len(table):
            raise RuntimeError("ClipAdam.step: every parameter is empty")
        self.n_chunks = chunks
        self._desc = _lib.ClipAdamDesc(n_segments=len(table), reserved=0, n_chunks=chunks,
                                       warm_up_steps=self.warm_up_steps, lr=self.base_lr, beta1=self.betas[0],
                                       beta2=self.betas[1], eps=self.eps, max_norm=self.max_norm)
        nbytes = ctypes.c_size_t()
        _lib.check(_lib.lib.ps_clip_adam_workspace_bytes(ctypes.byref(self._desc), ctypes.byref(nbytes)),
                   "ps_clip_adam_workspace_bytes")
        self._workspace = torch.zeros(nbytes.value, dtype=torch.uint8, device=self.device)
        self.table = torch.from_numpy(table).to(self.device)
        self._state = _lib.ClipAdamState(self.step_counter.data_ptr(), self.grad_norm.data_ptr())

    def step(self) -> None:
        """One optimiser step on the current stream.  The segment table is built on the first call: parameters,
        bucket views and moments must stay where they are afterwards (`reducer.zero_grad()` re-attaches a replaced
        `.grad`)."""
        if self.table is None:
            self._build()
        _lib.check(_lib.on_device(self.device, _lib.lib.ps_clip_adam_step, ctypes.byref(self._desc),
                                  self.table.data_ptr(), ctypes.byref(self._state), self._workspace.data_ptr(),
                                  self._workspace.numel(), torch.cuda.current_stream(self.device).cuda_stream),
                   "ps_clip_adam_step")
        self.steps += 1
