"""Gradient clipping, LR warm-up and Adam in float64 numpy, written from their formulas (test infrastructure: the
reference point of csrc/optimizer.cu and of pixelsplat_b200.optim.ClipAdam).

    total = sqrt(sum_i ||g_i||^2)                         (the L2 norm of the per-tensor L2 norms)
    coef  = min(1, max_norm / (total + 1e-6))
    t     = steps taken so far + 1
    lr_t  = lr * warm_up_factor(t - 1, W)
    m     = beta1 m + (1 - beta1) coef g
    v     = beta2 v + (1 - beta2) (coef g)^2
    p    -= lr_t / (1 - beta1^t) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
"""
from __future__ import annotations

import numpy as np


def warm_up_factor(steps_taken: int, warm_up_steps: int) -> float:
    """LinearLR(start_factor=1 / W, end_factor=1, total_iters=W) after `steps_taken` scheduler steps, closed form."""
    if warm_up_steps <= 0:
        return 1.0
    start = 1.0 / warm_up_steps
    return start + (1.0 - start) * min(steps_taken, warm_up_steps) / warm_up_steps


def total_norm(grads) -> float:
    return float(np.sqrt(sum(float(np.sum(np.square(np.asarray(g, np.float64)))) for g in grads)))


class AdamOracle:
    """State in float64; `step(grads)` takes one optimiser step and returns the gradient norm before clipping."""

    def __init__(self, params, lr=1.5e-4, warm_up_steps=2000, max_norm=0.5, betas=(0.9, 0.999), eps=1e-8):
        self.params = [np.array(p, np.float64) for p in params]
        self.exp_avg = [np.zeros_like(p) for p in self.params]
        self.exp_avg_sq = [np.zeros_like(p) for p in self.params]
        self.lr, self.warm_up_steps, self.max_norm, self.betas, self.eps = lr, warm_up_steps, max_norm, betas, eps
        self.steps = 0

    def lr_now(self) -> float:
        return self.lr * warm_up_factor(self.steps, self.warm_up_steps)

    def step(self, grads) -> float:
        b1, b2 = self.betas
        norm = total_norm(grads)
        coef = min(1.0, self.max_norm / (norm + 1e-6)) if norm == norm else float("nan")
        lr_t = self.lr_now()
        self.steps += 1
        bc1, bc2 = 1.0 - b1 ** self.steps, 1.0 - b2 ** self.steps
        for p, g, m, v in zip(self.params, grads, self.exp_avg, self.exp_avg_sq):
            g = coef * np.asarray(g, np.float64)
            m *= b1
            m += (1.0 - b1) * g
            v *= b2
            v += (1.0 - b2) * g * g
            p -= (lr_t / bc1) * m / (np.sqrt(v) / np.sqrt(bc2) + self.eps)
        return norm
