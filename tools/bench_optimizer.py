#!/usr/bin/env python
"""Times the optimiser end of a training step on the preset encoder (random initialisation, gradients of a realistic
scale in GradientReducer buckets):

    torch-foreach   clip_grad_norm_ + torch.optim.Adam(foreach=True)
    torch-fused     clip_grad_norm_ + torch.optim.Adam(fused=True)
    clip-adam       optim.ClipAdam (csrc/optimizer.cu)

each eagerly and inside a CUDA graph, in alternating rounds of one call, with CUDA events.  The torch arms run
capturable=True in both modes (a captured Adam needs it) and carry no LR schedule: LinearLR lives on the host and
cannot be replayed, which is part of why ClipAdam keeps the schedule on the device.  Before timing, the three arms
take one step from the same state and must agree on the parameters.

The algorithm needs 32 bytes per parameter (4 read for the norm; 16 read and 12 written for the update); the achieved
bytes/s over that figure is reported as a share of the H100 SXM data sheet's 3.35 TB/s.  The step is HBM-bound: it does
a handful of floating-point operations per 32 bytes.

Prints one JSON line.  Needs a GPU.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

BYTES_PER_PARAM = 32
HBM_PEAK = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=1.0, help="time filled by each arm's steps in each round")
    ap.add_argument("--grad-scale", type=float, default=1e-3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optimizer: no CUDA device; there is nothing to measure without one")
    from pixelsplat_b200.evaluation.presets import NUM_CONTEXT_VIEWS, encoder_cfg
    from pixelsplat_b200.encoder.encoder_epipolar import EncoderEpipolar
    from pixelsplat_b200.optim import ClipAdam, vectorised
    from pixelsplat_b200.parallel import GradientReducer
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)

    def make():
        torch.manual_seed(0)
        enc = EncoderEpipolar(encoder_cfg("re10k"), num_context_views=NUM_CONTEXT_VIEWS).to(dev)
        params = list(enc.parameters())
        reducer = GradientReducer(params)
        g = torch.Generator(device=dev).manual_seed(1)
        for b in reducer.buckets:
            b["flat"].copy_(args.grad_scale * torch.randn(b["flat"].shape, generator=g, device=dev))
        return params, reducer

    arms = {}
    for name in ("torch-foreach", "torch-fused", "clip-adam"):
        params, reducer = make()
        if name == "clip-adam":
            opt = ClipAdam(params, reducer, lr=1.5e-4, warm_up_steps=0, max_norm=0.5)
            step = opt.step
        else:
            opt = torch.optim.Adam(params, lr=1.5e-4, capturable=True, foreach=name == "torch-foreach",
                                   fused=name == "torch-fused")

            def step(opt=opt, params=params):
                torch.nn.utils.clip_grad_norm_(params, 0.5)
                opt.step()
        arms[name] = dict(params=params, reducer=reducer, opt=opt, step=step)

    # one step each from the same state: the arms must agree (clip_grad_norm_ rescales the torch arms' gradients in
    # place, so their buckets are refilled afterwards)
    for a in arms.values():
        a["step"]()
    torch.cuda.synchronize()
    ref = arms["torch-foreach"]["params"]
    agree = {}
    for name in ("torch-fused", "clip-adam"):
        num = sum(float((p - q).detach().double().norm()) ** 2 for p, q in zip(arms[name]["params"], ref)) ** 0.5
        den = 1.5e-4 * sum(p.numel() for p in ref) ** 0.5           # the norm of a step of lr in every element
        agree[name] = num / den
        assert agree[name] < 1e-3, f"{name} differs from torch-foreach by {agree[name]:.2e} of a step"
    n_params = sum(p.numel() for p in ref)
    n_tensors = len(ref)
    ca = arms["clip-adam"]["opt"]
    table = ca.table.cpu().numpy()
    vec_share = sum(int(r[4]) for r in table if vectorised(r)) / n_params

    def refill():
        for a in arms.values():
            g = torch.Generator(device=dev).manual_seed(1)
            for b in a["reducer"].buckets:
                b["flat"].copy_(args.grad_scale * torch.randn(b["flat"].shape, generator=g, device=dev))

    refill()
    graphs = {}
    for name, a in arms.items():
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                a["step"]()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            a["step"]()
        graphs[name] = g
    refill()

    def timed(fn, n):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(n):
            fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / n

    runs = {(name, mode): (arms[name]["step"] if mode == "eager" else graphs[name].replay)
            for name in arms for mode in ("eager", "graph")}
    counts = {}
    for key, fn in runs.items():                                   # warm-up and the step count that fills --seconds
        timed(fn, 10)
        counts[key] = max(10, int(args.seconds * 1e3 / timed(fn, 20)))
    times = {key: [] for key in runs}
    for _ in range(args.rounds):
        for key, fn in runs.items():
            times[key].append(timed(fn, counts[key]))
    med = {key: sorted(v)[len(v) // 2] for key, v in times.items()}

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    out = {"metric": "optimiser step of the re10k preset encoder: clip 0.5 + Adam, ms per step (median of rounds)",
           "card": smi or torch.cuda.get_device_name(0), "parameters": n_params, "tensors": n_tensors,
           "buckets": len(arms["clip-adam"]["reducer"].buckets), "chunks": ca.n_chunks,
           "float4_route_share_of_elements": vec_share, "rounds": args.rounds, "steps_per_round": {f"{k[0]}/{k[1]}": v for k, v in counts.items()},
           "ms": {f"{k[0]}/{k[1]}": v for k, v in med.items()},
           "ms_min_max": {f"{k[0]}/{k[1]}": [min(v), max(v)] for k, v in times.items()},
           "clip_adam_launches_per_step": ClipAdam.LAUNCHES_PER_STEP,
           "agreement_with_torch_foreach_in_steps_of_lr": agree,
           "bound": "HBM", "bytes_per_parameter": BYTES_PER_PARAM,
           "clip_adam_bytes_per_s": {m: BYTES_PER_PARAM * n_params / (med[("clip-adam", m)] * 1e-3)
                                     for m in ("eager", "graph")},
           "clip_adam_share_of_3.35TB/s": {m: BYTES_PER_PARAM * n_params / (med[("clip-adam", m)] * 1e-3) / HBM_PEAK
                                           for m in ("eager", "graph")}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
