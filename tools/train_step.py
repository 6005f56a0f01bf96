#!/usr/bin/env python
"""A bare training-step harness for BASELINE configs[2] / configs[3]: the full hot path inside one
optimisation step, data-parallel over GPUs.

    features [B, 2, 128, 256, 256]  (synthetic stand-in for the out-of-scope DINO/ResNet backbone)
      -> EpipolarTransformer                       (hot path, rows a8-a15; trainable)
      -> EncoderEpipolarTail                       (row f-1: high-res skip, depth predictor, to_gaussians,
                                                    fused GaussianAdapter kernel; trainable)
      -> DecoderSplattingCUDA, 4 target views/scene (hot path, rows a1-a7; V cameras share Gaussians)
      -> MSE -> backward, with the bucketed NCCL gradient all-reduce issued from backward hooks as buckets
         complete (pixelsplat_b200.parallel.GradientReducer: gradients live in flat buckets, no cat / copy-back)
      -> clip 0.5 -> Adam

--graph captures the WHOLE step (forward, backward, collectives, clip, Adam) into one CUDA graph after an eager
warm-up and replays it: the step is ~600 small kernels, and with 8 processes per node the Python launch path,
not the GPU, is what weak scaling loses to; a replayed graph has no launch path.

Replaces, for measurement purposes only, the reference's Lightning loop
(/root/reference/src/main.py:89-134, model_wrapper.py:108-151).  One process per GPU:

    python tools/train_step.py --batch 7
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tools/train_step.py --batch 7

Prints one JSON line from rank 0 (scenes/s and views/s over all ranks, per-phase milliseconds).
"""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=7, help="scenes per GPU (README.md:87: batch is per GPU)")
    ap.add_argument("--target-views", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--hw", type=int, default=256)
    ap.add_argument("--graph", action="store_true", help="capture the whole step in one CUDA graph and replay it")
    ap.add_argument("--bucket-mb", type=float, default=8.0)
    ap.add_argument("--legacy-allreduce", action="store_true", help="round-1 path: all-reduce after backward (A/B)")
    ap.add_argument("--unfused-loss", action="store_true", help="render an image, then torch MSE (A/B of the loss epilogue)")
    ap.add_argument("--depth-loss", action="store_true",
                    help="add LossDepth (re10k_depth_loss: weight 0.25, sigma 12, second derivative) on the fused depth")
    ap.add_argument("--two-pass-depth", action="store_true",
                    help="with --depth-loss: render the depth as a second pass (render_depth) instead (A/B)")
    ap.add_argument("--deterministic", action="store_true",
                    help="torch.use_deterministic_algorithms(True): fixed-order encoder and rasterizer gradients")
    args = ap.parse_args()
    if args.deterministic:                         # cuBLAS needs its workspace setting before its first call
        import os
        os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
        torch.use_deterministic_algorithms(True)
    from pixelsplat_b200 import parallel, synthetic
    from pixelsplat_b200.decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg
    from pixelsplat_b200.encoder import EpipolarTransformer, EpipolarTransformerCfg, ImageSelfAttentionCfg
    from pixelsplat_b200.encoder.encoder_tail import EncoderEpipolarTail, EncoderTailCfg
    from pixelsplat_b200.loss import LossDepth, LossDepthCfg, LossDepthCfgWrapper, mse_from_sse
    rank, world, local = parallel.init_distributed()
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    torch.manual_seed(0)                     # identical initial parameters on every rank
    cfg = EpipolarTransformerCfg(ImageSelfAttentionCfg(4, 10, 2, 4, 128, 128, 256), 10, 2, 4, 32, 128, 256, 4)
    enc = EpipolarTransformer(cfg, 128, num_context_views=2).to(dev)
    head = EncoderEpipolarTail(EncoderTailCfg()).to(dev)
    dec = DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"),
                               type("D", (), {"background_color": [0.0, 0.0, 0.0]})()).to(dev)
    params = list(enc.parameters()) + list(head.parameters())
    reducer = None if args.legacy_allreduce else parallel.GradientReducer(params, int(args.bucket_mb * 2 ** 20))
    opt = torch.optim.Adam(params, lr=1.5e-4, capturable=args.graph)
    B, T, HW = args.batch, args.target_views, args.hw
    g = torch.Generator().manual_seed(1234 + rank)          # per-rank data (main.py:106)
    feats = torch.randn(B, 2, 128, HW, HW, generator=g).to(dev)
    images = torch.rand(B, 2, 3, HW, HW, generator=g).to(dev)
    ctx_e = torch.eye(4).repeat(B, 2, 1, 1); ctx_e[:, 1, 0, 3] = 1.0
    ctx_k = synthetic.intrinsics_re10k(2)[None].repeat(B, 1, 1, 1)
    near_v, far_v = synthetic.bounds_from_baseline(1.0, HW, HW, 3.0 * HW, 0.5)
    tgt_e = torch.stack([synthetic.target_cameras(T, seed=rank * 100 + s) for s in range(B)])
    tgt_k = synthetic.intrinsics_re10k(T)[None].repeat(B, 1, 1, 1)
    target = torch.rand(B, T, 3, HW, HW, generator=g).to(dev)
    ctx_e, ctx_k, tgt_e, tgt_k = ctx_e.to(dev), ctx_k.to(dev), tgt_e.to(dev), tgt_k.to(dev)
    near_c, far_c = torch.full((B, 2), near_v, device=dev), torch.full((B, 2), far_v, device=dev)
    near_t, far_t = torch.full((B, T), near_v, device=dev), torch.full((B, T), far_v, device=dev)

    context = dict(image=images, extrinsics=ctx_e, intrinsics=ctx_k, near=near_c, far=far_c)
    loss_depth = LossDepth(LossDepthCfgWrapper(LossDepthCfg(0.25, 12.0, True)))
    depth_batch = {"target": {"near": near_t, "far": far_t, "image": target}}
    phases = ["encoder", "head", "render", "backward", "allreduce", "optimizer"]
    acc = {p: 0.0 for p in phases}

    timeline = []                                  # per timed step: the phase-boundary events (read at the end)

    def step(timed, record=True):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(phases) + 1)] if record else None
        mark = (lambda i: ev[i].record()) if record else (lambda i: None)
        mark(0)
        if reducer is not None:
            reducer.zero_grad()
        else:
            opt.zero_grad(set_to_none=True)
        f, _ = enc(feats, ctx_e, ctx_k, near_c, far_c); mark(1)
        gs = head(f, context, global_step=0); mark(2)
        fused_depth = "depth" if args.depth_loss and not args.two_pass_depth else None
        if args.unfused_loss:
            out = dec(gs, tgt_e, tgt_k, near_t, far_t, (HW, HW), depth_mode=fused_depth)
            loss = (out.color - target).square().mean()
        else:   # LossMse from the compositor's epilogue: no image tensor, no dL/dC tensor (row f-4)
            out, sse, _ = dec.forward_mse(gs, tgt_e, tgt_k, near_t, far_t, (HW, HW), target, want_color=False,
                                          depth_mode=fused_depth)
            loss = mse_from_sse(sse, (HW, HW))
        if args.depth_loss:
            depth = out.depth if fused_depth else dec.render_depth(gs, tgt_e, tgt_k, near_t, far_t, (HW, HW))
            loss = loss + loss_depth(type("O", (), {"depth": depth})(), depth_batch)
        mark(3)
        loss.backward(); mark(4)
        if reducer is not None:
            reducer.finish()                       # only the tail that backward did not hide
        else:
            parallel.allreduce_gradients(params)
        mark(5)
        torch.nn.utils.clip_grad_norm_(params, 0.5)
        opt.step(); mark(6)
        if timed and record:
            timeline.append(ev)                    # no host synchronisation inside the timed loop
        return loss

    if args.graph:   # the captured step freezes the binning capacity: leave room for the Gaussians to move
        from pixelsplat_b200 import rasterizer
        rasterizer.set_capacity_headroom(2.5)
    for _ in range(args.warmup):
        step(False)
    torch.cuda.synchronize()
    launch = "eager python"
    run = lambda: step(True)
    if args.graph:
        try:
            rasterizer.set_capacity_check("deferred")
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    step(False, record=False)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                static_loss = step(False, record=False)
            run = lambda: (graph.replay(), static_loss)[1]
            launch = "one CUDA graph per step (forward + backward + all-reduce + clip + Adam), replayed"
            for _ in range(2):
                run()
            torch.cuda.synchronize()
        except Exception as exc:                   # report and keep measuring eagerly
            import traceback
            traceback.print_exc()
            launch = f"eager python (graph capture failed: {type(exc).__name__}: {str(exc)[:200]})"
            torch.cuda.synchronize()
    if world > 1:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.steps):
        loss = run()
    t1.record()
    torch.cuda.synchronize()
    for ev in timeline:
        for i, p in enumerate(phases):
            acc[p] += ev[i].elapsed_time(ev[i + 1])
    sec = parallel.max_over_ranks(t0.elapsed_time(t1) * 1e-3, dev)
    if rank == 0:
        print(json.dumps({
            "config": f"configs[{2 if world == 1 else 3}]: 2-view {HW}x{HW}, batch {B}/GPU, {T} target views, "
                      f"EpipolarTransformer + splat render training step, world {world}",
            "scenes_per_s": world * B * args.steps / sec, "views_per_s": world * B * T * args.steps / sec,
            "ms_per_step": 1e3 * sec / args.steps,
            "phase_ms": ({p: acc[p] / len(timeline) for p in phases} if timeline else None),
            "launch": launch, "loss_path": "torch MSE on the rendered image" if args.unfused_loss else "fused compositor epilogue",
            "depth_loss": None if not args.depth_loss else ("two-pass render_depth" if args.two_pass_depth
                                                            else "fused depth channel"),
            "allreduce": ("after backward, torch.cat buckets (round-1 path)" if reducer is None else
                          f"{len(reducer.buckets)} flat buckets of <= {args.bucket_mb} MB, issued from backward hooks "
                          "(overlapped); phase 'allreduce' is the exposed tail only"),
            "deterministic": args.deterministic,
            "peak_gib": torch.cuda.max_memory_allocated() / 2 ** 30, "loss": float(loss),
            "n_gpus": world, "data": "synthetic", "dtype": "f32"}))
    if world > 1:
        torch.distributed.barrier()
        torch.cuda.synchronize()
        if args.graph:
            # a captured graph holds NCCL work of this communicator; tearing the process group down underneath it
            # blocks (observed: destroy_process_group never returned).  The measurement is done: leave directly.
            sys.stdout.flush()
            sys.stderr.flush()
            import os
            os._exit(0)
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
