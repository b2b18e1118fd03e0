#!/usr/bin/env python
"""Whole-model data-parallel training steps on synthetic clouds (SURVEY.md section 8 row (f)4).

    python tools/train_synth.py --task classification --la pseudo_grid --batch 16 --points 10000
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29533 \
        tools/train_synth.py --task scene_segmentation --la pospool_sincos --batch 8 --points 15000
    python tools/train_synth.py --task multi_part_segmentation --dataset shapenetpart --la pseudo_grid
    python tools/train_synth.py --task scene_segmentation --la pseudo_grid --amp bf16
    python tools/train_synth.py --task classification --deterministic --no-dropout --batch 2 --points 3000 --steps 3 --warmup 0

The reference's training step (function/train_modelnet_dist.py:254-297, train_s3dis_dist.py): forward, loss,
zero_grad, backward, SGD step, under DistributedDataParallel(broadcast_buffers=False) (:206); part segmentation as function/train_partnet_dist.py:274-282 (multi-shape
cross entropy on the list of per-shape logits, seeded shape and part labels) -- with this package's
networks (closerlook3d_b200/backbone.py: the reference's module tree on the fused neighbourhood operators).
Synthetic data (no datasets in the container): points on noisy unit-sphere shells (surface-like density, so the
shipped cfgs' radii see realistic neighbour counts), xyz (+1) as input features as the datasets provide them.
--amp bf16 | fp16 runs forward and loss under torch.autocast (fp16 with a torch.amp.GradScaler); the fused operators
take the 16-bit features autocast hands them and compute in fp32 inside.
--deterministic sets CUBLAS_WORKSPACE_CONFIG=:4096:8 before CUDA initialises and turns torch.use_deterministic_algorithms
on, so two runs from the same state give the same bits; the JSON line then carries every step's loss and a SHA-256 of
the final parameters and buffers to compare runs by.
Prints one JSON line: whole-model points/s (device time, max over ranks) and a reference-format checkpoint round trip.
"""
import argparse
import io
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

LA = {
    "pospool_xyz": ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="avg"))),
    "pospool_sincos": ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="avg"))),
    "adaptive_weight": ("adaptive_weight", dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1,
                                                                     reduction="avg"))),
    "pointwisemlp": ("pointwisemlp", dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))),
    "pseudo_grid": ("pseudo_grid", dict()),
}


def synth_batch(B, N, cin, seed, device, scale):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(B, N, 3, generator=g)
    xyz = d / d.norm(dim=-1, keepdim=True) * (0.5 + 0.02 * torch.randn(B, N, 1, generator=g)) * scale
    feats = torch.cat([torch.ones(B, 1, N), xyz.transpose(1, 2)], 1)[:, :cin] if cin == 4 else xyz.transpose(1, 2)
    mask = torch.ones(B, N, dtype=torch.int32)
    return xyz.contiguous().to(device), mask.to(device), feats.contiguous().to(device)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", default="classification", choices=["classification", "scene_segmentation",
                                                                     "multi_part_segmentation"])
    ap.add_argument("--dataset", default="partnet", choices=["partnet", "shapenetpart"],
                    help="multi_part_segmentation: the PartNet or ShapeNetPart settings")
    ap.add_argument("--la", default="pseudo_grid", choices=sorted(LA))
    ap.add_argument("--batch", type=int, default=None, help="clouds per GPU (default: the cfg's batch_size)")
    ap.add_argument("--points", type=int, default=None, help="points per cloud (default: the cfg's num_points)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ddp", action="store_true",
                    help="torch DistributedDataParallel (the reference's wrapper) instead of this package's flat "
                         "gradient buffer + one all-reduce per step (closerlook3d_b200/dist.py)")
    ap.add_argument("--amp", default="off", choices=["off", "bf16", "fp16"],
                    help="mixed precision: forward and loss under torch.autocast in this dtype (fp16 adds a GradScaler)")
    ap.add_argument("--deterministic", action="store_true",
                    help="torch.use_deterministic_algorithms(True) with CUBLAS_WORKSPACE_CONFIG=:4096:8: repeatable bits")
    ap.add_argument("--no-dropout", action="store_true", help="set every Dropout's p to 0")
    args = ap.parse_args()
    if args.deterministic:
        os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"   # read when cuBLAS initialises: before any CUDA work
        torch.use_deterministic_algorithms(True)
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    import torch.distributed as dist
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=device)
    from closerlook3d_b200 import backbone as bb, pt_utils
    la, over = LA[args.la]
    part = args.task == "multi_part_segmentation"
    cfg = bb.model_config(args.task, la, **over, **(dict(dataset=args.dataset) if part else {}))
    B = args.batch or (cfg.batch_size if part else (16 if args.task == "classification" else 8))
    N = args.points or cfg.num_points
    scale = 2.0 if args.task == "scene_segmentation" else 1.0      # S3DIS spheres: in_radius 2 m
    build = {"classification": bb.build_classification, "scene_segmentation": bb.build_scene_segmentation,
             "multi_part_segmentation": bb.build_multi_part_segmentation}[args.task]
    torch.manual_seed(0)
    if args.deterministic:   # the same start: kernel-point dispositions draw from numpy's global generator
        import numpy as np
        np.random.seed(0)
    model, criterion = build(cfg)
    model.init_weights()
    model = model.to(device).train()
    if args.no_dropout:
        for m in model.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
    opt = torch.optim.SGD(model.parameters(), lr=B * world / 16 * 0.002, momentum=0.98, weight_decay=0.001)
    net, flat = model, None
    if world > 1 and args.ddp:
        net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local_rank], broadcast_buffers=False)
    elif world > 1:
        from closerlook3d_b200.dist import FlatGradients
        for p in model.parameters():            # same start on every rank, as DDP's constructor does
            dist.broadcast(p.data, 0)
        flat = FlatGradients(model.parameters()).attach()
    batches = [synth_batch(B, N, cfg.input_features_dim, 100 * rank + i, device, scale) for i in range(3)]
    if args.task == "classification":
        targets = [torch.randint(0, cfg.num_classes, (B,), device=device) for _ in batches]
    elif part:
        from closerlook3d_b200 import synth
        labs = [synth.make_part_labels(B, N, cfg.num_parts, 100 * rank + i) for i in range(len(batches))]
        targets = [(lab["points_labels"].to(device), lab["shape_labels"].to(device)) for lab in labs]
    else:
        targets = [torch.randint(0, cfg.num_classes, (B, N), device=device) for _ in batches]

    amp_dtype = {"off": None, "bf16": torch.bfloat16, "fp16": torch.float16}[args.amp]
    scaler = torch.amp.GradScaler("cuda") if args.amp == "fp16" else None

    def step(i):
        xyz, mask, feats = batches[i % len(batches)]
        with torch.autocast("cuda", dtype=amp_dtype or torch.float32, enabled=amp_dtype is not None):
            pred = net(xyz, mask, feats)
            if args.task == "classification":
                loss = criterion(pred, targets[i % len(batches)])
            elif part:
                loss = criterion(pred, *targets[i % len(batches)])
            else:
                loss = criterion(pred, targets[i % len(batches)], mask.float())
        scaled = scaler.scale(loss) if scaler is not None else loss
        if flat is not None:
            flat.zero()                 # the gradients are views of one buffer: one memset, one all-reduce
            scaled.backward()
            flat.allreduce()
        else:
            opt.zero_grad(set_to_none=True)
            scaled.backward()
        if scaler is not None:
            scaler.step(opt)
            scaler.update()
        else:
            opt.step()
        return loss

    losses = []
    for i in range(args.warmup):
        losses.append(step(i).detach())
    pt_utils.cache_stats.update(hit=0, miss=0)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(device)
    if world > 1:
        dist.barrier()
    # one event per step boundary: mean AND median (a one-off stall -- allocator growth, a late NCCL channel set-up,
    # python GC -- moved the 10-step mean of an 8-GPU run by 2x); every statistic is the max over ranks
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    evs[0].record()
    for i in range(args.steps):
        loss = step(args.warmup + i)
        losses.append(loss.detach())
        evs[i + 1].record()
    torch.cuda.synchronize()
    per = sorted(evs[i].elapsed_time(evs[i + 1]) for i in range(args.steps))
    ms = torch.tensor([evs[0].elapsed_time(evs[-1]) / args.steps, per[len(per) // 2], per[-1]], device=device,
                      dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms_mean, ms_median, ms_worst = (float(v) for v in ms.tolist())
    peak_mb = torch.cuda.max_memory_allocated(device) / 2**20
    # checkpoint round trip in the reference's format (train_modelnet_dist.py:152-160: {'model': state_dict, ...})
    ok = None
    if rank == 0:
        buf = io.BytesIO()
        torch.save({"model": model.state_dict(), "optimizer": opt.state_dict(), "epoch": 1}, buf)
        buf.seek(0)
        ck = torch.load(buf, map_location="cpu")
        fresh = build(cfg)[0]
        fresh.load_state_dict(ck["model"], strict=True)
        ok = all(torch.equal(a.cpu(), b) for a, b in zip(model.state_dict().values(), fresh.state_dict().values()))
        import hashlib
        digest = hashlib.sha256()
        for k, v in model.state_dict().items():
            digest.update(k.encode())
            digest.update(v.detach().cpu().contiguous().reshape(-1).view(torch.uint8).numpy().tobytes())
        print(json.dumps({"what": "whole-model training step (fwd + loss + bwd + SGD), synthetic clouds",
                          "task": args.task, **({"dataset": args.dataset} if part else {}), "local_aggregation": args.la,
                          "amp": args.amp, "n_gpus": world, "clouds_per_gpu": B,
                          "points_per_cloud": N, "steps": args.steps, "ms_per_step": ms_mean,
                          "ms_per_step_median": ms_median, "ms_slowest_step": ms_worst,
                          "max_memory_allocated_MB": peak_mb,
                          "points_per_s": B * N * world / (ms_mean * 1e-3),
                          "points_per_s_median_step": B * N * world / (ms_median * 1e-3), "loss": float(loss.item()),
                          "neighbour_cache_per_step": {k: v / args.steps for k, v in pt_utils.cache_stats.items()},
                          "params_M": sum(p.numel() for p in model.parameters()) / 1e6,
                          "checkpoint_round_trip": ok, "deterministic": args.deterministic,
                          "losses": [float(v) for v in torch.stack(losses).float().cpu()],
                          "state_sha256": digest.hexdigest(), "launch": "eager (no CUDA graph); " + ("DDP broadcast_buffers=False" if args.ddp or world == 1 else
                                                                   "flat gradient buffer, one all-reduce per step")}))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
