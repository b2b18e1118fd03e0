#!/usr/bin/env python
"""The cost of SyncBatchNorm in the fused operators: one LocalAggregation training step with plain BatchNorm against
the same step after nn.SyncBatchNorm.convert_sync_batchnorm, per family, at the per-GPU shapes of BASELINE c3 and c4.

    torchrun --nproc-per-node 2 tools/bench_syncbn.py [--rounds 7] [--steps 20]

One process per GPU, NCCL.  Every rank holds the per-GPU shard of the config (c3: 8 clouds of 15000 points, c4: 4 of
10000).  Per family and shape: `rounds` alternations of plain / sync, each `steps` steps between two CUDA events
after a barrier and a warm-up -> ms per step on rank 0, median [min..max] over the rounds.  Prints the card's name
and power limit, then one JSON line per (family, shape).  The synchronised arm adds two all_gathers of a few KB per
fused BatchNorm and step (forward statistics, backward sums).

With fewer than two GPUs, or outside torchrun, nothing is timed: two ranks sharing one GPU over gloo would time gloo's
host round trips, not the exchange a multi-GPU run pays, so the script only reports that the cost was not measured.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from closerlook3d_b200 import pt_utils, synth  # noqa: E402
from closerlook3d_b200.config import baseline_config, la_config  # noqa: E402

FAMILIES = {
    "pospool-xyz-avg": ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="avg"))),
    "pospool-sincos-avg": ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="avg"))),
    "adaptive_weight": ("adaptive_weight", dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1,
                                                                     reduction="avg"))),
    "pseudo_grid": ("pseudo_grid", dict()),
    "pointwisemlp": ("pointwisemlp", dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))),
}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(step, steps):
    import torch.distributed as dist
    dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--configs", default="3,4")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    ngpu = torch.cuda.device_count()
    if world < 2 or ngpu < 2:
        print(json.dumps({"card": card() if ngpu else "no CUDA device", "gpus": ngpu, "world_size": world,
                          "result": "multi-rank SyncBatchNorm cost not measured: it needs torchrun over two or more "
                                    "GPUs (NCCL, one rank per GPU)"}), flush=True)
        return
    import torch.distributed as dist
    rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    if rank == 0:
        print(json.dumps({"card": card(), "world_size": world, "rounds": args.rounds, "steps": args.steps}), flush=True)
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    for i in (int(c) for c in args.configs.split(",")):
        t = baseline_config(i)
        B = max(1, t["B"] // t["gpus"])
        N, K, C = t["N"], t["K"], t["C"]
        d = {k: v.to(dev) for k, v in synth.make_cloud_batch(B, N, C, 1000 + i, b_offset=rank * B).items()}
        gout = torch.randn(B, C, N, device=dev, generator=torch.Generator(device=dev).manual_seed(rank))
        for fam, (la, over) in FAMILIES.items():
            torch.manual_seed(0)
            plain = LocalAggregation(C, C, synth.ball_radius(N, K), K, la_config(la, **over)).to(dev).train()
            arms = {"plain": plain, "sync": torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))}

            def step_of(mod):
                def step():
                    pt_utils.clear_neighbor_cache()   # every step searches, as a training step on a new batch does
                    f = d["features"].requires_grad_(True)
                    mod(d["xyz"], d["xyz"], d["mask"], d["mask"], f).backward(gout)
                    f.grad = None
                return step

            steps = {k: step_of(m) for k, m in arms.items()}
            for s in steps.values():
                timed(s, 3)
            ms = {k: [] for k in steps}
            for r in range(args.rounds):
                order = ("plain", "sync") if r % 2 == 0 else ("sync", "plain")
                for k in order:
                    ms[k].append(timed(steps[k], args.steps))
            if rank == 0:
                res = {k: f"{statistics.median(v):.3f} [{min(v):.3f}..{max(v):.3f}]" for k, v in ms.items()}
                print(json.dumps({"config": f"c{i}", "family": fam, "per_gpu": dict(B=B, N=N, K=K, C=C),
                                  "ms_per_step": res,
                                  "sync_minus_plain_median_ms": round(statistics.median(ms["sync"]) -
                                                                      statistics.median(ms["plain"]), 4)}), flush=True)
            del arms, steps
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
