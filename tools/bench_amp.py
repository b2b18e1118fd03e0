#!/usr/bin/env python
"""Mixed precision at the layout boundary: one LocalAggregation training step (forward + backward) per arm,
alternated, CUDA events per step and per libcl3d entry point.

    python tools/bench_amp.py [--configs 3 5] [--steps 30] [--rounds 5]

Arms: fp32 (features float32); bf16 (bfloat16 features through the entry points' dtype arguments); B (the fp32
operator behind explicit .float() / .to(bfloat16) conversions: what a caller without native 16-bit support would run).
c3 = PseudoGrid linear, B 8, N 15000, K 26, C 72; c5 = PosPool sin_cos avg, B 8 (one GPU's shard), N 40000, K 40,
C 144 (BASELINE.md).  Prints one JSON line per (config, arm): ms per step, median [min..max] over the rounds, and
the median ms per entry point; then the card, its power limit and SM clock.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

CONFIGS = {
    3: ("pseudo_grid", dict(), 8, 15000, 26, 72),
    5: ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="avg")), 8, 40000, 40, 144),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[3, 5])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    from closerlook3d_b200 import _lib, synth
    from closerlook3d_b200.config import la_config
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    dev = torch.device("cuda:0")
    for c in args.configs:
        la, over, B, N, K, C = CONFIGS[c]
        torch.manual_seed(0)
        d = synth.make_cloud_batch(B, N, C, 1)
        xyz, mask = d["xyz"].to(dev), d["mask"].to(dev)
        mod = LocalAggregation(C, C, synth.ball_radius(N, K), K, la_config(la, **over)).to(dev).train()
        f32 = d["features"].to(dev)
        g32 = torch.randn(B, C, N, device=dev)
        arms = {
            "fp32": (lambda f: mod(xyz, xyz, mask, mask, f), f32, g32),
            "bf16": (lambda f: mod(xyz, xyz, mask, mask, f), f32.bfloat16(), g32.bfloat16()),
            "B": (lambda f: mod(xyz, xyz, mask, mask, f.float()).to(f.dtype), f32.bfloat16(), g32.bfloat16()),
        }

        def step(arm):
            fn, f, g = arms[arm]
            f = f.detach().requires_grad_(True)
            fn(f).backward(g)

        for arm in arms:                      # warm every shape and allocation
            for _ in range(3):
                step(arm)
        res = {a: [] for a in arms}
        per_ep = {a: {} for a in arms}
        for _ in range(args.rounds):
            for arm in arms:                  # alternated within every round
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(args.steps):
                    step(arm)
                e1.record()
                torch.cuda.synchronize()
                res[arm].append(e0.elapsed_time(e1) / args.steps)
        for arm in arms:                      # per entry point in a separate pass (events around every call)
            _lib.profiler.start()
            for _ in range(args.steps):
                step(arm)
            for name, (calls, ms) in _lib.profiler.stop().items():
                per_ep[arm][name] = round(ms / args.steps, 4)
        for arm, v in res.items():
            v = sorted(v)
            print(json.dumps({"config": f"c{c}", "arm": arm, "B": B, "N": N, "K": K, "C": C,
                              "ms_per_step_median": v[len(v) // 2], "ms_min": v[0], "ms_max": v[-1],
                              "ms_per_step_per_entry_point": per_ep[arm]}), flush=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": q}))


if __name__ == "__main__":
    main()
