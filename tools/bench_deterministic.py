#!/usr/bin/env python
"""Deterministic mode against the default: one LocalAggregation training step per BASELINE config c1-c5, arms
alternated in one process, and the entry points the mode changes timed on their own.

    python tools/bench_deterministic.py [--configs 1,2,3,4,5] [--rounds 5] [--steps 20]

Per config (one GPU's shard: B of c4 / c5 divided by their 8 GPUs, as bench.py does): `rounds` alternations of
default / deterministic, each `steps` steps between two CUDA events after a warm-up -> ms per step, median
[min..max] over the rounds.  Per entry point (`_lib.profiler`, a separate pass): the list build
(cl3d_ball_query_csr, cl3d_build_csr), cl3d_pwmlp_bwd, cl3d_gather_max_bwd and cl3d_group_points_grad, ms per step.
The max-pool and group-points gradients run in a MaskedMaxPool / GroupingOperation step at the config's shape.
Prints one JSON line per config plus the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from closerlook3d_b200 import _lib, pt_utils, synth  # noqa: E402
from closerlook3d_b200.config import baseline_config  # noqa: E402

CHANGED = ("cl3d_ball_query_csr", "cl3d_build_csr", "cl3d_pwmlp_bwd", "cl3d_gather_max_bwd", "cl3d_group_points_grad")


def make_steps(i, dev):
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    t = baseline_config(i)
    B = max(1, t["B"] // t["gpus"])
    d = {k: v.to(dev) for k, v in synth.make_cloud_batch(B, t["N"], t["C"], 1000 + i).items()}
    r = synth.ball_radius(t["N"], t["K"])
    torch.manual_seed(0)
    mod = LocalAggregation(t["C"], t["C"], r, t["K"], t["cfg"]).to(dev).train()
    gout = torch.randn(B, t["C"], t["N"], device=dev)
    pool = pt_utils.MaskedMaxPool(t["N"] // 4, r, t["K"], 2 * r)

    def la_step():
        pt_utils.clear_neighbor_cache()           # every step searches, as a training step on a new batch does
        f = d["features"].requires_grad_(True)
        out = mod(d["xyz"], d["xyz"], d["mask"], d["mask"], f)
        out.backward(gout)
        f.grad = None

    def pool_step():   # max-pool and grouping gradients: the modules that reach the two gathers
        pt_utils.clear_neighbor_cache()
        f = d["features"].requires_grad_(True)
        _, _, sub = pool(d["xyz"], d["mask"], f)
        sub.sum().backward()
        nl = pt_utils.neighbors(d["xyz"], d["xyz"], d["mask"], d["mask"], r, t["K"]).wait()
        pt_utils.grouping_operation(f, nl.idx[:, : t["N"] // 16].contiguous()).sum().backward()
        f.grad = None

    return t, B, la_step, pool_step


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="1,2,3,4,5")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic.py needs a CUDA device")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"card": card[0] if card else "unknown"}), flush=True)
    for i in (int(c) for c in args.configs.split(",")):
        t, B, la_step, pool_step = make_steps(i, dev)
        res = {}
        for name, fn in (("la_step", la_step), ("pool_grouping_step", pool_step)):
            arms = {False: [], True: []}
            for det in (False, True):             # warm-up of both arms
                torch.use_deterministic_algorithms(det)
                timed(fn, 3)
            for _ in range(args.rounds):
                for det in (False, True):
                    torch.use_deterministic_algorithms(det)
                    arms[det].append(timed(fn, args.steps))
            torch.use_deterministic_algorithms(False)
            res[name] = {("deterministic" if det else "default"): dict(median=statistics.median(v), min=min(v),
                                                                       max=max(v)) for det, v in arms.items()}
        entry = {}
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            _lib.profiler.start()
            for _ in range(args.steps):
                la_step()
                pool_step()
            prof = _lib.profiler.stop()
            entry["deterministic" if det else "default"] = {
                k: prof[k][1] / args.steps for k in CHANGED if k in prof}
        torch.use_deterministic_algorithms(False)
        print(json.dumps({"config": t["name"], "B": B, "N": t["N"], "K": t["K"], "C": t["C"], "ms": res,
                          "entry_points_ms_per_step": entry}), flush=True)


if __name__ == "__main__":
    main()
