"""Where the neighbour search's time goes, on one GPU.

    python tools/bench_search.py [--launches 100] [--rounds 5] [--trace-dir DIR]

Per shape (c3 B=8 N=15000 K=26, c4 B=4 N=10000 K=32, c5 B=8 N=40000 K=40; query set = support set, one tensor passed
as both, as every non-strided layer does), on a ring of clouds from synth.make_cloud_batch:
  * `cl3d_ball_query_csr` as the step issues it (counted slots), CUDA events around `launches` calls per round:
    both phases, the search phase alone (phases=1) and the list phase alone (phases=2);
  * the split of one call into its kernels (grid build, ranked ball query, csr_scan + csr_place) from the device
    durations a torch.profiler pass records for the same calls.
Then, at c3, one torch.profiler trace of 10 CUDA-graph replays of the `bench.py` step (the same LocalAggregation
module and GraphedStep as bench.py, neighbour cache off): per replay, how long the main stream sits idle between its
last kernel before the aggregation forward and that forward -- the search time the step does not hide.
Prints medians and min..max over the rounds; needs a GPU and prints the card, its power limit and maximum SM clock.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from closerlook3d_b200 import _lib, ops, synth  # noqa: E402

SHAPES = [("c3", 8, 15000, 26), ("c4", 4, 10000, 32), ("c5", 8, 40000, 40)]
KERNELS = {"grid build": ("grid_build_fused_kernel",), "ball query": ("ball_query_grid_kernel",),
           "csr_scan + csr_place": ("csr_scan_kernel", "csr_place_kernel")}


def fmt(xs, unit="ms", scale=1.0):
    xs = [x * scale for x in xs]
    return f"{statistics.median(xs):.4f} {unit} [{min(xs):.4f}..{max(xs):.4f}]"


def make_ring(dev, B, N, K, n=4):
    r = synth.ball_radius(N, K)
    ring = []
    for t in range(n):
        d = synth.make_cloud_batch(B, N, 1, 1003 + 7919 * t)
        xyz, mask = d["xyz"].to(dev), d["mask"].to(dev)
        L = _lib.lib()
        wsb = L.cl3d_ball_query_csr_workspace_bytes(B, N, N, K, 0)
        ring.append(dict(xyz=xyz, mask=mask, idx=torch.empty(B, N, K, dtype=torch.int32, device=dev),
                         ncount=torch.empty(B, N, dtype=torch.int32, device=dev),
                         off=torch.empty(B, N + 1, dtype=torch.int32, device=dev),
                         ent=torch.empty(B, N * K, dtype=torch.int32, device=dev),
                         ws=torch.empty(wsb, dtype=torch.uint8, device=dev), wsb=wsb))
    return ring, r


def call(b, B, N, K, r, phases):
    """cl3d_ball_query_csr exactly as ops.ball_query(csr="counted") issues it, without the allocations"""
    L = _lib.lib()
    p = _lib.ptr
    _lib.check(L.cl3d_ball_query_csr(p(b["xyz"]), p(b["xyz"]), p(b["mask"]), p(b["mask"]), B, N, N, float(r), K,
                                     p(b["idx"]), None, p(b["ncount"]), 0, p(b["off"]), p(b["ent"]), p(b["ws"]),
                                     b["wsb"], 0, phases, 0, _lib.stream_ptr()), "cl3d_ball_query_csr")


def timed(fn, ring, launches):
    """ms per call, CUDA events around `launches` back-to-back calls"""
    for i in range(5):
        fn(ring[i % len(ring)])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(launches):
        fn(ring[i % len(ring)])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def kernel_split(fn, ring, launches):
    """{kernel: device ms per call} from one torch.profiler pass over `launches` calls"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(launches):
            fn(ring[i % len(ring)])
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            tot[e.name] = tot.get(e.name, 0.0) + e.device_time_total / 1e3
    return {k: tot[k] / launches for k in tot}


def exposed_search(dev, trace_dir):
    """c3 step as bench.py builds it, 10 graph replays under torch.profiler -> per-replay idle time of the main stream
    before the aggregation forward (us), plus the search kernels' own durations (us)"""
    import numpy as np
    from torch.profiler import ProfilerActivity, profile
    from closerlook3d_b200 import pt_utils
    from closerlook3d_b200.config import baseline_config
    from closerlook3d_b200.graphed import GraphedStep
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    spec = baseline_config(3)
    pt_utils.cache_enabled = False
    pt_utils.clear_neighbor_cache()
    torch.manual_seed(2003)
    np.random.seed(2003)
    r = synth.ball_radius(spec["N"], spec["K"])
    mod = LocalAggregation(spec["C"], spec["C"], r, spec["K"], spec["cfg"]).to(dev).train()
    ring = [{k: v.to(dev) for k, v in synth.make_cloud_batch(spec["B"], spec["N"], spec["C"], 1003 + 7919 * t).items()}
            for t in range(4)]
    gout = torch.randn(spec["B"], spec["C"], spec["N"], device=dev, generator=torch.Generator(device=dev).manual_seed(5))
    gs = GraphedStep(mod, ring[0]["xyz"], ring[0]["mask"], ring[0]["features"], gout)
    for i in range(10):
        gs.load(ring[i % 4]["xyz"], ring[i % 4]["mask"], ring[i % 4]["features"])
        gs.replay()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        for i in range(10):
            gs.load(ring[i % 4]["xyz"], ring[i % 4]["mask"], ring[i % 4]["features"])
            gs.replay()
        torch.cuda.synchronize()
    os.makedirs(trace_dir, exist_ok=True)
    path = os.path.join(trace_dir, "c3_step.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    search = [e for e in ev if e["name"].startswith("void cl3d::ball_query_grid_kernel") or
              e["name"].startswith("cl3d::ball_query_grid_kernel") or "ball_query_grid_kernel" in e["name"]]
    build = [e for e in ev if "grid_build_fused_kernel" in e["name"]]
    side = search[0]["args"]["stream"] if search else None
    idle, fwd_names = [], set()
    for s in search:
        s_end = s["ts"] + s["dur"]
        main = [e for e in ev if e["args"]["stream"] != side]
        nxt = next((e for e in main if e["ts"] >= s_end - 1.0), None)   # first main-stream kernel after the search
        if nxt is None:
            continue
        before = [e["ts"] + e["dur"] for e in main if e["ts"] + e["dur"] <= nxt["ts"] and e["ts"] >= s["ts"] - 2000]
        if not before:
            continue
        idle.append(nxt["ts"] - max(before))
        fwd_names.add(nxt["name"][:60])
    return dict(idle_us=idle, search_us=[e["dur"] for e in search], build_us=[e["dur"] for e in build],
                first_after=sorted(fwd_names), trace=path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--trace-dir", default=os.path.join(tempfile.gettempdir(), "cl3d_bench_search"),
                    help="where the c3 step trace is written")
    ap.add_argument("--no-trace", action="store_true", help="skip the c3 step trace")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_search.py: no CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0), flush=True)
    for name, B, N, K in SHAPES:
        ring, r = make_ring(dev, B, N, K)
        t = {"both phases": [], "search (phase 1)": [], "lists (phase 2)": []}
        for _ in range(args.rounds):
            t["both phases"].append(timed(lambda b: call(b, B, N, K, r, 3), ring, args.launches))
            t["search (phase 1)"].append(timed(lambda b: call(b, B, N, K, r, 1), ring, args.launches))
            t["lists (phase 2)"].append(timed(lambda b: call(b, B, N, K, r, 2), ring, args.launches))
        for k, v in t.items():
            print(f"{name} B={B} N={N} K={K}: cl3d_ball_query_csr {k}: {fmt(v)}", flush=True)
        split = {k: [] for k in KERNELS}
        for _ in range(args.rounds):
            per = kernel_split(lambda b: call(b, B, N, K, r, 3), ring, args.launches)
            for k, names in KERNELS.items():
                split[k].append(sum(v for n, v in per.items() if any(x in n for x in names)))
        for k, v in split.items():
            print(f"{name} B={B} N={N} K={K}: kernel {k}: {fmt(v)}", flush=True)
        del ring
        torch.cuda.empty_cache()
    if not args.no_trace:
        x = exposed_search(dev, args.trace_dir)
        print(f"c3 step (graph replay): main-stream idle before the forward: {fmt(x['idle_us'], 'us')} "
              f"(next kernel: {', '.join(x['first_after'])})", flush=True)
        print(f"c3 step (graph replay): ball_query_grid_kernel {fmt(x['search_us'], 'us')}, grid_build_fused_kernel "
              f"{fmt(x['build_us'], 'us') if x['build_us'] else 'n/a'}; trace {x['trace']}", flush=True)


if __name__ == "__main__":
    main()
