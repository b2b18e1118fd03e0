#!/usr/bin/env python
"""cl3d_gather_max_bwd (the MaskedMaxPool backward, default mode) at the S3DIS width-144 max-pool shapes, B = 8.

    python tools/time_pool_bwd.py [--other path/to/another/libcl3d.so]

Each library's 50 launches per round are captured in a CUDA graph, so host overhead stays out of the timing; CUDA events
around each replay; with --other the rounds alternate between this tree's library and the other build (ABBA order), and
the medians of both are printed beside the GPU's name and power limit.  Both libraries get the
same inputs; their gradients are compared (fp32 atomics in a different order may move the last bits)."""
import argparse
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from closerlook3d_b200 import _lib, ops, pt_utils, synth  # noqa: E402
from closerlook3d_b200._lib import ptr, stream_ptr  # noqa: E402

# (C, N, M, K): backbone.model_config("scene_segmentation") strided blocks at width 144
SHAPES = [(144, 15000, 4096, 26), (288, 4096, 1152, 31), (576, 1152, 304, 38), (1152, 304, 88, 41)]
B, ROUNDS, LAUNCHES = 8, 10, 50


def load(path):
    fn = ctypes.CDLL(os.path.abspath(path)).cl3d_gather_max_bwd
    fn.restype, fn.argtypes = _lib.SIGNATURES["cl3d_gather_max_bwd"]
    return fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", default=None, help="another build's libcl3d.so to alternate with")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    libs = {"this": load(_lib.SO_PATH)}
    if args.other:
        libs["other"] = load(args.other)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {torch.cuda.get_device_name(dev)} ({smi}); B={B}, {ROUNDS} rounds x {LAUNCHES} launches")
    for C, N, M, K in SHAPES:
        d = synth.make_cloud_batch(B, N, C, 100 + C)
        r = synth.ball_radius(N, K)
        xyz, mask = d["xyz"].to(dev), d["mask"].to(dev)
        q = xyz[:, :M].contiguous()
        qm = torch.ones(B, M, dtype=torch.int32, device=dev)
        idx = pt_utils.neighbors(q, xyz, qm, mask, r, K).wait().idx
        _, arg = ops.gather_max(d["features"].to(dev), idx)
        gout = torch.randn(B, C, M, device=dev)
        Cp = ops.padded_channels(C)
        out = {n: torch.empty(B, N, Cp, device=dev) for n in libs}

        def launch(n):
            _lib.check(libs[n](ptr(gout), 0, ptr(idx), ptr(arg), B, N, M, K, C, None, None, ptr(out[n]), stream_ptr()),
                       "cl3d_gather_max_bwd")

        times = {n: [] for n in libs}
        graphs = {}
        for n in libs:
            for _ in range(5):
                launch(n)
            torch.cuda.synchronize()
            graphs[n] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[n]):
                for _ in range(LAUNCHES):
                    launch(n)
            graphs[n].replay()
        for rnd in range(ROUNDS):
            order = list(libs) if rnd % 2 == 0 else list(libs)[::-1]
            for n in order:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                graphs[n].replay()
                e1.record()
                torch.cuda.synchronize()
                times[n].append(e0.elapsed_time(e1) * 1e3 / LAUNCHES)
        med = {n: sorted(t)[len(t) // 2] for n, t in times.items()}
        line = f"C={C} N={N} M={M} K={K}: " + ", ".join(
            f"{n} {med[n]:.2f} us (min {min(times[n]):.2f}, max {max(times[n]):.2f})" for n in libs)
        if "other" in libs:
            diff = float((out["this"] - out["other"]).abs().max()) / max(float(out["other"].abs().max()), 1e-30)
            line += f"; this/other {med['this'] / med['other']:.3f}; max rel diff {diff:.1e}"
        print(line, flush=True)
        pt_utils.clear_neighbor_cache()


if __name__ == "__main__":
    main()
