"""A/B of the PseudoGrid kernel generations on one GPU, forward and backward: the third-generation kernels (default)
against the second (CL3D_PG_V2=1), the arms alternated inside one process.

    python tools/bench_pg.py [--launches 200] [--rounds 5]

Per shape: inputs from synth.make_cloud_batch, lists from ops.ball_query + ops.build_csr, a ring of batches larger
than L2 so no launch finds its inputs there; ops.agg_bwd timed with CUDA events over `launches` calls per arm and
round after a warm-up (the library's per-entry-point profiler: events around cl3d_agg_fwd / cl3d_agg_bwd alone).
Prints, per shape, direction and arm, the median and the min..max over the rounds (ms per call), and the ratio of the
medians; for the c3 shape also the layout pass (cl3d_to_point_major of the features), which sits on the same step's
critical path.  Needs a GPU; prints the card, its power limit and maximum SM clock.
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from closerlook3d_b200 import _lib, ops, synth  # noqa: E402

L2_BYTES = 50e6
SHAPES = [("c3  B=8 N=15000 K=26 C=72", 8, 15000, 26, 72), ("c3  B=1 N=15000 K=26 C=72", 1, 15000, 26, 72),
          ("B=4 N=15000 K=26 C=128", 4, 15000, 26, 128), ("B=8 N=15000 K=26 C=36", 8, 15000, 26, 36)]


def make_ring(dev, B, N, K, C):
    per = B * N * (12 + 4 + 8 * C)
    n = min(16, max(2, int(1.6 * L2_BYTES // per) + 1))
    r = synth.ball_radius(N, K)
    gen = torch.Generator().manual_seed(11)
    kpts = (torch.rand(15, 3, generator=gen) - 0.5) * 0.8 * r
    kpts[0] = 0
    wk = torch.randn(15, C, generator=gen).to(dev)
    ring = []
    for t in range(n):
        d = {k: v.to(dev) for k, v in synth.make_cloud_batch(B, N, C, 1003 + 7919 * t).items()}
        idx, _, ncount = ops.ball_query(d["xyz"], d["xyz"], d["mask"], d["mask"], r, K, want_mask=False)
        off, ent = ops.build_csr(idx, ncount, N)
        gout = torch.randn(B, C, N, device=dev, generator=torch.Generator(device=dev).manual_seed(5 + t))
        ring.append(dict(xyz=d["xyz"], idx=idx, ncount=ncount, off=off, ent=ent,
                         feat_pm=ops.to_point_major(d["features"]), gpm=ops.to_point_major(gout)))
    return ring, r, kpts.to(dev), wk


def timed(fn, entry, ring, launches):
    """ms per call of the library entry point `entry` (CUDA events around each call, _lib.profiler)"""
    for i in range(10):
        fn(ring[i % len(ring)])
    torch.cuda.synchronize()
    _lib.profiler.start()
    for i in range(launches):
        fn(ring[i % len(ring)])
    calls, total_ms = _lib.profiler.stop()[entry]
    assert calls == launches
    return total_ms / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pg.py: no CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
    os.environ.pop("CL3D_PG_V2", None)
    for name, B, N, K, C in SHAPES:
        ring, r, kpts, wk = make_ring(dev, B, N, K, C)

        def bwd(b):
            return ops.agg_bwd(ops.FAM_PSEUDOGRID, ops.REDUCE["sum"], b["gpm"], b["feat_pm"], b["xyz"], b["xyz"], b["ncount"],
                               b["off"], b["ent"], kpts, wk, C, N, K, r, 0, 1, 15, 0.4 * r, 0)

        def fwd(b):
            return ops.agg_fwd(ops.FAM_PSEUDOGRID, ops.REDUCE["sum"], b["feat_pm"], b["xyz"], b["xyz"], b["idx"], b["ncount"],
                               kpts, wk, C, r, 0, 1, 15, 0.4 * r, 0)

        for what, fn, entry in (("fwd", fwd, "cl3d_agg_fwd"), ("bwd", bwd, "cl3d_agg_bwd")):
            t = {"v2": [], "v3": []}
            for _ in range(args.rounds):
                os.environ["CL3D_PG_V2"] = "1"
                try:
                    t["v2"].append(timed(fn, entry, ring, args.launches))
                finally:
                    del os.environ["CL3D_PG_V2"]
                t["v3"].append(timed(fn, entry, ring, args.launches))
            m2, m3 = statistics.median(t["v2"]), statistics.median(t["v3"])
            print(f"{name}: {what} v2 {m2:.4f} ms [{min(t['v2']):.4f}..{max(t['v2']):.4f}]  "
                  f"v3 {m3:.4f} ms [{min(t['v3']):.4f}..{max(t['v3']):.4f}]  v2/v3 = {m2 / m3:.2f}x", flush=True)
        if name.startswith("c3  B=8"):
            feats = [torch.randn(B, C, N, device=dev) for _ in range(2)]
            tl = [timed(lambda f: ops.to_point_major(f), "cl3d_to_point_major", feats, args.launches)
                  for _ in range(args.rounds)]
            print(f"{name}: cl3d_to_point_major {statistics.median(tl):.4f} ms [{min(tl):.4f}..{max(tl):.4f}]",
                  flush=True)


if __name__ == "__main__":
    main()
