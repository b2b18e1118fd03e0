#!/usr/bin/env python
"""bench.py -- local-aggregation hot path: points/s (forward + backward) on N H100s.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--config 1..5] [--impl ours|reference]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W

One "step" = one LocalAggregation call of the BASELINE.json configuration (default configs[2], the largest
single-GPU configuration: S3DIS Pseudo-Grid, B=8 N=15000 K=26 C=72 per GPU), forward AND backward (gradients w.r.t. the input
features and every parameter), INCLUDING the neighbour search (the neighbour-list cache is disabled, so no
step re-uses the previous step's search), on a fresh synthetic batch: a ring of pre-generated batches larger
than the 50 MB L2 is rotated so that no step finds its inputs in L2.  Multi-GPU: batches shard over ranks
(weak scaling: B per GPU is fixed), the only exchange is the NCCL all-reduce of parameter gradients, captured in
the step's CUDA graph.  The other four BASELINE configurations are measured the same way (device-timed) and
reported under "configs" in the same JSON line (c4/c5 at their per-GPU shard: B/8 clouds per GPU).

The JSON line follows the driver contract; extra objects:
  roofline      dominant entry point (by CUDA-event time): SURVEY section 8(d) algorithmic bytes of the step,
                (16C + 8K + 32) x points per launch, over that entry point's time vs the measured HBM peak
  cpu_baseline  the oracle port of the reference path on this box's host cores, bounded sample
  e2e           same metric through the public module API from pinned HOST buffers (H2D + D2H inside)
  ref_gpu       (informational) the reference's own CUDA extension (oracle/_ref) under the unfused python layer
`--impl reference` prints the reference arm: the reference's algorithm on the host cores (oracle port; the
reference's native ops are CUDA-only, every entry point is TORCH_CHECK(false, "CPU not supported")).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")  # one hardware queue per stream (copy / search / step)
import torch  # noqa: E402


def trace(msg):
    """progress to stderr when CL3D_BENCH_TRACE is set (multi-rank debugging)"""
    if os.environ.get("CL3D_BENCH_TRACE"):
        print(f"[bench rank {os.environ.get('RANK', '0')} t={time.perf_counter():.1f}] {msg}", file=sys.stderr, flush=True)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--config", type=int, default=3, help="BASELINE.json config index 1..5 (default 3 = configs[2], the "
                    "largest single-GPU configuration)")
    ap.add_argument("--no-extra-configs", action="store_true", help="skip the device-timed legs of the other configs")
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--batch", type=int, default=None, help="clouds per GPU (default: the config's B, or B/8 for 8-GPU configs)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-ref-gpu", action="store_true")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--no-e2e", action="store_true", help="skip the end-to-end leg (profiling captures: keeps the run to 3 steps)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed (output, d/dfeatures, "
                         "parameter gradients) as DIR/<name>.npy, float32, at most 64 MB in all")
    return ap.parse_args()


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    return 3350.0, "fallback (H100 SXM data sheet, HBM3)"


class ClockSampler:
    """SM clock and throttle reasons DURING the timed region.  A thread samples NVML about every millisecond; it is
    started before the warm-up so that it is in steady state (NVML initialised, thread scheduled) when the timed
    region begins, every sample carries a host time stamp, and only the samples between mark_start() and mark_stop()
    are reported.  (Round 1 started a 5 ms sampler between the barrier and the first event of a 6 ms region and
    caught nothing.)  nvidia-smi is only the fallback when NVML cannot be loaded: one polling nvidia-smi per rank
    stalls kernel launches at 8 GPUs."""
    Q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown," \
        "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown," \
        "clocks_event_reasons.sw_power_cap"
    NAMES = [(0x8, "hw_slowdown"), (0x40, "hw_thermal_slowdown"), (0x20, "sw_thermal_slowdown"), (0x4, "sw_power_cap")]

    def __init__(self, gpu_index, period_s=0.001):
        self.gpu, self.period = gpu_index, period_s
        self.nv = []          # (t, sm_mhz, sm_max_mhz, reasons bitmask)
        self.lines = []       # (t, nvidia-smi csv line)
        self.proc = None
        self.stop_ev = None
        self.err = None
        self.t0 = self.t1 = None

    def _nvml_handle(self):
        import pynvml
        pynvml.nvmlInit()
        try:
            uuid = str(torch.cuda.get_device_properties(self.gpu).uuid)
            return pynvml, pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid).encode())
        except Exception:
            return pynvml, pynvml.nvmlDeviceGetHandleByIndex(self.gpu)

    def _nvml_loop(self, nv, h, stop):
        mx = float(nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM))
        reasons = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or \
            getattr(nv, "nvmlDeviceGetCurrentClocksThrottleReasons")
        while not stop.is_set():
            try:
                self.nv.append((time.perf_counter(), float(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)), mx,
                                int(reasons(h))))
            except Exception as e:  # noqa: BLE001
                self.err = repr(e)[:120]
                break
            stop.wait(self.period)

    def start(self):
        try:
            nv, h = self._nvml_handle()
            nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)   # fail here, not in the thread
            self.stop_ev = threading.Event()
            self.nvt = threading.Thread(target=self._nvml_loop, args=(nv, h, self.stop_ev), daemon=True)
            self.nvt.start()
            return self
        except Exception as e:  # noqa: BLE001
            self.err = "nvml: " + repr(e)[:120]
            self.stop_ev = None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.gpu), f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "20"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception as e:  # noqa: BLE001
            self.err = (self.err or "") + " nvidia-smi: " + repr(e)[:120]
            self.proc = None
        return self

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append((time.perf_counter(), line.strip()))

    def mark_start(self):
        self.t0 = time.perf_counter()

    def mark_stop(self):
        self.t1 = time.perf_counter()

    def stop(self):
        if self.stop_ev is not None:
            self.stop_ev.set()
            self.nvt.join(timeout=1)
        if self.proc is not None:
            time.sleep(0.05)
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:
                self.proc.kill()
        t0, t1 = self.t0 or 0.0, self.t1 or float("inf")
        samples = [(sm, mx, r) for (t, sm, mx, r) in self.nv if t0 <= t <= t1]
        source = "nvml"
        if not samples and self.lines:
            source = "nvidia-smi"
            for t, ln in self.lines:
                f = [x.strip() for x in ln.split(",")]
                if len(f) < 8 or not (t0 <= t <= t1 + 0.02):
                    continue
                try:
                    bits = sum(b for (b, _), v in zip(self.NAMES, f[4:8]) if v.lower().startswith("active"))
                    samples.append((float(f[0]), float(f[1]), bits))
                except ValueError:
                    continue
        if not samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "samples": 0, "reasons": [],
                    "note": "no clock sample inside the timed region (" + (self.err or "sampler produced none") + ")",
                    "samples_total": len(self.nv) + len(self.lines)}
        bits = 0
        for _, _, r in samples:
            bits |= r
        return {"sm_mhz": statistics.median(x[0] for x in samples), "sm_min_mhz": min(x[0] for x in samples),
                "sm_max_mhz": max(x[1] for x in samples), "samples": len(samples),
                "reasons": sorted(n for b, n in self.NAMES if bits & b), "source": source,
                "window_ms": (t1 - t0) * 1e3 if self.t1 else None}


# algorithmic (compulsory) HBM bytes per POINT of each entry point, see DESIGN.md "Kernels"
def algo_bytes_per_point(name, C, K, Cout):
    Cop = (Cout + 7) & ~7
    table = {
        "cl3d_ball_query_algo": 16 + 16 + 4 * K + 4,            # support xyz+mask, query xyz+mask, idx, ncount
        "cl3d_to_point_major": 8 * C,
        "cl3d_to_channel_major": 8 * C,
        "cl3d_agg_fwd": 8 * C + 4 * K + 20,                    # f row in, agg out, idx, xyz, ncount
        "cl3d_agg_bwd": 8 * C + 4 * K + 20,
        "cl3d_bn_relu_fwd": 8 * C,
        "cl3d_bn_relu_bwd": 12 * C + 8 * C,                    # (grad_y, x) twice, g_pm out
        "cl3d_build_csr": 12 * K + 8,
        # three products per step, per call: [f|xyz] row in (or d/dfeat row out) + the 2*Cop-wide A|T row
        "cl3d_sgemm_algo": 4 * (C + 3) + 8 * Cop,
        "cl3d_pwmlp_fwd_stats": 8 * Cop + 8 * Cout + 2 * Cop + 4 * K + 16,
        "cl3d_pwmlp_fwd_out": 8 * Cout,
        "cl3d_pwmlp_bwd": 16 * Cout + 8 * Cop + 2 * Cop + 4 * K + 16 + 16 * Cop,
    }
    return table.get(name)


DUMP_BUDGET_BYTES = 64 << 20


def dump_outputs(out_dir, arrays):
    """Write {name: tensor} as out_dir/<name>.npy in float32.  Arrays that fit the budget are written whole (smallest
    first); each remaining array gets an equal share of what is left and is written as a fixed sample of its
    flattened elements (indices drawn once from a generator seeded with 0, sorted), so that two builds given the same
    arguments can be compared element for element."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    items = sorted(arrays.items(), key=lambda kv: kv[1].numel())
    left = (DUMP_BUDGET_BYTES - 4096 * len(items)) // 4   # room for the .npy headers
    written = {}
    for i, (name, t) in enumerate(items):
        flat = t.detach().float().reshape(-1)
        share = left // (len(items) - i)
        if flat.numel() > share:
            g = torch.Generator().manual_seed(0)
            idx = torch.randperm(flat.numel(), generator=g)[:share].sort().values
            flat = flat[idx.to(flat.device)]
            written[name] = f"sample of {share} of {t.numel()} elements, shape {list(t.shape)}"
        else:
            flat = flat.reshape(t.shape)
            written[name] = f"shape {list(t.shape)}"
        left -= flat.numel()
        np.save(os.path.join(out_dir, name + ".npy"), flat.cpu().numpy().astype(np.float32))
    return written


def build_module(spec, device):
    import numpy as np
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    from closerlook3d_b200 import synth
    i = spec["index"]
    torch.manual_seed(2000 + i)
    np.random.seed(2000 + i)
    r = synth.ball_radius(spec["N"], spec["K"])
    mod = LocalAggregation(spec["C"], spec["C"], r, spec["K"], spec["cfg"])
    return mod.to(device), r


class numa_local:
    """Bind the CALLING THREAD to the CPUs NVML reports as local to the GPU for the end-to-end leg: the pinned host
    buffers are allocated on that NUMA node (cudaHostAlloc places pages on the caller's node; the H2D copies are DMA
    from there) and the launching thread does not pay cross-socket latency per CUDA call; then restore the
    thread's affinity.  The intra-op thread pools are created before the first use (full mask), so the CPU legs
    of this script are not affected.  Any failure leaves the affinity untouched."""

    def __init__(self, device):
        self.device, self.saved, self.cpus = device, None, None

    def __enter__(self):
        try:
            import pynvml
            torch.ones(1 << 22).sum().item()          # create torch's CPU thread pool with the unrestricted mask
            pynvml.nvmlInit()
            uuid = str(torch.cuda.get_device_properties(self.device).uuid)
            try:
                h = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid).encode())
            except Exception:
                h = pynvml.nvmlDeviceGetHandleByIndex(self.device.index or 0)
            n = os.cpu_count() or 1
            words = pynvml.nvmlDeviceGetCpuAffinity(h, (n + 63) // 64)
            cpus = {64 * i + b for i, w in enumerate(words) for b in range(64) if (int(w) >> b) & 1}
            saved = os.sched_getaffinity(0)
            cpus &= saved
            if cpus and cpus != saved:
                os.sched_setaffinity(0, cpus)
                self.saved, self.cpus = saved, cpus
        except Exception:
            self.saved = None
        return self

    def __exit__(self, *exc):
        if self.saved is not None:
            try:
                os.sched_setaffinity(0, self.saved)
            except Exception:
                pass
        return False


def make_ring(spec, B_local, rank, device, min_bytes, pinned=False):
    """pre-generated batches; total size > min_bytes so consecutive steps never hit L2-resident inputs"""
    from closerlook3d_b200 import synth
    per = B_local * spec["N"] * (12 + 4 + 4 * spec["C"])
    n = max(2, int(min_bytes // per) + 1)
    n = min(n, 64)
    ring = []
    for t in range(n):
        d = synth.make_cloud_batch(B_local, spec["N"], spec["C"], 1000 + spec["index"] + 7919 * t + 104729 * rank,
                                   b_offset=rank * B_local)
        if pinned:
            ring.append({k: v.pin_memory() for k, v in d.items()})
        else:
            ring.append({k: v.to(device) for k, v in d.items()})
    return ring


def local_batch(args, spec):
    return args.batch or (spec["B"] if spec["gpus"] == 1 else max(1, spec["B"] // spec["gpus"]))


def device_leg(spec, B_local, rank, world, device, steps, warmup, use_graph=True, sampler=None, want_profile=False,
               keep=False, dump_dir=None):
    """Device-timed leg of one configuration: `warmup` untimed steps, then exactly `steps` steps between
    (barrier + synchronize) brackets, timed with CUDA events on the launch stream; MAX over ranks.
    Inputs are resident in HBM (a ring of batches larger than L2) when the timed region starts."""
    from closerlook3d_b200 import _lib, pt_utils
    from closerlook3d_b200 import dist as cdist
    import torch.distributed as dist
    pt_utils.cache_enabled = False  # every step searches its neighbours again (no cached outputs)
    pt_utils.clear_neighbor_cache()
    mod, radius = build_module(spec, device)
    mod.train()
    L2 = 50e6
    ring = make_ring(spec, B_local, rank, device, 1.6 * L2)
    C, N, K = spec["C"], spec["N"], spec["K"]
    gout = torch.randn(B_local, C, N, device=device, generator=torch.Generator(device=device).manual_seed(5))
    params = [p for p in mod.parameters()]
    L = _lib.lib()

    gs = None
    if use_graph:
        from closerlook3d_b200.graphed import GraphedStep
        b0 = ring[0]
        # forward + backward + (world > 1) the NCCL all-reduce of the parameter gradients: ONE graph
        gs = GraphedStep(mod, b0["xyz"], b0["mask"], b0["features"], gout)
    flat = None if use_graph else cdist.FlatGradients(params)

    def eager_step(batch, reduce_grads=True):
        f = batch["features"]
        f.requires_grad_(True)
        f.grad = None
        if flat is not None:
            flat.zero()
            flat.attach()
        else:
            for p in params:
                p.grad = None
        out = mod(batch["xyz"], batch["xyz"], batch["mask"], batch["mask"], f)
        out.backward(gout)
        if world > 1 and reduce_grads and flat is not None:
            flat.allreduce()
        return out

    def step(batch):
        if use_graph:
            gs.load(batch["xyz"], batch["mask"], batch["features"])  # this step's batch -> static buffers
            return gs.replay()
        return eager_step(batch)

    def last_step_arrays(out, batch):
        """what a caller of the step receives: the output, d/dfeatures and the parameter gradients"""
        if use_graph:
            f_grad, grads = gs.features.grad, gs.grads()
        else:
            f_grad, grads = batch["features"].grad, [p.grad for p in params if p.requires_grad]
        names = [n for n, p in mod.named_parameters() if p.requires_grad]
        arrays = {"out": out, "grad_features": f_grad}
        arrays.update({"grad_" + n: g for n, g in zip(names, grads) if g is not None})
        return arrays

    # kernels of one step (a graph replay does not pass through the library's launch counter: count one eager step)
    torch.cuda.synchronize()
    c0 = L.cl3d_launch_count()
    if use_graph:
        for p in params:
            p.grad = None
    tmp = {k: v.clone() for k, v in ring[0].items()}
    mod(tmp["xyz"], tmp["xyz"], tmp["mask"], tmp["mask"], tmp["features"].requires_grad_(True)).backward(gout)
    torch.cuda.synchronize()
    per_step = int(L.cl3d_launch_count() - c0)
    del tmp

    for w in range(warmup):
        step(ring[w % len(ring)])
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    e_all0, e_all1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()           # all ranks enter the timed region together ...
        torch.cuda.synchronize()  # ... with nothing pending on the device
    if sampler is not None:
        sampler.mark_start()
    t_wall0 = time.perf_counter()
    e_all0.record()
    for s in range(steps):
        b = ring[(warmup + s) % len(ring)]
        ev[s][0].record()
        out = step(b)
        ev[s][1].record()
    e_all1.record()
    torch.cuda.synchronize()
    t_wall = time.perf_counter() - t_wall0
    if sampler is not None:
        sampler.mark_stop()
    dumped = dump_outputs(dump_dir, last_step_arrays(out, b)) if dump_dir and rank == 0 and steps > 0 else None
    if world > 1:
        dist.barrier()
    total_ms = e_all0.elapsed_time(e_all1)
    per = sorted(a.elapsed_time(b) for a, b in ev)
    t = torch.tensor([total_ms, per[len(per) // 2]], device=device, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    total_ms, med_ms = float(t[0].item()), float(t[1].item())
    ms_per_step = total_ms / steps
    pts_per_step = B_local * N * world
    res = dict(value=pts_per_step / (ms_per_step * 1e-3), ms_per_step=ms_per_step, ms_per_step_median=med_ms,
               launches=per_step * steps, launches_per_step=per_step, B_local=B_local, wall_s=t_wall,
               points_per_step=pts_per_step, radius=radius)
    if dumped is not None:
        res["dumped"] = dumped

    # ---- per-entry-point device time (separate identical pass, CUDA events on the launch stream, eager: the
    #      events need the library calls, not a graph replay)
    if want_profile and rank == 0:
        for p in params:
            p.grad = None
        _lib.profiler.start()
        for s in range(steps):
            b = ring[(warmup + s) % len(ring)]
            f = b["features"]
            f.requires_grad_(True)
            f.grad = None
            mod(b["xyz"], b["xyz"], b["mask"], b["mask"], f).backward(gout)
        res["prof"] = _lib.profiler.stop()
    if keep:
        res.update(mod=mod, ring=ring, gs=gs, gout=gout)
    else:
        del gs, ring, mod
        torch.cuda.empty_cache()
    return res


def e2e_leg(args, spec, res, rank, world, device):
    """The same metric END TO END through the public API from pinned HOST buffers: every step's batch is copied
    host -> device inside the timed region and the step's result (+ the reduced parameter gradients) is read
    back.  With graphs: closerlook3d_b200.graphed.PipelinedTrainer overlaps the copy of batch i+1 with the replay
    of batch i (double-buffered static inputs) and reads results one step late."""
    import torch.distributed as dist
    B_local, mod, ring, gout = res["B_local"], res["mod"], res["ring"], res["gout"]
    use_graph = not args.no_graph
    with numa_local(device) as nl:
        hring = make_ring(spec, B_local, rank, device, 0.0, pinned=True)
        h2d = sum(v.numel() * v.element_size() for v in hring[0].values())
        nst = args.steps
        # the host link on its own: one batch, pinned -> device, 10 back-to-back copies (the e2e rate cannot exceed
        # points_per_batch / this time; the link is shared with the other tenants of the box)
        dbuf = {k: torch.empty_like(v, device=device) for k, v in hring[0].items()}
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for rep in range(2):
            ev0.record()
            for _ in range(10):
                for k, v in hring[0].items():
                    dbuf[k].copy_(v, non_blocking=True)
            ev1.record()
            torch.cuda.synchronize()
        h2d_ms = ev0.elapsed_time(ev1) / 10
        del dbuf
        if use_graph:
            from closerlook3d_b200.graphed import PipelinedTrainer
            b0 = ring[0]
            tr = PipelinedTrainer(mod, b0["xyz"], b0["mask"], b0["features"], gout)
            d2h = tr.d2h_bytes
            for w in range(4):
                tr.step(hring[w % len(hring)])
            tr.flush()
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            t0 = time.perf_counter()
            for s in range(nst):
                tr.step(hring[s % len(hring)])
            tr.flush()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            how = "PipelinedTrainer: H2D of batch i+1 overlaps the replay of batch i; results read one step late"
        else:
            from closerlook3d_b200 import dist as cdist
            params = [p for p in mod.parameters()]
            d2h = 4

            def e2e_step(hb):
                f = hb["features"].to(device, non_blocking=True).requires_grad_(True)
                x, m = hb["xyz"].to(device, non_blocking=True), hb["mask"].to(device, non_blocking=True)
                for p in params:
                    p.grad = None
                out = mod(x, x, m, m, f)
                out.backward(gout)
                cdist.allreduce_gradients(params)
                return float(out.sum().item())  # D2H read of the step's result
            for w in range(3):
                e2e_step(hring[w % len(hring)])
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            t0 = time.perf_counter()
            for s in range(nst):
                e2e_step(hring[s % len(hring)])
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            how = "serial: H2D, step, D2H"
    te = torch.tensor([dt], device=device, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(te, op=dist.ReduceOp.MAX)
    return {"value": res["points_per_step"] * nst / float(te.item()), "unit": "points/s", "h2d_bytes_per_step": int(h2d),
            "d2h_bytes_per_step": int(d2h), "d2h": "sum of the output + the (all-reduced) parameter gradients",
            "steps": nst, "ms_per_step": float(te.item()) / nst * 1e3, "how": how,
            "pinned_buffers": "allocated on the GPU-local NUMA node" if nl.cpus else "default placement",
            "h2d_copy_alone_ms": h2d_ms, "h2d_copy_alone_gbs": h2d / (h2d_ms * 1e-3) / 1e9,
            "timing": "host wall clock around all steps (copies inside), max over ranks"}


def cpu_reference_arm(spec, steps, warmup, budget_s=25.0):
    """the reference's algorithm on the host cores: oracle port (C/OpenMP restatement of the CUDA ops under the
    unfused python layer), forward + backward, on a bounded sample of the workload"""
    import oracle
    oracle.build()
    from oracle import ext as oext, la_oracle
    from closerlook3d_b200 import synth
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    import numpy as np
    i = spec["index"]
    torch.manual_seed(2000 + i)
    np.random.seed(2000 + i)
    r = synth.ball_radius(spec["N"], spec["K"])
    sd = LocalAggregation(spec["C"], spec["C"], r, spec["K"], spec["cfg"]).state_dict()
    # bounded sample: as many clouds of the workload as fit ~budget_s
    Bs = min(spec["B"], 2)
    orc = la_oracle.OracleLocalAggregation(oext, spec["la"], spec["C"], spec["C"], r, spec["K"], spec["cfg"], sd)

    def one(B):
        d = synth.make_cloud_batch(B, spec["N"], spec["C"], 1000 + i)
        f = d["features"].requires_grad_(True)
        t0 = time.perf_counter()
        out = orc(d["xyz"], d["xyz"], d["mask"], d["mask"], f)
        out.backward(torch.ones_like(out))
        return time.perf_counter() - t0

    # give the CPU arm its best thread count: all cores is not always fastest for these op sizes
    # (oversubscribed torch + OpenMP pools on a 100+ core host are far slower than 16-32 threads)
    ncores = os.cpu_count() or 1
    cands = sorted({c for c in (8, 16, 32, 64, ncores) if c <= ncores}) or [ncores]
    best_t, best_n = None, ncores
    for nt in cands:
        torch.set_num_threads(nt)
        oext.set_threads(nt)
        one(Bs)
        tt = min(one(Bs), one(Bs))
        if best_t is None or tt < best_t:
            best_t, best_n = tt, nt
    torch.set_num_threads(best_n)
    oext.set_threads(best_n)
    t = one(Bs)  # warm-up + calibration
    per_cloud = t / Bs
    n_steps = max(1, steps)
    Bs = int(max(1, min(spec["B"], budget_s / max(per_cloud, 1e-6) / (n_steps + max(0, warmup)))))
    for _ in range(max(0, warmup)):
        one(Bs)
    ts = [one(Bs) for _ in range(n_steps)]
    sec = sum(ts) / len(ts)
    return {"value": Bs * spec["N"] / sec, "unit": "points/s", "cores": best_n, "host_cores": ncores, "kind": "port",
            "threads_tried": cands, "ms_per_step": sec * 1e3,
            "sample": f"{Bs} of {spec['B']} clouds of the workload per step, fwd+bwd, {n_steps} steps"}


def ref_gpu_arm(spec, device, res):
    """informational: the reference's OWN CUDA extension (compiled unmodified into oracle/_ref) under the unfused
    python layer (oracle/la_oracle.py) on the same GPU and inputs, TF32 off -- timed, AND compared with this
    engine's outputs / gradients on the full-size batch it computes anyway (parity at the benchmarked shape)."""
    try:
        from oracle import build_ref, la_oracle
        ext = build_ref.load()
    except Exception as e:
        return {"unavailable": str(e)[:200]}
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    mod = res["mod"]
    sd = {k: v.detach().clone() for k, v in mod.state_dict().items()}
    orc = la_oracle.OracleLocalAggregation(ext, spec["la"], spec["C"], spec["C"], res["radius"], spec["K"], spec["cfg"],
                                           sd, device=device)
    ring = res["ring"]
    B, N, C = res["B_local"], spec["N"], spec["C"]
    gout = torch.ones(B, C, N, device=device)

    def one(b):
        f = b["features"].detach().clone().requires_grad_(True)
        out = orc(b["xyz"], b["xyz"], b["mask"], b["mask"], f)
        out.backward(gout)
        return out, f.grad

    try:
        # ---- parity on ring[0] (both sides start from the same parameters and running statistics)
        b = ring[0]
        f2 = b["features"].detach().clone().requires_grad_(True)
        is_max = spec["cfg"].get(spec["la"], {}).get("reduction") == "max" if isinstance(spec["cfg"], dict) else \
            getattr(getattr(spec["cfg"], spec["la"], None), "reduction", None) == "max"
        la_oracle.KEEP = {} if is_max else None
        o_ref = orc(b["xyz"], b["xyz"], b["mask"], b["mask"], f2)
        decided, undecided = None, 0
        if la_oracle.KEEP:
            # max over the neighbours: where two DISTINCT neighbours tie inside the tolerance, rounding picks the one
            # that receives the gradient (tests/test_local_aggregation_gpu.py); those positions get no upstream
            # gradient on either side
            key = "pwmlp_premax" if "pwmlp_premax" in la_oracle.KEEP else "premax"
            decided = la_oracle.argmax_is_decided(la_oracle.KEEP[key], la_oracle.KEEP["idx"],
                                                  relu=key == "pwmlp_premax")
            undecided = int((~decided).sum())
        la_oracle.KEEP = None
        for p in mod.parameters():
            p.grad = None
        f = b["features"].detach().clone().requires_grad_(True)
        out = mod(b["xyz"], b["xyz"], b["mask"], b["mask"], f)
        keep = ~((out.detach() > 0) != (o_ref.detach() > 0))   # ReLU sign flips inside the output tolerance
        flips = int((~keep).sum())
        if decided is not None:
            keep = keep & decided
        (o_ref * keep).sum().backward()
        (out * keep).sum().backward()
        torch.cuda.synchronize()
        e_out = float((out.detach() - o_ref.detach()).abs().max()) / max(1.0, float(o_ref.detach().abs().max()))
        e_g = float((f.grad - f2.grad).abs().max()) / max(1.0, float(f2.grad.abs().max()))
        parity = {"out_err": e_out, "grad_features_err": e_g, "relu_sign_flips": flips,
                  "undecided_maxima_masked": undecided, "tolerance": 1e-5, "ok": bool(e_out <= 1e-5 and e_g <= 1e-5),
                  "what": "this engine vs the reference CUDA ext + unfused layer, full per-GPU batch, fwd + bwd"}
        del o_ref, out, f, f2, keep, decided
        torch.cuda.empty_cache()
        for w in range(2):
            one(ring[w % len(ring)])
        torch.cuda.synchronize()
        n = 5
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in range(n):
            one(ring[(2 + s) % len(ring)])
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        return {"value": B * N / (ms * 1e-3), "unit": "points/s", "ms_per_step": ms, "parity": parity,
                "what": "reference CUDA ext (sm_90, unmodified) + unfused python layer, 1 GPU, fwd+bwd"}
    except Exception as e:  # e.g. out of memory on the inflated tensors
        return {"unavailable": str(e)[:200]}


def config_dict(workload, spec, B_local, world):
    """identical for both arms (the driver compares the two lines' `config`); how each arm runs is in `method`"""
    return {"workload": workload, "family": spec["la"], "clouds_per_gpu": B_local,
            "points_per_step": B_local * spec["N"] * world, "parallelism": f"dp{world}",
            "l2": "GPU arm: inputs rotate over a ring of pre-generated batches > 1.6x L2 (50 MB), no step finds its "
                  "inputs in L2"}


def shutdown_distributed(world, *graph_holders):
    """Leave torch.distributed cleanly.  CUDA graphs that captured NCCL collectives hold references on the
    communicator and ncclCommDestroy waits for them (measured: destroy_process_group() never returned while a
    GraphedStep with an in-graph all-reduce was alive), so every graph is released first; a watchdog ends the
    process if the teardown still stalls -- the JSON line has been printed by then."""
    if world <= 1:
        return
    import gc
    for h in graph_holders:
        if isinstance(h, dict):
            for k in ("gs", "mod", "ring", "gout"):
                h.pop(k, None)
    gc.collect()
    torch.cuda.synchronize()
    sys.stdout.flush()
    torch.distributed.barrier()          # rank 0 arrives after its single-rank legs; NCCL's own timeout bounds the wait
    t = threading.Timer(30.0, lambda: os._exit(0))
    t.daemon = True
    t.start()
    try:
        torch.distributed.destroy_process_group()
    finally:
        t.cancel()


def step_algo_bytes_per_point(C, K):
    """SURVEY.md section 8(d): compulsory HBM traffic of a fused fwd+bwd step, bytes per point"""
    return 16 * C + 8 * K + 32


def main():
    args = parse()
    # ONE JSON line on stdout: libraries (NCCL's version banner, OpenMP, ...) write to fd 1 as they please, so fd 1 is
    # pointed at stderr for the run and the line goes to a duplicate of the original stdout
    sys.stdout.flush()
    real_stdout = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    from closerlook3d_b200.config import baseline_config
    spec = baseline_config(args.config)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    metric = "aggregated points/sec (fwd+bwd), one LocalAggregation call incl. neighbour search"

    def workload_of(sp, idx):
        return f"configs[{idx - 1}]: {sp['name']} B={sp['B']} N={sp['N']} K={sp['K']} C={sp['C']}"
    workload = workload_of(spec, args.config)

    if args.impl == "reference":
        if rank != 0:
            return 0
        cb = cpu_reference_arm(spec, args.steps, args.warmup)
        line = {"impl": "reference", "metric": metric, "value": cb["value"], "unit": "points/s", "n_gpus": args.gpus,
                "steps": args.steps, "warmup": args.warmup, "ms_per_step": cb["ms_per_step"],
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                "config": config_dict(workload, spec, local_batch(args, spec), max(1, args.gpus)),
                "method": {"arm": "the reference's algorithm on the host cores (oracle port: C/OpenMP restatement of the "
                                  "CUDA ops under the unfused python layer), each step a bounded sample of the workload"},
                "cpu_baseline": cb,
                "e2e": {"value": cb["value"], "unit": "points/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        print(json.dumps(line), file=real_stdout, flush=True)
        return 0

    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (there is no CPU path for the product)")
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=device)
    trace("process group up")
    sampler = ClockSampler(torch.cuda.current_device()).start()   # steady state long before the timed region
    B_local = local_batch(args, spec)
    res = device_leg(spec, B_local, rank, world, device, args.steps, args.warmup, use_graph=not args.no_graph,
                     sampler=sampler, want_profile=True, keep=True, dump_dir=args.dump_outputs)
    clocks = sampler.stop()
    trace(f"device leg done: {res['ms_per_step']:.4f} ms/step")
    e2e = None if args.no_e2e else e2e_leg(args, spec, res, rank, world, device)
    trace("e2e leg done")

    # ---- the other BASELINE configurations, device-timed the same way (per-GPU shard of the 8-GPU configs)
    extra = {}
    if not args.no_extra_configs:
        for ci in (1, 2, 3, 4, 5):
            if ci == args.config:
                continue
            sp = baseline_config(ci)
            Bl = sp["B"] if sp["gpus"] == 1 else max(1, sp["B"] // sp["gpus"])
            st = min(args.steps, 30)
            try:
                r = device_leg(sp, Bl, rank, world, device, st, max(3, min(args.warmup, 5)),
                               use_graph=not args.no_graph)
                extra[f"c{ci}"] = {"workload": workload_of(sp, ci), "family": sp["la"], "clouds_per_gpu": Bl,
                                   "value": r["value"], "unit": "points/s", "ms_per_step": r["ms_per_step"],
                                   "ms_per_step_median": r["ms_per_step_median"], "steps": st, "n_gpus": world,
                                   "launches_per_step": r["launches_per_step"],
                                   "step_frac_of_hbm_roofline": step_algo_bytes_per_point(sp["C"], sp["K"]) *
                                   r["value"] / world / 1e9 / peaks()[0]}
            except Exception as e:  # noqa: BLE001
                extra[f"c{ci}"] = {"workload": workload_of(sp, ci), "error": str(e)[:200]}
            trace(f"extra config c{ci} done")
    if rank != 0:
        shutdown_distributed(world, res)
        return 0

    peak, peak_src = peaks()
    C, K, N = spec["C"], spec["K"], spec["N"]
    pts_local = res["B_local"] * N
    prof = res.get("prof") or {}
    kern = []
    for name, (calls, ms) in prof.items():
        ab = algo_bytes_per_point(name, C, K, C)
        per_launch_ms = ms / max(1, calls)
        kern.append({"entry": name, "calls_per_step": calls / args.steps, "ms_per_step": ms / args.steps,
                     "ms_per_call": per_launch_ms,
                     "kernel_model_gbs": (ab * pts_local / (per_launch_ms * 1e-3) / 1e9) if ab and per_launch_ms > 0 else None})
    # the dominant KERNEL is the longest single launch (an entry point called twice per step -- the search and,
    # beside the forward on the side stream, the transposed lists -- must not win on the sum of its calls)
    kern.sort(key=lambda k: -k["ms_per_call"])
    roof = None
    step_bytes = step_algo_bytes_per_point(C, K) * pts_local
    if kern:
        top = kern[0]
        # DRAM bytes per launch of the same entry point from an `ncu --set full` capture of this workload
        # (profiles/traffic.json, written by tools/ncu_traffic.py); null when no capture exists for the config
        traffic, traffic_src = None, None
        tp = os.path.join(ROOT, "profiles", "traffic.json")
        if os.path.exists(tp):
            with open(tp) as f:
                tj = json.load(f).get(f"c{args.config}", {})
            ent = tj.get(top["entry"])
            if ent and res["B_local"] == tj.get("_clouds_per_gpu", res["B_local"]):
                traffic = ent["dram_bytes_per_step"] / max(1.0, top["calls_per_step"])
                traffic_src = f"profiles/traffic.json ({tj.get('_report', 'ncu --set full')})"
        t_dom = top["ms_per_call"] * 1e-3
        achieved = step_bytes / t_dom / 1e9
        roof = {"bound": "hbm", "kernel": top["entry"], "achieved": achieved, "peak": peak, "unit": "GB/s",
                "frac": achieved / peak, "traffic": traffic, "traffic_source": traffic_src,
                "algo_bytes_per_launch": step_bytes,
                "algo_bytes_model": "SURVEY.md 8(d): (16C + 8K + 32) bytes/point x points per launch "
                                    f"= {step_algo_bytes_per_point(C, K)} x {pts_local}",
                "kernel_time_ms": top["ms_per_call"], "peak_source": peak_src,
                # share of the graph-replayed step (the entry points' own times sum to more than the step: the list
                # build runs beside the forward on the side stream and its elapsed time includes waiting for SMs)
                "share_of_step": top["ms_per_step"] / max(1e-9, res["ms_per_step"]),
                "step_frac": step_bytes / (res["ms_per_step"] * 1e-3) / 1e9 / peak,
                "kernel_model_frac": (top["kernel_model_gbs"] / peak) if top.get("kernel_model_gbs") else None}
    cb = None
    if not args.no_cpu_baseline and world == 1:      # contract: rank 0 at N=1 only
        cb = cpu_reference_arm(spec, 3, 1, budget_s=15.0)
    rg = None
    if not args.no_ref_gpu and world == 1:
        rg = ref_gpu_arm(spec, device, res)
    line = {"metric": metric, "value": res["value"], "unit": "points/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": res["ms_per_step"], "ms_per_step_median": res["ms_per_step_median"],
            "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": config_dict(workload, spec, res["B_local"], world),
            "method": {"launch": "CUDA graph replay of the captured step (fwd + bwd + NCCL all-reduce of the parameter "
                                 "gradients when n_gpus > 1); each step's batch is copied into the graph's static "
                                 "input buffers inside the timed region" if not args.no_graph else "eager launches",
                       "timing": "CUDA events around the K steps, (barrier + synchronize) on both sides, max over ranks",
                       "neighbour_cache": "disabled (search runs every step)"},
            "clocks": clocks, "gpu_launches": res["launches"], "gpu_launches_per_step": res["launches_per_step"],
            "dumped_outputs": res.get("dumped"), "e2e": e2e, "roofline": roof, "cpu_baseline": cb, "kernels": kern[:8], "configs": extra, "ref_gpu": rg}
    print(json.dumps(line), file=real_stdout, flush=True)
    trace("line printed")
    shutdown_distributed(world, res)
    trace("shut down")
    return 0


if __name__ == "__main__":
    sys.exit(main())
