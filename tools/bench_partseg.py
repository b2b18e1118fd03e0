"""The multi-shape part-segmentation head: the fused kernel (csrc/multihead.cu) against the reference's composition of
torch ops (oracle/part_seg_oracle.py part_seg_heads: per head Conv1d, BatchNorm1d, ReLU, Conv1d over every point), both
forward + backward in training mode, the arms alternated inside one process.

    python tools/bench_partseg.py [--iters 20] [--rounds 5] [--no-model] [--dtype fp32|bf16|fp16]

Head shapes: PartNet (B=8, N=10000, S=17) and ShapeNetPart (B=16, N=2048, S=16), C = 72.  The torch arm runs with
TF32 off (cuDNN and cuBLAS in fp32: the accuracy-matched comparison) and with cuDNN's default TF32 on.  Then one whole
training step of the part-segmentation network (width 144, AdaptiveWeight dp fc1 avg, multi-shape cross entropy,
backward) at each dataset's shape, with the fused head and with the torch head.  Prints ms per call, median
[min..max] over the rounds, each arm's peak of torch.cuda.max_memory_allocated over one call (above what was allocated
before it), and the card with its power limit and clock.  Needs a GPU.

--dtype bf16 | fp16: mixed precision as under torch.autocast.  The head arms take a 16-bit x (what the decoder hands
the heads under autocast) and 16-bit d/dlogits: the fused head against the reference's composition run under
torch.autocast ([h(x) for h in heads], its convolutions in the 16-bit type).  The whole-model arms are the step of
tools/train_synth.py --amp: forward and loss under torch.autocast, backward (fp16 through a GradScaler), SGD step.
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from closerlook3d_b200 import backbone as bb, partseg, synth  # noqa: E402
from oracle import part_seg_oracle  # noqa: E402

SHAPES = [("partnet", 8, 10000), ("shapenetpart", 16, 2048)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e!r})"
    return f"{torch.cuda.get_device_name()} | {q}"


def make_heads(C, num_parts, dev):
    torch.manual_seed(0)
    heads = nn.ModuleList(nn.Sequential(nn.Conv1d(C, C, 1, bias=False), nn.BatchNorm1d(C), nn.ReLU(inplace=True),
                                        nn.Conv1d(C, n, 1)) for n in num_parts)
    return heads.to(dev).train()


def head_arms(B, N, num_parts, dev, amp=None):
    C = 72
    heads = make_heads(C, num_parts, dev)
    dt = amp or torch.float32
    x = torch.relu(torch.randn(B, C, N, device=dev)).to(dt).requires_grad_(True)
    gs = [torch.randn(B, n, N, device=dev).to(dt) for n in num_parts]
    params = list(heads.parameters())
    if amp is not None:
        def run(fused):
            def call():
                with torch.autocast("cuda", dtype=amp):
                    out = partseg.multi_shape_heads_forward(heads, x) if fused else [h(x) for h in heads]
                torch.autograd.grad(out, [x] + params, gs)
            return call
        return {"fused": run(True), "torch under autocast": run(False)}
    st = {f"h.{s}.{k}": v for s, h in enumerate(heads) for k, v in h.state_dict(keep_vars=True).items()}
    hd = part_seg_oracle.heads_from_state(st, "h", len(num_parts))

    def fused():
        out = partseg.multi_shape_heads_forward(heads, x)
        torch.autograd.grad(out, [x] + params, gs)

    def torch_heads(tf32):
        def run():
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            out = part_seg_oracle.part_seg_heads(x, hd, True)
            torch.autograd.grad(out, [x] + params, gs)
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cuda.matmul.allow_tf32 = False
        return run
    return {"fused": fused, "torch tf32 off": torch_heads(False), "torch tf32 on": torch_heads(True)}


def model_arms(dataset, B, N, dev, amp=None):
    cfg = bb.model_config("multi_part_segmentation", "adaptive_weight", dataset=dataset,
                          adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1, reduction="avg"))
    torch.manual_seed(0)
    model, criterion = bb.build_multi_part_segmentation(cfg)
    model.init_weights()
    model = model.to(dev).train()
    d = synth.make_cloud_batch(B, N, cfg.input_features_dim, 5)
    xyz, mask, feats = d["xyz"].to(dev), d["mask"].to(dev), d["features"].to(dev)
    lab = synth.make_part_labels(B, N, cfg.num_parts, 6)
    pl, sl = lab["points_labels"].to(dev), lab["shape_labels"].to(dev)
    eligible = partseg.fused_eligible
    opt = torch.optim.SGD(model.parameters(), lr=B / 16 * 0.002, momentum=0.98, weight_decay=0.001)
    scaler = torch.amp.GradScaler("cuda") if amp == torch.float16 else None

    def step(fused):
        def run():
            partseg.fused_eligible = eligible if fused else (lambda heads, x: False)
            try:
                model.zero_grad(set_to_none=True)
                if amp is None:
                    criterion(model(xyz, mask, feats), pl, sl).backward()
                    return
                with torch.autocast("cuda", dtype=amp):       # tools/train_synth.py --amp
                    loss = criterion(model(xyz, mask, feats), pl, sl)
                if scaler is None:
                    loss.backward()
                    opt.step()
                else:
                    scaler.scale(loss).backward()
                    scaler.step(opt)
                    scaler.update()
            finally:
                partseg.fused_eligible = eligible
        return run
    if amp is None:
        return {"fused head": step(True), "torch head (tf32 off)": step(False)}
    return {"fused head": step(True), "torch head (autocast)": step(False)}


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def compare(title, arms, iters, rounds):
    for fn in arms.values():       # warm-up: library load, allocator, cuDNN algorithm choice
        fn()
        fn()
    torch.cuda.synchronize()
    peak = {}
    for k, fn in arms.items():     # each arm's own working memory: peak over one call above what it started with
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        peak[k] = (torch.cuda.max_memory_allocated() - base) / 2**20
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn, iters))
    base = statistics.median(res[next(iter(arms))])
    print(title)
    for k, v in res.items():
        med = statistics.median(v)
        print(f"  {k:24s} {med:8.3f} ms  [{min(v):.3f}..{max(v):.3f}]  x{med / base:.2f} of the first arm  "
              f"peak +{peak[k]:.0f} MB")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-model", action="store_true")
    ap.add_argument("--dtype", default="fp32", choices=["fp32", "bf16", "fp16"])
    a = ap.parse_args()
    amp = {"fp32": None, "bf16": torch.bfloat16, "fp16": torch.float16}[a.dtype]
    dev = torch.device("cuda")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    print("card:", card())
    for ds, B, N in SHAPES:
        num_parts = bb.PART_DATASETS[ds]["num_parts"]
        compare(f"head fwd+bwd {a.dtype}, {ds}: B={B} N={N} S={len(num_parts)} C=72 (ms per call)",
                head_arms(B, N, num_parts, dev, amp), a.iters, a.rounds)
    if not a.no_model:
        for ds, B, N in SHAPES:
            compare(f"whole-model training step {a.dtype}, {ds}: B={B} N={N} width 144 AdaptiveWeight (ms per step)",
                    model_arms(ds, B, N, dev, amp), max(2, a.iters // 5), max(3, a.rounds - 2))


if __name__ == "__main__":
    main()
