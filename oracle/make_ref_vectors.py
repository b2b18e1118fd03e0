#!/usr/bin/env python
"""Record what the UNMODIFIED reference python modules compute for the oracle pins of tests/test_oracle_cpu.py
(operator level) and tests/test_model_cpu.py (whole networks), as tests/golden/ref_*.pt.

TEST INFRASTRUCTURE ONLY.  Run where a reference checkout exists (CL3D_REFERENCE, see oracle/ref_loader.py):

    python -m oracle.make_ref_vectors

Inputs are the seeded synthetic clouds of closerlook3d_b200.synth, so only the reference's parameters, outputs and
gradients are stored; the tests rebuild the inputs and compare the oracle against these vectors.
"""
import copy
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the case tables live with the tests

from closerlook3d_b200 import synth  # noqa: E402
from oracle import ext, ref_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def plain(d):
    """EasyDict -> nested plain dict (picklable without the reference tree)"""
    return {k: plain(v) if isinstance(v, dict) else v for k, v in d.items()}


def pack(tensors):
    """{name: tensor} -> one flat tensor per dtype + the table to cut it apart (a zip record per tensor would cost
    more than the numbers themselves)"""
    table, flat = [], {}
    for k, t in tensors.items():
        dt = str(t.dtype)
        table.append((k, tuple(t.shape), dt))
        flat.setdefault(dt, []).append(t.detach().reshape(-1))
    return {"table": table, "flat": {dt: torch.cat(v) for dt, v in flat.items()}}


def unpack(p):
    out, off = {}, {}
    for k, shape, dt in p["table"]:
        n = 1
        for d in shape:
            n *= d
        o = off.get(dt, 0)
        out[k] = p["flat"][dt][o:o + n].reshape(shape).clone()
        off[dt] = o + n
    return out


def sample(t, n=256):
    """(flat indices, values) of a fixed seeded sample of at most n elements: keeps each file under 1 MB"""
    flat = t.reshape(-1)
    idx = torch.arange(flat.numel()) if flat.numel() <= n else \
        torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:n].sort().values
    return idx, flat[idx].clone()


def la_vectors():
    from test_oracle_cpu import LIVE_CASES, LA_SHAPE, live_case_id
    ns = ref_loader.load()
    B, N, K, C = LA_SHAPE
    for la_type, over in LIVE_CASES:
        torch.manual_seed(1)
        cfg = ref_loader.make_config(la_type, **over)
        r = synth.ball_radius(N, K)
        ref = ns.lao.LocalAggregation(C, C, r, K, cfg)
        sd = copy.deepcopy(ref.state_dict())
        d = synth.make_cloud_batch(B, N, C, 9)
        f = d["features"].clone().requires_grad_(True)
        out = ref(d["xyz"], d["xyz"], d["mask"], d["mask"], f)
        out.sum().backward()
        path = os.path.join(OUT, f"ref_la_{live_case_id(la_type, over)}.pt")
        torch.save({"la_type": la_type, "overrides": over, "cfg": plain(cfg), "state_dict": sd,
                    "out": out.detach(), "grad_features": f.grad}, path)
        print(path, os.path.getsize(path))


def model_vectors():
    import importlib
    from test_model_cpu import MODEL_CASES, ref_cfg, inputs, model_case_id
    ref_loader.load()
    build = importlib.import_module("models.build")
    for task, la, over in MODEL_CASES:
        cfg = ref_cfg(ref_loader.make_config(la, **over), task)
        torch.manual_seed(5)
        ref = (build.ClassificationModel if task == "classification" else build.SceneSegmentationModel)(
            cfg, cfg.backbone, cfg.head, cfg.num_classes, cfg.input_features_dim, cfg.radius, cfg.sampleDl,
            cfg.nsamples, cfg.npoints, cfg.width, cfg.depth, cfg.bottleneck_ratio)
        ref.init_weights()
        for m in ref.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        sd = copy.deepcopy(ref.state_dict())
        xyz, mask, feats = inputs(cfg.input_features_dim)
        ref.train()
        f = feats.clone().requires_grad_(True)
        out = ref(xyz, mask, f)
        g = torch.randn(out.shape, generator=torch.Generator().manual_seed(1))
        (out * g).sum().backward()
        sd_after = ref.state_dict()
        path = os.path.join(OUT, f"ref_model_{model_case_id(task, la)}.pt")
        grads = {n: sample(p.grad) for n, p in ref.named_parameters()}
        torch.save({"cfg": plain(cfg), "state_dict": pack(sd), "out": out.detach(), "grad_features": f.grad,
                    "grad_index": pack({n: i for n, (i, _) in grads.items()}),
                    "grad_params": pack({n: v for n, (_, v) in grads.items()}),
                    "running": pack({k: v for k, v in sd_after.items() if k.endswith(("running_mean", "running_var"))})},
                   path)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    la_vectors()
    model_vectors()
