#!/usr/bin/env python
"""Record what the UNMODIFIED reference multi-part segmentation network and criterion compute, for the pins of
tests/test_part_seg_cpu.py, as tests/golden/ref_model_multi_part_segmentation_<la>.pt.

TEST INFRASTRUCTURE ONLY.  Run where a reference checkout exists (CL3D_REFERENCE, see oracle/ref_loader.py):

    python -m oracle.make_part_seg_vectors

The small test network of tests/test_part_seg_cpu.py (its own case list), seeded clouds from
closerlook3d_b200.synth and labels from synth.make_part_labels; the storage format is that of
oracle/make_ref_vectors.py (pack / unpack / sample).
"""
import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the case table lives with the tests

from oracle import ref_loader  # noqa: E402
from oracle.make_ref_vectors import OUT, pack, plain, sample  # noqa: E402


def part_seg_vectors():
    import importlib
    from test_part_seg_cpu import PART_CASES, part_ref_cfg, part_inputs, PART_SEED
    ref_loader.load()
    build = importlib.import_module("models.build")
    for la, over in PART_CASES:
        cfg = part_ref_cfg(ref_loader.make_config(la, **over))
        torch.manual_seed(7)
        np.random.seed(7)    # PseudoGrid's kernel-point dispositions (models/utlis.py) draw from numpy
        ref, criterion = build.build_multi_part_segmentation(cfg)
        ref.init_weights()
        for m in ref.modules():   # non-trivial BatchNorm affine parameters
            if isinstance(m, torch.nn.BatchNorm1d):
                with torch.no_grad():
                    m.weight.uniform_(0.5, 1.5)
                    m.bias.uniform_(-0.2, 0.2)
        sd = copy.deepcopy(ref.state_dict())
        xyz, mask, feats, labels = part_inputs(cfg)
        ref.train()
        f = feats.clone().requires_grad_(True)
        out = ref(xyz, mask, f)
        loss = criterion(out, labels["points_labels"], labels["shape_labels"])
        loss.backward()
        sd_after = ref.state_dict()
        grads = {n: sample(p.grad) for n, p in ref.named_parameters() if p.grad is not None}
        path = os.path.join(OUT, f"ref_model_multi_part_segmentation_{la}.pt")
        torch.save({"cfg": plain(cfg), "state_dict": pack(sd), "seed": PART_SEED,
                    "out": pack({str(s): o.detach() for s, o in enumerate(out)}), "loss": loss.detach(),
                    "grad_features": f.grad,
                    "grad_index": pack({n: i for n, (i, _) in grads.items()}),
                    "grad_params": pack({n: v for n, (_, v) in grads.items()}),
                    "running": pack({k: v for k, v in sd_after.items() if k.endswith(("running_mean", "running_var"))})},
                   path)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    part_seg_vectors()
