"""Deterministic synthetic point clouds of the BASELINE.json shapes (SURVEY.md section 8d).

There are no datasets in the container, so every test and benchmark uses these generators:
  xyz      = torch.rand(B, N, 3)            unit cube, fp32
  features = torch.randn(B, C, N)
  masks    : cloud b has n_valid = N - (b mod 4) * floor(0.05 N) valid rows (valid PREFIX, as the reference's
             datasets build them: datasets/ModelNet40.py:186-196, S3DIS.py:307-314); padded rows are copies
             of random valid rows
  radius   = (1.5 * K * 3 / (4 pi N)) ** (1/3)   -> expected in-ball count ~ 1.5 K
all drawn from torch.Generator().manual_seed(seed) on CPU (so the same inputs exist with or without a GPU).
"""
import math

import torch


def ball_radius(N, K):
    return float((1.5 * K * 3.0 / (4.0 * math.pi * N)) ** (1.0 / 3.0))


def make_cloud_batch(B, N, C, seed, pad=True, b_offset=0):
    """Returns dict(xyz (B,N,3) f32, mask (B,N) i32, features (B,C,N) f32) on CPU.
    b_offset shifts the cloud index used for the padding pattern (rank sharding)."""
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(B, N, 3, generator=g)
    feats = torch.randn(B, C, N, generator=g)
    mask = torch.ones(B, N, dtype=torch.int32)
    if pad:
        for b in range(B):
            n_valid = N - ((b + b_offset) % 4) * int(0.05 * N)
            if n_valid < N:
                src = torch.randint(0, n_valid, (N - n_valid,), generator=g)
                xyz[b, n_valid:] = xyz[b, src]
                feats[b, :, n_valid:] = feats[b][:, src]
                mask[b, n_valid:] = 0
    return dict(xyz=xyz.contiguous(), mask=mask.contiguous(), features=feats.contiguous())


def baseline_inputs(i, B=None, seed=None, b_offset=0):
    """Inputs of BASELINE config i (1..5); B overrides the batch (per-GPU shard)."""
    from .config import baseline_config
    t = baseline_config(i)
    B = t["B"] if B is None else B
    d = make_cloud_batch(B, t["N"], t["C"], 1000 + i if seed is None else seed, b_offset=b_offset)
    d["radius"] = ball_radius(t["N"], t["K"])
    d["nsample"] = t["K"]
    d["spec"] = t
    return d


def make_part_labels(B, N, num_parts, seed):
    """Seeded labels of a multi-part segmentation batch, on CPU: shape_labels (B,) int64 in [0, S) and
    points_labels (B,N) int64 with points_labels[b] < num_parts[shape_labels[b]]."""
    g = torch.Generator().manual_seed(seed)
    shape_labels = torch.randint(0, len(num_parts), (B,), generator=g)
    u = torch.rand(B, N, generator=g)
    limit = torch.tensor([num_parts[int(s)] for s in shape_labels], dtype=torch.float64)[:, None]
    points_labels = (u.double() * limit).long().clamp_max(limit.long() - 1)
    return dict(shape_labels=shape_labels, points_labels=points_labels)
