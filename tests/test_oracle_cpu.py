"""CPU tests (-m "not gpu"): the oracle is pinned against
  (1) the golden fixtures made by the UNMODIFIED reference python modules (tests/golden, bit-exact),
  (2) outputs and feature gradients the unmodified reference modules computed on seeded clouds
      (tests/golden/ref_la_*.pt, recorded by oracle/make_ref_vectors.py),
  (3) an independent pure-python restatement of the ball-query rule on tiny inputs + structural properties.
"""
import copy
import glob
import math
import os

import pytest
import torch

from closerlook3d_b200 import synth
from closerlook3d_b200.config import AttrDict, la_config

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "la_*.pt")))


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p)[3:-3] for p in GOLD])
def test_oracle_reproduces_reference_golden(oracle_ext, path):
    from oracle import la_oracle
    g = torch.load(path, weights_only=False)
    cfg = la_config(g["la_type"], **g["overrides"])
    orc = la_oracle.OracleLocalAggregation(oracle_ext, g["la_type"], g["C"], g["C"], g["radius"], g["K"], cfg,
                                           g["state_dict"])
    idx, idx_mask = oracle_ext.masked_ordered_ball_query(g["query_xyz"], g["support_xyz"], g["query_mask"],
                                                         g["support_mask"], g["radius"], g["K"])
    assert torch.equal(idx, g["idx"]) and torch.equal(idx_mask, g["idx_mask"])
    f = g["features"].clone().requires_grad_(True)
    out = orc(g["query_xyz"], g["support_xyz"], g["query_mask"], g["support_mask"], f)
    (out * g["grad_out"]).sum().backward()
    assert torch.equal(out.detach(), g["out"])                       # same torch ops in the same order
    assert torch.equal(f.grad, g["grad_features"])
    # parameter gradients are reductions inside torch's CPU convolution / matmul kernels, whose summation order
    # depends on the host's instruction set: equal up to fp32 reordering, not bit for bit, across machines
    for k, v in orc.grads().items():
        want = g["grad_params"]["local_aggregation_operator." + k]
        assert float((v - want).abs().max()) <= 1e-6 * max(1.0, float(want.abs().max())), k
    for k, v in orc.st.items():
        if k.endswith(("running_mean", "running_var", "num_batches_tracked")):
            assert torch.equal(v, g["state_dict_after"]["local_aggregation_operator." + k]), k


LA_SHAPE = (2, 300, 10, 24)   # B, N, K, C
LIVE_CASES = [
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="avg"))),
    ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="sum"))),
    ("adaptive_weight", dict(adaptive_weight=dict(num_mlps=2, shared_channels=2, reduction="avg"))),
    ("pointwisemlp", dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))),
    ("pseudo_grid", dict()),
    # the max reductions the fused kernels of csrc/agg_max.cu are checked against
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="max"))),
    ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="max"))),
    ("adaptive_weight", dict(adaptive_weight=dict(num_mlps=1, shared_channels=1, reduction="max"))),
]


def live_case_id(la_type, over):
    v = over.get(la_type, {})
    return "_".join([la_type] + [f"{k}-{v[k]}" for k in sorted(v)])


def _attr(d):
    return AttrDict({k: _attr(v) if isinstance(v, dict) else v for k, v in d.items()})


@pytest.mark.parametrize("la_type,over", LIVE_CASES)
def test_oracle_matches_live_reference(oracle_ext, la_type, over):
    """the oracle == what the unmodified reference modules computed on the same seeded cloud, bit for bit"""
    from oracle import la_oracle
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", f"ref_la_{live_case_id(la_type, over)}.pt"),
                   weights_only=False)
    B, N, K, C = LA_SHAPE
    cfg = _attr(g["cfg"])
    r = synth.ball_radius(N, K)
    d = synth.make_cloud_batch(B, N, C, 9)
    f2 = d["features"].clone().requires_grad_(True)
    orc = la_oracle.OracleLocalAggregation(oracle_ext, la_type, C, C, r, K, cfg, g["state_dict"])
    o2 = orc(d["xyz"], d["xyz"], d["mask"], d["mask"], f2)
    o2.sum().backward()
    assert torch.equal(g["out"], o2) and torch.equal(g["grad_features"], f2.grad)


def _py_ball_query(q, s, qm, sm, radius, K):
    """independent, literal python restatement of masked_ordered_ball_query_gpu.cu:33-95 (tiny inputs only)"""
    import numpy as np
    f32 = np.float32
    B, M, _ = q.shape
    N = s.shape[1]
    idx = torch.zeros(B, M, K, dtype=torch.int32)
    msk = torch.zeros(B, M, K, dtype=torch.int32)
    r2 = f32(radius) * f32(radius)
    for b in range(B):
        for j in range(M):
            cand = []
            min_d, min_k = r2, 0
            qx, qy, qz = (f32(v) for v in q[b, j].tolist())
            for k in range(N):
                if sm[b, k] == 0:
                    break
                x, y, z = (f32(v) for v in s[b, k].tolist())
                dx, dy, dz = f32(qx - x), f32(qy - y), f32(qz - z)
                t = f32(dy * dy)
                t = f32(np.float64(dx) * np.float64(dx) + np.float64(t))    # fma: exact product, one rounding
                t = f32(np.float64(dz) * np.float64(dz) + np.float64(t))
                if t < r2:
                    if t < min_d:
                        min_d, min_k = t, k
                    if len(cand) >= 3 * K:
                        continue
                    cand.append((t, k))
            if len(cand) >= 3 * K and min_k > cand[-1][1]:
                cand[-1] = (min_d, min_k)
            cand.sort(key=lambda e: e[0])  # python's sort is stable
            cnt = len(cand)
            for i in range(K):
                if i < cnt:
                    idx[b, j, i], msk[b, j, i] = cand[i][1], 1
                else:
                    idx[b, j, i] = cand[i % cnt][1] if cnt else 0
            if qm[b, j] == 0:
                msk[b, j] = 0
    return idx, msk


@pytest.mark.parametrize("N,K,radius", [(40, 4, 0.35), (60, 3, 0.6), (25, 8, 0.2)])
def test_c_oracle_matches_python_restatement(oracle_ext, N, K, radius):
    d = synth.make_cloud_batch(2, N, 3, 50 + N)
    idx, msk = oracle_ext.masked_ordered_ball_query(d["xyz"], d["xyz"], d["mask"], d["mask"], radius, K)
    pidx, pmsk = _py_ball_query(d["xyz"], d["xyz"], d["mask"], d["mask"], radius, K)
    assert torch.equal(idx, pidx) and torch.equal(msk, pmsk)


def test_c_oracle_ball_query_properties(oracle_ext):
    B, N, K = 3, 500, 16
    d = synth.make_cloud_batch(B, N, 3, 5)
    r = synth.ball_radius(N, K)
    xyz, mask = d["xyz"], d["mask"]
    idx, msk = oracle_ext.masked_ordered_ball_query(xyz, xyz, mask, mask, r, K)
    nbr = torch.gather(xyz, 1, idx.long().view(B, -1, 1).expand(-1, -1, 3)).view(B, N, K, 3)
    d2 = ((nbr - xyz[:, :, None, :]) ** 2).sum(-1)
    assert bool((d2[msk.bool()] < r * r * (1 + 1e-5)).all())          # every valid neighbour is in the ball
    for b in range(B):
        nv = int(mask[b].sum())
        assert int(idx[b].max()) < nv                                   # padded supports are never returned
        valid = msk[b].bool()
        dd = d2[b].clone()
        dd[~valid] = float("inf")
        cnt = valid.sum(-1)
        for j in range(0, nv, 37):                                      # sorted by distance among valid slots
            c = int(cnt[j])
            assert bool((dd[j, 1:c] >= dd[j, :c - 1] - 1e-7).all())
            assert int(idx[b, j, 0]) == j or float(d2[b, j, 0]) == 0.0  # slot 0 = nearest = the query itself
        assert bool((msk[b, nv:] == 0).all())                           # padded queries: mask cleared


def test_c_oracle_group_points_and_grad(oracle_ext):
    g = torch.Generator().manual_seed(0)
    B, C, N, M, K = 2, 5, 40, 30, 4
    pts = torch.randn(B, C, N, generator=g)
    idx = torch.randint(0, N, (B, M, K), generator=g, dtype=torch.int32)
    out = oracle_ext.group_points(pts, idx)
    ref = torch.gather(pts.unsqueeze(2).expand(-1, -1, M, -1), 3, idx.long().unsqueeze(1).expand(-1, C, -1, -1))
    assert torch.equal(out, ref)
    go = torch.randn(B, C, M, K, generator=g)
    gp = oracle_ext.group_points_grad(go, idx, N)
    ref_g = torch.zeros(B, C, N).scatter_add_(2, idx.long().view(B, 1, -1).expand(-1, C, -1), go.reshape(B, C, -1))
    assert torch.allclose(gp, ref_g, atol=1e-5)


def test_c_oracle_nearest_and_subsample_properties(oracle_ext):
    d = synth.make_cloud_batch(2, 400, 3, 8)
    xyz, mask = d["xyz"], d["mask"]
    g = torch.Generator().manual_seed(1)
    q = torch.rand(2, 100, 3, generator=g)
    qm = torch.ones(2, 100, dtype=torch.int32)
    idx, m = oracle_ext.masked_nearest_query(q, xyz, qm, mask)
    for b in range(2):
        nv = int(mask[b].sum())
        dist = ((q[b][:, None] - xyz[b][None, :nv]) ** 2).sum(-1)
        assert torch.equal(idx[b, :, 0].long(), dist.argmin(1))
    sub, sm = oracle_ext.masked_grid_subsampling(xyz, mask, 120, 0.2)
    assert sub.shape == (2, 120, 3) and sm.shape == (2, 120)
    for b in range(2):
        n = int(sm[b].sum())
        assert 0 < n <= 120 and bool((sm[b, :n] == 1).all())
        cells = torch.floor(sub[b, :n] / 0.2)
        assert len({tuple(c.tolist()) for c in cells}) >= n - 2          # one barycentre per occupied voxel
        if n < 120:                                                       # cyclic padding with true sub points
            assert torch.equal(sub[b, n:], sub[b, torch.arange(n, 120) % n])
