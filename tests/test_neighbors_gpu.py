"""GPU parity: neighbour search + layout + compat gather, through the C ABI, against the oracle
(oracle/cl3d_oracle.c).  Index work is compared BIT-EXACT."""
import math

import pytest
import torch

from closerlook3d_b200 import synth

pytestmark = pytest.mark.gpu


def _cloud(B, N, seed, pad=True, kind="cube"):
    d = synth.make_cloud_batch(B, N, 8, seed, pad=pad)
    xyz = d["xyz"]
    g = torch.Generator().manual_seed(seed + 17)
    if kind == "clustered":  # dense blobs -> neighbourhoods with far more than 3K points
        c = torch.rand(B, 4, 3, generator=g)
        which = torch.randint(0, 4, (B, N), generator=g)
        xyz = c[torch.arange(B)[:, None], which] + 0.02 * torch.randn(B, N, 3, generator=g)
    elif kind == "lattice":  # exact distance ties and duplicates
        xyz = (torch.randint(0, 6, (B, N, 3), generator=g).float() * 0.125)
    elif kind == "sheet":  # degenerate extent along z
        xyz[..., 2] = 0.5
    xyz = xyz.contiguous()
    mask = d["mask"]
    # padded rows must duplicate valid rows (dataset convention)
    for b in range(B):
        nv = int(mask[b].sum())
        if nv < N:
            src = torch.randint(0, nv, (N - nv,), generator=g)
            xyz[b, nv:] = xyz[b, src]
    return xyz.contiguous(), mask


CASES = [
    # (B, N, M, K, radius or None, kind, algo) ; algo 0 auto, 1 brute, 2 grid
    (2, 1024, 1024, 16, None, "cube", 0),
    (2, 1024, 1024, 16, None, "cube", 2),
    (3, 777, 777, 9, None, "cube", 2),
    (3, 3000, 3000, 26, None, "cube", 0),
    (3, 3000, 3000, 26, None, "cube", 1),
    (2, 4096, 1000, 31, 0.2, "cube", 0),          # strided: fewer queries than supports
    (2, 2500, 2500, 8, 0.3, "cube", 2),            # cnt >> 3K everywhere: overwrite rule + candidate overflow
    (2, 3000, 3000, 16, 0.08, "clustered", 2),     # blobs: overflow fallback to index-order scan
    (2, 2048, 2048, 16, 0.126, "lattice", 2),      # ties in d2, duplicate points
    (2, 2048, 2048, 16, 0.126, "lattice", 1),
    (2, 3000, 3000, 12, 0.1, "sheet", 2),
    (1, 5, 5, 4, 0.5, "cube", 0),                  # tiny
    (1, 5, 5, 4, 0.5, "cube", 2),
    (2, 3000, 3000, 40, 0.02, "cube", 2),          # almost empty balls: cnt < K, cyclic padding
    (2, 15000, 15000, 16, 0.03, "cube", 2),        # 34^3 = 39304 cells > kFusedGridCells: cell counters in global memory
    (8, 15000, 15000, 26, None, "cube", 0),        # BASELINE c3 shape
]


@pytest.mark.parametrize("B,N,M,K,radius,kind,algo", CASES)
def test_ball_query_bit_exact(cuda, oracle_ext, B, N, M, K, radius, kind, algo):
    from closerlook3d_b200 import ops
    xyz, mask = _cloud(B, N, 100 + N + K, kind=kind)
    r = synth.ball_radius(N, K) if radius is None else radius
    if M == N:
        q, qm = xyz, mask
    else:
        g = torch.Generator().manual_seed(5)
        q = (xyz[:, :M] + 0.01 * torch.randn(B, M, 3, generator=g)).contiguous()
        qm = torch.ones(B, M, dtype=torch.int32)
        qm[:, M - M // 10:] = 0
    ref_idx, ref_mask = oracle_ext.masked_ordered_ball_query(q, xyz, qm, mask, r, K)
    idx, idx_mask, ncount = ops.ball_query(q.to(cuda), xyz.to(cuda), qm.to(cuda), mask.to(cuda), r, K, algo=algo)
    torch.cuda.synchronize()
    assert torch.equal(idx.cpu(), ref_idx), f"idx mismatch: {(idx.cpu() != ref_idx).sum().item()} entries"
    assert torch.equal(idx_mask.cpu(), ref_mask)
    # ncount = number of slots counted by the avg/sum reductions (feature_mask of the reference)
    fm = ref_mask + (1 - qm[:, :, None])
    assert torch.equal(ncount.cpu(), fm.sum(-1).to(torch.int32))
    assert torch.equal((torch.arange(K)[None, None, :] < ncount.cpu()[:, :, None]).to(torch.int32), fm)


def test_ball_query_query_outside_bbox(cuda, oracle_ext):
    from closerlook3d_b200 import ops
    xyz, mask = _cloud(2, 3000, 3)
    g = torch.Generator().manual_seed(9)
    q = (torch.rand(2, 500, 3, generator=g) * 3 - 1).contiguous()  # many queries far outside the unit cube
    qm = torch.ones(2, 500, dtype=torch.int32)
    # keep only queries with >= 1 neighbour (cnt == 0 is undefined behaviour in the reference)
    ref_idx, ref_mask = oracle_ext.masked_ordered_ball_query(q, xyz, qm, mask, 0.3, 16)
    idx, idx_mask, _ = ops.ball_query(q.to(cuda), xyz.to(cuda), qm.to(cuda), mask.to(cuda), 0.3, 16, algo=2)
    has = ref_mask.sum(-1) > 0
    assert torch.equal(idx.cpu()[has], ref_idx[has])
    assert torch.equal(idx_mask.cpu(), ref_mask)


@pytest.mark.parametrize("B,N,M", [(2, 1000, 3000), (3, 4096, 15000), (1, 7, 5)])
def test_nearest_query_bit_exact(cuda, oracle_ext, B, N, M):
    from closerlook3d_b200 import ops
    xyz, mask = _cloud(B, N, 40 + N)
    g = torch.Generator().manual_seed(11)
    q = torch.rand(B, M, 3, generator=g)
    qm = torch.ones(B, M, dtype=torch.int32)
    qm[:, M - M // 7:] = 0
    ref_idx, ref_mask = oracle_ext.masked_nearest_query(q, xyz, qm, mask)
    idx, idx_mask = ops.nearest_query(q.to(cuda), xyz.to(cuda), qm.to(cuda), mask.to(cuda))
    assert torch.equal(idx.cpu(), ref_idx[..., 0])
    assert torch.equal(idx_mask.cpu(), ref_mask[..., 0])


@pytest.mark.parametrize("offset,spread", [(0.0, 1.0), (25.0, 1.0), (0.0, 3.0)])
def test_nearest_query_grid_surface_cloud(cuda, oracle_ext, offset, spread):
    # the cell-ring walk (N > 2048) on surface-like supports (most cells empty: several rings per query), queries
    # well outside the supports' bounding box (spread 3), S3DIS-like coordinates far from the origin (offset 25),
    # exact duplicates among the supports (distance ties -> first index), masked tail, and against the tile scan
    from closerlook3d_b200 import ops
    B, N, M = 2, 6000, 9000
    g = torch.Generator().manual_seed(5)
    d = torch.randn(B, N, 3, generator=g)
    xyz = d / d.norm(dim=-1, keepdim=True) * (0.5 + 0.01 * torch.randn(B, N, 1, generator=g)) + offset
    xyz[:, 100:200] = xyz[:, 300:400]                      # duplicated points
    mask = torch.ones(B, N, dtype=torch.int32)
    mask[1, N - 500:] = 0
    q = (torch.rand(B, M, 3, generator=g) - 0.5) * 1.2 * spread + offset
    q[:, :300] = xyz[:, 100:400]                           # queries ON support points (distance 0, tied duplicates)
    qm = torch.ones(B, M, dtype=torch.int32)
    ref_idx, ref_mask = oracle_ext.masked_nearest_query(q, xyz.contiguous(), qm, mask)
    idx, idx_mask = ops.nearest_query(q.to(cuda), xyz.contiguous().to(cuda), qm.to(cuda), mask.to(cuda))
    assert torch.equal(idx.cpu(), ref_idx[..., 0])
    assert torch.equal(idx_mask.cpu(), ref_mask[..., 0])
    import os
    os.environ["CL3D_NN_BRUTE"] = "1"
    try:
        idx2, _ = ops.nearest_query(q.to(cuda), xyz.contiguous().to(cuda), qm.to(cuda), mask.to(cuda))
    finally:
        del os.environ["CL3D_NN_BRUTE"]
    assert torch.equal(idx2, idx)


def test_csr_is_transpose_of_idx(cuda, oracle_ext):
    from closerlook3d_b200 import ops
    B, N, K = 3, 2500, 16
    xyz, mask = _cloud(B, N, 77)
    r = synth.ball_radius(N, K)
    idx, _, ncount = ops.ball_query(xyz.to(cuda), xyz.to(cuda), mask.to(cuda), mask.to(cuda), r, K)
    off, ent = ops.build_csr(idx, ncount, N)
    idx, ncount, off, ent = idx.cpu(), ncount.cpu(), off.cpu(), ent.cpu()
    for b in range(B):
        assert off[b, 0] == 0
        total = int(ncount[b].sum())
        assert off[b, N] == total
        e = ent[b, :total].long()
        q, k = e // K, e % K
        assert bool((k < ncount[b][q]).all())
        tgt = idx[b][q, k].long()
        # entries are grouped by target in off order
        expect_tgt = torch.repeat_interleave(torch.arange(N), (off[b, 1:] - off[b, :-1]).long())
        assert torch.equal(tgt, expect_tgt)
        assert e.unique().numel() == total  # every counted slot exactly once


@pytest.mark.parametrize("B,C,N", [(2, 66, 1000), (3, 72, 4097), (1, 144, 33), (2, 3, 50)])
def test_layout_roundtrip(cuda, B, C, N):
    from closerlook3d_b200 import ops
    x = torch.randn(B, C, N, device=cuda)
    pm = ops.to_point_major(x)
    Cp = ops.padded_channels(C)
    assert pm.shape == (B, N, Cp)
    assert torch.equal(pm[:, :, :C], x.transpose(1, 2))
    assert bool((pm[:, :, C:] == 0).all())
    assert torch.equal(ops.to_channel_major(pm, C), x)


def test_group_points_and_grad(cuda, oracle_ext):
    from closerlook3d_b200 import ops
    B, C, N, M, K = 2, 10, 300, 200, 7
    g = torch.Generator().manual_seed(3)
    pts = torch.randn(B, C, N, generator=g)
    idx = torch.randint(0, N, (B, M, K), generator=g, dtype=torch.int32)
    go = torch.randn(B, C, M, K, generator=g)
    out = ops.group_points(pts.to(cuda), idx.to(cuda))
    assert torch.equal(out.cpu(), oracle_ext.group_points(pts, idx))
    gp = ops.group_points_grad(go.to(cuda), idx.to(cuda), N)
    ref = oracle_ext.group_points_grad(go, idx, N)
    # fp32 atomics: summation order differs (as in the reference itself) -> tolerance, not bit equality
    assert torch.allclose(gp.cpu(), ref, rtol=0, atol=1e-5)
