"""Ball query with ONE tensor as query and support set (and one mask tensor as both masks), as every non-strided layer
calls it: the grid kernel then walks the queries in cell order.  Index work is compared BIT-EXACT against the oracle
(oracle/cl3d_oracle.c); the transposed lists of the ranked search must be the transpose of idx."""
import pytest
import torch

from closerlook3d_b200 import synth
from test_neighbors_gpu import CASES, _cloud

pytestmark = pytest.mark.gpu

# every square case that reaches the grid kernel: cube, lattice ties, clustered overflow, sheet, almost-empty balls,
# the c3 shape; _cloud pads the tails of the clouds (mask zero, rows duplicating valid points)
SQUARE = [c for c in CASES if c[1] == c[2] and c[6] != 1]


def _check_reference(oracle_ext, xyz, mask, r, K, idx, idx_mask, ncount):
    ref_idx, ref_mask = oracle_ext.masked_ordered_ball_query(xyz, xyz, mask, mask, r, K)
    assert torch.equal(idx.cpu(), ref_idx), f"idx mismatch: {(idx.cpu() != ref_idx).sum().item()} entries"
    if idx_mask is not None:
        assert torch.equal(idx_mask.cpu(), ref_mask)
    fm = ref_mask + (1 - mask[:, :, None])
    assert torch.equal(ncount.cpu(), fm.sum(-1).to(torch.int32))


def _check_transpose(idx, ncount, off, ent, all_slots=False):
    """per support point, the list holds exactly the counted slots (q, k) whose idx is that point"""
    idx, ncount, off, ent = idx.cpu(), ncount.cpu(), off.cpu(), ent.cpu()
    B, M, K = idx.shape
    N = off.shape[1] - 1
    for b in range(B):
        counted = torch.full((M,), K, dtype=torch.int32) if all_slots else ncount[b]
        total = int(counted.sum())
        assert off[b, 0] == 0 and off[b, N] == total
        e = ent[b, :total].long()
        q, k = e // K, e % K
        assert bool((k < counted[q]).all())
        expect_tgt = torch.repeat_interleave(torch.arange(N), (off[b, 1:] - off[b, :-1]).long())
        assert torch.equal(idx[b][q, k].long(), expect_tgt)
        assert e.unique().numel() == total


@pytest.mark.parametrize("B,N,M,K,radius,kind,algo", SQUARE)
def test_same_tensor_bit_exact(cuda, oracle_ext, B, N, M, K, radius, kind, algo):
    from closerlook3d_b200 import ops
    xyz, mask = _cloud(B, N, 100 + N + K, kind=kind)
    r = synth.ball_radius(N, K) if radius is None else radius
    x, m = xyz.to(cuda), mask.to(cuda)
    idx, idx_mask, ncount = ops.ball_query(x, x, m, m, r, K, algo=algo)
    _check_reference(oracle_ext, xyz, mask, r, K, idx, idx_mask, ncount)


@pytest.mark.parametrize("B,N,M,K,radius,kind,algo", SQUARE)
@pytest.mark.parametrize("csr", ["counted", "all"])
def test_same_tensor_ranked_lists(cuda, oracle_ext, B, N, M, K, radius, kind, algo, csr):
    from closerlook3d_b200 import ops
    xyz, mask = _cloud(B, N, 100 + N + K, kind=kind)
    r = synth.ball_radius(N, K) if radius is None else radius
    x, m = xyz.to(cuda), mask.to(cuda)
    idx, _, ncount, (off, ent) = ops.ball_query(x, x, m, m, r, K, want_mask=False, algo=algo, csr=csr)
    _check_reference(oracle_ext, xyz, mask, r, K, idx, None, ncount)
    _check_transpose(idx, ncount, off, ent, all_slots=csr == "all")


def test_same_points_other_mask_tensor(cuda, oracle_ext):
    # same xyz pointer, equal mask values in a second tensor: the general (index-order) walk, same result
    from closerlook3d_b200 import ops
    B, N, K = 3, 5000, 26
    xyz, mask = _cloud(B, N, 8)
    r = synth.ball_radius(N, K)
    x, m = xyz.to(cuda), mask.to(cuda)
    m2 = m.clone()
    idx, idx_mask, ncount = ops.ball_query(x, x, m, m2, r, K)
    _check_reference(oracle_ext, xyz, mask, r, K, idx, idx_mask, ncount)
    idx1, idx_mask1, ncount1 = ops.ball_query(x, x, m, m, r, K)
    assert torch.equal(idx, idx1) and torch.equal(idx_mask, idx_mask1) and torch.equal(ncount, ncount1)


def test_same_tensor_graph_replay(cuda):
    # the ranked search captured in a CUDA graph, replayed on a new cloud, against an eager call on that cloud
    from closerlook3d_b200 import ops
    B, N, K = 4, 6000, 26
    r = synth.ball_radius(N, K)
    xyz0, mask0 = _cloud(B, N, 21)
    xyz1, mask1 = _cloud(B, N, 22)
    x, m = xyz0.to(cuda), mask0.to(cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.ball_query(x, x, m, m, r, K, want_mask=False, csr="counted")
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        idx, _, ncount, (off, ent) = ops.ball_query(x, x, m, m, r, K, want_mask=False, csr="counted")
    x.copy_(xyz1.to(cuda))
    m.copy_(mask1.to(cuda))
    g.replay()
    torch.cuda.synchronize()
    x2, m2 = xyz1.to(cuda), mask1.to(cuda)
    e_idx, _, e_ncount, (e_off, e_ent) = ops.ball_query(x2, x2, m2, m2, r, K, want_mask=False, csr="counted")
    assert torch.equal(idx, e_idx) and torch.equal(ncount, e_ncount) and torch.equal(off, e_off)
    _check_transpose(idx, ncount, off, ent)
