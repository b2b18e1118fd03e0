"""Third-generation PseudoGrid forward (csrc/pg.cu pg3_fwd_kernel: per-kernel-point sums U = h^T f on the tensor cores
with 3xTF32, then out = sum_k' Wk * U) against the second-generation kernel (CL3D_PG_V2=1) on the same inputs and
lists, and both against a float64 evaluation of the same sums.  Same terms and the same influences; the sums are
regrouped, so the comparison is to rounding, not bit for bit.  The BatchNorm partials keep their meaning: the moments
(count, sum, sum of squared deviations from the tile mean) of the output over each tile of 32 queries.  The forward takes the third generation up to 40
padded channels (C = 8, 36 below); the wider cases check that the dispatch still computes the same sums."""
import pytest
import torch

from closerlook3d_b200 import ops
from test_pg_v3_gpu import CASES, _case, _err, env

pytestmark = pytest.mark.gpu


def _fwd(c, influence):
    xyz = c["g"]["xyz"]
    agg, part = ops.agg_fwd(ops.FAM_PSEUDOGRID, ops.REDUCE["sum"], c["feat_pm"], xyz, xyz, c["idx"], c["ncount"],
                            c["kpts"], c["wk"], c["C"], c["r"], 0, 1, c["nkp"], c["extent"], influence)
    torch.cuda.synchronize()
    return agg, part


def _f64(c, influence):
    """agg (B,C,M) in float64 from the fp32 relative positions (gather of oracle.f64_ext)"""
    from oracle import f64_ext
    xyz, idx, K = c["g"]["xyz"], c["idx"], c["K"]
    sx = f64_ext.group_points(xyz.transpose(1, 2).contiguous(), idx)            # (B,3,M,K)
    dp = (sx - xyz.transpose(1, 2)[..., None]).permute(0, 2, 3, 1)               # support - query, fp32
    if influence == 1:
        h = torch.ones(*dp.shape[:3], c["nkp"], dtype=torch.float64, device=dp.device)
    else:
        dist = (dp[..., None, :].double() - c["kpts"].double()).pow(2).sum(-1).sqrt()
        h = (1.0 - dist / c["extent"]).clamp(min=0.0)                            # (B,M,K,nkp)
    h = h * (torch.arange(K, device=dp.device)[None, None, :] < c["ncount"][..., None])[..., None]
    fj = f64_ext.group_points(c["g"]["features"].double(), idx)                  # (B,C,M,K)
    return torch.einsum("bmkp,pc,bcmk->bcm", h, c["wk"].double(), fj)


def _tile_moments(agg):
    """(ntiles, 3, C) float64: count, sum and sum of squared deviations from the tile mean of agg over each tile of 32
    queries of each cloud"""
    B, C, M = agg.shape
    T = (M + 31) // 32
    present = (torch.arange(T * 32, device=agg.device) < M).view(T, 32)
    x = torch.zeros(B, C, T * 32, dtype=torch.float64, device=agg.device)
    x[..., :M] = agg.double()
    x = x.view(B, C, T, 32)
    n = present.sum(-1).double().expand(B, C, T)
    s = x.sum(-1)
    m2 = torch.where(present, (x - (s / n)[..., None]) ** 2, 0.0).sum(-1)
    return torch.stack([n, s, m2], -1).permute(0, 2, 3, 1).reshape(B * T, 3, C)   # row b * T + t


def _moments(part):
    return torch.stack(ops.bn_partial_moments(part), 1)


def _stats(part, C, count):
    rm, rv = torch.zeros(C, device=part.device), torch.ones(C, device=part.device)
    st = ops.bn_finalize(part, C, count, 1e-5, 1.0, True, rm, rv)
    return torch.stack([st[0], rv])   # mean, unbiased variance


@pytest.mark.parametrize("B,N,K,C,nkp,influence,thin", CASES)
@pytest.mark.parametrize("max_grid", [0, 1, 2, 5])   # 1 or 2 CTAs: each walks every tile of its share
def test_pg_v3_fwd_matches_v2_and_f64(cuda, B, N, K, C, nkp, influence, thin, max_grid):
    c = _case(cuda, B, N, K, C, nkp, 91 + N + C, thin)
    if K > 32:
        assert int(c["ncount"].max()) > 32                                       # several batches per query
    grid = dict(CL3D_TEST_MAX_GRID=max_grid) if max_grid else {}            # 5 CTAs: every CTA loops over many tiles
    with env(**grid):
        with env(CL3D_PG_V2=1):
            a2, p2 = _fwd(c, influence)
        a3, p3 = _fwd(c, influence)
        a3b, p3b = _fwd(c, influence)
    assert torch.equal(a3, a3b) and torch.equal(p3, p3b), "two runs of the same grid differ"
    assert _err(a3, a2) <= 1e-5, f"agg: v3 differs from v2 by {_err(a3, a2):.2e}"
    assert p3.shape == p2.shape
    m2, m3 = _moments(p2), _moments(p3)
    assert torch.equal(m3[:, 0], m2[:, 0]), "tile counts differ"
    assert _err(m3, m2) <= 1e-5, f"BatchNorm partials: v3 differs from v2 by {_err(m3, m2):.2e}"
    ref = _f64(c, influence)
    e2, e3 = _err(a2, ref), _err(a3, ref)
    mref = _tile_moments(ref)
    assert torch.equal(m3[:, 0], mref[:, 0])
    # per tile sum and sum of squares against float64 (the aggregation's error included), and the centred second
    # moment against that of the kernel's own output
    def sums(m):   # (ntiles, 2, C): sum and sum of squares
        return torch.stack([m[:, 1], m[:, 2] + m[:, 1] ** 2 / m[:, 0]], 1)

    assert torch.equal(m2[:, 0], mref[:, 0])
    ep2 = max(_err(sums(m2), sums(mref)), _err(m2[:, 2], _tile_moments(a2)[:, 2]))
    ep3 = max(_err(sums(m3), sums(mref)), _err(m3[:, 2], _tile_moments(a3)[:, 2]))
    print(f"float64 reference: agg v2 {e2:.2e} v3 {e3:.2e} | BatchNorm partials v2 {ep2:.2e} v3 {ep3:.2e}")
    assert e2 <= 5e-6, f"agg: v2 differs from float64 by {e2:.2e}"
    assert e3 <= 5e-6, f"agg: default dispatch differs from float64 by {e3:.2e}"
    assert e3 <= max(3 * e2, 2e-6), f"v3 {e3:.2e} against v2 {e2:.2e}"
    assert ep2 <= 1e-5, f"BatchNorm partials: v2 differ from float64 by {ep2:.2e}"
    assert ep3 <= 1e-5, f"BatchNorm partials: default dispatch differs from float64 by {ep3:.2e}"
    # BatchNorm statistics from the partials, as cl3d_bn_finalize merges them
    s2, s3 = _stats(p2, C, B * N), _stats(p3, C, B * N)
    assert float((s3 - s2).abs().max()) <= 1e-5 * max(1.0, float(s2.abs().max()))


def test_pg_v3_fwd_graph_replay_equals_eager(cuda):
    c = _case(cuda, 2, 3000, 26, 72, 15, 17)
    eager = _fwd(c, 0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _fwd(c, 0)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        xyz = c["g"]["xyz"]
        out = ops.agg_fwd(ops.FAM_PSEUDOGRID, ops.REDUCE["sum"], c["feat_pm"], xyz, xyz, c["idx"], c["ncount"],
                          c["kpts"], c["wk"], c["C"], c["r"], 0, 1, c["nkp"], c["extent"], 0)
    out[0].zero_()
    out[1].zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])


def test_pg_v3_fwd_dispatch(cuda):
    """up to 40 padded channels the forward takes pg3_fwd_kernel: its sums are regrouped, so its bits differ from the
    second generation's (CL3D_PG_V2=1); bench.py's default shape (S3DIS PseudoGrid: B=8, N=15000, K=26, C=72) keeps the
    second-generation forward, where it measured faster, so its bits are those of CL3D_PG_V2=1"""
    narrow = _case(cuda, 8, 15000, 26, 36, 15, 3)
    with env(CL3D_PG_V2=1):
        a2, _ = _fwd(narrow, 0)
    a3, _ = _fwd(narrow, 0)
    assert not torch.equal(a2, a3)
    assert _err(a3, a2) <= 1e-5
    c3 = _case(cuda, 8, 15000, 26, 72, 15, 3)
    with env(CL3D_PG_V2=1):
        a2, p2 = _fwd(c3, 0)
    a3, p3 = _fwd(c3, 0)
    assert torch.equal(a2, a3) and torch.equal(p2, p3)
