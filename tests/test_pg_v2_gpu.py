"""Second-generation PseudoGrid kernels (csrc/pg.cu: float4 lanes, packed fp32x2 FMA, compiled (h, weight-row)
entry lists, hardware square root) against the first-generation ones (csrc/agg.cu, IEEE square root, dense sums)
on the same inputs and the SAME transposed lists.  Same terms; the influences differ by the square-root
approximation (2^-22 relative), so the comparison is to rounding, not bit for bit."""
import os

import pytest
import torch

from closerlook3d_b200 import ops, synth

pytestmark = pytest.mark.gpu


def _inputs(cuda, B, N, K, C, seed):
    d = synth.make_cloud_batch(B, N, C, seed)
    g = {k: v.to(cuda) for k, v in d.items()}
    r = synth.ball_radius(N, K)
    idx, _, ncount = ops.ball_query(g["xyz"], g["xyz"], g["mask"], g["mask"], r, K, want_mask=False)
    gen = torch.Generator().manual_seed(seed + 1)
    kpts = (torch.rand(15, 3, generator=gen) - 0.5) * 0.8 * r
    kpts[0] = 0
    wk = torch.randn(15, C, generator=gen)
    return g, r, idx, ncount, kpts.to(cuda), wk.to(cuda)


@pytest.mark.parametrize("B,N,K,C,influence", [(2, 3000, 26, 72, 0), (3, 1500, 16, 36, 0), (2, 2100, 40, 128, 0),
                                               (2, 1200, 16, 72, 1), (8, 4000, 26, 72, 0)])
def test_pg_v2_matches_v1(cuda, B, N, K, C, influence):
    g, r, idx, ncount, kpts, wk = _inputs(cuda, B, N, K, C, 77 + N)
    extent = 0.4 * r
    feat_pm = ops.to_point_major(g["features"])
    gpm = ops.to_point_major(torch.randn(B, C, N, device=cuda, generator=torch.Generator(device=cuda).manual_seed(5)))
    off, ent = ops.build_csr(idx, ncount, N)

    def both():
        agg, part = ops.agg_fwd(ops.FAM_PSEUDOGRID, ops.REDUCE["sum"], feat_pm, g["xyz"], g["xyz"], idx, ncount, kpts, wk,
                                C, r, 0, 1, 15, extent, influence)
        gf, pg = ops.agg_bwd(ops.FAM_PSEUDOGRID, ops.REDUCE["sum"], gpm, feat_pm, g["xyz"], g["xyz"], ncount, off, ent,
                             kpts, wk, C, N, K, r, 0, 1, 15, extent, influence)
        torch.cuda.synchronize()
        return agg, part, gf, pg

    os.environ["CL3D_PG_V1"] = "1"
    try:
        a1, p1, g1, w1 = both()
    finally:
        del os.environ["CL3D_PG_V1"]
    a2, p2, g2, w2 = both()
    for x1, x2, what in ((g1, g2, "d/df"), (w1, w2, "d/dWk"), (a1, a2, "forward")):
        err = float((x1 - x2).abs().max()) / max(1.0, float(x1.abs().max()))
        assert err <= 5e-6, f"{what}: v2 differs from v1 by {err:.2e}"
    # BatchNorm partial moments (tile sizes are the same: 32 queries): counts, and the sums and sums of squared
    # deviations over the tiles
    (n1, s1, q1), (n2, s2, q2) = ops.bn_partial_moments(p1), ops.bn_partial_moments(p2)
    assert torch.equal(n1, n2)
    for x1, x2 in ((s1.sum(0), s2.sum(0)), (q1.sum(0), q2.sum(0))):
        assert float((x1 - x2).abs().max()) <= 1e-5 * max(1.0, float(x1.abs().max()))
