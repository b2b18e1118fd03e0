"""Third-generation PseudoGrid backward (csrc/pg.cu pg3_bwd_kernel: per-kernel-point sums U = h^T g on the tensor
cores with 3xTF32, d/dWk accumulated in registers) against the second-generation kernel (CL3D_PG_V2=1) on the same
inputs and the SAME transposed lists, and both against a float64 evaluation of the same sums.  Same terms and the
same influences; the sums are regrouped, so the comparison is to rounding, not bit for bit."""
import os
from contextlib import contextmanager

import pytest
import torch

from closerlook3d_b200 import ops, synth

pytestmark = pytest.mark.gpu

NKP_MAX = 16


@contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def _case(cuda, B, N, K, C, nkp, seed, thin_mask=False):
    d = synth.make_cloud_batch(B, N, C, seed)
    g = {k: v.to(cuda) for k, v in d.items()}
    if thin_mask:   # masked points are nobody's neighbour: their transposed lists are empty
        g["mask"] = g["mask"] * (torch.arange(N, device=cuda) % 3 != 0).to(g["mask"].dtype)[None, :]
    r = synth.ball_radius(N, K)
    idx, _, ncount = ops.ball_query(g["xyz"], g["xyz"], g["mask"], g["mask"], r, K, want_mask=False)
    gen = torch.Generator().manual_seed(seed + 1)
    kpts = (torch.rand(nkp, 3, generator=gen) - 0.5) * 0.8 * r
    kpts[0] = 0
    wk = torch.randn(nkp, C, generator=gen)
    gout = torch.randn(B, C, N, device=cuda, generator=torch.Generator(device=cuda).manual_seed(5))
    off, ent = ops.build_csr(idx, ncount, N)
    return dict(g=g, r=r, idx=idx, ncount=ncount, kpts=kpts.to(cuda), wk=wk.to(cuda), gout=gout, off=off, ent=ent,
                feat_pm=ops.to_point_major(g["features"]), gpm=ops.to_point_major(gout), extent=0.4 * r,
                B=B, N=N, K=K, C=C, nkp=nkp)


def _bwd(c, influence):
    xyz = c["g"]["xyz"]
    gf, gw = ops.agg_bwd(ops.FAM_PSEUDOGRID, ops.REDUCE["sum"], c["gpm"], c["feat_pm"], xyz, xyz, c["ncount"], c["off"],
                         c["ent"], c["kpts"], c["wk"], c["C"], c["N"], c["K"], c["r"], 0, 1, c["nkp"], c["extent"],
                         influence)
    torch.cuda.synchronize()
    return gf, gw


def _f64(c, influence):
    """d/df and d/dWk in float64 from the fp32 relative positions (gather / scatter-add of oracle.f64_ext)"""
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
    w = torch.einsum("bmkp,pc->bcmk", h, c["wk"].double())
    g64 = c["gout"].double()
    gf = f64_ext.group_points_grad(w * g64[..., None], idx, c["N"])
    fj = f64_ext.group_points(c["g"]["features"].double(), idx)                  # (B,C,M,K)
    gw = torch.einsum("bmkp,bcmk->pc", h, fj * g64[..., None])
    return gf, gw


def _err(x, ref):
    return float((x.double() - ref.double()).abs().max()) / max(1.0, float(ref.abs().max()))


CASES = [  # B, N, K, C, nkp, influence, thin mask
    (2, 3000, 26, 72, 15, 0, False), (3, 1500, 16, 36, 15, 0, False), (2, 2100, 40, 128, 15, 0, False),
    (2, 1200, 16, 72, 15, 1, False), (8, 4000, 26, 72, 15, 0, False),
    (2, 1500, 16, 8, 15, 0, False), (2, 1500, 40, 72, 16, 0, False), (2, 1500, 16, 72, 1, 0, False),
    (2, 1500, 40, 36, 16, 1, False), (2, 3000, 26, 72, 15, 0, True), (2, 1500, 16, 66, 15, 0, False),
]


@pytest.mark.parametrize("B,N,K,C,nkp,influence,thin", CASES)
@pytest.mark.parametrize("max_grid", [0, 5])
def test_pg_v3_matches_v2_and_f64(cuda, B, N, K, C, nkp, influence, thin, max_grid):
    c = _case(cuda, B, N, K, C, nkp, 91 + N + C, thin)
    if thin:
        assert int((c["off"][:, 1:] == c["off"][:, :-1]).sum()) > N // 4   # centre points with empty lists
    if K > 32:
        assert int((c["off"][:, 1:] - c["off"][:, :-1]).max()) > 32        # several batches per centre point
    grid = dict(CL3D_TEST_MAX_GRID=max_grid) if max_grid else {}            # 5 CTAs: every CTA loops over many tiles
    with env(**grid):
        with env(CL3D_PG_V2=1):
            f2, w2 = _bwd(c, influence)
        f3, w3 = _bwd(c, influence)
        f3b, w3b = _bwd(c, influence)
    assert torch.equal(f3, f3b) and torch.equal(w3, w3b), "two runs of the same grid differ"
    assert _err(f3, f2) <= 5e-6, f"d/df: v3 differs from v2 by {_err(f3, f2):.2e}"
    assert _err(w3, w2) <= 2e-5, f"d/dWk: v3 differs from v2 by {_err(w3, w2):.2e}"
    rf, rw = _f64(c, influence)
    e2 = (_err(f2, rf), _err(w2, rw))
    e3 = (_err(f3, rf), _err(w3, rw))
    print(f"float64 reference: v2 d/df {e2[0]:.2e} d/dWk {e2[1]:.2e} | v3 d/df {e3[0]:.2e} d/dWk {e3[1]:.2e}")
    assert max(e2) <= 5e-6, f"v2 (d/df, d/dWk) against float64: {e2}"
    assert e3[1] <= 5e-6, f"d/dWk: default dispatch differs from float64 by {e3[1]:.2e}"
    # the thin-mask case's d/df error follows the atomic order of its transposed lists: 1.3e-6 to 4.8e-6 measured
    if (B, N, K, C, nkp, influence, thin) in CASES[:5]:
        assert e3[0] <= 5e-6, f"d/df: default dispatch differs from float64 by {e3[0]:.2e}"
    assert e3[0] <= max(3 * e2[0], 2e-6) and e3[1] <= max(3 * e2[1], 5e-6), f"v3 {e3} against v2 {e2}"


def test_pg_v3_is_what_runs(cuda):
    """the shapes above take the third-generation kernel unless CL3D_PG_V2 is set: its d/dWk is not v2's bits"""
    c = _case(cuda, 2, 3000, 26, 72, 15, 7)
    with env(CL3D_PG_V2=1):
        _, w2 = _bwd(c, 0)
    _, w3 = _bwd(c, 0)
    assert not torch.equal(w2, w3)
