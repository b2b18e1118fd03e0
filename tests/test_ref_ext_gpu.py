"""GPU pins against the reference's OWN CUDA extension (oracle/_ref: the reference sources compiled unmodified
for sm_90 by oracle/build_ref.py):
  * the C restatement (oracle/cl3d_oracle.c) equals the reference kernels bit for bit  -> the oracle is pinned;
  * libcl3d equals the reference kernels bit for bit at the FULL BASELINE sizes, where the CPU oracle is slow.
Skipped when oracle/_ref has not been built (it is built in the container and travels with the snapshot)."""
import pytest
import torch

from closerlook3d_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref_ext():
    try:
        from oracle import build_ref
        return build_ref.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"oracle/_ref unavailable: {e}")


def _inputs(B, N, seed, cuda):
    d = synth.make_cloud_batch(B, N, 4, seed)
    return d, {k: v.to(cuda) for k, v in d.items()}


@pytest.mark.parametrize("B,N,K,radius", [(2, 1024, 16, None), (3, 3000, 26, None), (2, 2500, 8, 0.3), (2, 3000, 40, 0.02)])
def test_c_oracle_equals_reference_ball_query(cuda, oracle_ext, ref_ext, B, N, K, radius):
    d, g = _inputs(B, N, 60 + N + K, cuda)
    r = synth.ball_radius(N, K) if radius is None else radius
    ridx, rmask = ref_ext.masked_ordered_ball_query(g["xyz"], g["xyz"], g["mask"], g["mask"], r, K)
    oidx, omask = oracle_ext.masked_ordered_ball_query(d["xyz"], d["xyz"], d["mask"], d["mask"], r, K)
    assert torch.equal(ridx.cpu(), oidx) and torch.equal(rmask.cpu(), omask)


@pytest.mark.parametrize("cfg_index,B", [(2, 32), (3, 8), (4, 4), (5, 2)])
def test_libcl3d_equals_reference_ball_query_at_baseline_sizes(cuda, ref_ext, cfg_index, B):
    from closerlook3d_b200 import ops
    from closerlook3d_b200.config import baseline_config
    t = baseline_config(cfg_index)
    _, g = _inputs(B, t["N"], 1000 + cfg_index, cuda)
    r = synth.ball_radius(t["N"], t["K"])
    ridx, rmask = ref_ext.masked_ordered_ball_query(g["xyz"], g["xyz"], g["mask"], g["mask"], r, t["K"])
    idx, idx_mask, _ = ops.ball_query(g["xyz"], g["xyz"], g["mask"], g["mask"], r, t["K"])
    assert torch.equal(idx, ridx) and torch.equal(idx_mask, rmask)


def test_c_oracle_equals_reference_nearest_and_group(cuda, oracle_ext, ref_ext):
    d, g = _inputs(2, 1500, 5, cuda)
    gen = torch.Generator().manual_seed(2)
    q = torch.rand(2, 4000, 3, generator=gen)
    qm = torch.ones(2, 4000, dtype=torch.int32)
    ridx, rmask = ref_ext.masked_nearest_query(q.to(cuda), g["xyz"], qm.to(cuda), g["mask"])
    oidx, omask = oracle_ext.masked_nearest_query(q, d["xyz"], qm, d["mask"])
    assert torch.equal(ridx.cpu(), oidx) and torch.equal(rmask.cpu(), omask)
    idx = torch.randint(0, 1500, (2, 700, 9), generator=gen, dtype=torch.int32)
    pts = torch.randn(2, 11, 1500, generator=gen)
    assert torch.equal(ref_ext.group_points(pts.to(cuda), idx.to(cuda)).cpu(), oracle_ext.group_points(pts, idx))


@pytest.mark.parametrize("n,m,dl", [(1024, 300, 0.12), (3000, 1000, 0.07), (500, 600, 0.2)])
def test_c_oracle_equals_reference_grid_subsampling(cuda, oracle_ext, ref_ext, n, m, dl):
    d, g = _inputs(3, n, 9 + n, cuda)
    rs, rm = ref_ext.masked_grid_subsampling(g["xyz"], g["mask"], m, dl)
    os_, om = oracle_ext.masked_grid_subsampling(d["xyz"], d["mask"], m, dl)
    assert torch.equal(rm.cpu(), om)
    assert torch.equal(rs.cpu(), os_)
