"""The float64 reference (oracle.la_oracle over oracle.f64_ext, float64 state) against the fp32 oracle, which
tests/test_oracle_cpu.py and tests/golden pin to the reference.  Both evaluate the same functions; they may differ
by fp32 rounding only.  This pins the high-precision reference that tests/test_wide_layers_gpu.py measures the
kernels against to the already-pinned one, family by family, forward and backward."""
import copy

import pytest
import torch

from closerlook3d_b200 import synth
from closerlook3d_b200.config import la_config

# fp32 rounding of the fp32 oracle, relative to each tensor's max magnitude (measured: <= 1e-6; the BatchNorm
# normalisation of a channel with a small spread amplifies it a little)
TOL = 5e-6
PARAM_TOL = 2e-5


def _rel_err(a, b):
    return float((a.double() - b.double()).abs().max()) / max(1.0, float(b.double().abs().max()))


def _randomize_bn(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if "out_transform" in name or ".1." in name or "out_conv.1" in name:
                p.copy_((1.0 + 0.5 * torch.randn(p.shape, generator=g)) if name.endswith("weight")
                        else 0.5 * torch.randn(p.shape, generator=g))


def _run(ext, la_type, cfg, C, r, K, sd, q, s, qm, sm, feats, gout, train, dtype):
    from oracle import la_oracle
    is_max = la_type != "pseudo_grid" and cfg[la_type].get("reduction") == "max"
    la_oracle.KEEP = {} if is_max else None
    try:
        orc = la_oracle.OracleLocalAggregation(ext, la_type, C, C, r, K, cfg, sd, dtype=dtype)
        orc.training = train
        f = feats.detach().to(dtype or torch.float32, copy=True).requires_grad_(True)
        out = orc(q, s, qm, sm, f)
        keep = la_oracle.KEEP
    finally:
        la_oracle.KEEP = None
    return orc, f, out, keep


CASES = [
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="avg"))),
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="sum"))),
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="max"))),
    ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="avg"))),
    ("pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="max"))),
    ("adaptive_weight", dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1, reduction="avg"))),
    ("adaptive_weight", dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=4, reduction="max"))),
    ("pseudo_grid", dict()),
    ("pointwisemlp", dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))),
]


@pytest.mark.parametrize("strided", [False, True], ids=["self", "strided"])
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("la_type,over", CASES)
def test_f64_reference_matches_fp32_oracle(oracle_ext, la_type, over, train, strided):
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    from oracle import f64_ext, la_oracle
    B, N, K, C, seed = 2, 400, 12, 24, 17
    cfg = la_config(la_type, **over)
    torch.manual_seed(seed)
    r = synth.ball_radius(N, K)
    mod = LocalAggregation(C, C, r, K, cfg)
    _randomize_bn(mod, seed)
    sd = copy.deepcopy(mod.state_dict())
    d = synth.make_cloud_batch(B, N, C, seed)
    s, sm, feats = d["xyz"], d["mask"], d["features"]
    if strided:
        M = 120
        g = torch.Generator().manual_seed(seed + 1)
        q = (s[:, :M] + 0.1 * r * torch.randn(B, M, 3, generator=g)).contiguous()
        qm = torch.ones(B, M, dtype=torch.int32)
        qm[:, M - M // 8:] = 0
    else:
        q, qm = s, sm
    gout = torch.randn(B, C, q.shape[1], generator=torch.Generator().manual_seed(seed + 2), dtype=torch.float64)

    o32 = _run(oracle_ext, la_type, cfg, C, r, K, sd, q, s, qm, sm, feats, gout, train, None)
    o64 = _run(f64_ext, la_type, cfg, C, r, K, sd, q, s, qm, sm, feats, gout, train, torch.float64)
    (orc32, f32, out32, keep32), (orc64, f64, out64, keep64) = o32, o64
    assert out64.dtype == torch.float64 and f64.dtype == torch.float64
    assert all(v.dtype == torch.float64 for v in orc64.params().values())
    # where the ReLU or the arg-max over K is decided by rounding, neither side's gradient is meaningful
    flips = (out32.detach() > 0) != (out64.detach() > 0)
    assert int(flips.sum()) <= 2, int(flips.sum())
    gout = gout * (~flips)
    if keep64 is not None:
        pre = keep64["pwmlp_premax"] if la_type == "pointwisemlp" else keep64["premax"]
        decided = la_oracle.argmax_is_decided(pre, keep64["idx"], rel=1e-6, relu=la_type == "pointwisemlp")
        assert int((~decided).sum()) <= 4
        gout = gout * decided
    (out32 * gout.float()).sum().backward()
    (out64 * gout).sum().backward()

    assert _rel_err(out32.detach(), out64.detach()) <= TOL
    assert _rel_err(f32.grad, f64.grad) <= TOL
    g32, g64 = orc32.grads(), orc64.grads()
    assert set(g32) == set(g64) and g64
    for k in g64:
        assert _rel_err(g32[k], g64[k]) <= PARAM_TOL, k
    for k, v in orc64.st.items():
        if k.endswith(("running_mean", "running_var")):
            assert _rel_err(orc32.st[k], v) <= TOL, k
        elif k.endswith("num_batches_tracked"):
            assert int(orc32.st[k]) == int(v), k


def test_f64_grouping_is_the_adjoint_of_the_gather(oracle_ext):
    """f64_ext.group_points / group_points_grad equal the C restatement's on fp32 data, and keep float64"""
    from oracle import f64_ext
    g = torch.Generator().manual_seed(4)
    B, C, N, M, K = 2, 5, 50, 30, 7
    pts = torch.randn(B, C, N, generator=g)
    idx = torch.randint(0, N, (B, M, K), generator=g, dtype=torch.int32)
    gout = torch.randn(B, C, M, K, generator=g)
    assert torch.equal(f64_ext.group_points(pts, idx), oracle_ext.group_points(pts, idx))
    want = oracle_ext.group_points_grad(gout, idx, N)
    got = f64_ext.group_points_grad(gout.double(), idx, N)
    assert got.dtype == torch.float64
    assert float((got - want.double()).abs().max()) <= 1e-5
    d = synth.make_cloud_batch(B, N, 3, 4)
    r = synth.ball_radius(N, K)
    a = f64_ext.masked_ordered_ball_query(d["xyz"], d["xyz"], d["mask"], d["mask"], r, K)
    b = oracle_ext.masked_ordered_ball_query(d["xyz"], d["xyz"], d["mask"], d["mask"], r, K)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
