"""GPU parity of the fused LocalAggregation operators against the oracle (oracle/la_oracle.py on top of
oracle/cl3d_oracle.c), same seeded inputs, through the public module API (which calls the C ABI).

Tolerance (BASELINE.json north_star): fp32 outputs within 1e-5 of the reference path; gradients within 1e-5
relative to their max magnitude.  Neighbour indices are compared bit-exact in test_neighbors_gpu.py.
"""
import copy
import os
import re

import pytest
import torch

from closerlook3d_b200 import synth
from closerlook3d_b200.config import la_config

pytestmark = pytest.mark.gpu

TOL = 1e-5
# Parameter gradients are sums of B*M*K (~1e5..1e6) signed terms; BOTH sides accumulate them in fp32 in a
# different order, so their agreement is limited to ~1e-5 of the gradient's max magnitude (measured: <= 5e-6).
PARAM_TOL = 5e-5


def _rel_err(a, b):
    scale = max(1.0, float(b.abs().max()))
    return float((a - b).abs().max()) / scale


def _randomize_bn(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if "out_transform" in name or ".1." in name or "out_conv.1" in name:
                if name.endswith("weight"):
                    p.copy_(1.0 + 0.5 * torch.randn(p.shape, generator=g))
                else:
                    p.copy_(0.5 * torch.randn(p.shape, generator=g))


def run_case(cuda, oracle_ext, la_type, over, B, N, K, C, seed, M=None, radius=None, train=True, tol=TOL,
             param_tol=PARAM_TOL, oracle_device="cpu", offset=0.0):
    """oracle_device="cpu": la_oracle over the C restatement (oracle/cl3d_oracle.c) on the host;
    oracle_device=cuda: la_oracle over `oracle_ext` = the reference's OWN CUDA extension (oracle/_ref) on the GPU,
    i.e. the reference's GPU path itself (TF32 off) -- used at the full BASELINE sizes."""
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    from oracle import la_oracle
    cfg = la_config(la_type, **over)
    torch.manual_seed(seed)
    import numpy as np
    np.random.seed(seed)
    r = synth.ball_radius(N, K) if radius is None else radius
    mod = LocalAggregation(C, C, r, K, cfg)
    _randomize_bn(mod, seed)
    sd = copy.deepcopy(mod.state_dict())
    d = synth.make_cloud_batch(B, N, C, seed)
    xyz, mask, feats = d["xyz"], d["mask"], d["features"]
    if offset:
        xyz = (xyz + offset).contiguous()   # a scene far from the coordinate origin
    if M is None:
        q, qm = xyz, mask
    else:  # strided block: queries are a different (smaller) set near the supports
        g = torch.Generator().manual_seed(seed + 1)
        q = (xyz[:, :M] + 0.1 * r * torch.randn(B, M, 3, generator=g)).contiguous()  # every query keeps >= 1 neighbour
        qm = torch.ones(B, M, dtype=torch.int32)
        qm[:, M - M // 8:] = 0
    gout = torch.randn(B, C, q.shape[1], generator=torch.Generator().manual_seed(seed + 2))

    # ---- forward on both sides (the oracle follows the reference's GPU arithmetic for `/= radius`, see la_oracle)
    on_gpu = str(oracle_device) != "cpu"
    if on_gpu:   # the reference's arithmetic on its own device: nothing to emulate
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
    else:
        la_oracle.GPU_SCALAR_DIVISION = True
        la_oracle.DIM_MAT_FN = lambda fd: torch.pow(
            1.0 * 1000, (1.0 / fd) * torch.arange(fd, dtype=torch.float32).to(cuda)).cpu()   # reference :72-75 on its device
    orc = la_oracle.OracleLocalAggregation(oracle_ext, la_type, C, C, r, K, cfg, sd, device=oracle_device)
    orc.training = train
    od = oracle_device
    f_ref = feats.clone().to(od).requires_grad_(True)
    is_max = over.get(la_type, {}).get("reduction") == "max" and la_type != "pseudo_grid"
    la_oracle.KEEP = {} if is_max else None
    o_ref = orc(q.to(od), xyz.to(od), qm.to(od), mask.to(od), f_ref)
    decided = None
    if la_oracle.KEEP:
        # max over K: where the two best DISTINCT neighbours tie within the tolerance, rounding decides which one
        # receives the gradient (a discontinuity like the ReLU's); those (query, channel) positions get no
        # upstream gradient on either side
        if la_type == "pointwisemlp":     # post-ReLU activations through the 3xTF32 GEMM
            decided = la_oracle.argmax_is_decided(la_oracle.KEEP["pwmlp_premax"], la_oracle.KEEP["idx"]).cpu()
        else:                             # products of fp32 inputs: the two sides differ at rounding level only
            decided = la_oracle.argmax_is_decided(la_oracle.KEEP["premax"], la_oracle.KEEP["idx"], rel=2e-6,
                                                  relu=False).cpu()
        assert int((~decided).sum()) <= max(4, decided.numel() // 2000), f"{int((~decided).sum())} undecided maxima"
    la_oracle.KEEP = None
    mod = mod.to(cuda)
    mod.train(train)
    f = feats.to(cuda).requires_grad_(True)
    out = mod(q.to(cuda), xyz.to(cuda), qm.to(cuda), mask.to(cuda), f)
    # The final ReLU makes the gradient discontinuous at 0: an output that is +4e-6 on one side and 0 on the
    # other is inside the output tolerance but flips a whole BN channel's gradient.  Such elements (a handful
    # per million) get zero upstream gradient on BOTH sides, so the comparison is well-posed.
    la_oracle.GPU_SCALAR_DIVISION = False
    la_oracle.DIM_MAT_FN = None
    flips = (out.detach().cpu() > 0) != (o_ref.detach().cpu() > 0)
    assert int(flips.sum()) <= max(2, out.numel() // 100000), f"{int(flips.sum())} ReLU sign flips"
    gout = gout * (~flips)
    if decided is not None:
        gout = gout * decided
    (o_ref * gout.to(od)).sum().backward()
    (out * gout.to(cuda)).sum().backward()
    torch.cuda.synchronize()

    assert out.shape == o_ref.shape
    assert not torch.isnan(out).any()
    e_out = _rel_err(out.detach().cpu(), o_ref.detach().cpu())
    e_gf = _rel_err(f.grad.cpu(), f_ref.grad.cpu())
    assert e_out <= tol, f"output err {e_out}"
    assert e_gf <= tol, f"grad_features err {e_gf}"
    ref_grads = orc.grads()
    for name, p in mod.named_parameters():
        k = name[len("local_aggregation_operator."):]
        assert p.grad is not None, f"no grad for {name}"
        e = _rel_err(p.grad.cpu(), ref_grads[k].cpu())
        assert e <= param_tol, f"grad {name} err {e}"
    sd2 = mod.state_dict()
    for k, v in orc.st.items():
        if k.endswith(("running_mean", "running_var", "num_batches_tracked")):
            e = _rel_err(sd2["local_aggregation_operator." + k].float().cpu(), v.float().cpu())
            assert e <= tol, f"buffer {k} err {e}"
    return e_out, e_gf


PW = dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))
XYZ_MAX = dict(pospool=dict(position_embedding="xyz", reduction="max"))
SINCOS_MAX = dict(pospool=dict(position_embedding="sin_cos", reduction="max"))
AW_MAX = dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1, reduction="max"))
XYZ_AVG = dict(pospool=dict(position_embedding="xyz", reduction="avg"))
SINCOS_AVG = dict(pospool=dict(position_embedding="sin_cos", reduction="avg"))
AW = dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1, reduction="avg"))


@pytest.mark.parametrize("la_type,over,B,N,K,C", [
    ("pospool", XYZ_AVG, 2, 1024, 16, 66),                # BASELINE c1 (C=66: C=64 is illegal for PosPool)
    ("pospool", XYZ_AVG, 2, 1024, 16, 72),
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="sum")), 3, 700, 12, 9),
    ("pospool", SINCOS_AVG, 2, 1024, 16, 66),
    ("pospool", SINCOS_AVG, 2, 3000, 40, 144),            # c5 operator shape, smaller cloud
    ("pospool", XYZ_AVG, 2, 2500, 20, 288),               # channel chunking (C > 192)
    ("adaptive_weight", AW, 3, 1024, 16, 72),
    ("adaptive_weight", AW, 2, 3000, 32, 72),             # c4 operator shape, smaller cloud
    ("adaptive_weight", dict(adaptive_weight=dict(shared_channels=4, reduction="sum")), 2, 900, 16, 72),
    ("pseudo_grid", dict(), 2, 1024, 16, 72),
    ("pseudo_grid", dict(), 2, 3000, 26, 72),             # c3 operator shape, smaller cloud
    ("pseudo_grid", dict(pseudo_grid=dict(KP_influence="constant")), 2, 800, 16, 36),
    ("pseudo_grid", dict(), 2, 1500, 16, 144),            # two channel chunks
    ("pospool", XYZ_MAX, 2, 1024, 16, 66),                # fused max reduction (agg_max.cu)
    ("pospool", XYZ_MAX, 2, 1500, 40, 288),               # K > 32 (two rounds), three channel chunks
    ("pospool", SINCOS_MAX, 2, 1024, 16, 66),
    ("adaptive_weight", AW_MAX, 3, 1024, 16, 72),
    ("adaptive_weight", dict(adaptive_weight=dict(shared_channels=4, reduction="max")), 2, 900, 20, 72),
    ("pointwisemlp", PW, 2, 1024, 16, 66),
    ("pointwisemlp", PW, 4, 1024, 32, 72),                # c2 operator shape, smaller batch
    ("pointwisemlp", PW, 2, 2500, 20, 36),
    ("pointwisemlp", PW, 1, 600, 40, 144),                # two output-channel chunks, K > 32
])
def test_family_matches_oracle(cuda, oracle_ext, la_type, over, B, N, K, C):
    # 'constant' influence + BatchNorm: every kernel weight only rescales its channel, which BN removes, so
    # the exact kernel_weights gradient is 0 and both sides return rounding noise of size ~1 -> loose bound
    ptol = 2e-3 if over.get("pseudo_grid", {}).get("KP_influence") == "constant" else PARAM_TOL
    run_case(cuda, oracle_ext, la_type, over, B, N, K, C, seed=2000 + N + C, param_tol=ptol)


@pytest.mark.parametrize("la_type,over", [("pospool", XYZ_AVG), ("adaptive_weight", AW), ("pseudo_grid", dict()),
                                          ("pointwisemlp", PW)])
def test_scene_far_from_origin(cuda, oracle_ext, la_type, over):
    # S3DIS-like coordinates: |xyz| / radius ~ 150.  The relative positions are differences of nearby points, so the
    # result must not lose accuracy (PointWiseMLP's separable per-point / per-query terms are centred per cloud).
    run_case(cuda, oracle_ext, la_type, over, 2, 1024, 16, 72, seed=91, offset=25.0)


@pytest.mark.parametrize("la_type,over", [("pospool", XYZ_AVG), ("adaptive_weight", AW), ("pseudo_grid", dict()),
                                          ("pointwisemlp", PW)])
def test_strided_queries(cuda, oracle_ext, la_type, over):
    # queries != supports (strided bottleneck): M < N, padded queries, some queries with few neighbours
    run_case(cuda, oracle_ext, la_type, over, 3, 2400, 16, 72, seed=31, M=600, radius=0.15)


@pytest.mark.parametrize("la_type,over", [("pospool", XYZ_AVG), ("pseudo_grid", dict()), ("adaptive_weight", AW),
                                          ("pospool", SINCOS_AVG), ("pointwisemlp", PW)])
def test_eval_mode_uses_running_stats(cuda, oracle_ext, la_type, over):
    # forward with running statistics AND the backward through the frozen BatchNorm (fine-tuning with frozen BN)
    run_case(cuda, oracle_ext, la_type, over, 2, 1024, 16, 72, seed=77, train=False)


@pytest.mark.parametrize("la_type,over", [
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="max"))),
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="avg", output_conv=True))),
    ("adaptive_weight", dict(adaptive_weight=dict(num_mlps=2, shared_channels=2, reduction="avg"))),
    ("pseudo_grid", dict(pseudo_grid=dict(output_conv=True))),
    ("pointwisemlp", dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=2, reduction="max"))),
])
def test_composed_settings(cuda, oracle_ext, la_type, over):
    # settings outside the fused kernels run through the materialising GPU path (library conv: TF32 off)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    run_case(cuda, oracle_ext, la_type, over, 2, 600, 12, 36, seed=5, tol=2e-5)


def _declared_functions():
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "cl3d.h")) as fh:
        hdr = fh.read()
    return set(re.findall(r"\b(cl3d_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)))


@pytest.mark.parametrize("la_type,over,entries", [
    ("pseudo_grid", dict(), {"cl3d_to_point_major", "cl3d_agg_fwd", "cl3d_agg_bwd", "cl3d_bn_relu_fwd",
                             "cl3d_bn_relu_bwd"}),
    # the output is cl3d_bn_relu_fwd over the selected extremum
    pytest.param("pointwisemlp", PW, {"cl3d_sgemm_algo", "cl3d_pwmlp_fwd_stats", "cl3d_bn_relu_fwd", "cl3d_pwmlp_bwd",
                                      "cl3d_to_channel_major"}, id="pointwisemlp-output-bn_relu_fwd"),
])
def test_profiler_records_declared_entry_points(cuda, la_type, over, entries):
    # bench.py's kernel model and tools/bench_pg.py look the profiler's records up by the names include/cl3d.h declares
    from closerlook3d_b200 import _lib
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    B, N, K, C = 2, 1024, 16, 72
    torch.manual_seed(0)
    mod = LocalAggregation(C, C, synth.ball_radius(N, K), K, la_config(la_type, **over)).to(cuda)
    d = synth.make_cloud_batch(B, N, C, 0)
    xyz, mask = d["xyz"].to(cuda), d["mask"].to(cuda)
    f = d["features"].to(cuda).requires_grad_(True)
    _lib.profiler.start()
    try:
        mod(xyz, xyz, mask, mask, f).sum().backward()
    finally:
        recorded = set(_lib.profiler.stop())
    assert recorded <= _declared_functions(), f"recorded but not declared: {sorted(recorded - _declared_functions())}"
    assert entries <= recorded, f"not recorded: {sorted(entries - recorded)}"
