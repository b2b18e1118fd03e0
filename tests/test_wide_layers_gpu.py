"""GPU: every local-aggregation family at the channel widths and stage shapes the shipped networks run, against the
float64 reference (oracle.la_oracle over oracle.f64_ext, see tests/test_f64_reference_cpu.py).

The scene-segmentation ResNet (backbone.py:75-91, width 144, bottleneck ratio 2; npoints [4096, 1152, 304, 88],
nsamples [26, 31, 38, 41, 39], backbone.py:232-233) runs its LocalAggregation layers at C = 72 ... 1152 on fewer
points the wider they are; its "width x2" variant (the sin_cos config) at C = 144 ... 2304.  Each kernel chooses its
template instance and its number of channel chunks from C, so these widths run code that narrow layers never reach
(the dispatch rules are restated, and their coverage by the tables below asserted, in
test_case_tables_reach_every_instance).

Bars.  Outputs and d/dfeatures: 1e-5 per channel, max|err_c| / max(max|ref_c|, 1e-3 max|ref|), so that one wrong
channel or chunk of low magnitude cannot hide under the tensor's global maximum; the global bar of the other parity
tests as well.  Parameter gradients (sums of B*M*K fp32 terms in a different order): 5e-5 of their max magnitude.
The operator-level tests check the pre-BatchNorm aggregation per element against |err| <= 1e-5 * scale, scale =
the same reduction of the terms' absolute values.
"""
import copy

import pytest
import torch

from closerlook3d_b200 import synth
from closerlook3d_b200.config import la_config

TOL = 1e-5
PARAM_TOL = 5e-5

XYZ_AVG = dict(pospool=dict(position_embedding="xyz", reduction="avg"))
XYZ_MAX = dict(pospool=dict(position_embedding="xyz", reduction="max"))
SINCOS_AVG = dict(pospool=dict(position_embedding="sin_cos", reduction="avg"))
SINCOS_MAX = dict(pospool=dict(position_embedding="sin_cos", reduction="max"))
AW = dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1, reduction="avg"))
AW_MAX = dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1, reduction="max"))
AW_S4 = dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=4, reduction="sum"))
PG = dict()
PW = dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))

# (C, M, N, K) of the scene-segmentation network's LocalAggregation layers: strided (M = npoints[s], N = the
# previous stage's points) and plain (M = N).  res1's 72-wide layers run on the 15000-point input; here on 4096.
SCENE = [
    (72, 4096, 4096, 26),
    (144, 4096, 15000, 26),
    (144, 4096, 4096, 31),
    (288, 1152, 4096, 31),
    (288, 1152, 1152, 38),
    (576, 304, 1152, 38),
    (576, 304, 304, 41),
    (1152, 88, 304, 41),
    (1152, 88, 88, 39),
]
SCENE_X2 = [(2 * C, M, N, K) for C, M, N, K in SCENE]          # the width x2 network (PosPool sin_cos, c5)

FAMILIES = [("pospool", XYZ_AVG, SCENE), ("pospool", SINCOS_AVG, SCENE_X2), ("adaptive_weight", AW, SCENE),
            ("pseudo_grid", PG, SCENE), ("pointwisemlp", PW, SCENE)]
STAGE_CASES = [(t, o, C, M, N, K, True) for t, o, table in FAMILIES for C, M, N, K in table]

SMALL = (1024, 2048, 24)    # M, N, K of the instance-targeting cases
EXTRA_CASES = [
    # max reductions with several channel chunks (agg_max.cu: 96 channels per chunk)
    ("pospool", XYZ_MAX, 576, 304, 1152, 38, True),
    ("pospool", XYZ_MAX, 120, *SMALL, True),               # two chunks, the last one 24 wide
    ("pospool", SINCOS_MAX, 576, 304, 304, 41, True),
    ("adaptive_weight", AW_MAX, 1152, 88, 304, 41, True),
    ("adaptive_weight", AW_MAX, 120, *SMALL, True),
    # template instances no network layer above reaches
    ("pospool", SINCOS_AVG, 48, *SMALL, True),              # sin_cos PI = 1
    ("pospool", XYZ_AVG, 120, *SMALL, True),                # CI = 4
    ("adaptive_weight", AW, 24, *SMALL, True),              # CI = 1
    ("adaptive_weight", AW, 48, *SMALL, True),              # CI = 2
    ("adaptive_weight", AW, 120, *SMALL, True),             # CI = 4
    ("adaptive_weight", AW_S4, 144, *SMALL, True),          # CI = 5, shared channels
    ("adaptive_weight", AW, 192, *SMALL, True),             # CI = 6
    ("pseudo_grid", PG, 260, *SMALL, True),                 # chunks of 88, the last one with 84 real channels
    # eval mode (frozen BatchNorm) at the widest layer of each family
    ("pospool", XYZ_AVG, 1152, 88, 88, 39, False),
    ("pospool", SINCOS_AVG, 2304, 88, 88, 39, False),
    ("adaptive_weight", AW, 1152, 88, 88, 39, False),
    ("pseudo_grid", PG, 1152, 88, 88, 39, False),
    ("pointwisemlp", PW, 1152, 88, 88, 39, False),
]


def _family_id(la_type, over):
    v = over.get(la_type, {})
    tag = {"pospool": v.get("position_embedding", ""), "adaptive_weight": f"S{v.get('shared_channels', 1)}"}.get(
        la_type, "")
    return "-".join(x for x in (la_type, tag, v.get("reduction", "")) if x)


def _case_id(c):
    la_type, over, C, M, N, K, train = c
    return f"{_family_id(la_type, over)}-C{C}-M{M}-N{N}-K{K}" + ("" if train else "-eval")


def _rel_err(a, b):
    return float((a - b).abs().max()) / max(1.0, float(b.abs().max()))


def per_channel_err(a, b, scale=None):
    """max_c max|a_c - b_c| / max(max|s_c|, 1e-3 max|s|) over dim 1 (channels) of (B,C,...) tensors -> (err, c);
    s = b unless a `scale` tensor of the same shape is given"""
    C = b.shape[1]
    s = b if scale is None else scale
    e = (a.double() - b.double()).abs().transpose(0, 1).reshape(C, -1).max(1)[0]
    r = s.double().abs().transpose(0, 1).reshape(C, -1).max(1)[0]
    rel = e / r.clamp(min=1e-3 * max(float(r.max()), 1e-30))
    c = int(rel.argmax())
    return float(rel[c]), c


def _randomize_bn(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if "out_transform" in name or ".1." in name or "out_conv.1" in name:
                p.copy_((1.0 + 0.5 * torch.randn(p.shape, generator=g)) if name.endswith("weight")
                        else 0.5 * torch.randn(p.shape, generator=g))


def _cloud(B, C, M, N, K, seed):
    """supports, and queries: the supports themselves (M == N) or a strided subset near them"""
    r = synth.ball_radius(N, K)
    d = synth.make_cloud_batch(B, N, C, seed)
    xyz, mask, feats = d["xyz"], d["mask"], d["features"]
    if M == N:
        return r, xyz, mask, xyz, mask, feats
    g = torch.Generator().manual_seed(seed + 1)
    q = (xyz[:, :M] + 0.1 * r * torch.randn(B, M, 3, generator=g)).contiguous()
    qm = torch.ones(B, M, dtype=torch.int32)
    qm[:, M - M // 8:] = 0
    return r, xyz, mask, q, qm, feats


def run_wide(cuda, la_type, over, C, M, N, K, train=True, B=2, seed=None):
    """module API (fused kernels) vs the float64 reference on the GPU -> dict of the measured errors"""
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    from oracle import f64_ext, la_oracle
    seed = 7000 + C + M + K if seed is None else seed
    cfg = la_config(la_type, **over)
    torch.manual_seed(seed)
    r, xyz, mask, q, qm, feats = _cloud(B, C, M, N, K, seed)
    mod = LocalAggregation(C, C, r, K, cfg)
    _randomize_bn(mod, seed)
    sd = copy.deepcopy(mod.state_dict())
    gout = torch.randn(B, C, M, generator=torch.Generator().manual_seed(seed + 2), dtype=torch.float64).to(cuda)
    xyz_d, mask_d, q_d, qm_d = xyz.to(cuda), mask.to(cuda), q.to(cuda), qm.to(cuda)

    # ---- float64 reference on the GPU; dp and the sin_cos arguments follow the reference's fp32 GPU arithmetic
    is_max = la_type != "pseudo_grid" and cfg[la_type].get("reduction") == "max"
    la_oracle.GPU_SCALAR_DIVISION = True
    la_oracle.DIM_MAT_FN = lambda fd: torch.pow(
        1.0 * 1000, (1.0 / fd) * torch.arange(fd, dtype=torch.float32).to(cuda)).cpu()   # reference :72-75
    la_oracle.KEEP = {}
    try:
        orc = la_oracle.OracleLocalAggregation(f64_ext, la_type, C, C, r, K, cfg, sd, device=cuda,
                                               dtype=torch.float64)
        orc.training = train
        f_ref = feats.to(cuda, torch.float64).requires_grad_(True)
        o_ref = orc(q_d, xyz_d, qm_d, mask_d, f_ref)
        keep = la_oracle.KEEP
    finally:
        la_oracle.GPU_SCALAR_DIVISION = False
        la_oracle.DIM_MAT_FN = None
        la_oracle.KEEP = None
    pre_relu = keep.pop("pre_relu", None)
    decided = None
    if is_max:
        # the arg-max over K, decided by the float64 values: where the two best DISTINCT neighbours are closer than
        # fp32 rounding, either side may route the gradient to either of them
        if la_type == "pointwisemlp":
            decided = la_oracle.argmax_is_decided(keep["pwmlp_premax"], keep["idx"])
        else:
            decided = la_oracle.argmax_is_decided(keep["premax"], keep["idx"], rel=2e-6, relu=False)
        assert int((~decided).sum()) <= max(4, decided.numel() // 2000), f"{int((~decided).sum())} undecided maxima"
        del keep

    # ---- the fused path
    mod = mod.to(cuda)
    mod.train(train)
    f = feats.to(cuda).requires_grad_(True)
    out = mod(q_d, xyz_d, qm_d, mask_d, f)
    flips = (out.detach() > 0) != (o_ref.detach() > 0)       # the final ReLU decided by rounding
    assert int(flips.sum()) <= max(2, out.numel() // 100000), f"{int(flips.sum())} ReLU sign flips"
    gout = gout * (~flips)
    if decided is not None:
        gout = gout * decided
    (o_ref * gout).sum().backward()
    (out * gout.float()).sum().backward()
    torch.cuda.synchronize()

    assert out.shape == o_ref.shape and torch.isfinite(out).all()
    res = {}
    # The final ReLU leaves some channels with a few small positive outputs (BatchNorm shift beta < 0, small gamma):
    # their post-ReLU maximum is no measure of the channel's scale, the error of an output is that of its pre-ReLU
    # value.  So a channel's output error is measured against its pre-ReLU range (PointWiseMLP: max over K of the
    # BatchNorm output, since max_k relu(y) = relu(max_k y)); the post-ReLU ratio is reported beside it.
    res["out"], c_out = per_channel_err(out.detach(), o_ref.detach(), pre_relu)
    res["out_post_relu"] = per_channel_err(out.detach(), o_ref.detach())[0]
    res["grad_features"], c_gf = per_channel_err(f.grad, f_ref.grad)
    res["out_global"] = _rel_err(out.detach().double(), o_ref.detach())
    res["grad_features_global"] = _rel_err(f.grad.double(), f_ref.grad)
    ref_grads = orc.grads()
    params = {}
    for name, p in mod.named_parameters():
        k = name[len("local_aggregation_operator."):]
        assert p.grad is not None, f"no grad for {name}"
        params[k] = _rel_err(p.grad.double(), ref_grads[k])
    buffers = {}
    sd2 = mod.state_dict()
    for k, v in orc.st.items():
        if k.endswith(("running_mean", "running_var")):
            buffers[k] = _rel_err(sd2["local_aggregation_operator." + k].double(), v)
        elif k.endswith("num_batches_tracked"):
            assert int(sd2["local_aggregation_operator." + k]) == int(v), k
    print(f"\nWIDE {_family_id(la_type, over)} C={C} M={M} N={N} K={K} train={train}: "
          f"out/ch {res['out']:.2e} (c{c_out}; post-ReLU {res['out_post_relu']:.2e}) grad_f/ch {res['grad_features']:.2e} (c{c_gf}) "
          f"params {max(params.values()):.2e} buffers {max(buffers.values(), default=0.0):.2e} "
          f"peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")

    assert res["out"] <= TOL, f"output: channel {c_out} err {res['out']}"
    assert res["grad_features"] <= TOL, f"grad_features: channel {c_gf} err {res['grad_features']}"
    assert res["out_global"] <= TOL and res["grad_features_global"] <= TOL, res
    for k, e in params.items():
        assert e <= PARAM_TOL, f"grad {k} err {e}"
    for k, e in buffers.items():
        assert e <= TOL, f"buffer {k} err {e}"
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("case", STAGE_CASES + EXTRA_CASES, ids=_case_id)
def test_wide_layer_matches_f64_reference(cuda, oracle_ext, case):
    la_type, over, C, M, N, K, train = case
    torch.cuda.reset_peak_memory_stats()
    run_wide(cuda, la_type, over, C, M, N, K, train=train)


# --------------------------------------------------------------------------------------------------------------
# operator level: the pre-BatchNorm aggregation of ops.agg_fwd / ops.agg_bwd per element
# --------------------------------------------------------------------------------------------------------------
def _f64_terms(fam, dp, p0, p1, C, shared, extent, absolute):
    """(B,M,K,3) f32 relative positions -> per-channel weights w (B,C,M,K) float64 of each neighbour term
    f[j,c] * w_c, or (absolute=True) the bound of |w_c| from the absolute values of its own terms"""
    from closerlook3d_b200 import ops
    B, M, K, _ = dp.shape
    d64 = dp.double()
    if fam == ops.FAM_POSPOOL_XYZ:                                 # w_c = dp[c % 3]
        w = d64.permute(3, 0, 1, 2).repeat(C // 3, 1, 1, 1)        # (C,B,M,K)
        w = w.abs() if absolute else w
    elif fam == ops.FAM_POSPOOL_SINCOS:                            # c = axis*2F + t: sin (t < F) / cos of the pair
        F_ = C // 6
        arg = torch.div((100 * dp).unsqueeze(-1), p0.float()).double()   # fl32(fl32(100 dp) / dim): (B,M,K,3,F)
        if absolute:                                               # the hardware sine's error is absolute
            w = torch.ones(B, M, K, 3, 2 * F_, dtype=torch.float64, device=dp.device)
        else:
            w = torch.cat([torch.sin(arg), torch.cos(arg)], -1)
        w = w.reshape(B, M, K, C).permute(3, 0, 1, 2)
    elif fam == ops.FAM_ADAPTIVE_DP:                               # w_c = W[c//S] . dp + b[c//S]
        W, b = p0, p1
        if absolute:
            w = d64.abs() @ W.abs().t() + b.abs()
        else:
            w = d64 @ W.t() + b
        w = w.repeat_interleave(shared, dim=-1).permute(3, 0, 1, 2)
    else:                                                          # PseudoGrid: w_c = sum_k' Wk[k',c] h(k', dp)
        kp, Wk = p0, p1
        dist = torch.sqrt(((d64.unsqueeze(3) - kp.double()) ** 2).sum(-1)) / extent
        h = torch.clamp(1 - dist, min=0.0)
        if absolute:                                               # h = 1 - dist: its terms are 1 and dist
            h = (1 + dist) * (h > 0)
        w = (h @ (Wk.abs() if absolute else Wk)).permute(3, 0, 1, 2)
    return w.permute(1, 0, 2, 3)                                   # (B,C,M,K)


def _f64_reduce(f, idx, valid, cnt, w, reduction):
    from oracle import f64_ext
    terms = f64_ext.group_points(f, idx) * w
    if reduction == "max":
        return terms.masked_fill(~valid[:, None], float("-inf")).max(-1)[0]
    s = (terms * valid[:, None]).sum(-1)
    return s / cnt[:, None] if reduction == "avg" else s


OP_CASES = [
    # family, reduction, C, shared: the channel-chunked shapes
    ("xyz", "avg", 120, 1),        # agg_*_kernel<XYZ, 4>
    ("xyz", "sum", 576, 1),        # three chunks of 192
    ("sincos", "avg", 576, 1),     # gridDim.y = 3: the p0 > 0 pair lanes
    ("sincos", "sum", 2304, 1),
    ("aw", "avg", 120, 1),
    ("aw", "sum", 1152, 1),
    ("pg", "sum", 260, 1),         # uneven chunks, Cv < Cw in the last one
    ("pg", "sum", 576, 1),         # 4 x 116 + 112
    ("xyz", "max", 120, 1),        # agg_max.cu: two chunks, the last one 24 wide
    ("xyz", "max", 576, 1),
    ("sincos", "max", 576, 1),
    ("aw", "max", 1152, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("fam_name,reduction,C,shared", OP_CASES, ids=lambda v: str(v))
def test_chunked_aggregation_per_element(cuda, fam_name, reduction, C, shared):
    from closerlook3d_b200 import ops
    from closerlook3d_b200.kernel_points import create_kernel_points
    fam = {"xyz": ops.FAM_POSPOOL_XYZ, "sincos": ops.FAM_POSPOOL_SINCOS, "aw": ops.FAM_ADAPTIVE_DP,
           "pg": ops.FAM_PSEUDOGRID}[fam_name]
    B, M, N, K = 2, 600, 1800, 28
    seed = 300 + C
    g = torch.Generator().manual_seed(seed)
    d = synth.make_cloud_batch(B, N, C, seed)
    r = synth.ball_radius(N, K)
    s = d["xyz"].to(cuda)
    q = (d["xyz"][:, :M] + 0.1 * r * torch.randn(B, M, 3, generator=g)).contiguous().to(cuda)
    sm = d["mask"].to(cuda)
    qm = torch.ones(B, M, dtype=torch.int32, device=cuda)
    feats = d["features"].to(cuda)
    idx, idx_mask, ncount = ops.ball_query(q, s, qm, sm, r, K)
    assert int(ncount.min()) >= 1

    normalize = 0 if fam == ops.FAM_PSEUDOGRID else 1
    nkp, extent, p0, p1 = 0, 1.0, None, None
    if fam == ops.FAM_POSPOOL_SINCOS:
        fd = C // 6
        p0 = torch.pow(1.0 * 1000, (1.0 / fd) * torch.arange(fd, dtype=torch.float32).to(cuda)).contiguous()
    elif fam == ops.FAM_ADAPTIVE_DP:
        p0 = torch.randn(C // shared, 3, generator=g).to(cuda)
        p1 = (0.3 * torch.randn(C // shared, generator=g)).to(cuda)
    elif fam == ops.FAM_PSEUDOGRID:
        nkp = 15
        extent = 2 * 1.0 * r / 5.0
        kp = create_kernel_points(1.5 * extent, nkp, num_kernels=1, dimension=3, fixed="center").reshape(nkp, 3)
        p0 = torch.from_numpy(kp).float().to(cuda).contiguous()
        p1 = torch.randn(nkp, C, generator=g).to(cuda)
    red = ops.REDUCE[reduction]
    feat_pm = ops.to_point_major(feats)
    arg = torch.empty(B, M, feat_pm.shape[2], dtype=torch.uint8, device=cuda) if reduction == "max" else None
    agg, _ = ops.agg_fwd(fam, red, feat_pm, q, s, idx, ncount, p0, p1, C, r, normalize, shared, nkp, extent, 0,
                         want_bn_partial=True, arg=arg)

    # float64 reference over the same neighbour lists; dp in the kernels' fp32 arithmetic (fsub, fmul by 1/r)
    valid = torch.arange(K, device=cuda)[None, None, :] < ncount[:, :, None]
    sg = torch.gather(s, 1, idx.long().reshape(B, M * K, 1).expand(-1, -1, 3)).view(B, M, K, 3)
    dp = sg - q[:, :, None, :]
    if normalize:
        dp = dp * (torch.ones((), dtype=torch.float32) / torch.tensor(r, dtype=torch.float32)).to(cuda)
    cnt = ncount.double()
    f64 = feats.double().requires_grad_(True)
    # the learned parameters (float64 leaves) and the fixed ones (sin_cos wave lengths, kernel points)
    P = {ops.FAM_ADAPTIVE_DP: [p0, p1], ops.FAM_PSEUDOGRID: [p1]}.get(fam, [])
    P = [t.double().requires_grad_(True) for t in P]
    Pa = [t.detach().abs().requires_grad_(True) for t in P]

    def params(Q):
        return (Q[0], Q[1]) if fam == ops.FAM_ADAPTIVE_DP else ((p0, Q[0]) if fam == ops.FAM_PSEUDOGRID else (p0, None))

    w = _f64_terms(fam, dp, *params(P), C, shared, extent, False)
    ref = _f64_reduce(f64, idx, valid, cnt, w, reduction)
    fa = f64.detach().abs().requires_grad_(True)
    wa = _f64_terms(fam, dp, *params(Pa), C, shared, extent, True)
    scale = _f64_reduce(fa, idx, valid, cnt, wa, reduction)
    if reduction == "max":
        scale = torch.maximum(scale, ref.abs())
    err = (agg.double() - ref.detach()).abs()
    bad = err > TOL * scale.detach()
    worst = float((err / scale.detach().clamp(min=1e-30)).max())
    print(f"\nOP {fam_name} {reduction} C={C}: fwd {worst:.2e}")
    assert not bad.any(), f"{int(bad.sum())} elements, first (b,c,m) {bad.nonzero()[0].tolist()}, worst {worst}"
    assert per_channel_err(agg, ref.detach())[0] <= TOL
    if reduction == "max":   # the backward of the max routes through the forward's arg-max: see the module tests
        return

    gout = torch.randn(B, C, M, generator=g).to(cuda)
    csr_off, csr_ent = ops.build_csr(idx, ncount, N)
    gfeat, pg = ops.agg_bwd(fam, red, ops.to_point_major(gout), feat_pm, q, s, ncount, csr_off, csr_ent, p0, p1, C, N,
                            K, r, normalize, shared, nkp, extent, 0)
    grads = torch.autograd.grad(ref, [f64] + P, gout.double())
    grads_a = torch.autograd.grad(scale, [fa] + Pa, gout.double().abs())
    e = (gfeat.double() - grads[0]).abs()
    worst = float((e / grads_a[0].clamp(min=1e-30)).max())
    print(f"OP {fam_name} {reduction} C={C}: grad_features {worst:.2e}")
    assert (e <= TOL * grads_a[0]).all(), f"grad_features: worst {worst}"
    assert per_channel_err(gfeat, grads[0])[0] <= TOL
    if fam == ops.FAM_ADAPTIVE_DP:      # pg rows: d/d(Wx, Wy, Wz, bias) per channel (shared = 1)
        got = [pg[:3].t(), pg[3]]
    elif fam == ops.FAM_PSEUDOGRID:
        got = [pg]
    else:
        got = []
    for k, (a, b, sc) in enumerate(zip(got, grads[1:], grads_a[1:])):
        e = (a.double() - b).abs()
        worst = float((e / sc.clamp(min=1e-30)).max())
        print(f"OP {fam_name} {reduction} C={C}: param {k} {worst:.2e}")
        assert (e <= TOL * sc).all(), f"param grad {k}: worst {worst}"


# --------------------------------------------------------------------------------------------------------------
# CPU: the dispatch rules, restated, and the instances the case tables above reach
# --------------------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


def _padded(C):
    return (C + 7) & ~7


def agg_instance(C, pg=False):
    """agg.cu:851-855 pick_ci (cap kMaxCI = 6, agg_common.cuh:10; PseudoGrid 3) and launch_fwd's chunk count
    (agg.cu:826) -> (CI, chunks)"""
    Cp = _padded(C)
    ci = min(_cdiv(Cp, 32), 3 if pg else 6)
    return ci, _cdiv(Cp, 32 * ci)


def sincos_instance(C):
    """agg.cu:890-897 dispatch_sincos and launch_sincos' grid (agg.cu:877) -> (PI, gridDim.y)"""
    pi = min(_cdiv(C // 2, 32), 3)
    return pi, _cdiv(C // 2, 32 * pi)


def aggmax_instance(C):
    """agg_max.cu:250-256 pick_max (1, 2, else 3 channels per lane) and launch_max's grid (agg_max.cu:241)"""
    Cp = _padded(C)
    ci = min(_cdiv(Cp, 32), 3)
    return ci, _cdiv(Cp, 32 * ci)


def pg2_chunks(C):
    """pg.cu:206-207 pg_num_chunks / pg_chunk_width and pg2_kernel's per-chunk widths (pg.cu:237-240) -> list of
    (Cw, Cv) per chunk"""
    Cp = _padded(C)
    n = _cdiv(Cp, 128)
    W = (_cdiv(Cp, n) + 3) // 4 * 4
    return [(min(W, Cp - y * W), min(min(W, Cp - y * W), C - y * W)) for y in range(n)]


def pwmlp_instance(C):
    """pwmlp.cu:492-495 pw_ci (cap kPWMaxCI = 4) and launch_pw_fwd's grid (pwmlp.cu:503) -> (CI, chunks)"""
    Cop = _padded(C)
    ci = min(_cdiv(Cop, 32), 4)
    return ci, _cdiv(Cop, 32 * ci)


def pwmlp_ffma_products(C):
    """gemm.cu:321: AUTO sends an un-split product with k > 512 to the FMA kernel.  pwmlp.py:28 (k = Cpa) and
    pwmlp.py:71 (k = 2 Cop) are un-split -> how many of the two take the FMA kernel"""
    return int(_padded(C + 3) > 512) + int(2 * _padded(C) > 512)


def test_case_tables_reach_every_instance():
    mod = STAGE_CASES + EXTRA_CASES

    def widths(la_type, key=None, val=None):
        return {c[2] for c in mod if c[0] == la_type and (key is None or c[1][la_type].get(key) == val)}

    def fused(la_type, pe, reductions):
        return {c[2] for c in mod if c[0] == la_type and c[1][la_type].get("position_embedding", pe) == pe
                and c[1][la_type].get("reduction") in reductions}

    sum_red = ("avg", "sum")
    xyz, sincos = fused("pospool", "xyz", sum_red), fused("pospool", "sin_cos", sum_red)
    aw = fused("adaptive_weight", None, sum_red)
    # agg_fwd/bwd_kernel<*, 4>, every AdaptiveWeight instance, and multi-chunk launches
    assert 4 in {agg_instance(C)[0] for C in xyz}
    assert {agg_instance(C)[0] for C in aw} >= {1, 2, 4, 5, 6}
    assert max(agg_instance(C)[1] for C in xyz) >= 3 and max(agg_instance(C)[1] for C in aw) >= 3
    # sin_cos: PI = 1 and gridDim.y > 1 (the p0 > 0 pair lanes)
    assert 1 in {sincos_instance(C)[0] for C in sincos}
    assert max(sincos_instance(C)[1] for C in sincos) > 1
    # chunked PseudoGrid with an uneven last chunk, and with Cv < Cw in it
    pg = widths("pseudo_grid")
    assert any(len({cw for cw, _ in pg2_chunks(C)}) > 1 for C in pg)
    assert any(pg2_chunks(C)[-1][1] < pg2_chunks(C)[-1][0] for C in pg)
    # max reductions: >= 3 chunks for xyz and AdaptiveWeight, > 1 for sin_cos, an uneven last chunk
    mx = ("max",)
    assert max(aggmax_instance(C)[1] for C in fused("pospool", "xyz", mx)) >= 3
    assert max(aggmax_instance(C)[1] for C in fused("adaptive_weight", None, mx)) >= 3
    assert max(aggmax_instance(C)[1] for C in fused("pospool", "sin_cos", mx)) > 1
    assert any(_padded(C) % 96 for C in fused("pospool", "xyz", mx) if aggmax_instance(C)[1] > 1)
    # PointWiseMLP: > 2 output-channel chunks, and both un-split products on the FMA kernel
    pw = widths("pointwisemlp")
    assert max(pwmlp_instance(C)[1] for C in pw) > 2
    assert max(pwmlp_ffma_products(C) for C in pw) == 2
    # the operator-level table reaches the same chunked instances
    ops_c = {(f, r): C for f, r, C, _ in OP_CASES}
    assert agg_instance(ops_c[("xyz", "avg")])[0] == 4
    assert sincos_instance(ops_c[("sincos", "avg")])[1] > 1
    assert pg2_chunks(260)[-1] == (88, 84) and {cw for cw, _ in pg2_chunks(576)} == {116, 112}
    # and the widths of the shipped networks
    assert {C for C, _, _, _ in SCENE} == {72, 144, 288, 576, 1152}
    assert {C for C, _, _, _ in SCENE_X2} == {144, 288, 576, 1152, 2304}
