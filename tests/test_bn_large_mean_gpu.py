"""GPU: the training-mode BatchNorm statistics of every fused forward on channels whose mean dwarfs their spread.

Each forward writes per-tile moments (n, a centre c, sum (x - c), sum (x - c)^2) and cl3d_bn_finalize merges them in
double.  Raw fp32 sums of x and x^2 would lose about (mean/std)^2 * 2^-24 of the variance; nn.BatchNorm on CUDA
(Welford) has no such limit, and these layers replace it.

Inputs.  A strided layer per cloud: queries in a ball of radius rho*r around q0, supports in a ball of radius rho*r
around q0 + 0.8 r x, so every support is a neighbour of every query, all queries share their neighbours, and the
relative positions dp differ between queries by ~rho.  Features are off_c + sigma * noise (off_c = 0 on a quarter
of the channels).  The pre-BatchNorm value of every family then has |mean|/std ~ min(1/rho, off/sigma) on the offset
channels (PointWiseMLP's BatchNorm2d also spans the K neighbours, whose features differ by sigma).  rho and sigma
scale together with one factor, set from a first run so that the largest |mean|/std over the channels, measured in float64, lands on the target
(1e2, 1e3, 1e4), and the test asserts that it is within 2x of it.

Checks.
  1. statistics alone: save_stats and running_var of ops.bn_finalize(momentum=1) on the forward's own partials against
     the float64 mean and variance of the fp32 values that forward produced (PointWiseMLP never stores its B*M*K
     values y: they are rebuilt in float64 from the a' and T rows it read, y = a' + sgn * T[j_k]).  Bars: mean
     <= 1e-6 |mean| + 1e-7 std, variance <= 1e-5 relative.  A constant channel gives variance 0 exactly.
  2. the module, forward and backward, against the float64 reference, next to the same comparison for the
     reference's own fp32 composition (la_oracle in fp32 on the GPU, TF32 off): (x - mean) in fp32 loses
     ratio * 2^-24 of the spread in any fp32 implementation, so a fixed bar cannot hold at 1e4; the bar is
     err <= 2 err_ref32 + floor (1e-5 outputs and feature gradients, 5e-5 parameter gradients).
  3. two runs give the same partials and statistics bit for bit; a CUDA-graph replay equals the eager call.
"""
import contextlib
import copy
import math
import os

import pytest
import torch

from closerlook3d_b200 import ops
from closerlook3d_b200.config import la_config

pytestmark = pytest.mark.gpu

XYZ = lambda red: dict(pospool=dict(position_embedding="xyz", reduction=red))           # noqa: E731
SINCOS = lambda red: dict(pospool=dict(position_embedding="sin_cos", reduction=red))    # noqa: E731
AW = lambda red: dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1, reduction=red))  # noqa
PW = dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))

# one case per producer of BatchNorm partials: id -> (la_type, config override, C)
CASES = {
    "agg-xyz-avg": ("pospool", XYZ("avg"), 24),
    "agg-xyz-sum": ("pospool", XYZ("sum"), 24),
    "agg-aw-avg": ("adaptive_weight", AW("avg"), 24),
    "sincos-avg": ("pospool", SINCOS("avg"), 24),
    "aggmax-xyz": ("pospool", XYZ("max"), 24),
    "aggmax-sincos": ("pospool", SINCOS("max"), 24),
    "aggmax-aw": ("adaptive_weight", AW("max"), 24),
    "pg2-72": ("pseudo_grid", {}, 72),
    "pg2-144": ("pseudo_grid", {}, 144),          # two channel chunks
    "pg3-36": ("pseudo_grid", {}, 36),
    "pwmlp-72": ("pointwisemlp", PW, 72),
    "pwmlp-160": ("pointwisemlp", PW, 160),       # two output chunks of the forward
}
RATIOS = [1e2, 1e3, 1e4]
B, N, K = 2, 48, 16
M_ODD = 301                                           # last tile of each cloud partial


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def make_inputs(C, M, lam, seed, padded=False, const_channel=False):
    """rho = lam, sigma = 30 lam: both sources of spread (the queries' jitter; the features, which differ between the
    clouds and between a query's neighbours) scale together, so |mean|/std ~ 1 / lam in every family"""
    g = torch.Generator().manual_seed(seed)
    r = 0.1

    def ball(b, n):
        u = torch.randn(b, n, 3, generator=g, dtype=torch.float64)
        return u / u.norm(dim=-1, keepdim=True) * torch.rand(b, n, 1, generator=g, dtype=torch.float64) ** (1 / 3)

    q0 = 0.05 * torch.rand(1, 1, 3, generator=g, dtype=torch.float64)
    q = (q0 + lam * r * ball(B, M)).float().contiguous()
    s = (q0 + torch.tensor([0.8 * r, 0.0, 0.0], dtype=torch.float64) + lam * r * ball(1, N)).expand(B, N, 3)
    off = 1.0 + torch.rand(C, generator=g)
    off[::4] = 0.0                                            # ordinary channels beside the extreme ones
    sigma = torch.full((C,), 30.0 * lam)
    if const_channel:
        off[1], sigma[1] = 0.75, 0.0
    feats = off[None, :, None] + sigma[None, :, None] * torch.randn(B, C, N, generator=g)
    qm = torch.ones(B, M, dtype=torch.int32)
    if padded:
        qm[:, M - 3:] = 0
    return r, q, s.float().contiguous(), qm, torch.ones(B, N, dtype=torch.int32), feats.float().contiguous()


def make_module(la_type, over, C, r, seed, const_channel=False):
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    torch.manual_seed(seed)
    mod = LocalAggregation(C, C, r, K, la_config(la_type, **over))
    with torch.no_grad():
        for name, p in mod.named_parameters():
            if name.endswith("kernel_weights"):
                p.copy_(1.0 + 0.5 * torch.rand(p.shape))      # keeps PseudoGrid's offset channels offset
        if la_type == "pseudo_grid":   # a kernel point near dp = 0.8 r x, on the slope of its influence
            mod.local_aggregation_operator.K_points[1] = torch.tensor([0.75 * r, 0.0, 0.0])
        if const_channel:
            mod.local_aggregation_operator.mlps.conv0.weight[1].zero_()   # AdaptiveWeight: w = bias on channel 1
    return mod


class Capture:
    """records what the module's forward hands to ops.bn_finalize: the values it normalises and the partials"""

    def __init__(self, monkeypatch):
        self.calls = []
        fwd, pw = ops.agg_fwd, ops.pwmlp_fwd_stats

        def agg_fwd(*a, **k):
            agg, part = fwd(*a, **k)
            self.calls.append(dict(values=agg, partial=part))
            return agg, part

        def pwmlp_fwd_stats(ab_pm, wp, sgn, query_xyz, support_xyz, idx, Cout, radius):
            res = pw(ab_pm, wp, sgn, query_xyz, support_xyz, idx, Cout, radius)
            self.calls.append(dict(ab_pm=ab_pm, sgn=sgn, idx=idx, aq=res[1], partial=res[4], Cout=Cout))
            return res

        monkeypatch.setattr(ops, "agg_fwd", agg_fwd)
        monkeypatch.setattr(ops, "pwmlp_fwd_stats", pwmlp_fwd_stats)


def values64(call):
    """float64 (C, n) of the values BatchNorm normalises, as the kernel formed them"""
    if "values" in call:
        v = call["values"].double()                           # (B,C,M)
        return v.transpose(0, 1).reshape(v.shape[1], -1)
    Cout, aq, idx = call["Cout"], call["aq"].double(), call["idx"].long()
    Bq, Np, W = call["ab_pm"].shape
    Cop = W // 2
    T = call["ab_pm"][..., Cop:Cop + Cout].double() * call["sgn"].double()            # (B,N,Cout) sgn * T = bv
    Tk = torch.gather(T, 1, idx.reshape(Bq, -1, 1).expand(-1, -1, Cout)).view(*idx.shape, Cout)   # (B,M,K,Cout)
    y = aq[:, :, None, :Cout] + Tk                                                   # a' + bv[j_k]
    return y.permute(3, 0, 1, 2).reshape(Cout, -1)


def run_forward(cuda, case, M, target, seed, padded=False, const_channel=False, monkeypatch=None, lam=None):
    la_type, over, C = CASES[case]

    def once(lam):
        r, q, s, qm, sm, feats = make_inputs(C, M, lam, seed, padded, const_channel)
        mod = make_module(la_type, over, C, r, seed, const_channel).to(cuda).train()
        cap = Capture(monkeypatch)
        mod(q.to(cuda), s.to(cuda), qm.to(cuda), sm.to(cuda), feats.to(cuda))
        torch.cuda.synchronize()
        monkeypatch.undo()
        assert len(cap.calls) == 1
        x = values64(cap.calls[0])
        ratio = (x.mean(1).abs() / x.std(1, unbiased=False).clamp(min=1e-300))
        ratio[x.std(1) == 0] = 0
        return cap.calls[0], x, float(ratio.max())

    if lam is None:   # ratio ~ lam^-p (p = 1; 2 on sin_cos channels near cos = 1): fit p from two runs
        _, _, r1 = once(1e-2)
        _, _, r2 = once(1e-3)
        p = max(0.5, math.log10(r2 / r1))
        lam = 1e-2 * (r1 / target) ** (1.0 / p)
    call, x, ratio = once(lam)
    return call, x, ratio, lam


def check_stats(call, x, C, tag):
    n = x.shape[1]
    rm = torch.zeros(C, device=x.device)
    rv = torch.ones(C, device=x.device)
    stats = ops.bn_finalize(call["partial"], C, n, 1e-5, 1.0, True, rm, rv)
    torch.cuda.synchronize()
    mean, var = x.mean(1), x.var(1, unbiased=False)
    std = var.sqrt()
    e_mean = (stats[0].double() - mean).abs()
    assert torch.equal(stats[0], rm), "running_mean at momentum 1 is the batch mean"
    var_k = rv.double() * (n - 1) / n                            # unbiased running_var -> batch variance
    e_var = (var_k - var).abs()
    bad_m = e_mean > 1e-6 * mean.abs() + 1e-7 * std
    bad_v = e_var > 1e-5 * var
    rel_v = float((e_var / var.clamp(min=1e-300)).max())
    print(f"{tag}: max rel var err {rel_v:.2e}, max mean err / (|mean|+std) "
          f"{float((e_mean / (mean.abs() + std)).max()):.2e}")
    assert not bool(bad_m.any()), f"{tag}: mean off on channels {bad_m.nonzero().flatten().tolist()[:8]}"
    assert not bool(bad_v.any()), f"{tag}: variance off by up to {rel_v:.2e} (channels " \
                                  f"{bad_v.nonzero().flatten().tolist()[:8]})"
    inv = 1.0 / (var + 1e-5).sqrt()
    assert float(((stats[1].double() - inv).abs() / inv).max()) <= 1e-5
    return stats, rv


# ---------------------------------------------------------------------------------------------------------------
# 1. statistics
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("target", RATIOS, ids=lambda t: f"ratio{t:.0e}")
@pytest.mark.parametrize("case", list(CASES))
def test_bn_statistics_large_mean(cuda, monkeypatch, case, target):
    call, x, ratio, _ = run_forward(cuda, case, M_ODD, target, 11, monkeypatch=monkeypatch)
    assert target / 2 <= ratio <= 2 * target, f"construction gave ratio {ratio:.3g}, target {target:.0e}"
    check_stats(call, x, CASES[case][2], f"{case} ratio {ratio:.3g}")


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("shape", ["small_m", "padded", "max_grid5"])
def test_bn_statistics_edges(cuda, monkeypatch, case, shape):
    """M < 32 (one partial tile per cloud); padded queries, which count in BatchNorm as in the reference (their
    value -- 0 for avg / sum, the masked aggregate otherwise -- sits far from the others, so the ratio is not asserted
    there); five CTAs for the whole grid, so the persistent tile loops take many tiles each"""
    M = 20 if shape == "small_m" else M_ODD
    grid = {"CL3D_TEST_MAX_GRID": "5"} if shape == "max_grid5" else {}
    with env(**grid):
        call, x, ratio, _ = run_forward(cuda, case, M, 1e3, 23, padded=shape == "padded", monkeypatch=monkeypatch)
    if shape != "padded":
        assert 5e2 <= ratio <= 2e3, ratio
    check_stats(call, x, CASES[case][2], f"{case} {shape} ratio {ratio:.3g}")


def test_bn_statistics_constant_channel(cuda, monkeypatch):
    """AdaptiveWeight with W = 0 and a feature without noise on channel 1: every query aggregates the same value, so
    its variance is 0 exactly and running_var decays as torch's (1 - m) * old"""
    call, x, ratio, _ = run_forward(cuda, "agg-aw-avg", M_ODD, 1e3, 5, const_channel=True, monkeypatch=monkeypatch)
    assert float(x[1].std()) == 0.0
    C = CASES["agg-aw-avg"][2]
    check_stats(call, x, C, "constant channel")
    old = torch.rand(C, device=cuda) + 0.5
    rm, rv = torch.zeros(C, device=cuda), old.clone()
    stats = ops.bn_finalize(call["partial"], C, x.shape[1], 1e-5, 0.1, True, rm, rv)
    torch.cuda.synchronize()
    assert float(stats[1][1]) == pytest.approx(1.0 / (1e-5) ** 0.5, rel=1e-6)
    assert float(rv[1]) == float(((1 - torch.tensor(0.1, dtype=torch.float64)) * old[1].double()).float())


# ---------------------------------------------------------------------------------------------------------------
# 2. the module against float64, beside the reference's fp32 composition
# ---------------------------------------------------------------------------------------------------------------
def _rel(a, b):
    return float((a.double() - b.double()).abs().max()) / max(1e-30, float(b.abs().max()))


@pytest.mark.parametrize("target", RATIOS, ids=lambda t: f"ratio{t:.0e}")
@pytest.mark.parametrize("case", list(CASES))
def test_module_large_mean_matches_f64_like_fp32_reference(cuda, monkeypatch, case, target):
    from oracle import f64_ext, la_oracle
    la_type, over, C = CASES[case]
    _, _, _, rho = run_forward(cuda, case, M_ODD, target, 31, monkeypatch=monkeypatch)
    r, q, s, qm, sm, feats = make_inputs(C, M_ODD, rho, 31)
    mod = make_module(la_type, over, C, r, 31)
    with torch.no_grad():   # BatchNorm gamma / beta of a trained layer, not the identity
        for name, p in mod.named_parameters():
            if name.endswith((".1.weight", "out_transform.0.weight")):
                p.copy_(0.5 + torch.rand(p.shape))
            elif name.endswith((".1.bias", "out_transform.0.bias")):
                p.copy_(0.5 * torch.randn(p.shape))
    sd = copy.deepcopy(mod.state_dict())
    qd, sd_xyz, qmd, smd = q.to(cuda), s.to(cuda), qm.to(cuda), sm.to(cuda)
    cfg = la_config(la_type, **over)
    la_oracle.GPU_SCALAR_DIVISION = True
    la_oracle.DIM_MAT_FN = lambda fd: torch.pow(
        1.0 * 1000, (1.0 / fd) * torch.arange(fd, dtype=torch.float32).to(cuda)).cpu()
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    runs = {}
    try:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        for name, dt in (("f64", torch.float64), ("ref32", None)):
            la_oracle.KEEP = {}
            # f64_ext groups by a plain gather in the features' dtype: the fp32 run is the reference's composition
            orc = la_oracle.OracleLocalAggregation(f64_ext, la_type, C, C, r, K, cfg, sd, device=cuda, dtype=dt)
            f = feats.to(cuda, dt or torch.float32).requires_grad_(True)
            o = orc(qd, sd_xyz, qmd, smd, f)
            runs[name] = dict(out=o, f=f, orc=orc, keep=la_oracle.KEEP)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        la_oracle.GPU_SCALAR_DIVISION = False
        la_oracle.DIM_MAT_FN = None
        la_oracle.KEEP = None
    mod = mod.to(cuda).train()
    f = feats.to(cuda).requires_grad_(True)
    out = mod(qd, sd_xyz, qmd, smd, f)
    ref = runs["f64"]["out"].detach()
    # upstream gradient: zero where the final ReLU or an arg-max is decided by rounding in either fp32 path
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64).to(cuda)
    for o in (out, runs["ref32"]["out"]):
        gout = gout * ((o.detach() > 0) == (ref > 0))
    keep = runs["f64"]["keep"]
    if "pwmlp_premax" in keep:
        gout = gout * la_oracle.argmax_is_decided(keep["pwmlp_premax"], keep["idx"])
    elif "premax" in keep:
        gout = gout * la_oracle.argmax_is_decided(keep["premax"], keep["idx"], rel=2e-6, relu=False)
    (runs["f64"]["out"] * gout).sum().backward()
    (runs["ref32"]["out"] * gout.float()).sum().backward()
    (out * gout.float()).sum().backward()
    torch.cuda.synchronize()

    def errs(o, fgrad, grads, state):
        e = {"out": _rel(o.detach(), ref), "grad_features": _rel(fgrad, runs["f64"]["f"].grad)}
        g64 = runs["f64"]["orc"].grads()
        for k, v in grads.items():
            e["grad " + k] = _rel(v, g64[k])
        for k, v in runs["f64"]["orc"].st.items():
            if k.endswith(("running_mean", "running_var")):
                e[k] = _rel(state[k], v)
        return e

    ours = errs(out, f.grad, {n[len("local_aggregation_operator."):]: p.grad for n, p in mod.named_parameters()},
                {k[len("local_aggregation_operator."):]: v for k, v in mod.state_dict().items()})
    o32 = runs["ref32"]["orc"]
    ref32 = errs(runs["ref32"]["out"], runs["ref32"]["f"].grad, o32.grads(), o32.st)
    print(f"\n{case} rho {rho:.2e}: " + ", ".join(f"{k} {ours[k]:.2e}/{ref32[k]:.2e}" for k in ours))
    for k, e in ours.items():
        floor = 5e-5 if k.startswith("grad ") else 1e-5
        assert e <= 2 * ref32[k] + floor, f"{k}: {e:.2e} against the fp32 reference's {ref32[k]:.2e}"


# ---------------------------------------------------------------------------------------------------------------
# 3. determinism and graphs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_bn_partials_repeat_and_graph_replay(cuda, monkeypatch, case):
    la_type, over, C = CASES[case]
    call, x, ratio, rho = run_forward(cuda, case, M_ODD, 1e3, 41, monkeypatch=monkeypatch)
    call2, _, _, _ = run_forward(cuda, case, M_ODD, 1e3, 41, monkeypatch=monkeypatch, lam=rho)
    assert torch.equal(call["partial"], call2["partial"]), "two runs give different partials"
    n = x.shape[1]

    def fin(p, rm, rv):
        return ops.bn_finalize(p, C, n, 1e-5, 0.1, True, rm, rv)

    st = [(torch.zeros(C, device=cuda), torch.ones(C, device=cuda)) for _ in range(3)]
    s1, s2 = fin(call["partial"], *st[0]), fin(call2["partial"], *st[1])
    torch.cuda.synchronize()
    assert torch.equal(s1, s2) and torch.equal(st[0][0], st[1][0]) and torch.equal(st[0][1], st[1][1])
    if "values" not in call:
        return   # PointWiseMLP: its forward is graph-replayed with the module in test_graphed_gpu.py
    # graph: ops.agg_fwd then ops.bn_finalize, captured with the inputs of the module's call
    r, q, s, qm, sm, feats = make_inputs(C, M_ODD, rho, 41)
    mod = make_module(la_type, over, C, r, 41).to(cuda).train()
    args = []

    def rec(*a, **k):
        args.append((a, k))
        return fwd(*a, **k)

    fwd = ops.agg_fwd
    monkeypatch.setattr(ops, "agg_fwd", rec)
    mod(q.to(cuda), s.to(cuda), qm.to(cuda), sm.to(cuda), feats.to(cuda))
    monkeypatch.undo()
    a, k = args[0]
    eager_agg, eager_part = fwd(*a, **k)
    eager = fin(eager_part, *st[2])
    torch.cuda.synchronize()
    rm, rv = torch.zeros(C, device=cuda), torch.ones(C, device=cuda)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fin(fwd(*a, **k)[1], rm.clone(), rv.clone())
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_agg, g_part = fwd(*a, **k)
        g_stats = fin(g_part, rm, rv)
    g_agg.zero_()
    g_part.zero_()
    g_stats.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_agg, eager_agg) and torch.equal(g_part, eager_part) and torch.equal(g_stats, eager)
    assert torch.equal(rm, st[2][0]) and torch.equal(rv, st[2][1])
