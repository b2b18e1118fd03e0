"""GPU: float16 / bfloat16 features through every fused operator.

The rule (include/cl3d.h, CL3D_DTYPE_*): the features set the dtype of the output and of d/dfeatures; inside, every
buffer and every operation is fp32, and the only roundings are the one widening (exact) where the features enter and
the one narrowing where an output or gradient is stored.  So each operator on 16-bit features must give exactly
its fp32 result on the widened features, rounded once:  op(f_h) == op(f_h.float()).to(f_h.dtype).

Both arms of a comparison share their neighbour lists (the neighbour cache is keyed on the xyz tensors), so the
gather-form backward sums in the same order in both: bit-identical gradients where the path has no float atomics.
Paths with fp32 atomics (PointWiseMLP's red.add, the max-pool / grouping scatters) sum in a different order on every
run; there the 16-bit gradient must lie within one unit in the last place of the 16-bit type plus twice the
run-to-run spread of the fp32 arm, measured in the same test (a sum with cancellation can move by more than one
16-bit ulp of its small result from the order alone).
"""
import copy
import importlib.util
import os

import numpy as np
import pytest
import torch

from closerlook3d_b200 import synth
from closerlook3d_b200.config import la_config

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
_HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    spec = importlib.util.spec_from_file_location(f"_rp_{name}", os.path.join(_HERE, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


wide = _load("test_wide_layers_gpu")

# every kernel instance the wide-layer tables reach, plus the BASELINE c3 layer (PseudoGrid, K = 26, C = 72; B = 2
# instead of 8) and an odd N (16-bit channel-major rows only 2-byte aligned)
CASES = wide.STAGE_CASES + wide.EXTRA_CASES + [
    ("pseudo_grid", wide.PG, 72, 15000, 15000, 26, True),
    ("pseudo_grid", wide.PG, 72, 1001, 2049, 24, True),
    ("pospool", wide.XYZ_AVG, 72, 1001, 2049, 24, True),
    ("pospool", wide.SINCOS_MAX, 144, 1001, 2049, 24, True),
    ("adaptive_weight", wide.AW, 72, 1001, 2049, 24, True),
    ("pointwisemlp", wide.PW, 72, 1001, 2049, 24, True),
]


def ulp(x, dt):
    """one unit in the last place of dt at the magnitude of x (x in dt, returned as fp32)"""
    p, emin = (7, -126) if dt == torch.bfloat16 else (10, -14)
    _, e = torch.frexp(x.float())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float32), (e - 1).clamp(min=emin) - p)


def assert_within_ulp(a, b, dt, b2=None):
    """a (dt) within one ulp of dt of b, plus twice max|b - b2| when a second run b2 of the same arm is given"""
    assert a.dtype == dt
    spread = 0.0 if b2 is None else float((b.float() - b2.float()).abs().max())
    bh = b.to(dt)
    fin = torch.isfinite(bh)
    assert torch.equal(torch.isfinite(a), fin)
    d = (a.float() - bh.float()).abs()[fin]
    assert bool((d <= ulp(bh, dt)[fin] + 2 * spread).all()), (float(d.max()), spread)


def _two_arms(la_type, over, C, M, N, K, train, dt, cuda, seed):
    from closerlook3d_b200 import pt_utils
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    cfg = la_config(la_type, **over)
    torch.manual_seed(seed)
    np.random.seed(seed)
    r, xyz, mask, q, qm, feats = wide._cloud(2, C, M, N, K, seed)
    mod = LocalAggregation(C, C, r, K, cfg)
    wide._randomize_bn(mod, seed)
    mod = mod.to(cuda).train(train)
    mods = (copy.deepcopy(mod), copy.deepcopy(mod))
    xyz, mask, q, qm = xyz.to(cuda), mask.to(cuda), q.to(cuda), qm.to(cuda)
    f_h = feats.to(cuda, dt)
    gout = torch.randn(2, C, M, generator=torch.Generator().manual_seed(seed + 2)).to(cuda, dt)
    pt_utils.clear_neighbor_cache()
    res = []
    arms = [(mods[0], f_h, gout), (mods[1], f_h.float(), gout.float())]
    if la_type == "pointwisemlp":   # fp32 atomics: a second fp32 run measures the order spread
        arms.append((copy.deepcopy(mod), f_h.float(), gout.float()))
    for m, f, g in arms:
        f = f.clone().requires_grad_(True)
        out = m(q, xyz, qm, mask, f)
        out.backward(g)
        res.append((m, out.detach(), f.grad))
    pt_utils.clear_neighbor_cache()
    return res


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", CASES, ids=[wide._case_id(c) for c in CASES])
def test_operator_equals_fp32_on_widened_input(cuda, case, dt):
    la_type, over, C, M, N, K, train = case
    runs = _two_arms(la_type, over, C, M, N, K, train, dt, cuda, 9000 + C + M + K)
    (ma, out_a, g_a), (mb, out_b, g_b) = runs[:2]
    assert out_a.dtype == dt and g_a.dtype == dt
    assert torch.equal(out_a, out_b.to(dt))
    for (na, ba), (_, bb) in zip(ma.named_buffers(), mb.named_buffers()):
        assert torch.equal(ba, bb), na
    pw = la_type == "pointwisemlp"
    if pw:
        assert_within_ulp(g_a, g_b, dt, runs[2][2])
    else:
        assert torch.equal(g_a, g_b.to(dt))
    for (n, pa), (_, pb) in zip(ma.named_parameters(), mb.named_parameters()):
        assert pa.grad.dtype == torch.float32, n
        if pw:
            assert float((pa.grad - pb.grad).abs().max()) <= 1e-4 * max(1.0, float(pb.grad.abs().max())), n
        else:
            assert torch.equal(pa.grad, pb.grad), n


def _masked_inputs(cuda, dt, C=40, N=2049, seed=5):
    d = synth.make_cloud_batch(2, N, C, seed)
    return d["xyz"].to(cuda), d["mask"].to(cuda), d["features"].to(cuda, dt)


def _check_pair(fn, f_h, gshape_seed, dt):
    """fn(features) -> tensor; both arms, then output equality and gradients within one ulp"""
    fa = f_h.clone().requires_grad_(True)
    fb = f_h.float().requires_grad_(True)
    fc = f_h.float().requires_grad_(True)
    oa, ob, oc = fn(fa), fn(fb), fn(fc)
    assert oa.dtype == dt and torch.equal(oa, ob.to(dt))
    g = torch.randn(oa.shape, generator=torch.Generator().manual_seed(gshape_seed)).to(oa.device, dt)
    oa.backward(g)
    ob.backward(g.float())
    oc.backward(g.float())
    assert_within_ulp(fa.grad, fb.grad, dt, fc.grad)


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "fp16"])
def test_masked_layers_and_grouping(cuda, dt):
    from closerlook3d_b200 import pt_utils
    xyz, mask, f_h = _masked_inputs(cuda, dt)
    r = synth.ball_radius(2049, 24)
    pool = pt_utils.MaskedMaxPool(512, r, 24, r / 2)
    _check_pair(lambda f: pool(xyz, mask, f)[2], f_h, 1, dt)
    sub_xyz, sub_mask, _ = pool(xyz, mask, f_h)
    coarse = torch.randn(2, 40, sub_xyz.shape[1], generator=torch.Generator().manual_seed(2)).to(cuda, dt)
    for mode in ("nearest", "max"):
        up = pt_utils.MaskedUpsample(r, 24, mode=mode)
        _check_pair(lambda f: up(xyz, sub_xyz, mask, sub_mask, f), coarse, 3, dt)
    idx, _ = pt_utils.masked_ordered_ball_query(r, 24, sub_xyz, xyz, sub_mask, mask)
    _check_pair(lambda f: pt_utils.grouping_operation(f, idx), f_h, 4, dt)


def test_fp16_overflow_is_inf_where_the_cast_gives_inf_and_gradscaler_skips(cuda):
    """BatchNorm gamma 2e4 pushes outputs and gradients past 65504: the native path must give inf exactly where
    .to(float16) of the fp32 result does, and a GradScaler step over the fp32 parameter that fed the features skips."""
    from closerlook3d_b200 import pt_utils
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    dt, C, N, K = torch.float16, 72, 2049, 24
    torch.manual_seed(1)
    np.random.seed(1)
    d = synth.make_cloud_batch(2, N, C, 11)
    xyz, mask = d["xyz"].to(cuda), d["mask"].to(cuda)
    mod = LocalAggregation(C, C, synth.ball_radius(N, K), K, la_config("pseudo_grid")).to(cuda).train()
    with torch.no_grad():
        mod.local_aggregation_operator.out_transform[0].weight.fill_(2e4)
    ma, mb = copy.deepcopy(mod), copy.deepcopy(mod)
    x = torch.nn.Parameter(d["features"].to(cuda))          # fp32 leaf whose fp16 cast feeds the layer
    gout = torch.full((2, C, N), 1000.0, device=cuda, dtype=dt)
    pt_utils.clear_neighbor_cache()
    f_h = x.to(dt)
    out_a = ma(xyz, xyz, mask, mask, f_h)
    fb = f_h.detach().float().requires_grad_(True)
    out_b = mb(xyz, xyz, mask, mask, fb)
    assert bool(torch.isinf(out_b.to(dt)).any())
    assert torch.equal(out_a, out_b.detach().to(dt))
    scaler = torch.amp.GradScaler("cuda", init_scale=1.0)
    opt = torch.optim.SGD([x], lr=0.1)
    x0 = x.detach().clone()
    f_h.retain_grad()
    scaler.scale((out_a.float() * gout.float()).sum()).backward()
    (out_b * gout.float()).sum().backward()
    pt_utils.clear_neighbor_cache()
    ref = fb.grad.to(dt)
    assert bool(torch.isinf(ref).any())
    assert torch.equal(f_h.grad, ref)     # PseudoGrid: no float atomics, so the finite values agree too
    assert torch.equal(torch.isinf(f_h.grad), torch.isinf(ref))
    scaler.step(opt)
    scaler.update()
    assert torch.equal(x.detach(), x0)          # step skipped
    assert scaler.get_scale() < 1.0


# ---- whole networks under torch.autocast --------------------------------------------------------------------------
def _net_cfg(task, la, over):
    from closerlook3d_b200.backbone import model_config
    c = model_config(task, la, **over, **(dict(dataset="shapenetpart") if task == "multi_part_segmentation" else {}))
    c.width = 24
    c.radius, c.sampleDl = 0.06, 0.03
    c.npoints = [1024, 320, 96, 32]
    c.nsamples = [16, 18, 20, 18, 16]
    if task != "multi_part_segmentation":
        c.num_classes = 9
    return c


NETS = [
    ("classification", "pospool", dict(pospool=dict(position_embedding="xyz", reduction="avg"))),
    ("scene_segmentation", "pseudo_grid", dict()),
    ("multi_part_segmentation", "adaptive_weight",
     dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1, reduction="avg"))),
]


def _patch_to_upcast(model):
    """arm B: every fused module runs its fp32 path on the widened features and casts the result back"""
    from closerlook3d_b200 import pt_utils
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    for m in model.modules():
        if isinstance(m, (LocalAggregation, pt_utils.MaskedUpsample)):
            def fwd(*a, _f=m.forward):
                return _f(*a[:4], a[4].float()).to(a[4].dtype)
            m.forward = fwd
        elif isinstance(m, pt_utils.MaskedMaxPool):
            def fwd(xyz, mask, f, _f=m.forward):
                s, sm, o = _f(xyz, mask, f.float())
                return s, sm, o.to(f.dtype)
            m.forward = fwd


def _hook_16bit(model, dt, seen):
    from closerlook3d_b200 import pt_utils
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    hs = []
    for m in model.modules():
        if isinstance(m, (LocalAggregation, pt_utils.MaskedMaxPool, pt_utils.MaskedUpsample)):
            def pre(mod, args):
                assert args[-1].dtype == dt, (type(mod).__name__, args[-1].dtype)
                seen.append(type(mod).__name__)
            hs.append(m.register_forward_pre_hook(pre))
    return hs


def _net_step(model, criterion, task, dt, xyz, mask, feats, target):
    from closerlook3d_b200 import pt_utils
    pt_utils.clear_neighbor_cache()
    opt = torch.optim.SGD(model.parameters(), lr=1e-3)
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=dt):
        pred = model(xyz, mask, feats)
        if task == "classification":
            loss = criterion(pred, target)
        elif task == "multi_part_segmentation":
            loss = criterion(pred, *target)
        else:
            loss = criterion(pred, target, mask.float())
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    opt.step()
    logits = torch.cat([p.detach().float().reshape(-1) for p in (pred if isinstance(pred, (list, tuple)) else [pred])])
    return logits, float(loss), grads


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("task,la,over", NETS, ids=[f"{t[:5]}-{la}" for t, la, _ in NETS])
def test_whole_network_under_autocast(cuda, task, la, over, dt):
    from closerlook3d_b200 import backbone as bb
    cfg = _net_cfg(task, la, over)
    build = {"classification": bb.build_classification, "scene_segmentation": bb.build_scene_segmentation,
             "multi_part_segmentation": bb.build_multi_part_segmentation}[task]
    torch.manual_seed(3)
    np.random.seed(3)
    model, criterion = build(cfg)
    model.init_weights()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    B, N = 2, 3000
    d = synth.make_cloud_batch(B, N, cfg.input_features_dim, 21)
    xyz, mask, feats = d["xyz"].to(cuda), d["mask"].to(cuda), d["features"].to(cuda)
    if task == "classification":
        target = torch.randint(0, cfg.num_classes, (B,), generator=torch.Generator().manual_seed(4)).to(cuda)
    elif task == "multi_part_segmentation":
        lab = synth.make_part_labels(B, N, cfg.num_parts, 4)
        target = (lab["points_labels"].to(cuda), lab["shape_labels"].to(cuda))
    else:
        target = torch.randint(0, cfg.num_classes, (B, N), generator=torch.Generator().manual_seed(4)).to(cuda)
    sd = copy.deepcopy(model.state_dict())
    from closerlook3d_b200 import pt_utils
    det, overlap = torch.backends.cudnn.deterministic, pt_utils.overlap_enabled
    torch.backends.cudnn.deterministic = True
    # The neighbour search (whose int atomics order the transposed lists) normally runs on a side stream beside the
    # main stream's work, and that work differs between the arms (arm B adds its casts): each arm would then get its
    # own, repeatable list order.  In order on one stream, the list order depends on the search kernel alone.
    pt_utils.overlap_enabled = False
    try:
        runs = {}
        # one discarded step per arm first, then the arms alternated: every compared step runs in the same warm state
        # (the first step of a process schedules its atomics differently from the later ones)
        for arm in ("warm-native", "warm-B", "native", "B1", "N2", "B2", "N3", "B3", "N4", "B4"):
            model.load_state_dict(sd)
            m = model.to(cuda).train()
            m = copy.deepcopy(m)
            if "B" in arm:
                _patch_to_upcast(m)
            seen = []
            hs = _hook_16bit(m, dt, seen)
            runs[arm] = _net_step(m, criterion, task, dt, xyz, mask, feats, target)
            for h in hs:
                h.remove()
            assert "LocalAggregation" in seen
            if task != "classification":
                assert "MaskedUpsample" in seen
            assert "MaskedMaxPool" in seen
            assert all(torch.isfinite(p).all() for p in m.parameters())
    finally:
        torch.backends.cudnn.deterministic = det
        pt_utils.overlap_enabled = overlap
    (lo_n, loss_n, g_n), (lo_b, loss_b, g_b) = runs["native"], runs["B1"]
    g_bs = [runs[k][2] for k in ("B1", "B2", "B3", "B4")]
    g_ns = [runs[k][2] for k in ("native", "N2", "N3", "N4")]
    assert np.isfinite(loss_n) and bool(torch.isfinite(lo_n).all())
    assert torch.equal(lo_n, lo_b) and loss_n == loss_b

    # Gradients, per parameter tensor.  Native and arm B run the same fp32 arithmetic and round at the same points, so
    # they can differ only through the order of fp32 atomics: the max-pool and upsampling scatters and the transposed
    # neighbour lists the aggregation backward walks.
    #  * Parameters whose gradient the backward computes before reaching any of those (the classifier, the
    #    segmentation heads and the last decoder convolution behind the last upsampling): bit-identical.
    #  * Every other parameter: four runs of each arm measure that parameter's run-to-run spread; the closest
    #    native / arm-B pair must be no farther apart than twice the larger of the two arms' spreads (exactly equal
    #    where both arms repeat bit for bit).  Both arms sample the same atomics-order variation, and a single arm's
    #    few runs can miss it: arm B often repeats bit for bit while the native runs vary among themselves.
    assert set(g_n) == set(g_b)
    assert all(bool(torch.isfinite(g).all()) for g in g_n.values())
    atomic_free = {"classification": ("classifier.",),
                   "scene_segmentation": ("segmentation_head.head.", "segmentation_head.up_conv3."),
                   "multi_part_segmentation": ("segmentation_head.multi_shape_heads.",
                                               "segmentation_head.up_conv3.")}[task]

    def dist(a, b):
        return float((a - b).abs().max())

    n_free, bad = 0, []
    for name, g in g_n.items():
        if name.startswith(atomic_free):
            n_free += 1
            assert all(torch.equal(gn[name], gb[name]) for gn in g_ns for gb in g_bs), name
            continue
        spread_b = max(dist(a[name], b[name]) for i, a in enumerate(g_bs) for b in g_bs[i + 1:])
        spread_n = max(dist(a[name], b[name]) for i, a in enumerate(g_ns) for b in g_ns[i + 1:])
        err = min(dist(gn[name], gb[name]) for gn in g_ns for gb in g_bs)
        if err > 2 * max(spread_b, spread_n):
            bad.append((name, err, spread_b, spread_n))
    assert n_free > 0
    assert not bad, bad


# ---- CUDA graphs --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("la,over", [("pseudo_grid", dict()), ("pointwisemlp", wide.PW)])
def test_graphed_step_with_bf16_features(cuda, la, over):
    """A replay of a GraphedStep captured with bf16 example features gives the eager step's output bit for bit, which
    shows the 16-bit kernels are capturable.  The feature gradient is compared to the eager one within one bf16 ulp
    plus twice the eager step's own run-to-run spread, a deliberate relaxation of bit-identity: the eager step and the
    captured one each build their own transposed neighbour lists, whose order comes from int atomics, so the backward
    sums in a different order (the fp32 path varies the same way from run to run, BASELINE.md)."""
    from closerlook3d_b200 import pt_utils
    from closerlook3d_b200.graphed import GraphedStep
    from closerlook3d_b200.local_aggregation_operators import LocalAggregation
    dt, B, N, K, C = torch.bfloat16, 2, 2304, 16, 72
    torch.manual_seed(3)
    np.random.seed(3)
    mod = LocalAggregation(C, C, synth.ball_radius(N, K), K, la_config(la, **over)).to(cuda).train()
    b = {k: v.to(cuda) for k, v in synth.make_cloud_batch(B, N, C, 100).items()}
    feats = b["features"].to(dt)
    gout = torch.randn(B, C, N, generator=torch.Generator().manual_seed(1)).to(cuda, dt)
    was = pt_utils.cache_enabled
    pt_utils.cache_enabled = False
    try:
        eager = []
        for _ in range(2):      # twice: the run-to-run spread of the atomics-ordered backward
            f = feats.clone().requires_grad_(True)
            out_e = copy.deepcopy(mod)(b["xyz"], b["xyz"], b["mask"], b["mask"], f)
            out_e.backward(gout)
            eager.append((out_e.detach(), f.grad))
        gs = GraphedStep(copy.deepcopy(mod), b["xyz"], b["mask"], feats, gout)
        gs.load(b["xyz"], b["mask"], feats)
        gs.replay()
        torch.cuda.synchronize()
        assert gs.out.dtype == dt and gs.features.grad.dtype == dt
        assert torch.equal(gs.out, eager[0][0])
        # the backward's lists are ordered by atomics (eager and replay build their own)
        assert_within_ulp(gs.features.grad, eager[0][1], dt, eager[1][1])
    finally:
        pt_utils.cache_enabled = was
