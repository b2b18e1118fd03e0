"""GPU tests of the fused multi-shape part-segmentation head (csrc/multihead.cu, closerlook3d_b200/partseg.py) and of
the whole part-segmentation network.

The head is compared, same state, against the reference head restated in float64 (oracle/part_seg_oracle.py
part_seg_heads), in training and eval mode, with some heads receiving no gradient at all.  Bars per head against its
own scale: logits and d/dx 1e-5 of max, parameter gradients 5e-5 of max, running statistics 1e-5.  A position whose
float64 pre-ReLU value lies within 1e-5 of the scale of zero could take either side of the ReLU in fp32; the upstream
gradient of that head at that point is set to zero on both sides, so such a flip cannot move a gradient."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

from closerlook3d_b200 import synth

pytestmark = pytest.mark.gpu

PARTNET = [15, 9, 39, 11, 7, 4, 5, 10, 12, 10, 41, 6, 7, 24, 51, 11, 6]
SHAPENETPART = [4, 2, 2, 4, 4, 3, 3, 2, 4, 2, 6, 2, 3, 3, 3, 3]

# (id, C, num_parts, B, N, common offset of x)
HEAD_CASES = [
    ("partnet", 72, PARTNET, 8, 10000, 0.0),
    ("shapenetpart", 72, SHAPENETPART, 16, 2048, 0.0),
    ("c12-parts1-64", 12, [1, 64, 5], 3, 1000, 0.0),
    ("c36-single-head-offset", 36, [7], 2, 300, 50.0),
    ("c72-offset", 72, [64, 1, 3, 9], 2, 777, 50.0),
]


def make_heads(C, num_parts, seed, device):
    torch.manual_seed(seed)
    heads = nn.ModuleList()
    for n in num_parts:
        heads.append(nn.Sequential(nn.Conv1d(C, C, 1, bias=False), nn.BatchNorm1d(C), nn.ReLU(inplace=True),
                                   nn.Conv1d(C, n, 1, bias=True)))
    with torch.no_grad():
        for h in heads:
            nn.init.kaiming_normal_(h[0].weight)
            h[1].weight.uniform_(0.5, 1.5)
            h[1].bias.uniform_(-0.3, 0.3)
            h[1].running_var.uniform_(0.5, 2.0)
            h[3].bias.uniform_(-0.1, 0.1)
    return heads.to(device)


def make_x(B, C, N, offset, seed, device):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, C, N, generator=g)) + offset + 0.1 * torch.randn(C, 1, generator=g)
    return x.to(device)


def f64_heads(heads, x, training):
    from oracle import part_seg_oracle
    st = {}
    for s, h in enumerate(heads):
        for k, v in h.state_dict().items():
            t = v.detach().clone()
            if t.is_floating_point() and not k.endswith(("running_mean", "running_var")):
                t.requires_grad_(True)
            st[f"h.{s}.{k}"] = t
    hd = part_seg_oracle.heads_from_state(st, "h", len(heads), dtype=torch.float64)
    x64 = x.detach().double().requires_grad_(True)
    # pre-ReLU values, to find the positions a rounding difference could move across zero
    with torch.no_grad():
        pre = []
        for h in hd:
            y = torch.nn.functional.conv1d(x64, h["w1"])
            if training:
                m, v = y.mean((0, 2), keepdim=True), y.var((0, 2), unbiased=False, keepdim=True)
            else:
                m, v = h["rm"][None, :, None], h["rv"][None, :, None]
            pre.append((y - m) / torch.sqrt(v + 1e-5) * h["gamma"][None, :, None] + h["beta"][None, :, None])
    out = part_seg_oracle.part_seg_heads(x64, hd, training)
    return x64, hd, out, pre


def grads_for(outs, pre, used, seed):
    gen = torch.Generator(device=outs[0].device).manual_seed(seed)
    gs = []
    for s, o in enumerate(outs):
        if s not in used:
            gs.append(None)
            continue
        g = torch.randn(o.shape, device=o.device, generator=gen, dtype=torch.float32)
        band = 1e-5 * float(pre[s].abs().max())
        amb = (pre[s].abs() <= band).any(1)            # (B,N): some channel of this head is ambiguous at the point
        g[amb[:, None, :].expand_as(g)] = 0.0
        gs.append(g)
    return gs


def rel(a, b):
    return float((a.double() - b.double()).abs().max()) / max(1e-30, float(b.abs().max()))


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("case", HEAD_CASES, ids=[c[0] for c in HEAD_CASES])
def test_fused_head_matches_float64(cuda, case, training):
    from closerlook3d_b200.partseg import fused_eligible, multi_shape_heads_forward
    _, C, num_parts, B, N, offset = case
    heads = make_heads(C, num_parts, 1, cuda).train(training)
    x = make_x(B, C, N, offset, 2, cuda)
    if not training:   # running statistics that match the input's scale
        with torch.no_grad():
            for h in heads:
                y = torch.nn.functional.conv1d(x.double(), h[0].weight.double())
                h[1].running_mean.copy_(y.mean((0, 2)).float() + 0.05)
                h[1].running_var.copy_(y.var((0, 2)).float() * 1.1)
    assert fused_eligible(heads, x)
    x64, hd, out64, pre = f64_heads(heads, x, training)
    used = set(range(0, len(num_parts), 2)) if len(num_parts) > 1 else {0}
    xf = x.clone().requires_grad_(True)
    out = multi_shape_heads_forward(heads, xf)
    gs = grads_for(out, pre, used, 5)
    m = {}
    for s in range(len(num_parts)):
        assert out[s].shape == (B, num_parts[s], N)
        m[f"logits{s}"] = rel(out[s], out64[s])
    torch.autograd.backward([out[s] for s in used], [gs[s] for s in used])
    torch.autograd.backward([out64[s] for s in used], [gs[s].double() for s in used])
    m["dx"] = rel(xf.grad, x64.grad)
    for s, (h, h64) in enumerate(zip(heads, hd)):
        pairs = {"dW1": (h[0].weight.grad.squeeze(-1), h64["w1"].grad), "dgamma": (h[1].weight.grad, h64["gamma"].grad),
                 "dbeta": (h[1].bias.grad, h64["beta"].grad), "dW2": (h[3].weight.grad, h64["w2"].grad),
                 "db2": (h[3].bias.grad, h64["b2"].grad)}
        for k, (a, b) in pairs.items():
            if s in used:
                m[f"{k}{s}"] = rel(a.reshape(b.shape), b)
            else:
                assert h64[{"dW1": "w1", "dgamma": "gamma", "dbeta": "beta", "dW2": "w2", "db2": "b2"}[k]].grad is None
                assert float(a.abs().max()) == 0.0, (s, k)
        m[f"rm{s}"] = rel(h[1].running_mean, h64["rm"])
        m[f"rv{s}"] = rel(h[1].running_var, h64["rv"])
        assert int(h[1].num_batches_tracked) == (1 if training else 0)
    worst = {k: max(v for kk, v in m.items() if kk.startswith(k)) for k in
             ("logits", "dx", "dW1", "dgamma", "dbeta", "dW2", "db2", "rm", "rv")}
    print("MHEAD", case[0], "train" if training else "eval", {k: f"{v:.1e}" for k, v in worst.items()})
    assert worst["logits"] <= 1e-5 and worst["dx"] <= 1e-5, worst
    for k in ("dW1", "dgamma", "dbeta", "dW2", "db2"):
        assert worst[k] <= 5e-5, worst
    assert worst["rm"] <= 1e-5 and worst["rv"] <= 1e-5, worst


def _run(heads, x, gs):
    from closerlook3d_b200.partseg import multi_shape_heads_forward
    xf = x.clone().requires_grad_(True)
    out = multi_shape_heads_forward(heads, xf)
    used = [s for s, g in enumerate(gs) if g is not None]
    params = list(heads.parameters())
    grads = torch.autograd.grad([out[s] for s in used], [xf] + params, [gs[s] for s in used])
    return [o.detach().clone() for o in out], [g.clone() for g in grads]


def test_fused_head_is_deterministic_and_momentum_none(cuda):
    C, num_parts, B, N = 72, SHAPENETPART, 4, 2048
    heads = make_heads(C, num_parts, 3, cuda)
    x = make_x(B, C, N, 0.0, 4, cuda)
    gs = [torch.randn(B, n, N, device=cuda) if s % 3 else None for s, n in enumerate(num_parts)]
    h1, h2 = copy.deepcopy(heads), copy.deepcopy(heads)
    o1, g1 = _run(h1, x, gs)
    o2, g2 = _run(h2, x, gs)
    assert all(torch.equal(a, b) for a, b in zip(o1, o2))
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    assert all(torch.equal(a, b) for a, b in zip(h1.state_dict().values(), h2.state_dict().values()))
    # momentum=None: cumulative moving average over num_batches_tracked, as nn.BatchNorm1d
    from oracle import part_seg_oracle
    h3 = copy.deepcopy(heads)
    for h in h3:
        h[1].momentum = None
    st = {f"h.{s}.{k}": v.detach().clone() for s, h in enumerate(h3) for k, v in h.state_dict().items()}
    hd = part_seg_oracle.heads_from_state(st, "h", len(num_parts), dtype=torch.float64)
    for it in range(3):
        xi = make_x(B, C, N, 0.0, 10 + it, cuda)
        _run(h3, xi, gs)
        with torch.no_grad():
            part_seg_oracle.part_seg_heads(xi.double(), hd, True, momentum=None)
    for h, h64 in zip(h3, hd):
        assert int(h[1].num_batches_tracked) == 3
        assert rel(h[1].running_mean, h64["rm"]) <= 1e-5 and rel(h[1].running_var, h64["rv"]) <= 1e-5


def test_fused_head_cuda_graph_replay_matches_eager(cuda):
    C, num_parts, B, N = 72, PARTNET[:6], 2, 1500
    heads = make_heads(C, num_parts, 6, cuda)
    state0 = copy.deepcopy(heads.state_dict())
    xs = torch.zeros(B, C, N, device=cuda)
    gs = [torch.randn(B, n, N, device=cuda) if s != 2 else None for s, n in enumerate(num_parts)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            xs.copy_(make_x(B, C, N, 0.0, 0, cuda))
            _run(heads, xs, gs)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_g, grads_g = _run(heads, xs, gs)
    x_new = make_x(B, C, N, 1.0, 77, cuda)
    heads.load_state_dict(state0)
    xs.copy_(x_new)
    graph.replay()
    torch.cuda.synchronize()
    after_graph = copy.deepcopy(heads.state_dict())
    eager = copy.deepcopy(heads)
    eager.load_state_dict(state0)
    out_e, grads_e = _run(eager, x_new, gs)
    assert all(torch.equal(a, b) for a, b in zip(out_g, out_e))
    assert all(torch.equal(a, b) for a, b in zip(grads_g, grads_e))
    for k, v in eager.state_dict().items():
        assert torch.equal(v, after_graph[k]), k


@pytest.mark.parametrize("C,num_parts", [(130, [3, 5]), (136, [4]), (24, [65, 2])], ids=["c130", "c136", "parts65"])
def test_out_of_limit_inputs_take_the_torch_path(cuda, C, num_parts):
    from closerlook3d_b200.partseg import fused_eligible, multi_shape_heads_forward
    from oracle import part_seg_oracle
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    heads = make_heads(C, num_parts, 8, cuda)
    x = make_x(2, C, 500, 0.0, 9, cuda)
    assert not fused_eligible(heads, x)
    st = {f"h.{s}.{k}": v.detach().clone() for s, h in enumerate(heads) for k, v in h.state_dict().items()}
    hd = part_seg_oracle.heads_from_state(st, "h", len(num_parts), dtype=torch.float64)
    out = multi_shape_heads_forward(heads, x)
    ref = part_seg_oracle.part_seg_heads(x.double(), hd, True)
    for o, r in zip(out, ref):
        assert rel(o, r) <= 1e-5


@pytest.fixture(scope="module")
def ref_ext():
    try:
        from oracle import build_ref
        return build_ref.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"oracle/_ref unavailable: {e}")


NET_CASES = [
    ("partnet", "adaptive_weight", dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1,
                                                             reduction="avg"))),
    ("shapenetpart", "pseudo_grid", dict()),
]


@pytest.mark.parametrize("dataset,la,over", NET_CASES, ids=[f"{c[0]}-{c[1]}" for c in NET_CASES])
def test_whole_part_seg_network_matches_reference_gpu_path(cuda, ref_ext, dataset, la, over):
    """mirrors tests/test_model_gpu.py: this package's network (fused head) against the reference network restated
    over the reference's own CUDA extension, small width, the dataset's num_parts"""
    from closerlook3d_b200 import backbone as bb, pt_utils
    from oracle import part_seg_oracle
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = bb.model_config("multi_part_segmentation", la, dataset=dataset, **over)
    cfg.width = 24
    cfg.radius, cfg.sampleDl = 0.06, 0.03
    cfg.npoints = [1024, 320, 96, 32]
    cfg.nsamples = [16, 18, 20, 18, 16]
    torch.manual_seed(3)
    np.random.seed(3)
    model, criterion = bb.build_multi_part_segmentation(cfg)
    model.init_weights()
    sd = copy.deepcopy(model.state_dict())
    B, N = 2, 3000
    d = synth.make_cloud_batch(B, N, cfg.input_features_dim, 21)
    xyz, mask, feats = d["xyz"].to(cuda), d["mask"].to(cuda), d["features"].to(cuda)
    task = "multi_part_segmentation"
    orc = part_seg_oracle.OracleModel(ref_ext, cfg, sd, task, device=cuda)
    f_o = feats.clone().requires_grad_(True)
    out_o = orc(xyz, mask, f_o)

    model = bb.build_multi_part_segmentation(cfg)[0]
    model.load_state_dict({k: v.clone() for k, v in sd.items()}, strict=True)
    model = model.to(cuda).train()
    pt_utils.clear_neighbor_cache()
    pt_utils.cache_stats.update(hit=0, miss=0)
    f = feats.clone().requires_grad_(True)
    hook = model.backbone.register_forward_hook(lambda mod, args, res: setattr(model, "backbone_end_points", dict(res)))
    out = model(xyz, mask, f)
    hook.remove()
    assert pt_utils.cache_stats["hit"] == 5 and pt_utils.cache_stats["miss"] == 9, pt_utils.cache_stats
    assert orc.queries == 14
    assert len(out) == len(out_o) == cfg.num_classes

    def rel_l2(x, y):
        return float((x - y).norm()) / max(1e-20, float(y.norm()))

    def rel_max(x, y):
        return float((x - y).abs().max()) / max(1e-20, float(y.abs().max()))

    lab = synth.make_part_labels(B, N, cfg.num_parts, 4)
    pl, sl = lab["points_labels"].to(cuda), lab["shape_labels"].to(cuda)
    loss_o = part_seg_oracle.multi_shape_cross_entropy(out_o, pl, sl)
    loss = criterion(out, pl, sl)
    loss_o.backward()
    loss.backward()
    torch.cuda.synchronize()
    og = orc.grads()
    gscale = max(float(v.norm()) for v in og.values())
    m = {"logits_l2": max(rel_l2(a, b) for a, b in zip(out, out_o)),
         "logits_max": max(rel_max(a, b) for a, b in zip(out, out_o)),
         "loss": abs(float(loss) - float(loss_o)) / abs(float(loss_o)),
         "dfeat_l2": rel_l2(f.grad, f_o.grad), "dfeat_max": rel_max(f.grad, f_o.grad),
         "dparam_l2": max(float((p.grad - og[n]).norm()) for n, p in model.named_parameters()) / gscale}
    orc2 = part_seg_oracle.OracleModel(ref_ext, cfg, sd, task, device=cuda)
    gen = torch.Generator(device=cuda).manual_seed(9)
    f_p = (feats * (1.0 + 1e-6 * torch.randn(feats.shape, device=cuda, generator=gen))).requires_grad_(True)
    part_seg_oracle.multi_shape_cross_entropy(orc2(xyz, mask, f_p), pl, sl).backward()
    og2 = orc2.grads()
    m["ref_sens_dfeat_l2"] = rel_l2(f_p.grad, f_o.grad)
    m["ref_sens_dparam_l2"] = max(float((og2[n] - og[n]).norm()) for n in og) / gscale
    msd = model.state_dict()
    m["running_stats"] = max(rel_max(msd[k], v) for k, v in orc.st.items() if k.endswith(("running_mean", "running_var")))
    ep, ep_o = model.backbone_end_points, orc.end_points
    for st in range(1, 6):
        m[f"res{st}_l2"] = rel_l2(ep[f"res{st}_features"], ep_o[f"res{st}_features"])
        assert torch.equal(ep[f"res{st}_xyz"], ep_o[f"res{st}_xyz"]) and torch.equal(ep[f"res{st}_mask"], ep_o[f"res{st}_mask"])
    print("PARTSEG-PARITY", dataset, la, {k: f"{v:.2e}" for k, v in m.items()})
    assert m["res1_l2"] <= 2e-5 and m["res2_l2"] <= 2e-4, m
    assert m["res5_l2"] <= 2e-4 and m["logits_l2"] <= 2e-3 and m["logits_max"] <= 5e-2, m
    assert m["loss"] <= 1e-3, m
    assert m["dfeat_l2"] <= max(1e-4, 10 * m["ref_sens_dfeat_l2"]), m
    assert m["dparam_l2"] <= max(1e-4, 10 * m["ref_sens_dparam_l2"]), m
    assert m["running_stats"] <= 1e-2, m
    for h in model.segmentation_head.multi_shape_heads:
        assert int(h[1].num_batches_tracked) == 1
