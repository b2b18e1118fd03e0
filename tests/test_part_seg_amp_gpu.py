"""GPU tests of the fused multi-shape part-segmentation head on bf16 and fp16 input (csrc/multihead.cu,
closerlook3d_b200/partseg.py).

The rule (include/cl3d.h, CL3D_DTYPE_*): x, the logits, d/dlogits and d/dx take the 16-bit type; parameters, BatchNorm
statistics, saved state and every accumulator stay fp32.  So the 16-bit head on x16 is the fp32 head on x16.float()
with d/dlogits widened, rounded once: logits and d/dx equal bit for bit after the rounding, parameter gradients and
running statistics identical.  The helpers and shapes are those of test_part_seg_gpu.py."""
import copy
import importlib.util
import os

import numpy as np
import pytest
import torch

from closerlook3d_b200 import synth

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]
_HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    spec = importlib.util.spec_from_file_location(f"_psamp_{name}", os.path.join(_HERE, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


ps = _load("test_part_seg_gpu")

# (id, C, num_parts, B, N, common offset of x): the fp32 head cases, plus one point in one cloud.  N = 777 is odd: every
# 16-bit row but the first starts only 2-byte aligned.
CASES = ps.HEAD_CASES + [("b1-n1", 24, [3, 5], 1, 1, 0.0)]


def _heads(C, num_parts, B, N, offset, training, cuda, dt):
    heads = ps.make_heads(C, num_parts, 1, cuda).train(training)
    x16 = ps.make_x(B, C, N, offset, 2, cuda).to(dt)
    if not training:   # running statistics that match the input's scale
        with torch.no_grad():
            for h in heads:
                y = torch.nn.functional.conv1d(x16.double(), h[0].weight.double())
                h[1].running_mean.copy_(y.mean((0, 2)).float() + 0.05)
                h[1].running_var.copy_(y.var((0, 2), unbiased=False).float() * 1.1 + 1e-3)
    return heads, x16


def _used(num_parts):
    return set(range(0, len(num_parts), 2)) if len(num_parts) > 1 else {0}


class _CountApply:
    """counts the calls of partseg._MultiShapeHeads.apply (the fused path)"""

    def __enter__(self):
        from closerlook3d_b200 import partseg
        self.cls, self.calls = partseg._MultiShapeHeads, 0
        self.own = self.cls.__dict__.get("apply")       # None: inherited from torch.autograd.Function
        orig = self.cls.apply

        def apply(*a):
            self.calls += 1
            return orig(*a)
        self.cls.apply = apply
        return self

    def __exit__(self, *exc):
        if self.own is None:
            del self.cls.apply
        else:
            self.cls.apply = self.own


def _arm(heads, x, gs):
    """forward + backward of the used heads -> (logits, d/dx, parameter gradients)"""
    from closerlook3d_b200.partseg import multi_shape_heads_forward
    xf = x.clone().requires_grad_(True)
    with _CountApply() as n:
        out = multi_shape_heads_forward(heads, xf)
    assert n.calls == 1
    used = [s for s, g in enumerate(gs) if g is not None]
    torch.autograd.backward([out[s] for s in used], [gs[s] for s in used])
    return [o.detach() for o in out], xf.grad, [p.grad for p in heads.parameters()]


def _two_arms(heads, x16, gs16):
    """the 16-bit head on x16 and the fp32 head on x16.float() with widened d/dlogits, from the same state"""
    h16, h32 = copy.deepcopy(heads), copy.deepcopy(heads)
    a = _arm(h16, x16, gs16)
    b = _arm(h32, x16.float(), [None if g is None else g.float() for g in gs16])
    return (h16, a), (h32, b)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_16bit_head_is_the_fp32_head_on_widened_input_rounded_once(cuda, case, training, dt):
    from closerlook3d_b200.partseg import fused_eligible
    _, C, num_parts, B, N, offset = case
    heads, x16 = _heads(C, num_parts, B, N, offset, training, cuda, dt)
    assert fused_eligible(heads, x16)
    gen = torch.Generator(device=cuda).manual_seed(5)
    used = _used(num_parts)
    gs16 = [torch.randn(B, n, N, device=cuda, generator=gen).to(dt) if s in used else None
            for s, n in enumerate(num_parts)]
    (h16, (out16, dx16, pg16)), (h32, (out32, dx32, pg32)) = _two_arms(heads, x16, gs16)
    for s in range(len(num_parts)):
        assert out16[s].dtype == dt and out16[s].shape == (B, num_parts[s], N)
        assert torch.equal(out16[s], out32[s].to(dt)), s
    assert dx16.dtype == dt and torch.equal(dx16, dx32.to(dt))
    for (n, p), a, b in zip(h16.named_parameters(), pg16, pg32):
        assert p.dtype == torch.float32 and a.dtype == torch.float32, n
        assert torch.equal(a, b), n
        if int(n.split(".")[0]) not in used:
            assert float(a.abs().max()) == 0.0, n
    for (n, a), b in zip(h16.state_dict().items(), h32.state_dict().values()):
        assert a.dtype == b.dtype and torch.equal(a, b), n
    for h in h16:
        assert int(h[1].num_batches_tracked) == (1 if training else 0)


def _ulp(x, dt):
    """one unit in the last place of dt at the magnitude of x (fp32)"""
    p, emin = (7, -126) if dt == torch.bfloat16 else (10, -14)
    _, e = torch.frexp(x.float())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float32), (e - 1).clamp(min=emin) - p)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("case", ps.HEAD_CASES, ids=[c[0] for c in ps.HEAD_CASES])
def test_16bit_head_matches_float64(cuda, case, training, dt):
    """against the reference head in float64 on x16.double(): each logit within half a 16-bit ulp (at the larger
    magnitude of the two, so a value rounded across a power of two is covered) plus 1e-5 of the head's max, the fp32
    head's bar; d/dx the same against the float64 gradient.  Points where some channel's float64 pre-ReLU value lies
    within 1e-5 of the scale of zero could take either side of the ReLU: they are left out of the logits comparison and
    get no upstream gradient (ps.grads_for)."""
    from closerlook3d_b200.partseg import multi_shape_heads_forward
    _, C, num_parts, B, N, offset = case
    heads, x16 = _heads(C, num_parts, B, N, offset, training, cuda, dt)
    x64, hd, out64, pre = ps.f64_heads(heads, x16, training)
    used = _used(num_parts)
    gs = ps.grads_for(out64, pre, used, 5)
    gs16 = [None if g is None else g.to(dt) for g in gs]
    xf = x16.clone().requires_grad_(True)
    out = multi_shape_heads_forward(heads, xf)
    worst = 0.0
    for s in range(len(num_parts)):
        o, r = out[s].detach(), out64[s].detach()
        band = 1e-5 * float(pre[s].abs().max())
        keep = ~(pre[s].abs() <= band).any(1)[:, None, :].expand_as(o)
        d = (o.double() - r).abs()
        bar = 0.5 * torch.maximum(_ulp(o, dt), _ulp(r, dt)).double() + 1e-5 * float(r.abs().max())
        assert bool((d <= bar)[keep].all()), (s, float((d - bar)[keep].max()))
        worst = max(worst, float((d / bar)[keep].max()) if bool(keep.any()) else 0.0)
    torch.autograd.backward([out[s] for s in used], [gs16[s] for s in used])
    torch.autograd.backward([out64[s] for s in used], [gs16[s].double() for s in used])
    g, g64 = xf.grad, x64.grad
    bar = 0.5 * torch.maximum(_ulp(g, dt), _ulp(g64, dt)).double() + 1e-5 * float(g64.abs().max())
    assert g.dtype == dt and bool(((g.double() - g64).abs() <= bar).all())
    print("MHEAD16", case[0], dt, "train" if training else "eval", f"logits err/bar {worst:.2f}")


def test_fp16_overflow_is_inf_exactly_where_the_cast_overflows(cuda):
    """Head 0's output weights x1e4 push its logits past 65504; every head's x10 and d/dlogits of several thousand push
    d/dx past it.  The fp16 head must give inf exactly where .to(float16) of the fp32 head's result does."""
    dt, C, num_parts, B, N = torch.float16, 72, ps.SHAPENETPART, 2, 1000
    heads = ps.make_heads(C, num_parts, 11, cuda)
    with torch.no_grad():
        for h in heads:
            h[3].weight.mul_(10.0)
        heads[0][3].weight.mul_(1e4)
    x16 = ps.make_x(B, C, N, 0.0, 12, cuda).to(dt)
    gen = torch.Generator(device=cuda).manual_seed(13)
    gs16 = [(6000.0 * torch.randn(B, n, N, device=cuda, generator=gen)).to(dt) if s % 2 else None
            for s, n in enumerate(num_parts)]
    (_, (out16, dx16, pg16)), (_, (out32, dx32, pg32)) = _two_arms(heads, x16, gs16)
    ref = out32[0].to(dt)
    assert bool(torch.isinf(ref).any()) and bool(torch.isfinite(ref).any())
    assert all(torch.equal(a, b.to(dt)) for a, b in zip(out16, out32))
    ref = dx32.to(dt)
    assert bool(torch.isinf(ref).any()) and bool(torch.isfinite(ref).any())
    assert torch.equal(torch.isinf(dx16), torch.isinf(ref)) and torch.equal(dx16, ref)
    assert all(torch.equal(a, b) for a, b in zip(pg16, pg32))


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_16bit_head_repeats_bit_for_bit(cuda, dt):
    C, num_parts, B, N = 72, ps.SHAPENETPART, 4, 2047
    heads = ps.make_heads(C, num_parts, 3, cuda)
    x16 = ps.make_x(B, C, N, 0.0, 4, cuda).to(dt)
    gs16 = [torch.randn(B, n, N, device=cuda).to(dt) if s % 3 else None for s, n in enumerate(num_parts)]
    h1, h2 = copy.deepcopy(heads), copy.deepcopy(heads)
    o1, g1 = ps._run(h1, x16, gs16)
    o2, g2 = ps._run(h2, x16, gs16)
    assert o1[0].dtype == dt and g1[0].dtype == dt
    assert all(torch.equal(a, b) for a, b in zip(o1, o2))
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    assert all(torch.equal(a, b) for a, b in zip(h1.state_dict().values(), h2.state_dict().values()))


def test_bf16_head_cuda_graph_replay_matches_eager(cuda):
    dt, C, num_parts, B, N = torch.bfloat16, 72, ps.PARTNET[:6], 2, 1500
    heads = ps.make_heads(C, num_parts, 6, cuda)
    state0 = copy.deepcopy(heads.state_dict())
    xs = torch.zeros(B, C, N, device=cuda, dtype=dt)
    gs = [torch.randn(B, n, N, device=cuda).to(dt) if s != 2 else None for s, n in enumerate(num_parts)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            xs.copy_(ps.make_x(B, C, N, 0.0, 0, cuda))
            ps._run(heads, xs, gs)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_g, grads_g = ps._run(heads, xs, gs)
    x_new = ps.make_x(B, C, N, 1.0, 77, cuda).to(dt)
    heads.load_state_dict(state0)
    xs.copy_(x_new)
    graph.replay()
    torch.cuda.synchronize()
    after_graph = copy.deepcopy(heads.state_dict())
    eager = copy.deepcopy(heads)
    eager.load_state_dict(state0)
    out_e, grads_e = ps._run(eager, x_new, gs)
    assert out_g[0].dtype == dt and grads_g[0].dtype == dt
    assert all(torch.equal(a, b) for a, b in zip(out_g, out_e))
    assert all(torch.equal(a, b) for a, b in zip(grads_g, grads_e))
    for k, v in eager.state_dict().items():
        assert torch.equal(v, after_graph[k]), k


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_eligibility_needs_fp32_parameters(cuda, dt):
    """16-bit x with fp32 parameters takes the fused head; a head converted to bf16 wholesale keeps the reference's
    composition, whose result multi_shape_heads_forward returns"""
    from closerlook3d_b200.partseg import fused_eligible, multi_shape_heads_forward
    C, num_parts, B, N = 36, [4, 7, 2], 2, 500
    heads = ps.make_heads(C, num_parts, 21, cuda).eval()
    x16 = ps.make_x(B, C, N, 0.0, 22, cuda).to(dt)
    assert fused_eligible(heads, x16)
    low = copy.deepcopy(heads).to(torch.bfloat16)
    xb = x16.to(torch.bfloat16)
    assert not fused_eligible(low, xb)
    ref = [h(xb) for h in copy.deepcopy(low)]
    with _CountApply() as n:
        out = multi_shape_heads_forward(low, xb)
    assert n.calls == 0
    assert all(torch.equal(a, b) for a, b in zip(out, ref))
    one = copy.deepcopy(heads)          # a single 16-bit parameter is enough to decline
    one[1][3].bias.data = one[1][3].bias.data.to(dt)
    assert not fused_eligible(one, x16)


def test_whole_network_under_bf16_autocast_takes_the_fused_head(cuda):
    """A small ShapeNetPart network under bf16 autocast runs the fused head on the decoder's bf16 output.  Its logits
    and loss equal, bit for bit, those of the same network whose head input is widened to fp32 and whose logits are
    cast back to bf16."""
    from closerlook3d_b200 import backbone as bb, partseg, pt_utils
    rp = _load("test_reduced_precision_gpu")
    dt = torch.bfloat16
    cfg = rp._net_cfg("multi_part_segmentation", "pseudo_grid", dict())
    torch.manual_seed(3)
    np.random.seed(3)
    model, criterion = bb.build_multi_part_segmentation(cfg)
    model.init_weights()
    B, N = 2, 3000
    d = synth.make_cloud_batch(B, N, cfg.input_features_dim, 21)
    xyz, mask, feats = d["xyz"].to(cuda), d["mask"].to(cuda), d["features"].to(cuda)
    lab = synth.make_part_labels(B, N, cfg.num_parts, 4)
    pl, sl = lab["points_labels"].to(cuda), lab["shape_labels"].to(cuda)
    sd = copy.deepcopy(model.state_dict())
    fwd = partseg.multi_shape_heads_forward
    seen = []

    def widened(heads, x):
        seen.append(x.dtype)
        return [o.to(x.dtype) for o in fwd(heads, x.float())]

    det, overlap = torch.backends.cudnn.deterministic, pt_utils.overlap_enabled
    torch.backends.cudnn.deterministic = True
    pt_utils.overlap_enabled = False
    runs = {}
    try:
        for arm in ("warm", "native", "widened"):
            m = bb.build_multi_part_segmentation(cfg)[0]
            m.load_state_dict(sd)
            m = m.to(cuda).train()
            pt_utils.clear_neighbor_cache()
            import closerlook3d_b200.backbone as bbm
            bbm.multi_shape_heads_forward = widened if arm == "widened" else fwd
            try:
                with _CountApply() as n, torch.autocast("cuda", dtype=dt):
                    pred = m(xyz, mask, feats)
                    loss = criterion(pred, pl, sl)
            finally:
                bbm.multi_shape_heads_forward = fwd
            assert n.calls == 1
            assert all(p.dtype == dt for p in pred)
            runs[arm] = (torch.cat([p.detach().float().reshape(-1) for p in pred]), float(loss))
    finally:
        torch.backends.cudnn.deterministic = det
        pt_utils.overlap_enabled = overlap
    assert seen == [dt]
    (lo_n, loss_n), (lo_w, loss_w) = runs["native"], runs["widened"]
    assert bool(torch.isfinite(lo_n).all()) and np.isfinite(loss_n)
    assert torch.equal(lo_n, lo_w) and loss_n == loss_w
