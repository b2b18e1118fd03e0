"""Whole networks on the GPU (SURVEY.md section 8 row (f)4): this package's backbone + heads (closerlook3d_b200/backbone.py,
fused neighbourhood operators) against the reference networks restated in oracle/model_oracle.py on top of the
reference's OWN CUDA extension (oracle/_ref), same state dict, same inputs, forward and backward, TF32 off.
The restatement itself is pinned against the unmodified reference models in tests/test_model_cpu.py.

Tolerance: 10 aggregation layers + 4 pools + 30 training-mode BatchNorms deep (the last stage normalises over 64
samples), fp32 both sides, with ReLU / max discontinuities on the way: the per-stage features are compared so that the
error can be seen to START at rounding level (stage 1: ~1e-6) and grow with depth, instead of one loose end-to-end
bound; the subsampled coordinates and masks of every stage must be bit-identical."""
import copy

import numpy as np
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


def _cfg(task, la, over, width=24):
    from closerlook3d_b200.backbone import model_config
    c = model_config(task, la, **over)
    c.width = width
    c.radius, c.sampleDl = 0.06, 0.03
    c.npoints = [1024, 320, 96, 32]
    c.nsamples = [16, 18, 20, 18, 16]
    c.num_classes = 9
    return c


CASES = [
    ("classification", "pointwisemlp", dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))),
    ("scene_segmentation", "pseudo_grid", dict()),
    ("scene_segmentation", "pospool", dict(pospool=dict(position_embedding="sin_cos", reduction="avg"))),
    ("classification", "adaptive_weight", dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, shared_channels=1,
                                                                   reduction="avg"))),
]


@pytest.mark.parametrize("task,la,over", CASES, ids=[f"{c[0][:3]}-{c[1]}" for c in CASES])
def test_whole_model_matches_reference_gpu_path(cuda, ref_ext, task, la, over):
    from closerlook3d_b200 import backbone as bb, pt_utils
    from oracle import model_oracle
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = _cfg(task, la, over)
    torch.manual_seed(3)
    np.random.seed(3)
    build = bb.build_classification if task == "classification" else bb.build_scene_segmentation
    model, criterion = build(cfg)
    model.init_weights()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0          # the restatement has no dropout; everything else runs in training mode
    sd = copy.deepcopy(model.state_dict())
    B, N = 2, 3000
    d = synth.make_cloud_batch(B, N, cfg.input_features_dim, 21)
    xyz, mask, feats = d["xyz"].to(cuda), d["mask"].to(cuda), d["features"].to(cuda)

    orc = model_oracle.OracleModel(ref_ext, cfg, sd, task, device=cuda)
    f_o = feats.clone().requires_grad_(True)
    out_o = orc(xyz, mask, f_o)

    # a checkpoint in the reference's format round-trips through this package's model
    model = build(cfg)[0]
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    model.load_state_dict({k: v.clone() for k, v in sd.items()}, strict=True)
    model = model.to(cuda).train()
    pt_utils.clear_neighbor_cache()
    pt_utils.cache_stats.update(hit=0, miss=0)
    f = feats.clone().requires_grad_(True)
    hook = model.backbone.register_forward_hook(lambda mod, args, res: setattr(model, "backbone_end_points", dict(res)))
    out = model(xyz, mask, f)
    hook.remove()
    # 14 neighbour queries per backbone forward, 5 of them duplicates served by the cache (SURVEY 3.3)
    assert pt_utils.cache_stats["hit"] == 5 and pt_utils.cache_stats["miss"] == 9, pt_utils.cache_stats
    assert orc.queries == 14

    def rel_l2(x, y):
        return float((x - y).norm()) / max(1e-20, float(y.norm()))

    def rel_max(x, y):
        return float((x - y).abs().max()) / max(1e-20, float(y.abs().max()))

    g = torch.randn(out_o.shape, device=cuda, generator=torch.Generator(device=cuda).manual_seed(1))
    (out_o * g).sum().backward()
    (out * g).sum().backward()
    torch.cuda.synchronize()
    og = orc.grads()
    # parameter gradients against ONE scale (the largest gradient norm of the network): several parameters have an
    # analytically zero gradient (a bias in front of a BatchNorm) and hold pure rounding noise on both sides
    gscale = max(float(v.norm()) for v in og.values())
    m = {"logits_l2": rel_l2(out, out_o), "logits_max": rel_max(out, out_o),
         "dfeat_l2": rel_l2(f.grad, f_o.grad), "dfeat_max": rel_max(f.grad, f_o.grad),
         "dparam_l2": max(float((p.grad - og[n]).norm()) for n, p in model.named_parameters()) / gscale}
    # How sensitive is the REFERENCE network's own gradient to rounding-level noise?  Perturb the input features by
    # 1e-6 (relative) and differentiate the restated reference again: the gradient of a deep ReLU / max network with
    # training-mode BatchNorms moves by far more than 1e-6.  That measured sensitivity is the yardstick for the
    # gradient comparison (the forward values are compared at rounding level directly).
    orc2 = model_oracle.OracleModel(ref_ext, cfg, sd, task, device=cuda)
    gen = torch.Generator(device=cuda).manual_seed(9)
    f_p = (feats * (1.0 + 1e-6 * torch.randn(feats.shape, device=cuda, generator=gen))).requires_grad_(True)
    (orc2(xyz, mask, f_p) * g).sum().backward()
    og2 = orc2.grads()
    m["ref_sens_dfeat_l2"] = rel_l2(f_p.grad, f_o.grad)
    m["ref_sens_dparam_l2"] = max(float((og2[n] - og[n]).norm()) for n in og) / gscale
    msd = model.state_dict()
    m["running_stats"] = max(rel_max(msd[k], v) for k, v in orc.st.items() if k.endswith(("running_mean", "running_var")))
    ep, ep_o = model.backbone_end_points, orc.end_points
    for st in range(1, 6):   # per-stage features: the error grows with depth, it does not start large
        m[f"res{st}_l2"] = rel_l2(ep[f"res{st}_features"], ep_o[f"res{st}_features"])
        assert torch.equal(ep[f"res{st}_xyz"], ep_o[f"res{st}_xyz"]) and torch.equal(ep[f"res{st}_mask"], ep_o[f"res{st}_mask"])
    print("MODEL-PARITY", task, la, {k: f"{v:.2e}" for k, v in m.items()})
    # Deep network, discontinuous operators (ReLU, max over K, max-pool): a value that differs in the 7th digit at
    # layer 1 can flip a ReLU / an arg-max further down, so single elements may move by much more than the rounding
    # level while the bulk agrees to ~1e-6.  Hence norms for the bulk and a loose bound on the worst element.
    # Typical: stage-1 features ~1e-6, logits 1e-4..3e-4, gradients ~1e-2 in the 2-norm.
    assert m["res1_l2"] <= 2e-5 and m["res2_l2"] <= 2e-4, m
    assert m["res5_l2"] <= 2e-4 and m["logits_l2"] <= 2e-3 and m["logits_max"] <= 5e-2, m
    assert m["dfeat_l2"] <= max(1e-4, 10 * m["ref_sens_dfeat_l2"]), m
    assert m["dparam_l2"] <= max(1e-4, 10 * m["ref_sens_dparam_l2"]), m
    assert m["running_stats"] <= 1e-2, m
    # the loss of the task runs on the logits
    if task == "classification":
        loss = criterion(out.detach(), torch.randint(0, cfg.num_classes, (B,), device=cuda))
    else:
        loss = criterion(out.detach(), torch.randint(0, cfg.num_classes, (B, N), device=cuda), mask.float())
    assert torch.isfinite(loss)
