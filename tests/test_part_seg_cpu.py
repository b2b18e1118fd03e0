"""CPU tests (-m "not gpu") of the multi-part segmentation networks against what the UNMODIFIED reference network and
criterion (models/build.py:build_multi_part_segmentation, losses/multi_shape_cross_entropy.py) computed on seeded
clouds, recorded in tests/golden/ref_model_multi_part_segmentation_*.pt by oracle/make_part_seg_vectors.py:
  * closerlook3d_b200/backbone.py's MultiPartSegmentationModel has exactly the reference's state-dict keys, order and
    shapes (reference checkpoints load with strict=True);
  * oracle/part_seg_oracle.py reproduces the reference network and criterion forward and backward (it is the whole-model
    checker of tests/test_part_seg_gpu.py);
  * backbone.multi_shape_cross_entropy equals the reference criterion, value and gradient;
  * model_config("multi_part_segmentation") carries the shipped yaml settings, and shim.install() gives the
    reference's own builder this package's head (both need a reference checkout)."""
import os
import subprocess
import sys

import pytest
import torch

from closerlook3d_b200 import synth
from closerlook3d_b200.config import AttrDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PART_CASES = [
    ("pseudo_grid", dict()),
    ("pospool", dict(pospool=dict(position_embedding="xyz", reduction="avg"))),
]
PART_NUM_PARTS = [3, 1, 5, 2]   # uneven, one shape with a single part
PART_SEED = 31


def part_ref_cfg(cfg):
    """the reference's default config with the small test network's settings"""
    cfg.head, cfg.num_classes, cfg.num_parts, cfg.input_features_dim = "resnet_part_seg", 4, list(PART_NUM_PARTS), 3
    cfg.backbone, cfg.width, cfg.depth, cfg.bottleneck_ratio = "resnet", 12, 2, 2
    cfg.radius, cfg.sampleDl = 0.12, 0.06
    cfg.nsamples, cfg.npoints = [8, 9, 10, 9, 8], [96, 40, 16, 6]
    return cfg


def part_inputs(cfg):
    d = synth.make_cloud_batch(3, 256, cfg.input_features_dim, 12)
    return d["xyz"], d["mask"], d["features"], synth.make_part_labels(3, 256, cfg.num_parts, PART_SEED)


def _attr(d):
    return AttrDict({k: _attr(v) if isinstance(v, dict) else v for k, v in d.items()})


def _load(la):
    return torch.load(os.path.join(ROOT, "tests", "golden", f"ref_model_multi_part_segmentation_{la}.pt"),
                      weights_only=False)


@pytest.mark.parametrize("la,over", PART_CASES, ids=[c[0] for c in PART_CASES])
def test_part_seg_keys_and_oracle_match_reference(oracle_ext, la, over):
    from oracle import part_seg_oracle
    from oracle.make_ref_vectors import unpack
    ref = _load(la)
    cfg = _attr(ref["cfg"])
    sd = unpack(ref["state_dict"])

    # ---- (1) this package's network carries the same keys, order and shapes, and loads the reference checkpoint
    from closerlook3d_b200 import backbone as bb
    mine = bb.MultiPartSegmentationModel(cfg)
    msd = mine.state_dict()
    assert list(msd.keys()) == list(sd.keys())
    assert all(tuple(msd[k].shape) == tuple(sd[k].shape) for k in sd)
    mine.load_state_dict(sd, strict=True)
    assert [h[3].out_channels for h in mine.segmentation_head.multi_shape_heads] == PART_NUM_PARTS

    # ---- (2) the oracle restatement == the reference network and criterion, forward and backward, on CPU
    xyz, mask, feats, labels = part_inputs(cfg)
    orc = part_seg_oracle.OracleModel(oracle_ext, cfg, sd, "multi_part_segmentation")
    f_o = feats.clone().requires_grad_(True)
    out_o = orc(xyz, mask, f_o)
    assert orc.queries == 14
    out_ref = unpack(ref["out"])
    assert len(out_o) == len(out_ref) == len(PART_NUM_PARTS)
    for s, o in enumerate(out_o):
        r = out_ref[str(s)]
        assert o.shape == r.shape == (3, PART_NUM_PARTS[s], 256)
        assert float((o - r).abs().max()) <= 1e-6 * max(1.0, float(r.abs().max())), s
    loss = part_seg_oracle.multi_shape_cross_entropy(out_o, labels["points_labels"], labels["shape_labels"])
    assert abs(float(loss) - float(ref["loss"])) <= 1e-6 * abs(float(ref["loss"]))
    loss.backward()
    g_ref = ref["grad_features"]
    assert float((f_o.grad - g_ref).abs().max()) <= 1e-5 * max(1.0, float(g_ref.abs().max()))
    og = orc.grads()
    index = unpack(ref["grad_index"])
    for name, pg in unpack(ref["grad_params"]).items():
        assert name in og, name
        assert float((og[name].reshape(-1)[index[name]] - pg).abs().max()) <= 1e-5 * max(1.0, float(pg.abs().max())), name
    sd_after = unpack(ref["running"])
    for k, v in orc.st.items():
        if k.endswith(("running_mean", "running_var")):
            assert float((v - sd_after[k]).abs().max()) <= 1e-6 * max(1.0, float(sd_after[k].abs().max())), k
    # a shape that no sample selects still gets its (zero) gradient, as in the reference
    unused = set(range(len(PART_NUM_PARTS))) - set(labels["shape_labels"].tolist())
    assert unused
    for s in unused:
        assert float(og[f"segmentation_head.multi_shape_heads.{s}.3.weight"].abs().max()) == 0.0


def test_multi_shape_cross_entropy_matches_reference_criterion():
    from closerlook3d_b200.backbone import multi_shape_cross_entropy
    from oracle.part_seg_oracle import multi_shape_cross_entropy as ref_ce
    num_parts = [4, 1, 7, 3, 2]
    B, N = 5, 33
    lab = synth.make_part_labels(B, N, num_parts, 3)
    lab["shape_labels"][:] = torch.tensor([0, 2, 2, 1, 0])   # shapes 3 and 4 are selected by no sample
    for s in range(B):
        lab["points_labels"][s] = lab["points_labels"][s] % num_parts[int(lab["shape_labels"][s])]
    g = torch.Generator().manual_seed(0)
    base = [torch.randn(B, n, N, generator=g, dtype=torch.float64) * 3 for n in num_parts]
    a = [t.clone().requires_grad_(True) for t in base]
    b = [t.clone().requires_grad_(True) for t in base]
    la = multi_shape_cross_entropy(a, lab["points_labels"], lab["shape_labels"])
    lb = ref_ce(b, lab["points_labels"], lab["shape_labels"])
    assert abs(float(la) - float(lb)) <= 1e-12 * abs(float(lb))
    la.backward()
    lb.backward()
    for s in range(len(num_parts)):
        assert a[s].grad is not None and b[s].grad is not None
        assert torch.allclose(a[s].grad, b[s].grad, rtol=0, atol=1e-14), s
    assert float(a[3].grad.abs().max()) == 0.0 and float(a[4].grad.abs().max()) == 0.0


def test_synth_part_labels_respect_num_parts():
    num_parts = [15, 9, 1, 51]
    lab = synth.make_part_labels(6, 500, num_parts, 5)
    assert lab["shape_labels"].shape == (6,) and lab["points_labels"].shape == (6, 500)
    for b in range(6):
        n = num_parts[int(lab["shape_labels"][b])]
        assert int(lab["points_labels"][b].min()) >= 0 and int(lab["points_labels"][b].max()) < n
    again = synth.make_part_labels(6, 500, num_parts, 5)
    assert torch.equal(lab["points_labels"], again["points_labels"])


def _reference_root():
    from oracle.ref_loader import REF_ROOT
    if not os.path.isdir(os.path.join(REF_ROOT, "models")):
        pytest.skip(f"no reference checkout at {REF_ROOT} (set CL3D_REFERENCE)")
    return REF_ROOT


@pytest.mark.parametrize("dataset", ["partnet", "shapenetpart"])
def test_model_config_matches_shipped_yaml(dataset):
    import yaml
    from closerlook3d_b200.backbone import model_config
    root = _reference_root()
    files = sorted(os.listdir(os.path.join(root, "cfgs", dataset)))
    assert len(files) == 5
    for f in files:
        with open(os.path.join(root, "cfgs", dataset, f)) as fh:
            y = yaml.safe_load(fh)
        la = y["local_aggregation_type"]
        c = model_config("multi_part_segmentation", la, dataset=None if dataset == "partnet" else dataset)
        for k in ("datasets", "num_classes", "num_parts", "input_features_dim", "batch_size", "num_points", "backbone",
                  "head", "radius", "sampleDl", "nsamples", "npoints", "width", "depth", "bottleneck_ratio",
                  "bn_momentum"):
            if k in y:
                assert c[k] == y[k], (f, k, c[k], y[k])
        assert len(c.num_parts) == c.num_classes
        if "bn_momentum" not in y:
            assert c.bn_momentum == 0.1      # the reference's default (utils/config.py)
        if "num_points" not in y:
            assert c.num_points == 10000     # PartNet clouds


def test_shim_gives_reference_builder_the_fused_head():
    root = _reference_root()
    code = r'''
import sys
sys.path.insert(0, %r)
from closerlook3d_b200 import shim
shim.install(%r)
import models.build as mb, models.heads as mh, models.heads.segmentation_head as msh
from closerlook3d_b200.backbone import MultiPartSegHeadResNet
assert mb.MultiPartSegHeadResNet is MultiPartSegHeadResNet
assert mh.MultiPartSegHeadResNet is MultiPartSegHeadResNet and msh.MultiPartSegHeadResNet is MultiPartSegHeadResNet
assert mb.SceneSegHeadResNet is msh.SceneSegHeadResNet and mb.SceneSegHeadResNet.__module__ == "models.heads.segmentation_head"
cfg = shim.reference_config(%r + "/cfgs/partnet/pospool_xyz_avg.yaml")
cfg.width = 12
model, criterion = mb.build_multi_part_segmentation(cfg)
assert type(model.segmentation_head) is MultiPartSegHeadResNet
assert len(model.segmentation_head.multi_shape_heads) == 17
''' % (ROOT, root, root)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
