"""CPU tests (-m "not gpu") against what the UNMODIFIED reference networks (`models/`) computed on seeded clouds,
recorded in tests/golden/ref_model_*.pt by oracle/make_ref_vectors.py:
  * closerlook3d_b200/backbone.py has exactly the reference networks' state-dict keys and shapes (checkpoints load);
  * oracle/model_oracle.py reproduces the reference networks' forward and backward on CPU (it is the travelling
    whole-model checker of the GPU tests, so it is pinned here against the real thing)."""
import os

import pytest
import torch

from closerlook3d_b200 import synth
from closerlook3d_b200.config import AttrDict

MODEL_CASES = [
    ("classification", "pospool", dict(pospool=dict(position_embedding="xyz", reduction="avg"))),
    ("scene_segmentation", "adaptive_weight", dict(adaptive_weight=dict(weight_type="dp", num_mlps=1, reduction="avg"))),
    ("scene_segmentation", "pointwisemlp", dict(pointwisemlp=dict(feature_type="dp_fi_df", num_mlps=1, reduction="max"))),
]


def model_case_id(task, la):
    return f"{task}_{la}"


def ref_cfg(cfg, task):
    """the reference's default config with the small test network's settings"""
    if task == "classification":
        cfg.head, cfg.num_classes, cfg.input_features_dim = "resnet_cls", 7, 3
    else:
        cfg.head, cfg.num_classes, cfg.input_features_dim = "resnet_scene_seg", 5, 4
    cfg.backbone, cfg.width, cfg.depth, cfg.bottleneck_ratio = "resnet", 12, 2, 2
    cfg.radius, cfg.sampleDl = 0.12, 0.06
    cfg.nsamples, cfg.npoints = [8, 9, 10, 9, 8], [96, 40, 16, 6]
    return cfg


def inputs(cin):
    d = synth.make_cloud_batch(3, 256, cin, 12)
    return d["xyz"], d["mask"], d["features"]


def _attr(d):
    return AttrDict({k: _attr(v) if isinstance(v, dict) else v for k, v in d.items()})


@pytest.mark.parametrize("task,la,over", MODEL_CASES)
def test_model_oracle_and_backbone_keys_match_reference(oracle_ext, task, la, over):
    from oracle import model_oracle
    from oracle.make_ref_vectors import unpack
    ref = torch.load(os.path.join(os.path.dirname(__file__), "golden", f"ref_model_{model_case_id(task, la)}.pt"),
                     weights_only=False)
    cfg = _attr(ref["cfg"])
    sd = unpack(ref["state_dict"])

    # ---- (1) this package's networks carry the same keys and shapes, and load the reference checkpoint
    from closerlook3d_b200 import backbone as bb
    mine = (bb.ClassificationModel if task == "classification" else bb.SceneSegmentationModel)(cfg)
    msd = mine.state_dict()
    assert set(msd.keys()) == set(sd.keys())
    assert all(tuple(msd[k].shape) == tuple(sd[k].shape) for k in sd)
    assert list(msd.keys()) == list(sd.keys())
    mine.load_state_dict(sd, strict=True)

    # ---- (2) the oracle restatement == the reference model, forward and backward, on CPU
    xyz, mask, feats = inputs(cfg.input_features_dim)
    out_ref = ref["out"]
    orc = model_oracle.OracleModel(oracle_ext, cfg, sd, task)
    f_o = feats.clone().requires_grad_(True)
    out_o = orc(xyz, mask, f_o)
    assert orc.queries == 14                                   # 10 LocalAggregation + 4 MaskedMaxPool
    assert out_o.shape == out_ref.shape
    assert float((out_o - out_ref).abs().max()) <= 1e-6 * max(1.0, float(out_ref.abs().max()))
    g = torch.randn(out_ref.shape, generator=torch.Generator().manual_seed(1))
    (out_o * g).sum().backward()
    g_ref = ref["grad_features"]
    assert float((f_o.grad - g_ref).abs().max()) <= 1e-5 * max(1.0, float(g_ref.abs().max()))
    og = orc.grads()
    index = unpack(ref["grad_index"])
    for name, pg in unpack(ref["grad_params"]).items():   # a fixed sample of each parameter's gradient
        idx = index[name]
        assert name in og, name
        assert float((og[name].reshape(-1)[idx] - pg).abs().max()) <= 1e-5 * max(1.0, float(pg.abs().max())), name
    sd_after = unpack(ref["running"])
    for k, v in orc.st.items():
        if k.endswith(("running_mean", "running_var")):
            assert float((v - sd_after[k]).abs().max()) <= 1e-6 * max(1.0, float(sd_after[k].abs().max())), k
