"""oracle/part_seg_oracle.py -- torch restatement of the reference's multi-part segmentation network and criterion.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Extends oracle/model_oracle.py (backbone, decoder building blocks)
with the part-segmentation head and loss, for the tests of the fused multi-shape head:

  models/heads/segmentation_head.py:124-149  MultiPartSegHeadResNet.forward (part_seg_heads: any dtype, so the GPU
                                             tests can evaluate it in float64)
  models/build.py:84-86                      MultiPartSegmentationModel.forward
  models/losses/multi_shape_cross_entropy.py:6-23  MultiShapeCrossEntropy
Pinned against the unmodified reference network and criterion on CPU by tests/test_part_seg_cpu.py.
"""
import torch
import torch.nn.functional as F

from . import la_oracle, model_oracle


def heads_from_state(st, prefix, S, dtype=None):
    """the S shape heads of a state dict as dicts {w1, gamma, beta, rm, rv, nbt, w2, b2}; with `dtype` the tensors are
    converted copies (leaves that require grad where the source parameter does), else the state's own tensors"""
    names = dict(w1="0.weight", gamma="1.weight", beta="1.bias", rm="1.running_mean", rv="1.running_var",
                 w2="3.weight", b2="3.bias")
    heads = []
    for s in range(S):
        p = f"{prefix}.{s}."
        h = {}
        for k, n in names.items():
            t = st[p + n]
            if dtype is not None:
                t = t.detach().to(dtype).clone().requires_grad_(t.requires_grad)
            h[k] = t
        nbt = st.get(p + "1.num_batches_tracked")
        h["nbt"] = int(nbt) if nbt is not None else 0
        heads.append(h)
    return heads


def part_seg_heads(x, heads, training, momentum=0.1, eps=1e-5):
    """segmentation_head.py:145-149 with every head nn.Sequential(Conv1d, BatchNorm1d, ReLU, Conv1d+bias) written
    out: a list of S logits (B, num_parts[s], N) in x's dtype.  The running statistics of `heads` are updated in place
    (training); momentum None is nn.BatchNorm1d's cumulative average, 1 / num_batches_tracked."""
    out = []
    for h in heads:
        y = F.conv1d(x, h["w1"])
        m = momentum
        if training and momentum is None:
            h["nbt"] += 1
            m = 1.0 / h["nbt"]
        y = F.batch_norm(y, h["rm"], h["rv"], h["gamma"], h["beta"], training, 0.0 if m is None else m, eps)
        out.append(F.conv1d(F.relu(y), h["w2"], h["b2"]))
    return out


def multi_shape_cross_entropy(logits_all_shapes, points_labels, shape_labels):
    """losses/multi_shape_cross_entropy.py:11-23, as written there"""
    batch_size = shape_labels.shape[0]
    losses = 0
    for i in range(batch_size):
        sl = int(shape_labels[i])
        loss = F.cross_entropy(logits_all_shapes[sl][i].unsqueeze(0), points_labels[i].unsqueeze(0))
        losses += loss
        for isl in range(len(logits_all_shapes)):
            if isl == sl:
                continue
            losses += 0.0 * logits_all_shapes[isl][i].sum()
    return losses / batch_size


class OracleModel(model_oracle.OracleModel):
    """model_oracle.OracleModel with task "multi_part_segmentation" (state keys 'backbone....',
    'segmentation_head.up_conv*', 'segmentation_head.multi_shape_heads.*'); the other tasks as the base class"""

    def part_seg_head(self, ep):
        """segmentation_head.py:124-149: the scene decoder, then every shape head over every point"""
        f = ep["res5_features"]
        for i in range(4):
            fine, coarse = f"res{4 - i}", f"res{5 - i}"
            f = la_oracle.masked_upsample_nearest(self.ext, ep[fine + "_xyz"], ep[coarse + "_xyz"], ep[fine + "_mask"],
                                                  ep[coarse + "_mask"], f)
            f = self._conv_bn(torch.cat([f, ep[fine + "_features"]], 1), f"segmentation_head.up_conv{i}", relu=True,
                              momentum=0.1)
        self.head_input = f
        heads = heads_from_state(self.st, "segmentation_head.multi_shape_heads", self.cfg.num_classes)
        out = part_seg_heads(f, heads, self.training)
        if self.training:
            for s in range(len(heads)):
                self.st[f"segmentation_head.multi_shape_heads.{s}.1.num_batches_tracked"] += 1
        return out

    def __call__(self, xyz, mask, feats):
        if self.task != "multi_part_segmentation":
            return super().__call__(xyz, mask, feats)
        ep = self.backbone(xyz, mask, feats)
        self.end_points = ep
        return self.part_seg_head(ep)
