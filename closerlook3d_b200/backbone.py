"""Whole networks around the fused local aggregation: the reference's ResNet backbone, classifier and scene-segmentation
head, with the SAME module tree (=> the same state-dict keys: reference checkpoints load unmodified) on top of this
package's operators.

    reference (file:line)                                          here
    models/backbones/resnet.py:22-68    Bottleneck                 Bottleneck
    models/backbones/resnet.py:71-188   ResNet                     ResNet  (stages built in a loop)
    models/heads/classifier.py:6-52     ClassifierResNet           ClassifierResNet
    models/heads/segmentation_head.py:15-94  SceneSegHeadResNet    SceneSegHeadResNet
    models/heads/segmentation_head.py:97-149 MultiPartSegHeadResNet MultiPartSegHeadResNet (heads: partseg.py, fused)
    models/build.py:9-33,36-122         build_* / *Model           build_classification / build_scene_segmentation /
                                                                   build_multi_part_segmentation
    losses/multi_shape_cross_entropy.py MultiShapeCrossEntropy     multi_shape_cross_entropy

The reference's own `models/` also run on this package with zero edits through `shim.install()`; this module exists so
that the whole-model path is available (and testable on the GPU box) without the reference tree.  The 1x1 convolutions
and their BatchNorms are torch library calls exactly as in the reference; every neighbourhood operation (10
LocalAggregation calls, 4 MaskedMaxPool, the decoder's nearest upsampling) is this package's fused kernels, and the
duplicate neighbour queries of a forward pass (5 of 14) hit the neighbour-list cache.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .local_aggregation_operators import LocalAggregation
from .partseg import multi_shape_heads_forward
from .pt_utils import MaskedMaxPool, MaskedUpsample


def _conv_bn(cin, cout, momentum, relu):
    layers = [nn.Conv1d(cin, cout, kernel_size=1, bias=False), nn.BatchNorm1d(cout, momentum=momentum)]
    if relu:
        layers.append(nn.ReLU(inplace=True))
    return nn.Sequential(*layers)


class MultiInputSequential(nn.Sequential):
    """nn.Sequential over (xyz, mask, features) triples (resnet.py:14-19)"""

    def forward(self, *args):
        for m in self._modules.values():
            args = m(*args)
        return args


class Bottleneck(nn.Module):
    """conv1 (1x1 + BN + ReLU) -> LocalAggregation -> conv2 (1x1 + BN) -> + shortcut -> ReLU; a strided block first
    max-pools onto the grid-subsampled points (resnet.py:22-68)."""

    def __init__(self, in_channels, out_channels, bottleneck_ratio, radius, nsample, config, downsample=False,
                 sampleDl=None, npoint=None):
        super().__init__()
        self.in_channels, self.out_channels, self.downsample = in_channels, out_channels, downsample
        mid = out_channels // bottleneck_ratio
        if downsample:
            self.maxpool = MaskedMaxPool(npoint, radius, nsample, sampleDl)
        self.conv1 = _conv_bn(in_channels, mid, config.bn_momentum, relu=True)
        self.local_aggregation = LocalAggregation(mid, mid, radius, nsample, config)
        self.conv2 = _conv_bn(mid, out_channels, config.bn_momentum, relu=False)
        self.relu = nn.ReLU(inplace=True)
        if in_channels != out_channels:
            self.shortcut = _conv_bn(in_channels, out_channels, config.bn_momentum, relu=False)

    def forward(self, xyz, mask, features):
        if self.downsample:
            q_xyz, q_mask, identity = self.maxpool(xyz, mask, features)
        else:
            q_xyz, q_mask, identity = xyz, mask, features
        out = self.conv2(self.local_aggregation(q_xyz, xyz, q_mask, mask, self.conv1(features)))
        if self.in_channels != self.out_channels:
            identity = self.shortcut(identity)
        return q_xyz, q_mask, self.relu(out + identity)


class ResNet(nn.Module):
    """res1: conv1 + la1 + btnk1; res2..res5: one strided bottleneck (grid spacing, radius and width double) followed by
    depth-1 plain ones (resnet.py:71-188).  Returns the dict of per-stage (xyz, mask, features)."""

    def __init__(self, config, input_features_dim, radius, sampleDl, nsamples, npoints, width=144, depth=2,
                 bottleneck_ratio=2):
        super().__init__()
        self.input_features_dim = input_features_dim
        self.conv1 = _conv_bn(input_features_dim, width // 2, config.bn_momentum, relu=True)
        self.la1 = LocalAggregation(width // 2, width // 2, radius, nsamples[0], config)
        self.btnk1 = Bottleneck(width // 2, width, bottleneck_ratio, radius, nsamples[0], config)
        for stage in range(4):      # layer1 .. layer4
            seq = MultiInputSequential()
            sampleDl = sampleDl * 2
            seq.add_module("strided_bottleneck",
                           Bottleneck(width, 2 * width, bottleneck_ratio, radius, nsamples[stage], config, downsample=True,
                                      sampleDl=sampleDl, npoint=npoints[stage]))
            radius, width = radius * 2, width * 2
            for i in range(depth - 1):
                seq.add_module(f"bottlneck{i}",  # (sic) the reference's spelling is part of the checkpoint keys
                               Bottleneck(width, width, bottleneck_ratio, radius, nsamples[stage + 1], config))
            setattr(self, f"layer{stage + 1}", seq)

    def forward(self, xyz, mask, features, end_points=None):
        end_points = end_points if end_points else {}
        features = self.la1(xyz, xyz, mask, mask, self.conv1(features))
        state = self.btnk1(xyz, mask, features)
        for stage in range(5):
            if stage > 0:
                state = getattr(self, f"layer{stage}")(*state)
            for name, t in zip(("xyz", "mask", "features"), state):
                end_points[f"res{stage + 1}_{name}"] = t
        return end_points


class MaskedGlobalAvgPool1d(nn.Module):
    """mean of the features over the valid points of each cloud (classifier.py:6-14)"""

    def forward(self, mask, features):
        return features.sum(-1) / mask.sum(-1)[:, None]


class ClassifierResNet(nn.Module):
    """global average pool of res5 + three (Linear, BN, ReLU, Dropout) blocks + Linear (classifier.py:17-52)"""

    def __init__(self, num_classes, width):
        super().__init__()
        self.num_classes = num_classes
        self.pool = MaskedGlobalAvgPool1d()
        dims = [16 * width, 8 * width, 4 * width, 2 * width]
        layers = []
        for cin, cout in zip(dims[:-1], dims[1:]):
            layers += [nn.Linear(cin, cout), nn.BatchNorm1d(cout), nn.ReLU(inplace=True), nn.Dropout(0.5)]
        layers.append(nn.Linear(dims[-1], num_classes))
        self.classifier = nn.Sequential(*layers)

    def forward(self, end_points):
        return self.classifier(self.pool(end_points["res5_mask"], end_points["res5_features"]))


class SceneSegHeadResNet(nn.Module):
    """decoder: four times (nearest upsampling onto the finer stage, concat with its skip features, 1x1 conv + BN + ReLU),
    then the per-point classifier (segmentation_head.py:15-94)"""

    def __init__(self, num_classes, width, base_radius, nsamples):
        super().__init__()
        self.num_classes, self.base_radius, self.nsamples = num_classes, base_radius, nsamples
        cins = [24 * width, 8 * width, 4 * width, 2 * width]
        couts = [4 * width, 2 * width, width, width // 2]
        for i in range(4):
            setattr(self, f"up{i}", MaskedUpsample(radius=(8 >> i) * base_radius, nsample=nsamples[3 - i], mode="nearest"))
        for i in range(4):
            setattr(self, f"up_conv{i}", _conv_bn(cins[i], couts[i], 0.1, relu=True))
        self.head = nn.Sequential(*list(_conv_bn(width // 2, width // 2, 0.1, relu=True)),
                                  nn.Conv1d(width // 2, num_classes, kernel_size=1, bias=True))

    def forward(self, end_points):
        features = end_points["res5_features"]
        for i in range(4):
            fine, coarse = f"res{4 - i}", f"res{5 - i}"
            features = getattr(self, f"up{i}")(end_points[fine + "_xyz"], end_points[coarse + "_xyz"],
                                               end_points[fine + "_mask"], end_points[coarse + "_mask"], features)
            features = getattr(self, f"up_conv{i}")(torch.cat([features, end_points[fine + "_features"]], 1))
        return self.head(features)


class MultiPartSegHeadResNet(nn.Module):
    """the scene-segmentation decoder followed by one head per shape category, Conv1d(C,C) + BN + ReLU +
    Conv1d(C, num_parts[s]) with C = width/2, all run over every point (segmentation_head.py:97-149).  The heads run
    fused (partseg.py); forward returns the reference's list of S logits tensors (B, num_parts[s], N)."""

    def __init__(self, num_classes, width, base_radius, nsamples, num_parts):
        super().__init__()
        self.num_classes, self.base_radius, self.nsamples, self.num_parts = num_classes, base_radius, nsamples, num_parts
        cins = [24 * width, 8 * width, 4 * width, 2 * width]
        couts = [4 * width, 2 * width, width, width // 2]
        for i in range(4):
            setattr(self, f"up{i}", MaskedUpsample(radius=(8 >> i) * base_radius, nsample=nsamples[3 - i], mode="nearest"))
        for i in range(4):
            setattr(self, f"up_conv{i}", _conv_bn(cins[i], couts[i], 0.1, relu=True))
        self.multi_shape_heads = nn.ModuleList()
        for i in range(num_classes):
            self.multi_shape_heads.append(nn.Sequential(*list(_conv_bn(width // 2, width // 2, 0.1, relu=True)),
                                                        nn.Conv1d(width // 2, num_parts[i], kernel_size=1, bias=True)))

    def forward(self, end_points):
        features = end_points["res5_features"]
        for i in range(4):
            fine, coarse = f"res{4 - i}", f"res{5 - i}"
            features = getattr(self, f"up{i}")(end_points[fine + "_xyz"], end_points[coarse + "_xyz"],
                                               end_points[fine + "_mask"], end_points[coarse + "_mask"], features)
            features = getattr(self, f"up_conv{i}")(torch.cat([features, end_points[fine + "_features"]], 1))
        return multi_shape_heads_forward(self.multi_shape_heads, features)


class _Model(nn.Module):
    def _make_backbone(self, config):
        if config.backbone != "resnet":
            raise NotImplementedError(f"Backbone {config.backbone} not implemented")
        return ResNet(config, config.input_features_dim, config.radius, config.sampleDl, config.nsamples, config.npoints,
                      width=config.width, depth=config.depth, bottleneck_ratio=config.bottleneck_ratio)

    def init_weights(self):
        """kaiming-normal convolutions, zero biases (build.py:59-64)"""
        for m in self.modules():
            if isinstance(m, (nn.Conv1d, nn.Conv2d)):
                nn.init.kaiming_normal_(m.weight)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)


class ClassificationModel(_Model):
    """backbone + `classifier` (build.py:36-64): forward(xyz, mask, features) -> logits (B, num_classes)"""

    def __init__(self, config):
        super().__init__()
        self.backbone = self._make_backbone(config)
        if config.head != "resnet_cls":
            raise NotImplementedError(f"Head {config.head} not implemented in Classification Model")
        self.classifier = ClassifierResNet(config.num_classes, config.width)

    def forward(self, xyz, mask, features):
        return self.classifier(self.backbone(xyz, mask, features))


class SceneSegmentationModel(_Model):
    """backbone + `segmentation_head` (build.py:96-122): forward -> logits (B, num_classes, N)"""

    def __init__(self, config):
        super().__init__()
        self.backbone = self._make_backbone(config)
        if config.head != "resnet_scene_seg":
            raise NotImplementedError(f"Head {config.head} not implemented in Scene Segmentation Model")
        self.segmentation_head = SceneSegHeadResNet(config.num_classes, config.width, config.radius, config.nsamples)

    def forward(self, xyz, mask, features):
        return self.segmentation_head(self.backbone(xyz, mask, features))


class MultiPartSegmentationModel(_Model):
    """backbone + `segmentation_head` (build.py:66-90): forward -> list of S logits (B, num_parts[s], N)"""

    def __init__(self, config):
        super().__init__()
        self.backbone = self._make_backbone(config)
        if config.head != "resnet_part_seg":
            raise NotImplementedError(f"Head {config.head} not implemented in Multi-Part Segmentation Model")
        self.segmentation_head = MultiPartSegHeadResNet(config.num_classes, config.width, config.radius,
                                                        config.nsamples, config.num_parts)

    def forward(self, xyz, mask, features):
        return self.segmentation_head(self.backbone(xyz, mask, features))


def label_smoothing_cross_entropy(pred, target, smoothing_ratio=0.2):
    """the classification criterion (losses/label_smoothing_cross_entropy.py:6-21)"""
    n = pred.size(1)
    soft = torch.full_like(pred, smoothing_ratio / (n - 1)).scatter_(1, target.view(-1, 1), 1.0 - smoothing_ratio)
    return -(soft * F.log_softmax(pred, dim=1)).sum(1).mean()


def masked_cross_entropy(logit, target, mask):
    """the scene-segmentation criterion (losses/masked_cross_entropy.py:6-13)"""
    loss = F.cross_entropy(logit, target, reduction="none") * mask
    return loss.sum() / mask.sum()


def multi_shape_cross_entropy(logits_all_shapes, points_labels, shape_labels):
    """the part-segmentation criterion (losses/multi_shape_cross_entropy.py:6-23): per sample, the mean cross entropy
    of its own shape's logits over all N points (unmasked), plus 0 * the sum of every other shape's logits, over B.
    Written per head with a sample selector instead of a Python loop over samples: same value and gradients, no
    host synchronisation."""
    B = shape_labels.shape[0]
    loss = 0.0
    for s, logits in enumerate(logits_all_shapes):
        sel = shape_labels == s
        target = torch.where(sel[:, None], points_labels, torch.zeros_like(points_labels))
        ce = F.cross_entropy(logits, target, reduction="none").mean(1)
        loss = loss + torch.where(sel, ce, 0.0 * logits.sum((1, 2))).sum()
    return loss / B


def build_classification(config):
    return ClassificationModel(config), label_smoothing_cross_entropy


def build_scene_segmentation(config):
    return SceneSegmentationModel(config), masked_cross_entropy


def build_multi_part_segmentation(config):
    return MultiPartSegmentationModel(config), multi_shape_cross_entropy


# The shipped part-segmentation settings (cfgs/partnet/*.yaml, cfgs/shapenetpart/*.yaml): the same for every family
# except ShapeNetPart's PointWiseMLP batch (12).
PART_DATASETS = {
    "partnet": dict(datasets="partnet", num_classes=17,
                    num_parts=[15, 9, 39, 11, 7, 4, 5, 10, 12, 10, 41, 6, 7, 24, 51, 11, 6], input_features_dim=3,
                    batch_size=8, num_points=10000, radius=0.05, sampleDl=0.02, nsamples=[23, 38, 42, 40, 36],
                    npoints=[5120, 1024, 384, 64], bn_momentum=0.01),
    "shapenetpart": dict(datasets="shapenetpart", num_classes=16,
                         num_parts=[4, 2, 2, 4, 4, 3, 3, 2, 4, 2, 6, 2, 3, 3, 3, 3], input_features_dim=3,
                         batch_size=16, num_points=2048, radius=0.05, sampleDl=0.02, nsamples=[11, 25, 37, 36, 33],
                         npoints=[1280, 768, 192, 64], bn_momentum=0.1),
}


def model_config(task="classification", local_aggregation_type="pospool", dataset=None, **overrides):
    """A stand-alone config with the reference's model defaults (utils/config.py:20-33) and the shipped cfgs' stage
    settings: cfgs/modelnet/*.yaml for classification, cfgs/s3dis/*.yaml for scene segmentation, and for
    multi_part_segmentation cfgs/partnet/*.yaml (dataset=None or "partnet") or cfgs/shapenetpart/*.yaml
    (dataset="shapenetpart").  N of PartNet (no num_points key in its yaml) is the dataset's 10000 points."""
    from .config import la_config
    c = la_config(local_aggregation_type, **{k: v for k, v in overrides.items() if isinstance(v, dict)})
    c.backbone, c.width, c.depth, c.bottleneck_ratio = "resnet", 144, 2, 2
    if task == "classification":
        c.update(head="resnet_cls", num_classes=40, input_features_dim=3, radius=0.05, sampleDl=0.02,
                 nsamples=[20, 31, 38, 36, 34], npoints=[2048, 512, 128, 32], num_points=10000)
    elif task == "scene_segmentation":
        c.update(head="resnet_scene_seg", num_classes=13, input_features_dim=4, radius=0.1, sampleDl=0.04,
                 nsamples=[26, 31, 38, 41, 39], npoints=[4096, 1152, 304, 88], num_points=15000)
    elif task == "multi_part_segmentation":
        d = dict(PART_DATASETS[dataset or "partnet"])
        d["num_parts"], d["nsamples"], d["npoints"] = list(d["num_parts"]), list(d["nsamples"]), list(d["npoints"])
        if d["datasets"] == "shapenetpart" and local_aggregation_type == "pointwisemlp":
            d["batch_size"] = 12
        c.update(head="resnet_part_seg", **d)
    else:
        raise NotImplementedError(task)
    for k, v in overrides.items():
        if not isinstance(v, dict):
            c[k] = v
    return c
