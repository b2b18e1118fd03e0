"""Drop-in replacement for the reference's `models/local_aggregation_operators.py`
(/root/reference/pytorch/models/local_aggregation_operators.py): the same five classes
    PosPool (:16)  AdaptiveWeight (:115)  PointWiseMLP (:227)  PseudoGrid (:319)  LocalAggregation (:429)
with the same constructor / forward signatures and the same state-dict keys (checkpoints load unmodified),
but each forward is ONE fused pass over libcl3d's sm_90a kernels instead of the reference's
MaskedQueryAndGroup + ~10 elementwise torch ops over (B,C,M,K) tensors:

    neighbour search (grid hash, cached)  ->  fused gather + transform + reduce  ->  fused BN + ReLU

and each backward is a gather-form pass over transposed neighbour lists.  Settings no shipped cfg uses
(output_conv, num_mlps > 1, gaussian influence, ...) run through `_composed.py`, the same
mathematics on the materialising GPU kernels (still no CPU path).
"""
import math

import torch
import torch.nn as nn
from torch.autograd import Function

from . import _composed, ops
from . import pt_utils
from .kernel_points import create_kernel_points, weight_variable
from .pt_utils import MaskedQueryAndGroup


class _AggSpec:
    """static description of one fused aggregation (everything that is not a tensor)"""

    def __init__(self, family, reduction, radius, nsample, normalize, shared=1, nkp=0, extent=1.0, influence=0):
        self.family, self.reduction, self.radius, self.nsample = family, reduction, radius, nsample
        self.normalize, self.shared, self.nkp, self.extent, self.influence = normalize, shared, nkp, extent, influence


class _FusedAggBNReLU(Function):
    """agg = fused_aggregation(features) ; out = relu(batchnorm1d(agg))"""

    @staticmethod
    @ops.no_autocast
    def forward(ctx, features, p0, p1, bn_weight, bn_bias, spec, nl, query_xyz, support_xyz, bn):
        # features: fp32, fp16 or bf16; out and d/dfeatures come in that dtype, everything between is fp32
        B, C, N = features.shape
        M = query_xyz.shape[1]
        feat_pm = ops.to_point_major(features)   # overlaps the neighbour search running on the side stream
        arg = None
        if spec.reduction == ops.REDUCE["max"]:   # winning slot per (query, channel), read again by the backward
            arg = torch.empty(B, M, feat_pm.shape[2], dtype=torch.uint8, device=features.device)
        nl.wait()
        agg, partial = ops.agg_fwd(spec.family, spec.reduction, feat_pm, query_xyz, support_xyz, nl.idx, nl.ncount,
                                   p0, p1, C, spec.radius, spec.normalize, spec.shared, spec.nkp, spec.extent,
                                   spec.influence, want_bn_partial=bn.training or bn.running_mean is None, arg=arg)
        stats, training, sync = ops.bn_batch_stats(bn, partial, C, B * M)
        out = ops.bn_relu_fwd(agg, stats, bn_weight, bn_bias, dtype=features.dtype)
        if any(ctx.needs_input_grad):
            nl.prefetch_csr(all_slots=False)      # transposed lists for the backward, built behind the forward
        ctx.spec, ctx.nl, ctx.training, ctx.sync, ctx.N, ctx.dtype = spec, nl, training, sync, N, features.dtype
        needs_feat = spec.family in (ops.FAM_ADAPTIVE_DP, ops.FAM_PSEUDOGRID)
        ctx.save_for_backward(agg, stats, bn_weight, bn_bias, query_xyz, support_xyz, p0, p1,
                              feat_pm if needs_feat else None, arg)
        return out

    @staticmethod
    @ops.no_autocast
    def backward(ctx, grad_out):
        agg, stats, bn_weight, bn_bias, query_xyz, support_xyz, p0, p1, feat_pm, arg = ctx.saved_tensors
        spec, nl = ctx.spec, ctx.nl
        C = agg.shape[1]
        g_pm, dgamma, dbeta = ops.bn_relu_bwd(grad_out.contiguous(), agg, stats, bn_weight, bn_bias, ctx.training,
                                              sync=ctx.sync)
        off, ent = nl.csr()
        grad_feat, pg = ops.agg_bwd(spec.family, spec.reduction, g_pm, feat_pm, query_xyz, support_xyz, nl.ncount,
                                    off, ent, p0, p1, C, ctx.N, spec.nsample, spec.radius, spec.normalize,
                                    spec.shared, spec.nkp, spec.extent, spec.influence, arg=arg, dtype=ctx.dtype)
        gp0 = gp1 = None
        if spec.family == ops.FAM_ADAPTIVE_DP:  # pg: (4, C) rows x,y,z,bias per channel -> fold shared groups
            S = spec.shared
            gp0 = pg[:3].t().reshape(C // S, S, 3).sum(1).reshape(p0.shape)
            gp1 = pg[3].reshape(C // S, S).sum(1).reshape(p1.shape)
        elif spec.family == ops.FAM_PSEUDOGRID:
            gp1 = pg.reshape(p1.shape)
        return grad_feat, gp0, gp1, dgamma, dbeta, None, None, None, None, None


def _check_inputs(query_xyz, support_xyz, query_mask, support_mask, support_features):
    """the reference's CHECK_* macros (utils.h:9-30) -> RuntimeError"""
    from ._lib import require_cuda
    require_cuda(query_xyz, "query_xyz", torch.float32)
    require_cuda(support_xyz, "support_xyz", torch.float32)
    require_cuda(query_mask, "query_mask", torch.int32)
    require_cuda(support_mask, "support_mask", torch.int32)
    if not support_features.is_cuda:
        raise RuntimeError("points must be a CUDA tensor (CPU not supported)")
    if support_features.dtype not in ops.DTYPE_CODE:
        raise RuntimeError("points must be a float tensor (float32, float16 or bfloat16)")


def _out_block(module, in_channels, out_channels, momentum):
    """registers out_conv / out_transform exactly as the reference (:37-45) so state-dict keys match"""
    if module.output_conv:
        module.out_conv = nn.Sequential(
            nn.Conv1d(in_channels, out_channels, kernel_size=1, bias=False),
            nn.BatchNorm1d(out_channels, momentum=momentum),
            nn.ReLU(inplace=True))
    else:
        module.out_transform = nn.Sequential(
            nn.BatchNorm1d(out_channels, momentum=momentum),
            nn.ReLU(inplace=True))


class PosPool(nn.Module):
    def __init__(self, in_channels, out_channels, radius, nsample, config):
        """A PosPool operator for local aggregation (reference :16-45)."""
        super().__init__()
        self.in_channels, self.out_channels, self.radius, self.nsample = in_channels, out_channels, radius, nsample
        self.position_embedding = config.pospool.position_embedding
        self.reduction = config.pospool.reduction
        self.output_conv = config.pospool.output_conv or (self.in_channels != self.out_channels)
        self.grouper = MaskedQueryAndGroup(radius, nsample, use_xyz=False, ret_grouped_xyz=True, normalize_xyz=True)
        _out_block(self, in_channels, out_channels, config.bn_momentum)
        self._dim_mat = None

    def _fusable(self):
        return (not self.output_conv) and self.position_embedding in ("xyz", "sin_cos") and \
            (self.reduction in ("avg", "mean", "sum") or (self.reduction == "max" and self.nsample <= 256))

    @ops.no_autocast
    def forward(self, query_xyz, support_xyz, query_mask, support_mask, support_features):
        """(B,M,3),(B,N,3),(B,M) i32,(B,N) i32,(B,C,N) -> (B,C_out,M)   (reference :47-112)"""
        if self.position_embedding not in ("xyz", "sin_cos"):
            raise NotImplementedError(f'Position Embedding {self.position_embedding} not implemented in PosPool')
        if self.reduction not in ("max", "avg", "mean", "sum"):
            raise NotImplementedError(f'Reduction {self.reduction} not implemented in PosPool ')
        C = support_features.shape[1]
        if not self._fusable():
            return _composed.pospool(self, query_xyz, support_xyz, query_mask, support_mask, support_features)
        _check_inputs(query_xyz, support_xyz, query_mask, support_mask, support_features)
        if self.position_embedding == "xyz":
            if C % 3 != 0:  # the reference's view(B, C // 3, 3, ...) fails the same way (:67)
                raise RuntimeError(f"shape '[B, {C // 3}, 3, M, K]' is invalid for input with {C} channels")
            fam, p0 = ops.FAM_POSPOOL_XYZ, None
        else:
            if C % 6 != 0:
                raise RuntimeError(f"shape '[B, {C}, M, K]' is invalid for a {6 * (C // 6)}-channel embedding")
            fam = ops.FAM_POSPOOL_SINCOS
            if self._dim_mat is None or self._dim_mat.device != support_features.device or \
                    self._dim_mat.numel() != C // 6:
                fd = C // 6  # same torch expression as the reference (:72-74) for bit parity of the constants
                rng = torch.arange(fd, dtype=torch.float32).to(support_features.device)
                self._dim_mat = torch.pow(1.0 * 1000, (1.0 / fd) * rng).contiguous()
            p0 = self._dim_mat
        nl = pt_utils.neighbors(query_xyz, support_xyz, query_mask, support_mask, self.radius, self.nsample,
                                 csr="counted" if torch.is_grad_enabled() else None)
        spec = _AggSpec(fam, ops.REDUCE[self.reduction], self.radius, self.nsample, normalize=1)
        bn = self.out_transform[0]
        return _FusedAggBNReLU.apply(support_features.contiguous(), p0, None, bn.weight, bn.bias, spec, nl,
                                     query_xyz, support_xyz, bn)


class AdaptiveWeight(nn.Module):
    def __init__(self, in_channels, out_channels, radius, nsample, config):
        """A AdaptiveWeight operator for local aggregation (reference :115-168)."""
        super().__init__()
        self.in_channels, self.out_channels, self.radius, self.nsample = in_channels, out_channels, radius, nsample
        self.weight_type = config.adaptive_weight.weight_type
        self.weight_to_channels = {'dp': 3, 'df': in_channels, 'fj': in_channels, 'dp_df': 3 + in_channels,
                                   'dp_fj': 3 + in_channels, 'fi_df': 2 * in_channels,
                                   'dp_fi_df': 3 + 2 * in_channels, 'rscnn': 10}
        self.weight_input_channels = self.weight_to_channels[self.weight_type]
        self.num_mlps = config.adaptive_weight.num_mlps
        self.shared_channels = config.adaptive_weight.shared_channels
        self.weight_softmax = config.adaptive_weight.weight_softmax
        self.reduction = config.adaptive_weight.reduction
        self.output_conv = config.adaptive_weight.output_conv or (self.in_channels != self.out_channels)
        self.grouper = MaskedQueryAndGroup(radius, nsample, use_xyz=False, ret_grouped_xyz=True, normalize_xyz=True)
        self.mlps = nn.Sequential()
        self.mlps.add_module('conv0', nn.Conv2d(self.weight_input_channels, self.in_channels // self.shared_channels,
                                                kernel_size=1))
        for i in range(self.num_mlps - 1):
            self.mlps.add_module(f'relu{i}', nn.ReLU(inplace=True))
            self.mlps.add_module(f'conv{i + 1}', nn.Conv2d(self.in_channels // self.shared_channels,
                                                           self.in_channels // self.shared_channels, kernel_size=1))
        _out_block(self, in_channels, out_channels, config.bn_momentum)

    def _fusable(self):
        return (not self.output_conv) and self.num_mlps == 1 and \
            (self.reduction in ("avg", "mean", "sum") or (self.reduction == "max" and self.nsample <= 256))

    @ops.no_autocast
    def forward(self, query_xyz, support_xyz, query_mask, support_mask, support_features):
        """reference :170-224"""
        if self.weight_type != 'dp':
            raise NotImplementedError(f'Weight Type {self.weight_type} not implemented in AdaptiveWeight')
        if self.reduction not in ("max", "avg", "mean", "sum"):
            raise NotImplementedError(f'Reduction {self.reduction} not implemented in PosPool ')
        if not self._fusable():
            return _composed.adaptive_weight(self, query_xyz, support_xyz, query_mask, support_mask, support_features)
        _check_inputs(query_xyz, support_xyz, query_mask, support_mask, support_features)
        C = support_features.shape[1]
        S = self.shared_channels
        conv = self.mlps.conv0
        nl = pt_utils.neighbors(query_xyz, support_xyz, query_mask, support_mask, self.radius, self.nsample,
                                 csr="counted" if torch.is_grad_enabled() else None)
        spec = _AggSpec(ops.FAM_ADAPTIVE_DP, ops.REDUCE[self.reduction], self.radius, self.nsample, normalize=1,
                        shared=S)
        bn = self.out_transform[0]
        return _FusedAggBNReLU.apply(support_features.contiguous(), conv.weight.view(C // S, 3), conv.bias,
                                     bn.weight, bn.bias, spec, nl, query_xyz, support_xyz, bn)


class PseudoGrid(nn.Module):
    def __init__(self, in_channels, out_channels, radius, nsample, config):
        """A PseudoGrid operator for local aggregation (reference :319-366)."""
        super().__init__()
        self.in_channels, self.out_channels, self.radius, self.nsample = in_channels, out_channels, radius, nsample
        self.KP_influence = config.pseudo_grid.KP_influence
        self.num_kernel_points = config.pseudo_grid.num_kernel_points
        self.convolution_mode = config.pseudo_grid.convolution_mode
        self.output_conv = config.pseudo_grid.output_conv or (self.in_channels != self.out_channels)
        KP_extent = config.pseudo_grid.KP_extent
        fixed_kernel_points = config.pseudo_grid.fixed_kernel_points
        density_parameter = config.density_parameter
        self.extent = 2 * KP_extent * radius / density_parameter
        K_radius = 1.5 * self.extent
        K_points_numpy = create_kernel_points(K_radius, self.num_kernel_points, num_kernels=1, dimension=3,
                                              fixed=fixed_kernel_points)
        K_points_numpy = K_points_numpy.reshape((self.num_kernel_points, 3))
        self.register_buffer('K_points', torch.from_numpy(K_points_numpy).type(torch.float32))
        self.grouper = MaskedQueryAndGroup(radius, nsample, use_xyz=False, ret_grouped_xyz=True, normalize_xyz=False)
        self.kernel_weights = weight_variable([self.num_kernel_points, in_channels])
        _out_block(self, in_channels, out_channels, config.bn_momentum)

    def _fusable(self):
        return (not self.output_conv) and self.KP_influence in ("linear", "constant") and self.num_kernel_points <= 16

    @ops.no_autocast
    def forward(self, query_xyz, support_xyz, query_mask, support_mask, support_features):
        """reference :368-426"""
        if self.KP_influence not in ("constant", "linear", "gaussian"):
            raise ValueError('Unknown influence function type (config.KP_influence)')
        if self.convolution_mode != 'sum':
            raise NotImplementedError(f"convolution_mode:{self.convolution_mode} not support in PseudoGrid")
        if not self._fusable():
            return _composed.pseudo_grid(self, query_xyz, support_xyz, query_mask, support_mask, support_features)
        _check_inputs(query_xyz, support_xyz, query_mask, support_mask, support_features)
        nl = pt_utils.neighbors(query_xyz, support_xyz, query_mask, support_mask, self.radius, self.nsample,
                                 csr="counted" if torch.is_grad_enabled() else None)
        spec = _AggSpec(ops.FAM_PSEUDOGRID, ops.REDUCE["sum"], self.radius, self.nsample, normalize=0,
                        nkp=self.num_kernel_points, extent=self.extent,
                        influence=1 if self.KP_influence == "constant" else 0)
        bn = self.out_transform[0]
        return _FusedAggBNReLU.apply(support_features.contiguous(), self.K_points, self.kernel_weights, bn.weight,
                                     bn.bias, spec, nl, query_xyz, support_xyz, bn)


class PointWiseMLP(nn.Module):
    def __init__(self, in_channels, out_channels, radius, nsample, config):
        """A PointWiseMLP operator for local aggregation (reference :227-272)."""
        super().__init__()
        self.in_channels, self.out_channels, self.radius, self.nsample = in_channels, out_channels, radius, nsample
        self.feature_type = config.pointwisemlp.feature_type
        self.feature_input_channels = {'dp_fj': 3 + in_channels, 'fi_df': 2 * in_channels,
                                       'dp_fi_df': 3 + 2 * in_channels}
        self.feature_input_channels = self.feature_input_channels[self.feature_type]
        self.num_mlps = config.pointwisemlp.num_mlps
        self.reduction = config.pointwisemlp.reduction
        self.grouper = MaskedQueryAndGroup(radius, nsample, use_xyz=False, ret_grouped_xyz=True, normalize_xyz=True)
        bn_m = config.bn_momentum
        self.mlps = nn.Sequential()
        if self.num_mlps == 1:
            self.mlps.add_module('conv0', nn.Sequential(
                nn.Conv2d(self.feature_input_channels, self.out_channels, kernel_size=1, bias=False),
                nn.BatchNorm2d(self.out_channels, momentum=bn_m), nn.ReLU(inplace=True)))
        else:
            mfdim = max(self.in_channels // 2, 9)
            self.mlps.add_module('conv0', nn.Sequential(
                nn.Conv2d(self.feature_input_channels, mfdim, kernel_size=1, bias=False),
                nn.BatchNorm2d(mfdim, momentum=bn_m), nn.ReLU(inplace=True)))
            for i in range(self.num_mlps - 2):
                self.mlps.add_module(f'conv{i + 1}', nn.Sequential(
                    nn.Conv2d(mfdim, mfdim, kernel_size=1, bias=False),
                    nn.BatchNorm2d(mfdim, momentum=bn_m), nn.ReLU(inplace=True)))
            self.mlps.add_module(f'conv{self.num_mlps - 1}', nn.Sequential(
                nn.Conv2d(mfdim, self.out_channels, kernel_size=1, bias=False),
                nn.BatchNorm2d(self.out_channels, momentum=bn_m), nn.ReLU(inplace=True)))

    def _fusable(self):
        return self.num_mlps == 1 and self.reduction == "max"

    @ops.no_autocast
    def forward(self, query_xyz, support_xyz, query_mask, support_mask, support_features):
        """reference :274-316"""
        if self.feature_type != 'dp_fi_df':
            raise NotImplementedError(f'Feature Type {self.feature_type} not implemented in PointWiseMLP')
        if self.reduction not in ("max", "avg", "mean", "sum"):
            raise NotImplementedError(f'Reduction {self.reduction} not implemented in PointWiseMLP')
        if not self._fusable():
            return _composed.pointwise_mlp(self, query_xyz, support_xyz, query_mask, support_mask, support_features)
        _check_inputs(query_xyz, support_xyz, query_mask, support_mask, support_features)
        from . import pwmlp
        return pwmlp.forward(self, query_xyz, support_xyz, query_mask, support_mask, support_features)


class LocalAggregation(nn.Module):
    def __init__(self, in_channels, out_channels, radius, nsample, config):
        """LocalAggregation operators (reference :429-450): string dispatch on config.local_aggregation_type."""
        super().__init__()
        if config.local_aggregation_type == 'pospool':
            self.local_aggregation_operator = PosPool(in_channels, out_channels, radius, nsample, config)
        elif config.local_aggregation_type == 'adaptive_weight':
            self.local_aggregation_operator = AdaptiveWeight(in_channels, out_channels, radius, nsample, config)
        elif config.local_aggregation_type == 'pointwisemlp':
            self.local_aggregation_operator = PointWiseMLP(in_channels, out_channels, radius, nsample, config)
        elif config.local_aggregation_type == 'pseudo_grid':
            self.local_aggregation_operator = PseudoGrid(in_channels, out_channels, radius, nsample, config)
        else:
            raise NotImplementedError(f'LocalAggregation {config.local_aggregation_type} not implemented')

    def forward(self, query_xyz, support_xyz, query_mask, support_mask, support_features):
        """query_xyz (B,M,3), support_xyz (B,N,3), masks (B,M)/(B,N) int32, support_features (B,C_in,N)
        -> (B,C_out,M)   (reference :452-464).  support_features may be float32, float16 or bfloat16 (e.g. under
        torch.autocast): the output and the feature gradient come in that dtype, the arithmetic is fp32."""
        if support_features.is_cuda and support_features.device.index != torch.cuda.current_device():
            with torch.cuda.device(support_features.device):  # streams / launches belong to the tensors' device
                return self.local_aggregation_operator(query_xyz, support_xyz, query_mask, support_mask,
                                                       support_features)
        return self.local_aggregation_operator(query_xyz, support_xyz, query_mask, support_mask, support_features)
