"""Host side of the fused PointWiseMLP (feature_type 'dp_fi_df', num_mlps 1, reduction 'max').

Reference: /root/reference/pytorch/models/local_aggregation_operators.py:254-257,288-303.
The conv weight W (Cout, 3+2C) = [Wp | Wc | Wr] and sgn = sign(BN gamma) are folded once per call into
    wcat (2*Cop, C+3):  rows 0..Cout-1       = [Wc - Wr | 0 0 0]        -> A  = (Wc-Wr) f
                        rows Cop..Cop+Cout-1 = sgn * [Wr | Wp]          -> T  = sgn (Wr f + Wp s/r)
so that ONE per-point product over the augmented point-major matrix [f | s/r] yields both terms
(csrc/pwmlp.cu explains why y[o,q,k] = a'[q][o] + sgn*T[j_k][o] is the reference's function).  The folding / unfolding of the small weight matrices is one tiny kernel each way (cl3d_pwmlp_prep_weights /
cl3d_pwmlp_weight_grad).
"""
import torch
from torch.autograd import Function

from . import ops, pt_utils


class _FusedPointWiseMLP(Function):
    @staticmethod
    @ops.no_autocast
    def forward(ctx, features, conv_weight, bn_weight, bn_bias, nl, query_xyz, support_xyz, radius, bn):
        B, C, N = features.shape
        M, K = nl.idx.shape[1], nl.idx.shape[2]
        Cout = conv_weight.shape[0]
        Cop = ops.padded_channels(Cout)
        wcat, wp, sgn = ops.pwmlp_prep_weights(conv_weight.contiguous(), bn_weight, C, Cout)
        fa_pm = ops.to_point_major_aug(features, support_xyz, radius)          # (B,N,Cpa)
        Cpa = fa_pm.shape[2]
        # AB[p][n] = sum_c fa[p][c] * wcat[n][c]   (both row-padded to Cpa with zeros -> k runs over Cpa)
        ab_pm = ops.sgemm(fa_pm, Cpa, 1, wcat, 1, Cpa, B * N, 2 * Cop, Cpa).view(B, N, 2 * Cop)
        nl.wait()                                   # the search ran on the side stream, overlapping the product
        if any(ctx.needs_input_grad) and (bn.training or bn.running_mean is None or ops.deterministic_mode()):
            nl.prefetch_csr(all_slots=True)         # lists for the backward, built behind the forward kernels
        ysel, aq, sq, karg, partial = ops.pwmlp_fwd_stats(ab_pm, wp, sgn, query_xyz, support_xyz, nl.idx, Cout, radius)
        stats, training, sync = ops.bn_batch_stats(bn, partial, Cout, B * M * K)
        out = ops.bn_relu_fwd(ysel, stats, bn_weight, bn_bias, dtype=features.dtype)
        ctx.nl, ctx.radius, ctx.training, ctx.sync = nl, radius, training, sync
        ctx.dims = (B, C, N, M, K, Cout, Cop, Cpa)
        ctx.dtype = features.dtype
        # the backward recomputes the ReLU decision from ysel and the BatchNorm constants, not from `out`
        ctx.save_for_backward(fa_pm, ab_pm, wp, sgn, wcat, ysel, aq, sq, karg, stats, bn_weight, bn_bias, query_xyz,
                              support_xyz)
        return out

    @staticmethod
    @ops.no_autocast
    def backward(ctx, grad_out):
        (fa_pm, ab_pm, wp, sgn, wcat, ysel, aq, sq, karg, stats, bn_weight, bn_bias, query_xyz,
         support_xyz) = ctx.saved_tensors
        B, C, N, M, K, Cout, Cop, Cpa = ctx.dims
        nl = ctx.nl
        # eval mode (frozen BatchNorm): no batch-statistics terms -> no dense pass, no transposed lists needed, except
        # in deterministic mode, where every gradient row is gathered over the canonical lists
        det = ops.deterministic_mode()
        off, ent = nl.csr_all_slots() if ctx.training or det else (None, None)
        side = pt_utils._side_stream(ysel.device, priority=-1) if pt_utils.overlap_enabled else None
        grad_ab, grad_wp, dgamma, dbeta = ops.pwmlp_bwd(grad_out.contiguous(), bn_bias, ab_pm, wp, sgn, query_xyz, support_xyz, nl.idx,
                                                        off, ent, ysel, aq, sq, karg, stats, bn_weight, ctx.radius,
                                                        side_stream=side, training=ctx.training, deterministic=det,
                                                        sync=ctx.sync)
        P = B * N
        Cp = ops.padded_channels(C)
        # the two products of the backward are independent: the weight gradient runs on the side stream
        cur = torch.cuda.current_stream()
        side = pt_utils._side_stream(grad_ab.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            # d/dwcat (2Cop x Cpa) = grad_AB^T (2Cop x P) @ fa (P x Cpa): long reduction -> split-K
            splitk = max(1, min(1024, P // 128))   # ~128 points per partial sum (see cl3d_sgemm_algo)
            gwcat = ops.sgemm(grad_ab, 1, 2 * Cop, fa_pm, Cpa, 1, 2 * Cop, Cpa, P, splitk=splitk)
            gW = ops.pwmlp_weight_grad(gwcat, grad_wp, sgn, C, Cout)
        # d/dfeat (point-major) = grad_AB (P x 2Cop) @ wcat[:, :Cp] (2Cop x Cp; columns >= C are unused)
        gf_pm = ops.sgemm(grad_ab, 2 * Cop, 1, wcat, Cpa, 1, P, Cp, 2 * Cop, ldc=Cp).view(B, N, Cp)
        grad_feat = ops.to_channel_major(gf_pm, C, ctx.dtype)
        cur.wait_stream(side)
        return grad_feat, gW, dgamma, dbeta, None, None, None, None, None


def forward(module, query_xyz, support_xyz, query_mask, support_mask, support_features):
    conv, bn = module.mlps.conv0[0], module.mlps.conv0[1]
    # a differentiated forward in training mode needs the all-slots transposed lists (BatchNorm2d backward is dense)
    need_lists = torch.is_grad_enabled() and (bn.training or bn.running_mean is None or ops.deterministic_mode())
    nl = pt_utils.neighbors(query_xyz, support_xyz, query_mask, support_mask, module.radius, module.nsample,
                            csr="all" if need_lists else None)
    return _FusedPointWiseMLP.apply(support_features.contiguous(), conv.weight, bn.weight, bn.bias, nl, query_xyz,
                                    support_xyz, module.radius, bn)
