"""The multi-shape head of part segmentation (models/heads/segmentation_head.py:124-149) on the fused kernel.

The reference runs every shape's head, Conv1d(C,C) -> BatchNorm1d(C) -> ReLU -> Conv1d(C, num_parts[s]) + bias, over
every point of the batch, one after the other.  `multi_shape_heads_forward` runs all of them in one fused pass
(csrc/multihead.cu) and returns the reference's output, a list of S tensors (B, num_parts[s], N); they are views of
one buffer, nothing is copied.  The heads' parameters and buffers stay in the reference's module tree (state-dict
keys unchanged); BatchNorm keeps nn.BatchNorm1d's semantics in both modes, including the running-statistics update
and num_batches_tracked.

The fused path is taken when the input allows it: x is a CUDA fp32, fp16 or bf16 (B,C,N) tensor, padded C <= 128,
every num_parts <= 64, at most 32 heads, all head parameters and buffers are fp32, and all head BatchNorms share one
mode, momentum and eps and track running statistics.  Any other input runs the reference's own composition of torch
modules (so does a head converted wholesale to a 16-bit type), and so does a head whose BatchNorm is an
nn.SyncBatchNorm that synchronises (ops.bn_sync_group): the fused kernel keeps its statistics per GPU.

16-bit x (what the decoder hands the heads under torch.autocast) follows the library's dtype rule: the logits and
d/dx come back in x's dtype, d/dlogits must arrive in it, and everything in between -- parameters, BatchNorm
statistics, saved state, every accumulator -- stays fp32.  So the result is exactly the fp32 head on x.float(), rounded
once to x's dtype (fp16: inf exactly where that rounding overflows), and the parameter gradients and running
statistics are the fp32 run's, bit for bit.
"""
import torch

from . import _lib, ops


def _parts(heads):
    return [int(h[3].out_channels) for h in heads]


def fused_eligible(heads, x):
    """whether `multi_shape_heads_forward` takes the fused kernel for this input"""
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype in ops.DTYPE_CODE and x.dim() == 3):
        return False
    S, C = len(heads), x.shape[1]
    if not (1 <= S <= _lib.MHEAD_MAX_HEADS) or ops.padded_channels(C) > _lib.MHEAD_MAX_CHANNELS:
        return False
    if x.shape[0] < 1 or x.shape[2] < 1:
        return False
    bn0 = heads[0][1]
    for h in heads:
        conv1, bn, conv2 = h[0], h[1], h[3]
        if conv1.bias is not None or conv2.bias is None or not (1 <= conv2.out_channels <= _lib.MHEAD_MAX_PARTS):
            return False
        if conv1.weight.shape[:2] != (C, C) or conv2.weight.shape[1] != C:
            return False
        if not (bn.track_running_stats and bn.running_mean is not None and bn.affine):
            return False
        if ops.bn_sync_group(bn) is not None:   # cross-rank statistics: torch's SyncBatchNorm in the composition
            return False
        if (bn.training, bn.momentum, bn.eps) != (bn0.training, bn0.momentum, bn0.eps):
            return False
        for t in (conv1.weight, conv2.weight, conv2.bias, bn.weight, bn.bias, bn.running_mean, bn.running_var):
            if not (t.is_cuda and t.dtype == torch.float32 and t.device == x.device):
                return False
    return True


class _MultiShapeHeads(torch.autograd.Function):
    @staticmethod
    @ops.no_autocast
    def forward(ctx, x, w1, gamma, beta, w2, b2, meta):
        num_parts, bns, training, momentum, eps = meta
        x = x.contiguous()
        logits, save = ops.mhead_fwd(x, w1, gamma, beta, w2, b2, num_parts, [bn.running_mean for bn in bns],
                                     [bn.running_var for bn in bns], [bn.num_batches_tracked for bn in bns], eps,
                                     momentum, training)
        ctx.save_for_backward(x, w1, w2, save)
        ctx.num_parts, ctx.training = num_parts, training
        ctx.set_materialize_grads(False)
        B, _, N = x.shape
        outs, off = [], 0
        for n in num_parts:
            outs.append(logits[off:off + B * n * N].view(B, n, N))
            off += B * n * N
        return tuple(outs)

    @staticmethod
    @ops.no_autocast
    def backward(ctx, *grads):
        x, w1, w2, save = ctx.saved_tensors
        grads = [None if g is None else g.contiguous() for g in grads]
        gx, gw1, gg, gb, gw2, gb2 = ops.mhead_bwd(x, w1, w2, save, ctx.num_parts, grads, ctx.training)
        return gx, gw1, gg, gb, gw2, gb2, None


def multi_shape_heads_forward(heads, x):
    """[heads[s](x) for s] -- fused when `fused_eligible(heads, x)`, else exactly the reference's loop"""
    if not fused_eligible(heads, x):
        return [h(x) for h in heads]
    bns = [h[1] for h in heads]
    w1 = torch.stack([h[0].weight.squeeze(-1) for h in heads])
    gamma = torch.stack([bn.weight for bn in bns])
    beta = torch.stack([bn.bias for bn in bns])
    w2 = torch.cat([h[3].weight.squeeze(-1) for h in heads])
    b2 = torch.cat([h[3].bias for h in heads])
    meta = (_parts(heads), bns, bool(bns[0].training), bns[0].momentum, float(bns[0].eps))
    return list(_MultiShapeHeads.apply(x, w1, gamma, beta, w2, b2, meta))
