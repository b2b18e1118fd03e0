"""Unfused GPU path for operator settings that no shipped cfg uses (output_conv / C_in != C_out, num_mlps > 1,
gaussian influence, ...; the max reduction of PosPool / AdaptiveWeight is fused, csrc/agg_max.cu).  Same mathematics as the fused kernels and the reference
(/root/reference/pytorch/models/local_aggregation_operators.py), built from this package's materialising
kernels (MaskedQueryAndGroup -> cl3d_ball_query_algo + cl3d_group_points) and torch library ops on the GPU.
It exists so that every configuration the reference accepts runs here too; it is not the hot path.
16-bit features are widened to fp32 and the result is rounded back to their dtype (autocast off throughout), like
the fused operators.
"""
import functools

import torch
import torch.nn.functional as F


def _fp32(fn):
    @functools.wraps(fn)
    def call(m, q_xyz, s_xyz, q_mask, s_mask, feats):
        with torch.autocast("cuda", enabled=False):
            return fn(m, q_xyz, s_xyz, q_mask, s_mask, feats.float()).to(feats.dtype)
    return call


def _reduce(agg, idx_mask, query_mask, reduction):
    # reference :87-105 -- identical in all families
    if reduction == 'max':
        return agg.max(dim=-1)[0]
    fm = (idx_mask + (1 - query_mask[:, :, None]))[:, None, :, :]
    out = (agg * fm).sum(-1)
    if reduction in ('avg', 'mean'):
        out = out / fm.sum(-1)
    return out


def _out(module, out):
    return module.out_conv(out) if module.output_conv else module.out_transform(out)


@_fp32
def pospool(m, q_xyz, s_xyz, q_mask, s_mask, feats):
    B, C, M, K = feats.shape[0], feats.shape[1], q_xyz.shape[1], m.nsample
    gf, dp, idx_mask = m.grouper(q_xyz, s_xyz, q_mask, s_mask, feats)
    if m.position_embedding == 'xyz':
        agg = (dp.unsqueeze(1) * gf.view(B, C // 3, 3, M, K)).view(B, C, M, K)
    else:
        fd = C // 6
        rng = torch.arange(fd, dtype=torch.float32, device=feats.device)
        dim_mat = torch.pow(1.0 * 1000, (1.0 / fd) * rng)
        div = torch.div((100 * dp).unsqueeze(-1), dim_mat)
        emb = torch.cat([torch.sin(div), torch.cos(div)], -1).permute(0, 1, 4, 2, 3).contiguous().view(B, C, M, K)
        agg = gf * emb
    return _out(m, _reduce(agg, idx_mask, q_mask, m.reduction))


@_fp32
def adaptive_weight(m, q_xyz, s_xyz, q_mask, s_mask, feats):
    B, C, M, K, S = feats.shape[0], feats.shape[1], q_xyz.shape[1], m.nsample, m.shared_channels
    gf, dp, idx_mask = m.grouper(q_xyz, s_xyz, q_mask, s_mask, feats)
    w = m.mlps(dp).unsqueeze(2)
    agg = (gf.view(B, C // S, S, M, K) * w).view(B, C, M, K)
    return _out(m, _reduce(agg, idx_mask, q_mask, m.reduction))


@_fp32
def pointwise_mlp(m, q_xyz, s_xyz, q_mask, s_mask, feats):
    gf, dp, idx_mask = m.grouper(q_xyz, s_xyz, q_mask, s_mask, feats)
    center = gf[..., 0:1].expand(-1, -1, -1, m.nsample)
    x = m.mlps(torch.cat([dp, center, gf - center], 1))
    if m.reduction != 'max':
        x = x.clone()  # the reference multiplies the ReLU output in place here, which autograd rejects
    return _reduce(x, idx_mask, q_mask, m.reduction)


@_fp32
def pseudo_grid(m, q_xyz, s_xyz, q_mask, s_mask, feats):
    B, C, M, K = feats.shape[0], feats.shape[1], q_xyz.shape[1], m.nsample
    gf, dp, idx_mask = m.grouper(q_xyz, s_xyz, q_mask, s_mask, feats)
    sq = torch.sum((dp.permute(0, 2, 3, 1).unsqueeze(3) - m.K_points) ** 2, -1)  # (B,M,K,nkp)
    if m.KP_influence == 'constant':
        h = torch.ones_like(sq)
    elif m.KP_influence == 'linear':
        h = torch.clamp(1 - torch.sqrt(sq) / m.extent, min=0.0)
    else:  # 'gaussian' -- broken in the reference (torch.pow(float, 2), models/utlis.py:294); defined here
        h = torch.exp(-sq / (2 * (m.extent * 0.3) ** 2 + 1e-9))
    fm = idx_mask + (1 - q_mask[:, :, None])
    h = h.permute(0, 1, 3, 2) * fm[:, :, None, :]
    wf = torch.bmm(h.reshape(-1, m.num_kernel_points, K), gf.permute(0, 2, 3, 1).contiguous().view(-1, K, C))
    out = torch.sum(wf * m.kernel_weights, 1).view(B, M, C).transpose(1, 2)
    return _out(m, out)
