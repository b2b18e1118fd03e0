"""oracle/f64_ext.py -- the `ext` surface of oracle/ext.py for a float64 run of la_oracle, on CPU or GPU tensors.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The neighbour searches are the C restatement (oracle.ext) on fp32 CPU copies of the coordinates, so the indices
never come from the kernels under test; the results are moved back to the device of the query.  Grouping and its
gradient are plain torch gather / scatter-add in the dtype of their input, so features, parameters and gradients
stay float64 end to end while the coordinates (and with them the relative positions) keep the reference's fp32
arithmetic -- see la_oracle.OracleLocalAggregation(dtype=torch.float64).
"""
import torch

from . import ext as _c


def _cpu32(t):
    return t.detach().to("cpu").contiguous()


def masked_ordered_ball_query(query_xyz, support_xyz, query_mask, support_mask, radius, nsample):
    idx, idx_mask = _c.masked_ordered_ball_query(_cpu32(query_xyz), _cpu32(support_xyz), _cpu32(query_mask),
                                                 _cpu32(support_mask), radius, nsample)
    return [idx.to(query_xyz.device), idx_mask.to(query_xyz.device)]


def masked_nearest_query(query_xyz, support_xyz, query_mask, support_mask):
    idx, idx_mask = _c.masked_nearest_query(_cpu32(query_xyz), _cpu32(support_xyz), _cpu32(query_mask),
                                            _cpu32(support_mask))
    return [idx.to(query_xyz.device), idx_mask.to(query_xyz.device)]


def masked_grid_subsampling(points, mask, nsamples, sampleDl):
    sub, sub_mask = _c.masked_grid_subsampling(_cpu32(points), _cpu32(mask), nsamples, sampleDl)
    return [sub.to(points.device), sub_mask.to(points.device)]


def _flat_idx(idx, C, device):
    B, M, K = idx.shape
    return idx.to(device=device, dtype=torch.long).reshape(B, 1, M * K).expand(B, C, M * K)


def group_points(points, idx):
    """(B,C,N), (B,M,K) int -> (B,C,M,K) in the dtype of `points`"""
    B, C, _ = points.shape
    _, M, K = idx.shape
    return points.gather(2, _flat_idx(idx, C, points.device)).view(B, C, M, K)


def group_points_grad(grad_out, idx, n):
    """(B,C,M,K), (B,M,K) int, n -> (B,C,n): the adjoint of group_points"""
    B, C, M, K = grad_out.shape
    out = torch.zeros(B, C, int(n), dtype=grad_out.dtype, device=grad_out.device)
    return out.scatter_add_(2, _flat_idx(idx, C, grad_out.device), grad_out.reshape(B, C, M * K))
