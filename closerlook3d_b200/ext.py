"""Drop-in for the reference's pybind module `pt_custom_ops._ext`
(/root/reference/pytorch/ops/pt_custom_ops/_ext_src/src/bindings.cpp:6-15): the same five function names,
argument order and return shapes, on libcl3d's kernels.  Put it in sys.modules['pt_custom_ops._ext'] to run the
reference's own `pt_utils.py` / operator modules (unfused) on these kernels."""
from . import ops
from ._lib import require_cuda


def group_points(points, idx):
    require_cuda(points, "points", ops.F32)   # fp32 only, as the reference's CHECK_IS_FLOAT
    return ops.group_points(points, idx)


def group_points_grad(grad_out, idx, n):
    require_cuda(grad_out, "grad_out", ops.F32)
    return ops.group_points_grad(grad_out, idx, n)


def masked_ordered_ball_query(query_xyz, support_xyz, query_mask, support_mask, radius, nsample):
    idx, idx_mask, _ = ops.ball_query(query_xyz, support_xyz, query_mask, support_mask, radius, nsample,
                                      want_mask=True, want_ncount=False)
    return [idx, idx_mask]


def masked_nearest_query(query_xyz, support_xyz, query_mask, support_mask):
    idx, idx_mask = ops.nearest_query(query_xyz, support_xyz, query_mask, support_mask)
    return [idx.unsqueeze(-1), idx_mask.unsqueeze(-1)]


def masked_grid_subsampling(points, mask, nsamples, sampleDl):
    sub_xyz, sub_mask = ops.grid_subsample(points, mask, nsamples, sampleDl)
    return [sub_xyz, sub_mask]
