"""Thin tensor-level wrappers over the C ABI (include/cl3d.h): allocate outputs/workspaces with torch,
pass raw device pointers + the current CUDA stream.  No computation happens in Python."""
import ctypes

import torch

from . import _lib
from ._lib import check, ptr, require_cuda, stream_ptr

I32 = torch.int32
F32 = torch.float32

# element type of a channel-major feature tensor -> CL3D_DTYPE_* (include/cl3d.h).  The features set the dtype of
# every tensor that crosses the layout boundary; everything inside the library stays fp32.
DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def require_features(t, name):
    """CUDA, contiguous, float32 / float16 / bfloat16 -> the dtype code"""
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (CPU not supported)")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous tensor")
    if t.dtype not in DTYPE_CODE:
        raise RuntimeError(f"{name} must be a float tensor (float32, float16 or bfloat16)")
    return DTYPE_CODE[t.dtype]


def _on_device(fn):
    """Run `fn` with the CUDA device of its tensor arguments current (kernels, the stream passed to the library and
    the per-device attributes all belong to the CURRENT device), and refuse operands spread over several devices
    (the reference's ops have the same single-device contract)."""
    import functools

    @functools.wraps(fn)
    def call(*args, **kw):
        dev = None
        for a in list(args) + list(kw.values()):
            if isinstance(a, torch.Tensor) and a.is_cuda:
                if dev is None:
                    dev = a.device
                elif a.device != dev:
                    raise RuntimeError(f"{fn.__name__}: operands on different devices ({dev} and {a.device})")
        if dev is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kw)
        with torch.cuda.device(dev):
            return fn(*args, **kw)
    return call


def no_autocast(fn):
    """Run `fn` with CUDA autocast off.  The library's modules and autograd Functions decide dtypes themselves (the
    features' dtype at the layout boundary, fp32 inside), so no torch op of theirs may be recast by autocast."""
    import functools

    @functools.wraps(fn)
    def call(*args, **kw):
        with torch.autocast("cuda", enabled=False):
            return fn(*args, **kw)
    return call


def deterministic_mode(deterministic=None):
    """None -> torch's flag (torch.use_deterministic_algorithms) at the time of the call.  Under it the transposed
    neighbour lists are built in canonical order (ascending q*K + k) and the scatters take their gather forms, so
    every fused operator gives the same bits on every run."""
    return torch.are_deterministic_algorithms_enabled() if deterministic is None else bool(deterministic)


def padded_channels(C):
    return (C + 7) & ~7


PM_SLACK = 256  # CL3D_PM_SLACK: readable floats after the last row of every gathered point-major buffer


def _empty_pm(B, N, W, device):
    """(B,N,W) fp32 view of an allocation with PM_SLACK floats of slack behind it"""
    return torch.empty(B * N * W + PM_SLACK, dtype=F32, device=device)[:B * N * W].view(B, N, W)


@_on_device
def ball_query(query_xyz, support_xyz, query_mask, support_mask, radius, nsample, want_mask=True, want_ncount=True,
               algo=0, csr=None, after_search=None, deterministic=None):
    """-> (idx (B,M,K) i32, idx_mask (B,M,K) i32 | None, ncount (B,M) i32 | None); bit-exact with the
    reference's masked_ordered_ball_query (masked_ordered_ball_query_gpu.cu:11-96).
    csr = "counted" | "all": also build the transposed lists in the same call (cl3d_ball_query_csr) and return
    (idx, idx_mask, ncount, (csr_off, csr_ent)).  after_search(): called between the search and the list build (the
    caller records its "search done" event there, so consumers of idx do not wait for the lists).
    deterministic (None: torch's flag): the lists in canonical order."""
    require_cuda(query_xyz, "query_xyz", F32)
    require_cuda(support_xyz, "support_xyz", F32)
    require_cuda(query_mask, "query_mask", I32)
    require_cuda(support_mask, "support_mask", I32)
    B, M, _ = query_xyz.shape
    N = support_xyz.shape[1]
    K = int(nsample)
    dev = query_xyz.device
    L = _lib.lib()
    idx = torch.empty(B, M, K, dtype=I32, device=dev)
    idx_mask = torch.empty(B, M, K, dtype=I32, device=dev) if want_mask else None
    ncount = torch.empty(B, M, dtype=I32, device=dev) if (want_ncount or csr) else None
    if csr:
        assert csr in ("counted", "all")
        off = torch.empty(B, N + 1, dtype=I32, device=dev)
        ent = torch.empty(B, M * K, dtype=I32, device=dev)
        det = int(deterministic_mode(deterministic))
        wsb = L.cl3d_ball_query_csr_workspace_bytes(B, N, M, K, det)
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        args = (ptr(query_xyz), ptr(support_xyz), ptr(query_mask), ptr(support_mask), B, N, M, float(radius), K, ptr(idx),
                ptr(idx_mask), ptr(ncount), 1 if csr == "all" else 0, ptr(off), ptr(ent), ptr(ws), wsb, int(algo))
        if after_search is None:
            check(L.cl3d_ball_query_csr(*args, 3, det, stream_ptr()), "cl3d_ball_query_csr")
        else:
            check(L.cl3d_ball_query_csr(*args, 1, det, stream_ptr()), "cl3d_ball_query_csr (search)")
            after_search()
            check(L.cl3d_ball_query_csr(*args, 2, det, stream_ptr()), "cl3d_ball_query_csr (lists)")
        return idx, idx_mask, ncount, (off, ent)
    wsb = L.cl3d_ball_query_workspace_bytes(B, N, M, K)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    check(L.cl3d_ball_query_algo(ptr(query_xyz), ptr(support_xyz), ptr(query_mask), ptr(support_mask), B, N, M,
                                 float(radius), K, ptr(idx), ptr(idx_mask), ptr(ncount), ptr(ws), wsb, int(algo),
                                 stream_ptr()), "cl3d_ball_query")
    return idx, idx_mask, ncount


@_on_device
def nearest_query(query_xyz, support_xyz, query_mask, support_mask):
    """-> (idx (B,M) i32, idx_mask (B,M) i32)  (masked_nearest_query_gpu.cu:8-62)"""
    require_cuda(query_xyz, "query_xyz", F32)
    require_cuda(support_xyz, "support_xyz", F32)
    require_cuda(query_mask, "query_mask", I32)
    require_cuda(support_mask, "support_mask", I32)
    B, M, _ = query_xyz.shape
    N = support_xyz.shape[1]
    idx = torch.empty(B, M, dtype=I32, device=query_xyz.device)
    idx_mask = torch.empty(B, M, dtype=I32, device=query_xyz.device)
    L = _lib.lib()
    wsb = L.cl3d_nearest_query_workspace_bytes(B, N, M)      # 0: small cloud, tile scan; else the cell grid
    ws = torch.empty(wsb, dtype=torch.uint8, device=query_xyz.device) if wsb else None
    check(L.cl3d_nearest_query(ptr(query_xyz), ptr(support_xyz), ptr(query_mask), ptr(support_mask), B, N, M,
                               ptr(idx), ptr(idx_mask), ptr(ws), wsb, stream_ptr()), "cl3d_nearest_query")
    return idx, idx_mask


@_on_device
def build_csr(idx, ncount, N, deterministic=None):
    """transposed neighbour lists -> (csr_off (B,N+1) i32, csr_ent (B,M*K) i32); ncount None = all K slots.
    deterministic (None: torch's flag): each list in ascending q*K + k instead of atomic arrival order."""
    B, M, K = idx.shape
    dev = idx.device
    L = _lib.lib()
    if ncount is None:
        ncount = torch.full((B, M), K, dtype=I32, device=dev)
    det = int(deterministic_mode(deterministic))
    off = torch.empty(B, N + 1, dtype=I32, device=dev)
    ent = torch.empty(B, M * K, dtype=I32, device=dev)
    wsb = L.cl3d_csr_workspace_bytes(B, N, M, K, det)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    check(L.cl3d_build_csr(ptr(idx), ptr(ncount), B, N, M, K, ptr(off), ptr(ent), ptr(ws), wsb, det, stream_ptr()),
          "cl3d_build_csr")
    return off, ent


@_on_device
def to_point_major(x_cn):
    """(B,C,N) f32 / f16 / bf16 -> (B,N,Cp) fp32 zero-padded rows"""
    dt = require_features(x_cn, "features")
    B, C, N = x_cn.shape
    out = _empty_pm(B, N, padded_channels(C), x_cn.device)
    check(_lib.lib().cl3d_to_point_major(ptr(x_cn), dt, B, C, N, ptr(out), stream_ptr()), "cl3d_to_point_major")
    return out


@_on_device
def to_channel_major(x_nc, C, dtype=F32):
    """(B,N,Cp) fp32 -> (B,C,N) in `dtype`"""
    B, N, Cp = x_nc.shape
    assert Cp == padded_channels(C)
    out = torch.empty(B, C, N, dtype=dtype, device=x_nc.device)
    check(_lib.lib().cl3d_to_channel_major(ptr(x_nc), B, C, N, ptr(out), DTYPE_CODE[dtype], stream_ptr()),
          "cl3d_to_channel_major")
    return out


@_on_device
def group_points(points, idx):
    dt = require_features(points, "points")
    require_cuda(idx, "idx", I32)
    B, C, N = points.shape
    _, M, K = idx.shape
    out = torch.empty(B, C, M, K, dtype=points.dtype, device=points.device)
    check(_lib.lib().cl3d_group_points(ptr(points), dt, ptr(idx), B, C, N, M, K, ptr(out), stream_ptr()),
          "cl3d_group_points")
    return out


@_on_device
def group_points_grad(grad_out, idx, n, deterministic=None):
    """a 16-bit gradient is accumulated in fp32 and rounded once.  deterministic (None: torch's flag): gathered
    over the canonical transposed lists of idx instead of scattered with atomics"""
    dt = require_features(grad_out, "grad_out")
    require_cuda(idx, "idx", I32)
    B, C, M, K = grad_out.shape
    out = torch.empty(B, C, int(n), dtype=grad_out.dtype, device=grad_out.device)
    off = ent = acc = None
    if deterministic_mode(deterministic):
        off, ent = build_csr(idx, None, int(n), deterministic=True)
    elif dt:
        acc = torch.empty(B, C, int(n), dtype=F32, device=grad_out.device)
    check(_lib.lib().cl3d_group_points_grad(ptr(grad_out), dt, ptr(idx), B, C, int(n), M, K, ptr(off), ptr(ent),
                                            ptr(out), ptr(acc), stream_ptr()), "cl3d_group_points_grad")
    return out


@_on_device
def reduce_partials(partial):
    """(T,P) -> (P,)"""
    T, P = partial.shape
    out = torch.empty(P, dtype=F32, device=partial.device)
    check(_lib.lib().cl3d_reduce_partials(ptr(partial), T, P, ptr(out), stream_ptr()), "cl3d_reduce_partials")
    return out


# --------------------------------------------------------------------------------------------------
# fused aggregation + out_transform
# --------------------------------------------------------------------------------------------------
FAM_POSPOOL_XYZ, FAM_POSPOOL_SINCOS, FAM_ADAPTIVE_DP, FAM_PSEUDOGRID = 0, 1, 2, 3
REDUCE = {"avg": 0, "mean": 0, "sum": 1, "max": 2}
BN_PARTIAL_ROWS = 4  # CL3D_BN_PARTIAL_ROWS: per tile and channel n, centre c, sum (x - c), sum (x - c)^2


def bn_partial_buffer(ntiles, C, device):
    """(ntiles, BN_PARTIAL_ROWS, C) fp32: a forward's per-tile BatchNorm moments, rows of one tile contiguous"""
    return torch.empty(ntiles, BN_PARTIAL_ROWS, C, dtype=F32, device=device)


def bn_partial_moments(partial):
    """(ntiles, BN_PARTIAL_ROWS, C) -> float64 (n, sum, M2) per tile and channel, each (ntiles, C); M2 = the tile's
    sum of squared deviations from its own mean"""
    p = partial.double()
    n, c, d, q = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
    return n, n * c + d, q - d * d / n


@_on_device
def agg_fwd(family, reduction, feat_pm, query_xyz, support_xyz, idx, ncount, p0, p1, C, radius, normalize, shared=1,
            nkp=0, extent=1.0, influence=0, want_bn_partial=True, arg=None):
    """-> (agg (B,C,M), bn_partial (ntiles,BN_PARTIAL_ROWS,C) | None);
    arg = (B,M,Cp) uint8 buffer for the winning slots, required by (and only by) the max reduction"""
    B, N, Cp = feat_pm.shape
    M, K = idx.shape[1], idx.shape[2]
    L = _lib.lib()
    dev = feat_pm.device
    agg = torch.empty(B, C, M, dtype=F32, device=dev)
    partial = bn_partial_buffer(L.cl3d_agg_num_tiles(B, M), C, dev) if want_bn_partial else None
    check(L.cl3d_agg_fwd(family, reduction, ptr(feat_pm), ptr(query_xyz), ptr(support_xyz), ptr(idx), ptr(ncount),
                         ptr(p0), ptr(p1), B, N, M, K, C, float(radius), int(normalize), int(shared), int(nkp),
                         float(extent), int(influence), ptr(agg), ptr(partial), ptr(arg), stream_ptr()), "cl3d_agg_fwd")
    return agg, partial


@_on_device
def agg_bwd(family, reduction, g_pm, feat_pm, query_xyz, support_xyz, ncount, csr_off, csr_ent, p0, p1, C, N, K,
            radius, normalize, shared=1, nkp=0, extent=1.0, influence=0, arg=None, dtype=F32):
    """-> (grad_feat (B,C,N) in `dtype`, param_grad (P//C, C) fp32 | None)   P = 4C (adaptive: x,y,z,bias) or
    nkp*C; arg = the forward's winning slots (max reduction)"""
    B, M, Cp = g_pm.shape
    L = _lib.lib()
    dev = g_pm.device
    grad_feat = torch.empty(B, C, N, dtype=dtype, device=dev)
    P = L.cl3d_agg_num_params(family, C, shared, nkp)
    partial = None
    if P > 0:
        partial = torch.empty(L.cl3d_agg_bwd_num_blocks(B, N), P, dtype=F32, device=dev)
    check(L.cl3d_agg_bwd(family, reduction, ptr(g_pm), ptr(feat_pm), ptr(query_xyz), ptr(support_xyz), ptr(ncount),
                         ptr(csr_off), ptr(csr_ent), ptr(p0), ptr(p1), B, N, M, K, C, float(radius), int(normalize),
                         int(shared), int(nkp), float(extent), int(influence), ptr(grad_feat), DTYPE_CODE[dtype],
                         ptr(partial), ptr(arg), stream_ptr()), "cl3d_agg_bwd")
    pg = reduce_partials(partial).view(P // C, C) if P > 0 else None
    return grad_feat, pg


@_on_device
def bn_finalize(bn_partial, C, count, eps, momentum, training, running_mean, running_var):
    """-> save_stats (2,C): mean, invstd.  Updates running stats in place when training."""
    dev = running_mean.device if running_mean is not None else bn_partial.device
    stats = torch.empty(2, C, dtype=F32, device=dev)
    nt = bn_partial.shape[0] if bn_partial is not None else 0
    check(_lib.lib().cl3d_bn_finalize(ptr(bn_partial), nt, C, int(count), float(eps), float(momentum), int(training),
                                      ptr(running_mean), ptr(running_var), ptr(stats), stream_ptr()),
          "cl3d_bn_finalize")
    return stats


def bn_sync_group(bn):
    """The process group over which `bn` synchronises its batch statistics, or None.  torch's SyncBatchNorm rule: `bn`
    is an nn.SyncBatchNorm in training mode, torch.distributed is initialised, and its process group (bn.process_group,
    else WORLD) has more than one rank.  The one place that knows about nn.SyncBatchNorm: every other BatchNorm, and a
    SyncBatchNorm that torch would not synchronise, takes the per-GPU path."""
    if not (isinstance(bn, torch.nn.SyncBatchNorm) and bn.training):
        return None
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()):
        return None
    group = bn.process_group or dist.group.WORLD
    return group if dist.get_world_size(group) > 1 else None


def _gather_ranks(t, group):
    """(R, C) on every rank -> (W, R, C): one all_gather over `group`, rows in rank order"""
    import torch.distributed as dist
    W = dist.get_world_size(group)
    out = torch.empty(W, *t.shape, dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out.view(W * t.shape[0], *t.shape[1:]), t, group=group)
    return out


def bn_batch_stats(bn, partial, C, count):
    """The BatchNorm statistics a fused forward normalises with, as nn.BatchNorm in `bn`'s mode: batch statistics
    (updating the running ones, momentum=None as a cumulative average) when training or when there are no running
    statistics, else the running ones.  -> (save_stats (2,C): mean, invstd; training; sync).
    sync is None, or (process group, global count (1,) float64 on the device) when `bn` synchronises (bn_sync_group):
    the statistics are then those of every rank's values, gathered once and merged in rank order on the device."""
    training = bn.training or bn.running_mean is None
    momentum = bn.momentum if bn.momentum is not None else 0.0
    if training and bn.running_mean is not None:
        bn.num_batches_tracked.add_(1)
        if bn.momentum is None:
            momentum = 1.0 / float(bn.num_batches_tracked)
    group = bn_sync_group(bn)
    if group is None:
        return bn_finalize(partial, C, count, bn.eps, momentum, training, bn.running_mean, bn.running_var), training, None
    stats, count_all = bn_finalize_ranks(partial, C, count, bn.eps, momentum, bn.running_mean, bn.running_var, group)
    return stats, training, (group, count_all)


@_on_device
def bn_finalize_ranks(bn_partial, C, count, eps, momentum, running_mean, running_var, group):
    """Training statistics over every rank of `group`: this rank's (4,C) float64 record of its per-tile moments, one
    all_gather, the merge in rank order.  -> (save_stats (2,C), global count (1,) float64); updates the running
    statistics with the global count."""
    L = _lib.lib()
    dev = bn_partial.device
    record = torch.empty(4, C, dtype=torch.float64, device=dev)
    check(L.cl3d_bn_rank_moments(ptr(bn_partial), bn_partial.shape[0], C, int(count), ptr(record), stream_ptr()),
          "cl3d_bn_rank_moments")
    records = _gather_ranks(record, group)
    stats = torch.empty(2, C, dtype=F32, device=dev)
    count_all = torch.empty(1, dtype=torch.float64, device=dev)
    check(L.cl3d_bn_finalize_ranks(ptr(records), records.shape[0], C, float(eps), float(momentum), ptr(running_mean),
                                   ptr(running_var), ptr(stats), ptr(count_all), stream_ptr()), "cl3d_bn_finalize_ranks")
    return stats, count_all


def _global_sums(dgb, group):
    """this rank's (2,C) backward sums -> the sums over every rank of `group`, added in rank order"""
    rows = _gather_ranks(dgb, group)
    return reduce_partials(rows.view(rows.shape[0], -1))


@_on_device
def bn_relu_fwd(x, stats, gamma, beta, dtype=F32):
    """x (B,C,M) fp32 -> y in `dtype`"""
    B, C, M = x.shape
    y = torch.empty(B, C, M, dtype=dtype, device=x.device)
    check(_lib.lib().cl3d_bn_relu_fwd(ptr(x), ptr(stats), ptr(gamma), ptr(beta), B, C, M, ptr(y), DTYPE_CODE[dtype],
                                      stream_ptr()), "cl3d_bn_relu_fwd")
    return y


@_on_device
def bn_relu_bwd(grad_y, x, stats, gamma, beta, training, sync=None):
    """grad_y in the features' dtype -> (g_pm (B,M,Cp) point-major d/d(agg), dgamma (C,), dbeta (C,)), all fp32.
    sync: the forward's (process group, global count): d/d(agg) takes the batch-statistic sums of every rank;
    dgamma and dbeta stay this rank's"""
    dt = require_features(grad_y, "grad_y")
    B, C, M = x.shape
    L = _lib.lib()
    dev = x.device
    partial = torch.empty(L.cl3d_agg_num_tiles(B, M), 2, C, dtype=F32, device=dev)
    dgb = torch.empty(2, C, dtype=F32, device=dev)
    g_pm = _empty_pm(B, M, padded_channels(C), dev)
    if sync is None:
        check(L.cl3d_bn_relu_bwd(ptr(grad_y), dt, ptr(x), ptr(stats), ptr(gamma), ptr(beta), B, C, M, int(training),
                                 ptr(partial), ptr(dgb), ptr(g_pm), stream_ptr()), "cl3d_bn_relu_bwd")
        return g_pm, dgb[0], dgb[1]
    group, count = sync
    check(L.cl3d_bn_relu_bwd_stats(ptr(grad_y), dt, ptr(x), ptr(stats), ptr(gamma), ptr(beta), B, C, M, ptr(partial),
                                   ptr(dgb), stream_ptr()), "cl3d_bn_relu_bwd_stats")
    sums = _global_sums(dgb, group)
    check(L.cl3d_bn_relu_bwd_apply(ptr(grad_y), dt, ptr(x), ptr(stats), ptr(gamma), ptr(beta), B, C, M, int(training),
                                   ptr(sums), ptr(count), ptr(partial), ptr(g_pm), stream_ptr()), "cl3d_bn_relu_bwd_apply")
    return g_pm, dgb[0], dgb[1]


# --------------------------------------------------------------------------------------------------
# fp32 GEMM + fused PointWiseMLP
# --------------------------------------------------------------------------------------------------
GEMM_AUTO, GEMM_FFMA, GEMM_TC3X = 0, 1, 2


@_on_device
def sgemm(a, sa_m, sa_k, b, sb_k, sb_n, M, N, K, out=None, ldc=None, splitk=1, algo=GEMM_AUTO):
    """out[m][n] = sum_k a[m*sa_m + k*sa_k] * b[k*sb_k + n*sb_n]  (element strides; fp32 accuracy: 3xTF32 on
    the wgmma tensor cores, or the fp32 FMA kernel -- see cl3d.h)"""
    L = _lib.lib()
    dev = a.device
    ldc = N if ldc is None else ldc
    if out is None:
        out = _empty_pm(1, M, ldc, dev).view(M, ldc)
    wsb = L.cl3d_sgemm_workspace_bytes(M, N, splitk)
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=dev) if splitk > 1 else None
    check(L.cl3d_sgemm_algo(ptr(a), sa_m, sa_k, ptr(b), sb_k, sb_n, M, N, K, ptr(out), ldc, splitk, ptr(ws), wsb,
                            algo, stream_ptr()), "cl3d_sgemm")
    return out


@_on_device
def to_point_major_aug(x_cn, xyz, radius):
    """(B,C,N) f32 / f16 / bf16 features + (B,N,3) xyz -> (B,N,Cpa) fp32 rows [f | xyz/r | 0], Cpa = padded(C+3)"""
    dt = require_features(x_cn, "features")
    B, C, N = x_cn.shape
    out = torch.empty(B, N, padded_channels(C + 3), dtype=F32, device=x_cn.device)
    check(_lib.lib().cl3d_to_point_major_aug(ptr(x_cn), dt, ptr(xyz), B, C, N, float(radius), ptr(out),
                                             stream_ptr()), "cl3d_to_point_major_aug")
    return out


@_on_device
def pwmlp_prep_weights(conv_weight, gamma, C, Cout):
    """-> wcat (2Cop, Cpa) rows zero-padded to Cpa = padded(C+3), wp (Cout,3), sgn (Cout)"""
    dev = conv_weight.device
    Cop = padded_channels(Cout)
    wcat = torch.empty(2 * Cop, padded_channels(C + 3), dtype=F32, device=dev)
    wp = torch.empty(Cout, 3, dtype=F32, device=dev)
    sgn = torch.empty(Cout, dtype=F32, device=dev)
    check(_lib.lib().cl3d_pwmlp_prep_weights(ptr(conv_weight), ptr(gamma), C, Cout, ptr(wcat), ptr(wp), ptr(sgn),
                                             stream_ptr()), "cl3d_pwmlp_prep_weights")
    return wcat, wp, sgn


@_on_device
def pwmlp_weight_grad(gwcat, grad_wp, sgn, C, Cout):
    gW = torch.empty(Cout, 3 + 2 * C, 1, 1, dtype=F32, device=gwcat.device)
    check(_lib.lib().cl3d_pwmlp_weight_grad(ptr(gwcat), ptr(grad_wp), ptr(sgn), C, Cout, ptr(gW), stream_ptr()),
          "cl3d_pwmlp_weight_grad")
    return gW


@_on_device
def pwmlp_fwd_stats(ab_pm, wp, sgn, query_xyz, support_xyz, idx, Cout, radius):
    B, N, _ = ab_pm.shape
    M, K = idx.shape[1], idx.shape[2]
    L = _lib.lib()
    dev = ab_pm.device
    Cop = padded_channels(Cout)
    ysel = torch.empty(B, Cout, M, dtype=F32, device=dev)
    aq = _empty_pm(B, M, Cop, dev)
    sq = torch.empty(B, M, Cop, dtype=F32, device=dev)
    karg = torch.empty(B, M, Cop, dtype=torch.uint8, device=dev)
    partial = bn_partial_buffer(L.cl3d_agg_num_tiles(B, M), Cout, dev)
    check(L.cl3d_pwmlp_fwd_stats(ptr(ab_pm), ptr(wp), ptr(sgn), ptr(query_xyz), ptr(support_xyz), ptr(idx), B, N, M, K, Cout,
                                 float(radius), ptr(ysel), ptr(aq), ptr(sq), ptr(karg), ptr(partial), stream_ptr()),
          "cl3d_pwmlp_fwd_stats")
    return ysel, aq, sq, karg, partial


@_on_device
def pwmlp_bwd(grad_out, beta, ab_pm, wp, sgn, query_xyz, support_xyz, idx, csr_off, csr_ent, ysel, aq, sq, karg, stats,
              gamma, radius, side_stream=None, training=True, deterministic=None, sync=None):
    """grad_out in the features' dtype -> (grad_ab_pm (B,N,2Cop), grad_wp (3,Cout), dgamma (Cout), dbeta (Cout)), fp32;
    the ReLU decision is recomputed from ysel, stats, gamma and beta.  side_stream: a torch stream the library may fork
    onto (zero-fill + query pass run beside the gather pass), joined before it returns.  deterministic (None: torch's
    flag): no atomics, every grad_ab row gathered from the canonical all-slots lists csr_off / csr_ent (required then,
    in eval mode too).  sync: the forward's (process group, global count): the passes after the statistics take the
    batch-statistic sums of every rank; dgamma and dbeta stay this rank's"""
    dt = require_features(grad_out, "grad_out")
    B, N, C2 = ab_pm.shape
    Cout, M, K = ysel.shape[1], ysel.shape[2], idx.shape[2]
    L = _lib.lib()
    dev = ysel.device
    det = int(deterministic_mode(deterministic))
    partial = _empty_pm(1, 1, L.cl3d_pwmlp_bwd_scratch_floats(B, N, M, Cout, det), dev)  # partials + sc*dz (+ da') rows
    dgb = torch.empty(2, Cout, dtype=F32, device=dev)
    grad_ab = torch.empty(B, N, C2, dtype=F32, device=dev)
    grad_wp = torch.empty(3, Cout, dtype=F32, device=dev)
    side = ctypes.c_void_p(side_stream.cuda_stream) if side_stream is not None else None
    args = (ptr(grad_out), dt, ptr(beta), ptr(ab_pm), ptr(wp), ptr(sgn), ptr(query_xyz), ptr(support_xyz), ptr(idx),
            ptr(csr_off), ptr(csr_ent), ptr(ysel), ptr(aq), ptr(sq), ptr(karg), ptr(stats), ptr(gamma),
            B, N, M, K, Cout, float(radius), int(bool(training)), det, ptr(partial))
    if sync is None:
        check(L.cl3d_pwmlp_bwd(*args, ptr(dgb), ptr(grad_ab), ptr(grad_wp), stream_ptr(), side), "cl3d_pwmlp_bwd")
        return grad_ab, grad_wp, dgb[0], dgb[1]
    group, count = sync
    check(L.cl3d_pwmlp_bwd_stats(ptr(grad_out), dt, ptr(beta), ptr(ysel), ptr(stats), ptr(gamma), B, M, Cout,
                                 ptr(partial), ptr(dgb), stream_ptr()), "cl3d_pwmlp_bwd_stats")
    sums = _global_sums(dgb, group)
    check(L.cl3d_pwmlp_bwd_apply(*args, ptr(sums), ptr(count), ptr(grad_ab), ptr(grad_wp), stream_ptr(), side),
          "cl3d_pwmlp_bwd_apply")
    return grad_ab, grad_wp, dgb[0], dgb[1]


# --------------------------------------------------------------------------------------------------
# grid subsampling, fused max-pool
# --------------------------------------------------------------------------------------------------
@_on_device
def grid_subsample(points, mask, npoint, sampleDl):
    """-> (sub_xyz (B,m,3) f32, sub_mask (B,m) i32); bit-exact with masked_grid_subsampling_gpu.cu:11-153"""
    require_cuda(points, "points", F32)
    require_cuda(mask, "mask", I32)
    B, n, _ = points.shape
    m = int(npoint)
    L = _lib.lib()
    dev = points.device
    sub = torch.empty(B, m, 3, dtype=F32, device=dev)
    sm = torch.empty(B, m, dtype=I32, device=dev)
    wsb = L.cl3d_grid_subsample_workspace_bytes(B, n, m)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    check(L.cl3d_grid_subsample(ptr(points), ptr(mask), B, n, m, float(sampleDl), ptr(sub), ptr(sm), ptr(ws), wsb,
                                stream_ptr()), "cl3d_grid_subsample")
    return sub, sm


@_on_device
def gather_max(features, idx):
    """out[b,c,q] = max_k features[b,c,idx[b,q,k]] -> (out (B,C,M) in the features' dtype, arg (B,M,Cp) uint8)"""
    dt = require_features(features, "features")
    require_cuda(idx, "idx", I32)
    B, C, N = features.shape
    M, K = idx.shape[1], idx.shape[2]
    feat_pm = to_point_major(features)
    out = torch.empty(B, C, M, dtype=features.dtype, device=features.device)
    arg = torch.empty(B, M, feat_pm.shape[2], dtype=torch.uint8, device=features.device)
    check(_lib.lib().cl3d_gather_max_fwd(ptr(feat_pm), ptr(idx), B, N, M, K, C, ptr(out), dt, ptr(arg),
                                         stream_ptr()), "cl3d_gather_max_fwd")
    return out, arg


@_on_device
def gather_max_grad(grad_out, idx, arg, N, csr=None, deterministic=None):
    """-> d/dfeatures (B,C,N) in grad_out's dtype (accumulated in fp32, rounded once).  deterministic (None: torch's
    flag): gathered over the canonical all-slots lists of idx -- `csr` when the caller has them, else built here"""
    dt = require_features(grad_out, "grad_out")
    B, C, M = grad_out.shape
    K = idx.shape[2]
    off = ent = None
    if deterministic_mode(deterministic):
        off, ent = csr if csr is not None else build_csr(idx, None, N, deterministic=True)
    g_pm = torch.empty(B, N, padded_channels(C), dtype=F32, device=grad_out.device)
    check(_lib.lib().cl3d_gather_max_bwd(ptr(grad_out), dt, ptr(idx), ptr(arg), B, N, M, K, C, ptr(off), ptr(ent),
                                         ptr(g_pm), stream_ptr()), "cl3d_gather_max_bwd")
    return to_channel_major(g_pm, C, grad_out.dtype)


# ---- fused multi-shape part-segmentation head (multihead.cu) ------------------------------------------------------
def _mhead_desc(C, num_parts, running_means=None, running_vars=None, nbts=None, grads=None):
    d = _lib.MHeadDesc()
    d.S, d.C = len(num_parts), int(C)
    for s, n in enumerate(num_parts):
        d.num_parts[s] = int(n)
        if running_means is not None:
            d.running_mean[s] = running_means[s].data_ptr()
            d.running_var[s] = running_vars[s].data_ptr()
        if nbts is not None and nbts[s] is not None:
            d.num_batches_tracked[s] = nbts[s].data_ptr()
        if grads is not None and grads[s] is not None:
            d.grad_logits[s] = grads[s].data_ptr()
    return d


@_on_device
def mhead_fwd(x, w1, gamma, beta, w2, b2, num_parts, running_means, running_vars, nbts, eps, momentum, training):
    """All S heads over x (B,C,N) f32 / f16 / bf16: -> (logits in x's dtype, save fp32).  logits is flat: the
    concatenation over s of contiguous (B, num_parts[s], N) blocks.  w1 (S,C,C), gamma/beta (S,C), w2
    (sum num_parts, C), b2 (sum num_parts), all fp32.  momentum None = cumulative average (needs nbts).  Training
    updates the running statistics in place and adds one to every num_batches_tracked."""
    dt = require_features(x, "x")
    for t, n in ((w1, "w1"), (gamma, "gamma"), (beta, "beta"), (w2, "w2"), (b2, "b2")):
        require_cuda(t, n, F32)
    B, C, N = x.shape
    L = _lib.lib()
    d = _mhead_desc(C, num_parts, running_means, running_vars, nbts)
    dp = ctypes.addressof(d)
    logits = torch.empty(B * N * sum(num_parts), dtype=x.dtype, device=x.device)
    save = torch.empty(L.cl3d_mhead_save_floats(len(num_parts), C), dtype=F32, device=x.device)
    wsb = L.cl3d_mhead_fwd_workspace_bytes(dp, B, N)
    if wsb == 0:
        raise RuntimeError("cl3d_mhead_fwd_workspace_bytes: " + L.cl3d_last_error().decode("utf-8", "replace"))
    ws = torch.empty(wsb, dtype=torch.uint8, device=x.device)
    check(L.cl3d_mhead_fwd(dp, ptr(x), dt, B, N, ptr(w1), ptr(gamma), ptr(beta), ptr(w2), ptr(b2), float(eps),
                           -1.0 if momentum is None else float(momentum), int(bool(training)), ptr(logits), ptr(save),
                           ptr(ws), wsb, stream_ptr()), "cl3d_mhead_fwd")
    return logits, save


@_on_device
def mhead_bwd(x, w1, w2, save, num_parts, grads, training):
    """grads: per head d/dlogits (B, num_parts[s], N) contiguous in x's dtype, or None (zero).
    -> (grad_x in x's dtype, grad_w1, grad_gamma, grad_beta, grad_w2, grad_b2 fp32)"""
    dt = require_features(x, "x")
    for s, g in enumerate(grads):
        if g is not None and g.dtype != x.dtype:
            raise RuntimeError(f"grads[{s}] is {g.dtype}: d/dlogits must have x's dtype ({x.dtype})")
        if g is not None:
            require_cuda(g, f"grads[{s}]", x.dtype)
    B, C, N = x.shape
    S = len(num_parts)
    L = _lib.lib()
    d = _mhead_desc(C, num_parts, grads=grads)
    dp = ctypes.addressof(d)
    dev = x.device
    gx = torch.empty(B, C, N, dtype=x.dtype, device=dev)
    gw1 = torch.empty(S, C, C, dtype=F32, device=dev)
    gg = torch.empty(S, C, dtype=F32, device=dev)
    gb = torch.empty(S, C, dtype=F32, device=dev)
    gw2 = torch.empty(sum(num_parts), C, dtype=F32, device=dev)
    gb2 = torch.empty(sum(num_parts), dtype=F32, device=dev)
    wsb = L.cl3d_mhead_bwd_workspace_bytes(dp, B, N)
    if wsb == 0:
        raise RuntimeError("cl3d_mhead_bwd_workspace_bytes: " + L.cl3d_last_error().decode("utf-8", "replace"))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    check(L.cl3d_mhead_bwd(dp, ptr(x), dt, B, N, ptr(w1), ptr(w2), ptr(save), int(bool(training)), ptr(gx), ptr(gw1),
                           ptr(gg), ptr(gb), ptr(gw2), ptr(gb2), ptr(ws), wsb, stream_ptr()), "cl3d_mhead_bwd")
    return gx, gw1, gg, gb, gw2, gb2
