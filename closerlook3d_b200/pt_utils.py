"""Drop-in replacement for the reference's `pt_utils` module
(/root/reference/pytorch/ops/pt_custom_ops/pt_utils.py): same public names, constructor / forward
signatures, return shapes and autograd behaviour, running on libcl3d's sm_90a kernels.

    reference name (pt_utils.py line)            here
    grouping_operation            (:64)          GroupingOperation.apply      -> cl3d_group_points[_grad]
    masked_ordered_ball_query     (:80)          MaskedOrderedBallQuery.apply -> cl3d_ball_query_algo (grid hash)
    masked_nearest_query          (:95)          MaskedNearestQuery.apply     -> cl3d_nearest_query
    masked_grid_subsampling       (:111)         MaskedGridSubsampling.apply  -> cl3d_grid_subsample
    MaskedQueryAndGroup           (:114)         same forward contract (materialising compat path)
    MaskedNearestQueryAndGroup    (:147)
    MaskedMaxPool                 (:179)         fused: no (B,C,M,K) tensor
    MaskedUpsample                (:205)         nearest: fused gather of one row per query

The fused LocalAggregation operators (local_aggregation_operators.py in this package) do NOT go through
MaskedQueryAndGroup: they share its neighbour search via `neighbors()` below, which also caches the
neighbour lists so that the duplicate queries of a backbone forward (la1/btnk1, MaskedMaxPool + the strided
block's LocalAggregation: 5 of 14, SURVEY.md 3.3) are searched once.
"""
import collections

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function

from . import ops


# --------------------------------------------------------------------------------------------------
# neighbour lists + cache
# --------------------------------------------------------------------------------------------------
class NeighborList:
    """idx (B,M,K) i32, ncount (B,M) i32 [+ idx_mask (B,M,K) i32 on demand, CSR lists on demand].

    The search (and, when a backward will follow, the transposed lists) is enqueued on a side stream so that it
    overlaps the layout change / per-point product of the caller; `wait()` / `csr()` make the current stream
    wait for it.  Every use of the side stream starts with side.wait_stream(current), so memory allocated there
    is never recycled under a pending consumer."""

    def __init__(self, idx, ncount, idx_mask, N):
        self.idx, self.ncount, self._idx_mask, self.N = idx, ncount, idx_mask, N
        self._csr = None
        self._csr_all = None
        self._csr_det = self._csr_all_det = False   # whether each list set is canonical (ops.deterministic_mode)
        self.event = None
        self._csr_event = None
        self._csr_all_event = None

    def wait(self):
        if self.event is not None:
            torch.cuda.current_stream().wait_event(self.event)
        return self

    @property
    def idx_mask(self):
        if self._idx_mask is None:
            raise RuntimeError("idx_mask was not requested for this neighbour list")
        return self._idx_mask

    def _build(self, all_slots, det):
        return ops.build_csr(self.idx, None if all_slots else self.ncount, self.N, deterministic=det)

    def _have(self, all_slots, det):
        """lists of this kind exist and were built in mode `det` (a change of torch's flag rebuilds them)"""
        if all_slots:
            return self._csr_all is not None and self._csr_all_det == det
        return self._csr is not None and self._csr_det == det

    def _set(self, all_slots, det, csr, ev):
        if all_slots:
            self._csr_all, self._csr_all_det, self._csr_all_event = csr, det, ev
        else:
            self._csr, self._csr_det, self._csr_event = csr, det, ev

    def prefetch_csr(self, all_slots=False):
        """enqueue the transposed-list build on the side stream right behind the search"""
        det = ops.deterministic_mode()
        if self._have(all_slots, det):
            return
        side = _side_stream(self.idx.device)
        if self.event is not None:
            side.wait_event(self.event)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            csr = self._build(all_slots, det)
            ev = torch.cuda.Event()
            ev.record(side)
        self._set(all_slots, det, csr, ev)

    def _lists(self, all_slots):
        det = ops.deterministic_mode()
        if not self._have(all_slots, det):
            self.wait()
            self._set(all_slots, det, self._build(all_slots, det), None)
        else:
            ev = self._csr_all_event if all_slots else self._csr_event
            if ev is not None:
                torch.cuda.current_stream().wait_event(ev)
        return self._csr_all if all_slots else self._csr

    def csr(self):
        """transposed lists over the COUNTED slots (k < ncount): avg/sum families.  Canonical order while torch's
        deterministic flag is on."""
        return self._lists(False)

    def csr_all_slots(self):
        """transposed lists over ALL K slots (BatchNorm2d of PointWiseMLP sees every slot; the max-pool and
        group-points gradients' gather forms)"""
        return self._lists(True)


_SIDE = {}
overlap_enabled = True  # run the neighbour search on a side stream (fork/join), see NeighborList


def _side_stream(device, priority=0):
    """per-device helper stream; priority=-1: a second, high-priority one (its CTAs are scheduled first when it
    and the main stream both have a kernel pending -- used for short latency-bound passes beside a long one)"""
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device(), priority)
    st = _SIDE.get(key)
    if st is None:
        st = torch.cuda.Stream(device=device, priority=priority)
        _SIDE[key] = st
    return st


_CACHE = collections.OrderedDict()
_CACHE_SIZE = 8
cache_enabled = True
cache_stats = {"hit": 0, "miss": 0}


def _key(t):
    return (t.data_ptr(), tuple(t.shape), t._version, t.device.index)


def clear_neighbor_cache():
    _CACHE.clear()


def neighbors(query_xyz, support_xyz, query_mask, support_mask, radius, nsample, need_mask=False, overlap=None,
              csr=None):
    """Ball-query neighbour list for (query, support, radius, nsample), cached on tensor identity
    (data pointer + version; the cache keeps the key tensors alive so pointers cannot be recycled).
    With overlap (default: pt_utils.overlap_enabled) the search runs on a side stream; consumers call
    nl.wait() (the fused operators do) before touching nl.idx / nl.ncount.
    csr = "counted" | "all": a backward will follow -- the transposed lists are built in the same call as the
    search (ranks taken in its emit phase), not by a separate count / scan / fill afterwards."""
    key = (_key(query_xyz), _key(support_xyz), _key(query_mask), _key(support_mask), float(radius), int(nsample))
    if cache_enabled:
        hit = _CACHE.get(key)
        if hit is not None and (hit[0]._idx_mask is not None or not need_mask):
            _CACHE.move_to_end(key)
            cache_stats["hit"] += 1
            return hit[0]
    cache_stats["miss"] += 1
    overlap = overlap_enabled if overlap is None else overlap
    det = ops.deterministic_mode()
    lists = None
    if overlap:
        cur = torch.cuda.current_stream()
        side = _side_stream(query_xyz.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            ev = torch.cuda.Event()          # search done: idx / ncount final (the forward kernels wait for this one)
            res = ops.ball_query(query_xyz, support_xyz, query_mask, support_mask, radius, nsample,
                                 want_mask=need_mask, want_ncount=True, csr=csr,
                                 after_search=(lambda: ev.record(side)) if csr else None, deterministic=det)
            if not csr:
                ev.record(side)
            idx, idx_mask, ncount = res[:3]
            lists = res[3] if csr else None
            ev_lists = None
            if csr:                          # lists done: only the backward waits for this one
                ev_lists = torch.cuda.Event()
                ev_lists.record(side)
        nl = NeighborList(idx, ncount, idx_mask, support_xyz.shape[1])
        nl.event = ev
    else:
        res = ops.ball_query(query_xyz, support_xyz, query_mask, support_mask, radius, nsample,
                             want_mask=need_mask, want_ncount=True, csr=csr, deterministic=det)
        idx, idx_mask, ncount = res[:3]
        lists = res[3] if csr else None
        nl = NeighborList(idx, ncount, idx_mask, support_xyz.shape[1])
    if lists is not None:
        lists_event = ev_lists if overlap else None    # in-order on the current stream without overlap
        nl._set(csr == "all", det, lists, lists_event)
    if cache_enabled:
        _CACHE[key] = (nl, (query_xyz, support_xyz, query_mask, support_mask))
        while len(_CACHE) > _CACHE_SIZE:
            _CACHE.popitem(last=False)
    return nl


# --------------------------------------------------------------------------------------------------
# autograd functions with the reference's names
# --------------------------------------------------------------------------------------------------
class GroupingOperation(Function):
    """pt_utils.py:16-61"""

    @staticmethod
    @ops.no_autocast
    def forward(ctx, features, idx):
        ctx.for_backwards = (idx, features.size(2))
        return ops.group_points(features.contiguous(), idx)   # in the features' dtype (fp32, fp16 or bf16)

    @staticmethod
    @ops.no_autocast
    def backward(ctx, grad_out):
        idx, N = ctx.for_backwards
        return ops.group_points_grad(grad_out.contiguous(), idx, N), None


grouping_operation = GroupingOperation.apply


class MaskedOrderedBallQuery(Function):
    """pt_utils.py:67-77"""

    @staticmethod
    def forward(ctx, radius, nsample, query_xyz, support_xyz, query_mask, support_mask):
        nl = neighbors(query_xyz, support_xyz, query_mask, support_mask, radius, nsample, need_mask=True).wait()
        ctx.mark_non_differentiable(nl.idx, nl.idx_mask)
        return nl.idx, nl.idx_mask

    @staticmethod
    def backward(ctx, a=None, b=None):
        return None, None, None, None, None, None


masked_ordered_ball_query = MaskedOrderedBallQuery.apply


class MaskedNearestQuery(Function):
    """pt_utils.py:83-92; returns (B,M,1) tensors like the reference"""

    @staticmethod
    def forward(ctx, query_xyz, support_xyz, query_mask, support_mask):
        idx, idx_mask = ops.nearest_query(query_xyz, support_xyz, query_mask, support_mask)
        idx, idx_mask = idx.unsqueeze(-1), idx_mask.unsqueeze(-1)
        ctx.mark_non_differentiable(idx, idx_mask)
        return idx, idx_mask

    @staticmethod
    def backward(ctx, a=None, b=None):
        return None, None, None, None


masked_nearest_query = MaskedNearestQuery.apply


class MaskedGridSubsampling(Function):
    """pt_utils.py:98-108"""

    @staticmethod
    def forward(ctx, xyz, mask, npoint, sampleDl):
        sub_xyz, sub_mask = ops.grid_subsample(xyz, mask, npoint, sampleDl)
        ctx.mark_non_differentiable(sub_xyz, sub_mask)
        return sub_xyz, sub_mask

    @staticmethod
    def backward(ctx, a=None, b=None):
        return None, None, None, None


masked_grid_subsampling = MaskedGridSubsampling.apply


# --------------------------------------------------------------------------------------------------
# modules
# --------------------------------------------------------------------------------------------------
class MaskedQueryAndGroup(nn.Module):
    """pt_utils.py:114-144 (materialising compatibility path: returns the (B,C,M,K) tensors)."""

    def __init__(self, radius, nsample, use_xyz=True, ret_grouped_xyz=False, normalize_xyz=False):
        super().__init__()
        self.radius, self.nsample, self.use_xyz = radius, nsample, use_xyz
        self.ret_grouped_xyz = ret_grouped_xyz
        self.normalize_xyz = normalize_xyz

    def forward(self, query_xyz, support_xyz, query_mask, support_mask, features=None):
        idx, idx_mask = masked_ordered_ball_query(self.radius, self.nsample, query_xyz, support_xyz, query_mask,
                                                  support_mask)
        xyz_trans = support_xyz.transpose(1, 2).contiguous()
        grouped_xyz = grouping_operation(xyz_trans, idx)  # (B,3,M,K)
        grouped_xyz = grouped_xyz - query_xyz.transpose(1, 2).unsqueeze(-1)
        if self.normalize_xyz:
            grouped_xyz = grouped_xyz / self.radius
        if features is not None:
            grouped_features = grouping_operation(features, idx)
            new_features = torch.cat([grouped_xyz, grouped_features], dim=1) if self.use_xyz else grouped_features
        else:
            assert self.use_xyz, "Cannot have not features and not use xyz as a feature!"
            new_features = grouped_xyz
        if self.ret_grouped_xyz:
            return new_features, grouped_xyz, idx_mask
        return new_features, idx_mask


class MaskedNearestQueryAndGroup(nn.Module):
    """pt_utils.py:147-176"""

    def __init__(self, use_xyz=True, ret_grouped_xyz=False, normalize_xyz=False):
        super().__init__()
        self.use_xyz, self.ret_grouped_xyz, self.normalize_xyz = use_xyz, ret_grouped_xyz, normalize_xyz

    def forward(self, query_xyz, support_xyz, query_mask, support_mask, features=None):
        idx, idx_mask = masked_nearest_query(query_xyz, support_xyz, query_mask, support_mask)
        xyz_trans = support_xyz.transpose(1, 2).contiguous()
        grouped_xyz = grouping_operation(xyz_trans, idx)
        grouped_xyz = grouped_xyz - query_xyz.transpose(1, 2).unsqueeze(-1)
        if self.normalize_xyz:  # the reference reads self.radius here, which this class never defines (:160)
            raise AttributeError("'MaskedNearestQueryAndGroup' object has no attribute 'radius'")
        if features is not None:
            grouped_features = grouping_operation(features, idx)
            new_features = torch.cat([grouped_xyz, grouped_features], dim=1) if self.use_xyz else grouped_features
        else:
            assert self.use_xyz, "Cannot have not features and not use xyz as a feature!"
            new_features = grouped_xyz
        if self.ret_grouped_xyz:
            return new_features, grouped_xyz, idx_mask
        return new_features, idx_mask


class _GatherMax(Function):
    """out[b,c,q] = max_k f[b,c,idx[b,q,k]]  (fused MaskedMaxPool body: pt_utils.py:195-201); nl = the NeighborList
    of idx, whose cached all-slots lists the deterministic backward gathers over"""

    @staticmethod
    @ops.no_autocast
    def forward(ctx, features, idx, nl):
        out, arg = ops.gather_max(features, idx)   # in the features' dtype; the winning slots decide the backward
        ctx.save_for_backward(idx, arg)
        ctx.N, ctx.nl = features.shape[2], nl
        return out

    @staticmethod
    @ops.no_autocast
    def backward(ctx, grad_out):
        idx, arg = ctx.saved_tensors
        csr = ctx.nl.csr_all_slots() if ops.deterministic_mode() else None
        return ops.gather_max_grad(grad_out.contiguous(), idx, arg, ctx.N, csr=csr), None, None


class MaskedMaxPool(nn.Module):
    """pt_utils.py:179-202"""

    def __init__(self, npoint, radius, nsample, sampleDl):
        super().__init__()
        self.npoint, self.radius, self.nsample, self.sampleDl = npoint, radius, nsample, sampleDl

    def forward(self, xyz, mask, features):
        sub_xyz, sub_mask = masked_grid_subsampling(xyz, mask, self.npoint, self.sampleDl)
        sub_xyz = sub_xyz.contiguous()
        sub_mask = sub_mask.contiguous()
        nl = neighbors(sub_xyz, xyz, sub_mask, mask, self.radius, self.nsample).wait()
        sub_features = _GatherMax.apply(features.contiguous(), nl.idx, nl)
        return sub_xyz, sub_mask, sub_features


class MaskedUpsample(nn.Module):
    """pt_utils.py:205-227"""

    def __init__(self, radius, nsample, mode='nearest'):
        super().__init__()
        self.radius, self.nsample, self.mode = radius, nsample, mode

    def forward(self, up_xyz, xyz, up_mask, mask, features):
        if self.mode == 'nearest':
            idx, _ = masked_nearest_query(up_xyz, xyz, up_mask, mask)  # (B,M,1)
            return grouping_operation(features, idx)[..., 0].contiguous()
        elif self.mode == 'max':
            nl = neighbors(up_xyz, xyz, up_mask, mask, self.radius, self.nsample).wait()
            return _GatherMax.apply(features.contiguous(), nl.idx, nl)
        raise NotImplementedError(f"mode:{self.mode} not supported in MaskedUpsample")
