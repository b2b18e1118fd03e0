"""Data parallelism of the hot path: clouds are independent, so a batch shards over ranks by the batch
dimension and the only exchange is the all-reduce of parameter gradients (reference: DistributedSampler +
DistributedDataParallel(broadcast_buffers=False), /root/reference/pytorch/function/train_modelnet_dist.py:117,206;
BatchNorm statistics are per GPU by default, not synchronised).  One process per GPU, NCCL over NVLink/NVSwitch
(gloo on CPU in the tests).

A model converted with nn.SyncBatchNorm.convert_sync_batchnorm synchronises its BatchNorm statistics, fused operators
included: each fused BatchNorm then adds one all_gather of a small float64 record in the forward and one of its
(sum gy*xhat, sum gy) in the backward, over bn.process_group (ops.bn_sync_group, ops.bn_batch_stats).  dgamma and
dbeta stay per rank and travel with the parameter-gradient all-reduce.  Shards may be uneven (shard_range)."""
import torch
import torch.distributed as dist


def shard_range(total, world_size, rank):
    """contiguous [lo, hi) of `total` clouds owned by `rank` (earlier ranks take the remainder)"""
    base, rem = divmod(total, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def world_size():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


class FlatGradients:
    """ONE persistent buffer behind every parameter gradient (the reference's DDP keeps the same thing: a flat
    bucket whose slices are the .grad tensors, train_modelnet_dist.py:206).

    `attach()` points each p.grad at its slice of the buffer, so the backward accumulates straight into it and
    `allreduce()` is a single collective on memory that never moves: no per-step torch.cat, no copy back, and the
    collective can be captured in a CUDA graph (GraphedStep) because its address is static.
    """

    def __init__(self, params):
        self.params = [p for p in params if p.requires_grad]
        n = sum(p.numel() for p in self.params)
        dev = self.params[0].device if self.params else torch.device("cpu")
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        self.views = []
        o = 0
        for p in self.params:
            self.views.append(self.flat[o:o + p.numel()].view_as(p))
            o += p.numel()

    def attach(self):
        """p.grad <- view into the flat buffer (call once; survives zero())"""
        for p, v in zip(self.params, self.views):
            p.grad = v
        return self

    def zero(self):
        self.flat.zero_()

    def load(self, grads):
        """copy a list of gradient tensors (same order as the parameters) into the buffer: one kernel"""
        torch.cat([g.reshape(-1) for g in grads], out=self.flat)

    def allreduce(self, average=True):
        """sum (and divide by the world size) across ranks, in place; no-op on one rank"""
        w = world_size()
        if w == 1 or self.flat.numel() == 0:
            return self.flat
        dist.all_reduce(self.flat)
        if average:
            self.flat.mul_(1.0 / w)
        return self.flat


def allreduce_gradients(params, average=True):
    """All-reduce every parameter gradient with one collective.  If the gradients already live in one flat
    buffer (FlatGradients.attach) nothing is copied; otherwise they are flattened once and copied back."""
    params = [p for p in params if p.grad is not None]
    if not params or world_size() == 1:
        return
    g0 = params[0].grad
    base = g0._base if g0._base is not None else None
    if base is not None and base.dim() == 1 and all(p.grad._base is base for p in params) and \
            sum(p.grad.numel() for p in params) == base.numel():
        dist.all_reduce(base)
        if average:
            base.mul_(1.0 / world_size())
        return
    flat = torch.cat([p.grad.reshape(-1) for p in params])
    dist.all_reduce(flat)
    if average:
        flat /= world_size()
    o = 0
    for p in params:
        n = p.grad.numel()
        p.grad.copy_(flat[o:o + n].view_as(p.grad))
        o += n
