"""CUDA-graph replay of one LocalAggregation training step (forward + backward).

The hot path of a small cloud batch is ~40 short kernels; launched eagerly from Python the host cannot keep
the GPU busy: at the small BASELINE shapes the host time per step exceeds the kernel time.
`GraphedStep` captures the whole step -- neighbour search, layout change, fused aggregation, BN, and the
autograd backward -- once into a CUDA graph with static input / output buffers and replays it.  Nothing is
cached between replays: every replay runs the full search and aggregation on whatever the static input
buffers hold at that moment.
"""
import torch


class GraphedStep:
    """step = module(xyz, xyz, mask, mask, features) ; out.backward(grad_out) [; all-reduce of the gradients].

    static buffers (write your batch into them, then call replay()):
        .xyz (B,N,3) f32   .mask (B,N) i32   .features (B,C,N) f32   .grad_out (B,C_out,N) f32
    results after replay():
        .out (B,C_out,N), .features.grad,
        .param_grads   the parameter gradients THIS graph writes (static tensors, one per parameter, local to
                       this rank) -- several GraphedSteps over one module each own their set; p.grad only points
                       at the set of the graph captured last, so consumers must read the slot's own tensors,
        .flat_grad     one flat buffer with every parameter gradient, gathered inside the graph; with
                       allreduce=True (default: whenever torch.distributed is initialised with >1 rank) the NCCL
                       all-reduce (sum / world) of that buffer is captured in the graph as well, so a data-parallel
                       step is ONE graph launch: no per-step torch.cat, no eager collective.
        .grads()       views of .flat_grad shaped like the parameters (the reduced gradients).
        .result        (1 + n_param) f32: [sum(out) | flat_grad], assembled inside the graph: the step's device->host payload.
    """

    def __init__(self, module, xyz, mask, features, grad_out, warmup=3, allreduce=None, average=True):
        from . import dist as cdist
        from . import pt_utils
        self.module = module
        self.xyz = xyz.clone()
        self.mask = mask.clone()
        self.features = features.detach().clone().requires_grad_(True)
        self.grad_out = grad_out.clone()
        self.params = [p for p in module.parameters() if p.requires_grad]
        self.world = cdist.world_size()
        self.allreduce = (self.world > 1) if allreduce is None else (bool(allreduce) and self.world > 1)
        self.average = average
        self._cache_was = pt_utils.cache_enabled
        pt_utils.cache_enabled = False  # a captured search must never be skipped on replay
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._eager()
            if self.allreduce:  # communicator set-up must not happen inside the capture
                import torch.distributed as dist
                dist.all_reduce(torch.zeros(max(1, sum(p.numel() for p in self.params)), device=self.xyz.device))
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        try:  # parameters were created on the default stream; the captured backward accumulates on the capture stream
            torch.autograd.graph.set_warn_on_accumulate_grad_stream_mismatch(False)
        except Exception:
            pass
        self.graph = torch.cuda.CUDAGraph()
        self.features.grad = None
        for p in self.params:
            p.grad = None
        with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
            self.out = self.module(self.xyz, self.xyz, self.mask, self.mask, self.features)
            self.out.backward(self.grad_out)
            self.param_grads = [p.grad for p in self.params]
            self.flat_grad = torch.cat([g.reshape(-1) for g in self.param_grads]) if self.params else None
            if self.allreduce:
                import torch.distributed as dist
                dist.all_reduce(self.flat_grad)
                if average:
                    self.flat_grad.mul_(1.0 / self.world)
            # what leaves the device after a step: [sum of the output (stand-in for the loss) | parameter gradients]
            parts = [self.out.detach().sum().reshape(1)] + ([self.flat_grad] if self.flat_grad is not None else [])
            self.result = torch.cat(parts)
        pt_utils.cache_enabled = self._cache_was

    def _eager(self):
        self.features.grad = None
        for p in self.params:
            p.grad = None
        out = self.module(self.xyz, self.xyz, self.mask, self.mask, self.features)
        out.backward(self.grad_out)
        return out

    def load(self, xyz, mask, features, non_blocking=True):
        """copy a batch (device or pinned host tensors) into the static input buffers"""
        self.xyz.copy_(xyz, non_blocking=non_blocking)
        self.mask.copy_(mask, non_blocking=non_blocking)
        with torch.no_grad():
            self.features.copy_(features, non_blocking=non_blocking)

    def replay(self):
        self.graph.replay()
        return self.out

    def grads(self):
        """the (all-reduced, when data parallel) parameter gradients of the last replay: views of .flat_grad"""
        out, o = [], 0
        for p in self.params:
            out.append(self.flat_grad[o:o + p.numel()].view_as(p))
            o += p.numel()
        return out


class PipelinedTrainer:
    """End-to-end stepping from HOST batches: two GraphedSteps (double-buffered static inputs) and a copy stream,
    so the host->device copy of batch i+1 overlaps the replay of batch i; the step's result (sum of the output,
    a stand-in for the loss) is copied back asynchronously and read one step later.  Every batch is still
    copied, searched, aggregated and differentiated in full -- nothing is cached or skipped.  Under
    torch.distributed the gradient all-reduce is part of each slot's graph (GraphedStep.allreduce).

        tr = PipelinedTrainer(module, example_xyz, example_mask, example_features, grad_out)
        for host_batch in loader:            # pinned host tensors
            prev_loss = tr.step(host_batch)  # returns the result of the PREVIOUS step (None on the first)
        last = tr.flush()
    """

    def __init__(self, module, xyz, mask, features, grad_out, after_step=None):
        # each slot owns the gradient tensors its graph writes (slot.param_grads / slot.flat_grad / slot.grads());
        # module.parameters()[i].grad only aliases the LAST captured slot, so after_step must read the slot's own
        self.slots = [GraphedStep(module, xyz, mask, features, grad_out) for _ in range(2)]
        # high priority: its own hardware queue, so the H2D copies are never ordered behind the replay's kernels
        self.copy = torch.cuda.Stream(priority=-1)
        self.after_step = after_step            # after_step(slot): e.g. the optimizer step on slot.grads()
        nr = self.slots[0].result.numel()
        # per step the host receives the step's scalar result and the (reduced) parameter gradients
        self.result_host = [torch.zeros(nr, dtype=torch.float32).pin_memory() for _ in range(2)]
        self.d2h_bytes = 4 * nr
        self.done = [torch.cuda.Event(), torch.cuda.Event()]     # replay i finished (its buffers are free again)
        self.loaded = [torch.cuda.Event(), torch.cuda.Event()]   # inputs of slot i are on the device
        self.i = 0
        self.pending = None
        for e in self.done:
            e.record()

    def _issue_copy(self, slot, batch):
        s = self.slots[slot]
        self.copy.wait_event(self.done[slot])   # the previous replay on this slot no longer reads its inputs
        with torch.cuda.stream(self.copy):
            s.load(batch["xyz"], batch["mask"], batch["features"], non_blocking=True)
            self.loaded[slot].record(self.copy)

    def step(self, batch):
        slot = self.i & 1
        cur = torch.cuda.current_stream()
        self._issue_copy(slot, batch)
        cur.wait_event(self.loaded[slot])
        self.slots[slot].replay()
        if self.after_step is not None:
            self.after_step(self.slots[slot])
        self.result_host[slot].copy_(self.slots[slot].result, non_blocking=True)  # D2H: result + parameter gradients
        self.done[slot].record(cur)
        prev = None
        if self.pending is not None:
            pslot = self.pending
            self.done[pslot].synchronize()
            prev = float(self.result_host[pslot][0])
        self.pending = slot
        self.i += 1
        return prev

    def flush(self):
        if self.pending is None:
            return None
        self.done[self.pending].synchronize()
        v = float(self.result_host[self.pending][0])
        self.pending = None
        return v
