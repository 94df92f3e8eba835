"""Data-parallel plumbing: the one collective on the hot path is the gradient all-reduce (mean) the reference gets
from apex DistributedDataParallel (structure/model.py:27-34; per-rank batch = global / world,
data/data_loader.py:40-43).  One flat bucket (33 MB for CRNN) over NCCL / NVLink; CUDA-graph capturable."""
import torch
import torch.distributed as dist
from torch._utils import _flatten_dense_tensors, _unflatten_dense_tensors


def shard_range(n_items, rank, world):
    """[lo, hi) of this rank's slice of a global batch (reference: batch_size // world per rank)."""
    per = n_items // world
    return rank * per, (rank + 1) * per


def allreduce_mean_grads_(params, group=None):
    """In place: p.grad <- mean over ranks of p.grad, for every parameter that has a gradient."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return
    flat = _flatten_dense_tensors(grads)
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    flat.div_(dist.get_world_size(group))
    for g, s in zip(grads, _unflatten_dense_tensors(flat, grads)):
        g.copy_(s)


class FlatGrads:
    """The gradients of `params` as views into ONE flat fp32 buffer, in the given order (pass the parameters in backward order --
    decoder first -- and `buckets` > 1 to let the early buckets' all-reduce run while the rest of the backward is still computing).

    Flattening, reducing, dividing and copying back every step costs ~40 un-captured launches between two CUDA graphs, far
    more than the 33 MB transfer itself.  Here autograd
    accumulates straight into the views (`zero()` is one memset and keeps them attached), the collective is ONE in-place NCCL
    all-reduce with the AVG op (no separate divide) per bucket, and the optimizer reads the same views: no copies at all."""

    def __init__(self, params, buckets=1):
        self.params = [p for p in params if p.requires_grad]
        assert self.params and all(p.dtype == torch.float32 for p in self.params)
        dev = self.params[0].device
        n = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        self.spans = []
        o = 0
        for p in self.params:
            p.grad = self.flat[o:o + p.numel()].view_as(p)
            self.spans.append((o, o + p.numel()))
            o += p.numel()
        # bucket boundaries on parameter boundaries, roughly equal sizes
        buckets = max(1, min(buckets, len(self.params)))
        self.bounds = [0]
        for b in range(1, buckets):
            target = n * b // buckets
            cut = min((e for (_, e) in self.spans), key=lambda e: abs(e - target))
            if cut > self.bounds[-1]:
                self.bounds.append(cut)
        self.bounds.append(n)

    def zero(self):
        self.flat.zero_()

    def attached(self):
        """True while every parameter's .grad is still the view handed out (zero_grad(set_to_none=True) would detach them)."""
        return all(p.grad is not None and p.grad.data_ptr() == self.flat.data_ptr() + 4 * lo
                   for p, (lo, _) in zip(self.params, self.spans))

    def n_buckets(self):
        return len(self.bounds) - 1

    def bucket(self, i):
        return self.flat[self.bounds[i]:self.bounds[i + 1]]

    def allreduce_bucket_(self, i, group=None):
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            t = self.bucket(i)
            if dist.get_backend(group) == "nccl":
                dist.all_reduce(t, op=dist.ReduceOp.AVG, group=group)
            else:                                   # gloo (CPU tests) has no AVG
                dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
                t.div_(dist.get_world_size(group))

    def allreduce_(self, group=None):
        for i in range(self.n_buckets()):
            self.allreduce_bucket_(i, group)
