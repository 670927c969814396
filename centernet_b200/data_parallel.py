"""Training-side data parallelism (SURVEY 8e / row E2): one process per GPU, replicas hold full weights, and the
ONLY exchange per step is a bucketed NCCL all-reduce of the gradients over NVLink 4 / NVSwitch, launched from
autograd hooks while the rest of the backward is still running.

Replaces src/lib/models/data_parallel.py (single process, scatter -> replicate -> parallel_apply -> gather, the
gradient reduce-to-GPU0 hidden in `replicate`'s autograd) as used by trains/base_trainer.py:31-35:

    model_with_loss = DataParallel(model_with_loss, device_ids=gpus, chunk_sizes=chunk_sizes).to(device)
    output, loss, loss_stats = model_with_loss(batch); loss = loss.mean(); loss.backward(); optimizer.step()

Under `torchrun` (torch.distributed initialised) `DataParallel(...)` here returns a `ShardedDataParallel`: the
call site stays the same, every rank takes ITS chunk of the batch (`chunk_sizes`, opts.py:260-269 -- the first
GPU may get a smaller one), computes its own loss with its own focal normaliser `num_pos` (no cross-GPU
reduction, exactly as the reference where the loss lives inside the replicated module,
base_trainer.py:12-21) and the gradients come out as the MEAN over ranks -- what `loss.mean()` over the gathered
per-replica losses gives the reference.  Without torch.distributed it falls back to torch.nn.DataParallel.
"""
import torch
import torch.distributed as dist
from torch import nn


class GradientAllReducer(object):
    """Flat gradient buckets + overlapped all-reduce.

    Parameters are packed, in REVERSE registration order (gradients arrive roughly last layer first), into
    buckets of about `bucket_mb`; every `param.grad` is a view into its bucket's flat buffer, so nothing is
    copied.  A post-accumulate hook counts the gradients of a bucket and launches `all_reduce(async_op=True)`
    the moment the last one has landed; the collective runs on NCCL's stream under the remaining backward.
    `finish()` (queued automatically at the end of every backward) waits for the handles; the division by the
    world size is folded into the reduce (`ReduceOp.AVG` on NCCL, pre-scaled SUM elsewhere)."""

    def __init__(self, params, bucket_mb=25.0, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.params = [p for p in params if p.requires_grad]
        self.buckets = []          # dicts: flat, params, pending, handle
        self._of = {}
        cap = int(bucket_mb * 1024 * 1024)
        cur, cur_bytes = [], 0
        for p in reversed(self.params):
            nb = p.numel() * p.element_size()
            if cur and (cur_bytes + nb > cap or p.dtype != cur[0].dtype or p.device != cur[0].device):
                self._make_bucket(cur)
                cur, cur_bytes = [], 0
            cur.append(p)
            cur_bytes += nb
        if cur:
            self._make_bucket(cur)
        self._queued = False
        self._hooks = [p.register_post_accumulate_grad_hook(self._on_grad) for p in self.params]
        self.use_avg = dist.is_initialized() and dist.get_backend(group) == "nccl"

    def _make_bucket(self, plist):
        n = sum(p.numel() for p in plist)
        flat = torch.zeros(n, dtype=plist[0].dtype, device=plist[0].device)
        off = 0
        for p in plist:
            view = flat[off:off + p.numel()].view_as(p)
            if p.grad is not None:
                view.copy_(p.grad)
            p.grad = view                      # autograd accumulates in place into the bucket
            off += p.numel()
        b = {"flat": flat, "params": plist, "pending": len(plist), "handle": None}
        for p in plist:
            self._of[p] = b
        self.buckets.append(b)

    @property
    def nbytes(self):
        return sum(b["flat"].numel() * b["flat"].element_size() for b in self.buckets)

    def _on_grad(self, p):
        b = self._of[p]
        if p.grad.data_ptr() != b["flat"].data_ptr() + self._offset(b, p):
            # somebody replaced .grad (optimizer.zero_grad(set_to_none=True) + a fresh tensor): re-attach
            view = self._view(b, p)
            view.copy_(p.grad)
            p.grad = view
        b["pending"] -= 1
        if b["pending"] == 0:
            self._launch(b)
        if not self._queued:
            self._queued = True
            torch.autograd.Variable._execution_engine.queue_callback(self.finish)

    def _offset(self, b, p):
        off = 0
        for q in b["params"]:
            if q is p:
                return off * p.element_size()
            off += q.numel()
        raise KeyError

    def _view(self, b, p):
        off = self._offset(b, p) // p.element_size()
        return b["flat"][off:off + p.numel()].view_as(p)

    def _launch(self, b):
        if self.world == 1:
            return
        if self.use_avg:
            b["handle"] = dist.all_reduce(b["flat"], op=dist.ReduceOp.AVG, group=self.group, async_op=True)
        else:
            b["flat"].div_(self.world)
            b["handle"] = dist.all_reduce(b["flat"], op=dist.ReduceOp.SUM, group=self.group, async_op=True)

    def finish(self):
        """Waits for every outstanding bucket; buckets whose parameters got no gradient this step (unused
        heads) are reduced here so that all ranks issue the same collectives."""
        for b in self.buckets:
            if b["handle"] is None and b["pending"] != 0 and self.world > 1:
                self._launch(b)
        for b in self.buckets:
            if b["handle"] is not None:
                b["handle"].wait()
                b["handle"] = None
            b["pending"] = len(b["params"])
        self._queued = False

    def zero_grad(self):
        """Keeps the bucket views (use instead of optimizer.zero_grad(set_to_none=True))."""
        for b in self.buckets:
            b["flat"].zero_()

    def remove(self):
        for h in self._hooks:
            h.remove()


def _slice_batch(batch, lo, hi):
    if isinstance(batch, torch.Tensor):
        return batch[lo:hi]
    if isinstance(batch, dict):
        return {k: (v if k == "meta" else _slice_batch(v, lo, hi)) for k, v in batch.items()}
    if isinstance(batch, (list, tuple)):
        return type(batch)(_slice_batch(v, lo, hi) for v in batch)
    return batch


class ShardedDataParallel(nn.Module):
    """One replica of a one-process-per-GPU data-parallel job behind the reference's DataParallel call shape:
    forward(batch) runs `module` on THIS rank's chunk of `batch`; backward all-reduces (averages) the gradients."""

    def __init__(self, module, chunk_sizes=None, bucket_mb=25.0, group=None, scatter=True):
        super().__init__()
        self.module = module
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.chunk_sizes = list(chunk_sizes) if chunk_sizes is not None else None
        self.scatter = scatter          # False: the loader already yields per-rank shards
        for p in module.parameters():   # replicas start identical (replicate() broadcasts from GPU 0 in the reference)
            dist.broadcast(p.data, src=0, group=group)
        for bf in module.buffers():
            dist.broadcast(bf.data, src=0, group=group)
        self.reducer = GradientAllReducer(module.parameters(), bucket_mb=bucket_mb, group=group)

    def _bounds(self, n):
        if self.chunk_sizes is not None and len(self.chunk_sizes) == self.world and sum(self.chunk_sizes) == n:
            lo = sum(self.chunk_sizes[:self.rank])
            return lo, lo + self.chunk_sizes[self.rank]
        per = (n + self.world - 1) // self.world          # torch scatter: ceil-sized chunks
        return min(n, per * self.rank), min(n, per * (self.rank + 1))

    def forward(self, *inputs, **kwargs):
        if self.scatter and inputs:
            first = inputs[0]
            probe = first
            while isinstance(probe, dict):
                probe = next(v for k, v in probe.items() if k != "meta" and isinstance(v, (torch.Tensor, dict)))
            lo, hi = self._bounds(int(probe.shape[0]))
            inputs = tuple(_slice_batch(x, lo, hi) for x in inputs)
        return self.module(*inputs, **kwargs)

    def zero_grad(self, set_to_none=False):
        self.reducer.zero_grad()


def DataParallel(module, device_ids=None, output_device=None, dim=0, chunk_sizes=None):
    """Same signature as src/lib/models/data_parallel.py:119-128."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return ShardedDataParallel(module, chunk_sizes=chunk_sizes)
    return torch.nn.DataParallel(module, device_ids, output_device, dim)
