"""Batch-sharded data parallelism for the density pass (the reference has none; SURVEY 8e).

Every op on the path is per-sample, parameters are replicated, so the batch shards across ranks with
no data-path collective; `forward_kld` needs exactly one all-reduce of (sum log_q, count)."""
import torch
import torch.distributed as dist


def shard_rows(n_rows, rank, world_size):
    """Contiguous row range [lo, hi) of rank `rank`; remainders go to the first ranks."""
    base, rem = divmod(n_rows, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def all_reduce_kld(local_sum, local_count, group=None):
    """-(sum_r local_sum_r) / (sum_r local_count_r) with ONE collective on a 2-element fp64 tensor.
    local_sum: 0-dim tensor (sum of log_q over the local shard)."""
    buf = torch.stack([local_sum.to(torch.float64).reshape(()),
                       torch.full((), float(local_count), dtype=torch.float64, device=local_sum.device)])
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    return -(buf[0] / buf[1])


class _PendingLoss:
    """Result of an asynchronous data-parallel forward_kld: `.result()` makes the current stream wait for
    the collective and returns the 0-dim fp32 loss."""

    def __init__(self, buf, work):
        self._buf, self._work, self._val = buf, work, None

    def result(self):
        if self._val is None:
            if self._work is not None:
                self._work.wait()
            self._val = (-(self._buf[0] / self._buf[1])).to(torch.float32)
        return self._val


def forward_kld_dp(model, x_local, group=None, async_op=False):
    """Global forward KL over all ranks' shards: each rank runs the fused stack on its rows; the reduction
    kernel writes the rank's sum(log_q) straight into a 2-element fp64 buffer [sum, count] which is the
    operand of the ONE NCCL all-reduce.  No other device work, no host sync.

    async_op=True returns a handle instead of the tensor: the compute stream does not wait for the
    collective, so the next step's kernels are not serialised behind a 16-byte all-reduce (the buffers
    rotate through a ring of 8, the oldest is waited on before reuse)."""
    h = model._stack()
    if h is None or h.base is None:
        raise NotImplementedError("forward_kld_dp needs an all-native stack with a DiagGaussian or GaussianMixture base")
    ring = model.__dict__.get("_nfb_dp_ring")
    if ring is None or ring["bufs"][0].device != x_local.device:
        ring = {"bufs": [torch.zeros(2, dtype=torch.float64, device=x_local.device) for _ in range(8)],
                "pending": [None] * 8, "i": 0}
        model.__dict__["_nfb_dp_ring"] = ring
    i = ring["i"]
    ring["i"] = (i + 1) % 8
    if ring["pending"][i] is not None:
        ring["pending"][i].result()
        ring["pending"][i] = None
    buf = ring["bufs"][i]
    h.forward_kld(x_local, sum_out=buf)  # the reduction kernel writes [sum(log_q), rows]
    work = None
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        work = dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
        if not async_op:
            work = None
    pend = _PendingLoss(buf, work)
    if async_op:
        ring["pending"][i] = pend
        return pend
    return pend.result()


class GradientBuckets:
    """DDP-style gradient averaging for the training step (SURVEY 8e/8f-1): parameters are replicated, every
    rank back-propagates its shard of the batch, then the gradients are summed across ranks and divided by the
    GLOBAL row count (the loss is a mean over all rows, so ranks with ragged shards weight correctly when each
    rank's loss was taken over its local rows: g = sum_r n_r g_r / sum_r n_r).

    Gradients are packed into a few flat buffers (default 32 MB each: NVSwitch all-reduce cost is launch latency,
    not link count, so buckets are sized for few launches) and reduced with one collective per bucket, issued
    asynchronously in reverse parameter order (the order autograd finishes them); `finish()` waits and scatters
    the averages back into `.grad`.  Plain torch.distributed: NCCL on GPUs, gloo in the CPU tests."""

    def __init__(self, params, bucket_bytes=32 << 20, group=None):
        self.params = [p for p in params if p.requires_grad]
        self.group = group
        self.buckets, cur, size = [], [], 0
        for p in reversed(self.params):
            nbytes = p.numel() * p.element_size()
            if cur and (size + nbytes > bucket_bytes or p.dtype != cur[0].dtype or p.device != cur[0].device):
                self.buckets.append(cur)
                cur, size = [], 0
            cur.append(p)
            size += nbytes
        if cur:
            self.buckets.append(cur)
        self._flat = [None] * len(self.buckets)
        self._work = []

    def start(self, local_rows):
        """Launch the collectives.  `local_rows`: rows this rank's (mean) loss was computed over."""
        world = dist.get_world_size(self.group) if dist.is_available() and dist.is_initialized() else 1
        self._work = []
        self._rows = None
        if world == 1:
            return self
        first = self.buckets[0][0]
        self._rows = torch.tensor([float(local_rows)], dtype=torch.float64, device=first.device)
        for i, bucket in enumerate(self.buckets):
            n = sum(p.numel() for p in bucket)
            flat = self._flat[i]
            if flat is None or flat.numel() != n or flat.device != bucket[0].device or flat.dtype != bucket[0].dtype:
                flat = torch.empty(n, dtype=bucket[0].dtype, device=bucket[0].device)
                self._flat[i] = flat
            off = 0
            for p in bucket:
                g = p.grad if p.grad is not None else torch.zeros_like(p)
                flat[off:off + p.numel()].copy_(g.reshape(-1))
                off += p.numel()
            flat.mul_(float(local_rows))  # n_r g_r
            self._work.append(dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group, async_op=True))
        self._work.append(dist.all_reduce(self._rows, op=dist.ReduceOp.SUM, group=self.group, async_op=True))
        return self

    def finish(self):
        if not self._work:
            return
        for w in self._work:
            w.wait()
        total = float(self._rows.item())
        for flat, bucket in zip(self._flat, self.buckets):
            flat.div_(total)
            off = 0
            for p in bucket:
                g = flat[off:off + p.numel()].view_as(p)
                if p.grad is None:
                    p.grad = g.clone()
                else:
                    p.grad.copy_(g)
                off += p.numel()
        self._work = []
