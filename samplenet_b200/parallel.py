"""Batch-sharded data parallelism for SampleNet training on one multi-GPU node (SURVEY.md 8e).

The reference has no distributed code (every trainer pins one device, main.py:88).  Clouds are independent through
generator, projection, Chamfer and EMD, so the only cross-rank traffic of a training step is the gradient average of the
trainable parameters: ~250 k floats (1 MB) when only SampleNet trains (main.py:256-258).  At 1 MB an all-reduce over
NVLink 5 / NVSwitch is latency-bound, so the right shape is ONE collective per step over ONE flat bucket -- not DDP's
25 MB bucket heuristics, and not one collective per parameter:

  * all trainable parameters' `.grad` tensors are VIEWS into a single flat fp32 buffer (autograd accumulates in place);
  * `sync_gradients()` issues one `all_reduce(SUM)` on a side stream as soon as it is called after backward, then scales by
    1/world; `wait()` joins the streams before the optimizer step;
  * BatchNorm statistics stay per replica (standard DDP semantics; equals the reference at 32 clouds per GPU).

Forward + loss alone (the headline metric) need no collective at all: ranks are independent replicas.
Works with the `nccl` backend on GPUs and with `gloo` on CPU (the unit tests run it with world_size 2 on CPU).
"""
import torch
import torch.distributed as dist


class FlatBucketDataParallel(torch.nn.Module):
    def __init__(self, module, process_group=None, broadcast_from=0):
        super().__init__()
        self.module = module
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        params = [p for p in module.parameters() if p.requires_grad]
        if not params:
            raise ValueError("FlatBucketDataParallel: module has no trainable parameters")
        dev, dt = params[0].device, params[0].dtype
        if any(p.device != dev or p.dtype != dt for p in params):
            raise ValueError("FlatBucketDataParallel: parameters must share one device and dtype")
        self._params = params
        self.flat_grad = torch.zeros(sum(p.numel() for p in params), device=dev, dtype=dt)
        off = 0
        for p in params:
            n = p.numel()
            p.grad = self.flat_grad[off:off + n].view_as(p)  # autograd accumulates into the bucket in place
            off += n
        self._stream = torch.cuda.Stream(device=dev) if dev.type == "cuda" else None
        self._work = None
        # replicas start identical (parameters AND buffers, e.g. BatchNorm running statistics)
        if self.world > 1:
            with torch.no_grad():
                for t in list(module.parameters()) + list(module.buffers()):
                    dist.broadcast(t.data, src=broadcast_from, group=self.group)

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def zero_grad(self, set_to_none=False):  # keep the views: never set grads to None
        self.flat_grad.zero_()

    def bucket_bytes(self):
        return self.flat_grad.numel() * self.flat_grad.element_size()

    def sync_gradients(self):
        """One all-reduce over the flat bucket (async on a side stream for CUDA).  Call after backward()."""
        if self.world == 1:
            return
        for p in self._params:  # a parameter whose grad was replaced (e.g. by zero_grad(set_to_none=True)) would escape the bucket
            if p.grad is None or p.grad.data_ptr() < self.flat_grad.data_ptr() or \
                    p.grad.data_ptr() >= self.flat_grad.data_ptr() + self.bucket_bytes():
                raise RuntimeError("FlatBucketDataParallel: a parameter's .grad is no longer a view of the flat bucket "
                                   "(use wrapper.zero_grad(), not optimizer.zero_grad(set_to_none=True))")
        if self._stream is not None:
            self._stream.wait_stream(torch.cuda.current_stream(self.flat_grad.device))
            with torch.cuda.stream(self._stream):
                dist.all_reduce(self.flat_grad, op=dist.ReduceOp.SUM, group=self.group)
                self.flat_grad.mul_(1.0 / self.world)
        else:
            dist.all_reduce(self.flat_grad, op=dist.ReduceOp.SUM, group=self.group)
            self.flat_grad.mul_(1.0 / self.world)

    def wait(self):
        """Join the side stream (call before optimizer.step())."""
        if self._stream is not None and self.world > 1:
            torch.cuda.current_stream(self.flat_grad.device).wait_stream(self._stream)


def shard_batch(x, rank, world):
    """Contiguous batch shard of rank `rank` (global batch must divide evenly, as in the reference's fixed batch sizes)."""
    if x.shape[0] % world != 0:
        raise ValueError("global batch %d is not divisible by world size %d" % (x.shape[0], world))
    per = x.shape[0] // world
    return x[rank * per:(rank + 1) * per]
