"""CUDA-graph capture of a whole SampleNet step.

At the headline size (B=32, N=1024->64) the step is ~a dozen kernels of a few microseconds each; launched one by one from
Python the host is the bottleneck.  `GraphedStep` captures `net(x)` + `net.get_simplification_loss(...)` once into a CUDA
graph over static buffers and replays it: one host call per step.  This is the native replacement for what a tracing
compiler would do, and it is part of the public API:

    step = GraphedStep(net, batch_size=32, num_points=1024)            # forward + loss (no grad)
    simp, proj, loss = step(x_cuda)                                    # x already in HBM
    loss_host = step.run_from_host(x_pinned)                           # H2D copy + replay + D2H of the loss, synchronised
"""
import os

import torch

from . import _lib, ops


def _snapshot(module):
    """Clones of every parameter and buffer (BatchNorm running statistics, num_batches_tracked): graph construction runs real warm-up
    executions of the step on a placeholder batch, which must not leave a trace in the model."""
    return {k: v.detach().clone() for k, v in module.state_dict().items()}


def _restore(module, snap):
    with torch.no_grad():
        for k, v in module.state_dict().items():
            v.copy_(snap[k])           # in place: captured graphs keep pointing at the same storage


def _snapshot_optimizer(opt):
    return {p: {k: v.detach().clone() if torch.is_tensor(v) else v for k, v in st.items()} for p, st in opt.state.items()}


def _restore_optimizer(opt, snap):
    """In place, so that a captured graph keeps pointing at the same storage.  State the warm-up created (a parameter's first step) is
    zeroed, which is the state that first step creates for the ZERO_INIT_OPTIMIZERS only (check_capturable refuses the others)."""
    with torch.no_grad():
        for p, st in opt.state.items():
            old = snap.get(p)
            for k, v in st.items():
                if not torch.is_tensor(v):
                    if old is not None and k in old:
                        st[k] = old[k]
                elif old is None or k not in old:
                    v.zero_()
                else:
                    v.copy_(old[k])


# Optimizers whose lazily created per-parameter state is all zeros (step and every moment buffer), so that zeroing what a warm-up step
# created gives back the state before it.  Others are refused: NAdam creates mu_product = 1, ASGD eta = lr and mu = 1, and zeroing those
# would change every later step.  Exact classes: a subclass may create other state.
ZERO_INIT_OPTIMIZERS = (torch.optim.Adam, torch.optim.AdamW, torch.optim.Adamax, torch.optim.RAdam, torch.optim.RMSprop, torch.optim.Adadelta)


def check_capturable(optimizer, who):
    """ValueError unless `optimizer` can be captured and its warm-up undone: one of ZERO_INIT_OPTIMIZERS with capturable=True on every
    parameter group (a captured optimizer step keeps its step count on the device)."""
    names = ", ".join("torch.optim." + c.__name__ for c in ZERO_INIT_OPTIMIZERS)
    if type(optimizer) not in ZERO_INIT_OPTIMIZERS:
        raise ValueError("%s needs one of %s, constructed with capturable=True: it captures the optimizer step and undoes its "
                         "warm-up by zeroing the state that step created, which is the fresh state of those only; got %s"
                         % (who, names, type(optimizer).__name__))
    if not all(g.get("capturable", False) for g in optimizer.param_groups):
        raise ValueError("%s replays the optimizer step in a CUDA graph: construct the optimizer with capturable=True "
                         "(e.g. torch.optim.Adam(params, lr, capturable=True))" % who)


class CapturedStep:
    """One training step captured into a CUDA graph, with no trace of the capture left behind.

        cap = CapturedStep(body, modules, optimizer, counters=(runner, ("step", "epoch")), state=[accumulator])
        cap.replay()                    # one graph launch; cap.outputs is what body() returned at capture (static buffers)

    Construction snapshots every parameter and buffer of `modules`, the optimizer's state, the CUDA RNG state of the device, the named
    counters of `counters[0]` and the tensors in `state`; runs `warmup` real executions of body() on a side stream (they create the
    optimizer state, the autograd buffers and every kernel's one-time set-up); restores all of the above in place; then captures body()
    once.  The graph owns its own ops.PrimedWorkspaces, active around every execution of body(): the persistent generator scratch and the
    ticket word of the last-CTA reductions, so graphs replayed on different streams never share one.  The caller keeps body()'s inputs in
    static buffers and replays on its current stream.  `optimizer` must pass check_capturable."""

    def __init__(self, body, modules, optimizer=None, counters=None, state=(), device=None, warmup=3):
        if optimizer is not None:
            check_capturable(optimizer, type(self).__name__)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        self.workspaces = ops.PrimedWorkspaces()
        pw = self.workspaces

        def run():
            with ops.primed_workspaces(pw):
                return body()

        owner, names = counters if counters is not None else (None, ())
        self.stream = torch.cuda.Stream(device=dev)
        with torch.cuda.device(dev):
            snaps = [_snapshot(m) for m in modules]
            opt_snap = _snapshot_optimizer(optimizer) if optimizer is not None else None
            state_snap = [t.detach().clone() for t in state]
            rng = torch.cuda.get_rng_state(dev)
            counts = [getattr(owner, n) for n in names]
            self.stream.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(self.stream):
                for _ in range(warmup):
                    run()
                for m, s in zip(modules, snaps):
                    _restore(m, s)
                if optimizer is not None:
                    _restore_optimizer(optimizer, opt_snap)
                with torch.no_grad():
                    for t, s in zip(state, state_snap):
                        t.copy_(s)
            self.stream.synchronize()
            torch.cuda.set_rng_state(rng, dev)
            for n, v in zip(names, counts):
                setattr(owner, n, v)
            before = _lib.launch_count()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self.stream):
                self.outputs = run()
            self.launches_per_step = _lib.launch_count() - before

    def replay(self):
        self.graph.replay()


class PipelinedHostStep:
    """End-to-end streaming of host batches through two `GraphedStep`s (double buffering): the pinned host batch of a later step
    crosses PCIe on a copy stream while an earlier step computes, and up to two steps are in flight so the GPU always has the next
    graph queued while the host reads the previous loss.  Every step still ends with its loss on the host.

        pipe = PipelinedHostStep(net, 32, 1024)
        pipe.submit(batch0); pipe.launch()                 # step 0 in flight
        pipe.submit(batch1); pipe.launch()                 # step 1 queued behind it
        for i in range(2, steps):
            loss = pipe.finish()                           # loss of the oldest step in flight, on the host
            pipe.submit(batch_i); pipe.launch()            # its buffers are free again: refill and queue
        pipe.finish(); pipe.finish()
    """

    def __init__(self, net, batch_size, num_points, gamma=1, delta=0, device=None, side_readback=True):
        # side_readback: the 4-byte loss read-back runs on its own stream behind the graph instead of being the graph's last node, so the next
        # step's kernels (the other slot's graph, already queued) do not wait for a PCIe round trip between two steps
        self.side_readback = bool(side_readback)
        self.slots = [GraphedStep(net, batch_size, num_points, gamma, delta, device, loss_to_host=not self.side_readback) for _ in range(2)]
        self.device = self.slots[0].device
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self.d2h_stream = torch.cuda.Stream(device=self.device)
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]      # input of the slot has arrived
        self.computed = [torch.cuda.Event(), torch.cuda.Event()]   # the slot's graph has finished (side_readback)
        self.done = [torch.cuda.Event(), torch.cuda.Event()]       # graph + loss read-back of the slot have finished
        self.head = 0          # next slot to fill
        self.next_launch = 0   # next slot to launch
        self.submitted = []    # slots filled but not launched
        self.inflight = []     # slots launched but not finished (oldest first)
        self.launches_per_step = self.slots[0].launches_per_step
        for e in self.done:
            e.record(torch.cuda.current_stream(self.device))

    def submit(self, x_pinned):
        k = self.head
        if k in self.submitted or k in self.inflight:
            raise RuntimeError("PipelinedHostStep: both buffers are busy; call finish() first")
        self.copy_stream.wait_event(self.done[k])              # the graph that last read this buffer has finished (device-side wait)
        with torch.cuda.stream(self.copy_stream):
            self.slots[k].x.copy_(x_pinned, non_blocking=True)
            self.ready[k].record(self.copy_stream)
        self.submitted.append(k)
        self.head ^= 1

    def launch(self):
        """Enqueue the oldest submitted batch: graph replay + loss read-back (asynchronous)."""
        if not self.submitted:
            raise RuntimeError("PipelinedHostStep: nothing submitted")
        k = self.submitted.pop(0)
        st = torch.cuda.current_stream(self.device)
        st.wait_event(self.ready[k])
        g = self.slots[k]
        g.replay()
        if self.side_readback:
            self.computed[k].record(st)
            self.d2h_stream.wait_event(self.computed[k])
            with torch.cuda.stream(self.d2h_stream), torch.no_grad():
                g.loss_host.copy_(g.loss_flat, non_blocking=True)
                self.done[k].record(self.d2h_stream)
        else:                                                 # (the read-back into g.loss_host is the graph's last node)
            self.done[k].record(st)
        self.inflight.append(k)

    def finish(self):
        """Wait for the oldest step in flight and return its loss (host float)."""
        if not self.inflight:
            raise RuntimeError("PipelinedHostStep: nothing in flight")
        k = self.inflight.pop(0)
        self.done[k].synchronize()
        return float(self.slots[k].loss_host[0])

    def step(self):
        self.launch()
        return self.finish()

    def run_async(self, x):
        """Device-ordered variant for inputs that already live in HBM (or pinned host memory) when NO per-step host read-back is wanted:
        the batch is copied into the idle slot's capture buffer on the copy stream -- overlapping the other slot's graph, which is still
        running -- and that slot's graph is queued behind the copy.  Returns the slot (its static `simp`, `proj`, `loss` tensors are valid
        once the current stream reaches this point).  Do not mix with submit()/launch()/finish() on the same object."""
        k = self.head
        st = torch.cuda.current_stream(self.device)
        self.copy_stream.wait_event(self.done[k])              # the graph that last read this buffer has finished
        with torch.cuda.stream(self.copy_stream):
            self.slots[k].x.copy_(x, non_blocking=True)
            self.ready[k].record(self.copy_stream)
        st.wait_event(self.ready[k])
        self.slots[k].replay()
        self.done[k].record(st)
        self.head ^= 1
        return self.slots[k]


class GraphedStep:
    def __init__(self, net, batch_size, num_points, gamma=1, delta=0, device=None, warmup=2, loss_to_host=False):
        self.net = net
        self.loss_to_host = bool(loss_to_host)   # make the 4-byte loss read-back into pinned memory a node of the graph
        dev = torch.device(device) if device is not None else next(net.parameters()).device
        self.device = dev
        shape = (batch_size, num_points, 3) if net.input_shape == "bnc" else (batch_size, 3, num_points)
        self.x = torch.zeros(shape, device=dev)
        self.loss_host = torch.zeros(1).pin_memory()
        self.stream = torch.cuda.Stream(device=dev)
        m = net.num_out_points

        self._pw = ops.PrimedWorkspaces()   # this step's persistent generator scratch: no memset node in front of the kernel

        def body():
            with ops.primed_workspaces(self._pw):
                simp, proj = net(self.x)
            ref_bnc = self.x if net.input_shape == "bnc" else self.x.permute(0, 2, 1).contiguous()
            simp_bnc = simp if net.output_shape == "bnc" else simp.permute(0, 2, 1).contiguous()
            loss = net.get_simplification_loss(ref_bnc, simp_bnc, m, gamma, delta)
            return simp, proj, loss

        with torch.cuda.device(dev), torch.no_grad():
            snap = _snapshot(net)          # warm-up forwards in train mode would move the BatchNorm running statistics
            self.stream.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(self.stream):
                for _ in range(warmup):
                    body()
                _restore(net, snap)
            self.stream.synchronize()
            before = _lib.launch_count()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self.stream):
                self.simp, self.proj, self.loss = body()
                self.loss_flat = self.loss.reshape(1)
                if self.loss_to_host:
                    self.loss_host.copy_(self.loss_flat, non_blocking=True)     # the loss read-back is a node of the graph
            self.launches_per_step = _lib.launch_count() - before
        # SNB200_NO_GRAPH=1: launch the same kernels one by one instead of replaying the graph -- for profilers only (ncu cannot
        # attribute a cooperative launch inside a graph); results land in the same static buffers
        self._body = body
        self.eager = os.environ.get("SNB200_NO_GRAPH") == "1"

    def replay(self):
        if not self.eager:
            self.graph.replay()
            return
        with torch.no_grad():
            simp, proj, loss = self._body()
            self.simp.copy_(simp); self.proj.copy_(proj); self.loss.copy_(loss)
            if self.loss_to_host:
                self.loss_host.copy_(self.loss_flat, non_blocking=True)

    def __call__(self, x):
        """x: CUDA tensor shaped like the capture buffer (copied device-to-device), returns the static outputs."""
        self.x.copy_(x, non_blocking=True)
        self.replay()
        return self.simp, self.proj, self.loss

    def run_from_host(self, x_pinned):
        """End-to-end step: pinned host batch -> device, replay, loss back to the host (synchronised); returns float."""
        self.x.copy_(x_pinned, non_blocking=True)
        self.replay()
        if not self.loss_to_host:
            self.loss_host.copy_(self.loss_flat, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return float(self.loss_host[0])


class GraphedTrainStep:
    """One whole TRAINING step -- forward, simplification + projection loss, backward, ONE flat-bucket gradient all-reduce (when a
    process group is initialised) and the Adam update -- captured in a CUDA graph and replayed with one host call.

        step = GraphedTrainStep(net, batch_size=32, num_points=1024, lr=1e-3)      # net: SampleNet, "bnc" in/out, training mode
        loss = step(x_cuda)                                                          # 0-dim CUDA tensor (static buffer)

    The eager training step is ~120 small launches (the generator's backward recomputes through torch ops) and is bound by host
    launch overhead; the graph removes that.  The optimizer is `torch.optim.Adam(..., capturable=True)`; extra loss terms can be
    supplied as `extra_loss(simp, proj) -> scalar` (e.g. the task network's loss in the reference trainers)."""

    def __init__(self, net, batch_size, num_points, lr=1e-3, gamma=1, delta=0, alpha=0.01, lmbda=0.01, extra_loss=None, device=None, warmup=3):
        from .parallel import FlatBucketDataParallel

        dev = torch.device(device) if device is not None else next(net.parameters()).device
        self.net, self.device = net, dev
        if net.input_shape != "bnc" or net.output_shape != "bnc":
            raise ValueError("GraphedTrainStep expects a SampleNet with input_shape = output_shape = 'bnc'")
        self.ddp = FlatBucketDataParallel(net)
        params = [p for p in net.parameters() if p.requires_grad]
        # one fused multi-tensor Adam launch (torch's fused optimizer is capturable); gradients are written by the backward kernels straight
        # into the flat bucket's views (no per-parameter accumulate / zero-fill launches)
        self.optimizer = torch.optim.Adam(params, lr=lr, fused=True, capturable=True)
        net.direct_parameter_grads = True     # (one sampler forward per captured step)
        self.x = torch.zeros(batch_size, num_points, 3, device=dev)
        m = net.num_out_points

        def body():
            self.ddp.zero_grad()
            simp, proj = self.ddp(self.x)
            loss = alpha * net.get_simplification_loss(self.x, simp, m, gamma, delta) + lmbda * net.get_projection_loss()
            if extra_loss is not None:
                loss = loss + extra_loss(simp, proj)
            else:
                loss = loss + (proj * proj).mean() * 0.0 + proj.sum() * 0.0   # keeps the projection (and its backward) in the step
            loss.backward()
            self.ddp.sync_gradients()
            self.ddp.wait()
            self.optimizer.step()
            return loss.detach()

        # the warm-up executions are REAL optimizer steps on a placeholder batch: CapturedStep undoes them (parameters, BatchNorm buffers,
        # Adam moments and step counts) so that constructing the graphed step leaves the training trajectory untouched
        cap = CapturedStep(body, [net], self.optimizer, device=dev, warmup=warmup)
        with torch.cuda.device(dev):
            self.ddp.zero_grad()
        self.stream, self.graph, self._pw = cap.stream, cap.graph, cap.workspaces
        self.loss, self.launches_per_step = cap.outputs, cap.launches_per_step

    def __call__(self, x):
        self.x.copy_(x, non_blocking=True)
        self.graph.replay()
        return self.loss
