"""SampleNet(nn.Module) -- drop-in for registration/src/samplenet.py:22-187, on this package's sm_90a kernels.

Constructor signature, attribute names (`name`, `project`, `skip_projection`, ...), state-dict keys
(`conv1..5`, `bn1..5`, `fc1..4`, `bn_fc1..3`, `project._temperature`), return values (`simp, proj` in training,
`simp, match` in eval; contiguous, shaped per `output_shape`) and error behaviour follow the reference.
What changes is what runs underneath:

  reference (samplenet.py:90-104)                      | here
  -----------------------------------------------------+------------------------------------------------------------
  5 x (cuDNN conv1d, BatchNorm kernel, ReLU kernel),   | ONE persistent cooperative kernel: conv layers as 3xTF32 warpgroup
  torch.max, 3 x (Linear, BN, ReLU), Linear            | MMAs with activations kept on the SM, BN statistics exchanged between
                                                       | CTAs, max-pool and FC head in the same launch (csrc/conv_stack.cu);
                                                       | per-layer kernels outside its envelope (csrc/encoder_tc.cu, encoder.cu)
  KNN (python loop over B) + grouping + ~8 torch ops   | one fused kNN + softmax + weighted-gather launch (csrc/softproj.cu)
  eval: .cpu().numpy() -> numpy FPS loop -> .cuda()    | NN search + unique + FPS completion on the GPU (csrc/matching.cu)
  ChamferDistance: 2 launches + 4 torch reductions     | one fused two-direction launch + one reduction launch (csrc/chamfer.cu)

Backward: the projection, the loss and the generator have hand-written CUDA backward kernels.  The generator's (csrc/generator_bwd.cu,
nine launches, exact fp32, deterministic) starts from the raw conv outputs its training forward keeps.  Outside that kernel's envelope,
or with generator_backward = "torch", the generator's backward recomputes the layer stack with torch's stock conv/BN/linear ops
(activation checkpointing) -- the forward never uses them.
"""
import os
import warnings

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops, sputils
from .soft_projection import SoftProjection


# CUDA training route -> (envelope, training forward that keeps the activations, backward) in ops.  Both routes end in the same backward
# kernels (csrc/generator_bwd.cu); "layers" runs the per-layer tensor-core kernels for the shapes the persistent kernel does not take.
_ROUTE_OPS = {
    "fused": (ops.generator_backward_supported, ops.generator_train_forward, ops.generator_backward),
    "layers": (ops.generator_layers_backward_supported, ops.generator_layers_train_forward, ops.generator_layers_backward),
}
_GRAD_KEYS = ("weight", "bias", "bn_weight", "bn_bias")


class _GeneratorFunction(torch.autograd.Function):
    """simp_flat = generator(x).  Forward: this library's kernels.  Backward: this library's backward kernels where they cover the shape,
    otherwise a recompute with torch ops + autograd.

    `net` is a LayerTableGenerator; `net._route(...)` picks the path ("fused", "layers" or "torch"), and the route of the last training
    forward is `net.generator_route`."""

    @staticmethod
    def forward(ctx, net, x, layout, training, out_inner, *params):
        conv_specs, fc_specs = net._layer_specs()
        route = net._route(x, layout, conv_specs, fc_specs, training)
        if route == "torch":
            out, _ = ops.generator_forward(x, layout, conv_specs, fc_specs, training, out_inner, exact_fp32=net.generator_precision == "fp32")
        else:
            # forward that keeps every conv layer's raw output: the backward is then this library's own kernels, no recompute, no library GEMM
            out, _, ctx.cuda_saved = _ROUTE_OPS[route][1](x, layout, conv_specs, fc_specs, out_inner)
        if training:
            net.generator_route = route
        ctx.route = route
        ctx.net = net
        ctx.layout = layout
        ctx.training = training
        ctx.out_inner = out_inner
        ctx.save_for_backward(x, *params)
        return out

    @staticmethod
    def backward(ctx, g):
        x, *params = ctx.saved_tensors
        net = ctx.net
        if ctx.route != "torch":
            conv_specs, fc_specs = net._layer_specs()
            layers, k = [], 0   # per layer of the specs, its parameters in _generator_named_parameters order: w, b[, g, beta]
            for spec in conv_specs + fc_specs:
                n = 2 if spec["bn"] is None else 4
                layers.append(params[k:k + n])
                k += n
            cuda_backward = _ROUTE_OPS[ctx.route][2]
            if net.direct_parameter_grads and all(p.grad is not None and p.grad.is_contiguous() for p in params):
                # the kernels write straight into the parameters' .grad storage (e.g. views of FlatBucketDataParallel's bucket): no fresh
                # gradient tensors, no AccumulateGrad adds (35 launches per step).  OVERWRITES: valid when this is the only backward
                # contribution to the generator's parameters between two zero_grad() calls (one sampler forward per step).
                dest = [dict(zip(_GRAD_KEYS, [p.grad for p in ps] + [None, None])) for ps in layers]
                cuda_backward(x, ctx.layout, conv_specs, fc_specs, ctx.cuda_saved, g.contiguous(), ctx.out_inner, dest=dest)
                return (None,) * (5 + len(params))
            grads = cuda_backward(x, ctx.layout, conv_specs, fc_specs, ctx.cuda_saved, g.contiguous(), ctx.out_inner)
            return (None,) * 5 + tuple(gl[key].view_as(p) for ps, gl in zip(layers, grads) for key, p in zip(_GRAD_KEYS, ps))
        # the recompute runs the reference layer stack in true fp32 (torch's cuDNN default would be plain TF32)
        tf32_c, tf32_m = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            return _GeneratorFunction._backward(ctx, g, x, params, net, [n for n, _ in net._generator_named_parameters()])
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32_c, tf32_m

    @staticmethod
    def _backward(ctx, g, x, params, net, names):
        with torch.enable_grad():
            xs = x.detach().requires_grad_(ctx.needs_input_grad[1])
            ps = {n: p.detach().requires_grad_(p.requires_grad) for n, p in zip(names, params)}
            y = net._torch_generator(xs, ctx.layout, ctx.training, ps)
            if ctx.out_inner:
                b = y.shape[0]
                y = y.view(b, -1, ctx.out_inner).permute(0, 2, 1).reshape(b, -1)
            inputs = ([xs] if xs.requires_grad else []) + [p for p in ps.values() if p.requires_grad]
            grads = torch.autograd.grad(y, inputs, g, allow_unused=True) if inputs else []
        grads = list(grads)
        gx = grads.pop(0) if xs.requires_grad else None
        gp = [grads.pop(0) if p.requires_grad else None for p in ps.values()]
        return (None, gx, None, None, None, *gp)


class LayerTableGenerator(nn.Module):
    """A SampleNet generator given by its widths: 1x1 conv layers, each followed by BatchNorm and ReLU, a max-pool over the points, then
    FC layers with BatchNorm and ReLU as given per layer.  Parameters are `conv<i>` / `bn<i>` (i = 1..) and `fc<i>` / `bn_fc<i>` (the
    latter only on FC layers with BatchNorm).  Training runs the first of the class's CUDA_ROUTES whose envelope holds the shape, else the
    torch recompute (see _route).  Base of SampleNet and of the reconstruction and classification samplers."""

    CUDA_ROUTES = ("fused", "layers")   # tried in this order; SampleNet trains on "fused" only
    MAX_GENERATOR_BATCH = 256   # rows the FC head kernels hold per launch (snb200_generator_forward rejects more)
    # Registration order of the modules.  False: each layer, then its BatchNorm (conv1, bn1, conv2, ...).  True: every conv layer, every
    # conv BatchNorm, every FC layer, every FC BatchNorm -- SampleNet's order, the reference class's, so parameters() indices, optimiser
    # state and flat gradient buckets line up with its checkpoints.  BatchNorm initialisation draws no random numbers, so both orders
    # leave the same initial parameters under one seed.
    GROUPED_REGISTRATION = False

    def __init__(self, conv_widths, fc_widths, fc_bn, fc_relu, bn_eps, bn_momentum):
        super().__init__()
        if len(fc_bn) != len(fc_widths) - 1 or len(fc_relu) != len(fc_widths) - 1 or fc_widths[0] != conv_widths[-1]:
            raise ValueError("layer table: %s conv widths, %s FC widths, %d / %d FC flags" % (conv_widths, fc_widths, len(fc_bn), len(fc_relu)))
        self.n_conv, self.n_fc = len(conv_widths) - 1, len(fc_widths) - 1
        modules = []
        for i in range(self.n_conv):
            modules += [("conv%d" % (i + 1), nn.Conv1d(conv_widths[i], conv_widths[i + 1], 1)),
                        ("bn%d" % (i + 1), nn.BatchNorm1d(conv_widths[i + 1], eps=bn_eps, momentum=bn_momentum))]
        for i in range(self.n_fc):
            modules.append(("fc%d" % (i + 1), nn.Linear(fc_widths[i], fc_widths[i + 1])))
            if fc_bn[i]:
                modules.append(("bn_fc%d" % (i + 1), nn.BatchNorm1d(fc_widths[i + 1], eps=bn_eps, momentum=bn_momentum)))
        if self.GROUPED_REGISTRATION:
            modules.sort(key=lambda m: (m[0].startswith(("fc", "bn_fc")), m[0].startswith("bn")))   # stable: keeps the layer order
        for name, module in modules:
            self.add_module(name, module)
        self.fc_relu = [bool(r) for r in fc_relu]
        # "3xtf32": conv layers 2..5 on the tensor cores, error-compensated to fp32 accuracy (default);
        # "fp32":   exact-fp32 CUDA-core conv stack.  Not part of the reference signature; plain attribute.
        self.generator_precision = "3xtf32"
        # "cuda": hand-written backward kernels (csrc/generator_bwd.cu) wherever they cover the shape; "torch": recompute the layer stack
        # with stock torch ops and differentiate that (the round-1 path; also the fallback outside the CUDA backward's envelope)
        self.generator_backward = os.environ.get("SNB200_GENERATOR_BACKWARD", "cuda")
        # opt-in (set by GraphedTrainStep): the CUDA backward writes into existing .grad tensors instead of returning fresh ones
        self.direct_parameter_grads = False
        self.generator_route = None

    def _convs(self):
        return [(getattr(self, "conv%d" % i), getattr(self, "bn%d" % i)) for i in range(1, self.n_conv + 1)]

    def _fcs(self):
        return [(getattr(self, "fc%d" % i), getattr(self, "bn_fc%d" % i, None)) for i in range(1, self.n_fc + 1)]

    def _relus(self):
        return [True] * self.n_conv + self.fc_relu

    def _generator_named_parameters(self):
        out = []
        for i, (lin, bn) in enumerate(self._convs() + self._fcs()):
            out += [("l%d.w" % i, lin.weight), ("l%d.b" % i, lin.bias)]
            if bn is not None:
                out += [("l%d.g" % i, bn.weight), ("l%d.beta" % i, bn.bias)]
        return out

    @staticmethod
    def _bn_tuple(bn):
        return (bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum, bn.num_batches_tracked)

    def _layer_specs(self):
        specs = [dict(weight=lin.weight, bias=lin.bias, bn=None if bn is None else self._bn_tuple(bn), relu=relu)
                 for (lin, bn), relu in zip(self._convs() + self._fcs(), self._relus())]
        return specs[:self.n_conv], specs[self.n_conv:]

    def _route(self, x, layout, conv_specs, fc_specs, training):
        """The path of a generator call: in training mode the first of CUDA_ROUTES whose envelope holds the shape, otherwise "torch" (the
        forward kernels, and the torch recompute for the backward).  fp32 precision, generator_backward = "torch" and an input that needs
        its gradient take "torch" too: the training forwards keep activations on the 3xTF32 path only, and the CUDA backward computes no
        input gradient."""
        if training and self.generator_backward == "cuda" and self.generator_precision != "fp32" and not x.requires_grad:
            for route in self.CUDA_ROUTES:
                if _ROUTE_OPS[route][0](x, layout, conv_specs, fc_specs):
                    return route
        return "torch"

    def _torch_generator(self, x, layout, training, ps):
        """The layer stack in stock torch ops; used only to differentiate the generator.  The 1x1 convolutions are evaluated as ONE
        [B*N, C_in] x [C_in, C_out] matrix product per layer (points-major, the layout of this library's kernels): identical arithmetic,
        but the weight gradient becomes a single GEMM with a 32 768-long reduction instead of cuDNN's fp32 grouped-direct wgrad kernel
        (1.8 ms of a 3.2 ms training step at the headline size)."""
        b = x.shape[0]
        y = x.reshape(-1, 3) if layout == "bnc" else x.permute(0, 2, 1).reshape(-1, 3)
        for i, ((lin, bn), relu) in enumerate(zip(self._convs() + self._fcs(), self._relus())):
            w, bias = ps["l%d.w" % i], ps["l%d.b" % i]
            if i == self.n_conv:
                y = y.view(b, -1, y.shape[1]).max(dim=1)[0]          # max over the points of a cloud
            y = F.linear(y, w.reshape(w.shape[0], -1), bias)
            if bn is not None:
                if training:
                    y = F.batch_norm(y, None, None, ps["l%d.g" % i], ps["l%d.beta" % i], True, 0.0, bn.eps)
                else:
                    y = F.batch_norm(y, bn.running_mean, bn.running_var, ps["l%d.g" % i], ps["l%d.beta" % i], False, 0.0, bn.eps)
            if relu:
                y = F.relu(y)
        return y

    def _generate(self, x, layout, out_inner):
        if x.shape[0] > self.MAX_GENERATOR_BATCH:
            if self.training:
                raise RuntimeError("%s: training-mode batches are limited to %d clouds per call (BatchNorm over the batch runs inside one FC-head "
                                   "launch); got %d.  Split the batch (statistics are per call, as in the reference per GPU)." %
                                   (type(self).__name__, self.MAX_GENERATOR_BATCH, x.shape[0]))
            # eval mode: BatchNorm uses the running statistics, so the batch can be processed in chunks with identical results
            return torch.cat([self._generate(xc.contiguous(), layout, out_inner) for xc in x.split(self.MAX_GENERATOR_BATCH, dim=0)], dim=0)
        params = [p for _, p in self._generator_named_parameters()]
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
            return _GeneratorFunction.apply(self, x, layout, self.training, out_inner, *params)
        conv_specs, fc_specs = self._layer_specs()
        y, _ = ops.generator_forward(x, layout, conv_specs, fc_specs, self.training, out_inner, exact_fp32=self.generator_precision == "fp32")
        return y

    def _generate_points(self, x):
        """x (B, N, 3) -> generated points (B, M, 3): the (B, 3M) output reshaped as TF does (consecutive triples are points)."""
        if x.dim() != 3 or x.shape[2] != 3:
            raise RuntimeError("shape of x must be of [Batch x NumInPoints x 3]")
        x = x.contiguous()
        return x, self._generate(x, "bnc", 0).view(x.shape[0], -1, 3)

    def sample(self, x):
        return self.__call__(x)[1]

    def get_projection_loss(self):
        sigma = self.project.sigma
        if not self.training:
            return torch.tensor(0).to(sigma)
        return sigma


class SampleNet(LayerTableGenerator):
    """The registration sampler: convs 3-64-64-64-128-bottleneck and FC bottleneck-256-256-256-3M, BatchNorm (torch defaults) and ReLU on
    every layer but the last.  Trains on the fused route (the per-layer route for a bottleneck above 128) or the torch recompute."""

    CUDA_ROUTES = ("fused",)
    GROUPED_REGISTRATION = True

    def __init__(
        self,
        num_out_points,
        bottleneck_size,
        group_size,
        initial_temperature=1.0,
        is_temperature_trainable=True,
        min_sigma=1e-2,
        input_shape="bcn",
        output_shape="bcn",
        complete_fps=True,
        skip_projection=False,
    ):
        super().__init__([3, 64, 64, 64, 128, bottleneck_size], [bottleneck_size, 256, 256, 256, 3 * num_out_points], fc_bn=[True] * 3 + [False],
                         fc_relu=[True] * 3 + [False], bn_eps=1e-5, bn_momentum=0.1)
        self.num_out_points = num_out_points
        self.name = "samplenet"
        if bottleneck_size > 128:   # wider than the fused kernel's conv stack: the per-layer route
            self.CUDA_ROUTES = ("layers",)

        # projection and matching
        self.project = SoftProjection(group_size, initial_temperature, is_temperature_trainable, min_sigma)
        self.skip_projection = skip_projection
        self.complete_fps = complete_fps

        # input / output shapes
        if input_shape not in ["bcn", "bnc"]:
            raise ValueError("allowed shape are 'bcn' (batch * channels * num_in_points), 'bnc' ")
        if output_shape not in ["bcn", "bnc"]:
            raise ValueError("allowed shape are 'bcn' (batch * channels * num_in_points), 'bnc' ")
        if input_shape != output_shape:
            warnings.warn("SampleNet: input_shape is different to output_shape.")
        self.input_shape = input_shape
        self.output_shape = output_shape
        # project + Chamfer + loss reductions of (simp, x) in one launch when forward() runs in training mode ("bnc" in and out)
        self.fused_tail = True
        self._tail = None

    # ------------------------------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor):
        layout = self.input_shape
        cdim = 1 if layout == "bcn" else 2
        if x.dim() != 3 or x.shape[cdim] != 3:
            raise RuntimeError("shape of x must be of [Batch x 3 x NumInPoints]")
        x = x.contiguous()
        m = self.num_out_points
        # Drop the previous call's loss terms before this call's graph is built: they keep that graph, and with it the parameters'
        # gradient accumulators, alive, and an accumulator created on another stream would make a CUDA-graph capture of this step wait on it.
        self._tail = None

        # Generated points, produced directly in the layout of the input cloud (the FC head can store its (3, M) rows
        # transposed), so that projection / matching run without permuting the big cloud.
        y = self._generate(x, layout, m if layout == "bnc" else 0)
        simp_in = y.view(-1, m, 3) if layout == "bnc" else y.view(-1, 3, m)  # same layout as x

        match = None
        proj = None
        if self.training:
            if not self.skip_projection:
                if self.fused_tail and layout == "bnc" and self.output_shape == "bnc" and x.shape[1] <= 4096 and m <= 4096:
                    # projection + Chamfer + loss reductions of (simp, x) in one launch; the loss terms are kept for
                    # get_simplification_loss(x, simp, ...) (same tensors => no further launch)
                    sp = self.project
                    if sp._min_sigma_value is None:
                        sp._min_sigma_value = float(sp._min_sigma)
                    proj, loss_w1, terms = ops.ProjectAndLossFunction.apply(x, simp_in, sp._temperature, sp._group_size, 1, sp._min_sigma_value)
                    self._tail = (x, simp_in, x._version, simp_in._version, loss_w1, terms)
                else:
                    proj = self.project.project(x, simp_in, layout=layout)
            else:
                proj = simp_in
        else:  # Inference: nearest input point per generated point, unique, FPS completion -- all on the GPU
            x_bnc = x if layout == "bnc" else x.permute(0, 2, 1).contiguous()
            q_bnc = simp_in if layout == "bnc" else simp_in.permute(0, 2, 1).contiguous()
            _, idx1, _, _ = ops.nn_distance_forward(q_bnc.detach(), x_bnc.detach())
            match = sputils.nn_matching_cuda(x_bnc.detach(), idx1, m, complete_fps=self.complete_fps)  # B x M x 3

        # Change to output shapes
        def to_out(t, t_layout):
            if t is None or t_layout == self.output_shape:
                return t
            return t.permute(0, 2, 1)

        simp = to_out(simp_in, layout)
        proj = to_out(proj, layout)
        match = to_out(match, "bnc")

        simp = simp.contiguous()
        if proj is not None:
            proj = proj.contiguous()
        if match is not None:
            match = match.contiguous()

        out = proj if self.training else match
        return simp, out

    # Losses: at inference time there are no sampling losses (reference samplenet.py:167-187).
    def get_simplification_loss(self, ref_pc, samp_pc, pc_size, gamma=1, delta=0):
        if self.skip_projection or not self.training:
            return torch.tensor(0).to(ref_pc)
        # ref_pc and samp_pc are B x N x 3 matrices
        w = gamma + delta * pc_size
        tail = getattr(self, "_tail", None)
        if tail is not None and tail[0] is ref_pc and tail[1] is samp_pc and tail[2] == ref_pc._version and tail[3] == samp_pc._version:
            # the forward pass already evaluated Chamfer(samp, ref) and its reductions in the projection launch
            if w == 1:
                return tail[4]
            return tail[5][0] + tail[5][1] + w * tail[5][2]
        return ops.SimplificationLossFunction.apply(samp_pc, ref_pc, w)

    def get_projection_loss(self):
        sigma = self.project.sigma()
        if self.skip_projection or not self.training:
            return torch.tensor(0).to(sigma)
        return sigma
