"""The per-layer training path (ops.generator_layers_train_forward / generator_layers_backward) against float64, stage by stage.

Three float64 evaluations of the same layer stack, all routed through the max-pool at the kernel's own arg-max:
  * plain: float64 throughout;
  * kernel-valued: every conv layer's raw output z_l is replaced by its VALUE from the kernel's zsave[l]
    (z64 + (zsave[l] - z64).detach()), so BatchNorm statistics, ReLU masks and the pool's arg-max are the kernel's while gradients still
    flow through float64 weights, biases and BatchNorm parameters.  What remains between this and the CUDA backward is the backward
    kernels' own arithmetic, and it is held to a tight bar;
  * fp32-valued (the yardstick): the same replacement with the plain graph's own activations rounded to fp32.  No kernel is involved; its
    distance from the plain graph is how far ANY correct fp32 forward moves each gradient at that shape.  The end-to-end bar of a tensor
    is max(2e-4 * scale, K_YARDSTICK * that distance).

ReLU kinks at routed points.  Only the points the max-pool routes to carry more than an O(1/points) share of the gradient, and at 50 x 2048
they hold ~4 500 points x 704 conv units, a few of which lie within the fp32 forward's error (~1e-6 of |scale z| + |shift|) of their
ReLU kink.  Which side such a unit lands on moves its channel's BatchNorm shift gradient by up to 2 % in ANY fp32 implementation; that,
not a kernel bug, is why the float64 check once failed at this size.  So the kernel-valued graph applies the kernel's own fp32 masks
(kernel_masks), and cases are stepped to a seed with no routed unit within KINK_GUARD of a kink.  The end-to-end check therefore runs on
such a conditioned instance, and it is not fully independent of the kernel: in the plain and the fp32-valued graphs, units within
AMBIGUOUS of their kink take the kernel's fp32 mask (so the yardstick holds no mask-flip noise either).  Those pinned units are counted
and held to at most PINNED_BAR of the routed points' conv units (at least 4 units allowed); up to 40 of ~3e6 were pinned at 64 x 2048.

The forward is checked layer by layer (zsave[l] against float64 layer l applied to the kernel's own zsave[l-1]), together with the pooled
feature, the output and every BatchNorm layer's running statistics against PyTorch's update rule.  Cases cover the reconstruction,
classification (eps 1e-3, from TF variables) and registration tables, batch sizes up to 64 and clouds of 2048 points down to one point,
BCN input, a transposed output store, BatchNorm scales < 0 and channels whose pooled value is 0 in some clouds.  The CPU tests pin the
references: the plain graph is autograd of LayerTableGenerator._torch_generator, the route goes to the known point, and the running
statistics follow torch's BatchNorm1d."""
import copy
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from samplenet_b200 import ReconstructionSampleNet  # noqa: E402
from samplenet_b200.samplenet import LayerTableGenerator  # noqa: E402
from samplenet_b200.tf_variant import ClassificationSampleNet  # noqa: E402

# Bars, each about 10x the largest value measured over all cases on an H100 80GB HBM3 at a 400 W power limit (measured maxima in brackets)
FWD_Z_BAR = 2e-5        # [1.9e-6] |zsave[l] - float64 layer l| / the point's sum |terms|
FWD_FEAT_BAR = 2e-6     # [2.1e-7] pooled feature: / (|scale * z*| + |shift|)
FWD_OUT_BAR = 4e-5      # [3.7e-6] output: / max |out|
RUNNING_BAR = 2e-5      # [2.2e-6] running mean / variance: / (|previous| (1 - m) + m (|batch mean| + batch std)), resp. the expected variance
BWD_KERNEL_BAR = 3e-4   # [3.3e-5] CUDA backward against the kernel-valued float64 graph: / the tensor's scale
KINK_GUARD = 3e-7       # cases have no unit at a routed point closer than this to its ReLU kink (relative, see kink_distances)
AMBIGUOUS = 1e-5        # ... and units closer than this take the kernel's ReLU mask in the end-to-end reference
PINNED_BAR = 1e-4       # [1.3e-5] ... which may be at most this fraction of the routed points' conv units (or 4 units in small cases)
K_YARDSTICK = 4.0       # end to end: max(2e-4 * scale, K_YARDSTICK * the fp32-valued graph's distance from the plain one)


# ------------------------------------------------------------------------------------------------------------------ references
def _rows(x, layout):
    return (x if layout == "bnc" else x.permute(0, 2, 1)).reshape(-1, 3)


def _route(z, gamma, b):
    """(b, C) index of the point each (cloud, channel) pools: the first maximum of sign(gamma) * z, the raw last conv layer (the pool
    commutes with the monotone BatchNorm + ReLU map; it is a max where the BatchNorm scale is >= 0 and a min otherwise)."""
    sgn = torch.ones(z.shape[1], dtype=z.dtype, device=z.device) if gamma is None else torch.where(gamma >= 0, 1.0, -1.0).to(z)
    return (z.view(b, -1, z.shape[1]) * sgn).argmax(dim=1)


def reference64(net, x, layout, rw, zsave=None, route=None, out_inner=0, masks=None):
    """Float64 autograd of `net`'s layer stack (training-mode BatchNorm) for the upstream gradient rw.

    zsave: per conv layer, raw outputs whose VALUES replace the graph's (gradients still flow through the float64 parameters).
    route: (b, C) point per (cloud, channel) of the max-pool; default: the arg-max of the graph's own last conv layer.
    masks: per conv layer, a function (BatchNorm output, raw output) -> the ReLU mask to apply; default: the graph's own (> 0).
    Returns (gradients by parameter name, route, the raw conv outputs' values, the output)."""
    conv_specs, fc_specs = net._layer_specs()
    nconv = len(conv_specs)
    b = x.shape[0]
    ps = {nm: p.detach().double().requires_grad_(True) for nm, p in net._generator_named_parameters()}
    h = _rows(x.double(), layout)
    zs = []
    for i, spec in enumerate(conv_specs + fc_specs):
        if i == nconv:
            if route is None:
                route = _route(zs[-1], conv_specs[-1]["bn"][0].detach().double() if conv_specs[-1]["bn"] else None, b)
            h = torch.gather(h.view(b, -1, h.shape[1]), 1, route[:, None, :].to(h.device)).squeeze(1)
        w = ps["l%d.w" % i]
        h = F.linear(h, w.reshape(w.shape[0], -1), ps["l%d.b" % i])
        if i < nconv:
            if zsave is not None:
                h = h + (zsave[i].to(h) - h).detach()
            zs.append(h.detach())
        if spec["bn"] is not None:
            h = F.batch_norm(h, None, None, ps["l%d.g" % i], ps["l%d.beta" % i], True, 0.0, spec["bn"][4])
        if spec["relu"] and masks is not None and i < nconv:
            h = h * masks[i](h.detach(), zs[i]).to(h)
        elif spec["relu"]:
            h = torch.relu(h)
    if out_inner:
        h = h.view(b, -1, out_inner).permute(0, 2, 1).reshape(b, -1)
    g = torch.autograd.grad(h, list(ps.values()), rw.to(h))
    return dict(zip(ps, g)), route, zs, h.detach()


def _bn64(z, eps):
    """Training-mode BatchNorm statistics of z's rows in float64: (mean, biased variance, 1 / sqrt(variance + eps))."""
    z = z.double()
    mean, var = z.mean(0), z.var(0, unbiased=False)
    return mean, var, 1.0 / torch.sqrt(var + eps)


def _bn_act(z, spec):
    """relu(BN(z)) in float64 with z's own batch statistics."""
    g, beta, eps = spec["bn"][0].detach().double(), spec["bn"][1].detach().double(), spec["bn"][4]
    mean, _, inv = _bn64(z, eps)
    return torch.relu((z.double() - mean) * inv * g + beta)


def running_update64(prev_mean, prev_var, z, momentum):
    """PyTorch's training-mode update of BatchNorm running statistics from the rows of z, in float64: the momentum mix with the batch mean
    and the UNBIASED batch variance.  Returns (mean, variance, the batch's mean, std)."""
    z = z.double()
    cnt = z.shape[0]
    mean, var = z.mean(0), z.var(0, unbiased=False)
    unb = var * cnt / (cnt - 1) if cnt > 1 else var
    return ((1 - momentum) * prev_mean.double() + momentum * mean, (1 - momentum) * prev_var.double() + momentum * unb, mean, var.sqrt())


def _fc_chain64(net, feat, out_inner=0):
    """The FC layers in float64 from a given pooled feature: (output, each BatchNorm FC layer's pre-BatchNorm rows, smallest |pre-ReLU|)."""
    _, fc_specs = net._layer_specs()
    h = feat.double()
    pre, margin = [], float("inf")
    for spec in fc_specs:
        h = F.linear(h, spec["weight"].detach().double(), spec["bias"].detach().double())
        if spec["bn"] is not None:
            pre.append(h)
            mean, _, inv = _bn64(h, spec["bn"][4])
            h = (h - mean) * inv * spec["bn"][0].detach().double() + spec["bn"][1].detach().double()
        if spec["relu"]:
            margin = min(margin, h.abs().min().item())
            h = torch.relu(h)
    if out_inner:
        b = h.shape[0]
        h = h.view(b, -1, out_inner).permute(0, 2, 1).reshape(b, -1)
    return h, pre, margin


def kink_distances(net, zs, route):
    """Per conv layer, |BN(z)| / (|scale z| + |shift|) in float64 at the points the max-pool routes a gradient to (the only points whose
    conv units carry more than the BatchNorm backward's O(1/points) share; every point with route None): how close each of those ReLU
    masks is to flipping."""
    conv_specs, _ = net._layer_specs()
    if route is None:
        pts = slice(None)
    else:
        b = route.shape[0]
        pts = torch.unique((route + torch.arange(b, device=route.device)[:, None] * (zs[0].shape[0] // b)).flatten())
    out = []
    for z, spec in zip(zs, conv_specs):
        mean, _, inv = _bn64(z, spec["bn"][4])
        sc = spec["bn"][0].detach().double() * inv
        sh = spec["bn"][1].detach().double() - mean * sc
        zp = z[pts].double()
        out.append(((zp * sc + sh).abs() / (zp.abs() * sc.abs() + sh.abs())))
    return out


def kernel_masks(net, zs):
    """Per conv layer, the ReLU mask the CUDA backward applies to raw outputs zs: fmaf(scale, z, shift) > 0 with the fp32 scale
    gamma / sqrtf(var + eps) and shift beta - mean * scale.  The sign of a fused multiply-add is that of the exact value, which the float64
    product of the two fp32 factors plus the shift has too.  (Statistics are taken from zs in float64; the kernel's own double sums of
    fp32 tile sums can move scale or shift by an ulp, which run_case keeps away from the kink.)"""
    conv_specs, _ = net._layer_specs()
    out = []
    for z, spec in zip(zs, conv_specs):
        mean, var, _ = _bn64(z, spec["bn"][4])
        inv = 1.0 / torch.sqrt(var.float() + spec["bn"][4])
        sc = spec["bn"][0].detach().float() * inv
        sh = (spec["bn"][1].detach().double() - mean.float().double() * sc.double()).float()
        out.append((z.double() * sc.double() + sh.double()) > 0)
    return out


def _conv_forward64(net, x, layout):
    """Raw conv outputs of the plain float64 forward, and the pooled feature."""
    conv_specs, _ = net._layer_specs()
    b = x.shape[0]
    h, zs = _rows(x.double(), layout), []
    for spec in conv_specs:
        z = F.linear(h, spec["weight"].detach().double().reshape(spec["weight"].shape[0], -1), spec["bias"].detach().double())
        zs.append(z)
        h = _bn_act(z, spec)
    return zs, h.view(b, -1, h.shape[1]).max(dim=1)[0]


# ------------------------------------------------------------------------------------------------------------------ networks
M_OUT = 64


def _tf_variables(rng, m):
    """Sampler-scope variables of the classification trainer's TF graph (fc14b included), with non-trivial moving averages."""
    widths, fcw = [3, 64, 64, 64, 128, 128], [128, 256, 256, 256, 3 * m]
    layers = [("conv%d" % (i + 1), [1, 3, 1, 64] if i == 0 else [1, 1, widths[i], widths[i + 1]], widths[i + 1]) for i in range(5)]
    layers += [("fc1%db" % (i + 1), [fcw[i], fcw[i + 1]], fcw[i + 1]) for i in range(4)]
    v = {}
    for sc, shape, c in layers:
        sc = "sampler/" + sc
        fan_in = int(np.prod(shape[:-1]))
        v[sc + "/weights:0"] = (rng.standard_normal(shape) / np.sqrt(fan_in)).astype(np.float32)
        v[sc + "/biases:0"] = (0.1 * rng.standard_normal(c)).astype(np.float32)
        v[sc + "/bn/gamma:0"] = (1.0 + 0.2 * rng.standard_normal(c)).astype(np.float32)
        v[sc + "/bn/beta:0"] = (0.1 * rng.standard_normal(c)).astype(np.float32)
        v[sc + "/bn/moments/Squeeze/ExponentialMovingAverage:0"] = (0.1 * rng.standard_normal(c)).astype(np.float32)
        v[sc + "/bn/moments/Squeeze_1/ExponentialMovingAverage:0"] = (0.5 + rng.random(c)).astype(np.float32)
    return v


def make_net(table, seed):
    """rec: ReconstructionSampleNet; cls: ClassificationSampleNet.from_tf_variables (eps 1e-3, momentum 0.5); reg: the registration table
    as a LayerTableGenerator (so it trains on the per-layer entry points).  Shifts are perturbed and the running statistics start away
    from (0, 1), so that the momentum mix is visible."""
    torch.manual_seed(seed)
    if table == "rec":
        net = ReconstructionSampleNet(M_OUT)
    elif table == "cls":
        net = ClassificationSampleNet.from_tf_variables(_tf_variables(np.random.default_rng(seed), M_OUT))
    else:
        net = LayerTableGenerator([3, 64, 64, 64, 128, 128], [128, 256, 256, 256, 3 * M_OUT], [1, 1, 1, 0], [1, 1, 1, 0], 1e-5, 0.1)
    with torch.no_grad():
        for lin, bn in net._convs() + net._fcs():
            lin.bias.add_(0.1 * torch.randn_like(lin.bias))
            if bn is not None and table != "cls":
                bn.weight.add_(0.1 * torch.randn_like(bn.weight))
                bn.bias.add_(0.1 * torch.randn_like(bn.bias))
                bn.running_mean.copy_(0.2 * torch.randn_like(bn.running_mean))
                bn.running_var.copy_(0.5 + torch.rand_like(bn.running_var))
    return net


def apply_signs(net, x, layout):
    """About a quarter of every conv layer's channels get a BatchNorm scale < 0 (channels l % 4 + 4 k of layer l, the last layer's
    included); every 8th channel of the inner conv layers gets a shift of -1.5; and on channels 5 + 8 k (scale > 0) and 4 + 16 k (scale < 0,
    pooled at the cloud's arg-min) of the last conv layer the shift is set between two clouds' pooled extrema of scale * zhat (from the
    float64 forward), so that the pooled value after BatchNorm + ReLU is 0 in some clouds and not in others.  Returns those channels."""
    convs = net._convs()
    with torch.no_grad():
        for l, (_, bn) in enumerate(convs):
            bn.weight[(l % 4)::4] = -bn.weight[(l % 4)::4].abs()
            if l + 1 < len(convs):
                bn.bias[3::8] = -1.5
    zs, _ = _conv_forward64(net, x, layout)
    b = x.shape[0]
    bn = convs[-1][1]
    g = bn.weight.detach().double()
    _, _, inv = _bn64(zs[-1], bn.eps)
    zh = (zs[-1] - zs[-1].mean(0)) * inv
    peak = (zh * g).view(b, -1, zh.shape[1]).max(dim=1)[0]          # (b, C): the cloud's largest gamma * zhat
    dead = sorted(set(range(5, zh.shape[1], 8)) | set(range(4, zh.shape[1], 16)))   # 4 + 16 k: scale < 0, pooled at the arg-min
    with torch.no_grad():
        for c in dead:
            s = peak[:, c].sort()[0]
            lo, hi = max(0, b // 4 - 1), max(1, (3 * b) // 4)
            j = max(range(lo, min(hi, b - 1)), key=lambda k: (s[k + 1] - s[k]).item()) if b > 1 else 0
            thr = (s[j] + s[j + 1]) / 2 if b > 1 else s[0] + 1.0
            bn.bias[c] = float(-thr)
    return dead


def make_case(table, b, n, layout, signs, seed0, device, accept=None):
    """A network and a cloud batch with no FC pre-activation within 2e-5 of the ReLU kink (a flipped mask on one of the <= 64 rows moves
    every gradient in ANY fp32 implementation), found by stepping the seed."""
    for seed in range(seed0, seed0 + 30):
        net = make_net(table, seed).to(device).train()
        g = torch.Generator().manual_seed(seed)
        x = torch.rand(b, n, 3, generator=g) - 0.5
        x = (x if layout == "bnc" else x.permute(0, 2, 1).contiguous()).to(device)
        dead = apply_signs(net, x, layout) if signs else []
        _, feat = _conv_forward64(net, x, layout)
        if _fc_chain64(net, feat)[2] > 2e-5 and (accept is None or accept(net, x)):
            return net, x, dead
    raise AssertionError("no well-conditioned instance")


# ------------------------------------------------------------------------------------------------------------------ CPU pins
@pytest.mark.parametrize("table,layout,out_inner", [("rec", "bnc", 0), ("cls", "bcn", 0), ("reg", "bnc", M_OUT)])
def test_reference_is_autograd_of_the_torch_generator(table, layout, out_inner):
    """With no value replacement the reference is autograd of LayerTableGenerator._torch_generator in float64 (its max-pool, unrouted)."""
    net, x, _ = make_case(table, 3, 40, layout, True, 7, "cpu")
    rw = torch.randn(3, 3 * M_OUT, dtype=torch.float64)
    got, _, _, out = reference64(net, x, layout, rw, out_inner=out_inner)
    net64 = copy.deepcopy(net).double()
    ps = {nm: p.detach().requires_grad_(True) for nm, p in net64._generator_named_parameters()}
    y = net64._torch_generator(x.double(), layout, True, ps)
    if out_inner:
        y = y.view(3, -1, out_inner).permute(0, 2, 1).reshape(3, -1)
    want = dict(zip(ps, torch.autograd.grad(y, list(ps.values()), rw)))
    assert torch.allclose(out, y.detach(), rtol=0, atol=1e-12)
    for nm, g in want.items():
        assert (got[nm] - g).abs().max().item() <= 1e-12 * max(1.0, g.abs().max().item()), nm


def test_reference_routes_to_the_known_point():
    """A hand-built stack whose pooled channels are monotone in a point's x coordinate: a BatchNorm scale >= 0 pools the cloud's largest x,
    a scale < 0 its smallest, and a channel dead in a cloud sends that cloud nothing."""
    b, n = 2, 6
    net = LayerTableGenerator([3, 8, 8], [8, 4], [0], [0], 1e-5, 0.1).double().train()
    with torch.no_grad():
        for p in net.parameters():
            p.zero_()
        net.conv1.weight[:, 0, 0] = 1.0            # z1[c] = x
        net.bn1.weight.fill_(1.0)
        net.bn1.bias.fill_(10.0)                   # BN(x) + 10 > 0: ReLU passes, a1[c] is increasing in x
        net.conv2.weight[:, 0, 0] = 1.0            # z2[c] = a1[0]: increasing in x
        net.bn2.weight.copy_(torch.tensor([1.0, -1.0, 2.0, -0.5, 1.0, -1.0, 1.0, 1.0], dtype=torch.float64))
        net.bn2.bias.zero_()
        net.bn2.bias[6] = -50.0                    # dead in every cloud
        net.fc1.weight.copy_(torch.randn(4, 8, dtype=torch.float64))
    x = torch.rand(b, n, 3, dtype=torch.float64) - 0.5
    x[0, 4, 0], x[0, 1, 0] = 1.0, -1.0             # cloud 0: largest x at point 4, smallest at point 1
    x[1, 2, 0], x[1, 5, 0] = 1.0, -1.0             # cloud 1: largest at 2, smallest at 5
    rw = torch.randn(b, 4, dtype=torch.float64)
    g, route, zs, _ = reference64(net, x, "bnc", rw)
    big, small = torch.tensor([4, 2]), torch.tensor([1, 5])
    for c, gam in enumerate(net.bn2.weight.tolist()):
        assert torch.equal(route[:, c], big if gam >= 0 else small), (c, route[:, c])
    # fc1's weight gradient is rw^T . pooled feature, the pooled feature relu(BN(z2)) at the routed point
    y2 = _bn_act(zs[1], dict(bn=(net.bn2.weight, net.bn2.bias, None, None, net.bn2.eps))).view(b, n, 8)
    feat = torch.stack([y2[i, route[i]].diagonal() for i in range(b)])
    assert torch.equal(feat[:, 6], torch.zeros(b, dtype=torch.float64)) and (feat[:, :6] > 0).all()
    assert torch.allclose(g["l2.w"], rw.t() @ feat, rtol=1e-12, atol=1e-12)
    # an externally given route is followed as given
    g2, r2, _, _ = reference64(net, x, "bnc", rw, route=torch.zeros_like(route))
    assert torch.equal(r2, torch.zeros_like(route)) and not torch.allclose(g2["l2.w"], g["l2.w"])


@pytest.mark.parametrize("rows", [1, 2, 155])
def test_running_update_reference_is_torch_batchnorm(rows):
    torch.manual_seed(rows)
    bn = torch.nn.BatchNorm1d(16, eps=1e-3, momentum=0.3).double().train()
    with torch.no_grad():
        bn.running_mean.copy_(torch.randn(16)); bn.running_var.copy_(0.5 + torch.rand(16))
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    z = torch.randn(max(rows, 2), 16, dtype=torch.float64) * 3 + 1
    bn(z)
    m, v, _, _ = running_update64(rm0, rv0, z, 0.3)
    assert torch.allclose(m, bn.running_mean, rtol=1e-14, atol=1e-14) and torch.allclose(v, bn.running_var, rtol=1e-14, atol=1e-14)


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _flat_grads(specs, grads):
    out = {}
    for i, (spec, gl) in enumerate(zip(specs, grads)):
        out["l%d.w" % i], out["l%d.b" % i] = gl["weight"], gl["bias"]
        if spec["bn"] is not None:
            out["l%d.g" % i], out["l%d.beta" % i] = gl["bn_weight"], gl["bn_bias"]
    return out


def _bn_buffers(net):
    return [(bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()) for _, bn in net._convs() + net._fcs() if bn is not None]


def _restore(net, state):
    with torch.no_grad():
        for (_, bn), (m, v, t) in zip([lb for lb in net._convs() + net._fcs() if lb[1] is not None], state):
            bn.running_mean.copy_(m); bn.running_var.copy_(v); bn.num_batches_tracked.copy_(t)


def _run(sb, net, x, layout, rw, out_inner, route):
    conv_specs, fc_specs = net._layer_specs()
    train_forward = sb.ops.generator_layers_train_forward if route == "layers" else sb.ops.generator_train_forward
    backward = sb.ops.generator_layers_backward if route == "layers" else sb.ops.generator_backward
    with torch.no_grad():
        out, feat, saved = train_forward(x, layout, conv_specs, fc_specs, out_inner)
        zs = [z.clone() for z in saved[0]]
        grads = backward(x, layout, conv_specs, fc_specs, saved, rw, out_inner)
    if x.is_cuda:
        torch.cuda.synchronize()
    return out, feat, zs, _bn_buffers(net), _flat_grads(conv_specs + fc_specs, grads)


def zero_true_names(net):
    """Parameters whose true gradient is exactly 0: biases in front of a training-mode BatchNorm, and the last conv layer's BatchNorm shift
    when fc1 has BatchNorm (a constant added to a pooled channel is removed by its mean subtraction).  Both sides hold rounding noise."""
    conv_specs, fc_specs = net._layer_specs()
    specs = conv_specs + fc_specs
    out = {"l%d.b" % i for i, s in enumerate(specs) if s["bn"] is not None}
    if fc_specs[0]["bn"] is not None:
        out.add("l%d.beta" % (len(conv_specs) - 1))
    return out


def _scales(net, ref):
    """Per tensor, the scale its error is measured against: its largest entry, or for a tensor whose true gradient is 0, the largest
    entry of its layer's weight gradient (its rounding noise comes from the same dz sums)."""
    zt = zero_true_names(net)
    return {nm: max((ref["l%s.w" % nm[1:nm.index(".")]] if nm in zt else r).abs().max().item(), 1e-30) for nm, r in ref.items()}


def run_case(sb, table, b, n, layout="bnc", signs=False, out_inner=0, route="layers", seed0=None, device="cuda"):
    """Every stage check of one case.  Returns (report, info): report maps a check to (largest measured value, bar)."""
    def accept(net, x):
        # no ReLU unit at a routed point within a few fp32 ulps of the kink (kernel_masks could then disagree with the kernel)
        conv_specs, fc_specs = net._layer_specs()
        state = _bn_buffers(net)
        train_forward = sb.ops.generator_layers_train_forward if route == "layers" else sb.ops.generator_train_forward
        with torch.no_grad():
            zs = [z.clone() for z in train_forward(x, layout, conv_specs, fc_specs, out_inner)[2][0]]
        _restore(net, state)
        kd = kink_distances(net, zs, _route(zs[-1], conv_specs[-1]["bn"][0].detach(), x.shape[0]))
        return min(k.min().item() for k in kd) > KINK_GUARD

    net, x, dead = make_case(table, b, n, layout, signs, b * 131 + n if seed0 is None else seed0, device, accept)
    conv_specs, fc_specs = net._layer_specs()
    nconv = len(conv_specs)
    ok = (sb.ops.generator_layers_backward_supported if route == "layers" else sb.ops.generator_backward_supported)(x, layout, conv_specs, fc_specs)
    assert ok, (table, b, n, route)
    rw = torch.randn(b, fc_specs[-1]["weight"].shape[0], device=device, generator=torch.Generator(device=device).manual_seed(b + n))
    state0 = _bn_buffers(net)
    runs = []
    for _ in range(2):
        _restore(net, state0)
        runs.append(_run(sb, net, x, layout, rw, out_inner, route))
    (out, feat, zs, state1, grads), rerun = runs
    ident = torch.equal(out, rerun[0]) and torch.equal(feat, rerun[1]) and all(torch.equal(a, c) for a, c in zip(zs, rerun[2]))
    ident = ident and all(torch.equal(a, c) for s, t in zip(state1, rerun[3]) for a, c in zip(s, t))
    ident = ident and all(torch.equal(grads[k], rerun[4][k]) for k in grads)
    rep, info = {}, {"dead_clouds": None}

    def put(key, val, bar):
        old = rep.get(key, (0.0, bar))[0]
        rep[key] = (max(old, val), bar)

    put("bit_identical", 0.0 if ident else 1.0, 0.0)
    # ---- (a) forward, layer by layer from the kernel's own input
    for l, spec in enumerate(conv_specs):
        w = spec["weight"].detach().double().reshape(spec["weight"].shape[0], -1)
        bias = spec["bias"].detach().double()
        a = _rows(x.double(), layout) if l == 0 else _bn_act(zs[l - 1], conv_specs[l - 1])
        ref = F.linear(a, w, bias)
        terms = F.linear(a.abs(), w.abs(), bias.abs())
        put("fwd_z", ((zs[l].double() - ref).abs() / terms.clamp_min(1e-30)).max().item(), FWD_Z_BAR)
    sl = conv_specs[-1]
    mean, _, inv = _bn64(zs[-1], sl["bn"][4])
    sc = sl["bn"][0].detach().double() * inv
    sh = sl["bn"][1].detach().double() - mean * sc
    y = (zs[-1].double() * sc + sh).view(b, -1, sc.shape[0])
    ref_feat = torch.relu(y).max(dim=1)[0]
    fscale = (zs[-1].double().abs().view(b, -1, sc.shape[0]).max(dim=1)[0] * sc.abs() + sh.abs())
    put("fwd_feat", ((feat.double() - ref_feat).abs() / fscale).max().item(), FWD_FEAT_BAR)
    ref_out, fc_pre, _ = _fc_chain64(net, feat, out_inner)
    put("fwd_out", (out.double() - ref_out).abs().max().item() / ref_out.abs().max().item(), FWD_OUT_BAR)
    if dead:
        neg = sl["bn"][0].detach()[dead] < 0
        zero = (feat[:, dead] == 0)
        info["dead_clouds"] = (int(zero.sum()), zero.numel())
        info["dead_clouds_negative_scale"] = (int(zero[:, neg].sum()), int(zero[:, neg].numel()))
    # running statistics and num_batches_tracked: conv layers from the kernel's zsave, FC layers from the float64 head on its feature
    pre = [z for z in zs] + fc_pre
    bn_specs = [s for s in conv_specs + fc_specs if s["bn"] is not None]
    for spec, z, (m0, v0, t0), (m1, v1, t1) in zip(bn_specs, pre, state0, state1):
        mom = spec["bn"][5]
        em, ev, bmean, bstd = running_update64(m0, v0, z, mom)
        mscale = (1 - mom) * m0.double().abs() + mom * (bmean.abs() + bstd)
        put("running_mean", ((m1.double() - em).abs() / mscale).max().item(), RUNNING_BAR)
        put("running_var", ((v1.double() - ev).abs() / ev).max().item(), RUNNING_BAR)
        put("num_batches_tracked", float(int(t1) != int(t0) + 1), 0.0)
    # ---- (b) backward against the kernel-valued float64 graph, (c) end to end against the plain one
    kroute = _route(zs[-1], sl["bn"][0].detach(), b)
    km = kernel_masks(net, zs)
    r_kernel, route_k, _, _ = reference64(net, x, layout, rw, zsave=zs, out_inner=out_inner, masks=[lambda h, z, m=m: m for m in km])
    assert torch.equal(route_k, kroute)
    r_raw, _, zs64, _ = reference64(net, x, layout, rw, route=kroute, out_inner=out_inner)
    # units within AMBIGUOUS of the kink (relative to |scale z| + |shift|, float64) take the kernel's mask: a correct fp32 forward can
    # land on either side of them, and at a point the max-pool routes to, the side decides whole BatchNorm-shift entries
    mixed = [lambda h, z, m=m, d=d: torch.where(d < AMBIGUOUS, m, h > 0) for m, d in zip(km, kink_distances(net, zs64, None))]
    r_plain, _, _, _ = reference64(net, x, layout, rw, route=kroute, out_inner=out_inner, masks=mixed)
    r_fp32, _, _, _ = reference64(net, x, layout, rw, zsave=[z.float() for z in zs64], route=kroute, out_inner=out_inner, masks=mixed)
    kd_routed = kink_distances(net, zs64, kroute)
    info["ambiguous_routed_units"] = sum(int((k < AMBIGUOUS).sum()) for k in kd_routed)
    info["routed_units"] = sum(k.numel() for k in kd_routed)
    put("pinned_units_over_allowance", info["ambiguous_routed_units"] / max(4.0, PINNED_BAR * info["routed_units"]), 1.0)
    scale = _scales(net, r_plain)
    info["per_tensor"] = {}
    for nm in r_plain:
        got = grads[nm].double().reshape(r_plain[nm].shape)
        e_k = (got - r_kernel[nm]).abs().max().item() / scale[nm]
        e_p = (got - r_plain[nm]).abs().max().item() / scale[nm]
        e_raw = (got - r_raw[nm]).abs().max().item() / scale[nm]
        yard = (r_fp32[nm] - r_plain[nm]).abs().max().item() / scale[nm]
        fwd = (r_kernel[nm] - r_plain[nm]).abs().max().item() / scale[nm]
        bar = max(2e-4, K_YARDSTICK * yard)
        info["per_tensor"][nm] = dict(kernel=e_k, plain=e_p, raw_plain=e_raw, yardstick=yard, forward=fwd, bar=bar)
        put("bwd_vs_kernel_valued", e_k, BWD_KERNEL_BAR)
        put("bwd_vs_plain_over_bar", e_p / bar, 1.0)
    return rep, info


def _assert_report(rep, info):
    bad = {k: v for k, v in rep.items() if not v[0] <= v[1]}
    worst = {nm: d for nm, d in info.get("per_tensor", {}).items() if d["plain"] > d["bar"] or d["kernel"] > BWD_KERNEL_BAR}
    assert not bad, (bad, worst, "units pinned to the kernel's mask: %s of %s" % (info.get("ambiguous_routed_units"), info.get("routed_units")))


CASES = [
    # table, b, n, layout, signs, out_inner
    ("rec", 50, 2048, "bnc", False, 0),
    ("rec", 50, 2048, "bnc", True, 0),
    ("rec", 64, 2048, "bnc", True, 0),
    ("rec", 2, 2048, "bcn", True, 0),
    ("rec", 33, 129, "bnc", True, M_OUT),
    ("rec", 5, 31, "bnc", False, 0),
    ("rec", 8, 1, "bnc", True, 0),
    ("cls", 50, 2048, "bnc", True, 0),
    ("cls", 33, 129, "bcn", False, 0),
    ("cls", 8, 1, "bnc", True, 0),
    ("reg", 50, 2048, "bnc", True, 0),
    ("reg", 5, 31, "bnc", False, M_OUT),
]


@pytest.mark.gpu
@pytest.mark.parametrize("table,b,n,layout,signs,out_inner", CASES)
def test_per_layer_training_path_vs_float64(sb, table, b, n, layout, signs, out_inner):
    rep, info = run_case(sb, table, b, n, layout, signs, out_inner)
    if signs:
        _assert_dead_channels(info)
    _assert_report(rep, info)


def _assert_dead_channels(info):
    for key in ("dead_clouds", "dead_clouds_negative_scale"):
        dead, total = info[key]
        assert 0 < dead < total, (key, "no (cloud, channel) with a pooled value of 0, or all of them", dead, total)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,layout", [(32, 1024, "bnc"), (7, 1000, "bnc"), (16, 333, "bcn")])
def test_fused_training_path_with_negative_scales_vs_float64(sb, b, n, layout):
    """The fused path (persistent conv-stack kernel + the same backward kernels) on the registration table with BatchNorm scales < 0 and
    dead pooled channels: its own pooling of negative-scale channels and the shared pool backward.  7 x 1000 and 16 x 333 run one 64-point
    slice per CTA with a partial last slice (tests/test_write_sets.py checks that such launches write only their own buffers)."""
    rep, info = run_case(sb, "reg", b, n, layout, True, M_OUT if layout == "bnc" else 0, route="fused")
    _assert_dead_channels(info)
    _assert_report(rep, info)
