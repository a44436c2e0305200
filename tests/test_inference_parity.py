"""The inference path against float64 and the C oracle: the generator forward in eval mode (and in training mode past 64 clouds), and the
matching that turns generated points into input points, at the batch sizes the evaluators run (up to 256 clouds per call, 300 in two).

Generator.  ops.generator_forward with no gradient against reference64: LayerTableGenerator._torch_generator's layer stack evaluated in
float64, with the pooled feature and every BatchNorm layer's input kept (the CPU tests pin it against _torch_generator on a float64 copy of
the module and against the stock torch modules, in both modes).  Shapes are chosen from snb200_debug_conv_stack_partition on the device
and each asserts the branch it reaches: one to 32 slices per CTA, 33 (the per-layer route), slices touching 8 clouds and 9 (the per-layer
route), and a cloud spanning many slices; at 129 to 256 clouds the fused FC head stages its rows in two passes.  Tables: SampleNet(64),
SampleNet(1024), ClassificationSampleNet from TF variables (BatchNorm on every FC layer, eps 1e-3, the last with BatchNorm and no ReLU) and
ReconstructionSampleNet (256-wide conv layers: the per-layer route).  Every other route (separate head, per-layer kernels, exact fp32, the
two stand-alone entry points) is held to float64 on its own.  Parameters: BatchNorm scales < 0 on a quarter of every conv layer's
channels (the pool takes the minimum there), channels pooled to 0 in some clouds, running statistics from a float64 training pass over
another batch, perturbed.  The bar of feat and out is max(K_YARDSTICK * yardstick, FLOOR * the tensor's largest entry), the yardstick
being the larger distance from the plain float64 graph of (a) one that rounds every raw layer output to fp32 and (b) the graph in stock
torch fp32 ops: how far a correct fp32 forward moves the tensor at that shape.  Running statistics use the scales of
test_layers_training_parity.RUNNING_BAR and the same two yardstick graphs.  The floors, not the yardsticks, set nearly every bar: the
3xTF32 products keep about 21 bits, not fp32's 24, so the kernels sit up to 17 yardsticks from float64 (DESIGN section 2).

Matching.  csrc/matching.cu computes what the registration and reconstruction samplers' numpy matching computes: float64 distances
from the float32 points with every square and sum rounded, the first maximum, first-occurrence unique.  It is held bit for bit, points and
indices, to oracle.nn_matching and to matching_np, a float64 numpy model of those rules (pinned against the oracle on the CPU).  Mirror-symmetric clouds (a point and its
x<->y mirror, seeded on the diagonal) have exact numpy ties at the FPS arg-max that a fused multiply-add breaks; a CPU test proves with
exact rational arithmetic that they discriminate, and another checks that the kernel's SASS has no DFMA.

The bars are the constants below, each about 10x the largest value measured over all cases on an H100 80GB HBM3 at a 700 W power limit;
the measured maxima are in brackets beside them.
"""
import copy
import hashlib
import os
import shutil
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_layers_training_parity as tlp  # noqa: E402
import test_tf_variant as ttf  # noqa: E402
import test_write_sets as tws  # noqa: E402
from samplenet_b200 import ReconstructionSampleNet, SampleNet  # noqa: E402
from samplenet_b200.tf_variant import ClassificationSampleNet  # noqa: E402

K_YARDSTICK = 4.0      # [17] feat, out, running statistics: the bar is at least this many yardsticks (measured: the largest error / yardstick)
FLOOR = {"feat": 1e-4,  # [1.05e-5] ... and at least this fraction of the tensor's largest entry
         "out": 6e-4}   # [5.9e-5]
RUNNING_FLOOR = 2e-4   # [1.8e-5] running mean / variance, scales of test_layers_training_parity.RUNNING_BAR
M = 64


# ------------------------------------------------------------------------------------------------------------------ generator reference
def reference64(net, x, layout, training, out_inner=0, fp32_raw=False, dtype=torch.float64):
    """net's layer stack in float64 (_torch_generator's arithmetic; BatchNorm with batch statistics in training mode and the running ones
    in eval mode).  fp32_raw: round every raw layer output to fp32; dtype=torch.float32: the whole graph in stock torch fp32 ops (the two
    yardstick graphs).  Returns (out, feat, the rows entering each BatchNorm layer), in float64."""
    conv_specs, fc_specs = net._layer_specs()
    b = x.shape[0]
    h = tlp._rows(x.to(dtype), layout)
    feat, pre = None, []
    for i, spec in enumerate(conv_specs + fc_specs):
        if i == len(conv_specs):
            h = feat = h.view(b, -1, h.shape[1]).max(dim=1)[0]
        w = spec["weight"].detach().to(dtype)
        h = F.linear(h, w.reshape(w.shape[0], -1), spec["bias"].detach().to(dtype))
        if fp32_raw:
            h = h.float().double()
        if spec["bn"] is not None:
            g, beta, rm, rv, eps = (t.detach().to(dtype) if torch.is_tensor(t) else t for t in spec["bn"][:5])
            pre.append(h.double())
            h = F.batch_norm(h, None if training else rm, None if training else rv, g, beta, training, 0.0, eps)
        if spec["relu"]:
            h = torch.relu(h)
    if out_inner:
        h = h.view(b, -1, out_inner).permute(0, 2, 1).reshape(b, -1)
    return h.double(), feat.double(), pre


def yardsticks(net, x, layout, training, out_inner=0):
    """The two yardstick graphs: (out, feat, BatchNorm inputs) of the float64 graph with every raw layer output rounded to fp32, and of
    stock torch fp32 ops (TF32 off).  Rounding only the raw outputs leaves out the matrix products' accumulation error, about K times one
    rounding for K terms of mixed signs; the fp32 graph has it."""
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        return (reference64(net, x, layout, training, out_inner, fp32_raw=True),
                reference64(net, x, layout, training, out_inner, dtype=torch.float32))
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32


def _seed(*key):
    return int(hashlib.sha1(repr(key).encode()).hexdigest()[:8], 16)


def make_net(table, seed, layout="bnc"):
    torch.manual_seed(seed)
    if table == "reg64":
        return SampleNet(M, 128, 8, input_shape=layout, output_shape=layout)
    if table == "reg1024":
        return SampleNet(1024, 128, 8, input_shape=layout, output_shape=layout)
    if table == "cls":
        return ClassificationSampleNet.from_tf_variables(ttf.make_tf_variables(seed, m=M))
    return ReconstructionSampleNet(M)


def _bn_layers(net):
    return [bn for _, bn in net._convs() + net._fcs() if bn is not None]


def condition(net, x, layout, training, seed):
    """A case's parameters.  About a quarter of every conv layer's channels get a BatchNorm scale < 0 and every 8th channel of the inner
    conv layers a shift of -1.5; the running statistics are the batch statistics of a float64 training pass over another batch of 64
    clouds, perturbed (means by 0.1 std, variances by up to 20 %), so that eval-mode activations are of order 1; and with two clouds or
    more, channels 5 + 8 k (scale > 0) and 4 + 16 k (scale < 0) of the last conv layer get the shift that puts the pooled value after
    BatchNorm + ReLU at 0 in some clouds and not in others, in the mode the case runs.  Returns those channels."""
    g = torch.Generator().manual_seed(seed)
    convs = net._convs()
    with torch.no_grad():
        for l, (lin, bn) in enumerate(convs):
            lin.bias.add_(0.1 * torch.randn(lin.bias.shape, generator=g).to(lin.bias))
            if not isinstance(net, ClassificationSampleNet):
                bn.weight.add_(0.1 * torch.randn(bn.weight.shape, generator=g).to(bn.weight))
                bn.bias.add_(0.1 * torch.randn(bn.bias.shape, generator=g).to(bn.bias))
            bn.weight[(l % 4)::4] = -bn.weight[(l % 4)::4].abs()
            if l + 1 < len(convs):
                bn.bias[3::8] = -1.5
        other = (torch.rand(64, x.shape[1] if layout == "bnc" else x.shape[2], 3, generator=g) - 0.5).to(x.device)
        _, _, pre = reference64(net, other, "bnc", True)
        for bn, z in zip(_bn_layers(net), pre):
            mean, var = z.mean(0), z.var(0, unbiased=False)
            mean = mean + 0.1 * var.sqrt() * torch.randn(mean.shape, generator=g, dtype=torch.float64).to(mean)
            var = var * (0.8 + 0.4 * torch.rand(var.shape, generator=g, dtype=torch.float64).to(var)) + 1e-6
            bn.running_mean.copy_(mean); bn.running_var.copy_(var)
        b = x.shape[0]
        if b < 2:
            return []
        _, _, pre = reference64(net, x, layout, training)
        bn = convs[-1][1]
        z = pre[len(convs) - 1]
        mean, var = (z.mean(0), z.var(0, unbiased=False)) if training else (bn.running_mean.double(), bn.running_var.double())
        peak = ((z - mean) / torch.sqrt(var + bn.eps) * bn.weight.double()).view(b, -1, z.shape[1]).max(dim=1)[0]
        dead = sorted(set(range(5, z.shape[1], 8)) | set(range(4, z.shape[1], 16)))
        for c in dead:
            s = peak[:, c].sort()[0]
            lo, hi = max(0, b // 4 - 1), max(1, (3 * b) // 4)
            j = max(range(lo, min(hi, b - 1)), key=lambda k: (s[k + 1] - s[k]).item())
            bn.bias[c] = float(-(s[j] + s[j + 1]) / 2)
    return dead


# ------------------------------------------------------------------------------------------------------------------ matching reference
def sq_dist64(cloud64, q):
    """Squared distances in float64 from the point q to every row of cloud64, with numpy's rounding of a sum of squares over the last axis:
    each square rounded, then (x + y) + z."""
    e = (cloud64 - q) ** 2
    return (e[:, 0] + e[:, 1]) + e[:, 2]


def first_occurrences(seq):
    """The distinct entries of seq, in the order in which each first appears."""
    return list(dict.fromkeys(int(v) for v in seq))


def match_one(cloud, nn_idx, k):
    """Indices of one cloud's k matched points: the distinct nearest-neighbour indices in order of first appearance (a single one stays
    first), then farthest points from everything chosen so far, by float64 distance from the float32 coordinates, the lowest index on a
    tie."""
    c64 = cloud.astype(np.float64)
    chosen = first_occurrences(nn_idx)[:k]
    gap = np.full(len(c64), np.inf)
    for i in chosen:
        gap = np.minimum(gap, sq_dist64(c64, c64[i]))
    while len(chosen) < k:
        far = int(np.argmax(gap))          # np.argmax: the first of equal maxima
        chosen.append(far)
        gap = np.minimum(gap, sq_dist64(c64, c64[far]))
    return np.array(chosen, dtype=np.int64)


def matching_np(clouds, nn_idx, k, complete_fps=True):
    """The matching in numpy, float64: (matched points (B, k, 3), their indices (B, k), distinct nearest-neighbour indices per cloud (B,)).
    Without complete_fps the first k nearest-neighbour indices are taken as they are."""
    idx = nn_idx[:, :k].astype(np.int64) if not complete_fps else np.stack([match_one(c, i, k) for c, i in zip(clouds, nn_idx)])
    pts = np.take_along_axis(clouds, idx[..., None].repeat(3, -1), axis=1).astype(np.float64)
    return pts, idx, np.array([len(first_occurrences(i)) for i in nn_idx])


def symmetric_clouds(count, seed=0):
    """(count, 81, 3) float32: a seed point on the diagonal x = y, 40 random points with y scaled by 1e-3 (so that squared differences
    need more than 26 bits) and their x<->y mirrors.  In numpy a point and its mirror are exactly equidistant from the seed."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        half = rng.random((40, 3)) - 0.5
        half[:, 1] *= 1e-3
        half = half.astype(np.float32)
        diag = (rng.random((1, 3)) - 0.5).astype(np.float32)
        diag[0, 1] = diag[0, 0]
        out.append(np.concatenate([diag, half, half[:, [1, 0, 2]]]))
    return np.stack(out)


def matching_case(name):
    """(cloud (B, N, 3) float32, nearest-neighbour indices (B, k) int32, k, complete_fps) of a named case."""
    r = np.random.default_rng(_seed("matching", name))
    if name == "sym":
        pc = symmetric_clouds(64)
        return pc, np.zeros((64, 8), np.int32), 8, True
    b, n, k = {"b256": (256, 1024, 64), "order1024": (3, 1024, 1024), "order2048": (2, 2048, 2048), "one_seed": (8, 1024, 64),
               "few_seeds": (8, 1024, 200), "duplicates": (4, 1024, 200), "no_fps": (16, 1024, 48)}[name]
    pc = (r.random((b, n, 3)) - 0.5).astype(np.float32)
    idx = r.integers(0, n, size=(b, k)).astype(np.int32)
    if name == "one_seed":
        idx[:] = r.integers(0, n, size=(b, 1))
    elif name == "few_seeds":
        idx = np.take_along_axis(r.integers(0, n, size=(b, 3)), r.integers(0, 3, size=(b, k)), axis=1).astype(np.int32)
    elif name == "duplicates":     # 128 distinct points, each 8 times: FPS runs out of positive distances after 128 points
        pc = np.tile(pc[:, :128], (1, 8, 1))
        idx[:, 4:] = idx[:, :1]
    return pc, idx, k, name != "no_fps"


MATCHING_CASES = ["b256", "order1024", "order2048", "one_seed", "few_seeds", "duplicates", "no_fps", "sym"]


# ------------------------------------------------------------------------------------------------------------------ CPU pins
def _stock_forward(net64, x, training):
    """The float64 module's own submodules on a (B, 3, N) input: Conv1d, BatchNorm1d (updating its running statistics in training
    mode), ReLU, max over the points, Linear.  Returns (out, feat)."""
    net64.train(training)
    h = x.permute(0, 2, 1)
    for conv, bn in net64._convs():
        h = torch.relu(bn(conv(h)))
    feat = h = h.max(dim=2)[0]
    for (fc, bn), relu in zip(net64._fcs(), net64.fc_relu):
        h = fc(h)
        h = bn(h) if bn is not None else h
        h = torch.relu(h) if relu else h
    return h, feat


@pytest.mark.parametrize("table", ["reg64", "reg1024", "cls", "rec"])
@pytest.mark.parametrize("training", [False, True])
def test_reference64_is_the_float64_torch_generator(table, training):
    b, n = 5, 37
    net = make_net(table, 3)
    x = torch.rand(b, n, 3, generator=torch.Generator().manual_seed(4), dtype=torch.float64) - 0.5
    dead = condition(net, x.float(), "bnc", training, 5)
    net64 = copy.deepcopy(net).double()
    out, feat, pre = reference64(net, x, "bnc", training)
    ps = {nm: p for nm, p in net64._generator_named_parameters()}
    with torch.no_grad():
        y = net64._torch_generator(x, "bnc", training, ps)
        state0 = [(bn.running_mean.clone(), bn.running_var.clone()) for bn in _bn_layers(net64)]
        y_stock, feat_stock = _stock_forward(net64, x, training)
    assert (out - y).abs().max().item() <= 1e-12 * y.abs().max().item()
    assert (out - y_stock).abs().max().item() <= 1e-12 * y.abs().max().item()
    assert (feat - feat_stock).abs().max().item() <= 1e-12 * feat.abs().max().item()
    for bn, z, (m0, v0) in zip(_bn_layers(net64), pre, state0):
        if training:   # the rows reference64 keeps are what BatchNorm1d normalised: its running update is running_update64 of them
            em, ev, _, _ = tlp.running_update64(m0, v0, z, bn.momentum)
            assert torch.allclose(bn.running_mean, em, rtol=1e-12, atol=1e-14) and torch.allclose(bn.running_var, ev, rtol=1e-12, atol=1e-14)
        else:
            assert torch.equal(bn.running_mean, m0) and torch.equal(bn.running_var, v0)
    # the case construction: dead channels pooled to 0 in some clouds but not all, negative scales pooled at the minimum
    z = feat[:, dead]
    assert 0 < int((z == 0).sum()) < z.numel()
    neg = [c for c in dead if net._convs()[-1][1].weight[c] < 0]
    assert neg and 0 < int((feat[:, neg] == 0).sum()) < feat[:, neg].numel()
    if not training:
        assert 0.05 < out.abs().mean().item() < 20.0   # eval-mode activations of order 1
    # the yardstick graph differs from the plain one by fp32 rounding
    out32, _, _ = reference64(net, x, "bnc", training, fp32_raw=True)
    assert 0 < (out32 - out).abs().max().item() < 1e-4 * out.abs().max().item()


def test_matching_reference_is_the_oracle(oracle):
    """matching_np against the C oracle on every matching case that fits the CPU quickly, the symmetric clouds included: points exactly,
    the count of distinct seeds, and a single seed kept as the first index."""
    for name in ["sym", "one_seed", "few_seeds", "duplicates", "no_fps", "order1024"]:
        pc, idx, k, complete = matching_case(name)
        out, oi, nu = matching_np(pc, idx, k, complete)
        assert np.array_equal(out, oracle.nn_matching(pc, idx, k, complete)), name
        assert np.array_equal(nu, [len(np.unique(i)) for i in idx]), name
    pc, idx, k, _ = matching_case("one_seed")
    oi = matching_np(pc, idx, k)[1]
    assert np.array_equal(oi[:, 0], idx[:, 0]) and (oi[:, 1:] != oi[:, :1]).all()


def _fps_exact(pc, k, dist):
    """FPS from seed 0 to k points with the squared distance `dist`; returns (selected indices, at each step the indices tied at the
    maximum)."""
    n = len(pc)
    dmin = [dist(pc[0], pc[p]) for p in range(n)]
    sel, ties = [0], []
    while len(sel) < k:
        top = max(dmin)
        ties.append([p for p in range(n) if dmin[p] == top])
        sel.append(ties[-1][0])
        dmin = [min(dmin[p], dist(pc[sel[-1]], pc[p])) for p in range(n)]
    return sel, ties


def _d_rounded(s, p):       # numpy: every square and sum rounded, (dx^2 + dy^2) + dz^2
    dx, dy, dz = s[0] - p[0], s[1] - p[1], s[2] - p[2]
    return dx * dx + dy * dy + dz * dz


def _d_contracted(s, p):    # nvcc's contraction: fma(dz, dz, fma(dy, dy, dx * dx)), each fma rounded once
    dx, dy, dz = s[0] - p[0], s[1] - p[1], s[2] - p[2]
    inner = float(Fraction(dy) * Fraction(dy) + Fraction(dx * dx))
    return float(Fraction(dz) * Fraction(dz) + Fraction(inner))


def test_symmetric_clouds_discriminate_the_contraction():
    """At least one symmetric cloud has an exact numpy tie at an FPS arg-max that the contracted arithmetic breaks the other way, so a
    kernel that contracts fails the matching checks on them."""
    pc, _, k, _ = matching_case("sym")
    broken = 0
    for cloud in pc.astype(np.float64):
        pts = [tuple(map(float, row)) for row in cloud]
        sel, ties = _fps_exact(pts, k, _d_rounded)
        sel_c, _ = _fps_exact(pts, k, _d_contracted)
        if sel_c != sel:
            i = next(j for j in range(k) if sel[j] != sel_c[j])
            if len(ties[i - 1]) > 1 and sel_c[i] in ties[i - 1]:
                broken += 1
    assert broken >= 1


def _cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return exe if os.path.exists(exe) else None


def _lib_path():
    from samplenet_b200 import _lib

    return _lib.LIB_PATH


@pytest.mark.skipif(not os.path.exists(_lib_path()), reason="libsamplenet_b200.so has not been built")
@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump is not available")
def test_nn_matching_kernel_has_no_fma():
    """nn_matching_kernel rounds every square and sum of its float64 distances (no DFMA in its SASS), as numpy does."""
    sass = subprocess.run([_cuobjdump(), "-sass", _lib_path()], capture_output=True, text=True, check=True).stdout
    funcs = [f for f in sass.split("Function : ")[1:] if f.split()[0].startswith("_ZN3snb18nn_matching_kernel")]
    assert len(funcs) == 1
    assert funcs[0].count("DMUL") >= 6 and "DFMA" not in funcs[0]


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


# (b, n, the partition entry's answer on 132 SMs, persistent).  seg: clouds one slice may touch, (ppc - 1) / n + 2 (at most 8).
SHAPES = [
    (1, 1024, dict(per_cta=1, ppc=64), True),
    (2, 1024, dict(per_cta=1, ppc=64), True),
    (32, 1024, dict(per_cta=2), True),
    (33, 1024, dict(per_cta=2), True),
    (64, 1024, dict(per_cta=4), True),
    (65, 1024, dict(per_cta=4), True),
    (128, 1024, dict(per_cta=8), True),
    (129, 1024, dict(per_cta=8), True),
    (200, 1024, dict(per_cta=13), True),
    (256, 1024, dict(per_cta=16), True),
    (256, 2048, dict(per_cta=32), True),
    (256, 2112, dict(per_cta=32), True),
    (256, 2113, dict(per_cta=33), False),
    (256, 10, dict(seg=8, per_cta=1), True),
    (256, 9, dict(seg=9, per_cta=1), False),
    (8, 5000, dict(per_cta=3, ppc=128), True),
]
TABLES = ["reg64", "reg1024", "cls", "rec"]
PERSISTENT_TABLE = {"reg64": True, "reg1024": True, "cls": True, "rec": False}   # rec: 256-wide conv layers
ROUTES = {"default": {}, "separate_head": dict(separate_head=True), "per_layer_kernels": dict(per_layer_kernels=True),
          "exact_fp32": dict(exact_fp32=True), "unfused": None}


def _partition(sb, b, n):
    part = tws._partition(sb, b, n)
    part["seg"] = (part["ppc"] - 1) // n + 2
    return part


def _bar(key, yard, scale):
    return max(K_YARDSTICK * yard, FLOOR[key] * scale)


# Training mode on two clouds: an FC BatchNorm channel is +-1 times its scale, plus its shift, unless the two rows nearly coincide, where
# the output moves by up to 1 / (2 sqrt(eps)) times their difference's error.  The kernel's pooled feature is within 1e-5 of its scale
# of float64 there as everywhere, yet the output lands up to 13 yardsticks (2.6e-3 of its scale) away and the FC layers' running means
# up to 2x their bar; the output and the FC layers' running statistics are not compared below three rows (as in test_gpu_parity).
FC_WELL_CONDITIONED_ROWS = 3


def run_generator_case(sb, table, b, n, layout, training, route="default", expect=None, make=None, table_persistent=None, twice=False):
    """One generator call against float64.  Returns {check: (largest measured value, bar)} and the measured ratios.  make(table, seed):
    the net (default make_net); table_persistent: whether the persistent kernel takes the table (default PERSISTENT_TABLE); twice: run
    the call a second time from the same running statistics and require the same bits (outputs and statistics)."""
    dev = "cuda"
    seed = _seed(table, b, n, layout, training)
    net = (make or make_net)(table, seed).to(dev)
    x = (torch.rand(b, n, 3, generator=torch.Generator().manual_seed(seed)) - 0.5).to(dev)
    x = x if layout == "bnc" else x.permute(0, 2, 1).contiguous()
    dead = condition(net, x, layout, training, seed + 1)
    conv_specs, fc_specs = net._layer_specs()
    inner = net.num_out_points if layout == "bnc" else 0
    part = _partition(sb, b, n)
    persistent = part["per_cta"] <= 32 and part["seg"] <= 8 and part["grid"] <= 255
    if expect is not None:
        assert {k: part[k] for k in expect[0]} == expect[0] and persistent == expect[1], ("partition of %d x %d" % (b, n), part)
    state0 = [(bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()) for bn in _bn_layers(net)]
    def call():
        with torch.no_grad():
            if route == "unfused":
                return sb.ops.generator_forward_unfused(x, layout, conv_specs, fc_specs, training, inner)
            return sb.ops.generator_forward(x, layout, conv_specs, fc_specs, training, inner, **ROUTES[route])

    def restore():
        for bn, (m0, v0, t0) in zip(_bn_layers(net), state0):
            bn.running_mean.copy_(m0); bn.running_var.copy_(v0); bn.num_batches_tracked.copy_(t0)

    launches = sb._lib.launch_count()
    out, feat = call()
    torch.cuda.synchronize()
    launches = sb._lib.launch_count() - launches
    if route == "default":   # the persistent kernel runs the whole generator in one launch, the per-layer route in one per layer and more
        pt = PERSISTENT_TABLE[table] if table_persistent is None else table_persistent
        assert (launches == 1) == (persistent and pt), (launches, persistent, table)
    state1 = [(bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()) for bn in _bn_layers(net)]
    same = True
    if twice:
        restore()
        out2, feat2 = call()
        same = torch.equal(out, out2) and torch.equal(feat, feat2) and all(
            torch.equal(bn.running_mean, m1) and torch.equal(bn.running_var, v1) and torch.equal(bn.num_batches_tracked, t1)
            for bn, (m1, v1, t1) in zip(_bn_layers(net), state1))
    restore()
    out64, feat64, pre64 = reference64(net, x, layout, training, inner)
    yards = yardsticks(net, x, layout, training, inner)
    rep, ratios = {}, {}

    def put(key, val, bar):
        old = rep.get(key, (0.0, bar))
        rep[key] = (val, bar) if val / max(bar, 1e-300) > old[0] / max(old[1], 1e-300) or (val > 0 and bar == 0) else old

    if twice:
        put("second_call_differs", float(not same), 0.0)
    for i, (key, got, ref) in enumerate((("feat", feat, feat64), ("out", out, out64))):
        err = (got.double() - ref).abs().max().item()
        yard = max((y[1 - i] - ref).abs().max().item() for y in yards)
        scale = ref.abs().max().item()
        if key == "out" and training and b == 2:   # BatchNorm over two rows: see FC_WELL_CONDITIONED_ROWS
            continue
        put(key, err, _bar(key, yard, scale))
        ratios[key] = dict(err_over_scale=err / scale, err_over_yardstick=err / max(yard, 1e-300), yardstick_over_scale=yard / scale)
    if dead:
        z = feat64[:, dead]
        put("dead_channels_pooled_to_0_in_some_clouds", float(not 0 < int((z == 0).sum()) < z.numel()), 0.0)
    ratios["running"] = 0.0
    for l, (bn, z, (m0, v0, t0), (m1, v1, t1)) in enumerate(zip(_bn_layers(net), pre64, state0, state1)):
        if training and b < FC_WELL_CONDITIONED_ROWS and l >= len(conv_specs):
            continue
        if not training:
            put("eval_leaves_running_statistics", float(not (torch.equal(m0, m1) and torch.equal(v0, v1) and torch.equal(t0, t1))), 0.0)
            continue
        mom = bn.momentum
        em, ev, bmean, bstd = tlp.running_update64(m0, v0, z, mom)
        mscale = (1 - mom) * m0.double().abs() + mom * (bmean.abs() + bstd)
        e_m = ((m1.double() - em).abs() / mscale).max().item()
        e_v = ((v1.double() - ev).abs() / ev).max().item()
        yard_m = yard_v = 0.0
        for y in yards:
            ym, yv, _, _ = tlp.running_update64(m0, v0, y[2][l], mom)
            yard_m = max(yard_m, ((ym - em).abs() / mscale).max().item())
            yard_v = max(yard_v, ((yv - ev).abs() / ev).max().item())
        put("running_mean", e_m, max(RUNNING_FLOOR, K_YARDSTICK * yard_m))
        put("running_var", e_v, max(RUNNING_FLOOR, K_YARDSTICK * yard_v))
        put("num_batches_tracked", float(int(t1) != int(t0) + 1), 0.0)
        ratios["running"] = max(ratios["running"], e_m, e_v)
    return rep, ratios


def _assert_report(rep, ratios):
    bad = {k: v for k, v in rep.items() if not v[0] <= v[1]}
    assert not bad, (bad, ratios)


GEN_CASES = [pytest.param(table, b, n, layout, training, (expect, pers), id="%s-%dx%d-%s-%s" % (table, b, n, layout, "train" if training else "eval"))
             for (b, n, expect, pers) in SHAPES for table in TABLES for layout in ("bnc", "bcn") for training in (False, True)
             if b >= 2 or not training]


@pytest.mark.gpu
@pytest.mark.parametrize("table,b,n,layout,training,expect", GEN_CASES)
def test_generator_forward_vs_float64(sb, table, b, n, layout, training, expect):
    """The default route: the persistent kernel where the partition allows it, the per-layer route elsewhere (asserted)."""
    _assert_report(*run_generator_case(sb, table, b, n, layout, training, "default", expect))


ROUTE_CASES = [pytest.param(("reg64", "cls")[i % 2], b, n, ("bnc", "bcn")[(i // 2) % 2], training, route,
                            id="%s-%s-%dx%d-%s" % (route, ("reg64", "cls")[i % 2], b, n, "train" if training else "eval"))
               for i, (b, n, _, pers) in enumerate(SHAPES) if pers for route in ROUTES if route != "default" for training in (False, True)
               if b >= 2 or not training]


@pytest.mark.gpu
@pytest.mark.parametrize("table,b,n,layout,training,route", ROUTE_CASES)
def test_generator_routes_vs_float64(sb, table, b, n, layout, training, route):
    """The persistent conv stack with the cluster head, the per-layer tensor-core kernels, the exact-fp32 CUDA-core stack and the
    stand-alone encoder + FC-head entry points, each against float64 at the persistent kernel's shapes."""
    _assert_report(*run_generator_case(sb, table, b, n, layout, training, route))


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("name", MATCHING_CASES)
def test_nn_matching_vs_oracle(sb, oracle, name):
    """ops.nn_matching, points bit for bit against the oracle and indices against matching_np; the continued FPS against matching_np."""
    pc, idx, k, complete = matching_case(name)
    want = oracle.nn_matching(pc, idx, k, complete)
    out, oi = sb.ops.nn_matching(_t(pc), _t(idx, torch.int32), k, complete_fps=complete, return_idx=True)
    out, oi = out.cpu().numpy(), oi.cpu().numpy()
    assert np.array_equal(out.astype(np.float64), want)
    assert np.array_equal(np.take_along_axis(pc, oi[..., None].astype(np.int64).repeat(3, -1), axis=1), out)
    if not complete:
        assert np.array_equal(oi, idx[:, :k])
        return
    ref_pc, ref_idx, ref_nu = matching_np(pc, idx, k)
    assert np.array_equal(oi, ref_idx)
    got_pc, got_idx, got_nu = sb.sputils.simple_projection_and_continued_fps(_t(pc), _t(pc[:, :k]), _t(idx, torch.int32))
    assert np.array_equal(got_pc.cpu().numpy().astype(np.float64), ref_pc)
    assert np.array_equal(got_idx.cpu().numpy(), ref_idx)
    assert np.array_equal(got_nu.cpu().numpy()[:, 0], ref_nu)


def _generated_vs_float64(net, x, layout, simp, out_view):
    """(error, bar) of the generated points against the float64 generator on the same parameters."""
    out64, _, _ = reference64(net, x, layout, False)
    ref = out_view(out64)
    err = (simp.double() - ref).abs().max().item()
    return err, _bar("out", max((out_view(y[0]) - ref).abs().max().item() for y in yardsticks(net, x, layout, False)), ref.abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("b,layout", [(256, "bnc"), (300, "bcn")])
def test_samplenet_eval_end_to_end(sb, oracle, b, layout):
    """SampleNet(64).eval()(x) (300 clouds: two generator calls): simp within the generator bar of float64, match exactly the oracle's
    matching of the nearest input points of the kernel's own simp (nn_distance in the library's default, contracted, arithmetic)."""
    seed = _seed("samplenet", b, layout)
    net = make_net("reg64", seed, layout).cuda()
    x_bnc = (torch.rand(b, 1024, 3, generator=torch.Generator().manual_seed(seed)) - 0.5).cuda()
    x = x_bnc if layout == "bnc" else x_bnc.permute(0, 2, 1).contiguous()
    condition(net, x, layout, False, seed + 1)
    net.eval()
    with torch.no_grad():
        simp, match = net(x)
    simp_bnc = simp if layout == "bnc" else simp.permute(0, 2, 1)
    match_bnc = match if layout == "bnc" else match.permute(0, 2, 1)
    err, bar = _generated_vs_float64(net, x, layout, simp_bnc, lambda o: o.view(b, 3, M).permute(0, 2, 1))
    assert err <= bar, (err, bar)
    xs, ss = x_bnc.cpu().numpy(), simp_bnc.contiguous().cpu().numpy()
    want = oracle.nn_matching(xs, oracle.nn_distance(ss, xs, contract=True)[1], M)
    assert np.array_equal(match_bnc.cpu().numpy().astype(np.float64), want)


@pytest.mark.gpu
@pytest.mark.parametrize("table,b,n", [("cls", 256, 1024), ("rec", 50, 2048)])
def test_sampler_eval_end_to_end(sb, oracle, table, b, n):
    """ClassificationSampleNet and ReconstructionSampleNet in eval mode, checked the same way; the reconstruction sampler's continued FPS
    against matching_np."""
    seed = _seed("sampler", table, b, n)
    net = make_net(table, seed).cuda()
    x = (torch.rand(b, n, 3, generator=torch.Generator().manual_seed(seed)) - 0.5).cuda()
    condition(net, x, "bnc", False, seed + 1)
    net.eval()
    with torch.no_grad():
        simp, match = net(x)
    err, bar = _generated_vs_float64(net, x, "bnc", simp, lambda o: o.view(b, -1, 3))
    assert err <= bar, (err, bar)
    xs, ss = x.cpu().numpy(), simp.contiguous().cpu().numpy()
    nn_idx = oracle.nn_distance(ss, xs, contract=True)[1]
    want = oracle.nn_matching(xs, nn_idx, M) if table == "cls" else matching_np(xs, nn_idx, M)[0]
    assert np.array_equal(match.cpu().numpy().astype(np.float64), want)
