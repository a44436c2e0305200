"""The generator against float64 at last conv layers narrower than 128 channels, and at FC inputs that are not a multiple of four.

SampleNet(num_out_points, C) takes any bottleneck width C.  The persistent conv stack takes a last layer of 8 to 128 channels, the
per-layer tensor-core path one of 8 to 1024, so SampleNet(32, C) with C < 128 runs the fused kernel and its fused FC head; its training
step takes the torch route (the forward kernels, then a recompute for the backward), since the CUDA backward takes only the 128 -> 128
last pair.  The widths and what each reaches:

    C = 8     the smallest width: one 8-channel group; kr = 4 in the fused head (two K eighths of 4 columns, six empty)
    C = 40    one partly used 32-channel warp quarter in the conv stack; kr = 8 (the 4-wide loop, a last eighth of 4 columns)
    C = 64    the second 64-channel warpgroup idle; kr = 8
    C = 100   the second warpgroup partly used; kr = 16 with short eighths (eighth 6 holds 4 columns, eighth 7 none)
    C = 42    c_in & 3 = 2: scalar row staging, scalar weight staging, no weight TMA for fc1 in either head, the scalar K loop
    C = 127   c_in & 3 = 3, one channel short of the full tile

and two generic tables: "narrow8" (conv 3-32-32-8) and "narrow40" (conv 3-64-64-64-40), where a slice is parked in the weight matrix's
spare columns 64..127 (CsLayer::keep = 2) while the narrow last layer's weights are copied and zero-padded; and "unaligned" (conv ..-128-42,
FC 42-50-30-99, BatchNorm and ReLU on the first two): every FC input width is 2 mod 4 (no FC layer stages weights by TMA, in either head),
and the last 8-channel group of the 99-wide layer holds 3 channels.

Forward (GPU): test_inference_parity.run_generator_case on these nets -- out, feat and, in training mode, every BatchNorm layer's running
statistics and num_batches_tracked against float64, at that file's bars -- on every route: the default (persistent kernel and fused head,
repeated once for identical bits), the cluster head, the per-layer tensor-core kernels, the exact-fp32 CUDA-core stack and the two
stand-alone entry points.  Shapes come from snb200_debug_conv_stack_partition and each asserts its branch: one slice per CTA, two, three,
a ragged last slice with one and with three slices per CTA, one cloud (eval), and 200 clouds (the heads stage their rows in two passes).
snb200_debug_generator_plan asserts the conv path and head of every route.

Training step (GPU): SampleNet(32, C) trains on the torch route; one forward / backward of a random linear functional of the output on an
instance kept away from ReLU kinks and pooled ties, against float64 autograd of the same stack: output, every parameter gradient, the
running statistics.

CPU: the host answers at every width -- no CUDA backward, the persistent plan with the fused head, and SampleNet's route "torch"."""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_inference_parity as tip  # noqa: E402
import test_layers_training_parity as tlp  # noqa: E402
import test_sampler_training as tst  # noqa: E402
import test_write_sets as tws  # noqa: E402
from samplenet_b200 import _lib, samplenet  # noqa: E402
from samplenet_b200.samplenet import LayerTableGenerator, SampleNet  # noqa: E402

WIDTHS = (8, 40, 64, 100, 42, 127)
M = 32
# generic tables: conv widths, FC widths, FC BatchNorm, FC ReLU, sampled points (the last FC layer has 3 M outputs)
GENERIC = {
    "narrow8": ([3, 32, 32, 8], [8, 64, 96], [1, 0], [1, 0], 32),
    "narrow40": ([3, 64, 64, 64, 40], [40, 128, 96], [1, 0], [1, 0], 32),
    "unaligned": ([3, 64, 64, 64, 128, 42], [42, 50, 30, 99], [1, 1, 0], [1, 1, 0], 33),
}
TABLES = ["C%d" % c for c in WIDTHS] + sorted(GENERIC)


def widths(table):
    """(conv widths, FC widths, FC BatchNorm, FC ReLU) of a table."""
    if table in GENERIC:
        return GENERIC[table][:4]
    c = int(table[1:])
    return [3, 64, 64, 64, 128, c], [c, 256, 256, 256, 3 * M], [1, 1, 1, 0], [1, 1, 1, 0]


def make_net(table, seed):
    torch.manual_seed(seed)
    if table not in GENERIC:
        return SampleNet(M, int(table[1:]), 8, input_shape="bnc", output_shape="bnc")
    conv_w, fc_w, fc_bn, fc_relu, m = GENERIC[table]
    net = LayerTableGenerator(conv_w, fc_w, fc_bn, fc_relu, 1e-5, 0.1)
    net.num_out_points = m
    return net


def _c_tables(table):
    conv_w, fc_w, fc_bn, fc_relu = widths(table)
    return tst._table(conv_w, [1] * (len(conv_w) - 1), [1] * (len(conv_w) - 1)), tst._table(fc_w, fc_bn, fc_relu)


def _plan(lib, table, b, n, flags=0):
    """(conv path, fused head) snb200_generator_forward takes: path 0 persistent, 1 per-layer tensor-core, 2 exact fp32."""
    conv, fc = _c_tables(table)
    path, fuse = ctypes.c_int(-1), ctypes.c_int(-1)
    rc = lib.snb200_debug_generator_plan(b, n, len(conv), conv, len(fc), fc, flags, ctypes.byref(path), ctypes.byref(fuse))
    assert rc == 0, lib.snb200_last_error()
    return path.value, fuse.value


def head_rows(table):
    """Rows the fused head stages per pass (launch_conv_stack): 128 where they fit in 200 KB next to the partial sums and weight rows."""
    _, fc_w, _, _ = widths(table)
    hcmax, hcsum = max(fc_w[:-1]), sum(fc_w[:-1])
    for rs in (128, 96, 64, 32):
        if (rs * (hcmax + 1) + 2048 + 8 * hcsum) * 4 + 1024 <= 200 * 1024:
            return rs
    return 32


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _lib.lib()


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("table", TABLES)
def test_narrow_tables_take_the_persistent_plan_and_no_cuda_backward(lib, table):
    conv, fc = _c_tables(table)
    for b in (2, 4, 32, 64):
        for n in (256, 1024):
            assert lib.snb200_generator_backward_supported(b, n, len(conv), conv, len(fc), fc) == 0, (table, b, n)
            assert lib.snb200_generator_layers_backward_supported(b, n, len(conv), conv, len(fc), fc) == 0, (table, b, n)
    for b, n in ((1, 1024), (8, 1024), (32, 1024), (48, 1024), (40, 1000), (200, 1024)):
        assert _plan(lib, table, b, n) == (0, 1), (table, b, n)
        assert _plan(lib, table, b, n, _lib.GEN_SEPARATE_HEAD) == (0, 0)
        assert _plan(lib, table, b, n, _lib.GEN_PER_LAYER_KERNELS) == (1, 0)
        assert _plan(lib, table, b, n, _lib.GEN_EXACT_FP32) == (2, 0)


@pytest.mark.parametrize("c", WIDTHS)
def test_samplenet_narrow_route_is_torch(lib, monkeypatch, c):
    """SampleNet(32, C)'s training route with the library's own envelope answers (the ops wrappers need CUDA tensors, so the envelope is
    asked through the C tables of the same widths)."""
    net = SampleNet(M, c, 8)
    assert net.CUDA_ROUTES == ("fused",)
    asked = []

    def envelope(entry):
        def supported(x, layout, conv_specs, fc_specs):
            b, n = x.shape[0], x.shape[1] if layout == "bnc" else x.shape[2]
            conv = tst._table([3] + [s["weight"].shape[0] for s in conv_specs], [1] * len(conv_specs), [1] * len(conv_specs))
            fc = tst._table([c] + [s["weight"].shape[0] for s in fc_specs], [1, 1, 1, 0], [1, 1, 1, 0])
            asked.append(entry)
            return bool(getattr(lib, entry)(b, n, len(conv), conv, len(fc), fc))
        return supported
    for route, entry in (("fused", "snb200_generator_backward_supported"), ("layers", "snb200_generator_layers_backward_supported")):
        monkeypatch.setitem(samplenet._ROUTE_OPS, route, (envelope(entry),) + samplenet._ROUTE_OPS[route][1:])
    for b, n in ((4, 256), (32, 1024), (64, 1024)):
        assert net._route(torch.zeros(b, n, 3), "bnc", *net._layer_specs(), True) == "torch", (c, b, n)
    assert asked and set(asked) == {"snb200_generator_backward_supported"}


def test_head_rows_of_the_narrow_tables():
    assert all(head_rows(t) == 128 for t in TABLES)


# ------------------------------------------------------------------------------------------------------------------ GPU forward
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


# (b, n, the partition entry's answer on 132 SMs, what the case is there for)
SHAPES = {
    "b1": (1, 1024, dict(per_cta=1, partial=False)),
    "single": (8, 1024, dict(per_cta=1, partial=False)),
    "two": (32, 1024, dict(per_cta=2, partial=False)),
    "three": (48, 1024, dict(per_cta=3, partial=False)),
    "ragged1": (7, 1000, dict(per_cta=1, partial=True)),
    "ragged3": (40, 1000, dict(per_cta=3, partial=True)),
    "rows200": (200, 1024, dict(per_cta=13, partial=False)),
}


def _expect(sb, table, shape):
    b, n, want = SHAPES[shape]
    part = tws._partition(sb, b, n)
    assert {k: part[k] for k in want} == want, ("partition of %d x %d" % (b, n), part)
    if shape == "rows200":   # two staging passes of the fused head (and two or more row groups of the cluster head)
        assert head_rows(table) < b <= 2 * head_rows(table)
    return b, n, (dict(per_cta=want["per_cta"]), True)


def _run(sb, table, shape, layout, training, route, twice=False):
    b, n, expect = _expect(sb, table, shape)
    flags = {"default": 0, "separate_head": _lib.GEN_SEPARATE_HEAD, "per_layer_kernels": _lib.GEN_PER_LAYER_KERNELS,
             "exact_fp32": _lib.GEN_EXACT_FP32, "unfused": None}[route]
    if flags is not None:
        want = {"default": (0, 1), "separate_head": (0, 0), "per_layer_kernels": (1, 0), "exact_fp32": (2, 0)}[route]
        assert _plan(sb._lib.lib(), table, b, n, flags) == want, (table, b, n, route)
    rep, ratios = tip.run_generator_case(sb, table, b, n, layout, training, route, expect if route == "default" else None, make=make_net,
                                         table_persistent=True, twice=twice)
    tip._assert_report(rep, ratios)


FWD_CASES = [pytest.param(table, shape, layout, training, id="%s-%s-%s-%s" % (table, shape, layout, "train" if training else "eval"))
             for table in TABLES for shape in SHAPES for layout in ("bnc", "bcn") for training in (False, True)
             if SHAPES[shape][0] >= 2 or not training]


@pytest.mark.gpu
@pytest.mark.parametrize("table,shape,layout,training", FWD_CASES)
def test_narrow_forward_vs_float64(sb, table, shape, layout, training):
    """The default route: the persistent kernel with its fused head (one launch, asserted), a second call bit for bit."""
    _run(sb, table, shape, layout, training, "default", twice=True)


ROUTE_SHAPES = ("single", "ragged3", "rows200")
ROUTE_CASES = [pytest.param(table, shape, ("bnc", "bcn")[(i + j) % 2], training, route,
                            id="%s-%s-%s-%s" % (route, table, shape, "train" if training else "eval"))
               for i, table in enumerate(TABLES) for j, shape in enumerate(ROUTE_SHAPES)
               for route in ("separate_head", "per_layer_kernels", "exact_fp32", "unfused") for training in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("table,shape,layout,training,route", ROUTE_CASES)
def test_narrow_routes_vs_float64(sb, table, shape, layout, training, route):
    """The persistent conv stack with the cluster head, the per-layer tensor-core kernels (the tc_layer_kernel last layer with a partial
    N), the exact-fp32 CUDA-core stack and the stand-alone entry points, each against float64."""
    _run(sb, table, shape, layout, training, route)


# ------------------------------------------------------------------------------------------------------------------ GPU training step
STEP_WIDTHS = (8, 42, 64, 100, 127)
STEP_B, STEP_N = 4, 256
# an instance is used when, in its float64 forward, no conv unit's BatchNorm output is within KINK of 0, no FC BatchNorm output within
# FC_KINK of 0 (as test_gpu_parity's margin search), and no live pooled (cloud, channel) has its runner-up within TIE of the maximum
# (relative to the channel's largest |z| in the cloud): the fp32 recompute then takes float64's masks and routes.  Every point counts,
# not only the routed ones: through training-mode BatchNorm every point carries about 1 / (b n) of a layer's gradient, and at 4 x 256 a
# single flipped mask at an unrouted point moved conv layer 4's weight and shift gradients by 8e-4 of their scale (4x the bar)
KINK, FC_KINK, TIE = 3e-6, 2e-5, 1e-5


def _margins(net, x, layout):
    """(smallest conv unit |BatchNorm output|, smallest FC |BatchNorm output| ahead of a ReLU, smallest relative pooled gap)"""
    conv_specs, fc_specs = net._layer_specs()
    b = x.shape[0]
    with torch.no_grad():
        h = tlp._rows(x.double(), layout)
        us = []
        for spec in conv_specs:
            z = torch.nn.functional.linear(h, spec["weight"].double().reshape(spec["weight"].shape[0], -1), spec["bias"].double())
            u = torch.nn.functional.batch_norm(z, None, None, spec["bn"][0].double(), spec["bn"][1].double(), True, 0.0, spec["bn"][4])
            us.append(u)
            h = torch.relu(u)
        gamma = conv_specs[-1]["bn"][0].double()
        route = tlp._route(z, gamma, b)
        s = (z.view(b, -1, z.shape[1]) * torch.where(gamma >= 0, 1.0, -1.0).to(z)).sort(dim=1, descending=True)[0]
        live = torch.gather(h.view(b, -1, z.shape[1]), 1, route[:, None, :]).squeeze(1) > 0
        gap = ((s[:, 0] - s[:, 1]) / z.view(b, -1, z.shape[1]).abs().amax(dim=1))[live].min().item()
        kink = min(u.abs().min().item() for u in us)
        h = torch.gather(h.view(b, -1, h.shape[1]), 1, route[:, None, :]).squeeze(1)
        fc_kink = 1.0
        for spec in fc_specs:
            h = torch.nn.functional.linear(h, spec["weight"].double(), spec["bias"].double())
            if spec["bn"] is not None:
                h = torch.nn.functional.batch_norm(h, None, None, spec["bn"][0].double(), spec["bn"][1].double(), True, 0.0, spec["bn"][4])
            if spec["relu"]:
                fc_kink = min(fc_kink, h.abs().min().item())
                h = torch.relu(h)
    return kink, fc_kink, gap


def _step_instance(c, layout):
    for seed in range(100 + c, 160 + c):
        torch.manual_seed(seed)
        net = SampleNet(M, c, 8, input_shape=layout, output_shape=layout).cuda().train()
        with torch.no_grad():
            for p in net.parameters():
                if p.dim() == 1:
                    p.add_(0.1 * torch.randn_like(p))
            for bn in tip._bn_layers(net):
                bn.running_mean.copy_(0.1 * torch.randn_like(bn.running_mean)); bn.running_var.copy_(0.5 + torch.rand_like(bn.running_var))
        x = torch.rand(STEP_B, STEP_N, 3, device="cuda") - 0.5
        x = x if layout == "bnc" else x.permute(0, 2, 1).contiguous()
        kink, fc_kink, gap = _margins(net, x, layout)
        if kink > KINK and fc_kink > FC_KINK and gap > TIE:
            return net, x
    pytest.fail("no conditioned instance at C = %d" % c)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["bnc", "bcn"])
@pytest.mark.parametrize("c", STEP_WIDTHS)
def test_narrow_training_step_vs_float64_autograd(sb, c, layout):
    net, x = _step_instance(c, layout)
    b = x.shape[0]
    conv_specs, fc_specs = net._layer_specs()
    assert net._route(x, layout, conv_specs, fc_specs, True) == "torch"
    inner = M if layout == "bnc" else 0
    rw = torch.randn(b, 3 * M, device="cuda", generator=torch.Generator(device="cuda").manual_seed(c))
    named = net._generator_named_parameters()
    state0 = [(bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()) for bn in tip._bn_layers(net)]
    net.zero_grad()
    y = net._generate(x, layout, inner)
    (y * rw).sum().backward()
    assert net.generator_route == "torch"
    # test_layers_training_parity's end-to-end bar: per tensor max(2e-4, K_YARDSTICK * yardstick) of its scale, the yardstick being how far
    # the same graph with every conv layer's raw output rounded to fp32 lands from float64 (the scale of a tensor whose true gradient is 0
    # is its layer's weight gradient's)
    g64, route, zs64, out64 = tlp.reference64(net, x, layout, rw, out_inner=inner)
    g32, _, _, _ = tlp.reference64(net, x, layout, rw, zsave=[z.float() for z in zs64], route=route, out_inner=inner)
    scale = tlp._scales(net, g64)
    bad = {}
    yard = max((yy[0] - out64).abs().max().item() for yy in tip.yardsticks(net, x, layout, True, inner))
    err, bar = (y.detach().double() - out64).abs().max().item(), tip._bar("out", yard, out64.abs().max().item())
    if not err <= bar:
        bad["out"] = (err, bar)
    for nm, p in named:
        err = (p.grad.double().reshape(g64[nm].shape) - g64[nm]).abs().max().item() / scale[nm]
        yard = (g32[nm] - g64[nm]).abs().max().item() / scale[nm]
        if not err <= max(2e-4, tlp.K_YARDSTICK * yard):
            bad[nm] = dict(err_over_scale=err, yardstick=yard)
    _, _, pre = tip.reference64(net, x, layout, True)
    for i, (bn, z, (m0, v0, t0)) in enumerate(zip(tip._bn_layers(net), pre, state0)):
        em, ev, bmean, bstd = tlp.running_update64(m0, v0, z, bn.momentum)
        mscale = (1 - bn.momentum) * m0.double().abs() + bn.momentum * (bmean.abs() + bstd)
        e_m = ((bn.running_mean.double() - em).abs() / mscale).max().item()
        e_v = ((bn.running_var.double() - ev).abs() / ev).max().item()
        if not (e_m <= tip.RUNNING_FLOOR and e_v <= tip.RUNNING_FLOOR and int(bn.num_batches_tracked) == int(t0) + 1):
            bad["running%d" % i] = (e_m, e_v, int(bn.num_batches_tracked) - int(t0))
    assert not bad, bad
