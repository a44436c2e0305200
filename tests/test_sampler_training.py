"""Training the reconstruction and classification samplers on the per-layer CUDA path.

CPU: the host answers of the four snb200_generator_layers_* entry points (envelope, workspace sizes, rejections) on fake layer tables
that are never dereferenced.  GPU: the per-layer training forward against generator_forward(training, per-layer kernels), its backward
against float64 autograd, and whole ReconstructionStep / ClassificationStep steps on the new modules against the torch recompute."""
import copy
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BNC = 0
EXACT_FP32, PER_LAYER, PRIMED = 1, 8, 32
M3 = 192

_next_ptr = [0x40000]


def _ptr():
    _next_ptr[0] += 0x1000
    return _next_ptr[0]


def _table(widths, bn, relu, eps=1e-5, momentum=0.1):
    from samplenet_b200._lib import Layer
    arr = (Layer * (len(widths) - 1))()
    for i in range(len(widths) - 1):
        L = arr[i]
        L.c_in, L.c_out = widths[i], widths[i + 1]
        L.weight, L.bias = _ptr(), _ptr()
        if bn[i]:
            L.bn_weight, L.bn_bias, L.bn_running_mean, L.bn_running_var, L.bn_num_batches_tracked = _ptr(), _ptr(), _ptr(), _ptr(), _ptr()
            L.bn_eps, L.bn_momentum = eps, momentum
        L.relu = int(relu[i])
    return arr


# the three samplers' layer tables: reconstruction (FC without BatchNorm, 3 FC layers), classification (fc14b: BatchNorm, no ReLU),
# registration
TABLE_WIDTHS = {
    "reconstruction": ([3, 64, 128, 128, 256, 128], [128, 256, 256, M3], [0, 0, 0], [1, 1, 0], 1e-5),
    "classification": ([3, 64, 64, 64, 128, 128], [128, 256, 256, 256, M3], [1, 1, 1, 1], [1, 1, 1, 0], 1e-3),
    "registration": ([3, 64, 64, 64, 128, 128], [128, 256, 256, 256, M3], [1, 1, 1, 0], [1, 1, 1, 0], 1e-5),
}


def _tables(name, conv_widths=None, conv_relu=None):
    cw, fw, fbn, frelu, eps = TABLE_WIDTHS[name]
    cw = conv_widths or cw
    conv = _table(cw, [1] * (len(cw) - 1), conv_relu or [1] * (len(cw) - 1), eps)
    fc = _table(fw, fbn, frelu, eps)
    return conv, fc


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


@pytest.mark.parametrize("name", sorted(TABLE_WIDTHS))
def test_layers_envelope_and_workspace(lib, name):
    for n in (777, 2048):
        for b in (1, 2, 50, 64, 65):
            conv, fc = _tables(name)
            sup = lib.snb200_generator_layers_backward_supported(b, n, len(conv), conv, len(fc), fc)
            assert sup == int(2 <= b <= 64), (name, b, n, sup)
            ws = lib.snb200_generator_layers_backward_workspace_bytes(b, n, len(conv), conv, len(fc), fc)
            assert ws > 0, (name, b, n)
            # one backward, one workspace layout: the per-layer entry sizes it as the fused one does, wherever the fused path applies or not
            assert ws == lib.snb200_generator_backward_workspace_bytes(b, n, len(conv), conv, len(fc), fc), (name, b, n)
    # the fused envelope excludes the reconstruction and classification tables, and keeps the registration one
    conv, fc = _tables(name)
    assert lib.snb200_generator_backward_supported(32, 1024, 5, conv, len(fc), fc) == int(name == "registration")


@pytest.mark.parametrize("name", sorted(TABLE_WIDTHS))
def test_layers_envelope_rejects(lib, name):
    conv, fc = _tables(name, conv_relu=[1, 1, 0, 1, 1])     # a conv layer without ReLU
    assert lib.snb200_generator_layers_backward_supported(32, 1024, 5, conv, len(fc), fc) == 0
    conv, fc = _tables(name, conv_widths=[3, 64, 128, 256, 256, 128])   # a (256, 256) pair
    assert lib.snb200_generator_layers_backward_supported(32, 1024, 5, conv, len(fc), fc) == 0
    conv, fc = _tables(name)
    fc[len(fc) - 1].relu = 1                                 # ReLU on the output layer: its mask would need `out`
    assert lib.snb200_generator_layers_backward_supported(32, 1024, 5, conv, len(fc), fc) == 0


def _mutate(a, kind):
    if kind == "b65":
        a["b"] = 65
    elif kind == "b1":
        a["b"] = 1
    elif kind == "no_relu":
        a["conv"][2].relu = 0
    elif kind == "pair256":
        a["conv"], _ = _tables("reconstruction", conv_widths=[3, 64, 128, 256, 256, 128])
    elif kind == "fc_null":
        a["fc"] = None
    elif kind == "layout":
        a["layout"] = 7
    elif kind == "transpose_inner":
        a["oti"] = 5
    elif kind == "transpose_inner_negative":
        a["oti"] = -3
    elif kind == "zsave_entry_null":
        a["zsave"][3] = None
    elif kind == "flag_per_layer":
        a["flags"] = PER_LAYER
    elif kind == "flag_exact_fp32":
        a["flags"] = EXACT_FP32 | PRIMED
    else:
        raise AssertionError(kind)


# (entry, bad argument) -> return code: -1 SNB200_EINVAL, -2 SNB200_EWORKSPACE
_COMMON = {"b65": -1, "b1": -1, "no_relu": -1, "pair256": -1, "fc_null": -1, "layout": -1, "zsave_entry_null": -1, "workspace_short": -2,
           "transpose_inner": -1, "transpose_inner_negative": -1}
EXPECTED_RC = {"generator_layers_train_forward": dict(_COMMON, flag_per_layer=-1, flag_exact_fp32=-1), "generator_layers_backward": dict(_COMMON)}


def _call(lib, entry, a):
    from samplenet_b200._lib import LayerGrad
    nconv = 5
    nfc = 0 if a["fc"] is None else len(a["fc"])
    if entry == "generator_layers_train_forward":
        return lib.snb200_generator_layers_train_forward(a["b"], a["n"], a["layout"], _ptr(), nconv, a["conv"], nfc, a["fc"], _ptr(), a["oti"], _ptr(), a["zsave"],
                                                         a["flags"], a["ws"], a["wsb"], None)
    gconv, gfc = (LayerGrad * 9)(), (LayerGrad * 9)()
    return lib.snb200_generator_layers_backward(a["b"], a["n"], a["layout"], _ptr(), nconv, a["conv"], nfc, a["fc"], a["zsave"], _ptr(), _ptr(), a["oti"],
                                                gconv, gfc, a["ws"], a["wsb"], None)


@pytest.mark.parametrize("entry", sorted(EXPECTED_RC))
@pytest.mark.parametrize("name", ["reconstruction", "classification"])
def test_layers_rejections(lib, entry, name):
    for kind, want in EXPECTED_RC[entry].items():
        conv, fc = _tables(name)
        a = dict(b=32, n=1024, layout=BNC, conv=conv, fc=fc, oti=0, flags=0, ws=None, wsb=0, zsave=(ctypes.c_void_p * 5)(*[_ptr() for _ in range(5)]))
        if kind == "workspace_short":
            f = lib.snb200_generator_workspace_bytes if entry.endswith("forward") else lib.snb200_generator_layers_backward_workspace_bytes
            a.update(ws=_ptr(), wsb=f(32, 1024, 5, conv, len(fc), fc) - 1)
        else:
            _mutate(a, kind)
        rc = _call(lib, entry, a)
        msg = lib.snb200_last_error().decode()
        assert rc == want, (entry, kind, rc, msg)
        assert msg.startswith(entry + ":"), (entry, kind, msg)


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _module(sb, name, m=64):
    if name == "reconstruction":
        return sb.ReconstructionSampleNet(m)
    if name == "classification":
        return sb.ClassificationSampleNet(m)
    from samplenet_b200.samplenet import LayerTableGenerator
    return LayerTableGenerator([3, 64, 64, 64, 128, 128], [128, 256, 256, 256, 3 * m], [1, 1, 1, 0], [1, 1, 1, 0], 1e-5, 0.1)


def _cloud(b, n, layout, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(b, n, 3, generator=g) - 0.5).cuda()
    return x.permute(0, 2, 1).contiguous() if layout == "bcn" else x


def _bn_state(net):
    return [t.clone() for nm, t in net.state_dict().items() if "running" in nm or "num_batches" in nm]


@pytest.mark.gpu
@pytest.mark.parametrize("name,b,n,layout", [("reconstruction", 50, 2048, "bnc"), ("reconstruction", 2, 777, "bcn"), ("classification", 32, 1024, "bnc")])
def test_layers_train_forward_matches_per_layer_forward(sb, name, b, n, layout):
    torch.manual_seed(b + n)
    net = _module(sb, name).cuda().train()
    x = _cloud(b, n, layout, b * n)
    a, c = copy.deepcopy(net), copy.deepcopy(net)
    with torch.no_grad():
        out_a, feat_a = sb.ops.generator_forward(x, layout, *a._layer_specs(), True, 0, per_layer_kernels=True)
        out_c, feat_c, (zs, _) = sb.ops.generator_layers_train_forward(x, layout, *c._layer_specs(), 0)
    torch.cuda.synchronize()
    assert torch.equal(out_a, out_c) and torch.equal(feat_a, feat_c)
    for s, t in zip(_bn_state(a), _bn_state(c)):
        assert torch.equal(s, t)
    assert int(c.bn1.num_batches_tracked) == 1
    # the kept last conv layer reproduces the pooled feature: relu(BN(z)) with the batch statistics, max over each cloud's points
    z = zs[-1].double()
    bn = c._convs()[-1][1]
    y = torch.relu((z - z.mean(0)) / torch.sqrt(z.var(0, unbiased=False) + bn.eps) * bn.weight.double() + bn.bias.double())
    ref = y.view(b, n, -1).max(dim=1)[0]
    torch.testing.assert_close(feat_c.double(), ref, rtol=1e-5, atol=1e-5)


def _float64_reference(net, x, layout, zs, rw):
    """Float64 autograd through the same layer stack, the max-pool gathered at the arg-max of the kept fp32 activations (the route the
    forward took).  Returns {name: gradient}."""
    conv_specs, fc_specs = net._layer_specs()
    nconv = len(conv_specs)
    b = x.shape[0]
    zl = zs[nconv - 1].view(b, -1, zs[nconv - 1].shape[1])
    sgn = torch.where(conv_specs[-1]["bn"][0] >= 0, 1.0, -1.0)
    route = (zl * sgn).argmax(dim=1)
    named = net._generator_named_parameters()
    ps = {nm: p.detach().double().requires_grad_(True) for nm, p in named}
    h = (x.double() if layout == "bnc" else x.double().permute(0, 2, 1)).reshape(-1, 3)
    for i, spec in enumerate(conv_specs + fc_specs):
        if i == nconv:
            h = torch.gather(h.view(b, -1, h.shape[1]), 1, route[:, None, :]).squeeze(1)
        w = ps["l%d.w" % i]
        h = torch.nn.functional.linear(h, w.reshape(w.shape[0], -1), ps["l%d.b" % i])
        if spec["bn"] is not None:
            h = torch.nn.functional.batch_norm(h, None, None, ps["l%d.g" % i], ps["l%d.beta" % i], True, 0.0, spec["bn"][4])
        if spec["relu"]:
            h = torch.relu(h)
    g = torch.autograd.grad(h, list(ps.values()), rw.double())
    return dict(zip(ps, g))


def _fc_margin(net, x, layout):
    """Smallest |pre-ReLU value| of the FC layers (float64): a flipped mask on one of the <= 64 rows moves every gradient."""
    conv_specs, fc_specs = net._layer_specs()
    b = x.shape[0]
    with torch.no_grad():
        h = (x.double() if layout == "bnc" else x.double().permute(0, 2, 1)).reshape(-1, 3)
        margin = 1.0
        for i, spec in enumerate(conv_specs + fc_specs):
            if i == len(conv_specs):
                h = h.view(b, -1, h.shape[1]).max(dim=1)[0]
            h = torch.nn.functional.linear(h, spec["weight"].double().reshape(spec["weight"].shape[0], -1), spec["bias"].double())
            if spec["bn"] is not None:
                h = torch.nn.functional.batch_norm(h, None, None, spec["bn"][0].double(), spec["bn"][1].double(), True, 0.0, spec["bn"][4])
            if i >= len(conv_specs) and spec["relu"]:
                margin = min(margin, h.abs().min().item())
            if spec["relu"]:
                h = torch.relu(h)
    return margin


@pytest.mark.gpu
@pytest.mark.parametrize("name,b,n", [("reconstruction", 2, 777), ("reconstruction", 64, 1000), ("classification", 32, 1024),
                                      ("registration", 37, 1024)])
def test_layers_backward_vs_float64_autograd(sb, name, b, n):
    layout = "bnc"
    for seed in range(b + n, b + n + 20):
        torch.manual_seed(seed)
        net = _module(sb, name).cuda().train()
        with torch.no_grad():
            for p in net.parameters():
                if p.dim() == 1:
                    p.add_(0.1 * torch.randn_like(p))
        x = _cloud(b, n, layout, seed)
        if _fc_margin(net, x, layout) > 2e-5:
            break
    conv_specs, fc_specs = net._layer_specs()
    assert sb.ops.generator_layers_backward_supported(x, layout, conv_specs, fc_specs)
    rw = torch.randn(b, fc_specs[-1]["weight"].shape[0], device="cuda")
    runs = []
    for _ in range(2):
        with torch.no_grad():
            _, _, saved = sb.ops.generator_layers_train_forward(x, layout, conv_specs, fc_specs, 0)
            grads = sb.ops.generator_layers_backward(x, layout, conv_specs, fc_specs, saved, rw, 0)
        flat = []
        for gl in grads:
            flat += [gl["weight"], gl["bias"]] + ([gl["bn_weight"], gl["bn_bias"]] if gl["bn_weight"] is not None else [])
        runs.append([t.clone() for t in flat])
    assert all(torch.equal(a, c) for a, c in zip(*runs)), "per-layer CUDA backward is not run-to-run deterministic"
    ref = _float64_reference(net, x, layout, saved[0], rw)
    nconv = len(conv_specs)
    specs = conv_specs + fc_specs
    bad = []
    for (nm, r), got in zip(ref.items(), runs[0]):
        layer = int(nm[1:nm.index(".")])
        # true gradient exactly 0: biases in front of a training-mode BatchNorm, and the last conv layer's BN shift when fc1 has BatchNorm
        # (a constant added to a pooled channel is removed by its mean subtraction); both sides hold rounding noise there
        zero_true = (nm.endswith(".b") and specs[layer]["bn"] is not None) or (nm == "l%d.beta" % (nconv - 1) and fc_specs[0]["bn"] is not None)
        r = r.reshape(got.shape)
        err = (got.double() - r).abs().max().item()
        tol = 5e-3 if zero_true else 2e-4 * max(r.abs().max().item(), 1e-3)
        bad.append((nm, err, tol)) if err > tol else None
    assert not bad, (name, bad)


def _grads(net):
    return [p.grad.detach().clone() for p in net.parameters() if p.requires_grad]


def _compare_steps(net_cuda, net_torch, loss_fn):
    out = []
    for net in (net_cuda, net_torch):
        net.zero_grad(set_to_none=True)
        loss = loss_fn(net)
        loss.backward()
        out.append((float(loss), _grads(net)))
    assert net_cuda.generator_route == "layers" and net_torch.generator_route == "torch"
    (la, ga), (lc, gc) = out
    assert abs(la - lc) <= 1e-5 * abs(lc), (la, lc)
    # Both sides are fp32.  Parameters whose true gradient is 0 hold rounding noise on both sides: the biases of layers followed by a
    # training-mode BatchNorm and the last conv layer's BatchNorm shift when fc1 has BatchNorm.  The conv-side gradients sum ~1e5
    # point terms that largely cancel (BatchNorm removes the component along each layer's own output), so two fp32 evaluations agree
    # there to about 1e-3 of the tensor's largest entry.
    names = [nm for nm, p in net_cuda.named_parameters() if p.requires_grad]
    last_bn = "bn%d.bias" % net_cuda.n_conv
    bad = []
    for nm, a, c in zip(names, ga, gc):
        err, scale = (a - c).abs().max().item(), c.abs().max().item()
        layer = nm.split(".")[0]
        feeds_bn = layer.startswith("conv") or (layer.startswith("fc") and hasattr(net_cuda, "bn_" + layer))
        zero_true = (nm.endswith(".bias") and feeds_bn) or (nm == last_bn and hasattr(net_cuda, "bn_fc1"))
        if err > (5e-3 if zero_true else 2e-3 * max(scale, 1e-12)):
            bad.append((nm, err, scale))
    assert not bad, bad


def _pair(net):
    torch_net = copy.deepcopy(net)
    torch_net.generator_backward = "torch"
    net.generator_backward = "cuda"
    return net, torch_net


@pytest.mark.gpu
@pytest.mark.parametrize("ae_loss", ["chamfer", "emd"])
def test_reconstruction_step_on_the_per_layer_path(sb, ae_loss):
    from samplenet_b200 import tasknets, trainers
    B, N, M = 50, 2048, 64
    torch.manual_seed(5)
    net, ref = _pair(sb.ReconstructionSampleNet(M).cuda().train())
    ae = tasknets.PointNetAE(N, 128).cuda()
    x = _cloud(B, N, "bnc", 21)
    _compare_steps(net, ref, lambda s: trainers.ReconstructionStep(s, ae, M, ae_loss=ae_loss).loss(x)[0])


@pytest.mark.gpu
def test_classification_step_on_the_per_layer_path(sb):
    from samplenet_b200 import tasknets, trainers
    B, N, M = 32, 1024, 32
    torch.manual_seed(6)
    net, ref = _pair(sb.ClassificationSampleNet(M, group_size=7).cuda().train())
    cls = tasknets.PointNetCls().cuda()
    x = _cloud(B, N, "bnc", 22)
    y = torch.randint(0, 40, (B,), device="cuda")
    _compare_steps(net, ref, lambda s: trainers.ClassificationStep(s, cls, M).loss(x, y)[0])


def _tf_variables(seed=3, m=32):
    """Sampler-scope variables named and shaped as the classification trainer's TF graph creates them."""
    r = np.random.default_rng(seed)
    v = {}
    widths = [3, 64, 64, 64, 128, 128]
    fcw = [128, 256, 256, 256, 3 * m]
    layers = [("conv%d" % (i + 1), [1, 3, 1, 64] if i == 0 else [1, 1, widths[i], widths[i + 1]], widths[i + 1]) for i in range(5)]
    layers += [("fc1%db" % (i + 1), [fcw[i], fcw[i + 1]], fcw[i + 1]) for i in range(4)]
    for sc, shape, c in layers:
        sc = "sampler/" + sc
        v[sc + "/weights:0"] = (r.standard_normal(shape) * 0.2).astype(np.float32)
        v[sc + "/biases:0"] = (0.1 * r.standard_normal(c)).astype(np.float32)
        v[sc + "/bn/gamma:0"] = (1.0 + 0.2 * r.standard_normal(c)).astype(np.float32)
        v[sc + "/bn/beta:0"] = (0.1 * r.standard_normal(c)).astype(np.float32)
        v[sc + "/bn/moments/Squeeze/ExponentialMovingAverage:0"] = (0.1 * r.standard_normal(c)).astype(np.float32)
        v[sc + "/bn/moments/Squeeze_1/ExponentialMovingAverage:0"] = (0.5 + r.random(c)).astype(np.float32)
    return v


@pytest.mark.gpu
def test_classification_sampler_eval_matches_tf_generator_and_state_dict(sb):
    from samplenet_b200.tf_variant import TFSampleNetGenerator
    v = _tf_variables()
    net = sb.ClassificationSampleNet.from_tf_variables(v, group_size=7).cuda().eval()
    gen = TFSampleNetGenerator.from_tf_variables(v).cuda().eval()
    x = _cloud(16, 1024, "bnc", 23)
    simp, match = net(x)
    assert torch.equal(simp, gen(x))
    assert match.shape == (16, 32, 3)
    # state_dict round trip, then the same outputs in both modes
    other = sb.ClassificationSampleNet(32, group_size=7).cuda()
    other.load_state_dict(net.state_dict())
    other.eval()
    assert torch.equal(other(x)[0], simp)
    rec = sb.ReconstructionSampleNet(64).cuda().train()
    rec2 = sb.ReconstructionSampleNet(64).cuda().train()
    rec2.load_state_dict(rec.state_dict())
    xr = _cloud(4, 512, "bnc", 24)
    a, b = rec(xr), rec2(xr)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
