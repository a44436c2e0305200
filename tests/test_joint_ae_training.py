"""The autoencoder trained together with the reconstruction samplers (the reference's --fixed_ae False): the batch-statistics encoder's
parameter backward and running-statistics update (snb200_frozen_encoder_bstat_param_backward / _running_update, csrc/frozen_encoder_bstat.cu),
ops.EncoderBStatTrainFunction, CudaPointNetAE.prefixes in training mode, and ReconstructionStep / ProgressiveReconstructionStep(fixed_ae=False)
under SamplerTrainStep.

CPU: the exported symbols, the envelope and workspace sizes, the rejections, the steps' constructor contract.  GPU (H100): every parameter
gradient against float64 autograd of the contract with the kernel's masks and routes pinned, grad_x bit for bit the existing backward's,
determinism, the running statistics against a float64 ascending update, the write set, CudaPointNetAE.prefixes and the steps against the
plain module's ascending per-prefix loop, and the graphed and non-finite-skipping epochs."""
import copy
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import test_ae_batch_stats as bst  # noqa: E402
from samplenet_b200 import tasknets, trainers  # noqa: E402

# Bars (GPU): measured values on an H100 80GB HBM3 in brackets
PARAM_BAR = 1e-4      # [1.06e-5] every conv weight, gamma and beta gradient against pinned float64 autograd: / max |reference| of the tensor
BIAS_BAR = 1e-4       # [2.2e-6] conv bias gradients (zero in exact arithmetic): / max |reference| of the layer's weight gradient
RUNNING_BAR = 1e-6    # [2.1e-7] running mean / variance against the float64 ascending update on the forward's statistics: / (|reference| + 1)
ADAM_BAR = 2e-3       # [2.0e-4 at lr 1e-5] losses of five Adam steps, CudaPointNetAE against the plain module (TF32 off), as test_task_training
UPDATE_COS = 0.999    # [0.99983] cosine between the two routes' parameter updates over those five steps
PREFIX_LOSS_BAR = 1e-5
PREFIX_GRAD_BAR = 2e-3

AE = bst.AE
POW2 = bst.POW2
# (b, n, sizes): the bstat tests' shapes, the progressive plan, one prefix, sizes that are not multiples of 128.  The bstat tests' one-cloud
# case becomes five clouds: a group of two values has its variance from fp32 (sum, sum of squares) with most digits cancelled, which puts
# the gradients 2.8e-4 off the float64 statistics' (measured on an H100 at b = 2, sizes [1, 777]): a conditioning limit, not the kernel's.
GRAD_CASES = [(50, 2048, POW2), (5, 333, [1, 7, 64, 333]), (5, 777, [1, 777]), (50, 2048, [64]), (3, 1000, [100, 300, 555, 1000])]


def _wmax(widths=AE):
    return max(widths[i + 1] * (widths[i] + 1) for i in range(len(widths) - 1))


def _chunks(b, sizes):
    tiles = bst._rows(b, sizes) // 128
    tpc = -(-tiles // 256)
    return -(-tiles // tpc)


# ------------------------------------------------------------------------------------------------------------------ CPU
lib = bst.lib


def test_envelope_and_workspaces(lib):
    from samplenet_b200 import _lib

    for name in ("snb200_frozen_encoder_bstat_param_backward_supported", "snb200_frozen_encoder_bstat_param_backward_workspace_bytes",
                 "snb200_frozen_encoder_bstat_param_backward", "snb200_frozen_encoder_bstat_running_update"):
        assert name in _lib.exported_symbols() and getattr(lib, name) is not None
    t = bst._table(AE)
    sup = lambda b, n, sizes, table=t: lib.snb200_frozen_encoder_bstat_param_backward_supported(b, n, 5, table, len(sizes), bst._sz(sizes))
    wsb = lambda b, n, sizes: lib.snb200_frozen_encoder_bstat_param_backward_workspace_bytes(b, n, 5, t, len(sizes), bst._sz(sizes))
    for b, n, sizes in GRAD_CASES + [(3, 4096, [4096]), (2, 1, [1])]:
        assert sup(b, n, sizes) == 1
        bwd = lib.snb200_frozen_encoder_bstat_backward_workspace_bytes(b, n, 5, t, len(sizes), bst._sz(sizes))
        assert wsb(b, n, sizes) == bwd + bst._a256(_chunks(b, sizes) * _wmax() * 4)
    # the progressive plan: 217 600 packed rows in 1 700 tiles, 7 per chunk
    assert bst._rows(50, POW2) == 217600 and _chunks(50, POW2) == 243
    # the bstat envelope's edges
    assert sup(2, 2048, [16 * (i + 1) for i in range(16)]) == 1
    assert sup(2, 2048, [16 * (i + 1) for i in range(17)]) == 0
    assert sup(2, 2048, [64, 16]) == 0 and sup(2, 2048, [16, 16]) == 0
    assert sup(2, 2048, [0, 16]) == 0 and sup(2, 2048, [2049]) == 0
    assert sup(2, 4097, [16]) == 0
    assert sup(1024, 4096, [4096]) == 1 and sup(1025, 4096, [4096]) == 0
    assert sup(2, 2048, [16], bst._table(AE, bn=False)) == 0 and sup(2, 2048, [16], bst._table(AE, relu=0)) == 0
    # ... plus an unbiased variance for every prefix: b * s = 1 is refused, which the frozen envelope takes
    assert sup(1, 777, [1, 777]) == 0 and sup(1, 1, [1]) == 0 and sup(1, 777, [2, 777]) == 1
    assert lib.snb200_frozen_encoder_bstat_supported(1, 777, 5, t, 2, bst._sz([1, 777])) == 1
    assert wsb(1, 777, [1, 777]) == 0 and wsb(2, 2048, list(range(1, 18))) == 0


@pytest.mark.parametrize("case", ["prefixes", "unsorted", "n", "rows", "no_bn", "one_value"])
def test_entries_refuse_outside_the_envelope(lib, case):
    """Both entries return SNB200_EUNSUPPORTED before launching anything (without a GPU a launch would fail with SNB200_ECUDA instead)."""
    from samplenet_b200._lib import LayerGrad

    b, n, sizes, table = {"prefixes": (2, 2048, list(range(1, 18)), bst._table(AE)), "unsorted": (2, 2048, [64, 16], bst._table(AE)),
                          "n": (2, 4097, [16], bst._table(AE)), "rows": (1025, 4096, [4096], bst._table(AE)),
                          "no_bn": (2, 2048, [16], bst._table(AE, bn=False)), "one_value": (1, 777, [1, 777], bst._table(AE))}[case]
    buf = ctypes.c_void_p(bst._ptr())
    ws = ctypes.create_string_buffer(16)
    grads = (LayerGrad * 5)()
    for g in grads:
        g.weight, g.bias, g.bn_weight, g.bn_bias = bst._ptr(), bst._ptr(), bst._ptr(), bst._ptr()
    rc = lib.snb200_frozen_encoder_bstat_param_backward(b, n, buf, 5, table, len(sizes), bst._sz(sizes), buf, buf, buf, ctypes.addressof(ws),
                                                        1 << 40, buf, buf, grads, ctypes.addressof(ws), 1 << 40, None)
    assert rc == -4, rc
    assert lib.snb200_frozen_encoder_bstat_running_update(b, n, 5, table, len(sizes), bst._sz(sizes), buf, None) == -4


class _Sampler(torch.nn.Module):
    pass


def test_step_constructors():
    for make in (lambda ae, **kw: trainers.ReconstructionStep(_Sampler(), ae, 64, **kw),
                 lambda ae, **kw: trainers.ProgressiveReconstructionStep(_Sampler(), ae, **kw)):
        # the default freezes the autoencoder and sets eval mode, as before
        net = tasknets.PointNetAE(64).train()
        step = make(net)
        assert step.fixed_ae and not net.training and not any(p.requires_grad for p in net.parameters())
        # fixed_ae=False leaves the module alone, in either mode
        for mode in (True, False):
            net = tasknets.PointNetAE(64).train(mode)
            w = tasknets.CudaPointNetAE(net)
            step = make(w, fixed_ae=False)
            assert not step.fixed_ae and net.training == mode and all(p.requires_grad for p in net.parameters())
        with pytest.raises(ValueError, match="FrozenPointNetAE"):
            make(tasknets.FrozenPointNetAE(tasknets.PointNetAE(64)), fixed_ae=False)
        with pytest.raises(ValueError, match="ae_batch_stats"):
            make(tasknets.PointNetAE(64), fixed_ae=False, ae_batch_stats=True)
    with pytest.raises(ValueError, match="Chamfer"):
        trainers.ProgressiveReconstructionStep(_Sampler(), tasknets.PointNetAE(64), ae_loss="emd", fixed_ae=False)


# ------------------------------------------------------------------------------------------------------------------ GPU
sb = bst.sb


def _train_case(b, n, seed):
    net = bst._randomize(tasknets.PointNetAE(n_pc_points=2048), seed).cuda().train()
    x = (torch.rand(b, n, 3, generator=torch.Generator().manual_seed(seed + 1)) - 0.5).cuda()
    return net, x


def _pinned_param_grads64(net, x, sizes, zs, st, route, g):
    """Float64 autograd of sum(g * pooled) through the contract with the kernel's ReLU masks and routes pinned (see
    test_ae_batch_stats._pinned_grad64), with respect to every conv weight, conv bias, gamma and beta: [(dW, db, dgamma, dbeta)]."""
    leaves = [[t.detach().double().clone().requires_grad_(True) for t in (c.weight[:, :, 0], c.bias, bn.weight, bn.bias)]
              for c, bn in zip(net.convs, net.bns)]
    total = 0.0
    for p, s in enumerate(sizes):
        rows = bst._group_rows(x.shape[0], sizes, p, x.device)
        h = x[:, :s].double()
        for l, ((w, bias, gam, bet), bn) in enumerate(zip(leaves, net.bns)):
            z = h @ w.t() + bias
            mean = z.mean(dim=(0, 1))
            var = ((z - mean) ** 2).mean(dim=(0, 1))
            a = (z - mean) / torch.sqrt(var + bn.eps) * gam + bet
            sc, sh, _ = bst._kernel_scale_shift(bn, st[l][p])
            h = a * (zs[l][rows].double() * sc.double() + sh > 0)
        pooled = torch.gather(h, 1, route[p].long()[:, None, :]).squeeze(1)
        total = total + (pooled * g[p].double()).sum()
    flat = torch.autograd.grad(total, [t for layer in leaves for t in layer])
    return [flat[4 * i:4 * i + 4] for i in range(len(leaves))]


ALL = [(True, True, True, True)] * 5


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,sizes", GRAD_CASES)
def test_param_gradients_against_float64(sb, b, n, sizes):
    ops = sb.ops
    net, x = _train_case(b, n, 71)
    specs = tasknets._conv_specs(net)
    g = torch.randn(len(sizes), b, AE[-1], generator=torch.Generator().manual_seed(9)).cuda()
    pooled, route, stats, ws = ops.frozen_encoder_bstat_forward(x, specs, sizes)
    gx, grads = ops.frozen_encoder_bstat_param_backward(x, specs, sizes, pooled, route, stats, ws, g, ALL)
    # grad_x is bit for bit the existing backward's, and a second call gives the same parameter gradients bit for bit
    assert torch.equal(gx, ops.frozen_encoder_bstat_backward(x, specs, sizes, pooled, route, stats, ws, g))
    gx2, grads2 = ops.frozen_encoder_bstat_param_backward(x, specs, sizes, pooled, route, stats, ws, g, ALL)
    assert torch.equal(gx, gx2) and all(torch.equal(u, v) for a, c in zip(grads, grads2) for u, v in zip(a, c)), "not bit-identical on repeat"
    # without grad_x, and with a subset of the gradients: the same values
    none_x, part = ops.frozen_encoder_bstat_param_backward(x, specs, sizes, pooled, route, stats, ws, g, [(True, False, False, True)] * 5,
                                                           need_x=False)
    assert none_x is None and all(torch.equal(p_[0], a[0]) and torch.equal(p_[3], a[3]) and p_[1] is None for p_, a in zip(part, grads))
    st = ops.frozen_encoder_bstat_stats(stats, specs, len(sizes))
    ref = _pinned_param_grads64(net, x, sizes, bst._zsave(ws, bst._rows(b, sizes)), st, route, g)
    worst = {"weight": 0.0, "bias": 0.0, "gamma": 0.0, "beta": 0.0}
    for (dw, db, dg, dbt), (rw, rb, rg, rbt) in zip(grads, ref):
        rel = lambda got, want: ((got.double() - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()
        worst["weight"] = max(worst["weight"], rel(dw, rw))
        worst["gamma"] = max(worst["gamma"], rel(dg, rg))
        worst["beta"] = max(worst["beta"], rel(dbt, rbt))
        worst["bias"] = max(worst["bias"], ((db.double() - rb).abs().max() / rw.abs().max()).item())
    print("bstat param backward", b, n, len(sizes), worst)
    assert max(worst["weight"], worst["gamma"], worst["beta"]) <= PARAM_BAR and worst["bias"] <= BIAS_BAR, worst


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,sizes", [(50, 2048, POW2), (5, 333, [1, 7, 64, 333])])
def test_running_update_and_forward(sb, b, n, sizes):
    ops = sb.ops
    net, x = _train_case(b, n, 81)
    ref_net = copy.deepcopy(net)
    specs = tasknets._conv_specs(net)
    params = [t for c, bn in zip(net.convs, net.bns) for t in (c.weight, c.bias, bn.weight, bn.bias)]
    conv = [{"weight": c.weight, "bias": c.bias, "bn": tasknets._bn_spec(bn), "relu": True} for c, bn in zip(net.convs, net.bns)]
    want_p, want_r, want_s, _ = ops.frozen_encoder_bstat_forward(x, specs, sizes)
    before = {k: v.clone() for k, v in net.state_dict().items()}
    pooled, route, stats = ops.EncoderBStatTrainFunction.apply(x, conv, sizes, *params)
    # the forward is bit for bit the frozen one
    assert torch.equal(pooled, want_p) and torch.equal(route, want_r) and torch.equal(stats, want_s)
    st = ops.frozen_encoder_bstat_stats(stats, specs, len(sizes))
    worst = 0.0
    for l, bn in enumerate(ref_net.bns):
        rm, rv = bn.running_mean.double(), bn.running_var.double()
        for p, s in enumerate(sizes):
            cnt = b * s
            rm = (1 - bn.momentum) * rm + bn.momentum * st[l][p, 0]
            rv = (1 - bn.momentum) * rv + bn.momentum * st[l][p, 1] * cnt / (cnt - 1)
        for got, want in ((net.bns[l].running_mean, rm), (net.bns[l].running_var, rv)):
            worst = max(worst, ((got.double() - want).abs() / (want.abs() + 1)).max().item())
        assert int(net.bns[l].num_batches_tracked) == int(ref_net.bns[l].num_batches_tracked) + len(sizes)
    print("running statistics", b, n, len(sizes), worst)
    assert worst <= RUNNING_BAR, worst
    # nothing else of the module moved
    after = net.state_dict()
    assert all(torch.equal(before[k], after[k]) for k in before if "running" not in k and "num_batches" not in k)


@pytest.mark.gpu
def test_write_set(sb):
    """The parameter backward writes only the gradients it is given (and its workspace); the running update only the running buffers and
    counters: guard words around every gradient stay as they were, and the module is untouched."""
    from samplenet_b200 import _lib
    from samplenet_b200._lib import LayerGrad
    from samplenet_b200.ops import _p, _stream, make_layers

    ops, lib_ = sb.ops, _lib.lib()
    b, n, sizes = 5, 333, [1, 7, 64, 333]
    net, x = _train_case(b, n, 91)
    specs = tasknets._conv_specs(net)
    pooled, route, stats, ws = ops.frozen_encoder_bstat_forward(x, specs, sizes)
    g = torch.randn_like(pooled)
    _, want = ops.frozen_encoder_bstat_param_backward(x, specs, sizes, pooled, route, stats, ws, g, ALL, need_x=False)
    before = {k: v.clone() for k, v in net.state_dict().items()}
    conv, keep = make_layers(specs)
    G = 4096
    garr, bufs = (LayerGrad * 5)(), []
    for l in range(5):
        c_out, c_in = AE[l + 1], AE[l]
        sizes_l = {"weight": c_out * c_in, "bias": c_out, "bn_weight": c_out, "bn_bias": c_out}
        for k, cnt in sizes_l.items():
            if l == 2 and k == "bias":
                continue                                     # a NULL pointer is skipped
            buf = torch.full((G + cnt + G,), 7.0, device="cuda")
            setattr(garr[l], k, buf[G:].data_ptr())
            bufs.append((l, k, buf, cnt))
    inputs = {"x": x, "pooled": pooled, "route": route, "stats": stats, "fwd_workspace": ws, "grad_pooled": g}
    inputs_before = {k: v.clone() for k, v in inputs.items()}
    csz = bst._sz(sizes)
    wsb = lib_.snb200_frozen_encoder_bstat_param_backward_workspace_bytes(b, n, 5, conv, len(sizes), csz)
    bws = torch.empty(wsb, device="cuda", dtype=torch.uint8)
    _lib.check(lib_.snb200_frozen_encoder_bstat_param_backward(b, n, _p(x), 5, conv, len(sizes), csz, _p(pooled), _p(route), _p(stats), _p(ws),
                                                               ws.numel(), _p(g), None, garr, _p(bws), wsb, _stream()), "param backward")
    torch.cuda.synchronize()
    keys = ("weight", "bias", "bn_weight", "bn_bias")
    for l, k, buf, cnt in bufs:
        assert torch.all(buf[:G] == 7) and torch.all(buf[G + cnt:] == 7), (l, k)
        assert torch.equal(buf[G:G + cnt], want[l][keys.index(k)].reshape(-1)), (l, k)
    assert all(torch.equal(before[k], v) for k, v in net.state_dict().items())
    # its read-only inputs, the forward's outputs and workspace included, stay bit for bit
    assert all(torch.equal(inputs_before[k], v) for k, v in inputs.items()), [k for k, v in inputs.items() if not torch.equal(inputs_before[k], v)]
    # the running update: the running buffers and counters move, the parameters and the statistics it reads stay
    ops.frozen_encoder_bstat_running_update(x, [dict(s, bn=tasknets._bn_spec(bn)) for s, bn in zip(specs, net.bns)], sizes, stats)
    torch.cuda.synchronize()
    for k, v in net.state_dict().items():
        moved = not torch.equal(before[k], v)
        assert moved == ("running" in k or "num_batches" in k), k
    assert all(torch.equal(inputs_before[k], v) for k, v in inputs.items())
    # momentum=None (a cumulative average) is refused before anything runs
    with pytest.raises(ValueError, match="momentum=None"):
        ops.frozen_encoder_bstat_running_update(x, [dict(s, bn=tasknets._bn_spec(bn)[:5] + (None,)) for s, bn in zip(specs, net.bns)], sizes, stats)
    params = [t for c, bn in zip(net.convs, net.bns) for t in (c.weight, c.bias, bn.weight, bn.bias)]
    with pytest.raises(ValueError, match="momentum=None"):
        ops.EncoderBStatTrainFunction.apply(x, [dict(s, bn=tasknets._bn_spec(bn)[:5] + (None,)) for s, bn in zip(specs, net.bns)], sizes, *params)
    del keep


def _tf32_off(monkeypatch):
    bst._tf32_off(monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,sizes", [(50, 2048, POW2), (50, 2048, [64]), (5, 333, [1, 7, 64, 333])])
def test_prefixes_in_training_mode_against_the_module(sb, monkeypatch, b, n, sizes):
    """CudaPointNetAE.prefixes in training mode against the module's ascending loop (fp32, TF32 off): reconstructions, loss, the input's
    and every parameter's gradient, the running statistics; the route."""
    _tf32_off(monkeypatch)
    net, x = _train_case(b, n, 101)
    ref = copy.deepcopy(net)
    w = tasknets.CudaPointNetAE(net).train()
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    got = w.prefixes(xa, sizes)
    assert w.route == "cuda" and got.shape == (len(sizes), b, 2048, 3)
    want = torch.stack([ref(xb[:, :s].contiguous()) for s in sizes])
    target = torch.rand(b, 2048, 3, generator=torch.Generator().manual_seed(3)).cuda()
    lg = sum(((got[p] - target) ** 2).mean() for p in range(len(sizes)))
    lw = sum(((want[p] - target) ** 2).mean() for p in range(len(sizes)))
    lg.backward()
    lw.backward()
    rec_err = ((got - want).abs().max() / want.abs().max()).item()
    loss_err = abs(float(lg) - float(lw)) / abs(float(lw))
    gx_err = ((xa.grad - xb.grad).abs().max() / xb.grad.abs().max()).item()
    perr = max(((p.grad - q.grad).abs().max() / q.grad.abs().max().clamp_min(1e-30)).item()
               for (k, p), (_, q) in zip(net.named_parameters(), ref.named_parameters()) if not k.startswith("convs") or "bias" not in k)
    run_err = max(((a - c).abs() / (c.abs() + 1)).max().item() for (k, a), (_, c) in zip(net.state_dict().items(), ref.state_dict().items())
                  if "running" in k)
    print("prefixes", b, n, len(sizes), "rec", rec_err, "loss", loss_err, "grad_x", gx_err, "params", perr, "running", run_err)
    assert all(torch.equal(a, c) for k, a in net.state_dict().items() for k2, c in ref.state_dict().items() if k == k2 and "num_batches" in k)
    assert rec_err <= PREFIX_LOSS_BAR * 10 and loss_err <= PREFIX_LOSS_BAR, (rec_err, loss_err)
    assert gx_err <= PREFIX_GRAD_BAR and perr <= PREFIX_GRAD_BAR and run_err <= 2e-5, (gx_err, perr, run_err)


@pytest.mark.gpu
def test_prefixes_routes_and_fallbacks(sb):
    net, x = _train_case(3, 300, 111)
    w = tasknets.CudaPointNetAE(net).train()
    with torch.no_grad():
        w.prefixes(x, [16, 300])
        assert w.route == "cuda"
        w.prefixes(x, list(range(1, 18)))                              # 17 prefixes
        assert w.route == "module"
        w.prefixes(torch.rand(2, 4097, 3, device="cuda"), [16, 4097])  # n > 4096
        assert w.route == "module"
        # a one-value batch (b * s = 1) is outside the envelope; the module route then raises, as nn.BatchNorm1d refuses it
        assert not sb.ops.frozen_encoder_bstat_train_supported(1, 300, tasknets._conv_specs(net), [1, 300])
        with pytest.raises(ValueError):
            w.prefixes(x[:1], [1, 300])
        assert w.route == "module"
        net.bns[2].momentum = None                                    # a cumulative average
        w.prefixes(x, [16, 300])
        assert w.route == "module"
        net.bns[2].momentum = 0.1
        w.eval()
        got = w.prefixes(x, [16, 300])
        assert w.route == "frozen" and torch.equal(got, tasknets.FrozenPointNetAE(net).prefixes(x, [16, 300]))
    w.prefixes(x, [16, 300])                                           # eval mode with parameter gradients
    assert w.route == "module"


def _joint_runner(step_kind, sampler, ae, M, B=50, sizes=POW2, wrap=True, graphed=False, skip=False, lr=5e-4):
    """SamplerTrainStep over the sampler and the autoencoder trained together (fixed_ae=False), capturable Adam over both on every route:
    a capturable and a non-capturable Adam round differently."""
    a = tasknets.CudaPointNetAE(ae) if wrap else ae
    step = (trainers.ReconstructionStep(sampler, a, M, fixed_ae=False) if step_kind == "rec"
            else trainers.ProgressiveReconstructionStep(sampler, a, sizes=sizes, fixed_ae=False))
    opt = torch.optim.Adam(list(sampler.parameters()) + list(ae.parameters()), capturable=True)   # the same Adam eager and graphed
    return trainers.SamplerTrainStep(step, opt, batch_size=B, learning_rate=lr, graphed=graphed, skip_nonfinite=skip)


@pytest.mark.gpu
@pytest.mark.parametrize("step_kind", ["rec", "progressive_rec"])
def test_joint_steps_against_the_plain_module(sb, monkeypatch, step_kind):
    """Five Adam steps of the sampler and the autoencoder together: CudaPointNetAE against the plain PointNetAE, losses, running statistics
    and the parameter updates, at lr = 1e-5.  At the trainers' default 5e-4 the first loss agrees to 5e-7 and the five-step losses drift
    apart by up to 1.2e-2 (rec) and 4.7e-3 (progressive), but the sampler trained alone against the frozen autoencoder drifts as far between
    its two accepted routes (FrozenPointNetAE(batch_stats) against the plain module: 4.2e-2 and 5.2e-3, measured on an H100): the drift is
    the sampler's training dynamics at that rate, not the autoencoder's gradients (checked against float64 and the module above).  The
    updates are compared as one vector, by their cosine."""
    from test_sampler_training import _cloud

    _tf32_off(monkeypatch)
    B, N = 50, 2048
    M = 64 if step_kind == "rec" else 2048
    torch.manual_seed(7)
    sampler = sb.ReconstructionSampleNet(M).cuda().train()
    with torch.no_grad():
        _, proj = copy.deepcopy(sampler)(_cloud(B, N, "bnc", 31))
    ae = bst._conditioned_ae(proj, [M] if step_kind == "rec" else POW2, 61)
    out = {}
    for wrap in (True, False):
        s, a = copy.deepcopy(sampler), copy.deepcopy(ae)
        run = _joint_runner(step_kind, s, a, M, B=B, wrap=wrap, lr=1e-5)
        start = torch.cat([p.detach().reshape(-1) for p in list(s.parameters()) + list(a.parameters())])
        losses = [float(run(_cloud(B, N, "bnc", 40 + i))["loss"]) for i in range(5)]
        update = torch.cat([p.detach().reshape(-1) for p in list(s.parameters()) + list(a.parameters())]) - start
        out[wrap] = (losses, update.double(), a)
        if wrap:
            assert run.task.ae.route == "cuda"
    (lc, pc, ac), (lm, pm, am) = out[True], out[False]
    loss_err = max(abs(u - v) / abs(v) for u, v in zip(lc, lm))
    cos = (torch.dot(pc, pm) / (pc.norm() * pm.norm())).item()
    run_err = max(((u - v).abs() / (v.abs() + 1)).max().item() for bu, bv in zip(ac.bns, am.bns)
                  for u, v in ((bu.running_mean, bv.running_mean), (bu.running_var, bv.running_var)))
    print("joint step", step_kind, "losses", lc, lm, "loss", loss_err, "update cosine", cos, "running", run_err)
    assert loss_err <= ADAM_BAR and cos >= UPDATE_COS and run_err <= ADAM_BAR, (loss_err, cos, run_err)
    assert all(int(u.num_batches_tracked) == int(v.num_batches_tracked) for u, v in zip(ac.bns, am.bns))


def _state(run):
    st = {"s." + k: v.detach().clone() for k, v in run.task.sampler.state_dict().items()}
    st.update({"a." + k: v.detach().clone() for k, v in run.task.ae.state_dict().items()})
    for i, p in enumerate(run.optimizer.param_groups[0]["params"]):
        for k, v in run.optimizer.state.get(p, {}).items():
            st["opt.%d.%s" % (i, k)] = torch.as_tensor(v).detach().clone()
    return st


def _small_runner(sb, step_kind, **kw):
    torch.manual_seed(0)
    sampler = sb.ReconstructionSampleNet(32).cuda()
    ae = tasknets.PointNetAE(n_pc_points=256).cuda()
    return _joint_runner(step_kind, sampler, ae, 32, B=8, sizes=(8, 16, 32), **kw)


def _small_set():
    return (torch.rand(16, 256, 3, generator=torch.Generator().manual_seed(5)) - 0.5).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("step_kind", ["rec", "progressive_rec"])
def test_graphed_epochs_with_the_autoencoder_trained(sb, step_kind):
    """graphed=True gives the eager epochs bit for bit with the autoencoder trained: the returned dicts, both modules' parameters and
    buffers (running statistics and num_batches_tracked included), the optimiser state, the random numbers drawn and the step count."""
    x = _small_set()
    res = {}
    for graphed in (False, True):
        run = _small_runner(sb, step_kind, graphed=graphed)
        torch.manual_seed(11)
        res[graphed] = ([run.train_one_epoch(x) for _ in range(2)], _state(run), torch.cuda.get_rng_state(), run.step, run.task.ae.route)
    (eager, st_e, rng_e, step_e, route_e), (graph, st_g, rng_g, step_g, route_g) = res[False], res[True]
    assert route_e == route_g == "cuda"
    assert eager == graph and all(r["steps"] == 2 for r in graph)
    assert st_e.keys() == st_g.keys()
    for k in st_e:
        assert st_e[k].dtype == st_g[k].dtype and torch.equal(st_e[k], st_g[k]), k
    assert torch.equal(rng_e, rng_g) and step_e == step_g
    assert all(int(v) == 4 * (3 if step_kind == "progressive_rec" else 1) for k, v in st_g.items() if k.startswith("a.") and "num_batches" in k)


@pytest.mark.gpu
@pytest.mark.parametrize("graphed", [False, True])
def test_nonfinite_batch_leaves_both_modules(sb, graphed):
    """skip_nonfinite=True: a batch holding a NaN cloud leaves the sampler, the autoencoder and the optimiser state exactly as they were."""
    x = _small_set()
    run = _small_runner(sb, "progressive_rec", graphed=graphed, skip=True)
    assert int(run(x[:8])["skipped"]) == 0
    before = _state(run)
    bad = x[8:].clone()
    bad[3, 17] = float("nan")
    assert int(run(bad)["skipped"]) == 1
    after = _state(run)
    assert before.keys() == after.keys() and all(torch.equal(before[k], after[k]) for k in before)
