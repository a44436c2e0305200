"""The point-cloud autoencoder trained on CUDA (tasknets.CudaPointNetAE over ops.LayerStackFunction) and the task networks' training steps
(trainers.ClassifierTrainStep, trainers.AutoencoderTrainStep).

CPU: the two schedules against TF's staircase exponential_decay at step boundaries, and applied by a step of the plain classifier; the
wrapper's shared parameters, state-dict keys and refusal of CPU tensors.
GPU (H100): the routes; the wrapper's training step against float64 on conditioned instances (output, loss, every parameter gradient,
running statistics and num_batches_tracked); the backward against float64 on the kernel's own forward values and masks, with the
end-to-end gradient distance split into the backward's, the forward values' and the ReLU mask flips' shares; repeat backward passes
bit-identical; five Adam steps through AutoencoderTrainStep against the plain module.  Measured values are attached to the test reports."""
import copy
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from samplenet_b200 import tasknets, trainers  # noqa: E402

# Bars (GPU), about 10x the largest value measured on an H100 80GB HBM3 (in brackets)
OUT_BAR = 2e-5          # [8.1e-7] reconstruction against float64: / max |reference|
LOSS_BAR = 2e-5         # [1.1e-7] Chamfer / EMD of the reconstruction, relative to the float64 module's
GRAD_BAR = 2e-4         # [1.7e-5] every parameter gradient against float64 with the kernel's masks at ambiguous units: / its scale
BIAS_NOISE_BAR = 1e-5   # [7.7e-7] conv biases ahead of a BatchNorm (zero in exact arithmetic): largest |gradient| / the largest of all
BWD_KERNEL_BAR = 4e-5   # [3.5e-6] the CUDA backward against float64 on the kernel's own forward values and masks: / its scale
AMBIGUOUS = 1e-5        # units this close to their ReLU kink (relative) take the CUDA backward's mask in the float64 reference ...
FLIPPED_MAX = 200       # [19] ... which changes at most this many units' masks
RUNNING_BAR = 2e-5      # [2.1e-6] running mean / variance against the float64 module's: / max |reference|
ADAM_BAR = 2e-3         # [2.1e-4] losses of five Adam steps, wrapper against the plain module (TF32 off), relative
KINK_GUARD = 1e-7       # conditioned instances: no BatchNorm output of a routed point closer than this to the ReLU kink ...
TIE_GUARD = 1e-6        # ... and no pooled maximum closer than this (relative) to its runner-up


# ------------------------------------------------------------------------------------------------------------------ CPU
def _tf_staircase(base, global_step, decay_steps, rate):
    """tf.train.exponential_decay(..., staircase=True) as TF evaluates it: p = floor(global_step / decay_steps), base * rate^p."""
    import math

    return base * math.pow(rate, math.floor(global_step / decay_steps))


def test_classifier_schedules_at_step_boundaries():
    step = trainers.ClassifierTrainStep(torch.nn.Linear(1, 1), None, batch_size=32, base_lr=1e-3, decay_step=200000, decay_rate=0.7)
    for s in (0, 1, 6249, 6250, 6251, 12499, 12500, 80000, 81249, 81250, 10 ** 6):
        lr = max(_tf_staircase(1e-3, s * 32, 200000, 0.7), 1e-5)
        bn = min(0.99, 1 - _tf_staircase(0.5, s * 32, 200000.0, 0.5))
        assert step.learning_rate(s) == pytest.approx(lr, rel=1e-12, abs=0), s
        assert step.bn_decay(s) == pytest.approx(bn, rel=1e-12, abs=0), s
    assert step.learning_rate(6249) == 1e-3 and step.learning_rate(6250) == pytest.approx(7e-4)
    assert step.learning_rate(10 ** 6) == 1e-5                    # clipped
    assert step.bn_decay(0) == 0.5 and step.bn_decay(6250) == 0.75 and step.bn_decay(10 ** 6) == 0.99


@pytest.mark.parametrize("cls", [tasknets.PointNetCls, tasknets.PointNetClsTransforms])
def test_classifier_step_applies_the_schedules(cls):
    torch.manual_seed(0)
    net = cls(num_classes=5)
    opt = torch.optim.Adam(net.parameters(), lr=123.0)
    step = trainers.ClassifierTrainStep(net, opt, batch_size=4, decay_step=40)
    step.step = 10                                                 # 10 * 4 / 40: the first staircase step
    x, labels = torch.rand(4, 32, 3), torch.tensor([0, 1, 2, 3])
    before = copy.deepcopy(net.state_dict())
    loss, pred, correct = step(x, labels)
    assert step.step == 11 and opt.param_groups[0]["lr"] == pytest.approx(7e-4)
    bns = [m for m in net.modules() if isinstance(m, torch.nn.BatchNorm1d)]
    assert bns and all(m.momentum == pytest.approx(0.25) for m in bns)
    assert pred.shape == (4,) and correct == int((pred == labels).sum()) and torch.isfinite(loss)
    assert any(not torch.equal(before[k], v) for k, v in net.state_dict().items())


def test_autoencoder_step_refuses_unknown_loss():
    with pytest.raises(ValueError):
        trainers.AutoencoderTrainStep(tasknets.PointNetAE(), None, ae_loss="l2")


def test_cuda_ae_shares_the_module():
    ae = tasknets.PointNetAE(n_pc_points=64)
    w = tasknets.CudaPointNetAE(ae)
    assert [id(p) for p in w.parameters()] == [id(p) for p in ae.parameters()]
    assert list(w.state_dict()) == list(ae.state_dict())
    other = tasknets.PointNetAE(n_pc_points=64)
    w.load_state_dict(other.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(ae.state_dict().values(), other.state_dict().values()))
    outer = torch.nn.ModuleDict({"ae": w})                          # nested: the keys stay the module's under the parent's prefix
    assert list(outer.state_dict()) == ["ae." + k for k in ae.state_dict()]
    outer.load_state_dict(outer.state_dict())
    w.eval()
    assert not ae.training
    w.train()
    assert ae.training
    with pytest.raises(RuntimeError, match="CUDA-only"):
        w(torch.rand(4, 64, 3))


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    return ge.build()


@pytest.fixture()
def _tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


@pytest.mark.gpu
def test_routes(sb):
    torch.manual_seed(0)
    ae = tasknets.PointNetAE(n_pc_points=256).cuda()
    w = tasknets.CudaPointNetAE(ae).train()
    x = torch.rand(8, 300, 3, device="cuda")
    w(x)
    assert w.route == "cuda"
    for bad in (x[:1], torch.rand(65, 64, 3, device="cuda"), x.clone().requires_grad_(True)):
        w(bad)
        assert w.route == "module"
    ae.bns[2].momentum = None                                     # a cumulative average: the module's own update
    w(x)
    assert w.route == "module"
    ae.bns[2].momentum = 0.1
    w.eval()
    with torch.no_grad():
        y = w(x)
    assert w.route == "frozen" and torch.allclose(y, ae(x), rtol=1e-4, atol=1e-5)
    w(x)                                                          # grad enabled, parameters trainable: the module
    assert w.route == "module"
    ae.requires_grad_(False)
    w(x)
    assert w.route == "frozen"


def _ae64_pre(net64, x64):
    """Every conv layer's BatchNorm output (B, N, C) and the last layer's activation of the float64 module in training mode."""
    y, pre = x64.permute(0, 2, 1), []
    for conv, bn in zip(net64.convs, net64.bns):
        z = conv(y)
        m, v = z.mean(dim=(0, 2), keepdim=True), z.var(dim=(0, 2), unbiased=False, keepdim=True)
        t = (z - m) / torch.sqrt(v + bn.eps) * bn.weight[None, :, None] + bn.bias[None, :, None]
        pre.append(t.permute(0, 2, 1))
        y = torch.relu(t)
    return pre, y.permute(0, 2, 1)


def _conditioned(net64, x):
    """No routed point's BatchNorm output within KINK_GUARD of 0 in any conv layer, no live pooled maximum within TIE_GUARD of its
    runner-up."""
    pre, y = _ae64_pre(net64, x.double())
    top2 = y.topk(2, dim=1)[0]
    live = top2[:, 0] > 0
    if bool(((top2[:, 0] - top2[:, 1]) <= TIE_GUARD * top2[:, 0])[live].any()):
        return False
    routed = torch.zeros(y.shape[:2], dtype=torch.bool, device=x.device)
    routed.scatter_(1, y.argmax(dim=1), True)
    return not any(bool((t.abs()[routed] <= KINK_GUARD).any()) for t in pre)


def _case(b, n, n_out, bneck=128):
    for seed in range(40):
        torch.manual_seed(seed)
        ae = tasknets.PointNetAE(n_pc_points=n_out, bneck_size=bneck).cuda()
        x = (torch.rand(b, n, 3, generator=torch.Generator().manual_seed(seed)) - 0.5).cuda()
        if _conditioned(copy.deepcopy(ae).double(), x):
            return ae, x
    raise AssertionError("no conditioned instance among the seeds")


def _step64(net64, x, kind):
    """The float64 module's training forward: (reconstruction, its fp32 CUDA loss, the graph's output for a backward)."""
    net64.train()
    rec = net64(x.double())
    return rec.detach(), float(trainers.autoencoder_loss(rec.detach().float(), x, kind)), rec


class _Table:
    """The wrapper's layer stack with the names test_layers_training_parity.reference64 reads (l<i>.w / .b / .g / .beta, layer i in
    spec order), and each name's parameter name in the module."""

    def __init__(self, w):
        self.conv, self.fc, params = w._layer_stack()
        module_name = {id(p): nm for nm, p in w.net.named_parameters()}
        self.named, k = [], 0
        for i, spec in enumerate(self.conv + self.fc):
            for key in ("w", "b") if spec["bn"] is None else ("w", "b", "g", "beta"):
                self.named.append(("l%d.%s" % (i, key), params[k]))
                k += 1
        self.module_name = {nm: module_name[id(p)] for nm, p in self.named}

    def _layer_specs(self):
        return self.conv, self.fc

    def _generator_named_parameters(self):
        return self.named


def _rel_errs(got, ref, table):
    """(per tensor max |got - ref| / its scale, max(its own largest |ref|, 1e-3 of the largest of all); the largest |got| of the conv
    biases over the largest |ref| of all).  A conv bias ahead of a BatchNorm has a zero gradient in exact arithmetic: its fp32 value is
    rounding noise, held to an absolute bar."""
    top = max(float(t.abs().max()) for t in ref.values())
    biases = {table.module_name[nm] for nm, _ in table.named if nm.endswith(".b") and int(nm[1:nm.index(".")]) < len(table.conv)}
    rel = {nm: float((got[nm].double() - ref[nm]).abs().max()) / max(float(ref[nm].abs().max()), 1e-3 * top) for nm in ref if nm not in biases}
    return rel, max(float(got[nm].abs().max()) for nm in biases) / top


def _pinned_masks(table, zs64, zs_kernel):
    """ReLU masks for reference64: the graph's own (BatchNorm output > 0), except at units within AMBIGUOUS of their kink (relative to
    |scale z| + |shift|, float64), which take the CUDA backward's fp32 mask.  Returns (masks, number of pinned units whose mask differs
    from float64's)."""
    from test_layers_training_parity import _bn64, kernel_masks

    masks, flipped = [], 0
    for z64, km, spec in zip(zs64, kernel_masks(table, zs_kernel), table.conv):
        mean, _, inv = _bn64(z64, spec["bn"][4])
        sc = spec["bn"][0].detach().double() * inv
        sh = spec["bn"][1].detach().double() - mean * sc
        y = z64 * sc + sh
        amb = y.abs() <= AMBIGUOUS * (z64.abs() * sc.abs() + sh.abs())
        flipped += int((amb & (km != (y > 0))).sum())
        masks.append(lambda h, z, amb=amb, km=km: torch.where(amb, km, h > 0))
    return masks, flipped


def _saved(out):
    """The forward values CudaPointNetAE's LayerStackFunction kept for its backward: its autograd node is its ctx."""
    node = out.grad_fn
    while not hasattr(node, "cuda_saved"):
        node = node.next_functions[0][0]
    return node.cuda_saved


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,n_out,kind", [(50, 2048, 2048, "chamfer"), (50, 2048, 2048, "emd"), (5, 777, 512, "chamfer")])
def test_cuda_ae_step_against_float64(sb, record_property, _tf32_off, b, n, n_out, kind):
    """One training step of CudaPointNetAE against the float64 module fed the same gradient of the reconstruction: output, loss, running
    statistics and num_batches_tracked against the module; every parameter gradient against reference64 (test_layers_training_parity.py),
    float64 autograd of the same layer stack, with the max-pool at float64's own arg-max.

    ReLU kinks.  The BatchNorm backward makes every point's hidden units carry gradient, and a unit within the fp32 forward's error of its
    kink may take either side in ANY fp32 implementation; at a routed point that moves its channel's gradients by percents (DESIGN §4.8).
    So units within AMBIGUOUS of their kink take the CUDA backward's own mask in the reference, as in test_layers_training_parity.py; the
    ones whose mask that changes are counted."""
    from test_layers_training_parity import reference64

    ae, x = _case(b, n, n_out)
    w, net64 = tasknets.CudaPointNetAE(copy.deepcopy(ae)), copy.deepcopy(ae).double()
    table = _Table(tasknets.CudaPointNetAE(copy.deepcopy(ae)))
    w.train()
    rec = w(x)
    zs_kernel = _saved(rec)[0]
    r32 = rec.detach().requires_grad_(True)
    loss = trainers.autoencoder_loss(r32, x, kind)
    g, = torch.autograd.grad(loss, r32)
    rec.backward(g)
    assert w.route == "cuda"
    out64, loss64, _ = _step64(net64, x, kind)
    e_out = float((rec.detach().double() - out64).abs().max() / out64.abs().max())
    e_loss = abs(float(loss) - loss64) / abs(loss64)
    gf = g.reshape(b, -1)
    _, route64, zs64, _ = reference64(table, x, "bnc", gf)
    masks, flipped = _pinned_masks(table, zs64, zs_kernel)
    ref64, _, _, _ = reference64(table, x, "bnc", gf, route=route64, masks=masks)
    errs, bias_noise = _rel_errs({nm: p.grad for nm, p in w.net.named_parameters()},
                                 {table.module_name[nm]: t for nm, t in ref64.items()}, table)
    e_run = 0.0
    for bn, bn64 in zip(w.net.bns, net64.bns):
        for a, r in ((bn.running_mean, bn64.running_mean), (bn.running_var, bn64.running_var)):
            e_run = max(e_run, float((a.double() - r).abs().max() / r.abs().max()))
        assert int(bn.num_batches_tracked) == int(bn64.num_batches_tracked) == 1
    worst = max(errs, key=errs.get)
    for nm, v in (("out_err", e_out), ("loss_err", e_loss), ("running_err", e_run), ("grad_err", errs[worst]), ("grad_err_tensor", worst),
                  ("conv_bias_noise", bias_noise), ("flipped_pinned_units", flipped)):
        record_property(nm, v)
    assert e_out < OUT_BAR and e_loss < LOSS_BAR and e_run < RUNNING_BAR, (e_out, e_loss, e_run)
    assert errs[worst] < GRAD_BAR and bias_noise < BIAS_NOISE_BAR, (errs, bias_noise)
    assert flipped <= FLIPPED_MAX, flipped


@pytest.mark.gpu
def test_cuda_ae_backward_against_kernel_valued_float64(sb, record_property, _tf32_off):
    """The backward's own arithmetic at 50 x 2048: the training forward and backward entries on the wrapper's layer stack (what
    ops.LayerStackFunction calls) against reference64 with every raw conv output replaced by the kernel's saved value, the kernel's ReLU
    masks and the kernel's route.  Also recorded: the same float64 graph on its own values with the kernel's route and masks (the
    forward's share of the end-to-end distance), and with its own masks (what mask flips at routed units add)."""
    from test_layers_training_parity import _route, kernel_masks, reference64

    ops = sb.ops
    ae, x = _case(50, 2048, 2048)
    table = _Table(tasknets.CudaPointNetAE(copy.deepcopy(ae)))
    conv, fc = table._layer_specs()
    out, _, saved = ops.generator_layers_train_forward(x, "bnc", conv, fc)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(5)).cuda() / out.shape[1]
    grads = ops.generator_layers_backward(x, "bnc", conv, fc, saved, g)
    cuda, k = {}, 0
    for gl, spec in zip(grads, conv + fc):
        for key in ("weight", "bias", "bn_weight", "bn_bias")[:2 if spec["bn"] is None else 4]:
            cuda[table.module_name[table.named[k][0]]] = gl[key]
            k += 1
    zs = saved[0]
    route = _route(zs[-1].double(), conv[-1]["bn"][0].detach().double(), 50)
    km = kernel_masks(table, zs)
    fixed = [lambda h, z, m=m: m for m in km]
    named = lambda d: {table.module_name[nm]: t for nm, t in d.items()}
    kv, _, _, _ = reference64(table, x, "bnc", g, zsave=zs, route=route, masks=fixed)
    _, _, zs64, _ = reference64(table, x, "bnc", g, route=route)
    pinned, _ = _pinned_masks(table, zs64, zs)
    plain_pinned, _, _, _ = reference64(table, x, "bnc", g, route=route, masks=pinned)
    plain_own, _, _, _ = reference64(table, x, "bnc", g, route=route)
    bwd, bias_noise = _rel_errs(cuda, named(kv), table)
    fwd, _ = _rel_errs(named(kv), named(plain_pinned), table)
    flips, _ = _rel_errs(named(plain_pinned), named(plain_own), table)
    record_property("bwd_vs_kernel_valued", max(bwd.values()))
    record_property("conv_bias_noise", bias_noise)
    record_property("forward_values_share", max(fwd.values()))
    record_property("mask_flips_share", max(flips.values()))
    assert max(bwd.values()) < BWD_KERNEL_BAR and bias_noise < BIAS_NOISE_BAR, (bwd, bias_noise)


@pytest.mark.gpu
def test_backward_is_deterministic(sb):
    torch.manual_seed(1)
    ae = tasknets.PointNetAE(n_pc_points=2048).cuda()
    w = tasknets.CudaPointNetAE(ae).train()
    x = torch.rand(50, 2048, 3, device="cuda") - 0.5
    out = w(x)
    g = torch.randn_like(out)
    params = list(ae.parameters())
    g1 = torch.autograd.grad(out, params, g, retain_graph=True)
    g2 = torch.autograd.grad(out, params, g)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    # under a PrimedWorkspaces a second forward leaves what the first one saved alone
    with sb.ops.primed_workspaces(sb.ops.PrimedWorkspaces()):
        out_a = w(x)
        w(2 * x)
    ga = torch.autograd.grad(out_a, params, g)
    assert all(torch.allclose(a, b, rtol=1e-4, atol=1e-6 * float(b.abs().max())) for a, b in zip(ga, g1))
    # a frozen parameter gets a NULL gradient pointer; the others are those of the full backward (a new forward: its BatchNorm
    # statistics are double-precision atomic sums, equal to rounding)
    ae.convs[1].weight.requires_grad_(False)
    out = w(x)
    g3 = torch.autograd.grad(out, [p for p in params if p.requires_grad], g)
    assert all(torch.allclose(a, b, rtol=1e-4, atol=1e-6 * float(b.abs().max()))
               for a, b in zip(g3, [t for t, p in zip(g1, params) if p.requires_grad]))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["chamfer", "emd"])
def test_five_adam_steps_against_the_plain_module(sb, record_property, _tf32_off, kind):
    torch.manual_seed(2)
    ae = tasknets.PointNetAE(n_pc_points=2048).cuda()
    data = [(torch.rand(50, 2048, 3, generator=torch.Generator().manual_seed(10 + i)) - 0.5).cuda() for i in range(5)]
    losses = {}
    for cuda in (False, True):
        net = copy.deepcopy(ae)
        model = tasknets.CudaPointNetAE(net) if cuda else net
        step = trainers.AutoencoderTrainStep(model, torch.optim.Adam(model.parameters(), lr=5e-4), ae_loss=kind)
        losses[cuda] = [float(step(x)) for x in data]
        if cuda:
            assert model.route == "cuda"
    e = max(abs(a - b) / abs(a) for a, b in zip(losses[False], losses[True]))
    record_property("adam_loss_err", e)
    assert e < ADAM_BAR, losses


@pytest.mark.gpu
def test_fps_input(sb):
    torch.manual_seed(3)
    ae = tasknets.PointNetAE(n_pc_points=256).cuda()
    w = tasknets.CudaPointNetAE(ae)
    x = torch.rand(4, 1000, 3, device="cuda")
    step = trainers.AutoencoderTrainStep(w, torch.optim.Adam(w.parameters(), lr=1e-3), use_fps=True, n_sample_points=256)
    assert torch.isfinite(step(x)) and w.route == "cuda"
