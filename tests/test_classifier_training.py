"""The PointNet classifiers trained on CUDA (tasknets.CudaPointNetCls, tasknets.CudaPointNetClsTransforms) and the extended per-layer
training entries under them (snb200_generator_layers_ex_*: an activation input, a tapped layer, FC dropout and the input gradient).

CPU: shared parameters and state-dict keys, refusal of CPU tensors, the routes that need no device, the documented mask draws, and a float64
restatement of each classifier's CUDA split (three layer stacks for the transforms classifier) against the stock module with fixed masks.
GPU (H100): the extended entries with default arguments against the plain ones bit for bit on the per-layer path's tables; the cloud
input's gradient in both layouts; each addition against float64 autograd; whole steps against float64 fed the same masks (pinned at ReLU
kinks and pooled ties of the conv stack, guarded at the FC layers' kinks); five Adam steps against the plain module; bit-identical repeat
backward passes; saved buffers under PrimedWorkspaces; the write sets of the extended entries; the routes.  Measured values are attached
to the test reports."""
import copy
import ctypes
import os
import sys

import pytest
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from samplenet_b200 import tasknets, trainers  # noqa: E402

# Bars (GPU) against float64, relative to the reference's largest magnitude (see the recorded values)
LOGIT_BAR = 4e-4        # [4.0e-5] logits, and the loss, against the float64 module
GRAD_BAR = 1.5e-3       # [1.5e-4] every parameter gradient, whole steps (pinned, guarded) and each addition [2.5e-4] alike
NOISE_BAR = 3e-6        # [2.6e-7] gradients zero in exact arithmetic (_grad_errors): / the largest gradient
RUNNING_BAR = 1e-4      # running statistics
PART_BAR = 5e-5         # [4.2e-6] one addition of the extended entries on its own (small stacks): output
ADAM_BAR = 4e-2         # [4.0e-3] losses of five Adam steps, wrapper against the plain module (TF32 off), relative
AMBIGUOUS = 1e-5        # conv units this close to their ReLU kink (relative) take the CUDA backward's mask in the whole-step reference
TIE_BAR = 1e-4          # [3.1e-5] ... and the max-pool takes the CUDA forward's route, which may leave float64's own only at a gap this
                        # small (relative to the channel's largest activation; the transforms classifier's forward is within 4e-5)

CLASSES = (tasknets.PointNetCls, tasknets.PointNetClsTransforms)
WRAPPERS = {tasknets.PointNetCls: tasknets.CudaPointNetCls, tasknets.PointNetClsTransforms: tasknets.CudaPointNetClsTransforms}


class _FixedMask(nn.Module):
    """nn.Dropout with a given mask: x * mask (the mask already holds 0 or 1/(1-p))."""

    def __init__(self, mask):
        super().__init__()
        self.mask = mask

    def forward(self, x):
        return x * self.mask.to(x.dtype)


def _with_masks(net, masks):
    """A copy of a classifier whose dropouts apply `masks` (in the wrapper's order)."""
    net = copy.deepcopy(net)
    names = [n for n, _ in WRAPPERS[type(net)].DROPOUT]
    for name, m in zip(names, masks):
        setattr(net, name, _FixedMask(m))
    return net


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def _grad_errors(grads, grads64):
    """(largest relative error over the gradients, rounding noise): a gradient that is zero in exact arithmetic -- a bias ahead of a
    BatchNorm, the last conv layer's BatchNorm bias under fc1's BatchNorm over the batch -- has a float64 reference below 1e-6 of the
    largest one, and its fp32 value is measured against that largest gradient instead."""
    scale = max(float(r.abs().max()) for r in grads64)
    worst, noise = 0.0, 0.0
    for a, r in zip(grads, grads64):
        if float(r.abs().max()) <= 1e-6 * scale:
            noise = max(noise, float(a.abs().max()) / scale)
        else:
            worst = max(worst, _rel(a, r))
    return worst, noise


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("cls", CLASSES)
def test_wrapper_shares_the_module(cls):
    torch.manual_seed(0)
    net = cls(num_classes=7)
    w = WRAPPERS[cls](net)
    assert [id(p) for p in w.parameters()] == [id(p) for p in net.parameters()]
    assert list(w.state_dict()) == list(net.state_dict())
    outer = nn.Sequential(w)
    assert list(outer.state_dict()) == ["0." + k for k in net.state_dict()]
    other = cls(num_classes=7)
    other.load_state_dict(w.state_dict())                      # wrapper -> module
    w2 = WRAPPERS[cls](cls(num_classes=7))
    w2.load_state_dict(net.state_dict())                      # module -> wrapper
    nn.Sequential(WRAPPERS[cls](cls(num_classes=7))).load_state_dict(outer.state_dict())
    for a, b in zip(net.state_dict().values(), w2.state_dict().values()):
        assert torch.equal(a, b)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        w(torch.zeros(4, 64, 3))


@pytest.mark.parametrize("cls", CLASSES)
def test_routes_without_a_device(cls):
    """B = 1 and 42 (fc1's input next to its weight rows bounds the FC backward at 41 clouds) and momentum=None take the module's forward;
    these are decided before any layer table reaches the library."""
    w = WRAPPERS[cls](cls()).train()
    meta = lambda b: torch.empty(b, 1024, 3, device="meta")
    assert not w._cuda_supported(meta(1)) and not w._cuda_supported(meta(42))
    w.net.bns[3].momentum = None
    assert not w._cuda_supported(meta(32))


@pytest.mark.parametrize("cls", CLASSES)
def test_masks_rebuild_from_the_seed(cls):
    w = WRAPPERS[cls](cls())
    torch.manual_seed(5)
    masks = w.dropout_masks(6, "cpu")
    torch.manual_seed(5)
    again = [torch.empty(6, width).bernoulli_(1 - getattr(w.net, name).p).div_(1 - getattr(w.net, name).p) for name, width in w.DROPOUT]
    assert len(masks) == len(w.DROPOUT)
    for a, b in zip(masks, again):
        assert torch.equal(a, b)
    w.net.dp1.p = 0.0
    assert w.dropout_masks(6, "cpu")[0] is None


def _stack64(x, convs, fcs, masks=None, tap=None, pin=None):
    """Float64 restatement of one layer stack as the kernels run it: 1x1 convs with BatchNorm over the batch's points and ReLU, max-pool, FC
    layers with BatchNorm over the batch, a mask multiplying an FC layer's input.  Returns (out, pooled, tapped activation).
    pin (see _pin): the max-pool takes the CUDA forward's route, and conv units within AMBIGUOUS of their ReLU kink take its mask."""
    y, h = x, None
    for i, (c, bn) in enumerate(convs):
        z = y @ c.weight[:, :, 0].t() + c.bias
        zf = z.reshape(-1, z.shape[-1])
        sc = bn.weight / torch.sqrt(zf.var(0, unbiased=False) + bn.eps)
        sh = bn.bias - zf.mean(0) * sc
        y = z * sc + sh
        if pin is None or "kmask" not in pin:
            y = torch.relu(y)
        else:
            amb = (y.abs() <= AMBIGUOUS * ((z * sc).abs() + sh.abs())).detach()
            km = pin["kmask"][i].view(y.shape)
            pin["flipped"] += int((amb & (km != (y > 0))).sum())
            y = y * torch.where(amb, km, y > 0).detach().to(y)
        if i == tap:
            h = y
    if pin is None or "route" not in pin:
        pooled = y.max(dim=1)[0]
    else:
        pooled = y.gather(1, pin["route"][:, None, :]).squeeze(1)
        own = y.detach().argmax(dim=1)
        moved = own != pin["route"]
        gap = (y.detach().gather(1, own[:, None, :]) - y.detach().gather(1, pin["route"][:, None, :])).squeeze(1).abs()
        pin["rerouted"] += int(moved.sum())
        pin["reroute_gap"] = max(pin["reroute_gap"], float((gap[moved] / y.detach().abs().amax(dim=1)[moved]).max()) if bool(moved.any()) else 0.0)
    y = pooled
    for i, (lin, bn, relu) in enumerate(fcs):
        if masks and masks.get(i) is not None:
            y = y * masks[i]
        y = y @ lin.weight.t() + lin.bias
        if bn is not None:
            z = y
            sc = bn.weight / torch.sqrt(z.var(0, unbiased=False) + bn.eps)
            sh = bn.bias - z.mean(0) * sc
            y = z * sc + sh
            if relu and pin is not None:   # (kink guard of the FC layers: see test_train_step_against_float64)
                pin["fc_kinks"] += int((y.abs() <= AMBIGUOUS * ((z * sc).abs() + sh.abs())).sum())
        if relu:
            y = torch.relu(y)
    return y, pooled, h


def _split64(net, x, masks, pins=(None, None, None)):
    """The CUDA route's split of a classifier in float64 (module parameters as they are): logits and end_points.  pins: per layer stack,
    in the order the wrapper runs them, None or the CUDA forward's route and ReLU masks (_pin)."""
    if isinstance(net, tasknets.PointNetCls):
        head = [(net.fc1, net.bn_fc1, True), (net.fc2, net.bn_fc2, True), (net.fc3, None, False)]
        logits, gfv, _ = _stack64(x, list(zip(net.convs, net.bns)), head, {2: masks[0]}, pin=pins[0])
        return logits, {"GFV": gfv}
    t1n, t2n = net.transform_net1, net.transform_net2
    tfc = lambda t: [(t.fc1, t.bn_fc1, True), (t.fc2, t.bn_fc2, True), (t.transform, None, False)]
    convs = list(zip(net.convs, net.bns))
    t1 = t1n.to_matrix(_stack64(x, list(zip(t1n.convs, t1n.bns)), tfc(t1n), pin=pins[0])[0])
    x1 = x @ t1
    out2, _, h = _stack64(x1, convs[:2] + list(zip(t2n.convs, t2n.bns)), tfc(t2n), tap=1, pin=pins[1])
    t2 = t2n.to_matrix(out2)
    head = [(net.fc1, net.bn_fc1, True), (net.fc2, net.bn_fc2, True), (net.fc3, None, False)]
    logits, gfv, _ = _stack64(h @ t2, convs[2:], head, {1: masks[0], 2: masks[1]}, pin=pins[2])
    return logits, {"transform": t2, "GFV": gfv}


def _pin(zs, bns, b):
    """What the float64 reference takes from one CUDA layer stack's forward (its raw conv outputs zs): the max-pool's route, the first
    extreme of sign(gamma) * z of the last layer in fp32 as the kernel picks it, and per conv layer the ReLU mask the CUDA backward
    applies, fmaf(scale, z, shift) > 0 with the fp32 scale and shift (as test_layers_training_parity.kernel_masks)."""
    from test_layers_training_parity import _bn64

    kmask = []
    for z, bn in zip(zs, bns):
        mean, var, _ = _bn64(z, bn.eps)
        sc = bn.weight.detach().float() * (1.0 / torch.sqrt(var.float() + bn.eps))
        sh = (bn.bias.detach().double() - mean.float().double() * sc.double()).float()
        kmask.append((z.double() * sc.double() + sh.double()) > 0)
    sgn = torch.where(bns[-1].weight.detach() >= 0, 1.0, -1.0)
    route = (zs[-1].view(b, -1, zs[-1].shape[1]) * sgn).argmax(dim=1)
    return {"kmask": kmask, "route": route, "flipped": 0, "rerouted": 0, "reroute_gap": 0.0, "fc_kinks": 0}


@pytest.mark.parametrize("cls", CLASSES)
def test_split_reference_matches_the_module(cls):
    torch.manual_seed(1)
    net = cls(num_classes=10).double().train()
    for m in net.modules():
        if isinstance(m, nn.BatchNorm1d):
            nn.init.uniform_(m.weight, 0.5, 1.5); nn.init.uniform_(m.bias, -0.2, 0.2)
    if cls is tasknets.PointNetClsTransforms:
        for t in (net.transform_net1, net.transform_net2):
            nn.init.normal_(t.transform.weight, std=0.01)
    x = torch.randn(6, 100, 3, dtype=torch.float64)
    labels = torch.randint(0, 10, (6,))
    masks = [m.double() for m in WRAPPERS[cls](net).dropout_masks(6, "cpu")]
    ref = _with_masks(net, masks)
    logits, ep = ref(x)
    loss = ref.get_loss(logits, labels, ep)
    mine, ep2 = _split64(net, x, masks)
    assert torch.allclose(mine, logits, rtol=1e-10, atol=1e-10)
    assert torch.allclose(ep2["GFV"], ep["GFV"], rtol=1e-12, atol=1e-12)
    assert torch.allclose(net.get_loss(mine, labels, ep2), loss, rtol=1e-10, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    return ge.build()


@pytest.fixture()
def _tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


def _conditioned(cls, seed, classes=40):
    """A classifier instance whose BatchNorm affines keep activations away from degenerate scales (as a trained one would be)."""
    torch.manual_seed(seed)
    net = cls(num_classes=classes)
    for m in net.modules():
        if isinstance(m, nn.BatchNorm1d):
            nn.init.uniform_(m.weight, 0.5, 1.5); nn.init.uniform_(m.bias, -0.2, 0.2)
    if cls is tasknets.PointNetClsTransforms:
        for t in (net.transform_net1, net.transform_net2):
            nn.init.normal_(t.transform.weight, std=0.01)
    return net.cuda().train()


def _tables():
    """Layer tables (conv, fc) of the task networks and samplers the per-layer path trains."""
    from samplenet_b200 import tasknets as t

    out = []
    ae = t.PointNetAE(n_pc_points=128).cuda()
    out.append(("PointNetAE", list(zip(ae.convs, ae.bns)), [(l, None, i < 2) for i, l in enumerate(ae.dec)]))
    cls = t.PointNetCls().cuda()
    out.append(("PointNetCls", list(zip(cls.convs, cls.bns)), [(cls.fc1, cls.bn_fc1, True), (cls.fc2, cls.bn_fc2, True), (cls.fc3, None, False)]))
    return out


def _stack_grads(x, convs, fcs, g, masks=None, tap=-1, g_tap=None):
    """LayerStackFunction on the layers (convs, fcs): (out, feat, tap, [parameter gradients in spec order], x's gradient)."""
    from samplenet_b200 import ops

    conv, fc, params = tasknets._train_specs(convs, fcs)
    if tap >= 0:
        conv[tap]["tap"] = True
    for l, m in (masks or {}).items():
        fc[l]["dropout"] = m
    leaves = [p.detach().clone().requires_grad_() for p in params]
    res = ops.LayerStackFunction.apply(x, conv, fc, *leaves)
    outs = [res[0]] + ([res[2]] if tap >= 0 else [])
    gs = [g] + ([g_tap] if tap >= 0 else [])
    torch.autograd.backward([o for o, gg in zip(outs, gs) if gg is not None], [gg for gg in gs if gg is not None])
    return res[0].detach(), res[1], res[2].detach() if tap >= 0 else None, [p.grad for p in leaves], x.grad


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1])
def test_ex_defaults_match_the_plain_entries_bit_for_bit(sb, which):
    """LayerStackFunction runs the extended entries; with no tap, mask or input gradient they compute what the plain entries compute."""
    from samplenet_b200 import ops

    torch.manual_seed(3)
    name, convs, fcs = _tables()[which]
    bns = [bn for _, bn in convs] + [bn for _, bn, _ in fcs if bn is not None]
    x = torch.randn(8, 300, 3, device="cuda")
    g = torch.randn(8, fcs[-1][0].weight.shape[0], device="cuda")
    for m in bns:
        m.reset_running_stats()
    out, feat, _, grads, _ = _stack_grads(x, convs, fcs, g)
    run = [(m.running_mean.clone(), m.running_var.clone(), m.num_batches_tracked.clone()) for m in bns]
    for m in bns:
        m.reset_running_stats()
    conv, fc, _ = tasknets._train_specs(convs, fcs)
    out0, feat0, saved = ops.generator_layers_train_forward(x, "bnc", conv, fc)
    grads0 = [d[k] for d in ops.generator_layers_backward(x, "bnc", conv, fc, saved, g) for k in ("weight", "bias", "bn_weight", "bn_bias")
              if d[k] is not None]
    assert torch.equal(out, out0) and torch.equal(feat, feat0), name
    for (a, b, c), m in zip(run, bns):
        assert torch.equal(a, m.running_mean) and torch.equal(b, m.running_var) and torch.equal(c, m.num_batches_tracked), name
    assert len(grads) == len(grads0)
    for a, b in zip(grads, grads0):
        assert torch.equal(a, b.view_as(a)), name


def _float64_grads(x, convs, fcs, g, masks=None, tap=None, g_tap=None):
    """float64 autograd of _stack64 on copies of the layers: (out, [parameter gradients in spec order], x's gradient)."""
    convs64 = [(copy.deepcopy(c).double(), copy.deepcopy(bn).double()) for c, bn in convs]
    fcs64 = [(copy.deepcopy(l).double(), None if bn is None else copy.deepcopy(bn).double(), r) for l, bn, r in fcs]
    x64 = x.detach().double().requires_grad_()
    out, _, h = _stack64(x64, convs64, fcs64, {k: v.double() for k, v in (masks or {}).items()}, tap)
    loss = (out * g.double()).sum() + ((h * g_tap.double()).sum() if g_tap is not None else 0)
    loss.backward()
    params = [t for c, bn in convs64 for t in (c.weight, c.bias, bn.weight, bn.bias)]
    params += [t for l, bn, _ in fcs64 for t in ((l.weight, l.bias) if bn is None else (l.weight, l.bias, bn.weight, bn.bias))]
    return out.detach(), [p.grad for p in params], x64.grad


def _small_stack(c_in, seed):
    torch.manual_seed(seed)
    w = [c_in, 64, 64, 128, 256]
    convs = [(nn.Conv1d(w[i], w[i + 1], 1).cuda(), nn.BatchNorm1d(w[i + 1], eps=1e-3).cuda()) for i in range(4)]
    for _, bn in convs:
        nn.init.uniform_(bn.weight, 0.5, 1.5); nn.init.uniform_(bn.bias, 0.0, 0.3)
    fcs = [(nn.Linear(256, 128).cuda(), nn.BatchNorm1d(128, eps=1e-3).cuda(), True), (nn.Linear(128, 64).cuda(), nn.BatchNorm1d(64, eps=1e-3).cuda(), True),
           (nn.Linear(64, 10).cuda(), None, False)]
    return convs, fcs


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cloud_grad_in", "act_input", "tap", "tap_and_out", "dropout"])
def test_each_addition_against_float64(sb, record_property, _tf32_off, case):
    act = case == "act_input"
    convs, fcs = _small_stack(64 if act else 3, 11)
    b, n = 6, 200
    torch.manual_seed(12)
    x = (torch.randn(b, n, 64, device="cuda").relu() if act else torch.randn(b, n, 3, device="cuda")).requires_grad_(case in ("cloud_grad_in", "act_input"))
    g = torch.randn(b, 10, device="cuda")
    tap = 1 if case.startswith("tap") else -1
    g_tap = torch.randn(b, n, 64, device="cuda") * 1e-3 if tap >= 0 else None
    if case == "tap":
        g = None
    masks = {1: (torch.rand(b, 128, device="cuda") > 0.3).float() / 0.7, 2: (torch.rand(b, 64, device="cuda") > 0.3).float() / 0.7} \
        if case == "dropout" else None
    out, _, _, grads, gx = _stack_grads(x, convs, fcs, g, masks, tap, g_tap)
    ref, grads64, gx64 = _float64_grads(x, convs, fcs, torch.zeros(b, 10, device="cuda") if g is None else g, masks, tap if tap >= 0 else None, g_tap)
    worst, noise = _grad_errors(grads, grads64)
    record_property("out_rel", _rel(out, ref))
    record_property("grad_rel_max", worst)
    record_property("bias_noise", noise)
    assert _rel(out, ref) < PART_BAR and worst < GRAD_BAR and noise < NOISE_BAR
    if x.requires_grad:
        record_property("grad_in_rel", _rel(gx, gx64))
        assert _rel(gx, gx64) < GRAD_BAR


@pytest.mark.gpu
def test_all_ones_mask_is_bit_identical_to_none(sb):
    convs, fcs = _small_stack(3, 13)
    x = torch.randn(6, 200, 3, device="cuda")
    g = torch.randn(6, 10, device="cuda")
    a = _stack_grads(x, convs, fcs, g)
    ones = {1: torch.ones(6, 128, device="cuda"), 2: torch.ones(6, 64, device="cuda")}
    b = _stack_grads(x, convs, fcs, g, ones)
    assert torch.equal(a[0], b[0])
    for u, v in zip(a[3], b[3]):
        assert torch.equal(u, v)


def _cuda_step(cls, net, x, labels, masks):
    w = WRAPPERS[cls](net)
    w.dropout_masks = lambda b, device: masks
    logits, ep = w(x)
    assert w.route == "cuda"
    loss = w.get_loss(logits, labels, ep)
    loss.backward()
    return logits.detach(), loss.detach(), w


def _stack_bns(net):
    """The BatchNorms of each layer stack of the wrapper's split, in the order it runs them."""
    if isinstance(net, tasknets.PointNetCls):
        return [list(net.bns)]
    t1n, t2n = net.transform_net1, net.transform_net2
    return [list(t1n.bns), list(net.bns[:2]) + list(t2n.bns), list(net.bns[2:])]


@pytest.mark.gpu
@pytest.mark.parametrize("cls", CLASSES)
@pytest.mark.parametrize("b,n", [(32, 1024), (5, 777)])
def test_train_step_against_float64(sb, record_property, monkeypatch, _tf32_off, cls, b, n):
    """A whole ClassifierTrainStep-sized step of the wrapper against float64 fed the same masks: logits, loss (with the transform
    regulariser), running statistics and num_batches_tracked against the float64 module; every parameter gradient against the float64
    split (_split64) pinned to the CUDA forward where fp32 cannot decide: a conv unit within AMBIGUOUS of its ReLU kink takes the CUDA
    backward's mask, and the max-pool takes the CUDA forward's route (a route float64 would move is allowed only at a TIE_BAR tie).  Without
    the pins, the few units and pooled maxima within an fp32 rounding of a kink or a tie send a whole channel's gradient elsewhere."""
    from samplenet_b200 import ops

    net = _conditioned(cls, 21)
    ref = copy.deepcopy(net).double()
    for seed in range(22, 72):   # kink guard: the first batch with no FC unit within AMBIGUOUS of its ReLU kink in float64
        torch.manual_seed(seed)
        x = torch.randn(b, n, 3, device="cuda")
        labels = torch.randint(0, 40, (b,), device="cuda")
        masks = WRAPPERS[cls](net).dropout_masks(b, "cuda")
        guard = [{"fc_kinks": 0} for _ in range(3)]
        with torch.no_grad():
            _split64(ref, x.double(), [m.double() for m in masks], guard)
        if sum(gd["fc_kinks"] for gd in guard) == 0:
            break
    record_property("guard_seed", seed)
    saved, apply = [], ops.LayerStackFunction.apply

    def recording(*args):
        res = apply(*args)
        saved.append(res[0].grad_fn.cuda_saved[0])
        return res
    monkeypatch.setattr(ops.LayerStackFunction, "apply", recording)
    logits, loss, _ = _cuda_step(cls, net, x, labels, masks)
    ref = _with_masks(ref, [m.double() for m in masks])
    l64, ep64 = ref(x.double())
    loss64 = ref.get_loss(l64, labels, ep64)
    record_property("logits_rel", _rel(logits, l64))
    record_property("loss_rel", abs(float(loss) - float(loss64)) / abs(float(loss64)))
    assert _rel(logits, l64) < LOGIT_BAR and abs(float(loss) - float(loss64)) < LOGIT_BAR * abs(float(loss64))
    for (k, t), (_, t64) in zip(net.named_buffers(), ref.named_buffers()):
        if k.endswith("num_batches_tracked"):
            assert int(t) == int(t64) == 1, k
        else:
            assert _rel(t, t64) < RUNNING_BAR, k
    net64 = copy.deepcopy(_conditioned(cls, 21)).double()
    pins = [_pin(zs, bns, b) for zs, bns in zip(saved, _stack_bns(net))]
    p64, ep = _split64(net64, x.double(), [m.double() for m in masks], pins)
    net64.get_loss(p64, labels, ep).backward()
    names = [k for k, _ in net.named_parameters()]
    grads64 = [p.grad if p.grad is not None else torch.zeros_like(p) for p in net64.parameters()]
    worst, noise = _grad_errors([p.grad for p in net.parameters()], grads64)
    per = {k: _rel(p.grad, r) for k, p, r in zip(names, net.parameters(), grads64) if float(r.abs().max()) > 1e-6 * max(float(t.abs().max()) for t in grads64)}
    record_property("grad_rel_max", worst)
    record_property("grad_rel_max_at", max(per, key=per.get))
    record_property("bias_noise", noise)
    record_property("pinned_units_flipped", sum(pn["flipped"] for pn in pins))
    record_property("pool_rerouted", sum(pn["rerouted"] for pn in pins))
    record_property("pool_reroute_gap_max", max(pn["reroute_gap"] for pn in pins))
    record_property("fc_units_at_kink", sum(pn["fc_kinks"] for pn in pins))
    assert max(pn["reroute_gap"] for pn in pins) <= TIE_BAR
    # kink guard of the FC layers (the batch was drawn so): BatchNorm over 5 .. 32 rows makes a unit's mask move its whole channel, so no FC
    # unit may be within AMBIGUOUS of its kink (the conv units' masks are pinned instead: their channels hold thousands of points)
    assert sum(pn["fc_kinks"] for pn in pins) == 0
    assert worst < GRAD_BAR and noise < NOISE_BAR, (max(per, key=per.get), worst, noise)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", CLASSES)
def test_repeat_backward_is_bit_identical(sb, cls):
    net = _conditioned(cls, 31)
    x = torch.randn(16, 512, 3, device="cuda")
    labels = torch.randint(0, 40, (16,), device="cuda")
    masks = WRAPPERS[cls](net).dropout_masks(16, "cuda")
    state = copy.deepcopy(net.state_dict())
    grads = []
    for _ in range(2):
        net.load_state_dict(state)
        net.zero_grad()
        _cuda_step(cls, net, x, labels, masks)
        grads.append([p.grad.clone() for p in net.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", CLASSES)
def test_five_adam_steps_against_the_plain_module(sb, record_property, _tf32_off, cls):
    net = _conditioned(cls, 41)
    plain = copy.deepcopy(net)
    torch.manual_seed(42)
    batches = [(torch.randn(32, 1024, 3, device="cuda"), torch.randint(0, 40, (32,), device="cuda")) for _ in range(5)]
    w = WRAPPERS[cls](net)
    masks = [w.dropout_masks(32, "cuda") for _ in range(5)]
    it = iter(masks)
    w.dropout_masks = lambda b, device: next(it)
    plain_masked = _with_masks(plain, masks[0])
    s1 = trainers.ClassifierTrainStep(w, torch.optim.Adam(w.parameters(), lr=1e-3))
    s2 = trainers.ClassifierTrainStep(plain_masked, torch.optim.Adam(plain_masked.parameters(), lr=1e-3))
    worst = 0.0
    for k, (x, y) in enumerate(batches):
        for (name, _), m in zip(w.DROPOUT, masks[k]):
            getattr(plain_masked, name).mask = m
        l1, _, _ = s1(x, y)
        assert w.route == "cuda"
        l2, _, _ = s2(x, y)
        worst = max(worst, abs(float(l1) - float(l2)) / abs(float(l2)))
    record_property("loss_rel_max", worst)
    assert worst < ADAM_BAR


@pytest.mark.gpu
@pytest.mark.parametrize("cls", CLASSES)
def test_routes(sb, cls):
    net = _conditioned(cls, 51)
    w = WRAPPERS[cls](net)
    w(torch.randn(8, 256, 3, device="cuda"))
    assert w.route == "cuda"
    w(torch.randn(42, 64, 3, device="cuda"))
    assert w.route == "module"
    w(torch.randn(8, 256, 3, device="cuda", requires_grad=True))
    assert w.route == "module"
    net.requires_grad_(False)
    w.eval()
    with torch.no_grad():
        logits, _ = w(torch.randn(8, 256, 3, device="cuda"))
    assert w.route == "frozen" and logits.shape == (8, 40)


# ------------------------------------------------------------------------------------------------------------------ the C entries
# conv widths, FC widths, FC BatchNorm, FC ReLU, eps: the per-layer path's existing users (SampleNet at k = 128, the classification sampler
# at its 1024 bottleneck, the reconstruction sampler, PointNetAE) and a 128-wide first layer
EX_TABLES = {
    "SampleNet": ([3, 64, 64, 64, 128, 128], [128, 256, 256, 256, 192], [1, 1, 1, 0], [1, 1, 1, 0], 1e-5),
    "ClassificationSampleNet": ([3, 64, 64, 64, 128, 1024], [1024, 256, 256, 256, 192], [1, 1, 1, 1], [1, 1, 1, 0], 1e-3),
    "ReconstructionSampleNet": ([3, 64, 128, 128, 256, 128], [128, 256, 256, 192], [0, 0, 0], [1, 1, 0], 1e-3),
    "PointNetAE": ([3, 64, 128, 128, 256, 128], [128, 256, 256, 6144], [0, 0, 0], [1, 1, 0], 1e-3),
    "conv1-128": ([3, 128, 128, 128], [128, 256, 192], [1, 0], [1, 0], 1e-5),
}


def _ex_table(name, seed, alloc):
    """(conv specs, FC specs) of a table, every tensor from alloc(name, shape, fill, dtype)."""
    conv_w, fc_w, fc_bn, fc_relu, eps = EX_TABLES[name] if isinstance(name, str) else name
    g = torch.Generator().manual_seed(seed)

    def layer(nm, c_in, c_out, bn, relu):
        spec = dict(weight=alloc(nm + ".weight", (c_out, c_in), torch.randn(c_out, c_in, generator=g) / c_in ** 0.5),
                    bias=alloc(nm + ".bias", (c_out,), 0.1 * torch.randn(c_out, generator=g)), relu=bool(relu), bn=None)
        if bn:
            spec["bn"] = (alloc(nm + ".bn_weight", (c_out,), 1 + 0.2 * torch.randn(c_out, generator=g)),
                          alloc(nm + ".bn_bias", (c_out,), 0.1 * torch.randn(c_out, generator=g)),
                          alloc(nm + ".running_mean", (c_out,), torch.zeros(c_out)), alloc(nm + ".running_var", (c_out,), torch.ones(c_out)),
                          eps, 0.1, alloc(nm + ".num_batches_tracked", (1,), torch.zeros(1, dtype=torch.int64), torch.int64))
        return spec

    conv = [layer("conv%d" % i, conv_w[i], conv_w[i + 1], True, True) for i in range(len(conv_w) - 1)]
    return conv, [layer("fc%d" % i, fc_w[i], fc_w[i + 1], fc_bn[i], fc_relu[i]) for i in range(len(fc_w) - 1)]


def _plain_alloc(name, shape, fill, dtype=torch.float32):
    return fill.to("cuda", dtype).reshape(shape).contiguous()


class _Entries:
    """One training step through the C entries on caller-owned buffers (alloc), the plain ones or the extended ones."""

    def __init__(self, conv, fc, b, n, alloc, tag=""):
        import samplenet_b200 as sb

        self.sb, self.lib, self.alloc, self.tag = sb, sb._lib.lib(), alloc, tag
        self.conv_specs, self.fc_specs, self.b, self.n = conv, fc, b, n
        self.conv, _ = sb.ops.make_layers(conv)
        self.fc, _ = sb.ops.make_layers(fc)
        self.nc, self.nf = len(conv), len(fc)

    def bn_buffers(self):
        return [t for s in self.conv_specs + self.fc_specs if s["bn"] is not None for t in (s["bn"][2], s["bn"][3], s["bn"][6])]

    def forward(self, x, layout, ex=None):
        """ex: None (plain entry) or dict(act_input, tap, dropout: {fc layer: mask}).  Returns what it wrote."""
        a, lib, b, n = self.alloc, self.lib, self.b, self.n
        lay = self.sb._lib.BNC if layout == "bnc" else self.sb._lib.BCN
        wsb = int(lib.snb200_generator_workspace_bytes(b, n, self.nc, self.conv, self.nf, self.fc))
        self.ws = a(self.tag + "workspace", (wsb,), torch.zeros(wsb, dtype=torch.uint8), torch.uint8)
        self.zs = [a(self.tag + "zsave%d" % l, (b * n, self.conv[l].c_out), torch.zeros(b * n, self.conv[l].c_out)) for l in range(self.nc)]
        zp = (ctypes.c_void_p * self.nc)(*[z.data_ptr() for z in self.zs])
        self.out = a(self.tag + "out", (b, self.fc[self.nf - 1].c_out), torch.zeros(b, self.fc[self.nf - 1].c_out))
        self.feat = a(self.tag + "feat", (b, self.conv[self.nc - 1].c_out), torch.zeros(b, self.conv[self.nc - 1].c_out))
        self.x, self.layout, self.ex = x, lay, ex
        self.tap_out = None
        if ex is None:
            rc = lib.snb200_generator_layers_train_forward(b, n, lay, x.data_ptr(), self.nc, self.conv, self.nf, self.fc, self.out.data_ptr(), 0,
                                                           self.feat.data_ptr(), zp, 0, self.ws.data_ptr(), wsb, None)
        else:
            tap = ex.get("tap", -1)
            if tap >= 0:
                self.tap_out = a(self.tag + "tap_out", (b * n, self.conv[tap].c_out), torch.zeros(b * n, self.conv[tap].c_out))
            self.drop = (ctypes.c_void_p * self.nf)(*[ex.get("dropout", {}).get(l).data_ptr() if l in ex.get("dropout", {}) else None
                                                      for l in range(self.nf)])
            rc = lib.snb200_generator_layers_ex_train_forward(b, n, lay, int(ex.get("act_input", 0)), x.data_ptr(), self.nc, self.conv, self.nf,
                                                              self.fc, tap, None if self.tap_out is None else self.tap_out.data_ptr(), self.drop,
                                                              self.out.data_ptr(), 0, self.feat.data_ptr(), zp, 0, self.ws.data_ptr(), wsb, None)
        self.sb._lib.check(rc, "train forward")
        return [self.ws] + self.bn_buffers(), [self.out, self.feat] + self.zs + ([self.tap_out] if self.tap_out is not None else [])

    def backward(self, grad_out, grad_tap=None, grad_in=False):
        a, lib, b, n, ex = self.alloc, self.lib, self.b, self.n, self.ex
        act = int(ex.get("act_input", 0)) if ex else 0
        if ex is None:
            bwsb = int(lib.snb200_generator_layers_backward_workspace_bytes(b, n, self.nc, self.conv, self.nf, self.fc))
        else:
            bwsb = int(lib.snb200_generator_layers_ex_backward_workspace_bytes(b, n, act, self.nc, self.conv, self.nf, self.fc))
        bws = a(self.tag + "backward_workspace", (bwsb,), torch.zeros(bwsb, dtype=torch.uint8), torch.uint8)
        self.grads = []

        def gstructs(specs, kind):
            arr = (self.sb._lib.LayerGrad * len(specs))()
            for i, s in enumerate(specs):
                c_out, c_in = s["weight"].shape
                nm = "%sgrad.%s%d" % (self.tag, kind, i)
                g = [a(nm + ".weight", (c_out, c_in), torch.zeros(c_out, c_in)), a(nm + ".bias", (c_out,), torch.zeros(c_out))]
                if s["bn"] is not None:
                    g += [a(nm + ".bn_weight", (c_out,), torch.zeros(c_out)), a(nm + ".bn_bias", (c_out,), torch.zeros(c_out))]
                arr[i].weight, arr[i].bias = g[0].data_ptr(), g[1].data_ptr()
                arr[i].bn_weight, arr[i].bn_bias = (g[2].data_ptr(), g[3].data_ptr()) if len(g) > 2 else (None, None)
                self.grads.extend(g)
            return arr
        gconv, gfc = gstructs(self.conv_specs, "conv"), gstructs(self.fc_specs, "fc")
        zp = (ctypes.c_void_p * self.nc)(*[z.data_ptr() for z in self.zs])
        self.grad_in = a(self.tag + "grad_in", tuple(self.x.shape), torch.zeros(tuple(self.x.shape))) if grad_in else None
        self.backward_call = lambda: self._backward_call(grad_out, grad_tap, gconv, gfc, zp, bws, bwsb)
        self.backward_call()
        return [bws], self.grads + ([self.grad_in] if self.grad_in is not None else [])

    def _backward_call(self, grad_out, grad_tap, gconv, gfc, zp, bws, bwsb):
        lib, b, n, ex = self.lib, self.b, self.n, self.ex
        act = int(ex.get("act_input", 0)) if ex else 0
        if ex is None:
            rc = lib.snb200_generator_layers_backward(b, n, self.layout, self.x.data_ptr(), self.nc, self.conv, self.nf, self.fc, zp, self.ws.data_ptr(),
                                                      grad_out.data_ptr(), 0, gconv, gfc, bws.data_ptr(), bwsb, None)
        else:
            rc = lib.snb200_generator_layers_ex_backward(b, n, self.layout, act, self.x.data_ptr(), self.nc, self.conv, self.nf, self.fc, ex.get("tap", -1),
                                                         self.drop, zp, self.ws.data_ptr(), grad_out.data_ptr(), 0,
                                                         None if grad_tap is None else grad_tap.data_ptr(),
                                                         None if self.grad_in is None else self.grad_in.data_ptr(), gconv, gfc, bws.data_ptr(), bwsb, None)
        self.sb._lib.check(rc, "backward")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EX_TABLES))
def test_ex_entries_with_defaults_are_the_plain_entries(sb, name):
    """The extended entries with act_input = 0, tap = -1, no masks and grad_in = NULL against the plain generator_layers_* entries, bit for
    bit: output, pooled feature, saved activations, running statistics, num_batches_tracked and every gradient."""
    b, n = 8, 300
    conv, fc = _ex_table(name, 4, _plain_alloc)
    x = torch.randn(b, n, 3, generator=torch.Generator().manual_seed(5)).cuda()
    g = torch.randn(b, fc[-1]["weight"].shape[0], generator=torch.Generator().manual_seed(6)).cuda()
    e = _Entries(conv, fc, b, n, _plain_alloc)
    init = [t.clone() for t in e.bn_buffers()]
    runs = []
    for ex in (None, {}):
        for t, v in zip(e.bn_buffers(), init):
            t.copy_(v)
        _, fwd = e.forward(x, "bnc", ex)
        _, grads = e.backward(g)
        runs.append([t.clone() for t in fwd + e.bn_buffers() + grads])
    for i, (u, v) in enumerate(zip(*runs)):
        assert torch.equal(u, v), (name, i)


@pytest.mark.gpu
def test_cloud_input_gradient_in_both_layouts(sb):
    """grad_in of a cloud input in BCN is the BNC one transposed, bit for bit (the same per-point sums; BNC is checked against float64 in
    test_each_addition_against_float64), and so is every parameter gradient."""
    b, n = 6, 333
    conv, fc = _ex_table("SampleNet", 7, _plain_alloc)
    x = torch.randn(b, n, 3, generator=torch.Generator().manual_seed(8)).cuda()
    g = torch.randn(b, 192, generator=torch.Generator().manual_seed(9)).cuda()
    e = _Entries(conv, fc, b, n, _plain_alloc)
    init = [t.clone() for t in e.bn_buffers()]
    res = []
    for layout, xi in (("bnc", x), ("bcn", x.permute(0, 2, 1).contiguous())):
        for t, v in zip(e.bn_buffers(), init):
            t.copy_(v)
        e.forward(xi, layout, {})
        _, grads = e.backward(g, grad_in=True)
        res.append([t.clone() for t in grads])
    assert torch.equal(res[0][-1], res[1][-1].permute(0, 2, 1))
    assert float(res[0][-1].abs().max()) > 0
    for u, v in zip(res[0][:-1], res[1][:-1]):
        assert torch.equal(u, v)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cloud", "activation"])
def test_ex_entries_write_only_their_buffers(sb, case):
    """The extended entries with every addition on, every buffer carved from a poisoned arena (test_write_sets.py's harness): the forward
    writes its workspace, the BatchNorm buffers and, wholly, out, feat, the saved activations and tap_out; the backward its workspace and,
    wholly, every gradient and grad_in; nothing else."""
    from test_write_sets import POISON, Arena, assert_clean, run_checked

    arena = Arena()
    alloc = lambda nm, shape, fill, dtype=torch.float32: arena.carve(nm, shape, dtype=dtype, fill=fill.reshape(shape).to(dtype))
    b, n = 7, 333
    if case == "cloud":
        table = ([3, 64, 64, 64, 128, 1024], [1024, 512, 256, 40], [1, 1, 0], [1, 1, 0], 1e-3)
        x = alloc("x", (b, 3, n), torch.randn(b, 3, n))
        layout, ex = "bcn", {"tap": 1}
    else:
        table = ([64, 64, 128, 1024], [1024, 512, 256, 40], [1, 1, 0], [1, 1, 0], 1e-3)
        x = alloc("x", (b, n, 64), torch.randn(b, n, 64).relu())
        layout, ex = "bnc", {"act_input": 1, "tap": 0}
    conv, fc = _ex_table(table, 3, alloc)
    ex["dropout"] = {1: alloc("mask1", (b, 512), (torch.rand(b, 512) > 0.3).float() / 0.7),
                     2: alloc("mask2", (b, 256), (torch.rand(b, 256) > 0.3).float() / 0.7)}
    e = _Entries(conv, fc, b, n, alloc, "step.")
    poison = lambda ts: [t.view(torch.int32).fill_(POISON) for t in ts]
    w, full = e.forward(x, layout, ex)                      # carves the buffers; the checked call reissues it on them, outputs re-poisoned
    zp = (ctypes.c_void_p * e.nc)(*[z.data_ptr() for z in e.zs])
    poison(full)
    rep = run_checked(arena, "ex forward", lambda: e.sb._lib.check(e.lib.snb200_generator_layers_ex_train_forward(
        b, n, e.layout, int(ex.get("act_input", 0)), x.data_ptr(), e.nc, e.conv, e.nf, e.fc, ex["tap"], e.tap_out.data_ptr(), e.drop,
        e.out.data_ptr(), 0, e.feat.data_ptr(), zp, 0, e.ws.data_ptr(), e.ws.numel(), None), "ex forward"), w, full=full)
    grad_out = alloc("grad_out", (b, 40), torch.randn(b, 40))
    grad_tap = alloc("grad_tap", (b * n, 64), 1e-3 * torch.randn(b * n, 64))
    w, full = e.backward(grad_out, grad_tap, grad_in=True)
    poison(full)
    rep += run_checked(arena, "ex backward", e.backward_call, w, full=full)
    assert_clean(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", CLASSES)
def test_saved_buffers_survive_a_second_forward_under_primed_workspaces(sb, cls):
    """LayerStackFunction keeps its own saved activations and forward workspace even under an active PrimedWorkspaces: a second forward
    before the first one's backward leaves that backward's gradients bit for bit what they are without it."""
    from samplenet_b200 import ops

    net = _conditioned(cls, 61)
    w = WRAPPERS[cls](net)
    x1, x2 = torch.randn(8, 256, 3, device="cuda"), torch.randn(8, 256, 3, device="cuda")
    labels = torch.randint(0, 40, (8,), device="cuda")
    masks = w.dropout_masks(8, "cuda")
    w.dropout_masks = lambda b, device: masks
    grads = []
    for second in (False, True):
        net.zero_grad()
        with ops.primed_workspaces(ops.PrimedWorkspaces()):
            logits, ep = w(x1)
            if second:
                w(x2)
            w.get_loss(logits, labels, ep).backward()
        assert w.route == "cuda"
        grads.append([p.grad.clone() for p in net.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)
