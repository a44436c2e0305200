"""PCRNet trained on CUDA: the weight and bias gradients of the frozen encoder's and the frozen MLP's kernels (snb200_frozen_encoder_param_backward,
snb200_frozen_mlp_param_backward, ops.EncoderParamFunction / MLPParamFunction), registration.CudaPCRNet and RegistrationStep.create_model(cuda_task=True).

CPU: the entries' envelopes, workspace sizes and refusals (nothing launches), the wrapper's and the factory's refusals, the kernels' stack frames.
GPU (H100): dW / db against float64 on the kernels' own routes, masks and saved activations, with each element normalised by its sum of |terms|;
grad_in / grad_x bit-identical to the entries without parameter gradients; repeat runs bit-identical; CudaPCRNet plus the pose loss against
float64 autograd of PCRNet; whole train steps against the plain module; write sets.  Measured values are attached to the test reports."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from samplenet_b200 import registration as reg  # noqa: E402

# Bars (GPU), about 10x the largest value measured on an H100 80GB HBM3 (in brackets)
MLP_PARAM_BAR = 2e-6    # [1.8e-7] dW / db against float64 on the kernel's masks, per element / sum of |terms|
ENC_PARAM_BAR = 2.5e-6  # [2.2e-7] the same for the encoder, on the kernel's routes and masks
NET_BAR = 2e-5          # [1.7e-6] CudaPCRNet + pose loss against float64 autograd: per tensor, / max |reference|
STEP_BAR = 2e-5         # [2.0e-6] a first train step against the plain module (TF32 off): loss relative, each gradient / its max |value|
ADAM_BAR = 1e-4         # [1.9e-7] losses of five Adam steps, relative
JOINT_BAR = 5e-2        # [6.2e-3] the joint step's gradients: 64-point sampled clouds, unconditioned (see the test)

PCR_W = [2048, 1024, 1024, 512, 512, 256, 7]
ODD_W = [264, 40, 7]
PCR_CONV = [3, 64, 64, 64, 128, 1024]

_next_ptr = [0x90000]


def _ptr():
    _next_ptr[0] += 0x1000
    return _next_ptr[0]


def _table(widths, bn_at=None, relu_last=False):
    from samplenet_b200._lib import Layer
    arr = (Layer * (len(widths) - 1))()
    for i in range(len(widths) - 1):
        L = arr[i]
        L.c_in, L.c_out, L.weight, L.bias = widths[i], widths[i + 1], _ptr(), _ptr()
        if bn_at == i:
            L.bn_weight, L.bn_bias = _ptr(), _ptr()
        L.relu = int(i < len(widths) - 2 or relu_last)
    return arr


def _grads(nl, bn_at=None, misalign_at=None):
    from samplenet_b200._lib import LayerGrad
    arr = (LayerGrad * nl)()
    for i in range(nl):
        arr[i].weight, arr[i].bias = _ptr() + (4 if i == misalign_at else 0), _ptr()
        if i == bn_at:
            arr[i].bn_weight = _ptr()
    return arr


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


def _align(v):
    return (v + 255) // 256 * 256


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_param_entries_envelopes_and_workspaces(lib):
    t = _table(PCR_W)
    for b in (1, 7, 32, 64):
        assert lib.snb200_frozen_mlp_param_backward_supported(b, 6, t) == 1
        assert lib.snb200_frozen_mlp_param_backward_workspace_bytes(b, 6, t) == lib.snb200_frozen_mlp_backward_workspace_bytes(b, 6, t) > 0
    assert lib.snb200_frozen_mlp_param_backward_supported(5, 2, _table(ODD_W)) == 1
    assert lib.snb200_frozen_mlp_param_backward_supported(65, 6, t) == 0 and lib.snb200_frozen_mlp_param_backward_workspace_bytes(65, 6, t) == 0
    assert lib.snb200_frozen_mlp_param_backward_supported(32, 6, _table(PCR_W, bn_at=3)) == 0
    c = _table(PCR_CONV, relu_last=True)
    for b, n in ((64, 1024), (64, 64), (2, 1000), (5, 333), (1, 129)):
        assert lib.snb200_frozen_encoder_param_backward_supported(b, n, 5, c, 1) == 1
        # the route bits, then per hidden layer its dense dz rows and its chunk partials (at least 256 points per chunk, at most 256 chunks)
        pts = b * n
        chunks = min(256, (pts + 255) // 256)
        want = _align(pts * 32 * 4) + sum(_align(pts * PCR_CONV[l + 1] * 4) + _align(chunks * PCR_CONV[l + 1] * (PCR_CONV[l] + 1) * 4) for l in range(4))
        assert lib.snb200_frozen_encoder_param_backward_workspace_bytes(b, n, 5, c, 1) == want
        assert lib.snb200_frozen_encoder_backward_workspace_bytes(b, n, 5, c, 1) == _align(pts * 32 * 4)
    assert lib.snb200_frozen_encoder_param_backward_workspace_bytes(64, 1024, 5, c, 1) < 110 << 20
    assert lib.snb200_frozen_encoder_param_backward_supported(65, 64, 5, c, 1) == 0
    assert lib.snb200_frozen_encoder_param_backward_supported(8, 4097, 5, c, 1) == 0
    assert lib.snb200_frozen_encoder_param_backward_supported(8, 64, 5, c, 17) == 0
    cb = _table(PCR_CONV, bn_at=2, relu_last=True)
    assert lib.snb200_frozen_encoder_supported(8, 64, 5, cb, 1) == 1       # the frozen encoder takes BatchNorm ...
    assert lib.snb200_frozen_encoder_param_backward_supported(8, 64, 5, cb, 1) == 0 and \
        lib.snb200_frozen_encoder_param_backward_workspace_bytes(8, 64, 5, cb, 1) == 0     # ... the parameter backward does not


def test_param_entries_refuse_before_any_launch(lib):
    """Outside the envelope SNB200_EUNSUPPORTED (-4), bad gradient pointers and null arguments SNB200_EINVAL (-1), short workspaces
    SNB200_EWORKSPACE (-2), each with its message; the pointers are never dereferenced and this runs without a device."""
    big = 1 << 40
    z = (ctypes.c_void_p * 8)(*[_ptr() for _ in range(8)])

    def err():
        return lib.snb200_last_error().decode()

    t = _table(PCR_W)
    mlp = lambda b, tab, g, **kw: lib.snb200_frozen_mlp_param_backward(b, 6, tab, kw.get("x", _ptr()), z, _ptr(), kw.get("gin", _ptr()), g, _ptr(),
                                                                       kw.get("ws", big), None)
    assert mlp(65, t, _grads(6)) == -4 and err().startswith("frozen_mlp_param_backward: outside the frozen MLP's envelope")
    assert mlp(32, _table(PCR_W, bn_at=1), _grads(6)) == -4
    assert mlp(32, t, _grads(6, bn_at=2)) == -1 and "no BatchNorm" in err()
    assert mlp(32, t, _grads(6, misalign_at=4)) == -1 and "16-byte aligned" in err()
    assert mlp(32, t, None) == -1 and "grads is null" in err()
    assert mlp(32, t, _grads(6), x=None) == -1 and "null pointer" in err()          # layer 1's weight gradient reads `in`
    assert mlp(32, t, _grads(6), ws=lib.snb200_frozen_mlp_param_backward_workspace_bytes(32, 6, t) - 1) == -2
    assert lib.snb200_frozen_mlp_backward(32, 6, t, z, _ptr(), None, _ptr(), big, None) == -1    # the entry without parameters needs grad_in

    c = _table(PCR_CONV, relu_last=True)
    sizes = (ctypes.c_int * 1)(64)
    enc = lambda b, tab, g, **kw: lib.snb200_frozen_encoder_param_backward(b, 64, _ptr(), 5, tab, 1, sizes, _ptr(), _ptr(), z, _ptr(), kw.get("gx", _ptr()),
                                                                           g, _ptr(), kw.get("ws", big), None)
    assert enc(65, c, _grads(5)) == -4 and "frozen_encoder_param_backward: shape outside" in err()
    assert enc(8, _table(PCR_CONV, bn_at=0, relu_last=True), _grads(5)) == -4 and "no BatchNorm" in err()
    assert enc(8, c, _grads(5, bn_at=4)) == -1 and "no BatchNorm" in err()
    assert enc(8, c, _grads(5, misalign_at=0)) == -1 and "16-byte aligned" in err()
    assert enc(8, c, None) == -1 and "conv_grads is null" in err()
    assert enc(8, c, _grads(5), ws=lib.snb200_frozen_encoder_param_backward_workspace_bytes(8, 64, 5, c, 1) - 1) == -2
    assert enc(8, c, _grads(5), ws=lib.snb200_frozen_encoder_backward_workspace_bytes(8, 64, 5, c, 1)) == -2


def test_wrapper_and_factory():
    with pytest.raises(ValueError, match="one of them"):
        reg.RegistrationStep().create_model(frozen_task=True, cuda_task=True)
    with pytest.raises(ValueError, match="train_pcrnet"):
        reg.RegistrationStep(train_pcrnet=True).create_model(frozen_task=True)
    for train in (False, True):
        act = reg.RegistrationStep(sampler="none", train_pcrnet=train)
        torch.manual_seed(0)
        w = act.create_model(cuda_task=True)
        torch.manual_seed(0)
        plain = act.create_model()
        assert type(w) is reg.CudaPCRNet and isinstance(w, reg.FrozenPCRNet) and type(w.net) is reg.PCRNet and w.sampler is None
        assert w.training == train and w.net.training == train
        # the optimiser's parameter list and the state dict are the plain module's
        got = [p for p in w.parameters() if p.requires_grad]
        ref = [p for p in plain.parameters() if p.requires_grad]
        assert len(got) == len(ref) == (22 if train else 0) and all(a.shape == b.shape and torch.equal(a, b) for a, b in zip(got, ref))
        assert list(w.net.state_dict()) == list(plain.state_dict()) and all(k.startswith("net.") for k in w.state_dict())
        w.train(not train)
        assert w.training == (not train) and w.net.training == (not train)
    joint = reg.RegistrationStep(train_pcrnet=True, train_samplenet=True).create_model(cuda_task=True)
    assert joint.sampler.name == "samplenet" and joint.sampler.training
    assert sum(p.requires_grad for p in joint.parameters()) == 22 + sum(1 for p in joint.sampler.parameters() if p.requires_grad)
    x = torch.zeros(2, 16, 3)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        joint(x, x)


def _cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    return exe if os.path.exists(exe) else None


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump is not available")
def test_kernel_stack_frames(lib):
    from samplenet_b200 import _lib

    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = {}
    for i, line in enumerate(lines):
        m = re.search(r"Function (_ZN3snb\d+(frozen_mlp_backward_kernel|last_grad_kernel|hidden_grad_partial_kernel|chain_bwd_kernel)\S*):", line)
        if m:
            res = {k: int(v) for k, v in re.findall(r"(\w+(?:\[\d+\])?):(\d+)", lines[i + 1])}
            found[m.group(1)] = (m.group(2), res)
    kinds = sorted(k for k, _ in found.values())
    assert kinds.count("frozen_mlp_backward_kernel") == 4 and {"last_grad_kernel", "hidden_grad_partial_kernel", "chain_bwd_kernel"} <= set(kinds), kinds
    for name, (kind, res) in found.items():
        assert res["STACK"] <= (40 if kind == "chain_bwd_kernel" else 0), (name, res)


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _specs(widths, seed, relu_last=False, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(len(widths) - 1):
        w = (torch.randn(widths[i + 1], widths[i], generator=g) * scale / widths[i] ** 0.5).cuda()
        b = (0.1 * torch.randn(widths[i + 1], generator=g)).cuda()
        out.append({"weight": w, "bias": b, "bn": None, "relu": bool(i < len(widths) - 2 or relu_last)})
    return out


def _norm_err(got, ref, scale):
    """max over elements of |got - ref| / sum of |terms| (elements whose terms are all 0 must be exactly 0)."""
    got, ref, scale = got.double(), ref.double(), scale.double()
    zero = scale == 0
    assert bool((got[zero] == 0).all())
    return float(((got - ref).abs()[~zero] / scale[~zero]).max()) if bool((~zero).any()) else 0.0


def _mlp_ref(specs, x, asave, g):
    """float64 dW, db per layer and their |terms| sums, on the kernel's masks and saved activations."""
    acts = [x] + list(asave)
    r, ra, out = g.double(), g.double().abs(), []      # ra: the gradient's own sum of |terms|, carried down the chain
    for l in range(len(specs) - 1, -1, -1):
        if specs[l]["relu"]:
            m = (asave[l] > 0).double()
            r, ra = r * m, ra * m
        a = acts[l].double()
        out.append((r.t() @ a, r.sum(0), ra.t() @ a.abs(), ra.sum(0)))
        r, ra = r @ specs[l]["weight"].double(), ra @ specs[l]["weight"].double().abs()
    return out[::-1]


WANTS = {"all": (True, True), "weight": (True, False), "bias": (False, True), "none": (False, False)}


@pytest.mark.gpu
@pytest.mark.parametrize("widths,b", [(PCR_W, 1), (PCR_W, 7), (PCR_W, 32), (PCR_W, 64), (ODD_W, 5), (ODD_W, 64)])
def test_mlp_param_grads_against_float64(sb, record_property, widths, b):
    ops = sb.ops
    specs = _specs(widths, 100 + b)
    x = torch.randn(b, widths[0], generator=torch.Generator().manual_seed(b)).cuda()
    out, asave = ops.frozen_mlp_forward(x, specs)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(7)).cuda()
    gin_ref = ops.frozen_mlp_backward(specs, asave, g)
    ref = _mlp_ref(specs, x, asave, g)
    worst = 0.0
    for kind, (ww, wb) in WANTS.items():
        for need_x in (True, False):
            want = [(ww, wb)] * len(specs)
            gx, grads = ops.frozen_mlp_param_backward(x, specs, asave, g, want, need_x=need_x)
            gx2, grads2 = ops.frozen_mlp_param_backward(x, specs, asave, g, want, need_x=need_x)
            assert (gx is None) == (not need_x) and (gx is None or (torch.equal(gx, gin_ref) and torch.equal(gx, gx2)))
            for (dw, db), (dw2, db2), (rw, rb, sw, sbias) in zip(grads, grads2, ref):
                assert (dw is not None) == ww and (db is not None) == wb
                if ww:
                    assert torch.equal(dw, dw2)
                    worst = max(worst, _norm_err(dw, rw, sw))
                if wb:
                    assert torch.equal(db, db2)
                    worst = max(worst, _norm_err(db, rb, sbias))
    record_property("mlp_param_err", worst)
    assert worst < MLP_PARAM_BAR, worst


def _enc_case(b, n, seed, dead_channel=None, dup=None, widths=PCR_CONV):
    specs = _specs(widths, seed, relu_last=True)
    if dead_channel is not None:
        specs[-1]["bias"][dead_channel] = -1e3       # pooled to exactly 0 under the ReLU
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.rand(b, n, 3, generator=g) - 0.5
    if dup is not None:
        x[:, dup[1]] = x[:, dup[0]]
    return specs, x.cuda()


def _enc_ref(specs, x, zsave, pooled, route, gp):
    """float64 dW, db per layer and their |terms| sums on the kernel's routes, masks and saved activations."""
    P, B, C = pooled.shape
    N = x.shape[1]
    L = len(specs)
    acts = [x.reshape(B * N, 3).double()] + [torch.relu(z.double()) for z in zsave]
    coef = gp.double() * (pooled > 0).double()
    rows = (torch.arange(B, device=x.device)[None, :, None] * N + route.long()).reshape(-1)
    cols = torch.arange(C, device=x.device).repeat(P * B)
    dz = torch.zeros(B * N, C, dtype=torch.float64, device=x.device)
    dza = torch.zeros_like(dz)
    dz.index_put_((rows, cols), coef.reshape(-1), accumulate=True)
    dza.index_put_((rows, cols), coef.abs().reshape(-1), accumulate=True)
    out = []
    for l in range(L - 1, -1, -1):
        if l < L - 1:
            m = (zsave[l] > 0).double()
            dz, dza = dz * m, dza * m
        a = acts[l]
        out.append((dz.t() @ a, dz.sum(0), dza.t() @ a.abs(), dza.sum(0)))
        dz, dza = dz @ specs[l]["weight"].double(), dza @ specs[l]["weight"].double().abs()
    return out[::-1]


ENC_SHAPES = [pytest.param(64, 1024, [1024], id="64x1024"), pytest.param(64, 64, [64], id="64x64"), pytest.param(2, 1000, [100, 517, 1000], id="2x1000-3prefixes"),
              pytest.param(5, 333, [333], id="5x333"), pytest.param(1, 129, [129], id="1x129")]


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,sizes", ENC_SHAPES)
def test_encoder_param_grads_against_float64(sb, record_property, b, n, sizes, widths=PCR_CONV):
    ops = sb.ops
    specs, x = _enc_case(b, n, 3 * n + b, dead_channel=5, dup=(3, 7), widths=widths)
    pooled, route, zs = ops.frozen_encoder_forward(x, specs, sizes)
    assert bool((pooled[:, :, 5] == 0).all())
    assert not bool((route == 7).any())                           # duplicated points: the lowest index takes the maximum
    gp = torch.randn(pooled.shape, generator=torch.Generator().manual_seed(n)).cuda()
    gx_ref = ops.frozen_encoder_backward(x, specs, sizes, pooled, route, zs, gp)
    assert float(gx_ref[:, 7].abs().max()) == 0.0
    ref = _enc_ref(specs, x, zs, pooled, route, gp)
    worst = 0.0
    for kind in ("all", "weight", "bias"):
        want = [WANTS[kind]] * len(specs)
        for need_x in ((True, False) if kind == "all" else (True,)):
            gx, grads = ops.frozen_encoder_param_backward(x, specs, sizes, pooled, route, zs, gp, want, need_x=need_x)
            gx2, grads2 = ops.frozen_encoder_param_backward(x, specs, sizes, pooled, route, zs, gp, want, need_x=need_x)
            assert (gx is None) == (not need_x) and (gx is None or (torch.equal(gx, gx_ref) and torch.equal(gx, gx2)))
            for l, ((dw, db), (dw2, db2), (rw, rb, sw, sbias)) in enumerate(zip(grads, grads2, ref)):
                if dw is not None:
                    assert torch.equal(dw, dw2)
                    worst = max(worst, _norm_err(dw, rw, sw))
                    if l == len(specs) - 1:
                        assert float(dw[5].abs().max()) == 0.0
                if db is not None:
                    assert torch.equal(db, db2)
                    worst = max(worst, _norm_err(db, rb, sbias))
                    if l == len(specs) - 1:
                        assert float(db[5]) == 0.0
    record_property("enc_param_err", worst)
    assert worst < ENC_PARAM_BAR, worst


def _pcrnet64_at_routes(net, x0, x1, routes):
    """fc6's output of PCRNet in float64 with each max-pool taken at the given points (the kernel's routes)."""
    def feat(x, r):
        y = x
        for c in (net.feat.conv1, net.feat.conv2, net.feat.conv3, net.feat.conv4, net.feat.conv5):
            y = torch.relu(y @ c.weight[:, :, 0].t() + c.bias)
        return torch.gather(y, 1, r.long()[:, None, :])[:, 0, :], y
    f0, y0 = feat(x0, routes[0])
    f1, y1 = feat(x1, routes[1])
    h = torch.cat([f0, f1], dim=1)
    for i, l in enumerate((net.fc1, net.fc2, net.fc3, net.fc4, net.fc5, net.fc6)):
        h = h @ l.weight.t() + l.bias
        h = torch.relu(h) if i < 5 else h
    return h, (y0, y1)


def _pre_acts64(net, x):
    """Every conv pre-activation (B, N, C) and the last layer's activation, in float64."""
    y, pre = x, []
    for c in (net.feat.conv1, net.feat.conv2, net.feat.conv3, net.feat.conv4, net.feat.conv5):
        z = y @ c.weight[:, :, 0].t() + c.bias
        pre.append(z)
        y = torch.relu(z)
    return pre, y


def _conditioned(net64, x0, x1):
    """No pre-activation of a routed point (conv layers) or of the head within 1e-7 of 0 (at 1e-6 none of 100 seeds of
    PCRNet's default initialisation qualifies at B = 48).  (Pooled maxima within 1e-5 relative of their
    runner-up are left in: the reference takes the max-pool at the kernel's routes, and the routes are compared with float64's argmax
    wherever the runner-up is further away.)"""
    feats = []
    for x in (x0, x1):
        pre, y = _pre_acts64(net64, x.double())
        top2 = y.topk(2, dim=1)[0]
        routed = torch.zeros(x.shape[:2], dtype=torch.bool, device=x.device)
        routed.scatter_(1, y.argmax(dim=1), True)
        if any(bool((z.abs()[routed] <= 1e-7).any()) for z in pre):
            return False
        feats.append(top2[:, 0])
    h = torch.cat(feats, dim=1)
    for l in (net64.fc1, net64.fc2, net64.fc3, net64.fc4, net64.fc5):
        h = h @ l.weight.t() + l.bias
        if bool((h.abs() <= 1e-7).any()):
            return False
        h = torch.relu(h)
    return True


@pytest.mark.gpu
def test_cuda_pcrnet_and_pose_loss_against_float64(sb, record_property):
    """B = 48 (two 32-pair chunks), 16 points: all 22 parameter gradients and both cloud gradients of the fused pose loss, on a conditioned
    instance (no pre-activation of a routed point or of the head within 1e-7 of 0), the reference's max-pools taken at the kernel's routes."""
    B, M = 48, 16
    for seed in range(100):
        torch.manual_seed(seed)
        net = reg.PCRNet(input_shape="bnc").cuda()
        g = torch.Generator().manual_seed(seed)
        x0, x1 = (torch.rand(B, M, 3, generator=g) - 0.5).cuda(), (torch.rand(B, M, 3, generator=g) - 0.5).cuda()
        net64 = reg.PCRNet(input_shape="bnc").cuda().double()
        net64.load_state_dict(net.state_dict())
        ok = _conditioned(net64, x0, x1)
        if ok:
            break
    assert ok, "no conditioned instance among the seeds"
    gt = torch.cat([torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=1), 0.1 * torch.randn(B, 3, generator=g)], dim=1).cuda()
    w = reg.CudaPCRNet(net)
    a0, a1 = x0.clone().requires_grad_(True), x1.clone().requires_grad_(True)
    y = w.raw(a0, a1)
    terms, _ = sb.ops.PoseLossFunction.apply(y, a0, a1, gt)
    wts = torch.tensor([1.0, 0.0, 1.0, 0.0, 0.0], device="cuda")     # chamfer + norm_err: pcrnet_loss of LOSS_TYPE 0
    (terms * wts).sum().backward()
    routes = []
    for x in (x0, x1):     # the kernel's routes of this instance: float64's argmax wherever the runner-up is not within 1e-5 relative
        _, r, _ = sb.ops.frozen_encoder_forward(x.contiguous(), w._specs()[0], [M], keep_activations=False)
        routes.append(r[0])
        _, y64 = _pre_acts64(net64, x.double())
        top2 = y64.topk(2, dim=1)[0]
        clear = (top2[:, 0] - top2[:, 1]) > 1e-5 * top2[:, 0]
        assert torch.equal(r[0].long()[clear], y64.argmax(dim=1)[clear])      # (channels pooled to 0 tie at 0 and pass no gradient)
    d0, d1 = x0.double().requires_grad_(True), x1.double().requires_grad_(True)
    h, _ = _pcrnet64_at_routes(net64, d0, d1, routes)
    import test_frozen_pcrnet as tf
    _, i01, i10, _ = sb.ops.pose_loss_forward(y.detach(), x0, x1, gt)      # the Chamfer terms on the kernel's arg-mins
    t64, _, _, _ = tf.pose64(h, d0, d1, gt.double(), i01, i10)
    (t64 * wts.double()).sum().backward()
    errs = {}
    for (n, p), (_, p64) in zip(net.named_parameters(), net64.named_parameters()):
        errs[n] = float((p.grad.double() - p64.grad).abs().max() / p64.grad.abs().max())
    errs["x0"] = float((a0.grad.double() - d0.grad).abs().max() / d0.grad.abs().max())
    errs["x1"] = float((a1.grad.double() - d1.grad).abs().max() / d1.grad.abs().max())
    assert len(errs) == 24
    worst = max(errs.values())
    record_property("net_grad_err", worst)
    assert worst < NET_BAR, errs


def _step_data(b, n, seed=100):
    g = torch.Generator().manual_seed(seed)
    p0 = (torch.rand(b, n, 3, generator=g) - 0.5).cuda()
    vec = torch.cat([torch.nn.functional.normalize(torch.randn(b, 4, generator=g), dim=1), torch.zeros(b, 3)], dim=1).cuda()
    return p0, reg.QuaternionTransform(vec).rotate(p0), {"vec": vec, "inversion": torch.tensor([False])}


@pytest.fixture()
def _tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


def _grad_errs(ref, got):
    """Per parameter the largest difference relative to its own largest gradient, or to the largest of all where its own is below 1e-3 of
    that: gradients that vanish in exact arithmetic (a bias ahead of a BatchNorm) hold rounding noise in both variants."""
    assert ref.keys() == got.keys()
    top = max(float(g.abs().max()) for g in ref.values())
    return {n: float((got[n] - ref[n]).abs().max()) / max(float(ref[n].abs().max()), 1e-3 * top) for n in ref}


@pytest.mark.gpu
def test_train_step_against_the_plain_module(sb, record_property, _tf32_off):
    """RegistrationStep(sampler="none", train_pcrnet=True) at B = 32, N = 1024: the first step's loss and gradients, five Adam steps' losses,
    and the trained state dict in PCRNet and FrozenPCRNet."""
    data = _step_data(32, 1024)
    runs = {}
    for cuda in (False, True):
        act = reg.RegistrationStep(sampler="none", train_pcrnet=True)
        torch.manual_seed(0)
        model = act.create_model(cuda_task=cuda).cuda()
        if cuda:      # the kernel's routes are torch's argmax on these clouds
            for x in data[:2]:
                pooled, r, _ = sb.ops.frozen_encoder_forward(x.contiguous(), model._specs()[0], [1024], keep_activations=False)
                with torch.no_grad():
                    f = model.net.feat
                    y = x.permute(0, 2, 1)
                    for c in (f.conv1, f.conv2, f.conv3, f.conv4, f.conv5):
                        y = torch.relu(c(y))
                live = pooled[0] > 0           # (a channel pooled to 0 passes no gradient, whichever point it names)
                assert torch.equal(r[0].long()[live], y.argmax(dim=2)[live])
        opt = torch.optim.Adam(filter(lambda p: p.requires_grad, model.parameters()), lr=1e-3)
        losses, first = [], None
        for i in range(5):
            loss, rot, _ = act.train_step(model, data, opt, "cuda")
            losses.append(float(loss))
            if i == 0:
                net = model.net if cuda else model
                first = {n: p.grad.double().clone() for n, p in net.named_parameters()}
        runs[cuda] = (losses, first, model)
    (l0, g0, plain), (l1, g1, w) = runs[False], runs[True]
    assert len(g0) == 22
    errs = _grad_errs(g0, g1)
    e_loss = abs(l1[0] - l0[0]) / abs(l0[0])
    e_adam = max(abs(a - b) / abs(a) for a, b in zip(l0, l1))
    record_property("step_loss_err", e_loss); record_property("step_grad_err", max(errs.values())); record_property("adam_loss_err", e_adam)
    assert e_loss < STEP_BAR and max(errs.values()) < STEP_BAR, (e_loss, errs)
    assert e_adam < ADAM_BAR, (l0, l1)
    sd = w.net.state_dict()
    p = reg.PCRNet(input_shape="bnc").cuda()
    p.load_state_dict(sd)
    f = reg.FrozenPCRNet(reg.PCRNet(input_shape="bnc").cuda().requires_grad_(False).eval())
    f.net.load_state_dict(sd)
    assert all(torch.equal(a, b) for a, b in zip(p.state_dict().values(), sd.values()))


@pytest.mark.gpu
def test_joint_step_against_the_plain_module(sb, record_property, _tf32_off):
    """SampleNet 1024 -> 64 and PCRNet trained together (--train-pcrnet --train-samplenet): every gradient of the first step.  The sampled
    clouds are not conditioned: with 64 points a pooled maximum within fp32 rounding of its runner-up routes differently in torch's fp32
    convolutions and the encoder's 3xTF32 layers, which moves PCRNet's conv biases by up to 0.6 % of their largest gradient."""
    data = _step_data(32, 1024, seed=7)
    res = {}
    for cuda in (False, True):
        act = reg.RegistrationStep(num_out_points=64, train_pcrnet=True, train_samplenet=True)
        torch.manual_seed(0)
        model = act.create_model(cuda_task=cuda).cuda()
        opt = torch.optim.Adam(filter(lambda p: p.requires_grad, model.parameters()), lr=0.0)
        loss, _, _ = act.train_step(model, data, opt, "cuda")
        net = model.net if cuda else model
        res[cuda] = (float(loss), {n: p.grad.double().clone() for n, p in net.named_parameters() if p.grad is not None})
    (l0, g0), (l1, g1) = res[False], res[True]
    assert sum(n.startswith("sampler.") for n in g0) > 10 and sum(not n.startswith("sampler.") for n in g0) == 22
    errs = _grad_errs(g0, g1)
    top = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    record_property("joint_loss_err", abs(l1 - l0) / abs(l0)); record_property("joint_grad_err", top[0][1])
    assert abs(l1 - l0) / abs(l0) < STEP_BAR and top[0][1] < JOINT_BAR, (l0, l1, top)


# ------------------------------------------------------------------------------------------------------------------ write sets
@pytest.mark.gpu
@pytest.mark.parametrize("widths,b", [(PCR_W, 32), (ODD_W, 5)])
def test_mlp_param_backward_writes_only_its_buffers(sb, widths, b):
    from test_write_sets import Arena, _addr, run_checked
    arena = Arena(256 << 20)
    lib, ops = sb._lib.lib(), sb.ops
    g = torch.Generator().manual_seed(b)
    specs = []
    for i in range(len(widths) - 1):
        specs.append({"weight": arena.carve("w%d" % i, (widths[i + 1], widths[i]), fill=torch.randn(widths[i + 1], widths[i], generator=g) / widths[i] ** 0.5),
                      "bias": arena.carve("b%d" % i, (widths[i + 1],), fill=0.1 * torch.randn(widths[i + 1], generator=g)), "bn": None,
                      "relu": i < len(widths) - 2})
    table, _ = ops.make_layers(specs)
    nl = len(specs)
    x = arena.carve("x", (b, widths[0]), fill=torch.randn(b, widths[0], generator=g))
    out = arena.carve("out", (b, widths[-1]))
    asave = [arena.carve("asave%d" % l, (b, widths[l + 1])) for l in range(nl - 1)]
    ap = (ctypes.c_void_p * max(nl - 1, 1))(*[a.data_ptr() for a in asave])
    sb._lib.check(lib.snb200_frozen_mlp_forward(b, x.data_ptr(), nl, table, out.data_ptr(), ap, None, 0, None), "forward")
    go = arena.carve("grad_out", (b, widths[-1]), fill=torch.randn(b, widths[-1], generator=g))
    rep = []
    from samplenet_b200._lib import LayerGrad
    for case, (ww, wb, gin_on) in {"all": (1, 1, 1), "weights-no-grad-in": (1, 0, 0), "biases": (0, 1, 1)}.items():
        gin = arena.carve("grad_in.%s" % case, (b, widths[0])) if gin_on else None
        gw = [arena.carve("dW%d.%s" % (l, case), (widths[l + 1], widths[l])) if ww else None for l in range(nl)]
        gb = [arena.carve("db%d.%s" % (l, case), (widths[l + 1],)) if wb else None for l in range(nl)]
        arr = (LayerGrad * nl)()
        for l in range(nl):
            arr[l].weight, arr[l].bias = (gw[l].data_ptr() if ww else None), (gb[l].data_ptr() if wb else None)
        wsb = int(lib.snb200_frozen_mlp_param_backward_workspace_bytes(b, nl, table))
        ws = arena.carve("workspace.%s" % case, (wsb,), dtype=torch.uint8)
        rc = []
        full = [t for t in gw + gb + [gin] if t is not None]
        rep += run_checked(arena, "frozen_mlp_param_backward(%s)" % case, lambda: rc.append(lib.snb200_frozen_mlp_param_backward(
            b, nl, table, x.data_ptr(), ap, go.data_ptr(), None if gin is None else gin.data_ptr(), arr, _addr(ws), wsb, None)), [ws], full=full)
        assert rc[0] == 0, lib.snb200_last_error()
    assert not rep, "\n".join(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,sizes", [(5, 333, [333]), (2, 1000, [100, 517, 1000])])
def test_encoder_param_backward_writes_only_its_buffers(sb, b, n, sizes, widths=PCR_CONV):
    from test_write_sets import Arena, _addr, run_checked
    arena = Arena(512 << 20)
    lib, ops = sb._lib.lib(), sb.ops
    g = torch.Generator().manual_seed(n)
    specs = []
    for i in range(len(widths) - 1):
        ci, co = widths[i], widths[i + 1]
        specs.append({"weight": arena.carve("w%d" % i, (co, ci), fill=torch.randn(co, ci, generator=g) / ci ** 0.5),
                      "bias": arena.carve("b%d" % i, (co,), fill=0.1 * torch.randn(co, generator=g)), "bn": None, "relu": True})
    conv, _ = ops.make_layers(specs)
    nconv, npf, C = len(specs), len(sizes), widths[-1]
    csz = (ctypes.c_int * npf)(*sizes)
    x = arena.carve("x", (b, n, 3), fill=torch.rand(b, n, 3, generator=g) - 0.5)
    pooled, route = arena.carve("pooled", (npf, b, C)), arena.carve("route", (npf, b, C), dtype=torch.int32)
    zs = [arena.carve("zsave%d" % l, (b * n, widths[l + 1])) for l in range(nconv - 1)]
    zp = (ctypes.c_void_p * (nconv - 1))(*[z.data_ptr() for z in zs])
    fwsb = int(lib.snb200_frozen_encoder_workspace_bytes(b, n, nconv, conv, npf, 1))
    fws = arena.carve("forward_workspace", (fwsb,), dtype=torch.uint8)
    sb._lib.check(lib.snb200_frozen_encoder_forward(b, n, x.data_ptr(), nconv, conv, npf, csz, pooled.data_ptr(), route.data_ptr(), zp, _addr(fws), fwsb,
                                                    None), "forward")
    gp = arena.carve("grad_pooled", (npf, b, C), fill=torch.randn(npf, b, C, generator=g))
    rep = []
    from samplenet_b200._lib import LayerGrad
    for case, (ww, wb, gx_on) in {"all": (1, 1, 1), "all-no-grad-x": (1, 1, 0), "biases": (0, 1, 1)}.items():
        gx = arena.carve("grad_x.%s" % case, (b, n, 3)) if gx_on else None
        gw = [arena.carve("dW%d.%s" % (l, case), (widths[l + 1], widths[l])) if ww else None for l in range(nconv)]
        gb = [arena.carve("db%d.%s" % (l, case), (widths[l + 1],)) if wb else None for l in range(nconv)]
        arr = (LayerGrad * nconv)()
        for l in range(nconv):
            arr[l].weight, arr[l].bias = (gw[l].data_ptr() if ww else None), (gb[l].data_ptr() if wb else None)
        wsb = int(lib.snb200_frozen_encoder_param_backward_workspace_bytes(b, n, nconv, conv, npf))
        ws = arena.carve("workspace.%s" % case, (wsb,), dtype=torch.uint8)
        rc = []
        full = [t for t in gw + gb + [gx] if t is not None]
        rep += run_checked(arena, "frozen_encoder_param_backward(%s)" % case, lambda: rc.append(lib.snb200_frozen_encoder_param_backward(
            b, n, x.data_ptr(), nconv, conv, npf, csz, pooled.data_ptr(), route.data_ptr(), zp, gp.data_ptr(), None if gx is None else gx.data_ptr(), arr,
            _addr(ws), wsb, None)), [ws], full=full)
        assert rc[0] == 0, lib.snb200_last_error()
    assert not rep, "\n".join(rep)
