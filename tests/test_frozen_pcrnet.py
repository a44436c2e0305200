"""The frozen PCRNet and the registration task loss on CUDA (csrc/frozen_mlp.cu, csrc/pose_loss.cu, ops.FrozenMLPFunction /
PoseLossFunction, registration.FrozenPCRNet, RegistrationStep.create_model(frozen_task=True)).

CPU: a float64 restatement of PCRNet.forward and of compute_pcrnet_loss's five terms, pinned against float64 autograd of the torch code in
samplenet_b200.registration (with a brute-force Chamfer in place of the CUDA op); the C ABI's envelope, workspace sizes and rejections; the
wrapper's refusals.  GPU (H100): the MLP forward layer by layer and its backward against float64, the pose loss (terms, twist, arg-mins,
gradients) against float64, repeat runs bit-identical, the wrapper against the wrapped module, the reference fixtures through the frozen
path, and whole training steps against the plain module.  Measured values are attached to the test reports (record_property)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from samplenet_b200 import registration as reg  # noqa: E402

# Bars (GPU), about 10x the largest value measured on an H100 80GB HBM3 (in brackets)
MLP_FWD_BAR = 2.5e-6   # [2.4e-7] a layer's output against float64 on the kernel's own input: / (sum_k |in_k W_ok| + |bias_o|)
MLP_BWD_BAR = 2.5e-6   # [2.6e-7] grad_in against float64 with the kernel's masks: / max |reference|
POSE_TERM_BAR = 1e-5   # [1.2e-6] each of the five terms, relative (+ 1e-7 absolute)
POSE_TWIST_BAR = 1e-6  # [1.0e-7] twist, absolute
POSE_GRAD_BAR = 1e-5   # [9.8e-7] grad_y / grad_p0 / grad_p1 against float64 on the kernel's arg-mins: / max |reference|
STEP_BAR = 2e-5        # [2.0e-6] a whole step, frozen against plain (TF32 off): loss and rot_err relative, each gradient as described in the test

PCR_W = [2048, 1024, 1024, 512, 512, 256, 7]
ODD_W = [264, 40, 7]


# ------------------------------------------------------------------------------------------------------------------ references
def mlp64(ws, bs, x, relus):
    """Every layer's output in float64 from float64 weights."""
    acts = []
    for w, b, r in zip(ws, bs, relus):
        x = x @ w.t() + b
        x = torch.relu(x) if r else x
        acts.append(x)
    return acts


def pcrnet64(net, x0, x1):
    """fc6's output (B, 7) of PCRNet(input_shape='bnc') in float64."""
    def feat(x):
        y = x.double()
        for c in (net.feat.conv1, net.feat.conv2, net.feat.conv3, net.feat.conv4, net.feat.conv5):
            y = torch.relu(y @ c.weight[:, :, 0].double().t() + c.bias.double())
        return y.max(dim=1)[0]
    fcs = [net.fc1, net.fc2, net.fc3, net.fc4, net.fc5, net.fc6]
    return mlp64([l.weight.double() for l in fcs], [l.bias.double() for l in fcs], torch.cat([feat(x0), feat(x1)], dim=1), [1, 1, 1, 1, 1, 0])[-1]


def _rot64(q):
    """(B, 3, 3) of (w, x, y, z) quaternions, normalised with eps 1e-12 first."""
    q = q / q.norm(dim=1, keepdim=True).clamp_min(1e-12)
    w, x, y, z = q.unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], dim=1).view(-1, 3, 3)


def pose64(y, p0, p1, gt, idx01=None, idx10=None):
    """(terms (5,), twist, idx01, idx10) in the dtype of the inputs; with arg-mins given the Chamfer terms are evaluated on them."""
    q = y[:, :4] / y[:, :4].norm(dim=1, keepdim=True).clamp_min(1e-12)
    w, u = q[:, None, :1], q[:, None, 1:].expand(-1, p0.shape[1], -1)
    uv = torch.cross(u, p0, dim=2)
    e = p0 + 2 * (w * uv + torch.cross(u, uv, dim=2))
    d = ((p1[:, :, None, :] - e[:, None, :, :]) ** 2).sum(-1)            # [b, i (p1), j (e)]
    if idx01 is None:
        idx01, idx10 = d.argmin(dim=2), d.argmin(dim=1)
    c01 = torch.gather(d, 2, idx01.long()[:, :, None])[:, :, 0]
    c10 = torch.gather(d, 1, idx10.long()[:, None, :])[:, 0, :]
    chamfer = c01.mean() + c10.mean()
    qnorm = (((y[:, :4] ** 2).sum(1) - 1) ** 2).mean()
    m = _rot64(q) @ _rot64(gt[:, :4]).transpose(1, 2) - torch.eye(3, dtype=y.dtype, device=y.device)
    norm_err = (m ** 2).sum(dim=(1, 2)).mean()
    rot_err = (2 * torch.acos(2 * (q * gt[:, :4]).sum(1) ** 2 - 1)).mean()
    trans_err = (y[:, 4:] - gt[:, 4:]).abs().mean()
    return torch.stack([chamfer, qnorm, norm_err, rot_err, trans_err]), torch.cat([q, y[:, 4:]], dim=1), idx01, idx10


def torch_terms64(y, p0, p1, gt):
    """The five terms through the torch code of samplenet_b200.registration (brute-force Chamfer instead of the CUDA op)."""
    twist = torch.cat([F.normalize(y[:, :4], dim=1), y[:, 4:]], dim=1)
    est, gtt = reg.QuaternionTransform(twist), reg.QuaternionTransform(gt)
    e = est.rotate(p0)
    d = ((p1[:, :, None, :] - e[:, None, :, :]) ** 2).sum(-1)
    chamfer = d.min(dim=2)[0].mean() + d.min(dim=1)[0].mean()
    qnorm = torch.mean((torch.sum(y[:, :4] ** 2, dim=1) - 1) ** 2)
    rot_err, norm_err, trans_err = est.compute_errors(gtt)
    return torch.stack([chamfer, qnorm, norm_err, rot_err, trans_err])


def pose_case(b, m, seed, kind="random", device="cpu"):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(b, 7, generator=g)
    if kind == "conditioned":      # near-unit quaternions a moderate rotation away from the ground truth, small translations
        y[:, :4] = F.normalize(y[:, :4], dim=1) * (1 + 0.05 * torch.randn(b, 1, generator=g))
        y[:, 4:] *= 0.1
    gt = torch.cat([F.normalize(torch.randn(b, 4, generator=g), dim=1), 0.1 * torch.randn(b, 3, generator=g)], dim=1)
    p0 = torch.rand(b, m, 3, generator=g) - 0.5
    p1 = reg.QuaternionTransform(gt).rotate(p0) + 0.01 * torch.randn(b, m, 3, generator=g)
    return [t.to(device) for t in (y, p0, p1, gt)]


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("kind", ["random", "conditioned"])
def test_restatement_matches_float64_autograd_of_the_torch_code(kind):
    torch.manual_seed(3)
    net = reg.PCRNet(input_shape="bnc").double()
    y, p0, p1, gt = [t.double() for t in pose_case(3, 17, 5, kind)]
    # PCRNet.forward
    tw, pre = net(p0, p1)
    y_net = pcrnet64(net, p0, p1)
    assert torch.allclose(y_net[:, :4], pre, rtol=1e-12, atol=1e-14)
    assert torch.allclose(torch.cat([F.normalize(y_net[:, :4], dim=1), y_net[:, 4:]], dim=1), tw, rtol=1e-12, atol=1e-14)
    # the five terms and their gradients (rot_err is compared in value only: nothing differentiates it)
    a = [t.clone().requires_grad_(True) for t in (y, p0, p1)]
    c = [t.clone().requires_grad_(True) for t in (y, p0, p1)]
    ta, twist, _, _ = pose64(a[0], a[1], a[2], gt)
    tc = torch_terms64(c[0], c[1], c[2], gt)
    assert torch.allclose(ta, tc, rtol=1e-11, atol=1e-13), (ta, tc)
    wts = torch.tensor([1.0, 0.7, 1.3, 0.0, 0.4], dtype=torch.float64)
    (ta * wts).sum().backward(); (tc * wts).sum().backward()
    for u, v in zip(a, c):
        assert torch.allclose(u.grad, v.grad, rtol=1e-9, atol=1e-12)


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


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


def test_mlp_envelope_and_workspaces(lib):
    t = _table(PCR_W)
    for b in (1, 32, 64):
        assert lib.snb200_frozen_mlp_supported(b, 6, t) == 1
    assert lib.snb200_frozen_mlp_supported(5, 2, _table(ODD_W)) == 1
    assert lib.snb200_frozen_mlp_supported(64, 2, _table([4096, 4096, 1])) == 1
    for b in (0, 65, -1):
        assert lib.snb200_frozen_mlp_supported(b, 6, t) == 0
    assert lib.snb200_frozen_mlp_supported(32, 6, _table(PCR_W, bn_at=2)) == 0                  # BatchNorm
    assert lib.snb200_frozen_mlp_supported(32, 2, _table([260, 40, 7])) == 0                    # c_in not a multiple of 8
    assert lib.snb200_frozen_mlp_supported(32, 2, _table([264, 44, 7])) == 0                    # ... of a later layer
    assert lib.snb200_frozen_mlp_supported(32, 2, _table([4104, 40, 7])) == 0 and lib.snb200_frozen_mlp_supported(32, 2, _table([264, 4104, 7])) == 0
    assert lib.snb200_frozen_mlp_supported(32, 9, _table([64] * 10)) == 0                       # too many layers
    assert lib.snb200_frozen_mlp_supported(32, 0, t) == 0
    assert lib.snb200_frozen_mlp_supported(32, 6, _table(PCR_W, relu_last=True)) == 0           # no saved output to mask a last ReLU with
    bad_chain = _table(PCR_W); bad_chain[3].c_in = 1024
    assert lib.snb200_frozen_mlp_supported(32, 6, bad_chain) == 0
    # forward without asave: the hidden layers; with asave: nothing.  Backward: the layers' input-gradient blocks.  Monotone in b.
    hidden = sum(PCR_W[1:-1])
    assert lib.snb200_frozen_mlp_workspace_bytes(32, 6, t, 0) == 32 * hidden * 4
    assert lib.snb200_frozen_mlp_workspace_bytes(32, 6, t, 1) == 0
    prev_f = prev_b = 0
    for b in range(1, 65):
        f, bw = lib.snb200_frozen_mlp_workspace_bytes(b, 6, t, 0), lib.snb200_frozen_mlp_backward_workspace_bytes(b, 6, t)
        assert f > 0 and bw > 0 and f >= prev_f and bw >= prev_b
        prev_f, prev_b = f, bw
    assert lib.snb200_frozen_mlp_workspace_bytes(65, 6, t, 0) == 0 and lib.snb200_frozen_mlp_backward_workspace_bytes(0, 6, t) == 0
    assert lib.snb200_pose_loss_workspace_bytes(32, 64) > 0 and lib.snb200_pose_loss_workspace_bytes(256, 1024) >= lib.snb200_pose_loss_workspace_bytes(32, 64)
    assert lib.snb200_pose_loss_workspace_bytes(257, 64) == 0 and lib.snb200_pose_loss_workspace_bytes(32, 1025) == 0


def test_rejections_before_any_launch(lib):
    """Calls outside the envelope return SNB200_EUNSUPPORTED (-4), null / short workspaces SNB200_EWORKSPACE (-2), null pointers SNB200_EINVAL
    (-1), each with its message; nothing launches (the pointers here are never dereferenced, and this runs without a device)."""
    t = _table(PCR_W)
    z = (ctypes.c_void_p * 8)(*[_ptr() for _ in range(8)])
    big = 1 << 40

    def err():
        return lib.snb200_last_error().decode()

    assert lib.snb200_frozen_mlp_forward(65, _ptr(), 6, t, _ptr(), z, _ptr(), big, None) == -4 and err().startswith("frozen_mlp_forward: outside the frozen MLP's envelope")
    assert lib.snb200_frozen_mlp_backward(32, 6, _table(PCR_W, bn_at=0), z, _ptr(), _ptr(), _ptr(), big, None) == -4 and "frozen_mlp_backward" in err()
    assert lib.snb200_frozen_mlp_forward(32, None, 6, t, _ptr(), z, _ptr(), big, None) == -1 and "null pointer" in err()
    assert lib.snb200_frozen_mlp_forward(32, _ptr() + 4, 6, t, _ptr(), z, _ptr(), big, None) == -1 and "16-byte aligned" in err()
    need = lib.snb200_frozen_mlp_workspace_bytes(32, 6, t, 0)
    assert lib.snb200_frozen_mlp_forward(32, _ptr(), 6, t, _ptr(), None, None, big, None) == -2 and "workspace is null" in err()
    assert lib.snb200_frozen_mlp_forward(32, _ptr(), 6, t, _ptr(), None, _ptr(), need - 1, None) == -2 and "workspace" in err()
    needb = lib.snb200_frozen_mlp_backward_workspace_bytes(32, 6, t)
    assert lib.snb200_frozen_mlp_backward(32, 6, t, z, _ptr(), _ptr(), None, big, None) == -2
    assert lib.snb200_frozen_mlp_backward(32, 6, t, z, _ptr(), _ptr(), _ptr(), needb - 1, None) == -2
    assert lib.snb200_frozen_mlp_backward(32, 6, t, None, _ptr(), _ptr(), _ptr(), big, None) == -1
    p = [_ptr() for _ in range(12)]
    assert lib.snb200_pose_loss_forward(257, 64, *p[:8], _ptr(), big, _ptr(), None) == -4 and "pose_loss_forward: outside the pose loss's envelope" in err()
    assert lib.snb200_pose_loss_forward(32, 1025, *p[:8], _ptr(), big, _ptr(), None) == -4
    assert lib.snb200_pose_loss_forward(32, 0, *p[:8], _ptr(), big, _ptr(), None) == -4
    assert lib.snb200_pose_loss_forward(32, 64, *p[:8], None, big, _ptr(), None) == -2
    assert lib.snb200_pose_loss_forward(32, 64, *p[:8], _ptr(), lib.snb200_pose_loss_workspace_bytes(32, 64) - 1, _ptr(), None) == -2
    assert lib.snb200_pose_loss_forward(32, 64, *p[:8], _ptr(), big, None, None) == -1 and "null pointer" in err()
    assert lib.snb200_pose_loss_backward(0, 64, *p[:10], None) == -4
    assert lib.snb200_pose_loss_backward(32, 64, *p[:9], None, None) == -1


def test_wrapper_refusals_and_create_model():
    net = reg.PCRNet(input_shape="bnc").eval()
    x = torch.zeros(2, 16, 3)
    with pytest.raises(ValueError, match="gives no parameter gradients"):
        reg.FrozenPCRNet(net)(x, x)
    net.requires_grad_(False); net.eval()
    w = reg.FrozenPCRNet(net)
    assert not w.training
    with pytest.raises(ValueError, match="eval mode only"):
        w.train()
    with pytest.raises(ValueError, match="eval mode only"):
        w.train(True)
    w.eval()
    with pytest.raises(RuntimeError, match="CUDA-only"):
        w(x, x)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA-only"):
        reg.FrozenPCRNet(reg.PCRNet(input_shape="bnc").eval())(x, x)
    net.train()
    with pytest.raises(ValueError, match="training mode"):
        w(x, x)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        from samplenet_b200 import ops
        ops.pose_loss_forward(torch.zeros(2, 7), x, x, torch.zeros(2, 7))
    # the step's factory
    with pytest.raises(ValueError, match="train_pcrnet"):
        reg.RegistrationStep(train_pcrnet=True).create_model(frozen_task=True)
    plain = reg.RegistrationStep().create_model()
    assert type(plain) is reg.PCRNet
    act = reg.RegistrationStep()
    fr = act.create_model(frozen_task=True)
    assert type(fr) is reg.FrozenPCRNet and type(fr.net) is reg.PCRNet and fr.sampler is fr.net.sampler and fr.sampler.name == "samplenet"
    assert fr.sampler.training and not fr.net.feat.training and not fr.training
    # the wrapper owns no parameters: what a data-parallel wrapper of the sampler sees is unchanged
    assert [n for n, _ in fr.named_parameters()] == ["net." + n for n, _ in fr.net.named_parameters()]
    assert all(not p.requires_grad for n, p in fr.named_parameters() if not n.startswith("net.sampler."))
    fr.sampler = None
    assert fr.net.sampler is None and fr.sampler is None


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _mlp_case(widths, b, seed, conditioned=False):
    g = torch.Generator().manual_seed(seed)
    ws = [torch.randn(widths[i + 1], widths[i], generator=g) / widths[i] ** 0.5 for i in range(len(widths) - 1)]
    bs = [0.1 * torch.randn(widths[i + 1], generator=g) for i in range(len(widths) - 1)]
    x = torch.randn(b, widths[0], generator=g)
    relus = [1] * (len(widths) - 2) + [0]
    if conditioned:     # push every hidden pre-activation away from the ReLU kink (float64 forward, bias nudged per unit)
        h = x.double()
        for l in range(len(ws) - 1):
            z = h @ ws[l].double().t() + bs[l].double()
            near = z.abs().min(dim=0)[0] < 1e-3
            bs[l] = torch.where(near, bs[l] + 0.01, bs[l])
            h = torch.relu(h @ ws[l].double().t() + bs[l].double())
    specs = [{"weight": w.cuda(), "bias": b_.cuda(), "bn": None, "relu": bool(r)} for w, b_, r in zip(ws, bs, relus)]
    return ws, bs, relus, x.cuda(), specs


@pytest.mark.gpu
@pytest.mark.parametrize("widths", [PCR_W, ODD_W], ids=["pcrnet", "odd"])
@pytest.mark.parametrize("b", [1, 2, 31, 32, 64])
def test_mlp_forward_and_backward_against_float64(sb, record_property, widths, b):
    ws, bs, relus, x, specs = _mlp_case(widths, b, 10 + b)
    out, asave = sb.ops.frozen_mlp_forward(x, specs)
    out2, asave2 = sb.ops.frozen_mlp_forward(x, specs)
    out3, none = sb.ops.frozen_mlp_forward(x, specs, keep_activations=False)
    assert none is None and torch.equal(out, out2) and torch.equal(out, out3) and all(torch.equal(p, q) for p, q in zip(asave, asave2))
    acts = asave + [out]
    worst = 0.0
    for l in range(len(ws)):        # layer l in float64 on the kernel's own input
        src = (x if l == 0 else acts[l - 1]).double().cpu()
        w, bb = ws[l].double(), bs[l].double()
        z = src @ w.t() + bb
        ref = torch.relu(z) if relus[l] else z
        scale = src.abs() @ w.abs().t() + bb.abs()
        worst = max(worst, float(((acts[l].double().cpu() - ref).abs() / scale).max()))
    record_property("mlp_fwd_err", worst)
    assert worst < MLP_FWD_BAR, worst
    # backward with the kernel's masks
    g = torch.randn(b, widths[-1], generator=torch.Generator().manual_seed(b)).cuda()
    gx = sb.ops.frozen_mlp_backward(specs, asave, g)
    assert torch.equal(gx, sb.ops.frozen_mlp_backward(specs, asave, g))
    r = g.double().cpu()
    for l in range(len(ws) - 1, -1, -1):
        if relus[l]:
            r = r * (asave[l].cpu() > 0)
        r = r @ ws[l].double()
    err = float((gx.double().cpu() - r).abs().max() / r.abs().max())
    record_property("mlp_bwd_err", err)
    assert err < MLP_BWD_BAR, err


@pytest.mark.gpu
@pytest.mark.parametrize("widths,b", [(PCR_W, 32), (ODD_W, 5)], ids=["pcrnet", "odd"])
def test_mlp_end_to_end_on_conditioned_instances(sb, record_property, widths, b):
    ws, bs, relus, x, specs = _mlp_case(widths, b, 77, conditioned=True)
    xg = x.clone().requires_grad_(True)
    out = sb.ops.FrozenMLPFunction.apply(xg, specs)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(1)).cuda()
    (out * g).sum().backward()
    x64 = x.double().cpu().requires_grad_(True)
    ref = mlp64([w.double() for w in ws], [b_.double() for b_ in bs], x64, relus)[-1]
    (ref * g.double().cpu()).sum().backward()
    e_out = float((out.double().cpu() - ref).abs().max() / ref.abs().max())
    e_grad = float((xg.grad.double().cpu() - x64.grad).abs().max() / x64.grad.abs().max())
    record_property("mlp_e2e_out_err", e_out); record_property("mlp_e2e_grad_err", e_grad)
    assert e_out < 10 * MLP_FWD_BAR and e_grad < 10 * MLP_BWD_BAR, (e_out, e_grad)
    with pytest.raises(ValueError, match="envelope"):
        sb.ops.frozen_mlp_forward(torch.zeros(65, widths[0], device="cuda"), specs)
    with pytest.raises(ValueError, match="channels"):
        sb.ops.frozen_mlp_forward(torch.zeros(4, widths[0] + 8, device="cuda"), specs)


def _check_pose(sb, record_property, y, p0, p1, gt, tag):
    twist, i01, i10, terms = sb.ops.pose_loss_forward(y, p0, p1, gt)
    again = sb.ops.pose_loss_forward(y, p0, p1, gt)
    assert all(torch.equal(a, b) for a, b in zip((twist, i01, i10, terms), again))
    d = [t.double() for t in (y, p0, p1)]
    for t in d:
        t.requires_grad_(True)
    ref, tw64, _, _ = pose64(d[0], d[1], d[2], gt.double(), i01, i10)       # on the kernel's arg-mins
    e_terms = float(((terms.double() - ref).abs() / (ref.abs() + 1e-7 / POSE_TERM_BAR)).max())
    e_twist = float((twist.double() - tw64).abs().max())
    wts = torch.tensor([1.0, 0.7, 1.3, 0.0, 0.4], device="cuda")
    (ref * wts.double()).sum().backward()
    grads = sb.ops.pose_loss_backward(y, p0, p1, gt, i01, i10, wts)
    assert all(torch.equal(a, b) for a, b in zip(grads, sb.ops.pose_loss_backward(y, p0, p1, gt, i01, i10, wts)))
    e_grad = max(float((g.double() - t.grad).abs().max() / t.grad.abs().max()) for g, t in zip(grads, d))
    record_property("pose_term_err_" + tag, e_terms); record_property("pose_twist_err_" + tag, e_twist); record_property("pose_grad_err_" + tag, e_grad)
    assert e_terms < POSE_TERM_BAR and e_twist < POSE_TWIST_BAR and e_grad < POSE_GRAD_BAR, (e_terms, e_twist, e_grad)
    return twist, i01, i10, terms


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, 32, 256])
@pytest.mark.parametrize("m", [1, 7, 64, 1024])
def test_pose_loss_against_float64(sb, record_property, b, m):
    y, p0, p1, gt = pose_case(b, m, 1000 * b + m, "conditioned", "cuda")
    twist, i01, i10, _ = _check_pose(sb, record_property, y, p0, p1, gt, "b%d_m%d" % (b, m))
    # the arg-mins are ChamferDistance's (tie-free inputs) on the rotated cloud the kernel forms
    e = reg.QuaternionTransform(twist).rotate(p0)
    _, j01, _, j10 = sb.ops.nn_distance_forward(p1, e)
    same = float((i01 == j01).float().mean()), float((i10 == j10).float().mean())
    d = ((p1[:, :, None, :] - e[:, None, :, :]) ** 2).sum(-1) if m <= 64 else None
    if d is not None:       # and the true minima (float64 of the same e): equal wherever the runner-up is not within rounding
        dd = ((p1.double()[:, :, None, :] - e.double()[:, None, :, :]) ** 2).sum(-1)
        got = torch.gather(dd, 2, i01.long()[:, :, None])[:, :, 0]
        assert bool((got <= dd.min(dim=2)[0] * (1 + 1e-5) + 1e-12).all())
    assert same[0] > 0.9999 and same[1] > 0.9999, same


@pytest.mark.gpu
def test_pose_loss_ties_and_normalize_eps_path(sb, record_property):
    y, p0, p1, gt = pose_case(4, 64, 9, "conditioned", "cuda")
    # duplicated points: an identity estimate (e = p0 exactly) with p0's points 5 and 40 equal, and p1 = p0 -> ties go to the lowest index
    y[:, :4] = torch.tensor([1.0, 0.0, 0.0, 0.0], device="cuda")
    p0[:, 40] = p0[:, 5]
    p1 = p0.clone()
    _, i01, i10, terms = sb.ops.pose_loss_forward(y, p0, p1, gt)
    want = torch.arange(64, device="cuda", dtype=torch.int32).repeat(4, 1); want[:, 40] = 5
    assert torch.equal(i01, want) and torch.equal(i10, want) and float(terms[0]) == 0.0
    # an un-normalised row and a near-zero-norm row (|y[:4]| < 1e-12: normalize divides by eps, the twist's quaternion is not of unit length)
    y, p0, p1, gt = pose_case(4, 64, 10, "conditioned", "cuda")
    y[1, :4] *= 37.0
    y[2, :4] = torch.tensor([3e-14, -1e-14, 2e-14, 1e-14], device="cuda")
    twist, _, _, _ = _check_pose(sb, record_property, y, p0, p1, gt, "eps")
    assert abs(float(twist[1, :4].norm()) - 1) < 1e-6 and float(twist[2, :4].norm()) < 0.1
    assert torch.allclose(twist[2, :4], y[2, :4] / 1e-12, rtol=1e-6)


def _frozen_pair(seed, bottleneck=1024):
    torch.manual_seed(seed)
    net = reg.PCRNet(bottleneck, input_shape="bnc").requires_grad_(False).eval().cuda()
    return net, reg.FrozenPCRNet(net)


@pytest.fixture()
def _tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["bnc", "bcn"])
def test_wrapper_against_the_module(sb, record_property, _tf32_off, shape, bottleneck=1024):
    net, fr = _frozen_pair(5, bottleneck)
    net.input_shape = net.feat.input_shape = shape
    g = torch.Generator().manual_seed(2)
    x0, x1 = (torch.rand(32, 64, 3, generator=g) - 0.5).cuda(), (torch.rand(32, 64, 3, generator=g) - 0.5).cuda()
    a0, a1 = (x0, x1) if shape == "bnc" else (x0.permute(0, 2, 1).contiguous(), x1.permute(0, 2, 1).contiguous())
    a0.requires_grad_(True); a1.requires_grad_(True)
    tw, pre = fr(a0, a1)
    y64 = pcrnet64(net, x0, x1)
    e = float((pre.double() - y64[:, :4]).abs().max() / y64.abs().max())
    record_property("wrapper_out_err", e)
    assert e < 1e-5, e
    tw_m, pre_m = net(a0.detach(), a1.detach())
    assert torch.allclose(tw, tw_m, rtol=1e-3, atol=1e-5) and torch.allclose(pre, pre_m, rtol=1e-3, atol=1e-5)
    (tw.sum() + pre.sum()).backward()
    assert a0.grad is not None and a0.grad.shape == a0.shape and bool(torch.isfinite(a0.grad).all()) and float(a1.grad.abs().max()) > 0
    # outside the encoder's envelope (4097 points): the wrapped module runs
    if shape == "bnc":
        big = torch.rand(1, 4097, 3, device="cuda") - 0.5
        with torch.no_grad():
            assert torch.equal(fr(big, big)[0], net(big, big)[0])


@pytest.mark.gpu
def test_wrapper_chunks_batches_beyond_32_pairs(sb):
    net, fr = _frozen_pair(6)
    g = torch.Generator().manual_seed(3)
    x0, x1 = (torch.rand(48, 64, 3, generator=g) - 0.5).cuda().requires_grad_(True), (torch.rand(48, 64, 3, generator=g) - 0.5).cuda()
    tw, pre = fr(x0, x1)
    pre.square().sum().backward()
    h0 = [x0.detach()[:32].clone().requires_grad_(True), x0.detach()[32:].clone().requires_grad_(True)]
    halves = [fr(h0[0], x1[:32]), fr(h0[1], x1[32:])]
    assert torch.equal(tw, torch.cat([halves[0][0], halves[1][0]])) and torch.equal(pre, torch.cat([halves[0][1], halves[1][1]]))
    (halves[0][1].square().sum() + halves[1][1].square().sum()).backward()
    assert torch.equal(x0.grad, torch.cat([h0[0].grad, h0[1].grad]))


def _t(a):
    return torch.from_numpy(np.asarray(a)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("ncl", [1, 2])
def test_reference_fixture_through_the_frozen_path(sb, golden_dir, ncl):
    """tests/golden/registration_step_c{1,2}.npz (the reference's own Action on CPU) at the tolerances of the plain-module fixture test."""
    z = np.load(os.path.join(golden_dir, "registration_step_c%d.npz" % ncl))
    z2 = np.load(os.path.join(golden_dir, "samplenet_reg_b2.npz"))
    act = reg.RegistrationStep(num_sampled_clouds=ncl, alpha=float(z["alpha"]), lmbda=float(z["lmbda"]))
    torch.manual_seed(11)
    model = act.create_model(frozen_task=True)
    model.sampler.load_state_dict({k[3:]: torch.from_numpy(z2[k]) for k in z2.files if k.startswith("sd_")})
    model = model.cuda()
    model.sampler.train()
    igt = {"vec": _t(z["igt_vec"]), "inversion": torch.tensor([False])}
    data = (_t(z["p0"]), _t(z["p1"]), igt)
    pl, pinfo = act.compute_pcrnet_loss(model, (_t(z["p0_out"]), _t(z["p1_out"]), igt), "cuda")
    np.testing.assert_allclose(pinfo["est_transform"].vec.cpu().numpy(), z["twist"], rtol=2e-4, atol=2e-5)
    for key in ("chamfer_loss", "qnorm_loss", "norm_err", "trans_err", "rot_err"):
        np.testing.assert_allclose(float(pinfo[key]), float(z[key]), rtol=5e-4, atol=1e-6, err_msg=key)
    np.testing.assert_allclose(float(pl), float(z["pcrnet_loss"]), rtol=5e-4)
    if ncl == 2:
        model.zero_grad()
        sl2, sampled2, _ = act.compute_samplenet_loss(model, data, "cuda")
        pl2, _ = act.compute_pcrnet_loss(model, sampled2, "cuda")
        (pl2 + sl2).backward()
        worst = 0.0
        for name, p in model.sampler.named_parameters():
            ref = float(z["gnorm_" + name])
            if ref > 1e-3:
                worst = max(worst, abs(float(p.grad.double().norm()) - ref) / ref)
        assert worst < 5e-2, worst


def _step_data(b, n, dev="cuda"):
    g = torch.Generator().manual_seed(100)
    p0 = torch.rand(b, n, 3, generator=g) - 0.5
    vec = torch.cat([F.normalize(torch.randn(b, 4, generator=g), dim=1), torch.zeros(b, 3)], dim=1).to(dev)
    p0 = p0.to(dev)
    return p0, reg.QuaternionTransform(vec).rotate(p0), {"vec": vec, "inversion": torch.tensor([False])}


@pytest.mark.gpu
def test_whole_train_step_against_the_plain_module(sb, record_property, _tf32_off):
    data = _step_data(32, 1024)
    res = []
    for frozen in (False, True):
        act = reg.RegistrationStep(num_sampled_clouds=2)
        torch.manual_seed(0)
        model = act.create_model(frozen_task=frozen).cuda()
        model.sampler.train()
        ddp = act.wrap_data_parallel(model)      # world size 1: no process group; the flat bucket covers the sampler's parameters only
        assert ddp.bucket_bytes() == 4 * sum(p.numel() for p in model.sampler.parameters() if p.requires_grad)
        opt = torch.optim.SGD([p for p in model.sampler.parameters() if p.requires_grad], lr=0.0)
        loss, rot, _ = act.train_step(model, data, opt, "cuda")
        res.append((float(loss), float(rot), {n: p.grad.double().clone() for n, p in model.sampler.named_parameters() if p.grad is not None}))
    (l0, r0, g0), (l1, r1, g1) = res
    e_loss, e_rot = abs(l1 - l0) / abs(l0), abs(r1 - r0) / abs(r0)
    assert g0.keys() == g1.keys() and len(g0) > 10
    # Parameters whose gradient vanishes in exact arithmetic (a bias ahead of a BatchNorm; bn5's bias, a per-channel constant that bn_fc1's
    # batch statistics remove) hold rounding noise in both variants, 1e-9 .. 2e-8 here.  So a parameter is compared relative to its own largest
    # gradient when that is at least 1e-3 of the largest of all, and relative to the largest of all otherwise.
    top = max(float(g.abs().max()) for g in g0.values())
    per = sorted(((float((g1[n] - g0[n]).abs().max()) / (float(g0[n].abs().max()) if float(g0[n].abs().max()) >= 1e-3 * top else top), n,
                   float(g0[n].abs().max())) for n in g0), reverse=True)
    e_grad = per[0][0]
    record_property("step_loss_err", e_loss); record_property("step_rot_err", e_rot); record_property("step_grad_err", e_grad)
    assert e_loss < STEP_BAR and e_rot < STEP_BAR and e_grad < STEP_BAR, (e_loss, e_rot, top, per)


@pytest.mark.gpu
@pytest.mark.parametrize("sampler,n", [("fps", 1024), ("none", 1024), ("none", 1500)])
def test_steps_with_other_samplers_run(sb, sampler, n):
    """FPS samples both clouds to 64 points; "none" trains on the full clouds (1024 points: the pose loss's limit; 1500: beyond it, the
    torch ops run on the wrapper's output)."""
    data = _step_data(8, n)
    act = reg.RegistrationStep(num_sampled_clouds=2, sampler=sampler)
    torch.manual_seed(0)
    model = act.create_model(frozen_task=True).cuda()
    plain = reg.RegistrationStep(num_sampled_clouds=2, sampler=sampler)
    torch.manual_seed(0)
    ref = plain.create_model().cuda()
    # (nothing trains in these configurations -- PCRNet is frozen and the samplers have no parameters -- so the step is its forward half)
    sampled = act.non_learned_sampling(model, data, "cuda") if sampler == "fps" else data
    sampled_ref = plain.non_learned_sampling(ref, data, "cuda") if sampler == "fps" else data
    pl, info = act.compute_pcrnet_loss(model, sampled, "cuda")
    pl_ref, info_ref = plain.compute_pcrnet_loss(ref, sampled_ref, "cuda")
    assert abs(float(pl) - float(pl_ref)) <= 2e-3 * abs(float(pl_ref)) and abs(float(info["rot_err"]) - float(info_ref["rot_err"])) <= 2e-3 * float(info_ref["rot_err"])
