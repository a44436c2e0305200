"""PointNet with transform nets (tasknets.PointNetClsTransforms) and its frozen CUDA path (tasknets.FrozenPointNetClsTransforms): the
extended frozen encoder (activation input, tapped hidden layer; csrc/frozen_encoder.cu), the frozen MLP with eval-mode BatchNorm
(csrc/frozen_mlp.cu) and the point transform (csrc/point_transform.cu).

CPU: the module's float64 forward, loss and input gradient against a float64 restatement written from the TF graph (pointnet_cls.py +
transform_nets.py + tf_util.py) on TF-layout variables; from_tf_variables on a synthetic checkpoint against the same restatement; the new C
entries' envelopes, workspace sizes and rejections; the wrapper's refusals.  GPU (H100): each new kernel against float64 and bit-identical
on repeat, the whole wrapper against the float64 module, the classification steps with the wrapper against the plain module, and the
out-of-envelope fallback."""
import copy
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from samplenet_b200 import tasknets  # noqa: E402

# Bars (GPU).  The kernel bars are test_frozen_tasknets.py's / test_frozen_pcrnet.py's.
Z_BAR = 2e-5          # a stored raw output or tapped activation against float64 on the kernel's previous layer: / the point's sum |terms|
POOL_BAR = 2e-5       # pooled on the kernel's route: / (|scale| sum |terms| + |shift|)
BWD_BAR = 5e-6        # grad_in against float64 on the kernel's routes and masks: / max |reference|
MLP_FWD_BAR = 2.5e-6  # a layer's output against float64 on the kernel's input: / (|scale| (sum_k |in_k W_ok| + |bias_o|) + |shift|)
MLP_BWD_BAR = 2.5e-6  # grad_in against float64 with the kernel's masks: / max |reference|
PT_BAR = 1e-6         # point transform outputs and gradients against float64: / the sum of |terms| of each entry
NET_BAR = 1e-5        # the wrapper's logits / transform / loss against the float64 module: / max |reference|
NET_GRAD_BAR = 1e-4   # its gradient of get_loss to the points on a conditioned instance: / max |reference|
STEP_BAR = 2e-3       # whole steps, the sampler's gradients (test_frozen_tasknets.py's rule and bar)
GUARD = 1e-6          # conditioned instances: no pooled extreme this close to its runner-up, no routed unit this close to its ReLU kink
STEP_GUARD = 1e-7     # ... for the large cases (about 10^7 checked units per instance: 1e-6 is rarely met)


# ------------------------------------------------------------------------------------------------------------------ the TF graph in float64
def _ema(name, which):
    return "%s/bn/%s/bn/moments/%s/ExponentialMovingAverage" % (name, name, "Squeeze" if which == "mean" else "Squeeze_1")


def tf_graph64(V, x, label=None, reg_weight=0.001):
    """pointnet_cls.py get_model (is_training=False) + get_loss, from TF-named float64 tensors V (conv kernels (1, kw, Cin, Cout), FC weights
    (Cin, Cout)), on x (B, N, 3).  Returns (logits, transform (B, 64, 64), GFV, loss or None)."""
    def bn(v, name):
        return (v - V[_ema(name, "mean")]) / torch.sqrt(V[_ema(name, "var")] + 1e-3) * V[name + "/bn/gamma"] + V[name + "/bn/beta"]

    def conv(v, name):     # v (B, N, Cin): a [1, kw] kernel over a (B, N, 3, 1) image is the same contraction as a [1, 1] one over (B, N, 1, 3)
        w = V[name + "/weights"]
        w = w[0, :, 0, :] if w.shape[2] == 1 else w[0, 0]
        return torch.relu(bn(v @ w + V[name + "/biases"], name))

    def fc(v, name, with_bn=True):
        z = v @ V[name + "/weights"] + V[name + "/biases"]
        return torch.relu(bn(z, name)) if with_bn else z

    def tnet(v, scope, last, K):
        y = conv(conv(conv(v, scope + "/tconv1"), scope + "/tconv2"), scope + "/tconv3").max(dim=1)[0]
        y = fc(fc(y, scope + "/tfc1"), scope + "/tfc2")
        bias = V[scope + "/" + last + "/biases"] + torch.eye(K, dtype=y.dtype).flatten()    # the identity added to the bias in the graph
        return (y @ V[scope + "/" + last + "/weights"] + bias).reshape(-1, K, K)           # row-major reshape

    t1 = tnet(x, "transform_net1", "transform_XYZ", 3)
    h = conv(conv(torch.matmul(x, t1), "conv1"), "conv2")                                   # tf.matmul(point_cloud, transform)
    t2 = tnet(h, "transform_net2", "transform_feat", 64)
    y = conv(conv(conv(torch.matmul(h, t2), "conv3"), "conv4"), "conv5")
    gfv = y.max(dim=1)[0]
    logits = fc(fc(fc(gfv, "fc1"), "fc2"), "fc3", with_bn=False)
    loss = None
    if label is not None:
        d = t2 @ t2.transpose(1, 2) - torch.eye(64, dtype=t2.dtype)
        loss = F.cross_entropy(logits, label) + reg_weight * (d * d).sum() / 2                # tf.nn.l2_loss: half the sum over the batch
    return logits, t2, gfv, loss


def module_to_tf(net):
    """The module's parameters as TF variables (float64), converted here independently of from_tf_variables."""
    V = {}
    for name, kind, lin, bn in net.tf_layers():
        w = lin.weight.detach().double()
        if kind == "conv":
            w = w[:, :, 0].t()
            w = w[None, :, None, :] if w.shape[0] == 3 else w[None, None]
        else:
            w = w.t()
        V[name + "/weights"], V[name + "/biases"] = w.contiguous(), lin.bias.detach().double()
        if bn is not None:
            V[name + "/bn/gamma"], V[name + "/bn/beta"] = bn.weight.detach().double(), bn.bias.detach().double()
            V[_ema(name, "mean")], V[_ema(name, "var")] = bn.running_mean.double(), bn.running_var.double()
    return V


def randomized_net(seed, num_classes=40):
    """PointNetClsTransforms with BatchNorm away from the identity (a quarter of every layer's scales < 0) and transform layers away from
    zero, so that T1 and T2 are neither the identity nor symmetric."""
    torch.manual_seed(seed)
    net = tasknets.PointNetClsTransforms(num_classes)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                c = m.num_features
                gam = 0.5 + torch.rand(c, generator=g)
                gam[torch.randperm(c, generator=g)[: c // 4]] *= -1
                m.weight.copy_(gam); m.bias.copy_(0.3 * torch.randn(c, generator=g))
                m.running_mean.copy_(0.1 * torch.randn(c, generator=g)); m.running_var.copy_(0.5 + torch.rand(c, generator=g))
        for t, s in ((net.transform_net1.transform, 0.05), (net.transform_net2.transform, 0.01)):
            t.weight.copy_(s * torch.randn(t.weight.shape, generator=g)); t.bias.copy_(s * torch.randn(t.bias.shape, generator=g))
    return net.eval()


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_module_against_the_tf_graph_in_float64():
    net = randomized_net(1).double()
    x = (0.5 * torch.randn(3, 40, 3, dtype=torch.float64)).requires_grad_(True)
    label = torch.tensor([3, 17, 39])
    logits, ep = net(x)
    loss = net.get_loss(logits, label, ep)
    x2 = x.detach().clone().requires_grad_(True)
    l64, t64, gfv64, loss64 = tf_graph64(module_to_tf(net), x2, label)
    assert torch.allclose(logits, l64, rtol=1e-12, atol=1e-12) and torch.allclose(ep["transform"], t64, rtol=1e-12, atol=1e-13)
    assert torch.allclose(ep["GFV"], gfv64, rtol=1e-12, atol=1e-12) and abs(float(loss.detach() - loss64.detach())) < 1e-12 * abs(float(loss64.detach()))
    # the restatement is sensitive to what it pins: T @ x instead of x @ T, a transposed reshape, a mean instead of the half-sum
    t1 = net.transform_net1(x.detach().permute(0, 2, 1))
    assert not torch.allclose(torch.matmul(x.detach(), t1), torch.matmul(x.detach(), t1.transpose(1, 2)), atol=1e-6)
    assert not torch.allclose(ep["transform"], ep["transform"].transpose(1, 2), atol=1e-6)
    d = t64 @ t64.transpose(1, 2) - torch.eye(64, dtype=torch.float64)
    assert abs(float(loss64 - F.cross_entropy(l64, label)) - 0.001 * float((d * d).sum()) / 2) < 1e-12
    assert abs(float((d * d).sum()) / 2 - float((d * d).mean())) > 1e-6
    # the gradient of the loss to the points
    g, = torch.autograd.grad(loss, x)
    g64, = torch.autograd.grad(loss64, x2)
    assert torch.allclose(g, g64, rtol=1e-10, atol=1e-13)
    # the transform layers' parameters are TF's: zero-initialised, the identity added in forward
    fresh = tasknets.PointNetClsTransforms()
    assert float(fresh.transform_net2.transform.weight.abs().max()) == 0 and float(fresh.transform_net2.transform.bias.abs().max()) == 0
    assert torch.equal(fresh.transform_net1.to_matrix(torch.zeros(2, 9)), torch.eye(3).expand(2, 3, 3))


def _synthetic_checkpoint(seed, num_classes=40):
    """A name -> numpy array dict with TF shapes for every variable of the classifier, EMA names included (float32, as saved)."""
    rng = np.random.default_rng(seed)
    V = {k: v.numpy().astype(np.float32) for k, v in module_to_tf(randomized_net(seed, num_classes)).items()}
    for k in V:
        V[k] = (V[k] * (1 + 0.1 * rng.standard_normal(V[k].shape))).astype(np.float32)
        if k.endswith("Squeeze_1/ExponentialMovingAverage"):
            V[k] = np.abs(V[k]) + 0.1
    return V


def test_from_tf_variables_against_the_tf_graph():
    V = _synthetic_checkpoint(5, num_classes=10)
    assert sum(k.endswith("ExponentialMovingAverage") for k in V) == 2 * 17 and "transform_net2/transform_feat/biases" in V
    assert V["transform_net1/tconv1/weights"].shape == (1, 3, 1, 64) and V["transform_net2/tconv1/weights"].shape == (1, 1, 64, 64)
    net = tasknets.PointNetClsTransforms.from_tf_variables(V).double().eval()
    assert net.fc3.out_features == 10
    x = 0.5 * torch.randn(2, 30, 3, dtype=torch.float64)
    label = torch.tensor([1, 7])
    logits, ep = net(x)
    l64, t64, _, loss64 = tf_graph64({k: torch.from_numpy(v.astype(np.float64)) for k, v in V.items()}, x, label)
    assert torch.allclose(logits, l64, rtol=1e-10, atol=1e-10) and torch.allclose(ep["transform"], t64, rtol=1e-10, atol=1e-12)
    assert abs(float(net.get_loss(logits, label, ep) - loss64)) < 1e-10 * abs(float(loss64))
    # a missing weight, a missing moving average, an unknown name, each raise
    for drop in ("conv3/weights", _ema("transform_net1/tfc2", "var"), "transform_net2/transform_feat/biases"):
        W = dict(V); del W[drop]
        with pytest.raises(KeyError):
            tasknets.PointNetClsTransforms.from_tf_variables(W)
    W = dict(V); W["conv6/weights"] = np.zeros((1, 1, 4, 4), np.float32)
    with pytest.raises(KeyError, match="does not have"):
        tasknets.PointNetClsTransforms.from_tf_variables(W)
    W = dict(V); W["fc3/bn/gamma"] = np.ones(10, np.float32)
    with pytest.raises(KeyError):
        tasknets.PointNetClsTransforms.from_tf_variables(W)
    # the state dict round-trips: the transform layers hold TF's values, not TF's values plus the identity
    assert np.array_equal(net.transform_net2.transform.bias.detach().float().numpy(), V["transform_net2/transform_feat/biases"])


_next_ptr = [0x90000]


def _ptr():
    _next_ptr[0] += 0x1000
    return _next_ptr[0]


def _table(widths, bn=True, running=True):
    from samplenet_b200._lib import Layer
    arr = (Layer * (len(widths) - 1))()
    for i in range(len(widths) - 1):
        L = arr[i]
        L.c_in, L.c_out, L.weight, L.bias = widths[i], widths[i + 1], _ptr(), _ptr()
        if bn:
            L.bn_weight, L.bn_bias = _ptr(), _ptr()
            if running:
                L.bn_running_mean, L.bn_running_var = _ptr(), _ptr()
        L.bn_eps, L.bn_momentum, L.relu = 1e-3, 0.1, 1
    return arr


def _fc_table(widths, bn=True, running=True):
    t = _table(widths, bn, running)
    t[len(widths) - 2].relu = 0
    t[len(widths) - 2].bn_weight = t[len(widths) - 2].bn_bias = None
    return t


FRONT, BACK, TNET = [3, 64, 64, 64, 128, 1024], [64, 64, 128, 1024], [3, 64, 128, 1024]


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


def test_envelopes_and_workspaces(lib):
    front, back = _table(FRONT), _table(BACK)
    for b, n in ((1, 1), (32, 32), (32, 1024), (64, 4096), (5, 333)):
        assert lib.snb200_frozen_encoder_ex_supported(b, n, 0, 5, front, 1, 1) == 1
        assert lib.snb200_frozen_encoder_ex_supported(b, n, 1, 3, back, 1, -1) == 1
        assert lib.snb200_frozen_encoder_ex_supported(b, n, 1, 3, back, 4, 1) == 1
    for b, n in ((0, 32), (65, 32), (32, 4097)):
        assert lib.snb200_frozen_encoder_ex_supported(b, n, 1, 3, back, 1, -1) == 0
    # the tap is a hidden layer; an activation input is a tensor-core layer (c_in a multiple of 8 up to 256); a cloud input has 3 channels
    assert lib.snb200_frozen_encoder_ex_supported(32, 1024, 0, 5, front, 1, 4) == 0 and lib.snb200_frozen_encoder_ex_supported(32, 1024, 0, 5, front, 1, -2) == 0
    assert lib.snb200_frozen_encoder_ex_supported(32, 1024, 0, 5, front, 1, 3) == 1 and lib.snb200_frozen_encoder_ex_supported(32, 1024, 0, 5, front, 1, 0) == 1
    assert lib.snb200_frozen_encoder_ex_supported(32, 1024, 1, 3, _table([60, 64, 128, 1024]), 1, -1) == 0
    assert lib.snb200_frozen_encoder_ex_supported(32, 1024, 1, 3, _table([264, 64, 128, 1024]), 1, -1) == 0
    assert lib.snb200_frozen_encoder_ex_supported(32, 1024, 1, 1, _table([64, 1024]), 1, -1) == 0
    assert lib.snb200_frozen_encoder_ex_supported(32, 1024, 0, 3, back, 1, -1) == 0 and lib.snb200_frozen_encoder_ex_supported(32, 1024, 1, 5, front, 1, -1) == 0
    # the original entries are the cloud-input, no-tap case, and the workspaces are theirs
    for b, n in ((1, 32), (32, 1024), (5, 333)):
        assert lib.snb200_frozen_encoder_ex_supported(b, n, 0, 3, _table(TNET), 1, -1) == lib.snb200_frozen_encoder_supported(b, n, 3, _table(TNET), 1) == 1
        for z in (0, 1):
            assert lib.snb200_frozen_encoder_ex_workspace_bytes(b, n, 0, 5, front, 1, 1, z) == lib.snb200_frozen_encoder_workspace_bytes(b, n, 5, front, 1, z)
        assert lib.snb200_frozen_encoder_ex_backward_workspace_bytes(b, n, 0, 5, front, 1, 1) == lib.snb200_frozen_encoder_backward_workspace_bytes(b, n, 5, front, 1)
    assert lib.snb200_frozen_encoder_ex_workspace_bytes(32, 1024, 1, 3, back, 1, -1, 1) == 32 * (8 + 1) * 1024 * 8
    assert lib.snb200_frozen_encoder_ex_workspace_bytes(32, 1024, 1, 3, back, 1, -1, 0) == 32 * 9 * 1024 * 8 + 2 * 32 * 1024 * 128 * 4
    assert lib.snb200_frozen_encoder_ex_backward_workspace_bytes(32, 1024, 1, 3, back, 1, -1) == 32 * 1024 * 32 * 4
    assert lib.snb200_frozen_encoder_ex_workspace_bytes(65, 1024, 1, 3, back, 1, -1, 1) == 0
    # the MLP with BatchNorm: the old entries refuse BatchNorm, the new ones take it; workspaces as the old ones without it
    for w in ([1024, 512, 256, 9], [1024, 512, 256, 4096], [1024, 512, 256, 40]):
        t = _fc_table(w)
        assert lib.snb200_frozen_mlp_supported(32, 3, t) == 0
        for b in (1, 32, 64):
            assert lib.snb200_frozen_mlp_bn_supported(b, 3, t) == 1
        assert lib.snb200_frozen_mlp_bn_supported(65, 3, t) == 0
        plain = _fc_table(w, bn=False)
        assert lib.snb200_frozen_mlp_bn_supported(32, 3, plain) == lib.snb200_frozen_mlp_supported(32, 3, plain) == 1
        for b in (1, 32, 64):
            assert lib.snb200_frozen_mlp_bn_workspace_bytes(b, 3, t, 0) == lib.snb200_frozen_mlp_workspace_bytes(b, 3, plain, 0) == b * (512 + 256) * 4
            assert lib.snb200_frozen_mlp_bn_workspace_bytes(b, 3, t, 1) == 0
            assert lib.snb200_frozen_mlp_bn_backward_workspace_bytes(b, 3, t) == lib.snb200_frozen_mlp_backward_workspace_bytes(b, 3, plain) > 0
    relu_last = _fc_table([1024, 512, 256, 9]); relu_last[2].relu = 1
    assert lib.snb200_frozen_mlp_bn_supported(32, 3, relu_last) == 0
    assert lib.snb200_frozen_mlp_bn_supported(32, 2, _fc_table([1024, 4104, 9])) == 0
    # the point transform: K <= 64; the backward's workspace holds a partial grad_T per 128-point chunk (none for one chunk)
    for b, n, k in ((1, 1, 1), (32, 1024, 3), (32, 1024, 64), (65535, 128, 64)):
        assert lib.snb200_point_transform_supported(b, n, k) == 1
    for b, n, k in ((0, 32, 3), (65536, 32, 3), (32, 0, 3), (32, 32, 65), (32, 32, 0), (1, (1 << 24) + 1, 3)):
        assert lib.snb200_point_transform_supported(b, n, k) == 0 and lib.snb200_point_transform_workspace_bytes(b, n, k) == 0
    assert lib.snb200_point_transform_workspace_bytes(32, 128, 64) == 0 and lib.snb200_point_transform_workspace_bytes(32, 129, 64) == 32 * 2 * 4096 * 4
    assert lib.snb200_point_transform_workspace_bytes(32, 1024, 64) == 32 * 8 * 4096 * 4 and lib.snb200_point_transform_workspace_bytes(32, 1024, 3) == 32 * 8 * 9 * 4


def test_rejections_before_any_launch(lib):
    """Outside the envelope SNB200_EUNSUPPORTED (-4), short workspaces SNB200_EWORKSPACE (-2), null or misaligned pointers and missing running
    statistics SNB200_EINVAL (-1), each with its message; nothing launches (the pointers are never dereferenced: this runs without a device)."""
    big = 1 << 40
    z = (ctypes.c_void_p * 8)(*[_ptr() for _ in range(8)])
    one = (ctypes.c_int * 1)(1024)
    front, back = _table(FRONT), _table(BACK)

    def err():
        return lib.snb200_last_error().decode()

    def fwd(b, n, act, inp, nconv, t, sizes, tap, tap_out, ws=_ptr, wsb=big, zs=z):
        cs = (ctypes.c_int * len(sizes))(*sizes)
        return lib.snb200_frozen_encoder_ex_forward(b, n, act, inp, nconv, t, len(sizes), cs, _ptr(), _ptr(), tap, tap_out, zs, ws() if ws else None, wsb, None)

    def bwd(b, n, act, nconv, t, tap, grad_tap, wsb=big, zs=z):
        return lib.snb200_frozen_encoder_ex_backward(b, n, act, _ptr(), nconv, t, 1, one, _ptr(), _ptr(), zs, tap, grad_tap, _ptr(), _ptr(), _ptr(), wsb, None)

    who = "frozen_encoder_ex_forward: "
    assert fwd(65, 1024, 0, _ptr(), 5, front, [1024], 1, _ptr()) == -4 and err().startswith(who + "shape outside the frozen encoder's envelope")
    assert fwd(32, 1024, 0, _ptr(), 5, front, [1024], 4, _ptr()) == -4 and err().startswith(who + "shape outside")
    assert fwd(32, 1024, 1, _ptr(), 5, front, [1024], -1, None) == -4
    assert fwd(32, 1024, 1, _ptr(), 3, _table(BACK, running=False), [1024], -1, None) == -1 and "eval mode needs running statistics" in err()
    assert fwd(32, 1024, 1, _ptr(), 3, back, [512, 256], -1, None) == -1 and "prefix sizes must be ascending" in err()
    assert fwd(32, 1024, 0, _ptr(), 5, front, [1024], 1, None) == -1 and err() == who + "null pointer"
    assert fwd(32, 1024, 1, _ptr() + 4, 3, back, [1024], -1, None) == -1 and "16-byte aligned" in err()
    assert fwd(32, 1024, 0, _ptr(), 5, front, [1024], 1, _ptr() + 8) == -1 and "tap_out must be 16-byte aligned" in err()
    assert fwd(32, 1024, 0, _ptr(), 5, front, [1024], 1, _ptr(), ws=None) == -2 and "workspace is null" in err()
    need = lib.snb200_frozen_encoder_ex_workspace_bytes(32, 1024, 0, 5, front, 1, 1, 1)
    assert fwd(32, 1024, 0, _ptr(), 5, front, [1024], 1, _ptr(), wsb=need - 1) == -2 and err().startswith(who + "workspace")
    who = "frozen_encoder_ex_backward: "
    assert bwd(32, 4097, 1, 3, back, -1, None) == -4 and err().startswith(who + "shape outside")
    assert bwd(32, 1024, 0, 5, front, 1, None) == -1 and err() == who + "null pointer"
    assert bwd(32, 1024, 0, 5, front, 1, _ptr(), zs=None) == -1
    needb = lib.snb200_frozen_encoder_ex_backward_workspace_bytes(32, 1024, 0, 5, front, 1, 1)
    assert bwd(32, 1024, 0, 5, front, 1, _ptr(), wsb=needb - 1) == -2 and err().startswith(who + "workspace")
    # the MLP with BatchNorm
    t = _fc_table([1024, 512, 256, 9])
    assert lib.snb200_frozen_mlp_bn_forward(65, _ptr(), 3, t, _ptr(), z, _ptr(), big, None) == -4 and err().startswith("frozen_mlp_bn_forward: outside the frozen MLP's envelope")
    assert lib.snb200_frozen_mlp_bn_forward(32, _ptr(), 3, _fc_table([1024, 512, 256, 9], running=False), _ptr(), z, _ptr(), big, None) == -1
    assert "eval mode needs running statistics" in err()
    assert lib.snb200_frozen_mlp_bn_forward(32, None, 3, t, _ptr(), z, _ptr(), big, None) == -1 and err() == "frozen_mlp_bn_forward: null pointer"
    assert lib.snb200_frozen_mlp_bn_forward(32, _ptr() + 4, 3, t, _ptr(), z, _ptr(), big, None) == -1 and "16-byte aligned" in err()
    need = lib.snb200_frozen_mlp_bn_workspace_bytes(32, 3, t, 0)
    assert lib.snb200_frozen_mlp_bn_forward(32, _ptr(), 3, t, _ptr(), None, _ptr(), need - 1, None) == -2
    assert lib.snb200_frozen_mlp_bn_backward(32, 3, t, None, _ptr(), _ptr(), _ptr(), big, None) == -1 and err() == "frozen_mlp_bn_backward: null pointer"
    assert lib.snb200_frozen_mlp_bn_backward(32, 3, t, z, _ptr(), _ptr(), _ptr(), lib.snb200_frozen_mlp_bn_backward_workspace_bytes(32, 3, t) - 1, None) == -2
    assert lib.snb200_frozen_mlp_backward(32, 3, t, z, _ptr(), _ptr(), _ptr(), big, None) == -4    # the original entry still refuses BatchNorm
    # the point transform
    p = [_ptr() for _ in range(5)]
    assert lib.snb200_point_transform_forward(32, 1024, 65, p[0], p[1], p[2], None) == -4 and err().startswith("point_transform_forward: outside the point transform's envelope")
    assert lib.snb200_point_transform_forward(32, 1024, 64, p[0], None, p[2], None) == -1 and err() == "point_transform_forward: null pointer"
    assert lib.snb200_point_transform_backward(0, 1024, 64, *p, _ptr(), big, None) == -4
    assert lib.snb200_point_transform_backward(32, 1024, 64, *p[:4], None, _ptr(), big, None) == -1 and err() == "point_transform_backward: null pointer"
    assert lib.snb200_point_transform_backward(32, 1024, 64, *p, None, big, None) == -2 and "workspace is null" in err()
    assert lib.snb200_point_transform_backward(32, 1024, 64, *p, _ptr(), lib.snb200_point_transform_workspace_bytes(32, 1024, 64) - 1, None) == -2


def test_wrapper_refusals():
    net = tasknets.PointNetClsTransforms()
    x = torch.zeros(2, 16, 3)
    with pytest.raises(ValueError, match="gives no parameter gradients"):
        tasknets.FrozenPointNetClsTransforms(net.eval())(x)
    net.requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    assert not w.training and not hasattr(w, "prefixes")
    with pytest.raises(ValueError, match="eval mode only"):
        w.train()
    with pytest.raises(ValueError, match="eval mode only"):
        w.train(True)
    w.eval()
    net.train()
    with pytest.raises(ValueError, match="training mode"):
        w(x)
    net.eval()
    with pytest.raises(RuntimeError, match="CUDA-only"):   # CPU tensors: no fallback
        w(x)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA-only"):
        tasknets.FrozenPointNetClsTransforms(tasknets.PointNetClsTransforms().eval())(x)
    # the wrapper owns no parameters of its own
    assert [n for n, _ in w.named_parameters()] == ["net." + n for n, _ in net.named_parameters()]


# ------------------------------------------------------------------------------------------------------------------ GPU: kernels
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _stack(widths, seed):
    """A conv stack with randomized eval-mode BatchNorm (a quarter of the scales < 0), as an object with convs / bns, float32 on the GPU."""
    torch.manual_seed(seed)
    net = types.SimpleNamespace(convs=[torch.nn.Conv1d(widths[i], widths[i + 1], 1) for i in range(len(widths) - 1)],
                                bns=[torch.nn.BatchNorm1d(widths[i + 1], eps=1e-3) for i in range(len(widths) - 1)])
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for conv, bn in zip(net.convs, net.bns):
            c = bn.num_features
            conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) * (1.0 / conv.weight.shape[1]) ** 0.5)
            conv.bias.copy_(0.1 * torch.randn(c, generator=g))
            gam = 0.5 + torch.rand(c, generator=g)
            gam[torch.randperm(c, generator=g)[: c // 4]] *= -1
            bn.weight.copy_(gam); bn.bias.copy_(0.3 * torch.randn(c, generator=g))
            bn.running_mean.copy_(0.1 * torch.randn(c, generator=g)); bn.running_var.copy_(0.5 + torch.rand(c, generator=g))
    for m in net.convs + net.bns:
        m.cuda().eval().requires_grad_(False)
    return net


def _layers64(net):
    out = []
    for conv, bn in zip(net.convs, net.bns):
        sc = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
        out.append((conv.weight.double()[:, :, 0], conv.bias.double(), sc, bn.bias.double() - bn.running_mean.double() * sc))
    return out


def _fp32_scale_shift(bn):
    """The kernels' fp32 scale gamma * (1 / sqrtf(var + eps)) and shift beta - mean * scale, the latter's sign as the fused expression's."""
    inv = 1.0 / torch.sqrt(bn.running_var.float() + bn.eps)
    sc = bn.weight.float() * inv
    return sc.double(), bn.bias.double() - bn.running_mean.double() * sc.double()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["cloud_tap", "activation"])
@pytest.mark.parametrize("b,n", [(5, 333), (32, 1024), (1, 32)])
def test_encoder_ex_against_float64(sb, mode, b, n):
    widths, act, tap = (FRONT, False, 1) if mode == "cloud_tap" else (BACK, True, -1)
    net = _stack(widths, 7 + b)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(b, n, widths[0], device="cuda", generator=g) * (0.5 if not act else 1.0)
    if act:
        x = torch.relu(x)      # an activation: non-negative, as h2 of the network is not, but the kernel takes any values
    specs = tasknets._conv_specs(net)
    pooled, route, h, zs = sb.ops.frozen_encoder_ex_forward(x, specs, [n], act, tap)
    again = sb.ops.frozen_encoder_ex_forward(x, specs, [n], act, tap)
    assert torch.equal(pooled, again[0]) and torch.equal(route, again[1]) and all(torch.equal(p, q) for p, q in zip(zs, again[3]))
    assert (h is None) == (tap < 0) and (h is None or torch.equal(h, again[2]))
    if not act:    # the cloud-input, no-tap call is the original entry bit for bit
        p0, r0, z0 = sb.ops.frozen_encoder_forward(x, specs, [n])
        assert torch.equal(p0, pooled) and torch.equal(r0, route) and all(torch.equal(p, q) for p, q in zip(z0, zs))
    # layer by layer against float64 on the kernel's previous layer; the tap is relu(bn(z_tap)) of the stored z
    L = _layers64(net)
    hh = x.double()
    for l, (w, bb, sc, sh) in enumerate(L[:-1]):
        z64 = hh @ w.t() + bb
        terms = hh.abs() @ w.abs().t() + bb.abs()
        assert float(((zs[l].view(b, n, -1).double() - z64).abs() / terms).max()) <= Z_BAR, l
        hh = torch.relu(zs[l].view(b, n, -1).double() * sc + sh)
        if l == tap:
            s32, h32 = _fp32_scale_shift(net.bns[l])
            want = torch.relu(zs[l].view(b, n, -1).double() * s32 + h32)
            assert float((h.double() - want).abs().max() / (want.abs().max())) <= 1e-6
    w, bb, sc, sh = L[-1]
    terms = (hh.abs() @ w.abs().t() + bb.abs())
    aL = torch.relu((hh @ w.t() + bb) * sc + sh)
    idx = route[0].long()[:, None, :]
    err = (pooled[0].double() - torch.gather(aL, 1, idx)[:, 0]).abs() / (torch.gather(terms, 1, idx)[:, 0] * sc.abs() + sh.abs())
    assert float(err.max()) <= POOL_BAR
    # backward on the kernel's routes and masks, with a dense tap gradient
    gp = torch.randn(pooled.shape, device="cuda", generator=g)
    gt = torch.randn(b, n, widths[tap + 1], device="cuda", generator=g) if tap >= 0 else None
    gx = sb.ops.frozen_encoder_ex_backward(x, specs, [n], pooled, route, zs, gp, act, tap, gt)
    assert torch.equal(gx, sb.ops.frozen_encoder_ex_backward(x, specs, [n], pooled, route, zs, gp, act, tap, gt)), "not bit-identical"
    s_last, _ = _fp32_scale_shift(net.bns[-1])
    coef = gp[0].double() * s_last * (pooled[0] > 0).double()
    dA = torch.zeros(b, n, w.shape[1], dtype=torch.float64, device="cuda")
    dA.scatter_add_(1, route[0].long()[:, :, None].expand(b, -1, w.shape[1]), coef[:, :, None] * w[None])
    for l in range(len(L) - 2, -1, -1):
        if l == tap:
            dA = dA + gt.double()
        s32, h32 = _fp32_scale_shift(net.bns[l])
        mask = (zs[l].view(b, n, -1).double() * s32 + h32) > 0
        dA = (dA * s32 * mask) @ L[l][0]
    err = float((gx.double() - dA).abs().max() / dA.abs().max())
    assert err <= BWD_BAR, err
    if tap < 0:    # points nobody routes to get exactly 0
        rr = torch.zeros(b, n, dtype=torch.bool, device="cuda")
        live = pooled[0] > 0
        for bi in range(b):
            rr[bi, route[0, bi][live[bi]].long()] = True
        assert bool((gx[~rr] == 0).all())
    else:          # with a tap gradient every point gets one
        assert bool((gx.abs().sum(-1) > 0).all())
        gx_no_tap = sb.ops.frozen_encoder_ex_backward(x, specs, [n], pooled, route, zs, gp, act)
        gx_old = sb.ops.frozen_encoder_backward(x, specs, [n], pooled, route, zs, gp)
        assert torch.equal(gx_no_tap, gx_old)


def _mlp_bn_case(widths, b, seed):
    g = torch.Generator().manual_seed(seed)
    layers = []
    for i in range(len(widths) - 1):
        lin = torch.nn.Linear(widths[i], widths[i + 1])
        with torch.no_grad():
            lin.weight.copy_(torch.randn(lin.weight.shape, generator=g) / widths[i] ** 0.5); lin.bias.copy_(0.1 * torch.randn(widths[i + 1], generator=g))
        bn = None
        if i < len(widths) - 2:
            bn = torch.nn.BatchNorm1d(widths[i + 1], eps=1e-3)
            c = widths[i + 1]
            with torch.no_grad():
                gam = 0.5 + torch.rand(c, generator=g); gam[: c // 4] *= -1
                bn.weight.copy_(gam); bn.bias.copy_(0.3 * torch.randn(c, generator=g))
                bn.running_mean.copy_(0.1 * torch.randn(c, generator=g)); bn.running_var.copy_(0.5 + torch.rand(c, generator=g))
        layers.append((lin.cuda(), None if bn is None else bn.cuda().eval(), i < len(widths) - 2))
    return layers, torch.randn(b, widths[0], generator=g).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("widths", [[1024, 512, 256, 9], [1024, 512, 256, 4096], [1024, 512, 256, 40]], ids=["tnet1", "tnet2", "head"])
@pytest.mark.parametrize("b", [1, 5, 32, 64])
def test_mlp_bn_against_float64(sb, widths, b):
    layers, x = _mlp_bn_case(widths, b, 3 + b)
    specs = tasknets._fc_specs(layers)
    out, asave = sb.ops.frozen_mlp_forward(x, specs, batchnorm=True)
    out2, asave2 = sb.ops.frozen_mlp_forward(x, specs, batchnorm=True)
    out3, _ = sb.ops.frozen_mlp_forward(x, specs, keep_activations=False, batchnorm=True)
    assert torch.equal(out, out2) and torch.equal(out, out3) and all(torch.equal(p, q) for p, q in zip(asave, asave2))
    acts = asave + [out]
    for l, (lin, bn, relu) in enumerate(layers):    # layer l in float64 on the kernel's own input
        src = (x if l == 0 else acts[l - 1]).double()
        w, bb = lin.weight.detach().double(), lin.bias.detach().double()
        z = src @ w.t() + bb
        scale = src.abs() @ w.abs().t() + bb.abs()
        if bn is not None:
            sc = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
            sh = bn.bias.double() - bn.running_mean.double() * sc
            z, scale = z * sc + sh, scale * sc.abs() + sh.abs()
        ref = torch.relu(z) if relu else z
        err = float(((acts[l].double() - ref).abs() / scale).max())
        assert err < MLP_FWD_BAR, (l, err)
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(b)).cuda()
    gx = sb.ops.frozen_mlp_backward(specs, asave, gout, batchnorm=True)
    assert torch.equal(gx, sb.ops.frozen_mlp_backward(specs, asave, gout, batchnorm=True))
    r = gout.double()
    for l in range(len(layers) - 1, -1, -1):
        lin, bn, relu = layers[l]
        if relu:
            r = r * (asave[l] > 0)
        if bn is not None:
            r = r * _fp32_scale_shift(bn)[0]
        r = r @ lin.weight.detach().double()
    err = float((gx.double() - r).abs().max() / r.abs().max())
    assert err < MLP_BWD_BAR, err
    # without BatchNorm the new entries compute what the original ones do, bit for bit
    plain = [{**s, "bn": None} for s in specs]
    assert torch.equal(sb.ops.frozen_mlp_forward(x, plain, batchnorm=True)[0], sb.ops.frozen_mlp_forward(x, plain)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("k", [3, 64])
@pytest.mark.parametrize("b,n", [(1, 1), (5, 128), (32, 1024), (3, 333)])
def test_point_transform_against_float64(sb, k, b, n):
    g = torch.Generator(device="cuda").manual_seed(k + n)
    x = torch.randn(b, n, k, device="cuda", generator=g)
    T = torch.randn(b, k, k, device="cuda", generator=g) / k ** 0.5 + torch.eye(k, device="cuda")
    gout = torch.randn(b, n, k, device="cuda", generator=g)
    out = sb.ops.point_transform_forward(x, T)
    gx, gT = sb.ops.point_transform_backward(x, T, gout)
    assert torch.equal(out, sb.ops.point_transform_forward(x, T))
    gx2, gT2 = sb.ops.point_transform_backward(x, T, gout)
    assert torch.equal(gx, gx2) and torch.equal(gT, gT2)
    xd, Td, gd = x.double(), T.double(), gout.double()
    for got, ref, terms in ((out, xd @ Td, xd.abs() @ Td.abs()), (gx, gd @ Td.transpose(1, 2), gd.abs() @ Td.abs().transpose(1, 2)),
                            (gT, xd.transpose(1, 2) @ gd, xd.abs().transpose(1, 2) @ gd.abs())):
        err = float(((got.double() - ref).abs() / terms.clamp_min(1e-30)).max())
        assert err <= PT_BAR, err
    # the autograd Function: differentiable in both inputs
    xa, Ta = x.clone().requires_grad_(True), T.clone().requires_grad_(True)
    (sb.ops.PointTransformFunction.apply(xa, Ta) * gout).sum().backward()
    assert torch.equal(xa.grad, gx) and torch.equal(Ta.grad, gT)


# ------------------------------------------------------------------------------------------------------------------ GPU: the network
def _margin64(net64, x64):
    """The smallest relative distance, in the float64 forward, of a pooled extreme from its runner-up (each of the three pools) and of a
    unit whose ReLU decision reaches the gradient from its kink: every hidden unit of the points each pool routes to (in the conv layers in
    front of that pool, conv1 and conv2 included for the last two pools), the routed units, and the FC layers' hidden units."""
    m = float("inf")

    def run(convs_bns, y):
        raws, pres = [], []
        for conv, bn in convs_bns:
            z = y @ conv.weight[:, :, 0].t() + conv.bias
            sc = bn.weight / torch.sqrt(bn.running_var + bn.eps)
            sh = bn.bias - bn.running_mean * sc
            raws.append(z)
            pres.append(((z * sc + sh).abs() / ((z * sc).abs() + sh.abs())))
            y = torch.relu(z * sc + sh)
        return raws, pres, y, sc

    def pool_margin(z, sc, hidden, last):
        nonlocal m
        v = z * torch.where(sc >= 0, 1.0, -1.0).to(z)
        top = v.topk(min(2, v.shape[1]), dim=1)
        if v.shape[1] > 1:
            m = min(m, float(((top.values[:, 0] - top.values[:, 1]) / top.values[:, 0].abs()).min()))
        idx = top.indices[:, 0]                                      # (B, C): the routed point of each channel
        m = min(m, float(torch.gather(last, 1, idx[:, None, :]).min()))
        pts = [torch.unique(idx[i]) for i in range(idx.shape[0])]
        for p in hidden:
            m = min(m, min(float(p[i, pts[i]].min()) for i in range(idx.shape[0])))

    def fc_margin(layers, y):
        nonlocal m
        for lin, bn in layers:
            z = y @ lin.weight.t() + lin.bias
            sc = bn.weight / torch.sqrt(bn.running_var + bn.eps)
            sh = bn.bias - bn.running_mean * sc
            m = min(m, float(((z * sc + sh).abs() / ((z * sc).abs() + sh.abs())).min()))
            y = torch.relu(z * sc + sh)
        return y

    with torch.no_grad():
        t1n, t2n = net64.transform_net1, net64.transform_net2
        raws, pres, y, sc = run(list(zip(t1n.convs, t1n.bns)), x64)
        pool_margin(raws[-1], sc, pres[:-1], pres[-1])
        t1 = t1n.to_matrix(t1n.transform(fc_margin([(t1n.fc1, t1n.bn_fc1), (t1n.fc2, t1n.bn_fc2)], y.max(dim=1)[0])))
        fr, fp, h, _ = run(list(zip(net64.convs[:2], net64.bns[:2])), torch.matmul(x64, t1))
        raws, pres, y, sc = run(list(zip(t2n.convs, t2n.bns)), h)
        pool_margin(raws[-1], sc, fp + pres[:-1], pres[-1])
        t2 = t2n.to_matrix(t2n.transform(fc_margin([(t2n.fc1, t2n.bn_fc1), (t2n.fc2, t2n.bn_fc2)], y.max(dim=1)[0])))
        raws, pres, y, sc = run(list(zip(net64.convs[2:], net64.bns[2:])), torch.matmul(h, t2))
        pool_margin(raws[-1], sc, fp + pres[:-1], pres[-1])
        fc_margin([(net64.fc1, net64.bn_fc1), (net64.fc2, net64.bn_fc2)], y.max(dim=1)[0])
    return m


def _conditioned_case(b, n, guard, seed0=10, tries=40):
    """The first (net, x) from seed0 whose float64 forward has a _margin64 above guard, or the one with the largest margin."""
    best = None
    for seed in range(seed0, seed0 + tries):
        net = randomized_net(seed).cuda()
        x = 0.5 * torch.randn(b, n, 3, generator=torch.Generator().manual_seed(500 + seed)).cuda()
        m = _margin64(copy.deepcopy(net).double(), x.double())
        if best is None or m > best[0]:
            best = (m, net, x)
        if m > guard:
            break
    return best


@pytest.fixture()
def _tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n", [(1, 32), (5, 333), (1, 1024), (5, 32), (32, 32), (32, 333), (32, 1024), (70, 32)])
def test_wrapper_against_the_float64_module(sb, record_property, _tf32_off, b, n):
    large = b * n > 40000
    margin, net, x = _conditioned_case(b, n, STEP_GUARD if large else GUARD)
    net.requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    label = torch.randint(0, 40, (b,), generator=torch.Generator().manual_seed(b)).cuda()
    xa = x.clone().requires_grad_(True)
    logits, ep = w(xa)
    loss = w.get_loss(logits, label, ep)
    gx, = torch.autograd.grad(loss, xa)
    net64 = copy.deepcopy(net).double()
    x64 = x.double().requires_grad_(True)
    l64, ep64 = net64(x64)
    loss64 = net64.get_loss(l64, label, ep64)
    g64, = torch.autograd.grad(loss64, x64)
    e = {"logits": float((logits.double() - l64).abs().max() / l64.abs().max()),
         "transform": float((ep["transform"].double() - ep64["transform"]).abs().max() / ep64["transform"].abs().max()),
         "GFV": float((ep["GFV"].double() - ep64["GFV"]).abs().max() / ep64["GFV"].abs().max()),
         "loss": abs(float(loss) - float(loss64)) / abs(float(loss64)),
         "grad": float((gx.double() - g64).abs().max() / g64.abs().max())}
    for k, v in e.items():
        record_property("wrapper_%s_err" % k, v)
    record_property("margin", margin)
    assert e["logits"] <= NET_BAR and e["transform"] <= NET_BAR and e["GFV"] <= NET_BAR and e["loss"] <= NET_BAR, e
    assert e["grad"] <= (STEP_BAR if margin <= GUARD else NET_GRAD_BAR), (e, margin)
    assert ep["critical_set_idx"].dtype == torch.int64 and ep["critical_set_idx"].shape == (b, 1024)
    # repeat runs are bit-identical, and batches above 64 clouds equal their chunks
    logits2, ep2 = w(x)
    assert torch.equal(logits2, logits.detach()) and torch.equal(ep2["transform"], ep["transform"].detach())
    if b > 64:
        la, _ = w(x[:64].contiguous())
        lb, _ = w(x[64:].contiguous())
        assert torch.equal(torch.cat([la, lb]), logits2)


@pytest.mark.gpu
def test_outside_the_envelope_runs_the_module(sb):
    net = randomized_net(3).cuda().requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    x = 0.5 * torch.randn(2, 4097, 3, device="cuda")
    with torch.no_grad():
        lw, ew = w(x)
        ln, en = net(x)
    assert torch.equal(lw, ln) and torch.equal(ew["transform"], en["transform"])


@pytest.mark.gpu
@pytest.mark.parametrize("step", ["cls", "progressive_cls"])
def test_classification_steps_with_the_wrapper(sb, record_property, _tf32_off, step):
    from samplenet_b200 import trainers
    from test_sampler_training import _cloud
    B, N, M = 32, 1024, 32
    x = _cloud(B, N, "bnc", 31)
    torch.manual_seed(7)
    sampler = sb.ClassificationSampleNet(M, group_size=7).cuda().train()
    with torch.no_grad():
        _, proj = copy.deepcopy(sampler)(x)
    best = None
    for seed in range(40, 80):         # a task network well conditioned on the sampler's projected points
        net = randomized_net(seed).cuda()
        m = min(_margin64(copy.deepcopy(net).double(), proj[:, :s].double()) for s in ([M] if step == "cls" else [8, 16, 32]))
        if best is None or m > best[0]:
            best = (m, net)
        if m > STEP_GUARD:
            break
    record_property("margin", best[0])
    y = torch.randint(0, 40, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    runs = []
    for frozen in (True, True, False):
        s = copy.deepcopy(sampler)
        t = copy.deepcopy(best[1]).requires_grad_(False)
        t = tasknets.FrozenPointNetClsTransforms(t) if frozen else t
        st = trainers.ClassificationStep(s, t, M) if step == "cls" else trainers.ProgressiveClassificationStep(s, t, 8, M)
        loss, info = st.loss(x, y)
        loss.backward()
        runs.append((loss.detach(), {k: p.grad.detach().clone() for k, p in s.named_parameters() if p.grad is not None}))
    (la, ga), (lb, gb), (lt, gt) = runs
    assert torch.equal(la, lb) and all(torch.equal(ga[k], gb[k]) for k in ga), "frozen step not bit-identical run to run"
    e_loss = abs(float(la) - float(lt)) / abs(float(lt))
    assert ga.keys() == gt.keys() and len(ga) > 10
    # a parameter is measured against its own largest gradient when that is at least 1e-3 of the largest of all, else against that
    top = max(float(g.abs().max()) for g in gt.values())
    e_grad = max(float((ga[k] - gt[k]).abs().max()) / max(float(gt[k].abs().max()), 1e-3 * top) for k in gt)
    record_property("step_loss_err", e_loss); record_property("step_grad_err", e_grad)
    assert e_loss <= 1e-5 and e_grad <= STEP_BAR, (e_loss, e_grad, best[0])
