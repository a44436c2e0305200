"""The frozen PointNet task networks on CUDA (csrc/frozen_encoder.cu, ops.FrozenEncoderFunction, tasknets.FrozenPointNetCls /
FrozenPointNetAE): the conv stack once over the longest prefix, the max-pool of every prefix from running extrema, and the gradient to the
points through the routed points only.

CPU: the float64 restatement the GPU checks use, pinned against autograd of PointNetCls.eval() / PointNetAE.eval() on each prefix slice;
the C ABI's envelope, workspace sizes and rejections; the wrappers' refusals.  GPU (H100): the forward layer by layer against float64,
pooled values and routes (ties to the first index), bit-exact prefix invariance against one call per prefix, the backward against float64 on
the kernel's own routes and masks and end to end on conditioned instances, repeat runs bit-identical, the wrappers against the wrapped
modules, and the four training steps with the frozen wrapper against the plain module.  Every GPU case has BatchNorm scales < 0 on a quarter
of each layer's channels and last-layer channels pooled to 0 in some clouds but not all, and asserts both."""
import copy
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import test_layers_training_parity as ltp  # noqa: E402
from samplenet_b200 import tasknets  # noqa: E402

# Bars (GPU), about 10x the largest value measured on an H100 80GB HBM3 and no looser than test_layers_training_parity.py's
Z_BAR = 2e-5          # [1.4e-6] zsave[l] against float64 layer l on the kernel's zsave[l-1]: / the point's sum |terms|
POOL_BAR = 2e-5       # [1.3e-6] pooled on the kernel's route: / (|scale| sum |terms of z| + |shift|), the last layer's z bar
TIE_GAP = 1e-6        # the route must be THE arg-max where the runner-up is further than this (relative) from the extreme
BWD_BAR = 5e-6        # [6.1e-7] grad_x against float64 (kernel routes and masks, or plain on a conditioned instance): / max |reference|
GUARD = 1e-6          # conditioned instances: no routed unit this close to its ReLU kink, no pooled extreme this close to its runner-up
STEP_GUARD = 1e-7     # ... for the task networks of whole steps (~14 000 routed points x 320 hidden units per step: 1e-6 is rarely met)


# ------------------------------------------------------------------------------------------------------------------ references
def _layers64(net):
    """Per conv layer (W, b, scale, shift) in float64, from the module's eval-mode BatchNorm."""
    out = []
    for conv, bn in zip(net.convs, net.bns):
        sc = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
        out.append((conv.weight.detach().double()[:, :, 0], conv.bias.detach().double(), sc, bn.bias.detach().double() - bn.running_mean.detach().double() * sc))
    return out


def restate64(net, x, sizes, zs=None):
    """The frozen encoder in float64: raw conv outputs (B, N, c_l) and pooled (P, B, C), the max of each prefix taken at the first extreme
    of sign(scale) * z of the last layer.  zs: per hidden layer, raw outputs whose VALUES replace the graph's (gradients still flow)."""
    L = _layers64(net)
    h, raw = x.double(), []
    for l, (w, b, sc, sh) in enumerate(L):
        z = h @ w.t() + b
        if zs is not None and l < len(L) - 1:
            z = z + (zs[l].view(z.shape).double() - z).detach()
        raw.append(z)
        h = torch.relu(z * sc + sh)
    sgn = torch.where(L[-1][2] >= 0, 1.0, -1.0).to(h)
    pooled = []
    for s in sizes:
        idx = (raw[-1][:, :s].detach() * sgn).argmax(dim=1)   # first index on ties (CPU; on CUDA only where there are none)
        pooled.append(torch.gather(h, 1, idx[:, None, :]).squeeze(1))
    return raw, torch.stack(pooled)


def _fp32_masks(net, zs):
    """The ReLU masks the kernels decide: fmaf(z, scale, shift) > 0 with the fp32 eval-mode scale gamma * (1 / sqrtf(var + eps)) and shift
    beta - mean * scale (one rounding, as the contracted kernel expression); the sign of the exact fused value is that of this float64 sum."""
    out = []
    for z, bn in zip(zs, net.bns):
        inv = 1.0 / torch.sqrt(bn.running_var.detach().float() + bn.eps)
        sc = bn.weight.detach().float() * inv
        sh = (bn.bias.detach().double() - bn.running_mean.detach().float().double() * sc.double()).float()
        out.append((z.double() * sc.double() + sh.double() > 0, sc))
    return out


def grad_on_kernel_routes64(net, zs, pooled, route, g):
    """Float64 grad_x of sum(g * pooled) along the kernel's routes and its fp32 masks (hidden zsave values, routed coefficient
    g * scale * [pooled > 0])."""
    L = _layers64(net)
    masks = _fp32_masks(net, zs)
    P, B, C = pooled.shape
    N = zs[0].shape[0] // B
    w_last = L[-1][0]
    inv = 1.0 / torch.sqrt(net.bns[-1].running_var.detach().float() + net.bns[-1].eps)
    sc_last = (net.bns[-1].weight.detach().float() * inv).double()
    coef = g.double() * sc_last * (pooled > 0).double()
    dA = torch.zeros(B, N, w_last.shape[1], dtype=torch.float64, device=g.device)
    for p in range(P):
        idx = route[p].long()[:, :, None].expand(B, C, w_last.shape[1])
        dA.scatter_add_(1, idx, coef[p][:, :, None] * w_last[None])
    for l in range(len(L) - 2, -1, -1):
        m, sc = masks[l]
        dz = dA * sc.double() * m.view(B, N, -1).double()
        dA = dz @ L[l][0]
    return dA


# ------------------------------------------------------------------------------------------------------------------ networks
def _randomize(net, seed):
    """BatchNorm running statistics and affine parameters away from the identity, a quarter of every layer's scales < 0."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for conv, bn in zip(net.convs, net.bns):
            c = bn.num_features
            conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) * (1.0 / conv.weight.shape[1]) ** 0.5)
            conv.bias.copy_(0.1 * torch.randn(c, generator=g))
            gam = 0.5 + torch.rand(c, generator=g)
            gam[torch.randperm(c, generator=g)[: c // 4]] *= -1
            bn.weight.copy_(gam)
            bn.bias.copy_(0.3 * torch.randn(c, generator=g))
            bn.running_mean.copy_(0.1 * torch.randn(c, generator=g))
            bn.running_var.copy_(0.5 + torch.rand(c, generator=g))
    return net


DEAD = 16   # last-layer channels given a shift that pools them to 0 in about half of the clouds


def _kill_channels(net, x, sizes):
    """Shift DEAD last-layer channels (both scale signs) so that their longest prefix pools to 0 in some clouds but not in others."""
    raw, _ = restate64(net, x, [sizes[-1]])
    L = _layers64(net)
    sc = L[-1][2]
    bn = net.bns[-1]
    chans = torch.cat([torch.nonzero(sc >= 0)[: DEAD // 2, 0], torch.nonzero(sc < 0)[: DEAD // 2, 0]])
    ext = (raw[-1][:, : sizes[-1]] * sc).amax(dim=1)   # (B, C): max of scale * z, the pooled value before the shift
    with torch.no_grad():
        for k, c in enumerate(chans.tolist()):
            e = ext[:, c].sort()[0]
            # one cloud: alternate channels pooled to 0 and not
            h = (len(e) - 1) // 2
            mid = 0.5 * (e[h] + e[h + 1]) if len(e) > 1 else e[0] + (1.0 if k % 2 else -1.0)
            # shift = -mid: clouds with ext < mid pool to 0, the others do not
            bn.bias[c] = float(-mid + bn.running_mean[c].double() * sc[c])
    return chans


def make_case(kind, b, n, seed, dup=False):
    """(net, x, sizes, dead channels) on the GPU."""
    net = (tasknets.PointNetCls() if kind == "cls" else tasknets.PointNetAE(n_pc_points=2048)).double()
    _randomize(net, seed)
    g = torch.Generator().manual_seed(1000 + seed)
    x = torch.randn(b, n, 3, generator=g, dtype=torch.float64) * 0.5
    if dup:   # outlying points copied to later indices in the same tile and in later tiles: exact ties at many channels' extremes
        for i in range(4):
            x[:, i] *= 4.0
            for j in (i + 5, i + 131, min(n - 1, i + 263)):
                x[:, j] = x[:, i]
    x = x.float().double()
    sizes = SIZES[(kind, b, n)]
    dead = _kill_channels(net, x, sizes)
    return net.float().cuda().eval().requires_grad_(False), x.float().cuda(), sizes, dead


SIZES = {
    ("cls", 32, 1024): [8 * 2 ** i for i in range(8)],
    ("ae", 50, 2048): [16 * 2 ** i for i in range(8)],
    ("cls", 5, 333): [1, 7, 127, 128, 129, 300, 333],
    ("ae", 5, 333): [1, 7, 127, 128, 129, 300, 333],
    ("cls", 1, 1024): [8, 64, 1000, 1024],
    ("ae", 1, 777): [1, 128, 256, 777],
    ("cls", 4, 300): [3, 6, 130, 140, 300],
}
CASES = [("cls", 32, 1024, False), ("ae", 50, 2048, False), ("cls", 5, 333, False), ("ae", 5, 333, False), ("cls", 1, 1024, False),
         ("ae", 1, 777, False), ("cls", 4, 300, True)]


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("kind", ["cls", "ae"])
def test_restatement_matches_module_autograd_on_prefix_slices(kind):
    torch.manual_seed(3)
    net = _randomize((tasknets.PointNetCls() if kind == "cls" else tasknets.PointNetAE(n_pc_points=64)).double(), 4).eval()
    x = (torch.randn(3, 50, 3, dtype=torch.float64) * 0.5).requires_grad_(True)
    sizes = [1, 5, 17, 50]
    w = torch.randn(len(sizes), 3, net.bns[-1].num_features, dtype=torch.float64)
    _, pooled = restate64(net, x, sizes)
    mods = [net(x[:, :s])[1]["GFV"] if kind == "cls" else net.encode(x[:, :s]) for s in sizes]
    for p in range(len(sizes)):
        assert torch.allclose(pooled[p], mods[p], rtol=1e-12, atol=1e-12)
    g_re = torch.autograd.grad((w * pooled).sum(), x)[0]
    g_mod = torch.autograd.grad(sum((w[p] * mods[p]).sum() for p in range(len(sizes))), x)[0]
    assert torch.allclose(g_re, g_mod, rtol=1e-10, atol=1e-12)
    if kind == "cls":   # critical_set_idx of the module is the restatement's route where the pooled value is > 0
        _, ep = net(x)
        raw, _ = restate64(net, x, [50])
        sgn = torch.where(_layers64(net)[-1][2] >= 0, 1.0, -1.0).double()
        r = (raw[-1] * sgn).argmax(1)
        live = ep["GFV"] > 0
        assert torch.equal(ep["critical_set_idx"][live], r[live])


_next_ptr = [0x90000]


def _ptr():
    _next_ptr[0] += 0x1000
    return _next_ptr[0]


def _table(widths, eps=1e-3, running=True):
    from samplenet_b200._lib import Layer
    arr = (Layer * (len(widths) - 1))()
    for i in range(len(widths) - 1):
        L = arr[i]
        L.c_in, L.c_out = widths[i], widths[i + 1]
        L.weight, L.bias, L.bn_weight, L.bn_bias = _ptr(), _ptr(), _ptr(), _ptr()
        if running:
            L.bn_running_mean, L.bn_running_var = _ptr(), _ptr()
        L.bn_eps, L.bn_momentum, L.relu = eps, 0.1, 1
    return arr


CLS_W, AE_W = [3, 64, 64, 64, 128, 1024], [3, 64, 128, 128, 256, 128]


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


def test_envelope(lib):
    for w in (CLS_W, AE_W):
        t = _table(w)
        for b, n, P in ((1, 1, 1), (32, 1024, 8), (50, 2048, 8), (64, 4096, 16), (5, 333, 7)):
            assert lib.snb200_frozen_encoder_supported(b, n, 5, t, P) == 1, (w, b, n, P)
        for b, n, P in ((0, 1024, 8), (65, 1024, 8), (32, 4097, 8), (32, 0, 8), (32, 1024, 0), (32, 1024, 17)):
            assert lib.snb200_frozen_encoder_supported(b, n, 5, t, P) == 0, (w, b, n, P)
    # widths just outside: last layer 1032 wide, a 264-wide hidden layer, hidden width not a multiple of 8, 4 input channels, one layer
    for w in ([3, 64, 64, 64, 128, 1032], [3, 64, 128, 128, 264, 128], [3, 64, 60, 64, 128, 1024], [4, 64, 64, 64, 128, 1024], [3, 1024]):
        assert lib.snb200_frozen_encoder_supported(32, 1024, len(w) - 1, _table(w), 8) == 0, w
    assert lib.snb200_frozen_encoder_supported(32, 1024, 5, _table([3, 64, 64, 64, 128, 8]), 8) == 1


def test_workspace_sizes(lib):
    cls, ae = _table(CLS_W), _table(AE_W)
    # (tiles + prefixes) per cloud x C x (value + index); without zsave also two buffers of the widest hidden layer
    assert lib.snb200_frozen_encoder_workspace_bytes(32, 1024, 5, cls, 8, 1) == 32 * (8 + 8) * 1024 * 8
    assert lib.snb200_frozen_encoder_workspace_bytes(32, 1024, 5, cls, 8, 0) == 32 * 16 * 1024 * 8 + 2 * 32 * 1024 * 128 * 4
    assert lib.snb200_frozen_encoder_workspace_bytes(50, 2048, 5, ae, 8, 1) == 50 * (16 + 8) * 128 * 8
    assert lib.snb200_frozen_encoder_workspace_bytes(5, 333, 5, ae, 7, 1) == 5 * (3 + 7) * 128 * 8
    # backward: one bit per (point, last-layer channel)
    assert lib.snb200_frozen_encoder_backward_workspace_bytes(32, 1024, 5, cls, 8) == 32 * 1024 * 32 * 4
    assert lib.snb200_frozen_encoder_backward_workspace_bytes(50, 2048, 5, ae, 8) == 50 * 2048 * 4 * 4
    assert lib.snb200_frozen_encoder_workspace_bytes(65, 1024, 5, cls, 8, 1) == 0
    assert lib.snb200_frozen_encoder_backward_workspace_bytes(32, 1024, 5, cls, 17) == 0


def _call(lib, entry, b, n, table, sizes, ws_bytes, nconv=5):
    import ctypes
    cs = (ctypes.c_int * max(len(sizes), 1))(*sizes)
    z = (ctypes.c_void_p * 8)(*[_ptr() for _ in range(8)])
    if entry == "forward":
        rc = lib.snb200_frozen_encoder_forward(b, n, _ptr(), nconv, table, len(sizes), cs, _ptr(), _ptr(), z, _ptr(), ws_bytes, None)
    else:
        rc = lib.snb200_frozen_encoder_backward(b, n, _ptr(), nconv, table, len(sizes), cs, _ptr(), _ptr(), z, _ptr(), _ptr(), _ptr(), ws_bytes, None)
    return rc, lib.snb200_last_error().decode()


@pytest.mark.parametrize("entry", ["forward", "backward"])
def test_rejections(lib, entry):
    """Every malformed call returns SNB200_EINVAL (-1) or SNB200_EWORKSPACE (-2) with its message, before anything launches (the pointers
    here are never dereferenced)."""
    who = "frozen_encoder_%s: " % entry
    cls = _table(CLS_W)
    big = 1 << 40
    cases = [
        ((32, 1024, cls, [], big), -1, who + "1..16 prefixes expected"),
        ((32, 1024, cls, list(range(1, 18)), big), -1, who + "1..16 prefixes expected"),
        ((32, 1024, cls, [8, 8, 16], big), -1, who + "prefix sizes must be ascending"),
        ((32, 1024, cls, [16, 8], big), -1, who + "prefix sizes must be ascending"),
        ((32, 1024, cls, [0, 8], big), -1, who + "prefix sizes must be ascending"),
        ((32, 1024, cls, [8, 1025], big), -1, who + "prefix sizes must be ascending"),
        ((32, 1024, _table(CLS_W, running=False), [8], big), -1, who + "eval mode needs running statistics"),
        ((32, 1024, _table([3, 64, 64, 64, 128, 1032]), [8], big), -1, who + "shape outside the frozen encoder's envelope"),
        ((32, 1024, _table([3, 64, 128, 128, 264, 128]), [8], big), -1, who + "shape outside the frozen encoder's envelope"),
        ((65, 1024, cls, [8], big), -1, who + "shape outside the frozen encoder's envelope"),
        ((32, 4097, cls, [8], big), -1, who + "shape outside the frozen encoder's envelope"),
    ]
    need = (lib.snb200_frozen_encoder_workspace_bytes(32, 1024, 5, cls, 2, 1) if entry == "forward"
            else lib.snb200_frozen_encoder_backward_workspace_bytes(32, 1024, 5, cls, 2))
    cases.append(((32, 1024, cls, [8, 1024], need - 1), -2, who + "workspace"))
    for args, rc_want, msg in cases:
        rc, err = _call(lib, entry, *args)
        assert rc == rc_want and err.startswith(msg), (args[3], rc, err)


def test_wrapper_refusals():
    net = tasknets.PointNetCls()
    with pytest.raises(ValueError):   # parameters that require grad while grad is enabled: this path gives no parameter gradients
        tasknets.FrozenPointNetCls(net)(torch.zeros(2, 16, 3))
    net.requires_grad_(False)
    w = tasknets.FrozenPointNetCls(net)
    assert not w.training and not net.training
    with pytest.raises(ValueError):
        w.train()
    with pytest.raises(ValueError):
        w.train(True)
    w.eval()
    with pytest.raises(RuntimeError, match="CUDA-only"):   # CPU tensors: no fallback
        w(torch.zeros(2, 16, 3))
    ae = tasknets.FrozenPointNetAE(tasknets.PointNetAE(64).requires_grad_(False))
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ae.prefixes(torch.zeros(2, 16, 3), [8, 16])
    with pytest.raises(ValueError):
        ae.train()
    with torch.no_grad():   # grad disabled: grad-requiring parameters are fine (nothing would be differentiated)
        with pytest.raises(RuntimeError, match="CUDA-only"):
            tasknets.FrozenPointNetAE(tasknets.PointNetAE(64))(torch.zeros(2, 16, 3))


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _fwd(sb, net, x, sizes, keep=True):
    return sb.ops.frozen_encoder_forward(x, tasknets._conv_specs(net), sizes, keep_activations=keep)


def _check_forward(net, x, sizes, pooled, route, zs, dead):
    """Layer by layer against float64, pooled on the kernel's route, the route an arg-max.  Returns measured maxima."""
    B, N, _ = x.shape
    L = _layers64(net)
    rep = {}
    h = x.double()
    for l, (w, b, sc, sh) in enumerate(L[:-1]):
        z64 = h @ w.t() + b
        terms = h.abs() @ w.abs().t() + b.abs()
        rep["z%d" % l] = ((zs[l].view(B, N, -1).double() - z64).abs() / terms).max().item()
        h = torch.relu(zs[l].view(B, N, -1).double() * sc + sh)
    w, b, sc, sh = L[-1]
    zL = h @ w.t() + b
    aL = torch.relu(zL * sc + sh)
    at = torch.gather(aL, 1, route.long().permute(1, 0, 2).reshape(B, -1, w.shape[0])).view(B, len(sizes), -1).permute(1, 0, 2)
    terms = torch.gather(h.abs() @ w.abs().t() + b.abs(), 1, route.long().permute(1, 0, 2).reshape(B, -1, w.shape[0]))
    terms = terms.view(B, len(sizes), -1).permute(1, 0, 2)
    rep["pooled"] = ((pooled.double() - at).abs() / (terms * sc.abs() + sh.abs())).max().item()
    v = zL * torch.where(sc >= 0, 1.0, -1.0).to(zL)
    clear_total = 0
    for p, s in enumerate(sizes):
        top = v[:, :s].topk(min(2, s), dim=1)
        vr = torch.gather(v, 1, route[p].long()[:, None, :]).squeeze(1)
        assert (route[p] < s).all() and (route[p] >= 0).all()
        assert (vr >= top.values[:, 0] - TIE_GAP * top.values[:, 0].abs().clamp_min(1e-30)).all(), "route is not an extreme"
        if s > 1:
            clear = (top.values[:, 0] - top.values[:, 1]) > TIE_GAP * top.values[:, 0].abs()
        else:
            clear = torch.ones_like(route[p], dtype=torch.bool)
        clear_total += int(clear.sum())
        assert torch.equal(route[p][clear].long(), top.indices[:, 0][clear]), "route differs from the float64 arg-max"
    assert clear_total > 0
    # the case covers negative scales and channels pooled to 0 in some clouds but not all
    assert (sc < 0).any() and (sc > 0).any()
    last = pooled[-1][:, dead]
    assert (last == 0).any() and (last > 0).any(), "no channel pooled to 0 in some clouds but not all"
    if B > 1:
        assert ((last == 0).any(0) & (last > 0).any(0)).any()
    return rep


@pytest.mark.gpu
@pytest.mark.parametrize("kind,b,n,dup", CASES)
def test_forward_against_float64_and_prefix_invariance(sb, kind, b, n, dup):
    net, x, sizes, dead = make_case(kind, b, n, 11, dup)
    pooled, route, zs = _fwd(sb, net, x, sizes)
    rep = _check_forward(net, x, sizes, pooled, route, zs, dead)
    print("forward", kind, b, n, rep)
    assert max(v for k, v in rep.items() if k.startswith("z")) <= Z_BAR, rep
    assert rep["pooled"] <= POOL_BAR, rep
    # repeat: bit-identical; forward only (no zsave): the same pooled values and routes
    p2, r2, z2 = _fwd(sb, net, x, sizes)
    assert torch.equal(pooled, p2) and torch.equal(route, r2) and all(torch.equal(a, c) for a, c in zip(zs, z2))
    p3, r3, z3 = _fwd(sb, net, x, sizes, keep=False)
    assert z3 is None and torch.equal(pooled, p3) and torch.equal(route, r3)
    # prefix invariance, bit-exact: every prefix equals a one-prefix call on the slice
    for p, s in enumerate(sizes):
        ps, rs, zss = _fwd(sb, net, x[:, :s].contiguous(), [s])
        assert torch.equal(ps[0], pooled[p]) and torch.equal(rs[0], route[p]), (p, s)
        for a, c in zip(zss, zs):
            assert torch.equal(a.view(b, s, -1), c.view(b, n, -1)[:, :s]), (p, s)
    if dup:   # exact ties at the extremes go to the first index
        ties = 0
        for i in range(4):
            copies = torch.tensor([i + 5, i + 131, min(n - 1, i + 263)], device="cuda")
            for p, s in enumerate(sizes):
                hit = route[p] == i
                ties += int(hit.sum()) if s > i + 5 else 0
                for j in copies.tolist():
                    assert not (route[p] == j).any(), "a tied copy won over the first index"
        assert ties > 0, "no tie at an extreme"


def _margin(net64, x64, sizes):
    """The smallest relative distance of a pooled extreme from its runner-up and of a routed unit from its ReLU kink (relative to
    |scale z| + |shift|): every hidden unit of a point some prefix routes to, and the routed unit of the last layer itself."""
    b, n, _ = x64.shape
    raw, _ = restate64(net64, x64, sizes)
    L = _layers64(net64)
    sgn = torch.where(L[-1][2] >= 0, 1.0, -1.0).double()
    v = raw[-1] * sgn
    _, _, sc, sh = L[-1]
    pts, m = set(), float("inf")
    for s in sizes:
        top = v[:, :s].topk(min(2, s), dim=1)
        if s > 1:
            m = min(m, ((top.values[:, 0] - top.values[:, 1]) / top.values[:, 0].abs()).min().item())
        z = top.values[:, 0] * sgn
        m = min(m, ((z * sc + sh).abs() / ((z * sc).abs() + sh.abs())).min().item())
        pts.update((top.indices[:, 0] + torch.arange(b, device=x64.device)[:, None] * n).flatten().tolist())
    idx = torch.tensor(sorted(pts), device=x64.device)
    for z, (_, _, sc, sh) in zip(raw[:-1], L[:-1]):
        zp = z.reshape(-1, z.shape[-1])[idx]
        m = min(m, ((zp * sc + sh).abs() / ((zp * sc).abs() + sh.abs())).min().item())
    return m


def _conditioned(kind, b, n, seed0):
    """The first case from seed0 whose float64 forward has a _margin above GUARD."""
    for seed in range(seed0, seed0 + 40):
        net, x, sizes, dead = make_case(kind, b, n, seed)
        if _margin(copy.deepcopy(net).double().cpu(), x.double().cpu(), sizes) > GUARD:
            return net, x, sizes, dead
    raise AssertionError("no conditioned instance")


@pytest.mark.gpu
@pytest.mark.parametrize("kind,b,n,dup", CASES)
def test_backward_against_float64(sb, kind, b, n, dup):
    net, x, sizes, dead = make_case(kind, b, n, 11, dup)
    pooled, route, zs = _fwd(sb, net, x, sizes)
    g = torch.randn(pooled.shape, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
    specs = tasknets._conv_specs(net)
    gx = sb.ops.frozen_encoder_backward(x, specs, sizes, pooled, route, zs, g)
    gx2 = sb.ops.frozen_encoder_backward(x, specs, sizes, pooled, route, zs, g)
    assert torch.equal(gx, gx2), "backward not bit-identical run to run"
    ref = grad_on_kernel_routes64(net, [z.double() for z in zs], pooled, route, g)
    err = ((gx.double() - ref).abs().max() / ref.abs().max()).item()
    print("backward on kernel routes", kind, b, n, err)
    assert err <= BWD_BAR, err
    # points nobody routes to (with a live pooled value) get exactly 0
    live = pooled > 0
    rr = torch.zeros(b, n, dtype=torch.bool, device="cuda")
    for p in range(len(sizes)):
        for bi in range(b):
            rr[bi, route[p, bi][live[p, bi]].long()] = True
    assert (gx[~rr] == 0).all() and (~rr).any()


@pytest.mark.gpu
@pytest.mark.parametrize("kind,b,n", [("cls", 5, 333), ("ae", 5, 333), ("ae", 1, 777)])
def test_backward_end_to_end_on_conditioned_instances(sb, kind, b, n):
    net, x, sizes, _ = _conditioned(kind, b, n, 20)
    x.requires_grad_(True)
    g = torch.randn(len(sizes), b, net.bns[-1].num_features, generator=torch.Generator(device="cuda").manual_seed(6), device="cuda")
    pooled, _ = sb.ops.FrozenEncoderFunction.apply(x, tasknets._conv_specs(net), sizes)
    gx = torch.autograd.grad((pooled * g).sum(), x)[0]
    x64 = x.detach().double().cpu().requires_grad_(True)
    net64 = copy.deepcopy(net).double().cpu()
    _, p64 = restate64(net64, x64, sizes)
    ref = torch.autograd.grad((p64 * g.double().cpu()).sum(), x64)[0]
    err = ((gx.double().cpu() - ref).abs().max() / ref.abs().max()).item()
    print("backward end to end", kind, b, n, err)
    assert err <= BWD_BAR, err


def _tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,b,n,dup", [("cls", 32, 1024, False), ("ae", 50, 2048, False), ("cls", 5, 333, False), ("cls", 4, 300, True)])
def test_wrappers_against_the_modules(sb, monkeypatch, kind, b, n, dup):
    _tf32_off(monkeypatch)
    net, x, sizes, _ = make_case(kind, b, n, 11, dup)
    net64 = copy.deepcopy(net).double()
    with torch.no_grad():
        if kind == "cls":
            w = tasknets.FrozenPointNetCls(net)
            logits, ep = w(x)
            l64, ep64 = net64(x.double())
            assert ((logits.double() - l64).abs().max() / l64.abs().max()).item() <= 1e-5
            assert ((ep["GFV"].double() - ep64["GFV"]).abs().max() / ep64["GFV"].abs().max()).item() <= 1e-5
            # critical_set_idx where no near-tie exists (float64's CUDA argmax on exact ties is not defined)
            raw, _ = restate64(net64, x.double(), [n])
            v = raw[-1] * torch.where(_layers64(net64)[-1][2] >= 0, 1.0, -1.0).to(raw[-1])
            top = v.topk(2, dim=1).values
            clear = ((top[:, 0] - top[:, 1]) > TIE_GAP * top[:, 0].abs()) | (ep64["GFV"] == 0)
            assert ep["critical_set_idx"].dtype == torch.int64
            assert torch.equal(ep["critical_set_idx"][clear], ep64["critical_set_idx"][clear])
            pre = w.prefixes(x, sizes)
            want = torch.stack([net64(x[:, :s].double())[0] for s in sizes])
        else:
            w = tasknets.FrozenPointNetAE(net)
            out = w(x)
            o64 = net64(x.double())
            assert ((out.double() - o64).abs().max() / o64.abs().max()).item() <= 1e-5
            pre = w.prefixes(x, sizes)
            want = torch.stack([net64(x[:, :s].double()) for s in sizes])
        assert pre.shape == want.shape
        assert ((pre.double() - want).abs().max() / want.abs().max()).item() <= 1e-5


# ------------------------------------------------------------------------------------------------------------------ whole steps
def _task_net_conditioned(kind, proj, sizes, seed0):
    """A task network (random BatchNorm, a quarter of the scales < 0) whose _margin on the sampler's projected points exceeds STEP_GUARD,
    or the one with the largest margin over 40 seeds."""
    best = None
    for seed in range(seed0, seed0 + 40):
        net = _randomize((tasknets.PointNetCls() if kind == "cls" else tasknets.PointNetAE(n_pc_points=2048)).double(), seed).to(proj.device)
        m = _margin(net, proj.double(), sizes)
        if best is None or m > best[0]:
            best = (m, net)
        if m > STEP_GUARD:
            break
    print("task network margin", best[0])
    return best[1].float()


STEPS = ["cls", "progressive_cls", "rec", "progressive_rec"]


@pytest.mark.gpu
@pytest.mark.parametrize("step", STEPS)
def test_steps_with_the_frozen_wrapper(sb, monkeypatch, step):
    from samplenet_b200 import trainers
    from test_sampler_training import _cloud
    _tf32_off(monkeypatch)
    cls_like = step.endswith("cls")
    B, N = (32, 1024) if cls_like else (50, 2048)
    M = {"cls": 32, "progressive_cls": 1024, "rec": 64, "progressive_rec": 2048}[step]
    x = _cloud(B, N, "bnc", 31)
    torch.manual_seed(7)
    sampler = (sb.ClassificationSampleNet(M, group_size=7) if cls_like else sb.ReconstructionSampleNet(M)).cuda().train()
    with torch.no_grad():
        _, proj = copy.deepcopy(sampler)(x)
    sizes = {"cls": [M], "progressive_cls": [8 * 2 ** i for i in range(8)], "rec": [M], "progressive_rec": [16 * 2 ** i for i in range(8)]}[step]
    task = _task_net_conditioned("cls" if cls_like else "ae", proj, sizes, 40)
    y = torch.randint(0, 40, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))

    def run(s, t):
        if step == "cls":
            return trainers.ClassificationStep(s, t, M).loss(x, y)
        if step == "progressive_cls":
            return trainers.ProgressiveClassificationStep(s, t, 8, M).loss(x, y)
        if step == "rec":
            return trainers.ReconstructionStep(s, t, M).loss(x)
        return trainers.ProgressiveReconstructionStep(s, t).loss(x)

    runs = []
    for frozen in (True, True, False):
        s = copy.deepcopy(sampler)
        t = copy.deepcopy(task).requires_grad_(False)
        loss, info = run(s, tasknets.FrozenPointNetCls(t) if frozen and cls_like else tasknets.FrozenPointNetAE(t) if frozen else t)
        task_loss = info["loss_classifier" if cls_like else "loss_ae"]
        loss.backward()
        runs.append((loss.detach(), {k: p.grad.detach().clone() for k, p in s.named_parameters() if p.grad is not None}))
    (la, ga), (lb, gb), (lt, gt) = runs
    assert torch.equal(la, lb) and all(torch.equal(ga[k], gb[k]) for k in ga), "frozen step not bit-identical run to run"
    assert abs(float(la) - float(lt)) <= 1e-5 * abs(float(lt)), (float(la), float(lt))
    assert ga.keys() == gt.keys()
    # the rule of test_progressive_training._compare_routes: a generator tensor whose true gradient is 0 is measured against its layer's
    # weight gradient
    gen = dict(sampler._generator_named_parameters())
    by_name = {id(p): k for k, p in sampler.named_parameters()}
    alias = {by_name[id(p)]: k for k, p in gen.items()}
    scale = ltp._scales(sampler, {alias[k]: gt[k] for k in alias})
    errs = {k: ((ga[k] - gt[k]).abs().max().item() / (scale[alias[k]] if k in alias else max(gt[k].abs().max().item(), 1e-30))) for k in gt}
    worst = max(errs.values())
    print("step", step, "loss", float(la), float(lt), "task loss", float(task_loss), "worst grad", worst, max(errs, key=errs.get))
    assert worst <= 2e-3, worst
