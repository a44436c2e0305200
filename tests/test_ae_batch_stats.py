"""The frozen autoencoder normalised with each prefix's own batch statistics, as the reconstruction sampler trainers compute it:
PointNetAE.encode(x, batch_stats=True) (torch), FrozenPointNetAE(..., batch_stats=True) on the batch-statistics encoder
(snb200_frozen_encoder_bstat_*, csrc/frozen_encoder_bstat.cu), and ReconstructionStep / ProgressiveReconstructionStep(ae_batch_stats=True).

CPU: the torch route against a hand-written float64 restatement, per prefix and in both module modes; the module's state untouched; the
default call unchanged; the C ABI's envelope, workspace sizes and rejections.  GPU (H100): the forward layer by layer against float64 on the
kernel's own values (statistics, raw outputs, pooled values and routes), the backward against float64 autograd with the kernel's masks,
determinism and prefix invariance (bit for bit), the steps through the CUDA wrapper against the plain module, the module's state after steps
on every route, the fallbacks, and the entries' write set."""
import copy
import ctypes
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from samplenet_b200 import tasknets  # noqa: E402

# Bars (GPU): measured values on an H100 80GB HBM3 in brackets
STAT_BAR = 2e-5       # [2.6e-7] a group's mean and variance against float64 on the kernel's raw outputs: / mean of z^2
Z_BAR = 2e-5          # [1.5e-6] raw output of layer l against float64 on the kernel's layer l-1 and statistics: / the row's sum |terms|
POOL_BAR = 2e-5       # [8.3e-8] pooled on the kernel's route: / (|scale| |z| + |shift|)
GRAD_BAR = 1e-4       # [8.1e-6] grad_x against float64 autograd of the contract with the kernel's masks and routes: / max |reference|
STEP_LOSS_BAR = 1e-5  # as test_frozen_tasknets.test_steps_with_the_frozen_wrapper
STEP_GRAD_BAR = 2e-3

POW2 = [16 * 2 ** i for i in range(8)]
CASES = [(50, 2048, POW2), (5, 333, [1, 7, 64, 333]), (1, 777, [1, 777])]


def _a256(nbytes):
    return -(-nbytes // 256) * 256


def _randomize(net, seed):
    """Parameters and running statistics away from the identity, a quarter of every layer's BatchNorm scales < 0."""
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
            bn.running_mean.copy_(0.5 * torch.randn(c, generator=g))
            bn.running_var.copy_(0.2 + 2 * torch.rand(c, generator=g))
        for lin in net.dec:
            lin.weight.copy_(torch.randn(lin.weight.shape, generator=g) * (1.0 / lin.weight.shape[1]) ** 0.5)
    return net


def restate64(net, x, sizes):
    """The contract in float64, by hand: per prefix s, every conv layer normalised with the mean and biased variance over the B * s points
    of x[:, :s], ReLU, then the max over the points.  Returns (P, B, C)."""
    out = []
    for s in sizes:
        h = x[:, :s].double()
        for conv, bn in zip(net.convs, net.bns):
            z = h @ conv.weight.detach().double()[:, :, 0].t() + conv.bias.detach().double()
            mean = z.mean(dim=(0, 1))
            var = ((z - mean) ** 2).mean(dim=(0, 1))
            h = torch.relu((z - mean) / torch.sqrt(var + bn.eps) * bn.weight.detach().double() + bn.bias.detach().double())
        out.append(h.max(dim=1)[0])
    return torch.stack(out)


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("train_mode", [False, True])
def test_torch_route_against_float64(train_mode):
    net = _randomize(tasknets.PointNetAE(n_pc_points=64), 3).train(train_mode)
    x = torch.rand(4, 300, 3, generator=torch.Generator().manual_seed(4)) - 0.5
    sizes = [1, 7, 128, 300]
    state = {k: v.clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        got = torch.stack([net.encode(x[:, :s], batch_stats=True) for s in sizes])
        full = net(x, batch_stats=True)
    want = restate64(net, x, sizes)
    err = ((got.double() - want).abs().max() / want.abs().max()).item()
    assert err <= 1e-5, err
    assert torch.allclose(full.double(), net.decode(want[-1].float()).double(), rtol=1e-4, atol=1e-5)
    # nothing of the module changes, num_batches_tracked and the running statistics included
    after = net.state_dict()
    assert state.keys() == after.keys() and all(torch.equal(state[k], after[k]) for k in state)


def test_default_call_unchanged():
    net = _randomize(tasknets.PointNetAE(n_pc_points=64), 5).eval()
    x = torch.rand(3, 100, 3, generator=torch.Generator().manual_seed(6))
    with torch.no_grad():
        y = x.permute(0, 2, 1)
        for conv, bn in zip(net.convs, net.bns):
            y = F.relu(bn(conv(y)))
        want = net.decode(torch.max(y, 2)[0])
        assert torch.equal(net(x), want) and torch.equal(net.encode(x), torch.max(y, 2)[0])
        # eval-mode and batch-statistics results differ once the running statistics differ from the batch's
        assert not torch.allclose(net(x, batch_stats=True), want)


def test_cuda_wrapper_refuses_batch_stats_in_training_mode():
    w = tasknets.CudaPointNetAE(tasknets.PointNetAE(64)).train()
    with pytest.raises(ValueError):
        w(torch.zeros(2, 16, 3), batch_stats=True)


_next = [0x7000_0000]


def _ptr():
    _next[0] += 0x1000
    return _next[0]


AE = [3, 64, 128, 128, 256, 128]


def _table(widths, bn=True, relu=1):
    from samplenet_b200._lib import Layer

    arr = (Layer * (len(widths) - 1))()
    for i in range(len(widths) - 1):
        L = arr[i]
        L.c_in, L.c_out, L.weight, L.bias = widths[i], widths[i + 1], _ptr(), _ptr()
        if bn:
            L.bn_weight, L.bn_bias, L.bn_running_mean, L.bn_running_var = _ptr(), _ptr(), _ptr(), _ptr()
        L.bn_eps, L.bn_momentum, L.relu = 1e-3, 0.1, relu
    return arr


def _sz(sizes):
    return (ctypes.c_int * max(len(sizes), 1))(*sizes)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


def _rows(b, sizes):
    return b * sum(-(-s // 128) * 128 for s in sizes)


def test_envelope_and_workspaces(lib):
    from samplenet_b200 import _lib

    for name in ("snb200_frozen_encoder_bstat_supported", "snb200_frozen_encoder_bstat_workspace_bytes",
                 "snb200_frozen_encoder_bstat_backward_workspace_bytes", "snb200_frozen_encoder_bstat_forward", "snb200_frozen_encoder_bstat_backward"):
        assert name in _lib.exported_symbols() and getattr(lib, name) is not None
    t = _table(AE)
    sup = lambda b, n, sizes, table=t, nconv=5: lib.snb200_frozen_encoder_bstat_supported(b, n, nconv, table, len(sizes), _sz(sizes))
    for b, n, sizes in CASES + [(3, 4096, [4096]), (1, 1, [1])]:
        assert sup(b, n, sizes) == 1
        rows, tiles, np_ = _rows(b, sizes), _rows(b, sizes) // 128, len(sizes)
        fwd = sum(_a256(rows * c * 4) for c in AE[1:]) + _a256(tiles * 2 * 256 * 4) + 2 * _a256(tiles * 128 * 4)
        bwd = 2 * _a256(rows * 256 * 4) + _a256(rows * 3 * 4) + _a256(rows // 64 * 2 * 256 * 4) + _a256(np_ * 2 * 256 * 8)
        assert lib.snb200_frozen_encoder_bstat_workspace_bytes(b, n, 5, t, np_, _sz(sizes)) == fwd
        assert lib.snb200_frozen_encoder_bstat_backward_workspace_bytes(b, n, 5, t, np_, _sz(sizes)) == bwd
    # the progressive step's plan: 204 000 real and 217 600 packed rows
    assert _rows(50, POW2) == 217600 and 50 * sum(POW2) == 204000
    # the edges
    assert sup(2, 2048, [16 * (i + 1) for i in range(16)]) == 1
    assert sup(2, 2048, [16 * (i + 1) for i in range(17)]) == 0            # 17 prefixes
    assert sup(2, 2048, [64, 16]) == 0 and sup(2, 2048, [16, 16]) == 0   # unsorted, repeated
    assert sup(2, 2048, [0, 16]) == 0 and sup(2, 2048, [2049]) == 0      # outside [1, n]
    assert sup(2, 4097, [16]) == 0                                       # n > 4096
    assert sup(1024, 4096, [4096]) == 1 and sup(1025, 4096, [4096]) == 0  # 2^22 packed rows
    assert sup(2, 2048, [16], _table(AE, bn=False)) == 0                 # a layer without BatchNorm
    assert sup(2, 2048, [16], _table(AE, relu=0)) == 0                   # ... or without ReLU
    assert lib.snb200_frozen_encoder_bstat_workspace_bytes(2, 2048, 5, t, 17, _sz(list(range(1, 18)))) == 0


@pytest.mark.parametrize("case", ["prefixes", "unsorted", "n", "rows", "no_bn"])
def test_rejections(lib, case):
    """Outside the envelope both entries return SNB200_EUNSUPPORTED before launching anything (on a machine without a GPU a launch would
    fail with SNB200_ECUDA instead)."""
    b, n, sizes, table = {"prefixes": (2, 2048, list(range(1, 18)), _table(AE)), "unsorted": (2, 2048, [64, 16], _table(AE)),
                          "n": (2, 4097, [16], _table(AE)), "rows": (1025, 4096, [4096], _table(AE)),
                          "no_bn": (2, 2048, [16], _table(AE, bn=False))}[case]
    buf = ctypes.c_void_p(_ptr())
    ws = ctypes.create_string_buffer(16)
    rc = lib.snb200_frozen_encoder_bstat_forward(b, n, buf, 5, table, len(sizes), _sz(sizes), buf, buf, buf, ctypes.addressof(ws), 1 << 40, None)
    assert rc == -4, rc
    rc = lib.snb200_frozen_encoder_bstat_backward(b, n, 5, table, len(sizes), _sz(sizes), buf, buf, buf, ctypes.addressof(ws), 1 << 40, buf, buf,
                                                  ctypes.addressof(ws), 1 << 40, None)
    assert rc == -4, rc
    # a malformed table is SNB200_EINVAL
    bad = _table(AE)
    bad[2].c_in = 7
    assert lib.snb200_frozen_encoder_bstat_forward(2, 64, buf, 5, bad, 1, _sz([64]), buf, buf, buf, ctypes.addressof(ws), 1 << 40, None) == -1


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _tile0(b, sizes):
    t = [0]
    for s in sizes:
        t.append(t[-1] + b * (-(-s // 128)))
    return t


def _group_rows(b, sizes, p, device):
    """Packed rows of group p, cloud-major: (B, s) indices."""
    t0, tps, s = _tile0(b, sizes)[p], -(-sizes[p] // 128), sizes[p]
    base = (t0 + torch.arange(b, device=device) * tps) * 128
    return base[:, None] + torch.arange(s, device=device)[None]


def _zsave(ws, rows):
    out, off = [], 0
    for c in AE[1:]:
        out.append(ws[off:off + rows * c * 4].view(torch.float32).view(rows, c))
        off += _a256(rows * c * 4)
    return out


def _case(b, n, seed):
    net = _randomize(tasknets.PointNetAE(n_pc_points=2048), seed).cuda().eval().requires_grad_(False)
    x = (torch.rand(b, n, 3, generator=torch.Generator().manual_seed(seed + 1)) - 0.5).cuda()
    return net, x


def _kernel_scale_shift(bn, st):
    """The kernels' fp32 scale gamma * (1 / sqrtf(var + eps)) and the float64 sum of the (contracted) shift beta - mean * scale."""
    inv = 1.0 / torch.sqrt(st[1].float() + bn.eps)
    sc = bn.weight.float() * inv
    return sc, bn.bias.double() - st[0].float().double() * sc.double(), inv


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,sizes", CASES)
def test_forward_against_float64(sb, b, n, sizes):
    ops = sb.ops
    net, x = _case(b, n, 21)
    specs = tasknets._conv_specs(net)
    pooled, route, stats, ws = ops.frozen_encoder_bstat_forward(x, specs, sizes)
    st = ops.frozen_encoder_bstat_stats(stats, specs, len(sizes))
    zs = _zsave(ws, _rows(b, sizes))
    worst = {"stat": 0.0, "z": 0.0, "pool": 0.0}
    for p, s in enumerate(sizes):
        rows = _group_rows(b, sizes, p, x.device)
        h = x[:, :s].double()
        for l, (conv, bn) in enumerate(zip(net.convs, net.bns)):
            w, bias = conv.weight.double()[:, :, 0], conv.bias.double()
            z = zs[l][rows].double()                                            # (B, s, C) the kernel's raw output
            ref = h @ w.t() + bias
            worst["z"] = max(worst["z"], ((z - ref).abs() / (h.abs() @ w.abs().t() + bias.abs())).max().item())
            m64, v64 = z.mean(dim=(0, 1)), ((z - z.mean(dim=(0, 1))) ** 2).mean(dim=(0, 1))
            scale = (z * z).mean(dim=(0, 1)) + 1e-30
            worst["stat"] = max(worst["stat"], ((st[l][p, 0] - m64).abs() / scale.sqrt()).max().item(), ((st[l][p, 1] - v64).abs() / scale).max().item())
            sc, sh, _ = _kernel_scale_shift(bn, st[l][p])
            a = torch.relu(z * sc.double() + sh)
            h = a
        # the pool: the route is the first extreme of sign(gamma) * z over the prefix, pooled the activation there
        zl = zs[-1][rows].cpu()
        sgn = torch.where(net.bns[-1].weight.cpu() >= 0, 1.0, -1.0)
        assert torch.equal(route[p].long().cpu(), (zl * sgn).argmax(dim=1)), "route is not the first extreme"
        zr = torch.gather(zs[-1][rows], 1, route[p].long()[:, None, :]).squeeze(1).double()
        sc, sh, _ = _kernel_scale_shift(net.bns[-1], st[-1][p])
        want = torch.relu(zr * sc.double() + sh)
        worst["pool"] = max(worst["pool"], ((pooled[p].double() - want).abs() / (sc.double().abs() * zr.abs() + sh.abs())).max().item())
        # a one-row group: variance 0 up to the rounding of its fp32 square (the partials are fp32 sums of z and z^2)
        if b * s == 1:
            for l in range(len(AE) - 1):
                assert torch.all(st[l][p, 1] <= 2.0 ** -23 * st[l][p, 0] ** 2)
    # end to end against the float64 contract (conditioning, not a kernel bar)
    e2e = ((pooled.double() - restate64(net, x, sizes)).abs().max() / pooled.double().abs().max()).item()
    print("bstat forward", b, n, len(sizes), worst, "end to end", e2e)
    assert worst["stat"] <= STAT_BAR and worst["z"] <= Z_BAR and worst["pool"] <= POOL_BAR, worst


def _pinned_grad64(net, x, sizes, zs, st, route, g):
    """Float64 autograd of sum(g * pooled) through the contract, with the kernel's ReLU masks (decided from its raw outputs and fp32
    scale / shift) and routes pinned.  Returns (grad_x, units whose float64 sign differs from the kernel's mask)."""
    x64 = x.double().clone().requires_grad_(True)
    total, flipped = 0.0, 0
    for p, s in enumerate(sizes):
        rows = _group_rows(x.shape[0], sizes, p, x.device)
        h = x64[:, :s]
        for l, (conv, bn) in enumerate(zip(net.convs, net.bns)):
            z = h @ conv.weight.double()[:, :, 0].t() + conv.bias.double()
            mean = z.mean(dim=(0, 1))
            var = ((z - mean) ** 2).mean(dim=(0, 1))
            a = (z - mean) / torch.sqrt(var + bn.eps) * bn.weight.double() + bn.bias.double()
            sc, sh, _ = _kernel_scale_shift(bn, st[l][p])
            mask = zs[l][rows].double() * sc.double() + sh > 0
            flipped += int(((a.detach() > 0) != mask).sum())
            h = a * mask
        pooled = torch.gather(h, 1, route[p].long()[:, None, :]).squeeze(1)
        total = total + (pooled * g[p].double()).sum()
    return torch.autograd.grad(total, x64)[0], flipped


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,sizes", CASES)
def test_backward_and_determinism(sb, b, n, sizes):
    ops = sb.ops
    net, x = _case(b, n, 31)
    specs = tasknets._conv_specs(net)
    g = torch.randn(len(sizes), b, 128, generator=torch.Generator().manual_seed(5)).cuda()
    outs = []
    for _ in range(2):
        pooled, route, stats, ws = ops.frozen_encoder_bstat_forward(x, specs, sizes)
        gx = ops.frozen_encoder_bstat_backward(x, specs, sizes, pooled, route, stats, ws, g)
        outs.append((pooled, route, stats, gx))
    (p1, r1, s1, g1), (p2, r2, s2, g2) = outs
    assert torch.equal(p1, p2) and torch.equal(r1, r2) and torch.equal(s1, s2) and torch.equal(g1, g2), "not bit-identical on repeat"
    st = ops.frozen_encoder_bstat_stats(s1, specs, len(sizes))
    ref, flipped = _pinned_grad64(net, x, sizes, _zsave(ws, _rows(b, sizes)), st, r1, g)
    err = ((g1.double() - ref).abs().max() / ref.abs().max()).item()
    print("bstat backward", b, n, len(sizes), "grad", err, "flipped units", flipped)
    assert err <= GRAD_BAR, err
    # points past the longest prefix get exactly 0
    assert torch.all(g1[:, sizes[-1]:] == 0)
    # prefix invariance: prefix s of the multi-prefix call equals a one-prefix call on x[:, :s], bit for bit
    for p, s in enumerate(sizes):
        q, rq, sq, _ = ops.frozen_encoder_bstat_forward(x[:, :s].contiguous(), specs, [s])
        assert torch.equal(q[0], p1[p]) and torch.equal(rq[0], r1[p])
        assert all(torch.equal(a[0], b_[p]) for a, b_ in zip(ops.frozen_encoder_bstat_stats(sq, specs, 1), st))


def _tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)


@pytest.mark.gpu
def test_wrapper_and_fallbacks_against_the_module(sb, monkeypatch):
    _tf32_off(monkeypatch)
    net, x = _case(5, 333, 41)
    w = tasknets.FrozenPointNetAE(net)
    with torch.no_grad():
        for sizes in ([1, 7, 64, 333], [64, 7], [7, 7]):   # in the envelope, unsorted, repeated
            got = w.prefixes(x, sizes, batch_stats=True)
            want = torch.stack([net(x[:, :s], batch_stats=True) for s in sizes])
            assert ((got - want).abs().max() / want.abs().max()).item() <= 1e-5
        one = w(x, batch_stats=True)
        assert ((one - net(x, batch_stats=True)).abs().max() / one.abs().max()).item() <= 1e-5
        assert torch.equal(one, w.prefixes(x, [333], batch_stats=True)[0])
        # the default call is the eval-mode path, unchanged
        assert torch.equal(w(x), tasknets.FrozenPointNetAE(net)(x))
        # CudaPointNetAE passes the flag through on the frozen route
        assert torch.equal(tasknets.CudaPointNetAE(net).eval()(x, batch_stats=True), one)


@pytest.mark.gpu
def test_write_set(sb):
    """The entries write only pooled, route, stats, grad_x and their workspaces: the module's parameters and buffers stay bit for bit, and
    guard words around every output stay as they were."""
    ops = sb.ops
    net, x = _case(5, 333, 51)
    sizes = [1, 7, 64, 333]
    before = {k: v.clone() for k, v in net.state_dict().items()}
    specs = tasknets._conv_specs(net)
    pooled, route, stats, ws = ops.frozen_encoder_bstat_forward(x, specs, sizes)
    gx = ops.frozen_encoder_bstat_backward(x, specs, sizes, pooled, route, stats, ws, torch.ones_like(pooled))
    torch.cuda.synchronize()
    assert all(torch.equal(before[k], v) for k, v in net.state_dict().items())
    # outputs inside guarded buffers, through the C entries
    from samplenet_b200 import _lib
    from samplenet_b200.ops import _p, _stream, make_layers

    lib = _lib.lib()
    conv, keep = make_layers(specs)
    G = 4096
    P, B, C = pooled.shape
    buf_p = torch.full((G + P * B * C + G,), 7.0, device="cuda")
    buf_r = torch.full((G + P * B * C + G,), 7, device="cuda", dtype=torch.int32)
    buf_s = torch.full((G + stats.numel() + G,), 7.0, device="cuda", dtype=torch.float64)
    buf_g = torch.full((G + x.numel() + G,), 7.0, device="cuda")
    csz = _sz(sizes)
    wsb = lib.snb200_frozen_encoder_bstat_workspace_bytes(B, x.shape[1], 5, conv, P, csz)
    ws2 = torch.empty(wsb, device="cuda", dtype=torch.uint8)
    _lib.check(lib.snb200_frozen_encoder_bstat_forward(B, x.shape[1], _p(x), 5, conv, P, csz, buf_p[G:].data_ptr(), buf_r[G:].data_ptr(),
                                                       buf_s[G:].data_ptr(), _p(ws2), wsb, _stream()), "forward")
    bwb = lib.snb200_frozen_encoder_bstat_backward_workspace_bytes(B, x.shape[1], 5, conv, P, csz)
    bws = torch.empty(bwb, device="cuda", dtype=torch.uint8)
    gp = torch.ones(P * B * C, device="cuda")
    _lib.check(lib.snb200_frozen_encoder_bstat_backward(B, x.shape[1], 5, conv, P, csz, buf_p[G:].data_ptr(), buf_r[G:].data_ptr(),
                                                        buf_s[G:].data_ptr(), _p(ws2), wsb, _p(gp), buf_g[G:].data_ptr(), _p(bws), bwb,
                                                        _stream()), "backward")
    torch.cuda.synchronize()
    for buf, n_ in ((buf_p, P * B * C), (buf_r, P * B * C), (buf_s, stats.numel()), (buf_g, x.numel())):
        assert torch.all(buf[:G] == 7) and torch.all(buf[G + n_:] == 7)
    assert torch.equal(buf_p[G:G + P * B * C].view_as(pooled), pooled) and torch.equal(buf_g[G:G + x.numel()].view_as(gx), gx)
    assert all(torch.equal(before[k], v) for k, v in net.state_dict().items())
    del keep


def _margin(net, x, sizes):
    """The smallest relative distance, over the prefixes, of a hidden unit's BatchNorm output from its ReLU kink and of a pooled extreme
    from its runner-up, in float64 on the contract: where it is small, rounding alone can flip a mask or a route between two fp32 routes."""
    m = float("inf")
    for s in sizes:
        h = x[:, :s].double()
        for conv, bn in zip(net.convs, net.bns):
            z = h @ conv.weight.double()[:, :, 0].t() + conv.bias.double()
            mean = z.mean(dim=(0, 1))
            zh = (z - mean) / torch.sqrt(((z - mean) ** 2).mean(dim=(0, 1)) + bn.eps)
            a = zh * bn.weight.double() + bn.bias.double()
            m = min(m, (a.abs() / (zh.abs() * bn.weight.double().abs() + bn.bias.double().abs())).min().item())
            h = torch.relu(a)
        if s > 1:
            top = h.topk(2, dim=1).values
            gap = (top[:, 0] - top[:, 1]) / top[:, 0].abs().clamp_min(1e-30)
            m = min(m, gap[top[:, 0] > 0].min().item())
    return m


def _conditioned_ae(proj, sizes, seed0):
    """The autoencoder with the largest _margin on the sampler's projected points over 8 seeds."""
    best = None
    for seed in range(seed0, seed0 + 8):
        net = _randomize(tasknets.PointNetAE(n_pc_points=2048), seed).cuda()
        m = _margin(net, proj, sizes)
        if best is None or m > best[0]:
            best = (m, net)
    print("autoencoder margin", best[0])
    return best[1]


@pytest.mark.gpu
@pytest.mark.parametrize("step", ["rec", "progressive_rec"])
def test_steps_with_batch_statistics(sb, monkeypatch, step):
    """The steps with ae_batch_stats=True through FrozenPointNetAE against the plain module's torch route, the AE's state after steps on
    every route, and the flag taking effect."""
    import test_layers_training_parity as ltp
    from samplenet_b200 import trainers
    from test_sampler_training import _cloud

    _tf32_off(monkeypatch)
    B, N = 50, 2048
    M = 64 if step == "rec" else 2048
    x = _cloud(B, N, "bnc", 31)
    torch.manual_seed(7)
    sampler = sb.ReconstructionSampleNet(M).cuda().train()
    with torch.no_grad():
        _, proj = copy.deepcopy(sampler)(x)
    ae = _conditioned_ae(proj, [M] if step == "rec" else POW2, 61)
    state = {k: v.clone() for k, v in ae.state_dict().items()}

    def run(s, t, flag=True):
        if step == "rec":
            return trainers.ReconstructionStep(s, t, M, ae_batch_stats=flag).loss(x)
        return trainers.ProgressiveReconstructionStep(s, t, ae_batch_stats=flag).loss(x)

    runs = []
    for route in ("frozen", "frozen", "plain", "cuda"):
        s = copy.deepcopy(sampler)
        t = copy.deepcopy(ae).requires_grad_(False)
        wrapped = {"frozen": lambda: tasknets.FrozenPointNetAE(t), "plain": lambda: t, "cuda": lambda: tasknets.CudaPointNetAE(t)}[route]()
        loss, info = run(s, wrapped)
        loss.backward()
        after = t.state_dict()
        assert all(torch.equal(state[k], after[k]) for k in state), route
        runs.append((loss.detach(), {k: p.grad.detach().clone() for k, p in s.named_parameters() if p.grad is not None}))
    (la, ga), (lb, gb), (lt, gt), (lc, gc) = runs
    assert torch.equal(la, lb) and all(torch.equal(ga[k], gb[k]) for k in ga), "not bit-identical run to run"
    # CudaPointNetAE has no prefixes(): the progressive step calls it once per prefix, whose forward is bit for bit the one-pass forward
    # (prefix invariance); the gradients then add over the prefixes in autograd's order instead of the kernel's
    assert torch.equal(la, lc)
    loss_err = abs(float(la) - float(lt)) / abs(float(lt))
    gen = dict(sampler._generator_named_parameters())
    by_name = {id(p): k for k, p in sampler.named_parameters()}
    alias = {by_name[id(p)]: k for k, p in gen.items()}
    scale = ltp._scales(sampler, {alias[k]: gt[k] for k in alias})
    worst = []
    for gg in (ga, gc):
        assert gg.keys() == gt.keys()
        errs = {k: ((gg[k] - gt[k]).abs().max().item() / (scale[alias[k]] if k in alias else max(gt[k].abs().max().item(), 1e-30))) for k in gt}
        worst.append(max(errs.values()))
    # the flag takes effect: the running statistics differ from the batch's, so the eval-mode loss differs
    with torch.no_grad():
        s = copy.deepcopy(sampler)
        le, _ = run(s, tasknets.FrozenPointNetAE(copy.deepcopy(ae).requires_grad_(False)), flag=False)
    print("bstat step", step, "loss", float(la), float(lt), "rel", loss_err, "worst grad", worst, "eval-mode loss", float(le))
    assert loss_err <= STEP_LOSS_BAR and max(worst) <= STEP_GRAD_BAR, (loss_err, worst)
    assert abs(float(le) - float(la)) > 1e-3 * abs(float(la))
    # an epoch of SamplerTrainStep leaves the AE as it was
    t = copy.deepcopy(ae).requires_grad_(False)
    s = copy.deepcopy(sampler)
    inner = (trainers.ReconstructionStep(s, tasknets.FrozenPointNetAE(t), M, ae_batch_stats=True) if step == "rec"
             else trainers.ProgressiveReconstructionStep(s, tasknets.FrozenPointNetAE(t), ae_batch_stats=True))
    trainers.SamplerTrainStep(inner, torch.optim.Adam(s.parameters(), lr=1e-4), batch_size=B).train_one_epoch(x.repeat(2, 1, 1))
    assert all(torch.equal(state[k], v) for k, v in t.state_dict().items())
