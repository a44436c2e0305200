"""Every prefix of PointNet with transform nets in one frozen CUDA pass: FrozenPointNetClsTransforms.prefixes() on the segmented frozen
encoder (snb200_frozen_encoder_seg_*, csrc/frozen_encoder.cu) and the segmented point transform (snb200_point_transform_seg_*,
csrc/point_transform.cu).

CPU: the new symbols are bound, the workspace queries match the carve, ops.Segments builds the table the entries expect, and every new entry
refuses shapes outside its envelope before anything launches.  GPU (H100): prefixes() against the float64 module on each prefix, against
forward() per prefix (bit for bit where the rows are computed the same way), determinism and chunking, the progressive classification step
and evaluation curve against the plain module, the fallbacks, and the new entries' write sets."""
import copy
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from samplenet_b200 import tasknets  # noqa: E402
from test_frozen_cls_transforms import (BACK, FRONT, GUARD, NET_BAR, NET_GRAD_BAR, STEP_BAR, STEP_GUARD, _conditioned_case,  # noqa: E402
                                        _margin64, _ptr, _table, randomized_net)

POW2 = [2, 4, 8, 16, 32, 64, 128, 256, 512, 1024]


def _padded_total(sizes, b):
    return b * sum(-(-s // 128) * 128 for s in sizes)


def _a256(nbytes):
    return -(-nbytes // 256) * 256


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


def test_symbols_and_workspaces(lib):
    from samplenet_b200 import _lib

    for name in ("snb200_frozen_encoder_seg_supported", "snb200_frozen_encoder_seg_workspace_bytes", "snb200_frozen_encoder_seg_backward_workspace_bytes",
                 "snb200_frozen_encoder_seg_forward", "snb200_frozen_encoder_seg_backward", "snb200_point_transform_seg_supported",
                 "snb200_point_transform_seg_workspace_bytes", "snb200_point_transform_seg_forward", "snb200_point_transform_seg_backward"):
        assert name in _lib.exported_symbols() and getattr(lib, name) is not None
    front, back = _table(FRONT), _table(BACK)
    for sizes, b in ((POW2, 32), ([1, 7, 64, 333], 5), (POW2[2:], 64), ([4096] * 1, 64)):
        total, num, ml = _padded_total(sizes, b), len(sizes) * b, max(sizes)
        tiles = total // 128
        assert lib.snb200_frozen_encoder_seg_supported(num, total, ml, 0, 5, front, 1) == 1
        assert lib.snb200_frozen_encoder_seg_supported(num, total, ml, 1, 3, back, -1) == 1
        # forward: a value and a row per (tile, channel); without zsave two ping-pong buffers of the widest hidden layer
        assert lib.snb200_frozen_encoder_seg_workspace_bytes(num, total, ml, 1, 3, back, -1, 1) == _a256(2 * tiles * 1024 * 4)
        assert lib.snb200_frozen_encoder_seg_workspace_bytes(num, total, ml, 0, 5, front, 1, 0) == _a256(2 * tiles * 1024 * 4) + 2 * _a256(total * 128 * 4)
        # backward: one bit per (row, channel)
        assert lib.snb200_frozen_encoder_seg_backward_workspace_bytes(num, total, ml, 1, 3, back, -1) == _a256(total * 32 * 4)
        # the transform's backward: one partial grad_T per 128-row chunk
        for k in (3, 64):
            assert lib.snb200_point_transform_seg_supported(num, total, ml, k) == 1
            assert lib.snb200_point_transform_seg_workspace_bytes(num, total, ml, k) == _a256(tiles * k * k * 4)
    # the envelope: rows, segments per row count, length, layer table
    assert lib.snb200_frozen_encoder_seg_supported(1, 1 << 22, 4096, 1, 3, back, -1) == 1
    assert lib.snb200_frozen_encoder_seg_supported(1, (1 << 22) + 1, 4096, 1, 3, back, -1) == 0
    assert lib.snb200_frozen_encoder_seg_supported(9, 1024, 128, 1, 3, back, -1) == 0      # 9 segments cannot each start a tile of 8
    assert lib.snb200_frozen_encoder_seg_supported(8, 1024, 128, 1, 3, back, -1) == 1
    assert lib.snb200_frozen_encoder_seg_supported(1, 8192, 4097, 1, 3, back, -1) == 0
    assert lib.snb200_frozen_encoder_seg_supported(0, 1024, 128, 1, 3, back, -1) == 0
    assert lib.snb200_frozen_encoder_seg_supported(8, 1024, 128, 0, 3, back, -1) == 0      # a cloud input has 3 channels
    assert lib.snb200_frozen_encoder_seg_supported(8, 1024, 128, 0, 5, front, 4) == 0      # the tap is a hidden layer
    assert lib.snb200_frozen_encoder_seg_workspace_bytes(9, 1024, 128, 1, 3, back, -1, 1) == 0
    assert lib.snb200_point_transform_seg_supported(8, 1024, 128, 65) == 0 and lib.snb200_point_transform_seg_supported(9, 1024, 128, 64) == 0
    assert lib.snb200_point_transform_seg_supported(1, 1 << 22, 4096, 64) == 1 and lib.snb200_point_transform_seg_supported(1, 128, 4097, 3) == 0
    assert lib.snb200_point_transform_seg_workspace_bytes(9, 1024, 128, 64) == 0


def test_segment_table():
    from samplenet_b200 import ops

    s = ops.Segments([1, 7, 128, 129, 333], 3, "cpu")
    assert s.num == 15 and s.max_len == 333 and s.sizes == [1, 7, 128, 129, 333] and s.b == 3
    want_len = [1] * 3 + [7] * 3 + [128] * 3 + [129] * 3 + [333] * 3
    want_pad = [128] * 3 + [128] * 3 + [128] * 3 + [256] * 3 + [384] * 3
    want_off = [sum(want_pad[:j]) for j in range(15)]
    assert s.table.dtype == torch.int32 and tuple(s.table.shape) == (15, 2)
    assert s.table[:, 0].tolist() == want_off and s.table[:, 1].tolist() == want_len
    assert s.total == sum(want_pad) == _padded_total([1, 7, 128, 129, 333], 3)
    assert all(o % ops.SEG_TILE == 0 for o in want_off)
    rows = s.rows()
    assert rows.tolist() == [o + i for o, n in zip(want_off, want_len) for i in range(n)]
    # segment j = p * B + b is prefix p of cloud b
    assert int(s.table[1 * 3 + 2, 1]) == 7 and int(s.table[4 * 3 + 0, 0]) == want_off[12]


def test_rejections_before_any_launch(lib):
    """Outside the envelope SNB200_EUNSUPPORTED (-4), short workspaces SNB200_EWORKSPACE (-2), null or misaligned pointers SNB200_EINVAL (-1);
    the pointers are never dereferenced and the launch counter does not move (this runs without a device)."""
    big = 1 << 40
    z = (ctypes.c_void_p * 8)(*[_ptr() for _ in range(8)])
    front, back = _table(FRONT), _table(BACK)
    before = lib.snb200_launch_count()

    def err():
        return lib.snb200_last_error().decode()

    def efwd(num, total, ml, seg, act, nconv, t, tap, tap_out, wsb=big):
        return lib.snb200_frozen_encoder_seg_forward(num, total, ml, seg, act, _ptr(), nconv, t, _ptr(), _ptr(), tap, tap_out, z, _ptr(), wsb, None)

    def ebwd(num, total, ml, seg, act, nconv, t, tap, grad_tap, wsb=big):
        return lib.snb200_frozen_encoder_seg_backward(num, total, ml, seg, act, _ptr(), nconv, t, _ptr(), _ptr(), z, tap, grad_tap, _ptr(), _ptr(),
                                                      _ptr(), wsb, None)

    assert efwd(9, 1024, 128, _ptr(), 1, 3, back, -1, None) == -4 and "outside the segmented frozen encoder's envelope" in err()
    assert efwd(8, 1024, 4097, _ptr(), 1, 3, back, -1, None) == -4
    assert efwd(8, 1024, 128, _ptr(), 0, 5, front, 4, _ptr()) == -4
    assert efwd(8, 1024, 128, None, 1, 3, back, -1, None) == -1 and "segment table" in err()
    assert efwd(8, 1024, 128, _ptr() + 4, 1, 3, back, -1, None) == -1 and "8-byte aligned" in err()
    assert efwd(8, 1024, 128, _ptr(), 0, 5, front, 1, None) == -1 and "null pointer" in err()
    assert efwd(8, 1024, 128, _ptr(), 1, 3, _table(BACK, running=False), -1, None) == -1
    assert efwd(8, 1024, 128, _ptr(), 1, 3, back, -1, None, wsb=16) == -2
    assert ebwd(9, 1024, 128, _ptr(), 1, 3, back, -1, None) == -4
    assert ebwd(8, 1024, 128, _ptr(), 0, 5, front, 1, None) == -1 and "null pointer" in err()
    assert ebwd(8, 1024, 128, _ptr(), 1, 3, back, -1, None, wsb=16) == -2

    def tfwd(num, total, ml, k, src_b, src_n, sizes):
        cs = (ctypes.c_int * max(len(sizes), 1))(*sizes)
        return lib.snb200_point_transform_seg_forward(num, total, ml, _ptr(), k, src_b, src_n, len(sizes), cs, _ptr(), _ptr(), _ptr(), None)

    def tbwd(num, total, ml, k, src_b, src_n, sizes, wsb=big):
        cs = (ctypes.c_int * max(len(sizes), 1))(*sizes)
        return lib.snb200_point_transform_seg_backward(num, total, ml, _ptr(), k, src_b, src_n, len(sizes), cs, _ptr(), _ptr(), _ptr(), _ptr(), _ptr(),
                                                       _ptr(), wsb, None)

    assert tfwd(8, 1024, 128, 65, 0, 0, []) == -4 and "segmented point transform's envelope" in err()
    assert tfwd(17, 17 * 128, 128, 3, 1, 128, list(range(1, 18))) == -4                      # 17 prefixes
    assert tfwd(65536, 65536 * 128, 1, 3, 65536, 1, [1]) == -4
    assert tfwd(6, 768, 128, 3, 2, 128, [64, 128]) == -1 and "num_seg = num_prefix * src_b" in err()
    assert tfwd(4, 512, 128, 3, 2, 128, [128, 64]) == -1 and "ascending" in err()
    assert tfwd(4, 512, 100, 3, 2, 128, [64, 128]) == -1 and "ascending" in err()              # a size above max_len
    assert tbwd(8, 1024, 128, 64, 0, 0, [], wsb=16) == -2
    assert tbwd(8, 1024, 128, 65, 0, 0, []) == -4
    assert lib.snb200_launch_count() == before


def test_prefixes_only_for_a_module_on_cuda():
    """A wrapper around a module that is not on a CUDA device has no prefixes (the one-pass route is CUDA-only), so the progressive step and
    evaluator keep their per-prefix calls for it; the wrapper's other behaviour is unchanged."""
    net = tasknets.PointNetClsTransforms().eval().requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    assert not hasattr(w, "prefixes") and hasattr(w, "_prefixes")
    with pytest.raises(AttributeError, match="prefixes"):
        w.prefixes


@pytest.mark.gpu
def test_prefixes_refusals_on_cuda(sb):
    net = randomized_net(2).cuda().requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    assert hasattr(w, "prefixes") and hasattr(tasknets.FrozenPointNetCls(tasknets.PointNetCls().cuda().eval().requires_grad_(False)), "prefixes")
    x = torch.zeros(2, 16, 3)
    with pytest.raises(RuntimeError, match="CUDA-only"):       # CPU tensors: no fallback
        w.prefixes(x, [4, 16])
    net.train()
    with pytest.raises(ValueError, match="training mode"):
        w.prefixes(x.cuda(), [4, 16])
    net.eval()
    net.fc3.weight.requires_grad_(True)
    with pytest.raises(ValueError, match="gives no parameter gradients"):
        w.prefixes(x.cuda(), [4, 16])


@pytest.mark.gpu
def test_wrapper_fallback_rules(sb):
    """Which calls take the segmented path (decided on the host, before anything launches)."""
    w = tasknets.FrozenPointNetClsTransforms(randomized_net(2).cuda().requires_grad_(False))
    ok = lambda b, n, s: w._prefixes_supported(b, n, s)
    assert ok(32, 1024, POW2) and ok(5, 333, [1, 7, 64, 333]) and ok(70, 1024, POW2[2:]) and ok(3, 4096, [4096])
    assert not ok(32, 1024, [4, 2, 8])                       # not ascending
    assert not ok(32, 1024, [2, 2, 8])                       # a repeat
    assert not ok(4, 1024, list(range(1, 18)))                # more than 16 sizes
    assert not ok(4, 100, [50, 101]) and not ok(4, 100, [0, 50])
    assert not ok(2, 4097, [8, 4097])                        # N above the frozen encoder's 4096
    assert not ok(2, 1024, [])


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


@pytest.fixture()
def _tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


def _prefix_case(b, n, sizes, guard, seed0=10, tries=30):
    """The first (net, x) from seed0 whose float64 forward on every prefix has a _margin64 above guard, or the one with the largest margin."""
    best = None
    for seed in range(seed0, seed0 + tries):
        net = randomized_net(seed).cuda()
        x = 0.5 * torch.randn(b, n, 3, generator=torch.Generator().manual_seed(500 + seed)).cuda()
        n64, x64 = copy.deepcopy(net).double(), x.double()
        m = min(_margin64(n64, x64[:, :s]) for s in sizes)
        if best is None or m > best[0]:
            best = (m, net, x)
        if m > guard:
            break
    return best


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,sizes", [(32, 1024, POW2), (5, 333, [1, 7, 64, 333]), (70, 1024, POW2[2:])], ids=["32x1024", "5x333", "70x1024"])
def test_prefixes_against_float64(sb, record_property, _tf32_off, b, n, sizes):
    large = b * n > 40000
    margin, net, x = _prefix_case(b, n, sizes, STEP_GUARD if large else GUARD)
    net.requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    label = torch.randint(0, 40, (b,), generator=torch.Generator().manual_seed(b)).cuda()
    xa = x.clone().requires_grad_(True)
    logits, eps = w.prefixes(xa, sizes, return_end_points=True)
    assert logits.shape == (len(sizes), b, 40) and len(eps) == len(sizes)
    loss = sum(w.get_loss(logits[p], label, eps[p]) for p in range(len(sizes)))
    gx, = torch.autograd.grad(loss, xa)
    net64 = copy.deepcopy(net).double()
    x64 = x.double().requires_grad_(True)
    loss64, e = 0.0, {"logits": 0.0, "transform": 0.0, "GFV": 0.0, "loss": 0.0}
    for p, s in enumerate(sizes):
        l64, ep64 = net64(x64[:, :s])
        lp64 = net64.get_loss(l64, label, ep64)
        loss64 = loss64 + lp64
        e["logits"] = max(e["logits"], float((logits[p].double() - l64).abs().max() / l64.abs().max()))
        e["transform"] = max(e["transform"], float((eps[p]["transform"].double() - ep64["transform"]).abs().max() / ep64["transform"].abs().max()))
        e["GFV"] = max(e["GFV"], float((eps[p]["GFV"].double() - ep64["GFV"]).abs().max() / ep64["GFV"].abs().max()))
        e["loss"] = max(e["loss"], abs(float(w.get_loss(logits[p], label, eps[p])) - float(lp64)) / abs(float(lp64)))
        assert eps[p]["critical_set_idx"].dtype == torch.int64 and eps[p]["critical_set_idx"].shape == (b, 1024)
        assert int(eps[p]["critical_set_idx"].max()) < s
    g64, = torch.autograd.grad(loss64, x64)
    e["grad"] = float((gx.double() - g64).abs().max() / g64.abs().max())
    # the same gradient through forward() prefix by prefix: a prefix of one point makes the transforms' gradients steep, so the bar is also
    # the per-prefix route's own error on this instance
    xf = x.clone().requires_grad_(True)
    lf = 0.0
    for s in sizes:
        lg, ep = w(xf[:, :s])
        lf = lf + w.get_loss(lg, label, ep)
    gf, = torch.autograd.grad(lf, xf)
    e["grad_forward"] = float((gf.double() - g64).abs().max() / g64.abs().max())
    for k, v in e.items():
        record_property("prefixes_%s_err" % k, v)
    record_property("margin", margin)
    assert e["logits"] <= NET_BAR and e["transform"] <= NET_BAR and e["GFV"] <= NET_BAR and e["loss"] <= NET_BAR, e
    assert e["grad"] <= max(STEP_BAR if margin <= GUARD else NET_GRAD_BAR, 2 * e["grad_forward"]), (e, margin)
    # points beyond the largest prefix get exactly 0
    if sizes[-1] < n:
        assert float(gx[:, sizes[-1]:].abs().max()) == 0.0


@pytest.mark.gpu
def test_prefixes_against_forward(sb):
    """prefixes() against forward(x[:, :s]) prefix by prefix.  Bit for bit where each row is computed the same way: T-Net 1's pooled features
    (one frozen-encoder pass over every prefix, per-row tensor-core layers), and, given the same T, the segmented point transform's rows, the
    segmented encoder's pools, routes and tapped rows and both gradients (per-point transform chains, the same per-row layer kernels, the
    same chunk sums).  Not bit for bit: T1, T2 and the logits, because the frozen MLP's summation depends on its row count (P * B rows in
    64-row calls against B rows per prefix), and everything downstream of T1; those agree within fp32 rounding."""
    from samplenet_b200 import ops

    net = randomized_net(11).cuda().requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    b, n, sizes = 6, 300, [1, 5, 128, 129, 300]
    x = 0.5 * torch.randn(b, n, 3, generator=torch.Generator().manual_seed(3)).cuda()
    with torch.no_grad():
        logits, eps = w.prefixes(x, sizes, return_end_points=True)
        for p, s in enumerate(sizes):
            lf, ef = w(x[:, :s].contiguous())
            for got, want in ((logits[p], lf), (eps[p]["transform"], ef["transform"]), (eps[p]["GFV"], ef["GFV"])):
                assert float((got - want).abs().max()) <= 2e-5 * float(want.abs().max()), (p, s)
    # the kernels, bit for bit on the same inputs
    P = w._plan()
    segs = ops.Segments(sizes, b, x.device)
    g = torch.Generator(device="cuda").manual_seed(5)
    T1 = torch.eye(3, device="cuda") + 0.1 * torch.randn(segs.num, 3, 3, device="cuda", generator=g)
    T2 = torch.eye(64, device="cuda") + 0.05 * torch.randn(segs.num, 64, 64, device="cuda", generator=g)
    pooled1, _, _ = ops.frozen_encoder_forward(x, P["t1_conv"], sizes)
    x1 = ops.point_transform_seg_forward(x, T1, segs, True)
    pad = torch.ones(segs.total, dtype=torch.bool, device="cuda")
    pad[segs.rows()] = False
    assert float(x1[pad].abs().max()) == 0.0
    pooled2, route2, h, zs2 = ops.frozen_encoder_seg_forward(x1, P["front"], segs, False, 1)
    h2 = ops.point_transform_seg_forward(h, T2, segs, False)
    pooled3, route3, _, zs3 = ops.frozen_encoder_seg_forward(h2, P["back"], segs, True, -1)
    gp2, gp3 = torch.randn_like(pooled2), torch.randn_like(pooled3)
    gh = torch.randn(segs.total, 64, device="cuda", generator=g)
    gin3 = ops.frozen_encoder_seg_backward(h2, P["back"], segs, pooled3, route3, zs3, gp3, True)
    assert float(gin3[pad].abs().max()) == 0.0
    gh2, gT2 = ops.point_transform_seg_backward(h, T2, segs, False, gin3)
    gx1 = ops.frozen_encoder_seg_backward(x1, P["front"], segs, pooled2, route2, zs2, gp2, False, 1, gh)
    assert float(gx1[pad].abs().max()) == 0.0
    gx, gT1 = ops.point_transform_seg_backward(x, T1, segs, True, gx1)
    gx_want = torch.zeros_like(x)
    for p, s in enumerate(sizes):
        pf, _, _ = ops.frozen_encoder_forward(x[:, :s].contiguous(), P["t1_conv"], [s])
        assert torch.equal(pooled1[p], pf[0])
        js = slice(p * b, (p + 1) * b)
        rows = torch.stack([torch.arange(int(segs.table[j, 0]), int(segs.table[j, 0]) + s, device="cuda") for j in range(p * b, (p + 1) * b)])
        xs = x[:, :s].contiguous()
        x1p = ops.point_transform_forward(xs, T1[js].contiguous())
        assert torch.equal(x1[rows], x1p)
        q2, r2, hp, z2 = ops.frozen_encoder_ex_forward(x1p, P["front"], [s], False, 1)
        assert torch.equal(pooled2[js], q2[0]) and torch.equal(route2[js], r2[0]) and torch.equal(h[rows], hp)
        h2p = ops.point_transform_forward(hp, T2[js].contiguous())
        assert torch.equal(h2[rows], h2p)
        q3, r3, _, z3 = ops.frozen_encoder_ex_forward(h2p, P["back"], [s], True, -1)
        assert torch.equal(pooled3[js], q3[0]) and torch.equal(route3[js], r3[0])
        gi3 = ops.frozen_encoder_ex_backward(h2p, P["back"], [s], q3, r3, z3, gp3[js][None].contiguous(), True)
        assert torch.equal(gin3[rows], gi3)
        ghp, gTp = ops.point_transform_backward(hp, T2[js].contiguous(), gi3)
        assert torch.equal(gh2[rows], ghp) and torch.equal(gT2[js], gTp)
        gxp = ops.frozen_encoder_ex_backward(x1p, P["front"], [s], q2, r2, z2, gp2[js][None].contiguous(), False, 1, gh[rows].contiguous())
        assert torch.equal(gx1[rows], gxp)
        gxs, gT1p = ops.point_transform_backward(xs, T1[js].contiguous(), gxp)
        assert torch.equal(gT1[js], gT1p)
        gx_want[:, :s] += gxs                                                 # the prefixes of a point in ascending order
    assert torch.equal(gx, gx_want)


@pytest.mark.gpu
def test_determinism_and_chunks(sb):
    net = randomized_net(12).cuda().requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    x = 0.5 * torch.randn(70, 512, 3, generator=torch.Generator().manual_seed(4)).cuda()
    sizes = [8, 64, 100, 512]

    def run(xx):
        xa = xx.clone().requires_grad_(True)
        logits, eps = w.prefixes(xa, sizes, return_end_points=True)
        loss = sum((logits[p] ** 2).sum() + (eps[p]["transform"] ** 2).sum() for p in range(len(sizes)))
        gx, = torch.autograd.grad(loss, xa)
        return logits.detach(), torch.stack([e["transform"] for e in eps]).detach(), gx

    a, b_ = run(x), run(x)
    assert all(torch.equal(u, v) for u, v in zip(a, b_)), "prefixes() not bit-identical run to run"
    lo, hi = run(x[:64].contiguous()), run(x[64:].contiguous())
    assert torch.equal(torch.cat([lo[0], hi[0]], dim=1), a[0]) and torch.equal(torch.cat([lo[1], hi[1]], dim=1), a[1])
    assert torch.equal(torch.cat([lo[2], hi[2]]), a[2])


@pytest.mark.gpu
def test_fallbacks_equal_forward_per_prefix(sb):
    net = randomized_net(13).cuda().requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    x = 0.5 * torch.randn(3, 256, 3, generator=torch.Generator().manual_seed(6)).cuda()
    big = 0.5 * torch.randn(2, 4100, 3, generator=torch.Generator().manual_seed(7)).cuda()
    with torch.no_grad():
        for xx, sizes in ((x, [64, 8, 256]), (x, list(range(1, 18))), (big, [16, 4100])):
            logits, eps = w.prefixes(xx, sizes, return_end_points=True)
            for p, s in enumerate(sizes):
                lf, ef = w(xx[:, :s].contiguous())
                assert torch.equal(logits[p], lf) and torch.equal(eps[p]["transform"], ef["transform"])
            assert torch.equal(w.prefixes(xx, sizes), logits)


@pytest.mark.gpu
def test_progressive_step_against_the_plain_module(sb, record_property, _tf32_off):
    from samplenet_b200 import trainers
    from test_sampler_training import _cloud

    B, N = 32, 1024
    x = _cloud(B, N, "bnc", 31)
    torch.manual_seed(7)
    sampler = sb.ClassificationSampleNet(N, group_size=7).cuda().train()
    with torch.no_grad():
        _, proj = copy.deepcopy(sampler)(x)
    best = None
    for seed in range(40, 60):
        net = randomized_net(seed).cuda()
        n64 = copy.deepcopy(net).double()
        m = min(_margin64(n64, proj[:, :s].double()) for s in POW2)
        if best is None or m > best[0]:
            best = (m, net)
        if m > STEP_GUARD:
            break
    record_property("margin", best[0])
    y = torch.randint(0, 40, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    runs = []
    for frozen in (True, False):
        s = copy.deepcopy(sampler)
        t = copy.deepcopy(best[1]).requires_grad_(False)
        t = tasknets.FrozenPointNetClsTransforms(t) if frozen else t
        st = trainers.ProgressiveClassificationStep(s, t, 2, N)
        assert st.sizes == POW2
        loss, info = st.loss(x, y)
        loss.backward()
        runs.append((loss.detach(), {k: p.grad.detach().clone() for k, p in s.named_parameters() if p.grad is not None}))
    (la, ga), (lt, gt) = runs
    # the loss holds every prefix's transform regulariser: without them it would be smaller by their sum
    with torch.no_grad():
        _, proj2 = copy.deepcopy(sampler)(x)
        reg = sum(0.001 * 0.5 * float(((t2 := best[1](proj2[:, :s])[1]["transform"]) @ t2.transpose(1, 2) - torch.eye(64, device="cuda")).pow(2).sum())
                  for s in POW2)
    assert reg > 1e3 * abs(float(la) - float(lt))
    e_loss = abs(float(la) - float(lt)) / abs(float(lt))
    assert ga.keys() == gt.keys() and len(ga) > 10
    top = max(float(g.abs().max()) for g in gt.values())
    e_grad = max(float((ga[k] - gt[k]).abs().max()) / max(float(gt[k].abs().max()), 1e-3 * top) for k in gt)
    record_property("step_loss_err", e_loss); record_property("step_grad_err", e_grad)
    assert e_loss <= 1e-5 and e_grad <= STEP_BAR, (e_loss, e_grad, best[0])


@pytest.mark.gpu
def test_evaluation_curve_against_the_plain_module(sb, _tf32_off):
    from samplenet_b200 import evaluation

    margin, net, x = _conditioned_case(16, 256, GUARD, seed0=20, tries=20)
    net.requires_grad_(False)
    sizes = [1, 2, 4, 8, 16, 32, 64, 128, 256]
    labels = torch.randint(0, 40, (16,), generator=torch.Generator().manual_seed(2)).cuda()
    ev_p = evaluation.ProgressiveClassificationEvaluator(None, net)
    ev_w = evaluation.ProgressiveClassificationEvaluator(None, tasknets.FrozenPointNetClsTransforms(net))
    with torch.no_grad():
        lp, lw = ev_p.logits(x, sizes), ev_w.logits(x, sizes)
    assert float((lw - lp).abs().max()) <= 1e-4 * float(lp.abs().max())
    # records whose float32 prediction is not within the two paths' rounding of a tie
    top2 = lp.topk(2, dim=2)[0]
    clear = (top2[..., 0] - top2[..., 1]) > 1e-4 * float(lp.abs().max())
    assert torch.equal(lw.argmax(2)[clear], lp.argmax(2)[clear]) and float(clear.double().mean()) > 0.95
    got_w, got_p = ev_w.evaluate(x, labels, sizes, ordered=x), ev_p.evaluate(x, labels, sizes, ordered=x)
    if bool(clear.all()):
        assert (got_w["accuracy"] == got_p["accuracy"]).all(), (got_w["accuracy"], got_p["accuracy"])


# ------------------------------------------------------------------------------------------------------------------ GPU: write sets
@pytest.mark.gpu
def test_new_entries_write_only_their_buffers(sb):
    from samplenet_b200 import _lib, ops
    from test_write_sets import Arena, assert_clean, run_checked

    lib = _lib.lib()
    arena = Arena(nbytes=192 << 20)
    net = randomized_net(14).cuda().requires_grad_(False)
    P = tasknets.FrozenPointNetClsTransforms(net)._plan()
    b, n, sizes = 3, 200, [5, 130, 200]
    segs = ops.Segments(sizes, b, "cuda")
    tot, num, ml = segs.total, segs.num, segs.max_len
    g = torch.Generator(device="cuda").manual_seed(1)
    rnd = lambda *shape: torch.randn(*shape, device="cuda", generator=g)
    seg = arena.carve("seg", (num, 2), torch.int32, fill=segs.table)
    sz = (ctypes.c_int * len(sizes))(*sizes)
    x = arena.carve("x", (b, n, 3), fill=0.5 * rnd(b, n, 3))
    T1 = arena.carve("T1", (num, 3, 3), fill=torch.eye(3, device="cuda") + 0.1 * rnd(num, 3, 3))
    x1 = arena.carve("x1", (tot, 3))
    rep = run_checked(arena, "transform prefix forward", lambda: _lib.check(lib.snb200_point_transform_seg_forward(
        num, tot, ml, seg.data_ptr(), 3, b, n, len(sizes), sz, x.data_ptr(), T1.data_ptr(), x1.data_ptr(), None), "fwd"), full=[x1])
    front, keep_f = ops.make_layers(P["front"])
    c = [l.c_out for l in front]
    zs = [arena.carve("z%d" % l, (tot, c[l])) for l in range(4)]
    zp = (ctypes.c_void_p * 4)(*[z.data_ptr() for z in zs])
    pooled, route = arena.carve("pooled", (num, 1024)), arena.carve("route", (num, 1024), torch.int32)
    h = arena.carve("h", (tot, 64))
    wsb = int(lib.snb200_frozen_encoder_seg_workspace_bytes(num, tot, ml, 0, 5, front, 1, 1))
    ws = arena.carve("enc ws", wsb, torch.uint8)
    rep += run_checked(arena, "encoder forward", lambda: _lib.check(lib.snb200_frozen_encoder_seg_forward(
        num, tot, ml, seg.data_ptr(), 0, x1.data_ptr(), 5, front, pooled.data_ptr(), route.data_ptr(), 1, h.data_ptr(), zp, ws.data_ptr(), wsb,
        None), "efwd"), writes=[ws], full=[pooled, route, h] + zs)
    gp, gh = arena.carve("gp", (num, 1024), fill=rnd(num, 1024)), arena.carve("gh", (tot, 64), fill=rnd(tot, 64))
    gx1 = arena.carve("gx1", (tot, 3))
    bwb = int(lib.snb200_frozen_encoder_seg_backward_workspace_bytes(num, tot, ml, 0, 5, front, 1))
    bws = arena.carve("enc bws", bwb, torch.uint8)
    rep += run_checked(arena, "encoder backward", lambda: _lib.check(lib.snb200_frozen_encoder_seg_backward(
        num, tot, ml, seg.data_ptr(), 0, x1.data_ptr(), 5, front, pooled.data_ptr(), route.data_ptr(), zp, 1, gh.data_ptr(), gp.data_ptr(),
        gx1.data_ptr(), bws.data_ptr(), bwb, None), "ebwd"), writes=[bws], full=[gx1])
    T2 = arena.carve("T2", (num, 64, 64), fill=torch.eye(64, device="cuda") + 0.05 * rnd(num, 64, 64))
    h2 = arena.carve("h2", (tot, 64))
    rep += run_checked(arena, "transform packed forward", lambda: _lib.check(lib.snb200_point_transform_seg_forward(
        num, tot, ml, seg.data_ptr(), 64, 0, 0, 0, sz, h.data_ptr(), T2.data_ptr(), h2.data_ptr(), None), "pfwd"), full=[h2])
    gh2 = arena.carve("gh2", (tot, 64), fill=rnd(tot, 64))
    gin, gT2 = arena.carve("gin", (tot, 64)), arena.carve("gT2", (num, 64, 64))
    twb = int(lib.snb200_point_transform_seg_workspace_bytes(num, tot, ml, 64))
    tws = arena.carve("pt ws", twb, torch.uint8)
    rep += run_checked(arena, "transform packed backward", lambda: _lib.check(lib.snb200_point_transform_seg_backward(
        num, tot, ml, seg.data_ptr(), 64, 0, 0, 0, sz, h.data_ptr(), T2.data_ptr(), gh2.data_ptr(), gin.data_ptr(), gT2.data_ptr(), tws.data_ptr(),
        twb, None), "pbwd"), writes=[tws], full=[gin, gT2])
    gx, gT1 = arena.carve("gx", (b, n, 3)), arena.carve("gT1", (num, 3, 3))
    twb3 = int(lib.snb200_point_transform_seg_workspace_bytes(num, tot, ml, 3))
    tws3 = arena.carve("pt ws 3", twb3, torch.uint8)
    rep += run_checked(arena, "transform prefix backward", lambda: _lib.check(lib.snb200_point_transform_seg_backward(
        num, tot, ml, seg.data_ptr(), 3, b, n, len(sizes), sz, x.data_ptr(), T1.data_ptr(), gx1.data_ptr(), gx.data_ptr(), gT1.data_ptr(),
        tws3.data_ptr(), twb3, None), "xbwd"), writes=[tws3], full=[gx, gT1])
    del keep_f
    assert_clean(rep)
