"""The frozen encoder's forward over many prefixes (csrc/frozen_encoder.cu, snb200_frozen_encoder_curve_*, ops.frozen_encoder_curve_forward):
every sample size of a progressive curve from one pass of the conv stack, and the evaluator route that takes it.

CPU: the C ABI's envelope, workspace sizes and rejections; the Python layer's refusals.  GPU (H100): pooled and route bit for bit what
snb200_frozen_encoder_forward gives 16 sizes at a time over the whole envelope's edges (negative BatchNorm scales and duplicated points,
so exact ties); one case against float64; routes in [0, n) on NaN and Inf clouds; the entry's write set; ProgressiveClassificationEvaluator
on FrozenPointNetCls with every size in one call against the 16-size route, and FrozenPointNetClsTransforms unchanged."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import test_frozen_tasknets as tft  # noqa: E402
import test_write_sets as tws  # noqa: E402
from samplenet_b200 import tasknets  # noqa: E402

EINVAL, EWORKSPACE, EUNSUPPORTED = -1, -2, -4
LOGIT_TOL = 1e-5      # logits of the two evaluator routes: |difference| / max |logit| (the FC head's GEMMs see P * B rows against 16 * B)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


def _sizes(sizes):
    sizes = list(sizes)
    return len(sizes), (ctypes.c_int * max(len(sizes), 1))(*sizes)


def _supported(lib, b, n, table, sizes, nconv=5):
    return lib.snb200_frozen_encoder_curve_supported(b, n, nconv, table, *_sizes(sizes))


def _ws(lib, b, n, table, sizes, nconv=5):
    return lib.snb200_frozen_encoder_curve_workspace_bytes(b, n, nconv, table, *_sizes(sizes))


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_curve_envelope(lib):
    for w in (tft.CLS_W, tft.AE_W):
        t = tft._table(w)
        for b, n, sizes in ((1, 1, [1]), (64, 4096, [1]), (64, 4096, range(1, 4097)), (32, 1024, range(8, 1025)), (5, 333, [333]),
                            (1, 129, [1, 128, 129])):
            assert _supported(lib, b, n, t, sizes) == 1, (w, b, n)
        for b, n, sizes in ((32, 1024, []), (32, 1024, [8, 4]), (32, 1024, [8, 8]), (32, 1024, [1, 2, 2, 3]), (32, 1024, [0, 8]),
                            (32, 1024, [8, 1025]), (32, 1024, [-1]), (65, 1024, [8]), (0, 1024, [8]), (32, 4097, [8]), (32, 0, [1])):
            assert _supported(lib, b, n, t, sizes) == 0, (w, b, n, list(sizes)[:4])
        assert _supported(lib, 4, 16, t, range(1, 18)) == 0        # more sizes than points: one of them repeats or lies outside [1, n]
        assert lib.snb200_frozen_encoder_curve_supported(4, 16, 5, t, 1, None) == 0
    for w in ([3, 64, 64, 64, 128, 1032], [3, 64, 128, 128, 264, 128], [3, 64, 60, 64, 128, 1024], [4, 64, 64, 64, 128, 1024], [3, 1024]):
        assert _supported(lib, 32, 1024, tft._table(w), range(1, 1025), nconv=len(w) - 1) == 0, w
    assert _supported(lib, 32, 1024, tft._table([3, 64, 64, 64, 128, 8]), range(1, 1025)) == 1
    # the 16-prefix entry keeps its envelope
    assert lib.snb200_frozen_encoder_supported(32, 1024, 5, tft._table(tft.CLS_W), 17) == 0


def test_curve_workspace_sizes(lib):
    cls, ae = tft._table(tft.CLS_W), tft._table(tft.AE_W)

    def a256(x):
        return (x + 255) // 256 * 256

    # tile records (value + index per cloud, tile and channel), two buffers of the widest hidden layer, then the sizes and the tiles + 1
    # first-prefix entries; no boundary records (they go to pooled / route)
    assert _ws(lib, 32, 1024, cls, range(1, 1025)) == 32 * 8 * 1024 * 8 + 2 * 32 * 1024 * 128 * 4 + a256((1024 + 9) * 4)
    assert _ws(lib, 32, 1024, cls, range(8, 1025)) == 32 * 8 * 1024 * 8 + 2 * 32 * 1024 * 128 * 4 + a256((1017 + 9) * 4)
    assert _ws(lib, 50, 2048, ae, range(1, 2049)) == 50 * 16 * 128 * 8 + 2 * a256(50 * 2048 * 256 * 4) + a256((2048 + 17) * 4)
    assert _ws(lib, 5, 333, ae, [333]) == a256(5 * 3 * 128 * 8) + 2 * a256(5 * 333 * 256 * 4) + a256((1 + 4) * 4)
    assert _ws(lib, 64, 4096, cls, range(1, 4097)) == 64 * 32 * 1024 * 8 + 2 * 64 * 4096 * 128 * 4 + a256((4096 + 33) * 4)
    assert _ws(lib, 65, 1024, cls, range(1, 1025)) == 0
    assert _ws(lib, 32, 1024, cls, [8, 8]) == 0
    assert _ws(lib, 32, 4097, cls, [8]) == 0
    assert _ws(lib, 32, 1024, tft._table([3, 64, 64, 64, 128, 1032]), [8]) == 0


def test_curve_rejections(lib):
    """Every malformed call returns its error code with its message before anything launches (the pointers are never dereferenced)."""
    who = "frozen_encoder_curve_forward: "
    cls = tft._table(tft.CLS_W)
    big = 1 << 40
    cases = [
        ((32, 1024, cls, [], big), EINVAL, who + "1..n=1024 sizes expected"),
        ((4, 16, cls, range(1, 18), big), EINVAL, who + "1..n=16 sizes expected"),
        ((32, 1024, cls, [8, 8, 16], big), EINVAL, who + "sizes must be ascending and distinct"),
        ((32, 1024, cls, [16, 8], big), EINVAL, who + "sizes must be ascending and distinct"),
        ((32, 1024, cls, [0, 8], big), EINVAL, who + "sizes must be ascending and distinct"),
        ((32, 1024, cls, [8, 1025], big), EINVAL, who + "sizes must be ascending and distinct"),
        ((32, 1024, tft._table(tft.CLS_W, running=False), [8], big), EINVAL, who + "eval mode needs running statistics"),
        ((32, 1024, tft._table([3, 64, 64, 64, 128, 1032]), [8], big), EUNSUPPORTED, who + "shape outside the frozen encoder's envelope"),
        ((65, 1024, cls, [8], big), EUNSUPPORTED, who + "shape outside the frozen encoder's envelope"),
        ((32, 4097, cls, [8], big), EUNSUPPORTED, who + "shape outside the frozen encoder's envelope"),
        ((32, 1024, cls, range(1, 1025), _ws(lib, 32, 1024, cls, range(1, 1025)) - 1), EWORKSPACE, who + "workspace"),
    ]
    for (b, n, table, sizes, wsb), rc_want, msg in cases:
        rc = lib.snb200_frozen_encoder_curve_forward(b, n, tft._ptr(), 5, table, *_sizes(sizes), tft._ptr(), tft._ptr(), tft._ptr(), wsb, None)
        err = lib.snb200_last_error().decode()
        assert rc == rc_want and err.startswith(msg), (list(sizes)[:4], rc, err)


def test_python_refusals():
    from samplenet_b200 import ops

    net = tasknets.PointNetCls().requires_grad_(False).eval()
    specs = tasknets._conv_specs(net)
    x = torch.zeros(2, 40, 3)
    for bad in ([], [8, 4], [8, 8], [0, 8], [8, 41]):
        with pytest.raises(ValueError, match="ascending, distinct"):
            ops.frozen_encoder_curve_forward(x, specs, bad)
    with pytest.raises(ValueError):
        ops.frozen_encoder_curve_forward(torch.zeros(2, 40), specs, [8])
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.frozen_encoder_curve_forward(x, specs, range(1, 41))
    with pytest.raises(RuntimeError, match="CUDA-only"):     # more than 16 sizes without a gradient: the curve entry, CUDA-only
        with torch.no_grad():
            tasknets.FrozenPointNetCls(net).prefixes(x, range(1, 41))
    assert tasknets.FrozenPointNetCls.ONE_PASS_PREFIXES and not getattr(tasknets.FrozenPointNetClsTransforms, "ONE_PASS_PREFIXES", False)


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _net(kind, seed):
    """A frozen PointNetCls (C = 1024) or PointNetAE (C = 128) on the GPU with BatchNorm away from the identity, a quarter of every layer's
    scales < 0."""
    net = tasknets.PointNetCls() if kind == "cls" else tasknets.PointNetAE(n_pc_points=2048, bneck_size=128)
    return tft._randomize(net, seed).cuda().eval().requires_grad_(False)


def _cloud(b, n, seed):
    """b clouds of n points; the first four points copied to later indices in the same tile and in later tiles (exact ties at extremes)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, n, 3, generator=g) * 0.5
    for i in range(min(4, n)):
        x[:, i] *= 4.0
        for j in (i + 5, i + 131, i + 263):
            if j < n:
                x[:, j] = x[:, i]
    return x.cuda()


def _by_16(sb, x, specs, sizes):
    """snb200_frozen_encoder_forward 16 sizes at a time (the reference route), forward only."""
    parts = [sb.ops.frozen_encoder_forward(x, specs, sizes[i:i + 16], keep_activations=False)[:2] for i in range(0, len(sizes), 16)]
    return torch.cat([p for p, _ in parts]), torch.cat([r for _, r in parts])


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, 5, 32, 64])
@pytest.mark.parametrize("n", [1, 127, 128, 129, 333, 1024, 2048, 4096])
@pytest.mark.parametrize("kind", ["cls", "ae"])
def test_curve_bit_identical_to_16_at_a_time(sb, kind, n, b):
    net = _net(kind, 7 + n + b)
    specs = tasknets._conv_specs(net)
    x = _cloud(b, n, n * 100 + b)
    C = net.bns[-1].num_features
    assert (net.bns[-1].weight < 0).any()
    for sizes in (list(range(1, n + 1)), list(range(8, n + 1))):
        if not sizes:
            continue
        pooled, route = sb.ops.frozen_encoder_curve_forward(x, specs, sizes)
        assert pooled.shape == (len(sizes), b, C) and route.shape == (len(sizes), b, C) and route.dtype == torch.int32
        p16, r16 = _by_16(sb, x, specs, sizes)
        assert torch.equal(_bits(pooled), _bits(p16)), (kind, n, b, sizes[0])
        assert torch.equal(route, r16), (kind, n, b, sizes[0])
        lens = torch.tensor(sizes, device="cuda", dtype=torch.int32)[:, None, None]
        assert (route >= 0).all() and (route < lens).all()
        del pooled, route, p16, r16


@pytest.mark.gpu
def test_curve_ties_go_to_the_first_index(sb):
    net, n = _net("cls", 3), 333
    x = _cloud(5, n, 4)
    sizes = list(range(1, n + 1))
    _, route = sb.ops.frozen_encoder_curve_forward(x, tasknets._conv_specs(net), sizes)
    ties = 0
    for i in range(4):
        for p, s in enumerate(sizes):
            ties += int((route[p] == i).sum()) if s > i + 5 else 0
            for j in (i + 5, i + 131, i + 263):
                assert not (route[p] == j).any(), "a tied copy won over the first index"
    assert ties > 0, "no tie at an extreme"


@pytest.mark.gpu
def test_curve_against_float64(sb):
    """Every size of 5 clouds of 333 points against the float64 restatement, with the frozen encoder's bars (the hidden layers checked on the
    same kernels' saved outputs)."""
    net, x, _, dead = tft.make_case("cls", 5, 333, 11, sizes=[333])
    specs = tasknets._conv_specs(net)
    sizes = list(range(1, 334))
    pooled, route = sb.ops.frozen_encoder_curve_forward(x, specs, sizes)
    _, _, zs = sb.ops.frozen_encoder_forward(x, specs, [333])
    rep = tft._check_forward(net, x, sizes, pooled, route, zs, dead)
    print("curve forward", rep)
    assert max(v for k, v in rep.items() if k.startswith("z")) <= tft.Z_BAR, rep
    assert rep["pooled"] <= tft.POOL_BAR, rep


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["cls", "ae"])
def test_curve_routes_in_bounds_on_nonfinite_clouds(sb, kind):
    net, b, n = _net(kind, 5), 4, 300
    x = _cloud(b, n, 9)
    x[0] = float("nan")                                   # a cloud of NaN
    x[1, 7], x[1, 200, 1] = float("inf"), float("-inf")   # Inf points
    x[2, 150:] = float("nan")                             # NaN in the later tiles only
    x[3, 0, 2], x[3, 299] = float("nan"), float("inf")
    specs = tasknets._conv_specs(net)
    sizes = list(range(1, n + 1))
    pooled, route = sb.ops.frozen_encoder_curve_forward(x, specs, sizes)
    lens = torch.tensor(sizes, device="cuda", dtype=torch.int32)[:, None, None]
    assert (route >= 0).all() and (route < lens).all()
    p16, r16 = _by_16(sb, x, specs, sizes)
    assert torch.equal(route, r16) and torch.equal(_bits(pooled), _bits(p16))


@pytest.mark.gpu
@pytest.mark.parametrize("widths,b,n,sizes", [
    pytest.param(tft.CLS_W, 5, 333, list(range(1, 334)), id="cls-every-size"),
    pytest.param(tft.AE_W, 3, 129, list(range(8, 130)), id="ae-from-8"),
    pytest.param(tft.CLS_W, 2, 300, [1, 128, 129, 300], id="cls-few-sizes"),
])
def test_curve_writes_only_its_buffers(sb, widths, b, n, sizes):
    arena = tws.Arena(nbytes=256 << 20)
    lib, ops = sb._lib.lib(), sb.ops
    specs = tws.make_fc_table(arena, "enc", widths, [1] * (len(widths) - 1), bn=True, seed=b)
    conv, _ = ops.make_layers(specs)
    nconv, (npf, csz) = len(specs), _sizes(sizes)
    g = torch.Generator().manual_seed(n)
    x = arena.carve("x", (b, n, 3), fill=torch.rand(b, n, 3, generator=g) - 0.5)
    C = widths[-1]
    pooled, route = arena.carve("pooled", (npf, b, C)), arena.carve("route", (npf, b, C), dtype=torch.int32)
    wsb = int(lib.snb200_frozen_encoder_curve_workspace_bytes(b, n, nconv, conv, npf, csz))
    ws = arena.carve("workspace", (wsb,), dtype=torch.uint8)
    rc = []
    rep = tws.run_checked(arena, "frozen_encoder_curve_forward", lambda: rc.append(lib.snb200_frozen_encoder_curve_forward(
        b, n, x.data_ptr(), nconv, conv, npf, csz, pooled.data_ptr(), route.data_ptr(), tws._addr(ws), wsb, None)), [ws], full=[pooled, route])
    assert rc == [0], lib.snb200_last_error()
    tws.assert_clean(rep)


class _FrozenClsBy16(tasknets.FrozenPointNetCls):
    """FrozenPointNetCls as the evaluator took it before: prefixes() 16 sizes per call."""
    ONE_PASS_PREFIXES = False


def _evaluator_setup(sb, n_clouds, n_points, seed=0):
    torch.manual_seed(seed)
    sampler = sb.ClassificationSampleNet(32).cuda()
    net = tft._randomize(tasknets.PointNetCls(), seed + 1).cuda().requires_grad_(False).eval()
    g = torch.Generator().manual_seed(seed + 2)
    pcs = (torch.rand(n_clouds, n_points, 3, generator=g) * 2 - 1).cuda()
    labels = torch.randint(0, 40, (n_clouds,), generator=g).cuda()
    return sampler, net, pcs, labels


@pytest.mark.gpu
def test_progressive_evaluator_dense_curve_against_16_size_route(sb, monkeypatch):
    sampler, net, pcs, labels = _evaluator_setup(sb, 40, 256)
    new = sb.ProgressiveClassificationEvaluator(sampler, tasknets.FrozenPointNetCls(net))
    old = sb.ProgressiveClassificationEvaluator(sampler, _FrozenClsBy16(net))
    ordered = new.order(pcs)
    sizes = list(range(1, 257))
    calls = []
    real = sb.ops.frozen_encoder_curve_forward
    monkeypatch.setattr(sb.ops, "frozen_encoder_curve_forward", lambda *a: calls.append(len(a[2])) or real(*a))
    with torch.no_grad():
        ln = torch.cat([new.logits(ordered[s:s + 32].contiguous(), sizes) for s in range(0, 40, 32)], dim=1)
        assert calls == [256, 256]                     # one encoder pass per batch of clouds, every size in it
        lo = torch.cat([old.logits(ordered[s:s + 32].contiguous(), sizes) for s in range(0, 40, 32)], dim=1)
    tol = LOGIT_TOL * float(lo.abs().max())
    diff = float((ln - lo).abs().max())
    print("logits: max |difference| %.3g, tolerance %.3g" % (diff, tol))
    assert diff <= tol
    # accuracy on the clouds whose top-two margin exceeds twice the tolerance at every size (so both routes must agree on the class)
    top2 = lo.topk(2, dim=2).values
    clear = ((top2[..., 0] - top2[..., 1]) > 2 * tol).all(dim=0)
    keep = torch.nonzero(clear).flatten()
    print("clouds with a clear margin at every size: %d of 40" % keep.numel())
    assert keep.numel() >= 8, "too few clouds with a clear margin at every size: %d" % keep.numel()
    top2k = lo[:, keep].topk(2, dim=2).values
    assert float((top2k[..., 0] - top2k[..., 1]).min()) > 2 * tol
    a_new = new.evaluate(pcs[keep], labels[keep], sizes, ordered=ordered[keep])
    a_old = old.evaluate(pcs[keep], labels[keep], sizes, ordered=ordered[keep])
    assert np.array_equal(a_new["accuracy"], a_old["accuracy"])
    # and the reference's default dense range 8..N through evaluate() on every cloud: the same shape, one pass per batch
    calls.clear()
    out = new.evaluate(pcs, labels, range(8, 257), ordered=ordered)
    assert out["accuracy"].shape == (249,) and calls == [249, 249]
    # retrieval goes through the same route: unsorted sizes, the descriptors within the logits' tolerance
    rs = [1, 2, 3, 64, 100, 128, 129, 200, 255, 256, 17, 5, 6, 7, 8, 9, 10]
    calls.clear()
    r = new.retrieval(pcs, labels, rs, ordered=ordered)
    assert calls == [17, 17] and r["map"].shape == (17,) and np.isfinite(r["map"]).all()
    with torch.no_grad():
        dn = new._per_size(ordered[:32].contiguous(), rs, "retrieval_vectors")
        do = old._per_size(ordered[:32].contiguous(), rs, "retrieval_vectors")
    assert float((dn - do).abs().max()) <= LOGIT_TOL * float(do.abs().max())


@pytest.mark.gpu
def test_transforms_classifier_keeps_its_16_size_route(sb, monkeypatch):
    torch.manual_seed(2)
    net = tasknets.PointNetClsTransforms().cuda().eval().requires_grad_(False)
    w = tasknets.FrozenPointNetClsTransforms(net)
    g = torch.Generator().manual_seed(3)
    ordered = (torch.rand(6, 128, 3, generator=g) * 2 - 1).cuda()
    ev = sb.ProgressiveClassificationEvaluator(None, w)
    sizes = list(range(1, 41))
    seen = []
    cls = tasknets.FrozenPointNetClsTransforms
    real = cls._prefixes      # what the prefixes property returns
    monkeypatch.setattr(cls, "_prefixes", lambda self, x, s, **k: seen.append(list(s)) or real(self, x, s, **k))
    with torch.no_grad():
        got = ev.logits(ordered, sizes)
        assert seen == [sizes[0:16], sizes[16:32], sizes[32:40]]
        want = torch.cat([real(w, ordered, sizes[i:i + 16]) for i in range(0, 40, 16)])
    assert torch.equal(got, want)
