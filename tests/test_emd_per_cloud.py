"""Per-cloud EMD without the match tensor (csrc/emd.cu: approxmatch_kernel<false> + the match_cost kernels with rebuilt weights;
ops.emd_per_cloud, ops.EMDCostFunction) against the composition it replaces: cost = match_cost(xyz1, xyz2, approx_match(xyz1, xyz2)),
gradients = grad_cost[b] * match_cost_grad on that match.  Every comparison is torch.equal: the weights are rebuilt with the final pass's
expression from the same ratios, and every sum runs in the stored route's order.

CPU: the C entries are declared and in the ctypes table, and the envelope and workspace queries answer at its corners.
GPU (H100): parity on approx_match's launch-plan cases, the callers switched to it (autoencoder_loss, the evaluator's EMD curve, three
AutoencoderTrainStep steps eager and graphed), peak memory at the autoencoder size, rejections, write sets and run-to-run repeats.
"""
import os
import re
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_emd_parity as tep  # noqa: E402
import test_write_sets as tws  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ["snb200_emd_per_cloud_supported", "snb200_emd_per_cloud_workspace_bytes", "snb200_emd_per_cloud", "snb200_emd_per_cloud_backward"]
MAX_B, MAX_N, MAX_M = 65535, 1 << 24, 65520   # m: the largest match_cost takes
LEVELS = 10


@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------- CPU
def test_entries_are_declared_and_bound():
    from samplenet_b200 import _lib

    header = open(os.path.join(ROOT, "include", "samplenet_b200.h")).read()
    for name in ENTRIES:
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _lib._SIGNATURES, name


def test_envelope_and_workspace_at_the_corners(sb):
    lib = sb._lib.lib()

    def ws(b, n, m):   # grid word (256 B), the per-cloud vectors of approx_match, the 16 slab partials per cloud: each 256-byte aligned
        up = lambda x: (x + 255) // 256 * 256
        return 256 + up(b * (n + m) * (1 + LEVELS) * 4) + up(b * 16 * 4)

    for b, n, m in [(1, 1, 1), (MAX_B, 1, 1), (1, MAX_N, 1), (1, 1, MAX_M), (MAX_B, MAX_N, MAX_M), (50, 2048, 2048)]:
        assert lib.snb200_emd_per_cloud_supported(b, n, m) == 1, (b, n, m)
        assert lib.snb200_emd_per_cloud_workspace_bytes(b, n, m) == ws(b, n, m), (b, n, m)
    for b, n, m in [(0, 1, 1), (MAX_B + 1, 1, 1), (1, 0, 1), (1, MAX_N + 1, 1), (1, 1, 0), (1, 1, MAX_M + 1), (-1, 5, 5)]:
        assert lib.snb200_emd_per_cloud_supported(b, n, m) == 0, (b, n, m)
        assert lib.snb200_emd_per_cloud_workspace_bytes(b, n, m) == 0, (b, n, m)
    assert ws(50, 2048, 2048) < 64 << 20


# ---------------------------------------------------------------------------------------------------- GPU: parity
def _composed(sb, x1, x2, grad_cost):
    """The route being replaced: approx_match, match_cost, match_cost_grad on a repeated xyz2, gradients scaled after the kernel."""
    if x2.shape[0] != x1.shape[0]:
        x2 = x2.repeat(x1.shape[0] // x2.shape[0], 1, 1)
    match = sb.ops.approx_match(x1, x2, exact=False)
    cost = sb.ops.match_cost_forward(x1, x2, match)
    g1, g2 = sb.ops.match_cost_grad(x1, x2, match)
    return cost, g1 * grad_cost.view(-1, 1, 1), g2 * grad_cost.view(-1, 1, 1)


def _rand_case(b, n, m, b2, seed):
    g = _gen(seed)
    return torch.rand(b, n, 3, generator=g).cuda(), torch.rand(b2, m, 3, generator=g).cuda()


# approx_match's launch-plan cases of test_emd_parity, n != m both ways, b = 1, n % 4 != 0 (the scalar path), the autoencoder size,
# 800 pairs against 50 clouds, and m past 48 KB of the cost kernel's shared memory up to the largest m the composition runs (65472: the
# stored match_cost kernel's 32 bytes of static shared memory sit beside its 48 KB of staged points)
CASES = {
    "dup_4x512x512": None, "thin_3x5000x13": None, "wide_7x999x3000": None, "one_1x1x1": None, "one_2x1x700": None,
    "one_2x700x1": None, "small_200x64x64": None,
    "n_gt_m_5x1024x256": (5, 1024, 256, 5), "n_lt_m_5x256x1024": (5, 256, 1024, 5), "b1_1x2048x1024": (1, 2048, 1024, 1),
    "scalar_3x1001x777": (3, 1001, 777, 3), "ae_50x2048x2048": (50, 2048, 2048, 50), "repeat_800x512x512_b2_50": (800, 512, 512, 50),
    "big_m_1x2048x16384": (1, 2048, 16384, 1), "max_m_2x256x65472": (2, 256, 65472, 2),
}


def _case(name):
    if CASES[name] is None:
        return tep._clouds(name)
    b, n, m, b2 = CASES[name]
    return _rand_case(b, n, m, b2, sum(map(ord, name)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_cost_and_gradients_equal_the_match_route(sb, name):
    x1, x2 = _case(name)
    b = x1.shape[0]
    grad_cost = (torch.rand(b, generator=_gen(7)) - 0.3).cuda()
    cost, ws = sb.ops.emd_per_cloud_forward(x1, x2)
    g1, g2 = sb.ops.emd_per_cloud_backward(x1, x2, grad_cost, ws)
    want_cost, want_g1, want_g2 = _composed(sb, x1, x2, grad_cost)
    assert torch.equal(cost, want_cost), (cost - want_cost).abs().max()
    assert torch.equal(g1, want_g1), (g1 - want_g1).abs().max()
    assert torch.equal(g2, want_g2), (g2 - want_g2).abs().max()
    assert torch.equal(sb.ops.emd_per_cloud(x1, x2), cost)


@pytest.mark.gpu
def test_largest_m_runs(sb):
    """m = 65520, the envelope's corner, past what the composition runs: finite costs and gradients, the same bits twice."""
    x1, x2 = _rand_case(2, 64, MAX_M, 1, 41)
    grad_cost = torch.ones(2, device="cuda")
    outs = []
    for _ in range(2):
        cost, ws = sb.ops.emd_per_cloud_forward(x1, x2)
        outs.append((cost,) + sb.ops.emd_per_cloud_backward(x1, x2, grad_cost, ws))
    assert all(bool(torch.isfinite(t).all()) for t in outs[0]) and bool((outs[0][0] > 0).all())
    assert all(torch.equal(a, c) for a, c in zip(*outs))


@pytest.mark.gpu
def test_one_gradient_alone(sb, monkeypatch):
    """grad1 or grad2 alone (the other pointer null) is the same bits as with both, and EMDCostFunction runs only the pass an input needs."""
    lib = sb._lib.lib()
    x1, x2 = _rand_case(6, 640, 700, 3, 21)
    grad_cost = (torch.rand(6, generator=_gen(22)) - 0.5).cuda()
    _, ws = sb.ops.emd_per_cloud_forward(x1, x2)
    g1, g2 = sb.ops.emd_per_cloud_backward(x1, x2, grad_cost, ws)
    assert sb.ops.emd_per_cloud_backward(x1, x2, grad_cost, ws, need2=False)[1] is None
    assert torch.equal(sb.ops.emd_per_cloud_backward(x1, x2, grad_cost, ws, need2=False)[0], g1)
    assert torch.equal(sb.ops.emd_per_cloud_backward(x1, x2, grad_cost, ws, need1=False)[1], g2)
    assert lib.snb200_emd_per_cloud_backward(6, 640, x1.data_ptr(), 700, x2.data_ptr(), 3, grad_cost.data_ptr(), None, None, ws.data_ptr(),
                                             ws.numel(), None) == -1
    asked, backward = [], sb.ops.emd_per_cloud_backward

    def recording(*args):
        asked.append(args[4:])
        return backward(*args)

    monkeypatch.setattr(sb.ops, "emd_per_cloud_backward", recording)
    x = x1.clone().requires_grad_(True)
    (sb.ops.EMDCostFunction.apply(x, x2) * grad_cost).sum().backward()
    assert torch.equal(x.grad, g1)
    y2 = x2.clone().requires_grad_(True)
    (sb.ops.EMDCostFunction.apply(x1, y2) * grad_cost).sum().backward()
    assert torch.equal(y2.grad, g2.view(2, 3, 700, 3).sum(0))
    assert asked == [(True, False), (False, True)]


@pytest.mark.gpu
def test_callers_keep_the_composition_outside_the_envelope(sb):
    """n > 2^24 is outside the per-cloud envelope but inside the composition's: autoencoder_loss still returns, through the composition."""
    from samplenet_b200 import tf_ops, trainers

    x0, gt = _rand_case(1, MAX_N + 4, 2, 1, 31)
    assert not sb.ops.emd_per_cloud_supported(x0, gt)
    x = x0.clone().requires_grad_(True)
    loss = trainers.autoencoder_loss(x, gt, "emd")
    loss.backward()
    y = x0.clone().requires_grad_(True)
    ref = tf_ops.match_cost(y, gt, tf_ops.approx_match(y, gt)).mean()
    ref.backward()
    assert torch.equal(loss, ref) and torch.equal(x.grad, y.grad)


@pytest.mark.gpu
def test_peak_memory_at_the_autoencoder_size(sb):
    """50 x 2048^2: the per-cloud call allocates its cost and workspace (9 MB); the match route holds the 838 MB match tensor."""
    x1, x2 = _rand_case(50, 2048, 2048, 50, 3)
    sb.ops.emd_per_cloud(x1, x2)
    torch.cuda.synchronize()
    for fn, lo, hi in ((lambda: sb.ops.emd_per_cloud(x1, x2), 0, 64 << 20),
                       (lambda: sb.ops.match_cost_forward(x1, x2, sb.ops.approx_match(x1, x2)), 50 * 2048 * 2048 * 4, None)):
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        assert peak >= lo and (hi is None or peak < hi), peak


@pytest.mark.gpu
def test_autograd_form_and_repeat_reduction(sb):
    """EMDCostFunction under .mean() and a weighted sum: loss and both gradients equal MatchCostFunction on approx_match's match; with
    xyz2 repeated every b2 clouds the gradient to xyz2 is the per-pair gradient summed over the repeats."""
    p1, p2 = tep._clouds("wide_7x999x3000")
    weights = (torch.rand(7, generator=_gen(9)) - 0.3).cuda()
    for reduce in (lambda c: c.mean(), lambda c: (c * weights).sum()):
        x1, x2 = p1.clone().requires_grad_(True), p2.clone().requires_grad_(True)
        loss = reduce(sb.ops.EMDCostFunction.apply(x1, x2))
        loss.backward()
        y1, y2 = p1.clone().requires_grad_(True), p2.clone().requires_grad_(True)
        ref = reduce(sb.tf_ops.match_cost(y1, y2, sb.tf_ops.approx_match(y1, y2)))
        ref.backward()
        assert torch.equal(loss, ref) and torch.equal(x1.grad, y1.grad) and torch.equal(x2.grad, y2.grad)
    a, c = _rand_case(12, 300, 200, 3, 12)
    x2 = c.clone().requires_grad_(True)
    sb.ops.EMDCostFunction.apply(a, x2).sum().backward()
    _, _, g2 = _composed(sb, a, c, torch.ones(12, device="cuda"))
    assert torch.equal(x2.grad, g2.view(4, 3, 200, 3).sum(0))


# ---------------------------------------------------------------------------------------------------- GPU: the callers
def _composed_ae_loss(x_reconstr, gt, kind="chamfer"):
    """trainers.autoencoder_loss(..., "emd") written out as the match-tensor composition."""
    from samplenet_b200 import tf_ops

    assert kind == "emd"
    return tf_ops.match_cost(x_reconstr, gt, tf_ops.approx_match(x_reconstr, gt)).mean()


@pytest.mark.gpu
def test_autoencoder_loss_equals_the_written_out_composition(sb):
    from samplenet_b200 import tf_ops, trainers

    x0, gt = _rand_case(50, 2048, 2048, 50, 50)
    x = x0.clone().requires_grad_(True)
    loss = trainers.autoencoder_loss(x, gt, "emd")
    loss.backward()
    y = x0.clone().requires_grad_(True)
    ref = tf_ops.match_cost(y, gt, tf_ops.approx_match(y, gt)).mean()
    ref.backward()
    assert torch.equal(loss, ref) and torch.equal(x.grad, y.grad)


@pytest.mark.gpu
def test_reconstruction_evaluator_emd_curve_equals_the_written_out_composition(sb, monkeypatch):
    from samplenet_b200 import tasknets, tf_ops

    torch.manual_seed(5)
    sampler = sb.ReconstructionSampleNet(64).cuda()
    net = tasknets.PointNetAE(n_pc_points=256).cuda().eval().requires_grad_(False)
    ae = tasknets.FrozenPointNetAE(net)
    pcs = (torch.rand(12, 256, 3, generator=_gen(6)) - 0.5).cuda()
    sizes = [64, 1, 16, 32, 8]
    ev = sb.ReconstructionEvaluator(sampler, ae, ae_loss="emd")
    sampled, _ = ev.get_samples(pcs)
    got = ev.get_loss_ae_per_pc_progressive(pcs, sampled, sizes, batch_size=5)
    single = ev.get_loss_ae_per_pc(pcs, sampled, batch_size=5)

    def composed(self, recon, gt):
        gt = gt.repeat(recon.shape[0] // gt.shape[0], 1, 1)
        return tf_ops.match_cost(recon, gt, tf_ops.approx_match(recon, gt))

    monkeypatch.setattr(sb.ReconstructionEvaluator, "_loss", composed)
    assert torch.equal(got, ev.get_loss_ae_per_pc_progressive(pcs, sampled, sizes, batch_size=5))
    assert torch.equal(single, ev.get_loss_ae_per_pc(pcs, sampled, batch_size=5))


@pytest.mark.gpu
@pytest.mark.parametrize("graphed", [False, True])
def test_autoencoder_train_steps_equal_the_written_out_composition(sb, monkeypatch, graphed):
    """Three AutoencoderTrainStep(ae_loss="emd") steps: losses, parameters and Adam state bit for bit those of the same steps with the
    loss written out as approx_match + match_cost."""
    from samplenet_b200 import tasknets, trainers

    data = (torch.rand(3, 16, 512, 3, generator=_gen(4)) - 0.5).cuda()

    def run():
        torch.manual_seed(0)
        ae = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=512)).cuda()
        opt = torch.optim.Adam(ae.parameters(), lr=5e-4, capturable=True)
        step = trainers.AutoencoderTrainStep(ae, opt, ae_loss="emd", n_sample_points=512, batch_size=16, graphed=graphed)
        losses = [step(x).clone() for x in data]
        state = {k: v.detach().clone() for k, v in ae.state_dict().items()}
        for i, p in enumerate(ae.parameters()):
            state.update({"opt.%d.%s" % (i, k): torch.as_tensor(v).detach().clone() for k, v in opt.state[p].items()})
        return losses, state

    losses, state = run()
    monkeypatch.setattr(trainers, "autoencoder_loss", _composed_ae_loss)
    want_losses, want_state = run()
    assert all(torch.equal(a, b) for a, b in zip(losses, want_losses))
    assert state.keys() == want_state.keys()
    for k in state:
        assert torch.equal(state[k], want_state[k]), k


# ---------------------------------------------------------------------------------------------------- GPU: contract
@pytest.mark.gpu
def test_rejections_launch_nothing(sb):
    lib = sb._lib.lib()
    x1, x2 = _rand_case(4, 64, 32, 2, 1)
    wsb = int(lib.snb200_emd_per_cloud_workspace_bytes(4, 64, 32))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    cost, gc = torch.empty(4, device="cuda"), torch.ones(4, device="cuda")
    g1, g2 = torch.empty(4, 64, 3, device="cuda"), torch.empty(4, 32, 3, device="cuda")
    p = lambda t: t.data_ptr()
    before = sb._lib.launch_count()

    def both(b, n, m, b2, w, wb, xa=p(x1), xb=p(x2)):
        return (lib.snb200_emd_per_cloud(b, n, xa, m, xb, b2, p(cost), w, wb, None),
                lib.snb200_emd_per_cloud_backward(b, n, xa, m, xb, b2, p(gc), p(g1), p(g2), w, wb, None))

    einval, ews, eunsup = -1, -2, -4
    for args, rc, text in [((4, 0, 32, 2, p(ws), wsb), einval, "bad sizes"), ((4, 64, 0, 2, p(ws), wsb), einval, "bad sizes"),
                           ((-1, 64, 32, 1, p(ws), wsb), einval, "bad sizes"), ((4, 64, 32, 3, p(ws), wsb), einval, "must divide"),
                           ((4, 64, 32, 0, p(ws), wsb), einval, "must divide"), ((4, 64, 32, 8, p(ws), wsb), einval, "must divide"),
                           ((4, 64, MAX_M + 1, 2, p(ws), wsb), eunsup, "envelope"), ((MAX_B + 1, 64, 32, 1, p(ws), wsb), eunsup, "envelope"),
                           ((4, 64, 32, 2, p(ws), wsb - 1), ews, "workspace"), ((4, 64, 32, 2, None, wsb), ews, "workspace is null")]:
        for got, who in zip(both(*args), ("emd_per_cloud", "emd_per_cloud_backward")):
            assert got == rc, (args, who, got)
        assert text in lib.snb200_last_error().decode()
    assert both(4, 64, 32, 2, p(ws), wsb, xa=None) == (einval, einval)
    assert both(0, 64, 32, 1, None, 0) == (0, 0)
    with pytest.raises(ValueError, match="must divide"):
        sb.ops.emd_per_cloud(x1, x2[:1].expand(3, -1, -1))
    with pytest.raises(ValueError, match="expects"):
        sb.ops.emd_per_cloud(x1[..., :2], x2)
    with pytest.raises(RuntimeError, match="without a backward"):
        sb.ops.emd_per_cloud(x1.clone().requires_grad_(True), x2)
    assert sb.ops.emd_per_cloud(torch.zeros(0, 5, 3, device="cuda"), torch.zeros(1, 7, 3, device="cuda")).shape == (0,)
    assert sb._lib.launch_count() == before


@pytest.mark.gpu
@pytest.mark.parametrize("b,b2,n,m", [(6, 2, 300, 200), (3, 3, 1001, 17), (8, 4, 64, 2048), (1, 1, 1, 1)])
def test_writes_only_its_buffers_and_repeats_bit_for_bit(sb, b, b2, n, m):
    """The forward writes its cost and workspace; the backward writes grad1 and grad2 and reads the workspace without writing it.  Two
    calls on the same inputs in fresh buffers give the same bits."""
    lib = sb._lib.lib()
    arena = tws.Arena(256 << 20)
    g = _gen(n + m)
    vals = (torch.rand(b, n, 3, generator=g), torch.rand(b2, m, 3, generator=g), torch.rand(b, generator=g) - 0.5)
    wsb = int(lib.snb200_emd_per_cloud_workspace_bytes(b, n, m))
    rep, rc, outs = [], [], []
    for i in range(2):
        x1 = arena.carve("call%d.xyz1" % i, (b, n, 3), fill=vals[0])
        x2 = arena.carve("call%d.xyz2" % i, (b2, m, 3), fill=vals[1])
        gc = arena.carve("call%d.grad_cost" % i, (b,), fill=vals[2])
        cost, ws = arena.carve("call%d.cost" % i, (b,)), arena.carve("call%d.workspace" % i, (wsb,), dtype=torch.uint8)
        g1, g2 = arena.carve("call%d.grad1" % i, (b, n, 3)), arena.carve("call%d.grad2" % i, (b, m, 3))
        rep += tws.run_checked(arena, "emd_per_cloud #%d" % i, lambda: rc.append(lib.snb200_emd_per_cloud(
            b, n, x1.data_ptr(), m, x2.data_ptr(), b2, cost.data_ptr(), tws._addr(ws), wsb, None)), [ws], full=[cost])
        rep += tws.run_checked(arena, "emd_per_cloud_backward #%d" % i, lambda: rc.append(lib.snb200_emd_per_cloud_backward(
            b, n, x1.data_ptr(), m, x2.data_ptr(), b2, gc.data_ptr(), g1.data_ptr(), g2.data_ptr(), tws._addr(ws), wsb, None)),
            full=[g1, g2])
        outs.append((cost.clone(), g1.clone(), g2.clone()))
    assert rc == [0] * 4, lib.snb200_last_error()
    tws.assert_clean(rep)
    assert all(torch.equal(a, c) for a, c in zip(*outs))
