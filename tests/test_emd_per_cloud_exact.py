"""Per-cloud EMD in the exact (parity) mode (csrc/emd.cu: approxmatch_exact_kernel<false> + the match_cost kernels rebuilding each weight
with emd_exact_match_value; ops.emd_per_cloud(..., exact=True), ops.EMDCostFunction.apply(..., True)) against the composition it replaces:
cost = match_cost(xyz1, xyz2, approx_match(xyz1, xyz2, exact=True)), gradients = grad_cost[b] * match_cost_grad on that match.  Every
comparison is torch.equal: the exact kernel's arithmetic is unchanged, each stored match element is (((0 + w7) + w6) + ... + w-2) in
round-to-nearest adds of the kernel's own level terms, and every cost and gradient sum runs in the stored route's order.

CPU: the snb200_emd_per_cloud_mode family is declared and bound, rejects bad arguments before any launch, and its flags = 0 case answers
what the original four entries answer.
GPU (H100): parity at the autoencoder size and on uneven shapes, a repeated target batch, the callers under SNB200_EMD_EXACT_EXP=1, peak
memory, run-to-run repeats and non-finite clouds.
"""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ["snb200_emd_per_cloud_mode_supported", "snb200_emd_per_cloud_mode_workspace_bytes", "snb200_emd_per_cloud_mode",
           "snb200_emd_per_cloud_mode_backward"]
EXACT = 1                  # SNB200_EMD_EXACT
MAX_B, MAX_PTS = 65535, 25600   # the exact envelope: b, and n + m (2 * (n + m) floats of shared memory in 200 KB)
EINVAL, EWORKSPACE, EUNSUPPORTED = -1, -2, -4


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
        decl = re.search(r"\b%s\(([^;]*)\);" % name, header)
        assert decl, name
        assert len(_lib._SIGNATURES[name][1]) == decl.group(1).count(",") + 1, name


def test_flags_zero_is_the_original_family(sb):
    lib = sb._lib.lib()
    for b, n, m in [(1, 1, 1), (MAX_B, 1, 1), (1, 1 << 24, 1), (1, 1, 65520), (50, 2048, 2048), (0, 1, 1), (MAX_B + 1, 1, 1),
                    (1, (1 << 24) + 1, 1), (1, 1, 65521), (1, 0, 1), (-1, 5, 5), (3, 20000, 20000)]:
        assert lib.snb200_emd_per_cloud_mode_supported(b, n, m, 0) == lib.snb200_emd_per_cloud_supported(b, n, m), (b, n, m)
        assert lib.snb200_emd_per_cloud_mode_workspace_bytes(b, n, m, 0) == lib.snb200_emd_per_cloud_workspace_bytes(b, n, m), (b, n, m)


def test_exact_envelope_and_workspace(sb):
    lib = sb._lib.lib()
    for b, n, m in [(1, 1, 1), (MAX_B, 1, 1), (1, MAX_PTS - 1, 1), (1, 1, MAX_PTS - 1), (7, 12800, 12800), (50, 2048, 2048)]:
        assert lib.snb200_emd_per_cloud_mode_supported(b, n, m, EXACT) == 1, (b, n, m)
        assert lib.snb200_emd_per_cloud_mode_workspace_bytes(b, n, m, EXACT) == lib.snb200_emd_per_cloud_workspace_bytes(b, n, m) > 0
    for b, n, m in [(0, 1, 1), (MAX_B + 1, 1, 1), (1, 0, 1), (1, 1, 0), (-1, 5, 5), (1, MAX_PTS, 1), (1, 12800, 12801), (1, 1 << 30, 1 << 30)]:
        assert lib.snb200_emd_per_cloud_mode_supported(b, n, m, EXACT) == 0, (b, n, m)
        assert lib.snb200_emd_per_cloud_mode_workspace_bytes(b, n, m, EXACT) == 0, (b, n, m)


def test_exact_rejections_launch_nothing(sb):
    """Every rejection returns before a launch, with its message; b = 0 launches nothing.  The pointers are never dereferenced, so
    stand-in addresses serve without a device."""
    lib = sb._lib.lib()
    P = 1 << 20                                        # a stand-in device address
    wsb = int(lib.snb200_emd_per_cloud_mode_workspace_bytes(4, 64, 32, EXACT))
    before = sb._lib.launch_count()

    def both(b, n, m, b2, w=P, wb=wsb, xa=P, out=P):   # out: the forward's cost and the backward's grad_cost
        return (lib.snb200_emd_per_cloud_mode(b, n, xa, m, P, b2, out, EXACT, w, wb, None),
                lib.snb200_emd_per_cloud_mode_backward(b, n, xa, m, P, b2, out, P, P, EXACT, w, wb, None))

    for args, kw, rc, text in [((-1, 64, 32, 1), {}, EINVAL, "bad sizes"), ((4, 0, 32, 2), {}, EINVAL, "bad sizes"),
                               ((4, 64, 0, 2), {}, EINVAL, "bad sizes"),
                               ((4, 25000, 601, 2), {}, EUNSUPPORTED, "exact mode's envelope"),
                               ((MAX_B + 1, 64, 32, 1), {}, EUNSUPPORTED, "exact mode's envelope"),
                               ((4, 64, 32, 3), {}, EINVAL, "must divide"), ((4, 64, 32, 0), {}, EINVAL, "must divide"),
                               ((4, 64, 32, 8), {}, EINVAL, "must divide"),
                               ((4, 64, 32, 2), {"xa": None}, EINVAL, "null pointer"), ((4, 64, 32, 2), {"out": None}, EINVAL, "null pointer"),
                               ((4, 64, 32, 2), {"wb": wsb - 1}, EWORKSPACE, "workspace"),
                               ((4, 64, 32, 2), {"w": None}, EWORKSPACE, "workspace is null")]:
        for got, who in zip(both(*args, **kw), ("emd_per_cloud", "emd_per_cloud_backward")):
            assert got == rc, (args, kw, who, got)
        assert text in lib.snb200_last_error().decode(), (args, kw, lib.snb200_last_error())
    # the backward needs at least one of its gradients
    assert lib.snb200_emd_per_cloud_mode_backward(4, 64, P, 32, P, 2, P, None, None, EXACT, P, wsb, None) == EINVAL
    assert "null pointer" in lib.snb200_last_error().decode()
    # n + m = 25600 is inside; the fast envelope's large m is outside the exact one but still inside the fast one
    assert lib.snb200_emd_per_cloud_mode(0, 25599, None, 1, None, 1, None, EXACT, None, 0, None) == 0
    assert lib.snb200_emd_per_cloud_mode(0, 64, None, 32, None, 1, None, EXACT, None, 0, None) == 0
    assert lib.snb200_emd_per_cloud_mode_backward(0, 64, None, 32, None, 1, None, None, None, EXACT, None, 0, None) == 0
    assert lib.snb200_emd_per_cloud_mode(2, 64, P, 30000, P, 1, P, EXACT, P, 1 << 40, None) == EUNSUPPORTED
    assert lib.snb200_emd_per_cloud_mode_supported(2, 64, 30000, 0) == 1
    assert sb._lib.launch_count() == before


# ---------------------------------------------------------------------------------------------------- GPU: parity
def _rand_case(b, n, m, b2, seed):
    g = _gen(seed)
    return torch.rand(b, n, 3, generator=g).cuda(), torch.rand(b2, m, 3, generator=g).cuda()


def _composed(sb, x1, x2, grad_cost):
    """The route being replaced: exact approx_match, match_cost and match_cost_grad on a repeated xyz2, gradients scaled after the kernel."""
    if x2.shape[0] != x1.shape[0]:
        x2 = x2.repeat(x1.shape[0] // x2.shape[0], 1, 1)
    match = sb.ops.approx_match(x1, x2, exact=True)
    cost = sb.ops.match_cost_forward(x1, x2, match)
    g1, g2 = sb.ops.match_cost_grad(x1, x2, match)
    return cost, g1 * grad_cost.view(-1, 1, 1), g2 * grad_cost.view(-1, 1, 1)


# (b, n, m, b2): the autoencoder size, n % 4 == 0 with m > n, n % 4 != 0 (the scalar kernels) with a short m, uneven integer
# multipliers both ways, one point against five, and 16 x 3 reconstructions against 3 targets
CASES = {"ae_50x2048x2048": (50, 2048, 2048, 50), "vec_4x64x1024": (4, 64, 1024, 4), "scalar_3x1531x77": (3, 1531, 77, 3),
         "n_gt_m_4x100x33": (4, 100, 33, 4), "n_lt_m_4x33x100": (4, 33, 100, 4), "one_1x1x5": (1, 1, 5, 1),
         "repeat_48x256x256_b2_3": (48, 256, 256, 3)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_exact_cost_and_gradients_equal_the_match_route(sb, name):
    b, n, m, b2 = CASES[name]
    x1, x2 = _rand_case(b, n, m, b2, sum(map(ord, name)))
    grad_cost = (torch.rand(b, generator=_gen(7)) - 0.3).cuda()
    cost, ws = sb.ops.emd_per_cloud_forward(x1, x2, exact=True)
    g1, g2 = sb.ops.emd_per_cloud_backward(x1, x2, grad_cost, ws, exact=True)
    want_cost, want_g1, want_g2 = _composed(sb, x1, x2, grad_cost)
    assert torch.equal(cost, want_cost), (cost - want_cost).abs().max()
    assert torch.equal(g1, want_g1), (g1 - want_g1).abs().max()
    assert torch.equal(g2, want_g2), (g2 - want_g2).abs().max()
    assert torch.equal(sb.ops.emd_per_cloud(x1, x2, exact=True), cost)
    if b2 < b:   # the autograd form sums the per-pair gradients to xyz2 over the repeats
        y1, y2 = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
        (sb.ops.EMDCostFunction.apply(y1, y2, True) * grad_cost).sum().backward()
        assert torch.equal(y1.grad, want_g1)
        assert torch.equal(y2.grad, want_g2.view(b // b2, b2, m, 3).sum(0))


@pytest.mark.gpu
def test_exact_differs_from_fast(sb):
    """The flag reaches the kernels: the two modes' costs differ (the fast mode's ex2.approx differs from the exact exponential)."""
    x1, x2 = _rand_case(4, 256, 256, 4, 13)
    assert not torch.equal(sb.ops.emd_per_cloud(x1, x2, exact=True), sb.ops.emd_per_cloud(x1, x2))
    assert torch.equal(sb.ops.emd_per_cloud(x1, x2), sb.ops.match_cost_forward(x1, x2, sb.ops.approx_match(x1, x2, exact=False)))


@pytest.mark.gpu
def test_exact_repeats_bit_for_bit(sb):
    x1, x2 = _rand_case(6, 300, 200, 3, 17)
    grad_cost = (torch.rand(6, generator=_gen(18)) - 0.5).cuda()
    outs = []
    for _ in range(2):
        cost, ws = sb.ops.emd_per_cloud_forward(x1, x2, exact=True)
        outs.append((cost,) + sb.ops.emd_per_cloud_backward(x1, x2, grad_cost, ws, exact=True))
    assert all(torch.equal(a, c) for a, c in zip(*outs))


@pytest.mark.gpu
def test_exact_nonfinite_clouds(sb):
    """NaN and Inf coordinates: the route is NaN exactly where the composition is, equal elsewhere, and the kernels finish."""
    x1, x2 = _rand_case(4, 128, 96, 4, 23)
    x1[0, 5, 1] = float("nan")
    x2[1, 7, 0] = float("inf")
    x1[2, 0, 2] = float("-inf")
    grad_cost = torch.ones(4, device="cuda")
    cost, ws = sb.ops.emd_per_cloud_forward(x1, x2, exact=True)
    g1, g2 = sb.ops.emd_per_cloud_backward(x1, x2, grad_cost, ws, exact=True)
    torch.cuda.synchronize()
    for got, want in zip((cost, g1, g2), _composed(sb, x1, x2, grad_cost)):
        assert torch.equal(torch.isnan(got), torch.isnan(want))
        keep = ~torch.isnan(want)
        assert torch.equal(got[keep], want[keep])
    assert bool(torch.isnan(cost[0])) and bool(torch.isfinite(cost[3]))


# ---------------------------------------------------------------------------------------------------- GPU: the callers
@pytest.fixture
def exact_env(monkeypatch):
    monkeypatch.setenv("SNB200_EMD_EXACT_EXP", "1")
    return monkeypatch


def _count_forwards(sb, monkeypatch):
    """Record the `exact` of every per-cloud forward, to show the callers take the route."""
    seen, forward = [], sb.ops.emd_per_cloud_forward

    def recording(xyz1, xyz2, exact=False):
        seen.append(exact)
        return forward(xyz1, xyz2, exact)

    monkeypatch.setattr(sb.ops, "emd_per_cloud_forward", recording)
    return seen


def _composed_ae_loss(x_reconstr, gt, kind="chamfer"):
    """trainers.autoencoder_loss(..., "emd") written out as the match-tensor composition (approx_match follows SNB200_EMD_EXACT_EXP)."""
    from samplenet_b200 import tf_ops

    assert kind == "emd"
    return tf_ops.match_cost(x_reconstr, gt, tf_ops.approx_match(x_reconstr, gt)).mean()


@pytest.mark.gpu
def test_autoencoder_loss_in_exact_mode(sb, exact_env):
    from samplenet_b200 import trainers

    seen = _count_forwards(sb, exact_env)
    x0, gt = _rand_case(8, 512, 512, 8, 50)
    x = x0.clone().requires_grad_(True)
    loss = trainers.autoencoder_loss(x, gt, "emd")
    loss.backward()
    y = x0.clone().requires_grad_(True)
    ref = _composed_ae_loss(y, gt, "emd")
    ref.backward()
    assert seen == [True]
    assert torch.equal(loss, ref) and torch.equal(x.grad, y.grad)


@pytest.mark.gpu
def test_autoencoder_train_step_in_exact_mode(sb, exact_env):
    """One AutoencoderTrainStep(ae_loss="emd") step: loss, parameters and Adam state bit for bit those of the written-out composition."""
    from samplenet_b200 import tasknets, trainers

    seen = _count_forwards(sb, exact_env)
    data = (torch.rand(16, 512, 3, generator=_gen(4)) - 0.5).cuda()

    def run():
        torch.manual_seed(0)
        ae = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=512)).cuda()
        opt = torch.optim.Adam(ae.parameters(), lr=5e-4, capturable=True)
        step = trainers.AutoencoderTrainStep(ae, opt, ae_loss="emd", n_sample_points=512, batch_size=16)
        loss = step(data).clone()
        state = {k: v.detach().clone() for k, v in ae.state_dict().items()}
        for i, p in enumerate(ae.parameters()):
            state.update({"opt.%d.%s" % (i, k): torch.as_tensor(v).detach().clone() for k, v in opt.state[p].items()})
        return loss, state

    loss, state = run()
    assert seen and all(seen)
    exact_env.setattr(trainers, "autoencoder_loss", _composed_ae_loss)
    want_loss, want_state = run()
    assert torch.equal(loss, want_loss)
    assert state.keys() == want_state.keys()
    for k in state:
        assert torch.equal(state[k], want_state[k]), k


@pytest.mark.gpu
def test_reconstruction_evaluator_exact_emd_curve(sb, exact_env):
    from samplenet_b200 import tasknets, tf_ops

    seen = _count_forwards(sb, exact_env)
    torch.manual_seed(5)
    sampler = sb.ReconstructionSampleNet(64).cuda()
    net = tasknets.PointNetAE(n_pc_points=256).cuda().eval().requires_grad_(False)
    ae = tasknets.FrozenPointNetAE(net)
    pcs = (torch.rand(12, 256, 3, generator=_gen(6)) - 0.5).cuda()
    sizes = [64, 8, 32]
    ev = sb.ReconstructionEvaluator(sampler, ae, ae_loss="emd")
    sampled, _ = ev.get_samples(pcs)
    got = ev.get_loss_ae_per_pc_progressive(pcs, sampled, sizes, batch_size=5)
    assert seen and all(seen)

    def composed(self, recon, gt):
        gt = gt.repeat(recon.shape[0] // gt.shape[0], 1, 1)
        return tf_ops.match_cost(recon, gt, tf_ops.approx_match(recon, gt))

    exact_env.setattr(sb.ReconstructionEvaluator, "_loss", composed)
    assert torch.equal(got, ev.get_loss_ae_per_pc_progressive(pcs, sampled, sizes, batch_size=5))


@pytest.mark.gpu
def test_exact_peak_memory_at_the_autoencoder_size(sb, exact_env):
    """50 x 2048^2 in exact mode: the loss forward + backward stays within 100 MB above its inputs; the composition holds the 839 MB
    match tensor."""
    from samplenet_b200 import trainers

    x0, gt = _rand_case(50, 2048, 2048, 50, 3)
    for fn, lo, hi in ((trainers.autoencoder_loss, 0, 100 << 20), (_composed_ae_loss, 50 * 2048 * 2048 * 4, None)):
        x = x0.clone().requires_grad_(True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn(x, gt, "emd").backward()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        assert peak >= lo and (hi is None or peak < hi), peak
