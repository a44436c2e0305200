"""Training the progressive samplers on the CUDA generator backward: FC output layers of any width.

fc_bwd_kernel streams the upper layer's dz and W_up through shared memory in chunks of upper channels (a multiple of 4, chosen on the
host from the 200 KB budget), so the backward's envelope no longer depends on the output layer's width.  3 M output channels with
M = 341 (cls / registration at B = 32) and M = 209 (rec at B = 50) are the first widths that did not fit whole; 3 x 341 = 1023 and
3 x 209 = 627 leave a c_up % 4 tail of 3.

CPU: the host envelope and workspace sizes of the wide tables.  GPU: the per-layer and fused training paths on wide samplers with the
stage checks of test_layers_training_parity.py (forward, running statistics, backward against the kernel-valued float64 graph and end to
end against plain float64 on a conditioned instance, each run repeated and bit-identical), and whole ProgressiveClassificationStep /
ProgressiveReconstructionStep steps against the torch recompute."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import test_layers_training_parity as ltp  # noqa: E402
from test_sampler_training import _cloud, _pair  # noqa: E402

_next_ptr = [0x80000]


def _ptr():
    _next_ptr[0] += 0x1000
    return _next_ptr[0]


def _table(widths, bn, relu, eps=1e-5, momentum=0.1):
    from samplenet_b200._lib import Layer
    arr = (Layer * (len(widths) - 1))()
    for i in range(len(widths) - 1):
        L = arr[i]
        L.c_in, L.c_out = widths[i], widths[i + 1]
        L.weight, L.bias = _ptr(), _ptr()
        if bn[i]:
            L.bn_weight, L.bn_bias, L.bn_running_mean, L.bn_running_var, L.bn_num_batches_tracked = _ptr(), _ptr(), _ptr(), _ptr(), _ptr()
            L.bn_eps, L.bn_momentum = eps, momentum
        L.relu = int(relu[i])
    return arr


def _tables(name, m):
    """Fake (never dereferenced) layer tables of ReconstructionSampleNet(m), ClassificationSampleNet(m) and SampleNet(m, 128)."""
    if name == "rec":
        return _table([3, 64, 128, 128, 256, 128], [1] * 5, [1] * 5), _table([128, 256, 256, 3 * m], [0, 0, 0], [1, 1, 0])
    eps, mom = (1e-3, 0.5) if name == "cls" else (1e-5, 0.1)
    fc_bn = [1, 1, 1, 1] if name == "cls" else [1, 1, 1, 0]
    return _table([3, 64, 64, 64, 128, 128], [1] * 5, [1] * 5, eps, mom), _table([128, 256, 256, 256, 3 * m], fc_bn, [1, 1, 1, 0], eps, mom)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


WIDE = [("cls", m, b) for m in (341, 512, 1024) for b in (2, 32, 64)] + [("rec", m, 50) for m in (209, 256, 2048)]


@pytest.mark.parametrize("name,m,b", WIDE)
def test_wide_output_layers_are_in_the_per_layer_envelope(lib, name, m, b):
    conv, fc = _tables(name, m)
    for n in (777, 1024, 2048):
        assert lib.snb200_generator_layers_backward_supported(b, n, 5, conv, len(fc), fc) == 1, (name, m, b, n)
        # one backward, one workspace layout: streaming the upper layer adds no workspace
        ws = lib.snb200_generator_layers_backward_workspace_bytes(b, n, 5, conv, len(fc), fc)
        assert ws > 0 and ws == lib.snb200_generator_backward_workspace_bytes(b, n, 5, conv, len(fc), fc), (name, m, b, n)


@pytest.mark.parametrize("name,m", [("cls", 1024), ("rec", 2048), ("reg", 1024)])
def test_wide_tables_keep_the_rest_of_the_envelope(lib, name, m):
    for b in (1, 65):
        conv, fc = _tables(name, m)
        assert lib.snb200_generator_layers_backward_supported(b, 1024, 5, conv, len(fc), fc) == 0, (name, b)
        assert lib.snb200_generator_backward_supported(b, 1024, 5, conv, len(fc), fc) == 0, (name, b)
    conv, fc = _tables(name, m)
    fc[len(fc) - 1].relu = 1   # ReLU on the output layer: its mask would need `out`
    assert lib.snb200_generator_layers_backward_supported(32, 1024, 5, conv, len(fc), fc) == 0


def test_registration_table_at_1024_points_routes_fused(lib):
    conv, fc = _tables("reg", 1024)
    assert lib.snb200_generator_backward_supported(32, 1024, 5, conv, 4, fc) == 1
    assert lib.snb200_generator_layers_backward_supported(32, 1024, 5, conv, 4, fc) == 1
    ws = lib.snb200_generator_backward_workspace_bytes(32, 1024, 5, conv, 4, fc)
    assert ws > 0 and ws == lib.snb200_generator_layers_backward_workspace_bytes(32, 1024, 5, conv, 4, fc)


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


# (table, M, b, n, layout, signs) and the chunks fc_bwd_kernel streams the 3 M-wide output layer in: cls 1024 at b = 32 in 4 (1020 channels
# each but the last), rec 2048 at b = 50 in 10 (624), rec 209 at b = 64 in 2 (452 + 175: a tail of 3), cls 341 at b = 32 in 2 (1020 + 3:
# the last chunk is the tail alone), cls 341 at b = 16 in 1 with its tail of 3.  (The cls table's smallest batch is 16, not 2: BatchNorm
# over the FC layers' 2 rows differences two nearly equal values, and an fp32 FC head, torch's included, is then 2e-4 .. 4e-4 of the
# output away from float64, 5x the forward bar.)
PER_LAYER_CASES = [
    ("cls", 1024, 32, 1024, "bnc", True),
    ("rec", 2048, 50, 2048, "bnc", True),
    ("rec", 209, 64, 2048, "bnc", True),
    ("cls", 341, 32, 1024, "bnc", True),
    ("cls", 341, 16, 777, "bcn", True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("table,m,b,n,layout,signs", PER_LAYER_CASES)
def test_wide_per_layer_training_path_vs_float64(sb, monkeypatch, table, m, b, n, layout, signs):
    monkeypatch.setattr(ltp, "M_OUT", m)
    rep, info = ltp.run_case(sb, table, b, n, layout, signs, 0)
    if signs:
        ltp._assert_dead_channels(info)
    ltp._assert_report(rep, info)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["bnc", "bcn"])
def test_wide_fused_training_path_vs_float64(sb, monkeypatch, layout):
    """SampleNet(1024)'s table on the fused path at 32 x 1024 (several 128-point slices per CTA), BNC with the transposed store of its
    3072-wide output."""
    m = 1024
    monkeypatch.setattr(ltp, "M_OUT", m)
    rep, info = ltp.run_case(sb, "reg", 32, 1024, layout, True, m if layout == "bnc" else 0, route="fused")
    ltp._assert_dead_channels(info)
    ltp._assert_report(rep, info)
    net = sb.SampleNet(m, 128, group_size=7, input_shape="bnc", output_shape="bnc").cuda().train()
    net(torch.rand(32, 1024, 3, device="cuda") - 0.5)
    assert net.generator_route == "fused"


STEP_GUARD = 1e-6   # whole steps: no routed conv unit this close to its ReLU kink, no pooled extreme this close to its runner-up


def _conditioned_sampler(make, x, seed0):
    """(seed, sampler) for the first seed from seed0 whose float64 forward on x has no conv unit at a point the max-pool routes to within
    STEP_GUARD of its ReLU kink (relative to |scale z| + |shift|, ltp.kink_distances) and no pooled (cloud, channel) whose runner-up
    point is within STEP_GUARD of the extreme (relative).  The CUDA route keeps the forward's own fp32 masks and arg-max; the torch
    recompute takes its own.  A unit on different sides of its kink in the two moves whole gradients apart: measured on unconditioned
    instances, up to 2e-3 of conv2.weight (rec, a unit 6e-8 from its kink) and 1.7e-1 of fc1's BatchNorm shift (cls, 2e-7); every flip
    seen was within 3e-7."""
    b = x.shape[0]
    for seed in range(seed0, seed0 + 40):
        torch.manual_seed(seed)
        net = make()
        zs, _ = ltp._conv_forward64(net, x, "bnc")
        gam = net._layer_specs()[0][-1]["bn"][0].detach().double()
        route = ltp._route(zs[-1], gam, b)
        kink = min(k.min().item() for k in ltp.kink_distances(net, zs, route))
        top2 = (zs[-1].view(b, -1, zs[-1].shape[1]) * torch.where(gam >= 0, 1.0, -1.0).to(zs[-1])).topk(2, dim=1)[0]
        gap = ((top2[:, 0] - top2[:, 1]) / top2[:, 0].abs()).min().item()
        if kink > STEP_GUARD and gap > STEP_GUARD:
            return seed, net
    raise AssertionError("no conditioned sampler")


def _compare_routes(net, loss_fn):
    """One step on the CUDA backward, repeated (loss and gradients bit-identical), against the same step with generator_backward="torch"
    (loss within 1e-5, every gradient within 2e-3 of its scale: its largest entry, or for a generator tensor whose true gradient is 0 --
    ltp.zero_true_names: rounding noise on both sides -- the largest entry of its layer's weight gradient, as in ltp._scales)."""
    net, ref = _pair(net)
    runs = []
    for n in (net, net, ref):
        n.zero_grad(set_to_none=True)
        loss = loss_fn(n)
        loss.backward()
        runs.append((loss.detach().clone(), {k: p.grad.detach().clone() for k, p in n.named_parameters() if p.requires_grad}, n.generator_route))
    (la, ga, ra), (lb, gb, _), (lt, gt, rt) = runs
    assert (ra, rt) == ("layers", "torch")
    assert torch.equal(la, lb) and all(torch.equal(ga[k], gb[k]) for k in ga), "CUDA step not bit-identical run to run"
    assert abs(float(la) - float(lt)) <= 1e-5 * abs(float(lt)), (float(la), float(lt))
    gen = dict(net._generator_named_parameters())
    by_name = {id(p): k for k, p in net.named_parameters()}
    alias = {by_name[id(p)]: k for k, p in gen.items()}   # module name -> "l<i>.<w|b|g|beta>"
    scale = ltp._scales(net, {alias[k]: gt[k] for k in alias})
    bad = []
    for k in gt:
        sc = scale[alias[k]] if k in alias else max(gt[k].abs().max().item(), 1e-30)
        err = (ga[k] - gt[k]).abs().max().item() / sc
        if err > 2e-3:
            bad.append((k, err))
    assert not bad, bad


@pytest.mark.gpu
def test_progressive_classification_step_on_the_per_layer_path(sb, monkeypatch):
    from samplenet_b200 import tasknets, trainers
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)   # the frozen classifier's input gradient, run to run
    B, N, M = 32, 1024, 1024
    x = _cloud(B, N, "bnc", 25)
    _, net = _conditioned_sampler(lambda: sb.ClassificationSampleNet(M, group_size=7).cuda().train(), x, 8)
    cls = tasknets.PointNetCls().cuda()
    y = torch.randint(0, 40, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    _compare_routes(net, lambda s: trainers.ProgressiveClassificationStep(s, cls, 8, M).loss(x, y)[0])


@pytest.mark.gpu
def test_progressive_reconstruction_step_on_the_per_layer_path(sb, monkeypatch):
    from samplenet_b200 import tasknets, trainers
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)   # the frozen AE's input gradient, run to run
    B, N = 50, 2048
    x = _cloud(B, N, "bnc", 26)
    _, net = _conditioned_sampler(lambda: sb.ReconstructionSampleNet(N).cuda().train(), x, 8)
    ae = tasknets.PointNetAE(N, 128).cuda()
    _compare_routes(net, lambda s: trainers.ProgressiveReconstructionStep(s, ae).loss(x)[0])
    # the loss against the reference's per-prefix structure: one AE loss and one simplification loss (weight s / 64) per prefix
    step = trainers.ProgressiveReconstructionStep(net, ae)
    sizes = [16 * 2 ** i for i in range(8)]
    assert step.sizes == sizes
    with torch.no_grad():
        total, _ = step.loss(x)
        simp, proj = net(x)
        loss_ae = sum(trainers.autoencoder_loss(ae(proj[:, :s].contiguous()), x) for s in sizes) / len(sizes)
        loss_simp = sum(trainers.autoencoder_simplification_loss(x, simp[:, :s].contiguous(), s)[0] for s in sizes) / len(sizes)
        want = loss_ae + 0.01 * loss_simp + 1e-4 * net.get_projection_loss()
        per_prefix = trainers.progressive_simplification_loss(x, simp, sizes, 0, 1 / 64.0, one_pass=False) / len(sizes)
    assert abs(float(total) - float(want)) <= 1e-5 * abs(float(want)), (float(total), float(want))
    assert abs(float(per_prefix) - float(loss_simp)) <= 1e-5 * abs(float(loss_simp))


def test_progressive_reconstruction_step_rejects_emd():
    from samplenet_b200 import trainers
    with pytest.raises(ValueError):
        trainers.ProgressiveReconstructionStep(torch.nn.Identity(), torch.nn.Identity(), ae_loss="emd")
