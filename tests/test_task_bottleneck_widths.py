"""The frozen task-network encoders and PCRNet's CUDA path against float64 at last conv layers other than 128 and 1024 channels, and a full
16-prefix pack.

PointNetAE(n_pc_points, bneck_size), PCRNet(bottleneck_size) and PointNetFeatures(bottleneck_size) take any bottleneck width C, and the
frozen encoder, the batch-statistics encoder and the parameter backward take a last conv layer of 8 to 1024 channels.  The width decides
which code runs:

    C = 8     tc_layer_kernel<64, PFX>: masked columns, four row ranges in the epilogue; one partial route word (8 of 32 bits)
    C = 40    <64>, not a multiple of 32: a partial route word, a partial 32-channel block of bs_reduce_kernel
    C = 100   <128>, masked
    C = 200   <256>, masked, one block; two 128-channel passes of bs_bwd_layer_kernel, the second partial
    C = 256   <256>, one full block: the edge between one block and several
    C = 300   two blocks over grid.y, the second 44 channels wide
    C = 520   three blocks, the third 8 channels wide
    C = 1000  four blocks, the last 232 channels wide; 32 route words, the last one partial

Every width is a multiple of 4, so PCRNet's first FC layer (2 C inputs) stays inside the frozen MLP's envelope (c_in a multiple of 8).

GPU (H100), each case at the bars of the module whose check it runs:
  eval frozen encoder   FrozenPointNetAE's encoder, test_frozen_tasknets: pooled and route per prefix against float64 (the route the first
                        extreme), repeat calls and one-prefix calls on x[:, :s] bit for bit, exact ties to the first index, channels pooled to
                        exactly 0 in some clouds; grad_x against float64 on the kernel's routes, unrouted points exactly 0;
  batch statistics      test_ae_batch_stats: statistics, raw outputs and pool against float64, grad_x against pinned float64 autograd,
                        repeat calls and one-prefix calls bit for bit;
  PCRNet                test_pcrnet_training / test_frozen_pcrnet: the parameter backward's dW, db and grad_x against float64, the frozen
                        MLP forward, backward and parameter backward with the 2C-wide input, FrozenPCRNet against the module and float64,
                        and at two widths (one block, three blocks) CudaPCRNet with the pose loss against float64 autograd and a whole
                        train step against the plain module; each asserts that the wrapper ran the kernels, not its module fallback;
  autoencoder step      CudaPointNetAE's training step at 40 and 300 takes the module route (the CUDA backward takes only the 256 -> 128
                        last layer): the route, and the reconstruction and loss against the float64 module;
  prefix cap            16 prefixes with several boundaries in one tile and sizes 128k - 1, 128k, 128k + 1, through the eval encoder
                        (classifier and autoencoder), the batch-statistics encoder and the parameter backward.
CPU: every width inside each envelope, FrozenPCRNet's module route where 2C is not a multiple of 8, CudaPointNetAE's route per width."""
import copy
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import test_ae_batch_stats as tab  # noqa: E402
import test_frozen_pcrnet as tfp  # noqa: E402
import test_frozen_tasknets as tft  # noqa: E402
import test_pcrnet_training as tpt  # noqa: E402
import test_sampler_training as tst  # noqa: E402
import test_task_training as ttr  # noqa: E402
from samplenet_b200 import registration as reg  # noqa: E402
from samplenet_b200 import tasknets, trainers  # noqa: E402

WIDTHS = (8, 40, 100, 200, 256, 300, 520, 1000)
AE_CONV = [3, 64, 128, 128, 256]            # PointNetAE's conv layers ahead of the bottleneck
PCR_CONV = [3, 64, 64, 64, 128]             # PointNetFeatures'
PCR_FC = [1024, 1024, 512, 512, 256, 7]     # PCRNet's FC layers after the 2C-wide concatenated feature

# (b, n, prefixes, duplicated points): a ragged multi-prefix shape off the tile grid, and the progressive reconstruction trainer's plan
SHAPES = {"ragged": (5, 333, [1, 7, 127, 128, 129, 300, 333], True), "pow2": (50, 2048, [16 * 2 ** i for i in range(8)], False)}
# the prefix cap: 16 ascending sizes, five boundaries in tile 0, 128k - 1 / 128k / 128k + 1 at k = 1, 2, 3
PFX16 = [1, 2, 3, 5, 8, 127, 128, 129, 200, 255, 256, 257, 383, 384, 385, 1000]
PFX_B, PFX_N = 3, 1000


def ae_widths(c):
    return AE_CONV + [c]


def pcr_widths(c):
    return PCR_CONV + [c]


def mlp_widths(c):
    return [2 * c] + PCR_FC


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_prefix_cap_sizes():
    assert len(PFX16) == 16 and PFX16 == sorted(set(PFX16)) and PFX16[-1] == PFX_N
    in_tile0 = [s for s in PFX16 if s <= 128]
    assert len(in_tile0) >= 5 and all(k * 128 + d in PFX16 for k in (1, 2, 3) for d in (-1, 0, 1))


def test_width_table():
    """Each width reaches the path it is listed for: the tensor-core kernel's padded width (64 / 128 / 256), its blocks of 256 channels and
    the last block's width, the route words and the last word's bits, and bs_bwd_layer_kernel's 128-channel passes."""
    nout = lambda c: 64 if c <= 64 else 128 if c <= 128 else 256
    blocks = lambda c: -(-c // 256)
    got = {c: (nout(c), blocks(c), c - 256 * (blocks(c) - 1), -(-c // 32), c % 32, -(-c // 128)) for c in WIDTHS}
    assert got == {8: (64, 1, 8, 1, 8, 1), 40: (64, 1, 40, 2, 8, 1), 100: (128, 1, 100, 4, 4, 1), 200: (256, 1, 200, 7, 8, 2),
                   256: (256, 1, 256, 8, 0, 2), 300: (256, 2, 44, 10, 12, 3), 520: (256, 3, 8, 17, 8, 5), 1000: (256, 4, 232, 32, 8, 8)}
    assert all(2 * c % 8 == 0 for c in WIDTHS)


@pytest.mark.parametrize("c", WIDTHS)
def test_widths_inside_the_envelopes(lib, c):
    """The host answers of every entry this file runs at width c, at the shapes it runs them: the frozen encoder (autoencoder table, up to
    16 prefixes, 17 refused), the batch-statistics encoder, the parameter backward (PCRNet's table without BatchNorm) and the frozen MLP with
    its 2C-wide input."""
    import ctypes

    ae, pcr = tft._table(ae_widths(c)), tpt._table(pcr_widths(c), relu_last=True)
    bst = tab._table(ae_widths(c))
    for b, n, sizes, _ in list(SHAPES.values()) + [(PFX_B, PFX_N, PFX16, True)]:
        assert lib.snb200_frozen_encoder_supported(b, n, 5, ae, len(sizes)) == 1, (c, b, n)
        assert lib.snb200_frozen_encoder_param_backward_supported(b, n, 5, pcr, len(sizes)) == 1, (c, b, n)
        csz = (ctypes.c_int * len(sizes))(*sizes)
        assert lib.snb200_frozen_encoder_bstat_supported(b, n, 5, bst, len(sizes), csz) == 1, (c, b, n)
    assert lib.snb200_frozen_encoder_supported(PFX_B, PFX_N, 5, ae, 17) == 0
    # PCRNet's table at the shapes FrozenPCRNet / CudaPCRNet stack template and source into (2 x 32 pairs of 64 or 1024 points)
    for b, n in ((64, 64), (64, 1024), (48, 16), (2, 1000), (5, 333)):
        assert lib.snb200_frozen_encoder_supported(b, n, 5, pcr, 1) == 1
        assert lib.snb200_frozen_encoder_param_backward_supported(b, n, 5, pcr, 1) == 1
    mlp = tpt._table(mlp_widths(c))
    for b in (1, 7, 31, 32, 64):
        assert lib.snb200_frozen_mlp_supported(b, 6, mlp) == 1 and lib.snb200_frozen_mlp_param_backward_supported(b, 6, mlp) == 1


def test_frozen_pcrnet_module_route_where_2c_is_not_a_multiple_of_8(lib):
    """At C = 102 the encoder takes the table but the frozen MLP does not take a 204-wide input, so FrozenPCRNet.raw returns None and the
    wrapper runs the module (checked on the GPU by test_frozen_pcrnet_at_102_runs_the_module)."""
    assert lib.snb200_frozen_encoder_supported(64, 1024, 5, tpt._table(pcr_widths(102), relu_last=True), 1) == 1
    assert lib.snb200_frozen_mlp_supported(32, 6, tpt._table(mlp_widths(102))) == 0
    assert lib.snb200_frozen_mlp_supported(32, 6, tpt._table(mlp_widths(100))) == 1


@pytest.mark.parametrize("c", WIDTHS + (128,))
def test_cuda_ae_route_per_width(lib, monkeypatch, c):
    """CudaPointNetAE's training-mode route with the library's own envelope (asked through C tables of the module's widths: the ops
    wrappers need CUDA tensors).  The CUDA backward takes the 256 -> 128 last layer only, so every width here but 128 runs the module."""
    from samplenet_b200 import ops

    asked = []

    def supported(x, conv_specs, fc_specs):
        conv = tst._table([3] + [s["weight"].shape[0] for s in conv_specs], [1] * len(conv_specs), [1] * len(conv_specs))
        fc = tst._table([c] + [s["weight"].shape[0] for s in fc_specs], [0] * len(fc_specs), [int(s["relu"]) for s in fc_specs])
        asked.append((x.shape[0], x.shape[1]))
        return bool(lib.snb200_generator_layers_ex_supported(x.shape[0], x.shape[1], 0, len(conv_specs), conv, len(fc_specs), fc, -1, None))

    monkeypatch.setattr(ops, "generator_layers_ex_supported", supported)
    w = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=512, bneck_size=c)).train()
    conv_specs, _, _ = w._layer_stack()
    assert [s["weight"].shape[0] for s in conv_specs] == ae_widths(c)[1:]
    for b, n in ((2, 64), (5, 777), (50, 2048)):
        assert w._cuda_supported(torch.zeros(b, n, 3)) == (c == 128), (c, b, n)
    assert len(asked) == 3


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


@pytest.fixture()
def tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)


CASES = [pytest.param(c, shape, id="C%d-%s" % (c, shape)) for c in WIDTHS for shape in SHAPES]


@pytest.mark.gpu
@pytest.mark.parametrize("c,shape", CASES)
def test_eval_encoder_forward(sb, c, shape):
    b, n, sizes, dup = SHAPES[shape]
    tft.test_forward_against_float64_and_prefix_invariance(sb, "ae", b, n, dup, width=c, sizes=sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("c,shape", CASES)
def test_eval_encoder_backward(sb, c, shape):
    b, n, sizes, dup = SHAPES[shape]
    tft.test_backward_against_float64(sb, "ae", b, n, dup, width=c, sizes=sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("c,shape", CASES)
def test_batch_stats_forward(sb, c, shape):
    b, n, sizes, _ = SHAPES[shape]
    tab.test_forward_against_float64(sb, b, n, sizes, bneck=c)


@pytest.mark.gpu
@pytest.mark.parametrize("c,shape", CASES)
def test_batch_stats_backward(sb, c, shape):
    b, n, sizes, _ = SHAPES[shape]
    tab.test_backward_and_determinism(sb, b, n, sizes, bneck=c)


@pytest.mark.gpu
@pytest.mark.parametrize("c", WIDTHS)
def test_frozen_wrapper_against_the_module(sb, tf32_off, c):
    """FrozenPointNetAE's eval forward and prefixes against the float64 module, and its batch-statistics prefixes against the module, at
    the wrappers' bar."""
    net, x, sizes, _ = tft.make_case("ae", 5, 333, 11, True, c, SHAPES["ragged"][2])
    w, net64 = tasknets.FrozenPointNetAE(net), copy.deepcopy(net).double()
    with torch.no_grad():
        out, o64 = w(x), net64(x.double())
        assert ((out.double() - o64).abs().max() / o64.abs().max()).item() <= 1e-5
        pre, want = w.prefixes(x, sizes), torch.stack([net64(x[:, :s].double()) for s in sizes])
        assert ((pre.double() - want).abs().max() / want.abs().max()).item() <= 1e-5
        # batch statistics: as test_ae_batch_stats.test_wrapper_and_fallbacks_against_the_module
        got, want = w.prefixes(x, sizes, batch_stats=True), torch.stack([net(x[:, :s], batch_stats=True) for s in sizes])
        assert ((got - want).abs().max() / want.abs().max()).item() <= 1e-5


PCR_SHAPES = [pytest.param(64, 1024, [1024], id="64x1024"), pytest.param(2, 1000, [100, 517, 1000], id="2x1000-3prefixes"),
              pytest.param(5, 333, [333], id="5x333")]


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,sizes", PCR_SHAPES)
@pytest.mark.parametrize("c", WIDTHS)
def test_pcrnet_encoder_param_grads(sb, record_property, c, b, n, sizes):
    tpt.test_encoder_param_grads_against_float64(sb, record_property, b, n, sizes, widths=pcr_widths(c))


@pytest.mark.gpu
@pytest.mark.parametrize("c", WIDTHS)
def test_pcrnet_mlp_with_the_2c_input(sb, record_property, c):
    for b in (1, 31, 64):
        tfp.test_mlp_forward_and_backward_against_float64(sb, record_property, mlp_widths(c), b)
    for b in (7, 64):
        tpt.test_mlp_param_grads_against_float64(sb, record_property, mlp_widths(c), b)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["bnc", "bcn"])
@pytest.mark.parametrize("c", WIDTHS)
def test_frozen_pcrnet_against_the_module(sb, record_property, tf32_off, c, shape):
    """test_frozen_pcrnet's wrapper check at width c, after asserting that the wrapper runs the kernels there: FrozenPCRNet.raw returns
    None, and forward the module's result, outside their envelopes."""
    net, fr = tfp._frozen_pair(5, c)
    x = torch.rand(32, 64, 3, device="cuda") - 0.5
    with torch.no_grad():
        assert fr.raw(x, x) is not None
    tfp.test_wrapper_against_the_module(sb, record_property, None, shape, bottleneck=c)


@pytest.mark.gpu
def test_frozen_pcrnet_at_102_runs_the_module(sb):
    net, fr = tfp._frozen_pair(5, 102)
    g = torch.Generator().manual_seed(2)
    x0, x1 = (torch.rand(4, 64, 3, generator=g) - 0.5).cuda(), (torch.rand(4, 64, 3, generator=g) - 0.5).cuda()
    with torch.no_grad():
        assert fr.raw(x0, x1) is None
        assert all(torch.equal(a, b) for a, b in zip(fr(x0, x1), net(x0, x1)))


def _pcrnet_at(monkeypatch, c):
    """Make reg.PCRNet default to a c-wide bottleneck, for the tests that build PCRNet(input_shape=...) (RegistrationStep.create_model
    among them)."""
    class PCRNetC(reg.PCRNet):
        def __init__(self, bottleneck_size=c, input_shape="bcn"):
            super().__init__(bottleneck_size, input_shape)

    monkeypatch.setattr(reg, "PCRNet", PCRNetC)


STEP_WIDTHS = (200, 520)   # one 256-channel block, three


@pytest.mark.gpu
@pytest.mark.parametrize("c", STEP_WIDTHS)
def test_cuda_pcrnet_and_pose_loss(sb, record_property, monkeypatch, c):
    _pcrnet_at(monkeypatch, c)
    assert reg.PCRNet(input_shape="bnc").feat.conv5.out_channels == c
    tpt.test_cuda_pcrnet_and_pose_loss_against_float64(sb, record_property)


@pytest.mark.gpu
@pytest.mark.parametrize("c", STEP_WIDTHS)
def test_cuda_pcrnet_train_step(sb, record_property, monkeypatch, tf32_off, c):
    """test_pcrnet_training's train step at width c, counting the CudaPCRNet encoder and head calls: every step runs the kernels (one
    stacked encoder call and one head call for 32 pairs of equal size), none falls back to the module."""
    _pcrnet_at(monkeypatch, c)
    assert reg.RegistrationStep(sampler="none", train_pcrnet=True).create_model(cuda_task=True).net.fc1.in_features == 2 * c
    calls = {"encode": 0, "head": 0}

    def counted(name):
        fn = getattr(reg.CudaPCRNet, "_" + name)

        def call(*args):
            calls[name] += 1
            return fn(*args)
        return staticmethod(call)

    for name in calls:
        monkeypatch.setattr(reg.CudaPCRNet, "_" + name, counted(name))
    tpt.test_train_step_against_the_plain_module(sb, record_property, None)
    assert calls == {"encode": 5, "head": 5}, calls   # five steps of 32 pairs


@pytest.mark.gpu
@pytest.mark.parametrize("c", (40, 300))
def test_cuda_ae_step_takes_the_module_route(sb, tf32_off, c):
    """At a bottleneck the CUDA backward does not take, CudaPointNetAE's training step runs the wrapped module (no kernel of this project
    runs here): the route, every parameter's gradient present, and the reconstruction and its loss against the float64 module at
    test_task_training's bars."""
    ae, x = ttr._case(5, 777, 512, bneck=c)
    w, net64 = tasknets.CudaPointNetAE(copy.deepcopy(ae)).train(), copy.deepcopy(ae).double()
    rec = w(x)
    assert w.route == "module"
    loss = trainers.autoencoder_loss(rec, x, "chamfer")
    loss.backward()
    assert all(p.grad is not None for p in w.parameters())
    out64, loss64, _ = ttr._step64(net64, x, "chamfer")
    e_out = float((rec.detach().double() - out64).abs().max() / out64.abs().max())
    e_loss = abs(float(loss) - loss64) / abs(loss64)
    assert e_out < ttr.OUT_BAR and e_loss < ttr.LOSS_BAR, (e_out, e_loss)


# ------------------------------------------------------------------------------------------------------------------ GPU, the prefix cap
PFX_CASES = [pytest.param("cls", None, id="cls"), pytest.param("ae", None, id="ae-C128"), pytest.param("ae", 300, id="ae-C300")]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,c", PFX_CASES)
def test_prefix_cap_eval_encoder(sb, kind, c):
    tft.test_forward_against_float64_and_prefix_invariance(sb, kind, PFX_B, PFX_N, True, width=c, sizes=PFX16)
    tft.test_backward_against_float64(sb, kind, PFX_B, PFX_N, True, width=c, sizes=PFX16)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [128, 300])
def test_prefix_cap_batch_stats(sb, c):
    tab.test_forward_against_float64(sb, PFX_B, PFX_N, PFX16, bneck=c)
    tab.test_backward_and_determinism(sb, PFX_B, PFX_N, PFX16, bneck=c)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [1024, 300])
def test_prefix_cap_param_backward(sb, record_property, c):
    tpt.test_encoder_param_grads_against_float64(sb, record_property, PFX_B, PFX_N, PFX16, widths=pcr_widths(c))


# ------------------------------------------------------------------------------------------------------------------ GPU, buffers
# Every buffer of these calls -- inputs, layer tables, outputs, workspaces -- is carved from test_write_sets' arena, whose every other word
# holds a NaN pattern: a write outside the call's buffers, or an output element left unwritten, is reported by run_checked.
ARENA_ENC = [pytest.param(ae_widths(8), 1, 4, 300, [8, 100, 300], id="C8-tap1"),
             pytest.param(ae_widths(300), -1, 5, 333, [1, 7, 127, 128, 129, 333], id="C300"),
             pytest.param(ae_widths(1000), -1, PFX_B, PFX_N, PFX16, id="C1000-16prefixes")]


@pytest.mark.gpu
@pytest.mark.parametrize("widths,tap,b,n,sizes", ARENA_ENC)
def test_eval_encoder_writes_only_its_buffers(sb, widths, tap, b, n, sizes):
    import test_write_sets as tws

    tws.test_frozen_encoder_ex_writes_only_its_buffers(sb, tws.Arena(), widths, 0, tap, b, n, sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [8, 300])
def test_param_backward_writes_only_its_buffers(sb, c):
    tpt.test_encoder_param_backward_writes_only_its_buffers(sb, 2, 1000, [100, 517, 1000], widths=pcr_widths(c))


@pytest.mark.gpu
@pytest.mark.parametrize("c,b,n,sizes", [pytest.param(300, 5, 333, [1, 7, 127, 128, 129, 333], id="C300"),
                                         pytest.param(1000, PFX_B, PFX_N, PFX16, id="C1000-16prefixes")])
def test_batch_stats_buffers(sb, c, b, n, sizes):
    """The batch-statistics entries on arena buffers: each writes only its outputs and workspace, writes every output element, and its
    results equal those of the same call on freshly allocated buffers bit for bit, so no value read outside the inputs or before it
    was written (here a NaN) reaches them."""
    import ctypes

    import test_write_sets as tws

    lib, ops = sb._lib.lib(), sb.ops
    arena = tws.Arena()
    specs = tws.make_fc_table(arena, "ae", ae_widths(c), [1] * 5, bn=True, seed=c)
    conv, _ = ops.make_layers(specs)
    P, csz = len(sizes), (ctypes.c_int * len(sizes))(*sizes)
    assert lib.snb200_frozen_encoder_bstat_supported(b, n, 5, conv, P, csz)
    g = torch.Generator().manual_seed(n)
    x = arena.carve("x", (b, n, 3), fill=torch.rand(b, n, 3, generator=g) - 0.5)
    nstat = P * 2 * sum(ae_widths(c)[1:])
    pooled, route = arena.carve("pooled", (P, b, c)), arena.carve("route", (P, b, c), dtype=torch.int32)
    stats = arena.carve("stats", (nstat,), dtype=torch.float64)
    wsb = int(lib.snb200_frozen_encoder_bstat_workspace_bytes(b, n, 5, conv, P, csz))
    ws = arena.carve("forward_workspace", (wsb,), dtype=torch.uint8)
    gp = arena.carve("grad_pooled", (P, b, c), fill=torch.randn(P, b, c, generator=g))
    gx = arena.carve("grad_x", (b, n, 3))
    bwsb = int(lib.snb200_frozen_encoder_bstat_backward_workspace_bytes(b, n, 5, conv, P, csz))
    bws = arena.carve("backward_workspace", (bwsb,), dtype=torch.uint8)
    rc = []
    rep = tws.run_checked(arena, "frozen_encoder_bstat_forward", lambda: rc.append(lib.snb200_frozen_encoder_bstat_forward(
        b, n, x.data_ptr(), 5, conv, P, csz, pooled.data_ptr(), route.data_ptr(), stats.data_ptr(), tws._addr(ws), wsb, None)), [ws],
        full=[pooled, route, stats])
    rep += tws.run_checked(arena, "frozen_encoder_bstat_backward", lambda: rc.append(lib.snb200_frozen_encoder_bstat_backward(
        b, n, 5, conv, P, csz, pooled.data_ptr(), route.data_ptr(), stats.data_ptr(), tws._addr(ws), wsb, gp.data_ptr(), gx.data_ptr(),
        tws._addr(bws), bwsb, None)), [bws], full=[gx])
    assert rc == [0, 0], lib.snb200_last_error()
    tws.assert_clean(rep)
    p2, r2, s2, ws2 = ops.frozen_encoder_bstat_forward(x.clone(), specs, sizes)
    g2 = ops.frozen_encoder_bstat_backward(x.clone(), specs, sizes, p2, r2, s2, ws2, gp.clone())
    assert torch.equal(pooled, p2) and torch.equal(route, r2) and torch.equal(stats, s2) and torch.equal(gx, g2)
    assert bool(torch.isfinite(gx).all()) and bool(torch.isfinite(pooled).all())
