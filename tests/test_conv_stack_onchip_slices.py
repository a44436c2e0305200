"""The multi-slice conv stack keeps up to two slices per CTA on chip between layers (csrc/conv_stack.cu, CsLayer::keep): the last slice a
layer visits stays in the accumulator staging buffer, the slice before it in the weight matrix's spare columns 64..127 while both layers
have K <= 64, and the rest go through L2.  The layers walk their slices forwards and backwards in turn, so which slice sits where depends on
the number of slices per CTA, the layer table, the mode and the batch's last, partly filled slice.  Every placement here is checked against
the per-layer tensor-core kernels and the exact-fp32 CUDA-core path at the tolerances of test_gpu_parity.py, and a second launch must
return the same bits."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HEADLINE = [3, 64, 64, 64, 128, 128]
MID128_K32 = [3, 32, 128, 64, 32, 128]   # a 128-wide middle layer (no spare columns around it) and K = 32 layers on either side


@pytest.fixture(scope="module")
def sb():
    import samplenet_b200

    samplenet_b200._lib.lib()  # fail loudly if the CUDA library is missing
    return samplenet_b200


def _n(t):
    return t.detach().cpu().numpy()


def _partition(sb, b, n):
    v = [ctypes.c_int() for _ in range(5)]
    sb._lib.check(sb._lib.lib().snb200_debug_conv_stack_partition(b, n, *[ctypes.byref(t) for t in v]), "debug_conv_stack_partition")
    ppc, slices, grid, per_cta, _ = (t.value for t in v)
    return dict(ppc=ppc, slices=slices, grid=grid, per_cta=per_cta, ragged=(b * n) % ppc != 0)


def _shape(sb, per_cta, n, ragged, fill=0.75):
    """a batch of n-point clouds whose partition on this device gives per_cta slices to the busiest CTA, with the last round of slices about
    `fill` full (so some CTAs have one slice fewer), and a partly filled last slice or none"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for b in range(max(1, round((per_cta - 1 + fill) * sms * 128 / n)), 1024):
        p = _partition(sb, b, n)
        if p["per_cta"] == per_cta and p["ragged"] == ragged:
            return b, p
    pytest.fail("no batch of %d-point clouds gives %d slices per CTA (ragged=%s)" % (n, per_cta, ragged))


def _params(widths, seed):
    """conv layers (BatchNorm + ReLU each) of the given widths and one FC layer with BatchNorm, on the GPU"""
    g = torch.Generator().manual_seed(seed)

    def layer(ci, co):
        return dict(weight=torch.randn(co, ci, generator=g) / ci ** 0.5, bias=0.1 * torch.randn(co, generator=g),
                    gamma=1 + 0.3 * torch.randn(co, generator=g), beta=0.2 * torch.randn(co, generator=g),
                    mean=0.1 * torch.randn(co, generator=g), var=0.5 + torch.rand(co, generator=g))

    conv = [{k: v.cuda() for k, v in layer(widths[i], widths[i + 1]).items()} for i in range(len(widths) - 1)]
    fc = [{k: v.cuda() for k, v in layer(widths[-1], 40).items()}]
    return conv, fc


def _specs(params, relu_last=True):
    """layer specs over fresh copies of the running statistics (training launches update them in place)"""
    return [dict(weight=p["weight"], bias=p["bias"], bn=(p["gamma"], p["beta"], p["mean"].clone(), p["var"].clone(), 1e-5, 0.1),
                 relu=relu_last or i + 1 < len(params)) for i, p in enumerate(params)]


def _check(sb, x, layout, widths, training, seed):
    conv_p, fc_p = _params(widths, seed)
    runs = []
    for kw in (dict(), dict(), dict(per_layer_kernels=True), dict(exact_fp32=True)):
        conv, fc = _specs(conv_p), _specs(fc_p, relu_last=False)
        out, feat = sb.ops.generator_forward(x, layout, conv, fc, training, **kw)
        runs.append((out.clone(), feat.clone(), [s["bn"][2] for s in conv + fc] + [s["bn"][3] for s in conv + fc]))
    (out, feat, stats), (out2, feat2, stats2) = runs[:2]
    assert torch.isfinite(out).all() and torch.isfinite(feat).all()
    assert torch.equal(out, out2) and torch.equal(feat, feat2)
    assert all(torch.equal(a, b) for a, b in zip(stats, stats2))
    for o, f, st in runs[2:]:
        np.testing.assert_allclose(_n(feat), _n(f), rtol=3e-4, atol=3e-5)
        np.testing.assert_allclose(_n(out), _n(o), rtol=2e-3, atol=2e-4)
        for a, b in zip(stats, st):
            np.testing.assert_allclose(_n(a), _n(b), rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("per_cta", [1, 2, 3, 8])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_slices_per_cta(sb, per_cta, training):
    """1 (the single-slice kernel), 2 (the headline: held slice + spare columns, one deferred park), 3 (one slice through L2) and 8 slices
    per CTA, full slices"""
    b, p = _shape(sb, per_cta, 1024, ragged=False)
    assert p["per_cta"] == per_cta
    torch.manual_seed(per_cta)
    x = torch.rand(b, 1024, 3, device="cuda") - 0.5
    _check(sb, x, "bnc", HEADLINE, training, seed=per_cta)


@pytest.mark.parametrize("per_cta,fill", [(2, 0.1), (3, 0.75)])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_ragged_last_slice(sb, per_cta, fill, training):
    """a batch that ends inside its last slice, and clouds that straddle slices; just over one round of slices, the slices have 96 points
    (24 per thread)"""
    b, p = _shape(sb, per_cta, 1000, ragged=True, fill=fill)
    assert p["ragged"] and p["per_cta"] == per_cta
    torch.manual_seed(10 + per_cta)
    x = torch.rand(b, 1000, 3, device="cuda") - 0.5
    _check(sb, x, "bnc", HEADLINE, training, seed=10 + per_cta)


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_bcn_input(sb, training):
    b, _ = _shape(sb, 2, 1024, ragged=False)
    torch.manual_seed(20)
    x = torch.rand(b, 3, 1024, device="cuda") - 0.5
    _check(sb, x, "bcn", HEADLINE, training, seed=20)


@pytest.mark.parametrize("per_cta", [2, 3])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_wide_middle_layer_and_k32(sb, per_cta, training):
    """widths 32, 128, 64, 32, 128: the spare columns hold a slice only between the 64 -> 32 and 32 -> 128 layers; around the 128-wide
    layer only the staging buffer does"""
    b, _ = _shape(sb, per_cta, 1024, ragged=False)
    torch.manual_seed(30 + per_cta)
    x = torch.rand(b, 1024, 3, device="cuda") - 0.5
    _check(sb, x, "bnc", MID128_K32, training, seed=30 + per_cta)


@pytest.mark.parametrize("per_cta,ragged", [(2, False), (3, True)])
def test_training_forward_with_saved_outputs(sb, per_cta, ragged):
    """training with gradients: every slice's raw outputs are still written for the backward pass while the next layer reads them from
    chip; the saved outputs, the pooled feature and the output against the per-layer training forward, and a second launch bit for bit"""
    n = 1000 if ragged else 1024
    b, p = _shape(sb, per_cta, n, ragged)
    assert b <= 64 and p["per_cta"] == per_cta
    torch.manual_seed(40 + per_cta)
    net = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train()
    with torch.no_grad():
        for bn in [net.bn1, net.bn2, net.bn3, net.bn4, net.bn5]:
            bn.weight.copy_(1 + 0.3 * torch.randn_like(bn.weight)); bn.bias.copy_(0.2 * torch.randn_like(bn.bias))
    x = torch.rand(b, n, 3, device="cuda") - 0.5
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    res = []
    for fwd in (sb.ops.generator_train_forward, sb.ops.generator_train_forward, sb.ops.generator_layers_train_forward):
        net.load_state_dict(sd)
        conv, fc = net._layer_specs()
        out, feat, (zs, _) = fwd(x, "bnc", conv, fc)
        res.append((out.clone(), feat.clone(), [z.clone() for z in zs]))
    (out, feat, zs), (out2, feat2, zs2), (out3, feat3, zs3) = res
    assert torch.equal(out, out2) and torch.equal(feat, feat2)
    assert all(torch.equal(a, c) for a, c in zip(zs, zs2))
    np.testing.assert_allclose(_n(feat), _n(feat3), rtol=3e-4, atol=3e-5)
    np.testing.assert_allclose(_n(out), _n(out3), rtol=2e-3, atol=2e-4)
    for l, (a, c) in enumerate(zip(zs, zs3)):
        np.testing.assert_allclose(_n(a), _n(c), rtol=3e-4, atol=3e-5, err_msg="layer %d" % (l + 1))
