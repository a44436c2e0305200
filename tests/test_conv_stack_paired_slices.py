"""The multi-slice conv stack runs its 64-wide layers (K <= 64, c_out <= 64, not the last) over two of a CTA's slices per pass, one per half
of the CTA (csrc/conv_stack.cu, CsLayer::pair); with an odd number of slices the last one is a pass of its own.  Which slice of a pass sits
in which half of the staging buffer, and which thread re-reads which rows from L2, depends on the slice count, the walking direction and
the neighbouring layers being paired or not.  These shapes mix pairs and single passes in one layer, end a batch inside a pair, and put
paired and serial layers next to each other both ways; each is checked against the per-layer tensor-core kernels and the exact-fp32 path
at the tolerances of test_conv_stack_onchip_slices.py, with repeated launches bit for bit."""
import numpy as np
import pytest
import torch

from test_conv_stack_onchip_slices import HEADLINE, _check, _n, _shape

pytestmark = pytest.mark.gpu

# 128 -> 64 (serial, K = 128) feeds 64 -> 64 (paired), which feeds 64 -> 128 (serial, K = 64, not the last layer)
MIXED = [3, 64, 128, 64, 64, 128, 128]


@pytest.fixture(scope="module")
def sb():
    import samplenet_b200

    samplenet_b200._lib.lib()  # fail loudly if the CUDA library is missing
    return samplenet_b200


@pytest.mark.parametrize("per_cta", [3, 5])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_odd_slice_counts(sb, per_cta, training):
    """pairs and a single pass in the same layer, walked forwards and backwards"""
    b, p = _shape(sb, per_cta, 1024, ragged=False)
    assert p["per_cta"] == per_cta
    torch.manual_seed(50 + per_cta)
    x = torch.rand(b, 1024, 3, device="cuda") - 0.5
    _check(sb, x, "bnc", HEADLINE, training, seed=50 + per_cta)


@pytest.mark.parametrize("per_cta,fill", [(2, 0.75), (4, 0.75)])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_ragged_last_pair(sb, per_cta, fill, training):
    """the batch ends inside the second slice of a CTA's last pair"""
    b, p = _shape(sb, per_cta, 1000, ragged=True, fill=fill)
    assert p["ragged"] and p["per_cta"] == per_cta
    torch.manual_seed(60 + per_cta)
    x = torch.rand(b, 1000, 3, device="cuda") - 0.5
    _check(sb, x, "bnc", HEADLINE, training, seed=60 + per_cta)


@pytest.mark.parametrize("per_cta", [2, 3, 4])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_paired_and_serial_neighbours(sb, per_cta, training):
    """a serial layer feeding a paired one and a paired one feeding a serial 64-wide-in layer that is not the last"""
    b, _ = _shape(sb, per_cta, 1024, ragged=False)
    torch.manual_seed(70 + per_cta)
    x = torch.rand(b, 1024, 3, device="cuda") - 0.5
    _check(sb, x, "bnc", MIXED, training, seed=70 + per_cta)


def test_saved_outputs_and_backward(sb):
    """training with gradients at an odd slice count: every layer's saved raw outputs against the per-layer training forward, the CUDA
    backward on top of each, and a second launch bit for bit"""
    per_cta, n = 3, 1024
    b, p = _shape(sb, per_cta, n, ragged=False)
    assert b <= 64 and p["per_cta"] == per_cta   # (the CUDA backward's envelope)
    torch.manual_seed(80 + per_cta)
    net = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train()
    with torch.no_grad():
        for bn in [net.bn1, net.bn2, net.bn3, net.bn4, net.bn5]:
            bn.weight.copy_(1 + 0.3 * torch.randn_like(bn.weight)); bn.bias.copy_(0.2 * torch.randn_like(bn.bias))
    x = torch.rand(b, n, 3, device="cuda") - 0.5
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    res = []
    for fwd, bwd in ((sb.ops.generator_train_forward, sb.ops.generator_backward), (sb.ops.generator_train_forward, sb.ops.generator_backward),
                     (sb.ops.generator_layers_train_forward, sb.ops.generator_layers_backward)):
        net.load_state_dict(sd)
        conv, fc = net._layer_specs()
        out, feat, saved = fwd(x, "bnc", conv, fc)
        grad_out = torch.randn(out.shape, generator=torch.Generator().manual_seed(90 + per_cta)).cuda()
        grads = bwd(x, "bnc", conv, fc, saved, grad_out)
        torch.cuda.synchronize()
        res.append((out.clone(), feat.clone(), [z.clone() for z in saved[0]], [{k: v.clone() for k, v in g.items() if v is not None} for g in grads]))
    (out, feat, zs, gr), (out2, feat2, zs2, gr2), (out3, feat3, zs3, gr3) = res
    assert torch.equal(out, out2) and torch.equal(feat, feat2)
    assert all(torch.equal(a, c) for a, c in zip(zs, zs2))
    assert all(torch.equal(a[k], c[k]) for a, c in zip(gr, gr2) for k in a)
    np.testing.assert_allclose(_n(feat), _n(feat3), rtol=3e-4, atol=3e-5)
    np.testing.assert_allclose(_n(out), _n(out3), rtol=2e-3, atol=2e-4)
    for l, (a, c) in enumerate(zip(zs, zs3)):
        np.testing.assert_allclose(_n(a), _n(c), rtol=3e-4, atol=3e-5, err_msg="layer %d" % (l + 1))
    for l, (a, c) in enumerate(zip(gr, gr3)):
        # (zero gradients, so rounding noise only: a conv bias in front of a training BatchNorm, and the last conv layer's BatchNorm shift,
        # which moves every cloud's pooled feature alike and is taken out again by the first FC layer's BatchNorm)
        for k in ("weight", "bn_weight", "bn_bias"):
            if k not in a or (k == "bn_bias" and l == 4):
                continue
            scale = float(c[k].abs().max()) + 1e-12
            np.testing.assert_allclose(_n(a[k]) / scale, _n(c[k]) / scale, rtol=0, atol=2e-3, err_msg="layer %d %s" % (l + 1, k))
