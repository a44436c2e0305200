"""The generator modules without a GPU: SampleNet and the reconstruction / classification samplers as layer-table generators.  Parameter and
state-dict order, initial parameters under a seed, the layer table handed to the kernels, the torch recompute against a stock
Conv1d / BatchNorm1d / Linear stack, the choice of training route, and the batch limit.  Nothing here launches a kernel: the route's
envelope functions are replaced, and the batch check raises before any launch."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from samplenet_b200 import samplenet
from samplenet_b200.rec_sampler import ReconstructionSampleNet
from samplenet_b200.samplenet import SampleNet
from samplenet_b200.tf_variant import ClassificationSampleNet

# named_parameters() / state_dict() keys in order, as the modules registered them before they were built on one layer-table class
SAMPLENET_PARAMETERS = [
    'conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias', 'conv4.weight', 'conv4.bias',
    'conv5.weight', 'conv5.bias', 'bn1.weight', 'bn1.bias', 'bn2.weight', 'bn2.bias', 'bn3.weight', 'bn3.bias', 'bn4.weight',
    'bn4.bias', 'bn5.weight', 'bn5.bias', 'fc1.weight', 'fc1.bias', 'fc2.weight', 'fc2.bias', 'fc3.weight', 'fc3.bias', 'fc4.weight',
    'fc4.bias', 'bn_fc1.weight', 'bn_fc1.bias', 'bn_fc2.weight', 'bn_fc2.bias', 'bn_fc3.weight', 'bn_fc3.bias', 'project._temperature'
]

SAMPLENET_STATE = [
    'conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias', 'conv4.weight', 'conv4.bias',
    'conv5.weight', 'conv5.bias', 'bn1.weight', 'bn1.bias', 'bn1.running_mean', 'bn1.running_var', 'bn1.num_batches_tracked',
    'bn2.weight', 'bn2.bias', 'bn2.running_mean', 'bn2.running_var', 'bn2.num_batches_tracked', 'bn3.weight', 'bn3.bias',
    'bn3.running_mean', 'bn3.running_var', 'bn3.num_batches_tracked', 'bn4.weight', 'bn4.bias', 'bn4.running_mean', 'bn4.running_var',
    'bn4.num_batches_tracked', 'bn5.weight', 'bn5.bias', 'bn5.running_mean', 'bn5.running_var', 'bn5.num_batches_tracked', 'fc1.weight',
    'fc1.bias', 'fc2.weight', 'fc2.bias', 'fc3.weight', 'fc3.bias', 'fc4.weight', 'fc4.bias', 'bn_fc1.weight', 'bn_fc1.bias',
    'bn_fc1.running_mean', 'bn_fc1.running_var', 'bn_fc1.num_batches_tracked', 'bn_fc2.weight', 'bn_fc2.bias', 'bn_fc2.running_mean',
    'bn_fc2.running_var', 'bn_fc2.num_batches_tracked', 'bn_fc3.weight', 'bn_fc3.bias', 'bn_fc3.running_mean', 'bn_fc3.running_var',
    'bn_fc3.num_batches_tracked', 'project._temperature'
]

RECONSTRUCTION_PARAMETERS = [
    'conv1.weight', 'conv1.bias', 'bn1.weight', 'bn1.bias', 'conv2.weight', 'conv2.bias', 'bn2.weight', 'bn2.bias', 'conv3.weight',
    'conv3.bias', 'bn3.weight', 'bn3.bias', 'conv4.weight', 'conv4.bias', 'bn4.weight', 'bn4.bias', 'conv5.weight', 'conv5.bias',
    'bn5.weight', 'bn5.bias', 'fc1.weight', 'fc1.bias', 'fc2.weight', 'fc2.bias', 'fc3.weight', 'fc3.bias', 'project._temperature'
]

RECONSTRUCTION_STATE = [
    'conv1.weight', 'conv1.bias', 'bn1.weight', 'bn1.bias', 'bn1.running_mean', 'bn1.running_var', 'bn1.num_batches_tracked',
    'conv2.weight', 'conv2.bias', 'bn2.weight', 'bn2.bias', 'bn2.running_mean', 'bn2.running_var', 'bn2.num_batches_tracked',
    'conv3.weight', 'conv3.bias', 'bn3.weight', 'bn3.bias', 'bn3.running_mean', 'bn3.running_var', 'bn3.num_batches_tracked',
    'conv4.weight', 'conv4.bias', 'bn4.weight', 'bn4.bias', 'bn4.running_mean', 'bn4.running_var', 'bn4.num_batches_tracked',
    'conv5.weight', 'conv5.bias', 'bn5.weight', 'bn5.bias', 'bn5.running_mean', 'bn5.running_var', 'bn5.num_batches_tracked',
    'fc1.weight', 'fc1.bias', 'fc2.weight', 'fc2.bias', 'fc3.weight', 'fc3.bias', 'project._temperature'
]

CLASSIFICATION_PARAMETERS = [
    'conv1.weight', 'conv1.bias', 'bn1.weight', 'bn1.bias', 'conv2.weight', 'conv2.bias', 'bn2.weight', 'bn2.bias', 'conv3.weight',
    'conv3.bias', 'bn3.weight', 'bn3.bias', 'conv4.weight', 'conv4.bias', 'bn4.weight', 'bn4.bias', 'conv5.weight', 'conv5.bias',
    'bn5.weight', 'bn5.bias', 'fc1.weight', 'fc1.bias', 'bn_fc1.weight', 'bn_fc1.bias', 'fc2.weight', 'fc2.bias', 'bn_fc2.weight',
    'bn_fc2.bias', 'fc3.weight', 'fc3.bias', 'bn_fc3.weight', 'bn_fc3.bias', 'fc4.weight', 'fc4.bias', 'bn_fc4.weight', 'bn_fc4.bias',
    'project._temperature'
]

CLASSIFICATION_STATE = [
    'conv1.weight', 'conv1.bias', 'bn1.weight', 'bn1.bias', 'bn1.running_mean', 'bn1.running_var', 'bn1.num_batches_tracked',
    'conv2.weight', 'conv2.bias', 'bn2.weight', 'bn2.bias', 'bn2.running_mean', 'bn2.running_var', 'bn2.num_batches_tracked',
    'conv3.weight', 'conv3.bias', 'bn3.weight', 'bn3.bias', 'bn3.running_mean', 'bn3.running_var', 'bn3.num_batches_tracked',
    'conv4.weight', 'conv4.bias', 'bn4.weight', 'bn4.bias', 'bn4.running_mean', 'bn4.running_var', 'bn4.num_batches_tracked',
    'conv5.weight', 'conv5.bias', 'bn5.weight', 'bn5.bias', 'bn5.running_mean', 'bn5.running_var', 'bn5.num_batches_tracked',
    'fc1.weight', 'fc1.bias', 'bn_fc1.weight', 'bn_fc1.bias', 'bn_fc1.running_mean', 'bn_fc1.running_var', 'bn_fc1.num_batches_tracked',
    'fc2.weight', 'fc2.bias', 'bn_fc2.weight', 'bn_fc2.bias', 'bn_fc2.running_mean', 'bn_fc2.running_var', 'bn_fc2.num_batches_tracked',
    'fc3.weight', 'fc3.bias', 'bn_fc3.weight', 'bn_fc3.bias', 'bn_fc3.running_mean', 'bn_fc3.running_var', 'bn_fc3.num_batches_tracked',
    'fc4.weight', 'fc4.bias', 'bn_fc4.weight', 'bn_fc4.bias', 'bn_fc4.running_mean', 'bn_fc4.running_var', 'bn_fc4.num_batches_tracked',
    'project._temperature'
]

# registration/src/samplenet.py:40-59 creates conv1..5, bn1..5, fc1..4, bn_fc1..3, then the projection
REFERENCE_MODULE_ORDER = ["conv%d" % i for i in range(1, 6)] + ["bn%d" % i for i in range(1, 6)] + ["fc%d" % i for i in range(1, 5)] + \
    ["bn_fc%d" % i for i in range(1, 4)] + ["project"]

# name -> (constructor, conv widths, FC widths, BatchNorm per FC layer, ReLU per FC layer, BatchNorm eps, momentum, parameter keys, state keys)
MODULES = {
    "samplenet64": (lambda: SampleNet(64, 128, 8), [3, 64, 64, 64, 128, 128], [128, 256, 256, 256, 192], [1, 1, 1, 0], [1, 1, 1, 0], 1e-5, 0.1,
                    SAMPLENET_PARAMETERS, SAMPLENET_STATE),
    "samplenet1024": (lambda: SampleNet(1024, 128, 8), [3, 64, 64, 64, 128, 128], [128, 256, 256, 256, 3072], [1, 1, 1, 0], [1, 1, 1, 0], 1e-5,
                      0.1, SAMPLENET_PARAMETERS, SAMPLENET_STATE),
    "reconstruction": (lambda: ReconstructionSampleNet(64), [3, 64, 128, 128, 256, 128], [128, 256, 256, 192], [0, 0, 0], [1, 1, 0], 1e-5, 0.1,
                       RECONSTRUCTION_PARAMETERS, RECONSTRUCTION_STATE),
    "classification": (lambda: ClassificationSampleNet(32), [3, 64, 64, 64, 128, 128], [128, 256, 256, 256, 96], [1, 1, 1, 1], [1, 1, 1, 0],
                       1e-3, 0.5, CLASSIFICATION_PARAMETERS, CLASSIFICATION_STATE),
}


@pytest.mark.parametrize("name", sorted(MODULES))
def test_parameter_and_state_order(name):
    make, *_, params, state = MODULES[name]
    net = make()
    assert [k for k, _ in net.named_parameters()] == params
    assert list(net.state_dict()) == state
    if name.startswith("samplenet"):
        order = [k.split(".")[0] for k, _ in net.named_parameters()]
        assert [m for i, m in enumerate(order) if m not in order[:i]] == REFERENCE_MODULE_ORDER


@pytest.mark.parametrize("name", sorted(MODULES))
def test_initial_parameters_follow_the_seed(name):
    """Each Conv1d / Linear draws its initial values in layer order (conv1..., fc1...); BatchNorm draws none."""
    make, cw, fw = MODULES[name][:3]
    torch.manual_seed(11)
    net = make()
    torch.manual_seed(11)
    convs = [nn.Conv1d(cw[i], cw[i + 1], 1) for i in range(len(cw) - 1)]
    fcs = [nn.Linear(fw[i], fw[i + 1]) for i in range(len(fw) - 1)]
    for (lin, bn), want in zip(net._convs() + net._fcs(), convs + fcs):
        assert torch.equal(lin.weight, want.weight) and torch.equal(lin.bias, want.bias)
        if bn is not None:
            assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))
    assert torch.equal(net.project._temperature, torch.tensor(1.0))


@pytest.mark.parametrize("name", sorted(MODULES))
def test_layer_specs(name):
    make, cw, fw, fbn, frelu, eps, momentum = MODULES[name][:7]
    net = make()
    conv_specs, fc_specs = net._layer_specs()
    assert [s["weight"].shape[:2] for s in conv_specs] == [(cw[i + 1], cw[i]) for i in range(len(cw) - 1)]
    assert [s["weight"].shape for s in fc_specs] == [(fw[i + 1], fw[i]) for i in range(len(fw) - 1)]
    assert [s["relu"] for s in conv_specs + fc_specs] == [True] * (len(cw) - 1) + [bool(r) for r in frelu]
    assert [s["bn"] is not None for s in conv_specs + fc_specs] == [True] * (len(cw) - 1) + [bool(b) for b in fbn]
    for spec, (lin, bn) in zip(conv_specs + fc_specs, net._convs() + net._fcs()):
        assert spec["weight"] is lin.weight and spec["bias"] is lin.bias
        if bn is not None:
            assert all(t is m for t, m in zip(spec["bn"], (bn.weight, bn.bias, bn.running_mean, bn.running_var, None, None, bn.num_batches_tracked))
                       if m is not None)
            assert spec["bn"][4:6] == (eps, momentum)


def _stock(net, x_bcn, training):
    """The same layer stack as stock modules (on a copy: training-mode BatchNorm updates its running statistics)."""
    net = copy.deepcopy(net).train(training)
    y = x_bcn
    for lin, bn in net._convs():
        y = F.relu(bn(lin(y)))
    y = y.max(dim=2)[0]
    for (lin, bn), relu in zip(net._fcs(), net.fc_relu):
        y = lin(y)
        if bn is not None:
            y = bn(y)
        if relu:
            y = F.relu(y)
    return y


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("layout", ["bnc", "bcn"])
@pytest.mark.parametrize("name", sorted(MODULES))
def test_torch_generator_matches_stock_modules(name, layout, training):
    torch.manual_seed(3)
    net = MODULES[name][0]().double()
    with torch.no_grad():
        for _, bn in net._convs() + net._fcs():
            if bn is not None:
                bn.weight.normal_(1.0, 0.3), bn.bias.normal_(0.0, 0.3), bn.running_mean.normal_(0.0, 0.2), bn.running_var.uniform_(0.5, 2.0)
    x = torch.rand(5, 3, 200, dtype=torch.float64) - 0.5
    ps = dict(net._generator_named_parameters())
    got = net._torch_generator(x.permute(0, 2, 1).contiguous() if layout == "bnc" else x, layout, training, ps)
    torch.testing.assert_close(got, _stock(net, x, training), rtol=1e-12, atol=1e-12)


def _envelopes(monkeypatch, fused, layers):
    """Replace the two CUDA routes' envelope functions by constant answers."""
    for route, ok in (("fused", fused), ("layers", layers)):
        monkeypatch.setitem(samplenet._ROUTE_OPS, route, (lambda *a, ok=ok: ok,) + samplenet._ROUTE_OPS[route][1:])


def _route(net, x=None, training=True):
    x = torch.zeros(4, 256, 3) if x is None else x
    return net._route(x, "bnc", *net._layer_specs(), training)


@pytest.mark.parametrize("name", sorted(MODULES))
def test_route(monkeypatch, name):
    net = MODULES[name][0]()
    sampler = not name.startswith("samplenet")
    for fused, layers, want in ((True, True, "fused"), (True, False, "fused"), (False, True, "layers" if sampler else "torch"),
                                (False, False, "torch")):
        _envelopes(monkeypatch, fused, layers)
        assert _route(net) == want, (fused, layers)
    _envelopes(monkeypatch, True, True)
    assert _route(net, training=False) == "torch"
    assert _route(net, x=torch.zeros(4, 256, 3, requires_grad=True)) == "torch"
    for attr, value in (("generator_precision", "fp32"), ("generator_backward", "torch")):
        other = copy.deepcopy(net)
        setattr(other, attr, value)
        assert _route(other) == "torch", attr
    assert net.generator_route is None


@pytest.mark.parametrize("make,shape", [(lambda: SampleNet(64, 128, 8), (257, 3, 64)), (lambda: ReconstructionSampleNet(64), (257, 64, 3)),
                                        (lambda: ClassificationSampleNet(32), (257, 64, 3))])
def test_training_batch_limit(make, shape):
    net = make().train()
    with pytest.raises(RuntimeError, match="^%s: training-mode batches are limited to 256 clouds" % type(net).__name__):
        net(torch.zeros(*shape))
