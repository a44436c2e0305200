"""TensorFlow-variant SampleNet generator (classification) on this package's kernels, fed from TF-named variables.

The classification trainer builds the generator with `tf_util` layers under `tf.variable_scope("sampler")`
(classification/train_samplenet.py:154-161, models/samplenet_model.py:22-112): five 1x1 "conv2d" layers (the first with a [1,3]
kernel over the xyz axis), a max-pool over the points and four fully connected layers, ALL of them -- including the last one,
`fc14b`, which has no activation -- followed by `batch_norm_template` (eps 1e-3, exponential moving averages of the batch moments,
tf_util.py:478-519).  That differs from the registration (torch) class in three ways the torch `SampleNet` cannot express -- BatchNorm on
the output layer, eps, and the variable layout -- while the C ABI's layer table can, so this module only translates names and layouts:

    TF variable (scope "sampler/")                               shape               ->  layer-table entry
    conv1/weights                                                 [1, 3, 1, 64]       ->  weight (64, 3)
    conv{2..5}/weights                                            [1, 1, Cin, Cout]   ->  weight (Cout, Cin)
    fc1{1..4}b/weights                                            [Cin, Cout]         ->  weight (Cout, Cin)
    <layer>/biases                                                [Cout]              ->  bias
    <layer>/bn/gamma, <layer>/bn/beta                             [Cout]              ->  bn weight / bias
    <layer>/bn/.../moments/Squeeze/ExponentialMovingAverage       [Cout]              ->  running mean
    <layer>/bn/.../moments/Squeeze_1/ExponentialMovingAverage     [Cout]              ->  running var
    temperature (soft_projection.py:33-38)                        []                  ->  SoftProjection temperature

`bn_decay` d of the TF graph is torch's momentum 1 - d.  One documented difference: TF averages the BIASED batch variance, the
kernels (like torch) fold the UNBIASED one into the running variance; training-mode outputs (batch statistics) and eval-mode
outputs (given running statistics) are unaffected.
"""
import re

import numpy as np
import torch
from torch import nn

from . import ops, sputils, tf_ops
from .samplenet import LayerTableGenerator

CONV_SCOPES = ("conv1", "conv2", "conv3", "conv4", "conv5")
FC_SCOPES = ("fc11b", "fc12b", "fc13b", "fc14b")
BN_EPS = 1e-3  # tf_util.py:518

_EMA_MEAN = re.compile(r"moments/Squeeze/ExponentialMovingAverage$")
_EMA_VAR = re.compile(r"moments/Squeeze_1/ExponentialMovingAverage$")


def _strip(name):
    return name[:-2] if name.endswith(":0") else name


def _find(variables, scope, layer, leaf):
    """`leaf` is a literal suffix below `<scope>/<layer>/` or a compiled pattern for the EMA shadow variables, whose names repeat
    the scope (`conv1/bn/conv1/bn/moments/Squeeze/ExponentialMovingAverage` in checkpoints written by the reference)."""
    prefix = (scope.rstrip("/") + "/" if scope else "") + layer + "/"
    hits = []
    for k in variables:
        kk = _strip(k)
        if not kk.startswith(prefix):
            continue
        rest = kk[len(prefix):]
        if (leaf.search(rest) if hasattr(leaf, "search") else rest == leaf):
            hits.append(k)
    if len(hits) > 1:
        raise KeyError("ambiguous TF variable for %s%s: %s" % (prefix, getattr(leaf, "pattern", leaf), hits))
    return variables[hits[0]] if hits else None


def layer_tables_from_tf(variables, scope="sampler", conv_scopes=CONV_SCOPES, fc_scopes=FC_SCOPES):
    """variables: mapping TF variable name -> numpy array (e.g. from tf.train.load_checkpoint / np.load).
    Returns (conv, fc): lists of dict(weight (Cout,Cin), bias, gamma, beta, mean, var, relu) in numpy, torch layout."""
    def one(layer, kind, relu):
        w = _find(variables, scope, layer, "weights")
        if w is None:
            raise KeyError("TF variable %s/%s/weights not found" % (scope, layer))
        w = np.asarray(w, dtype=np.float32)
        if kind == "conv":
            if w.ndim != 4 or w.shape[0] != 1:
                raise ValueError("%s/weights: expected a [1, kw, Cin, Cout] kernel, got %s" % (layer, w.shape))
            if w.shape[1] == 3 and w.shape[2] == 1:          # conv1: [1,3] kernel over the xyz axis of the (B,N,3,1) image
                w2 = w[0, :, 0, :].T
            elif w.shape[1] == 1:
                w2 = w[0, 0].T
            else:
                raise ValueError("%s/weights: unsupported kernel shape %s" % (layer, w.shape))
        else:
            if w.ndim != 2:
                raise ValueError("%s/weights: expected [Cin, Cout], got %s" % (layer, w.shape))
            w2 = w.T
        c_out = w2.shape[0]
        b = _find(variables, scope, layer, "biases")
        d = dict(weight=np.ascontiguousarray(w2), bias=np.zeros(c_out, np.float32) if b is None else np.asarray(b, np.float32), relu=relu)
        g = _find(variables, scope, layer, "bn/gamma")
        if g is not None:
            be = _find(variables, scope, layer, "bn/beta")
            mu = _find(variables, scope, layer, _EMA_MEAN)
            va = _find(variables, scope, layer, _EMA_VAR)
            d.update(gamma=np.asarray(g, np.float32), beta=np.zeros(c_out, np.float32) if be is None else np.asarray(be, np.float32),
                     mean=np.zeros(c_out, np.float32) if mu is None else np.asarray(mu, np.float32),
                     var=np.ones(c_out, np.float32) if va is None else np.asarray(va, np.float32))
        for k, v in d.items():
            if k != "relu" and k != "weight" and v.shape != (c_out,):
                raise ValueError("%s: %s has shape %s, expected (%d,)" % (layer, k, v.shape, c_out))
        return d

    conv = [one(s, "conv", True) for s in conv_scopes]
    fc = [one(s, "fc", i + 1 < len(fc_scopes)) for i, s in enumerate(fc_scopes)]   # fc14b: activation_fn=None (samplenet_model.py:100-108)
    for a, b in zip((conv + fc)[:-1], (conv + fc)[1:]):
        if b["weight"].shape[1] != a["weight"].shape[0]:
            raise ValueError("layer widths do not chain: %s -> %s" % (a["weight"].shape, b["weight"].shape))
    if conv[0]["weight"].shape[1] != 3:
        raise ValueError("conv1 must read xyz")
    return conv, fc


class TFSampleNetGenerator(nn.Module):
    """`get_model` of classification/models/samplenet_model.py as a torch module over `snb200_generator_forward`:
    `forward(point_cloud (B,N,3)) -> (B, num_output_points, 3)`.  Forward only (the TF trainers' optimiser is not restated)."""

    def __init__(self, conv, fc, bn_decay=0.5):
        super().__init__()
        self.n_conv, self.n_fc = len(conv), len(fc)
        self.momentum = 1.0 - float(bn_decay)
        for i, d in enumerate(conv + fc):
            self.register_parameter("l%d_weight" % i, nn.Parameter(torch.from_numpy(d["weight"]).clone(), requires_grad=False))
            self.register_parameter("l%d_bias" % i, nn.Parameter(torch.from_numpy(d["bias"]).clone(), requires_grad=False))
            setattr(self, "l%d_relu" % i, bool(d["relu"]))
            setattr(self, "l%d_bn" % i, "gamma" in d)
            if "gamma" in d:
                self.register_parameter("l%d_gamma" % i, nn.Parameter(torch.from_numpy(d["gamma"]).clone(), requires_grad=False))
                self.register_parameter("l%d_beta" % i, nn.Parameter(torch.from_numpy(d["beta"]).clone(), requires_grad=False))
                self.register_buffer("l%d_mean" % i, torch.from_numpy(d["mean"]).clone())
                self.register_buffer("l%d_var" % i, torch.from_numpy(d["var"]).clone())
        self.num_output_points = fc[-1]["weight"].shape[0] // 3

    @classmethod
    def from_tf_variables(cls, variables, scope="sampler", bn_decay=0.5):
        conv, fc = layer_tables_from_tf(variables, scope)
        return cls(conv, fc, bn_decay)

    def specs(self):
        out = []
        for i in range(self.n_conv + self.n_fc):
            bn = None
            if getattr(self, "l%d_bn" % i):
                bn = (getattr(self, "l%d_gamma" % i), getattr(self, "l%d_beta" % i), getattr(self, "l%d_mean" % i), getattr(self, "l%d_var" % i),
                      BN_EPS, self.momentum)
            out.append(dict(weight=getattr(self, "l%d_weight" % i), bias=getattr(self, "l%d_bias" % i), bn=bn, relu=getattr(self, "l%d_relu" % i)))
        return out[:self.n_conv], out[self.n_conv:]

    def forward(self, point_cloud):
        conv, fc = self.specs()
        # TF reshapes the (B, 3M) output to (B, M, 3): consecutive triples are points -- no transposed store
        out, _ = ops.generator_forward(point_cloud, "bnc", conv, fc, self.training, 0)
        return out.view(out.shape[0], -1, 3)


class ClassificationSampleNet(LayerTableGenerator):
    """The classification sampler (`get_model` of classification/models/samplenet_model.py:22-112 with its SoftProjection,
    classification/soft_projection.py) as a trainable module: 1x1 convs 64-64-64-128-bottleneck and FC 256-256-256-3M, BatchNorm
    (eps 1e-3, momentum 1 - bn_decay) on all nine layers, ReLU on all but `fc14b`; sigma = T^2.  `forward(point_cloud (B,N,3))` returns
    (simplified (B, M, 3), projected (B, M, 3)) in training and (simplified, matched) in eval, where matched are the input points nearest
    to the generated ones, completed by farthest point sampling.  `fc14b`'s BatchNorm without ReLU is outside the persistent kernel:
    training runs the per-layer CUDA path.  Parameters: random init, or the sampler scope of a TF checkpoint (`from_tf_variables`)."""

    def __init__(self, num_out_points, bottleneck_size=128, group_size=7, initial_temperature=1.0, is_temperature_trainable=True, bn_decay=0.5):
        m = num_out_points
        super().__init__([3, 64, 64, 64, 128, bottleneck_size], [bottleneck_size, 256, 256, 256, 3 * m], fc_bn=[True] * 4,
                         fc_relu=[True, True, True, False], bn_eps=BN_EPS, bn_momentum=1.0 - float(bn_decay))
        self.num_out_points = m
        self.name = "samplenet"
        self.complete_fps = True
        self.project = tf_ops.SoftProjection(group_size, initial_temperature, is_temperature_trainable, sigma_mode="cls")

    @classmethod
    def from_tf_variables(cls, variables, group_size=7, scope="sampler", bn_decay=0.5, initial_temperature=1.0, is_temperature_trainable=True):
        """Same variables as TFSampleNetGenerator.from_tf_variables (layer_tables_from_tf); the widths are read from them."""
        conv, fc = layer_tables_from_tf(variables, scope)
        if len(conv) != 5 or len(fc) != 4 or not all("gamma" in d for d in conv + fc):
            raise ValueError("the classification sampler has 5 conv and 4 FC layers, each with BatchNorm")
        net = cls(fc[-1]["weight"].shape[0] // 3, conv[-1]["weight"].shape[0], group_size, initial_temperature, is_temperature_trainable, bn_decay)
        with torch.no_grad():
            for (lin, bn), d in zip(net._convs() + net._fcs(), conv + fc):
                if tuple(lin.weight.shape[:2]) != d["weight"].shape:
                    raise ValueError("layer width %s does not match the module's %s" % (d["weight"].shape, tuple(lin.weight.shape[:2])))
                lin.weight.copy_(torch.from_numpy(d["weight"]).view_as(lin.weight))
                lin.bias.copy_(torch.from_numpy(d["bias"]))
                bn.weight.copy_(torch.from_numpy(d["gamma"])); bn.bias.copy_(torch.from_numpy(d["beta"]))
                bn.running_mean.copy_(torch.from_numpy(d["mean"])); bn.running_var.copy_(torch.from_numpy(d["var"]))
        return net

    def forward(self, point_cloud):
        x, simp = self._generate_points(point_cloud)
        if self.training:
            proj, _, _ = self.project(x, simp)
            return simp, proj
        _, idx, _, _ = ops.nn_distance_forward(simp.detach(), x.detach())
        return simp, sputils.nn_matching_cuda(x.detach(), idx, self.num_out_points, complete_fps=self.complete_fps)

    def get_simplification_loss(self, ref_pc, samp_pc, pc_size, gamma=1, delta=0):
        """samplenet_model.py:176-188; 0 in eval mode."""
        if not self.training:
            return torch.tensor(0).to(ref_pc)
        return tf_ops.get_simplification_loss(ref_pc, samp_pc, pc_size, gamma, delta)
