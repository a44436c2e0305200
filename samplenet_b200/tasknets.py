"""Task networks of the classification and reconstruction trainers, restated in stock torch ops (SURVEY.md 8f rank 1).  They are CALLERS
of the hot path -- frozen while the sampler trains (train_samplenet.py:227-232, sampler/train_samplenet.py:100-118) -- so they stay plain
torch modules; only the layer stacks' structure, widths, BatchNorm placement and eps follow the reference:

    PointNetCls   classification/models/pointnet_cls_basic.py:55-136 (vanilla PointNet: 3-64-64-64-128-1024 1x1 convs with BN, max-pool,
                  fc 512 - fc 256 - dropout(keep 0.7) - fc 40; tf_util batch norm eps 1e-3); get_loss = mean sparse softmax cross-entropy
    PointNetClsTransforms  classification/models/pointnet_cls.py + transform_nets.py (PointNet with its input and feature transform nets,
                  the classification trainers' default classifier); get_loss adds reg_weight * l2_loss(T2 T2^T - I)
    PointNetAE    reconstruction/src/ae_templates.py:24-37 + encoders_decoders.py (encoder 64-128-128-256-bneck 1x1 convs with BN + ReLU and
                  max symmetry; decoder FC 256-256-n*3, ReLU between, no BN), output reshaped to (B, n, 3)
"""
import torch
import torch.nn as nn
import torch.nn.functional as F


class PointNetCls(nn.Module):
    def __init__(self, num_classes=40, bn_eps=1e-3):
        super().__init__()
        w = [3, 64, 64, 64, 128, 1024]
        self.convs = nn.ModuleList([nn.Conv1d(w[i], w[i + 1], 1) for i in range(5)])
        self.bns = nn.ModuleList([nn.BatchNorm1d(w[i + 1], eps=bn_eps) for i in range(5)])
        self.fc1, self.bn_fc1 = nn.Linear(1024, 512), nn.BatchNorm1d(512, eps=bn_eps)
        self.fc2, self.bn_fc2 = nn.Linear(512, 256), nn.BatchNorm1d(256, eps=bn_eps)
        self.dp1 = nn.Dropout(p=0.3)
        self.fc3 = nn.Linear(256, num_classes)

    def forward(self, point_cloud):
        """point_cloud (B, N, 3) -> (logits (B, classes), end_points)."""
        y = point_cloud.permute(0, 2, 1)
        for conv, bn in zip(self.convs, self.bns):
            y = F.relu(bn(conv(y)))
        end_points = {"critical_set_idx": torch.argmax(y, dim=2)}
        y = torch.max(y, 2)[0]
        end_points["GFV"] = y
        v = self.descriptor(y)
        end_points["retrieval_vectors"] = v
        return self.fc3(v), end_points

    def descriptor(self, y):
        """fc3's input from the pooled feature (B, 1024): dp1(relu(bn_fc2(fc2(relu(bn_fc1(fc1(y))))))), (B, 256).  pointnet_cls_basic.py has
        no retrieval end point; this is the layer pointnet_cls.py:111 exports as "retrieval_vectors", and in eval mode (dropout the
        identity) it is relu(bn_fc2(fc2(.)))."""
        y = F.relu(self.bn_fc1(self.fc1(y)))
        return self.dp1(F.relu(self.bn_fc2(self.fc2(y))))

    def head(self, y):
        """The FC head on the pooled feature (B, 1024) -> logits."""
        return self.fc3(self.descriptor(y))

    @staticmethod
    def get_loss(pred, label, end_points=None):
        return F.cross_entropy(pred, label.long())


class TransformNet(nn.Module):
    """transform_nets.py input_transform_net (c_in 3, K 3) / feature_transform_net (c_in 64, K 64): 1x1 convs c_in-64-128-1024 (BN + ReLU),
    max over the points, FC 1024-512-256 (BN + ReLU), then `transform` Linear(256, K*K) without activation.  TF initialises the last layer's
    weights and biases to 0 and adds the identity to the bias in the graph; so does `forward` here, and the state dict keeps TF's values.
    forward(y (B, c_in, N)) -> T (B, K, K), row-major reshape."""

    def __init__(self, c_in, k, bn_eps=1e-3):
        super().__init__()
        w = [c_in, 64, 128, 1024]
        self.k = k
        self.convs = nn.ModuleList([nn.Conv1d(w[i], w[i + 1], 1) for i in range(3)])
        self.bns = nn.ModuleList([nn.BatchNorm1d(w[i + 1], eps=bn_eps) for i in range(3)])
        self.fc1, self.bn_fc1 = nn.Linear(1024, 512), nn.BatchNorm1d(512, eps=bn_eps)
        self.fc2, self.bn_fc2 = nn.Linear(512, 256), nn.BatchNorm1d(256, eps=bn_eps)
        self.transform = nn.Linear(256, k * k)
        nn.init.zeros_(self.transform.weight)
        nn.init.zeros_(self.transform.bias)

    def to_matrix(self, raw):
        """The transform layer's output (B, K*K) plus the identity, reshaped row-major to (B, K, K)."""
        return (raw + torch.eye(self.k, dtype=raw.dtype, device=raw.device).flatten()).view(-1, self.k, self.k)

    def forward(self, y):
        for conv, bn in zip(self.convs, self.bns):
            y = F.relu(bn(conv(y)))
        y = torch.max(y, 2)[0]
        y = F.relu(self.bn_fc1(self.fc1(y)))
        y = F.relu(self.bn_fc2(self.fc2(y)))
        return self.to_matrix(self.transform(y))


class PointNetClsTransforms(nn.Module):
    """PointNet with transform nets (classification/models/pointnet_cls.py): T1 = transform_net1(x) (3x3), x1 = x @ T1; conv1 3-64, conv2
    64-64 -> h; T2 = transform_net2(h) (64x64), h2 = h @ T2; conv3 64-64, conv4 64-128, conv5 128-1024 -> max -> GFV; FC 1024-512 (BN + ReLU),
    dropout, FC 512-256 (BN + ReLU), dropout, FC 256-40.  All BatchNorms eps 1e-3.  forward(point_cloud (B, N, 3)) -> (logits (B, classes),
    end_points with "transform" (T2), "critical_set_idx", "GFV" and "retrieval_vectors", fc3's input).  Parameters: random init, or the classifier's TF variables
    (from_tf_variables)."""

    def __init__(self, num_classes=40, bn_eps=1e-3):
        super().__init__()
        self.transform_net1 = TransformNet(3, 3, bn_eps)
        self.transform_net2 = TransformNet(64, 64, bn_eps)
        w = [3, 64, 64, 64, 128, 1024]
        self.convs = nn.ModuleList([nn.Conv1d(w[i], w[i + 1], 1) for i in range(5)])
        self.bns = nn.ModuleList([nn.BatchNorm1d(w[i + 1], eps=bn_eps) for i in range(5)])
        self.fc1, self.bn_fc1 = nn.Linear(1024, 512), nn.BatchNorm1d(512, eps=bn_eps)
        self.fc2, self.bn_fc2 = nn.Linear(512, 256), nn.BatchNorm1d(256, eps=bn_eps)
        self.dp1, self.dp2 = nn.Dropout(p=0.3), nn.Dropout(p=0.3)
        self.fc3 = nn.Linear(256, num_classes)

    def forward(self, point_cloud):
        t1 = self.transform_net1(point_cloud.permute(0, 2, 1))
        y = torch.matmul(point_cloud, t1).permute(0, 2, 1)          # tf.matmul(point_cloud, transform): rows times T
        for conv, bn in zip(self.convs[:2], self.bns[:2]):
            y = F.relu(bn(conv(y)))
        t2 = self.transform_net2(y)
        y = torch.matmul(y.permute(0, 2, 1), t2).permute(0, 2, 1)
        for conv, bn in zip(self.convs[2:], self.bns[2:]):
            y = F.relu(bn(conv(y)))
        end_points = {"transform": t2, "critical_set_idx": torch.argmax(y, dim=2)}
        y = torch.max(y, 2)[0]
        end_points["GFV"] = y
        v = self.descriptor(y)
        end_points["retrieval_vectors"] = v
        return self.fc3(v), end_points

    def descriptor(self, y):
        """fc3's input from the pooled feature (B, 1024), (B, 256): fc2's output after dp2, pointnet_cls.py:111's "retrieval_vectors"; in
        eval mode relu(bn_fc2(fc2(.)))."""
        y = self.dp1(F.relu(self.bn_fc1(self.fc1(y))))
        return self.dp2(F.relu(self.bn_fc2(self.fc2(y))))

    def head(self, y):
        """The FC head on the pooled feature (B, 1024) -> logits."""
        return self.fc3(self.descriptor(y))

    @staticmethod
    def get_loss(pred, label, end_points, reg_weight=0.001):
        """Mean sparse softmax cross-entropy + reg_weight * tf.nn.l2_loss(T2 T2^T - I): half the sum of squares over the WHOLE batch (not a
        mean, so the regulariser grows with the batch size), as pointnet_cls.py's get_loss."""
        t = end_points["transform"]
        d = torch.matmul(t, t.transpose(1, 2)) - torch.eye(t.shape[1], dtype=t.dtype, device=t.device)
        return F.cross_entropy(pred, label.long()) + reg_weight * 0.5 * (d * d).sum()

    def tf_layers(self):
        """(TF layer name, kind, torch layer, BatchNorm or None) of every variable-holding layer, in the graph's order."""
        out = []
        for scope, tn, last in (("transform_net1", self.transform_net1, "transform_XYZ"), ("transform_net2", self.transform_net2, "transform_feat")):
            out += [("%s/tconv%d" % (scope, i + 1), "conv", c, b) for i, (c, b) in enumerate(zip(tn.convs, tn.bns))]
            out += [(scope + "/tfc1", "fc", tn.fc1, tn.bn_fc1), (scope + "/tfc2", "fc", tn.fc2, tn.bn_fc2), (scope + "/" + last, "fc", tn.transform, None)]
        out += [("conv%d" % (i + 1), "conv", c, b) for i, (c, b) in enumerate(zip(self.convs, self.bns))]
        return out + [("fc1", "fc", self.fc1, self.bn_fc1), ("fc2", "fc", self.fc2, self.bn_fc2), ("fc3", "fc", self.fc3, None)]

    @classmethod
    def from_tf_variables(cls, variables, scope="", bn_eps=1e-3):
        """The classifier from a TF variable name -> array mapping, as train_classifier.py saves it (the model variables: weights, biases, bn
        gamma / beta and the moving averages of every layer; no optimiser slots).  The classifier's variables carry no scope
        (train_samplenet.py restores every non-sampler variable under its plain name).  Conv kernels are (1, kw, Cin, Cout), FC weights
        (Cin, Cout).  A missing or an extra name raises KeyError."""
        from .tf_variant import layer_from_tf

        net = cls(num_classes=layer_from_tf(variables, scope, "fc3", "fc", False)["weight"].shape[0], bn_eps=bn_eps)
        used = set()
        with torch.no_grad():
            for name, kind, lin, bn in net.tf_layers():
                before = len(used)
                d = layer_from_tf(variables, scope, name, kind, False, used)
                want = 6 if bn is not None else 2
                if len(used) - before != want or (bn is None) != ("gamma" not in d):
                    raise KeyError("TF variables of %s: %d found, %d expected (weights, biases%s)"
                                   % (name, len(used) - before, want, ", bn gamma / beta / moving mean / variance" if bn is not None else ""))
                if tuple(lin.weight.shape[:2]) != d["weight"].shape:
                    raise ValueError("%s: width %s does not match the module's %s" % (name, d["weight"].shape, tuple(lin.weight.shape[:2])))
                lin.weight.copy_(torch.from_numpy(d["weight"]).view_as(lin.weight))
                lin.bias.copy_(torch.from_numpy(d["bias"]))
                if bn is not None:
                    bn.weight.copy_(torch.from_numpy(d["gamma"])); bn.bias.copy_(torch.from_numpy(d["beta"]))
                    bn.running_mean.copy_(torch.from_numpy(d["mean"])); bn.running_var.copy_(torch.from_numpy(d["var"]))
        extra = sorted(set(variables) - used)
        if extra:
            raise KeyError("TF variables that PointNet with transform nets does not have: %s" % extra[:8])
        return net


class PointNetAE(nn.Module):
    def __init__(self, n_pc_points=2048, bneck_size=128, bn_eps=1e-3):
        super().__init__()
        w = [3, 64, 128, 128, 256, bneck_size]
        self.convs = nn.ModuleList([nn.Conv1d(w[i], w[i + 1], 1) for i in range(5)])
        self.bns = nn.ModuleList([nn.BatchNorm1d(w[i + 1], eps=bn_eps) for i in range(5)])
        self.dec = nn.ModuleList([nn.Linear(bneck_size, 256), nn.Linear(256, 256), nn.Linear(256, n_pc_points * 3)])
        self.n_pc_points = n_pc_points

    def encode(self, x, batch_stats=False):
        """x (B, N, 3) -> (B, bneck).  batch_stats=True: every BatchNorm normalises with the mean and biased variance of this batch's B * N
        points, in either module mode, and no buffer is touched -- the frozen autoencoder of the reconstruction sampler trainers, which run
        it under the training flag with every moving-average decay at 1."""
        y = x.permute(0, 2, 1)
        for conv, bn in zip(self.convs, self.bns):
            if batch_stats:
                y = F.relu(F.batch_norm(conv(y), None, None, bn.weight, bn.bias, training=True, eps=bn.eps))
            else:
                y = F.relu(bn(conv(y)))
        return torch.max(y, 2)[0]

    def decode(self, z):
        y = F.relu(self.dec[0](z))
        y = F.relu(self.dec[1](y))
        return self.dec[2](y).view(-1, self.n_pc_points, 3)

    def forward(self, x, batch_stats=False):
        return self.decode(self.encode(x, batch_stats))


# ------------------------------------------------------------------------------------------------- frozen task networks on CUDA
def _conv_specs(net):
    return [{"weight": conv.weight, "bias": conv.bias, "bn": (bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum),
             "relu": True} for conv, bn in zip(net.convs, net.bns)]


class _FrozenEncoder(nn.Module):
    """A frozen task network whose conv stack and max-pool run on the CUDA frozen encoder (csrc/frozen_encoder.cu): eval-mode BatchNorm,
    gradient to the points only, every prefix of a cloud from one shared pass.  The wrapped module's parameters and buffers are shared,
    not copied.  Evaluation mode only: train(True) raises, and so does a call with grad enabled while a wrapped parameter requires grad
    (this path gives no parameter gradients)."""

    def __init__(self, net):
        super().__init__()
        self.net = net
        super().train(False)

    def train(self, mode=True):
        if mode:
            raise ValueError("%s evaluates in eval mode only" % type(self).__name__)
        return super().train(False)

    def _check_frozen(self):
        if self.net.training:
            raise ValueError("%s: the wrapped module is in training mode" % type(self).__name__)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.net.parameters()):
            raise ValueError("%s gives no parameter gradients: freeze the wrapped module (requires_grad_(False)) or disable grad"
                             % type(self).__name__)

    def _pooled(self, x, sizes):
        """(pooled, route) of every prefix x[:, :s]: more than 16 sizes without a gradient to x run on the forward-only curve entry (one pass
        of the conv stack for all of them), everything else on FrozenEncoderFunction."""
        self._check_frozen()
        from . import ops

        if len(sizes) > ops.FROZEN_MAX_PREFIX and not (torch.is_grad_enabled() and x.requires_grad):
            return ops.frozen_encoder_curve_forward(x.contiguous(), _conv_specs(self.net), sizes)
        return ops.FrozenEncoderFunction.apply(x, _conv_specs(self.net), sizes)


def _critical_set(gfv, route):
    # torch.argmax of an all-zero channel is 0
    return torch.where(gfv > 0, route.long(), torch.zeros_like(route, dtype=torch.long))


class FrozenPointNetCls(_FrozenEncoder):
    """PointNetCls(classifier) on the CUDA frozen encoder: forward(x) -> (logits, end_points) as the module; prefixes(x, sizes) ->
    (P, B, classes) logits of x[:, :s] for every s in sizes, and with return_end_points=True also one end_points dict per prefix ("GFV",
    "critical_set_idx", "retrieval_vectors").  prefixes takes any number of ascending sizes in one encoder pass when no gradient is needed
    (ONE_PASS_PREFIXES), and up to 16 with a gradient to x."""

    ONE_PASS_PREFIXES = True

    def forward(self, point_cloud):
        pooled, route = self._pooled(point_cloud, [point_cloud.shape[1]])
        y = pooled[0]
        v = self.net.descriptor(y)
        return self.net.fc3(v), {"critical_set_idx": _critical_set(y, route[0]), "GFV": y, "retrieval_vectors": v}

    def prefixes(self, x, sizes, return_end_points=False):
        pooled, route = self._pooled(x, sizes)
        p, b, c = pooled.shape
        v = self.net.descriptor(pooled.reshape(p * b, c))
        logits = self.net.fc3(v).view(p, b, -1)
        if not return_end_points:
            return logits
        v = v.view(p, b, -1)
        return logits, [{"GFV": pooled[i], "critical_set_idx": _critical_set(pooled[i], route[i]), "retrieval_vectors": v[i]} for i in range(p)]

    def get_loss(self, pred, label, end_points=None):
        return self.net.get_loss(pred, label, end_points)


class FrozenPointNetAE(_FrozenEncoder):
    """PointNetAE(ae) on the CUDA frozen encoder: forward(x) -> (B, n_pc_points, 3) as the module; prefixes(x, sizes) ->
    (P, B, n_pc_points, 3) reconstructions of x[:, :s] for every s in sizes.

    batch_stats=True (forward, encode, prefixes): every BatchNorm normalises with the batch statistics of each prefix, over its B * s points,
    as PointNetAE.encode(x[:, :s], batch_stats=True) does, on the batch-statistics encoder (csrc/frozen_encoder_bstat.cu): every prefix from
    one pass, the whole batch in one call (the statistics couple the clouds).  Outside that encoder's envelope (unsorted or repeated sizes,
    more than 16 of them, N > 4096, more than 2^22 packed rows) each prefix runs the module's torch route instead."""

    def encode(self, x, batch_stats=False):
        if batch_stats:
            return self._bstat_pooled(x, [x.shape[1]])[0]
        return self._pooled(x, [x.shape[1]])[0][0]

    def forward(self, x, batch_stats=False):
        return self.net.decode(self.encode(x, batch_stats))

    def prefixes(self, x, sizes, batch_stats=False):
        pooled = self._bstat_pooled(x, sizes) if batch_stats else self._pooled(x, sizes)[0]
        p, b, c = pooled.shape
        return self.net.decode(pooled.reshape(p * b, c)).view(p, b, self.net.n_pc_points, 3)

    def _bstat_pooled(self, x, sizes):
        """(P, B, bneck) pooled features of x[:, :s] for every s in sizes, each prefix normalised with its own batch statistics."""
        from . import ops

        self._check_frozen()
        sizes = [int(s) for s in sizes]
        specs = _conv_specs(self.net)
        if x.dim() == 3 and x.shape[2] == 3 and ops.frozen_encoder_bstat_supported(x.shape[0], x.shape[1], specs, sizes):
            if not x.is_cuda:
                raise RuntimeError("samplenet_b200: the input is on %s; the ops are CUDA-only (no CPU fallback)" % x.device)
            return ops.FrozenEncoderBStatFunction.apply(x, specs, sizes)[0]
        return torch.stack([self.net.encode(x[:, :s], batch_stats=True) for s in sizes])


def _fc_specs(layers):
    """(Linear, BatchNorm1d or None, relu) -> frozen-MLP specs sharing the module's tensors."""
    return [{"weight": lin.weight, "bias": lin.bias, "relu": relu,
             "bn": None if bn is None else (bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum)} for lin, bn, relu in layers]


class FrozenPointNetClsTransforms(_FrozenEncoder):
    """PointNetClsTransforms(classifier) frozen, on CUDA kernels; forward(x (B, N, 3)) -> (logits, end_points) as the module, with a
    differentiable end_points["transform"], so the module's get_loss (cross-entropy + the transform regulariser) applies unchanged.  Gradients
    reach the points only, through both transform nets:

        T1      transform_net1's conv stack and pool on the frozen encoder, its FC layers on the frozen MLP with BatchNorm
        x1      x @ T1 (point transform)
        h, T2   conv1, conv2 and transform_net2's conv stack as ONE frozen-encoder call on x1 that also returns h = conv2's activation;
                transform_net2's FC layers on the frozen MLP
        GFV     h @ T2, then conv3 .. conv5 and the pool as one frozen-encoder call from that activation
        logits  the head on the frozen MLP with BatchNorm (dropout is the identity in eval mode); end_points["retrieval_vectors"] is the
                head's fc2 activation, fc3's input, as that call writes it (not differentiable)

    Batches above 64 clouds run in chunks; shapes outside the kernels' envelopes run the wrapped module.
    prefixes(x, sizes) gives every prefix x[:, :s] from one chain of launches, although T1 and T2 depend on the prefix: every (prefix, cloud)
    pair is one segment of a packed buffer (ops.Segments), and the per-point layers and the point transforms run on all segments at once
    (see _prefix_chunk).  prefixes exists while the wrapped module's parameters are on a CUDA device: the one-pass route is CUDA-only (even
    its plan needs CUDA tensors), so for a module elsewhere the attribute is absent and callers that look for it (ProgressiveClassificationStep,
    ProgressiveClassificationEvaluator) keep calling the wrapper once per prefix, as they did before the route existed."""

    MAX_CLOUDS = 64
    MAX_PREFIXES = 16   # the frozen encoder's prefix pools per pass (T-Net 1)

    def _plan(self):
        net = self.net
        t1, t2 = net.transform_net1, net.transform_net2
        tn_fc = lambda t: _fc_specs([(t.fc1, t.bn_fc1, True), (t.fc2, t.bn_fc2, True), (t.transform, None, False)])
        front = _conv_specs(net)[:2] + _conv_specs(t2)
        return {"t1_conv": _conv_specs(t1), "t1_fc": tn_fc(t1), "front": front, "t2_fc": tn_fc(t2), "back": _conv_specs(net)[2:],
                "head": _fc_specs([(net.fc1, net.bn_fc1, True), (net.fc2, net.bn_fc2, True), (net.fc3, None, False)])}

    def supported(self, b, n):
        """Whether (b <= 64 clouds of) n points run on the CUDA path."""
        from . import ops

        P = self._plan()
        b = min(b, self.MAX_CLOUDS)
        return (b >= 1 and ops.frozen_encoder_supported(b, n, P["t1_conv"], 1) and ops.frozen_encoder_ex_supported(b, n, P["front"], 1, False, 1)
                and ops.frozen_encoder_ex_supported(b, n, P["back"], 1, True) and ops.point_transform_supported(b, n, 64)
                and all(ops.frozen_mlp_supported(b, P[k], batchnorm=True) for k in ("t1_fc", "t2_fc", "head")))

    def _chunk(self, x, P):
        from . import ops

        n = x.shape[1]
        pooled1, _ = ops.FrozenEncoderFunction.apply(x, P["t1_conv"], [n])
        t1 = self.net.transform_net1.to_matrix(ops.FrozenMLPBNFunction.apply(pooled1[0], P["t1_fc"]))
        x1 = ops.PointTransformFunction.apply(x, t1)
        pooled2, _, h = ops.FrozenEncoderExFunction.apply(x1, P["front"], [n], False, 1)
        t2 = self.net.transform_net2.to_matrix(ops.FrozenMLPBNFunction.apply(pooled2[0], P["t2_fc"]))
        h2 = ops.PointTransformFunction.apply(h, t2)
        pooled3, route3 = ops.FrozenEncoderExFunction.apply(h2, P["back"], [n], True, -1)
        gfv = pooled3[0]
        logits, v = ops.FrozenMLPBNFunction.apply(gfv, P["head"], True)
        return logits, t2, _critical_set(gfv, route3[0]), gfv, v

    def forward(self, point_cloud):
        self._check_frozen()
        if point_cloud.dim() != 3 or point_cloud.shape[2] != 3 or not self.supported(point_cloud.shape[0], point_cloud.shape[1]):
            return self.net(point_cloud)
        if not point_cloud.is_cuda:
            raise RuntimeError("samplenet_b200: the input is on %s; the ops are CUDA-only (no CPU fallback)" % point_cloud.device)
        P = self._plan()
        parts = [self._chunk(point_cloud[s:s + self.MAX_CLOUDS].contiguous(), P) for s in range(0, point_cloud.shape[0], self.MAX_CLOUDS)]
        logits, t2, crit, gfv, v = parts[0] if len(parts) == 1 else [torch.cat(t) for t in zip(*parts)]
        return logits, {"transform": t2, "critical_set_idx": crit, "GFV": gfv, "retrieval_vectors": v}

    def _prefixes_supported(self, b, n, sizes):
        """Whether prefixes(x (b, n, 3), sizes) runs on the segmented path: 1..16 ascending sizes in [1, n], and every kernel's envelope at
        a chunk of min(b, 64) clouds."""
        from . import ops

        if not sizes or len(sizes) > self.MAX_PREFIXES or sizes[0] < 1 or sizes[-1] > n or any(a >= c for a, c in zip(sizes, sizes[1:])):
            return False
        if not self.supported(b, n):
            return False
        P, b = self._plan(), min(b, self.MAX_CLOUDS)
        num, max_len = len(sizes) * b, sizes[-1]
        total = b * sum(-(-s // ops.SEG_TILE) * ops.SEG_TILE for s in sizes)
        return (ops.frozen_encoder_supported(b, n, P["t1_conv"], len(sizes)) and ops.frozen_encoder_seg_supported(num, total, max_len, P["front"], False, 1)
                and ops.frozen_encoder_seg_supported(num, total, max_len, P["back"], True) and ops.point_transform_seg_supported(num, total, max_len, 64))

    def _rows(self, rows, specs, last_hidden=False):
        """The frozen MLP on the rows of a (P * B, C) tensor, 64 rows per call; with last_hidden=True (out, the last hidden layer's
        activation)."""
        from . import ops

        parts = [ops.FrozenMLPBNFunction.apply(rows[i:i + self.MAX_CLOUDS], specs, last_hidden) for i in range(0, rows.shape[0], self.MAX_CLOUDS)]
        return [torch.cat(t) for t in zip(*parts)] if last_hidden else torch.cat(parts)

    def _prefix_chunk(self, x, sizes, P):
        """prefixes() of at most 64 clouds: (logits, T2, critical_set_idx, GFV), each (P, B, ...).  Segment j = p * B + b is prefix p of cloud b.
            1. T-Net 1's conv stack once on x with every prefix's pool (its layers are per point; only the pool depends on the prefix);
            2. T-Net 1's FC layers on the P * B pooled rows, 64 per call -> T1 per segment;
            3. x1 = x[b, :s_p] @ T1[p, b] for every segment, read from x in place (prefix source) into the packed buffer;
            4. conv1, conv2 (tapped: h) and T-Net 2's convs, one pool per segment;  5. T-Net 2's FC layers -> T2 per segment;
            6. h2 = h @ T2 per segment (packed source);  7. conv3 .. conv5, one pool per segment;  8. the head."""
        from . import ops

        b, np_ = x.shape[0], len(sizes)
        segs = ops.Segments(sizes, b, x.device)
        tn1, tn2 = self.net.transform_net1, self.net.transform_net2
        pooled1, _ = ops.FrozenEncoderFunction.apply(x, P["t1_conv"], sizes)
        t1 = tn1.to_matrix(self._rows(pooled1.reshape(np_ * b, -1), P["t1_fc"]))
        x1 = ops.PointTransformSegFunction.apply(x, t1, segs, True)
        pooled2, _, h = ops.FrozenEncoderSegFunction.apply(x1, P["front"], segs, False, 1)
        t2 = tn2.to_matrix(self._rows(pooled2, P["t2_fc"]))
        h2 = ops.PointTransformSegFunction.apply(h, t2, segs, False)
        gfv, route3 = ops.FrozenEncoderSegFunction.apply(h2, P["back"], segs, True, -1)
        logits, v = self._rows(gfv, P["head"], True)
        view = lambda t: t.view(np_, b, *t.shape[1:])
        return view(logits), view(t2), view(_critical_set(gfv, route3)), view(gfv), view(v)

    @property
    def prefixes(self):
        """prefixes(x, sizes, return_end_points=False), offered while the wrapped module is on a CUDA device (see the class docstring)."""
        if not all(p.is_cuda for p in self.net.parameters()):
            raise AttributeError("%s.prefixes: the one pass over every prefix needs the wrapped module on a CUDA device" % type(self).__name__)
        return self._prefixes

    def _prefixes(self, x, sizes, return_end_points=False):
        """(P, B, classes) logits of x[:, :s] for every s in sizes, differentiable in x; with return_end_points=True also one end_points dict
        per prefix, as forward's ("transform" differentiable, "GFV", "critical_set_idx", "retrieval_vectors"), so get_loss keeps the transform regulariser.
        Sizes that are not ascending, more than 16 of them, sizes outside [1, N] or shapes outside the kernels' envelopes run forward on
        each prefix instead (the same results, one chain per prefix)."""
        self._check_frozen()
        sizes = [int(s) for s in sizes]
        if x.dim() != 3 or x.shape[2] != 3 or not self._prefixes_supported(x.shape[0], x.shape[1], sizes):
            outs = [self.forward(x[:, :s].contiguous()) for s in sizes]
            logits = torch.stack([o[0] for o in outs])
            return (logits, [o[1] for o in outs]) if return_end_points else logits
        if not x.is_cuda:
            raise RuntimeError("samplenet_b200: the input is on %s; the ops are CUDA-only (no CPU fallback)" % x.device)
        P = self._plan()
        parts = [self._prefix_chunk(x[s:s + self.MAX_CLOUDS].contiguous(), sizes, P) for s in range(0, x.shape[0], self.MAX_CLOUDS)]
        logits, t2, crit, gfv, v = parts[0] if len(parts) == 1 else [torch.cat(t, dim=1) for t in zip(*parts)]
        if not return_end_points:
            return logits
        return logits, [{"transform": t2[p], "critical_set_idx": crit[p], "GFV": gfv[p], "retrieval_vectors": v[p]} for p in range(len(sizes))]

    def get_loss(self, pred, label, end_points, reg_weight=0.001):
        return self.net.get_loss(pred, label, end_points, reg_weight)


# ------------------------------------------------------------------------------------------------- task networks trained on CUDA
def _bn_spec(bn):
    return (bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum, bn.num_batches_tracked)


class _TrainableTaskNet(nn.Module):
    """Base of the task networks trained on CUDA.  The wrapped module (`.net`) keeps its parameters and buffers: the optimiser takes
    `parameters()`, and `state_dict()` / `load_state_dict()` use the module's own keys (no `net.` prefix), so checkpoints move freely
    between the module and its wrapper.  `route` is the path of the last forward:

        "cuda"    training mode, on the per-layer training kernels (ops.LayerStackFunction)
        "frozen"  eval mode with no parameter gradient wanted, on the module's frozen wrapper
        "module"  the wrapped module's own forward: shapes outside the kernels' envelope (BatchNorm over the batch cannot be split), an
                  input that needs its gradient, BatchNorm with momentum=None (a cumulative average), eval mode with parameter gradients

    The mode is the wrapped module's (`net.training`); train() / eval() on the wrapper set it.  CPU tensors raise."""

    def __init__(self, net):
        super().__init__()
        self.net = net
        self.route = None
        self._register_state_dict_hook(_TrainableTaskNet._strip_prefix)
        self._register_load_state_dict_pre_hook(_TrainableTaskNet._add_prefix)

    @staticmethod
    def _strip_prefix(module, state_dict, prefix, local_metadata):
        for k in [k for k in state_dict if k.startswith(prefix + "net.")]:
            state_dict[prefix + k[len(prefix) + 4:]] = state_dict.pop(k)

    @staticmethod
    def _add_prefix(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        for k in [k for k in state_dict if k.startswith(prefix) and not k.startswith(prefix + "net.")]:
            state_dict[prefix + "net." + k[len(prefix):]] = state_dict.pop(k)

    def _layer_stack(self):
        """(conv specs, FC specs, parameters in spec order) of the stack that runs on the training kernels."""
        raise NotImplementedError

    def _cuda_trainable(self, x, conv_specs, fc_specs, check_envelope=True):
        from . import ops

        if x.requires_grad or x.dim() != 3 or x.shape[2] != conv_specs[0]["weight"].shape[1]:
            return False
        if any(s["bn"] is not None and s["bn"][5] is None for s in conv_specs + fc_specs):
            return False
        return ops.generator_layers_ex_supported(x, conv_specs, fc_specs) if check_envelope else True

    def _cuda_supported(self, x):
        """Whether a training-mode forward on x runs on the CUDA kernels."""
        return self._cuda_trainable(x, *self._layer_stack()[:2])

    def _pick_route(self, x):
        if not x.is_cuda:
            raise RuntimeError("samplenet_b200: the input is on %s; the ops are CUDA-only (no CPU fallback)" % x.device)
        if self.net.training:
            self.route = "cuda" if self._cuda_supported(x) else "module"
        elif torch.is_grad_enabled() and any(p.requires_grad for p in self.net.parameters()):
            self.route = "module"
        else:
            self.route = "frozen"
        return self.route

    def _train_stack(self, x):
        """(out, feat) of the layer stack on the CUDA training kernels."""
        from . import ops

        conv_specs, fc_specs, params = self._layer_stack()
        return ops.LayerStackFunction.apply(x.contiguous(), conv_specs, fc_specs, *params)


class CudaPointNetAE(_TrainableTaskNet):
    """PointNetAE(ae) trained on CUDA: forward(x (B, N, 3)) -> (B, n_pc_points, 3) as the module.  In training mode the encoder's conv stack
    with BatchNorm over the batch, the max-pool and the decoder run on the per-layer training kernels, forward and backward (every
    parameter's gradient, the running statistics and num_batches_tracked as nn.BatchNorm1d updates them); 2 <= B <= 64 clouds of any number
    of points.  Eval mode runs FrozenPointNetAE.  prefixes(x, sizes) reconstructs every prefix x[:, :s], in training mode from one pass of
    the batch-statistics encoder trained.  See _TrainableTaskNet for the routes."""

    def _layer_stack(self):
        net = self.net
        conv = [{"weight": c.weight, "bias": c.bias, "bn": _bn_spec(bn), "relu": True} for c, bn in zip(net.convs, net.bns)]
        fc = [{"weight": l.weight, "bias": l.bias, "bn": None, "relu": i < 2} for i, l in enumerate(net.dec)]
        params = [t for c, bn in zip(net.convs, net.bns) for t in (c.weight, c.bias, bn.weight, bn.bias)]
        return conv, fc, params + [t for l in net.dec for t in (l.weight, l.bias)]

    def forward(self, x, batch_stats=False):
        """batch_stats=True (eval mode only): BatchNorm with the batch's own statistics and no buffer touched, on the "frozen" and "module"
        routes (see PointNetAE.encode).  Training mode raises ValueError: it normalises with the batch statistics already, and updates the
        running ones."""
        if batch_stats and self.net.training:
            raise ValueError("CudaPointNetAE: batch_stats=True is for eval mode; training mode already normalises with the batch statistics "
                             "and updates the running ones")
        route = self._pick_route(x)
        if route == "cuda":
            return self._train_stack(x)[0].view(-1, self.net.n_pc_points, 3)
        if route == "frozen":
            return FrozenPointNetAE(self.net)(x, batch_stats=True) if batch_stats else FrozenPointNetAE(self.net)(x)
        return self.net(x, batch_stats=True) if batch_stats else self.net(x)

    def prefixes(self, x, sizes):
        """(P, B, n_pc_points, 3): the reconstruction of x[:, :s] for every s in sizes, what `torch.stack([net(x[:, :s]) for s in sizes])`
        computes on the module, the running statistics included.  Training mode: every encoder BatchNorm normalises prefix s with its own
        batch statistics and the running statistics move once per prefix in ascending order, on the batch-statistics encoder trained
        (ops.EncoderBStatTrainFunction: every prefix from one pass, gradients to x and to every encoder parameter); the decoder runs in torch
        on the (P B, bneck) pooled features.  Outside that encoder's envelope (see ops.frozen_encoder_bstat_train_supported) or with a
        BatchNorm of momentum=None, the module's ascending per-prefix loop ("module").  Eval mode: FrozenPointNetAE.prefixes ("frozen") when
        no parameter gradient is wanted, the module's loop otherwise."""
        from . import ops

        if not x.is_cuda:
            raise RuntimeError("samplenet_b200: the input is on %s; the ops are CUDA-only (no CPU fallback)" % x.device)
        net, sizes = self.net, [int(s) for s in sizes]
        if net.training:
            conv, _, params = self._layer_stack()
            if (x.dim() == 3 and x.shape[2] == 3 and all(s["bn"][5] is not None for s in conv)
                    and ops.frozen_encoder_bstat_train_supported(x.shape[0], x.shape[1], conv, sizes)):
                self.route = "cuda"
                pooled = ops.EncoderBStatTrainFunction.apply(x, conv, sizes, *params[:4 * len(conv)])[0]
                p, b, c = pooled.shape
                return net.decode(pooled.reshape(p * b, c)).view(p, b, net.n_pc_points, 3)
            self.route = "module"
        elif torch.is_grad_enabled() and any(p.requires_grad for p in net.parameters()):
            self.route = "module"
        else:
            self.route = "frozen"
            return FrozenPointNetAE(net).prefixes(x, sizes)
        return torch.stack([net(x[:, :s].contiguous()) for s in sizes])


def _train_specs(convs, fcs):
    """(conv specs, FC specs, parameters in spec order) of a layer stack trained on CUDA: convs [(Conv1d, BatchNorm1d)] with ReLU, fcs
    [(Linear, BatchNorm1d or None, relu)]."""
    conv = [{"weight": c.weight, "bias": c.bias, "bn": _bn_spec(bn), "relu": True} for c, bn in convs]
    fc = [{"weight": l.weight, "bias": l.bias, "bn": None if bn is None else _bn_spec(bn), "relu": relu} for l, bn, relu in fcs]
    params = [t for c, bn in convs for t in (c.weight, c.bias, bn.weight, bn.bias)]
    return conv, fc, params + [t for l, bn, _ in fcs for t in ((l.weight, l.bias) if bn is None else (l.weight, l.bias, bn.weight, bn.bias))]


class _CudaClassifier(_TrainableTaskNet):
    """The PointNet classifiers trained on CUDA.  In the "cuda" route the wrapper draws the dropout masks itself: one per nn.Dropout of the
    module (`DROPOUT`: its name and the width of the FC input it masks), in that order, each
        torch.empty(B, width, device=x.device).bernoulli_(1 - p).div_(1 - p)
    on torch's default CUDA generator with the module's p (p = 0: no mask, no draw).  Those draws are the wrapper's only random numbers, so
    re-seeding the generator rebuilds them.  end_points hold "GFV", the pooled feature (detached), and for the transforms classifier
    "transform"; "critical_set_idx" is not produced in training mode (neither get_loss nor the classification trainer reads it).  get_loss
    is the module's."""

    DROPOUT = ()
    MAX_CLOUDS = 41   # fc1's 1024-channel input and weight rows in the FC backward's shared memory

    def _stack_inputs(self, x):
        """(input of the stack, the stack) of every layer-stack call of a training-mode forward on x."""
        return [(x, self._layer_stack())]

    def _cuda_supported(self, x):
        if x.dim() != 3:
            return False
        stacks = self._stack_inputs(x)
        if not (2 <= x.shape[0] <= self.MAX_CLOUDS and all(self._cuda_trainable(xi, c, f, False) for xi, (c, f, _) in stacks)):
            return False
        return all(self._cuda_trainable(xi, c, f) for xi, (c, f, _) in stacks)

    def dropout_masks(self, b, device):
        """The masks of one training-mode forward of b clouds, drawn as the class documents; None for a dropout with p = 0."""
        masks = []
        for name, width in self.DROPOUT:
            p = getattr(self.net, name).p
            masks.append(torch.empty(b, width, device=device).bernoulli_(1 - p).div_(1 - p) if p > 0 else None)
        return masks

    def get_loss(self, *args, **kwargs):
        return self.net.get_loss(*args, **kwargs)


class CudaPointNetCls(_CudaClassifier):
    """PointNetCls(classifier) trained on CUDA: forward(x (B, N, 3)) -> (logits, end_points) as the module.  In training mode the conv stack
    with BatchNorm over the batch, the max-pool and the FC head with its dropout run on the per-layer training kernels, forward and backward
    (every parameter's gradient, the running statistics and num_batches_tracked as nn.BatchNorm1d updates them); 2 <= B <= 41 clouds of any
    number of points.  Eval mode runs FrozenPointNetCls.  See _CudaClassifier for the masks and _TrainableTaskNet for the routes."""

    DROPOUT = (("dp1", 256),)

    def _layer_stack(self):
        net = self.net
        return _train_specs(list(zip(net.convs, net.bns)), [(net.fc1, net.bn_fc1, True), (net.fc2, net.bn_fc2, True), (net.fc3, None, False)])

    def forward(self, point_cloud):
        route = self._pick_route(point_cloud)
        if route == "frozen":
            return FrozenPointNetCls(self.net)(point_cloud)
        if route == "module":
            return self.net(point_cloud)
        from . import ops

        conv, fc, params = self._layer_stack()
        fc[2]["dropout"] = self.dropout_masks(point_cloud.shape[0], point_cloud.device)[0]
        logits, gfv = ops.LayerStackFunction.apply(point_cloud.contiguous(), conv, fc, *params)
        return logits, {"GFV": gfv}


class CudaPointNetClsTransforms(_CudaClassifier):
    """PointNetClsTransforms(classifier) trained on CUDA: forward(x (B, N, 3)) -> (logits, end_points) as the module, with a differentiable
    end_points["transform"] (T2), so the module's get_loss (cross-entropy + the transform regulariser) applies unchanged.  A training-mode
    forward is three calls of the per-layer training kernels, as FrozenPointNetClsTransforms splits the network:

        T1      transform_net1 on x (no gradient to x); x1 = x @ T1 (point transform)
        h, T2   conv1, conv2 and transform_net2's conv stack as ONE stack on x1 that also returns h = conv2's activation (each layer's
                BatchNorm statistics are its own, so merging them changes none); the gradient reaches x1, and h's through the tap
        logits  h2 = h @ T2, then conv3 .. conv5, the pool and the head with its two dropouts as one stack reading the activation h2

    2 <= B <= 41 clouds of any number of points.  Eval mode runs FrozenPointNetClsTransforms.  See _CudaClassifier for the masks and
    _TrainableTaskNet for the routes."""

    DROPOUT = (("dp1", 512), ("dp2", 256))

    def _stacks(self):
        net = self.net
        t1, t2 = net.transform_net1, net.transform_net2
        tn_fc = lambda t: [(t.fc1, t.bn_fc1, True), (t.fc2, t.bn_fc2, True), (t.transform, None, False)]
        convs = list(zip(net.convs, net.bns))
        front = _train_specs(convs[:2] + list(zip(t2.convs, t2.bns)), tn_fc(t2))
        front[0][1]["tap"] = True
        return (_train_specs(list(zip(t1.convs, t1.bns)), tn_fc(t1)), front,
                _train_specs(convs[2:], [(net.fc1, net.bn_fc1, True), (net.fc2, net.bn_fc2, True), (net.fc3, None, False)]))

    def _layer_stack(self):
        return self._stacks()[2]

    def _stack_inputs(self, x):
        s1, s2, s3 = self._stacks()
        return [(x, s1), (x, s2), (torch.empty(x.shape[0], x.shape[1], s3[0][0]["weight"].shape[1], device="meta"), s3)]

    def forward(self, point_cloud):
        route = self._pick_route(point_cloud)
        if route == "frozen":
            return FrozenPointNetClsTransforms(self.net)(point_cloud)
        if route == "module":
            return self.net(point_cloud)
        from . import ops

        net, x = self.net, point_cloud.contiguous()
        masks = self.dropout_masks(x.shape[0], x.device)
        (c1, f1, p1), (c2, f2, p2), (c3, f3, p3) = self._stacks()
        t1 = net.transform_net1.to_matrix(ops.LayerStackFunction.apply(x, c1, f1, *p1)[0])
        x1 = ops.PointTransformFunction.apply(x, t1)
        out2, _, h = ops.LayerStackFunction.apply(x1, c2, f2, *p2)
        t2 = net.transform_net2.to_matrix(out2)
        h2 = ops.PointTransformFunction.apply(h, t2)
        f3[1]["dropout"], f3[2]["dropout"] = masks
        logits, gfv = ops.LayerStackFunction.apply(h2, c3, f3, *p3)
        return logits, {"transform": t2, "GFV": gfv}
