"""Task networks of the classification and reconstruction trainers, restated in stock torch ops (SURVEY.md 8f rank 1).  They are CALLERS
of the hot path -- frozen while the sampler trains (train_samplenet.py:227-232, sampler/train_samplenet.py:100-118) -- so they stay plain
torch modules; only the layer stacks' structure, widths, BatchNorm placement and eps follow the reference:

    PointNetCls   classification/models/pointnet_cls_basic.py:55-136 (vanilla PointNet: 3-64-64-64-128-1024 1x1 convs with BN, max-pool,
                  fc 512 - fc 256 - dropout(keep 0.7) - fc 40; tf_util batch norm eps 1e-3); get_loss = mean sparse softmax cross-entropy
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
        return self.head(y), end_points

    def head(self, y):
        """The FC head on the pooled feature (B, 1024) -> logits."""
        y = F.relu(self.bn_fc1(self.fc1(y)))
        y = F.relu(self.bn_fc2(self.fc2(y)))
        return self.fc3(self.dp1(y))

    @staticmethod
    def get_loss(pred, label, end_points=None):
        return F.cross_entropy(pred, label.long())


class PointNetAE(nn.Module):
    def __init__(self, n_pc_points=2048, bneck_size=128, bn_eps=1e-3):
        super().__init__()
        w = [3, 64, 128, 128, 256, bneck_size]
        self.convs = nn.ModuleList([nn.Conv1d(w[i], w[i + 1], 1) for i in range(5)])
        self.bns = nn.ModuleList([nn.BatchNorm1d(w[i + 1], eps=bn_eps) for i in range(5)])
        self.dec = nn.ModuleList([nn.Linear(bneck_size, 256), nn.Linear(256, 256), nn.Linear(256, n_pc_points * 3)])
        self.n_pc_points = n_pc_points

    def encode(self, x):
        y = x.permute(0, 2, 1)
        for conv, bn in zip(self.convs, self.bns):
            y = F.relu(bn(conv(y)))
        return torch.max(y, 2)[0]

    def decode(self, z):
        y = F.relu(self.dec[0](z))
        y = F.relu(self.dec[1](y))
        return self.dec[2](y).view(-1, self.n_pc_points, 3)

    def forward(self, x):
        return self.decode(self.encode(x))


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

    def _pooled(self, x, sizes):
        if self.net.training:
            raise ValueError("%s: the wrapped module is in training mode" % type(self).__name__)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.net.parameters()):
            raise ValueError("%s gives no parameter gradients: freeze the wrapped module (requires_grad_(False)) or disable grad"
                             % type(self).__name__)
        from . import ops

        return ops.FrozenEncoderFunction.apply(x, _conv_specs(self.net), sizes)


class FrozenPointNetCls(_FrozenEncoder):
    """PointNetCls(classifier) on the CUDA frozen encoder: forward(x) -> (logits, end_points) as the module; prefixes(x, sizes) ->
    (P, B, classes) logits of x[:, :s] for every s in sizes."""

    def forward(self, point_cloud):
        pooled, route = self._pooled(point_cloud, [point_cloud.shape[1]])
        y = pooled[0]
        # torch.argmax of an all-zero channel is 0
        end_points = {"critical_set_idx": torch.where(y > 0, route[0].long(), torch.zeros_like(route[0], dtype=torch.long)), "GFV": y}
        return self.net.head(y), end_points

    def prefixes(self, x, sizes):
        pooled, _ = self._pooled(x, sizes)
        p, b, c = pooled.shape
        return self.net.head(pooled.reshape(p * b, c)).view(p, b, -1)

    def get_loss(self, pred, label, end_points=None):
        return self.net.get_loss(pred, label, end_points)


class FrozenPointNetAE(_FrozenEncoder):
    """PointNetAE(ae) on the CUDA frozen encoder: forward(x) -> (B, n_pc_points, 3) as the module; prefixes(x, sizes) ->
    (P, B, n_pc_points, 3) reconstructions of x[:, :s] for every s in sizes."""

    def encode(self, x):
        return self._pooled(x, [x.shape[1]])[0][0]

    def forward(self, x):
        return self.net.decode(self.encode(x))

    def prefixes(self, x, sizes):
        pooled, _ = self._pooled(x, sizes)
        p, b, c = pooled.shape
        return self.net.decode(pooled.reshape(p * b, c)).view(p, b, self.net.n_pc_points, 3)
