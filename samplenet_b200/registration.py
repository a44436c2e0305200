"""The registration trainer's step, restated over this package (SURVEY.md 8f ranks 1 and 4): the callers of the hot path.

    PCRNet / PointNetFeatures     registration/models/pcrnet.py:8-82         (task network; stock torch layers, same state-dict keys)
    QuaternionTransform           registration/src/qdataset.py:17-119        ((w,x,y,z) quaternion + translation, kornia-free)
    qrot / qinv                   registration/src/quaternion.py:35-53, qinv
    random_transforms / on_unit_cube / CudaQuaternionFixedDataset / get_datasets
                                  registration/src/qdataset.py:122-179, src/pctransforms.py:162-166,
                                  data/modelnet_loader_torch.py:102-116, main.py:601-637 (the set on the device, one launch per batch)
    RegistrationStep              registration/main.py:221-247 (hyper-parameters), :249-298 (create_model), :485-498
                                  (non_learned_sampling), :500-538
                                  (compute_samplenet_loss), :540-553 (compute_sampling_consistency), :555-598 (compute_pcrnet_loss),
                                  :306-362 (train_1: loss = pcrnet_loss + sampler_loss; zero_grad; backward; step),
                                  :306-362 (train_1 over an epoch), :364-414 (eval_1), :416-483 (test_1)

The sampler is this package's SampleNet (CUDA kernels) or, for `sampler="fps"` / `"random"`, its FPSSampler / RandomSampler, Chamfer is this package's ChamferDistance; the task network is the reference's
architecture in stock torch ops (it is a caller of the path, not the path).  `RegistrationStep.train_step` is one iteration of
`Action.train_1`; with torch.distributed initialised the sampler's gradients go through `FlatBucketDataParallel` (one flat all-reduce).
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .chamfer_distance import ChamferDistance
from .evaluation import eval_mode, precision_curve
from .parallel import FlatBucketDataParallel
from .samplenet import SampleNet
from .samplers import FPSSampler, RandomSampler
from .trainers import _StepGraph


# ----------------------------------------------------------------------------------------------------- task network
class PointNetFeatures(nn.Module):
    def __init__(self, bottleneck_size=1024, input_shape="bcn"):
        super().__init__()
        if input_shape not in ["bcn", "bnc"]:
            raise ValueError("allowed shape are 'bcn' (batch * channels * num_in_points), 'bnc' ")
        self.input_shape = input_shape
        self.conv1 = torch.nn.Conv1d(3, 64, 1)
        self.conv2 = torch.nn.Conv1d(64, 64, 1)
        self.conv3 = torch.nn.Conv1d(64, 64, 1)
        self.conv4 = torch.nn.Conv1d(64, 128, 1)
        self.conv5 = torch.nn.Conv1d(128, bottleneck_size, 1)

    def forward(self, x):
        if self.input_shape == "bnc":
            x = x.permute(0, 2, 1)
        if x.shape[1] != 3:
            raise RuntimeError("shape of x must be of [Batch x 3 x NumInPoints]")
        y = F.relu(self.conv1(x))
        y = F.relu(self.conv2(y))
        y = F.relu(self.conv3(y))
        y = F.relu(self.conv4(y))
        y = F.relu(self.conv5(y))
        return torch.max(y, 2)[0].contiguous()


class PCRNet(nn.Module):
    def __init__(self, bottleneck_size=1024, input_shape="bcn"):
        super().__init__()
        if input_shape not in ["bcn", "bnc"]:
            raise ValueError("allowed shape are 'bcn' (batch * channels * num_in_points), 'bnc' ")
        self.input_shape = input_shape
        self.feat = PointNetFeatures(bottleneck_size, input_shape)
        self.fc1 = nn.Linear(bottleneck_size * 2, 1024)
        self.fc2 = nn.Linear(1024, 1024)
        self.fc3 = nn.Linear(1024, 512)
        self.fc4 = nn.Linear(512, 512)
        self.fc5 = nn.Linear(512, 256)
        self.fc6 = nn.Linear(256, 7)
        self.sampler = None

    def forward(self, x0, x1):
        y = torch.cat([self.feat(x0), self.feat(x1)], dim=1)
        y = F.relu(self.fc1(y))
        y = F.relu(self.fc2(y))
        y = F.relu(self.fc3(y))
        y = F.relu(self.fc4(y))
        y = F.relu(self.fc5(y))
        y = self.fc6(y)
        pre_normalized_quat = y[:, 0:4]
        normalized_quat = F.normalize(pre_normalized_quat, dim=1)
        return torch.cat([normalized_quat, y[:, 4:]], dim=1), pre_normalized_quat


class FrozenPCRNet(nn.Module):
    """PCRNet(pcrnet) frozen, on CUDA kernels: template and source through the frozen encoder (csrc/frozen_encoder.cu) as one stacked call
    when they have the same size and as one call each when they do not (one sampled cloud against a full one), the six Linear layers
    through the frozen MLP (csrc/frozen_mlp.cu); gradients reach the two clouds only.  forward(x0, x1) ->
    (twist, pre_normalized_quat) as the module.  The wrapped module's parameters are shared, not copied.  Evaluation mode only: train(True)
    raises, and so does a call with grad enabled while a wrapped parameter requires grad (this path gives no parameter gradients).
    Shapes outside the kernels' envelopes run the wrapped module."""

    # Clouds per frozen-encoder call: 32 pairs stacked.  Clouds of two sizes go through one call per size, still 32 pairs at a time: the MLP
    # sums in an order that depends on its row count, and one chunk size for both keeps a batch's output the concatenation of its chunks'.
    ENCODER_ROWS = 64

    def __init__(self, pcrnet):
        super().__init__()
        self.net = pcrnet
        self.training = False      # the wrapped module (and the sampler attached to it) keep their own modes

    @property
    def sampler(self):
        return self.net.sampler

    def __setattr__(self, name, value):
        if name == "sampler":     # nn.Module would register a module-valued attribute on the wrapper instead
            self.net.sampler = value
        else:
            super().__setattr__(name, value)

    @property
    def input_shape(self):
        return self.net.input_shape

    def train(self, mode=True):
        if mode:
            raise ValueError("%s evaluates in eval mode only" % type(self).__name__)
        return super().train(False)

    def _specs(self):
        f = self.net.feat
        conv = [{"weight": c.weight, "bias": c.bias, "bn": None, "relu": True} for c in (f.conv1, f.conv2, f.conv3, f.conv4, f.conv5)]
        fcs = (self.net.fc1, self.net.fc2, self.net.fc3, self.net.fc4, self.net.fc5, self.net.fc6)
        return conv, [{"weight": l.weight, "bias": l.bias, "bn": None, "relu": i < 5} for i, l in enumerate(fcs)]

    def _check_call(self):
        if self.net.training:
            raise ValueError("%s: the wrapped module is in training mode" % type(self).__name__)
        if torch.is_grad_enabled() and any(p.requires_grad for n, p in self.net.named_parameters() if not n.startswith("sampler.")):
            raise ValueError("%s gives no parameter gradients: freeze the wrapped module (requires_grad_(False)) or disable grad"
                             % type(self).__name__)

    @staticmethod
    def _encode(clouds, conv, m):
        from . import ops

        return ops.FrozenEncoderFunction.apply(clouds, conv, [m])[0]

    @staticmethod
    def _head(feat, fc):
        from . import ops

        return ops.FrozenMLPFunction.apply(feat, fc)

    def supported(self, b, m0, m1):
        """Whether b pairs of a template of m0 points and a source of m1 are inside the kernels' envelopes (raw does not return None)."""
        from . import ops

        conv, fc = self._specs()
        half = self.ENCODER_ROWS // 2
        if b < 1 or not ops.frozen_mlp_supported(min(b, half), fc):
            return False
        if m0 == m1:
            return ops.frozen_encoder_supported(min(2 * b, self.ENCODER_ROWS), m0, conv, 1)
        return ops.frozen_encoder_supported(min(b, half), m0, conv, 1) and ops.frozen_encoder_supported(min(b, half), m1, conv, 1)

    def raw(self, x0, x1):
        """fc6's output (B, 7), or None when a shape is outside the kernels' envelopes."""
        self._check_call()
        if self.net.input_shape == "bcn":
            x0, x1 = x0.permute(0, 2, 1), x1.permute(0, 2, 1)
        if x0.dim() != 3 or x0.shape[2] != 3 or x1.dim() != 3 or x1.shape[2] != 3:
            raise RuntimeError("shape of x must be of [Batch x 3 x NumInPoints]" if self.net.input_shape == "bcn" else
                               "shape of x must be of [Batch x NumInPoints x 3]")
        for t in (x0, x1):
            if not t.is_cuda:
                raise RuntimeError("samplenet_b200: the input is on %s; the ops are CUDA-only (no CPU fallback)" % t.device)
        b, m0, m1 = x0.shape[0], x0.shape[1], x1.shape[1]
        if x1.shape[0] != b or not self.supported(b, m0, m1):
            return None
        conv, fc = self._specs()
        half = self.ENCODER_ROWS // 2
        rows = []
        for s in range(0, b, half):     # up to 32 pairs: the encoder's pooled features of template and source, then their MLP rows
            c0, c1 = x0[s:s + half], x1[s:s + half]
            if m0 == m1:                # one (2 B', m, 3) cloud batch
                pooled = self._encode(torch.cat([c0, c1], dim=0).contiguous(), conv, m0)
                f0, f1 = pooled[0, :c0.shape[0]], pooled[0, c0.shape[0]:]
            else:
                f0, f1 = self._encode(c0.contiguous(), conv, m0)[0], self._encode(c1.contiguous(), conv, m1)[0]
            rows.append(self._head(torch.cat([f0, f1], dim=1), fc))
        return rows[0] if len(rows) == 1 else torch.cat(rows, dim=0)

    def forward(self, x0, x1):
        y = self.raw(x0, x1)
        if y is None:
            return self.net(x0, x1)
        pre_normalized_quat = y[:, 0:4]
        return torch.cat([F.normalize(pre_normalized_quat, dim=1), y[:, 4:]], dim=1), pre_normalized_quat


class CudaPCRNet(FrozenPCRNet):
    """PCRNet(pcrnet) on the same CUDA kernels as FrozenPCRNet, trainable: the parameters that require grad receive gradients
    (csrc/frozen_encoder.cu and csrc/frozen_mlp.cu's parameter backward; PCRNet has no BatchNorm and no dropout, so its training forward is
    the frozen forward).  forward(x0, x1) -> (twist, pre_normalized_quat) as the module, template and source of up to 32 pairs through the
    encoder calls FrozenPCRNet makes (autograd adds the parameter gradients of two calls in a fixed order); shapes outside the kernels'
    envelopes run the wrapped module.  train(mode) sets the wrapped module's mode (and its
    sampler's, as nn.Module.train does).  The parameters are the wrapped module's: an optimiser over filter(requires_grad, parameters())
    sees what it sees on a plain PCRNet, and net.state_dict() keeps PCRNet's keys."""

    def __init__(self, pcrnet):
        super().__init__(pcrnet)
        self.training = pcrnet.training

    def train(self, mode=True):
        return nn.Module.train(self, mode)

    def _check_call(self):
        pass

    @staticmethod
    def _encode(clouds, conv, m):
        from . import ops

        params = [t for c in conv for t in (c["weight"], c["bias"])]
        return ops.EncoderParamFunction.apply(clouds, [m], [c["relu"] for c in conv], *params)[0]

    @staticmethod
    def _head(feat, fc):
        from . import ops

        return ops.MLPParamFunction.apply(feat, [l["relu"] for l in fc], *[t for l in fc for t in (l["weight"], l["bias"])])


# ----------------------------------------------------------------------------------------------------- quaternions
def qrot(q, v):
    """Rotate v (*, 3) by the (w, x, y, z) quaternion q (*, 4)  (registration/src/quaternion.py:35-53)."""
    shape = list(v.shape)
    q = q.reshape(-1, 4)
    v = v.reshape(-1, 3)
    qvec = q[:, 1:]
    uv = torch.cross(qvec, v, dim=1)
    uuv = torch.cross(qvec, uv, dim=1)
    return (v + 2 * (q[:, :1] * uv + uuv)).view(shape)


def qinv(q):
    """Conjugate of a (w, x, y, z) quaternion."""
    return torch.cat([q[..., :1], -q[..., 1:]], dim=-1)


def quaternion_to_rotation_matrix(quaternion):
    """(x, y, z, w) -> (.., 3, 3); what `kornia.geometry.conversions.quaternion_to_rotation_matrix` computes (qdataset.py:74-75)."""
    q = F.normalize(quaternion, p=2, dim=-1, eps=1e-12)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    one = torch.ones_like(x)
    m = torch.stack([one - (tyy + tzz), txy - twz, txz + twy, txy + twz, one - (txx + tzz), tyz - twx, txz - twy, tyz + twx, one - (txx + tyy)], dim=-1)
    return m.view(quaternion.shape[:-1] + (3, 3))


class QuaternionTransform:
    def __init__(self, vec, inverse=False):
        self._inversion = torch.tensor([inverse])
        self.vec = vec.view([-1, 7])

    @staticmethod
    def from_dict(d, device):
        return QuaternionTransform(d["vec"].to(device), d["inversion"][0].item())

    def inverse(self):
        return QuaternionTransform(torch.cat([qinv(self.quat()), -self.trans()], dim=1), inverse=(not self.inversion()))

    def as_dict(self):
        return {"inversion": self._inversion, "vec": self.vec}

    def quat(self):
        return self.vec[:, 0:4]

    def trans(self):
        return self.vec[:, 4:]

    def inversion(self):
        return self._inversion[0].item()

    def compute_errors(self, other):
        q1, q2 = self.quat(), other.quat()
        R1 = quaternion_to_rotation_matrix(q1[..., [1, 2, 3, 0]])
        R2 = quaternion_to_rotation_matrix(q2[..., [1, 2, 3, 0]])
        R1_R2inv = torch.bmm(R1, R2.transpose(1, 2))
        rot_err = torch.mean(2 * torch.acos(2 * (torch.sum(q1 * q2, dim=1)) ** 2 - 1))
        eye = torch.eye(3).unsqueeze(0).expand([R1_R2inv.shape[0], -1, -1]).to(R1_R2inv)
        norm_err = torch.mean(torch.sum((R1_R2inv - eye) ** 2, dim=(1, 2)))
        trans_err = torch.mean(torch.sqrt((self.trans() - other.trans()) ** 2))
        return rot_err, norm_err, trans_err

    def rotate(self, p):
        if p.dim() == 2:
            assert self.vec.shape[0] == 1
            return qrot(self.quat().expand([p.shape[0], -1]), p)
        quat = self.quat().unsqueeze(1).expand([-1, p.shape[1], -1]).contiguous()
        return qrot(quat, p)


def rad_to_deg(rad):
    return 180 / math.pi * rad


# ----------------------------------------------------------------------------------------------------- the data set
def random_transforms(count, seed, max_rotation_deg=45, max_translation=0):
    """The fixed transform table of QuaternionFixedDataset(data, repeat, seed) (qdataset.py:122-144), (count, 7) float32 rows
    (w, x, y, z, tx, ty, tz), bit for bit: per record uniform(-r, r, 3) then uniform(-t, t, 3) (the translation draws are consumed at t = 0
    too), euler_to_quaternion(rot, "xyz") in float64 with qmul's term order, negated, then rounded to float32.  The draws come from a
    private np.random.RandomState(seed); numpy's global state is left alone."""
    rs = np.random.RandomState(seed)
    max_rotation = np.pi / 180 * max_rotation_deg
    u = rs.random_sample((count, 6))        # uniform(low, high) is low + (high - low) * random_sample(), in draw order
    rot = -max_rotation + (max_rotation - -max_rotation) * u[:, :3]
    trans = -max_translation + (max_translation - -max_translation) * u[:, 3:]
    half = rot / 2
    c, s, z = np.cos(half), np.sin(half), np.zeros(count)
    rx = np.stack([c[:, 0], s[:, 0], z, z], axis=1)
    ry = np.stack([c[:, 1], z, s[:, 1], z], axis=1)
    rz = np.stack([c[:, 2], z, z, s[:, 2]], axis=1)

    def qmul(q, r):   # registration/src/quaternion.py:14-32: terms[a, b] = r[a] q[b], summed left to right
        t = r[:, :, None] * q[:, None, :]
        return np.stack([t[:, 0, 0] - t[:, 1, 1] - t[:, 2, 2] - t[:, 3, 3], t[:, 0, 1] + t[:, 1, 0] - t[:, 2, 3] + t[:, 3, 2],
                         t[:, 0, 2] + t[:, 1, 3] + t[:, 2, 0] - t[:, 3, 1], t[:, 0, 3] - t[:, 1, 2] + t[:, 2, 1] + t[:, 3, 0]], axis=1)

    quat = -qmul(qmul(rx, ry), rz)
    return np.concatenate([quat, trans], axis=1).astype(np.float32)


def on_unit_cube(points):
    """OnUnitCube.method2 (registration/src/pctransforms.py:162-166) per cloud of points (..., N, 3): divide by the largest axis extent,
    then subtract the mean.  Torch ops on the points' device."""
    c = points.amax(dim=-2) - points.amin(dim=-2)
    v = points / c.amax(dim=-1, keepdim=True).unsqueeze(-1)
    return v - v.mean(dim=-2, keepdim=True)


class CudaQuaternionFixedDataset:
    """ModelNetCls(num_points, OnUnitCube) + QuaternionFixedDataset(repeat, seed) (registration/data/modelnet_loader_torch.py,
    registration/src/qdataset.py:122-179) on the device.  points (S, P, 3), numpy or a tensor, is the set as read from the h5 files; the
    first min(P, num_points) points of each cloud are kept and put on the unit cube once, at construction (the reference normalises each
    item over the same point set, so only the summation order of the mean differs).  Record r is cloud r % S with transform row r of
    random_transforms(S * repeat, seed).  batch(records) builds the pairs of any records with one ops.registration_pairs launch, each cloud
    in a fresh random point order (torch's CUDA generator; numpy's permutation stream is not reproduced).  The set lives on the points'
    device when they are a CUDA tensor, on the current CUDA device otherwise."""

    def __init__(self, points, num_points=1024, repeat=1, seed=0):
        if not isinstance(points, torch.Tensor):
            points = torch.from_numpy(np.ascontiguousarray(points))
        if points.dim() != 3 or points.shape[2] != 3 or points.shape[0] < 1 or points.shape[1] < 1:
            raise ValueError("CudaQuaternionFixedDataset expects points of shape (clouds >= 1, points >= 1, 3), got %s" % (tuple(points.shape),))
        if int(num_points) < 1 or int(repeat) < 1:
            raise ValueError("num_points and repeat must be >= 1, got %r and %r" % (num_points, repeat))
        dev = points.device if points.is_cuda else torch.device("cuda", torch.cuda.current_device())
        self.num_points = min(points.shape[1], int(num_points))
        self.clouds = on_unit_cube(points[:, :self.num_points].to(device=dev, dtype=torch.float32)).contiguous()
        self.len_data, self.repeat, self.seed = points.shape[0], int(repeat), seed
        self.transforms = torch.from_numpy(random_transforms(len(self), seed)).to(dev)

    def __len__(self):
        return self.len_data * self.repeat

    @property
    def device(self):
        return self.clouds.device

    def batch(self, records):
        """(p0, p1, igt) for the records (a (B,) integer tensor or sequence): p0 (B, n, 3) the clouds in a random point order, p1 = p0 rotated
        by each record's fixed quaternion, igt = {"vec": (B, 7) on the device, "inversion": tensor([False]) on the host}, as the reference's
        DataLoader collates them.  One launch; the records are not range-checked (that would read them back)."""
        from . import ops

        if not isinstance(records, torch.Tensor):
            records = torch.tensor(records, dtype=torch.int32)
        p0, p1, vec = ops.registration_pairs(self.clouds, records.to(self.device), self.transforms)
        return p0, p1, {"vec": vec, "inversion": torch.tensor([False])}

    def batches(self, batch_size, shuffle=False, drop_last=False):
        """Yield batch() over every record in order, or shuffled with torch.randperm on the device; the last partial batch is yielded unless
        drop_last, as DataLoader(batch_size, shuffle, drop_last) does."""
        total = len(self)
        order = (torch.randperm(total, device=self.device, dtype=torch.int32) if shuffle
                 else torch.arange(total, device=self.device, dtype=torch.int32))
        for s in range(0, total, batch_size):
            if drop_last and s + batch_size > total:
                return
            yield self.batch(order[s:s + batch_size])


def get_datasets(train_points, test_points, num_points=1024, test=False):
    """get_datasets of registration/main.py:601-637 on CudaQuaternionFixedDataset, the h5 files read by the caller: (trainset, testset)
    with repeat = max(int(5000 / S), 1) and seed 0 for the training set and repeat 1, seed 0 for the test set; with test=True
    (None, the test set with repeat 5 and seed 1)."""
    if test:
        return None, CudaQuaternionFixedDataset(test_points, num_points, repeat=5, seed=1)
    train_repeats = max(int(5000 / len(train_points)), 1)
    return (CudaQuaternionFixedDataset(train_points, num_points, repeat=train_repeats, seed=0),
            CudaQuaternionFixedDataset(test_points, num_points, repeat=1, seed=0))


# ----------------------------------------------------------------------------------------------------- the step
class RegistrationStep:
    """`Action` of registration/main.py: same hyper-parameter names, same loss assembly.  `sampler` is main.py's --sampler:
    "samplenet" (default), "fps", "random" or "none".

    graphed=True runs every whole batch of train_1 as one CUDA-graph replay instead of the step's launches from Python, with the same
    results bit for bit (parameters, buffers, optimiser state, CUDA RNG state, returned means).  The graph holds train_step on static p0, p1
    and igt["vec"] buffers -- the losses, zero_grad, backward, optimizer.step() -- and the addition of (loss, rot_err) into a float64
    accumulator.  Building each batch (the pairs launch and its key draw), its device-to-device copy into the static buffers, zeroing the
    accumulator and the one read-back stay outside.  The step is captured at the first batch of the first train_1 call, so a checkpoint
    restored before that is what is captured, and never again.  A trailing smaller batch (DataLoader's last partial batch) runs eagerly on
    the same parameters and optimiser state and its row is added last.  The runner holds one model, one optimiser, one batch shape and
    one igt["inversion"] value (a host tensor, read at capture): another raises ValueError.  Refused with ValueError before any capture:
    sampler "fps" (it draws its permutation on the CPU generator on every call, which a graph would freeze), wrap_data_parallel, an
    optimiser that fails graphs.check_capturable (main.py's Adam and RMSprop pass with capturable=True, its SGD does not), a model that is
    not a FrozenPCRNet or CudaPCRNet with input_shape "bnc", and a batch on which compute_pcrnet_loss would leave the fused CUDA path.  A
    graphed runner keeps a private memory pool and the static buffers for its lifetime."""

    SAMPLERS = ("samplenet", "fps", "random", "none")

    def __init__(self, num_out_points=64, bottleneck_size=128, group_size=8, alpha=0.01, lmbda=0.01, gamma=1, delta=0, loss_type=0,
                 num_sampled_clouds=2, skip_projection=False, train_samplenet=True, train_pcrnet=False, sampler="samplenet", graphed=False):
        if sampler not in self.SAMPLERS:
            raise ValueError("sampler must be one of %s, got %r" % (", ".join(self.SAMPLERS), sampler))
        self.graphed = bool(graphed)
        if self.graphed and sampler == "fps":
            raise ValueError("RegistrationStep(graphed=True) cannot train with sampler='fps': FPSSampler draws its point permutation on the "
                             "CPU generator on every call, and a graph would replay one permutation")
        self.SAMPLER = sampler
        self.ALPHA, self.LMBDA, self.GAMMA, self.DELTA = alpha, lmbda, gamma, delta
        self.NUM_OUT_POINTS, self.BOTTLNECK_SIZE, self.GROUP_SIZE = num_out_points, bottleneck_size, group_size
        self.LOSS_TYPE, self.NUM_SAMPLED_CLOUDS, self.SKIP_PROJECTION = loss_type, num_sampled_clouds, skip_projection
        self.TRAIN_SAMPLENET, self.TRAIN_PCRNET = train_samplenet, train_pcrnet
        self._ddp = None
        self._graph = None          # graphed: the trainers._StepGraph of the one model and optimiser, made by the first train_1
        self._inversion = None      # graphed: igt["inversion"] of the captured batch

    def create_model(self, frozen_task=False, cuda_task=False):
        """The task network with the sampler attached.  frozen_task=True returns it wrapped in FrozenPCRNet (the CUDA path of the frozen
        task half); that needs train_pcrnet=False.  cuda_task=True returns it wrapped in CudaPCRNet (the same kernels with parameter
        gradients), with train_pcrnet True or False."""
        if frozen_task and cuda_task:
            raise ValueError("frozen_task and cuda_task select two different wrappers: pass one of them")
        if frozen_task and self.TRAIN_PCRNET:
            raise ValueError("frozen_task=True runs PCRNet frozen: it cannot be combined with train_pcrnet=True")
        model = PCRNet(input_shape="bnc")
        model.requires_grad_(self.TRAIN_PCRNET)
        model.train(self.TRAIN_PCRNET)
        if self.SAMPLER == "samplenet":
            sampler = SampleNet(num_out_points=self.NUM_OUT_POINTS, bottleneck_size=self.BOTTLNECK_SIZE, group_size=self.GROUP_SIZE,
                                initial_temperature=1.0, input_shape="bnc", output_shape="bnc", skip_projection=self.SKIP_PROJECTION)
            sampler.requires_grad_(self.TRAIN_SAMPLENET)
            sampler.train(self.TRAIN_SAMPLENET)
        elif self.SAMPLER == "fps":
            sampler = FPSSampler(self.NUM_OUT_POINTS, permute=True, input_shape="bnc", output_shape="bnc")
        elif self.SAMPLER == "random":
            sampler = RandomSampler(self.NUM_OUT_POINTS, input_shape="bnc", output_shape="bnc")
        else:
            sampler = None
        model.sampler = sampler
        if frozen_task:
            return FrozenPCRNet(model)
        return CudaPCRNet(model) if cuda_task else model

    def non_learned_sampling(self, model, data, device):
        """Sample p1 (and p0 when NUM_SAMPLED_CLOUDS == 2) with the FPS or random sampler."""
        p0, p1, igt = data
        p0, p1 = p0.to(device), p1.to(device)
        p1_samp = model.sampler(p1)
        if self.NUM_SAMPLED_CLOUDS == 1:
            return (p0, p1_samp, igt)
        return (model.sampler(p0), p1_samp, igt)

    def compute_samplenet_loss(self, model, data, device):
        p0, p1, igt = data
        p0, p1 = p0.to(device), p1.to(device)
        p1_simplified, p1_projected = model.sampler(p1)
        p1_loss = model.sampler.get_simplification_loss(p1, p1_simplified, self.NUM_OUT_POINTS, self.GAMMA, self.DELTA)
        if self.NUM_SAMPLED_CLOUDS == 1:
            simplification_loss = p1_loss
            sampled_data = (p0, p1_projected, igt)
        else:
            p0_simplified, p0_projected = model.sampler(p0)
            p0_loss = model.sampler.get_simplification_loss(p0, p0_simplified, self.NUM_OUT_POINTS, self.GAMMA, self.DELTA)
            simplification_loss = 0.5 * (p1_loss + p0_loss)
            sampled_data = (p0_projected, p1_projected, igt)
        projection_loss = model.sampler.get_projection_loss()
        samplenet_loss = self.ALPHA * simplification_loss + self.LMBDA * projection_loss
        return samplenet_loss, sampled_data, {"simplification_loss": simplification_loss, "projection_loss": projection_loss}

    def compute_sampling_consistency(self, sampled_data, device):
        p0s, p1s, igt = sampled_data
        p0s, p1s = p0s.to(device), p1s.to(device)
        p0s_est = QuaternionTransform.from_dict(igt, device).inverse().rotate(p1s)
        c01, c10 = ChamferDistance()(p0s, p0s_est)
        return torch.mean(c01) + torch.mean(c10)

    def compute_pcrnet_loss(self, model, data, device, epoch=0):
        p0, p1, igt = data
        p0, p1 = p0.to(device), p1.to(device)
        if isinstance(model, FrozenPCRNet):
            fused = self._frozen_pcrnet_loss(model, p0, p1, igt, device)
            if fused is not None:
                return fused
        twist, pre_normalized_quat = model(p0, p1)
        qnorm_loss = torch.mean((torch.sum(pre_normalized_quat ** 2, dim=1) - 1) ** 2)
        est_transform = QuaternionTransform(twist)
        gt_transform = QuaternionTransform.from_dict(igt, device)
        p1_est = est_transform.rotate(p0)
        c01, c10 = ChamferDistance()(p1, p1_est)
        chamfer_loss = torch.mean(c01) + torch.mean(c10)
        rot_err, norm_err, trans_err = est_transform.compute_errors(gt_transform)
        pcrnet_loss = 1.0 * norm_err + 1.0 * chamfer_loss if self.LOSS_TYPE == 0 else chamfer_loss
        return pcrnet_loss, {"chamfer_loss": chamfer_loss, "qnorm_loss": qnorm_loss, "rot_err": rad_to_deg(rot_err), "norm_err": norm_err,
                             "trans_err": trans_err, "est_transform": est_transform}

    def _frozen_pcrnet_loss(self, model, p0, p1, igt, device):
        """compute_pcrnet_loss on the CUDA path: frozen encoder -> frozen MLP -> one fused pose-loss launch (ops.PoseLossFunction).  None
        when a shape is outside a kernel's envelope (the caller then runs the torch ops on the wrapper's output).  The template and the
        source may differ in size (one sampled cloud)."""
        from . import ops

        if (model.input_shape != "bnc" or p0.dim() != 3 or p1.dim() != 3 or p0.shape[0] != p1.shape[0]
                or not ops.pose_loss_supported(p0.shape[0], p0.shape[1], p1.shape[1])):
            return None
        y = model.raw(p0, p1)
        if y is None:
            return None
        gt_vec = QuaternionTransform.from_dict(igt, device).vec.to(torch.float32)
        terms, twist = ops.PoseLossFunction.apply(y, p0, p1, gt_vec)
        chamfer_loss, qnorm_loss, norm_err, rot_err, trans_err = terms.unbind(0)
        pcrnet_loss = 1.0 * norm_err + 1.0 * chamfer_loss if self.LOSS_TYPE == 0 else chamfer_loss
        return pcrnet_loss, {"chamfer_loss": chamfer_loss, "qnorm_loss": qnorm_loss, "rot_err": rad_to_deg(rot_err), "norm_err": norm_err,
                             "trans_err": trans_err, "est_transform": QuaternionTransform(twist)}

    # one iteration of Action.train_1 (main.py:306-362); data-parallel when torch.distributed is initialised
    def wrap_data_parallel(self, model):
        if self.graphed:
            raise ValueError("RegistrationStep(graphed=True) runs on one GPU: build it with graphed=False to train data-parallel")
        self._ddp = FlatBucketDataParallel(model.sampler)
        return self._ddp

    def train_step(self, model, data, optimizer, device):
        name = model.sampler.name if model.sampler is not None else None
        if name == "samplenet":
            sampler_loss, sampled_data, info = self.compute_samplenet_loss(model, data, device)
        else:  # main.py:321-330: no sampler loss; train_1 samples only with FPS, other samplers train on the full clouds
            sampled_data = self.non_learned_sampling(model, data, device) if name == "fps" else data
            zero = torch.tensor(0, dtype=torch.float32)
            sampler_loss, info = zero, {"simplification_loss": zero, "projection_loss": zero}
        pcrnet_loss, pinfo = self.compute_pcrnet_loss(model, sampled_data, device)
        loss = pcrnet_loss + sampler_loss
        if self._ddp is not None:
            self._ddp.zero_grad()
        else:
            optimizer.zero_grad()
        loss.backward()
        if self._ddp is not None:
            self._ddp.sync_gradients()
            self._ddp.wait()
        optimizer.step()
        return loss.detach(), pinfo["rot_err"].detach(), info

    def train_1(self, model, batches, optimizer, device, epoch=0):
        """`Action.train_1` (main.py:306-362): train_step over every (p0, p1, igt) of `batches` (a CudaQuaternionFixedDataset's batches(...)
        or a DataLoader) -> (ave_vloss, ave_gloss), the means over the batches of the total loss and of the rotation error in degrees.  The
        per-batch values are summed in float64 on the device, in batch order as the reference's host sums of .item(), and read back once.
        As in the reference, a trailing batch of one cloud fails in a training SampleNet's BatchNorm: pass drop_last=True, or a batch size
        that leaves no such remainder.  With graphed=True every whole batch is one graph replay (see the class)."""
        if self.graphed:
            return self._train_1_graphed(model, batches, optimizer, device)
        acc = None
        count = 0
        for data in batches:
            loss, rot_err, _ = self.train_step(model, data[0:3], optimizer, device)
            row = self._row(loss, rot_err)
            acc = row if acc is None else acc + row
            count += 1
        if acc is None:
            raise ValueError("train_1: no batches")
        ave = acc.cpu()
        return float(ave[0]) / count, float(ave[1]) / count

    @staticmethod
    def _row(loss, rot_err):
        return torch.stack([loss.reshape(()), rot_err.reshape(()).to(loss.device)]).double()

    # ------------------------------------------------------------------------------------------------- graphed train_1
    def _graph_runner(self, model, optimizer):
        """The runner's _StepGraph, made on the first call; ValueError, before any CUDA work, for what the graph cannot hold."""
        if self._graph is not None:
            if model is not self._graph.modules[0] or optimizer is not self._graph.optimizer:
                raise ValueError("RegistrationStep(graphed=True) holds the model and the optimiser of its first train_1 call; build another "
                                 "RegistrationStep for another model or optimiser")
            return self._graph
        if not isinstance(model, FrozenPCRNet) or model.input_shape != "bnc":
            raise ValueError("RegistrationStep(graphed=True) needs the CUDA task network, create_model(frozen_task=True) or "
                             "create_model(cuda_task=True) with input_shape 'bnc', got %s: the plain PCRNet's torch ops would be "
                             "captured instead of the fused pose loss" % type(model).__name__)
        if model.sampler is not None and model.sampler.name == "fps":
            raise ValueError("RegistrationStep(graphed=True) cannot train with an FPS sampler: it draws its point permutation on the CPU "
                             "generator on every call, and a graph would replay one permutation")
        from .graphs import check_capturable

        check_capturable(optimizer, "RegistrationStep(graphed=True)")
        self._graph = _StepGraph(self, self._graph_step, [model], optimizer, ())
        return self._graph

    def _check_capture(self, model, p0, p1):
        """ValueError unless train_step on this batch runs the fused CUDA path (compute_pcrnet_loss would otherwise run torch ops)."""
        from . import ops

        if p0.dim() != 3 or p1.dim() != 3 or p0.shape[2] != 3 or p1.shape[2] != 3 or p1.shape[0] != p0.shape[0]:
            raise ValueError("RegistrationStep(graphed=True) expects p0 and p1 of shape (batch, points, 3), got %s and %s"
                             % (tuple(p0.shape), tuple(p1.shape)))
        b, m0, m1 = p0.shape[0], p0.shape[1], p1.shape[1]
        if model.sampler is not None and model.sampler.name == "samplenet":   # the clouds compute_pcrnet_loss sees
            m1 = model.sampler.num_out_points
            m0 = m1 if self.NUM_SAMPLED_CLOUDS == 2 else m0
        if not (ops.pose_loss_supported(b, m0, m1) and model.supported(b, m0, m1)):
            raise ValueError("RegistrationStep(graphed=True): %d pairs of %d and %d points are outside the CUDA task network's and the pose "
                             "loss's envelopes" % (b, m0, m1))

    def _graph_step(self, p0, p1, vec):
        loss, rot_err, _ = self.train_step(self._graph.modules[0], (p0, p1, {"vec": vec, "inversion": self._inversion}),
                                           self._graph.optimizer, p0.device)
        return None, [loss.reshape(()), rot_err.reshape(())]

    def _train_1_graphed(self, model, batches, optimizer, device):
        g = self._graph_runner(model, optimizer)
        count, partial = 0, False
        for data in batches:
            p0, p1, igt = data[0:3]
            if partial:
                raise ValueError("RegistrationStep(graphed=True): only the last batch of an epoch may be smaller than the captured batch")
            if g.captured is None:
                self._check_capture(model, p0, p1)
                self._inversion = igt["inversion"].clone()
            elif bool(igt["inversion"][0]) != bool(self._inversion[0]):
                raise ValueError("RegistrationStep(graphed=True) captured igt['inversion'] = %s; got %s"
                                 % (bool(self._inversion[0]), bool(igt["inversion"][0])))
            p0, p1, vec = p0.to(device), p1.to(device), igt["vec"].to(device)
            s0, s1 = (None, None) if g.captured is None else (g.inputs[0].shape, g.inputs[1].shape)
            if s0 is not None and p0.shape[0] < s0[0] and p1.shape[0] == p0.shape[0] and p0.shape[1:] == s0[1:] and p1.shape[1:] == s1[1:]:
                # a smaller batch of the captured clouds (a trailing partial batch): eagerly, on the parameters and optimiser state the
                # graph updates, its row added last
                if count == 0:
                    g.acc.zero_()
                loss, rot_err, _ = self.train_step(model, (p0, p1, igt), optimizer, device)
                g.acc += self._row(loss, rot_err)
                partial = True
            else:
                g.bind(p0, p1, vec)
                g.replay(None, first_of_epoch=count == 0)      # no schedule: captured once
            count += 1
        if count == 0:
            raise ValueError("train_1: no batches")
        ave = g.acc.cpu()
        return float(ave[0]) / count, float(ave[1]) / count

    # ------------------------------------------------------------------------------------------------- evaluation
    def _sample_for_eval(self, model, data, device, samplers):
        """(sampler_loss, sampled_data) as eval_1 / test_1 choose them: main.py:378-389 samples with "samplenet" and "fps" (`samplers`),
        :428-437 with "random" as well; any other sampler leaves the clouds whole."""
        name = model.sampler.name if model.sampler is not None else None
        if name == "samplenet":
            sampler_loss, sampled_data, _ = self.compute_samplenet_loss(model, data, device)
            return sampler_loss, sampled_data
        zero = torch.tensor(0, dtype=torch.float32)
        return zero, (self.non_learned_sampling(model, data, device) if name in samplers else data)

    def eval_1(self, model, batches, device, epoch=0):
        """`Action.eval_1` (main.py:364-414): (ave_vloss, ave_gloss), the means over the batches of the total loss and of the rotation error
        in degrees.  `batches` yields (p0, p1, igt) with igt = {"vec": (B, 7), "inversion": tensor([False])}.  The task network and the
        sampler run in eval mode and get their modes back; the per-batch values stay on the device and are read back once."""
        net = model.net if isinstance(model, FrozenPCRNet) else model
        rows = []
        with eval_mode(net):
            for data in batches:
                sampler_loss, sampled_data = self._sample_for_eval(model, data[0:3], device, ("fps",))
                pcrnet_loss, info = self.compute_pcrnet_loss(model, sampled_data, device, epoch)
                rows.append(torch.stack([(pcrnet_loss + sampler_loss.to(pcrnet_loss.device)).float(), info["rot_err"].float()]))
            if not rows:
                raise ValueError("eval_1: no batches")
            ave = torch.stack(rows).double().mean(dim=0).cpu()
        return float(ave[0]), float(ave[1])

    def test_1(self, model, batches, device, epoch=0):
        """`Action.test_1` (main.py:416-483) on batches of any size: per record the rotation error (degrees), the translation error and the
        sampling consistency the reference's batch-1 loop appends, then the precision curve over np.arange(0, 180, 0.5), its AUC and the
        means / standard deviations it prints.  A batch changes nothing for a record beyond fp32 rounding: every network is in eval mode
        and every op works per cloud, so a record's values do not depend on its neighbours (a few 1e-4 degrees between batch sizes, from
        summation orders that depend on the row count; the "fps" and "random" samplers draw from the random generator per call, so
        their records repeat only under the same batching and seed).  With a FrozenPCRNet a batch is one pass: model.raw and
        one ops.pose_eval launch for every pair; a plain PCRNet, or a shape outside the kernels' envelopes, runs the torch ops record by
        record.  One host read-back for the whole call."""
        from . import ops

        net = model.net if isinstance(model, FrozenPCRNet) else model
        cols = []        # (3, B) per batch: rot_err in degrees, trans_err, consistency
        with eval_mode(net):
            for data in batches:
                _, (p0s, p1s, igt) = self._sample_for_eval(model, data[0:3], device, ("fps", "random"))
                p0s, p1s = p0s.to(device), p1s.to(device)
                gt_vec = QuaternionTransform.from_dict(igt, device).vec.to(torch.float32)
                y = None
                if (isinstance(model, FrozenPCRNet) and model.input_shape == "bnc" and p0s.dim() == 3 and p1s.dim() == 3
                        and p0s.shape[0] == p1s.shape[0] and ops.pose_eval_supported(p0s.shape[0], p0s.shape[1], m1=p1s.shape[1])):
                    y = model.raw(p0s, p1s)
                if y is not None:
                    per_pair, _ = ops.pose_eval(y, p0s, p1s, gt_vec, p0s, p1s)
                    cols.append(torch.stack([rad_to_deg(per_pair[:, 3]), per_pair[:, 4], per_pair[:, 5]]))
                    continue
                for i in range(p0s.shape[0]):
                    one = (p0s[i:i + 1], p1s[i:i + 1], {"vec": gt_vec[i:i + 1], "inversion": igt["inversion"]})
                    _, info = self.compute_pcrnet_loss(model, one, device, epoch)
                    cols.append(torch.stack([info["rot_err"], info["trans_err"], self.compute_sampling_consistency(one, device)]).float()[:, None])
            if not cols:
                raise ValueError("test_1: no batches")
            rot, trans, cons = torch.cat(cols, dim=1).cpu().numpy().astype(np.float64)
        x, y, auc = precision_curve(rot)
        return {"rotation_errors": rot, "trans_errs": trans, "consistency_errors": cons, "precision_x": x, "precision_y": y, "auc": auc,
                "mean_rotation_error": float(np.mean(rot)), "std_rotation_error": float(np.std(rot)),
                "mean_trans_err": float(np.mean(trans)), "std_trans_err": float(np.std(trans)),
                "mean_consistency_error": float(np.mean(cons)), "std_consistency_error": float(np.std(cons))}
