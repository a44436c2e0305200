"""The registration trainer's step, restated over this package (SURVEY.md 8f ranks 1 and 4): the callers of the hot path.

    PCRNet / PointNetFeatures     registration/models/pcrnet.py:8-82         (task network; stock torch layers, same state-dict keys)
    QuaternionTransform           registration/src/qdataset.py:17-119        ((w,x,y,z) quaternion + translation, kornia-free)
    qrot / qinv                   registration/src/quaternion.py:35-53, qinv
    RegistrationStep              registration/main.py:221-247 (hyper-parameters), :249-298 (create_model), :485-498
                                  (non_learned_sampling), :500-538
                                  (compute_samplenet_loss), :540-553 (compute_sampling_consistency), :555-598 (compute_pcrnet_loss),
                                  :306-362 (train_1: loss = pcrnet_loss + sampler_loss; zero_grad; backward; step)

The sampler is this package's SampleNet (CUDA kernels) or, for `sampler="fps"` / `"random"`, its FPSSampler / RandomSampler, Chamfer is this package's ChamferDistance; the task network is the reference's
architecture in stock torch ops (it is a caller of the path, not the path).  `RegistrationStep.train_step` is one iteration of
`Action.train_1`; with torch.distributed initialised the sampler's gradients go through `FlatBucketDataParallel` (one flat all-reduce).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .chamfer_distance import ChamferDistance
from .parallel import FlatBucketDataParallel
from .samplenet import SampleNet
from .samplers import FPSSampler, RandomSampler


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


# ----------------------------------------------------------------------------------------------------- the step
class RegistrationStep:
    """`Action` of registration/main.py: same hyper-parameter names, same loss assembly.  `sampler` is main.py's --sampler:
    "samplenet" (default), "fps", "random" or "none"."""

    SAMPLERS = ("samplenet", "fps", "random", "none")

    def __init__(self, num_out_points=64, bottleneck_size=128, group_size=8, alpha=0.01, lmbda=0.01, gamma=1, delta=0, loss_type=0,
                 num_sampled_clouds=2, skip_projection=False, train_samplenet=True, train_pcrnet=False, sampler="samplenet"):
        if sampler not in self.SAMPLERS:
            raise ValueError("sampler must be one of %s, got %r" % (", ".join(self.SAMPLERS), sampler))
        self.SAMPLER = sampler
        self.ALPHA, self.LMBDA, self.GAMMA, self.DELTA = alpha, lmbda, gamma, delta
        self.NUM_OUT_POINTS, self.BOTTLNECK_SIZE, self.GROUP_SIZE = num_out_points, bottleneck_size, group_size
        self.LOSS_TYPE, self.NUM_SAMPLED_CLOUDS, self.SKIP_PROJECTION = loss_type, num_sampled_clouds, skip_projection
        self.TRAIN_SAMPLENET, self.TRAIN_PCRNET = train_samplenet, train_pcrnet
        self._ddp = None

    def create_model(self):
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
        return model

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

    # one iteration of Action.train_1 (main.py:306-362); data-parallel when torch.distributed is initialised
    def wrap_data_parallel(self, model):
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
