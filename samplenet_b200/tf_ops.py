"""TF-named functional surface, as torch functions on CUDA tensors, so that the classification / reconstruction trainers
can be restated 1:1 (SURVEY.md 8b):

    nn_distance          classification/structural_losses/tf_nndistance.py:12-47
    approx_match         classification/structural_losses/tf_approxmatch.py:13-33   (no gradient, like ops.NoGradient)
    match_cost           classification/structural_losses/tf_approxmatch.py:35-64   (grads to xyz1, xyz2 only)
    knn_point            classification/grouping/tf_grouping.py:64-91
    group_point          classification/grouping/tf_grouping.py:46-61
    farthest_point_sample  reconstruction/external/sampling/tf_sampling.py:65-76  (no gradient, like ops.NoGradient)
    gather_point         reconstruction/external/sampling/tf_sampling.py:42-61   (grad to inp: the scatter-add of GatherPointGrad)
    SoftProjection       classification/soft_projection.py:8-82 and reconstruction/src/soft_projection.py:19-95
    get_simplification_loss   classification/models/samplenet_model.py:176-188, reconstruction/src/samplenet_pointnet_ae.py:165-189
All tensors are BNC float32.
"""
import torch
import torch.nn as nn

from . import ops


def nn_distance(xyz1, xyz2):
    """-> (dist1 (B,N), idx1 (B,N) int32, dist2 (B,M), idx2 (B,M) int32); squared distances; differentiable in xyz1, xyz2."""
    return ops.NNDistanceFunction.apply(xyz1, xyz2)


def approx_match(xyz1, xyz2, exact=None):
    """xyz1 (B, #dataset, 3), xyz2 (B, #query, 3) -> match (B, #query, #dataset).  No gradient.
    exact=True / SNB200_EMD_EXACT_EXP=1: the parity kernel (bit-identical to the CPU oracle); default: the fast kernel."""
    with torch.no_grad():
        return ops.approx_match(xyz1.detach(), xyz2.detach(), exact=exact)


def match_cost(xyz1, xyz2, match):
    """-> cost (B,); differentiable in xyz1 and xyz2."""
    return ops.MatchCostFunction.apply(xyz1, xyz2, match)


def knn_point(k, xyz1, xyz2):
    """xyz1 (B, ndataset, 3) dataset, xyz2 (B, npoint, 3) queries -> val (B, npoint, k) squared distances ascending,
    idx (B, npoint, k) int32.  Ties are ordered by index."""
    o = ops.knn_soft_project_forward(xyz1, xyz2, k, "bnc", want=("idx", "val"))
    return o["val"], o["idx"]


def group_point(points, idx):
    """points (B, ndataset, C), idx (B, npoint, nsample) -> (B, npoint, nsample, C); differentiable in points."""
    return ops.GroupPointFunction.apply(points, idx.to(torch.int32), "bnc")


def farthest_point_sample(npoint, inp):
    """npoint: int, inp (B, N, 3) -> idx (B, npoint) int32: the indices of tf_sampling's FarthestPointSample kernel.  No gradient."""
    with torch.no_grad():
        return ops.farthest_point_sample(inp.detach() if isinstance(inp, torch.Tensor) else inp, npoint, "bnc")


def gather_point(inp, idx):
    """inp (B, N, 3), idx (B, npoint) -> (B, npoint, 3); differentiable in inp."""
    if not isinstance(inp, torch.Tensor) or inp.dim() != 3 or inp.shape[2] != 3:
        raise ValueError("gather_point expects (batch_size, num_points, 3) inp, got %s" % (getattr(inp, "shape", type(inp).__name__),))
    return ops.gather_point(inp, idx, "bnc")


class SoftProjection(nn.Module):
    """TF-flavoured SoftProjection: __call__(point_cloud, query_cloud, hard=False) -> (projected (B,M,3),
    weights (B,M,k,1), dist (B,M,k,1)); `.sigma` is exposed for the projection loss.

    sigma_mode: "cls" -> sigma = T**2 (classification/soft_projection.py:41);
                "rec" -> sigma = max(T, min_sigma)**2 (reconstruction/src/soft_projection.py:51-54, min_sigma = 1e-2)."""

    def __init__(self, group_size, initial_temperature=1.0, is_temperature_trainable=True, sigma_mode="cls", min_sigma=1e-2):
        super().__init__()
        if sigma_mode not in ("cls", "rec"):
            raise ValueError("sigma_mode must be 'cls' or 'rec'")
        self._group_size = group_size
        self._temperature = nn.Parameter(torch.tensor(initial_temperature, dtype=torch.float32),
                                         requires_grad=is_temperature_trainable)
        self._sigma_mode = sigma_mode
        self._min_sigma = float(min_sigma)

    @property
    def sigma(self):
        if self._sigma_mode == "cls":
            return self._temperature ** 2
        return torch.clamp(self._temperature, min=self._min_sigma) ** 2

    def forward(self, point_cloud, query_cloud, hard=False):
        return self.project(point_cloud, query_cloud, hard)

    def project(self, point_cloud, query_cloud, hard=False):
        mode = 2 if self._sigma_mode == "cls" else 3
        proj, _, w, d, _ = ops.SoftProjectFunction.apply(point_cloud, query_cloud, self._temperature, None, self._group_size, "bnc",
                                                         bool(hard), True, False, mode, self._min_sigma)
        return proj, w.unsqueeze(-1), d.unsqueeze(-1)


def get_simplification_loss(ref_pc, samp_pc, pc_size, gamma=1, delta=0):
    """classification/models/samplenet_model.py:176-188."""
    return ops.SimplificationLossFunction.apply(samp_pc, ref_pc, gamma + delta * pc_size)
