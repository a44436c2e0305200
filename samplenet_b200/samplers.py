"""The non-learned baseline samplers of registration/main.py (`--sampler fps` / `--sampler random`), on this package's kernels.

    FPSSampler     registration/src/fps.py             farthest point sampling (csrc/fps.cu) + the selected points from the same launch
    RandomSampler  registration/src/random_sampling.py a random subset per cloud, gathered by the group_point kernel

Same constructor arguments, `.name`, errors, warnings and return value as the reference modules, and the same RNG calls, so seeded
runs draw the same permutations.
"""
import warnings

import torch

from . import ops

_SHAPE_ERROR = "allowed shape are 'bcn' (batch * channels * num_in_points), 'bnc' "


def _check_shapes(who, input_shape, output_shape):
    if input_shape not in ["bcn", "bnc"]:
        raise ValueError(_SHAPE_ERROR)
    if output_shape not in ["bcn", "bnc"]:
        raise ValueError(_SHAPE_ERROR)
    if input_shape != output_shape:
        warnings.warn("%s: input_shape is different to output_shape." % who)


class FPSSampler(torch.nn.Module):
    """Farthest point sampling of `num_out_points` points per cloud; forward(x) -> y in `output_shape`.

    permute=True first shuffles the points of every cloud with one `torch.randperm(N)` on the default CPU generator (fps.py:31-33), so
    the start point -- FPS always starts at index 0 -- is random.

    The indices are those of tf_sampling's FarthestPointSample kernel.  The reference calls pointnet2's furthest_point_sample, whose
    source is not part of the reference tree, so parity with that kernel's ties cannot be pinned; both start at index 0 and take the
    farthest point each round.

    Deviation: for input_shape="bcn" the reference's fps(x) would read the 3 channels as points (its only caller passes "bnc"); here a
    "bcn" cloud is sampled along its point axis (and permute shuffles that axis)."""

    def __init__(self, num_out_points, permute, input_shape="bcn", output_shape="bcn"):
        super().__init__()
        self.num_out_points = num_out_points
        self.permute = permute
        self.name = "fps"
        _check_shapes("FPS", input_shape, output_shape)
        self.input_shape = input_shape
        self.output_shape = output_shape

    def forward(self, x: torch.Tensor):
        if self.permute:
            if self.input_shape == "bnc":
                _, N, _ = x.shape
                x = x[:, torch.randperm(N), :]
            else:
                _, _, N = x.shape
                x = x[:, :, torch.randperm(N)]
        if torch.is_grad_enabled() and x.requires_grad:  # gather_operation is differentiable in x: gather through autograd
            idx = ops.farthest_point_sample(x.detach(), self.num_out_points, self.input_shape)
            y = ops.gather_point(x, idx, self.input_shape)
        else:  # the points come from the sampling launch itself
            _, y = ops.farthest_point_sample(x, self.num_out_points, self.input_shape, return_points=True)
        if self.input_shape != self.output_shape:
            y = y.permute(0, 2, 1).contiguous()
        return y


class RandomSampler(torch.nn.Module):
    """`num_out_points` points per cloud drawn without replacement: per cloud one `torch.randperm(N, dtype=int32, device=x.device)`
    (random_sampling.py:33-39), gathered on the GPU; forward(x) -> y in `output_shape`, differentiable in x like the reference's
    gather_operation."""

    def __init__(self, num_out_points, input_shape="bcn", output_shape="bcn"):
        super().__init__()
        self.num_out_points = num_out_points
        self.name = "random"
        _check_shapes("RandomSampler", input_shape, output_shape)
        self.input_shape = input_shape
        self.output_shape = output_shape

    def forward(self, x: torch.Tensor):
        if self.input_shape == "bnc":
            x = x.permute(0, 2, 1).contiguous()
        B, _, N = x.shape
        idx = torch.zeros(B, self.num_out_points, dtype=torch.int32, device=x.device)
        for i in range(B):
            rand_perm = torch.randperm(N, dtype=torch.int32, device=x.device)
            idx[i] = rand_perm[:self.num_out_points]
        y = ops.gather_point(x, idx, "bcn")
        if self.output_shape == "bnc":
            y = y.permute(0, 2, 1).contiguous()
        return y
