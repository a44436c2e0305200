"""ReconstructionSampleNet -- the sampler of the reconstruction trainer (reconstruction/src/samplers.py:13-41,
samplenet_pointnet_ae.py:46-189) as a trainable torch module on this package's kernels.

Network (encoders_decoders.py:24-131 with the sampler's arguments): 1x1 convs 64-128-128-256-128, each followed by BatchNorm (tflearn,
decay 0.9 = torch momentum 0.1, eps 1e-5) and ReLU; a max-pool over the points; FC 256-256 with ReLU and no BatchNorm; a linear FC to 3M
whose output is reshaped to (B, M, 3) as TF does (consecutive triples are points).  Projection: the reconstruction SoftProjection
(sigma = max(T, 1e-2)^2).  In eval mode the generated points are matched to the input and completed by farthest point sampling
(`simple_projection_and_continued_fps`).

The 256-wide conv layers and the FC layers without BatchNorm are outside the persistent conv-stack kernel: training runs the per-layer
path (tensor-core layer kernels that keep every raw conv output, then the backward kernels of csrc/generator_bwd.cu).
"""
import torch

from . import ops, sputils, tf_ops, trainers
from .samplenet import LayerTableGenerator


class ReconstructionSampleNet(LayerTableGenerator):
    def __init__(self, num_out_points, group_size=16, initial_temperature=1.0, is_temperature_trainable=True):
        m = num_out_points
        super().__init__([3, 64, 128, 128, 256, 128], [128, 256, 256, 3 * m], fc_bn=[False] * 3, fc_relu=[True, True, False],
                         bn_eps=1e-5, bn_momentum=0.1)
        self.num_out_points = m
        self.name = "samplenet"
        self.project = tf_ops.SoftProjection(group_size, initial_temperature, is_temperature_trainable, sigma_mode="rec")

    def forward(self, x):
        """x (B, N, 3) -> (simplified (B, M, 3), projected (B, M, 3)) in training, (simplified, matched (B, M, 3)) in eval."""
        x, simp = self._generate_points(x)
        if self.training:
            proj, _, _ = self.project(x, simp)
            return simp, proj
        _, idx, _, _ = ops.nn_distance_forward(simp.detach(), x.detach())
        match, _, _ = sputils.simple_projection_and_continued_fps(x.detach(), simp, idx)
        return simp, match

    def get_simplification_loss(self, ref_pc, samp_pc, pc_size, is_denoising=False):
        """samplenet_pointnet_ae.py:165-189 (weight pc_size / 64 on the input -> sample term); 0 in eval mode."""
        if not self.training:
            return torch.tensor(0).to(ref_pc)
        return trainers.autoencoder_simplification_loss(ref_pc, samp_pc, pc_size, is_denoising)[0]
