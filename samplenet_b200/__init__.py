"""samplenet_b200 -- SampleNet's sampling-and-loss hot path as hand-written sm_90a CUDA behind the reference's Python API.

    from samplenet_b200 import SampleNet, SoftProjection, ChamferDistance, sputils            # registration (torch) names
    from samplenet_b200.tf_ops import nn_distance, approx_match, match_cost, knn_point, ...   # classification / reconstruction names

Importing the package does not need a GPU; calling any op does, and raises if the CUDA library is missing
(no CPU fallback).
"""
from . import _lib, ops, sputils, tf_ops  # noqa: F401
from .graphs import GraphedStep, PipelinedHostStep, GraphedTrainStep  # noqa: F401
from .chamfer_distance import ChamferDistance, ChamferDistanceFunction  # noqa: F401
from .samplenet import SampleNet  # noqa: F401
from .soft_projection import SoftProjection, knn_point  # noqa: F401
from .samplers import FPSSampler, RandomSampler  # noqa: F401
from .rec_sampler import ReconstructionSampleNet  # noqa: F401
from .tf_variant import ClassificationSampleNet  # noqa: F401
from .registration import CudaPCRNet, FrozenPCRNet  # noqa: F401
from .tasknets import CudaPointNetAE, CudaPointNetCls, CudaPointNetClsTransforms, PointNetClsTransforms, FrozenPointNetClsTransforms  # noqa: F401
from . import evaluation  # noqa: F401
from .evaluation import ClassificationEvaluator, ClassifierEvaluator, ProgressiveClassificationEvaluator, ReconstructionEvaluator  # noqa: F401

__all__ = ["CudaPCRNet", "CudaPointNetAE", "CudaPointNetCls", "CudaPointNetClsTransforms", "FrozenPCRNet", "PointNetClsTransforms", "FrozenPointNetClsTransforms", "SampleNet", "SoftProjection", "ChamferDistance", "ChamferDistanceFunction", "knn_point", "sputils", "tf_ops", "ops", "GraphedStep", "PipelinedHostStep", "GraphedTrainStep",
           "FPSSampler", "RandomSampler", "ReconstructionSampleNet", "ClassificationSampleNet",
           "evaluation", "ClassificationEvaluator", "ClassifierEvaluator", "ProgressiveClassificationEvaluator", "ReconstructionEvaluator"]
