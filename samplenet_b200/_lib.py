"""ctypes loader for libsamplenet_b200.so (the C-ABI CUDA library, include/samplenet_b200.h).

There is NO fallback: if the shared library is missing or a call fails, an exception is raised.  The product path never
touches oracle/ or any CPU implementation.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libsamplenet_b200.so")

BNC, BCN = 0, 1
DIST_FMA, DIST_UNFUSED = 0, 1
GEN_EXACT_FP32 = 1
GEN_PROFILE_SKIP_HEAD = 2
GEN_PROFILE_SKIP_CONV = 4
GEN_PER_LAYER_KERNELS = 8
GEN_SEPARATE_HEAD = 16
GEN_WORKSPACE_PRIMED = 32
EMD_EXACT = 1
SIGMA_VALUE, SIGMA_FROM_T_REG, SIGMA_FROM_T_CLS, SIGMA_FROM_T_REC = 0, 1, 2, 3

_c_float_p = ctypes.c_void_p  # raw device pointers travel as integers
_vp = ctypes.c_void_p
_int = ctypes.c_int
_size = ctypes.c_size_t
_float = ctypes.c_float


class Layer(ctypes.Structure):
    """Mirror of `snb200_layer`."""

    _fields_ = [
        ("c_in", _int), ("c_out", _int),
        ("weight", _vp), ("bias", _vp), ("bn_weight", _vp), ("bn_bias", _vp),
        ("bn_running_mean", _vp), ("bn_running_var", _vp), ("bn_num_batches_tracked", _vp),
        ("bn_eps", _float), ("bn_momentum", _float), ("relu", _int),
    ]


class LayerGrad(ctypes.Structure):
    """Mirror of `snb200_layer_grad`."""

    _fields_ = [("weight", _vp), ("bias", _vp), ("bn_weight", _vp), ("bn_bias", _vp)]


class GuardCheck(ctypes.Structure):
    """Mirror of `snb200_guard_check`."""

    _fields_ = [("ptr", _vp), ("count", _int), ("dtype", _int)]


class GuardRestore(ctypes.Structure):
    """Mirror of `snb200_guard_restore`."""

    _fields_ = [("live", _vp), ("snapshot", _vp), ("bytes", ctypes.c_longlong)]


_SIGNATURES = {
    # name: (restype, argtypes)
    "snb200_last_error": (ctypes.c_char_p, []),
    "snb200_version": (_int, []),
    "snb200_launch_count": (ctypes.c_ulonglong, []),
    "snb200_nn_distance_forward": (_int, [_int, _int, _vp, _int, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "snb200_nn_distance_backward": (_int, [_int, _int, _vp, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "snb200_chamfer_per_cloud_workspace_bytes": (_size, [_int, _int, _int]),
    "snb200_chamfer_per_cloud": (_int, [_int, _int, _vp, _int, _vp, _int, _vp, _vp, _size, _vp]),
    "snb200_simplification_loss_workspace_bytes": (_size, [_int, _int, _int]),
    "snb200_simplification_loss_forward": (_int, [_int, _int, _vp, _int, _vp, _float, _vp, _vp, _vp, _vp, _vp, _vp, _size, _int, _vp]),
    "snb200_knn_soft_project_forward": (_int, [_int, _int, _int, _int, _int, _vp, _vp, _vp, _int, _float, _int, _vp, _int, _vp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "snb200_soft_project_backward_workspace_bytes": (_size, [_int, _int, _int, _int, _int]),
    "snb200_soft_project_backward": (_int, [_int, _int, _int, _int, _int, _vp, _vp, _vp, _int, _float, _vp, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _size, _vp]),
    "snb200_project_and_loss_workspace_bytes": (_size, [_int, _int, _int]),
    "snb200_project_and_loss_forward": (_int, [_int, _int, _int, _int, _vp, _vp, _vp, _int, _float, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _float, _vp, _vp, _size, _vp, _int, _vp]),
    "snb200_group_point": (_int, [_int, _int, _int, _int, _int, _int, _vp, _vp, _vp, _vp]),
    "snb200_group_point_grad": (_int, [_int, _int, _int, _int, _int, _int, _vp, _vp, _vp, _vp]),
    "snb200_encoder_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer)]),
    "snb200_encoder_forward": (_int, [_int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, _vp, _vp, _size, _vp]),
    "snb200_generator_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer)]),
    "snb200_generator_forward": (_int, [_int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer), _int, _vp, _int, _vp, _int, _vp, _size, _vp]),
    "snb200_generator_backward_supported": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer)]),
    "snb200_generator_train_forward": (_int, [_int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer), _vp, _int, _vp,
                                              ctypes.POINTER(_vp), _int, _vp, _size, _vp]),
    "snb200_generator_backward_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer)]),
    "snb200_generator_backward": (_int, [_int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer), ctypes.POINTER(_vp), _vp, _vp, _int,
                                         ctypes.POINTER(LayerGrad), ctypes.POINTER(LayerGrad), _vp, _size, _vp]),
    "snb200_generator_layers_backward_supported": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer)]),
    "snb200_generator_layers_train_forward": (_int, [_int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer), _vp, _int, _vp,
                                                     ctypes.POINTER(_vp), _int, _vp, _size, _vp]),
    "snb200_generator_layers_backward_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer)]),
    "snb200_generator_layers_backward": (_int, [_int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer), ctypes.POINTER(_vp), _vp, _vp,
                                                _int, ctypes.POINTER(LayerGrad), ctypes.POINTER(LayerGrad), _vp, _size, _vp]),
    "snb200_generator_layers_ex_supported": (_int, [_int, _int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer), _int,
                                                    ctypes.POINTER(_vp)]),
    "snb200_generator_layers_ex_train_forward": (_int, [_int, _int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer), _int,
                                                        _vp, ctypes.POINTER(_vp), _vp, _int, _vp, ctypes.POINTER(_vp), _int, _vp, _size, _vp]),
    "snb200_generator_layers_ex_backward_workspace_bytes": (_size, [_int, _int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer)]),
    "snb200_generator_layers_ex_backward": (_int, [_int, _int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer), _int,
                                                   ctypes.POINTER(_vp), ctypes.POINTER(_vp), _vp, _vp, _int, _vp, _vp, ctypes.POINTER(LayerGrad),
                                                   ctypes.POINTER(LayerGrad), _vp, _size, _vp]),
    "snb200_debug_tc_gemm": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, _vp]),
    "snb200_fc_head_workspace_bytes": (_size, [_int, _int, ctypes.POINTER(Layer)]),
    "snb200_fc_head_forward": (_int, [_int, _vp, _int, ctypes.POINTER(Layer), _int, _vp, _int, _vp, _size, _vp]),
    "snb200_progressive_loss_workspace_bytes": (_size, [_int, _int, _int, _int]),
    "snb200_progressive_loss_forward": (_int, [_int, _int, _int, _vp, _vp, _int, ctypes.POINTER(_int), ctypes.POINTER(_float), _vp, _vp, _vp, _vp, _vp, _vp, _size,
                                               _vp, _int, _vp]),
    "snb200_frozen_encoder_supported": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int]),
    "snb200_frozen_encoder_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int, _int]),
    "snb200_frozen_encoder_backward_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int]),
    "snb200_frozen_encoder_forward": (_int, [_int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp, ctypes.POINTER(_vp), _vp, _size,
                                             _vp]),
    "snb200_frozen_encoder_backward": (_int, [_int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp, ctypes.POINTER(_vp), _vp, _vp,
                                              _vp, _size, _vp]),
    "snb200_frozen_encoder_curve_supported": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int)]),
    "snb200_frozen_encoder_curve_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int)]),
    "snb200_frozen_encoder_curve_forward": (_int, [_int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp, _vp, _size, _vp]),
    "snb200_frozen_mlp_supported": (_int, [_int, _int, ctypes.POINTER(Layer)]),
    "snb200_frozen_mlp_workspace_bytes": (_size, [_int, _int, ctypes.POINTER(Layer), _int]),
    "snb200_frozen_mlp_forward": (_int, [_int, _vp, _int, ctypes.POINTER(Layer), _vp, ctypes.POINTER(_vp), _vp, _size, _vp]),
    "snb200_frozen_mlp_backward_workspace_bytes": (_size, [_int, _int, ctypes.POINTER(Layer)]),
    "snb200_frozen_mlp_backward": (_int, [_int, _int, ctypes.POINTER(Layer), ctypes.POINTER(_vp), _vp, _vp, _vp, _size, _vp]),
    "snb200_frozen_encoder_param_backward_supported": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int]),
    "snb200_frozen_encoder_param_backward_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int]),
    "snb200_frozen_encoder_param_backward": (_int, [_int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp,
                                                    ctypes.POINTER(_vp), _vp, _vp, ctypes.POINTER(LayerGrad), _vp, _size, _vp]),
    "snb200_frozen_mlp_param_backward_supported": (_int, [_int, _int, ctypes.POINTER(Layer)]),
    "snb200_frozen_mlp_param_backward_workspace_bytes": (_size, [_int, _int, ctypes.POINTER(Layer)]),
    "snb200_frozen_mlp_param_backward": (_int, [_int, _int, ctypes.POINTER(Layer), _vp, ctypes.POINTER(_vp), _vp, _vp, ctypes.POINTER(LayerGrad), _vp,
                                                _size, _vp]),
    "snb200_frozen_encoder_ex_supported": (_int, [_int, _int, _int, _int, ctypes.POINTER(Layer), _int, _int]),
    "snb200_frozen_encoder_ex_workspace_bytes": (_size, [_int, _int, _int, _int, ctypes.POINTER(Layer), _int, _int, _int]),
    "snb200_frozen_encoder_ex_backward_workspace_bytes": (_size, [_int, _int, _int, _int, ctypes.POINTER(Layer), _int, _int]),
    "snb200_frozen_encoder_ex_forward": (_int, [_int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp, _int, _vp,
                                                ctypes.POINTER(_vp), _vp, _size, _vp]),
    "snb200_frozen_encoder_ex_backward": (_int, [_int, _int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp,
                                                 ctypes.POINTER(_vp), _int, _vp, _vp, _vp, _vp, _size, _vp]),
    "snb200_frozen_mlp_bn_supported": (_int, [_int, _int, ctypes.POINTER(Layer)]),
    "snb200_frozen_mlp_bn_workspace_bytes": (_size, [_int, _int, ctypes.POINTER(Layer), _int]),
    "snb200_frozen_mlp_bn_forward": (_int, [_int, _vp, _int, ctypes.POINTER(Layer), _vp, ctypes.POINTER(_vp), _vp, _size, _vp]),
    "snb200_frozen_mlp_bn_backward_workspace_bytes": (_size, [_int, _int, ctypes.POINTER(Layer)]),
    "snb200_frozen_mlp_bn_backward": (_int, [_int, _int, ctypes.POINTER(Layer), ctypes.POINTER(_vp), _vp, _vp, _vp, _size, _vp]),
    "snb200_point_transform_supported": (_int, [_int, _int, _int]),
    "snb200_point_transform_workspace_bytes": (_size, [_int, _int, _int]),
    "snb200_point_transform_forward": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp]),
    "snb200_point_transform_backward": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _size, _vp]),
    "snb200_frozen_encoder_seg_supported": (_int, [_int, _int, _int, _int, _int, ctypes.POINTER(Layer), _int]),
    "snb200_frozen_encoder_seg_workspace_bytes": (_size, [_int, _int, _int, _int, _int, ctypes.POINTER(Layer), _int, _int]),
    "snb200_frozen_encoder_seg_backward_workspace_bytes": (_size, [_int, _int, _int, _int, _int, ctypes.POINTER(Layer), _int]),
    "snb200_frozen_encoder_seg_forward": (_int, [_int, _int, _int, _vp, _int, _vp, _int, ctypes.POINTER(Layer), _vp, _vp, _int, _vp,
                                                 ctypes.POINTER(_vp), _vp, _size, _vp]),
    "snb200_frozen_encoder_seg_backward": (_int, [_int, _int, _int, _vp, _int, _vp, _int, ctypes.POINTER(Layer), _vp, _vp, ctypes.POINTER(_vp),
                                                  _int, _vp, _vp, _vp, _vp, _size, _vp]),
    "snb200_frozen_encoder_bstat_supported": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int)]),
    "snb200_frozen_encoder_bstat_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int)]),
    "snb200_frozen_encoder_bstat_backward_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int)]),
    "snb200_frozen_encoder_bstat_forward": (_int, [_int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp, _vp, _vp,
                                                   _size, _vp]),
    "snb200_frozen_encoder_bstat_backward": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp, _vp, _vp,
                                                    _size, _vp, _vp, _vp, _size, _vp]),
    "snb200_frozen_encoder_bstat_param_backward_supported": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int)]),
    "snb200_frozen_encoder_bstat_param_backward_workspace_bytes": (_size, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int)]),
    "snb200_frozen_encoder_bstat_param_backward": (_int, [_int, _int, _vp, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp, _vp,
                                                          _vp, _size, _vp, _vp, ctypes.POINTER(LayerGrad), _vp, _size, _vp]),
    "snb200_frozen_encoder_bstat_running_update": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(_int), _vp, _vp]),
    "snb200_point_transform_seg_supported": (_int, [_int, _int, _int, _int]),
    "snb200_point_transform_seg_workspace_bytes": (_size, [_int, _int, _int, _int]),
    "snb200_point_transform_seg_forward": (_int, [_int, _int, _int, _vp, _int, _int, _int, _int, ctypes.POINTER(_int), _vp, _vp, _vp, _vp]),
    "snb200_point_transform_seg_backward": (_int, [_int, _int, _int, _vp, _int, _int, _int, _int, ctypes.POINTER(_int), _vp, _vp, _vp, _vp, _vp,
                                                   _vp, _size, _vp]),
    "snb200_pose_loss_workspace_bytes": (_size, [_int, _int]),
    "snb200_pose_loss_forward": (_int, [_int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _size, _vp, _vp]),
    "snb200_pose_loss_backward": (_int, [_int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "snb200_pose_eval_supported": (_int, [_int, _int, _int]),
    "snb200_pose_eval": (_int, [_int, _int, _vp, _vp, _vp, _vp, _int, _vp, _vp, _vp, _vp, _vp]),
    "snb200_pose_loss_ex_supported": (_int, [_int, _int, _int]),
    "snb200_pose_loss_ex_workspace_bytes": (_size, [_int, _int, _int]),
    "snb200_pose_loss_ex_forward": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _size, _vp, _vp]),
    "snb200_pose_loss_ex_backward": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "snb200_pose_eval_ex": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, _int, _int, _vp, _vp, _vp, _vp, _vp]),
    "snb200_approxmatch_workspace_bytes": (_size, [_int, _int, _int]),
    "snb200_approxmatch": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, _size, _vp]),
    "snb200_approxmatch_mode": (_int, [_int, _int, _int, _vp, _vp, _vp, _int, _vp, _size, _vp]),
    "snb200_matchcost_workspace_bytes": (_size, [_int]),
    "snb200_matchcost": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, _vp, _size, _vp]),
    "snb200_matchcostgrad": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, _vp, _vp]),
    "snb200_emd_per_cloud_supported": (_int, [_int, _int, _int]),
    "snb200_emd_per_cloud_workspace_bytes": (_size, [_int, _int, _int]),
    "snb200_emd_per_cloud": (_int, [_int, _int, _vp, _int, _vp, _int, _vp, _vp, _size, _vp]),
    "snb200_emd_per_cloud_backward": (_int, [_int, _int, _vp, _int, _vp, _int, _vp, _vp, _vp, _vp, _size, _vp]),
    "snb200_emd_per_cloud_mode_supported": (_int, [_int, _int, _int, _int]),
    "snb200_emd_per_cloud_mode_workspace_bytes": (_size, [_int, _int, _int, _int]),
    "snb200_emd_per_cloud_mode": (_int, [_int, _int, _vp, _int, _vp, _int, _vp, _int, _vp, _size, _vp]),
    "snb200_emd_per_cloud_mode_backward": (_int, [_int, _int, _vp, _int, _vp, _int, _vp, _vp, _vp, _int, _vp, _size, _vp]),
    "snb200_nn_matching": (_int, [_int, _int, _int, _int, _vp, _vp, _int, _vp, _vp, _vp]),
    "snb200_farthest_point_sample": (_int, [_int, _int, _int, _int, _vp, _vp, _vp, _vp]),
    "snb200_rotate_jitter": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, ctypes.c_double, ctypes.c_double, _vp]),
    "snb200_ae_augment": (_int, [_int, _int, _vp, _vp, _vp, _int, ctypes.c_double, ctypes.c_double, _int, _vp]),
    "snb200_registration_pairs": (_int, [_int, _int, _int, _int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "snb200_retrieval_metrics_supported": (_int, [_int, _int, _int, _int, _int]),
    "snb200_retrieval_metrics": (_int, [_int, _int, _int, _vp, _vp, _vp, _vp, _int, _int, _vp, _vp, _vp, _vp]),
    "snb200_nonfinite_guard": (_int, [ctypes.POINTER(GuardCheck), _int, ctypes.POINTER(GuardRestore), _int, _vp, _vp, _vp, _vp]),
    "snb200_debug_farthest_point_sample": (_int, [_int, _int, _int, _int, _vp, _vp, _vp, _int, _vp]),
    "snb200_debug_conv_stack_partition": (_int, [_int, _int] + [ctypes.POINTER(_int)] * 5),
    "snb200_debug_generator_plan": (_int, [_int, _int, _int, ctypes.POINTER(Layer), _int, ctypes.POINTER(Layer), _int] + [ctypes.POINTER(_int)] * 2),
    "snb200_debug_project_and_loss_plan": (_int, [_int, _int, _int] + [ctypes.POINTER(_int)] * 7),
    "snb200_debug_progressive_loss_plan": (_int, [_int, _int, _int] + [ctypes.POINTER(_int)] * 5),
    "snb200_debug_simplification_loss_plan": (_int, [_int, ctypes.POINTER(_int)]),
}

_lib = None


class SampleNetB200Error(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle.  Raises ImportError loudly if the library was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "samplenet_b200: %s not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `python samplenet_b200/csrc/build.py`). There is no CPU fallback." % LIB_PATH
            )
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(h, name)  # AttributeError if the symbol is missing: fail loudly
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def exported_symbols():
    return sorted(_SIGNATURES)


def check(rc, what):
    if rc != 0:
        msg = lib().snb200_last_error().decode("utf-8", "replace")
        if rc == -1:
            raise ValueError("%s: %s" % (what, msg))
        raise SampleNetB200Error("%s failed (rc=%d): %s" % (what, rc, msg))


def launch_count():
    return int(lib().snb200_launch_count())
