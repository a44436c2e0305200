"""ctypes binding of oracle/_ref/libsamplenet_ref_cuda.so: the REFERENCE's own CUDA kernels (compiled unmodified for sm_90 from the
sources of the reference tree by oracle/Makefile), callable on torch CUDA tensors.

TEST / MEASUREMENT INFRASTRUCTURE, NOT PRODUCT.  Used by tests/ (a second, GPU-side oracle: the reference's kernels on identical inputs)
and by bench.py's `gpu_reference` leg (the "reference on the GPU" row).  samplenet_b200/ never imports this.

The reference launchers run on the LEGACY DEFAULT STREAM (`<<<grid, block>>>`), exactly as in the reference; call these functions with
torch's default stream current (torch's default stream is that stream), never inside a CUDA-graph capture.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "_ref", "libsamplenet_ref_cuda.so")
_LIB = None


def available():
    return os.path.exists(_PATH)


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(_PATH)
        for name in dir(_LIB):
            pass
    return _LIB


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _f(t):
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    return t


def _check_stream(t):
    assert torch.cuda.current_stream(t.device) == torch.cuda.default_stream(t.device), "reference kernels run on the legacy default stream"


def chamfer_forward(xyz1, xyz2):
    """registration ChamferDistanceKernelLauncher: (dist1 (b,n), idx1, dist2 (b,m), idx2)."""
    xyz1, xyz2 = _f(xyz1), _f(xyz2); _check_stream(xyz1)
    b, n, _ = xyz1.shape; m = xyz2.shape[1]
    d1 = torch.empty(b, n, device=xyz1.device); d2 = torch.empty(b, m, device=xyz1.device)
    i1 = torch.empty(b, n, device=xyz1.device, dtype=torch.int32); i2 = torch.empty(b, m, device=xyz1.device, dtype=torch.int32)
    _lib().refcu_chamfer_forward(b, n, _p(xyz1), m, _p(xyz2), _p(d1), _p(i1), _p(d2), _p(i2))
    return d1, i1, d2, i2


def chamfer_backward(xyz1, xyz2, g1, i1, g2, i2):
    xyz1, xyz2, g1, g2 = _f(xyz1), _f(xyz2), _f(g1), _f(g2); _check_stream(xyz1)
    b, n, _ = xyz1.shape; m = xyz2.shape[1]
    gx1 = torch.zeros_like(xyz1); gx2 = torch.zeros_like(xyz2)      # (chamfer_distance.py:47-48 allocates zeros)
    _lib().refcu_chamfer_backward(b, n, _p(xyz1), m, _p(xyz2), _p(g1), _p(i1), _p(g2), _p(i2), _p(gx1), _p(gx2))
    return gx1, gx2


def nn_distance(xyz1, xyz2):
    """TF NmDistanceKernelLauncher."""
    xyz1, xyz2 = _f(xyz1), _f(xyz2); _check_stream(xyz1)
    b, n, _ = xyz1.shape; m = xyz2.shape[1]
    d1 = torch.empty(b, n, device=xyz1.device); d2 = torch.empty(b, m, device=xyz1.device)
    i1 = torch.empty(b, n, device=xyz1.device, dtype=torch.int32); i2 = torch.empty(b, m, device=xyz1.device, dtype=torch.int32)
    _lib().refcu_nn_distance(b, n, _p(xyz1), m, _p(xyz2), _p(d1), _p(i1), _p(d2), _p(i2))
    return d1, i1, d2, i2


def approx_match(xyz1, xyz2):
    """approxmatchLauncher: match (b, m, n); temp = (b, (n+m)*2) floats (tf_approxmatch.cpp:168)."""
    xyz1, xyz2 = _f(xyz1), _f(xyz2); _check_stream(xyz1)
    b, n, _ = xyz1.shape; m = xyz2.shape[1]
    match = torch.empty(b, m, n, device=xyz1.device)
    temp = torch.empty(b, (n + m) * 2, device=xyz1.device)
    _lib().refcu_approxmatch(b, n, m, _p(xyz1), _p(xyz2), _p(match), _p(temp))
    return match


def match_cost(xyz1, xyz2, match):
    xyz1, xyz2, match = _f(xyz1), _f(xyz2), _f(match); _check_stream(xyz1)
    b, n, _ = xyz1.shape; m = xyz2.shape[1]
    out = torch.empty(b, device=xyz1.device)
    _lib().refcu_matchcost(b, n, m, _p(xyz1), _p(xyz2), _p(match), _p(out))
    return out


def match_cost_grad(xyz1, xyz2, match):
    xyz1, xyz2, match = _f(xyz1), _f(xyz2), _f(match); _check_stream(xyz1)
    b, n, _ = xyz1.shape; m = xyz2.shape[1]
    g1 = torch.empty_like(xyz1); g2 = torch.empty_like(xyz2)
    _lib().refcu_matchcostgrad(b, n, m, _p(xyz1), _p(xyz2), _p(match), _p(g1), _p(g2))
    return g1, g2


def selection_sort(dist, k):
    """selectionSortLauncher on a (b, m, n) distance matrix: (idx (b,m,n) int32, val (b,m,n)); the first k entries of each row are the
    k smallest, ascending (tf_grouping.py:31-45)."""
    dist = _f(dist); _check_stream(dist)
    b, m, n = dist.shape
    outi = torch.empty(b, m, n, device=dist.device, dtype=torch.int32)
    out = torch.empty(b, m, n, device=dist.device)
    _lib().refcu_selection_sort(b, n, m, int(k), _p(dist), _p(outi), _p(out))
    return outi, out


def knn_point(k, xyz1, xyz2):
    """tf_grouping.knn_point (tf_grouping.py:64-91): TF evaluates the (b, m, n) squared-distance matrix with elementwise ops and a
    reduce_sum over the 3 coordinates, then runs the selection-sort kernel; here the matrix is evaluated by torch in the same order."""
    diff = xyz2[:, :, None, :] - xyz1[:, None, :, :]
    sq = diff * diff
    dist = ((sq[..., 0] + sq[..., 1]) + sq[..., 2]).contiguous()
    outi, out = selection_sort(dist, k)
    return out[:, :, :k].contiguous(), outi[:, :, :k].contiguous()


def group_point(points, idx):
    points = _f(points); _check_stream(points)
    b, n, c = points.shape
    _, m, ns = idx.shape
    out = torch.empty(b, m, ns, c, device=points.device)
    _lib().refcu_group_point(b, n, c, m, ns, _p(points), _p(idx.contiguous()), _p(out))
    return out


def farthest_point_sample(npoint, inp):
    """tf_sampling.farthest_point_sample(npoint, inp (b,n,3)) -> idx (b, npoint) int32 (temp = (32, n) floats, tf_sampling.cpp)."""
    inp = _f(inp); _check_stream(inp)
    b, n, _ = inp.shape
    temp = torch.empty(32, n, device=inp.device)
    out = torch.empty(b, npoint, device=inp.device, dtype=torch.int32)
    _lib().refcu_farthest_point_sampling(b, n, int(npoint), _p(inp), _p(temp), _p(out))
    return out
