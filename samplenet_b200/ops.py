"""torch-facing wrappers of the C-ABI kernels: argument checks, output allocation, autograd Functions.

Every function launches on torch's CURRENT CUDA stream and never synchronises, so whole steps can be captured into
CUDA graphs.  CPU tensors are rejected: there is no fallback path.
"""
import ctypes
import math
import os
import threading

import torch

from . import _lib
from ._lib import BCN, BNC, DIST_FMA, DIST_UNFUSED, Layer, LayerGrad, check, lib

_LAYOUTS = {"bnc": BNC, "bcn": BCN}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _req(t, name, dtype=torch.float32):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise RuntimeError("samplenet_b200: %s is on %s; the ops are CUDA-only (no CPU fallback)" % (name, t.device))
    if t.dtype != dtype:
        raise TypeError("%s must be %s, got %s" % (name, dtype, t.dtype))
    return t.contiguous()


def _layout(s):
    try:
        return _LAYOUTS[s]
    except KeyError:
        raise ValueError("layout must be 'bnc' or 'bcn', got %r" % (s,))


def _sigma_grad_to_t(gs, t, sigma_mode, sigma_floor):
    """d/dT from d/dsigma for the temperature modes of the kernels (sigma_mode 1: max(T^2, floor); 2: T^2; 3: max(T, floor)^2)."""
    if sigma_mode == 1:
        return gs * torch.where(t * t > sigma_floor, 2.0 * t, torch.zeros_like(t))
    if sigma_mode == 2:
        return gs * 2.0 * t
    if sigma_mode == 3:
        return gs * torch.where(t > sigma_floor, 2.0 * t, torch.zeros_like(t))
    return gs


# ----------------------------------------------------------------------------------------------------- Chamfer
def nn_distance_forward(xyz1, xyz2, unfused=False):
    """dist1 (B,n), idx1 (B,n) int32, dist2 (B,m), idx2 (B,m) int32 for BNC clouds xyz1 (B,n,3), xyz2 (B,m,3)."""
    xyz1, xyz2 = _req(xyz1, "xyz1"), _req(xyz2, "xyz2")
    if xyz1.dim() != 3 or xyz2.dim() != 3 or xyz1.shape[2] != 3 or xyz2.shape[2] != 3:
        raise ValueError("nn_distance expects (batch, points, 3) tensors, got %s and %s" % (tuple(xyz1.shape), tuple(xyz2.shape)))
    if xyz1.shape[0] != xyz2.shape[0]:
        raise ValueError("nn_distance: batch sizes differ (%d vs %d)" % (xyz1.shape[0], xyz2.shape[0]))
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    with torch.cuda.device(xyz1.device):
        dist1 = torch.empty(b, n, device=xyz1.device, dtype=torch.float32)
        dist2 = torch.empty(b, m, device=xyz1.device, dtype=torch.float32)
        idx1 = torch.empty(b, n, device=xyz1.device, dtype=torch.int32)
        idx2 = torch.empty(b, m, device=xyz1.device, dtype=torch.int32)
        check(lib().snb200_nn_distance_forward(b, n, _p(xyz1), m, _p(xyz2), _p(dist1), _p(idx1), _p(dist2), _p(idx2),
                                               DIST_UNFUSED if unfused else DIST_FMA, _stream()), "nn_distance_forward")
    return dist1, idx1, dist2, idx2


def nn_distance_backward(xyz1, xyz2, g1, idx1, g2, idx2):
    xyz1, xyz2, g1, g2 = _req(xyz1, "xyz1"), _req(xyz2, "xyz2"), _req(g1, "grad_dist1"), _req(g2, "grad_dist2")
    idx1, idx2 = _req(idx1, "idx1", torch.int32), _req(idx2, "idx2", torch.int32)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    with torch.cuda.device(xyz1.device):
        gx1 = torch.empty_like(xyz1)
        gx2 = torch.empty_like(xyz2)
        check(lib().snb200_nn_distance_backward(b, n, _p(xyz1), m, _p(xyz2), _p(g1), _p(idx1), _p(g2), _p(idx2), _p(gx1), _p(gx2),
                                                _stream()), "nn_distance_backward")
    return gx1, gx2


class NNDistanceFunction(torch.autograd.Function):
    """Mirrors ChamferDistanceFunction (registration/src/chamfer_distance/chamfer_distance.py:14-61) and the TF op pair
    NnDistance / NnDistanceGrad (classification/structural_losses/tf_nndistance.py:12-47): returns all four outputs;
    the index outputs are non-differentiable."""

    @staticmethod
    def forward(ctx, xyz1, xyz2, unfused=False):
        dist1, idx1, dist2, idx2 = nn_distance_forward(xyz1, xyz2, unfused)
        ctx.save_for_backward(xyz1.contiguous(), xyz2.contiguous(), idx1, idx2)
        ctx.mark_non_differentiable(idx1, idx2)
        return dist1, idx1, dist2, idx2

    @staticmethod
    def backward(ctx, g1, gi1, g2, gi2):
        xyz1, xyz2, idx1, idx2 = ctx.saved_tensors
        if g1 is None:
            g1 = torch.zeros(idx1.shape, device=xyz1.device, dtype=torch.float32)
        if g2 is None:
            g2 = torch.zeros(idx2.shape, device=xyz1.device, dtype=torch.float32)
        gx1, gx2 = nn_distance_backward(xyz1, xyz2, g1, idx1, g2, idx2)
        return gx1, gx2, None


def _no_grad_inputs(what, *tensors):
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
        raise RuntimeError("%s is an evaluation op without a backward: call it under torch.no_grad() or detach its inputs" % what)


def chamfer_per_cloud(xyz1, xyz2):
    """Per-cloud Chamfer means (csrc/chamfer.cu): sums (B, 2) = (mean_i dist1[b, i], mean_j dist2[b, j]) of xyz1 (B, n, 3) against
    xyz2 (B2, m, 3), where B2 divides B and cloud b of xyz1 is compared with cloud b % B2 of xyz2 (B2 == B: cloud with cloud; B2 < B: the
    stacked prefixes' reconstructions against the one input batch, without repeat()).  The distances are nn_distance_forward's; neither
    distances nor indices are written.  Run to run bit-identical.  No gradient."""
    xyz1, xyz2 = _req(xyz1, "xyz1"), _req(xyz2, "xyz2")
    _no_grad_inputs("chamfer_per_cloud", xyz1, xyz2)
    if xyz1.dim() != 3 or xyz2.dim() != 3 or xyz1.shape[2] != 3 or xyz2.shape[2] != 3:
        raise ValueError("chamfer_per_cloud expects (batch, points, 3) tensors, got %s and %s" % (tuple(xyz1.shape), tuple(xyz2.shape)))
    b, n, _ = xyz1.shape
    b2, m, _ = xyz2.shape
    if xyz2.device != xyz1.device:
        raise ValueError("chamfer_per_cloud: xyz1 is on %s and xyz2 on %s" % (xyz1.device, xyz2.device))
    if b2 < 1 or b % b2 != 0 or n < 1 or m < 1:
        raise ValueError("chamfer_per_cloud: xyz2's %d clouds must divide xyz1's %d, and no cloud may be empty" % (b2, b))
    with torch.cuda.device(xyz1.device):
        sums = torch.empty(b, 2, device=xyz1.device)
        if b:
            wsb = int(lib().snb200_chamfer_per_cloud_workspace_bytes(b, n, m))
            ws = torch.empty(max(wsb, 4), device=xyz1.device, dtype=torch.uint8)
            check(lib().snb200_chamfer_per_cloud(b, n, _p(xyz1), m, _p(xyz2), b2, _p(sums), _p(ws), wsb, _stream()), "chamfer_per_cloud")
    return sums


def simplification_loss_forward(samp, ref, weight21, unfused=False):
    """Fused Chamfer + reductions.  Returns (out4, dist1, idx1, dist2, idx2); out4 = [mean c12, mean max c12, mean c21, loss]."""
    samp, ref = _req(samp, "samp_pc"), _req(ref, "ref_pc")
    if samp.dim() != 3 or ref.dim() != 3 or samp.shape[2] != 3 or ref.shape[2] != 3 or samp.shape[0] != ref.shape[0]:
        raise ValueError("simplification loss expects (B,M,3) and (B,N,3) tensors")
    b, n, _ = samp.shape
    m = ref.shape[1]
    dev = samp.device
    with torch.cuda.device(dev):
        dist1 = torch.empty(b, n, device=dev); dist2 = torch.empty(b, m, device=dev)
        idx1 = torch.empty(b, n, device=dev, dtype=torch.int32); idx2 = torch.empty(b, m, device=dev, dtype=torch.int32)
        out4 = torch.empty(4, device=dev)
        check(lib().snb200_simplification_loss_forward(b, n, _p(samp), m, _p(ref), float(weight21), _p(dist1), _p(idx1), _p(dist2), _p(idx2),
                                                       _p(out4), None, 0, DIST_UNFUSED if unfused else DIST_FMA, _stream()),
              "simplification_loss_forward")
    return out4, dist1, idx1, dist2, idx2


class SimplificationLossFunction(torch.autograd.Function):
    """loss = mean(c12) + mean_b(max c12) + w * mean(c21), c12/c21 = Chamfer(samp, ref)
    (registration/src/samplenet.py:171-181).  Backward routes through the deterministic Chamfer backward kernel."""

    @staticmethod
    def forward(ctx, samp, ref, weight21):
        out4, dist1, idx1, dist2, idx2 = simplification_loss_forward(samp, ref, weight21)
        ctx.save_for_backward(samp.contiguous(), ref.contiguous(), dist1, idx1, idx2)
        ctx.w = float(weight21)
        return out4[3].clone()

    @staticmethod
    def backward(ctx, g):
        samp, ref, dist1, idx1, idx2 = ctx.saved_tensors
        b, n = dist1.shape
        m = idx2.shape[1]
        # d loss / d dist1[b,j] = 1/(b n) + [j == argmax_j dist1[b]] / b ;  d loss / d dist2 = w / (b m)
        g1 = torch.full((b, n), 1.0 / (b * n), device=samp.device)
        am = dist1.argmax(dim=1, keepdim=True)
        g1.scatter_add_(1, am, torch.full((b, 1), 1.0 / b, device=samp.device))
        g2 = torch.full((b, m), ctx.w / (b * m), device=samp.device)
        g1 = g1 * g
        g2 = g2 * g
        gs, gr = nn_distance_backward(samp, ref, g1, idx1, g2, idx2)
        return gs, gr, None


# ----------------------------------------------------------------------------------------------------- kNN / projection
def knn_soft_project_forward(points, query, k, layout, sigma=None, hard=False, feats=None, want=("proj",), unfused=False,
                             sigma_mode=0, sigma_floor=0.0):
    """One fused launch.  `want` is a subset of {"proj","prop","idx","val","weights","dist"}; returns a dict of tensors.
    sigma_mode / sigma_floor: how the `sigma` scalar is interpreted (see SNB200_SIGMA_* in the header)."""
    lay = _layout(layout)
    points, query = _req(points, "point_cloud"), _req(query, "query_cloud")
    if points.dim() != 3 or query.dim() != 3 or points.shape[0] != query.shape[0]:
        raise ValueError("soft projection expects 3-D clouds with equal batch sizes")
    cdim = 2 if lay == BNC else 1
    if points.shape[cdim] != 3 or query.shape[cdim] != 3:
        raise ValueError("soft projection: channel dimension must be 3 for layout %r, got %s / %s" % (layout, tuple(points.shape), tuple(query.shape)))
    b = points.shape[0]
    n = points.shape[1] if lay == BNC else points.shape[2]
    m = query.shape[1] if lay == BNC else query.shape[2]
    k = int(k)
    dev = points.device
    f = 0
    if feats is not None:
        feats = _req(feats, "point_features")
        f = feats.shape[2] if lay == BNC else feats.shape[1]
        nf = feats.shape[1] if lay == BNC else feats.shape[2]
        if nf != n or feats.shape[0] != b:
            raise ValueError("point_features must cover the same points as point_cloud")
    if sigma is not None:
        sigma = _req(sigma.reshape(1), "sigma")
    out = {}
    with torch.cuda.device(dev):
        if "proj" in want:
            out["proj"] = torch.empty_like(query)
        if "prop" in want:
            out["prop"] = torch.empty((b, m, f) if lay == BNC else (b, f, m), device=dev)
        if "idx" in want:
            out["idx"] = torch.empty(b, m, k, device=dev, dtype=torch.int32)
        if "val" in want:
            out["val"] = torch.empty(b, m, k, device=dev)
        if "weights" in want:
            out["weights"] = torch.empty(b, m, k, device=dev)
        if "dist" in want:
            out["dist"] = torch.empty(b, m, k, device=dev)
        check(lib().snb200_knn_soft_project_forward(
            b, n, m, k, lay, _p(points), _p(query), _p(sigma), int(sigma_mode), float(sigma_floor), int(bool(hard)), _p(feats), f,
            _p(out.get("proj")), _p(out.get("prop")),
            _p(out.get("idx")), _p(out.get("val")), _p(out.get("weights")), _p(out.get("dist")), DIST_UNFUSED if unfused else DIST_FMA,
            _stream()), "knn_soft_project_forward")
    return out


def soft_project_backward(points, query, sigma, feats, idx, weights, grad_proj, grad_prop, layout, need_points, need_query, need_feats,
                          need_sigma, sigma_mode=0, sigma_floor=0.0):
    lay = _layout(layout)
    b = points.shape[0]
    n = points.shape[1] if lay == BNC else points.shape[2]
    m = query.shape[1] if lay == BNC else query.shape[2]
    k = idx.shape[2]
    f = 0 if feats is None else (feats.shape[2] if lay == BNC else feats.shape[1])
    dev = points.device
    with torch.cuda.device(dev):
        gp = torch.empty_like(points) if need_points else None
        gq = torch.empty_like(query) if need_query else None
        gf = torch.empty_like(feats) if (need_feats and feats is not None) else None
        gs = torch.empty(1, device=dev) if need_sigma else None
        wsb = lib().snb200_soft_project_backward_workspace_bytes(b, n, m, k, f)
        ws = torch.empty(max(int(wsb), 4), device=dev, dtype=torch.uint8)
        gproj = None if grad_proj is None else _req(grad_proj, "grad_proj")
        gprop = None if grad_prop is None else _req(grad_prop, "grad_prop")
        check(lib().snb200_soft_project_backward(
            b, n, m, k, lay, _p(points), _p(query), _p(sigma), int(sigma_mode), float(sigma_floor), _p(feats), f, _p(idx), _p(weights),
            _p(gproj), _p(gprop), _p(gp), _p(gq),
            _p(gf), _p(gs), _p(ws), int(wsb), _stream()), "soft_project_backward")
    return gp, gq, gf, gs


class SoftProjectFunction(torch.autograd.Function):
    """(points, query, t[, feats]) -> (proj, prop, weights, dist, idx); differentiable in points, query, t, feats.

    `t` is either sigma itself (sigma_mode 0) or the temperature parameter, in which case the kernel evaluates the
    sub-project's clamp (sigma_mode 1: max(T^2, floor) registration; 2: T^2 classification; 3: max(T, floor)^2 reconstruction)
    and the chain rule d sigma / d T is applied here in backward."""

    @staticmethod
    def forward(ctx, points, query, t, feats, k, layout, hard, want_proj, want_prop, sigma_mode=0, sigma_floor=0.0):
        want = ["idx", "weights", "dist"]
        if want_proj:
            want.append("proj")
        if want_prop:
            want.append("prop")
        points = points.contiguous(); query = query.contiguous()
        sig = t.detach().reshape(1).contiguous()
        o = knn_soft_project_forward(points, query, k, layout, sig, hard, feats, want, sigma_mode=sigma_mode, sigma_floor=sigma_floor)
        ctx.layout = layout
        ctx.hard = hard
        ctx.has_feats = feats is not None
        ctx.sigma_mode, ctx.sigma_floor = int(sigma_mode), float(sigma_floor)
        ctx.save_for_backward(points, query, sig, feats.contiguous() if feats is not None else None, o["idx"], o["weights"])
        proj = o.get("proj"); prop = o.get("prop")
        # weights / dist are returned for inspection (the TF SoftProjection returns them too); only the projection and the propagated features
        # carry gradients, as in every reference caller -- marked so autograd does not pretend otherwise
        ctx.mark_non_differentiable(o["idx"], o["weights"], o["dist"])
        ctx.sigma_shape = t.shape
        dev = points.device
        if proj is None:
            proj = torch.empty(0, device=dev)
        if prop is None:
            prop = torch.empty(0, device=dev)
        return proj, prop, o["weights"], o["dist"], o["idx"]

    @staticmethod
    def backward(ctx, g_proj, g_prop, g_w, g_d, g_i):
        points, query, sig, feats, idx, weights = ctx.saved_tensors
        if ctx.hard:
            raise NotImplementedError("hard projection is not differentiable (registration/src/soft_projection.py:144-145)")
        if g_proj is not None and g_proj.numel() == 0:
            g_proj = None
        if g_prop is not None and g_prop.numel() == 0:
            g_prop = None
        if g_proj is None and g_prop is None:
            return (None,) * 11
        need = ctx.needs_input_grad
        gp, gq, gf, gs = soft_project_backward(points, query, sig, feats, idx, weights, g_proj, g_prop, ctx.layout, need[0], need[1],
                                               need[3] and ctx.has_feats, need[2], ctx.sigma_mode, ctx.sigma_floor)
        if gs is not None:
            gs = _sigma_grad_to_t(gs, sig, ctx.sigma_mode, ctx.sigma_floor).reshape(ctx.sigma_shape)
        return gp, gq, gs, gf, None, None, None, None, None, None, None


_TICKETS = {}


def _ticket(dev):
    """One zero-initialised device counter per (GPU, stream) for the last-CTA reductions (fused tail, progressive loss); the kernels leave
    it zero.  Launches that share a word are stream-ordered by construction; concurrent launches on different streams get different
    words.  (A kernel that traps leaves the context unusable anyway.)  The C ABI takes the word as an argument.
    With a PrimedWorkspaces active the word is that object's own instead: a captured launch keeps the word of its capture but replays on
    the caller's stream, so a graph must not share the word of a stream (or of another graph)."""
    pw = getattr(_ACTIVE_PW, "pw", None)
    if pw is not None:
        return pw.ticket(dev)
    key = (dev.type, dev.index, torch.cuda.current_stream(dev).cuda_stream)   # launches on different streams never share a word
    t = _TICKETS.get(key)
    if t is None:
        t = torch.zeros(1, device=dev, dtype=torch.int32)
        _TICKETS[key] = t
    return t


_CONSTANTS = {}


def _device_constant(values, dtype, dev):
    """A read-only device copy of a short host list, made once per (values, dtype, device): the per-call host-to-device copy it replaces
    synchronises the host and cannot be captured in a CUDA graph.  Callers never write into it."""
    key = (tuple(values), dtype, dev.type, dev.index)
    t = _CONSTANTS.get(key)
    if t is None:
        t = torch.tensor(list(values), dtype=dtype, device=dev)
        _CONSTANTS[key] = t
    return t


def project_and_loss_forward(ref, samp, k, t, sigma_mode, sigma_floor, weight21, unfused=False):
    """One launch: proj, (idx, weights, dist) for the projection backward, Chamfer dist/idx both ways, out4 loss terms."""
    ref, samp = _req(ref, "ref_pc"), _req(samp, "samp_pc")
    b, n, _ = ref.shape
    m = samp.shape[1]
    dev = ref.device
    tt = _req(t.detach().reshape(1), "temperature")
    with torch.cuda.device(dev):
        proj = torch.empty_like(samp)
        idx = torch.empty(b, m, k, device=dev, dtype=torch.int32)
        w = torch.empty(b, m, k, device=dev); d = torch.empty(b, m, k, device=dev)
        dist1 = torch.empty(b, m, device=dev); idx1 = torch.empty(b, m, device=dev, dtype=torch.int32)
        dist2 = torch.empty(b, n, device=dev); idx2 = torch.empty(b, n, device=dev, dtype=torch.int32)
        out4 = torch.empty(4, device=dev)
        wsb = int(lib().snb200_project_and_loss_workspace_bytes(b, m, n))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_project_and_loss_forward(b, n, m, int(k), _p(ref), _p(samp), _p(tt), int(sigma_mode), float(sigma_floor), _p(proj), _p(idx),
                                                    _p(w), _p(d), _p(dist1), _p(idx1), _p(dist2), _p(idx2), float(weight21), _p(out4), _p(ws), wsb,
                                                    _p(_ticket(dev)), DIST_UNFUSED if unfused else DIST_FMA, _stream()), "project_and_loss_forward")
    return proj, idx, w, d, dist1, idx1, dist2, idx2, out4


class ProjectAndLossFunction(torch.autograd.Function):
    """(ref, samp, temperature) -> (proj, loss_w1, terms): the projection of `samp` onto `ref` together with the simplification
    loss of (samp, ref) evaluated for weight 1 (`loss_w1`) and its three terms (`terms` = [mean c12, mean max c12, mean c21]).
    Backward = soft-projection backward + Chamfer backward (both deterministic kernels)."""

    @staticmethod
    def forward(ctx, ref, samp, t, k, sigma_mode, sigma_floor):
        ref = ref.contiguous(); samp = samp.contiguous()
        proj, idx, w, d, dist1, idx1, dist2, idx2, out4 = project_and_loss_forward(ref, samp, k, t, sigma_mode, sigma_floor, 1.0)
        ctx.save_for_backward(ref, samp, t.detach().reshape(1).contiguous(), idx, w, dist1, idx1, idx2)
        ctx.sigma_mode, ctx.sigma_floor, ctx.t_shape = int(sigma_mode), float(sigma_floor), t.shape
        return proj, out4[3], out4[:3]

    @staticmethod
    def backward(ctx, g_proj, g_unit, g_terms):
        ref, samp, tt, idx, w, dist1, idx1, idx2 = ctx.saved_tensors
        need = ctx.needs_input_grad
        b, m = dist1.shape
        n = idx2.shape[1]
        dev = ref.device
        g_ref = g_samp = g_t = None
        if g_proj is not None:
            gp, gq, _, gs = soft_project_backward(ref, samp, tt, None, idx, w, g_proj.contiguous(), None, "bnc", need[0], need[1], False, need[2],
                                                  ctx.sigma_mode, ctx.sigma_floor)
            g_ref, g_samp = gp, gq
            if gs is not None:
                g_t = _sigma_grad_to_t(gs, tt, ctx.sigma_mode, ctx.sigma_floor).reshape(ctx.t_shape)
        if g_unit is not None or g_terms is not None:
            zero = torch.zeros((), device=dev)
            gu = g_unit if g_unit is not None else zero
            gt = g_terms if g_terms is not None else torch.zeros(3, device=dev)
            a0, a1, a2 = gu + gt[0], gu + gt[1], gu + gt[2]
            g1 = (a0 / (b * m)).expand(b, m).clone()
            g1.scatter_add_(1, dist1.argmax(dim=1, keepdim=True), (a1 / b).expand(b, 1).contiguous())
            g2 = (a2 / (b * n)).expand(b, n).contiguous()
            gs_c, gr_c = nn_distance_backward(samp, ref, g1, idx1, g2, idx2)
            g_samp = gs_c if g_samp is None else g_samp + gs_c
            if need[0]:
                g_ref = gr_c if g_ref is None else g_ref + gr_c
        return (g_ref if need[0] else None), g_samp, g_t, None, None, None


# ----------------------------------------------------------------------------------------------------- progressive loss
def progressive_loss_forward(ref, samp, sizes, weights, unfused=False):
    """One launch: dist1/idx1 (B,M), dist2/idx2 (B,P,N) for the P prefixes `sizes` of the ordered samples, terms (3P+1,)."""
    ref, samp = _req(ref, "ref_pc"), _req(samp, "samp_pc")
    b, n, _ = ref.shape
    m = samp.shape[1]
    npf = len(sizes)
    dev = ref.device
    csz = (ctypes.c_int * npf)(*[int(v) for v in sizes])
    cw = (ctypes.c_float * npf)(*[float(v) for v in weights])
    with torch.cuda.device(dev):
        dist1 = torch.empty(b, m, device=dev); idx1 = torch.empty(b, m, device=dev, dtype=torch.int32)
        dist2 = torch.empty(b, npf, n, device=dev); idx2 = torch.empty(b, npf, n, device=dev, dtype=torch.int32)
        terms = torch.empty(3 * npf + 1, device=dev)
        wsb = int(lib().snb200_progressive_loss_workspace_bytes(b, n, m, npf))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_progressive_loss_forward(b, n, m, _p(ref), _p(samp), npf, csz, cw, _p(dist1), _p(idx1), _p(dist2), _p(idx2), _p(terms), _p(ws), wsb,
                                                    _p(_ticket(dev)), DIST_UNFUSED if unfused else DIST_FMA, _stream()), "progressive_loss_forward")
    return dist1, idx1, dist2, idx2, terms


class ProgressiveLossFunction(torch.autograd.Function):
    """sum over prefixes s of [mean(c12[:s]) + mean_b(max c12[:s]) + w_s mean(c21^(s))]  (train_samplenet_progressive.py:196-220) in one
    forward launch; backward = one deterministic Chamfer-backward launch over the concatenated prefix index sets."""

    @staticmethod
    def forward(ctx, samp, ref, sizes, weights):
        samp = samp.contiguous(); ref = ref.contiguous()
        dist1, idx1, dist2, idx2, terms = progressive_loss_forward(ref, samp, sizes, weights)
        ctx.save_for_backward(samp, ref, dist1, idx1, idx2)
        ctx.sizes, ctx.weights = [int(v) for v in sizes], [float(v) for v in weights]
        return terms[3 * len(sizes)].clone(), terms[:3 * len(sizes)].view(len(sizes), 3)

    @staticmethod
    def backward(ctx, g, g_terms):
        samp, ref, dist1, idx1, idx2 = ctx.saved_tensors
        b, m = dist1.shape
        npf, n = idx2.shape[1], idx2.shape[2]
        dev = samp.device
        sizes = _device_constant(ctx.sizes, torch.int64, dev)
        w = _device_constant(ctx.weights, torch.float32, dev)
        gt = g_terms if g_terms is not None else torch.zeros(npf, 3, device=dev)
        gg = g if g is not None else torch.zeros((), device=dev)
        a0 = gg + gt[:, 0]; a1 = gg + gt[:, 1]; a2 = gg * w + gt[:, 2]           # d total / d term, per prefix
        # mean(c12[:s]) : every j < s gets 1/(b s);  as a function of j: sum over prefixes with s > j
        j = torch.arange(m, device=dev)
        cover = (sizes[None, :] > j[:, None]).to(dist1.dtype)                     # (m, P)
        g1 = (cover * (a0 / (b * sizes.to(dist1.dtype)))[None, :]).sum(1)[None, :].expand(b, m).clone()
        # mean_b max(c12[:s]) : the FIRST j < s attaining the running maximum, as argmax routes the max term in the other two loss
        # paths (torch.cummax's indices would give the last one on ties)
        run_max = torch.cummax(dist1, dim=1).values[:, sizes - 1]                 # (b, P)
        am = (dist1[:, None, :] == run_max[:, :, None]).to(torch.int32).argmax(dim=2)   # (b, P); the first hit is always < s
        g1.scatter_add_(1, am, (a1 / b)[None, :].expand(b, npf).contiguous())
        g2 = (a2 / (b * n))[None, :, None].expand(b, npf, n).reshape(b, npf * n).contiguous()
        ref_rep = ref[:, None].expand(b, npf, n, 3).reshape(b, npf * n, 3).contiguous()
        gs, gr = nn_distance_backward(samp, ref_rep, g1.contiguous(), idx1, g2, idx2.reshape(b, npf * n).contiguous())
        return gs, gr.view(b, npf, n, 3).sum(1), None, None


def group_point(points, idx, layout="bnc"):
    lay = _layout(layout)
    points, idx = _req(points, "points"), _req(idx, "idx", torch.int32)
    b = points.shape[0]
    if lay == BNC:
        n, c = points.shape[1], points.shape[2]
    else:
        c, n = points.shape[1], points.shape[2]
    _, m, ns = idx.shape
    with torch.cuda.device(points.device):
        out = torch.empty((b, m, ns, c) if lay == BNC else (b, c, m, ns), device=points.device)
        check(lib().snb200_group_point(b, n, c, m, ns, lay, _p(points), _p(idx), _p(out), _stream()), "group_point")
    return out


def group_point_grad(points_shape, idx, grad_out, layout="bnc"):
    lay = _layout(layout)
    idx, grad_out = _req(idx, "idx", torch.int32), _req(grad_out, "grad_out")
    b = points_shape[0]
    if lay == BNC:
        n, c = points_shape[1], points_shape[2]
    else:
        c, n = points_shape[1], points_shape[2]
    _, m, ns = idx.shape
    with torch.cuda.device(idx.device):
        gp = torch.empty(tuple(points_shape), device=idx.device)
        check(lib().snb200_group_point_grad(b, n, c, m, ns, lay, _p(grad_out), _p(idx), _p(gp), _stream()), "group_point_grad")
    return gp


class GroupPointFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, idx, layout):
        ctx.save_for_backward(idx)
        ctx.shape = tuple(points.shape)
        ctx.layout = layout
        return group_point(points, idx, layout)

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        return group_point_grad(ctx.shape, idx, g, ctx.layout), None, None


# ----------------------------------------------------------------------------------------------------- generator
def make_layers(specs):
    """specs: list of dicts(weight, bias, bn=(weight,bias,running_mean,running_var,eps,momentum[,num_batches_tracked]) or None, relu=bool)."""
    arr = (Layer * len(specs))()
    keep = []
    for i, s in enumerate(specs):
        w = _req(s["weight"].reshape(s["weight"].shape[0], -1), "weight")
        bias = _req(s["bias"], "bias") if s.get("bias") is not None else torch.zeros(w.shape[0], device=w.device)
        keep += [w, bias]
        arr[i].c_out, arr[i].c_in = w.shape[0], w.shape[1]
        arr[i].weight, arr[i].bias = w.data_ptr(), bias.data_ptr()
        bn = s.get("bn")
        if bn is not None:
            gw, gb, rm, rv, eps, mom = bn[:6]
            nbt = bn[6] if len(bn) > 6 else None
            gw, gb = _req(gw, "bn.weight"), _req(gb, "bn.bias")
            keep += [gw, gb]
            arr[i].bn_weight, arr[i].bn_bias = gw.data_ptr(), gb.data_ptr()
            arr[i].bn_running_mean = None if rm is None else rm.data_ptr()
            arr[i].bn_running_var = None if rv is None else rv.data_ptr()
            arr[i].bn_eps, arr[i].bn_momentum = float(eps), float(0.1 if mom is None else mom)
            if nbt is not None:
                if nbt.dtype != torch.int64 or not nbt.is_cuda:
                    raise TypeError("num_batches_tracked must be an int64 CUDA tensor")
                arr[i].bn_num_batches_tracked = nbt.data_ptr()
            else:
                arr[i].bn_num_batches_tracked = None
        else:
            arr[i].bn_weight = arr[i].bn_bias = arr[i].bn_running_mean = arr[i].bn_running_var = arr[i].bn_num_batches_tracked = None
            arr[i].bn_eps, arr[i].bn_momentum = 0.0, 0.0
        arr[i].relu = int(bool(s.get("relu", False)))
    return arr, keep


class PrimedWorkspaces:
    """Generator workspaces that persist across calls (one per size), zero-initialised once.  With one of these active
    (`with primed_workspaces(pw): ...`) `generator_forward` passes SNB200_GEN_WORKSPACE_PRIMED: the persistent kernel cleans its own
    scratch, so no memset is issued in front of it.  The owner promises the calls that share a buffer are stream-ordered
    (GraphedStep / GraphedTrainStep own one each); plain calls outside such a context allocate and memset per call as before.  While one
    is active, the fused tail and the progressive loss take its own ticket word (`ticket`) instead of their stream's."""

    def __init__(self):
        self.bufs = {}
        self.uses = {}     # training forwards per size since primed_workspaces(self) was entered (see saved)

    def get(self, dev, nbytes):
        key = (dev.index, int(nbytes))
        t = self.bufs.get(key)
        if t is None:
            t = torch.zeros(max(int(nbytes), 256), device=dev, dtype=torch.uint8)
            self.bufs[key] = t
        return t

    def saved(self, dev, nbytes, shapes):
        """(workspace, activation buffers) of a training forward, which its backward reads: the k-th training forward of a size since
        primed_workspaces(self) was entered gets the k-th pair.  So a step that runs the generator twice at one size before its backward
        (the registration sampler on the template and on the source) keeps both forwards' buffers, and every execution of the step maps
        its calls to the same buffers.  The first pair is get(dev, nbytes) and get_named(dev, "zsave", shapes)."""
        key = (dev.index, int(nbytes), tuple(tuple(s) for s in shapes))
        k = self.uses.get(key, 0)
        self.uses[key] = k + 1
        if k == 0:
            return self.get(dev, nbytes), self.get_named(dev, "zsave", shapes)
        wkey = (dev.index, int(nbytes), k)
        ws = self.bufs.get(wkey)
        if ws is None:
            ws = torch.zeros(max(int(nbytes), 256), device=dev, dtype=torch.uint8)
            self.bufs[wkey] = ws
        return ws, self.get_named(dev, ("zsave", k), shapes)

    def get_named(self, dev, name, shapes):
        """Persistent float buffers (e.g. the activations kept for the backward pass), one list per (device, name, shapes)."""
        key = (dev.index, name, tuple(tuple(s) for s in shapes))
        t = self.bufs.get(key)
        if t is None:
            t = [torch.empty(*s, device=dev) for s in shapes]
            self.bufs[key] = t
        return t

    def ticket(self, dev):
        """This object's zero-initialised ticket word for the last-CTA reductions (see _ticket), one per device."""
        key = (dev.index, "ticket")
        t = self.bufs.get(key)
        if t is None:
            t = torch.zeros(1, device=dev, dtype=torch.int32)
            self.bufs[key] = t
        return t


_ACTIVE_PW = threading.local()


class primed_workspaces:
    def __init__(self, pw):
        self.pw = pw

    def __enter__(self):
        self.prev = getattr(_ACTIVE_PW, "pw", None)
        _ACTIVE_PW.pw = self.pw
        self.pw.uses = {}
        return self.pw

    def __exit__(self, *exc):
        _ACTIVE_PW.pw = self.prev
        return False


def _generator_args(x, layout, conv_specs, fc_specs):
    """Prologue of the generator wrappers: layout code, batch, points per cloud and the two C layer tables, with the tensors the tables
    point into (keep them alive until the call has been issued)."""
    lay = _layout(layout)
    if x.dim() != 3 or x.shape[2 if lay == BNC else 1] != 3:
        raise RuntimeError("shape of x must be of [Batch x 3 x NumInPoints]")
    b = x.shape[0]
    n = x.shape[1] if lay == BNC else x.shape[2]
    conv, keep_conv = make_layers(conv_specs)
    fc, keep_fc = make_layers(fc_specs)
    return lay, b, n, conv, fc, keep_conv + keep_fc


def _workspace(dev, nbytes, primed=False):
    """(buffer, flag): with `primed` and a PrimedWorkspaces active, its persistent buffer and SNB200_GEN_WORKSPACE_PRIMED; otherwise a
    fresh buffer and 0."""
    pw = getattr(_ACTIVE_PW, "pw", None) if primed else None
    if pw is not None:
        return pw.get(dev, nbytes), _lib.GEN_WORKSPACE_PRIMED
    return torch.empty(max(nbytes, 4), device=dev, dtype=torch.uint8), 0


def generator_forward(x, layout, conv_specs, fc_specs, training, out_transpose_inner=0, exact_fp32=False, _profile_flags=0, per_layer_kernels=False, separate_head=False):
    """x (B,N,3)/(B,3,N) -> (out (B, c_out_last), feat (B, c_conv_last)): conv stack + max-pool + FC head in ONE C-ABI call.
    Default: conv layers on the tensor cores (wgmma, 3xTF32) + cluster-fused FC head; exact_fp32=True: CUDA-core conv stack."""
    lay, b, n, conv, fc, keep = _generator_args(x, layout, conv_specs, fc_specs)
    x = _req(x, "x")
    dev = x.device
    flags = ((_lib.GEN_EXACT_FP32 if exact_fp32 else 0) | (_lib.GEN_PER_LAYER_KERNELS if per_layer_kernels else 0)
             | (_lib.GEN_SEPARATE_HEAD if separate_head else 0) | int(_profile_flags))
    with torch.cuda.device(dev):
        wsb = int(lib().snb200_generator_workspace_bytes(b, n, len(conv_specs), conv, len(fc_specs), fc))
        ws, primed = _workspace(dev, wsb, primed=not _profile_flags)
        feat = torch.empty(b, conv[len(conv_specs) - 1].c_out, device=dev)
        out = torch.empty(b, fc[len(fc_specs) - 1].c_out, device=dev)
        check(lib().snb200_generator_forward(b, n, lay, _p(x), len(conv_specs), conv, len(fc_specs), fc, int(bool(training)), _p(out),
                                             int(out_transpose_inner), _p(feat), flags | primed, _p(ws), wsb, _stream()), "generator_forward")
    del keep
    return out, feat


def generator_backward_supported(x, layout, conv_specs, fc_specs):
    """True when the CUDA backward (csrc/generator_bwd.cu) covers this shape: the persistent conv-stack envelope, 2 <= B <= 64,
    BatchNorm + ReLU on every conv layer."""
    _, b, n, conv, fc, keep = _generator_args(x, layout, conv_specs, fc_specs)
    return bool(lib().snb200_generator_backward_supported(b, n, len(conv_specs), conv, len(fc_specs), fc))


def generator_layers_backward_supported(x, layout, conv_specs, fc_specs):
    """True when the per-layer training path covers this shape (snb200_generator_layers_backward_supported): conv widths up to 256 in the
    pairs the backward kernels take, or a last layer 128 -> C with C a multiple of 64 up to 1024, BatchNorm + ReLU on every conv layer, FC
    layers with any BatchNorm / ReLU combination but no ReLU on the last one, 2 <= B <= 64 (fewer where fc1's input and weight rows fill
    the backward kernel's shared memory: B <= 41 at C = 1024), any number of points."""
    _, b, n, conv, fc, keep = _generator_args(x, layout, conv_specs, fc_specs)
    return bool(lib().snb200_generator_layers_backward_supported(b, n, len(conv_specs), conv, len(fc_specs), fc))


def _train_forward(entry, x, layout, conv_specs, fc_specs, out_transpose_inner):
    lay, b, n, conv, fc, keep = _generator_args(x, layout, conv_specs, fc_specs)
    x = _req(x, "x")
    dev = x.device
    with torch.cuda.device(dev):
        wsb = int(lib().snb200_generator_workspace_bytes(b, n, len(conv_specs), conv, len(fc_specs), fc))
        shapes = [(b * n, conv[l].c_out) for l in range(len(conv_specs))]
        pw = getattr(_ACTIVE_PW, "pw", None)
        if pw is not None:
            (ws, zs), primed = pw.saved(dev, wsb, shapes), _lib.GEN_WORKSPACE_PRIMED
        else:
            ws, primed = _workspace(dev, wsb)
            zs = [torch.empty(*s, device=dev) for s in shapes]
        zp = (ctypes.c_void_p * len(zs))(*[z.data_ptr() for z in zs])
        feat = torch.empty(b, conv[len(conv_specs) - 1].c_out, device=dev)
        out = torch.empty(b, fc[len(fc_specs) - 1].c_out, device=dev)
        check(getattr(lib(), "snb200_" + entry)(b, n, lay, _p(x), len(conv_specs), conv, len(fc_specs), fc, _p(out), int(out_transpose_inner), _p(feat),
                                                zp, primed, _p(ws), wsb, _stream()), entry)
    del keep
    return out, feat, (zs, ws)


def generator_train_forward(x, layout, conv_specs, fc_specs, out_transpose_inner=0):
    """Training-mode forward that keeps what the CUDA backward needs.  Returns (out, feat, saved) with saved = (zsave list, workspace)."""
    return _train_forward("generator_train_forward", x, layout, conv_specs, fc_specs, out_transpose_inner)


def generator_layers_train_forward(x, layout, conv_specs, fc_specs, out_transpose_inner=0):
    """The per-layer path's training forward (tensor-core layer kernels + cluster FC head; the same results as generator_forward(training,
    per_layer_kernels=True)) that keeps what generator_layers_backward needs.  Returns (out, feat, saved) like generator_train_forward."""
    return _train_forward("generator_layers_train_forward", x, layout, conv_specs, fc_specs, out_transpose_inner)


def _backward(entry, x, layout, conv_specs, fc_specs, saved, grad_out, out_transpose_inner, dest):
    lay, b, n, conv, fc, keep = _generator_args(x, layout, conv_specs, fc_specs)
    x = _req(x, "x"); grad_out = _req(grad_out, "grad_out")
    dev = x.device
    zs, fwd_ws = saved
    grads = []

    def grad_structs(specs):
        arr = (LayerGrad * len(specs))()
        for i, s in enumerate(specs):
            w = s["weight"]
            if dest is not None:
                g = dest[len(grads)]
            else:
                g = {"weight": torch.empty_like(w), "bias": torch.empty(w.shape[0], device=dev) if s.get("bias") is not None else None,
                     "bn_weight": None, "bn_bias": None}
                if s.get("bn") is not None:
                    g["bn_weight"] = torch.empty(w.shape[0], device=dev); g["bn_bias"] = torch.empty(w.shape[0], device=dev)
            arr[i].weight, arr[i].bias = _p(g["weight"]), _p(g["bias"])
            arr[i].bn_weight, arr[i].bn_bias = _p(g["bn_weight"]), _p(g["bn_bias"])
            grads.append(g)
        return arr

    with torch.cuda.device(dev):
        gconv = grad_structs(conv_specs)
        gfc = grad_structs(fc_specs)
        wsb = int(getattr(lib(), "snb200_%s_workspace_bytes" % entry)(b, n, len(conv_specs), conv, len(fc_specs), fc))
        ws, _ = _workspace(dev, wsb)
        zp = (ctypes.c_void_p * len(zs))(*[z.data_ptr() for z in zs])
        check(getattr(lib(), "snb200_" + entry)(b, n, lay, _p(x), len(conv_specs), conv, len(fc_specs), fc, zp, _p(fwd_ws), _p(grad_out),
                                                int(out_transpose_inner), gconv, gfc, _p(ws), wsb, _stream()), entry)
    del keep
    return grads


def generator_backward(x, layout, conv_specs, fc_specs, saved, grad_out, out_transpose_inner=0, dest=None):
    """Gradients of every generator parameter (hand-written CUDA; csrc/generator_bwd.cu).  Returns a list, in layer order (conv then fc), of
    dicts {weight, bias, bn_weight, bn_bias} (bn_* None for layers without BatchNorm).  dest: optional list of such dicts of preallocated
    contiguous tensors the kernels write into (e.g. the parameters' .grad views of a flat bucket) instead of fresh tensors."""
    return _backward("generator_backward", x, layout, conv_specs, fc_specs, saved, grad_out, out_transpose_inner, dest)


def generator_layers_backward(x, layout, conv_specs, fc_specs, saved, grad_out, out_transpose_inner=0, dest=None):
    """generator_backward for what generator_layers_train_forward saved (the same kernels; 256-wide conv layers split over the grid)."""
    return _backward("generator_layers_backward", x, layout, conv_specs, fc_specs, saved, grad_out, out_transpose_inner, dest)


def _layers_ex_args(x, conv_specs, fc_specs):
    """Prologue of the extended per-layer entries: (act_input, b, n, conv table, FC table, tap, dropout pointer array, keep).  x is the cloud
    (B, N, 3), or an activation (B, N, c_in) when layer 1 takes c_in != 3 channels.  A conv spec with "tap": True is the tapped layer; an FC
    spec's "dropout" is the (B, c_in) mask of its input."""
    conv, keep_conv = make_layers(conv_specs)
    fc, keep_fc = make_layers(fc_specs)
    c_in = conv[0].c_in
    if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.shape[2] != c_in:
        raise ValueError("the layer stack expects its input of shape (batch, points, %d), got %s" % (c_in, tuple(getattr(x, "shape", ()))))
    taps = [i for i, s in enumerate(conv_specs) if s.get("tap")]
    if len(taps) > 1:
        raise ValueError("at most one tapped conv layer, got %s" % taps)
    b, n = x.shape[0], x.shape[1]
    masks = []
    for l, s in enumerate(fc_specs):
        m = s.get("dropout")
        if m is not None:
            m = _req(m, "dropout mask")
            if tuple(m.shape) != (b, fc[l].c_in):
                raise ValueError("FC layer %d's dropout mask must be (%d, %d), got %s" % (l, b, fc[l].c_in, tuple(m.shape)))
        masks.append(m)
    drop = (ctypes.c_void_p * len(fc_specs))(*[None if m is None else m.data_ptr() for m in masks])
    return int(c_in != 3), b, n, conv, fc, taps[0] if taps else -1, drop, keep_conv + keep_fc + [m for m in masks if m is not None]


def generator_layers_ex_supported(x, conv_specs, fc_specs):
    """snb200_generator_layers_ex_supported for the layer stack of LayerStackFunction: x (its input), taps and dropout as there."""
    act, b, n, conv, fc, tap, drop, keep = _layers_ex_args(x, conv_specs, fc_specs)
    return bool(lib().snb200_generator_layers_ex_supported(b, n, act, len(conv_specs), conv, len(fc_specs), fc, tap, drop))


_LAYER_GRAD_KEYS = ("weight", "bias", "bn_weight", "bn_bias")


class LayerStackFunction(torch.autograd.Function):
    """(x, conv_specs, fc_specs, *params) -> (out (B, c_out_last), feat (B, c_conv_last)[, tap (B, N, c_tap)]): a trainable task-network layer
    stack -- 1x1 convs with BatchNorm over the batch and ReLU, max-pool, FC head -- on the per-layer training path
    (snb200_generator_layers_ex_train_forward / _backward).  `params` are the tensors the specs hold, per layer in spec order: weight, bias[,
    BatchNorm weight, bias].  They are inputs so that needs_input_grad decides which gradients the backward writes; the others are NULL
    pointers.  The forward updates the running statistics (and num_batches_tracked) the specs point to.
      x        the cloud (B, N, 3), or an activation (B, N, c_in) that layer 1 reads as it is when it takes c_in != 3 channels.  Differentiable.
      tap      a conv spec with "tap": True also returns its activation relu(bn(z)), differentiable.
      dropout  an FC spec's "dropout": a (B, c_in) mask (0 or 1/(1-p)) multiplying that layer's input, in the forward and the backward.
    feat is not differentiable.  The saved activations and forward workspace are this call's own (never a PrimedWorkspaces buffer), so
    forwards may run ahead of backwards."""

    @staticmethod
    def forward(ctx, x, conv_specs, fc_specs, *params):
        x = _req(x, "x")
        act, b, n, conv, fc, tap, drop, keep = _layers_ex_args(x, conv_specs, fc_specs)
        nconv, nfc = len(conv_specs), len(fc_specs)
        dev = x.device
        with torch.cuda.device(dev):
            # fresh buffers even under an active PrimedWorkspaces: a second forward before this backward must not overwrite what it keeps
            wsb = int(lib().snb200_generator_workspace_bytes(b, n, nconv, conv, nfc, fc))
            ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
            zs = [torch.empty(b * n, conv[l].c_out, device=dev) for l in range(nconv)]
            zp = (ctypes.c_void_p * nconv)(*[z.data_ptr() for z in zs])
            feat = torch.empty(b, conv[nconv - 1].c_out, device=dev)
            out = torch.empty(b, fc[nfc - 1].c_out, device=dev)
            h = torch.empty(b, n, conv[tap].c_out, device=dev) if tap >= 0 else None
            check(lib().snb200_generator_layers_ex_train_forward(b, n, BNC, act, _p(x), nconv, conv, nfc, fc, tap, _p(h), drop, _p(out), 0, _p(feat),
                                                                 zp, 0, _p(ws), wsb, _stream()), "generator_layers_ex_train_forward")
        ctx.conv_specs, ctx.fc_specs, ctx.cuda_saved = conv_specs, fc_specs, (zs, ws)
        ctx.save_for_backward(x, *params)
        ctx.mark_non_differentiable(feat)
        del keep
        return (out, feat) if h is None else (out, feat, h)

    @staticmethod
    def backward(ctx, g, g_feat, *g_tap):
        x, *params = ctx.saved_tensors
        gt = g_tap[0] if g_tap else None
        if g is None and gt is None:
            return (None,) * (3 + len(params))
        need = ctx.needs_input_grad[3:]
        act, b, n, conv, fc, tap, drop, keep = _layers_ex_args(x, ctx.conv_specs, ctx.fc_specs)
        nconv, nfc = len(ctx.conv_specs), len(ctx.fc_specs)
        dev = x.device
        grads, flat = [], []

        def grad_structs(specs, k):
            arr = (LayerGrad * len(specs))()
            for i, s in enumerate(specs):
                d = dict.fromkeys(_LAYER_GRAD_KEYS)
                for key in _LAYER_GRAD_KEYS[:2 if s["bn"] is None else 4]:
                    d[key] = torch.empty_like(params[k]) if need[k] else None
                    flat.append(d[key])
                    k += 1
                arr[i].weight, arr[i].bias, arr[i].bn_weight, arr[i].bn_bias = (_p(d[key]) for key in _LAYER_GRAD_KEYS)
            return arr, k

        with torch.cuda.device(dev):
            gconv, k = grad_structs(ctx.conv_specs, 0)
            gfc, _ = grad_structs(ctx.fc_specs, k)
            g = torch.zeros(b, fc[nfc - 1].c_out, device=dev) if g is None else _req(g, "grad_out")
            gt = None if gt is None else _req(gt, "grad_tap")
            gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
            wsb = int(lib().snb200_generator_layers_ex_backward_workspace_bytes(b, n, act, nconv, conv, nfc, fc))
            ws, _ = _workspace(dev, wsb)
            zs, fwd_ws = ctx.cuda_saved
            zp = (ctypes.c_void_p * nconv)(*[z.data_ptr() for z in zs])
            check(lib().snb200_generator_layers_ex_backward(b, n, BNC, act, _p(x), nconv, conv, nfc, fc, tap, drop, zp, _p(fwd_ws), _p(g), 0, _p(gt),
                                                            _p(gx), gconv, gfc, _p(ws), wsb, _stream()), "generator_layers_ex_backward")
        del keep
        return (gx, None, None, *flat)


def generator_forward_unfused(x, layout, conv_specs, fc_specs, training, out_transpose_inner=0):
    """Same result through the two stand-alone entry points snb200_encoder_forward + snb200_fc_head_forward: the exact-fp32
    CUDA-core conv stack, then the generator's cluster head twice, once for the pool and once for the FC layers.  Bit for bit
    what generator_forward(..., exact_fp32=True) returns, running statistics and num_batches_tracked included."""
    lay, b, n, conv, fc, keep = _generator_args(x, layout, conv_specs, fc_specs)
    x = _req(x, "x")
    dev = x.device
    with torch.cuda.device(dev):
        ws1b = int(lib().snb200_encoder_workspace_bytes(b, n, len(conv_specs), conv))
        ws2b = int(lib().snb200_fc_head_workspace_bytes(b, len(fc_specs), fc))
        ws1, _ = _workspace(dev, ws1b)
        ws2, _ = _workspace(dev, ws2b)
        feat = torch.empty(b, conv[len(conv_specs) - 1].c_out, device=dev)
        out = torch.empty(b, fc[len(fc_specs) - 1].c_out, device=dev)
        check(lib().snb200_encoder_forward(b, n, lay, _p(x), len(conv_specs), conv, int(bool(training)), _p(feat), _p(ws1), ws1b, _stream()),
              "encoder_forward")
        check(lib().snb200_fc_head_forward(b, _p(feat), len(fc_specs), fc, int(bool(training)), _p(out), int(out_transpose_inner), _p(ws2), ws2b, _stream()),
              "fc_head_forward")
    del keep
    return out, feat


# ----------------------------------------------------------------------------------------------------- frozen encoder over prefixes
def _frozen_args(x, conv_specs, sizes):
    """(b, n, P, C layer table, host sizes array, tensors to keep alive) of a frozen-encoder call; x is (B, N, 3)."""
    if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.shape[2] != 3:
        raise ValueError("the frozen encoder expects x of shape (batch, points, 3)")
    b, n = x.shape[0], x.shape[1]
    conv, keep = make_layers(conv_specs)
    sizes = [int(s) for s in sizes]
    csz = (ctypes.c_int * max(len(sizes), 1))(*sizes)
    return b, n, len(sizes), conv, csz, keep


def frozen_encoder_forward(x, conv_specs, sizes, keep_activations=True):
    """A frozen conv stack (eval-mode BatchNorm) and its max-pool over every prefix x[:, :s], s in `sizes`, in one shared pass
    (csrc/frozen_encoder.cu).  Returns (pooled (P, B, C), route (P, B, C) int32: the point each value comes from, zsave: the hidden layers'
    raw outputs (B*N, c_l) for the backward, or None with keep_activations=False)."""
    x = _req(x, "x")
    b, n, npf, conv, csz, keep = _frozen_args(x, conv_specs, sizes)
    nconv = len(conv_specs)
    dev = x.device
    with torch.cuda.device(dev):
        c = conv[nconv - 1].c_out
        pooled = torch.empty(npf, b, c, device=dev)
        route = torch.empty(npf, b, c, device=dev, dtype=torch.int32)
        zs = [torch.empty(b * n, conv[l].c_out, device=dev) for l in range(nconv - 1)] if keep_activations else None
        zp = (ctypes.c_void_p * (nconv - 1))(*[z.data_ptr() for z in zs]) if keep_activations else None
        wsb = int(lib().snb200_frozen_encoder_workspace_bytes(b, n, nconv, conv, npf, int(keep_activations)))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_forward(b, n, _p(x), nconv, conv, npf, csz, _p(pooled), _p(route), zp, _p(ws), wsb, _stream()),
              "frozen_encoder_forward")
    del keep
    return pooled, route, zs


def frozen_encoder_backward(x, conv_specs, sizes, pooled, route, zsave, grad_pooled):
    """Gradient with respect to x (B, N, 3) of sum(grad_pooled * pooled) through the frozen encoder (no parameter gradients)."""
    x, pooled, grad_pooled = _req(x, "x"), _req(pooled, "pooled"), _req(grad_pooled, "grad_pooled")
    route = _req(route, "route", torch.int32)
    b, n, npf, conv, csz, keep = _frozen_args(x, conv_specs, sizes)
    nconv = len(conv_specs)
    dev = x.device
    with torch.cuda.device(dev):
        gx = torch.empty_like(x)
        zp = (ctypes.c_void_p * (nconv - 1))(*[z.data_ptr() for z in zsave])
        wsb = int(lib().snb200_frozen_encoder_backward_workspace_bytes(b, n, nconv, conv, npf))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_backward(b, n, _p(x), nconv, conv, npf, csz, _p(pooled), _p(route), zp, _p(grad_pooled), _p(gx), _p(ws), wsb,
                                                   _stream()), "frozen_encoder_backward")
    del keep
    return gx


def frozen_encoder_supported(b, n, conv_specs, num_prefix):
    conv, keep = make_layers(conv_specs)
    return bool(lib().snb200_frozen_encoder_supported(int(b), int(n), len(conv_specs), conv, int(num_prefix)))


FROZEN_MAX_PREFIX = 16     # prefixes per frozen_encoder_forward call; frozen_encoder_curve_forward takes up to N


def _curve_sizes(sizes, n):
    """The host array of a frozen_encoder_curve call: 1 to n ascending, distinct sizes in [1, n], else ValueError."""
    sizes = [int(s) for s in sizes]
    if not sizes or sizes[0] < 1 or sizes[-1] > n or any(a >= c for a, c in zip(sizes, sizes[1:])):
        raise ValueError("frozen_encoder_curve: sizes must be ascending, distinct and in [1, %d]" % n)
    return (ctypes.c_int * len(sizes))(*sizes)


def frozen_encoder_curve_forward(x, conv_specs, sizes):
    """frozen_encoder_forward's (pooled (P, B, C), route (P, B, C) int32) for any number of sizes, up to every s in [1, N], from one pass of
    the conv stack (csrc/frozen_encoder.cu, the _curve entries): bit for bit what frozen_encoder_forward gives 16 sizes at a time.  Forward
    only, no gradient; sizes ascending and distinct."""
    if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.shape[2] != 3:
        raise ValueError("the frozen encoder expects x of shape (batch, points, 3)")
    csz = _curve_sizes(sizes, x.shape[1])
    x = _req(x, "x")
    b, n, _, conv, _, keep = _frozen_args(x, conv_specs, [])
    npf, nconv = len(csz), len(conv_specs)
    dev = x.device
    with torch.cuda.device(dev):
        c = conv[nconv - 1].c_out
        pooled = torch.empty(npf, b, c, device=dev)
        route = torch.empty(npf, b, c, device=dev, dtype=torch.int32)
        wsb = int(lib().snb200_frozen_encoder_curve_workspace_bytes(b, n, nconv, conv, npf, csz))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_curve_forward(b, n, _p(x), nconv, conv, npf, csz, _p(pooled), _p(route), _p(ws), wsb, _stream()),
              "frozen_encoder_curve_forward")
    del keep
    return pooled, route


def frozen_encoder_curve_supported(b, n, conv_specs, sizes):
    """Whether frozen_encoder_curve_forward takes b clouds of n points with these sizes (ascending, distinct, in [1, n])."""
    conv, keep = make_layers(conv_specs)
    sizes = [int(s) for s in sizes]
    csz = (ctypes.c_int * max(len(sizes), 1))(*sizes)
    return bool(lib().snb200_frozen_encoder_curve_supported(int(b), int(n), len(conv_specs), conv, len(sizes), csz))


class FrozenEncoderFunction(torch.autograd.Function):
    """(x (B, N, 3), conv_specs, sizes) -> (pooled (P, B, C), route (P, B, C) int32): the frozen encoder's max-pool over every prefix
    x[:, :s], from one shared pass.  Differentiable in x only (the parameters are frozen); route is not differentiable."""

    @staticmethod
    def forward(ctx, x, conv_specs, sizes):
        x = x.contiguous()
        pooled, route, zs = frozen_encoder_forward(x, conv_specs, sizes, keep_activations=ctx.needs_input_grad[0])
        ctx.conv_specs, ctx.sizes = conv_specs, [int(s) for s in sizes]
        ctx.save_for_backward(x, pooled, route, *(zs or []))
        ctx.mark_non_differentiable(route)
        return pooled, route

    @staticmethod
    def backward(ctx, g, g_route):
        x, pooled, route, *zs = ctx.saved_tensors
        if g is None:
            return None, None, None
        return frozen_encoder_backward(x, ctx.conv_specs, ctx.sizes, pooled, route, zs, g.contiguous()), None, None


# ----------------------------------------------------------------------------------------------------- frozen encoder, batch statistics
def _bstat_args(conv_specs, sizes):
    conv, keep = make_layers(conv_specs)
    sizes = [int(s) for s in sizes]
    return conv, len(sizes), (ctypes.c_int * max(len(sizes), 1))(*sizes), keep


def frozen_encoder_bstat_supported(b, n, conv_specs, sizes):
    """Whether the frozen encoder with per-prefix batch statistics (csrc/frozen_encoder_bstat.cu) takes B = b clouds of n points and the
    prefix sizes `sizes`: 1..16 ascending distinct sizes in [1, n], n <= 4096, b * sum(pad128(s)) <= 2^22 rows, and the frozen encoder's
    layer table with BatchNorm, a bias and ReLU on every layer."""
    conv, npf, csz, keep = _bstat_args(conv_specs, sizes)
    return bool(lib().snb200_frozen_encoder_bstat_supported(int(b), int(n), len(conv_specs), conv, npf, csz))


def frozen_encoder_bstat_stats(stats, conv_specs, num_prefix):
    """The forward's flat `stats` (float64) as one (P, 2, c_out_l) view per layer: per prefix the mean and biased variance of the layer's raw
    output over that prefix's B * s points."""
    out, off = [], 0
    for spec in conv_specs:
        c = spec["weight"].shape[0]
        out.append(stats[off:off + num_prefix * 2 * c].view(num_prefix, 2, c))
        off += num_prefix * 2 * c
    return out


def frozen_encoder_bstat_forward(x, conv_specs, sizes):
    """A frozen conv stack whose BatchNorms normalise with the batch statistics of each prefix x[:, :s], s in `sizes`, and its max-pool, in
    one pass (csrc/frozen_encoder_bstat.cu).  Returns (pooled (P, B, C), route (P, B, C) int32, stats (flat float64, see
    frozen_encoder_bstat_stats), ws: the workspace holding every layer's raw output, which the backward reads).  Nothing of the layer table
    is written, the running statistics included."""
    x = _req(x, "x")
    if x.dim() != 3 or x.shape[2] != 3:
        raise ValueError("the frozen encoder expects x of shape (batch, points, 3)")
    b, n = x.shape[0], x.shape[1]
    conv, npf, csz, keep = _bstat_args(conv_specs, sizes)
    nconv, dev = len(conv_specs), x.device
    with torch.cuda.device(dev):
        pooled = torch.empty(npf, b, conv[nconv - 1].c_out, device=dev)
        route = torch.empty(npf, b, conv[nconv - 1].c_out, device=dev, dtype=torch.int32)
        stats = torch.empty(npf * 2 * sum(conv[l].c_out for l in range(nconv)), device=dev, dtype=torch.float64)
        wsb = int(lib().snb200_frozen_encoder_bstat_workspace_bytes(b, n, nconv, conv, npf, csz))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_bstat_forward(b, n, _p(x), nconv, conv, npf, csz, _p(pooled), _p(route), _p(stats), _p(ws), wsb,
                                                        _stream()), "frozen_encoder_bstat_forward")
    del keep
    return pooled, route, stats, ws


def frozen_encoder_bstat_backward(x, conv_specs, sizes, pooled, route, stats, ws, grad_pooled):
    """Gradient with respect to x (B, N, 3) of sum(grad_pooled * pooled) through the batch-statistics encoder, from the forward's outputs
    and workspace (no parameter gradients)."""
    x, pooled, grad_pooled = _req(x, "x"), _req(pooled, "pooled"), _req(grad_pooled, "grad_pooled")
    route = _req(route, "route", torch.int32)
    stats = _req(stats, "stats", torch.float64)
    b, n = x.shape[0], x.shape[1]
    conv, npf, csz, keep = _bstat_args(conv_specs, sizes)
    nconv, dev = len(conv_specs), x.device
    with torch.cuda.device(dev):
        gx = torch.empty_like(x)
        wsb = int(lib().snb200_frozen_encoder_bstat_backward_workspace_bytes(b, n, nconv, conv, npf, csz))
        bws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_bstat_backward(b, n, nconv, conv, npf, csz, _p(pooled), _p(route), _p(stats), _p(ws), ws.numel(),
                                                         _p(grad_pooled), _p(gx), _p(bws), wsb, _stream()), "frozen_encoder_bstat_backward")
    del keep
    return gx


class FrozenEncoderBStatFunction(torch.autograd.Function):
    """(x (B, N, 3), conv_specs, sizes) -> (pooled (P, B, C), route (P, B, C) int32, stats flat float64): the frozen encoder with every
    BatchNorm normalised by the batch statistics of each prefix x[:, :s] (the mean and biased variance over its B * s points), from one
    pass.  Differentiable in x only, through pooled (the statistics' dependence on x included); route and stats are not differentiable."""

    @staticmethod
    def forward(ctx, x, conv_specs, sizes):
        x = x.contiguous()
        pooled, route, stats, ws = frozen_encoder_bstat_forward(x, conv_specs, sizes)
        ctx.conv_specs, ctx.sizes = conv_specs, [int(s) for s in sizes]
        if ctx.needs_input_grad[0]:
            ctx.save_for_backward(x, pooled, route, stats, ws)
        ctx.mark_non_differentiable(route, stats)
        return pooled, route, stats

    @staticmethod
    def backward(ctx, g, g_route, g_stats):
        if g is None:
            return None, None, None
        x, pooled, route, stats, ws = ctx.saved_tensors
        return frozen_encoder_bstat_backward(x, ctx.conv_specs, ctx.sizes, pooled, route, stats, ws, g.contiguous()), None, None


# ----------------------------------------------------------------------------------------------------- batch-statistics encoder, trained
def frozen_encoder_bstat_train_supported(b, n, conv_specs, sizes):
    """Whether the batch-statistics encoder trains (frozen_encoder_bstat_param_backward, frozen_encoder_bstat_running_update) on B = b
    clouds of n points and `sizes`: frozen_encoder_bstat_supported's envelope with b * s >= 2 for every prefix."""
    conv, npf, csz, keep = _bstat_args(conv_specs, sizes)
    return bool(lib().snb200_frozen_encoder_bstat_param_backward_supported(int(b), int(n), len(conv_specs), conv, npf, csz))


_BN_GRAD_KEYS = ("weight", "bias", "bn_weight", "bn_bias")


def frozen_encoder_bstat_param_backward(x, conv_specs, sizes, pooled, route, stats, ws, grad_pooled, want, need_x=True):
    """frozen_encoder_bstat_backward with parameter gradients (csrc/frozen_encoder_bstat.cu), from the forward's outputs and workspace.
    want: per layer (weight?, bias?, bn weight?, bn bias?).  Returns (grad_x (B, N, 3) or None without need_x, [(dW (c_out, c_in), db,
    dgamma, dbeta), each None where not wanted, per layer]); grad_x is bit for bit frozen_encoder_bstat_backward's."""
    what = "frozen_encoder_bstat_param_backward"
    x, pooled, grad_pooled = _req(x, "x"), _req(pooled, "pooled"), _req(grad_pooled, "grad_pooled")
    route = _req(route, "route", torch.int32)
    stats = _req(stats, "stats", torch.float64)
    b, n = x.shape[0], x.shape[1]
    conv, npf, csz, keep = _bstat_args(conv_specs, sizes)
    nconv, dev = len(conv_specs), x.device
    with torch.cuda.device(dev):
        gx = torch.empty_like(x) if need_x else None
        garr, grads = (LayerGrad * nconv)(), []
        for i, w in enumerate(want):
            c_out, c_in = conv[i].c_out, conv[i].c_in
            g = [torch.empty(c_out, c_in, device=dev) if w[0] else None] + [torch.empty(c_out, device=dev) if f else None for f in w[1:]]
            for key, t in zip(_BN_GRAD_KEYS, g):
                setattr(garr[i], key, _p(t))
            grads.append(tuple(g))
        wsb = int(lib().snb200_frozen_encoder_bstat_param_backward_workspace_bytes(b, n, nconv, conv, npf, csz))
        bws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_bstat_param_backward(b, n, _p(x), nconv, conv, npf, csz, _p(pooled), _p(route), _p(stats), _p(ws),
                                                               ws.numel(), _p(grad_pooled), _p(gx), garr, _p(bws), wsb, _stream()), what)
    del keep
    return gx, grads


def frozen_encoder_bstat_running_update(x, conv_specs, sizes, stats):
    """Move the running statistics the specs point to (and num_batches_tracked) as nn.BatchNorm1d does in training mode for each prefix
    x[:, :s] in ascending order, from the forward's `stats` (snb200_frozen_encoder_bstat_running_update, one launch).  A BatchNorm with
    momentum=None (torch's cumulative average) raises ValueError: the update is the exponential one."""
    for i, spec in enumerate(conv_specs):
        if spec.get("bn") is not None and spec["bn"][5] is None:
            raise ValueError("frozen_encoder_bstat_running_update: layer %d's BatchNorm has momentum=None (a cumulative average); the update "
                             "is nn.BatchNorm1d's exponential average with a momentum" % i)
    stats = _req(stats, "stats", torch.float64)
    b, n = x.shape[0], x.shape[1]
    conv, npf, csz, keep = _bstat_args(conv_specs, sizes)
    with torch.cuda.device(stats.device):
        check(lib().snb200_frozen_encoder_bstat_running_update(b, n, len(conv_specs), conv, npf, csz, _p(stats), _stream()),
              "frozen_encoder_bstat_running_update")
    del keep


class EncoderBStatTrainFunction(torch.autograd.Function):
    """(x (B, N, 3), conv_specs, sizes, *params) -> (pooled (P, B, C), route (P, B, C) int32, stats flat float64): the autoencoder's encoder
    in training mode over every prefix x[:, :s] from one pass: every BatchNorm normalises prefix s with its own batch statistics, and the
    running statistics the specs point to move once per prefix in ascending order (nn.BatchNorm1d's update; num_batches_tracked + P).
    `params` are the tensors the specs hold, per layer: conv weight, conv bias, BatchNorm weight, BatchNorm bias.  They are inputs so that
    needs_input_grad decides which gradients the backward writes; the others are NULL pointers.  Differentiable in x and params through
    pooled; route and stats are not differentiable.  A BatchNorm with momentum=None raises ValueError (before anything launches).  No host
    synchronisation: the call can be captured in a CUDA graph."""

    @staticmethod
    def forward(ctx, x, conv_specs, sizes, *params):
        if any(s.get("bn") is not None and s["bn"][5] is None for s in conv_specs):
            raise ValueError("EncoderBStatTrainFunction: a BatchNorm with momentum=None (a cumulative average) is not supported")
        x = x.contiguous()
        sizes = [int(s) for s in sizes]
        pooled, route, stats, ws = frozen_encoder_bstat_forward(x, conv_specs, sizes)
        frozen_encoder_bstat_running_update(x, conv_specs, sizes, stats)
        ctx.conv_specs, ctx.sizes, ctx.param_shapes = conv_specs, sizes, [p.shape for p in params]
        if any(ctx.needs_input_grad):
            ctx.save_for_backward(x, pooled, route, stats, ws)
        ctx.mark_non_differentiable(route, stats)
        return pooled, route, stats

    @staticmethod
    def backward(ctx, g, g_route, g_stats):
        need = ctx.needs_input_grad
        nparams = len(ctx.param_shapes)
        if g is None:
            return (None,) * (3 + nparams)
        x, pooled, route, stats, ws = ctx.saved_tensors
        g = g.contiguous()
        want = [tuple(need[3 + 4 * i:7 + 4 * i]) for i in range(nparams // 4)]
        if not any(any(w) for w in want):
            return (frozen_encoder_bstat_backward(x, ctx.conv_specs, ctx.sizes, pooled, route, stats, ws, g), None, None) + (None,) * nparams
        gx, grads = frozen_encoder_bstat_param_backward(x, ctx.conv_specs, ctx.sizes, pooled, route, stats, ws, g, want, need_x=need[0])
        flat = [t for layer in grads for t in layer]
        return (gx, None, None, *[None if t is None else t.view(ctx.param_shapes[i]) for i, t in enumerate(flat)])


# ----------------------------------------------------------------------------------------------------- frozen MLP head
# The two families of C entries: "frozen_mlp" (no BatchNorm) and "frozen_mlp_bn" (eval-mode BatchNorm allowed on any layer); same kernels.
def _mlp_entry(name, bn):
    return getattr(lib(), "snb200_%s_%s" % ("frozen_mlp_bn" if bn else "frozen_mlp", name))


def _mlp_args(x, fc_specs, what, bn=False):
    """(b, layer table, tensors to keep alive) of a frozen-MLP call; x is (B, c_in of the first layer)."""
    if not isinstance(x, torch.Tensor) or x.dim() != 2:
        raise ValueError("%s expects a (batch, channels) tensor" % what)
    fc, keep = make_layers(fc_specs)
    if x.shape[1] != fc[0].c_in:
        raise ValueError("%s: %d channels given, the first layer takes %d" % (what, x.shape[1], fc[0].c_in))
    if not _mlp_entry("supported", bn)(x.shape[0], len(fc_specs), fc):
        raise ValueError("%s: %d rows through %s are outside the frozen MLP's envelope (1..64 rows, c_in a multiple of 8 up to 4096, c_out up "
                         "to 4096, %s, no ReLU on the last layer)" % (what, x.shape[0], [(l.c_in, l.c_out) for l in fc],
                                                                       "eval-mode BatchNorm allowed" if bn else "no BatchNorm"))
    return x.shape[0], fc, keep


def frozen_mlp_supported(b, fc_specs, batchnorm=False):
    fc, keep = make_layers(fc_specs)
    return bool(_mlp_entry("supported", batchnorm)(int(b), len(fc_specs), fc))


def frozen_mlp_forward(x, fc_specs, keep_activations=True, batchnorm=False):
    """A frozen stack of Linear (+ ReLU) layers on x (B <= 64, C) (csrc/frozen_mlp.cu).  Returns (out (B, c_out_last), asave: the hidden
    layers' activations for the backward, or None with keep_activations=False).  batchnorm=True: the layers may carry eval-mode BatchNorm
    (`bn` of the specs, applied from the running statistics behind the bias)."""
    what = "frozen_mlp_bn_forward" if batchnorm else "frozen_mlp_forward"
    x = _req(x, "x")
    b, fc, keep = _mlp_args(x, fc_specs, what, batchnorm)
    nl = len(fc_specs)
    dev = x.device
    with torch.cuda.device(dev):
        out = torch.empty(b, fc[nl - 1].c_out, device=dev)
        asave = [torch.empty(b, fc[l].c_out, device=dev) for l in range(nl - 1)] if keep_activations else None
        ap = (ctypes.c_void_p * max(nl - 1, 1))(*[a.data_ptr() for a in asave]) if keep_activations else None
        wsb = int(_mlp_entry("workspace_bytes", batchnorm)(b, nl, fc, int(keep_activations)))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(_mlp_entry("forward", batchnorm)(b, _p(x), nl, fc, _p(out), ap, _p(ws), wsb, _stream()), what)
    del keep
    return out, asave


def frozen_mlp_backward(fc_specs, asave, grad_out, batchnorm=False):
    """Gradient with respect to the input (B, c_in_0) of sum(grad_out * out) through the frozen MLP (no parameter gradients)."""
    what = "frozen_mlp_bn_backward" if batchnorm else "frozen_mlp_backward"
    grad_out = _req(grad_out, "grad_out")
    fc, keep = make_layers(fc_specs)
    nl = len(fc_specs)
    if grad_out.dim() != 2 or grad_out.shape[1] != fc[nl - 1].c_out or len(asave) != nl - 1:
        raise ValueError("%s expects grad_out (batch, %d) and %d saved activations" % (what, fc[nl - 1].c_out, nl - 1))
    b = grad_out.shape[0]
    asave = [_req(a, "asave") for a in asave]
    if any(tuple(a.shape) != (b, fc[l].c_out) for l, a in enumerate(asave)):
        raise ValueError("%s: saved activations do not match the layer table" % what)
    if not _mlp_entry("supported", batchnorm)(b, nl, fc):
        raise ValueError("%s: outside the frozen MLP's envelope" % what)
    dev = grad_out.device
    with torch.cuda.device(dev):
        gx = torch.empty(b, fc[0].c_in, device=dev)
        ap = (ctypes.c_void_p * max(nl - 1, 1))(*[a.data_ptr() for a in asave])
        wsb = int(_mlp_entry("backward_workspace_bytes", batchnorm)(b, nl, fc))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(_mlp_entry("backward", batchnorm)(b, nl, fc, ap, _p(grad_out), _p(gx), _p(ws), wsb, _stream()), what)
    del keep
    return gx


class FrozenMLPFunction(torch.autograd.Function):
    """(x (B, C), fc_specs) -> out (B, c_out_last) through a frozen MLP.  Differentiable in x only (the parameters are frozen)."""

    @staticmethod
    def forward(ctx, x, fc_specs):
        out, asave = frozen_mlp_forward(x.contiguous(), fc_specs, keep_activations=ctx.needs_input_grad[0])
        ctx.fc_specs = fc_specs
        ctx.save_for_backward(*(asave or []))
        return out

    @staticmethod
    def backward(ctx, g):
        return frozen_mlp_backward(ctx.fc_specs, list(ctx.saved_tensors), g.contiguous()), None


class FrozenMLPBNFunction(torch.autograd.Function):
    """(x (B, C), fc_specs) -> out (B, c_out_last) through a frozen MLP whose layers may carry eval-mode BatchNorm (the snb200_frozen_mlp_bn_*
    entries).  Differentiable in x only (the parameters are frozen).  With last_hidden=True -> (out, the last hidden layer's activation, as
    the same launches write it for the backward; not differentiable)."""

    @staticmethod
    def forward(ctx, x, fc_specs, last_hidden=False):
        keep = ctx.needs_input_grad[0]
        out, asave = frozen_mlp_forward(x.contiguous(), fc_specs, keep_activations=keep or last_hidden, batchnorm=True)
        ctx.fc_specs = fc_specs
        ctx.save_for_backward(*(asave if keep else []))
        if not last_hidden:
            return out
        ctx.mark_non_differentiable(asave[-1])
        return out, asave[-1]

    @staticmethod
    def backward(ctx, g, *_):
        return frozen_mlp_backward(ctx.fc_specs, list(ctx.saved_tensors), g.contiguous(), batchnorm=True), None, None


# ----------------------------------------------------------------------------------------------------- parameter gradients (no BatchNorm)
def _grad_table(specs, want):
    """(snb200_layer_grad array, [(dW (c_out, c_in) or None, db (c_out) or None) per layer]): fresh tensors for what `want`, a (weight?, bias?)
    pair per layer, asks for; NULL pointers elsewhere."""
    arr = (LayerGrad * len(specs))()
    out = []
    for i, (s, (ww, wb)) in enumerate(zip(specs, want)):
        w = s["weight"].reshape(s["weight"].shape[0], -1)
        gw = torch.empty(w.shape, device=w.device) if ww else None
        gb = torch.empty(w.shape[0], device=w.device) if wb else None
        arr[i].weight, arr[i].bias, arr[i].bn_weight, arr[i].bn_bias = _p(gw), _p(gb), None, None
        out.append((gw, gb))
    return arr, out


def frozen_encoder_param_backward_supported(b, n, conv_specs, num_prefix):
    conv, keep = make_layers(conv_specs)
    return bool(lib().snb200_frozen_encoder_param_backward_supported(int(b), int(n), len(conv_specs), conv, int(num_prefix)))


def frozen_encoder_param_backward(x, conv_specs, sizes, pooled, route, zsave, grad_pooled, want, need_x=True):
    """frozen_encoder_backward with weight and bias gradients, for conv layers without BatchNorm (csrc/frozen_encoder.cu).  want: per layer
    (weight?, bias?).  Returns (grad_x (B, N, 3) or None without need_x, [(dW (c_out, c_in) or None, db or None) per layer])."""
    what = "frozen_encoder_param_backward"
    x, pooled, grad_pooled = _req(x, "x"), _req(pooled, "pooled"), _req(grad_pooled, "grad_pooled")
    route = _req(route, "route", torch.int32)
    b, n, npf, conv, csz, keep = _frozen_args(x, conv_specs, sizes)
    nconv = len(conv_specs)
    if not lib().snb200_frozen_encoder_param_backward_supported(b, n, nconv, conv, npf):
        raise ValueError("%s: (%d, %d) clouds through %s are outside the envelope (the frozen encoder's, no BatchNorm)"
                         % (what, b, n, [(l.c_in, l.c_out) for l in conv]))
    dev = x.device
    with torch.cuda.device(dev):
        gx = torch.empty_like(x) if need_x else None
        garr, grads = _grad_table(conv_specs, want)
        zp = (ctypes.c_void_p * (nconv - 1))(*[z.data_ptr() for z in zsave])
        wsb = int(lib().snb200_frozen_encoder_param_backward_workspace_bytes(b, n, nconv, conv, npf))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_param_backward(b, n, _p(x), nconv, conv, npf, csz, _p(pooled), _p(route), zp, _p(grad_pooled), _p(gx),
                                                         garr, _p(ws), wsb, _stream()), what)
    del keep
    return gx, grads


def frozen_mlp_param_backward(x, fc_specs, asave, grad_out, want, need_x=True):
    """frozen_mlp_backward with weight and bias gradients (csrc/frozen_mlp.cu); x (B, c_in_0) is the head's input.  want: per layer
    (weight?, bias?).  Returns (grad_in or None without need_x, [(dW (c_out, c_in) or None, db or None) per layer])."""
    what = "frozen_mlp_param_backward"
    x, grad_out = _req(x, "x"), _req(grad_out, "grad_out")
    b, fc, keep = _mlp_args(x, fc_specs, what)
    nl = len(fc_specs)
    asave = [_req(a, "asave") for a in asave]
    if tuple(grad_out.shape) != (b, fc[nl - 1].c_out) or len(asave) != nl - 1 or any(tuple(a.shape) != (b, fc[l].c_out) for l, a in enumerate(asave)):
        raise ValueError("%s expects grad_out (%d, %d) and %d saved activations matching the layer table" % (what, b, fc[nl - 1].c_out, nl - 1))
    dev = x.device
    with torch.cuda.device(dev):
        gx = torch.empty_like(x) if need_x else None
        garr, grads = _grad_table(fc_specs, want)
        ap = (ctypes.c_void_p * max(nl - 1, 1))(*[a.data_ptr() for a in asave])
        wsb = int(lib().snb200_frozen_mlp_param_backward_workspace_bytes(b, nl, fc))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_mlp_param_backward(b, nl, fc, _p(x), ap, _p(grad_out), _p(gx), garr, _p(ws), wsb, _stream()), what)
    del keep
    return gx, grads


def _param_specs(relus, params):
    """Layer specs without BatchNorm from the flat (weight, bias, weight, bias, ...) parameter list of an autograd Function."""
    return [{"weight": params[2 * i], "bias": params[2 * i + 1], "bn": None, "relu": bool(r)} for i, r in enumerate(relus)]


def _param_grads(ctx, grads):
    """The gradients an autograd Function returns for its parameter inputs, shaped as the parameters."""
    out = []
    for i, (gw, gb) in enumerate(grads):
        out.append(None if gw is None else gw.view(ctx.param_shapes[2 * i]))
        out.append(gb)
    return out


class EncoderParamFunction(torch.autograd.Function):
    """(x (B, N, 3), sizes, relus, w_1, b_1, ..., w_L, b_L) -> (pooled (P, B, C), route (P, B, C) int32): the frozen encoder over conv layers
    without BatchNorm (weights (c_out, c_in[, 1])), differentiable in x and in every weight and bias; which gradients are computed follows
    needs_input_grad.  Parameter gradients come from snb200_frozen_encoder_param_backward, the gradient of x alone from
    snb200_frozen_encoder_backward (bit-identical to the former's grad_x)."""

    @staticmethod
    def forward(ctx, x, sizes, relus, *params):
        x = x.contiguous()
        specs = _param_specs(relus, params)
        pooled, route, zs = frozen_encoder_forward(x, specs, sizes, keep_activations=any(ctx.needs_input_grad))
        ctx.specs, ctx.sizes, ctx.param_shapes = specs, [int(s) for s in sizes], [None if p is None else p.shape for p in params]
        ctx.save_for_backward(x, pooled, route, *(zs or []))
        ctx.mark_non_differentiable(route)
        return pooled, route

    @staticmethod
    def backward(ctx, g, g_route):
        x, pooled, route, *zs = ctx.saved_tensors
        need = ctx.needs_input_grad
        want = [(need[3 + 2 * i], need[4 + 2 * i]) for i in range(len(ctx.specs))]
        if g is None:
            return (None,) * (3 + 2 * len(ctx.specs))
        if not any(w or b for w, b in want):
            return (frozen_encoder_backward(x, ctx.specs, ctx.sizes, pooled, route, zs, g.contiguous()), None, None) + (None,) * (2 * len(want))
        gx, grads = frozen_encoder_param_backward(x, ctx.specs, ctx.sizes, pooled, route, zs, g.contiguous(), want, need_x=need[0])
        return (gx, None, None, *_param_grads(ctx, grads))


class MLPParamFunction(torch.autograd.Function):
    """(x (B, C), relus, w_1, b_1, ..., w_L, b_L) -> out (B, c_out_last) through the frozen MLP's kernels, differentiable in x and in every
    weight and bias; which gradients are computed follows needs_input_grad (snb200_frozen_mlp_param_backward, or snb200_frozen_mlp_backward
    for the gradient of x alone)."""

    @staticmethod
    def forward(ctx, x, relus, *params):
        x = x.contiguous()
        specs = _param_specs(relus, params)
        out, asave = frozen_mlp_forward(x, specs, keep_activations=any(ctx.needs_input_grad))
        ctx.specs, ctx.param_shapes = specs, [None if p is None else p.shape for p in params]
        ctx.save_for_backward(x, *(asave or []))
        return out

    @staticmethod
    def backward(ctx, g):
        x, *asave = ctx.saved_tensors
        need = ctx.needs_input_grad
        want = [(need[2 + 2 * i], need[3 + 2 * i]) for i in range(len(ctx.specs))]
        if not any(w or b for w, b in want):
            return (frozen_mlp_backward(ctx.specs, asave, g.contiguous()), None) + (None,) * (2 * len(want))
        gx, grads = frozen_mlp_param_backward(x, ctx.specs, asave, g.contiguous(), want, need_x=need[0])
        return (gx, None, *_param_grads(ctx, grads))


# ----------------------------------------------------------------------------------------------------- frozen encoder: activation input, tap
def frozen_encoder_ex_supported(b, n, conv_specs, num_prefix, act_input=False, tap=-1):
    conv, keep = make_layers(conv_specs)
    return bool(lib().snb200_frozen_encoder_ex_supported(int(b), int(n), int(bool(act_input)), len(conv_specs), conv, int(num_prefix), int(tap)))


def _frozen_ex_args(x, conv_specs, sizes, act_input, what):
    """(b, n, P, layer table, host sizes, keep) of an extended frozen-encoder call; x is the cloud (B, N, 3) or an activation (B, N, c_in)."""
    conv, keep = make_layers(conv_specs)
    c_in = conv[0].c_in if act_input else 3
    if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.shape[2] != c_in:
        raise ValueError("%s expects %s of shape (batch, points, %d)" % (what, "an activation" if act_input else "x", c_in))
    sizes = [int(s) for s in sizes]
    csz = (ctypes.c_int * max(len(sizes), 1))(*sizes)
    return x.shape[0], x.shape[1], len(sizes), conv, csz, keep


def frozen_encoder_ex_forward(x, conv_specs, sizes, act_input=False, tap=-1, keep_activations=True):
    """The frozen encoder of frozen_encoder_forward, reading the cloud x (B, N, 3) or with act_input=True an activation x (B, N, c_in) as layer
    1's input, and with tap = t >= 0 also returning hidden layer t's activation relu(bn(z_t)) (B, N, c_t).  Returns (pooled (P, B, C), route,
    tapped activation or None, zsave or None)."""
    what = "frozen_encoder_ex_forward"
    x = _req(x, "x")
    b, n, npf, conv, csz, keep = _frozen_ex_args(x, conv_specs, sizes, act_input, what)
    nconv = len(conv_specs)
    dev = x.device
    with torch.cuda.device(dev):
        c = conv[nconv - 1].c_out
        pooled = torch.empty(npf, b, c, device=dev)
        route = torch.empty(npf, b, c, device=dev, dtype=torch.int32)
        h = torch.empty(b, n, conv[tap].c_out, device=dev) if tap >= 0 else None
        zs = [torch.empty(b * n, conv[l].c_out, device=dev) for l in range(nconv - 1)] if keep_activations else None
        zp = (ctypes.c_void_p * (nconv - 1))(*[z.data_ptr() for z in zs]) if keep_activations else None
        wsb = int(lib().snb200_frozen_encoder_ex_workspace_bytes(b, n, int(bool(act_input)), nconv, conv, npf, int(tap), int(keep_activations)))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_ex_forward(b, n, int(bool(act_input)), _p(x), nconv, conv, npf, csz, _p(pooled), _p(route), int(tap), _p(h),
                                                     zp, _p(ws), wsb, _stream()), what)
    del keep
    return pooled, route, h, zs


def frozen_encoder_ex_backward(x, conv_specs, sizes, pooled, route, zsave, grad_pooled, act_input=False, tap=-1, grad_tap=None):
    """Gradient with respect to x ((B, N, 3) or the activation (B, N, c_in)) of sum(grad_pooled * pooled) + sum(grad_tap * tapped activation);
    grad_tap=None: no gradient reached the tapped activation."""
    what = "frozen_encoder_ex_backward"
    x, pooled, grad_pooled = _req(x, "x"), _req(pooled, "pooled"), _req(grad_pooled, "grad_pooled")
    route = _req(route, "route", torch.int32)
    b, n, npf, conv, csz, keep = _frozen_ex_args(x, conv_specs, sizes, act_input, what)
    if grad_tap is None:
        tap = -1
    else:
        grad_tap = _req(grad_tap, "grad_tap")
        if tap < 0 or tuple(grad_tap.shape) != (b, n, conv[tap].c_out):
            raise ValueError("%s: grad_tap must be (batch, points, channels of layer %d)" % (what, tap))
    nconv = len(conv_specs)
    dev = x.device
    with torch.cuda.device(dev):
        gx = torch.empty_like(x)
        zp = (ctypes.c_void_p * (nconv - 1))(*[z.data_ptr() for z in zsave])
        wsb = int(lib().snb200_frozen_encoder_ex_backward_workspace_bytes(b, n, int(bool(act_input)), nconv, conv, npf, int(tap)))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_ex_backward(b, n, int(bool(act_input)), _p(x), nconv, conv, npf, csz, _p(pooled), _p(route), zp, int(tap),
                                                      _p(grad_tap), _p(grad_pooled), _p(gx), _p(ws), wsb, _stream()), what)
    del keep
    return gx


class FrozenEncoderExFunction(torch.autograd.Function):
    """(x, conv_specs, sizes, act_input, tap) -> (pooled (P, B, C), route (P, B, C) int32[, h (B, N, c_tap) with tap >= 0]): the frozen encoder
    from the cloud or an activation, with a tapped hidden activation.  Differentiable in x through pooled and h (the parameters are frozen)."""

    @staticmethod
    def forward(ctx, x, conv_specs, sizes, act_input=False, tap=-1):
        x = x.contiguous()
        pooled, route, h, zs = frozen_encoder_ex_forward(x, conv_specs, sizes, act_input, tap, keep_activations=ctx.needs_input_grad[0])
        ctx.conv_specs, ctx.sizes, ctx.act_input, ctx.tap = conv_specs, [int(s) for s in sizes], act_input, tap
        ctx.save_for_backward(x, pooled, route, *(zs or []))
        ctx.mark_non_differentiable(route)
        return (pooled, route) if h is None else (pooled, route, h)

    @staticmethod
    def backward(ctx, g, g_route, *g_h):
        x, pooled, route, *zs = ctx.saved_tensors
        gh = g_h[0] if g_h else None
        if g is None and gh is None:
            return None, None, None, None, None
        g = torch.zeros_like(pooled) if g is None else g.contiguous()
        gx = frozen_encoder_ex_backward(x, ctx.conv_specs, ctx.sizes, pooled, route, zs, g, ctx.act_input, ctx.tap,
                                        None if gh is None else gh.contiguous())
        return gx, None, None, None, None


# ----------------------------------------------------------------------------------------------------- point transform
def _pt_args(x, T, what):
    x, T = _req(x, "x"), _req(T, "T")
    if x.dim() != 3 or T.dim() != 3 or T.shape[0] != x.shape[0] or T.shape[1] != x.shape[2] or T.shape[2] != x.shape[2]:
        raise ValueError("%s expects x (batch, points, k) and T (batch, k, k), got %s and %s" % (what, tuple(x.shape), tuple(T.shape)))
    b, n, k = x.shape
    if not point_transform_supported(b, n, k):
        raise ValueError("%s: outside the point transform's envelope (1..65535 clouds of 1..2^24 points, k <= 64), got %s" % (what, tuple(x.shape)))
    return x, T, b, n, k


def point_transform_supported(b, n, k):
    return bool(lib().snb200_point_transform_supported(int(b), int(n), int(k)))


def point_transform_forward(x, T):
    """out[b, i, :] = x[b, i, :] @ T[b] for x (B, N, K), T (B, K, K), K <= 64 (csrc/point_transform.cu)."""
    x, T, b, n, k = _pt_args(x, T, "point_transform_forward")
    with torch.cuda.device(x.device):
        out = torch.empty_like(x)
        check(lib().snb200_point_transform_forward(b, n, k, _p(x), _p(T), _p(out), _stream()), "point_transform_forward")
    return out


def point_transform_backward(x, T, grad_out):
    """(grad_x = grad_out @ T^T, grad_T = sum over points of x^T grad_out) of sum(grad_out * (x @ T)); bit-identical run to run."""
    x, T, b, n, k = _pt_args(x, T, "point_transform_backward")
    grad_out = _req(grad_out, "grad_out")
    if grad_out.shape != x.shape:
        raise ValueError("point_transform_backward: grad_out must have x's shape %s" % (tuple(x.shape),))
    dev = x.device
    with torch.cuda.device(dev):
        gx, gT = torch.empty_like(x), torch.empty_like(T)
        wsb = int(lib().snb200_point_transform_workspace_bytes(b, n, k))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_point_transform_backward(b, n, k, _p(x), _p(T), _p(grad_out), _p(gx), _p(gT), _p(ws), wsb, _stream()),
              "point_transform_backward")
    return gx, gT


class PointTransformFunction(torch.autograd.Function):
    """(x (B, N, K), T (B, K, K)) -> x @ T per cloud, differentiable in x and T."""

    @staticmethod
    def forward(ctx, x, T):
        x, T = x.contiguous(), T.contiguous()
        ctx.save_for_backward(x, T)
        return point_transform_forward(x, T)

    @staticmethod
    def backward(ctx, g):
        x, T = ctx.saved_tensors
        gx, gT = point_transform_backward(x, T, g.contiguous())
        return gx, gT


# ----------------------------------------------------------------------------------------------------- segments of a packed buffer
SEG_TILE = 128     # a segment starts on a 128-row tile of the frozen encoder's tensor-core layers; the rows up to the next one are padding


class Segments:
    """The prefixes x[b, :s] of B clouds, s in `sizes` (ascending), as the segments of one packed buffer: segment j = p * B + b is prefix p of
    cloud b, at rows [offset_j, offset_j + sizes[p]), each offset a multiple of SEG_TILE and the segments in order.  `table` (P*B, 2) int32 on
    the device is the C entries' segment table; `total` the packed rows, padding included."""

    def __init__(self, sizes, b, device):
        self.sizes, self.b = [int(s) for s in sizes], int(b)
        lengths = [s for s in self.sizes for _ in range(self.b)]
        padded = [-(-s // SEG_TILE) * SEG_TILE for s in lengths]
        offsets = [0]
        for p in padded[:-1]:
            offsets.append(offsets[-1] + p)
        self.offsets, self.lengths = offsets, lengths
        self.total, self.max_len, self.num = offsets[-1] + padded[-1], max(lengths), len(lengths)
        self.table = _device_constant([v for o, n in zip(offsets, lengths) for v in (o, n)], torch.int32, torch.device(device)).view(-1, 2)

    def rows(self):
        """Every segment row of the packed buffer in segment order (padding left out), as an index tensor on the table's device."""
        return torch.cat([torch.arange(o, o + n, device=self.table.device) for o, n in zip(self.offsets, self.lengths)])


def frozen_encoder_seg_supported(num_seg, total, max_len, conv_specs, act_input=False, tap=-1):
    conv, keep = make_layers(conv_specs)
    return bool(lib().snb200_frozen_encoder_seg_supported(int(num_seg), int(total), int(max_len), int(bool(act_input)), len(conv_specs), conv, int(tap)))


def _seg_input(x, conv, act_input, segs, what):
    c_in = conv[0].c_in if act_input else 3
    if not isinstance(x, torch.Tensor) or x.dim() != 2 or x.shape[0] != segs.total or x.shape[1] != c_in:
        raise ValueError("%s expects a packed (%d, %d) input" % (what, segs.total, c_in))


def frozen_encoder_seg_forward(x, conv_specs, segs, act_input=False, tap=-1, keep_activations=True):
    """The frozen encoder over the segments `segs` (a Segments) of a packed buffer x (total, 3 or c_in) (csrc/frozen_encoder.cu): one pool per
    segment.  Returns (pooled (num_seg, C), route (num_seg, C) int32: the row within the segment, the tapped activation (total, c_tap) or None,
    zsave or None)."""
    what = "frozen_encoder_seg_forward"
    x = _req(x, "x")
    conv, keep = make_layers(conv_specs)
    _seg_input(x, conv, act_input, segs, what)
    nconv, dev, ai = len(conv_specs), x.device, int(bool(act_input))
    with torch.cuda.device(dev):
        c = conv[nconv - 1].c_out
        pooled = torch.empty(segs.num, c, device=dev)
        route = torch.empty(segs.num, c, device=dev, dtype=torch.int32)
        h = torch.empty(segs.total, conv[tap].c_out, device=dev) if tap >= 0 else None
        zs = [torch.empty(segs.total, conv[l].c_out, device=dev) for l in range(nconv - 1)] if keep_activations else None
        zp = (ctypes.c_void_p * (nconv - 1))(*[z.data_ptr() for z in zs]) if keep_activations else None
        wsb = int(lib().snb200_frozen_encoder_seg_workspace_bytes(segs.num, segs.total, segs.max_len, ai, nconv, conv, int(tap), int(keep_activations)))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_seg_forward(segs.num, segs.total, segs.max_len, _p(segs.table), ai, _p(x), nconv, conv, _p(pooled), _p(route),
                                                      int(tap), _p(h), zp, _p(ws), wsb, _stream()), what)
    del keep
    return pooled, route, h, zs


def frozen_encoder_seg_backward(x, conv_specs, segs, pooled, route, zsave, grad_pooled, act_input=False, tap=-1, grad_tap=None):
    """Gradient with respect to the packed x of sum(grad_pooled * pooled) + sum(grad_tap * tapped activation); rows outside every segment
    get 0.  grad_tap=None: no gradient reached the tapped activation."""
    what = "frozen_encoder_seg_backward"
    x, pooled, grad_pooled = _req(x, "x"), _req(pooled, "pooled"), _req(grad_pooled, "grad_pooled")
    route = _req(route, "route", torch.int32)
    conv, keep = make_layers(conv_specs)
    _seg_input(x, conv, act_input, segs, what)
    if grad_tap is None:
        tap = -1
    else:
        grad_tap = _req(grad_tap, "grad_tap")
        if tap < 0 or tuple(grad_tap.shape) != (segs.total, conv[tap].c_out):
            raise ValueError("%s: grad_tap must be (total rows, channels of layer %d)" % (what, tap))
    nconv, dev, ai = len(conv_specs), x.device, int(bool(act_input))
    with torch.cuda.device(dev):
        gx = torch.empty_like(x)
        zp = (ctypes.c_void_p * (nconv - 1))(*[z.data_ptr() for z in zsave])
        wsb = int(lib().snb200_frozen_encoder_seg_backward_workspace_bytes(segs.num, segs.total, segs.max_len, ai, nconv, conv, int(tap)))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_frozen_encoder_seg_backward(segs.num, segs.total, segs.max_len, _p(segs.table), ai, _p(x), nconv, conv, _p(pooled), _p(route),
                                                       zp, int(tap), _p(grad_tap), _p(grad_pooled), _p(gx), _p(ws), wsb, _stream()), what)
    del keep
    return gx


class FrozenEncoderSegFunction(torch.autograd.Function):
    """(x packed (total, 3 or c_in), conv_specs, segs, act_input, tap) -> (pooled (num_seg, C), route (num_seg, C) int32[, h (total, c_tap) with
    tap >= 0]): the frozen encoder over the segments of a packed buffer.  Differentiable in x through pooled and h."""

    @staticmethod
    def forward(ctx, x, conv_specs, segs, act_input=False, tap=-1):
        x = x.contiguous()
        pooled, route, h, zs = frozen_encoder_seg_forward(x, conv_specs, segs, act_input, tap, keep_activations=ctx.needs_input_grad[0])
        ctx.conv_specs, ctx.segs, ctx.act_input, ctx.tap = conv_specs, segs, act_input, tap
        ctx.save_for_backward(x, pooled, route, *(zs or []))
        ctx.mark_non_differentiable(route)
        return (pooled, route) if h is None else (pooled, route, h)

    @staticmethod
    def backward(ctx, g, g_route, *g_h):
        x, pooled, route, *zs = ctx.saved_tensors
        gh = g_h[0] if g_h else None
        if g is None and gh is None:
            return None, None, None, None, None
        g = torch.zeros_like(pooled) if g is None else g.contiguous()
        gx = frozen_encoder_seg_backward(x, ctx.conv_specs, ctx.segs, pooled, route, zs, g, ctx.act_input, ctx.tap,
                                         None if gh is None else gh.contiguous())
        return gx, None, None, None, None


def point_transform_seg_supported(num_seg, total, max_len, k):
    return bool(lib().snb200_point_transform_seg_supported(int(num_seg), int(total), int(max_len), int(k)))


def _pt_seg_args(x, T, segs, prefix, what):
    x, T = _req(x, "x"), _req(T, "T")
    k = x.shape[-1]
    if prefix:
        ok = x.dim() == 3 and x.shape[0] == segs.b and x.shape[1] >= segs.max_len
        src_b, src_n, np_, sizes = x.shape[0], x.shape[1], len(segs.sizes), segs.sizes
    else:
        ok = x.dim() == 2 and x.shape[0] == segs.total
        src_b, src_n, np_, sizes = 0, 0, 0, []
    if not ok or tuple(T.shape) != (segs.num, k, k):
        raise ValueError("%s expects x %s and T (%d, k, k), got %s and %s" % (what, "(B, N >= max(sizes), k)" if prefix else "(total, k) packed",
                                                                              segs.num, tuple(x.shape), tuple(T.shape)))
    csz = (ctypes.c_int * max(np_, 1))(*sizes)
    return x, T, k, src_b, src_n, np_, csz


def point_transform_seg_forward(x, T, segs, prefix):
    """Segment j of the packed output (segs.total, k) is its rows times T[j] (T (num_seg, k, k)), padding rows 0 (csrc/point_transform.cu).
    prefix=True: x is the unpacked (B, N, k) input and segment p * B + b reads x[b, :sizes[p]]; prefix=False: x is packed as the output."""
    what = "point_transform_seg_forward"
    x, T, k, src_b, src_n, np_, csz = _pt_seg_args(x, T, segs, prefix, what)
    with torch.cuda.device(x.device):
        out = torch.empty(segs.total, k, device=x.device)
        check(lib().snb200_point_transform_seg_forward(segs.num, segs.total, segs.max_len, _p(segs.table), k, src_b, src_n, np_, csz, _p(x), _p(T),
                                                       _p(out), _stream()), what)
    return out


def point_transform_seg_backward(x, T, segs, prefix, grad_out):
    """(grad_x shaped as x, grad_T (num_seg, k, k)) of sum(grad_out * point_transform_seg_forward(x, T, segs, prefix)); with prefix=True
    grad_x[b, i] sums the prefixes holding point i in ascending order.  Bit-identical run to run."""
    what = "point_transform_seg_backward"
    x, T, k, src_b, src_n, np_, csz = _pt_seg_args(x, T, segs, prefix, what)
    grad_out = _req(grad_out, "grad_out")
    if tuple(grad_out.shape) != (segs.total, k):
        raise ValueError("%s: grad_out must be (%d, %d)" % (what, segs.total, k))
    dev = x.device
    with torch.cuda.device(dev):
        gx, gT = torch.empty_like(x), torch.empty_like(T)
        wsb = int(lib().snb200_point_transform_seg_workspace_bytes(segs.num, segs.total, segs.max_len, k))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_point_transform_seg_backward(segs.num, segs.total, segs.max_len, _p(segs.table), k, src_b, src_n, np_, csz, _p(x), _p(T),
                                                        _p(grad_out), _p(gx), _p(gT), _p(ws), wsb, _stream()), what)
    return gx, gT


class PointTransformSegFunction(torch.autograd.Function):
    """(x, T (num_seg, k, k), segs, prefix) -> packed (segs.total, k): each segment's rows times its own T, differentiable in x and T."""

    @staticmethod
    def forward(ctx, x, T, segs, prefix):
        x, T = x.contiguous(), T.contiguous()
        ctx.save_for_backward(x, T)
        ctx.segs, ctx.prefix = segs, prefix
        return point_transform_seg_forward(x, T, segs, prefix)

    @staticmethod
    def backward(ctx, g):
        x, T = ctx.saved_tensors
        gx, gT = point_transform_seg_backward(x, T, ctx.segs, ctx.prefix, g.contiguous())
        return gx, gT, None, None


# ----------------------------------------------------------------------------------------------------- registration pose loss
POSE_TERMS = ("chamfer_loss", "qnorm_loss", "norm_err", "rot_err", "trans_err")


def _pose_args(y, p0, p1, igt, what):
    y, p0, p1, igt = _req(y, "y"), _req(p0, "p0"), _req(p1, "p1"), _req(igt, "igt")
    if (p0.dim() != 3 or p0.shape[2] != 3 or p1.dim() != 3 or p1.shape[2] != 3 or p1.shape[0] != p0.shape[0] or tuple(y.shape) != (p0.shape[0], 7)
            or igt.shape != y.shape):
        raise ValueError("%s expects y and igt (batch, 7) and p0, p1 (batch, points, 3) of one batch, got %s, %s, %s, %s"
                         % (what, tuple(y.shape), tuple(igt.shape), tuple(p0.shape), tuple(p1.shape)))
    b, m0, m1 = p0.shape[0], p0.shape[1], p1.shape[1]
    if not pose_loss_supported(b, m0, m1):
        raise ValueError("%s: 1..256 pairs of clouds of 1..1024 points expected, got %d pairs of %d and %d" % (what, b, m0, m1))
    return y, p0, p1, igt, b, m0, m1


def pose_loss_supported(b, m0, m1=None):
    """Whether b pairs of a template of m0 points and a source of m1 (default m0) are inside the pose loss's envelope."""
    m1 = m0 if m1 is None else m1
    return 1 <= b <= 256 and 1 <= m0 <= 1024 and 1 <= m1 <= 1024


def pose_loss_forward(y, p0, p1, igt):
    """One launch (csrc/pose_loss.cu): twist (B, 7), the Chamfer arg-mins idx01 (B, M1) / idx10 (B, M0) int32 and terms (5,) = POSE_TERMS
    (rot_err in radians) of the raw PCRNet output y (B, 7), the template p0 (B, M0, 3), the source p1 (B, M1, 3) and the ground truth
    igt (B, 7).  M0 and M1 may differ (one sampled cloud against a full one); each Chamfer mean is over its own cloud."""
    y, p0, p1, igt, b, m0, m1 = _pose_args(y, p0, p1, igt, "pose_loss_forward")
    dev = y.device
    with torch.cuda.device(dev):
        twist = torch.empty(b, 7, device=dev)
        idx01 = torch.empty(b, m1, device=dev, dtype=torch.int32); idx10 = torch.empty(b, m0, device=dev, dtype=torch.int32)
        terms = torch.empty(5, device=dev)
        wsb = int(lib().snb200_pose_loss_ex_workspace_bytes(b, m0, m1))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_pose_loss_ex_forward(b, m0, m1, _p(y), _p(p0), _p(p1), _p(igt), _p(twist), _p(idx01), _p(idx10), _p(terms), _p(ws), wsb,
                                                _p(_ticket(dev)), _stream()), "pose_loss_forward")
    return twist, idx01, idx10, terms


def pose_loss_backward(y, p0, p1, igt, idx01, idx10, grad_terms):
    """(grad_y (B, 7), grad_p0 (B, M0, 3), grad_p1 (B, M1, 3)) of sum(grad_terms * terms); rot_err's entry is ignored (it is reported, not
    trained on)."""
    y, p0, p1, igt, b, m0, m1 = _pose_args(y, p0, p1, igt, "pose_loss_backward")
    idx01, idx10, grad_terms = _req(idx01, "idx01", torch.int32), _req(idx10, "idx10", torch.int32), _req(grad_terms, "grad_terms")
    if tuple(idx01.shape) != (b, m1) or tuple(idx10.shape) != (b, m0) or grad_terms.numel() != 5:
        raise ValueError("pose_loss_backward expects idx01 (batch, source points), idx10 (batch, template points) and 5 grad_terms")
    dev = y.device
    with torch.cuda.device(dev):
        gy, g0, g1 = torch.empty_like(y), torch.empty_like(p0), torch.empty_like(p1)
        check(lib().snb200_pose_loss_ex_backward(b, m0, m1, _p(y), _p(p0), _p(p1), _p(igt), _p(idx01), _p(idx10), _p(grad_terms), _p(gy), _p(g0),
                                                 _p(g1), _stream()), "pose_loss_backward")
    return gy, g0, g1


class PoseLossFunction(torch.autograd.Function):
    """(y, p0, p1, igt) -> (terms (5,) = POSE_TERMS, twist (B, 7)).  Differentiable in y, p0 and p1 through every term but rot_err; twist is
    not differentiable (it is the reported estimate).  p0 and p1 may hold different numbers of points."""

    @staticmethod
    def forward(ctx, y, p0, p1, igt):
        y, p0, p1, igt = y.contiguous(), p0.contiguous(), p1.contiguous(), igt.contiguous()
        twist, idx01, idx10, terms = pose_loss_forward(y, p0, p1, igt)
        ctx.save_for_backward(y, p0, p1, igt, idx01, idx10)
        ctx.mark_non_differentiable(twist)
        return terms, twist

    @staticmethod
    def backward(ctx, g_terms, g_twist):
        y, p0, p1, igt, idx01, idx10 = ctx.saved_tensors
        gy, g0, g1 = pose_loss_backward(y, p0, p1, igt, idx01, idx10, g_terms.contiguous())
        return gy, g0, g1, None


POSE_EVAL_COLUMNS = POSE_TERMS + ("consistency",)


def pose_eval_supported(b, m, ms=None, m1=None, ms1=None):
    """Whether pose_eval takes b pairs of a template of m points and a source of m1 (default m) and, when ms is given, a sampled pair of ms
    and ms1 (default ms) points."""
    return pose_loss_supported(b, m, m1) and (ms is None or pose_loss_supported(b, ms, ms1))


def pose_eval(y, p0, p1, igt, p0s=None, p1s=None):
    """One launch (csrc/pose_loss.cu), forward only: (per_pair (B, 6) = POSE_EVAL_COLUMNS of every pair, twist (B, 7)).  Columns 0-4 are
    pose_loss_forward's terms of that pair alone (rot_err in radians), so their mean over the pairs is its `terms` up to the rounding of
    that mean; `consistency` is compute_sampling_consistency (registration/main.py:540-553) of the sampled pair p0s (B, Ms0, 3), p1s
    (B, Ms1, 3), which may be p0, p1 themselves, and 0 when they are not given.  p0 (B, M0, 3) and p1 (B, M1, 3) may differ in size, and so
    may p0s and p1s.  1..256 pairs of clouds of 1..1024 points.  No gradient."""
    y, p0, p1, igt, b, m0, m1 = _pose_args(y, p0, p1, igt, "pose_eval")
    if (p0s is None) != (p1s is None):
        raise ValueError("pose_eval: the sampled pair needs both p0s and p1s")
    ms0 = ms1 = 0
    if p0s is not None:
        p0s, p1s = _req(p0s, "p0s"), _req(p1s, "p1s")
        if p0s.dim() != 3 or p0s.shape[2] != 3 or p0s.shape[0] != b or p1s.dim() != 3 or p1s.shape[2] != 3 or p1s.shape[0] != b:
            raise ValueError("pose_eval expects p0s, p1s (batch, points, 3) with the batch of p0, got %s, %s" % (tuple(p0s.shape), tuple(p1s.shape)))
        ms0, ms1 = p0s.shape[1], p1s.shape[1]
        if not pose_loss_supported(b, ms0, ms1):
            raise ValueError("pose_eval: 1..1024 sampled points expected, got %d and %d" % (ms0, ms1))
    _no_grad_inputs("pose_eval", y, p0, p1, igt, p0s, p1s)
    dev = y.device
    if any(t is not None and t.device != dev for t in (p0, p1, igt, p0s, p1s)):
        raise ValueError("pose_eval: the inputs are on different devices")
    with torch.cuda.device(dev):
        per_pair, twist = torch.empty(b, 6, device=dev), torch.empty(b, 7, device=dev)
        check(lib().snb200_pose_eval_ex(b, m0, m1, _p(y), _p(p0), _p(p1), _p(igt), ms0, ms1, _p(p0s), _p(p1s), _p(per_pair), _p(twist), _stream()),
              "pose_eval")
    return per_pair, twist


# ----------------------------------------------------------------------------------------------------- EMD
def _emd_clouds(what, xyz1, xyz2):
    """(b, n, m) of two BNC clouds with equal batch sizes; ValueError before any launch otherwise."""
    if xyz1.dim() != 3 or xyz2.dim() != 3 or xyz1.shape[2] != 3 or xyz2.shape[2] != 3 or xyz1.shape[0] != xyz2.shape[0]:
        raise ValueError("%s expects (batch_size,num_points,3) xyz1 and xyz2 with equal batch sizes" % what)
    return xyz1.shape[0], xyz1.shape[1], xyz2.shape[1]


def _emd_match(match, b, n, m):
    if tuple(match.shape) != (b, m, n):
        raise ValueError("MatchCost expects (batch_size,#query,#dataset) match shape, got %s" % (tuple(match.shape),))


def emd_exact_mode():
    """True when SNB200_EMD_EXACT_EXP=1 in the environment selects approx_match's parity kernel by default."""
    return os.environ.get("SNB200_EMD_EXACT_EXP", "0") == "1"


def approx_match(xyz1, xyz2, exact=None):
    """exact=True (or SNB200_EMD_EXACT_EXP=1 in the environment): the parity kernel -- exact exponential, index-order float sums, the
    reference's level order; bit-identical to the CPU oracle.  Default: the fast kernel (ex2.approx, blocked sums)."""
    if exact is None:
        exact = emd_exact_mode()
    xyz1, xyz2 = _req(xyz1, "xyz1"), _req(xyz2, "xyz2")
    b, n, m = _emd_clouds("ApproxMatch", xyz1, xyz2)
    dev = xyz1.device
    with torch.cuda.device(dev):
        match = torch.empty(b, m, n, device=dev)
        wsb = int(lib().snb200_approxmatch_workspace_bytes(b, n, m))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_approxmatch_mode(b, n, m, _p(xyz1), _p(xyz2), _p(match), _lib.EMD_EXACT if exact else 0, _p(ws), wsb, _stream()), "approxmatch")
    return match


def match_cost_forward(xyz1, xyz2, match):
    xyz1, xyz2, match = _req(xyz1, "xyz1"), _req(xyz2, "xyz2"), _req(match, "match")
    b, n, m = _emd_clouds("MatchCost", xyz1, xyz2)
    _emd_match(match, b, n, m)
    dev = xyz1.device
    with torch.cuda.device(dev):
        cost = torch.empty(b, device=dev)
        wsb = int(lib().snb200_matchcost_workspace_bytes(b))
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_matchcost(b, n, m, _p(xyz1), _p(xyz2), _p(match), _p(cost), _p(ws), wsb, _stream()), "matchcost")
    return cost


def match_cost_grad(xyz1, xyz2, match):
    xyz1, xyz2, match = _req(xyz1, "xyz1"), _req(xyz2, "xyz2"), _req(match, "match")
    b, n, m = _emd_clouds("MatchCost", xyz1, xyz2)
    _emd_match(match, b, n, m)
    with torch.cuda.device(xyz1.device):
        g1 = torch.empty_like(xyz1); g2 = torch.empty_like(xyz2)
        check(lib().snb200_matchcostgrad(b, n, m, _p(xyz1), _p(xyz2), _p(match), _p(g1), _p(g2), _stream()), "matchcostgrad")
    return g1, g2


class MatchCostFunction(torch.autograd.Function):
    """tf_approxmatch.py:35-64: cost (B,), gradients to xyz1 and xyz2 only, scaled by grad_cost[b]."""

    @staticmethod
    def forward(ctx, xyz1, xyz2, match):
        ctx.save_for_backward(xyz1.contiguous(), xyz2.contiguous(), match.contiguous())
        return match_cost_forward(xyz1, xyz2, match)

    @staticmethod
    def backward(ctx, g):
        xyz1, xyz2, match = ctx.saved_tensors
        g1, g2 = match_cost_grad(xyz1, xyz2, match)
        return g1 * g.view(-1, 1, 1), g2 * g.view(-1, 1, 1), None


def _emd_per_cloud_args(xyz1, xyz2):
    """(b, n, m, b2) of xyz1 (B, n, 3) against xyz2 (B2, m, 3) with B2 dividing B; ValueError before any launch otherwise."""
    if xyz1.dim() != 3 or xyz2.dim() != 3 or xyz1.shape[2] != 3 or xyz2.shape[2] != 3:
        raise ValueError("emd_per_cloud expects (batch, points, 3) tensors, got %s and %s" % (tuple(xyz1.shape), tuple(xyz2.shape)))
    b, n, _ = xyz1.shape
    b2, m, _ = xyz2.shape
    if xyz2.device != xyz1.device:
        raise ValueError("emd_per_cloud: xyz1 is on %s and xyz2 on %s" % (xyz1.device, xyz2.device))
    if b2 < 1 or b % b2 != 0 or n < 1 or m < 1:
        raise ValueError("emd_per_cloud: xyz2's %d clouds must divide xyz1's %d, and no cloud may be empty" % (b2, b))
    return b, n, m, b2


def emd_per_cloud_forward(xyz1, xyz2):
    """(cost (B,), workspace): the per-cloud EMD of csrc/emd.cu and the workspace holding the ratios its backward rebuilds the match from."""
    xyz1, xyz2 = _req(xyz1, "xyz1"), _req(xyz2, "xyz2")
    b, n, m, b2 = _emd_per_cloud_args(xyz1, xyz2)
    dev = xyz1.device
    with torch.cuda.device(dev):
        cost = torch.empty(b, device=dev)
        wsb = int(lib().snb200_emd_per_cloud_workspace_bytes(b, n, m)) if b else 0
        ws = torch.empty(max(wsb, 4), device=dev, dtype=torch.uint8)
        check(lib().snb200_emd_per_cloud(b, n, _p(xyz1), m, _p(xyz2), b2, _p(cost), _p(ws), wsb, _stream()), "emd_per_cloud")
    return cost, ws


def emd_per_cloud_supported(xyz1, xyz2):
    """Whether emd_per_cloud takes these clouds: (B, n, 3) and (B2, m, 3) with B2 dividing B, B <= 65535, n <= 2^24, m <= 65520.  Outside,
    callers keep the match-tensor composition (and its errors)."""
    if xyz1.dim() != 3 or xyz2.dim() != 3 or xyz1.shape[2] != 3 or xyz2.shape[2] != 3 or xyz2.shape[0] < 1 or xyz1.shape[0] % xyz2.shape[0]:
        return False
    return bool(lib().snb200_emd_per_cloud_supported(xyz1.shape[0], xyz1.shape[1], xyz2.shape[1]))


def emd_per_cloud_backward(xyz1, xyz2, grad_cost, ws, need1=True, need2=True):
    """(grad1 (B, n, 3), grad2 (B, m, 3) per pair) for the workspace emd_per_cloud_forward returned; a gradient not needed is None and
    its pass does not run."""
    xyz1, xyz2, grad_cost = _req(xyz1, "xyz1"), _req(xyz2, "xyz2"), _req(grad_cost, "grad_cost")
    b, n, m, b2 = _emd_per_cloud_args(xyz1, xyz2)
    if tuple(grad_cost.shape) != (b,):
        raise ValueError("emd_per_cloud_backward: grad_cost must have shape (%d,), got %s" % (b, tuple(grad_cost.shape)))
    dev = xyz1.device
    with torch.cuda.device(dev):
        g1 = torch.empty(b, n, 3, device=dev) if need1 else None
        g2 = torch.empty(b, m, 3, device=dev) if need2 else None
        if not (need1 or need2):
            return g1, g2
        check(lib().snb200_emd_per_cloud_backward(b, n, _p(xyz1), m, _p(xyz2), b2, _p(grad_cost), _p(g1), _p(g2), _p(ws), ws.numel(), _stream()),
              "emd_per_cloud_backward")
    return g1, g2


def emd_per_cloud(xyz1, xyz2):
    """Per-cloud EMD, (B,): match_cost(xyz1, xyz2, approx_match(xyz1, xyz2)) bit for bit (the fast mode), without the (B, m, n) match
    tensor.  xyz1 (B, n, 3), xyz2 (B2, m, 3) with B2 dividing B: cloud b of xyz1 is matched with cloud b % B2 of xyz2 (B2 < B: the
    stacked prefixes' reconstructions against the one input batch, without repeat()).  Run to run bit-identical.  No gradient: see
    EMDCostFunction."""
    _no_grad_inputs("emd_per_cloud", xyz1, xyz2)
    return emd_per_cloud_forward(xyz1, xyz2)[0]


class EMDCostFunction(torch.autograd.Function):
    """The per-cloud EMD with gradients: EMDCostFunction.apply(xyz1, xyz2) is MatchCostFunction.apply(xyz1, xyz2, approx_match(xyz1, xyz2))
    bit for bit, cost and both gradients (the match counts as a constant, as approx_match has no gradient), without the match tensor.
    The forward keeps its workspace (the per-level ratios, 44 * B * (n + m) bytes) for the backward.  With B2 < B clouds in xyz2 the
    per-pair gradients to xyz2 are summed over the repeats.  The pass of a gradient no input needs does not run (the target cloud of a
    loss usually needs none)."""

    @staticmethod
    def forward(ctx, xyz1, xyz2):
        cost, ws = emd_per_cloud_forward(xyz1, xyz2)
        ctx.save_for_backward(xyz1.contiguous(), xyz2.contiguous(), ws)
        return cost

    @staticmethod
    def backward(ctx, g):
        xyz1, xyz2, ws = ctx.saved_tensors
        g1, g2 = emd_per_cloud_backward(xyz1, xyz2, g.contiguous(), ws, ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        if g2 is not None and xyz2.shape[0] != xyz1.shape[0]:
            g2 = g2.view(-1, *xyz2.shape).sum(dim=0)
        return g1, g2


# ----------------------------------------------------------------------------------------------------- inference matching
def nn_matching(full_pc, nn_idx, k, complete_fps=True, return_idx=False):
    """GPU twin of sputils.nn_matching: full_pc (B,N,3), nn_idx (B,T) int32 -> (B,k,3)."""
    full_pc, nn_idx = _req(full_pc, "full_pc"), _req(nn_idx, "idx", torch.int32)
    b, n, _ = full_pc.shape
    t = nn_idx.shape[1]
    with torch.cuda.device(full_pc.device):
        out = torch.empty(b, k, 3, device=full_pc.device)
        oi = torch.empty(b, k, device=full_pc.device, dtype=torch.int32) if return_idx else None
        check(lib().snb200_nn_matching(b, n, t, int(k), _p(full_pc), _p(nn_idx), int(bool(complete_fps)), _p(out), _p(oi), _stream()),
              "nn_matching")
    return (out, oi) if return_idx else out


# ----------------------------------------------------------------------------------------------------- farthest point sampling
def farthest_point_sample(inp, m, layout="bnc", return_points=False, _threads=0):
    """Farthest point sampling of m points per cloud: inp (B,N,3) for layout "bnc" or (B,3,N) for "bcn" -> idx (B,m) int32, and with
    return_points=True also the selected points (B,m,3) / (B,3,m) in the same layout, written by the same launch.
    The indices are those of tf_sampling's farthestpointsamplingKernel (see include/samplenet_b200.h).  1 <= N <= 16384, m >= 1
    (m > N repeats index 0).  No gradient."""
    lay = _layout(layout)
    if not isinstance(inp, torch.Tensor) or inp.dim() != 3 or inp.shape[2 if lay == BNC else 1] != 3:
        raise ValueError("farthest_point_sample expects (batch, points, 3) for 'bnc' or (batch, 3, points) for 'bcn', got %s"
                         % (tuple(inp.shape) if isinstance(inp, torch.Tensor) else type(inp).__name__,))
    if isinstance(m, bool) or int(m) != m or m < 1:
        raise ValueError("farthest_point_sample: the number of samples must be a positive integer, got %r" % (m,))
    m = int(m)
    b = inp.shape[0]
    n = inp.shape[1 if lay == BNC else 2]
    if n < 1:
        raise ValueError("farthest_point_sample: empty clouds")
    inp = _req(inp, "inp")
    with torch.cuda.device(inp.device):
        idx = torch.empty(b, m, device=inp.device, dtype=torch.int32)
        pts = torch.empty((b, m, 3) if lay == BNC else (b, 3, m), device=inp.device) if return_points else None
        check(lib().snb200_debug_farthest_point_sample(b, n, m, lay, _p(inp), _p(idx), _p(pts), int(_threads), _stream()) if _threads else
              lib().snb200_farthest_point_sample(b, n, m, lay, _p(inp), _p(idx), _p(pts), _stream()), "farthest_point_sample")
    return (idx, pts) if return_points else idx


def gather_point(inp, idx, layout="bnc"):
    """tf_sampling.gather_point / pointnet2 gather_operation: inp (B,N,C) "bnc" or (B,C,N) "bcn", idx (B,m) -> (B,m,C) / (B,C,m);
    differentiable in inp (deterministic scatter-add: the group_point kernels with one neighbour)."""
    if not isinstance(idx, torch.Tensor) or idx.dim() != 2:
        raise ValueError("gather_point expects idx of shape (batch, m)")
    if not isinstance(inp, torch.Tensor) or inp.dim() != 3 or inp.shape[0] != idx.shape[0]:
        raise ValueError("gather_point expects inp of shape (batch, points, channels) with the batch of idx")
    out = GroupPointFunction.apply(inp, idx.to(torch.int32)[..., None], layout)
    return out[:, :, :, 0] if layout == "bcn" else out[:, :, 0, :]


# ----------------------------------------------------------------------------------------------------- augmentation
def _aug_shape(points, what):
    if not isinstance(points, torch.Tensor) or points.dim() != 3 or points.shape[2] != 3 or points.shape[1] < 1:
        raise ValueError("%s expects points of shape (batch, points >= 1, 3), got %s"
                         % (what, tuple(points.shape) if isinstance(points, torch.Tensor) else type(points).__name__))
    if points.shape[1] > 1 << 24:
        raise ValueError("%s: clouds of at most 2^24 points, got %d" % (what, points.shape[1]))
    return points.shape


def rotate_jitter(points, sigma=0.01, clip=0.05, key=None):
    """classification/train_classifier.py:217-221 (provider.rotate_point_cloud, then provider.jitter_point_cloud) in one launch: each cloud of
    points (B, N, 3) rotated about y by its own angle drawn uniformly in [0, 2 pi), then every coordinate moved by clip(sigma * normal, -clip,
    clip) (sigma = 0: no jitter).  Returns a new (B, N, 3) tensor.  The random numbers come from Philox4x32-10 under a key of two 64-bit words
    (include/samplenet_b200.h, snb200_rotate_jitter); key=None draws the key on the device from torch's default CUDA generator, one draw per
    call and no host read, so torch.manual_seed repeats the result and the call can be captured in a CUDA graph.  key: an int64 tensor of 2
    words on the points' device.  No gradient."""
    b, n, _ = _aug_shape(points, "rotate_jitter")
    sigma, clip = float(sigma), float(clip)
    if not sigma >= 0.0 or (sigma > 0.0 and not clip > 0.0):
        raise ValueError("rotate_jitter: sigma must be >= 0 and clip > 0 (sigma=%r clip=%r)" % (sigma, clip))
    points = _req(points, "points")
    with torch.cuda.device(points.device):
        if key is None:
            key = torch.empty(2, dtype=torch.int64, device=points.device).random_()
        elif not isinstance(key, torch.Tensor) or key.dtype != torch.int64 or key.numel() != 2 or key.device != points.device:
            raise ValueError("rotate_jitter: key must be an int64 tensor of 2 words on %s" % (points.device,))
        key = key.contiguous()
        out = torch.empty_like(points)
        check(lib().snb200_rotate_jitter(b, n, 1, _p(points), _p(out), None, _p(key), sigma, clip, _stream()), "rotate_jitter")
    return out


def rotate_by_angles(points, angles):
    """provider.rotate_point_cloud_by_angle for every angle at once (the votes of evaluate_classifier.py:163-167): points (B, N, 3) and a host
    sequence of V float64 angles -> (V, B, N, 3), replica v rotated about y by angles[v].  One launch.  No gradient."""
    b, n, _ = _aug_shape(points, "rotate_by_angles")
    angles = [float(a) for a in angles]
    if not angles:
        raise ValueError("rotate_by_angles: at least one angle")
    points = _req(points, "points")
    with torch.cuda.device(points.device):
        ang = torch.tensor(angles, dtype=torch.float64).to(points.device)
        out = torch.empty((len(angles), b, n, 3), dtype=torch.float32, device=points.device)
        check(lib().snb200_rotate_jitter(b, n, len(angles), _p(points), _p(out), _p(ang), None, 0.0, 0.0, _stream()), "rotate_by_angles")
    return out


def ae_augment(points, mu=None, sigma=None, z_rotate=False, out=None, key=None):
    """general_utils.apply_augmentations (reconstruction/src/general_utils.py:100-117) in one launch: with sigma given, every coordinate of
    points (B, N, 3) plus a normal draw of mean mu (None: 0) and standard deviation sigma, in float64 and rounded to float32 (mu without
    sigma is a ValueError, as the reference reads mu only with gauss_augment's sigma); then, with
    z_rotate, the whole batch times ONE matrix, rand_rotation_matrix() with its third row and column set to (0, 0, 1) (not orthogonal in
    general, as in the reference).  Writes and returns `out` ((B, N, 3) float32, contiguous, on the points' device; None: a new tensor;
    `points` itself: in place).  The random numbers come from Philox4x32-10 under a key of two 64-bit words (include/samplenet_b200.h,
    snb200_ae_augment); key=None draws the key on the device from torch's default CUDA generator, one draw per call and no host read, so
    torch.manual_seed repeats the result and the call can be captured in a CUDA graph.  No gradient."""
    b, n, _ = _aug_shape(points, "ae_augment")
    gauss = sigma is not None
    if mu is not None and not gauss:
        raise ValueError("ae_augment: mu=%r without sigma (the noise is drawn only when sigma is given)" % (mu,))
    mu, sigma = float(0.0 if mu is None else mu), float(0.0 if sigma is None else sigma)
    if gauss and not (math.isfinite(mu) and math.isfinite(sigma) and sigma >= 0.0):
        raise ValueError("ae_augment: the noise needs finite mu and sigma >= 0 (mu=%r sigma=%r)" % (mu, sigma))
    if out is not None and (not isinstance(out, torch.Tensor) or out.shape != points.shape or out.dtype != torch.float32
                            or out.device != points.device or not out.is_contiguous()):
        raise ValueError("ae_augment: out must be a contiguous float32 tensor of the points' shape and device")
    points = _req(points, "points")
    with torch.cuda.device(points.device):
        if not (gauss or z_rotate):
            key = None
        elif key is None:
            key = torch.empty(2, dtype=torch.int64, device=points.device).random_()
        elif not isinstance(key, torch.Tensor) or key.dtype != torch.int64 or key.numel() != 2 or key.device != points.device:
            raise ValueError("ae_augment: key must be an int64 tensor of 2 words on %s" % (points.device,))
        else:
            key = key.contiguous()
        out = torch.empty_like(points) if out is None else out
        check(lib().snb200_ae_augment(b, n, _p(points), _p(out), _p(key), int(gauss), mu, sigma, int(bool(z_rotate)), _stream()), "ae_augment")
    return out


def registration_pairs(clouds, records, transforms, key=None, return_perm=False):
    """The registration trainer's pairs for a batch of records in one launch (ModelNetCls.__getitem__ + QuaternionFixedDataset.__getitem__,
    registration/data/modelnet_loader_torch.py:102-116, registration/src/qdataset.py:160-179): clouds (S, N, 3) float32 already on the unit
    cube, records (B,) int32 or int64 indices in [0, len(transforms)), transforms (R, 7) float32 rows (w, x, y, z, tx, ty, tz).  Record r
    takes cloud r % S and row r.  -> (p0 (B, N, 3), p1 (B, N, 3), vec (B, 7)) and, with return_perm, perm (B, N) int32: p0 is the cloud
    in a random point order, p1 = qrot(q_r, p0) in float32, vec the row.  The point order comes from Philox4x32-10 under a key of two
    64-bit words (include/samplenet_b200.h, snb200_registration_pairs); key=None draws the key on the device from torch's default CUDA
    generator, one draw per call and no host read, so torch.manual_seed repeats the batch and the call can be captured in a CUDA graph.
    The records are not range-checked on the host (that would read them back).  N <= 2048.  No gradient."""
    if not isinstance(clouds, torch.Tensor) or clouds.dim() != 3 or clouds.shape[2] != 3 or clouds.shape[0] < 1 or clouds.shape[1] < 1:
        raise ValueError("registration_pairs expects clouds of shape (clouds >= 1, points >= 1, 3), got %s"
                         % ((tuple(clouds.shape) if isinstance(clouds, torch.Tensor) else type(clouds).__name__),))
    if clouds.shape[1] > 2048:
        raise ValueError("registration_pairs: clouds of at most 2048 points, got %d" % clouds.shape[1])
    if not isinstance(records, torch.Tensor) or records.dim() != 1 or records.dtype not in (torch.int32, torch.int64):
        raise ValueError("registration_pairs expects records as a 1-d int32 or int64 tensor")
    if not isinstance(transforms, torch.Tensor) or transforms.dim() != 2 or transforms.shape[1] != 7 or transforms.shape[0] < 1:
        raise ValueError("registration_pairs expects transforms of shape (records >= 1, 7)")
    s, n, _ = clouds.shape
    b = records.shape[0]
    clouds, transforms = _req(clouds, "clouds"), _req(transforms, "transforms")
    records = _req(records, "records", records.dtype)
    dev = clouds.device
    if records.device != dev or transforms.device != dev:
        raise ValueError("registration_pairs: clouds, records and transforms must be on one device")
    with torch.cuda.device(dev):
        records = records.to(torch.int32).contiguous()
        if key is None:
            key = torch.empty(2, dtype=torch.int64, device=dev).random_()
        elif not isinstance(key, torch.Tensor) or key.dtype != torch.int64 or key.numel() != 2 or key.device != dev:
            raise ValueError("registration_pairs: key must be an int64 tensor of 2 words on %s" % (dev,))
        key = key.contiguous()
        p0 = torch.empty((b, n, 3), dtype=torch.float32, device=dev)
        p1 = torch.empty_like(p0)
        vec = torch.empty((b, 7), dtype=torch.float32, device=dev)
        perm = torch.empty((b, n), dtype=torch.int32, device=dev) if return_perm else None
        check(lib().snb200_registration_pairs(b, n, s, transforms.shape[0], _p(clouds), _p(records), _p(transforms), _p(key), _p(p0), _p(p1),
                                              _p(vec), _p(perm), _stream()), "registration_pairs")
    return (p0, p1, vec, perm) if return_perm else (p0, p1, vec)


# ----------------------------------------------------------------------------------------------------- shape retrieval
def retrieval_metrics(queries, query_labels, database=None, database_labels=None, recall_levels=11, exclude_diagonal=None):
    """Shape-retrieval metrics of descriptors (csrc/retrieval.cu; the contract is snb200_retrieval_metrics in include/samplenet_b200.h):
    queries (Q, D) float32 and query_labels (Q,) against database (M, D) and database_labels (M,), every query ranking the whole database by
    squared L2 distance, ties by index.  database=None ranks queries against themselves leaving each query's own row out (leave-one-out).
    exclude_diagonal=True with a database of as many rows leaves database row i out of query i's results (each query's own shape in another
    form); its default is database=None.
    -> {"ap" (Q,) float64, "precision" (Q, recall_levels) float64 (interpolated precision at recall l / (recall_levels - 1)),
    "num_relevant" (Q,) int32} on the device; a query without a relevant result has NaN ap and precision.  One launch; nothing is read back.
    Outside the kernel's envelope (Q <= 2^20, M <= 16384, D <= 1024, 2 <= recall_levels <= 101) it raises with the kernel's message."""
    if (database is None) != (database_labels is None):
        raise ValueError("retrieval_metrics: give database and database_labels together, or neither (leave-one-out)")
    exclude = database is None if exclude_diagonal is None else bool(exclude_diagonal)
    same = database is None
    if same:
        database, database_labels = queries, query_labels
    for name, t in (("queries", queries), ("database", database)):
        if not isinstance(t, torch.Tensor) or t.dim() != 2:
            raise ValueError("retrieval_metrics: %s must be a (rows, D) tensor" % name)
    if queries.shape[1] != database.shape[1]:
        raise ValueError("retrieval_metrics: queries have %d columns, the database %d" % (queries.shape[1], database.shape[1]))
    for name, t, rows in (("query_labels", query_labels, queries.shape[0]), ("database_labels", database_labels, database.shape[0])):
        if not isinstance(t, torch.Tensor) or t.numel() != rows or t.is_floating_point():
            raise ValueError("retrieval_metrics: %s must be an integer tensor of %d labels" % (name, rows))
    queries, database = _req(queries, "queries"), _req(database, "database")
    dev = queries.device
    if database.device != dev or query_labels.device != dev or database_labels.device != dev:
        raise ValueError("retrieval_metrics: descriptors and labels must be on one device")
    q, m, d, L = queries.shape[0], database.shape[0], queries.shape[1], int(recall_levels)
    with torch.cuda.device(dev):
        ql = query_labels.reshape(-1).to(torch.int32).contiguous()
        dl = ql if same else database_labels.reshape(-1).to(torch.int32).contiguous()
        ap = torch.empty(q, dtype=torch.float64, device=dev)
        prec = torch.empty(q, max(L, 1), dtype=torch.float64, device=dev)
        nrel = torch.empty(q, dtype=torch.int32, device=dev)
        check(lib().snb200_retrieval_metrics(q, m, d, _p(queries), _p(ql), _p(database), _p(dl), int(exclude), L, _p(ap), _p(prec), _p(nrel),
                                             _stream()), "retrieval_metrics")
    return {"ap": ap, "precision": prec, "num_relevant": nrel}


# ----------------------------------------------------------------------------------------------------- non-finite step guard
_GUARD_DTYPES = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.bfloat16: 3}


def _guard_tensor(t, dev, what):
    if not isinstance(t, torch.Tensor) or t.device != dev or not t.is_contiguous():
        raise ValueError("nonfinite guard: every %s tensor must be a contiguous tensor on %s" % (what, dev))
    if t.is_complex() or t.numel() >= 2 ** 31:
        raise ValueError("nonfinite guard: %s tensors must be real with fewer than 2^31 elements, got %s of %d" % (what, t.dtype, t.numel()))


class NonfiniteGuard:
    """One caller's device state of snb200_nonfinite_guard (include/samplenet_b200.h): the state words the kernels leave zero, the 0/1
    result of the last call (`skipped`, int32, 0-dim) and the number of calls that restored (`skip_count`, int32, 0-dim).  Calls on
    different streams, or in different CUDA graphs, need guards of their own.

        guard = NonfiniteGuard(device)
        skipped = guard(checked, live, snapshots)

    If any element of a floating tensor in `checked` is NaN or +-Inf, every snapshots[i] is copied over live[i] bit for bit; otherwise
    nothing is written but the result.  Integer tensors in `checked` are finite and passed over.  Two launches for up to 384 tensors per
    table, no read-back, capturable; returns `skipped`."""

    def __init__(self, device):
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        self.state = torch.zeros(2, dtype=torch.int32, device=dev)
        self.skipped = torch.zeros((), dtype=torch.int32, device=dev)
        self.skip_count = torch.zeros((), dtype=torch.int32, device=dev)

    def __call__(self, checked, live, snapshots):
        dev = self.device
        chk = []
        for t in checked:
            _guard_tensor(t, dev, "checked")
            if t.is_floating_point():
                code = _GUARD_DTYPES.get(t.dtype)
                if code is None:
                    raise ValueError("nonfinite guard: unsupported floating dtype %s" % t.dtype)
                chk.append((t.data_ptr(), t.numel(), code))
        live, snapshots = list(live), list(snapshots)
        if len(live) != len(snapshots):
            raise ValueError("nonfinite guard: %d live tensors but %d snapshots" % (len(live), len(snapshots)))
        rst = []
        for a, s in zip(live, snapshots):
            _guard_tensor(a, dev, "live")
            _guard_tensor(s, dev, "snapshot")
            if a.dtype != s.dtype or a.shape != s.shape:
                raise ValueError("nonfinite guard: a snapshot %s %s does not match its live tensor %s %s"
                                 % (s.dtype, tuple(s.shape), a.dtype, tuple(a.shape)))
            rst.append((a.data_ptr(), s.data_ptr(), a.numel() * a.element_size()))
        ct = (_lib.GuardCheck * max(len(chk), 1))(*chk)
        rt = (_lib.GuardRestore * max(len(rst), 1))(*rst)
        with torch.cuda.device(dev):
            check(lib().snb200_nonfinite_guard(ct, len(chk), rt, len(rst), _p(self.state), _p(self.skipped), _p(self.skip_count), _stream()),
                  "nonfinite_guard")
        return self.skipped


# ----------------------------------------------------------------------------------------------------- test hook
def debug_tc_gemm(A, W, bias):
    """D = A @ W.T + bias through the wgmma layer kernel (3xTF32).  A (rows, c_in), W (c_out, c_in), bias (c_out)."""
    A, W, bias = _req(A, "A"), _req(W, "W"), _req(bias, "bias")
    rows, c_in = A.shape
    c_out = W.shape[0]
    with torch.cuda.device(A.device):
        D = torch.empty(rows, c_out, device=A.device)
        check(lib().snb200_debug_tc_gemm(rows, c_in, c_out, _p(A), _p(W), _p(bias), _p(D), _stream()), "debug_tc_gemm")
    return D
