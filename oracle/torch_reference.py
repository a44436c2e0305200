"""Plain-torch CPU restatement of the reference's SampleNet step (test infrastructure, NOT product):

    registration/src/samplenet.py:82-161   forward (train mode): conv/BN/ReLU x5 -> max -> FC/BN/ReLU x3 -> FC -> soft projection
    registration/src/samplenet.py:171-181  get_simplification_loss

The layer stack is stock torch (nn.Conv1d / BatchNorm1d / Linear run by torch's CPU kernels, exactly what the reference
executes on CPU); kNN + soft projection go through the C oracle (the reference's knn_cuda / pointnet2 are CUDA-only);
Chamfer goes through the reference's own CPU code in oracle/_ref when present, else the C oracle.
Used by bench.py (cpu_baseline and --impl reference) and by tests.  Only importable from those places.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import oracle as orc


class ReferenceGenerator(nn.Module):
    """Same parameter names / registration order as registration/src/samplenet.py:40-60."""

    def __init__(self, num_out_points, bottleneck_size):
        super().__init__()
        self.num_out_points = num_out_points
        w = [3, 64, 64, 64, 128, bottleneck_size]
        for i in range(5):
            setattr(self, "conv%d" % (i + 1), nn.Conv1d(w[i], w[i + 1], 1))
        for i in range(5):
            setattr(self, "bn%d" % (i + 1), nn.BatchNorm1d(w[i + 1]))
        f = [bottleneck_size, 256, 256, 256, 3 * num_out_points]
        for i in range(4):
            setattr(self, "fc%d" % (i + 1), nn.Linear(f[i], f[i + 1]))
        for i in range(3):
            setattr(self, "bn_fc%d" % (i + 1), nn.BatchNorm1d(256))

    def forward(self, x_bcn):
        y = x_bcn
        for i in range(1, 6):
            y = F.relu(getattr(self, "bn%d" % i)(getattr(self, "conv%d" % i)(y)))
        y = torch.max(y, 2)[0]
        for i in range(1, 4):
            y = F.relu(getattr(self, "bn_fc%d" % i)(getattr(self, "fc%d" % i)(y)))
        y = self.fc4(y)
        return y.view(-1, 3, self.num_out_points)


_POOL = {}


def _pool(workers):
    from concurrent.futures import ThreadPoolExecutor
    if workers not in _POOL:
        _POOL[workers] = ThreadPoolExecutor(max_workers=workers)
    return _POOL[workers]


def _over_clouds(fn, workers, *arrays):
    """Run fn(chunk of every array) over contiguous chunks of the batch on `workers` threads (the C calls release the GIL) and
    concatenate the results -- clouds are independent, so this is how the CPU path uses all host threads."""
    b = arrays[0].shape[0]
    if workers <= 1 or b <= 1:
        return fn(*arrays)
    w = min(workers, b)
    bounds = [(b * i) // w for i in range(w + 1)]
    futs = [_pool(w).submit(fn, *[np.ascontiguousarray(a[bounds[i]:bounds[i + 1]]) for a in arrays]) for i in range(w)]
    parts = [f.result() for f in futs]
    return tuple(np.concatenate([p[j] for p in parts], axis=0) for j in range(len(parts[0])))


def cpu_generator(gen, x_bnc):
    """The layer stack (torch CPU kernels, torch's intra-op threads): x (B,N,3) torch -> simp (B,M,3) numpy."""
    with torch.no_grad():
        return gen(x_bnc.permute(0, 2, 1)).permute(0, 2, 1).contiguous().numpy()


def cpu_pairwise(x_bnc, simp, k, sigma, gamma=1.0, delta=0.0, workers=1):
    """kNN + soft projection (C oracle) and Chamfer (the reference's CPU code when oracle/_ref exists) + the loss reductions,
    cloud-parallel on `workers` threads.  Returns (proj, loss)."""
    x = x_bnc.numpy()
    _, idx = _over_clouds(lambda a, q: orc.knn_point(k, a, q, contract=False, tie_mode=0), workers, x, simp)
    proj, _, _ = _over_clouds(lambda a, q, i: orc.soft_project(a, q, i, float(sigma)), workers, x, simp, idx)
    if orc.have_ref():
        c12, _, c21, _ = _over_clouds(lambda q, a: orc.ref_chamfer_forward(q, a), workers, simp, x)
    else:
        c12, _, c21, _ = _over_clouds(lambda q, a: orc.nn_distance(q, a), workers, simp, x)
    m = simp.shape[1]
    loss = np.float32(c12.mean(dtype=np.float32) + c12.max(axis=1).mean(dtype=np.float32) + np.float32(gamma + delta * m) * c21.mean(dtype=np.float32))
    return proj, loss


def cpu_step(gen, x_bnc, k, sigma, gamma=1.0, delta=0.0, workers=1):
    """One forward (train mode) + simplification loss on the CPU.  x_bnc: torch (B,N,3) float32.  Returns (simp, proj, loss).
    workers > 1: kNN / projection / Chamfer run cloud-parallel on that many threads (the layer stack uses torch's own threads)."""
    simp = cpu_generator(gen, x_bnc)
    proj, loss = cpu_pairwise(x_bnc, simp, k, sigma, gamma, delta, workers)
    return simp, proj, loss


# ------------------------------------------------------------------------------------------------- the reference ON THE GPU (row G0)
class GpuReferenceStep:
    """The reference's GPU path for the headline step, assembled from what exists on the box (SURVEY.md 8d (iv), BASELINE.md G0):
      * the layer stack: stock torch modules on CUDA (cuDNN / cuBLAS / ATen BatchNorm kernels, TF32 off like the fp32 reference);
      * kNN: the reference uses KNN_CUDA 0.2 (not in the tree): torch.cdist + topk stand-in, the rest of SoftProjection.project in the
        reference's own torch ops (registration/src/soft_projection.py:75-127: gather, softmax over -d/sigma, weighted sum);
      * Chamfer: the REFERENCE'S OWN CUDA kernels compiled unmodified for sm_90 (oracle/_ref/libsamplenet_ref_cuda.so), two launches on
        the legacy default stream + the four torch reductions of get_simplification_loss (samplenet.py:171-181).
    Eager launches on the default stream, as the reference trainer issues them.  Measurement infrastructure, not product."""

    def __init__(self, num_out_points, bottleneck, k, device):
        from . import ref_cuda

        self.refcu = ref_cuda
        self.dev = device
        torch.manual_seed(0)
        self.gen = ReferenceGenerator(num_out_points, bottleneck).to(device).train()
        self.k = k
        self.m = num_out_points
        self.sigma = 1.0

    def generator(self, x_bnc):
        return self.gen(x_bnc.permute(0, 2, 1)).permute(0, 2, 1).contiguous()

    def project(self, x_bnc, simp):
        d = torch.cdist(simp, x_bnc)                              # (B, M, N)
        _, idx = torch.topk(d, self.k, dim=2, largest=False)      # KNN_CUDA stand-in
        grouped = torch.gather(x_bnc[:, None].expand(-1, simp.shape[1], -1, -1), 2, idx[..., None].expand(-1, -1, -1, 3))   # (B, M, k, 3)
        dist = ((grouped - simp[:, :, None, :]) ** 2).sum(-1) / self.sigma
        w = torch.softmax(-dist, dim=2)
        return (w[..., None] * grouped).sum(2)

    def chamfer_loss(self, x_bnc, simp):
        c12, _, c21, _ = self.refcu.chamfer_forward(simp, x_bnc)
        return torch.mean(c12) + torch.mean(torch.max(c12, dim=1)[0]) + torch.mean(c21)

    def step(self, x_bnc):
        simp = self.generator(x_bnc)
        proj = self.project(x_bnc, simp)
        return simp, proj, self.chamfer_loss(x_bnc, simp)


def time_gpu_reference(x_pool, num_out_points, bottleneck, k, steps=100, warmup=10):
    """us per step of GpuReferenceStep (eager, default stream, CUDA events) + per-stage times.  x_pool: (P, B, N, 3) CUDA tensor."""
    dev = x_pool.device
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref = GpuReferenceStep(num_out_points, bottleneck, k, dev)
        npool = x_pool.shape[0]

        def timed(fn, reps):
            for i in range(warmup):
                fn(i)
            torch.cuda.synchronize(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(reps):
                fn(i)
            b.record(); b.synchronize()
            return a.elapsed_time(b) * 1e3 / reps

        out = {}
        with torch.no_grad():
            out["step_us"] = timed(lambda i: ref.step(x_pool[i % npool]), steps)
            simp = ref.generator(x_pool[0])
            out["generator_us"] = timed(lambda i: ref.generator(x_pool[i % npool]), steps)
            out["knn_project_us"] = timed(lambda i: ref.project(x_pool[i % npool], simp), steps)
            out["chamfer_loss_us"] = timed(lambda i: ref.chamfer_loss(x_pool[i % npool], simp), steps)
            out["chamfer_kernels_only_us"] = timed(lambda i: ref.refcu.chamfer_forward(simp, x_pool[i % npool]), steps)
            # the torch part replayed from a CUDA graph (what a maintainer gets from torch.cuda.graphs without touching a kernel); the
            # reference's Chamfer launchers use the legacy stream and cannot be captured, so they stay eager behind it
            try:
                xs = x_pool[0].clone()
                s = torch.cuda.Stream(device=dev)
                s.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(s):
                    for _ in range(3):
                        sg = ref.generator(xs); ref.project(xs, sg)
                torch.cuda.current_stream(dev).wait_stream(s)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    sg = ref.generator(xs); pg = ref.project(xs, sg)

                def graphed(i):
                    xs.copy_(x_pool[i % npool], non_blocking=True)
                    g.replay()
                    return ref.chamfer_loss(xs, sg)

                out["step_graphed_torch_part_us"] = timed(graphed, steps)
            except Exception as exc:
                out["step_graphed_torch_part_error"] = str(exc)[:200]
        out["note"] = ("reference-on-GPU: stock torch layer stack (cuDNN/cuBLAS/ATen, TF32 off) + torch.cdist/topk kNN stand-in for KNN_CUDA + the "
                       "reference's SoftProjection torch ops + the reference's own Chamfer CUDA kernels compiled for sm_90; eager launches on the "
                       "default stream as in the reference trainer")
        return out
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
