"""GPU parity against the REFERENCE'S OWN CUDA KERNELS: the .cu files of the reference compiled unmodified (oracle/Makefile,
oracle/ref_cuda_shim.cu) and run on the inputs below; their outputs are stored in tests/golden/reference_cuda.npz
(tests/golden/make_reference_cuda_golden.py, a seeded sample of the entries of the large outputs) and compared with this library's
kernels on identical inputs -- north_star: "outputs match the reference's own TF/CUDA ops on identical inputs (kNN indices and match
assignments bit-exact, distances/losses within a stated fp32 tolerance)".
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CHAMFER_CASES = [(32, 64, 1024), (4, 37, 129), (2, 513, 511), (32, 1024, 1024), (50, 2048, 2048), (3, 5, 2000)]
KNN_CASES = [(32, 1024, 64, 8), (32, 1024, 32, 7), (4, 2048, 64, 16), (3, 200, 17, 3), (2, 1024, 1024, 7)]
EMD_CASES = [(64, 64), (96, 32), (300, 300), (2048, 2048)]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_cuda.npz")


def sample_positions(size, key, count=512):
    """The fixed sample of flat positions stored for an output of `size` entries (all of them when it is small)."""
    if size <= count:
        return np.arange(size)
    rng = np.random.default_rng(sum(key.encode()) * 7919 + size)
    return np.sort(rng.choice(size, count, replace=False))


@pytest.fixture(scope="module")
def sb():
    import samplenet_b200

    samplenet_b200._lib.lib()
    return samplenet_b200


@pytest.fixture(scope="module")
def ref():
    return dict(np.load(GOLDEN))


def _clouds(seed, b, n, m, noise=0.02):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(b, n, 3, generator=g) - 0.5
    if m <= n:
        q = x[:, torch.randperm(n, generator=g)[:m]] + noise * torch.randn(b, m, 3, generator=g)
    else:
        q = torch.rand(b, m, 3, generator=g) - 0.5
    return x.cuda().contiguous(), q.cuda().contiguous()


def _emd_inputs(n, m):
    """Two clouds and a seeded match matrix (b, m, n) with the magnitudes of a real assignment (rows of about unit mass)."""
    b = 2 if n < 2048 else 1
    g = torch.Generator().manual_seed(n + m)
    a = torch.rand(b, n, 3, generator=g).cuda(); c = torch.rand(b, m, 3, generator=g).cuda()
    match_in = (torch.rand(b, m, n, generator=torch.Generator().manual_seed(7 * n + m)) * (2.0 / n)).cuda()
    return a, c, match_in


def _at(t, key):
    a = t.detach().cpu().numpy()
    return a.reshape(-1)[sample_positions(a.size, key)]


@pytest.mark.parametrize("b,n,m", CHAMFER_CASES)
def test_chamfer_forward_equals_reference_kernels(sb, ref, b, n, m):
    """registration ChamferDistanceKernel and TF NmDistanceKernel (same algorithm, two files, identical outputs): indices AND squared
    distances bit-identical to this library's kernel in its default (FMA-contracted, what nvcc gives the reference) arithmetic."""
    x, q = _clouds(b + n + m, b, m, n)          # xyz1 = q (b, n, 3), xyz2 = x (b, m, 3)
    outs = sb.ops.nn_distance_forward(q, x)
    torch.cuda.synchronize()
    for name, t in zip(("d1", "i1", "d2", "i2"), outs):
        key = "chamfer_%d_%d_%d_%s" % (b, n, m, name)
        assert np.array_equal(_at(t, key), ref[key]), key


def test_chamfer_backward_vs_reference_kernels(sb, ref):
    x, q = _clouds(3, 8, 1024, 64)
    d1, i1, d2, i2 = sb.ops.nn_distance_forward(q, x)
    g = torch.Generator().manual_seed(5)
    g1 = torch.rand(d1.shape, generator=g).cuda(); g2 = torch.rand(d2.shape, generator=g).cuda()
    gx1, gx2 = sb.ops.nn_distance_backward(q, x, g1, i1, g2, i2)
    torch.cuda.synchronize()   # (the reference uses float atomics: order-dependent rounding)
    np.testing.assert_allclose(_at(gx1, "chamfer_bwd_gx1"), ref["chamfer_bwd_gx1"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(_at(gx2, "chamfer_bwd_gx2"), ref["chamfer_bwd_gx2"], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("b,n,m,k", KNN_CASES)
def test_knn_equals_reference_selection_sort(sb, ref, b, n, m, k):
    """tf_grouping.knn_point = TF distance matrix + the reference's selection-sort kernel (tf_grouping_g.cu:83-123): neighbour indices
    bit-exact (tie-free inputs), squared distances bit-exact in this library's unfused arithmetic mode (three roundings, the order TF's
    elementwise graph evaluates); group_point on those indices bit-exact."""
    x, q = _clouds(b * 7 + k, b, n, m)
    o = sb.ops.knn_soft_project_forward(x, q, k, "bnc", want=("idx", "val"), unfused=True)
    ours = sb.tf_ops.group_point(x, o["idx"])
    torch.cuda.synchronize()
    key = "knn_%d_%d_%d_%d_" % (b, n, m, k)
    assert np.array_equal(_at(o["idx"], key + "idx"), ref[key + "idx"])
    assert np.array_equal(_at(o["val"], key + "val"), ref[key + "val"])
    assert np.array_equal(_at(ours, key + "gp"), ref[key + "gp"])


@pytest.mark.parametrize("n,m", EMD_CASES)
def test_emd_vs_reference_kernels(sb, ref, n, m):
    """approxmatch / matchcost / matchcostgrad of tf_approxmatch_g.cu (float, __expf, 512-thread tree reductions) on identical inputs.
    The reference GPU kernel is itself only an approximation of its CPU twin (its self-test flags |diff| > 1e-2, approxmatch.cpp:222);
    this library's fast kernel and its exact mode are both compared, and cost / gradients on an identical match matrix."""
    a, c, match_in = _emd_inputs(n, m)
    key = "emd_%d_%d_" % (n, m)
    fast = sb.tf_ops.approx_match(a, c)
    torch.cuda.synchronize()
    assert float(np.abs(_at(fast, key + "match") - ref[key + "match"]).max()) < 5e-3
    if n <= 300:
        exact = sb.tf_ops.approx_match(a, c, exact=True)
        torch.cuda.synchronize()
        assert float(np.abs(_at(exact, key + "match") - ref[key + "match"]).max()) < 5e-3
        # assignments: equal wherever the reference's own top-2 gap exceeds that tolerance
        rm, ex = ref[key + "match_rows"], exact[:, :16].cpu().numpy()
        assert float(np.abs(ex - rm).max()) < 5e-3
        am, ar = ex.argmax(axis=2), rm.argmax(axis=2)
        gap = np.take_along_axis(rm, ar[..., None], 2)[..., 0] - np.take_along_axis(rm, am[..., None], 2)[..., 0]
        assert bool((gap < 5e-3).all())
    oc = sb.ops.match_cost_forward(a, c, match_in)
    og1, og2 = sb.ops.match_cost_grad(a, c, match_in)
    torch.cuda.synchronize()
    np.testing.assert_allclose(oc.cpu().numpy(), ref[key + "cost"], rtol=2e-5)
    np.testing.assert_allclose(og1.cpu().numpy(), ref[key + "grad1"], rtol=2e-4, atol=2e-5)
    np.testing.assert_allclose(og2.cpu().numpy(), ref[key + "grad2"], rtol=2e-4, atol=2e-5)
