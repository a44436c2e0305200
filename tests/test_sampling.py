"""Farthest point sampling (csrc/fps.cu), gather_point and the FPS / random baseline samplers.

The indices must be bit-exact against the reference's own farthestpointsamplingKernel: its outputs on the inputs below are stored in
tests/golden/reference_cuda_sampling.npz (tests/golden/make_reference_sampling_golden.py, from oracle/_ref/libsamplenet_ref_cuda.so),
and tests/fps_oracle.c restates the kernel in plain C as a second, CPU-side check.
"""
import ctypes
import os
import subprocess
import warnings

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "reference_cuda_sampling.npz")

# name -> (b, n, m, kind)
FPS_CASES = {
    "rec_sort": (50, 2048, 2048, "rand"),       # SamplerAutoEncoder.sort: a full 2048-of-2048 ordering
    "reg_baseline": (32, 1024, 64, "rand"),     # registration --sampler fps
    "tiny": (3, 20, 12, "rand"),                # n < 32
    "ragged": (4, 777, 300, "rand"),            # n not a multiple of 32 or 512
    "ragged_1537": (2, 1537, 700, "rand"),
    "past_smem_cache": (2, 5000, 800, "rand"),  # n > 3072: the reference reads these points from global memory
    "modelnet_10k": (2, 10000, 1024, "rand"),
    "max_16384": (2, 16384, 1024, "rand"),
    "m_gt_n": (3, 100, 160, "rand"),            # index 0 repeats once every point is taken
    "duplicates": (4, 1024, 700, "dup"),
    "lattice": (2, 1000, 400, "lattice"),
    "identical": (2, 700, 40, "same"),
}
GATHER_CASES = {"gather_ragged": ("ragged", 11), "gather_reg": ("reg_baseline", 12)}


def fps_input(name):
    """The seeded (b, n, 3) float32 cloud of a case (numpy)."""
    b, n, m, kind = FPS_CASES[name]
    g = torch.Generator().manual_seed(sum(name.encode()) * 31 + n)
    if kind == "rand":
        x = torch.rand(b, n, 3, generator=g) - 0.5
    elif kind == "dup":  # 300 distinct points, each repeated, in a shuffled order
        base = torch.rand(b, 300, 3, generator=g) - 0.5
        x = base[:, torch.randint(0, 300, (n,), generator=g)]
    elif kind == "lattice":  # 10 x 10 x 10 integer lattice: many exactly equal distances
        a = torch.arange(10, dtype=torch.float32)
        grid = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
        x = torch.stack([grid[torch.randperm(n, generator=g)] for _ in range(b)])
    else:
        x = (torch.rand(b, 1, 3, generator=g) - 0.5).expand(b, n, 3)
    return x.contiguous().numpy().astype(np.float32)


def gather_indices(name):
    """Indices with duplicates for the gather_point checks: (b, 2m) drawn with replacement."""
    case, seed = GATHER_CASES[name]
    b, n, m, _ = FPS_CASES[case]
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, n, (b, 2 * m), generator=g, dtype=torch.int32).numpy()


# ----------------------------------------------------------------------------------------------------- CPU oracle
@pytest.fixture(scope="session")
def fps_oracle(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("fps_oracle") / "libfps_oracle.so")
    subprocess.run(["cc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "fps_oracle.c"), "-lm"], check=True)
    lib = ctypes.CDLL(so)
    fp = ctypes.POINTER(ctypes.c_float)
    ip = ctypes.POINTER(ctypes.c_int)
    lib.fps_oracle.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, fp, ip, fp]

    def run(x, m):
        x = np.ascontiguousarray(x, dtype=np.float32)
        b, n, _ = x.shape
        idx = np.empty((b, m), np.int32)
        scratch = np.empty(n, np.float32)
        lib.fps_oracle(b, n, m, x.ctypes.data_as(fp), idx.ctypes.data_as(ip), scratch.ctypes.data_as(fp))
        return idx

    return run


@pytest.fixture(scope="session")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="session")
def oracle_idx(fps_oracle):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = fps_oracle(fps_input(name), FPS_CASES[name][2])
        return cache[name]

    return get


@pytest.mark.parametrize("name", sorted(FPS_CASES))
def test_oracle_matches_reference_kernel(name, golden, oracle_idx):
    assert np.array_equal(oracle_idx(name), golden["fps_" + name].astype(np.int32))


def test_golden_covers_the_tie_rule(golden):
    """The stored cases exercise ties: index 0 repeats in m > n, and an all-identical cloud selects point 0 every round."""
    assert np.all(golden["fps_m_gt_n"][:, 100:] == 0)
    assert np.all(golden["fps_identical"] == 0)
    assert np.array_equal(np.sort(golden["fps_rec_sort"].astype(np.int64), axis=1), np.tile(np.arange(2048), (50, 1)))


def test_argument_errors_raise_value_error():
    from samplenet_b200 import ops, tf_ops

    x = torch.zeros(2, 16, 3)
    with pytest.raises(ValueError):
        ops.farthest_point_sample(torch.zeros(2, 16, 4), 4)
    with pytest.raises(ValueError):
        ops.farthest_point_sample(torch.zeros(16, 3), 4)
    with pytest.raises(ValueError):
        ops.farthest_point_sample(torch.zeros(2, 16, 3), 4, layout="bcn")
    with pytest.raises(ValueError):
        ops.farthest_point_sample(x, 0)
    with pytest.raises(ValueError):
        ops.farthest_point_sample(x, 2.5)
    with pytest.raises(ValueError):
        ops.farthest_point_sample(x, 4, layout="nbc")
    with pytest.raises(ValueError):
        ops.farthest_point_sample(torch.zeros(2, 0, 3), 4)
    with pytest.raises(ValueError):
        tf_ops.farthest_point_sample(-1, x)
    with pytest.raises(ValueError):
        tf_ops.gather_point(torch.zeros(2, 16, 4), torch.zeros(2, 4, dtype=torch.int32))
    with pytest.raises(ValueError):
        ops.gather_point(x, torch.zeros(3, 4, dtype=torch.int32))


def test_cpu_tensors_raise_runtime_error():
    from samplenet_b200 import ops, tf_ops

    with pytest.raises(RuntimeError):
        ops.farthest_point_sample(torch.zeros(2, 16, 3), 4)
    with pytest.raises(RuntimeError):
        tf_ops.farthest_point_sample(4, torch.zeros(2, 16, 3))
    with pytest.raises(RuntimeError):
        tf_ops.gather_point(torch.zeros(2, 16, 3), torch.zeros(2, 4, dtype=torch.int32))


def test_abi_validates_before_launching():
    """The C entry point rejects bad sizes and clouds above 16384 points before touching the device."""
    from samplenet_b200 import _lib

    lib = _lib.lib()
    fake = ctypes.c_void_p(256)
    assert lib.snb200_farthest_point_sample(0, 16, 4, _lib.BNC, None, None, None, None) == 0  # empty batch: nothing to do
    assert lib.snb200_farthest_point_sample(1, 16, 0, _lib.BNC, fake, fake, None, None) == -1
    assert lib.snb200_farthest_point_sample(1, 0, 4, _lib.BNC, fake, fake, None, None) == -1
    assert lib.snb200_farthest_point_sample(1, 16, 4, 7, fake, fake, None, None) == -1
    assert lib.snb200_farthest_point_sample(1, 16, 4, _lib.BNC, None, fake, None, None) == -1
    assert lib.snb200_farthest_point_sample(1, 16385, 4, _lib.BNC, fake, fake, None, None) == -4
    assert b"16384" in lib.snb200_last_error()
    assert lib.snb200_debug_farthest_point_sample(1, 16, 4, _lib.BNC, fake, fake, None, 384, None) == -1


def test_sampler_constructors_behave_as_the_reference():
    from samplenet_b200 import FPSSampler, RandomSampler

    s = FPSSampler(64, permute=True, input_shape="bnc", output_shape="bnc")
    assert (s.name, s.num_out_points, s.permute, s.input_shape, s.output_shape) == ("fps", 64, True, "bnc", "bnc")
    r = RandomSampler(32)
    assert (r.name, r.num_out_points, r.input_shape, r.output_shape) == ("random", 32, "bcn", "bcn")
    for cls, args in ((FPSSampler, (8, False)), (RandomSampler, (8,))):
        with pytest.raises(ValueError, match="allowed shape"):
            cls(*args, input_shape="nbc")
        with pytest.raises(ValueError, match="allowed shape"):
            cls(*args, output_shape="cnb")
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            cls(*args, input_shape="bnc", output_shape="bcn")
        assert any("input_shape is different to output_shape" in str(x.message) for x in w)
    assert not list(FPSSampler(8, True).parameters()) and not list(RandomSampler(8).parameters())


def test_registration_step_rejects_unknown_sampler():
    from samplenet_b200.registration import RegistrationStep

    with pytest.raises(ValueError):
        RegistrationStep(sampler="poisson")
    assert RegistrationStep(sampler="none").create_model().sampler is None
    assert RegistrationStep(sampler="random").create_model().sampler.name == "random"


# ----------------------------------------------------------------------------------------------------- GPU
gpu = pytest.mark.gpu


def _thread_configs(n):
    return [t for t, cap in ((256, 4096), (512, 8192), (1024, 16384)) if n <= cap]


@gpu
@pytest.mark.parametrize("name", sorted(FPS_CASES))
def test_indices_bit_exact_vs_reference_kernel(name, golden, oracle_idx):
    from samplenet_b200 import ops, tf_ops

    b, n, m, _ = FPS_CASES[name]
    x = torch.from_numpy(fps_input(name)).cuda()
    want = golden["fps_" + name].astype(np.int32)
    got = tf_ops.farthest_point_sample(m, x)
    assert got.dtype == torch.int32 and tuple(got.shape) == (b, m)
    got = got.cpu().numpy()
    assert np.array_equal(got, want)
    assert np.array_equal(got, oracle_idx(name))
    for t in _thread_configs(n):  # every configuration the kernel can take for this size, not only the one chosen by default
        assert np.array_equal(ops.farthest_point_sample(x, m, _threads=t).cpu().numpy(), want), t


@gpu
@pytest.mark.parametrize("name", ["ragged", "rec_sort", "modelnet_10k", "tiny", "m_gt_n"])
def test_bcn_equals_bnc_and_fused_points_equal_gather(name):
    from samplenet_b200 import ops

    b, n, m, _ = FPS_CASES[name]
    x = torch.from_numpy(fps_input(name)).cuda()
    i_bnc, p_bnc = ops.farthest_point_sample(x, m, "bnc", return_points=True)
    i_bcn, p_bcn = ops.farthest_point_sample(x.permute(0, 2, 1).contiguous(), m, "bcn", return_points=True)
    assert torch.equal(i_bnc, i_bcn)
    ref = torch.gather(x, 1, i_bnc.long()[..., None].expand(b, m, 3))
    assert torch.equal(p_bnc, ref)
    assert torch.equal(p_bcn, ref.permute(0, 2, 1))
    assert torch.equal(ops.farthest_point_sample(x, m), i_bnc)


@gpu
def test_too_many_points_raises():
    from samplenet_b200 import ops

    with pytest.raises(RuntimeError, match="16384"):
        ops.farthest_point_sample(torch.zeros(1, 16385, 3, device="cuda"), 4)
    assert ops.farthest_point_sample(torch.zeros(0, 10, 3, device="cuda"), 4).shape == (0, 4)


@gpu
@pytest.mark.parametrize("name", sorted(GATHER_CASES))
def test_gather_point_forward_and_backward(name, golden):
    from samplenet_b200 import tf_ops

    case = GATHER_CASES[name][0]
    xn = fps_input(case)
    idx_np = gather_indices(name)
    x = torch.from_numpy(xn).cuda().requires_grad_(True)
    idx = torch.from_numpy(idx_np).cuda()
    y = tf_ops.gather_point(x, idx)
    assert tuple(y.shape) == (idx.shape[0], idx.shape[1], 3)
    assert np.array_equal(y.detach().cpu().numpy(), golden[name])
    g = torch.randn(y.shape, generator=torch.Generator().manual_seed(3)).cuda()
    grads = []
    for _ in range(2):
        x.grad = None
        y = tf_ops.gather_point(x, idx)
        y.backward(g)
        grads.append(x.grad.clone())
    assert torch.equal(grads[0], grads[1]), "the gather_point gradient must be deterministic"
    want = np.zeros(xn.shape, np.float64)
    gn = g.cpu().numpy().astype(np.float64)
    for bi in range(xn.shape[0]):
        np.add.at(want[bi], idx_np[bi], gn[bi])
    assert np.max(np.abs(grads[0].cpu().numpy() - want)) <= 1e-5 * max(1.0, np.abs(want).max())


@gpu
def test_cuda_graph_replay_equals_eager():
    from samplenet_b200 import ops

    x = torch.from_numpy(fps_input("reg_baseline")).cuda()
    eager_i, eager_p = ops.farthest_point_sample(x, 64, return_points=True)
    eager_g = ops.gather_point(x, eager_i)
    static_x = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            ops.farthest_point_sample(static_x, 64, return_points=True)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gi, gp = ops.farthest_point_sample(static_x, 64, return_points=True)
        gg = ops.gather_point(static_x, gi)
    static_x.copy_(torch.flip(x, dims=[0]))
    graph.replay()
    torch.cuda.synchronize()
    fi, fp = ops.farthest_point_sample(torch.flip(x, dims=[0]).contiguous(), 64, return_points=True)
    assert torch.equal(gi, fi) and torch.equal(gp, fp)
    static_x.copy_(x)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(gi, eager_i) and torch.equal(gp, eager_p) and torch.equal(gg, eager_g)


def _gather_bcn(x, idx):  # pointnet2 gather_operation: (B, C, N), (B, m) -> (B, C, m)
    return torch.gather(x, 2, idx.long()[:, None, :].expand(x.shape[0], x.shape[1], idx.shape[1]))


@gpu
@pytest.mark.parametrize("shapes", [("bnc", "bnc"), ("bcn", "bcn"), ("bnc", "bcn")])
def test_fps_sampler_matches_reference_module(shapes, fps_oracle):
    """registration/src/fps.py restated with the same RNG call (torch.randperm(N) on the default CPU generator) and the C oracle's FPS."""
    from samplenet_b200 import FPSSampler

    in_s, out_s = shapes
    x = torch.from_numpy(fps_input("reg_baseline")).cuda()
    xin = x if in_s == "bnc" else x.permute(0, 2, 1).contiguous()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sampler = FPSSampler(64, permute=True, input_shape=in_s, output_shape=out_s)
    torch.manual_seed(1234)
    y = sampler(xin)
    torch.manual_seed(1234)
    xp = x[:, torch.randperm(x.shape[1]), :]
    idx = torch.from_numpy(fps_oracle(xp.cpu().numpy(), 64)).cuda()
    want = _gather_bcn(xp.permute(0, 2, 1).contiguous(), idx)
    if out_s == "bnc":
        want = want.permute(0, 2, 1).contiguous()
    assert torch.equal(y, want)
    # differentiable in x, like gather_operation
    xg = xin.clone().requires_grad_(True)
    torch.manual_seed(1234)
    sampler(xg).sum().backward()
    assert float(xg.grad.sum()) == pytest.approx(64 * 3 * x.shape[0])


@gpu
@pytest.mark.parametrize("shapes", [("bnc", "bnc"), ("bcn", "bcn"), ("bcn", "bnc")])
def test_random_sampler_matches_reference_module(shapes):
    """registration/src/random_sampling.py restated: one torch.randperm(N, dtype=int32, device=x.device) per cloud."""
    from samplenet_b200 import RandomSampler

    in_s, out_s = shapes
    x = torch.from_numpy(fps_input("reg_baseline")).cuda()
    xin = x if in_s == "bnc" else x.permute(0, 2, 1).contiguous()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sampler = RandomSampler(64, input_shape=in_s, output_shape=out_s)
    torch.manual_seed(99)
    y = sampler(xin)
    torch.manual_seed(99)
    xb = x.permute(0, 2, 1).contiguous()
    B, _, N = xb.shape
    idx = torch.zeros(B, 64, dtype=torch.int32, device=x.device)
    for i in range(B):
        idx[i] = torch.randperm(N, dtype=torch.int32, device=x.device)[:64]
    want = _gather_bcn(xb, idx)
    if out_s == "bnc":
        want = want.permute(0, 2, 1).contiguous()
    assert torch.equal(y, want)


@gpu
@pytest.mark.parametrize("sampler", ["fps", "random", "none"])
def test_registration_step_with_baseline_samplers(sampler):
    from samplenet_b200.registration import RegistrationStep

    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    step = RegistrationStep(num_out_points=64, train_pcrnet=True, sampler=sampler)
    model = step.create_model().to(dev)
    assert (model.sampler.name if model.sampler is not None else "none") == sampler
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-4)
    p0 = torch.rand(8, 1024, 3) - 0.5
    p1 = torch.rand(8, 1024, 3) - 0.5
    vec = torch.cat([torch.nn.functional.normalize(torch.randn(8, 4), dim=1), 0.1 * torch.randn(8, 3)], 1)  # (w,x,y,z) + translation
    igt = {"vec": vec, "inversion": torch.tensor([False])}
    loss, rot_err, info = step.train_step(model, (p0, p1, igt), opt, dev)
    assert torch.isfinite(loss) and torch.isfinite(rot_err)
    assert float(info["simplification_loss"]) == 0.0 and float(info["projection_loss"]) == 0.0
    if sampler == "fps":
        sampled = step.non_learned_sampling(model, (p0, p1, igt), dev)
        assert sampled[0].shape == (8, 64, 3) and sampled[1].shape == (8, 64, 3)
