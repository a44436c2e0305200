"""The registration step with one sampled cloud (registration/main.py --num-sampled-clouds 1): the full template against the sampled
source through the CUDA path -- the pose loss's _ex entries (csrc/pose_loss.cu with a template of m0 points and a source of m1),
FrozenPCRNet / CudaPCRNet with one encoder call per cloud size, RegistrationStep's fused loss and test_1's batched route.

CPU: the float64 restatement at m0 != m1 against float64 autograd of the torch code; the _ex entries' envelope, workspace sizes and
rejections (nothing launches).  GPU (H100): the _ex kernels against float64 at four shapes and on exact duplicates, bit for bit the plain
entries at equal sizes, run to run bit-identical, their write sets; pose_eval_ex against the per-record torch loop and the reference's
fixture; whole train steps (frozen task, and PCRNet trained jointly with the sampler) against the plain module; chunking beyond 32 pairs;
test_1 against the per-record loop."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from samplenet_b200 import registration as reg  # noqa: E402
import test_frozen_pcrnet as tfp  # noqa: E402

STEP_BAR = tfp.STEP_BAR     # a whole step against the plain module (TF32 off): loss, rot_err and each sampler gradient
JOINT_BAR = 5e-2            # the joint step's gradients, as test_pcrnet_training's joint step (64-point clouds, unconditioned)


def case2(b, m0, m1, seed, kind="conditioned", device="cpu"):
    """pose_case with a template of m0 points and a source of m1: the source is the rotated template's first m1 points (or a random cloud
    of m1 when m1 > m0) plus noise."""
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(b, 7, generator=g)
    if kind == "conditioned":
        y[:, :4] = F.normalize(y[:, :4], dim=1) * (1 + 0.05 * torch.randn(b, 1, generator=g))
        y[:, 4:] *= 0.1
    gt = torch.cat([F.normalize(torch.randn(b, 4, generator=g), dim=1), 0.1 * torch.randn(b, 3, generator=g)], dim=1)
    p0 = torch.rand(b, m0, 3, generator=g) - 0.5
    src = p0[:, :m1] if m1 <= m0 else torch.rand(b, m1, 3, generator=g) - 0.5
    p1 = reg.QuaternionTransform(gt).rotate(src.contiguous()) + 0.01 * torch.randn(b, m1, 3, generator=g)
    return [t.to(device) for t in (y, p0, p1, gt)]


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("kind", ["random", "conditioned"])
@pytest.mark.parametrize("m0,m1", [(23, 9), (5, 17)])
def test_restatement_at_two_sizes_matches_float64_autograd(kind, m0, m1):
    y, p0, p1, gt = [t.double() for t in case2(3, m0, m1, 5, kind)]
    a = [t.clone().requires_grad_(True) for t in (y, p0, p1)]
    c = [t.clone().requires_grad_(True) for t in (y, p0, p1)]
    ta, _, i01, i10 = tfp.pose64(a[0], a[1], a[2], gt)
    assert i01.shape == (3, m1) and i10.shape == (3, m0)
    tc = tfp.torch_terms64(c[0], c[1], c[2], gt)
    assert torch.allclose(ta, tc, rtol=1e-11, atol=1e-13), (ta, tc)
    wts = torch.tensor([1.0, 0.7, 1.3, 0.0, 0.4], dtype=torch.float64)
    (ta * wts).sum().backward(); (tc * wts).sum().backward()
    for u, v in zip(a, c):
        assert torch.allclose(u.grad, v.grad, rtol=1e-9, atol=1e-12)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    from samplenet_b200 import _lib

    return _lib.lib()


def test_ex_envelope_and_workspace(lib):
    from samplenet_b200 import ops

    for b, m0, m1 in [(1, 1, 1), (32, 1024, 64), (3, 1, 1024), (256, 1024, 1024), (5, 777, 33)]:
        assert lib.snb200_pose_loss_ex_supported(b, m0, m1) == 1 and ops.pose_loss_supported(b, m0, m1)
        assert lib.snb200_pose_loss_ex_workspace_bytes(b, m0, m1) == lib.snb200_pose_loss_workspace_bytes(b, max(m0, m1)) == b * 8 * 4
        assert ops.pose_eval_supported(b, m0, m0, m1=m1, ms1=m1)
    for b, m0, m1 in [(0, 64, 64), (257, 64, 64), (32, 1025, 64), (32, 64, 1025), (32, 0, 64), (32, 64, 0)]:
        assert lib.snb200_pose_loss_ex_supported(b, m0, m1) == 0 and not ops.pose_loss_supported(b, m0, m1)
        assert lib.snb200_pose_loss_ex_workspace_bytes(b, m0, m1) == 0
    # the existing calls keep their meaning: one size for both clouds
    assert ops.pose_loss_supported(32, 64) and not ops.pose_loss_supported(32, 1025)
    assert ops.pose_eval_supported(4, 64, 1024) and not ops.pose_eval_supported(4, 64, 1024, ms1=1025) and not ops.pose_eval_supported(4, 64, m1=0)


def test_ex_rejections_launch_nothing(lib):
    from samplenet_b200 import _lib

    p = [tfp._ptr() for _ in range(12)]
    big = 1 << 40

    def err():
        return lib.snb200_last_error().decode()

    before = _lib.launch_count()
    assert lib.snb200_pose_loss_ex_forward(257, 64, 64, *p[:8], tfp._ptr(), big, tfp._ptr(), None) == -4
    assert "pose_loss_ex_forward: outside the pose loss's envelope" in err()
    assert lib.snb200_pose_loss_ex_forward(32, 1024, 1025, *p[:8], tfp._ptr(), big, tfp._ptr(), None) == -4 and "m1=1025" in err()
    assert lib.snb200_pose_loss_ex_forward(32, 0, 64, *p[:8], tfp._ptr(), big, tfp._ptr(), None) == -4
    assert lib.snb200_pose_loss_ex_forward(32, 1024, 64, *p[:8], None, big, tfp._ptr(), None) == -2
    assert lib.snb200_pose_loss_ex_forward(32, 1024, 64, *p[:8], tfp._ptr(), lib.snb200_pose_loss_ex_workspace_bytes(32, 1024, 64) - 1,
                                           tfp._ptr(), None) == -2
    assert lib.snb200_pose_loss_ex_forward(32, 1024, 64, *p[:8], tfp._ptr(), big, None, None) == -1 and "null pointer" in err()
    assert lib.snb200_pose_loss_ex_backward(32, 64, 1025, *p[:10], None) == -4 and "pose_loss_ex_backward" in err()
    assert lib.snb200_pose_loss_ex_backward(32, 1024, 64, *p[:9], None, None) == -1
    # pose_eval_ex: the pose pair, the sampled pair (only checked when given), and a half-given sampled pair
    ev = lambda b, m0, m1, ms0, ms1, p0s, p1s: lib.snb200_pose_eval_ex(b, m0, m1, *p[:4], ms0, ms1, p0s, p1s, p[4], p[5], None)  # noqa: E731
    assert ev(4, 1025, 64, 0, 0, None, None) == -4 and "pose_eval_ex: outside the envelope" in err()
    assert ev(4, 1024, 64, 1024, 1025, p[6], p[7]) == -4
    assert ev(4, 1024, 64, 0, 64, p[6], p[7]) == -4
    assert ev(4, 1024, 64, 1024, 64, p[6], None) == -1 and "both p0s and p1s" in err()
    assert _lib.launch_count() == before


# ------------------------------------------------------------------------------------------------------------------ GPU
sb = tfp.sb
_tf32_off = tfp._tf32_off


def _plain_forward(lib, y, p0, p1, igt):
    """The plain C entry (one size) through ctypes: (twist, idx01, idx10, terms)."""
    from samplenet_b200 import ops

    b, m = p0.shape[0], p0.shape[1]
    twist, terms = torch.empty(b, 7, device="cuda"), torch.empty(5, device="cuda")
    i01, i10 = torch.empty(b, m, device="cuda", dtype=torch.int32), torch.empty(b, m, device="cuda", dtype=torch.int32)
    wsb = int(lib.snb200_pose_loss_workspace_bytes(b, m))
    ws, ticket = torch.empty(wsb, device="cuda", dtype=torch.uint8), torch.zeros(1, device="cuda", dtype=torch.int32)
    assert lib.snb200_pose_loss_forward(b, m, y.data_ptr(), p0.data_ptr(), p1.data_ptr(), igt.data_ptr(), twist.data_ptr(), i01.data_ptr(),
                                        i10.data_ptr(), terms.data_ptr(), ws.data_ptr(), wsb, ticket.data_ptr(), ops._stream()) == 0
    return twist, i01, i10, terms


def _plain_backward(lib, y, p0, p1, igt, i01, i10, gt):
    from samplenet_b200 import ops

    gy, g0, g1 = torch.empty_like(y), torch.empty_like(p0), torch.empty_like(p1)
    assert lib.snb200_pose_loss_backward(p0.shape[0], p0.shape[1], y.data_ptr(), p0.data_ptr(), p1.data_ptr(), igt.data_ptr(), i01.data_ptr(),
                                         i10.data_ptr(), gt.data_ptr(), gy.data_ptr(), g0.data_ptr(), g1.data_ptr(), ops._stream()) == 0
    return gy, g0, g1


def _plain_eval(lib, y, p0, p1, igt, p0s=None, p1s=None):
    from samplenet_b200 import ops

    b, m = p0.shape[0], p0.shape[1]
    per_pair, twist = torch.empty(b, 6, device="cuda"), torch.empty(b, 7, device="cuda")
    ms = 0 if p0s is None else p0s.shape[1]
    assert lib.snb200_pose_eval(b, m, y.data_ptr(), p0.data_ptr(), p1.data_ptr(), igt.data_ptr(), ms, ops._p(p0s), ops._p(p1s),
                                per_pair.data_ptr(), twist.data_ptr(), ops._stream()) == 0
    return per_pair, twist


@pytest.mark.gpu
@pytest.mark.parametrize("b,m0,m1", [(32, 1024, 64), (5, 777, 33), (3, 1, 1024), (256, 1024, 1024)])
def test_pose_loss_ex_against_float64(sb, record_property, b, m0, m1):
    """Terms, twist, arg-mins and the three gradients against float64 on the kernel's arg-mins, at the bars of test_frozen_pcrnet; repeat
    runs bit-identical (tfp._check_pose)."""
    y, p0, p1, gt = case2(b, m0, m1, 1000 * b + m0 + m1, "conditioned", "cuda")
    twist, i01, i10, terms = tfp._check_pose(sb, record_property, y, p0, p1, gt, "b%d_m%d_%d" % (b, m0, m1))
    assert i01.shape == (b, m1) and i10.shape == (b, m0)
    e = reg.QuaternionTransform(twist).rotate(p0)
    _, j01, _, j10 = sb.ops.nn_distance_forward(p1, e)       # the arg-mins are ChamferDistance's on the rotated cloud the kernel forms
    same = float((i01 == j01).float().mean()), float((i10 == j10).float().mean())
    assert same[0] > 0.9999 and same[1] > 0.9999, same


@pytest.mark.gpu
def test_pose_loss_ex_ties_go_to_the_lowest_index(sb):
    """An identity estimate with exact duplicates: template points 5, 40 and 80 equal, the source the template's first 64 points."""
    y, p0, _, gt = case2(4, 100, 64, 9, "conditioned", "cuda")
    y[:, :4] = torch.tensor([1.0, 0.0, 0.0, 0.0], device="cuda")
    p0[:, 40] = p0[:, 5]; p0[:, 80] = p0[:, 5]
    p1 = p0[:, :64].clone()
    _, i01, i10, terms = sb.ops.pose_loss_forward(y, p0, p1, gt)
    want01 = torch.arange(64, device="cuda", dtype=torch.int32).repeat(4, 1); want01[:, 40] = 5
    assert torch.equal(i01, want01)
    d = ((p0.double().cpu()[:, :, None, :] - p1.double().cpu()[:, None, :, :]) ** 2).sum(-1)     # [b, j (template), i (source)]
    want10 = d.argmin(dim=2).int(); want10[:, :64] = want01.cpu(); want10[:, 80] = 5
    assert torch.equal(i10.cpu(), want10)
    assert float(terms[0]) > 0
    gy, g0, g1 = sb.ops.pose_loss_backward(y, p0, p1, gt, i01, i10, torch.tensor([1.0, 0, 0, 0, 0], device="cuda"))
    assert bool(torch.isfinite(g0).all()) and bool(torch.isfinite(g1).all())


@pytest.mark.gpu
@pytest.mark.parametrize("b,m", [(1, 1), (32, 64), (7, 1024), (256, 1024)])
def test_ex_at_equal_sizes_is_the_plain_entries_bit_for_bit(sb, b, m):
    lib = sb._lib.lib()
    y, p0, p1, gt = tfp.pose_case(b, m, 77 + b + m, "conditioned", "cuda")
    fwd_ex, fwd = sb.ops.pose_loss_forward(y, p0, p1, gt), _plain_forward(lib, y, p0, p1, gt)
    assert all(torch.equal(a, c) for a, c in zip(fwd_ex, fwd))
    wts = torch.tensor([1.0, 0.7, 1.3, 3.0, 0.4], device="cuda")
    bwd_ex, bwd = sb.ops.pose_loss_backward(y, p0, p1, gt, fwd[1], fwd[2], wts), _plain_backward(lib, y, p0, p1, gt, fwd[1], fwd[2], wts)
    assert all(torch.equal(a, c) for a, c in zip(bwd_ex, bwd))
    ms = max(1, m // 2)
    p0s, p1s = p0[:, :ms].contiguous(), p1[:, -ms:].contiguous()
    for pair in ((None, None), (p0s, p1s)):
        ev_ex, ev = sb.ops.pose_eval(y, p0, p1, gt, *pair), _plain_eval(lib, y, p0, p1, gt, *pair)
        assert all(torch.equal(a, c) for a, c in zip(ev_ex, ev))


@pytest.mark.gpu
@pytest.mark.parametrize("b,m0,m1,ms0,ms1", [(32, 1024, 64, 1024, 64), (5, 33, 777, 0, 0), (1, 1, 1024, 17, 1000), (3, 64, 1024, 1024, 1)])
def test_ex_entries_write_only_their_buffers(sb, b, m0, m1, ms0, ms1):
    from test_write_sets import Arena, _addr, _vp, assert_clean, run_checked

    lib = sb._lib.lib()
    arena = Arena(256 << 20)
    g = torch.Generator().manual_seed(b + m0 + m1)
    q = torch.randn(b, 4, generator=g)
    y = arena.carve("y", (b, 7), fill=torch.cat([q * 1.3, 0.1 * torch.randn(b, 3, generator=g)], 1))
    igt = arena.carve("igt", (b, 7), fill=torch.cat([q / q.norm(dim=1, keepdim=True), 0.1 * torch.randn(b, 3, generator=g)], 1))
    p0 = arena.carve("p0", (b, m0, 3), fill=torch.rand(b, m0, 3, generator=g) - 0.5)
    p1 = arena.carve("p1", (b, m1, 3), fill=torch.rand(b, m1, 3, generator=g) - 0.5)
    wsb = int(lib.snb200_pose_loss_ex_workspace_bytes(b, m0, m1))
    twist, terms = arena.carve("twist", (b, 7)), arena.carve("terms", (5,))
    idx01, idx10 = arena.carve("idx01", (b, m1), dtype=torch.int32), arena.carve("idx10", (b, m0), dtype=torch.int32)
    ws = arena.carve("workspace", (wsb,), dtype=torch.uint8)
    ticket = arena.carve("ticket", (1,), dtype=torch.int32, fill=torch.zeros(1, dtype=torch.int32))
    rc = []
    rep = run_checked(arena, "pose_loss_ex_forward", lambda: rc.append(lib.snb200_pose_loss_ex_forward(
        b, m0, m1, y.data_ptr(), p0.data_ptr(), p1.data_ptr(), igt.data_ptr(), twist.data_ptr(), idx01.data_ptr(), idx10.data_ptr(),
        terms.data_ptr(), _addr(ws), wsb, ticket.data_ptr(), None)), [ws, ticket], full=[twist, idx01, idx10, terms], zero=[(ticket, "ticket")])
    gt = arena.carve("grad_terms", (5,), fill=torch.tensor([1.0, 0.5, 0.25, 3.0, 2.0]))
    gy, g0, g1 = arena.carve("grad_y", (b, 7)), arena.carve("grad_p0", (b, m0, 3)), arena.carve("grad_p1", (b, m1, 3))
    rep += run_checked(arena, "pose_loss_ex_backward", lambda: rc.append(lib.snb200_pose_loss_ex_backward(
        b, m0, m1, y.data_ptr(), p0.data_ptr(), p1.data_ptr(), igt.data_ptr(), idx01.data_ptr(), idx10.data_ptr(), gt.data_ptr(), gy.data_ptr(),
        g0.data_ptr(), g1.data_ptr(), None)), full=[gy, g0, g1])
    p0s = arena.carve("p0s", (b, ms0, 3), fill=torch.rand(b, ms0, 3, generator=g) - 0.5) if ms0 else None
    p1s = arena.carve("p1s", (b, ms1, 3), fill=torch.rand(b, ms1, 3, generator=g) - 0.5) if ms1 else None
    per_pair, etw = arena.carve("per_pair", (b, 6)), arena.carve("eval_twist", (b, 7))
    rep += run_checked(arena, "pose_eval_ex", lambda: rc.append(lib.snb200_pose_eval_ex(
        b, m0, m1, y.data_ptr(), p0.data_ptr(), p1.data_ptr(), igt.data_ptr(), ms0, ms1, _vp(p0s), _vp(p1s), per_pair.data_ptr(), etw.data_ptr(),
        None)), full=[per_pair, etw])
    assert rc == [0, 0, 0], lib.snb200_last_error()
    assert_clean(rep)
    assert bool((per_pair[:, 5] != 0).all()) if ms0 else bool((per_pair[:, 5] == 0).all())


@pytest.mark.gpu
def test_pose_eval_ex_against_the_per_record_loop_and_the_fixture(sb, golden_dir):
    """Per pair as test_1's record loop computes it (compute_pcrnet_loss of the plain torch ops on a 1024-point template and a 64-point
    source, then compute_sampling_consistency between them), and the reference's consistency of registration_step_c1.npz."""
    b = 8
    y, p0, p1, gt = case2(b, 1024, 64, 31, "conditioned", "cuda")
    per_pair, _ = sb.ops.pose_eval(y, p0, p1, gt, p0, p1)
    step = reg.RegistrationStep(num_sampled_clouds=1)

    class _Fixed(torch.nn.Module):         # a "model" whose output is y: compute_pcrnet_loss's torch ops on it
        def __init__(self, y):
            super().__init__()
            self.y = y

        def forward(self, x0, x1):
            return torch.cat([F.normalize(self.y[:, :4], dim=1), self.y[:, 4:]], dim=1), self.y[:, :4]
    for i in range(b):
        one = (p0[i:i + 1], p1[i:i + 1], {"vec": gt[i:i + 1], "inversion": torch.tensor([False])})
        _, info = step.compute_pcrnet_loss(_Fixed(y[i:i + 1]), one, "cuda")
        want = torch.stack([info["chamfer_loss"], info["qnorm_loss"], info["norm_err"], info["rot_err"] * np.pi / 180, info["trans_err"],
                            step.compute_sampling_consistency(one, "cuda")])
        tol = torch.tensor([1e-5, 1e-5, 1e-5, 2e-3, 1e-5, 1e-5], device="cuda")
        assert bool(((per_pair[i] - want).abs() <= tol * (want.abs() + 1e-3)).all()), (i, per_pair[i], want)
    z = np.load(os.path.join(golden_dir, "registration_step_c1.npz"))
    p0s, p1s, igt = (torch.from_numpy(z[k]).cuda() for k in ("p0_out", "p1_out", "igt_vec"))
    assert p0s.shape[1] == 1024 and p1s.shape[1] == 64
    col, _ = sb.ops.pose_eval(igt, p0s, p1s, igt, p0s, p1s)
    np.testing.assert_allclose(float(col[:, 5].double().mean()), float(z["consistency"]), rtol=5e-4)


def _step_data(b, n, seed=100):
    g = torch.Generator().manual_seed(seed)
    p0 = (torch.rand(b, n, 3, generator=g) - 0.5).cuda()
    vec = torch.cat([F.normalize(torch.randn(b, 4, generator=g), dim=1), torch.zeros(b, 3)], dim=1).cuda()
    return p0, reg.QuaternionTransform(vec).rotate(p0), {"vec": vec, "inversion": torch.tensor([False])}


def _no_module_forward(monkeypatch):
    def refuse(self, *a):
        raise AssertionError("the wrapped PCRNet's forward ran: the step left the CUDA path")
    monkeypatch.setattr(reg.PCRNet, "forward", refuse)


@pytest.mark.gpu
def test_whole_train_step_at_one_sampled_cloud_against_the_plain_module(sb, record_property, _tf32_off, monkeypatch):
    """B = 32, N = 1024 -> 64, frozen_task=True against the plain module: loss, rot_err and every sampler gradient.  The frozen run never
    calls the wrapped module's forward."""
    data = _step_data(32, 1024)
    res = []
    for frozen in (False, True):
        act = reg.RegistrationStep(num_sampled_clouds=1)
        torch.manual_seed(0)
        model = act.create_model(frozen_task=frozen).cuda()
        model.sampler.train()
        opt = torch.optim.SGD([p for p in model.sampler.parameters() if p.requires_grad], lr=0.0)
        with monkeypatch.context() as mp:
            if frozen:
                _no_module_forward(mp)
            loss, rot, _ = act.train_step(model, data, opt, "cuda")
        res.append((float(loss), float(rot), {n: p.grad.double().clone() for n, p in model.sampler.named_parameters() if p.grad is not None}))
    (l0, r0, g0), (l1, r1, g1) = res
    e_loss, e_rot = abs(l1 - l0) / abs(l0), abs(r1 - r0) / abs(r0)
    assert g0.keys() == g1.keys() and len(g0) > 10
    top = max(float(g.abs().max()) for g in g0.values())       # as test_frozen_pcrnet's whole step: vanishing gradients against the largest
    per = sorted(((float((g1[n] - g0[n]).abs().max()) / (float(g0[n].abs().max()) if float(g0[n].abs().max()) >= 1e-3 * top else top), n)
                  for n in g0), reverse=True)
    record_property("step1_loss_err", e_loss); record_property("step1_rot_err", e_rot); record_property("step1_grad_err", per[0][0])
    assert e_loss < STEP_BAR and e_rot < STEP_BAR and per[0][0] < STEP_BAR, (e_loss, e_rot, per[:5])


@pytest.mark.gpu
def test_joint_step_at_one_sampled_cloud_against_the_plain_module(sb, record_property, _tf32_off, monkeypatch):
    """cuda_task=True with train_pcrnet and train_samplenet: all 22 PCRNet gradients and the sampler's, test_pcrnet_training's
    normalisation and bars."""
    from test_pcrnet_training import _grad_errs

    data = _step_data(32, 1024, seed=7)
    res = {}
    for cuda in (False, True):
        act = reg.RegistrationStep(num_out_points=64, num_sampled_clouds=1, train_pcrnet=True, train_samplenet=True)
        torch.manual_seed(0)
        model = act.create_model(cuda_task=cuda).cuda()
        opt = torch.optim.Adam(filter(lambda p: p.requires_grad, model.parameters()), lr=0.0)
        with monkeypatch.context() as mp:
            if cuda:
                _no_module_forward(mp)
            loss, _, _ = act.train_step(model, data, opt, "cuda")
        net = model.net if cuda else model
        res[cuda] = (float(loss), {n: p.grad.double().clone() for n, p in net.named_parameters() if p.grad is not None})
    (l0, g0), (l1, g1) = res[False], res[True]
    assert sum(n.startswith("sampler.") for n in g0) > 10 and sum(not n.startswith("sampler.") for n in g0) == 22
    errs = _grad_errs(g0, g1)
    top = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    record_property("joint1_loss_err", abs(l1 - l0) / abs(l0)); record_property("joint1_grad_err", top[0][1])
    assert abs(l1 - l0) / abs(l0) < STEP_BAR and top[0][1] < JOINT_BAR, (l0, l1, top)


@pytest.mark.gpu
@pytest.mark.parametrize("trainable", [False, True])
def test_chunks_of_two_sizes_beyond_32_pairs(sb, trainable):
    """48 pairs of a 256-point template and a 64-point source: bit for bit the concatenation of 32 + 16, outputs and cloud gradients (and,
    trained, the parameter gradients of two runs)."""
    torch.manual_seed(6)
    net = reg.PCRNet(input_shape="bnc").cuda()
    if trainable:
        w = reg.CudaPCRNet(net)
    else:
        net.requires_grad_(False).eval()
        w = reg.FrozenPCRNet(net)
    g = torch.Generator().manual_seed(3)
    x0, x1 = (torch.rand(48, 256, 3, generator=g) - 0.5).cuda(), (torch.rand(48, 64, 3, generator=g) - 0.5).cuda()

    def run(parts):
        outs, grads = [], []
        for s, e in parts:
            a0, a1 = x0[s:e].clone().requires_grad_(True), x1[s:e].clone().requires_grad_(True)
            tw, pre = w(a0, a1)
            (pre.square().sum() + tw[:, 4:].sum()).backward()
            outs.append((tw.detach(), pre.detach())); grads.append((a0.grad, a1.grad))
        return [torch.cat([o[k] for o in outs]) for k in range(2)] + [torch.cat([gr[k] for gr in grads]) for k in range(2)]
    whole, halves = run([(0, 48)]), run([(0, 32), (32, 48)])
    assert all(torch.equal(a, c) for a, c in zip(whole, halves))
    if trainable:       # run to run: the parameter gradients of the two encoder calls are added in a fixed order
        net.zero_grad(set_to_none=True)
        run([(0, 48)])
        first = [p.grad.clone() for p in net.parameters()]
        net.zero_grad(set_to_none=True)
        run([(0, 48)])
        assert all(torch.equal(a, p.grad) for a, p in zip(first, net.parameters()))


@pytest.mark.gpu
@pytest.mark.parametrize("sampler", ["samplenet", "fps", "random"])
def test_test_1_at_one_sampled_cloud(sb, sampler, monkeypatch):
    """Batches of 20 through FrozenPCRNet and one pose_eval launch against the per-record torch loop (the plain module, batch 1), with the
    samplenet sampler in eval mode; "fps" and "random" draw per call, so they run and are not compared."""
    torch.manual_seed(0)
    step = reg.RegistrationStep(num_out_points=64, sampler=sampler, num_sampled_clouds=1)
    model = step.create_model(frozen_task=True).cuda()
    g = torch.Generator().manual_seed(4)
    n = 40
    q = F.normalize(torch.randn(n, 4, generator=g), dim=1)
    vec = torch.cat([q, 0.1 * torch.randn(n, 3, generator=g)], dim=1).cuda()
    p0 = (torch.rand(n, 1024, 3, generator=g) * 2 - 1).cuda()
    p1 = reg.qrot(q.cuda()[:, None, :].expand(-1, 1024, -1).contiguous(), p0)

    def batches(bs):
        return [(p0[s:s + bs], p1[s:s + bs], {"vec": vec[s:s + bs], "inversion": torch.tensor([False])}) for s in range(0, n, bs)]
    calls = []
    monkeypatch.setattr(sb.ops, "pose_eval", lambda *a, _f=sb.ops.pose_eval: calls.append(a[1].shape[1:2] + a[2].shape[1:2]) or _f(*a))
    with monkeypatch.context() as mp:
        _no_module_forward(mp)
        got = step.test_1(model, batches(20), "cuda")
    assert calls == [(1024, 64)] * 2
    assert got["rotation_errors"].shape == (n,) and np.isfinite(got["consistency_errors"]).all()
    if sampler != "samplenet":
        return
    one = step.test_1(model.net, batches(1), "cuda")
    for key in ("rotation_errors", "trans_errs", "consistency_errors"):      # 3xTF32 tensor-core layers against cuBLAS fp32, as test_evaluation
        assert np.allclose(got[key], one[key], rtol=5e-3, atol=5e-3), (key, np.abs(got[key] - one[key]).max())
