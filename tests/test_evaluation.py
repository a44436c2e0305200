"""The evaluators (samplenet_b200/evaluation.py, RegistrationStep.eval_1 / test_1) and their two kernels, pose_eval and chamfer_per_cloud.

Host tests: the ABI symbols and signatures, the envelope predicates, the metric restatements (precision curve / AUC, per-class accuracy,
NRE) against numpy loops written from the reference's lines, mode restoration.  GPU tests: the kernels against float64 torch and against
the ops they restate, run-to-run bit identity, rejections outside the envelope, and every evaluator against its one-record-at-a-time form.
"""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import samplenet_b200 as sb
from samplenet_b200 import _lib, evaluation as ev, ops, registration as reg, sputils, tasknets, trainers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------- host
def test_abi_symbols_and_signatures():
    header = open(os.path.join(ROOT, "include", "samplenet_b200.h")).read()
    flat = re.sub(r"\s+", " ", header)
    want = {
        "snb200_pose_eval_supported": "int snb200_pose_eval_supported(int b, int m, int ms);",
        "snb200_pose_eval": "int snb200_pose_eval(int b, int m, const float *y, const float *p0, const float *p1, const float *igt, int ms, "
                            "const float *p0s, const float *p1s, float *per_pair, float *twist, snb200_stream_t stream);",
        "snb200_chamfer_per_cloud_workspace_bytes": "size_t snb200_chamfer_per_cloud_workspace_bytes(int b, int n, int m);",
        "snb200_chamfer_per_cloud": "int snb200_chamfer_per_cloud(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, float *sums, "
                                    "void *workspace, size_t workspace_bytes, snb200_stream_t stream);",
    }
    for name, decl in want.items():
        assert decl in flat, name
        assert name in _lib.exported_symbols()
        assert len(_lib._SIGNATURES[name][1]) == decl.count(",") + 1
    lib = _lib.lib()     # loading binds every symbol: a missing one raises
    assert lib.snb200_pose_eval_supported(1, 1, 1) == 1 and lib.snb200_pose_eval_supported(256, 1024, 1024) == 1
    for bad in ((0, 64, 64), (257, 64, 64), (4, 0, 64), (4, 1025, 64), (4, 64, 0), (4, 64, 1025)):
        assert lib.snb200_pose_eval_supported(*bad) == 0, bad
    assert lib.snb200_chamfer_per_cloud_workspace_bytes(400, 2048, 2048) >= 400 * 2 * 4
    assert lib.snb200_chamfer_per_cloud_workspace_bytes(0, 8, 8) == 0


def test_envelope_predicates_and_host_rejections():
    assert ops.pose_eval_supported(1, 1) and ops.pose_eval_supported(256, 1024, 1024)
    assert not ops.pose_eval_supported(257, 64) and not ops.pose_eval_supported(4, 64, 1025) and not ops.pose_eval_supported(0, 64)
    lib = _lib.lib()
    one = ctypes.c_void_p(16)    # never dereferenced: the calls below are rejected before any launch
    before = _lib.launch_count()
    assert lib.snb200_pose_eval(257, 64, one, one, one, one, 0, None, None, one, one, None) != 0
    assert lib.snb200_pose_eval(4, 64, one, one, one, one, 2000, one, one, one, one, None) != 0
    assert lib.snb200_pose_eval(4, 64, one, one, one, one, 64, one, None, one, one, None) != 0
    assert lib.snb200_chamfer_per_cloud(6, 8, one, 8, one, 4, one, one, 1 << 20, None) != 0      # 4 does not divide 6
    assert lib.snb200_chamfer_per_cloud(6, 8, one, 8, one, 3, one, None, 0, None) != 0           # no workspace
    assert _lib.launch_count() == before
    with pytest.raises(RuntimeError):
        ops.pose_eval(torch.zeros(2, 7), torch.zeros(2, 4, 3), torch.zeros(2, 4, 3), torch.zeros(2, 7))     # CPU tensors
    with pytest.raises(RuntimeError):
        ops.chamfer_per_cloud(torch.zeros(2, 4, 3), torch.zeros(2, 4, 3))


def test_precision_curve_against_reference_loop():
    rng = np.random.RandomState(0)
    rotation_errors = np.concatenate([rng.rand(50) * 200, [0.0, 0.5, 179.5, 180.0]])
    n_samples = len(rotation_errors)            # main.py:461-477
    x = np.arange(0.0, 180.0, 0.5)
    y = np.zeros(len(x))
    for idx, err in enumerate(x):
        y[idx] = np.sum(rotation_errors <= err) / n_samples
    auc = np.sum(y) / len(x)
    gx, gy, gauc = ev.precision_curve(rotation_errors)
    assert np.array_equal(gx, x) and np.array_equal(gy, y) and gauc == auc


def _reference_class_accuracy(pred_val, labels, num_classes):
    total_seen_class = [0] * num_classes        # evaluate_samplenet.py:236-258
    total_correct_class = [0] * num_classes
    pred = np.argmax(pred_val, 1)
    for i in range(len(labels)):
        l = labels[i]
        total_seen_class[l] += 1
        total_correct_class[l] += pred[i] == l
    return np.sum(pred == labels) / float(len(labels)), np.array(total_correct_class) / np.array(total_seen_class, dtype=float)


def test_classification_metrics_against_reference_loop():
    g = torch.Generator().manual_seed(1)
    logits = torch.randn(200, 7, generator=g)
    labels = torch.randint(0, 7, (200,), generator=g)
    pred, seen, correct = ev.classification_counts(logits, labels)
    acc, per_class, avg = ev.class_accuracies(seen.numpy(), correct.numpy())
    racc, rper = _reference_class_accuracy(logits.numpy(), labels.numpy(), 7)
    assert np.array_equal(pred.numpy(), np.argmax(logits.numpy(), 1))
    assert acc == racc and np.array_equal(per_class, rper) and avg == np.mean(rper)
    # a class nobody belongs to: NaN there and in the mean, as the reference's division
    _, seen, correct = ev.classification_counts(logits, labels, num_classes=9)
    _, per_class, avg = ev.class_accuracies(seen.numpy(), correct.numpy())
    assert np.isnan(per_class[7:]).all() and np.isnan(avg)


def test_nre_and_eval_mode_restore():
    a, b = np.array([1.0, 3.0]), np.array([2.0, 2.0])
    assert np.array_equal(ev.nre(a, b), a / b) and torch.equal(ev.nre(torch.tensor(a), torch.tensor(b)), torch.tensor(a / b))
    net = torch.nn.Sequential(torch.nn.Linear(2, 2), torch.nn.BatchNorm1d(2), torch.nn.Sequential(torch.nn.Dropout()))
    net.train()
    net[1].eval()            # a mixed state comes back as it was, module by module
    with ev.eval_mode(net, None):
        assert not any(m.training for m in net.modules()) and not torch.is_grad_enabled()
    assert net.training and net[0].training and not net[1].training and net[2].training and net[2][0].training
    with pytest.raises(KeyError):
        with ev.eval_mode(net):
            raise KeyError("restored on the way out of an exception too")
    assert net.training and not net[1].training


# ----------------------------------------------------------------------------------------------------- fixtures
def _dev():
    return torch.device("cuda")


def _rand_quat(g, b, near_identity=False):
    q = torch.randn(b, 4, generator=g)
    if near_identity:
        q = torch.tensor([1.0, 0, 0, 0]) + 1e-3 * q
    return q / q.norm(dim=1, keepdim=True)


def _pose_case(seed, b, m, ms=None, near_identity=False):
    g = torch.Generator().manual_seed(seed)
    qg = _rand_quat(g, b, near_identity)
    igt = torch.cat([qg, 0.3 * torch.randn(b, 3, generator=g)], dim=1)
    p0 = torch.rand(b, m, 3, generator=g) * 2 - 1
    p1 = reg.qrot(qg[:, None, :].expand(-1, m, -1).contiguous(), p0) + 0.01 * torch.randn(b, m, 3, generator=g)
    scale = 0.5 + torch.rand(b, 1, generator=g)       # the raw quaternion is not of unit length
    y = torch.cat([(qg + (1e-3 if near_identity else 0.2) * torch.randn(b, 4, generator=g)) * scale, igt[:, 4:] + 0.1 * torch.randn(b, 3, generator=g)], dim=1)
    ms = m if ms is None else ms
    p0s, p1s = p0[:, torch.randperm(m, generator=g)[:ms]].contiguous(), p1[:, torch.randperm(m, generator=g)[:ms]].contiguous()
    return [t.to(_dev()) for t in (y, p0, p1, igt, p0s, p1s)]


def _chamfer64(a, b):
    d = ((a[:, :, None, :].double() - b[:, None, :, :].double()) ** 2).sum(-1)
    return d.min(dim=2)[0].mean(dim=1), d.min(dim=1)[0].mean(dim=1)


def _pose_reference64(y, p0, p1, igt, p0s, p1s):
    """Per pair, in float64, with registration.py's quaternion maths."""
    y, p0, p1, igt, p0s, p1s = [t.double().cpu() for t in (y, p0, p1, igt, p0s, p1s)]
    q = y[:, :4] / y[:, :4].norm(dim=1, keepdim=True).clamp_min(1e-12)
    est, gt = reg.QuaternionTransform(torch.cat([q, y[:, 4:]], dim=1)), reg.QuaternionTransform(igt)
    c01, c10 = _chamfer64(p1, est.rotate(p0))
    R1 = reg.quaternion_to_rotation_matrix(q[:, [1, 2, 3, 0]])
    R2 = reg.quaternion_to_rotation_matrix(igt[:, [1, 2, 3, 0]])
    eye = torch.eye(3, dtype=torch.float64)
    s01, s10 = _chamfer64(p0s, gt.inverse().rotate(p1s))
    return torch.stack([c01 + c10, ((y[:, :4] ** 2).sum(1) - 1) ** 2, ((R1 @ R2.transpose(1, 2) - eye) ** 2).sum(dim=(1, 2)),
                        2 * torch.acos((2 * (q * igt[:, :4]).sum(1) ** 2 - 1).clamp(-1, 1)), (y[:, 4:] - igt[:, 4:]).abs().mean(1), s01 + s10], dim=1)


# ----------------------------------------------------------------------------------------------------- pose_eval
@gpu
@pytest.mark.parametrize("b,m,ms,near", [(1, 1, 1, False), (32, 64, 64, False), (32, 64, 17, True), (3, 1000, 1024 - 24, False), (256, 64, 64, False),
                                         (2, 1024, 1024, True)])
def test_pose_eval_against_float64_and_pose_loss(b, m, ms, near):
    y, p0, p1, igt, p0s, p1s = _pose_case(10 + b + m, b, m, ms, near)
    per_pair, twist = ops.pose_eval(y, p0, p1, igt, p0s, p1s)
    ref = _pose_reference64(y, p0, p1, igt, p0s, p1s)
    got = per_pair.double().cpu()
    # fp32 against float64: 1e-5 relative on the sums of squares; acos near 1 loses half the digits (rot_err of a near-identity error)
    for col, name in enumerate(ops.POSE_EVAL_COLUMNS):
        tol = dict(rtol=2e-3, atol=2e-3) if name == "rot_err" else dict(rtol=1e-4, atol=1e-6)
        assert torch.allclose(got[:, col], ref[:, col], **tol), (name, (got[:, col] - ref[:, col]).abs().max())
    # the forward's batch means are the means of the per-pair columns: same arithmetic per pair, only the last mean is rounded differently
    twist_f, _, _, terms = ops.pose_loss_forward(y, p0, p1, igt)
    assert torch.equal(twist, twist_f)
    assert torch.allclose(per_pair[:, :5].double().mean(dim=0), terms.double(), rtol=1e-5, atol=1e-7)
    if b == 1:      # one pair: nothing to average, bit equality except the Chamfer term's two divisions
        assert torch.equal(per_pair[0, 1:5], terms[1:5])
    # run to run, and without the sampled pair
    again, _ = ops.pose_eval(y, p0, p1, igt, p0s, p1s)
    assert torch.equal(per_pair, again)
    bare, _ = ops.pose_eval(y, p0, p1, igt)
    assert torch.equal(bare[:, :5], per_pair[:, :5]) and bool((bare[:, 5] == 0).all())
    # a pair's row does not depend on the batch around it
    k = b // 2
    alone, _ = ops.pose_eval(y[k:k + 1], p0[k:k + 1], p1[k:k + 1], igt[k:k + 1], p0s[k:k + 1], p1s[k:k + 1])
    assert torch.equal(alone[0], per_pair[k])


@gpu
def test_pose_eval_consistency_against_compute_sampling_consistency():
    b, m = 8, 64
    y, p0, p1, igt, p0s, p1s = _pose_case(3, b, m)
    per_pair, _ = ops.pose_eval(y, p0, p1, igt, p0s, p1s)
    step = reg.RegistrationStep()
    for i in range(b):
        one = (p0s[i:i + 1], p1s[i:i + 1], {"vec": igt[i:i + 1], "inversion": torch.tensor([False])})
        want = step.compute_sampling_consistency(one, _dev())
        assert torch.allclose(per_pair[i, 5], want, rtol=1e-5, atol=1e-8)


@gpu
def test_pose_eval_rejections_launch_nothing():
    y, p0, p1, igt, p0s, p1s = _pose_case(4, 4, 32)
    before = _lib.launch_count()
    big = torch.zeros(4, 1025, 3, device=_dev())
    with pytest.raises(ValueError):
        ops.pose_eval(y, big, big, igt)
    with pytest.raises(ValueError):
        ops.pose_eval(y, p0, p1, igt, big, big)
    with pytest.raises(ValueError):
        ops.pose_eval(y, p0, p1, igt, p0s, None)
    with pytest.raises(ValueError):
        ops.pose_eval(y[:3], p0, p1, igt)
    with pytest.raises(RuntimeError):
        ops.pose_eval(y.clone().requires_grad_(True), p0, p1, igt)
    many = torch.zeros(257, 7, device=_dev())
    with pytest.raises(ValueError):
        ops.pose_eval(many, torch.zeros(257, 8, 3, device=_dev()), torch.zeros(257, 8, 3, device=_dev()), many)
    assert _lib.launch_count() == before
    with torch.no_grad():
        ops.pose_eval(y.clone().requires_grad_(True), p0, p1, igt)


# ----------------------------------------------------------------------------------------------------- chamfer_per_cloud
@gpu
@pytest.mark.parametrize("b,n,m", [(4, 64, 1024), (16, 2048, 2048), (3, 77, 1531), (2, 1, 5), (1, 5000, 333)])
def test_chamfer_per_cloud_against_nn_distance_and_float64(b, n, m):
    g = torch.Generator().manual_seed(b * 7 + n)
    x1, x2 = torch.randn(b, n, 3, generator=g).to(_dev()), torch.randn(b, m, 3, generator=g).to(_dev())
    before = _lib.launch_count()
    sums = ops.chamfer_per_cloud(x1, x2)
    assert _lib.launch_count() == before + 2
    d1, _, d2, _ = ops.nn_distance_forward(x1, x2)
    # the same distances; only the order of the fp32 sum differs
    assert torch.allclose(sums[:, 0], d1.mean(1), rtol=2e-6 * math.sqrt(n) + 1e-6) and torch.allclose(sums[:, 1], d2.mean(1), rtol=2e-6 * math.sqrt(m) + 1e-6)
    assert torch.allclose(sums[:, 0].double(), d1.double().mean(1), rtol=1e-5) and torch.allclose(sums[:, 1].double(), d2.double().mean(1), rtol=1e-5)
    for i in range(min(b, 3)):      # float64, a cloud at a time (the (2048, 2048) distance matrix is 100 MB)
        r1, r2 = _chamfer64(x1[i:i + 1], x2[i:i + 1])
        assert torch.allclose(sums[i].double(), torch.cat([r1, r2]), rtol=1e-4, atol=1e-7)
    assert torch.equal(sums, ops.chamfer_per_cloud(x1, x2))


@gpu
@pytest.mark.parametrize("p,b2,n,m", [(8, 50, 2048, 2048), (3, 5, 100, 333)])
def test_chamfer_per_cloud_repeated_reference(p, b2, n, m):
    g = torch.Generator().manual_seed(p)
    x1, x2 = torch.randn(p * b2, n, 3, generator=g).to(_dev()), torch.randn(b2, m, 3, generator=g).to(_dev())
    assert torch.equal(ops.chamfer_per_cloud(x1, x2), ops.chamfer_per_cloud(x1, x2.repeat(p, 1, 1)))
    with pytest.raises(ValueError):
        ops.chamfer_per_cloud(x1[:-1], x2)
    with pytest.raises(RuntimeError):
        ops.chamfer_per_cloud(x1.clone().requires_grad_(True), x2)


# ----------------------------------------------------------------------------------------------------- registration
def _reg_batches(n_records, batch, n_points=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    qg = _rand_quat(g, n_records)
    vec = torch.cat([qg, torch.zeros(n_records, 3)], dim=1)
    p0 = torch.rand(n_records, n_points, 3, generator=g) * 2 - 1
    p1 = reg.qrot(qg[:, None, :].expand(-1, n_points, -1).contiguous(), p0)
    return [(p0[s:s + batch].to(_dev()), p1[s:s + batch].to(_dev()), {"vec": vec[s:s + batch].to(_dev()), "inversion": torch.tensor([False])})
            for s in range(0, n_records, batch)]


def _reg_model(sampler, frozen, seed=0):
    torch.manual_seed(seed)
    step = reg.RegistrationStep(num_out_points=32, sampler=sampler, num_sampled_clouds=2)
    model = step.create_model(frozen_task=frozen).to(_dev())
    net = model.net if frozen else model
    for mod in net.modules():      # running statistics that are not the identity
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.running_mean.normal_(0, 0.1); mod.running_var.uniform_(0.5, 1.5)
    return step, model


class _Readbacks:
    """Counts the device-to-host reads of CUDA tensors that Python can see: .item(), .cpu(), .tolist(), .numpy() via .cpu()."""

    def __enter__(self):
        self.count, self._saved = 0, {}
        for name in ("item", "cpu", "tolist"):
            orig = getattr(torch.Tensor, name)
            self._saved[name] = orig

            def patched(t, *a, _orig=orig, **k):
                if t.is_cuda:
                    self.count += 1
                return _orig(t, *a, **k)
            setattr(torch.Tensor, name, patched)
        return self

    def __exit__(self, *exc):
        for name, orig in self._saved.items():
            setattr(torch.Tensor, name, orig)


@gpu
@pytest.mark.parametrize("frozen", [True, False])
@pytest.mark.parametrize("sampler", ["samplenet", "none"])
def test_test_1_batched_equals_record_by_record(sampler, frozen):
    step, model = _reg_model(sampler, frozen)
    n = 64 if frozen else 16
    with _Readbacks() as rb:
        got = step.test_1(model, _reg_batches(n, 32 if frozen else 8), _dev())
    assert rb.count == 1, "one host read-back per call"
    one = step.test_1(model, _reg_batches(n, 1), _dev())
    assert got["rotation_errors"].shape == (n,)
    for key in ("rotation_errors", "trans_errs", "consistency_errors"):
        # the frozen encoder and MLP are per-row kernels and pose_eval is per pair; the torch path's cuBLAS picks its algorithm by batch size
        assert np.allclose(got[key], one[key], rtol=1e-4, atol=1e-4), (key, np.abs(got[key] - one[key]).max())
    x, yy, auc = ev.precision_curve(got["rotation_errors"])
    assert np.array_equal(got["precision_y"], yy) and got["auc"] == auc and np.array_equal(got["precision_x"], np.arange(0.0, 180.0, 0.5))
    assert got["mean_rotation_error"] == np.mean(got["rotation_errors"]) and got["std_consistency_error"] == np.std(got["consistency_errors"])
    assert np.isfinite(got["rotation_errors"]).all() and (got["rotation_errors"] >= 0).all() and (got["rotation_errors"] <= 360).all()


@gpu
def test_test_1_frozen_against_plain_model():
    step, model = _reg_model("samplenet", True)
    batches = _reg_batches(32, 32)
    frozen, plain = step.test_1(model, batches, _dev()), step.test_1(model.net, batches, _dev())
    for key in ("rotation_errors", "trans_errs", "consistency_errors"):     # 3xTF32 tensor-core layers against cuBLAS fp32
        assert np.allclose(frozen[key], plain[key], rtol=5e-3, atol=5e-3), (key, np.abs(frozen[key] - plain[key]).max())


@gpu
@pytest.mark.parametrize("sampler", ["fps", "random"])
def test_test_1_baseline_samplers_run(sampler):
    step, model = _reg_model(sampler, True)
    torch.manual_seed(5)
    got = step.test_1(model, _reg_batches(40, 16), _dev())
    assert got["rotation_errors"].shape == (40,) and np.isfinite(got["consistency_errors"]).all() and 0 <= got["auc"] <= 1
    # the sampled pair holds input points that correspond under the ground truth only by chance: the consistency is positive
    assert (got["consistency_errors"] > 0).all()


@gpu
@pytest.mark.parametrize("frozen", [True, False])
def test_eval_1_means_modes_and_one_readback(frozen):
    step, model = _reg_model("samplenet", frozen)
    net = model.net if frozen else model
    net.sampler.train()
    if not frozen:
        net.feat.train()
    flags = [m.training for m in net.modules()]
    batches = _reg_batches(24, 8)
    with _Readbacks() as rb:
        vloss, gloss = step.eval_1(model, batches, _dev(), epoch=3)
    assert rb.count == 1
    assert [m.training for m in net.modules()] == flags
    # main.py:391-407 batch by batch
    net.eval()
    with torch.no_grad():
        vs, gs = [], []
        for data in batches:
            sl, sd, _ = step.compute_samplenet_loss(model, data, _dev())
            pl, info = step.compute_pcrnet_loss(model, sd, _dev())
            vs.append((pl + sl).item()); gs.append(info["rot_err"].item())
    assert vloss == pytest.approx(np.mean(vs), rel=1e-6) and gloss == pytest.approx(np.mean(gs), rel=1e-6)


# ----------------------------------------------------------------------------------------------------- classification
def _randomise_bn(net, seed):
    g = torch.Generator().manual_seed(seed)
    for mod in net.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.running_mean.copy_(0.1 * torch.randn(mod.num_features, generator=g))
            mod.running_var.copy_(0.5 + torch.rand(mod.num_features, generator=g))
            mod.weight.data.copy_(0.5 + torch.rand(mod.num_features, generator=g))


def _cls_setup(m=32, n_clouds=24, n_points=256, seed=0, frozen=True):
    torch.manual_seed(seed)
    sampler = sb.ClassificationSampleNet(m).to(_dev())
    net = tasknets.PointNetCls().to(_dev())
    _randomise_bn(sampler, seed + 1); _randomise_bn(net, seed + 2)
    net.requires_grad_(False).eval()
    g = torch.Generator().manual_seed(seed + 3)
    pcs = (torch.rand(n_clouds, n_points, 3, generator=g) * 2 - 1).to(_dev())
    labels = torch.randint(0, 40, (n_clouds,), generator=g).to(_dev())
    return sampler, (tasknets.FrozenPointNetCls(net) if frozen else net), net, pcs, labels


@gpu
@pytest.mark.parametrize("match_output", [True, False])
def test_classification_evaluator_against_reference_loop(match_output):
    sampler, cls, net, pcs, labels = _cls_setup()
    sampler.train()
    evaluator = sb.ClassificationEvaluator(sampler, cls, 32, match_output=match_output)
    with _Readbacks() as rb:
        out = evaluator.evaluate(pcs, labels, batch_size=10)
    assert rb.count == 1 and sampler.training
    # the same logits through the reference's counting loop
    sampler.eval()
    with torch.no_grad():
        parts = [sampler(pcs[s:s + 10]) for s in range(0, 24, 10)]
        simp, matched = torch.cat([a for a, _ in parts]), torch.cat([b for _, b in parts])
        assert torch.equal(out["simplified"], simp) and torch.equal(out["sampled"], matched)
        logits, end_points = cls(matched if match_output else simp)
        _, idx, _, _ = ops.nn_distance_forward(simp, pcs)
        hard = torch.gather(pcs, 1, idx.long()[:, :, None].expand(-1, -1, 3))
    assert torch.equal(out["hard_projected"], hard)          # evaluate_samplenet.py: the hard projection is the nearest input point
    assert out["soft_projected"].shape == simp.shape and not torch.equal(out["soft_projected"], hard)
    racc, rper = _reference_class_accuracy(logits.cpu().numpy(), labels.cpu().numpy(), 40)
    assert np.array_equal(out["predictions"], logits.argmax(1).cpu().numpy())
    assert out["accuracy"] == racc and np.array_equal(out["class_accuracy"], rper, equal_nan=True)
    assert out["mean_unique_idx"] == np.mean([np.size(np.unique(r)) for r in idx.cpu().numpy()])
    assert out["mean_loss"] == pytest.approx(float(net.get_loss(logits, labels)), rel=1e-5)


@gpu
def test_progressive_order_against_nn_matching():
    sampler, cls, _, pcs, _ = _cls_setup(n_clouds=6)
    evaluator = sb.ProgressiveClassificationEvaluator(sampler, cls)
    ordered = evaluator.order(pcs, batch_size=6)
    with torch.no_grad():
        simp, _ = sampler.eval()(pcs)
        _, idx, _, _ = ops.nn_distance_forward(simp, pcs)
    want = sputils.nn_matching(pcs.cpu().numpy(), idx.cpu().numpy(), pcs.shape[1])      # the numpy-signature one, k = N
    assert np.array_equal(ordered.cpu().numpy().astype(np.float64), want)
    # a reordering: every cloud keeps its points
    assert torch.equal(torch.sort(ordered.view(6, -1), dim=1)[0], torch.sort(pcs.view(6, -1), dim=1)[0])


@gpu
def test_progressive_curve_prefixes_against_size_by_size_and_dense():
    sampler, cls, net, pcs, labels = _cls_setup(n_clouds=20, n_points=128)
    frozen_ev, plain_ev = sb.ProgressiveClassificationEvaluator(sampler, cls), sb.ProgressiveClassificationEvaluator(sampler, net)
    ordered = frozen_ev.order(pcs)
    sizes = [128, 8, 16, 32, 64, 1, 100, 2, 4, 77]        # 10 sizes, not sorted: the answer comes back in the caller's order
    with torch.no_grad():
        lf, lp = frozen_ev.logits(ordered, sizes), plain_ev.logits(ordered, sizes)
    assert torch.allclose(lf, lp, rtol=2e-3, atol=2e-3)
    # records whose float32 prediction is not within the tensor-core path's error of a tie
    top2 = lp.topk(2, dim=2)[0]
    clear = ((top2[..., 0] - top2[..., 1]) > 5e-3)
    assert clear.float().mean() > 0.2
    assert torch.equal(lf.argmax(2)[clear], lp.argmax(2)[clear])
    with _Readbacks() as rb:
        got = frozen_ev.evaluate(pcs, labels, sizes, batch_size=8, ordered=ordered)
    assert rb.count == 1
    want = (lf.argmax(2) == labels[None]).double().mean(1).cpu().numpy()
    assert got["sizes"] == sizes and np.allclose(got["accuracy"], want)
    if bool(clear.all()):
        assert np.array_equal(got["accuracy"], plain_ev.evaluate(pcs, labels, sizes, ordered=ordered)["accuracy"])
    dense = frozen_ev.evaluate(pcs, labels, range(1, 129), ordered=ordered)       # the reference's dense evaluation: 8 passes of 16 prefixes
    assert dense["accuracy"].shape == (128,) and dense["accuracy"][127] == got["accuracy"][0] and dense["accuracy"][76] == got["accuracy"][9]
    with pytest.raises(ValueError):
        frozen_ev.evaluate(pcs, labels, [0, 4], ordered=ordered)


# ----------------------------------------------------------------------------------------------------- reconstruction
def _rec_setup(m=64, n_clouds=12, n_points=2048, seed=0, frozen=True):
    torch.manual_seed(seed)
    sampler = sb.ReconstructionSampleNet(m).to(_dev())
    net = tasknets.PointNetAE(n_pc_points=n_points).to(_dev())
    _randomise_bn(sampler, seed + 1); _randomise_bn(net, seed + 2)
    net.requires_grad_(False).eval()
    g = torch.Generator().manual_seed(seed + 3)
    pcs = (torch.rand(n_clouds, n_points, 3, generator=g) - 0.5).to(_dev())
    return sampler, (tasknets.FrozenPointNetAE(net) if frozen else net), net, pcs


@gpu
@pytest.mark.parametrize("frozen", [True, False])
def test_reconstruction_samples_and_per_cloud_loss(frozen):
    sampler, ae, net, pcs = _rec_setup(frozen=frozen)
    sampler.train()
    evaluator = sb.ReconstructionEvaluator(sampler, ae)
    sampled_pc, sample_idx = evaluator.get_samples(pcs, batch_size=5)
    assert sampler.training
    with torch.no_grad():
        parts = [sampler.eval()(pcs[s:s + 5]) for s in range(0, pcs.shape[0], 5)]
        simp, matched = torch.cat([a for a, _ in parts]), torch.cat([b for _, b in parts])
        _, idx, _, _ = ops.nn_distance_forward(simp, pcs)
        want_pc, want_idx, _ = sputils.simple_projection_and_continued_fps(pcs, simp, idx)
    assert torch.equal(sampled_pc, want_pc) and torch.equal(sample_idx, want_idx) and torch.equal(sampled_pc, matched)
    assert torch.equal(torch.gather(pcs, 1, sample_idx.long()[:, :, None].expand(-1, -1, 3)), sampled_pc)
    recon = evaluator.get_reconstructions_from_sampled(sampled_pc, batch_size=5)
    assert recon.shape == pcs.shape
    loss = evaluator.get_loss_ae_per_pc(pcs, sampled_pc, batch_size=5)
    with torch.no_grad():        # sampler_progressive_autoencoder.py:156-161: the graph once per cloud
        loop = torch.stack([trainers.autoencoder_loss(ae(sampled_pc[i:i + 1]), pcs[i:i + 1]) for i in range(pcs.shape[0])])
    assert torch.allclose(loss, loop, rtol=2e-5, atol=1e-8), (loss - loop).abs().max()
    with _Readbacks() as rb:
        out = evaluator.evaluate(pcs, batch_size=5)
    assert rb.count == 1
    assert np.allclose(out["ae_loss_per_pc"], loss.cpu().numpy(), rtol=1e-6) and out["nre"] == pytest.approx(np.mean(out["ae_loss_per_pc"] / out["ae_loss_per_pc_ref"]))
    assert np.isfinite(out["nre_per_pc"]).all() and (out["nre_per_pc"] > 0).all()


class _WholeCloud(torch.nn.Module):
    name = "identity"

    def forward(self, x):
        return x


@gpu
def test_nre_of_the_whole_cloud_is_one_and_baselines_run():
    _, ae, _, pcs = _rec_setup(n_clouds=6)
    out = sb.ReconstructionEvaluator(_WholeCloud(), ae).evaluate(pcs)
    # the sample is the cloud reordered by FPS completion; max-pooling does not see the order
    assert np.allclose(out["nre_per_pc"], 1.0, rtol=1e-4) and out["nre"] == pytest.approx(1.0, rel=1e-4)
    for baseline in (sb.FPSSampler(64, permute=False, input_shape="bnc", output_shape="bnc"), sb.RandomSampler(64, input_shape="bnc", output_shape="bnc")):
        res = sb.ReconstructionEvaluator(baseline, ae).evaluate(pcs, sizes=[16, 64])
        assert res["nre_per_pc"].shape == (2, 6) and np.isfinite(res["nre"]).all() and res["sampled_pc"].shape == (6, 64, 3)
    emd = sb.ReconstructionEvaluator(sb.FPSSampler(64, permute=False, input_shape="bnc", output_shape="bnc"), ae, ae_loss="emd")
    loss = emd.get_loss_ae_per_pc(pcs[:2], emd.get_samples(pcs[:2])[0])
    assert loss.shape == (2,) and bool(torch.isfinite(loss).all())


@gpu
def test_progressive_reconstruction_curve_prefixes_against_size_by_size():
    sampler, ae, net, pcs = _rec_setup(m=256, n_clouds=10)
    sizes = [16, 32, 64, 128, 256, 8, 100, 1]
    fe, pe = sb.ReconstructionEvaluator(sampler, ae), sb.ReconstructionEvaluator(sampler, net)
    sampled_pc, _ = fe.get_samples(pcs)
    got = fe.get_loss_ae_per_pc_progressive(pcs, sampled_pc, sizes, batch_size=4)
    want = pe.get_loss_ae_per_pc_progressive(pcs, sampled_pc, sizes, batch_size=10)
    assert got.shape == (8, 10) and torch.allclose(got, want, rtol=5e-3, atol=1e-6), (got - want).abs().max()
    assert torch.allclose(got[4], fe.get_loss_ae_per_pc(pcs, sampled_pc), rtol=1e-4)
    out = fe.evaluate(pcs, sizes=sizes)
    assert out["nre"].shape == (8,) and out["ae_loss_per_pc"].shape == (8, 10)
