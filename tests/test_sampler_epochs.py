"""The SampleNet trainers' epochs on the device (trainers.SamplerTrainStep, AutoencoderTrainStep.train_one_epoch) and the reconstruction
trainers' augmentation on CUDA (snb200_ae_augment in csrc/augment.cu, ops.ae_augment).

CPU: the classification and reconstruction schedules at step and epoch boundaries; ClassifierTrainStep's schedules unchanged by the shared
functions; the entry's export and argument checks, which launch nothing; the op's argument errors and refusal of CPU tensors; an epoch
needs one whole batch.
GPU (H100): the kernel against a float64 numpy restatement of apply_augmentations on the documented Philox stream (within one float32 ulp);
the noise's moments and the rotation block's entries against numpy's rand_rotation_matrix; seeding, CUDA graph replays, the write set and
in-place calls; every epoch bit for bit against a loop of __call__ over the same permutation, with and without augmentation, and the
reconstruction epoch's EMD division and recomposed loss; one device-to-host copy per epoch; the BatchNorm schedule reaching the generator's
running statistics on the fused and per-layer routes."""
import copy
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from samplenet_b200 import ops, tasknets, trainers  # noqa: E402
from test_classifier_augmentation import ANGLE_WORD, KEY, _key_tensor, _key_words, _within_ulp, box_muller, philox, u53  # noqa: E402

RUNNING_ULPS = 4   # running statistics against (1 - m) R + m S in float64: float32 ulps of the terms' magnitudes


# ----------------------------------------------------------------------------------------------------- numpy restatement
def _philox_args(key):
    k0, k1 = key
    return (k1 & 0xFFFFFFFF, k1 >> 32, k0 & 0xFFFFFFFF, k0 >> 32)


def rotation_from_uniforms(u0, u1, u2):
    """general_utils.rand_rotation_matrix (deflection 1) from its three uniforms, in float64, with the third row and column set to (0, 0, 1)
    as apply_augmentations does."""
    theta, phi, z = u0 * 2.0 * 1.0 * np.pi, u1 * 2.0 * np.pi, u2 * 2.0 * 1.0
    r = np.sqrt(z)
    v = np.array([np.sin(phi) * r, np.cos(phi) * r, np.sqrt(2.0 - z)])
    st, ct = np.sin(theta), np.cos(theta)
    m = (np.outer(v, v) - np.eye(3)).dot(np.array([[ct, st, 0], [-st, ct, 0], [0, 0, 1]]))
    m[0, 2] = m[2, 0] = m[1, 2] = m[2, 1] = 0
    m[2, 2] = 1
    return m


def drawn_rotation(key):
    wa = philox(0, ANGLE_WORD, *_philox_args(key))
    wb = philox(1, ANGLE_WORD, *_philox_args(key))
    return rotation_from_uniforms(float(u53(wa[0], wa[1])), float(u53(wa[2], wa[3])), float(u53(wb[0], wb[1])))


def restate(points, key, mu, sigma, z_rotate):
    """apply_augmentations on the documented random stream: (B, N, 3) float32 -> float32."""
    b, n, _ = points.shape
    x = points.astype(np.float32)
    if sigma is not None:
        cloud = np.arange(b, dtype=np.uint64)[:, None]
        j = 2 * np.arange(n, dtype=np.uint64)[None, :]
        zx, zy = box_muller(philox(cloud, j, *_philox_args(key)))
        zz, _ = box_muller(philox(cloud, j + np.uint64(1), *_philox_args(key)))
        x = (x.astype(np.float64) + (mu + sigma * np.stack([zx, zy, zz], axis=-1))).astype(np.float32)
    if z_rotate:
        x = x.astype(np.float64).dot(drawn_rotation(key)).astype(np.float32)
    return x


def _tf_staircase(base, global_step, decay_steps, rate):
    return base * math.pow(rate, math.floor(global_step / decay_steps))


# ----------------------------------------------------------------------------------------------------- CPU
def _cpu_steps():
    sampler, task = torch.nn.Linear(1, 1), torch.nn.Linear(1, 1)
    return trainers.ClassificationStep(sampler, task, 32), trainers.ReconstructionStep(sampler, task, 64)


def test_sampler_schedules_at_step_and_epoch_boundaries():
    cls_step, rec_step = _cpu_steps()
    run = trainers.SamplerTrainStep(cls_step, None)
    assert run.batch_size == 32 and run.base_lr == 0.01
    for s in (0, 1, 18749, 18750, 18751, 37499, 37500, 131249, 131250, 10 ** 6):   # 600000 / 32 = 18750 steps per staircase step
        run.step = s
        assert run.learning_rate() == pytest.approx(max(_tf_staircase(0.01, s * 32, 600000, 0.7), 1e-5), rel=1e-12, abs=0), s
        assert run.bn_momentum() == pytest.approx(1 - min(0.99, 1 - _tf_staircase(0.5, s * 32, 600000.0, 0.5)), rel=1e-12, abs=0), s
    run.step = 18750
    assert run.learning_rate() == pytest.approx(7e-3) and run.bn_momentum() == pytest.approx(0.25)
    run.step = 10 ** 6
    assert run.learning_rate() == 1e-5 and run.bn_momentum() == pytest.approx(0.01)

    run = trainers.SamplerTrainStep(rec_step, None)
    assert run.batch_size == 50 and run.bn_momentum() is None
    for e in (0, 1, 10 ** 4):
        run.epoch = e
        assert run.learning_rate() == 5e-4
    run = trainers.SamplerTrainStep(rec_step, None, learning_rate=1e-3, decay_steps=10)
    for e in (0, 9, 10, 11, 19, 20, 59, 60, 1000):
        run.epoch = e
        run.step = 12345   # the reconstruction schedule counts epochs, not steps
        assert run.learning_rate() == pytest.approx(max(_tf_staircase(1e-3, e, 10, 0.5), 1e-5), rel=1e-12, abs=0), e
    run.epoch = 1000
    assert run.learning_rate() == 1e-5


def test_sampler_train_step_rejects_what_its_task_does_not_have():
    cls_step, rec_step = _cpu_steps()
    with pytest.raises(TypeError):
        trainers.SamplerTrainStep(object(), None)
    for kw in ({"z_rotate": True}, {"gauss_augment": {"mu": 0.0, "sigma": 0.01}}, {"decay_steps": 10}):
        with pytest.raises(ValueError):
            trainers.SamplerTrainStep(cls_step, None, **kw)
    for kw in ({"decay_step": 10}, {"decay_rate": 0.5}, {"gauss_augment": {"sigma": 0.01}}, {"gauss_augment": {"mu": 0.0, "sigma": None}},
               {"gauss_augment": 0.01}):
        with pytest.raises(ValueError):
            trainers.SamplerTrainStep(rec_step, None, **kw)
    with pytest.raises(ValueError):
        trainers.AutoencoderTrainStep(tasknets.PointNetAE(), None, gauss_augment={"mu": 0.0})
    with pytest.raises(ValueError):
        trainers.SamplerTrainStep(cls_step, None)(torch.rand(2, 8, 3))   # classification needs labels


def test_classifier_train_step_schedules_are_unchanged():
    for bs, lr, ds, dr in ((32, 1e-3, 200000, 0.7), (24, 0.01, 600000, 0.7), (7, 3e-4, 1000, 0.5)):
        step = trainers.ClassifierTrainStep(torch.nn.Linear(1, 1), None, batch_size=bs, base_lr=lr, decay_step=ds, decay_rate=dr)
        for s in list(range(0, 40)) + [ds // bs - 1, ds // bs, ds // bs + 1, 10 * ds // bs, 10 ** 6]:
            assert step.learning_rate(s) == max(trainers.staircase_decay(lr, s * bs, ds, dr), 1e-5)
            assert step.bn_decay(s) == min(0.99, 1.0 - trainers.staircase_decay(0.5, s * bs, float(ds), 0.5))


def test_library_exports_the_entry():
    from samplenet_b200 import _lib

    assert "snb200_ae_augment" in _lib.exported_symbols()
    assert hasattr(_lib.lib(), "snb200_ae_augment")
    assert "int snb200_ae_augment(" in open(os.path.join(os.path.dirname(HERE), "include", "samplenet_b200.h")).read()


def test_entry_rejects_bad_arguments_and_launches_nothing():
    from samplenet_b200 import _lib

    lib = _lib.lib()
    f = lambda *a: lib.snb200_ae_augment(*a, None)
    P, Q, K = 1 << 32, 1 << 36, 1 << 44      # never dereferenced: every call below fails its checks or has b = 0
    inf, nan = float("inf"), float("nan")
    before = _lib.launch_count()
    bad = [(1, 0, P, Q, K, 1, 0.0, 0.01, 1),                  # n = 0
           (1, (1 << 24) + 1, P, Q, K, 1, 0.0, 0.01, 1),      # n > 2^24
           (-1, 4, P, Q, K, 1, 0.0, 0.01, 1),                 # b < 0
           (2, 4, P, Q, K, 1, 0.0, -0.01, 0),                 # sigma < 0
           (2, 4, P, Q, K, 1, 0.0, nan, 0),                   # sigma NaN
           (2, 4, P, Q, K, 1, 0.0, inf, 0),                   # sigma infinite
           (2, 4, P, Q, K, 1, nan, 0.01, 0),                  # mu NaN
           (2, 4, P, Q, K, 1, -inf, 0.01, 1),                 # mu infinite
           (2, 4, None, Q, K, 1, 0.0, 0.01, 1),               # null input
           (2, 4, P, None, K, 0, 0.0, 0.0, 1),                # null output
           (2, 4, P, Q, None, 1, 0.0, 0.01, 0),               # noise needs the key
           (2, 4, P, Q, None, 0, 0.0, 0.0, 1),                # the rotation needs the key
           (2, 4, P, P + 12, K, 1, 0.0, 0.01, 1),             # partial overlap
           (2, 4, P + 12, P, K, 0, 0.0, 0.0, 1)]
    for args in bad:
        assert f(*args) == -1, args
    assert f(0, 4, None, None, None, 1, 0.0, 0.01, 1) == 0     # b = 0: nothing to do
    assert _lib.launch_count() == before


def test_ops_argument_errors_and_cpu_tensors():
    x = torch.rand(2, 8, 3)
    for bad in (torch.rand(2, 8, 2), torch.rand(8, 3), torch.rand(2, 0, 3), np.zeros((2, 8, 3), np.float32)):
        with pytest.raises(ValueError):
            ops.ae_augment(bad, sigma=0.01)
    for mu, sigma in ((0.0, -0.1), (0.0, float("nan")), (float("inf"), 0.01), (0.0, float("inf")), (0.1, None)):
        with pytest.raises(ValueError):
            ops.ae_augment(x, mu, sigma)
    for out in (torch.empty(2, 8, 3, dtype=torch.float64), torch.empty(2, 9, 3), torch.empty(2, 3, 8).transpose(1, 2), np.zeros((2, 8, 3))):
        with pytest.raises(ValueError):
            ops.ae_augment(x, sigma=0.01, out=out)
    with pytest.raises(RuntimeError):
        ops.ae_augment(x, sigma=0.01)
    with pytest.raises(RuntimeError):
        ops.ae_augment(x, z_rotate=True)


def test_an_epoch_needs_one_whole_batch():
    cls_step, rec_step = _cpu_steps()
    x, y = torch.rand(31, 8, 3), torch.zeros(31, dtype=torch.int64)
    with pytest.raises(ValueError, match="whole batch"):
        trainers.SamplerTrainStep(cls_step, None).train_one_epoch(x, y)
    with pytest.raises(ValueError, match="whole batch"):
        trainers.SamplerTrainStep(rec_step, None).train_one_epoch(torch.rand(49, 8, 3))
    with pytest.raises(ValueError, match="whole batch"):
        trainers.AutoencoderTrainStep(tasknets.PointNetAE(n_pc_points=8), None, batch_size=50).train_one_epoch(torch.rand(49, 8, 3))


# ----------------------------------------------------------------------------------------------------- GPU: the kernel
MODES = {"noise": (0.01, 0.02, False), "rotate": (None, None, True), "both": (-0.03, 0.05, True)}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("b,n", [(1, 1), (50, 2048), (64, 4096), (2, 1100000)])   # the last one takes the stride loop (> 4096 * 256 points)
def test_ae_augment_matches_the_float64_restatement(b, n, mode):
    mu, sigma, z_rotate = MODES[mode]
    g = torch.Generator().manual_seed(b * 7 + n)
    x = torch.rand(b, n, 3, generator=g) * 2 - 1
    got = ops.ae_augment(x.cuda(), mu, sigma, z_rotate, key=_key_tensor(KEY)).cpu().numpy()
    ref = restate(x.numpy(), KEY, mu, sigma, z_rotate)
    ok = _within_ulp(got, ref)
    assert ok.all(), (int((~ok).sum()), float(np.abs(got - ref).max()))
    if mode == "rotate":   # z is left as it is
        assert np.array_equal(got[..., 2].view(np.int32), x.numpy()[..., 2].view(np.int32))


@pytest.mark.gpu
def test_no_augmentation_copies_and_empty_batches():
    x = torch.rand(3, 500, 3, device="cuda")
    assert torch.equal(ops.ae_augment(x), x)
    assert ops.ae_augment(torch.empty(0, 10, 3, device="cuda"), sigma=0.1, z_rotate=True).shape == (0, 10, 3)


@pytest.mark.gpu
def test_noise_moments_and_rotation_entries_against_numpy(record_property):
    from scipy import stats

    mu, sigma = 0.1, 0.02
    x = torch.zeros(64, 4096, 3, device="cuda")
    d = ops.ae_augment(x, mu, sigma, key=_key_tensor(KEY)).double().flatten().cpu().numpy()
    N = d.size
    record_property("noise_mean_err", float(d.mean() - mu))
    record_property("noise_std_rel_err", float(d.std() / sigma - 1))
    assert abs(d.mean() - mu) <= 6 * sigma / math.sqrt(N)
    assert abs(d.std() / sigma - 1) <= 6 * math.sqrt(0.5 / N) + 1e-6     # + the float32 rounding of mu + noise

    draws = 3000
    e = torch.zeros(1, 2, 3, device="cuda")
    e[0, 0, 0] = 1.0                                  # (1, 0, 0) dot R is R's first row, (0, 1, 0) its second
    e[0, 1, 1] = 1.0
    torch.manual_seed(4)
    got = torch.stack([ops.ae_augment(e, z_rotate=True)[0, :, :2] for _ in range(draws)]).double().cpu().numpy().reshape(draws, 4)
    rng = np.random.RandomState(5)
    ref = np.stack([rotation_from_uniforms(*rng.uniform(size=3))[:2, :2].reshape(4) for _ in range(draws)])
    for k in range(4):
        p = stats.ks_2samp(got[:, k], ref[:, k]).pvalue
        record_property("rotation_entry_%d_ks_p" % k, p)
        assert p > 1e-3, (k, p)


@pytest.mark.gpu
def test_seeding_repeats_and_graph_replays_draw_new_keys():
    x = torch.rand(8, 500, 3, device="cuda")
    torch.manual_seed(7)
    a = ops.ae_augment(x, 0.0, 0.01, True)
    torch.manual_seed(7)
    b = ops.ae_augment(x, 0.0, 0.01, True)
    torch.manual_seed(8)
    c = ops.ae_augment(x, 0.0, 0.01, True)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert not torch.equal(b, ops.ae_augment(x, 0.0, 0.01, True))

    xh = torch.rand(4, 300, 3, generator=torch.Generator().manual_seed(3)) - 0.5
    xd = xh.cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            ops.ae_augment(xd, 0.0, 0.01, True)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        key = torch.empty(2, dtype=torch.int64, device="cuda").random_()
        out = ops.ae_augment(xd, 0.0, 0.01, True, key=key)
        out_default = ops.ae_augment(xd, 0.0, 0.01, True)
    keys, outs = set(), []
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        words = _key_words(key)
        keys.add(words)
        assert _within_ulp(out.cpu().numpy(), restate(xh.numpy(), words, 0.0, 0.01, True)).all()
        outs.append(out_default.clone())
    assert len(keys) == 3
    assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[2])


@pytest.mark.gpu
def test_only_out_is_written_and_in_place_matches():
    from samplenet_b200 import _lib

    lib = _lib.lib()
    b, n, pad = 3, 333, 1000
    x = torch.rand(b, n, 3, device="cuda") - 0.5
    key = _key_tensor(KEY)
    for gauss, z_rotate in ((1, 0), (0, 1), (1, 1), (0, 0)):
        buf = torch.full((b * n * 3 + 2 * pad,), float("nan"), device="cuda")
        buf[:pad] = 7.0
        buf[-pad:] = -3.0
        x0 = x.clone()
        rc = lib.snb200_ae_augment(b, n, x.data_ptr(), buf[pad:].data_ptr(), key.data_ptr(), gauss, 0.0, 0.02, z_rotate,
                                   torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize()
        assert torch.all(buf[:pad] == 7.0) and torch.all(buf[-pad:] == -3.0)
        assert not torch.isnan(buf[pad:-pad]).any()
        assert torch.equal(x, x0)
    ref = ops.ae_augment(x, 0.0, 0.02, True, key=key)
    y = x.clone()
    assert ops.ae_augment(y, 0.0, 0.02, True, out=y, key=key) is y
    assert torch.equal(y, ref)
    z = torch.empty_like(x)
    assert ops.ae_augment(x, 0.0, 0.02, True, out=z, key=key) is z and torch.equal(z, ref)


# ----------------------------------------------------------------------------------------------------- GPU: the epochs
B, N_SET, N_PTS, M = 8, 21, 256, 32        # 2 whole batches of 8; the last 5 clouds are the remainder
GAUSS = {"mu": 0.0, "sigma": 0.01}


def _set(seed, n=N_SET, points=N_PTS, classes=5):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, points, 3, generator=g) - 0.5).cuda(), torch.randint(0, classes, (n,), generator=g).cuda()


def _sampler_runner(task, augment):
    """A SamplerTrainStep around a fresh step of the given task with frozen CUDA task networks; Adam over the sampler."""
    import samplenet_b200 as sb

    torch.manual_seed(0)
    if task in ("cls", "progressive_cls"):
        sampler = sb.ClassificationSampleNet(M, group_size=7).cuda()
        net = tasknets.PointNetClsTransforms(num_classes=5).cuda().eval().requires_grad_(False)
        step = (trainers.ClassificationStep(sampler, tasknets.FrozenPointNetClsTransforms(net), M) if task == "cls"
                else trainers.ProgressiveClassificationStep(sampler, tasknets.FrozenPointNetClsTransforms(net), 8, M))
    else:
        sampler = sb.ReconstructionSampleNet(M).cuda()
        ae = tasknets.FrozenPointNetAE(tasknets.PointNetAE(n_pc_points=N_PTS).cuda().eval().requires_grad_(False))
        step = (trainers.ProgressiveReconstructionStep(sampler, ae, sizes=(8, 16, 32)) if task == "progressive_rec"
                else trainers.ReconstructionStep(sampler, ae, M, ae_loss="emd" if task == "rec_emd" else "chamfer"))
    kw = {"gauss_augment": GAUSS, "z_rotate": True} if augment else {}
    return trainers.SamplerTrainStep(step, torch.optim.Adam(sampler.parameters(), lr=1e-3), batch_size=B, **kw)


def _assert_same_training_state(a_module, b_module, a_opt, b_opt):
    sa, sb_ = a_module.state_dict(), b_module.state_dict()
    for k in sa:
        assert torch.equal(sa[k], sb_[k]), k
    pa, pb = list(a_module.parameters()), list(b_module.parameters())
    for p, q in zip(pa, pb):
        st_a, st_b = a_opt.state.get(p, {}), b_opt.state.get(q, {})
        assert st_a.keys() == st_b.keys()
        for k in st_a:
            assert torch.equal(torch.as_tensor(st_a[k]), torch.as_tensor(st_b[k])), k


def _manual_then_epoch(run_a, run_b, x, y, seed):
    """run_b: a Python loop of __call__ over the permutation the epoch draws; run_a: train_one_epoch on the set with the remainder poisoned."""
    torch.manual_seed(seed)
    perm = torch.randperm(x.shape[0], device="cuda")
    steps = x.shape[0] // B
    sums = {}
    for s in range(steps):
        idx = perm[s * B:(s + 1) * B]
        r = run_b(x[idx], None if y is None else y[idx])
        for k, v in r.items():
            sums[k] = sums.get(k, 0.0) + float(v)
    x_nan = x.clone()
    x_nan[perm[steps * B:]] = float("nan")            # the remainder is not used
    torch.manual_seed(seed)
    res = run_a.train_one_epoch(x_nan, y)
    return res, sums, steps


SAMPLER_CASES = [("cls", False), ("progressive_cls", False), ("rec", False), ("rec", True), ("rec_emd", False), ("rec_emd", True),
                 ("progressive_rec", False), ("progressive_rec", True)]


@pytest.mark.gpu
@pytest.mark.parametrize("task,augment", SAMPLER_CASES)
def test_sampler_epoch_is_the_loop_of_steps_and_returns_the_reference_numbers(task, augment):
    run_a, run_b = _sampler_runner(task, augment), _sampler_runner(task, augment)
    cls_like = task.endswith("cls")
    x, y = _set(1)
    res, sums, steps = _manual_then_epoch(run_a, run_b, x, y if cls_like else None, 21)
    assert res["steps"] == steps == 2 and run_a.step == run_b.step == 2 and run_a.epoch == 1
    assert all(math.isfinite(v) for v in res.values())
    means = {k: v / steps for k, v in sums.items()}
    if cls_like:
        assert res["loss"] == means["loss"] and res["loss_classifier"] == means["loss_classifier"]
        if task == "cls":                           # the step returns pred: accuracy over the clouds seen
            assert res["accuracy"] == sums["correct"] / (steps * B)
        else:
            assert "accuracy" not in res
    else:
        # _single_epoch_train (samplenet_pointnet_ae.py:291-353): the means, loss_ae / N with EMD, the loss recomposed from the means
        loss_ae = means["loss_ae"] / (N_PTS if task == "rec_emd" else 1)
        assert res["loss_ae"] == loss_ae
        assert res["loss"] == loss_ae + run_a.task.alpha * means["loss_simplification"] + run_a.task.lmbda * means["loss_projection"]
    assert res["loss_simplification"] == means["loss_simplification"] and res["loss_projection"] == means["loss_projection"]
    _assert_same_training_state(run_a.task.sampler, run_b.task.sampler, run_a.optimizer, run_b.optimizer)


AE_CASES = [("chamfer", False, False), ("chamfer", True, False), ("emd", False, False), ("emd", True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("loss,augment,denoising", AE_CASES)
def test_autoencoder_epoch_is_the_loop_of_steps(loss, augment, denoising):
    def make():
        torch.manual_seed(0)
        ae = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=N_PTS).cuda())
        kw = {"gauss_augment": GAUSS, "z_rotate": True} if augment else {}
        return trainers.AutoencoderTrainStep(ae, torch.optim.Adam(ae.parameters(), lr=5e-4), ae_loss=loss, n_sample_points=N_PTS,
                                             batch_size=B, denoising=denoising, **kw)

    run_a, run_b = make(), make()
    x, _ = _set(2)
    torch.manual_seed(31)
    perm = torch.randperm(N_SET, device="cuda")
    total = 0.0
    for s in range(N_SET // B):
        total += float(run_b(x[perm[s * B:(s + 1) * B]]))
    x_nan = x.clone()
    x_nan[perm[(N_SET // B) * B:]] = float("nan")
    torch.manual_seed(31)
    res = run_a.train_one_epoch(x_nan)
    assert run_a.ae.route == "cuda"
    assert res["steps"] == 2
    assert res["loss"] == total / 2 / (N_PTS if loss == "emd" else 1)        # pointnet_ae.py:186-192
    _assert_same_training_state(run_a.ae, run_b.ae, run_a.optimizer, run_b.optimizer)


@pytest.mark.gpu
def test_denoising_scores_against_the_clean_batch():
    torch.manual_seed(0)
    ae = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=N_PTS).cuda())
    ae_a, ae_b = copy.deepcopy(ae), copy.deepcopy(ae)
    run = trainers.AutoencoderTrainStep(ae_a, torch.optim.SGD(ae_a.parameters(), lr=0.0), n_sample_points=N_PTS, denoising=True,
                                        gauss_augment=GAUSS, z_rotate=True)
    ref = trainers.AutoencoderTrainStep(ae_b, torch.optim.SGD(ae_b.parameters(), lr=0.0), n_sample_points=N_PTS)
    x, _ = _set(3, n=B)
    torch.manual_seed(4)
    got = run(x)
    torch.manual_seed(4)
    aug = ops.ae_augment(x, 0.0, 0.01, True)
    assert torch.equal(got, ref(aug, x))


def _dtoh_copies(fn):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, sum(e.count for e in prof.key_averages() if "DtoH" in e.key)


@pytest.mark.gpu
@pytest.mark.parametrize("task", ["cls", "rec_aug", "ae_aug"])
def test_one_read_back_per_epoch(task):
    x, y = _set(4, n=3 * B + 1)
    if task == "ae_aug":
        ae = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=N_PTS).cuda())
        run = trainers.AutoencoderTrainStep(ae, torch.optim.Adam(ae.parameters()), n_sample_points=N_PTS, batch_size=B, gauss_augment=GAUSS,
                                            z_rotate=True)
        epoch = lambda: run.train_one_epoch(x)
    else:
        run = _sampler_runner("cls" if task == "cls" else "rec", task == "rec_aug")
        epoch = lambda: run.train_one_epoch(x, y if task == "cls" else None)
    epoch()                                           # first calls: module loads, cached host constants
    res, copies = _dtoh_copies(epoch)
    assert res["steps"] == 3
    assert copies == 1, copies


def _bn_layers(sampler):
    return [m for m in sampler.modules() if isinstance(m, torch.nn.BatchNorm1d)]


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["fused", "layers"])
def test_bn_schedule_reaches_the_generator_running_statistics(route):
    """Step s sets momentum m_s = 1 - pointnet_bn_decay(s) on the sampler's BatchNorm layers.  A copy of the sampler taken before the step
    and run once with momentum 1 holds the step's batch statistics S (batch mean and unbiased variance), so after the step each running
    statistic must be (1 - m_s) R + m_s S, R its value before, up to the float32 rounding of that update (RUNNING_ULPS)."""
    import samplenet_b200 as sb

    def make():
        if route == "fused":
            return sb.SampleNet(M, 128, 7, input_shape="bnc", output_shape="bnc").cuda()
        return sb.ClassificationSampleNet(M, group_size=7).cuda()

    torch.manual_seed(0)
    sampler = make()
    net = tasknets.PointNetCls(num_classes=5).cuda().eval().requires_grad_(False)
    bs, n_pts = 16, 1024
    run = trainers.SamplerTrainStep(trainers.ClassificationStep(sampler, tasknets.FrozenPointNetCls(net), M),
                                    torch.optim.Adam(sampler.parameters(), lr=1e-3), batch_size=bs, decay_step=2 * bs)
    x, y = _set(5, n=4 * bs, points=n_pts)
    momenta = []
    for s in range(4):
        xb, yb = x[s * bs:(s + 1) * bs], y[s * bs:(s + 1) * bs]
        before = [(bn.running_mean.clone(), bn.running_var.clone()) for bn in _bn_layers(sampler)]
        probe = make().train()                       # a copy (deepcopy does not take the fused forward's saved loss terms)
        probe.load_state_dict(sampler.state_dict())
        for bn in _bn_layers(probe):
            bn.momentum = 1.0
        probe(xb)
        assert probe.generator_route == route
        stats_s = [(bn.running_mean.clone(), bn.running_var.clone()) for bn in _bn_layers(probe)]
        run(xb, yb)
        m = 1.0 - trainers.pointnet_bn_decay(s, bs, 2 * bs)
        momenta.append(m)
        assert sampler.generator_route == route
        for bn, (r_mean, r_var), (s_mean, s_var) in zip(_bn_layers(sampler), before, stats_s):
            assert bn.momentum == m
            for got, r, st in ((bn.running_mean, r_mean, s_mean), (bn.running_var, r_var, s_var)):
                want = (1 - m) * r.double() + m * st.double()
                scale = (1 - m) * r.double().abs() + m * st.double().abs()
                err = (got.double() - want).abs()
                assert bool((err <= RUNNING_ULPS * 2.0 ** -24 * scale + 1e-30).all()), (s, float((err / scale.clamp_min(1e-30)).max()))
    assert momenta == [0.5, 0.5, 0.25, 0.25]
    assert all(int(bn.num_batches_tracked) == 4 for bn in _bn_layers(sampler))
