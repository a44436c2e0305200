"""The classifier trainer's augmentation and the rotation-vote evaluation on CUDA: snb200_rotate_jitter (csrc/augment.cu), ops.rotate_jitter /
ops.rotate_by_angles, ClassifierTrainStep(augment=True) and train_one_epoch, evaluation.ClassifierEvaluator.

CPU: a numpy restatement of Philox4x32-10 against the Random123 known answers; the entry's argument checks, which launch nothing; the ops'
argument errors and refusal of CPU tensors; train_one_epoch and the one-vote evaluator on the plain modules against host restatements of
train_classifier.py's loops.
GPU (H100): the kernel against a float64 numpy restatement of provider.py at several shapes, with a supplied key (within one float32 ulp);
the fixed-angle votes; the distributions of the angles and of the clipped jitter; seeding; CUDA graph replays; the write set; the training
step and epoch bit for bit against their manual compositions; the evaluator against a per-vote restatement, with the plain module and the
frozen wrapper."""
import copy
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from samplenet_b200 import evaluation, ops, tasknets, trainers  # noqa: E402

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)
ANGLE_WORD = 0xFFFFFFFF
KEY = (0x243F6A8885A308D3, 0x13198A2E03707344)   # a key with both halves of both words set
FRONT_BAR = 1e-4     # frozen wrapper's summed vote logits against the plain module (TF32 off): / max |logit|


# ----------------------------------------------------------------------------------------------------- numpy restatement
def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on arrays of uint64 holding 32-bit words (broadcast), as Random123 / curand_Philox4x32_10."""
    c = [np.asarray(v, dtype=np.uint64) & MASK32 for v in (c0, c1, c2, c3)]
    k = [np.uint64(k0) & MASK32, np.uint64(k1) & MASK32]
    for _ in range(10):
        p0, p1 = np.uint64(M0) * c[0], np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & MASK32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & MASK32]
        k = [(k[0] + np.uint64(W0)) & MASK32, (k[1] + np.uint64(W1)) & MASK32]
    return c


def u53(wa, wb):
    return ((wa >> np.uint64(5)).astype(np.float64) * 67108864.0 + (wb >> np.uint64(6)).astype(np.float64)) * (1.0 / 9007199254740992.0)


def box_muller(w):
    u1, u2 = u53(w[0], w[1]), u53(w[2], w[3])
    r = np.sqrt(-2.0 * np.log(1.0 - u1))
    return r * np.cos(2.0 * np.pi * u2), r * np.sin(2.0 * np.pi * u2)


def _rot(pc, angle):
    """provider.rotate_point_cloud_by_angle on one cloud: np.dot(pc, R) in float64."""
    c, s = np.cos(angle), np.sin(angle)
    return np.dot(pc.reshape(-1, 3), np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]]))


def drawn_angles(num_clouds, key):
    k0, k1 = key
    w = philox(np.arange(num_clouds, dtype=np.uint64), ANGLE_WORD, k1 & 0xFFFFFFFF, k1 >> 32, k0 & 0xFFFFFFFF, k0 >> 32)
    return u53(w[0], w[1]) * 2 * np.pi


def restate(points, key, sigma, clip):
    """rotate_point_cloud, then jitter_point_cloud, on the documented random stream: (B, N, 3) float32 -> float32."""
    b, n, _ = points.shape
    k0, k1 = key
    ang = drawn_angles(b, key)
    rot = np.stack([_rot(points[i].astype(np.float64), ang[i]) for i in range(b)]).astype(np.float32)
    if sigma == 0:
        return rot
    cloud = np.arange(b, dtype=np.uint64)[:, None]
    j = 2 * np.arange(n, dtype=np.uint64)[None, :]
    args = (k1 & 0xFFFFFFFF, k1 >> 32, k0 & 0xFFFFFFFF, k0 >> 32)
    zx, zy = box_muller(philox(cloud, j, *args))
    zz, _ = box_muller(philox(cloud, j + np.uint64(1), *args))
    jit = np.clip(sigma * np.stack([zx, zy, zz], axis=-1), -clip, clip)
    return (rot.astype(np.float64) + jit).astype(np.float32)


def _within_ulp(got, ref):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    ulp = np.maximum(np.spacing(np.abs(ref)), np.spacing(np.abs(got)))
    return np.abs(got.astype(np.float64) - ref.astype(np.float64)) <= ulp


def _key_tensor(key, dev="cuda"):
    return torch.tensor([k - (1 << 64) if k >= 1 << 63 else k for k in key], dtype=torch.int64, device=dev)


def _key_words(t):
    return tuple(int(v) & 0xFFFFFFFFFFFFFFFF for v in t.cpu().tolist())


# ----------------------------------------------------------------------------------------------------- CPU
def test_philox_restatement_reproduces_the_random123_known_answers():
    cases = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
             ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in cases:
        assert tuple(int(v) for v in philox(*ctr, *key)) == want


def test_library_exports_the_augmentation_entry():
    from samplenet_b200 import _lib

    assert "snb200_rotate_jitter" in _lib.exported_symbols()
    assert hasattr(_lib.lib(), "snb200_rotate_jitter")
    assert "int snb200_rotate_jitter(" in open(os.path.join(os.path.dirname(HERE), "include", "samplenet_b200.h")).read()


def test_entry_rejects_bad_arguments_and_launches_nothing():
    from samplenet_b200 import _lib

    lib = _lib.lib()
    f = lambda *a: lib.snb200_rotate_jitter(*a, None)
    P, Q, A, K = 1 << 32, 1 << 36, 1 << 40, 1 << 44      # never dereferenced: every call below fails its checks or has b = 0
    before = _lib.launch_count()
    bad = [(1, 0, 1, P, Q, None, K, 0.01, 0.05),                 # n = 0
           (1, (1 << 24) + 1, 1, P, Q, None, K, 0.01, 0.05),     # n > 2^24
           (-1, 4, 1, P, Q, None, K, 0.01, 0.05),                # b < 0
           (1, 4, 0, P, Q, A, K, 0.0, 0.0),                      # replicas = 0
           (65536, 4, 65536, P, Q, A, None, 0.0, 0.0),           # b * replicas beyond the grid
           (2, 4, 2, P, Q, None, K, 0.01, 0.05),                 # drawn angles with replicas > 1
           (2, 4, 1, P, Q, None, K, -0.01, 0.05),                # sigma < 0
           (2, 4, 1, P, Q, None, K, float("nan"), 0.05),         # sigma NaN
           (2, 4, 1, P, Q, None, K, 0.01, 0.0),                  # clip = 0 while jittering
           (2, 4, 1, P, Q, None, K, 0.01, -1.0),                 # clip < 0 while jittering
           (2, 4, 1, None, Q, None, K, 0.01, 0.05),              # null input
           (2, 4, 1, P, None, None, K, 0.01, 0.05),              # null output
           (2, 4, 1, P, Q, None, None, 0.0, 0.0),                # drawn angles need the key
           (2, 4, 1, P, Q, A, None, 0.01, 0.05),                 # jitter needs the key
           (2, 4, 1, P, P + 12, None, K, 0.01, 0.05),            # partial overlap
           (2, 4, 3, P, P, A, None, 0.0, 0.0)]                   # in place with replicas > 1
    for args in bad:
        assert f(*args) == -1, args
    assert f(0, 4, 1, None, None, None, None, 0.01, 0.05) == 0          # b = 0: nothing to do
    assert f(0, 4, 1, None, None, None, None, 0.0, 0.0) == 0
    assert _lib.launch_count() == before


def test_ops_argument_errors_and_cpu_tensors():
    x = torch.rand(2, 8, 3)
    for bad in (torch.rand(2, 8, 2), torch.rand(8, 3), torch.rand(2, 0, 3), np.zeros((2, 8, 3), np.float32)):
        with pytest.raises(ValueError):
            ops.rotate_jitter(bad)
        with pytest.raises(ValueError):
            ops.rotate_by_angles(bad, [0.0])
    for sigma, clip in ((-0.1, 0.05), (float("nan"), 0.05), (0.01, 0.0), (0.01, -1.0)):
        with pytest.raises(ValueError):
            ops.rotate_jitter(x, sigma, clip)
    with pytest.raises(ValueError):
        ops.rotate_by_angles(x, [])
    with pytest.raises(RuntimeError):
        ops.rotate_jitter(x)
    with pytest.raises(RuntimeError):
        ops.rotate_jitter(x, 0.0, 0.0)
    with pytest.raises(RuntimeError):
        ops.rotate_by_angles(x, [0.0, 1.0])
    with pytest.raises(ValueError):
        trainers.ClassifierTrainStep(torch.nn.Linear(1, 1), None, augment=True, clip=0.0)
    with pytest.raises(ValueError):
        trainers.ClassifierTrainStep(torch.nn.Linear(1, 1), None, augment=True, sigma=-1.0)
    for v in (0, -1, 1.5, True):
        with pytest.raises(ValueError):
            evaluation.ClassifierEvaluator(torch.nn.Linear(1, 1), num_votes=v)


def _small_net(cls, seed, classes=5):
    torch.manual_seed(seed)
    net = cls(num_classes=classes)
    if cls is tasknets.PointNetClsTransforms:   # T2 away from the identity, so that the regulariser counts
        torch.nn.init.normal_(net.transform_net2.transform.weight, std=0.05)
    return net


def test_train_one_epoch_is_the_host_loop_on_the_plain_module():
    g = torch.Generator().manual_seed(0)
    x, y = torch.rand(21, 64, 3, generator=g) - 0.5, torch.randint(0, 5, (21,), generator=g)
    net_a = _small_net(tasknets.PointNetCls, 1)
    net_b = copy.deepcopy(net_a)
    sa = trainers.ClassifierTrainStep(net_a, torch.optim.Adam(net_a.parameters(), lr=1e-3), batch_size=8)
    sb = trainers.ClassifierTrainStep(net_b, torch.optim.Adam(net_b.parameters(), lr=1e-3), batch_size=8)
    torch.manual_seed(5)
    res = sa.train_one_epoch(x, y)
    torch.manual_seed(5)
    perm = torch.randperm(21)
    loss_sum, correct = 0.0, 0
    for s in range(2):
        idx = perm[s * 8:(s + 1) * 8]
        loss, _, c = sb(x[idx], y[idx])
        loss_sum += float(loss)
        correct += c
    assert res["steps"] == 2 and sa.step == sb.step == 2
    assert res["mean_loss"] == loss_sum / 2 and res["accuracy"] == correct / 16
    for p, q in zip(net_a.parameters(), net_b.parameters()):
        assert torch.equal(p, q)
    with pytest.raises(ValueError):
        sa.train_one_epoch(x[:7], y[:7])


@pytest.mark.parametrize("cls", (tasknets.PointNetCls, tasknets.PointNetClsTransforms))
def test_one_vote_evaluator_is_eval_one_epoch_on_the_plain_module(cls):
    g = torch.Generator().manual_seed(2)
    x, y = torch.rand(19, 64, 3, generator=g) - 0.5, torch.randint(0, 5, (19,), generator=g)
    net = _small_net(cls, 3).eval()
    res = evaluation.ClassifierEvaluator(net).evaluate(x, y, batch_size=8, num_classes=5)
    preds, loss_sum = [], 0.0
    with torch.no_grad():
        for s in range(0, 19, 8):
            logits, ep = net(x[s:s + 8])
            loss_sum += float(net.get_loss(logits, y[s:s + 8], ep)) * logits.shape[0]
            preds.append(logits.argmax(1))
    pred = torch.cat(preds).numpy()
    assert np.array_equal(res["predictions"], pred)
    assert res["mean_loss"] == pytest.approx(loss_sum / 19, rel=1e-12)
    assert res["accuracy"] == np.mean(pred == y.numpy())
    assert len(res["class_accuracy"]) == 5


# ----------------------------------------------------------------------------------------------------- GPU: the kernel
@pytest.mark.gpu
@pytest.mark.parametrize("b,n", [(1, 1), (5, 777), (32, 1024), (64, 2048), (3, 16384)])
def test_rotate_jitter_matches_the_float64_restatement(b, n):
    g = torch.Generator().manual_seed(b * 7 + n)
    x = (torch.rand(b, n, 3, generator=g) * 2 - 1)
    got = ops.rotate_jitter(x.cuda(), 0.01, 0.05, key=_key_tensor(KEY)).cpu().numpy()
    ref = restate(x.numpy(), KEY, 0.01, 0.05)
    ok = _within_ulp(got, ref)
    assert ok.all(), (int((~ok).sum()), float(np.abs(got - ref).max()))
    rot = ops.rotate_jitter(x.cuda(), 0.0, 0.0, key=_key_tensor(KEY)).cpu().numpy()     # sigma = 0: the rotation alone
    assert _within_ulp(rot, restate(x.numpy(), KEY, 0.0, 0.0)).all()
    assert np.array_equal(rot[..., 1].view(np.int32), x.numpy()[..., 1].view(np.int32))   # y is left as it is
    empty = ops.rotate_jitter(torch.empty(0, n, 3, device="cuda"), key=_key_tensor(KEY))
    assert empty.shape == (0, n, 3)


@pytest.mark.gpu
def test_rotate_by_angles_matches_rotate_point_cloud_by_angle():
    V = 12
    g = torch.Generator().manual_seed(11)
    x = torch.rand(32, 1024, 3, generator=g) * 2 - 1
    angles = [v / float(V) * np.pi * 2 for v in range(V)]
    got = ops.rotate_by_angles(x.cuda(), angles).cpu().numpy()
    assert got.shape == (V, 32, 1024, 3)
    xs = x.numpy()
    for v in range(V):
        ref = np.stack([_rot(xs[i].astype(np.float64), angles[v]) for i in range(32)]).astype(np.float32)
        assert _within_ulp(got[v], ref).all(), v
        assert np.array_equal(got[v][..., 1].view(np.int32), xs[..., 1].view(np.int32))
    assert np.array_equal(got[0].view(np.int32), xs.view(np.int32))     # a rotation by 0 is the identity bit for bit


@pytest.mark.gpu
def test_distributions_of_the_angles_and_the_jitter(record_property):
    from scipy import stats

    b, n = 4096, 1024
    x = torch.zeros(b, n, 3, device="cuda")
    x[:, 0, 0] = 1.0                                 # point 0 of every cloud at (1, 0, 0): its rotation shows the angle
    rot = ops.rotate_jitter(x, 0.0, 0.0, key=_key_tensor(KEY))
    ang = torch.remainder(torch.atan2(rot[:, 0, 2].double(), rot[:, 0, 0].double()), 2 * math.pi).cpu().numpy()
    assert np.allclose(ang, drawn_angles(b, KEY), atol=1e-6)
    ks = stats.kstest(ang, stats.uniform(0, 2 * np.pi).cdf)
    record_property("angle_ks_p", ks.pvalue)
    assert ks.pvalue > 1e-3

    sigma, clip = 0.01, 0.015                        # clip at 1.5 sigma: about 13 % of the draws land on the bounds
    key2 = _key_tensor((KEY[1], KEY[0]))
    jit = ops.rotate_jitter(x, sigma, clip, key=key2)
    d = jit.double() - ops.rotate_jitter(x, 0.0, 0.0, key=key2).double()     # the same angles: the jitter alone
    assert float(d.abs().max()) <= clip + float(np.spacing(np.float32(1.0)))
    z = d[:, 1:].flatten().cpu().numpy()             # the points at the origin: the jitter up to its float32 rounding
    N = z.size
    a = clip / sigma
    p_out = 2 * stats.norm.cdf(-a)
    var = sigma ** 2 * ((1 - p_out) - 2 * a * stats.norm.pdf(a)) + clip ** 2 * p_out
    mean, var_hat = float(z.mean()), float(z.var())
    record_property("jitter_mean", mean)
    record_property("jitter_var_rel_err", var_hat / var - 1)
    assert abs(mean) <= 6 * math.sqrt(var / N)
    assert abs(var_hat - var) <= 6 * math.sqrt(2.0 / N) * var
    on_bound = np.abs(np.abs(z) - clip) <= 1e-9
    frac = float(on_bound.mean())
    assert abs(frac - p_out) <= 6 * math.sqrt(p_out * (1 - p_out) / N)
    inner = z[~on_bound][:200000]
    ks = stats.kstest(inner, stats.truncnorm(-a, a, scale=sigma).cdf)
    record_property("jitter_ks_p", ks.pvalue)
    assert ks.pvalue > 1e-3


@pytest.mark.gpu
def test_seeding_repeats_and_a_new_seed_changes():
    x = torch.rand(8, 500, 3, device="cuda")
    torch.manual_seed(7)
    a = ops.rotate_jitter(x)
    torch.manual_seed(7)
    b = ops.rotate_jitter(x)
    torch.manual_seed(8)
    c = ops.rotate_jitter(x)
    assert torch.equal(a, b)
    assert not torch.equal(a, c)
    d = ops.rotate_jitter(x)
    assert not torch.equal(b, d)


@pytest.mark.gpu
def test_graph_replays_draw_a_new_key_each():
    g = torch.Generator().manual_seed(3)
    xh = torch.rand(4, 300, 3, generator=g) - 0.5
    x = xh.cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            ops.rotate_jitter(x)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        key = torch.empty(2, dtype=torch.int64, device="cuda").random_()
        out = ops.rotate_jitter(x, key=key)
        out_default = ops.rotate_jitter(x)
    keys, outs = set(), []
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        words = _key_words(key)
        keys.add(words)
        assert _within_ulp(out.cpu().numpy(), restate(xh.numpy(), words, 0.01, 0.05)).all()
        outs.append(out_default.clone())
    assert len(keys) == 3
    assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[2])


@pytest.mark.gpu
def test_only_out_is_written_and_in_place_matches():
    from samplenet_b200 import _lib

    lib = _lib.lib()
    b, n, V, pad = 3, 333, 4, 1000
    x = torch.rand(b, n, 3, device="cuda") - 0.5
    key = _key_tensor(KEY)
    angles = torch.tensor([0.3, 1.0, 2.0, 5.5], dtype=torch.float64, device="cuda")
    for replicas, ang, sigma in ((1, None, 0.01), (V, angles, 0.0), (V, angles, 0.02)):
        size = replicas * b * n * 3
        buf = torch.full((size + 2 * pad,), float("nan"), device="cuda")
        buf[:pad] = 7.0
        buf[-pad:] = -3.0
        x0 = x.clone()
        rc = lib.snb200_rotate_jitter(b, n, replicas, x.data_ptr(), buf[pad:].data_ptr(), None if ang is None else ang.data_ptr(), key.data_ptr(),
                                      sigma, 0.05, torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize()
        assert torch.all(buf[:pad] == 7.0) and torch.all(buf[-pad:] == -3.0)
        assert not torch.isnan(buf[pad:-pad]).any()
        assert torch.equal(x, x0)
    y = x.clone()
    ref = ops.rotate_jitter(x, key=key)
    rc = lib.snb200_rotate_jitter(b, n, 1, y.data_ptr(), y.data_ptr(), None, key.data_ptr(), 0.01, 0.05, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    assert torch.equal(y, ref)


# ----------------------------------------------------------------------------------------------------- GPU: training
def _gpu_batch(n, seed, classes=40):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, 1024, 3, generator=g) * 2 - 1).cuda(), torch.randint(0, classes, (n,), generator=g).cuda()


WRAPPERS = ((tasknets.PointNetCls, tasknets.CudaPointNetCls), (tasknets.PointNetClsTransforms, tasknets.CudaPointNetClsTransforms))


def _pair(cls, wrap, **kw):
    torch.manual_seed(0)
    net = cls().cuda()
    out = []
    for _ in range(2):
        w = wrap(copy.deepcopy(net))
        out.append((w, trainers.ClassifierTrainStep(w, torch.optim.Adam(w.parameters(), lr=1e-3), **kw)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("cls,wrap", WRAPPERS)
def test_augmented_step_is_the_manual_composition(cls, wrap):
    (wa, sa), (wb, sb) = _pair(cls, wrap)
    sa.augment = True
    x, y = _gpu_batch(32, 1)
    for seed in (10, 11):
        torch.manual_seed(seed)
        la, pa, ca = sa(x, y)
        torch.manual_seed(seed)
        key = torch.empty(2, dtype=torch.int64, device="cuda").random_()
        lb, pb, cb = sb(ops.rotate_jitter(x, 0.01, 0.05, key=key), y)
        assert wa.route == wb.route == "cuda"
        assert torch.equal(la, lb) and torch.equal(pa, pb) and ca == cb
        for p, q in zip(wa.parameters(), wb.parameters()):
            assert torch.equal(p, q)


@pytest.mark.gpu
@pytest.mark.parametrize("cls,wrap", WRAPPERS)
def test_train_one_epoch_is_the_host_loop_of_steps(cls, wrap):
    B, n = 16, 53
    (wa, sa), (wb, sb) = _pair(cls, wrap, batch_size=B, augment=True)
    init = copy.deepcopy(wa.state_dict())
    x, y = _gpu_batch(n, 2)
    torch.manual_seed(21)
    perm = torch.randperm(n, device="cuda")
    losses, correct = [], 0
    for s in range(n // B):
        idx = perm[s * B:(s + 1) * B]
        loss, _, c = sb(x[idx], y[idx])
        losses.append(float(loss))
        correct += c
    x_nan = x.clone()
    x_nan[perm[(n // B) * B:]] = float("nan")        # the remainder is not used
    torch.manual_seed(21)
    res = sa.train_one_epoch(x_nan, y)
    assert res["steps"] == n // B
    assert res["mean_loss"] == sum(losses) / len(losses)
    assert res["accuracy"] == correct / ((n // B) * B)
    for p, q in zip(wa.parameters(), wb.parameters()):
        assert torch.equal(p, q)
    after = copy.deepcopy(wa.state_dict())
    wa.load_state_dict(init)
    sa.optimizer = torch.optim.Adam(wa.parameters(), lr=1e-3)
    sa.step = 0
    torch.manual_seed(21)
    again = sa.train_one_epoch(x_nan, y)             # a re-seeded epoch repeats bit for bit
    assert again == res
    for k, v in wa.state_dict().items():
        assert torch.equal(v, after[k]), k


# ----------------------------------------------------------------------------------------------------- GPU: evaluation
@pytest.fixture
def _tf32_off(monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


def _per_vote(net, x, y, V, batch_size, regulariser_once=False):
    """evaluate_classifier.py:128-222 restated: numpy rotations per vote, one classifier call per vote (or, regulariser_once, the wrong
    single get_loss over all V * b rows).  -> (summed logits (n, C) float64, mean loss, the largest |logit| of one vote)."""
    angles = [v / float(V) * np.pi * 2 for v in range(V)]
    xs, out, loss_sum, top = x.cpu().numpy(), [], 0.0, 0.0
    with torch.no_grad():
        for s in range(0, x.shape[0], batch_size):
            pc, lab = xs[s:s + batch_size], y[s:s + batch_size]
            b = pc.shape[0]
            rot = [torch.from_numpy(np.stack([_rot(pc[i].astype(np.float64), a) for i in range(b)]).astype(np.float32)).cuda() for a in angles]
            summed, batch_loss = torch.zeros(b, 40, dtype=torch.float64, device="cuda"), 0.0
            if regulariser_once:
                logits, ep = net(torch.cat(rot))
                summed = logits.double().view(V, b, -1).sum(0)
                batch_loss = float(net.get_loss(logits, lab.repeat(V), ep)) * b
            else:
                for r in rot:
                    logits, ep = net(r)
                    top = max(top, float(logits.abs().max()))
                    summed += logits.double()
                    batch_loss += float(net.get_loss(logits, lab, ep)) * b / float(V)
            out.append(summed)
            loss_sum += batch_loss
    return torch.cat(out), loss_sum / x.shape[0], top


def _margin(logits):
    top = torch.topk(logits, 2, dim=1).values
    return (top[:, 0] - top[:, 1]).cpu().numpy()


@pytest.mark.gpu
def test_twelve_votes_match_the_per_vote_restatement(_tf32_off, record_property):
    torch.manual_seed(4)
    net = tasknets.PointNetCls().cuda().eval()
    x, y = _gpu_batch(70, 3)
    res = evaluation.ClassifierEvaluator(net, num_votes=12).evaluate(x, y, batch_size=32, num_classes=40)
    summed, mean_loss, _ = _per_vote(net, x, y, 12, 32)
    pred = summed.argmax(1).cpu().numpy()
    record_property("min_margin", float(_margin(summed).min()))
    assert np.array_equal(res["predictions"], pred)
    assert res["mean_loss"] == pytest.approx(mean_loss, rel=1e-6)
    acc, per_class, avg = evaluation.class_accuracies(*[t.cpu().numpy() for t in evaluation.classification_counts(summed, y, 40)[1:]])
    assert res["accuracy"] == acc
    assert np.array_equal(res["class_accuracy"], per_class, equal_nan=True)


@pytest.mark.gpu
def test_transform_regulariser_is_taken_per_vote(_tf32_off, record_property):
    net = _small_net(tasknets.PointNetClsTransforms, 5, classes=40).cuda().eval()
    x, y = _gpu_batch(40, 4)
    res = evaluation.ClassifierEvaluator(net, num_votes=3).evaluate(x, y, batch_size=16)
    _, per_vote, _ = _per_vote(net, x, y, 3, 16)
    _, once, _ = _per_vote(net, x, y, 3, 16, regulariser_once=True)
    record_property("per_vote", per_vote)
    record_property("once", once)
    assert res["mean_loss"] == pytest.approx(per_vote, rel=1e-5)
    assert abs(once - per_vote) > 1e-3 * abs(per_vote)


@pytest.mark.gpu
def test_frozen_wrapper_votes_agree_with_the_plain_module(_tf32_off, record_property):
    torch.manual_seed(6)
    net = tasknets.PointNetClsTransforms().cuda().eval().requires_grad_(False)
    frozen = tasknets.FrozenPointNetClsTransforms(net)
    x, y = _gpu_batch(70, 5)
    V = 12
    angles = [v / float(V) * np.pi * 2 for v in range(V)]
    with torch.no_grad():
        rot = ops.rotate_by_angles(x[:32].contiguous(), angles).flatten(0, 1)
        lf, lp = frozen(rot)[0], net(rot)[0]
    err = float((lf - lp).abs().max() / lp.abs().max())
    record_property("frozen_logit_err", err)
    assert err <= FRONT_BAR
    rf = evaluation.ClassifierEvaluator(frozen, num_votes=V).evaluate(x, y)
    rp = evaluation.ClassifierEvaluator(net, num_votes=V).evaluate(x, y)
    summed, _, top = _per_vote(net, x, y, V, 32)
    sure = _margin(summed) > 2 * V * FRONT_BAR * top   # each side's vote sum is within V * FRONT_BAR * top of the exact one
    record_property("decided", int(sure.sum()))
    assert sure.sum() >= 60
    assert np.array_equal(rf["predictions"][sure], rp["predictions"][sure])
    assert rf["mean_loss"] == pytest.approx(rp["mean_loss"], rel=1e-4)
