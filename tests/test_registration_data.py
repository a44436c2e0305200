"""The registration trainer's data path on CUDA: snb200_registration_pairs (csrc/registration_data.cu), ops.registration_pairs,
registration.random_transforms / on_unit_cube / CudaQuaternionFixedDataset / get_datasets and RegistrationStep.train_1.

CPU: random_transforms bit for bit against the reference's QuaternionFixedDataset tables (tests/golden/registration_data.npz, written by
make_registration_data_golden.py from the reference's own classes); on_unit_cube against ModelNetCls.__getitem__'s normalised items; the
entry's argument checks, which launch nothing; the ops' argument errors and refusal of CPU tensors; get_datasets' repeats and seeds; train_1
on a plain PCRNet against the host loop of train_step and .item().
GPU (H100): the permutation against the Philox restatement of test_classifier_augmentation, p0 exactly, p1 bit for bit against a float32
restatement of qrot and within 1e-6 of float64, vec, at four sizes with records that wrap past the set; the reference fixture's pairs; seeding,
CUDA graph replays and the distribution of one point's position; the write set; train_1 bit for bit against a manual loop with CudaPCRNet, and
eval_1 / test_1 over the set's batches against explicit batches."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from samplenet_b200 import ops, registration  # noqa: E402
from test_classifier_augmentation import philox  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "registration_data.npz")
KEY = (0x243F6A8885A308D3, 0x13198A2E03707344)   # a key with both halves of both words set
EUNSUPPORTED = -4


# ----------------------------------------------------------------------------------------------------- restatements
def restate_perm(b, n, key):
    """perm (b, n) of the documented stream: Philox4x32-10 with key (lo32(k0), hi32(k0)), counter (i, j, lo32(k1), hi32(k1)), sort keys
    ((w0 << 32 | w1) & ~0x7FF) | j in ascending order."""
    k0, k1 = key
    i = np.arange(b, dtype=np.uint64)[:, None]
    j = np.arange(n, dtype=np.uint64)[None, :]
    w = philox(i, j, k1 & 0xFFFFFFFF, k1 >> 32, k0 & 0xFFFFFFFF, k0 >> 32)
    keys = (((w[0] << np.uint64(32)) | w[1]) & ~np.uint64(0x7FF)) | j
    return np.argsort(keys, axis=1).astype(np.int32)


def qrot_np(q, v):
    """registration.qrot in q's and v's dtype, one rounding per operation: uv = qvec x v, uuv = qvec x uv, v + 2 (w uv + uuv)."""
    w, x, y, z = (q[:, None, c] for c in range(4))
    vx, vy, vz = v[..., 0], v[..., 1], v[..., 2]
    ux, uy, uz = y * vz - z * vy, z * vx - x * vz, x * vy - y * vx
    wx, wy, wz = y * uz - z * uy, z * ux - x * uz, x * uy - y * ux
    two = v.dtype.type(2)
    return np.stack([vx + two * (w * ux + wx), vy + two * (w * uy + wy), vz + two * (w * uz + wz)], axis=-1)


def _key_tensor(key, dev="cuda"):
    return torch.tensor([k - (1 << 64) if k >= 1 << 63 else k for k in key], dtype=torch.int64, device=dev)


def _key_words(t):
    return tuple(int(v) & 0xFFFFFFFFFFFFFFFF for v in t.cpu().tolist())


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


# ----------------------------------------------------------------------------------------------------- CPU
def test_random_transforms_are_the_reference_tables_bit_for_bit():
    z = np.load(GOLDEN)
    for seed, count in ((0, 4925), (1, 500)):
        got = registration.random_transforms(count, seed)
        want = z["transforms_seed%d" % seed]
        assert got.dtype == np.float32 and got.shape == (count, 7)
        assert np.array_equal(_bits(got), _bits(want)), seed
    state = np.random.get_state()[1].copy()
    registration.random_transforms(10, 3)
    assert np.array_equal(np.random.get_state()[1], state)        # numpy's global state is left alone


def test_on_unit_cube_matches_the_reference_items():
    z = np.load(GOLDEN)
    m = int(z["num_points"])
    clouds = z["clouds"]
    cube = registration.on_unit_cube(torch.from_numpy(clouds[:, :m])).numpy()
    for r in range(z["p0"].shape[0]):
        got = cube[r % clouds.shape[0]][z["perm"][r]]
        assert np.abs(got.astype(np.float64) - z["p0"][r]).max() <= 1e-6, r


def test_library_exports_the_entry():
    from samplenet_b200 import _lib

    assert "snb200_registration_pairs" in _lib.exported_symbols()
    assert hasattr(_lib.lib(), "snb200_registration_pairs")
    assert "int snb200_registration_pairs(" in open(os.path.join(os.path.dirname(HERE), "include", "samplenet_b200.h")).read()


def test_entry_rejects_bad_arguments_and_launches_nothing():
    from samplenet_b200 import _lib

    lib = _lib.lib()
    f = lambda *a: lib.snb200_registration_pairs(*a, None)
    C, R, T, K = 1 << 32, 1 << 33, 1 << 34, 1 << 35                 # never dereferenced: every call below fails its checks or has b = 0
    P0, P1, V, PM = 1 << 40, 1 << 41, 1 << 42, 1 << 43
    ok = (4, 16, 3, 12, C, R, T, K, P0, P1, V, PM)

    def with_(**kw):
        names = ("b", "n", "s", "num_records", "clouds", "records", "transforms", "key", "p0", "p1", "vec", "perm")
        a = dict(zip(names, ok))
        a.update(kw)
        return tuple(a[k] for k in names)

    before = _lib.launch_count()
    bad = [with_(b=-1), with_(n=0), with_(s=0), with_(num_records=0),
           with_(clouds=None), with_(records=None), with_(transforms=None), with_(key=None), with_(p0=None), with_(p1=None), with_(vec=None),
           with_(p1=P0 + 4 * 16 * 3 * 4 - 4),            # p1 starts inside p0
           with_(vec=P1 + 8),                            # vec inside p1
           with_(perm=P0 + 64),                          # perm inside p0
           with_(p0=C + 4),                              # p0 overlaps the clouds
           with_(vec=R), with_(perm=T + 4), with_(p1=K + 8 - 4)]
    for args in bad:
        assert f(*args) == -1, args
    assert f(*with_(n=2049)) == EUNSUPPORTED
    assert f(*with_(n=1 << 20)) == EUNSUPPORTED
    assert f(*with_(b=0, clouds=None, records=None, transforms=None, key=None, p0=None, p1=None, vec=None, perm=None)) == 0
    assert _lib.launch_count() == before


def test_ops_argument_errors_and_cpu_tensors():
    clouds, records, tr = torch.rand(3, 8, 3), torch.arange(4, dtype=torch.int32), torch.rand(5, 7)
    for bad in (torch.rand(3, 8, 2), torch.rand(8, 3), torch.rand(0, 8, 3), torch.rand(3, 0, 3), torch.rand(3, 2049, 3),
                np.zeros((3, 8, 3), np.float32)):
        with pytest.raises(ValueError):
            ops.registration_pairs(bad, records, tr)
    for bad in (torch.arange(4.0), torch.zeros(2, 2, dtype=torch.int32), [0, 1]):
        with pytest.raises(ValueError):
            ops.registration_pairs(clouds, bad, tr)
    for bad in (torch.rand(5, 6), torch.rand(7), torch.rand(0, 7)):
        with pytest.raises(ValueError):
            ops.registration_pairs(clouds, records, bad)
    with pytest.raises(RuntimeError):
        ops.registration_pairs(clouds, records, tr)
    with pytest.raises(RuntimeError):
        ops.registration_pairs(clouds, records, tr, key=torch.zeros(2, dtype=torch.int64), return_perm=True)
    for bad in (np.zeros((2, 8, 2), np.float32), np.zeros((0, 8, 3), np.float32)):
        with pytest.raises(ValueError):
            registration.CudaQuaternionFixedDataset(bad)
    with pytest.raises(ValueError):
        registration.CudaQuaternionFixedDataset(np.zeros((2, 8, 3), np.float32), repeat=0)


def test_get_datasets_takes_the_reference_repeats_and_seeds(monkeypatch):
    made = []

    class Recorder:
        def __init__(self, points, num_points=1024, repeat=1, seed=0):
            made.append((points, num_points, repeat, seed))

    monkeypatch.setattr(registration, "CudaQuaternionFixedDataset", Recorder)
    train, test = np.zeros((197, 4, 3), np.float32), np.zeros((50, 4, 3), np.float32)
    a, b = registration.get_datasets(train, test, num_points=512)
    assert isinstance(a, Recorder) and isinstance(b, Recorder)
    assert [m[1:] for m in made] == [(512, 25, 0), (512, 1, 0)] and made[0][0] is train and made[1][0] is test
    made.clear()
    registration.get_datasets(np.zeros((6000, 4, 3), np.float32), test)
    assert made[0][2] == 1                                  # max(int(5000 / S), 1)
    made.clear()
    a, b = registration.get_datasets(None, test, test=True)
    assert a is None and [m[1:] for m in made] == [(1024, 5, 1)]


def _cpu_chamfer():
    class Chamfer(torch.nn.Module):   # squared distances to the nearest neighbour, as ChamferDistance, in torch ops on the host
        def forward(self, a, b):
            d = ((a[:, :, None, :] - b[:, None, :, :]) ** 2).sum(-1)
            return d.min(dim=2)[0], d.min(dim=1)[0]

    return Chamfer


def test_train_1_is_the_host_loop_of_train_step_on_the_plain_module(monkeypatch):
    monkeypatch.setattr(registration, "ChamferDistance", _cpu_chamfer())
    act = registration.RegistrationStep(sampler="none", train_pcrnet=True)
    torch.manual_seed(0)
    net_a = act.create_model()
    net_b = copy.deepcopy(net_a)
    g = torch.Generator().manual_seed(1)
    tr = torch.from_numpy(registration.random_transforms(10, 0))
    batches = []
    for s, e in ((0, 4), (4, 8), (8, 10)):
        p0 = registration.on_unit_cube(torch.rand(e - s, 32, 3, generator=g))
        batches.append((p0, registration.QuaternionTransform(tr[s:e]).rotate(p0), {"vec": tr[s:e], "inversion": torch.tensor([False])}))
    opt_a = torch.optim.Adam(filter(lambda p: p.requires_grad, net_a.parameters()), lr=1e-3)
    opt_b = torch.optim.Adam(filter(lambda p: p.requires_grad, net_b.parameters()), lr=1e-3)
    vloss, gloss = act.train_1(net_a, batches, opt_a, "cpu")
    v, gl = 0.0, 0.0
    for data in batches:                                   # main.py:306-362
        loss, rot, _ = act.train_step(net_b, data, opt_b, "cpu")
        v += loss.item()
        gl += rot.item()
    assert vloss == v / 3 and gloss == gl / 3
    for p, q in zip(net_a.parameters(), net_b.parameters()):
        assert torch.equal(p, q)
    with pytest.raises(ValueError):
        act.train_1(net_a, [], opt_a, "cpu")


# ----------------------------------------------------------------------------------------------------- GPU: the kernel
def _set(s, n, num_records, seed):
    g = torch.Generator().manual_seed(seed)
    clouds = (torch.rand(s, n, 3, generator=g) - 0.5) * torch.tensor([1.0, 0.7, 0.4])     # the size of a cloud on the unit cube
    return clouds.cuda(), torch.from_numpy(registration.random_transforms(num_records, seed)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("n", (1, 7, 1024, 2048))
def test_pairs_are_the_documented_draw(n):
    s, num_records, b = 3, 12, 10
    clouds, tr = _set(s, n, num_records, n)
    records = torch.tensor([0, 11, 4, 5, 3, 9, 1, 7, 11, 2], dtype=torch.int32, device="cuda")   # wraps past s; a repeat
    p0, p1, vec, perm = ops.registration_pairs(clouds, records, tr, key=_key_tensor(KEY), return_perm=True)
    assert p0.shape == p1.shape == (b, n, 3) and vec.shape == (b, 7) and perm.shape == (b, n) and perm.dtype == torch.int32
    want_perm = restate_perm(b, n, KEY)
    assert np.array_equal(perm.cpu().numpy(), want_perm)
    rec, c, t = records.cpu().numpy(), clouds.cpu().numpy(), tr.cpu().numpy()
    gathered = np.stack([c[rec[i] % s][want_perm[i]] for i in range(b)])
    assert np.array_equal(_bits(p0.cpu().numpy()), _bits(gathered))
    q = t[rec, :4]
    got1 = p1.cpu().numpy()
    assert np.array_equal(_bits(got1), _bits(qrot_np(q, gathered)))
    assert np.abs(got1.astype(np.float64) - qrot_np(q.astype(np.float64), gathered.astype(np.float64))).max() <= 1e-6
    assert np.array_equal(_bits(vec.cpu().numpy()), _bits(t[rec]))
    p0b, p1b, vecb = ops.registration_pairs(clouds, records.long(), tr, key=_key_tensor(KEY))      # int64 records, no perm: the same pairs
    assert torch.equal(p0b, p0) and torch.equal(p1b, p1) and torch.equal(vecb, vec)


@pytest.mark.gpu
def test_more_than_2048_points_is_unsupported():
    from samplenet_b200 import _lib

    n = 2049
    clouds, tr = torch.zeros(2, n, 3, device="cuda"), torch.zeros(2, 7, device="cuda")
    records, key = torch.zeros(1, dtype=torch.int32, device="cuda"), _key_tensor(KEY)
    p0, p1 = torch.empty(1, n, 3, device="cuda"), torch.empty(1, n, 3, device="cuda")
    vec = torch.empty(1, 7, device="cuda")
    before = _lib.launch_count()
    rc = _lib.lib().snb200_registration_pairs(1, n, 2, 2, clouds.data_ptr(), records.data_ptr(), tr.data_ptr(), key.data_ptr(), p0.data_ptr(),
                                              p1.data_ptr(), vec.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
    assert rc == EUNSUPPORTED and _lib.launch_count() == before


@pytest.mark.gpu
def test_pairs_match_the_reference_fixture():
    z = np.load(GOLDEN)
    ds = registration.CudaQuaternionFixedDataset(z["clouds"], num_points=int(z["num_points"]), repeat=int(z["repeat"]), seed=0)
    b = z["p0"].shape[0]
    assert len(ds) == b and ds.clouds.shape == (3, int(z["num_points"]), 3)
    records = torch.arange(b, dtype=torch.int32, device="cuda")
    p0, p1, vec, perm = ops.registration_pairs(ds.clouds, records, ds.transforms, return_perm=True)
    assert np.array_equal(_bits(vec.cpu().numpy()), _bits(z["vec"]))
    ours, theirs = np.empty_like(z["p1"]), np.empty_like(z["p1"])
    pm = perm.cpu().numpy()
    for i in range(b):                                     # undo both point orders
        ours[i, pm[i]] = p1[i].cpu().numpy()
        theirs[i, z["perm"][i]] = z["p1"][i]
    assert np.abs(ours.astype(np.float64) - theirs).max() <= 1e-6
    bp0, bp1, igt = ds.batch(records)                      # the set's batch: the same clouds and transforms, a new point order
    assert igt["inversion"].device.type == "cpu" and not bool(igt["inversion"][0])
    assert torch.equal(igt["vec"], vec)
    assert torch.equal(torch.sort(bp0.view(b, -1), dim=1)[0], torch.sort(p0.view(b, -1), dim=1)[0])


@pytest.mark.gpu
def test_seeding_repeats_graphs_replay_new_keys_and_one_point_lands_uniformly():
    from scipy import stats

    clouds, tr = _set(4, 300, 8, 3)
    records = torch.tensor([0, 5, 7, 2], dtype=torch.int32, device="cuda")
    torch.manual_seed(7)
    a = ops.registration_pairs(clouds, records, tr, return_perm=True)
    torch.manual_seed(7)
    b = ops.registration_pairs(clouds, records, tr, return_perm=True)
    torch.manual_seed(8)
    c = ops.registration_pairs(clouds, records, tr, return_perm=True)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not torch.equal(a[3], c[3]) and not torch.equal(a[0], c[0])
    d = ops.registration_pairs(clouds, records, tr, return_perm=True)
    assert not torch.equal(c[3], d[3])

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            ops.registration_pairs(clouds, records, tr)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        key = torch.empty(2, dtype=torch.int64, device="cuda").random_()
        _, _, _, perm = ops.registration_pairs(clouds, records, tr, key=key, return_perm=True)
        _, _, _, perm_default = ops.registration_pairs(clouds, records, tr, return_perm=True)
    keys, outs = set(), []
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        words = _key_words(key)
        keys.add(words)
        assert np.array_equal(perm.cpu().numpy(), restate_perm(4, 300, words))
        outs.append(perm_default.clone())
    assert len(keys) == 3
    assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[2])

    n, pairs = 64, 4096
    small, tr_small = _set(1, n, 1, 4)
    torch.manual_seed(11)
    _, _, _, perm = ops.registration_pairs(small, torch.zeros(pairs, dtype=torch.int32, device="cuda"), tr_small, return_perm=True)
    assert torch.equal(torch.sort(perm, dim=1)[0], torch.arange(n, dtype=torch.int32, device="cuda").expand(pairs, n))
    where = (perm == 0).int().argmax(dim=1).cpu().numpy()
    counts = np.bincount(where, minlength=n)
    assert stats.chisquare(counts).pvalue > 1e-3


@pytest.mark.gpu
def test_only_the_outputs_are_written():
    from samplenet_b200 import _lib

    b, n, s, pad = 5, 333, 3, 1000
    clouds, tr = _set(s, n, 9, 5)
    records = torch.tensor([8, 0, 4, 3, 7], dtype=torch.int32, device="cuda")
    key = _key_tensor(KEY)
    inputs = [t.clone() for t in (clouds, records, tr, key)]
    ref = ops.registration_pairs(clouds, records, tr, key=key, return_perm=True)
    for with_perm in (True, False):
        bufs = []
        for size, dtype, canary in ((b * n * 3, torch.float32, float("nan")), (b * n * 3, torch.float32, float("nan")), (b * 7, torch.float32, float("nan")),
                                    (b * n, torch.int32, -7)):
            buf = torch.full((size + 2 * pad,), canary, dtype=dtype, device="cuda")
            buf[:pad] = 7
            buf[-pad:] = -3
            bufs.append(buf)
        rc = _lib.lib().snb200_registration_pairs(b, n, s, 9, clouds.data_ptr(), records.data_ptr(), tr.data_ptr(), key.data_ptr(),
                                                  *[buf[pad:].data_ptr() for buf in bufs[:3]], bufs[3][pad:].data_ptr() if with_perm else None,
                                                  torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize()
        for buf in bufs:
            assert torch.all(buf[:pad] == 7) and torch.all(buf[-pad:] == -3)
        for buf, want in zip(bufs[:3], ref[:3]):
            assert torch.equal(buf[pad:-pad], want.flatten())
        if with_perm:
            assert torch.equal(bufs[3][pad:-pad], ref[3].flatten())
        else:
            assert torch.all(bufs[3][pad:-pad] == -7)
        for t, t0 in zip((clouds, records, tr, key), inputs):
            assert torch.equal(t, t0)


# ----------------------------------------------------------------------------------------------------- GPU: the trainer
def _gpu_set(num_clouds, points, num_points, repeat, seed=0):
    g = torch.Generator().manual_seed(seed)
    raw = torch.rand(num_clouds, points, 3, generator=g) * torch.tensor([1.0, 0.8, 0.5])
    return registration.CudaQuaternionFixedDataset(raw.numpy(), num_points=num_points, repeat=repeat, seed=seed)


@pytest.mark.gpu
def test_train_1_on_the_set_is_the_manual_loop_with_cuda_pcrnet():
    act = registration.RegistrationStep(sampler="none", train_pcrnet=True)
    torch.manual_seed(0)
    model_a = act.create_model(cuda_task=True).cuda()
    model_b = copy.deepcopy(model_a)
    ds = _gpu_set(5, 300, 256, 3)
    assert len(ds) == 15
    opt_a = torch.optim.Adam(filter(lambda p: p.requires_grad, model_a.parameters()), lr=1e-3)
    opt_b = torch.optim.Adam(filter(lambda p: p.requires_grad, model_b.parameters()), lr=1e-3)
    torch.manual_seed(3)
    vloss, gloss = act.train_1(model_a, ds.batches(4, shuffle=True), opt_a, "cuda")
    torch.manual_seed(3)
    v, gl, sizes = 0.0, 0.0, []
    for data in ds.batches(4, shuffle=True):
        sizes.append(data[0].shape[0])
        loss, rot, _ = act.train_step(model_b, data, opt_b, "cuda")
        v += loss.item()
        gl += rot.item()
    assert sizes == [4, 4, 4, 3]                            # the last partial batch is kept, as DataLoader(drop_last=False)
    assert vloss == v / 4 and gloss == gl / 4
    for p, q in zip(model_a.parameters(), model_b.parameters()):
        assert torch.equal(p, q)
    assert [d[0].shape[0] for d in ds.batches(4, drop_last=True)] == [4, 4, 4]


@pytest.mark.gpu
def test_eval_1_and_test_1_over_the_set_are_the_calls_over_explicit_batches():
    act = registration.RegistrationStep(sampler="none")
    torch.manual_seed(1)
    model = act.create_model(frozen_task=True).cuda()
    ds = _gpu_set(7, 1100, 1024, 6, seed=2)
    assert len(ds) == 42 and ds.num_points == 1024

    def explicit():
        return [ds.batch(torch.arange(s, min(s + 32, len(ds)), dtype=torch.int32)) for s in range(0, len(ds), 32)]

    torch.manual_seed(5)
    e1 = act.eval_1(model, ds.batches(32), "cuda")
    torch.manual_seed(5)
    e2 = act.eval_1(model, explicit(), "cuda")
    assert e1 == e2
    torch.manual_seed(6)
    t1 = act.test_1(model, ds.batches(32), "cuda")
    torch.manual_seed(6)
    t2 = act.test_1(model, explicit(), "cuda")
    assert len(t1["rotation_errors"]) == 42
    for k in ("rotation_errors", "trans_errs", "consistency_errors"):
        assert np.array_equal(t1[k], t2[k]), k
    assert t1["auc"] == t2["auc"]
