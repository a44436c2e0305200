"""Non-finite input: the index contract of the distance, matching and pool kernels, the non-finite step guard (ops.NonfiniteGuard,
snb200_nonfinite_guard) and skip_nonfinite=True on the training runners (trainers.SamplerTrainStep, ClassifierTrainStep,
AutoencoderTrainStep).

CPU: the entry is declared and in the ctypes table; skip_nonfinite refuses an optimiser whose state the guard cannot restore.
GPU (H100): every index an entry writes stays in range on NaN / Inf clouds, and the finite clouds of a batch holding a NaN cloud give what
they give alone, bit for bit; the guard against a torch restatement, bit for bit, eager and captured, writing only its own buffers; the
runners, eager and graphed, leave everything as it was across a non-finite step, count skipped steps, and change nothing on finite data."""
import ctypes
import os
import re
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from samplenet_b200 import _lib, ops, tasknets, trainers  # noqa: E402

B, N_PTS, M, CLASSES = 8, 256, 32, 5
NAN = float("nan")


# ----------------------------------------------------------------------------------------------------- CPU
def test_guard_entry_is_declared_and_mirrored():
    hdr = open(os.path.join(ROOT, "include", "samplenet_b200.h")).read()
    assert re.search(r"\bint snb200_nonfinite_guard\s*\(", hdr)
    assert "snb200_nonfinite_guard" in _lib.exported_symbols()
    # the ctypes mirrors have the C layout: pointer, int, int / pointer, pointer, long long
    assert ctypes.sizeof(_lib.GuardCheck) == 16 and _lib.GuardCheck.count.offset == 8 and _lib.GuardCheck.dtype.offset == 12
    assert ctypes.sizeof(_lib.GuardRestore) == 24 and _lib.GuardRestore.bytes.offset == 16


def test_skip_nonfinite_refuses_optimizers_it_cannot_restore():
    lin = torch.nn.Linear(3, 3)
    cls_step = trainers.ClassificationStep(torch.nn.Linear(1, 1), torch.nn.Linear(1, 1), 32)
    makers = [lambda opt: trainers.SamplerTrainStep(cls_step, opt, skip_nonfinite=True),
              lambda opt: trainers.ClassifierTrainStep(lin, opt, skip_nonfinite=True),
              lambda opt: trainers.AutoencoderTrainStep(lin, opt, skip_nonfinite=True)]
    for make in makers:
        with pytest.raises(ValueError, match="capturable=True"):          # the step count of a non-capturable Adam lives on the host
            make(torch.optim.Adam(lin.parameters()))
        with pytest.raises(ValueError, match="torch.optim.Adam, torch.optim.AdamW"):   # NAdam's fresh state is not zeros
            make(torch.optim.NAdam(lin.parameters(), capturable=True))
        with pytest.raises(ValueError):
            make(torch.optim.SGD(lin.parameters(), lr=0.1))
    # the default takes any optimiser, as before
    assert trainers.ClassifierTrainStep(lin, torch.optim.SGD(lin.parameters(), lr=0.1))._skip is None


# ----------------------------------------------------------------------------------------------------- GPU: index contract
POISON = ["query_nan", "ref_nan", "inf", "both_nan"]
BAD = 1                                         # the poisoned cloud of a batch of 3


def _pair(poison, b=3, n=300, m=40, seed=0):
    """(ref (b,n,3), samp (b,m,3)) finite, and the same with cloud BAD poisoned."""
    g = torch.Generator().manual_seed(seed)
    ref, samp = torch.rand(b, n, 3, generator=g) - 0.5, torch.rand(b, m, 3, generator=g) - 0.5
    r2, s2 = ref.clone(), samp.clone()
    if poison in ("query_nan", "both_nan"):
        s2[BAD] = NAN
    if poison in ("ref_nan", "both_nan"):
        r2[BAD] = NAN
    if poison == "inf":
        r2[BAD, 0::2] = float("inf")
        r2[BAD, 1::2] = -float("inf")
        s2[BAD, : m // 2, 1] = float("inf")
    return ref.cuda(), samp.cuda(), r2.cuda(), s2.cuda()


def _in_range(idx, n):
    assert idx.dtype == torch.int32
    assert int(idx.min()) >= 0 and int(idx.max()) < n, (int(idx.min()), int(idx.max()), n)


def _same_finite(a, b):
    """Outputs of the finite clouds (every cloud but BAD) equal bit for bit."""
    keep = [i for i in range(a.shape[0]) if i != BAD]
    assert torch.equal(a[keep], b[keep])


@pytest.mark.gpu
@pytest.mark.parametrize("poison", POISON)
def test_nn_distance_and_simplification_loss_indices_stay_in_range(poison):
    ref, samp, r2, s2 = _pair(poison)
    n, m = ref.shape[1], samp.shape[1]
    clean = ops.nn_distance_forward(samp, ref)
    bad = ops.nn_distance_forward(s2, r2)
    _in_range(bad[1], n)
    _in_range(bad[3], m)
    if poison != "inf":
        assert torch.equal(bad[1][BAD], torch.zeros_like(bad[1][BAD]))     # nothing compares: index 0, as tf_nndistance
    for a, c in zip(bad, clean):
        _same_finite(a, c)
    g1, g2 = torch.ones_like(clean[0]), torch.ones_like(clean[2])
    gc = ops.nn_distance_backward(samp, ref, g1, clean[1], g2, clean[3])
    gb = ops.nn_distance_backward(s2, r2, g1, bad[1], g2, bad[3])
    for a, c in zip(gb, gc):
        _same_finite(a, c)
    out_c = ops.simplification_loss_forward(samp, ref, 1.0)
    out_b = ops.simplification_loss_forward(s2, r2, 1.0)
    _in_range(out_b[2], n)
    _in_range(out_b[4], m)
    for a, c in zip(out_b[1:], out_c[1:]):
        _same_finite(a, c)
    assert not torch.isfinite(out_b[0][3])                                # the loss stays non-finite
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("poison", POISON)
def test_projection_indices_stay_in_range(poison):
    ref, samp, r2, s2 = _pair(poison)
    n, m = ref.shape[1], samp.shape[1]
    sigma = torch.full((1,), 0.05, device="cuda")
    want = ("proj", "idx", "weights", "dist")
    clean = ops.knn_soft_project_forward(ref, samp, 7, "bnc", sigma=sigma, want=want)
    bad = ops.knn_soft_project_forward(r2, s2, 7, "bnc", sigma=sigma, want=want)
    _in_range(bad["idx"], n)
    for k in want:
        _same_finite(bad[k], clean[k])
    t = torch.full((1,), 0.3, device="cuda")
    clean = ops.project_and_loss_forward(ref, samp, 7, t, _lib.SIGMA_FROM_T_CLS, 0.0, 1.0)
    bad = ops.project_and_loss_forward(r2, s2, 7, t, _lib.SIGMA_FROM_T_CLS, 0.0, 1.0)
    for i, bound in ((1, n), (5, n), (7, m)):
        _in_range(bad[i], bound)
    for a, c in zip(bad[:8], clean[:8]):
        _same_finite(a, c)
    # and through autograd: the backward kernels index with what the forward wrote
    grads = []
    for r, s in ((ref, samp), (r2, s2)):
        sq = s.clone().requires_grad_(True)
        proj, loss, _ = ops.ProjectAndLossFunction.apply(r, sq, t, 7, _lib.SIGMA_FROM_T_CLS, 0.0)
        (proj.sum() + loss).backward()
        grads.append(sq.grad)
    torch.cuda.synchronize()
    assert grads[1].shape == grads[0].shape


@pytest.mark.gpu
@pytest.mark.parametrize("poison", POISON)
def test_progressive_loss_indices_stay_in_range(poison):
    ref, samp, r2, s2 = _pair(poison)
    n, m = ref.shape[1], samp.shape[1]
    sizes, w = [8, 16, m], [1.0, 1.0, 1.0]
    clean = ops.progressive_loss_forward(ref, samp, sizes, w)
    bad = ops.progressive_loss_forward(r2, s2, sizes, w)
    _in_range(bad[1], n)
    _in_range(bad[3], m)
    for a, c in zip(bad[:4], clean[:4]):
        _same_finite(a, c)
    assert not torch.isfinite(bad[4][-1])
    sq = s2.clone().requires_grad_(True)
    total, _ = ops.ProgressiveLossFunction.apply(sq, r2, sizes, w)
    total.backward()
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("poison", POISON)
def test_nn_matching_completion_stays_in_range(poison):
    ref, samp, r2, s2 = _pair(poison)
    n, m = ref.shape[1], samp.shape[1]
    for r, s in ((ref, samp), (r2, s2)):
        _, idx1, _, _ = ops.nn_distance_forward(s, r)
        few = idx1[:, :4].contiguous()                   # 4 seeds, completed to m points by farthest point sampling
        out, oi = ops.nn_matching(r, few, m, complete_fps=True, return_idx=True)
        _in_range(oi, n)
        if r is ref:
            clean = (out, oi)
    _same_finite(out, clean[0])
    _same_finite(oi, clean[1])
    if poison == "ref_nan":                               # numpy's argmax: the first NaN distance wins
        assert int(oi[BAD, 4]) == 0
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["fused", "layers"])
@pytest.mark.parametrize("poison", ["nan_cloud", "inf_cloud", "all_nan"])
def test_generator_backward_pool_argmax_on_nonfinite_clouds(route, poison):
    """SampleNet trains on the fused route, the classification sampler on the per-layer one; both end in the pool arg-max of
    generator_bwd.cu.  A NaN or Inf cloud poisons the BatchNorm statistics of the whole batch, so what is checked is that the step runs
    through and leaves a gradient on every parameter (the arg-max it routes by is the one the kernel reads with)."""
    import samplenet_b200 as sb

    torch.manual_seed(0)
    if route == "fused":
        net = sb.SampleNet(M, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train()
    else:
        net = sb.ClassificationSampleNet(M, group_size=7).cuda().train()
    g = torch.Generator().manual_seed(1)
    x = torch.rand(4, 1024, 3, generator=g) - 0.5
    if poison == "nan_cloud":
        x[1] = NAN
    elif poison == "inf_cloud":
        x[1, :, 0] = float("inf")
    else:
        x[:] = NAN
    simp, proj = net(x.cuda())
    assert net.generator_route == route
    (simp.sum() + proj.sum()).backward()
    torch.cuda.synchronize()
    assert all(p.grad is not None for p in net.parameters() if p.requires_grad)


# ----------------------------------------------------------------------------------------------------- GPU: the guard kernel
def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _reference_guard(checked, live, snaps):
    """The guard restated with torch: isfinite over the floating checked tensors, then where() per pair on the bits."""
    bad = any(not bool(torch.isfinite(t).all()) for t in checked if t.is_floating_point())
    return bad, [_bits(s).clone() if bad else _bits(a).clone() for a, s in zip(live, snaps)]


def _tables(seed, count=40):
    g = torch.Generator().manual_seed(seed)
    dtypes = [torch.float32, torch.float64, torch.float16, torch.bfloat16, torch.int64, torch.float32]
    live, snaps, checked = [], [], []
    for i in range(count):
        dt = dtypes[i % len(dtypes)]
        n = int(torch.randint(1, 20000 if i % 7 == 0 else 300, (1,), generator=g))
        mk = (lambda: torch.randint(-9, 9, (n,), generator=g)) if not dt.is_floating_point else (lambda: torch.randn(n, generator=g))
        a, s, c = mk().to(dt), mk().to(dt), mk().to(dt)
        if dt.is_floating_point:
            s[::5] = -0.0                                 # a signed zero and NaN payloads must come back exactly
            s.view(-1)[1::11] = NAN
            if dt == torch.float32:
                s.view(torch.int32)[2::13] = 0x7fc01234   # a quiet NaN with a payload
        live.append(a.cuda()); snaps.append(s.cuda()); checked.append(c.cuda())
    return checked, live, snaps


def _check_guard(guard, checked, live, snaps):
    bad, want = _reference_guard(checked, live, snaps)
    before = guard.skip_count.item()
    ck_bits = [_bits(c).clone() for c in checked]
    sn_bits = [_bits(s).clone() for s in snaps]
    skipped = guard(checked, live, snaps)
    torch.cuda.synchronize()
    assert int(skipped) == int(bad) and int(guard.skip_count) == before + int(bad)
    for a, w in zip(live, want):
        assert torch.equal(_bits(a), w)
    assert all(torch.equal(_bits(c), b) for c, b in zip(checked, ck_bits))
    assert all(torch.equal(_bits(s), b) for s, b in zip(snaps, sn_bits))
    assert int(guard.state.abs().sum()) == 0                       # left zero for the next call


@pytest.mark.gpu
@pytest.mark.parametrize("count", [40, 900])        # 900: more than one launch's table on each side
def test_guard_matches_torch_restatement(count):
    guard = ops.NonfiniteGuard("cuda")
    checked, live, snaps = _tables(3, count)
    _check_guard(guard, checked, live, snaps)                     # all finite: nothing restored
    last = [t for t in checked if t.is_floating_point()][-1]
    last.view(-1)[-1] = float("inf")                              # only the last element of the last checked tensor
    _check_guard(guard, checked, live, snaps)
    last.view(-1)[-1] = 0.0
    checked[0].view(-1)[0] = NAN                                   # the first element of the first
    _check_guard(guard, checked, live, snaps)
    checked[0].view(-1)[0] = 1.0
    ints = [torch.full((5,), 2 ** 62, dtype=torch.int64, device="cuda")]       # integers are finite, whatever their bits
    _check_guard(guard, ints, live, snaps)
    _check_guard(guard, [], [], [])                                # empty tables: only the result is written
    assert int(guard.skip_count) == 2


@pytest.mark.gpu
def test_guard_inside_a_cuda_graph():
    guard = ops.NonfiniteGuard("cuda")
    checked, live, snaps = _tables(4, 30)
    src = [c.clone() for c in checked]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        guard(checked, live, snaps)                                 # warm-up: finite, nothing restored
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        guard(checked, live, snaps)
    for poison in (False, True, False, True):
        for c, o in zip(checked, src):
            c.copy_(o)
        if poison:
            checked[5].view(-1)[3] = NAN
        for a in live:                                             # fresh live values each replay
            a.copy_(a.flip(0))
        bad, want = _reference_guard(checked, live, snaps)
        assert bad == poison
        graph.replay()
        torch.cuda.synchronize()
        assert int(guard.skipped) == int(poison)
        for a, w in zip(live, want):
            assert torch.equal(_bits(a), w)
    assert int(guard.skip_count) == 2


@pytest.mark.gpu
def test_guard_writes_only_its_buffers():
    """Every tensor a view of one arena, with guard bands of a canary pattern between them: after a restoring call only the live tensors
    and the guard's own result words differ."""
    sizes = [1, 17, 4099, 3, 70000, 255]
    pad = 64
    total = sum(sizes) * 3 + pad * (3 * len(sizes) + 1)
    arena = torch.full((total,), -123.25, device="cuda")
    views, off = [], pad
    for _ in range(3):
        for n in sizes:
            views.append(arena[off:off + n])
            off += n + pad
    checked, live, snaps = views[:6], views[6:12], views[12:]
    for i, t in enumerate(views):
        t.copy_(torch.arange(t.numel(), device="cuda", dtype=torch.float32) * (i + 1))
    checked[4][-1] = NAN
    expect = arena.clone()
    for a, s in zip(live, snaps):
        o = (a.data_ptr() - arena.data_ptr()) // 4
        expect[o:o + a.numel()] = s
    guard = ops.NonfiniteGuard("cuda")
    words = torch.full((8,), 7, dtype=torch.int32, device="cuda")
    guard.skipped, guard.skip_count = words[2], words[5]          # results land in the middle of a canary buffer
    guard(checked, live, snaps)
    torch.cuda.synchronize()
    assert torch.equal(_bits(arena), _bits(expect))
    assert words.tolist() == [7, 7, 1, 7, 7, 8, 7, 7]


# ----------------------------------------------------------------------------------------------------- GPU: the runners
def _set(seed, n, nan_clouds=()):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, N_PTS, 3, generator=g) - 0.5
    for i in nan_clouds:
        x[i, 7] = NAN
    return x.cuda(), torch.randint(0, CLASSES, (n,), generator=g).cuda()


def _runner(case, graphed, skip=True):
    import samplenet_b200 as sb

    torch.manual_seed(0)
    if case == "cls":
        sampler = sb.ClassificationSampleNet(M, group_size=7).cuda()
        net = tasknets.PointNetClsTransforms(num_classes=CLASSES).cuda().eval().requires_grad_(False)
        step = trainers.ClassificationStep(sampler, tasknets.FrozenPointNetClsTransforms(net), M)
        return trainers.SamplerTrainStep(step, torch.optim.Adam(sampler.parameters(), lr=1e-3, capturable=True), batch_size=B,
                                         graphed=graphed, skip_nonfinite=skip)
    if case == "classifier":
        net = tasknets.CudaPointNetCls(tasknets.PointNetCls(num_classes=CLASSES)).cuda()
        return trainers.ClassifierTrainStep(net, torch.optim.Adam(net.parameters(), lr=1e-3, capturable=True), batch_size=B, graphed=graphed,
                                            skip_nonfinite=skip)
    ae = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=N_PTS)).cuda()
    return trainers.AutoencoderTrainStep(ae, torch.optim.Adam(ae.parameters(), lr=5e-4, capturable=True), n_sample_points=N_PTS, batch_size=B,
                                         graphed=graphed, skip_nonfinite=skip)


def _module(run):
    if isinstance(run, trainers.SamplerTrainStep):
        return run.task.sampler
    return run.net if isinstance(run, trainers.ClassifierTrainStep) else run.ae


def _state(run):
    module = _module(run)
    st = {"m." + k: v.detach().clone() for k, v in module.state_dict().items()}
    for i, p in enumerate(module.parameters()):
        for k, v in run.optimizer.state.get(p, {}).items():
            st["opt.%d.%s" % (i, k)] = torch.as_tensor(v).detach().clone()
    return st


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(_bits(a[k].reshape(-1)), _bits(b[k].reshape(-1))), k


def _call(run, x, y):
    """One step: (its outputs but the skip flag, as clones; the skip flag)."""
    if isinstance(run, trainers.SamplerTrainStep):
        out = run(x, y)
        return [v.clone() for k, v in out.items() if k != "skipped"], int(out["skipped"]) if "skipped" in out else None
    out = run(x, y) if isinstance(run, trainers.ClassifierTrainStep) else run(x)
    out = out if isinstance(out, tuple) else (out,)
    rest = [v.clone() if torch.is_tensor(v) else v for v in out[:-1]] if run._skip is not None else list(out)
    return rest, int(out[-1]) if run._skip is not None else None


def _same_outputs(a, b):
    assert len(a) == len(b)
    for u, v in zip(a, b):
        assert (torch.equal(u, v) if torch.is_tensor(u) else u == v)


CASES = ["cls", "classifier", "autoencoder"]


@pytest.mark.gpu
@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graphed"])
@pytest.mark.parametrize("case", CASES)
def test_a_nan_batch_is_skipped_and_leaves_no_trace(case, graphed):
    x, y = _set(1, 3 * B)
    bad = x[B:2 * B].clone()
    bad[3, 11] = NAN
    batches = [x[:B], bad, x[B:2 * B], x[2 * B:]]
    a, b = _runner(case, graphed), _runner(case, graphed)
    outs_a, outs_b = [], []
    torch.manual_seed(5)
    outs_a.append(_call(a, batches[0], y[:B]))
    before = _state(a)
    _, skipped = _call(a, batches[1], y[:B])
    torch.cuda.synchronize()
    assert skipped == 1
    _assert_same(before, _state(a))                            # parameters, buffers, optimiser state: as before the step
    torch.manual_seed(5)
    outs_b.append(_call(b, batches[0], y[:B]))
    if hasattr(b, "step"):
        b.step += 1                                             # the batch was consumed: the schedule advanced
    for i, xb in enumerate(batches[2:]):
        torch.manual_seed(20 + i)                               # (dropout draws of the skipped step are not replayed)
        outs_a.append(_call(a, xb, y[:B]))
        torch.manual_seed(20 + i)
        outs_b.append(_call(b, xb, y[:B]))
    for (oa, sa), (ob, sb_) in zip(outs_a, outs_b):
        assert sa == sb_ == 0
        _same_outputs(oa, ob)
    _assert_same(_state(a), _state(b))


@pytest.mark.gpu
@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graphed"])
def test_a_sampler_with_a_nan_weight_skips_every_step(graphed):
    run = _runner("cls", graphed)
    with torch.no_grad():
        next(run.task.sampler.parameters()).view(-1)[0] = NAN
    before = {k: v for k, v in _state(run).items() if not k.startswith("opt.")}
    x, y = _set(2, 4 * B)
    res = run.train_one_epoch(x, y)
    assert res["skipped_steps"] == res["steps"] == 4 and run.step == 4
    assert all(v != v for k, v in res.items() if k not in ("steps", "skipped_steps"))   # means over no step: NaN
    after = _state(run)
    _assert_same(before, {k: v for k, v in after.items() if not k.startswith("opt.")})
    for k, v in after.items():
        if k.startswith("opt."):
            assert not v.any(), k                               # the state its first step created: zeros, the fresh state


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_epoch_counts_the_batches_holding_a_nan_cloud(case):
    n = 5 * B + 3
    nan_clouds = (2, 17, 18, 40)
    x, y = _set(3, n, nan_clouds)
    results = {}
    for graphed in (False, True):
        run = _runner(case, graphed)
        torch.manual_seed(9)
        perm = torch.randperm(n, device="cuda").cpu()             # the permutation the epoch is about to draw
        want = sum(any(int(i) in nan_clouds for i in perm[s * B:(s + 1) * B]) for s in range(n // B))
        torch.manual_seed(9)
        res = run.train_one_epoch(x, y) if case != "autoencoder" else run.train_one_epoch(x)
        assert res["skipped_steps"] == want and 1 <= want < res["steps"]
        results[graphed] = (res, _state(run))
    assert results[False][0] == results[True][0]                   # the graphed epoch is the eager epoch, bit for bit
    _assert_same(results[False][1], results[True][1])


@pytest.mark.gpu
@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graphed"])
@pytest.mark.parametrize("case", CASES)
def test_on_finite_data_the_guard_changes_nothing(case, graphed):
    x, y = _set(4, 2 * B + 3)
    results = {}
    for skip in (False, True):
        run = _runner(case, graphed, skip)
        torch.manual_seed(10)
        res = [run.train_one_epoch(x, y) if case != "autoencoder" else run.train_one_epoch(x) for _ in range(2)]
        if skip:
            assert all(r.pop("skipped_steps") == 0 for r in res)
        results[skip] = (res, _state(run), torch.cuda.get_rng_state())
    assert results[False][0] == results[True][0]
    _assert_same(results[False][1], results[True][1])
    assert torch.equal(results[False][2], results[True][2])
