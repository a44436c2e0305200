"""The training runners with graphed=True (trainers.SamplerTrainStep, ClassifierTrainStep, AutoencoderTrainStep): every step one CUDA-graph
replay through graphs.CapturedStep, bit for bit the eager runner.

CPU: a non-capturable optimiser, or one whose lazily created state is not all zeros, is refused at construction, naming the fix; for every
optimiser accepted, zeroing the state its first step created gives the state a fresh optimiser starts from.
GPU (H100): two epochs of a graphed runner against an eager twin with the same seed, model and optimiser configuration -- every parameter
and buffer, the optimiser state, the returned dicts and the CUDA RNG state after the epochs equal -- for every step the runners wrap, with
augmentation and dropout; a schedule that crosses staircase boundaries mid-epoch (captured again); capturing leaves the model, the
optimiser, the RNG state and the counters as they were; a replayed epoch issues no launch from the host; another shape, dtype or device
raises; each captured step has its own ticket word; the classifier's epochs with every other accepted optimiser."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from samplenet_b200 import _lib, graphs, tasknets, trainers  # noqa: E402

B, N_SET, N_PTS, M, CLASSES = 8, 21, 256, 32, 5      # 2 whole batches of 8 per epoch; the last 5 clouds are the remainder
GAUSS = {"mu": 0.0, "sigma": 0.01}


# ----------------------------------------------------------------------------------------------------- CPU
def test_non_capturable_optimizer_is_refused_at_construction():
    lin = torch.nn.Linear(3, 3)
    cls_step = trainers.ClassificationStep(torch.nn.Linear(1, 1), torch.nn.Linear(1, 1), 32)
    rec_step = trainers.ReconstructionStep(torch.nn.Linear(1, 1), torch.nn.Linear(1, 1), 64)
    makers = [lambda opt: trainers.SamplerTrainStep(cls_step, opt, graphed=True),
              lambda opt: trainers.SamplerTrainStep(rec_step, opt, graphed=True),
              lambda opt: trainers.ClassifierTrainStep(lin, opt, graphed=True),
              lambda opt: trainers.AutoencoderTrainStep(lin, opt, graphed=True)]
    for make in makers:
        for opt in (torch.optim.Adam(lin.parameters()), torch.optim.SGD(lin.parameters(), lr=0.1), None):
            with pytest.raises(ValueError, match="capturable=True"):
                make(opt)
        assert make(torch.optim.Adam(lin.parameters(), capturable=True)).graphed
    # one group without it is enough to refuse
    opt = torch.optim.Adam([{"params": [lin.weight], "capturable": True}, {"params": [lin.bias], "capturable": False}])
    with pytest.raises(ValueError):
        trainers.ClassifierTrainStep(lin, opt, graphed=True)
    # the default stays eager and takes any optimiser
    assert not trainers.ClassifierTrainStep(lin, torch.optim.SGD(lin.parameters(), lr=0.1)).graphed
    # capturable, but their first step creates state that is not zero (NAdam's mu_product, ASGD's eta and mu); a subclass may create other state
    class MyAdam(torch.optim.Adam):
        pass

    for opt in (torch.optim.NAdam(lin.parameters(), capturable=True), torch.optim.ASGD(lin.parameters(), capturable=True),
                MyAdam(lin.parameters(), capturable=True)):
        with pytest.raises(ValueError, match="torch.optim.Adam, torch.optim.AdamW"):
            trainers.ClassifierTrainStep(lin, opt, graphed=True)
    for cls in graphs.ZERO_INIT_OPTIMIZERS:
        assert trainers.ClassifierTrainStep(lin, cls(lin.parameters(), lr=0.1, capturable=True), graphed=True).graphed


ZERO_INIT_KW = {torch.optim.Adam: {"amsgrad": True}, torch.optim.RMSprop: {"momentum": 0.9, "centered": True}}


def _steps_after_restore(cls, kw):
    """Parameters after three steps of a fresh optimiser, and of one whose first step was taken and undone (the parameter copied back, the
    state restored as CapturedStep restores it from an empty snapshot) -- on the CPU, so not capturable; the state created is the same."""
    torch.manual_seed(0)
    a = torch.nn.Parameter(torch.randn(7))
    b = torch.nn.Parameter(a.detach().clone())
    opt_a, opt_b = cls([a], lr=0.1, **kw), cls([b], lr=0.1, **kw)
    g = torch.randn(7)
    a.grad = g.clone()
    opt_a.step()
    with torch.no_grad():
        a.copy_(b)
    graphs._restore_optimizer(opt_a, {})
    for i in range(3):
        a.grad, b.grad = g * (i + 1), g * (i + 1)
        opt_a.step()
        opt_b.step()
    return a, b


def test_zeroing_created_state_is_the_fresh_state_for_every_accepted_optimizer():
    for cls in graphs.ZERO_INIT_OPTIMIZERS:
        a, b = _steps_after_restore(cls, ZERO_INIT_KW.get(cls, {}))
        assert torch.equal(a, b), cls.__name__
    for cls in (torch.optim.NAdam, torch.optim.ASGD):        # why those are refused: zeroing is not their fresh state
        a, b = _steps_after_restore(cls, {})
        assert not torch.equal(a, b), cls.__name__


# ----------------------------------------------------------------------------------------------------- GPU helpers
def _set(seed, n=N_SET, points=N_PTS):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, points, 3, generator=g) - 0.5).cuda(), torch.randint(0, CLASSES, (n,), generator=g).cuda()


def _adam(params, lr=1e-3):
    return torch.optim.Adam(params, lr=lr, capturable=True)


def _runner(case, graphed, optimizer=None, **kw):
    """A fresh runner of the given case; the same seed gives the same model."""
    import samplenet_b200 as sb

    torch.manual_seed(0)
    if case in ("cls", "progressive_cls"):
        sampler = sb.ClassificationSampleNet(M, group_size=7).cuda()
        if case == "cls":
            net = tasknets.PointNetClsTransforms(num_classes=CLASSES).cuda().eval().requires_grad_(False)
            step = trainers.ClassificationStep(sampler, tasknets.FrozenPointNetClsTransforms(net), M)
        else:
            net = tasknets.PointNetCls(num_classes=CLASSES).cuda().eval().requires_grad_(False)
            step = trainers.ProgressiveClassificationStep(sampler, tasknets.FrozenPointNetCls(net), 8, M)
        return trainers.SamplerTrainStep(step, _adam(sampler.parameters()), batch_size=B, graphed=graphed, **kw)
    if case in ("rec_chamfer", "rec_emd", "progressive_rec"):
        sampler = sb.ReconstructionSampleNet(M).cuda()
        ae = tasknets.FrozenPointNetAE(tasknets.PointNetAE(n_pc_points=N_PTS).cuda().eval().requires_grad_(False))
        if case == "progressive_rec":
            step = trainers.ProgressiveReconstructionStep(sampler, ae, sizes=(8, 16, 32), ae_batch_stats=True)
            aug = {}
        else:
            step = trainers.ReconstructionStep(sampler, ae, M, ae_loss=case[4:])
            aug = {"gauss_augment": GAUSS, "z_rotate": True}
        return trainers.SamplerTrainStep(step, _adam(sampler.parameters()), batch_size=B, graphed=graphed, **aug, **kw)
    if case in ("classifier", "classifier_transforms"):
        net = (tasknets.CudaPointNetCls(tasknets.PointNetCls(num_classes=CLASSES)) if case == "classifier"
               else tasknets.CudaPointNetClsTransforms(tasknets.PointNetClsTransforms(num_classes=CLASSES))).cuda()
        opt = _adam(net.parameters()) if optimizer is None else optimizer(net.parameters())
        return trainers.ClassifierTrainStep(net, opt, batch_size=B, augment=True, graphed=graphed, **kw)
    ae = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=N_PTS)).cuda()
    return trainers.AutoencoderTrainStep(ae, _adam(ae.parameters(), 5e-4), n_sample_points=N_PTS, batch_size=B, gauss_augment=GAUSS,
                                         z_rotate=True, graphed=graphed, **kw)


def _parts(run):
    """(trained module, frozen task network or None, optimiser, labels needed)."""
    if isinstance(run, trainers.SamplerTrainStep):
        return run.task.sampler, run.task.classifier if run.classification else run.task.ae, run.optimizer, run.classification
    if isinstance(run, trainers.ClassifierTrainStep):
        return run.net, None, run.optimizer, True
    return run.ae, None, run.optimizer, False


def _epoch(run, x, y):
    return run.train_one_epoch(x, y) if _parts(run)[3] else run.train_one_epoch(x)


def _state(run):
    """Every parameter and buffer of the modules the step touches, and the optimiser state, as clones."""
    module, task, opt, _ = _parts(run)
    st = {"m." + k: v.detach().clone() for k, v in module.state_dict().items()}
    if task is not None:
        st.update({"t." + k: v.detach().clone() for k, v in task.state_dict().items()})
    for i, p in enumerate(module.parameters()):
        for k, v in opt.state.get(p, {}).items():
            st["opt.%d.%s" % (i, k)] = torch.as_tensor(v).detach().clone()
    return st


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k


CASES = ["cls", "progressive_cls", "rec_chamfer", "rec_emd", "progressive_rec", "classifier", "classifier_transforms", "autoencoder"]


# ----------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_graphed_epochs_are_the_eager_epochs_bit_for_bit(case):
    x, y = _set(1)
    results = {}
    for graphed in (False, True):
        run = _runner(case, graphed)
        torch.manual_seed(11)
        results[graphed] = ([_epoch(run, x, y) for _ in range(2)], _state(run), torch.cuda.get_rng_state(), getattr(run, "step", None))
    (eager, st_e, rng_e, step_e), (graph, st_g, rng_g, step_g) = results[False], results[True]
    assert eager == graph
    assert all(r["steps"] == 2 for r in graph)
    _assert_same(st_e, st_g)
    assert torch.equal(rng_e, rng_g)          # the same random numbers were drawn: permutations, augmentation keys, dropout masks
    assert step_e == step_g


OTHER_OPTIMIZERS = [c for c in graphs.ZERO_INIT_OPTIMIZERS if c is not torch.optim.Adam]


@pytest.mark.gpu
@pytest.mark.parametrize("cls", OTHER_OPTIMIZERS, ids=lambda c: c.__name__)
def test_graphed_epochs_with_the_other_accepted_optimizers(cls):
    make = lambda params: cls(params, lr=1e-3, capturable=True, **ZERO_INIT_KW.get(cls, {}))
    x, y = _set(6)
    results = {}
    for graphed in (False, True):
        run = _runner("classifier", graphed, optimizer=make)
        torch.manual_seed(13)
        results[graphed] = ([_epoch(run, x, y) for _ in range(2)], _state(run), torch.cuda.get_rng_state())
    assert results[False][0] == results[True][0]
    _assert_same(results[False][1], results[True][1])
    assert torch.equal(results[False][2], results[True][2])


@pytest.mark.gpu
def test_each_captured_step_has_its_own_ticket_word():
    """The progressive loss's last-CTA reduction keeps the word it was captured with and replays on the caller's stream: two graphs must not
    share a word, nor take the stream's."""
    from samplenet_b200 import ops

    x, y = _set(7)
    runs = [_runner("progressive_cls", True) for _ in range(2)]
    for run in runs:
        run.train_one_epoch(x, y)
    words = [run._graph.captured.workspaces.ticket(x.device).data_ptr() for run in runs]
    assert words[0] != words[1]
    assert ops._ticket(x.device).data_ptr() not in words


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cls", "classifier", "rec_chamfer"])
def test_schedule_boundaries_capture_again_and_match_eager(case):
    """Staircases every 2 steps (3 steps per epoch, so boundaries fall inside epochs) or, for reconstruction, every epoch."""
    kw = {"decay_steps": 1} if case == "rec_chamfer" else {"decay_step": 2 * B}
    x, y = _set(2, n=3 * B + 2)
    results = {}
    for graphed in (False, True):
        run = _runner(case, graphed, **kw)
        torch.manual_seed(12)
        res, captures = [], []
        for _ in range(3):
            res.append(_epoch(run, x, y))
            captures.append(run._graph.key if graphed else None)
        results[graphed] = (res, _state(run), torch.cuda.get_rng_state())
        if graphed:
            assert len(set(captures)) == 3            # the graph of the last step differs in each epoch
    assert results[False][0] == results[True][0]
    _assert_same(results[False][1], results[True][1])
    assert torch.equal(results[False][2], results[True][2])


@pytest.mark.gpu
def test_capture_leaves_model_optimizer_rng_and_counters_as_they_were():
    """Mid-training: an eager runner has taken steps (the optimiser has state), then its step is captured."""
    run = _runner("classifier_transforms", False)
    x, y = _set(3, n=B)
    torch.manual_seed(5)
    for _ in range(2):
        run(x, y)
    before, rng, step = _state(run), torch.cuda.get_rng_state(), run.step
    acc = torch.arange(3, dtype=torch.float64, device="cuda")

    def body():
        out, terms = run._step(x, y)
        acc.add_(torch.stack([t.double() for t in terms] + [terms[0].double()]))
        return out

    cap = graphs.CapturedStep(body, [run.net], run.optimizer, counters=(run, ("step",)), state=[acc])
    torch.cuda.synchronize()
    _assert_same(before, _state(run))
    assert torch.equal(torch.cuda.get_rng_state(), rng) and run.step == step
    assert torch.equal(acc, torch.arange(3, dtype=torch.float64, device="cuda"))
    assert cap.launches_per_step > 0

    # one replay is the eager runner's next step: a twin that took the same two steps takes it eagerly, from the same RNG state
    twin = _runner("classifier_transforms", False)
    torch.manual_seed(5)
    for _ in range(2):
        twin(x, y)
    assert torch.equal(torch.cuda.get_rng_state(), rng)
    cap.replay()
    loss, pred, _ = cap.outputs
    torch.cuda.set_rng_state(rng)
    t_loss, t_pred, _ = twin(x, y)
    assert torch.equal(loss, t_loss) and torch.equal(pred, t_pred)
    run.step += 1
    _assert_same(_state(twin), _state(run))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["classifier", "rec_chamfer"])
def test_a_replayed_epoch_launches_nothing_from_the_host(case):
    run = _runner(case, True)
    x, y = _set(4)
    _epoch(run, x, y)                                 # captures
    before = _lib.launch_count()
    res = _epoch(run, x, y)
    torch.cuda.synchronize()
    assert _lib.launch_count() == before
    assert res["steps"] == 2


@pytest.mark.gpu
def test_another_shape_raises():
    run = _runner("classifier", True)
    x, y = _set(5)
    run.train_one_epoch(x, y)
    with pytest.raises(ValueError, match="one captured input"):
        run.train_one_epoch(x[:, :128].contiguous(), y)
    with pytest.raises(ValueError, match="one captured input"):
        run(x[:B + 1], y[:B + 1])
    with pytest.raises(ValueError, match="one captured input"):           # another dtype is refused, not cast
        run(x[:B].double(), y[:B])
    with pytest.raises(ValueError, match="one captured input"):
        run.train_one_epoch(x, y.int())
    loss, pred, correct = run(x[:B], y[:B])           # the captured shape still runs
    assert loss.shape == () and pred.shape == (B,) and 0 <= correct <= B

    ae = _runner("autoencoder", True)
    ae.train_one_epoch(x)
    with pytest.raises(ValueError, match="one captured input"):
        ae(x[:B, :128].contiguous())
    with pytest.raises(ValueError, match="gt=None"):
        ae(x[:B], x[:B])
