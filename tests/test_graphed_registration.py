"""RegistrationStep(graphed=True): every whole batch of train_1 one CUDA-graph replay through trainers._StepGraph and graphs.CapturedStep,
bit for bit the eager train_1.

CPU: what the graph cannot hold is refused with ValueError before any CUDA work -- the FPS sampler, data-parallel training, an optimiser
that is not capturable (SGD among them), a plain PCRNet, and clouds outside the pose loss's envelope; the eager default takes all of them.
GPU (H100): two graphed epochs against an eager twin from the same seed -- the returned means, every parameter and buffer, the optimiser
state and the CUDA RNG state after each epoch equal -- for SampleNet with the frozen PCRNet (one and two sampled clouds), PCRNet trained
alone and both trained jointly, each with capturable Adam and RMSprop, over sets whose last batch is partial; a capture after an eager
epoch; a replayed epoch issues no launch from the host; each runner's graph has its own ticket word; another shape, inversion value,
model or optimiser raises."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from samplenet_b200 import _lib, registration  # noqa: E402

B, CLOUDS, RAW_POINTS, N = 8, 5, 300, 256      # 5 clouds x 4 repeats = 20 records: batches of 8, 8 and 4


class _Untouched:
    """A batch iterable that fails the test if train_1 reaches it."""

    def __iter__(self):
        raise AssertionError("train_1 read a batch before refusing")


# ----------------------------------------------------------------------------------------------------- CPU
def test_refusals_come_before_any_cuda_work():
    with pytest.raises(ValueError, match="sampler='fps'"):
        registration.RegistrationStep(sampler="fps", graphed=True)
    registration.RegistrationStep(sampler="fps")                     # the eager default takes it

    act = registration.RegistrationStep(graphed=True)
    model = act.create_model(frozen_task=True)
    with pytest.raises(ValueError, match="one GPU"):
        act.wrap_data_parallel(model)
    assert act._ddp is None

    params = [p for p in model.parameters() if p.requires_grad]
    for opt in (torch.optim.Adam(params, lr=1e-3), torch.optim.RMSprop(params, lr=1e-3), torch.optim.SGD(params, lr=1e-3)):
        with pytest.raises(ValueError, match="capturable=True"):
            act.train_1(model, _Untouched(), opt, "cuda")
    with pytest.raises(ValueError, match="torch.optim.Adam"):         # capturable, but its created state is not zero
        act.train_1(model, _Untouched(), torch.optim.NAdam(params, lr=1e-3, capturable=True), "cuda")

    plain = registration.RegistrationStep(graphed=True)
    net = plain.create_model()
    with pytest.raises(ValueError, match="PCRNet"):
        plain.train_1(net, _Untouched(), torch.optim.Adam([p for p in net.parameters() if p.requires_grad], capturable=True), "cuda")

    # an FPS sampler attached to the model is refused too, whatever the step was built with
    act = registration.RegistrationStep(sampler="none", train_pcrnet=True, graphed=True)
    model = act.create_model(cuda_task=True)
    model.sampler = registration.FPSSampler(16, permute=True, input_shape="bnc", output_shape="bnc")
    with pytest.raises(ValueError, match="FPS sampler"):
        act.train_1(model, _Untouched(), torch.optim.Adam(model.parameters(), capturable=True), "cuda")


def test_clouds_outside_the_pose_loss_are_refused_before_capture():
    act = registration.RegistrationStep(sampler="none", train_pcrnet=True, graphed=True)
    model = act.create_model(cuda_task=True)
    opt = torch.optim.Adam(model.parameters(), capturable=True)
    big = torch.zeros(2, 2048, 3)                                     # above the pose loss's 1024 points; CPU tensors, never copied
    igt = {"vec": torch.zeros(2, 7), "inversion": torch.tensor([False])}
    with pytest.raises(ValueError, match="envelopes"):
        act.train_1(model, [(big, big, igt)], opt, "cuda")
    assert act._graph.captured is None


# ----------------------------------------------------------------------------------------------------- GPU helpers
def _set(seed=0, clouds=CLOUDS, repeat=4):
    g = torch.Generator().manual_seed(seed)
    raw = torch.rand(clouds, RAW_POINTS, 3, generator=g) * torch.tensor([1.0, 0.8, 0.5])
    return registration.CudaQuaternionFixedDataset(raw.numpy(), num_points=N, repeat=repeat, seed=seed)


CONFIGS = {
    "samplenet_frozen_2": ({"sampler": "samplenet", "num_sampled_clouds": 2}, {"frozen_task": True}),
    "samplenet_frozen_1": ({"sampler": "samplenet", "num_sampled_clouds": 1}, {"frozen_task": True}),
    "pcrnet": ({"sampler": "none", "train_pcrnet": True}, {"cuda_task": True}),
    "samplenet_joint": ({"sampler": "samplenet", "train_pcrnet": True}, {"cuda_task": True}),
}
OPTIMIZERS = {"adam": lambda ps: torch.optim.Adam(ps, lr=1e-3, capturable=True),
              "rmsprop": lambda ps: torch.optim.RMSprop(ps, lr=1e-4, capturable=True)}


def _runner(config, graphed, optimizer="adam"):
    """(step, model, optimiser); the same seed gives the same model."""
    step_kw, model_kw = CONFIGS[config]
    act = registration.RegistrationStep(num_out_points=32, graphed=graphed, **step_kw)
    torch.manual_seed(0)
    model = act.create_model(**model_kw).cuda()
    return act, model, OPTIMIZERS[optimizer]([p for p in model.parameters() if p.requires_grad])


def _state(model, opt):
    """Every parameter and buffer of the model (the sampler's BatchNorm statistics included) and the optimiser state, as clones."""
    st = {"m." + k: v.detach().clone() for k, v in model.state_dict().items()}
    for i, p in enumerate(model.parameters()):
        for k, v in opt.state.get(p, {}).items():
            st["opt.%d.%s" % (i, k)] = torch.as_tensor(v).detach().clone()
    return st


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and torch.equal(a[k], b[k]), k


def _epochs(act, model, opt, ds, epochs, seed=11):
    """train_1 over fresh shuffled batches `epochs` times: [(returned means, CUDA RNG state after the epoch)]."""
    torch.manual_seed(seed)
    out = []
    for _ in range(epochs):
        res = act.train_1(model, ds.batches(B, shuffle=True), opt, "cuda")
        out.append((res, torch.cuda.get_rng_state()))
    return out


def _assert_epochs_equal(a, b):
    assert len(a) == len(b)
    for (res_a, rng_a), (res_b, rng_b) in zip(a, b):
        assert res_a == res_b
        assert torch.equal(rng_a, rng_b)          # the same random numbers were drawn: permutations and the pairs' keys


# ----------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("optimizer", sorted(OPTIMIZERS))
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_graphed_epochs_are_the_eager_epochs_bit_for_bit(config, optimizer):
    ds = _set()
    assert [d[0].shape[0] for d in ds.batches(B)] == [8, 8, 4]      # a trailing partial batch of more than one cloud
    results = {}
    for graphed in (False, True):
        act, model, opt = _runner(config, graphed, optimizer)
        results[graphed] = (_epochs(act, model, opt, ds, 2), _state(model, opt))
        if graphed:
            assert act._graph.captured is not None
    _assert_epochs_equal(results[False][0], results[True][0])
    _assert_same(results[False][1], results[True][1])
    assert all(v == v for (res, _) in results[True][0] for v in res)    # finite means, not a pair of NaNs that compare unequal anyway


@pytest.mark.gpu
def test_capture_after_an_eager_epoch_continues_the_eager_run():
    ds = _set(1)
    eager, model_e, opt_e = _runner("samplenet_frozen_2", False)
    want = _epochs(eager, model_e, opt_e, ds, 3)

    first, model, opt = _runner("samplenet_frozen_2", False)
    torch.manual_seed(11)
    got = [(first.train_1(model, ds.batches(B, shuffle=True), opt, "cuda"), torch.cuda.get_rng_state())]
    graphed = registration.RegistrationStep(num_out_points=32, sampler="samplenet", graphed=True)
    for _ in range(2):                                 # the optimiser has state: the capture restores it, then replays from it
        got.append((graphed.train_1(model, ds.batches(B, shuffle=True), opt, "cuda"), torch.cuda.get_rng_state()))
    _assert_epochs_equal(want, got)
    _assert_same(_state(model_e, opt_e), _state(model, opt))


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["samplenet_frozen_2", "pcrnet"])
def test_a_replayed_epoch_launches_nothing_from_the_host(config):
    ds = _set(2, clouds=4)                             # 16 records: two whole batches, no partial one
    act, model, opt = _runner(config, True)
    act.train_1(model, ds.batches(B, shuffle=True), opt, "cuda")          # captures
    batches = list(ds.batches(B, shuffle=True))       # the pairs launches happen here
    torch.cuda.synchronize()
    before = _lib.launch_count()
    vloss, gloss = act.train_1(model, batches, opt, "cuda")
    torch.cuda.synchronize()
    assert _lib.launch_count() == before
    assert act._graph.captured.launches_per_step > 0
    assert vloss == vloss and gloss == gloss


@pytest.mark.gpu
def test_each_runner_has_its_own_ticket_word():
    """The pose loss's last-CTA reduction keeps the word it was captured with and replays on the caller's stream: two runners' graphs must
    not share a word, nor take the stream's."""
    from samplenet_b200 import ops

    ds = _set(3)
    runs = [_runner("samplenet_frozen_2", True) for _ in range(2)]
    for act, model, opt in runs:
        act.train_1(model, ds.batches(B, shuffle=True), opt, "cuda")
    dev = ds.device
    words = [act._graph.captured.workspaces.ticket(dev).data_ptr() for act, _, _ in runs]
    assert words[0] != words[1]
    assert ops._ticket(dev).data_ptr() not in words


@pytest.mark.gpu
def test_another_shape_inversion_model_or_optimizer_raises():
    ds = _set(4)
    act, model, opt = _runner("samplenet_frozen_2", True)
    act.train_1(model, ds.batches(B, shuffle=True), opt, "cuda")
    p0, p1, igt = ds.batch(list(range(B)))
    with pytest.raises(ValueError, match="one captured input"):                  # other clouds
        act.train_1(model, [(p0[:, :128].contiguous(), p1[:, :128].contiguous(), igt)], opt, "cuda")
    q0, q1, qgt = ds.batch(list(range(B + 2)))
    with pytest.raises(ValueError, match="one captured input"):                  # a larger batch
        act.train_1(model, [(q0, q1, qgt)], opt, "cuda")
    with pytest.raises(ValueError, match="inversion"):
        act.train_1(model, [(p0, p1, {"vec": igt["vec"], "inversion": torch.tensor([True])})], opt, "cuda")
    with pytest.raises(ValueError, match="only the last batch"):                 # a smaller batch that is not the last
        act.train_1(model, [(p0[:4], p1[:4], {"vec": igt["vec"][:4], "inversion": igt["inversion"]}), (p0, p1, igt)], opt, "cuda")
    _, other, other_opt = _runner("samplenet_frozen_2", False)
    with pytest.raises(ValueError, match="model and the optimiser"):
        act.train_1(other, [(p0, p1, igt)], opt, "cuda")
    with pytest.raises(ValueError, match="model and the optimiser"):
        act.train_1(model, [(p0, p1, igt)], other_opt, "cuda")
    vloss, gloss = act.train_1(model, [(p0, p1, igt)], opt, "cuda")               # the captured shape still runs
    assert vloss == vloss and gloss == gloss
