"""Shape retrieval: the classifiers' retrieval vectors (fc3's input) on every classifier path, csrc/retrieval.cu (snb200_retrieval_metrics)
against a float64 numpy restatement of its contract over float32 sequential distances, and the evaluators built on it.  The host part
(envelope, ABI, the restatement on hand-worked cases) runs without a GPU."""
import ctypes
import os
import re
import subprocess
import zlib

import numpy as np
import pytest
import torch

import samplenet_b200 as sb
from samplenet_b200 import _lib, evaluation as ev, ops, tasknets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
NAMES = ("snb200_retrieval_metrics_supported", "snb200_retrieval_metrics")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _lib.lib()


# ----------------------------------------------------------------------------------------------------- the restatement
def distances32(q, x, chunk=64):
    """d(q, x) = sum_k fl(fl(q_k - x_k)^2), left to right in float32."""
    q, x = np.asarray(q, np.float32), np.asarray(x, np.float32)
    out = np.empty((q.shape[0], x.shape[0]), np.float32)
    for s in range(0, q.shape[0], chunk):
        acc = np.zeros((min(chunk, q.shape[0] - s), x.shape[0]), np.float32)
        for k in range(q.shape[1]):
            d = q[s:s + chunk, None, k] - x[None, :, k]
            acc = acc + d * d
        out[s:s + chunk] = acc
    return out


def metrics64(dist, qlab, xlab, exclude, levels):
    """(ap, prec, num_relevant) from the definitions: results by (d, index), AP = ordered float64 sum of hits/k over relevant ranks / R,
    prec[l] = max hits/k over ranks with hits * (L - 1) >= l * R."""
    qn, m = dist.shape
    ap, prec, nrel = np.full(qn, np.nan), np.full((qn, levels), np.nan), np.zeros(qn, np.int32)
    for i in range(qn):
        idx = np.arange(m)
        if exclude:
            idx = idx[idx != i]
        order = idx[np.argsort(dist[i, idx], kind="stable")]
        rel = np.asarray(xlab)[order] == qlab[i]
        hits = np.cumsum(rel)
        R = int(hits[-1]) if hits.size else 0
        nrel[i] = R
        if R == 0:
            continue
        k = np.arange(1, order.size + 1)
        terms = hits[rel] / k[rel]
        ap[i] = np.cumsum(terms)[-1] / R
        for l in range(levels):
            ok = hits * (levels - 1) >= l * R
            prec[i, l] = np.max(hits[ok] / k[ok])
    return ap, prec, nrel


def test_restatement_on_hand_worked_cases():
    # all relevant: AP 1, every precision 1
    ap, prec, r = metrics64(np.array([[0.3, 0.1, 0.2]], np.float32), [5], [5, 5, 5], False, 11)
    assert ap[0] == 1.0 and np.all(prec == 1.0) and r[0] == 3
    # one relevant item at rank r: AP 1/r and a flat curve at 1/r
    for rank in (1, 2, 5):
        d = np.arange(6, dtype=np.float32)[None]
        lab = [0] * 6
        lab[rank - 1] = 1
        ap, prec, r = metrics64(d, [1], lab, False, 11)
        assert ap[0] == 1.0 / rank and np.all(prec == 1.0 / rank) and r[0] == 1
    # relevant at ranks 1 and 3: AP (1 + 2/3) / 2; the curve is 1 up to recall 1/2, then 2/3
    ap, prec, _ = metrics64(np.array([[0.0, 1.0, 2.0]], np.float32), [1], [1, 0, 1], False, 5)
    assert ap[0] == (1.0 + 2.0 / 3.0) / 2 and np.array_equal(prec[0], [1, 1, 1, 2 / 3, 2 / 3])
    # no relevant item: NaN, and left out of the mean
    ap, prec, r = metrics64(np.zeros((1, 4), np.float32), [9], [0, 1, 2, 3], False, 11)
    assert np.isnan(ap[0]) and np.all(np.isnan(prec)) and r[0] == 0
    m = {"ap": torch.tensor([0.5, float("nan"), 1.0], dtype=torch.float64), "num_relevant": torch.tensor([2, 0, 1], dtype=torch.int32),
         "precision": torch.tensor([[1.0, 0.5], [float("nan")] * 2, [1.0, 1.0]], dtype=torch.float64)}
    means, count = ev._retrieval_means(m)
    assert int(count) == 2 and means.tolist() == [0.75, 1.0, 0.75]
    # equal distances rank by index: the relevant item at index 2 behind two irrelevant ties is rank 3
    ap, _, _ = metrics64(np.full((1, 4), 0.5, np.float32), [1], [0, 0, 1, 0], False, 11)
    assert ap[0] == 1.0 / 3.0
    # leave-one-out drops the query's own row: its own label does not count
    ap, _, r = metrics64(np.array([[0.0, 1.0, 2.0]], np.float32), [1], [1, 0, 1], True, 11)
    assert r[0] == 1 and ap[0] == 0.5


def test_distance_restatement_rounds_each_step():
    q, x = np.array([[1e8, 1.0, -1.0]], np.float32), np.array([[0.0, 0.0, 0.0]], np.float32)
    # float32: 1e16 + 1 + 1 stays 1e16 when each sum is rounded
    assert distances32(q, x)[0, 0] == np.float32(np.float32(1e8) * np.float32(1e8))


# ----------------------------------------------------------------------------------------------------- host
def test_abi_header_table_and_exports_agree(lib):
    hdr = open(os.path.join(ROOT, "include", "samplenet_b200.h")).read()
    for name in NAMES:
        assert re.search(r"\b%s\s*\(" % name, hdr) and name in _lib.exported_symbols() and hasattr(lib, name)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert all(re.search(r" T %s$" % n, out, re.M) for n in NAMES)


def test_envelope_corners_and_bounds(lib):
    ok = lib.snb200_retrieval_metrics_supported
    for q, m, d, L, ex in ((1, 1, 1, 2, 0), (1, 1, 1, 2, 1), (1 << 20, 16384, 1024, 101, 0), (16384, 16384, 1024, 101, 1), (2468, 9843, 256, 11, 0)):
        assert ok(q, m, d, L, ex) == 1, (q, m, d, L, ex)
    for q, m, d, L, ex in ((1, 16385, 8, 11, 0), (1, 8, 1025, 11, 0), (1, 8, 8, 1, 0), (1, 8, 8, 102, 0), (7, 8, 8, 11, 1), ((1 << 20) + 1, 8, 8, 11, 0),
                           (0, 8, 8, 11, 0), (1, 0, 8, 11, 0), (1, 8, 0, 11, 0)):
        assert ok(q, m, d, L, ex) == 0, (q, m, d, L, ex)


@pytest.mark.parametrize("q,m,d,L,ex,bound", [(1, 16385, 8, 11, 0, "16384"), (1, 8, 1025, 11, 0, "1024"), (1, 8, 8, 1, 0, "101"),
                                              (1, 8, 8, 102, 0, "101"), (7, 8, 8, 11, 1, "exclude_diagonal")])
def test_outside_the_envelope_returns_unsupported_before_touching_memory(lib, q, m, d, L, ex, bound):
    before = _lib.launch_count()
    bogus = ctypes.c_void_p(16)      # never dereferenced: the envelope is checked from the sizes alone
    rc = lib.snb200_retrieval_metrics(q, m, d, bogus, bogus, bogus, bogus, ex, L, bogus, bogus, bogus, None)
    assert rc == -4 and _lib.launch_count() == before
    msg = lib.snb200_last_error().decode()
    assert msg.startswith("retrieval_metrics") and bound in msg


def test_ops_rejects_cpu_tensors_and_bad_shapes():
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.retrieval_metrics(torch.zeros(3, 4), torch.zeros(3, dtype=torch.int64))
    with pytest.raises(ValueError):
        ops.retrieval_metrics(torch.zeros(3, 4), torch.zeros(2, dtype=torch.int64))
    with pytest.raises(ValueError):
        ops.retrieval_metrics(torch.zeros(3, 4), torch.zeros(3, dtype=torch.int64), torch.zeros(5, 4))


# ----------------------------------------------------------------------------------------------------- the kernel on the GPU
def _labels(g, n, classes=40):
    """Uneven classes: class c drawn with weight c + 1."""
    w = np.arange(1, classes + 1, dtype=np.float64)
    return g.choice(classes, size=n, p=w / w.sum()).astype(np.int32)


def _case(name):
    g = np.random.default_rng(zlib.crc32(name.encode()))
    if name == "loo_2468":
        x = g.standard_normal((2468, 256)).astype(np.float32)
        return x, _labels(g, 2468), None, None
    if name == "2468x9843":
        return (g.standard_normal((2468, 256)).astype(np.float32), _labels(g, 2468), g.standard_normal((9843, 256)).astype(np.float32),
                _labels(g, 9843))
    if name == "300x16384x1024":
        return (g.standard_normal((300, 1024)).astype(np.float32), _labels(g, 300, 7), g.standard_normal((16384, 1024)).astype(np.float32),
                _labels(g, 16384, 7))
    if name == "1x1x1":
        return np.array([[0.5]], np.float32), np.array([3], np.int32), np.array([[-0.25]], np.float32), np.array([3], np.int32)
    if name == "7x5x3":
        return g.standard_normal((7, 3)).astype(np.float32), _labels(g, 7, 3), g.standard_normal((5, 3)).astype(np.float32), _labels(g, 5, 3)
    if name == "duplicates":     # repeated rows: many distances exactly equal, ranked by index
        base = g.integers(-2, 3, size=(40, 9)).astype(np.float32)
        x = base[g.integers(0, 40, size=3000)]
        return x[:500].copy(), _labels(g, 500, 5), x, _labels(g, 3000, 5)
    if name == "singleton_class":     # leave-one-out where query 17's class has no other member
        x = g.standard_normal((600, 61)).astype(np.float32)
        lab = _labels(g, 600, 6)
        lab[17] = 99
        return x, lab, None, None
    raise KeyError(name)


def _run(q, ql, x, xl, levels):
    dev = torch.device("cuda")
    t = lambda a: torch.from_numpy(a).to(dev)
    if x is None:
        return ops.retrieval_metrics(t(q), t(ql), recall_levels=levels)
    return ops.retrieval_metrics(t(q), t(ql), t(x), t(xl), recall_levels=levels)


@gpu
@pytest.mark.parametrize("name,levels", [("loo_2468", 11), ("2468x9843", 11), ("300x16384x1024", 101), ("1x1x1", 2), ("7x5x3", 11),
                                         ("duplicates", 11), ("singleton_class", 21)])
def test_kernel_equals_the_float64_restatement(name, levels):
    q, ql, x, xl = _case(name)
    got = {k: v.cpu().numpy() for k, v in _run(q, ql, x, xl, levels).items()}
    exclude = x is None
    dist = distances32(q, q if exclude else x)
    ap, prec, nrel = metrics64(dist, ql, ql if exclude else xl, exclude, levels)
    assert np.array_equal(got["num_relevant"], nrel)
    assert np.array_equal(got["precision"], prec, equal_nan=True)       # a maximum of exactly rounded quotients: no rounding freedom
    assert np.array_equal(np.isnan(got["ap"]), np.isnan(ap))
    live = ~np.isnan(ap)
    np.testing.assert_array_max_ulp(got["ap"][live], ap[live], maxulp=1)
    if name == "singleton_class":
        assert np.isnan(got["ap"][17]) and nrel[17] == 0
    if name == "duplicates":
        assert (np.diff(np.sort(dist, axis=1), axis=1) == 0).mean() > 0.5


@gpu
def test_kernel_is_deterministic_and_writes_only_its_outputs(lib):
    q, ql, x, xl = _case("2468x9843")
    dev = torch.device("cuda")
    q, ql, x, xl = (torch.from_numpy(a).to(dev) for a in (q[:333], ql[:333], x[:5000], xl[:5000]))
    n, L, pad = 333, 11, 64
    canary = float.fromhex("0x1.dead0beefp+7")
    ap_buf = torch.full((n + 2 * pad,), canary, dtype=torch.float64, device=dev)
    prec_buf = torch.full((n * L + 2 * pad,), canary, dtype=torch.float64, device=dev)
    nrel_buf = torch.full((n + 2 * pad,), -777, dtype=torch.int32, device=dev)
    ins = [t.clone() for t in (q, ql, x, xl)]
    outs = []
    for _ in range(3):
        rc = lib.snb200_retrieval_metrics(n, 5000, 256, q.data_ptr(), ql.data_ptr(), x.data_ptr(), xl.data_ptr(), 0, L, ap_buf[pad:].data_ptr(),
                                          prec_buf[pad:].data_ptr(), nrel_buf[pad:].data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize()
        for buf, lo, hi, fill in ((ap_buf, pad, pad + n, canary), (prec_buf, pad, pad + n * L, canary), (nrel_buf, pad, pad + n, -777)):
            assert bool((buf[:lo] == fill).all()) and bool((buf[hi:] == fill).all())
        outs.append((ap_buf.clone(), prec_buf.clone(), nrel_buf.clone()))
    assert all(torch.equal(a, b) for o in outs[1:] for a, b in zip(o, outs[0]))
    assert all(torch.equal(a, b) for a, b in zip(ins, (q, ql, x, xl)))
    assert not bool((nrel_buf[pad:pad + n] == -777).any())


@gpu
def test_ops_outside_the_envelope_raises_with_the_kernel_message():
    dev = torch.device("cuda")
    with pytest.raises(_lib.SampleNetB200Error, match="16384"):
        ops.retrieval_metrics(torch.zeros(2, 4, device=dev), torch.zeros(2, dtype=torch.int32, device=dev), torch.zeros(16385, 4, device=dev),
                              torch.zeros(16385, dtype=torch.int32, device=dev))
    with pytest.raises(_lib.SampleNetB200Error, match="101"):
        ops.retrieval_metrics(torch.zeros(2, 4, device=dev), torch.zeros(2, dtype=torch.int32, device=dev), recall_levels=1)


# ----------------------------------------------------------------------------------------------------- the descriptors
def _randomise_bn(net, seed):
    g = torch.Generator().manual_seed(seed)
    for mod in net.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.running_mean.copy_(0.1 * torch.randn(mod.num_features, generator=g))
            mod.running_var.copy_(0.5 + torch.rand(mod.num_features, generator=g))
            mod.weight.data.copy_(0.5 + torch.rand(mod.num_features, generator=g))


def _classifier(kind, seed=0):
    torch.manual_seed(seed)
    net = (tasknets.PointNetCls() if kind == "basic" else tasknets.PointNetClsTransforms()).cuda()
    _randomise_bn(net, seed + 1)
    return net.requires_grad_(False).eval()


def _by_hand(net, gfv):
    return torch.relu(net.bn_fc2(net.fc2(torch.relu(net.bn_fc1(net.fc1(gfv))))))


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@gpu
@pytest.mark.parametrize("kind", ["basic", "transforms"])
def test_retrieval_vectors_on_every_classifier_path(kind, monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    net = _classifier(kind)
    frozen = tasknets.FrozenPointNetCls(net) if kind == "basic" else tasknets.FrozenPointNetClsTransforms(net)
    b = 40 if kind == "basic" else 70      # FrozenPointNetCls takes up to 64 clouds; the transforms wrapper runs 70 in two chunks
    x = (torch.rand(b, 200, 3, generator=torch.Generator().manual_seed(5)) * 2 - 1).cuda()
    with torch.no_grad():
        logits, ep = net(x)
        flog, fep = frozen(x)
    # the module: fc3's input, and logits as the head computes them
    assert ep["retrieval_vectors"].shape == (b, 256)
    assert torch.equal(ep["retrieval_vectors"], _by_hand(net, ep["GFV"])) and torch.equal(logits, net.fc3(_by_hand(net, ep["GFV"])))
    # the frozen wrapper: the module's descriptor of its own GFV, and of the module's within the frozen-path bar
    assert set(fep) == set(ep)
    assert _rel(fep["retrieval_vectors"], _by_hand(net, fep["GFV"])) <= 1e-5
    assert _rel(fep["retrieval_vectors"], ep["retrieval_vectors"]) <= 1e-4 and _rel(flog, logits) <= 1e-4
    # logits as the parent computed them: the same head call, bit for bit
    with torch.no_grad():
        if kind == "basic":
            assert torch.equal(flog, net.head(fep["GFV"]))
        else:
            P = frozen._plan()
            old = torch.cat([ops.FrozenMLPBNFunction.apply(fep["GFV"][s:s + 64].contiguous(), P["head"]) for s in (0, 64)])
            assert torch.equal(flog, old)
    # every prefix: prefix s equals forward(x[:, :s])
    sizes = [1, 7, 64, 128, 200]
    with torch.no_grad():
        plog, peps = frozen.prefixes(x, sizes, return_end_points=True)
        for i, s in enumerate(sizes):
            slog, sep = frozen(x[:, :s].contiguous())
            assert set(peps[i]) == set(sep)
            assert _rel(peps[i]["retrieval_vectors"], sep["retrieval_vectors"]) <= 1e-5 and _rel(plog[i], slog) <= 1e-5
            assert torch.equal(peps[i]["GFV"], sep["GFV"]) or _rel(peps[i]["GFV"], sep["GFV"]) <= 1e-5
        if kind == "transforms":
            gfv, head = torch.stack([e["GFV"] for e in peps]), frozen._plan()["head"]
            old = torch.cat([frozen._rows(gfv[:, s:s + 64].flatten(0, 1), head).view(len(sizes), -1, plog.shape[2]) for s in (0, 64)], dim=1)
            assert torch.equal(plog, old)
            assert torch.equal(frozen.prefixes(x, sizes), plog)


@gpu
def test_frozen_transforms_logits_keep_their_gradient():
    net = _classifier("transforms")
    frozen = tasknets.FrozenPointNetClsTransforms(net)
    x = (torch.rand(5, 64, 3, generator=torch.Generator().manual_seed(2)) * 2 - 1).cuda().requires_grad_(True)
    logits, ep = frozen(x)
    assert not ep["retrieval_vectors"].requires_grad
    logits.sum().backward()
    g1 = x.grad.clone()
    x.grad = None
    logits2, _ = frozen(x)
    logits2.sum().backward()
    assert torch.equal(g1, x.grad) and torch.isfinite(g1).all()


# ----------------------------------------------------------------------------------------------------- the evaluators
class _Readbacks:
    """Counts the device-to-host reads of CUDA tensors that Python can see: .item(), .cpu(), .tolist()."""

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


def _clouds(n, points, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, points, 3, generator=g) * 2 - 1).cuda(), torch.randint(0, 5, (n,), generator=g).cuda()


@gpu
@pytest.mark.parametrize("sampler_kind", ["samplenet", "fps"])
def test_retrieval_evaluator_equals_metrics_on_hand_gathered_descriptors(sampler_kind):
    torch.manual_seed(0)
    sampler = sb.ClassificationSampleNet(32).cuda() if sampler_kind == "samplenet" else sb.FPSSampler(32, False, "bnc", "bnc")
    net = _classifier("transforms")
    cls = tasknets.FrozenPointNetClsTransforms(net)
    pcs, labels = _clouds(40, 256, 3)
    evaluator = sb.RetrievalEvaluator(sampler, cls, 32)
    with _Readbacks() as rb:
        out = evaluator.evaluate(pcs, labels, batch_size=16)
    assert rb.count == 1
    with torch.no_grad():
        ce = sb.ClassificationEvaluator(sampler, cls, 32)
        if hasattr(sampler, "eval"):
            sampler.eval()
        desc = torch.cat([cls(ce.clouds(pcs[s:s + 16])["sampled"])[1]["retrieval_vectors"] for s in range(0, 40, 16)])
        want = ops.retrieval_metrics(desc, labels)
    wap = want["ap"].cpu().numpy()
    assert np.array_equal(out["ap"], wap, equal_nan=True)
    live = want["num_relevant"].cpu().numpy() > 0
    assert out["num_queries"] == int(live.sum())
    assert out["map"] == pytest.approx(float(wap[live].mean()), rel=1e-12)
    assert np.allclose(out["precision"], want["precision"].cpu().numpy()[live].mean(axis=0), rtol=1e-12)
    assert np.array_equal(out["recall_levels"], np.linspace(0, 1, 11))


class _MeanDescriptor(torch.nn.Module):
    """A stand-in classifier whose descriptor is the cloud's centroid (three channels)."""

    def forward(self, x):
        v = x.mean(dim=1)
        return v, {"retrieval_vectors": v}


@gpu
def test_class_separated_descriptors_give_map_one_and_complete_equals_leave_one_out():
    g = torch.Generator().manual_seed(9)
    labels = torch.randint(0, 6, (90,), generator=g)
    pcs = (torch.rand(90, 128, 3, generator=g) * 0.1 + labels[:, None, None].float() * 5).cuda()
    evaluator = sb.RetrievalEvaluator(None, _MeanDescriptor(), 32)
    loo = evaluator.evaluate(pcs, labels.cuda(), batch_size=32)
    assert loo["map"] == 1.0 and np.all(loo["precision"] == 1.0)
    pcs2 = (torch.rand(90, 128, 3, generator=g) * 2 - 1).cuda()
    net = _classifier("basic")
    ev2 = sb.RetrievalEvaluator(None, tasknets.FrozenPointNetCls(net), 32)
    a, b = ev2.evaluate(pcs2, labels.cuda()), ev2.evaluate(pcs2, labels.cuda(), database="complete")
    assert np.array_equal(a["ap"], b["ap"], equal_nan=True) and a["map"] == b["map"] and np.array_equal(a["precision"], b["precision"])
    with pytest.raises(ValueError):
        ev2.evaluate(pcs2, labels.cuda(), database="train")


@gpu
def test_progressive_retrieval_equals_the_evaluator_per_size():
    torch.manual_seed(0)
    sampler = sb.ClassificationSampleNet(64).cuda()
    net = _classifier("basic")
    pcs, labels = _clouds(24, 1024, 4)
    plain, frozen = sb.ProgressiveClassificationEvaluator(sampler, net), sb.ProgressiveClassificationEvaluator(sampler, tasknets.FrozenPointNetCls(net))
    ordered = frozen.order(pcs, batch_size=8)
    sizes = [8, 32, 1024]
    with _Readbacks() as rb:
        got = plain.retrieval(pcs, labels, sizes, batch_size=8, ordered=ordered)
    assert rb.count == 1 and got["sizes"] == sizes and got["precision"].shape == (3, 11)
    for i, s in enumerate(sizes):
        want = sb.RetrievalEvaluator(None, net, s).evaluate(ordered[:, :s].contiguous(), labels, batch_size=8)
        assert got["map"][i] == want["map"] and np.array_equal(got["precision"][i], want["precision"])
    with _Readbacks() as rb:
        fg = frozen.retrieval(pcs, labels, [1024, 8, 32], batch_size=8, ordered=ordered)
    assert rb.count == 1
    assert np.allclose(fg["map"], got["map"][[2, 0, 1]], atol=0.02)
    with pytest.raises(ValueError):
        plain.retrieval(pcs, labels, [0, 4], ordered=ordered)
