"""Backward kernels downstream of the generator against plain float64 torch autograd on the CPU: the soft projection
(csrc/softproj.cu, every sigma mode and public entry point), the fused projection + simplification-loss tail, the Chamfer
backward (csrc/chamfer.cu), the progressive loss and group_point_grad / gather_point.

The float64 graph is evaluated on the kernels' own routing -- the kNN indices of knn_soft_project_forward, the Chamfer
idx1 / idx2 and the FIRST arg-max of the kernel's fp32 dist1 -- exactly as the generator backward test does with its
max-pool routing.  The forward tests prove those indices bit-exact; recomputing them in float64 would turn near-ties into
spurious failures.  What remains is rounding, and each bar is written at its comparison as

    max |kernel - float64| <= c * scale

where the scale is the float64 tensor's max |value|, or, where a gradient is a sum whose terms can cancel (cloud points
shared by many queries, the temperature), the largest sum of |terms| in float64.  Sigma is chosen from the data so that
d / sigma stays <= 10 over the neighbours: a steeper softmax amplifies fp32 rounding legitimately.

The tests without the `gpu` mark pin the float64 references themselves (against the reference class's fixture, the C
oracle and the per-prefix definition of the progressive loss), so a wrong yardstick cannot pass a wrong kernel.
"""
import os

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def sb():
    import samplenet_b200

    samplenet_b200._lib.lib()  # fail loudly if the CUDA library is missing
    return samplenet_b200


def _cpu64(t):
    return t.detach().to("cpu", torch.float64)


def _leaf(t):
    return _cpu64(t).requires_grad_(True)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bnc(t, layout):
    """(b, c, n) -> (b, n, c) view for layout 'bcn'."""
    return t if layout == "bnc" else t.transpose(1, 2)


def _abs_scatter(idx, terms, n):
    """sum of |terms| per target point: idx (b, E) long, terms (b, E, c) -> (b, n, c)."""
    b, _, c = terms.shape
    out = torch.zeros(b, n, c, dtype=torch.float64)
    return out.scatter_add_(1, idx[..., None].expand(b, idx.shape[1], c), terms.abs())


class _Bars:
    """Collects every comparison of a test, prints its error in units of the scale, and fails at the end with all of them."""

    def __init__(self):
        self.failed = []

    def check(self, what, got, ref, scale, bar):
        err = float((_cpu64(got) - ref).abs().max())
        scale = float(scale)
        if scale == 0.0:   # every term is exactly zero (k = 1: the softmax is constant): so must the kernel's result be
            print("%-34s err %.2e  (scale 0)" % (what, err))
        else:
            print("%-34s err/scale %.2e  (bar %.0e)" % (what, err / scale, bar))
        if not err <= bar * scale:
            self.failed.append("%s: max err %.3e > %.0e * %.3e" % (what, err, bar, scale))

    def done(self):
        assert not self.failed, "\n".join(self.failed)


# ---------------------------------------------------------------------------------------------------- float64 references
def _sigma64(t, mode, floor):
    """sigma as the reference classes evaluate it: 0 sigma itself, 1 max(T^2, floor) (registration), 2 T^2 (classification),
    3 max(T, floor)^2 (reconstruction)."""
    if mode == 0:
        return t
    if mode == 1:
        return torch.clamp(t * t, min=floor)
    if mode == 2:
        return t * t
    return torch.clamp(t, min=floor) ** 2


def _softproj64(points, query, t, feats, idx, mode, floor):
    """Soft projection of BNC float64 clouds on the given neighbour indices idx (b, m, k): d = |g - q|^2 / sigma,
    w = softmax(-d), proj = sum w g, prop = sum w F[idx].  Also returns the intermediates the error scales are built from."""
    b, m, k = idx.shape
    bi = torch.arange(b)[:, None, None]
    g = points[bi, idx]                                   # (b, m, k, 3) the neighbours
    qb = query[:, :, None, :].expand(b, m, k, 3)
    s = _sigma64(t, mode, floor)
    d = ((g - qb) ** 2).sum(-1) / s
    w = torch.softmax(-d, dim=-1)
    out = {"proj": (w[..., None] * g).sum(2), "g": g, "qb": qb, "d": d, "s": s, "w": w}
    if feats is not None:
        out["fg"] = feats[bi, idx]
        out["prop"] = (w[..., None] * out["fg"]).sum(2)
    return out


def _sq(a):
    return (a ** 2).sum(-1)


def _first_argmax(d):
    """Index of the FIRST maximum along dim 1 (torch.argmax's documented tie rule)."""
    return d.argmax(dim=1)


def _simp64(ref, samp, w21, i1, i2, am):
    """Simplification loss terms [mean c12, mean_b max c12, mean c21] and loss on given routing: i1 (b, s) samp -> ref,
    i2 (b, n) ref -> samp, am (b,) the arg-max of c12."""
    bi = torch.arange(ref.shape[0])[:, None]
    c12 = _sq(samp - ref[bi, i1])
    c21 = _sq(ref - samp[bi, i2])
    terms = torch.stack([c12.mean(), c12.gather(1, am[:, None]).mean(), c21.mean()])
    return terms[0] + terms[1] + w21 * terms[2], terms


def _progressive64(ref, samp, sizes, weights, idx1, idx2, dist1):
    """The progressive loss in one pass, like csrc/progressive.cu: c12 of all ordered samples once, prefix s takes c12[:, :s] and
    its max term at the first index attaining the running maximum of dist1; idx2 (b, P, n) the ref -> prefix indices.
    Returns (total, terms (P, 3))."""
    b, m = idx1.shape
    bi = torch.arange(b)
    sz = torch.tensor(sizes)
    c12 = _sq(samp - ref[bi[:, None], idx1])                                     # (b, m)
    cover = (torch.arange(m)[None, :] < sz[:, None]).to(torch.float64)           # (P, m)
    t0 = (c12[:, None, :] * cover).sum((0, 2)) / (b * sz.to(torch.float64))
    run_max = torch.cummax(dist1, dim=1).values[:, sz - 1]                       # (b, P)
    am = (dist1[:, None, :] == run_max[:, :, None]).to(torch.int32).argmax(2)    # (b, P) first j attaining it
    t1 = c12.gather(1, am).mean(0)
    t2 = _sq(ref[:, None] - samp[bi[:, None, None], idx2]).mean((0, 2))          # (P,)
    terms = torch.stack([t0, t1, t2], 1)
    return (t0 + t1 + torch.tensor(weights, dtype=torch.float64) * t2).sum(), terms


# ---------------------------------------------------------------------------------------------------- CPU: pin the yardsticks
def test_softproj_reference_reproduces_reference_fixture(oracle, golden_dir):
    """The float64 soft projection reproduces the reference class's own outputs and all four gradients
    (registration/src/soft_projection.py, B=3, N=200, M=17, k=8, F=5, BCN, sigma = max(T^2, 1e-4), T = 0.7)."""
    z = np.load(os.path.join(golden_dir, "softproj_reg.npz"))
    k = int(z["k"])
    _, idx = oracle.knn_point(k, z["point_cloud"].transpose(0, 2, 1), z["query_cloud"].transpose(0, 2, 1), tie_mode=1)
    P, Q, F = (torch.from_numpy(z[key]).double().requires_grad_(True) for key in ("point_cloud", "query_cloud", "feats"))
    T = torch.tensor(float(z["temperature"]), dtype=torch.float64, requires_grad=True)
    o = _softproj64(_bnc(P, "bcn"), _bnc(Q, "bcn"), T, _bnc(F, "bcn"), torch.from_numpy(idx).long(), 1, float(z["min_sigma"]))
    proj, prop = o["proj"].transpose(1, 2), o["prop"].transpose(1, 2)
    # the fixture is the reference's fp32 evaluation: forward values agree to fp32 rounding
    np.testing.assert_allclose(proj.detach().numpy(), z["proj"], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(prop.detach().numpy(), z["prop"], rtol=2e-6, atol=2e-6)
    L = (proj * torch.from_numpy(z["r1"]).double()).sum() + (prop * torch.from_numpy(z["r2"]).double()).sum()
    gP, gQ, gF, gT = torch.autograd.grad(L, [P, Q, F, T])
    bars = _Bars()
    # fp32 rounding of the fixture's own autograd graph (softmax backward over k = 8, sums over the cloud; measured <= 2e-7)
    for name, got, want in (("grad_point_cloud", gP, "grad_point_cloud"), ("grad_query_cloud", gQ, "grad_query_cloud"),
                            ("grad_feats", gF, "grad_feats"), ("grad_temperature", gT, "grad_temperature")):
        ref = torch.from_numpy(np.asarray(z[want])).double()
        bars.check("fixture " + name, got, ref, float(ref.abs().max()), 2e-6)
    bars.done()


def test_softproj_reference_forward_equals_oracle(oracle):
    """The float64 forward equals the C oracle's soft projection (fp32, sequential) on random inputs with features."""
    for seed, (b, n, m, k, f, sigma) in enumerate([(2, 300, 40, 8, 3, 0.01), (1, 64, 64, 1, 2, 0.3), (3, 500, 20, 32, 5, 0.05)]):
        g = _gen(seed)
        pts = (torch.rand(b, n, 3, generator=g) - 0.5).numpy()
        qry = (torch.rand(b, m, 3, generator=g) - 0.5).numpy()
        ft = torch.randn(b, n, f, generator=g).numpy()
        _, idx = oracle.knn_point(k, pts, qry, contract=True, tie_mode=1)
        proj, w, d, prop = oracle.soft_project(pts, qry, idx, sigma, feats=ft)
        sig = float(np.float32(sigma))
        o = _softproj64(torch.from_numpy(pts).double(), torch.from_numpy(qry).double(), torch.tensor(sig, dtype=torch.float64),
                        torch.from_numpy(ft).double(), torch.from_numpy(idx).long(), 0, 0.0)
        np.testing.assert_allclose(o["proj"].numpy(), proj, rtol=1e-5, atol=1e-6)   # fp32 rounding of the oracle
        np.testing.assert_allclose(o["prop"].numpy(), prop, rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(o["w"].numpy(), w, rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(o["d"].numpy(), d, rtol=1e-5, atol=1e-7)


def test_progressive_reference_equals_per_prefix_sum(oracle):
    """The one-pass float64 progressive loss equals the sum over prefixes of the simplification loss of each prefix, each with
    its own nearest-neighbour search and first-maximum routing, in value and gradient -- also with a duplicated outlier that is
    the maximum of several prefixes.  Each prefix's loss also equals the C oracle's simplification loss."""
    g = _gen(3)
    b, n, m, sizes = 3, 400, 64, [2, 4, 9, 16, 40, 64]
    ref0 = torch.rand(b, n, 3, generator=g, dtype=torch.float64) - 0.5
    samp0 = torch.rand(b, m, 3, generator=g, dtype=torch.float64) - 0.5
    samp0[:, 3] = samp0[:, 10] = samp0[:, 40] = torch.tensor([1.5, 1.5, 1.5], dtype=torch.float64)   # the max from s = 4 on, tied from s = 16 on
    weights = [1.0 + 0.01 * s for s in sizes]
    ref, samp = ref0.clone().requires_grad_(True), samp0.clone().requires_grad_(True)
    D = _sq(samp0[:, :, None] - ref0[:, None])                # (b, m, n) squared distances, elementwise (no matmul shortcut)
    idx1 = D.argmin(2)
    dist1 = D.gather(2, idx1[..., None])[..., 0]
    idx2 = torch.stack([D[:, :s].argmin(1) for s in sizes], 1)
    total, terms = _progressive64(ref, samp, sizes, weights, idx1, idx2, dist1)
    ref2, samp2 = ref0.clone().requires_grad_(True), samp0.clone().requires_grad_(True)
    per = []
    for s, w in zip(sizes, weights):
        Ds = _sq(samp0[:, :s, None] - ref0[:, None])              # a stand-alone nearest-neighbour search per prefix
        i1 = Ds.argmin(2)
        am = _first_argmax(Ds.gather(2, i1[..., None])[..., 0])
        loss, t = _simp64(ref2, samp2[:, :s], w, i1, Ds.argmin(1), am)
        per.append((loss, t))
        want = oracle.simplification_loss(ref0.float().numpy(), samp0[:, :s].float().numpy(), s, 1.0, 0.01)
        assert abs(float(loss.detach()) - float(want)) <= 1e-5 * abs(float(want))   # the oracle runs in fp32
    assert torch.allclose(total, sum(p[0] for p in per), rtol=1e-12, atol=0)
    assert torch.allclose(terms, torch.stack([p[1] for p in per]), rtol=1e-12, atol=0)
    gr, gs = torch.autograd.grad(total, [ref, samp])
    gr2, gs2 = torch.autograd.grad(sum(p[0] for p in per), [ref2, samp2])
    assert torch.allclose(gr, gr2, rtol=1e-10, atol=1e-14) and torch.allclose(gs, gs2, rtol=1e-10, atol=1e-14)
    assert float(gs[:, 10].abs().max()) > 0 and float(gs[:, 3].norm()) > float(gs[:, 10].norm())   # the max terms went to index 3


# ---------------------------------------------------------------------------------------------------- GPU: soft projection
def _clouds(seed, b, n, m, f, layout, kind):
    """Points uniform in the unit cube, queries near cloud points; kind 'hub': every query within 1e-3 of point 0 (which is then a
    neighbour of all of them); 'dup': a block of duplicated cloud points with queries among them."""
    g = _gen(seed)
    pts = torch.rand(b, n, 3, generator=g) - 0.5
    if kind == "dup":
        pts[:, n // 2:n // 2 + n // 8] = pts[:, :n // 8]
        qry = pts[:, torch.randint(0, n // 8, (m,), generator=g)] + 0.01 * torch.randn(b, m, 3, generator=g)
    elif kind == "hub":
        qry = pts[:, :1] + 1e-3 * torch.randn(b, m, 3, generator=g)
    else:
        qry = pts[:, torch.randint(0, n, (m,), generator=g)] + 0.02 * torch.randn(b, m, 3, generator=g)
    ft = torch.randn(b, n, f, generator=g) if f else None
    lay = (lambda t: t.contiguous()) if layout == "bnc" else (lambda t: t.transpose(1, 2).contiguous())
    return lay(pts).cuda(), lay(qry).cuda(), (lay(ft).cuda() if f else None)


def _knn(sb, P, Q, k, layout):
    """The kernel's neighbour indices, and sigma = max squared neighbour distance / 10 (so d / sigma <= 10)."""
    o = sb.ops.knn_soft_project_forward(P, Q, k, layout, want=("idx", "val"))
    return o["idx"].long().cpu(), float(o["val"].max()) / 10.0


def _temperature(mode, sig, clamped=False, negative=False):
    """(t, floor) so that the mode's sigma(t) == sig; clamped: the floor is active (sigma == floor resp. floor^2 == sig)."""
    if mode == 0:
        return sig, 0.0
    r = float(np.sqrt(sig))
    if mode == 1:
        return (0.5 * r, sig) if clamped else (r, 1e-4 * sig)
    if mode == 2:
        return (-r if negative else r), 0.0
    return (0.5 * r, r) if clamped else (r, 0.01 * r)


def _entry(layout, mode, f):
    """Which public entry point drives a case: the registration module for sigma mode 1 (BCN, or BNC projection), the TF-flavoured
    module for modes 2 / 3 (BNC projection), the autograd Function itself otherwise (mode 0, BNC features, BCN with modes 2 / 3)."""
    if mode == 1 and (layout == "bcn" or f == 0):
        return "module"
    if mode in (2, 3) and layout == "bnc" and f == 0:
        return "tf"
    return "function"


def _softproj_gpu(sb, entry, P, Q, F, k, layout, mode, t0, floor, want=("proj", "prop"), need=("points", "query", "feats", "t"),
                  upstream=None):
    """One forward + backward through `entry`.  upstream(proj, prop) -> scalar loss.  Returns the outputs, the gradients
    (None where not asked for) and the temperature value the module holds (fp32)."""
    P = P.clone().requires_grad_("points" in need)
    Q = Q.clone().requires_grad_("query" in need)
    F = None if F is None else F.clone().requires_grad_("feats" in need)
    want_proj, want_prop = "proj" in want, "prop" in want and F is not None
    if entry == "module":
        mod = sb.SoftProjection(k, initial_temperature=t0, min_sigma=floor).cuda()
        T = mod._temperature
        T.requires_grad_("t" in need)
        if layout == "bnc":
            proj, prop = mod.project(P, Q, layout="bnc"), None
        elif want_proj and want_prop:
            proj, prop = mod(P, Q, F, action="project_and_propagate")
        elif want_prop:
            proj, prop = None, mod(P, Q, F, action="propagate")
        else:
            proj, prop = mod(P, Q), None
    elif entry == "tf":
        mod = sb.tf_ops.SoftProjection(k, initial_temperature=t0, is_temperature_trainable="t" in need,
                                       sigma_mode="cls" if mode == 2 else "rec", min_sigma=floor).cuda()
        T = mod._temperature
        proj, prop = mod(P, Q)[0], None
    else:
        T = torch.tensor(t0, device="cuda", requires_grad="t" in need)
        proj, prop, _, _, _ = sb.ops.SoftProjectFunction.apply(P, Q, T, F, k, layout, False, want_proj, want_prop, mode, floor)
        proj = proj if want_proj else None
        prop = prop if want_prop else None
    L = upstream(proj, prop)
    L.backward()
    return {"proj": proj, "prop": prop, "points": P.grad, "query": Q.grad, "feats": None if F is None else F.grad, "t": T.grad,
            "t_value": float(T.detach())}


def _softproj_compare(bars, got, P, Q, F, idx, layout, mode, floor, upstream, need):
    """float64 autograd of the same upstream loss on the kernel's idx.  Scales: max |ref| for the outputs, the largest per-query
    sum of |terms| for the query, the largest per-point sum of |terms| for the cloud and the features, the sum of |terms| for the
    temperature.  Bars: about 10x the largest error measured on an H100 over all the cases of this file."""
    P64, Q64 = _leaf(P), _leaf(Q)
    F64 = None if F is None else _leaf(F)
    T64 = torch.tensor(got["t_value"], dtype=torch.float64, requires_grad=True)
    floor = float(np.float32(floor))     # the modules hand the floor to the kernel as fp32
    o = _softproj64(_bnc(P64, layout), _bnc(Q64, layout), T64, None if F64 is None else _bnc(F64, layout), idx, mode, floor)
    proj = _bnc(o["proj"], layout) if got["proj"] is not None else None
    prop = _bnc(o["prop"], layout) if got["prop"] is not None else None
    L = upstream(proj, prop)
    leaves = [P64, Q64, T64] + ([F64] if F64 is not None else [])
    inter = [o["g"], o["qb"], o["d"]] + ([o["fg"]] if F64 is not None else [])
    gr = torch.autograd.grad(L, leaves + inter, allow_unused=True)
    gP, gQ, gT = gr[:3]
    gF = gr[3] if F64 is not None else None
    dg, dqb, dd = gr[len(leaves):len(leaves) + 3]
    dfg = gr[-1] if F64 is not None else None
    b, m, k = idx.shape
    n = P.shape[1] if layout == "bnc" else P.shape[2]
    zero = lambda t: torch.zeros(1, dtype=torch.float64) if t is None else t
    if proj is not None:   # forward: fp32 softmax and weighted sums (measured <= 3.3e-7)
        bars.check("proj", got["proj"], proj.detach(), proj.detach().abs().max(), 2e-6)
    if prop is not None:
        bars.check("prop", got["prop"], prop.detach(), prop.detach().abs().max(), 2e-6)
    if "points" in need:
        scale = _abs_scatter(idx.reshape(b, m * k), zero(dg).reshape(b, m * k, 3), n).max()
        # fp32 exp of d <= 10 and the softmax backward's w (a - sum w a) (measured <= 1.5e-6)
        bars.check("grad points", got["points"], gP, scale, 1e-5)
    else:
        assert got["points"] is None
    if "query" in need:
        bars.check("grad query", got["query"], gQ, zero(dqb).abs().sum(2).max(), 1e-5)   # as the cloud (measured <= 1.2e-6)
    else:
        assert got["query"] is None
    if F is not None and "feats" in need and got["prop"] is not None:
        scale = _abs_scatter(idx.reshape(b, m * k), dfg.reshape(b, m * k, -1), n).max()
        bars.check("grad feats", got["feats"], gF, scale, 1e-6)   # sums of w * grad_prop: no cancellation inside a term (<= 1.0e-7)
    elif F is not None and "feats" not in need:
        assert got["feats"] is None
    if "t" in need:
        clamped = (mode == 1 and got["t_value"] ** 2 <= floor) or (mode == 3 and got["t_value"] <= floor)
        if clamped:   # sigma is the floor: it does not depend on T, the gradient is exactly 0
            assert float(got["t"]) == 0.0 and float(gT) == 0.0, float(got["t"])
        else:
            dsdt = 1.0 if mode == 0 else 2.0 * abs(got["t_value"])
            scale = (dd * o["d"].detach() / o["s"].detach()).abs().sum() * dsdt
            bars.check("grad T", got["t"].reshape(()), gT, scale, 1e-6)   # against the sum of |terms| (measured <= 6e-8)
    else:
        assert got["t"] is None


def _rand_upstream(seed, P, Q, F, m, layout):
    """L = sum(proj * r1) + sum(prop * r2), r1 / r2 fixed random tensors in the outputs' layout (CUDA for the kernel, float64 CPU
    for the reference)."""
    g = _gen(seed)
    b = P.shape[0]
    f = 0 if F is None else (F.shape[2] if layout == "bnc" else F.shape[1])
    r1 = torch.randn((b, m, 3) if layout == "bnc" else (b, 3, m), generator=g)
    r2 = torch.randn((b, m, f) if layout == "bnc" else (b, f, m), generator=g)

    def up(proj, prop):
        dev = (proj if proj is not None else prop).device
        dt = (proj if proj is not None else prop).dtype
        L = 0
        if proj is not None:
            L = L + (proj * r1.to(dev, dt)).sum()
        if prop is not None:
            L = L + (prop * r2.to(dev, dt)).sum()
        return L
    return up


# b, n, m, k, layout, sigma mode, features, data
SOFTPROJ_CASES = [
    (2, 1024, 64, 8, "bnc", 1, 0, "plain"),        # headline
    (3, 200, 17, 8, "bcn", 1, 5, "plain"),         # the reference fixture's shape
    (32, 1024, 32, 7, "bnc", 2, 0, "plain"),       # classification, sigma = T^2 (negative T: the chain rule's sign)
    (4, 2048, 64, 16, "bnc", 3, 0, "plain"),       # reconstruction, sigma = max(T, floor)^2; 8 gather CTAs per cloud
    (2, 1024, 1024, 7, "bnc", 1, 3, "plain"),      # m k = 7168: four gather tiles, with features
    (1, 2048, 2048, 16, "bcn", 0, 3, "plain"),     # sigma given directly; m k = 32768
    (2, 9001, 40, 32, "bnc", 1, 33, "plain"),      # multi-tile forward (neighbours from global memory), k = 32, F > 32
    (3, 77, 300, 1, "bcn", 2, 64, "plain"),        # k = 1, m > n
    (2, 1500, 512, 8, "bcn", 1, 4, "hub"),         # point 0 is a neighbour of all 512 queries: one thread sums across two tiles
    (2, 512, 100, 8, "bnc", 2, 0, "dup"),          # duplicated cloud points
    (2, 600, 300, 6, "bnc", 0, 5, "dup"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,k,layout,mode,f,kind", SOFTPROJ_CASES)
def test_soft_projection_backward_vs_float64(sb, b, n, m, k, layout, mode, f, kind):
    P, Q, F = _clouds(b * 7 + n + m + k, b, n, m, f, layout, kind)
    idx, sig = _knn(sb, P, Q, k, layout)
    t0, floor = _temperature(mode, sig, negative=(mode == 2 and b == 32))
    entry = _entry(layout, mode, f)
    up = _rand_upstream(n + m, P, Q, F, m, layout)
    runs = [_softproj_gpu(sb, entry, P, Q, F, k, layout, mode, t0, floor, upstream=up) for _ in range(2)]
    for key in ("proj", "prop", "points", "query", "feats", "t"):   # no float atomics anywhere: run to run bit-identical
        a, c = runs[0][key], runs[1][key]
        assert (a is None and c is None) or torch.equal(a, c), key
    bars = _Bars()
    _softproj_compare(bars, runs[0], P, Q, F, idx, layout, mode, floor, up, ("points", "query", "feats", "t"))
    bars.done()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,layout,f", [(1, "bcn", 5), (3, "bnc", 0)])
def test_soft_projection_temperature_below_floor(sb, mode, layout, f):
    """T^2 <= floor (mode 1) or T <= floor (mode 3): sigma is the floor, dL/dT is exactly 0 and every other gradient still matches."""
    b, n, m, k = 3, 700, 90, 8
    P, Q, F = _clouds(mode, b, n, m, f, layout, "plain")
    idx, sig = _knn(sb, P, Q, k, layout)
    t0, floor = _temperature(mode, sig, clamped=True)
    up = _rand_upstream(mode, P, Q, F, m, layout)
    got = _softproj_gpu(sb, _entry(layout, mode, f), P, Q, F, k, layout, mode, t0, floor, upstream=up)
    assert got["t"] is not None
    bars = _Bars()
    _softproj_compare(bars, got, P, Q, F, idx, layout, mode, floor, up, ("points", "query", "feats", "t"))
    bars.done()


@pytest.mark.gpu
@pytest.mark.parametrize("want,need", [
    (("proj",), ("points", "query", "feats", "t")),     # projection only: the features get no gradient
    (("prop",), ("points", "query", "feats", "t")),     # propagation only: the cloud through the weights alone
    (("proj", "prop"), ("query", "feats", "t")),        # cloud not requiring grad
    (("proj", "prop"), ("points", "query", "feats")),   # frozen temperature
    (("proj", "prop"), ("feats",)),
])
def test_soft_projection_gradient_subsets(sb, want, need):
    """Gradients that were not asked for are None; the others equal the full float64 graph's."""
    b, n, m, k, f, layout = 2, 700, 300, 8, 6, "bcn"
    P, Q, F = _clouds(11, b, n, m, f, layout, "plain")
    idx, sig = _knn(sb, P, Q, k, layout)
    t0, floor = _temperature(1, sig)
    up = _rand_upstream(12, P, Q, F, m, layout)
    got = _softproj_gpu(sb, "module", P, Q, F, k, layout, 1, t0, floor, want=want, need=need, upstream=up)
    if "prop" not in want:
        assert got["prop"] is None and (got["feats"] is None or float(got["feats"].abs().max()) == 0.0)
    bars = _Bars()
    _softproj_compare(bars, got, P, Q, F, idx, layout, 1, floor, up, need)
    bars.done()


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["sum", "permuted"])
def test_soft_projection_expanded_and_permuted_upstream(sb, form):
    """An expanded (proj.sum()) or non-contiguous (a permuted proj) upstream gradient is read correctly."""
    b, n, m, k, f = 2, 1024, 200, 8, 4
    P, Q, F = _clouds(21, b, n, m, f, "bnc", "plain")
    idx, sig = _knn(sb, P, Q, k, "bnc")
    t0, floor = _temperature(0, sig)
    r = torch.randn(b, 3, m, generator=_gen(22))
    rf = torch.randn(b, f, m, generator=_gen(23))

    def up(proj, prop):
        if form == "sum":
            return proj.sum() + prop.sum()
        dev, dt = proj.device, proj.dtype
        return (proj.permute(0, 2, 1) * r.to(dev, dt)).sum() + (prop.permute(0, 2, 1) * rf.to(dev, dt)).sum()

    got = _softproj_gpu(sb, "function", P, Q, F, k, "bnc", 0, t0, floor, upstream=up)
    bars = _Bars()
    _softproj_compare(bars, got, P, Q, F, idx, "bnc", 0, floor, up, ("points", "query", "feats", "t"))
    bars.done()


# ---------------------------------------------------------------------------------------------------- GPU: fused tail
@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,k,clamped", [(32, 1024, 64, 8, False), (32, 1024, 32, 7, False), (32, 1024, 1024, 7, False),
                                             (50, 2048, 64, 16, False), (8, 1024, 64, 8, True)])
def test_fused_tail_backward_vs_float64(sb, b, n, m, k, clamped):
    """ProjectAndLossFunction (SampleNet's training tail): projection + simplification loss (mean c12 + mean_b max c12 + mean c21)
    in one launch, backward = soft-projection backward + Chamfer backward.  The ref cloud requires grad, so both parts of its gradient
    are summed; every output (projection, loss, the three terms) carries an upstream gradient."""
    g = _gen(b + n + m + k)
    x = (torch.rand(b, n, 3, generator=g) - 0.5).cuda()
    s = (x.cpu()[:, torch.randperm(n, generator=g)[:m]] + 0.02 * torch.randn(b, m, 3, generator=g)).cuda()
    idx, sig = _knn(sb, x, s, k, "bnc")
    t0, floor = _temperature(1, sig, clamped=clamped)
    r = torch.randn(b, m, 3, generator=g)
    cu, ct = 0.7, torch.tensor([0.3, -1.1, 0.5])
    _, _, _, _, dist1, idx1, _, idx2, _ = sb.ops.project_and_loss_forward(x, s, k, torch.tensor([t0], device="cuda"), 1, floor, 1.0)
    X, S = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
    T = torch.tensor(t0, device="cuda", requires_grad=True)
    proj, loss, terms = sb.ops.ProjectAndLossFunction.apply(X, S, T, k, 1, floor)
    ((proj * r.cuda()).sum() + cu * loss + (terms * ct.cuda()).sum()).backward()
    # float64 on the kernel's routing
    X64, S64 = _leaf(x), _leaf(s)
    T64 = torch.tensor(float(T.detach()), dtype=torch.float64, requires_grad=True)
    fl = float(np.float32(floor))
    o = _softproj64(X64, S64, T64, None, idx, 1, fl)
    loss64, terms64 = _simp64(X64, S64, 1.0, idx1.long().cpu(), idx2.long().cpu(), _first_argmax(dist1.cpu()))
    L = (o["proj"] * r.double()).sum() + cu * loss64 + (terms64 * ct.double()).sum()
    gX, gS, gT, dd = torch.autograd.grad(L, [X64, S64, T64, o["d"]])
    bars = _Bars()
    # bars about 10x the largest error measured on an H100 over these cases
    bars.check("proj", proj, o["proj"].detach(), o["proj"].detach().abs().max(), 2e-6)   # fp32 softmax / weighted sum (<= 1.9e-7)
    bars.check("loss", loss, loss64.detach(), abs(float(loss64.detach())), 1e-6)         # fp32 means over up to 100k distances (<= 8e-8)
    bars.check("terms", terms, terms64.detach(), terms64.detach().abs().max(), 1e-6)
    # the projection backward plus the Chamfer backward's per-point sums (measured <= 9.5e-7)
    bars.check("grad ref", X.grad, gX, gX.abs().max(), 1e-5)
    bars.check("grad samp", S.grad, gS, gS.abs().max(), 1e-5)
    if clamped:
        assert float(T.grad) == 0.0 and float(gT) == 0.0
    else:
        bars.check("grad T", T.grad, gT, (dd * o["d"].detach() / o["s"].detach()).abs().sum() * 2 * abs(float(T64.detach())), 1e-6)   # (<= 2e-8)
    bars.done()


# ---------------------------------------------------------------------------------------------------- GPU: Chamfer backward
def _chamfer64(x1, x2, i1, i2, g1, g2):
    """float64 L = sum g1 |x1 - x2[i1]|^2 + sum g2 |x2 - x1[i2]|^2; returns (dL/dx1, dL/dx2, scale1, scale2) with the per-point sum
    of |terms| (own term + every term scattered onto the point) as scales."""
    b = x1.shape[0]
    X1, X2 = _leaf(x1), _leaf(x2)
    bi = torch.arange(b)[:, None]
    e1, e2 = X2[bi, i1], X1[bi, i2]
    L = (_sq(X1 - e1) * g1).sum() + (_sq(X2 - e2) * g2).sum()
    gx1, gx2, de1, de2 = torch.autograd.grad(L, [X1, X2, e1, e2])
    s1 = (de1.abs() + _abs_scatter(i2, de2, x1.shape[1])).max()     # own term = -dL/de
    s2 = (de2.abs() + _abs_scatter(i1, de1, x2.shape[1])).max()
    return gx1, gx2, s1, s2


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,hub", [(2, 256, 128, False), (2, 257, 128, False), (2, 256, 127, False),   # either side of the owner switch
                                       (1, 64, 5000, False), (1, 5000, 64, False),                      # warp per owner, multi-tile index list
                                       (3, 2049, 2047, False), (2, 6000, 70, False),
                                       (2, 3000, 200, True)])                                           # one xyz2 point nearest to all of xyz1
def test_chamfer_backward_vs_float64(sb, b, n, m, hub):
    g = _gen(b * 100 + n + m)
    x1 = torch.rand(b, n, 3, generator=g) - 0.5
    x2 = torch.rand(b, m, 3, generator=g) - 0.5
    if hub:
        x2[:, 0] = 0.0
        x1 = 1e-3 * torch.randn(b, n, 3, generator=g)
    g1, g2 = torch.randn(b, n, generator=g), torch.randn(b, m, generator=g)
    x1c, x2c = x1.cuda(), x2.cuda()
    _, i1, _, i2 = sb.ops.nn_distance_forward(x1c, x2c)
    if hub:
        assert int(i1.max()) == 0
    runs = [sb.ops.nn_distance_backward(x1c, x2c, g1.cuda(), i1, g2.cuda(), i2) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])   # deterministic: no atomics
    r1, r2, s1, s2 = _chamfer64(x1, x2, i1.long().cpu(), i2.long().cpu(), g1.double(), g2.double())
    bars = _Bars()
    # fp32 products and the per-owner sums in ascending index order: 1e-6 of the sum of |terms| (measured <= 7.5e-8 on an H100)
    bars.check("grad xyz1", runs[0][0], r1, s1, 1e-6)
    bars.check("grad xyz2", runs[0][1], r2, s2, 1e-6)
    bars.done()


@pytest.mark.gpu
@pytest.mark.parametrize("used", ["dist1", "dist2"])
def test_chamfer_module_with_one_output_used(sb, used):
    """ChamferDistance with one output unused: its upstream gradient arrives as zeros."""
    g = _gen(31)
    b, n, m = 3, 700, 1500
    x1, x2 = torch.rand(b, n, 3, generator=g) - 0.5, torch.rand(b, m, 3, generator=g) - 0.5
    w = torch.randn(b, n if used == "dist1" else m, generator=g)
    A, C = x1.cuda().requires_grad_(True), x2.cuda().requires_grad_(True)
    d1, d2 = sb.ChamferDistance()(A, C)
    ((d1 if used == "dist1" else d2) * w.cuda()).sum().backward()
    _, i1, _, i2 = sb.ops.nn_distance_forward(x1.cuda(), x2.cuda())
    z1, z2 = (w.double(), torch.zeros(b, m, dtype=torch.float64)) if used == "dist1" else (torch.zeros(b, n, dtype=torch.float64), w.double())
    r1, r2, s1, s2 = _chamfer64(x1, x2, i1.long().cpu(), i2.long().cpu(), z1, z2)
    bars = _Bars()
    bars.check("grad xyz1", A.grad, r1, s1, 1e-6)   # as above
    bars.check("grad xyz2", C.grad, r2, s2, 1e-6)
    bars.done()


@pytest.mark.gpu
def test_simplification_loss_tied_maximum_goes_to_first_index(sb):
    """Duplicated samples tied for max c12: the max term's gradient goes to the first of them, as argmax does."""
    g = _gen(41)
    b, n, m = 4, 1024, 64
    ref = torch.rand(b, n, 3, generator=g) - 0.5
    samp = ref[:, :m] + 0.05 * torch.randn(b, m, 3, generator=g)
    samp[:, 9] = samp[:, 30] = samp[:, 51] = torch.tensor([1.5, -1.5, 1.5])
    R, S = ref.cuda().requires_grad_(True), samp.cuda().requires_grad_(True)
    w21 = 1.3
    sb.ops.SimplificationLossFunction.apply(S, R, w21).backward()
    _, dist1, idx1, _, idx2 = sb.ops.simplification_loss_forward(samp.cuda(), ref.cuda(), w21)
    d = dist1.cpu()
    assert torch.equal(d[:, 9], d[:, 30]) and torch.equal(d[:, 9], d[:, 51]) and bool((d.argmax(1) == 9).all())
    R64, S64 = _leaf(ref), _leaf(samp)
    loss, _ = _simp64(R64, S64, w21, idx1.long().cpu(), idx2.long().cpu(), _first_argmax(d))
    gR, gS = torch.autograd.grad(loss, [R64, S64])
    bars = _Bars()
    # fp32 Chamfer backward against the tensor's max |value|; a max term at the wrong sample is an O(1) error (measured <= 1.4e-7)
    bars.check("grad samp", S.grad, gS, gS.abs().max(), 2e-6)
    bars.check("grad ref", R.grad, gR, gR.abs().max(), 2e-6)
    bars.done()


# ---------------------------------------------------------------------------------------------------- GPU: progressive loss
@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,sizes,dup", [
    (4, 1024, 1024, [2, 4, 8, 16, 32, 64, 128, 256, 512, 1024], False),
    (3, 500, 300, [7, 50, 299, 300], False),
    (32, 1024, 1024, [8, 16, 32, 64, 128, 256, 512, 1024], False),
    (4, 1024, 64, [2, 4, 8, 16, 32, 64], True),     # a duplicated outlier: the maximum from s = 4 on, tied from s = 16 on
])
def test_progressive_backward_vs_float64(sb, b, n, m, sizes, dup):
    """ProgressiveLossFunction (one forward launch, one Chamfer-backward launch over all prefixes) against the float64 per-prefix
    formula on the kernel's indices, each prefix's max term routed to the FIRST index attaining the running maximum."""
    from samplenet_b200 import trainers

    g = _gen(b + n + m)
    x = torch.rand(b, n, 3, generator=g) - 0.5
    s = torch.rand(b, m, 3, generator=g) - 0.5
    if dup:
        s[:, 3] = s[:, 10] = s[:, 40] = torch.tensor([1.5, 1.5, -1.5])
    weights = [1.0 + 0.01 * v for v in sizes]
    dist1, idx1, _, idx2, _ = sb.ops.progressive_loss_forward(x.cuda(), s.cuda(), sizes, weights)
    if dup:
        d = dist1.cpu()
        assert torch.equal(d[:, 3], d[:, 10]) and torch.equal(d[:, 3], d[:, 40])
    ct = torch.randn(len(sizes), 3, generator=g)
    X, S = x.cuda().requires_grad_(True), s.cuda().requires_grad_(True)
    total, terms = sb.ops.ProgressiveLossFunction.apply(S, X, sizes, weights)
    (0.8 * total + (terms * ct.cuda()).sum()).backward()
    X64, S64 = _leaf(x), _leaf(s)
    total64, terms64 = _progressive64(X64, S64, sizes, weights, idx1.long().cpu(), idx2.long().cpu(), dist1.cpu().double())
    gX, gS = torch.autograd.grad(0.8 * total64 + (terms64 * ct.double()).sum(), [X64, S64])
    bars = _Bars()
    bars.check("total", total, total64.detach(), abs(float(total64.detach())), 1e-6)   # fp32 means (measured <= 6.5e-8)
    # fp32 Chamfer backward over the concatenated prefix index sets, summed over up to 10 prefixes whose terms can cancel
    # (measured <= 1.1e-6 on an H100)
    bars.check("grad samp", S.grad, gS, gS.abs().max(), 1e-5)
    bars.check("grad ref", X.grad, gX, gX.abs().max(), 1e-5)
    bars.done()
    if dup:   # the one-pass and the per-prefix paths agree with a tied maximum too
        s1, s2 = s.cuda().requires_grad_(True), s.cuda().requires_grad_(True)
        trainers.progressive_simplification_loss(x.cuda(), s1, sizes, 1, 0.01, one_pass=True).backward()
        trainers.progressive_simplification_loss(x.cuda(), s2, sizes, 1, 0.01, one_pass=False).backward()
        err = float((s1.grad - s2.grad).abs().max())
        assert err <= 1e-5 * float(s2.grad.abs().max()), err   # as above


# ---------------------------------------------------------------------------------------------------- GPU: group_point_grad
@pytest.mark.gpu
@pytest.mark.parametrize("b,n,c,m,ns,kind", [(2, 300, 7, 40, 5, "plain"), (2, 1024, 3, 1024, 7, "plain"),   # m ns = 7168: four tiles
                                             (3, 100, 64, 512, 16, "hub"), (4, 1000, 3, 64, 1, "gather")])
@pytest.mark.parametrize("layout", ["bnc", "bcn"])
def test_group_point_grad_vs_float64(sb, b, n, c, m, ns, kind, layout):
    """group_point_grad (deterministic gather per source point) against float64 index_add, both layouts; 'gather' goes through
    gather_point as the FPS / random samplers do, 'hub' sends 3/4 of all indices to point 0."""
    g = _gen(b + n + c + m + ns)
    pts = torch.randn(b, n, c, generator=g)
    idx = torch.randint(0, n, (b, m, ns), generator=g)
    if kind == "hub":
        idx[torch.rand(b, m, ns, generator=g) < 0.75] = 0
    P = (pts if layout == "bnc" else pts.transpose(1, 2)).contiguous().cuda()
    go = torch.randn((b, m, ns, c) if layout == "bnc" else (b, c, m, ns), generator=g)
    if kind == "gather":
        go = go[..., 0, :] if layout == "bnc" else go[..., 0]
    runs = []
    for _ in range(2):
        Pl = P.clone().requires_grad_(True)
        if kind == "gather":
            out = sb.ops.gather_point(Pl, idx[..., 0].cuda(), layout)
        else:
            out = sb.ops.GroupPointFunction.apply(Pl, idx.to(torch.int32).cuda(), layout)
        assert out.shape == go.shape
        (out * go.cuda()).sum().backward()
        runs.append(Pl.grad)
    assert torch.equal(runs[0], runs[1])   # deterministic: no atomics
    go_bnc = go.double()
    if layout == "bcn":   # (b, c, m, ns) -> (b, m, ns, c), or (b, c, m) -> (b, m, c) for gather_point
        go_bnc = go_bnc.permute(0, 2, 3, 1) if kind != "gather" else go_bnc.permute(0, 2, 1)
    terms = go_bnc.reshape(b, m * ns, c)
    flat = idx.reshape(b, m * ns)
    ref = torch.zeros(b, n, c, dtype=torch.float64).scatter_add_(1, flat[..., None].expand(b, m * ns, c), terms)
    scale = _abs_scatter(flat, terms, n).max()
    bars = _Bars()
    bars.check("grad points", runs[0], _bnc(ref, layout), scale, 1e-6)   # fp32 sums in ascending index order (measured <= 1e-7)
    bars.done()
