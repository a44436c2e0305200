"""EMD kernels (csrc/emd.cu: approx_match, match_cost, match_cost_grad) against the C oracle, the exact-mode kernel and float64,
at the reconstruction autoencoder's batch sizes and on every branch of approx_match's launch plan.

The fast `approxmatch_kernel` is a persistent grid (two CTAs per SM) that cuts the b * nrows flat rows of each phase into one
chunk per CTA; a row is shared by S lanes, a chunk longer than a pass's row slots puts two rows on each slot (its own unrolled
loop and odd-column tail), and a chunk may straddle two clouds.  Which of these run depends on b, n, m and the SM count, so
`emd_plan` restates the launcher's plan and every case asserts the branches it is there to reach.

Yardsticks, each pinned here or elsewhere:
  - the C oracle (pinned against the reference's CPU code in test_oracle_pinning.py), run on a few sampled clouds of each
    batch -- the first, the last and one whose rows cross a CTA chunk boundary -- because it costs about a second per 2048^2
    cloud;
  - exact mode (approx_match(exact=True), one CTA per cloud), checked bit-exact against the oracle on those sampled clouds and
    then used as the reference for every cloud;
  - `_schedule64`, the ten-level schedule in float64 with the reference's arithmetic (levels 7 ... -2, level 0 at -2, the 1e-9
    terms, integer-division multipliers), pinned against the oracle by a CPU test below;
  - `_cost_grad64`, cost = sum match * |x1 - x2| and grad = sum match * d / max(|d|, 1e-10) in float64 on the kernel's own match.

Each bar is written at its comparison with the largest error measured over the cases on an H100 80GB HBM3 (SXM) at a 700 W
power limit; the bars are about 10x those maxima unless the comment there says otherwise.
"""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

EMD_THREADS, EMD_TILE, MC_SLABS = 512, 1024, 16     # csrc/emd.cu: kEmdThreads, kEmdTile, kMcSlabs


@pytest.fixture(scope="module")
def sb():
    import samplenet_b200

    samplenet_b200._lib.lib()  # fail loudly if the CUDA library is missing
    return samplenet_b200


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------- the launch plan
def _lane_counts(cn, S):
    """Columns each of the S lanes of a row takes from a tile of cn columns (j == lane mod S)."""
    return [(cn - l + S - 1) // S for l in range(min(S, cn))]


def emd_plan(b, n, m, sms, per_sm=2):
    """launch_approxmatch's grid and lanes per row, and what emd_row_pass does with them in each phase: phase 1 and 3 rows are
    xyz1 points over xyz2 columns, phase 2 the other way round.  Per phase: rows per CTA, whether any chunk takes the two-row
    branch and whether its odd-column tail runs, whether the single-row branch runs, the share of chunks that straddle two
    clouds, the column tiles, and a cloud whose rows cross a CTA chunk boundary."""
    rows = b * min(n, m)
    grid = per_sm * sms
    S = 1
    while S < 32 and rows * (S * 2) <= grid * EMD_THREADS // 2 and min(n, m) // (S * 2) >= 16:
        S *= 2
    grid = max(1, min(grid, (rows * S + 31) // 32))
    slots = EMD_THREADS // S
    plan = {"grid": grid, "S": S, "slots": slots,
            "multiL": 1 if n >= m else m // n, "multiR": n // m if n >= m else 1,
            "vec": n % 4 == 0, "empty_slabs": m < MC_SLABS}
    for phase, nrows, ncols in (("p1", n, m), ("p2", m, n)):
        total = b * nrows
        per = -(-total // grid)
        tiles = [min(EMD_TILE, ncols - c0) for c0 in range(0, ncols, EMD_TILE)]
        two = single = False
        chunks = crossing = 0
        for cta in range(grid):
            lo = min(total, per * cta)
            hi = min(total, lo + per)
            f0 = lo
            while f0 < hi:
                bi0 = f0 // nrows
                cap, split = min(hi, (bi0 + 2) * nrows), (bi0 + 1) * nrows
                t = cap - f0 > slots and cap <= split
                fend = min(cap, f0 + (2 if t else 1) * slots)
                two, single = two or t, single or not t
                chunks += 1
                crossing += fend > split
                f0 = fend
        cuts = [g * per for g in range(grid // 2, grid) if g * per < total and (g * per) % nrows]
        plan[phase] = {
            "per": per, "tiles": tiles, "two": two, "single": single, "cross": crossing / chunks,
            "two_tail": two and any(c % 2 for cn in tiles for c in _lane_counts(cn, S)),
            "cross_cloud": cuts[0] // nrows if cuts else None,
        }
    plan["p3"] = plan["p1"]     # phase 3 walks the rows of phase 1
    return plan


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# b, n, m, what the case is there for (a predicate on the plan, stated for the SM count of the device it runs on)
CASES = {
    "selfcheck_32x4096x1024": (32, 4096, 1024, lambda p: p["S"] == 2 and p["p1"]["two"] and p["p2"]["single"] and not p["p2"]["two"]
                               and p["p2"]["cross"] > 0 and p["multiR"] == 4 and len(p["p2"]["tiles"]) == 4),
    "ae_50x2048x2048": (50, 2048, 2048, lambda p: p["S"] == 1 and not p["p1"]["two"] and not p["p2"]["two"] and p["p1"]["cross"] > 0
                        and p["vec"]),
    "odd_72x2047x2047": (72, 2047, 2047, lambda p: p["S"] == 1 and p["p1"]["two_tail"] and p["p2"]["two_tail"]
                         and p["p1"]["tiles"][-1] == 1023 and not p["vec"]),
    "small_200x64x64": (200, 64, 64, lambda p: p["p1"]["cross"] > 0.5 and p["p2"]["cross"] > 0.5 and p["p1"]["per"] < p["slots"]),
    "thin_3x5000x13": (3, 5000, 13, lambda p: p["S"] == 1 and p["grid"] == 2 and p["p1"]["two_tail"] and p["multiR"] == 384
                       and p["empty_slabs"] and len(p["p2"]["tiles"]) == 5),
    "wide_7x999x3000": (7, 999, 3000, lambda p: p["S"] == 8 and p["multiL"] == 3 and p["p1"]["tiles"][-1] == 952),
    "dup_4x512x512": (4, 512, 512, lambda p: p["vec"]),
    "one_1x1x1": (1, 1, 1, lambda p: p["grid"] == 1 and p["S"] == 1),
    "one_2x1x700": (2, 1, 700, lambda p: p["grid"] == 1 and p["multiL"] == 700),
    "one_2x700x1": (2, 700, 1, lambda p: p["grid"] == 1 and p["multiR"] == 700),
}


def _clouds(name, device="cuda"):
    """Uniform clouds in the unit cube.  'dup': xyz2 is a permutation of xyz1, xyz1 holds exact duplicates (zero-distance pairs
    whose gradient term must be 0, not NaN) and one pair is 3e-11 apart, inside the 1e-10 clamp of the gradient's norm."""
    b, n, m, _ = CASES[name]
    g = _gen(sum(map(ord, name)))
    x1 = torch.rand(b, n, 3, generator=g)
    x2 = torch.rand(b, m, 3, generator=g)
    if name.startswith("dup"):
        x1[:, 256:320] = x1[:, :64]
        x1[:, 5] = 0.0
        x2 = x1[:, torch.randperm(n, generator=g)].clone()
        x2[:, (x2 == 0).all(2)[0].nonzero()[0, 0]] = torch.tensor([3e-11, 0.0, 0.0])
    return x1.to(device), x2.to(device)


# ---------------------------------------------------------------------------------------------------- float64 references
def _schedule64(x1, x2, chunk=1 << 25):
    """approx_match's ten-level schedule (tf_approxmatch_g.cu:21-160) in float64, on the device of the inputs: match (b, m, n)."""
    b, n, _ = x1.shape
    m = x2.shape[1]
    multiL, multiR = (1.0, float(n // m)) if n >= m else (float(m // n), 1.0)
    out = torch.empty(b, m, n, dtype=torch.float64, device=x1.device)
    step = max(1, chunk // (n * m))
    for s in range(0, b, step):
        a, c = x1[s:s + step].double(), x2[s:s + step].double()
        d = sum((a[:, :, None, i] - c[:, None, :, i]) ** 2 for i in range(3))              # (bs, n, m)
        remainL = torch.full(a.shape[:2], multiL, dtype=torch.float64, device=a.device)
        remainR = torch.full(c.shape[:2], multiR, dtype=torch.float64, device=a.device)
        match = torch.zeros_like(d)
        for j in range(7, -3, -1):
            level = 0.0 if j == -2 else -(4.0 ** j)
            e = torch.exp(level * d)
            ratioL = remainL / (1e-9 + (e * remainR[:, None, :]).sum(2))
            sumr = (e * ratioL[:, :, None]).sum(1) * remainR
            ratioR = torch.clamp(remainR / (sumr + 1e-9), max=1.0) * remainR
            remainR = torch.clamp(remainR - sumr, min=0.0)
            w = e * ratioL[:, :, None] * ratioR[:, None, :]
            match += w
            remainL = torch.clamp(remainL - w.sum(2), min=0.0)
        out[s:s + step] = match.transpose(1, 2)
    return out


def _cost_grad64(x1, x2, match, chunk=1 << 24):
    """cost (b,), grad1 (b, n, 3), grad2 (b, m, 3) in float64 from the fp32 inputs, and the per-point sums of |match| that scale
    the gradients: s1 (b, n) over xyz2, s2 (b, m) over xyz1."""
    b, n, _ = x1.shape
    m = x2.shape[1]
    dev = x1.device
    cost = torch.empty(b, dtype=torch.float64, device=dev)
    g1 = torch.empty(b, n, 3, dtype=torch.float64, device=dev)
    g2 = torch.empty(b, m, 3, dtype=torch.float64, device=dev)
    step = max(1, chunk // max(1, n * m))
    for s in range(0, b, step):
        a, c, w = x1[s:s + step].double(), x2[s:s + step].double(), match[s:s + step].double()
        d = [a[:, None, :, i] - c[:, :, None, i] for i in range(3)]                         # (bs, m, n): x1[k] - x2[l]
        r = torch.sqrt(d[0] ** 2 + d[1] ** 2 + d[2] ** 2)
        cost[s:s + step] = (w * r).sum((1, 2))
        inv = w / torch.clamp(r, min=1e-10)
        g1[s:s + step] = torch.stack([(di * inv).sum(1) for di in d], -1)
        g2[s:s + step] = -torch.stack([(di * inv).sum(2) for di in d], -1)
    absm = match.double().abs()
    return cost, g1, g2, absm.sum(1), absm.sum(2)


class _Bars:
    """Collects every comparison of a test, prints its error, and fails at the end with all of them."""

    def __init__(self, case):
        self.case, self.failed = case, []

    def check(self, what, err, bar):
        err = float(err)
        print("%-24s %-34s %.2e  (bar %.0e)" % (self.case, what, err, bar))
        if not err <= bar:
            self.failed.append("%s: %.3e > %.0e" % (what, err, bar))

    def done(self):
        assert not self.failed, "\n".join(self.failed)


def _rel(got, want, scale):
    """max over elements of |got - want| / scale (scale broadcast to the elements; 0 / 0 counts as 0)."""
    err = (got.double() - want).abs()
    scale = scale.double().expand_as(err)
    return float(torch.where(err == 0, torch.zeros_like(err), err / scale).max()) if err.numel() else 0.0


# ---------------------------------------------------------------------------------------------------- CPU: pin the yardsticks
@pytest.mark.parametrize("n,m", [(64, 64), (96, 32), (40, 120), (77, 77)])
def test_schedule64_equals_oracle(oracle, n, m):
    """The float64 schedule reproduces the oracle's fp32 match, its cost and its conservation.  The match bar is loose because the
    oracle runs the schedule in fp32: where a point's remaining mass runs towards zero, the next level's ratio divides rounding
    errors by it (measured <= 1.4e-4 absolute; the cost, a sum over the whole match, <= 4.1e-7 relative)."""
    g = _gen(n * 7 + m)
    x1, x2 = torch.rand(2, n, 3, generator=g), torch.rand(2, m, 3, generator=g)
    want = torch.from_numpy(oracle.approx_match(x1.numpy(), x2.numpy())).double()
    got = _schedule64(x1, x2)
    assert float((got - want).abs().max()) <= 1e-3
    cost = _cost_grad64(x1, x2, got)[0]
    ocost = torch.from_numpy(oracle.match_cost(x1.numpy(), x2.numpy(), want.float().numpy())).double()
    assert float(((cost - ocost).abs() / ocost).max()) <= 4e-6
    lo, hi = min(n, m), max(n, m)
    tot = got.sum(1) if n <= m else got.sum(2)
    assert float((tot - hi // lo).abs().max()) <= 1e-7 * (hi // lo)    # measured <= 1.5e-8


def test_cost_grad64_equals_oracle(oracle):
    """The written-out float64 cost and gradients equal the oracle's (double accumulators over fp32 terms) on a dense random
    match, including zero-distance pairs (term 0) and a pair inside the 1e-10 norm clamp (term match * d / 1e-10)."""
    g = _gen(5)
    x1, x2 = torch.rand(2, 50, 3, generator=g), torch.rand(2, 70, 3, generator=g)
    x2[:, 3] = x1[:, 7]
    x1[:, 0] = 0.0
    x2[:, 0] = torch.tensor([3e-11, 0.0, 0.0])
    match = torch.rand(2, 70, 50, generator=g)
    cost, g1, g2, s1, s2 = _cost_grad64(x1, x2, match)
    a, c, mt = x1.numpy(), x2.numpy(), match.numpy()
    oc = torch.from_numpy(oracle.match_cost(a, c, mt)).double()
    o1, o2 = (torch.from_numpy(t).double() for t in oracle.match_cost_grad(a, c, mt))
    assert _rel(cost, oc, cost) <= 1e-6
    assert _rel(o1, g1, s1[..., None]) <= 1e-6 and _rel(o2, g2, s2[..., None]) <= 1e-6
    assert torch.isfinite(g1).all() and torch.isfinite(g2).all()
    y1, y2 = x1.double().requires_grad_(True), x2.double().requires_grad_(True)    # the autograd graph has the same gradient
    a1, a2 = torch.autograd.grad(_cost64_graph(y1, y2, match).sum(), [y1, y2])
    assert _rel(a1, g1, s1[..., None]) <= 1e-12 and _rel(a2, g2, s2[..., None]) <= 1e-12
    # the clamped pair alone: (0 - 3e-11) / 1e-10 of its weight, on both sides
    lone = torch.zeros_like(match)
    lone[0, 0, 0] = 0.5
    _, g1, g2, _, _ = _cost_grad64(x1, x2, lone)
    o1, o2 = oracle.match_cost_grad(a, c, lone.numpy())
    for got in (g1[0, 0, 0], -g2[0, 0, 0], o1[0, 0, 0], -o2[0, 0, 0]):
        assert abs(float(got) + 0.15) <= 1e-6


def test_plan_at_132_sms():
    """The plan of each case on a 132-SM H100 SXM, as stated where the case list was chosen."""
    plans = {k: emd_plan(b, n, m, 132) for k, (b, n, m, _) in CASES.items()}
    for name, (b, n, m, reaches) in CASES.items():
        assert reaches(plans[name]), name
    p = plans["selfcheck_32x4096x1024"]
    assert p["grid"] == 264 and p["p1"]["per"] == 497 and p["p1"]["two"] and not p["p1"]["two_tail"]
    p = plans["ae_50x2048x2048"]
    assert p["grid"] == 264 and p["p1"]["per"] == 388
    p = plans["odd_72x2047x2047"]
    assert p["p1"]["two"] and p["p2"]["two"] and p["p1"]["per"] == 559
    assert plans["small_200x64x64"]["p1"]["per"] == 49
    p = plans["thin_3x5000x13"]
    assert p["p1"]["per"] == 7500 and p["p2"]["single"] and p["p2"]["tiles"][-1] == 904
    # the batch sizes of the other EMD tests (b <= 3, n <= 2048) never reach S = 1 or the two-row branch
    for b, n, m in [(1, 2048, 2048), (2, 1024, 1024), (3, 77, 77), (2, 300, 300), (2, 40, 120), (2, 96, 32)]:
        p = emd_plan(b, n, m, 132)
        assert p["S"] >= 2 and not p["p1"]["two"] and not p["p2"]["two"]


# ---------------------------------------------------------------------------------------------------- GPU: approx_match
def _sampled(plan, b):
    """The first and last cloud, and one whose rows cross a CTA chunk boundary."""
    cross = plan["p1"]["cross_cloud"]
    return sorted({0, b - 1} | ({cross} if cross is not None else set()))


def _oracle_clouds(oracle, x1, x2, clouds):
    """The oracle's match of the given clouds, one thread per cloud (the C call releases the GIL)."""
    a, c = x1.cpu().numpy(), x2.cpu().numpy()
    with ThreadPoolExecutor(len(clouds)) as ex:
        return list(ex.map(lambda i: oracle.approx_match(a[i:i + 1], c[i:i + 1])[0], clouds))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_approx_match_parity(sb, oracle, name):
    b, n, m, reaches = CASES[name]
    plan = emd_plan(b, n, m, _sms())
    assert reaches(plan), (name, plan)
    x1, x2 = _clouds(name)
    bars = _Bars(name)
    exact = sb.ops.approx_match(x1, x2, exact=True)
    fast = sb.ops.approx_match(x1, x2)
    assert fast.shape == exact.shape == (b, m, n)
    # exact mode is still the oracle's arithmetic at this size, so it can stand in for it on every cloud
    clouds = _sampled(plan, b)
    for i, want in zip(clouds, _oracle_clouds(oracle, x1, x2, clouds)):
        assert np.array_equal(exact[i].cpu().numpy(), want), (name, i)

    # the fast match against exact mode, every cloud: values, and the arg-max assignments wherever exact mode's top-2 gap exceeds
    # the value bar (as test_gpu_parity.py).  The bar is the reference's own GPU-vs-CPU threshold (approxmatch.cpp:222) at every
    # size, looser than test_gpu_parity.py's 2e-3 for n <= 300: ex2.approx and the blocked row sums are amplified by the schedule
    # wherever a point's remaining mass runs towards zero, and over the 200 clouds of the 64^2 case the worst one reaches 7.7e-3
    # (at most 3.4e-3 on the other cases).  That is the cloud's own arithmetic, not the batch's: the same cloud launched alone
    # is checked below.
    tol = 1e-2
    per_cloud = (fast - exact).abs().amax((1, 2))
    bars.check("fast - exact match", per_cloud.max(), tol)
    for dim in (1, 2):
        am, ao = fast.argmax(dim), exact.argmax(dim)
        gap = exact.gather(dim, ao.unsqueeze(dim)) - exact.gather(dim, am.unsqueeze(dim))
        bars.check("arg-max gap (dim %d)" % dim, gap.max(), tol)

    # per-cloud EMD cost of the fast match against the float64 schedule's own cost
    m64 = _schedule64(x1, x2)
    c64 = _cost_grad64(x1, x2, m64)[0]
    cf = _cost_grad64(x1, x2, fast)[0]
    # (measured <= 9.9e-5 for the fast match and 4.5e-5 for exact mode, both on the zero-distance case whose cost is near 0)
    bars.check("cost(fast) / cost(f64) - 1", ((cf - c64).abs() / c64).max(), 1e-3)
    bars.check("cost(exact) / cost(f64) - 1", ((_cost_grad64(x1, x2, exact)[0] - c64).abs() / c64).max(), 1e-3)

    # conservation: the smaller side fully assigned, no point over its mass, and the same per-point totals as float64, relative
    # to the point's mass (measured <= 5.8e-5, 1.2e-6 and 5.8e-5)
    lo = min(n, m)
    tot2, tot1 = fast.double().sum(2), fast.double().sum(1)     # per xyz2 point, per xyz1 point
    full = tot2 if n >= m else tot1
    bars.check("smaller side assigned", (full - max(n, m) // lo).abs().max() / (max(n, m) // lo), 6e-4)
    over = max(float((tot1 - plan["multiL"]).max()) / plan["multiL"], float((tot2 - plan["multiR"]).max()) / plan["multiR"])
    bars.check("over mass", max(over, 0.0), 1e-5)
    bars.check("totals vs float64", max(float((tot1 - m64.sum(1)).abs().max()) / plan["multiL"],
                                        float((tot2 - m64.sum(2)).abs().max()) / plan["multiR"]), 6e-4)

    # batch invariance: the crossing cloud and the cloud furthest from exact mode, each launched alone, where it takes another
    # grid and chunking and, at the large batches, another S (measured <= 2.8e-5)
    for i in sorted({clouds[len(clouds) // 2], int(per_cloud.argmax())}):
        alone = sb.ops.approx_match(x1[i:i + 1].contiguous(), x2[i:i + 1].contiguous())
        bars.check("cloud %d alone - in batch" % i, (alone[0] - fast[i]).abs().max(), 3e-4)
    # run to run: bit-identical
    assert torch.equal(sb.ops.approx_match(x1, x2), fast)
    assert torch.equal(sb.ops.approx_match(x1, x2, exact=True), exact)
    bars.done()


# ---------------------------------------------------------------------------------------------------- GPU: match_cost / grad
def _misaligned(match):
    """A copy of `match` 4 bytes past a 16-byte boundary: the kernels' scalar path although n % 4 == 0."""
    buf = torch.empty(match.numel() + 1, device=match.device)[1:].view(match.shape)
    buf.copy_(match)
    assert buf.data_ptr() % 16 == 4
    return buf


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_match_cost_and_grad_parity(sb, name):
    b, n, m, _ = CASES[name]
    x1, x2 = _clouds(name)
    bars = _Bars(name)
    own = sb.ops.approx_match(x1, x2)
    dense = torch.rand(b, m, n, generator=_gen(b + n + m), device="cpu").cuda()
    inputs = [("own", own), ("dense", dense)]
    if n % 4 == 0:
        inputs += [("own misaligned", _misaligned(own)), ("dense misaligned", _misaligned(dense))]
    for what, match in inputs:
        cost = sb.ops.match_cost_forward(x1, x2, match)
        g1, g2 = sb.ops.match_cost_grad(x1, x2, match)
        c64, w1, w2, s1, s2 = _cost_grad64(x1, x2, match)
        # fp32 terms summed in fp32 (measured <= 2.7e-7 for the cost and 4.4e-7 for the gradients, relative to the sum of |terms|)
        bars.check(what + " cost", _rel(cost, c64, c64), 3e-6)
        bars.check(what + " grad1", _rel(g1, w1, s1[..., None]), 5e-6)
        bars.check(what + " grad2", _rel(g2, w2, s2[..., None]), 5e-6)
        assert torch.equal(sb.ops.match_cost_forward(x1, x2, match), cost)
        r1, r2 = sb.ops.match_cost_grad(x1, x2, match)
        assert torch.equal(r1, g1) and torch.equal(r2, g2)
    bars.done()


# ---------------------------------------------------------------------------------------------------- GPU: autograd and trainer
def _cost64_graph(x1, x2, match):
    """float64 autograd graph of the written-out cost (b,) on a fixed match.  Below |d| = 1e-10 a pair's term is |d|^2 / 2e-10
    instead of |d| (at most 5e-11 of its weight): its gradient is then d / 1e-10, the kernels' clamped norm, and 0 at d = 0."""
    d = x1[:, None, :, :] - x2[:, :, None, :]
    d2 = (d * d).sum(-1)
    r = torch.where(d2 >= 1e-20, torch.sqrt(torch.clamp(d2, min=1e-20)), d2 / 2e-10)
    return (match.double() * r).sum((1, 2))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["dup_4x512x512", "thin_3x5000x13", "wide_7x999x3000"])
def test_match_cost_autograd(sb, name):
    """tf_ops.match_cost backward with the expanded (stride 0) upstream gradient of .mean() and with a weighted vector, against
    float64 autograd (measured <= 4.5e-8 for the loss and 3.4e-7 for the gradients, scaled as in the test above)."""
    b, n, m, _ = CASES[name]
    bars = _Bars(name)
    p1, p2 = _clouds(name)
    match = sb.tf_ops.approx_match(p1, p2)
    weights = torch.rand(b, generator=_gen(9)).cuda() - 0.3
    for what, reduce in (("mean", lambda c: c.mean()), ("weighted", lambda c: (c * weights).sum())):
        x1, x2 = p1.clone().requires_grad_(True), p2.clone().requires_grad_(True)
        loss = reduce(sb.tf_ops.match_cost(x1, x2, match))
        loss.backward()
        y1, y2 = p1.double().requires_grad_(True), p2.double().requires_grad_(True)
        ref = reduce(_cost64_graph(y1, y2, match))
        ref.backward()
        up = torch.full((b,), 1.0 / b, dtype=torch.float64, device="cuda") if what == "mean" else weights.double()
        absm = match.double().abs()
        bars.check(what + " loss", abs(float(loss) - float(ref)) / float(_cost64_graph(p1.double(), p2.double(), match).mul(up.abs()).sum()), 3e-6)
        bars.check(what + " grad xyz1", _rel(x1.grad, y1.grad, (absm.sum(1) * up.abs()[:, None])[..., None]), 5e-6)
        bars.check(what + " grad xyz2", _rel(x2.grad, y2.grad, (absm.sum(2) * up.abs()[:, None])[..., None]), 5e-6)
    bars.done()


@pytest.mark.gpu
def test_autoencoder_emd_loss_b50(sb):
    """trainers.autoencoder_loss(x, gt, "emd") at the reconstruction AE size (B = 50, 2048 points each): loss and both input
    gradients against float64 autograd of the written-out cost on the kernel's own match (approx_match has no gradient).
    Measured: 6.9e-8 for the loss, 3.9e-7 for the gradients."""
    from samplenet_b200 import trainers

    b, n = 50, 2048
    g = _gen(50)
    x0, gt0 = torch.rand(b, n, 3, generator=g).cuda(), torch.rand(b, n, 3, generator=g).cuda()
    x, gt = x0.clone().requires_grad_(True), gt0.clone().requires_grad_(True)
    loss = trainers.autoencoder_loss(x, gt, "emd")
    loss.backward()
    match = sb.tf_ops.approx_match(x0, gt0)
    bars = _Bars("ae_b50")
    y, ygt = x0.double().requires_grad_(True), gt0.double().requires_grad_(True)
    ref = 0.0
    for s in range(0, b, 10):   # ten clouds per graph keeps the float64 intermediates at a few GB
        part = _cost64_graph(y[s:s + 10], ygt[s:s + 10], match[s:s + 10]).sum() / b
        part.backward()
        ref += float(part)
    absm = match.double().abs() / b
    bars.check("loss", abs(float(loss) - ref) / ref, 3e-6)
    bars.check("grad x", _rel(x.grad, y.grad, absm.sum(1)[..., None]), 5e-6)
    bars.check("grad gt", _rel(gt.grad, ygt.grad, absm.sum(2)[..., None]), 5e-6)
    bars.done()


# ---------------------------------------------------------------------------------------------------- GPU: argument checks
@pytest.mark.gpu
def test_emd_argument_rejections(sb):
    """Shapes the kernels would read past are rejected with ValueError before anything is launched."""
    z = lambda *s: torch.zeros(*s, device="cuda")
    before = sb._lib.launch_count()
    bad_clouds = [(z(3, 8, 3), z(2, 5, 3)), (z(8, 3), z(5, 3)), (z(3, 8, 2), z(3, 5, 3)), (z(3, 8, 3), z(3, 5, 4)),
                  (z(1, 3, 8, 3), z(1, 3, 5, 3))]
    for a, c in bad_clouds:
        with pytest.raises(ValueError, match="ApproxMatch expects"):
            sb.ops.approx_match(a, c)
        with pytest.raises(ValueError, match="MatchCost expects"):
            sb.ops.match_cost_forward(a, c, z(3, 5, 8))
        with pytest.raises(ValueError, match="MatchCost expects"):
            sb.ops.match_cost_grad(a, c, z(3, 5, 8))
    a, c = z(3, 8, 3), z(3, 5, 3)
    for mt in (z(3, 8, 5), z(2, 5, 8), z(3, 5, 8, 1), z(15, 8), z(3, 5, 9)):
        for fn in (sb.ops.match_cost_forward, sb.ops.match_cost_grad):
            with pytest.raises(ValueError, match="match shape"):
                fn(a, c, mt)
    assert sb._lib.launch_count() == before


@pytest.mark.gpu
def test_emd_empty_batch(sb):
    """b = 0: empty results and no launch."""
    z = lambda *s: torch.zeros(*s, device="cuda")
    before = sb._lib.launch_count()
    for exact in (False, True):
        assert sb.ops.approx_match(z(0, 7, 3), z(0, 5, 3), exact=exact).shape == (0, 5, 7)
    assert sb.ops.match_cost_forward(z(0, 7, 3), z(0, 5, 3), z(0, 5, 7)).shape == (0,)
    g1, g2 = sb.ops.match_cost_grad(z(0, 7, 3), z(0, 5, 3), z(0, 5, 7))
    assert g1.shape == (0, 7, 3) and g2.shape == (0, 5, 3)
    assert sb._lib.launch_count() == before
