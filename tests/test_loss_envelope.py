"""The three simplification-loss entries across their launch plans: the fused projection + loss tail (csrc/tail.cu,
snb200_project_and_loss_forward), the progressive loss over every prefix (csrc/progressive.cu, snb200_progressive_loss_forward) and the
separate Chamfer + one-CTA reduction (csrc/chamfer.cu, snb200_simplification_loss_forward).

Each case names the branch of its entry's planner it is there for, and asserts it through the plan entries of
include/samplenet_b200_debug.h, so a planner change cannot move a case off its branch silently.  The planners assume a fixed 132 SMs: a
plan does not depend on the device, and the CPU tests pin every case's branch and the plans' agreement with the workspace queries.

GPU checks:
  * indices and distances bit-exact against the C oracle (on a spread of clouds where the whole batch would take the oracle seconds) and
    bit-identical to the stand-alone routes (knn_soft_project_forward, nn_distance_forward, one nn_distance per prefix), in both
    arithmetic modes;
  * forward values and gradients against float64 on the kernels' own routing, with the bars of test_backward_parity.py (each written at
    its comparison);
  * batch invariance, run-to-run repeats with the ticket word back at zero, inputs 4 bytes off 16-byte alignment, and write sets.
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_backward_parity as tbp  # noqa: E402
import test_write_sets as tws  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W21 = 1.3                          # weight of the input -> sample term (a value other than 1 checks the multiply)
W21_32 = float(np.float32(W21))    # what the kernels receive
ORACLE_OPS = 6e8                   # oracle work per call (pairs x (k + 1) for the kNN) above which it sees a spread of clouds only
ORACLE_PAIRS = 3e8                 # (query, candidate) pairs above which the Chamfer-only checks leave the oracle out


@pytest.fixture(scope="module")
def sb():
    import __graft_entry__ as ge

    ge.build()
    import samplenet_b200

    return samplenet_b200


# ---------------------------------------------------------------------------------------------------- plans
def tail_plan(sb, b, n_ref, n_samp):
    v = [ctypes.c_int() for _ in range(7)]
    sb._lib.check(sb._lib.lib().snb200_debug_project_and_loss_plan(b, n_ref, n_samp, *[ctypes.byref(t) for t in v]), "debug_project_and_loss_plan")
    p = dict(zip(("knn_ctas", "s1", "tiles1", "ntiles", "smem_floats", "cap_clouds", "tma"), (t.value for t in v)))
    p["passes"] = -(-b // p["cap_clouds"])
    p["partial_cta"] = n_samp % 8 != 0           # the last projection CTA has idle warps
    p["scalar_samp"] = n_samp % 4 != 0           # the direction-1 role stages the samples with the scalar loop
    p["register_knn"] = n_ref <= 1024            # the kNN keeps a lane's 32 distances in registers
    return p


def prog_plan(sb, b, n, m):
    v = [ctypes.c_int() for _ in range(5)]
    sb._lib.check(sb._lib.lib().snb200_debug_progressive_loss_plan(b, n, m, *[ctypes.byref(t) for t in v]), "debug_progressive_loss_plan")
    p = dict(zip(("s_a", "tiles_a", "s2", "tiles2", "cl_batch"), (t.value for t in v)))
    p["passes"] = -(-b // p["cl_batch"])
    p["last_pass"] = b - (p["passes"] - 1) * p["cl_batch"]   # clouds in the final reduction's last staging pass
    p["cand_tiles"] = -(-n // 4096)              # role A's candidate tiles
    p["scalar_samp"] = m % 4 != 0                # role B stages the samples with the scalar loop
    return p


def reduce_threads(sb, b):
    t = ctypes.c_int()
    sb._lib.check(sb._lib.lib().snb200_debug_simplification_loss_plan(b, ctypes.byref(t)), "debug_simplification_loss_plan")
    return t.value


def _check_branch(plan, expect, what):
    got = {k: plan[k] for k in expect}
    assert got == expect, (what, plan)


# (b, n_ref, n_samp, k, branch)
TAIL_CASES = [
    pytest.param(1, 1, 1, 1, dict(tma=0, passes=1, partial_cta=True), id="1x1x1-k1"),
    pytest.param(1, 32, 1, 32, dict(tma=1, knn_ctas=1, partial_cta=True), id="1x32x1-k32"),
    pytest.param(2, 1024, 63, 8, dict(partial_cta=True, scalar_samp=True, tma=1, register_knn=True), id="2x1024x63-partial-cta"),
    pytest.param(3, 1025, 65, 16, dict(register_knn=False, tma=0, scalar_samp=True), id="3x1025x65-generic-knn"),
    pytest.param(32, 1024, 64, 8, dict(passes=1, tma=1, partial_cta=False), id="32x1024x64-headline"),
    pytest.param(50, 2048, 64, 16, dict(passes=1, register_knn=False), id="50x2048x64-rec"),
    pytest.param(154, 1024, 64, 8, dict(cap_clouds=153, passes=2), id="154x1024x64-two-passes"),
    pytest.param(2048, 1024, 64, 8, dict(cap_clouds=153, passes=14), id="2048x1024x64-saturated"),
    pytest.param(12, 8, 4096, 8, dict(ntiles=513, s1=32, cap_clouds=11, passes=2), id="12x8x4096-513-slots"),
    pytest.param(9, 4096, 4096, 32, dict(tma=1, passes=1, ntiles=528), id="9x4096x4096-k32"),
    pytest.param(5, 4095, 4095, 7, dict(tma=0, partial_cta=True, scalar_samp=True), id="5x4095x4095-ragged"),
    pytest.param(1, 4096, 1, 1, dict(tma=1, knn_ctas=1), id="1x4096x1-k1"),
]

_FIB = [1, 2, 3, 5, 8, 13, 21, 34, 55, 89, 144, 233, 377, 610, 987, 1500]
# (b, n, m, sizes, duplicated outlier at (j, j + 1) -- j + 1 a prefix boundary -- or None, branch)
PROG_CASES = [
    pytest.param(1, 1, 1, [1], None, dict(passes=1, cand_tiles=1), id="1x1x1"),
    pytest.param(1, 33, 31, list(range(1, 17)), None, dict(scalar_samp=True), id="1x33x31-16-prefixes"),
    pytest.param(9, 1024, 1024, [2 ** i for i in range(1, 11)], None, dict(cl_batch=8, passes=2, last_pass=1), id="9x1024x1024-second-pass"),
    pytest.param(32, 1024, 1022, [2 ** i for i in range(1, 10)] + [1022], 63, dict(scalar_samp=True, cl_batch=8), id="32x1024x1022-scalar-staging"),
    pytest.param(50, 2048, 2048, [2 ** i for i in range(4, 12)], None, dict(cl_batch=5, passes=10), id="50x2048x2048-rec"),
    pytest.param(3, 5000, 4096, [1, 7, 4095, 4096], None, dict(cand_tiles=2, cl_batch=2), id="3x5000x4096-two-tiles"),
    pytest.param(2, 4097, 1531, _FIB, 376, dict(cand_tiles=2, scalar_samp=True), id="2x4097x1531-last-prefix-below-m"),
    pytest.param(64, 1024, 4096, [4, 16, 64, 256, 1024, 2048, 3001, 4096], None, dict(s_a=1, passes=32), id="64x1024x4096-32-passes"),
]

# (b, n_ref, n_samp, reduce threads)
SIMP_CASES = [
    pytest.param(1, 1, 1, 32, id="1x1x1"),
    pytest.param(31, 1024, 64, 992, id="31x1024x64-31-warps"),
    pytest.param(33, 1024, 64, 1024, id="33x1024x64-warps-loop"),
    pytest.param(5, 1023, 77, 160, id="5x1023x77-scalar-sums"),
    pytest.param(2048, 1024, 64, 1024, id="2048x1024x64"),
    pytest.param(50, 2048, 2048, 1024, id="50x2048x2048-rec"),
]


# ---------------------------------------------------------------------------------------------------- CPU: the plan entries
def test_plan_entries_answer_without_a_device(sb):
    """The three plan entries are declared in the debug header, bound in the ctypes table, and answer in a process that sees no CUDA
    device, the same as here; they reject bad sizes."""
    hdr = open(os.path.join(ROOT, "include", "samplenet_b200_debug.h")).read()
    for name in ("snb200_debug_project_and_loss_plan", "snb200_debug_progressive_loss_plan", "snb200_debug_simplification_loss_plan"):
        assert "int %s(" % name in hdr and name in sb._lib.exported_symbols(), name
    script = ("import ctypes, importlib.util, json, sys\n"
              "spec = importlib.util.spec_from_file_location('l', sys.argv[1]); m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)\n"
              "L = m.lib(); v = [ctypes.c_int() for _ in range(7)]; w = [ctypes.c_int() for _ in range(5)]; t = ctypes.c_int()\n"
              "r = [L.snb200_debug_project_and_loss_plan(2048, 1024, 64, *[ctypes.byref(x) for x in v]),\n"
              "     L.snb200_debug_progressive_loss_plan(50, 2048, 2048, *[ctypes.byref(x) for x in w]),\n"
              "     L.snb200_debug_simplification_loss_plan(33, ctypes.byref(t))]\n"
              "print(json.dumps([r, [x.value for x in v], [x.value for x in w], t.value]))\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", script, os.path.join(ROOT, "samplenet_b200", "_lib.py")], env=env, capture_output=True, text=True,
                         timeout=120)
    assert out.returncode == 0, out.stderr
    rc, tv, pv, threads = json.loads(out.stdout.strip().splitlines()[-1])
    assert rc == [0, 0, 0]
    tp, pp = tail_plan(sb, 2048, 1024, 64), prog_plan(sb, 50, 2048, 2048)
    assert tv == [tp[k] for k in ("knn_ctas", "s1", "tiles1", "ntiles", "smem_floats", "cap_clouds", "tma")]
    assert pv == [pp[k] for k in ("s_a", "tiles_a", "s2", "tiles2", "cl_batch")] and threads == reduce_threads(sb, 33) == 1024
    L, o = sb._lib.lib(), ctypes.c_int()
    assert L.snb200_debug_project_and_loss_plan(0, 1024, 64, *[ctypes.byref(o)] * 7) == -1
    assert L.snb200_debug_project_and_loss_plan(1, 1024, 64, *([ctypes.byref(o)] * 6 + [None])) == -1
    assert L.snb200_debug_progressive_loss_plan(1, 0, 64, *[ctypes.byref(o)] * 5) == -1
    assert L.snb200_debug_simplification_loss_plan(0, ctypes.byref(o)) == -1
    assert L.snb200_debug_simplification_loss_plan(1, None) == -1


def test_plans_agree_with_the_workspace_queries(sb):
    """Over a sweep of shapes: the tail's partial slots per cloud are knn_ctas + tiles1 and fill its workspace exactly, the final
    reduction's staged clouds fit its shared memory, the progressive loss's partials fit its workspace, and the reduction launch has one
    warp per cloud up to 1024 threads."""
    L = sb._lib.lib()
    for b in (1, 2, 3, 31, 32, 33, 153, 154, 1000, 2048, 65535):
        for n_ref in (1, 7, 32, 1023, 1024, 1025, 2048, 4095, 4096):
            for n_samp in (1, 8, 63, 64, 65, 1024, 4095, 4096):
                p = tail_plan(sb, b, n_ref, n_samp)
                assert p["knn_ctas"] == -(-n_samp // 8) and p["ntiles"] == p["knn_ctas"] + p["tiles1"], (b, n_ref, n_samp, p)
                assert int(L.snb200_project_and_loss_workspace_bytes(b, n_samp, n_ref)) == b * p["ntiles"] * 2 * 4, (b, n_ref, n_samp, p)
                assert p["s1"] in (1, 2, 4, 8, 16, 32) and p["tiles1"] == -(-n_ref // (256 // p["s1"] * 2)), (b, n_ref, n_samp, p)
                assert p["smem_floats"] == max(1024, 3 * max(n_ref, n_samp))
                assert p["cap_clouds"] == max(1, p["smem_floats"] // 2 // p["ntiles"]) and p["tma"] == (n_ref % 4 == 0)
        assert reduce_threads(sb, b) == min(1024, 32 * b)
    for b in (1, 2, 9, 50, 64, 1000):
        for n in (1, 33, 1024, 4096, 4097, 9000):
            for m in (1, 31, 1022, 2048, 4096):
                p = prog_plan(sb, b, n, m)
                assert p["tiles2"] == -(-n // (256 // p["s2"])) and p["s2"] in (1, 2, 4, 8, 16, 32), (b, n, m, p)
                assert 1 <= p["cl_batch"] <= 8 and (p["cl_batch"] == 1 or 64 + p["cl_batch"] * m <= 12 * 1024), (b, n, m, p)
                for npf in (1, 16):
                    assert b * p["tiles2"] * npf * 4 <= int(L.snb200_progressive_loss_workspace_bytes(b, n, m, npf)), (b, n, m, p)


def test_cases_reach_their_branches(sb):
    """Every GPU case of this file is on the branch it names (also asserted by the case itself on the GPU)."""
    for p in TAIL_CASES:
        b, n, m, k, expect = p.values
        _check_branch(tail_plan(sb, b, n, m), expect, p.id)
    for p in PROG_CASES:
        b, n, m, sizes, dup, expect = p.values
        _check_branch(prog_plan(sb, b, n, m), expect, p.id)
        assert len(sizes) <= 16 and sizes == sorted(set(sizes)) and sizes[-1] <= m
        assert dup is None or dup + 1 in sizes
    for p in SIMP_CASES:
        b, n, m, threads = p.values
        assert reduce_threads(sb, b) == threads, p.id
    # direction 1's lanes per query change with the batch: the batch-invariance test compares different merges
    assert tail_plan(sb, 1, 1024, 64)["s1"] != tail_plan(sb, 2048, 1024, 64)["s1"]
    assert prog_plan(sb, 1, 1024, 4096)["s_a"] != prog_plan(sb, 64, 1024, 4096)["s_a"]


# ---------------------------------------------------------------------------------------------------- helpers
def _oracle_clouds(b, ops_per_cloud):
    """Clouds the oracle checks: all of them when that is cheap, else an even spread that keeps the first and the last."""
    count = max(2, int(ORACLE_OPS // max(ops_per_cloud, 1)))
    if count >= b:
        return list(range(b))
    return sorted(set(np.linspace(0, b - 1, count).round().astype(int).tolist()))


def _np(t):
    return t.detach().cpu().numpy()


def _tail_clouds(seed, b, n, m, outlier=None):
    """Input cloud uniform in the unit cube; samples near input points (with replacement when m > n); outlier = (j1, j2): two samples
    at the same far point, tied for the largest c12."""
    g = tbp._gen(seed)
    x = torch.rand(b, n, 3, generator=g) - 0.5
    pick = torch.randperm(n, generator=g)[:m] if m <= n else torch.randint(0, n, (m,), generator=g)
    s = x[:, pick] + 0.02 * torch.randn(b, m, 3, generator=g)
    if outlier is not None:
        s[:, outlier[0]] = s[:, outlier[1]] = torch.tensor([1.5, -1.5, 1.5])
    return x.cuda(), s.cuda()


def _tail(sb, x, s, k, t0, mode, floor, unfused):
    names = ("proj", "idx", "weights", "dist", "dist1", "idx1", "dist2", "idx2", "out4")
    out = sb.ops.project_and_loss_forward(x, s, k, torch.tensor([t0], device="cuda"), mode, floor, W21, unfused=unfused)
    return dict(zip(names, out))


def _tail_exact(sb, oracle, out, x, s, k, t0, mode, floor, unfused):
    """Indices and distances bit-exact against the oracle and the stand-alone routes; proj, weights and dist_over_sigma bit-identical
    to knn_soft_project_forward's."""
    b, n, m = x.shape[0], x.shape[1], s.shape[1]
    sel = _oracle_clouds(b, n * m * (k + 1))
    xs, ss = _np(x)[sel], _np(s)[sel]
    _, oi = oracle.knn_point(k, xs, ss, contract=not unfused, tie_mode=1)
    assert np.array_equal(_np(out["idx"])[sel], oi), "knn_idx vs oracle"
    od1, oi1, od2, oi2 = oracle.nn_distance(ss, xs, contract=not unfused)
    for key, want in (("dist1", od1), ("idx1", oi1), ("dist2", od2), ("idx2", oi2)):
        assert np.array_equal(_np(out[key])[sel], want), key + " vs oracle"
    o = sb.ops.knn_soft_project_forward(x, s, k, "bnc", sigma=torch.tensor([t0], device="cuda"), want=("proj", "idx", "weights", "dist"),
                                        unfused=unfused, sigma_mode=mode, sigma_floor=floor)
    for key in ("proj", "idx", "weights", "dist"):
        assert torch.equal(out[key], o[key]), key + " vs knn_soft_project_forward"
    d1, i1, d2, i2 = sb.ops.nn_distance_forward(s, x, unfused=unfused)
    for key, want in (("dist1", d1), ("idx1", i1), ("dist2", d2), ("idx2", i2)):
        assert torch.equal(out[key], want), key + " vs nn_distance_forward"


def _tail_values(bars, out, x, s, mode, floor, tag):
    """proj and out4 against float64 on the kernel's routing."""
    X64, S64 = tbp._cpu64(x), tbp._cpu64(s)
    T64 = torch.tensor(float(np.float32(out["t0"])), dtype=torch.float64)
    o = tbp._softproj64(X64, S64, T64, None, out["idx"].long().cpu(), mode, float(np.float32(floor)))
    # fp32 softmax and weighted sums (bar of test_backward_parity; measured <= 2.3e-7)
    bars.check(tag + " proj", out["proj"], o["proj"], o["proj"].abs().max(), 2e-6)
    loss64, terms64 = tbp._simp64(X64, S64, W21_32, out["idx1"].long().cpu(), out["idx2"].long().cpu(), tbp._first_argmax(out["dist1"].cpu()))
    # fp32 sums over up to 2M distances in a fixed order (measured <= 1.4e-7)
    bars.check(tag + " loss", out["out4"][3], loss64, abs(float(loss64)), 1e-6)
    bars.check(tag + " terms", out["out4"][:3], terms64, terms64.abs().max(), 1e-6)


def _tail_backward(sb, bars, x, s, k, t0, mode, floor, seed, tag="", still=()):
    """ProjectAndLossFunction backward (soft-projection backward + Chamfer backward) against float64 autograd on the kernel's routing,
    with an upstream gradient on proj (except on the samples `still`), the loss and all three terms."""
    b, m = s.shape[0], s.shape[1]
    g = tbp._gen(seed)
    r = torch.randn(b, m, 3, generator=g)
    r[:, list(still)] = 0.0
    cu, ct = 0.7, torch.tensor([0.3, -1.1, 0.5])
    X, S = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
    T = torch.tensor(t0, device="cuda", requires_grad=True)
    proj, loss, terms = sb.ops.ProjectAndLossFunction.apply(X, S, T, k, mode, floor)
    ((proj * r.cuda()).sum() + cu * loss + (terms * ct.cuda()).sum()).backward()
    fwd = sb.ops.project_and_loss_forward(x, s, k, torch.tensor([t0], device="cuda"), mode, floor, 1.0)
    idx, dist1, idx1, idx2 = fwd[1].long().cpu(), fwd[4].cpu(), fwd[5].long().cpu(), fwd[7].long().cpu()
    X64, S64 = tbp._leaf(x), tbp._leaf(s)
    T64 = torch.tensor(float(T.detach()), dtype=torch.float64, requires_grad=True)
    fl = float(np.float32(floor))
    o = tbp._softproj64(X64, S64, T64, None, idx, mode, fl)
    loss64, terms64 = tbp._simp64(X64, S64, 1.0, idx1, idx2, tbp._first_argmax(dist1))
    L = (o["proj"] * r.double()).sum() + cu * loss64 + (terms64 * ct.double()).sum()
    gX, gS, gT, dd = torch.autograd.grad(L, [X64, S64, T64, o["d"]])
    # the projection backward plus the Chamfer backward's per-point sums (bars of test_backward_parity; measured <= 2.7e-6 over this file's
    # tail cases on an H100 at 700 W, the sums over up to 2048 clouds and 4096-point clouds included)
    bars.check(tag + "grad ref", X.grad, gX, gX.abs().max(), 1e-5)
    bars.check(tag + "grad samp", S.grad, gS, gS.abs().max(), 1e-5)
    tv = float(T64.detach())
    clamped = (mode == 1 and tv * tv <= fl) or (mode == 3 and tv <= fl)
    if clamped:   # sigma is the floor: the temperature gets exactly nothing
        assert float(T.grad) == 0.0 and float(gT) == 0.0, float(T.grad)
    else:
        dsdt = 1.0 if mode == 0 else 2.0 * abs(tv)
        bars.check(tag + "grad T", T.grad, gT, (dd * o["d"].detach() / o["s"].detach()).abs().sum() * dsdt, 1e-6)
    return dist1


def _sigma(sb, x, s, k):
    """sigma = the largest squared neighbour distance / 10, so that d / sigma <= 10 (tbp._knn)."""
    return tbp._knn(sb, x, s, k, "bnc")[1]


# ---------------------------------------------------------------------------------------------------- GPU: fused tail
@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,k,expect", TAIL_CASES)
def test_tail_vs_oracle_and_float64(sb, oracle, b, n, m, k, expect):
    _check_branch(tail_plan(sb, b, n, m), expect, (b, n, m))
    seed = b + n + m + k
    x, s = _tail_clouds(seed, b, n, m)
    t0, floor = tbp._temperature(1, _sigma(sb, x, s, k))
    bars = tbp._Bars()
    for unfused in (False, True):
        out = _tail(sb, x, s, k, t0, 1, floor, unfused)
        out["t0"] = t0
        _tail_exact(sb, oracle, out, x, s, k, t0, 1, floor, unfused)
        _tail_values(bars, out, x, s, 1, floor, "unfused" if unfused else "fma")
    _tail_backward(sb, bars, x, s, k, t0, 1, floor, seed)
    bars.done()


# sigma mode (0 sigma itself, 1 max(T^2, floor), 2 T^2, 3 max(T, floor)^2), floor active, negative temperature
SIGMA_MODES = [(0, False, False), (1, True, False), (2, False, True), (3, False, False), (3, True, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,k", [(2, 1024, 63, 8), (3, 1025, 65, 16), (12, 8, 4096, 8)])
@pytest.mark.parametrize("mode,clamped,negative", SIGMA_MODES)
def test_tail_sigma_modes(sb, oracle, b, n, m, k, mode, clamped, negative):
    """Every sigma mode, with the floor active and not, through the same launch: the projection outputs bit-identical to the stand-alone
    projection's, values and gradients (the temperature's exactly 0 under the floor) against float64."""
    seed = 7 * b + n + m + mode
    x, s = _tail_clouds(seed, b, n, m)
    t0, floor = tbp._temperature(mode, _sigma(sb, x, s, k), clamped=clamped, negative=negative)
    bars = tbp._Bars()
    out = _tail(sb, x, s, k, t0, mode, floor, False)
    out["t0"] = t0
    _tail_exact(sb, oracle, out, x, s, k, t0, mode, floor, False)
    _tail_values(bars, out, x, s, mode, floor, "mode %d" % mode)
    _tail_backward(sb, bars, x, s, k, t0, mode, floor, seed)
    bars.done()


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,k", [(32, 1024, 64, 8), (2, 1024, 63, 8), (12, 8, 4096, 8)])
def test_tail_tied_maximum_goes_to_first_index(sb, oracle, b, n, m, k):
    """Two samples at one far point tie for the largest c12, the second in another projection CTA (the last one): the max term and its
    gradient go to the first, as argmax does.  The two carry no upstream gradient on their projection: their neighbours lie 2 to 3 units
    away at d / sigma near 10, and the cancelling terms of that softmax gradient (measured 6.5e-6 of max |grad samp| on an H100) would set
    the error scale instead of the routing this test is about."""
    j1, j2 = 9, m - 1
    x, s = _tail_clouds(b + m, b, n, m, outlier=(j1, j2))
    t0, floor = tbp._temperature(1, _sigma(sb, x, s, k))
    bars = tbp._Bars()
    out = _tail(sb, x, s, k, t0, 1, floor, False)
    out["t0"] = t0
    _tail_exact(sb, oracle, out, x, s, k, t0, 1, floor, False)
    d = out["dist1"].cpu()
    assert torch.equal(d[:, j1], d[:, j2]) and bool((d.argmax(1) == j1).all())
    _tail_values(bars, out, x, s, 1, floor, "tied")
    _tail_backward(sb, bars, x, s, k, t0, 1, floor, b + m, still=(j1, j2))
    bars.done()


# ---------------------------------------------------------------------------------------------------- GPU: progressive loss
def _prog_clouds(seed, b, n, m, dup):
    g = tbp._gen(seed)
    x = torch.rand(b, n, 3, generator=g) - 0.5
    s = torch.rand(b, m, 3, generator=g) - 0.5
    if dup is not None:   # the maximum of the prefix ending at dup + 1, tied with the first sample of the next prefix
        s[:, dup] = s[:, dup + 1] = torch.tensor([1.5, 1.5, -1.5])
    return x.cuda(), s.cuda()


def _weights(sizes):
    return [1.0 + 0.01 * v for v in sizes]


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,sizes,dup,expect", PROG_CASES)
def test_progressive_vs_oracle_and_float64(sb, oracle, b, n, m, sizes, dup, expect):
    _check_branch(prog_plan(sb, b, n, m), expect, (b, n, m))
    seed = b + n + m + len(sizes)
    x, s = _prog_clouds(seed, b, n, m, dup)
    w = _weights(sizes)
    w32 = [float(np.float32(v)) for v in w]
    npf = len(sizes)
    bars = tbp._Bars()
    X64, S64 = tbp._cpu64(x), tbp._cpu64(s)
    use_oracle = b * n * (m + sum(sizes)) <= ORACLE_PAIRS
    for unfused in (False, True):
        tag = "unfused" if unfused else "fma"
        d1, i1, d2, i2, terms = sb.ops.progressive_loss_forward(x, s, sizes, w, unfused=unfused)
        e1, j1, _, _ = sb.ops.nn_distance_forward(s, x, unfused=unfused)
        assert torch.equal(d1, e1) and torch.equal(i1, j1), tag + " dist1 / idx1 vs nn_distance_forward"
        if use_oracle:
            od1, oi1, _, _ = oracle.nn_distance(_np(s), _np(x), contract=not unfused)
            assert np.array_equal(_np(d1), od1) and np.array_equal(_np(i1), oi1), tag + " dist1 / idx1 vs oracle"
        for p, sz in enumerate(sizes):
            _, _, e2, j2 = sb.ops.nn_distance_forward(s[:, :sz].contiguous(), x, unfused=unfused)
            assert torch.equal(d2[:, p], e2) and torch.equal(i2[:, p], j2), "%s prefix %d: dist2 / idx2 vs nn_distance_forward" % (tag, sz)
            if use_oracle:
                _, _, od2, oi2 = oracle.nn_distance(_np(s)[:, :sz], _np(x), contract=not unfused)
                assert np.array_equal(_np(d2[:, p]), od2) and np.array_equal(_np(i2[:, p]), oi2), "%s prefix %d vs oracle" % (tag, sz)
        if dup is not None:
            dd = d1.cpu()
            assert torch.equal(dd[:, dup], dd[:, dup + 1]) and bool((dd.argmax(1) == dup).all())
        total64, terms64 = tbp._progressive64(X64, S64, sizes, w32, i1.long().cpu(), i2.long().cpu(), d1.cpu().double())
        # fp32 means in a fixed order (bars of test_backward_parity; measured <= 2.2e-7)
        bars.check(tag + " total", terms[3 * npf], total64, abs(float(total64)), 1e-6)
        bars.check(tag + " terms", terms[:3 * npf].view(npf, 3), terms64, terms64.abs().max(), 1e-6)
    # backward (the FMA route, as the trainers run it)
    d1, i1, _, i2, _ = sb.ops.progressive_loss_forward(x, s, sizes, w)
    ct = torch.randn(npf, 3, generator=tbp._gen(seed + 1))
    X, S = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
    total, terms = sb.ops.ProgressiveLossFunction.apply(S, X, sizes, w)
    (0.8 * total + (terms * ct.cuda()).sum()).backward()
    XL, SL = tbp._leaf(x), tbp._leaf(s)
    total64, terms64 = tbp._progressive64(XL, SL, sizes, w32, i1.long().cpu(), i2.long().cpu(), d1.cpu().double())
    gX, gS = torch.autograd.grad(0.8 * total64 + (terms64 * ct.double()).sum(), [XL, SL])
    # fp32 Chamfer backward over the concatenated prefix index sets (measured <= 2.7e-6)
    bars.check("grad samp", S.grad, gS, gS.abs().max(), 1e-5)
    bars.check("grad ref", X.grad, gX, gX.abs().max(), 1e-5)
    bars.done()


# ---------------------------------------------------------------------------------------------------- GPU: separate simplification loss
@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,threads", SIMP_CASES)
def test_simplification_loss_vs_float64(sb, oracle, b, n, m, threads):
    """chamfer_forward_kernel + simplification_reduce_kernel: dist / idx bit-identical to the fused tail's (and to the oracle where that
    is cheap), out4 against float64, SimplificationLossFunction's backward against float64 autograd."""
    assert reduce_threads(sb, b) == threads
    x, s = _tail_clouds(b + n + m, b, n, m)
    bars = tbp._Bars()
    X64, S64 = tbp._cpu64(x), tbp._cpu64(s)
    for unfused in (False, True):
        tag = "unfused" if unfused else "fma"
        out4, d1, i1, d2, i2 = sb.ops.simplification_loss_forward(s, x, W21, unfused=unfused)
        t = _tail(sb, x, s, 1, 1.0, 0, 0.0, unfused)
        for key, got in (("dist1", d1), ("idx1", i1), ("dist2", d2), ("idx2", i2)):
            assert torch.equal(got, t[key]), "%s %s vs the fused tail" % (tag, key)
        if b * n * m <= ORACLE_PAIRS:
            od1, oi1, od2, oi2 = oracle.nn_distance(_np(s), _np(x), contract=not unfused)
            assert all(np.array_equal(_np(a), c) for a, c in ((d1, od1), (i1, oi1), (d2, od2), (i2, oi2))), tag + " vs oracle"
        loss64, terms64 = tbp._simp64(X64, S64, W21_32, i1.long().cpu(), i2.long().cpu(), tbp._first_argmax(d1.cpu()))
        bars.check(tag + " loss", out4[3], loss64, abs(float(loss64)), 1e-6)     # fp32 sums in a fixed order (measured <= 1.3e-7)
        bars.check(tag + " terms", out4[:3], terms64, terms64.abs().max(), 1e-6)
    R, S = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
    (0.9 * sb.ops.SimplificationLossFunction.apply(S, R, W21)).backward()
    _, d1, i1, _, i2 = sb.ops.simplification_loss_forward(s, x, W21)
    RL, SL = tbp._leaf(x), tbp._leaf(s)
    loss64, _ = tbp._simp64(RL, SL, W21_32, i1.long().cpu(), i2.long().cpu(), tbp._first_argmax(d1.cpu()))
    gR, gS = torch.autograd.grad(0.9 * loss64, [RL, SL])
    bars.check("grad samp", S.grad, gS, gS.abs().max(), 1e-5)   # fp32 Chamfer backward (bar of the fused tail's gradients; measured <= 1.9e-7)
    bars.check("grad ref", R.grad, gR, gR.abs().max(), 1e-5)
    bars.done()


# ---------------------------------------------------------------------------------------------------- GPU: all three entries
@pytest.mark.gpu
def test_batch_invariance(sb):
    """The first and the last cloud of each entry's largest batch, run alone at b = 1, give bit-identical per-cloud outputs, although
    the planners pick other lanes per query there (a different lexicographic merge)."""
    b, n, m, k = 2048, 1024, 64, 8
    x, s = _tail_clouds(5, b, n, m)
    t0 = 0.1
    full = _tail(sb, x, s, k, t0, 1, 1e-4, False)
    simp = sb.ops.simplification_loss_forward(s, x, W21)
    for c in (0, b - 1):
        one = _tail(sb, x[c:c + 1].contiguous(), s[c:c + 1].contiguous(), k, t0, 1, 1e-4, False)
        for key in ("proj", "idx", "weights", "dist", "dist1", "idx1", "dist2", "idx2"):
            assert torch.equal(full[key][c:c + 1], one[key]), ("tail", c, key)
        alone = sb.ops.simplification_loss_forward(s[c:c + 1].contiguous(), x[c:c + 1].contiguous(), W21)
        for i in range(1, 5):
            assert torch.equal(simp[i][c:c + 1], alone[i]), ("simplification", c, i)
    b, n, m, sizes = 64, 1024, 4096, [4, 16, 64, 256, 1024, 2048, 3001, 4096]
    x, s = _prog_clouds(6, b, n, m, None)
    full = sb.ops.progressive_loss_forward(x, s, sizes, _weights(sizes))
    for c in (0, b - 1):
        one = sb.ops.progressive_loss_forward(x[c:c + 1].contiguous(), s[c:c + 1].contiguous(), sizes, _weights(sizes))
        for i in range(4):
            assert torch.equal(full[i][c:c + 1], one[i]), ("progressive", c, i)


@pytest.mark.gpu
def test_repeats_are_bit_identical_and_the_ticket_returns_to_zero(sb):
    """The tail and the progressive loss alternate on one ticket word (the stream's): it is zero after every call, and every output of
    a repeated call -- out4 and terms included -- is bit-identical."""
    xt, st = _tail_clouds(8, 154, 1024, 64)
    xp, sp = _prog_clouds(9, 9, 1024, 1024, None)
    sizes = [2 ** i for i in range(1, 11)]
    ticket = sb.ops._ticket(xt.device)
    runs = {"tail": [], "progressive": [], "simplification": []}
    for _ in range(2):
        runs["tail"].append(list(_tail(sb, xt, st, 8, 0.1, 1, 1e-4, False).values()))
        torch.cuda.synchronize()
        assert int(ticket) == 0
        runs["progressive"].append(list(sb.ops.progressive_loss_forward(xp, sp, sizes, _weights(sizes))))
        torch.cuda.synchronize()
        assert int(ticket) == 0
        runs["simplification"].append(list(sb.ops.simplification_loss_forward(st, xt, W21)))
    for name, (a, c) in runs.items():
        assert all(torch.equal(u, v) for u, v in zip(a, c)), name


def _offset(t):
    """A copy of t whose data starts 4 bytes past a 16-byte boundary (a view of buf[1:])."""
    buf = torch.empty(t.numel() + 1, device=t.device, dtype=t.dtype)
    buf[1:].copy_(t.flatten())
    v = buf[1:].view(t.shape)
    assert v.data_ptr() % 16 == 4 and v.is_contiguous()
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["tail", "progressive", "simplification"])
def test_unaligned_inputs_give_the_aligned_results(sb, entry):
    """ref and samp 4 bytes off 16-byte alignment: the TMA stagings fall back to the scalar loops, and every output is bit-identical."""
    if entry == "tail":
        x, s = _tail_clouds(10, 32, 1024, 64)
        assert tail_plan(sb, 32, 1024, 64)["tma"] == 1
        run = lambda a, c: list(_tail(sb, a, c, 8, 0.1, 1, 1e-4, False).values())
    elif entry == "progressive":
        x, s = _prog_clouds(11, 9, 1024, 1024, None)
        sizes = [2 ** i for i in range(1, 11)]
        run = lambda a, c: list(sb.ops.progressive_loss_forward(a, c, sizes, _weights(sizes)))
    else:
        x, s = _tail_clouds(12, 33, 1024, 64)
        run = lambda a, c: list(sb.ops.simplification_loss_forward(c, a, W21))
    want, got = run(x, s), run(_offset(x), _offset(s))
    for i, (a, c) in enumerate(zip(want, got)):
        assert torch.equal(a, c), (entry, i)


# ---------------------------------------------------------------------------------------------------- GPU: write sets
@pytest.fixture(scope="module")
def arena_store(sb):
    return {}


@pytest.fixture
def arena(arena_store):
    a = arena_store.get("a")
    if a is None:
        a = arena_store["a"] = tws.Arena(512 << 20)
    a.words.fill_(tws.POISON)
    a.off, a.regions = tws.GUARD, []
    return a


def _zero_ticket(arena, tag):
    return arena.carve(tag + ".ticket", (1,), dtype=torch.int32, fill=torch.zeros(1, dtype=torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,k,skew", [(2, 1024, 63, 8, 0), (154, 1024, 64, 8, 0), (9, 4096, 4096, 32, 0), (5, 4095, 4095, 7, 4),
                                          (12, 8, 4096, 8, 4)])
def test_tail_writes_only_its_buffers(sb, arena, b, n, m, k, skew):
    """Three calls in a row, each on its own buffers, dist_over_sigma given and not; the workspace carved at exactly its queried size and
    the ticket back at zero after each."""
    lib = sb._lib.lib()
    wsb = int(lib.snb200_project_and_loss_workspace_bytes(b, m, n))
    x, s = _tail_clouds(b + n, b, n, m)
    rep, rc = [], []
    for i, with_dos in enumerate((True, False, True)):
        tag = "call%d" % i
        ref = arena.carve(tag + ".ref", (b, n, 3), skew=skew, fill=x.cpu())
        samp = arena.carve(tag + ".samp", (b, m, 3), skew=skew, fill=s.cpu())
        sig = arena.carve(tag + ".sigma", (1,), fill=torch.tensor([0.3]))
        proj = arena.carve(tag + ".proj", (b, m, 3), skew=skew)
        kidx = arena.carve(tag + ".knn_idx", (b, m, k), dtype=torch.int32, skew=skew)
        wts = arena.carve(tag + ".weights", (b, m, k), skew=skew)
        dos = arena.carve(tag + ".dist_over_sigma", (b, m, k), skew=skew) if with_dos else None
        d1, i1 = arena.carve(tag + ".dist1", (b, m), skew=skew), arena.carve(tag + ".idx1", (b, m), dtype=torch.int32, skew=skew)
        d2, i2 = arena.carve(tag + ".dist2", (b, n), skew=skew), arena.carve(tag + ".idx2", (b, n), dtype=torch.int32, skew=skew)
        out4 = arena.carve(tag + ".out4", (4,), skew=skew)
        ws = arena.carve(tag + ".workspace", (wsb,), dtype=torch.uint8)
        ticket = _zero_ticket(arena, tag)
        outs = [proj, kidx, wts, d1, i1, d2, i2, out4] + ([dos] if with_dos else [])
        rep += tws.run_checked(arena, "%s project_and_loss_forward(dist_over_sigma=%d)" % (tag, with_dos), lambda: rc.append(
            lib.snb200_project_and_loss_forward(b, n, m, k, ref.data_ptr(), samp.data_ptr(), sig.data_ptr(), 1, 1e-4, proj.data_ptr(),
                                                kidx.data_ptr(), wts.data_ptr(), tws._vp(dos), d1.data_ptr(), i1.data_ptr(), d2.data_ptr(),
                                                i2.data_ptr(), W21, out4.data_ptr(), tws._addr(ws), wsb, ticket.data_ptr(), 0, None)),
            [ws, ticket], full=outs, zero=[(ticket, tag + " ticket")])
    assert rc == [0] * 3, lib.snb200_last_error()
    tws.assert_clean(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,sizes,skew", [(1, 33, 31, list(range(1, 17)), 0), (9, 1024, 1024, [2 ** i for i in range(1, 11)], 0),
                                              (2, 4097, 1531, _FIB, 4), (64, 1024, 4096, [4, 16, 64, 256, 1024, 2048, 3001, 4096], 0),
                                              (3, 5000, 4096, [1, 7, 4095, 4096], 4)])
def test_progressive_writes_only_its_buffers(sb, arena, b, n, m, sizes, skew):
    lib = sb._lib.lib()
    npf = len(sizes)
    wsb = int(lib.snb200_progressive_loss_workspace_bytes(b, n, m, npf))
    csz = (ctypes.c_int * npf)(*sizes)
    cw = (ctypes.c_float * npf)(*_weights(sizes))
    x, s = _prog_clouds(b + n, b, n, m, None)
    rep, rc = [], []
    for i in range(2):
        tag = "call%d" % i
        ref = arena.carve(tag + ".ref", (b, n, 3), skew=skew, fill=x.cpu())
        samp = arena.carve(tag + ".samp", (b, m, 3), skew=skew, fill=s.cpu())
        d1, i1 = arena.carve(tag + ".dist1", (b, m), skew=skew), arena.carve(tag + ".idx1", (b, m), dtype=torch.int32, skew=skew)
        d2, i2 = arena.carve(tag + ".dist2", (b, npf, n), skew=skew), arena.carve(tag + ".idx2", (b, npf, n), dtype=torch.int32, skew=skew)
        terms = arena.carve(tag + ".terms", (3 * npf + 1,), skew=skew)
        ws = arena.carve(tag + ".workspace", (wsb,), dtype=torch.uint8)
        ticket = _zero_ticket(arena, tag)
        rep += tws.run_checked(arena, tag + " progressive_loss_forward", lambda: rc.append(lib.snb200_progressive_loss_forward(
            b, n, m, ref.data_ptr(), samp.data_ptr(), npf, csz, cw, d1.data_ptr(), i1.data_ptr(), d2.data_ptr(), i2.data_ptr(), terms.data_ptr(),
            tws._addr(ws), wsb, ticket.data_ptr(), 0, None)), [ws, ticket], full=[d1, i1, d2, i2, terms], zero=[(ticket, tag + " ticket")])
    assert rc == [0] * 2, lib.snb200_last_error()
    tws.assert_clean(rep)


@pytest.mark.gpu
@pytest.mark.parametrize("b,n,m,skew", [(1, 1, 1, 0), (33, 1024, 64, 0), (5, 1023, 77, 4), (2048, 1024, 64, 0)])
def test_simplification_loss_writes_only_its_buffers(sb, arena, b, n, m, skew):
    lib = sb._lib.lib()
    wsb = int(lib.snb200_simplification_loss_workspace_bytes(b, m, n))
    x, s = _tail_clouds(b + m, b, n, m)
    rep, rc = [], []
    for i in range(2):
        tag = "call%d" % i
        ref = arena.carve(tag + ".ref", (b, n, 3), skew=skew, fill=x.cpu())
        samp = arena.carve(tag + ".samp", (b, m, 3), skew=skew, fill=s.cpu())
        d1, i1 = arena.carve(tag + ".dist1", (b, m), skew=skew), arena.carve(tag + ".idx1", (b, m), dtype=torch.int32, skew=skew)
        d2, i2 = arena.carve(tag + ".dist2", (b, n), skew=skew), arena.carve(tag + ".idx2", (b, n), dtype=torch.int32, skew=skew)
        out4 = arena.carve(tag + ".out4", (4,), skew=skew)
        ws = arena.carve(tag + ".workspace", (wsb,), dtype=torch.uint8)
        rep += tws.run_checked(arena, tag + " simplification_loss_forward", lambda: rc.append(lib.snb200_simplification_loss_forward(
            b, m, samp.data_ptr(), n, ref.data_ptr(), W21, d1.data_ptr(), i1.data_ptr(), d2.data_ptr(), i2.data_ptr(), out4.data_ptr(),
            tws._addr(ws), wsb, 0, None)), [ws], full=[d1, i1, d2, i2, out4])
    assert rc == [0] * 2, lib.snb200_last_error()
    tws.assert_clean(rep)
