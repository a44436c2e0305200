"""GPU parity tests (run on a GPU with `-m gpu`): the CUDA path, called through the C-ABI library via the
package's public API, against the CPU oracle on the same seeded inputs, against the committed golden fixtures
(generated from the reference's own Python classes, tests/golden/make_golden.py), against the reference's own CPU code
compiled into oracle/_ref, and -- at BASELINE.json's full sizes -- through size-independent properties.

Bars: indices bit-exact; squared distances bit-exact against the oracle evaluated in the same arithmetic mode
(SNB200_DIST_FMA <-> oracle contract=True, SNB200_DIST_UNFUSED <-> oracle contract=False == the reference CPU code);
floating-point results of softmax / reductions within the tolerance written at each assert.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

REF_CPU = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_cpu.npz")))   # tests/golden/make_reference_cpu_golden.py


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device="cuda")


def _n(t):
    return t.detach().cpu().numpy()


def _rng(seed):
    return np.random.default_rng(seed)


@pytest.fixture(scope="module")
def sb():
    import samplenet_b200

    samplenet_b200._lib.lib()  # fail loudly if the CUDA library is missing
    return samplenet_b200


# ------------------------------------------------------------------------------------------------ Chamfer forward
@pytest.mark.parametrize("b,n,m", [(1, 1, 1), (2, 64, 1024), (3, 37, 129), (2, 513, 511), (1, 1024, 64), (4, 5, 3), (2, 33, 4099), (1, 6000, 70)])
def test_chamfer_forward_bitexact(sb, oracle, b, n, m):
    r = _rng(b * 1000 + n + m)
    a = r.standard_normal((b, n, 3)).astype(np.float32)
    c = r.standard_normal((b, m, 3)).astype(np.float32)
    if n > 4:
        a[:, 3] = a[:, 1]  # duplicated points: exact ties, lowest index must win
    if m > 4:
        c[:, 4] = c[:, 0]
    for unfused in (False, True):
        d1, i1, d2, i2 = sb.ops.nn_distance_forward(_t(a), _t(c), unfused=unfused)
        e1, j1, e2, j2 = oracle.nn_distance(a, c, contract=not unfused)
        assert np.array_equal(_n(i1), j1) and np.array_equal(_n(i2), j2)
        assert np.array_equal(_n(d1), e1) and np.array_equal(_n(d2), e2)
    # the reference's own CPU code, compiled unmodified, on these inputs
    d1, i1, d2, i2 = sb.ops.nn_distance_forward(_t(a), _t(c), unfused=True)
    rd1, ri1, rd2, ri2 = (REF_CPU["chamfer_%d_%d_%d_%s" % (b, n, m, s)] for s in ("d1", "i1", "d2", "i2"))
    assert np.array_equal(_n(i1), ri1) and np.array_equal(_n(i2), ri2)
    assert np.array_equal(_n(d1), rd1) and np.array_equal(_n(d2), rd2)


def test_chamfer_lattice_ties(sb, oracle):
    g = np.stack(np.meshgrid(np.arange(6), np.arange(6), np.arange(6), indexing="ij"), -1).reshape(1, -1, 3).astype(np.float32)
    q = (g[:, ::5] + np.float32(0.5)).copy()  # equidistant from 8 lattice points each
    d1, i1, d2, i2 = sb.ops.nn_distance_forward(_t(q), _t(g))
    e1, j1, e2, j2 = oracle.nn_distance(q, g, contract=True)
    assert np.array_equal(_n(i1), j1) and np.array_equal(_n(i2), j2)


def test_chamfer_backward_and_module(sb, oracle, golden_dir):
    z = np.load(os.path.join(golden_dir, "chamfer_reg.npz"))
    a = _t(z["xyz1"]).requires_grad_(True)
    c = _t(z["xyz2"]).requires_grad_(True)
    d1, d2 = sb.ChamferDistance()(a, c)
    # reference autograd Function ran the CPU (unfused) arithmetic: distances agree to 1 ulp-ish
    np.testing.assert_allclose(_n(d1), z["dist1"], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(_n(d2), z["dist2"], rtol=1e-6, atol=1e-7)
    ((d1 * _t(z["w1"])).sum() + (d2 * _t(z["w2"])).sum()).backward()
    np.testing.assert_allclose(_n(a.grad), z["grad_xyz1"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(_n(c.grad), z["grad_xyz2"], rtol=1e-5, atol=1e-6)
    # larger random case against the oracle's sequential backward (many-to-one scatter)
    r = _rng(5)
    x1 = r.standard_normal((3, 64, 3)).astype(np.float32); x2 = r.standard_normal((3, 1500, 3)).astype(np.float32)
    g1 = r.standard_normal((3, 64)).astype(np.float32); g2 = r.standard_normal((3, 1500)).astype(np.float32)
    _, i1, _, i2 = oracle.nn_distance(x1, x2, contract=True)
    gx1, gx2 = sb.ops.nn_distance_backward(_t(x1), _t(x2), _t(g1), _t(i1, torch.int32), _t(g2), _t(i2, torch.int32))
    ox1, ox2 = oracle.nn_distance_grad(x1, x2, g1, i1, g2, i2)
    np.testing.assert_allclose(_n(gx1), ox1, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(_n(gx2), ox2, rtol=2e-5, atol=2e-5)
    # determinism: two runs are bit-identical (the reference's atomics are not)
    gy1, gy2 = sb.ops.nn_distance_backward(_t(x1), _t(x2), _t(g1), _t(i1, torch.int32), _t(g2), _t(i2, torch.int32))
    assert torch.equal(gx1, gy1) and torch.equal(gx2, gy2)


# ------------------------------------------------------------------------------------------------ kNN / projection
@pytest.mark.parametrize("b,n,m,k", [(2, 1024, 64, 8), (2, 1024, 32, 7), (1, 2048, 64, 16), (3, 200, 17, 3), (2, 35, 9, 1),
                                     (1, 64, 5, 32), (1, 4100, 6, 8), (2, 9001, 3, 16), (1, 40, 40, 32)])
@pytest.mark.parametrize("layout", ["bnc", "bcn"])
def test_knn_and_soft_projection_vs_oracle(sb, oracle, b, n, m, k, layout):
    r = _rng(n * 13 + m + k)
    pts = r.standard_normal((b, n, 3)).astype(np.float32)
    sel = r.permutation(n)[:m]
    qry = (pts[:, sel] + 0.05 * r.standard_normal((b, m, 3))).astype(np.float32)
    sigma = np.float32(0.37)
    P, Q = (_t(pts), _t(qry)) if layout == "bnc" else (_t(pts.transpose(0, 2, 1)), _t(qry.transpose(0, 2, 1)))
    for unfused in (False, True):
        o = sb.ops.knn_soft_project_forward(P, Q, k, layout, _t([sigma]), want=("proj", "idx", "val", "weights", "dist"), unfused=unfused)
        val, idx = oracle.knn_point(k, pts, qry, contract=not unfused, tie_mode=1)
        assert np.array_equal(_n(o["idx"]), idx)
        assert np.array_equal(_n(o["val"]), val)
        proj, w, d = oracle.soft_project(pts, qry, idx, float(sigma))
        gp = _n(o["proj"]) if layout == "bnc" else _n(o["proj"]).transpose(0, 2, 1)
        np.testing.assert_allclose(gp, proj, rtol=2e-6, atol=2e-6)
        np.testing.assert_allclose(_n(o["weights"]), w, rtol=2e-6, atol=1e-7)
        np.testing.assert_allclose(_n(o["dist"]), d, rtol=1e-6, atol=0)
    # reference selection-sort tie order (tie_mode=0) coincides on tie-free inputs
    _, idx0 = oracle.knn_point(k, pts, qry, contract=True, tie_mode=0)
    assert np.array_equal(idx0, oracle.knn_point(k, pts, qry, contract=True, tie_mode=1)[1])


def test_knn_duplicate_points_tie_contract(sb, oracle):
    """Duplicated cloud points (pctransforms.py:145-146 creates them): sorted by (distance, index)."""
    r = _rng(3)
    pts = r.standard_normal((2, 128, 3)).astype(np.float32)
    pts[:, 64:] = pts[:, :64]
    qry = pts[:, 5:25].copy()
    o = sb.ops.knn_soft_project_forward(_t(pts), _t(qry), 6, "bnc", want=("idx", "val"))
    val, idx = oracle.knn_point(6, pts, qry, contract=True, tie_mode=1)
    assert np.array_equal(_n(o["idx"]), idx) and np.array_equal(_n(o["val"]), val)


def test_reference_selftest_known_answers_on_gpu(sb):
    """registration/src/soft_projection.py:158-284 and classification/soft_projection.py:86-161 golden vectors."""
    A = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [5, 4, 4], [4, 5, 4], [4, 4, 5], [8, 7, 7], [7, 8, 7], [7, 7, 8]], np.float32)
    Bc = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [5, 5, 5], [7, 7, 8], [7, 7, 8.5]], np.float32)
    feats = np.arange(1, 31, dtype=np.float32).reshape(6, 5)
    exp_feat = np.array([[6.0, 7.0, 8.0, 9.0, 10.0], [2.459, 3.459, 4.459, 5.459, 6.459], [2.459, 3.459, 4.459, 5.459, 6.459],
                         [16.0, 17.0, 18.0, 19.0, 20.0], [16.0, 17.0, 18.0, 19.0, 20.0], [16.0, 17.0, 18.0, 19.0, 20.0],
                         [22.113, 23.113, 24.113, 25.113, 26.113], [22.113, 23.113, 24.113, 25.113, 26.113],
                         [23.189, 24.189, 25.189, 26.189, 27.189]], np.float32)
    exp_cloud = np.array([[0.333, 0.333, 0.333], [1, 0, 0], [1, 0, 0], [4.333, 4.333, 4.333], [7, 7, 8], [7, 7, 8]], np.float32)
    exp_hard = np.array([[1, 0, 0], [1, 0, 0], [1, 0, 0], [5, 4, 4], [7, 7, 8], [7, 7, 8]], np.float32)
    # torch flavour (BCN)
    sp = sb.SoftProjection(3, initial_temperature=1.0).cuda()
    prop = sp.propagate(_t(Bc.T[None]), _t(feats.T[None]), _t(A.T[None]))
    assert np.abs(_n(prop)[0].T - exp_feat).max() < 6e-4
    sd = sp.state_dict(); sd["_temperature"] = torch.tensor(0.1); sp.load_state_dict(sd)
    proj = sp.project(_t(A.T[None]), _t(Bc.T[None]))
    assert np.abs(_n(proj)[0].T - exp_cloud).max() < 6e-4
    # TF flavour (BNC), batch of 2 with the scaled cloud, T=0.01, soft and hard
    tp = sb.tf_ops.SoftProjection(3, initial_temperature=0.01).cuda()
    pc = _t(np.stack([A, A * 3])); qc = _t(np.stack([Bc, Bc * 3]))
    soft, w, d = tp(pc, qc)
    hard, wh, _ = tp(pc, qc, hard=True)
    assert w.shape == (2, 6, 3, 1) and d.shape == (2, 6, 3, 1)
    assert np.abs(_n(soft)[0] - exp_cloud).max() < 1.1e-3 and np.abs(_n(soft)[1] - 3 * exp_cloud).max() < 3.1e-3
    assert np.abs(_n(hard)[0] - exp_hard).max() < 1e-6 and np.abs(_n(hard)[1] - 3 * exp_hard).max() < 1e-6


def test_soft_projection_module_vs_reference_fixture(sb, golden_dir):
    z = np.load(os.path.join(golden_dir, "softproj_reg.npz"))
    sp = sb.SoftProjection(int(z["k"]), initial_temperature=float(z["temperature"]), min_sigma=float(z["min_sigma"])).cuda()
    pc = _t(z["point_cloud"]).requires_grad_(True); qc = _t(z["query_cloud"]).requires_grad_(True)
    ft = _t(z["feats"]).requires_grad_(True)
    pp, pf = sp(pc, qc, ft, action="project_and_propagate")
    np.testing.assert_allclose(_n(pp), z["proj"], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(_n(pf), z["prop"], rtol=2e-6, atol=2e-6)
    ((pp * _t(z["r1"])).sum() + (pf * _t(z["r2"])).sum()).backward()
    np.testing.assert_allclose(_n(qc.grad), z["grad_query_cloud"], rtol=2e-4, atol=2e-5)
    np.testing.assert_allclose(_n(pc.grad), z["grad_point_cloud"], rtol=2e-4, atol=2e-5)
    np.testing.assert_allclose(_n(ft.grad), z["grad_feats"], rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(_n(sp._temperature.grad), z["grad_temperature"], rtol=2e-4, atol=1e-5)
    np.testing.assert_allclose(_n(sp(pc.detach(), qc.detach())), z["only_proj"], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(_n(sp(pc.detach(), qc.detach(), ft.detach(), action="propagate")), z["only_prop"], rtol=2e-6, atol=2e-6)
    with pytest.raises(ValueError):
        sp(pc, qc, action="nonsense")
    d, i = sb.knn_point(4, pc.detach(), qc.detach())
    assert d.shape == (3, 4, 17) and i.dtype == torch.int64 and bool((d[:, 1:] >= d[:, :-1]).all())


def test_group_point_and_grad(sb, oracle):
    r = _rng(9)
    pts = r.standard_normal((2, 300, 7)).astype(np.float32)
    idx = r.integers(0, 300, size=(2, 40, 5)).astype(np.int32)
    idx[:, :, 1] = idx[:, :, 0]  # repeated indices inside a group
    p = _t(pts).requires_grad_(True)
    out = sb.tf_ops.group_point(p, _t(idx, torch.int32))
    assert np.array_equal(_n(out), oracle.group_point(pts, idx))
    go = r.standard_normal(out.shape).astype(np.float32)
    out.backward(_t(go))
    np.testing.assert_allclose(_n(p.grad), oracle.group_point_grad(pts.shape, idx, go), rtol=1e-5, atol=1e-5)
    # BCN flavour (pointnet2 grouping_operation)
    ob = sb.ops.group_point(_t(pts.transpose(0, 2, 1)), _t(idx, torch.int32), "bcn")
    assert np.array_equal(_n(ob), oracle.group_point(pts, idx).transpose(0, 3, 1, 2))


# ------------------------------------------------------------------------------------------------ SampleNet end to end
def _load_net(sb, z, **kw):
    net = sb.SampleNet(64, 128, group_size=8, initial_temperature=1.0, **kw)
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd_")}
    net.load_state_dict(sd)  # reference state-dict keys load as-is
    return net.cuda()


def test_samplenet_config0_vs_reference_fixture(sb, golden_dir):
    """BASELINE config 0: registration SampleNet fwd + soft-proj (+ both losses, backward), B=2, N=1024->64, k=8.

    With B=2 the BatchNorm over the batch in the FC head is ill-conditioned: the reference's own fp32 output sits 2.8e-4
    away from its fp64 evaluation (fixture key simp_fp64) and moves by 8e-5 when torch uses a different thread count.  So
    (a) the generator is judged against the fp64 yardstick, and (b) everything downstream is compared on IDENTICAL inputs
    (the reference's own simp), where tight tolerances are meaningful."""
    z = np.load(os.path.join(golden_dir, "samplenet_reg_b2.npz"))
    net = _load_net(sb, z, input_shape="bnc", output_shape="bnc")
    net.train()
    x = _t(z["x"])
    simp, proj = net(x)
    assert simp.is_contiguous() and proj.is_contiguous() and simp.shape == (2, 64, 3) and proj.shape == (2, 64, 3)
    # (a) generator: no further from the fp64 truth than twice the reference's own fp32 error
    err_ref = np.abs(z["simp"].astype(np.float64) - z["simp_fp64"]).max()
    err_ours = np.abs(_n(simp).astype(np.float64) - z["simp_fp64"]).max()
    assert err_ours <= 2.0 * err_ref + 1e-6, (err_ours, err_ref)
    np.testing.assert_allclose(_n(proj), z["proj"], rtol=0, atol=1.5e-3)  # end-to-end sanity (noise amplified by the kNN switch points)
    # (b) projection, losses and their gradients on the reference's own simp
    simp_ref = _t(z["simp"]).requires_grad_(True)
    proj_id = net.project.project(x, simp_ref.detach(), layout="bnc")
    np.testing.assert_allclose(_n(proj_id), z["proj"], rtol=2e-6, atol=2e-6)
    loss_s = net.get_simplification_loss(x, simp_ref, 64, 1, 0)
    loss_p = net.get_projection_loss()
    assert abs(float(loss_s.detach()) - float(z["loss_simplification"])) < 1e-5 * max(1.0, abs(float(z["loss_simplification"])))  # north_star bar
    np.testing.assert_allclose(_n(loss_p), z["loss_projection"], rtol=1e-6)
    # in the reference graph the returned `simp` only feeds the simplification loss (proj hangs off the pre-permute tensor),
    # so fixture grad_simp == 0.01 * d loss_s / d simp
    (0.01 * loss_s).backward()
    np.testing.assert_allclose(_n(simp_ref.grad), z["grad_simp"], rtol=2e-4, atol=1e-7)
    # temperature: d/dT [0.01 * sigma + sum(proj * rw)] with proj computed from the reference's simp
    net.zero_grad()
    (0.01 * loss_p + (proj_id * _t(z["rw"])).sum()).backward()
    np.testing.assert_allclose(_n(net.project._temperature.grad), z["grad_temperature"], rtol=2e-4, atol=1e-5)
    # (c) whole step end to end runs and yields finite gradients for every parameter (values are checked at a
    # well-conditioned batch size in test_generator_backward_matches_torch_autograd: at B=2 they are rounding noise)
    net.zero_grad()
    simp2, proj2 = net(x)
    total = 0.01 * net.get_simplification_loss(x, simp2, 64, 1, 0) + 0.01 * net.get_projection_loss() + (proj2 * _t(z["rw"])).sum()
    total.backward()
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in net.parameters())
    # BatchNorm running statistics after training steps follow PyTorch's momentum rule: compare after ONE step on a fresh net
    net1 = _load_net(sb, z, input_shape="bnc", output_shape="bnc").train()
    net1(x)
    sd = net1.state_dict()
    for key in z.files:
        if key.startswith("after_"):
            np.testing.assert_allclose(_n(sd[key[6:]]).astype(np.float64), z[key].astype(np.float64), rtol=5e-4, atol=3e-5, err_msg=key)


def test_samplenet_eval_matching_vs_reference_fixture(sb, oracle, golden_dir):
    z = np.load(os.path.join(golden_dir, "samplenet_reg_b2.npz"))
    e = np.load(os.path.join(golden_dir, "samplenet_reg_b2_eval.npz"))
    # (a) the matching kernel alone on the reference's NN indices: exact
    out = sb.sputils.nn_matching_cuda(_t(z["x"]), _t(e["nn_idx"], torch.int32), 64, complete_fps=True)
    assert np.array_equal(_n(out), e["match"].astype(np.float32))
    assert np.array_equal(sb.sputils.nn_matching(z["x"], e["nn_idx"], 64), oracle.nn_matching(z["x"], e["nn_idx"], 64))
    out2 = sb.sputils.nn_matching_cuda(_t(z["x"]), _t(e["nn_idx"], torch.int32), 64, complete_fps=False)
    assert np.array_equal(_n(out2), np.take_along_axis(z["x"], e["nn_idx"][..., None].astype(np.int64).repeat(3, -1), axis=1))
    # (b) the whole eval forward, starting from a state after one training step like the fixture did
    net = _load_net(sb, z, input_shape="bnc", output_shape="bnc")
    net.train(); net(_t(z["x"])); net.eval()
    with torch.no_grad():
        simp, match = net(_t(z["x"]))
    np.testing.assert_allclose(_n(simp), e["simp_eval"], rtol=0, atol=1e-3)  # B=2 BatchNorm conditioning, see config0 test
    assert match.shape == (2, 64, 3)
    # every matched point is a point of the input cloud, and (NN assignment being stable under 1e-4 perturbations for
    # all but near-tie queries) nearly all rows coincide with the reference's
    same = (np.abs(_n(match) - e["match"].astype(np.float32)).max(-1) == 0).mean()
    assert same > 0.9
    assert float(net.get_simplification_loss(_t(z["x"]), simp, 64)) == 0.0 and float(net.get_projection_loss()) == 0.0


@pytest.mark.parametrize("shapes", [("bcn", "bcn"), ("bnc", "bcn"), ("bcn", "bnc")])
def test_samplenet_layout_variants_agree(sb, golden_dir, shapes):
    import warnings

    z = np.load(os.path.join(golden_dir, "samplenet_reg_b2.npz"))
    base = _load_net(sb, z, input_shape="bnc", output_shape="bnc").train()
    simp0, proj0 = base(_t(z["x"]))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        net = _load_net(sb, z, input_shape=shapes[0], output_shape=shapes[1])
    net.train()
    x = _t(z["x"]) if shapes[0] == "bnc" else _t(z["x"].transpose(0, 2, 1)).contiguous()
    simp, proj = net(x)
    assert simp.is_contiguous() and proj.is_contiguous()
    if shapes[1] == "bcn":
        assert simp.shape == (2, 3, 64)
        simp, proj = simp.permute(0, 2, 1), proj.permute(0, 2, 1)
    # same arithmetic whatever the layout: bit-identical generator output, projection to fp32 rounding
    assert torch.equal(simp, simp0)
    np.testing.assert_allclose(_n(proj), _n(proj0), rtol=1e-6, atol=1e-6)
    with pytest.raises(RuntimeError):
        net(torch.zeros(2, 4, 10, device="cuda"))


@pytest.mark.parametrize("precision", ["3xtf32", "fp32"])
def test_generator_vs_torch_fp32_reference(sb, precision):
    """The conv/BN/FC stack is a floating-point kernel: compare with plain torch fp32 (CPU) on the headline shape,
    plus the rec widths (reconstruction/src/samplers.py:22-36) and a ragged cloud size through the C-ABI layer API."""
    torch.manual_seed(0)
    net = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc")
    x = torch.rand(32, 1024, 3) - 0.5
    net.train()
    ps = {n: p for n, p in net._generator_named_parameters()}
    ref = net._torch_generator(x, "bnc", True, ps).detach()  # stock torch ops on CPU
    netc = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc")
    netc.load_state_dict(net.state_dict()); netc.cuda().train()
    netc.generator_precision = precision
    with torch.no_grad():
        y = netc._generate(x.cuda(), "bnc", 0)
    np.testing.assert_allclose(_n(y), ref.numpy(), rtol=2e-4, atol=5e-5)  # outputs are O(0.5): fp32 rounding through 9 normalised layers
    # eval mode (running statistics)
    net.eval(); netc.eval()
    ref_e = net._torch_generator(x, "bnc", False, ps).detach()
    with torch.no_grad():
        y_e = netc._generate(x.cuda(), "bnc", 0)
    # netc's running stats were updated by the training forward above, net's were not: sync them first
    net.load_state_dict(netc.state_dict()); ref_e = net._torch_generator(x, "bnc", False, {n: p for n, p in net._generator_named_parameters()}).detach()
    np.testing.assert_allclose(_n(y_e), ref_e.numpy(), rtol=2e-4, atol=2e-5)


def test_generator_backward_matches_torch_autograd(sb):
    """Generator backward (recompute with stock torch ops) == autograd of the reference layer stack, B=32."""
    torch.manual_seed(5)
    torch.backends.cudnn.allow_tf32 = False        # the torch stack on the GPU would otherwise run its convs in plain TF32
    torch.backends.cuda.matmul.allow_tf32 = False
    net = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train()
    net.generator_backward = "torch"     # (the fallback path; the CUDA backward has its own test against float64 below)
    x = (torch.rand(32, 1024, 3, device="cuda") - 0.5)
    g = torch.randn(32, 64, 3, device="cuda")
    simp, _ = net(x)
    simp.backward(g)
    mine = {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}
    net.zero_grad()
    ps = {n: p for n, p in net._generator_named_parameters()}
    y = net._torch_generator(x, "bnc", True, ps).view(32, 3, 64).permute(0, 2, 1)
    y.backward(g)
    for n, p in net.named_parameters():
        if n.startswith("project"):
            continue
        ref = p.grad
        assert n in mine, n
        assert (mine[n] - ref).abs().max().item() <= 1e-4 * ref.abs().max().item() + 1e-7, n
    # and the forward values agree with the same stack to fp32 accuracy
    np.testing.assert_allclose(_n(simp), _n(y), rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize("b,n,m,layout", [(32, 1024, 64, "bnc"), (16, 333, 32, "bcn"), (7, 1000, 64, "bnc"), (64, 512, 64, "bnc")])
def test_generator_cuda_backward_vs_float64_autograd(sb, b, n, m, layout):
    """The hand-written generator backward (csrc/generator_bwd.cu: FC, max-pool, conv dgrad + wgrad with fused BatchNorm backward) against a
    FLOAT64 torch autograd evaluation of the same layer stack (registration/src/samplenet.py:90-104).

    The max-pool sends each (cloud, channel) gradient to ONE point; two points within rounding of the maximum make that choice -- and with
    it every upstream gradient -- discontinuous, so two correct fp32 implementations can disagree at the percent level (stock torch fp32
    vs float64 does, see tools/diag_bwd.py).  The float64 graph therefore gathers at the arg-max of THIS library's own saved activations
    (same routing on both sides); what remains is rounding: every gradient within 2e-4 of its tensor's scale, and bit-identical from run
    to run (no float atomics)."""
    # a well-conditioned instance: no FC pre-activation within 2e-5 of the ReLU kink (a flipped mask on one of the <= 64 rows moves every
    # gradient at the percent level, in ANY fp32 implementation), found by stepping the seed
    for seed in range(b + n, b + n + 20):
        torch.manual_seed(seed)
        net = sb.SampleNet(m, 128, group_size=8, input_shape=layout, output_shape=layout).cuda().train()
        net.generator_backward = "cuda"
        with torch.no_grad():
            for p in net.parameters():
                if p.dim() == 1:
                    p.add_(0.1 * torch.randn_like(p))
        x = torch.rand(b, n, 3, device="cuda") - 0.5
        if layout == "bcn":
            x = x.permute(0, 2, 1).contiguous()
        with torch.no_grad():
            ps = {nm: p.double() for nm, p in net._generator_named_parameters()}
            h = (x.double() if layout == "bnc" else x.double().permute(0, 2, 1)).reshape(-1, 3)
            margin = 1.0
            for i, (lin, bn) in enumerate(net._convs() + net._fcs()):
                if i == 5:
                    h = h.view(b, n, -1).max(dim=1)[0]
                h = torch.nn.functional.linear(h, ps["l%d.w" % i].reshape(ps["l%d.w" % i].shape[0], -1), ps["l%d.b" % i])
                if bn is not None:
                    h = torch.nn.functional.batch_norm(h, None, None, ps["l%d.g" % i], ps["l%d.beta" % i], True, 0.0, bn.eps)
                    if i >= 5:
                        margin = min(margin, h.abs().min().item())
                    h = torch.relu(h)
        if margin > 2e-5:
            break
    conv_specs, fc_specs = net._layer_specs()
    assert sb.ops.generator_backward_supported(x, layout, conv_specs, fc_specs)
    out_inner = m if layout == "bnc" else 0
    rw = torch.randn(b, 3 * m, device="cuda")
    names = [k for k, _ in net._generator_named_parameters()]
    params = [p for _, p in net._generator_named_parameters()]
    runs = []
    for _ in range(2):
        net.zero_grad()
        y = net._generate(x, layout, out_inner)
        (y * rw).sum().backward()
        runs.append([p.grad.detach().clone() for p in params])
    assert all(torch.equal(a, c) for a, c in zip(*runs)), "CUDA backward is not run-to-run deterministic"
    # routing: arg-max of the last conv layer's BN output per (cloud, channel), from the activations the forward kept
    with torch.no_grad():
        _, _, (zs, ws) = sb.ops.generator_train_forward(x, layout, conv_specs, fc_specs, out_inner)
        z5 = zs[4].view(b, n, -1)
        sgn = torch.where(net.bn5.weight >= 0, 1.0, -1.0)                     # the pool takes the max of the raw output where the BN scale is >= 0
        route = (z5 * sgn).argmax(dim=1)                                      # (b, C), exact comparisons on the kept fp32 activations
    ps64 = {nm: p.detach().double().requires_grad_(True) for nm, p in zip(names, params)}
    h = (x.double() if layout == "bnc" else x.double().permute(0, 2, 1)).reshape(-1, 3)
    layers = net._convs() + net._fcs()
    for i, (lin, bn) in enumerate(layers):
        if i == 5:
            h = torch.gather(h.view(b, n, -1), 1, route[:, None, :]).squeeze(1)   # the max-pool, routed
        h = torch.nn.functional.linear(h, ps64["l%d.w" % i].reshape(ps64["l%d.w" % i].shape[0], -1), ps64["l%d.b" % i])
        if bn is not None:
            h = torch.nn.functional.batch_norm(h, None, None, ps64["l%d.g" % i], ps64["l%d.beta" % i], True, 0.0, bn.eps)
            h = torch.relu(h)
    if out_inner:
        h = h.view(b, -1, out_inner).permute(0, 2, 1).reshape(b, -1)
    g64 = torch.autograd.grad(h, list(ps64.values()), rw.double())
    for nm, got, ref in zip(names, runs[0], g64):
        ref = ref.reshape(got.shape)
        scale = max(ref.abs().max().item(), 1e-3)
        err = (got.double() - ref).abs().max().item()
        # biases in front of a training-mode BatchNorm: true gradient exactly 0, both sides hold rounding noise of the layer's dz sums
        # parameters whose TRUE gradient is exactly zero hold rounding noise on both sides: biases in front of a training-mode BatchNorm,
        # and bn5's shift (a constant added to a pooled channel is removed by bn_fc1's mean subtraction)
        zero_true = (nm.endswith(".b") and nm != "l8.b") or nm == "l4.beta"
        tol = 5e-3 if zero_true else 2e-4 * scale
        assert err <= tol, (nm, err, scale)
    np.testing.assert_allclose(_n(y), h.detach().float().cpu().numpy(), rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("b,n", [(32, 1024), (2, 1024), (7, 1000), (37, 1024), (3, 77), (70, 500), (64, 1024), (128, 1024), (41, 1999)])
def test_conv_stack_kernel_vs_per_layer_kernels_and_fp32(sb, b, n):
    """The persistent cooperative conv-stack kernel (activations resident in registers / shared memory) == the per-layer tensor-core kernels ==
    the exact-fp32 CUDA-core path, training and eval mode, full and ragged slices, one slice per CTA and (shapes with more than 128
    points per SM) several slices per CTA with the raw layer outputs parked in L2 between layers."""
    torch.manual_seed(b * 1000 + n)
    net = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda()
    with torch.no_grad():
        for bn in [net.bn1, net.bn2, net.bn3, net.bn4, net.bn5]:
            bn.weight.copy_(1 + 0.3 * torch.randn_like(bn.weight)); bn.bias.copy_(0.2 * torch.randn_like(bn.bias))
            bn.running_mean.copy_(0.1 * torch.randn_like(bn.running_mean)); bn.running_var.copy_(0.5 + torch.rand_like(bn.running_var))
    x = torch.rand(b, n, 3, device="cuda") - 0.5
    conv, fc = net._layer_specs()
    for training in (True, False):
        sd = {k: v.clone() for k, v in net.state_dict().items()}
        outs = []
        for kw in (dict(), dict(separate_head=True), dict(per_layer_kernels=True), dict(exact_fp32=True)):
            net.load_state_dict(sd)
            out, feat = sb.ops.generator_forward(x, "bnc", conv, fc, training, 64, **kw)
            outs.append((out.clone(), feat.clone(), {k: v.clone() for k, v in net.state_dict().items() if "running" in k}))
        for o, f, st in outs[1:]:
            np.testing.assert_allclose(_n(outs[0][1]), _n(f), rtol=3e-4, atol=3e-5)
            if b >= 3:   # (with 2 rows the BatchNorm of the FC head is ill-conditioned, see the config-0 test)
                np.testing.assert_allclose(_n(outs[0][0]), _n(o), rtol=2e-3, atol=2e-4)
            for k in st:
                if b < 3 and "bn_fc" in k:
                    continue
                np.testing.assert_allclose(_n(outs[0][2][k]), _n(st[k]), rtol=1e-4, atol=1e-6, err_msg=k)


@pytest.mark.parametrize("b", [56, 65])
def test_conv_stack_multislice_eval_is_race_free(sb, b):
    """Eval mode has no grid-wide synchronisation between the conv layers, so CTAs of a multi-slice launch drift layers apart: the parked
    activations of a slice must occupy the same bytes in every layer (fixed row stride), or a fast CTA's 128-wide rows overwrite a slow CTA's
    64-wide rows.  That race corrupted one cloud in about every second launch -- repeated launches against the exact-fp32 path."""
    torch.manual_seed(b)
    net = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().eval()
    with torch.no_grad():
        for bn in [net.bn1, net.bn2, net.bn3, net.bn4, net.bn5]:
            bn.running_mean.copy_(0.1 * torch.randn_like(bn.running_mean)); bn.running_var.copy_(0.5 + torch.rand_like(bn.running_var))
    x = torch.rand(b, 1024, 3, device="cuda") - 0.5
    conv, fc = net._layer_specs()
    ref = sb.ops.generator_forward(x, "bnc", conv, fc, False, 64, exact_fp32=True)[1].clone()
    for _ in range(8):
        for kw in (dict(), dict(separate_head=True)):
            feat = sb.ops.generator_forward(x, "bnc", conv, fc, False, 64, **kw)[1]
            np.testing.assert_allclose(_n(feat), _n(ref), rtol=3e-4, atol=3e-5)


def test_conv_stack_statistics_range_guard(sb):
    """The BatchNorm statistics between the conv layers travel as fixed-point words (conv_stack.cu, cs_fx_*): inputs of any scale stay exact
    (layer 1 is normalised analytically), and a layer whose pre-activations leave the representable range (|z| beyond ~3e4) must poison the
    launch -- NaN rows -- instead of returning numbers computed from clipped statistics."""
    torch.manual_seed(5)
    net = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train()
    conv, fc = net._layer_specs()
    x = torch.rand(32, 1024, 3, device="cuda") - 0.5
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    for scale in (1.0, 1e3, 1e-3):
        net.load_state_dict(sd)
        o1, f1 = sb.ops.generator_forward(x * scale, "bnc", conv, fc, True, 64)
        net.load_state_dict(sd)
        o2, f2 = sb.ops.generator_forward(x * scale, "bnc", conv, fc, True, 64, per_layer_kernels=True)
        assert torch.isfinite(o1).all()
        np.testing.assert_allclose(_n(f1), _n(f2), rtol=3e-4, atol=3e-5)
    with torch.no_grad():
        net.conv2.weight.mul_(1e6)
    conv, fc = net._layer_specs()
    o3, _ = sb.ops.generator_forward(x, "bnc", conv, fc, True, 64)
    assert torch.isnan(o3).all()
    net.load_state_dict(sd)
    conv, fc = net._layer_specs()
    o4, _ = sb.ops.generator_forward(x, "bnc", conv, fc, True, 64)   # the next launch is clean again
    assert torch.isfinite(o4).all()


def test_generator_rec_widths_and_ragged_sizes(sb):
    torch.manual_seed(1)
    import torch.nn.functional as F
    widths = [3, 64, 128, 128, 256, 128]
    b, n = 5, 777
    x = torch.randn(b, n, 3)
    Ws = [torch.randn(widths[i + 1], widths[i]) / widths[i] ** 0.5 for i in range(5)]
    bs = [0.1 * torch.randn(widths[i + 1]) for i in range(5)]
    gs = [1 + 0.2 * torch.randn(widths[i + 1]) for i in range(5)]
    be = [0.1 * torch.randn(widths[i + 1]) for i in range(5)]
    y = x.permute(0, 2, 1)
    for i in range(5):
        y = F.relu(F.batch_norm(F.conv1d(y, Ws[i][:, :, None], bs[i]), None, None, gs[i], be[i], True, 0.0, 1e-3))
    ref = y.max(2)[0]
    conv = [dict(weight=Ws[i].cuda(), bias=bs[i].cuda(), bn=(gs[i].cuda(), be[i].cuda(), None, None, 1e-3, 0.1), relu=True) for i in range(5)]
    fcw = torch.eye(128).cuda()
    fc = [dict(weight=fcw, bias=torch.zeros(128).cuda(), bn=None, relu=False)]
    for kw in (dict(), dict(exact_fp32=True)):
        out, feat = sb.ops.generator_forward(x.cuda(), "bnc", conv, fc, True, **kw)
        np.testing.assert_allclose(_n(feat), ref.numpy(), rtol=3e-4, atol=3e-5)
        np.testing.assert_allclose(_n(out), ref.numpy(), rtol=3e-4, atol=3e-5)
    out, feat = sb.ops.generator_forward_unfused(x.cuda(), "bnc", conv, fc, True)  # stand-alone encoder / FC-head entry points
    np.testing.assert_allclose(_n(feat), ref.numpy(), rtol=3e-4, atol=3e-5)
    np.testing.assert_allclose(_n(out), ref.numpy(), rtol=3e-4, atol=3e-5)
    # a batch beyond one warp of rows (FC head row groups) and BCN input
    xb = torch.randn(70, 3, 130)
    y = xb
    for i in range(5):
        y = F.relu(F.batch_norm(F.conv1d(y, Ws[i][:, :, None], bs[i]), None, None, gs[i], be[i], True, 0.0, 1e-3))
    refb = y.max(2)[0]
    fc2 = [dict(weight=(torch.randn(40, 128) / 11).cuda(), bias=torch.randn(40).cuda(), bn=((1 + 0.1 * torch.randn(40)).cuda(), torch.randn(40).cuda(), None, None, 1e-5, 0.1), relu=True)]
    refo = F.relu(F.batch_norm(F.linear(refb, fc2[0]["weight"].cpu(), fc2[0]["bias"].cpu()), None, None, fc2[0]["bn"][0].cpu(), fc2[0]["bn"][1].cpu(), True, 0.0, 1e-5))
    for kw in (dict(), dict(exact_fp32=True)):
        out, feat = sb.ops.generator_forward(xb.cuda(), "bcn", conv, fc2, True, **kw)
        np.testing.assert_allclose(_n(feat), refb.numpy(), rtol=3e-4, atol=3e-5)
        np.testing.assert_allclose(_n(out), refo.numpy(), rtol=1e-3, atol=1e-4)


# ------------------------------------------------------------------------------------------------ losses
def test_simplification_loss_fused_and_tf_names(sb, oracle):
    r = _rng(21)
    ref = r.standard_normal((4, 1024, 3)).astype(np.float32)
    samp = (ref[:, :64] + 0.1 * r.standard_normal((4, 64, 3))).astype(np.float32)
    for gamma, delta in ((1, 0), (0.5, 0.01)):
        out = sb.tf_ops.get_simplification_loss(_t(ref), _t(samp), 64, gamma, delta)
        np.testing.assert_allclose(float(out), float(oracle.simplification_loss(ref, samp, 64, gamma, delta, contract=True)), rtol=3e-6)
    d1, i1, d2, i2 = sb.tf_ops.nn_distance(_t(samp), _t(ref))
    e1, j1, e2, j2 = oracle.nn_distance(samp, ref, contract=True)
    assert np.array_equal(_n(i1), j1) and np.array_equal(_n(d2), e2) and i1.dtype == torch.int32
    # autograd of the fused loss == autograd of the composed torch expression over ChamferDistance
    s1 = _t(samp).requires_grad_(True); s2 = _t(samp).requires_grad_(True)
    sb.tf_ops.get_simplification_loss(_t(ref), s1, 64, 1, 0).backward()
    c12, c21 = sb.ChamferDistance()(s2, _t(ref))
    (c12.mean() + c12.max(dim=1)[0].mean() + c21.mean()).backward()
    np.testing.assert_allclose(_n(s1.grad), _n(s2.grad), rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("n,m", [(64, 64), (96, 32), (40, 120), (77, 77), (300, 300), (1024, 1024)])
def test_emd_exact_mode_bitexact_vs_oracle(sb, oracle, n, m):
    """north_star: match ASSIGNMENTS bit-exact.  approx_match(exact=True) (C flag SNB200_EMD_EXACT; env SNB200_EMD_EXACT_EXP=1) evaluates
    the reference's level schedule with the oracle's arithmetic operation for operation (correctly rounded exp, index-order float sums, no
    FMA contraction): the whole `match` tensor -- hence every arg-max assignment -- equals the oracle's bit for bit, and the assignments
    equal those of the reference's own CPU code (oracle/_ref approxmatch_cpu, double accumulators) on these tie-free random inputs."""
    r = _rng(n * 13 + m)
    b = 3 if n < 1024 else 2
    a = r.random((b, n, 3)).astype(np.float32)
    c = r.random((b, m, 3)).astype(np.float32)
    mt = _n(sb.tf_ops.approx_match(_t(a), _t(c), exact=True))
    omt = oracle.approx_match(a, c)
    assert mt.shape == omt.shape == (b, m, n)
    assert np.array_equal(mt.argmax(axis=2), omt.argmax(axis=2)) and np.array_equal(mt.argmax(axis=1), omt.argmax(axis=1))
    assert np.array_equal(mt, omt), np.abs(mt - omt).max()
    if n <= 300:   # the assignments of the reference's own CPU code on these inputs
        assert np.array_equal(mt.argmax(axis=2), REF_CPU["emd_assign_%d_%d" % (n, m)])
    # the fast kernel against the exact one: same assignments wherever the exact top-2 gap exceeds the fast kernel's value tolerance
    fast = _n(sb.tf_ops.approx_match(_t(a), _t(c)))
    tol = 2e-3 if n <= 300 else 1e-2      # (the reference's own GPU-vs-CPU self-check flags > 1e-2, approxmatch.cpp:222; the error grows with n)
    assert np.abs(fast - mt).max() < tol
    am, ao = fast.argmax(axis=2), mt.argmax(axis=2)
    gap = np.take_along_axis(mt, ao[..., None], 2)[..., 0] - np.take_along_axis(mt, am[..., None], 2)[..., 0]
    assert (gap < tol).all()


@pytest.mark.parametrize("n,m", [(64, 64), (96, 32), (40, 120), (77, 77), (300, 300), (2048, 2048)])
def test_emd_vs_oracle(sb, oracle, n, m):
    r = _rng(n * 7 + m)
    b = 3 if n == 77 else (2 if n < 2048 else 1)   # (3 x 77 rows: the persistent grid's row chunks straddle cloud boundaries)
    a = r.random((b, n, 3)).astype(np.float32)
    c = r.random((b, m, 3)).astype(np.float32)
    mt = sb.tf_ops.approx_match(_t(a), _t(c))
    assert mt.shape == (b, m, n)
    omt = oracle.approx_match(a, c)
    # same algorithm, different summation order + exp2f vs expf: the reference flags |diff| > 1e-2 (approxmatch.cpp:222)
    assert np.abs(_n(mt) - omt).max() < 2e-3
    # match assignments: the strongest partner of every xyz2 point agrees, except where the oracle's own top two weights are
    # closer than the value tolerance above (then either is "the" assignment)
    am, ao = np.argmax(_n(mt), axis=2), np.argmax(omt, axis=2)
    gap = np.take_along_axis(omt, ao[..., None], 2)[..., 0] - np.take_along_axis(omt, am[..., None], 2)[..., 0]
    assert (gap < 2e-3).all() and (am == ao).mean() > 0.97
    # on IDENTICAL match input the cost and gradient kernels are compared tightly
    x1 = _t(a).requires_grad_(True); x2 = _t(c).requires_grad_(True)
    cost = sb.tf_ops.match_cost(x1, x2, _t(omt))
    np.testing.assert_allclose(_n(cost), oracle.match_cost(a, c, omt), rtol=2e-5)
    gw = r.random(b).astype(np.float32)
    (cost * _t(gw)).sum().backward()
    g1, g2 = oracle.match_cost_grad(a, c, omt)
    np.testing.assert_allclose(_n(x1.grad), g1 * gw[:, None, None], rtol=2e-4, atol=2e-5)
    np.testing.assert_allclose(_n(x2.grad), g2 * gw[:, None, None], rtol=2e-4, atol=2e-5)
    # conservation: the smaller side is fully assigned
    tot = _n(mt).sum(axis=1) if n <= m else _n(mt).sum(axis=2)
    np.testing.assert_allclose(tot, max(n, m) // min(n, m), rtol=3e-3)



# ------------------------------------------------------------------------------------------------ full sizes vs the oracle, bit-exact
@pytest.mark.parametrize("b,n,m,k", [(32, 1024, 64, 8), (32, 1024, 1024, 7), (50, 2048, 2048, 16)])
def test_full_size_bitexact_vs_oracle(sb, oracle, b, n, m, k):
    """BASELINE.json's full sizes (headline reg, progressive cls, rec AE) against the C oracle: Chamfer indices + distances and kNN
    indices + distances BIT-EXACT in both arithmetic modes; projection / weights / simplification loss within fp32 tolerance; the
    fused tail (projection + Chamfer + loss in one launch) identical to the stand-alone kernels."""
    r = _rng(b + n + m + k)
    x = (r.random((b, n, 3)) - 0.5).astype(np.float32)
    q = (x[:, r.permutation(n)[:m]] + 0.02 * r.standard_normal((b, m, 3))).astype(np.float32)
    xt, qt = _t(x), _t(q)
    for unfused in (False, True):
        d1, i1, d2, i2 = sb.ops.nn_distance_forward(qt, xt, unfused=unfused)
        od1, oi1, od2, oi2 = oracle.nn_distance(q, x, contract=not unfused)
        assert np.array_equal(_n(i1), oi1) and np.array_equal(_n(i2), oi2)
        assert np.array_equal(_n(d1), od1) and np.array_equal(_n(d2), od2)
    sigma = 0.05
    o = sb.ops.knn_soft_project_forward(xt, qt, k, "bnc", torch.tensor([sigma], device="cuda"), want=("proj", "idx", "val", "weights", "dist"))
    ov, oi = oracle.knn_point(k, x, q, contract=True, tie_mode=1)
    assert np.array_equal(_n(o["idx"]), oi) and np.array_equal(_n(o["val"]), ov)
    pr, w, dd = oracle.soft_project(x, q, oi, sigma)
    np.testing.assert_allclose(_n(o["proj"]), pr, rtol=1e-5, atol=2e-6)
    np.testing.assert_allclose(_n(o["weights"]), w.reshape(b, m, k), rtol=2e-5, atol=1e-7)
    loss = sb.ops.simplification_loss_forward(qt, xt, 1.0)[0]
    ref = oracle.simplification_loss(x, q, m, 1, 0, contract=True)
    assert abs(float(loss[3]) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref)))   # north_star bar
    if k <= 32 and n <= 4096 and m <= 4096:
        t = torch.tensor([0.4], device="cuda")
        pj, idx, ww, dk, fd1, fi1, fd2, fi2, out4 = sb.ops.project_and_loss_forward(xt, qt, k, t, 1, 1e-2, 1.0)
        assert np.array_equal(_n(idx), oi) and np.array_equal(_n(fi1), oracle.nn_distance(q, x, contract=True)[1])
        assert np.array_equal(_n(fd1), oracle.nn_distance(q, x, contract=True)[0]) and np.array_equal(_n(fi2), oracle.nn_distance(q, x, contract=True)[3])
        assert abs(float(out4[3]) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref)))
        pr2, _, _ = oracle.soft_project(x, q, oi, 0.16)
        np.testing.assert_allclose(_n(pj), pr2, rtol=1e-5, atol=2e-6)


def test_samplenet_headline_vs_reference_fixture(sb, golden_dir):
    """The HEADLINE size (B=32, N=1024 -> 64, k=8) against the reference's own classes (tests/golden/make_golden.py fixture 4; weights of
    fixture 1): generator, projection, both losses, the running statistics and EVERY parameter gradient of
    0.01 * loss_s + 0.01 * loss_p + sum(proj * rw).

    Tolerances.  The reference's fp32 CPU run and this library's 3xTF32 + fp32 run both approximate the exact (fp64) network; the
    fixture carries the fp64 evaluation, so the generator is asked to be no further from the truth than 2x the reference itself, plus a
    direct bound.  Everything downstream of `simp` is compared on IDENTICAL inputs (the reference's own simp) at tight tolerances, and
    the whole step end to end at the loss level with the north_star 1e-5 bar relaxed only by the measured generator noise."""
    z = np.load(os.path.join(golden_dir, "samplenet_reg_b32.npz"))
    z2 = np.load(os.path.join(golden_dir, "samplenet_reg_b2.npz"))
    net = _load_net(sb, z2, input_shape="bnc", output_shape="bnc").train()
    x = _t(z["x"])
    simp, proj = net(x)
    err_ref = np.abs(z["simp"].astype(np.float64) - z["simp_fp64"]).max()
    err_ours = np.abs(_n(simp).astype(np.float64) - z["simp_fp64"]).max()
    assert err_ours <= 2.0 * err_ref + 1e-6, (err_ours, err_ref)
    np.testing.assert_allclose(_n(simp), z["simp"], rtol=0, atol=5e-5)
    # end to end the projection is discontinuous where a generated point's k-th and (k+1)-th neighbours swap under 1e-6 perturbations of simp:
    # all but a handful of the 2048 projected points must agree tightly (identical-input comparisons follow)
    bad_pts = (np.abs(_n(proj) - z["proj"]).max(axis=2) > 2e-4).sum()
    assert bad_pts <= 8, bad_pts
    loss_e2e = net.get_simplification_loss(x, simp, 64, 1, 0)
    assert abs(float(loss_e2e) - float(z["loss_simplification"])) < 2e-5 * max(1.0, abs(float(z["loss_simplification"])))
    # identical inputs: the reference's own simp
    simp_ref = _t(z["simp"]).requires_grad_(True)
    # the fixture's kNN stand-in evaluates distances without FMA contraction (torch CPU): in that arithmetic mode the projection agrees
    # everywhere; in the default mode (the reference CUDA kernels' contraction) a point whose 8th / 9th neighbours are 1 ulp apart may switch
    sig = net.project.sigma().detach().reshape(1)
    pu = sb.ops.knn_soft_project_forward(x, simp_ref.detach(), 8, "bnc", sig, want=("proj",), unfused=True)["proj"]
    np.testing.assert_allclose(_n(pu), z["proj"], rtol=2e-6, atol=2e-6)
    proj_id = net.project.project(x, simp_ref.detach(), layout="bnc")
    assert (np.abs(_n(proj_id) - z["proj"]).max(axis=2) > 2e-6).sum() <= 4
    loss_s = net.get_simplification_loss(x, simp_ref, 64, 1, 0)
    assert abs(float(loss_s.detach()) - float(z["loss_simplification"])) < 1e-5 * max(1.0, abs(float(z["loss_simplification"])))   # north_star bar
    np.testing.assert_allclose(_n(net.get_projection_loss()), z["loss_projection"], rtol=1e-6)
    (0.01 * loss_s).backward()
    np.testing.assert_allclose(_n(simp_ref.grad), z["grad_simp"], rtol=2e-4, atol=1e-8)
    # whole training step: every parameter's gradient norm, and a few gradients element-wise
    net.zero_grad()
    simp2, proj2 = net(x)
    (0.01 * net.get_simplification_loss(x, simp2, 64, 1, 0) + 0.01 * net.get_projection_loss() + (proj2 * _t(z["rw"])).sum()).backward()
    for name, p in net.named_parameters():
        ref = float(z["gnorm_" + name])
        got = float(p.grad.double().norm())
        # conv/fc biases in front of a training-mode BatchNorm (and bn5's shift, removed by bn_fc1's mean subtraction) have an exactly-zero
        # true gradient: both sides hold rounding noise there
        zero_true = name in ("conv1.bias", "conv2.bias", "conv3.bias", "conv4.bias", "conv5.bias", "fc1.bias", "fc2.bias", "fc3.bias", "bn5.bias")
        if zero_true or ref < 1e-4:
            assert got < 1e-2 and ref < 1e-2, (name, got, ref)
        elif name == "project._temperature":
            # ONE 8th/9th-neighbour switch moves this scalar by 10 %: on the fixture, perturbing the reference's own simp by 1e-7 flips it
            # between -0.379 and -0.417 in plain torch fp32.  Checked below on the kernel's own neighbour sets instead.
            assert 0.7 * ref <= got <= 1.3 * ref, (name, got, ref)
        else:   # end to end the step is discontinuous (kNN neighbour switches, max-pool / ReLU routing under 1e-6 perturbations of the forward):
            # norms within 1 %; the backward kernels themselves are held to 2e-4 against float64 in test_generator_cuda_backward_vs_float64_autograd
            assert abs(got - ref) <= 1e-2 * ref + 1e-6, (name, got, ref)
    # element-wise: a neighbour switch at one generated point moves the gradient of that point's three coordinates (and whatever they feed)
    # by a finite amount, so a few elements may sit outside the band; the bulk must agree
    def bulk_close(got, ref, rtol, atol, max_bad_frac):
        got, ref = _n(got).astype(np.float64), np.asarray(ref, dtype=np.float64)
        bad = np.abs(got - ref) > atol + rtol * np.abs(ref)
        assert bad.mean() <= max_bad_frac, (float(bad.mean()), float(np.abs(got - ref).max()))
    bulk_close(net.fc4.bias.grad, z["grad_fc4_bias"], 1e-2, 1e-3, 0.06)
    for got, key in ((net.conv1.weight.grad, "grad_conv1_weight"), (net.bn3.weight.grad, "grad_bn3_weight"),
                     (net.fc2.weight.grad[:4], "grad_fc2_weight_rows"), (net.conv4.weight.grad[:4], "grad_conv4_weight_rows")):
        bulk_close(got, z[key], 2e-2, 2e-2 * float(np.abs(z[key]).max()), 0.02)
    # temperature gradient on fixed routing: the kernel's own neighbour indices, torch float64 autograd of softmax(-d / sigma) . neighbours
    net.zero_grad()
    rw = _t(z["rw"])
    sq = _t(z["simp"])
    o = sb.ops.knn_soft_project_forward(x, sq, 8, "bnc", net.project.sigma().detach().reshape(1), want=("idx",))
    pj = net.project.project(x, sq, layout="bnc")
    ((pj * rw).sum() + 0.01 * net.get_projection_loss()).backward()
    T = net.project._temperature.detach().double().clone().requires_grad_(True)
    xd, qd = x.double(), sq.double()
    nb = torch.gather(xd[:, None].expand(-1, 64, -1, -1), 2, o["idx"].long()[..., None].expand(-1, -1, -1, 3))
    sg = torch.clamp(T ** 2, min=1e-4)
    w = torch.softmax(-((qd[:, :, None, :] - nb) ** 2).sum(-1) / sg, dim=2)
    ((w[..., None] * nb).sum(2) * rw.double()).sum().add(0.01 * sg).backward()
    assert abs(float(net.project._temperature.grad) - float(T.grad)) <= 2e-4 * abs(float(T.grad)), (float(net.project._temperature.grad), float(T.grad))
    # running statistics after ONE training forward of a fresh net
    net1 = _load_net(sb, z2, input_shape="bnc", output_shape="bnc").train()
    net1(x)
    np.testing.assert_allclose(_n(net1.bn5.running_mean), z["after_bn5_running_mean"], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(_n(net1.bn5.running_var), z["after_bn5_running_var"], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(_n(net1.bn_fc3.running_var), z["after_bn_fc3_running_var"], rtol=2e-3, atol=1e-6)


@pytest.mark.parametrize("ncl", [1, 2])
def test_registration_step_vs_reference_action_fixture(sb, golden_dir, ncl):
    """One registration training step's loss assembly (samplenet_b200.registration.RegistrationStep) against the reference's own
    `Action.compute_samplenet_loss / compute_pcrnet_loss / compute_sampling_consistency` (registration/main.py:500-598) run on CPU
    through tests/golden/make_golden.py (fixture 5).  PCRNet is rebuilt from the same seed; the sampler carries fixture 1's weights."""
    from samplenet_b200.registration import RegistrationStep

    z = np.load(os.path.join(golden_dir, "registration_step_c%d.npz" % ncl))
    z2 = np.load(os.path.join(golden_dir, "samplenet_reg_b2.npz"))
    act = RegistrationStep(num_sampled_clouds=ncl, alpha=float(z["alpha"]), lmbda=float(z["lmbda"]))
    torch.manual_seed(11)
    model = act.create_model()
    model.sampler.load_state_dict({k[3:]: torch.from_numpy(z2[k]) for k in z2.files if k.startswith("sd_")})
    model = model.cuda()
    model.sampler.train()
    igt = {"vec": _t(z["igt_vec"]), "inversion": torch.tensor([False])}
    data = (_t(z["p0"]), _t(z["p1"]), igt)
    sl, sampled, info = act.compute_samplenet_loss(model, data, "cuda")
    # B=4: the FC head's BatchNorm over 4 rows amplifies generator rounding (see the B=2 fixture test); loss-level tolerances follow
    np.testing.assert_allclose(float(info["simplification_loss"]), float(z["simplification_loss"]), rtol=2e-3)
    np.testing.assert_allclose(float(info["projection_loss"]), float(z["projection_loss"]), rtol=1e-6)
    np.testing.assert_allclose(float(sl), float(z["samplenet_loss"]), rtol=2e-3)
    np.testing.assert_allclose(_n(sampled[1]), z["p1_out"], rtol=0, atol=2e-3)
    # task side on IDENTICAL sampled clouds (the reference's own outputs)
    ref_sampled = (_t(z["p0_out"]), _t(z["p1_out"]), igt)
    pl, pinfo = act.compute_pcrnet_loss(model, ref_sampled, "cuda")
    np.testing.assert_allclose(_n(pinfo["est_transform"].vec), z["twist"], rtol=2e-4, atol=2e-5)
    for key in ("chamfer_loss", "qnorm_loss", "norm_err", "trans_err", "rot_err"):
        np.testing.assert_allclose(float(pinfo[key]), float(z[key]), rtol=5e-4, atol=1e-6, err_msg=key)
    np.testing.assert_allclose(float(pl), float(z["pcrnet_loss"]), rtol=5e-4)
    cons = act.compute_sampling_consistency(ref_sampled, "cuda")
    np.testing.assert_allclose(float(cons), float(z["consistency"]), rtol=1e-5, atol=1e-8)
    if ncl == 2:   # the whole step backward (train_1): gradient norms of the sampler's parameters
        model.zero_grad()
        sl2, sampled2, _ = act.compute_samplenet_loss(model, data, "cuda")
        pl2, _ = act.compute_pcrnet_loss(model, sampled2, "cuda")
        (pl2 + sl2).backward()
        worst = 0.0
        for name, p in model.sampler.named_parameters():
            ref = float(z["gnorm_" + name])
            if ref > 1e-3:
                worst = max(worst, abs(float(p.grad.double().norm()) - ref) / ref)
        assert worst < 5e-2, worst    # (B=4 BatchNorm in the head: a loose, conditioning-limited bound; B=32 is checked at 2e-3 above)


# ------------------------------------------------------------------------------------------------ full-size properties
def test_full_size_properties(sb):
    """BASELINE sizes, checked through size-independent properties (the oracle would take minutes here)."""
    g = torch.Generator(device="cuda").manual_seed(0)
    for (b, n, m, k) in [(32, 1024, 64, 8), (32, 1024, 1024, 7), (50, 2048, 2048, 16)]:
        x = torch.rand(b, n, 3, device="cuda", generator=g) - 0.5
        q = x[:, torch.randperm(n, device="cuda")[:m]] + 0.02 * torch.randn(b, m, 3, device="cuda", generator=g)
        d1, i1, d2, i2 = sb.ops.nn_distance_forward(q, x)
        # (1) the reported distance is the distance to the reported index; (2) nothing is closer (torch.cdist bound)
        gq = torch.gather(x, 1, i1.long()[..., None].expand(-1, -1, 3))
        assert torch.allclose(((gq - q) ** 2).sum(-1), d1, rtol=1e-5, atol=1e-7)
        full = torch.cdist(q, x) ** 2
        assert bool((d1 <= full.min(2)[0] * (1 + 1e-4) + 1e-6).all()) and bool((d2 <= full.min(1)[0] * (1 + 1e-4) + 1e-6).all())
        # (3) symmetry: swapping the clouds swaps the outputs bit-exactly
        e2, j2, e1, j1 = sb.ops.nn_distance_forward(x, q)
        assert torch.equal(d1, e1) and torch.equal(i1, j1) and torch.equal(d2, e2) and torch.equal(i2, j2)
        # (4) kNN: sorted, first neighbour == Chamfer NN, weights sum to one, projection inside the neighbours' bounding box
        o = sb.ops.knn_soft_project_forward(x, q, k, "bnc", torch.tensor([0.05], device="cuda"), want=("proj", "idx", "val", "weights"))
        assert bool((o["val"][..., 1:] >= o["val"][..., :-1]).all())
        assert torch.equal(o["idx"][..., 0], i1) and torch.equal(o["val"][..., 0], d1)
        assert torch.allclose(o["weights"].sum(-1), torch.ones(b, m, device="cuda"), atol=1e-5)
        nb = torch.gather(x[:, None].expand(-1, m, -1, -1), 2, o["idx"].long()[..., None].expand(-1, -1, -1, 3))
        assert bool((o["proj"] <= nb.max(2)[0] + 1e-5).all()) and bool((o["proj"] >= nb.min(2)[0] - 1e-5).all())
        # (5) idempotence: projecting cloud points onto the cloud with k=1 returns them
        p1 = sb.ops.knn_soft_project_forward(x, x[:, :m].contiguous(), 1, "bnc", torch.tensor([1.0], device="cuda"))["proj"]
        assert torch.equal(p1, x[:, :m])


def test_cuda_graph_capture_of_a_step(sb, golden_dir):
    z = np.load(os.path.join(golden_dir, "samplenet_reg_b2.npz"))
    net = _load_net(sb, z, input_shape="bnc", output_shape="bnc").train()
    x = _t(z["x"])
    with torch.no_grad():
        simp0, proj0 = net(x); l0 = net.get_simplification_loss(x, simp0, 64)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            net(x)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            simp, proj = net(x); loss = net.get_simplification_loss(x, simp, 64)
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(simp, simp0) and torch.equal(proj, proj0) and torch.equal(loss, l0)


def test_graphed_step_and_host_pipeline_agree_with_eager(sb):
    """GraphedStep / PipelinedHostStep (two steps in flight, loss read-back inside the graph) return, batch by batch, exactly what the
    eager calls return -- BatchNorm running statistics advance identically, so the nets are cloned per path."""
    torch.manual_seed(0)
    nets = []
    for _ in range(3):
        torch.manual_seed(0)
        nets.append(sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train())
    g = torch.Generator().manual_seed(5)
    batches = [(torch.rand(8, 256, 3, generator=g) - 0.5).pin_memory() for _ in range(5)]
    eager = []
    with torch.no_grad():
        for xb in batches:
            x = xb.cuda()
            simp, _ = nets[0](x)
            eager.append(float(nets[0].get_simplification_loss(x, simp, 64)))
    step = sb.GraphedStep(nets[1], 8, 256)
    # the capture itself ran the step (warm-up + capture do not replay): restore the state the eager net started from
    nets[1].load_state_dict(nets[2].state_dict())
    graphed = [float(step(xb.cuda())[2]) for xb in batches]
    assert graphed == eager
    pipe = sb.PipelinedHostStep(nets[2], 8, 256)
    torch.manual_seed(0)
    fresh = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train()
    nets[2].load_state_dict(fresh.state_dict())
    piped = []
    for j, xb in enumerate(batches):
        if j >= 2:
            piped.append(pipe.finish())
        pipe.submit(xb); pipe.launch()
    piped += [pipe.finish(), pipe.finish()]
    assert piped == eager
    with pytest.raises(RuntimeError):
        pipe.finish()


def test_primed_generator_workspace_is_self_cleaning(sb):
    """SNB200_GEN_WORKSPACE_PRIMED: the persistent kernel cleans its own scratch, so repeated calls on one kept workspace give exactly
    the per-call-memset results -- also after a call that took a non-self-cleaning path on the same workspace."""
    torch.manual_seed(0)
    net = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train()
    conv, fc = net._layer_specs()
    g = torch.Generator().manual_seed(3)
    xs = [(torch.rand(32, 1024, 3, generator=g) - 0.5).cuda() for _ in range(3)]
    with torch.no_grad():
        want = [sb.ops.generator_forward(x, "bnc", conv, fc, True, 64)[0].clone() for x in xs]
        pw = sb.ops.PrimedWorkspaces()
        with sb.ops.primed_workspaces(pw):
            got = [sb.ops.generator_forward(x, "bnc", conv, fc, True, 64)[0].clone() for x in xs]
            sb.ops.generator_forward(xs[0], "bnc", conv, fc, True, 64, per_layer_kernels=True)       # dirties, then re-zeroes the head
            again = sb.ops.generator_forward(xs[1], "bnc", conv, fc, True, 64)[0].clone()
        assert len(pw.bufs) == 1
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert torch.equal(again, want[1])


def test_graphed_train_step_matches_eager_step(sb):
    """One captured training step (forward, losses, backward, Adam) == the same step issued eagerly: same loss, same updated weights."""
    def make():
        torch.manual_seed(0)
        return sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train()
    g = torch.Generator().manual_seed(9)
    xs = [(torch.rand(8, 256, 3, generator=g) - 0.5).cuda() for _ in range(3)]
    ref = make()
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    losses = []
    for x in xs:
        opt.zero_grad()
        simp, proj = ref(x)
        loss = 0.01 * ref.get_simplification_loss(x, simp, 64) + 0.01 * ref.get_projection_loss() + (proj * proj).mean() * 0.0 + proj.sum() * 0.0
        loss.backward(); opt.step()
        losses.append(float(loss))
    net = make()
    init = {k: v.clone() for k, v in net.state_dict().items()}
    step = sb.GraphedTrainStep(net, 8, 256, lr=1e-3)
    # warm-up + capture trained on the (zero) static buffer: rewind parameters, BatchNorm buffers and Adam's state
    net.load_state_dict(init)
    for st in step.optimizer.state.values():
        for v in st.values():
            if torch.is_tensor(v):
                v.zero_()
    got = [float(step(x)) for x in xs]
    np.testing.assert_allclose(got, losses, rtol=2e-4)
    # Parameters: Adam normalises every gradient by its own magnitude, so parameters whose true gradient is zero (biases in front
    # of a BatchNorm) random-walk by +-lr on rounding noise in BOTH runs; compare the ones with a real gradient.
    sd, rd = net.state_dict(), ref.state_dict()
    for k in ("fc4.weight", "fc4.bias", "project._temperature", "bn_fc3.weight"):
        a, r = _n(sd[k]).ravel(), _n(rd[k]).ravel()
        bad = np.abs(a - r) > 3e-4 + 1e-3 * np.abs(r)       # (single elements with a near-zero gradient also random-walk by +-lr per step)
        assert bad.mean() <= 1e-3 and np.abs(a - r).max() < 3.5e-3, (k, bad.sum(), np.abs(a - r).max())
        assert not torch.equal(sd[k], init[k]), k
    assert int(sd["bn1.num_batches_tracked"]) == int(rd["bn1.num_batches_tracked"]) == 3


def test_cpu_tensors_are_rejected(sb):
    with pytest.raises(RuntimeError):
        sb.ChamferDistance()(torch.zeros(1, 4, 3), torch.zeros(1, 4, 3))
    with pytest.raises(ValueError):
        sb.ops.knn_soft_project_forward(torch.zeros(1, 8, 3, device="cuda"), torch.zeros(1, 2, 3, device="cuda"), 33, "bnc", want=("idx",))
    with pytest.raises(ValueError):
        sb.ops.knn_soft_project_forward(torch.zeros(1, 4, 3, device="cuda"), torch.zeros(1, 2, 3, device="cuda"), 5, "bnc", want=("idx",))


# ------------------------------------------------------------------------------------------------ tensor-core layer bring-up
@pytest.mark.parametrize("rows,c_in,c_out", [(128, 64, 64), (300, 64, 128), (256, 128, 128), (128, 32, 64), (128, 128, 256)])
def test_tc_gemm_3xtf32(sb, rows, c_in, c_out):
    """wgmma tf32 x3 (hi/lo split) must reproduce an fp32 GEMM to ~1e-6 relative."""
    g = torch.Generator(device="cuda").manual_seed(rows + c_in + c_out)
    A = torch.randn(rows, c_in, device="cuda", generator=g)
    W = torch.randn(c_out, c_in, device="cuda", generator=g) / c_in ** 0.5
    bias = torch.randn(c_out, device="cuda", generator=g)
    ref = (A.double() @ W.double().T + bias.double())
    D = sb.ops.debug_tc_gemm(A, W, bias)
    torch.cuda.synchronize()
    err = (D.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 5e-6 * scale, (err, scale)


def test_fused_tail_matches_separate_kernels(sb, oracle):
    """projection + Chamfer + loss reductions in one launch == the stand-alone kernels, forward and backward; the cache in
    SampleNet only answers for the very tensors forward() returned."""
    torch.manual_seed(11)
    net = sb.SampleNet(64, 128, group_size=8, input_shape="bnc", output_shape="bnc").cuda().train()
    x = torch.rand(8, 1024, 3, device="cuda") - 0.5
    outs = []
    for fused in (True, False):
        net.fused_tail = fused
        net.zero_grad()
        simp, proj = net(x)
        loss = net.get_simplification_loss(x, simp, 64, 1, 0)
        loss2 = net.get_simplification_loss(x, simp, 64, 0.5, 0.01)
        (loss + 0.3 * loss2 + (proj ** 2).sum()).backward()
        outs.append((proj.detach().clone(), loss.detach().clone(), loss2.detach().clone(), net.fc4.weight.grad.clone(), net.project._temperature.grad.clone()))
    for a, c in zip(outs[0], outs[1]):
        np.testing.assert_allclose(_n(a), _n(c), rtol=2e-5, atol=1e-6)
    # oracle check of the fused launch itself, identical inputs
    xs = _n(x); ss = _n(simp)
    proj_f, idx_f, w_f, d_f, d1, i1, d2, i2, out4 = sb.ops.project_and_loss_forward(x, simp.detach(), 8, net.project._temperature, 1, 1e-2, 1.0)
    _, idx = oracle.knn_point(8, xs, ss, contract=True, tie_mode=1)
    assert np.array_equal(_n(idx_f), idx)
    e1, j1, e2, j2 = oracle.nn_distance(ss, xs, contract=True)
    assert np.array_equal(_n(i1), j1) and np.array_equal(_n(i2), j2) and np.array_equal(_n(d1), e1) and np.array_equal(_n(d2), e2)
    np.testing.assert_allclose(float(out4[3]), float(oracle.simplification_loss(xs, ss, 64, 1, 0, contract=True)), rtol=3e-6)
    # cache discipline: a different (equal-valued) tensor, or an in-place edit, must not be answered from the cache
    net.fused_tail = True
    simp, proj = net(x)
    l_hit = net.get_simplification_loss(x, simp, 64)
    l_miss = net.get_simplification_loss(x, simp.clone(), 64)
    np.testing.assert_allclose(float(l_hit), float(l_miss), rtol=1e-6)
    with torch.no_grad():
        simp.mul_(1.5)
    l_edit = net.get_simplification_loss(x, simp, 64)
    assert abs(float(l_edit) - float(l_hit)) > 1e-4
    # deterministic: the ticket counter is left at zero and two launches agree bit for bit
    a = sb.ops.project_and_loss_forward(x, ss_t := simp.detach(), 8, net.project._temperature, 1, 1e-2, 1.0)[-1].clone()
    c = sb.ops.project_and_loss_forward(x, ss_t, 8, net.project._temperature, 1, 1e-2, 1.0)[-1].clone()
    assert torch.equal(a, c) and int(sb.ops._ticket(x.device)) == 0


def test_rec_continued_fps_matches_reference_semantics(sb, oracle):
    """reconstruction's inference matching `simple_projection_and_continued_fps` (samplenet_pointnet_ae.py:494-549): restated in numpy
    line by line below (float64 distances, first-maximum arg-max, order-preserving unique) and compared exactly."""
    r = _rng(77)
    B, N, k = 5, 2048, 64
    pc = r.random((B, N, 3)).astype(np.float32)
    gen = (pc[:, r.permutation(N)[:k]] + 0.05 * r.standard_normal((B, k, 3))).astype(np.float32)
    _, idx1, _, _ = sb.ops.nn_distance_forward(_t(gen), _t(pc))
    idx = _n(idx1)
    idx[:, 5] = idx[:, 3]; idx[:, 17] = idx[:, 0]            # force duplicates
    out_pc, out_idx, nu = sb.sputils.simple_projection_and_continued_fps(_t(pc), _t(gen), _t(idx, torch.int32))

    def calc(p0, pts):
        return ((p0 - pts) ** 2).sum(axis=1)

    for ii in range(B):
        _, first = np.unique(idx[ii], return_index=True)
        best = idx[ii][np.sort(first)]
        t = best.size
        far = np.zeros((k, 3)); sel = np.zeros(k, dtype=int)
        far[:t] = pc[ii][best]; sel[:t] = best
        d = calc(far[0], pc[ii].astype(np.float64))
        for i in range(1, t):
            d = np.minimum(d, calc(far[i], pc[ii].astype(np.float64)))
        for i in range(t, k):
            sel[i] = np.argmax(d); far[i] = pc[ii][sel[i]]
            d = np.minimum(d, calc(far[i], pc[ii].astype(np.float64)))
        assert int(nu[ii]) == t
        assert np.array_equal(_n(out_idx[ii]), sel)
        assert np.array_equal(_n(out_pc[ii]), far.astype(np.float32))
