"""One small invocation of every kernel family through the public API -- the workload for compute-sanitizer
(memcheck / racecheck / synccheck / initcheck):   compute-sanitizer --tool racecheck python tools/sanitize_ops.py [families...]
Sizes are small: the sanitizers slow kernels 10-100x and the persistent kernels spin on grid barriers."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import samplenet_b200 as sb
from samplenet_b200 import tf_ops

fam = set(sys.argv[1:]) or {"chamfer", "softproj", "tail", "generator", "emd", "matching", "group", "train", "progressive", "fps", "layers", "frozen",
                                "wide", "augment", "pairs"}
torch.manual_seed(0)
dev = torch.device("cuda:0")
x = (torch.rand(4, 256, 3, device=dev) - 0.5)
q = (x[:, :32] + 0.02 * torch.randn(4, 32, 3, device=dev)).contiguous()
if "chamfer" in fam:
    a, b = q.clone().requires_grad_(True), x.clone().requires_grad_(True)
    d1, d2 = sb.ChamferDistance()(a, b)
    (d1.mean() + d2.mean()).backward()
    tf_ops.nn_distance(q, x)
    print("chamfer ok")
if "softproj" in fam:
    sp = sb.SoftProjection(8, 1.0).to(dev)
    pc, qc = x.permute(0, 2, 1).contiguous().requires_grad_(True), q.permute(0, 2, 1).contiguous().requires_grad_(True)
    feats = torch.rand(4, 5, 256, device=dev, requires_grad=True)
    pr, prop = sp(pc, qc, feats, action="project_and_propagate")
    (pr.sum() + prop.sum()).backward()
    tf_ops.knn_point(7, x, q)
    print("softproj ok")
if "group" in fam:
    _, idx = tf_ops.knn_point(4, x, q)
    pts = x.clone().requires_grad_(True)
    tf_ops.group_point(pts, idx).sum().backward()
    print("group ok")
if "generator" in fam or "tail" in fam or "train" in fam:
    net = sb.SampleNet(32, 128, group_size=8, input_shape="bnc", output_shape="bnc").to(dev).train()
    if "generator" in fam:
        with torch.no_grad():
            conv, fc = net._layer_specs()
            sb.ops.generator_forward(x, "bnc", conv, fc, True, 32)
            sb.ops.generator_forward(x, "bnc", conv, fc, True, 32, per_layer_kernels=True)
            sb.ops.generator_forward(x, "bnc", conv, fc, True, 32, exact_fp32=True)
            net.eval(); net(x); net.train()
        print("generator ok")
    if "tail" in fam:
        with torch.no_grad():
            simp, proj = net(x)
            net.get_simplification_loss(x, simp, 32)
        print("tail ok")
    if "train" in fam:
        simp, proj = net(x)
        loss = net.get_simplification_loss(x, simp, 32) + 0.01 * net.get_projection_loss() + proj.sum() * 0.0
        loss.backward()
        print("train ok")
if "layers" in fam:   # the per-layer training path: snb200_generator_layers_* (256-wide conv layers, FC layers without BatchNorm / ReLU)
    # ReconstructionSampleNet(1401): at 4 clouds fc_bwd_kernel streams its 4203-wide output layer in two chunks, the second with a tail of 3
    for netl in (sb.ReconstructionSampleNet(16).to(dev).train(), sb.ClassificationSampleNet(16).to(dev).train(),
                 sb.ReconstructionSampleNet(1401).to(dev).train()):
        conv, fc = netl._layer_specs()
        assert sb.ops.generator_layers_backward_supported(x, "bnc", conv, fc)
        with torch.no_grad():
            out, _, saved = sb.ops.generator_layers_train_forward(x, "bnc", conv, fc, 0)
            sb.ops.generator_layers_backward(x, "bnc", conv, fc, saved, torch.randn_like(out), 0)
    print("layers ok")
if "emd" in fam:
    a = torch.rand(2, 96, 3, device=dev).requires_grad_(True)
    b = torch.rand(2, 64, 3, device=dev).requires_grad_(True)
    match = tf_ops.approx_match(a, b)
    tf_ops.match_cost(a, b, match).sum().backward()
    # the per-cloud route (approxmatch_kernel<false>, the rebuilt cost and gradient kernels): xyz2 repeated every 2 clouds, the vector
    # (n % 4 == 0) and scalar paths, m over two of the rebuilt kernels' 512-point tiles; then one gradient alone
    for n in (96, 97):
        a = torch.rand(4, n, 3, device=dev).requires_grad_(True)
        b = torch.rand(2, 600, 3, device=dev).requires_grad_(True)
        sb.ops.EMDCostFunction.apply(a, b).sum().backward()
        sb.ops.EMDCostFunction.apply(a, b.detach()).sum().backward()
        with torch.no_grad():
            sb.ops.emd_per_cloud(a, b)
    print("emd ok")
if "progressive" in fam:
    from samplenet_b200 import trainers
    so = torch.rand(4, 64, 3, device=dev, requires_grad=True)
    xr = x.clone().requires_grad_(True)
    trainers.progressive_simplification_loss(xr, so, [2, 4, 8, 16, 32, 64]).backward()
    print("progressive ok")
if "emd" in fam:
    tf_ops.approx_match(torch.rand(2, 48, 3, device=dev), torch.rand(2, 32, 3, device=dev), exact=True)
    print("emd exact ok")
if "multislice" in fam:   # more than 128 points per SM: every CTA of the persistent generator kernel walks two slices per layer (not in the default set:
    xb = torch.rand(40, 1024, 3, device=dev) - 0.5   # one CTA per SM x 512 threads under racecheck take minutes)
    netb = sb.SampleNet(32, 128, group_size=8, input_shape="bnc", output_shape="bnc").to(dev).train()
    simp, proj = netb(xb)
    (netb.get_simplification_loss(xb, simp, 32) + proj.sum() * 0.0).backward()
    print("multislice ok")
if "matching" in fam:
    _, idx1, _, _ = sb.ops.nn_distance_forward(q, x)
    sb.sputils.nn_matching_cuda(x, idx1, 32)
    print("matching ok")
if "fps" in fam:   # every configuration: 256 threads with coordinates in registers, 512 and 1024 reading them from shared memory
    for n, t in ((256, 256), (200, 512), (9000, 1024)):
        xs = torch.rand(2, n, 3, device=dev) - 0.5
        sb.ops.farthest_point_sample(xs, 40, return_points=True, _threads=t)
    pts = x.clone().requires_grad_(True)
    tf_ops.gather_point(pts, tf_ops.farthest_point_sample(300, x)).sum().backward()   # m > n: index 0 repeats
    print("fps ok")
if "frozen" in fam:   # the frozen task networks over prefixes: 1024-wide last layer in 4 channel blocks, prefixes off the 128-point tile grid;
    # then a last layer whose second block is partial, and the batch-statistics encoder
    from samplenet_b200 import tasknets
    for wrap, net in ((tasknets.FrozenPointNetCls, tasknets.PointNetCls()), (tasknets.FrozenPointNetAE, tasknets.PointNetAE(256))):
        w = wrap(net.to(dev).requires_grad_(False))
        xf = (torch.rand(2, 200, 3, device=dev) - 0.5).requires_grad_(True)
        w.prefixes(xf, [1, 7, 128, 129, 200]).sum().backward()
        with torch.no_grad():
            w(xf)
    # a 300-wide bottleneck (a 256-channel block and a 44-channel one), eval and batch statistics, forward and backward
    w = tasknets.FrozenPointNetAE(tasknets.PointNetAE(256, bneck_size=300).to(dev).requires_grad_(False))
    xf = (torch.rand(2, 200, 3, device=dev) - 0.5).requires_grad_(True)
    w.prefixes(xf, [1, 7, 128, 129, 200]).sum().backward()
    w.prefixes(xf, [1, 7, 128, 129, 200], batch_stats=True).sum().backward()
    print("frozen ok")
if "wide" in fam:   # bottleneck 320: a 256-channel block plus a partial one, two output slices of the wide backward; then eval at 1024
    netw = sb.SampleNet(32, 320, group_size=8, input_shape="bnc", output_shape="bnc").to(dev).train()
    xw = torch.rand(3, 200, 3, device=dev) - 0.5
    simp, proj = netw(xw)
    (netw.get_simplification_loss(xw, simp, 32) + proj.sum() * 0.0).backward()
    assert netw.generator_route == "layers", netw.generator_route
    with torch.no_grad():
        sb.SampleNet(32, 1024, group_size=8).to(dev).eval()(torch.rand(3, 3, 200, device=dev) - 0.5)
    print("wide ok")
if "augment" in fam:   # drawn angles with jitter, a partial last tile, fixed angles over replicas, in place
    xa = torch.rand(3, 300, 3, device=dev) - 0.5
    sb.ops.rotate_jitter(xa)
    sb.ops.rotate_by_angles(xa, [0.0, 1.0, 2.0])
    key = torch.empty(2, dtype=torch.int64, device=dev).random_()
    sb._lib.check(sb._lib.lib().snb200_rotate_jitter(3, 300, 1, xa.data_ptr(), xa.data_ptr(), None, key.data_ptr(), 0.01, 0.05,
                                                     torch.cuda.current_stream().cuda_stream), "rotate_jitter")
    print("augment ok")
if "pairs" in fam:   # n below one tile of keys (pads sort last), records wrapping past the set, with and without perm
    clouds = torch.rand(3, 300, 3, device=dev) - 0.5
    tr = torch.from_numpy(sb.registration.random_transforms(7, 0)).to(dev)
    rec = torch.tensor([6, 0, 4, 2], dtype=torch.int32, device=dev)
    sb.ops.registration_pairs(clouds, rec, tr, return_perm=True)
    sb.ops.registration_pairs(clouds, rec, tr)
    print("pairs ok")
torch.cuda.synchronize()
print("sanitize_ops done")
