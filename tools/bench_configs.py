"""Secondary configurations of BASELINE.json (configs[1..4]) -- one JSON line each.  Not the driver's bench (that is bench.py, the
headline metric); these lines document what the same kernels do at the classification / reconstruction / progressive shapes and
what a training step (forward + backward + flat-bucket all-reduce + Adam) costs.

    python tools/bench_configs.py                      # 1 GPU: cls, rec (+AE Chamfer/EMD), progressive, train step
    torchrun --nproc-per-node N ... tools/bench_configs.py --only train     # DDP training step on N GPUs (NCCL all-reduce)

Synthetic clouds (unit-cube normalised, seed fixed), random-init weights, fp32.  Timing: CUDA events, warm, R repetitions; the
forward+loss configurations replay a CUDA graph (as bench.py does), the training step and the kernel-level lines run eagerly.
"""
import argparse, json, os, sys, time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import samplenet_b200 as sb
from samplenet_b200 import ops, tf_ops

PEAKS = {"hbm_gbs": 6480.8}
try:
    mp = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
    PEAKS["hbm_gbs"] = float(mp["hbm_gbs"])
except Exception:
    pass


def clouds(b, n, seed, dev):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.rand(b, n, 3, generator=g) - 0.5
    x = x - x.mean(dim=1, keepdim=True)
    x = x / (x.abs().amax(dim=(1, 2), keepdim=True) * 2)
    return x.to(dev).contiguous()


def time_us(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record(); b.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def graph_us(fn, reps=10, replays=10):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn(); fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(replays):
        g.replay()
    b.record(); b.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * replays)


def emit(d):
    print(json.dumps(d), flush=True)


def cfg_cls(dev):
    """configs[1]: classification SampleNet N=1024->32, k=7 (train_samplenet.py:155-176): generator + projection + simplification loss."""
    B, N, M, K = 32, 1024, 32, 7
    torch.manual_seed(0)
    net = sb.SampleNet(M, 128, group_size=K, input_shape="bnc", output_shape="bnc").to(dev).train()
    x = clouds(B, N, 1, dev)
    step = sb.GraphedStep(net, B, N)
    us = time_us(lambda: step(x), reps=200, warm=20)
    emit({"config": "cls SampleNet fwd(train)+soft-proj+simplification loss, B=32, N=1024->32, k=7", "us_per_step": us, "clouds_per_s": B / (us * 1e-6),
          "launches_per_step": int(step.launches_per_step)})


def cfg_rec(dev):
    """configs[2]: reconstruction sampler N=2048->64, k=16 (samplers.py:22-36 widths) + AE losses Chamfer / EMD at 2048 x 2048, B=50."""
    B, N, M, K = 50, 2048, 64, 16
    torch.manual_seed(0)
    widths = [3, 64, 128, 128, 256, 128]
    fcw = [128, 256, 256, 256, 3 * M]
    convs = [torch.nn.Conv1d(widths[i], widths[i + 1], 1).to(dev) for i in range(5)]
    bns = [torch.nn.BatchNorm1d(widths[i + 1]).to(dev) for i in range(5)]
    fcs = [torch.nn.Linear(fcw[i], fcw[i + 1]).to(dev) for i in range(4)]
    fbns = [torch.nn.BatchNorm1d(256).to(dev) for _ in range(3)]
    bt = lambda bn: (bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum, bn.num_batches_tracked)
    conv_specs = [dict(weight=c.weight, bias=c.bias, bn=bt(b), relu=True) for c, b in zip(convs, bns)]
    fc_specs = [dict(weight=l.weight, bias=l.bias, bn=bt(fbns[i]) if i < 3 else None, relu=i < 3) for i, l in enumerate(fcs)]
    x = clouds(B, N, 2, dev)
    temp = torch.ones(1, device=dev)
    with torch.no_grad():
        def fwd():
            out, _ = ops.generator_forward(x, "bnc", conv_specs, fc_specs, True, M)
            simp = out.view(B, M, 3)
            return ops.project_and_loss_forward(x, simp, K, temp, 3, 1e-2, 1.0)
        us = graph_us(fwd, reps=5, replays=10)
        emit({"config": "rec sampler fwd(train, widths 64-128-128-256-128)+soft-proj(k=16, sigma=max(T,min)^2)+simplification loss, B=50, N=2048->64",
              "us_per_step": us, "clouds_per_s": B / (us * 1e-6),
              "note": "800 tiles and a 256-wide layer are outside the persistent conv-stack kernel's envelope: per-layer launches (wgmma where the layer shape allows, exact-fp32 CUDA cores otherwise)"})
        # AE losses on (reconstruction, ground truth) 2048 x 2048
        r = clouds(B, N, 3, dev)
        us_cd = graph_us(lambda: ops.nn_distance_forward(r, x), reps=5, replays=10)
        pairs = 2.0 * B * N * N
        emit({"config": "rec AE Chamfer nn_distance 2048<->2048, B=50", "us": us_cd, "clouds_per_s": B / (us_cd * 1e-6),
              "pair_evals_per_s": pairs / (us_cd * 1e-6), "pair_gflops": 8 * pairs / (us_cd * 1e-6) / 1e9,
              "hbm_gbs_algorithmic": B * (12 * 2 * N + 8 * 2 * N) / (us_cd * 1e-6) / 1e9, "bound": "fp32 issue (65 k pair evaluations per point pair of tiles vs 20 B/point)"})
        match = ops.approx_match(r, x)
        us_am = time_us(lambda: ops.approx_match(r, x), reps=5, warm=1)
        us_mc = time_us(lambda: ops.match_cost_forward(r, x, match), reps=10, warm=2)
        us_mg = time_us(lambda: ops.match_cost_grad(r, x, match), reps=10, warm=2)
        mbytes = B * N * N * 4
        exp_pairs = 30.0 * B * N * N     # 10 levels x 3 passes (SURVEY.md 8a8)
        emit({"config": "rec AE EMD approx_match n=m=2048, B=50", "us": us_am, "clouds_per_s": B / (us_am * 1e-6), "exp_pairs_per_s": exp_pairs / (us_am * 1e-6),
              "match_bytes": mbytes, "hbm_gbs_if_match_written_once": mbytes / (us_am * 1e-6) / 1e9, "bound": "MUFU (exp) / FMA: 126 M exp-pairs per cloud"})
        emit({"config": "rec AE EMD match_cost n=m=2048, B=50", "us": us_mc, "hbm_gbs": mbytes / (us_mc * 1e-6) / 1e9, "hbm_frac": mbytes / (us_mc * 1e-6) / 1e9 / PEAKS["hbm_gbs"],
              "bound": "hbm (reads match once: %.0f MB)" % (mbytes / 1e6)})
        emit({"config": "rec AE EMD match_cost_grad n=m=2048, B=50", "us": us_mg, "hbm_gbs": 2 * mbytes / (us_mg * 1e-6) / 1e9, "hbm_frac": 2 * mbytes / (us_mg * 1e-6) / 1e9 / PEAKS["hbm_gbs"],
              "bound": "hbm (reads match once per gradient side)"})


def cfg_progressive(dev):
    """configs[3]: SampleNetProgressive, M = N = 1024, k = 7, simplification loss summed over prefix sizes 8..1024
    (train_samplenet_progressive.py:157-224)."""
    B, N, M, K = 32, 1024, 1024, 7
    torch.manual_seed(0)
    net = sb.SampleNet(M, 128, group_size=K, input_shape="bnc", output_shape="bnc").to(dev).train()
    net.fused_tail = False
    x = clouds(B, N, 4, dev)
    sizes = [8, 16, 32, 64, 128, 256, 512, 1024]
    with torch.no_grad():
        def fwd():
            simp, proj = net(x)
            tot = 0
            for s in sizes:
                tot = tot + tf_ops.get_simplification_loss(x, simp[:, :s].contiguous(), s)
            return proj, tot
        us = graph_us(fwd, reps=3, replays=10)
    emit({"config": "progressive SampleNet fwd(train)+soft-proj(1024 queries, k=7)+simplification loss over prefixes 8..1024, B=32, N=1024->1024, one Chamfer launch per prefix",
          "us_per_step": us, "clouds_per_s": B / (us * 1e-6), "prefix_sizes": sizes})
    from samplenet_b200 import trainers
    with torch.no_grad():
        def fwd1():
            simp, proj = net(x)
            return proj, trainers.progressive_simplification_loss(x, simp, sizes)
        us1 = graph_us(fwd1, reps=3, replays=10)
        simp, _ = net(x)
        us_loss8 = graph_us(lambda: trainers.progressive_simplification_loss(x, simp, sizes, one_pass=False), reps=5, replays=10)
        us_loss1 = graph_us(lambda: trainers.progressive_simplification_loss(x, simp, sizes, one_pass=True), reps=5, replays=10)
    emit({"config": "progressive SampleNet fwd(train)+soft-proj(1024 queries, k=7)+ONE-PASS prefix loss (csrc/progressive.cu), B=32, N=1024->1024",
          "us_per_step": us1, "clouds_per_s": B / (us1 * 1e-6), "prefix_sizes": sizes, "loss_only_us_one_pass": us_loss1, "loss_only_us_per_prefix_launches": us_loss8})


def cfg_train(dev, rank, world):
    """configs[4]: training step, batch-sharded: forward + simplification/projection loss + backward + ONE flat-bucket all-reduce + Adam,
    32 clouds per GPU (registration/main.py:507-529 restated on synthetic clouds; the task network is out of scope)."""
    B, N, M, K = 32, 1024, 64, 8
    torch.manual_seed(0)
    net = sb.SampleNet(M, 128, group_size=K, input_shape="bnc", output_shape="bnc").to(dev).train()
    from samplenet_b200.parallel import FlatBucketDataParallel
    ddp = FlatBucketDataParallel(net)
    opt = torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=1e-3)
    xs = [clouds(B, N, 100 * rank + i, dev) for i in range(4)]

    def one(i):
        ddp.zero_grad()
        simp, proj = ddp(xs[i % 4])
        loss = net.get_simplification_loss(xs[i % 4], simp, M) + net.get_projection_loss() + (proj * proj).mean()
        loss.backward()
        ddp.sync_gradients()
        ddp.wait()
        opt.step()
        return loss

    for i in range(5):
        one(i)
    if world > 1:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    steps = 50
    a.record()
    for i in range(steps):
        one(i)
    b.record(); b.synchronize()
    ms = a.elapsed_time(b)
    if world > 1:
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        ms = float(t.item())
    # the same step captured in one CUDA graph
    torch.manual_seed(0)
    net2 = sb.SampleNet(M, 128, group_size=K, input_shape="bnc", output_shape="bnc").to(dev).train()
    gstep = sb.GraphedTrainStep(net2, B, N, lr=1e-3)
    for i in range(5):
        gstep(xs[i % 4])
    if world > 1:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    a.record()
    for i in range(steps):
        gstep(xs[i % 4])
    b.record(); b.synchronize()
    msg = a.elapsed_time(b)
    if world > 1:
        t = torch.tensor([msg], device=dev, dtype=torch.float64)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        msg = float(t.item())
    ar_us = None
    if world > 1:   # the collective alone: one all-reduce of the flat gradient bucket, back to back (device time, max over ranks)
        flat = ddp.flat_grad
        for _ in range(10):
            torch.distributed.all_reduce(flat)
        torch.distributed.barrier(); torch.cuda.synchronize()
        a.record()
        for _ in range(100):
            torch.distributed.all_reduce(flat)
        b.record(); b.synchronize()
        t = torch.tensor([a.elapsed_time(b) * 10.0], device=dev, dtype=torch.float64)   # us per all-reduce
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        ar_us = float(t.item())
    if rank == 0:
        emit({"config": "gradient all-reduce alone: flat bucket of %d bytes over NCCL (NVLink/NVSwitch), back to back" % ddp.bucket_bytes(), "n_gpus": world, "us_per_allreduce": ar_us})
    if rank == 0:
        emit({"config": "training step in ONE CUDA graph (samplenet_b200.GraphedTrainStep): fwd + losses + backward + flat-bucket all-reduce + Adam, 32 clouds/GPU",
              "n_gpus": world, "ms_per_step": msg / steps, "clouds_per_s": world * B * steps / (msg * 1e-3), "loss": float(gstep.loss),
              "library_launches_per_step": int(gstep.launches_per_step)})
    if rank == 0:
        emit({"config": "training step: SampleNet fwd + simplification/projection loss + backward + flat-bucket all-reduce (%d B) + Adam, 32 clouds/GPU, eager" % ddp.bucket_bytes(),
              "n_gpus": world, "ms_per_step": ms / steps, "clouds_per_s": world * B * steps / (ms * 1e-3),
              "note": "generator, Chamfer and projection backward are this library's kernels (csrc/generator_bwd.cu); eager launches, host-launch-bound"})


def cfg_task_steps(dev):
    """configs[1..3] END TO END with their (frozen) task networks: whole training steps -- sampler forward, task network forward, all losses,
    backward into the sampler, Adam -- eager, as the reference trainers run them (samplenet_b200.trainers / .registration / .tasknets)."""
    from samplenet_b200 import trainers, tasknets

    def run(name, B, loss_fn, params, reps=20):
        opt = torch.optim.Adam(params, lr=1e-3)

        def one():
            opt.zero_grad(set_to_none=True)
            loss = loss_fn()
            loss.backward()
            opt.step()
            return loss
        us = time_us(one, reps=reps, warm=5)
        emit({"config": name, "ms_per_step": us / 1e3, "clouds_per_s": B / (us * 1e-6), "loss": float(one())})

    torch.manual_seed(0)
    # classification: N=1024 -> 32, k=7, frozen PointNet classifier
    B, N, M = 32, 1024, 32
    net = sb.SampleNet(M, 128, group_size=7, input_shape="bnc", output_shape="bnc").to(dev).train()
    cls = tasknets.PointNetCls().to(dev)
    step = trainers.ClassificationStep(net, cls, M)
    x = clouds(B, N, 11, dev); y = torch.randint(0, 40, (B,), device=dev)
    run("cls training step end to end: SampleNet(1024->32,k=7) + frozen PointNet classifier, loss_cls + 30*simplification + projection, backward, Adam; B=32",
        B, lambda: step.loss(x, y)[0], [p for p in net.parameters() if p.requires_grad])
    # progressive classification: one generator pass, 8 prefixes
    Mp = 1024
    netp = sb.SampleNet(Mp, 128, group_size=7, input_shape="bnc", output_shape="bnc").to(dev).train()
    stepp = trainers.ProgressiveClassificationStep(netp, cls, 8, Mp)
    run("progressive cls training step end to end: SampleNet(1024->1024,k=7), classifier + one-pass prefix loss on 8 prefixes, backward, Adam; B=32",
        B, lambda: stepp.loss(x, y)[0], [p for p in netp.parameters() if p.requires_grad], reps=10)
    # reconstruction: N=2048 -> 64, k=16, frozen AE, Chamfer AE loss (EMD variant timed separately at the kernel level)
    Br, Nr, Mr = 50, 2048, 64
    netr = sb.SampleNet(Mr, 128, group_size=16, input_shape="bnc", output_shape="bnc").to(dev).train()
    ae = tasknets.PointNetAE(Nr, 128).to(dev)
    stepr = trainers.ReconstructionStep(netr, ae, Mr)
    xr = clouds(Br, Nr, 12, dev)
    run("rec training step end to end: SampleNet(2048->64,k=16) + frozen PointNet AE, Chamfer AE loss + simplification + projection, backward, Adam; B=50",
        Br, lambda: stepr.loss(xr)[0], [p for p in netr.parameters() if p.requires_grad], reps=10)
    stepe = trainers.ReconstructionStep(netr, ae, Mr, ae_loss="emd")
    run("rec training step end to end with the EMD AE loss (approx_match + match_cost 2048x2048); B=50",
        Br, lambda: stepe.loss(xr)[0], [p for p in netr.parameters() if p.requires_grad], reps=5)


def cfg_registration_ddp(dev, rank, world):
    """configs[4]: registration PCRNet + SampleNet, batch-sharded over the ranks (32 sample pairs per GPU: global B = 32 x world), the step of
    registration/main.py:306-362 (train_1) through samplenet_b200.registration.RegistrationStep: two sampler passes (template + source),
    frozen PCRNet, quaternion + Chamfer task loss, backward into the sampler, ONE flat-bucket NCCL all-reduce, Adam."""
    from samplenet_b200.registration import RegistrationStep, QuaternionTransform

    B, N = 32, 1024
    act = RegistrationStep(num_sampled_clouds=2)
    torch.manual_seed(0)
    model = act.create_model().to(dev)
    model.sampler.train()
    ddp = act.wrap_data_parallel(model)
    opt = torch.optim.Adam([p for p in model.sampler.parameters() if p.requires_grad], lr=1e-3)
    g = torch.Generator().manual_seed(100 + rank)
    p0 = clouds(B, N, 200 + rank, dev)
    quat = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=1).to(dev)
    vec = torch.cat([quat, torch.zeros(B, 3, device=dev)], dim=1)
    igt = {"vec": vec, "inversion": torch.tensor([False])}
    p1 = QuaternionTransform(vec).rotate(p0)
    data = (p0, p1, igt)
    for _ in range(5):
        act.train_step(model, data, opt, dev)
    if world > 1:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    steps = 30
    a.record()
    for _ in range(steps):
        loss, rot, _ = act.train_step(model, data, opt, dev)
    b.record(); b.synchronize()
    ms = a.elapsed_time(b)
    if world > 1:
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        ms = float(t.item())
    if rank == 0:
        emit({"config": "registration training step (PCRNet frozen + SampleNet, 2 sampled clouds, quaternion + Chamfer task loss), batch-sharded DDP, "
                        "global B = %d, flat-bucket all-reduce %d B, eager" % (B * world, ddp.bucket_bytes()),
              "n_gpus": world, "ms_per_step": ms / steps, "sample_pairs_per_s": world * B * steps / (ms * 1e-3), "loss": float(loss)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="all")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); lr = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device("cuda", lr)
    torch.cuda.set_device(dev)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=dev)
    try:
        if rank == 0 and args.only in ("all", "cls"):
            cfg_cls(dev)
        if rank == 0 and args.only in ("all", "rec"):
            cfg_rec(dev)
        if rank == 0 and args.only in ("all", "progressive"):
            cfg_progressive(dev)
        if rank == 0 and args.only in ("all", "tasks"):
            cfg_task_steps(dev)
        if args.only in ("all", "train"):
            cfg_train(dev, rank, world)
        if args.only in ("all", "train", "registration"):
            cfg_registration_ddp(dev, rank, world)
    finally:
        if world > 1:
            torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
