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


def card_and_power_limit(dev):
    """(card name, power limit) of the device the numbers were taken on (nvidia-smi query; power limit "unknown" without it)."""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(dev.index)], capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return torch.cuda.get_device_name(dev), power


def cfg_sampler_training(dev, rounds=5):
    """The reconstruction and classification samplers' own training steps (ReconstructionSampleNet / ClassificationSampleNet on the
    per-layer CUDA path) against the same steps with generator_backward="torch" (torch recompute of the layer stack), alternating the two
    in one process: rec B=50, N=2048 -> 64, k=16, frozen PointNet AE (Chamfer and EMD AE loss); cls B=32, N=1024 -> 32, k=7, frozen
    PointNet classifier.  Eager steps (forward, losses, backward, Adam); median over `rounds` alternations."""
    from samplenet_b200 import trainers, tasknets
    torch.manual_seed(0)
    Br, Nr, Mr = 50, 2048, 64
    netr = sb.ReconstructionSampleNet(Mr, group_size=16).to(dev).train()
    ae = tasknets.PointNetAE(Nr, 128).to(dev)
    xr = clouds(Br, Nr, 13, dev)
    B, N, M = 32, 1024, 32
    netc = sb.ClassificationSampleNet(M, group_size=7).to(dev).train()
    cls = tasknets.PointNetCls().to(dev)
    x = clouds(B, N, 14, dev); y = torch.randint(0, 40, (B,), device=dev)
    cases = [
        ("rec sampler training step (ReconstructionSampleNet 2048->64, k=16) + frozen PointNet AE, Chamfer AE loss; B=50", Br, netr,
         lambda: trainers.ReconstructionStep(netr, ae, Mr).loss(xr)[0], 10),
        ("rec sampler training step (ReconstructionSampleNet 2048->64, k=16) + frozen PointNet AE, EMD AE loss; B=50", Br, netr,
         lambda: trainers.ReconstructionStep(netr, ae, Mr, ae_loss="emd").loss(xr)[0], 5),
        ("cls sampler training step (ClassificationSampleNet 1024->32, k=7) + frozen PointNet classifier; B=32", B, netc,
         lambda: trainers.ClassificationStep(netc, cls, M).loss(x, y)[0], 20),
    ]
    alternate_backward_routes(dev, cases, rounds)


def alternate_backward_routes(dev, cases, rounds):
    """Per case (name, batch, sampler, loss_fn, reps): eager steps (forward, losses, backward, Adam) with the sampler's CUDA backward and
    with generator_backward="torch", alternated in one process; one line with the medians over `rounds` alternations, the routes taken,
    the card and its power limit."""
    card, power = card_and_power_limit(dev)
    for name, b, net, loss_fn, reps in cases:
        opt = torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=1e-4)

        def one():
            opt.zero_grad(set_to_none=True)
            loss = loss_fn()
            loss.backward()
            opt.step()
            return loss
        times, routes = {"cuda": [], "torch": []}, {}
        for _ in range(rounds):
            for mode in ("cuda", "torch"):
                net.generator_backward = mode
                times[mode].append(time_us(one, reps=reps, warm=2))
                routes[mode] = net.generator_route
        net.generator_backward = "cuda"
        med = {k: sorted(v)[len(v) // 2] / 1e3 for k, v in times.items()}
        emit({"config": name, "card": card, "power_limit": power, "ms_per_step_cuda_backward": med["cuda"], "ms_per_step_torch_backward": med["torch"],
              "speedup": med["torch"] / med["cuda"], "clouds_per_s_cuda": b / (med["cuda"] * 1e-3), "generator_route": routes})


def cfg_progressive_training(dev, rounds=5):
    """The progressive trainers' steps on the wide samplers, whose output layers (3072 and 6144 channels) the CUDA backward streams
    through shared memory: cls B=32, N=1024, ClassificationSampleNet(1024), k=7, frozen PointNet classifier on the prefixes 8..1024;
    rec B=50, N=2048, ReconstructionSampleNet(2048), k=16, frozen PointNet AE, Chamfer AE loss on the prefixes 16..2048.  CUDA backward
    and generator_backward="torch" alternated as in cfg_sampler_training."""
    from samplenet_b200 import trainers, tasknets
    torch.manual_seed(0)
    B, N, M = 32, 1024, 1024
    netc = sb.ClassificationSampleNet(M, group_size=7).to(dev).train()
    cls = tasknets.PointNetCls().to(dev)
    x = clouds(B, N, 15, dev); y = torch.randint(0, 40, (B,), device=dev)
    stepc = trainers.ProgressiveClassificationStep(netc, cls, 8, M)
    Br, Nr = 50, 2048
    netr = sb.ReconstructionSampleNet(Nr, group_size=16).to(dev).train()
    ae = tasknets.PointNetAE(Nr, 128).to(dev)
    xr = clouds(Br, Nr, 16, dev)
    stepr = trainers.ProgressiveReconstructionStep(netr, ae)
    alternate_backward_routes(dev, [
        ("progressive cls sampler training step (ClassificationSampleNet 1024->1024, k=7) + frozen PointNet classifier on 8 prefixes; B=32", B,
         netc, lambda: stepc.loss(x, y)[0], 5),
        ("progressive rec sampler training step (ReconstructionSampleNet 2048->2048, k=16) + frozen PointNet AE, Chamfer AE loss on 8 prefixes; "
         "B=50", Br, netr, lambda: stepr.loss(xr)[0], 5),
    ], rounds)


class fp32_only:
    """cuDNN / cuBLAS TF32 off inside the block (restored after)."""

    def __enter__(self):
        self.prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.prev
        return False


def cfg_frozen_tasknets(dev, rounds=5):
    """The four sampler training steps with the stock torch task network and with its CUDA frozen wrapper (tasknets.FrozenPointNetCls /
    FrozenPointNetAE: one shared pass over every prefix), alternated in one process, median over `rounds`: cls 1024 -> 32, progressive cls
    1024 -> 1024 on the prefixes 8..1024 (B=32), rec 2048 -> 64, progressive rec 2048 -> 2048 on the prefixes 16..2048 (B=50).  Also the
    task network's forward + backward alone on the prefixes, both ways.  Timings run the torch side with torch's default cuDNN TF32 setting,
    printed with each line; the two routes' losses and gradients are compared at the timed sizes with TF32 off (fp32 on both sides), the
    sampler gradients as the largest difference over all its tensors relative to the largest gradient entry."""
    import copy

    from samplenet_b200 import trainers, tasknets
    card, power = card_and_power_limit(dev)
    torch.manual_seed(0)
    B, N, Br, Nr = 32, 1024, 50, 2048
    x = clouds(B, N, 17, dev); y = torch.randint(0, 40, (B,), device=dev)
    xr = clouds(Br, Nr, 18, dev)
    cls = tasknets.PointNetCls().to(dev).requires_grad_(False).eval()
    ae = tasknets.PointNetAE(Nr, 128).to(dev).requires_grad_(False).eval()
    both = {"cls": (cls, tasknets.FrozenPointNetCls(cls)), "ae": (ae, tasknets.FrozenPointNetAE(ae))}
    psz_c, psz_r = [8 * 2 ** i for i in range(8)], [16 * 2 ** i for i in range(8)]
    steps = [
        ("cls step (ClassificationSampleNet 1024->32, k=7) + PointNet classifier; B=32", B, sb.ClassificationSampleNet(32, group_size=7), "cls",
         lambda s, t: trainers.ClassificationStep(s, t, 32).loss(x, y), 20),
        ("progressive cls step (ClassificationSampleNet 1024->1024, k=7) + PointNet classifier on 8 prefixes; B=32", B,
         sb.ClassificationSampleNet(1024, group_size=7), "cls", lambda s, t: trainers.ProgressiveClassificationStep(s, t, 8, 1024).loss(x, y), 5),
        ("rec step (ReconstructionSampleNet 2048->64, k=16) + PointNet AE, Chamfer AE loss; B=50", Br, sb.ReconstructionSampleNet(64, group_size=16),
         "ae", lambda s, t: trainers.ReconstructionStep(s, t, 64).loss(xr), 10),
        ("progressive rec step (ReconstructionSampleNet 2048->2048, k=16) + PointNet AE, Chamfer AE loss on 8 prefixes; B=50", Br,
         sb.ReconstructionSampleNet(2048, group_size=16), "ae", lambda s, t: trainers.ProgressiveReconstructionStep(s, t).loss(xr), 5),
    ]
    for name, b, net, kind, loss_fn, reps in steps:
        net = net.to(dev).train()
        # the two routes' outputs on the same sampler state, before any optimiser step
        res = {}
        with fp32_only():
            for way, task in zip(("torch", "frozen"), both[kind]):
                s = copy.deepcopy(net)
                loss = loss_fn(s, task)[0]
                loss.backward()
                res[way] = (float(loss), {k: p.grad.detach() for k, p in s.named_parameters() if p.grad is not None})
        gt = res["torch"][1]
        gdiff = max((res["frozen"][1][k] - g).abs().max().item() for k, g in gt.items()) / max(g.abs().max().item() for g in gt.values())
        opt = torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=1e-4)
        times = {"torch": [], "frozen": []}
        for _ in range(rounds):
            for way, task in zip(("torch", "frozen"), both[kind]):
                def one():
                    opt.zero_grad(set_to_none=True)
                    loss = loss_fn(net, task)[0]
                    loss.backward()
                    opt.step()
                    return loss
                times[way].append(time_us(one, reps=reps, warm=2))
        med = {k: sorted(v)[len(v) // 2] / 1e3 for k, v in times.items()}
        emit({"config": "frozen_tasknets: " + name, "card": card, "power_limit": power, "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32,
              "ms_per_step_torch_task_net": med["torch"], "ms_per_step_frozen_task_net": med["frozen"], "speedup": med["torch"] / med["frozen"],
              "clouds_per_s_frozen": b / (med["frozen"] * 1e-3),               "loss_rel_diff_fp32": abs(res["frozen"][0] - res["torch"][0]) / abs(res["torch"][0]), "sampler_grad_max_diff_fp32": gdiff})
    # the task network alone on the prefixes: forward + backward to the points
    for name, kind, xx, sizes in (("PointNet classifier on 8 prefixes 8..1024 of 32 x 1024", "cls", x, psz_c),
                                  ("PointNet AE encoder + decoder on 8 prefixes 16..2048 of 50 x 2048", "ae", xr, psz_r)):
        torch_net, frozen = both[kind]
        g = torch.randn(len(sizes), xx.shape[0], 40 if kind == "cls" else Nr * 3, device=dev)

        def run_torch():
            p = xx.detach().requires_grad_(True)
            outs = [torch_net(p[:, :s].contiguous()) for s in sizes]
            outs = [o[0] if kind == "cls" else o.reshape(o.shape[0], -1) for o in outs]
            torch.autograd.backward(outs, list(g))
            return p.grad

        def run_frozen():
            p = xx.detach().requires_grad_(True)
            out = frozen.prefixes(p, sizes)
            out.reshape(len(sizes), xx.shape[0], -1).backward(g)
            return p.grad
        times = {"torch": [], "frozen": []}
        for _ in range(rounds):
            times["torch"].append(time_us(run_torch, reps=10, warm=2))
            times["frozen"].append(time_us(run_frozen, reps=10, warm=2))
        with fp32_only():
            ga, gb = run_torch(), run_frozen()
        med = {k: sorted(v)[len(v) // 2] / 1e3 for k, v in times.items()}
        emit({"config": "frozen_tasknets: task network forward + backward alone, " + name, "card": card, "power_limit": power,
              "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32, "ms_torch": med["torch"], "ms_frozen": med["frozen"],
              "speedup": med["torch"] / med["frozen"], "grad_x_max_diff_fp32": ((ga - gb).abs().max() / ga.abs().max()).item()})


def cuda_kernels_per_call(fn):
    """CUDA kernels one call of fn launches, counted by a separate torch.profiler pass (not timed)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA and "emcpy" not in e.key and "emset" not in e.key)


def cfg_cls_transforms(dev, rounds=5):
    """PointNet with transform nets (the classification trainer's default classifier), plain torch module against its CUDA frozen wrapper
    (tasknets.FrozenPointNetClsTransforms), alternated in one process, median over `rounds`: the ClassificationStep with
    ClassificationSampleNet(32, k=7) at B=32, N=1024 (forward, losses, backward, Adam); the task network's forward + get_loss + backward to
    the points alone on 32 x 32 and 32 x 1024 points; forward-only evaluation on 32 x 1024.  CUDA kernels per call from a separate profiler
    pass.  The torch side runs with torch's default cuDNN TF32 setting, printed with each line."""
    from samplenet_b200 import trainers, tasknets
    card, power = card_and_power_limit(dev)
    torch.manual_seed(0)
    B, N, M = 32, 1024, 32
    net = tasknets.PointNetClsTransforms().to(dev).requires_grad_(False).eval()
    both = {"torch": net, "frozen": tasknets.FrozenPointNetClsTransforms(net)}
    x = clouds(B, N, 19, dev); y = torch.randint(0, 40, (B,), device=dev)
    sampler = sb.ClassificationSampleNet(M, group_size=7).to(dev).train()
    opt = torch.optim.Adam([p for p in sampler.parameters() if p.requires_grad], lr=1e-4)

    def step(task):
        def one():
            opt.zero_grad(set_to_none=True)
            loss = trainers.ClassificationStep(sampler, task, M).loss(x, y)[0]
            loss.backward()
            opt.step()
            return loss
        return one

    def fwd_bwd(task, pts):
        def one():
            p = pts.detach().requires_grad_(True)
            logits, ep = task(p)
            task.get_loss(logits, y, ep).backward()
            return p.grad
        return one

    def fwd(task, pts):
        def one():
            with torch.no_grad():
                return task(pts)[0]
        return one

    x32 = clouds(B, 32, 20, dev)
    cases = [("ClassificationStep, ClassificationSampleNet(1024->32, k=7) + PointNet with transform nets, B=32", step, 20),
             ("task network forward + get_loss + backward to the points, 32 x 32", lambda t: fwd_bwd(t, x32), 20),
             ("task network forward + get_loss + backward to the points, 32 x 1024", lambda t: fwd_bwd(t, x), 20),
             ("task network forward only, 32 x 1024", lambda t: fwd(t, x), 20)]
    for name, make, reps in cases:
        times = {"torch": [], "frozen": []}
        for _ in range(rounds):
            for way in ("torch", "frozen"):
                times[way].append(time_us(make(both[way]), reps=reps, warm=2))
        med = {k: sorted(v)[len(v) // 2] / 1e3 for k, v in times.items()}
        kern = {k: cuda_kernels_per_call(make(both[k])) for k in both}
        emit({"config": "cls_transforms: " + name, "card": card, "power_limit": power, "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32,
              "ms_torch": med["torch"], "ms_frozen": med["frozen"], "speedup": med["torch"] / med["frozen"],
              "cuda_kernels_torch": kern["torch"], "cuda_kernels_frozen": kern["frozen"]})


def cfg_wide_bottleneck(dev, rounds=5):
    """Samplers with a wide bottleneck (the trainers' --bottleneck-size / --bottleneck_size) at B=32, N=1024: the classification
    sampler's step (ClassificationSampleNet 1024->32, k=7, frozen PointNet classifier) at bottlenecks 1024 and 320 (a partial last
    output slice) and SampleNet(64, 1024)'s own losses (not RegistrationStep: PCRNet's cost is not the sampler's), each on the
    per-layer CUDA backward against generator_backward="torch", alternated; then the C=512 classification generator's training-mode forward
    on the tensor cores against generator_precision="fp32" (the exact CUDA-core conv stack), alternated, median over `rounds`."""
    from samplenet_b200 import trainers, tasknets
    torch.manual_seed(0)
    B, N = 32, 1024
    netc = sb.ClassificationSampleNet(32, bottleneck_size=1024, group_size=7).to(dev).train()
    cls = tasknets.PointNetCls().to(dev)
    x = clouds(B, N, 15, dev); y = torch.randint(0, 40, (B,), device=dev)
    netr = sb.SampleNet(64, 1024, 8, input_shape="bnc", output_shape="bnc").to(dev).train()
    # 320 = one full output slice of 256 channels and one of 64 that the wide backward runs at the full slice width
    net3 = sb.ClassificationSampleNet(32, bottleneck_size=320, group_size=7).to(dev).train()

    def reg_loss():
        simp, proj = netr(x)
        return netr.get_simplification_loss(x, simp, 64) + 0.01 * netr.get_projection_loss() + (proj * proj).mean()
    cases = [
        ("wide_bottleneck: cls sampler training step (ClassificationSampleNet 1024->32, k=7, bottleneck 1024) + frozen PointNet classifier; "
         "B=32", B, netc, lambda: trainers.ClassificationStep(netc, cls, 32).loss(x, y)[0], 10),
        ("wide_bottleneck: SampleNet(64, 1024) training step, simplification + projection losses; B=32, N=1024", B, netr, reg_loss, 10),
        ("wide_bottleneck: cls sampler training step (ClassificationSampleNet 1024->32, k=7, bottleneck 320) + frozen PointNet classifier; "
         "B=32", B, net3, lambda: trainers.ClassificationStep(net3, cls, 32).loss(x, y)[0], 10),
    ]
    alternate_backward_routes(dev, cases, rounds)
    card, power = card_and_power_limit(dev)
    net5 = sb.ClassificationSampleNet(32, bottleneck_size=512, group_size=7).to(dev).train()
    times = {"3xtf32": [], "fp32": []}
    for _ in range(rounds):
        for prec in ("3xtf32", "fp32"):
            net5.generator_precision = prec
            with torch.no_grad():
                times[prec].append(time_us(lambda: net5._generate(x, "bnc", 0), reps=20, warm=3))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    emit({"config": "wide_bottleneck: generator training-mode forward, classification table with bottleneck 512; B=32, N=1024", "card": card,
          "power_limit": power, "us_tensor_cores": med["3xtf32"], "us_fp32_cuda_cores": med["fp32"], "speedup": med["fp32"] / med["3xtf32"]})


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
        if rank == 0 and args.only in ("all", "sampler_training"):
            cfg_sampler_training(dev)
        if rank == 0 and args.only in ("all", "progressive_training"):
            cfg_progressive_training(dev)
        if rank == 0 and args.only in ("all", "frozen_tasknets"):
            cfg_frozen_tasknets(dev)
        if rank == 0 and args.only in ("all", "cls_transforms"):
            cfg_cls_transforms(dev)
        if rank == 0 and args.only in ("all", "wide_bottleneck"):
            cfg_wide_bottleneck(dev)
        if args.only in ("all", "train"):
            cfg_train(dev, rank, world)
        if args.only in ("all", "train", "registration"):
            cfg_registration_ddp(dev, rank, world)
    finally:
        if world > 1:
            torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
