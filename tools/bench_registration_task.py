"""Measure the registration trainer's task half (frozen PCRNet + quaternion / Chamfer pose loss) plain against frozen_task=True.

    python tools/bench_registration_task.py [--steps 200] [--blocks 5] [--out DIR] [--num-sampled-clouds {1,2}]

One process, one GPU.  Builds RegistrationStep(num_sampled_clouds=2) (or 1: the sampled source against the full 1024-point template) at
B=32, N=1024 -> 64 twice from the same seed and the data of
tools/bench_configs.py's cfg_registration_ddp, warms both, then times alternating plain / frozen blocks with device events:
  (a) the task half alone: compute_pcrnet_loss on fixed sampled clouds + backward to the clouds;
  (b) the whole train_step.
Reports the median and the spread over the blocks, the CUDA kernels per step of each from a separate torch.profiler pass, the two new
kernel families' device time against the bytes their shapes imply (the MLP's weights once per pass), and the largest difference of the last
step's loss and sampled-cloud gradients between the variants.  Prints one JSON line.  Needs a GPU: it fails without one.

    python tools/bench_registration_task.py --train-pcrnet [--steps 50] [--blocks 5]

PCRNet's own training run instead: train_step of the plain module against create_model(cuda_task=True), Adam(lr=1e-3) over
filter(requires_grad, parameters()), at sampler="none" (B=32, N=1024: --train-pcrnet) and for the joint step (SampleNet 1024 -> 64 with
--train-pcrnet --train-samplenet), alternating blocks.  Reports the card and its power limit, the median and spread per variant, kernels
per step, the parameter-gradient kernels' device time against the bytes and FLOP their shapes imply, and the first step's differences in
loss and gradients (both variants from the same initial state).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

B, N, M = 32, 1024, 64
MLP_WIDTHS = [2048, 1024, 1024, 512, 512, 256, 7]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def make(frozen, dev, num_sampled_clouds=2):
    from bench_configs import clouds
    from samplenet_b200.registration import QuaternionTransform, RegistrationStep

    act = RegistrationStep(num_sampled_clouds=num_sampled_clouds)
    torch.manual_seed(0)
    model = act.create_model(frozen_task=frozen).to(dev)
    model.sampler.train()
    opt = torch.optim.Adam([p for p in model.sampler.parameters() if p.requires_grad], lr=1e-3)
    g = torch.Generator().manual_seed(100)
    p0 = clouds(B, N, 200, dev)
    quat = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=1).to(dev)
    vec = torch.cat([quat, torch.zeros(B, 3, device=dev)], dim=1)
    igt = {"vec": vec, "inversion": torch.tensor([False])}
    return act, model, opt, (p0, QuaternionTransform(vec).rotate(p0), igt)


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record(); b.synchronize()
    return a.elapsed_time(b) * 1e3 / steps     # us per step


def kernels_per_step(fn, steps=5, keys=("frozen_mlp_forward", "frozen_mlp_backward", "frozen_mlp_sum", "pose_loss_forward", "pose_loss_backward")):
    """(CUDA kernels per step, {kernel-name key: device us per step}) from a profiler pass of its own."""
    from torch.profiler import ProfilerActivity, profile

    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    count, fam = 0, {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and not ev.name.lower().startswith(("memcpy", "memset")):
            count += 1
            for key in keys:
                if key in ev.name:
                    fam[key] = fam.get(key, 0.0) + ev.device_time / steps
    return count / steps, fam


CONV_WIDTHS = [3, 64, 64, 64, 128, 1024]
PARAM_KERNELS = ("frozen_mlp_backward", "frozen_mlp_sum", "chain_bwd", "route_mark", "last_grad", "hidden_grad_partial", "reduce_partials")


def make_training(joint, cuda, dev, num_sampled_clouds=2):
    from bench_configs import clouds
    from samplenet_b200.registration import QuaternionTransform, RegistrationStep

    act = (RegistrationStep(num_out_points=M, num_sampled_clouds=num_sampled_clouds, train_pcrnet=True, train_samplenet=True) if joint
           else RegistrationStep(sampler="none", train_pcrnet=True))
    torch.manual_seed(0)
    model = act.create_model(cuda_task=cuda).to(dev)
    opt = torch.optim.Adam(filter(lambda p: p.requires_grad, model.parameters()), lr=1e-3)
    g = torch.Generator().manual_seed(100)
    p0 = clouds(B, N, 200, dev)
    quat = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=1).to(dev)
    vec = torch.cat([quat, torch.zeros(B, 3, device=dev)], dim=1)
    return act, model, opt, (p0, QuaternionTransform(vec).rotate(p0), {"vec": vec, "inversion": torch.tensor([False])})


def param_kernel_work(n_enc, rows):
    """Bytes and FLOP the parameter-gradient kernels' shapes imply per step: the encoder's dense dz rows written and read once, the hidden
    layers' dz^T a products over every point, the routed rows of conv4's output gathered once per (cloud, channel); the MLP's weight gradients
    written once, its dW products over `rows`, and its weights read once."""
    pts = 2 * rows * n_enc
    hid = CONV_WIDTHS[1:-1]
    enc_flop = 2 * pts * sum((CONV_WIDTHS[l] + 1) * CONV_WIDTHS[l + 1] for l in range(4)) + 2 * 2 * rows * CONV_WIDTHS[-1] * CONV_WIDTHS[-2]
    enc_bytes = 4 * (2 * pts * sum(hid) + 2 * rows * CONV_WIDTHS[-1] * CONV_WIDTHS[-2] + sum(CONV_WIDTHS[l] * CONV_WIDTHS[l + 1] for l in range(5)))
    mlp_params = sum(MLP_WIDTHS[i] * MLP_WIDTHS[i + 1] for i in range(6))
    return {"encoder_bytes": enc_bytes, "encoder_flop": enc_flop, "mlp_bytes": 4 * 2 * mlp_params, "mlp_flop": 2 * 2 * rows * mlp_params}


def train_pcrnet_main(args, dev):
    res = {"card": card(), "B": B, "N": N, "M": M, "steps_per_block": args.steps, "blocks": args.blocks}
    if args.num_sampled_clouds != 2:
        res["num_sampled_clouds"] = args.num_sampled_clouds
    for tag, joint in (("none", False), ("joint", True)):
        # first-step differences from the same initial state, with TF32 off (the plain module's convolutions allow it by default)
        tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        first = {}
        for cuda in (False, True):
            act, model, opt, data = make_training(joint, cuda, dev, args.num_sampled_clouds)
            loss, _, _ = act.train_step(model, data, opt, dev)
            net = model.net if cuda else model
            first[cuda] = (float(loss), {n: p.grad.double().clone() for n, p in net.named_parameters() if p.grad is not None})
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        (l0, g0), (l1, g1) = first[False], first[True]
        top = max(float(g.abs().max()) for g in g0.values())      # (a bias ahead of a BatchNorm: rounding noise, compared to the largest)
        rel = {n: float((g1[n] - g0[n]).abs().max()) / max(float(g0[n].abs().max()), 1e-3 * top) for n in g0}
        worst = max(rel, key=rel.get)
        res["%s_first_step" % tag] = {"loss_plain": l0, "loss_cuda": l1, "loss_rel_diff": abs(l1 - l0) / abs(l0), "worst_grad": worst,
                                      "worst_grad_rel_diff_of_max": rel[worst], "grads_compared": len(rel)}
        variants = {n: make_training(joint, n == "cuda", dev, args.num_sampled_clouds) for n in ("plain", "cuda")}
        fns = {n: (lambda v=v: v[0].train_step(v[1], v[3], v[2], dev)) for n, v in variants.items()}
        for n in fns:
            for _ in range(5):
                fns[n]()
        torch.cuda.synchronize()
        t = {n: [] for n in fns}
        for _ in range(args.blocks):
            for n in fns:
                t[n].append(timed(fns[n], args.steps))
        for n in fns:
            res["%s_%s_us" % (tag, n)] = {"median": statistics.median(t[n]), "min": min(t[n]), "max": max(t[n])}
        res["%s_speedup_of_medians" % tag] = res["%s_plain_us" % tag]["median"] / res["%s_cuda_us" % tag]["median"]
        for n in fns:
            k, fam = kernels_per_step(fns[n], keys=PARAM_KERNELS)
            res["%s_%s_kernels_per_step" % (tag, n)] = k
            if n == "cuda":
                res["%s_cuda_kernel_us_per_step" % tag] = fam
        work = param_kernel_work(M if joint else N, B)
        res["%s_param_kernel_work" % tag] = work
        fam = res["%s_cuda_kernel_us_per_step" % tag]
        enc_us = sum(fam.get(k, 0.0) for k in ("chain_bwd", "last_grad", "hidden_grad_partial", "reduce_partials"))
        mlp_us = fam.get("frozen_mlp_backward", 0.0) + fam.get("frozen_mlp_sum", 0.0)
        if enc_us:
            res["%s_encoder_backward_GBps_GFLOPs" % tag] = [work["encoder_bytes"] / enc_us * 1e-3, work["encoder_flop"] / enc_us * 1e-3]
        if mlp_us:
            res["%s_mlp_backward_GBps_GFLOPs" % tag] = [work["mlp_bytes"] / mlp_us * 1e-3, work["mlp_flop"] / mlp_us * 1e-3]
        del variants, fns
        torch.cuda.empty_cache()
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the dumped last-step tensors")
    ap.add_argument("--train-pcrnet", action="store_true", help="time PCRNet's training step (plain against cuda_task=True) instead")
    ap.add_argument("--num-sampled-clouds", type=int, choices=(1, 2), default=2,
                    help="2 samples template and source, 1 the source only (main.py --num-sampled-clouds)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_registration_task: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    if args.train_pcrnet:
        return train_pcrnet_main(args, dev)
    variants = {name: make(name == "frozen", dev, args.num_sampled_clouds) for name in ("plain", "frozen")}

    # fixed sampled clouds for the task half: the plain variant's projected points of its first forward
    act, model, _, data = variants["plain"]
    with torch.no_grad():
        _, sampled, _ = act.compute_samplenet_loss(model, data, dev)
    s0, s1 = sampled[0].detach().clone(), sampled[1].detach().clone()
    last = {}

    def task_fn(name):
        act, model, _, data = variants[name]

        def run():
            a0, a1 = s0.clone().requires_grad_(True), s1.clone().requires_grad_(True)
            loss, info = act.compute_pcrnet_loss(model, (a0, a1, data[2]), dev)
            loss.backward()
            last[name] = (loss.detach(), a0.grad, a1.grad, info["rot_err"].detach())
        return run

    def step_fn(name):
        act, model, opt, data = variants[name]
        return lambda: act.train_step(model, data, opt, dev)

    res = {"card": card(), "B": B, "N": N, "M": M, "steps_per_block": args.steps, "blocks": args.blocks}
    if args.num_sampled_clouds != 2:
        res["num_sampled_clouds"] = args.num_sampled_clouds
    for what, mk in (("task_half", task_fn), ("train_step", step_fn)):
        fns = {n: mk(n) for n in variants}
        for n in fns:
            for _ in range(10):
                fns[n]()
        torch.cuda.synchronize()
        t = {n: [] for n in fns}
        for _ in range(args.blocks):
            for n in fns:
                t[n].append(timed(fns[n], args.steps))
        for n in fns:
            res["%s_%s_us" % (what, n)] = {"median": statistics.median(t[n]), "min": min(t[n]), "max": max(t[n])}
        res["%s_speedup_of_medians" % what] = res["%s_plain_us" % what]["median"] / res["%s_frozen_us" % what]["median"]
        if what == "task_half":
            d = [float((a.double() - b.double()).abs().max()) for a, b in zip(last["plain"], last["frozen"])]
            res["task_half_max_abs_diff"] = {"loss": d[0], "grad_p0": d[1], "grad_p1": d[2], "rot_err_deg": d[3],
                                             "grad_p0_max_abs": float(last["plain"][1].abs().max())}
            if args.out:
                os.makedirs(args.out, exist_ok=True)
                torch.save({n: [x.cpu() for x in v] for n, v in last.items()}, os.path.join(args.out, "registration_task_last_step.pt"))
    for what, mk in (("task_half", task_fn), ("train_step", step_fn)):
        for n in variants:
            k, fam = kernels_per_step(mk(n))
            res["%s_%s_kernels_per_step" % (what, n)] = k
            if what == "task_half" and n == "frozen":
                mlp_bytes = 4 * sum(MLP_WIDTHS[i] * MLP_WIDTHS[i + 1] for i in range(6))     # every weight once per pass
                res["kernel_us_per_step"] = fam
                res["mlp_weight_bytes_per_pass"] = mlp_bytes
                if fam.get("frozen_mlp_forward"):
                    res["mlp_forward_GBps"] = mlp_bytes / fam["frozen_mlp_forward"] * 1e-3
                if fam.get("frozen_mlp_backward"):
                    res["mlp_backward_GBps"] = mlp_bytes / (fam["frozen_mlp_backward"] + fam.get("frozen_mlp_sum", 0.0)) * 1e-3
    print(json.dumps(res))


if __name__ == "__main__":
    main()
