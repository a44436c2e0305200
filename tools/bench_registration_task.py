"""Measure the registration trainer's task half (frozen PCRNet + quaternion / Chamfer pose loss) plain against frozen_task=True.

    python tools/bench_registration_task.py [--steps 200] [--blocks 5] [--out DIR]

One process, one GPU.  Builds RegistrationStep(num_sampled_clouds=2) at B=32, N=1024 -> 64 twice from the same seed and the data of
tools/bench_configs.py's cfg_registration_ddp, warms both, then times alternating plain / frozen blocks with device events:
  (a) the task half alone: compute_pcrnet_loss on fixed sampled clouds + backward to the clouds;
  (b) the whole train_step.
Reports the median and the spread over the blocks, the CUDA kernels per step of each from a separate torch.profiler pass, the two new
kernel families' device time against the bytes their shapes imply (the MLP's weights once per pass), and the largest difference of the last
step's loss and sampled-cloud gradients between the variants.  Prints one JSON line.  Needs a GPU: it fails without one.
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


def make(frozen, dev):
    from bench_configs import clouds
    from samplenet_b200.registration import QuaternionTransform, RegistrationStep

    act = RegistrationStep(num_sampled_clouds=2)
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


def kernels_per_step(fn, steps=5):
    """(CUDA kernels per step, {kernel-name prefix: device us per step}) from a profiler pass of its own."""
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
            for key in ("frozen_mlp_forward", "frozen_mlp_backward", "frozen_mlp_sum", "pose_loss_forward", "pose_loss_backward"):
                if key in ev.name:
                    fam[key] = fam.get(key, 0.0) + ev.device_time / steps
    return count / steps, fam


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the dumped last-step tensors")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_registration_task: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    variants = {name: make(name == "frozen", dev) for name in ("plain", "frozen")}

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
