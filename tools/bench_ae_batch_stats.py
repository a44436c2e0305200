"""Time the reconstruction sampler steps with the frozen autoencoder normalised by each prefix's batch statistics (ae_batch_stats=True), on:

    frozen_bstat  tasknets.FrozenPointNetAE: every prefix from one pass of the batch-statistics encoder (csrc/frozen_encoder_bstat.cu)
    torch_bstat   the plain tasknets.PointNetAE, PointNetAE.encode(..., batch_stats=True) per prefix (fp32: TF32 off), the same objective
    frozen_eval   tasknets.FrozenPointNetAE with eval-mode BatchNorm (ae_batch_stats=False): today's default, a different objective, for
                  context only

    python tools/bench_ae_batch_stats.py [--steps 10] [--blocks 5]

One process, one GPU.  Steps: trainers.ReconstructionStep(ReconstructionSampleNet(64), ae, 64) and
trainers.ProgressiveReconstructionStep(ReconstructionSampleNet(2048), ae) (sizes 16 .. 2048) at B = 50, N = 2048: the sampler's forward,
the losses, the backward and an Adam step, every route from the same initial state and batch.  Also the autoencoder's encoder alone at the
progressive sizes, forward and backward to the points ("encoder").  The routes alternate in blocks timed with device events; the median and
the spread over the blocks are reported, and CUDA kernels per call come from a separate torch.profiler pass.  The card's name, power limit
and SM clock limit are read in the same run and printed with the numbers.  Prints one JSON line.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_registration_task import card, kernels_per_step, timed  # noqa: E402

B, N = 50, 2048
SIZES = [16 * 2 ** i for i in range(8)]
ROUTES = ("frozen_bstat", "torch_bstat", "frozen_eval")


def _ae(dev):
    from samplenet_b200 import tasknets

    torch.manual_seed(0)
    return tasknets.PointNetAE(n_pc_points=N).to(dev).eval().requires_grad_(False)


def _wrap(route, net):
    from samplenet_b200 import tasknets

    return net if route == "torch_bstat" else tasknets.FrozenPointNetAE(net)


def make_step(progressive):
    def make(route, dev):
        import samplenet_b200 as sb
        from samplenet_b200 import trainers

        net = _ae(dev)
        torch.manual_seed(1)
        sampler = sb.ReconstructionSampleNet(N if progressive else 64).to(dev).train()
        flag = route != "frozen_eval"
        step = (trainers.ProgressiveReconstructionStep(sampler, _wrap(route, net), SIZES, ae_batch_stats=flag) if progressive
                else trainers.ReconstructionStep(sampler, _wrap(route, net), 64, ae_batch_stats=flag))
        opt = torch.optim.Adam(sampler.parameters(), lr=1e-4)
        x = (torch.rand(B, N, 3, generator=torch.Generator().manual_seed(2)) - 0.5).to(dev)

        def run():
            opt.zero_grad(set_to_none=True)
            loss, _ = step.loss(x)
            loss.backward()
            opt.step()
            return loss

        return run
    return make


def make_encoder(route, dev):
    net = _ae(dev)
    w = _wrap(route, net)
    x = (torch.rand(B, N, 3, generator=torch.Generator().manual_seed(3)) - 0.5).to(dev).requires_grad_(True)
    g = torch.randn(len(SIZES), B, net.convs[-1].out_channels, generator=torch.Generator().manual_seed(4)).to(dev)

    def run():
        if route == "torch_bstat":
            pooled = torch.stack([net.encode(x[:, :s], batch_stats=True) for s in SIZES])
        elif route == "frozen_bstat":
            pooled = w._bstat_pooled(x, SIZES)
        else:
            pooled = w._pooled(x, SIZES)[0]
        return torch.autograd.grad((pooled * g).sum(), x)[0]

    return run


def bench(make_fn, steps, blocks, dev):
    fns = {r: make_fn(r, dev) for r in ROUTES}
    for r in ROUTES:
        for _ in range(3):
            fns[r]()
    torch.cuda.synchronize()
    t = {r: [] for r in ROUTES}
    for _ in range(blocks):
        for r in ROUTES:
            t[r].append(timed(fns[r], steps))
    out = {}
    for r in ROUTES:
        out[r + "_us"] = {"median": statistics.median(t[r]), "min": min(t[r]), "max": max(t[r])}
        out[r + "_kernels"] = kernels_per_step(fns[r], steps=2, keys=())[0]
    out["frozen_bstat_vs_torch_bstat"] = out["torch_bstat_us"]["median"] / out["frozen_bstat_us"]["median"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--blocks", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ae_batch_stats: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False   # the torch route is the fp32 baseline
    torch.backends.cudnn.allow_tf32 = False
    res = {"card": card(), "B": B, "N": N, "sizes": SIZES, "steps_per_block": args.steps, "blocks": args.blocks}
    res["encoder"] = bench(make_encoder, args.steps, args.blocks, dev)
    torch.cuda.empty_cache()
    res["rec_step"] = bench(make_step(False), args.steps, args.blocks, dev)
    torch.cuda.empty_cache()
    res["progressive_step"] = bench(make_step(True), args.steps, args.blocks, dev)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
