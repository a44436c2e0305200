"""Time the reconstruction samplers trained together with their autoencoder (fixed_ae=False, the reference's --fixed_ae False), on:

    cuda   tasknets.CudaPointNetAE: the encoder over every prefix from one pass of the batch-statistics encoder trained
           (ops.EncoderBStatTrainFunction: forward, running statistics, gradients to the points and to every encoder parameter)
    torch  the plain tasknets.PointNetAE in training mode, one call per prefix (fp32: TF32 off)

    python tools/bench_joint_ae.py [--steps 10] [--blocks 5] [--epoch-batches 4]

One process, one GPU, B = 50, N = 2048, every route from the same initial state and batch.  Four comparisons:
    encoder           the autoencoder's encoder alone over the 8 progressive prefixes (16 .. 2048): forward, then the backward with every
                      encoder parameter's gradient and the points' gradient
    progressive_step  trainers.ProgressiveReconstructionStep(ReconstructionSampleNet(2048), ae, fixed_ae=False) with Adam over both modules
    rec_step          trainers.ReconstructionStep(ReconstructionSampleNet(64), ae, 64, fixed_ae=False) (2048 -> 64), Adam over both
    progressive_epoch SamplerTrainStep.train_one_epoch of the progressive step over --epoch-batches batches, eager and graphed=True
The routes alternate in blocks timed with device events; the median and the spread over the blocks are reported, and CUDA kernels per
call come from a separate torch.profiler pass.  The card's name, power limit and SM clock limit are read in the same run and printed with
the numbers.  Prints one JSON line.  Needs a GPU.
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


def _ae(route, dev):
    from samplenet_b200 import tasknets

    torch.manual_seed(0)
    net = tasknets.PointNetAE(n_pc_points=N).to(dev).train()
    return net, (tasknets.CudaPointNetAE(net) if route.startswith("cuda") else net)


def _step(progressive, route, dev, graphed=False):
    import samplenet_b200 as sb
    from samplenet_b200 import trainers

    net, ae = _ae(route, dev)
    torch.manual_seed(1)
    sampler = sb.ReconstructionSampleNet(N if progressive else 64).to(dev).train()
    step = (trainers.ProgressiveReconstructionStep(sampler, ae, SIZES, fixed_ae=False) if progressive
            else trainers.ReconstructionStep(sampler, ae, 64, fixed_ae=False))
    opt = torch.optim.Adam(list(sampler.parameters()) + list(net.parameters()), lr=1e-4, capturable=graphed)
    return trainers.SamplerTrainStep(step, opt, batch_size=B, graphed=graphed)


def make_step(progressive):
    def make(route, dev):
        run = _step(progressive, route, dev)
        x = (torch.rand(B, N, 3, generator=torch.Generator().manual_seed(2)) - 0.5).to(dev)
        return lambda: run(x)["loss"]
    return make


def make_epoch(batches):
    def make(route, dev):
        run = _step(True, route, dev, graphed=route.endswith("graphed"))
        x = (torch.rand(batches * B, N, 3, generator=torch.Generator().manual_seed(2)) - 0.5).to(dev)
        return lambda: run.train_one_epoch(x)
    return make


def make_encoder(route, dev):
    from samplenet_b200 import ops

    net, ae = _ae(route, dev)
    x = (torch.rand(B, N, 3, generator=torch.Generator().manual_seed(3)) - 0.5).to(dev).requires_grad_(True)
    g = torch.randn(len(SIZES), B, net.convs[-1].out_channels, generator=torch.Generator().manual_seed(4)).to(dev)
    conv, _, params = ae._layer_stack() if route == "cuda" else (None, None, None)
    enc = [t for c, bn in zip(net.convs, net.bns) for t in (c.weight, c.bias, bn.weight, bn.bias)]

    def run():
        if route == "cuda":
            pooled = ops.EncoderBStatTrainFunction.apply(x, conv, SIZES, *params[:4 * len(conv)])[0]
        else:
            pooled = torch.stack([net.encode(x[:, :s]) for s in SIZES])
        return torch.autograd.grad((pooled * g).sum(), [x] + enc)[0]

    return run


def bench(make_fn, routes, steps, blocks, dev):
    fns = {r: make_fn(r, dev) for r in routes}
    for r in routes:
        for _ in range(3):
            fns[r]()
    torch.cuda.synchronize()
    t = {r: [] for r in routes}
    for _ in range(blocks):
        for r in routes:
            t[r].append(timed(fns[r], steps))
    out = {}
    for r in routes:
        out[r + "_us"] = {"median": statistics.median(t[r]), "min": min(t[r]), "max": max(t[r])}
        out[r + "_kernels"] = kernels_per_step(fns[r], steps=2, keys=())[0]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--epoch-batches", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_joint_ae: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cuda.matmul.allow_tf32 = False   # the torch route is the fp32 baseline
    torch.backends.cudnn.allow_tf32 = False
    res = {"card": card(), "B": B, "N": N, "sizes": SIZES, "steps_per_block": args.steps, "blocks": args.blocks}
    for name, make_fn in (("encoder", make_encoder), ("progressive_step", make_step(True)), ("rec_step", make_step(False))):
        res[name] = bench(make_fn, ("cuda", "torch"), args.steps, args.blocks, dev)
        res[name]["cuda_vs_torch"] = res[name]["torch_us"]["median"] / res[name]["cuda_us"]["median"]
        torch.cuda.empty_cache()
    ep = bench(make_epoch(args.epoch_batches), ("cuda_eager", "cuda_graphed", "torch_eager", "torch_graphed"), 1, args.blocks, dev)
    ep["batches"] = args.epoch_batches
    ep["cuda_graphed_vs_eager"] = ep["cuda_eager_us"]["median"] / ep["cuda_graphed_us"]["median"]
    ep["cuda_graphed_vs_torch_eager"] = ep["torch_eager_us"]["median"] / ep["cuda_graphed_us"]["median"]
    res["progressive_epoch"] = ep
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
