"""Time the progressive classification step and curve with PointNet with transform nets as the frozen task network, on three routes:

    module      the plain module (tasknets.PointNetClsTransforms), one call per prefix
    per_prefix  tasknets.FrozenPointNetClsTransforms one prefix at a time (its forward on x[:, :s])
    prefixes    tasknets.FrozenPointNetClsTransforms.prefixes: every prefix in one chain of launches over packed segments

    python tools/bench_progressive_cls_transforms.py [--steps 20] [--blocks 5]

One process, one GPU.  The step is trainers.ProgressiveClassificationStep(ClassificationSampleNet(1024), classifier, 2, 1024) at B = 32,
N = 1024 (sizes 2, 4, ..., 1024): the sampler's forward, the classifier and simplification losses of every prefix, the backward and an
Adam step, every route from the same initial state and batch.  The curve is evaluation.ProgressiveClassificationEvaluator.evaluate on 256
ordered clouds of 1024 points at the same 10 sizes (batches of 32, one read-back).  The routes alternate in blocks timed with device events;
the median and the spread over the blocks are reported, and kernels per step come from a separate torch.profiler pass.  TF32 is at torch's
default.  The card's name, power limit and SM clock limit are printed with the numbers.  Prints one JSON line.  Needs a GPU.
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

B, N, CURVE_CLOUDS = 32, 1024, 256
ROUTES = ("module", "per_prefix", "prefixes")


class PerPrefix(torch.nn.Module):
    """The frozen wrapper without prefixes(): the step and the evaluator then call it once per prefix."""

    def __init__(self, wrapper):
        super().__init__()
        self.w = wrapper

    def forward(self, x):
        return self.w(x)

    def get_loss(self, *args, **kwargs):
        return self.w.get_loss(*args, **kwargs)


def classifier(route, net):
    from samplenet_b200 import tasknets

    if route == "module":
        return net
    w = tasknets.FrozenPointNetClsTransforms(net)
    return PerPrefix(w) if route == "per_prefix" else w


def make_step(route, dev):
    import samplenet_b200 as sb
    from samplenet_b200 import tasknets, trainers

    torch.manual_seed(0)
    net = tasknets.PointNetClsTransforms(40).to(dev).eval().requires_grad_(False)
    sampler = sb.ClassificationSampleNet(N).to(dev).train()
    step = trainers.ProgressiveClassificationStep(sampler, classifier(route, net), 2, N)
    opt = torch.optim.Adam(sampler.parameters(), lr=1e-3)
    g = torch.Generator().manual_seed(1)
    x, y = (torch.rand(B, N, 3, generator=g) - 0.5).to(dev), torch.randint(0, 40, (B,), generator=g).to(dev)

    def run():
        opt.zero_grad(set_to_none=True)
        loss, _ = step.loss(x, y)
        loss.backward()
        opt.step()
        return loss

    return run


def make_curve(route, dev):
    from samplenet_b200 import evaluation, tasknets

    torch.manual_seed(0)
    net = tasknets.PointNetClsTransforms(40).to(dev).eval().requires_grad_(False)
    ev = evaluation.ProgressiveClassificationEvaluator(None, classifier(route, net))
    g = torch.Generator().manual_seed(2)
    x, y = (torch.rand(CURVE_CLOUDS, N, 3, generator=g) - 0.5).to(dev), torch.randint(0, 40, (CURVE_CLOUDS,), generator=g).to(dev)
    sizes = [2 ** i for i in range(1, 11)]

    def run():
        with torch.no_grad():
            return ev.evaluate(x, y, sizes, ordered=x)["accuracy"]

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
    out["prefixes_vs_per_prefix"] = out["per_prefix_us"]["median"] / out["prefixes_us"]["median"]
    out["prefixes_vs_module"] = out["module_us"]["median"] / out["prefixes_us"]["median"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_progressive_cls_transforms: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "B": B, "N": N, "curve_clouds": CURVE_CLOUDS, "steps_per_block": args.steps, "blocks": args.blocks}
    res["step"] = bench(make_step, args.steps, args.blocks, dev)
    torch.cuda.empty_cache()
    res["curve"] = bench(make_curve, max(1, args.steps // 10), args.blocks, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
