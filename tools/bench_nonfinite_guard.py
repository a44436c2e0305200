"""Time the sampler epochs with skip_nonfinite on and off (trainers.SamplerTrainStep), eager and graphed, alternated.

    python tools/bench_nonfinite_guard.py [--blocks 5] [--cls-clouds 1280] [--rec-clouds 500] [--out FILE]

    cls32     trainers.ClassificationStep: ClassificationSampleNet(32, k = 7) in front of a frozen PointNetClsTransforms, B = 32, N = 1024
    cls1024   the same with ClassificationSampleNet(1024): about a million sampler parameters, the largest table the guard checks and copies
    rec       trainers.ReconstructionStep: ReconstructionSampleNet(64) in front of a frozen PointNetAE, Chamfer, B = 50, N = 2048

Synthetic finite sets, so no step is skipped and the guard's cost is its snapshot copy and its check; with the guard off the epochs run
exactly as before.  Every epoch starts from the same network and optimiser state.  For every (case, eager/graphed) the guard-on and
guard-off epochs alternate in blocks; the medians over the blocks and the per-step difference are reported, with the card's name, power
limit and SM clock limit.  Prints one JSON line.  Needs a GPU.
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

from bench_classifier_epoch import wall  # noqa: E402
from bench_registration_task import card  # noqa: E402

CLASSES = 40


def make_runner(case, dev, graphed, skip):
    import samplenet_b200 as sb
    from samplenet_b200 import tasknets, trainers

    torch.manual_seed(0)
    if case.startswith("cls"):
        m = int(case[3:])
        sampler = sb.ClassificationSampleNet(m, group_size=7).to(dev)
        net = tasknets.PointNetClsTransforms(num_classes=CLASSES).to(dev).eval().requires_grad_(False)
        step = trainers.ClassificationStep(sampler, tasknets.FrozenPointNetClsTransforms(net), m)
        opt = torch.optim.Adam(sampler.parameters(), lr=0.01, capturable=True)
    else:
        sampler = sb.ReconstructionSampleNet(64).to(dev)
        ae = tasknets.FrozenPointNetAE(tasknets.PointNetAE(n_pc_points=2048).to(dev).eval().requires_grad_(False))
        step = trainers.ReconstructionStep(sampler, ae, 64)
        opt = torch.optim.Adam(sampler.parameters(), lr=5e-4, capturable=True)
    return trainers.SamplerTrainStep(step, opt, graphed=graphed, skip_nonfinite=skip)


def make_epoch(case, dev, graphed, skip, x, y):
    """(epoch, reset, steps): one epoch on the device-resident set, and a reset to the initial sampler and an empty optimiser state."""
    from samplenet_b200 import graphs

    run = make_runner(case, dev, graphed, skip)
    init = {k: v.detach().clone() for k, v in run.task.sampler.state_dict().items()}

    def reset():
        with torch.no_grad():
            for k, v in run.task.sampler.state_dict().items():
                v.copy_(init[k])
        graphs._restore_optimizer(run.optimizer, {})    # in place: a captured step points at the state tensors
        run.step = run.epoch = 0

    def epoch():
        res = run.train_one_epoch(x, y) if case.startswith("cls") else run.train_one_epoch(x)
        if skip and res["skipped_steps"]:
            raise FloatingPointError("%s: %d steps skipped on a finite set" % (case, res["skipped_steps"]))
        return res

    return epoch, reset, run, run.batch_size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--cls-clouds", type=int, default=1280)
    ap.add_argument("--rec-clouds", type=int, default=500)
    ap.add_argument("--cases", default="cls32,cls1024,rec")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nonfinite_guard needs a GPU")
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    result = {"card": card(), "blocks": args.blocks}
    for case in args.cases.split(","):
        n, pts = (args.cls_clouds, 1024) if case.startswith("cls") else (args.rec_clouds, 2048)
        x = (torch.rand(n, pts, 3, generator=g) - 0.5).to(dev)
        y = torch.randint(0, CLASSES, (n,), generator=g).to(dev)
        for graphed in (False, True):
            routes = {skip: make_epoch(case, dev, graphed, skip, x, y) for skip in (False, True)}
            params = sum(p.numel() for p in routes[True][2].task.sampler.parameters())
            steps = n // routes[True][3]
            t = {False: [], True: []}
            for block in range(args.blocks + 1):
                for skip, (epoch, reset, _, _) in routes.items():
                    reset()
                    print("%s graphed=%s guard=%s block %d" % (case, graphed, skip, block), file=sys.stderr, flush=True)
                    dt = wall(epoch)
                    if block:                             # block 0 warms up (and captures)
                        t[skip].append(dt)
            off, on = statistics.median(t[False]), statistics.median(t[True])
            result["%s_%s" % (case, "graphed" if graphed else "eager")] = {
                "sampler_params": params, "steps": steps,
                "guard_off_s": {"median": off, "min": min(t[False]), "max": max(t[False])},
                "guard_on_s": {"median": on, "min": min(t[True]), "max": max(t[True])},
                "guard_us_per_step": (on - off) * 1e6 / steps,
            }
            del routes
            torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
