"""Measure the per-cloud EMD (ops.emd_per_cloud / ops.EMDCostFunction) against the match-tensor route it replaces.

    python tools/bench_emd.py [--rounds 5] [--clouds 500] [--quick]

One process, one GPU, synthetic clouds from fixed seeds.  Each case runs the old route (approx_match + match_cost [+ match_cost_grad]
through a (B, M, N) match tensor, written out here as the package ran it before) and the new one, warmed on their own shapes and then
timed in alternating rounds with device events around whole calls; medians and the spread over the rounds, and the peak of
torch.cuda.max_memory_allocated above what was allocated before the call:

  ae_train_eager / ae_train_graphed   one AutoencoderTrainStep(ae_loss="emd") step at B = 50, N = 2048 (CudaPointNetAE), eager and as
                                      a CUDA-graph replay (the graph of each route is captured once and replayed)
  eval_curve                          ReconstructionEvaluator(FPS sampler, FrozenPointNetAE, ae_loss="emd").evaluate at the sizes 16, 32,
                                      ..., 2048 over `clouds` clouds (all eight prefixes x 50 reconstructions per batch in one loss call)
  forward                             the per-cloud cost alone at 50 x 2048^2

Both routes give the same bits (tests/test_emd_per_cloud.py); the tool checks the forward case's outputs.  Prints one JSON line with the
card, its power limit and maximum SM clock.  Needs a GPU: it fails without one.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def measure(fn):
    """(milliseconds, peak bytes allocated above the allocation before the call) of one call ending in a device synchronise."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), torch.cuda.max_memory_allocated() - base


def composed_ae_loss(x_reconstr, gt, loss="emd"):
    from samplenet_b200 import tf_ops

    return tf_ops.match_cost(x_reconstr, gt, tf_ops.approx_match(x_reconstr, gt)).mean()


def composed_eval_loss(self, recon, gt):
    from samplenet_b200 import tf_ops

    gt = gt.repeat(recon.shape[0] // gt.shape[0], 1, 1) if recon.shape[0] != gt.shape[0] else gt
    return tf_ops.match_cost(recon, gt, tf_ops.approx_match(recon, gt))


class Route:
    """Switches the package's EMD callers between the per-cloud route ("new") and the match-tensor composition ("old")."""

    def __init__(self):
        from samplenet_b200 import evaluation, trainers

        self.trainers, self.evaluation = trainers, evaluation
        self.new = (trainers.autoencoder_loss, evaluation.ReconstructionEvaluator._loss)

    def set(self, which):
        loss, ev = self.new if which == "new" else (composed_ae_loss, composed_eval_loss)
        self.trainers.autoencoder_loss = loss
        self.evaluation.ReconstructionEvaluator._loss = ev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--clouds", type=int, default=500)
    ap.add_argument("--quick", action="store_true", help="two rounds, 100 clouds")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_emd.py needs a CUDA device")
    if args.quick:
        args.rounds, args.clouds = 2, 100
    import samplenet_b200 as sb
    from samplenet_b200 import ops, tasknets, trainers

    route = Route()
    g = torch.Generator().manual_seed(0)
    B, N = 50, 2048
    batch = (torch.rand(B, N, 3, generator=g) - 0.5).cuda()
    pcs = (torch.rand(args.clouds, N, 3, generator=g) - 0.5).cuda()
    x1, x2 = torch.rand(B, N, 3, generator=g).cuda(), torch.rand(B, N, 3, generator=g).cuda()

    def ae_step(graphed):
        torch.manual_seed(0)
        ae = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=N)).cuda()
        opt = torch.optim.Adam(ae.parameters(), lr=5e-4, capturable=True)
        step = trainers.AutoencoderTrainStep(ae, opt, ae_loss="emd", n_sample_points=N, batch_size=B, graphed=graphed)
        return lambda: step(batch)

    net = tasknets.PointNetAE(n_pc_points=N).cuda().eval().requires_grad_(False)
    evaluator = sb.ReconstructionEvaluator(sb.FPSSampler(N, permute=False, input_shape="bnc", output_shape="bnc"), tasknets.FrozenPointNetAE(net),
                                           ae_loss="emd")
    sizes = [2 ** k for k in range(4, 12)]   # 16, 32, ..., 2048

    def fwd(which):
        if which == "new":
            return lambda: ops.emd_per_cloud(x1, x2)
        return lambda: ops.match_cost_forward(x1, x2, ops.approx_match(x1, x2))

    same = {}
    route.set("old"); ref = fwd("old")()
    route.set("new"); same["forward"] = bool(torch.equal(fwd("new")(), ref))
    cases = {}
    for name in ("ae_train_eager", "ae_train_graphed", "eval_curve", "forward"):
        calls = {}
        for which in ("old", "new"):
            route.set(which)
            if name.startswith("ae_train"):
                calls[which] = ae_step(name.endswith("graphed"))
            elif name == "eval_curve":
                calls[which] = lambda: evaluator.evaluate(pcs, sizes=sizes)
            else:
                calls[which] = fwd(which)
            calls[which]()          # warm-up (and the capture of a graphed step)
        times, peaks = {"old": [], "new": []}, {"old": 0, "new": 0}
        for _ in range(args.rounds):
            for which in ("old", "new"):
                route.set(which)
                ms, peak = measure(calls[which])
                times[which].append(ms)
                peaks[which] = max(peaks[which], peak)
        cases[name] = {w: {"median_ms": round(statistics.median(times[w]), 3), "min_ms": round(min(times[w]), 3), "max_ms": round(max(times[w]), 3),
                           "peak_alloc_mb": round(peaks[w] / 2 ** 20, 1)} for w in ("old", "new")}
        cases[name]["speedup"] = round(cases[name]["old"]["median_ms"] / cases[name]["new"]["median_ms"], 3)
    route.set("new")
    print(json.dumps({"card": card(), "rounds": args.rounds, "clouds": args.clouds, "sizes": sizes, "same_bits": same, "cases": cases}))


if __name__ == "__main__":
    main()
