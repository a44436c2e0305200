"""Measure the exact-mode (SNB200_EMD_EXACT_EXP=1) EMD autoencoder loss through the per-cloud route against the match-tensor composition.

    python tools/bench_emd_exact.py [--rounds 5] [--batch 50] [--points 2048]

One process, one GPU, synthetic clouds from a fixed seed.  The case is trainers.autoencoder_loss(x, gt, "emd") forward + backward (the
gradient to the reconstruction x) at B = 50, N = M = 2048 in the exact mode:

  old   approx_match(exact) + match_cost + match_cost_grad through the (B, M, N) match tensor, written out here as the package ran it
        before (the exact approx_match zero-fills the match and read-modify-writes it once per level)
  new   ops.EMDCostFunction in the exact mode: the exact levels keep their ratios, and the cost and gradient passes rebuild every match
        element from them (one double-precision exponential per level and pair in each pass)

Both are warmed, then timed in alternating rounds with device events around whole calls (each call ends in a device synchronise):
medians, the spread over the rounds, and the peak of torch.cuda.max_memory_allocated above what was allocated before the call.  The tool
checks that both routes give the same loss and gradient bits.  Prints one JSON line with the card, its power limit and maximum SM clock.
Needs a GPU: it fails without one.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_emd import card, composed_ae_loss, measure  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=50)
    ap.add_argument("--points", type=int, default=2048)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_emd_exact.py needs a CUDA device")
    os.environ["SNB200_EMD_EXACT_EXP"] = "1"
    from samplenet_b200 import ops, trainers

    assert ops.emd_exact_mode()
    B, N = args.batch, args.points
    g = torch.Generator().manual_seed(0)
    x0, gt = (torch.rand(B, N, 3, generator=g) - 0.5).cuda(), (torch.rand(B, N, 3, generator=g) - 0.5).cuda()
    if not ops.emd_per_cloud_supported(x0, gt, exact=True):
        sys.exit("B=%d N=%d is outside the exact per-cloud envelope" % (B, N))
    routes = {"old": composed_ae_loss, "new": trainers.autoencoder_loss}

    def call(which):
        x = x0.clone().requires_grad_(True)
        loss = routes[which](x, gt, "emd")
        loss.backward()
        return loss.detach(), x.grad

    out = {w: call(w) for w in ("old", "new")}   # warm-up, and the bits of each route
    same = all(torch.equal(a, b) for a, b in zip(out["old"], out["new"]))
    del out
    times, peaks = {"old": [], "new": []}, {"old": 0, "new": 0}
    for _ in range(args.rounds):
        for which in ("old", "new"):
            ms, peak = measure(lambda: call(which))
            times[which].append(ms)
            peaks[which] = max(peaks[which], peak)
    res = {w: {"median_ms": round(statistics.median(times[w]), 2), "min_ms": round(min(times[w]), 2), "max_ms": round(max(times[w]), 2),
               "peak_alloc_mb": round(peaks[w] / 2 ** 20, 1)} for w in ("old", "new")}
    res["speedup"] = round(res["old"]["median_ms"] / res["new"]["median_ms"], 3)
    print(json.dumps({"card": card(), "case": "autoencoder_loss emd exact fwd+bwd", "B": B, "N": N, "rounds": args.rounds, "same_bits": same,
                      "routes": res}))


if __name__ == "__main__":
    main()
