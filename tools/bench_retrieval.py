"""Measure shape retrieval (ops.retrieval_metrics, RetrievalEvaluator, ProgressiveClassificationEvaluator.retrieval).

    python tools/bench_retrieval.py [--rounds 5] [--quick]

One process, one GPU, synthetic data from fixed seeds at ModelNet40's test size (2468 clouds of 1024 points, 40 labels), every variant
warmed on its own shapes and then timed in alternating rounds with device events around whole calls; medians and the spread:

  kernel       ops.retrieval_metrics alone on 256-wide descriptors, (2468, 2468) leave-one-out and (2468, 9843), against the torch
               composition on the same descriptors: cdist(compute_mode="donot_use_mm_for_euclid_dist") + stable argsort + cumsum.  Achieved
               rate over the 3 * Q * M * D operations the distance needs, and the torch route's peak memory over its inputs
  evaluator    RetrievalEvaluator.evaluate with ClassificationSampleNet(32) and FrozenPointNetClsTransforms, leave-one-out
  progressive  a 10-size curve: ProgressiveClassificationEvaluator.retrieval through FrozenPointNetCls.prefixes(), against size by size
               through the plain PointNetCls

Prints one JSON line with the card, its power limit and maximum SM clock.  Needs a GPU: it fails without one.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_evaluation import alternate, card, clouds  # noqa: E402


def torch_route(q, ql, x, xl, exclude, levels):
    """The composition the kernel replaces: the same metrics from a (Q, M) distance matrix and a stable sort of it."""
    d = torch.cdist(q, x, compute_mode="donot_use_mm_for_euclid_dist")
    if exclude:
        d.fill_diagonal_(float("inf"))
    order = torch.argsort(d, dim=1, stable=True)
    if exclude:
        order = order[:, :-1]
    rel = (xl[order] == ql[:, None]).double()
    hits = torch.cumsum(rel, dim=1)
    k = torch.arange(1, order.shape[1] + 1, device=q.device, dtype=torch.float64)
    R = hits[:, -1]
    ap = (rel * hits / k).sum(dim=1) / R
    ratio = torch.where(rel > 0, hits / k, torch.zeros_like(hits))
    suffix = torch.flip(torch.cummax(torch.flip(ratio, [1]), dim=1)[0], [1])
    lv = torch.arange(levels, device=q.device, dtype=torch.float64)[None, :] * R[:, None]
    first = torch.searchsorted(hits.contiguous(), (lv / (levels - 1)).contiguous())      # first rank with hits >= l * R / (L - 1)
    prec = torch.gather(suffix, 1, first.clamp(max=order.shape[1] - 1))
    return ap, prec


def bench_kernel(dev, rounds, q_n, m_n, d):
    from samplenet_b200 import ops

    g = torch.Generator().manual_seed(7)
    q = torch.randn(q_n, d, generator=g).to(dev)
    ql = torch.randint(0, 40, (q_n,), generator=g).to(dev)
    exclude = m_n is None
    x, xl = (q, ql) if exclude else (torch.randn(m_n, d, generator=g).to(dev), torch.randint(0, 40, (m_n,), generator=g).to(dev))
    m_n = x.shape[0]
    kern = (lambda: ops.retrieval_metrics(q, ql)) if exclude else (lambda: ops.retrieval_metrics(q, ql, x, xl))
    fns = {"kernel": lambda: (kern(), torch.cuda.synchronize()), "torch_cdist_argsort_cumsum": lambda: (torch_route(q, ql, x, xl, exclude, 11),
                                                                                                         torch.cuda.synchronize())}
    t = alternate(fns, rounds)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ap_t, _ = torch_route(q, ql, x, xl, exclude, 11)
    torch.cuda.synchronize()
    torch_peak = torch.cuda.max_memory_allocated() - base
    torch.cuda.reset_peak_memory_stats()
    out = kern()
    torch.cuda.synchronize()
    kernel_peak = torch.cuda.max_memory_allocated() - base
    ops_needed = 3.0 * q_n * m_n * d
    return {"Q": q_n, "M": m_n, "D": d, "leave_one_out": exclude, "ms_per_call": t,
            "kernel_tflops": ops_needed / (t["kernel"]["median"] * 1e-3) / 1e12,
            "torch_tflops": ops_needed / (t["torch_cdist_argsort_cumsum"]["median"] * 1e-3) / 1e12,
            "speedup_of_medians": t["torch_cdist_argsort_cumsum"]["median"] / t["kernel"]["median"],
            "torch_peak_mb_over_inputs": torch_peak / 2 ** 20, "kernel_peak_mb_over_inputs": kernel_peak / 2 ** 20,
            "max_abs_diff_ap_vs_torch": float((out["ap"] - ap_t).abs().max())}


def bench_evaluator(dev, rounds, n):
    import samplenet_b200 as sb
    from samplenet_b200 import tasknets

    torch.manual_seed(0)
    sampler = sb.ClassificationSampleNet(32).to(dev)
    net = tasknets.PointNetClsTransforms().to(dev).requires_grad_(False).eval()
    ev = sb.RetrievalEvaluator(sampler, tasknets.FrozenPointNetClsTransforms(net), 32)
    pcs, labels = clouds(n, 1024, 3, dev), torch.randint(0, 40, (n,), generator=torch.Generator().manual_seed(4)).to(dev)
    fns = {"evaluate_batch_32": lambda: ev.evaluate(pcs, labels, batch_size=32)}
    return {"clouds": n, "ms_per_call": alternate(fns, rounds)}


def bench_progressive(dev, rounds, n):
    import samplenet_b200 as sb
    from samplenet_b200 import tasknets

    torch.manual_seed(0)
    sampler = sb.ClassificationSampleNet(64).to(dev)
    net = tasknets.PointNetCls().to(dev).requires_grad_(False).eval()
    frozen, plain = sb.ProgressiveClassificationEvaluator(sampler, tasknets.FrozenPointNetCls(net)), sb.ProgressiveClassificationEvaluator(sampler, net)
    pcs, labels = clouds(n, 1024, 5, dev), torch.randint(0, 40, (n,), generator=torch.Generator().manual_seed(6)).to(dev)
    ordered = frozen.order(pcs)
    sizes = [2, 4, 8, 16, 32, 64, 128, 256, 512, 1024]
    fns = {"prefixes_10_sizes": lambda: frozen.retrieval(pcs, labels, sizes, ordered=ordered),
           "size_by_size_plain_10_sizes": lambda: plain.retrieval(pcs, labels, sizes, ordered=ordered)}
    a, b = frozen.retrieval(pcs, labels, sizes, ordered=ordered), plain.retrieval(pcs, labels, sizes, ordered=ordered)
    return {"clouds": n, "sizes": sizes, "ms_per_call": alternate(fns, rounds), "max_abs_diff_map": float(abs(a["map"] - b["map"]).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--quick", action="store_true", help="small sizes: a rehearsal of the script, not a measurement")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_retrieval: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n = 256 if args.quick else 2468
    res = {"card": card(), "rounds": args.rounds, "quick": args.quick}
    res["kernel"] = [bench_kernel(dev, args.rounds, n, None, 256), bench_kernel(dev, args.rounds, n, 1024 if args.quick else 9843, 256)]
    res["evaluator"] = bench_evaluator(dev, args.rounds, n)
    res["progressive"] = bench_progressive(dev, args.rounds, n)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
