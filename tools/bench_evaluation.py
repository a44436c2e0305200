"""Measure the evaluators (samplenet_b200/evaluation.py, RegistrationStep.test_1) batched against the reference's one-record way.

    python tools/bench_evaluation.py [--rounds 5] [--records 1024] [--quick]

One process, one GPU, synthetic clouds from fixed seeds, every variant warmed on its own shapes and then timed in alternating rounds
with device events around whole calls (each call ends in its one host read-back); medians and the spread over the rounds:

  registration    test_1 over `records` pairs (N=1024 -> 64 points, both clouds sampled by SampleNet, frozen PCRNet) at batch 1 (the
                  reference's loop), 32 and 256 (one ops.pose_eval launch per batch)
  classification  the progressive curve of 256 clouds of 1024 points at 10 sizes and dense (1024 sizes), frozen PointNet classifier
                  through prefixes(); the 10 sizes also size by size through the plain module
  reconstruction  the progressive per-cloud AE loss of 50 clouds of 2048 points at 8 sizes: ops.chamfer_per_cloud on the 400
                  reconstructions against nn_distance + torch means on a repeated reference, and the two alone on the same tensors

Prints one JSON line with the card, its power limit and maximum SM clock.  Needs a GPU: it fails without one.
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


def timed_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record(); b.synchronize()
    return a.elapsed_time(b)


def alternate(fns, rounds):
    """{name: {"median", "min", "max"} in ms}: every variant warmed once, then `rounds` rounds that run the variants one after another."""
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    t = {n: [] for n in fns}
    for _ in range(rounds):
        for n, fn in fns.items():
            t[n].append(timed_ms(fn))
    return {n: {"median": statistics.median(v), "min": min(v), "max": max(v)} for n, v in t.items()}


def clouds(n, points, seed, dev, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(n, points, 3, generator=g) * 2 - 1) * scale).to(dev)


def bench_registration(dev, records, rounds):
    from samplenet_b200.registration import RegistrationStep, qrot

    step = RegistrationStep(num_sampled_clouds=2)
    torch.manual_seed(0)
    model = step.create_model(frozen_task=True).to(dev)
    g = torch.Generator().manual_seed(1)
    quat = torch.nn.functional.normalize(torch.randn(records, 4, generator=g), dim=1).to(dev)
    p0 = clouds(records, 1024, 2, dev)
    p1 = qrot(quat[:, None, :].expand(-1, 1024, -1).contiguous(), p0)
    vec = torch.cat([quat, torch.zeros(records, 3, device=dev)], dim=1)

    def batches(bs):
        return [(p0[s:s + bs], p1[s:s + bs], {"vec": vec[s:s + bs], "inversion": torch.tensor([False])}) for s in range(0, records, bs)]

    out, fns = {}, {}
    for bs in (1, 32, 256):
        data = batches(bs)
        fns["batch_%d" % bs] = lambda data=data, bs=bs: out.__setitem__(bs, step.test_1(model, data, dev))
    res = {"records": records, "ms_per_call": alternate(fns, rounds)}
    res["speedup_of_medians_over_batch_1"] = {k: res["ms_per_call"]["batch_1"]["median"] / v["median"] for k, v in res["ms_per_call"].items()}
    res["max_abs_diff_rot_deg_vs_batch_1"] = {bs: float(abs(out[bs]["rotation_errors"] - out[1]["rotation_errors"]).max()) for bs in (32, 256)}
    return res


def bench_classification(dev, rounds, n_clouds, n_points):
    import samplenet_b200 as sb
    from samplenet_b200 import tasknets

    torch.manual_seed(0)
    sampler = sb.ClassificationSampleNet(64).to(dev)
    net = tasknets.PointNetCls().to(dev).requires_grad_(False).eval()
    pcs, labels = clouds(n_clouds, n_points, 3, dev), torch.randint(0, 40, (n_clouds,), generator=torch.Generator().manual_seed(4)).to(dev)
    frozen, plain = sb.ProgressiveClassificationEvaluator(sampler, tasknets.FrozenPointNetCls(net)), sb.ProgressiveClassificationEvaluator(sampler, net)
    ordered = frozen.order(pcs)
    sizes = [max(1, n_points >> k) for k in range(9, -1, -1)]
    sizes = sorted(set(sizes))
    fns = {"prefixes_%d_sizes" % len(sizes): lambda: frozen.evaluate(pcs, labels, sizes, ordered=ordered),
           "size_by_size_plain_%d_sizes" % len(sizes): lambda: plain.evaluate(pcs, labels, sizes, ordered=ordered),
           "prefixes_dense_%d_sizes" % n_points: lambda: frozen.evaluate(pcs, labels, range(1, n_points + 1), ordered=ordered),
           "order": lambda: (frozen.order(pcs), torch.cuda.synchronize())}
    return {"clouds": n_clouds, "points": n_points, "sizes": sizes, "ms_per_call": alternate(fns, rounds)}


def bench_reconstruction(dev, rounds, n_clouds, sizes):
    import samplenet_b200 as sb
    from samplenet_b200 import ops, tasknets

    torch.manual_seed(0)
    sampler = sb.ReconstructionSampleNet(max(sizes)).to(dev)
    net = tasknets.PointNetAE(2048).to(dev).requires_grad_(False).eval()
    ae = tasknets.FrozenPointNetAE(net)
    pcs = clouds(n_clouds, 2048, 5, dev, 0.5)
    evaluator = sb.ReconstructionEvaluator(sampler, ae)
    sampled_pc, _ = evaluator.get_samples(pcs)
    with torch.no_grad():
        recon = ae.prefixes(sampled_pc, sizes).flatten(0, 1).contiguous()
    p = len(sizes)

    def per_cloud():
        return ops.chamfer_per_cloud(recon, pcs).sum(dim=1)

    def nn_means():
        d1, _, d2, _ = ops.nn_distance_forward(recon, pcs.repeat(p, 1, 1))
        return d1.mean(dim=1) + d2.mean(dim=1)

    class _NNMeans(sb.ReconstructionEvaluator):      # the evaluator with the loss the kernel replaces
        def _loss(self, r, gt):
            d1, _, d2, _ = ops.nn_distance_forward(r.contiguous(), gt.repeat(r.shape[0] // gt.shape[0], 1, 1))
            return d1.mean(dim=1) + d2.mean(dim=1)

    old = _NNMeans(sampler, ae)
    fns = {"kernel_chamfer_per_cloud": lambda: (per_cloud(), torch.cuda.synchronize()),
           "kernel_nn_distance_plus_means": lambda: (nn_means(), torch.cuda.synchronize()),
           "curve_chamfer_per_cloud": lambda: evaluator.get_loss_ae_per_pc_progressive(pcs, sampled_pc, sizes).cpu(),
           "curve_nn_distance_plus_means": lambda: old.get_loss_ae_per_pc_progressive(pcs, sampled_pc, sizes).cpu()}
    res = {"clouds": n_clouds, "sizes": sizes, "reconstructions": p * n_clouds, "ms_per_call": alternate(fns, rounds)}
    res["max_rel_diff"] = float(((per_cloud() - nn_means()).abs() / nn_means()).max())
    res["bytes_not_written"] = 2 * p * n_clouds * 2048 * 8 + p * n_clouds * 2048 * 12     # dist + idx both ways, and the repeated reference
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--records", type=int, default=1024)
    ap.add_argument("--quick", action="store_true", help="small sizes: a rehearsal of the script, not a measurement")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluation: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "rounds": args.rounds, "quick": args.quick}
    res["registration_test_1"] = bench_registration(dev, 256 if args.quick else args.records, args.rounds)
    res["classification_progressive"] = bench_classification(dev, args.rounds, 32 if args.quick else 256, 256 if args.quick else 1024)
    res["reconstruction_progressive"] = bench_reconstruction(dev, args.rounds, 10 if args.quick else 50, [16, 32, 64, 128, 256, 512, 1024, 2048])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
