"""Time the task networks' training steps on CUDA against the plain modules: the point-cloud autoencoder (tasknets.CudaPointNetAE) and the
two PointNet classifiers (tasknets.CudaPointNetCls, tasknets.CudaPointNetClsTransforms).

    python tools/bench_task_training.py [--steps 50] [--blocks 5]

One process, one GPU.  AutoencoderTrainStep at B = 50, N = 2048 (reconstruction/autoencoder/train_ae.py's size) with the Chamfer and with
the EMD loss, Adam(lr=5e-4), both variants from the same initial state and batch.  The variants alternate in blocks of --steps steps timed
with device events; the median and the spread over the blocks are reported.  Kernels per step come from a separate torch.profiler pass.
ClassifierTrainStep at B = 32, N = 1024 (classification/train_classifier.py's size), Adam(lr=1e-3), 40 classes, with TF32 at torch's default
and off (the plain module's convolutions and matmuls then run in exact fp32, as the wrapper's backward does); the step's loss is reported.
The card's name, power limit and SM clock limit are printed with the numbers.  Prints one JSON line.  Needs a GPU: it fails without one.
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


def make(kind, cuda, dev):
    from samplenet_b200 import tasknets, trainers

    torch.manual_seed(0)
    ae = tasknets.PointNetAE(n_pc_points=N).to(dev)
    model = tasknets.CudaPointNetAE(ae) if cuda else ae
    step = trainers.AutoencoderTrainStep(model, torch.optim.Adam(model.parameters(), lr=5e-4), ae_loss=kind)
    x = (torch.rand(B, N, 3, generator=torch.Generator().manual_seed(1)) - 0.5).to(dev)
    return model, (lambda: step(x))


CB, CN = 32, 1024


def make_classifier(cls_name, cuda, dev):
    from samplenet_b200 import tasknets, trainers

    torch.manual_seed(0)
    net = getattr(tasknets, cls_name)(num_classes=40).to(dev)
    model = getattr(tasknets, "Cuda" + cls_name)(net) if cuda else net
    step = trainers.ClassifierTrainStep(model, torch.optim.Adam(model.parameters(), lr=1e-3), batch_size=CB)
    g = torch.Generator().manual_seed(1)
    x, y = (torch.rand(CB, CN, 3, generator=g) - 0.5).to(dev), torch.randint(0, 40, (CB,), generator=g).to(dev)
    return model, (lambda: step(x, y)[0])


def bench_pair(make_fn, args):
    """Warm both variants, then alternate them in blocks; (times per variant, kernels per step, the last losses)."""
    variants = {n: make_fn(n == "cuda") for n in ("plain", "cuda")}
    fns = {n: v[1] for n, v in variants.items()}
    for n in fns:
        for _ in range(5):
            fns[n]()
    assert variants["cuda"][0].route == "cuda", variants["cuda"][0].route
    torch.cuda.synchronize()
    t = {n: [] for n in fns}
    for _ in range(args.blocks):
        for n in fns:
            t[n].append(timed(fns[n], args.steps))
    out = {}
    for n in fns:
        out[n + "_us"] = {"median": statistics.median(t[n]), "min": min(t[n]), "max": max(t[n])}
        out[n + "_kernels_per_step"] = kernels_per_step(fns[n], keys=())[0]
        out[n + "_loss"] = float(fns[n]())
    out["speedup_of_medians"] = out["plain_us"]["median"] / out["cuda_us"]["median"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--blocks", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_task_training: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "B": B, "N": N, "steps_per_block": args.steps, "blocks": args.blocks}
    for kind in ("chamfer", "emd"):
        variants = {n: make(kind, n == "cuda", dev) for n in ("plain", "cuda")}
        fns = {n: v[1] for n, v in variants.items()}
        for n in fns:
            for _ in range(5):
                fns[n]()
        assert variants["cuda"][0].route == "cuda", variants["cuda"][0].route
        torch.cuda.synchronize()
        t = {n: [] for n in fns}
        for _ in range(args.blocks):
            for n in fns:
                t[n].append(timed(fns[n], args.steps))
        for n in fns:
            res["%s_%s_us" % (kind, n)] = {"median": statistics.median(t[n]), "min": min(t[n]), "max": max(t[n])}
            res["%s_%s_kernels_per_step" % (kind, n)] = kernels_per_step(fns[n], keys=())[0]
        res["%s_speedup_of_medians" % kind] = res["%s_plain_us" % kind]["median"] / res["%s_cuda_us" % kind]["median"]
        del variants, fns
        torch.cuda.empty_cache()
    for cls_name in ("PointNetCls", "PointNetClsTransforms"):
        for tf32 in (True, False):
            prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = prev[0] and tf32
            r = bench_pair(lambda cuda: make_classifier(cls_name, cuda, dev), args)
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
            res["%s_B%d_N%d_tf32_%s" % (cls_name, CB, CN, "default" if tf32 else "off")] = r
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
