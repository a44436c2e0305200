"""Time the SampleNet trainers' epochs and the autoencoder's epoch with the data on the host, in the reference's structure, and on the device
(trainers.SamplerTrainStep, AutoencoderTrainStep.train_one_epoch), and the reconstruction augmentation kernel (ops.ae_augment).

    python tools/bench_sampler_epoch.py [--blocks 3] [--cls-clouds 9840] [--rec-clouds 4000] [--profile-steps 20]

Synthetic data: the classification set at ModelNet40's training size (9840 clouds of N = 1024 points, 40 classes), the reconstruction set
4000 clouds of N = 2048 points.

    cls_epoch   trainers.ClassificationStep: ClassificationSampleNet(32, k = 7) in front of a frozen PointNetClsTransforms
                (tasknets.FrozenPointNetClsTransforms), B = 32, Adam over the sampler
    rec_epoch   trainers.ReconstructionStep: ReconstructionSampleNet(64) in front of a frozen PointNetAE (tasknets.FrozenPointNetAE), Chamfer,
                B = 50, with the configuration's gauss_augment {"mu": 0, "sigma": 0.01} and z_rotate
    ae_epoch    trainers.AutoencoderTrainStep on tasknets.CudaPointNetAE, Chamfer, B = 50, with the same augmentation

Each epoch runs two routes, alternated in blocks:
    host    the reference's structure: a numpy shuffle, per batch the numpy augmentation (apply_augmentations, restated below) when on, a
            copy through pinned memory to the device, the step's __call__, and a read-back of its loss terms, as sess.run's float returns
    device  train_one_epoch on the device-resident set: a device shuffle, ops.ae_augment when on, one read-back per epoch
    graphed the same with graphed=True and a capturable Adam: every step one CUDA-graph replay
Every epoch starts from the same initial network and optimiser state.  The median and the spread over the blocks are reported.  TF32 is
at torch's default.  A non-finite loss stops the measurement.

    ae_augment  the kernel with a fixed key and device events at B = 50, N = 2048 and at 1024 clouds of 2048 points, noise and rotation and
                rotation alone: time per call, achieved bytes/s (12 bytes read and 12 written per point) and its share of the H100 SXM data
                sheet's 3.35 TB/s; and the numpy augmentation of one batch with the host clock.

    steps       a separate torch.profiler run of the device and graphed epochs on --profile-steps batches: GPU-busy time per step, device
                activities per step, and, unprofiled, the wall time per step (bench_classifier_epoch.step_profile)

The card's name, power limit and SM clock limit are printed with the numbers.  Prints one JSON line.  Needs a GPU.
"""
import argparse
import copy
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_classifier_epoch import _event_us, step_profile, wall  # noqa: E402
from bench_registration_task import card  # noqa: E402

CLASSES = 40
GAUSS = {"mu": 0.0, "sigma": 0.01}
HBM_BYTES_PER_S = 3.35e12


# ----------------------------------------------------------------------------------------------------- general_utils.py restated
def rand_rotation_matrix():
    theta, phi, z = np.random.uniform(size=(3,))
    theta, phi, z = theta * 2.0 * np.pi, phi * 2.0 * np.pi, z * 2.0
    r = np.sqrt(z)
    v = (np.sin(phi) * r, np.cos(phi) * r, np.sqrt(2.0 - z))
    st, ct = np.sin(theta), np.cos(theta)
    return (np.outer(v, v) - np.eye(3)).dot(np.array(((ct, st, 0), (-st, ct, 0), (0, 0, 1))))


def apply_augmentations(batch, gauss_augment, z_rotate):
    batch = batch.copy()
    if gauss_augment is not None:
        batch += np.random.normal(gauss_augment["mu"], gauss_augment["sigma"], batch.shape)
    if z_rotate:
        r = rand_rotation_matrix()
        r[0, 2] = r[2, 0] = r[1, 2] = r[2, 1] = 0
        r[2, 2] = 1
        batch = batch.dot(r)
    return batch


# ----------------------------------------------------------------------------------------------------- routes
def make_runner(kind, dev, n_points, graphed=False):
    import samplenet_b200 as sb
    from samplenet_b200 import tasknets, trainers

    torch.manual_seed(0)
    adam = lambda params, lr: torch.optim.Adam(params, lr=lr, capturable=graphed)
    if kind == "cls":
        sampler = sb.ClassificationSampleNet(32, group_size=7).to(dev)
        net = tasknets.PointNetClsTransforms(num_classes=CLASSES).to(dev).eval().requires_grad_(False)
        step = trainers.ClassificationStep(sampler, tasknets.FrozenPointNetClsTransforms(net), 32)
        return trainers.SamplerTrainStep(step, adam(sampler.parameters(), 0.01), graphed=graphed), 32
    if kind == "rec":
        sampler = sb.ReconstructionSampleNet(64).to(dev)
        ae = tasknets.FrozenPointNetAE(tasknets.PointNetAE(n_pc_points=n_points).to(dev).eval().requires_grad_(False))
        step = trainers.ReconstructionStep(sampler, ae, 64)
        return trainers.SamplerTrainStep(step, adam(sampler.parameters(), 5e-4), gauss_augment=GAUSS, z_rotate=True, graphed=graphed), 50
    ae = tasknets.CudaPointNetAE(tasknets.PointNetAE(n_pc_points=n_points).to(dev))
    return trainers.AutoencoderTrainStep(ae, adam(ae.parameters(), 5e-4), n_sample_points=n_points, batch_size=50,
                                         gauss_augment=GAUSS, z_rotate=True, graphed=graphed), 50


def _finite(values, what):
    """Stops the measurement at the first non-finite loss read back (after each host step, after each device epoch), so that no number is
    reported for a run whose sampler has gone non-finite.  It does not keep the steps before that read-back from running on such a
    sampler (DESIGN §7)."""
    if not all(np.isfinite(v) for v in values):
        raise FloatingPointError("%s: non-finite loss terms %s" % (what, values))


def make_epoch(kind, route, data, dev):
    """(epoch, reset): one epoch of the route, and a reset of the trained module and the optimiser to their initial state, so that every
    timed epoch trains the same network from the same start."""
    x_host, y_host, x_dev, y_dev = data
    n_points = x_host.shape[1]
    run, b = make_runner(kind, dev, n_points, graphed=route == "graphed")
    module = run.ae if kind == "ae" else run.task.sampler
    init_module, init_opt = copy.deepcopy(module.state_dict()), copy.deepcopy(run.optimizer.state_dict())

    def reset():
        module.load_state_dict(init_module)            # copies in place
        if route == "graphed":
            # in place as well: the captured optimizer step points at the state tensors, which load_state_dict would replace.  The initial
            # state is empty, so every tensor the first step created goes back to zero.
            from samplenet_b200 import graphs

            graphs._restore_optimizer(run.optimizer, {})
        else:
            run.optimizer.load_state_dict(init_opt)
        if kind != "ae":
            run.step = run.epoch = 0

    if route in ("device", "graphed"):
        def device():
            res = run.train_one_epoch(x_dev, y_dev) if kind == "cls" else run.train_one_epoch(x_dev)
            _finite([v for k, v in res.items() if k != "steps"], "%s device epoch" % kind)

        return device, reset
    pin_x = torch.empty(b, n_points, 3).pin_memory()
    pin_y = torch.empty(b, dtype=torch.int64).pin_memory()
    # __call__ runs with the augmentation off: the host route augments in numpy
    if kind != "cls":
        run.gauss_augment, run.z_rotate = None, False

    def host():
        idx = np.arange(x_host.shape[0])
        np.random.shuffle(idx)
        for s in range(x_host.shape[0] // b):
            sel = idx[s * b:(s + 1) * b]
            batch = x_host[sel] if kind == "cls" else apply_augmentations(x_host[sel], GAUSS, True)
            pin_x.copy_(torch.from_numpy(np.asarray(batch, dtype=np.float32)))
            xb = pin_x.to(dev, non_blocking=True)
            if kind == "cls":
                pin_y.copy_(torch.from_numpy(y_host[sel]))
                r = run(xb, pin_y.to(dev, non_blocking=True))
            elif kind == "rec":
                r = run(xb)
            else:
                r = {"loss": run(xb)}
            # the per-step read-back, as sess.run's float returns; it also frees the pinned buffers for the next batch
            _finite([float(v) for v in r.values()], "%s host step %d" % (kind, s))

    return host, reset


def alternate(routes, blocks):
    """routes: {name: (epoch, reset)}.  One untimed epoch of each, then `blocks` rounds of timed epochs in turn, each after a reset."""
    t = {k: [] for k in routes}
    for block in range(blocks + 1):
        for k, (epoch, reset) in routes.items():
            reset()
            print("epoch %s block %d" % (k, block), file=sys.stderr, flush=True)
            dt = wall(epoch)
            if block:
                t[k].append(dt)
    return {k + "_s": {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in t.items()}


def bench_augment(dev, x_host, launches=500, host_reps=20, big=1024):
    from samplenet_b200 import ops

    key = torch.empty(2, dtype=torch.int64, device=dev).random_()
    out = {}
    for name, clouds in (("B50", 50), ("B%d" % big, big)):
        x = torch.rand(clouds, 2048, 3, device=dev)
        bytes_ = 2 * clouds * 2048 * 3 * 4
        for mode, kw in (("noise_rotate", {"mu": 0.0, "sigma": 0.01, "z_rotate": True}), ("rotate", {"z_rotate": True})):
            us = _event_us(lambda: ops.ae_augment(x, key=key, **kw), launches if clouds == 50 else 50)
            out["%s_%s" % (name, mode)] = {"us": us, "GBps": bytes_ / (us * 1e3), "of_3.35TBps": bytes_ / (us * 1e-6) / HBM_BYTES_PER_S}
        del x
    xb50 = torch.rand(50, 2048, 3, device=dev)
    out["B50_call_us"] = _event_us(lambda: ops.ae_augment(xb50, 0.0, 0.01, True), launches)   # with the key draw, as the steps call it
    t0 = time.perf_counter()
    for _ in range(host_reps):
        apply_augmentations(x_host[:50], GAUSS, True)
    out["numpy_B50_us"] = (time.perf_counter() - t0) * 1e6 / host_reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--cls-clouds", type=int, default=9840)
    ap.add_argument("--rec-clouds", type=int, default=4000)
    ap.add_argument("--profile-steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampler_epoch: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    np.random.seed(0)
    rng = np.random.default_rng(1)
    x_cls = rng.random((args.cls_clouds, 1024, 3), dtype=np.float32) - 0.5
    y_cls = rng.integers(0, CLASSES, args.cls_clouds).astype(np.int64)
    x_rec = rng.random((args.rec_clouds, 2048, 3), dtype=np.float32) - 0.5
    sets = {"cls": (x_cls, y_cls, torch.from_numpy(x_cls).to(dev), torch.from_numpy(y_cls).to(dev)),
            "rec": (x_rec, None, torch.from_numpy(x_rec).to(dev), None)}
    res = {"card": card(), "blocks": args.blocks, "cls_clouds": args.cls_clouds, "rec_clouds": args.rec_clouds}
    res["ae_augment"] = bench_augment(dev, x_rec)
    for kind in ("cls", "rec", "ae"):
        data = sets["cls" if kind == "cls" else "rec"]
        r = alternate({route: make_epoch(kind, route, data, dev) for route in ("host", "device", "graphed")}, args.blocks)
        r["device_vs_host"] = r["host_s"]["median"] / r["device_s"]["median"]
        r["graphed_vs_device"] = r["device_s"]["median"] / r["graphed_s"]["median"]
        res[kind + "_epoch"] = r
        print(kind, json.dumps(r), file=sys.stderr, flush=True)
        torch.cuda.empty_cache()
        b = 32 if kind == "cls" else 50
        small = tuple(None if t is None else t[:args.profile_steps * b] for t in data)
        res[kind + "_steps"] = {route: step_profile(make_epoch(kind, route, small, dev)[0], args.profile_steps) for route in ("device", "graphed")}
        print(kind, json.dumps(res[kind + "_steps"]), file=sys.stderr, flush=True)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
