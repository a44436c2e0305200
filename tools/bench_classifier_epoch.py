"""Time the classification trainer's augmented training epoch and the rotation-vote evaluation (classification/train_classifier.py and
evaluate_classifier.py) with the data on the host and on the device.

    python tools/bench_classifier_epoch.py [--blocks 3] [--train-clouds 9840] [--test-clouds 2468] [--profile-clouds 640]

Synthetic data at ModelNet40's sizes: 9840 training clouds and 2468 test clouds of N = 1024 points, 40 classes, batches of B = 32.

    epoch        one training epoch of tasknets.CudaPointNetCls and CudaPointNetClsTransforms through trainers.ClassifierTrainStep:
                   host    the reference's loop: shuffle, then per batch provider.rotate_point_cloud + jitter_point_cloud in numpy (restated
                           below), a copy through pinned memory to the device and ClassifierTrainStep.__call__ (one read-back per step)
                   device  ClassifierTrainStep(augment=True).train_one_epoch on the device-resident set (one read-back per epoch)
                   graphed the same with graphed=True and a capturable Adam: every step one CUDA-graph replay
    steps        a separate torch.profiler run of the device and graphed epochs on --profile-clouds clouds: GPU-busy time per step (the
                 sum of the device activities' durations), device activities per step, and, unprofiled, the wall time per step
    augment      ops.rotate_jitter on one batch of 32 clouds with device events over 1000 calls: as the step calls it (the key draw and the
                 kernel) and with a fixed key (the kernel alone); its throughput at 4096 clouds; against the numpy functions timed with the
                 host clock and the pinned copy of their output, which the host route adds
    evaluation   evaluation.ClassifierEvaluator at 1 and 12 votes through FrozenPointNetClsTransforms on the test set, against a loop over
                 votes in the reference's structure: per vote ops.rotate_by_angles with one angle, one classifier call and get_loss

The routes alternate in blocks; the median and the spread over the blocks are reported.  TF32 is at torch's default.  The card's name,
power limit and SM clock limit are printed with the numbers.  Prints one JSON line.  Needs a GPU.
"""
import argparse
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

from bench_registration_task import card  # noqa: E402

B, N, CLASSES = 32, 1024, 40


# ----------------------------------------------------------------------------------------------------- provider.py restated
def rotate_point_cloud(batch_data):
    rotated_data = np.zeros(batch_data.shape, dtype=np.float32)
    for k in range(batch_data.shape[0]):
        rotation_angle = np.random.uniform() * 2 * np.pi
        cosval, sinval = np.cos(rotation_angle), np.sin(rotation_angle)
        rotation_matrix = np.array([[cosval, 0, sinval], [0, 1, 0], [-sinval, 0, cosval]])
        rotated_data[k, ...] = np.dot(batch_data[k, ...].reshape((-1, 3)), rotation_matrix)
    return rotated_data


def jitter_point_cloud(batch_data, sigma=0.01, clip=0.05):
    jittered_data = np.clip(sigma * np.random.randn(*batch_data.shape), -1 * clip, clip)
    jittered_data += batch_data
    return jittered_data


# ----------------------------------------------------------------------------------------------------- routes
def make_epoch(wrapper_name, route, data, dev):
    from samplenet_b200 import tasknets, trainers

    x_host, y_host, x_dev, y_dev = data
    torch.manual_seed(0)
    module = tasknets.PointNetCls() if wrapper_name == "CudaPointNetCls" else tasknets.PointNetClsTransforms()
    w = getattr(tasknets, wrapper_name)(module.to(dev))
    graphed = route == "graphed"
    opt = torch.optim.Adam(w.parameters(), lr=1e-3, capturable=graphed)
    step = trainers.ClassifierTrainStep(w, opt, batch_size=B, augment=(route != "host"), graphed=graphed)
    if route != "host":
        return lambda: step.train_one_epoch(x_dev, y_dev)
    pin_x = torch.empty(B, N, 3).pin_memory()
    pin_y = torch.empty(B, dtype=torch.int64).pin_memory()

    def run():
        idx = np.arange(x_host.shape[0])
        np.random.shuffle(idx)
        for s in range(x_host.shape[0] // B):
            sel = idx[s * B:(s + 1) * B]
            pin_x.copy_(torch.from_numpy(jitter_point_cloud(rotate_point_cloud(x_host[sel])).astype(np.float32)))
            pin_y.copy_(torch.from_numpy(y_host[sel]))
            step(pin_x.to(dev, non_blocking=True), pin_y.to(dev, non_blocking=True))   # __call__ reads back, so the buffers are free after it

    return run


def make_eval(route, votes, data, dev):
    from samplenet_b200 import evaluation, ops, tasknets

    x, y = data
    torch.manual_seed(0)
    frozen = tasknets.FrozenPointNetClsTransforms(tasknets.PointNetClsTransforms().to(dev).eval().requires_grad_(False))
    if route == "evaluator":
        ev = evaluation.ClassifierEvaluator(frozen, num_votes=votes)
        return lambda: ev.evaluate(x, y)["accuracy"]
    angles = [v / float(votes) * np.pi * 2 for v in range(votes)]

    def run():
        preds, loss_sum = [], 0.0
        with torch.no_grad():
            for s in range(0, x.shape[0], B):
                pc, lab = x[s:s + B], y[s:s + B]
                summed, batch_loss = 0.0, 0.0
                for a in angles:
                    pred, end_points = frozen(ops.rotate_by_angles(pc, [a])[0])
                    summed = summed + pred.double()
                    batch_loss = batch_loss + frozen.get_loss(pred, lab, end_points).double() * pc.shape[0] / votes
                loss_sum = loss_sum + batch_loss
                preds.append(summed.argmax(1))
        return float((torch.cat(preds) == y).double().mean()), float(loss_sum / x.shape[0])

    return run


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def alternate(fns, blocks):
    for fn in fns.values():
        fn()
    t = {k: [] for k in fns}
    for _ in range(blocks):
        for k, fn in fns.items():
            t[k].append(wall(fn))
    return {k + "_s": {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in t.items()}


def step_profile(epoch, steps):
    """epoch() runs `steps` steps.  After one untimed epoch (a graphed runner captures there): the wall time per step of one epoch, and in
    a separate epoch under torch.profiler the GPU-busy time per step (the sum of the CUDA activities' durations: kernels, memsets, copies)
    and the number of those activities per step."""
    from torch.profiler import ProfilerActivity, profile

    epoch()
    wall_s = wall(epoch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        epoch()
        torch.cuda.synchronize()
    acts = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    busy_us = sum(getattr(e, "device_time", None) or e.cuda_time for e in acts)
    return {"wall_ms_per_step": wall_s * 1e3 / steps, "gpu_busy_ms_per_step": busy_us / 1e3 / steps, "gpu_activities_per_step": len(acts) / steps}


def _event_us(fn, launches):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(10):
        fn()
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / launches


def bench_augment(x_host, dev, launches=1000, host_reps=50, big=4096):
    """One batch: ops.rotate_jitter as the step calls it (the key draw and the kernel) and the kernel alone with a fixed key; the throughput
    at `big` clouds (the kernel with a fixed key); the numpy functions and the pinned copy of their output."""
    from samplenet_b200 import ops

    xb = torch.from_numpy(x_host[:B]).to(dev)
    key = torch.empty(2, dtype=torch.int64, device=dev).random_()
    call_us = _event_us(lambda: ops.rotate_jitter(xb), launches)
    kernel_us = _event_us(lambda: ops.rotate_jitter(xb, key=key), launches)
    xbig = torch.rand(big, N, 3, device=dev)
    big_us = _event_us(lambda: ops.rotate_jitter(xbig, key=key), 50)
    pin = torch.empty(B, N, 3).pin_memory()
    t0 = time.perf_counter()
    for _ in range(host_reps):
        out = jitter_point_cloud(rotate_point_cloud(x_host[:B])).astype(np.float32)
    numpy_us = (time.perf_counter() - t0) * 1e6 / host_reps
    t0 = time.perf_counter()
    for _ in range(host_reps):
        pin.copy_(torch.from_numpy(out))
        pin.to(dev, non_blocking=True)
        torch.cuda.synchronize()
    copy_us = (time.perf_counter() - t0) * 1e6 / host_reps
    big_bytes = 2 * big * N * 3 * 4
    return {"rotate_jitter_call_us": call_us, "rotate_jitter_fixed_key_us": kernel_us, "numpy_us": numpy_us, "pinned_copy_us": copy_us,
            "big_clouds": big, "big_us": big_us, "big_GBps": big_bytes / (big_us * 1e3), "big_points_per_s": big * N / (big_us * 1e-6)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--train-clouds", type=int, default=9840)
    ap.add_argument("--test-clouds", type=int, default=2468)
    ap.add_argument("--profile-clouds", type=int, default=640)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_classifier_epoch: no CUDA device (this measurement has no CPU path)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    np.random.seed(0)
    rng = np.random.default_rng(1)
    x_host = (rng.random((args.train_clouds, N, 3), dtype=np.float32) * 2 - 1)
    y_host = rng.integers(0, CLASSES, args.train_clouds).astype(np.int64)
    train = (x_host, y_host, torch.from_numpy(x_host).to(dev), torch.from_numpy(y_host).to(dev))
    test = (torch.from_numpy(rng.random((args.test_clouds, N, 3), dtype=np.float32) * 2 - 1).to(dev),
            torch.from_numpy(rng.integers(0, CLASSES, args.test_clouds)).to(dev))
    res = {"card": card(), "B": B, "N": N, "train_clouds": args.train_clouds, "test_clouds": args.test_clouds, "blocks": args.blocks,
           "steps_per_epoch": args.train_clouds // B}
    res["augment"] = bench_augment(x_host, dev)
    for name in ("CudaPointNetCls", "CudaPointNetClsTransforms"):
        r = alternate({route: make_epoch(name, route, train, dev) for route in ("host", "device", "graphed")}, args.blocks)
        r["device_vs_host"] = r["host_s"]["median"] / r["device_s"]["median"]
        r["graphed_vs_device"] = r["device_s"]["median"] / r["graphed_s"]["median"]
        res["epoch_" + name] = r
        torch.cuda.empty_cache()
        small = tuple(t[:args.profile_clouds] for t in train)
        res["steps_" + name] = {route: step_profile(make_epoch(name, route, small, dev), args.profile_clouds // B) for route in ("device", "graphed")}
        torch.cuda.empty_cache()
    for votes in (1, 12):
        r = alternate({route: make_eval(route, votes, test, dev) for route in ("evaluator", "vote_loop")}, args.blocks)
        r["evaluator_vs_vote_loop"] = r["vote_loop_s"]["median"] / r["evaluator_s"]["median"]
        res["eval_%d_votes" % votes] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
