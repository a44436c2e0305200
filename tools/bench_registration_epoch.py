"""Time one training epoch of the registration trainer (registration/main.py:306-362) with the reference's host data path and with the
device-resident set.

    python tools/bench_registration_epoch.py [--blocks 3] [--clouds 197] [--points 2048] [--profile-steps 20]

Synthetic data at the "car" set's size: 197 training clouds of 2048 points, repeated int(5000 / 197) = 25 times, so an epoch is 4925
records in 154 batches of B = 32, N = 1024 points per cloud.

    epoch        one epoch of RegistrationStep.train_step over the set, for two models:
                   pcrnet     sampler="none", train_pcrnet=True, create_model(cuda_task=True) (the README's PCRNet run)
                   samplenet  sampler="samplenet", create_model(frozen_task=True), Adam over the sampler
                 along three routes:
                   host    the reference's data path, restated below: ModelNetCls.__getitem__ (a numpy permutation of the first N points),
                           OnUnitCube.method2 and QuaternionFixedDataset.__getitem__ (qrot on the host) in a
                           DataLoader(batch_size=32, shuffle=True, num_workers=4), then train_step and two .item() calls per batch
                   device  registration.CudaQuaternionFixedDataset(...).batches(32, shuffle=True) + RegistrationStep.train_1 (one read-back)
                   graphed the same with RegistrationStep(graphed=True) and Adam(capturable=True): every whole batch one CUDA-graph
                           replay, the trailing partial batch (4925 = 153 x 32 + 29) eager
    data         the same two data paths without a step: the DataLoader epoch with each batch copied to the device, and the set's batches
    pairs        ops.registration_pairs at B = 32 with device events over 1000 calls, as batch() calls it (the key draw and the kernel) and
                 with a fixed key (the kernel alone), its throughput at B = 4096, and its share of the device route's mean step
    steps        a separate torch.profiler run of the device and graphed routes over --profile-steps whole batches, for each model: GPU-busy
                 time per step, device activities per step, and, unprofiled, the wall time per step (bench_classifier_epoch.step_profile)

The routes alternate in blocks; the median and the spread over the blocks are reported.  TF32 is at torch's default.  The card's name,
power limit and SM clock limit are printed with the numbers.  Prints one JSON line.  Needs a GPU.
"""
import argparse
import itertools
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_classifier_epoch import _event_us, alternate, step_profile  # noqa: E402
from bench_registration_task import card  # noqa: E402

B, N, WORKERS = 32, 1024, 4


# ----------------------------------------------------------------------------------------------------- the reference's data path restated
class HostModelNetCls(torch.utils.data.Dataset):
    """ModelNetCls(num_points, Compose([PointcloudToTensor(), OnUnitCube()])) over clouds already read (modelnet_loader_torch.py:102-116)."""

    def __init__(self, points, num_points):
        self.points, self.num_points = points, min(points.shape[1], num_points)

    def __getitem__(self, idx):
        pt_idxs = np.arange(0, self.num_points)
        np.random.shuffle(pt_idxs)
        current_points = torch.from_numpy(self.points[idx, pt_idxs].copy()).float()
        c = torch.max(current_points, dim=0)[0] - torch.min(current_points, dim=0)[0]     # OnUnitCube.method2
        v = current_points / torch.max(c)
        return v - v.mean(dim=0, keepdim=True), torch.zeros(1, dtype=torch.int64)

    def __len__(self):
        return self.points.shape[0]


class HostQuaternionFixedDataset(torch.utils.data.Dataset):
    """QuaternionFixedDataset(data, repeat, seed) (qdataset.py:122-179): a fixed QuaternionTransform per record, p1 = rotate(p0) on the host."""

    def __init__(self, data, repeat=1, seed=0):
        from samplenet_b200.registration import QuaternionTransform, random_transforms

        self.data, self.len_data = data, len(data)
        self.transforms = [QuaternionTransform(torch.from_numpy(row[None].copy())) for row in random_transforms(len(data) * repeat, seed)]

    def __len__(self):
        return len(self.transforms)

    def __getitem__(self, index):
        p0, _ = self.data[index % self.len_data]
        gt = self.transforms[index]
        return p0, gt.rotate(p0), gt.as_dict()


# ----------------------------------------------------------------------------------------------------- routes
def make_model(kind, dev, graphed=False):
    from samplenet_b200.registration import RegistrationStep

    torch.manual_seed(0)
    if kind == "pcrnet":
        act = RegistrationStep(sampler="none", train_pcrnet=True, graphed=graphed)
        model = act.create_model(cuda_task=True).to(dev)
    else:
        act = RegistrationStep(sampler="samplenet", graphed=graphed)
        model = act.create_model(frozen_task=True).to(dev)
    opt = torch.optim.Adam(filter(lambda p: p.requires_grad, model.parameters()), lr=1e-3, capturable=graphed)
    return act, model, opt


def make_epoch(kind, route, loader, ds, dev, steps=None):
    """One epoch of the route; steps: only the first `steps` batches of each epoch (device and graphed routes)."""
    act, model, opt = make_model(kind, dev, graphed=route == "graphed")
    if route in ("device", "graphed"):
        return lambda: act.train_1(model, itertools.islice(ds.batches(B, shuffle=True), steps), opt, dev)

    def run():   # main.py:306-362 over the DataLoader: two .item() calls per batch
        vloss, gloss, count = 0.0, 0.0, 0
        for data in loader:
            loss, rot, _ = act.train_step(model, data, opt, dev)
            vloss += loss.item()
            gloss += rot.item()
            count += 1
        return vloss / count, gloss / count

    return run


def make_data(route, loader, ds, dev):
    if route == "device":
        def run():
            for p0, p1, igt in ds.batches(B, shuffle=True):
                pass
        return run

    def run():
        for p0, p1, igt in loader:
            p0.to(dev), p1.to(dev), igt["vec"].to(dev)
    return run


def bench_pairs(ds, dev, launches=1000, big=4096):
    from samplenet_b200 import ops

    rec = torch.randperm(len(ds), device=dev, dtype=torch.int32)[:B]
    key = torch.empty(2, dtype=torch.int64, device=dev).random_()
    call_us = _event_us(lambda: ops.registration_pairs(ds.clouds, rec, ds.transforms), launches)
    kernel_us = _event_us(lambda: ops.registration_pairs(ds.clouds, rec, ds.transforms, key=key), launches)
    rec_big = torch.randint(0, len(ds), (big,), device=dev, dtype=torch.int32)
    big_us = _event_us(lambda: ops.registration_pairs(ds.clouds, rec_big, ds.transforms, key=key), 50)
    n = ds.num_points
    big_bytes = big * n * (12 + 24) + big * (4 + 2 * 28)     # gathered points read once, p0 and p1 written; records, rows read, vec written
    return {"call_us_B32": call_us, "fixed_key_us_B32": kernel_us, "big_pairs": big, "big_us": big_us, "big_GBps": big_bytes / (big_us * 1e3),
            "big_pairs_per_s": big / (big_us * 1e-6)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--clouds", type=int, default=197)
    ap.add_argument("--points", type=int, default=2048)
    ap.add_argument("--profile-steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_registration_epoch: no CUDA device (this measurement has no CPU path)")
    from samplenet_b200 import registration

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    np.random.seed(0)
    rng = np.random.default_rng(1)
    points = (rng.random((args.clouds, args.points, 3), dtype=np.float32) * np.array([2.0, 1.2, 0.8], np.float32) - 0.5).astype(np.float32)
    repeat = max(int(5000 / args.clouds), 1)
    host_set = HostQuaternionFixedDataset(HostModelNetCls(points, N), repeat=repeat, seed=0)
    loader = torch.utils.data.DataLoader(host_set, batch_size=B, shuffle=True, num_workers=WORKERS)
    ds = registration.CudaQuaternionFixedDataset(points, num_points=N, repeat=repeat, seed=0)
    steps = (len(ds) + B - 1) // B
    res = {"card": card(), "B": B, "N": N, "clouds": args.clouds, "points": args.points, "records": len(ds), "steps_per_epoch": steps,
           "workers": WORKERS, "blocks": args.blocks}
    res["pairs"] = bench_pairs(ds, dev)
    r = alternate({route: make_data(route, loader, ds, dev) for route in ("host", "device")}, args.blocks)
    r["device_vs_host"] = r["host_s"]["median"] / r["device_s"]["median"]
    res["data"] = r
    for kind in ("pcrnet", "samplenet"):
        r = alternate({route: make_epoch(kind, route, loader, ds, dev) for route in ("host", "device", "graphed")}, args.blocks)
        r["device_vs_host"] = r["host_s"]["median"] / r["device_s"]["median"]
        r["graphed_vs_device"] = r["device_s"]["median"] / r["graphed_s"]["median"]
        for route in ("host", "device", "graphed"):
            r[route + "_step_ms"] = r[route + "_s"]["median"] * 1e3 / steps
        r["pairs_call_share_of_device_step"] = res["pairs"]["call_us_B32"] * 1e-3 / r["device_step_ms"]
        res["epoch_" + kind] = r
        print(kind, json.dumps(r), file=sys.stderr, flush=True)
        torch.cuda.empty_cache()
        res["steps_" + kind] = {route: step_profile(make_epoch(kind, route, loader, ds, dev, steps=args.profile_steps), args.profile_steps)
                                for route in ("device", "graphed")}
        print(kind, json.dumps(res["steps_" + kind]), file=sys.stderr, flush=True)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
