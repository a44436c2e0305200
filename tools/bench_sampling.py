"""Times farthest point sampling: this library's kernel (csrc/fps.cu) against the reference's farthestpointsamplingKernel
(oracle/_ref/libsamplenet_ref_cuda.so, when built) in the same process, with CUDA events after warm-up.

    python tools/bench_sampling.py [--reps R] [--sweep-only | --no-sweep]

One JSON line per configuration: us per call, us per round (call / (m - 1)), speedup over the reference kernel, and the card's name
and power limit read in the same run.  The sweep lines time every threads-per-CTA setting on both sides of each size threshold of the
kernel's automatic choice (fps.cu: fps_auto_threads), which is how that choice was made.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from samplenet_b200 import ops  # noqa: E402

# (label, b, n, m): the callers' workloads
WORKLOADS = [
    ("rec_sort", 50, 2048, 2048),      # SamplerAutoEncoder.sort / pointnet_ae: gather_point(x, farthest_point_sample(2048, x))
    ("ae_use_fps_256", 50, 2048, 256),  # pointnet_ae.py use_fps
    ("ae_use_fps_1024", 50, 2048, 1024),
    ("reg_baseline", 32, 1024, 64),    # registration --sampler fps
    ("large_16384", 8, 16384, 1024),
]
# both sides of the automatic thresholds (n <= 1024: 256 threads, n <= 4096: 512, else 1024)
SWEEP = [("sweep", 50, n, 1024) for n in (512, 1024, 1536, 2048, 4096, 5000, 8192)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        power, clock = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
    except Exception:
        power, clock = "unknown", "unknown"
    return name, power, clock


def time_us(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1000.0 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sweep-only", action="store_true")
    ap.add_argument("--no-sweep", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sampling.py measures on a GPU"
    try:
        from oracle import ref_cuda
        have_ref = ref_cuda.available()
    except Exception:
        have_ref = False
    name, power, clock = card()
    g = torch.Generator().manual_seed(0)
    rows = ([] if args.sweep_only else WORKLOADS) + ([] if args.no_sweep else SWEEP)
    for label, b, n, m in rows:
        x = (torch.rand(b, n, 3, generator=g) - 0.5).cuda()
        rec = {"workload": label, "b": b, "n": n, "m": m, "gpu": name, "power_limit": power, "max_sm_clock": clock}
        want = ops.farthest_point_sample(x, m)
        threads = [0] if label != "sweep" else [t for t, cap in ((256, 4096), (512, 8192), (1024, 16384)) if n <= cap]
        for t in threads:
            got = ops.farthest_point_sample(x, m, _threads=t)
            assert torch.equal(got, want), (label, t)
            us = time_us(lambda: ops.farthest_point_sample(x, m, _threads=t), args.reps)
            key = "snb200" if t == 0 else "snb200_t%d" % t
            rec[key + "_us"] = round(us, 1)
            rec[key + "_us_per_round"] = round(us / max(m - 1, 1), 4)
        us = time_us(lambda: ops.farthest_point_sample(x, m, return_points=True), args.reps)
        rec["snb200_with_points_us"] = round(us, 1)
        if have_ref and label != "sweep":
            ref = ref_cuda.farthest_point_sample(m, x)
            torch.cuda.synchronize()
            rec["indices_equal_reference"] = bool(torch.equal(ref, want))
            rus = time_us(lambda: ref_cuda.farthest_point_sample(m, x), max(args.reps // 2, 3))
            rec["reference_us"] = round(rus, 1)
            rec["reference_us_per_round"] = round(rus / max(m - 1, 1), 4)
            if "snb200_us" in rec:
                rec["speedup"] = round(rus / rec["snb200_us"], 2)
        elif label != "sweep":
            rec["reference_us"] = "not measured (oracle/_ref not built)"
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
