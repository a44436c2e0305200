"""Phase timeline of the persistent conv stack (`conv_stack_kernel`) at the headline shape: where a launch's time goes, per layer and slice.

    python tools/conv_stack_timeline.py [--source A.cu [--source B.cu]] [--rounds R] [--reps N] [--batch 32] [--json OUT]

Each source (default: the package's own conv_stack.cu) is compiled with -DSNB200_CS_TIMELINE into a copy of the library in a temporary
directory (the other objects are the in-tree build's).  With that macro, thread 0 of every CTA stamps %clock64 and %globaltimer at the
phase boundaries of the launch (see CS_TL in conv_stack.cu); the default build contains no stamp.  Each build then runs in a child
process, the builds alternating for R rounds: SampleNet(64, 128, group_size=8) in train mode on the bench's synthetic batch, the
generator forward (conv stack + fused FC head, one launch) warmed up and then launched N times, one synchronise and read-back per
launch.  Intervals are taken from %clock64 (per-CTA cycle counts) and converted to microseconds with each CTA's own clock rate
(cycles over globaltimer nanoseconds across the launch).  For every interval the table prints the median and the maximum over the CTAs,
each the median over the N launches.

Phases per (tensor layer, slice):
  reload   the slice's input: the parked raw rows from L2 (layer 1: the points and layer 1 on CUDA cores)
  prep     BatchNorm / ReLU of the input, TF32 hi / lo split and operand stores, up to the CTA barrier
  mma      the MMAs of thread 0's warpgroup: first weight load up to wgmma.wait_group 0
  staging  accumulator fragments -> shared memory -> this thread's channel, with the CTA barriers around it
  stats    statistics, extrema and parking of the raw outputs
per layer: `xchg` = end of the previous layer (phase 0 for the first) up to the statistics exchange being done (cs_fx_collect and the
CTA barriers that share it) and `tail` = last slice up to the end of the layer (the statistics contribution; the grid barrier in the last
layer); per launch: phase 0 (input moments and their grid barrier) and the head (pool finalise + FC head) as one interval each.
"""
import argparse
import ctypes
import glob
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "samplenet_b200", "csrc")
PHASES = ("reload", "prep", "mma", "staging", "stats")


def _build_module():
    import importlib.util

    spec = importlib.util.spec_from_file_location("snb200_build", os.path.join(CSRC, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def build_variant(source, outdir):
    """conv_stack.cu from `source` with the timeline stamps, linked with the in-tree objects of every other source -> outdir/lib/*.so"""
    bm = _build_module()
    bm.build()   # the in-tree objects (no-op when they are current)
    objs = [o for o in sorted(glob.glob(os.path.join(bm.OBJ, "*.o"))) if os.path.basename(o) != "conv_stack.o"]
    obj = os.path.join(outdir, "conv_stack_timeline.o")
    cmd = [bm.NVCC] + bm.FLAGS + ["-DSNB200_CS_TIMELINE", "-I", CSRC, "-I", os.path.join(ROOT, "include"), "-c", source, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s" % (source, r.stderr))
    lib = os.path.join(outdir, "lib", "libsamplenet_b200.so")
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    cmd = [bm.NVCC, "-shared", "-o", lib, obj] + objs + ["-gencode", "arch=compute_90a,code=" + bm.ARCH, "-lcudart_static", "-Xcompiler", "-fPIC"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s" % r.stderr)
    return lib


def _intervals(st, nl, ns, per_layer, head):
    """one CTA's stamps [stamps][2] -> {name: microseconds}; intervals with a missing end point are left out"""
    c, t = st[:, 0].astype("float64"), st[:, 1].astype("float64")
    end = head + 1
    if not (c[0] and c[end]) or t[end] <= t[0]:
        return None
    cyc_per_us = (c[end] - c[0]) / ((t[end] - t[0]) * 1e-3)
    out = {"_mhz": cyc_per_us}

    def iv(name, a, b):
        if c[a] and c[b]:
            out[name] = (c[b] - c[a]) / cyc_per_us

    iv("phase0", 0, 1)
    iv("conv_total", 0, head)
    iv("head", head, end)
    prev_end = 1
    for l in range(1, nl + 1):
        base = 2 + (l - 1) * per_layer
        iv("L%d xchg" % l, prev_end, base)
        prev = base
        for s in range(ns):
            for k, ph in enumerate(PHASES):
                a = base + 1 + 5 * s + k
                if c[a]:
                    iv("L%d s%d %s" % (l, s, ph), prev, a)
                    prev = a
        iv("L%d tail" % l, prev, base + per_layer - 1)
        prev_end = base + per_layer - 1
    return out


def run_child(lib_path, reps, batch, warmup):
    """load the timeline library, launch the generator, return {interval: [median over CTAs, max over CTAs] per launch}"""
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch

    import samplenet_b200 as sb

    sb._lib.LIB_PATH = lib_path
    h = sb._lib.lib()
    raw = ctypes.CDLL(lib_path)   # the same loaded image: the two timeline entries are not part of the bound C ABI
    mc, msl, pl, hd = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    nst = raw.snb200_cs_timeline_layout(ctypes.byref(mc), ctypes.byref(msl), ctypes.byref(pl), ctypes.byref(hd))
    assert h is not None and nst > 0
    buf = np.zeros((mc.value, nst, 2), dtype=np.uint64)
    fn = raw.snb200_cs_timeline
    fn.argtypes = [ctypes.c_void_p, ctypes.c_size_t]

    import bench

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    net = sb.SampleNet(bench.M, bench.BOTTLENECK, group_size=bench.K_NN, initial_temperature=1.0, input_shape="bnc", output_shape="bnc").to(dev).train()
    x = bench.synth_batch(0, b=batch).to(dev)
    conv, fc = net._layer_specs()
    nl = len(conv) - 1
    per = {}
    mhz = []
    with torch.no_grad():
        for _ in range(warmup):
            sb.ops.generator_forward(x, "bnc", conv, fc, True, bench.M)
        torch.cuda.synchronize()
        assert fn(buf.ctypes.data, buf.nbytes) == nst
        for _ in range(reps):
            sb.ops.generator_forward(x, "bnc", conv, fc, True, bench.M)
            torch.cuda.synchronize()
            assert fn(buf.ctypes.data, buf.nbytes) == nst
            ctas = [iv for iv in (_intervals(buf[i], nl, msl.value, pl.value, hd.value) for i in range(mc.value)) if iv]
            mhz.append(statistics.median(iv["_mhz"] for iv in ctas))
            names = {k for iv in ctas for k in iv if k != "_mhz"}
            for k in names:
                vals = [iv[k] for iv in ctas if k in iv]
                per.setdefault(k, []).append((statistics.median(vals), max(vals), len(vals)))
    res = {k: [statistics.median(v[0] for v in vs), statistics.median(v[1] for v in vs), vs[0][2]] for k, vs in per.items()}
    return {"intervals": res, "sm_mhz": statistics.median(mhz), "gpu": torch.cuda.get_device_name(0), "layers": nl}


def _order(name):
    if not name.startswith("L"):
        return (0 if name == "phase0" else 99, 0, 0, name)
    parts = name.split()
    l = int(parts[0][1:])
    if parts[1] == "xchg":
        return (l, -1, 0, "")
    if parts[1] == "tail":
        return (l, 99, 0, "")
    return (l, int(parts[1][1:]), PHASES.index(parts[2]), "")


def print_table(label, runs):
    """runs: child results of one build (one per round) -> one markdown table, medians over the rounds"""
    keys = sorted(set().union(*(r["intervals"].keys() for r in runs)), key=_order)
    print("\n### %s  (%s, SM clock ~%.0f MHz, %d round(s))" % (label, runs[0]["gpu"], statistics.median(r["sm_mhz"] for r in runs), len(runs)))
    print("| interval | median over CTAs, µs | max over CTAs, µs | CTAs |")
    print("|---|---|---|---|")
    for k in keys:
        vs = [r["intervals"][k] for r in runs if k in r["intervals"]]
        print("| %s | %.2f | %.2f | %d |" % (k, statistics.median(v[0] for v in vs), statistics.median(v[1] for v in vs), vs[0][2]))
    # the slice body summed over slices and layers, per phase (median CTA)
    print("| **per phase, all layers and slices** | | | |")
    for ph in PHASES + ("xchg", "tail"):
        tot = sum(statistics.median(r["intervals"][k][0] for r in runs if k in r["intervals"]) for k in keys if k.endswith(" " + ph))
        print("| %s | %.2f | | |" % (ph, tot))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--source", action="append", help="conv_stack.cu to instrument (repeatable; default: the package's)")
    ap.add_argument("--label", action="append", help="a name per --source")
    ap.add_argument("--rounds", type=int, default=2, help="child runs per build, builds alternating")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--json", default=None, help="write every child's raw result here")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        print("TIMELINE_JSON " + json.dumps(run_child(a.child, a.reps, a.batch, a.warmup)))
        return
    sources = a.source or [os.path.join(CSRC, "conv_stack.cu")]
    labels = a.label or [os.path.relpath(s, ROOT) for s in sources]
    with tempfile.TemporaryDirectory(prefix="cs_timeline_") as tmp:
        libs = []
        for i, s in enumerate(sources):
            d = os.path.join(tmp, "v%d" % i)
            os.makedirs(d)
            libs.append(build_variant(os.path.abspath(s), d))
        results = {lab: [] for lab in labels}
        for _ in range(a.rounds):
            for lab, lib in zip(labels, libs):
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", lib, "--reps", str(a.reps), "--batch", str(a.batch),
                                    "--warmup", str(a.warmup)], capture_output=True, text=True, cwd=ROOT)
                line = [ln for ln in r.stdout.splitlines() if ln.startswith("TIMELINE_JSON ")]
                if r.returncode != 0 or not line:
                    raise RuntimeError("timeline run failed (%s):\n%s\n%s" % (lab, r.stdout[-2000:], r.stderr[-4000:]))
                results[lab].append(json.loads(line[0][len("TIMELINE_JSON "):]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)
    for lab in labels:
        print_table(lab, results[lab])


if __name__ == "__main__":
    main()
