"""Warm, in-graph time of each stage of the step: a CUDA graph holding R back-to-back launches of ONE stage is replayed and
the CUDA-event time is divided by R.  This is the marginal cost of the stage inside the real step graph (launch gap
included), which the cold-cache, serialised ncu launch list overstates for the small kernels.

    python tools/kernel_times.py [--batch 32] > kernel_times.json
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import samplenet_b200 as sb  # noqa: E402


def graph_time(fn, reps=20, replays=20):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn(); fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(replays):
        g.replay()
    b.record(); b.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * replays)  # us per launch of the stage


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--points", type=int, default=1024)
    ap.add_argument("--out-points", type=int, default=64)
    ap.add_argument("--k", type=int, default=8)
    a = ap.parse_args()
    B, N, M, K = a.batch, a.points, a.out_points, a.k
    torch.manual_seed(0)
    net = sb.SampleNet(M, 128, group_size=K, input_shape="bnc", output_shape="bnc").cuda().train()
    x = (torch.rand(B, N, 3, device="cuda") - 0.5)
    conv, fc = net._layer_specs()
    out = {}
    with torch.no_grad():
        simp = net(x)[0].detach()
        sigma = net.project.sigma().detach().reshape(1).contiguous()
        out["generator_total"] = graph_time(lambda: sb.ops.generator_forward(x, "bnc", conv, fc, True, M))
        out["generator_conv_only"] = graph_time(lambda: sb.ops.generator_forward(x, "bnc", conv, fc, True, M, _profile_flags=2))
        out["generator_head_only_cluster_kernel"] = graph_time(lambda: sb.ops.generator_forward(x, "bnc", conv, fc, True, M, _profile_flags=4))
        out["generator_total_separate_head"] = graph_time(lambda: sb.ops.generator_forward(x, "bnc", conv, fc, True, M, separate_head=True))
        out["generator_exact_fp32_total"] = graph_time(lambda: sb.ops.generator_forward(x, "bnc", conv, fc, True, M, exact_fp32=True), reps=5)
        widths = [64, 64, 64, 128, 128]
        for l in range(1, 5):
            A = torch.randn(B * N, widths[l - 1], device="cuda")
            W = torch.randn(widths[l], widths[l - 1], device="cuda") / widths[l - 1] ** 0.5
            bias = torch.zeros(widths[l], device="cuda")
            out["tc_layer_%d_%dto%d" % (l + 1, widths[l - 1], widths[l])] = graph_time(lambda: sb.ops.debug_tc_gemm(A, W, bias))
        out["knn_softproj"] = graph_time(lambda: sb.ops.knn_soft_project_forward(x, simp, K, "bnc", sigma, want=("proj", "idx", "weights", "dist")))
        out["chamfer_fwd"] = graph_time(lambda: sb.ops.nn_distance_forward(simp, x))
        out["chamfer_fwd+reduce"] = graph_time(lambda: sb.ops.simplification_loss_forward(simp, x, 1.0))
        out["tail_fused_project_chamfer_loss"] = graph_time(lambda: sb.ops.project_and_loss_forward(x, simp, K, net.project._temperature, 1, 1e-2, 1.0))
        xb = torch.empty_like(x)
        out["input_copy_d2d"] = graph_time(lambda: xb.copy_(x))
        step = sb.GraphedStep(net, B, N)
        a_, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(5):
            step(x)
        torch.cuda.synchronize()
        a_.record()
        for _ in range(200):
            step(x)
        b_.record(); b_.synchronize()
        out["whole_step_graph"] = a_.elapsed_time(b_) * 1e3 / 200
        out["launches_per_step"] = int(step.launches_per_step)
    out["unit"] = "us per launch, warm, in-graph"
    out["shape"] = dict(B=B, N=N, M=M, k=K)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
