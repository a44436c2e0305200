/* samplenet_b200_debug.h -- test and benchmark entry points of libsamplenet_b200.so.  NOT part of the drop-in surface (include/samplenet_b200.h):
 * one tensor-core GEMM through the wgmma layer kernel, farthest point sampling with the threads per CTA forced, and the launch plans of
 * the conv stack, the generator and the simplification-loss entries.  Used by tools/ and tests only. */
#ifndef SAMPLENET_B200_DEBUG_H
#define SAMPLENET_B200_DEBUG_H
#include "samplenet_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Unit-test hook of the wgmma layer kernel (csrc/encoder_tc.cu): D (rows, c_out) = A (rows, c_in) * W (c_out, c_in)^T + bias
 * as 3xTF32 on the tensor cores, no BatchNorm.  c_in % 8 == 0, 8 <= c_in, c_out <= 256. */
int snb200_debug_tc_gemm(int rows, int c_in, int c_out, const float *A, const float *W, const float *bias, float *D,
                         snb200_stream_t stream);

/* snb200_farthest_point_sample with the threads per CTA forced (256, 512 or 1024; 0 = the library's choice by cloud size), so that one
 * GPU session can time every configuration on both sides of the size thresholds (tools/bench_sampling.py). */
int snb200_debug_farthest_point_sample(int b, int n, int m, int layout, const float *inp, int *idx, float *out_points, int threads,
                                       snb200_stream_t stream);

/* Host-only: how the persistent conv-stack kernel (csrc/conv_stack.cu) partitions a batch of b clouds of n points on the current device --
 * points per slice, slices, CTAs, slices per CTA (1 = the single-slice instantiation, which keeps activations in registers; more = the
 * multi-slice one) and pool partial slots per cloud.  Whether the kernel applies to a layer table is a separate question. */
int snb200_debug_conv_stack_partition(int b, int n, int *ppc, int *slices, int *grid, int *per_cta, int *slots);

/* Host-only: the path snb200_generator_forward takes for these tables, batch and flags (SNB200_GEN_*) on the current device --
 * conv_path 0 = the persistent conv-stack kernel, 1 = the per-layer tensor-core kernels, 2 = the exact-fp32 CUDA-core stack, 3 = no conv
 * stage (profiling) -- and fuse_head = 1 when the persistent kernel runs the pool and FC head itself (else the cluster head launch). */
int snb200_debug_generator_plan(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc, int flags,
                                int *conv_path, int *fuse_head);

/* Host-only launch plans of the simplification-loss entries.  The pairwise planners assume a fixed 132 SMs, so a plan does not depend on
 * the device.  snb200_project_and_loss_forward (csrc/tail.cu): projection CTAs per cloud, the input -> generated scan's lanes per query
 * (s1) and CTAs per cloud (tiles1), partial slots per cloud (ntiles = knn_ctas + tiles1), the floats of dynamic shared memory the final
 * reduction stages partials through, the clouds it stages per pass, and tma_preissue = 1 when the projection role requests the input cloud
 * by TMA before it waits on the previous grid (n_ref % 4 == 0; ref must also be 16-byte aligned). */
int snb200_debug_project_and_loss_plan(int b, int n_ref, int n_samp, int *knn_ctas, int *s1, int *tiles1, int *ntiles, int *smem_floats,
                                       int *cap_clouds, int *tma_preissue);
/* snb200_progressive_loss_forward (csrc/progressive.cu): the sample -> input scan's lanes per query (s_a) and CTAs per cloud (tiles_a),
 * the input -> sample scan's lanes per reference point (s2) and CTAs per cloud (tiles2), and the clouds whose dist1 rows the final
 * reduction stages at a time (cl_batch). */
int snb200_debug_progressive_loss_plan(int b, int n, int m, int *s_a, int *tiles_a, int *s2, int *tiles2, int *cl_batch);
/* snb200_simplification_loss_forward (csrc/chamfer.cu): the threads of its one-CTA reduction launch. */
int snb200_debug_simplification_loss_plan(int b, int *reduce_threads);

#ifdef __cplusplus
}
#endif
#endif
