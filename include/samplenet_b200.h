/*
 * samplenet_b200.h -- C ABI of libsamplenet_b200.so: SampleNet's sampling-and-loss hot path as
 * hand-written sm_90a CUDA.  This is the drop-in boundary: every entry point below replaces one of the
 * reference's native launchers (cited per function, paths relative to the reference tree) and keeps that
 * launcher's calling convention -- plain sizes + raw DEVICE pointers owned by the caller -- with three
 * deliberate differences (SURVEY.md 8b):
 *   1. every call takes the CUDA stream to launch on (the reference launchers use the legacy default stream);
 *   2. every call returns 0 on success or a negative SNB200_E* code and records a message retrievable with
 *      snb200_last_error() (the reference printf()s and carries on);
 *   3. the library allocates nothing: scratch is passed in, sized by the matching *_workspace_bytes() query.
 * All entry points are re-entrant (no global state besides the thread-local error string) and asynchronous
 * (they only enqueue work on `stream`; they never synchronise, so they can be captured into CUDA graphs).
 *
 * Layout tags: SNB200_BNC = (batch, points, channels) contiguous (the TF ops and ChamferDistance);
 *              SNB200_BCN = (batch, channels, points) contiguous (registration/src SoftProjection / SampleNet).
 * dtypes: float32 and int32 only (snb200_nonfinite_guard also takes float64, float16 and bfloat16).
 *
 * Index contract: every int32 index an entry point writes, and every index a kernel computes and then reads memory with, lies in
 * [0, n) of the array it indexes, for any float input including NaN and +-Inf.  Distances keep what they compute (+Inf, NaN), so a
 * loss over them stays non-finite and visible.  A query with no candidate comparing below +Inf gets:
 *   nn_distance / simplification loss / progressive loss (idx1, idx2)    index 0, as the reference's tf_nndistance kernel
 *   knn_soft_project, project_and_loss (knn_idx, and idx1 there)         index n - 1 in the lanes no candidate filled
 *   nn_matching's farthest-point completion                              numpy's argmax: the first NaN distance wins
 *   the generator backward's pool arg-max (a channel of NaN)             point 0
 *   farthest_point_sample, the frozen encoders' pool routes, pose loss   always in range (their scans start from a real point)
 */
#ifndef SAMPLENET_B200_H
#define SAMPLENET_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SNB200_OK 0
#define SNB200_EINVAL (-1)   /* bad size / null pointer / unsupported argument */
#define SNB200_EWORKSPACE (-2) /* workspace too small */
#define SNB200_ECUDA (-3)    /* CUDA runtime reported an error at launch */
#define SNB200_EUNSUPPORTED (-4)

#define SNB200_BNC 0
#define SNB200_BCN 1

/* flags for the distance kernels */
#define SNB200_DIST_FMA 0      /* d = fma(dz,dz,fma(dx,dx,dy*dy)): the arithmetic nvcc gives the reference CUDA kernels (bit-identical results) */
#define SNB200_DIST_UNFUSED 1  /* d = (dx*dx+dy*dy)+dz*dz, three roundings: the arithmetic of the reference CPU code */

/* how the `sigma` device scalar of the projection entry points is interpreted (sigma_mode); `sigma_floor` is the clamp:
 *   SIGMA_VALUE       *sigma is sigma itself
 *   SIGMA_FROM_T_REG  *sigma is the temperature T, sigma = max(T*T, floor)      registration/src/soft_projection.py:97-99
 *   SIGMA_FROM_T_CLS  *sigma is T, sigma = T*T                                   classification/soft_projection.py:41
 *   SIGMA_FROM_T_REC  *sigma is T, sigma = max(T, floor)^2                       reconstruction/src/soft_projection.py:51-54
 * (evaluating sigma inside the kernel removes two elementwise launches from every forward) */
#define SNB200_SIGMA_VALUE 0
#define SNB200_SIGMA_FROM_T_REG 1
#define SNB200_SIGMA_FROM_T_CLS 2
#define SNB200_SIGMA_FROM_T_REC 3

typedef void *snb200_stream_t; /* a cudaStream_t */

const char *snb200_last_error(void);
int snb200_version(void);
/* number of kernels this library has launched from the calling thread since load (bench.py's gpu_launches) */
unsigned long long snb200_launch_count(void);

/* ---------------------------------------------------------------------------------------------------------
 * Chamfer / nn_distance.  xyz1 (b,n,3), xyz2 (b,m,3) BNC; dist1,idx1 (b,n); dist2,idx2 (b,m).
 * Replaces ChamferDistanceKernelLauncher (registration/src/chamfer_distance/chamfer_distance.cpp:4-12,
 * chamfer_distance.cu:139-155) and NmDistanceKernelLauncher (classification/structural_losses/tf_nndistance.cpp:168,
 * tf_nndistance_g.cu:128-131).  Squared L2 distance to the nearest neighbour and its index; lowest index wins ties.
 * Both directions are computed by ONE launch.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_nn_distance_forward(int b, int n, const float *xyz1, int m, const float *xyz2, float *dist1, int *idx1,
                               float *dist2, int *idx2, int flags, snb200_stream_t stream);

/* Replaces ChamferDistanceGradKernelLauncher (chamfer_distance.cpp:14-24, chamfer_distance.cu:189-209) and
 * NmDistanceGradKernelLauncher (tf_nndistance.cpp:208).  grad_xyz1 (b,n,3) and grad_xyz2 (b,m,3) are overwritten
 * (the launcher zeroes them itself, like the reference's cudaMemset).  Deterministic: no float atomics. */
int snb200_nn_distance_backward(int b, int n, const float *xyz1, int m, const float *xyz2, const float *grad_dist1,
                                const int *idx1, const float *grad_dist2, const int *idx2, float *grad_xyz1,
                                float *grad_xyz2, snb200_stream_t stream);

/* Per-cloud Chamfer means for evaluation (reconstruction/src/sampler_progressive_autoencoder.py:145-177 get_loss_ae_per_pc):
 * sums (b,2) = { mean_i dist1[bi,i], mean_j dist2[bi,j] } of xyz1[bi] (n points) against xyz2[bi % b2] (m points); xyz2 holds b2 clouds
 * (b2 divides b; b2 == b compares cloud with cloud).  The distances are those of snb200_nn_distance_forward with flags 0; no dist / idx
 * array is written.  Per-CTA partials in the workspace are added in tile order: no float atomics, run to run bit-identical. */
size_t snb200_chamfer_per_cloud_workspace_bytes(int b, int n, int m);
int snb200_chamfer_per_cloud(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, float *sums, void *workspace,
                             size_t workspace_bytes, snb200_stream_t stream);

/* Fused simplification loss (registration/src/samplenet.py:171-181, classification/models/samplenet_model.py:176-188):
 * nn_distance(samp, ref) + the three reductions (two launches on `stream`).  out4 (device, 4 floats) =
 * { mean(dist1), mean_b(max_n dist1), mean(dist2), loss = out[0] + out[1] + (gamma + delta*pc_size) * out[2] }.
 * dist/idx outputs as in snb200_nn_distance_forward (needed by the backward).  workspace: see query. */
size_t snb200_simplification_loss_workspace_bytes(int b, int n, int m);
int snb200_simplification_loss_forward(int b, int n, const float *samp, int m, const float *ref, float weight21,
                                       float *dist1, int *idx1, float *dist2, int *idx2, float *out4, void *workspace,
                                       size_t workspace_bytes, int flags, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * kNN + soft projection, fused: for every query point the k nearest points of the cloud (brute force,
 * sorted by (squared distance, index)), then -- if `proj` is given -- dist/sigma, softmax over the k
 * neighbours and the weighted average of the neighbours (and of their features).
 * Replaces, in one launch: knn_cuda.KNN + pointnet2 grouping_operation + the torch ops of
 * registration/src/soft_projection.py:75-152; and tf_grouping.py:64-91 knn_point (three (B,M,N[,3]) temporaries
 * + selectionSortLauncher, tf_grouping.cpp:108) + groupPointLauncher (:142) + classification/soft_projection.py:46-82.
 *   points (b,n,3) / query (b,m,3) in `layout`; feats (b,n,f) BNC or (b,f,n) BCN, may be NULL (f = 0).
 *   sigma: DEVICE pointer to one float, already clamped by the caller (the three sub-projects clamp differently).
 *   hard != 0: one-hot weights on the nearest neighbour (TF SoftProjection(hard=True)).
 * Outputs (each may be NULL): proj (b,m,3)/(b,3,m) in `layout`; prop like feats with n->m;
 *   knn_idx (b,m,k) int32; knn_val (b,m,k) squared distances ascending; weights (b,m,k); dist_over_sigma (b,m,k).
 * 1 <= k <= 32, k <= n.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_knn_soft_project_forward(int b, int n, int m, int k, int layout, const float *points, const float *query,
                                    const float *sigma, int sigma_mode, float sigma_floor, int hard, const float *feats, int f, float *proj, float *prop,
                                    int *knn_idx, float *knn_val, float *weights, float *dist_over_sigma, int flags,
                                    snb200_stream_t stream);

/* Backward of the soft projection given the saved knn_idx and weights.  grad_proj in `layout` (may be NULL),
 * grad_prop like prop (may be NULL).  Outputs (each may be NULL): grad_points, grad_query in `layout` (overwritten),
 * grad_feats like feats (overwritten), grad_sigma: DEVICE pointer to one float (overwritten), the gradient with respect to
 * SIGMA (for the FROM_T modes the caller applies d sigma / d T).
 * Replaces the autograd graph of registration/src/soft_projection.py:92-152 and groupPointGradLauncher
 * (tf_grouping.cpp:173).  workspace: see query. */
size_t snb200_soft_project_backward_workspace_bytes(int b, int n, int m, int k, int f);
int snb200_soft_project_backward(int b, int n, int m, int k, int layout, const float *points, const float *query,
                                 const float *sigma, int sigma_mode, float sigma_floor, const float *feats, int f, const int *knn_idx,
                                 const float *weights, const float *grad_proj, const float *grad_prop,
                                 float *grad_points, float *grad_query, float *grad_feats, float *grad_sigma,
                                 void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* The tail of a SampleNet training step in ONE launch: soft projection of the generated points onto the input cloud
 * (registration/src/samplenet.py:114) + nn_distance(samp, ref) + the simplification-loss reductions (samplenet.py:175-180).
 * ref (b,n_ref,3), samp (b,n_samp,3) BNC.  Outputs: proj (b,n_samp,3), knn_idx / weights / dist_over_sigma (b,n_samp,k) (saved
 * for the projection backward), dist1/idx1 (b,n_samp), dist2/idx2 (b,n_ref), out4 as in snb200_simplification_loss_forward.
 * workspace: snb200_project_and_loss_workspace_bytes() bytes of partial sums; ticket: DEVICE unsigned that must be zero at
 * the first call and is left zero by every call (allocate once, never touch).  n_ref <= 4096 (one shared-memory tile).
 * Launched as a programmatic dependent launch: `ref` may be read before the kernel waits for the previous kernel on `stream` to finish,
 * so that kernel must not write `ref` (SampleNet puts the generator there, which only reads it); `samp` is read after the wait. */
size_t snb200_project_and_loss_workspace_bytes(int b, int n_samp, int n_ref);
int snb200_project_and_loss_forward(int b, int n_ref, int n_samp, int k, const float *ref, const float *samp, const float *sigma,
                                    int sigma_mode, float sigma_floor, float *proj, int *knn_idx, float *weights,
                                    float *dist_over_sigma, float *dist1, int *idx1, float *dist2, int *idx2, float weight21,
                                    float *out4, void *workspace, size_t workspace_bytes, unsigned *ticket, int flags,
                                    snb200_stream_t stream);

/* group_point: points (b,n,c) BNC [or (b,c,n) BCN], idx (b,m,ns) -> out (b,m,ns,c) BNC [or (b,c,m,ns) BCN].
 * Replaces groupPointLauncher / groupPointGradLauncher (tf_grouping.cpp:142,173; tf_grouping_g.cu:40-78) and
 * pointnet2 grouping_operation.  The grad launcher overwrites grad_points (zeroes it first). */
int snb200_group_point(int b, int n, int c, int m, int ns, int layout, const float *points, const int *idx, float *out,
                       snb200_stream_t stream);
int snb200_group_point_grad(int b, int n, int c, int m, int ns, int layout, const float *grad_out, const int *idx,
                            float *grad_points, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * SampleNet generator (registration/src/samplenet.py:40-60,90-104; rec widths reconstruction/src/samplers.py:22-36):
 * x -> 5 x [1x1 conv + BatchNorm + ReLU] -> max over points -> 3 x [Linear + BatchNorm + ReLU] -> Linear.
 * --------------------------------------------------------------------------------------------------------- */
#define SNB200_MAX_CONV_LAYERS 8
#define SNB200_MAX_FC_LAYERS 8
typedef struct snb200_layer {
    int c_in, c_out;
    const float *weight;  /* (c_out, c_in) row-major: Conv1d.weight[:, :, 0] / Linear.weight */
    const float *bias;    /* (c_out) */
    const float *bn_weight, *bn_bias;   /* (c_out) gamma/beta, NULL => no BatchNorm after this layer */
    float *bn_running_mean, *bn_running_var; /* (c_out) updated in training mode when non-NULL */
    long long *bn_num_batches_tracked;  /* int64 device scalar, +1 per training forward when non-NULL (torch BatchNorm bookkeeping) */
    float bn_eps, bn_momentum;
    int relu;             /* apply ReLU after (BatchNorm of) this layer */
} snb200_layer;

/* Per-point MLP + global max-pool.  x (b,n,3) in `layout`; feat (b, c_last).  training != 0 uses batch statistics
 * over all b*n positions (and updates the running stats), else the running stats.  workspace: see query.  Computes what
 * snb200_generator_forward computes for feat with SNB200_GEN_EXACT_FP32: the same CUDA-core conv stack and pool kernels. */
size_t snb200_encoder_workspace_bytes(int b, int n, int num_layers, const snb200_layer *layers);
int snb200_encoder_forward(int b, int n, int layout, const float *x, int num_layers, const snb200_layer *layers,
                           int training, float *feat, void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* The whole generator in one call: conv stack -> max-pool -> FC head -> out (b, c_out_last) [+ feat (b, c_conv_last), may be
 * NULL].  Default path: ONE persistent cooperative launch -- layers 2.. of the conv stack on the tensor cores (wgmma
 * tf32, 3xTF32 error-compensated, fp32 register accumulators), layer 1 evaluated on the fly with its BatchNorm statistics
 * derived from the input moments, the max-pool and all FC layers on the same grid (conv widths 32/64/128, up to 32 slices of
 * 128 points per SM).  Other shapes: one tensor-core launch per layer (hidden layers up to 256 channels, the last one up to 1024 in
 * blocks of 256) + a thread-block-cluster FC head (a pooled feature of up to 1024 channels).  flags & SNB200_GEN_EXACT_FP32 selects the
 * exact-fp32 CUDA-core conv stack instead (also taken automatically for widths the tensor path does not cover).  b <= 256.  Training-mode pre-BatchNorm activations must stay below ~3e4 in magnitude on the default
 * path (fixed-point statistics exchange); beyond that the call returns NaN rows. */
#define SNB200_GEN_EXACT_FP32 1
#define SNB200_GEN_PER_LAYER_KERNELS 8 /* tensor-core path as one launch per layer instead of the persistent conv-stack kernel */
#define SNB200_GEN_SEPARATE_HEAD 16 /* keep the pool + FC head as its own thread-block-cluster launch */
#define SNB200_GEN_WORKSPACE_PRIMED 32 /* the caller keeps `workspace` across calls and its first 256 bytes are zero (freshly zeroed or as the
                                         previous PRIMED call left them): the persistent kernel cleans the rest itself, no memset in front */
#define SNB200_GEN_PROFILE_SKIP_HEAD 2 /* profiling only: stop after the conv stack (out is not written) */
#define SNB200_GEN_PROFILE_SKIP_CONV 4 /* profiling only: run only the pool + FC head on whatever the workspace holds */
size_t snb200_generator_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc);
int snb200_generator_forward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                             const snb200_layer *fc, int training, float *out, int out_transpose_inner, float *feat, int flags,
                             void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Generator TRAINING step: forward that keeps what the backward needs, and the backward itself
 * (replaces `loss.backward()` through registration/src/samplenet.py:90-104 -- stock cuDNN / cuBLAS / ATen kernels in the reference).
 *   snb200_generator_backward_supported(...) != 0 : shapes covered (the persistent conv-stack envelope, 2 <= b <= 64, BN + ReLU layers)
 *   snb200_generator_train_forward : snb200_generator_forward + `zsave`: per conv layer l a (b*n, c_out_l) float buffer that receives
 *                                    the layer's raw output; `workspace` must stay untouched until the backward has run
 *   snb200_generator_backward      : grad_out (b, c_out_last) in the layout snb200_generator_forward stores `out` -> gradients of
 *                                    every weight / bias / BatchNorm weight / BatchNorm bias (null pointers are skipped)
 * --------------------------------------------------------------------------------------------------------- */
typedef struct snb200_layer_grad {
    float *weight, *bias, *bn_weight, *bn_bias;
} snb200_layer_grad;
int snb200_generator_backward_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc);
int snb200_generator_train_forward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                                   const snb200_layer *fc, float *out, int out_transpose_inner, float *feat, float *const *zsave, int flags,
                                   void *workspace, size_t workspace_bytes, snb200_stream_t stream);
size_t snb200_generator_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc);
int snb200_generator_backward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                              const snb200_layer *fc, float *const *zsave, void *forward_workspace, const float *grad_out,
                              int out_transpose_inner, const snb200_layer_grad *conv_grads, const snb200_layer_grad *fc_grads,
                              void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* The same training step for the shapes the persistent kernel does not take: the reconstruction sampler (conv widths 64-128-128-256-128,
 * FC layers with ReLU and no BatchNorm) and the classification sampler (BatchNorm without ReLU on the last FC layer), at any number of
 * points.  Same argument lists as the four calls above; the forward is the per-layer tensor-core path (SNB200_GEN_PER_LAYER_KERNELS)
 * and computes exactly what snb200_generator_forward(training, SNB200_GEN_PER_LAYER_KERNELS) computes.
 *   snb200_generator_layers_backward_supported(...) != 0 : conv1 with 64 or 128 channels; later conv layers (64,64), (64,128), (128,128),
 *       (128,256) or (256,128), and the last one also (128,C) with C a multiple of 64 up to 1024 (the samplers' bottleneck); BatchNorm +
 *       ReLU on every conv layer; FC layers with any BatchNorm / ReLU combination except ReLU on the last one, inputs of at most 1024
 *       channels, outputs of any width; 2 <= b <= 64, and at most as many rows as fit fc1's input next to its weight rows in the FC
 *       backward's 200 KB of shared memory (b <= 41 for a 1024-channel last conv layer)
 *   snb200_generator_layers_train_forward : flags 0 or SNB200_GEN_WORKSPACE_PRIMED; zsave as for snb200_generator_train_forward */
int snb200_generator_layers_backward_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc);
int snb200_generator_layers_train_forward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                                          const snb200_layer *fc, float *out, int out_transpose_inner, float *feat, float *const *zsave, int flags,
                                          void *workspace, size_t workspace_bytes, snb200_stream_t stream);
size_t snb200_generator_layers_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc);
int snb200_generator_layers_backward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                                     const snb200_layer *fc, float *const *zsave, void *forward_workspace, const float *grad_out,
                                     int out_transpose_inner, const snb200_layer_grad *conv_grads, const snb200_layer_grad *fc_grads,
                                     void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* The per-layer training step with four additions, for the PointNet classifiers (classification/models/pointnet_cls_basic.py, and
 * pointnet_cls.py + transform_nets.py, whose conv stack a per-cloud transform splits).  Same kernels; the vocabulary of
 * snb200_frozen_encoder_ex_*:
 *   act_input = 0: `in` is the cloud (b,n,3) in `layout`, as above.  act_input = 1: `in` is a (b*n, c_in) activation (16-byte aligned) that
 *       layer 1 reads as it is (no BatchNorm, no ReLU in front of it); layer 1 is then a tensor-core layer like the hidden ones, its
 *       BatchNorm statistics taken from its own output.
 *   tap = -1: none.  tap = t in [0, num_conv - 2]: hidden layer t's activation a_t = relu(bn(z_t)) is also written to tap_out (b*n, c_out_t,
 *       16-byte aligned), exactly the values layer t + 1 consumes.
 *   fc_dropout[num_fc] (or NULL: none): per FC layer NULL or a (b, c_in) mask multiplying that layer's input, entries 0 or 1/(1-p).  The
 *       forward stores the masked input, and the backward reads it and takes the gradient through the same mask.  fc_dropout[num_fc] must
 *       be the same in the forward and the backward.
 * The backward adds:
 *   grad_tap (b*n, c_out_t, 16-byte aligned) or NULL: added to the gradient of a_t point by point, before a_t's ReLU mask and BatchNorm
 *       backward.
 *   grad_in: the gradient of `in`, (b,n,3) in `layout` or (b*n, c_in) (16-byte aligned), overwritten; NULL: not computed.  Per point a fixed
 *       order over the channels; no float atomics, so a repeat backward is bit-identical.
 *   The parameter gradients are as above.
 * snb200_generator_layers_ex_supported(...) != 0 : the envelope of snb200_generator_layers_backward_supported, and with act_input = 1 layer 1
 *   64 -> 64 or 64 -> 128; a tap only on a layer of 64 output channels that is not directly under a wide last layer (128 -> C > 256); no
 *   mask on fc1's input (the pooled feature).  Outside it the calls return SNB200_EUNSUPPORTED and launch nothing.  The forward workspace is
 *   snb200_generator_workspace_bytes'; the backward's depends on act_input.
 * snb200_generator_layers_train_forward / _backward are these entries with act_input = 0, tap = -1, no masks and grad_in = NULL. */
int snb200_generator_layers_ex_supported(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc,
                                         int tap, const float *const *fc_dropout);
int snb200_generator_layers_ex_train_forward(int b, int n, int layout, int act_input, const float *in, int num_conv, const snb200_layer *conv,
                                             int num_fc, const snb200_layer *fc, int tap, float *tap_out, const float *const *fc_dropout,
                                             float *out, int out_transpose_inner, float *feat, float *const *zsave, int flags,
                                             void *workspace, size_t workspace_bytes, snb200_stream_t stream);
size_t snb200_generator_layers_ex_backward_workspace_bytes(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_fc,
                                                           const snb200_layer *fc);
int snb200_generator_layers_ex_backward(int b, int n, int layout, int act_input, const float *in, int num_conv, const snb200_layer *conv,
                                        int num_fc, const snb200_layer *fc, int tap, const float *const *fc_dropout, float *const *zsave,
                                        void *forward_workspace, const float *grad_out, int out_transpose_inner, const float *grad_tap,
                                        float *grad_in, const snb200_layer_grad *conv_grads, const snb200_layer_grad *fc_grads,
                                        void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* Fully connected head on the pooled feature: in (b, c_in0) -> out (b, c_out_last).  BatchNorm over the batch.
 * out_transpose_inner = M > 0: each output row, logically (c_out_last/M, M) -- the reference's y.view(-1, 3, M),
 * samplenet.py:104 -- is stored transposed as (M, c_out_last/M), i.e. directly in BNC order; 0 = stored as is (BCN).
 * b <= 256.  Runs the FC-head kernel of snb200_generator_forward's non-fused paths, so chained behind snb200_encoder_forward
 * it gives bit for bit what snb200_generator_forward gives with SNB200_GEN_EXACT_FP32.  `in` must be 16-byte aligned when c_in0
 * is a multiple of 4 (SNB200_EINVAL otherwise); inputs too wide for its shared memory (together with the layers' 16-row weight
 * slices) return SNB200_EUNSUPPORTED. */
size_t snb200_fc_head_workspace_bytes(int b, int num_layers, const snb200_layer *layers);
int snb200_fc_head_forward(int b, const float *in, int num_layers, const snb200_layer *layers, int training, float *out,
                           int out_transpose_inner, void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * SampleNetProgressive: the simplification loss summed over prefixes of an ORDERED sample set, one launch
 * (replaces the per-prefix NnDistance ops + reductions of classification/train_samplenet_progressive.py:172-230).
 *   ref (b,n,3), samp (b,m,3); sizes[num_prefix] ascending prefix lengths (<= m, <= 16 of them); weights[p] = gamma + delta * sizes[p]
 *   dist1/idx1 (b,m): sample -> nearest input point (prefix p uses the slice [:sizes[p]])
 *   dist2/idx2 (b,num_prefix,n): input point -> nearest of the first sizes[p] samples
 *   terms (3*num_prefix + 1): per prefix [mean dist1[:s], mean_b max dist1[:s], mean dist2_p], then the total loss
 *   ticket: one zero-initialised unsigned, left zero.  sizes / weights are HOST arrays.
 * --------------------------------------------------------------------------------------------------------- */
size_t snb200_progressive_loss_workspace_bytes(int b, int n, int m, int num_prefix);
int snb200_progressive_loss_forward(int b, int n, int m, const float *ref, const float *samp, int num_prefix, const int *sizes, const float *weights,
                                    float *dist1, int *idx1, float *dist2, int *idx2, float *terms, void *workspace, size_t workspace_bytes,
                                    unsigned *ticket, int flags, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * A FROZEN PointNet encoder over every prefix of a cloud, from one shared pass (the task networks the sampler trainers put behind the
 * sampler: classification/models/pointnet_cls_basic.py, reconstruction/src/ae_templates.py; evaluated per prefix in
 * classification/train_samplenet_progressive.py and reconstruction/src/samplenet_progressive_pointnet_ae.py).
 *   x (b,n,3) BNC; conv: num_conv layers, 1x1 conv l: z_l = W_l a_{l-1} + b_l, a_l = relu(scale_l z_l + shift_l) with eval-mode BatchNorm
 *   from the running statistics (or identity without BatchNorm); sizes[num_prefix]: ascending prefix lengths in [1, n] (HOST array).
 *   pooled (num_prefix, b, C): pooled[p,b,c] = max over i < sizes[p] of a_L[b,i,c];
 *   route  (num_prefix, b, C) int32: the point that max comes from, the first extreme of z_L in the direction of sign(scale) (max for
 *          scale >= 0, min otherwise), the lowest index on ties;
 *   zsave: per hidden layer l < num_conv - 1 a (b*n, c_out_l) float buffer that receives its raw output, or NULL (forward only: the
 *          hidden layers then live in the workspace, sized with with_zsave = 0).
 * The backward gives the gradient with respect to x only (the parameters are frozen): grad_pooled (num_prefix, b, C) -> grad_x (b,n,3),
 * overwritten; points no prefix routes to get exactly 0.  No float atomics: run to run bit-identical.
 *   snb200_frozen_encoder_supported(...) != 0 : 1 <= b <= 64, 1 <= n <= 4096, 1 <= num_prefix <= 16, 2..8 conv layers, conv1 3 -> a
 *       multiple of 8 up to 256, hidden layers as the tensor-core layer kernels take them (c_in a multiple of 8 up to 256, c_out 8..256),
 *       last layer c_in a multiple of 8 up to 256 and c_out 8..1024 (PointNetCls 3-64-64-64-128-1024, PointNetAE 3-64-128-128-256-128).
 * --------------------------------------------------------------------------------------------------------- */
int snb200_frozen_encoder_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix);
size_t snb200_frozen_encoder_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, int with_zsave);
size_t snb200_frozen_encoder_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix);
int snb200_frozen_encoder_forward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                  float *pooled, int *route, float *const *zsave, void *workspace, size_t workspace_bytes,
                                  snb200_stream_t stream);
int snb200_frozen_encoder_backward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                   const float *pooled, const int *route, float *const *zsave, const float *grad_pooled, float *grad_x,
                                   void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The same frozen encoder's forward over MANY prefixes, up to every sample size of a progressive curve (classification/evaluate_from_files.py
 * --dense_eval 1 classifies the first s points of each ordered cloud for every s), from one pass of the conv stack.
 *   x (b,n,3) BNC and the layer table as snb200_frozen_encoder_forward; sizes[num_sizes]: 1 to n ascending, distinct lengths in [1, n] (HOST
 *   array).  pooled, route (num_sizes, b, C): exactly the values, routes and tie rule of snb200_frozen_encoder_forward, bit for bit what that
 *   entry gives called on the same sizes 16 at a time.  Forward only: no zsave, no backward.
 *   The sizes reach the kernels through the workspace: the call stages them there, with a table of each 128-point tile's first boundary, by
 *   one host-to-device copy on `stream` from pageable memory, so the call may not be captured into a CUDA graph.  Besides that table the
 *   workspace holds one record per (cloud, 128-point tile, channel) and the hidden layers' activations; the boundary records are written
 *   into pooled / route and finished there.
 *   Every route entry lies in [0, n) for any float input (non-finite included), as for snb200_frozen_encoder_forward.
 *   snb200_frozen_encoder_curve_supported(...) != 0 : snb200_frozen_encoder_supported's envelope (1 <= b <= 64, 1 <= n <= 4096, the same
 *       layer table) with 1 <= num_sizes <= n sizes that are ascending, distinct and in [1, n]; _workspace_bytes returns 0 outside it.  The
 *       forward returns SNB200_EINVAL for bad sizes and SNB200_EUNSUPPORTED for a shape outside the envelope, and launches nothing then.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_frozen_encoder_curve_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_sizes, const int *sizes);
size_t snb200_frozen_encoder_curve_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_sizes, const int *sizes);
int snb200_frozen_encoder_curve_forward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_sizes, const int *sizes,
                                        float *pooled, int *route, void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The same frozen encoder (same kernels, same workspaces) with two additions, for a conv stack split by a per-cloud transform (PointNet with
 * its transform nets: classification/models/pointnet_cls.py + transform_nets.py):
 *   act_input = 0: `in` is the cloud (b,n,3) BNC, as above.  act_input = 1: `in` is a (b*n, c_in) activation (16-byte aligned) that layer 1
 *       reads as it is (no BatchNorm, no ReLU in front of it); layer 1 is then a tensor-core layer like the hidden ones.
 *   tap = -1: none.  tap = t in [0, num_conv - 2]: hidden layer t's activation a_t = relu(scale_t z_t + shift_t) is also written to tap_out
 *       (b*n, c_out_t, 16-byte aligned), exactly the values layer t + 1 consumes.
 * The backward gives grad_in, (b,n,3) or (b*n, c_in), of sum(grad_pooled * pooled) + [tap >= 0] sum(grad_tap * a_t): grad_tap (b*n, c_out_t)
 * is added to the routed gradient of a_t point by point in a fixed order.  The backward's tap may be -1 after a tapped forward (no gradient
 * reached a_t).  Points that no prefix routes to and, with a tap, every point, run the chain from the highest layer with a gradient; without
 * a tap, points no prefix routes to get exactly 0.  No float atomics: run to run bit-identical.
 *   snb200_frozen_encoder_ex_supported(...) != 0 : the envelope above, with layer 1 as a hidden layer (c_in a multiple of 8 up to 256, c_out
 *       8..256) when act_input = 1.  Outside it the calls return SNB200_EUNSUPPORTED and launch nothing.
 * snb200_frozen_encoder_ex_supported(b, n, 0, ...conv, num_prefix, -1) is snb200_frozen_encoder_supported(b, n, ...), and so on: the original
 * entries are these with a cloud input and no tap.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_frozen_encoder_ex_supported(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_prefix, int tap);
size_t snb200_frozen_encoder_ex_workspace_bytes(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_prefix, int tap,
                                                int with_zsave);
size_t snb200_frozen_encoder_ex_backward_workspace_bytes(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_prefix,
                                                         int tap);
int snb200_frozen_encoder_ex_forward(int b, int n, int act_input, const float *in, int num_conv, const snb200_layer *conv, int num_prefix,
                                     const int *sizes, float *pooled, int *route, int tap, float *tap_out, float *const *zsave,
                                     void *workspace, size_t workspace_bytes, snb200_stream_t stream);
int snb200_frozen_encoder_ex_backward(int b, int n, int act_input, const float *in, int num_conv, const snb200_layer *conv, int num_prefix,
                                      const int *sizes, const float *pooled, const int *route, float *const *zsave, int tap,
                                      const float *grad_tap, const float *grad_pooled, float *grad_in, void *workspace,
                                      size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The same frozen encoder (same kernels) over the SEGMENTS of a packed buffer instead of the prefixes of clouds, so that rows which depend on
 * their prefix (PointNet with transform nets: x[:, :s] @ T1(s)) share one pass.
 *   in: a packed buffer of `total` rows, 3 channels (act_input = 0: points) or c_in channels (act_input = 1: an activation, 16-byte aligned).
 *   seg (num_seg, 2) int32, DEVICE memory, 8-byte aligned: segment j is rows [seg[j][0], seg[j][0] + seg[j][1]).  The table is the caller's
 *       and is not read on the host: offsets ascending, each a multiple of 128 (a segment starts its own 128-row tile; the rows up to the next
 *       multiple of 128 are its padding, which the kernels read and otherwise ignore), lengths in [1, max_len], and every segment with its
 *       padding inside `total` rows.
 *   pooled (num_seg, C): the max over segment j's rows of a_L; route (num_seg, C) int32: its row within the segment (the first extreme of
 *       z_L in the direction of sign(scale), the lowest row on ties).  tap, tap_out (total, c_out_t) and zsave (total, c_out_l) as in _ex_.
 *   backward: grad_in (total, 3 or c_in), overwritten; rows outside every segment get exactly 0, and so do rows no segment routes to when
 *       tap = -1.  Point -> segment instead of point -> (cloud, prefix): one segment per row, so the chain takes one coefficient per channel.
 *       No float atomics: run to run bit-identical.
 *   snb200_frozen_encoder_seg_supported(...) != 0 : the layer table of snb200_frozen_encoder_ex_supported, and
 *       total <= 2^22 rows             (an element offset of a (total, 256) hidden activation stays below 2^31),
 *       1 <= num_seg <= ceil(total/128) (each segment starts its own tile),
 *       1 <= max_len <= 4096           (the frozen encoder's cloud size).
 *     Outside it the calls return SNB200_EUNSUPPORTED and launch nothing.  The workspaces depend on total and the layer table only.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_frozen_encoder_seg_supported(int num_seg, int total, int max_len, int act_input, int num_conv, const snb200_layer *conv, int tap);
size_t snb200_frozen_encoder_seg_workspace_bytes(int num_seg, int total, int max_len, int act_input, int num_conv, const snb200_layer *conv, int tap,
                                                 int with_zsave);
size_t snb200_frozen_encoder_seg_backward_workspace_bytes(int num_seg, int total, int max_len, int act_input, int num_conv, const snb200_layer *conv,
                                                          int tap);
int snb200_frozen_encoder_seg_forward(int num_seg, int total, int max_len, const int *seg, int act_input, const float *in, int num_conv,
                                      const snb200_layer *conv, float *pooled, int *route, int tap, float *tap_out, float *const *zsave,
                                      void *workspace, size_t workspace_bytes, snb200_stream_t stream);
int snb200_frozen_encoder_seg_backward(int num_seg, int total, int max_len, const int *seg, int act_input, const float *in, int num_conv,
                                       const snb200_layer *conv, const float *pooled, const int *route, float *const *zsave, int tap,
                                       const float *grad_tap, const float *grad_pooled, float *grad_in, void *workspace, size_t workspace_bytes,
                                       snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The frozen encoder with every BatchNorm normalised by the BATCH statistics of each prefix, as the reconstruction sampler trainers run
 * their frozen autoencoder (reconstruction/src/samplenet_pointnet_ae.py:229 and samplenet_progressive_pointnet_ae.py:260 set tflearn's
 * training flag; --fixed_ae sets every moving-average decay to 1, so the autoencoder's state never changes).
 *   x (b,n,3) BNC; conv: the frozen encoder's layer table, BatchNorm, bias and ReLU on every layer; sizes[num_prefix] HOST, ascending.
 *   Layer l on prefix p: a = relu(gamma (z - mean_p) / sqrt(var_p + eps) + beta), mean_p and the BIASED variance var_p over the b * sizes[p]
 *   points of x[:, :sizes[p]].  The running statistics are neither read nor written.
 *   pooled, route (num_prefix, b, C) as snb200_frozen_encoder_forward; stats (double): per layer l in layer order a (num_prefix, 2, c_out_l)
 *       block of (mean, biased variance) per prefix.
 *   The forward workspace keeps every layer's raw output; the backward reads it (fwd_workspace) with pooled, route and stats, and writes
 *   grad_x (b,n,3) of sum(grad_pooled * pooled), the statistics' dependence on x included (no parameter gradients).  Points past the
 *   longest prefix get exactly 0.  No float atomics: run to run bit-identical.
 *   snb200_frozen_encoder_bstat_supported(...) != 0 : 1 <= num_prefix <= 16 ascending distinct sizes in [1, n], 1 <= n <= 4096, b >= 1,
 *       b * sum(pad128(sizes[p])) <= 2^22 packed rows, and the layer table of snb200_frozen_encoder_supported with BatchNorm, bias and ReLU
 *       on every layer.  Outside it the calls return SNB200_EUNSUPPORTED and launch nothing; the workspace queries return 0.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_frozen_encoder_bstat_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes);
size_t snb200_frozen_encoder_bstat_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes);
size_t snb200_frozen_encoder_bstat_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes);
int snb200_frozen_encoder_bstat_forward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                        float *pooled, int *route, double *stats, void *workspace, size_t workspace_bytes, snb200_stream_t stream);
int snb200_frozen_encoder_bstat_backward(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                         const float *pooled, const int *route, const double *stats, const void *fwd_workspace,
                                         size_t fwd_workspace_bytes, const float *grad_pooled, float *grad_x, void *workspace,
                                         size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The batch-statistics encoder TRAINED: the autoencoder fine-tuned together with the reconstruction sampler (--fixed_ae False,
 * reconstruction/src/samplenet_pointnet_ae.py:191-214, samplenet_progressive_pointnet_ae.py:242-245).  The forward is
 * snb200_frozen_encoder_bstat_forward, unchanged.
 *   snb200_frozen_encoder_bstat_param_backward: what snb200_frozen_encoder_bstat_backward takes, plus x (b,n,3) and
 *       conv_grads[num_conv] (snb200_layer_grad): weight (c_out, c_in), bias, bn_weight and bn_bias per layer, overwritten; a NULL pointer
 *       is skipped.  Writes the gradients of sum(grad_pooled * pooled) with respect to every conv weight, conv bias, gamma and beta, the
 *       statistics' dependence on the weights included; grad_x may be NULL, and otherwise is bit for bit snb200_frozen_encoder_bstat_backward's
 *       (the same chain).  With r_g = 1/sqrt(var_g + eps), zhat = (z - mean_g) r_g, dy the gradient of the BatchNorm output under the ReLU mask:
 *         dbeta = sum_g sum_{rows in g} dy, dgamma = sum_g sum_{rows in g} dy zhat (groups ascending, in double);
 *         dz = gamma r_g (dy - mean_g dy - zhat mean_g(dy zhat)); dW_l = sum_rows dz (x) a_{l-1} (a_0 = x, a_{l-1} recomputed from the
 *         saved raw output with the forward's relu(fmaf(z, scale, shift))), db_l = sum_rows dz (0 in exact arithmetic, written all the same).
 *       The rows are summed in fixed chunks of tiles (fp32), the chunks added in a fixed order; no float atomics: run to run bit-identical.
 *   snb200_frozen_encoder_bstat_running_update: one launch; stats is the forward's.  For each prefix in ascending order, every layer's
 *       bn_running_mean / bn_running_var (where non-NULL) move as nn.BatchNorm1d moves them: momentum bn_momentum, the variance unbiased
 *       with N/(N-1), N = b * sizes[p]; bn_num_batches_tracked (where non-NULL) goes up by num_prefix.
 *   The envelope is snb200_frozen_encoder_bstat_supported's plus b * sizes[p] >= 2 for every prefix (a one-value batch has no unbiased
 *   variance).  Outside it the calls return SNB200_EUNSUPPORTED and launch nothing; the workspace query returns 0.  Neither entry writes
 *   an index.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_frozen_encoder_bstat_param_backward_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes);
size_t snb200_frozen_encoder_bstat_param_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix,
                                                                  const int *sizes);
int snb200_frozen_encoder_bstat_param_backward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix,
                                               const int *sizes, const float *pooled, const int *route, const double *stats,
                                               const void *fwd_workspace, size_t fwd_workspace_bytes, const float *grad_pooled, float *grad_x,
                                               const snb200_layer_grad *conv_grads, void *workspace, size_t workspace_bytes,
                                               snb200_stream_t stream);
int snb200_frozen_encoder_bstat_running_update(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                               const double *stats, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The frozen encoder's backward with weight and bias gradients, for a conv stack without BatchNorm (PCRNet's encoder trained:
 * registration/main.py --train-pcrnet).  The forward is snb200_frozen_encoder_forward with zsave; PCRNet has no BatchNorm and no dropout,
 * so its training forward is the frozen one.
 *   conv_grads[num_conv] (snb200_layer_grad): weight (c_out, c_in) 16-byte aligned and bias (c_out) per layer, overwritten; a NULL pointer
 *       is skipped; bn_weight / bn_bias must be NULL (SNB200_EINVAL otherwise).  grad_x may be NULL (no gradient to the points).
 *   last layer L:   dW_L[c,:] = sum over clouds b, then prefixes p, of g[p,b,c] [pooled > 0] a_{L-1}[b, route[p,b,c], :]; db_L[c] the sum of
 *                   the coefficients (a channel pooled to 0 under ReLU gets exactly 0);
 *   hidden layers:  dW_l = sum over points of dz_l^T a_{l-1} (a_0 = x), db_l = sum dz_l, dz_l from the same chain as grad_x; the points are
 *                   summed in fixed chunks, the chunks added in a fixed order.  No float atomics: run to run bit-identical, and grad_x is
 *                   bit for bit snb200_frozen_encoder_backward's.
 *   workspace: the route bits plus each hidden layer's gradient rows (b*n, c_out_l) and per-chunk partials, all counted by the query.
 *   snb200_frozen_encoder_param_backward_supported(...) != 0 : snb200_frozen_encoder_supported's envelope with no BatchNorm on any layer;
 *       outside it the call returns SNB200_EUNSUPPORTED and launches nothing.
 * snb200_frozen_encoder_backward is this entry with no parameter gradients.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_frozen_encoder_param_backward_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix);
size_t snb200_frozen_encoder_param_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix);
int snb200_frozen_encoder_param_backward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                         const float *pooled, const int *route, float *const *zsave, const float *grad_pooled, float *grad_x,
                                         const snb200_layer_grad *conv_grads, void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * A FROZEN fully connected head on at most 64 rows, with the gradient to its input only (PCRNet's 2048-1024-1024-512-512-256-7 head,
 * registration/models/pcrnet.py:46-82, frozen while the sampler trains: registration/main.py:256-258).
 *   in (b, c_in_0); layer l: a_l = act(W_l a_{l-1} + bias_l), act = ReLU where layers[l].relu, identity otherwise; out (b, c_out_last).
 *   asave: per hidden layer l < num_layers - 1 a (b, c_out_l) float buffer that receives a_l (kept for the backward), or NULL (forward only:
 *          the hidden layers then live in the workspace, sized with with_save = 0; with with_save = 1 the forward needs no workspace).
 * The backward gives grad_in (b, c_in_0) = d sum(grad_out * out) / d in, overwritten; a ReLU's mask is a_l > 0 of the saved activation.
 * One launch per layer chained by programmatic dependent launch (plus one that adds the first layer's partial blocks when its output
 * channels were split); every weight is read once per pass; no float atomics: run to run bit-identical.
 *   snb200_frozen_mlp_supported(...) != 0 : 1 <= b <= 64, 1..SNB200_MAX_FC_LAYERS layers chained c_out -> c_in, c_in a multiple of 8 up to
 *       4096, c_out 1..4096, no BatchNorm on any layer, ReLU on any subset of the hidden layers (none on the last one, whose output is
 *       not saved).  Outside it the calls return SNB200_EUNSUPPORTED and launch nothing.  `in`, asave[l] and the weights are 16-byte aligned.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_frozen_mlp_supported(int b, int num_layers, const snb200_layer *layers);
size_t snb200_frozen_mlp_workspace_bytes(int b, int num_layers, const snb200_layer *layers, int with_save);
int snb200_frozen_mlp_forward(int b, const float *in, int num_layers, const snb200_layer *layers, float *out, float *const *asave,
                              void *workspace, size_t workspace_bytes, snb200_stream_t stream);
size_t snb200_frozen_mlp_backward_workspace_bytes(int b, int num_layers, const snb200_layer *layers);
int snb200_frozen_mlp_backward(int b, int num_layers, const snb200_layer *layers, float *const *asave, const float *grad_out, float *grad_in,
                               void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* The same backward with weight and bias gradients (PCRNet's head trained: registration/main.py --train-pcrnet).
 *   in (b, c_in_0): the head's input, read for grads[0].weight (may be NULL otherwise); grads[num_layers] (snb200_layer_grad): weight
 *   (c_out, c_in) 16-byte aligned and bias (c_out) per layer, overwritten, a NULL pointer skipped, bn_weight / bn_bias NULL (SNB200_EINVAL
 *   otherwise).  dW_l[o,k] = sum_r g[r,o] a_{l-1}[r,k] and db_l[o] = sum_r g[r,o] over the rows in row order, g the gradient of layer l's
 *   pre-activation; grad_in may be NULL and is otherwise bit for bit snb200_frozen_mlp_backward's.  Same kernels (an epilogue of the input
 *   gradient's), same workspace, same envelope; run to run bit-identical.  snb200_frozen_mlp_backward is this entry with no parameter
 *   gradients. */
int snb200_frozen_mlp_param_backward_supported(int b, int num_layers, const snb200_layer *layers);
size_t snb200_frozen_mlp_param_backward_workspace_bytes(int b, int num_layers, const snb200_layer *layers);
int snb200_frozen_mlp_param_backward(int b, int num_layers, const snb200_layer *layers, const float *in, float *const *asave, const float *grad_out,
                                     float *grad_in, const snb200_layer_grad *grads, void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The same frozen MLP (same kernels, same workspaces) with eval-mode BatchNorm allowed on any layer (the FC layers of PointNet's classifier
 * and transform nets, classification/models/pointnet_cls.py + transform_nets.py, frozen while the sampler trains).
 *   layer l with BatchNorm: a_l = act(fmaf(z_l, scale, shift)), z_l = W_l a_{l-1} + bias_l, scale = gamma / sqrtf(running_var + eps),
 *   shift = beta - running_mean * scale, evaluated per call from the layer's own parameters as the frozen encoder does.  The running
 *   statistics are required (SNB200_EINVAL without them).  The backward's gradient of z_l is grad a_l * [a_l > 0 where ReLU] * scale.
 *   snb200_frozen_mlp_bn_supported(...) != 0 : the envelope of snb200_frozen_mlp_supported with BatchNorm allowed (SNB200_EUNSUPPORTED outside).
 * --------------------------------------------------------------------------------------------------------- */
int snb200_frozen_mlp_bn_supported(int b, int num_layers, const snb200_layer *layers);
size_t snb200_frozen_mlp_bn_workspace_bytes(int b, int num_layers, const snb200_layer *layers, int with_save);
int snb200_frozen_mlp_bn_forward(int b, const float *in, int num_layers, const snb200_layer *layers, float *out, float *const *asave,
                                 void *workspace, size_t workspace_bytes, snb200_stream_t stream);
size_t snb200_frozen_mlp_bn_backward_workspace_bytes(int b, int num_layers, const snb200_layer *layers);
int snb200_frozen_mlp_bn_backward(int b, int num_layers, const snb200_layer *layers, float *const *asave, const float *grad_out, float *grad_in,
                                  void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * A per-cloud K x K transform of points or point features (PointNet's input and feature transforms: `tf.matmul(point_cloud, transform)` in
 * classification/models/pointnet_cls.py, rows times T).
 *   in (b,n,k), T (b,k,k) row-major;  forward: out[b,i,:] = in[b,i,:] @ T[b]  (out (b,n,k), overwritten).
 *   backward: grad_in[b,i,:] = grad_out[b,i,:] @ T[b]^T  and  grad_T[b] = sum_i in[b,i,:]^T grad_out[b,i,:]  (both overwritten).  The sum over
 *   points runs in a fixed order (chunks of 128 points, added in chunk order): no float atomics, run to run bit-identical.
 *   workspace: the backward's per-chunk partial grad_T, snb200_point_transform_workspace_bytes (0 for clouds of at most 128 points); the
 *   forward takes none.  1 <= b <= 65535, 1 <= n <= 2^24, 1 <= k <= 64 (SNB200_EUNSUPPORTED otherwise; nothing launches).
 * --------------------------------------------------------------------------------------------------------- */
int snb200_point_transform_supported(int b, int n, int k);
size_t snb200_point_transform_workspace_bytes(int b, int n, int k);
int snb200_point_transform_forward(int b, int n, int k, const float *in, const float *T, float *out, snb200_stream_t stream);
int snb200_point_transform_backward(int b, int n, int k, const float *in, const float *T, const float *grad_out, float *grad_in, float *grad_T,
                                    void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* The point transform over the segments of a packed buffer (the layout of snb200_frozen_encoder_seg_*: seg (num_seg, 2) int32 in device
 * memory, offsets multiples of 128 in ascending order, padding to the next multiple of 128): segment j multiplies its rows by its own T[j]
 * (T (num_seg, k, k)).  out (total, k): segment rows as snb200_point_transform_forward makes each row, padding rows 0.
 *   num_prefix = 0, packed source: `in` is a (total, k) packed buffer in the same layout; grad_in (total, k), padding rows 0.
 *   num_prefix > 0, prefix source: `in` is an unpacked (src_b, src_n, k) input; segment j = p * src_b + b reads rows [0, sizes[p]) of cloud b
 *       (its length must be sizes[p]; sizes a HOST array, ascending in [1, min(src_n, max_len)]).  No prefix is copied.  grad_in (src_b, src_n,
 *       k): grad_in[b, i] is the sum over the prefixes p with sizes[p] > i, in ascending p, of that segment row's gradient; one owner per point,
 *       no atomics; points beyond every prefix get 0.
 *   grad_T[j] = sum of in^T grad_out over segment j's rows, in chunks of 128 rows added in chunk order (as snb200_point_transform_backward).
 *   workspace: the backward's per-chunk partials, snb200_point_transform_seg_workspace_bytes; the forward takes none.  Run to run
 *   bit-identical.
 *   snb200_point_transform_seg_supported(...) != 0 : total <= 2^22, 1 <= num_seg <= ceil(total/128), 1 <= max_len <= 4096, 1 <= k <= 64; a
 *   prefix source adds 1..16 prefixes of src_b <= 65535 clouds (SNB200_EUNSUPPORTED otherwise; nothing launches). */
int snb200_point_transform_seg_supported(int num_seg, int total, int max_len, int k);
size_t snb200_point_transform_seg_workspace_bytes(int num_seg, int total, int max_len, int k);
int snb200_point_transform_seg_forward(int num_seg, int total, int max_len, const int *seg, int k, int src_b, int src_n, int num_prefix,
                                       const int *sizes, const float *in, const float *T, float *out, snb200_stream_t stream);
int snb200_point_transform_seg_backward(int num_seg, int total, int max_len, const int *seg, int k, int src_b, int src_n, int num_prefix,
                                        const int *sizes, const float *in, const float *T, const float *grad_out, float *grad_in, float *grad_T,
                                        void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The registration task loss behind PCRNet's last layer (registration/main.py:555-598 compute_pcrnet_loss; src/qdataset.py:93-119
 * compute_errors / rotate; src/quaternion.py:35-53 qrot), one launch forward and one backward.
 *   y (b,7) raw fc6 output; p0, p1 (b,m,3) BNC; igt (b,7) ground truth (w,x,y,z, t).
 *   twist (b,7): y[:4] / max(|y[:4]|, 1e-12), then y[4:] as is;  e = qrot(twist[:4], p0): the rotation only, the translation is not applied
 *   idx01 (b,m): for p1[i] the nearest e[j];  idx10 (b,m): for e[j] the nearest p1[i]  (squared distances, lowest index on ties)
 *   terms (5): chamfer_loss = mean c01 + mean c10 over b*m; qnorm_loss = mean (|y[:4]|^2 - 1)^2; norm_err = mean |R(q) R(q_gt)^T - I|_F^2;
 *              rot_err = mean 2 acos(2 (q . q_gt)^2 - 1) in radians; trans_err = mean |y[4:] - t_gt|
 *   workspace: per-pair sums, added in pair order by the last CTA; ticket: one zero-initialised unsigned, left zero.
 * The backward takes grad_terms (5, device; the entry of rot_err is ignored: nothing differentiates it) and overwrites grad_y (b,7),
 * grad_p0 and grad_p1 (b,m,3).  The Chamfer gradient is gathered per point inside the CTA: no float atomics, run to run bit-identical.
 * 1 <= b <= 256, 1 <= m <= 1024 (SNB200_EUNSUPPORTED otherwise; nothing launches).
 * --------------------------------------------------------------------------------------------------------- */
size_t snb200_pose_loss_workspace_bytes(int b, int m);
int snb200_pose_loss_forward(int b, int m, const float *y, const float *p0, const float *p1, const float *igt, float *twist, int *idx01,
                             int *idx10, float *terms, void *workspace, size_t workspace_bytes, unsigned *ticket, snb200_stream_t stream);
int snb200_pose_loss_backward(int b, int m, const float *y, const float *p0, const float *p1, const float *igt, const int *idx01,
                              const int *idx10, const float *grad_terms, float *grad_y, float *grad_p0, float *grad_p1, snb200_stream_t stream);

/* Evaluation form of the pose loss (registration/main.py:416-483 test_1 wants the errors of every pair): forward only, one launch.
 *   per_pair (b,6): chamfer = mean c01 + mean c10 of that pair; qnorm; norm_err; rot_err in radians; trans_err; consistency =
 *                   mean c01 + mean c10 of p0s against qrot(conj(igt[:4]), p1s) (main.py:540-553), 0 when p0s and p1s are null.
 *   p0s, p1s (b,ms,3): the sampled pair, both or neither; they may be p0, p1.  twist (b,7) as the forward.
 * The arithmetic, tie rule and in-pair summation order are the forward's, so the mean over pairs of columns 0-4 is its `terms` up to the
 * rounding of that last mean.  No workspace.  1 <= b <= 256, 1 <= m, ms <= 1024 (SNB200_EUNSUPPORTED otherwise; nothing launches). */
int snb200_pose_eval_supported(int b, int m, int ms);
int snb200_pose_eval(int b, int m, const float *y, const float *p0, const float *p1, const float *igt, int ms, const float *p0s,
                     const float *p1s, float *per_pair, float *twist, snb200_stream_t stream);

/* The pose loss and its evaluation form with clouds of two sizes (registration/main.py --num-sampled-clouds 1 samples the source only: the
 * full template against the sampled source, main.py:492-496, :514-516).  Each entry is its plain namesake above with p0 (b,m0,3) and
 * p1 (b,m1,3):
 *   idx01 (b,m1): for p1[i] the nearest of the m0 points of e;  idx10 (b,m0): for e[j] the nearest of the m1 points of p1;
 *   chamfer_loss = sum c01 / (b*m1) + sum c10 / (b*m0) (the reference's mean(dist1) + mean(dist2), main.py:573-577);
 *   grad_p0 (b,m0,3), grad_p1 (b,m1,3);
 *   pose_eval_ex: p0s (b,ms0,3), p1s (b,ms1,3); consistency = mean over p0s + mean over qrot(conj(igt[:4]), p1s).
 * With m0 == m1 (and ms0 == ms1) every output is bit-identical to the plain entry's: the plain entries are these with one size.
 * snb200_pose_loss_ex_supported: 1 <= b <= 256, 1 <= m0, m1 <= 1024; pose_eval_ex needs it for (b, m0, m1) and, with the sampled pair,
 * for (b, ms0, ms1).  SNB200_EUNSUPPORTED otherwise; nothing launches.  The workspace is the plain forward's (0 outside the envelope). */
int snb200_pose_loss_ex_supported(int b, int m0, int m1);
size_t snb200_pose_loss_ex_workspace_bytes(int b, int m0, int m1);
int snb200_pose_loss_ex_forward(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, float *twist,
                                int *idx01, int *idx10, float *terms, void *workspace, size_t workspace_bytes, unsigned *ticket,
                                snb200_stream_t stream);
int snb200_pose_loss_ex_backward(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, const int *idx01,
                                 const int *idx10, const float *grad_terms, float *grad_y, float *grad_p0, float *grad_p1, snb200_stream_t stream);
int snb200_pose_eval_ex(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, int ms0, int ms1,
                        const float *p0s, const float *p1s, float *per_pair, float *twist, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * EMD.  xyz1 (b,n,3), xyz2 (b,m,3), match (b,m,n), cost (b), grad1 (b,n,3), grad2 (b,m,3).
 * Replace approxmatchLauncher / matchcostLauncher / matchcostgradLauncher
 * (classification/structural_losses/tf_approxmatch.cpp:141-143, tf_approxmatch_g.cu:181,227,293-294).
 * `temp` of the reference (tf_approxmatch.cpp:168) is the workspace here.
 * --------------------------------------------------------------------------------------------------------- */
size_t snb200_approxmatch_workspace_bytes(int b, int n, int m);
int snb200_approxmatch(int b, int n, int m, const float *xyz1, const float *xyz2, float *match, void *workspace,
                       size_t workspace_bytes, snb200_stream_t stream);
/* flags & SNB200_EMD_EXACT: the parity mode -- exact exponential (exp in double, rounded to float), one float accumulator per row summed in
 * index order, the reference's level order and per-level read-modify-write of `match`: operation-for-operation the arithmetic of the CPU
 * oracle, so match values AND arg-max assignments are bit-identical to it (workspace unused).  Without the flag: the fast kernel. */
#define SNB200_EMD_EXACT 1
int snb200_approxmatch_mode(int b, int n, int m, const float *xyz1, const float *xyz2, float *match, int flags, void *workspace,
                            size_t workspace_bytes, snb200_stream_t stream);
size_t snb200_matchcost_workspace_bytes(int b);
int snb200_matchcost(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *cost,
                     void *workspace, size_t workspace_bytes, snb200_stream_t stream);
int snb200_matchcostgrad(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *grad1,
                         float *grad2, snb200_stream_t stream);

/* Per-cloud EMD without the match tensor: cost (b) = snb200_matchcost(xyz1, xyz2, snb200_approxmatch(xyz1, xyz2)) bit for bit, where
 * xyz1 (b,n,3) and xyz2 (b2,m,3) with b2 dividing b, and pair bi matches xyz1[bi] with xyz2[bi % b2] (b2 == b: cloud with cloud).  The
 * levels run as snb200_approxmatch runs them; the match values are rebuilt where the cost and gradient kernels need them from the
 * per-level ratios kept in the workspace.  Nothing of size b x m x n is stored.
 * The backward takes grad_cost (b) and the workspace the forward filled (unchanged since) and writes grad1 (b,n,3) and grad2 (b,m,3), per
 * pair even when b2 < b: grad_cost[bi] times snb200_matchcostgrad's outputs on that match, bit for bit.  Either of grad1 / grad2 may be
 * null (not both): that gradient is then not computed, which saves its pass.  No float atomics.
 * Envelope (snb200_emd_per_cloud_supported != 0): 1 <= b <= 65535, 1 <= n <= 2^24, 1 <= m <= 65520 (the m snb200_matchcost takes); the
 * workspace query answers 0 outside
 * it.  b = 0 launches nothing.  These four entries are the _mode family below with flags = 0. */
int snb200_emd_per_cloud_supported(int b, int n, int m);
size_t snb200_emd_per_cloud_workspace_bytes(int b, int n, int m);
int snb200_emd_per_cloud(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, float *cost, void *workspace,
                         size_t workspace_bytes, snb200_stream_t stream);
int snb200_emd_per_cloud_backward(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, const float *grad_cost, float *grad1,
                                  float *grad2, const void *workspace, size_t workspace_bytes, snb200_stream_t stream);
/* The per-cloud EMD in either mode.  flags = 0: the entries above.  flags & SNB200_EMD_EXACT: cost = snb200_matchcost(xyz1, xyz2,
 * snb200_approxmatch_mode(xyz1, xyz2, SNB200_EMD_EXACT)) and the gradients grad_cost[bi] times snb200_matchcostgrad's on that match, bit
 * for bit, with the same b2 repeat, null-gradient rule and workspace use.  The exact levels run one CTA per cloud as the exact approx_match
 * does, but write no match: each level's ratios go to the workspace, and every match element is rebuilt from them in the exact mode's
 * own arithmetic.  Workspace: the same size in both modes, 256 + align256(44 * b * (n + m)) + align256(64 * b) bytes (a grid-barrier word,
 * 11 floats per point and cloud, 16 cost partials per cloud).  Exact envelope: 1 <= b <= 65535, n >= 1, m >= 1, n + m <= 25600 (the
 * exact kernel's 200 KB of shared-memory vectors, as for snb200_approxmatch_mode); outside it the entries return SNB200_EUNSUPPORTED
 * before any launch and the queries answer 0.  The backward takes the flags its forward was given. */
int snb200_emd_per_cloud_mode_supported(int b, int n, int m, int flags);
size_t snb200_emd_per_cloud_mode_workspace_bytes(int b, int n, int m, int flags);
int snb200_emd_per_cloud_mode(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, float *cost, int flags, void *workspace,
                              size_t workspace_bytes, snb200_stream_t stream);
int snb200_emd_per_cloud_mode_backward(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, const float *grad_cost, float *grad1,
                                       float *grad2, int flags, const void *workspace, size_t workspace_bytes, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Inference matching on the GPU (registration/src/samplenet.py:119-141 + sputils.py:7-41): order-preserving unique
 * of the NN indices, then farthest-point-sampling completion to k points.  full_pc (b,n,3) BNC, nn_idx (b,t),
 * out (b,k,3) BNC, out_idx (b,k) (may be NULL).  complete_fps == 0 -> plain gather of the first k indices.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_nn_matching(int b, int n, int t, int k, const float *full_pc, const int *nn_idx, int complete_fps, float *out,
                       int *out_idx, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Farthest point sampling.  inp (b,n,3) BNC or (b,3,n) BCN; idx (b,m) int32; out_points (b,m,3) / (b,3,m) in `layout`, may be NULL:
 * when given, the selected coordinates are written too (the gather every caller does next, without a second launch).
 * Replaces farthestpointsamplingLauncher (reconstruction/external/sampling/tf_sampling.cpp:98-120, tf_sampling_g.cu:203-205) and
 * returns the same indices: idx[0] = 0, then each round the point farthest (fma-contracted squared distance, as the reference kernel)
 * from the points selected so far; equal maxima go to the smallest (k mod 512, k div 512), the reference's thread order.  m > n is
 * allowed (index 0 repeats once every point is taken).  b >= 0, m >= 1, 1 <= n <= 16384 (larger clouds: SNB200_EUNSUPPORTED).
 * No workspace (the reference's `temp` of 32*n floats is not needed).  No gradient.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_farthest_point_sample(int b, int n, int m, int layout, const float *inp, int *idx, float *out_points, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The classification trainer's augmentation in one launch: rotation about the up axis, then jitter (classification/train_classifier.py:217-221:
 * provider.rotate_point_cloud + provider.jitter_point_cloud, provider.py:35-53, :76-87), and the evaluation votes' fixed rotations
 * (evaluate_classifier.py:163-167, provider.rotate_point_cloud_by_angle).
 *   in (b,n,3) BNC; out (replicas,b,n,3): replica r of cloud c is in[c] rotated about y by angles[r] (angles (replicas,) float64 on the device),
 *       or, with angles == NULL (replicas must be 1), by an angle drawn for each cloud.  As np.dot(pc, R), R = [[c,0,s],[0,1,0],[-s,0,c]]:
 *       x' = x*c - z*s, y' = y, z' = x*s + z*c in float64, rounded to float32.
 *   sigma > 0: jitter, out = fl32(fl32(rot) + clip(sigma*z, -clip, clip)) with the normal z, the clip and the sum in float64.  sigma = 0: none.
 *   key: 2 words on the device, read only when angles == NULL or sigma > 0.
 * Random numbers (numpy's MT19937 stream is not reproduced; this stream does not depend on the launch configuration):
 *   Philox4x32-10 (Random123; curand_Philox4x32_10 in curand_philox4x32_x.h) with key (lo32(k0), hi32(k0)) and counter
 *       (cloud, j, lo32(k1), hi32(k1)), cloud the output cloud r*b + c, giving the words (w0, w1, w2, w3);
 *   u(wa, wb) = ((wa >> 5) * 2^26 + (wb >> 6)) * 2^-53 in float64 (numpy's 53-bit construction);
 *   angle: j = 0xFFFFFFFF, angle = u(w0, w1) * 2 * pi (np.random.uniform() * 2 * np.pi);
 *   jitter of point i: j = 2i gives the normals of x and y, j = 2i+1 the normal of z; for each, u1 = u(w0,w1), u2 = u(w2,w3),
 *       r = sqrt(-2 log(1 - u1)), z0 = r cos(2 pi u2), z1 = r sin(2 pi u2), all in float64 (x: z0 and y: z1 of j = 2i; z: z0 of j = 2i+1).
 * 1 <= n <= 2^24 (2i+1 stays below the angle's j), replicas >= 1, b * replicas <= 2^31 - 1 (the grid); b = 0 does nothing.  sigma >= 0, and
 * clip > 0 while sigma > 0 (provider.py asserts it).  In place (in == out) only with replicas == 1; no other overlap.  SNB200_EINVAL otherwise.
 * Writes `out` only.  No gradient.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_rotate_jitter(int b, int n, int replicas, const float *in, float *out, const double *angles, const unsigned long long *key, double sigma,
                         double clip, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The reconstruction trainers' augmentation in one launch (general_utils.apply_augmentations, reconstruction/src/general_utils.py:100-117, as
 * the autoencoder and sampler epochs apply it to every batch): Gaussian noise, then one z-rotation for the whole batch.
 *   in (b,n,3) BNC; out (b,n,3).
 *   gauss != 0: every coordinate v becomes fl32(v + (mu + sigma*z)) with a standard normal z, the product and both sums in float64
 *       (batch += np.random.normal(mu, sigma, batch.shape) on a float32 batch).
 *   z_rotate != 0: then (x, y, z) becomes (fl32(x*R00 + y*R10), fl32(x*R01 + y*R11), z) in float64 (batch.dot(R), row vectors), R being
 *       rand_rotation_matrix() (general_utils.py:16-52, deflection 1) with R[0,2] = R[2,0] = R[1,2] = R[2,1] = 0 and R[2,2] = 1.  Its upper
 *       2x2 block is that of a random 3-D rotation, so R is in general not orthogonal; it is restated as the reference has it.  One R per
 *       launch: theta = u0 * 2 * pi, phi = u1 * 2 * pi, zeta = u2 * 2, r = sqrt(zeta), V = (sin(phi) r, cos(phi) r, sqrt(2 - zeta)),
 *       R = (V V^T - I) [[cos theta, sin theta, 0], [-sin theta, cos theta, 0], [0, 0, 1]] in float64.
 *   key: 2 words on the device, read only when gauss or z_rotate.
 * Random numbers (numpy's MT19937 stream is not reproduced; this stream does not depend on the launch configuration): snb200_rotate_jitter's
 *   Philox4x32-10 words, uniform and Box-Muller with counter (c, j, lo32(k1), hi32(k1)):
 *   noise of point i of cloud c: j = 2i gives the normals of x and y, j = 2i+1 the normal of z (x: z0 and y: z1 of j = 2i; z: z0 of j = 2i+1);
 *   rotation: u0 = u(w0, w1), u1 = u(w2, w3) of the counter (0, 0xFFFFFFFF), u2 = u(w0, w1) of (1, 0xFFFFFFFF).
 * 1 <= n <= 2^24, b >= 0 (b = 0 does nothing).  mu and sigma finite and sigma >= 0 while gauss.  Neither gauss nor z_rotate copies in to out.
 * In place (in == out) or no overlap; SNB200_EINVAL otherwise.  Writes `out` only.  No gradient.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_ae_augment(int b, int n, const float *in, float *out, const unsigned long long *key, int gauss, double mu, double sigma, int z_rotate,
                      snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * The registration trainer's pairs in one launch: ModelNetCls.__getitem__'s random point order (registration/data/modelnet_loader_torch.py:
 * 102-116) over a set already on the unit cube, then QuaternionFixedDataset.__getitem__'s fixed rotation (registration/src/qdataset.py:160-179).
 *   clouds (s,n,3) BNC; records (b,) int32 on the device; transforms (num_records,7) rows (w, x, y, z, tx, ty, tz); key: 2 words on the device.
 *   Pair i takes r = records[i], cloud r % s and transform row r.  records is not read on the host: 0 <= records[i] < num_records is the
 *   caller's precondition.
 *   perm (b,n) int32, optional (NULL: not written): perm[i] lists 0..n-1 in ascending order of the sort keys
 *       ((w0 << 32 | w1) & ~0x7FF) | j, (w0, w1) the first two words of Philox4x32-10 (Random123; curand_Philox4x32_10) with key
 *       (lo32(k0), hi32(k0)) and counter (i, j, lo32(k1), hi32(k1)).  The keys are unique, so perm[i] is a permutation; numpy's
 *       np.random.shuffle stream is not reproduced.
 *   p0 (b,n,3): p0[i,j] = clouds[r % s, perm[i,j]], copied exactly.
 *   p1 (b,n,3): p1[i,j] = qrot(q_r, p0[i,j]) in float32 in registration.qrot's order, every product, difference and sum rounded (no FMA):
 *       uv = qvec x v, uuv = qvec x uv, p1 = v + 2 (w uv + uuv).  The translation is not applied (QuaternionTransform.rotate).
 *   vec (b,7): vec[i] = transforms[r].
 * 1 <= n <= 2048 (SNB200_EUNSUPPORTED above), b >= 0 (b = 0 does nothing), s >= 1, num_records >= 1; the outputs overlap neither each other
 * nor the inputs.  SNB200_EINVAL otherwise.  Writes p0, p1, vec and perm only.  No gradient, no workspace.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_registration_pairs(int b, int n, int s, int num_records, const float *clouds, const int *records, const float *transforms,
                              const unsigned long long *key, float *p0, float *p1, float *vec, int *perm, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Shape-retrieval metrics of descriptor sets (the classifiers' end_points["retrieval_vectors"], classification/models/pointnet_cls.py:111):
 * every query ranks the whole database; average precision and the interpolated precision curve of that ranking.
 *   queries (q,d), database (m,d) float32 row-major; query_labels (q,), database_labels (m,) int32.
 *   exclude_diagonal != 0 (needs q == m): database item i is never a result for query i (leave-one-out; database may be queries).
 *   Distance: d(a, x) = sum_{k=0..d-1} fl(fl(a_k - x_k)^2), accumulated left to right in float32, every product and sum rounded (no
 *       contraction): numpy's float32 ((a - x) ** 2) summed sequentially.  Independent of tiling, batch and launch shape.
 *   Order: the m' results (m, minus the excluded item) sorted by (d, index) ascending (numpy's argsort(kind="stable")); a NaN distance ranks
 *       after +inf.  rel(k) = [label of the k-th result == query label], hits(k) = sum_{j<=k} rel(j), R = hits(m').
 *   ap (q,) float64: (sum over k of rel(k) * hits(k) / k, each term hits / k in float64, summed in rank order) / R.
 *   prec (q, levels) float64: prec[l] = max over k with hits(k) * (levels - 1) >= l * R (in integers) of hits(k) / k, l = 0 .. levels - 1.
 *   num_relevant (q,) int32: R.  With R = 0, ap and the whole prec row are NaN.
 * Writes ap, prec and num_relevant only, each entry once; no workspace, no float atomics, run to run bit-identical.  Asynchronous on `stream`.
 * snb200_retrieval_metrics_supported(...) != 0 : 1 <= q <= 2^20, 1 <= m <= 16384, 1 <= d <= 1024, 2 <= levels <= 101, q == m when
 *   exclude_diagonal.  Outside it the entry returns SNB200_EUNSUPPORTED, names the bound in snb200_last_error and launches nothing.
 * --------------------------------------------------------------------------------------------------------- */
int snb200_retrieval_metrics_supported(int q, int m, int d, int levels, int exclude_diagonal);
int snb200_retrieval_metrics(int q, int m, int d, const float *queries, const int *query_labels, const float *database, const int *database_labels,
                             int exclude_diagonal, int levels, double *ap, double *prec, int *num_relevant, snb200_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Non-finite step guard: undo a training step that went non-finite, on the device, with no read-back.
 *   checks[num_checks]      tensors to test; an element is non-finite when its exponent bits are all ones (NaN, +-Inf).  dtype is one
 *                           of SNB200_GUARD_F32 / F64 / F16 / BF16; integer tensors are finite by construction and are not listed.
 *   restores[num_restores]  (live, snapshot, bytes) pairs: when any checked element is non-finite, every snapshot is copied over its live
 *                           tensor bit for bit (-0.0 and NaN payloads included), and nothing is copied otherwise.
 *   state                   DEVICE, 2 unsigned words, zero at the first call and left zero by every call (allocate once, never touch);
 *                           concurrent calls need their own.
 *   skipped                 DEVICE int, may be NULL: 1 if this call restored, else 0.
 *   skip_count              DEVICE int, may be NULL: incremented when this call restored.
 * The tables are HOST arrays, copied into the launches' parameters: a captured call keeps the tables of its capture.  Two launches (check,
 * then restore) for up to 384 entries per table, one more per further 384; no allocation, no float atomics.
 * --------------------------------------------------------------------------------------------------------- */
#define SNB200_GUARD_F32 0
#define SNB200_GUARD_F64 1
#define SNB200_GUARD_F16 2
#define SNB200_GUARD_BF16 3

typedef struct {
    const void *ptr;          /* DEVICE */
    int count;                /* elements */
    int dtype;                /* SNB200_GUARD_* */
} snb200_guard_check;

typedef struct {
    void *live;               /* DEVICE */
    const void *snapshot;     /* DEVICE */
    long long bytes;
} snb200_guard_restore;

int snb200_nonfinite_guard(const snb200_guard_check *checks, int num_checks, const snb200_guard_restore *restores, int num_restores,
                           unsigned *state, int *skipped, int *skip_count, snb200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SAMPLENET_B200_H */
