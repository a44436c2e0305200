// generator_bwd.cu -- backward pass of the SampleNet generator (registration/main.py:348-352 `loss.backward()` through
// samplenet.py:90-104) as hand-written CUDA: no cuBLAS / ATen BatchNorm kernels on the training step.
//
// The same kernels serve both training paths: the fused one (snb200_generator_train_forward) and the per-layer one
// (snb200_generator_layers_train_forward: tensor-core layer kernels + cluster FC head, for the reconstruction / classification samplers).
// The forward conv-stack kernel (conv_stack.cu) keeps, when asked, every conv layer's raw output z_l (points x channels, with bias) --
// 58.7 MB at the headline size, written from the registers that hold it anyway while the CTA waits at the statistics barrier; the
// per-layer (sum, sumsq) statistics and the FC head's inputs stay in the forward workspace.  Backward, top down:
//   fc_bwd_kernel        x4   one FC layer: recompute z (tiny), BatchNorm-over-the-batch backward, dW / db / dgamma / dbeta for the 8
//                              output channels of a CTA (deterministic: a CTA owns its rows), dZ to global; the layer's input gradient
//                              dZ_up . W_up is evaluated by the consumer (the next kernel) for its own channels only, streaming the
//                              upper layer through shared memory in chunks of channels when it is too wide to stage whole
//   pool_bwd_kernel      x1   grad of the pooled feature (fc1's input gradient), arg-max of the last conv layer per (cloud, channel)
//                              = the only points that receive a gradient through the max-pool, and that layer's BatchNorm sums
//   conv_bwd_kernel<Ci,Cs,Co> x4 one conv layer l (conv5 .. conv2) per launch, persistent over 32-point tiles (input channels in Cs-wide
//                              slices over grid.y: the 256-wide layers of the per-layer training path, see the kernel):
//                              dz_l = gamma/sigma (dy_l - mean(dy_l) - zhat_l mean(dy_l zhat_l))        (BatchNorm backward, on load)
//                              dy_{l-1} = (dz_l W_l) * [y_{l-1} > 0]            (dgrad, 4x8 / 2x8 register tiles, fp32 FFMA)
//                              dW_l += dz_l^T a_{l-1}, db_l += sum dz_l          (wgrad, 8x8 register tiles, per-CTA partials)
//                              and the BatchNorm sums of layer l-1 (sum dy, sum dy zhat) for the next launch
//   conv1_bwd_kernel     x1   dW_1 = dz_1^T x (K = 3), db_1
//   reduce_partials_kernel x1 per-CTA weight-gradient partials -> gradients, fixed order (bit-reproducible)
// Exact fp32 arithmetic (CUDA cores): the products are the same 4.3 GFLOP a cuBLAS SGEMM backward performs; what goes away is the
// ~120 library launches, the recompute of the forward in stock ops and every activation / mask / BatchNorm intermediate in HBM.
#include "encoder_internal.cuh"
#include <string.h>

namespace snb {

constexpr int kFcbThreads = 256;
constexpr int kFcbMaxRows = 64;

// ------------------------------------------------------------------------------------------------------------------ FC layer
struct FcBwdParams {
    int b, c_in, c_out;
    const float *a_in;          // (b, c_in) the layer's input (post-activation of the layer below / pooled feature; dropout-masked if any)
    const float *a_out;         // (b, c_out) the layer's OUTPUT as the forward stored it (post-ReLU), or null: the ReLU mask the forward used
    const float *weight, *bias, *gamma, *beta;
    float eps;
    int has_bn, relu;
    // gradient wrt this layer's OUTPUT: either grad_out (top layer; column permutation out_inner as in the forward store) ...
    const float *grad_out; int out_inner;
    // ... or dZ_up (b, c_up) . W_up (c_up, c_out), its c_up upper channels staged u_chunk at a time (fcb_chunk)
    const float *dz_up, *w_up; int c_up, u_chunk;
    const float *mask;          // (b, c_out) the layer above's dropout mask (the forward stored this layer's output masked), or null
    float *dz;                  // (b, c_out) written here
    float *g_weight, *g_bias, *g_gamma, *g_beta;   // (c_out, c_in), (c_out), (c_out), (c_out); any may be null
};

// (rows, cols) of a row-major global array with row stride lds -> shared memory with row stride ld, 8 independent loads per thread and pass
__device__ __forceinline__ void fcb_stage(float *dst, int ld, const float *__restrict__ src, int lds, int rows, int cols, int tid)
{
    const int total = rows * cols;
    for (int e0 = tid; e0 < total; e0 += kFcbThreads * 8) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int e = e0 + u * kFcbThreads, r = e / cols;
            v[u] = e < total ? __ldg(src + (size_t)r * lds + (e - r * cols)) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int e = e0 + u * kFcbThreads;
            if (e < total) { const int r = e / cols, k = e - r * cols; dst[r * ld + k] = v[u]; }
        }
    }
}

__global__ void __launch_bounds__(kFcbThreads) fc_bwd_kernel(const __grid_constant__ FcBwdParams P)
{
    extern __shared__ __align__(16) float fsm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b = P.b, I = P.c_in, O = P.c_out;
    const int U = P.dz_up ? P.u_chunk : 0;             // upper channels per chunk: c_up (one chunk), or a multiple of 4
    float *sA = fsm;                                   // [b][I + 1]
    float *sU = sA + (size_t)b * (I + 1);              // [b][U + 1]  (a chunk of the dz of the layer above)
    float *sWr = sU + (size_t)(U ? b * (U + 1) : 0);   // [8][I] this CTA's weight rows
    const int c = blockIdx.x * 8 + warp;               // the channel of this warp
    const bool cv = c < O;
    float *sWu = sWr + 8 * I + warp * U;               // this warp's chunk of its column of the upper layer's weight: w_up[u0 + u][c], u < U
    // staging: every load of a thread is in flight before its first store (one load -> one store per iteration cost an L2 round trip each:
    // ncu put 60 % of this kernel's stall samples on these stores)
    fcb_stage(sA, I + 1, P.a_in, I, b, I, tid);
    {
        const int rows = min(8, O - (int)blockIdx.x * 8);
        fcb_stage(sWr, I, P.weight + (size_t)blockIdx.x * 8 * I, I, rows, I, tid);
        for (int e = rows * I + tid; e < 8 * I; e += kFcbThreads) sWr[e] = 0.f;
    }
    // gradient wrt this layer's output from the layer above: dout[r] = sum_u dz_up[r][u] w_up[u][c], rows r = lane, lane + 32 (b <= 64),
    // over the upper channels in chunks.  Each chunk but the last holds a multiple of 4 of them, so the four interleaved accumulators see
    // the same u order as one pass over all c_up would give them, and the c_up % 4 tail is left in the last chunk.  The top layer makes
    // one pass that stages nothing of a layer above.
    float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    const int nchunk = U ? (P.c_up + U - 1) / U : 1;
    int un = 0;                                        // channels in the current chunk
    for (int k = 0; k < nchunk; k++) {
        const int u0 = k * U;
        un = U ? min(U, P.c_up - u0) : 0;
        if (k) __syncthreads();                        // every warp is done with the previous chunk
        if (un && cv) {   // (this warp's own region: filled before the CTA barrier, in flight together with the staging loads)
            for (int v0 = lane; v0 < un; v0 += 32 * 8) {
                float v[8];
#pragma unroll
                for (int j = 0; j < 8; j++) { const int u = v0 + 32 * j; v[j] = u < un ? __ldg(P.w_up + (size_t)(u0 + u) * O + c) : 0.f; }
#pragma unroll
                for (int j = 0; j < 8; j++) { const int u = v0 + 32 * j; if (u < un) sWu[u] = v[j]; }
            }
            __syncwarp();
        }
        if (un) fcb_stage(sU, U + 1, P.dz_up + u0, P.c_up, b, un, tid);
        __syncthreads();
        if (cv) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int r = lane + 32 * h;
                if (r < b) {
                    const float *su = sU + r * (U + 1);
                    for (int u = 0; u + 4 <= un; u += 4) {
                        acc[h][0] = fmaf(su[u], sWu[u], acc[h][0]); acc[h][1] = fmaf(su[u + 1], sWu[u + 1], acc[h][1]);
                        acc[h][2] = fmaf(su[u + 2], sWu[u + 2], acc[h][2]); acc[h][3] = fmaf(su[u + 3], sWu[u + 3], acc[h][3]);
                    }
                }
            }
        }
    }
    if (!cv) return;
    float dout[2] = {0.f, 0.f}, z[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int r = lane + 32 * h;
        if (r < b) {
            if (P.dz_up) {
                const float *su = sU + r * (U + 1);   // the last chunk: its c_up % 4 tail
                for (int u = un - (P.c_up & 3); u < un; u++) acc[h][0] = fmaf(su[u], sWu[u], acc[h][0]);
                dout[h] = (acc[h][0] + acc[h][1]) + (acc[h][2] + acc[h][3]);
                if (P.mask) dout[h] *= P.mask[(size_t)r * O + c];   // through the dropout of the layer above's input
            } else {
                const int oc = (P.out_inner > 0) ? (c % P.out_inner) * (O / P.out_inner) + c / P.out_inner : c;
                dout[h] = P.grad_out[(size_t)r * O + oc];
            }
            const float *wr = sWr + warp * I, *sa = sA + r * (I + 1);
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
            int k = 0;
            for (; k + 4 <= I; k += 4) {
                a0 = fmaf(sa[k], wr[k], a0); a1 = fmaf(sa[k + 1], wr[k + 1], a1); a2 = fmaf(sa[k + 2], wr[k + 2], a2); a3 = fmaf(sa[k + 3], wr[k + 3], a3);
            }
            for (; k < I; k++) a0 = fmaf(sa[k], wr[k], a0);
            z[h] = ((a0 + a1) + (a2 + a3)) + (P.bias ? P.bias[c] : 0.f);
        }
    }
    float dzv[2];
    if (P.has_bn) {
        const float inv_b = 1.f / (float)b;
        float s = (lane < b ? z[0] : 0.f) + (lane + 32 < b ? z[1] : 0.f);
        const float mean = warp_sum(s) * inv_b;
        float d0 = lane < b ? z[0] - mean : 0.f, d1 = lane + 32 < b ? z[1] - mean : 0.f;
        const float var = warp_sum(d0 * d0 + d1 * d1) * inv_b;
        const float invstd = rsqrtf(var + P.eps);
        const float gam = P.gamma[c], bet = P.beta[c];
        float zh[2] = {d0 * invstd, d1 * invstd}, dy[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            // the ReLU mask is the one the FORWARD applied (its stored output), not a recomputation: a pre-activation within rounding of
            // zero must not get a gradient the forward pass did not see (one flipped element of a 32..64-row batch moves every row)
            const float y = (P.a_out && lane + 32 * h < b) ? P.a_out[(size_t)(lane + 32 * h) * O + c] : fmaf(gam, zh[h], bet);
            dy[h] = (lane + 32 * h < b && (!P.relu || y > 0.f)) ? dout[h] : 0.f;
        }
        const float s1 = warp_sum(dy[0] + dy[1]);
        const float s2 = warp_sum(dy[0] * zh[0] + dy[1] * zh[1]);
        const float coef = gam * invstd;
#pragma unroll
        for (int h = 0; h < 2; h++) dzv[h] = (lane + 32 * h < b) ? coef * (dy[h] - s1 * inv_b - zh[h] * s2 * inv_b) : 0.f;
        if (lane == 0) { if (P.g_gamma) P.g_gamma[c] = s2; if (P.g_beta) P.g_beta[c] = s1; }
    } else {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int r = lane + 32 * h;
            const float y = (P.a_out && r < b) ? P.a_out[(size_t)r * O + c] : z[h];   // the forward's mask, as above
            dzv[h] = (r < b && (!P.relu || y > 0.f)) ? dout[h] : 0.f;
        }
    }
#pragma unroll
    for (int h = 0; h < 2; h++)
        if (lane + 32 * h < b) P.dz[(size_t)(lane + 32 * h) * O + c] = dzv[h];
    const float dbias = warp_sum(dzv[0] + dzv[1]);
    if (lane == 0 && P.g_bias) P.g_bias[c] = dbias;
    if (P.g_weight) {   // dW[c][k] = sum_r dz[r][c] a_in[r][k]: lanes over k, rows broadcast by shuffle
        for (int k0 = 0; k0 < I; k0 += 32) {
            const int k = k0 + lane;
            float acc = 0.f;
            for (int r = 0; r < b; r++) {
                const float d = __shfl_sync(kFullMask, dzv[r >> 5], r & 31);
                if (k < I) acc = fmaf(d, sA[r * (I + 1) + k], acc);
            }
            if (k < I) P.g_weight[(size_t)c * I + k] = acc;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------ max-pool
struct PoolBwdParams {
    int b, n, C;                 // C = channels of the last conv layer
    const float *z;              // (b*n, C) raw output of the last conv layer
    const double *stats;         // [2][C]
    const float *gamma, *beta; float eps; int has_bn, relu;
    const float *dz1, *w1; int c1;   // fc1: dZ (b, c1), weight (c1, C): grad of the pooled feature = dz1 . w1
    int *pstar;                  // (b, C): flat point index of the arg-max
    float *gval;                 // (b, C): gradient arriving at that point (after the ReLU mask)
    double *s12;                 // [2][C] zeroed: sum dy, sum dy*zhat of the last conv layer
};

// CTA = (cloud, block of 128 channels): thread (grp, c) serves channel 128 blockIdx.y + c, and c below is that layer-wide channel
__global__ void __launch_bounds__(1024) pool_bwd_kernel(const __grid_constant__ PoolBwdParams P)
{
    __shared__ float sDz1[1024];
    __shared__ float sRed[8][128];
    __shared__ int sIdx[8][128];
    __shared__ float sDf[128];
    const int tid = threadIdx.x, grp = tid >> 7, cl = tid & 127, c = (int)blockIdx.y * 128 + cl;
    const int cloud = blockIdx.x, C = P.C;
    for (int e = tid; e < P.c1; e += 1024) sDz1[e] = P.dz1[(size_t)cloud * P.c1 + e];
    __syncthreads();
    // grad of the pooled feature for channel c: sum_u dz1[u] w1[u][c], u split over the 8 groups
    float acc = 0.f;
    if (c < C) {
        const int per = (P.c1 + 7) / 8;
        for (int u = grp * per; u < min(P.c1, (grp + 1) * per); u++) acc = fmaf(sDz1[u], __ldg(P.w1 + (size_t)u * C + c), acc);
    }
    sRed[grp][cl] = acc;
    __syncthreads();
    if (grp == 0) { float t = 0.f; for (int g2 = 0; g2 < 8; g2++) t += sRed[g2][cl]; sDf[cl] = t; }
    __syncthreads();
    // arg-max of y = BN(z) over the cloud's points (first index among equals), 8 point groups per channel
    float sc = 1.f, sh = 0.f, mean = 0.f, invstd = 1.f;
    if (c < C && P.has_bn) {
        const double cnt = (double)P.b * P.n;
        const double m = P.stats[c] / cnt;
        double v = P.stats[C + c] / cnt - m * m;
        if (v < 0) v = 0;
        mean = (float)m; invstd = 1.0f / sqrtf((float)v + P.eps);
        sc = P.gamma[c] * invstd; sh = P.beta[c] - mean * sc;
    }
    // The forward pools the RAW layer output (max where the BatchNorm scale is >= 0, min otherwise: the max-pool commutes with the monotone
    // BN + ReLU map), by exact comparisons: the same rule here -- first index among equal values -- so the gradient goes to the very point
    // whose value the forward used.  `best` is kept as sign * z.
    const float sgn = sc >= 0.f ? 1.f : -1.f;
    float best = -INFINITY; int bi = 0x7fffffff;
    if (c < C) {
        const float *zc = P.z + (size_t)cloud * P.n * C + c;
        for (int p = grp; p < P.n; p += 8) {   // (batching these loads 8 at a time measured 3x slower: 60 vs 20 us under ncu)
            const float y = sgn * zc[(size_t)p * C];
            if (y > best) { best = y; bi = p; }
        }
    }
    __syncthreads();
    sRed[grp][cl] = best; sIdx[grp][cl] = bi;
    __syncthreads();
    if (grp == 0 && c < C) {
        for (int g2 = 1; g2 < 8; g2++) {
            const float o = sRed[g2][cl]; const int oi = sIdx[g2][cl];
            if (o > best || (o == best && oi < bi)) { best = o; bi = oi; }
        }
        if (bi == 0x7fffffff) bi = 0;   // no value compared above -inf (NaN in the channel): point 0, as nn_distance
        const size_t flat = (size_t)cloud * P.n + bi;
        const float zstar = P.z[flat * C + c];
        const float g = (!P.relu || fmaf(sc, zstar, sh) > 0.f) ? sDf[cl] : 0.f;
        const float zh = (zstar - mean) * invstd;
        P.pstar[(size_t)cloud * C + c] = (int)flat;
        P.gval[(size_t)cloud * C + c] = g;
        atomicAdd(P.s12 + c, (double)g);
        atomicAdd(P.s12 + C + c, (double)(g * zh));
    }
}

// ------------------------------------------------------------------------------------------------------------------ conv layers
constexpr int kCbThreads = 256;
constexpr int kCbTP = 32;       // points per tile

struct ConvBwdParams {
    long long P; int n;                      // points, points per cloud
    const float *z;                          // (P, COUT) raw output of this layer
    const float *dy;                         // (P, COUT) dense gradient after the ReLU mask, or null: sparse (pstar, gval)
    const int *pstar; const float *gval;
    const double *stats, *s12;               // this layer: [2][COUT] (sum, sumsq) and (sum dy, sum dy zhat)
    const float *gamma; float eps;
    const float *weight;                     // (COUT, CIN)
    const float *z_in;                       // (P, CIN) raw output of the layer below
    const double *stats_in; const float *gamma_in, *beta_in; float eps_in;
    float *dy_in;                            // (P, CIN) out: gradient wrt the layer below's BN output, ReLU mask applied
    double *s12_in;                          // [2][CIN] zeroed: its BatchNorm sums
    const float *a_in;                       // (P, CIN) or null: layer 1 reading an activation -- a_0 = a_in as it is (z_in, stats_in,
                                             // s12_in unused), and dy_in, if not null, receives the dgrad unmasked
    const float *grad_tap;                   // (P, CIN) or null: added to the dgrad before the layer below's ReLU mask
    float *part;                             // [grid][COUT*CIN + COUT] weight / bias gradient partials of this launch
    float *g_gamma, *g_beta;                 // (COUT)
    // wide last layer (conv_bwd_kernel<..., WIDE>): its cw output channels in slices of COUT over grid.z; the arrays above indexed by an
    // output channel hold cw of them, and each slice leaves its share of dz W (unmasked) in dpart[slice] (P, CIN) for dgrad_combine_kernel
    int cw; float *dpart;
};

// CIN: the layer's input channels (the row stride of z_in / dy_in / W); CS: the slice of them this CTA owns, [blockIdx.y * CS, + CS).
// Layers up to 128 x 128 take the whole input in one CTA (CS == CIN).  The 256-wide layers split it into 64-channel slices over grid.y --
// their W would be 128 KB of shared memory and their wgrad tile 128 accumulators per thread otherwise; each CTA of a point range
// recomputes the full dz tile (BatchNorm backward on load, cheap) and owns its slice of W, of the dgrad output, of the wgrad partials and
// of the layer below's sums.  A 256-wide dz tile needs more than 128 registers per thread to run without spilling: one CTA per SM.
// WIDE: the last layer when it is wider than one CTA's dz tile and W (128 -> up to 1024).  grid.z walks its output channels in slices of
// COUT ([COUT blockIdx.z, +COUT), the last one possibly partial): each CTA computes dz and the wgrad partial of its slice, and its slice's
// part of the dgrad, which dgrad_combine_kernel sums over the slices in slice order before the ReLU mask and the layer below's sums.
template <int CIN, int CS, int COUT, bool SPARSE, bool WIDE = false>
__global__ void __launch_bounds__(kCbThreads, COUT > 128 ? 1 : 2) conv_bwd_kernel(const __grid_constant__ ConvBwdParams Q)
{
    constexpr int LDZ = COUT + 4, LDA = CS + 4;
    constexpr int NCB = CS / 8;                        // dgrad: 8-wide input-channel blocks
    constexpr int PPT = kCbTP * NCB / kCbThreads;      // points per thread in dgrad (2 for CS=128, 1 for CS=64)
    constexpr int WCO = COUT >= 128 ? 8 : 4;           // wgrad register tile
    constexpr int WCI = COUT * CS / kCbThreads / WCO;
    constexpr int NWCI = CS / WCI;
    static_assert(PPT >= 1 && WCI >= 4 && WCI <= 8 && WCI % 4 == 0 && CIN % CS == 0, "tile shapes");
    // an activation input and a tapped layer below (a_in, grad_tap) are compiled into the 64-input-channel layers only: the classifiers
    // need no other, and the 128 x 128 layer, at its 128-register cap, spills more with them
    constexpr bool EX = CIN == 64 && !WIDE;
    extern __shared__ __align__(16) float csm[];
    float *sW = csm;                                   // [COUT][CS]
    float *sDz = sW + COUT * CS;                       // [TP][LDZ]
    float *sA = sDz + kCbTP * LDZ;                     // [TP][LDA]   a_{l-1} = relu(BN(z_{l-1})), this CTA's channels
    float *sV = sA + kCbTP * LDA;                      // per-channel vectors: coef, m1, m2, mean, invstd [COUT] | sc_in, sh_in, mean_in, invstd_in [CS]
    float *vCoef = sV, *vM1 = sV + COUT, *vM2 = sV + 2 * COUT, *vMean = sV + 3 * COUT, *vInv = sV + 4 * COUT;
    float *vSc = sV + 5 * COUT, *vSh = vSc + CS, *vMeanI = vSc + 2 * CS, *vInvI = vSc + 3 * CS;
    const int tid = threadIdx.x;
    const int c0 = CS == CIN ? 0 : (int)blockIdx.y * CS;   // first input channel of this CTA
    const bool lead = CS == CIN || blockIdx.y == 0;         // writes what every CTA of a point range computes alike (bias, BN grads)
    const int CW = WIDE ? Q.cw : COUT;                      // the layer's output channels (row stride of z, pstar, gval)
    const int co0 = WIDE ? (int)blockIdx.z * COUT : 0;      // first output channel of this CTA's slice
    const int nco = WIDE ? min(COUT, CW - co0) : COUT;      // ... and how many it has (a multiple of 4); dz is 0 beyond
    const double cnt = (double)Q.P;
    for (int c = tid; c < COUT; c += kCbThreads) {
        if (WIDE && c >= nco) { vMean[c] = 0.f; vInv[c] = 0.f; vCoef[c] = 0.f; vM1[c] = 0.f; vM2[c] = 0.f; continue; }
        const int cg = co0 + c;
        const double m = Q.stats[cg] / cnt;
        double v = Q.stats[CW + cg] / cnt - m * m;
        if (v < 0) v = 0;
        const float invstd = 1.0f / sqrtf((float)v + Q.eps);
        vMean[c] = (float)m; vInv[c] = invstd;
        vCoef[c] = Q.gamma[cg] * invstd;
        vM1[c] = (float)(Q.s12[cg] / cnt); vM2[c] = (float)(Q.s12[CW + cg] / cnt);
        if (blockIdx.x == 0 && lead) { if (Q.g_gamma) Q.g_gamma[cg] = (float)Q.s12[CW + cg]; if (Q.g_beta) Q.g_beta[cg] = (float)Q.s12[cg]; }
    }
    for (int c = (EX && Q.a_in) ? CS : tid; c < CS; c += kCbThreads) {
        const double m = Q.stats_in[c0 + c] / cnt;
        double v = Q.stats_in[CIN + c0 + c] / cnt - m * m;
        if (v < 0) v = 0;
        const float invstd = 1.0f / sqrtf((float)v + Q.eps_in);
        const float sc = Q.gamma_in[c0 + c] * invstd;
        vSc[c] = sc; vSh[c] = Q.beta_in[c0 + c] - (float)m * sc; vMeanI[c] = (float)m; vInvI[c] = invstd;
    }
    for (int e = tid; e < COUT * CS / 4; e += kCbThreads) {
        const int r = e / (CS / 4), k4 = (e - r * (CS / 4)) * 4;
        const size_t src = CS == CIN ? (size_t)e * 4 : (size_t)(co0 + r) * CIN + c0 + k4;
        reinterpret_cast<float4 *>(sW)[e] = (WIDE && r >= nco) ? make_float4(0.f, 0.f, 0.f, 0.f)
                                                                : __ldg(reinterpret_cast<const float4 *>(Q.weight + src));
    }

    // dgrad mapping: thread -> (point block pb, input-channel block cb)
    const int cb = tid % NCB, pb = tid / NCB;          // pb in [0, TP / PPT)
    // wgrad mapping: thread -> (cob, cib)
    const int cib = tid % NWCI, cob = tid / NWCI;
    float wacc[WCO][WCI];
    float bacc[WCO];
#pragma unroll
    for (int i = 0; i < WCO; i++) { bacc[i] = 0.f;
#pragma unroll
        for (int j = 0; j < WCI; j++) wacc[i][j] = 0.f; }
    float s1acc[8], s2acc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) { s1acc[j] = 0.f; s2acc[j] = 0.f; }

    const long long ntiles = (Q.P + kCbTP - 1) / kCbTP;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const long long p0 = t * kCbTP;
        __syncthreads();   // previous tile's consumers are done (and the per-channel vectors / weights are staged)
        // ---- prologue: dz tile (BatchNorm backward on load) and the layer-below activation tile
        for (int e = tid; e < kCbTP * COUT / 4; e += kCbThreads) {
            const int p = e / (COUT / 4), c4 = (e - p * (COUT / 4)) * 4;
            const long long gp = p0 + p;
            float4 dz4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (gp < Q.P && (!WIDE || c4 < nco)) {
                const float4 z4 = __ldg(reinterpret_cast<const float4 *>(Q.z + gp * CW + co0 + c4));
                float4 dy4;
                if (SPARSE) {
                    const int cloud = (int)(gp / Q.n);
                    const int4 ps = __ldg(reinterpret_cast<const int4 *>(Q.pstar + (size_t)cloud * CW + co0 + c4));
                    const float4 gv = __ldg(reinterpret_cast<const float4 *>(Q.gval + (size_t)cloud * CW + co0 + c4));
                    dy4.x = ps.x == (int)gp ? gv.x : 0.f; dy4.y = ps.y == (int)gp ? gv.y : 0.f;
                    dy4.z = ps.z == (int)gp ? gv.z : 0.f; dy4.w = ps.w == (int)gp ? gv.w : 0.f;
                } else {
                    dy4 = __ldg(reinterpret_cast<const float4 *>(Q.dy + gp * COUT + c4));
                }
                dz4.x = vCoef[c4 + 0] * (dy4.x - vM1[c4 + 0] - (z4.x - vMean[c4 + 0]) * vInv[c4 + 0] * vM2[c4 + 0]);
                dz4.y = vCoef[c4 + 1] * (dy4.y - vM1[c4 + 1] - (z4.y - vMean[c4 + 1]) * vInv[c4 + 1] * vM2[c4 + 1]);
                dz4.z = vCoef[c4 + 2] * (dy4.z - vM1[c4 + 2] - (z4.z - vMean[c4 + 2]) * vInv[c4 + 2] * vM2[c4 + 2]);
                dz4.w = vCoef[c4 + 3] * (dy4.w - vM1[c4 + 3] - (z4.w - vMean[c4 + 3]) * vInv[c4 + 3] * vM2[c4 + 3]);
            }
            *reinterpret_cast<float4 *>(sDz + p * LDZ + c4) = dz4;
        }
        for (int e = tid; e < kCbTP * CS / 4; e += kCbThreads) {
            const int p = e / (CS / 4), c4 = (e - p * (CS / 4)) * 4;
            const long long gp = p0 + p;
            float4 a4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (EX && gp < Q.P && Q.a_in) {
                a4 = __ldg(reinterpret_cast<const float4 *>(Q.a_in + gp * CIN + c0 + c4));
            } else if (gp < Q.P) {
                const float4 z4 = __ldg(reinterpret_cast<const float4 *>(Q.z_in + gp * CIN + c0 + c4));
                a4.x = fmaxf(fmaf(vSc[c4 + 0], z4.x, vSh[c4 + 0]), 0.f); a4.y = fmaxf(fmaf(vSc[c4 + 1], z4.y, vSh[c4 + 1]), 0.f);
                a4.z = fmaxf(fmaf(vSc[c4 + 2], z4.z, vSh[c4 + 2]), 0.f); a4.w = fmaxf(fmaf(vSc[c4 + 3], z4.w, vSh[c4 + 3]), 0.f);
            }
            *reinterpret_cast<float4 *>(sA + p * LDA + c4) = a4;
        }
        __syncthreads();
        // ---- dgrad: out[p][ci] = sum_co dz[p][co] W[co][ci], PPT points x 8 input channels per thread, co in steps of 4
        {
            float o[PPT][8];
#pragma unroll
            for (int i = 0; i < PPT; i++)
#pragma unroll
                for (int j = 0; j < 8; j++) o[i][j] = 0.f;
#pragma unroll 2
            for (int co = 0; co < COUT; co += 4) {
                float4 d[PPT];
#pragma unroll
                for (int i = 0; i < PPT; i++) d[i] = *reinterpret_cast<const float4 *>(sDz + (pb * PPT + i) * LDZ + co);
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    // this thread's 8 input channels are [4 cb, 4 cb + 4) and [CS/2 + 4 cb, CS/2 + 4 cb + 4): a quarter warp's 16-byte reads
                    // are then 128 contiguous bytes (an 8-wide block per thread would put lanes cb and cb + 4 on the same banks)
                    const float4 w0 = *reinterpret_cast<const float4 *>(sW + (co + q) * CS + cb * 4);
                    const float4 w1 = *reinterpret_cast<const float4 *>(sW + (co + q) * CS + CS / 2 + cb * 4);
#pragma unroll
                    for (int i = 0; i < PPT; i++) {
                        const float dv = q == 0 ? d[i].x : (q == 1 ? d[i].y : (q == 2 ? d[i].z : d[i].w));
                        o[i][0] = fmaf(dv, w0.x, o[i][0]); o[i][1] = fmaf(dv, w0.y, o[i][1]); o[i][2] = fmaf(dv, w0.z, o[i][2]); o[i][3] = fmaf(dv, w0.w, o[i][3]);
                        o[i][4] = fmaf(dv, w1.x, o[i][4]); o[i][5] = fmaf(dv, w1.y, o[i][5]); o[i][6] = fmaf(dv, w1.z, o[i][6]); o[i][7] = fmaf(dv, w1.w, o[i][7]);
                    }
                }
            }
            // epilogue: ReLU mask of the layer below, store, and its BatchNorm sums (WIDE: the slice's unmasked share, combined later)
#pragma unroll
            for (int i = 0; i < PPT; i++) {
                const long long gp = p0 + pb * PPT + i;
                if (WIDE && gp < Q.P) {
                    float *dp = Q.dpart + ((size_t)blockIdx.z * Q.P + gp) * CIN + c0;
                    *reinterpret_cast<float4 *>(dp + cb * 4) = make_float4(o[i][0], o[i][1], o[i][2], o[i][3]);
                    *reinterpret_cast<float4 *>(dp + CS / 2 + cb * 4) = make_float4(o[i][4], o[i][5], o[i][6], o[i][7]);
                } else if (EX && gp < Q.P && Q.a_in) {   // the gradient of the stack's input (if wanted): no ReLU in front of layer 1
                    if (Q.dy_in) {
                        *reinterpret_cast<float4 *>(Q.dy_in + gp * CIN + c0 + cb * 4) = make_float4(o[i][0], o[i][1], o[i][2], o[i][3]);
                        *reinterpret_cast<float4 *>(Q.dy_in + gp * CIN + c0 + CS / 2 + cb * 4) = make_float4(o[i][4], o[i][5], o[i][6], o[i][7]);
                    }
                } else if (gp < Q.P) {
                    if (EX && Q.grad_tap) {   // the tapped activation's own gradient joins the one through this layer
                        const float4 ta = __ldg(reinterpret_cast<const float4 *>(Q.grad_tap + gp * CIN + c0 + cb * 4));
                        const float4 tb = __ldg(reinterpret_cast<const float4 *>(Q.grad_tap + gp * CIN + c0 + CS / 2 + cb * 4));
                        o[i][0] += ta.x; o[i][1] += ta.y; o[i][2] += ta.z; o[i][3] += ta.w;
                        o[i][4] += tb.x; o[i][5] += tb.y; o[i][6] += tb.z; o[i][7] += tb.w;
                    }
                    const float4 za = __ldg(reinterpret_cast<const float4 *>(Q.z_in + gp * CIN + c0 + cb * 4));
                    const float4 zb = __ldg(reinterpret_cast<const float4 *>(Q.z_in + gp * CIN + c0 + CS / 2 + cb * 4));
                    const float zv[8] = {za.x, za.y, za.z, za.w, zb.x, zb.y, zb.z, zb.w};
                    float dyv[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const int c = (j < 4 ? 0 : CS / 2) + cb * 4 + (j & 3);
                        const float y = fmaf(vSc[c], zv[j], vSh[c]);
                        const float zh = (zv[j] - vMeanI[c]) * vInvI[c];
                        dyv[j] = y > 0.f ? o[i][j] : 0.f;
                        s1acc[j] += dyv[j];
                        s2acc[j] = fmaf(dyv[j], zh, s2acc[j]);
                    }
                    *reinterpret_cast<float4 *>(Q.dy_in + gp * CIN + c0 + cb * 4) = make_float4(dyv[0], dyv[1], dyv[2], dyv[3]);
                    *reinterpret_cast<float4 *>(Q.dy_in + gp * CIN + c0 + CS / 2 + cb * 4) = make_float4(dyv[4], dyv[5], dyv[6], dyv[7]);
                }
            }
        }
        // ---- wgrad: dW[co][ci] += sum_p dz[p][co] a[p][ci]
#pragma unroll 4
        for (int p = 0; p < kCbTP; p++) {
            float dzr[WCO], ar[WCI];
#pragma unroll
            for (int i = 0; i < WCO; i += 4) {
                const float4 t4 = *reinterpret_cast<const float4 *>(sDz + p * LDZ + cob * WCO + i);
                dzr[i] = t4.x; dzr[i + 1] = t4.y; dzr[i + 2] = t4.z; dzr[i + 3] = t4.w;
            }
#pragma unroll
            for (int j = 0; j < WCI; j += 4) {   // columns [4 cib, +4) (and [CS/2 + 4 cib, +4) when WCI = 8): conflict-free 16-byte reads
                const float4 t4 = *reinterpret_cast<const float4 *>(sA + p * LDA + (j ? CS / 2 : 0) + cib * 4);
                ar[j] = t4.x; ar[j + 1] = t4.y; ar[j + 2] = t4.z; ar[j + 3] = t4.w;
            }
#pragma unroll
            for (int i = 0; i < WCO; i++) {
                if (cib == 0) bacc[i] += dzr[i];
#pragma unroll
                for (int j = 0; j < WCI; j++) wacc[i][j] = fmaf(dzr[i], ar[j], wacc[i][j]);
            }
        }
    }
    // ---- per-CTA results: weight / bias partials (plain stores, reduced in fixed order later); BatchNorm sums of the layer below.
    // The partial of point range blockIdx.x is one [COUT][CIN] + [COUT] block; the CTAs of a split layer fill disjoint columns of it.
    // WIDE: the [CW][CIN] + [CW] block of all slices, this CTA's rows co0 + [0, nco).
    float *part = Q.part + (size_t)blockIdx.x * ((size_t)CW * CIN + CW);
#pragma unroll
    for (int i = 0; i < WCO; i++) {
        if (WIDE && cob * WCO + i >= nco) continue;
        const int co = co0 + cob * WCO + i;
#pragma unroll
        for (int j = 0; j < WCI; j += 4)
            *reinterpret_cast<float4 *>(part + (size_t)co * CIN + c0 + (j ? CS / 2 : 0) + cib * 4) = make_float4(wacc[i][j], wacc[i][j + 1], wacc[i][j + 2], wacc[i][j + 3]);
        if (cib == 0 && lead) part[(size_t)CW * CIN + co] = bacc[i];
    }
    if (WIDE || (EX && Q.a_in)) return;   // (layer 1 reading an activation: no layer below)
    __syncthreads();
    float *sR = sDz;  // [TP/PPT point blocks][2][CS] fixed-order combine of the per-thread sums
    constexpr int NPB = kCbTP / PPT;
    static_assert(NPB * 2 * CS <= kCbTP * LDZ + kCbTP * LDA, "reduction scratch");
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int c = (j < 4 ? 0 : CS / 2) + cb * 4 + (j & 3);
        sR[(pb * 2 + 0) * CS + c] = s1acc[j]; sR[(pb * 2 + 1) * CS + c] = s2acc[j];
    }
    __syncthreads();
    for (int e = tid; e < 2 * CS; e += kCbThreads) {
        const int which = e / CS, c = e - which * CS;
        float s = 0.f;
        for (int k = 0; k < NPB; k++) s += sR[(k * 2 + which) * CS + c];
        atomicAdd(Q.s12_in + which * CIN + c0 + c, (double)s);
    }
}

// The wide last layer's dgrad: dy_in = (sum over its output slices of dpart, in slice order) * [y_in > 0], and the layer below's BatchNorm
// sums, each with the expressions of conv_bwd_kernel's epilogue.  Thread = (row r of R = 256 / c_in, channel c); the CTAs stride over the
// points, and each adds its per-channel sums (fixed order inside the CTA) into s12_in.
struct DgradCombineParams {
    long long P; int c_in, nslices;
    const float *dpart;                      // [nslices][P][c_in]
    const float *z_in; const double *stats_in; const float *gamma_in, *beta_in; float eps_in;
    float *dy_in; double *s12_in;
};
__global__ void __launch_bounds__(256) dgrad_combine_kernel(const __grid_constant__ DgradCombineParams Q)
{
    __shared__ float sR[2][256];
    const int tid = threadIdx.x, C = Q.c_in, R = 256 / C, c = tid % C, r = tid / C;
    const double cnt = (double)Q.P;
    const double m = Q.stats_in[c] / cnt;
    double v = Q.stats_in[C + c] / cnt - m * m;
    if (v < 0) v = 0;
    const float invstd = 1.0f / sqrtf((float)v + Q.eps_in);
    const float sc = Q.gamma_in[c] * invstd, sh = Q.beta_in[c] - (float)m * sc, mean = (float)m;
    float s1 = 0.f, s2 = 0.f;
    for (long long p = (long long)blockIdx.x * R + r; p < Q.P; p += (long long)gridDim.x * R) {
        float d = 0.f;
        for (int k = 0; k < Q.nslices; k++) d += __ldcs(Q.dpart + ((size_t)k * Q.P + p) * C + c);
        const float zv = __ldg(Q.z_in + p * C + c);
        const float y = fmaf(sc, zv, sh);
        const float zh = (zv - mean) * invstd;
        const float dy = y > 0.f ? d : 0.f;
        Q.dy_in[p * C + c] = dy;
        s1 += dy;
        s2 = fmaf(dy, zh, s2);
    }
    sR[0][tid] = s1; sR[1][tid] = s2;
    __syncthreads();
    if (r == 0) {
        for (int k = 1; k < R; k++) { s1 += sR[0][k * C + c]; s2 += sR[1][k * C + c]; }
        atomicAdd(Q.s12_in + c, (double)s1);
        atomicAdd(Q.s12_in + C + c, (double)s2);
    }
}

// conv1 (3 -> C): dW = dz^T x, db = sum dz; lanes over channels (C <= 128: up to 4 per lane), warps over points
struct Conv1BwdParams {
    long long P; int n, C, layout;
    const float *x, *z, *dy; const double *stats, *s12; const float *gamma; float eps;
    float *part;                  // [grid][C*3 + C]
    float *g_gamma, *g_beta;
    const float *weight;          // (C, 3)
    float *grad_x;                // x's shape and layout, or null: grad_x[p] = dz_p W, per point one warp's sum over its channel lanes
};
__global__ void __launch_bounds__(256) conv1_bwd_kernel(const __grid_constant__ Conv1BwdParams Q)
{
    __shared__ float sRed[8][128 * 4];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int C = Q.C;
    const double cnt = (double)Q.P;
    float coef[4], m1[4], m2[4], mean[4], inv[4], acc[4][4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int c = lane + 32 * u;
        coef[u] = m1[u] = m2[u] = mean[u] = 0.f; inv[u] = 1.f;
#pragma unroll
        for (int k = 0; k < 4; k++) acc[u][k] = 0.f;
        if (c < C) {
            const double m = Q.stats[c] / cnt;
            double v = Q.stats[C + c] / cnt - m * m;
            if (v < 0) v = 0;
            inv[u] = 1.0f / sqrtf((float)v + Q.eps); mean[u] = (float)m; coef[u] = Q.gamma[c] * inv[u];
            m1[u] = (float)(Q.s12[c] / cnt); m2[u] = (float)(Q.s12[C + c] / cnt);
            if (blockIdx.x == 0 && warp == 0) { if (Q.g_gamma) Q.g_gamma[c] = (float)Q.s12[C + c]; if (Q.g_beta) Q.g_beta[c] = (float)Q.s12[c]; }
        }
    }
    // 4 of this warp's points per pass: their loads are issued together (the loop is a chain of HBM round trips otherwise), the
    // accumulation stays in point order
    const long long pstride = (long long)gridDim.x * 8;
    for (long long pb = (long long)blockIdx.x * 8 + warp; pb < Q.P; pb += 4 * pstride) {
        float xs[4][3], zs[4][4], ds[4][4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const long long p = pb + j * pstride;
            const bool in = p < Q.P;
            const long long pc = in ? p : 0;
            if (Q.layout == SNB200_BNC) { xs[j][0] = Q.x[pc * 3 + 0]; xs[j][1] = Q.x[pc * 3 + 1]; xs[j][2] = Q.x[pc * 3 + 2]; }
            else { const long long cl = pc / Q.n, pi = pc - cl * Q.n; xs[j][0] = Q.x[(cl * 3 + 0) * Q.n + pi]; xs[j][1] = Q.x[(cl * 3 + 1) * Q.n + pi]; xs[j][2] = Q.x[(cl * 3 + 2) * Q.n + pi]; }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int c = lane + 32 * u;
                const bool ok = in && c < C;
                zs[j][u] = ok ? __ldg(Q.z + pc * C + c) : 0.f;
                ds[j][u] = ok ? __ldg(Q.dy + pc * C + c) : 0.f;
            }
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const long long p = pb + j * pstride;
            if (p < Q.P) {   // (warp-uniform)
                float gx[3] = {0.f, 0.f, 0.f};
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    if (lane + 32 * u < C) {
                        const float dz = coef[u] * (ds[j][u] - m1[u] - (zs[j][u] - mean[u]) * inv[u] * m2[u]);
                        acc[u][0] = fmaf(dz, xs[j][0], acc[u][0]); acc[u][1] = fmaf(dz, xs[j][1], acc[u][1]); acc[u][2] = fmaf(dz, xs[j][2], acc[u][2]); acc[u][3] += dz;
                        if (Q.grad_x) {
                            const float *w = Q.weight + (size_t)(lane + 32 * u) * 3;
                            gx[0] = fmaf(dz, __ldg(w), gx[0]); gx[1] = fmaf(dz, __ldg(w + 1), gx[1]); gx[2] = fmaf(dz, __ldg(w + 2), gx[2]);
                        }
                    }
                }
                if (Q.grad_x) {   // channel lanes in the butterfly's fixed order: every point's gradient is one warp's, stored once
#pragma unroll
                    for (int k = 0; k < 3; k++) gx[k] = warp_sum(gx[k]);
                    if (lane < 3) {
                        const float g = lane == 0 ? gx[0] : (lane == 1 ? gx[1] : gx[2]);
                        if (Q.layout == SNB200_BNC) Q.grad_x[p * 3 + lane] = g;
                        else { const long long cl = p / Q.n, pi = p - cl * Q.n; Q.grad_x[(cl * 3 + lane) * Q.n + pi] = g; }
                    }
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < 4; u++)
#pragma unroll
        for (int k = 0; k < 4; k++) sRed[warp][(lane + 32 * u) * 4 + k] = acc[u][k];
    __syncthreads();
    float *part = Q.part + (size_t)blockIdx.x * (C * 4);
    for (int e = tid; e < C * 4; e += 256) {
        float s = 0.f;
        for (int w = 0; w < 8; w++) s += sRed[w][e];
        const int c = e >> 2, k = e & 3;
        if (k < 3) part[c * 3 + k] = s; else part[C * 3 + c] = s;
    }
}

// gradient = sum over the launch's CTAs of its partial, in CTA order (bit-reproducible)
// blockIdx.y = job (conv layer).  A CTA = 32 columns x 8 part groups; a column is V consecutive gradient elements (V = 4: one 16-byte load
// per part), a group sums its contiguous share of the launch's CTA partials in CTA order with 8 loads in flight, the 8 group sums are then
// added in group order: a fixed order, so the gradients are bit-reproducible.  (One thread per element walking all ~300 parts, as in the
// first version, had 0.5 MB in flight on the whole GPU and ran at 10 % of HBM bandwidth.)
constexpr int kRpGroups = 8;
template <int V>
__device__ __forceinline__ void reduce_partials_body(const ReduceJob &J, float (*sAcc)[32][4])
{
    const int total = J.nw + J.nb, ncol = (total + V - 1) / V;
    const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
    const int per = (J.nparts + kRpGroups - 1) / kRpGroups;
    const int k0 = min(J.nparts, grp * per), k1 = min(J.nparts, k0 + per);
    for (int c0 = blockIdx.x * 32; c0 < ncol; c0 += gridDim.x * 32) {
        const int col = c0 + lane;
        float s[4] = {0.f, 0.f, 0.f, 0.f};
        if (col < ncol) {
            const float *p = J.part + (size_t)col * V;
            int k = k0;
            for (; k + 8 <= k1; k += 8) {
                float v[8][4];
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    if (V == 4) {
                        const float4 t = __ldcs(reinterpret_cast<const float4 *>(p + (size_t)(k + u) * total));
                        v[u][0] = t.x; v[u][1] = t.y; v[u][2] = t.z; v[u][3] = t.w;
                    } else {
                        v[u][0] = __ldcs(p + (size_t)(k + u) * total); v[u][1] = v[u][2] = v[u][3] = 0.f;
                    }
                }
#pragma unroll
                for (int u = 0; u < 8; u++)
#pragma unroll
                    for (int i = 0; i < V; i++) s[i] += v[u][i];
            }
            for (; k < k1; k++) {
                if (V == 4) {
                    const float4 t = __ldcs(reinterpret_cast<const float4 *>(p + (size_t)k * total));
                    s[0] += t.x; s[1] += t.y; s[2] += t.z; s[3] += t.w;
                } else {
                    s[0] += __ldcs(p + (size_t)k * total);
                }
            }
        }
        __syncthreads();   // (the previous column block's sums have been consumed)
#pragma unroll
        for (int i = 0; i < 4; i++) sAcc[grp][lane][i] = s[i];
        __syncthreads();
        if (grp == 0 && col < ncol) {
#pragma unroll
            for (int i = 0; i < V; i++) {
                float t = 0.f;
#pragma unroll
                for (int g = 0; g < kRpGroups; g++) t += sAcc[g][lane][i];
                const int e = col * V + i;
                if (e < J.nw) { if (J.g_weight) J.g_weight[e] = t; }
                else if (e < total && J.g_bias) J.g_bias[e - J.nw] = t;
            }
        }
    }
}
__global__ void __launch_bounds__(256) reduce_partials_kernel(const __grid_constant__ ReduceParams R)
{
    __shared__ float sAcc[kRpGroups][32][4];
    const ReduceJob &J = R.job[blockIdx.y];
    const int total = J.nw + J.nb;
    if ((total & 3) == 0 && (reinterpret_cast<uintptr_t>(J.part) & 15) == 0) reduce_partials_body<4>(J, sAcc);
    else reduce_partials_body<1>(J, sAcc);
}

// ------------------------------------------------------------------------------------------------------------------ host side
static size_t cb_smem_bytes(int cin, int cout) { return ((size_t)cout * cin + (size_t)kCbTP * (cout + 4) + (size_t)kCbTP * (cin + 4) + 5 * cout + 4 * cin) * sizeof(float); }
static int c1_grid(long long P) { return (int)min((long long)(4 * num_sms()), (P + 7) / 8); }
static int cb_grid(long long P) { return (int)min((long long)(2 * num_sms()), (P + kCbTP - 1) / kCbTP); }

// fc_bwd_kernel's shared memory, in floats: the layer's input [b][c_in + 1] and the CTA's 8 weight rows, plus for a layer below another
// one a chunk of `chunk` upper channels: their dz [b][chunk + 1] and each warp's slice of its upper-weight column [8][chunk]
constexpr size_t kFcbSmemFloats = 200 * 1024 / sizeof(float);
static size_t fcb_smem_floats(int b, int c_in, int chunk)
{
    return (size_t)b * (c_in + 1) + 8 * (size_t)c_in + (chunk ? (size_t)b * (chunk + 1) + 8 * (size_t)chunk : 0);
}
// Upper channels per chunk for a layer below one of c_up channels: all of them when they fit (one chunk), else the most that fit, rounded
// down to a multiple of 4 (the kernel's accumulators stay in step across chunks); 0 when not even 4 fit.
static int fcb_chunk(int b, int c_in, int c_up)
{
    const size_t base = fcb_smem_floats(b, c_in, 0) + b;
    const size_t fit = base < kFcbSmemFloats ? (kFcbSmemFloats - base) / (b + 8) : 0;
    return fit >= (size_t)c_up ? c_up : (int)(fit & ~(size_t)3);
}

// What both training paths' backward needs of the tables: BatchNorm + ReLU on every conv layer, 2 <= b <= 64 (an FC warp holds the
// batch), conv1 at most 128 channels (conv1_bwd_kernel), fc1 at most 1024 output channels (pool_bwd_kernel), each FC layer's input and
// weight rows in shared memory next to at least one chunk of the layer above (any width: fc_bwd_kernel streams it).  With fc1's input
// the pooled feature, that caps the batch at 41 clouds for a 1024-channel last conv layer.
static bool backward_tables_supported(int b, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc)
{
    if (b > kFcbMaxRows || b < 2 || conv[0].c_out > 128) return false;
    for (int l = 0; l < nconv; l++) if (!conv[l].bn_weight || !conv[l].relu) return false;
    for (int l = 0; l < nfc; l++) {
        if (fc[l].c_in > 1024 || fcb_smem_floats(b, fc[l].c_in, 0) > kFcbSmemFloats) return false;
        if (l + 1 < nfc && fcb_chunk(b, fc[l].c_in, fc[l + 1].c_out) == 0) return false;
    }
    return fc[0].c_out <= 1024;
}

// conv layers 2.. that conv_bwd_kernel is instantiated for; `wide` adds the 256-channel pairs (input channels split over grid.y)
static bool conv_bwd_pair_supported(int ci, int co, bool wide)
{
    if ((ci == 64 && co == 64) || (ci == 64 && co == 128) || (ci == 128 && co == 128)) return true;
    return wide && ((ci == 128 && co == 256) || (ci == 256 && co == 128));
}

// The last layer 128 -> C that runs as output slices (conv_bwd_kernel<..., WIDE>): C a multiple of 64 above 128, up to 1024 (256 has a
// pair of its own).
constexpr int kCbWideSlice = 256;
static bool conv_bwd_wide_last(int ci, int co) { return ci == 128 && co > 128 && co != 256 && co % 64 == 0 && co <= 1024; }
static int cb_wide_slices(int co) { return (co + kCbWideSlice - 1) / kCbWideSlice; }
// point ranges of a wide layer: cb_grid's CTAs shared among the output slices, so its weight-gradient partials stay as large as a
// 256-channel layer's (a 128 -> 1024 layer over cb_grid point ranges would need 139 MB of them)
static int cb_wide_grid(long long P, int co) { return (int)min((long long)max(1, 2 * num_sms() / cb_wide_slices(co)), (P + kCbTP - 1) / kCbTP); }
static int layer_grid(long long P, int nconv, const snb200_layer *conv, int l, bool act_input)
{
    if (l == 0 && !act_input) return c1_grid(P);
    return (l == nconv - 1 && conv_bwd_wide_last(conv[l].c_in, conv[l].c_out)) ? cb_wide_grid(P, conv[l].c_out) : cb_grid(P);
}

bool generator_backward_supported(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc)
{
    if (!conv_stack_supported(b, n, nconv, conv) || !backward_tables_supported(b, nconv, conv, nfc, fc) || conv[nconv - 1].c_out > 128) return false;
    for (int l = 1; l < nconv; l++) if (!conv_bwd_pair_supported(conv[l].c_in, conv[l].c_out, false)) return false;
    for (int l = 0; l < nfc; l++) if ((fc[l].bn_weight != nullptr) != (fc[l].relu != 0)) return false;
    return true;
}

// The per-layer path: the forward is the tensor-core layer kernels (any batch of points), so only the backward kernels bound the shapes.
// An FC layer may have BatchNorm and ReLU in any combination, except that the last one has no ReLU: its ReLU mask would have to come
// from `out`, which the backward does not receive.
bool generator_layers_backward_supported(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc)
{
    return generator_layers_ex_supported(b, n, 0, nconv, conv, nfc, fc, -1, nullptr);
}

// act_input: layer 1 is one of conv_bwd_kernel's pairs with 64 input channels.  tap: a hidden layer whose gradient the next layer's
// conv_bwd_kernel epilogue completes, one with 64 input channels (see EX in the kernel).  Dropout on any FC input but fc1's.
bool generator_layers_ex_supported(int b, int n, int act_input, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc, int tap,
                                   const float *const *fc_dropout)
{
    if (n < 1 || nconv < 2) return false;
    if (act_input ? conv[0].c_in != 64 || !conv_bwd_pair_supported(64, conv[0].c_out, true) : (conv[0].c_in != 3 || (conv[0].c_out != 64 && conv[0].c_out != 128)))
        return false;
    if (!backward_tables_supported(b, nconv, conv, nfc, fc) || fc[nfc - 1].relu) return false;
    bool wide_last = false;
    for (int l = 1; l < nconv; l++) {
        wide_last = l == nconv - 1 && conv_bwd_wide_last(conv[l].c_in, conv[l].c_out);
        if (!wide_last && !conv_bwd_pair_supported(conv[l].c_in, conv[l].c_out, true)) return false;
    }
    if (tap < -1 || tap > nconv - 2 || (tap >= 0 && (conv[tap].c_out != 64 || (tap == nconv - 2 && wide_last)))) return false;
    return !(fc_dropout && fc_dropout[0]);
}

struct BwdWorkspace {
    float *dy[2]; double *s12[SNB200_MAX_CONV_LAYERS]; char *s12_base; size_t s12_bytes;
    int *pstar; float *gval; float *dzfc[SNB200_MAX_FC_LAYERS]; float *part[SNB200_MAX_CONV_LAYERS];
    float *dpart;   // a wide last layer's dgrad per output slice (null, 0 bytes, otherwise)
    size_t total;
};
static BwdWorkspace carve_bwd_ws(void *base, int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc, bool act_input)
{
    BwdWorkspace W;
    WsCarver c(base);
    const long long P = (long long)b * n;
    int maxc = 8;
    for (int l = 0; l + 1 < nconv; l++) maxc = max(maxc, conv[l].c_out);
    W.dy[0] = c.take<float>((size_t)P * maxc);
    W.dy[1] = c.take<float>((size_t)P * maxc);
    const size_t s12_off = c.off;
    for (int l = 0; l < nconv; l++) W.s12[l] = c.take<double>((size_t)2 * conv[l].c_out);
    W.s12_base = reinterpret_cast<char *>(W.s12[0]);
    W.s12_bytes = c.off - s12_off;
    const int C = conv[nconv - 1].c_out;
    W.pstar = c.take<int>((size_t)b * C);
    W.gval = c.take<float>((size_t)b * C);
    for (int l = 0; l < nfc; l++) W.dzfc[l] = c.take<float>((size_t)b * fc[l].c_out);
    for (int l = 0; l < nconv; l++)
        W.part[l] = c.take<float>((size_t)layer_grid(P, nconv, conv, l, act_input) * ((size_t)conv[l].c_out * conv[l].c_in + conv[l].c_out));
    const snb200_layer &LL = conv[nconv - 1];
    const bool wide = nconv > 1 && conv_bwd_wide_last(LL.c_in, LL.c_out);
    W.dpart = wide ? c.take<float>((size_t)cb_wide_slices(LL.c_out) * P * LL.c_in) : nullptr;
    W.total = c.off;
    return W;
}
size_t generator_backward_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc, bool act_input)
{
    return carve_bwd_ws(nullptr, b, n, nconv, conv, nfc, fc, act_input).total;
}

// the wide last layer: output slices over grid.z, then their dgrad summed, masked and reduced into the layer below's sums
static int launch_conv_bwd_wide(const ConvBwdParams &Q, int grid, cudaStream_t stream)
{
    constexpr int CIN = 128, CS = 64;
    const size_t smem = cb_smem_bytes(CS, kCbWideSlice);
    static PerDeviceOnce once;
    if (once.first()) cudaFuncSetAttribute(conv_bwd_kernel<CIN, CS, kCbWideSlice, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int ns = cb_wide_slices(Q.cw);
    conv_bwd_kernel<CIN, CS, kCbWideSlice, true, true><<<dim3(grid, CIN / CS, ns), kCbThreads, smem, stream>>>(Q);
    if (int rc = check_launch("generator backward: wide conv layer")) return rc;
    DgradCombineParams D;
    D.P = Q.P; D.c_in = CIN; D.nslices = ns; D.dpart = Q.dpart;
    D.z_in = Q.z_in; D.stats_in = Q.stats_in; D.gamma_in = Q.gamma_in; D.beta_in = Q.beta_in; D.eps_in = Q.eps_in;
    D.dy_in = Q.dy_in; D.s12_in = Q.s12_in;
    const long long rows = (Q.P + 1) / 2;   // 256 / CIN point rows per CTA and pass
    dgrad_combine_kernel<<<(int)min((long long)(2 * num_sms()), rows), 256, 0, stream>>>(D);
    return check_launch("generator backward: wide conv layer combine");
}

template <int CIN, int CS, int COUT>
static int launch_conv_bwd(const ConvBwdParams &Q, bool sparse, int grid, cudaStream_t stream)
{
    const size_t smem = cb_smem_bytes(CS, COUT);
    static PerDeviceOnce once;
    if (once.first()) {
        cudaFuncSetAttribute(conv_bwd_kernel<CIN, CS, COUT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        cudaFuncSetAttribute(conv_bwd_kernel<CIN, CS, COUT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    }
    const dim3 g(grid, CIN / CS);
    if (sparse) conv_bwd_kernel<CIN, CS, COUT, true><<<g, kCbThreads, smem, stream>>>(Q);
    else conv_bwd_kernel<CIN, CS, COUT, false><<<g, kCbThreads, smem, stream>>>(Q);
    return check_launch("generator backward: conv layer");
}

int launch_generator_backward(int b, int n, int layout, const float *x, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc,
                              float *const *zsave, void *fwd_workspace, const float *grad_out, int out_transpose_inner,
                              const snb200_layer_grad *gconv, const snb200_layer_grad *gfc, void *workspace, cudaStream_t stream, const GenEx *ex)
{
    const long long P = (long long)b * n;
    const bool act_input = ex && ex->act_input;
    BwdWorkspace W = carve_bwd_ws(workspace, b, n, nconv, conv, nfc, fc, act_input);
    GenWorkspaceView V = generator_workspace_view(fwd_workspace, b, n, nconv, conv, nfc, fc);
    cudaMemsetAsync(W.s12_base, 0, W.s12_bytes, stream);
    // ---- FC head, top down
    static PerDeviceOnce once_fc;
    if (once_fc.first()) cudaFuncSetAttribute(fc_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kFcbSmemFloats * sizeof(float)));
    for (int l = nfc - 1; l >= 0; l--) {
        FcBwdParams F;
        memset(&F, 0, sizeof(F));
        F.b = b; F.c_in = fc[l].c_in; F.c_out = fc[l].c_out; F.a_in = V.ll[l];
        F.a_out = (l + 1 < nfc && fc[l].relu) ? V.ll[l + 1] : nullptr;
        F.weight = fc[l].weight; F.bias = fc[l].bias; F.gamma = fc[l].bn_weight; F.beta = fc[l].bn_bias; F.eps = fc[l].bn_eps;
        F.has_bn = fc[l].bn_weight != nullptr; F.relu = fc[l].relu;
        if (l == nfc - 1) { F.grad_out = grad_out; F.out_inner = out_transpose_inner; }
        else {
            F.dz_up = W.dzfc[l + 1]; F.w_up = fc[l + 1].weight; F.c_up = fc[l + 1].c_out; F.u_chunk = fcb_chunk(b, F.c_in, F.c_up);
            F.mask = ex ? ex->fc_dropout[l + 1] : nullptr;
        }
        F.dz = W.dzfc[l];
        F.g_weight = gfc[l].weight; F.g_bias = gfc[l].bias; F.g_gamma = gfc[l].bn_weight; F.g_beta = gfc[l].bn_bias;
        const size_t smem = fcb_smem_floats(b, F.c_in, F.u_chunk) * sizeof(float);
        fc_bwd_kernel<<<(F.c_out + 7) / 8, kFcbThreads, smem, stream>>>(F);
        int rc = check_launch("generator backward: fc layer");
        if (rc) return rc;
    }
    // ---- max-pool
    const int L = nconv - 1, C = conv[L].c_out;
    {
        PoolBwdParams Q;
        memset(&Q, 0, sizeof(Q));
        Q.b = b; Q.n = n; Q.C = C; Q.z = zsave[L]; Q.stats = V.stats[L]; Q.gamma = conv[L].bn_weight; Q.beta = conv[L].bn_bias; Q.eps = conv[L].bn_eps;
        Q.has_bn = 1; Q.relu = conv[L].relu; Q.dz1 = W.dzfc[0]; Q.w1 = fc[0].weight; Q.c1 = fc[0].c_out;
        Q.pstar = W.pstar; Q.gval = W.gval; Q.s12 = W.s12[L];
        pool_bwd_kernel<<<dim3(b, (C + 127) / 128), 1024, 0, stream>>>(Q);
        int rc = check_launch("generator backward: pool");
        if (rc) return rc;
    }
    // ---- conv layers L .. 1 (.. 0 when layer 1 reads an activation)
    for (int l = L; l >= (act_input ? 0 : 1); l--) {
        const int grid = layer_grid(P, nconv, conv, l, act_input);
        ConvBwdParams Q;
        memset(&Q, 0, sizeof(Q));
        Q.P = P; Q.n = n; Q.z = zsave[l];
        const bool sparse = (l == L);
        if (sparse) { Q.pstar = W.pstar; Q.gval = W.gval; } else Q.dy = W.dy[l & 1];
        Q.stats = V.stats[l]; Q.s12 = W.s12[l]; Q.gamma = conv[l].bn_weight; Q.eps = conv[l].bn_eps; Q.weight = conv[l].weight;
        if (l == 0) { Q.a_in = x; Q.dy_in = ex->grad_in; }
        else {
            Q.z_in = zsave[l - 1]; Q.stats_in = V.stats[l - 1]; Q.gamma_in = conv[l - 1].bn_weight; Q.beta_in = conv[l - 1].bn_bias;
            Q.eps_in = conv[l - 1].bn_eps; Q.dy_in = W.dy[(l - 1) & 1]; Q.s12_in = W.s12[l - 1];
            Q.grad_tap = (ex && ex->tap == l - 1) ? ex->grad_tap : nullptr;
        }
        Q.part = W.part[l];
        Q.g_gamma = gconv[l].bn_weight; Q.g_beta = gconv[l].bn_bias;
        int rc;
        const int ci = conv[l].c_in, co = conv[l].c_out;
        if (l == L && conv_bwd_wide_last(ci, co)) { Q.cw = co; Q.dpart = W.dpart; rc = launch_conv_bwd_wide(Q, grid, stream); }
        else if (ci == 128 && co == 128) rc = launch_conv_bwd<128, 128, 128>(Q, sparse, grid, stream);
        else if (ci == 64 && co == 128) rc = launch_conv_bwd<64, 64, 128>(Q, sparse, grid, stream);
        else if (ci == 128 && co == 256) rc = launch_conv_bwd<128, 64, 256>(Q, sparse, grid, stream);
        else if (ci == 256 && co == 128) rc = launch_conv_bwd<256, 64, 128>(Q, sparse, grid, stream);
        else rc = launch_conv_bwd<64, 64, 64>(Q, sparse, grid, stream);
        if (rc) return rc;
    }
    // ---- conv1
    const int g1 = c1_grid(P);
    if (!act_input) {
        Conv1BwdParams Q;
        memset(&Q, 0, sizeof(Q));
        Q.P = P; Q.n = n; Q.C = conv[0].c_out; Q.layout = layout; Q.x = x; Q.z = zsave[0]; Q.dy = W.dy[0];
        Q.stats = V.stats[0]; Q.s12 = W.s12[0]; Q.gamma = conv[0].bn_weight; Q.eps = conv[0].bn_eps; Q.part = W.part[0];
        Q.g_gamma = gconv[0].bn_weight; Q.g_beta = gconv[0].bn_bias;
        Q.weight = conv[0].weight; Q.grad_x = ex ? ex->grad_in : nullptr;
        conv1_bwd_kernel<<<g1, 256, 0, stream>>>(Q);
        int rc = check_launch("generator backward: conv1");
        if (rc) return rc;
    }
    // ---- partials -> gradients
    ReduceParams R;
    memset(&R, 0, sizeof(R));
    R.njobs = nconv;
    for (int l = 0; l < nconv; l++) {
        R.job[l].part = W.part[l]; R.job[l].nparts = layer_grid(P, nconv, conv, l, act_input);
        R.job[l].nw = conv[l].c_out * conv[l].c_in; R.job[l].nb = conv[l].c_out;
        R.job[l].g_weight = gconv[l].weight; R.job[l].g_bias = gconv[l].bias;
    }
    return launch_reduce_partials(R, stream, "generator backward: reduce");
}

int launch_reduce_partials(const ReduceParams &R, cudaStream_t stream, const char *what)
{
    reduce_partials_kernel<<<dim3(128, R.njobs), 256, 0, stream>>>(R);   // 128 x 32 columns x 4 elements per sweep: one sweep up to 128 x 128
    return check_launch(what);
}

}  // namespace snb
