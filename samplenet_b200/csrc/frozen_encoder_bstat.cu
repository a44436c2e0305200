// frozen_encoder_bstat.cu -- a frozen PointNet encoder whose BatchNorms normalise with the batch statistics of each prefix, over every
// prefix of a cloud in one pass, and its gradient with respect to the points.
//
// This is what the reconstruction sampler trainers compute: the autoencoder is frozen (its parameters and moving averages never change), but
// its encoder runs under the training flag, so every conv layer normalises its input with the mean and biased variance of the batch it sees,
// and the progressive trainer rebuilds the encoder per prefix, so prefix p is normalised over its own B * s_p points.  Past layer 1 every
// prefix therefore has its own activations.
//
// Layout (PrefixPack, encoder_internal.cuh).  Each (prefix p, cloud b) pair is one segment of a packed buffer: rows
// [B sum_{q<p} pad(s_q) + b pad(s_p), + s_p), pad rounding up to the 128-row tile of the tensor-core layers.  No tile straddles two segments,
// so a tile belongs to exactly one group (prefix), and the group of prefix p is a contiguous range of tiles.  Padding rows are read as zeros
// by the layers and excluded from every statistic and pool.
//   forward   layer 1's per-tile (sum, sumsq) from bs_l1_partial_kernel; layers 2 .. L on tc_layer_kernel<..., GRP> (3xTF32 wgmma), whose
//             prologue normalises with the tile's group statistics and whose epilogue stores z and leaves per-tile partials; bs_reduce_kernel
//             turns each layer's partials into per-group (mean, biased variance) in double, adding a group's tiles in a fixed order relative
//             to its first tile; the last layer keeps the segment pool's per-tile records (the extreme of z in the direction of sign(gamma)
//             does not depend on the statistics), and bs_pool_kernel applies the group's scale and shift.
//   backward  dense, because the mean terms of a training-mode BatchNorm give every point of a group a share:
//               dz = scale_g (dy - mean_g dy - zhat mean_g(dy zhat)),   dy_{l-1} = (dz W_l) * [a_{l-1} > 0]
//             The top layer's dy is the pool's routed coefficient, so its group sums come from the routes alone (bs_top_sums_kernel).
//             bs_bwd_layer_kernel (fp32 CUDA cores) builds dz on load, multiplies by W_l, applies the layer below's mask (recomputed from
//             the saved z with the forward's expression) and leaves per-64-row partials of the layer below's sums, which bs_reduce_kernel
//             turns into group means.  Layer 1's dgrad lands in a packed (rows, 3) buffer; bs_gather_kernel sums, for every point, the
//             prefixes that hold it in ascending order (one writer per point).
// No floating-point atomics anywhere: repeat calls are bit-identical.  A group's reductions read only its own tiles, in an order relative
// to its first tile, so prefix s of a multi-prefix call equals a one-prefix call on x[:, :s] bit for bit.
//
// The autoencoder trained with the sampler (snb200_frozen_encoder_bstat_param_backward, _running_update) runs the same forward and the same
// backward chain, which gives grad_x bit for bit, and adds, layer by layer while the chain's buffers for that layer are live:
//   gamma, beta   bs_bn_grad_kernel: dbeta = sum_g sum_{rows in g} dy, dgamma = sum_g sum_{rows in g} dy zhat, from the group means the
//                 chain already reduced (times B s_g), groups ascending, in double;
//   W, b          bs_wgrad_partial_kernel: dW_l = sum_rows dz_l (x) a_{l-1}, db_l = sum_rows dz_l over one chunk of tiles per CTA (a 64 x 64
//                 output tile, 4 x 4 per thread, fp32 CUDA cores), dz built on load from dy (the top layer: the pool's routes) and the
//                 group statistics in bs_bwd_layer_kernel's expression, a_{l-1} recomputed from the saved z_{l-1} with the forward's
//                 relu(fmaf(z, scale, shift)) (a_0 = x); reduce_partials_kernel adds the chunks in a fixed order.  Padding rows enter nothing.
//   running stats bs_running_update_kernel, one launch after the forward: per prefix in ascending order, nn.BatchNorm1d's momentum update
//                 with the unbiased variance (bn_running_step, the generator head's arithmetic), and num_batches_tracked + num_prefix.
#include "encoder_internal.cuh"

namespace snb {

constexpr int kBsMaxN = 4096;
constexpr long long kBsMaxRows = 1ll << 22;   // packed rows: an element offset of a (rows, 256) activation stays below 2^31
constexpr int kBsBwdRows = 64;            // backward: rows per CTA (half a tile, so inside one segment)
constexpr int kBsBwdCo = 128;             // ... output channels staged per pass
constexpr int kBsBwdCi = 64;              // ... input channels per CTA (grid.y)
constexpr int kBsLdz = kBsBwdCo + 4;

// ---- forward, layer 1: per-tile (sum, sumsq) of z_1 = W_1 x + b_1 over the tile's rows, in the expression of tc_layer_kernel's prologue
__global__ void __launch_bounds__(256) bs_l1_partial_kernel(const __grid_constant__ PrefixPack S, const float *__restrict__ x,
                                                            const float *__restrict__ w1, const float *__restrict__ b1, int c1,
                                                            float *__restrict__ part)
{
    __shared__ float sX[kTcM * 3];
    int g, cloud, i0, rows;
    pack_tile(S, blockIdx.x, g, cloud, i0, rows);
    const float *xc = x + ((size_t)cloud * S.n + i0) * 3;
    for (int e = threadIdx.x; e < rows * 3; e += blockDim.x) sX[e] = xc[e];
    __syncthreads();
    for (int c = threadIdx.x; c < c1; c += blockDim.x) {
        const float wx = w1[c * 3 + 0], wy = w1[c * 3 + 1], wz = w1[c * 3 + 2], bc = b1[c];
        float sm = 0.f, ss = 0.f;
        for (int r = 0; r < rows; r++) {
            const float v = fmaf(wz, sX[r * 3 + 2], fmaf(wy, sX[r * 3 + 1], wx * sX[r * 3 + 0])) + bc;
            sm += v;
            ss = fmaf(v, v, ss);
        }
        part[(size_t)blockIdx.x * 2 * c1 + c] = sm;
        part[((size_t)blockIdx.x * 2 + 1) * c1 + c] = ss;
    }
}

// ---- per-group reduction of (units, 2, C) partials, `unit` rows each: one CTA per (group, 32 channels); warp w adds the group's units
// w, w + 8, ... (counted from the group's first unit) in double, and warp 0 adds the eight warps in order.  fwd: out (np, 2, C) = (mean,
// biased variance) over the group's B * s_p rows; otherwise (mean of the first sum, mean of the second).
__global__ void __launch_bounds__(256) bs_reduce_kernel(const __grid_constant__ PrefixPack S, const float *__restrict__ part, int C, int unit,
                                                        int fwd, double *__restrict__ out)
{
    __shared__ double sR[8][2][32];
    const int g = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, c = blockIdx.y * 32 + lane;
    const long long u0 = (long long)S.tile0[g] * kTcM / unit, u1 = (long long)S.tile0[g + 1] * kTcM / unit;
    double s1 = 0.0, s2 = 0.0;
    if (c < C)
        for (long long u = u0 + warp; u < u1; u += 8) {
            s1 += (double)part[(size_t)u * 2 * C + c];
            s2 += (double)part[((size_t)u * 2 + 1) * C + c];
        }
    sR[warp][0][lane] = s1;
    sR[warp][1][lane] = s2;
    __syncthreads();
    if (warp != 0 || c >= C) return;
    double t1 = 0.0, t2 = 0.0;
    for (int w = 0; w < 8; w++) { t1 += sR[w][0][lane]; t2 += sR[w][1][lane]; }
    const double cnt = (double)S.b * (double)S.sizes[g];
    const double m = t1 / cnt;
    double v = t2 / cnt;
    if (fwd) {
        v -= m * m;
        if (v < 0) v = 0;
    }
    out[(size_t)g * 2 * C + c] = m;
    out[((size_t)g * 2 + 1) * C + c] = v;
}

// ---- forward, pool: one thread per (group, cloud, channel) walks its segment's tile records, then applies the group's scale and shift
__global__ void __launch_bounds__(256) bs_pool_kernel(const __grid_constant__ PrefixPack S, int C, const float *__restrict__ gamma,
                                                      const float *__restrict__ beta, float eps, const double *__restrict__ stats,
                                                      const float *__restrict__ tile_val, const int *__restrict__ tile_idx,
                                                      float *__restrict__ pooled, int *__restrict__ route)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)S.np * S.b * C) return;
    const int c = (int)(e % C), j = (int)(e / C), g = j / S.b, cloud = j % S.b;
    const int tps = tc_tiles_per_cloud(S.sizes[g]), t0 = S.tile0[g] + cloud * tps;
    float run;
    int run_i;
    seg_tile_extreme(tile_val, tile_idx, C, c, t0, t0 + tps, run, run_i);
    const double *st = stats + (size_t)g * 2 * C;
    float sc, sh;
    bn_group_scale_shift(st[c], st[C + c], gamma[c], beta[c], eps, sc, sh);
    pooled[e] = fmaxf(fmaf(gamma[c] < 0.f ? -run : run, sc, sh), 0.f);
    route[e] = run_i;
}

// ---- backward, top layer: the group means of dy and dy * zhat, where dy is the pool's coefficient at its routed row.  One thread per
// (group, channel) adds the clouds in order.
__global__ void __launch_bounds__(256) bs_top_sums_kernel(const __grid_constant__ PrefixPack S, int C, const float *__restrict__ gamma,
                                                          const float *__restrict__ beta, float eps, const double *__restrict__ stats,
                                                          const float *__restrict__ z, const float *__restrict__ pooled,
                                                          const int *__restrict__ route, const float *__restrict__ grad_pooled,
                                                          double *__restrict__ m12)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= S.np * C) return;
    const int g = e / C, c = e % C;
    const double *st = stats + (size_t)g * 2 * C;
    const float mean = (float)st[c], invstd = 1.0f / sqrtf((float)st[C + c] + eps);
    double s1 = 0.0, s2 = 0.0;
    for (int cloud = 0; cloud < S.b; cloud++) {
        const size_t o = ((size_t)g * S.b + cloud) * C + c;
        if (!(pooled[o] > 0.f)) continue;
        const float d = grad_pooled[o];
        const float zh = (z[(size_t)pack_row(S, g, cloud, route[o]) * C + c] - mean) * invstd;
        s1 += (double)d;
        s2 += (double)(d * zh);
    }
    const double cnt = (double)S.b * (double)S.sizes[g];
    m12[(size_t)g * 2 * C + c] = s1 / cnt;
    m12[((size_t)g * 2 + 1) * C + c] = s2 / cnt;
}

struct BsBwdParams {
    PrefixPack S;
    int C, K;                                  // this layer's output and input channels
    const float *z;                            // (rows, C) raw output of this layer
    const double *stats, *m12;                 // (np, 2, C): (mean, var) and (mean dy, mean dy zhat) per group
    const float *gamma, *beta; float eps;
    const float *dy;                           // (rows, C) masked gradient of this layer's BatchNorm output, or null: the top layer's
    const float *pooled; const int *route; const float *grad_pooled;   // ... pool coefficients (np, b, C)
    const float *weight;                       // (C, K)
    const float *z_in;                         // (rows, K) raw output of the layer below, or null: layer 1 (dgrad to the points)
    const double *stats_in; const float *gamma_in, *beta_in; float eps_in;
    float *dy_in;                              // (rows, K): masked gradient of the layer below; layer 1: (rows, 3) gradient of the points
    float *part_in;                            // (rows / 64, 2, K): per-CTA sums of dy_in and dy_in * zhat_in (layers above 1)
};

// One CTA per (64 rows, 64 input channels).  dz is built on load, 128 output channels at a time, with W's matching rows; each thread keeps
// 2 rows x 8 input channels ([4 cb, +4) and [32 + 4 cb, +4)).  Partials of the layer below's sums: per thread over its 2 rows, then over
// the 32 row pairs in order.
__global__ void __launch_bounds__(256) bs_bwd_layer_kernel(const __grid_constant__ BsBwdParams Q)
{
    extern __shared__ __align__(16) float bsm[];
    float *sDz = bsm;                                // [64][kBsLdz]
    float *sW = sDz + kBsBwdRows * kBsLdz;           // [128][64]
    float *vCoef = sW + kBsBwdCo * kBsBwdCi, *vM1 = vCoef + kBsBwdCo, *vM2 = vM1 + kBsBwdCo, *vMean = vM2 + kBsBwdCo, *vInv = vMean + kBsBwdCo;
    float *vSc = vInv + kBsBwdCo, *vSh = vSc + kBsBwdCi, *vMeanI = vSh + kBsBwdCi, *vInvI = vMeanI + kBsBwdCi;
    const PrefixPack &S = Q.S;
    const int tid = threadIdx.x, C = Q.C, K = Q.K, ci0 = blockIdx.y * kBsBwdCi;
    const int unit = blockIdx.x, tile = unit / (kTcM / kBsBwdRows), r0 = (unit % (kTcM / kBsBwdRows)) * kBsBwdRows;
    int g, cloud, i0, trows;
    pack_tile(S, tile, g, cloud, i0, trows);
    const int nr = max(0, min(kBsBwdRows, trows - r0));
    const long long prow0 = (long long)tile * kTcM + r0;
    const size_t gb = ((size_t)g * S.b + cloud) * C;   // this segment's pool records
    if (Q.z_in) {
        const double *st = Q.stats_in + (size_t)g * 2 * K;
        for (int c = tid; c < kBsBwdCi; c += blockDim.x) {
            float sc = 0.f, sh = 0.f, mean = 0.f, inv = 0.f;
            if (ci0 + c < K) {
                bn_group_scale_shift(st[ci0 + c], st[K + ci0 + c], Q.gamma_in[ci0 + c], Q.beta_in[ci0 + c], Q.eps_in, sc, sh);
                mean = (float)st[ci0 + c];
                inv = 1.0f / sqrtf((float)st[K + ci0 + c] + Q.eps_in);
            }
            vSc[c] = sc; vSh[c] = sh; vMeanI[c] = mean; vInvI[c] = inv;
        }
    }
    const int rp = tid >> 3, cb = tid & 7;
    float o[2][8];
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) o[i][j] = 0.f;
    for (int co0 = 0; co0 < C && nr > 0; co0 += kBsBwdCo) {
        __syncthreads();   // the previous pass's readers are done
        for (int c = tid; c < kBsBwdCo; c += blockDim.x) {
            float coef = 0.f, m1 = 0.f, m2 = 0.f, mean = 0.f, inv = 0.f;
            if (co0 + c < C) {
                const int cg = co0 + c;
                const double *st = Q.stats + (size_t)g * 2 * C, *mm = Q.m12 + (size_t)g * 2 * C;
                mean = (float)st[cg];
                inv = 1.0f / sqrtf((float)st[C + cg] + Q.eps);
                coef = Q.gamma[cg] * inv;
                m1 = (float)mm[cg];
                m2 = (float)mm[C + cg];
            }
            vCoef[c] = coef; vM1[c] = m1; vM2[c] = m2; vMean[c] = mean; vInv[c] = inv;
        }
        for (int e = tid; e < kBsBwdCo * kBsBwdCi; e += blockDim.x) {
            const int co = e / kBsBwdCi, ci = e % kBsBwdCi;
            sW[e] = (co0 + co < C && ci0 + ci < K) ? __ldg(Q.weight + (size_t)(co0 + co) * K + ci0 + ci) : 0.f;
        }
        __syncthreads();
        for (int e = tid; e < kBsBwdRows * kBsBwdCo; e += blockDim.x) {
            const int r = e / kBsBwdCo, co = e % kBsBwdCo, cg = co0 + co;
            float dz = 0.f;
            if (r < nr && cg < C) {
                const float z = Q.z[(size_t)(prow0 + r) * C + cg];
                float dy;
                if (Q.dy) dy = Q.dy[(size_t)(prow0 + r) * C + cg];
                else dy = (Q.route[gb + cg] == i0 + r0 + r && Q.pooled[gb + cg] > 0.f) ? Q.grad_pooled[gb + cg] : 0.f;
                dz = vCoef[co] * (dy - vM1[co] - (z - vMean[co]) * vInv[co] * vM2[co]);
            }
            sDz[r * kBsLdz + co] = dz;
        }
        __syncthreads();
#pragma unroll 4
        for (int co = 0; co < kBsBwdCo; co++) {
            const float d0 = sDz[(2 * rp) * kBsLdz + co], d1 = sDz[(2 * rp + 1) * kBsLdz + co];
            const float4 w0 = *reinterpret_cast<const float4 *>(sW + co * kBsBwdCi + cb * 4);
            const float4 w1 = *reinterpret_cast<const float4 *>(sW + co * kBsBwdCi + 32 + cb * 4);
            const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
            for (int j = 0; j < 8; j++) {
                o[0][j] = fmaf(d0, wv[j], o[0][j]);
                o[1][j] = fmaf(d1, wv[j], o[1][j]);
            }
        }
    }
    if (!Q.z_in) {   // layer 1: the gradient of the points, rows of 3
        for (int i = 0; i < 2; i++) {
            const int r = 2 * rp + i;
            if (r >= nr || cb != 0) continue;
            for (int j = 0; j < K; j++) Q.dy_in[(size_t)(prow0 + r) * 3 + j] = o[i][j];
        }
        return;
    }
    float s1[8], s2[8];
#pragma unroll
    for (int j = 0; j < 8; j++) { s1[j] = 0.f; s2[j] = 0.f; }
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int r = 2 * rp + i;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int c = h * 32 + cb * 4;   // local input channel of o[i][4h .. 4h+3]
            if (r >= nr || ci0 + c >= K) continue;
            const size_t off = (size_t)(prow0 + r) * K + ci0 + c;
            const float4 z4 = __ldg(reinterpret_cast<const float4 *>(Q.z_in + off));
            const float zv[4] = {z4.x, z4.y, z4.z, z4.w};
            float dv[4];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const float zh = (zv[q] - vMeanI[c + q]) * vInvI[c + q];
                dv[q] = fmaf(zv[q], vSc[c + q], vSh[c + q]) > 0.f ? o[i][4 * h + q] : 0.f;
                s1[4 * h + q] += dv[q];
                s2[4 * h + q] = fmaf(dv[q], zh, s2[4 * h + q]);
            }
            *reinterpret_cast<float4 *>(Q.dy_in + off) = make_float4(dv[0], dv[1], dv[2], dv[3]);
        }
    }
    __syncthreads();
    float *sR = sDz;   // [32 row pairs][2][64]
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int c = (j < 4 ? 0 : 32) + cb * 4 + (j & 3);
        sR[(rp * 2 + 0) * kBsBwdCi + c] = s1[j];
        sR[(rp * 2 + 1) * kBsBwdCi + c] = s2[j];
    }
    __syncthreads();
    if (tid < 2 * kBsBwdCi) {
        const int which = tid / kBsBwdCi, c = tid % kBsBwdCi;
        float s = 0.f;
        for (int k = 0; k < kBsBwdRows / 2; k++) s += sR[(k * 2 + which) * kBsBwdCi + c];
        if (ci0 + c < K) Q.part_in[((size_t)unit * 2 + which) * K + ci0 + c] = s;
    }
}

// ---- backward, last step: grad_x[cloud, i] = sum over the prefixes holding point i, ascending, of the packed gradient rows
__global__ void __launch_bounds__(256) bs_gather_kernel(const __grid_constant__ PrefixPack S, const float *__restrict__ gpk, float *__restrict__ grad_x)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)S.b * S.n) return;
    const int cloud = (int)(e / S.n), i = (int)(e % S.n);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int p = 0; p < S.np; p++) {
        if (i >= S.sizes[p]) continue;
        const float *r = gpk + (size_t)pack_row(S, p, cloud, i) * 3;
        a0 += r[0]; a1 += r[1]; a2 += r[2];
    }
    grad_x[e * 3 + 0] = a0; grad_x[e * 3 + 1] = a1; grad_x[e * 3 + 2] = a2;
}

// ---- parameter backward, BatchNorm: one thread per channel adds B s_g times the group means of dy and dy zhat over the groups, ascending
__global__ void __launch_bounds__(256) bs_bn_grad_kernel(const __grid_constant__ PrefixPack S, int C, const double *__restrict__ m12,
                                                         float *__restrict__ dgamma, float *__restrict__ dbeta)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s1 = 0.0, s2 = 0.0;
    for (int g = 0; g < S.np; g++) {
        const double cnt = (double)S.b * (double)S.sizes[g];
        s1 += m12[(size_t)g * 2 * C + c] * cnt;
        s2 += m12[((size_t)g * 2 + 1) * C + c] * cnt;
    }
    if (dbeta) dbeta[c] = (float)s1;
    if (dgamma) dgamma[c] = (float)s2;
}

// ---- parameter backward, weights and bias: per CTA one chunk of tiles (blockIdx.x) and one 64 x 64 tile of (output channel, input channel)
// (blockIdx.y); the sums run over the chunk's rows in order, the bias (a column of ones) alongside in tile column block 0.  Partials:
// (chunks, C K + C).
constexpr int kBwTile = 64, kBwRows = 32, kBwMaxChunks = 256;
struct BsWgradParams {
    PrefixPack S;
    int C, K, tiles_per_chunk;
    const float *z;                            // (rows, C) raw output of this layer
    const double *stats, *m12;                 // (np, 2, C): (mean, var) and (mean dy, mean dy zhat) per group
    const float *gamma; float eps;
    const float *dy;                           // (rows, C) masked gradient of this layer's BatchNorm output, or null: the top layer's
    const float *pooled; const int *route; const float *grad_pooled;   // ... pool coefficients (np, b, C)
    const float *x;                            // layer 1: the cloud (b, n, 3)
    const float *z_in;                         // (rows, K) raw output of the layer below, or null (layer 1)
    const double *stats_in; const float *gamma_in, *beta_in; float eps_in;
    float *part;
};

__global__ void __launch_bounds__(256) bs_wgrad_partial_kernel(const __grid_constant__ BsWgradParams Q)
{
    __shared__ __align__(16) float sdz[kBwRows][kBwTile];
    __shared__ __align__(16) float sa[kBwRows][kBwTile];
    __shared__ float vCoef[kBwTile], vM1[kBwTile], vM2[kBwTile], vMean[kBwTile], vInv[kBwTile], vSc[kBwTile], vSh[kBwTile];
    const PrefixPack &S = Q.S;
    const int C = Q.C, K = Q.K, otiles = (C + kBwTile - 1) / kBwTile;
    const int o0 = ((int)blockIdx.y % otiles) * kBwTile, k0 = ((int)blockIdx.y / otiles) * kBwTile;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int t0 = (int)blockIdx.x * Q.tiles_per_chunk, t1 = min(S.tile0[S.np], t0 + Q.tiles_per_chunk);
    float acc[4][4] = {}, bsum = 0.f;
    for (int tile = t0; tile < t1; tile++) {
        int g, cloud, i0, trows;
        pack_tile(S, tile, g, cloud, i0, trows);
        const long long prow0 = (long long)tile * kTcM;
        const size_t gb = ((size_t)g * S.b + cloud) * C;   // this segment's pool records
        __syncthreads();   // the previous tile's readers of the coefficients are done
        if (tid < kBwTile) {
            const int cg = o0 + tid;
            float coef = 0.f, m1 = 0.f, m2 = 0.f, mean = 0.f, inv = 0.f;
            if (cg < C) {
                const double *st = Q.stats + (size_t)g * 2 * C, *mm = Q.m12 + (size_t)g * 2 * C;
                mean = (float)st[cg];
                inv = 1.0f / sqrtf((float)st[C + cg] + Q.eps);
                coef = Q.gamma[cg] * inv;
                m1 = (float)mm[cg];
                m2 = (float)mm[C + cg];
            }
            vCoef[tid] = coef; vM1[tid] = m1; vM2[tid] = m2; vMean[tid] = mean; vInv[tid] = inv;
        } else if (tid < 2 * kBwTile && Q.z_in) {
            const int c = tid - kBwTile, kg = k0 + c;
            float sc = 0.f, sh = 0.f;
            if (kg < K) {
                const double *st = Q.stats_in + (size_t)g * 2 * K;
                bn_group_scale_shift(st[kg], st[K + kg], Q.gamma_in[kg], Q.beta_in[kg], Q.eps_in, sc, sh);
            }
            vSc[c] = sc; vSh[c] = sh;
        }
        __syncthreads();
        for (int r0 = 0; r0 < trows; r0 += kBwRows) {
            const int rows = min(kBwRows, trows - r0);
            for (int i = tid; i < kBwRows * kBwTile; i += 256) {
                const int r = i / kBwTile, c = i % kBwTile, cg = o0 + c, kg = k0 + c;
                const long long prow = prow0 + r0 + r;
                float dz = 0.f, a = 0.f;
                if (r < rows) {
                    if (cg < C) {
                        const float z = Q.z[(size_t)prow * C + cg];
                        float dy;
                        if (Q.dy) dy = Q.dy[(size_t)prow * C + cg];
                        else dy = (Q.route[gb + cg] == i0 + r0 + r && Q.pooled[gb + cg] > 0.f) ? Q.grad_pooled[gb + cg] : 0.f;
                        dz = vCoef[c] * (dy - vM1[c] - (z - vMean[c]) * vInv[c] * vM2[c]);
                    }
                    if (kg < K)
                        a = Q.z_in ? fmaxf(fmaf(Q.z_in[(size_t)prow * K + kg], vSc[c], vSh[c]), 0.f)
                                   : Q.x[((size_t)cloud * S.n + i0 + r0 + r) * 3 + kg];
                }
                sdz[r][c] = dz;
                sa[r][c] = a;
            }
            __syncthreads();
            for (int r = 0; r < rows; r++) {
                const float4 gv4 = *reinterpret_cast<const float4 *>(&sdz[r][ty * 4]);
                const float4 av4 = *reinterpret_cast<const float4 *>(&sa[r][tx * 4]);
                const float gv[4] = {gv4.x, gv4.y, gv4.z, gv4.w}, av[4] = {av4.x, av4.y, av4.z, av4.w};
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) acc[i][j] = fmaf(gv[i], av[j], acc[i][j]);
            }
            if (k0 == 0 && tid < kBwTile)
                for (int r = 0; r < rows; r++) bsum += sdz[r][tid];
            __syncthreads();
        }
    }
    float *part = Q.part + (size_t)blockIdx.x * ((size_t)C * K + C);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int o = o0 + ty * 4 + i;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int k = k0 + tx * 4 + j;
            if (o < C && k < K) part[(size_t)o * K + k] = acc[i][j];
        }
    }
    if (k0 == 0 && tid < kBwTile && o0 + tid < C) part[(size_t)C * K + o0 + tid] = bsum;
}

// ---- running statistics: one thread per (channel, layer = blockIdx.y) walks the prefixes in ascending order
struct BsRunningUpdate {
    PrefixPack S;
    int c[SNB200_MAX_CONV_LAYERS];
    const double *stats[SNB200_MAX_CONV_LAYERS];
    float *mean[SNB200_MAX_CONV_LAYERS], *var[SNB200_MAX_CONV_LAYERS];
    long long *nbt[SNB200_MAX_CONV_LAYERS];
    float momentum[SNB200_MAX_CONV_LAYERS];
};

__global__ void __launch_bounds__(256) bs_running_update_kernel(const __grid_constant__ BsRunningUpdate U)
{
    const int l = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x, C = U.c[l];
    if (c == 0 && U.nbt[l]) *U.nbt[l] += U.S.np;
    if (c >= C) return;
    const double *st = U.stats[l];
    for (int g = 0; g < U.S.np; g++)
        bn_running_step(U.mean[l], U.var[l], c, st[(size_t)g * 2 * C + c], st[((size_t)g * 2 + 1) * C + c], (double)U.S.b * (double)U.S.sizes[g],
                        U.momentum[l]);
}

// ------------------------------------------------------------------------------------------------------------------ host side
bool frozen_encoder_ex_supported(int b, int n, int act_input, int nconv, const snb200_layer *conv, int np, int tap);   // frozen_encoder.cu

bool frozen_encoder_bstat_supported(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes)
{
    if (b < 1 || n < 1 || n > kBsMaxN || np < 1 || np > kMaxPrefix || !sizes) return false;
    long long rows = 0;
    for (int p = 0; p < np; p++) {
        if (sizes[p] < 1 || sizes[p] > n || (p > 0 && sizes[p] <= sizes[p - 1])) return false;
        rows += (long long)b * tc_tiles_per_cloud(sizes[p]) * kTcM;
    }
    if (rows > kBsMaxRows) return false;
    if (!frozen_encoder_ex_supported(1, 1, 0, nconv, conv, 1, -1)) return false;
    for (int l = 0; l < nconv; l++)
        if (!conv[l].bn_weight || !conv[l].bn_bias || !conv[l].bias || !conv[l].relu) return false;
    return true;
}

// training: also an unbiased variance for every prefix (b * sizes[0] >= 2), as torch's BatchNorm refuses a one-value batch
bool frozen_encoder_bstat_train_supported(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes)
{
    return frozen_encoder_bstat_supported(b, n, nconv, conv, np, sizes) && (long long)b * sizes[0] >= 2;
}

static long long bs_rows(const PrefixPack &S) { return (long long)S.tile0[S.np] * kTcM; }

// the parameter backward's chunks of tiles: at most kBwMaxChunks of tiles_per_chunk tiles each
static int bs_tiles_per_chunk(const PrefixPack &S) { return (S.tile0[S.np] + kBwMaxChunks - 1) / kBwMaxChunks; }
static int bs_chunks(const PrefixPack &S) { return (S.tile0[S.np] + bs_tiles_per_chunk(S) - 1) / bs_tiles_per_chunk(S); }

// forward workspace: every layer's raw output (rows, c_out_l), the per-tile partials of the widest layer, the last layer's tile records
struct BsFwdWorkspace { float *z[SNB200_MAX_CONV_LAYERS]; float *part; float *tile_val; int *tile_idx; size_t total; };

static BsFwdWorkspace carve_bs_fwd(void *base, const PrefixPack &S, int nconv, const snb200_layer *conv)
{
    BsFwdWorkspace W;
    memset(&W, 0, sizeof(W));
    WsCarver c(base);
    const long long rows = bs_rows(S), tiles = S.tile0[S.np];
    int cmax = 0;
    for (int l = 0; l < nconv; l++) {
        W.z[l] = c.take<float>((size_t)rows * conv[l].c_out);
        cmax = max(cmax, conv[l].c_out);
    }
    W.part = c.take<float>((size_t)tiles * 2 * cmax);
    W.tile_val = c.take<float>((size_t)tiles * conv[nconv - 1].c_out);
    W.tile_idx = c.take<int>((size_t)tiles * conv[nconv - 1].c_out);
    W.total = c.off;
    return W;
}

// backward workspace: two (rows, widest hidden layer) gradient buffers, the packed point gradient, per-64-row partials, the group means;
// with parameter gradients then the weight-gradient chunk partials of the largest layer (one layer at a time)
struct BsBwdWorkspace { float *dy[2]; float *gpk; float *part; double *m12; float *wpart; size_t total; };

static BsBwdWorkspace carve_bs_bwd(void *base, const PrefixPack &S, int nconv, const snb200_layer *conv, bool params)
{
    BsBwdWorkspace W;
    WsCarver c(base);
    const long long rows = bs_rows(S);
    int hid = 0, cmax = 0;
    size_t wmax = 0;
    for (int l = 0; l < nconv; l++) {
        if (l < nconv - 1) hid = max(hid, conv[l].c_out);
        cmax = max(cmax, conv[l].c_out);
        wmax = max(wmax, (size_t)conv[l].c_out * (conv[l].c_in + 1));
    }
    W.dy[0] = c.take<float>((size_t)rows * hid);
    W.dy[1] = c.take<float>((size_t)rows * hid);
    W.gpk = c.take<float>((size_t)rows * 3);
    W.part = c.take<float>((size_t)(rows / kBsBwdRows) * 2 * hid);
    W.m12 = c.take<double>((size_t)S.np * 2 * cmax);
    W.wpart = params ? c.take<float>((size_t)bs_chunks(S) * wmax) : nullptr;
    W.total = c.off;
    return W;
}

size_t frozen_encoder_bstat_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes)
{
    return carve_bs_fwd(nullptr, prefix_pack(b, n, np, sizes), nconv, conv).total;
}

size_t frozen_encoder_bstat_backward_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, bool params)
{
    return carve_bs_bwd(nullptr, prefix_pack(b, n, np, sizes), nconv, conv, params).total;
}

// stats: per layer l a (np, 2, c_out_l) block of doubles, in layer order
static double *bs_stats(double *stats, int np, const snb200_layer *conv, int l)
{
    size_t off = 0;
    for (int q = 0; q < l; q++) off += (size_t)np * 2 * conv[q].c_out;
    return stats + off;
}

static int bs_reduce(const PrefixPack &S, const float *part, int C, int unit, int fwd, double *out, cudaStream_t stream, const char *what)
{
    bs_reduce_kernel<<<dim3(S.np, (C + 31) / 32), 256, 0, stream>>>(S, part, C, unit, fwd, out);
    return check_launch(what);
}

int launch_frozen_encoder_bstat_forward(int b, int n, const float *x, int nconv, const snb200_layer *conv, int np, const int *sizes, float *pooled,
                                        int *route, double *stats, void *workspace, cudaStream_t stream)
{
    const PrefixPack S = prefix_pack(b, n, np, sizes);
    const BsFwdWorkspace W = carve_bs_fwd(workspace, S, nconv, conv);
    const int tiles = S.tile0[np];
    const snb200_layer &L0 = conv[0];
    bs_l1_partial_kernel<<<tiles, 256, 0, stream>>>(S, x, L0.weight, L0.bias, L0.c_out, W.part);
    if (int rc = check_launch("batch-statistics encoder layer 1 partials")) return rc;
    if (int rc = bs_reduce(S, W.part, L0.c_out, kTcM, 1, bs_stats(stats, np, conv, 0), stream, "batch-statistics encoder statistics")) return rc;
    for (int l = 1; l < nconv; l++) {
        const snb200_layer &L = conv[l], &Lp = conv[l - 1];
        const bool last = l == nconv - 1;
        TcLayerParams P;
        memset(&P, 0, sizeof(P));
        P.b = 1; P.n = tiles * kTcM; P.tiles_per_cloud = tiles; P.c_in = L.c_in; P.c_out = L.c_out;
        if (l == 1) { P.x = x; P.x_layout = SNB200_BNC; P.w1 = Lp.weight; P.b1 = Lp.bias; P.out1 = W.z[0]; }
        else P.in = W.z[l - 1];
        P.in_has_bn = 1; P.in_gamma = Lp.bn_weight; P.in_beta = Lp.bn_bias; P.in_eps = Lp.bn_eps; P.in_relu = 1;
        P.weight = L.weight; P.bias = L.bias; P.out = W.z[l];
        P.pack = S; P.grp_in_stats = bs_stats(stats, np, conv, l - 1); P.grp_part = W.part;
        if (last) { P.pool_gamma = L.bn_weight; P.tile_val = W.tile_val; P.tile_idx = W.tile_idx; }
        if (int rc = launch_tc_layer(P, stream)) return rc;
        if (int rc = bs_reduce(S, W.part, L.c_out, kTcM, 1, bs_stats(stats, np, conv, l), stream, "batch-statistics encoder statistics")) return rc;
    }
    const snb200_layer &LL = conv[nconv - 1];
    const long long threads = (long long)np * b * LL.c_out;
    bs_pool_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(S, LL.c_out, LL.bn_weight, LL.bn_bias, LL.bn_eps,
                                                                          bs_stats(stats, np, conv, nconv - 1), W.tile_val, W.tile_idx, pooled, route);
    return check_launch("batch-statistics encoder pool");
}

static size_t bs_bwd_smem() { return ((size_t)kBsBwdRows * kBsLdz + kBsBwdCo * kBsBwdCi + 5 * kBsBwdCo + 4 * kBsBwdCi) * sizeof(float); }

// The weight / bias and gamma / beta gradients of layer l, while the chain's m12 and dy of layer l are live (before its dgrad reduces the
// layer below's sums into m12)
static int bs_param_grads(const PrefixPack &S, const BsBwdParams &Q, const float *x, const snb200_layer_grad &G, const BsBwdWorkspace &W,
                          cudaStream_t stream)
{
    if (G.bn_weight || G.bn_bias) {
        bs_bn_grad_kernel<<<(Q.C + 255) / 256, 256, 0, stream>>>(S, Q.C, Q.m12, G.bn_weight, G.bn_bias);
        if (int rc = check_launch("batch-statistics encoder backward: BatchNorm parameters")) return rc;
    }
    if (!G.weight && !G.bias) return SNB200_OK;
    BsWgradParams P;
    memset(&P, 0, sizeof(P));
    P.S = S; P.C = Q.C; P.K = Q.K; P.tiles_per_chunk = bs_tiles_per_chunk(S);
    P.z = Q.z; P.stats = Q.stats; P.m12 = Q.m12; P.gamma = Q.gamma; P.eps = Q.eps;
    P.dy = Q.dy; P.pooled = Q.pooled; P.route = Q.route; P.grad_pooled = Q.grad_pooled;
    P.x = x; P.z_in = Q.z_in; P.stats_in = Q.stats_in; P.gamma_in = Q.gamma_in; P.beta_in = Q.beta_in; P.eps_in = Q.eps_in;
    P.part = W.wpart;
    const unsigned tiles = (unsigned)(((Q.C + kBwTile - 1) / kBwTile) * ((Q.K + kBwTile - 1) / kBwTile));
    bs_wgrad_partial_kernel<<<dim3((unsigned)bs_chunks(S), tiles), 256, 0, stream>>>(P);
    if (int rc = check_launch("batch-statistics encoder backward: weight partials")) return rc;
    ReduceParams R;
    memset(&R, 0, sizeof(R));
    R.njobs = 1;
    R.job[0].part = W.wpart; R.job[0].nparts = bs_chunks(S); R.job[0].nw = Q.C * Q.K; R.job[0].nb = Q.C;
    R.job[0].g_weight = G.weight; R.job[0].g_bias = G.bias;
    return launch_reduce_partials(R, stream, "batch-statistics encoder backward: weight reduce");
}

// grads == NULL: the gradient of the points alone.  Otherwise also every parameter gradient grads points to (x is read for layer 1's
// weights), and grad_x may be NULL; the chain that gives grad_x is the same either way.
int launch_frozen_encoder_bstat_backward(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, const float *pooled,
                                         const int *route, const double *stats, const void *fwd_workspace, const float *grad_pooled, float *grad_x,
                                         void *workspace, cudaStream_t stream, const float *x, const snb200_layer_grad *grads)
{
    const PrefixPack S = prefix_pack(b, n, np, sizes);
    const BsFwdWorkspace F = carve_bs_fwd(const_cast<void *>(fwd_workspace), S, nconv, conv);
    const BsBwdWorkspace W = carve_bs_bwd(workspace, S, nconv, conv, grads != nullptr);
    double *st = const_cast<double *>(stats);
    const snb200_layer &LL = conv[nconv - 1];
    bs_top_sums_kernel<<<(np * LL.c_out + 255) / 256, 256, 0, stream>>>(S, LL.c_out, LL.bn_weight, LL.bn_bias, LL.bn_eps,
                                                                       bs_stats(st, np, conv, nconv - 1), F.z[nconv - 1], pooled, route,
                                                                       grad_pooled, W.m12);
    if (int rc = check_launch("batch-statistics encoder backward: top sums")) return rc;
    static PerDeviceOnce once;
    if (once.first()) cudaFuncSetAttribute(bs_bwd_layer_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bs_bwd_smem());
    const unsigned units = (unsigned)(S.tile0[np] * (kTcM / kBsBwdRows));
    for (int l = nconv - 1; l >= 0; l--) {
        const snb200_layer &L = conv[l];
        BsBwdParams Q;
        memset(&Q, 0, sizeof(Q));
        Q.S = S; Q.C = L.c_out; Q.K = L.c_in; Q.z = F.z[l]; Q.stats = bs_stats(st, np, conv, l); Q.m12 = W.m12;
        Q.gamma = L.bn_weight; Q.beta = L.bn_bias; Q.eps = L.bn_eps;
        if (l == nconv - 1) { Q.pooled = pooled; Q.route = route; Q.grad_pooled = grad_pooled; }
        else Q.dy = W.dy[l & 1];
        Q.weight = L.weight;
        if (l > 0) {
            const snb200_layer &Lp = conv[l - 1];
            Q.z_in = F.z[l - 1]; Q.stats_in = bs_stats(st, np, conv, l - 1); Q.gamma_in = Lp.bn_weight; Q.beta_in = Lp.bn_bias; Q.eps_in = Lp.bn_eps;
            Q.dy_in = W.dy[(l - 1) & 1]; Q.part_in = W.part;
        } else {
            Q.dy_in = W.gpk;
        }
        if (grads)
            if (int rc = bs_param_grads(S, Q, x, grads[l], W, stream)) return rc;
        if (l == 0 && !grad_x) break;
        bs_bwd_layer_kernel<<<dim3(units, (L.c_in + kBsBwdCi - 1) / kBsBwdCi), 256, bs_bwd_smem(), stream>>>(Q);
        if (int rc = check_launch("batch-statistics encoder backward: layer")) return rc;
        if (l > 0)
            if (int rc = bs_reduce(S, W.part, L.c_in, kBsBwdRows, 0, W.m12, stream, "batch-statistics encoder backward: sums")) return rc;
    }
    if (!grad_x) return SNB200_OK;
    const long long pts = (long long)b * n;
    bs_gather_kernel<<<(unsigned)((pts + 255) / 256), 256, 0, stream>>>(S, W.gpk, grad_x);
    return check_launch("batch-statistics encoder backward: gather");
}

int launch_frozen_encoder_bstat_running_update(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, const double *stats,
                                               cudaStream_t stream)
{
    BsRunningUpdate U;
    memset(&U, 0, sizeof(U));
    U.S = prefix_pack(b, n, np, sizes);
    int cmax = 0;
    for (int l = 0; l < nconv; l++) {
        U.c[l] = conv[l].c_out; U.stats[l] = bs_stats(const_cast<double *>(stats), np, conv, l);
        U.mean[l] = conv[l].bn_running_mean; U.var[l] = conv[l].bn_running_var; U.nbt[l] = conv[l].bn_num_batches_tracked;
        U.momentum[l] = conv[l].bn_momentum;
        cmax = max(cmax, conv[l].c_out);
    }
    bs_running_update_kernel<<<dim3((cmax + 255) / 256, nconv), 256, 0, stream>>>(U);
    return check_launch("batch-statistics encoder running statistics");
}

}  // namespace snb
