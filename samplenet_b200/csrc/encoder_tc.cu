// encoder_tc.cu -- the per-point MLP layers of the SampleNet generator on the tensor cores (warpgroup MMA, wgmma).
//
// Why tensor cores here and nowhere else: the conv stack (samplenet.py:90-94: 64->64->64->128->128 per point, 32 768
// points per step) is the one genuine dense contraction on the hot path (2.1 GFLOP of the step's 2.2).  Why 3xTF32: the
// reference computes these layers in fp32 and SampleNet's loss parity bar is 1e-5, which a single TF32/BF16 pass cannot
// hold.  Each fp32 operand is split exactly into hi = x & 0xffffe000 (representable in TF32) and lo = x - hi; the tile
// product is accumulated in fp32 registers as  A_hi*W_hi + A_hi*W_lo + A_lo*W_hi  (the dropped lo*lo term is < 2^-22 relative),
// i.e. three wgmma.m64n64k8.tf32 per K-step and 64-column tile into the same accumulator.
//
// Kernel shape (one launch per layer, CTA = 128 points x all output channels, two warpgroups of 64 points each):
//   prologue  all 256 threads: load the previous layer's RAW output tile, apply its BatchNorm+ReLU, split hi/lo and write
//             both into shared memory in the canonical K-major SWIZZLE_128B operand layout (rows of 128 B = 32 fp32 along K,
//             16-byte chunks XOR-swizzled with row%8, 8-row groups 1024 B apart); same for the weight tile (N rows);
//   MMA       every warpgroup issues 3 x 4 x (c_out/64) wgmma (M=64, N=64, K=8) per 32-wide K chunk, both operands from shared
//             memory; the next chunk's global loads fly while they run;
//   epilogue  accumulators + bias into a padded shared-memory copy of the tile, raw store to HBM from there, and column sums /
//             sums of squares (BatchNorm statistics) or column max/min (last layer, for the max-pool) reduced by one thread per
//             channel in a fixed order.  A training forward that keeps its activations for the backward stores the last layer's raw
//             output too, and layer 1's (out1) from the operand prologue that evaluates it.
// The layer's interface (workspace, statistics, extrema) is the one of the CUDA-core path in encoder.cu.
// A last layer wider than 256 channels (up to kTcMaxLastOut) runs as blocks of 256 output channels over grid.y; every narrower layer is one
// block.  tc_layer_kernel<NOUT, true> is the last layer of a frozen encoder (frozen_encoder.cu): no output store, and an epilogue that keeps
// the first extreme of sign(scale) * z per channel at every prefix boundary inside the tile (up to kMaxPrefix sizes in the kernel parameters,
// or any number in device memory with a per-tile table of the first boundary), or over a packed segment's rows in the tile (tc_seg_pool).
// tc_layer_kernel<NOUT, PFX, true> normalises its input with the statistics of the tile's group in the PrefixPack layout and leaves per-tile
// (sum, sumsq) partials instead of adding into global statistics (frozen_encoder_bstat.cu); with PFX it stores z and keeps the segment
// pool's per-tile records.  launch_tc_layer launches every instantiation.
#include "encoder_internal.cuh"

namespace snb {

constexpr int kTcThreads = 256;
constexpr int kTcKC = 32;   // K chunk resident in shared memory: one swizzle atom of 32 fp32 (128 B rows)

// byte offset of the 16-byte chunk `chunk` (0..7) of row `row` inside one [rows x 128 B] swizzle atom
__device__ __forceinline__ uint32_t sw128_off(int row, int chunk) { return (uint32_t)row * 128u + (uint32_t)((chunk ^ (row & 7)) << 4); }

__device__ __forceinline__ void split_store(unsigned char *hi_base, unsigned char *lo_base, uint32_t off, float4 v)
{
    float4 h, l;
    h.x = tf32_hi(v.x); l.x = v.x - h.x;
    h.y = tf32_hi(v.y); l.y = v.y - h.y;
    h.z = tf32_hi(v.z); l.z = v.z - h.z;
    h.w = tf32_hi(v.w); l.w = v.w - h.w;
    *reinterpret_cast<float4 *>(hi_base + off) = h;
    *reinterpret_cast<float4 *>(lo_base + off) = l;
}

// The segment pool: one thread per channel walks the tile's first `rows` rows of the staged tile (all inside one segment) in order, strict
// '>' keeping the first index among equal values; the index is relative to the segment's first row, i0 being the tile's first row in it.
template <int LD>
__device__ __forceinline__ void tc_seg_pool(const TcLayerParams &P, const float *sStage, int tile, int coff, int c_out, int rows, int i0)
{
    const int c = threadIdx.x;
    if (c >= c_out) return;
    const int cg = coff + c;
    const bool neg = P.pool_gamma && __ldg(P.pool_gamma + cg) < 0.f;
    float best = neg ? -sStage[c] : sStage[c];
    int arg = 0;
    for (int r = 1; r < rows; r++) {
        const float v = neg ? -sStage[r * LD + c] : sStage[r * LD + c];
        if (v > best) { best = v; arg = r; }
    }
    P.tile_val[(size_t)tile * P.c_out + cg] = best;
    P.tile_idx[(size_t)tile * P.c_out + cg] = i0 + arg;
}

// The CTA computes the output channels [256 blockIdx.y, +256) of its tile (all of them when gridDim.y == 1); every per-channel output --
// raw store, BatchNorm statistics, extrema -- goes to the layer-wide channel coff + c.  PFX: the prefix-pool epilogue of a frozen encoder's
// last layer (see TcLayerParams).  GRP: grouped statistics (see TcLayerParams).
template <int NOUT, bool PFX, bool GRP = false>  // padded output width: 64, 128 or 256 (NOUT / 64 wgmma tiles per warpgroup)
__global__ void __launch_bounds__(kTcThreads, (NOUT <= 128 ? 2 : 1)) tc_layer_kernel(const __grid_constant__ TcLayerParams P)
{
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    // operand buffers, one 32-wide K atom each: [rows][128 B]
    constexpr uint32_t kAtomA = kTcM * 128, kAtomB = NOUT * 128;
    constexpr int NA = (kTcM * 8) / kTcThreads;   // float4 loads per thread for the A atom (4)
    constexpr int NB = (NOUT * 8) / kTcThreads;   // ... for the B atom (2 / 4 / 8)
    constexpr int NT = NOUT / 64;                 // m64n64 accumulator tiles per warpgroup
    constexpr int LD = NOUT + 1;
    constexpr int H = kTcThreads / NOUT;          // row ranges in the epilogue reduction (4 / 2 / 1)
    unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // swizzle atoms start on 1024-byte boundaries
    unsigned char *sAhi = smem;
    unsigned char *sAlo = sAhi + kAtomA;
    unsigned char *sBhi = sAlo + kAtomA;
    unsigned char *sBlo = sBhi + kAtomB;
    float *sStage = reinterpret_cast<float *>(smem);  // epilogue: [128][NOUT+1] floats, aliases the operand buffers
    float *sPart = sStage + kTcM * LD;                // [H][NOUT][4] partial reductions
    __shared__ float sScale[256], sShift[256];
    __shared__ float sX[kTcM * 3], sW1[256 * 3], sB1[256];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2;                     // warpgroup: A rows [64 wg, 64 wg + 64) of the tile
    const int tile = blockIdx.x;
    const int cloud = tile / P.tiles_per_cloud;
    const int p0 = (tile % P.tiles_per_cloud) * kTcM;
    int np = min(kTcM, P.n - p0);
    int grp = 0, g_cloud = 0, g_i0 = 0;
    if constexpr (GRP) pack_tile(P.pack, tile, grp, g_cloud, g_i0, np);
    const int coff = (int)blockIdx.y * 256;
    const int c_in = P.c_in, c_out = min(256, P.c_out - coff);   // this block's channels
    const float *weight = P.weight + (size_t)coff * c_in, *bias = P.bias + coff;

    for (int c = tid; c < c_in; c += kTcThreads) {
        float sc = 1.f, sh = 0.f;
        if constexpr (GRP) {
            const double *st = P.grp_in_stats + (size_t)grp * 2 * c_in;
            if (P.in_has_bn) bn_group_scale_shift(st[c], st[c_in + c], P.in_gamma[c], P.in_beta[c], P.in_eps, sc, sh);
        } else if (P.in_has_bn) {
            bn_scale_shift(P.in_stats, c_in, c, (double)P.b * (double)P.n, P.in_gamma, P.in_beta, P.in_run_mean, P.in_run_var, P.in_eps,
                           P.in_training, sc, sh);
        }
        sScale[c] = sc;
        sShift[c] = sh;
    }
    if (P.x) {  // stage the 128 points of this tile and the first layer's weights
        if constexpr (GRP) {
            const float *xc = P.x + ((size_t)g_cloud * P.pack.n + g_i0) * 3;
            for (int e = tid; e < kTcM * 3; e += kTcThreads) sX[e] = (e / 3 < np) ? xc[e] : 0.f;
        } else {
            const float *xc = P.x + (size_t)cloud * P.n * 3;
            for (int e = tid; e < kTcM * 3; e += kTcThreads) {
                const int r = e / 3, c = e % 3;
                sX[e] = (r < np) ? (P.x_layout == SNB200_BNC ? xc[(size_t)(p0 + r) * 3 + c] : xc[(size_t)c * P.n + p0 + r]) : 0.f;
            }
        }
        for (int e = tid; e < c_in * 3; e += kTcThreads) sW1[e] = P.w1[e];
        for (int e = tid; e < c_in; e += kTcThreads) sB1[e] = P.b1 ? P.b1[e] : 0.f;
    }
    __syncthreads();

    float acc[NT][32];
#pragma unroll
    for (int j = 0; j < NT; j++)
#pragma unroll
        for (int i = 0; i < 32; i++) acc[j][i] = 0.f;
    const float *in_tile = P.x ? nullptr : P.in + ((size_t)cloud * P.n + p0) * c_in;
    const int nchunks = (c_in + kTcKC - 1) / kTcKC;
    // the thread's u-th 16-byte chunk of an atom is (row tid / 8 + 32 u, chunk tid % 8): every one has the same swizzle phase, so its
    // byte offset is that of u = 0 plus 32 rows of 128 B per u
    const uint32_t soff = sw128_off(tid >> 3, tid & 7);
    constexpr uint32_t kRowsPerU = kTcThreads / 8;
    for (int kc = 0; kc < nchunks; kc++) {
        const int k0 = kc * kTcKC;
        // ---- 1. all global loads of this K chunk go out first (NA + NB independent 16-byte loads per thread) ...
        float4 av[NA], wv[NB];
#pragma unroll
        for (int u = 0; u < NA; u++) {
            const int e = tid + u * kTcThreads, row = e >> 3, k = k0 + (e & 7) * 4;
            av[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (!P.x && row < np && k < c_in) av[u] = __ldg(reinterpret_cast<const float4 *>(in_tile + (size_t)row * c_in + k));
        }
#pragma unroll
        for (int u = 0; u < NB; u++) {
            const int e = tid + u * kTcThreads, row = e >> 3, k = k0 + (e & 7) * 4;
            wv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (row < c_out && k < c_in) wv[u] = __ldg(reinterpret_cast<const float4 *>(weight + (size_t)row * c_in + k));
        }
        // ---- 2. ... and fly while the tensor cores finish the previous chunk (its operands live in the same buffers)
        if (kc > 0) {
            wg_wait_all();
            __syncthreads();
        }
        // ---- 3. BatchNorm + ReLU of the previous layer, hi/lo split, swizzled store
#pragma unroll
        for (int u = 0; u < NA; u++) {
            const int e = tid + u * kTcThreads, row = e >> 3, ch = e & 7, k = k0 + ch * 4;
            float4 v = av[u];
            if (row < np && k < c_in) {
                if (P.x) {  // layer 1 on the fly: y = (w0*x + w1*y + w2*z) + b
                    const float px = sX[row * 3 + 0], py = sX[row * 3 + 1], pz = sX[row * 3 + 2];
                    v.x = fmaf(sW1[(k + 0) * 3 + 2], pz, fmaf(sW1[(k + 0) * 3 + 1], py, sW1[(k + 0) * 3 + 0] * px)) + sB1[k + 0];
                    v.y = fmaf(sW1[(k + 1) * 3 + 2], pz, fmaf(sW1[(k + 1) * 3 + 1], py, sW1[(k + 1) * 3 + 0] * px)) + sB1[k + 1];
                    v.z = fmaf(sW1[(k + 2) * 3 + 2], pz, fmaf(sW1[(k + 2) * 3 + 1], py, sW1[(k + 2) * 3 + 0] * px)) + sB1[k + 2];
                    v.w = fmaf(sW1[(k + 3) * 3 + 2], pz, fmaf(sW1[(k + 3) * 3 + 1], py, sW1[(k + 3) * 3 + 0] * px)) + sB1[k + 3];
                    // a CTA owns its 128 points and walks all of layer 1's channels (the K chunks) once: each value is stored exactly once
                    if (P.out1 && blockIdx.y == 0) *reinterpret_cast<float4 *>(P.out1 + ((size_t)cloud * P.n + p0 + row) * c_in + k) = v;
                }
                v.x = fmaf(v.x, sScale[k + 0], sShift[k + 0]); v.y = fmaf(v.y, sScale[k + 1], sShift[k + 1]);
                v.z = fmaf(v.z, sScale[k + 2], sShift[k + 2]); v.w = fmaf(v.w, sScale[k + 3], sShift[k + 3]);
                if (P.in_relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
                // a tapped activation: stored once, as out1 is
                if (P.in_act_out && blockIdx.y == 0) *reinterpret_cast<float4 *>(P.in_act_out + ((size_t)cloud * P.n + p0 + row) * c_in + k) = v;
            }
            split_store(sAhi, sAlo, soff + (uint32_t)u * kRowsPerU * 128u, v);
        }
#pragma unroll
        for (int u = 0; u < NB; u++) split_store(sBhi, sBlo, soff + (uint32_t)u * kRowsPerU * 128u, wv[u]);
        fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor cores (async proxy)
        __syncthreads();
        // ---- 4. each warpgroup: its 64 rows x all NOUT columns, 3 MMAs per K step of 8 and 64-column tile
        wg_fence();
        const int ksteps = min(kTcKC, c_in - k0) / 8;
#pragma unroll 1
        for (int ks = 0; ks < ksteps; ks++) {
            const uint32_t kin = (uint32_t)ks * 32u;  // byte advance inside the atom: 32 B per K=8 step
            const uint32_t arow = (uint32_t)wg * 64u * 128u;
            const uint64_t a_hi = wg_sdesc(smem_u32(sAhi) + arow + kin);
            const uint64_t a_lo = wg_sdesc(smem_u32(sAlo) + arow + kin);
            const uint32_t acc_in = (kc > 0 || ks > 0) ? 1u : 0u;
#pragma unroll
            for (int j = 0; j < NT; j++) {
                const uint32_t brow = (uint32_t)j * 64u * 128u;
                const uint64_t b_hi = wg_sdesc(smem_u32(sBhi) + brow + kin);
                const uint64_t b_lo = wg_sdesc(smem_u32(sBlo) + brow + kin);
                wg_mma_ss_n64(acc[j], a_lo, b_hi, acc_in);   // small terms first, the dominant hi*hi last
                wg_mma_ss_n64(acc[j], a_hi, b_lo, 1u);
                wg_mma_ss_n64(acc[j], a_hi, b_hi, 1u);
            }
        }
        wg_commit();
    }
    wg_wait_all();
    __syncthreads();   // both warpgroups are done with the operand buffers: the staging tile may overwrite them

    // ---- epilogue: accumulators (+bias) -> padded shared-memory copy of the tile -> HBM raw store (one contiguous block)
    {
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < NT; j++) {
#pragma unroll
            for (int jj = 0; jj < 8; jj++) {
                const int c = j * 64 + jj * 8 + cq;
                const float b0 = (c < c_out) ? __ldg(bias + c) : 0.f, b1 = (c + 1 < c_out) ? __ldg(bias + c + 1) : 0.f;
                sStage[r0 * LD + c] = acc[j][4 * jj + 0] + b0;
                sStage[r0 * LD + c + 1] = acc[j][4 * jj + 1] + b1;
                sStage[(r0 + 8) * LD + c] = acc[j][4 * jj + 2] + b0;
                sStage[(r0 + 8) * LD + c + 1] = acc[j][4 * jj + 3] + b1;
            }
        }
    }
    __syncthreads();
    if constexpr (PFX && !GRP) {
        if (P.seg) {
            // segment pool: the tile lies inside one segment, whose rows past its length are padding
            const int j = seg_find(P.seg, P.num_seg, p0);
            if (j < 0) return;
            const int2 s = __ldg(P.seg + j);
            tc_seg_pool<LD>(P, sStage, tile, coff, c_out, min(np, s.x + s.y - p0), p0 - s.x);
            return;
        }
        // prefix pool: one thread per channel walks the tile's rows in order, as tc_seg_pool does; a prefix's value does not depend on how
        // the tiles are later combined (max is exact).  The tile's boundaries are prefixes p .. pe - 1: scanned for in the parameter array,
        // or read from the per-tile table when the sizes are a device array.
        const int c = tid;
        if (c < c_out) {
            const int cg = coff + c;
            const bool neg = P.pool_gamma && __ldg(P.pool_gamma + cg) < 0.f;   // scale = gamma / sqrt(var + eps) has gamma's sign
            float best = neg ? -sStage[c] : sStage[c];
            const int *sizes = P.pack.sizes;
            int arg = p0, p = 0, pe = P.pack.np;
            if (P.pfx_first) {
                sizes = P.pfx_sizes;
                p = __ldg(P.pfx_first + p0 / kTcM);
                pe = __ldg(P.pfx_first + p0 / kTcM + 1);
            } else {
                while (p < pe && sizes[p] <= p0) p++;
            }
            for (int r = 0; r < np; r++) {
                const float v = neg ? -sStage[r * LD + c] : sStage[r * LD + c];
                if (v > best) { best = v; arg = p0 + r; }
                for (; p < pe && sizes[p] == p0 + r + 1; p++) {
                    const size_t o = ((size_t)p * P.b + cloud) * P.c_out + cg;
                    P.bound_val[o] = best;
                    P.bound_idx[o] = arg;
                }
            }
            P.tile_val[(size_t)tile * P.c_out + cg] = best;
            P.tile_idx[(size_t)tile * P.c_out + cg] = arg;
        }
        return;
    }
    if (P.out) {
        float *obase = P.out + ((size_t)cloud * P.n + p0) * P.c_out + coff;   // (points x P.c_out): contiguous rows when one block
        for (int e = tid; e < np * c_out; e += kTcThreads) {
            const int r = e / c_out, c = e - r * c_out;
            obase[(size_t)r * P.c_out + c] = sStage[r * LD + c];
        }
    }
    // ---- per-channel reductions over the tile's valid rows: H row ranges in parallel, combined in fixed order
    {
        const int c = tid % NOUT, h = tid / NOUT;
        const int r_lo = h * (kTcM / H), r_hi = min(np, (h + 1) * (kTcM / H));
        float sm = 0.f, ss = 0.f, mx = -INFINITY, mn = INFINITY;
        for (int r = r_lo; r < r_hi; r++) {
            const float v = sStage[r * LD + c];
            sm += v; ss = fmaf(v, v, ss); mx = fmaxf(mx, v); mn = fminf(mn, v);
        }
        float *pp = sPart + ((size_t)h * NOUT + c) * 4;
        pp[0] = sm; pp[1] = ss; pp[2] = mx; pp[3] = mn;
        __syncthreads();
        if (h == 0 && c < c_out) {
            for (int g = 1; g < H; g++) {
                const float *o = sPart + ((size_t)g * NOUT + c) * 4;
                sm += o[0]; ss += o[1]; mx = fmaxf(mx, o[2]); mn = fminf(mn, o[3]);
            }
            if constexpr (GRP) {
                P.grp_part[(size_t)tile * 2 * P.c_out + coff + c] = sm;
                P.grp_part[((size_t)tile * 2 + 1) * P.c_out + coff + c] = ss;
            } else if (P.out_stats) {
                atomicAdd(P.out_stats + coff + c, (double)sm);
                atomicAdd(P.out_stats + P.c_out + coff + c, (double)ss);
            }
            if (P.tile_max) {
                P.tile_max[(size_t)tile * P.c_out + coff + c] = mx;
                P.tile_min[(size_t)tile * P.c_out + coff + c] = mn;
            }
        }
    }
    if constexpr (PFX && GRP) {
        // the segment pool, the index being the point within the cloud's prefix (the tile is looked up again here rather than kept live
        // through the MMA loop)
        int rows;
        pack_tile(P.pack, tile, grp, g_cloud, g_i0, rows);
        tc_seg_pool<LD>(P, sStage, tile, coff, c_out, rows, g_i0);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Input moments -> BatchNorm statistics of the first layer, analytically.  Layer 1 is affine in the point (y = W1 p + b1),
// so sum_y[c] = cnt*(w_c.mu + b_c) and sum_y2[c] = cnt*(var_c + mean_c^2) with var_c = w_c^T Cov(p) w_c.  Twelve sums over the
// cloud (fp32 per thread, fp64 across threads) replace an 8.4 MB activation write + read and a full pass of statistics.
// The last CTA to arrive converts the moments into the (sum, sumsq) layout every other layer uses.
// mom: [0..2] sum p, [3..8] sum xx,xy,xz,yy,yz,zz ; counter: arrival count (both zeroed by the caller's memset)
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) x_moments_kernel(int b, int n, int layout, const float *__restrict__ x, double *mom, unsigned *counter,
                                                        const float *__restrict__ w1, const float *__restrict__ b1, int c1, double *stats0)
{
    __shared__ double s_red[9][8];
    __shared__ bool s_last;
    const long long total = (long long)b * n;
    float acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
        const long long bi = i / n, p = i % n;
        float px, py, pz;
        if (layout == SNB200_BNC) { const float *q = x + (bi * n + p) * 3; px = q[0]; py = q[1]; pz = q[2]; }
        else { const float *q = x + bi * n * 3 + p; px = q[0]; py = q[n]; pz = q[2 * (size_t)n]; }
        acc[0] += px; acc[1] += py; acc[2] += pz;
        acc[3] = fmaf(px, px, acc[3]); acc[4] = fmaf(px, py, acc[4]); acc[5] = fmaf(px, pz, acc[5]);
        acc[6] = fmaf(py, py, acc[6]); acc[7] = fmaf(py, pz, acc[7]); acc[8] = fmaf(pz, pz, acc[8]);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < 9; j++) {
        double v = (double)acc[j];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
        if (lane == 0) s_red[j][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x < 9) {
        double v = 0;
        for (int w = 0; w < 8; w++) v += s_red[threadIdx.x][w];
        atomicAdd(mom + threadIdx.x, v);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    const double cnt = (double)total;
    volatile double *vm = mom;
    const double mx = vm[0] / cnt, my = vm[1] / cnt, mz = vm[2] / cnt;
    const double cxx = vm[3] / cnt - mx * mx, cxy = vm[4] / cnt - mx * my, cxz = vm[5] / cnt - mx * mz;
    const double cyy = vm[6] / cnt - my * my, cyz = vm[7] / cnt - my * mz, czz = vm[8] / cnt - mz * mz;
    for (int c = threadIdx.x; c < c1; c += 256) {
        const double a0 = w1[c * 3 + 0], a1 = w1[c * 3 + 1], a2 = w1[c * 3 + 2];
        const double mean = a0 * mx + a1 * my + a2 * mz + (b1 ? (double)b1[c] : 0.0);
        double var = a0 * a0 * cxx + a1 * a1 * cyy + a2 * a2 * czz + 2.0 * (a0 * a1 * cxy + a0 * a2 * cxz + a1 * a2 * cyz);
        if (var < 0) var = 0;
        stats0[c] = cnt * mean;
        stats0[c1 + c] = cnt * (var + mean * mean);
    }
}

int launch_x_moments(int b, int n, int layout, const float *x, double *mom, unsigned *counter, const float *w1, const float *b1, int c1,
                     double *stats0, cudaStream_t stream)
{
    const long long total = (long long)b * n;
    int blocks = (int)((total + 255) / 256);
    if (blocks > kNumSMs) blocks = kNumSMs;
    x_moments_kernel<<<blocks, 256, 0, stream>>>(b, n, layout, x, mom, counter, w1, b1, c1, stats0);
    return check_launch("encoder input moments");
}

static size_t tc_smem_bytes(int nout)
{
    const size_t operands = 2 * (size_t)kTcM * 128 + 2 * (size_t)nout * 128;
    const size_t stage = (size_t)kTcM * (nout + 1) * sizeof(float) + (size_t)kTcThreads * 4 * sizeof(float);
    return (operands > stage ? operands : stage) + 1024;  // + alignment slack (the kernel rounds the base up to 1024 bytes)
}

bool tc_layer_supported(int c_in, int c_out) { return c_in % 8 == 0 && c_in >= 8 && c_in <= 256 && c_out >= 8 && c_out <= 256; }
bool tc_last_layer_supported(int c_in, int c_out) { return tc_layer_supported(c_in, 8) && c_out >= 8 && c_out <= kTcMaxLastOut; }

// every instantiation, [pool][grouped][NOUT 64 / 128 / 256], and the error text of a launch
static void (*const kTcKernels[2][2][3])(TcLayerParams) = {
    {{tc_layer_kernel<64, false>, tc_layer_kernel<128, false>, tc_layer_kernel<256, false>},
     {tc_layer_kernel<64, false, true>, tc_layer_kernel<128, false, true>, tc_layer_kernel<256, false, true>}},
    {{tc_layer_kernel<64, true>, tc_layer_kernel<128, true>, tc_layer_kernel<256, true>},
     {tc_layer_kernel<64, true, true>, tc_layer_kernel<128, true, true>, tc_layer_kernel<256, true, true>}}};
static const char *const kTcWhat[2][2] = {{"encoder tensor-core layer", "batch-statistics encoder layer"},
                                          {"frozen encoder last layer", "batch-statistics encoder last layer"}};

int launch_tc_layer(const TcLayerParams &P, cudaStream_t stream)
{
    static PerDeviceOnce once;
    if (once.first())
        for (auto &by_grp : kTcKernels)
            for (auto &by_nout : by_grp)
                for (int i = 0; i < 3; i++) cudaFuncSetAttribute(by_nout[i], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem_bytes(64 << i));
    const int pool = P.tile_val != nullptr, grp = P.grp_part != nullptr, i = P.c_out <= 64 ? 0 : (P.c_out <= 128 ? 1 : 2);
    dim3 grid(P.b * P.tiles_per_cloud, (P.c_out + 255) / 256);
    kTcKernels[pool][grp][i]<<<grid, kTcThreads, tc_smem_bytes(64 << i), stream>>>(P);
    return check_launch(kTcWhat[pool][grp]);
}

int launch_tc_stack(int b, int n, int layout, const float *x, int nconv, const snb200_layer *conv, int training, double *const *stats,
                    float *const *zsave, float *const *act, const TcStackTail &tail, cudaStream_t stream, const float *act_in, int tap,
                    float *tap_out)
{
    for (int l = act_in ? 0 : 1; l < nconv; l++) {
        const snb200_layer &L = conv[l];
        const bool last = l == nconv - 1, pool = last && (tail.num_prefix > 0 || tail.seg);
        TcLayerParams P;
        memset(&P, 0, sizeof(P));
        P.b = b; P.n = n; P.tiles_per_cloud = tc_tiles_per_cloud(n); P.c_in = L.c_in; P.c_out = L.c_out;
        if (l == 0) {
            P.in = act_in;   // identity input: no BatchNorm, no ReLU
        } else {
            const snb200_layer &Lp = conv[l - 1];
            if (l == 1 && !act_in) { P.x = x; P.x_layout = layout; P.w1 = Lp.weight; P.b1 = Lp.bias; P.out1 = zsave ? zsave[0] : nullptr; }
            else P.in = zsave ? zsave[l - 1] : act[(l - 1) & 1];
            P.in_has_bn = Lp.bn_weight != nullptr; P.in_stats = stats ? stats[l - 1] : nullptr;
            P.in_gamma = Lp.bn_weight; P.in_beta = Lp.bn_bias; P.in_run_mean = Lp.bn_running_mean; P.in_run_var = Lp.bn_running_var;
            P.in_eps = Lp.bn_eps; P.in_relu = Lp.relu; P.in_training = training;
            if (l - 1 == tap) P.in_act_out = tap_out;
        }
        P.weight = L.weight; P.bias = L.bias;
        P.out_stats = (training && L.bn_weight) ? stats[l] : nullptr;
        if (!last) P.out = zsave ? zsave[l] : act[l & 1];
        else if (!pool) { P.out = zsave ? zsave[l] : nullptr; P.tile_max = tail.tile_max; P.tile_min = tail.tile_min; }
        else {
            P.pack.np = tail.num_prefix; P.pool_gamma = L.bn_weight;
            if (tail.dev_first) { P.pfx_sizes = tail.sizes; P.pfx_first = tail.dev_first; }
            else for (int p = 0; p < tail.num_prefix; p++) P.pack.sizes[p] = tail.sizes[p];
            P.bound_val = tail.bound_val; P.bound_idx = tail.bound_idx; P.tile_val = tail.tile_val; P.tile_idx = tail.tile_idx;
            P.seg = tail.seg; P.num_seg = tail.num_seg;
        }
        if (int rc = launch_tc_layer(P, stream)) return rc;
    }
    return SNB200_OK;
}

// Unit-test entry: D (rows, c_out) = A (rows, c_in) * W (c_out, c_in)^T + bias through the tensor-core layer kernel with no
// BatchNorm, rows = b*n points.
int launch_tc_gemm_debug(int rows, int c_in, int c_out, const float *A, const float *W, const float *bias, float *D, cudaStream_t stream)
{
    TcLayerParams P;
    memset(&P, 0, sizeof(P));
    P.in = A; P.c_in = c_in; P.c_out = c_out; P.b = 1; P.n = rows; P.tiles_per_cloud = tc_tiles_per_cloud(rows);
    P.weight = W; P.bias = bias; P.out = D;
    return launch_tc_layer(P, stream);
}

}  // namespace snb
