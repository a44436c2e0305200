// frozen_encoder.cu -- a frozen PointNet encoder (eval-mode BatchNorm, no parameter gradients) evaluated over every prefix of a cloud in one
// shared pass, and its gradient with respect to the points.
//
// With BatchNorm in eval mode every conv layer is a per-point function: point i's activations are the same in every prefix that holds it,
// and only the max-pool depends on the prefix.  So
//   forward   layers 1 .. L-1 run once over all n points on the tensor-core layer kernels (encoder_tc.cu), each raw output kept in zsave;
//             the last layer (up to 1024 channels, 256 per CTA over grid.y) never stores its output: its epilogue keeps, per (tile,
//             channel), the first extreme of sign(scale) * z over the tile's rows and emits it at every prefix boundary inside the tile and
//             at the tile's end (tc_layer_kernel<NOUT, true>); prefix_combine_kernel folds those into pooled / route for every prefix;
//   backward  only the points the pool routes to get a gradient.  For each (prefix p, cloud b, channel c) the coefficient
//             g[p,b,c] * scale_c * [pooled > 0] lands on route[p,b,c]; route_mark_kernel sets one bit per (point, channel) that receives
//             any, and chain_bwd_kernel (one warp per point) sums, for each of its point's channels in channel order, the coefficients of
//             the prefixes routed to it in prefix order, multiplies by W_L, and runs the point-local chain dz_l = dA_l * scale_l * mask_l,
//             dA_{l-1} = dz_l W_l down to dX = dz_1 W_1.  Masks are recomputed from zsave with the forward's own fp32 expression
//             (fmaf(z, scale, shift) > 0, the same bn_scale_shift), so they are the forward's decisions bit for bit.  No float atomics,
//             no dense (points x channels) gradient buffer; points nobody routes to get exactly 0.
// The extended entries (snb200_frozen_encoder_ex_*) run the same kernels with two additions, for a network whose conv stack is split by a
// per-cloud transform (PointNet with its transform nets):
//   activation input  layer 1 is a tensor-core layer too, reading a (b*n, c_in) activation as it is; the backward's last step writes
//                     dA_0 = dz_1 W_1 (b*n, c_in) instead of dX;
//   tap               hidden layer t's activation a_t is also stored (by the prologue of layer t + 1, which evaluates it anyway), and the
//                     backward takes a dense gradient for it: the chain adds it to dA_t of every point, in a fixed order, and a point that no
//                     prefix routes to starts its chain at layer t instead of being skipped.
// The segmented entries (snb200_frozen_encoder_seg_*) take a packed buffer of segments instead of prefixes of clouds, so that rows which
// depend on their prefix (x[:, :s] @ T1(s) in PointNet with transform nets) can share one pass: one pool per segment, each segment starting
// on a tile (see "segments" below).
// The parameter backward (snb200_frozen_encoder_param_backward, conv stacks without BatchNorm: PCRNet trained) adds the weight and bias
// gradients, every sum in a fixed order (no float atomics):
//   last layer L   last_grad_kernel, one warp per channel c: dW_L[c,:] = sum over clouds b, then prefixes p (ascending) of
//                  coef[p,b,c] a_{L-1}[b, route[p,b,c], :] and db_L[c] = sum coef, coef the chain's g * scale * [pooled > 0]; a_{L-1} is
//                  recomputed from zsave with the forward's activation expression;
//   hidden layers  the chain also stores dz_l of every point (zeros where nothing routes) as dense (b*n, c_out_l) rows in the workspace;
//                  hidden_grad_partial_kernel sums dz_l^T [a_{l-1} | 1] over one chunk of points in point order per CTA (a 64 x 64 output
//                  tile, 4 x 4 per thread), and the generator's reduce_partials_kernel adds the chunks in a fixed order.
// The curve entries (snb200_frozen_encoder_curve_*) run the forward over any number of prefixes, up to every size 1 .. n: the sizes are
// staged in the workspace, and the serial walk of prefix_combine_kernel becomes a running extreme over the tiles and an element-parallel
// combine (see "many prefixes" below).
#include "encoder_internal.cuh"

#include <vector>

namespace snb {

constexpr int kFeMaxHidden = 256;     // widest hidden layer (tc_layer_supported)
constexpr int kFeWarps = 8;           // chain_bwd_kernel: one point per warp at a time

struct FrozenLayer {
    const float *weight, *gamma, *beta, *run_mean, *run_var;
    float eps;
    int c_in, c_out, has_bn, relu;
};

struct FrozenParams {
    int b, n, nconv, np, tiles;
    int tap;                    // hidden layer whose activation gradient grad_tap holds, or -1
    int sizes[kMaxPrefix];
    FrozenLayer L[SNB200_MAX_CONV_LAYERS];
    // segments (the _seg entries): b = num_seg segments (offset, length) of a packed buffer of `rows` rows, np = 1, n unused
    const int2 *seg;
    long long rows;
};

struct FrozenZsave {
    const float *z[SNB200_MAX_CONV_LAYERS];   // raw outputs of the hidden layers, (b * n, c_out_l)
};

struct FrozenDz {
    float *dz[SNB200_MAX_CONV_LAYERS];        // per hidden layer the gradient of its raw output, (b * n, c_out_l), or all NULL: not stored
};

static FrozenParams frozen_params(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, int tap = -1)
{
    FrozenParams F;
    memset(&F, 0, sizeof(F));
    F.b = b; F.n = n; F.nconv = nconv; F.np = np; F.tiles = tc_tiles_per_cloud(n); F.tap = tap; F.rows = (long long)b * n;
    for (int p = 0; p < np; p++) F.sizes[p] = sizes[p];
    for (int l = 0; l < nconv; l++) {
        const snb200_layer &s = conv[l];
        F.L[l] = FrozenLayer{s.weight, s.bn_weight, s.bn_bias, s.bn_running_mean, s.bn_running_var, s.bn_eps, s.c_in, s.c_out, s.bn_weight != nullptr, s.relu};
    }
    return F;
}

// the eval-mode scale / shift of layer l's channel c, exactly as the forward kernels evaluate them
__device__ __forceinline__ void frozen_scale_shift(const FrozenLayer &L, int c, float &sc, float &sh)
{
    sc = 1.f; sh = 0.f;
    if (L.has_bn) bn_scale_shift(nullptr, L.c_out, c, 0.0, L.gamma, L.beta, L.run_mean, L.run_var, L.eps, 0, sc, sh);
}

// layer l's activation from its raw output, the expression of the forward's next-layer prologue
__device__ __forceinline__ float frozen_act(const FrozenLayer &L, float z, float sc, float sh)
{
    const float a = fmaf(z, sc, sh);
    return L.relu ? fmaxf(a, 0.f) : a;
}

// ---- forward: per-tile extrema -> pooled / route of every prefix.  One thread per (cloud, channel) walks the tiles in order: a prefix whose
// last point lies in tile t takes the tiles before t whole and tile t's boundary record; ties keep the earlier tile (the lower index).
__global__ void __launch_bounds__(256) prefix_combine_kernel(const __grid_constant__ FrozenParams F, const float *__restrict__ tile_val,
                                                             const int *__restrict__ tile_idx, const float *__restrict__ bound_val,
                                                             const int *__restrict__ bound_idx, float *__restrict__ pooled, int *__restrict__ route)
{
    const FrozenLayer &L = F.L[F.nconv - 1];
    const int C = L.c_out;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= F.b * C) return;
    const int bi = e / C, c = e % C;
    float sc, sh;
    frozen_scale_shift(L, c, sc, sh);
    const bool neg = L.has_bn && L.gamma[c] < 0.f;
    float run = -INFINITY;
    int run_i = -1, t = 0;
    for (int p = 0; p < F.np; p++) {
        const int last = (F.sizes[p] - 1) / kTcM;
        for (; t < last; t++) {
            const size_t o = ((size_t)bi * F.tiles + t) * C + c;
            const float v = tile_val[o];
            if (run_i < 0 || v > run) { run = v; run_i = tile_idx[o]; }
        }
        const size_t o = ((size_t)p * F.b + bi) * C + c;
        float v = bound_val[o];
        int vi = bound_idx[o];
        if (run_i >= 0 && !(v > run)) { v = run; vi = run_i; }
        float a = fmaf(neg ? -v : v, sc, sh);
        if (L.relu) a = fmaxf(a, 0.f);
        pooled[o] = a;
        route[o] = vi;
    }
}

// ---- forward over many prefixes (the _curve entries), step 1: per (cloud, channel) the tile records become, in place, the running extreme
// of the tiles before each one (index -1 before tile 0), with prefix_combine_kernel's rule: the first tile is taken, a later one only on '>'.
__global__ void __launch_bounds__(256) curve_carry_kernel(int b, int tiles, int C, float *__restrict__ tile_val, int *__restrict__ tile_idx)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= b * C) return;
    const int bi = e / C, c = e % C;
    float run = -INFINITY;
    int run_i = -1;
    for (int t = 0; t < tiles; t++) {
        const size_t o = ((size_t)bi * tiles + t) * C + c;
        const float v = tile_val[o];
        const int vi = tile_idx[o];
        tile_val[o] = run;
        tile_idx[o] = run_i;
        if (run_i < 0 || v > run) { run = v; run_i = vi; }
    }
}

// step 2: one thread per (prefix, cloud, channel) finishes the boundary record the last layer left in pooled / route: the carry of the tiles
// before the boundary's tile wins ties (prefix_combine_kernel's expression), then the BatchNorm and ReLU of the pooled value.  grid.x walks
// the (prefix, cloud) rows, grid.y blocks of 256 channels.
__global__ void __launch_bounds__(256) curve_combine_kernel(const __grid_constant__ FrozenParams F, const int *__restrict__ sizes,
                                                            const float *__restrict__ carry_val, const int *__restrict__ carry_idx,
                                                            float *__restrict__ pooled, int *__restrict__ route)
{
    const FrozenLayer &L = F.L[F.nconv - 1];
    const int C = L.c_out, c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const int row = blockIdx.x, p = row / F.b, bi = row - p * F.b;
    const size_t t = (size_t)bi * F.tiles + (__ldg(sizes + p) - 1) / kTcM, e = (size_t)row * C + c;
    const float run = carry_val[t * C + c];
    const int run_i = carry_idx[t * C + c];
    float v = pooled[e];
    int vi = route[e];
    if (run_i >= 0 && !(v > run)) { v = run; vi = run_i; }
    float sc, sh;
    frozen_scale_shift(L, c, sc, sh);
    const bool neg = L.has_bn && L.gamma[c] < 0.f;
    float a = fmaf(neg ? -v : v, sc, sh);
    if (L.relu) a = fmaxf(a, 0.f);
    pooled[e] = a;
    route[e] = vi;
}

// ---- forward, segments: one thread per (segment, channel) walks the segment's tile records
__global__ void __launch_bounds__(256) seg_combine_kernel(const __grid_constant__ FrozenParams F, const float *__restrict__ tile_val,
                                                          const int *__restrict__ tile_idx, float *__restrict__ pooled, int *__restrict__ route)
{
    const FrozenLayer &L = F.L[F.nconv - 1];
    const int C = L.c_out;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= F.b * C) return;
    const int j = e / C, c = e % C;
    float sc, sh;
    frozen_scale_shift(L, c, sc, sh);
    const bool neg = L.has_bn && L.gamma[c] < 0.f;
    const int2 s = F.seg[j];
    float run;
    int run_i;
    seg_tile_extreme(tile_val, tile_idx, C, c, s.x / kTcM, (s.x + s.y - 1) / kTcM + 1, run, run_i);
    float a = fmaf(neg ? -run : run, sc, sh);
    if (L.relu) a = fmaxf(a, 0.f);
    pooled[e] = a;
    route[e] = run_i;
}

// ---- backward 1: one bit per (point, channel) that some prefix routes a nonzero coefficient to (integer atomics: the result is exact)
__global__ void __launch_bounds__(256) route_mark_kernel(const __grid_constant__ FrozenParams F, const float *__restrict__ pooled,
                                                         const int *__restrict__ route, unsigned *__restrict__ bits, int words)
{
    const FrozenLayer &L = F.L[F.nconv - 1];
    const int C = L.c_out;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= F.np * F.b * C) return;
    const int c = e % C, bi = (e / C) % F.b;
    if (L.relu && !(pooled[e] > 0.f)) return;
    const size_t row = (F.seg ? (size_t)F.seg[bi].x : (size_t)bi * F.n) + route[e];   // a segment's route is relative to its first row
    atomicOr(bits + row * words + (c >> 5), 1u << (c & 31));
}

// ---- backward 2: one warp per point, every step in a fixed order
__global__ void __launch_bounds__(kFeWarps * 32) chain_bwd_kernel(const __grid_constant__ FrozenParams F, const float *__restrict__ pooled,
                                                                  const int *__restrict__ route, const float *__restrict__ grad_pooled,
                                                                  const unsigned *__restrict__ bits, int words,
                                                                  const __grid_constant__ FrozenZsave Z, const float *__restrict__ grad_tap,
                                                                  float *__restrict__ grad_x, const __grid_constant__ FrozenDz D)
{
    extern __shared__ float s_fe[];
    // [scale | shift] of every layer behind each other, then per warp two vectors of kFeMaxHidden
    int off[SNB200_MAX_CONV_LAYERS + 1];
    off[0] = 0;
    for (int l = 0; l < F.nconv; l++) off[l + 1] = off[l] + 2 * F.L[l].c_out;
    for (int l = 0; l < F.nconv; l++)
        for (int c = threadIdx.x; c < F.L[l].c_out; c += blockDim.x) frozen_scale_shift(F.L[l], c, s_fe[off[l] + c], s_fe[off[l] + F.L[l].c_out + c]);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float *dA = s_fe + off[F.nconv] + warp * 2 * kFeMaxHidden;   // gradient of the current layer's activation
    float *dz = dA + kFeMaxHidden;                                // ... of its raw output
    const FrozenLayer &LL = F.L[F.nconv - 1];
    const int C = LL.c_out, K = LL.c_in, c0 = F.L[0].c_in;
    const float *sc_last = s_fe + off[F.nconv - 1];
    for (long long pt = (long long)blockIdx.x * kFeWarps + warp; pt < F.rows; pt += (long long)gridDim.x * kFeWarps) {
        // (cloud, point), or with segments (segment, row within it); a packed row outside every segment gets 0 as one nobody routes to
        int bi, i;
        if (F.seg) {
            bi = seg_find(F.seg, F.b, pt);
            i = bi < 0 ? 0 : (int)(pt - F.seg[bi].x);
        } else {
            bi = (int)(pt / F.n); i = (int)(pt % F.n);
        }
        const unsigned word = lane < words ? bits[pt * words + lane] : 0u;
        const bool routed = __any_sync(kFullMask, word != 0u);
        if (bi < 0 || (!routed && F.tap < 0)) {
            if (grad_x)
                for (int j = lane; j < c0; j += 32) grad_x[pt * c0 + j] = 0.f;
            if (D.dz[0])
                for (int l = 0; l < F.nconv - 1; l++)
                    for (int k = lane; k < F.L[l].c_out; k += 32) D.dz[l][pt * F.L[l].c_out + k] = 0.f;
            continue;
        }
        // last layer: dA_{L-1}[k] = sum over the point's channels c (ascending) of D_c W_L[c, k], D_c = sum over prefixes p routed here
        // (ascending) of g[p,b,c] * scale_c.  Without any, the chain starts at the tapped layer with dA = 0.
        const int top = routed ? F.nconv - 2 : F.tap;
        for (int k = lane; k < F.L[top].c_out; k += 32) dA[k] = 0.f;
        __syncwarp();
        for (int w = 0; w < (routed ? words : 0); w++) {
            unsigned m = __shfl_sync(kFullMask, word, w);
            while (m) {
                const int c = w * 32 + __ffs(m) - 1;
                m &= m - 1;
                float d = 0.f;
                for (int p = 0; p < F.np; p++) {
                    const size_t o = ((size_t)p * F.b + bi) * C + c;
                    if (route[o] == i && (!LL.relu || pooled[o] > 0.f)) d += grad_pooled[o] * sc_last[c];
                }
                const float *wr = LL.weight + (size_t)c * K;
                for (int k = lane; k < K; k += 32) dA[k] = fmaf(d, __ldg(wr + k), dA[k]);
            }
        }
        __syncwarp();
        // hidden layers, top down
        for (int l = top; l >= 0; l--) {
            const FrozenLayer &L = F.L[l];
            const float *sc = s_fe + off[l], *sh = sc + L.c_out;
            const float *zr = Z.z[l] + pt * L.c_out;
            const float *gt = l == F.tap ? grad_tap + pt * L.c_out : nullptr;   // the dense gradient of this layer's activation, if tapped
            for (int k = lane; k < L.c_out; k += 32) {
                const bool on = !L.relu || fmaf(zr[k], sc[k], sh[k]) > 0.f;
                const float d = gt ? dA[k] + gt[k] : dA[k];
                dz[k] = on ? d * sc[k] : 0.f;
                if (D.dz[0]) D.dz[l][pt * L.c_out + k] = dz[k];
            }
            __syncwarp();
            if (l == 0 && !grad_x) break;
            // dA_{l-1} = dz_l W_l; below layer 1 this is the gradient of the input (the cloud's 3 coordinates or the input activation)
            float *dst = l > 0 ? dA : grad_x + pt * c0;
            for (int j = lane; j < L.c_in; j += 32) {
                float a = 0.f;
                for (int k = 0; k < L.c_out; k++) a = fmaf(dz[k], __ldg(L.weight + (size_t)k * L.c_in + j), a);
                dst[j] = a;
            }
            __syncwarp();
        }
    }
}

// ---- parameter backward (layers without BatchNorm: scale 1, shift 0), last layer: one warp per channel.  The (cloud, prefix) terms are
// walked 32 at a time in order; each lane fetches one term's coefficient and route, and the warp then gathers the routed rows of a_{L-1}
// one after the other (lane = input channel).
constexpr int kFeKPerLane = kFeMaxHidden / 32;
__global__ void __launch_bounds__(kFeWarps * 32) last_grad_kernel(const __grid_constant__ FrozenParams F, const float *__restrict__ pooled,
                                                                  const int *__restrict__ route, const float *__restrict__ grad_pooled,
                                                                  const __grid_constant__ FrozenZsave Z, float *__restrict__ dW, float *__restrict__ db)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const FrozenLayer &LL = F.L[F.nconv - 1], &LP = F.L[F.nconv - 2];
    const int C = LL.c_out, K = LL.c_in, c = (int)blockIdx.x * kFeWarps + warp;
    if (c >= C) return;
    float acc[kFeKPerLane];
#pragma unroll
    for (int j = 0; j < kFeKPerLane; j++) acc[j] = 0.f;
    const float *a_prev = Z.z[F.nconv - 2];
    float bsum = 0.f;
    const int terms = F.b * F.np;     // b * n <= 2^18: a row index fits an int
    for (int q0 = 0; q0 < terms; q0 += 32) {
        const int q = q0 + lane, bi = q / F.np, p = q % F.np;
        float d = 0.f;
        int row = -1;
        if (q < terms) {
            const size_t o = ((size_t)p * F.b + bi) * C + c;
            if (!LL.relu || pooled[o] > 0.f) { d = grad_pooled[o]; row = bi * F.n + route[o]; }
        }
        const int cnt = min(32, terms - q0);
#pragma unroll 4
        for (int t = 0; t < cnt; t++) {
            const float dt = __shfl_sync(kFullMask, d, t);
            const int rt = __shfl_sync(kFullMask, row, t);
            if (rt < 0) continue;
            const float *zr = a_prev + (size_t)rt * K;
#pragma unroll
            for (int j = 0; j < kFeKPerLane; j++) {
                const int k = lane + 32 * j;
                if (k < K) acc[j] = fmaf(dt, frozen_act(LP, zr[k], 1.f, 0.f), acc[j]);
            }
            bsum += dt;
        }
    }
#pragma unroll
    for (int j = 0; j < kFeKPerLane; j++)
        if (dW && lane + 32 * j < K) dW[(size_t)c * K + lane + 32 * j] = acc[j];
    if (db && lane == 0) db[c] = bsum;
}

// ---- parameter backward, hidden layers: per CTA one chunk of points and one 64 x 64 tile of (output channel, input channel) of one layer;
// the sums run over the chunk's points in order, the bias (a column of ones) alongside in tile column block 0.  Partials: (chunks, nw + nb).
constexpr int kHgTile = 64, kHgPts = 32;
struct HiddenGradJobs {
    int njobs, chunks, chunk_pts;
    int layer[SNB200_MAX_CONV_LAYERS];
    float *part[SNB200_MAX_CONV_LAYERS];
};
__global__ void __launch_bounds__(256) hidden_grad_partial_kernel(const __grid_constant__ FrozenParams F, const float *__restrict__ x,
                                                                  const __grid_constant__ FrozenZsave Z, const __grid_constant__ FrozenDz D,
                                                                  const __grid_constant__ HiddenGradJobs J)
{
    __shared__ __align__(16) float sdz[kHgPts][kHgTile];
    __shared__ __align__(16) float sa[kHgPts][kHgTile];
    const int l = J.layer[blockIdx.z];
    const FrozenLayer &L = F.L[l];
    const int C = L.c_out, K = L.c_in;
    const int otiles = (C + kHgTile - 1) / kHgTile, ktiles = (K + kHgTile - 1) / kHgTile;
    if ((int)blockIdx.y >= otiles * ktiles) return;
    const int o0 = ((int)blockIdx.y % otiles) * kHgTile, k0 = ((int)blockIdx.y / otiles) * kHgTile;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const long long pts = (long long)F.b * F.n;
    const long long p0 = (long long)blockIdx.x * J.chunk_pts, p1 = min(pts, p0 + J.chunk_pts);
    const float *dzl = D.dz[l], *zin = l > 0 ? Z.z[l - 1] : nullptr;
    float acc[4][4] = {}, bsum = 0.f;
    for (long long s0 = p0; s0 < p1; s0 += kHgPts) {
        for (int i = tid; i < kHgPts * kHgTile; i += 256) {
            const int r = i / kHgTile, c = i % kHgTile;
            const long long pt = s0 + r;
            const bool in_pt = pt < p1;
            sdz[r][c] = (in_pt && o0 + c < C) ? dzl[pt * C + o0 + c] : 0.f;
            float a = 0.f;
            if (in_pt && k0 + c < K) {
                a = zin ? frozen_act(F.L[l - 1], zin[pt * K + k0 + c], 1.f, 0.f) : x[pt * K + k0 + c];
            }
            sa[r][c] = a;
        }
        __syncthreads();
        const int rows = (int)min((long long)kHgPts, p1 - s0);
        for (int r = 0; r < rows; r++) {
            const float4 g = *reinterpret_cast<const float4 *>(&sdz[r][ty * 4]);
            const float4 a = *reinterpret_cast<const float4 *>(&sa[r][tx * 4]);
            const float gv[4] = {g.x, g.y, g.z, g.w}, av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(gv[i], av[j], acc[i][j]);
        }
        if (k0 == 0 && tid < kHgTile)
            for (int r = 0; r < rows; r++) bsum += sdz[r][tid];
        __syncthreads();
    }
    float *part = J.part[blockIdx.z] + (size_t)blockIdx.x * ((size_t)C * K + C);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int o = o0 + ty * 4 + i;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int k = k0 + tx * 4 + j;
            if (o < C && k < K) part[(size_t)o * K + k] = acc[i][j];
        }
    }
    if (k0 == 0 && tid < kHgTile && o0 + tid < C) part[(size_t)C * K + o0 + tid] = bsum;
}

// ------------------------------------------------------------------------------------------------------------------ host side
// act_input: layer 1 reads a (b*n, c_in) activation (a tensor-core layer like the others); tap: -1 or a hidden layer
bool frozen_encoder_ex_supported(int b, int n, int act_input, int nconv, const snb200_layer *conv, int np, int tap)
{
    if (b < 1 || b > 64 || n < 1 || n > 4096 || np < 1 || np > kMaxPrefix) return false;
    if (nconv < 2 || nconv > SNB200_MAX_CONV_LAYERS || tap < -1 || tap > nconv - 2) return false;
    if (act_input) {
        if (!tc_layer_supported(conv[0].c_in, conv[0].c_out)) return false;
    } else if (conv[0].c_in != 3 || conv[0].c_out % 8 != 0 || conv[0].c_out > kFeMaxHidden) {
        return false;
    }
    for (int l = 1; l < nconv - 1; l++)
        if (!tc_layer_supported(conv[l].c_in, conv[l].c_out)) return false;
    const snb200_layer &L = conv[nconv - 1];
    return L.c_in % 8 == 0 && L.c_in >= 8 && L.c_in <= kFeMaxHidden && L.c_out >= 8 && L.c_out <= kTcMaxLastOut;
}

bool frozen_encoder_supported(int b, int n, int nconv, const snb200_layer *conv, int np) { return frozen_encoder_ex_supported(b, n, 0, nconv, conv, np, -1); }

struct FrozenWorkspace { float *tile_val; int *tile_idx; float *bound_val; int *bound_idx; float *act[2]; size_t total; };

// one block of tile and boundary records (a value and a point index each), then without zsave two ping-pong buffers of the widest hidden layer
static FrozenWorkspace carve_frozen_ws(void *base, int b, int n, int nconv, const snb200_layer *conv, int np, bool with_zsave)
{
    FrozenWorkspace W;
    WsCarver c(base);
    const size_t C = conv[nconv - 1].c_out, tile_recs = (size_t)b * tc_tiles_per_cloud(n) * C, bound_recs = (size_t)np * b * C;
    W.tile_val = c.take<float>(2 * (tile_recs + bound_recs));
    W.tile_idx = reinterpret_cast<int *>(W.tile_val + tile_recs);
    W.bound_val = reinterpret_cast<float *>(W.tile_idx + tile_recs);
    W.bound_idx = reinterpret_cast<int *>(W.bound_val + bound_recs);
    int w = 0;
    for (int l = 0; l < nconv - 1; l++) w = max(w, conv[l].c_out);
    W.act[0] = with_zsave ? nullptr : c.take<float>((size_t)b * n * w);
    W.act[1] = with_zsave ? nullptr : c.take<float>((size_t)b * n * w);
    W.total = c.off;
    return W;
}

size_t frozen_encoder_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int np, int with_zsave)
{
    return carve_frozen_ws(nullptr, b, n, nconv, conv, np, with_zsave).total;
}

// the backward's workspace: the route bits; with parameter gradients then each hidden layer's dense dz rows and its chunk partials
struct FrozenBwdWorkspace { unsigned *bits; float *dz[SNB200_MAX_CONV_LAYERS]; float *part[SNB200_MAX_CONV_LAYERS]; int chunks, chunk_pts; size_t total; };

static FrozenBwdWorkspace carve_frozen_bwd_ws(void *base, int b, int n, int nconv, const snb200_layer *conv, bool params)
{
    FrozenBwdWorkspace W;
    memset(&W, 0, sizeof(W));
    WsCarver c(base);
    const long long pts = (long long)b * n;
    W.bits = c.take<unsigned>((size_t)pts * ((conv[nconv - 1].c_out + 31) / 32));
    W.chunks = (int)min(256ll, (pts + 255) / 256);     // at least 256 points per chunk, at most 256 chunks
    W.chunk_pts = (int)((pts + W.chunks - 1) / W.chunks);
    if (params)
        for (int l = 0; l < nconv - 1; l++) {
            W.dz[l] = c.take<float>((size_t)pts * conv[l].c_out);
            W.part[l] = c.take<float>((size_t)W.chunks * conv[l].c_out * (conv[l].c_in + 1));
        }
    W.total = c.off;
    return W;
}

size_t frozen_encoder_backward_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int, bool params)
{
    return carve_frozen_bwd_ws(nullptr, b, n, nconv, conv, params).total;
}

static FrozenZsave frozen_zsave(int nconv, float *const *zsave)
{
    FrozenZsave Z;
    memset(&Z, 0, sizeof(Z));
    for (int l = 0; l < nconv - 1; l++) Z.z[l] = zsave[l];
    return Z;
}

// The chain backward of the F.rows rows (points, or packed rows with segments): the route bits, then chain_bwd_kernel when it has something
// to write (grad_in, or D's dense dz rows).
static int launch_frozen_chain(const FrozenParams &F, const snb200_layer *conv, const float *pooled, const int *route, float *const *zsave,
                               const float *grad_pooled, unsigned *bits, const float *grad_tap, float *grad_in, const FrozenDz &D,
                               cudaStream_t stream)
{
    const int C = conv[F.nconv - 1].c_out, words = (C + 31) / 32;
    cudaMemsetAsync(bits, 0, (size_t)F.rows * words * sizeof(unsigned), stream);
    route_mark_kernel<<<(unsigned)(((long long)F.np * F.b * C + 255) / 256), 256, 0, stream>>>(F, pooled, route, bits, words);
    if (int rc = check_launch(F.seg ? "frozen encoder segment route marks" : "frozen encoder route marks")) return rc;
    if (!grad_in && !D.dz[0]) return SNB200_OK;
    size_t smem = (size_t)kFeWarps * 2 * kFeMaxHidden;
    for (int l = 0; l < F.nconv; l++) smem += 2 * (size_t)conv[l].c_out;
    smem *= sizeof(float);   // at most 8 * 512 + 2 * (7 * 256 + 1024) floats: 38 912 bytes, below the 48 KB default
    const long long blocks = (F.rows + kFeWarps - 1) / kFeWarps, cap = 16ll * num_sms();
    chain_bwd_kernel<<<(int)(blocks < cap ? blocks : cap), kFeWarps * 32, smem, stream>>>(F, pooled, route, grad_pooled, bits, words,
                                                                                         frozen_zsave(F.nconv, zsave), grad_tap, grad_in, D);
    return check_launch(F.seg ? "frozen encoder segment backward chain" : "frozen encoder backward chain");
}

// in: the cloud (b, n, 3), or with act_input the (b*n, c_in) activation layer 1 reads; tap_out: hidden layer tap's activation (tap >= 0)
int launch_frozen_encoder_forward(int b, int n, const float *in, int nconv, const snb200_layer *conv, int np, const int *sizes, float *pooled,
                                  int *route, float *const *zsave, void *workspace, cudaStream_t stream, int act_input, int tap, float *tap_out)
{
    const FrozenParams F = frozen_params(b, n, nconv, conv, np, sizes);
    const int C = conv[nconv - 1].c_out;
    const FrozenWorkspace W = carve_frozen_ws(workspace, b, n, nconv, conv, np, zsave != nullptr);
    // eval mode without statistics; the last layer leaves the prefix pool's records instead of its output
    if (int rc = launch_tc_stack(b, n, SNB200_BNC, act_input ? nullptr : in, nconv, conv, 0, nullptr, zsave, W.act,
                                 TcStackTail{nullptr, nullptr, np, sizes, W.bound_val, W.bound_idx, W.tile_val, W.tile_idx}, stream,
                                 act_input ? in : nullptr, tap, tap_out))
        return rc;
    prefix_combine_kernel<<<(b * C + 255) / 256, 256, 0, stream>>>(F, W.tile_val, W.tile_idx, W.bound_val, W.bound_idx, pooled, route);
    return check_launch("frozen encoder prefix combine");
}

// grad_x: (b, n, c_in of layer 1), or NULL with `grads`; tap >= 0: grad_tap (b*n, c_out_tap) is the gradient of that hidden layer's
// activation.  grads: per layer the weight / bias gradients to write (NULL pointers skipped; the workspace then holds the parameter part),
// or NULL; x is read for grads[0].weight.
int launch_frozen_encoder_backward(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, const float *pooled,
                                   const int *route, float *const *zsave, const float *grad_pooled, float *grad_x, void *workspace,
                                   cudaStream_t stream, int tap, const float *grad_tap, const float *x, const snb200_layer_grad *grads)
{
    const FrozenParams F = frozen_params(b, n, nconv, conv, np, sizes, tap);
    const int C = conv[nconv - 1].c_out;
    const FrozenBwdWorkspace W = carve_frozen_bwd_ws(workspace, b, n, nconv, conv, grads != nullptr);
    HiddenGradJobs J;
    memset(&J, 0, sizeof(J));
    J.chunks = W.chunks; J.chunk_pts = W.chunk_pts;
    ReduceParams R;
    memset(&R, 0, sizeof(R));
    FrozenDz D;
    memset(&D, 0, sizeof(D));
    for (int l = 0; grads && l < nconv - 1; l++) {
        if (!grads[l].weight && !grads[l].bias) continue;
        J.layer[J.njobs] = l; J.part[J.njobs] = W.part[l]; J.njobs++;
        ReduceJob &rj = R.job[R.njobs++];
        rj.part = W.part[l]; rj.nparts = W.chunks; rj.nw = conv[l].c_out * conv[l].c_in; rj.nb = conv[l].c_out;
        rj.g_weight = grads[l].weight; rj.g_bias = grads[l].bias;
    }
    if (J.njobs)
        for (int l = 0; l < nconv - 1; l++) D.dz[l] = W.dz[l];
    int rc = launch_frozen_chain(F, conv, pooled, route, zsave, grad_pooled, W.bits, grad_tap, grad_x, D, stream);
    if (rc) return rc;
    const FrozenZsave Z = frozen_zsave(nconv, zsave);
    const snb200_layer_grad *gl = grads ? grads + nconv - 1 : nullptr;
    if (gl && (gl->weight || gl->bias)) {
        last_grad_kernel<<<(C + kFeWarps - 1) / kFeWarps, kFeWarps * 32, 0, stream>>>(F, pooled, route, grad_pooled, Z, gl->weight, gl->bias);
        if ((rc = check_launch("frozen encoder backward: last layer parameters"))) return rc;
    }
    if (!J.njobs) return SNB200_OK;
    int tiles = 0;
    for (int j = 0; j < J.njobs; j++) {
        const snb200_layer &L = conv[J.layer[j]];
        tiles = max(tiles, ((L.c_out + kHgTile - 1) / kHgTile) * ((L.c_in + kHgTile - 1) / kHgTile));
    }
    hidden_grad_partial_kernel<<<dim3((unsigned)W.chunks, (unsigned)tiles, (unsigned)J.njobs), 256, 0, stream>>>(F, x, Z, D, J);
    if ((rc = check_launch("frozen encoder backward: hidden layer partials"))) return rc;
    return launch_reduce_partials(R, stream, "frozen encoder backward: hidden layer reduce");
}

// ------------------------------------------------------------------------------------------------------------------ many prefixes
// The _curve entries: the forward of the frozen encoder with a cloud input over up to n prefixes, every sample size of a progressive curve.
// The hidden layers run once as above; the last layer's epilogue reads the sizes from the workspace, where the call stages them with a
// table of each tile's first boundary (one host-to-device copy on the stream), and writes every boundary record straight into pooled /
// route.  curve_carry_kernel and curve_combine_kernel then finish them in place, so the workspace holds only the tile records.  The tie
// rule is prefix_combine_kernel's, so the results are bit for bit those of the 16-prefix entry.
bool frozen_encoder_curve_supported(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes)
{
    if (!sizes || np < 1 || !frozen_encoder_ex_supported(b, n, 0, nconv, conv, 1, -1) || np > n) return false;
    for (int p = 0; p < np; p++)
        if (sizes[p] < 1 || sizes[p] > n || (p > 0 && sizes[p] <= sizes[p - 1])) return false;
    return true;
}

// the tile records and the hidden layers' ping-pong buffers of carve_frozen_ws, then the staged sizes and per-tile first prefixes
struct CurveWorkspace { FrozenWorkspace F; int *sizes, *first; size_t total; };

static CurveWorkspace carve_curve_ws(void *base, int b, int n, int nconv, const snb200_layer *conv, int np)
{
    CurveWorkspace W;
    W.F = carve_frozen_ws(base, b, n, nconv, conv, 0, false);
    WsCarver c(base);
    c.off = W.F.total;
    W.sizes = c.take<int>((size_t)np + tc_tiles_per_cloud(n) + 1);
    W.first = W.sizes ? W.sizes + np : nullptr;
    W.total = c.off;
    return W;
}

size_t frozen_encoder_curve_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int np)
{
    return carve_curve_ws(nullptr, b, n, nconv, conv, np).total;
}

int launch_frozen_encoder_curve_forward(int b, int n, const float *x, int nconv, const snb200_layer *conv, int np, const int *sizes, float *pooled,
                                        int *route, void *workspace, cudaStream_t stream)
{
    const int C = conv[nconv - 1].c_out, tiles = tc_tiles_per_cloud(n);
    const CurveWorkspace W = carve_curve_ws(workspace, b, n, nconv, conv, np);
    // the sizes, then per tile t of a cloud the first prefix whose last point sizes[p] - 1 lies in tile t or later (tiles + 1 entries)
    std::vector<int> staged(sizes, sizes + np);
    for (int t = 0, p = 0; t <= tiles; t++) {
        while (p < np && (sizes[p] - 1) / kTcM < t) p++;
        staged.push_back(p);
    }
    // from pageable memory: the copy returns once the source has been taken, so `staged` may go out of scope
    if (cudaMemcpyAsync(W.sizes, staged.data(), staged.size() * sizeof(int), cudaMemcpyHostToDevice, stream) != cudaSuccess) {
        set_error("frozen encoder curve: staging the sizes failed: %s", cudaGetErrorString(cudaGetLastError()));
        return SNB200_ECUDA;
    }
    TcStackTail tail;
    memset(&tail, 0, sizeof(tail));
    tail.num_prefix = np; tail.sizes = W.sizes; tail.dev_first = W.first;
    tail.bound_val = pooled; tail.bound_idx = route; tail.tile_val = W.F.tile_val; tail.tile_idx = W.F.tile_idx;
    if (int rc = launch_tc_stack(b, n, SNB200_BNC, x, nconv, conv, 0, nullptr, nullptr, W.F.act, tail, stream)) return rc;
    curve_carry_kernel<<<(b * C + 255) / 256, 256, 0, stream>>>(b, tiles, C, W.F.tile_val, W.F.tile_idx);
    if (int rc = check_launch("frozen encoder curve carry")) return rc;
    FrozenParams F = frozen_params(b, n, nconv, conv, 0, nullptr);
    F.np = np;
    curve_combine_kernel<<<dim3((unsigned)(np * b), (unsigned)((C + 255) / 256)), 256, 0, stream>>>(F, W.sizes, W.F.tile_val, W.F.tile_idx, pooled,
                                                                                                     route);
    return check_launch("frozen encoder curve combine");
}

// ------------------------------------------------------------------------------------------------------------------ segments
// The _seg entries run the same kernels on a packed buffer of `total` rows holding num_seg segments (offset, length), each offset a multiple of
// kTcM (so no tile straddles two segments) and the segments in ascending offset order.  The hidden layers are row-local, so they run as one
// cloud of `total` points; only the last layer's epilogue (one record per tile), seg_combine_kernel and the backward's point -> segment map
// know about segments.
//   rows      total <= 2^22: an element offset of a (total, 256) hidden activation, the widest, stays below 2^31;
//   segments  each starts on its own tile, so num_seg <= ceil(total / 128) <= 2^15, and num_seg * C <= 2^25 threads in seg_combine_kernel;
//   length    max_len <= 4096, the frozen encoder's cloud size: a route is a row within its segment.
constexpr long long kFeSegMaxRows = 1ll << 22;
constexpr int kFeSegMaxLen = 4096;

bool frozen_encoder_seg_supported(int num_seg, int total, int max_len, int act_input, int nconv, const snb200_layer *conv, int tap)
{
    if (num_seg < 1 || total < 1 || total > kFeSegMaxRows || max_len < 1 || max_len > kFeSegMaxLen) return false;
    if ((long long)num_seg * kTcM > ((long long)total + kTcM - 1) / kTcM * kTcM) return false;
    return frozen_encoder_ex_supported(1, 1, act_input, nconv, conv, 1, tap);   // the layer table, as the _ex entries take it
}

size_t frozen_encoder_seg_workspace_bytes(int total, int nconv, const snb200_layer *conv, int with_zsave)
{
    return carve_frozen_ws(nullptr, 1, total, nconv, conv, 0, with_zsave).total;
}

size_t frozen_encoder_seg_backward_workspace_bytes(int total, int nconv, const snb200_layer *conv)
{
    return carve_frozen_bwd_ws(nullptr, 1, total, nconv, conv, false).total;
}

static FrozenParams frozen_seg_params(int num_seg, int total, const int2 *seg, int nconv, const snb200_layer *conv, int tap)
{
    FrozenParams F = frozen_params(num_seg, 0, nconv, conv, 0, nullptr, tap);
    F.np = 1; F.seg = seg; F.rows = total;
    return F;
}

int launch_frozen_encoder_seg_forward(int num_seg, int total, const int2 *seg, const float *in, int nconv, const snb200_layer *conv, float *pooled,
                                      int *route, float *const *zsave, void *workspace, cudaStream_t stream, int act_input, int tap, float *tap_out)
{
    const FrozenParams F = frozen_seg_params(num_seg, total, seg, nconv, conv, tap);
    const int C = conv[nconv - 1].c_out;
    const FrozenWorkspace W = carve_frozen_ws(workspace, 1, total, nconv, conv, 0, zsave != nullptr);
    TcStackTail tail;
    memset(&tail, 0, sizeof(tail));
    tail.tile_val = W.tile_val; tail.tile_idx = W.tile_idx; tail.seg = seg; tail.num_seg = num_seg;
    if (int rc = launch_tc_stack(1, total, SNB200_BNC, act_input ? nullptr : in, nconv, conv, 0, nullptr, zsave, W.act, tail, stream,
                                 act_input ? in : nullptr, tap, tap_out))
        return rc;
    seg_combine_kernel<<<(unsigned)(((long long)num_seg * C + 255) / 256), 256, 0, stream>>>(F, W.tile_val, W.tile_idx, pooled, route);
    return check_launch("frozen encoder segment combine");
}

int launch_frozen_encoder_seg_backward(int num_seg, int total, const int2 *seg, int nconv, const snb200_layer *conv, const float *pooled,
                                       const int *route, float *const *zsave, const float *grad_pooled, float *grad_in, void *workspace,
                                       cudaStream_t stream, int tap, const float *grad_tap)
{
    const FrozenParams F = frozen_seg_params(num_seg, total, seg, nconv, conv, tap);
    const FrozenBwdWorkspace W = carve_frozen_bwd_ws(workspace, 1, total, nconv, conv, false);
    FrozenDz D;
    memset(&D, 0, sizeof(D));
    return launch_frozen_chain(F, conv, pooled, route, zsave, grad_pooled, W.bits, grad_tap, grad_in, D, stream);
}

}  // namespace snb
