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
#include "encoder_internal.cuh"

namespace snb {

constexpr int kFeMaxPrefix = 16;
constexpr int kFeTile = 128;          // points per tile of the tensor-core layer kernels (kTcM)
constexpr int kFeMaxHidden = 256;     // widest hidden layer (tc_layer_supported)
constexpr int kFeWarps = 8;           // chain_bwd_kernel: one point per warp at a time

struct FrozenLayer {
    const float *weight, *gamma, *beta, *run_mean, *run_var;
    float eps;
    int c_in, c_out, has_bn, relu;
};

struct FrozenParams {
    int b, n, nconv, np, tiles;
    int sizes[kFeMaxPrefix];
    FrozenLayer L[SNB200_MAX_CONV_LAYERS];
};

struct FrozenZsave {
    const float *z[SNB200_MAX_CONV_LAYERS];   // raw outputs of the hidden layers, (b * n, c_out_l)
};

static FrozenParams frozen_params(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes)
{
    FrozenParams F;
    memset(&F, 0, sizeof(F));
    F.b = b; F.n = n; F.nconv = nconv; F.np = np; F.tiles = (n + kFeTile - 1) / kFeTile;
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
        const int last = (F.sizes[p] - 1) / kFeTile;
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
    const int i = route[e];
    atomicOr(bits + ((size_t)bi * F.n + i) * words + (c >> 5), 1u << (c & 31));
}

// ---- backward 2: one warp per point, every step in a fixed order
__global__ void __launch_bounds__(kFeWarps * 32) chain_bwd_kernel(const __grid_constant__ FrozenParams F, const float *__restrict__ pooled,
                                                                  const int *__restrict__ route, const float *__restrict__ grad_pooled,
                                                                  const unsigned *__restrict__ bits, int words,
                                                                  const __grid_constant__ FrozenZsave Z, float *__restrict__ grad_x)
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
    const int C = LL.c_out, K = LL.c_in;
    const float *sc_last = s_fe + off[F.nconv - 1];
    for (long long pt = (long long)blockIdx.x * kFeWarps + warp; pt < (long long)F.b * F.n; pt += (long long)gridDim.x * kFeWarps) {
        const int bi = (int)(pt / F.n), i = (int)(pt % F.n);
        const unsigned word = lane < words ? bits[pt * words + lane] : 0u;
        if (!__any_sync(kFullMask, word != 0u)) {
            if (lane < 3) grad_x[pt * 3 + lane] = 0.f;
            continue;
        }
        // last layer: dA_{L-1}[k] = sum over the point's channels c (ascending) of D_c W_L[c, k], D_c = sum over prefixes p routed here
        // (ascending) of g[p,b,c] * scale_c
        for (int k = lane; k < K; k += 32) dA[k] = 0.f;
        __syncwarp();
        for (int w = 0; w < words; w++) {
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
        for (int l = F.nconv - 2; l >= 0; l--) {
            const FrozenLayer &L = F.L[l];
            const float *sc = s_fe + off[l], *sh = sc + L.c_out;
            const float *zr = Z.z[l] + pt * L.c_out;
            for (int k = lane; k < L.c_out; k += 32) {
                const bool on = !L.relu || fmaf(zr[k], sc[k], sh[k]) > 0.f;
                dz[k] = on ? dA[k] * sc[k] : 0.f;
            }
            __syncwarp();
            if (l > 0) {
                for (int j = lane; j < L.c_in; j += 32) {
                    float a = 0.f;
                    for (int k = 0; k < L.c_out; k++) a = fmaf(dz[k], __ldg(L.weight + (size_t)k * L.c_in + j), a);
                    dA[j] = a;
                }
            } else if (lane < 3) {
                float a = 0.f;
                for (int k = 0; k < L.c_out; k++) a = fmaf(dz[k], __ldg(L.weight + (size_t)k * 3 + lane), a);
                grad_x[pt * 3 + lane] = a;
            }
            __syncwarp();
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------ host side
bool frozen_encoder_supported(int b, int n, int nconv, const snb200_layer *conv, int np)
{
    if (b < 1 || b > 64 || n < 1 || n > 4096 || np < 1 || np > kFeMaxPrefix) return false;
    if (nconv < 2 || nconv > SNB200_MAX_CONV_LAYERS || conv[0].c_in != 3) return false;
    if (conv[0].c_out % 8 != 0 || conv[0].c_out > kFeMaxHidden) return false;
    for (int l = 1; l < nconv - 1; l++)
        if (!tc_layer_supported(conv[l].c_in, conv[l].c_out)) return false;
    const snb200_layer &L = conv[nconv - 1];
    return L.c_in % 8 == 0 && L.c_in >= 8 && L.c_in <= kFeMaxHidden && L.c_out >= 8 && L.c_out <= kTcMaxLastOut;
}

struct FrozenWorkspace { float *tile_val; int *tile_idx; float *bound_val; int *bound_idx; float *act[2]; size_t total; };

// one block of tile and boundary records (a value and a point index each), then without zsave two ping-pong buffers of the widest hidden layer
static FrozenWorkspace carve_frozen_ws(void *base, int b, int n, int nconv, const snb200_layer *conv, int np, bool with_zsave)
{
    FrozenWorkspace W;
    WsCarver c(base);
    const size_t C = conv[nconv - 1].c_out, tile_recs = (size_t)b * ((n + kFeTile - 1) / kFeTile) * C, bound_recs = (size_t)np * b * C;
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

size_t frozen_encoder_backward_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int)
{
    return align_up((size_t)b * n * ((conv[nconv - 1].c_out + 31) / 32) * sizeof(unsigned), 256);
}

int launch_frozen_encoder_forward(int b, int n, const float *x, int nconv, const snb200_layer *conv, int np, const int *sizes, float *pooled,
                                  int *route, float *const *zsave, void *workspace, cudaStream_t stream)
{
    const FrozenParams F = frozen_params(b, n, nconv, conv, np, sizes);
    const int C = conv[nconv - 1].c_out;
    const FrozenWorkspace W = carve_frozen_ws(workspace, b, n, nconv, conv, np, zsave != nullptr);
    // eval mode without statistics; the last layer leaves the prefix pool's records instead of its output
    if (int rc = launch_tc_stack(b, n, SNB200_BNC, x, nconv, conv, 0, nullptr, zsave, W.act,
                                 TcStackTail{nullptr, nullptr, np, sizes, W.bound_val, W.bound_idx, W.tile_val, W.tile_idx}, stream))
        return rc;
    prefix_combine_kernel<<<(b * C + 255) / 256, 256, 0, stream>>>(F, W.tile_val, W.tile_idx, W.bound_val, W.bound_idx, pooled, route);
    return check_launch("frozen encoder prefix combine");
}

int launch_frozen_encoder_backward(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, const float *pooled,
                                   const int *route, float *const *zsave, const float *grad_pooled, float *grad_x, void *workspace,
                                   cudaStream_t stream)
{
    const FrozenParams F = frozen_params(b, n, nconv, conv, np, sizes);
    const int C = conv[nconv - 1].c_out, words = (C + 31) / 32;
    unsigned *bits = static_cast<unsigned *>(workspace);
    cudaMemsetAsync(bits, 0, (size_t)b * n * words * sizeof(unsigned), stream);
    route_mark_kernel<<<(np * b * C + 255) / 256, 256, 0, stream>>>(F, pooled, route, bits, words);
    int rc = check_launch("frozen encoder route marks");
    if (rc) return rc;
    FrozenZsave Z;
    memset(&Z, 0, sizeof(Z));
    for (int l = 0; l < nconv - 1; l++) Z.z[l] = zsave[l];
    size_t smem = (size_t)kFeWarps * 2 * kFeMaxHidden;
    for (int l = 0; l < nconv; l++) smem += 2 * (size_t)conv[l].c_out;
    smem *= sizeof(float);   // at most 8 * 512 + 2 * (7 * 256 + 1024) floats: 38 912 bytes, below the 48 KB default
    const long long pts = (long long)b * n;
    const long long blocks = (pts + kFeWarps - 1) / kFeWarps, cap = 16ll * num_sms();
    const int grid = (int)(blocks < cap ? blocks : cap);
    chain_bwd_kernel<<<grid, kFeWarps * 32, smem, stream>>>(F, pooled, route, grad_pooled, bits, words, Z, grad_x);
    return check_launch("frozen encoder backward chain");
}

}  // namespace snb
