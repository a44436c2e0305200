// encoder.cu -- SampleNet generator: per-point MLP (1x1 conv + BatchNorm + ReLU stack) on the CUDA cores, and the stand-alone
// encoder / FC-head entry points.
//
// Reference behaviour restated (not ported): registration/src/samplenet.py:90-104 runs, per layer, a cuDNN/cuBLAS conv,
// a BatchNorm kernel and a ReLU kernel, each round-tripping the (B,C,N) activation tensor; then torch.max and four
// Linear+BN+ReLU triples.  reconstruction/src/samplers.py:22-36 and classification/models/samplenet_model.py:31-108 are the
// same stack with other widths / BN epsilon.
//
// This file is the exact-fp32 CUDA-core path (every product and sum in fp32, like the reference's CPU path):
//   * one launch per conv layer.  The layer kernel applies the PREVIOUS layer's BatchNorm + ReLU while it loads its input
//     tile (so normalised activations never exist in memory), multiplies by the weight tile out of shared memory with an
//     8x8 register tile per thread, adds the bias, writes the raw (pre-BN) output once, and accumulates the per-channel
//     sum / sum-of-squares that training-mode BatchNorm needs (fp32 inside the tile, fp64 atomics across tiles);
//   * the last conv layer never writes its activation: it only emits per-tile max / min of the raw output, from which
//     max_n relu(bn(y)) follows exactly because the BN affine map is monotone per channel;
//   * the pool and the FC head are the generator's cluster head (fc_head_cluster_kernel, generator.cu): the stand-alone
//     snb200_encoder_forward runs it with no FC layers, snb200_fc_head_forward with no pool.
// The wgmma tensor-core variant of the conv stack lives in encoder_tc.cu.
#include "encoder_internal.cuh"

namespace snb {

constexpr int kEncThreads = 256;
constexpr int kEncKC = 32;  // K chunk staged in shared memory per step

struct ConvLayerParams {
    // input: either the cloud itself (first layer) or the previous layer's raw output (points-major, `c_in` wide)
    const float *in;
    long long in_cloud_stride;  // floats between consecutive clouds
    int in_stride_p, in_stride_c;
    int c_in, c_out;
    int b, n, tiles_per_cloud;
    // BatchNorm + ReLU of the PREVIOUS layer, applied on load (nullptrs => identity)
    const double *in_stats;        // [2][c_in] sum, sumsq over b*n positions (training) or nullptr
    const float *in_gamma, *in_beta, *in_run_mean, *in_run_var;
    float in_eps;
    int in_relu, in_has_bn, in_training;
    // this layer
    const float *weight, *bias;    // (c_out, c_in), (c_out)
    float *out;                    // raw output (b*n, c_out) or nullptr for the last layer
    double *out_stats;             // [2][c_out] or nullptr (no BN after this layer / eval mode)
    float *tile_max, *tile_min;    // (b*tiles_per_cloud, c_out) or nullptr
};

// CC = output channels per CTA (64 or 128); thread tile 8 points x 8 channels; TP = points per CTA.
template <int CC>
__global__ void __launch_bounds__(kEncThreads) conv_layer_kernel(const __grid_constant__ ConvLayerParams P)
{
    constexpr int TXN = CC / 8;             // threads along channels
    constexpr int TYN = kEncThreads / TXN;  // threads along points
    constexpr int TP = TYN * 8;             // points per CTA: 256 (CC=64) or 128 (CC=128)
    extern __shared__ __align__(16) float smem[];
    float *sA = smem;                        // [kEncKC][TP]
    float *sW = sA + kEncKC * TP;            // [kEncKC][CC]
    float *sScale = sW + kEncKC * CC;        // [c_in]
    float *sShift = sScale + P.c_in;         // [c_in]
    float *sRed = sShift + P.c_in;           // [TYN][CC] (epilogue reductions)

    const int tid = threadIdx.x;
    const int tx = tid % TXN, ty = tid / TXN;
    const int tile = blockIdx.x;
    const int cloud = tile / P.tiles_per_cloud;
    const int p0 = (tile % P.tiles_per_cloud) * TP;
    const int np = min(TP, P.n - p0);
    const int c0 = blockIdx.y * CC;
    const int c_in = P.c_in;

    // ---- prologue: BatchNorm(+ReLU) of the previous layer as a per-channel affine map
    for (int c = tid; c < c_in; c += kEncThreads) {
        float sc = 1.f, sh = 0.f;
        if (P.in_has_bn)
            bn_scale_shift(P.in_stats, c_in, c, (double)P.b * (double)P.n, P.in_gamma, P.in_beta, P.in_run_mean, P.in_run_var, P.in_eps,
                           P.in_training, sc, sh);
        sScale[c] = sc;
        sShift[c] = sh;
    }
    __syncthreads();

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i][j] = 0.f;

    const float *in_cloud = P.in + (size_t)cloud * P.in_cloud_stride;
    for (int k0 = 0; k0 < c_in; k0 += kEncKC) {
        const int kn = min(kEncKC, c_in - k0);
        // A tile: sA[k][p] = relu(bn(in[p][k0+k])), zero for p >= np.  lane -> point (conflict-free stores).
        for (int e = tid; e < kEncKC * TP; e += kEncThreads) {
            const int p = e % TP, k = e / TP;
            float v = 0.f;
            if (p < np && k < kn) {
                v = __ldg(in_cloud + (size_t)(p0 + p) * P.in_stride_p + (size_t)(k0 + k) * P.in_stride_c);
                v = fmaf(v, sScale[k0 + k], sShift[k0 + k]);
                if (P.in_relu) v = fmaxf(v, 0.f);
            }
            sA[k * TP + p] = v;
        }
        // W tile: sW[k][c] = W[c0+c][k0+k] (row-major (c_out, c_in)).  Lanes run along c so the transposed store is
        // bank-conflict free; the strided global reads stay in L1/L2 (the whole weight matrix is <= 128 KB).
        for (int e = tid; e < kEncKC * CC; e += kEncThreads) {
            const int c = e % CC, k = e / CC;
            float v = 0.f;
            if (k < kn && c0 + c < P.c_out) v = __ldg(P.weight + (size_t)(c0 + c) * c_in + k0 + k);
            sW[k * CC + c] = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int k = 0; k < kn; k++) {
            const float4 a0 = *reinterpret_cast<const float4 *>(sA + k * TP + ty * 8);
            const float4 a1 = *reinterpret_cast<const float4 *>(sA + k * TP + ty * 8 + 4);
            const float4 w0 = *reinterpret_cast<const float4 *>(sW + k * CC + tx * 8);
            const float4 w1 = *reinterpret_cast<const float4 *>(sW + k * CC + tx * 8 + 4);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int j = 0; j < 8; j++) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
        }
        __syncthreads();
    }

    // ---- epilogue: bias, raw store, statistics, per-tile extrema
    float bias[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int c = c0 + tx * 8 + j;
        bias[j] = (c < P.c_out) ? __ldg(P.bias + c) : 0.f;
    }
    float s[8], ss[8], mx[8], mn[8];
#pragma unroll
    for (int j = 0; j < 8; j++) { s[j] = 0.f; ss[j] = 0.f; mx[j] = -INFINITY; mn[j] = INFINITY; }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int p = ty * 8 + i;
        const bool pv = p < np;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const float v = acc[i][j] + bias[j];
            acc[i][j] = v;
            if (pv) { s[j] += v; ss[j] = fmaf(v, v, ss[j]); mx[j] = fmaxf(mx[j], v); mn[j] = fminf(mn[j], v); }
        }
        if (P.out && pv) {
            float *o = P.out + ((size_t)cloud * P.n + p0 + p) * P.c_out + c0 + tx * 8;
            if (c0 + tx * 8 + 8 <= P.c_out && (P.c_out & 3) == 0) {
                *reinterpret_cast<float4 *>(o) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
                *reinterpret_cast<float4 *>(o + 4) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
            } else {
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (c0 + tx * 8 + j < P.c_out) o[j] = acc[i][j];
            }
        }
    }
    // cross-thread reductions over the TYN point groups, fixed order
    if (P.out_stats) {
#pragma unroll
        for (int j = 0; j < 8; j++) sRed[ty * CC + tx * 8 + j] = s[j];
        __syncthreads();
        if (tid < CC && c0 + tid < P.c_out) {
            float t = 0.f;
            for (int r = 0; r < TYN; r++) t += sRed[r * CC + tid];
            atomicAdd(P.out_stats + c0 + tid, (double)t);
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; j++) sRed[ty * CC + tx * 8 + j] = ss[j];
        __syncthreads();
        if (tid < CC && c0 + tid < P.c_out) {
            float t = 0.f;
            for (int r = 0; r < TYN; r++) t += sRed[r * CC + tid];
            atomicAdd(P.out_stats + P.c_out + c0 + tid, (double)t);
        }
        __syncthreads();
    }
    if (P.tile_max) {
#pragma unroll
        for (int j = 0; j < 8; j++) sRed[ty * CC + tx * 8 + j] = mx[j];
        __syncthreads();
        if (tid < CC && c0 + tid < P.c_out) {
            float t = -INFINITY;
            for (int r = 0; r < TYN; r++) t = fmaxf(t, sRed[r * CC + tid]);
            P.tile_max[(size_t)tile * P.c_out + c0 + tid] = t;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; j++) sRed[ty * CC + tx * 8 + j] = mn[j];
        __syncthreads();
        if (tid < CC && c0 + tid < P.c_out) {
            float t = INFINITY;
            for (int r = 0; r < TYN; r++) t = fminf(t, sRed[r * CC + tid]);
            P.tile_min[(size_t)tile * P.c_out + c0 + tid] = t;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
static int enc_tp(int c_out) { return c_out > 64 ? 128 : 256; }
int simt_tiles_per_cloud(int n, int c_last) { return (n + enc_tp(c_last) - 1) / enc_tp(c_last); }

struct EncWorkspace {
    float *act[2];
    double *stats[SNB200_MAX_CONV_LAYERS];
    float *tile_max, *tile_min;
    size_t stats_bytes;
    char *stats_base;
    size_t total;
};

static EncWorkspace carve_encoder_ws(void *base, int b, int n, int num_layers, const snb200_layer *layers)
{
    EncWorkspace W;
    WsCarver c(base);
    int maxc = 0;
    for (int l = 0; l + 1 < num_layers; l++) maxc = max(maxc, layers[l].c_out);
    W.act[0] = c.take<float>((size_t)b * n * maxc);
    W.act[1] = c.take<float>((size_t)b * n * maxc);
    const size_t stats_off = c.off;
    for (int l = 0; l < num_layers; l++) W.stats[l] = c.take<double>((size_t)2 * layers[l].c_out);
    W.stats_base = reinterpret_cast<char *>(W.stats[0]);
    W.stats_bytes = c.off - stats_off;
    const int c_last = layers[num_layers - 1].c_out;
    const int tpc = simt_tiles_per_cloud(n, c_last);
    W.tile_max = c.take<float>((size_t)b * tpc * c_last);
    W.tile_min = c.take<float>((size_t)b * tpc * c_last);
    W.total = c.off;
    return W;
}

size_t encoder_workspace_bytes(int b, int n, int num_layers, const snb200_layer *layers)
{
    return carve_encoder_ws(nullptr, b, n, num_layers, layers).total;
}

int launch_simt_conv_stack(int b, int n, int layout, const float *x, int num_layers, const snb200_layer *layers, int training, float *act0,
                           float *act1, double *const *stats, float *tile_max, float *tile_min, cudaStream_t stream)
{
    float *act[2] = {act0, act1};
    for (int l = 0; l < num_layers; l++) {
        const snb200_layer &L = layers[l];
        ConvLayerParams P;
        memset(&P, 0, sizeof(P));
        P.b = b; P.n = n; P.c_in = L.c_in; P.c_out = L.c_out;
        if (l == 0) {
            P.in = x;
            P.in_cloud_stride = (long long)n * 3;
            P.in_stride_p = layout == SNB200_BNC ? 3 : 1;
            P.in_stride_c = layout == SNB200_BNC ? 1 : n;
            P.in_has_bn = 0; P.in_relu = 0;
        } else {
            const snb200_layer &Lp = layers[l - 1];
            P.in = act[(l - 1) & 1];
            P.in_cloud_stride = (long long)n * Lp.c_out;
            P.in_stride_p = Lp.c_out; P.in_stride_c = 1;
            P.in_has_bn = Lp.bn_weight != nullptr;
            P.in_stats = stats[l - 1];
            P.in_gamma = Lp.bn_weight; P.in_beta = Lp.bn_bias; P.in_run_mean = Lp.bn_running_mean; P.in_run_var = Lp.bn_running_var;
            P.in_eps = Lp.bn_eps; P.in_relu = Lp.relu; P.in_training = training;
        }
        P.weight = L.weight; P.bias = L.bias;
        const bool last = (l == num_layers - 1);
        P.out = last ? nullptr : act[l & 1];
        P.out_stats = (training && L.bn_weight) ? stats[l] : nullptr;
        P.tile_max = last ? tile_max : nullptr;
        P.tile_min = last ? tile_min : nullptr;
        const int CC = L.c_out > 64 ? 128 : 64;
        const int TP = enc_tp(L.c_out);
        P.tiles_per_cloud = simt_tiles_per_cloud(n, L.c_out);
        dim3 grid(b * P.tiles_per_cloud, (L.c_out + CC - 1) / CC);
        const int TYN = kEncThreads / (CC / 8);
        const size_t smem = ((size_t)kEncKC * TP + (size_t)kEncKC * CC + 2 * (size_t)L.c_in + (size_t)TYN * CC) * sizeof(float);
        static PerDeviceOnce attr_once;
        if (attr_once.first()) {
            cudaFuncSetAttribute(conv_layer_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
            cudaFuncSetAttribute(conv_layer_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        }
        if (smem > 100 * 1024) { set_error("encoder: layer %d too wide for the shared-memory tile (c_in=%d)", l, L.c_in); return SNB200_EUNSUPPORTED; }
        if (CC == 64) conv_layer_kernel<64><<<grid, kEncThreads, smem, stream>>>(P);
        else conv_layer_kernel<128><<<grid, kEncThreads, smem, stream>>>(P);
        int rc = check_launch("encoder conv layer");
        if (rc) return rc;
    }
    return SNB200_OK;
}

int launch_encoder_forward(int b, int n, int layout, const float *x, int num_layers, const snb200_layer *layers, int training, float *feat,
                           void *workspace, cudaStream_t stream)
{
    EncWorkspace W = carve_encoder_ws(workspace, b, n, num_layers, layers);
    if (training) cudaMemsetAsync(W.stats_base, 0, W.stats_bytes, stream);
    int rc0 = launch_simt_conv_stack(b, n, layout, x, num_layers, layers, training, W.act[0], W.act[1], W.stats, W.tile_max, W.tile_min, stream);
    if (rc0) return rc0;
    HeadParams H{};
    fill_pool_params(H, b, n, simt_tiles_per_cloud(n, layers[num_layers - 1].c_out), num_layers, layers, training, W.stats, W.tile_max,
                     W.tile_min, feat);
    return launch_fc_head_cluster(H, stream);
}

struct FcHeadWorkspace { float *buf[2]; size_t total; };   // ping-pong hidden layers

static FcHeadWorkspace carve_fc_head_ws(void *base, int b, int num_layers, const snb200_layer *layers)
{
    FcHeadWorkspace W;
    WsCarver c(base);
    int maxc = 1;
    for (int l = 0; l + 1 < num_layers; l++) maxc = max(maxc, layers[l].c_out);
    W.buf[0] = c.take<float>((size_t)b * maxc);
    W.buf[1] = c.take<float>((size_t)b * maxc);
    W.total = c.off;
    return W;
}

size_t fc_head_workspace_bytes(int b, int num_layers, const snb200_layer *layers)
{
    return carve_fc_head_ws(nullptr, b, num_layers, layers).total;
}

int launch_fc_head_forward(int b, const float *in, int num_layers, const snb200_layer *layers, int training, float *out, int out_transpose_inner,
                           void *workspace, cudaStream_t stream)
{
    if ((layers[0].c_in & 3) == 0 && (reinterpret_cast<uintptr_t>(in) & 15) != 0) {   // the head reads such rows as float4
        set_error("fc_head_forward: input of %d channels must be 16-byte aligned", layers[0].c_in);
        return SNB200_EINVAL;
    }
    const FcHeadWorkspace W = carve_fc_head_ws(workspace, b, num_layers, layers);
    HeadParams H{};
    H.b = b; H.training = training;
    H.feat = const_cast<float *>(in);   // tile_max stays null: the FC layers read `in`, nothing is pooled
    fill_fc_params(H, num_layers, layers, out, out_transpose_inner);
    H.act[0] = W.buf[0]; H.act[1] = W.buf[1];
    return launch_fc_head_cluster(H, stream);
}

}  // namespace snb
