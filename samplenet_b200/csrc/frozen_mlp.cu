// frozen_mlp.cu -- a fully connected head without BatchNorm statistics applied to at most 64 rows, with the gradient to its input and
// optionally to its weights and biases (PCRNet's 2048-1024-1024-512-512-256-7 head behind the frozen encoder: registration/models/pcrnet.py:46-82,
// frozen while the sampler trains, trained in PCRNet's own run).
//
// The work is a skinny GEMM per layer: 16 MB of weights against <= 64 activation rows.  One launch per layer, chained on the stream by
// programmatic dependent launch (every kernel requests its first weights, then waits for the previous grid, then touches activations), so
// the layers need no host synchronisation and the next layer's CTAs are resident when the previous layer drains.  A cooperative
// single-launch design would need a grid barrier per layer and would pin the grid to one wave for the 4096-wide envelope; the per-layer
// launches keep each layer's own tiling.
//
//   forward  out[r, o] = act(bias[o] + sum_k in[r, k] W[o, k])
//       A CTA owns OT (8 or 4) output channels and all rows; W rows are read along k exactly once (cp.async, 16-byte granules, K tiles of
//       256 double buffered together with the matching activation tile).  Lanes split k, a thread holds an 8-row x OT tile of accumulators,
//       the warps are (row group, k split); the lanes' and k splits' partial sums are combined through shared memory in a fixed order.
//   backward grad_in[r, k] = sum_o (grad_out[r, o] * [a[r, o] > 0]) W[o, k]
//       The same row-major W is read in column slices of 32 floats: a warp's load of W[o, k0 .. k0 + 32) is one whole 128-byte segment, no
//       transposed copy exists.  Lane = column, a thread holds one accumulator per row, the warps split o; g = grad_out * mask is staged per
//       128 output channels and read back as broadcast float4.  When c_in / 32 column slices do not fill the machine the o range is split
//       over grid.y and each split writes its partial (b, c_in) block; the consumer (the next layer's staging, or the final reduce kernel)
//       adds the blocks in split order.  No float atomics anywhere: run to run bit-identical.
//   parameter gradients (snb200_frozen_mlp_param_backward: PCRNet trained)  dW[o, k] = sum_r g[r, o] a_{l-1}[r, k], db[o] = sum_r g[r, o]
//       An epilogue of the same kernel on the same staged g: the CTA keeps its own 32 columns of the layer input (`in` for layer 1, the
//       saved activation below otherwise) in shared memory behind the g tile; per staged step each warp walks its 16 output channels, a lane
//       sums its column over the rows in row order and the warp stores one whole 128-byte row segment of dW per channel.  db is summed the
//       same way by the CTAs of column slice 0.  Every dW / db element has one owner CTA; the grad_in arithmetic is unchanged.
// Eval-mode BatchNorm (the snb200_frozen_mlp_bn_* entries: the FC layers of PointNet's classifier and transform nets): the forward's epilogue
// is a = act(fmaf(z, scale, shift)) with scale / shift from the running statistics by bn_scale_shift, the conv layers' expression, evaluated
// from the layer's own parameters (nothing is folded into the weights); the backward stages g * [a > 0] * scale.
#include "encoder_internal.cuh"

namespace snb {

constexpr int kMlpThreads = 256;
constexpr int kMlpMaxRows = 64;
constexpr int kMlpMaxWidth = 4096;
constexpr int kMlpKT = 256;        // forward: input channels staged per step
constexpr int kMlpBwdCols = 32;    // backward: columns of W per CTA = one 128-byte segment per weight row
constexpr int kMlpBwdOC = 128;     // backward: output channels of g staged per step (16 per warp)
constexpr int kMlpMaxSplit = 8;

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src, int src_bytes)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(src_bytes) : "memory");   // the rest is zero-filled
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ------------------------------------------------------------------------------------------------------------------ forward
// the eval-mode BatchNorm of one layer (gamma == nullptr: none)
struct MlpBN {
    const float *gamma, *beta, *run_mean, *run_var;
    float eps;
};

__device__ __forceinline__ float mlp_bn_scale(const MlpBN &bn, int c_out, int o, float *shift)
{
    float sc, sh;
    bn_scale_shift(nullptr, c_out, o, 0.0, bn.gamma, bn.beta, bn.run_mean, bn.run_var, bn.eps, 0, sc, sh);
    if (shift) *shift = sh;
    return sc;
}

template <int OT>
__global__ void __launch_bounds__(kMlpThreads) frozen_mlp_forward_kernel(const float *__restrict__ in, const float *__restrict__ W, const float *__restrict__ bias,
                                                                         float *__restrict__ out, int b, int c_in, int c_out, int relu, int rgp,
                                                                         const __grid_constant__ MlpBN bn)
{
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rows = rgp * 8;                          // rgp: row groups of 8, a power of two (1, 2, 4, 8)
    const int stage = (rows + OT) * kMlpKT;            // floats of one stage: activations [rows][KT], then weights [OT][KT]
    const int o0 = (int)blockIdx.x * OT;
    const int rg = warp & (rgp - 1), ks = warp / rgp, KS = (kMlpThreads / 32) / rgp;
    const int nchunks = (c_in + kMlpKT - 1) / kMlpKT;
    constexpr int G = kMlpKT / 4;                      // 16-byte granules per staged row

    auto load_w = [&](int chunk, int s) {
        float *dst = sm + s * stage + rows * kMlpKT;
        for (int i = tid; i < OT * G; i += kMlpThreads) {
            const int o = i / G, k = chunk * kMlpKT + (i % G) * 4;
            const bool ok = (o0 + o < c_out) && (k < c_in);
            cp_async16(dst + o * kMlpKT + (i % G) * 4, ok ? W + (size_t)(o0 + o) * c_in + k : W, ok ? 16 : 0);
        }
    };
    auto load_a = [&](int chunk, int s) {
        float *dst = sm + s * stage;
        for (int i = tid; i < rows * G; i += kMlpThreads) {
            const int r = i / G, k = chunk * kMlpKT + (i % G) * 4;
            const bool ok = (r < b) && (k < c_in);
            cp_async16(dst + r * kMlpKT + (i % G) * 4, ok ? in + (size_t)r * c_in + k : in, ok ? 16 : 0);
        }
    };

    load_w(0, 0);                                             // the weights do not depend on the previous grid
    asm volatile("griddepcontrol.wait;" ::: "memory");        // ... the activations do; nothing is written to global memory before this
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    load_a(0, 0);
    cp_async_commit();

    float acc[8][OT];
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
        for (int o = 0; o < OT; o++) acc[r][o] = 0.f;

    for (int c = 0; c < nchunks; c++) {
        if (c + 1 < nchunks) {
            load_w(c + 1, (c + 1) & 1);
            load_a(c + 1, (c + 1) & 1);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float *A = sm + (c & 1) * stage + rg * 8 * kMlpKT;
        const float *B = sm + (c & 1) * stage + rows * kMlpKT;
        for (int j = ks; j < kMlpKT / 32; j += KS) {
            const int k = lane + 32 * j;
            float a[8], w[OT];
#pragma unroll
            for (int r = 0; r < 8; r++) a[r] = A[r * kMlpKT + k];
#pragma unroll
            for (int o = 0; o < OT; o++) w[o] = B[o * kMlpKT + k];
#pragma unroll
            for (int r = 0; r < 8; r++)
#pragma unroll
                for (int o = 0; o < OT; o++) acc[r][o] = fmaf(a[r], w[o], acc[r][o]);
        }
        __syncthreads();
    }
    // the lanes' (k mod 32) and the k splits' partial sums, added in a fixed order: thread t's tile at red[t][.] (odd stride: conflict-free)
    constexpr int T = 8 * OT;
    float *red = sm;
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
        for (int o = 0; o < OT; o++) red[tid * (T + 1) + r * OT + o] = acc[r][o];
    __syncthreads();
    for (int q = tid; q < rgp * T; q += kMlpThreads) {
        const int rgq = q / T, i = q % T;
        float s = 0.f;
        for (int sp = 0; sp < KS; sp++) {
            const float *src = red + (size_t)((rgq + rgp * sp) * 32) * (T + 1) + i;
#pragma unroll 8
            for (int l = 0; l < 32; l++) s += src[l * (T + 1)];
        }
        const int r = rgq * 8 + i / OT, o = o0 + i % OT;
        if (r < b && o < c_out) {
            s += bias ? __ldg(bias + o) : 0.f;
            if (bn.gamma) {
                float sh;
                const float sc = mlp_bn_scale(bn, c_out, o, &sh);
                s = fmaf(s, sc, sh);
            }
            out[(size_t)r * c_out + o] = relu ? fmaxf(s, 0.f) : s;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------ backward
struct MlpBwdParams {
    const float *g;          // (g_splits, b, c_out): the blocks are added in order; grad_out itself has one block
    const float *mask;       // (b, c_out) saved post-ReLU activation of this layer, or NULL (no ReLU)
    const float *W;          // (c_out, c_in)
    float *dst;              // (gridDim.y, b, c_in), or NULL: no input gradient (layer 1 of a call without grad_in)
    const float *act;        // (b, c_in) the layer's input, read when dW is set
    float *dW, *db;          // (c_out, c_in) / (c_out) parameter gradients, or NULL
    int g_splits, b, c_in, c_out, o_per_split;
    MlpBN bn;                // the gradient of z is g * mask * scale
};

template <int RB>
__global__ void __launch_bounds__(kMlpThreads) frozen_mlp_backward_kernel(const __grid_constant__ MlpBwdParams P)
{
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int col = (int)blockIdx.x * kMlpBwdCols + lane;
    const bool colok = col < P.c_in;
    const int oa = (int)blockIdx.y * P.o_per_split, ob = min(P.c_out, oa + P.o_per_split);
    constexpr int U = kMlpBwdOC / (kMlpThreads / 32);   // output channels per warp and step (16)

    auto load_w = [&](int oc, float *w) {
#pragma unroll
        for (int u = 0; u < U; u++) {
            const int o = oc + warp * U + u;
            w[u] = (colok && o < ob) ? __ldg(P.W + (size_t)o * P.c_in + col) : 0.f;     // the warp reads W[o, k0 .. k0 + 32): one 128-byte segment
        }
    };
    float wv[U], wn[U];
    load_w(oa, wv);                                           // the weights do not depend on the previous grid
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    float *sa = sm + RB * kMlpBwdOC;                          // the layer input's 32 columns of this CTA, [RB][32], behind the g tile
    if (P.dW)
        for (int i = tid; i < RB * kMlpBwdCols; i += kMlpThreads) {
            const int r = i / kMlpBwdCols, c = (int)blockIdx.x * kMlpBwdCols + i % kMlpBwdCols;
            sa[i] = (r < P.b && c < P.c_in) ? P.act[(size_t)r * P.c_in + c] : 0.f;
        }

    float acc[RB];
#pragma unroll
    for (int r = 0; r < RB; r++) acc[r] = 0.f;
    const size_t blk = (size_t)P.b * P.c_out;
    for (int oc = oa; oc < ob; oc += kMlpBwdOC) {
        for (int i = tid; i < RB * kMlpBwdOC; i += kMlpThreads) {
            const int r = i / kMlpBwdOC, o = oc + i % kMlpBwdOC;
            float v = 0.f;
            if (r < P.b && o < ob) {
                const size_t e = (size_t)r * P.c_out + o;
                for (int s = 0; s < P.g_splits; s++) v += P.g[s * blk + e];
                if (P.mask && !(P.mask[e] > 0.f)) v = 0.f;
                else if (P.bn.gamma) v *= mlp_bn_scale(P.bn, P.c_out, o, nullptr);
            }
            sm[i] = v;
        }
        __syncthreads();
        load_w(oc + kMlpBwdOC, wn);          // next step's weights in flight under this step's FMAs (zeros past the end of the range)
#pragma unroll
        for (int r = 0; r < RB; r++) {
            const float4 *g4 = reinterpret_cast<const float4 *>(sm + r * kMlpBwdOC + warp * U);
#pragma unroll
            for (int u4 = 0; u4 < U / 4; u4++) {
                const float4 gv = g4[u4];
                acc[r] = fmaf(gv.x, wv[u4 * 4 + 0], acc[r]);
                acc[r] = fmaf(gv.y, wv[u4 * 4 + 1], acc[r]);
                acc[r] = fmaf(gv.z, wv[u4 * 4 + 2], acc[r]);
                acc[r] = fmaf(gv.w, wv[u4 * 4 + 3], acc[r]);
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) wv[u] = wn[u];
        if (P.dW) {      // dW[o, k0 .. k0 + 32) of the warp's 16 channels, the rows summed in row order
#pragma unroll 1
            for (int u = 0; u < U; u++) {
                const int o = oc + warp * U + u;
                const float *gc = sm + warp * U + u;
                float s = 0.f;
                for (int r = 0; r < P.b; r++) s = fmaf(gc[r * kMlpBwdOC], sa[r * kMlpBwdCols + lane], s);
                if (colok && o < ob) P.dW[(size_t)o * P.c_in + col] = s;
            }
        }
        if (P.db && blockIdx.x == 0 && lane < U) {
            const int o = oc + warp * U + lane;
            float s = 0.f;
            for (int r = 0; r < P.b; r++) s += sm[r * kMlpBwdOC + warp * U + lane];
            if (o < ob) P.db[o] = s;
        }
        __syncthreads();
    }
    if (!P.dst) return;
    // the warps' partial sums (each over its own output channels), added in warp order
    float *red = sm;
#pragma unroll
    for (int r = 0; r < RB; r++) red[(warp * RB + r) * 32 + lane] = acc[r];
    __syncthreads();
    float *dst = P.dst + (size_t)blockIdx.y * P.b * P.c_in;
    for (int i = tid; i < RB * 32; i += kMlpThreads) {
        const int r = i / 32, l = i % 32, c = (int)blockIdx.x * kMlpBwdCols + l;
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < kMlpThreads / 32; w++) s += red[(w * RB + r) * 32 + l];
        if (r < P.b && c < P.c_in) dst[(size_t)r * P.c_in + c] = s;
    }
}

__global__ void __launch_bounds__(kMlpThreads) frozen_mlp_sum_splits_kernel(const float *__restrict__ parts, int splits, int count, float *__restrict__ out)
{
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int i = (int)blockIdx.x * kMlpThreads + (int)threadIdx.x;
    if (i >= count) return;
    float s = 0.f;
    for (int p = 0; p < splits; p++) s += parts[(size_t)p * count + i];
    out[i] = s;
}

// ------------------------------------------------------------------------------------------------------------------ host
// allow_bn: eval-mode BatchNorm on any layer (the snb200_frozen_mlp_bn_* entries)
bool frozen_mlp_supported(int b, int nl, const snb200_layer *L, bool allow_bn)
{
    if (b < 1 || b > kMlpMaxRows || nl < 1 || nl > SNB200_MAX_FC_LAYERS || !L) return false;
    for (int l = 0; l < nl; l++) {
        if (L[l].c_in < 8 || L[l].c_in > kMlpMaxWidth || (L[l].c_in % 8) != 0) return false;
        if (L[l].c_out < 1 || L[l].c_out > kMlpMaxWidth) return false;
        if (!allow_bn && (L[l].bn_weight || L[l].bn_bias)) return false;
        if (l > 0 && L[l].c_in != L[l - 1].c_out) return false;
    }
    return !L[nl - 1].relu;     // the last layer's output is not saved, so there is no mask to take a ReLU's gradient from
}

static MlpBN mlp_bn(const snb200_layer &L) { return MlpBN{L.bn_weight, L.bn_bias, L.bn_running_mean, L.bn_running_var, L.bn_eps}; }

static int mlp_row_groups(int b)
{
    int rgp = 1;
    while (rgp * 8 < b) rgp *= 2;
    return rgp;
}

static int mlp_fwd_ot(int c_out) { return (c_out + 7) / 8 >= kNumSMs * 3 / 4 ? 8 : 4; }

// how many blocks the output channels of layer l's backward are split into (grid.y), and the channels per block (a multiple of the staging step)
static void mlp_bwd_split(const snb200_layer &L, int *splits, int *o_per_split)
{
    const int slices = (L.c_in + kMlpBwdCols - 1) / kMlpBwdCols;
    int s = max(1, min(kMlpMaxSplit, kNumSMs / slices));
    int per = (int)align_up((size_t)(L.c_out + s - 1) / s, kMlpBwdOC);
    *o_per_split = per;
    *splits = (L.c_out + per - 1) / per;
}

// hidden activations of a forward without `asave`: one (b, c_out_l) buffer per hidden layer (distinct buffers: a layer's output is never
// overwritten while an earlier launch may still read it)
static size_t mlp_fwd_carve(void *base, int b, int nl, const snb200_layer *L, float **hidden)
{
    WsCarver ws(base);
    for (int l = 0; l < nl - 1; l++) {
        float *p = ws.take<float>((size_t)b * L[l].c_out);
        if (hidden) hidden[l] = p;
    }
    return ws.off;
}
size_t frozen_mlp_workspace_bytes(int b, int nl, const snb200_layer *L, int with_save) { return with_save ? 0 : mlp_fwd_carve(nullptr, b, nl, L, nullptr); }

// per layer l the (splits_l, b, c_in_l) blocks of its input gradient (layer 0 writes grad_in directly when it is not split)
static size_t mlp_bwd_carve(void *base, int b, int nl, const snb200_layer *L, float **parts)
{
    WsCarver ws(base);
    for (int l = 0; l < nl; l++) {
        int s, per;
        mlp_bwd_split(L[l], &s, &per);
        float *p = (l == 0 && s == 1) ? nullptr : ws.take<float>((size_t)s * b * L[l].c_in);
        if (parts) parts[l] = p;
    }
    return ws.off > 0 ? ws.off : 256;
}
size_t frozen_mlp_backward_workspace_bytes(int b, int nl, const snb200_layer *L) { return mlp_bwd_carve(nullptr, b, nl, L, nullptr); }

template <class... KArgs, class... Args>
static int mlp_launch(const char *what, void (*kernel)(KArgs...), dim3 grid, size_t smem, cudaStream_t stream, Args... args)
{
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid; cfg.blockDim = dim3(kMlpThreads); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;   // may be scheduled while the previous layer drains; it waits for it itself
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, args...);
    if (e != cudaSuccess) { set_error("%s: launch failed: %s", what, cudaGetErrorString(e)); cudaGetLastError(); return SNB200_ECUDA; }
    return check_launch(what);
}

static size_t mlp_fwd_smem(int rgp, int ot) { return sizeof(float) * (size_t)max(2 * (rgp * 8 + ot) * kMlpKT, kMlpThreads * (8 * ot + 1)); }

int launch_frozen_mlp_forward(int b, const float *in, int nl, const snb200_layer *L, float *out, float *const *asave, void *workspace, cudaStream_t stream)
{
    static PerDeviceOnce once;
    if (once.first()) {
        cudaFuncSetAttribute(frozen_mlp_forward_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mlp_fwd_smem(8, 8));
        cudaFuncSetAttribute(frozen_mlp_forward_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mlp_fwd_smem(8, 4));
    }
    float *hidden[SNB200_MAX_FC_LAYERS] = {};
    if (asave) for (int l = 0; l < nl - 1; l++) hidden[l] = asave[l];
    else mlp_fwd_carve(workspace, b, nl, L, hidden);
    const int rgp = mlp_row_groups(b);
    const float *src = in;
    for (int l = 0; l < nl; l++) {
        float *dst = l == nl - 1 ? out : hidden[l];
        const int ot = mlp_fwd_ot(L[l].c_out);
        const dim3 grid((unsigned)((L[l].c_out + ot - 1) / ot));
        const int rc = mlp_launch("frozen_mlp_forward", ot == 8 ? frozen_mlp_forward_kernel<8> : frozen_mlp_forward_kernel<4>, grid, mlp_fwd_smem(rgp, ot),
                                  stream, src, L[l].weight, L[l].bias, dst, b, L[l].c_in, L[l].c_out, L[l].relu, rgp, mlp_bn(L[l]));
        if (rc) return rc;
        src = dst;
    }
    return SNB200_OK;
}

// grads: per layer the weight / bias gradients to write (NULL pointers skipped), or NULL for none; `in` is read only for grads[0].weight.
// grad_in may be NULL when grads asks for something.
int launch_frozen_mlp_backward(int b, int nl, const snb200_layer *L, float *const *asave, const float *grad_out, float *grad_in, void *workspace,
                               cudaStream_t stream, const float *in, const snb200_layer_grad *grads)
{
    static PerDeviceOnce once;
    if (once.first()) cudaFuncSetAttribute(frozen_mlp_backward_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    float *parts[SNB200_MAX_FC_LAYERS] = {};
    mlp_bwd_carve(workspace, b, nl, L, parts);
    const int rb = mlp_row_groups(b) * 8;
    const float *g = grad_out;
    int g_splits = 1;
    for (int l = nl - 1; l >= 0; l--) {
        MlpBwdParams P;
        int s;
        mlp_bwd_split(L[l], &s, &P.o_per_split);
        P.g = g; P.g_splits = g_splits; P.mask = L[l].relu ? asave[l] : nullptr; P.W = L[l].weight;
        P.dst = parts[l] ? parts[l] : grad_in;
        P.act = l == 0 ? in : asave[l - 1];
        P.dW = grads ? grads[l].weight : nullptr; P.db = grads ? grads[l].bias : nullptr;
        P.b = b; P.c_in = L[l].c_in; P.c_out = L[l].c_out; P.bn = mlp_bn(L[l]);
        const dim3 grid((unsigned)((L[l].c_in + kMlpBwdCols - 1) / kMlpBwdCols), (unsigned)s);
        const size_t smem = (size_t)rb * 1024;      // max(g tile rb x 128 + input columns rb x 32, warp partials 8 x rb x 32) floats
        void (*kernel)(MlpBwdParams) = rb == 8 ? frozen_mlp_backward_kernel<8> : rb == 16 ? frozen_mlp_backward_kernel<16>
                                       : rb == 32 ? frozen_mlp_backward_kernel<32> : frozen_mlp_backward_kernel<64>;
        if (int rc = mlp_launch("frozen_mlp_backward", kernel, grid, smem, stream, P)) return rc;
        g = P.dst; g_splits = s;
    }
    if (parts[0] && grad_in) {
        const int count = b * L[0].c_in;
        return mlp_launch("frozen_mlp_backward", frozen_mlp_sum_splits_kernel, dim3((unsigned)((count + kMlpThreads - 1) / kMlpThreads)), 0, stream,
                          (const float *)parts[0], g_splits, count, grad_in);
    }
    return SNB200_OK;
}

}  // namespace snb
