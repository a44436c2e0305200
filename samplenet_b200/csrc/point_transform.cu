// point_transform.cu -- a per-cloud K x K transform of points or point features, and its backward (PointNet's input and feature transforms:
// classification/models/pointnet_cls.py `tf.matmul(point_cloud, transform)`: rows times T).
//
//   forward   out[b, i, :] = in[b, i, :] @ T[b]                         K <= 64
//   backward  grad_in[b, i, :] = grad_out[b, i, :] @ T[b]^T
//             grad_T[b] = sum_i in[b, i, :]^T grad_out[b, i, :]
//
// A CTA owns kPtRows points of one cloud and stages them with T[b] (row stride K + 1: the backward reads T along its rows from consecutive
// threads) in shared memory; every output is one thread's fmaf chain in ascending index order.  The backward's CTA also forms its chunk's
// partial grad_T (one thread per entry, its points in order); with more than one chunk per cloud the partials go to the workspace and a
// second kernel adds them in chunk order.  No float atomics: run to run bit-identical.
// Folding T into per-cloud conv weights is not done: it would break the 128-point tensor-core tiles of the following layer for small clouds.
#include "common.cuh"

namespace snb {

constexpr int kPtThreads = 256;
constexpr int kPtRows = 128;      // points per CTA
constexpr int kPtMaxK = 64;

static size_t pt_smem_bytes(int k, bool backward) { return sizeof(float) * ((size_t)k * (k + 1) + (size_t)(backward ? 2 : 1) * kPtRows * k); }

// T[b] into sT (stride k + 1) and rows [i0, i0 + rows) of the (n, k) matrices a (and g) into sA (and sG)
__device__ __forceinline__ void pt_stage(int k, int rows, const float *T, const float *a, const float *g, float *sT, float *sA, float *sG)
{
    for (int e = threadIdx.x; e < k * k; e += kPtThreads) sT[(e / k) * (k + 1) + e % k] = T[e];
    for (int e = threadIdx.x; e < rows * k; e += kPtThreads) {
        sA[e] = a[e];
        if (g) sG[e] = g[e];
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kPtThreads) point_transform_fwd_kernel(int n, int k, const float *__restrict__ in, const float *__restrict__ T,
                                                                         float *__restrict__ out)
{
    extern __shared__ float s_pt[];
    const int bi = blockIdx.y, i0 = blockIdx.x * kPtRows, rows = min(kPtRows, n - i0);
    float *sT = s_pt, *sA = sT + k * (k + 1);
    const size_t base = ((size_t)bi * n + i0) * k;
    pt_stage(k, rows, T + (size_t)bi * k * k, in + base, nullptr, sT, sA, nullptr);
    for (int e = threadIdx.x; e < rows * k; e += kPtThreads) {
        const int r = e / k, j = e % k;
        float acc = 0.f;
        for (int q = 0; q < k; q++) acc = fmaf(sA[r * k + q], sT[q * (k + 1) + j], acc);
        out[base + e] = acc;
    }
}

// grad_in of the CTA's points, and its chunk's partial grad_T: to gT (b, k, k) directly when the cloud is one chunk, else to
// part (b, chunks, k, k)
__global__ void __launch_bounds__(kPtThreads) point_transform_bwd_kernel(int n, int k, const float *__restrict__ in, const float *__restrict__ T,
                                                                         const float *__restrict__ grad_out, float *__restrict__ grad_in,
                                                                         float *__restrict__ gT, float *__restrict__ part)
{
    extern __shared__ float s_pt[];
    const int bi = blockIdx.y, i0 = blockIdx.x * kPtRows, rows = min(kPtRows, n - i0);
    float *sT = s_pt, *sA = sT + k * (k + 1), *sG = sA + kPtRows * k;
    const size_t base = ((size_t)bi * n + i0) * k;
    pt_stage(k, rows, T + (size_t)bi * k * k, in + base, grad_out + base, sT, sA, sG);
    for (int e = threadIdx.x; e < rows * k; e += kPtThreads) {
        const int r = e / k, q = e % k;
        float acc = 0.f;
        for (int j = 0; j < k; j++) acc = fmaf(sG[r * k + j], sT[q * (k + 1) + j], acc);
        grad_in[base + e] = acc;
    }
    float *dst = gridDim.x == 1 ? gT + (size_t)bi * k * k : part + ((size_t)bi * gridDim.x + blockIdx.x) * k * k;
    for (int e = threadIdx.x; e < k * k; e += kPtThreads) {
        const int q = e / k, j = e % k;
        float acc = 0.f;
        for (int r = 0; r < rows; r++) acc = fmaf(sA[r * k + q], sG[r * k + j], acc);
        dst[e] = acc;
    }
}

__global__ void __launch_bounds__(kPtThreads) point_transform_sum_kernel(int b, int chunks, int kk, const float *__restrict__ part, float *__restrict__ gT)
{
    const int e = blockIdx.x * kPtThreads + threadIdx.x;
    if (e >= b * kk) return;
    const int bi = e / kk, q = e % kk;
    const float *p = part + (size_t)bi * chunks * kk + q;
    float s = 0.f;
    for (int c = 0; c < chunks; c++) s += p[(size_t)c * kk];
    gT[e] = s;
}

// ------------------------------------------------------------------------------------------------------------------ host
bool point_transform_supported(int b, int n, int k) { return b >= 1 && b <= 65535 && n >= 1 && n <= (1 << 24) && k >= 1 && k <= kPtMaxK; }

static int pt_chunks(int n) { return (n + kPtRows - 1) / kPtRows; }

size_t point_transform_workspace_bytes(int b, int n, int k)
{
    const int c = pt_chunks(n);
    return c == 1 ? 0 : align_up((size_t)b * c * k * k * sizeof(float), 256);
}

static void pt_attributes()
{
    static PerDeviceOnce once;
    if (once.first()) {
        cudaFuncSetAttribute(point_transform_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pt_smem_bytes(kPtMaxK, false));
        cudaFuncSetAttribute(point_transform_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pt_smem_bytes(kPtMaxK, true));
    }
}

int launch_point_transform_forward(int b, int n, int k, const float *in, const float *T, float *out, cudaStream_t stream)
{
    pt_attributes();
    point_transform_fwd_kernel<<<dim3(pt_chunks(n), b), kPtThreads, pt_smem_bytes(k, false), stream>>>(n, k, in, T, out);
    return check_launch("point transform forward");
}

int launch_point_transform_backward(int b, int n, int k, const float *in, const float *T, const float *grad_out, float *grad_in, float *grad_T,
                                    void *workspace, cudaStream_t stream)
{
    pt_attributes();
    const int chunks = pt_chunks(n);
    float *part = static_cast<float *>(workspace);
    point_transform_bwd_kernel<<<dim3(chunks, b), kPtThreads, pt_smem_bytes(k, true), stream>>>(n, k, in, T, grad_out, grad_in, grad_T, part);
    if (int rc = check_launch("point transform backward")) return rc;
    if (chunks == 1) return SNB200_OK;
    point_transform_sum_kernel<<<(b * k * k + kPtThreads - 1) / kPtThreads, kPtThreads, 0, stream>>>(b, chunks, k * k, part, grad_T);
    return check_launch("point transform backward sum");
}

}  // namespace snb
