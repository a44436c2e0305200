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

// ------------------------------------------------------------------------------------------------------------------ segments
// Segment j of a packed buffer (offset off_j, a multiple of kPtRows, and length len_j; the rows up to the next multiple of kPtRows are its
// padding) multiplies its rows by its own T[j].  Its rows come from
//   prefix source (np > 0)  rows [0, len_j) of cloud j % src_b of an unpacked (src_b, src_n, k) input, segment j = p * src_b + b being prefix
//                           p of cloud b (len_j = sizes[p]): no prefix copy is materialised;
//   packed source (np = 0)  rows [off_j, off_j + len_j) of a packed (total, k) input laid out as the output.
// Every output element is the fmaf chain of the per-cloud kernels, so a row comes out as point_transform_fwd_kernel makes it.  The forward
// writes the padding rows as 0, as does the packed source's grad_in.  grad_T[j]: per chunk of kPtRows rows a partial (in packed tile
// off_j / kPtRows + chunk of the workspace), added in chunk order.  The prefix source's grad_in[b, i] is the sum over the prefixes p with
// sizes[p] > i, in ascending p, of grad_out[off_{p,b} + i] @ T[p,b]^T: one CTA owns each point, no atomics.
struct PtSegParams {
    const int2 *seg;
    int num_seg, k, src_b, src_n, np;
    int sizes[16];
};

__device__ __forceinline__ const float *pt_seg_source(const PtSegParams &S, const float *in, int j, int2 s, int i0)
{
    return S.np ? in + ((size_t)(j % S.src_b) * S.src_n + i0) * S.k : in + ((size_t)s.x + i0) * S.k;
}

__global__ void __launch_bounds__(kPtThreads) point_transform_seg_fwd_kernel(const __grid_constant__ PtSegParams S, const float *__restrict__ in,
                                                                             const float *__restrict__ T, float *__restrict__ out)
{
    extern __shared__ float s_pt[];
    const int k = S.k, j = blockIdx.x, i0 = blockIdx.y * kPtRows;
    const int2 s = S.seg[j];
    const int rows_pad = min(kPtRows, (s.y + kPtRows - 1) / kPtRows * kPtRows - i0), rows = min(kPtRows, s.y - i0);
    if (rows_pad <= 0) return;
    float *sT = s_pt, *sA = sT + k * (k + 1);
    pt_stage(k, rows, T + (size_t)j * k * k, pt_seg_source(S, in, j, s, i0), nullptr, sT, sA, nullptr);
    float *o = out + ((size_t)s.x + i0) * k;
    for (int e = threadIdx.x; e < rows_pad * k; e += kPtThreads) {
        const int r = e / k, c = e % k;
        float acc = 0.f;
        if (r < rows)
            for (int q = 0; q < k; q++) acc = fmaf(sA[r * k + q], sT[q * (k + 1) + c], acc);
        o[e] = acc;
    }
}

// per (segment, chunk): the partial grad_T, and for the packed source grad_in of the chunk's rows (padding 0)
__global__ void __launch_bounds__(kPtThreads) point_transform_seg_bwd_kernel(const __grid_constant__ PtSegParams S, const float *__restrict__ in,
                                                                             const float *__restrict__ T, const float *__restrict__ grad_out,
                                                                             float *__restrict__ grad_in, float *__restrict__ part)
{
    extern __shared__ float s_pt[];
    const int k = S.k, j = blockIdx.x, i0 = blockIdx.y * kPtRows;
    const int2 s = S.seg[j];
    const int rows_pad = min(kPtRows, (s.y + kPtRows - 1) / kPtRows * kPtRows - i0), rows = min(kPtRows, s.y - i0);
    if (rows_pad <= 0) return;
    float *sT = s_pt, *sA = sT + k * (k + 1), *sG = sA + kPtRows * k;
    const size_t base = ((size_t)s.x + i0) * k;
    pt_stage(k, rows, T + (size_t)j * k * k, pt_seg_source(S, in, j, s, i0), grad_out + base, sT, sA, sG);
    if (!S.np)
        for (int e = threadIdx.x; e < rows_pad * k; e += kPtThreads) {
            const int r = e / k, q = e % k;
            float acc = 0.f;
            if (r < rows)
                for (int c = 0; c < k; c++) acc = fmaf(sG[r * k + c], sT[q * (k + 1) + c], acc);
            grad_in[base + e] = acc;
        }
    float *dst = part + ((size_t)s.x / kPtRows + blockIdx.y) * k * k;
    for (int e = threadIdx.x; e < k * k; e += kPtThreads) {
        const int q = e / k, c = e % k;
        float acc = 0.f;
        for (int r = 0; r < rows; r++) acc = fmaf(sA[r * k + q], sG[r * k + c], acc);
        dst[e] = acc;
    }
}

__global__ void __launch_bounds__(kPtThreads) point_transform_seg_sum_kernel(const __grid_constant__ PtSegParams S, const float *__restrict__ part,
                                                                             float *__restrict__ gT)
{
    const int kk = S.k * S.k;
    const long long e = (long long)blockIdx.x * kPtThreads + threadIdx.x;
    if (e >= (long long)S.num_seg * kk) return;
    const int j = (int)(e / kk), q = (int)(e % kk);
    const int2 s = S.seg[j];
    const float *p = part + (size_t)(s.x / kPtRows) * kk + q;
    float acc = 0.f;
    for (int c = 0; c < (s.y + kPtRows - 1) / kPtRows; c++) acc += p[(size_t)c * kk];
    gT[e] = acc;
}

// prefix source: grad_in of kPtRows points of one cloud, the prefixes that hold them in ascending order
__global__ void __launch_bounds__(kPtThreads) point_transform_seg_prefix_grad_kernel(const __grid_constant__ PtSegParams S, const float *__restrict__ T,
                                                                                     const float *__restrict__ grad_out, float *__restrict__ grad_in)
{
    extern __shared__ float s_pt[];
    const int k = S.k, bi = blockIdx.y, i0 = blockIdx.x * kPtRows, rows = min(kPtRows, S.src_n - i0);
    float *sT = s_pt, *sG = sT + k * (k + 1), *sAcc = sG + kPtRows * k;
    for (int e = threadIdx.x; e < rows * k; e += kPtThreads) sAcc[e] = 0.f;   // each element stays with its thread throughout
    for (int p = 0; p < S.np; p++) {
        if (S.sizes[p] <= i0) continue;
        const int rp = min(rows, S.sizes[p] - i0), j = p * S.src_b + bi;
        __syncthreads();   // the previous prefix's operands are read
        pt_stage(k, rp, T + (size_t)j * k * k, grad_out + ((size_t)S.seg[j].x + i0) * k, nullptr, sT, sG, nullptr);
        for (int e = threadIdx.x; e < rp * k; e += kPtThreads) {
            const int r = e / k, q = e % k;
            float acc = 0.f;
            for (int c = 0; c < k; c++) acc = fmaf(sG[r * k + c], sT[q * (k + 1) + c], acc);
            sAcc[e] += acc;
        }
    }
    float *g = grad_in + ((size_t)bi * S.src_n + i0) * k;
    for (int e = threadIdx.x; e < rows * k; e += kPtThreads) g[e] = sAcc[e];
}

// Envelope: total <= 2^22 packed rows and segments of at most 4096 rows (the frozen encoder's _seg envelope), k <= 64; every segment starts
// on its own chunk of kPtRows rows, so num_seg <= ceil(total / kPtRows).  A prefix source has 1..16 prefixes of at most 65535 clouds
// (grid.y of the prefix gradient).
bool point_transform_seg_supported(int num_seg, int total, int max_len, int k)
{
    if (num_seg < 1 || total < 1 || total > (1 << 22) || max_len < 1 || max_len > 4096 || k < 1 || k > kPtMaxK) return false;
    return (long long)num_seg * kPtRows <= ((long long)total + kPtRows - 1) / kPtRows * kPtRows;
}

size_t point_transform_seg_workspace_bytes(int total, int k) { return align_up((size_t)pt_chunks(total) * k * k * sizeof(float), 256); }

static size_t pt_prefix_grad_smem_bytes(int k) { return sizeof(float) * ((size_t)k * (k + 1) + 2 * (size_t)kPtRows * k); }

static void pt_seg_attributes()
{
    static PerDeviceOnce once;
    if (once.first()) {
        cudaFuncSetAttribute(point_transform_seg_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pt_smem_bytes(kPtMaxK, false));
        cudaFuncSetAttribute(point_transform_seg_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pt_smem_bytes(kPtMaxK, true));
        cudaFuncSetAttribute(point_transform_seg_prefix_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)pt_prefix_grad_smem_bytes(kPtMaxK));
    }
}

static PtSegParams pt_seg_params(int num_seg, const int2 *seg, int k, int src_b, int src_n, int np, const int *sizes)
{
    PtSegParams S;
    memset(&S, 0, sizeof(S));
    S.seg = seg; S.num_seg = num_seg; S.k = k; S.np = np; S.src_b = np ? src_b : 0; S.src_n = np ? src_n : 0;
    for (int p = 0; p < np; p++) S.sizes[p] = sizes[p];
    return S;
}

int launch_point_transform_seg_forward(int num_seg, int max_len, const int2 *seg, int k, int src_b, int src_n, int np, const int *sizes,
                                       const float *in, const float *T, float *out, cudaStream_t stream)
{
    pt_seg_attributes();
    const PtSegParams S = pt_seg_params(num_seg, seg, k, src_b, src_n, np, sizes);
    point_transform_seg_fwd_kernel<<<dim3(num_seg, pt_chunks(max_len)), kPtThreads, pt_smem_bytes(k, false), stream>>>(S, in, T, out);
    return check_launch("point transform segments forward");
}

int launch_point_transform_seg_backward(int num_seg, int max_len, const int2 *seg, int k, int src_b, int src_n, int np, const int *sizes,
                                        const float *in, const float *T, const float *grad_out, float *grad_in, float *grad_T, void *workspace,
                                        cudaStream_t stream)
{
    pt_seg_attributes();
    const PtSegParams S = pt_seg_params(num_seg, seg, k, src_b, src_n, np, sizes);
    float *part = static_cast<float *>(workspace);
    point_transform_seg_bwd_kernel<<<dim3(num_seg, pt_chunks(max_len)), kPtThreads, pt_smem_bytes(k, true), stream>>>(S, in, T, grad_out, grad_in, part);
    if (int rc = check_launch("point transform segments backward")) return rc;
    point_transform_seg_sum_kernel<<<(unsigned)(((long long)num_seg * k * k + kPtThreads - 1) / kPtThreads), kPtThreads, 0, stream>>>(S, part, grad_T);
    if (int rc = check_launch("point transform segments backward sum")) return rc;
    if (!np) return SNB200_OK;
    point_transform_seg_prefix_grad_kernel<<<dim3(pt_chunks(src_n), src_b), kPtThreads, pt_prefix_grad_smem_bytes(k), stream>>>(S, T, grad_out, grad_in);
    return check_launch("point transform segments prefix gradient");
}

}  // namespace snb
