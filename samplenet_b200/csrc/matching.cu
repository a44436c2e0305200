// matching.cu -- inference-time matching on the GPU: order-preserving unique of the nearest-neighbour indices followed by
// farthest-point-sampling completion.
//
// Reference behaviour restated (not ported): registration/src/samplenet.py:119-141 copies x, y and idx to the host,
// runs numpy per cloud (sputils.py:7-41: np.unique(return_index) + a Python FPS loop in float64) and copies the result
// back -- two PCIe round trips and a device sync per batch.  Here one CTA per cloud does the same arithmetic (float64
// distances, first-maximum arg-max, first-occurrence unique) out of shared memory; nothing leaves the device.
#include "common.cuh"

namespace snb {

constexpr int kMatchThreads = 512;

// numpy's ((p0 - points) ** 2).sum(axis=1): every square and both sums rounded, left to right.  Written with explicit intrinsics:
// `dx * dx + dy * dy + dz * dz` is contracted by nvcc into fma(dz, dz, fma(dy, dy, dx * dx)), which breaks numpy's exact ties (a point
// and its x<->y mirror are equidistant from a seed on the diagonal in numpy, not under the contraction) and so moves the FPS completion.
__device__ __forceinline__ double dist2_numpy(double dx, double dy, double dz)
{
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// np.argmax's order: does candidate (a, ai) come before the running (b, bi)?  The first NaN wins, then the first maximum.  Every point
// beats the initial (-1, INT_MAX) of a thread without points, so the index read back is always one of the cloud's.
__device__ __forceinline__ bool argmax_before(double a, int ai, double b, int bi)
{
    if (a != a) return b == b || ai < bi;
    return b == b && (a > b || (a == b && ai < bi));
}

__global__ void __launch_bounds__(kMatchThreads) nn_matching_kernel(int n, int t, int k, const float *__restrict__ full_pc,
                                                                    const int *__restrict__ nn_idx, int complete_fps, float *__restrict__ out,
                                                                    int *__restrict__ out_idx)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // layout: double dmin[n]; int first_pos[n]; int sel[k]; reduction scratch
    double *dmin = reinterpret_cast<double *>(smem_raw);
    int *first_pos = reinterpret_cast<int *>(dmin + n);
    int *sel = first_pos + n;
    __shared__ double s_rv[kMatchThreads / 32];
    __shared__ int s_ri[kMatchThreads / 32];
    __shared__ int s_count;
    __shared__ int s_scan[kMatchThreads];

    const int bi = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float *pc = full_pc + (size_t)bi * n * 3;
    const int *idx = nn_idx + (size_t)bi * t;
    float *o = out + (size_t)bi * k * 3;

    if (!complete_fps) {  // sputils.py:40: plain gather of the first k indices
        for (int i = tid; i < k; i += kMatchThreads) {
            const int ii = idx[i];
            o[i * 3 + 0] = pc[ii * 3 + 0]; o[i * 3 + 1] = pc[ii * 3 + 1]; o[i * 3 + 2] = pc[ii * 3 + 2];
            if (out_idx) out_idx[(size_t)bi * k + i] = ii;
        }
        return;
    }

    // ---- _unique (sputils.py:26-28): keep first occurrences, in order of first occurrence
    for (int p = tid; p < n; p += kMatchThreads) first_pos[p] = 0x7fffffff;
    __syncthreads();
    for (int i = tid; i < t; i += kMatchThreads) atomicMin(&first_pos[idx[i]], i);
    __syncthreads();
    // ordered compaction of {i : first_pos[idx[i]] == i} by a block-wide scan over chunks of kMatchThreads entries
    if (tid == 0) s_count = 0;
    __syncthreads();
    for (int i0 = 0; i0 < t; i0 += kMatchThreads) {
        const int i = i0 + tid;
        const int flag = (i < t && first_pos[idx[i]] == i) ? 1 : 0;
        s_scan[tid] = flag;
        __syncthreads();
        for (int off = 1; off < kMatchThreads; off <<= 1) {  // Hillis-Steele inclusive scan
            const int v = (tid >= off) ? s_scan[tid - off] : 0;
            __syncthreads();
            s_scan[tid] += v;
            __syncthreads();
        }
        const int base = s_count;
        if (flag) {
            const int pos = base + s_scan[tid] - 1;
            if (pos < k) sel[pos] = idx[i];
        }
        __syncthreads();
        if (tid == 0) s_count = base + s_scan[kMatchThreads - 1];
        __syncthreads();
    }
    const int nseed = min(s_count, k);

    // ---- distances to the seeds (sputils.py:15-17), float64 like numpy's promotion of float32 - float64
    for (int p = tid; p < n; p += kMatchThreads) {
        const double px = pc[p * 3 + 0], py = pc[p * 3 + 1], pz = pc[p * 3 + 2];
        double best = 0.0;
        for (int i = 0; i < nseed; i++) {
            const int si = sel[i];
            const double dx = (double)pc[si * 3 + 0] - px, dy = (double)pc[si * 3 + 1] - py, dz = (double)pc[si * 3 + 2] - pz;
            const double d = dist2_numpy(dx, dy, dz);
            if (i == 0 || d < best || d != d) best = d;   // np.minimum: a NaN propagates
        }
        dmin[p] = best;
    }
    __syncthreads();

    // ---- FPS completion (sputils.py:19-22): np.argmax returns the FIRST maximum
    for (int i = nseed; i < k; i++) {
        double bv = -1.0;
        int bidx = 0x7fffffff;
        for (int p = tid; p < n; p += kMatchThreads) {
            const double v = dmin[p];
            if (v > bv || (v != v && bv == bv)) { bv = v; bidx = p; }  // ascending p per thread: first maximum (first NaN) within the thread
        }
        for (int off = 16; off > 0; off >>= 1) {
            const double ov = __shfl_xor_sync(kFullMask, bv, off);
            const int oi = __shfl_xor_sync(kFullMask, bidx, off);
            if (argmax_before(ov, oi, bv, bidx)) { bv = ov; bidx = oi; }
        }
        if (lane == 0) { s_rv[warp] = bv; s_ri[warp] = bidx; }
        __syncthreads();
        if (tid == 0) {
            double v = s_rv[0];
            int ix = s_ri[0];
            for (int w = 1; w < kMatchThreads / 32; w++)
                if (argmax_before(s_rv[w], s_ri[w], v, ix)) { v = s_rv[w]; ix = s_ri[w]; }
            sel[i] = ix;
        }
        __syncthreads();
        const int si = sel[i];
        const double sx = pc[si * 3 + 0], sy = pc[si * 3 + 1], sz = pc[si * 3 + 2];
        for (int p = tid; p < n; p += kMatchThreads) {
            const double dx = sx - (double)pc[p * 3 + 0], dy = sy - (double)pc[p * 3 + 1], dz = sz - (double)pc[p * 3 + 2];
            const double d = dist2_numpy(dx, dy, dz);
            if (d < dmin[p] || d != d) dmin[p] = d;
        }
        __syncthreads();
    }
    for (int i = tid; i < k; i += kMatchThreads) {
        const int si = sel[i];
        o[i * 3 + 0] = pc[si * 3 + 0]; o[i * 3 + 1] = pc[si * 3 + 1]; o[i * 3 + 2] = pc[si * 3 + 2];
        if (out_idx) out_idx[(size_t)bi * k + i] = si;
    }
}

int launch_nn_matching(int b, int n, int t, int k, const float *full_pc, const int *nn_idx, int complete_fps, float *out, int *out_idx,
                       cudaStream_t stream)
{
    const size_t smem = (size_t)n * sizeof(double) + (size_t)n * sizeof(int) + (size_t)k * sizeof(int);
    if (smem > 200 * 1024) { set_error("nn_matching: cloud of %d points does not fit the shared-memory working set", n); return SNB200_EUNSUPPORTED; }
    static PerDeviceOnce once;
    if (once.first()) cudaFuncSetAttribute(nn_matching_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    nn_matching_kernel<<<b, kMatchThreads, smem, stream>>>(n, t, k, full_pc, nn_idx, complete_fps, out, out_idx);
    return check_launch("nn_matching");
}

}  // namespace snb
