// fps.cu -- farthest point sampling (tf_sampling's FarthestPointSample), one CTA per cloud, optionally fused with the gather of the
// selected coordinates.
//
// Contract: the same indices as farthestpointsamplingKernel (reconstruction/external/sampling/tf_sampling_g.cu:105-170):
//   idx[0] = 0, running minimum starts at 1e38f;
//   round j: d_k = fma(dz, dz, fma(dx, dx, dy*dy)) with d? = p_k.? - p_sel.? (the contraction nvcc gives the reference kernel),
//            dmin_k = fminf(d_k, dmin_k), select the largest dmin;
//   ties: the reference's 512 threads scan their points k = t, t + 512, ... keeping a candidate on strict '>', and its tree keeps the lower
//         slot unless strictly smaller, so among equal maxima the smallest (k mod 512, k div 512) wins.  Here that order is the tie rank
//         ((k & 511) << 5) | (k >> 9) (n <= 16384, so k >> 9 < 32).
//
// Design (DESIGN.md 4.3): the op is m-1 strictly dependent rounds, so its cost is the latency of one round.  The reference pays a global
// read-modify-write of its `temp` array per point and a 9-level shared-memory tree with 10 barriers per round, on a fixed grid of 32 CTAs
// (two waves at B = 50).  Here:
//   * grid = b: every cloud has its own CTA and all clouds run in one wave (B <= 132 on an H100 SXM);
//   * each thread keeps the running minimum of its P points in registers, and their coordinates too (P <= 8) or, for large clouds, in shared
//     memory as structure-of-arrays (conflict-free: consecutive threads read consecutive points);
//   * each warp reduces (distance bits, tie rank) with two redux.sync (non-negative floats order like their bit patterns), the winning lane
//     writes (bits, rank) and its coordinates into a per-warp slot of a double-buffered array indexed by the round's parity;
//   * ONE __syncthreads per round; after it every warp reduces the slots itself, so every thread knows the winner and its coordinates
//     without a second barrier or a global read.  Double buffering makes the single barrier sufficient: the slots a warp writes in round j+1
//     were last read in round j-1, before every warp arrived at round j's barrier.
// Within a thread the points are visited in ascending tie rank, so a strict '>' keeps the reference's winner without comparing ranks.
#include "common.cuh"

namespace snb {

constexpr int kFpsMaxPoints = 16384;
constexpr int kFpsRegMaxPPT = 8;   // up to 8 points per thread keep their coordinates in registers; more read them from shared memory

// the j-th point a thread visits (k = t + jj * T), ordered so that its tie ranks ascend.  For T >= 512, jj = j: k & 511 is fixed per thread
// and k >> 9 grows with j.  For T < 512 a thread owns R = 512 / T residues mod 512 (t, t + T, ...): visit all points of the first residue
// (ascending k >> 9), then the next.
template <int T, int P>
__device__ __forceinline__ constexpr int fps_visit(int j)
{
    constexpr int R = T >= 512 ? 1 : 512 / T;
    constexpr int I = P >= R ? P / R : 1;
    return (R == 1 || P < R) ? j : (j / I) + R * (j % I);
}

__device__ __forceinline__ int fps_rank(int k) { return ((k & 511) << 5) | (k >> 9); }

template <int T, int P, bool kSmemXYZ>
__global__ void __launch_bounds__(T) fps_kernel(int n, int m, int layout, const float *__restrict__ inp, int *__restrict__ idx,
                                                float *__restrict__ out_points)
{
    constexpr int NW = T / 32;
    static_assert(NW <= 32, "one lane per warp slot");
    extern __shared__ __align__(16) float s_xyz[];  // kSmemXYZ: x[n], y[n], z[n]
    __shared__ int2 s_key[2][NW];                   // (distance bits, tie rank) of each warp's winner, by round parity
    __shared__ float4 s_pt[2][NW];                  // its coordinates

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t cloud = blockIdx.x;
    const float *pc = inp + cloud * (size_t)n * 3;
    int *oi = idx + cloud * (size_t)m;
    float *op = out_points ? out_points + cloud * (size_t)m * 3 : nullptr;
    // coordinate c of point k in the caller's layout
    auto ld = [&](int k, int c) { return layout == SNB200_BNC ? __ldg(pc + (size_t)k * 3 + c) : __ldg(pc + (size_t)c * n + k); };
    auto st = [&](int j, float x, float y, float z) {
        if (layout == SNB200_BNC) { op[(size_t)j * 3 + 0] = x; op[(size_t)j * 3 + 1] = y; op[(size_t)j * 3 + 2] = z; }
        else { op[j] = x; op[(size_t)m + j] = y; op[2 * (size_t)m + j] = z; }
    };

    float px[kSmemXYZ ? 1 : P], py[kSmemXYZ ? 1 : P], pz[kSmemXYZ ? 1 : P];
    float dmin[P];
#pragma unroll
    for (int j = 0; j < P; j++) {
        const int k = tid + fps_visit<T, P>(j) * T;
        dmin[j] = k < n ? 1e38f : -1.0f;  // padding never wins: its bits are a negative int below the initial best of -1
        if (!kSmemXYZ) {
            px[j] = k < n ? ld(k, 0) : 0.f; py[j] = k < n ? ld(k, 1) : 0.f; pz[j] = k < n ? ld(k, 2) : 0.f;
        }
    }
    if (kSmemXYZ) {
        for (int k = tid; k < n; k += T) { s_xyz[k] = ld(k, 0); s_xyz[n + k] = ld(k, 1); s_xyz[2 * n + k] = ld(k, 2); }
        __syncthreads();
    }
    float sx = ld(0, 0), sy = ld(0, 1), sz = ld(0, 2);
    if (tid == 0) {
        oi[0] = 0;
        if (op) st(0, sx, sy, sz);
    }

    for (int r = 1; r < m; r++) {
        int bb = -1, bk = 0;
        float bx = 0.f, by = 0.f, bz = 0.f;
#pragma unroll
        for (int j = 0; j < P; j++) {
            const int k = tid + fps_visit<T, P>(j) * T;
            float x, y, z;
            if (kSmemXYZ) {
                const int kk = k < n ? k : 0;
                x = s_xyz[kk]; y = s_xyz[n + kk]; z = s_xyz[2 * n + kk];
            } else {
                x = px[j]; y = py[j]; z = pz[j];
            }
            const float dx = __fsub_rn(x, sx), dy = __fsub_rn(y, sy), dz = __fsub_rn(z, sz);
            const float d = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
            dmin[j] = fminf(d, dmin[j]);
            const int bits = __float_as_int(dmin[j]);
            if (bits > bb) { bb = bits; bk = k; bx = x; by = y; bz = z; }
        }
        // warp winner: largest distance, then smallest tie rank
        const int wb = __reduce_max_sync(kFullMask, bb);
        const int wr = __reduce_min_sync(kFullMask, bb == wb ? fps_rank(bk) : 0x7fffffff);
        const int par = r & 1;
        // one lane (tie ranks are distinct per point), or every lane of a warp that holds only padding, all writing the same (-1, 0)
        if (bb == wb && fps_rank(bk) == wr) {
            s_key[par][warp] = make_int2(wb, wr);
            s_pt[par][warp] = make_float4(bx, by, bz, 0.f);
        }
        __syncthreads();
        // CTA winner, reduced by every warp on its own
        const int2 key = lane < NW ? s_key[par][lane] : make_int2(-2, 0x7fffffff);
        const int cb = __reduce_max_sync(kFullMask, key.x);
        const int cr = __reduce_min_sync(kFullMask, key.x == cb ? key.y : 0x7fffffff);
        const int src = __ffs(__ballot_sync(kFullMask, key.x == cb && key.y == cr)) - 1;
        float4 w = lane < NW ? s_pt[par][lane] : make_float4(0.f, 0.f, 0.f, 0.f);
        sx = __shfl_sync(kFullMask, w.x, src); sy = __shfl_sync(kFullMask, w.y, src); sz = __shfl_sync(kFullMask, w.z, src);
        if (tid == 0) {
            oi[r] = ((cr & 31) << 9) | (cr >> 5);
            if (op) st(r, sx, sy, sz);
        }
    }
}

// Threads per CTA by cloud size, chosen by measurement (tools/bench_sampling.py sweep, B = 50, m = 1024, H100 SXM 80 GB at 700 W; DESIGN.md 6).
// A round costs its reductions and its barrier more than its arithmetic, so fewer, fuller threads win: 256 threads beat 512 at n = 512
// (354 vs 420 us), 1536, 2048 (491 vs 510 us) and 4096 (560 vs 657 us).  The exception is 513..1024 points, where 512 threads with two
// points each beat 256 with four (366 vs 401 us).  Above 4096 points 256 threads would need more than 16 points each (spills), and 512
// beat 1024 (915 vs 1047 us at n = 5000); above 8192 only 1024 threads fit 16 points each.
static int fps_auto_threads(int n)
{
    if (n <= 512) return 256;
    if (n <= 1024) return 512;
    if (n <= 4096) return 256;
    if (n <= 8192) return 512;
    return 1024;
}

static int ceil_pow2(int v)
{
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

template <int T, int P>
static int fps_launch_tp(int b, int n, int m, int layout, const float *inp, int *idx, float *out_points, cudaStream_t stream)
{
    constexpr bool kSmem = P > kFpsRegMaxPPT;
    const size_t smem = kSmem ? (size_t)n * 3 * sizeof(float) : 0;
    if (kSmem) {
        static PerDeviceOnce once;
        if (once.first()) cudaFuncSetAttribute(fps_kernel<T, P, kSmem>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFpsMaxPoints * 3 * (int)sizeof(float));
    }
    fps_kernel<T, P, kSmem><<<b, T, smem, stream>>>(n, m, layout, inp, idx, out_points);
    return check_launch("farthest_point_sample");
}

template <int T>
static int fps_launch_t(int p, int b, int n, int m, int layout, const float *inp, int *idx, float *out_points, cudaStream_t stream)
{
    switch (p) {
    case 1: return fps_launch_tp<T, 1>(b, n, m, layout, inp, idx, out_points, stream);
    case 2: return fps_launch_tp<T, 2>(b, n, m, layout, inp, idx, out_points, stream);
    case 4: return fps_launch_tp<T, 4>(b, n, m, layout, inp, idx, out_points, stream);
    case 8: return fps_launch_tp<T, 8>(b, n, m, layout, inp, idx, out_points, stream);
    case 16: return fps_launch_tp<T, 16>(b, n, m, layout, inp, idx, out_points, stream);
    }  // more than 16 points per thread would spill (ptxas hoists the shared-memory coordinates into registers where the budget allows)
    set_error("farthest_point_sample: %d threads cannot hold %d points", T, n);
    return SNB200_EUNSUPPORTED;
}

// threads = 0: by cloud size; 256 / 512 / 1024: forced (tools/bench_sampling.py sweeps them)
int launch_farthest_point_sample(int b, int n, int m, int layout, const float *inp, int *idx, float *out_points, int threads, cudaStream_t stream)
{
    if (n > kFpsMaxPoints) {
        set_error("farthest_point_sample: clouds of up to %d points are supported, got n=%d", kFpsMaxPoints, n);
        return SNB200_EUNSUPPORTED;
    }
    if (threads == 0) threads = fps_auto_threads(n);
    const int p = ceil_pow2((n + threads - 1) / threads);
    switch (threads) {
    case 256: return fps_launch_t<256>(p, b, n, m, layout, inp, idx, out_points, stream);
    case 512: return fps_launch_t<512>(p, b, n, m, layout, inp, idx, out_points, stream);
    case 1024: return fps_launch_t<1024>(p, b, n, m, layout, inp, idx, out_points, stream);
    }
    set_error("farthest_point_sample: threads per CTA must be 256, 512 or 1024, got %d", threads);
    return SNB200_EINVAL;
}

}  // namespace snb
