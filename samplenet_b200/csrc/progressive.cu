// progressive.cu -- SampleNetProgressive's simplification loss in ONE launch.
//
// Reference (classification/train_samplenet_progressive.py:172-230, reconstruction twin samplenet_pointnet_ae.py:196-220): the generator
// emits M ORDERED points; for every prefix size s in {s_0 < s_1 < ... } (powers of two in the reference) the graph slices the first s
// points and calls get_simplification_loss -> one NnDistance op + 4 reductions per prefix (10 ops pairs for 2..1024).
// Both Chamfer directions of ALL prefixes come out of one pass over the pair matrix:
//   * sample -> input  : the nearest input point of sample j does not depend on the prefix; dist1 of prefix s is the slice [:s];
//   * input  -> sample : the nearest of the first s samples is a running prefix minimum over the sample index.  A reference point is
//     owned by S lanes, lane l scans the samples l, l + S, ... and records its running (distance, index) minimum at every prefix
//     boundary; the lanes' records are merged lexicographically, which reproduces the strict-'<' lowest-index rule of the reference
//     kernel for every prefix.
// Loss terms are reduced in a fixed order: per-CTA partials, the last CTA to finish (ticket) combines them (bit-reproducible).
#include "pairwise_device.cuh"

namespace snb {

constexpr int kPgMaxPrefix = 16;
constexpr int kPgThreads = 256;
constexpr int kPgQ = 2;     // queries register-blocked per thread in the sample -> input scan

struct ProgParams {
    int b, n, m, np;                 // clouds, input points, ordered samples, prefixes
    int sizes[kPgMaxPrefix];         // ascending, <= m
    float w21[kPgMaxPrefix];         // weight of the input -> sample term of each prefix (gamma + delta * size)
    const float *ref, *samp;
    ChamferDir d0;                   // samples (queries) -> input cloud (candidates): dist1 / idx1
    int S2, tiles2;                  // input -> samples: lanes per reference point, CTAs per cloud
    float *dist2; int *idx2;         // (b, np, n)
    float *partial;                  // (b, tiles2, np): per-CTA sums of dist2
    unsigned *ticket;
    float *terms;                    // (np, 3) then [3*np] = total loss
    int cl_batch;                    // clouds whose dist1 rows the final reduction stages at a time (1..8)
};

template <bool kFma>
__global__ void __launch_bounds__(kPgThreads) progressive_loss_kernel(const __grid_constant__ ProgParams P)
{
    extern __shared__ __align__(16) float s_dyn[];
    __shared__ uint64_t bar;
    __shared__ float s_red[kPgThreads / 32][kPgMaxPrefix];
    __shared__ unsigned s_ticket;
    const int n0 = P.b * P.d0.tiles;
    const int total_ctas = n0 + P.b * P.tiles2;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { mbar_init(&bar, 1); fence_mbar_init(); }
    __syncthreads();
    if ((int)blockIdx.x < n0) {
        // ---- role A: sample -> input (prefix independent)
        const int bi = (int)blockIdx.x / P.d0.tiles, tile = (int)blockIdx.x % P.d0.tiles;
        chamfer_dir<kPgQ, kFma>(P.d0, tile, bi, s_dyn, &bar);
    } else {
        // ---- role B: input -> samples with prefix minima
        const int bi = ((int)blockIdx.x - n0) / P.tiles2, tile = ((int)blockIdx.x - n0) % P.tiles2;
        const int S = P.S2, groups = kPgThreads / S;
        const int g = threadIdx.x / S, l = threadIdx.x % S;
        const int i = tile * groups + g;                           // reference point of this lane group
        const bool live = i < P.n;
        const float *rp = P.ref + ((size_t)bi * P.n + min(i, P.n - 1)) * 3;
        const float qx = __ldg(rp), qy = __ldg(rp + 1), qz = __ldg(rp + 2);
        uint32_t phase = 0;
        stage_floats(s_dyn, P.samp + (size_t)bi * P.m * 3, P.m * 3, &bar, phase);
        // lane l scans the samples j = l, l + S, l + 2S, ... (neighbouring lanes read neighbouring points: conflict-free shared-memory reads);
        // at a prefix boundary s its running minimum covers {j < s, j = l mod S}, and the lexicographic merge over the S lanes below gives
        // the minimum over all j < s with the lowest index among equal distances
        float best = INFINITY; int besti = 0x7fffffff;
        float rec[kPgMaxPrefix]; int reci[kPgMaxPrefix];
        int j = l;
#pragma unroll
        for (int p = 0; p < kPgMaxPrefix; p++) {
            if (p < P.np) {
                const int end = P.sizes[p];
#pragma unroll 4
                for (; j < end; j += S) {
                    const float d = sqdist<kFma>(s_dyn[j * 3 + 0] - qx, s_dyn[j * 3 + 1] - qy, s_dyn[j * 3 + 2] - qz);   // (candidate - query)
                    if (d < best) { best = d; besti = j; }
                }
                rec[p] = best; reci[p] = besti;      // minimum over this lane's samples below the prefix boundary (INF if none)
            }
        }
        float psum[kPgMaxPrefix];
#pragma unroll
        for (int p = 0; p < kPgMaxPrefix; p++) {
            psum[p] = 0.f;
            if (p < P.np) {
                float v = rec[p]; int vi = reci[p];
                for (int o = S >> 1; o > 0; o >>= 1) {
                    const float ov = __shfl_xor_sync(kFullMask, v, o);
                    const int oi = __shfl_xor_sync(kFullMask, vi, o);
                    if (ov < v || (ov == v && oi < vi)) { v = ov; vi = oi; }
                }
                if (vi == 0x7fffffff) vi = 0;   // nothing compared below +inf (NaN/Inf coordinates): index 0, as nn_distance
                if (live && l == 0) {
                    P.dist2[((size_t)bi * P.np + p) * P.n + i] = v;
                    P.idx2[((size_t)bi * P.np + p) * P.n + i] = vi;
                    psum[p] = v;
                }
            }
        }
        // CTA partial per prefix, fixed order
#pragma unroll
        for (int p = 0; p < kPgMaxPrefix; p++) {
            if (p < P.np) {
                const float s = warp_sum(psum[p]);
                if (lane == 0) s_red[warp][p] = s;
            }
        }
        __syncthreads();
        if ((int)threadIdx.x < P.np) {
            float t = 0.f;
            for (int w = 0; w < kPgThreads / 32; w++) t += s_red[w][threadIdx.x];
            P.partial[((size_t)bi * P.tiles2 + tile) * P.np + threadIdx.x] = t;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_ticket = atomicAdd(P.ticket, 1u);
    }
    __syncthreads();
    if (s_ticket != (unsigned)total_ctas - 1u) return;
    // ---- last CTA: every dist1 value and every partial is visible (each CTA fenced before taking its ticket)
    __threadfence();
    float *s_t = s_dyn;    // [np][3] accumulators over clouds, then the total
    for (int e2 = threadIdx.x; e2 < P.np * 3; e2 += kPgThreads) s_t[e2] = 0.f;
    __shared__ float s_seg[kPgThreads / 32][kPgMaxPrefix][2];
    __syncthreads();
    const float *d1 = P.d0.dist;
    // dist1 of kPgThreads / 32 clouds at a time is pulled into shared memory with independent, coalesced loads (one L2 round trip), then a
    // warp per cloud forms the per-segment sums / maxima and the prefix over the segments -- everything in a fixed order
    float *s_d1 = s_dyn + 64;                                   // [8 clouds][m] behind the accumulators
    const int kCl = P.cl_batch;
    for (int c0 = 0; c0 < P.b; c0 += kCl) {
        const int ncl = min(kCl, P.b - c0);
        const int tot = ncl * P.m;
        __syncthreads();
        for (int e0 = threadIdx.x; e0 < tot; e0 += kPgThreads * 8) {
            float v8[8];
#pragma unroll
            for (int u = 0; u < 8; u++) v8[u] = (e0 + u * kPgThreads < tot) ? __ldcg(d1 + (size_t)c0 * P.m + e0 + u * kPgThreads) : 0.f;
#pragma unroll
            for (int u = 0; u < 8; u++)
                if (e0 + u * kPgThreads < tot) s_d1[e0 + u * kPgThreads] = v8[u];
        }
        __syncthreads();
        const int bi = c0 + warp;
        if (warp < ncl) {
            int lo = 0;
            for (int p = 0; p < P.np; p++) {
                float s = 0.f, mx = -INFINITY;
                for (int jj = lo + lane; jj < P.sizes[p]; jj += 32) { const float v = s_d1[warp * P.m + jj]; s += v; mx = fmaxf(mx, v); }
                s = warp_sum(s); mx = warp_max(mx);
                if (lane == 0) { s_seg[warp][p][0] = s; s_seg[warp][p][1] = mx; }
                lo = P.sizes[p];
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 0; w < kCl && c0 + w < P.b; w++) {
                float run_s = 0.f, run_m = -INFINITY;
                for (int p = 0; p < P.np; p++) {
                    run_s += s_seg[w][p][0]; run_m = fmaxf(run_m, s_seg[w][p][1]);
                    s_t[p * 3 + 0] += run_s / (float)P.sizes[p];
                    s_t[p * 3 + 1] += run_m;
                }
            }
        }
        __syncthreads();
    }
    {   // per-prefix sums of the input -> sample partials: all threads pull the (cloud, tile) partials with independent loads, then a
        // fixed-order tree (bit-reproducible)
        __shared__ float s_tree[kPgThreads];
        const int nparts = P.b * P.tiles2;
        for (int p = 0; p < P.np; p++) {
            float t = 0.f;
            for (int e2 = threadIdx.x; e2 < nparts; e2 += kPgThreads) t += __ldcg(P.partial + (size_t)e2 * P.np + p);
            s_tree[threadIdx.x] = t;
            __syncthreads();
            for (int o = kPgThreads / 2; o > 0; o >>= 1) {
                if ((int)threadIdx.x < o) s_tree[threadIdx.x] += s_tree[threadIdx.x + o];
                __syncthreads();
            }
            if (threadIdx.x == 0) s_t[p * 3 + 2] = s_tree[0];
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) {
        float total = 0.f;
        for (int p = 0; p < P.np; p++) {
            const float t0 = s_t[p * 3 + 0] / (float)P.b, t1 = s_t[p * 3 + 1] / (float)P.b, t2 = s_t[p * 3 + 2] / ((float)P.b * (float)P.n);
            P.terms[p * 3 + 0] = t0; P.terms[p * 3 + 1] = t1; P.terms[p * 3 + 2] = t2;
            total += t0 + t1 + P.w21[p] * t2;
        }
        P.terms[P.np * 3] = total;
        *P.ticket = 0u;
    }
}

size_t progressive_workspace_bytes(int b, int n, int m, int np)
{
    // worst case tiles2 = n (one reference point per CTA would never be planned; S2 <= 32 -> groups >= 8)
    const int tiles2_max = (n + 7) / 8;
    return (size_t)b * tiles2_max * np * sizeof(float) + 256;
}

// The launch plan of progressive_loss_kernel, computed in one place for the launcher and snb200_debug_progressive_loss_plan: role A's
// scan (P.d0: lanes per query, tiles), role B's lanes per reference point and tiles, the clouds the final reduction stages at a time, and
// the dynamic shared memory.
static size_t progressive_plan(ProgParams &P, int b, int n, int m)
{
    P.d0.nq = m; P.d0.nc = n;
    plan_chamfer_dir(P.d0, b, kPgQ, 2 * kNumSMs);
    // lanes per reference point: enough CTAs to fill the machine a few times over, at least 32 samples per lane
    int S = 1;
    while (S < 32 && m / (S * 2) >= 32 && (long long)b * ((n + kPgThreads / S - 1) / (kPgThreads / S)) < 4ll * kNumSMs) S *= 2;
    P.S2 = S;
    P.tiles2 = (n + kPgThreads / S - 1) / (kPgThreads / S);
    P.cl_batch = max(1, min(kPgThreads / 32, (12 * 1024 - 64) / m));   // at most 48 KB of staging (keeps several CTAs per SM)
    return (size_t)max(max(max(min(n, kChamferTile), m) * 3, 64 + P.cl_batch * m), 64) * sizeof(float);
}

void progressive_plan_query(int b, int n, int m, int *s_a, int *tiles_a, int *s2, int *tiles2, int *cl_batch)
{
    ProgParams P;
    memset(&P, 0, sizeof(P));
    progressive_plan(P, b, n, m);
    *s_a = P.d0.S; *tiles_a = P.d0.tiles; *s2 = P.S2; *tiles2 = P.tiles2; *cl_batch = P.cl_batch;
}

int launch_progressive_loss(int b, int n, int m, const float *ref, const float *samp, int np, const int *sizes, const float *w21, float *dist1, int *idx1,
                            float *dist2, int *idx2, float *terms, void *workspace, unsigned *ticket, int flags, cudaStream_t stream)
{
    ProgParams P;
    memset(&P, 0, sizeof(P));
    P.b = b; P.n = n; P.m = m; P.np = np; P.ref = ref; P.samp = samp;
    for (int p = 0; p < np; p++) { P.sizes[p] = sizes[p]; P.w21[p] = w21[p]; }
    P.d0.q = samp; P.d0.c = ref; P.d0.dist = dist1; P.d0.idx = idx1;
    const size_t smem = progressive_plan(P, b, n, m);
    P.dist2 = dist2; P.idx2 = idx2; P.partial = reinterpret_cast<float *>(workspace); P.ticket = ticket; P.terms = terms;
    static PerDeviceOnce once;
    if (once.first()) {
        cudaFuncSetAttribute(progressive_loss_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        cudaFuncSetAttribute(progressive_loss_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    }
    const int grid = b * (P.d0.tiles + P.tiles2);
    if (flags & SNB200_DIST_UNFUSED) progressive_loss_kernel<false><<<grid, kPgThreads, smem, stream>>>(P);
    else progressive_loss_kernel<true><<<grid, kPgThreads, smem, stream>>>(P);
    return check_launch("progressive loss");
}

}  // namespace snb
