// chamfer.cu -- nn_distance (Chamfer) forward / backward and the fused simplification loss.
//
// Reference behaviour restated (not ported): registration/src/chamfer_distance/chamfer_distance.cu:6-137 and
// classification/structural_losses/tf_nndistance_g.cu:5-157 launch the same one-thread-per-query kernel twice over a
// fixed (32,16) grid; with 64 queries per cloud that leaves 64 of 8192 threads per batch row working, and the
// result round-trips through global memory once per 512-candidate chunk.
//
// Design: ONE launch covers both directions.  A query is owned by a group of S lanes (S = 1..32, chosen
// per direction from the shape so that small problems still spread over all SMs); each lane of the group scans
// the candidates j == lane (mod S) out of a shared-memory tile that was filled by a single TMA bulk copy
// (cp.async.bulk, AoS xyz kept as in HBM: a stride of 3 words across lanes is bank-conflict free), Q queries are
// register-blocked per thread so that every candidate read from shared memory feeds Q distance evaluations, and the
// group's partial minima are merged by log2(S) shuffle steps on the (distance, index) pair, lowest index winning
// ties exactly like the reference's strict '<' scan.
#include "pairwise_device.cuh"

namespace snb {

template <int Q, bool kFma>
__global__ void __launch_bounds__(kChamferThreads) chamfer_forward_kernel(const __grid_constant__ ChamferParams P)
{
    extern __shared__ __align__(16) float s_c[];
    __shared__ uint64_t bar;
    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    __syncthreads();
    const int bi = blockIdx.y;
    if ((int)blockIdx.x < P.d[0].tiles)
        chamfer_dir<Q, kFma>(P.d[0], blockIdx.x, bi, s_c, &bar);
    else
        chamfer_dir<Q, kFma>(P.d[1], blockIdx.x - P.d[0].tiles, bi, s_c, &bar);
}

int launch_chamfer_forward(int b, int n, const float *xyz1, int m, const float *xyz2, float *dist1, int *idx1, float *dist2,
                           int *idx2, int flags, cudaStream_t stream)
{
    ChamferParams P;
    P.d[0] = {xyz1, xyz2, dist1, idx1, n, m, 1, 0};
    P.d[1] = {xyz2, xyz1, dist2, idx2, m, n, 1, 0};
    // register blocking (every candidate read from shared memory feeds Q distance evaluations) only pays when BOTH directions
    // have many queries; with a short side (64 generated points) it would idle most of the CTA
    const long long pairs = (long long)b * n * m;
    const int Q = (pairs >= (1ll << 24) && min(n, m) >= 1024) ? 4 : 1;
    plan_chamfer_dir(P.d[0], b, Q, 2 * kNumSMs);
    plan_chamfer_dir(P.d[1], b, Q, 2 * kNumSMs);
    const int max_nc = max(n, m);
    const size_t smem = (size_t)min(max_nc, kChamferTile) * 3 * sizeof(float);
    dim3 grid(P.d[0].tiles + P.d[1].tiles, b);
    const bool unfused = (flags & SNB200_DIST_UNFUSED) != 0;
    static PerDeviceOnce attr_once;  // 48 KB tile + the static mbarrier exceeds the default 48 KB window: opt in once
    if (attr_once.first()) {
        cudaFuncSetAttribute(chamfer_forward_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
        cudaFuncSetAttribute(chamfer_forward_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
        cudaFuncSetAttribute(chamfer_forward_kernel<4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
        cudaFuncSetAttribute(chamfer_forward_kernel<4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
    }
#define SNB_LAUNCH_CHAMFER(QQ, FMA) chamfer_forward_kernel<QQ, FMA><<<grid, kChamferThreads, smem, stream>>>(P)
    if (Q == 4) {
        if (unfused) SNB_LAUNCH_CHAMFER(4, false); else SNB_LAUNCH_CHAMFER(4, true);
    } else {
        if (unfused) SNB_LAUNCH_CHAMFER(1, false); else SNB_LAUNCH_CHAMFER(1, true);
    }
#undef SNB_LAUNCH_CHAMFER
    return check_launch("nn_distance_forward");
}

// ------------------------------------------------------------------------------------------------------------------
// Per-cloud Chamfer means (evaluation: reconstruction/src/sampler_progressive_autoencoder.py:145-177 get_loss_ae_per_pc wants one scalar
// per cloud): sums[bi] = (mean_i dist1[bi, i], mean_j dist2[bi, j]) of xyz1[bi] against xyz2[bi % b2], with no dist / idx array written.
// The direction scan is chamfer_forward_kernel's own (same expression, same contraction, same planner); each CTA reduces the minima of
// its queries in a fixed order (lanes by the shuffle tree, warps in index order) into one partial, and a second small launch adds a
// cloud's partials in tile order.  No float atomics: run to run bit-identical.
// ------------------------------------------------------------------------------------------------------------------
struct ChamferCloudParams {
    ChamferDir d[2];       // dist = idx = null; q / c are the bases of xyz1 and xyz2
    int b2;                // xyz2 holds b2 clouds and repeats: cloud bi of xyz1 is compared with cloud bi % b2
    float *partial;        // (b, tiles0 + tiles1)
};

template <int Q>
__global__ void __launch_bounds__(kChamferThreads) chamfer_per_cloud_kernel(const __grid_constant__ ChamferCloudParams P)
{
    extern __shared__ __align__(16) float s_c[];
    __shared__ uint64_t bar;
    __shared__ float s_red[kChamferThreads / 32];
    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    __syncthreads();
    const int bi = blockIdx.y, dir = (int)blockIdx.x < P.d[0].tiles ? 0 : 1;
    const int b1 = bi, b2 = bi % P.b2;
    ChamferDir D = P.d[dir];      // this cloud's view: the scan then runs as batch row 0
    D.q += (size_t)(dir == 0 ? b1 : b2) * D.nq * 3;
    D.c += (size_t)(dir == 0 ? b2 : b1) * D.nc * 3;
    float my_sum = 0.f, my_max = 0.f;
    chamfer_dir<Q, true>(D, dir == 0 ? blockIdx.x : blockIdx.x - P.d[0].tiles, 0, s_c, &bar, &my_sum, &my_max);
    my_sum = warp_sum(my_sum);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = my_sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < kChamferThreads / 32; w++) t += s_red[w];
        P.partial[(size_t)bi * gridDim.x + blockIdx.x] = t;
    }
}

__global__ void chamfer_per_cloud_combine_kernel(int b, int tiles0, int tiles1, int n, int m, const float *__restrict__ partial, float *__restrict__ sums)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;   // (cloud, direction)
    if (i >= 2 * b) return;
    const int bi = i >> 1, dir = i & 1;
    const float *p = partial + (size_t)bi * (tiles0 + tiles1) + (dir ? tiles0 : 0);
    float t = 0.f;
    for (int k = 0; k < (dir ? tiles1 : tiles0); k++) t += p[k];
    sums[i] = t / (float)(dir ? m : n);
}

static int plan_chamfer_per_cloud(ChamferCloudParams &P, int b, int n, const float *xyz1, int m, const float *xyz2)
{
    P.d[0] = {xyz1, xyz2, nullptr, nullptr, n, m, 1, 0};
    P.d[1] = {xyz2, xyz1, nullptr, nullptr, m, n, 1, 0};
    const int Q = ((long long)b * n * m >= (1ll << 24) && min(n, m) >= 1024) ? 4 : 1;      // as launch_chamfer_forward
    plan_chamfer_dir(P.d[0], b, Q, 2 * kNumSMs);
    plan_chamfer_dir(P.d[1], b, Q, 2 * kNumSMs);
    return Q;
}

size_t chamfer_per_cloud_workspace_bytes(int b, int n, int m)
{
    ChamferCloudParams P;
    plan_chamfer_per_cloud(P, b, n, nullptr, m, nullptr);
    return (size_t)b * (P.d[0].tiles + P.d[1].tiles) * sizeof(float);
}

int launch_chamfer_per_cloud(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, float *sums, void *workspace, cudaStream_t stream)
{
    ChamferCloudParams P;
    const int Q = plan_chamfer_per_cloud(P, b, n, xyz1, m, xyz2);
    P.b2 = b2;
    P.partial = static_cast<float *>(workspace);
    const size_t smem = (size_t)min(max(n, m), kChamferTile) * 3 * sizeof(float);
    dim3 grid(P.d[0].tiles + P.d[1].tiles, b);
    static PerDeviceOnce attr_once;
    if (attr_once.first()) {
        cudaFuncSetAttribute(chamfer_per_cloud_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
        cudaFuncSetAttribute(chamfer_per_cloud_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
    }
    if (Q == 4) chamfer_per_cloud_kernel<4><<<grid, kChamferThreads, smem, stream>>>(P);
    else chamfer_per_cloud_kernel<1><<<grid, kChamferThreads, smem, stream>>>(P);
    if (int rc = check_launch("chamfer_per_cloud")) return rc;
    chamfer_per_cloud_combine_kernel<<<(2 * b + 255) / 256, 256, 0, stream>>>(b, P.d[0].tiles, P.d[1].tiles, n, m, P.partial, sums);
    return check_launch("chamfer_per_cloud_combine");
}

// ------------------------------------------------------------------------------------------------------------------
// Backward.  Reference: chamfer_distance.cu:158-209 zeroes both gradients and then scatters with float atomicAdd
// (summation order varies run to run).  Here each output point is owned by one thread that (a) writes its own
// "direct" term 2*g*(a - b[idx]) and (b) gathers the terms scattered onto it by scanning the other side's index
// array out of shared memory in ascending order: deterministic, no atomics, no memset.
//   grad_xyz1[j] =  2 g1[j] (x1[j] - x2[idx1[j]])  -  sum_{i: idx2[i]==j} 2 g2[i] (x2[i] - x1[j])
//   grad_xyz2[i] =  2 g2[i] (x2[i] - x1[idx2[i]])  -  sum_{j: idx1[j]==i} 2 g1[j] (x1[j] - x2[i])
// The scan is O(n*m) integer compares per cloud -- the same pair count the forward pass already walks.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kBwdThreads = 256;
constexpr int kBwdTile = 2048;

struct ChamferBwdDir {
    const float *own;        // (b, no, 3) points owned by this direction's threads
    const float *other;      // (b, nt, 3)
    const float *g_own;      // (b, no) grad wrt own dist
    const int *idx_own;      // (b, no) index into other
    const float *g_other;    // (b, nt)
    const int *idx_other;    // (b, nt) index into own
    float *grad_own;         // (b, no, 3)
    int no, nt, tiles;
    int lanes;               // threads per owned point: 1 or 32
};
struct ChamferBwdParams {
    ChamferBwdDir d[2];
};

// S = D.lanes threads share one owned point (S = 32 when a direction has few owners and a long index array to scan -- the 64 generated
// points against 1024 input points at the headline size: one thread per owner would leave 64 threads walking 1024 entries each): lane s
// scans entries s, s + S, ... and the partial sums are combined by a fixed shuffle tree, so the result stays bit-reproducible.
__device__ __forceinline__ void chamfer_bwd_dir(const ChamferBwdDir &D, int tile, int bi, int *s_idx, float *s_g)
{
    const int S = D.lanes;
    const int j = tile * (kBwdThreads / S) + (int)threadIdx.x / S;
    const int sl = (int)threadIdx.x % S;
    const bool live = j < D.no;
    const float *own = D.own + (size_t)bi * D.no * 3;
    const float *oth = D.other + (size_t)bi * D.nt * 3;
    float ax = 0, ay = 0, az = 0, gx = 0, gy = 0, gz = 0;
    if (live) {
        ax = own[j * 3 + 0]; ay = own[j * 3 + 1]; az = own[j * 3 + 2];
        if (sl == 0) {
            const int j2 = D.idx_own[(size_t)bi * D.no + j];
            const float g = D.g_own[(size_t)bi * D.no + j] * 2;
            gx = g * (ax - oth[j2 * 3 + 0]);
            gy = g * (ay - oth[j2 * 3 + 1]);
            gz = g * (az - oth[j2 * 3 + 2]);
        }
    }
    for (int t0 = 0; t0 < D.nt; t0 += kBwdTile) {
        const int tn = min(kBwdTile, D.nt - t0);
        __syncthreads();
        for (int i = threadIdx.x; i < tn; i += kBwdThreads) {
            s_idx[i] = D.idx_other[(size_t)bi * D.nt + t0 + i];
            s_g[i] = D.g_other[(size_t)bi * D.nt + t0 + i];
        }
        __syncthreads();
        if (live) {
            for (int i = sl; i < tn; i += S) {
                if (s_idx[i] == j) {  // rare: on average nt/no hits per owner
                    const float g = s_g[i] * 2;
                    gx -= g * (oth[(t0 + i) * 3 + 0] - ax);
                    gy -= g * (oth[(t0 + i) * 3 + 1] - ay);
                    gz -= g * (oth[(t0 + i) * 3 + 2] - az);
                }
            }
        }
    }
    if (S > 1) {   // (S = 32: a warp per owner; every lane of the warp takes part, live or not)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            gx += __shfl_down_sync(kFullMask, gx, o);
            gy += __shfl_down_sync(kFullMask, gy, o);
            gz += __shfl_down_sync(kFullMask, gz, o);
        }
    }
    if (live && sl == 0) {
        float *go = D.grad_own + ((size_t)bi * D.no + j) * 3;
        go[0] = gx; go[1] = gy; go[2] = gz;
    }
}

__global__ void __launch_bounds__(kBwdThreads) chamfer_backward_kernel(const __grid_constant__ ChamferBwdParams P)
{
    __shared__ int s_idx[kBwdTile];
    __shared__ float s_g[kBwdTile];
    if ((int)blockIdx.x < P.d[0].tiles)
        chamfer_bwd_dir(P.d[0], blockIdx.x, blockIdx.y, s_idx, s_g);
    else
        chamfer_bwd_dir(P.d[1], blockIdx.x - P.d[0].tiles, blockIdx.y, s_idx, s_g);
}

int launch_chamfer_backward(int b, int n, const float *xyz1, int m, const float *xyz2, const float *grad_dist1, const int *idx1,
                            const float *grad_dist2, const int *idx2, float *grad_xyz1, float *grad_xyz2, cudaStream_t stream)
{
    ChamferBwdParams P;
    const int s1 = (n <= 256 && m >= 128) ? 32 : 1, s2 = (m <= 256 && n >= 128) ? 32 : 1;
    P.d[0] = {xyz1, xyz2, grad_dist1, idx1, grad_dist2, idx2, grad_xyz1, n, m, (n * s1 + kBwdThreads - 1) / kBwdThreads, s1};
    P.d[1] = {xyz2, xyz1, grad_dist2, idx2, grad_dist1, idx1, grad_xyz2, m, n, (m * s2 + kBwdThreads - 1) / kBwdThreads, s2};
    dim3 grid(P.d[0].tiles + P.d[1].tiles, b);
    chamfer_backward_kernel<<<grid, kBwdThreads, 0, stream>>>(P);
    return check_launch("nn_distance_backward");
}

// ------------------------------------------------------------------------------------------------------------------
// Simplification-loss reductions (registration/src/samplenet.py:176-180): three deterministic means in one small
// launch that runs after the forward kernel on the same stream.
//   out[0] = mean(dist1), out[1] = mean_b(max_n dist1), out[2] = mean(dist2), out[3] = out[0]+out[1]+w*out[2]
// One CTA: per-cloud partials are produced by warps in a fixed order and summed in a fixed order (the reference
// uses four separate torch reductions; values agree to fp32 rounding).
// ------------------------------------------------------------------------------------------------------------------
// all of a lane's loads are issued before the first add (the arrays are a few KB: latency, not bandwidth, is the cost)
__device__ __forceinline__ void lane_sum_max(const float *__restrict__ p, int n, int lane, float &sum, float &mx)
{
    sum = 0.f; mx = -INFINITY;
    if (((reinterpret_cast<uintptr_t>(p) & 15) == 0) && (n & 3) == 0) {
        const float4 *q = reinterpret_cast<const float4 *>(p);
        const int n4 = n >> 2;
        for (int j0 = lane; j0 < n4; j0 += 32 * 8) {
            float4 v[8];
#pragma unroll
            for (int u = 0; u < 8; u++) v[u] = (j0 + u * 32 < n4) ? __ldg(q + j0 + u * 32) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int u = 0; u < 8; u++)
                if (j0 + u * 32 < n4) {
                    sum += (v[u].x + v[u].y) + (v[u].z + v[u].w);
                    mx = fmaxf(mx, fmaxf(fmaxf(v[u].x, v[u].y), fmaxf(v[u].z, v[u].w)));
                }
        }
    } else {
        for (int j = lane; j < n; j += 32) { const float v = __ldg(p + j); sum += v; mx = fmaxf(mx, v); }
    }
}

__global__ void __launch_bounds__(1024) simplification_reduce_kernel(int b, int n, int m, const float *__restrict__ dist1,
                                                                    const float *__restrict__ dist2, float w, float *__restrict__ out4)
{
    __shared__ float s_sum1[32], s_max1[32], s_sum2[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    float acc1 = 0, accmax = 0, acc2 = 0;  // per-warp accumulators over the clouds this warp owns (lane 0 meaningful)
    for (int bi = warp; bi < b; bi += nwarps) {
        float s1, mx, s2, unused;
        lane_sum_max(dist1 + (size_t)bi * n, n, lane, s1, mx);
        lane_sum_max(dist2 + (size_t)bi * m, m, lane, s2, unused);
        s1 = warp_sum(s1);
        mx = warp_max(mx);
        s2 = warp_sum(s2);
        acc1 += s1; accmax += mx; acc2 += s2;
    }
    if (lane == 0) { s_sum1[warp] = acc1; s_max1[warp] = accmax; s_sum2[warp] = acc2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float t1 = 0, tm = 0, t2 = 0;
        for (int i = 0; i < nwarps; i++) { t1 += s_sum1[i]; tm += s_max1[i]; t2 += s_sum2[i]; }
        const float c12 = t1 / ((float)b * (float)n);
        const float mc = tm / (float)b;
        const float c21 = t2 / ((float)b * (float)m);
        out4[0] = c12; out4[1] = mc; out4[2] = c21;
        out4[3] = c12 + mc + w * c21;
    }
}

// One warp per cloud up to 32 clouds, then 1024 threads whose warps loop over the clouds (also snb200_debug_simplification_loss_plan).
int simplification_reduce_threads(int b) { return (b >= 32) ? 1024 : max(32, b * 32); }

int launch_simplification_reduce(int b, int n, int m, const float *dist1, const float *dist2, float w, float *out4, cudaStream_t stream)
{
    simplification_reduce_kernel<<<1, simplification_reduce_threads(b), 0, stream>>>(b, n, m, dist1, dist2, w, out4);
    return check_launch("simplification_loss_reduce");
}

}  // namespace snb
