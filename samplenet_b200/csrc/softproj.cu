// softproj.cu -- fused brute-force kNN + temperature softmax + weighted gather (SoftProjection), its backward,
// and group_point / group_point_grad.
//
// Reference behaviour restated (not ported):
//   registration/src/soft_projection.py:75-152  knn_cuda.KNN (python loop over the batch, full N x M distance matrix per
//       cloud, insertion sort) -> pointnet2 grouping_operation -> ~8 small torch kernels;
//   classification/grouping/tf_grouping.py:64-91 + tf_grouping_g.cu:83-123  two tiled (B,M,N,3) tensors, a (B,M,N)
//       distance tensor, then a selection sort that runs ONE CTA per batch element over global memory.
//
// Design: one warp owns one query.  The cloud tile sits in shared memory (one TMA bulk copy per CTA; AoS for BNC
// input -- a stride of 3 words across lanes is conflict free -- or three SoA rows for BCN input), the 32 lanes evaluate 32
// candidates per step, and the running top-k lives in registers ACROSS the warp: lane i holds the i-th best
// (distance, index).  A candidate enters only if it beats the current k-th best (one ballot per 32 candidates); an insert
// is two shuffles and two selects per lane, independent of k.  Candidates are inserted in ascending index order with a
// strict '<', so the list is sorted by (distance, index) -- the documented tie contract.  The pair matrix is never
// materialised, and the softmax / weighted average run in the same warp on the k survivors.
#include "pairwise_device.cuh"

namespace snb {

template <int kLayout, bool kFma>
__global__ void __launch_bounds__(kSpThreads) knn_softproj_kernel(const __grid_constant__ SoftProjParams P)
{
    extern __shared__ __align__(16) float s_pts[];
    __shared__ uint64_t bar;
    knn_softproj_body<kLayout, kFma>(P, blockIdx.x, blockIdx.y, s_pts, &bar);
}

int launch_knn_softproj(int b, int n, int m, int k, int layout, const float *points, const float *query, const float *sigma, int sigma_mode,
                        float sigma_floor, int hard,
                        const float *feats, int f, float *proj, float *prop, int *knn_idx, float *knn_val, float *weights,
                        float *dist_over_sigma, int flags, cudaStream_t stream)
{
    SoftProjParams P;
    P.b = b; P.n = n; P.m = m; P.k = k; P.f = f;
    P.points = points; P.query = query; P.sigma = sigma; P.sigma_mode = sigma_mode; P.sigma_floor = sigma_floor; P.feats = feats; P.hard = hard;
    P.proj = proj; P.prop = prop; P.knn_idx = knn_idx; P.knn_val = knn_val; P.weights = weights; P.dist_over_sigma = dist_over_sigma;
    P.nn_dist = nullptr; P.nn_idx = nullptr;
    // one query per warp until the grid exceeds ~8 CTAs per SM, then amortise the tile staging over more queries
    int qpw = 1;
    while ((long long)b * ((m + kSpWarps * qpw - 1) / (kSpWarps * qpw)) > 8ll * kNumSMs && qpw < 16) qpw *= 2;
    if (n > kSpTile) qpw = 1;  // multi-tile clouds restage per query round; keep rounds minimal
    P.queries_per_warp = qpw;
    dim3 grid((m + kSpWarps * qpw - 1) / (kSpWarps * qpw), b);
    const size_t smem = (size_t)min(n, kSpTile) * 3 * sizeof(float);
    const bool unfused = (flags & SNB200_DIST_UNFUSED) != 0;
    static PerDeviceOnce attr_once;  // 48 KB tile + the static mbarrier exceeds the default 48 KB window: opt in once
    if (attr_once.first()) {
        cudaFuncSetAttribute(knn_softproj_kernel<SNB200_BNC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
        cudaFuncSetAttribute(knn_softproj_kernel<SNB200_BNC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
        cudaFuncSetAttribute(knn_softproj_kernel<SNB200_BCN, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
        cudaFuncSetAttribute(knn_softproj_kernel<SNB200_BCN, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
    }
    if (layout == SNB200_BNC) {
        if (unfused) knn_softproj_kernel<SNB200_BNC, false><<<grid, kSpThreads, smem, stream>>>(P);
        else knn_softproj_kernel<SNB200_BNC, true><<<grid, kSpThreads, smem, stream>>>(P);
    } else {
        if (unfused) knn_softproj_kernel<SNB200_BCN, false><<<grid, kSpThreads, smem, stream>>>(P);
        else knn_softproj_kernel<SNB200_BCN, true><<<grid, kSpThreads, smem, stream>>>(P);
    }
    return check_launch("knn_soft_project_forward");
}

// ------------------------------------------------------------------------------------------------------------------
// Backward of the soft projection (autograd graph of registration/src/soft_projection.py:92-152).
// Per query (one warp, lane i = neighbour i), with g_i the neighbour, q the query, s = sigma, d_i = |g_i-q|^2/s,
// w = softmax(-d), proj = sum_i w_i g_i, prop_c = sum_i w_i F_c[idx_i]:
//   a_i   = <grad_proj, g_i> + sum_c grad_prop_c F_c[idx_i]          (dL/dw_i)
//   t_i   = w_i (a_i - sum_j w_j a_j)                                (dL/d(-d_i))
//   dL/dd_i = -t_i ;  dL/dg_i = w_i grad_proj + dL/dd_i * 2 (g_i - q)/s ; dL/dq = -sum_i dL/dd_i * 2 (g_i - q)/s
//   dL/ds = sum_i dL/dd_i * (-d_i / s) ;  dL/dF_c[idx_i] += w_i grad_prop_c
// grad_query is written directly.  The scatters onto the cloud (grad_points, grad_feats) are made deterministic the
// same way as the Chamfer backward: pass 1 stores the per-(query, neighbour) contribution in the workspace, pass 2 lets
// every cloud point gather its contributions by scanning that cloud's (m*k) index list in ascending order.
// grad_sigma: per-CTA partials in the workspace, summed in fixed order by the last pass.
// ------------------------------------------------------------------------------------------------------------------
struct SoftProjBwdParams {
    int b, n, m, k, f;
    const float *points, *query, *sigma, *feats;
    int sigma_mode; float sigma_floor;
    const int *knn_idx;
    const float *weights, *grad_proj, *grad_prop;
    float *grad_query;
    float *contrib;       // workspace (b, m, k, 3): dL/dg_i per (query, neighbour)   [only if grad_points]
    float *wcontrib;      // workspace: unused (weights are re-read)
    float *sigma_partial; // workspace (b * m) per-query dL/dsigma
};

template <int kLayout>
__global__ void __launch_bounds__(kSpThreads) softproj_bwd_query_kernel(const __grid_constant__ SoftProjBwdParams P)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bi = blockIdx.y;
    const int qi = blockIdx.x * kSpWarps + warp;
    if (qi >= P.m) return;
    const int n = P.n, m = P.m, k = P.k, f = P.f;
    const float *pts = P.points + (size_t)bi * n * 3;
    const float *qry = P.query + (size_t)bi * m * 3;
    const bool has = lane < k;
    const size_t o = ((size_t)bi * m + qi) * k + lane;
    const int li = has ? P.knn_idx[o] : 0;
    const float w = has ? P.weights[o] : 0.0f;
    const float qx = ld_coord<kLayout>(qry, m, qi, 0), qy = ld_coord<kLayout>(qry, m, qi, 1), qz = ld_coord<kLayout>(qry, m, qi, 2);
    float gx = 0, gy = 0, gz = 0;
    if (has) { gx = ld_coord<kLayout>(pts, n, li, 0); gy = ld_coord<kLayout>(pts, n, li, 1); gz = ld_coord<kLayout>(pts, n, li, 2); }
    float px = 0, py = 0, pz = 0;
    if (P.grad_proj) {
        const float *gp = P.grad_proj + (size_t)bi * m * 3;
        px = ld_coord<kLayout>(gp, m, qi, 0); py = ld_coord<kLayout>(gp, m, qi, 1); pz = ld_coord<kLayout>(gp, m, qi, 2);
    }
    float a = px * gx + py * gy + pz * gz;
    if (P.grad_prop && has) {
        const float *ft = P.feats + (size_t)bi * n * f;
        const float *gpr = P.grad_prop + (size_t)bi * m * f;
        for (int c = 0; c < f; c++) {
            const float gpc = kLayout == SNB200_BNC ? gpr[(size_t)qi * f + c] : gpr[(size_t)c * m + qi];
            const float fv = kLayout == SNB200_BNC ? ft[(size_t)li * f + c] : ft[(size_t)c * n + li];
            a += gpc * fv;
        }
    }
    if (!has) a = 0;
    const float wa = warp_sum(w * a);
    const float t = w * (a - wa);   // dL/d(-d_i)
    const float ddd = -t;           // dL/dd_i
    const float sigma = resolve_sigma(P.sigma, P.sigma_mode, P.sigma_floor);
    const float dx = gx - qx, dy = gy - qy, dz = gz - qz;
    const float two_over_s = 2.0f / sigma;
    const float cx = ddd * two_over_s * dx, cy = ddd * two_over_s * dy, cz = ddd * two_over_s * dz;  // via the distance
    if (P.grad_query) {
        const float sx = warp_sum(has ? -cx : 0.f), sy = warp_sum(has ? -cy : 0.f), sz = warp_sum(has ? -cz : 0.f);
        if (lane == 0) {
            float *gq = P.grad_query + (size_t)bi * m * 3;
            if (kLayout == SNB200_BNC) { gq[(size_t)qi * 3 + 0] = sx; gq[(size_t)qi * 3 + 1] = sy; gq[(size_t)qi * 3 + 2] = sz; }
            else { gq[qi] = sx; gq[(size_t)m + qi] = sy; gq[2 * (size_t)m + qi] = sz; }
        }
    }
    if (P.contrib && has) {
        float *cb = P.contrib + o * 3;
        cb[0] = w * px + cx; cb[1] = w * py + cy; cb[2] = w * pz + cz;
    }
    if (P.sigma_partial) {
        const float d_over_s = (dx * dx + dy * dy + dz * dz) / sigma;
        const float gs = warp_sum(has ? ddd * (-d_over_s / sigma) : 0.f);
        if (lane == 0) P.sigma_partial[(size_t)bi * m + qi] = gs;
    }
}

// pass 2: every cloud point gathers the contributions addressed to it (ascending (query, neighbour) order)
struct SoftProjGatherParams {
    int b, n, m, k, f;
    const int *knn_idx;
    const float *contrib;     // (b, m*k, 3) or NULL
    const float *weights;     // (b, m*k)
    const float *grad_prop;   // (b, m, f)/(b, f, m) or NULL
    float *grad_points;       // layout, or NULL
    float *grad_feats;        // like feats, or NULL
    const float *sigma_partial;
    float *grad_sigma;
    int total_queries;
};

constexpr int kGatherTile = 2048;

template <int kLayout>
__global__ void __launch_bounds__(256) softproj_bwd_gather_kernel(const __grid_constant__ SoftProjGatherParams P)
{
    __shared__ int s_idx[kGatherTile];
    const int bi = blockIdx.y;
    const int p = blockIdx.x * 256 + threadIdx.x;
    const int n = P.n, m = P.m, k = P.k, f = P.f;
    const int mk = m * k;
    const bool live = p < n;
    float ax = 0, ay = 0, az = 0;
    // grad_sigma: CTA (0,0) sums the per-query partials in a fixed order
    if (P.grad_sigma && blockIdx.x == 0 && blockIdx.y == 0) {
        __shared__ float s_part[256];
        float acc = 0;
        for (int i = threadIdx.x; i < P.total_queries; i += 256) acc += P.sigma_partial[i];
        s_part[threadIdx.x] = acc;
        __syncthreads();
        for (int s = 128; s > 0; s >>= 1) {
            if (threadIdx.x < s) s_part[threadIdx.x] += s_part[threadIdx.x + s];
            __syncthreads();
        }
        if (threadIdx.x == 0) *P.grad_sigma = s_part[0];
    }
    if (!P.grad_points && !P.grad_feats) return;
    if (P.grad_feats && live) {
        float *gf = P.grad_feats + (size_t)bi * n * f;
        for (int c = 0; c < f; c++) {
            if (kLayout == SNB200_BNC) gf[(size_t)p * f + c] = 0.f; else gf[(size_t)c * n + p] = 0.f;
        }
    }
    for (int t0 = 0; t0 < mk; t0 += kGatherTile) {
        const int tn = min(kGatherTile, mk - t0);
        __syncthreads();
        for (int i = threadIdx.x; i < tn; i += 256) s_idx[i] = P.knn_idx[(size_t)bi * mk + t0 + i];
        __syncthreads();
        if (live) {
            for (int i = 0; i < tn; i++) {
                if (s_idx[i] == p) {
                    const size_t e = (size_t)bi * mk + t0 + i;
                    if (P.grad_points) {
                        ax += P.contrib[e * 3 + 0]; ay += P.contrib[e * 3 + 1]; az += P.contrib[e * 3 + 2];
                    }
                    if (P.grad_feats) {
                        const float w = P.weights[e];
                        const int qi = (t0 + i) / k;
                        const float *gpr = P.grad_prop + (size_t)bi * m * f;
                        float *gf = P.grad_feats + (size_t)bi * n * f;
                        for (int c = 0; c < f; c++) {
                            const float gpc = kLayout == SNB200_BNC ? gpr[(size_t)qi * f + c] : gpr[(size_t)c * m + qi];
                            if (kLayout == SNB200_BNC) gf[(size_t)p * f + c] += w * gpc; else gf[(size_t)c * n + p] += w * gpc;
                        }
                    }
                }
            }
        }
    }
    if (P.grad_points && live) {
        float *gp = P.grad_points + (size_t)bi * n * 3;
        if (kLayout == SNB200_BNC) { gp[(size_t)p * 3 + 0] = ax; gp[(size_t)p * 3 + 1] = ay; gp[(size_t)p * 3 + 2] = az; }
        else { gp[p] = ax; gp[(size_t)n + p] = ay; gp[2 * (size_t)n + p] = az; }
    }
}

size_t softproj_bwd_workspace(int b, int n, int m, int k, int f)
{
    (void)n; (void)f;
    return align_up((size_t)b * m * k * 3 * sizeof(float), 256) + align_up((size_t)b * m * sizeof(float), 256);
}

int launch_softproj_backward(int b, int n, int m, int k, int layout, const float *points, const float *query, const float *sigma,
                             int sigma_mode, float sigma_floor, const float *feats, int f, const int *knn_idx, const float *weights, const float *grad_proj,
                             const float *grad_prop, float *grad_points, float *grad_query, float *grad_feats, float *grad_sigma,
                             void *workspace, cudaStream_t stream)
{
    float *contrib = reinterpret_cast<float *>(workspace);
    float *sigma_partial = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + align_up((size_t)b * m * k * 3 * sizeof(float), 256));
    SoftProjBwdParams P;
    P.b = b; P.n = n; P.m = m; P.k = k; P.f = f;
    P.points = points; P.query = query; P.sigma = sigma; P.sigma_mode = sigma_mode; P.sigma_floor = sigma_floor; P.feats = feats;
    P.knn_idx = knn_idx; P.weights = weights;
    P.grad_proj = grad_proj; P.grad_prop = grad_prop; P.grad_query = grad_query;
    P.contrib = grad_points ? contrib : nullptr; P.wcontrib = nullptr;
    P.sigma_partial = grad_sigma ? sigma_partial : nullptr;
    dim3 grid((m + kSpWarps - 1) / kSpWarps, b);
    if (layout == SNB200_BNC) softproj_bwd_query_kernel<SNB200_BNC><<<grid, kSpThreads, 0, stream>>>(P);
    else softproj_bwd_query_kernel<SNB200_BCN><<<grid, kSpThreads, 0, stream>>>(P);
    int rc = check_launch("soft_project_backward(query pass)");
    if (rc) return rc;
    if (!grad_points && !grad_feats && !grad_sigma) return SNB200_OK;
    SoftProjGatherParams G;
    G.b = b; G.n = n; G.m = m; G.k = k; G.f = f; G.knn_idx = knn_idx; G.contrib = contrib; G.weights = weights;
    G.grad_prop = grad_prop; G.grad_points = grad_points; G.grad_feats = (grad_prop ? grad_feats : nullptr);
    G.sigma_partial = sigma_partial; G.grad_sigma = grad_sigma; G.total_queries = b * m;
    dim3 grid2((n + 255) / 256, b);
    if (!grad_points && !G.grad_feats) grid2 = dim3(1, 1);
    if (layout == SNB200_BNC) softproj_bwd_gather_kernel<SNB200_BNC><<<grid2, 256, 0, stream>>>(G);
    else softproj_bwd_gather_kernel<SNB200_BCN><<<grid2, 256, 0, stream>>>(G);
    rc = check_launch("soft_project_backward(gather pass)");
    if (rc) return rc;
    if (grad_feats && !grad_prop) {
        cudaMemsetAsync(grad_feats, 0, (size_t)b * n * f * sizeof(float), stream);
    }
    return SNB200_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// group_point / group_point_grad (tf_grouping_g.cu:40-78; pointnet2 grouping_operation).  The reference runs one CTA
// per batch element; here one thread per output element, coalesced along the channel (BNC) or neighbour (BCN) axis.
// The gradient gathers deterministically per source point instead of atomicAdd.
// ------------------------------------------------------------------------------------------------------------------
template <int kLayout>
__global__ void group_point_kernel(int b, int n, int c, int m, int ns, const float *__restrict__ points, const int *__restrict__ idx,
                                   float *__restrict__ out)
{
    const size_t total = (size_t)b * m * ns * c;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        if (kLayout == SNB200_BNC) {  // out (b, m, ns, c)
            const int l = e % c;
            const size_t r = e / c;  // (b, m, ns) flattened
            const int bi = r / ((size_t)m * ns);
            const int ii = idx[r];
            out[e] = points[((size_t)bi * n + ii) * c + l];
        } else {  // out (b, c, m, ns), points (b, c, n)
            const size_t mn = (size_t)m * ns;
            const size_t r = e % mn;
            const size_t bc = e / mn;
            const int bi = bc / c;
            const int ii = idx[(size_t)bi * mn + r];
            out[e] = points[bc * n + ii];
        }
    }
}

template <int kLayout>
__global__ void __launch_bounds__(256) group_point_grad_kernel(int b, int n, int c, int m, int ns, const float *__restrict__ grad_out,
                                                               const int *__restrict__ idx, float *__restrict__ grad_points)
{
    __shared__ int s_idx[kGatherTile];
    const int bi = blockIdx.y;
    const int p = blockIdx.x * 256 + threadIdx.x;
    const int mk = m * ns;
    const bool live = p < n;
    float *gp = grad_points + (size_t)bi * n * c;
    if (live)
        for (int l = 0; l < c; l++) { if (kLayout == SNB200_BNC) gp[(size_t)p * c + l] = 0.f; else gp[(size_t)l * n + p] = 0.f; }
    for (int t0 = 0; t0 < mk; t0 += kGatherTile) {
        const int tn = min(kGatherTile, mk - t0);
        __syncthreads();
        for (int i = threadIdx.x; i < tn; i += 256) s_idx[i] = idx[(size_t)bi * mk + t0 + i];
        __syncthreads();
        if (live) {
            for (int i = 0; i < tn; i++) {
                if (s_idx[i] == p) {
                    for (int l = 0; l < c; l++) {
                        if (kLayout == SNB200_BNC) gp[(size_t)p * c + l] += grad_out[((size_t)bi * mk + t0 + i) * c + l];
                        else gp[(size_t)l * n + p] += grad_out[((size_t)bi * c + l) * mk + t0 + i];
                    }
                }
            }
        }
    }
}

int launch_group_point(int b, int n, int c, int m, int ns, int layout, const float *points, const int *idx, float *out, cudaStream_t stream)
{
    const size_t total = (size_t)b * m * ns * c;
    size_t nb = (total + 255) / 256;
    if (nb > (size_t)kNumSMs * 16) nb = (size_t)kNumSMs * 16;
    const int blocks = (int)nb;
    if (layout == SNB200_BNC) group_point_kernel<SNB200_BNC><<<blocks, 256, 0, stream>>>(b, n, c, m, ns, points, idx, out);
    else group_point_kernel<SNB200_BCN><<<blocks, 256, 0, stream>>>(b, n, c, m, ns, points, idx, out);
    return check_launch("group_point");
}

int launch_group_point_grad(int b, int n, int c, int m, int ns, int layout, const float *grad_out, const int *idx, float *grad_points,
                            cudaStream_t stream)
{
    dim3 grid((n + 255) / 256, b);
    if (layout == SNB200_BNC) group_point_grad_kernel<SNB200_BNC><<<grid, 256, 0, stream>>>(b, n, c, m, ns, grad_out, idx, grad_points);
    else group_point_grad_kernel<SNB200_BCN><<<grid, 256, 0, stream>>>(b, n, c, m, ns, grad_out, idx, grad_points);
    return check_launch("group_point_grad");
}

}  // namespace snb
