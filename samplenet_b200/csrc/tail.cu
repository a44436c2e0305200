// tail.cu -- the SampleNet step's tail in ONE launch: soft projection of the generated points (fused kNN + softmax + gather),
// Chamfer nn_distance between generated and input cloud (both directions) and the three simplification-loss reductions.
//
// In the reference these are knn_cuda.KNN + grouping + ~8 torch ops (samplenet.py:114), then -- when the trainer asks for the
// loss -- two Chamfer launches and four reductions (samplenet.py:175-180).  The projection and the Chamfer distances depend
// only on (x, simp), not on each other, so they run as different CTA roles of one grid: the projection CTAs also deliver the
// generated->input Chamfer direction (the nearest neighbour is the head of the top-k list), the other CTAs scan input->generated;
// the per-CTA partial sums / maxima are combined by the last CTA to finish (ticket counter) in a fixed order, which keeps the
// loss bit-reproducible.  Launched with the programmatic-dependent-launch attribute: each role waits for the producer of `simp`
// (griddepcontrol.wait) only right before it first reads `simp`, after the input cloud's tile has been requested.
#include "pairwise_device.cuh"

namespace snb {

struct TailParams {
    SoftProjParams sp;      // kNN + projection role (BNC)
    ChamferParams ch;       // d[0]: samp -> ref, d[1]: ref -> samp
    int knn_ctas;           // CTAs along x of the projection role
    int b, n_samp, n_ref;
    float w21;              // weight of the ref->samp term
    float *partial;         // (b, chamfer_ctas, 2): per-CTA sum / max of its distances
    unsigned *ticket;       // zero before the launch; reset to zero by the last CTA
    float *out4;            // mean(d1), mean_b(max d1), mean(d2), loss
    unsigned smem_floats;   // dynamic shared memory available to the final reduction
};

constexpr int kTailQ = 2;   // queries register-blocked per thread in the input->generated scan

template <bool kFma>
__global__ void __launch_bounds__(256) tail_fused_kernel(const __grid_constant__ TailParams P)
{
    extern __shared__ __align__(16) float s_dyn[];
    __shared__ uint64_t bar;
    __shared__ float s_rs[8], s_rm[8];
    __shared__ unsigned s_ticket;
    // 1-D grid, projection CTAs first: they are the long pole (a dependent top-k chain per query), so they must all be in the
    // first wave; the short Chamfer tiles fill in behind them.  The projection role also IS the generated->input Chamfer
    // direction: the nearest neighbour of a query is lane 0 of its top-k list (same arithmetic, same lowest-index tie rule), so
    // dist1 / idx1 and their loss reductions come out of it for free and only the input->generated direction is scanned separately.
    // Programmatic dependent launch: this grid may be scheduled while the producer of `samp` (the generator kernel) is still
    // draining -- its launch latency, CTA start-up and the staging of the input cloud are hidden -- and each role executes
    // griddepcontrol.wait (previous grid complete and flushed) right before its first read of `samp`.
    const int n_knn = P.b * P.knn_ctas;
    const int ntiles = P.knn_ctas + P.ch.d[1].tiles;      // partial slots per cloud: projection CTAs, then direction-1 tiles
    float my_sum = 0.f, my_max = -INFINITY;
    int bi, slot;
    if ((int)blockIdx.x < n_knn) {   // ---- role A: projection + direction 0
        bi = (int)blockIdx.x / P.knn_ctas;
        slot = (int)blockIdx.x % P.knn_ctas;
        knn_softproj_body<SNB200_BNC, kFma>(P.sp, slot, bi, s_dyn, &bar, &my_sum, &my_max, true);   // waits on the previous grid itself
    } else {                         // ---- role B: one tile of direction 1
        bi = ((int)blockIdx.x - n_knn) / P.ch.d[1].tiles;
        const int cx = ((int)blockIdx.x - n_knn) % P.ch.d[1].tiles;
        slot = P.knn_ctas + cx;
        if (threadIdx.x == 0) {
            mbar_init(&bar, 1);
            fence_mbar_init();
        }
        __syncthreads();
        asm volatile("griddepcontrol.wait;" ::: "memory");     // the candidates ARE the previous grid's output
        chamfer_dir<kTailQ, kFma>(P.ch.d[1], cx, bi, s_dyn, &bar, &my_sum, &my_max);
    }
    // CTA partials (fixed order: warp shuffle tree, then warps in index order)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    my_sum = warp_sum(my_sum);
    my_max = warp_max(my_max);
    if (lane == 0) { s_rs[warp] = my_sum; s_rm[warp] = my_max; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float ts = 0.f, tm = -INFINITY;
        for (int w = 0; w < 8; w++) { ts += s_rs[w]; tm = fmaxf(tm, s_rm[w]); }
        float *pp = P.partial + ((size_t)bi * ntiles + slot) * 2;
        pp[0] = ts; pp[1] = tm;
        __threadfence();
        s_ticket = atomicAdd(P.ticket, 1u);
    }
    __syncthreads();
    if (s_ticket != (unsigned)(P.b * ntiles) - 1u) return;
    // ---- last CTA: combine (every partial is visible: each writer fenced before taking its ticket).  The partials are pulled
    //      into shared memory with all loads in flight (one L2 round trip), then summed per cloud and across clouds in a fixed order.
    __threadfence();
    __shared__ float s_a[256], s_b[256], s_c[256];
    float a1 = 0.f, amax = 0.f, a2 = 0.f;
    const int t0 = P.knn_ctas;
    float2 *s_p = reinterpret_cast<float2 *>(s_dyn);
    const int cap_clouds = max(1, (int)(P.smem_floats / 2) / ntiles);           // clouds per shared-memory pass
    for (int cbase = 0; cbase < P.b; cbase += cap_clouds) {
        const int nc = min(cap_clouds, P.b - cbase);
        const int ne = nc * ntiles;
        __syncthreads();
        const float2 *src = reinterpret_cast<const float2 *>(P.partial) + (size_t)cbase * ntiles;
        for (int e0 = threadIdx.x; e0 < ne; e0 += 256 * 4) {
            float2 v[4];
#pragma unroll
            for (int u = 0; u < 4; u++) v[u] = (e0 + u * 256 < ne) ? __ldcg(src + e0 + u * 256) : make_float2(0.f, 0.f);
#pragma unroll
            for (int u = 0; u < 4; u++)
                if (e0 + u * 256 < ne) s_p[e0 + u * 256] = v[u];
        }
        __syncthreads();
        for (int c = threadIdx.x; c < nc; c += 256) {
            const float2 *pp = s_p + (size_t)c * ntiles;
            float s1 = 0.f, mx = -INFINITY, s2 = 0.f;
            for (int t = 0; t < t0; t++) { s1 += pp[t].x; mx = fmaxf(mx, pp[t].y); }
            for (int t = t0; t < ntiles; t++) s2 += pp[t].x;
            a1 += s1; amax += mx; a2 += s2;
        }
    }
    s_a[threadIdx.x] = a1; s_b[threadIdx.x] = amax; s_c[threadIdx.x] = a2;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            s_a[threadIdx.x] += s_a[threadIdx.x + s]; s_b[threadIdx.x] += s_b[threadIdx.x + s]; s_c[threadIdx.x] += s_c[threadIdx.x + s];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float c12 = s_a[0] / ((float)P.b * (float)P.n_samp);
        const float mc = s_b[0] / (float)P.b;
        const float c21 = s_c[0] / ((float)P.b * (float)P.n_ref);
        P.out4[0] = c12; P.out4[1] = mc; P.out4[2] = c21;
        P.out4[3] = c12 + mc + P.w21 * c21;
        *P.ticket = 0u;   // ready for the next launch
    }
}

// The launch plan of tail_fused_kernel, computed in one place for the launcher, the workspace query and snb200_debug_project_and_loss_plan.
// One CTA per SM for direction 1 is enough here: the grid also carries the projection CTAs and should stay within a single wave.
struct TailPlan {
    int knn_ctas;       // projection CTAs per cloud (kSpWarps queries each)
    int s1, tiles1;     // direction 1 (ref -> samp): lanes per query, CTAs per cloud
    int ntiles;         // partial slots per cloud: knn_ctas + tiles1
    size_t smem;        // dynamic shared memory: one staged cloud, at least 4 KB for the final reduction
    int cap_clouds;     // clouds the final reduction stages per pass (the kernel's own formula)
    int tma_preissue;   // the projection role requests the cloud by TMA before griddepcontrol.wait (also needs a 16-byte aligned ref)
};

static TailPlan tail_plan(int b, int n_ref, int n_samp)
{
    TailPlan T;
    T.knn_ctas = (n_samp + kSpWarps - 1) / kSpWarps;
    ChamferDir d1 = {nullptr, nullptr, nullptr, nullptr, n_ref, n_samp, 1, 0};
    plan_chamfer_dir(d1, b, kTailQ, kNumSMs);
    T.s1 = d1.S; T.tiles1 = d1.tiles;
    T.ntiles = T.knn_ctas + T.tiles1;
    T.smem = (size_t)min(max(n_ref, n_samp), kSpTile) * 3 * sizeof(float);
    if (T.smem < 4096) T.smem = 4096;
    T.cap_clouds = max(1, (int)(T.smem / sizeof(float) / 2) / T.ntiles);
    T.tma_preissue = n_ref % 4 == 0;
    return T;
}

void tail_plan_query(int b, int n_ref, int n_samp, int *knn_ctas, int *s1, int *tiles1, int *ntiles, int *smem_floats, int *cap_clouds, int *tma_preissue)
{
    const TailPlan T = tail_plan(b, n_ref, n_samp);
    *knn_ctas = T.knn_ctas; *s1 = T.s1; *tiles1 = T.tiles1; *ntiles = T.ntiles;
    *smem_floats = (int)(T.smem / sizeof(float)); *cap_clouds = T.cap_clouds; *tma_preissue = T.tma_preissue;
}

size_t tail_workspace_bytes(int b, int n_samp, int n_ref)
{
    return (size_t)b * tail_plan(b, n_ref, n_samp).ntiles * 2 * sizeof(float);
}

int launch_tail_fused(int b, int n_ref, int n_samp, int k, const float *ref, const float *samp, const float *sigma, int sigma_mode, float sigma_floor,
                      float *proj, int *knn_idx, float *weights, float *dist_over_sigma, float *dist1, int *idx1, float *dist2, int *idx2,
                      float w21, float *out4, float *partial, unsigned *ticket, int flags, cudaStream_t stream)
{
    const TailPlan T = tail_plan(b, n_ref, n_samp);
    TailParams P;
    memset(&P, 0, sizeof(P));
    SoftProjParams &S = P.sp;
    S.b = b; S.n = n_ref; S.m = n_samp; S.k = k; S.f = 0; S.queries_per_warp = 1;
    S.points = ref; S.query = samp; S.sigma = sigma; S.sigma_mode = sigma_mode; S.sigma_floor = sigma_floor; S.hard = 0;
    S.proj = proj; S.knn_idx = knn_idx; S.weights = weights; S.dist_over_sigma = dist_over_sigma;
    P.knn_ctas = T.knn_ctas;
    P.ch.d[0] = {samp, ref, dist1, idx1, n_samp, n_ref, 1, 0};
    P.ch.d[1] = {ref, samp, dist2, idx2, n_ref, n_samp, T.s1, T.tiles1};
    P.ch.d[0].tiles = 0;            // direction 0 (generated -> input) rides on the projection role
    S.nn_dist = dist1; S.nn_idx = idx1;
    P.b = b; P.n_samp = n_samp; P.n_ref = n_ref; P.w21 = w21; P.partial = partial; P.ticket = ticket; P.out4 = out4;
    P.smem_floats = (unsigned)(T.smem / sizeof(float));
    static PerDeviceOnce once;
    if (once.first()) {
        cudaFuncSetAttribute(tail_fused_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
        cudaFuncSetAttribute(tail_fused_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 56 * 1024);
        cudaFuncSetAttribute(tail_fused_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(tail_fused_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    }
    dim3 grid((unsigned)((long long)b * T.ntiles));
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid; cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = T.smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;     // may start before the previous kernel of the stream has drained
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    cudaError_t e = (flags & SNB200_DIST_UNFUSED) ? cudaLaunchKernelEx(&cfg, tail_fused_kernel<false>, P) : cudaLaunchKernelEx(&cfg, tail_fused_kernel<true>, P);
    if (e != cudaSuccess) { set_error("project_and_simplification_loss: launch failed: %s", cudaGetErrorString(e)); cudaGetLastError(); return SNB200_ECUDA; }
    return check_launch("project_and_simplification_loss");
}

}  // namespace snb
