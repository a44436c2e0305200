// generator.cu -- orchestration of the whole SampleNet generator (samplenet.py:90-104): path selection, workspace layout, and the
// cluster pool + FC-head kernel of the non-fused paths and of the stand-alone encoder / FC-head entry points (encoder.cu).
//
//   path (training step at the headline size)                                          launches
//   default        cudaMemsetAsync(statistics, barrier word, FC exchange buffers)         (memset node)
//                  conv_stack_kernel   conv 1..5 + pool + fc1..fc4, persistent cooperative   1      (conv_stack.cu)
//   per-layer      memset; x_moments_kernel; tc_layer_kernel x4; fc_head_cluster_kernel      6      (encoder_tc.cu, here)
//   exact fp32     memset; conv_layer_kernel x5; fc_head_cluster_kernel                      6      (encoder.cu, here)
//   The default applies when the conv widths are 32/64/128 and the batch has at most 32 slices of 128 points per SM
//   (conv_stack_supported: one slice per SM keeps activations in registers; with more than one, up to two slices per SM stay in shared
//   memory between layers and the rest park in L2 -- still one launch); everything else falls through to the per-layer tensor-core path, then to exact fp32.
//   plan_generator makes every one of these decisions once (conv path, fused head, self-cleaning workspace, the pool partials per cloud
//   the head reads); launch_generator_forward then runs the conv stage and, unless it is fused, the cluster head.
//
// fc_head_cluster_kernel: the FC head (samplenet.py:99-104: 128->256->256->256->3M on B rows, BatchNorm over the batch) is tiny
// (7 MFLOP, 0.86 MB of weights) but has four layer-to-layer dependencies.  ONE thread-block cluster of 16 CTAs runs all of it:
// every CTA owns a slice of the output channels of each layer (so BatchNorm over the batch never leaves a warp: lane = batch
// row), activations are exchanged through a 32 KB global scratch that stays in L2, and layers are separated by cluster
// barriers.  The same kernel first turns the last conv layer's per-tile extrema into the pooled feature and applies every
// BatchNorm running-statistics update exactly once.  (The default path runs the head inside conv_stack_kernel instead.)  Either half
// can run alone: snb200_encoder_forward launches it with no FC layers, snb200_fc_head_forward with no pool (tile_max == nullptr).
#include "encoder_internal.cuh"
#include <cooperative_groups.h>
#include <string.h>
namespace cg = cooperative_groups;

namespace snb {

constexpr int kHeadThreads = 256;      // 8 warps = 8 K slices; lanes = 8 row quads x 4 channel quads
constexpr int kHeadChPerCta = 16;
constexpr int kHeadMaxCluster = 16;
constexpr int kHeadSmemBytes = 200 * 1024;
// row stride (floats) of a layer's weight slice in shared memory: 4 floats of padding, and a multiple of 4 whatever c_in so that the
// float4 weight reads stay 16-byte aligned
__host__ __device__ constexpr int head_ldw(int c_in) { return ((c_in + 3) & ~3) + 4; }

// RG = number of 32-row groups of the batch (b <= 32*RG).  256 threads = 8 warps.
// Everything here is a latency chain (4 dependent layers on <= 256 rows), so the kernel is organised around keeping loads
// off that chain and shared-memory wavefronts low:
//   * the weight slices of ALL layers do not depend on activations: they are fetched by TMA bulk copies (one mbarrier per
//     layer, one row per issuing thread) the moment the kernel starts;
//   * per-channel parameters (bias, gamma, beta, running stats) are read into registers before the layer's math;
//   * the per-CTA product [32 rows x c_in] x [c_in x 16 channels] is register-tiled 4 rows x 4 channels per thread with the
//     K range split over the 8 warps (2 LDS.128 wavefronts per 16 FMAs), partial sums are combined through shared memory in a
//     fixed order, and the combine leaves lane = batch row, warp = channel so BatchNorm over the batch is two warp shuffles.
template <int RG>
__global__ void __launch_bounds__(kHeadThreads) fc_head_cluster_kernel(const __grid_constant__ HeadParams P)
{
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = cluster.block_rank(), csize = cluster.num_blocks();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    extern __shared__ __align__(16) float smem[];
    __shared__ uint64_t wbar[SNB200_MAX_FC_LAYERS];
    __shared__ float *s_wptr[SNB200_MAX_FC_LAYERS];
    // s_in  : [k_chunk][36]          one row group of a K range of the input, transposed (k-major), 4-row float4 reads
    // s_w   : per layer [16][ldw]     this CTA's first 16-channel weight slice, row-major like in HBM (head_ldw)
    // s_part: [8 warps][32 rows][17]  partial dot products of the K slices
    const int kch = P.k_chunk;
    float *s_in = smem;
    float *s_part;
    if (tid == 0) {
        float *p = smem + (size_t)kch * 36;
        for (int l = 0; l < P.num_fc; l++) { s_wptr[l] = p; p += (size_t)kHeadChPerCta * head_ldw(P.fc[l].c_in); }
        for (int l = 0; l < P.num_fc; l++) mbar_init(&wbar[l], 1);
        fence_mbar_init();
        for (int l = 0; l < P.num_fc; l++) {   // arm every layer's barrier with the bytes its slice will deliver
            const HeadLayer &L = P.fc[l];
            const int per_cta = (L.c_out + csize - 1) / csize;
            const int c_lo = rank * per_cta, c_hi = min(L.c_out, c_lo + per_cta);
            const int nch = max(0, min(kHeadChPerCta, c_hi - c_lo));
            const bool tma_ok = (L.c_in & 3) == 0 && (reinterpret_cast<uintptr_t>(L.weight) & 15) == 0;
            if (tma_ok && nch > 0) mbar_expect_tx(&wbar[l], (uint32_t)nch * L.c_in * 4u);
        }
    }
    __syncthreads();
    {
        float *p = smem + (size_t)kch * 36;
        for (int l = 0; l < P.num_fc; l++) p += (size_t)kHeadChPerCta * head_ldw(P.fc[l].c_in);
        s_part = p;
    }
    // ---- weight prefetch: thread t issues row (t % 16) of layer (t / 16)
    if (tid < P.num_fc * kHeadChPerCta) {
        const int l = tid / kHeadChPerCta, jrow = tid % kHeadChPerCta;
        const HeadLayer &L = P.fc[l];
        const int per_cta = (L.c_out + csize - 1) / csize;
        const int c_lo = rank * per_cta, c_hi = min(L.c_out, c_lo + per_cta);
        const int nch = max(0, min(kHeadChPerCta, c_hi - c_lo));
        const bool tma_ok = (L.c_in & 3) == 0 && (reinterpret_cast<uintptr_t>(L.weight) & 15) == 0;
        if (tma_ok && jrow < nch)
            tma_load_1d(s_wptr[l] + (size_t)jrow * head_ldw(L.c_in), L.weight + (size_t)(c_lo + jrow) * L.c_in, (uint32_t)L.c_in * 4u, &wbar[l]);
    }

    // ---- phase 0: pooled feature (this CTA's share) and the conv stack's running statistics (spread over the cluster).
    // tile_max == nullptr: the caller gives the FC input in feat, and there is nothing to pool.
    if (P.tile_max) {
        const int total = P.b * P.c_feat;
        const double inv = 1.0 / P.count;
        for (int e = rank * kHeadThreads + tid; e < total; e += csize * kHeadThreads) {
            const int bi = e / P.c_feat, c = e % P.c_feat;
            float mx = -INFINITY, mn = INFINITY;
            const float *tm = P.tile_max + (size_t)bi * P.tiles_per_cloud * P.c_feat + c;
            const float *tn = P.tile_min + (size_t)bi * P.tiles_per_cloud * P.c_feat + c;
#pragma unroll 8
            for (int t = 0; t < P.tiles_per_cloud; t++) {
                mx = fmaxf(mx, __ldg(tm + (size_t)t * P.c_feat));
                mn = fminf(mn, __ldg(tn + (size_t)t * P.c_feat));
            }
            float v = mx;
            if (P.last_has_bn) {
                float mean, var;
                if (P.training) {
                    const double m = P.last_stats[c] * inv;
                    double vv = P.last_stats[P.c_feat + c] * inv - m * m;
                    if (vv < 0) vv = 0;
                    mean = (float)m; var = (float)vv;
                } else {
                    mean = P.last_run_mean[c]; var = P.last_run_var[c];
                }
                const float sc = P.last_gamma[c] * (1.0f / sqrtf(var + P.last_eps));
                const float sh = P.last_beta[c] - mean * sc;
                v = sc >= 0.f ? fmaf(mx, sc, sh) : fmaf(mn, sc, sh);  // max over points of a monotone map
            }
            if (P.last_relu) v = fmaxf(v, 0.f);
            P.feat[e] = v;
            if (P.keep_inputs) P.ll[0][e] = v;
        }
        if (P.training) {   // training mode never reads the running buffers, so the update can go anywhere in the kernel
            int base = 0;
            const int gt = rank * kHeadThreads + tid, gn = csize * kHeadThreads;
            for (int l = 0; l < P.ru_num; l++) {
                for (int c = gt - base; c < P.ru_c[l]; c += gn) {
                    if (c < 0) continue;
                    const double m = P.ru_stats[l][c] * inv;
                    double v = P.ru_stats[l][P.ru_c[l] + c] * inv - m * m;
                    if (v < 0) v = 0;
                    const double unb = P.count > 1 ? v * (P.count / (P.count - 1)) : v;
                    const float mom = P.ru_momentum[l];
                    if (P.ru_mean[l]) P.ru_mean[l][c] = (1.f - mom) * P.ru_mean[l][c] + mom * (float)m;
                    if (P.ru_var[l]) P.ru_var[l][c] = (1.f - mom) * P.ru_var[l][c] + mom * (float)unb;
                }
                base = (base + P.ru_c[l]) % gn;
            }
        }
    }
    if (rank == csize - 1 && tid < P.num_counters) *P.counters[tid] += 1;
    cluster.sync();

    // ---- FC layers
    const float *cur = P.feat;
    for (int l = 0; l < P.num_fc; l++) {
        const HeadLayer &L = P.fc[l];
        const bool last = (l == P.num_fc - 1);
        float *dst = last ? P.out : (P.keep_inputs ? P.ll[l + 1] : P.act[l & 1]);   // kept: the next layer's input, read by its backward
        const int c_in = L.c_in, ldw = head_ldw(c_in);
        const int per_cta = (L.c_out + csize - 1) / csize;
        const int c_lo = rank * per_cta, c_hi = min(L.c_out, c_lo + per_cta);
        const bool vec = (c_in & 3) == 0;   // input rows are then read as float4: fc1's input must be 16-byte aligned
        const bool tma_ok = vec && (reinterpret_cast<uintptr_t>(L.weight) & 15) == 0;
        float *sw = s_wptr[l];
        for (int cb = c_lo; cb < c_hi; cb += kHeadChPerCta) {      // passes of 16 channels (one pass unless c_out > 16*cluster)
            const int nch = min(kHeadChPerCta, c_hi - cb);
            // per-channel parameters of the two channels this warp finishes (warp, warp+8): loads start now
            float pb[2], pg[2], pbe[2], prm[2], prv[2];
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const int c = cb + warp + 8 * j;
                const bool cv = (warp + 8 * j) < nch;
                pb[j] = (cv && L.bias) ? __ldg(L.bias + c) : 0.f;
                pg[j] = (cv && L.has_bn) ? __ldg(L.gamma + c) : 1.f;
                pbe[j] = (cv && L.has_bn) ? __ldg(L.beta + c) : 0.f;
                prm[j] = (cv && L.has_bn && L.run_mean) ? L.run_mean[c] : 0.f;
                prv[j] = (cv && L.has_bn && L.run_var) ? L.run_var[c] : 1.f;
            }
            if (cb == c_lo && tma_ok) {
                mbar_wait(&wbar[l], 0);                           // prefetched slice has landed
            } else {
                __syncthreads();
                for (int e = tid; e < kHeadChPerCta * c_in; e += kHeadThreads) {
                    const int jr = e / c_in, k = e % c_in;
                    sw[jr * ldw + k] = (jr < nch) ? __ldg(L.weight + (size_t)(cb + jr) * c_in + k) : 0.f;
                }
            }
            float y[RG][2];   // finished pre-activation of (row = g*32 + lane, channel = warp + 8*j)
#pragma unroll
            for (int g = 0; g < RG; g++) {
                y[g][0] = 0.f; y[g][1] = 0.f;
                const int r0 = g * 32;
                if (r0 < P.b) {   // uniform
                    const int rn = min(32, P.b - r0);
                    // register-tiled partial product: lane -> rows 4*rg..+3, channels cgp, cgp+4, cgp+8, cgp+12 (bank-conflict-free weight reads);
                    // warp -> K slice
                    const int rg = lane & 7, cgp = lane >> 3;
                    const int kr = ((c_in + 31) / 32) * 4;                    // K per warp, multiple of 4
                    const int k_lo = warp * kr, k_hi = min(c_in, k_lo + kr);
                    float acc[4][4];
#pragma unroll
                    for (int r = 0; r < 4; r++)
#pragma unroll
                        for (int j = 0; j < 4; j++) acc[r][j] = 0.f;
                    // the input's K range is staged k_chunk at a time (one chunk unless the layer is too wide for the tile; k_chunk is then
                    // a multiple of 4): every warp still walks its K slice in ascending k with the same groups of 4, so a chunked sum is
                    // the one-chunk sum
                    for (int kc0 = 0; kc0 < c_in; kc0 += kch) {
                        const int kc1 = min(c_in, kc0 + kch);
                        __syncthreads();
                        // input rows r0..r0+rn-1, transposed into s_in[k - kc0][r]; written by other CTAs of this kernel: plain loads,
                        // all of a thread's loads in flight before the first store
                        if (vec) {
                            // lane = batch row (conflict-free transposed stores), warps stride over the 16-byte k groups;
                            // up to 8 loads per thread in flight before the first store
                            const int q = (kc1 - kc0) >> 2;
                            const float *src = cur + (size_t)(r0 + min(lane, rn - 1)) * c_in + kc0;
                            for (int q0 = warp; q0 < q; q0 += 8 * 8) {
                                float4 v[8];
#pragma unroll
                                for (int u = 0; u < 8; u++) {
                                    const int kq = q0 + 8 * u;
                                    v[u] = (kq < q) ? *(reinterpret_cast<const float4 *>(src) + kq) : make_float4(0, 0, 0, 0);
                                }
#pragma unroll
                                for (int u = 0; u < 8; u++) {
                                    const int kq = q0 + 8 * u;
                                    if (kq < q) {
                                        const float4 t = (lane < rn) ? v[u] : make_float4(0, 0, 0, 0);
                                        s_in[(kq * 4 + 0) * 36 + lane] = t.x; s_in[(kq * 4 + 1) * 36 + lane] = t.y;
                                        s_in[(kq * 4 + 2) * 36 + lane] = t.z; s_in[(kq * 4 + 3) * 36 + lane] = t.w;
                                    }
                                }
                            }
                        } else {
                            for (int e = tid; e < 32 * (kc1 - kc0); e += kHeadThreads) {
                                const int r = e & 31, k = e >> 5;
                                s_in[k * 36 + r] = (r < rn) ? cur[(size_t)(r0 + r) * c_in + kc0 + k] : 0.f;
                            }
                        }
                        __syncthreads();
                        int k = max(k_lo, kc0);
                        const int ke = min(k_hi, kc1);
                        for (; k + 4 <= ke; k += 4) {
                            float4 a[4], wv[4];
#pragma unroll
                            for (int i = 0; i < 4; i++) a[i] = *reinterpret_cast<const float4 *>(s_in + (k - kc0 + i) * 36 + rg * 4);
#pragma unroll
                            for (int j = 0; j < 4; j++) wv[j] = *reinterpret_cast<const float4 *>(sw + (cgp + 4 * j) * ldw + k);
#pragma unroll
                            for (int j = 0; j < 4; j++) {
                                acc[0][j] = fmaf(a[3].x, wv[j].w, fmaf(a[2].x, wv[j].z, fmaf(a[1].x, wv[j].y, fmaf(a[0].x, wv[j].x, acc[0][j]))));
                                acc[1][j] = fmaf(a[3].y, wv[j].w, fmaf(a[2].y, wv[j].z, fmaf(a[1].y, wv[j].y, fmaf(a[0].y, wv[j].x, acc[1][j]))));
                                acc[2][j] = fmaf(a[3].z, wv[j].w, fmaf(a[2].z, wv[j].z, fmaf(a[1].z, wv[j].y, fmaf(a[0].z, wv[j].x, acc[2][j]))));
                                acc[3][j] = fmaf(a[3].w, wv[j].w, fmaf(a[2].w, wv[j].z, fmaf(a[1].w, wv[j].y, fmaf(a[0].w, wv[j].x, acc[3][j]))));
                            }
                        }
                        for (; k < ke; k++) {
                            const float4 a = *reinterpret_cast<const float4 *>(s_in + (k - kc0) * 36 + rg * 4);
#pragma unroll
                            for (int j = 0; j < 4; j++) {
                                const float wj = sw[(cgp + 4 * j) * ldw + k];
                                acc[0][j] = fmaf(a.x, wj, acc[0][j]); acc[1][j] = fmaf(a.y, wj, acc[1][j]);
                                acc[2][j] = fmaf(a.z, wj, acc[2][j]); acc[3][j] = fmaf(a.w, wj, acc[3][j]);
                            }
                        }
                    }
#pragma unroll
                    for (int r = 0; r < 4; r++)
#pragma unroll
                        for (int j = 0; j < 4; j++) s_part[(warp * 32 + rg * 4 + r) * 17 + cgp + 4 * j] = acc[r][j];
                    __syncthreads();
#pragma unroll
                    for (int j = 0; j < 2; j++) {   // fixed-order combination of the 8 K slices: lane = row, warp (+8) = channel
                        float t = 0.f;
#pragma unroll
                        for (int w8 = 0; w8 < 8; w8++) t += s_part[(w8 * 32 + lane) * 17 + warp + 8 * j];
                        y[g][j] = t;
                    }
                }
            }
            // bias, BatchNorm over the batch (rows live in lanes x row groups), activation, store
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const int c = cb + warp + 8 * j;
                const bool cv = (warp + 8 * j) < nch;   // warp-uniform
                float scale = 1.f, shift = 0.f;
#pragma unroll
                for (int g = 0; g < RG; g++) y[g][j] += pb[j];
                if (L.has_bn && cv) {
                    float mean, var;
                    if (P.training) {
                        float sm = 0.f;
#pragma unroll
                        for (int g = 0; g < RG; g++)
                            if (g * 32 + lane < P.b) sm += y[g][j];
                        mean = warp_sum(sm) / (float)P.b;
                        float q = 0.f;
#pragma unroll
                        for (int g = 0; g < RG; g++)
                            if (g * 32 + lane < P.b) { const float d = y[g][j] - mean; q = fmaf(d, d, q); }
                        q = warp_sum(q);
                        var = q / (float)P.b;
                        if (lane == 0) {
                            const float unb = P.b > 1 ? q / (float)(P.b - 1) : var;
                            if (L.run_mean) L.run_mean[c] = (1.f - L.momentum) * prm[j] + L.momentum * mean;
                            if (L.run_var) L.run_var[c] = (1.f - L.momentum) * prv[j] + L.momentum * unb;
                        }
                    } else {
                        mean = prm[j]; var = prv[j];
                    }
                    const float invstd = 1.0f / sqrtf(var + L.eps);
                    scale = pg[j] * invstd;
                    shift = pbe[j] - mean * scale;
                }
                if (cv) {
#pragma unroll
                    for (int g = 0; g < RG; g++) {
                        const int row = g * 32 + lane;
                        if (row < P.b) {
                            float v = L.has_bn ? fmaf(y[g][j], scale, shift) : y[g][j];
                            if (L.relu) v = fmaxf(v, 0.f);
                            // the next layer's dropout: its input, and what its backward reads as that input, is the masked value
                            if (L.out_mask) v *= __ldg(L.out_mask + (size_t)row * L.c_out + c);
                            const int oc = (last && P.out_inner > 0) ? (c % P.out_inner) * (L.c_out / P.out_inner) + c / P.out_inner : c;
                            dst[(size_t)row * L.c_out + oc] = v;
                        }
                    }
                }
            }
        }
        cur = dst;
        cluster.sync();   // the next layer reads every CTA's slice
    }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
struct GenWorkspace {
    float *act[2];
    char *stats_base; size_t stats_bytes;
    double *mom; unsigned *counter; float *ll[SNB200_MAX_FC_LAYERS + 1];
    double *stats[SNB200_MAX_CONV_LAYERS];
    float *tile_max, *tile_min;
    float *feat;
    float *head_act[2];
    size_t total;
};

static GenWorkspace carve_gen_ws(void *base, int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc)
{
    GenWorkspace W{};
    WsCarver c(base);
    // the first 256 bytes: the input moments (16 doubles), then the grid-barrier and exit words -- the words a SNB200_GEN_WORKSPACE_PRIMED
    // caller keeps zero between calls (include/samplenet_b200.h), so they lead the workspace
    const size_t stats_off = c.off;
    W.stats_base = c.take<char>(256);
    W.mom = reinterpret_cast<double *>(W.stats_base);
    W.counter = reinterpret_cast<unsigned *>(W.stats_base + 16 * sizeof(double));
    for (int l = 0; l < nconv; l++)   // canonical [2C] block + one line per accumulator
        W.stats[l] = c.take<double>((size_t)(1 + kStatStride) * 2 * conv[l].c_out);
    for (int l = 0; l < nfc; l++)   // exchange buffers of the fused head (zeroed with the statistics): the input of FC layer l, null beyond
        W.ll[l] = c.take<float>((size_t)b * (l == 0 ? conv[nconv - 1].c_out : fc[l - 1].c_out));
    W.stats_bytes = c.off - stats_off;
    int maxc = 8;
    for (int l = 0; l + 1 < nconv; l++) maxc = max(maxc, conv[l].c_out);
    W.act[0] = c.take<float>((size_t)b * n * maxc);
    W.act[1] = c.take<float>((size_t)b * n * maxc);
    const int c_last = conv[nconv - 1].c_out;
    const int tpc = max((n + 127) / 128, (n + 63) / 64 + 1);  // upper bound over all paths (128- / 256-point tiles; conv-stack (cloud, CTA) slots)
    W.tile_max = c.take<float>((size_t)b * tpc * c_last);
    W.tile_min = c.take<float>((size_t)b * tpc * c_last);
    W.feat = c.take<float>((size_t)b * c_last);
    int maxf = 8;
    for (int l = 0; l < nfc; l++) maxf = max(maxf, fc[l].c_out);
    W.head_act[0] = c.take<float>((size_t)b * maxf);
    W.head_act[1] = c.take<float>((size_t)b * maxf);
    W.total = c.off;
    return W;
}

size_t generator_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc)
{
    return carve_gen_ws(nullptr, b, n, nconv, conv, nfc, fc).total;
}

void fill_pool_params(HeadParams &H, int b, int n, int tpc, int nconv, const snb200_layer *conv, int training, double *const *stats,
                      float *tile_max, float *tile_min, float *feat)
{
    const snb200_layer &LL = conv[nconv - 1];
    H.b = b; H.training = training; H.c_feat = LL.c_out; H.tiles_per_cloud = tpc;
    H.tile_max = tile_max; H.tile_min = tile_min; H.last_stats = stats[nconv - 1];
    H.last_gamma = LL.bn_weight; H.last_beta = LL.bn_bias; H.last_run_mean = LL.bn_running_mean; H.last_run_var = LL.bn_running_var;
    H.last_eps = LL.bn_eps; H.last_has_bn = LL.bn_weight != nullptr; H.last_relu = LL.relu;
    H.count = (double)b * (double)n;
    H.feat = feat;
    if (!training) return;
    for (int l = 0; l < nconv; l++) {
        const snb200_layer &L = conv[l];
        if (!L.bn_weight) continue;
        if (L.bn_running_mean || L.bn_running_var) {
            H.ru_stats[H.ru_num] = stats[l]; H.ru_mean[H.ru_num] = L.bn_running_mean; H.ru_var[H.ru_num] = L.bn_running_var;
            H.ru_momentum[H.ru_num] = L.bn_momentum; H.ru_c[H.ru_num] = L.c_out;
            H.ru_num++;
        }
        if (L.bn_num_batches_tracked) H.counters[H.num_counters++] = L.bn_num_batches_tracked;
    }
}

void fill_fc_params(HeadParams &H, int nfc, const snb200_layer *fc, float *out, int out_transpose_inner)
{
    H.num_fc = nfc;
    for (int l = 0; l < nfc; l++) {
        HeadLayer &D = H.fc[l];
        D.c_in = fc[l].c_in; D.c_out = fc[l].c_out; D.weight = fc[l].weight; D.bias = fc[l].bias; D.gamma = fc[l].bn_weight; D.beta = fc[l].bn_bias;
        D.run_mean = fc[l].bn_running_mean; D.run_var = fc[l].bn_running_var; D.eps = fc[l].bn_eps; D.momentum = fc[l].bn_momentum;
        D.has_bn = fc[l].bn_weight != nullptr; D.relu = fc[l].relu;
        if (H.training && fc[l].bn_weight && fc[l].bn_num_batches_tracked) H.counters[H.num_counters++] = fc[l].bn_num_batches_tracked;
    }
    H.out = out; H.out_inner = out_transpose_inner;
}

static void fill_head_params(HeadParams &H, int b, int n, int tpc, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc, int training,
                             float *out, int out_transpose_inner, float *feat_out, const GenWorkspace &W)
{
    memset(&H, 0, sizeof(H));
    fill_pool_params(H, b, n, tpc, nconv, conv, training, W.stats, W.tile_max, W.tile_min, feat_out ? feat_out : W.feat);
    fill_fc_params(H, nfc, fc, out, out_transpose_inner);
    H.act[0] = W.head_act[0]; H.act[1] = W.head_act[1];
    for (int l = 0; l <= SNB200_MAX_FC_LAYERS; l++) H.ll[l] = W.ll[l];
}

// act_input: layer 1 reads an activation, so it is a tensor-core layer like the hidden ones
static bool tc_stack_supported(int nconv, const snb200_layer *conv, bool act_input)
{
    if (nconv < 2) return false;
    if (act_input ? !tc_layer_supported(conv[0].c_in, conv[0].c_out) : (conv[0].c_in != 3 || conv[0].c_out % 8 != 0 || conv[0].c_out > 256)) return false;
    for (int l = 1; l + 1 < nconv; l++)
        if (!tc_layer_supported(conv[l].c_in, conv[l].c_out)) return false;
    return tc_last_layer_supported(conv[nconv - 1].c_in, conv[nconv - 1].c_out);
}

GenWorkspaceView generator_workspace_view(void *fwd_workspace, int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc)
{
    GenWorkspace W = carve_gen_ws(fwd_workspace, b, n, nconv, conv, nfc, fc);
    GenWorkspaceView V;
    for (int l = 0; l < SNB200_MAX_CONV_LAYERS; l++) V.stats[l] = l < nconv ? W.stats[l] : nullptr;
    for (int l = 0; l <= SNB200_MAX_FC_LAYERS; l++) V.ll[l] = W.ll[l];
    return V;
}

// ---- path selection
enum class GenConv {
    Persistent,   // conv_stack_kernel (conv_stack.cu), one cooperative launch
    PerLayerTc,   // x_moments_kernel + tc_layer_kernel per layer (encoder_tc.cu)
    ExactFp32,    // conv_layer_kernel per layer (encoder.cu)
    HeadOnly,     // SNB200_GEN_PROFILE_SKIP_CONV: no conv stage, the head reads whatever the workspace holds
};
struct GenPlan {
    GenConv conv;
    bool fuse_head;        // the persistent kernel runs the pool + FC head as its tail (no cluster-head launch)
    bool self_clean;       // ... and cleans its own workspace (SNB200_GEN_WORKSPACE_PRIMED): no memset in front of it
    int tiles_per_cloud;   // per-cloud pool partials the conv stage leaves for the head
};

static GenPlan plan_generator(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc, int flags, bool act_input)
{
    const bool use_tc = !(flags & SNB200_GEN_EXACT_FP32) && tc_stack_supported(nconv, conv, act_input);
    const bool cs_ok = use_tc && !act_input && conv_stack_supported(b, n, nconv, conv);
    GenPlan P;
    if (flags & SNB200_GEN_PROFILE_SKIP_CONV) P.conv = GenConv::HeadOnly;
    else if (cs_ok && !(flags & SNB200_GEN_PER_LAYER_KERNELS)) P.conv = GenConv::Persistent;
    else P.conv = use_tc ? GenConv::PerLayerTc : GenConv::ExactFp32;
    P.fuse_head = P.conv == GenConv::Persistent && !(flags & (SNB200_GEN_PROFILE_SKIP_HEAD | SNB200_GEN_SEPARATE_HEAD)) && b <= 256;
    for (int l = 0; l < nfc; l++) P.fuse_head = P.fuse_head && fc[l].c_in <= 1024;
    // SNB200_GEN_WORKSPACE_PRIMED: the caller keeps this workspace for this call sequence and its first 256 bytes (moments, barrier
    // and exit words) are zero -- freshly zeroed, or as the previous PRIMED call left them.  The fused persistent kernel then cleans the
    // rest itself; every other path memsets as usual and re-zeroes those 256 bytes at the end.
    P.self_clean = (flags & SNB200_GEN_WORKSPACE_PRIMED) && P.fuse_head;
    // head-only profiling reads the layout the default path (the persistent kernel where it applies) leaves behind
    if (P.conv == GenConv::Persistent || (P.conv == GenConv::HeadOnly && cs_ok)) P.tiles_per_cloud = conv_stack_slots_per_cloud(b, n);
    else if (use_tc) P.tiles_per_cloud = tc_tiles_per_cloud(n);
    else P.tiles_per_cloud = simt_tiles_per_cloud(n, conv[nconv - 1].c_out);
    return P;
}

// snb200_debug_generator_plan: the conv path (0 persistent, 1 per-layer tensor-core, 2 exact fp32, 3 head only) and whether the head is fused
void generator_plan_debug(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc, int flags, int *conv_path, int *fuse_head)
{
    const GenPlan P = plan_generator(b, n, nconv, conv, nfc, fc, flags, false);
    *conv_path = (int)P.conv;
    *fuse_head = P.fuse_head ? 1 : 0;
}

// ---- pool + FC head as its own cluster launch
int launch_fc_head_cluster(const HeadParams &H, cudaStream_t stream)
{
    const int nfc = H.num_fc;
    int cmax = 0, max_out = 0;
    size_t wfloats = 0;
    for (int l = 0; l < nfc; l++) {
        cmax = max(cmax, H.fc[l].c_in); max_out = max(max_out, H.fc[l].c_out);
        wfloats += (size_t)kHeadChPerCta * head_ldw(H.fc[l].c_in);
    }
    // cluster size: enough CTAs that the widest layer is a single 16-channel pass per CTA, or without FC layers that every thread pools
    // one value, capped at 16 (non-portable size)
    int csize = 1;
    if (nfc) while (csize < kHeadMaxCluster && csize * kHeadChPerCta < max_out) csize *= 2;
    else while (csize < kHeadMaxCluster && (long long)csize * kHeadThreads < (long long)H.b * H.c_feat) csize *= 2;
    // the input tile stages every K at once where that fits, else the most K that fits, a multiple of 32; the pool alone uses none
    const size_t fixed = nfc ? wfloats + (size_t)8 * 32 * 17 : 0, cap = kHeadSmemBytes / sizeof(float);
    int kch = cmax;
    if (fixed + (size_t)cmax * 36 > cap) kch = fixed < cap ? (int)(((cap - fixed) / 36) & ~(size_t)31) : 0;
    const size_t smem = (fixed + (size_t)kch * 36) * sizeof(float);
    const int rg = nfc ? (H.b + 31) / 32 : 1;   // the pool has no row groups: any batch
    if (rg > 8) { set_error("FC head: batch %d exceeds the limit of 256 rows", H.b); return SNB200_EUNSUPPORTED; }
    if (kch < cmax && kch < 32) { set_error("FC head: width %d too large for the shared-memory tile", cmax); return SNB200_EUNSUPPORTED; }
    HeadParams Hk = H;
    Hk.k_chunk = kch;
    using HeadKernel = void (*)(HeadParams);
    static const HeadKernel kernels[4] = {fc_head_cluster_kernel<1>, fc_head_cluster_kernel<2>, fc_head_cluster_kernel<4>, fc_head_cluster_kernel<8>};
    static PerDeviceOnce once;
    if (once.first())
        for (HeadKernel k : kernels) {
            cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kHeadSmemBytes);
            cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(csize); cfg.blockDim = dim3(kHeadThreads); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = csize; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    const HeadKernel kernel = kernels[rg == 1 ? 0 : rg == 2 ? 1 : rg <= 4 ? 2 : 3];   // RG = 1, 2, 4, 8 row groups
    cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, Hk);
    if (e != cudaSuccess) { set_error("FC head: launch failed: %s", cudaGetErrorString(e)); cudaGetLastError(); return SNB200_ECUDA; }
    return check_launch("FC head");
}

int launch_generator_forward(int b, int n, int layout, const float *x, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc,
                             int training, float *out, int out_transpose_inner, float *feat_out, int flags, void *workspace, cudaStream_t stream,
                             float *const *zsave, const GenEx *ex)
{
    GenWorkspace W = carve_gen_ws(workspace, b, n, nconv, conv, nfc, fc);
    const bool act_input = ex && ex->act_input;   // x is then the (b*n, c_in) activation
    const GenPlan plan = plan_generator(b, n, nconv, conv, nfc, fc, flags, act_input);
    const bool persistent = plan.conv == GenConv::Persistent;
    if ((training || persistent) && !plan.self_clean) cudaMemsetAsync(W.stats_base, 0, W.stats_bytes, stream);   // statistics, moments, grid-barrier counter
    struct Rezero {   // non-self-cleaning paths leave the head of a PRIMED workspace as they found it
        bool on; char *p; cudaStream_t s;
        ~Rezero() { if (on) cudaMemsetAsync(p, 0, 256, s); }
    } rezero{(flags & SNB200_GEN_WORKSPACE_PRIMED) && !plan.self_clean, W.stats_base, stream};
    HeadParams H;
    fill_head_params(H, b, n, plan.tiles_per_cloud, nconv, conv, nfc, fc, training, out, out_transpose_inner, feat_out, W);
    if (ex)
        for (int l = 0; l + 1 < nfc; l++) H.fc[l].out_mask = ex->fc_dropout[l + 1];
    int rc = SNB200_OK;
    if (persistent)
        rc = launch_conv_stack(b, n, layout, x, nconv, conv, training, W.stats, W.mom, W.counter, W.tile_max, W.tile_min, plan.fuse_head ? &H : nullptr,
                               plan.self_clean ? W.stats_base + 256 : nullptr, W.stats_bytes - 256, stream, zsave, W.act);
    else if (plan.conv == GenConv::PerLayerTc) {
        if (training && conv[0].bn_weight && !act_input)
            rc = launch_x_moments(b, n, layout, x, W.mom, W.counter, conv[0].weight, conv[0].bias, conv[0].c_out, W.stats[0], stream);
        if (!rc) rc = launch_tc_stack(b, n, layout, x, nconv, conv, training, W.stats, zsave, W.act, TcStackTail{W.tile_max, W.tile_min}, stream,
                                      act_input ? x : nullptr, ex ? ex->tap : -1, ex ? ex->tap_out : nullptr);
        H.keep_inputs = zsave != nullptr;
    }
    else if (plan.conv == GenConv::ExactFp32)
        rc = launch_simt_conv_stack(b, n, layout, x, nconv, conv, training, W.act[0], W.act[1], W.stats, W.tile_max, W.tile_min, stream);
    if (rc || plan.fuse_head || (flags & SNB200_GEN_PROFILE_SKIP_HEAD)) return rc;
    return launch_fc_head_cluster(H, stream);
}

}  // namespace snb
