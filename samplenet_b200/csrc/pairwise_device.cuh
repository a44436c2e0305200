// pairwise_device.cuh -- device bodies of the pairwise-distance kernels (fused kNN + soft projection, Chamfer direction
// scan), shared by their stand-alone kernels (softproj.cu, chamfer.cu) and by the fused SampleNet tail kernel (tail.cu).
#pragma once
#include "common.cuh"

namespace snb {


constexpr int kSpWarps = 8;
constexpr int kSpThreads = kSpWarps * 32;
constexpr int kSpTile = 4096;  // points per shared-memory stage (48 KB)

struct SoftProjParams {
    int b, n, m, k, f;
    int queries_per_warp;
    const float *points, *query, *sigma, *feats;
    int sigma_mode; float sigma_floor;
    int hard;
    float *proj, *prop;
    int *knn_idx;
    float *knn_val, *weights, *dist_over_sigma;
    float *nn_dist;   // optional (b, m): distance to the nearest neighbour == nn_distance's dist1 of (query -> points)
    int *nn_idx;      // optional (b, m): its index                         == idx1
};

__device__ __forceinline__ float resolve_sigma(const float *p, int mode, float floor_v)
{
    const float t = __ldg(p);
    if (mode == SNB200_SIGMA_FROM_T_REG) return fmaxf(t * t, floor_v);
    if (mode == SNB200_SIGMA_FROM_T_CLS) return t * t;
    if (mode == SNB200_SIGMA_FROM_T_REC) { const float u = fmaxf(t, floor_v); return u * u; }
    return t;
}

template <int kLayout>
__device__ __forceinline__ float ld_coord(const float *base, int npts, int p, int c)
{
    return kLayout == SNB200_BNC ? base[(size_t)p * 3 + c] : base[(size_t)c * npts + p];
}

// Body of the fused kNN + soft projection for CTA (bx, bi); s_pts: dynamic shared memory (BNC: [tile*3] AoS; BCN: 3 rows of
// `tile_cap`), bar: an mbarrier in shared memory (initialised here).
template <int kLayout, bool kFma>
__device__ __forceinline__ void knn_softproj_body(const SoftProjParams &P, int bx, int bi, float *s_pts, uint64_t *barp,
                                                  float *acc_sum = nullptr, float *acc_max = nullptr, bool pdl = false)
{
    uint64_t &bar = *barp;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = P.n, m = P.m, k = P.k;
    const int tile_cap = min(n, kSpTile);

    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    __syncthreads();

    const float *pts = P.points + (size_t)bi * n * 3;
    const float *qry = P.query + (size_t)bi * m * 3;
    const int qpw = P.queries_per_warp;
    const int q_first = (bx * kSpWarps + warp) * qpw;

    uint32_t phase = 0;
    const int ntiles = (n + kSpTile - 1) / kSpTile;
    // Programmatic dependent launch (fused tail): the cloud does not depend on the producer of the queries, so its tile is requested
    // BEFORE this grid synchronises on the previous one; the queries are only read after griddepcontrol.wait.
    bool preissued = false;
    if (pdl) {
        const bool tma_ok = kLayout == SNB200_BNC && ntiles == 1 && ((reinterpret_cast<uintptr_t>(pts) & 15) == 0) && (((n * 3) & 3) == 0) && n > 0;
        if (tma_ok) {
            if (threadIdx.x == 0) {
                mbar_expect_tx(&bar, (uint32_t)n * 12u);
                tma_load_1d(s_pts, pts, (uint32_t)n * 12u, &bar);
            }
            preissued = true;
        }
        asm volatile("griddepcontrol.wait;" ::: "memory");
    }

    // With a single tile (the common case: n <= 4096) the cloud is staged once and reused for all queries of the CTA.
    // With several tiles each query walks the tiles in order; the CTA restages per (query round, tile).
    for (int qr = 0; qr < qpw; qr++) {
        const int qi = q_first + qr;
        const bool live = qi < m;  // warp-uniform
        float qx = 0, qy = 0, qz = 0;
        if (live) {
            qx = ld_coord<kLayout>(qry, m, qi, 0);
            qy = ld_coord<kLayout>(qry, m, qi, 1);
            qz = ld_coord<kLayout>(qry, m, qi, 2);
        }
        float lv = INFINITY;      // lane i: i-th smallest distance so far
        int li = 0x7fffffff;      //         and its index
        float thr = INFINITY;     // current k-th best (warp-uniform)

        for (int t = 0; t < ntiles; t++) {
            const int p0 = t * kSpTile;
            const int pn = min(kSpTile, n - p0);
            if (ntiles > 1 || qr == 0) {
                if (!(t == 0 && qr == 0)) __syncthreads();
                if (preissued && t == 0 && qr == 0) {
                    mbar_wait(&bar, phase);   // the tile requested before griddepcontrol.wait
                    phase ^= 1;
                } else if (kLayout == SNB200_BNC) {
                    stage_floats(s_pts, pts + (size_t)p0 * 3, pn * 3, &bar, phase);
                } else {
                    // three rows; issue them back to back on the same barrier when TMA-eligible
                    stage_floats(s_pts + 0 * tile_cap, pts + 0 * (size_t)n + p0, pn, &bar, phase);
                    stage_floats(s_pts + 1 * tile_cap, pts + 1 * (size_t)n + p0, pn, &bar, phase);
                    stage_floats(s_pts + 2 * tile_cap, pts + 2 * (size_t)n + p0, pn, &bar, phase);
                }
            }
            // One insertion into the warp-resident sorted list (lane i = i-th smallest so far, ascending by (distance, index)):
            // candidates arrive in ascending index order, so strict '<' keeps the lower index first among equal distances.
#define SNB_KNN_INSERT(V, VI)                                                   \
            do {                                                                \
                const float up_v = __shfl_up_sync(kFullMask, lv, 1);            \
                const int up_i = __shfl_up_sync(kFullMask, li, 1);              \
                if (lane > 0 && (V) < up_v) { lv = up_v; li = up_i; }           \
                else if ((V) < lv) { lv = (V); li = (VI); }                     \
            } while (0)
            // Bound from the lane minima `mn` of a tile: the k-th smallest of the 32 lane minima is an upper bound of the k-th
            // neighbour distance (k distinct candidates lie at or below it), so only the handful of candidates at or below it
            // have to go through the list instead of every running improvement (~k(1+ln(n/k)) for a cold list).
#define SNB_KNN_BOUND(MN)                                                                                       \
            do {                                                                                                \
                int rank = 0;                                                                                   \
                _Pragma("unroll") for (int jj = 0; jj < 32; jj++) {                                             \
                    const float o = __shfl_sync(kFullMask, (MN), jj);                                           \
                    rank += (o < (MN) || (o == (MN) && jj < lane)) ? 1 : 0;                                     \
                }                                                                                               \
                const unsigned kth = __ballot_sync(kFullMask, rank == k - 1);                                   \
                if (kth) { /* (no lane has that rank only when NaNs break the ordering: keep the running bound) */ \
                    const float tau = __shfl_sync(kFullMask, (MN), __ffs(kth) - 1);                             \
                    if (tau < INFINITY) thr = fminf(thr, __uint_as_float(__float_as_uint(tau) + 1u)); /* admit d <= tau */ \
                }                                                                                               \
            } while (0)
            if (live && pn <= 1024) {
                // Register path (the SampleNet sizes): the 32 distances of a lane stay in registers between the bound pass and the
                // insertion pass, so every pair is evaluated once.
                float d[32];
                float mn = INFINITY;
#pragma unroll
                for (int u = 0; u < 32; u++) {
                    const int j = u * 32 + lane;
                    float dd = INFINITY;
                    if (j < pn) {
                        float cx, cy, cz;
                        if (kLayout == SNB200_BNC) {
                            cx = s_pts[j * 3 + 0]; cy = s_pts[j * 3 + 1]; cz = s_pts[j * 3 + 2];
                        } else {
                            cx = s_pts[j]; cy = s_pts[tile_cap + j]; cz = s_pts[2 * tile_cap + j];
                        }
                        dd = sqdist<kFma>(cx - qx, cy - qy, cz - qz);  // (dataset - query), tf_grouping.py:84
                    }
                    d[u] = dd;
                    mn = (dd < mn) ? dd : mn;
                }
                SNB_KNN_BOUND(mn);
#pragma unroll
                for (int u = 0; u < 32; u++) {
                    unsigned mask = __ballot_sync(kFullMask, d[u] < thr);
                    if (mask) {
                        while (mask) {
                            const int src = __ffs(mask) - 1;
                            mask &= mask - 1;
                            const float v = __shfl_sync(kFullMask, d[u], src);
                            const int vi = p0 + u * 32 + src;
                            SNB_KNN_INSERT(v, vi);
                        }
                        thr = fminf(thr, __shfl_sync(kFullMask, lv, k - 1));
                    }
                }
            } else if (live) {
                // Generic path (tiles of up to kSpTile points): bound pass, then the distances are recomputed (bit-identical).
                float mn = INFINITY;
#pragma unroll 4
                for (int j = lane; j < pn; j += 32) {
                    float cx, cy, cz;
                    if (kLayout == SNB200_BNC) {
                        cx = s_pts[j * 3 + 0]; cy = s_pts[j * 3 + 1]; cz = s_pts[j * 3 + 2];
                    } else {
                        cx = s_pts[j]; cy = s_pts[tile_cap + j]; cz = s_pts[2 * tile_cap + j];
                    }
                    const float dd = sqdist<kFma>(cx - qx, cy - qy, cz - qz);
                    mn = (dd < mn) ? dd : mn;
                }
                SNB_KNN_BOUND(mn);
                for (int base = 0; base < pn; base += 128) {
                    float d[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        const int j = base + u * 32 + lane;
                        float dd = INFINITY;
                        if (j < pn) {
                            float cx, cy, cz;
                            if (kLayout == SNB200_BNC) {
                                cx = s_pts[j * 3 + 0]; cy = s_pts[j * 3 + 1]; cz = s_pts[j * 3 + 2];
                            } else {
                                cx = s_pts[j]; cy = s_pts[tile_cap + j]; cz = s_pts[2 * tile_cap + j];
                            }
                            dd = sqdist<kFma>(cx - qx, cy - qy, cz - qz);
                        }
                        d[u] = dd;
                    }
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        unsigned mask = __ballot_sync(kFullMask, d[u] < thr);
                        if (mask) {
                            while (mask) {
                                const int src = __ffs(mask) - 1;
                                mask &= mask - 1;
                                const float v = __shfl_sync(kFullMask, d[u], src);
                                const int vi = p0 + base + u * 32 + src;
                                SNB_KNN_INSERT(v, vi);
                            }
                            thr = fminf(thr, __shfl_sync(kFullMask, lv, k - 1));
                        }
                    }
                }
            }
#undef SNB_KNN_INSERT
#undef SNB_KNN_BOUND
        }
        if (!live) continue;

        // ---- lanes 0..k-1 now hold the k nearest neighbours, ascending by (distance, index)
        const bool has = lane < k;
        const size_t o = ((size_t)bi * m + qi) * k + lane;
        li = min(li, n - 1);  // only reachable with NaN/Inf coordinates (nothing ever beat +inf): stay in bounds
        if (P.knn_idx && has) P.knn_idx[o] = li;
        if (P.knn_val && has) P.knn_val[o] = lv;
        if (lane == 0) {   // the first neighbour is the nn_distance result of this query (same arithmetic, same tie rule)
            if (P.nn_dist) P.nn_dist[(size_t)bi * m + qi] = lv;
            if (P.nn_idx) P.nn_idx[(size_t)bi * m + qi] = li;
            if (acc_sum) { *acc_sum += lv; *acc_max = fmaxf(*acc_max, lv); }
        }
        if (!P.proj && !P.prop && !P.weights && !P.dist_over_sigma) continue;

        // neighbour coordinates: from global (L2-resident; the tile in shared memory may be a later one)
        float gx = 0, gy = 0, gz = 0;
        if (has && ntiles == 1) {          // the whole cloud is still staged
            if (kLayout == SNB200_BNC) { gx = s_pts[li * 3 + 0]; gy = s_pts[li * 3 + 1]; gz = s_pts[li * 3 + 2]; }
            else { gx = s_pts[li]; gy = s_pts[tile_cap + li]; gz = s_pts[2 * tile_cap + li]; }
        } else if (has) {
            gx = ld_coord<kLayout>(pts, n, li, 0);
            gy = ld_coord<kLayout>(pts, n, li, 1);
            gz = ld_coord<kLayout>(pts, n, li, 2);
        }
        // soft_projection.py:92-95: sum((grouped - query)^2) / sigma, evaluated like torch does (separate
        // subtract, square, sum over xyz in order, true division)
        const float sigma = resolve_sigma(P.sigma, P.sigma_mode, P.sigma_floor);
        const float dx = gx - qx, dy = gy - qy, dz = gz - qz;
        const float dist = __fdiv_rn(sqdist<false>(dx, dy, dz), sigma);
        // soft_projection.py:143: softmax(-dist) over the k neighbours
        const float neg = has ? -dist : -INFINITY;
        const float mx = warp_max(neg);
        float e = has ? expf(neg - mx) : 0.0f;
        const float sum = warp_sum(e);
        float w = __fdiv_rn(e, sum);
        if (P.hard) w = (lane == 0) ? 1.0f : 0.0f;  // tf.one_hot(tf.argmax(weights)): the nearest neighbour
        if (P.weights && has) P.weights[o] = w;
        if (P.dist_over_sigma && has) P.dist_over_sigma[o] = dist;
        if (P.proj) {
            const float px = warp_sum(w * gx), py = warp_sum(w * gy), pz = warp_sum(w * gz);
            if (lane == 0) {
                float *pr = P.proj + (size_t)bi * m * 3;
                if (kLayout == SNB200_BNC) {
                    pr[(size_t)qi * 3 + 0] = px; pr[(size_t)qi * 3 + 1] = py; pr[(size_t)qi * 3 + 2] = pz;
                } else {
                    pr[0 * (size_t)m + qi] = px; pr[1 * (size_t)m + qi] = py; pr[2 * (size_t)m + qi] = pz;
                }
            }
        }
        if (P.prop) {  // soft_projection.py:120-136: propagate features with the same weights; lanes over channels
            const int f = P.f;
            const float *ft = P.feats + (size_t)bi * n * f;
            float *po = P.prop + (size_t)bi * m * f;
            for (int c0 = 0; c0 < f; c0 += 32) {
                const int c = c0 + lane;
                float acc = 0;
                for (int s = 0; s < k; s++) {
                    const float ws = __shfl_sync(kFullMask, w, s);
                    const int is = __shfl_sync(kFullMask, li, s);
                    if (c < f) acc += ws * (kLayout == SNB200_BNC ? ft[(size_t)is * f + c] : ft[(size_t)c * n + is]);
                }
                if (c < f) {
                    if (kLayout == SNB200_BNC) po[(size_t)qi * f + c] = acc; else po[(size_t)c * m + qi] = acc;
                }
            }
        }
    }
}


constexpr int kChamferThreads = 256;
constexpr int kChamferTile = 4096;  // candidates per shared-memory stage (48 KB)

struct ChamferDir {
    const float *q;   // queries   (b, nq, 3)
    const float *c;   // candidates (b, nc, 3)
    float *dist;      // (b, nq), or null: nothing is stored
    int *idx;         // (b, nq), with dist
    int nq, nc;
    int S;            // lanes per query (power of two <= 32)
    int tiles;        // CTAs along x for this direction
};

struct ChamferParams {
    ChamferDir d[2];
};

// Choose the lanes-per-query S of one direction (Q = queries register-blocked per thread): no more thread slots per CTA than
// there are queries (a 64-query direction must not leave 3/4 of a 256-thread CTA idle), then enough CTAs to reach `target_ctas`,
// but never fewer than 16 candidates per lane (the log2(S) merge would dominate).
inline void plan_chamfer_dir(ChamferDir &D, int b, int Q, int target_ctas)
{
    int S = 1;
    while (S < 32) {
        if (D.nc / (S * 2) < 16) break;
        const int per_cta = (kChamferThreads / S) * Q;
        const long long ctas = (long long)b * ((D.nq + per_cta - 1) / per_cta);
        if (per_cta <= D.nq && ctas >= target_ctas) break;
        S *= 2;
    }
    D.S = S;
    const int per_cta = (kChamferThreads / S) * Q;
    D.tiles = (D.nq + per_cta - 1) / per_cta;
}

template <int Q, bool kFma>
__device__ __forceinline__ void chamfer_dir(const ChamferDir &D, int tile, int bi, float *s_c, uint64_t *bar, float *acc_sum = nullptr,
                                            float *acc_max = nullptr)
{
    const int S = D.S;
    const int groups = kChamferThreads / S;  // query groups per CTA
    const int g = threadIdx.x / S;           // my group
    const int l = threadIdx.x % S;           // my lane inside the group
    const int q0 = (tile * groups + g) * Q;  // first of my Q queries

    const float *qp = D.q + (size_t)bi * D.nq * 3;
    const float *cp = D.c + (size_t)bi * D.nc * 3;

    float qx[Q], qy[Q], qz[Q], best[Q];
    int besti[Q];
#pragma unroll
    for (int t = 0; t < Q; t++) {
        const int qi = min(q0 + t, D.nq - 1);  // clamp: out-of-range slots compute a duplicate and are not stored
        qx[t] = __ldg(qp + qi * 3 + 0);
        qy[t] = __ldg(qp + qi * 3 + 1);
        qz[t] = __ldg(qp + qi * 3 + 2);
        best[t] = INFINITY;
        besti[t] = 0x7fffffff;
    }

    uint32_t phase = 0;
    for (int c0 = 0; c0 < D.nc; c0 += kChamferTile) {
        const int cn = min(kChamferTile, D.nc - c0);
        if (c0 > 0) __syncthreads();  // everyone finished with the previous tile
        stage_floats(s_c, cp + (size_t)c0 * 3, cn * 3, bar, phase);
#pragma unroll 4
        for (int j = l; j < cn; j += S) {
            const float cx = s_c[j * 3 + 0], cy = s_c[j * 3 + 1], cz = s_c[j * 3 + 2];
#pragma unroll
            for (int t = 0; t < Q; t++) {
                // (candidate - query), as chamfer_distance.cu:30-33
                const float d = sqdist<kFma>(cx - qx[t], cy - qy[t], cz - qz[t]);
                if (d < best[t]) {  // strict '<' and ascending j per lane: lowest index among equal distances
                    best[t] = d;
                    besti[t] = c0 + j;
                }
            }
        }
    }
    // merge the S partial results of the group: lexicographic min on (distance, index)
#pragma unroll
    for (int t = 0; t < Q; t++) {
        for (int o = S >> 1; o > 0; o >>= 1) {
            const float od = __shfl_xor_sync(kFullMask, best[t], o);
            const int oi = __shfl_xor_sync(kFullMask, besti[t], o);
            if (od < best[t] || (od == best[t] && oi < besti[t])) {
                best[t] = od;
                besti[t] = oi;
            }
        }
        if (l == 0 && q0 + t < D.nq) {
            if (D.dist) {   // null when only the reductions are wanted (chamfer_per_cloud)
                D.dist[(size_t)bi * D.nq + q0 + t] = best[t];
                D.idx[(size_t)bi * D.nq + q0 + t] = besti[t];
            }
            if (acc_sum) { *acc_sum += best[t]; *acc_max = fmaxf(*acc_max, best[t]); }   // this thread's share of the loss reductions
        }
    }
}


}  // namespace snb
