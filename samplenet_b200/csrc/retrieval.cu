// retrieval.cu -- shape-retrieval metrics of descriptor sets: for every query, the whole database ranked by squared L2 distance, then
// average precision and the interpolated precision-recall curve of that ranking, without a (Q, M) matrix in global memory.
//
// Contract (include/samplenet_b200.h, snb200_retrieval_metrics): d(q, x) = sum_k fl(fl(q_k - x_k)^2) accumulated left to right in float32
// with every product and sum rounded (no contraction, as matching.cu rounds for numpy); results ordered by (d, index); AP summed in float64
// in rank order; interpolated precision compared in integers.
//
// Design (DESIGN.md 4.14): one CTA takes kQ queries.  Pass 1 streams the database through shared memory in tiles of kThreads rows x kKC
// columns: thread t owns row j * kThreads + t of every tile and accumulates its kQ distances in registers, column by column, so the order of
// the sum is the contract's whatever the tile shape.  Pass 2, per query: each distance becomes a unique 46-bit key (float bits << 14 |
// index; non-negative floats order like their bits, and the index breaks ties), one cub::BlockRadixSort ranks them, a block scan of the
// relevance flags gives hits(k), every relevant rank writes hits/k to shared memory at position hits - 1, and one thread sums those terms in
// order while the other warps take the suffix maxima the interpolated curve needs.  The excluded item and the padding rows get the all-ones
// key and sort last.
#include "common.cuh"

#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>

namespace snb {

constexpr int kKC = 32;                         // database columns per staged tile
constexpr int kTileStride = kKC + 4;            // padded row stride: float4 reads of 8 consecutive rows hit distinct bank groups
constexpr int kIndexBits = 14;                  // M <= 16384
constexpr int kKeyBits = 31 + kIndexBits + 1;   // distance bits, index, and the bit that puts the pad key above every real key
constexpr unsigned long long kPadKey = ~0ull;
constexpr unsigned kCanonicalNan = 0x7FC00000u; // every NaN distance ranks as one value, after +inf, by index (numpy's argsort)

template <int kThreads, int kItems>
constexpr size_t retrieval_union_bytes()
{
    using Sort = cub::BlockRadixSort<unsigned long long, kThreads, kItems>;
    size_t a = sizeof(typename Sort::TempStorage), b = (size_t)kThreads * kTileStride * sizeof(float), c = (size_t)kThreads * kItems * sizeof(double);
    size_t m = a > b ? a : b;
    m = m > c ? m : c;
    return (m + 15) / 16 * 16;
}

__device__ __forceinline__ float sq_diff_rn(float q, float x)
{
    const float d = __fsub_rn(q, x);
    return __fmul_rn(d, d);
}

template <int kThreads, int kItems, int kQ>
__global__ void __launch_bounds__(kThreads) retrieval_kernel(int Q, int M, int D, int dpad, int vec4, const float *__restrict__ queries,
                                                             const int *__restrict__ qlab, const float *__restrict__ db, const int *__restrict__ dblab,
                                                             int exclude, int L, double *__restrict__ ap, double *__restrict__ prec,
                                                             int *__restrict__ num_relevant)
{
    using Sort = cub::BlockRadixSort<unsigned long long, kThreads, kItems>;
    using Scan = cub::BlockScan<int, kThreads>;
    constexpr size_t kUnion = retrieval_union_bytes<kThreads, kItems>();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ typename Scan::TempStorage scan_tmp;
    // layout: one region used in turn as the database tile (pass 1), the sort's storage and the AP terms (pass 2); then the kQ queries
    float *tile = reinterpret_cast<float *>(smem_raw);
    typename Sort::TempStorage &sort_tmp = *reinterpret_cast<typename Sort::TempStorage *>(smem_raw);
    double *terms = reinterpret_cast<double *>(smem_raw);
    float *qs = reinterpret_cast<float *>(smem_raw + kUnion);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int q0 = blockIdx.x * kQ;
    for (int e = tid; e < kQ * dpad; e += kThreads) {   // zero columns beyond D add +0 to a non-negative sum: no change
        const int t = e / dpad, k = e - t * dpad;
        qs[e] = (q0 + t < Q && k < D) ? queries[(size_t)(q0 + t) * D + k] : 0.f;
    }

    // ---- pass 1: distances, kQ x kItems per thread
    float acc[kQ][kItems];
#pragma unroll
    for (int t = 0; t < kQ; ++t)
#pragma unroll
        for (int j = 0; j < kItems; ++j) acc[t][j] = 0.f;
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
        const int r0 = j * kThreads;
        if (r0 >= M) break;
        for (int k0 = 0; k0 < dpad; k0 += kKC) {
            __syncthreads();   // the previous tile is consumed (and, the first time, the queries are staged)
            if (vec4) {
                for (int e = tid; e < kThreads * (kKC / 4); e += kThreads) {
                    const int r = e / (kKC / 4), c = (e % (kKC / 4)) * 4, row = r0 + r, col = k0 + c;
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (row < M && col < D) v = __ldg(reinterpret_cast<const float4 *>(db + (size_t)row * D + col));
                    *reinterpret_cast<float4 *>(tile + r * kTileStride + c) = v;
                }
            } else {
                for (int e = tid; e < kThreads * kKC; e += kThreads) {
                    const int r = e / kKC, c = e % kKC, row = r0 + r, col = k0 + c;
                    tile[r * kTileStride + c] = (row < M && col < D) ? __ldg(db + (size_t)row * D + col) : 0.f;
                }
            }
            __syncthreads();
            const float *xr = tile + tid * kTileStride;
#pragma unroll
            for (int c = 0; c < kKC; c += 4) {
                const float4 xv = *reinterpret_cast<const float4 *>(xr + c);
#pragma unroll
                for (int t = 0; t < kQ; ++t) {
                    const float4 qv = *reinterpret_cast<const float4 *>(qs + t * dpad + k0 + c);
                    float a = acc[t][j];
                    a = __fadd_rn(a, sq_diff_rn(qv.x, xv.x));
                    a = __fadd_rn(a, sq_diff_rn(qv.y, xv.y));
                    a = __fadd_rn(a, sq_diff_rn(qv.z, xv.z));
                    a = __fadd_rn(a, sq_diff_rn(qv.w, xv.w));
                    acc[t][j] = a;
                }
            }
        }
    }

    // ---- pass 2: rank, then AP and the interpolated curve, one query at a time
    const double nan = __longlong_as_double(0x7FF8000000000000LL);
    const int nwarps = kThreads / 32;
#pragma unroll
    for (int t = 0; t < kQ; ++t) {
        const int qi = q0 + t;
        if (qi >= Q) break;
        __syncthreads();   // the shared region is free: the last tile, or the previous query's terms, have been read
        unsigned long long keys[kItems];
#pragma unroll
        for (int j = 0; j < kItems; ++j) {
            const int m = j * kThreads + tid;
            const float d = acc[t][j];
            const unsigned bits = isnan(d) ? kCanonicalNan : __float_as_uint(d);
            keys[j] = (m < M && !(exclude && m == qi)) ? ((unsigned long long)bits << kIndexBits | (unsigned)m) : kPadKey;
        }
        Sort(sort_tmp).Sort(keys, 0, kKeyBits);   // blocked: thread tid holds ranks tid * kItems + i (0-based)
        const int ql = qlab[qi];
        unsigned relmask = 0;
        int count = 0;
#pragma unroll
        for (int i = 0; i < kItems; ++i) {
            const bool rel = keys[i] != kPadKey && dblab[keys[i] & ((1u << kIndexBits) - 1)] == ql;
            relmask |= (unsigned)rel << i;
            count += rel;
        }
        int before, R;
        Scan(scan_tmp).ExclusiveSum(count, before, R);
        __syncthreads();   // every thread is done with the sort's storage before the terms overwrite it
        int h = before;
#pragma unroll
        for (int i = 0; i < kItems; ++i)
            if (relmask >> i & 1u) {
                ++h;
                terms[h - 1] = (double)h / (double)(tid * kItems + i + 1);
            }
        __syncthreads();
        if (tid == 0) {
            num_relevant[qi] = R;
            double s = 0.0;
            for (int j = 0; j < R; ++j) s = __dadd_rn(s, terms[j]);
            ap[qi] = R > 0 ? s / (double)R : nan;
        }
        // prec_l = max over relevant ranks with hits * (L - 1) >= l * R of hits / k: the maximum of terms[j0 - 1 ..], j0 the first such hits
        for (int l = warp - 1; warp > 0 && l < L; l += nwarps - 1) {
            double v = nan;
            if (R > 0) {
                const int j0 = max(1, (l * R + L - 2) / (L - 1));
                v = 0.0;
                for (int j = j0 - 1 + lane; j < R; j += 32) v = fmax(v, terms[j]);
                for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(kFullMask, v, o));
            }
            if (lane == 0) prec[(size_t)qi * L + l] = v;
        }
    }
}

template <int kThreads, int kItems, int kQ>
static int launch_tier(int Q, int M, int D, const float *queries, const int *qlab, const float *db, const int *dblab, int exclude, int L, double *ap,
                       double *prec, int *num_relevant, cudaStream_t stream)
{
    constexpr size_t kUnion = retrieval_union_bytes<kThreads, kItems>();
    const int dpad = (D + kKC - 1) / kKC * kKC;
    const size_t smem = kUnion + (size_t)kQ * dpad * sizeof(float);
    auto kernel = retrieval_kernel<kThreads, kItems, kQ>;
    static PerDeviceOnce once;
    if (once.first()) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kUnion + (size_t)kQ * 1024 * sizeof(float)));
    const int vec4 = D % 4 == 0 && ((uintptr_t)db & 15) == 0;
    kernel<<<(Q + kQ - 1) / kQ, kThreads, smem, stream>>>(Q, M, D, dpad, vec4, queries, qlab, db, dblab, exclude, L, ap, prec, num_relevant);
    return check_launch("retrieval_metrics");
}

bool retrieval_metrics_supported(int Q, int M, int D, int L, int exclude)
{
    return Q >= 1 && Q <= (1 << 20) && M >= 1 && M <= (1 << kIndexBits) && D >= 1 && D <= 1024 && L >= 2 && L <= 101 && (!exclude || Q == M);
}

// The tier is the smallest sort that holds M keys; small databases take several queries per CTA, so each database row staged in shared
// memory serves them all.
int launch_retrieval_metrics(int Q, int M, int D, const float *queries, const int *qlab, const float *db, const int *dblab, int exclude, int L,
                             double *ap, double *prec, int *num_relevant, cudaStream_t stream)
{
    if (M <= 2048) return launch_tier<256, 8, 4>(Q, M, D, queries, qlab, db, dblab, exclude, L, ap, prec, num_relevant, stream);
    if (M <= 4096) return launch_tier<256, 16, 2>(Q, M, D, queries, qlab, db, dblab, exclude, L, ap, prec, num_relevant, stream);
    if (M <= 8192) return launch_tier<512, 16, 1>(Q, M, D, queries, qlab, db, dblab, exclude, L, ap, prec, num_relevant, stream);
    return launch_tier<512, 32, 1>(Q, M, D, queries, qlab, db, dblab, exclude, L, ap, prec, num_relevant, stream);
}

}  // namespace snb
