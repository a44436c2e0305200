// emd.cu -- approx_match / match_cost / match_cost_grad (EMD).
//
// Reference behaviour restated (not ported): classification/structural_losses/tf_approxmatch_g.cu:1-295.  The reference
// runs ONE CTA of 512 threads per cloud on a fixed grid of 32 CTAs (so at most 32 of the 132 SMs of an H100 ever work), keeps the
// remain/ratio vectors in global scratch, zeroes `match` and then read-modify-writes it once per level (10 sweeps).
//
// Design (approx_match): a persistent cooperative grid (two 512-thread CTAs per SM) walks the flat (cloud, row) index space
// in equal chunks, so every SM works whatever the batch size is; inside a CTA a row is shared by S lanes that each take the
// columns j == lane (mod S) and merge by shuffles; the opposite side (xyz + its per-point weight, as float4) is staged through
// shared memory in tiles, for up to two consecutive clouds at once (a chunk that straddles a cloud boundary still costs one sweep).
// The per-point vectors live in a small global scratch that stays in L2; the 30 phases are separated by a hand-written grid
// barrier.  The ten levels only update those vectors (the per-level ratios are kept), and `match` is written ONCE by a final pass
// that re-evaluates the ten weights of a pair in registers in level order -- no zero-fill, no read-modify-write sweeps.
// exp(level*d) is evaluated as ex2(level*log2e * d) with one MUFU.EX2 (ex2.approx.ftz; the argument is <= 0, results below the
// normal range flush to zero), so values agree with the CPU oracle to fp32 rounding (not the reference's __expf).
// match_cost / match_cost_grad are streaming kernels that read `match` exactly once with 16-byte loads, eight in flight per thread.
#include "common.cuh"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace snb {

constexpr int kEmdThreads = 512;
constexpr int kEmdTile = 1024;  // opposite-side points per shared-memory tile (float4 each: 16 KB)
constexpr int kEmdLevels = 10;  // tf_approxmatch_g.cu:13: j = 7 ... -2

struct EmdParams {
    int b, n, m;
    int b2;          // xyz2 holds b2 clouds (b2 divides b); pair bi matches xyz1[bi] with xyz2[bi % b2]
    int S;           // lanes per row
    const float *xyz1, *xyz2;
    float *match;    // (b, m, n)
    float *temp;     // per cloud: remainL[n], remainR[m], then per level ratioL[n], ratioR[m]
    unsigned *counter;   // grid-barrier word, zero at launch
};

__device__ __forceinline__ float emd_sq(float ax, float ay, float az, float bx, float by, float bz)
{
    const float dx = bx - ax, dy = by - ay, dz = bz - az;
    return dx * dx + dy * dy + dz * dz;
}
// 2^x for x <= 0: one MUFU.EX2; results below the normal range flush to zero (they are below 1e-38 of a weight that is <= 1)
__device__ __forceinline__ float emd_ex2(float x)
{
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float emd_level2(int lev)   // level = -4^lev (0 at the last level); exp(level*d) == exp2(level*log2(e)*d)
{
    const float level = (lev == -2) ? 0.f : -powf(4.0f, (float)lev);
    return level * 1.44269504088896340736f;
}
// One match value rebuilt from the kept per-level ratios:  match[l][k] = sum_lev exp(level_lev * d(k,l)) * ratioL_lev[k] * ratioR_lev[l],
// summed in level order.  The final pass of approxmatch_kernel and the kernels that rebuild match values instead of reading them share
// this expression; the roundings are spelled out (squared distance dy*dy, then + dx*dx and + dz*dz as FMAs, the contraction the
// compiler chose for the final pass's plain expression; (ex2 * rl) * rr + acc as one FMA)
// so every caller obtains the same bits whatever the compiler would contract around it.
__device__ __forceinline__ float emd_sq_rn(float ax, float ay, float az, float bx, float by, float bz)
{
    const float dx = bx - ax, dy = by - ay, dz = bz - az;
    return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}
__device__ __forceinline__ float emd_match_value(float d2, const float *lv2, const float *rl, const float *rr)
{
    float acc = 0.f;
#pragma unroll
    for (int li = 0; li < kEmdLevels; li++) acc = __fmaf_rn(__fmul_rn(emd_ex2(__fmul_rn(lv2[li], d2)), rl[li]), rr[li], acc);
    return acc;
}
__device__ __forceinline__ void emd_level2_all(float *lv2)
{
#pragma unroll
    for (int li = 0; li < kEmdLevels; li++) lv2[li] = emd_level2(7 - li);
}

__device__ __forceinline__ void emd_grid_barrier(unsigned *counter, unsigned target)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1u);
        unsigned v, spin = 0;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
            if (++spin > (1u << 28)) __trap();
        } while (v < target);
    }
    __syncthreads();
}

// Row sums over ALL clouds of the batch:  acc[bi][row] = sum_col exp2(level2 * |row - col|^2) * w[bi][col].
// The b * nrows rows are one flat index space cut into equal contiguous chunks, one per CTA (a chunk may straddle clouds), so the
// whole grid is busy whatever b is (the reference -- and a cluster-per-cloud split -- leave SMs idle unless b divides the chip).
// Inside a CTA a row is shared by S lanes that take the columns j == lane (mod S); the column side (xyz + w as float4) is staged
// through shared memory in tiles; two rows are register-blocked per thread slot when the chunk is long enough.
// ROW / COL strides: rows are points of `prow` (nrows per cloud), columns points of `pcol` (ncols per cloud); `wcol` and the
// vectors `finish` touches are per-cloud vectors addressed through `vec_stride`.  `prow` holds brow clouds and `pcol` bcol (each divides b):
// pair bi reads the points of cloud bi % brow and bi % bcol.
template <typename F>
__device__ __forceinline__ void emd_row_pass(int b, int nrows, int ncols, const float *prow, int brow, const float *pcol, int bcol, const float *wcol,
                                             size_t vec_stride, float level2, int S, float4 (*s_o)[kEmdTile], F &&finish)
{
    const long long total = (long long)b * nrows;
    const long long per = (total + gridDim.x - 1) / gridDim.x;
    const long long lo = min(total, per * blockIdx.x), hi = min(total, lo + per);
    const int slots = kEmdThreads / S;              // row slots per pass
    const int slot = threadIdx.x / S, l_in = threadIdx.x % S;
    // A pass covers up to `slots` (or 2 x slots) consecutive flat rows taken from at most TWO consecutive clouds: the column tiles of
    // both clouds are staged side by side and every thread reads the tile of its own row's cloud, so a chunk that straddles a cloud
    // boundary still costs one sweep over the columns (a per-cloud loop would cost two and stall the whole grid at the next barrier).
    for (long long f0 = lo; f0 < hi;) {
        const int bi0 = (int)(f0 / nrows);
        const long long cap = min(hi, (long long)(bi0 + 2) * nrows);             // rows of clouds bi0 and bi0 + 1 only
        const long long split = (long long)(bi0 + 1) * nrows;                    // first flat row of cloud bi0 + 1
        const bool two = (cap - f0) > slots && cap <= split;                     // second row per slot only inside one cloud (shares the LDS)
        const long long fend = min(cap, f0 + (two ? 2 : 1) * (long long)slots);
        const bool second_cloud = fend > split;                                  // CTA-uniform
        const long long fa = f0 + slot, fb = f0 + slots + slot;
        const bool la = fa < fend, lb = two && fb < fend;
        const int sel = (la && fa >= split) ? 1 : 0;
        const int bia = bi0 + sel;
        const int ra = (int)(fa - (long long)bia * nrows), rb = (int)(fb - (long long)bi0 * nrows);
        float xa = 0, ya = 0, za = 0, xb = 0, yb = 0, zb = 0;
        if (la) { const float *pr = prow + ((size_t)(bia % brow) * nrows + ra) * 3; xa = pr[0]; ya = pr[1]; za = pr[2]; }
        if (lb) { const float *pr = prow + ((size_t)(bi0 % brow) * nrows + rb) * 3; xb = pr[0]; yb = pr[1]; zb = pr[2]; }
        // the per-pair chain LDS -> 6 FMA-pipe ops -> MUFU -> FMA is ~70 cycles long: four independent accumulators (times the
        // unroll) keep enough pairs in flight per thread for the issue slots to be the limit, not that latency
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (int c0 = 0; c0 < ncols; c0 += kEmdTile) {
            const int cn = min(kEmdTile, ncols - c0);
            __syncthreads();
            for (int q = 0; q < (second_cloud ? 2 : 1); q++) {
                const float *pc = pcol + (size_t)((bi0 + q) % bcol) * ncols * 3;
                const float *wc = wcol + (size_t)(bi0 + q) * vec_stride;
                for (int c = threadIdx.x; c < cn; c += kEmdThreads)
                    s_o[q][c] = make_float4(pc[(c0 + c) * 3 + 0], pc[(c0 + c) * 3 + 1], pc[(c0 + c) * 3 + 2], wc[c0 + c]);
            }
            __syncthreads();
            const float4 *so = s_o[sel];
            if (la && two) {   // one shared-memory read feeds two rows: a0/a2 row a, a1/a3 row b
                int c = l_in;
#pragma unroll 2
                for (; c + S < cn; c += 2 * S) {
                    const float4 o0 = so[c], o1 = so[c + S];
                    a0 = fmaf(emd_ex2(level2 * emd_sq(xa, ya, za, o0.x, o0.y, o0.z)), o0.w, a0);
                    a1 = fmaf(emd_ex2(level2 * emd_sq(xb, yb, zb, o0.x, o0.y, o0.z)), o0.w, a1);
                    a2 = fmaf(emd_ex2(level2 * emd_sq(xa, ya, za, o1.x, o1.y, o1.z)), o1.w, a2);
                    a3 = fmaf(emd_ex2(level2 * emd_sq(xb, yb, zb, o1.x, o1.y, o1.z)), o1.w, a3);
                }
                if (c < cn) {
                    const float4 o0 = so[c];
                    a0 = fmaf(emd_ex2(level2 * emd_sq(xa, ya, za, o0.x, o0.y, o0.z)), o0.w, a0);
                    a1 = fmaf(emd_ex2(level2 * emd_sq(xb, yb, zb, o0.x, o0.y, o0.z)), o0.w, a1);
                }
            } else if (la) {
                int c = l_in;
#pragma unroll 2
                for (; c + 3 * S < cn; c += 4 * S) {
                    const float4 o0 = so[c], o1 = so[c + S], o2 = so[c + 2 * S], o3 = so[c + 3 * S];
                    a0 = fmaf(emd_ex2(level2 * emd_sq(xa, ya, za, o0.x, o0.y, o0.z)), o0.w, a0);
                    a1 = fmaf(emd_ex2(level2 * emd_sq(xa, ya, za, o1.x, o1.y, o1.z)), o1.w, a1);
                    a2 = fmaf(emd_ex2(level2 * emd_sq(xa, ya, za, o2.x, o2.y, o2.z)), o2.w, a2);
                    a3 = fmaf(emd_ex2(level2 * emd_sq(xa, ya, za, o3.x, o3.y, o3.z)), o3.w, a3);
                }
                for (; c < cn; c += S) {
                    const float4 o0 = so[c];
                    a0 = fmaf(emd_ex2(level2 * emd_sq(xa, ya, za, o0.x, o0.y, o0.z)), o0.w, a0);
                }
            }
        }
        if (two) { a0 += a2; a1 += a3; } else { a0 = (a0 + a1) + (a2 + a3); a1 = 0.f; }
        for (int o = S >> 1; o > 0; o >>= 1) {
            a0 += __shfl_xor_sync(kFullMask, a0, o);
            a1 += __shfl_xor_sync(kFullMask, a1, o);
        }
        if (l_in == 0) {
            if (la) finish(bia, ra, a0);
            if (lb) finish(bi0, rb, a1);
        }
        f0 = fend;
    }
}

// The reference read-modify-writes the (b, m, n) match tensor once per level (10 sweeps, 17 GB at the AE size).  Here the ten
// levels only update the per-point vectors (the per-level ratioL / ratioR are kept: 10 x (n + m) floats per cloud), and `match`
// is produced by ONE final pass that re-evaluates the ten weights of a pair in registers, in level order, and writes it once:
//   match[l][k] = sum_lev exp(level_lev * d(k,l)) * ratioL_lev[k] * ratioR_lev[l]
// One extra exp per pair and level buys the removal of all match traffic but the final store.
// kStoreMatch = false stops after the levels: the ratios stay in the workspace and the per-cloud EMD kernels below rebuild the match
// values from them where they need them (emd_match_value), so no (b, m, n) tensor exists at all.
// Persistent cooperative grid (2 CTAs per SM), phases separated by a grid barrier (31 per launch).
template <bool kStoreMatch>
__global__ void __launch_bounds__(kEmdThreads, 2) approxmatch_kernel(const __grid_constant__ EmdParams P)
{
    const int n = P.n, m = P.m, S = P.S, b = P.b;
    const size_t vs = (size_t)(n + m) * (1 + kEmdLevels);    // floats of per-point vectors per cloud
    float *remainL = P.temp, *remainR = remainL + n;          // + bi * vs
    float *ratios = remainR + m;                              // [level][ratioL (n) | ratioR (m)]
    unsigned *counter = P.counter;
    const unsigned G = gridDim.x;
    unsigned epoch = 0;

    __shared__ float4 s_o[2][kEmdTile];

    float multiL, multiR;  // tf_approxmatch_g.cu:4-10 (integer division)
    if (n >= m) { multiL = 1; multiR = (float)(n / m); } else { multiL = (float)(m / n); multiR = 1; }
    for (long long e = (long long)blockIdx.x * kEmdThreads + threadIdx.x; e < (long long)b * (n + m); e += (long long)G * kEmdThreads) {
        const int bi = (int)(e / (n + m)), j = (int)(e - (long long)bi * (n + m));
        (P.temp + (size_t)bi * vs)[j] = j < n ? multiL : multiR;
    }
    emd_grid_barrier(counter, ++epoch * G);

    for (int lev = 7, li = 0; lev >= -2; lev--, li++) {
        const float level2 = emd_level2(lev);
        float *ratioL = ratios + (size_t)li * (n + m), *ratioR = ratioL + n;   // + bi * vs

        // ---- phase 1 (:27-60): ratioL[k] = remainL[k] / (1e-9 + sum_l exp(level*d) * remainR[l])
        emd_row_pass(b, n, m, P.xyz1, b, P.xyz2, P.b2, remainR, vs, level2, S, s_o,
                     [&](int bi, int k, float suml) { ratioL[bi * vs + k] = remainL[bi * vs + k] / (suml + 1e-9f); });
        emd_grid_barrier(counter, ++epoch * G);
        // ---- phase 2 (:75-111): per xyz2 point l: sumr = remainR[l] * sum_k exp(level*d) * ratioL[k]
        emd_row_pass(b, m, n, P.xyz2, P.b2, P.xyz1, b, ratioL, vs, level2, S, s_o, [&](int bi, int l, float sumr) {
            const float rr = remainR[bi * vs + l];
            sumr *= rr;
            const float consumption = fminf(rr / (sumr + 1e-9f), 1.0f);
            ratioR[bi * vs + l] = consumption * rr;
            remainR[bi * vs + l] = fmaxf(0.0f, rr - sumr);
        });
        emd_grid_barrier(counter, ++epoch * G);
        // ---- phase 3 (:127-160) without the match update: remainL[k] -= sum_l exp(level*d) * ratioL[k] * ratioR[l]
        emd_row_pass(b, n, m, P.xyz1, b, P.xyz2, P.b2, ratioR, vs, level2, S, s_o,
                     [&](int bi, int k, float suml) { remainL[bi * vs + k] = fmaxf(0.0f, remainL[bi * vs + k] - suml * ratioL[bi * vs + k]); });
        emd_grid_barrier(counter, ++epoch * G);
    }
    if constexpr (!kStoreMatch) return;

    // ---- final pass: work item = (cloud, block of 512 k, chunk of kFinTile l); thread = k (coalesced stores along k); ten weights
    //      per pair, summed in level order
    float lv2[kEmdLevels];
    emd_level2_all(lv2);
    float *s_r = reinterpret_cast<float *>(&s_o[0][0]);     // [tile l][kEmdLevels] ratioR of the staged columns (reuses the tile buffer)
    constexpr int kFinTile = (kEmdTile * 4) / (kEmdLevels + 3);   // columns per stage: xyz (3) + ten ratios
    float *s_xyz = s_r + kFinTile * kEmdLevels;
    const int kblocks = (n + kEmdThreads - 1) / kEmdThreads, lchunks = (m + kFinTile - 1) / kFinTile;
    const long long items = (long long)b * kblocks * lchunks;
    for (long long it = blockIdx.x; it < items; it += G) {
        const int lc = (int)(it % lchunks);
        const int kb = (int)((it / lchunks) % kblocks);
        const int bi = (int)(it / ((long long)lchunks * kblocks));
        const float *p1 = P.xyz1 + (size_t)bi * n * 3, *p2 = P.xyz2 + (size_t)bi * m * 3;
        const float *rat = ratios + (size_t)bi * vs;
        float *match = P.match + (size_t)bi * n * m;
        const int k = kb * kEmdThreads + threadIdx.x;
        const bool live = k < n;
        float x1 = 0, y1 = 0, z1 = 0, rl[kEmdLevels];
        if (live) { x1 = p1[k * 3 + 0]; y1 = p1[k * 3 + 1]; z1 = p1[k * 3 + 2]; }
#pragma unroll
        for (int li = 0; li < kEmdLevels; li++) rl[li] = live ? rat[(size_t)li * (n + m) + k] : 0.f;
        const int l0 = lc * kFinTile, ln = min(kFinTile, m - l0);
        __syncthreads();
        for (int e = threadIdx.x; e < ln * kEmdLevels; e += kEmdThreads) {
            const int l = e / kEmdLevels, li = e - l * kEmdLevels;
            s_r[e] = rat[(size_t)li * (n + m) + n + l0 + l];
        }
        for (int e = threadIdx.x; e < ln * 3; e += kEmdThreads) s_xyz[e] = p2[(size_t)l0 * 3 + e];
        __syncthreads();
        if (live) {
#pragma unroll 2
            for (int l = 0; l < ln; l++) {
                const float d2 = emd_sq_rn(x1, y1, z1, s_xyz[l * 3 + 0], s_xyz[l * 3 + 1], s_xyz[l * 3 + 2]);
                const float acc = emd_match_value(d2, lv2, rl, s_r + l * kEmdLevels);
                __stcs(match + (size_t)(l0 + l) * n + k, acc);     // written once, read later by other kernels: streaming store
            }
        }
    }
}

struct EmdWorkspace { unsigned *counter; float *temp; size_t total; };

static EmdWorkspace carve_approxmatch_ws(void *base, int b, int n, int m)
{
    EmdWorkspace W;
    WsCarver c(base);
    W.counter = c.take<unsigned>(1);   // grid-barrier word, alone in the first 256 bytes
    W.temp = c.take<float>(0);         // then the per-cloud vectors up to the end, unpadded
    W.total = c.off + (size_t)b * (n + m) * (1 + kEmdLevels) * sizeof(float);
    return W;
}

size_t approxmatch_workspace_bytes(int b, int n, int m) { return carve_approxmatch_ws(nullptr, b, n, m).total; }

// The ten levels (and with kStoreMatch the final pass) on the cooperative grid.  The grid size and the lanes per row S fix the row
// chunking and with it the bits of every ratio, so both instantiations take them from this one rule for the same (b, n, m).
template <bool kStoreMatch>
static int launch_approxmatch_levels(int b, int n, int m, const float *xyz1, const float *xyz2, int b2, float *match, unsigned *counter,
                                     float *temp, cudaStream_t stream)
{
    EmdParams P;
    P.b = b; P.n = n; P.m = m; P.b2 = b2; P.xyz1 = xyz1; P.xyz2 = xyz2; P.match = match;
    P.counter = counter; P.temp = temp;
    // grid: every SM gets two CTAs unless the batch is too small to give each CTA rows
    int per_sm = 0;
    const int sms = num_sms();
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, approxmatch_kernel<kStoreMatch>, kEmdThreads, 0);
    if (per_sm < 1) { set_error("approxmatch: kernel does not fit an SM"); return SNB200_ECUDA; }
    const long long rows = (long long)b * min(n, m);
    int grid = min(per_sm, 2) * sms;
    // lanes per row for the reductions: spread short batches over the idle threads (>= 16 columns per lane)
    int S = 1;
    while (S < 32 && rows * (S * 2) <= (long long)grid * kEmdThreads / 2 && min(n, m) / (S * 2) >= 16) S *= 2;
    P.S = S;
    const long long warps_needed = (rows * S + 31) / 32;   // keep the whole grid unless CTAs would get less than a warp of rows
    grid = (int)max(1ll, min((long long)grid, warps_needed));
    cudaMemsetAsync(P.counter, 0, sizeof(unsigned), stream);
    void *args[] = {(void *)&P};
    cudaError_t e = cudaLaunchCooperativeKernel((const void *)approxmatch_kernel<kStoreMatch>, dim3(grid), dim3(kEmdThreads), args, 0, stream);
    if (e != cudaSuccess) { set_error("approxmatch: cooperative launch failed: %s", cudaGetErrorString(e)); cudaGetLastError(); return SNB200_ECUDA; }
    return check_launch("approxmatch");
}

int launch_approxmatch(int b, int n, int m, const float *xyz1, const float *xyz2, float *match, void *workspace, cudaStream_t stream)
{
    if (b == 0) return SNB200_OK;
    const EmdWorkspace W = carve_approxmatch_ws(workspace, b, n, m);
    return launch_approxmatch_levels<true>(b, n, m, xyz1, xyz2, b, match, W.counter, W.temp, stream);
}

// ------------------------------------------------------------------------------------------------------------------
// Exact mode (SNB200_EMD_EXACT): the parity path.  The fast kernel above evaluates exp as one MUFU.EX2 and sums a row with S lanes x 4
// accumulators; the level schedule then amplifies those roundings wherever `remain` runs towards zero, so its `match` agrees with the
// CPU oracle to ~1e-3 absolute only and arg-max assignments can flip at near-ties.  This kernel reproduces the oracle's arithmetic
// operation by operation (oracle/samplenet_oracle.c:orc_approxmatch, itself a restatement of tf_approxmatch_g.cu:21-160 in the
// reference's level order 7 ... -2): one thread owns a row and accumulates over the columns IN INDEX ORDER in one float accumulator,
// no FMA contraction, exp(d) evaluated in double and rounded to float (both sides obtain the correctly rounded float exponential),
// `match` zero-filled and read-modify-written per level like the reference.  One CTA per cloud, per-point vectors in shared memory.
// kStoreMatch = false is the per-cloud EMD's exact route: the same arithmetic with no `match` at all; each level's ratioL / ratioR go
// to the workspace instead, laid out as approxmatch_kernel<false> leaves them, and the match_cost kernels below rebuild every match
// element from them (emd_exact_match_value).
// ------------------------------------------------------------------------------------------------------------------
constexpr int kEmdExactThreads = 1024;
constexpr int kEmdExactSmemMax = 200 * 1024;   // remainL, remainR, ratioL, ratioR: 2 * (n + m) floats, so n + m <= 25600

__device__ __forceinline__ float emd_exact_exp(float level, float x1, float y1, float z1, float x2, float y2, float z2)
{
    const float dx = __fsub_rn(x2, x1), dy = __fsub_rn(y2, y1), dz = __fsub_rn(z2, z1);
    const float s = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    return (float)exp((double)__fmul_rn(level, s));
}
__device__ __forceinline__ float emd_exact_level(int j)   // -4^j, exact; 0 at the last level (j = -2)
{
    float level = 0.f;
    if (j != -2) { level = 1.f; for (int e = 0; e < (j < 0 ? -j : j); e++) level = (j < 0) ? level * 0.25f : level * 4.f; level = -level; }
    return level;
}
// level j's weight of the pair (xyz1 point, xyz2 point): what phase 3 adds to match[l][k] and to remainL's sum
__device__ __forceinline__ float emd_exact_term(float level, float x1, float y1, float z1, float x2, float y2, float z2, float rl, float rr)
{
    return __fmul_rn(__fmul_rn(emd_exact_exp(level, x1, y1, z1, x2, y2, z2), rl), rr);
}
// One exact-mode match element rebuilt from the kept per-level ratios: the stored kernel zero-fills it and adds level 7's term, then
// level 6's, ... level -2's, each with __fadd_rn, so (((0 + w7) + w6) + ... + w-2) is its value bit for bit.
__device__ __forceinline__ float emd_exact_match_value(float x1, float y1, float z1, float x2, float y2, float z2, const float *rl, const float *rr)
{
    float acc = 0.f;
#pragma unroll
    for (int li = 0; li < kEmdLevels; li++) acc = __fadd_rn(acc, emd_exact_term(emd_exact_level(7 - li), x1, y1, z1, x2, y2, z2, rl[li], rr[li]));
    return acc;
}

// match (b, m, n) with kStoreMatch; otherwise ratios: pair bi, level li: ratioL (n) at ratios + bi * vs + li * (n + m), ratioR (m) after it.
// Pair bi reads xyz2[bi % b2].
template <bool kStoreMatch>
__global__ void __launch_bounds__(kEmdExactThreads) approxmatch_exact_kernel(int n, int m, int b2, const float *__restrict__ xyz1,
                                                                            const float *__restrict__ xyz2, float *__restrict__ match,
                                                                            float *__restrict__ ratios, size_t vs)
{
    extern __shared__ float s_vec[];   // remainL[n] remainR[m] ratioL[n] ratioR[m]
    float *remainL = s_vec, *remainR = s_vec + n, *ratioL = s_vec + n + m, *ratioR = s_vec + 2 * n + m;
    const int bi = blockIdx.x, tid = threadIdx.x;
    const float *p1 = xyz1 + (size_t)bi * n * 3, *p2 = xyz2 + (size_t)(bi % b2) * m * 3;
    float *mt = kStoreMatch ? match + (size_t)bi * n * m : nullptr;
    float *rat = kStoreMatch ? nullptr : ratios + (size_t)bi * vs;
    float multiL, multiR;   // tf_approxmatch_g.cu:4-10 (integer division)
    if (n >= m) { multiL = 1.f; multiR = (float)(n / m); } else { multiL = (float)(m / n); multiR = 1.f; }
    if constexpr (kStoreMatch)
        for (size_t j = tid; j < (size_t)n * m; j += kEmdExactThreads) mt[j] = 0.f;
    for (int j = tid; j < n; j += kEmdExactThreads) remainL[j] = multiL;
    for (int j = tid; j < m; j += kEmdExactThreads) remainR[j] = multiR;
    __syncthreads();
    for (int j = 7; j >= -2; j--) {
        const float level = emd_exact_level(j);
        float *ratL = kStoreMatch ? nullptr : rat + (size_t)(7 - j) * (n + m), *ratR = kStoreMatch ? nullptr : ratL + n;
        for (int k = tid; k < n; k += kEmdExactThreads) {
            const float x1 = p1[k * 3 + 0], y1 = p1[k * 3 + 1], z1 = p1[k * 3 + 2];
            float suml = 1e-9f;
            for (int l = 0; l < m; l++)
                suml = __fadd_rn(suml, __fmul_rn(emd_exact_exp(level, x1, y1, z1, p2[l * 3 + 0], p2[l * 3 + 1], p2[l * 3 + 2]), remainR[l]));
            ratioL[k] = __fdiv_rn(remainL[k], suml);
            if constexpr (!kStoreMatch) ratL[k] = ratioL[k];
        }
        __syncthreads();
        for (int l = tid; l < m; l += kEmdExactThreads) {
            const float x2 = p2[l * 3 + 0], y2 = p2[l * 3 + 1], z2 = p2[l * 3 + 2];
            float sumr = 0.f;
            for (int k = 0; k < n; k++)
                sumr = __fadd_rn(sumr, __fmul_rn(emd_exact_exp(level, p1[k * 3 + 0], p1[k * 3 + 1], p1[k * 3 + 2], x2, y2, z2), ratioL[k]));
            const float rr = remainR[l];
            sumr = __fmul_rn(sumr, rr);
            const float consumption = fminf(__fdiv_rn(rr, __fadd_rn(sumr, 1e-9f)), 1.0f);
            ratioR[l] = __fmul_rn(consumption, rr);
            remainR[l] = fmaxf(0.0f, __fsub_rn(rr, sumr));
            if constexpr (!kStoreMatch) ratR[l] = ratioR[l];
        }
        __syncthreads();
        for (int k = tid; k < n; k += kEmdExactThreads) {
            const float x1 = p1[k * 3 + 0], y1 = p1[k * 3 + 1], z1 = p1[k * 3 + 2];
            const float rl = ratioL[k];
            float suml = 0.f;
            for (int l = 0; l < m; l++) {
                const float w = emd_exact_term(level, x1, y1, z1, p2[l * 3 + 0], p2[l * 3 + 1], p2[l * 3 + 2], rl, ratioR[l]);
                if constexpr (kStoreMatch) mt[(size_t)l * n + k] = __fadd_rn(mt[(size_t)l * n + k], w);
                suml = __fadd_rn(suml, w);
            }
            remainL[k] = fmaxf(0.0f, __fsub_rn(remainL[k], suml));
        }
        __syncthreads();
    }
}

template <bool kStoreMatch>
static int launch_approxmatch_exact_kernel(int b, int n, int m, int b2, const float *xyz1, const float *xyz2, float *match, float *ratios, size_t vs,
                                           cudaStream_t stream)
{
    const size_t smem = (size_t)2 * (n + m) * sizeof(float);
    static PerDeviceOnce once;
    if (once.first()) cudaFuncSetAttribute(approxmatch_exact_kernel<kStoreMatch>, cudaFuncAttributeMaxDynamicSharedMemorySize, kEmdExactSmemMax);
    approxmatch_exact_kernel<kStoreMatch><<<b, kEmdExactThreads, smem, stream>>>(n, m, b2, xyz1, xyz2, match, ratios, vs);
    return check_launch("approxmatch exact");
}

int launch_approxmatch_exact(int b, int n, int m, const float *xyz1, const float *xyz2, float *match, cudaStream_t stream)
{
    if (b == 0) return SNB200_OK;
    const size_t smem = (size_t)2 * (n + m) * sizeof(float);
    if (smem > kEmdExactSmemMax) { set_error("approxmatch (exact mode): %d + %d points exceed the shared-memory vectors", n, m); return SNB200_EUNSUPPORTED; }
    return launch_approxmatch_exact_kernel<true>(b, n, m, b, xyz1, xyz2, match, nullptr, 0, stream);
}

// ------------------------------------------------------------------------------------------------------------------
// match_cost (:183-225): cost[b] = sum_{k,l} match[b][l][k] * ||xyz1[k] - xyz2[l]||.
// Streaming kernels: `match` is read exactly once, 16 bytes per thread and load (k runs fastest in memory), several loads in
// flight per thread; per-CTA partials are combined in slab order by a second tiny kernel (deterministic).
//
// The same kernels serve the per-cloud EMD (kRebuild): there no match tensor exists, and each weight is rebuilt where the kernel would
// have loaded it, from the per-level ratios approxmatch_kernel<false> left in the workspace, with the final pass's expression
// (emd_match_value).  The weights are then the bits the stored tensor would hold and every sum runs in the same order, so cost and
// gradients are bit for bit those of the stored route.  The rebuilt route also takes xyz2 with b2 clouds (pair bi uses xyz2[bi % b2]) and
// applies grad_cost[bi] to each finished gradient component as one multiply.  In the exact mode the ratios are those of
// approxmatch_exact_kernel<false> and each weight is rebuilt with the exact kernel's own expression (emd_exact_match_value).
// ------------------------------------------------------------------------------------------------------------------
constexpr int kMcThreads = 256;
constexpr int kMcSlabs = 16;

// where the kernels take their match weights: loaded from `match`, or rebuilt from the ratios of the fast or the exact levels
enum class EmdSrc { kStored, kFast, kExact };

// match[l][k] of the pair (xyz1 point k, xyz2 point l) rebuilt from its ten ratioL (rl) and ratioR (rr); lv2: emd_level2_all
template <EmdSrc kSrc>
__device__ __forceinline__ float emd_rebuilt_value(float x1, float y1, float z1, float x2, float y2, float z2, const float *lv2, const float *rl,
                                                   const float *rr)
{
    if constexpr (kSrc == EmdSrc::kExact) return emd_exact_match_value(x1, y1, z1, x2, y2, z2, rl, rr);
    else return emd_match_value(emd_sq_rn(x1, y1, z1, x2, y2, z2), lv2, rl, rr);
}

struct EmdWeights {
    const float *match;       // stored: (b, m, n)
    const float *ratios;      // rebuilt: pair bi, level li: ratioL (n) at ratios + bi * vs + li * (n + m), ratioR (m) right after it
    size_t vs;
    int b2;                   // xyz2 holds b2 clouds (b2 == b on the stored route)
    const float *grad_cost;   // rebuilt backward: (b)
};

// the ten ratioL of point k (or ratioR of point n + l)
__device__ __forceinline__ void emd_ratios_of(const float *rat, int n, int m, int j, float *r)
{
#pragma unroll
    for (int li = 0; li < kEmdLevels; li++) r[li] = rat[(size_t)li * (n + m) + j];
}
// stage the ten ratios of points j0 .. j0 + cnt - 1 (offset `side`: 0 for ratioL, n for ratioR) as [point][level], as the final pass does
__device__ __forceinline__ void emd_stage_ratios(float *s_r, const float *rat, int n, int m, int side, int j0, int cnt)
{
    for (int e = threadIdx.x; e < cnt * kEmdLevels; e += blockDim.x) {
        const int j = e / kEmdLevels, li = e - j * kEmdLevels;
        s_r[e] = rat[(size_t)li * (n + m) + side + j0 + j];
    }
}

template <bool kVec, EmdSrc kSrc>
__global__ void __launch_bounds__(kMcThreads, kSrc == EmdSrc::kExact ? 1 : 0) matchcost_partial_kernel(int b, int n, int m, const float *__restrict__ xyz1, const float *__restrict__ xyz2,
                                                                      const EmdWeights Wt, float *__restrict__ partial)
{
    constexpr bool kRebuild = kSrc != EmdSrc::kStored;
    __shared__ float s_red[kMcThreads / 32];
    extern __shared__ float s_p2[];     // the slab's xyz2 points (rebuilt: then their ratioR, [l][level])
    const int bi = blockIdx.y, slab = blockIdx.x;
    const int l_beg = (int)((long long)m * slab / kMcSlabs), l_end = (int)((long long)m * (slab + 1) / kMcSlabs);
    const float *p1 = xyz1 + (size_t)bi * n * 3, *p2 = xyz2 + (size_t)(bi % Wt.b2) * m * 3;
    const float *mt = kRebuild ? nullptr : Wt.match + (size_t)bi * n * m;
    const float *rat = kRebuild ? Wt.ratios + (size_t)bi * Wt.vs : nullptr;
    float *s_rr = s_p2 + (size_t)(l_end - l_beg) * 3;
    float lv2[kEmdLevels];
    emd_level2_all(lv2);
    for (int i = threadIdx.x; i < (l_end - l_beg) * 3; i += kMcThreads) s_p2[i] = p2[(size_t)l_beg * 3 + i];
    if (kRebuild) emd_stage_ratios(s_rr, rat, n, m, n, l_beg, l_end - l_beg);
    __syncthreads();
    float sub = 0.f;
    if (kVec) {
        for (int k4 = threadIdx.x; k4 < (n >> 2); k4 += kMcThreads) {
            float x1[4], y1[4], z1[4], rl[4][kEmdLevels];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                x1[u] = p1[(k4 * 4 + u) * 3 + 0]; y1[u] = p1[(k4 * 4 + u) * 3 + 1]; z1[u] = p1[(k4 * 4 + u) * 3 + 2];
                if (kRebuild) emd_ratios_of(rat, n, m, k4 * 4 + u, rl[u]);
            }
            const float4 *row = kRebuild ? nullptr : reinterpret_cast<const float4 *>(mt + (size_t)l_beg * n) + k4;
            const size_t stride4 = (size_t)(n >> 2);
            const int nl = l_end - l_beg;
            for (int lb = 0; lb < nl; lb += 8) {   // 8 independent 16-byte loads in flight per thread, then the arithmetic
                float4 w[8];
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    if (kRebuild) {
                        const int l = lb + u;
                        w[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (l < nl) {
                            const float x2 = s_p2[l * 3 + 0], y2 = s_p2[l * 3 + 1], z2 = s_p2[l * 3 + 2];
                            const float *rr = s_rr + l * kEmdLevels;
                            w[u].x = emd_rebuilt_value<kSrc>(x1[0], y1[0], z1[0], x2, y2, z2, lv2, rl[0], rr);
                            w[u].y = emd_rebuilt_value<kSrc>(x1[1], y1[1], z1[1], x2, y2, z2, lv2, rl[1], rr);
                            w[u].z = emd_rebuilt_value<kSrc>(x1[2], y1[2], z1[2], x2, y2, z2, lv2, rl[2], rr);
                            w[u].w = emd_rebuilt_value<kSrc>(x1[3], y1[3], z1[3], x2, y2, z2, lv2, rl[3], rr);
                        }
                    } else {
                        w[u] = (lb + u < nl) ? __ldcs(row + (size_t)(lb + u) * stride4) : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    const int l = min(lb + u, nl - 1);
                    const float x2 = s_p2[l * 3 + 0], y2 = s_p2[l * 3 + 1], z2 = s_p2[l * 3 + 2];
                    sub += sqrtf(emd_sq(x1[0], y1[0], z1[0], x2, y2, z2)) * w[u].x;
                    sub += sqrtf(emd_sq(x1[1], y1[1], z1[1], x2, y2, z2)) * w[u].y;
                    sub += sqrtf(emd_sq(x1[2], y1[2], z1[2], x2, y2, z2)) * w[u].z;
                    sub += sqrtf(emd_sq(x1[3], y1[3], z1[3], x2, y2, z2)) * w[u].w;
                }
            }
        }
    } else {
        for (int k = threadIdx.x; k < n; k += kMcThreads) {
            const float x1 = p1[k * 3 + 0], y1 = p1[k * 3 + 1], z1 = p1[k * 3 + 2];
            float rl[kEmdLevels];
            if (kRebuild) emd_ratios_of(rat, n, m, k, rl);
#pragma unroll 4
            for (int l = l_beg; l < l_end; l++) {
                const float x2 = s_p2[(l - l_beg) * 3 + 0], y2 = s_p2[(l - l_beg) * 3 + 1], z2 = s_p2[(l - l_beg) * 3 + 2];
                const float w = kRebuild ? emd_rebuilt_value<kSrc>(x1, y1, z1, x2, y2, z2, lv2, rl, s_rr + (l - l_beg) * kEmdLevels)
                                         : mt[(size_t)l * n + k];
                sub += sqrtf(emd_sq(x1, y1, z1, x2, y2, z2)) * w;
            }
        }
    }
    sub = warp_sum(sub);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = sub;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < kMcThreads / 32; i++) t += s_red[i];
        partial[bi * kMcSlabs + slab] = t;
    }
}
__global__ void matchcost_final_kernel(int b, const float *__restrict__ partial, float *__restrict__ cost)
{
    const int bi = blockIdx.x * blockDim.x + threadIdx.x;
    if (bi < b) {
        float t = 0.f;
        for (int s = 0; s < kMcSlabs; s++) t += partial[bi * kMcSlabs + s];
        cost[bi] = t;
    }
}

// grad1 (:263-291): grad1[k] = sum_l match[l][k] * (x1-x2) / max(|x1-x2|, 1e-10).  CTA = 8 warps over a block of k: lane = k (vector
// path: 4 consecutive k), warp w takes the rows l == w (mod 8) with 8 loads in flight; the 8 partial sums of a k are combined through
// shared memory in warp order (deterministic).  The rebuilt route stages half a tile of xyz2 with its ratioR: a warp still visits its
// rows in increasing l, as the groups of 64 rows stay aligned, so the sums are the same.
constexpr int kMgThreads = 256;
template <bool kVec, EmdSrc kSrc>
__global__ void __launch_bounds__(kMgThreads) matchcostgrad1_kernel(int b, int n, int m, const float *__restrict__ xyz1, const float *__restrict__ xyz2,
                                                                   const EmdWeights Wt, float *__restrict__ grad1)
{
    constexpr bool kRebuild = kSrc != EmdSrc::kStored;
    constexpr int W = kVec ? 4 : 1;
    constexpr int kTile = kRebuild ? kEmdTile / 2 : kEmdTile;
    __shared__ float s_o[kTile * 3];
    __shared__ float s_rr[kRebuild ? kTile * kEmdLevels : 1];
    __shared__ float s_acc[8][32 * W * 3];
    const int bi = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k0 = (blockIdx.x * 32 + lane) * W;
    const bool live = k0 < n;
    const float *p1 = xyz1 + (size_t)bi * n * 3, *p2 = xyz2 + (size_t)(bi % Wt.b2) * m * 3;
    const float *mt = kRebuild ? nullptr : Wt.match + (size_t)bi * n * m;
    const float *rat = kRebuild ? Wt.ratios + (size_t)bi * Wt.vs : nullptr;
    float lv2[kEmdLevels];
    emd_level2_all(lv2);
    float x1[W], y1[W], z1[W], dx[W], dy[W], dz[W], rl[W][kEmdLevels];
#pragma unroll
    for (int u = 0; u < W; u++) {
        const int k = min(k0 + u, n - 1);
        x1[u] = p1[k * 3 + 0]; y1[u] = p1[k * 3 + 1]; z1[u] = p1[k * 3 + 2];
        dx[u] = dy[u] = dz[u] = 0.f;
        if (kRebuild) emd_ratios_of(rat, n, m, k, rl[u]);
    }
    for (int l0 = 0; l0 < m; l0 += kTile) {
        const int ln = min(kTile, m - l0);
        __syncthreads();
        for (int i = threadIdx.x; i < ln * 3; i += kMgThreads) s_o[i] = p2[(size_t)l0 * 3 + i];
        if (kRebuild) emd_stage_ratios(s_rr, rat, n, m, n, l0, ln);
        __syncthreads();
        if (live) {
            for (int lb = warp; lb < ln; lb += 8 * 8) {
                float w[8][W];
#pragma unroll
                for (int q = 0; q < 8; q++) {
                    const int l = lb + 8 * q;
                    if (kRebuild) {
                        const float x2 = s_o[min(l, ln - 1) * 3 + 0], y2 = s_o[min(l, ln - 1) * 3 + 1], z2 = s_o[min(l, ln - 1) * 3 + 2];
#pragma unroll
                        for (int u = 0; u < W; u++)
                            w[q][u] = (l < ln) ? emd_rebuilt_value<kSrc>(x1[u], y1[u], z1[u], x2, y2, z2, lv2, rl[u], s_rr + l * kEmdLevels) : 0.f;
                    } else if (kVec) {
                        const float4 v = (l < ln) ? __ldcs(reinterpret_cast<const float4 *>(mt + (size_t)(l0 + l) * n + k0)) : make_float4(0.f, 0.f, 0.f, 0.f);
                        w[q][0] = v.x; w[q][W > 1 ? 1 : 0] = v.y; w[q][W > 2 ? 2 : 0] = v.z; w[q][W > 3 ? 3 : 0] = v.w;
                    } else {
                        w[q][0] = (l < ln) ? __ldcs(mt + (size_t)(l0 + l) * n + k0) : 0.f;
                    }
                }
#pragma unroll
                for (int q = 0; q < 8; q++) {
                    const int l = min(lb + 8 * q, ln - 1);
                    const float x2 = s_o[l * 3 + 0], y2 = s_o[l * 3 + 1], z2 = s_o[l * 3 + 2];
#pragma unroll
                    for (int u = 0; u < W; u++) {
                        const float ex = x1[u] - x2, ey = y1[u] - y2, ez = z1[u] - z2;
                        const float d = w[q][u] * rsqrtf(fmaxf(ex * ex + ey * ey + ez * ez, 1e-20f));
                        dx[u] += ex * d; dy[u] += ey * d; dz[u] += ez * d;
                    }
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < W; u++) {
        s_acc[warp][(lane * W + u) * 3 + 0] = dx[u]; s_acc[warp][(lane * W + u) * 3 + 1] = dy[u]; s_acc[warp][(lane * W + u) * 3 + 2] = dz[u];
    }
    __syncthreads();
    const float g = kRebuild ? Wt.grad_cost[bi] : 1.f;
    for (int e = threadIdx.x; e < 32 * W * 3; e += kMgThreads) {
        const int k = blockIdx.x * 32 * W + e / 3;
        if (k < n) {
            float t = 0.f;
#pragma unroll
            for (int w8 = 0; w8 < 8; w8++) t += s_acc[w8][e];
            grad1[((size_t)bi * n) * 3 + (size_t)blockIdx.x * 32 * W * 3 + e] = kRebuild ? __fmul_rn(t, g) : t;
        }
    }
}

// grad2 (:229-262): grad2[l] = sum_k match[l][k] * (x2-x1) / max(|x2-x1|, 1e-10); one warp per l, lanes along k (coalesced; vector
// path: 4 consecutive k per lane and load), xyz1 staged in shared memory.  The rebuilt route stages half a tile of xyz1 with its ratioL
// (a multiple of 32 x 4 points, so each lane still visits the same k in the same order).
template <bool kVec, EmdSrc kSrc>
__global__ void __launch_bounds__(256, kSrc == EmdSrc::kExact ? 1 : 0) matchcostgrad2_kernel(int b, int n, int m, const float *__restrict__ xyz1, const float *__restrict__ xyz2,
                                                             const EmdWeights Wt, float *__restrict__ grad2)
{
    constexpr bool kRebuild = kSrc != EmdSrc::kStored;
    constexpr int W = kVec ? 4 : 1;
    constexpr int kTile = kRebuild ? kEmdTile / 2 : kEmdTile;
    __shared__ float s_p1[kTile * 3];
    __shared__ float s_rl[kRebuild ? kTile * kEmdLevels : 1];
    const int bi = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int l = blockIdx.x * 8 + warp;
    const bool live = l < m;
    const float *p1 = xyz1 + (size_t)bi * n * 3, *p2 = xyz2 + (size_t)(bi % Wt.b2) * m * 3;
    const float *mt = kRebuild ? nullptr : Wt.match + (size_t)bi * n * m + (size_t)min(l, m - 1) * n;
    const float *rat = kRebuild ? Wt.ratios + (size_t)bi * Wt.vs : nullptr;
    float lv2[kEmdLevels], rr[kEmdLevels];
    emd_level2_all(lv2);
    if (kRebuild) emd_ratios_of(rat, n, m, n + min(l, m - 1), rr);
    float x2 = 0, y2 = 0, z2 = 0;
    if (live) { x2 = p2[l * 3 + 0]; y2 = p2[l * 3 + 1]; z2 = p2[l * 3 + 2]; }
    float sx = 0, sy = 0, sz = 0;
    for (int k0 = 0; k0 < n; k0 += kTile) {
        const int kn = min(kTile, n - k0);
        __syncthreads();
        for (int i = threadIdx.x; i < kn * 3; i += 256) s_p1[i] = p1[(size_t)k0 * 3 + i];
        if (kRebuild) emd_stage_ratios(s_rl, rat, n, m, 0, k0, kn);
        __syncthreads();
        if (live) {
#pragma unroll 4
            for (int k = lane * W; k < kn; k += 32 * W) {
                float w[W];
                if (kRebuild) {
#pragma unroll
                    for (int u = 0; u < W; u++)
                        w[u] = emd_rebuilt_value<kSrc>(s_p1[(k + u) * 3 + 0], s_p1[(k + u) * 3 + 1], s_p1[(k + u) * 3 + 2], x2, y2, z2, lv2,
                                                       s_rl + (k + u) * kEmdLevels, rr);
                } else if (kVec) {
                    const float4 v = __ldcs(reinterpret_cast<const float4 *>(mt + k0 + k));
                    w[0] = v.x; w[W > 1 ? 1 : 0] = v.y; w[W > 2 ? 2 : 0] = v.z; w[W > 3 ? 3 : 0] = v.w;
                } else {
                    w[0] = __ldcs(mt + k0 + k);
                }
#pragma unroll
                for (int u = 0; u < W; u++) {
                    const float ex = x2 - s_p1[(k + u) * 3 + 0], ey = y2 - s_p1[(k + u) * 3 + 1], ez = z2 - s_p1[(k + u) * 3 + 2];
                    const float d = w[u] * rsqrtf(fmaxf(ex * ex + ey * ey + ez * ez, 1e-20f));
                    sx += ex * d; sy += ey * d; sz += ez * d;
                }
            }
        }
    }
    sx = warp_sum(sx); sy = warp_sum(sy); sz = warp_sum(sz);
    if (live && lane == 0) {
        float *g = grad2 + ((size_t)bi * m + l) * 3;
        if (kRebuild) {
            const float gc = Wt.grad_cost[bi];
            g[0] = __fmul_rn(sx, gc); g[1] = __fmul_rn(sy, gc); g[2] = __fmul_rn(sz, gc);
        } else {
            g[0] = sx; g[1] = sy; g[2] = sz;
        }
    }
}

static bool emd_vec_ok(int n, const float *match) { return (n & 3) == 0 && (reinterpret_cast<uintptr_t>(match) & 15) == 0; }

static constexpr size_t matchcost_smem(int m, bool rebuild) { return (size_t)((m + kMcSlabs - 1) / kMcSlabs + 1) * (rebuild ? 3 + kEmdLevels : 3) * sizeof(float); }

// The rebuilt route stages 13 floats per point of a slab instead of 3, so it opts in to more than 48 KB of dynamic shared memory to take
// every m the stored route takes (kEmdPerCloudMaxM below).
constexpr int kMcRebuildSmemMax = 212992;

template <EmdSrc kSrc>
static int launch_matchcost_kernels(int b, int n, int m, const float *xyz1, const float *xyz2, const EmdWeights &Wt, bool vec, float *cost,
                                    float *partial, cudaStream_t stream)
{
    const size_t smem = matchcost_smem(m, kSrc != EmdSrc::kStored);
    if (kSrc != EmdSrc::kStored) {
        static PerDeviceOnce once;
        if (once.first()) {
            cudaFuncSetAttribute(matchcost_partial_kernel<true, kSrc>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMcRebuildSmemMax);
            cudaFuncSetAttribute(matchcost_partial_kernel<false, kSrc>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMcRebuildSmemMax);
        }
    }
    if (vec) matchcost_partial_kernel<true, kSrc><<<dim3(kMcSlabs, b), kMcThreads, smem, stream>>>(b, n, m, xyz1, xyz2, Wt, partial);
    else matchcost_partial_kernel<false, kSrc><<<dim3(kMcSlabs, b), kMcThreads, smem, stream>>>(b, n, m, xyz1, xyz2, Wt, partial);
    int rc = check_launch("matchcost(partial)");
    if (rc) return rc;
    matchcost_final_kernel<<<(b + 127) / 128, 128, 0, stream>>>(b, partial, cost);
    return check_launch("matchcost(final)");
}

// grad1 / grad2 null: that gradient is not computed (the rebuilt route, for a cloud that needs no gradient; the stored route passes both)
template <EmdSrc kSrc>
static int launch_matchcostgrad_kernels(int b, int n, int m, const float *xyz1, const float *xyz2, const EmdWeights &Wt, bool vec, float *grad1,
                                        float *grad2, cudaStream_t stream)
{
    if (grad1) {
        if (vec) matchcostgrad1_kernel<true, kSrc><<<dim3((n + 127) / 128, b), kMgThreads, 0, stream>>>(b, n, m, xyz1, xyz2, Wt, grad1);
        else matchcostgrad1_kernel<false, kSrc><<<dim3((n + 31) / 32, b), kMgThreads, 0, stream>>>(b, n, m, xyz1, xyz2, Wt, grad1);
        if (int rc = check_launch("matchcostgrad1")) return rc;
    }
    if (!grad2) return SNB200_OK;
    if (vec) matchcostgrad2_kernel<true, kSrc><<<dim3((m + 7) / 8, b), 256, 0, stream>>>(b, n, m, xyz1, xyz2, Wt, grad2);
    else matchcostgrad2_kernel<false, kSrc><<<dim3((m + 7) / 8, b), 256, 0, stream>>>(b, n, m, xyz1, xyz2, Wt, grad2);
    return check_launch("matchcostgrad2");
}

int launch_matchcost(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *cost, float *partial, cudaStream_t stream)
{
    if (matchcost_smem(m, false) > 48 * 1024) { set_error("matchcost: m=%d too large", m); return SNB200_EUNSUPPORTED; }
    const EmdWeights Wt{match, nullptr, 0, b, nullptr};
    return launch_matchcost_kernels<EmdSrc::kStored>(b, n, m, xyz1, xyz2, Wt, emd_vec_ok(n, match), cost, partial, stream);
}

int launch_matchcostgrad(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *grad1, float *grad2, cudaStream_t stream)
{
    const EmdWeights Wt{match, nullptr, 0, b, nullptr};
    return launch_matchcostgrad_kernels<EmdSrc::kStored>(b, n, m, xyz1, xyz2, Wt, emd_vec_ok(n, match), grad1, grad2, stream);
}

// ------------------------------------------------------------------------------------------------------------------
// Per-cloud EMD: match_cost(xyz1, xyz2, approx_match(xyz1, xyz2)) and its gradients without the (b, m, n) match tensor.  The forward
// runs the ten levels (approxmatch_kernel<false>, same launch rule, same workspace vectors), then the match_cost kernels with rebuilt
// weights; the backward runs the match_cost_grad kernels with rebuilt weights from the ratios the forward left in the workspace.
// The exact mode runs approxmatch_exact_kernel<false> instead, which leaves its ratios in the same places (its remain vectors stay in
// shared memory and the grid-barrier word is unused), and rebuilds the weights with the exact expression.
// Workspace: the grid-barrier word, the per-cloud vectors of approx_match, the slab partials of match_cost.
// ------------------------------------------------------------------------------------------------------------------
struct EmdPerCloudWorkspace { unsigned *counter; float *temp; float *partial; size_t total; };

static EmdPerCloudWorkspace carve_emd_per_cloud_ws(void *base, int b, int n, int m)
{
    EmdPerCloudWorkspace W;
    WsCarver c(base);
    W.counter = c.take<unsigned>(1);
    W.temp = c.take<float>((size_t)b * (n + m) * (1 + kEmdLevels));
    W.partial = c.take<float>((size_t)b * kMcSlabs);
    W.total = c.off;
    return W;
}

// envelope: b is a grid dimension; m is the stored route's limit (match_cost stages a 16th of xyz2 in 48 KB of shared memory), which the
// rebuilt route reaches with its larger dynamic shared memory; n is bounded where the kernels' 32-bit point offsets still have ample room.
// The exact mode is bounded by the exact kernel's shared-memory vectors, as approx_match's exact mode is.
constexpr int kEmdPerCloudMaxN = 1 << 24, kEmdPerCloudMaxM = 65520;
constexpr int kEmdExactMaxPoints = kEmdExactSmemMax / (2 * (int)sizeof(float));   // n + m
static_assert(matchcost_smem(kEmdPerCloudMaxM, false) <= 48 * 1024 && matchcost_smem(kEmdPerCloudMaxM + 1, false) > 48 * 1024, "m envelope");
static_assert(matchcost_smem(kEmdPerCloudMaxM, true) <= kMcRebuildSmemMax, "rebuilt cost kernel's shared memory");
static_assert(kEmdExactMaxPoints < kEmdPerCloudMaxM, "the exact envelope lies inside the cost kernel's");

bool emd_per_cloud_supported(int b, int n, int m, bool exact)
{
    if (exact) return b >= 1 && b <= 65535 && n >= 1 && m >= 1 && (long long)n + m <= kEmdExactMaxPoints;
    return b >= 1 && b <= 65535 && n >= 1 && n <= kEmdPerCloudMaxN && m >= 1 && m <= kEmdPerCloudMaxM;
}

size_t emd_per_cloud_workspace_bytes(int b, int n, int m) { return carve_emd_per_cloud_ws(nullptr, b, n, m).total; }

static EmdWeights emd_rebuilt_weights(const EmdPerCloudWorkspace &W, int n, int m, int b2, const float *grad_cost)
{
    const size_t vs = (size_t)(n + m) * (1 + kEmdLevels);
    return EmdWeights{nullptr, W.temp + (size_t)(n + m), vs, b2, grad_cost};   // the ratios follow remainL / remainR in each cloud's block
}

int launch_emd_per_cloud(int b, int n, int m, const float *xyz1, const float *xyz2, int b2, bool exact, float *cost, void *workspace, cudaStream_t stream)
{
    if (b == 0) return SNB200_OK;
    const EmdPerCloudWorkspace W = carve_emd_per_cloud_ws(workspace, b, n, m);
    const EmdWeights Wt = emd_rebuilt_weights(W, n, m, b2, nullptr);
    if (exact) {
        if (int rc = launch_approxmatch_exact_kernel<false>(b, n, m, b2, xyz1, xyz2, nullptr, W.temp + (size_t)(n + m), Wt.vs, stream)) return rc;
        return launch_matchcost_kernels<EmdSrc::kExact>(b, n, m, xyz1, xyz2, Wt, (n & 3) == 0, cost, W.partial, stream);
    }
    if (int rc = launch_approxmatch_levels<false>(b, n, m, xyz1, xyz2, b2, nullptr, W.counter, W.temp, stream)) return rc;
    return launch_matchcost_kernels<EmdSrc::kFast>(b, n, m, xyz1, xyz2, Wt, (n & 3) == 0, cost, W.partial, stream);
}

int launch_emd_per_cloud_backward(int b, int n, int m, const float *xyz1, const float *xyz2, int b2, bool exact, const float *grad_cost, float *grad1,
                                  float *grad2, const void *workspace, cudaStream_t stream)
{
    if (b == 0) return SNB200_OK;
    const EmdPerCloudWorkspace W = carve_emd_per_cloud_ws(const_cast<void *>(workspace), b, n, m);
    const EmdWeights Wt = emd_rebuilt_weights(W, n, m, b2, grad_cost);
    if (exact) return launch_matchcostgrad_kernels<EmdSrc::kExact>(b, n, m, xyz1, xyz2, Wt, (n & 3) == 0, grad1, grad2, stream);
    return launch_matchcostgrad_kernels<EmdSrc::kFast>(b, n, m, xyz1, xyz2, Wt, (n & 3) == 0, grad1, grad2, stream);
}

}  // namespace snb
