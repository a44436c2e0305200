// common.cuh -- shared device/host helpers for libsamplenet_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <math.h>

#include "../../include/samplenet_b200.h"

#ifndef __CUDA_ARCH__
#define SNB_HOST_ONLY 1
#endif

namespace snb {

constexpr int kNumSMs = 132;  // H100 SXM: num_sms() when the device cannot be queried, and the fixed count of the pairwise planners
constexpr int kStatStride = 16;     // doubles between two BatchNorm statistics accumulators of the conv-stack kernel: one per 128-byte line, so that the
                                   // CTAs' fp64 atomics on different channels do not serialise in the same L2 line

// ------------------------------------------------------------------------------------------- host side
void set_error(const char *fmt, ...);
void count_launch(int n = 1);

inline int check_launch(const char *what)
{
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
        return SNB200_ECUDA;
    }
    count_launch();
    return SNB200_OK;
}

#define SNB_REQUIRE(cond, ...)               \
    do {                                     \
        if (!(cond)) {                       \
            snb::set_error(__VA_ARGS__);     \
            return SNB200_EINVAL;            \
        }                                    \
    } while (0)

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Bump allocator over a workspace: take<T>(count) hands out the next sub-buffer, 256-byte aligned, and `off` is the size so far.  On a null
// base every pointer is null, so one carve function both reports a workspace's size and lays it out.
struct WsCarver {
    char *base;
    size_t off = 0;
    explicit WsCarver(void *b) : base(static_cast<char *>(b)) {}
    template <class T> T *take(size_t count)
    {
        T *p = base ? reinterpret_cast<T *>(base + off) : nullptr;
        off += align_up(count * sizeof(T), 256);
        return p;
    }
};

// SM count of the current device, queried once per device; kNumSMs when the device cannot be queried.
inline int num_sms()
{
    static int sms[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return kNumSMs;
    if (!sms[dev]) {
        int v = 0;
        sms[dev] = (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) ? v : kNumSMs;
    }
    return sms[dev];
}

// cudaFuncSetAttribute is per device: run the opt-in once per (kernel family, device).
struct PerDeviceOnce {
    bool done[64] = {};
    bool first()
    {
        int d = 0;
        if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) return true;
        if (done[d]) return false;
        done[d] = true;
        return true;
    }
};

// ------------------------------------------------------------------------------------------- device side
#ifdef __CUDACC__

constexpr unsigned kFullMask = 0xffffffffu;

// Squared distance in the two evaluation orders of the reference (see include/samplenet_b200.h flags).
template <bool kFma>
__device__ __forceinline__ float sqdist(float dx, float dy, float dz)
{
    if (kFma) {
        // the contraction nvcc applies to (dx*dx + dy*dy) + dz*dz in the reference kernels (chamfer_distance.cu:33-36, tf_nndistance_g.cu:25-28;
        // SASS: FMUL dy*dy, FFMA dx*dx + ., FFMA dz*dz + .): results are bit-identical to the reference's own CUDA ops
        return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
    } else {
        return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    }
}

// ---- mbarrier + 1-D TMA bulk copy (cp.async.bulk, SASS: UBLKCP) -------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// global -> shared bulk copy; dst/src 16-byte aligned, bytes a multiple of 16
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Stage `nfloats` contiguous floats from global to shared with the whole CTA.
// Fast path: one elected thread issues a TMA bulk copy (needs 16 B alignment of both ends and nfloats % 4 == 0),
// everyone waits on the mbarrier.  Slow path (ragged sizes): coalesced LDG/STS.  Both paths end with the data visible
// to all threads of the CTA.  `phase` is the caller-tracked mbarrier parity (flipped here when the TMA path is used).
__device__ __forceinline__ void stage_floats(float *smem_dst, const float *gmem_src, int nfloats, uint64_t *bar, uint32_t &phase)
{
    const bool tma_ok = ((reinterpret_cast<uintptr_t>(gmem_src) & 15) == 0) && ((nfloats & 3) == 0) && nfloats > 0 &&
                        ((smem_u32(smem_dst) & 15) == 0);
    if (tma_ok) {
        if (threadIdx.x == 0) {
            mbar_expect_tx(bar, (uint32_t)nfloats * 4u);
            tma_load_1d(smem_dst, gmem_src, (uint32_t)nfloats * 4u, bar);
        }
        mbar_wait(bar, phase);
        phase ^= 1;
    } else {
        for (int i = threadIdx.x; i < nfloats; i += blockDim.x) smem_dst[i] = __ldg(gmem_src + i);
        __syncthreads();
    }
}

// ---- warpgroup MMA (wgmma, SASS: HGMMA), kind tf32, fp32 accumulators in registers -------------------------
// Shared-memory matrix descriptor: start >> 4 [0,14) | LBO >> 4 [16,30) | SBO >> 4 [32,46) | base offset [49,52) | layout [62,64).
// K-major SWIZZLE_128B operands (rows of 128 B = 32 fp32 along K, 16-byte chunks XOR-swizzled with row % 8, 8-row groups 1024 B
// apart): SBO = 1024 B, LBO unused (1), layout 1 = SWIZZLE_128B; the atom must start on a 1024-byte boundary.  A K step of 8 tf32
// advances the start address by 32 bytes.
constexpr unsigned kWgDescHiSw128 = 64u | (1u << 30);   // bits [32,64) of the descriptor
__device__ __forceinline__ uint64_t wg_sdesc(uint32_t smem_addr)
{
    return (uint64_t)((smem_addr >> 4) & 0x3fffu) | (1ull << 16) | ((uint64_t)kWgDescHiSw128 << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// Accumulator fragment of one m64n64 tile (32 floats per thread, warp w of the warpgroup, g = lane / 4, t = lane % 4):
//   d[4j + 0] = (row 16w + g, col 8j + 2t), d[4j + 1] = (row 16w + g, col 8j + 2t + 1), d[4j + 2 / 3] = the same columns of row 16w + g + 8
#define SNB_WG_D32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
                   "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define SNB_WG_D32_OPS(d)                                                                                                     \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),     \
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),    \
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),    \
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// D[64 x 64] (+)= A[64 x 8] . B[8 x 64], both operands in shared memory (descriptors)
__device__ __forceinline__ void wg_mma_ss_n64(float *d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " SNB_WG_D32 ", %32, %33, p, 1, 1;\n"
        "}\n"
        : SNB_WG_D32_OPS(d)
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// ... with A from registers: a[0] = (row 16w + g, k t), a[1] = (row 16w + g + 8, k t), a[2] / a[3] = the same rows at k t + 4
__device__ __forceinline__ void wg_mma_rs_n64(float *d, const uint32_t *a, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " SNB_WG_D32 ", {%32, %33, %34, %35}, %36, p, 1, 1;\n"
        "}\n"
        : SNB_WG_D32_OPS(d)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}

// exact split of an fp32 value into a TF32 head and an fp32 remainder (3xTF32: A_lo.B_hi + A_hi.B_lo + A_hi.B_hi)
__device__ __forceinline__ float tf32_hi(float v) { return __uint_as_float(__float_as_uint(v) & 0xffffe000u); }

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(kFullMask, v, o));
    return v;
}

#endif  // __CUDACC__
}  // namespace snb
