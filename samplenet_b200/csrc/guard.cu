// guard.cu -- the non-finite step guard (snb200_nonfinite_guard): after a training step, one launch checks a table of tensors for NaN/Inf
// and a second one, only when the check found one, copies every snapshot back over its live tensor.
//
//   check    one CTA per chunk of kGuardCheckChunk elements of a checked tensor; a non-finite element (exponent bits all ones) ORs 1 into
//            the flag word.  Integer atomics only.
//   restore  one CTA per chunk of kGuardCopyChunk bytes of a (live, snapshot) pair; every CTA reads the flag and copies its chunk only when
//            it is set.  The copy moves bits, so -0.0 and NaN payloads come back exactly.  The last CTA to finish (ticket) writes the call's
//            0/1 result, adds it to the optional skip counter and zeroes the flag and the ticket for the next call.
// The tables travel as kernel parameters: the launch (and a graph node capturing it) owns a copy, nothing is allocated and nothing is read
// back.  A table larger than one launch's parameter space is split over more launches of the same kernel; only the last restore launch
// finishes the call.
#include "common.cuh"

namespace snb {

constexpr int kGuardThreads = 256;
constexpr int kGuardCheckChunk = 8192;          // elements per check CTA
constexpr long long kGuardCopyChunk = 65536;    // bytes per restore CTA
// entries per launch: 20 B (check) or 28 B (restore) each with its CTA offset, about 8 and 11 KB of parameters, inside sm_90's 32 KB
constexpr int kGuardChecksPerLaunch = 384;
constexpr int kGuardRestoresPerLaunch = 384;

struct GuardCheckParams {
    int num;                                    // entries in this launch
    int first[kGuardChecksPerLaunch + 1];       // first CTA of each entry; first[num] = grid size
    snb200_guard_check e[kGuardChecksPerLaunch];
    unsigned *state;                            // [0] flag, [1] ticket
};

struct GuardRestoreParams {
    int num;
    int first[kGuardRestoresPerLaunch + 1];
    snb200_guard_restore e[kGuardRestoresPerLaunch];
    unsigned *state;
    int finish;                                 // the call's last restore launch: write the result and zero the state
    int *skipped;
    int *skip_count;
};

// the entry owning CTA `b`: the last i with first[i] <= b (entries without elements own no CTA)
__device__ __forceinline__ int guard_entry(const int *first, int num, int b)
{
    int lo = 0, hi = num - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (first[mid] <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}

template <typename T>
__device__ __forceinline__ bool guard_chunk_bad(const void *ptr, long long lo, long long hi, T mask)
{
    const T *p = static_cast<const T *>(ptr);
    bool bad = false;
    for (long long i = lo + threadIdx.x; i < hi; i += kGuardThreads) bad |= (__ldg(p + i) & mask) == mask;
    return bad;
}

__global__ void __launch_bounds__(kGuardThreads) nonfinite_check_kernel(const __grid_constant__ GuardCheckParams P)
{
    const int i = guard_entry(P.first, P.num, (int)blockIdx.x);
    const snb200_guard_check &E = P.e[i];
    const long long lo = (long long)((int)blockIdx.x - P.first[i]) * kGuardCheckChunk;
    const long long hi = min((long long)E.count, lo + kGuardCheckChunk);
    bool bad;
    switch (E.dtype) {
        case SNB200_GUARD_F64: bad = guard_chunk_bad<unsigned long long>(E.ptr, lo, hi, 0x7ff0000000000000ull); break;
        case SNB200_GUARD_F16: bad = guard_chunk_bad<unsigned short>(E.ptr, lo, hi, (unsigned short)0x7c00); break;
        case SNB200_GUARD_BF16: bad = guard_chunk_bad<unsigned short>(E.ptr, lo, hi, (unsigned short)0x7f80); break;
        default: bad = guard_chunk_bad<unsigned>(E.ptr, lo, hi, 0x7f800000u); break;
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(P.state, 1u);
}

__global__ void __launch_bounds__(kGuardThreads) nonfinite_restore_kernel(const __grid_constant__ GuardRestoreParams P)
{
    const unsigned flag = *reinterpret_cast<volatile unsigned *>(P.state);
    if (flag && P.num > 0) {
        const int i = guard_entry(P.first, P.num, (int)blockIdx.x);
        const snb200_guard_restore &E = P.e[i];
        const long long lo = (long long)((int)blockIdx.x - P.first[i]) * kGuardCopyChunk;
        const long long hi = min(E.bytes, lo + kGuardCopyChunk);
        unsigned char *dst = static_cast<unsigned char *>(E.live);
        const unsigned char *src = static_cast<const unsigned char *>(E.snapshot);
        long long v = lo;
        if ((((uintptr_t)dst | (uintptr_t)src) & 15) == 0) {   // chunks start at multiples of 64 KB: 16-byte words from `lo` on
            const long long nv = (hi - lo) >> 4;
            for (long long k = threadIdx.x; k < nv; k += kGuardThreads)
                reinterpret_cast<uint4 *>(dst + lo)[k] = reinterpret_cast<const uint4 *>(src + lo)[k];
            v = lo + (nv << 4);
        }
        for (long long k = v + threadIdx.x; k < hi; k += kGuardThreads) dst[k] = src[k];
    }
    if (!P.finish) return;
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(P.state + 1, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;
    // every CTA of this launch has read the flag (each took its ticket after): the state can be zeroed for the next call
    __threadfence();
    const int f = flag ? 1 : 0;
    if (P.skipped) *P.skipped = f;
    if (P.skip_count) *P.skip_count += f;
    P.state[0] = 0u;
    P.state[1] = 0u;
}

// CTAs per entry: ceil(size / chunk), none for an empty one
template <typename E, typename F>
static int guard_plan(int *first, const E *e, int num, F ctas_of)
{
    long long total = 0;
    for (int i = 0; i < num; i++) {
        first[i] = (int)total;
        total += ctas_of(e[i]);
    }
    first[num] = (int)total;
    return (int)total;
}

int launch_nonfinite_guard(const snb200_guard_check *checks, int num_checks, const snb200_guard_restore *restores, int num_restores,
                           unsigned *state, int *skipped, int *skip_count, cudaStream_t stream)
{
    for (int c0 = 0; c0 < num_checks; c0 += kGuardChecksPerLaunch) {
        GuardCheckParams P;
        P.num = min(kGuardChecksPerLaunch, num_checks - c0);
        P.state = state;
        for (int i = 0; i < P.num; i++) P.e[i] = checks[c0 + i];
        const int grid = guard_plan(P.first, P.e, P.num, [](const snb200_guard_check &x) {
            return (long long)((x.count + kGuardCheckChunk - 1) / kGuardCheckChunk);
        });
        if (grid == 0) continue;
        nonfinite_check_kernel<<<grid, kGuardThreads, 0, stream>>>(P);
        const int rc = check_launch("nonfinite_guard (check)");
        if (rc) return rc;
    }
    int r0 = 0;
    do {
        GuardRestoreParams P;
        P.num = min(kGuardRestoresPerLaunch, num_restores - r0);
        P.state = state;
        P.finish = r0 + P.num >= num_restores;
        P.skipped = skipped;
        P.skip_count = skip_count;
        for (int i = 0; i < P.num; i++) P.e[i] = restores[r0 + i];
        int grid = guard_plan(P.first, P.e, P.num, [](const snb200_guard_restore &x) { return (x.bytes + kGuardCopyChunk - 1) / kGuardCopyChunk; });
        r0 += P.num;
        if (grid == 0 && !P.finish) continue;
        if (grid == 0) { P.num = 0; grid = 1; }      // nothing to copy: one CTA finishes the call
        nonfinite_restore_kernel<<<grid, kGuardThreads, 0, stream>>>(P);
        const int rc = check_launch("nonfinite_guard (restore)");
        if (rc) return rc;
    } while (r0 < num_restores);
    return SNB200_OK;
}

}  // namespace snb
