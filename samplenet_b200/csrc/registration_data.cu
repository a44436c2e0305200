// registration_data.cu -- the registration trainer's per-record data path in one launch: ModelNetCls.__getitem__'s point permutation
// (registration/data/modelnet_loader_torch.py:102-116) on a set already on the unit cube, then QuaternionFixedDataset.__getitem__'s fixed
// rotation of p0 into p1 (registration/src/qdataset.py:160-179, QuaternionTransform.rotate without the translation).
//
// Contract (include/samplenet_b200.h, snb200_registration_pairs): pair i takes record r = records[i], cloud r % s and transform row r;
//   perm[i] is 0..n-1 in ascending order of the Philox sort keys ((w0 << 32 | w1) & ~0x7FF) | j, p0[i, j] = clouds[r % s, perm[i, j]],
//   p1[i, j] = qrot(q_r, p0[i, j]) in float32 in the operation order of registration.qrot (no contraction), vec[i] = transforms[r].
//
// Design (DESIGN.md 4.11): one CTA per pair.  The n <= 2048 sort keys go through one cub::BlockRadixSort of 256 threads x 8 keys in shared
// memory (the low 11 bits of a key are its point index, so the sorted keys are the permutation and no values travel with them; the padding
// keys of j >= n are all ones and sort last).  The sort leaves the ranks striped over the threads, so the writes of perm, p0 and p1 are
// coalesced; the gather reads one cloud of at most 24 KB, which stays in L1.
#include "common.cuh"

#include <cub/block/block_radix_sort.cuh>
#include <curand_philox4x32_x.h>

namespace snb {

constexpr int kPairThreads = 256;
constexpr int kPairItems = 8;                                   // kPairThreads * kPairItems = 2048, the largest n
constexpr unsigned long long kPointBits = 0x7FFull;             // the sort key's low 11 bits hold j
constexpr unsigned long long kPadKey = ~0ull;                   // above every real key: j <= 2046 whenever a pad exists

__global__ void __launch_bounds__(kPairThreads) registration_pairs_kernel(int n, int s, const float *__restrict__ clouds,
                                                                          const int *__restrict__ records, const float *__restrict__ transforms,
                                                                          const unsigned long long *__restrict__ key, float *__restrict__ p0,
                                                                          float *__restrict__ p1, float *__restrict__ vec, int *__restrict__ perm)
{
    using Sort = cub::BlockRadixSort<unsigned long long, kPairThreads, kPairItems>;
    __shared__ typename Sort::TempStorage tmp;

    const unsigned i = blockIdx.x;
    const int r = records[i];
    const unsigned long long k0 = key[0], k1 = key[1];
    const uint2 k = make_uint2((unsigned)k0, (unsigned)(k0 >> 32));

    unsigned long long keys[kPairItems];
#pragma unroll
    for (int t = 0; t < kPairItems; ++t) {   // blocked: thread x holds j = x * 8 + t
        const unsigned j = (unsigned)(threadIdx.x * kPairItems + t);
        if ((int)j < n) {
            const uint4 w = curand_Philox4x32_10(make_uint4(i, j, (unsigned)k1, (unsigned)(k1 >> 32)), k);
            keys[t] = ((((unsigned long long)w.x << 32) | w.y) & ~kPointBits) | j;
        } else {
            keys[t] = kPadKey;
        }
    }
    Sort(tmp).SortBlockedToStriped(keys);   // striped: thread x holds ranks x + 256 t

    const float *__restrict__ src = clouds + (size_t)(r % s) * n * 3;
    const float *__restrict__ tr = transforms + (size_t)r * 7;
    const float qw = tr[0], qx = tr[1], qy = tr[2], qz = tr[3];
    const size_t base = (size_t)i * n;
#pragma unroll
    for (int t = 0; t < kPairItems; ++t) {
        const int rank = threadIdx.x + t * kPairThreads;
        if (rank >= n) break;
        const int j = (int)(keys[t] & kPointBits);
        const float vx = src[3 * j], vy = src[3 * j + 1], vz = src[3 * j + 2];
        // registration.qrot: uv = qvec x v, uuv = qvec x uv, out = v + 2 (w uv + uuv); torch.cross(a, b) = (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0)
        const float ux = __fsub_rn(__fmul_rn(qy, vz), __fmul_rn(qz, vy));
        const float uy = __fsub_rn(__fmul_rn(qz, vx), __fmul_rn(qx, vz));
        const float uz = __fsub_rn(__fmul_rn(qx, vy), __fmul_rn(qy, vx));
        const float wx = __fsub_rn(__fmul_rn(qy, uz), __fmul_rn(qz, uy));
        const float wy = __fsub_rn(__fmul_rn(qz, ux), __fmul_rn(qx, uz));
        const float wz = __fsub_rn(__fmul_rn(qx, uy), __fmul_rn(qy, ux));
        const size_t o = (base + rank) * 3;
        p0[o] = vx;
        p0[o + 1] = vy;
        p0[o + 2] = vz;
        p1[o] = __fadd_rn(vx, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(qw, ux), wx)));
        p1[o + 1] = __fadd_rn(vy, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(qw, uy), wy)));
        p1[o + 2] = __fadd_rn(vz, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(qw, uz), wz)));
        if (perm) perm[base + rank] = j;
    }
    if (threadIdx.x < 7) vec[(size_t)i * 7 + threadIdx.x] = tr[threadIdx.x];
}

int launch_registration_pairs(int b, int n, int s, const float *clouds, const int *records, const float *transforms, const unsigned long long *key,
                              float *p0, float *p1, float *vec, int *perm, cudaStream_t stream)
{
    registration_pairs_kernel<<<(unsigned)b, kPairThreads, 0, stream>>>(n, s, clouds, records, transforms, key, p0, p1, vec, perm);
    return check_launch("registration_pairs");
}

}  // namespace snb
