// augment.cu -- the classification trainer's training augmentation (classification/train_classifier.py:217-221: provider.rotate_point_cloud,
// then provider.jitter_point_cloud) and the evaluation votes (provider.rotate_point_cloud_by_angle), one launch for a whole batch.
//
// Contract (include/samplenet_b200.h, snb200_rotate_jitter): out[r, c] = in[c] rotated about y by the angle of (r, c), then jittered:
//   x' = x c - z s,  y' = y,  z' = x s + z c  in float64 (np.dot(pc, R) with R = [[c,0,s],[0,1,0],[-s,0,c]]), rounded to float32;
//   jitter: out = fl32(fl32(rot) + clip(sigma * z, -clip, clip)) with the normal z and the sum in float64.
// The random numbers come from Philox4x32-10 (Random123, curand's header-only curand_Philox4x32_10), one counter per (cloud, word index),
// so the stream does not depend on the launch configuration.  See the header for the mapping.
//
// Design (DESIGN.md 4.10): memory-bound, 12 bytes in and 12 out per point.  One CTA row per output cloud (grid.x = replicas * b), point tiles
// of 256 threads along grid.y with a stride loop; every thread evaluates its cloud's angle itself (one Philox block and a sincos: cheaper
// than a barrier), then one point at a time: two Philox blocks, two logs, two square roots and two sincos in float64 when jittering.
#include "common.cuh"

#include <curand_philox4x32_x.h>

namespace snb {

constexpr int kAugThreads = 256;
constexpr int kAugMaxTilesY = 4096;                     // grid.y; larger clouds take the stride loop
constexpr unsigned kAngleWord = 0xFFFFFFFFu;            // the counter's second word for a cloud's angle (point words are 2i and 2i + 1 < 2^25)
constexpr double kPi = 3.141592653589793116;            // fl64(pi)
constexpr double kTwoPi = 2.0 * kPi;                    // exact

// numpy's 53-bit uniform double from two 32-bit words (random_standard_uniform: (a >> 5) * 2^26 + (b >> 6), times 2^-53)
__device__ __forceinline__ double uniform53(unsigned wa, unsigned wb)
{
    return ((double)(wa >> 5) * 67108864.0 + (double)(wb >> 6)) * (1.0 / 9007199254740992.0);
}

// Box-Muller on (u(w0, w1), u(w2, w3)): r = sqrt(-2 log(1 - u1)), (r cos(2 pi u2), r sin(2 pi u2))
__device__ __forceinline__ double2 box_muller(uint4 w)
{
    const double u1 = uniform53(w.x, w.y), u2 = uniform53(w.z, w.w);
    const double r = sqrt(-2.0 * log(1.0 - u1));
    double s, c;
    sincos(kTwoPi * u2, &s, &c);
    return make_double2(r * c, r * s);
}

__device__ __forceinline__ double jitter(double v, double sigma, double clip)
{
    return fmin(fmax(sigma * v, -clip), clip);   // np.clip(sigma * randn, -clip, clip)
}

__global__ void __launch_bounds__(kAugThreads) rotate_jitter_kernel(int b, int n, const float *in, float *out,   // in == out in place
                                                                    const double *__restrict__ angles, const unsigned long long *__restrict__ key,
                                                                    double sigma, double clip)
{
    const unsigned cloud = blockIdx.x;   // output cloud r * b + c
    const int r = (int)(cloud / (unsigned)b), c = (int)(cloud - (unsigned)r * (unsigned)b);
    uint2 k = make_uint2(0u, 0u);
    unsigned k1lo = 0u, k1hi = 0u;
    if (key) {
        const unsigned long long k0 = key[0], k1 = key[1];
        k = make_uint2((unsigned)k0, (unsigned)(k0 >> 32));
        k1lo = (unsigned)k1;
        k1hi = (unsigned)(k1 >> 32);
    }
    double ang;
    if (angles) {
        ang = angles[r];
    } else {
        const uint4 w = curand_Philox4x32_10(make_uint4(cloud, kAngleWord, k1lo, k1hi), k);
        ang = uniform53(w.x, w.y) * 2.0 * kPi;   // np.random.uniform() * 2 * np.pi, left to right
    }
    double sn, cs;
    sincos(ang, &sn, &cs);
    const float *src = in + (size_t)c * n * 3;
    float *dst = out + (size_t)cloud * n * 3;
    for (int i = blockIdx.y * kAugThreads + threadIdx.x; i < n; i += gridDim.y * kAugThreads) {
        const double x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
        float ox = (float)(x * cs - z * sn), oy = (float)y, oz = (float)(x * sn + z * cs);
        if (sigma > 0.0) {
            const double2 nxy = box_muller(curand_Philox4x32_10(make_uint4(cloud, 2u * (unsigned)i, k1lo, k1hi), k));
            const double nz = box_muller(curand_Philox4x32_10(make_uint4(cloud, 2u * (unsigned)i + 1u, k1lo, k1hi), k)).x;
            ox = (float)((double)ox + jitter(nxy.x, sigma, clip));
            oy = (float)((double)oy + jitter(nxy.y, sigma, clip));
            oz = (float)((double)oz + jitter(nz, sigma, clip));
        }
        dst[3 * i] = ox;
        dst[3 * i + 1] = oy;
        dst[3 * i + 2] = oz;
    }
}

int launch_rotate_jitter(int b, int n, int replicas, const float *in, float *out, const double *angles, const unsigned long long *key, double sigma,
                         double clip, cudaStream_t stream)
{
    const int tiles = (n + kAugThreads - 1) / kAugThreads;
    const dim3 grid((unsigned)b * (unsigned)replicas, tiles < kAugMaxTilesY ? tiles : kAugMaxTilesY);
    rotate_jitter_kernel<<<grid, kAugThreads, 0, stream>>>(b, n, in, out, angles, sigma > 0.0 || !angles ? key : nullptr, sigma, clip);
    return check_launch("rotate_jitter");
}

}  // namespace snb
