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

// The reconstruction trainers' augmentation (general_utils.apply_augmentations): Gaussian noise on every coordinate, then one z-rotation for
// the whole batch (include/samplenet_b200.h, snb200_ae_augment).  Same grid and stream mapping as rotate_jitter: cloud c takes the counters
// (c, 2i) and (c, 2i + 1) for point i's three normals.  The matrix's three uniforms come from the counters (0, kAngleWord) and (1, kAngleWord),
// which no point uses; every thread derives the same matrix from them (two Philox blocks, two sincos and two square roots, no barrier).
__global__ void __launch_bounds__(kAugThreads) ae_augment_kernel(int n, const float *in, float *out, const unsigned long long *__restrict__ key,
                                                                 int gauss, double mu, double sigma, int z_rotate)
{
    const unsigned cloud = blockIdx.x;
    uint2 k = make_uint2(0u, 0u);
    unsigned k1lo = 0u, k1hi = 0u;
    if (key) {
        const unsigned long long k0 = key[0], k1 = key[1];
        k = make_uint2((unsigned)k0, (unsigned)(k0 >> 32));
        k1lo = (unsigned)k1;
        k1hi = (unsigned)(k1 >> 32);
    }
    // rand_rotation_matrix() (deflection 1) with R[0,2] = R[2,0] = R[1,2] = R[2,1] = 0 and R[2,2] = 1: only the upper 2x2 block is used
    double r00 = 1.0, r01 = 0.0, r10 = 0.0, r11 = 1.0;
    if (z_rotate) {
        const uint4 wa = curand_Philox4x32_10(make_uint4(0u, kAngleWord, k1lo, k1hi), k);
        const uint4 wb = curand_Philox4x32_10(make_uint4(1u, kAngleWord, k1lo, k1hi), k);
        const double theta = uniform53(wa.x, wa.y) * 2.0 * 1.0 * kPi, phi = uniform53(wa.z, wa.w) * 2.0 * kPi, z = uniform53(wb.x, wb.y) * 2.0 * 1.0;
        const double r = sqrt(z);
        double sp, cp, st, ct;
        sincos(phi, &sp, &cp);
        sincos(theta, &st, &ct);
        const double v0 = __dmul_rn(sp, r), v1 = __dmul_rn(cp, r);
        // M = (V V^T - I) Rz with Rz = [[ct, st, 0], [-st, ct, 0], [0, 0, 1]]; the third column of V V^T - I meets Rz's zero entries
        const double a00 = __dmul_rn(v0, v0) - 1.0, a01 = __dmul_rn(v0, v1), a10 = __dmul_rn(v1, v0), a11 = __dmul_rn(v1, v1) - 1.0;
        r00 = __dadd_rn(__dmul_rn(a00, ct), __dmul_rn(a01, -st));
        r01 = __dadd_rn(__dmul_rn(a00, st), __dmul_rn(a01, ct));
        r10 = __dadd_rn(__dmul_rn(a10, ct), __dmul_rn(a11, -st));
        r11 = __dadd_rn(__dmul_rn(a10, st), __dmul_rn(a11, ct));
    }
    const float *src = in + (size_t)cloud * n * 3;
    float *dst = out + (size_t)cloud * n * 3;
    for (int i = blockIdx.y * kAugThreads + threadIdx.x; i < n; i += gridDim.y * kAugThreads) {
        float x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
        if (gauss) {   // batch += np.random.normal(mu, sigma, batch.shape): mu + sigma * normal and the sum in float64, stored as float32
            const double2 nxy = box_muller(curand_Philox4x32_10(make_uint4(cloud, 2u * (unsigned)i, k1lo, k1hi), k));
            const double nz = box_muller(curand_Philox4x32_10(make_uint4(cloud, 2u * (unsigned)i + 1u, k1lo, k1hi), k)).x;
            x = (float)__dadd_rn((double)x, __dadd_rn(mu, __dmul_rn(sigma, nxy.x)));
            y = (float)__dadd_rn((double)y, __dadd_rn(mu, __dmul_rn(sigma, nxy.y)));
            z = (float)__dadd_rn((double)z, __dadd_rn(mu, __dmul_rn(sigma, nz)));
        }
        if (z_rotate) {   // batch.dot(R) in float64, rounded to float32 when fed; z' = z exactly
            const float ox = (float)__dadd_rn(__dmul_rn((double)x, r00), __dmul_rn((double)y, r10));
            y = (float)__dadd_rn(__dmul_rn((double)x, r01), __dmul_rn((double)y, r11));
            x = ox;
        }
        dst[3 * i] = x;
        dst[3 * i + 1] = y;
        dst[3 * i + 2] = z;
    }
}

int launch_ae_augment(int b, int n, const float *in, float *out, const unsigned long long *key, int gauss, double mu, double sigma, int z_rotate,
                      cudaStream_t stream)
{
    const int tiles = (n + kAugThreads - 1) / kAugThreads;
    const dim3 grid((unsigned)b, tiles < kAugMaxTilesY ? tiles : kAugMaxTilesY);
    ae_augment_kernel<<<grid, kAugThreads, 0, stream>>>(n, in, out, gauss || z_rotate ? key : nullptr, gauss, mu, sigma, z_rotate);
    return check_launch("ae_augment");
}

}  // namespace snb
