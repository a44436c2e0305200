// pose_loss.cu -- the registration task loss behind PCRNet's last layer, one launch forward and one backward.
//
// Reference (registration/main.py:555-598 compute_pcrnet_loss, src/qdataset.py:17-119, src/quaternion.py:35-53): from the raw output
// y (b, 7) of fc6 and the two sampled clouds
//     q = y[:4] / max(|y[:4]|, 1e-12), twist = (q, y[4:])                     F.normalize
//     e_j = v_j + 2 (q_w (u x v_j) + u x (u x v_j)),  u = q[1:], v = p0        qrot: the rotation only, the translation is not applied
//     chamfer_loss = mean_i min_j |p1_i - e_j|^2 + mean_j min_i |e_j - p1_i|^2  (lowest index on ties; each mean over its own cloud)
//     qnorm_loss   = mean (|y[:4]|^2 - 1)^2
//     norm_err     = mean |R(q) R(q_gt)^T - I|_F^2, both quaternions normalised once more inside the conversion
//     rot_err      = mean 2 acos(2 (q . q_gt)^2 - 1)      (reported; it has no gradient here, as nothing differentiates it in the trainer)
//     trans_err    = mean |y[4:] - t_gt|
// The template p0 has m0 points and the source p1 m1 (equal when both clouds are sampled, 1024 against the sampled source when only the
// source is: main.py:492-496).  One CTA per pair; the per-pair sums go to the workspace and the last CTA to finish (ticket) adds them in
// pair order.  The backward recomputes q and e, gathers the Chamfer gradient per point (every point scans the other cloud's arg-mins in
// index order: nothing is scattered, no atomics), rotates it back to p0 and reduces the quaternion's gradient over the points in a fixed
// order.
#include "common.cuh"

namespace snb {

constexpr int kPoseThreads = 256;
constexpr int kPoseMaxPoints = 1024;
constexpr int kPoseMaxPairs = 256;
constexpr int kPosePart = 8;           // floats per pair in the workspace: sum c01, sum c10, qnorm, norm, rot, trans
constexpr float kPoseEps = 1e-12f;

// u = v / max(|v|, eps); returns |v|
__device__ __forceinline__ float normalize4(const float *v, float *u)
{
    const float n = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);
    const float d = fmaxf(n, kPoseEps);
#pragma unroll
    for (int k = 0; k < 4; k++) u[k] = v[k] / d;
    return n;
}
// gradient of normalize4: gu -> gv, given its output u and |v|
__device__ __forceinline__ void normalize4_grad(const float *u, float n, const float *gu, float *gv)
{
    if (n > kPoseEps) {
        const float d = u[0] * gu[0] + u[1] * gu[1] + u[2] * gu[2] + u[3] * gu[3];
#pragma unroll
        for (int k = 0; k < 4; k++) gv[k] = (gu[k] - u[k] * d) / n;
    } else {
#pragma unroll
        for (int k = 0; k < 4; k++) gv[k] = gu[k] / kPoseEps;
    }
}
__device__ __forceinline__ void cross3(const float *a, const float *b, float *c)
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}
// q = (w, x, y, z), not necessarily of unit length: the formula of qrot as it stands
__device__ __forceinline__ void qrot3(const float *q, const float *v, float *e)
{
    float uv[3], uuv[3];
    cross3(q + 1, v, uv);
    cross3(q + 1, uv, uuv);
#pragma unroll
    for (int k = 0; k < 3; k++) e[k] = v[k] + 2.f * (q[0] * uv[k] + uuv[k]);
}
// rotation matrix (row major) of the unit quaternion q = (w, x, y, z)
__device__ __forceinline__ void rotmat(const float *q, float *R)
{
    const float w = q[0], x = q[1], y = q[2], z = q[3];
    const float tx = 2.f * x, ty = 2.f * y, tz = 2.f * z;
    const float twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1.f - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1.f - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.f - (txx + tyy);
}
// gradient of rotmat: G = dL/dR -> g = dL/d(w, x, y, z)
__device__ __forceinline__ void rotmat_grad(const float *q, const float *G, float *g)
{
    const float w = q[0], x = q[1], y = q[2], z = q[3];
    g[0] = 2.f * (-z * G[1] + y * G[2] + z * G[3] - x * G[5] - y * G[6] + x * G[7]);
    g[1] = 2.f * (y * G[1] + z * G[2] + y * G[3] - 2.f * x * G[4] - w * G[5] + z * G[6] + w * G[7] - 2.f * x * G[8]);
    g[2] = 2.f * (-2.f * y * G[0] + x * G[1] + w * G[2] + x * G[3] + z * G[5] - w * G[6] + z * G[7] - 2.f * y * G[8]);
    g[3] = 2.f * (-2.f * z * G[0] - w * G[1] + x * G[2] + w * G[3] - 2.f * z * G[4] + y * G[5] + x * G[6] + y * G[7]);
}
// M = R1 R2^T - I
__device__ __forceinline__ void rel_rot_minus_eye(const float *R1, const float *R2, float *M)
{
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
            M[i * 3 + j] = R1[i * 3] * R2[j * 3] + R1[i * 3 + 1] * R2[j * 3 + 1] + R1[i * 3 + 2] * R2[j * 3 + 2] - (i == j ? 1.f : 0.f);
}

struct PoseParams {
    int b, m0, m1;
    const float *y, *p0, *p1, *igt;
    float *twist; int *idx01, *idx10;
    float *terms, *partial; unsigned *ticket;
    const float *grad_terms; float *grad_y, *grad_p0, *grad_p1;
};

// stage p1 (m1 points) and e = qrot(q, p0) (m0 points); q is the normalised quaternion
__device__ __forceinline__ void pose_stage(const float *p0, const float *p1, int m0, int m1, const float *q, float *s_p1, float *s_e)
{
    for (int j = threadIdx.x; j < max(m0, m1); j += kPoseThreads) {
        if (j < m0) {
            const float v[3] = {__ldg(p0 + j * 3), __ldg(p0 + j * 3 + 1), __ldg(p0 + j * 3 + 2)};
            float e[3];
            qrot3(q, v, e);
            s_e[j * 3] = e[0]; s_e[j * 3 + 1] = e[1]; s_e[j * 3 + 2] = e[2];
        }
        if (j < m1) { s_p1[j * 3] = __ldg(p1 + j * 3); s_p1[j * 3 + 1] = __ldg(p1 + j * 3 + 1); s_p1[j * 3 + 2] = __ldg(p1 + j * 3 + 2); }
    }
}
__device__ __forceinline__ void pose_stage(const PoseParams &P, int bi, const float *q, float *s_p1, float *s_e)
{
    pose_stage(P.p0 + (size_t)bi * P.m0 * 3, P.p1 + (size_t)bi * P.m1 * 3, P.m0, P.m1, q, s_p1, s_e);
}

// Chamfer sums of the two staged clouds: t01 = sum_i min_j |p1_i - e_j|^2, t10 = sum_j min_i |e_j - p1_i|^2 (lowest index on ties), valid in
// thread 0.  Items [0, m1): p1_i against the m0 points of e (c01 / idx01); items [m1, m1 + m0): e_j against the m1 points of p1 (c10 /
// idx10).  The arg-mins go to idx01 (m1 entries) / idx10 (m0 entries) unless they are null.  Lanes, then warps in order: one fixed
// summation order, the same item-to-thread mapping for any split of the items between the two clouds.
__device__ __forceinline__ void pose_chamfer_sums(const float *s_p1, const float *s_e, int m0, int m1, int *idx01, int *idx10, float (*s_red)[2],
                                                  float &t01, float &t10)
{
    const int tid = (int)threadIdx.x;
    float sum01 = 0.f, sum10 = 0.f;
    for (int it = tid; it < m1 + m0; it += kPoseThreads) {
        const bool back = it >= m1;
        const int i = back ? it - m1 : it, nc = back ? m1 : m0;
        const float *qs = back ? s_e : s_p1, *cs = back ? s_p1 : s_e;
        const float qx = qs[i * 3], qy = qs[i * 3 + 1], qz = qs[i * 3 + 2];
        float best = INFINITY; int besti = 0;
#pragma unroll 4
        for (int j = 0; j < nc; j++) {
            const float d = sqdist<true>(cs[j * 3] - qx, cs[j * 3 + 1] - qy, cs[j * 3 + 2] - qz);
            if (d < best) { best = d; besti = j; }
        }
        if (idx01) (back ? idx10 : idx01)[i] = besti;
        if (back) sum10 += best; else sum01 += best;
    }
    sum01 = warp_sum(sum01); sum10 = warp_sum(sum10);
    if ((tid & 31) == 0) { s_red[tid >> 5][0] = sum01; s_red[tid >> 5][1] = sum10; }
    __syncthreads();
    t01 = 0.f; t10 = 0.f;
    if (tid == 0)
        for (int w = 0; w < kPoseThreads / 32; w++) { t01 += s_red[w][0]; t10 += s_red[w][1]; }
}

// The terms of one pair that need no cloud: out = (qnorm, norm_err, rot_err in radians, sum_k |y[4+k] - t_gt[k]|); y is the raw output, q its
// normalised quaternion, gt the ground truth (w, x, y, z, t).
__device__ __forceinline__ void pose_pair_terms(const float *y, const float *q, const float *gt, float *out)
{
    float qg[4] = {__ldg(gt), __ldg(gt + 1), __ldg(gt + 2), __ldg(gt + 3)};
    const float s = y[0] * y[0] + y[1] * y[1] + y[2] * y[2] + y[3] * y[3];
    float n1[4], n2[4], R1[9], R2[9], M[9];
    normalize4(q, n1); normalize4(qg, n2);
    rotmat(n1, R1); rotmat(n2, R2);
    rel_rot_minus_eye(R1, R2, M);
    float nerr = 0.f;
#pragma unroll
    for (int k = 0; k < 9; k++) nerr += M[k] * M[k];
    const float dot = q[0] * qg[0] + q[1] * qg[1] + q[2] * qg[2] + q[3] * qg[3];
    float terr = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) { const float d = y[4 + k] - __ldg(gt + 4 + k); terr += sqrtf(d * d); }
    out[0] = (s - 1.f) * (s - 1.f); out[1] = nerr; out[2] = 2.f * acosf(2.f * dot * dot - 1.f); out[3] = terr;
}

__global__ void __launch_bounds__(kPoseThreads) pose_loss_forward_kernel(const __grid_constant__ PoseParams P)
{
    __shared__ float s_p1[kPoseMaxPoints * 3], s_e[kPoseMaxPoints * 3];
    __shared__ float s_red[kPoseThreads / 32][2];
    __shared__ unsigned s_ticket;
    const int bi = (int)blockIdx.x, tid = (int)threadIdx.x, m0 = P.m0, m1 = P.m1;
    float y[7], q[4];
#pragma unroll
    for (int k = 0; k < 7; k++) y[k] = __ldg(P.y + bi * 7 + k);
    normalize4(y, q);
    pose_stage(P, bi, q, s_p1, s_e);
    __syncthreads();
    float t01, t10;
    pose_chamfer_sums(s_p1, s_e, m0, m1, P.idx01 + (size_t)bi * m1, P.idx10 + (size_t)bi * m0, s_red, t01, t10);
    if (tid == 0) {
        float t[4];
        pose_pair_terms(y, q, P.igt + bi * 7, t);
        float *part = P.partial + (size_t)bi * kPosePart;
        part[0] = t01; part[1] = t10; part[2] = t[0]; part[3] = t[1]; part[4] = t[2]; part[5] = t[3];
#pragma unroll
        for (int k = 0; k < 7; k++) P.twist[bi * 7 + k] = k < 4 ? q[k] : y[k];
        __threadfence();
        s_ticket = atomicAdd(P.ticket, 1u);
    }
    __syncthreads();
    if (s_ticket != (unsigned)P.b - 1u) return;
    // ---- last CTA: every pair's partial is visible (each CTA fenced before taking its ticket); thread t adds column t in pair order
    __threadfence();
    if (tid < 6) {
        float t = 0.f;
        for (int p = 0; p < P.b; p++) t += __ldcg(P.partial + (size_t)p * kPosePart + tid);
        s_p1[tid] = t;
    }
    __syncthreads();
    if (tid == 0) {
        const float fb = (float)P.b;
        P.terms[0] = s_p1[0] / (fb * (float)m1) + s_p1[1] / (fb * (float)m0);
        P.terms[1] = s_p1[2] / fb;
        P.terms[2] = s_p1[3] / fb;
        P.terms[3] = s_p1[4] / fb;
        P.terms[4] = s_p1[5] / (3.f * fb);
        *P.ticket = 0u;
    }
}

__global__ void __launch_bounds__(kPoseThreads) pose_loss_backward_kernel(const __grid_constant__ PoseParams P)
{
    __shared__ float s_p1[kPoseMaxPoints * 3], s_e[kPoseMaxPoints * 3];
    __shared__ int s_i01[kPoseMaxPoints], s_i10[kPoseMaxPoints];
    __shared__ float s_red[kPoseThreads / 32][4];
    const int bi = (int)blockIdx.x, tid = (int)threadIdx.x, m0 = P.m0, m1 = P.m1;
    float y[7], q[4];
#pragma unroll
    for (int k = 0; k < 7; k++) y[k] = __ldg(P.y + bi * 7 + k);
    const float ny = normalize4(y, q);
    pose_stage(P, bi, q, s_p1, s_e);
    for (int j = tid; j < max(m0, m1); j += kPoseThreads) {     // clamped: a caller's index never addresses outside the staged clouds
        if (j < m1) s_i01[j] = min(max(__ldg(P.idx01 + (size_t)bi * m1 + j), 0), m0 - 1);
        if (j < m0) s_i10[j] = min(max(__ldg(P.idx10 + (size_t)bi * m0 + j), 0), m1 - 1);
    }
    __syncthreads();
    // d loss / d c01_i = g / (b m1), d loss / d c10_j = g / (b m0).  A point's own term is scaled by (own weight / other weight) = m_oth /
    // m_own and the sum by the other cloud's weight: with m0 == m1 the ratio is exactly 1 and the arithmetic is that of one shared weight.
    const float g_src = __ldg(P.grad_terms) / ((float)P.b * (float)m0), g_tpl = __ldg(P.grad_terms) / ((float)P.b * (float)m1);
    const float r_src = (float)m0 / (float)m1, r_tpl = (float)m1 / (float)m0;
    float gq[4] = {0.f, 0.f, 0.f, 0.f};                                    // this thread's share of d loss / d q through the rotation
    for (int it = tid; it < m1 + m0; it += kPoseThreads) {
        const bool back = it >= m1;
        const int i = back ? it - m1 : it, n_oth = back ? m1 : m0;
        const float r = back ? r_tpl : r_src, g_ch = back ? g_tpl : g_src;
        // the point's own term, then the terms of the other cloud's points whose nearest neighbour it is, in index order
        const float *own = back ? s_e : s_p1, *oth = back ? s_p1 : s_e;
        const int *own_idx = back ? s_i10 : s_i01, *oth_idx = back ? s_i01 : s_i10;
        const float x0 = own[i * 3], x1 = own[i * 3 + 1], x2 = own[i * 3 + 2];
        const int nn = own_idx[i];
        float g[3] = {r * (x0 - oth[nn * 3]), r * (x1 - oth[nn * 3 + 1]), r * (x2 - oth[nn * 3 + 2])};
        for (int j = 0; j < n_oth; j++)
            if (oth_idx[j] == i) { g[0] -= oth[j * 3] - x0; g[1] -= oth[j * 3 + 1] - x1; g[2] -= oth[j * 3 + 2] - x2; }
#pragma unroll
        for (int k = 0; k < 3; k++) g[k] *= 2.f * g_ch;
        if (!back) {
            float *dst = P.grad_p1 + ((size_t)bi * m1 + i) * 3;
            dst[0] = g[0]; dst[1] = g[1]; dst[2] = g[2];
        } else {
            // e = v + 2 (w (u x v) + u x (u x v)) is linear in v with matrix A = I + 2 w [u]x + 2 [u]x^2, so grad_v = g - 2 w (u x g) + 2 u x (u x g)
            const float *p0 = P.p0 + ((size_t)bi * m0 + i) * 3;
            const float v[3] = {__ldg(p0), __ldg(p0 + 1), __ldg(p0 + 2)};
            const float *u = q + 1;
            float ug[3], uug[3], uv[3], vg[3];
            cross3(u, g, ug); cross3(u, ug, uug); cross3(u, v, uv); cross3(v, g, vg);
            float *dst = P.grad_p0 + ((size_t)bi * m0 + i) * 3;
#pragma unroll
            for (int k = 0; k < 3; k++) dst[k] = g[k] - 2.f * q[0] * ug[k] + 2.f * uug[k];
            const float udv = u[0] * v[0] + u[1] * v[1] + u[2] * v[2], gdu = g[0] * u[0] + g[1] * u[1] + g[2] * u[2], gdv = g[0] * v[0] + g[1] * v[1] + g[2] * v[2];
            gq[0] += 2.f * (g[0] * uv[0] + g[1] * uv[1] + g[2] * uv[2]);
#pragma unroll
            for (int k = 0; k < 3; k++) gq[1 + k] += 2.f * q[0] * vg[k] + 2.f * (g[k] * udv + v[k] * gdu - 2.f * u[k] * gdv);
        }
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const float s = warp_sum(gq[k]);
        if ((tid & 31) == 0) s_red[tid >> 5][k] = s;
    }
    __syncthreads();
    if (tid != 0) return;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        float t = 0.f;
        for (int w = 0; w < kPoseThreads / 32; w++) t += s_red[w][k];
        gq[k] = t;
    }
    // norm_err = |R(n1) R(n2)^T - I|^2 / b with n1 = normalize(q): d / d R1 = 2 M R2
    const float *gt = P.igt + bi * 7;
    float qg[4] = {__ldg(gt), __ldg(gt + 1), __ldg(gt + 2), __ldg(gt + 3)};
    float n1[4], n2[4], R1[9], R2[9], M[9], G[9], gn1[4], gq2[4];
    const float nq = normalize4(q, n1);
    normalize4(qg, n2);
    rotmat(n1, R1); rotmat(n2, R2);
    rel_rot_minus_eye(R1, R2, M);
    const float g_ne = 2.f * __ldg(P.grad_terms + 2) / (float)P.b;
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) G[i * 3 + j] = g_ne * (M[i * 3] * R2[j] + M[i * 3 + 1] * R2[3 + j] + M[i * 3 + 2] * R2[6 + j]);
    rotmat_grad(n1, G, gn1);
    normalize4_grad(n1, nq, gn1, gq2);
#pragma unroll
    for (int k = 0; k < 4; k++) gq[k] += gq2[k];
    float gy[4];
    normalize4_grad(q, ny, gq, gy);
    const float s = y[0] * y[0] + y[1] * y[1] + y[2] * y[2] + y[3] * y[3];
    const float g_qn = __ldg(P.grad_terms + 1) / (float)P.b * 4.f * (s - 1.f);       // d (s - 1)^2 / d y_k = 4 (s - 1) y_k
    const float g_tr = __ldg(P.grad_terms + 4) / (3.f * (float)P.b);
#pragma unroll
    for (int k = 0; k < 4; k++) P.grad_y[bi * 7 + k] = gy[k] + g_qn * y[k];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float d = y[4 + k] - __ldg(gt + 4 + k);
        P.grad_y[bi * 7 + 4 + k] = g_tr * (d > 0.f ? 1.f : d < 0.f ? -1.f : 0.f);
    }
}

// Evaluation: the same terms per pair instead of their batch means, and the sampling consistency of the pair (main.py:540-553:
// Chamfer(p0s, qrot(conj(q_gt), p1s)), the rotation only; p0s has ms0 points and p1s ms1).  Forward only; no arg-mins are written and
// nothing is combined across CTAs.
struct PoseEvalParams {
    int m0, m1, ms0, ms1;
    const float *y, *p0, *p1, *igt, *p0s, *p1s;
    float *per_pair, *twist;
};

__global__ void __launch_bounds__(kPoseThreads) pose_eval_kernel(const __grid_constant__ PoseEvalParams P)
{
    __shared__ float s_p1[kPoseMaxPoints * 3], s_e[kPoseMaxPoints * 3];
    __shared__ float s_red[kPoseThreads / 32][2];
    const int bi = (int)blockIdx.x, tid = (int)threadIdx.x, m0 = P.m0, m1 = P.m1, ms0 = P.ms0, ms1 = P.ms1;
    float y[7], q[4];
#pragma unroll
    for (int k = 0; k < 7; k++) y[k] = __ldg(P.y + bi * 7 + k);
    normalize4(y, q);
    pose_stage(P.p0 + (size_t)bi * m0 * 3, P.p1 + (size_t)bi * m1 * 3, m0, m1, q, s_p1, s_e);
    __syncthreads();
    float t01, t10, c01 = 0.f, c10 = 0.f;
    pose_chamfer_sums(s_p1, s_e, m0, m1, nullptr, nullptr, s_red, t01, t10);
    const float *gt = P.igt + bi * 7;
    if (P.p0s) {
        const float qi[4] = {__ldg(gt), -__ldg(gt + 1), -__ldg(gt + 2), -__ldg(gt + 3)};
        __syncthreads();     // every thread is done with the staged pair and thread 0 with s_red
        // the rotated cloud is p1s (staged as e), the queries of c01 are p0s's points
        pose_stage(P.p1s + (size_t)bi * ms1 * 3, P.p0s + (size_t)bi * ms0 * 3, ms1, ms0, qi, s_p1, s_e);
        __syncthreads();
        pose_chamfer_sums(s_p1, s_e, ms1, ms0, nullptr, nullptr, s_red, c01, c10);
    }
    if (tid != 0) return;
    float t[4];
    pose_pair_terms(y, q, gt, t);
    float *out = P.per_pair + (size_t)bi * 6;
    out[0] = t01 / (float)m1 + t10 / (float)m0;
    out[1] = t[0]; out[2] = t[1]; out[3] = t[2]; out[4] = t[3] / 3.f;
    out[5] = P.p0s ? c01 / (float)ms0 + c10 / (float)ms1 : 0.f;
#pragma unroll
    for (int k = 0; k < 7; k++) P.twist[bi * 7 + k] = k < 4 ? q[k] : y[k];
}

bool pose_loss_supported(int b, int m0, int m1)
{
    return b >= 1 && b <= kPoseMaxPairs && m0 >= 1 && m0 <= kPoseMaxPoints && m1 >= 1 && m1 <= kPoseMaxPoints;
}
size_t pose_loss_workspace_bytes(int b) { return (size_t)b * kPosePart * sizeof(float); }

int launch_pose_eval(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, int ms0, int ms1, const float *p0s,
                     const float *p1s, float *per_pair, float *twist, cudaStream_t stream)
{
    const PoseEvalParams P = {m0, m1, ms0, ms1, y, p0, p1, igt, p0s, p1s, per_pair, twist};
    pose_eval_kernel<<<b, kPoseThreads, 0, stream>>>(P);
    return check_launch("pose_eval");
}

int launch_pose_loss_forward(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, float *twist, int *idx01, int *idx10,
                             float *terms, void *workspace, unsigned *ticket, cudaStream_t stream)
{
    PoseParams P;
    memset(&P, 0, sizeof(P));
    P.b = b; P.m0 = m0; P.m1 = m1; P.y = y; P.p0 = p0; P.p1 = p1; P.igt = igt; P.twist = twist; P.idx01 = idx01; P.idx10 = idx10; P.terms = terms;
    P.partial = static_cast<float *>(workspace); P.ticket = ticket;
    pose_loss_forward_kernel<<<b, kPoseThreads, 0, stream>>>(P);
    return check_launch("pose_loss_forward");
}

int launch_pose_loss_backward(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, const int *idx01, const int *idx10,
                              const float *grad_terms, float *grad_y, float *grad_p0, float *grad_p1, cudaStream_t stream)
{
    PoseParams P;
    memset(&P, 0, sizeof(P));
    P.b = b; P.m0 = m0; P.m1 = m1; P.y = y; P.p0 = p0; P.p1 = p1; P.igt = igt; P.idx01 = const_cast<int *>(idx01); P.idx10 = const_cast<int *>(idx10);
    P.grad_terms = grad_terms; P.grad_y = grad_y; P.grad_p0 = grad_p0; P.grad_p1 = grad_p1;
    pose_loss_backward_kernel<<<b, kPoseThreads, 0, stream>>>(P);
    return check_launch("pose_loss_backward");
}

}  // namespace snb
