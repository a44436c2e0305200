/* fps_oracle.c -- plain-C restatement of tf_sampling's farthest point sampling, the CPU oracle of tests/test_sampling.py (compiled by
 * the test with -ffp-contract=off, so every rounding below is the one written).  Test infrastructure, not product.
 *
 * farthestpointsamplingKernel (reconstruction/external/sampling/tf_sampling_g.cu:105-170), launched as <<<32, 512>>> (:203-205):
 *   idx[0] = 0 (:114-116), running minimum 1e38 (:118);
 *   round j (:124-168): from the last selected point s, d = (x2-x1)^2 + (y2-y1)^2 + (z2-z1)^2 (:142), which nvcc contracts to
 *   fma(dz, dz, fma(dx, dx, dy*dy)); dmin = min(d, dmin) (:143); the largest dmin wins.
 *   Ties: thread t = k mod 512 scans k = t, t+512, ... and keeps a candidate on strict '>' (:146-149); the tree keeps the lower slot
 *   unless it is strictly smaller (:153-163).  So among equal maxima the smallest (k mod 512, k div 512) wins.
 */
#include <math.h>

static int tie_before(int a, int b) /* a precedes b in the reference's thread order */
{
    if ((a & 511) != (b & 511)) return (a & 511) < (b & 511);
    return (a >> 9) < (b >> 9);
}

/* inp (b, n, 3), idx (b, m), dmin: n floats of scratch */
void fps_oracle(int b, int n, int m, const float *inp, int *idx, float *dmin)
{
    for (int i = 0; i < b; i++) {
        const float *p = inp + (long)i * n * 3;
        int *o = idx + (long)i * m;
        for (int k = 0; k < n; k++) dmin[k] = 1e38f;
        int old = 0;
        o[0] = 0;
        for (int j = 1; j < m; j++) {
            const float x1 = p[old * 3 + 0], y1 = p[old * 3 + 1], z1 = p[old * 3 + 2];
            float best = -1.0f;
            int besti = 0;
            for (int k = 0; k < n; k++) {
                const float dx = p[k * 3 + 0] - x1, dy = p[k * 3 + 1] - y1, dz = p[k * 3 + 2] - z1;
                const float d = fmaf(dz, dz, fmaf(dx, dx, dy * dy));
                const float d2 = fminf(d, dmin[k]);
                dmin[k] = d2;
                if (d2 > best || (d2 == best && tie_before(k, besti))) {
                    best = d2;
                    besti = k;
                }
            }
            old = besti;
            o[j] = old;
        }
    }
}
