// ref_cuda_shim.cu -- compiles the REFERENCE's own CUDA kernels, unmodified, from the reference tree (oracle/Makefile REF; nothing is
// copied into this repo) for sm_90, behind extern "C" wrappers that take raw device pointers, so that
//   * tests/golden/make_reference_cuda_golden.py can record the reference's GPU ops as a second oracle (its own kernels on identical
//     inputs, stored for tests/test_vs_reference_cuda.py), and
//   * bench.py can time "the reference on the GPU" (SURVEY.md 8d (iv), BASELINE.md row G0) next to this library.
// Output: oracle/_ref/libsamplenet_ref_cuda.so (git-ignored).  Test / measurement infrastructure, not product.
//
//   registration/src/chamfer_distance/chamfer_distance.cu        ChamferDistanceKernelLauncher (:139-155), ...GradKernelLauncher (:193-209)
//   classification/structural_losses/tf_nndistance_g.cu           NmDistanceKernelLauncher (:128), NmDistanceGradKernelLauncher (:152)
//   classification/structural_losses/tf_approxmatch_g.cu          approxmatchLauncher (:180), matchcostLauncher (:226), matchcostgradLauncher (:292)
//   classification/grouping/tf_grouping_g.cu                      selectionSortLauncher (:129), groupPointLauncher (:133), groupPointGradLauncher (:137)
//   reconstruction/external/sampling/tf_sampling_g.cu             farthestpointsamplingLauncher (:203), gatherpointLauncher (:206)
// All launchers use the legacy default stream, exactly as the reference does.
#include <cstdio>
#define GOOGLE_CUDA 1
#include "registration/src/chamfer_distance/chamfer_distance.cu"
#include "classification/structural_losses/tf_nndistance_g.cu"
#include "classification/structural_losses/tf_approxmatch_g.cu"
#include "classification/grouping/tf_grouping_g.cu"
#include "reconstruction/external/sampling/tf_sampling_g.cu"

#define REF_API extern "C" __attribute__((visibility("default")))

REF_API void refcu_chamfer_forward(int b, int n, const float *xyz1, int m, const float *xyz2, float *d1, int *i1, float *d2, int *i2)
{ ChamferDistanceKernelLauncher(b, n, xyz1, m, xyz2, d1, i1, d2, i2); }
REF_API void refcu_chamfer_backward(int b, int n, const float *xyz1, int m, const float *xyz2, const float *g1, const int *i1, const float *g2, const int *i2,
                                    float *gx1, float *gx2)
{ ChamferDistanceGradKernelLauncher(b, n, xyz1, m, xyz2, g1, i1, g2, i2, gx1, gx2); }
REF_API void refcu_nn_distance(int b, int n, const float *xyz1, int m, const float *xyz2, float *d1, int *i1, float *d2, int *i2)
{ NmDistanceKernelLauncher(b, n, xyz1, m, xyz2, d1, i1, d2, i2); }
REF_API void refcu_nn_distance_grad(int b, int n, const float *xyz1, int m, const float *xyz2, const float *g1, const int *i1, const float *g2, const int *i2,
                                    float *gx1, float *gx2)
{ NmDistanceGradKernelLauncher(b, n, xyz1, m, xyz2, g1, i1, g2, i2, gx1, gx2); }
REF_API void refcu_approxmatch(int b, int n, int m, const float *xyz1, const float *xyz2, float *match, float *temp)
{ approxmatchLauncher(b, n, m, xyz1, xyz2, match, temp); }
REF_API void refcu_matchcost(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *out)
{ matchcostLauncher(b, n, m, xyz1, xyz2, match, out); }
REF_API void refcu_matchcostgrad(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *g1, float *g2)
{ matchcostgradLauncher(b, n, m, xyz1, xyz2, match, g1, g2); }
REF_API void refcu_selection_sort(int b, int n, int m, int k, const float *dist, int *outi, float *out)
{ selectionSortLauncher(b, n, m, k, dist, outi, out); }
REF_API void refcu_group_point(int b, int n, int c, int m, int nsample, const float *points, const int *idx, float *out)
{ groupPointLauncher(b, n, c, m, nsample, points, idx, out); }
REF_API void refcu_group_point_grad(int b, int n, int c, int m, int nsample, const float *grad_out, const int *idx, float *grad_points)
{ groupPointGradLauncher(b, n, c, m, nsample, grad_out, idx, grad_points); }
REF_API void refcu_farthest_point_sampling(int b, int n, int m, const float *inp, float *temp, int *out)
{ farthestpointsamplingLauncher(b, n, m, inp, temp, out); }
REF_API void refcu_gather_point(int b, int n, int m, const float *inp, const int *idx, float *out)
{ gatherpointLauncher(b, n, m, inp, idx, out); }
