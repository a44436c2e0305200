// api.cu -- the extern "C" boundary of libsamplenet_b200.so (see include/samplenet_b200.h).
// Argument validation + dispatch only; kernels live in chamfer.cu / softproj.cu / encoder.cu (CUDA-core conv stack) / generator.cu
// (pool + FC head, also of the stand-alone encoder and FC-head entries) / emd.cu / matching.cu / fps.cu.
#include "encoder_internal.cuh"
#include "../../include/samplenet_b200_debug.h"
#include <string.h>

#include <cmath>

namespace snb {

static thread_local char g_err[512] = "";
static thread_local unsigned long long g_launches = 0;

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches += (unsigned long long)n; }

// kernels (defined in the other translation units)
int launch_chamfer_forward(int b, int n, const float *xyz1, int m, const float *xyz2, float *dist1, int *idx1, float *dist2, int *idx2, int flags,
                           cudaStream_t stream);
size_t chamfer_per_cloud_workspace_bytes(int b, int n, int m);
int launch_chamfer_per_cloud(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, float *sums, void *workspace, cudaStream_t stream);
int launch_chamfer_backward(int b, int n, const float *xyz1, int m, const float *xyz2, const float *grad_dist1, const int *idx1,
                            const float *grad_dist2, const int *idx2, float *grad_xyz1, float *grad_xyz2, cudaStream_t stream);
int launch_simplification_reduce(int b, int n, int m, const float *dist1, const float *dist2, float w, float *out4, cudaStream_t stream);
int launch_knn_softproj(int b, int n, int m, int k, int layout, const float *points, const float *query, const float *sigma, int sigma_mode,
                        float sigma_floor, int hard,
                        const float *feats, int f, float *proj, float *prop, int *knn_idx, float *knn_val, float *weights,
                        float *dist_over_sigma, int flags, cudaStream_t stream);
size_t softproj_bwd_workspace(int b, int n, int m, int k, int f);
int launch_softproj_backward(int b, int n, int m, int k, int layout, const float *points, const float *query, const float *sigma,
                             int sigma_mode, float sigma_floor, const float *feats, int f, const int *knn_idx, const float *weights, const float *grad_proj,
                             const float *grad_prop, float *grad_points, float *grad_query, float *grad_feats, float *grad_sigma,
                             void *workspace, cudaStream_t stream);
int launch_group_point(int b, int n, int c, int m, int ns, int layout, const float *points, const int *idx, float *out, cudaStream_t stream);
int launch_group_point_grad(int b, int n, int c, int m, int ns, int layout, const float *grad_out, const int *idx, float *grad_points,
                            cudaStream_t stream);
size_t encoder_workspace_bytes(int b, int n, int num_layers, const snb200_layer *layers);
int launch_encoder_forward(int b, int n, int layout, const float *x, int num_layers, const snb200_layer *layers, int training, float *feat,
                           void *workspace, cudaStream_t stream);
size_t fc_head_workspace_bytes(int b, int num_layers, const snb200_layer *layers);
int launch_fc_head_forward(int b, const float *in, int num_layers, const snb200_layer *layers, int training, float *out, int out_transpose_inner,
                           void *workspace, cudaStream_t stream);
size_t approxmatch_workspace_bytes(int b, int n, int m);
int launch_approxmatch(int b, int n, int m, const float *xyz1, const float *xyz2, float *match, void *workspace, cudaStream_t stream);
int launch_approxmatch_exact(int b, int n, int m, const float *xyz1, const float *xyz2, float *match, cudaStream_t stream);
int launch_matchcost(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *cost, float *partial, cudaStream_t stream);
int launch_matchcostgrad(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *grad1, float *grad2, cudaStream_t stream);
constexpr int kEmdPerCloudMaxN = 1 << 24, kEmdPerCloudMaxM = 65520;   // emd.cu
bool emd_per_cloud_supported(int b, int n, int m);
size_t emd_per_cloud_workspace_bytes(int b, int n, int m);
int launch_emd_per_cloud(int b, int n, int m, const float *xyz1, const float *xyz2, int b2, float *cost, void *workspace, cudaStream_t stream);
int launch_emd_per_cloud_backward(int b, int n, int m, const float *xyz1, const float *xyz2, int b2, const float *grad_cost, float *grad1,
                                  float *grad2, const void *workspace, cudaStream_t stream);
int launch_nn_matching(int b, int n, int t, int k, const float *full_pc, const int *nn_idx, int complete_fps, float *out, int *out_idx,
                       cudaStream_t stream);
int launch_farthest_point_sample(int b, int n, int m, int layout, const float *inp, int *idx, float *out_points, int threads, cudaStream_t stream);
int launch_rotate_jitter(int b, int n, int replicas, const float *in, float *out, const double *angles, const unsigned long long *key, double sigma,
                         double clip, cudaStream_t stream);
int launch_ae_augment(int b, int n, const float *in, float *out, const unsigned long long *key, int gauss, double mu, double sigma, int z_rotate,
                      cudaStream_t stream);
int launch_registration_pairs(int b, int n, int s, const float *clouds, const int *records, const float *transforms, const unsigned long long *key,
                              float *p0, float *p1, float *vec, int *perm, cudaStream_t stream);
bool retrieval_metrics_supported(int q, int m, int d, int levels, int exclude);
int launch_retrieval_metrics(int q, int m, int d, const float *queries, const int *qlab, const float *db, const int *dblab, int exclude, int levels,
                             double *ap, double *prec, int *num_relevant, cudaStream_t stream);

int launch_nonfinite_guard(const snb200_guard_check *checks, int num_checks, const snb200_guard_restore *restores, int num_restores,
                           unsigned *state, int *skipped, int *skip_count, cudaStream_t stream);

int launch_tc_gemm_debug(int rows, int c_in, int c_out, const float *A, const float *W, const float *bias, float *D, cudaStream_t stream);
bool tc_layer_supported(int c_in, int c_out);
void conv_stack_partition(int b, int n, int *ppc, int *slices, int *grid, int *per_cta, int *slots);
void generator_plan_debug(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc, int flags, int *conv_path, int *fuse_head);

size_t generator_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc);
int launch_generator_forward(int b, int n, int layout, const float *x, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc,
                             int training, float *out, int out_transpose_inner, float *feat_out, int flags, void *workspace, cudaStream_t stream,
                             float *const *zsave = nullptr, const GenEx *ex = nullptr);
bool generator_backward_supported(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc);
bool generator_layers_backward_supported(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc);
size_t generator_backward_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc, bool act_input = false);
int launch_generator_backward(int b, int n, int layout, const float *x, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc,
                              float *const *zsave, void *fwd_workspace, const float *grad_out, int out_transpose_inner,
                              const snb200_layer_grad *gconv, const snb200_layer_grad *gfc, void *workspace, cudaStream_t stream,
                              const GenEx *ex = nullptr);

size_t tail_workspace_bytes(int b, int n_samp, int n_ref);
size_t progressive_workspace_bytes(int b, int n, int m, int np);
int launch_progressive_loss(int b, int n, int m, const float *ref, const float *samp, int np, const int *sizes, const float *w21, float *dist1, int *idx1,
                            float *dist2, int *idx2, float *terms, void *workspace, unsigned *ticket, int flags, cudaStream_t stream);
int launch_tail_fused(int b, int n_ref, int n_samp, int k, const float *ref, const float *samp, const float *sigma, int sigma_mode, float sigma_floor,
                      float *proj, int *knn_idx, float *weights, float *dist_over_sigma, float *dist1, int *idx1, float *dist2, int *idx2,
                      float w21, float *out4, float *partial, unsigned *ticket, int flags, cudaStream_t stream);

bool frozen_encoder_supported(int b, int n, int nconv, const snb200_layer *conv, int np);
bool frozen_encoder_ex_supported(int b, int n, int act_input, int nconv, const snb200_layer *conv, int np, int tap);
size_t frozen_encoder_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int np, int with_zsave);
size_t frozen_encoder_backward_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int np, bool params = false);
int launch_frozen_encoder_forward(int b, int n, const float *x, int nconv, const snb200_layer *conv, int np, const int *sizes, float *pooled,
                                  int *route, float *const *zsave, void *workspace, cudaStream_t stream, int act_input = 0, int tap = -1,
                                  float *tap_out = nullptr);
int launch_frozen_encoder_backward(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, const float *pooled,
                                   const int *route, float *const *zsave, const float *grad_pooled, float *grad_x, void *workspace,
                                   cudaStream_t stream, int tap = -1, const float *grad_tap = nullptr, const float *x = nullptr,
                                   const snb200_layer_grad *grads = nullptr);

bool frozen_encoder_curve_supported(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes);
size_t frozen_encoder_curve_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int np);
int launch_frozen_encoder_curve_forward(int b, int n, const float *x, int nconv, const snb200_layer *conv, int np, const int *sizes, float *pooled,
                                        int *route, void *workspace, cudaStream_t stream);

bool frozen_encoder_seg_supported(int num_seg, int total, int max_len, int act_input, int nconv, const snb200_layer *conv, int tap);
size_t frozen_encoder_seg_workspace_bytes(int total, int nconv, const snb200_layer *conv, int with_zsave);
size_t frozen_encoder_seg_backward_workspace_bytes(int total, int nconv, const snb200_layer *conv);
int launch_frozen_encoder_seg_forward(int num_seg, int total, const int2 *seg, const float *in, int nconv, const snb200_layer *conv, float *pooled,
                                      int *route, float *const *zsave, void *workspace, cudaStream_t stream, int act_input, int tap, float *tap_out);
int launch_frozen_encoder_seg_backward(int num_seg, int total, const int2 *seg, int nconv, const snb200_layer *conv, const float *pooled,
                                       const int *route, float *const *zsave, const float *grad_pooled, float *grad_in, void *workspace,
                                       cudaStream_t stream, int tap, const float *grad_tap);

bool frozen_encoder_bstat_supported(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes);
bool frozen_encoder_bstat_train_supported(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes);
size_t frozen_encoder_bstat_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes);
size_t frozen_encoder_bstat_backward_workspace_bytes(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, bool params = false);
int launch_frozen_encoder_bstat_forward(int b, int n, const float *x, int nconv, const snb200_layer *conv, int np, const int *sizes, float *pooled,
                                        int *route, double *stats, void *workspace, cudaStream_t stream);
int launch_frozen_encoder_bstat_backward(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, const float *pooled,
                                         const int *route, const double *stats, const void *fwd_workspace, const float *grad_pooled, float *grad_x,
                                         void *workspace, cudaStream_t stream, const float *x = nullptr, const snb200_layer_grad *grads = nullptr);
int launch_frozen_encoder_bstat_running_update(int b, int n, int nconv, const snb200_layer *conv, int np, const int *sizes, const double *stats,
                                               cudaStream_t stream);

bool frozen_mlp_supported(int b, int nl, const snb200_layer *layers, bool allow_bn);
size_t frozen_mlp_workspace_bytes(int b, int nl, const snb200_layer *layers, int with_save);
size_t frozen_mlp_backward_workspace_bytes(int b, int nl, const snb200_layer *layers);
int launch_frozen_mlp_forward(int b, const float *in, int nl, const snb200_layer *layers, float *out, float *const *asave, void *workspace,
                              cudaStream_t stream);
int launch_frozen_mlp_backward(int b, int nl, const snb200_layer *layers, float *const *asave, const float *grad_out, float *grad_in, void *workspace,
                               cudaStream_t stream, const float *in = nullptr, const snb200_layer_grad *grads = nullptr);

bool point_transform_supported(int b, int n, int k);
size_t point_transform_workspace_bytes(int b, int n, int k);
int launch_point_transform_forward(int b, int n, int k, const float *in, const float *T, float *out, cudaStream_t stream);
int launch_point_transform_backward(int b, int n, int k, const float *in, const float *T, const float *grad_out, float *grad_in, float *grad_T,
                                    void *workspace, cudaStream_t stream);
bool point_transform_seg_supported(int num_seg, int total, int max_len, int k);
size_t point_transform_seg_workspace_bytes(int total, int k);
int launch_point_transform_seg_forward(int num_seg, int max_len, const int2 *seg, int k, int src_b, int src_n, int np, const int *sizes,
                                       const float *in, const float *T, float *out, cudaStream_t stream);
int launch_point_transform_seg_backward(int num_seg, int max_len, const int2 *seg, int k, int src_b, int src_n, int np, const int *sizes,
                                        const float *in, const float *T, const float *grad_out, float *grad_in, float *grad_T, void *workspace,
                                        cudaStream_t stream);

bool pose_loss_supported(int b, int m0, int m1);
size_t pose_loss_workspace_bytes(int b);
int launch_pose_loss_forward(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, float *twist, int *idx01,
                             int *idx10, float *terms, void *workspace, unsigned *ticket, cudaStream_t stream);
int launch_pose_loss_backward(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, const int *idx01,
                              const int *idx10, const float *grad_terms, float *grad_y, float *grad_p0, float *grad_p1, cudaStream_t stream);
int launch_pose_eval(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, int ms0, int ms1, const float *p0s,
                     const float *p1s, float *per_pair, float *twist, cudaStream_t stream);

static int check_layers(const char *who, int num_layers, const snb200_layer *layers, int max_layers)
{
    SNB_REQUIRE(layers != nullptr && num_layers >= 1 && num_layers <= max_layers, "%s: num_layers=%d out of range [1,%d]", who, num_layers, max_layers);
    for (int l = 0; l < num_layers; l++) {
        SNB_REQUIRE(layers[l].c_in >= 1 && layers[l].c_out >= 1, "%s: layer %d has non-positive width", who, l);
        SNB_REQUIRE(layers[l].weight != nullptr, "%s: layer %d has no weight", who, l);
        SNB_REQUIRE(l == 0 || layers[l].c_in == layers[l - 1].c_out, "%s: layer %d c_in=%d does not match previous c_out=%d", who, l,
                    layers[l].c_in, layers[l - 1].c_out);
        SNB_REQUIRE((layers[l].bn_weight == nullptr) == (layers[l].bn_bias == nullptr), "%s: layer %d needs both BN weight and bias", who, l);
    }
    return SNB200_OK;
}

// The two layer tables of a generator: each well formed, and the FC head taking the conv stack's output width.
static int check_generator_tables(const char *who, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc)
{
    if (int rc = check_layers(who, nconv, conv, SNB200_MAX_CONV_LAYERS)) return rc;
    if (int rc = check_layers(who, nfc, fc, SNB200_MAX_FC_LAYERS)) return rc;
    SNB_REQUIRE(fc[0].c_in == conv[nconv - 1].c_out, "%s: FC input width %d != conv output width %d", who, fc[0].c_in, conv[nconv - 1].c_out);
    return SNB200_OK;
}

// BatchNorm of one layer table: eval mode reads the running statistics, and BatchNorm over the batch rows (`over_batch`: the FC layers)
// needs more than one row in training mode.
static int check_batchnorm(const char *who, const char *what, int num_layers, const snb200_layer *layers, int training, bool over_batch, int b)
{
    for (int l = 0; l < num_layers; l++) {
        SNB_REQUIRE(training || !layers[l].bn_weight || (layers[l].bn_running_mean && layers[l].bn_running_var),
                    "%s: eval mode needs running statistics (%s layer %d)", who, what, l);
        SNB_REQUIRE(!(training && over_batch && layers[l].bn_weight && b < 2), "%s: training-mode BatchNorm needs more than 1 row (%s layer %d)", who, what, l);
    }
    return SNB200_OK;
}

static int check_workspace(const char *who, const void *workspace, size_t have, size_t need)
{
    if (!workspace) set_error("%s: workspace is null (%zu bytes needed)", who, need);
    else if (have < need) set_error("%s: workspace %zu < %zu bytes", who, have, need);
    else return SNB200_OK;
    return SNB200_EWORKSPACE;
}

}  // namespace snb

using namespace snb;

#define SNB_API extern "C" __attribute__((visibility("default")))

SNB_API const char *snb200_last_error(void) { return g_err; }
SNB_API int snb200_version(void) { return 100; }
SNB_API unsigned long long snb200_launch_count(void) { return g_launches; }

SNB_API int snb200_nn_distance_forward(int b, int n, const float *xyz1, int m, const float *xyz2, float *dist1, int *idx1, float *dist2, int *idx2,
                                       int flags, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1, "nn_distance_forward: bad sizes b=%d n=%d m=%d", b, n, m);
    SNB_REQUIRE(b <= 65535, "nn_distance_forward: batch %d exceeds the grid limit 65535", b);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(xyz1 && xyz2 && dist1 && idx1 && dist2 && idx2, "nn_distance_forward: null pointer");
    return launch_chamfer_forward(b, n, xyz1, m, xyz2, dist1, idx1, dist2, idx2, flags, (cudaStream_t)stream);
}

SNB_API int snb200_nn_distance_backward(int b, int n, const float *xyz1, int m, const float *xyz2, const float *grad_dist1, const int *idx1,
                                        const float *grad_dist2, const int *idx2, float *grad_xyz1, float *grad_xyz2, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1 && b <= 65535, "nn_distance_backward: bad sizes b=%d n=%d m=%d", b, n, m);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(xyz1 && xyz2 && grad_dist1 && idx1 && grad_dist2 && idx2 && grad_xyz1 && grad_xyz2, "nn_distance_backward: null pointer");
    return launch_chamfer_backward(b, n, xyz1, m, xyz2, grad_dist1, idx1, grad_dist2, idx2, grad_xyz1, grad_xyz2, (cudaStream_t)stream);
}

SNB_API size_t snb200_simplification_loss_workspace_bytes(int, int, int) { return 0; }

SNB_API int snb200_simplification_loss_forward(int b, int n, const float *samp, int m, const float *ref, float weight21, float *dist1, int *idx1,
                                               float *dist2, int *idx2, float *out4, void *, size_t, int flags, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 1 && n >= 1 && m >= 1 && b <= 65535, "simplification_loss_forward: bad sizes b=%d n=%d m=%d", b, n, m);
    SNB_REQUIRE(samp && ref && dist1 && idx1 && dist2 && idx2 && out4, "simplification_loss_forward: null pointer");
    int rc = launch_chamfer_forward(b, n, samp, m, ref, dist1, idx1, dist2, idx2, flags, (cudaStream_t)stream);
    if (rc) return rc;
    return launch_simplification_reduce(b, n, m, dist1, dist2, weight21, out4, (cudaStream_t)stream);
}

SNB_API int snb200_knn_soft_project_forward(int b, int n, int m, int k, int layout, const float *points, const float *query, const float *sigma,
                                            int sigma_mode, float sigma_floor, int hard, const float *feats, int f, float *proj, float *prop, int *knn_idx, float *knn_val,
                                            float *weights, float *dist_over_sigma, int flags, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1 && b <= 65535, "knn_soft_project_forward: bad sizes b=%d n=%d m=%d", b, n, m);
    SNB_REQUIRE(k >= 1 && k <= 32, "knn_soft_project_forward: group size k=%d outside the supported range [1,32]", k);
    SNB_REQUIRE(k <= n, "knn_soft_project_forward: k=%d exceeds the number of points n=%d", k, n);
    SNB_REQUIRE(layout == SNB200_BNC || layout == SNB200_BCN, "knn_soft_project_forward: unknown layout %d", layout);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(points && query, "knn_soft_project_forward: null input");
    const bool needs_sigma = proj || prop || weights || dist_over_sigma;
    SNB_REQUIRE(!needs_sigma || sigma, "knn_soft_project_forward: sigma is required for projection outputs");
    SNB_REQUIRE(sigma_mode >= 0 && sigma_mode <= 3, "knn_soft_project_forward: unknown sigma_mode %d", sigma_mode);
    SNB_REQUIRE(!prop || (feats && f >= 1), "knn_soft_project_forward: prop requested without features");
    return launch_knn_softproj(b, n, m, k, layout, points, query, sigma, sigma_mode, sigma_floor, hard, feats, f, proj, prop, knn_idx, knn_val, weights, dist_over_sigma,
                               flags, (cudaStream_t)stream);
}

SNB_API size_t snb200_soft_project_backward_workspace_bytes(int b, int n, int m, int k, int f) { return softproj_bwd_workspace(b, n, m, k, f); }

SNB_API int snb200_soft_project_backward(int b, int n, int m, int k, int layout, const float *points, const float *query, const float *sigma,
                                         int sigma_mode, float sigma_floor, const float *feats, int f, const int *knn_idx, const float *weights, const float *grad_proj,
                                         const float *grad_prop, float *grad_points, float *grad_query, float *grad_feats, float *grad_sigma,
                                         void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 1 && n >= 1 && m >= 1 && k >= 1 && k <= 32 && b <= 65535, "soft_project_backward: bad sizes b=%d n=%d m=%d k=%d", b, n, m, k);
    SNB_REQUIRE(layout == SNB200_BNC || layout == SNB200_BCN, "soft_project_backward: unknown layout %d", layout);
    SNB_REQUIRE(points && query && sigma && knn_idx && weights, "soft_project_backward: null input");
    SNB_REQUIRE(grad_proj || grad_prop, "soft_project_backward: no upstream gradient");
    SNB_REQUIRE(!grad_prop || (feats && f >= 1), "soft_project_backward: grad_prop without features");
    if (int rc = check_workspace("soft_project_backward", workspace, workspace_bytes, softproj_bwd_workspace(b, n, m, k, f))) return rc;
    return launch_softproj_backward(b, n, m, k, layout, points, query, sigma, sigma_mode, sigma_floor, feats, f, knn_idx, weights, grad_proj, grad_prop, grad_points,
                                    grad_query, grad_feats, grad_sigma, workspace, (cudaStream_t)stream);
}

SNB_API size_t snb200_project_and_loss_workspace_bytes(int b, int n_samp, int n_ref)
{
    if (b < 1 || n_samp < 1 || n_ref < 1) return 0;
    return tail_workspace_bytes(b, n_samp, n_ref);
}

SNB_API int snb200_project_and_loss_forward(int b, int n_ref, int n_samp, int k, const float *ref, const float *samp, const float *sigma,
                                            int sigma_mode, float sigma_floor, float *proj, int *knn_idx, float *weights, float *dist_over_sigma,
                                            float *dist1, int *idx1, float *dist2, int *idx2, float weight21, float *out4, void *workspace,
                                            size_t workspace_bytes, unsigned *ticket, int flags, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 1 && b <= 65535 && n_ref >= 1 && n_samp >= 1, "project_and_loss_forward: bad sizes b=%d n_ref=%d n_samp=%d", b, n_ref, n_samp);
    SNB_REQUIRE(n_ref <= 4096 && n_samp <= 4096, "project_and_loss_forward: clouds above 4096 points need the separate entry points (n_ref=%d n_samp=%d)", n_ref, n_samp);
    SNB_REQUIRE(k >= 1 && k <= 32 && k <= n_ref, "project_and_loss_forward: group size k=%d outside [1, min(32, n_ref)]", k);
    SNB_REQUIRE(sigma_mode >= 0 && sigma_mode <= 3, "project_and_loss_forward: unknown sigma_mode %d", sigma_mode);
    SNB_REQUIRE(ref && samp && sigma && proj && knn_idx && weights && dist1 && idx1 && dist2 && idx2 && out4 && ticket, "project_and_loss_forward: null pointer");
    if (int rc = check_workspace("project_and_loss_forward", workspace, workspace_bytes, tail_workspace_bytes(b, n_samp, n_ref))) return rc;
    return launch_tail_fused(b, n_ref, n_samp, k, ref, samp, sigma, sigma_mode, sigma_floor, proj, knn_idx, weights, dist_over_sigma, dist1, idx1, dist2,
                             idx2, weight21, out4, reinterpret_cast<float *>(workspace), ticket, flags, (cudaStream_t)stream);
}

SNB_API int snb200_group_point(int b, int n, int c, int m, int ns, int layout, const float *points, const int *idx, float *out, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && c >= 1 && m >= 1 && ns >= 1, "group_point: bad sizes");
    SNB_REQUIRE(layout == SNB200_BNC || layout == SNB200_BCN, "group_point: unknown layout %d", layout);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(points && idx && out, "group_point: null pointer");
    return launch_group_point(b, n, c, m, ns, layout, points, idx, out, (cudaStream_t)stream);
}

SNB_API int snb200_group_point_grad(int b, int n, int c, int m, int ns, int layout, const float *grad_out, const int *idx, float *grad_points,
                                    snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && c >= 1 && m >= 1 && ns >= 1 && b <= 65535, "group_point_grad: bad sizes");
    SNB_REQUIRE(layout == SNB200_BNC || layout == SNB200_BCN, "group_point_grad: unknown layout %d", layout);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(grad_out && idx && grad_points, "group_point_grad: null pointer");
    return launch_group_point_grad(b, n, c, m, ns, layout, grad_out, idx, grad_points, (cudaStream_t)stream);
}

SNB_API size_t snb200_encoder_workspace_bytes(int b, int n, int num_layers, const snb200_layer *layers)
{
    if (check_layers("encoder_workspace_bytes", num_layers, layers, SNB200_MAX_CONV_LAYERS) || b < 1 || n < 1) return 0;
    return encoder_workspace_bytes(b, n, num_layers, layers);
}

SNB_API int snb200_encoder_forward(int b, int n, int layout, const float *x, int num_layers, const snb200_layer *layers, int training, float *feat,
                                   void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    if (int rc = check_layers("encoder_forward", num_layers, layers, SNB200_MAX_CONV_LAYERS)) return rc;
    SNB_REQUIRE(b >= 1 && n >= 1, "encoder_forward: bad sizes b=%d n=%d", b, n);
    SNB_REQUIRE(layout == SNB200_BNC || layout == SNB200_BCN, "encoder_forward: unknown layout %d", layout);
    SNB_REQUIRE(layers[0].c_in == 3, "encoder_forward: first layer must take 3 input channels, got %d", layers[0].c_in);
    SNB_REQUIRE(x && feat, "encoder_forward: null pointer");
    if (int rc = check_batchnorm("encoder_forward", "conv", num_layers, layers, training, false, b)) return rc;
    if (int rc = check_workspace("encoder_forward", workspace, workspace_bytes, encoder_workspace_bytes(b, n, num_layers, layers))) return rc;
    return launch_encoder_forward(b, n, layout, x, num_layers, layers, training, feat, workspace, (cudaStream_t)stream);
}

SNB_API size_t snb200_generator_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc)
{
    if (check_generator_tables("generator_workspace_bytes", num_conv, conv, num_fc, fc) || b < 1 || n < 1) return 0;
    return generator_workspace_bytes(b, n, num_conv, conv, num_fc, fc);
}

SNB_API int snb200_generator_forward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                                     const snb200_layer *fc, int training, float *out, int out_transpose_inner, float *feat, int flags,
                                     void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    if (int rc = check_generator_tables("generator_forward", num_conv, conv, num_fc, fc)) return rc;
    SNB_REQUIRE(b >= 1 && b <= 256 && n >= 1, "generator_forward: bad sizes b=%d (1..256) n=%d", b, n);
    SNB_REQUIRE(layout == SNB200_BNC || layout == SNB200_BCN, "generator_forward: unknown layout %d", layout);
    SNB_REQUIRE(conv[0].c_in == 3, "generator_forward: first layer must take 3 input channels, got %d", conv[0].c_in);
    SNB_REQUIRE(x && out, "generator_forward: null pointer");
    SNB_REQUIRE(out_transpose_inner >= 0 && (out_transpose_inner == 0 || fc[num_fc - 1].c_out % out_transpose_inner == 0),
                "generator_forward: out_transpose_inner=%d does not divide the output width %d", out_transpose_inner, fc[num_fc - 1].c_out);
    if (int rc = check_batchnorm("generator_forward", "conv", num_conv, conv, training, false, b)) return rc;
    if (int rc = check_batchnorm("generator_forward", "fc", num_fc, fc, training, true, b)) return rc;
    if (int rc = check_workspace("generator_forward", workspace, workspace_bytes, generator_workspace_bytes(b, n, num_conv, conv, num_fc, fc))) return rc;
    return launch_generator_forward(b, n, layout, x, num_conv, conv, num_fc, fc, training, out, out_transpose_inner, feat, flags, workspace,
                                    (cudaStream_t)stream);
}

SNB_API int snb200_generator_backward_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc)
{
    if (check_generator_tables("generator_backward_supported", num_conv, conv, num_fc, fc) || b < 1 || n < 1) return 0;
    return generator_backward_supported(b, n, num_conv, conv, num_fc, fc) ? 1 : 0;
}

// The two training routes, fused (the persistent conv-stack kernel) and per-layer (tensor-core layer kernels, for the shapes the persistent
// kernel does not take), keep every conv layer's raw output for the same backward kernels and check their calls alike.
struct TrainRoute {
    const char *train_forward, *backward;                                                               // entry names: the messages' prefix
    bool (*supported)(int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc);   // the route's envelope
    int accepted_flags, forced_flags;                                                                   // of the training forward
};
static const TrainRoute kFused = {"generator_train_forward", "generator_backward", generator_backward_supported,
                                  ~(SNB200_GEN_EXACT_FP32 | SNB200_GEN_PER_LAYER_KERNELS | SNB200_GEN_SEPARATE_HEAD | SNB200_GEN_PROFILE_SKIP_CONV |
                                    SNB200_GEN_PROFILE_SKIP_HEAD), 0};
static const TrainRoute kLayers = {"generator_layers_train_forward", "generator_layers_backward", generator_layers_backward_supported,
                                   SNB200_GEN_WORKSPACE_PRIMED, SNB200_GEN_PER_LAYER_KERNELS};

// The route's envelope; with the extended entries' additions (ex != nullptr) that of snb200_generator_layers_ex_supported, answered with
// SNB200_EUNSUPPORTED instead of SNB200_EINVAL.
static int check_train_envelope(const TrainRoute &r, const char *who, int b, int n, int num_conv, const snb200_layer *conv, int num_fc,
                                const snb200_layer *fc, const GenEx *ex)
{
    if (ex ? generator_layers_ex_supported(b, n, ex->act_input, num_conv, conv, num_fc, fc, ex->tap, ex->fc_dropout)
           : r.supported(b, n, num_conv, conv, num_fc, fc))
        return SNB200_OK;
    set_error("%s: shape outside the envelope of this route's CUDA backward (b=%d n=%d)", who, b, n);
    return ex ? SNB200_EUNSUPPORTED : SNB200_EINVAL;
}

static int train_forward_checked(const TrainRoute &r, int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                                 const snb200_layer *fc, float *out, int out_transpose_inner, float *feat, float *const *zsave, int flags,
                                 void *workspace, size_t workspace_bytes, snb200_stream_t stream, const GenEx *ex = nullptr)
{
    const char *who = r.train_forward;
    SNB_REQUIRE(zsave != nullptr, "%s: zsave is null", who);
    if (int rc = check_generator_tables(who, num_conv, conv, num_fc, fc)) return rc;
    SNB_REQUIRE(b >= 1 && n >= 1 && x && out, "%s: bad arguments", who);
    SNB_REQUIRE(layout == SNB200_BNC || layout == SNB200_BCN, "%s: unknown layout %d", who, layout);
    SNB_REQUIRE(out_transpose_inner >= 0 && (out_transpose_inner == 0 || fc[num_fc - 1].c_out % out_transpose_inner == 0),
                "%s: out_transpose_inner=%d does not divide the output width %d", who, out_transpose_inner, fc[num_fc - 1].c_out);
    if (int rc = check_train_envelope(r, who, b, n, num_conv, conv, num_fc, fc, ex)) return rc;
    SNB_REQUIRE(!(flags & ~r.accepted_flags), "%s: flags 0x%x select a path that does not keep activations", who, flags);
    for (int l = 0; l < num_conv; l++) SNB_REQUIRE(zsave[l] != nullptr, "%s: zsave[%d] is null", who, l);
    if (ex) {
        SNB_REQUIRE(!ex->act_input || ((uintptr_t)x & 15) == 0, "%s: the activation input must be 16-byte aligned", who);
        SNB_REQUIRE(ex->tap < 0 || (ex->tap_out && ((uintptr_t)ex->tap_out & 15) == 0), "%s: tap_out must be a 16-byte aligned buffer", who);
    }
    if (int rc = check_workspace(who, workspace, workspace_bytes, generator_workspace_bytes(b, n, num_conv, conv, num_fc, fc))) return rc;
    return launch_generator_forward(b, n, layout, x, num_conv, conv, num_fc, fc, 1, out, out_transpose_inner, feat, flags | r.forced_flags, workspace,
                                    (cudaStream_t)stream, zsave, ex);
}

static int backward_checked(const TrainRoute &r, int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                            const snb200_layer *fc, float *const *zsave, void *forward_workspace, const float *grad_out, int out_transpose_inner,
                            const snb200_layer_grad *conv_grads, const snb200_layer_grad *fc_grads, void *workspace, size_t workspace_bytes, snb200_stream_t stream,
                            const GenEx *ex = nullptr)
{
    const char *who = r.backward;
    if (int rc = check_generator_tables(who, num_conv, conv, num_fc, fc)) return rc;
    SNB_REQUIRE(x && zsave && forward_workspace && grad_out && conv_grads && fc_grads, "%s: null pointer", who);
    SNB_REQUIRE(layout == SNB200_BNC || layout == SNB200_BCN, "%s: unknown layout %d", who, layout);
    SNB_REQUIRE(out_transpose_inner >= 0 && (out_transpose_inner == 0 || fc[num_fc - 1].c_out % out_transpose_inner == 0),
                "%s: out_transpose_inner=%d does not divide the output width %d", who, out_transpose_inner, fc[num_fc - 1].c_out);
    if (int rc = check_train_envelope(r, who, b, n, num_conv, conv, num_fc, fc, ex)) return rc;
    for (int l = 0; l < num_conv; l++) SNB_REQUIRE(zsave[l] != nullptr, "%s: zsave[%d] is null", who, l);
    const bool act_input = ex && ex->act_input;
    if (ex) {
        SNB_REQUIRE(!ex->grad_tap || (ex->tap >= 0 && ((uintptr_t)ex->grad_tap & 15) == 0), "%s: grad_tap needs a tap and 16-byte alignment", who);
        SNB_REQUIRE(!act_input || (((uintptr_t)x & 15) == 0 && ((uintptr_t)ex->grad_in & 15) == 0),
                    "%s: the activation input and its gradient must be 16-byte aligned", who);
    }
    if (int rc = check_workspace(who, workspace, workspace_bytes, generator_backward_workspace_bytes(b, n, num_conv, conv, num_fc, fc, act_input)))
        return rc;
    return launch_generator_backward(b, n, layout, x, num_conv, conv, num_fc, fc, zsave, forward_workspace, grad_out, out_transpose_inner, conv_grads,
                                     fc_grads, workspace, (cudaStream_t)stream, ex);
}

SNB_API int snb200_generator_train_forward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                                           const snb200_layer *fc, float *out, int out_transpose_inner, float *feat, float *const *zsave, int flags,
                                           void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    return train_forward_checked(kFused, b, n, layout, x, num_conv, conv, num_fc, fc, out, out_transpose_inner, feat, zsave, flags, workspace, workspace_bytes, stream);
}

SNB_API size_t snb200_generator_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc)
{
    if (check_generator_tables("generator_backward_workspace_bytes", num_conv, conv, num_fc, fc) || b < 1 || n < 1) return 0;
    return generator_backward_workspace_bytes(b, n, num_conv, conv, num_fc, fc);
}

SNB_API int snb200_generator_backward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                                      const snb200_layer *fc, float *const *zsave, void *forward_workspace, const float *grad_out,
                                      int out_transpose_inner, const snb200_layer_grad *conv_grads, const snb200_layer_grad *fc_grads,
                                      void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    return backward_checked(kFused, b, n, layout, x, num_conv, conv, num_fc, fc, zsave, forward_workspace, grad_out, out_transpose_inner, conv_grads, fc_grads,
                            workspace, workspace_bytes, stream);
}

SNB_API int snb200_generator_layers_backward_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc)
{
    if (check_generator_tables("generator_layers_backward_supported", num_conv, conv, num_fc, fc) || b < 1 || n < 1) return 0;
    return generator_layers_backward_supported(b, n, num_conv, conv, num_fc, fc) ? 1 : 0;
}

SNB_API int snb200_generator_layers_train_forward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                                                  const snb200_layer *fc, float *out, int out_transpose_inner, float *feat, float *const *zsave,
                                                  int flags, void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    return train_forward_checked(kLayers, b, n, layout, x, num_conv, conv, num_fc, fc, out, out_transpose_inner, feat, zsave, flags, workspace, workspace_bytes, stream);
}

SNB_API size_t snb200_generator_layers_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc)
{
    return snb200_generator_backward_workspace_bytes(b, n, num_conv, conv, num_fc, fc);
}

SNB_API int snb200_generator_layers_backward(int b, int n, int layout, const float *x, int num_conv, const snb200_layer *conv, int num_fc,
                                             const snb200_layer *fc, float *const *zsave, void *forward_workspace, const float *grad_out,
                                             int out_transpose_inner, const snb200_layer_grad *conv_grads, const snb200_layer_grad *fc_grads,
                                             void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    return backward_checked(kLayers, b, n, layout, x, num_conv, conv, num_fc, fc, zsave, forward_workspace, grad_out, out_transpose_inner, conv_grads, fc_grads,
                            workspace, workspace_bytes, stream);
}

// The extended entries' additions, checked before anything launches.
static int make_gen_ex(const char *who, int num_fc, int act_input, int tap, float *tap_out, const float *const *fc_dropout, const float *grad_tap,
                       float *grad_in, GenEx &ex)
{
    SNB_REQUIRE(act_input == 0 || act_input == 1, "%s: act_input must be 0 or 1, got %d", who, act_input);
    SNB_REQUIRE(num_fc >= 1 && num_fc <= SNB200_MAX_FC_LAYERS, "%s: num_fc=%d out of range", who, num_fc);
    memset(&ex, 0, sizeof(ex));
    ex.act_input = act_input; ex.tap = tap; ex.tap_out = tap_out; ex.grad_tap = grad_tap; ex.grad_in = grad_in;
    for (int l = 0; l < num_fc; l++) ex.fc_dropout[l] = fc_dropout ? fc_dropout[l] : nullptr;
    return SNB200_OK;
}

SNB_API int snb200_generator_layers_ex_supported(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc,
                                                 int tap, const float *const *fc_dropout)
{
    if (check_generator_tables("generator_layers_ex_supported", num_conv, conv, num_fc, fc) || b < 1 || n < 1 || (act_input != 0 && act_input != 1)) return 0;
    return generator_layers_ex_supported(b, n, act_input, num_conv, conv, num_fc, fc, tap, fc_dropout) ? 1 : 0;
}

SNB_API int snb200_generator_layers_ex_train_forward(int b, int n, int layout, int act_input, const float *in, int num_conv, const snb200_layer *conv,
                                                     int num_fc, const snb200_layer *fc, int tap, float *tap_out, const float *const *fc_dropout,
                                                     float *out, int out_transpose_inner, float *feat, float *const *zsave, int flags,
                                                     void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    GenEx ex;
    if (int rc = make_gen_ex("generator_layers_ex_train_forward", num_fc, act_input, tap, tap_out, fc_dropout, nullptr, nullptr, ex)) return rc;
    TrainRoute r = kLayers;
    r.train_forward = "generator_layers_ex_train_forward";
    return train_forward_checked(r, b, n, layout, in, num_conv, conv, num_fc, fc, out, out_transpose_inner, feat, zsave, flags, workspace,
                                 workspace_bytes, stream, &ex);
}

SNB_API size_t snb200_generator_layers_ex_backward_workspace_bytes(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_fc,
                                                                   const snb200_layer *fc)
{
    if (check_generator_tables("generator_layers_ex_backward_workspace_bytes", num_conv, conv, num_fc, fc) || b < 1 || n < 1) return 0;
    return generator_backward_workspace_bytes(b, n, num_conv, conv, num_fc, fc, act_input != 0);
}

SNB_API int snb200_generator_layers_ex_backward(int b, int n, int layout, int act_input, const float *in, int num_conv, const snb200_layer *conv,
                                                int num_fc, const snb200_layer *fc, int tap, const float *const *fc_dropout, float *const *zsave,
                                                void *forward_workspace, const float *grad_out, int out_transpose_inner, const float *grad_tap,
                                                float *grad_in, const snb200_layer_grad *conv_grads, const snb200_layer_grad *fc_grads,
                                                void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    GenEx ex;
    if (int rc = make_gen_ex("generator_layers_ex_backward", num_fc, act_input, tap, nullptr, fc_dropout, grad_tap, grad_in, ex)) return rc;
    TrainRoute r = kLayers;
    r.backward = "generator_layers_ex_backward";
    return backward_checked(r, b, n, layout, in, num_conv, conv, num_fc, fc, zsave, forward_workspace, grad_out, out_transpose_inner, conv_grads,
                            fc_grads, workspace, workspace_bytes, stream, &ex);
}

SNB_API int snb200_debug_tc_gemm(int rows, int c_in, int c_out, const float *A, const float *W, const float *bias, float *D,
                                 snb200_stream_t stream)
{
    SNB_REQUIRE(rows >= 1 && tc_layer_supported(c_in, c_out), "debug_tc_gemm: unsupported shape rows=%d c_in=%d c_out=%d", rows, c_in, c_out);
    SNB_REQUIRE(A && W && bias && D, "debug_tc_gemm: null pointer");
    return launch_tc_gemm_debug(rows, c_in, c_out, A, W, bias, D, (cudaStream_t)stream);
}

SNB_API size_t snb200_fc_head_workspace_bytes(int b, int num_layers, const snb200_layer *layers)
{
    if (check_layers("fc_head_workspace_bytes", num_layers, layers, SNB200_MAX_FC_LAYERS) || b < 1) return 0;
    return fc_head_workspace_bytes(b, num_layers, layers);
}

SNB_API int snb200_fc_head_forward(int b, const float *in, int num_layers, const snb200_layer *layers, int training, float *out,
                                   int out_transpose_inner, void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    if (int rc = check_layers("fc_head_forward", num_layers, layers, SNB200_MAX_FC_LAYERS)) return rc;
    SNB_REQUIRE(b >= 1 && b <= 256, "fc_head_forward: batch %d outside the supported range [1,256]", b);
    SNB_REQUIRE(in && out, "fc_head_forward: null pointer");
    SNB_REQUIRE(out_transpose_inner >= 0 && (out_transpose_inner == 0 || layers[num_layers - 1].c_out % out_transpose_inner == 0),
                "fc_head_forward: out_transpose_inner=%d does not divide the output width %d", out_transpose_inner, layers[num_layers - 1].c_out);
    if (int rc = check_batchnorm("fc_head_forward", "fc", num_layers, layers, training, true, b)) return rc;
    if (int rc = check_workspace("fc_head_forward", workspace, workspace_bytes, fc_head_workspace_bytes(b, num_layers, layers))) return rc;
    return launch_fc_head_forward(b, in, num_layers, layers, training, out, out_transpose_inner, workspace, (cudaStream_t)stream);
}

SNB_API size_t snb200_progressive_loss_workspace_bytes(int b, int n, int m, int num_prefix) { return progressive_workspace_bytes(b, n, m, num_prefix); }

SNB_API int snb200_progressive_loss_forward(int b, int n, int m, const float *ref, const float *samp, int num_prefix, const int *sizes, const float *weights,
                                            float *dist1, int *idx1, float *dist2, int *idx2, float *terms, void *workspace, size_t workspace_bytes,
                                            unsigned *ticket, int flags, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 1 && n >= 1 && m >= 1, "progressive_loss: bad sizes b=%d n=%d m=%d", b, n, m);
    SNB_REQUIRE(num_prefix >= 1 && num_prefix <= 16 && sizes && weights, "progressive_loss: 1..16 prefixes expected, got %d", num_prefix);
    SNB_REQUIRE(m <= 4096, "progressive_loss: at most 4096 ordered samples (one shared-memory tile), got %d", m);
    for (int p = 0; p < num_prefix; p++)
        SNB_REQUIRE(sizes[p] >= 1 && sizes[p] <= m && (p == 0 || sizes[p] > sizes[p - 1]), "progressive_loss: prefix sizes must be ascending in [1, m]");
    SNB_REQUIRE(ref && samp && dist1 && idx1 && dist2 && idx2 && terms && ticket, "progressive_loss: null pointer");
    if (int rc = check_workspace("progressive_loss", workspace, workspace_bytes, progressive_workspace_bytes(b, n, m, num_prefix))) return rc;
    return launch_progressive_loss(b, n, m, ref, samp, num_prefix, sizes, weights, dist1, idx1, dist2, idx2, terms, workspace, ticket, flags, (cudaStream_t)stream);
}

// Parameter gradients of layers without BatchNorm: no BatchNorm gradient pointers, weight gradients 16-byte aligned like the weights.
static int check_layer_grads(const char *who, int num_layers, const snb200_layer_grad *grads)
{
    for (int l = 0; l < num_layers; l++) {
        SNB_REQUIRE(!grads[l].bn_weight && !grads[l].bn_bias, "%s: layer %d has no BatchNorm: its bn_weight / bn_bias gradients must be NULL", who, l);
        SNB_REQUIRE(((uintptr_t)grads[l].weight & 15) == 0, "%s: layer %d's weight gradient must be 16-byte aligned", who, l);
    }
    return SNB200_OK;
}

// The frozen encoder over prefixes (frozen_encoder.cu): argument checks shared by the forward and the backward, before anything launches.
// The extended entries (act_input, tap) answer a shape outside the envelope with SNB200_EUNSUPPORTED, the original ones with SNB200_EINVAL.
static int check_frozen_encoder(const char *who, int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                bool ex = false, int act_input = 0, int tap = -1)
{
    if (int rc = check_layers(who, num_conv, conv, SNB200_MAX_CONV_LAYERS)) return rc;
    SNB_REQUIRE(num_prefix >= 1 && num_prefix <= 16, "%s: 1..16 prefixes expected, got %d", who, num_prefix);
    SNB_REQUIRE(sizes != nullptr, "%s: sizes is null", who);
    SNB_REQUIRE(b >= 1 && n >= 1, "%s: bad sizes b=%d n=%d", who, b, n);
    for (int p = 0; p < num_prefix; p++)
        SNB_REQUIRE(sizes[p] >= 1 && sizes[p] <= n && (p == 0 || sizes[p] > sizes[p - 1]), "%s: prefix sizes must be ascending in [1, n=%d]", who, n);
    if (int rc = check_batchnorm(who, "conv", num_conv, conv, 0, false, b)) return rc;
    if (!frozen_encoder_ex_supported(b, n, act_input, num_conv, conv, num_prefix, tap)) {
        set_error("%s: shape outside the frozen encoder's envelope (b=%d n=%d, %d conv layers)", who, b, n, num_conv);
        return ex ? SNB200_EUNSUPPORTED : SNB200_EINVAL;
    }
    return SNB200_OK;
}

SNB_API int snb200_frozen_encoder_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix)
{
    if (check_layers("frozen_encoder_supported", num_conv, conv, SNB200_MAX_CONV_LAYERS)) return 0;
    return frozen_encoder_supported(b, n, num_conv, conv, num_prefix) ? 1 : 0;
}

SNB_API size_t snb200_frozen_encoder_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, int with_zsave)
{
    if (!snb200_frozen_encoder_supported(b, n, num_conv, conv, num_prefix)) return 0;
    return frozen_encoder_workspace_bytes(b, n, num_conv, conv, num_prefix, with_zsave);
}

SNB_API size_t snb200_frozen_encoder_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix)
{
    if (!snb200_frozen_encoder_supported(b, n, num_conv, conv, num_prefix)) return 0;
    return frozen_encoder_backward_workspace_bytes(b, n, num_conv, conv, num_prefix);
}

SNB_API int snb200_frozen_encoder_forward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                          float *pooled, int *route, float *const *zsave, void *workspace, size_t workspace_bytes,
                                          snb200_stream_t stream)
{
    if (int rc = check_frozen_encoder("frozen_encoder_forward", b, n, num_conv, conv, num_prefix, sizes)) return rc;
    SNB_REQUIRE(x && pooled && route, "frozen_encoder_forward: null pointer");
    if (zsave)
        for (int l = 0; l < num_conv - 1; l++) SNB_REQUIRE(zsave[l] != nullptr, "frozen_encoder_forward: zsave[%d] is null", l);
    if (int rc = check_workspace("frozen_encoder_forward", workspace, workspace_bytes,
                                 frozen_encoder_workspace_bytes(b, n, num_conv, conv, num_prefix, zsave != nullptr)))
        return rc;
    return launch_frozen_encoder_forward(b, n, x, num_conv, conv, num_prefix, sizes, pooled, route, zsave, workspace, (cudaStream_t)stream);
}

// The backward with and without parameter gradients (conv_grads NULL: the original entry, gradient to x only, x required).
static int encoder_backward_checked(const char *who, int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix,
                                    const int *sizes, const float *pooled, const int *route, float *const *zsave, const float *grad_pooled,
                                    float *grad_x, const snb200_layer_grad *conv_grads, void *workspace, size_t workspace_bytes,
                                    snb200_stream_t stream)
{
    if (conv_grads) {
        if (int rc = check_layers(who, num_conv, conv, SNB200_MAX_CONV_LAYERS)) return rc;
        if (!snb200_frozen_encoder_param_backward_supported(b, n, num_conv, conv, num_prefix)) {
            set_error("%s: shape outside the envelope of the frozen encoder's parameter backward (b=%d n=%d, %d conv layers, no BatchNorm)", who, b,
                      n, num_conv);
            return SNB200_EUNSUPPORTED;
        }
        if (int rc = check_layer_grads(who, num_conv, conv_grads)) return rc;
    }
    if (int rc = check_frozen_encoder(who, b, n, num_conv, conv, num_prefix, sizes, conv_grads != nullptr)) return rc;
    SNB_REQUIRE(x && pooled && route && zsave && grad_pooled && (grad_x || conv_grads), "%s: null pointer", who);
    for (int l = 0; l < num_conv - 1; l++) SNB_REQUIRE(zsave[l] != nullptr, "%s: zsave[%d] is null", who, l);
    if (int rc = check_workspace(who, workspace, workspace_bytes,
                                 frozen_encoder_backward_workspace_bytes(b, n, num_conv, conv, num_prefix, conv_grads != nullptr)))
        return rc;
    return launch_frozen_encoder_backward(b, n, num_conv, conv, num_prefix, sizes, pooled, route, zsave, grad_pooled, grad_x, workspace,
                                          (cudaStream_t)stream, -1, nullptr, x, conv_grads);
}

SNB_API int snb200_frozen_encoder_backward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                           const float *pooled, const int *route, float *const *zsave, const float *grad_pooled, float *grad_x,
                                           void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    return encoder_backward_checked("frozen_encoder_backward", b, n, x, num_conv, conv, num_prefix, sizes, pooled, route, zsave, grad_pooled, grad_x,
                                    nullptr, workspace, workspace_bytes, stream);
}

// The frozen encoder's backward with weight and bias gradients, for conv stacks without BatchNorm (PCRNet's encoder trained).
SNB_API int snb200_frozen_encoder_param_backward_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix)
{
    if (check_layers("frozen_encoder_param_backward_supported", num_conv, conv, SNB200_MAX_CONV_LAYERS)) return 0;
    for (int l = 0; l < num_conv; l++)
        if (conv[l].bn_weight || conv[l].bn_bias) return 0;
    return frozen_encoder_supported(b, n, num_conv, conv, num_prefix) ? 1 : 0;
}

SNB_API size_t snb200_frozen_encoder_param_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix)
{
    if (!snb200_frozen_encoder_param_backward_supported(b, n, num_conv, conv, num_prefix)) return 0;
    return frozen_encoder_backward_workspace_bytes(b, n, num_conv, conv, num_prefix, true);
}

SNB_API int snb200_frozen_encoder_param_backward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix,
                                                 const int *sizes, const float *pooled, const int *route, float *const *zsave,
                                                 const float *grad_pooled, float *grad_x, const snb200_layer_grad *conv_grads, void *workspace,
                                                 size_t workspace_bytes, snb200_stream_t stream)
{
    const char *who = "frozen_encoder_param_backward";
    SNB_REQUIRE(conv_grads != nullptr, "%s: conv_grads is null", who);
    return encoder_backward_checked(who, b, n, x, num_conv, conv, num_prefix, sizes, pooled, route, zsave, grad_pooled, grad_x, conv_grads,
                                    workspace, workspace_bytes, stream);
}

// The frozen encoder with an activation input and a tapped hidden layer (frozen_encoder.cu, the same kernels).
SNB_API int snb200_frozen_encoder_ex_supported(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_prefix, int tap)
{
    if (check_layers("frozen_encoder_ex_supported", num_conv, conv, SNB200_MAX_CONV_LAYERS)) return 0;
    return frozen_encoder_ex_supported(b, n, act_input, num_conv, conv, num_prefix, tap) ? 1 : 0;
}

SNB_API size_t snb200_frozen_encoder_ex_workspace_bytes(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_prefix, int tap,
                                                        int with_zsave)
{
    if (!snb200_frozen_encoder_ex_supported(b, n, act_input, num_conv, conv, num_prefix, tap)) return 0;
    return frozen_encoder_workspace_bytes(b, n, num_conv, conv, num_prefix, with_zsave);
}

SNB_API size_t snb200_frozen_encoder_ex_backward_workspace_bytes(int b, int n, int act_input, int num_conv, const snb200_layer *conv, int num_prefix,
                                                                 int tap)
{
    if (!snb200_frozen_encoder_ex_supported(b, n, act_input, num_conv, conv, num_prefix, tap)) return 0;
    return frozen_encoder_backward_workspace_bytes(b, n, num_conv, conv, num_prefix);
}

SNB_API int snb200_frozen_encoder_ex_forward(int b, int n, int act_input, const float *in, int num_conv, const snb200_layer *conv, int num_prefix,
                                             const int *sizes, float *pooled, int *route, int tap, float *tap_out, float *const *zsave,
                                             void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    const char *who = "frozen_encoder_ex_forward";
    if (int rc = check_frozen_encoder(who, b, n, num_conv, conv, num_prefix, sizes, true, act_input, tap)) return rc;
    SNB_REQUIRE(in && pooled && route && (tap < 0 || tap_out), "%s: null pointer", who);
    SNB_REQUIRE(!act_input || ((uintptr_t)in & 15) == 0, "%s: an activation input must be 16-byte aligned", who);
    SNB_REQUIRE(tap < 0 || ((uintptr_t)tap_out & 15) == 0, "%s: tap_out must be 16-byte aligned", who);
    if (zsave)
        for (int l = 0; l < num_conv - 1; l++) SNB_REQUIRE(zsave[l] != nullptr, "%s: zsave[%d] is null", who, l);
    if (int rc = check_workspace(who, workspace, workspace_bytes, frozen_encoder_workspace_bytes(b, n, num_conv, conv, num_prefix, zsave != nullptr)))
        return rc;
    return launch_frozen_encoder_forward(b, n, in, num_conv, conv, num_prefix, sizes, pooled, route, zsave, workspace, (cudaStream_t)stream, act_input,
                                         tap, tap >= 0 ? tap_out : nullptr);
}

SNB_API int snb200_frozen_encoder_ex_backward(int b, int n, int act_input, const float *in, int num_conv, const snb200_layer *conv, int num_prefix,
                                              const int *sizes, const float *pooled, const int *route, float *const *zsave, int tap,
                                              const float *grad_tap, const float *grad_pooled, float *grad_in, void *workspace,
                                              size_t workspace_bytes, snb200_stream_t stream)
{
    const char *who = "frozen_encoder_ex_backward";
    if (int rc = check_frozen_encoder(who, b, n, num_conv, conv, num_prefix, sizes, true, act_input, tap)) return rc;
    SNB_REQUIRE(in && pooled && route && zsave && grad_pooled && grad_in && (tap < 0 || grad_tap), "%s: null pointer", who);
    for (int l = 0; l < num_conv - 1; l++) SNB_REQUIRE(zsave[l] != nullptr, "%s: zsave[%d] is null", who, l);
    if (int rc = check_workspace(who, workspace, workspace_bytes, frozen_encoder_backward_workspace_bytes(b, n, num_conv, conv, num_prefix)))
        return rc;
    return launch_frozen_encoder_backward(b, n, num_conv, conv, num_prefix, sizes, pooled, route, zsave, grad_pooled, grad_in, workspace,
                                          (cudaStream_t)stream, tap, tap >= 0 ? grad_tap : nullptr);
}

// The frozen encoder's forward over many prefixes (frozen_encoder.cu, the same layer kernels).  Sizes are checked on the host before
// anything launches: bad sizes are SNB200_EINVAL, a shape outside the envelope SNB200_EUNSUPPORTED.
SNB_API int snb200_frozen_encoder_curve_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_sizes, const int *sizes)
{
    if (check_layers("frozen_encoder_curve_supported", num_conv, conv, SNB200_MAX_CONV_LAYERS)) return 0;
    return frozen_encoder_curve_supported(b, n, num_conv, conv, num_sizes, sizes) ? 1 : 0;
}

SNB_API size_t snb200_frozen_encoder_curve_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_sizes, const int *sizes)
{
    if (!snb200_frozen_encoder_curve_supported(b, n, num_conv, conv, num_sizes, sizes)) return 0;
    return frozen_encoder_curve_workspace_bytes(b, n, num_conv, conv, num_sizes);
}

SNB_API int snb200_frozen_encoder_curve_forward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_sizes, const int *sizes,
                                                float *pooled, int *route, void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    const char *who = "frozen_encoder_curve_forward";
    if (int rc = check_layers(who, num_conv, conv, SNB200_MAX_CONV_LAYERS)) return rc;
    SNB_REQUIRE(b >= 1 && n >= 1, "%s: bad sizes b=%d n=%d", who, b, n);
    SNB_REQUIRE(sizes != nullptr && num_sizes >= 1 && num_sizes <= n, "%s: 1..n=%d sizes expected, got %d", who, n, num_sizes);
    for (int p = 0; p < num_sizes; p++)
        SNB_REQUIRE(sizes[p] >= 1 && sizes[p] <= n && (p == 0 || sizes[p] > sizes[p - 1]), "%s: sizes must be ascending and distinct in [1, n=%d]",
                    who, n);
    if (int rc = check_batchnorm(who, "conv", num_conv, conv, 0, false, b)) return rc;
    if (!frozen_encoder_curve_supported(b, n, num_conv, conv, num_sizes, sizes)) {
        set_error("%s: shape outside the frozen encoder's envelope (b=%d n=%d, %d conv layers)", who, b, n, num_conv);
        return SNB200_EUNSUPPORTED;
    }
    SNB_REQUIRE(x && pooled && route, "%s: null pointer", who);
    if (int rc = check_workspace(who, workspace, workspace_bytes, frozen_encoder_curve_workspace_bytes(b, n, num_conv, conv, num_sizes))) return rc;
    return launch_frozen_encoder_curve_forward(b, n, x, num_conv, conv, num_sizes, sizes, pooled, route, workspace, (cudaStream_t)stream);
}

// The frozen encoder over the segments of a packed buffer (frozen_encoder.cu, the same kernels).  The segment table is the caller's (device
// memory); everything checked here is on the host, before anything launches.
static int check_frozen_encoder_seg(const char *who, int num_seg, int total, int max_len, const int *seg, int act_input, int num_conv,
                                    const snb200_layer *conv, int tap)
{
    if (int rc = check_layers(who, num_conv, conv, SNB200_MAX_CONV_LAYERS)) return rc;
    if (int rc = check_batchnorm(who, "conv", num_conv, conv, 0, false, 1)) return rc;
    if (!frozen_encoder_seg_supported(num_seg, total, max_len, act_input, num_conv, conv, tap)) {
        set_error("%s: outside the segmented frozen encoder's envelope (%d segments of at most %d rows in %d rows, %d conv layers, tap %d): "
                  "1..ceil(total/128) segments, total <= 2^22, max_len <= 4096, the layer table of snb200_frozen_encoder_ex_supported", who,
                  num_seg, max_len, total, num_conv, tap);
        return SNB200_EUNSUPPORTED;
    }
    SNB_REQUIRE(seg && ((uintptr_t)seg & 7) == 0, "%s: the segment table must be a non-null, 8-byte aligned (num_seg, 2) int32 array", who);
    return SNB200_OK;
}

SNB_API int snb200_frozen_encoder_seg_supported(int num_seg, int total, int max_len, int act_input, int num_conv, const snb200_layer *conv, int tap)
{
    if (check_layers("frozen_encoder_seg_supported", num_conv, conv, SNB200_MAX_CONV_LAYERS)) return 0;
    return frozen_encoder_seg_supported(num_seg, total, max_len, act_input, num_conv, conv, tap) ? 1 : 0;
}

SNB_API size_t snb200_frozen_encoder_seg_workspace_bytes(int num_seg, int total, int max_len, int act_input, int num_conv, const snb200_layer *conv,
                                                         int tap, int with_zsave)
{
    if (!snb200_frozen_encoder_seg_supported(num_seg, total, max_len, act_input, num_conv, conv, tap)) return 0;
    return frozen_encoder_seg_workspace_bytes(total, num_conv, conv, with_zsave);
}

SNB_API size_t snb200_frozen_encoder_seg_backward_workspace_bytes(int num_seg, int total, int max_len, int act_input, int num_conv,
                                                                  const snb200_layer *conv, int tap)
{
    if (!snb200_frozen_encoder_seg_supported(num_seg, total, max_len, act_input, num_conv, conv, tap)) return 0;
    return frozen_encoder_seg_backward_workspace_bytes(total, num_conv, conv);
}

SNB_API int snb200_frozen_encoder_seg_forward(int num_seg, int total, int max_len, const int *seg, int act_input, const float *in, int num_conv,
                                              const snb200_layer *conv, float *pooled, int *route, int tap, float *tap_out, float *const *zsave,
                                              void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    const char *who = "frozen_encoder_seg_forward";
    if (int rc = check_frozen_encoder_seg(who, num_seg, total, max_len, seg, act_input, num_conv, conv, tap)) return rc;
    SNB_REQUIRE(in && pooled && route && (tap < 0 || tap_out), "%s: null pointer", who);
    SNB_REQUIRE(!act_input || ((uintptr_t)in & 15) == 0, "%s: an activation input must be 16-byte aligned", who);
    SNB_REQUIRE(tap < 0 || ((uintptr_t)tap_out & 15) == 0, "%s: tap_out must be 16-byte aligned", who);
    if (zsave)
        for (int l = 0; l < num_conv - 1; l++) SNB_REQUIRE(zsave[l] != nullptr, "%s: zsave[%d] is null", who, l);
    if (int rc = check_workspace(who, workspace, workspace_bytes, frozen_encoder_seg_workspace_bytes(total, num_conv, conv, zsave != nullptr)))
        return rc;
    return launch_frozen_encoder_seg_forward(num_seg, total, reinterpret_cast<const int2 *>(seg), in, num_conv, conv, pooled, route, zsave, workspace,
                                             (cudaStream_t)stream, act_input, tap, tap >= 0 ? tap_out : nullptr);
}

SNB_API int snb200_frozen_encoder_seg_backward(int num_seg, int total, int max_len, const int *seg, int act_input, const float *in, int num_conv,
                                               const snb200_layer *conv, const float *pooled, const int *route, float *const *zsave, int tap,
                                               const float *grad_tap, const float *grad_pooled, float *grad_in, void *workspace,
                                               size_t workspace_bytes, snb200_stream_t stream)
{
    const char *who = "frozen_encoder_seg_backward";
    if (int rc = check_frozen_encoder_seg(who, num_seg, total, max_len, seg, act_input, num_conv, conv, tap)) return rc;
    SNB_REQUIRE(in && pooled && route && zsave && grad_pooled && grad_in && (tap < 0 || grad_tap), "%s: null pointer", who);
    for (int l = 0; l < num_conv - 1; l++) SNB_REQUIRE(zsave[l] != nullptr, "%s: zsave[%d] is null", who, l);
    if (int rc = check_workspace(who, workspace, workspace_bytes, frozen_encoder_seg_backward_workspace_bytes(total, num_conv, conv))) return rc;
    return launch_frozen_encoder_seg_backward(num_seg, total, reinterpret_cast<const int2 *>(seg), num_conv, conv, pooled, route, zsave, grad_pooled,
                                              grad_in, workspace, (cudaStream_t)stream, tap, tap >= 0 ? grad_tap : nullptr);
}

// The frozen encoder with batch statistics per prefix (frozen_encoder_bstat.cu).  A malformed layer table is SNB200_EINVAL; a well-formed
// call outside the envelope is SNB200_EUNSUPPORTED.  Everything is decided on the host, before anything launches.
// train: the entries of the autoencoder trained with the sampler, whose envelope adds b * sizes[0] >= 2 (an unbiased variance).
static int check_frozen_encoder_bstat(const char *who, int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                      bool train = false)
{
    if (int rc = check_layers(who, num_conv, conv, SNB200_MAX_CONV_LAYERS)) return rc;
    if (!(train ? frozen_encoder_bstat_train_supported : frozen_encoder_bstat_supported)(b, n, num_conv, conv, num_prefix, sizes)) {
        set_error("%s: outside the batch-statistics encoder's envelope (b=%d n=%d, %d prefixes, %d conv layers): 1..16 ascending distinct sizes "
                  "in [1, n], n <= 4096, b * sum(pad128(size)) <= 2^22 rows, the frozen encoder's layer table with BatchNorm, bias and ReLU on "
                  "every layer%s", who, b, n, num_prefix, num_conv, train ? ", b * size >= 2 for every prefix" : "");
        return SNB200_EUNSUPPORTED;
    }
    return SNB200_OK;
}

SNB_API int snb200_frozen_encoder_bstat_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes)
{
    if (check_layers("frozen_encoder_bstat_supported", num_conv, conv, SNB200_MAX_CONV_LAYERS)) return 0;
    return frozen_encoder_bstat_supported(b, n, num_conv, conv, num_prefix, sizes) ? 1 : 0;
}

SNB_API size_t snb200_frozen_encoder_bstat_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes)
{
    if (!snb200_frozen_encoder_bstat_supported(b, n, num_conv, conv, num_prefix, sizes)) return 0;
    return frozen_encoder_bstat_workspace_bytes(b, n, num_conv, conv, num_prefix, sizes);
}

SNB_API size_t snb200_frozen_encoder_bstat_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix,
                                                                    const int *sizes)
{
    if (!snb200_frozen_encoder_bstat_supported(b, n, num_conv, conv, num_prefix, sizes)) return 0;
    return frozen_encoder_bstat_backward_workspace_bytes(b, n, num_conv, conv, num_prefix, sizes);
}

SNB_API int snb200_frozen_encoder_bstat_forward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix,
                                                const int *sizes, float *pooled, int *route, double *stats, void *workspace, size_t workspace_bytes,
                                                snb200_stream_t stream)
{
    const char *who = "frozen_encoder_bstat_forward";
    if (int rc = check_frozen_encoder_bstat(who, b, n, num_conv, conv, num_prefix, sizes)) return rc;
    SNB_REQUIRE(x && pooled && route && stats, "%s: null pointer", who);
    if (int rc = check_workspace(who, workspace, workspace_bytes, frozen_encoder_bstat_workspace_bytes(b, n, num_conv, conv, num_prefix, sizes)))
        return rc;
    return launch_frozen_encoder_bstat_forward(b, n, x, num_conv, conv, num_prefix, sizes, pooled, route, stats, workspace, (cudaStream_t)stream);
}

SNB_API int snb200_frozen_encoder_bstat_backward(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                                 const float *pooled, const int *route, const double *stats, const void *fwd_workspace,
                                                 size_t fwd_workspace_bytes, const float *grad_pooled, float *grad_x, void *workspace,
                                                 size_t workspace_bytes, snb200_stream_t stream)
{
    const char *who = "frozen_encoder_bstat_backward";
    if (int rc = check_frozen_encoder_bstat(who, b, n, num_conv, conv, num_prefix, sizes)) return rc;
    SNB_REQUIRE(pooled && route && stats && grad_pooled && grad_x, "%s: null pointer", who);
    if (int rc = check_workspace(who, fwd_workspace, fwd_workspace_bytes, frozen_encoder_bstat_workspace_bytes(b, n, num_conv, conv, num_prefix, sizes)))
        return rc;
    if (int rc = check_workspace(who, workspace, workspace_bytes,
                                 frozen_encoder_bstat_backward_workspace_bytes(b, n, num_conv, conv, num_prefix, sizes)))
        return rc;
    return launch_frozen_encoder_bstat_backward(b, n, num_conv, conv, num_prefix, sizes, pooled, route, stats, fwd_workspace, grad_pooled, grad_x,
                                                workspace, (cudaStream_t)stream);
}

// The batch-statistics encoder trained (the autoencoder fine-tuned with the sampler): parameter gradients and the running statistics.
SNB_API int snb200_frozen_encoder_bstat_param_backward_supported(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix,
                                                                 const int *sizes)
{
    if (check_layers("frozen_encoder_bstat_param_backward_supported", num_conv, conv, SNB200_MAX_CONV_LAYERS)) return 0;
    return frozen_encoder_bstat_train_supported(b, n, num_conv, conv, num_prefix, sizes) ? 1 : 0;
}

SNB_API size_t snb200_frozen_encoder_bstat_param_backward_workspace_bytes(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix,
                                                                          const int *sizes)
{
    if (!snb200_frozen_encoder_bstat_param_backward_supported(b, n, num_conv, conv, num_prefix, sizes)) return 0;
    return frozen_encoder_bstat_backward_workspace_bytes(b, n, num_conv, conv, num_prefix, sizes, true);
}

SNB_API int snb200_frozen_encoder_bstat_param_backward(int b, int n, const float *x, int num_conv, const snb200_layer *conv, int num_prefix,
                                                       const int *sizes, const float *pooled, const int *route, const double *stats,
                                                       const void *fwd_workspace, size_t fwd_workspace_bytes, const float *grad_pooled, float *grad_x,
                                                       const snb200_layer_grad *conv_grads, void *workspace, size_t workspace_bytes,
                                                       snb200_stream_t stream)
{
    const char *who = "frozen_encoder_bstat_param_backward";
    if (int rc = check_frozen_encoder_bstat(who, b, n, num_conv, conv, num_prefix, sizes, true)) return rc;
    SNB_REQUIRE(x && pooled && route && stats && grad_pooled && conv_grads, "%s: null pointer", who);
    if (int rc = check_workspace(who, fwd_workspace, fwd_workspace_bytes, frozen_encoder_bstat_workspace_bytes(b, n, num_conv, conv, num_prefix, sizes)))
        return rc;
    if (int rc = check_workspace(who, workspace, workspace_bytes,
                                 frozen_encoder_bstat_backward_workspace_bytes(b, n, num_conv, conv, num_prefix, sizes, true)))
        return rc;
    return launch_frozen_encoder_bstat_backward(b, n, num_conv, conv, num_prefix, sizes, pooled, route, stats, fwd_workspace, grad_pooled, grad_x,
                                                workspace, (cudaStream_t)stream, x, conv_grads);
}

SNB_API int snb200_frozen_encoder_bstat_running_update(int b, int n, int num_conv, const snb200_layer *conv, int num_prefix, const int *sizes,
                                                       const double *stats, snb200_stream_t stream)
{
    const char *who = "frozen_encoder_bstat_running_update";
    if (int rc = check_frozen_encoder_bstat(who, b, n, num_conv, conv, num_prefix, sizes, true)) return rc;
    SNB_REQUIRE(stats, "%s: null pointer", who);
    return launch_frozen_encoder_bstat_running_update(b, n, num_conv, conv, num_prefix, sizes, stats, (cudaStream_t)stream);
}

// The frozen MLP head (frozen_mlp.cu).  Anything outside the envelope is SNB200_EUNSUPPORTED, decided on the host: nothing launches.
// allow_bn: the snb200_frozen_mlp_bn_* entries, which take eval-mode BatchNorm (running statistics required) on any layer.
static int check_frozen_mlp(const char *who, int b, int num_layers, const snb200_layer *layers, bool allow_bn = false)
{
    if (!frozen_mlp_supported(b, num_layers, layers, allow_bn)) {
        set_error("%s: outside the frozen MLP's envelope (b=%d, %d layers): 1 <= b <= 64, 1..%d layers %s, c_in a multiple of 8 up to "
                  "4096, c_out 1..4096, no ReLU on the last layer", who, b, num_layers, SNB200_MAX_FC_LAYERS,
                  allow_bn ? "with or without BatchNorm" : "without BatchNorm");
        return SNB200_EUNSUPPORTED;
    }
    if (allow_bn)
        if (int rc = check_batchnorm(who, "fc", num_layers, layers, 0, true, b)) return rc;
    for (int l = 0; l < num_layers; l++)
        SNB_REQUIRE(layers[l].weight && ((uintptr_t)layers[l].weight & 15) == 0, "%s: layer %d needs a 16-byte aligned weight", who, l);
    return SNB200_OK;
}

static int mlp_forward_checked(const char *who, bool allow_bn, int b, const float *in, int num_layers, const snb200_layer *layers, float *out,
                               float *const *asave, void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    if (int rc = check_frozen_mlp(who, b, num_layers, layers, allow_bn)) return rc;
    SNB_REQUIRE(in && out, "%s: null pointer", who);
    SNB_REQUIRE(((uintptr_t)in & 15) == 0, "%s: `in` must be 16-byte aligned", who);
    if (asave)
        for (int l = 0; l < num_layers - 1; l++)
            SNB_REQUIRE(asave[l] && ((uintptr_t)asave[l] & 15) == 0, "%s: asave[%d] is null or not 16-byte aligned", who, l);
    const size_t need = frozen_mlp_workspace_bytes(b, num_layers, layers, asave != nullptr);
    if (need)
        if (int rc = check_workspace(who, workspace, workspace_bytes, need)) return rc;
    return launch_frozen_mlp_forward(b, in, num_layers, layers, out, asave, workspace, (cudaStream_t)stream);
}

// grads NULL: the input gradient only (grad_in required); otherwise grad_in may be NULL, and `in` is required for a layer-1 weight gradient.
static int mlp_backward_checked(const char *who, bool allow_bn, int b, int num_layers, const snb200_layer *layers, const float *in,
                                float *const *asave, const float *grad_out, float *grad_in, const snb200_layer_grad *grads, void *workspace,
                                size_t workspace_bytes, snb200_stream_t stream)
{
    if (int rc = check_frozen_mlp(who, b, num_layers, layers, allow_bn)) return rc;
    if (grads)
        if (int rc = check_layer_grads(who, num_layers, grads)) return rc;
    SNB_REQUIRE(grad_out && (grad_in || grads) && (asave || num_layers == 1) && (in || !grads || !grads[0].weight), "%s: null pointer", who);
    for (int l = 0; l < num_layers - 1; l++) SNB_REQUIRE(asave[l] != nullptr, "%s: asave[%d] is null", who, l);
    if (int rc = check_workspace(who, workspace, workspace_bytes, frozen_mlp_backward_workspace_bytes(b, num_layers, layers))) return rc;
    return launch_frozen_mlp_backward(b, num_layers, layers, asave, grad_out, grad_in, workspace, (cudaStream_t)stream, in, grads);
}

SNB_API int snb200_frozen_mlp_supported(int b, int num_layers, const snb200_layer *layers) { return frozen_mlp_supported(b, num_layers, layers, false) ? 1 : 0; }

SNB_API size_t snb200_frozen_mlp_workspace_bytes(int b, int num_layers, const snb200_layer *layers, int with_save)
{
    return frozen_mlp_supported(b, num_layers, layers, false) ? frozen_mlp_workspace_bytes(b, num_layers, layers, with_save) : 0;
}

SNB_API size_t snb200_frozen_mlp_backward_workspace_bytes(int b, int num_layers, const snb200_layer *layers)
{
    return frozen_mlp_supported(b, num_layers, layers, false) ? frozen_mlp_backward_workspace_bytes(b, num_layers, layers) : 0;
}

SNB_API int snb200_frozen_mlp_forward(int b, const float *in, int num_layers, const snb200_layer *layers, float *out, float *const *asave,
                                      void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    return mlp_forward_checked("frozen_mlp_forward", false, b, in, num_layers, layers, out, asave, workspace, workspace_bytes, stream);
}

SNB_API int snb200_frozen_mlp_backward(int b, int num_layers, const snb200_layer *layers, float *const *asave, const float *grad_out, float *grad_in,
                                       void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    return mlp_backward_checked("frozen_mlp_backward", false, b, num_layers, layers, nullptr, asave, grad_out, grad_in, nullptr, workspace,
                                workspace_bytes, stream);
}

// The same backward with weight and bias gradients (PCRNet's head trained).
SNB_API int snb200_frozen_mlp_param_backward_supported(int b, int num_layers, const snb200_layer *layers)
{
    return frozen_mlp_supported(b, num_layers, layers, false) ? 1 : 0;
}

SNB_API size_t snb200_frozen_mlp_param_backward_workspace_bytes(int b, int num_layers, const snb200_layer *layers)
{
    return frozen_mlp_supported(b, num_layers, layers, false) ? frozen_mlp_backward_workspace_bytes(b, num_layers, layers) : 0;
}

SNB_API int snb200_frozen_mlp_param_backward(int b, int num_layers, const snb200_layer *layers, const float *in, float *const *asave,
                                             const float *grad_out, float *grad_in, const snb200_layer_grad *grads, void *workspace,
                                             size_t workspace_bytes, snb200_stream_t stream)
{
    const char *who = "frozen_mlp_param_backward";
    SNB_REQUIRE(grads != nullptr, "%s: grads is null", who);
    return mlp_backward_checked(who, false, b, num_layers, layers, in, asave, grad_out, grad_in, grads, workspace, workspace_bytes, stream);
}

// The same MLP with eval-mode BatchNorm allowed on any layer.
SNB_API int snb200_frozen_mlp_bn_supported(int b, int num_layers, const snb200_layer *layers) { return frozen_mlp_supported(b, num_layers, layers, true) ? 1 : 0; }

SNB_API size_t snb200_frozen_mlp_bn_workspace_bytes(int b, int num_layers, const snb200_layer *layers, int with_save)
{
    return frozen_mlp_supported(b, num_layers, layers, true) ? frozen_mlp_workspace_bytes(b, num_layers, layers, with_save) : 0;
}

SNB_API size_t snb200_frozen_mlp_bn_backward_workspace_bytes(int b, int num_layers, const snb200_layer *layers)
{
    return frozen_mlp_supported(b, num_layers, layers, true) ? frozen_mlp_backward_workspace_bytes(b, num_layers, layers) : 0;
}

SNB_API int snb200_frozen_mlp_bn_forward(int b, const float *in, int num_layers, const snb200_layer *layers, float *out, float *const *asave,
                                         void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    return mlp_forward_checked("frozen_mlp_bn_forward", true, b, in, num_layers, layers, out, asave, workspace, workspace_bytes, stream);
}

SNB_API int snb200_frozen_mlp_bn_backward(int b, int num_layers, const snb200_layer *layers, float *const *asave, const float *grad_out,
                                          float *grad_in, void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    return mlp_backward_checked("frozen_mlp_bn_backward", true, b, num_layers, layers, nullptr, asave, grad_out, grad_in, nullptr, workspace,
                                workspace_bytes, stream);
}

// The point transform (point_transform.cu).
static int check_point_transform(const char *who, int b, int n, int k)
{
    if (!point_transform_supported(b, n, k)) {
        set_error("%s: outside the point transform's envelope: 1 <= b <= 65535 clouds of 1 <= n <= 2^24 points, 1 <= k <= 64, got b=%d n=%d k=%d", who,
                  b, n, k);
        return SNB200_EUNSUPPORTED;
    }
    return SNB200_OK;
}

SNB_API int snb200_point_transform_supported(int b, int n, int k) { return point_transform_supported(b, n, k) ? 1 : 0; }

SNB_API size_t snb200_point_transform_workspace_bytes(int b, int n, int k) { return point_transform_supported(b, n, k) ? point_transform_workspace_bytes(b, n, k) : 0; }

SNB_API int snb200_point_transform_forward(int b, int n, int k, const float *in, const float *T, float *out, snb200_stream_t stream)
{
    if (int rc = check_point_transform("point_transform_forward", b, n, k)) return rc;
    SNB_REQUIRE(in && T && out, "point_transform_forward: null pointer");
    return launch_point_transform_forward(b, n, k, in, T, out, (cudaStream_t)stream);
}

SNB_API int snb200_point_transform_backward(int b, int n, int k, const float *in, const float *T, const float *grad_out, float *grad_in, float *grad_T,
                                            void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    if (int rc = check_point_transform("point_transform_backward", b, n, k)) return rc;
    SNB_REQUIRE(in && T && grad_out && grad_in && grad_T, "point_transform_backward: null pointer");
    const size_t need = point_transform_workspace_bytes(b, n, k);
    if (need)
        if (int rc = check_workspace("point_transform_backward", workspace, workspace_bytes, need)) return rc;
    return launch_point_transform_backward(b, n, k, in, T, grad_out, grad_in, grad_T, workspace, (cudaStream_t)stream);
}

// The point transform over the segments of a packed buffer; num_prefix > 0 reads the prefixes of an unpacked (src_b, src_n, k) input.
static int check_point_transform_seg(const char *who, int num_seg, int total, int max_len, const int *seg, int k, int src_b, int src_n, int num_prefix,
                                     const int *sizes)
{
    if (!point_transform_seg_supported(num_seg, total, max_len, k) || num_prefix < 0 || num_prefix > 16 || (num_prefix && src_b > 65535)) {
        set_error("%s: outside the segmented point transform's envelope: 1..ceil(total/128) segments of at most max_len <= 4096 rows in "
                  "total <= 2^22 rows, 1 <= k <= 64, 0..16 prefixes of at most 65535 clouds; got %d segments, total %d, max_len %d, k %d, "
                  "%d prefixes of %d clouds", who, num_seg, total, max_len, k, num_prefix, src_b);
        return SNB200_EUNSUPPORTED;
    }
    SNB_REQUIRE(seg && ((uintptr_t)seg & 7) == 0, "%s: the segment table must be a non-null, 8-byte aligned (num_seg, 2) int32 array", who);
    if (num_prefix) {
        SNB_REQUIRE(sizes && src_b >= 1 && src_n >= 1 && num_seg == num_prefix * src_b, "%s: a prefix source needs sizes and num_seg = num_prefix * src_b",
                    who);
        for (int p = 0; p < num_prefix; p++)
            SNB_REQUIRE(sizes[p] >= 1 && sizes[p] <= src_n && sizes[p] <= max_len && (p == 0 || sizes[p] > sizes[p - 1]),
                        "%s: prefix sizes must be ascending in [1, min(src_n=%d, max_len=%d)]", who, src_n, max_len);
    }
    return SNB200_OK;
}

SNB_API int snb200_point_transform_seg_supported(int num_seg, int total, int max_len, int k)
{
    return point_transform_seg_supported(num_seg, total, max_len, k) ? 1 : 0;
}

SNB_API size_t snb200_point_transform_seg_workspace_bytes(int num_seg, int total, int max_len, int k)
{
    return point_transform_seg_supported(num_seg, total, max_len, k) ? point_transform_seg_workspace_bytes(total, k) : 0;
}

SNB_API int snb200_point_transform_seg_forward(int num_seg, int total, int max_len, const int *seg, int k, int src_b, int src_n, int num_prefix,
                                               const int *sizes, const float *in, const float *T, float *out, snb200_stream_t stream)
{
    const char *who = "point_transform_seg_forward";
    if (int rc = check_point_transform_seg(who, num_seg, total, max_len, seg, k, src_b, src_n, num_prefix, sizes)) return rc;
    SNB_REQUIRE(in && T && out, "%s: null pointer", who);
    return launch_point_transform_seg_forward(num_seg, max_len, reinterpret_cast<const int2 *>(seg), k, src_b, src_n, num_prefix, sizes, in, T, out,
                                              (cudaStream_t)stream);
}

SNB_API int snb200_point_transform_seg_backward(int num_seg, int total, int max_len, const int *seg, int k, int src_b, int src_n, int num_prefix,
                                                const int *sizes, const float *in, const float *T, const float *grad_out, float *grad_in,
                                                float *grad_T, void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    const char *who = "point_transform_seg_backward";
    if (int rc = check_point_transform_seg(who, num_seg, total, max_len, seg, k, src_b, src_n, num_prefix, sizes)) return rc;
    SNB_REQUIRE(in && T && grad_out && grad_in && grad_T, "%s: null pointer", who);
    if (int rc = check_workspace(who, workspace, workspace_bytes, point_transform_seg_workspace_bytes(total, k))) return rc;
    return launch_point_transform_seg_backward(num_seg, max_len, reinterpret_cast<const int2 *>(seg), k, src_b, src_n, num_prefix, sizes, in, T,
                                               grad_out, grad_in, grad_T, workspace, (cudaStream_t)stream);
}

// The fused pose loss (pose_loss.cu).  The plain entries are the _ex entries with one point count for both clouds.
static int check_pose_loss(const char *who, int b, int m0, int m1)
{
    if (!pose_loss_supported(b, m0, m1)) {
        if (m0 == m1)
            set_error("%s: outside the pose loss's envelope: 1 <= b <= 256 pairs of 1 <= m <= 1024 points, got b=%d m=%d", who, b, m0);
        else
            set_error("%s: outside the pose loss's envelope: 1 <= b <= 256 pairs of 1 <= m0, m1 <= 1024 points, got b=%d m0=%d m1=%d", who, b, m0, m1);
        return SNB200_EUNSUPPORTED;
    }
    return SNB200_OK;
}

static int pose_loss_forward_checked(const char *who, int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt,
                                     float *twist, int *idx01, int *idx10, float *terms, void *workspace, size_t workspace_bytes, unsigned *ticket,
                                     snb200_stream_t stream)
{
    if (int rc = check_pose_loss(who, b, m0, m1)) return rc;
    SNB_REQUIRE(y && p0 && p1 && igt && twist && idx01 && idx10 && terms && ticket, "%s: null pointer", who);
    if (int rc = check_workspace(who, workspace, workspace_bytes, pose_loss_workspace_bytes(b))) return rc;
    return launch_pose_loss_forward(b, m0, m1, y, p0, p1, igt, twist, idx01, idx10, terms, workspace, ticket, (cudaStream_t)stream);
}

static int pose_loss_backward_checked(const char *who, int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt,
                                      const int *idx01, const int *idx10, const float *grad_terms, float *grad_y, float *grad_p0, float *grad_p1,
                                      snb200_stream_t stream)
{
    if (int rc = check_pose_loss(who, b, m0, m1)) return rc;
    SNB_REQUIRE(y && p0 && p1 && igt && idx01 && idx10 && grad_terms && grad_y && grad_p0 && grad_p1, "%s: null pointer", who);
    return launch_pose_loss_backward(b, m0, m1, y, p0, p1, igt, idx01, idx10, grad_terms, grad_y, grad_p0, grad_p1, (cudaStream_t)stream);
}

static int pose_eval_checked(const char *who, int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, int ms0,
                             int ms1, const float *p0s, const float *p1s, float *per_pair, float *twist, snb200_stream_t stream)
{
    const bool sampled = p0s || p1s;
    if (!pose_loss_supported(b, m0, m1) || (sampled && !pose_loss_supported(b, ms0, ms1))) {
        if (m0 == m1 && ms0 == ms1)
            set_error("%s: outside the envelope: 1 <= b <= 256 pairs of 1 <= m, ms <= 1024 points, got b=%d m=%d ms=%d", who, b, m0, ms0);
        else
            set_error("%s: outside the envelope: 1 <= b <= 256 pairs of 1 <= m0, m1, ms0, ms1 <= 1024 points, got b=%d m0=%d m1=%d ms0=%d ms1=%d",
                      who, b, m0, m1, ms0, ms1);
        return SNB200_EUNSUPPORTED;
    }
    SNB_REQUIRE(y && p0 && p1 && igt && per_pair && twist, "%s: null pointer", who);
    SNB_REQUIRE(!sampled || (p0s && p1s), "%s: the sampled pair needs both p0s and p1s", who);
    return launch_pose_eval(b, m0, m1, y, p0, p1, igt, ms0, ms1, p0s, p1s, per_pair, twist, (cudaStream_t)stream);
}

SNB_API size_t snb200_pose_loss_workspace_bytes(int b, int m) { return pose_loss_supported(b, m, m) ? pose_loss_workspace_bytes(b) : 0; }

SNB_API int snb200_pose_loss_forward(int b, int m, const float *y, const float *p0, const float *p1, const float *igt, float *twist, int *idx01,
                                     int *idx10, float *terms, void *workspace, size_t workspace_bytes, unsigned *ticket, snb200_stream_t stream)
{
    return pose_loss_forward_checked("pose_loss_forward", b, m, m, y, p0, p1, igt, twist, idx01, idx10, terms, workspace, workspace_bytes, ticket,
                                     stream);
}

SNB_API int snb200_pose_loss_backward(int b, int m, const float *y, const float *p0, const float *p1, const float *igt, const int *idx01,
                                      const int *idx10, const float *grad_terms, float *grad_y, float *grad_p0, float *grad_p1, snb200_stream_t stream)
{
    return pose_loss_backward_checked("pose_loss_backward", b, m, m, y, p0, p1, igt, idx01, idx10, grad_terms, grad_y, grad_p0, grad_p1, stream);
}

SNB_API int snb200_pose_eval_supported(int b, int m, int ms) { return pose_loss_supported(b, m, m) && pose_loss_supported(b, ms, ms) ? 1 : 0; }

SNB_API int snb200_pose_eval(int b, int m, const float *y, const float *p0, const float *p1, const float *igt, int ms, const float *p0s,
                             const float *p1s, float *per_pair, float *twist, snb200_stream_t stream)
{
    return pose_eval_checked("pose_eval", b, m, m, y, p0, p1, igt, ms, ms, p0s, p1s, per_pair, twist, stream);
}

SNB_API int snb200_pose_loss_ex_supported(int b, int m0, int m1) { return pose_loss_supported(b, m0, m1) ? 1 : 0; }

SNB_API size_t snb200_pose_loss_ex_workspace_bytes(int b, int m0, int m1) { return pose_loss_supported(b, m0, m1) ? pose_loss_workspace_bytes(b) : 0; }

SNB_API int snb200_pose_loss_ex_forward(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, float *twist,
                                        int *idx01, int *idx10, float *terms, void *workspace, size_t workspace_bytes, unsigned *ticket,
                                        snb200_stream_t stream)
{
    return pose_loss_forward_checked("pose_loss_ex_forward", b, m0, m1, y, p0, p1, igt, twist, idx01, idx10, terms, workspace, workspace_bytes,
                                     ticket, stream);
}

SNB_API int snb200_pose_loss_ex_backward(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, const int *idx01,
                                         const int *idx10, const float *grad_terms, float *grad_y, float *grad_p0, float *grad_p1,
                                         snb200_stream_t stream)
{
    return pose_loss_backward_checked("pose_loss_ex_backward", b, m0, m1, y, p0, p1, igt, idx01, idx10, grad_terms, grad_y, grad_p0, grad_p1,
                                      stream);
}

SNB_API int snb200_pose_eval_ex(int b, int m0, int m1, const float *y, const float *p0, const float *p1, const float *igt, int ms0, int ms1,
                                const float *p0s, const float *p1s, float *per_pair, float *twist, snb200_stream_t stream)
{
    return pose_eval_checked("pose_eval_ex", b, m0, m1, y, p0, p1, igt, ms0, ms1, p0s, p1s, per_pair, twist, stream);
}

SNB_API size_t snb200_chamfer_per_cloud_workspace_bytes(int b, int n, int m)
{
    return (b >= 1 && b <= 65535 && n >= 1 && m >= 1) ? chamfer_per_cloud_workspace_bytes(b, n, m) : 0;
}

SNB_API int snb200_chamfer_per_cloud(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, float *sums, void *workspace,
                                     size_t workspace_bytes, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1, "chamfer_per_cloud: bad sizes b=%d n=%d m=%d", b, n, m);
    SNB_REQUIRE(b <= 65535, "chamfer_per_cloud: batch %d exceeds the grid limit 65535", b);
    SNB_REQUIRE(b2 >= 1 && b2 <= (b > 0 ? b : 1) && b % b2 == 0, "chamfer_per_cloud: xyz2 repeats every b2=%d clouds, which must divide b=%d", b2, b);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(xyz1 && xyz2 && sums, "chamfer_per_cloud: null pointer");
    if (int rc = check_workspace("chamfer_per_cloud", workspace, workspace_bytes, chamfer_per_cloud_workspace_bytes(b, n, m))) return rc;
    return launch_chamfer_per_cloud(b, n, xyz1, m, xyz2, b2, sums, workspace, (cudaStream_t)stream);
}

SNB_API size_t snb200_approxmatch_workspace_bytes(int b, int n, int m) { return approxmatch_workspace_bytes(b, n, m); }

SNB_API int snb200_approxmatch(int b, int n, int m, const float *xyz1, const float *xyz2, float *match, void *workspace, size_t workspace_bytes,
                               snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1, "approxmatch: bad sizes b=%d n=%d m=%d", b, n, m);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(xyz1 && xyz2 && match, "approxmatch: null pointer");
    if (int rc = check_workspace("approxmatch", workspace, workspace_bytes, approxmatch_workspace_bytes(b, n, m))) return rc;
    return launch_approxmatch(b, n, m, xyz1, xyz2, match, workspace, (cudaStream_t)stream);
}

SNB_API int snb200_approxmatch_mode(int b, int n, int m, const float *xyz1, const float *xyz2, float *match, int flags, void *workspace,
                                    size_t workspace_bytes, snb200_stream_t stream)
{
    if (!(flags & SNB200_EMD_EXACT)) return snb200_approxmatch(b, n, m, xyz1, xyz2, match, workspace, workspace_bytes, stream);
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1, "approxmatch: bad sizes b=%d n=%d m=%d", b, n, m);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(xyz1 && xyz2 && match, "approxmatch: null pointer");
    return launch_approxmatch_exact(b, n, m, xyz1, xyz2, match, (cudaStream_t)stream);
}

SNB_API size_t snb200_matchcost_workspace_bytes(int b) { return (size_t)b * 16 * sizeof(float); }

SNB_API int snb200_matchcost(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *cost, void *workspace,
                             size_t workspace_bytes, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1 && b <= 65535, "matchcost: bad sizes b=%d n=%d m=%d", b, n, m);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(xyz1 && xyz2 && match && cost, "matchcost: null pointer");
    if (int rc = check_workspace("matchcost", workspace, workspace_bytes, snb200_matchcost_workspace_bytes(b))) return rc;
    return launch_matchcost(b, n, m, xyz1, xyz2, match, cost, reinterpret_cast<float *>(workspace), (cudaStream_t)stream);
}

SNB_API int snb200_matchcostgrad(int b, int n, int m, const float *xyz1, const float *xyz2, const float *match, float *grad1, float *grad2,
                                 snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1 && b <= 65535, "matchcostgrad: bad sizes b=%d n=%d m=%d", b, n, m);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(xyz1 && xyz2 && match && grad1 && grad2, "matchcostgrad: null pointer");
    return launch_matchcostgrad(b, n, m, xyz1, xyz2, match, grad1, grad2, (cudaStream_t)stream);
}

SNB_API int snb200_emd_per_cloud_supported(int b, int n, int m) { return emd_per_cloud_supported(b, n, m) ? 1 : 0; }

SNB_API size_t snb200_emd_per_cloud_workspace_bytes(int b, int n, int m) { return emd_per_cloud_supported(b, n, m) ? emd_per_cloud_workspace_bytes(b, n, m) : 0; }

// sizes, repeat and envelope: the checks both per-cloud EMD entries make before their pointers
static int emd_per_cloud_checks(const char *who, int b, int n, int m, int b2)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1, "%s: bad sizes b=%d n=%d m=%d", who, b, n, m);
    SNB_REQUIRE(b2 >= 1 && b2 <= (b > 0 ? b : 1) && b % b2 == 0, "%s: xyz2 repeats every b2=%d clouds, which must divide b=%d", who, b2, b);
    if (b > 0 && !emd_per_cloud_supported(b, n, m)) {
        set_error("%s: b=%d n=%d m=%d is outside the envelope (b <= 65535, n <= %d, m <= %d)", who, b, n, m, kEmdPerCloudMaxN, kEmdPerCloudMaxM);
        return SNB200_EUNSUPPORTED;
    }
    return SNB200_OK;
}

SNB_API int snb200_emd_per_cloud(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, float *cost, void *workspace,
                                 size_t workspace_bytes, snb200_stream_t stream)
{
    if (int rc = emd_per_cloud_checks("emd_per_cloud", b, n, m, b2)) return rc;
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(xyz1 && xyz2 && cost, "emd_per_cloud: null pointer");
    if (int rc = check_workspace("emd_per_cloud", workspace, workspace_bytes, emd_per_cloud_workspace_bytes(b, n, m))) return rc;
    return launch_emd_per_cloud(b, n, m, xyz1, xyz2, b2, cost, workspace, (cudaStream_t)stream);
}

SNB_API int snb200_emd_per_cloud_backward(int b, int n, const float *xyz1, int m, const float *xyz2, int b2, const float *grad_cost, float *grad1,
                                          float *grad2, const void *workspace, size_t workspace_bytes, snb200_stream_t stream)
{
    if (int rc = emd_per_cloud_checks("emd_per_cloud_backward", b, n, m, b2)) return rc;
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(xyz1 && xyz2 && grad_cost && (grad1 || grad2), "emd_per_cloud_backward: null pointer");
    if (int rc = check_workspace("emd_per_cloud_backward", workspace, workspace_bytes, emd_per_cloud_workspace_bytes(b, n, m))) return rc;
    return launch_emd_per_cloud_backward(b, n, m, xyz1, xyz2, b2, grad_cost, grad1, grad2, workspace, (cudaStream_t)stream);
}

SNB_API int snb200_nn_matching(int b, int n, int t, int k, const float *full_pc, const int *nn_idx, int complete_fps, float *out, int *out_idx,
                               snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && t >= 1 && k >= 1, "nn_matching: bad sizes b=%d n=%d t=%d k=%d", b, n, t, k);
    SNB_REQUIRE(complete_fps || k <= t, "nn_matching: without FPS completion k=%d must not exceed the number of indices t=%d", k, t);
    SNB_REQUIRE(k <= n, "nn_matching: k=%d exceeds the number of points n=%d", k, n);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(full_pc && nn_idx && out, "nn_matching: null pointer");
    return launch_nn_matching(b, n, t, k, full_pc, nn_idx, complete_fps, out, out_idx, (cudaStream_t)stream);
}

static int fps_checked(const char *who, int b, int n, int m, int layout, const float *inp, int *idx, float *out_points, int threads, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && m >= 1, "%s: bad sizes b=%d n=%d m=%d (npoint must be positive)", who, b, n, m);
    SNB_REQUIRE(layout == SNB200_BNC || layout == SNB200_BCN, "%s: unknown layout %d", who, layout);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(inp && idx, "%s: null pointer", who);
    return launch_farthest_point_sample(b, n, m, layout, inp, idx, out_points, threads, (cudaStream_t)stream);
}

SNB_API int snb200_farthest_point_sample(int b, int n, int m, int layout, const float *inp, int *idx, float *out_points, snb200_stream_t stream)
{
    return fps_checked("farthest_point_sample", b, n, m, layout, inp, idx, out_points, 0, stream);
}

SNB_API int snb200_rotate_jitter(int b, int n, int replicas, const float *in, float *out, const double *angles, const unsigned long long *key,
                                 double sigma, double clip, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && n <= (1 << 24) && replicas >= 1, "rotate_jitter: bad sizes b=%d n=%d replicas=%d (1 <= n <= 2^24)", b, n,
                replicas);
    SNB_REQUIRE((long long)b * replicas <= 0x7FFFFFFFLL, "rotate_jitter: b * replicas = %lld clouds exceed the grid", (long long)b * replicas);
    SNB_REQUIRE(angles || replicas == 1, "rotate_jitter: drawn angles (angles == NULL) need replicas == 1, got %d", replicas);
    SNB_REQUIRE(sigma >= 0.0, "rotate_jitter: sigma must be >= 0, got %g", sigma);
    SNB_REQUIRE(sigma == 0.0 || clip > 0.0, "rotate_jitter: clip must be > 0 when jittering, got %g", clip);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(in && out, "rotate_jitter: null pointer");
    SNB_REQUIRE(key || (angles && sigma == 0.0), "rotate_jitter: the key is null but angles are drawn or sigma > 0");
    const uintptr_t i0 = (uintptr_t)in, i1 = i0 + (size_t)b * n * 3 * sizeof(float);
    const uintptr_t o0 = (uintptr_t)out, o1 = o0 + (size_t)replicas * b * n * 3 * sizeof(float);
    SNB_REQUIRE((replicas == 1 && i0 == o0) || i1 <= o0 || o1 <= i0, "rotate_jitter: out overlaps in (in place only as in == out with replicas == 1)");
    return launch_rotate_jitter(b, n, replicas, in, out, angles, key, sigma, clip, (cudaStream_t)stream);
}

SNB_API int snb200_ae_augment(int b, int n, const float *in, float *out, const unsigned long long *key, int gauss, double mu, double sigma,
                              int z_rotate, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && n <= (1 << 24), "ae_augment: bad sizes b=%d n=%d (1 <= n <= 2^24)", b, n);
    SNB_REQUIRE(!gauss || (std::isfinite(mu) && std::isfinite(sigma) && sigma >= 0.0), "ae_augment: need finite mu and sigma >= 0, got mu=%g sigma=%g",
                mu, sigma);
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(in && out, "ae_augment: null pointer");
    SNB_REQUIRE(key || !(gauss || z_rotate), "ae_augment: the key is null but noise or a rotation is drawn");
    const uintptr_t i0 = (uintptr_t)in, i1 = i0 + (size_t)b * n * 3 * sizeof(float);
    const uintptr_t o0 = (uintptr_t)out, o1 = o0 + (size_t)b * n * 3 * sizeof(float);
    SNB_REQUIRE(i0 == o0 || i1 <= o0 || o1 <= i0, "ae_augment: out overlaps in (in place only as in == out)");
    return launch_ae_augment(b, n, in, out, key, gauss, mu, sigma, z_rotate, (cudaStream_t)stream);
}

SNB_API int snb200_registration_pairs(int b, int n, int s, int num_records, const float *clouds, const int *records, const float *transforms,
                                      const unsigned long long *key, float *p0, float *p1, float *vec, int *perm, snb200_stream_t stream)
{
    SNB_REQUIRE(b >= 0 && n >= 1 && s >= 1 && num_records >= 1, "registration_pairs: bad sizes b=%d n=%d s=%d num_records=%d", b, n, s,
                num_records);
    if (n > 2048) {
        snb::set_error("registration_pairs: n=%d points per cloud exceed the sort's 2048", n);
        return SNB200_EUNSUPPORTED;
    }
    if (b == 0) return SNB200_OK;
    SNB_REQUIRE(clouds && records && transforms && key && p0 && p1 && vec, "registration_pairs: null pointer");
    struct Span {
        uintptr_t lo, hi;
    };
    auto span = [](const void *p, size_t bytes) { return Span{(uintptr_t)p, (uintptr_t)p + bytes}; };
    const size_t pts = (size_t)b * n * 3 * sizeof(float);
    const Span out[4] = {span(p0, pts), span(p1, pts), span(vec, (size_t)b * 7 * sizeof(float)), span(perm, perm ? (size_t)b * n * sizeof(int) : 0)};
    const Span in[4] = {span(clouds, (size_t)s * n * 3 * sizeof(float)), span(records, (size_t)b * sizeof(int)),
                        span(transforms, (size_t)num_records * 7 * sizeof(float)), span(key, 2 * sizeof(unsigned long long))};
    auto apart = [](Span a, Span c) { return a.lo == a.hi || c.lo == c.hi || a.hi <= c.lo || c.hi <= a.lo; };
    for (int o = 0; o < 4; ++o) {
        for (int q = o + 1; q < 4; ++q) SNB_REQUIRE(apart(out[o], out[q]), "registration_pairs: outputs %d and %d overlap", o, q);
        for (int q = 0; q < 4; ++q) SNB_REQUIRE(apart(out[o], in[q]), "registration_pairs: output %d overlaps input %d", o, q);
    }
    return launch_registration_pairs(b, n, s, clouds, records, transforms, key, p0, p1, vec, perm, (cudaStream_t)stream);
}

SNB_API int snb200_retrieval_metrics_supported(int q, int m, int d, int levels, int exclude_diagonal)
{
    return retrieval_metrics_supported(q, m, d, levels, exclude_diagonal) ? 1 : 0;
}

SNB_API int snb200_retrieval_metrics(int q, int m, int d, const float *queries, const int *query_labels, const float *database,
                                     const int *database_labels, int exclude_diagonal, int levels, double *ap, double *prec, int *num_relevant,
                                     snb200_stream_t stream)
{
    if (!retrieval_metrics_supported(q, m, d, levels, exclude_diagonal)) {
        snb::set_error("retrieval_metrics: outside the envelope 1 <= q <= 2^20, 1 <= m <= 16384, 1 <= d <= 1024, 2 <= levels <= 101, q == m with "
                       "exclude_diagonal; got q=%d m=%d d=%d levels=%d exclude_diagonal=%d", q, m, d, levels, exclude_diagonal);
        return SNB200_EUNSUPPORTED;
    }
    SNB_REQUIRE(queries && query_labels && database && database_labels && ap && prec && num_relevant, "retrieval_metrics: null pointer");
    return launch_retrieval_metrics(q, m, d, queries, query_labels, database, database_labels, exclude_diagonal, levels, ap, prec, num_relevant,
                                    (cudaStream_t)stream);
}

SNB_API int snb200_debug_farthest_point_sample(int b, int n, int m, int layout, const float *inp, int *idx, float *out_points, int threads,
                                               snb200_stream_t stream)
{
    return fps_checked("debug_farthest_point_sample", b, n, m, layout, inp, idx, out_points, threads, stream);
}

SNB_API int snb200_debug_conv_stack_partition(int b, int n, int *ppc, int *slices, int *grid, int *per_cta, int *slots)
{
    SNB_REQUIRE(b >= 1 && n >= 1, "debug_conv_stack_partition: bad sizes b=%d n=%d", b, n);
    SNB_REQUIRE(ppc && slices && grid && per_cta && slots, "debug_conv_stack_partition: null pointer");
    conv_stack_partition(b, n, ppc, slices, grid, per_cta, slots);
    return SNB200_OK;
}

SNB_API int snb200_debug_generator_plan(int b, int n, int num_conv, const snb200_layer *conv, int num_fc, const snb200_layer *fc, int flags,
                                        int *conv_path, int *fuse_head)
{
    if (int rc = check_generator_tables("debug_generator_plan", num_conv, conv, num_fc, fc)) return rc;
    SNB_REQUIRE(b >= 1 && n >= 1, "debug_generator_plan: bad sizes b=%d n=%d", b, n);
    SNB_REQUIRE(conv_path && fuse_head, "debug_generator_plan: null pointer");
    generator_plan_debug(b, n, num_conv, conv, num_fc, fc, flags, conv_path, fuse_head);
    return SNB200_OK;
}

SNB_API int snb200_nonfinite_guard(const snb200_guard_check *checks, int num_checks, const snb200_guard_restore *restores, int num_restores,
                                   unsigned *state, int *skipped, int *skip_count, snb200_stream_t stream)
{
    SNB_REQUIRE(num_checks >= 0 && num_restores >= 0, "nonfinite_guard: bad table sizes %d, %d", num_checks, num_restores);
    SNB_REQUIRE((checks || num_checks == 0) && (restores || num_restores == 0) && state, "nonfinite_guard: null pointer");
    for (int i = 0; i < num_checks; i++) {
        SNB_REQUIRE(checks[i].count >= 0 && (checks[i].ptr || checks[i].count == 0), "nonfinite_guard: check %d has a bad span", i);
        SNB_REQUIRE(checks[i].dtype >= SNB200_GUARD_F32 && checks[i].dtype <= SNB200_GUARD_BF16, "nonfinite_guard: check %d has unknown dtype %d",
                    i, checks[i].dtype);
    }
    for (int i = 0; i < num_restores; i++)
        SNB_REQUIRE(restores[i].bytes >= 0 && ((restores[i].live && restores[i].snapshot) || restores[i].bytes == 0),
                    "nonfinite_guard: restore %d has a bad span", i);
    return launch_nonfinite_guard(checks, num_checks, restores, num_restores, state, skipped, skip_count, (cudaStream_t)stream);
}
