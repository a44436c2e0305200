// encoder_internal.cuh -- declarations shared by encoder.cu (CUDA-core path), encoder_tc.cu (tensor-core path), conv_stack.cu,
// generator.cu, generator_bwd.cu, the frozen encoders (frozen_encoder.cu, frozen_encoder_bstat.cu) and point_transform.cu.
#pragma once
#include "common.cuh"

namespace snb {

constexpr int kTcM = 128;        // points per tile of the tensor-core layer kernels (one CTA, UMMA M)
constexpr int kMaxPrefix = 16;   // most prefixes one frozen pass evaluates

__host__ __device__ __forceinline__ int tc_tiles_per_cloud(int n) { return (n + kTcM - 1) / kTcM; }

// The grouped-prefix layout: the prefixes x[c, :sizes[p]] of b clouds of n points, packed prefix by prefix and cloud by cloud, each
// (prefix, cloud) segment padded to whole tiles.  No tile straddles two segments, and group p (prefix p) owns tiles [tile0[p], tile0[p + 1]).
struct PrefixPack {
    int np, b, n;
    int sizes[kMaxPrefix];        // ascending prefix lengths
    int tile0[kMaxPrefix + 1];    // tile0[np]: the number of tiles
};

inline PrefixPack prefix_pack(int b, int n, int np, const int *sizes)
{
    PrefixPack S;
    memset(&S, 0, sizeof(S));
    S.np = np; S.b = b; S.n = n;
    for (int p = 0; p < np; p++) {
        S.sizes[p] = sizes[p];
        S.tile0[p + 1] = S.tile0[p] + b * tc_tiles_per_cloud(sizes[p]);
    }
    return S;
}

// tile -> (group, cloud, first point of the tile within the cloud, rows of the tile inside its segment)
__device__ __forceinline__ void pack_tile(const PrefixPack &S, int tile, int &g, int &cloud, int &i0, int &rows)
{
    g = 0;
    while (tile >= S.tile0[g + 1]) g++;
    const int tps = tc_tiles_per_cloud(S.sizes[g]), local = tile - S.tile0[g];
    cloud = local / tps;
    i0 = (local - cloud * tps) * kTcM;
    rows = min(kTcM, S.sizes[g] - i0);
}

// packed row of point i of (group g, cloud)
__device__ __forceinline__ long long pack_row(const PrefixPack &S, int g, int cloud, int i)
{
    return ((long long)S.tile0[g] + (long long)cloud * tc_tiles_per_cloud(S.sizes[g])) * kTcM + i;
}

// scale/shift of a BatchNorm given either batch statistics or running statistics (the per-layer kernels of encoder.cu / encoder_tc.cu)
__device__ __forceinline__ void bn_scale_shift(const double *stats, int c_total, int c, double count, const float *gamma, const float *beta,
                                               const float *run_mean, const float *run_var, float eps, int training, float &scale, float &shift)
{
    float mean, var;
    if (training) {
        const double m = stats[c] / count;
        double v = stats[c_total + c] / count - m * m;
        if (v < 0) v = 0;
        mean = (float)m;
        var = (float)v;
    } else {
        mean = run_mean[c];
        var = run_var[c];
    }
    const float invstd = 1.0f / sqrtf(var + eps);
    scale = gamma[c] * invstd;
    shift = beta[c] - mean * scale;
}

struct TcLayerParams {
    // FIRST mode (x != nullptr): the A operand is layer 1 (3 -> c_in, weights w1/b1) evaluated on the fly from the cloud,
    // its BatchNorm statistics having been derived analytically from the input moments (x_moments_kernel).
    const float *x;             // cloud (b, n, 3) BNC or (b, 3, n) BCN, or nullptr
    int x_layout;
    const float *w1, *b1;       // (c_in, 3), (c_in)
    float *out1;                // FIRST mode: layer 1's raw output (b*n, c_in) is stored here when non-null (training forward that keeps it)
    const float *in;           // previous layer's raw output (b*n, c_in) row-major (x == nullptr)
    float *in_act_out;          // or nullptr: the input's activation relu(bn(in)) (b*n, c_in), as the prologue evaluates it, is stored here too
    int c_in, c_out;
    int b, n, tiles_per_cloud;
    const double *in_stats;
    const float *in_gamma, *in_beta, *in_run_mean, *in_run_var;
    float in_eps;
    int in_relu, in_has_bn, in_training;
    const float *weight, *bias;
    float *out;                 // raw output or nullptr (last layer)
    double *out_stats;          // or nullptr
    float *tile_max, *tile_min; // or nullptr
    // Pool of a frozen encoder's last layer (tile_val != nullptr): grid.y walks blocks of 256 output channels, nothing is stored but the
    // first extreme of sign(scale) * z (value and point index) over the tile's rows.  Prefix pool (pack.np > 0): at every prefix boundary
    // pack.sizes[p] inside the tile and at the tile's end.
    PrefixPack pack;            // the prefix pool's np / sizes, or with GRP the whole layout
    // Many prefixes (pfx_sizes != nullptr): the pack.np ascending sizes are a device array instead of pack.sizes, and pfx_first
    // (tiles_per_cloud + 1 entries, device) holds per tile of a cloud the first prefix whose boundary lies in it: tile t's boundaries are
    // prefixes pfx_first[t] .. pfx_first[t + 1] - 1.
    const int *pfx_sizes, *pfx_first;
    const float *pool_gamma;    // the layer's BatchNorm weight (its sign is the sign of the scale), or nullptr (no BatchNorm: max)
    float *bound_val;           // (num_prefix, b, c_out): sign * z of the extreme over [tile start, sizes[p]) in the tile holding sizes[p] - 1
    int *bound_idx;
    float *tile_val;            // (b * tiles_per_cloud, c_out): ... over the whole tile
    int *tile_idx;
    // Segment pool (seg != nullptr, b == 1, pack.np == 0): the rows are a packed buffer of num_seg segments (offset, length), each
    // starting on a tile; tile_val / tile_idx get the extreme over the tile's rows inside its segment, the index relative to the segment's
    // first row.  Tiles of padding rows record nothing.
    const int2 *seg;
    int num_seg;
    // Grouped statistics (grp_part != nullptr, tc_layer_kernel<..., GRP = true>, frozen_encoder_bstat.cu): b == 1, and the n rows are the
    // packed prefixes of pack.  FIRST mode reads the cloud x (pack.b, pack.n, 3) BNC at the tile's (cloud, point offset).
    const double *grp_in_stats;   // (pack.np, 2, c_in): mean and biased variance of the input layer's raw output per group
    float *grp_part;              // (tiles, 2, c_out): sum and sum of squares of the output over each tile's rows inside its segment
};

// scale / shift of a BatchNorm from a group's mean and biased variance, in the float expressions of bn_scale_shift's training branch
__device__ __forceinline__ void bn_group_scale_shift(double m, double v, float gamma, float beta, float eps, float &scale, float &shift)
{
    const float mean = (float)m, var = (float)v;
    const float invstd = 1.0f / sqrtf(var + eps);
    scale = gamma * invstd;
    shift = beta - mean * scale;
}

// One nn.BatchNorm1d running-statistics step of channel c from a batch's mean m and biased variance v over `count` values: momentum `mom`,
// the variance made unbiased with count / (count - 1).  NULL buffers are skipped.
__device__ __forceinline__ void bn_running_step(float *run_mean, float *run_var, int c, double m, double v, double count, float mom)
{
    const double unb = count > 1 ? v * (count / (count - 1)) : v;
    if (run_mean) run_mean[c] = (1.f - mom) * run_mean[c] + mom * (float)m;
    if (run_var) run_var[c] = (1.f - mom) * run_var[c] + mom * (float)unb;
}

// The segment holding packed row r (segments in ascending offset order, device table), or -1 for a row outside every segment.
__device__ __forceinline__ int seg_find(const int2 *__restrict__ seg, int num_seg, long long r)
{
    int lo = 0, hi = num_seg - 1, j = -1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        if (seg[mid].x <= r) { j = mid; lo = mid + 1; }
        else hi = mid - 1;
    }
    return (j >= 0 && r < (long long)seg[j].x + seg[j].y) ? j : -1;
}

// The first extreme over one segment's tile records t0 .. t1 - 1 of channel c, value and index (ties keep the earlier tile)
__device__ __forceinline__ void seg_tile_extreme(const float *__restrict__ tile_val, const int *__restrict__ tile_idx, int C, int c, int t0, int t1,
                                                 float &run, int &run_i)
{
    run = tile_val[(size_t)t0 * C + c];
    run_i = tile_idx[(size_t)t0 * C + c];
    for (int t = t0 + 1; t < t1; t++) {
        const float v = tile_val[(size_t)t * C + c];
        if (v > run) { run = v; run_i = tile_idx[(size_t)t * C + c]; }
    }
}

// One tc_layer_kernel launch, the instantiation chosen by P: a pool (tile_val) or not, grouped statistics (grp_part) or not.  A grouped layer
// with the pool is the last one: it keeps the segment pool's per-tile records and stores z too.
int launch_tc_layer(const TcLayerParams &P, cudaStream_t stream);
constexpr int kTcMaxLastOut = 1024;   // widest last layer of a tensor-core stack (blocks of 256 output channels over grid.y)
bool tc_layer_supported(int c_in, int c_out);        // a hidden layer: up to 256 channels in and out
bool tc_last_layer_supported(int c_in, int c_out);   // the last layer: up to 256 in, kTcMaxLastOut out
int launch_x_moments(int b, int n, int layout, const float *x, double *mom, unsigned *counter, const float *w1, const float *b1, int c1,
                     double *stats0, cudaStream_t stream);
// The last layer's epilogue in launch_tc_stack: per-tile extrema, or with num_prefix > 0 the prefix pool of a frozen encoder, or with seg the
// segment pool (see TcLayerParams).  sizes is a host array of at most kMaxPrefix entries, or with dev_first != nullptr a device array of
// any length and dev_first its per-tile first prefixes (TcLayerParams::pfx_sizes / pfx_first).
struct TcStackTail {
    float *tile_max, *tile_min; int num_prefix; const int *sizes; float *bound_val; int *bound_idx; float *tile_val; int *tile_idx;
    const int2 *seg; int num_seg;
    const int *dev_first;
};
// Layers 2 .. nconv on the tensor-core layer kernels, layer 1 evaluated in layer 2's prologue from x.  stats: the per-layer BatchNorm statistics,
// or nullptr (eval mode without them).  With zsave every stored raw output goes to zsave[l], layer 1's included; otherwise the hidden layers
// ping-pong through act[0] / act[1].
// act_in != nullptr (x unused): layer 1 is a tensor-core layer too, reading the (b*n, c_in) activation act_in as it is (identity input).
// tap >= 0: hidden layer tap's activation relu(bn(z_tap)) is also stored to tap_out (b*n, c_out_tap) by the prologue of layer tap + 1.
int launch_tc_stack(int b, int n, int layout, const float *x, int nconv, const snb200_layer *conv, int training, double *const *stats,
                    float *const *zsave, float *const *act, const TcStackTail &tail, cudaStream_t stream, const float *act_in = nullptr,
                    int tap = -1, float *tap_out = nullptr);
// CUDA-core conv stack: writes per-tile extrema of the last layer and (training) per-layer statistics
int launch_simt_conv_stack(int b, int n, int layout, const float *x, int num_layers, const snb200_layer *layers, int training, float *act0,
                           float *act1, double *const *stats, float *tile_max, float *tile_min, cudaStream_t stream);
int simt_tiles_per_cloud(int n, int c_last);   // per-tile extrema per cloud written by launch_simt_conv_stack (its `tiles_per_cloud`)

// pool + FC head description (generator.cu builds it; the cluster kernel and the fused tail of the conv-stack kernel consume it)
struct HeadLayer {
    int c_in, c_out;
    const float *weight, *bias, *gamma, *beta;
    float *run_mean, *run_var;
    float eps, momentum;
    int has_bn, relu;
    const float *out_mask;   // (b, c_out) dropout mask of the next layer's input, multiplied into this layer's stored output, or null
};

struct HeadParams {
    int b, training;
    // pooling of the last conv layer
    int c_feat, tiles_per_cloud;
    const float *tile_max, *tile_min;   // cluster head: tile_max == nullptr means no pool, feat holds the FC input
    const double *last_stats;
    int stat_rep;                // 0: (sum, sumsq) of every conv layer are the plain [2][C] block; 1: the accumulators the conv-stack kernel adds into
                                 // are spread one per 128-byte line behind that block: accumulator idx at stats[2C + idx * kStatStride]
    const float *last_gamma, *last_beta, *last_run_mean, *last_run_var;
    float last_eps;
    int last_has_bn, last_relu;
    double count;
    float *feat;                 // (b, c_feat) global: pooled feature (also an API output)
    // running-statistics updates of the conv layers
    int ru_num;
    const double *ru_stats[SNB200_MAX_CONV_LAYERS];
    int ru_rep[SNB200_MAX_CONV_LAYERS];   // replicas behind each of them (see stat_rep)
    float *ru_mean[SNB200_MAX_CONV_LAYERS];
    float *ru_var[SNB200_MAX_CONV_LAYERS];
    float ru_momentum[SNB200_MAX_CONV_LAYERS];
    int ru_c[SNB200_MAX_CONV_LAYERS];
    // FC layers
    int num_fc;
    HeadLayer fc[SNB200_MAX_FC_LAYERS];
    float *act[2];               // (b, max width) scratch
    float *out;                  // (b, c_out_last)
    int out_inner;
    // torch BatchNorm bookkeeping: int64 counters incremented once per training forward
    int num_counters;
    long long *counters[SNB200_MAX_CONV_LAYERS + SNB200_MAX_FC_LAYERS];
    float *ll[SNB200_MAX_FC_LAYERS + 1];   // fused head: self-validating exchange buffers, zero at launch: [0] pooled feature (b, c_feat),
                                           // [l+1] output of FC layer l (b, c_out); a word of 0 means "not stored yet"
    int keep_inputs;             // cluster head: also store every FC layer's input in ll[l] (training forward that keeps activations)
    int k_chunk;                 // cluster head: FC input channels staged per pass (the widest input, or fewer when that does not fit)
};

// Filling a zeroed HeadParams (generator.cu).  fill_pool_params: the pool of the last conv layer's per-tile extrema into feat (b, c_last)
// with the conv layers' batch statistics stats[l], and in training their running-statistics updates and num_batches_tracked counters.
// fill_fc_params (after H.b and H.training are set): the FC layers from H.feat to out, and in training their counters.
void fill_pool_params(HeadParams &H, int b, int n, int tpc, int nconv, const snb200_layer *conv, int training, double *const *stats,
                      float *tile_max, float *tile_min, float *feat);
void fill_fc_params(HeadParams &H, int nfc, const snb200_layer *fc, float *out, int out_transpose_inner);
// fc_head_cluster_kernel as one thread-block cluster; H.num_fc == 0 runs the pool alone, H.tile_max == nullptr the FC layers alone.
int launch_fc_head_cluster(const HeadParams &H, cudaStream_t stream);

// persistent cooperative conv-stack kernel (conv_stack.cu); head != nullptr fuses the pool + FC head into the same launch
bool conv_stack_supported(int b, int n, int nconv, const snb200_layer *conv);
int conv_stack_slots_per_cloud(int b, int n);   // pool partials per cloud written by the conv-stack kernel (its `tiles_per_cloud`)
int launch_conv_stack(int b, int n, int layout, const float *x, int nconv, const snb200_layer *conv, int training, double *const *stats,
                      double *mom, unsigned *barrier, float *tile_max, float *tile_min, const HeadParams *head,
                      char *clean_ptr, size_t clean_bytes, cudaStream_t stream, float *const *zsave = nullptr, float *const *act = nullptr);

// the pieces of the generator's forward workspace the backward pass reads (generator.cu carves the workspace, generator_bwd.cu reads it)
struct GenWorkspaceView {
    const double *stats[SNB200_MAX_CONV_LAYERS];
    const float *ll[SNB200_MAX_FC_LAYERS + 1];
};
GenWorkspaceView generator_workspace_view(void *fwd_workspace, int b, int n, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc);

// The per-layer training path's additions (snb200_generator_layers_ex_*).  A null GenEx, or one with act_input = 0, tap = -1 and null
// pointers, is the plain per-layer path.
struct GenEx {
    int act_input;              // the stack's input is a (b*n, c_in) activation layer 1 reads as it is, instead of the cloud
    int tap;                    // -1, or the hidden layer whose activation relu(bn(z_tap)) the forward stores to tap_out
    float *tap_out;             // forward
    const float *grad_tap;      // backward: (b*n, c_out_tap) added to the gradient of a_tap, or null
    float *grad_in;             // backward: gradient of the stack's input, or null
    const float *fc_dropout[SNB200_MAX_FC_LAYERS];   // per FC layer: (b, c_in) mask multiplying its input, or null (never layer 0)
};
bool generator_layers_ex_supported(int b, int n, int act_input, int nconv, const snb200_layer *conv, int nfc, const snb200_layer *fc, int tap,
                                   const float *const *fc_dropout);

// Per-chunk weight-gradient partials -> gradients in a fixed order (generator_bwd.cu; also the frozen encoder's parameter backward).  A job's
// partials are nparts blocks of nw + nb floats, weights (c_out, c_in) row-major then biases; a NULL g_weight / g_bias is skipped.
struct ReduceJob { const float *part; int nparts; int nw, nb; float *g_weight, *g_bias; };
struct ReduceParams { int njobs; ReduceJob job[SNB200_MAX_CONV_LAYERS]; };
int launch_reduce_partials(const ReduceParams &R, cudaStream_t stream, const char *what);

}  // namespace snb
