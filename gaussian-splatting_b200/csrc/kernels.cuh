// kernels.cuh -- argument blocks and host launchers of the rasterizer kernels.
#pragma once
#include "common.cuh"
#include "geom.cuh"

namespace gsb {

// per-gaussian gradient accumulator written by the backward blend kernel (float, 48 B stride):
//   0..4 raw moments of t = dL/d(power): sum t dx, t dy, t dx^2, t dx dy, t dy^2   5 opacity  6,7,8 rgb  9 inverse depth  10,11 pad
// (the feature pass, features.cu, adds its terms of a feature loss into 0..5 of the same rows)
constexpr int DACC_STRIDE = 12;

// ---- view-batch variants: per-view arrays are laid out [V][...] with uniform strides (in elements) ----
constexpr int GSB_MAX_VIEWS = 16;
constexpr int GSB_MAX_PEERS = 16;
struct CamArgsBatch {
    int V;
    CamArgs cam[GSB_MAX_VIEWS];
};
struct PreFwdBatchStrides { size_t splat /* float4 */, per_gauss /* u32 / uint2 arrays */, radii; };
struct PreBwdBatchStrides { size_t splat /* float4 */, dacc /* float */, means2D /* float */; };

// Split SH input (gsb_forward_split_sh / gsb_backward_split_sh, single-view kernels only): `shs` points at the DC rows
// [P,1,3] and `rest` at the remaining coefficients [P,M-1,3] (NULL when M == 1); the kernels assemble the joint row in
// shared memory.  Every other launch leaves `rest` (and `dL_drest`) NULL.
struct PreFwdArgs {
    int P;
    const float *means, *shs, *colors, *opac, *scales, *rots, *cov_pre;
    const float *rest;
    float4 *splat;        // [P*3]
    uint32_t *depth_key;  // [P] float bits of view depth, 0xffffffff when culled
    uint32_t *depth_idx;  // [P] identity, sorted along with the keys
    uint32_t *tiles;      // [P] tiles touched after exact culling
    uint2 *rect;          // [P] x0|x1<<16, y0|y1<<16 reference 3-sigma tile rectangle
    int *radii;           // [P] output
    int cull;             // 1: exact tile culling, 0: reference rectangle (debug / A-B)
};

// Fused reduce-scatter (gsb_backward_batch_peer): gaussians [r * rows_per_rank, (r + 1) * rows_per_rank) are OWNED by rank r;
// every rank adds its gradient rows straight into the owner's buffer.  delta[r] = byte offset that turns an address inside THIS
// rank's gradient buffer into the same location of rank r's buffer as mapped into this process (0 for r == rank).
struct PeerTable {
    int world;              // 0 = no peers (plain local output)
    int rows_per_rank;      // multiple of the per-gaussian kernels' block size
    long long delta[GSB_MAX_PEERS];
};

struct PreBwdArgs {
    int P;
    const float *means, *shs, *opac, *scales, *rots, *cov_pre;
    const float4 *splat;
    const float *dacc;    // [P*DACC_STRIDE]
    int p_begin, p_end;   // gaussian range of this launch (chunked backward: the caller reduces finished chunks meanwhile)
    GsbGrads g;
    PeerTable peer;       // world > 0: outputs are ADDED into the owners' buffers (view-batch kernel, TMA rows only)
    const float *rest;    // split SH input: shs = DC rows, g.dL_dshs = their gradient, rest / dL_drest the other coefficients
    float *dL_drest;
    float *cam_part;      // non-NULL: camera gradient requested; per-warp partials [V][CAM_TERMS][cam_slots(p_end - p_begin)]
};

// Camera gradient (gsb_backward_camera / gsb_backward_batch_camera): the 27 per-gaussian terms of preprocess.cu's CamGrad
// (viewmatrix rows 0..3 x columns 0..2, projmatrix rows 0..3 x columns 0, 1, 3, campos), summed per warp by K8 and then over
// the warps by camera_grad_reduce_kernel.  dL/dbg = sum over pixels of final_T * dL/dcolor: CAM_BG_BLOCKS partials per view
// and channel (camera_bg_partial_kernel), summed by the same reduce kernel.  No float atomics: every sum has a fixed order.
constexpr int CAM_TERMS = 27;
constexpr int CAM_OUTPUTS = 16 + 16 + 3 + 3;
constexpr int CAM_BG_BLOCKS = 128;
struct CamReduceArgs {
    int V, nslots;               // views; warp partials per view (0: no gaussians)
    float *part;                 // [V][CAM_TERMS][nslots]
    float *bg_part;              // [V][3][CAM_BG_BLOCKS] scratch
    float *dview, *dproj, *dcampos, *dbg;   // [V][16], [V][16], [V][3], [V][3]; NULL = not requested
    const float *final_T;        // view v: final_T + v * sv_image, [npix]
    size_t sv_image, npix;
    const float *dL_dcolor;      // [V][3][npix]
};
size_t cam_slots(int n_gauss);   // warp partials of one view for a K8 launch over n_gauss gaussians

struct BinArgs {
    int P;
    int num_tiles, gx;
    // view-batch launches (blockIdx.y = view): strides between the views' arrays, in elements; 0 for single view
    size_t sv_gauss;          // order / tiles / rect / offsets
    size_t sv_splat;          // float4
    size_t sv_scan;           // scan_state
    size_t sv_inst;           // instance arrays (capacity)
    const uint32_t *order;    // [P] gaussian ids in depth order
    const uint32_t *tiles;    // [P]
    const uint2 *rect;        // [P]
    const float4 *splat;
    uint32_t *offsets;        // [P] exclusive scan of tiles in depth order
    unsigned long long *scan_state;   // [V][scan_state_count(P)] scan scratch, zeroed by launch_tile_scan
    unsigned long long *total;  // device scalar: D
};

// Blend launches cover V views (blockIdx.y): every per-view array is base + view * stride (strides in elements; 0 and V = 1
// for the single-view call).  tile_order (optional, [V][tiles]): blockIdx.x -> tile id permutation (heavy tiles first).
struct RenderFwdArgs {
    int W, H, gx, gy, V;
    size_t sv_ranges, sv_list, sv_splat /* float4 */, sv_color, sv_depth, sv_image;
    const uint2 *ranges;
    const uint32_t *point_list;
    const uint32_t *tile_order;
    const float4 *splat;
    const float *bg[GSB_MAX_VIEWS];
    float *out_color, *out_invdepth, *final_T;
    uint32_t *n_contrib;
};

struct RenderBwdArgs {
    int W, H, gx, gy, V;
    size_t sv_ranges, sv_list, sv_splat /* float4 */, sv_color, sv_depth, sv_image, sv_dacc;
    const uint2 *ranges;
    const uint32_t *point_list;
    const uint32_t *tile_order;
    const float4 *splat;
    const uint32_t *n_contrib;
    const float *out_color, *out_invdepth;   // forward outputs
    const float *dL_dcolor, *dL_dinvdepth;
    float *dacc;
    // rendered-alpha gradient (alpha = 1 - final_T): dL_dalpha [V][H*W] at stride sv_depth, final_T at stride sv_image; NULL =
    // no alpha term.  Appended last so that the parameter offsets of the kernels that do not read them stay where they were.
    const float *final_T, *dL_dalpha;
    // deterministic backward (DESIGN.md section 7.9), NULL = the plain kernel: det_part [V][sv_list * 2][DACC_STRIDE] partial rows,
    // det_mark [V][sv_list * 2] bytes, zeroed by the caller; appended last, as above
    float *det_part;
    uint8_t *det_mark;
};

// alpha[v][p] = 1 - final_T[v][p] for V <= GSB_MAX_VIEWS forward states (any mix of single-view and view-batch calls)
struct AlphaArgs {
    int V;
    size_t npix;
    const float *final_T[GSB_MAX_VIEWS];
    float *out;           // [V][npix]
};

// Rendered feature maps (features.cu, DESIGN.md section 7.7): F[v][c][p] = sum_k w_k(p) features[id_k][c] with the forward's blend
// weights, channels in groups of 4 or 8 (blockIdx.z) and views in blockIdx.y.  Every view is one forward state of its own
// (any forward entry point); the backward adds its moment and opacity terms into rows view * P + id of `dacc` (the same rows
// render_bwd_kernel fills) and dL/dfeatures, summed over the views, into dL_dfeatures.
constexpr int FEAT_MAX_CHANNELS = 128;
struct FeatView {
    const uint2 *ranges;
    const uint32_t *point_list, *tile_order;
    const float4 *splat;
    const uint32_t *n_contrib;
};
struct FeatArgs {
    int W, H, gx, gy, V, C, P;
    FeatView view[GSB_MAX_VIEWS];
    const float *features;                  // [P, C]
    float *out;                             // forward: [V, C, H*W]
    const float *out_features, *dL_dout;    // backward: the forward's output and its gradient, [V, C, H*W]
    float *dacc;                            // backward: [V * P, DACC_STRIDE], zeroed by the caller
    float *dL_dfeatures;                    // backward: [P, C], added into; NULL = not requested
};

// Contribution statistics (contrib.cu, DESIGN.md section 7.8): for every pair a forward state accepted, count[id] += 1,
// weight_sum[id] += w and weight_max[id] = max(., w) with w = alpha T, over V <= GSB_MAX_VIEWS states (blockIdx.y = view).
struct ContribArgs {
    int W, H, gx, gy, V, P;
    FeatView view[GSB_MAX_VIEWS];
    long long *count;              // [P], added into
    float *weight_sum;             // [P], added into
    uint32_t *weight_max_bits;     // [P] float bits (w >= 0), max-ed into
};

// split: a.shs / a.rest are the split SH input (see PreFwdArgs)
int launch_preprocess_fwd(const CamArgs &ca, const PreFwdArgs &a, bool split, bool debug, cudaStream_t stream);
int launch_preprocess_bwd(const CamArgs &ca, const PreBwdArgs &a, bool split, bool accumulate, bool debug, cudaStream_t stream);
int launch_preprocess_fwd_batch(const CamArgsBatch &cb, const PreFwdArgs &a, const PreFwdBatchStrides &st, bool debug, cudaStream_t stream);
int launch_preprocess_bwd_batch(const CamArgsBatch &cb, const PreBwdArgs &a, const PreBwdBatchStrides &st, bool accumulate, bool debug,
                                cudaStream_t stream);
int launch_mark_visible(int P, const float *means, const float *view, uint8_t *present, cudaStream_t stream);
int launch_camera_grad_reduce(const CamReduceArgs &r, bool accumulate, bool debug, cudaStream_t stream);

size_t scan_state_count(int P);
// V > 1: blockIdx.y = view, arrays offset by the BinArgs strides; totals / n_dev are arrays of V counts
int launch_tile_scan(const BinArgs &a, int V, bool debug, cudaStream_t stream);
// async forward: counts[GSB_MAX_VIEWS] = max(counts[GSB_MAX_VIEWS], counts[0..V))  (running maximum the host polls later)
int launch_count_max(unsigned long long *counts, int V, bool debug, cudaStream_t stream);
// also fills dg.ghist, the digit histograms of the tile sort of the emitted keys (sort_prepare before, sort_pairs(hist_ready) after)
int launch_emit(const BinArgs &a, int V, uint32_t *inst_tile, uint32_t *inst_gauss, int64_t cap, const SortDigits &dg, bool debug,
                cudaStream_t stream);
int launch_tile_ranges(const uint32_t *sorted_tiles, int64_t D, const unsigned long long *n_dev, int num_tiles,
                       uint2 *ranges, int V, size_t sv_inst, bool debug, cudaStream_t stream);

int launch_render_fwd(const RenderFwdArgs &a, bool debug, cudaStream_t stream);
int launch_render_bwd(const RenderBwdArgs &a, bool debug, cudaStream_t stream);
int launch_alpha(const AlphaArgs &a, bool debug, cudaStream_t stream);
// deterministic backward (deterministic.cu, DESIGN.md section 7.9): scratch of V views of capn list positions each
struct DetScratch {
    int64_t capn;
    float *part;                      // [V][capn * 2][DACC_STRIDE] partial rows of render_bwd_kernel<..., DET>
    uint8_t *mark;                    // [V][capn * 2] written-pair marks, zeroed before the blend launch
    uint32_t *keys, *vals, *keys_alt, *vals_alt;   // [V][capn] (gaussian id, list position) pairs of the grouping sort
    unsigned long long *count;        // [GSB_MAX_VIEWS] instances per view
    char *sortscr;
};
size_t det_carve(void *base, int64_t capn, int V, DetScratch &d);    // base NULL: size only
// after launch_render_bwd(a) with a.det_part / a.det_mark from d: every row view * P + g of dacc, g < P, is stored
int launch_det_reduce(const RenderBwdArgs &a, const DetScratch &d, int P, float *dacc, bool debug, cudaStream_t stream);
int launch_render_features(const FeatArgs &a, bool debug, cudaStream_t stream);
int launch_render_features_bwd(const FeatArgs &a, bool debug, cudaStream_t stream);
int launch_contribution(const ContribArgs &a, bool debug, cudaStream_t stream);
int launch_tile_order(const uint2 *ranges, int V, int num_tiles, uint32_t *order, bool debug, cudaStream_t stream);
int launch_l1_loss_grad(const float *img, const float *gt, int64_t n, float scale, float *grad, float *loss_accum,
                        cudaStream_t stream);
int launch_photometric_loss_grad(const float *img, const float *gt, int C, int H, int W, float lambda_dssim, bool clamp_input,
                                 float *grad, float *loss_accum, float *maps, cudaStream_t stream);

// optimizer step and densification on the flat store (optim.cu, densify.cu)
int launch_adam_step(int64_t P, int sh_coeffs, float *params, const float *grads, float *m, float *v, float *act,
                     const uint8_t *visible, const float step_size[6], float beta1, float beta2, float eps, const float bias2_sqrt[6],
                     uint32_t skip_groups, cudaStream_t stream);
int launch_activate(int64_t P, int sh_coeffs, const float *params, float *act, cudaStream_t stream);
// SparseGaussianAdam: up to GSB_MAX_SPARSE_GROUPS [N, width] groups, rows with visible[i] == 0 untouched (optim.cu)
int launch_sparse_adam_step(const GsbSparseAdamGroup *groups, int n_groups, const uint8_t *visible, int64_t N, float beta1, float beta2,
                            cudaStream_t stream);
size_t densify_scratch_bytes(int64_t P, int n_children);
// exclusive scan of n uint32 (in == out allowed); partials: scan_u32_partials(n) words; *total receives the sum
size_t scan_u32_partials(int64_t n);
int scan_u32_exclusive(const uint32_t *in, uint32_t *out, size_t n, uint32_t *partials, uint32_t *total, cudaStream_t stream);
// 3-nearest-neighbour mean squared distance (knn.cu)
size_t knn_scratch_bytes(int64_t P);
int launch_knn_mean_dist2(const float *points, int64_t P, float *out, void *scratch, cudaStream_t stream);
int launch_densify_plan(int64_t P, int sh_coeffs, int n_children, const float *params, const float *grad_accum, const float *denom,
                        float grad_threshold, float size_limit, float min_opacity, float world_limit, void *scratch,
                        uint32_t **counters_dev, cudaStream_t stream);
int launch_densify_apply(int64_t P, int sh_coeffs, int n_children, const float *params, const float *m, const float *v, void *scratch,
                         const float *unit_samples, int64_t n_split, int64_t P_new, float *new_params, float *new_m, float *new_v,
                         cudaStream_t stream);
// prune_points on the store: scratch of densify_scratch_bytes(P, 1); plan = keep flags, their exclusive scan and the source row
// of every output row (*counter_dev: the device word holding P_new), apply = the densify gather of the kept rows
int launch_prune_plan(int64_t P, const uint8_t *remove, void *scratch, uint32_t **counter_dev, cudaStream_t stream);
int launch_prune_apply(int64_t P, int sh_coeffs, const float *params, const float *m, const float *v, const void *scratch, int64_t P_new,
                       float *new_params, float *new_m, float *new_v, cudaStream_t stream);

}  // namespace gsb
