/*
 * gs_b200.h -- C ABI of libgs_b200.so, the H100 (sm_90a) differentiable 3D-Gaussian-splatting
 * rasterizer.  Plain C: raw device pointers, explicit sizes, explicit stream, int error codes.
 * No torch types, no exceptions.  Process-wide state, all of it listed here: the tuning options
 * (gsb_set_option: set them before the first call and leave them alone while calls are in flight),
 * the launch counter and the kernel-timing records (diagnostics, mutex-guarded).  Per host thread:
 * the last error string, the deterministic switch (gsb_set_deterministic) and one pinned read-back slot +
 * event per device.
 * Threading: any number of host threads may call concurrently (different streams / devices); the
 * reference calls from its single training thread (train.py), one process per GPU.
 *
 * What each entry point replaces in the reference (graphdeco-inria/gaussian-splatting):
 * the reference reaches this path ONLY through the python package imported at
 *   /root/reference/gaussian_renderer/__init__.py:14
 *       from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
 * constructed at :36-52 and called at :91-110.  The package's native side
 * (submodules/diff-gaussian-rasterization @ 59f5f77e: rasterize_points.cu, cuda_rasterizer/)
 * is an EMPTY directory in /root/reference, so no file:line exists for the pybind functions;
 * by name (BASELINE.json north_star) they are
 *   _C.rasterize_gaussians           -> gsb_forward
 *   _C.rasterize_gaussians_backward  -> gsb_backward
 *   _C.mark_visible                  -> gsb_mark_visible
 * The reference-side binding a maintainer adds is a ctypes stub: INTEGRATION.md.
 *
 * Conventions
 *  - all tensors float32, contiguous, on the device that is current when the call is made;
 *  - viewmatrix / projmatrix are the TRANSPOSED 4x4 matrices of scene/cameras.py:86-88,
 *    flattened row-major (element [r][c] at 4*r+c), i.e. p_view = [x y z 1] * viewmatrix;
 *  - shs is [P, sh_coeffs, 3]; sh_degree is the ACTIVE degree (0..3)
 *    (gaussian_renderer/__init__.py:45,76);
 *  - every kernel is enqueued on `stream`; the only host synchronisation is the read-back of
 *    the instance count inside gsb_forward;
 *  - memory is obtained through the caller's allocator so that it lives in the caller's pool
 *    (torch caching allocator): scratch is released by the caller after the call returns,
 *    GEOM / BINNING / IMAGE must stay alive until gsb_backward has been enqueued.
 */
#ifndef GS_B200_H
#define GS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSB_ABI_VERSION 6

/* error codes (0 = ok); gsb_last_error() holds the message of the calling thread's last failure */
#define GSB_OK 0
#define GSB_ERR_ARGUMENT 1
#define GSB_ERR_CUDA 2
#define GSB_ERR_ALLOC 3
#define GSB_ERR_OVERFLOW 4

/* buffer classes passed to the allocator */
#define GSB_BUF_GEOM 0     /* per-gaussian forward state, kept for backward   */
#define GSB_BUF_BINNING 1  /* sorted per-tile gaussian lists + tile ranges    */
#define GSB_BUF_IMAGE 2    /* per-pixel final transmittance + contributor count */
#define GSB_BUF_SCRATCH0 3 /* temporaries, may be freed when the call returns */
#define GSB_BUF_SCRATCH1 4
#define GSB_BUF_SCRATCH2 5

/* returns a device pointer aligned to >= 256 bytes, or NULL */
typedef void *(*gsb_alloc_fn)(void *ctx, int32_t which, size_t bytes);

/* the 13 fields of GaussianRasterizationSettings (gaussian_renderer/__init__.py:36-50)
 * plus the coefficient count of the shs tensor */
typedef struct GsbSettings {
    int32_t image_height;
    int32_t image_width;
    float tanfovx;
    float tanfovy;
    const float *bg;         /* device [3]  */
    float scale_modifier;
    const float *viewmatrix; /* device [16] */
    const float *projmatrix; /* device [16] */
    int32_t sh_degree;
    const float *campos;     /* device [3]  */
    int32_t prefiltered;
    int32_t debug;           /* !=0: synchronise + check after every kernel */
    int32_t antialiasing;
    int32_t sh_coeffs;       /* M of shs[P,M,3]; 0 when colors_precomp is given */
} GsbSettings;

/* arguments of GaussianRasterizer.forward (gaussian_renderer/__init__.py:102-110).
 * Exactly one of shs / colors_precomp and one of (scales+rotations) / cov3D_precomp is non-NULL. */
typedef struct GsbInputs {
    int32_t P;
    const float *means3D;        /* [P,3] */
    const float *shs;            /* [P,M,3] or NULL */
    const float *colors_precomp; /* [P,3] or NULL */
    const float *opacities;      /* [P] */
    const float *scales;         /* [P,3] or NULL */
    const float *rotations;      /* [P,4] or NULL */
    const float *cov3D_precomp;  /* [P,6] or NULL */
} GsbInputs;

/* forward state handed back to gsb_backward (plain data; the caller owns the three buffers) */
typedef struct GsbState {
    int32_t P;
    int32_t num_tiles;
    int64_t num_rendered;   /* D: (gaussian, tile) instances after exact tile culling */
    int64_t num_visible;    /* gaussians with radius > 0 (-1: not counted) */
    int64_t binning_capacity; /* instances the binning buffer was sized for (>= num_rendered) */
    void *geom;
    size_t geom_bytes;
    void *binning;
    size_t binning_bytes;
    void *image;
    size_t image_bytes;
    /* typed views into the buffers above (set by the forward call; the view-batch call packs V views per buffer) */
    const void *splat;        /* [P] 48-byte records */
    const uint32_t *point_list; /* [num_rendered] gaussian ids grouped by tile, depth-ordered inside a tile */
    const void *ranges;       /* [num_tiles] uint2 [begin, end) into point_list */
    const float *final_T;     /* [H*W] */
    const uint32_t *n_contrib; /* [H*W] */
    const void *tile_order;   /* [num_tiles] uint32 blend-launch order of the tiles, or NULL (option tile_order) */
} GsbState;

/* gradient outputs of the autograd.Function's backward; NULL pointers are skipped */
typedef struct GsbGrads {
    float *dL_dmeans3D;      /* [P,3] */
    float *dL_dmeans2D;      /* [P,3]  (x,y = gradient of the NDC 2D mean, z = 0) */
    float *dL_dshs;          /* [P,M,3] */
    float *dL_dcolors;       /* [P,3] */
    float *dL_dopacities;    /* [P] */
    float *dL_dscales;       /* [P,3] */
    float *dL_drotations;    /* [P,4] */
    float *dL_dcov3D;        /* [P,6] */
} GsbGrads;

/* Forward: preprocess -> depth sort -> tile binning -> tile sort -> tile ranges -> blend.
 * out_color [3,H,W], out_radii [P] int32, out_invdepth [H*W].
 * capacity_hint: the caller's estimate of the instance count (0 = none).  With an estimate the binning and
 * blend kernels are enqueued before the host waits for the true count, so the device never idles on the
 * read-back; if the true count exceeds the estimate the tail is re-run exactly (results never depend on it). */
int32_t gsb_forward(const GsbSettings *settings, const GsbInputs *in, float *out_color,
                    int32_t *out_radii, float *out_invdepth, int64_t capacity_hint, gsb_alloc_fn alloc,
                    void *alloc_ctx, GsbState *state_out, void *cuda_stream);

/* Backward.  out_color / out_invdepth are the forward call's outputs (the front-to-back backward blend
 * reads them); dL_dinvdepth may be NULL.  accumulate != 0 adds into the gradient tensors instead of
 * overwriting them (view-batch path: one buffer summed over views). */
int32_t gsb_backward(const GsbSettings *settings, const GsbInputs *in, const GsbState *state,
                     const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                     const float *dL_dinvdepth, const GsbGrads *grads, int32_t accumulate,
                     gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);

/* Split SH input: the DC coefficient and the remaining ones in two tensors (GaussianRasterizer.forward(dc=..., shs=...),
 * what scene.GaussianModel keeps as _features_dc / _features_rest), so no [P,M,3] concatenation is needed per view.
 *   dc [P,1,3];  rest [P,M-1,3], or NULL when M == 1;  settings->sh_coeffs = M counts both;  in->shs must be NULL.
 * Backward: dL_ddc [P,1,3] and dL_drest [P,M-1,3] receive the SH gradient (either may be NULL); grads->dL_dshs must be
 * NULL.  Single-view calls only; results are those of gsb_forward / gsb_backward on the concatenated tensor. */
typedef struct GsbSplitSH {
    const float *dc;
    const float *rest;
    float *dL_ddc;
    float *dL_drest;
} GsbSplitSH;
int32_t gsb_forward_split_sh(const GsbSettings *settings, const GsbInputs *in, const GsbSplitSH *split, float *out_color,
                             int32_t *out_radii, float *out_invdepth, int64_t capacity_hint, gsb_alloc_fn alloc,
                             void *alloc_ctx, GsbState *state_out, void *cuda_stream);
int32_t gsb_backward_split_sh(const GsbSettings *settings, const GsbInputs *in, const GsbSplitSH *split, const GsbState *state,
                              const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                              const float *dL_dinvdepth, const GsbGrads *grads, int32_t accumulate,
                              gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);

/* Camera gradients: gsb_backward (split == NULL) or gsb_backward_split_sh that also returns dL/d of the camera tensors of
 * `settings` (a learnable pose, a learnable background).  Every output is optional; with cam_grads NULL or all four fields
 * NULL the call is gsb_backward / gsb_backward_split_sh.  Outputs have the layout of the matching settings input (viewmatrix /
 * projmatrix: transposed, row-major, [r][c] at 4r+c) and are written (accumulate != 0: added to).  Conventions:
 *  - the gradient is that of the forward as computed: the 1.3x frustum clamp of x/z, y/z is a constant (no gradient through
 *    a clamped coordinate), the SH clamp to 0 and the anti-aliasing factor act as in dL/dmeans3D, and a gaussian that no
 *    pixel blended contributes nothing;
 *  - column 3 of the viewmatrix and column 2 of the projmatrix are never read by the forward: their gradient is 0;
 *  - dL/dcampos is 0 with colors_precomp (campos only enters through the SH view direction);
 *  - dL/dbg[c] = sum over pixels of final transmittance * dL/dcolor[c].
 * The per-gaussian terms are summed per warp inside the backward preprocess kernel and then over the warps by one small kernel
 * in a fixed order (no float atomics): repeated calls give identical bits.  No host synchronisation.
 * Not available on gsb_backward_batch_chunked / gsb_backward_batch_peer: the per-view sum would have to span the gaussian
 * chunks (which the caller consumes while later chunks run) or the ranks. */
typedef struct GsbCameraGrads {
    float *dL_dviewmatrix;  /* [16] (batch: [V,16]) or NULL, layout of the viewmatrix input */
    float *dL_dprojmatrix;  /* [16] (batch: [V,16]) or NULL */
    float *dL_dcampos;      /* [3]  (batch: [V,3])  or NULL */
    float *dL_dbg;          /* [3]  (batch: [V,3])  or NULL */
} GsbCameraGrads;
int32_t gsb_backward_camera(const GsbSettings *settings, const GsbInputs *in, const GsbSplitSH *split /* NULL = joint shs */,
                            const GsbState *state, const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                            const float *dL_dinvdepth, const GsbGrads *grads, const GsbCameraGrads *cam_grads, int32_t accumulate,
                            gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);

/* Rendered alpha (accumulated opacity), DESIGN.md section 7.6:
 *     alpha[p] = 1 - final_T[p]
 * where final_T is the transmittance after the last gaussian pixel p blended, under the forward's rules (the 1/255 cut-off,
 * the 0.99 cap, the T < 1e-4 stop): the final_T every forward call leaves in its state and uses for the background term, so
 * color = C_fg + (1 - alpha) * bg holds as computed.  Alpha does not depend on bg (dL/dbg of the camera gradient is unchanged
 * by an alpha loss); empty or fully culled scenes give alpha = 0 and zero gradients.
 *
 * gsb_alpha: out_alpha [V, height*width] from V forward states (states[v] of any forward call: single view, split SH, view
 * batch, async view batch; height x width must be their image size).  One launch, no host synchronisation.  It reads only the
 * states' IMAGE buffers, which must still be alive. */
int32_t gsb_alpha(int32_t V, const GsbState *states, int32_t height, int32_t width, float *out_alpha, void *cuda_stream);

/* Backward with a gradient on the rendered alpha: gsb_backward_camera (split NULL = joint shs; cam_grads NULL = no camera
 * gradient) plus dL_dalpha [H*W].  With dL_dalpha NULL the call is gsb_backward_camera: the same kernels are launched.  The
 * alpha term enters the per-gaussian gradients (means, opacity, scales / rotations or cov3D, means2D) and the camera
 * gradient; it adds nothing to the colour / SH gradients. */
int32_t gsb_backward_alpha(const GsbSettings *settings, const GsbInputs *in, const GsbSplitSH *split /* NULL = joint shs */,
                           const GsbState *state, const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                           const float *dL_dinvdepth, const float *dL_dalpha, const GsbGrads *grads,
                           const GsbCameraGrads *cam_grads, int32_t accumulate, gsb_alloc_fn alloc, void *alloc_ctx,
                           void *cuda_stream);
/* (view batch: gsb_backward_batch_alpha, after gsb_backward_batch_peer below) */

/* View-batch variants (DESIGN.md section 5): V <= 16 cameras of equal image size against the SAME gaussians.
 * The per-gaussian parameters are read once for all views (preprocess), the V depth sorts / scans / tile sorts
 * run as single batched launches, and there is ONE host read-back (V instance counts) per call.
 * out_color [V,3,H,W], out_radii [V,P], out_invdepth [V,H*W]; states[V] (buffers are shared, the typed views differ).
 * Backward: dL_dcolor [V,3,H,W], dL_dinvdepth [V,H*W] or NULL; every gradient in `grads` is the SUM over the V views
 * and is written once (accumulate != 0: added to the existing contents), except dL_dmeans2D which is [V,P,3]. */
int32_t gsb_forward_batch(int32_t V, const GsbSettings *settings, const GsbInputs *in, float *out_color,
                          int32_t *out_radii, float *out_invdepth, int64_t capacity_hint, gsb_alloc_fn alloc,
                          void *alloc_ctx, GsbState *states, void *cuda_stream);
int32_t gsb_backward_batch(int32_t V, const GsbSettings *settings, const GsbInputs *in, const GsbState *states,
                           const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                           const float *dL_dinvdepth, const GsbGrads *grads, int32_t accumulate,
                           gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);
/* gsb_backward_batch that also returns each view's camera gradient (GsbCameraGrads; outputs [V,16] / [V,3], one row per view). */
int32_t gsb_backward_batch_camera(int32_t V, const GsbSettings *settings, const GsbInputs *in, const GsbState *states,
                                  const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                                  const float *dL_dinvdepth, const GsbGrads *grads, const GsbCameraGrads *cam_grads,
                                  int32_t accumulate, gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);

/* gsb_forward_batch without ANY host synchronisation (what lets the host enqueue whole training steps ahead of the
 * device, and what a CUDA-graph capture of the step needs).  `capacity` (> 0) is the per-view instance capacity of the
 * binning buffers and is final: there is no read-back and no repair.  counts_dev: device array of 17 uint64 owned by the
 * caller; the call leaves the V instance counts in counts_dev[0..V) and folds them into the running maximum
 * counts_dev[16] (zero it once).  A view whose count exceeds `capacity` is rendered from a TRUNCATED list (no out-of-
 * bounds access): the caller polls counts_dev[16] whenever convenient (e.g. every N steps) and, if it ever exceeded the
 * capacity, discards those steps and re-runs them with a larger one.  states[v].num_rendered is -1 (device-only). */
int32_t gsb_forward_batch_async(int32_t V, const GsbSettings *settings, const GsbInputs *in, float *out_color,
                                int32_t *out_radii, float *out_invdepth, int64_t capacity, uint64_t *counts_dev,
                                gsb_alloc_fn alloc, void *alloc_ctx, GsbState *states, void *cuda_stream);

/* gsb_backward_batch with the last kernel (preprocess backward, which writes the gradient tensors) cut into n_chunks
 * gaussian ranges.  After chunk c has been ENQUEUED, on_chunk(ctx, c, p_begin, p_end) is called on the host: rows
 * [p_begin, p_end) of every gradient tensor are final once the work enqueued so far on the stream completes, so the
 * caller can record an event and start reducing that range on another stream (data-parallel all-reduce overlapped with
 * the remaining chunks).  on_chunk may be NULL. */
typedef void (*gsb_chunk_fn)(void *ctx, int32_t chunk, int32_t p_begin, int32_t p_end);
int32_t gsb_backward_batch_chunked(int32_t V, const GsbSettings *settings, const GsbInputs *in, const GsbState *states,
                                   const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                                   const float *dL_dinvdepth, const GsbGrads *grads, int32_t accumulate,
                                   int32_t n_chunks, gsb_chunk_fn on_chunk, void *chunk_ctx, gsb_alloc_fn alloc,
                                   void *alloc_ctx, void *cuda_stream);

/* FUSED REDUCE-SCATTER of the data-parallel gradients (one process per GPU of a node).  gsb_backward_batch whose last kernel does
 * not write this rank's gradient buffer but ADDS every row into the buffer of the rank that OWNS the row -- over NVLink, as TMA
 * bulk reduce-adds (one per 192-byte SH row, four per 128-gaussian block for the narrow tensors) issued while the kernel computes.
 * Rank r owns gaussians [r * rows_per_rank, (r + 1) * rows_per_rank); rows_per_rank is a multiple of 128 and
 * world * rows_per_rank >= P; every gradient tensor has world * rows_per_rank rows (the padding rows receive zeros).
 * `grads` points into THIS rank's buffer; base[r] is rank r's buffer as mapped into this process (gsb_peer_open), base[rank] the
 * local one, all with the same internal layout.  Protocol (caller): owners zero their rows; barrier; this call on every rank;
 * barrier; the owned rows now hold the sum over ranks -- all-gather them (or step the owned slice and all-gather parameters).
 * dL_dmeans2D (per-view, not reduced) is written locally as usual.  Needs option pre_tma (default) and SH tensors. */
typedef struct GsbPeerTable {
    int32_t world, rank;
    int32_t rows_per_rank;
    int32_t reserved;
    void *base[16];
} GsbPeerTable;
int32_t gsb_backward_batch_peer(int32_t V, const GsbSettings *settings, const GsbInputs *in, const GsbState *states,
                                const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                                const float *dL_dinvdepth, const GsbGrads *grads, const GsbPeerTable *peers,
                                gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);

/* View-batch backward with a gradient on the rendered alpha (see gsb_alpha), dL_dalpha [V, H*W] or NULL, in every mode of the
 * view-batch backward:
 *  - plain (n_chunks 1, on_chunk NULL, peers NULL): gsb_backward_batch, or gsb_backward_batch_camera with cam_grads;
 *  - n_chunks > 1 (1..64) or on_chunk != NULL: gsb_backward_batch_chunked;
 *  - peers != NULL: gsb_backward_batch_peer (the outputs are always added into the owners' buffers; accumulate is ignored).
 * cam_grads is not available with chunks or peers, as for the existing entry points.  With dL_dalpha NULL the call is the
 * matching existing entry point: the same kernels are launched. */
int32_t gsb_backward_batch_alpha(int32_t V, const GsbSettings *settings, const GsbInputs *in, const GsbState *states,
                                 const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                                 const float *dL_dinvdepth, const float *dL_dalpha, const GsbGrads *grads,
                                 const GsbCameraGrads *cam_grads, const GsbPeerTable *peers, int32_t accumulate,
                                 int32_t n_chunks, gsb_chunk_fn on_chunk, void *chunk_ctx, gsb_alloc_fn alloc,
                                 void *alloc_ctx, void *cuda_stream);

/* Rendered feature maps, DESIGN.md section 7.7: C view-independent per-gaussian channels composited with the forward's own
 * blend weights,
 *     F[c][p] = sum_k alpha_k T_k features[id_k][c]
 * under the forward's rules (the 1/255 cut-off, the 0.99 cap, the T < 1e-4 stop), with background 0 (composite with gsb_alpha
 * if needed).  Channels 3j..3j+2 equal, bit for bit, the colour output of the same gaussians rendered with colors_precomp =
 * features[:, 3j:3j+3] and bg = 0.  Channel counts 1..GSB_MAX_FEATURE_CHANNELS.
 *
 * gsb_render_features: out [V, channels, height*width] from V forward states (states[v] of any forward call: single view, split
 * SH, view batch, async view batch; P and height x width must be theirs) and features [P, channels].  One launch, no host
 * synchronisation; it reads the states' BINNING, GEOM and IMAGE buffers, which must still be alive.  features may be NULL
 * only when P == 0. */
#define GSB_MAX_FEATURE_CHANNELS 128
int32_t gsb_render_features(int32_t V, const GsbState *states, int32_t height, int32_t width, int32_t P, int32_t channels,
                            const float *features, float *out, void *cuda_stream);

/* Per-gaussian contribution statistics, DESIGN.md section 7.8: the usage scores of contribution-based pruning.  A forward state
 * accepts a pair (pixel p, gaussian k) exactly when gsb_render_features does (power <= 0, alpha >= 1/255, list position <=
 * n_contrib[p]); its blend weight is w_k(p) = alpha_k T_k, bit-equal to the weight of the blend.  Over the pixels of the V states:
 *     count[k]      (int64)   += number of accepted pairs
 *     weight_sum[k] (float32) += sum of w_k(p)
 *     weight_max[k] (float32)  = max(weight_max[k], max of w_k(p))
 * The outputs are ADDED into (max: max-ed into) so that views and calls accumulate; the caller zeroes them (weight_max >= 0
 * then, and stays 0 for a gaussian without an accepted pair).  count and weight_max are deterministic; weight_sum depends on
 * the order of float atomics.  The gaussian that would take T below 1e-4 is not blended and not counted.
 * states[v] of any forward call (single view, split SH, view batch, async view batch); P and height x width must be theirs.
 * One launch (none when P == 0), no host synchronisation; the states' BINNING, GEOM and IMAGE buffers must still be alive.
 * count 8-byte aligned, weight_sum / weight_max 4-byte aligned; they may be NULL only when P == 0. */
int32_t gsb_contribution(int32_t V, const GsbState *states, int32_t height, int32_t width, int32_t P, int64_t *count,
                         float *weight_sum, float *weight_max, void *cuda_stream);

/* The feature term of a backward call.  NULL pointers: no feature loss (dL_dout_features) or no feature gradient
 * (dL_dfeatures).  A NULL features pointer together with a non-NULL output is an error (unless P == 0). */
typedef struct GsbFeatures {
    int32_t channels;                /* C, 1..GSB_MAX_FEATURE_CHANNELS */
    const float *features;           /* [P, C], as given to gsb_render_features */
    const float *out_features;       /* [V, C, H*W]: gsb_render_features' output for these states */
    const float *dL_dout_features;   /* [V, C, H*W] or NULL */
    float *dL_dfeatures;             /* [P, C] or NULL: written (added with accumulate), summed over the views */
} GsbFeatures;

/* Backward with a feature term: gsb_backward_alpha (split NULL = joint shs, cam_grads NULL = no camera gradient, dL_dalpha
 * NULL = no alpha term) plus `features`.  The feature loss enters the per-gaussian gradients (means, opacity, scales /
 * rotations or cov3D, means2D), the camera gradient and dL_dfeatures; it adds nothing to the colour / SH gradients or dL/dbg.
 * With features NULL the call is gsb_backward_alpha: the same kernels are launched.  Otherwise one more launch, after the
 * colour pass, when dL_dout_features is given and the state holds instances. */
int32_t gsb_backward_features(const GsbSettings *settings, const GsbInputs *in, const GsbSplitSH *split /* NULL = joint shs */,
                              const GsbState *state, const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                              const float *dL_dinvdepth, const float *dL_dalpha, const GsbGrads *grads,
                              const GsbCameraGrads *cam_grads, const GsbFeatures *features, int32_t accumulate,
                              gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);

/* View-batch backward with a feature term: gsb_backward_batch_alpha plus `features` (out_features / dL_dout_features
 * [V, C, H*W]; dL_dfeatures [P, C] is the sum over the views).  With features NULL the call is gsb_backward_batch_alpha in
 * every mode.  With features, only the plain and camera modes exist: n_chunks > 1, on_chunk or peers return
 * GSB_ERR_ARGUMENT.  As with camera gradients, those protocols cover the per-gaussian gradient rows of GsbGrads only:
 * dL_dfeatures is neither handed out chunk by chunk nor added into the owner ranks' buffers. */
int32_t gsb_backward_batch_features(int32_t V, const GsbSettings *settings, const GsbInputs *in, const GsbState *states,
                                    const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                                    const float *dL_dinvdepth, const float *dL_dalpha, const GsbGrads *grads,
                                    const GsbCameraGrads *cam_grads, const GsbFeatures *features, const GsbPeerTable *peers,
                                    int32_t accumulate, int32_t n_chunks, gsb_chunk_fn on_chunk, void *chunk_ctx,
                                    gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);

/* Lets kernels launched on the CURRENT device dereference pointers into `peer_device`'s memory (cudaDeviceEnablePeerAccess;
 * already-enabled is not an error).  Needed once per peer before gsb_backward_batch_peer is given peer-mapped buffers. */
int32_t gsb_enable_peer_access(int32_t peer_device);
/* Peer-visible device memory for the ranks of one node (one process per GPU).  gsb_peer_alloc: cudaMalloc (zero-filled) on the
 * current device + its 64-byte CUDA-IPC handle, which the caller ships to the other processes by any means; gsb_peer_open: maps
 * another process's allocation into this one, on the current device (the device whose kernels will use it); _close / _free undo. */
int32_t gsb_peer_alloc(size_t bytes, void **ptr, uint8_t *handle64);
int32_t gsb_peer_open(const uint8_t *handle64, void **ptr);
int32_t gsb_peer_close(void *ptr);
int32_t gsb_peer_free(void *ptr);

/* Frustum test only (GaussianRasterizer.markVisible): present[i] = 1 if view-space z > 0.2 */
int32_t gsb_mark_visible(int32_t P, const float *means3D, const float *viewmatrix,
                         const float *projmatrix, uint8_t *present, void *cuda_stream);

/* Stand-alone stable LSD radix sort of (u32 key, u32 value) pairs on bits [begin_bit,end_bit):
 * the replacement of the reference's cub::DeviceRadixSort call, exported for tests.
 * keys/vals are overwritten with the sorted result; scratch is obtained through alloc. */
int32_t gsb_sort_pairs(uint32_t *keys, uint32_t *vals, int64_t n, int32_t begin_bit, int32_t end_bit,
                       gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);

/* Fused L1 photometric loss of the step after the path (train.py:120-126 with render()'s clamp,
 * gaussian_renderer/__init__.py:119): *loss_accum += scale * sum |clamp(image,0,1) - target| and
 * grad_out = d(that)/d(image).  n (elements) must be a multiple of 4; pointers 16-byte aligned. */
int32_t gsb_l1_loss_grad(const float *image, const float *target, int64_t n, float scale, float *grad_out,
                         float *loss_accum, void *cuda_stream);

/* The reference training step's photometric loss fused with its gradient (SURVEY.md section 8(f) #2):
 *   loss = (1 - lambda) * mean|x - y| + lambda * (1 - SSIM(x, y)),  x = clamp(image, 0, 1) when clamp_input != 0 (render()'s
 *   clamp, gaussian_renderer/__init__.py:119, with its gradient mask) and x = image otherwise (the fused_ssim drop-in)
 * (train.py:120-126, utils/loss_utils.py:40-86; 11x11 gaussian window, sigma 1.5, zero padding).  image / target are
 * [channels, height, width]; grad_out = d loss / d image; loss_accum[0] += loss - lambda (add lambda on the host side,
 * or pre-load it), loss_accum[1] += sum|x - y| * (1-lambda > 0), loss_accum[2] += sum of the SSIM map. */
int32_t gsb_photometric_loss_grad(const float *image, const float *target, int32_t channels, int32_t height,
                                  int32_t width, float lambda_dssim, int32_t clamp_input, float *grad_out,
                                  float *loss_accum, gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream);

/* ---- Training state around the path (SURVEY.md section 8(f) rows 3 and 1) -------------------------------------
 * The gaussians' RAW parameters live in ONE flat float buffer ("store"), group after group, each group [P, width]
 * row-major.  With M = sh_coeffs:
 *     xyz [P,3] | features [P,M,3] (row 0 = f_dc, rows 1.. = f_rest) | opacity [P,1] | scaling [P,3] | rotation [P,4]
 * = (11 + 3M) floats per gaussian (59 at SH degree 3).  Gradients, exp_avg and exp_avg_sq use the same layout, so the
 * data-parallel reduction is one all-reduce of one buffer and the optimizer is one launch.  The gradient buffer holds
 * dLoss/d(ACTIVATED value) -- exactly what gsb_backward writes -- for the activations of scene/gaussian_model.py:33-46:
 * identity (xyz, features), sigmoid (opacity), exp (scaling), normalize (rotation).
 * `act` (8 floats per gaussian: sigmoid(opacity)[P] | exp(scaling)[P,3] | normalize(rotation)[P,4]) are the activated
 * tensors the rasterizer reads; the optimizer rewrites them, so no separate activation pass runs between steps. */
typedef struct GsbAdamArgs {
    int64_t P;
    int32_t sh_coeffs;
    int32_t skip_groups;      /* bit g set: group g (order below) is left untouched -- the reference's optimizer.step() skips a
                                 parameter that densify_and_prune / reset_opacity has just replaced (its .grad is None) */
    float *params;            /* store, updated in place */
    const float *grads;       /* dLoss/d activated, same layout */
    float *exp_avg;
    float *exp_avg_sq;
    float *act;               /* rewritten from the updated parameters; may be NULL */
    const uint8_t *visible;   /* NULL = every gaussian; else rows with visible[i] == 0 are left untouched */
    float step_size[6];       /* lr_g / (1 - beta1^t_g) for xyz, f_dc, f_rest, opacity, scaling, rotation */
    float bias2_sqrt[6];      /* sqrt(1 - beta2^t_g); t_g is the group's OWN step count (torch.optim.Adam keeps one per parameter) */
    float beta1, beta2, eps;
} GsbAdamArgs;

/* torch.optim.Adam (no weight decay, no amsgrad; scene/gaussian_model.py:176-199, train.py:178-186) over the six parameter
 * groups in one launch, with the activation backward (autograd's part in the reference) and the re-activation fused in:
 *   g_raw = J_act^T g;  m += (1-b1)(g_raw - m);  v = b2 v + (1-b2) g_raw^2;  p -= step_size * m / (sqrt(v)/bias2_sqrt + eps) */
int32_t gsb_adam_step(const GsbAdamArgs *args, void *cuda_stream);

/* SparseGaussianAdam (train.py --optimizer_type sparse_adam) over separate per-parameter tensors: every group is [N, width]
 * row-major, float32, contiguous; param / grad / exp_avg / exp_avg_sq of one group share the layout.  Rows with
 * visible[i] == 0 are neither read nor written.  Visible rows take the update of gsb_adam_step with step_size = lr and
 * bias2_sqrt = 1 (no bias correction):
 *   m += (1-b1)(g - m);  v = b2 v + (1-b2) g^2;  p -= lr * m / (sqrt(v) + eps)
 * One launch for 1..GSB_MAX_SPARSE_GROUPS groups; no host synchronisation. */
#define GSB_MAX_SPARSE_GROUPS 8
typedef struct GsbSparseAdamGroup {
    float *param;
    const float *grad;
    float *exp_avg;
    float *exp_avg_sq;
    int32_t width;            /* floats per row (> 0) */
    float lr;
    float eps;
} GsbSparseAdamGroup;
int32_t gsb_sparse_adam_step(const GsbSparseAdamGroup *groups, int32_t n_groups, const uint8_t *visible, int64_t N,
                             float beta1, float beta2, void *cuda_stream);

/* act <- activations of the store (after initialisation, densification or an opacity reset) */
int32_t gsb_activate(int64_t P, int32_t sh_coeffs, const float *params, float *act, void *cuda_stream);

/* densify_and_prune (scene/gaussian_model.py:399-469) as a plan (classification + two scans; one host read-back) and one
 * gather that writes the new store and its Adam moments.  Row order of the result is the reference's:
 *   surviving originals | surviving clones | surviving children, copy-major (child k of the j-th split gaussian at k*n_split + j)
 * Survivors keep their moments, new rows start at zero (:359-397).  Every threshold is passed in already multiplied out:
 *   clone  if mean grad >= grad_threshold and max(exp(scaling)) <= size_limit   (size_limit = percent_dense * extent)
 *   split  if mean grad >= grad_threshold and max(exp(scaling)) >  size_limit   (children: scaling / (0.8 * n_children))
 *   prune  if sigmoid(opacity) < min_opacity, or (world_limit >= 0 and max(exp(scaling)) > world_limit = 0.1 * extent)
 * The screen-size test of :462 never fires in the reference (max_radii2D is zeroed by densification_postfix first) and
 * is therefore absent.  grad_threshold must be > 0 (a clone is never split). */
typedef struct GsbDensifyArgs {
    int64_t P;
    int32_t sh_coeffs;
    int32_t n_children;       /* 2 in the reference */
    const float *params;      /* old store and moments */
    const float *exp_avg;
    const float *exp_avg_sq;
    const float *grad_accum;  /* [P] accumulated view-space gradient norm */
    const float *denom;       /* [P] how many views accumulated */
    float grad_threshold, size_limit, min_opacity, world_limit;
    void *scratch;            /* gsb_densify_scratch_bytes(P, n_children) bytes; written by plan, read by apply */
} GsbDensifyArgs;
size_t gsb_densify_scratch_bytes(int64_t P, int32_t n_children);
/* counts = { n_clone, n_split, n_pruned, P_new }.  Synchronises the stream once (the caller needs n_split to draw the
 * samples and P_new to size the new store -- the reference synchronises a dozen times here). */
int32_t gsb_densify_plan(const GsbDensifyArgs *args, int64_t counts[4], void *cuda_stream);
/* unit_samples: [n_children * n_split, 3] standard normals (the draw of torch.normal at :409). */
int32_t gsb_densify_apply(const GsbDensifyArgs *args, const float *unit_samples, int64_t n_split, int64_t P_new,
                          float *new_params, float *new_exp_avg, float *new_exp_avg_sq, void *cuda_stream);

/* prune_points(mask) (scene/gaussian_model.py:349-364) on the store: rows with remove[i] != 0 go, the survivors keep their order
 * and their Adam moments.  scratch: gsb_densify_scratch_bytes(P, 1) bytes, written by plan and read by apply.
 * gsb_prune_plan: keep flags, their exclusive scan and the source row of every output row; *P_new = survivors.  Synchronises
 *   the stream once (the caller sizes the new store with P_new).
 * gsb_prune_apply: one gather of the kept rows into new_params / new_exp_avg / new_exp_avg_sq (store layout of P_new rows). */
int32_t gsb_prune_plan(int64_t P, const uint8_t *remove, void *scratch, int64_t *P_new, void *cuda_stream);
int32_t gsb_prune_apply(int64_t P, int32_t sh_coeffs, const float *params, const float *exp_avg, const float *exp_avg_sq,
                        const void *scratch, int64_t P_new, float *new_params, float *new_exp_avg, float *new_exp_avg_sq,
                        void *cuda_stream);

/* Mean squared distance from every point to its three nearest other points: the replacement of
 * simple_knn._C.distCUDA2 (scene/gaussian_model.py:21,159 -- initial scales).  points [P,3], out [P]; exact (uniform grid
 * sized on the device, no host synchronisation); scratch through alloc. */
int32_t gsb_knn_mean_dist2(const float *points, int64_t P, float *out, gsb_alloc_fn alloc, void *alloc_ctx,
                           void *cuda_stream);

const char *gsb_last_error(void);
int32_t gsb_abi_version(void);
/* number of kernels this library has launched in this process since the last reset */
int64_t gsb_launch_count(void);
void gsb_reset_launch_count(void);
/* CUDA-event time of the launches of kernel `name` ("" = all) recorded on their launching stream since
 * the last reset, while option "time_kernels" was 1 (blend kernels) or 2 (all).  Synchronises on the events. */
int32_t gsb_kernel_time(const char *name, double *total_ms, int64_t *launches, int32_t reset);
/* Deterministic backward switch of the CALLING HOST THREAD (off by default); returns the previous value.  Per thread
 * because autograd runs CUDA backwards on its own device threads.  While it is on, every gradient output of every backward
 * entry point (single view, split SH, camera, alpha; view batch plain, camera, chunked, after a sync or async forward) is a
 * function of the forward state and the loss gradients alone: the blend kernel stores its per-(list entry, warp) sums
 * instead of adding them with float atomics, and they are summed per gaussian in ascending list order.  Repeating a call
 * gives identical bits whatever the CTA scheduling, the "tile_order" option or the chunking.  The values differ from the
 * default path only by float reassociation.  Costs 4 + ceil(ceil(log2 P) / 8) kernel launches more per call and scratch
 * (GSB_BUF_SCRATCH2) of about 114 bytes per instance of the forward's capacity, per view.
 * No deterministic implementation, GSB_ERR_ARGUMENT while it is on: a feature term with a feature-map gradient
 * (gsb_backward_features, gsb_backward_batch_features) and peers (gsb_backward_batch_peer, gsb_backward_batch_alpha /
 * _features with a peer table).  Not covered (float atomics, whatever the switch): gsb_contribution's weight_sum and the
 * loss scalars of gsb_l1_loss_grad / gsb_photometric_loss_grad (their gradients are per pixel and deterministic). */
int32_t gsb_set_deterministic(int32_t on);
/* tuning knobs (integers): "cull", "sort_small", "tile_order", "pre_tma", "time_kernels"; returns 0 if known */
int32_t gsb_set_option(const char *name, int32_t value);

#ifdef __cplusplus
}
#endif
#endif /* GS_B200_H */
