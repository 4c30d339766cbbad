// abi.cu -- extern "C" entry points of libgs_b200.so (include/gs_b200.h) and the host-side
// orchestration of the forward / backward kernel sequences.
#include <stdarg.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "kernels.cuh"

namespace gsb {

static thread_local char g_err[512] = "";
static thread_local int g_deterministic = 0;    // gsb_set_deterministic: per host thread, like the last error
int64_t g_launch_count = 0;

int g_time_kernels = 0;

// ---- kernel timing records ----
struct TimerRec { char name[32]; cudaEvent_t e0, e1; };
static std::vector<TimerRec *> g_timer_recs;
static std::mutex g_timer_mutex;

void *timer_begin(const char *name, cudaStream_t stream) {
    if (g_time_kernels == 1 && strncmp(name, "render_", 7) != 0) return nullptr;
    TimerRec *r = new TimerRec();
    strncpy(r->name, name, sizeof(r->name) - 1);
    r->name[sizeof(r->name) - 1] = 0;
    if (cudaEventCreate(&r->e0) != cudaSuccess || cudaEventCreate(&r->e1) != cudaSuccess) { delete r; return nullptr; }
    cudaEventRecord(r->e0, stream);
    return r;
}

void timer_end(void *token, cudaStream_t stream) {
    TimerRec *r = static_cast<TimerRec *>(token);
    cudaEventRecord(r->e1, stream);
    std::lock_guard<std::mutex> lock(g_timer_mutex);
    g_timer_recs.push_back(r);
}

static int opt_cull = 1;
static int opt_tile_order = 1;    // blend CTAs take the tiles by descending list length (render.cu tile_order_kernel), so that the
                                  // heavy tiles start in the first wave and the light ones fill the tail of the launch; 0 = off

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_launch(const char *what, bool debug, cudaStream_t stream) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && debug) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) {
        set_error("kernel %s failed: %s", what, cudaGetErrorString(e));
        return GSB_ERR_CUDA;
    }
    return GSB_OK;
}

// pinned read-back slot for the instance count: one per (host thread, device), created on first use, so that two host
// threads driving the same device (a viewer next to the training thread) never share a slot or its event
static unsigned long long *pinned_slot() {
    static thread_local unsigned long long *slots[64] = {nullptr};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    if (!slots[dev]) {
        void *p = nullptr;
        if (cudaHostAlloc(&p, 256, cudaHostAllocDefault) != cudaSuccess) return nullptr;
        slots[dev] = static_cast<unsigned long long *>(p);
    }
    return slots[dev];
}

static cudaEvent_t readback_event() {
    static thread_local cudaEvent_t evs[64] = {nullptr};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    if (!evs[dev] && cudaEventCreateWithFlags(&evs[dev], cudaEventDisableTiming) != cudaSuccess) return nullptr;
    return evs[dev];
}

static int bits_for(uint32_t max_value) {
    int b = 1;
    while (b < 32 && (max_value >> b) != 0u) ++b;
    return b;
}

static int make_cam(const GsbSettings *s, CamArgs &c) {
    if (!s->bg || !s->viewmatrix || !s->projmatrix || !s->campos) {
        set_error("settings: bg / viewmatrix / projmatrix / campos must be device pointers");
        return GSB_ERR_ARGUMENT;
    }
    if (s->image_width <= 0 || s->image_height <= 0 || s->image_width > 16 * 65535 || s->image_height > 16 * 65535) {
        set_error("settings: bad image size %d x %d", s->image_width, s->image_height);
        return GSB_ERR_ARGUMENT;
    }
    if (s->sh_degree < 0 || s->sh_degree > 3) {
        set_error("settings: sh_degree %d outside 0..3", s->sh_degree);
        return GSB_ERR_ARGUMENT;
    }
    c.view = s->viewmatrix; c.proj = s->projmatrix; c.campos = s->campos; c.bg = s->bg;
    c.tanfovx = s->tanfovx; c.tanfovy = s->tanfovy;
    c.W = s->image_width; c.H = s->image_height;
    c.focal_x = c.W / (2.0f * s->tanfovx);
    c.focal_y = c.H / (2.0f * s->tanfovy);
    c.scale_modifier = s->scale_modifier;
    c.gx = (c.W + TILE - 1) / TILE; c.gy = (c.H + TILE - 1) / TILE;
    c.sh_degree = s->sh_degree; c.sh_coeffs = s->sh_coeffs; c.antialiasing = s->antialiasing;
    return GSB_OK;
}

// split: the split SH input of gsb_forward_split_sh / gsb_backward_split_sh (its dc takes the place of in->shs), or NULL
static int check_inputs(const GsbSettings *s, const GsbInputs *in, const GsbSplitSH *split = nullptr) {
    if (in->P < 0) { set_error("inputs: P < 0"); return GSB_ERR_ARGUMENT; }
    if (in->P > 0 && (!in->means3D || !in->opacities)) { set_error("inputs: means3D / opacities missing"); return GSB_ERR_ARGUMENT; }
    if (split) {
        if (in->shs) { set_error("split SH input: in->shs must be NULL (dc and rest carry the coefficients)"); return GSB_ERR_ARGUMENT; }
        if (split->dc && in->colors_precomp) { set_error("split SH input: dc given together with colors_precomp"); return GSB_ERR_ARGUMENT; }
        if (split->rest && s->sh_coeffs == 1) { set_error("split SH input: rest given with sh_coeffs == 1"); return GSB_ERR_ARGUMENT; }
        if (in->P > 0 && split->dc && !split->rest && s->sh_coeffs > 1) {
            set_error("split SH input: rest missing for sh_coeffs == %d", s->sh_coeffs);
            return GSB_ERR_ARGUMENT;
        }
    }
    const float *sh = split ? split->dc : in->shs;
    if (in->P > 0 && ((sh != nullptr) == (in->colors_precomp != nullptr))) {
        set_error("inputs: provide exactly one of shs / colors_precomp");
        return GSB_ERR_ARGUMENT;
    }
    const bool sr = in->scales != nullptr && in->rotations != nullptr;
    if (in->P > 0 && (sr == (in->cov3D_precomp != nullptr))) {
        set_error("inputs: provide exactly one of (scales, rotations) / cov3D_precomp");
        return GSB_ERR_ARGUMENT;
    }
    if (sh && s->sh_coeffs < (s->sh_degree + 1) * (s->sh_degree + 1)) {
        set_error("inputs: shs has %d coefficients, degree %d needs %d", s->sh_coeffs, s->sh_degree,
                  (s->sh_degree + 1) * (s->sh_degree + 1));
        return GSB_ERR_ARGUMENT;
    }
    return GSB_OK;
}

// camera gradient outputs: NULL (or every field NULL) = not requested; a requested output must be a 4-byte aligned pointer
static int check_cam_grads(const char *fn, const GsbCameraGrads *cg, bool &want) {
    want = false;
    if (!cg) return GSB_OK;
    float *const outs[4] = {cg->dL_dviewmatrix, cg->dL_dprojmatrix, cg->dL_dcampos, cg->dL_dbg};
    for (float *p : outs) {
        if (!p) continue;
        if (reinterpret_cast<size_t>(p) & 3) {
            set_error("%s: camera gradient outputs must be 4-byte aligned float pointers", fn);
            return GSB_ERR_ARGUMENT;
        }
        want = true;
    }
    return GSB_OK;
}

static void *do_alloc(gsb_alloc_fn alloc, void *ctx, int which, size_t bytes) {
    void *p = alloc(ctx, which, bytes < 256 ? 256 : bytes);
    if (!p) set_error("allocator returned NULL for buffer %d (%zu bytes)", which, bytes);
    return p;
}

struct ImageView { float *final_T; uint32_t *n_contrib; };
static size_t carve_image(void *base, size_t npix, ImageView &v) {
    Carver c(base);
    v.final_T = c.take<float>(npix);
    v.n_contrib = c.take<uint32_t>(npix);
    return c.bytes();
}
struct BinningView { uint32_t *point_list; uint2 *ranges; uint32_t *tile_order; };
static size_t carve_binning(void *base, int64_t D, int num_tiles, BinningView &v) {
    Carver c(base);
    v.point_list = c.take<uint32_t>((size_t)(D > 0 ? D : 1));
    v.ranges = c.take<uint2>((size_t)num_tiles);
    v.tile_order = c.take<uint32_t>((size_t)num_tiles);
    return c.bytes();
}

}  // namespace gsb

using namespace gsb;

extern "C" {

const char *gsb_last_error(void) { return g_err; }
int32_t gsb_abi_version(void) { return GSB_ABI_VERSION; }
int32_t gsb_set_deterministic(int32_t on) {
    const int32_t prev = g_deterministic;
    g_deterministic = on != 0;
    return prev;
}
int64_t gsb_launch_count(void) { return g_launch_count; }
void gsb_reset_launch_count(void) { g_launch_count = 0; }

int32_t gsb_set_option(const char *name, int32_t value) {
    if (!name) return 1;
    if (!strcmp(name, "cull")) { opt_cull = value; return 0; }
    if (!strcmp(name, "time_kernels")) { g_time_kernels = value; return 0; }
    if (!strcmp(name, "sort_small")) { g_sort_force_small = value; return 0; }
    if (!strcmp(name, "tile_order")) { opt_tile_order = value; return 0; }
    if (!strcmp(name, "pre_tma")) { g_pre_tma = value; return 0; }
    return 1;
}

int32_t gsb_kernel_time(const char *name, double *total_ms, int64_t *launches, int32_t reset) {
    // waits for the recorded events; name == NULL or "" sums every kernel
    std::lock_guard<std::mutex> lock(g_timer_mutex);
    double ms = 0.0;
    int64_t n = 0;
    for (TimerRec *r : g_timer_recs) {
        if (name && name[0] && strcmp(name, r->name) != 0) continue;
        float t = 0.f;
        if (cudaEventSynchronize(r->e1) == cudaSuccess && cudaEventElapsedTime(&t, r->e0, r->e1) == cudaSuccess) {
            ms += t;
            ++n;
        }
    }
    if (reset) {
        for (TimerRec *r : g_timer_recs) { cudaEventDestroy(r->e0); cudaEventDestroy(r->e1); delete r; }
        g_timer_recs.clear();
    }
    if (total_ms) *total_ms = ms;
    if (launches) *launches = n;
    return GSB_OK;
}

// optional heavy-tiles-first permutation for the blend launches (option tile_order); lives behind the tile ranges in BINNING
static int maybe_tile_order(const uint2 *ranges, int V, int num_tiles, uint32_t *order, bool debug, cudaStream_t stream) {
    if (!opt_tile_order) return GSB_OK;
    return launch_tile_order(ranges, V, num_tiles, order, debug, stream);
}

// shared body of gsb_forward (split == NULL) and gsb_forward_split_sh
static int forward_impl(const char *fn, const GsbSettings *s, const GsbInputs *in, const GsbSplitSH *split, float *out_color,
                        int32_t *out_radii, float *out_invdepth, int64_t capacity_hint, gsb_alloc_fn alloc, void *alloc_ctx,
                        GsbState *st, void *cuda_stream) {
    if (!s || !in || !out_color || (!out_radii && in->P > 0) || !out_invdepth || !alloc || !st) {
        set_error("%s: NULL argument", fn);
        return GSB_ERR_ARGUMENT;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    const bool debug = s->debug != 0;
    CamArgs cam;
    int rc = make_cam(s, cam);
    if (rc) return rc;
    rc = check_inputs(s, in, split);
    if (rc) return rc;
    const int P = in->P;
    const int num_tiles = cam.gx * cam.gy;
    const int tile_bits = bits_for((uint32_t)num_tiles);
    const size_t npix = (size_t)cam.W * cam.H;
    memset(st, 0, sizeof(*st));
    st->P = P; st->num_tiles = num_tiles; st->num_visible = -1;

    // ---- per-gaussian state ----
    const size_t Pn = (size_t)(P > 0 ? P : 1);
    st->geom_bytes = align_up(Pn * SPLAT_F4 * sizeof(float4), 256);
    st->geom = do_alloc(alloc, alloc_ctx, GSB_BUF_GEOM, st->geom_bytes);
    if (!st->geom) return GSB_ERR_ALLOC;
    float4 *splat = static_cast<float4 *>(st->geom);

    // ---- per-pixel state (allocated up front so that nothing host-side sits between binning and blending) ----
    ImageView iv;
    st->image_bytes = carve_image(nullptr, npix, iv);
    st->image = do_alloc(alloc, alloc_ctx, GSB_BUF_IMAGE, st->image_bytes);
    if (!st->image) return GSB_ERR_ALLOC;
    carve_image(st->image, npix, iv);

    uint32_t *key, *idx, *key_alt, *idx_alt, *tiles, *offsets; uint2 *rect; unsigned long long *scan_state, *total; char *sortscr;
    auto carve0 = [&](Carver &c) {
        key = c.take<uint32_t>(Pn); idx = c.take<uint32_t>(Pn); key_alt = c.take<uint32_t>(Pn); idx_alt = c.take<uint32_t>(Pn);
        tiles = c.take<uint32_t>(Pn); rect = c.take<uint2>(Pn); offsets = c.take<uint32_t>(Pn);
        scan_state = c.take<unsigned long long>(scan_state_count(P)); total = c.take<unsigned long long>(4);
        sortscr = c.take<char>(sort_scratch_bytes(P));
    };
    Carver c0(nullptr);
    carve0(c0);
    void *scr0 = do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH0, c0.bytes());
    if (!scr0) return GSB_ERR_ALLOC;
    Carver c0r(scr0);
    carve0(c0r);

    BinArgs ba;
    ba.P = P; ba.num_tiles = num_tiles; ba.gx = cam.gx; ba.order = idx; ba.tiles = tiles; ba.rect = rect; ba.splat = splat;
    ba.offsets = offsets; ba.scan_state = scan_state; ba.total = total;
    ba.sv_gauss = 0; ba.sv_splat = 0; ba.sv_scan = 0; ba.sv_inst = 0;
    st->splat = splat; st->final_T = iv.final_T; st->n_contrib = iv.n_contrib;

    // binning + blend for an instance capacity `cap`; the true count is read by the kernels from *n_dev when given
    BinningView bv;
    auto bin_and_blend = [&](int64_t cap, const unsigned long long *n_dev) -> int {
        st->binning_capacity = cap;
        st->binning_bytes = carve_binning(nullptr, cap, num_tiles, bv);
        st->binning = do_alloc(alloc, alloc_ctx, GSB_BUF_BINNING, st->binning_bytes);
        if (!st->binning) return GSB_ERR_ALLOC;
        carve_binning(st->binning, cap, num_tiles, bv);
        st->point_list = bv.point_list; st->ranges = bv.ranges; st->tile_order = opt_tile_order ? bv.tile_order : nullptr;
        int r;
        if (cap > 0 && P > 0) {
            const size_t Dn = (size_t)cap;
            Carver c1(nullptr);
            c1.take<uint32_t>(Dn); c1.take<uint32_t>(Dn); c1.take<uint32_t>(Dn); c1.take<char>(sort_scratch_bytes(cap));
            void *scr1 = do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH1, c1.bytes());
            if (!scr1) return GSB_ERR_ALLOC;
            Carver c1r(scr1);
            uint32_t *inst_tile = c1r.take<uint32_t>(Dn), *inst_tile_alt = c1r.take<uint32_t>(Dn), *inst_gauss_alt = c1r.take<uint32_t>(Dn);
            char *sortscr1 = c1r.take<char>(sort_scratch_bytes(cap));
            SortDigits dg;
            r = sort_prepare(cap, 1, 0, tile_bits, sortscr1, stream, &dg);
            if (r) return r;
            r = launch_emit(ba, 1, inst_tile, bv.point_list, cap, dg, debug, stream);
            if (r) return r;
            r = sort_pairs(inst_tile, bv.point_list, inst_tile_alt, inst_gauss_alt, cap, n_dev, 0, tile_bits, sortscr1, debug, stream, 1, 0,
                           true);
            if (r) return r;
            r = launch_tile_ranges(inst_tile, cap, n_dev, num_tiles, bv.ranges, 1, 0, debug, stream);
            if (r) return r;
        } else {
            r = launch_tile_ranges(nullptr, 0, nullptr, num_tiles, bv.ranges, 1, 0, debug, stream);
            if (r) return r;
        }
        r = maybe_tile_order(bv.ranges, 1, num_tiles, bv.tile_order, debug, stream);
        if (r) return r;
        RenderFwdArgs ra;
        memset(&ra, 0, sizeof(ra));
        ra.W = cam.W; ra.H = cam.H; ra.gx = cam.gx; ra.gy = cam.gy; ra.V = 1;
        ra.ranges = bv.ranges; ra.point_list = bv.point_list; ra.tile_order = static_cast<const uint32_t *>(st->tile_order);
        ra.splat = splat; ra.bg[0] = s->bg; ra.out_color = out_color; ra.out_invdepth = out_invdepth; ra.final_T = iv.final_T;
        ra.n_contrib = iv.n_contrib;
        return launch_render_fwd(ra, debug, stream);
    };

    int64_t D = 0;
    if (P > 0) {
        PreFwdArgs pa;
        pa.P = P; pa.means = in->means3D; pa.shs = split ? split->dc : in->shs; pa.colors = in->colors_precomp; pa.opac = in->opacities;
        pa.scales = in->scales; pa.rots = in->rotations; pa.cov_pre = in->cov3D_precomp;
        pa.rest = split ? split->rest : nullptr;
        pa.splat = splat; pa.depth_key = key; pa.depth_idx = idx; pa.tiles = tiles; pa.rect = rect; pa.radii = out_radii;
        pa.cull = opt_cull;
        rc = launch_preprocess_fwd(cam, pa, split != nullptr, debug, stream);
        if (rc) return rc;
        // gaussians by depth (culled ones carry key 0xffffffff and sort to the end)
        rc = sort_pairs(key, idx, key_alt, idx_alt, P, nullptr, 0, 32, sortscr, debug, stream);
        if (rc) return rc;
        rc = launch_tile_scan(ba, 1, debug, stream);
        if (rc) return rc;
        // The instance count D sizes the binning buffers, so it has to reach the host: ONE read-back per forward.
        unsigned long long *h = pinned_slot();
        cudaEvent_t ev = readback_event();
        if (!h || !ev) { set_error("pinned read-back slot unavailable"); return GSB_ERR_CUDA; }
        GSB_CUDA(cudaMemcpyAsync(h, total, sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
        GSB_CUDA(cudaEventRecord(ev, stream));
        bool blended = false;
        if (capacity_hint > 0 && capacity_hint < (1ll << 31)) {
            // Speculate: with the caller's capacity estimate (e.g. the previous frame's count plus slack) the rest of
            // the forward pass is enqueued BEFORE waiting for the count, so the GPU keeps running while the host waits.
            rc = bin_and_blend(capacity_hint, total);
            if (rc) return rc;
            blended = true;
        }
        GSB_CUDA(cudaEventSynchronize(ev));
        if (*h >= (1ull << 31)) {
            set_error("instance count %llu exceeds 2^31", *h);
            return GSB_ERR_OVERFLOW;
        }
        D = (int64_t)*h;
        if (!blended || D > capacity_hint) {   // exact path, also the (rare) repair when the estimate was too small
            rc = bin_and_blend(D, nullptr);
            if (rc) return rc;
        }
    } else {
        rc = bin_and_blend(0, nullptr);
        if (rc) return rc;
    }
    st->num_rendered = D;
    return GSB_OK;
}

int32_t gsb_forward(const GsbSettings *s, const GsbInputs *in, float *out_color, int32_t *out_radii,
                    float *out_invdepth, int64_t capacity_hint, gsb_alloc_fn alloc, void *alloc_ctx, GsbState *st,
                    void *cuda_stream) {
    return forward_impl("gsb_forward", s, in, nullptr, out_color, out_radii, out_invdepth, capacity_hint, alloc, alloc_ctx, st,
                        cuda_stream);
}

int32_t gsb_forward_split_sh(const GsbSettings *s, const GsbInputs *in, const GsbSplitSH *split, float *out_color,
                             int32_t *out_radii, float *out_invdepth, int64_t capacity_hint, gsb_alloc_fn alloc,
                             void *alloc_ctx, GsbState *st, void *cuda_stream) {
    if (!split) { set_error("gsb_forward_split_sh: NULL argument"); return GSB_ERR_ARGUMENT; }
    return forward_impl("gsb_forward_split_sh", s, in, split, out_color, out_radii, out_invdepth, capacity_hint, alloc, alloc_ctx, st,
                        cuda_stream);
}

// Camera-gradient scratch of a K8 launch over P gaussians and V views: the warp partials and the dL/dbg partials.  Fills the
// scratch pointers of `r` and returns the caller's PreBwdArgs::cam_part.
static float *carve_cam_scratch(gsb_alloc_fn alloc, void *alloc_ctx, int V, int P, CamReduceArgs &r) {
    r.V = V;
    r.nslots = (int)cam_slots(P);
    auto carve = [&](Carver &c) {
        r.part = c.take<float>((size_t)V * CAM_TERMS * (r.nslots > 0 ? r.nslots : 1));
        r.bg_part = c.take<float>((size_t)V * 3 * CAM_BG_BLOCKS);
    };
    Carver c0(nullptr);
    carve(c0);
    void *scr = do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH1, c0.bytes());
    if (!scr) return nullptr;
    Carver c1(scr);
    carve(c1);
    return r.part;
}

static void set_cam_outputs(const GsbCameraGrads *cg, CamReduceArgs &r) {
    r.dview = cg->dL_dviewmatrix; r.dproj = cg->dL_dprojmatrix; r.dcampos = cg->dL_dcampos; r.dbg = cg->dL_dbg;
}

static bool misaligned(const void *p) { return (reinterpret_cast<size_t>(p) & 3) != 0; }

// the feature term of a backward call (NULL = none); `launch` = the feature blend pass runs (a feature loss is given)
static int check_features(const char *fn, const GsbFeatures *ft, int P, bool &launch) {
    launch = false;
    if (!ft) return GSB_OK;
    if (ft->channels < 1 || ft->channels > GSB_MAX_FEATURE_CHANNELS) {
        set_error("%s: feature channels %d outside 1..%d", fn, ft->channels, GSB_MAX_FEATURE_CHANNELS);
        return GSB_ERR_ARGUMENT;
    }
    if (!ft->features && P > 0 && (ft->out_features || ft->dL_dout_features || ft->dL_dfeatures)) {
        set_error("%s: feature outputs given without features", fn);
        return GSB_ERR_ARGUMENT;
    }
    if (ft->dL_dout_features && !ft->out_features) {
        set_error("%s: dL_dout_features given without out_features", fn);
        return GSB_ERR_ARGUMENT;
    }
    if (misaligned(ft->features) || misaligned(ft->out_features) || misaligned(ft->dL_dout_features) || misaligned(ft->dL_dfeatures)) {
        set_error("%s: feature tensors must be 4-byte aligned float pointers", fn);
        return GSB_ERR_ARGUMENT;
    }
    launch = ft->dL_dout_features != nullptr && P > 0;
    return GSB_OK;
}

// a state's view for the feature kernels; false when it does not hold a forward of P gaussians over num_tiles tiles
static bool feat_view(const GsbState &st, int P, int num_tiles, FeatView &v) {
    if (st.P != P || st.num_tiles != num_tiles || !st.ranges || !st.point_list || !st.splat || !st.n_contrib) return false;
    v.ranges = static_cast<const uint2 *>(st.ranges); v.point_list = st.point_list;
    v.tile_order = static_cast<const uint32_t *>(st.tile_order); v.splat = static_cast<const float4 *>(st.splat);
    v.n_contrib = st.n_contrib;
    return true;
}

// deterministic backward, first half: the partial rows and marks of the blend launch `ra` over V views of cap list positions
// (GSB_BUF_SCRATCH2); launch_det_reduce after the blend launch stores the accumulator rows
static int det_begin(const char *fn, gsb_alloc_fn alloc, void *alloc_ctx, int64_t cap, int V, DetScratch &d, RenderBwdArgs &ra,
                     cudaStream_t stream) {
    if (cap >= ((int64_t)1 << 30)) { set_error("%s: deterministic backward: capacity %lld exceeds 2^30", fn, (long long)cap); return GSB_ERR_OVERFLOW; }
    const int64_t capn = cap > 0 ? cap : 1;
    void *scr = do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH2, det_carve(nullptr, capn, V, d));
    if (!scr) return GSB_ERR_ALLOC;
    det_carve(scr, capn, V, d);
    GSB_CUDA(cudaMemsetAsync(d.mark, 0, (size_t)V * capn * 2, stream));
    ra.det_part = d.part; ra.det_mark = d.mark;
    return GSB_OK;
}

// shared body of gsb_backward (split == NULL), gsb_backward_split_sh, gsb_backward_camera (cam_grads != NULL),
// gsb_backward_alpha (dL_dalpha != NULL) and gsb_backward_features (feat != NULL)
static int backward_impl(const char *fn, const GsbSettings *s, const GsbInputs *in, const GsbSplitSH *split, const GsbState *st,
                         const float *out_color, const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth,
                         const GsbGrads *grads, int32_t accumulate, gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream,
                         const GsbCameraGrads *cam_grads = nullptr, const float *dL_dalpha = nullptr,
                         const GsbFeatures *feat = nullptr) {
    if (!s || !in || !st || !out_color || !out_invdepth || !dL_dcolor || !grads || !alloc) {
        set_error("%s: NULL argument", fn);
        return GSB_ERR_ARGUMENT;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    const bool debug = s->debug != 0;
    CamArgs cam;
    int rc = make_cam(s, cam);
    if (rc) return rc;
    rc = check_inputs(s, in, split);
    if (rc) return rc;
    bool want_cam = false;
    rc = check_cam_grads(fn, cam_grads, want_cam);
    if (rc) return rc;
    if (split && grads->dL_dshs) {
        set_error("%s: grads->dL_dshs must be NULL (dL_ddc / dL_drest receive the SH gradient)", fn);
        return GSB_ERR_ARGUMENT;
    }
    const int P = in->P;
    if (P != st->P || st->num_tiles != cam.gx * cam.gy || !st->splat || !st->ranges || !st->final_T) {
        set_error("%s: state does not match the inputs (P %d vs %d)", fn, P, st->P);
        return GSB_ERR_ARGUMENT;
    }
    bool want_feat = false;
    rc = check_features(fn, feat, P, want_feat);
    if (rc) return rc;
    const bool det = g_deterministic != 0;
    if (det && want_feat) {
        set_error("%s: the feature backward has no deterministic implementation (gsb_set_deterministic is on)", fn);
        return GSB_ERR_ARGUMENT;
    }
    if (feat && feat->dL_dfeatures && !accumulate && P > 0)
        GSB_CUDA(cudaMemsetAsync(feat->dL_dfeatures, 0, (size_t)P * feat->channels * sizeof(float), stream));
    CamReduceArgs cr;
    memset(&cr, 0, sizeof(cr));
    if (want_cam) {
        if (!carve_cam_scratch(alloc, alloc_ctx, 1, P, cr)) return GSB_ERR_ALLOC;
        set_cam_outputs(cam_grads, cr);
        cr.final_T = st->final_T; cr.sv_image = 0; cr.npix = (size_t)cam.W * cam.H; cr.dL_dcolor = dL_dcolor;
    }
    if (P == 0) return want_cam ? launch_camera_grad_reduce(cr, accumulate != 0, debug, stream) : GSB_OK;
    const size_t dacc_bytes = align_up((size_t)P * DACC_STRIDE * sizeof(float), 256);
    float *dacc = static_cast<float *>(do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH0, dacc_bytes));
    if (!dacc) return GSB_ERR_ALLOC;
    if (!det || st->num_rendered == 0) GSB_CUDA(cudaMemsetAsync(dacc, 0, dacc_bytes, stream));     // det: det_reduce stores every row
    const float4 *splat = static_cast<const float4 *>(st->splat);

    if (st->num_rendered != 0) {
        RenderBwdArgs ra;
        memset(&ra, 0, sizeof(ra));
        ra.W = cam.W; ra.H = cam.H; ra.gx = cam.gx; ra.gy = cam.gy; ra.V = 1;
        ra.ranges = static_cast<const uint2 *>(st->ranges); ra.point_list = st->point_list;
        ra.tile_order = static_cast<const uint32_t *>(st->tile_order);
        ra.splat = splat; ra.n_contrib = st->n_contrib; ra.dL_dcolor = dL_dcolor;
        ra.dL_dinvdepth = dL_dinvdepth; ra.dacc = dacc; ra.out_color = out_color; ra.out_invdepth = out_invdepth;
        ra.final_T = st->final_T; ra.dL_dalpha = dL_dalpha;
        DetScratch ds;
        if (det && (rc = det_begin(fn, alloc, alloc_ctx, st->binning_capacity, 1, ds, ra, stream))) return rc;
        rc = launch_render_bwd(ra, debug, stream);
        if (rc) return rc;
        if (det && (rc = launch_det_reduce(ra, ds, P, dacc, debug, stream))) return rc;
        if (want_feat) {     // adds its terms into the same accumulator rows (linear in the loss gradient)
            FeatArgs fa;
            memset(&fa, 0, sizeof(fa));
            fa.W = cam.W; fa.H = cam.H; fa.gx = cam.gx; fa.gy = cam.gy; fa.V = 1; fa.C = feat->channels; fa.P = P;
            if (!feat_view(*st, P, cam.gx * cam.gy, fa.view[0])) {
                set_error("%s: state has no binning", fn);
                return GSB_ERR_ARGUMENT;
            }
            fa.features = feat->features; fa.out_features = feat->out_features; fa.dL_dout = feat->dL_dout_features;
            fa.dacc = dacc; fa.dL_dfeatures = feat->dL_dfeatures;
            rc = launch_render_features_bwd(fa, debug, stream);
            if (rc) return rc;
        }
    }
    PreBwdArgs pa;
    pa.P = P; pa.means = in->means3D; pa.shs = split ? split->dc : in->shs; pa.opac = in->opacities; pa.scales = in->scales;
    pa.rots = in->rotations; pa.cov_pre = in->cov3D_precomp; pa.splat = splat; pa.dacc = dacc; pa.g = *grads;
    pa.rest = split ? split->rest : nullptr;
    pa.dL_drest = split ? split->dL_drest : nullptr;
    if (split) pa.g.dL_dshs = split->dL_ddc;
    pa.p_begin = 0; pa.p_end = P;
    pa.peer.world = 0;
    pa.cam_part = want_cam ? cr.part : nullptr;
    rc = launch_preprocess_bwd(cam, pa, split != nullptr, accumulate != 0, debug, stream);
    if (rc || !want_cam) return rc;
    return launch_camera_grad_reduce(cr, accumulate != 0, debug, stream);
}

int32_t gsb_backward(const GsbSettings *s, const GsbInputs *in, const GsbState *st, const float *out_color,
                     const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth,
                     const GsbGrads *grads, int32_t accumulate, gsb_alloc_fn alloc, void *alloc_ctx,
                     void *cuda_stream) {
    return backward_impl("gsb_backward", s, in, nullptr, st, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads, accumulate,
                         alloc, alloc_ctx, cuda_stream);
}

int32_t gsb_backward_split_sh(const GsbSettings *s, const GsbInputs *in, const GsbSplitSH *split, const GsbState *st,
                              const float *out_color, const float *out_invdepth, const float *dL_dcolor,
                              const float *dL_dinvdepth, const GsbGrads *grads, int32_t accumulate,
                              gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream) {
    if (!split) { set_error("gsb_backward_split_sh: NULL argument"); return GSB_ERR_ARGUMENT; }
    return backward_impl("gsb_backward_split_sh", s, in, split, st, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads,
                         accumulate, alloc, alloc_ctx, cuda_stream);
}

int32_t gsb_backward_camera(const GsbSettings *s, const GsbInputs *in, const GsbSplitSH *split, const GsbState *st,
                            const float *out_color, const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth,
                            const GsbGrads *grads, const GsbCameraGrads *cam_grads, int32_t accumulate, gsb_alloc_fn alloc,
                            void *alloc_ctx, void *cuda_stream) {
    return backward_impl("gsb_backward_camera", s, in, split, st, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads, accumulate,
                         alloc, alloc_ctx, cuda_stream, cam_grads);
}

int32_t gsb_backward_alpha(const GsbSettings *s, const GsbInputs *in, const GsbSplitSH *split, const GsbState *st,
                           const float *out_color, const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth,
                           const float *dL_dalpha, const GsbGrads *grads, const GsbCameraGrads *cam_grads, int32_t accumulate,
                           gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream) {
    if (dL_dalpha && (reinterpret_cast<size_t>(dL_dalpha) & 3)) {
        set_error("gsb_backward_alpha: dL_dalpha must be a 4-byte aligned float pointer");
        return GSB_ERR_ARGUMENT;
    }
    return backward_impl("gsb_backward_alpha", s, in, split, st, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads, accumulate,
                         alloc, alloc_ctx, cuda_stream, cam_grads, dL_dalpha);
}

int32_t gsb_alpha(int32_t V, const GsbState *states, int32_t height, int32_t width, float *out_alpha, void *cuda_stream) {
    if (!states || !out_alpha || V < 1 || V > GSB_MAX_VIEWS || height <= 0 || width <= 0) {
        set_error("gsb_alpha: NULL argument, V=%d outside 1..%d or bad image size %d x %d", V, GSB_MAX_VIEWS, height, width);
        return GSB_ERR_ARGUMENT;
    }
    AlphaArgs a;
    memset(&a, 0, sizeof(a));
    a.V = V; a.npix = (size_t)height * width; a.out = out_alpha;
    for (int v = 0; v < V; ++v) {
        // the IMAGE buffer holds final_T and n_contrib of npix pixels each (carve_image): a smaller one is another image size
        if (!states[v].final_T || !states[v].image ||
            (const char *)states[v].final_T + a.npix * sizeof(float) > (const char *)states[v].image + states[v].image_bytes) {
            set_error("gsb_alpha: state %d has no forward image of %d x %d pixels", v, width, height);
            return GSB_ERR_ARGUMENT;
        }
        a.final_T[v] = states[v].final_T;
    }
    return launch_alpha(a, false, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_backward_features(const GsbSettings *s, const GsbInputs *in, const GsbSplitSH *split, const GsbState *st,
                              const float *out_color, const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth,
                              const float *dL_dalpha, const GsbGrads *grads, const GsbCameraGrads *cam_grads,
                              const GsbFeatures *features, int32_t accumulate, gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream) {
    if (misaligned(dL_dalpha)) {
        set_error("gsb_backward_features: dL_dalpha must be a 4-byte aligned float pointer");
        return GSB_ERR_ARGUMENT;
    }
    return backward_impl("gsb_backward_features", s, in, split, st, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads,
                         accumulate, alloc, alloc_ctx, cuda_stream, cam_grads, dL_dalpha, features);
}

int32_t gsb_render_features(int32_t V, const GsbState *states, int32_t height, int32_t width, int32_t P, int32_t channels,
                            const float *features, float *out, void *cuda_stream) {
    if (!states || !out || V < 1 || V > GSB_MAX_VIEWS || height <= 0 || width <= 0 || P < 0 || (P > 0 && !features)) {
        set_error("gsb_render_features: NULL argument, V=%d outside 1..%d, bad image size %d x %d or P=%d", V, GSB_MAX_VIEWS, height,
                  width, P);
        return GSB_ERR_ARGUMENT;
    }
    if (channels < 1 || channels > GSB_MAX_FEATURE_CHANNELS) {
        set_error("gsb_render_features: channels %d outside 1..%d", channels, GSB_MAX_FEATURE_CHANNELS);
        return GSB_ERR_ARGUMENT;
    }
    if (misaligned(features) || misaligned(out)) {
        set_error("gsb_render_features: features and out must be 4-byte aligned float pointers");
        return GSB_ERR_ARGUMENT;
    }
    FeatArgs a;
    memset(&a, 0, sizeof(a));
    a.W = width; a.H = height; a.gx = (width + TILE - 1) / TILE; a.gy = (height + TILE - 1) / TILE; a.V = V; a.C = channels; a.P = P;
    a.features = features; a.out = out;
    const size_t npix = (size_t)height * width;
    for (int v = 0; v < V; ++v) {
        // the IMAGE buffer holds final_T and n_contrib of npix pixels each (carve_image): a smaller one is another image size
        if (!feat_view(states[v], P, a.gx * a.gy, a.view[v]) || !states[v].image ||
            (const char *)states[v].n_contrib + npix * sizeof(uint32_t) > (const char *)states[v].image + states[v].image_bytes) {
            set_error("gsb_render_features: state %d is not a forward of %d gaussians over %d x %d pixels", v, P, width, height);
            return GSB_ERR_ARGUMENT;
        }
    }
    return launch_render_features(a, false, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_contribution(int32_t V, const GsbState *states, int32_t height, int32_t width, int32_t P, int64_t *count,
                         float *weight_sum, float *weight_max, void *cuda_stream) {
    if (!states || V < 1 || V > GSB_MAX_VIEWS || height <= 0 || width <= 0 || P < 0 ||
        (P > 0 && (!count || !weight_sum || !weight_max))) {
        set_error("gsb_contribution: NULL argument, V=%d outside 1..%d, bad image size %d x %d or P=%d", V, GSB_MAX_VIEWS, height,
                  width, P);
        return GSB_ERR_ARGUMENT;
    }
    if ((reinterpret_cast<size_t>(count) & 7) || misaligned(weight_sum) || misaligned(weight_max)) {
        set_error("gsb_contribution: count must be 8-byte, weight_sum and weight_max 4-byte aligned");
        return GSB_ERR_ARGUMENT;
    }
    ContribArgs a;
    memset(&a, 0, sizeof(a));
    a.W = width; a.H = height; a.gx = (width + TILE - 1) / TILE; a.gy = (height + TILE - 1) / TILE; a.V = V; a.P = P;
    a.count = reinterpret_cast<long long *>(count); a.weight_sum = weight_sum;
    a.weight_max_bits = reinterpret_cast<uint32_t *>(weight_max);
    const size_t npix = (size_t)height * width;
    for (int v = 0; v < V; ++v) {
        if (states[v].P != P) {
            set_error("gsb_contribution: state %d holds %d gaussians, not %d", v, states[v].P, P);
            return GSB_ERR_ARGUMENT;
        }
        if (P == 0) continue;
        // the IMAGE buffer holds final_T and n_contrib of npix pixels each (carve_image): a smaller one is another image size
        if (!feat_view(states[v], P, a.gx * a.gy, a.view[v]) || !states[v].image ||
            (const char *)states[v].n_contrib + npix * sizeof(uint32_t) > (const char *)states[v].image + states[v].image_bytes) {
            set_error("gsb_contribution: state %d is not a forward of %d gaussians over %d x %d pixels", v, P, width, height);
            return GSB_ERR_ARGUMENT;
        }
    }
    return launch_contribution(a, false, static_cast<cudaStream_t>(cuda_stream));
}

static int check_batch(int32_t V, const GsbSettings *s, const GsbInputs *in, CamArgsBatch &cb) {
    if (V < 1 || V > GSB_MAX_VIEWS) { set_error("view batch: V=%d outside 1..%d", V, GSB_MAX_VIEWS); return GSB_ERR_ARGUMENT; }
    cb.V = V;
    for (int v = 0; v < V; ++v) {
        int rc = make_cam(&s[v], cb.cam[v]);
        if (rc) return rc;
        rc = check_inputs(&s[v], in);
        if (rc) return rc;
        if (cb.cam[v].W != cb.cam[0].W || cb.cam[v].H != cb.cam[0].H || cb.cam[v].sh_degree != cb.cam[0].sh_degree ||
            cb.cam[v].sh_coeffs != cb.cam[0].sh_coeffs) {
            set_error("view batch: all views must share image size and SH configuration");
            return GSB_ERR_ARGUMENT;
        }
    }
    if (in->colors_precomp || in->cov3D_precomp) {
        set_error("view batch: precomputed colours / covariances are per view; use the single-view call");
        return GSB_ERR_ARGUMENT;
    }
    return GSB_OK;
}

// shared body of gsb_forward_batch (counts read back, capacity repaired) and gsb_forward_batch_async (no host
// synchronisation at all: fixed capacity, counts and their running maximum stay on the device)
static int forward_batch_impl(int32_t V, const GsbSettings *s, const GsbInputs *in, float *out_color, int32_t *out_radii,
                              float *out_invdepth, int64_t capacity_hint, unsigned long long *counts_dev, gsb_alloc_fn alloc,
                              void *alloc_ctx, GsbState *states, cudaStream_t stream) {
    const bool async = counts_dev != nullptr;
    CamArgsBatch cb;
    int rc = check_batch(V, s, in, cb);
    if (rc) return rc;
    const bool debug = s[0].debug != 0;
    const CamArgs &c0 = cb.cam[0];
    const int P = in->P;
    const int num_tiles = c0.gx * c0.gy;
    const int tile_bits = bits_for((uint32_t)num_tiles);
    const size_t npix = (size_t)c0.W * c0.H;
    const size_t Pn = align_up((size_t)P, 64);     // per-view stride of the per-gaussian u32 arrays

    // ---- state buffers, V views each ----
    const size_t sv_splat = (size_t)P * SPLAT_F4;  // float4
    const size_t geom_bytes = align_up((size_t)V * sv_splat * sizeof(float4), 256);
    float4 *splat = static_cast<float4 *>(do_alloc(alloc, alloc_ctx, GSB_BUF_GEOM, geom_bytes));
    if (!splat) return GSB_ERR_ALLOC;
    ImageView iv0;
    const size_t image_bytes = carve_image(nullptr, npix, iv0);
    char *image = static_cast<char *>(do_alloc(alloc, alloc_ctx, GSB_BUF_IMAGE, (size_t)V * image_bytes));
    if (!image) return GSB_ERR_ALLOC;
    for (int v = 0; v < V; ++v) {
        GsbState *st = &states[v];
        memset(st, 0, sizeof(*st));
        st->P = P; st->num_tiles = num_tiles; st->num_visible = -1;
        st->geom = splat; st->geom_bytes = geom_bytes; st->image = image; st->image_bytes = (size_t)V * image_bytes;
        st->splat = splat + (size_t)v * sv_splat;
        ImageView iv;
        carve_image(image + (size_t)v * image_bytes, npix, iv);
        st->final_T = iv.final_T; st->n_contrib = iv.n_contrib;
    }

    // ---- per-gaussian scratch, [V][Pn] ----
    const size_t np = scan_state_count(P);
    uint32_t *key, *idx, *key_alt, *idx_alt, *tiles, *offsets; uint2 *rect; unsigned long long *scan_state, *total; char *sortscr;
    auto carve0 = [&](Carver &c) {
        key = c.take<uint32_t>(V * Pn); idx = c.take<uint32_t>(V * Pn); key_alt = c.take<uint32_t>(V * Pn); idx_alt = c.take<uint32_t>(V * Pn);
        tiles = c.take<uint32_t>(V * Pn); rect = c.take<uint2>(V * Pn); offsets = c.take<uint32_t>(V * Pn);
        scan_state = c.take<unsigned long long>(V * np); total = c.take<unsigned long long>(GSB_MAX_VIEWS);
        sortscr = c.take<char>(sort_scratch_bytes(P, V));
    };
    Carver c0n(nullptr);
    carve0(c0n);
    void *scr0 = do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH0, c0n.bytes());
    if (!scr0) return GSB_ERR_ALLOC;
    Carver c0r(scr0);
    carve0(c0r);
    if (async) total = counts_dev;     // the caller's buffer: the counts outlive the call

    PreFwdArgs pa;
    pa.P = P; pa.means = in->means3D; pa.shs = in->shs; pa.colors = nullptr; pa.opac = in->opacities;
    pa.scales = in->scales; pa.rots = in->rotations; pa.cov_pre = nullptr; pa.rest = nullptr;
    pa.splat = splat; pa.depth_key = key; pa.depth_idx = idx; pa.tiles = tiles; pa.rect = rect; pa.radii = out_radii;
    pa.cull = opt_cull;
    PreFwdBatchStrides ps;
    ps.splat = sv_splat; ps.per_gauss = Pn; ps.radii = (size_t)P;
    rc = launch_preprocess_fwd_batch(cb, pa, ps, debug, stream);
    if (rc) return rc;
    rc = sort_pairs(key, idx, key_alt, idx_alt, P, nullptr, 0, 32, sortscr, debug, stream, V, Pn);
    if (rc) return rc;
    BinArgs ba;
    ba.P = P; ba.num_tiles = num_tiles; ba.gx = c0.gx; ba.order = idx; ba.tiles = tiles; ba.rect = rect; ba.splat = splat;
    ba.offsets = offsets; ba.scan_state = scan_state; ba.total = total;
    ba.sv_gauss = Pn; ba.sv_splat = sv_splat; ba.sv_scan = np; ba.sv_inst = 0;
    rc = launch_tile_scan(ba, V, debug, stream);
    if (rc) return rc;
    unsigned long long *h = nullptr;
    cudaEvent_t ev = nullptr;
    if (async) {
        rc = launch_count_max(total, V, debug, stream);     // counts_dev[GSB_MAX_VIEWS] = max(itself, the V counts)
        if (rc) return rc;
    } else {
        h = pinned_slot();
        ev = readback_event();
        if (!h || !ev) { set_error("pinned read-back slot unavailable"); return GSB_ERR_CUDA; }
        GSB_CUDA(cudaMemcpyAsync(h, total, (size_t)V * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
        GSB_CUDA(cudaEventRecord(ev, stream));
    }

    auto bin_and_blend = [&](int64_t cap) -> int {
        // BINNING: [V][cap] point lists, then [V][num_tiles] ranges, then [V][num_tiles] tile order
        const size_t capn = (size_t)(cap > 0 ? cap : 1);
        const size_t pl_bytes = align_up((size_t)V * capn * 4, 256);
        const size_t rg_bytes = align_up((size_t)V * num_tiles * sizeof(uint2), 256);
        const size_t bin_bytes = pl_bytes + rg_bytes + align_up((size_t)V * num_tiles * sizeof(uint32_t), 256);
        char *bin = static_cast<char *>(do_alloc(alloc, alloc_ctx, GSB_BUF_BINNING, bin_bytes));
        if (!bin) return GSB_ERR_ALLOC;
        uint32_t *point_list = reinterpret_cast<uint32_t *>(bin);
        uint2 *ranges = reinterpret_cast<uint2 *>(bin + pl_bytes);
        uint32_t *tile_order = reinterpret_cast<uint32_t *>(bin + pl_bytes + rg_bytes);
        for (int v = 0; v < V; ++v) {
            states[v].binning = bin; states[v].binning_bytes = bin_bytes; states[v].binning_capacity = cap;
            states[v].point_list = point_list + (size_t)v * capn; states[v].ranges = ranges + (size_t)v * num_tiles;
            states[v].tile_order = opt_tile_order ? tile_order + (size_t)v * num_tiles : nullptr;
        }
        int r;
        if (cap > 0) {
            Carver c1(nullptr);
            c1.take<uint32_t>(V * capn); c1.take<uint32_t>(V * capn); c1.take<uint32_t>(V * capn); c1.take<char>(sort_scratch_bytes(cap, V));
            void *scr1 = do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH1, c1.bytes());
            if (!scr1) return GSB_ERR_ALLOC;
            Carver c1r(scr1);
            uint32_t *inst_tile = c1r.take<uint32_t>(V * capn), *inst_tile_alt = c1r.take<uint32_t>(V * capn);
            uint32_t *inst_gauss_alt = c1r.take<uint32_t>(V * capn);
            char *sortscr1 = c1r.take<char>(sort_scratch_bytes(cap, V));
            BinArgs bb = ba;
            bb.sv_inst = capn;
            SortDigits dg;
            r = sort_prepare(cap, V, 0, tile_bits, sortscr1, stream, &dg);
            if (r) return r;
            r = launch_emit(bb, V, inst_tile, point_list, cap, dg, debug, stream);
            if (r) return r;
            r = sort_pairs(inst_tile, point_list, inst_tile_alt, inst_gauss_alt, cap, total, 0, tile_bits, sortscr1, debug, stream, V, capn,
                           true);
            if (r) return r;
            r = launch_tile_ranges(inst_tile, cap, total, num_tiles, ranges, V, capn, debug, stream);
            if (r) return r;
        } else {
            r = launch_tile_ranges(nullptr, 0, nullptr, num_tiles, ranges, V, 0, debug, stream);
            if (r) return r;
        }
        r = maybe_tile_order(ranges, V, num_tiles, tile_order, debug, stream);
        if (r) return r;
        // ONE blend launch for the V views
        RenderFwdArgs ra;
        memset(&ra, 0, sizeof(ra));
        ra.W = c0.W; ra.H = c0.H; ra.gx = c0.gx; ra.gy = c0.gy; ra.V = V;
        ra.sv_ranges = (size_t)num_tiles; ra.sv_list = capn; ra.sv_splat = sv_splat; ra.sv_color = 3 * npix; ra.sv_depth = npix;
        ra.sv_image = image_bytes / sizeof(float);
        ra.ranges = ranges; ra.point_list = point_list; ra.tile_order = opt_tile_order ? tile_order : nullptr; ra.splat = splat;
        for (int v = 0; v < V; ++v) ra.bg[v] = s[v].bg;
        ra.out_color = out_color; ra.out_invdepth = out_invdepth;
        ra.final_T = const_cast<float *>(states[0].final_T); ra.n_contrib = const_cast<uint32_t *>(states[0].n_contrib);
        return launch_render_fwd(ra, debug, stream);
    };

    if (async) {
        for (int v = 0; v < V; ++v) states[v].num_rendered = -1;     // known to the device only
        return bin_and_blend(capacity_hint);
    }
    bool blended = false;
    if (capacity_hint > 0 && capacity_hint < (1ll << 30)) {
        rc = bin_and_blend(capacity_hint);
        if (rc) return rc;
        blended = true;
    }
    GSB_CUDA(cudaEventSynchronize(ev));
    int64_t dmax = 0;
    for (int v = 0; v < V; ++v) {
        if (h[v] >= (1ull << 30)) { set_error("instance count %llu exceeds 2^30", h[v]); return GSB_ERR_OVERFLOW; }
        states[v].num_rendered = (int64_t)h[v];
        if ((int64_t)h[v] > dmax) dmax = (int64_t)h[v];
    }
    if (!blended || dmax > capacity_hint) {
        rc = bin_and_blend(dmax);
        if (rc) return rc;
    }
    return GSB_OK;
}

int32_t gsb_forward_batch(int32_t V, const GsbSettings *s, const GsbInputs *in, float *out_color, int32_t *out_radii,
                          float *out_invdepth, int64_t capacity_hint, gsb_alloc_fn alloc, void *alloc_ctx, GsbState *states,
                          void *cuda_stream) {
    if (!s || !in || !out_color || !out_radii || !out_invdepth || !alloc || !states || in->P <= 0) {
        set_error("gsb_forward_batch: NULL argument or empty input");
        return GSB_ERR_ARGUMENT;
    }
    return forward_batch_impl(V, s, in, out_color, out_radii, out_invdepth, capacity_hint, nullptr, alloc, alloc_ctx, states,
                              static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_forward_batch_async(int32_t V, const GsbSettings *s, const GsbInputs *in, float *out_color, int32_t *out_radii,
                                float *out_invdepth, int64_t capacity, uint64_t *counts_dev, gsb_alloc_fn alloc, void *alloc_ctx,
                                GsbState *states, void *cuda_stream) {
    if (!s || !in || !out_color || !out_radii || !out_invdepth || !alloc || !states || in->P <= 0 || !counts_dev) {
        set_error("gsb_forward_batch_async: NULL argument or empty input");
        return GSB_ERR_ARGUMENT;
    }
    if (capacity <= 0 || capacity >= (1ll << 30)) {
        set_error("gsb_forward_batch_async: capacity %lld outside 1..2^30-1", (long long)capacity);
        return GSB_ERR_ARGUMENT;
    }
    static_assert(sizeof(uint64_t) == sizeof(unsigned long long), "count type");
    return forward_batch_impl(V, s, in, out_color, out_radii, out_invdepth, capacity, reinterpret_cast<unsigned long long *>(counts_dev),
                              alloc, alloc_ctx, states, static_cast<cudaStream_t>(cuda_stream));
}

// shared body of gsb_backward_batch / gsb_backward_batch_chunked
static int backward_batch_impl(int32_t V, const GsbSettings *s, const GsbInputs *in, const GsbState *states, const float *out_color,
                               const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth, const GsbGrads *grads,
                               int32_t accumulate, int32_t n_chunks, gsb_chunk_fn on_chunk, void *chunk_ctx, gsb_alloc_fn alloc,
                               void *alloc_ctx, cudaStream_t stream, const GsbPeerTable *peers = nullptr,
                               const GsbCameraGrads *cam_grads = nullptr, const float *dL_dalpha = nullptr,
                               const GsbFeatures *feat = nullptr) {
    CamArgsBatch cb;
    int rc = check_batch(V, s, in, cb);
    if (rc) return rc;
    bool want_cam = false;
    rc = check_cam_grads("gsb_backward_batch_camera", cam_grads, want_cam);
    if (rc) return rc;
    bool want_feat = false;
    rc = check_features("gsb_backward_batch_features", feat, in->P, want_feat);
    if (rc) return rc;
    if (feat && (peers || n_chunks > 1 || on_chunk)) {
        set_error("gsb_backward_batch_features: features are not available on the chunked or peer backward");
        return GSB_ERR_ARGUMENT;
    }
    const bool det = g_deterministic != 0;
    if (det && (want_feat || peers)) {
        set_error("gsb_backward_batch: the %s has no deterministic implementation (gsb_set_deterministic is on)",
                  want_feat ? "feature backward" : "peer reduce-scatter");
        return GSB_ERR_ARGUMENT;
    }
    const bool debug = s[0].debug != 0;
    const CamArgs &c0 = cb.cam[0];
    const int P = in->P;
    const size_t npix = (size_t)c0.W * c0.H;
    bool any = false, uniform = true;
    for (int v = 0; v < V; ++v) {
        if (states[v].P != P || states[v].num_tiles != c0.gx * c0.gy || !states[v].splat || !states[v].ranges || !states[v].final_T) {
            set_error("gsb_backward_batch: state %d does not match the inputs", v);
            return GSB_ERR_ARGUMENT;
        }
        any = any || states[v].num_rendered != 0;
        // the batched blend launch addresses view v at base + v * stride: the states must come from ONE forward_batch call
        if (v > 0 && (states[v].binning != states[0].binning || states[v].image != states[0].image || states[v].geom != states[0].geom))
            uniform = false;
    }
    if (!uniform) { set_error("gsb_backward_batch: states of different forward calls"); return GSB_ERR_ARGUMENT; }
    const size_t sv_dacc = (size_t)P * DACC_STRIDE;
    const size_t dacc_bytes = align_up((size_t)V * sv_dacc * sizeof(float), 256);
    float *dacc = static_cast<float *>(do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH0, dacc_bytes));
    if (!dacc) return GSB_ERR_ALLOC;
    if (!det || !any) GSB_CUDA(cudaMemsetAsync(dacc, 0, dacc_bytes, stream));     // det: det_reduce stores every row
    if (feat && feat->dL_dfeatures && !accumulate)
        GSB_CUDA(cudaMemsetAsync(feat->dL_dfeatures, 0, (size_t)P * feat->channels * sizeof(float), stream));
    const size_t sv_splat = V > 1 ? (size_t)((const float4 *)states[1].splat - (const float4 *)states[0].splat) : 0;
    if (any) {
        RenderBwdArgs ra;
        memset(&ra, 0, sizeof(ra));
        ra.W = c0.W; ra.H = c0.H; ra.gx = c0.gx; ra.gy = c0.gy; ra.V = V;
        if (V > 1) {
            ra.sv_ranges = (size_t)((const uint2 *)states[1].ranges - (const uint2 *)states[0].ranges);
            ra.sv_list = (size_t)(states[1].point_list - states[0].point_list);
            ra.sv_image = (size_t)(states[1].n_contrib - states[0].n_contrib);
        }
        ra.sv_splat = sv_splat; ra.sv_color = 3 * npix; ra.sv_depth = npix; ra.sv_dacc = sv_dacc;
        ra.ranges = static_cast<const uint2 *>(states[0].ranges); ra.point_list = states[0].point_list;
        ra.tile_order = static_cast<const uint32_t *>(states[0].tile_order);
        ra.splat = static_cast<const float4 *>(states[0].splat); ra.n_contrib = states[0].n_contrib;
        ra.dL_dcolor = dL_dcolor; ra.dL_dinvdepth = dL_dinvdepth; ra.dacc = dacc; ra.out_color = out_color; ra.out_invdepth = out_invdepth;
        ra.final_T = states[0].final_T; ra.dL_dalpha = dL_dalpha;     // final_T and n_contrib share the IMAGE stride sv_image
        DetScratch ds;
        if (det && (rc = det_begin("gsb_backward_batch", alloc, alloc_ctx, states[0].binning_capacity, V, ds, ra, stream))) return rc;
        rc = launch_render_bwd(ra, debug, stream);
        if (rc) return rc;
        if (det && (rc = launch_det_reduce(ra, ds, P, dacc, debug, stream))) return rc;
        if (want_feat) {     // adds into the same accumulator rows, view v at rows v * P + id
            FeatArgs fa;
            memset(&fa, 0, sizeof(fa));
            fa.W = c0.W; fa.H = c0.H; fa.gx = c0.gx; fa.gy = c0.gy; fa.V = V; fa.C = feat->channels; fa.P = P;
            for (int v = 0; v < V; ++v) {
                if (!feat_view(states[v], P, c0.gx * c0.gy, fa.view[v])) {
                    set_error("gsb_backward_batch_features: state %d has no binning", v);
                    return GSB_ERR_ARGUMENT;
                }
            }
            fa.features = feat->features; fa.out_features = feat->out_features; fa.dL_dout = feat->dL_dout_features;
            fa.dacc = dacc; fa.dL_dfeatures = feat->dL_dfeatures;
            rc = launch_render_features_bwd(fa, debug, stream);
            if (rc) return rc;
        }
    }
    PreBwdArgs pa;
    pa.P = P; pa.means = in->means3D; pa.shs = in->shs; pa.opac = in->opacities; pa.scales = in->scales; pa.rots = in->rotations;
    pa.cov_pre = nullptr; pa.splat = static_cast<const float4 *>(states[0].splat); pa.dacc = dacc; pa.g = *grads;
    pa.rest = nullptr; pa.dL_drest = nullptr;
    pa.peer.world = 0;
    pa.cam_part = nullptr;
    CamReduceArgs cr;
    memset(&cr, 0, sizeof(cr));
    if (want_cam) {
        // the per-view sums cover every gaussian: one K8 launch, in this rank's process
        if (peers || n_chunks > 1) {
            set_error("camera gradients: not available on the chunked or peer backward (the sum would span chunks or ranks)");
            return GSB_ERR_ARGUMENT;
        }
        if (!carve_cam_scratch(alloc, alloc_ctx, V, P, cr)) return GSB_ERR_ALLOC;
        set_cam_outputs(cam_grads, cr);
        cr.final_T = states[0].final_T; cr.sv_image = V > 1 ? (size_t)(states[1].final_T - states[0].final_T) : 0;
        cr.npix = npix; cr.dL_dcolor = dL_dcolor;
        pa.cam_part = cr.part;
    }
    if (peers) {
        if (peers->world < 1 || peers->world > GSB_MAX_PEERS || peers->rank < 0 || peers->rank >= peers->world ||
            (int64_t)peers->rows_per_rank * peers->world < P) {
            set_error("gsb_backward_batch_peer: bad peer table (world %d, rank %d, rows_per_rank %d, P %d)", peers->world, peers->rank,
                      peers->rows_per_rank, P);
            return GSB_ERR_ARGUMENT;
        }
        pa.peer.world = peers->world; pa.peer.rows_per_rank = peers->rows_per_rank;
        for (int r = 0; r < GSB_MAX_PEERS; ++r)
            pa.peer.delta[r] = r < peers->world ? (long long)((const char *)peers->base[r] - (const char *)peers->base[peers->rank]) : 0;
    }
    PreBwdBatchStrides ps;
    ps.splat = sv_splat; ps.dacc = sv_dacc; ps.means2D = (size_t)P * 3;
    // gaussian-range chunks: chunk c's gradients are final when its launch completes, so the caller can start reducing
    // them (on_chunk: e.g. enqueue an all-reduce of the chunk's rows on another stream) while the next chunk computes
    if (n_chunks < 1) n_chunks = 1;
    const int step = (int)align_up((size_t)ceil_div(P, n_chunks), 256);
    for (int c = 0, p0 = 0; p0 < P; ++c, p0 += step) {
        pa.p_begin = p0; pa.p_end = p0 + step < P ? p0 + step : P;
        rc = launch_preprocess_bwd_batch(cb, pa, ps, accumulate != 0, debug, stream);
        if (rc) return rc;
        if (on_chunk) on_chunk(chunk_ctx, c, pa.p_begin, pa.p_end);
    }
    return want_cam ? launch_camera_grad_reduce(cr, accumulate != 0, debug, stream) : GSB_OK;
}

int32_t gsb_backward_batch(int32_t V, const GsbSettings *s, const GsbInputs *in, const GsbState *states, const float *out_color,
                           const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth, const GsbGrads *grads,
                           int32_t accumulate, gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream) {
    if (!s || !in || !states || !out_color || !out_invdepth || !dL_dcolor || !grads || !alloc || in->P <= 0) {
        set_error("gsb_backward_batch: NULL argument or empty input");
        return GSB_ERR_ARGUMENT;
    }
    return backward_batch_impl(V, s, in, states, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads, accumulate, 1, nullptr, nullptr,
                               alloc, alloc_ctx, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_backward_batch_camera(int32_t V, const GsbSettings *s, const GsbInputs *in, const GsbState *states, const float *out_color,
                                  const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth, const GsbGrads *grads,
                                  const GsbCameraGrads *cam_grads, int32_t accumulate, gsb_alloc_fn alloc, void *alloc_ctx,
                                  void *cuda_stream) {
    if (!s || !in || !states || !out_color || !out_invdepth || !dL_dcolor || !grads || !alloc || in->P <= 0) {
        set_error("gsb_backward_batch_camera: NULL argument or empty input");
        return GSB_ERR_ARGUMENT;
    }
    return backward_batch_impl(V, s, in, states, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads, accumulate, 1, nullptr, nullptr,
                               alloc, alloc_ctx, static_cast<cudaStream_t>(cuda_stream), nullptr, cam_grads);
}

int32_t gsb_backward_batch_peer(int32_t V, const GsbSettings *s, const GsbInputs *in, const GsbState *states, const float *out_color,
                                const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth, const GsbGrads *grads,
                                const GsbPeerTable *peers, gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream) {
    if (!s || !in || !states || !out_color || !out_invdepth || !dL_dcolor || !grads || !alloc || in->P <= 0 || !peers) {
        set_error("gsb_backward_batch_peer: NULL argument or empty input");
        return GSB_ERR_ARGUMENT;
    }
    return backward_batch_impl(V, s, in, states, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads, 1, 1, nullptr, nullptr, alloc,
                               alloc_ctx, static_cast<cudaStream_t>(cuda_stream), peers);
}

int32_t gsb_backward_batch_chunked(int32_t V, const GsbSettings *s, const GsbInputs *in, const GsbState *states, const float *out_color,
                                   const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth, const GsbGrads *grads,
                                   int32_t accumulate, int32_t n_chunks, gsb_chunk_fn on_chunk, void *chunk_ctx, gsb_alloc_fn alloc,
                                   void *alloc_ctx, void *cuda_stream) {
    if (!s || !in || !states || !out_color || !out_invdepth || !dL_dcolor || !grads || !alloc || in->P <= 0 || n_chunks < 1 || n_chunks > 64) {
        set_error("gsb_backward_batch_chunked: NULL argument, empty input or n_chunks outside 1..64");
        return GSB_ERR_ARGUMENT;
    }
    return backward_batch_impl(V, s, in, states, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads, accumulate, n_chunks, on_chunk,
                               chunk_ctx, alloc, alloc_ctx, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_backward_batch_alpha(int32_t V, const GsbSettings *s, const GsbInputs *in, const GsbState *states, const float *out_color,
                                 const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth, const float *dL_dalpha,
                                 const GsbGrads *grads, const GsbCameraGrads *cam_grads, const GsbPeerTable *peers, int32_t accumulate,
                                 int32_t n_chunks, gsb_chunk_fn on_chunk, void *chunk_ctx, gsb_alloc_fn alloc, void *alloc_ctx,
                                 void *cuda_stream) {
    if (!s || !in || !states || !out_color || !out_invdepth || !dL_dcolor || !grads || !alloc || in->P <= 0 || n_chunks < 1 ||
        n_chunks > 64) {
        set_error("gsb_backward_batch_alpha: NULL argument, empty input or n_chunks outside 1..64");
        return GSB_ERR_ARGUMENT;
    }
    if (dL_dalpha && (reinterpret_cast<size_t>(dL_dalpha) & 3)) {
        set_error("gsb_backward_batch_alpha: dL_dalpha must be a 4-byte aligned float pointer");
        return GSB_ERR_ARGUMENT;
    }
    // the existing entry points' mode selection: peers take the peer path (always adding), else chunks, else plain
    if (peers) { accumulate = 1; n_chunks = 1; on_chunk = nullptr; }
    return backward_batch_impl(V, s, in, states, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads, accumulate, n_chunks, on_chunk,
                               chunk_ctx, alloc, alloc_ctx, static_cast<cudaStream_t>(cuda_stream), peers, cam_grads, dL_dalpha);
}

int32_t gsb_backward_batch_features(int32_t V, const GsbSettings *s, const GsbInputs *in, const GsbState *states, const float *out_color,
                                    const float *out_invdepth, const float *dL_dcolor, const float *dL_dinvdepth, const float *dL_dalpha,
                                    const GsbGrads *grads, const GsbCameraGrads *cam_grads, const GsbFeatures *features,
                                    const GsbPeerTable *peers, int32_t accumulate, int32_t n_chunks, gsb_chunk_fn on_chunk,
                                    void *chunk_ctx, gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream) {
    if (!s || !in || !states || !out_color || !out_invdepth || !dL_dcolor || !grads || !alloc || in->P <= 0 || n_chunks < 1 ||
        n_chunks > 64) {
        set_error("gsb_backward_batch_features: NULL argument, empty input or n_chunks outside 1..64");
        return GSB_ERR_ARGUMENT;
    }
    if (misaligned(dL_dalpha)) {
        set_error("gsb_backward_batch_features: dL_dalpha must be a 4-byte aligned float pointer");
        return GSB_ERR_ARGUMENT;
    }
    // gsb_backward_batch_alpha's mode selection (backward_batch_impl refuses features with chunks or peers)
    if (peers) { accumulate = 1; n_chunks = 1; on_chunk = nullptr; }
    return backward_batch_impl(V, s, in, states, out_color, out_invdepth, dL_dcolor, dL_dinvdepth, grads, accumulate, n_chunks, on_chunk,
                               chunk_ctx, alloc, alloc_ctx, static_cast<cudaStream_t>(cuda_stream), peers, cam_grads, dL_dalpha,
                               features);
}

// ---- peer memory (one process per GPU of a node): allocation + CUDA IPC, for the fused reduce-scatter ----
#ifdef GSB_HOST_EMUL   // tests/host_emul: one process, plain pointers; the IPC entry points do not exist there
int32_t gsb_enable_peer_access(int32_t) { return GSB_OK; }
int32_t gsb_peer_alloc(size_t bytes, void **ptr, uint8_t *) { *ptr = calloc(1, bytes ? bytes : 1); return *ptr ? GSB_OK : GSB_ERR_ALLOC; }
int32_t gsb_peer_open(const uint8_t *, void **) { set_error("gsb_peer_open: no IPC on the host build"); return GSB_ERR_CUDA; }
int32_t gsb_peer_close(void *) { return GSB_OK; }
int32_t gsb_peer_free(void *ptr) { free(ptr); return GSB_OK; }
#else
int32_t gsb_enable_peer_access(int32_t peer_device) {
    int dev = -1;
    GSB_CUDA(cudaGetDevice(&dev));
    if (peer_device == dev) return GSB_OK;
    int can = 0;
    GSB_CUDA(cudaDeviceCanAccessPeer(&can, dev, peer_device));
    if (!can) { set_error("device %d cannot access device %d as a peer", dev, peer_device); return GSB_ERR_CUDA; }
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) { (void)cudaGetLastError(); return GSB_OK; }
    if (e != cudaSuccess) { set_error("cudaDeviceEnablePeerAccess(%d) failed: %s", peer_device, cudaGetErrorString(e)); return GSB_ERR_CUDA; }
    return GSB_OK;
}

int32_t gsb_peer_alloc(size_t bytes, void **ptr, uint8_t *handle64) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    if (!ptr || !handle64 || bytes == 0) { set_error("gsb_peer_alloc: bad argument"); return GSB_ERR_ARGUMENT; }
    GSB_CUDA(cudaMalloc(ptr, bytes));
    GSB_CUDA(cudaMemset(*ptr, 0, bytes));
    cudaIpcMemHandle_t h;
    GSB_CUDA(cudaIpcGetMemHandle(&h, *ptr));
    memcpy(handle64, &h, 64);
    return GSB_OK;
}

int32_t gsb_peer_open(const uint8_t *handle64, void **ptr) {
    if (!ptr || !handle64) { set_error("gsb_peer_open: bad argument"); return GSB_ERR_ARGUMENT; }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    // opened on the CURRENT device (the one whose kernels will dereference it): the lazy flag sets up peer access to the
    // exporting device's memory for exactly this mapping
    GSB_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return GSB_OK;
}

int32_t gsb_peer_close(void *ptr) {
    if (ptr) GSB_CUDA(cudaIpcCloseMemHandle(ptr));
    return GSB_OK;
}

int32_t gsb_peer_free(void *ptr) {
    if (ptr) GSB_CUDA(cudaFree(ptr));
    return GSB_OK;
}
#endif

int32_t gsb_mark_visible(int32_t P, const float *means3D, const float *viewmatrix, const float *projmatrix,
                         uint8_t *present, void *cuda_stream) {
    (void)projmatrix;
    if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) {
        set_error("gsb_mark_visible: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    return launch_mark_visible(P, means3D, viewmatrix, present, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_l1_loss_grad(const float *image, const float *target, int64_t n, float scale, float *grad_out,
                         float *loss_accum, void *cuda_stream) {
    if (n < 0 || (n > 0 && (!image || !target || !grad_out || !loss_accum))) {
        set_error("gsb_l1_loss_grad: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    return launch_l1_loss_grad(image, target, n, scale, grad_out, loss_accum, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_photometric_loss_grad(const float *image, const float *target, int32_t channels, int32_t height, int32_t width,
                                  float lambda_dssim, int32_t clamp_input, float *grad_out, float *loss_accum, gsb_alloc_fn alloc,
                                  void *alloc_ctx, void *cuda_stream) {
    if (channels < 0 || height < 0 || width < 0 || !alloc ||
        ((size_t)channels * height * width > 0 && (!image || !target || !grad_out || !loss_accum))) {
        set_error("gsb_photometric_loss_grad: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    const size_t n = (size_t)channels * height * width;
    if (n == 0) return GSB_OK;
    float *maps = static_cast<float *>(do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH2, 3 * n * sizeof(float)));
    if (!maps) return GSB_ERR_ALLOC;
    return launch_photometric_loss_grad(image, target, channels, height, width, lambda_dssim, clamp_input != 0, grad_out, loss_accum, maps,
                                        static_cast<cudaStream_t>(cuda_stream));
}

static bool store_fits_u32(int64_t P, int32_t sh_coeffs, int32_t n_children) {
    const int64_t width = 11 + 3 * (int64_t)sh_coeffs;
    return P >= 0 && P * width < ((int64_t)1 << 32) - 4096 && P * (2 + (int64_t)n_children) < ((int64_t)1 << 32) - 4096;
}

int32_t gsb_adam_step(const GsbAdamArgs *a, void *cuda_stream) {
    if (!a || a->P < 0 || a->sh_coeffs < 1 || !store_fits_u32(a->P, a->sh_coeffs, 0) ||
        (a->P > 0 && (!a->params || !a->grads || !a->exp_avg || !a->exp_avg_sq)) || (a->skip_groups & ~0x3f)) {
        set_error("gsb_adam_step: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    for (int g = 0; g < 6; ++g)
        if (!((a->skip_groups >> g) & 1) && !(a->bias2_sqrt[g] > 0.0f)) {
            set_error("gsb_adam_step: bias2_sqrt[%d] must be > 0", g);
            return GSB_ERR_ARGUMENT;
        }
    if ((a->skip_groups & 0x3f) == 0x3f) return GSB_OK;
    return launch_adam_step(a->P, a->sh_coeffs, a->params, a->grads, a->exp_avg, a->exp_avg_sq, a->act, a->visible, a->step_size,
                            a->beta1, a->beta2, a->eps, a->bias2_sqrt, (uint32_t)a->skip_groups, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_sparse_adam_step(const GsbSparseAdamGroup *groups, int32_t n_groups, const uint8_t *visible, int64_t N, float beta1,
                             float beta2, void *cuda_stream) {
    if (!groups || n_groups < 1 || n_groups > GSB_MAX_SPARSE_GROUPS || N < 0 || (N > 0 && !visible)) {
        set_error("gsb_sparse_adam_step: bad argument (n_groups %d outside 1..%d, N %lld)", n_groups, GSB_MAX_SPARSE_GROUPS, (long long)N);
        return GSB_ERR_ARGUMENT;
    }
    for (int k = 0; k < n_groups; ++k) {
        const GsbSparseAdamGroup &g = groups[k];
        if (g.width <= 0 || N * (int64_t)g.width >= ((int64_t)1 << 31) ||
            (N > 0 && (!g.param || !g.grad || !g.exp_avg || !g.exp_avg_sq))) {
            set_error("gsb_sparse_adam_step: group %d: width %d must be positive, N * width below 2^31, pointers non-NULL", k, g.width);
            return GSB_ERR_ARGUMENT;
        }
    }
    return launch_sparse_adam_step(groups, n_groups, visible, N, beta1, beta2, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_activate(int64_t P, int32_t sh_coeffs, const float *params, float *act, void *cuda_stream) {
    if (P < 0 || sh_coeffs < 1 || !store_fits_u32(P, sh_coeffs, 0) || (P > 0 && (!params || !act))) {
        set_error("gsb_activate: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    return launch_activate(P, sh_coeffs, params, act, static_cast<cudaStream_t>(cuda_stream));
}

size_t gsb_densify_scratch_bytes(int64_t P, int32_t n_children) { return densify_scratch_bytes(P < 0 ? 0 : P, n_children < 1 ? 1 : n_children); }

static bool densify_args_ok(const GsbDensifyArgs *a) {
    return a && a->P >= 0 && a->sh_coeffs >= 1 && a->n_children >= 1 && a->n_children <= 8 &&
           store_fits_u32(a->P, a->sh_coeffs, a->n_children) && (a->P == 0 || (a->params && a->scratch));
}

int32_t gsb_densify_plan(const GsbDensifyArgs *a, int64_t counts[4], void *cuda_stream) {
    if (!densify_args_ok(a) || !counts || (a->P > 0 && (!a->grad_accum || !a->denom)) || !(a->grad_threshold > 0.0f)) {
        set_error("gsb_densify_plan: bad argument (grad_threshold must be > 0)");
        return GSB_ERR_ARGUMENT;
    }
    counts[0] = counts[1] = counts[2] = counts[3] = 0;
    if (a->P == 0) return GSB_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    uint32_t *dev = nullptr;
    const int e = launch_densify_plan(a->P, a->sh_coeffs, a->n_children, a->params, a->grad_accum, a->denom, a->grad_threshold,
                                      a->size_limit, a->min_opacity, a->world_limit, a->scratch, &dev, stream);
    if (e) return e;
    uint32_t host[8];
    GSB_CUDA(cudaMemcpyAsync(host, dev, sizeof(host), cudaMemcpyDeviceToHost, stream));
    GSB_CUDA(cudaStreamSynchronize(stream));
    for (int k = 0; k < 4; ++k) counts[k] = host[k];
    if (host[4] != host[1]) {
        set_error("gsb_densify_plan: split count mismatch (%u vs %u)", host[4], host[1]);
        return GSB_ERR_CUDA;
    }
    return GSB_OK;
}

int32_t gsb_densify_apply(const GsbDensifyArgs *a, const float *unit_samples, int64_t n_split, int64_t P_new, float *new_params,
                          float *new_exp_avg, float *new_exp_avg_sq, void *cuda_stream) {
    if (!densify_args_ok(a) || n_split < 0 || P_new < 0 || (n_split > 0 && !unit_samples) ||
        !store_fits_u32(P_new, a->sh_coeffs, 0) ||
        (P_new > 0 && (!new_params || !new_exp_avg || !new_exp_avg_sq || !a->exp_avg || !a->exp_avg_sq))) {
        set_error("gsb_densify_apply: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    if (a->P == 0) return GSB_OK;
    return launch_densify_apply(a->P, a->sh_coeffs, a->n_children, a->params, a->exp_avg, a->exp_avg_sq, a->scratch, unit_samples,
                                n_split, P_new, new_params, new_exp_avg, new_exp_avg_sq, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_prune_plan(int64_t P, const uint8_t *remove, void *scratch, int64_t *P_new, void *cuda_stream) {
    if (P < 0 || !P_new || !store_fits_u32(P, 1, 1) || (P > 0 && (!remove || !scratch))) {
        set_error("gsb_prune_plan: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    *P_new = 0;
    if (P == 0) return GSB_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    uint32_t *dev = nullptr;
    const int e = launch_prune_plan(P, remove, scratch, &dev, stream);
    if (e) return e;
    uint32_t host = 0;
    GSB_CUDA(cudaMemcpyAsync(&host, dev, sizeof(host), cudaMemcpyDeviceToHost, stream));
    GSB_CUDA(cudaStreamSynchronize(stream));
    *P_new = host;
    return GSB_OK;
}

int32_t gsb_prune_apply(int64_t P, int32_t sh_coeffs, const float *params, const float *exp_avg, const float *exp_avg_sq,
                        const void *scratch, int64_t P_new, float *new_params, float *new_exp_avg, float *new_exp_avg_sq,
                        void *cuda_stream) {
    if (P < 0 || sh_coeffs < 1 || P_new < 0 || P_new > P || !store_fits_u32(P, sh_coeffs, 1) ||
        (P_new > 0 && (!params || !exp_avg || !exp_avg_sq || !scratch || !new_params || !new_exp_avg || !new_exp_avg_sq))) {
        set_error("gsb_prune_apply: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    return launch_prune_apply(P, sh_coeffs, params, exp_avg, exp_avg_sq, scratch, P_new, new_params, new_exp_avg, new_exp_avg_sq,
                              static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_knn_mean_dist2(const float *points, int64_t P, float *out, gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream) {
    if (P < 0 || P >= ((int64_t)1 << 31) || !alloc || (P > 0 && (!points || !out))) {
        set_error("gsb_knn_mean_dist2: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    if (P == 0) return GSB_OK;
    void *scr = do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH0, knn_scratch_bytes(P));
    if (!scr) return GSB_ERR_ALLOC;
    return launch_knn_mean_dist2(points, P, out, scr, static_cast<cudaStream_t>(cuda_stream));
}

int32_t gsb_sort_pairs(uint32_t *keys, uint32_t *vals, int64_t n, int32_t begin_bit, int32_t end_bit,
                       gsb_alloc_fn alloc, void *alloc_ctx, void *cuda_stream) {
    if (n < 0 || (n > 0 && (!keys || !vals)) || !alloc || begin_bit < 0 || end_bit > 32 || begin_bit > end_bit) {
        set_error("gsb_sort_pairs: bad argument");
        return GSB_ERR_ARGUMENT;
    }
    if (n == 0) return GSB_OK;
    Carver c(nullptr);
    c.take<uint32_t>((size_t)n); c.take<uint32_t>((size_t)n); c.take<char>(sort_scratch_bytes(n));
    void *scr = do_alloc(alloc, alloc_ctx, GSB_BUF_SCRATCH0, c.bytes());
    if (!scr) return GSB_ERR_ALLOC;
    Carver cr(scr);
    uint32_t *ka = cr.take<uint32_t>((size_t)n), *va = cr.take<uint32_t>((size_t)n);
    char *ss = cr.take<char>(sort_scratch_bytes(n));
    return sort_pairs(keys, vals, ka, va, n, nullptr, begin_bit, end_bit, ss, false, static_cast<cudaStream_t>(cuda_stream));
}

}  // extern "C"
