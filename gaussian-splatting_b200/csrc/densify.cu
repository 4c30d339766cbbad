// densify.cu -- densify_and_prune with the optimizer-state surgery (SURVEY.md section 8(f) #1; scene/gaussian_model.py:316-469)
// on the flat store.  The reference builds the new tensors with ~60 boolean-mask gathers and cats and a dozen host
// synchronisations; here the decision for every possible output row is taken in one pass over the P originals
// (classify), two exclusive scans give the split ranks and the output positions, and ONE gather writes the new store and
// both Adam moments (byte mover: reads and writes each surviving float once).
//
// Candidate slots, in the reference's final row order (N = n_children):
//   [0, P)              original i             kept unless split or pruned
//   [P, 2P)             clone of i             exists if clone-selected; kept unless pruned (same opacity / scale as i)
//   [2P + kP, 2P+(k+1)P) child k of i          exists if split-selected; kept unless pruned with the CHILD's scale
#include "common.cuh"
#include "kernels.cuh"

namespace gsb {

constexpr int DS_THREADS = 256, DS_ITEMS = 8, DS_CHUNK = DS_THREADS * DS_ITEMS;

struct StoreLayout {
    uint32_t P, F;                              // rows, floats per features row
    __host__ __device__ size_t feat() const { return 3u * (size_t)P; }
    __host__ __device__ size_t op() const { return feat() + (size_t)F * P; }
    __host__ __device__ size_t sc() const { return op() + P; }
    __host__ __device__ size_t rot() const { return sc() + 3u * (size_t)P; }
    __host__ __device__ size_t total() const { return rot() + 4u * (size_t)P; }
};

// scratch carving (device): keep flags / output positions [S], split flags / ranks [P], source slot of every output row [S],
// scan partials, counters
struct DensifyScratch {
    uint32_t *pos, *rank, *src, *partials, *counters;   // counters: n_clone, n_split, n_pruned, P_new, n_split (scan total)
};

static size_t partial_count(int64_t n) { return (size_t)ceil_div(n > 0 ? n : 1, DS_CHUNK) + 1; }

static DensifyScratch carve_densify(void *base, int64_t P, int n_children, size_t *bytes) {
    const size_t S = (size_t)(2 + n_children) * (size_t)P;
    Carver c(static_cast<char *>(base));
    DensifyScratch s;
    s.pos = c.take<uint32_t>(S);
    s.rank = c.take<uint32_t>((size_t)P);
    s.src = c.take<uint32_t>(S);
    s.partials = c.take<uint32_t>(partial_count((int64_t)S));
    s.counters = c.take<uint32_t>(8);
    if (bytes) *bytes = c.bytes();
    return s;
}

size_t densify_scratch_bytes(int64_t P, int n_children) {
    size_t b = 0;
    carve_densify(nullptr, P, n_children, &b);
    return b;
}

// ---- exclusive scan of uint32 (three small kernels; in == out allowed) -------------------------------------------------
__device__ __forceinline__ uint32_t block_excl_scan(const uint32_t v, uint32_t *warp_sums, uint32_t &total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t n = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += n;
    }
    if (lane == 31) warp_sums[w] = inc;
    __syncthreads();
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (int k = 0; k < DS_THREADS / 32; ++k) {
        const uint32_t s = warp_sums[k];
        if (k < w) base += s;
        tot += s;
    }
    total = tot;
    __syncthreads();
    return base + inc - v;
}

__global__ void __launch_bounds__(DS_THREADS)
ds_reduce_kernel(const uint32_t *__restrict__ in, const size_t n, uint32_t *__restrict__ partials) {
    __shared__ uint32_t warp_sums[DS_THREADS / 32];
    const size_t first = (size_t)blockIdx.x * DS_CHUNK + (size_t)threadIdx.x * DS_ITEMS;
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < DS_ITEMS; ++k)
        if (first + k < n) s += in[first + k];
    uint32_t total;
    block_excl_scan(s, warp_sums, total);
    if (threadIdx.x == 0) partials[blockIdx.x] = total;
}

__global__ void __launch_bounds__(DS_THREADS)
ds_partials_kernel(uint32_t *partials, const int n, uint32_t *total_out) {
    __shared__ uint32_t warp_sums[DS_THREADS / 32];
    uint32_t carry = 0;
    for (int base = 0; base < n; base += DS_THREADS) {
        const int i = base + threadIdx.x;
        const uint32_t v = i < n ? partials[i] : 0u;
        uint32_t total;
        const uint32_t excl = block_excl_scan(v, warp_sums, total);
        if (i < n) partials[i] = carry + excl;
        carry += total;
    }
    if (threadIdx.x == 0) *total_out = carry;
}

__global__ void __launch_bounds__(DS_THREADS)
ds_apply_kernel(const uint32_t *in, uint32_t *out, const size_t n, const uint32_t *__restrict__ partials) {
    __shared__ uint32_t warp_sums[DS_THREADS / 32];
    const size_t first = (size_t)blockIdx.x * DS_CHUNK + (size_t)threadIdx.x * DS_ITEMS;
    uint32_t v[DS_ITEMS], s = 0;
#pragma unroll
    for (int k = 0; k < DS_ITEMS; ++k) {
        v[k] = first + k < n ? in[first + k] : 0u;
        s += v[k];
    }
    uint32_t total;
    uint32_t run = block_excl_scan(s, warp_sums, total) + partials[blockIdx.x];
#pragma unroll
    for (int k = 0; k < DS_ITEMS; ++k) {
        if (first + k < n) out[first + k] = run;
        run += v[k];
    }
}

static int exclusive_scan_u32(const uint32_t *in, uint32_t *out, size_t n, uint32_t *partials, uint32_t *total, cudaStream_t stream) {
    const int chunks = (int)ceil_div((int64_t)(n > 0 ? n : 1), DS_CHUNK);
    GSB_LAUNCH("densify_scan_reduce", false, stream, ds_reduce_kernel, chunks, DS_THREADS, 0, in, n, partials);
    GSB_LAUNCH("densify_scan_partials", false, stream, ds_partials_kernel, 1, DS_THREADS, 0, partials, chunks, total);
    GSB_LAUNCH("densify_scan_apply", false, stream, ds_apply_kernel, chunks, DS_THREADS, 0, in, out, n, partials);
    return GSB_OK;
}

// shared with knn.cu
size_t scan_u32_partials(int64_t n) { return partial_count(n); }
int scan_u32_exclusive(const uint32_t *in, uint32_t *out, size_t n, uint32_t *partials, uint32_t *total, cudaStream_t stream) {
    return exclusive_scan_u32(in, out, n, partials, total, stream);
}

// ---- classification ------------------------------------------------------------------------------------------------------
struct ClassifyArgs {
    uint32_t P;
    int N;
    const float *opacity, *scaling, *accum, *denom;
    float grad_threshold, size_limit, min_opacity, world_limit;
    uint32_t *keep, *split, *counters;
};

__global__ void __launch_bounds__(DS_THREADS)
densify_classify_kernel(const ClassifyArgs a) {
    const uint32_t i = blockIdx.x * DS_THREADS + threadIdx.x;
    uint32_t n_clone = 0, n_split = 0, n_pruned = 0;
    if (i < a.P) {
        float g = a.accum[i] / a.denom[i];                                   // grads = xyz_gradient_accum / denom; NaN -> 0 (:453-454)
        if (isnan(g)) g = 0.0f;
        const float s0 = a.scaling[3u * (size_t)i], s1 = a.scaling[3u * (size_t)i + 1], s2 = a.scaling[3u * (size_t)i + 2];
        const float e0 = expf(s0), e1 = expf(s1), e2 = expf(s2);
        const float big = fmaxf(e0, fmaxf(e1, e2));
        const bool hot_clone = fabsf(g) >= a.grad_threshold;                 // torch.norm(grads, dim=-1) of a [P,1] tensor (:434)
        const bool hot_split = g >= a.grad_threshold;                        // padded_grad >= threshold (:404)
        const bool clone = hot_clone && big <= a.size_limit;
        const bool split = hot_split && big > a.size_limit;
        const bool transparent = 1.0f / (1.0f + expf(-a.opacity[i])) < a.min_opacity;
        const bool drop_self = transparent || (a.world_limit >= 0.0f && big > a.world_limit);
        const float den = 0.8f * (float)a.N;                                 // children: log(scale / (0.8 N)) (:411), re-activated
        const float c_big = fmaxf(expf(logf(e0 / den)), fmaxf(expf(logf(e1 / den)), expf(logf(e2 / den))));
        const bool drop_child = transparent || (a.world_limit >= 0.0f && c_big > a.world_limit);
        a.keep[i] = (!split && !drop_self) ? 1u : 0u;
        a.keep[a.P + i] = (clone && !drop_self) ? 1u : 0u;
        for (int k = 0; k < a.N; ++k) a.keep[(size_t)(2 + k) * a.P + i] = (split && !drop_child) ? 1u : 0u;
        a.split[i] = split ? 1u : 0u;
        n_clone = clone;
        n_split = split;
        n_pruned = ((!split && drop_self) ? 1u : 0u) + ((clone && drop_self) ? 1u : 0u) + ((split && drop_child) ? (uint32_t)a.N : 0u);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        n_clone += __shfl_xor_sync(0xffffffffu, n_clone, o);
        n_split += __shfl_xor_sync(0xffffffffu, n_split, o);
        n_pruned += __shfl_xor_sync(0xffffffffu, n_pruned, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (n_clone) atomicAdd(a.counters + 0, n_clone);
        if (n_split) atomicAdd(a.counters + 1, n_split);
        if (n_pruned) atomicAdd(a.counters + 2, n_pruned);
    }
}

// source slot of every output row
__global__ void __launch_bounds__(DS_THREADS)
densify_invert_kernel(const uint32_t *__restrict__ keep_pos, const uint32_t *__restrict__ total, const size_t S, uint32_t *__restrict__ src) {
    const size_t c = (size_t)blockIdx.x * DS_THREADS + threadIdx.x;
    if (c >= S) return;
    const uint32_t here = keep_pos[c], next = c + 1 < S ? keep_pos[c + 1] : *total;
    if (next != here) src[here] = (uint32_t)c;       // exclusive scan of 0/1 flags: the slot is kept iff the position advances
}

// ---- gather ---------------------------------------------------------------------------------------------------------------
struct GatherArgs {
    StoreLayout o, n;                     // old and new layouts
    int N;
    uint32_t n_split;
    const float *p, *m, *v;               // old store
    float *np, *nm, *nv;                  // new store
    const uint32_t *src, *rank;
    const float *unit;                    // [N * n_split, 3]
};

__global__ void __launch_bounds__(DS_THREADS)
densify_gather_kernel(const GatherArgs a) {
    const size_t e = (size_t)blockIdx.x * DS_THREADS + threadIdx.x;
    if (e >= a.n.total()) return;
    // decode (group, row, column) of the NEW store
    int grp; uint32_t w; size_t nbase, obase;
    if (e < a.n.feat()) { grp = 0; w = 3; nbase = 0; obase = 0; }
    else if (e < a.n.op()) { grp = 1; w = a.n.F; nbase = a.n.feat(); obase = a.o.feat(); }
    else if (e < a.n.sc()) { grp = 2; w = 1; nbase = a.n.op(); obase = a.o.op(); }
    else if (e < a.n.rot()) { grp = 3; w = 3; nbase = a.n.sc(); obase = a.o.sc(); }
    else { grp = 4; w = 4; nbase = a.n.rot(); obase = a.o.rot(); }
    const uint32_t rel = (uint32_t)(e - nbase);
    const uint32_t r = rel / w, col = rel - r * w;
    const uint32_t c = a.src[r];
    const uint32_t kind = c / a.o.P, i = c - kind * a.o.P;         // 0 original, 1 clone, 2 + k child k
    const size_t oe = obase + (size_t)i * w + col;
    float val = a.p[oe];
    if (kind >= 2u) {
        if (grp == 0) {
            // new_xyz = R(q_i) (unit * exp(scaling_i)) + xyz_i  (:406-410)
            const float *q = a.p + a.o.rot() + 4u * (size_t)i, *s = a.p + a.o.sc() + 3u * (size_t)i;
            const float *u = a.unit + 3u * ((size_t)(kind - 2u) * a.n_split + a.rank[i]);
            const float nq = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
            const float r0 = q[0] / nq, x = q[1] / nq, y = q[2] / nq, z = q[3] / nq;
            const float t0 = u[0] * expf(s[0]), t1 = u[1] * expf(s[1]), t2 = u[2] * expf(s[2]);
            float R0, R1, R2;
            if (col == 0) { R0 = 1.f - 2.f * (y * y + z * z); R1 = 2.f * (x * y - r0 * z); R2 = 2.f * (x * z + r0 * y); }
            else if (col == 1) { R0 = 2.f * (x * y + r0 * z); R1 = 1.f - 2.f * (x * x + z * z); R2 = 2.f * (y * z - r0 * x); }
            else { R0 = 2.f * (x * z - r0 * y); R1 = 2.f * (y * z + r0 * x); R2 = 1.f - 2.f * (x * x + y * y); }
            val = (R0 * t0 + R1 * t1 + R2 * t2) + val;
        } else if (grp == 3) {
            val = logf(expf(val) / (0.8f * (float)a.N));
        }
    }
    a.np[e] = val;
    a.nm[e] = kind == 0u ? a.m[oe] : 0.0f;
    a.nv[e] = kind == 0u ? a.v[oe] : 0.0f;
}

int launch_densify_plan(int64_t P, int sh_coeffs, int n_children, const float *params, const float *grad_accum, const float *denom,
                        float grad_threshold, float size_limit, float min_opacity, float world_limit, void *scratch,
                        uint32_t **counters_dev, cudaStream_t stream) {
    const DensifyScratch s = carve_densify(scratch, P, n_children, nullptr);
    const size_t S = (size_t)(2 + n_children) * (size_t)P;
    StoreLayout L{(uint32_t)P, 3u * (uint32_t)sh_coeffs};
    cudaError_t err = cudaMemsetAsync(s.counters, 0, 8 * sizeof(uint32_t), stream);
    if (err != cudaSuccess) { set_error("densify: memset failed: %s", cudaGetErrorString(err)); return GSB_ERR_CUDA; }
    ClassifyArgs a;
    a.P = (uint32_t)P; a.N = n_children;
    a.opacity = params + L.op(); a.scaling = params + L.sc(); a.accum = grad_accum; a.denom = denom;
    a.grad_threshold = grad_threshold; a.size_limit = size_limit; a.min_opacity = min_opacity; a.world_limit = world_limit;
    a.keep = s.pos; a.split = s.rank; a.counters = s.counters;
    GSB_LAUNCH("densify_classify", false, stream, densify_classify_kernel, (uint32_t)ceil_div(P, DS_THREADS), DS_THREADS, 0, a);
    int e = exclusive_scan_u32(s.rank, s.rank, (size_t)P, s.partials, s.counters + 4, stream);
    if (e) return e;
    e = exclusive_scan_u32(s.pos, s.pos, S, s.partials, s.counters + 3, stream);
    if (e) return e;
    GSB_LAUNCH("densify_invert", false, stream, densify_invert_kernel, (uint32_t)ceil_div((int64_t)S, DS_THREADS), DS_THREADS, 0, s.pos,
               s.counters + 3, S, s.src);
    *counters_dev = s.counters;
    return GSB_OK;
}

int launch_densify_apply(int64_t P, int sh_coeffs, int n_children, const float *params, const float *m, const float *v, void *scratch,
                         const float *unit_samples, int64_t n_split, int64_t P_new, float *new_params, float *new_m, float *new_v,
                         cudaStream_t stream) {
    if (P_new == 0) return GSB_OK;
    const DensifyScratch s = carve_densify(scratch, P, n_children, nullptr);
    GatherArgs a;
    a.o = StoreLayout{(uint32_t)P, 3u * (uint32_t)sh_coeffs};
    a.n = StoreLayout{(uint32_t)P_new, 3u * (uint32_t)sh_coeffs};
    a.N = n_children; a.n_split = (uint32_t)n_split;
    a.p = params; a.m = m; a.v = v; a.np = new_params; a.nm = new_m; a.nv = new_v;
    a.src = s.src; a.rank = s.rank; a.unit = unit_samples;
    GSB_LAUNCH("densify_gather", false, stream, densify_gather_kernel, (uint32_t)ceil_div((int64_t)a.n.total(), DS_THREADS), DS_THREADS, 0, a);
    return GSB_OK;
}

// ---- prune_points (scene/gaussian_model.py:349-364): the densify pipeline with originals only --------------------------------
// keep flags -> exclusive scan (output positions, P_new) -> source row of every output row -> densify_gather_kernel with
// n_children = 1 and no clone / child slot kept, i.e. every output row an original that keeps its moments.
__global__ void __launch_bounds__(DS_THREADS)
prune_keep_kernel(const uint8_t *__restrict__ remove, const uint32_t P, uint32_t *__restrict__ keep) {
    const uint32_t i = blockIdx.x * DS_THREADS + threadIdx.x;
    if (i < P) keep[i] = remove[i] ? 0u : 1u;
}

int launch_prune_plan(int64_t P, const uint8_t *remove, void *scratch, uint32_t **counter_dev, cudaStream_t stream) {
    const DensifyScratch s = carve_densify(scratch, P, 1, nullptr);
    GSB_LAUNCH("prune_keep", false, stream, prune_keep_kernel, (uint32_t)ceil_div(P, DS_THREADS), DS_THREADS, 0, remove, (uint32_t)P, s.pos);
    const int e = exclusive_scan_u32(s.pos, s.pos, (size_t)P, s.partials, s.counters + 3, stream);
    if (e) return e;
    GSB_LAUNCH("densify_invert", false, stream, densify_invert_kernel, (uint32_t)ceil_div(P, DS_THREADS), DS_THREADS, 0, s.pos,
               s.counters + 3, (size_t)P, s.src);
    *counter_dev = s.counters + 3;
    return GSB_OK;
}

int launch_prune_apply(int64_t P, int sh_coeffs, const float *params, const float *m, const float *v, const void *scratch, int64_t P_new,
                       float *new_params, float *new_m, float *new_v, cudaStream_t stream) {
    if (P_new == 0) return GSB_OK;
    const DensifyScratch s = carve_densify(const_cast<void *>(scratch), P, 1, nullptr);
    GatherArgs a;
    a.o = StoreLayout{(uint32_t)P, 3u * (uint32_t)sh_coeffs};
    a.n = StoreLayout{(uint32_t)P_new, 3u * (uint32_t)sh_coeffs};
    a.N = 1; a.n_split = 0u;
    a.p = params; a.m = m; a.v = v; a.np = new_params; a.nm = new_m; a.nv = new_v;
    a.src = s.src; a.rank = s.rank; a.unit = nullptr;
    GSB_LAUNCH("densify_gather", false, stream, densify_gather_kernel, (uint32_t)ceil_div((int64_t)a.n.total(), DS_THREADS), DS_THREADS, 0, a);
    return GSB_OK;
}

}  // namespace gsb
