// contrib.cu -- per-gaussian contribution statistics of finished forward states (gsb_contribution; DESIGN.md section 7.8).
//
// For every pair (pixel p, gaussian k) a forward accepted -- power <= 0, alpha >= 1/255, list position <= n_contrib[p], the
// rules of render_features_kernel (features.cu) -- with blend weight w_k(p) = alpha_k T_k:
//     count[k] += 1,   weight_sum[k] += w_k(p),   weight_max[k] = max(weight_max[k], w_k(p))
// summed over the pixels of every view of the launch.  These are the usage scores of contribution-based pruning (sum of
// weights, max weight, number of pixels).
//
// Nothing is binned again: the kernel reads a forward state (ranges, point_list, tile_order, the 48-byte splat records and
// n_contrib) in K6's layout -- one pixel per thread, a warp per 8x4 patch, patch-mask compaction -- and walks each pixel's list
// up to n_contrib with render_features_kernel's per-pair arithmetic, so w is bit-equal to the weight the blend used.  Per
// staged entry the warp reduces its 32 pixels first (ballot popcount, shuffle sum, max over the float bits, w >= 0) and lane 0
// issues at most one atomic of each kind: global atomics per (warp, entry) with a hit, never per pair.  (Reducing the 8 warps
// of a CTA in shared memory first, one global atomic per (CTA, entry), measured slower on the H100: DESIGN.md section 7.8.)
#include "blend_common.cuh"

namespace gsb {

constexpr int CONTRIB_RB = 256;     // gaussians staged per round
constexpr int CONTRIB_MINB = 4;     // CTAs per SM the kernel is compiled for (register table in DESIGN.md section 7.8)

struct alignas(16) ContribRec {
    ulonglong2 w0;      // {(x, y), (A', C')} as two f32x2 (blend_common.cuh stage_scale)
    float bp, op;       // B', opacity
    uint32_t id, pad;   // gaussian id
};

// the forward state of view v, selected with uniform compares (a dynamic index would copy the parameter block to local memory)
__device__ __forceinline__ FeatView contrib_view(const ContribArgs &a, const int v) {
    FeatView f = a.view[0];
#pragma unroll
    for (int k = 1; k < GSB_MAX_VIEWS; ++k)
        if (k == v) f = a.view[k];
    return f;
}

__device__ __forceinline__ uint8_t stage_contrib(ContribRec &dst, const float4 *splat, const uint32_t g, const float ox, const float oy) {
    const float4 *rec = splat + (size_t)g * SPLAT_F4;
    float4 q0 = __ldg(rec), q1 = __ldg(rec + 1);
    const float4 q2 = __ldg(rec + 2);
    const uint8_t mask = (uint8_t)patch_mask(q0.x, q0.y, q0.z, q0.w, q1.x, q2.z, ox, oy);
    stage_scale(q0, q1);
    dst.w0 = make_ulonglong2(pk(q0.x, q0.y), pk(q0.z, q0.w));
    dst.bp = q1.x; dst.op = q1.y; dst.id = g; dst.pad = 0u;
    return mask;
}

__global__ void __launch_bounds__(256, CONTRIB_MINB)
contribution_kernel(const ContribArgs a) {
    constexpr int WARPS = 8;
    __shared__ ContribRec srec[CONTRIB_RB];
    __shared__ uint8_t smask[CONTRIB_RB];
    __shared__ uint8_t slist[WARPS][CONTRIB_RB];
    __shared__ uint32_t s_max;
    const int v = (int)blockIdx.y;
    const FeatView f = contrib_view(a, v);
    const int tile = f.tile_order ? (int)f.tile_order[blockIdx.x] : (int)blockIdx.x;
    const int tile_x = tile % a.gx, tile_y = tile / a.gx;
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    const int px = tile_x * TILE + (w & 1) * 8 + (l & 7);     // warp w owns patch w: bit w of the staged masks
    const int py = tile_y * TILE + (w >> 1) * 4 + (l >> 3);
    const bool inside = px < a.W && py < a.H;
    const size_t pid = inside ? (size_t)py * a.W + px : 0;
    const f32x2 negp = pk(-(float)px, -(float)py);
    const float ox = (float)(tile_x * TILE), oy = (float)(tile_y * TILE);
    const uint2 range = f.ranges[tile];
    const uint32_t last = inside ? f.n_contrib[pid] : 0u;
    const int wmax = (int)__reduce_max_sync(0xffffffffu, last);
    // largest n_contrib over the CTA's pixels: list entries behind it blend no pixel of the tile
    if (threadIdx.x == 0) s_max = 0u;
    __syncthreads();
    if (l == 0) atomicMax(&s_max, (uint32_t)wmax);
    __syncthreads();
    const int todo = (int)s_max;

    float T = 1.0f;
    for (int base = 0; base < todo; base += CONTRIB_RB) {
        __syncthreads();
        const int n = min(CONTRIB_RB, todo - base);
        if ((int)threadIdx.x < n)
            smask[threadIdx.x] = stage_contrib(srec[threadIdx.x], f.splat, f.point_list[range.x + base + threadIdx.x], ox, oy);
        __syncthreads();
        const int cnt = compact_hits(smask, max(0, min(n, wmax - base)), 1u << w, slist[w]);
        for (int k = 0; k < cnt; ++k) {
            const int j = slist[w][k];
            const ContribRec &r = srec[j];
            // render_features_kernel's arithmetic, operation for operation
            const f32x2 d2 = add2((f32x2)r.w0.x, negp);
            const f32x2 u2 = mul2(mul2((f32x2)r.w0.y, d2), d2);
            float dx, dy, Axx, Cyy;
            unpk(d2, dx, dy);
            unpk(u2, Axx, Cyy);
            const float power = power2_at(Axx, Cyy, __fmul_rn(r.bp, dx), dy);
            const float alpha = fminf(ALPHA_MAX, __fmul_rn(r.op, ex2_approx(power)));
            const bool ok = alpha >= ALPHA_MIN && power <= 0.0f && (uint32_t)(base + j + 1) <= last;
            const float wgt = ok ? __fmul_rn(alpha, T) : 0.0f;
            T = ok ? __fmul_rn(T, __fsub_rn(1.0f, alpha)) : T;
            const uint32_t hits = __ballot_sync(0xffffffffu, ok);
            if (hits == 0u) continue;                                       // warp-uniform
            float s = wgt;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            const uint32_t mbits = __reduce_max_sync(0xffffffffu, __float_as_uint(wgt));   // w >= 0: bit order = value order
            if (l == 0) {
                atomicAdd(reinterpret_cast<unsigned long long *>(a.count) + r.id, (unsigned long long)__popc(hits));
                atomicAdd(a.weight_sum + r.id, s);
                atomicMax(a.weight_max_bits + r.id, mbits);
            }
        }
    }
}

int launch_contribution(const ContribArgs &a, bool debug, cudaStream_t stream) {
    const int tiles = a.gx * a.gy;
    if (tiles <= 0 || a.P == 0) return GSB_OK;
    if (a.V < 1 || a.V > GSB_MAX_VIEWS || tiles > 0x7fffffff / GSB_MAX_VIEWS) {
        set_error("contribution: bad launch geometry (V=%d, tiles=%d)", a.V, tiles);
        return GSB_ERR_ARGUMENT;
    }
    GSB_LAUNCH("contribution", debug, stream, contribution_kernel, dim3(tiles, a.V, 1), 256, 0, a);
    return GSB_OK;
}

}  // namespace gsb
