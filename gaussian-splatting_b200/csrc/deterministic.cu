// deterministic.cu -- the second half of the deterministic backward (DESIGN.md section 7.9).
//
// With the deterministic switch on, render_bwd_kernel<..., DET = true> does not add a warp's per-gaussian sums into the
// accumulator rows with red.add (whose order depends on CTA scheduling): it stores them into a partial row per (list
// position, warp) and marks the pair.  This file turns those partials into the accumulator rows in a fixed order:
//   det_count    per view, the instance count = the largest tile-range end (no host read-back: the async forward works);
//   det_prepare  keys = a copy of point_list (gaussian ids; the state itself is left alone), values = list positions;
//   sort_pairs   stable onesweep sort on ceil(log2 P) key bits, batched over the views: each gaussian's positions come out
//                ascending, i.e. in ascending tile id, independently of scheduling;
//   det_reduce   one thread per (view, gaussian): the marked partials of its positions, warp 0 then warp 1, summed in float32
//                from 0 and stored as the full accumulator row (zero without entries).
// preprocess_bwd then reads the rows exactly as it reads the red.add ones.
#include "kernels.cuh"

namespace gsb {

__global__ void __launch_bounds__(256)
det_count_kernel(const uint2 *__restrict__ ranges, const int num_tiles, const size_t sv_ranges, unsigned long long *__restrict__ count) {
    __shared__ uint32_t s_max;
    ranges += blockIdx.x * sv_ranges;
    if (threadIdx.x == 0) s_max = 0u;
    __syncthreads();
    uint32_t m = 0u;
    for (int t = threadIdx.x; t < num_tiles; t += 256) m = max(m, ranges[t].y);
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0) atomicMax(&s_max, m);
    __syncthreads();
    if (threadIdx.x == 0) count[blockIdx.x] = s_max;
}

__global__ void __launch_bounds__(256)
det_prepare_kernel(const uint32_t *__restrict__ point_list, const size_t sv_list, const unsigned long long *__restrict__ count,
                   uint32_t *__restrict__ keys, uint32_t *__restrict__ vals, const size_t sv) {
    const size_t v = blockIdx.y;
    const int64_t n = (int64_t)count[v];
    point_list += v * sv_list; keys += v * sv; vals += v * sv;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
        keys[i] = point_list[i];
        vals[i] = (uint32_t)i;
    }
}

// nsum: the partial slots K7 wrote (9, or 10 with the inverse-depth sum)
__global__ void __launch_bounds__(256)
det_reduce_kernel(const uint32_t *__restrict__ keys, const uint32_t *__restrict__ vals, const unsigned long long *__restrict__ count,
                  const float *__restrict__ part, const uint8_t *__restrict__ mark, const size_t sv, const int P, const int nsum,
                  float *__restrict__ dacc) {
    const int g = blockIdx.x * 256 + threadIdx.x;
    if (g >= P) return;
    const size_t v = blockIdx.y;
    const int64_t n = (int64_t)count[v];
    keys += v * sv; vals += v * sv; part += v * sv * 2 * DACC_STRIDE; mark += v * sv * 2;
    int64_t lo = 0, hi = n;     // first sorted entry with key >= g
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < (uint32_t)g) lo = mid + 1; else hi = mid;
    }
    float acc[10];
#pragma unroll
    for (int s = 0; s < 10; ++s) acc[s] = 0.0f;
    for (int64_t i = lo; i < n && keys[i] == (uint32_t)g; ++i) {
        const size_t pos = vals[i];
#pragma unroll
        for (int w = 0; w < 2; ++w) {
            if (!mark[pos * 2 + w]) continue;
            const float4 *r = reinterpret_cast<const float4 *>(part + (pos * 2 + w) * DACC_STRIDE);
            const float4 a = r[0], b = r[1];
            const float2 c = *reinterpret_cast<const float2 *>(r + 2);
            const float x[10] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y};
#pragma unroll
            for (int s = 0; s < 10; ++s)
                if (s < nsum) acc[s] = __fadd_rn(acc[s], x[s]);
        }
    }
    float4 *out = reinterpret_cast<float4 *>(dacc + (v * (size_t)P + g) * DACC_STRIDE);
    out[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    out[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    out[2] = make_float4(acc[8], acc[9], 0.0f, 0.0f);
}

size_t det_carve(void *base, int64_t capn, int V, DetScratch &d) {
    Carver c(base);
    const size_t n = (size_t)V * capn;
    d.part = c.take<float>(n * 2 * DACC_STRIDE);
    d.mark = c.take<uint8_t>(n * 2);
    d.keys = c.take<uint32_t>(n); d.vals = c.take<uint32_t>(n);
    d.keys_alt = c.take<uint32_t>(n); d.vals_alt = c.take<uint32_t>(n);
    d.count = c.take<unsigned long long>(GSB_MAX_VIEWS);
    d.sortscr = c.take<char>(sort_scratch_bytes(capn, V));
    d.capn = capn;
    return c.bytes();
}

int launch_det_reduce(const RenderBwdArgs &a, const DetScratch &d, int P, float *dacc, bool debug, cudaStream_t stream) {
    if (P <= 0) return GSB_OK;
    const int V = a.V, num_tiles = a.gx * a.gy;
    const size_t sv = (size_t)d.capn;
    if (V > 1 && a.sv_list != sv) {
        set_error("det_reduce: point-list stride %zu differs from the capacity %zu", a.sv_list, sv);
        return GSB_ERR_ARGUMENT;
    }
    GSB_LAUNCH("det_count", debug, stream, det_count_kernel, V, 256, 0, a.ranges, num_tiles, a.sv_ranges, d.count);
    const int64_t pblocks = ceil_div(d.capn, 256 * 4);
    GSB_LAUNCH("det_prepare", debug, stream, det_prepare_kernel, dim3((unsigned)(pblocks < NUM_SMS * 16 ? pblocks : NUM_SMS * 16), V), 256,
               0, a.point_list, a.sv_list, d.count, d.keys, d.vals, sv);
    int bits = 1;
    while (bits < 32 && ((uint32_t)(P - 1) >> bits) != 0u) ++bits;
    int rc = sort_pairs(d.keys, d.vals, d.keys_alt, d.vals_alt, d.capn, d.count, 0, bits, d.sortscr, debug, stream, V, sv);
    if (rc) return rc;
    GSB_LAUNCH("det_reduce", debug, stream, det_reduce_kernel, dim3((unsigned)ceil_div(P, 256), V), 256, 0, d.keys, d.vals, d.count,
               d.part, d.mark, sv, P, a.dL_dinvdepth ? 10 : 9, dacc);
    return GSB_OK;
}

}  // namespace gsb
