// binning.cu -- tile binning: scan of tiles-touched in depth order (K2), instance emission with the tile sort's digit
// histograms (K3) and per-tile ranges of the tile-sorted instance list (K5).
//
// Replaces the cub::DeviceScan::InclusiveSum call, duplicateWithKeys and identifyTileRanges of the
// reference's cuda_rasterizer/rasterizer_impl.cu (named in BASELINE.json north_star; absent from
// /root/reference).  Difference in structure, same resulting order: gaussians are first sorted by
// depth, instances are emitted in that order with the TILE id as the only key, and a stable sort on
// the tile id (radix_sort.cu) then yields per-tile lists ordered by (depth, gaussian index) -- exactly
// what one stable sort on tile<<32|depth keys gives.
#include "kernels.cuh"

namespace gsb {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_IPT = 8;
constexpr int SCAN_CHUNK = SCAN_THREADS * SCAN_IPT;

// per view: a ticket counter, then one status word per chunk (decoupled look-back)
size_t scan_state_count(int P) { return (size_t)ceil_div(P > 0 ? P : 1, SCAN_CHUNK) + 1; }

__device__ __forceinline__ uint32_t block_exclusive_scan_256(const uint32_t v, uint32_t *warp_sums, uint32_t &block_total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[w] = incl;
    __syncthreads();
    uint32_t prefix = 0, total = 0;
#pragma unroll
    for (int k = 0; k < SCAN_THREADS / 32; ++k) {
        const uint32_t s = warp_sums[k];
        if (k < w) prefix += s;
        total += s;
    }
    block_total = total;
    __syncthreads();
    return prefix + incl - v;
}

// status word of a chunk: bits 63..62 = 0 not ready | 1 chunk total | 2 inclusive prefix; bits 61..0 = the sum
#define SCAN_FLAG_AGG (1ull << 62)
#define SCAN_FLAG_PREFIX (2ull << 62)
#define SCAN_VALUE_MASK ((1ull << 62) - 1ull)

// K2: offsets[r] = sum of tiles[order[r']] over r' < r, in one pass.  Chunks take tickets, so a chunk only waits for chunks
// that started before it; warp 0 finds the chunk's prefix by walking back over 32 predecessors' status words at a time.
// The 64-bit running sum gives the exact per-view total (the host rejects totals >= 2^31; offsets are that sum mod 2^32).
__global__ void __launch_bounds__(SCAN_THREADS)
tile_scan_kernel(BinArgs a) {
    __shared__ uint32_t warp_sums[SCAN_THREADS / 32];
    __shared__ uint32_t s_chunk;
    __shared__ unsigned long long s_prefix;
    a.order += blockIdx.y * a.sv_gauss; a.tiles += blockIdx.y * a.sv_gauss; a.offsets += blockIdx.y * a.sv_gauss;
    unsigned long long *ticket = a.scan_state + blockIdx.y * a.sv_scan;
    volatile unsigned long long *status = ticket + 1;
    if (threadIdx.x == 0) s_chunk = (uint32_t)atomicAdd(ticket, 1ull);
    __syncthreads();
    const uint32_t b = s_chunk;
    const int base = (int)b * SCAN_CHUNK + threadIdx.x * SCAN_IPT;
    uint32_t v[SCAN_IPT];
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_IPT; ++k) {
        const int r = base + k;
        v[k] = r < a.P ? a.tiles[a.order[r]] : 0u;
        s += v[k];
    }
    uint32_t total;
    const uint32_t excl = block_exclusive_scan_256(s, warp_sums, total);
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        unsigned long long prefix = 0;
        if (b == 0) {
            if (lane == 0) status[0] = SCAN_FLAG_PREFIX | total;
        } else {
            if (lane == 0) status[b] = SCAN_FLAG_AGG | total;
            for (int64_t q = (int64_t)b - 1 - lane;; q -= 32) {
                unsigned long long w = q >= 0 ? status[q] : SCAN_FLAG_PREFIX;
                while (!__all_sync(0xffffffffu, (w >> 62) != 0ull))
                    if ((w >> 62) == 0ull) w = status[q];
                // the nearest inclusive prefix ends the walk: sum the lanes up to it
                const uint32_t at_prefix = __ballot_sync(0xffffffffu, (w >> 62) == 2ull);
                unsigned long long x = (at_prefix == 0u || lane < __ffs(at_prefix)) ? (w & SCAN_VALUE_MASK) : 0ull;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
                prefix += x;
                if (at_prefix) break;
            }
            if (lane == 0) status[b] = SCAN_FLAG_PREFIX | ((prefix + total) & SCAN_VALUE_MASK);
        }
        if (lane == 0) {
            s_prefix = prefix;
            if (b == gridDim.x - 1) a.total[blockIdx.y] = prefix + total;
        }
    }
    __syncthreads();
    uint32_t run = (uint32_t)s_prefix + excl;
#pragma unroll
    for (int k = 0; k < SCAN_IPT; ++k) {
        const int r = base + k;
        if (r < a.P) a.offsets[r] = run;
        run += v[k];
    }
}

int launch_tile_scan(const BinArgs &a, int V, bool debug, cudaStream_t stream) {
    const int nchunks = (int)ceil_div(a.P, SCAN_CHUNK);
    GSB_CUDA(cudaMemsetAsync(a.scan_state, 0, ((size_t)(V - 1) * a.sv_scan + scan_state_count(a.P)) * sizeof(unsigned long long), stream));
    GSB_LAUNCH("tile_scan", debug, stream, tile_scan_kernel, dim3(nchunks, V), SCAN_THREADS, 0, a);
    return GSB_OK;
}

__global__ void count_max_kernel(unsigned long long *counts, const int V) {
    unsigned long long m = counts[GSB_MAX_VIEWS];
    for (int v = 0; v < V; ++v) m = counts[v] > m ? counts[v] : m;
    counts[GSB_MAX_VIEWS] = m;
}

int launch_count_max(unsigned long long *counts, int V, bool debug, cudaStream_t stream) {
    GSB_LAUNCH("count_max", debug, stream, count_max_kernel, 1, 1, 0, counts, V);
    return GSB_OK;
}

// K3: writes (tile id, gaussian id) for every tile the cull ellipse of a gaussian meets, gaussians in depth order.
// Each lane walks the tiles of one gaussian (the rows and spans of cull_rows / cull_span, or the whole rectangle when culling
// is off); the 32 gaussians of a warp are consecutive depth ranks, so their instances form one contiguous slot range, which
// the warp stages in shared memory a window at a time and stores with consecutive lanes on consecutive slots.  The block also
// counts the digits of the tile sort's passes (dg) over the slots it wrote, so that sort_pairs needs no histogram kernel.
constexpr int EMIT_THREADS = 256;
constexpr int EMIT_WINDOW = 256;   // slots per warp and round
static_assert(EMIT_THREADS == GSB_SORT_RADIX, "one histogram bin per thread");

__global__ void __launch_bounds__(EMIT_THREADS)
emit_kernel(BinArgs a, uint32_t *__restrict__ inst_tile, uint32_t *__restrict__ inst_gauss, const uint32_t cap, const SortDigits dg) {
    __shared__ uint32_t s_tile[EMIT_THREADS / 32][EMIT_WINDOW], s_gauss[EMIT_THREADS / 32][EMIT_WINDOW];
    __shared__ uint32_t hist[GSB_SORT_MAX_PASSES][GSB_SORT_RADIX];
    a.order += blockIdx.y * a.sv_gauss; a.tiles += blockIdx.y * a.sv_gauss; a.rect += blockIdx.y * a.sv_gauss;
    a.offsets += blockIdx.y * a.sv_gauss; a.splat += blockIdx.y * a.sv_splat;
    inst_tile += blockIdx.y * a.sv_inst; inst_gauss += blockIdx.y * a.sv_inst;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    for (int p = 0; p < dg.npass; ++p) hist[p][tid] = 0;

    // this lane's gaussian and its slots [start, start + n)
    const int r = blockIdx.x * EMIT_THREADS + tid;
    uint32_t g = 0, n = 0, start = 0;
    if (r < a.P) {
        g = a.order[r];
        n = a.tiles[g];
        if (n) {
            start = a.offsets[r];
            // speculative capacity (abi.cu): never write past it; the host re-runs binning when the count did not fit
            n = start < cap ? min(n, cap - start) : 0u;
        }
    }
    // tile walk: row ty of [ty, ty1), columns [tx, tx1) of that row still to come
    CullGeom cg;
    int ty = 0, ty1 = 0, tx = 0, tx1 = 0;
    bool whole = false;
    if (n) {
        const float4 q0 = a.splat[(size_t)g * SPLAT_F4], q1 = a.splat[(size_t)g * SPLAT_F4 + 1], q2 = a.splat[(size_t)g * SPLAT_F4 + 2];
        const uint2 rc = a.rect[g];
        cg.cx = q0.x; cg.cy = q0.y; cg.A = q0.z; cg.B = q0.w; cg.C = q1.x; cg.lim = q2.z;
        cg.rx0 = (int)(rc.x & 0xffffu); cg.rx1 = (int)(rc.x >> 16);
        cg.ry0 = (int)(rc.y & 0xffffu); cg.ry1 = (int)(rc.y >> 16);
        whole = cg.lim > 1.0e38f;     // culling disabled: the whole rectangle
        if (whole) { ty = cg.ry0; ty1 = cg.ry1; } else cull_rows(cg, ty, ty1);
        ty -= 1;
        tx = tx1 = 0;
    }
    auto advance_row = [&]() {
        while (tx >= tx1 && ++ty < ty1) {
            if (whole) { tx = cg.rx0; tx1 = cg.rx1; } else cull_span(cg, ty, tx, tx1);
        }
    };
    if (n) advance_row();
    __syncthreads();     // histogram zeroed

    const uint32_t active = __ballot_sync(0xffffffffu, n != 0u);
    if (active) {
        const int first = __ffs(active) - 1, last = 31 - __clz(active);
        const uint32_t lo = __shfl_sync(0xffffffffu, start, first), hi = __shfl_sync(0xffffffffu, start + n, last);
        uint32_t k = 0;
        for (uint32_t base = lo; base < hi; base += EMIT_WINDOW) {
            const uint32_t end = min(hi, base + EMIT_WINDOW);
            for (; k < n && start + k < end; ++k) {
                uint32_t t = (uint32_t)a.num_tiles;   // past the last tile: never taken when count and emit agree
                if (ty < ty1) {
                    t = (uint32_t)(ty * a.gx + tx);
                    ++tx;
                    advance_row();
                }
                s_tile[w][start + k - base] = t;
                s_gauss[w][start + k - base] = g;
            }
            __syncwarp();
            for (uint32_t j = lane; j < end - base; j += 32) {
                const uint32_t t = s_tile[w][j];
                inst_tile[base + j] = t;
                inst_gauss[base + j] = s_gauss[w][j];
#pragma unroll
                for (int p = 0; p < GSB_SORT_MAX_PASSES; ++p)
                    if (p < dg.npass) atomicAdd(&hist[p][(t >> dg.shift[p]) & dg.mask[p]], 1u);
            }
            __syncwarp();
        }
    }
    __syncthreads();
    uint32_t *ghist = dg.ghist + blockIdx.y * (GSB_SORT_MAX_PASSES * GSB_SORT_RADIX);
    for (int p = 0; p < dg.npass; ++p) {
        const uint32_t c = hist[p][tid];
        if (c) atomicAdd(&ghist[p * GSB_SORT_RADIX + tid], c);
    }
}

int launch_emit(const BinArgs &a, int V, uint32_t *inst_tile, uint32_t *inst_gauss, int64_t cap, const SortDigits &dg, bool debug,
                cudaStream_t stream) {
    GSB_LAUNCH("emit", debug, stream, emit_kernel, dim3((int)ceil_div(a.P, EMIT_THREADS), V), EMIT_THREADS, 0, a, inst_tile, inst_gauss,
               (uint32_t)cap, dg);
    return GSB_OK;
}

// K5: ranges[t] = [first, last+1) of tile t in the tile-sorted instance list (ranges pre-zeroed)
__global__ void __launch_bounds__(256)
tile_ranges_kernel(const uint32_t *__restrict__ sorted_tiles, int64_t D, const unsigned long long *__restrict__ n_dev,
                   const int num_tiles, uint2 *ranges, const size_t sv_inst) {
    sorted_tiles += blockIdx.y * sv_inst; ranges += (size_t)blockIdx.y * num_tiles;
    if (n_dev) D = min((int64_t)n_dev[blockIdx.y], D);
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= D) return;
    const uint32_t t = sorted_tiles[i];
    if (t >= (uint32_t)num_tiles) return;
    if (i == 0 || sorted_tiles[i - 1] != t) ranges[t].x = (uint32_t)i;
    if (i == D - 1 || sorted_tiles[i + 1] != t) ranges[t].y = (uint32_t)(i + 1);
}

int launch_tile_ranges(const uint32_t *sorted_tiles, int64_t D, const unsigned long long *n_dev, int num_tiles,
                       uint2 *ranges, int V, size_t sv_inst, bool debug, cudaStream_t stream) {
    GSB_CUDA(cudaMemsetAsync(ranges, 0, (size_t)V * num_tiles * sizeof(uint2), stream));
    if (D <= 0) return GSB_OK;
    GSB_LAUNCH("tile_ranges", debug, stream, tile_ranges_kernel, dim3((int)ceil_div(D, 256), V), 256, 0, sorted_tiles, D, n_dev,
               num_tiles, ranges, sv_inst);
    return GSB_OK;
}

}  // namespace gsb
