// radix_sort.cu -- stable LSD radix sort of (u32 key, u32 value) pairs, 8 bits per pass.
//
// Replaces the reference's cub::DeviceRadixSort::SortPairs call (named in BASELINE.json
// north_star; the call site lives in the absent cuda_rasterizer/rasterizer_impl.cu).
//
// The reference sorts D 64-bit keys (tile << 32 | depth) in one 6-pass sort.  Here the same
// order is produced by two much smaller sorts (DESIGN.md "binning"):
//   1. gaussians by depth bits      (P pairs, 4 passes)
//   2. instances by tile id, STABLE (D pairs, ceil(log2(tiles)/8) = 2 passes)
// because instances are emitted in depth order and a stable sort keeps that order per tile.
//
// One upfront kernel builds the digit histograms of every pass; each pass is then ONE kernel ("onesweep", below):
// keys and values are read once and written once per pass (16 B / pair).  The round-1 three-kernel-per-pass version
// (histogram / row scan / scatter) and an 8-keys-per-thread block size are gone from the build; git has them.
#include "common.cuh"

namespace gsb {

constexpr int RADIX_BITS = 8;
constexpr int RADIX = 1 << RADIX_BITS;
constexpr int SORT_THREADS = 256;
// keys per thread: 16 for large inputs; 4 below ~2.4 M keys so that even the 1 M-gaussian depth sort fills
// the SMs with several blocks each (the first version ran 245 blocks of 4096 keys: latency bound)
constexpr int SORT_IPT_BIG = 16;
constexpr int SORT_IPT_SMALL = 4;
constexpr int64_t SORT_SMALL_LIMIT = NUM_SMS * 4 * 1024;   // below ~0.5 M keys: 1024-key blocks to fill the SMs
int g_sort_force_small = 0;   // option "sort_small": 1 = 4 keys per thread for every size, -1 = never (A/B, tests)
static inline int sort_ipt(int64_t n) {
    if (g_sort_force_small < 0) return SORT_IPT_BIG;
    return (g_sort_force_small || n < SORT_SMALL_LIMIT) ? SORT_IPT_SMALL : SORT_IPT_BIG;
}
// runs CALL with the compile-time constant I = keys per thread
#define SORT_WITH_IPT(ipt, CALL)                                       \
    switch (ipt) {                                                     \
        case SORT_IPT_SMALL: { constexpr int I = SORT_IPT_SMALL; CALL; } break; \
        default: { constexpr int I = SORT_IPT_BIG; CALL; } break;      \
    }

// ------------------------------------------------------------------------------------------------
// Single-pass-per-digit variant ("onesweep"): one upfront kernel builds the global digit histograms of
// every pass, then each pass is ONE kernel whose blocks obtain their per-digit offsets by decoupled
// look-back over a status word per (block, digit) -- no per-pass histogram / row-scan kernels, keys and
// values are read once and written once per pass (16 B / pair).
//   status word: bits 31..30 = 0 not ready | 1 block aggregate | 2 inclusive prefix; bits 29..0 = count.
// Blocks take a ticket from an atomic counter, so a block only ever waits for blocks that started before
// it: forward progress does not depend on the hardware's block scheduling order.
// ------------------------------------------------------------------------------------------------
#define OS_FLAG_AGG (1u << 30)
#define OS_FLAG_PREFIX (2u << 30)
#define OS_VALUE_MASK ((1u << 30) - 1u)
constexpr int OS_MAX_PASSES = GSB_SORT_MAX_PASSES;
static_assert(RADIX == GSB_SORT_RADIX, "histogram layout shared with binning.cu");

struct OnesweepPasses {
    int npass;
    int shift[OS_MAX_PASSES];
    uint32_t mask[OS_MAX_PASSES];
};

__global__ void __launch_bounds__(256)
onesweep_hist_kernel(const uint32_t *__restrict__ keys, uint32_t *__restrict__ ghist, int64_t n,
                     const unsigned long long *__restrict__ n_dev, const OnesweepPasses ps, const size_t sv) {
    __shared__ uint32_t hist[OS_MAX_PASSES][RADIX];
    keys += blockIdx.y * sv; ghist += blockIdx.y * (OS_MAX_PASSES * RADIX);   // view-batch: blockIdx.y = view
    if (n_dev) n = min((int64_t)n_dev[blockIdx.y], n);
    for (int p = 0; p < ps.npass; ++p) hist[p][threadIdx.x] = 0;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
        const uint32_t k = keys[i];
        for (int p = 0; p < ps.npass; ++p) atomicAdd(&hist[p][(k >> ps.shift[p]) & ps.mask[p]], 1u);
    }
    __syncthreads();
    for (int p = 0; p < ps.npass; ++p) {
        const uint32_t c = hist[p][threadIdx.x];
        if (c) atomicAdd(&ghist[p * RADIX + threadIdx.x], c);
    }
}

// compile-time knobs of the ranking loop (A/B builds through GSB_LIBRARY; tools/sort_ab.py times the variants)
#ifndef GSB_OS_GROUP
#define GSB_OS_GROUP 8      // MATCH.ANY instructions issued back to back before their counter chains
#endif
#ifndef GSB_OS_MINB
#define GSB_OS_MINB 3       // resident CTAs per SM the register allocation must allow
#endif
#ifndef GSB_OS_BALLOT
#define GSB_OS_BALLOT 1     // 1: peers from nine ballots instead of MATCH.ANY
#endif

__device__ __forceinline__ uint32_t digit_peers(const uint32_t d) {
#if GSB_OS_BALLOT
    uint32_t peers = 0xffffffffu;
#pragma unroll
    for (int bit = 0; bit <= RADIX_BITS; ++bit) {          // bit RADIX_BITS separates the out-of-range lanes (d == RADIX)
        const bool one = (d >> bit) & 1u;
        const uint32_t b = __ballot_sync(0xffffffffu, one);
        peers &= one ? b : ~b;
    }
    return peers;
#else
    return __match_any_sync(0xffffffffu, d);
#endif
}

template <int SORT_IPT>
__global__ void __launch_bounds__(SORT_THREADS, SORT_IPT >= 16 ? GSB_OS_MINB : 4)
onesweep_pass_kernel(const uint32_t *__restrict__ keys_in, const uint32_t *__restrict__ vals_in,
                     uint32_t *__restrict__ keys_out, uint32_t *__restrict__ vals_out,
                     const uint32_t *__restrict__ ghist, volatile uint32_t *status, uint32_t *ticket, int64_t n,
                     const unsigned long long *__restrict__ n_dev, int shift, uint32_t mask, const size_t sv,
                     const size_t sv_status) {
    constexpr int SORT_KPB = SORT_THREADS * SORT_IPT;
    {   // view-batch: blockIdx.y = view
        const size_t v = blockIdx.y;
        keys_in += v * sv; vals_in += v * sv; keys_out += v * sv; vals_out += v * sv;
        ghist += v * (OS_MAX_PASSES * RADIX); status += v * sv_status; ticket += v * OS_MAX_PASSES;
    }
    __shared__ uint32_t warp_cnt[SORT_THREADS / 32][RADIX];
    __shared__ uint32_t warp_sums[8];
    __shared__ uint32_t s_ticket;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (n_dev) n = min((int64_t)n_dev[blockIdx.y], n);
    if (tid == 0) s_ticket = atomicAdd(ticket, 1u);
#pragma unroll
    for (int k = 0; k < SORT_THREADS / 32; ++k) warp_cnt[k][tid] = 0;
    __syncthreads();
    const uint32_t b = s_ticket;
    if ((int64_t)b * SORT_KPB >= n) return;

    // global base of digit `tid`: exclusive scan of the 256 digit totals of this pass
    const uint32_t tot = ghist[tid];
    uint32_t incl = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[w] = incl;
    __syncthreads();
    uint32_t digit_base = incl - tot;
#pragma unroll
    for (int k = 0; k < 8; ++k)
        if (k < w) digit_base += warp_sums[k];

    // stable local ranks, block order = (warp, round, lane)
    const int64_t seg = (int64_t)b * SORT_KPB + (int64_t)w * (32 * SORT_IPT);
    uint32_t key[SORT_IPT], rank[SORT_IPT];
    const uint32_t lt_mask = (1u << lane) - 1u;
    // The rounds are chained through the warp's digit counters, but the MATCH.ANY that finds a round's peers is not: issue
    // a group of them back to back (ncu: 31 % of this kernel's stall samples sat on the first consumer of MATCH.ANY when
    // every round waited for its own match) and only then walk the counter chain.
    constexpr int GROUP = SORT_IPT < GSB_OS_GROUP ? SORT_IPT : GSB_OS_GROUP;
#pragma unroll
    for (int g0 = 0; g0 < SORT_IPT; g0 += GROUP) {
        uint32_t peers[GROUP];
#pragma unroll
        for (int j = 0; j < GROUP; ++j) {
            const int r = g0 + j;
            const int64_t idx = seg + r * 32 + lane;
            const bool valid = idx < n;
            key[r] = valid ? keys_in[idx] : 0xffffffffu;
            const uint32_t d = valid ? ((key[r] >> shift) & mask) : (uint32_t)RADIX;
            peers[j] = digit_peers(d);
        }
#pragma unroll
        for (int j = 0; j < GROUP; ++j) {
            const int r = g0 + j;
            const bool valid = seg + r * 32 + lane < n;
            const uint32_t d = (key[r] >> shift) & mask;
            const int leader = __ffs(peers[j]) - 1;
            uint32_t base = 0;
            if (lane == leader && valid) {
                base = warp_cnt[w][d];
                warp_cnt[w][d] = base + __popc(peers[j]);
            }
            base = __shfl_sync(0xffffffffu, base, leader);
            rank[r] = base + __popc(peers[j] & lt_mask);
            __syncwarp();
        }
    }
    __syncthreads();

    // per-digit block count; warp_cnt becomes the exclusive prefix over warps (position inside the block's digit run)
    uint32_t cnt = 0;
#pragma unroll
    for (int k = 0; k < SORT_THREADS / 32; ++k) {
        const uint32_t c = warp_cnt[k][tid];
        warp_cnt[k][tid] = cnt;
        cnt += c;
    }
    // decoupled look-back for digit `tid`
    volatile uint32_t *my = status + (size_t)b * RADIX + tid;
    uint32_t excl = 0;
    if (b == 0) {
        *my = cnt | OS_FLAG_PREFIX;
    } else {
        *my = cnt | OS_FLAG_AGG;
        // Walk back over the predecessors' status words, eight loads in flight at a time: with ~300 blocks resident
        // most predecessors only show an aggregate, so the walk is long and must not be one L2 round trip per step.
        int64_t pb = (int64_t)b - 1;
        bool found = false;
        while (!found) {
            uint32_t v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int64_t q = pb - u;
                v[u] = q >= 0 ? status[(size_t)q * RADIX + tid] : OS_FLAG_PREFIX;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                if (!found) {
                    while ((v[u] >> 30) == 0u) v[u] = status[(size_t)(pb - u) * RADIX + tid];
                    excl += v[u] & OS_VALUE_MASK;
                    found = (v[u] >> 30) == 2u;
                }
            }
            pb -= 8;
        }
        *my = ((excl + cnt) & OS_VALUE_MASK) | OS_FLAG_PREFIX;
    }

    // Local reorder: the block's pairs are first put in digit order in shared memory, then written out so that
    // consecutive threads write consecutive addresses inside each digit's run.  A direct scatter writes one 4-byte
    // element per 32-byte sector (12.5 % sector efficiency); runs of KPB/256 keys fill whole sectors.
    __shared__ uint32_t sk[SORT_KPB], svals[SORT_KPB];
    __shared__ uint32_t loff[RADIX], gpos[RADIX];
    {   // exclusive scan of cnt over the 256 digits -> local start of each digit's run
        uint32_t inc = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t2 = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t2;
        }
        __syncthreads();                 // warp_sums is reused: everyone has finished reading it for digit_base
        if (lane == 31) warp_sums[w] = inc;
        __syncthreads();
        uint32_t lo = inc - cnt;
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (k < w) lo += warp_sums[k];
        loff[tid] = lo;
        gpos[tid] = digit_base + excl;
    }
    __syncthreads();
    const int64_t block_start = (int64_t)b * SORT_KPB;
    const int block_n = (int)min((int64_t)SORT_KPB, n - block_start);
#pragma unroll
    for (int r = 0; r < SORT_IPT; ++r) {
        const int64_t idx = seg + r * 32 + lane;
        if (idx < n) {
            const uint32_t d = (key[r] >> shift) & mask;
            const uint32_t lp = loff[d] + warp_cnt[w][d] + rank[r];
            sk[lp] = key[r];
            svals[lp] = vals_in[idx];
        }
    }
    __syncthreads();
    for (int i = tid; i < block_n; i += SORT_THREADS) {
        const uint32_t k2 = sk[i];
        const uint32_t d = (k2 >> shift) & mask;
        const uint32_t pos = gpos[d] + ((uint32_t)i - loff[d]);
        keys_out[pos] = k2;
        vals_out[pos] = svals[i];
    }
}

static size_t onesweep_scratch_bytes(int64_t n, int V) {
    const int64_t nblocks = ceil_div(n > 0 ? n : 1, SORT_THREADS * sort_ipt(n));
    return align_up((size_t)GSB_SORT_MAX_VIEWS * OS_MAX_PASSES * RADIX * 4 + 256 + (size_t)V * OS_MAX_PASSES * nblocks * RADIX * 4, 256);
}

// the key bits are split EVENLY over the fewest passes (13 tile bits = 7 + 6, not 8 + 5): a pass with fewer digits writes
// longer runs per digit out of every block
static int onesweep_passes(int begin_bit, int end_bit, OnesweepPasses &ps) {
    ps.npass = 0;
    const int total_bits = end_bit - begin_bit, npass = (total_bits + RADIX_BITS - 1) / RADIX_BITS;
    if (npass > OS_MAX_PASSES) { set_error("onesweep: more than %d passes", OS_MAX_PASSES); return GSB_ERR_ARGUMENT; }
    for (int p = 0, bit = begin_bit; p < npass; ++p) {
        const int bits = total_bits / npass + (p < total_bits % npass ? 1 : 0);
        ps.shift[p] = bit;
        ps.mask[p] = (1u << bits) - 1u;
        bit += bits;
        ++ps.npass;
    }
    return GSB_OK;
}

// scratch layout: ghist[16 views][4][256] | ticket[16][4] (256 B) | status[V][npass][nblocks][256]
static size_t onesweep_zero_bytes(int64_t n, int V, int npass) {
    const int64_t nblocks = ceil_div(n, SORT_THREADS * sort_ipt(n));
    return (size_t)GSB_SORT_MAX_VIEWS * OS_MAX_PASSES * RADIX * 4 + 256 + (size_t)V * npass * nblocks * RADIX * 4;
}

static int onesweep_sort(uint32_t *keys, uint32_t *vals, uint32_t *keys_alt, uint32_t *vals_alt, int64_t n,
                         const unsigned long long *n_dev, int begin_bit, int end_bit, void *scratch, bool debug,
                         cudaStream_t stream, int V, size_t sv, bool hist_ready) {
    OnesweepPasses ps;
    int rc = onesweep_passes(begin_bit, end_bit, ps);
    if (rc) return rc;
    const int ipt = sort_ipt(n);
    const int nblocks = (int)ceil_div(n, SORT_THREADS * ipt);
    uint32_t *ghist = static_cast<uint32_t *>(scratch);
    uint32_t *ticket = ghist + GSB_SORT_MAX_VIEWS * OS_MAX_PASSES * RADIX;
    uint32_t *status = ticket + 64;
    const size_t sv_status = (size_t)ps.npass * nblocks * RADIX;
    if (!hist_ready) {
        GSB_CUDA(cudaMemsetAsync(scratch, 0, onesweep_zero_bytes(n, V, ps.npass), stream));
        const int hist_blocks = (int)(ceil_div(n, 256 * 16) < NUM_SMS * 8 ? ceil_div(n, 256 * 16) : NUM_SMS * 8);
        GSB_LAUNCH("sort_hist", debug, stream, onesweep_hist_kernel, dim3(hist_blocks, V), 256, 0, keys, ghist, n, n_dev, ps, sv);
    }
    uint32_t *kin = keys, *vin = vals, *kout = keys_alt, *vout = vals_alt;
    for (int p = 0; p < ps.npass; ++p) {
        uint32_t *st = status + (size_t)p * nblocks * RADIX;
        SORT_WITH_IPT(ipt, GSB_LAUNCH("sort_scatter", debug, stream, onesweep_pass_kernel<I>, dim3(nblocks, V), SORT_THREADS, 0, kin, vin,
                                 kout, vout, ghist + p * RADIX, st, ticket + p, n, n_dev, ps.shift[p], ps.mask[p], sv, sv_status));
        uint32_t *t = kin; kin = kout; kout = t;
        t = vin; vin = vout; vout = t;
    }
    if (ps.npass & 1) {
        const size_t bytes = V > 1 ? ((size_t)(V - 1) * sv + (size_t)n) * 4 : (size_t)n * 4;
        GSB_CUDA(cudaMemcpyAsync(keys, keys_alt, bytes, cudaMemcpyDeviceToDevice, stream));
        GSB_CUDA(cudaMemcpyAsync(vals, vals_alt, bytes, cudaMemcpyDeviceToDevice, stream));
    }
    return GSB_OK;
}

size_t sort_scratch_bytes(int64_t n, int V) { return onesweep_scratch_bytes(n, V); }

int sort_prepare(int64_t n, int V, int begin_bit, int end_bit, void *scratch, cudaStream_t stream, SortDigits *out) {
    OnesweepPasses ps;
    int rc = onesweep_passes(begin_bit, end_bit, ps);
    if (rc) return rc;
    out->npass = ps.npass;
    for (int p = 0; p < OS_MAX_PASSES; ++p) {
        out->shift[p] = p < ps.npass ? ps.shift[p] : 0;
        out->mask[p] = p < ps.npass ? ps.mask[p] : 0u;
    }
    out->ghist = static_cast<uint32_t *>(scratch);
    if (n > 0) GSB_CUDA(cudaMemsetAsync(scratch, 0, onesweep_zero_bytes(n, V, ps.npass), stream));
    return GSB_OK;
}

int sort_pairs(uint32_t *keys, uint32_t *vals, uint32_t *keys_alt, uint32_t *vals_alt, int64_t n,
               const unsigned long long *n_dev, int begin_bit, int end_bit, void *scratch, bool debug,
               cudaStream_t stream, int V, size_t sv, bool hist_ready) {
    if (n <= 0 || end_bit <= begin_bit) return GSB_OK;
    if (n >= (int64_t)1 << 30) {
        set_error("sort_pairs: n=%lld does not fit 30-bit positions", (long long)n);
        return GSB_ERR_OVERFLOW;
    }
    if (V > GSB_SORT_MAX_VIEWS) { set_error("sort_pairs: more than %d views", GSB_SORT_MAX_VIEWS); return GSB_ERR_ARGUMENT; }
    return onesweep_sort(keys, vals, keys_alt, vals_alt, n, n_dev, begin_bit, end_bit, scratch, debug, stream, V, sv, hist_ready);
}

}  // namespace gsb
