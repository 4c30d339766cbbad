// common.cuh -- shared definitions for the sm_90a rasterizer kernels.
#pragma once
#ifdef GSB_HOST_EMUL        // tests/host_emul: these sources compiled for the CPU by the test-suite (never a product build)
#include "cuda_shim.h"
#else
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <stdio.h>

#include "../../include/gs_b200.h"

namespace gsb {

// ---- splatting constants (same set as oracle/torch_oracle.py UNVERIFIED_VS_REFERENCE) ----
constexpr int TILE = 16;
constexpr int TILE_PIX = TILE * TILE;
constexpr float NEAR_CULL = 0.2f;
constexpr float FRUSTUM_CLAMP = 1.3f;
constexpr float DILATION = 0.3f;
constexpr float AA_FLOOR = 0.000025f;
constexpr float ALPHA_MIN = 1.0f / 255.0f;
constexpr float ALPHA_MAX = 0.99f;
constexpr float T_STOP = 0.0001f;
constexpr float W_EPS = 0.0000001f;

// SH constants: /root/reference/utils/sh_utils.py:26-54
constexpr float SH_C0 = 0.28209479177387814f;
constexpr float SH_C1 = 0.4886025119029199f;
__device__ constexpr float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                       -1.0925484305920792f, 0.5462742152960396f};
__device__ constexpr float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                       0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                       -0.5900435899266435f};

// ---- per-gaussian forward record gathered by the blend kernels: 3 x float4 = 48 B ----
//   q0 = { x, y, conic.A, conic.B }      pixel-space mean, inverse dilated 2D covariance
//   q1 = { conic.C, opacity, r, g }      opacity already multiplied by the AA factor
//   q2 = { b, 1/depth, depth, bits }     bits: low 3 = SH clamp flags
constexpr int SPLAT_F4 = 3;

// ---- single-instruction approximate math (MUFU), for CULLING GEOMETRY ONLY ------------------------------------
// The culling tests are conservative by construction (padded limits and spans), so <= 2 ulp approximations are
// fine there, and as inline PTX they are evaluated identically wherever they appear (the counting and the emitting
// pass must agree bit for bit).  Projection / covariance / blending arithmetic never uses these.
#ifdef GSB_HOST_EMUL
inline float sqrt_apx(const float x) { return sqrtf(x); }
inline float div_apx(const float a, const float b) { return a / b; }
inline float rcp_apx(const float x) { return 1.0f / x; }
#else
__device__ __forceinline__ float sqrt_apx(const float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float div_apx(const float a, const float b) { float y; asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(y) : "f"(a), "f"(b)); return y; }
__device__ __forceinline__ float rcp_apx(const float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
#endif

// ---- TMA bulk copies (cp.async.bulk: SASS UBLKCP / UBLKRED) and the mbarrier they complete on ------------------------------
// 1-D bulk copies need no tensor map: 16-byte aligned source / destination, size a multiple of 16.  Used by the per-gaussian
// kernels to move SH rows (192 B each) between global and shared memory without a single LDG / STG / index instruction.
#ifdef GSB_HOST_EMUL     // tests/host_emul: synchronous copies; the barrier degenerates to nothing (each thread waits for its own row)
inline void mbar_init(unsigned long long *, int) {}
inline void mbar_expect_tx(unsigned long long *, uint32_t) {}
inline void mbar_wait(unsigned long long *, uint32_t) {}
inline void bulk_g2s(void *smem_dst, const void *gsrc, uint32_t bytes, unsigned long long *) { memcpy(smem_dst, gsrc, bytes); }
inline void bulk_s2g(void *gdst, const void *smem_src, uint32_t bytes) { memcpy(gdst, smem_src, bytes); }
inline void bulk_s2g_add_f32(float *gdst, const float *smem_src, uint32_t bytes) { for (uint32_t k = 0; k < bytes / 4; ++k) gdst[k] += smem_src[k]; }
inline void bulk_store_fence() {}
inline void bulk_store_commit_and_wait() {}
#else
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, const int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, const uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, const uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "LAB_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra LAB_DONE;\n\t"
        "bra LAB_WAIT;\n\t"
        "LAB_DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, const uint32_t bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void *gdst, const void *smem_src, const uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_s2g_add_f32(float *gdst, const float *smem_src, const uint32_t bytes) {
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
// generic-proxy writes to shared memory -> visible to the async proxy (before a bulk store reads them)
__device__ __forceinline__ void bulk_store_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// the issuing thread's bulk stores have finished READING shared memory (required before the CTA exits or reuses it)
__device__ __forceinline__ void bulk_store_commit_and_wait() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
#endif

// ---- host-side plumbing -------------------------------------------------------------------
void set_error(const char *fmt, ...);
extern int64_t g_launch_count;
int check_launch(const char *what, bool debug, cudaStream_t stream);

// per-kernel CUDA-event timing on the launching stream (option "time_kernels": 1 = blend kernels only,
// 2 = every kernel); read back with gsb_kernel_time()
extern int g_time_kernels;
void *timer_begin(const char *name, cudaStream_t stream);
void timer_end(void *token, cudaStream_t stream);

// the launch itself; dynamic shared memory is declared through GSB_DYNAMIC_SMEM so that both spellings stay in one place
#ifdef GSB_HOST_EMUL
#define GSB_KERNEL_LAUNCH(kernel, grid, block, smem, stream, ...) \
    gsb_emul_launch(dim3(grid), dim3(block), (size_t)(smem), [&] { kernel(__VA_ARGS__); })
#define GSB_DYNAMIC_SMEM(type, name) type *name = reinterpret_cast<type *>(gsb_emul_dynamic_smem())
#else
#define GSB_KERNEL_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define GSB_DYNAMIC_SMEM(type, name) extern __shared__ type name[]
#endif

#define GSB_LAUNCH(name, debug, stream, kernel, grid, block, smem, ...)                         \
    do {                                                                                        \
        void *_tok = gsb::g_time_kernels ? gsb::timer_begin(name, (stream)) : nullptr;          \
        GSB_KERNEL_LAUNCH(kernel, grid, block, smem, stream, __VA_ARGS__);                      \
        if (_tok) gsb::timer_end(_tok, (stream));                                               \
        ++gsb::g_launch_count;                                                                  \
        int _e = gsb::check_launch(name, (debug), (stream));                                    \
        if (_e) return _e;                                                                      \
    } while (0)

#define GSB_CUDA(expr)                                                                          \
    do {                                                                                        \
        cudaError_t _err = (expr);                                                              \
        if (_err != cudaSuccess) {                                                              \
            gsb::set_error("%s failed: %s", #expr, cudaGetErrorString(_err));                   \
            return GSB_ERR_CUDA;                                                                \
        }                                                                                       \
    } while (0)

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// SMs of the target GPU (H100 SXM), for the grid-stride kernels whose grid is sized to fill the device once
constexpr int NUM_SMS = 132;

// bump carver over one allocation
struct Carver {
    char *base;
    size_t off;
    explicit Carver(void *p) : base(static_cast<char *>(p)), off(0) {}
    template <typename T>
    T *take(size_t count) {
        off = align_up(off, 256);
        T *p = base ? reinterpret_cast<T *>(base + off) : nullptr;
        off += count * sizeof(T);
        return p;
    }
    size_t bytes() const { return align_up(off, 256); }
};

// ---- radix sort / scan (radix_sort.cu) ----------------------------------------------------
size_t sort_scratch_bytes(int64_t n, int V = 1);
// Stable LSD sort of pairs on bits [begin_bit, end_bit).  Result is left in (keys, vals);
// (keys_alt, vals_alt) are ping-pong buffers of the same size; scratch >= sort_scratch_bytes(n).
// n sizes the launch; if n_dev != NULL the kernels sort min(*n_dev, n) pairs (count known only on the device).
// V > 1 (view batch): V independent sorts in the same launches; view v's arrays start at base + v * sv elements and
// n_dev is an array of V counts.
// hist_ready: the scratch was zeroed and its digit histograms filled by the caller (sort_prepare), so the sort skips both.
int sort_pairs(uint32_t *keys, uint32_t *vals, uint32_t *keys_alt, uint32_t *vals_alt, int64_t n,
               const unsigned long long *n_dev, int begin_bit, int end_bit, void *scratch, bool debug,
               cudaStream_t stream, int V = 1, size_t sv = 0, bool hist_ready = false);
constexpr int GSB_SORT_MAX_VIEWS = 16, GSB_SORT_MAX_PASSES = 4, GSB_SORT_RADIX = 256;
// The digits of a sort_pairs call: pass p sorts on (key >> shift[p]) & mask[p].  ghist[view][pass][digit] are the counts of
// the keys that will be sorted, which a kernel that produces the keys can build (binning.cu emit) instead of sort_pairs.
struct SortDigits {
    int npass;
    int shift[GSB_SORT_MAX_PASSES];
    uint32_t mask[GSB_SORT_MAX_PASSES];
    uint32_t *ghist;   // [GSB_SORT_MAX_VIEWS][GSB_SORT_MAX_PASSES][GSB_SORT_RADIX]
};
// Zeroes the scratch of a later sort_pairs(..., hist_ready = true) call with the same n, V and bits, and describes its digits.
int sort_prepare(int64_t n, int V, int begin_bit, int end_bit, void *scratch, cudaStream_t stream, SortDigits *out);
extern int g_sort_force_small;
extern int g_pre_tma;

}  // namespace gsb
