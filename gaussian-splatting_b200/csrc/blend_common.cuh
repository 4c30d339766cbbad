// blend_common.cuh -- helpers of the blend kernels (render.cu): staged-record scaling, the pinned exponent, packed f32x2 arithmetic,
// the transposed warp reductions of the backward pass.
#pragma once
#include "kernels.cuh"
#include "patch_cull.cuh"

namespace gsb {

constexpr int MP_R = 128;           // gaussians staged per round
constexpr float LOG2E = 1.4426950408889634f;

#ifdef GSB_HOST_EMUL     // tests/host_emul: the approximate instructions become their libm counterparts
inline float ex2_approx(const float x) { return exp2f(x); }
inline float rcp_approx(const float x) { return 1.0f / x; }
#else
__device__ __forceinline__ float ex2_approx(const float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// 1/x, one MUFU.RCP (<= 1 ulp); x = 1 - alpha is in [0.01, 1], no special cases to handle
__device__ __forceinline__ float rcp_approx(const float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
#endif

// staged record: q0 = {x, y, A', C'}, q1 = {B', opacity, r, g} with A' = -0.5 log2e A, B' = -log2e B, C' = -0.5 log2e C.
// (x, y) and (A', C') are 64-bit register pairs after the 128-bit shared-memory load, i.e. ready-made f32x2 operands:
// (dx, dy) = (x, y) - pixel is ONE packed add and (A' dx dx, C' dy dy) two packed multiplies.
__device__ __forceinline__ void stage_scale(float4 &q0, float4 &q1) {
    const float a = __fmul_rn(q0.z, -0.5f * LOG2E), b = __fmul_rn(q0.w, -LOG2E), c = __fmul_rn(q1.x, -0.5f * LOG2E);
    q0.z = a; q0.w = c; q1.x = b;
}

// log2-domain exponent at offset (dx, dy); pinned operation order: forward and backward must agree bit for bit
__device__ __forceinline__ float power2_at(const float Axx, const float Cyy, const float Bx, const float dy) {
    return __fmaf_rn(Bx, dy, __fadd_rn(Axx, Cyy));
}

// lane L ends with the warp total of value (L >> 2): 9 shuffles
__device__ __forceinline__ float reduce8_transposed(const float v0, const float v1, const float v2, const float v3,
                                                    const float v4, const float v5, const float v6, const float v7) {
    const int lane = threadIdx.x & 31;
    const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
    const float k0 = (b4 ? v4 : v0) + __shfl_xor_sync(0xffffffffu, b4 ? v0 : v4, 16);
    const float k1 = (b4 ? v5 : v1) + __shfl_xor_sync(0xffffffffu, b4 ? v1 : v5, 16);
    const float k2 = (b4 ? v6 : v2) + __shfl_xor_sync(0xffffffffu, b4 ? v2 : v6, 16);
    const float k3 = (b4 ? v7 : v3) + __shfl_xor_sync(0xffffffffu, b4 ? v3 : v7, 16);
    const float m0 = (b3 ? k2 : k0) + __shfl_xor_sync(0xffffffffu, b3 ? k0 : k2, 8);
    const float m1 = (b3 ? k3 : k1) + __shfl_xor_sync(0xffffffffu, b3 ? k1 : k3, 8);
    float r = (b2 ? m1 : m0) + __shfl_xor_sync(0xffffffffu, b2 ? m0 : m1, 4);
    r += __shfl_xor_sync(0xffffffffu, r, 2);
    r += __shfl_xor_sync(0xffffffffu, r, 1);
    return r;
}

// lanes 0..15 end with the total of v0, lanes 16..31 with the total of v1: 5 shuffles
__device__ __forceinline__ float reduce2_transposed(const float v0, const float v1) {
    const bool b4 = threadIdx.x & 16;
    float r = (b4 ? v1 : v0) + __shfl_xor_sync(0xffffffffu, b4 ? v0 : v1, 16);
    r += __shfl_xor_sync(0xffffffffu, r, 8);
    r += __shfl_xor_sync(0xffffffffu, r, 4);
    r += __shfl_xor_sync(0xffffffffu, r, 2);
    r += __shfl_xor_sync(0xffffffffu, r, 1);
    return r;
}

// Lane roles of reduce10_transposed: bits 4, 3, 2 and 1 of the lane id, from lane_mask = 1 << lane.  Each role is then ONE
// test of one register against a constant (a kernel keeps lane_mask opaque in a register, so a loop does not rebuild it
// from the lane id; there are not enough predicate registers to keep all four roles resident).
struct LaneBits {
    bool b4, b3, b2, b1;
};
__device__ __forceinline__ LaneBits lane_bits(const uint32_t lane_mask) {
    return LaneBits{(lane_mask & 0xffff0000u) != 0u, (lane_mask & 0xff00ff00u) != 0u, (lane_mask & 0xf0f0f0f0u) != 0u,
                    (lane_mask & 0xccccccccu) != 0u};
}

// Warp totals of ten per-lane sums v[0..9] (nine with TEN = false: v[9] is not read) in 12 shuffles (5 + 3 + 2 + 1 + 1).
// Lane L ends with the total of sum  (L & 2) ? 4 + 5 b4 : 2 b2 + b3 + 5 b4  (bK = bit K of L), so lanes
// 0, 8, 4, 12, 2, 16, 24, 20, 28, 18 hold sums 0..9.  Without v[9], the lanes that would hold it hold sum 4 as well.
template <bool TEN>
__device__ __forceinline__ float reduce10_transposed(const float (&v)[10], const LaneBits &L) {
    float k[5];
#pragma unroll
    for (int i = 0; i < 4; ++i) k[i] = (L.b4 ? v[i + 5] : v[i]) + __shfl_xor_sync(0xffffffffu, L.b4 ? v[i] : v[i + 5], 16);
    if (TEN) k[4] = (L.b4 ? v[9] : v[4]) + __shfl_xor_sync(0xffffffffu, L.b4 ? v[4] : v[9], 16);
    else     k[4] = v[4] + __shfl_xor_sync(0xffffffffu, v[4], 16);
    const float m0 = (L.b3 ? k[1] : k[0]) + __shfl_xor_sync(0xffffffffu, L.b3 ? k[0] : k[1], 8);
    const float m1 = (L.b3 ? k[3] : k[2]) + __shfl_xor_sync(0xffffffffu, L.b3 ? k[2] : k[3], 8);
    const float m2 = k[4] + __shfl_xor_sync(0xffffffffu, k[4], 8);
    const float n0 = (L.b2 ? m1 : m0) + __shfl_xor_sync(0xffffffffu, L.b2 ? m0 : m1, 4);
    const float n1 = m2 + __shfl_xor_sync(0xffffffffu, m2, 4);
    float r = (L.b1 ? n1 : n0) + __shfl_xor_sync(0xffffffffu, L.b1 ? n0 : n1, 2);
    r += __shfl_xor_sync(0xffffffffu, r, 1);
    return r;
}

// ---- FP32 pairs: two pixels (or two coordinates) carried as one 64-bit register pair ----
// sm_90 has no packed FP32 instruction, so every pair operation is two scalar round-to-nearest instructions (the _rn
// intrinsics also keep the compiler from contracting a multiply and an add into an FMA, which would change the bits
// the forward and backward kernels must agree on).  The pair type stays: the staged record is read with 128-bit
// shared-memory loads that deliver exactly these register pairs, and the pack / unpack moves cost no instruction.
typedef unsigned long long f32x2;
#ifdef GSB_HOST_EMUL
inline f32x2 pk(const float lo, const float hi) { f32x2 r; float t[2] = {lo, hi}; memcpy(&r, t, 8); return r; }
inline void unpk(const f32x2 v, float &lo, float &hi) { float t[2]; memcpy(t, &v, 8); lo = t[0]; hi = t[1]; }
#else
__device__ __forceinline__ f32x2 pk(const float lo, const float hi) { f32x2 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void unpk(const f32x2 v, float &lo, float &hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
#endif
__device__ __forceinline__ f32x2 fma2(const f32x2 a, const f32x2 b, const f32x2 c) {
    float al, ah, bl, bh, cl, ch;
    unpk(a, al, ah); unpk(b, bl, bh); unpk(c, cl, ch);
    return pk(__fmaf_rn(al, bl, cl), __fmaf_rn(ah, bh, ch));
}
__device__ __forceinline__ f32x2 mul2(const f32x2 a, const f32x2 b) {
    float al, ah, bl, bh;
    unpk(a, al, ah); unpk(b, bl, bh);
    return pk(__fmul_rn(al, bl), __fmul_rn(ah, bh));
}
__device__ __forceinline__ f32x2 add2(const f32x2 a, const f32x2 b) {
    float al, ah, bl, bh;
    unpk(a, al, ah); unpk(b, bl, bh);
    return pk(__fadd_rn(al, bl), __fadd_rn(ah, bh));
}
__device__ __forceinline__ f32x2 sub2(const f32x2 a, const f32x2 b) {
    float al, ah, bl, bh;
    unpk(a, al, ah); unpk(b, bl, bh);
    return pk(__fsub_rn(al, bl), __fsub_rn(ah, bh));
}
__device__ __forceinline__ f32x2 pk1(const float v) { return pk(v, v); }
__device__ __forceinline__ float lo_of(const f32x2 v) { float a, b; unpk(v, a, b); return a; }
__device__ __forceinline__ float hi_of(const f32x2 v) { float a, b; unpk(v, a, b); return b; }
__device__ __forceinline__ float hsum(const f32x2 v) { float a, b; unpk(v, a, b); return a + b; }

}  // namespace gsb
