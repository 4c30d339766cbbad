// render.cu -- the blend kernels (K6 forward, K7 backward).  One launch covers all V views of a batch
// (blockIdx.y = view, blockIdx.x = position in the tile order), so the V tails of a per-view launch sequence
// collapse into one.
//
// Replaces FORWARD::renderCUDA / BACKWARD::renderCUDA of the reference's cuda_rasterizer/{forward,backward}.cu
// (named in BASELINE.json north_star; absent from /root/reference, SURVEY.md section 0).  Blend rules restated in
// oracle/gs_oracle.c.
//
// Data movement: a tile's sorted gaussian ids are contiguous in point_list; the 48-byte splat records they point
// to are gathered from the L2-resident record table (P * 48 B) into shared memory, 256 (forward) / 128 (backward)
// at a time.  One 16x16 tile per CTA.  While a record is staged its 2 ln(255 o) ellipse is intersected with the
// eight 8x4 patches of the tile (patch_cull.cuh); every warp walks only the records that reach its own pixels.
//
// Forward (render_fwd_kernel): one pixel per thread, a warp owns an 8x4 patch; exponent in the log2 domain (conic
// pre-scaled while staging): one MUFU.EX2 per (pixel, gaussian).
//
// Backward (render_bwd_kernel): 2x2 pixels per thread (a warp owns a 16x8 band), so the shared-memory reads, loop
// overhead and the cross-lane reduction of the ten per-gaussian gradient terms are paid once per four pixels; the
// four pixels are plain scalars (sm_90 has no packed FP32 arithmetic).  The pass walks FRONT to back with two scalars
// of state per pixel (T and U = S - F, F the running dL-weighted front colour) instead of the ten the back-to-front
// recursion carries:
//     dL/dalpha_k = T_k g_k - (S - F_k) / (1 - alpha_k),   g_k = dLdC . c_k + dLdD / z_k,
//     S = dLdC . C_out + dLdD D_out,   F_k = sum_{j<=k} alpha_j T_j g_j
// (algebraically the recursion of oracle/gs_oracle.c; background enters through C_out).  The geometric gradient
// terms are accumulated as raw moments of d(power) (sum t dx, t dy, t dx^2, t dx dy, t dy^2) and turned into
// mean / conic gradients once per gaussian in preprocess_bwd.
// The round-1 history of both kernels (v0 one-pixel back-to-front pair, scalar 2x2, patch-slot and prefetch
// variants) is in git (render.cu / render_mp.cu / render_ps.cu before round 2).
#include "blend_common.cuh"

namespace gsb {

constexpr int RB = 256;  // gaussians staged per round, forward
// CTAs per SM the backward kernels with the alpha channel are compiled for (no spills on sm_90a; DESIGN.md section 7.6)
constexpr int ALPHA_MINB = 14, ALPHA_DEPTH_MINB = 12;

// One staged gaussian = ONE 48-byte shared-memory record, so that the blend loops form one address per list entry and read the
// record with two or three 128-bit loads at fixed offsets.  (Separate arrays meant one address computation each, the third one --
// behind the alpha test -- rebuilt from the CTA's shared-window base every iteration for lack of registers.)
struct alignas(16) StagedRec {
    ulonglong2 w0;      // {(x, y), (A', C')} as two f32x2
    float4 q1;          // {B', opacity, r, g}
    float b, inv_z;
    uint32_t row;       // backward: row of the gradient accumulator (view * P + gaussian id)
    uint32_t pad;       // deterministic backward: the entry's position in the view's point list
};
static_assert(sizeof(StagedRec) == 48, "three 16-byte units");

__device__ __forceinline__ void stage_record(StagedRec &dst, float4 q0, float4 q1, const float4 q2, const uint32_t row,
                                             const uint32_t pad = 0u) {
    stage_scale(q0, q1);   // conic pre-scaled for the log2-domain exponent (blend_common.cuh): q0 = {x, y, A', C'}, q1 = {B', o, r, g}
    dst.w0 = make_ulonglong2(pk(q0.x, q0.y), pk(q0.z, q0.w));
    dst.q1 = q1;
    dst.b = q2.x; dst.inv_z = q2.y; dst.row = row; dst.pad = pad;
}

// per-view base pointers of a batched launch (blockIdx.y = view)
struct FwdView {
    const uint2 *ranges;
    const uint32_t *point_list, *order;
    const float4 *splat;
    const float *bg;
    float *out_color, *out_invdepth, *final_T;
    uint32_t *n_contrib;
};

__device__ __forceinline__ const float *select_bg(const float *const (&bg)[GSB_MAX_VIEWS], const int v) {
    const float *p = bg[0];
#pragma unroll
    for (int k = 1; k < GSB_MAX_VIEWS; ++k)
        if (k == v) p = bg[k];
    return p;
}

__device__ __forceinline__ FwdView fwd_view(const RenderFwdArgs &a) {
    const size_t v = blockIdx.y;
    FwdView f;
    f.ranges = a.ranges + v * a.sv_ranges;
    f.point_list = a.point_list + v * a.sv_list;
    f.order = a.tile_order ? a.tile_order + v * a.sv_ranges : nullptr;
    f.splat = a.splat + v * a.sv_splat;
    f.bg = select_bg(a.bg, (int)v);
    f.out_color = a.out_color + v * a.sv_color;
    f.out_invdepth = a.out_invdepth + v * a.sv_depth;
    f.final_T = a.final_T + v * a.sv_image;
    f.n_contrib = a.n_contrib + v * a.sv_image;
    return f;
}

// One CTA per 16x16 tile, eight warps.  (The alternative, CTAs of four warps on 16x8 half tiles, has fewer warps to wait for at
// the two barriers of a staging round but stages every record twice.)
__global__ void __launch_bounds__(256, 6)
render_fwd_kernel(const RenderFwdArgs a) {
    constexpr int WARPS = 8, NT = 32 * WARPS;
    __shared__ StagedRec srec[RB];
    __shared__ uint8_t smask[RB];
    __shared__ uint8_t slist[WARPS][RB];
    const FwdView f = fwd_view(a);
    const int tile = f.order ? (int)f.order[blockIdx.x] : (int)blockIdx.x;
    const int tile_x = tile % a.gx, tile_y = tile / a.gx;
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    const int px = tile_x * TILE + (w & 1) * 8 + (l & 7);     // warp w owns patch w: bit w of the staged masks
    const int py = tile_y * TILE + (w >> 1) * 4 + (l >> 3);
    const bool inside = px < a.W && py < a.H;
    const f32x2 negp = pk(-(float)px, -(float)py);
    const float ox = (float)(tile_x * TILE), oy = (float)(tile_y * TILE);
    const uint2 range = f.ranges[tile];
    const int todo = (int)(range.y - range.x);
    const int rounds = (todo + RB - 1) / RB;

    bool done = !inside;
    float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, Dp = 0.f;
    uint32_t last = 0;

    for (int rd = 0; rd < rounds; ++rd) {
        if (__syncthreads_count(done) == NT) break;
        const int idx = rd * RB + threadIdx.x;
        if (idx < todo) {
            const uint32_t g = f.point_list[range.x + idx];
            const float4 *rec = f.splat + (size_t)g * SPLAT_F4;
            const float4 q0 = __ldg(rec), q1 = __ldg(rec + 1), q2 = __ldg(rec + 2);
            smask[threadIdx.x] = (uint8_t)patch_mask(q0.x, q0.y, q0.z, q0.w, q1.x, q2.z, ox, oy);
            stage_record(srec[threadIdx.x], q0, q1, q2, 0u);
        }
        __syncthreads();
        const int n = min(RB, todo - rd * RB);
        const int cnt = compact_hits(smask, n, 1u << w, slist[w]);
        // The loop bound is per lane: a pixel that is done sets its bound to zero (one move) instead of carrying a flag through
        // the loop condition; the index of the last contributor is kept as the list position and turned into `last` once per round.
        int lim = done ? 0 : cnt;
        int lastj = -1;
        for (int k = 0; k < lim; ++k) {
            const int j = slist[w][k];
            const StagedRec &r = srec[j];
            const ulonglong2 w0 = r.w0;
            const float4 q1 = r.q1;
            // Same roundings as the backward kernel (x - px == x + (-px) in IEEE arithmetic; each pair lane is an ordinary
            // round-to-nearest multiply), so both passes agree bit for bit on alpha.
            const f32x2 d2 = add2((f32x2)w0.x, negp);
            const f32x2 u2 = mul2(mul2((f32x2)w0.y, d2), d2);
            float dx, dy, Axx, Cyy;
            unpk(d2, dx, dy);
            unpk(u2, Axx, Cyy);
            const float power = power2_at(Axx, Cyy, __fmul_rn(q1.x, dx), dy);
            const float alpha = fminf(ALPHA_MAX, __fmul_rn(q1.y, ex2_approx(power)));
            const float test_T = __fmul_rn(T, __fsub_rn(1.0f, alpha));
            // No branch in the loop body: 94 % of the warp's iterations have at least one accepting lane (ncu source page), so the
            // accept block runs anyway; predicating it saves the branch and its reconvergence pair.
            const bool hit = alpha >= ALPHA_MIN && power <= 0.0f;       // both rejections (power > 0 is a rounding rarity)
            const bool go = hit && !(test_T < T_STOP);
            lim = (hit && !go) ? 0 : lim;                                // the stop test ends this pixel's loop
            const float wgt = go ? __fmul_rn(alpha, T) : 0.0f;
            C0 = __fmaf_rn(q1.z, wgt, C0); C1 = __fmaf_rn(q1.w, wgt, C1); C2 = __fmaf_rn(r.b, wgt, C2);
            Dp = __fmaf_rn(r.inv_z, wgt, Dp);
            T = go ? test_T : T;
            lastj = go ? j : lastj;
        }
        done = done || (cnt != 0 && lim == 0);      // bound zeroed by the stop test
        if (lastj >= 0) last = (uint32_t)(rd * RB + lastj + 1);
    }
    if (inside) {
        const size_t pid = (size_t)py * a.W + px, HW = (size_t)a.W * a.H;
        f.final_T[pid] = T;
        f.n_contrib[pid] = last;
        f.out_color[pid] = C0 + T * __ldg(f.bg);
        f.out_color[HW + pid] = C1 + T * __ldg(f.bg + 1);
        f.out_color[2 * HW + pid] = C2 + T * __ldg(f.bg + 2);
        f.out_invdepth[pid] = Dp;
    }
}

// *p += v (relaxed, device scope, no return value) on the lanes with `on`, as ONE predicated instruction
__device__ __forceinline__ void red_add_on(float *p, const bool on, const float v) {
#ifdef GSB_HOST_EMUL
    if (on) atomicAdd(p, v);
#else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p red.global.add.f32 [%0], %2;\n\t}"
                 ::"l"(p), "r"((uint32_t)on), "f"(v) : "memory");
#endif
}

// Backward.  Scalar IEEE round-to-nearest arithmetic (sm_90 has no packed FP32 instruction, so pairs would buy nothing).
// Per list entry a lane evaluates its four pixels with the forward kernel's operations, then, if any lane of the warp
// blends the gaussian:
//   * U = S - F is carried instead of F, so dL/dalpha = T g - U / (1 - alpha) is one multiply and one FMA on the reciprocal;
//   * the five raw moments are formed once per lane from four basis sums of G dL/dalpha (all four pixels, column 1, row 1,
//     pixel (1, 1)): with dx0 = x - px0, sum t dx = dx0 s - s_c, sum t dx^2 = dx0 sum t dx - dx1 s_c, and alike for y and xy;
//   * they are multiplied by the opacity once, after the reduction (t = o G dL/dalpha is linear in o), on the lanes that
//     hold them;
//   * ONE transposed shuffle network (12 shuffles) reduces the nine or ten sums, whose lanes add them to the accumulator row
//     with one predicated reduction instruction.
// ALPHA: the rendered alpha A = 1 - final_T is one more channel whose per-gaussian "colour" is 1 and whose background is 0:
// g_k += dL/dA and S += dL/dA * A.  Then T_k - (A - F_k) / (1 - alpha_k) = T_final / (1 - alpha_k) = dA/dalpha_k, as it must.
// It has no colour gradient, so the accumulator row and the reduction are those of the plain kernel.
// DET (deterministic backward, DESIGN.md section 7.9): the same sums are STORED, not added: warp w's sums for list position
// pos go to partial row (pos * 2 + w) of the view, and the warp marks byte pos * 2 + w; det_reduce (deterministic.cu) adds
// the marked partials of every gaussian in ascending list order.
template <bool DEPTH, bool ALPHA, int MINB, bool DET = false>
__global__ void __launch_bounds__(64, MINB)
render_bwd_kernel(const RenderBwdArgs a) {
    constexpr int NT = 64;
    __shared__ StagedRec srec[MP_R];
    __shared__ uint32_t s_max;
    __shared__ uint8_t smask[MP_R];
    __shared__ uint8_t slist[2][MP_R];
    const size_t v = blockIdx.y;
    const uint2 *const ranges = a.ranges + v * a.sv_ranges;
    const uint32_t *const point_list = a.point_list + v * a.sv_list;
    const float4 *const splat = a.splat + v * a.sv_splat;
    const uint32_t *const n_contrib = a.n_contrib + v * a.sv_image;
    const float *const dL_dcolor = a.dL_dcolor + v * a.sv_color;
    const float *const out_color = a.out_color + v * a.sv_color;
    // accumulator rows are addressed as (view * P + gaussian) from the batch's base: the per-view offset goes into the staged
    // record once per 128 entries instead of being rebuilt in the loop (five uniform-pipe instructions per iteration before)
    const uint32_t row0 = (uint32_t)(v * (a.sv_dacc / DACC_STRIDE));
    const int tile = a.tile_order ? (int)a.tile_order[v * a.sv_ranges + blockIdx.x] : (int)blockIdx.x;
    const int ox = (tile % a.gx) * TILE, oy = (tile / a.gx) * TILE;
    const float fox = (float)ox, foy = (float)oy;
    const int t = threadIdx.x;
    const int px0 = ox + 2 * (t & 7), py0 = oy + 2 * (t >> 3);
    const uint2 range = ranges[tile];
    const size_t HW = (size_t)a.W * a.H;

    // per-pixel state: pixel i = 2 r + c is (px0 + c, py0 + r).  U = S - F (see above); rem = n_contrib - base, so that the
    // pixel blends list entry j of the current round (position base + j + 1) iff j < rem.
    float T[4], U[4], dL0[4], dL1[4], dL2[4], dLd[4], dLa[4];
    int rem[4];
    uint32_t my_max = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int px = px0 + (i & 1), py = py0 + (i >> 1);
        uint32_t last = 0u;
        float vS = 0.f, v0 = 0.f, v1 = 0.f, v2 = 0.f, vd = 0.f, va = 0.f;
        if (px < a.W && py < a.H) {
            const size_t pid = (size_t)py * a.W + px;
            last = n_contrib[pid];
            v0 = dL_dcolor[pid]; v1 = dL_dcolor[HW + pid]; v2 = dL_dcolor[2 * HW + pid];
            vS = v0 * out_color[pid] + v1 * out_color[HW + pid] + v2 * out_color[2 * HW + pid];
            if (DEPTH) { vd = a.dL_dinvdepth[v * a.sv_depth + pid]; vS += vd * a.out_invdepth[v * a.sv_depth + pid]; }
            if (ALPHA) { va = a.dL_dalpha[v * a.sv_depth + pid]; vS += va * (1.0f - a.final_T[v * a.sv_image + pid]); }
        }
        my_max = max(my_max, last);
        T[i] = 1.0f; U[i] = vS; dL0[i] = v0; dL1[i] = v1; dL2[i] = v2; dLd[i] = vd; dLa[i] = va;
        rem[i] = (int)last;
    }
    if (t == 0) s_max = 0;
    __syncthreads();
    my_max = __reduce_max_sync(0xffffffffu, my_max);
    if ((t & 31) == 0) atomicMax(&s_max, my_max);
    __syncthreads();
    const int todo = (int)s_max;
    const int my_todo = (int)my_max;
    // After reduce10_transposed a lane holds sum `slot` (= its float slot in the accumulator row); one lane per sum adds it:
    // lanes 0, 8, 4, 12, 2, 16, 24, 20, 28 (and 18 with the depth sum), i.e. the bits of ADDS.
    constexpr uint32_t ADDS = DEPTH ? 0x11151115u : 0x11111115u;

    for (int base = 0; base < todo; base += MP_R) {
        __syncthreads();
        const int n = min(MP_R, todo - base);
        for (int k = t; k < n; k += NT) {
            const uint32_t g = point_list[range.x + base + k];
            const float4 *rec = splat + (size_t)g * SPLAT_F4;
            const float4 q0 = __ldg(rec), q1 = __ldg(rec + 1), q2 = __ldg(rec + 2);
            smask[k] = (uint8_t)patch_mask(q0.x, q0.y, q0.z, q0.w, q1.x, q2.z, fox, foy);
            stage_record(srec[k], q0, q1, q2, row0 + g, DET ? range.x + (uint32_t)(base + k) : 0u);
        }
        __syncthreads();
        // The loop's per-thread constants are formed here, once per round, from an opaque copy of the thread index: hoisted
        // out of the round loop they would be live across the staging above, which then spills.  Inside the loop they are
        // neither rebuilt nor recomputed: the pixel coordinates, the lane's address in accumulator row 0 (the loop adds
        // row * 48 bytes) and lane_mask = 1 << lane, of which every lane role is one test.
        int tr = t;
#ifndef GSB_HOST_EMUL
        asm volatile("" : "+r"(tr));
#endif
        const int lane = tr & 31;
        const int slot = (lane & 2) ? 4 + 5 * (lane >> 4) : ((lane >> 1) & 2) + ((lane >> 3) & 1) + 5 * (lane >> 4);
        // DET: the lane's address in the warp's partial row of list position 0 (the loop adds pos * 96 bytes)
        float *dacc_lane = (DET ? a.det_part + (v * a.sv_list * 2 + (size_t)(tr >> 5)) * DACC_STRIDE : a.dacc) + slot;
        uint32_t lane_mask = 1u << lane;
#ifndef GSB_HOST_EMUL
        asm volatile("" : "+l"(dacc_lane), "+r"(lane_mask));
#endif
        const float fx0 = fox + (float)(2 * (tr & 7)), fy0 = foy + (float)(2 * (tr >> 3));    // exact: px0, py0
        const float fx1 = __fadd_rn(fx0, 1.0f), fy1 = __fadd_rn(fy0, 1.0f);
        const int nw = max(0, min(n, my_todo - base));
        const int cnt = compact_hits(smask, nw, 0xfu << (4 * (tr >> 5)), slist[tr >> 5]);
        for (int kk = 0; kk < cnt; ++kk) {
            const int j = (int)slist[t >> 5][kk];
            const StagedRec &rec = srec[j];
            const float4 q1 = rec.q1;                    // {B', o, r, g}
            float x, y, A, C;                            // A', C'
            unpk((f32x2)rec.w0.x, x, y);
            unpk((f32x2)rec.w0.y, A, C);
            // the forward kernel's operations (x - px == x + (-px)), so that both passes agree bit for bit on alpha
            const float dx[2] = {__fsub_rn(x, fx0), __fsub_rn(x, fx1)}, dy[2] = {__fsub_rn(y, fy0), __fsub_rn(y, fy1)};
            float G[4], al[4];
            bool valid[4];
            bool any = false;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float dxc = dx[i & 1], dyr = dy[i >> 1];
                const float p = power2_at(__fmul_rn(__fmul_rn(A, dxc), dxc), __fmul_rn(__fmul_rn(C, dyr), dyr), __fmul_rn(q1.x, dxc), dyr);
                G[i] = ex2_approx(p);
                al[i] = fminf(ALPHA_MAX, __fmul_rn(q1.y, G[i]));
                valid[i] = (p <= 0.0f) && (al[i] >= ALPHA_MIN) && (j < rem[i]);
                any = any || valid[i];
            }
            if (!__any_sync(0xffffffffu, any)) continue;
            const float cb = rec.b, cd = rec.inv_z;
            float Gd[4], sum[10];                        // sum: the accumulator row's slots 0..9 (moments still without o)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                // invalid pixels: alpha = 0 and G = 0 make every contribution below exactly zero
                const float ai = valid[i] ? al[i] : 0.0f, Gi = valid[i] ? G[i] : 0.0f;
                const float w = __fmul_rn(ai, T[i]);
                float g = __fmaf_rn(dL2[i], cb, __fmaf_rn(dL1[i], q1.w, __fmul_rn(dL0[i], q1.z)));
                if (DEPTH) g = __fmaf_rn(dLd[i], cd, g);
                if (ALPHA) g = __fadd_rn(g, dLa[i]);
                U[i] = __fmaf_rn(-w, g, U[i]);
                const float om = __fsub_rn(1.0f, ai);
                Gd[i] = __fmul_rn(Gi, __fmaf_rn(-U[i], rcp_approx(om), __fmul_rn(T[i], g)));     // G dL/dalpha
                T[i] = __fmul_rn(T[i], om);
                if (i == 0) {     // the sums START at the first pixel's terms (0 + x is not folded away: it turns -0 into +0)
                    sum[6] = __fmul_rn(w, dL0[i]); sum[7] = __fmul_rn(w, dL1[i]); sum[8] = __fmul_rn(w, dL2[i]);
                    sum[9] = DEPTH ? __fmul_rn(w, dLd[i]) : 0.0f;
                } else {
                    sum[6] = __fmaf_rn(w, dL0[i], sum[6]); sum[7] = __fmaf_rn(w, dL1[i], sum[7]); sum[8] = __fmaf_rn(w, dL2[i], sum[8]);
                    if (DEPTH) sum[9] = __fmaf_rn(w, dLd[i], sum[9]);
                }
            }
            // basis sums over the pixels of column 1 and of row 1; sum 5 (opacity) is the sum over all four
            const float s_c = __fadd_rn(Gd[1], Gd[3]), s_r = __fadd_rn(Gd[2], Gd[3]);
            sum[5] = __fadd_rn(__fadd_rn(Gd[0], Gd[2]), s_c);
            sum[0] = __fmaf_rn(dx[0], sum[5], -s_c);                                   // sum G dL/dalpha dx
            sum[1] = __fmaf_rn(dy[0], sum[5], -s_r);                                   // ... dy
            sum[2] = __fmaf_rn(dx[0], sum[0], -__fmul_rn(dx[1], s_c));                 // ... dx^2
            sum[3] = __fmaf_rn(dy[0], sum[0], __fmaf_rn(-dx[0], s_r, Gd[3]));          // ... dx dy
            sum[4] = __fmaf_rn(dy[0], sum[1], -__fmul_rn(dy[1], s_r));                 // ... dy^2
            const LaneBits lb = lane_bits(lane_mask);
            float r = reduce10_transposed<DEPTH>(sum, lb);
            r = lb.b4 ? r : __fmul_rn(r, q1.y);          // lanes 0..15 hold sums 0..4: the moments' opacity factor
            if (DET) {
                if (lane_mask & ADDS) dacc_lane[(size_t)rec.pad * (2 * DACC_STRIDE)] = r;
                if (lane_mask & 1u) a.det_mark[(v * a.sv_list + rec.pad) * 2 + (size_t)(tr >> 5)] = 1u;
            } else {
                red_add_on(dacc_lane + (size_t)rec.row * DACC_STRIDE, (lane_mask & ADDS) != 0u, r);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) rem[i] -= MP_R;
    }
}

// Tile order for the blend launches: tiles by DESCENDING list length (longest-processing-time-first), so that the heavy
// tiles start in the first wave and the light ones fill the tail.  One block per view: a counting sort of the tiles on
// a 256-bin quantisation of their list length.
__global__ void __launch_bounds__(256)
tile_order_kernel(const uint2 *__restrict__ ranges, const int num_tiles, uint32_t *__restrict__ order) {
    __shared__ uint32_t cnt[256], warp_sums[8];
    ranges += (size_t)blockIdx.x * num_tiles; order += (size_t)blockIdx.x * num_tiles;
    cnt[threadIdx.x] = 0u;
    __syncthreads();
    // bin 0 = longest: 255 - min(255, len / 16 rounded into 0..255 with a log-ish top)
    auto bin_of = [](const uint2 r) {
        const uint32_t len = r.y - r.x;
        const uint32_t q = len < 2048u ? (len >> 4) : min(255u, 128u + ((len - 2048u) >> 7));
        return 255u - q;
    };
    for (int t = threadIdx.x; t < num_tiles; t += 256) atomicAdd(&cnt[bin_of(ranges[t])], 1u);
    __syncthreads();
    // exclusive scan of the 256 bins
    const uint32_t c = cnt[threadIdx.x];
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)(threadIdx.x & 31) >= o) incl += n;
    }
    if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = incl;
    __syncthreads();
    uint32_t basev = 0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) basev += warp_sums[w];
    __syncthreads();
    cnt[threadIdx.x] = basev + incl - c;
    __syncthreads();
    // placement (order inside a bin is irrelevant: the permutation only schedules CTAs, results do not depend on it)
    for (int t = threadIdx.x; t < num_tiles; t += 256) order[atomicAdd(&cnt[bin_of(ranges[t])], 1u)] = (uint32_t)t;
}

static int check_views(const char *what, int V, int tiles) {
    if (V < 1 || V > GSB_MAX_VIEWS || tiles > 0x7fffffff / GSB_MAX_VIEWS) {
        set_error("%s: bad launch geometry (V=%d, tiles=%d)", what, V, tiles);
        return GSB_ERR_ARGUMENT;
    }
    return GSB_OK;
}

int launch_tile_order(const uint2 *ranges, int V, int num_tiles, uint32_t *order, bool debug, cudaStream_t stream) {
    if (num_tiles <= 0) return GSB_OK;
    int rc = check_views("tile_order", V, num_tiles);
    if (rc) return rc;
    GSB_LAUNCH("tile_order", debug, stream, tile_order_kernel, V, 256, 0, ranges, num_tiles, order);
    return GSB_OK;
}

int launch_render_fwd(const RenderFwdArgs &a, bool debug, cudaStream_t stream) {
    const int tiles = a.gx * a.gy;
    if (tiles <= 0) return GSB_OK;
    int rc = check_views("render_fwd", a.V, tiles);
    if (rc) return rc;
    GSB_LAUNCH("render_fwd", debug, stream, render_fwd_kernel, dim3(tiles, a.V), 256, 0, a);
    return GSB_OK;
}

template <bool DET>
static int launch_render_bwd_t(const RenderBwdArgs &a, const int tiles, bool debug, cudaStream_t stream) {
    const char *name = DET ? "render_bwd_det" : "render_bwd";
    if (a.dL_dalpha) {   // register budgets: DESIGN.md section 7.6
        if (a.dL_dinvdepth) {
            GSB_LAUNCH(name, debug, stream, (render_bwd_kernel<true, true, ALPHA_DEPTH_MINB, DET>), dim3(tiles, a.V), 64, 0, a);
        } else {
            GSB_LAUNCH(name, debug, stream, (render_bwd_kernel<false, true, ALPHA_MINB, DET>), dim3(tiles, a.V), 64, 0, a);
        }
    } else if (a.dL_dinvdepth) {
        GSB_LAUNCH(name, debug, stream, (render_bwd_kernel<true, false, 12, DET>), dim3(tiles, a.V), 64, 0, a);
    } else {   // register budget for 16 CTAs/SM (64 registers, no spills on sm_90a)
        GSB_LAUNCH(name, debug, stream, (render_bwd_kernel<false, false, 16, DET>), dim3(tiles, a.V), 64, 0, a);
    }
    return GSB_OK;
}

int launch_render_bwd(const RenderBwdArgs &a, bool debug, cudaStream_t stream) {
    const int tiles = a.gx * a.gy;
    if (tiles <= 0) return GSB_OK;
    int rc = check_views("render_bwd", a.V, tiles);
    if (rc) return rc;
    if (a.dL_dalpha && !a.final_T) {
        set_error("render_bwd: dL_dalpha without final_T");
        return GSB_ERR_ARGUMENT;
    }
    if ((a.det_part == nullptr) != (a.det_mark == nullptr)) {
        set_error("render_bwd: deterministic partials without marks");
        return GSB_ERR_ARGUMENT;
    }
    if (a.det_part) return launch_render_bwd_t<true>(a, tiles, debug, stream);
    return launch_render_bwd_t<false>(a, tiles, debug, stream);
}

// Rendered alpha of V forward states: one launch, blockIdx.y = view.  The forward leaves final_T in every state's IMAGE buffer;
// nothing else is read.
__global__ void __launch_bounds__(256)
alpha_kernel(const AlphaArgs a) {
    const float *T = a.final_T[0];
#pragma unroll
    for (int k = 1; k < GSB_MAX_VIEWS; ++k)
        if (k == (int)blockIdx.y) T = a.final_T[k];
    float *out = a.out + (size_t)blockIdx.y * a.npix;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < a.npix; i += (size_t)gridDim.x * 256)
        out[i] = __fsub_rn(1.0f, __ldg(T + i));
}

int launch_alpha(const AlphaArgs &a, bool debug, cudaStream_t stream) {
    if (a.npix == 0) return GSB_OK;
    if (a.V < 1 || a.V > GSB_MAX_VIEWS) {
        set_error("alpha: bad launch geometry (V=%d)", a.V);
        return GSB_ERR_ARGUMENT;
    }
    const size_t blocks = (a.npix + 255) / 256;
    GSB_LAUNCH("render_alpha", debug, stream, alpha_kernel, dim3((unsigned)(blocks < 4096 ? blocks : 4096), a.V), 256, 0, a);
    return GSB_OK;
}

}  // namespace gsb
