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
// two pixels of a row share every per-gaussian operand and are carried as f32x2 register pairs.  The pass walks
// FRONT to back with two scalars of state per pixel (T and the running dL-weighted front colour F) instead of the
// ten the back-to-front recursion carries:
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
    uint32_t pad;
};
static_assert(sizeof(StagedRec) == 48, "three 16-byte units");

__device__ __forceinline__ void stage_record(StagedRec &dst, float4 q0, float4 q1, const float4 q2, const uint32_t row) {
    stage_scale(q0, q1);   // conic pre-scaled for the log2-domain exponent (blend_common.cuh): q0 = {x, y, A', C'}, q1 = {B', o, r, g}
    dst.w0 = make_ulonglong2(pk(q0.x, q0.y), pk(q0.z, q0.w));
    dst.q1 = q1;
    dst.b = q2.x; dst.inv_z = q2.y; dst.row = row; dst.pad = 0u;
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

// *(float *)(base + off) += v (relaxed, device scope, no return value) for the lanes with off >= 0, as ONE predicated instruction
__device__ __forceinline__ void red_add_if(char *base, const int off, const float v) {
#ifdef GSB_HOST_EMUL
    if (off >= 0) atomicAdd(reinterpret_cast<float *>(base + off), v);
#else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ge.s32 p, %1, 0;\n\t@p red.global.add.f32 [%0], %2;\n\t}"
                 ::"l"(base + (off < 0 ? 0 : off)), "r"(off), "f"(v) : "memory");
#endif
}

// Backward.  Arithmetic per lane is IEEE round-to-nearest (the f32x2 helpers are pairs of _rn scalar instructions).
// ALPHA: the rendered alpha A = 1 - final_T is one more channel whose per-gaussian "colour" is 1 and whose background is 0:
// g_k += dL/dA and S += dL/dA * A.  Then T_k - (A - F_k) / (1 - alpha_k) = T_final / (1 - alpha_k) = dA/dalpha_k, as it must.
// It has no colour gradient, so the accumulator row, the shuffle networks and the reduction are those of the plain kernel.
template <bool DEPTH, bool ALPHA, int MINB>
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
    const uint32_t want = 0xfu << (4 * (threadIdx.x >> 5));
    const int tile = a.tile_order ? (int)a.tile_order[v * a.sv_ranges + blockIdx.x] : (int)blockIdx.x;
    const int ox = (tile % a.gx) * TILE, oy = (tile / a.gx) * TILE;
    const int t = threadIdx.x;
    const int px0 = ox + 2 * (t & 7), py0 = oy + 2 * (t >> 3);
    const float fx0 = (float)px0, fy0 = (float)py0;
    const uint2 range = ranges[tile];
    const size_t HW = (size_t)a.W * a.H;

    // per-pixel state, packed by row: element c of row r is pixel (px0 + c, py0 + r)
    f32x2 T[2], F[2], S[2], dL0[2], dL1[2], dL2[2], dLd[2], dLa[2];
    uint32_t last[4];
    uint32_t my_max = 0;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float vS[2] = {0.f, 0.f}, v0[2] = {0.f, 0.f}, v1[2] = {0.f, 0.f}, v2[2] = {0.f, 0.f}, vd[2] = {0.f, 0.f}, va[2] = {0.f, 0.f};
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int px = px0 + c, py = py0 + r;
            last[2 * r + c] = 0u;
            if (px < a.W && py < a.H) {
                const size_t pid = (size_t)py * a.W + px;
                last[2 * r + c] = n_contrib[pid];
                v0[c] = dL_dcolor[pid]; v1[c] = dL_dcolor[HW + pid]; v2[c] = dL_dcolor[2 * HW + pid];
                vS[c] = v0[c] * out_color[pid] + v1[c] * out_color[HW + pid] + v2[c] * out_color[2 * HW + pid];
                if (DEPTH) { vd[c] = a.dL_dinvdepth[v * a.sv_depth + pid]; vS[c] += vd[c] * a.out_invdepth[v * a.sv_depth + pid]; }
                if (ALPHA) { va[c] = a.dL_dalpha[v * a.sv_depth + pid]; vS[c] += va[c] * (1.0f - a.final_T[v * a.sv_image + pid]); }
            }
            my_max = max(my_max, last[2 * r + c]);
        }
        T[r] = pk1(1.0f); F[r] = pk1(0.0f); S[r] = pk(vS[0], vS[1]);
        dL0[r] = pk(v0[0], v0[1]); dL1[r] = pk(v1[0], v1[1]); dL2[r] = pk(v2[0], v2[1]); dLd[r] = pk(vd[0], vd[1]);
        dLa[r] = pk(va[0], va[1]);
    }
    if (t == 0) s_max = 0;
    __syncthreads();
    my_max = __reduce_max_sync(0xffffffffu, my_max);
    if ((t & 31) == 0) atomicMax(&s_max, my_max);
    __syncthreads();
    const int todo = (int)s_max;
    const int my_todo = (int)my_max;
    const f32x2 one2 = pk1(1.0f);
    const int lane = t & 31;
    int red_off = (lane & 3) == 0 ? 4 * (lane >> 2) : (lane == 1 ? 32 : (DEPTH && lane == 17 ? 36 : -1));
#ifndef GSB_HOST_EMUL
    asm volatile("" : "+r"(red_off));      // opaque from here on: kept in a register instead of being rebuilt from the lane id in the loop
#endif

    for (int base = 0; base < todo; base += MP_R) {
        __syncthreads();
        const int n = min(MP_R, todo - base);
        for (int k = t; k < n; k += NT) {
            const uint32_t g = point_list[range.x + base + k];
            const float4 *rec = splat + (size_t)g * SPLAT_F4;
            const float4 q0 = __ldg(rec), q1 = __ldg(rec + 1), q2 = __ldg(rec + 2);
            smask[k] = (uint8_t)patch_mask(q0.x, q0.y, q0.z, q0.w, q1.x, q2.z, (float)ox, (float)oy);
            stage_record(srec[k], q0, q1, q2, row0 + g);
        }
        __syncthreads();
        const int nw = max(0, min(n, my_todo - base));
        const int cnt = compact_hits(smask, nw, want, slist[t >> 5]);
        for (int kk = 0; kk < cnt; ++kk) {
            const int j = (int)slist[t >> 5][kk];
            const StagedRec &rec = srec[j];
            const float4 q1 = rec.q1;
            float4 q0;                                   // {x, y, A', C'}
            unpk((f32x2)rec.w0.x, q0.x, q0.y);
            unpk((f32x2)rec.w0.y, q0.z, q0.w);
            const uint32_t pos = (uint32_t)(base + j + 1);
            // column-packed terms (shared by both rows): dx, A' dx^2, B' dx
            const f32x2 dx2 = pk(q0.x - fx0, q0.x - (fx0 + 1.0f));   // same rounding as the forward kernel
            const f32x2 Axx2 = mul2(mul2(pk1(q0.z), dx2), dx2);
            const f32x2 Bx2 = mul2(pk1(q1.x), dx2);
            float dy[2], Cyy[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                dy[r] = q0.y - (fy0 + (float)r);
                Cyy[r] = __fmul_rn(__fmul_rn(q0.w, dy[r]), dy[r]);
            }
            float G[4], al[4];
            bool valid[4];
            bool any = false;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                // power2_at(Axx, Cyy, Bx, dy) = fma(Bx, dy, Axx + Cyy), both columns at once
                const f32x2 p2 = fma2(Bx2, pk1(dy[r]), add2(Axx2, pk1(Cyy[r])));
                float p[2];
                unpk(p2, p[0], p[1]);
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int i = 2 * r + c;
                    G[i] = ex2_approx(p[c]);
                    al[i] = fminf(ALPHA_MAX, __fmul_rn(q1.y, G[i]));
                    valid[i] = (p[c] <= 0.0f) && (al[i] >= ALPHA_MIN) && (pos <= last[i]);
                    any = any || valid[i];
                }
            }
            if (!__any_sync(0xffffffffu, any)) continue;
            const float2 q2 = make_float2(rec.b, rec.inv_z);
            f32x2 m_x = pk1(0.f), m_y = m_x, m_xx = m_x, m_xy = m_x, m_yy = m_x, g_o = m_x, g_r = m_x, g_g = m_x, g_b = m_x, g_d = m_x;
            const f32x2 cr = pk1(q1.z), cg = pk1(q1.w), cb = pk1(q2.x), cd = pk1(q2.y), op2 = pk1(q1.y);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int i0 = 2 * r, i1 = 2 * r + 1;
                // invalid lanes: alpha = 0 and G = 0 make every contribution below exactly zero
                const f32x2 ai = pk(valid[i0] ? al[i0] : 0.0f, valid[i1] ? al[i1] : 0.0f);
                const f32x2 Gm = pk(valid[i0] ? G[i0] : 0.0f, valid[i1] ? G[i1] : 0.0f);
                const f32x2 w = mul2(ai, T[r]);
                f32x2 g = fma2(dL2[r], cb, fma2(dL1[r], cg, mul2(dL0[r], cr)));
                if (DEPTH) g = fma2(dLd[r], cd, g);
                if (ALPHA) g = add2(g, dLa[r]);
                F[r] = fma2(w, g, F[r]);
                if (r == 0) {
                    g_r = mul2(w, dL0[r]); g_g = mul2(w, dL1[r]); g_b = mul2(w, dL2[r]);
                    if (DEPTH) g_d = mul2(w, dLd[r]);
                } else {
                    g_r = fma2(w, dL0[r], g_r); g_g = fma2(w, dL1[r], g_g); g_b = fma2(w, dL2[r], g_b);
                    if (DEPTH) g_d = fma2(w, dLd[r], g_d);
                }
                const f32x2 om = sub2(one2, ai);
                float om0, om1;
                unpk(om, om0, om1);
                const f32x2 rcp = pk(rcp_approx(om0), rcp_approx(om1));
                // dL/dalpha = T g - (S - F) / (1 - alpha); multiplied by G (0 for invalid lanes) wherever it is used
                const f32x2 dLda = sub2(mul2(T[r], g), mul2(sub2(S[r], F[r]), rcp));
                T[r] = mul2(T[r], om);
                const f32x2 Gd = mul2(Gm, dLda);
                const f32x2 tt = mul2(op2, Gd);
                const f32x2 dy2 = pk1(dy[r]);
                const f32x2 u = mul2(tt, dx2), vv = mul2(tt, dy2);
                if (r == 0) {     // the sums START at the first row's terms (0 + x is not folded away: it turns -0 into +0)
                    g_o = Gd; m_x = u; m_y = vv;
                    m_xx = mul2(u, dx2); m_xy = mul2(u, dy2); m_yy = mul2(vv, dy2);
                } else {
                    g_o = add2(g_o, Gd); m_x = add2(m_x, u); m_y = add2(m_y, vv);
                    m_xx = fma2(u, dx2, m_xx); m_xy = fma2(u, dy2, m_xy); m_yy = fma2(vv, dy2, m_yy);
                }
            }
            // both shuffle networks are issued before the atomic so that their (independent) chains overlap
            const float ra = reduce8_transposed(hsum(m_x), hsum(m_y), hsum(m_xx), hsum(m_xy), hsum(m_yy), hsum(g_o), hsum(g_r), hsum(g_g));
            float rb;
            if (DEPTH) {
                rb = reduce2_transposed(hsum(g_b), hsum(g_d));
            } else {
                rb = hsum(g_b);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) rb += __shfl_xor_sync(0xffffffffu, rb, o);
            }
            // ONE predicated reduction instruction for the ten sums: lanes 0, 4, ..., 28 hold sums 0..7 (ra), lane 1 (and 17 with a
            // depth gradient) the remaining ones (rb); red_off is the lane's byte offset into the 48-byte accumulator row or -1
            // (computed once per thread: the loop used to rebuild the lane roles and branch around two atomics every iteration).
            red_add_if(reinterpret_cast<char *>(a.dacc + (size_t)rec.row * DACC_STRIDE), red_off, red_off >= 32 ? rb : ra);
        }
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

int launch_render_bwd(const RenderBwdArgs &a, bool debug, cudaStream_t stream) {
    const int tiles = a.gx * a.gy;
    if (tiles <= 0) return GSB_OK;
    int rc = check_views("render_bwd", a.V, tiles);
    if (rc) return rc;
    if (a.dL_dalpha && !a.final_T) {
        set_error("render_bwd: dL_dalpha without final_T");
        return GSB_ERR_ARGUMENT;
    }
    if (a.dL_dalpha) {   // register budgets: DESIGN.md section 7.6
        if (a.dL_dinvdepth) {
            GSB_LAUNCH("render_bwd", debug, stream, (render_bwd_kernel<true, true, ALPHA_DEPTH_MINB>), dim3(tiles, a.V), 64, 0, a);
        } else {
            GSB_LAUNCH("render_bwd", debug, stream, (render_bwd_kernel<false, true, ALPHA_MINB>), dim3(tiles, a.V), 64, 0, a);
        }
    } else if (a.dL_dinvdepth) {
        GSB_LAUNCH("render_bwd", debug, stream, (render_bwd_kernel<true, false, 12>), dim3(tiles, a.V), 64, 0, a);
    } else {   // register budget for 16 CTAs/SM (64 registers, no spills on sm_90a)
        GSB_LAUNCH("render_bwd", debug, stream, (render_bwd_kernel<false, false, 16>), dim3(tiles, a.V), 64, 0, a);
    }
    return GSB_OK;
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
