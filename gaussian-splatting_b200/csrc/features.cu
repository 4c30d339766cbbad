// features.cu -- rendered feature maps: C per-gaussian channels composited with the forward's own blend weights
// (gsb_render_features, gsb_backward_features, gsb_backward_batch_features; DESIGN.md section 7.7).
//
//     F[c][p] = sum_k w_k(p) features[id_k][c],   w_k = alpha_k T_k,   background 0
//
// Nothing is binned again: both kernels read a forward state (ranges, point_list, tile_order, the 48-byte splat records and
// n_contrib) and accept exactly the pairs render_bwd_kernel reproduces: power <= 0, alpha >= 1/255 and list position <=
// n_contrib.  The per-pair arithmetic is that of the blend kernels (render.cu): the same staging scale, the same exponent
// with the same roundings, fmaf(f, w, F) in list order.  So the forward equals, bit for bit, the colour output of a
// colors_precomp call with a black background whose colours are three of the feature channels.
//
// Channels go in groups of G = 4 or 8 (blockIdx.z, the last group padded with zeros); views in blockIdx.y, each one a forward
// state of its own (any forward entry point, up to GSB_MAX_VIEWS per launch).  Every group recomputes the exponents: the
// blend weights are cheaper to recompute than to store.  A staged gaussian is one shared-memory record: its conic, opacity
// and id next to the group's G feature values, read with 128-bit broadcast loads.
//
// Backward (render_features_bwd_kernel): render_bwd_kernel's front-to-back scheme with one channel group as the "colour",
//     dL/dalpha_k = T_k g_k - (S - F_k) / (1 - alpha_k),   g_k = sum_c dL/dF_c f_kc,   S = sum_c dL/dF_c F_out_c
// (F_k the running dL-weighted front sum).  dL/dalpha is linear in the loss gradient, so every group ADDS its raw-moment and
// opacity terms into the first six floats of the accumulator row that render_bwd_kernel fills; preprocess_bwd turns the
// summed row into the mean, conic, opacity and camera gradients unchanged.  dL/dfeatures[id][c] = sum_p w_k(p) dL/dF_c(p)
// is reduced across the warp and added with one red.add per sum, summed over the views of a batch.
#include "blend_common.cuh"

namespace gsb {

constexpr int FEAT_RB = 256;   // gaussians staged per round, forward (the backward stages MP_R)
// CTAs per SM the kernels are compiled for (no spills on sm_90a; register table in DESIGN.md section 7.7)
constexpr int FEAT_FWD_MINB = 4, FEAT_BWD_MINB4 = 12, FEAT_BWD_MINB8 = 8;

template <int G>
struct alignas(16) FeatRec {
    ulonglong2 w0;      // {(x, y), (A', C')} as two f32x2 (blend_common.cuh stage_scale)
    float bp, op;       // B', opacity
    uint32_t id, pad;   // gaussian id
    float f[G];         // features[id][c0 .. c0 + G), 0 past the last channel
};

// the forward state of view v: kernel parameters selected with uniform compares instead of a dynamic index (which would
// copy the whole parameter block to local memory)
__device__ __forceinline__ FeatView pick_view(const FeatArgs &a, const int v) {
    FeatView f = a.view[0];
#pragma unroll
    for (int k = 1; k < GSB_MAX_VIEWS; ++k)
        if (k == v) f = a.view[k];
    return f;
}

template <int G>
__device__ __forceinline__ uint8_t stage_feat(FeatRec<G> &dst, const float4 *splat, const uint32_t g, const FeatArgs &a, const int c0,
                                              const float ox, const float oy) {
    const float4 *rec = splat + (size_t)g * SPLAT_F4;
    float4 q0 = __ldg(rec), q1 = __ldg(rec + 1);
    const float4 q2 = __ldg(rec + 2);
    const uint8_t mask = (uint8_t)patch_mask(q0.x, q0.y, q0.z, q0.w, q1.x, q2.z, ox, oy);
    stage_scale(q0, q1);
    dst.w0 = make_ulonglong2(pk(q0.x, q0.y), pk(q0.z, q0.w));
    dst.bp = q1.x; dst.op = q1.y; dst.id = g; dst.pad = 0u;
    const float *src = a.features + (size_t)g * a.C + c0;
#pragma unroll
    for (int c = 0; c < G; ++c) dst.f[c] = c0 + c < a.C ? __ldg(src + c) : 0.0f;
    return mask;
}

template <int G>
__device__ __forceinline__ void load_feats(const FeatRec<G> &r, float (&fv)[G]) {
#pragma unroll
    for (int c = 0; c < G; c += 4) {
        const float4 q = *reinterpret_cast<const float4 *>(&r.f[c]);
        fv[c] = q.x; fv[c + 1] = q.y; fv[c + 2] = q.z; fv[c + 3] = q.w;
    }
}

// largest n_contrib over the CTA's pixels (list entries behind it blend no pixel of the tile); `mine` = this thread's
__device__ __forceinline__ int tile_max(uint32_t mine, uint32_t *s_max) {
    if (threadIdx.x == 0) *s_max = 0u;
    __syncthreads();
    mine = __reduce_max_sync(0xffffffffu, mine);
    if ((threadIdx.x & 31) == 0) atomicMax(s_max, mine);
    __syncthreads();
    return (int)*s_max;
}

// Forward: K6's layout (one pixel per thread, a warp owns an 8x4 patch), walking each pixel's list up to n_contrib.
template <int G>
__global__ void __launch_bounds__(256, FEAT_FWD_MINB)
render_features_kernel(const FeatArgs a) {
    constexpr int WARPS = 8;
    __shared__ FeatRec<G> srec[FEAT_RB];
    __shared__ uint8_t smask[FEAT_RB];
    __shared__ uint8_t slist[WARPS][FEAT_RB];
    __shared__ uint32_t s_max;
    const int v = (int)blockIdx.y, c0 = (int)blockIdx.z * G;
    const FeatView f = pick_view(a, v);
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
    const int todo = tile_max(last, &s_max);

    float T = 1.0f, acc[G];
#pragma unroll
    for (int c = 0; c < G; ++c) acc[c] = 0.0f;
    for (int base = 0; base < todo; base += FEAT_RB) {
        __syncthreads();
        const int n = min(FEAT_RB, todo - base);
        if ((int)threadIdx.x < n)
            smask[threadIdx.x] = stage_feat<G>(srec[threadIdx.x], f.splat, f.point_list[range.x + base + threadIdx.x], a, c0, ox, oy);
        __syncthreads();
        const int cnt = compact_hits(smask, max(0, min(n, wmax - base)), 1u << w, slist[w]);
        for (int k = 0; k < cnt; ++k) {
            const int j = slist[w][k];
            const FeatRec<G> &r = srec[j];
            // render_fwd_kernel's arithmetic, operation for operation
            const f32x2 d2 = add2((f32x2)r.w0.x, negp);
            const f32x2 u2 = mul2(mul2((f32x2)r.w0.y, d2), d2);
            float dx, dy, Axx, Cyy;
            unpk(d2, dx, dy);
            unpk(u2, Axx, Cyy);
            const float power = power2_at(Axx, Cyy, __fmul_rn(r.bp, dx), dy);
            const float alpha = fminf(ALPHA_MAX, __fmul_rn(r.op, ex2_approx(power)));
            const bool ok = alpha >= ALPHA_MIN && power <= 0.0f && (uint32_t)(base + j + 1) <= last;
            const float wgt = ok ? __fmul_rn(alpha, T) : 0.0f;
            float fv[G];
            load_feats<G>(r, fv);
#pragma unroll
            for (int c = 0; c < G; ++c) acc[c] = __fmaf_rn(fv[c], wgt, acc[c]);
            T = ok ? __fmul_rn(T, __fsub_rn(1.0f, alpha)) : T;
        }
    }
    if (inside) {
        const size_t HW = (size_t)a.W * a.H;
        float *out = a.out + ((size_t)v * a.C + c0) * HW + pid;
#pragma unroll
        for (int c = 0; c < G; ++c)
            if (c0 + c < a.C) out[c * HW] = acc[c];
    }
}

// *p += v (relaxed, device scope, no return value) for the lanes with `on`, as ONE predicated instruction
__device__ __forceinline__ void red_add_pred(float *p, const bool on, const float v) {
#ifdef GSB_HOST_EMUL
    if (on) atomicAdd(p, v);
#else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p red.global.add.f32 [%0], %2;\n\t}"
                 ::"l"(p), "r"((uint32_t)on), "f"(v) : "memory");
#endif
}

// Backward: K7's layout (2x2 pixels per thread carried as f32x2 row pairs, a warp owns a 16x8 band, 128 records per round).
template <int G, int MINB>
__global__ void __launch_bounds__(64, MINB)
render_features_bwd_kernel(const FeatArgs a) {
    constexpr int NT = 64;
    __shared__ FeatRec<G> srec[MP_R];
    __shared__ uint32_t s_max;
    __shared__ uint8_t smask[MP_R];
    __shared__ uint8_t slist[2][MP_R];
    const int v = (int)blockIdx.y, c0 = (int)blockIdx.z * G;
    const FeatView f = pick_view(a, v);
    const size_t row0 = (size_t)v * a.P;
    const uint32_t want = 0xfu << (4 * (threadIdx.x >> 5));
    const int tile = f.tile_order ? (int)f.tile_order[blockIdx.x] : (int)blockIdx.x;
    const int ox = (tile % a.gx) * TILE, oy = (tile / a.gx) * TILE;
    const int t = threadIdx.x;
    const int px0 = ox + 2 * (t & 7), py0 = oy + 2 * (t >> 3);
    const float fx0 = (float)px0, fy0 = (float)py0;
    const uint2 range = f.ranges[tile];
    const size_t HW = (size_t)a.W * a.H;
    const float *const dLdF = a.dL_dout + ((size_t)v * a.C + c0) * HW;
    const float *const Fout = a.out_features + ((size_t)v * a.C + c0) * HW;

    // per-pixel state, packed by row: element c of row r is pixel (px0 + c, py0 + r)
    f32x2 T[2], F[2], S[2], dL[G][2];
    uint32_t last[4];
    uint32_t my_max = 0;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        float vS[2] = {0.f, 0.f}, vd[G][2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int px = px0 + c, py = py0 + r;
            last[2 * r + c] = 0u;
#pragma unroll
            for (int ch = 0; ch < G; ++ch) vd[ch][c] = 0.f;
            if (px < a.W && py < a.H) {
                const size_t pid = (size_t)py * a.W + px;
                last[2 * r + c] = f.n_contrib[pid];
#pragma unroll
                for (int ch = 0; ch < G; ++ch)
                    if (c0 + ch < a.C) {
                        vd[ch][c] = dLdF[ch * HW + pid];
                        vS[c] += vd[ch][c] * Fout[ch * HW + pid];
                    }
            }
            my_max = max(my_max, last[2 * r + c]);
        }
        T[r] = pk1(1.0f); F[r] = pk1(0.0f); S[r] = pk(vS[0], vS[1]);
#pragma unroll
        for (int ch = 0; ch < G; ++ch) dL[ch][r] = pk(vd[ch][0], vd[ch][1]);
    }
    my_max = __reduce_max_sync(0xffffffffu, my_max);
    const int todo = tile_max(my_max, &s_max);
    const int my_todo = (int)my_max;
    const f32x2 one2 = pk1(1.0f);
    // ONE predicated red.add per lane and pair: lane 4k holds sum k of ra (k < 6: accumulator float k; 6, 7: channels 0, 1);
    // with G = 8 lane 4k + 1 holds sum k of rb (channel 2 + k, k < 6); with G = 4 lanes 1 and 17 hold channels 2 and 3
    const int lane = t & 31;
    int acc_k = -1, fch = -1;
    if ((lane & 3) == 0) {
        if ((lane >> 2) < 6) acc_k = lane >> 2; else fch = (lane >> 2) - 6;
    } else if (G == 8 && (lane & 3) == 1 && (lane >> 2) < 6) {
        fch = 2 + (lane >> 2);
    } else if (G == 4 && (lane == 1 || lane == 17)) {
        fch = lane == 1 ? 2 : 3;
    }
    if (fch >= 0 && (c0 + fch >= a.C || !a.dL_dfeatures)) fch = -1;
    const bool red_on = acc_k >= 0 || fch >= 0;
    const bool from_rb = (lane & 3) != 0;

    for (int base = 0; base < todo; base += MP_R) {
        __syncthreads();
        const int n = min(MP_R, todo - base);
        for (int k = t; k < n; k += NT)
            smask[k] = stage_feat<G>(srec[k], f.splat, f.point_list[range.x + base + k], a, c0, (float)ox, (float)oy);
        __syncthreads();
        const int nw = max(0, min(n, my_todo - base));
        const int cnt = compact_hits(smask, nw, want, slist[t >> 5]);
        for (int kk = 0; kk < cnt; ++kk) {
            const int j = (int)slist[t >> 5][kk];
            const FeatRec<G> &rec = srec[j];
            float4 q0;                                   // {x, y, A', C'}
            unpk((f32x2)rec.w0.x, q0.x, q0.y);
            unpk((f32x2)rec.w0.y, q0.z, q0.w);
            const float op = rec.op;
            const uint32_t pos = (uint32_t)(base + j + 1);
            // render_bwd_kernel's exponent and acceptance, operation for operation
            const f32x2 dx2 = pk(q0.x - fx0, q0.x - (fx0 + 1.0f));
            const f32x2 Axx2 = mul2(mul2(pk1(q0.z), dx2), dx2);
            const f32x2 Bx2 = mul2(pk1(rec.bp), dx2);
            float dy[2], Cyy[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                dy[r] = q0.y - (fy0 + (float)r);
                Cyy[r] = __fmul_rn(__fmul_rn(q0.w, dy[r]), dy[r]);
            }
            float Gs[4], al[4];
            bool valid[4];
            bool any = false;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const f32x2 p2 = fma2(Bx2, pk1(dy[r]), add2(Axx2, pk1(Cyy[r])));
                float p[2];
                unpk(p2, p[0], p[1]);
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int i = 2 * r + c;
                    Gs[i] = ex2_approx(p[c]);
                    al[i] = fminf(ALPHA_MAX, __fmul_rn(op, Gs[i]));
                    valid[i] = (p[c] <= 0.0f) && (al[i] >= ALPHA_MIN) && (pos <= last[i]);
                    any = any || valid[i];
                }
            }
            if (!__any_sync(0xffffffffu, any)) continue;
            float fv[G];
            load_feats<G>(rec, fv);
            f32x2 m_x = pk1(0.f), m_y = m_x, m_xx = m_x, m_xy = m_x, m_yy = m_x, g_o = m_x, gf[G];
            const f32x2 op2 = pk1(op);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int i0 = 2 * r, i1 = 2 * r + 1;
                // invalid lanes: alpha = 0 and G = 0 make every contribution below exactly zero
                const f32x2 ai = pk(valid[i0] ? al[i0] : 0.0f, valid[i1] ? al[i1] : 0.0f);
                const f32x2 Gm = pk(valid[i0] ? Gs[i0] : 0.0f, valid[i1] ? Gs[i1] : 0.0f);
                const f32x2 w = mul2(ai, T[r]);
                f32x2 g = mul2(dL[0][r], pk1(fv[0]));
#pragma unroll
                for (int ch = 1; ch < G; ++ch) g = fma2(dL[ch][r], pk1(fv[ch]), g);
                F[r] = fma2(w, g, F[r]);
#pragma unroll
                for (int ch = 0; ch < G; ++ch) gf[ch] = r == 0 ? mul2(w, dL[ch][r]) : fma2(w, dL[ch][r], gf[ch]);
                const f32x2 om = sub2(one2, ai);
                float om0, om1;
                unpk(om, om0, om1);
                const f32x2 rcp = pk(rcp_approx(om0), rcp_approx(om1));
                const f32x2 dLda = sub2(mul2(T[r], g), mul2(sub2(S[r], F[r]), rcp));
                T[r] = mul2(T[r], om);
                const f32x2 Gd = mul2(Gm, dLda);
                const f32x2 tt = mul2(op2, Gd);
                const f32x2 dy2 = pk1(dy[r]);
                const f32x2 u = mul2(tt, dx2), vv = mul2(tt, dy2);
                if (r == 0) {
                    g_o = Gd; m_x = u; m_y = vv;
                    m_xx = mul2(u, dx2); m_xy = mul2(u, dy2); m_yy = mul2(vv, dy2);
                } else {
                    g_o = add2(g_o, Gd); m_x = add2(m_x, u); m_y = add2(m_y, vv);
                    m_xx = fma2(u, dx2, m_xx); m_xy = fma2(u, dy2, m_xy); m_yy = fma2(vv, dy2, m_yy);
                }
            }
            const float ra = reduce8_transposed(hsum(m_x), hsum(m_y), hsum(m_xx), hsum(m_xy), hsum(m_yy), hsum(g_o), hsum(gf[0]),
                                                hsum(gf[1]));
            float rb;
            if constexpr (G == 8)
                rb = reduce8_transposed(hsum(gf[2]), hsum(gf[3]), hsum(gf[4]), hsum(gf[5]), hsum(gf[6]), hsum(gf[7]), 0.f, 0.f);
            else
                rb = reduce2_transposed(hsum(gf[2]), hsum(gf[3]));
            float *dst = fch >= 0 ? a.dL_dfeatures + (size_t)rec.id * a.C + (c0 + fch) : a.dacc + (row0 + rec.id) * DACC_STRIDE + acc_k;
            red_add_pred(dst, red_on, from_rb ? rb : ra);
        }
    }
}

static int check_feat_launch(const char *what, const FeatArgs &a, const int tiles) {
    if (a.V < 1 || a.V > GSB_MAX_VIEWS || a.C < 1 || a.C > FEAT_MAX_CHANNELS || tiles > 0x7fffffff / GSB_MAX_VIEWS) {
        set_error("%s: bad launch geometry (V=%d, C=%d, tiles=%d)", what, a.V, a.C, tiles);
        return GSB_ERR_ARGUMENT;
    }
    return GSB_OK;
}

int launch_render_features(const FeatArgs &a, bool debug, cudaStream_t stream) {
    const int tiles = a.gx * a.gy;
    if (tiles <= 0) return GSB_OK;
    int rc = check_feat_launch("render_features", a, tiles);
    if (rc) return rc;
    if (a.C <= 4) {
        GSB_LAUNCH("render_features", debug, stream, render_features_kernel<4>, dim3(tiles, a.V, 1), 256, 0, a);
    } else {
        GSB_LAUNCH("render_features", debug, stream, render_features_kernel<8>, dim3(tiles, a.V, (a.C + 7) / 8), 256, 0, a);
    }
    return GSB_OK;
}

int launch_render_features_bwd(const FeatArgs &a, bool debug, cudaStream_t stream) {
    const int tiles = a.gx * a.gy;
    if (tiles <= 0) return GSB_OK;
    int rc = check_feat_launch("render_features_bwd", a, tiles);
    if (rc) return rc;
    if (a.C <= 4) {
        GSB_LAUNCH("render_features_bwd", debug, stream, (render_features_bwd_kernel<4, FEAT_BWD_MINB4>), dim3(tiles, a.V, 1), 64, 0, a);
    } else {
        GSB_LAUNCH("render_features_bwd", debug, stream, (render_features_bwd_kernel<8, FEAT_BWD_MINB8>), dim3(tiles, a.V, (a.C + 7) / 8),
                   64, 0, a);
    }
    return GSB_OK;
}

}  // namespace gsb
