// preprocess.cu -- per-gaussian kernels: forward projection (K1), backward chain rule (K8) and the
// frustum-only visibility test (K9).  One thread per gaussian, 256-thread blocks.
//
// Replaces preprocessCUDA / BACKWARD::preprocessCUDA / checkFrustum of the reference's
// cuda_rasterizer/{forward,backward,auxiliary}.* (named in BASELINE.json north_star; the files are
// absent from /root/reference, SURVEY.md section 0).  The cited in-tree formulae:
//   SH -> RGB ........ /root/reference/utils/sh_utils.py:57-112, gaussian_renderer/__init__.py:76-80
//   Sigma = L L^T .... /root/reference/utils/general_utils.py:78-110, scene/gaussian_model.py:33-37
//   matrices ......... /root/reference/scene/cameras.py:86-89 (transposed, row-vector convention)
#include "geom.cuh"
#include "kernels.cuh"

namespace gsb {

constexpr int PRE_THREADS = 128;

// SH rows ([3*M] floats per gaussian, 192 B at degree 3) dominate this kernel's traffic.  A thread-per-gaussian
// access would touch 32 different 128-byte lines per warp instruction, so the block's rows are moved between
// global and shared memory with fully coalesced accesses and each thread works on its own row in shared memory
// (row stride padded to an odd word count: conflict-free).
__host__ __device__ __forceinline__ int sh_row_stride(const int n) { return n | 1; }

// Second layout (VEC, option pre_tma): rows 16-byte aligned at a stride of an ODD number of 16-byte units.  A row is then one TMA
// bulk copy (cp.async.bulk, 192 B at SH degree 3) in either direction -- no load / store / index instruction at all -- and its
// owner reads and writes it as float4: the 8 rows of a quarter warp fall into 8 different 16-byte bank groups (conflict-free).
__host__ __device__ __forceinline__ int sh_row_stride_vec(const int n) { return 4 * (((n + 3) >> 2) | 1); }
template <bool VEC>
__device__ __forceinline__ int sh_stride(const int n) { return VEC ? sh_row_stride_vec(n) : sh_row_stride(n); }

// element e of a row <-> coefficient k = e / 3, channel c = e % 3; every index below is a compile-time constant after unrolling
#define GSB_SH_QUADS(m, nfloats, q, ...)                                                       \
    _Pragma("unroll") for (int m = 0; m < 12; ++m) {                                           \
        if (4 * m < (nfloats)) {                                                               \
            float4 _v = (q)[m];                                                                \
            float vv[4] = {_v.x, _v.y, _v.z, _v.w};                                            \
            __VA_ARGS__                                                                        \
        }                                                                                      \
    }

// rgb += sum_{k < nb} bas[k] * row[3k + c]
template <bool VEC>
__device__ __forceinline__ void sh_eval(const float *row, const float (&bas)[16], const int nb, float &r, float &g, float &b) {
    if (VEC) {
        const float4 *q = reinterpret_cast<const float4 *>(row);
        float acc[3] = {r, g, b};
        GSB_SH_QUADS(m, 3 * nb, q,
                     _Pragma("unroll") for (int i = 0; i < 4; ++i) {
                         const int e = 4 * m + i, k = e / 3, c = e % 3;
                         if (k < nb) acc[c] += bas[k] * vv[i];
                     })
        r = acc[0]; g = acc[1]; b = acc[2];
    } else {
#pragma unroll
        for (int k = 0; k < 16; ++k) {   // compile-time bound: bas[] stays in registers
            if (k < nb) { r += bas[k] * row[3 * k]; g += bas[k] * row[3 * k + 1]; b += bas[k] * row[3 * k + 2]; }
        }
    }
}

// dd{x,y,z} += sum_{1 <= k < nb} b{x,y,z}[k] * (row[3k] d0 + row[3k+1] d1 + row[3k+2] d2)
template <bool VEC>
__device__ __forceinline__ void sh_dir_grad(const float *row, const float (&d)[3], const float (&bx)[16], const float (&by)[16],
                                            const float (&bz)[16], const int nb, float &ddx, float &ddy, float &ddz) {
    if (VEC) {
        const float4 *q = reinterpret_cast<const float4 *>(row);
        float sk[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) sk[k] = 0.f;
        GSB_SH_QUADS(m, 3 * nb, q,
                     _Pragma("unroll") for (int i = 0; i < 4; ++i) {
                         const int e = 4 * m + i, k = e / 3, c = e % 3;
                         if (k >= 1 && k < nb) sk[k] = c == 0 ? vv[i] * d[0] : sk[k] + vv[i] * d[c];
                     })
#pragma unroll
        for (int k = 1; k < 16; ++k)
            if (k < nb) { ddx += bx[k] * sk[k]; ddy += by[k] * sk[k]; ddz += bz[k] * sk[k]; }
    } else {
#pragma unroll
        for (int k = 1; k < 16; ++k) {   // compile-time bound: bx/by/bz stay in registers
            if (k < nb) {
                const float s = row[3 * k] * d[0] + row[3 * k + 1] * d[1] + row[3 * k + 2] * d[2];
                ddx += bx[k] * s; ddy += by[k] * s; ddz += bz[k] * s;
            }
        }
    }
}

// gradient row: row[3k + c] (+)= bas[k] d[c] for k < nb; with ADD = false the rest of the row (k >= nb, up to M) is zeroed
template <bool VEC, bool ADD>
__device__ __forceinline__ void sh_grad_row(float *row, const float (&bas)[16], const float (&d)[3], const int nb, const int M) {
    if (VEC) {
        float4 *q = reinterpret_cast<float4 *>(row);
        GSB_SH_QUADS(m, ADD ? 3 * nb : 3 * M, q,
                     _Pragma("unroll") for (int i = 0; i < 4; ++i) {
                         const int e = 4 * m + i, k = e / 3, c = e % 3;
                         const float t = k < nb ? bas[k] * d[c] : 0.f;
                         vv[i] = ADD ? vv[i] + t : t;
                     }
                     q[m] = make_float4(vv[0], vv[1], vv[2], vv[3]);)
    } else {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            if (ADD) {
                if (k < nb) { row[3 * k] += bas[k] * d[0]; row[3 * k + 1] += bas[k] * d[1]; row[3 * k + 2] += bas[k] * d[2]; }
            } else if (k < M) {
                const float bk = k < nb ? bas[k] : 0.f;
                row[3 * k] = bk * d[0]; row[3 * k + 1] = bk * d[1]; row[3 * k + 2] = bk * d[2];
            }
        }
        if (!ADD)
            for (int k = 16; k < M; ++k) { row[3 * k] = 0.f; row[3 * k + 1] = 0.f; row[3 * k + 2] = 0.f; }
    }
}

// TMA staging of the block's SH rows: one bulk copy per row, issued by the row's owner, completing on one mbarrier
__device__ __forceinline__ void tma_rows_in(const float *__restrict__ g, float *s, unsigned long long *bar, const int row0,
                                            const int nrows, const int n) {
    if (threadIdx.x == 0) mbar_init(bar, 1);
    __syncthreads();
    if (threadIdx.x == 0) mbar_expect_tx(bar, (uint32_t)(nrows * n) * 4u);
    if ((int)threadIdx.x < nrows)
        bulk_g2s(s + threadIdx.x * sh_row_stride_vec(n), g + (size_t)(row0 + threadIdx.x) * n, (uint32_t)n * 4u, bar);
    mbar_wait(bar, 0u);
}

// the owner's (gradient) row back to global memory: bulk store, or bulk reduce-add (ACC)
template <bool ACC>
__device__ __forceinline__ void tma_row_out(float *__restrict__ g, const float *row, const int i, const int n, const bool live) {
    bulk_store_fence();
    if (live) {
        if (ACC) bulk_s2g_add_f32(g + (size_t)i * n, row, (uint32_t)n * 4u);
        else bulk_s2g(g + (size_t)i * n, row, (uint32_t)n * 4u);
    }
    bulk_store_commit_and_wait();
}

// global -> shared: first `ncols` floats of each of the block's rows (row length n).  When both n and ncols
// are multiples of four (SH degree 1 and 3 rows: 12 and 48 floats) the block's rows are fetched as 128-bit loads (a quarter of the load instructions and of the index
// arithmetic; the row stride in shared memory stays odd, so the four words are stored one by one); otherwise word by word.
__device__ __forceinline__ void stage_rows_in(const float *__restrict__ g, float *s, const int row0, const int nrows,
                                              const int n, const int ncols) {
    const int stride = sh_row_stride(n);
    const float *gb = g + (size_t)row0 * n;
    if (((n | ncols) & 3) == 0 && ((reinterpret_cast<size_t>(gb) & 15) == 0)) {
        const int q = ncols >> 2, total = nrows * q;        // float4 per row, float4 in the block
        const float inv = 1.0f / (float)q;
        for (int base = 0; base < total; base += 4 * PRE_THREADS) {
            float4 v[4];
            int si[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int idx = base + u * PRE_THREADS + threadIdx.x;
                si[u] = -1;
                if (idx < total) {
                    const int r = (int)(((float)idx + 0.5f) * inv), c = idx - r * q;
                    si[u] = r * stride + 4 * c;
                    v[u] = __ldg(reinterpret_cast<const float4 *>(gb + (size_t)r * n) + c);
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (si[u] >= 0) { s[si[u]] = v[u].x; s[si[u] + 1] = v[u].y; s[si[u] + 2] = v[u].z; s[si[u] + 3] = v[u].w; }
        }
        return;
    }
    const int total = nrows * ncols;
    const float inv = 1.0f / (float)ncols;
    for (int base = 0; base < total; base += 4 * PRE_THREADS) {
        float v[4];
        int si[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int idx = base + u * PRE_THREADS + threadIdx.x;
            si[u] = -1;
            if (idx < total) {
                const int r = (int)(((float)idx + 0.5f) * inv), c = idx - r * ncols;
                si[u] = r * stride + c;
                v[u] = __ldg(gb + (size_t)r * n + c);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (si[u] >= 0) s[si[u]] = v[u];
    }
}

// shared -> global: full rows (contiguous in global memory); ACC adds into the destination.  128-bit stores (and loads, for
// ACC) when the row length is a multiple of four floats.
template <bool ACC>
__device__ __forceinline__ void stage_rows_out(float *__restrict__ g, const float *s, const int row0, const int nrows,
                                               const int n) {
    const int stride = sh_row_stride(n);
    float *gb = g + (size_t)row0 * n;
    if ((n & 3) == 0 && ((reinterpret_cast<size_t>(gb) & 15) == 0)) {
        const int q = n >> 2, total = nrows * q;
        const float inv = 1.0f / (float)q;
        float4 *gb4 = reinterpret_cast<float4 *>(gb);
        for (int base = 0; base < total; base += 4 * PRE_THREADS) {
            float4 v[4];
            int gi[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int idx = base + u * PRE_THREADS + threadIdx.x;
                gi[u] = -1;
                if (idx < total) {
                    const int r = (int)(((float)idx + 0.5f) * inv), c = idx - r * q;
                    const float *sp = s + r * stride + 4 * c;
                    gi[u] = idx;
                    v[u] = make_float4(sp[0], sp[1], sp[2], sp[3]);
                    if (ACC) { const float4 o = gb4[idx]; v[u].x += o.x; v[u].y += o.y; v[u].z += o.z; v[u].w += o.w; }
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (gi[u] >= 0) gb4[gi[u]] = v[u];
        }
        return;
    }
    const int total = nrows * n;
    const float inv = 1.0f / (float)n;
    for (int base = 0; base < total; base += 4 * PRE_THREADS) {
        float v[4];
        int gi[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int idx = base + u * PRE_THREADS + threadIdx.x;
            gi[u] = -1;
            if (idx < total) {
                const int r = (int)(((float)idx + 0.5f) * inv), c = idx - r * n;
                gi[u] = idx;
                v[u] = s[r * stride + c];
                if (ACC) v[u] += gb[idx];
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (gi[u] >= 0) gb[gi[u]] = v[u];
    }
}

// ---- third staging source: split SH input (DC rows [P,1,3] and rest rows [P,M-1,3] in two tensors) ----------------------------
// Each source's span for the block ([nrows, n] floats) is contiguous in global memory and is moved with word accesses,
// consecutive threads on consecutive words (coalesced), into / out of columns [col0, col0 + ncols) of the joint rows that
// stage_rows_in lays out in shared memory (odd word stride).  Everything after staging is the joint path's code.
__device__ __forceinline__ void stage_span_in(const float *__restrict__ g, float *s, const int row0, const int nrows, const int n,
                                              const int ncols, const int stride, const int col0) {
    if (ncols <= 0) return;
    const float *gb = g + (size_t)row0 * n;
    const int total = nrows * ncols;
    const float inv = 1.0f / (float)ncols;
    for (int base = 0; base < total; base += 4 * PRE_THREADS) {
        float v[4];
        int si[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int idx = base + u * PRE_THREADS + threadIdx.x;
            si[u] = -1;
            if (idx < total) {
                const int r = (int)(((float)idx + 0.5f) * inv), c = idx - r * ncols;
                si[u] = r * stride + col0 + c;
                v[u] = __ldg(gb + (size_t)r * n + c);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (si[u] >= 0) s[si[u]] = v[u];
    }
}

template <bool ACC>
__device__ __forceinline__ void stage_span_out(float *__restrict__ g, const float *s, const int row0, const int nrows, const int n,
                                               const int stride, const int col0) {
    if (!g || n <= 0) return;
    float *gb = g + (size_t)row0 * n;
    const int total = nrows * n;
    const float inv = 1.0f / (float)n;
    for (int base = 0; base < total; base += 4 * PRE_THREADS) {
        float v[4];
        int gi[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int idx = base + u * PRE_THREADS + threadIdx.x;
            gi[u] = -1;
            if (idx < total) {
                const int r = (int)(((float)idx + 0.5f) * inv), c = idx - r * n;
                gi[u] = idx;
                v[u] = s[r * stride + col0 + c];
                if (ACC) v[u] += gb[idx];
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (gi[u] >= 0) gb[gi[u]] = v[u];
    }
}

// first `ncols` floats of the block's joint rows (row length n = 3M) from the two split tensors (rest may be NULL: M == 1)
__device__ __forceinline__ void stage_split_rows_in(const float *__restrict__ dc, const float *__restrict__ rest, float *s, const int row0,
                                                    const int nrows, const int n, const int ncols) {
    const int stride = sh_row_stride(n);
    stage_span_in(dc, s, row0, nrows, 3, min(ncols, 3), stride, 0);
    if (rest) stage_span_in(rest, s, row0, nrows, n - 3, ncols - 3, stride, 3);
}

// full joint (gradient) rows back to the two split tensors; a NULL destination is skipped
template <bool ACC>
__device__ __forceinline__ void stage_split_rows_out(float *__restrict__ ddc, float *__restrict__ drest, const float *s, const int row0,
                                                     const int nrows, const int n) {
    const int stride = sh_row_stride(n);
    stage_span_out<ACC>(ddc, s, row0, nrows, 3, stride, 0);
    stage_span_out<ACC>(drest, s, row0, nrows, n - 3, stride, 3);
}

// one gaussian, one view: everything of K1 after the SH row has been staged
template <bool VEC>
__device__ __forceinline__ void preprocess_fwd_body(const CamParams &cam, const PreFwdArgs &a, const int i, const float *sh_row) {
    // defaults for a culled gaussian
    uint32_t key = 0xffffffffu, ntiles = 0;
    int radius_out = 0;
    float4 q0 = make_float4(0.f, 0.f, 0.f, 0.f), q1 = q0, q2 = q0;
    uint2 rect = make_uint2(0u, 0u);
    bool write_all = false;

    const float px = a.means[3 * i], py = a.means[3 * i + 1], pz = a.means[3 * i + 2];
    const float *v = cam.view, *pm = cam.proj;
    const float tz = v[2] * px + v[6] * py + v[10] * pz + v[14];
    if (tz > NEAR_CULL) {
        const float hx = pm[0] * px + pm[4] * py + pm[8] * pz + pm[12];
        const float hy = pm[1] * px + pm[5] * py + pm[9] * pz + pm[13];
        const float hw = pm[3] * px + pm[7] * py + pm[11] * pz + pm[15];
        const float pw = 1.0f / (hw + W_EPS);
        const float ndcx = hx * pw, ndcy = hy * pw;

        float c6[6];
        if (a.cov_pre) {
#pragma unroll
            for (int k = 0; k < 6; ++k) c6[k] = a.cov_pre[6 * (size_t)i + k];
        } else {
            const float4 q = reinterpret_cast<const float4 *>(a.rots)[i];
            cov3d_from_scale_rot(a.scales[3 * i], a.scales[3 * i + 1], a.scales[3 * i + 2], cam.scale_modifier, q, c6);
        }
        Cov2D cv;
        cov2d(cam, px, py, pz, c6, cv);
        const float det0 = cv.a * cv.c - cv.b * cv.b;
        const float ca_ = cv.a + DILATION, cc_ = cv.c + DILATION, cb_ = cv.b;
        const float det = ca_ * cc_ - cb_ * cb_;
        float hscale = 1.0f;
        if (cam.antialiasing) hscale = sqrtf(fmaxf(AA_FLOOR, det0 / det));
        if (det != 0.0f) {
            const float det_inv = 1.0f / det;
            const float mid = 0.5f * (ca_ + cc_);
            const float root = sqrtf(fmaxf(0.1f, mid * mid - det));
            const float lam = fmaxf(mid + root, mid - root);
            const float radius = ceilf(3.0f * sqrtf(lam));
            const float sx = ((ndcx + 1.0f) * cam.W - 1.0f) * 0.5f;
            const float sy = ((ndcy + 1.0f) * cam.H - 1.0f) * 0.5f;
            int x0 = (int)((sx - radius) / TILE), y0 = (int)((sy - radius) / TILE);
            int x1 = (int)((sx + radius + TILE - 1) / TILE), y1 = (int)((sy + radius + TILE - 1) / TILE);
            x0 = min(cam.gx, max(0, x0)); x1 = min(cam.gx, max(0, x1));
            y0 = min(cam.gy, max(0, y0)); y1 = min(cam.gy, max(0, y1));
            if ((x1 - x0) * (y1 - y0) != 0) {
                float r = 0.f, g = 0.f, b = 0.f;
                uint32_t bits = 8u;  // bit 3: visible
                if (a.colors) {
                    r = a.colors[3 * (size_t)i]; g = a.colors[3 * (size_t)i + 1]; b = a.colors[3 * (size_t)i + 2];
                } else {
                    const float dx = px - cam.campos[0], dy = py - cam.campos[1], dz = pz - cam.campos[2];
                    const float inv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
                    float bas[16];
                    sh_basis(cam.sh_degree, dx * inv, dy * inv, dz * inv, bas);
                    const int nb = (cam.sh_degree + 1) * (cam.sh_degree + 1);
                    sh_eval<VEC>(sh_row, bas, nb, r, g, b);
                    r += 0.5f; g += 0.5f; b += 0.5f;
                    if (r < 0.f) { bits |= 1u; r = 0.f; }
                    if (g < 0.f) { bits |= 2u; g = 0.f; }
                    if (b < 0.f) { bits |= 4u; b = 0.f; }
                }
                const float opacity = a.opac[i] * hscale;
                const float A = cc_ * det_inv, B = -cb_ * det_inv, C = ca_ * det_inv;
                CullGeom cg;
                cg.cx = sx; cg.cy = sy; cg.A = A; cg.B = B; cg.C = C;
                cg.rx0 = x0; cg.ry0 = y0; cg.rx1 = x1; cg.ry1 = y1;
                if (a.cull) {
                    cg.lim = cull_limit(opacity);
                    ntiles = cull_count(cg);
                } else {
                    cg.lim = 3.0e38f;
                    ntiles = (uint32_t)((x1 - x0) * (y1 - y0));
                }
                q0 = make_float4(sx, sy, A, B);
                q1 = make_float4(C, opacity, r, g);
                q2 = make_float4(b, 1.0f / tz, cg.lim, __uint_as_float(bits));
                rect = make_uint2((uint32_t)x0 | ((uint32_t)x1 << 16), (uint32_t)y0 | ((uint32_t)y1 << 16));
                key = __float_as_uint(tz);
                radius_out = (int)radius;
                write_all = true;
            }
        }
    }
    float4 *rec = a.splat + (size_t)i * SPLAT_F4;
    if (write_all) { rec[0] = q0; rec[1] = q1; }
    rec[2] = q2;
    a.depth_key[i] = key;
    a.depth_idx[i] = (uint32_t)i;
    a.tiles[i] = ntiles;
    a.rect[i] = rect;
    a.radii[i] = radius_out;
}

// SPLIT: split SH input (a.shs = DC rows, a.rest = the other coefficients), staged into the scalar row layout (TMA false)
template <bool TMA, bool SPLIT = false>
__global__ void __launch_bounds__(PRE_THREADS)
preprocess_fwd_kernel(const CamArgs ca, const PreFwdArgs a) {
    __shared__ CamParams cam;
    __shared__ unsigned long long bar;
    GSB_DYNAMIC_SMEM(float4, sh_rows4);
    float *sh_rows = reinterpret_cast<float *>(sh_rows4);
    load_cam(ca, cam);
    const int row0 = blockIdx.x * PRE_THREADS;
    const int nrows = min(PRE_THREADS, a.P - row0);
    const int shn = 3 * ca.sh_coeffs;
    if (a.shs) {
        if (SPLIT) stage_split_rows_in(a.shs, a.rest, sh_rows, row0, nrows, shn, 3 * (ca.sh_degree + 1) * (ca.sh_degree + 1));
        else if (TMA) tma_rows_in(a.shs, sh_rows, &bar, row0, nrows, shn);
        else stage_rows_in(a.shs, sh_rows, row0, nrows, shn, 3 * (ca.sh_degree + 1) * (ca.sh_degree + 1));
    }
    __syncthreads();
    const int i = row0 + threadIdx.x;
    if (i >= a.P) return;
    preprocess_fwd_body<TMA>(cam, a, i, sh_rows + threadIdx.x * sh_stride<TMA>(shn));
}

// View-batch K1: the gaussians' parameters (236 B each at SH degree 3, 192 B of it the SH row) are read ONCE and
// projected through every camera of the batch; per-view outputs are [V][...] arrays with uniform strides.
template <bool TMA>
__global__ void __launch_bounds__(PRE_THREADS)
preprocess_fwd_batch_kernel(const CamArgsBatch cb, const PreFwdArgs a, const PreFwdBatchStrides st) {
    __shared__ CamParams cams[GSB_MAX_VIEWS];
    __shared__ unsigned long long bar;
    GSB_DYNAMIC_SMEM(float4, sh_rows4);
    float *sh_rows = reinterpret_cast<float *>(sh_rows4);
    for (int v = 0; v < cb.V; ++v) load_cam(cb.cam[v], cams[v]);
    const int row0 = blockIdx.x * PRE_THREADS;
    const int nrows = min(PRE_THREADS, a.P - row0);
    const int shn = 3 * cb.cam[0].sh_coeffs;
    if (a.shs) {
        if (TMA) tma_rows_in(a.shs, sh_rows, &bar, row0, nrows, shn);
        else stage_rows_in(a.shs, sh_rows, row0, nrows, shn, 3 * (cb.cam[0].sh_degree + 1) * (cb.cam[0].sh_degree + 1));
    }
    __syncthreads();
    const int i = row0 + threadIdx.x;
    if (i >= a.P) return;
    for (int v = 0; v < cb.V; ++v) {
        PreFwdArgs av = a;
        av.splat += (size_t)v * st.splat; av.depth_key += (size_t)v * st.per_gauss; av.depth_idx += (size_t)v * st.per_gauss;
        av.tiles += (size_t)v * st.per_gauss; av.rect += (size_t)v * st.per_gauss; av.radii += (size_t)v * st.radii;
        preprocess_fwd_body<TMA>(cams[v], av, i, sh_rows + threadIdx.x * sh_stride<TMA>(shn));
    }
}

// d basis / d(x,y,z)
__device__ __forceinline__ void sh_basis_grad(const int deg, const float x, const float y, const float z, float bx[16],
                                              float by[16], float bz[16]) {
#pragma unroll
    for (int k = 0; k < 16; ++k) bx[k] = by[k] = bz[k] = 0.0f;
    if (deg < 1) return;
    by[1] = -SH_C1; bz[2] = SH_C1; bx[3] = -SH_C1;
    if (deg < 2) return;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    bx[4] = SH_C2[0] * y; by[4] = SH_C2[0] * x;
    by[5] = SH_C2[1] * z; bz[5] = SH_C2[1] * y;
    bx[6] = SH_C2[2] * -2.0f * x; by[6] = SH_C2[2] * -2.0f * y; bz[6] = SH_C2[2] * 4.0f * z;
    bx[7] = SH_C2[3] * z; bz[7] = SH_C2[3] * x;
    bx[8] = SH_C2[4] * 2.0f * x; by[8] = SH_C2[4] * -2.0f * y;
    if (deg < 3) return;
    bx[9] = SH_C3[0] * 6.0f * xy; by[9] = SH_C3[0] * (3.0f * xx - 3.0f * yy);
    bx[10] = SH_C3[1] * yz; by[10] = SH_C3[1] * xz; bz[10] = SH_C3[1] * xy;
    bx[11] = SH_C3[2] * -2.0f * xy; by[11] = SH_C3[2] * (4.0f * zz - xx - 3.0f * yy); bz[11] = SH_C3[2] * 8.0f * yz;
    bx[12] = SH_C3[3] * -6.0f * xz; by[12] = SH_C3[3] * -6.0f * yz;
    bz[12] = SH_C3[3] * (6.0f * zz - 3.0f * xx - 3.0f * yy);
    bx[13] = SH_C3[4] * (4.0f * zz - 3.0f * xx - yy); by[13] = SH_C3[4] * -2.0f * xy; bz[13] = SH_C3[4] * 8.0f * xz;
    bx[14] = SH_C3[5] * 2.0f * xz; by[14] = SH_C3[5] * -2.0f * yz; bz[14] = SH_C3[5] * (xx - yy);
    bx[15] = SH_C3[6] * (3.0f * xx - 3.0f * yy); by[15] = SH_C3[6] * -6.0f * xy;
}

template <bool ACC>
__device__ __forceinline__ void put(float *p, const float v) {
    if (ACC) *p += v; else *p = v;
}

// gradient of one gaussian through one view
struct ViewGrad {
    float gm[3], g_m2[2], g_op, g_rgb[3], g_sc[3], g_rot[4], dS[6], d_rgb_sh[3], bas[16];
};

// One gaussian's contribution to the camera gradient (CAMGRAD instantiations), x~ = [x, y, z, 1]:
//   t[3r + c]       dL/dV[r][c],  r < 4, c < 3   (column 3 of the viewmatrix is never read: its gradient is 0)
//   t[12 + 3r + k]  dL/dPM[r][c], r < 4, c = 0, 1, 3 for k = 0, 1, 2   (column 2 is never read)
//   t[24 + c]       dL/dcampos[c]
struct CamGrad {
    float t[CAM_TERMS];
};

__device__ __forceinline__ void cam_zero(CamGrad &cg) {
#pragma unroll
    for (int k = 0; k < CAM_TERMS; ++k) cg.t[k] = 0.f;
}

// Warp sum of the 27 terms (xor butterfly: a fixed order, every lane ends with the sum); lane 0 writes the warp's partial to
// column `slot` of the [CAM_TERMS][nslots] panel.  Every lane of the warp must call this.
__device__ __forceinline__ void cam_warp_partial(CamGrad &cg, float *panel, const int nslots, const int slot) {
#pragma unroll
    for (int k = 0; k < CAM_TERMS; ++k) {
        float s = cg.t[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        cg.t[k] = s;
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < CAM_TERMS; ++k) panel[(size_t)k * nslots + slot] = cg.t[k];
    }
}

// K8 for one gaussian and one view: chain rule from the blend kernel's accumulators (mean2D / conic or raw moments, opacity,
// rgb, inverse depth) to the rasterizer inputs.  Every field of `o` is written.
// Returns false when the gaussian received no gradient in this view (all fields of `o` are zero then).
// CAMGRAD: `*cg` receives the gaussian's camera gradient terms (all zero when it returns false).
template <bool VEC, bool CAMGRAD = false>
__device__ __forceinline__ bool preprocess_bwd_view(const CamParams &cam, const PreBwdArgs &a, const int i, const float *sh_row,
                                                    const uint32_t bits, ViewGrad &o, CamGrad *cg = nullptr) {
    if (CAMGRAD) cam_zero(*cg);
    float (&gm)[3] = o.gm; float (&g_m2)[2] = o.g_m2; float &g_op = o.g_op; float (&g_rgb)[3] = o.g_rgb;
    float (&g_sc)[3] = o.g_sc; float (&g_rot)[4] = o.g_rot; float (&dS)[6] = o.dS; float (&d_rgb_sh)[3] = o.d_rgb_sh;
    float (&bas)[16] = o.bas;
    gm[0] = gm[1] = gm[2] = 0.f; g_m2[0] = g_m2[1] = 0.f; g_op = 0.f; g_rgb[0] = g_rgb[1] = g_rgb[2] = 0.f;
    g_sc[0] = g_sc[1] = g_sc[2] = 0.f; g_rot[0] = g_rot[1] = g_rot[2] = g_rot[3] = 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) dS[k] = 0.f;
    d_rgb_sh[0] = d_rgb_sh[1] = d_rgb_sh[2] = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) bas[k] = 0.f;
    const bool visible = (bits & 8u) != 0u;
    const int nb = (cam.sh_degree + 1) * (cam.sh_degree + 1);
    const int M = cam.sh_coeffs;
    (void)M;

    if (visible) {
        const float4 *acc = reinterpret_cast<const float4 *>(a.dacc + (size_t)i * DACC_STRIDE);
        const float4 A0 = acc[0], A1 = acc[1], A2 = acc[2];
        // A gaussian no pixel blended in this view (occluded, or behind every pixel's stopping point) has an all-zero
        // accumulator row: every gradient below would be an exact zero, so the chain rule is skipped.
        if (A0.x == 0.f && A0.y == 0.f && A0.z == 0.f && A0.w == 0.f && A1.x == 0.f && A1.y == 0.f && A1.z == 0.f && A1.w == 0.f &&
            A2.x == 0.f && A2.y == 0.f)
            return false;
        // the accumulator holds raw moments of t = dL/d(power):  sum t dx, t dy, t dx^2, t dx dy, t dy^2   (render.cu)
        const float4 r0 = a.splat[(size_t)i * SPLAT_F4], r1 = a.splat[(size_t)i * SPLAT_F4 + 1];
        const float cA = r0.z, cB = r0.w, cC = r1.x;
        const float Mx = A0.x, My = A0.y, Mxx = A0.z, Mxy = A0.w, Myy = A1.x;
        const float d_m2x = (-cA * Mx - cB * My) * (0.5f * cam.W);
        const float d_m2y = (-cC * My - cB * Mx) * (0.5f * cam.H);
        const float dA = -0.5f * Mxx, dB = -Mxy, dC = -0.5f * Myy;
        const float d_w = A1.y;
        const float d_rgb[3] = {A1.z, A1.w, A2.x};
        const float d_invd = A2.y;
        g_m2[0] = d_m2x; g_m2[1] = d_m2y;
        const float px = a.means[3 * i], py = a.means[3 * i + 1], pz = a.means[3 * i + 2];

        // colour
        if (a.shs) {
            const float dx = px - cam.campos[0], dy = py - cam.campos[1], dz = pz - cam.campos[2];
            const float inv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
            const float ux = dx * inv, uy = dy * inv, uz = dz * inv;
            float bx[16], by[16], bz[16];
            sh_basis(cam.sh_degree, ux, uy, uz, bas);
            sh_basis_grad(cam.sh_degree, ux, uy, uz, bx, by, bz);
            d_rgb_sh[0] = (bits & 1u) ? 0.f : d_rgb[0];
            d_rgb_sh[1] = (bits & 2u) ? 0.f : d_rgb[1];
            d_rgb_sh[2] = (bits & 4u) ? 0.f : d_rgb[2];
            float ddx = 0.f, ddy = 0.f, ddz = 0.f;
            sh_dir_grad<VEC>(sh_row, d_rgb_sh, bx, by, bz, nb, ddx, ddy, ddz);
            const float dot = ux * ddx + uy * ddy + uz * ddz;
            gm[0] += (ddx - ux * dot) * inv; gm[1] += (ddy - uy * dot) * inv; gm[2] += (ddz - uz * dot) * inv;
            if (CAMGRAD) {   // the view direction is mean - campos: campos takes minus this part of dL/dmean
                cg->t[24] = -(ddx - ux * dot) * inv; cg->t[25] = -(ddy - uy * dot) * inv; cg->t[26] = -(ddz - uz * dot) * inv;
            }
        } else {
            g_rgb[0] = d_rgb[0]; g_rgb[1] = d_rgb[1]; g_rgb[2] = d_rgb[2];
        }

        // conic -> dilated 2D covariance
        float c6[6];
        float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
        float sc[3] = {0.f, 0.f, 0.f};
        if (a.cov_pre) {
#pragma unroll
            for (int k = 0; k < 6; ++k) c6[k] = a.cov_pre[6 * (size_t)i + k];
        } else {
            q = reinterpret_cast<const float4 *>(a.rots)[i];
            sc[0] = a.scales[3 * i]; sc[1] = a.scales[3 * i + 1]; sc[2] = a.scales[3 * i + 2];
            cov3d_from_scale_rot(sc[0], sc[1], sc[2], cam.scale_modifier, q, c6);
        }
        Cov2D cv;
        cov2d(cam, px, py, pz, c6, cv);
        const float a0 = cv.a, b = cv.b, c0 = cv.c;
        const float a_ = a0 + DILATION, c_ = c0 + DILATION;
        const float det = a_ * c_ - b * b;
        const float dinv2 = 1.0f / (det * det + 0.0000001f);
        float dL_da = dinv2 * (-c_ * c_ * dA + b * c_ * dB - b * b * dC);
        float dL_dc = dinv2 * (-b * b * dA + a_ * b * dB - a_ * a_ * dC);
        float dL_db = dinv2 * (2.f * b * c_ * dA - (det + 2.f * b * b) * dB + 2.f * a_ * b * dC);
        g_op = d_w;
        if (cam.antialiasing) {
            const float det0 = a0 * c0 - b * b;
            const float ratio = det0 / det;
            const float hs = sqrtf(fmaxf(AA_FLOOR, ratio));
            g_op = d_w * hs;
            if (ratio > AA_FLOOR) {
                const float d_ratio = d_w * a.opac[i] / (2.0f * hs);
                dL_da += d_ratio * (c0 / det - det0 * c_ / (det * det));
                dL_dc += d_ratio * (a0 / det - det0 * a_ / (det * det));
                dL_db += d_ratio * (-2.f * b / det + det0 * 2.f * b / (det * det));
            }
        }

        // 2D covariance -> Sigma and M = J R
        const float *M0 = cv.M0, *M1 = cv.M1;
        dS[0] = M0[0] * M0[0] * dL_da + M0[0] * M1[0] * dL_db + M1[0] * M1[0] * dL_dc;
        dS[3] = M0[1] * M0[1] * dL_da + M0[1] * M1[1] * dL_db + M1[1] * M1[1] * dL_dc;
        dS[5] = M0[2] * M0[2] * dL_da + M0[2] * M1[2] * dL_db + M1[2] * M1[2] * dL_dc;
        dS[1] = 2.f * M0[0] * M0[1] * dL_da + (M0[0] * M1[1] + M0[1] * M1[0]) * dL_db + 2.f * M1[0] * M1[1] * dL_dc;
        dS[2] = 2.f * M0[0] * M0[2] * dL_da + (M0[0] * M1[2] + M0[2] * M1[0]) * dL_db + 2.f * M1[0] * M1[2] * dL_dc;
        dS[4] = 2.f * M0[1] * M0[2] * dL_da + (M0[1] * M1[2] + M0[2] * M1[1]) * dL_db + 2.f * M1[1] * M1[2] * dL_dc;
        const float S0[3] = {c6[0], c6[1], c6[2]}, S1[3] = {c6[1], c6[3], c6[4]}, S2[3] = {c6[2], c6[4], c6[5]};
        const float SM0[3] = {S0[0] * M0[0] + S0[1] * M0[1] + S0[2] * M0[2], S1[0] * M0[0] + S1[1] * M0[1] + S1[2] * M0[2],
                              S2[0] * M0[0] + S2[1] * M0[1] + S2[2] * M0[2]};
        const float SM1[3] = {S0[0] * M1[0] + S0[1] * M1[1] + S0[2] * M1[2], S1[0] * M1[0] + S1[1] * M1[1] + S1[2] * M1[2],
                              S2[0] * M1[0] + S2[1] * M1[1] + S2[2] * M1[2]};
        float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
        float dMv0[3], dMv1[3];   // dL/dM (CAMGRAD only)
        const float *v = cam.view;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float dM0 = 2.f * dL_da * SM0[c] + dL_db * SM1[c];
            const float dM1 = 2.f * dL_dc * SM1[c] + dL_db * SM0[c];
            dJ00 += dM0 * v[4 * c + 0]; dJ02 += dM0 * v[4 * c + 2];
            dJ11 += dM1 * v[4 * c + 1]; dJ12 += dM1 * v[4 * c + 2];
            if (CAMGRAD) { dMv0[c] = dM0; dMv1[c] = dM1; }
        }
        const float tz = cv.tz, tz2 = 1.0f / (tz * tz), tz3 = tz2 / tz;
        const float fx = cam.focal_x, fy = cam.focal_y;
        const float dtx = cv.cx ? 0.0f : -fx * tz2 * dJ02;
        const float dty = cv.cy ? 0.0f : -fy * tz2 * dJ12;
        float dtz = -fx * tz2 * dJ00 - fy * tz2 * dJ11 + 2.f * fx * cv.tx * tz3 * dJ02 + 2.f * fy * cv.ty * tz3 * dJ12;
        dtz -= d_invd * tz2;
#pragma unroll
        for (int c = 0; c < 3; ++c) gm[c] += dtx * v[4 * c + 0] + dty * v[4 * c + 1] + dtz * v[4 * c + 2];
        const float xt[4] = {px, py, pz, 1.0f};
        if (CAMGRAD) {
            // p_view = x~ V: dL/dV[r][c] = x~_r dL/dp_view[c].  M = J Rw2c with Rw2c[k][c] = V[c][k] adds
            // dL/dV[c][k] += sum_i dL/dM[i][c] J[i][k] on the rotation block (J01 = J10 = 0, J's tx / ty are the clamped ones)
            const float J00 = fx / tz, J02 = -(fx * cv.tx) / (tz * tz), J11 = fy / tz, J12 = -(fy * cv.ty) / (tz * tz);
#pragma unroll
            for (int r = 0; r < 4; ++r) { cg->t[3 * r] = xt[r] * dtx; cg->t[3 * r + 1] = xt[r] * dty; cg->t[3 * r + 2] = xt[r] * dtz; }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                cg->t[3 * c] += dMv0[c] * J00;
                cg->t[3 * c + 1] += dMv1[c] * J11;
                cg->t[3 * c + 2] += dMv0[c] * J02 + dMv1[c] * J12;
            }
        }

        // NDC 2D mean -> 3D mean
        {
            const float *pm = cam.proj;
            const float hx = pm[0] * px + pm[4] * py + pm[8] * pz + pm[12];
            const float hy = pm[1] * px + pm[5] * py + pm[9] * pz + pm[13];
            const float hw = pm[3] * px + pm[7] * py + pm[11] * pz + pm[15];
            const float pw = 1.0f / (hw + W_EPS);
            const float mul1 = hx * pw * pw, mul2 = hy * pw * pw;
#pragma unroll
            for (int c = 0; c < 3; ++c)
                gm[c] += (pm[4 * c + 0] * pw - pm[4 * c + 3] * mul1) * d_m2x + (pm[4 * c + 1] * pw - pm[4 * c + 3] * mul2) * d_m2y;
            if (CAMGRAD) {
                // p_hom = x~ PM, ndc = p_hom.xy / (p_hom.w + eps): dL/dPM[r][c] = x~_r dL/dp_hom[c] for c = 0, 1, 3
                const float gx = pw * d_m2x, gy = pw * d_m2y, gw = -(mul1 * d_m2x + mul2 * d_m2y);
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    cg->t[12 + 3 * r] = xt[r] * gx; cg->t[12 + 3 * r + 1] = xt[r] * gy; cg->t[12 + 3 * r + 2] = xt[r] * gw;
                }
            }
        }

        // Sigma -> scale, rotation
        if (!a.cov_pre) {
            float R[9];
            quat_to_R(q, R);
            const float mod = cam.scale_modifier;
            const float sp[3] = {mod * sc[0], mod * sc[1], mod * sc[2]};
            const float Gm[9] = {dS[0], 0.5f * dS[1], 0.5f * dS[2], 0.5f * dS[1], dS[3], 0.5f * dS[4],
                                 0.5f * dS[2], 0.5f * dS[4], dS[5]};
            float dR[9];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                float ds = 0.f;
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const float dl = 2.f * (Gm[3 * r] * R[k] + Gm[3 * r + 1] * R[3 + k] + Gm[3 * r + 2] * R[6 + k]) * sp[k];
                    ds += dl * R[3 * r + k];
                    dR[3 * r + k] = dl * sp[k];
                }
                g_sc[k] = mod * ds;
            }
            const float r = q.x, x = q.y, y = q.z, z = q.w;
            g_rot[0] = 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
            g_rot[1] = 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - 2.f * x * dR[4] - r * dR[5] + z * dR[6] + r * dR[7] - 2.f * x * dR[8]);
            g_rot[2] = 2.f * (-2.f * y * dR[0] + x * dR[1] + r * dR[2] + x * dR[3] + z * dR[5] - r * dR[6] + z * dR[7] - 2.f * y * dR[8]);
            g_rot[3] = 2.f * (-2.f * z * dR[0] - r * dR[1] + x * dR[2] + r * dR[3] - 2.f * z * dR[4] + y * dR[5] + x * dR[6] + y * dR[7]);
        }
    }

    return visible;
}

template <bool ACC>
__device__ __forceinline__ void write_gauss_grads(const PreBwdArgs &a, const int i, const float gm[3], const float g_op,
                                                  const float g_rgb[3], const float g_sc[3], const float g_rot[4], const float dS[6]) {
    if (a.g.dL_dmeans3D) {
        put<ACC>(a.g.dL_dmeans3D + 3 * (size_t)i, gm[0]); put<ACC>(a.g.dL_dmeans3D + 3 * (size_t)i + 1, gm[1]);
        put<ACC>(a.g.dL_dmeans3D + 3 * (size_t)i + 2, gm[2]);
    }
    if (a.g.dL_dopacities) put<ACC>(a.g.dL_dopacities + i, g_op);
    if (a.g.dL_dcolors) {
#pragma unroll
        for (int c = 0; c < 3; ++c) put<ACC>(a.g.dL_dcolors + 3 * (size_t)i + c, g_rgb[c]);
    }
    if (a.cov_pre) {
        if (a.g.dL_dcov3D) {
#pragma unroll
            for (int k = 0; k < 6; ++k) put<ACC>(a.g.dL_dcov3D + 6 * (size_t)i + k, dS[k]);
        }
    } else {
        if (a.g.dL_dscales) {
#pragma unroll
            for (int k = 0; k < 3; ++k) put<ACC>(a.g.dL_dscales + 3 * (size_t)i + k, g_sc[k]);
        }
        if (a.g.dL_drotations) {
#pragma unroll
            for (int k = 0; k < 4; ++k) put<ACC>(a.g.dL_drotations + 4 * (size_t)i + k, g_rot[k]);
        }
    }
}

// ---- fused reduce-scatter: the block's gradients leave as bulk reduce-adds into the OWNER rank's memory ----------------------
__device__ __forceinline__ long long peer_delta(const PeerTable &t, const int row0) {
    const int owner = row0 / t.rows_per_rank;          // uniform per block: rows_per_rank is a multiple of PRE_THREADS
    long long d = t.delta[0];
#pragma unroll
    for (int k = 1; k < GSB_MAX_PEERS; ++k)
        if (k == owner) d = t.delta[k];
    return d;
}
template <typename T>
__device__ __forceinline__ T *shift_ptr(T *p, const long long bytes) {
    return reinterpret_cast<T *>(reinterpret_cast<char *>(p) + bytes);
}

// K8, one view.  SPLIT: split SH input and gradient (a.shs / a.g.dL_dshs = DC rows, a.rest / a.dL_drest = the rest; TMA false).
// CAMGRAD: every warp also writes its sum of the camera gradient terms to a.cam_part ([CAM_TERMS][4 * gridDim.x]).
template <bool ACC, bool TMA, bool SPLIT = false, bool CAMGRAD = false>
__global__ void __launch_bounds__(PRE_THREADS)
preprocess_bwd_kernel(const CamArgs ca, const PreBwdArgs a) {
    __shared__ CamParams cam;
    __shared__ unsigned long long bar;
    GSB_DYNAMIC_SMEM(float4, sh_rows4);
    float *sh_rows = reinterpret_cast<float *>(sh_rows4);
    load_cam(ca, cam);
    const int row0 = a.p_begin + blockIdx.x * PRE_THREADS;      // gaussians [p_begin, p_end) of this launch
    const int nrows = min(PRE_THREADS, a.p_end - row0);
    const int shn = 3 * ca.sh_coeffs;
    const int nb = (ca.sh_degree + 1) * (ca.sh_degree + 1);
    if (a.shs) {
        if (SPLIT) stage_split_rows_in(a.shs, a.rest, sh_rows, row0, nrows, shn, 3 * nb);
        else if (TMA) tma_rows_in(a.shs, sh_rows, &bar, row0, nrows, shn);
        else stage_rows_in(a.shs, sh_rows, row0, nrows, shn, 3 * nb);
    }
    __syncthreads();
    const int i = row0 + threadIdx.x;
    const bool live = i < a.p_end;
    const int M = cam.sh_coeffs;
    float *sh_row = sh_rows + threadIdx.x * sh_stride<TMA>(shn);
    ViewGrad g;
    CamGrad cg;
    if (live) preprocess_bwd_view<TMA, CAMGRAD>(cam, a, i, sh_row, __float_as_uint(a.splat[(size_t)i * SPLAT_F4 + 2].w), g, &cg);
    if (CAMGRAD) {
        if (!live) cam_zero(cg);
        cam_warp_partial(cg, a.cam_part, PRE_THREADS / 32 * gridDim.x, blockIdx.x * (PRE_THREADS / 32) + threadIdx.x / 32);
    }

    // SH gradient rows go out through shared memory (coalesced / one bulk store); each thread rewrites only its own row
    if ((a.g.dL_dshs || (SPLIT && a.dL_drest)) && a.shs) {
        if (live) sh_grad_row<TMA, false>(sh_row, g.bas, g.d_rgb_sh, nb, M);
        if (TMA) {
            tma_row_out<ACC>(a.g.dL_dshs, sh_row, i, shn, live);
        } else {
            __syncthreads();
            if (SPLIT) stage_split_rows_out<ACC>(a.g.dL_dshs, a.dL_drest, sh_rows, row0, nrows, shn);
            else stage_rows_out<ACC>(a.g.dL_dshs, sh_rows, row0, nrows, shn);
        }
    }
    if (!live) return;
    if (a.g.dL_dmeans2D) {
        put<ACC>(a.g.dL_dmeans2D + 3 * (size_t)i, g.g_m2[0]); put<ACC>(a.g.dL_dmeans2D + 3 * (size_t)i + 1, g.g_m2[1]);
        put<ACC>(a.g.dL_dmeans2D + 3 * (size_t)i + 2, 0.f);
    }
    write_gauss_grads<ACC>(a, i, g.gm, g.g_op, g.g_rgb, g.g_sc, g.g_rot, g.dS);
}

// View-batch K8: parameters read once, the V views' accumulators chained one after the other, the per-gaussian
// gradient summed over views in registers (SH: in a second shared-memory row) and written ONCE.
// Per-view arrays (dacc, splat, means2D gradient) are [V][...] with uniform strides.
// CAMGRAD: view v's warp partials of the camera gradient go to panel v of a.cam_part ([V][CAM_TERMS][4 * gridDim.x]).
template <bool ACC, bool TMA, bool CAMGRAD = false>
__global__ void __launch_bounds__(PRE_THREADS)
preprocess_bwd_batch_kernel(const CamArgsBatch cb, const PreBwdArgs a, const PreBwdBatchStrides st) {
    __shared__ CamParams cams[GSB_MAX_VIEWS];
    __shared__ unsigned long long bar;
    GSB_DYNAMIC_SMEM(float4, sh_rows4);
    float *sh_rows = reinterpret_cast<float *>(sh_rows4);
    for (int v = 0; v < cb.V; ++v) load_cam(cb.cam[v], cams[v]);
    const int row0 = a.p_begin + blockIdx.x * PRE_THREADS;      // gaussians [p_begin, p_end) of this launch
    const int nrows = min(PRE_THREADS, a.p_end - row0);
    const int shn = 3 * cb.cam[0].sh_coeffs;
    const int nb = (cb.cam[0].sh_degree + 1) * (cb.cam[0].sh_degree + 1);
    float *grad_rows = sh_rows + PRE_THREADS * sh_stride<TMA>(shn);
    if (a.shs) {
        if (TMA) tma_rows_in(a.shs, sh_rows, &bar, row0, nrows, shn);
        else stage_rows_in(a.shs, sh_rows, row0, nrows, shn, 3 * nb);
    }
    __syncthreads();
    const int i = row0 + threadIdx.x;
    const bool live = i < a.p_end;
    const int M = cb.cam[0].sh_coeffs;
    const float *sh_row = sh_rows + threadIdx.x * sh_stride<TMA>(shn);
    float *gr = grad_rows + threadIdx.x * sh_stride<TMA>(shn);
    float gm[3] = {0.f, 0.f, 0.f}, g_op = 0.f, g_rgb[3] = {0.f, 0.f, 0.f}, g_sc[3] = {0.f, 0.f, 0.f};
    float g_rot[4] = {0.f, 0.f, 0.f, 0.f}, dS[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const bool want_sh = a.g.dL_dshs && a.shs;
    // view v of a live gaussian: its gradient added to the sums above (CAMGRAD: its camera terms written to *cg)
    auto one_view = [&](const int v, CamGrad *cg) {
        PreBwdArgs av = a;
        av.splat += (size_t)v * st.splat; av.dacc += (size_t)v * st.dacc;
        const uint32_t bits = __float_as_uint(av.splat[(size_t)i * SPLAT_F4 + 2].w);
        if (!(bits & 8u)) {
            if (a.g.dL_dmeans2D) {
                float *m2 = a.g.dL_dmeans2D + (size_t)v * st.means2D + 3 * (size_t)i;
                m2[0] = 0.f; m2[1] = 0.f; m2[2] = 0.f;
            }
            return;
        }
        ViewGrad g;
        if (!preprocess_bwd_view<TMA, CAMGRAD>(cams[v], av, i, sh_row, bits, g, cg)) {
            if (a.g.dL_dmeans2D) {
                float *m2 = a.g.dL_dmeans2D + (size_t)v * st.means2D + 3 * (size_t)i;
                m2[0] = 0.f; m2[1] = 0.f; m2[2] = 0.f;
            }
            return;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) { gm[c] += g.gm[c]; g_rgb[c] += g.g_rgb[c]; g_sc[c] += g.g_sc[c]; }
#pragma unroll
        for (int c = 0; c < 4; ++c) g_rot[c] += g.g_rot[c];
#pragma unroll
        for (int c = 0; c < 6; ++c) dS[c] += g.dS[c];
        g_op += g.g_op;
        if (want_sh) sh_grad_row<TMA, true>(gr, g.bas, g.d_rgb_sh, nb, M);
        if (a.g.dL_dmeans2D) {
            float *m2 = a.g.dL_dmeans2D + (size_t)v * st.means2D + 3 * (size_t)i;
            m2[0] = g.g_m2[0]; m2[1] = g.g_m2[1]; m2[2] = 0.f;
        }
    };
    if (live) {
        if (want_sh) {
            if (TMA) {
                float4 *gq = reinterpret_cast<float4 *>(gr);
                for (int k = 0; 4 * k < 3 * M; ++k) gq[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            } else {
                for (int k = 0; k < 3 * M; ++k) gr[k] = 0.f;
            }
        }
#ifdef GSB_PRE_UNROLL
        constexpr int kViewUnroll = GSB_PRE_UNROLL;
#else
        constexpr int kViewUnroll = 1;
#endif
        if (!CAMGRAD) {
#pragma unroll kViewUnroll
            for (int v = 0; v < cb.V; ++v) one_view(v, nullptr);
        }
    }
    if (CAMGRAD) {
        // every lane of the block runs every view (compute or zero, then the warp sum): no lane may skip a shuffle
        const int nslots = PRE_THREADS / 32 * gridDim.x, slot = blockIdx.x * (PRE_THREADS / 32) + threadIdx.x / 32;
        for (int v = 0; v < cb.V; ++v) {
            CamGrad cg;
            cam_zero(cg);
            if (live) one_view(v, &cg);
            cam_warp_partial(cg, a.cam_part + (size_t)v * CAM_TERMS * nslots, nslots, slot);
        }
    }
    if (TMA && a.peer.world > 0) {
        // Fused reduce-scatter.  SH gradient rows: one bulk reduce-add per row into the owner's buffer.  Narrow gradients (11
        // floats per gaussian): staged as four dense [128, w] panels in the (now dead) parameter rows, one bulk reduce-add each --
        // four NVLink-sized transactions per block instead of 11 scalar atomics per gaussian.  Threads past the end add zeros
        // into the padding rows of the owner's buffer (the buffers hold world * rows_per_rank rows).
        const long long dlt = peer_delta(a.peer, row0);
        if (want_sh) tma_row_out<true>(shift_ptr(a.g.dL_dshs, dlt), gr, i, shn, live);
        __syncthreads();                                   // every thread is done reading its parameter row
        float *pan = sh_rows;                              // [128,3] xyz | [128] opacity | [128,3] scales | [128,4] rotations
        const int t = threadIdx.x;
#pragma unroll
        for (int c = 0; c < 3; ++c) { pan[3 * t + c] = live ? gm[c] : 0.f; pan[4 * PRE_THREADS + 3 * t + c] = live ? g_sc[c] : 0.f; }
        pan[3 * PRE_THREADS + t] = live ? g_op : 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) pan[7 * PRE_THREADS + 4 * t + c] = live ? g_rot[c] : 0.f;
        bulk_store_fence();
        __syncthreads();
        if (t == 0 && a.g.dL_dmeans3D) bulk_s2g_add_f32(shift_ptr(a.g.dL_dmeans3D, dlt) + 3 * (size_t)row0, pan, 3 * PRE_THREADS * 4);
        if (t == 1 && a.g.dL_dopacities) bulk_s2g_add_f32(shift_ptr(a.g.dL_dopacities, dlt) + (size_t)row0, pan + 3 * PRE_THREADS, PRE_THREADS * 4);
        if (t == 2 && a.g.dL_dscales) bulk_s2g_add_f32(shift_ptr(a.g.dL_dscales, dlt) + 3 * (size_t)row0, pan + 4 * PRE_THREADS, 3 * PRE_THREADS * 4);
        if (t == 3 && a.g.dL_drotations) bulk_s2g_add_f32(shift_ptr(a.g.dL_drotations, dlt) + 4 * (size_t)row0, pan + 7 * PRE_THREADS, 4 * PRE_THREADS * 4);
        if (t < 4) bulk_store_commit_and_wait();
        return;
    }
    if (want_sh) {
        if (TMA) {
            tma_row_out<ACC>(a.g.dL_dshs, gr, i, shn, live);
        } else {
            __syncthreads();
            stage_rows_out<ACC>(a.g.dL_dshs, grad_rows, row0, nrows, shn);
        }
    }
    if (!live) return;
    write_gauss_grads<ACC>(a, i, gm, g_op, g_rgb, g_sc, g_rot, dS);
}

__global__ void __launch_bounds__(PRE_THREADS)
mark_visible_kernel(const int P, const float *__restrict__ means, const float *__restrict__ view, uint8_t *present) {
    const int i = blockIdx.x * PRE_THREADS + threadIdx.x;
    if (i >= P) return;
    const float tz = __ldg(view + 2) * means[3 * i] + __ldg(view + 6) * means[3 * i + 1] + __ldg(view + 10) * means[3 * i + 2] + __ldg(view + 14);
    present[i] = tz > NEAR_CULL ? 1 : 0;
}

// Option pre_tma: SH rows move between global and shared memory as TMA bulk copies (one per row) and are accessed as float4.
// Needs 16-byte rows (n = 3 M a multiple of 4: SH degree 1 and 3 tensors) and 16-byte aligned tensors.
int g_pre_tma = 1;   // TMA bulk copies of the SH rows in the per-gaussian kernels; 0 = off (A/B)
static bool use_tma_rows(const float *shs, const float *dshs, int sh_coeffs) {
    return g_pre_tma && shs && ((3 * sh_coeffs) & 3) == 0 && (reinterpret_cast<size_t>(shs) & 15) == 0 &&
           (reinterpret_cast<size_t>(dshs) & 15) == 0;
}
static size_t sh_smem_bytes(bool tma, int sh_coeffs, int rows_per_thread) {
    const int n = 3 * sh_coeffs;
    return (size_t)rows_per_thread * PRE_THREADS * (tma ? sh_row_stride_vec(n) : sh_row_stride(n)) * sizeof(float);
}
#define GSB_PRE_LAUNCH(kernel, grid, smem, ...)                                                                             \
    do {                                                                                                                    \
        if ((smem) > 40 * 1024) GSB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(smem))); \
        GSB_LAUNCH(name, debug, stream, kernel, grid, PRE_THREADS, smem, __VA_ARGS__);                                      \
    } while (0)

// split: split SH input (12-byte DC rows next to the rest rows: no TMA row copies, the scalar row layout is staged from both)
int launch_preprocess_fwd(const CamArgs &ca, const PreFwdArgs &a, bool split, bool debug, cudaStream_t stream) {
    if (a.P <= 0) return GSB_OK;
    const char *name = "preprocess_fwd";
    const bool tma = !split && use_tma_rows(a.shs, nullptr, ca.sh_coeffs);
    const size_t smem = a.shs ? sh_smem_bytes(tma, ca.sh_coeffs, 1) : 0;
    const int grid = (int)ceil_div(a.P, PRE_THREADS);
    if (split) GSB_PRE_LAUNCH((preprocess_fwd_kernel<false, true>), grid, smem, ca, a);
    else if (tma) GSB_PRE_LAUNCH(preprocess_fwd_kernel<true>, grid, smem, ca, a);
    else GSB_PRE_LAUNCH(preprocess_fwd_kernel<false>, grid, smem, ca, a);
    return GSB_OK;
}

int launch_preprocess_bwd(const CamArgs &ca, const PreBwdArgs &a, bool split, bool accumulate, bool debug, cudaStream_t stream) {
    if (a.P <= 0 || a.p_end <= a.p_begin) return GSB_OK;
    const char *name = "preprocess_bwd";
    const int grid = (int)ceil_div(a.p_end - a.p_begin, PRE_THREADS);
    const bool tma = !split && use_tma_rows(a.shs, a.g.dL_dshs, ca.sh_coeffs);
    const size_t smem = a.shs ? sh_smem_bytes(tma, ca.sh_coeffs, 1) : 0;
    if (a.cam_part) {   // camera gradient: the accumulate switch only concerns the per-gaussian outputs here
        if (split) {
            if (accumulate) GSB_PRE_LAUNCH((preprocess_bwd_kernel<true, false, true, true>), grid, smem, ca, a);
            else GSB_PRE_LAUNCH((preprocess_bwd_kernel<false, false, true, true>), grid, smem, ca, a);
        } else if (accumulate) {
            if (tma) GSB_PRE_LAUNCH((preprocess_bwd_kernel<true, true, false, true>), grid, smem, ca, a);
            else GSB_PRE_LAUNCH((preprocess_bwd_kernel<true, false, false, true>), grid, smem, ca, a);
        } else {
            if (tma) GSB_PRE_LAUNCH((preprocess_bwd_kernel<false, true, false, true>), grid, smem, ca, a);
            else GSB_PRE_LAUNCH((preprocess_bwd_kernel<false, false, false, true>), grid, smem, ca, a);
        }
    } else if (split) {
        if (accumulate) GSB_PRE_LAUNCH((preprocess_bwd_kernel<true, false, true>), grid, smem, ca, a);
        else GSB_PRE_LAUNCH((preprocess_bwd_kernel<false, false, true>), grid, smem, ca, a);
    } else if (accumulate) {
        if (tma) GSB_PRE_LAUNCH((preprocess_bwd_kernel<true, true>), grid, smem, ca, a);
        else GSB_PRE_LAUNCH((preprocess_bwd_kernel<true, false>), grid, smem, ca, a);
    } else {
        if (tma) GSB_PRE_LAUNCH((preprocess_bwd_kernel<false, true>), grid, smem, ca, a);
        else GSB_PRE_LAUNCH((preprocess_bwd_kernel<false, false>), grid, smem, ca, a);
    }
    return GSB_OK;
}

int launch_preprocess_fwd_batch(const CamArgsBatch &cb, const PreFwdArgs &a, const PreFwdBatchStrides &st, bool debug, cudaStream_t stream) {
    if (a.P <= 0) return GSB_OK;
    const char *name = "preprocess_fwd";
    const bool tma = use_tma_rows(a.shs, nullptr, cb.cam[0].sh_coeffs);
    const size_t smem = a.shs ? sh_smem_bytes(tma, cb.cam[0].sh_coeffs, 1) : 0;
    const int grid = (int)ceil_div(a.P, PRE_THREADS);
    if (tma) GSB_PRE_LAUNCH(preprocess_fwd_batch_kernel<true>, grid, smem, cb, a, st);
    else GSB_PRE_LAUNCH(preprocess_fwd_batch_kernel<false>, grid, smem, cb, a, st);
    return GSB_OK;
}

int launch_preprocess_bwd_batch(const CamArgsBatch &cb, const PreBwdArgs &a, const PreBwdBatchStrides &st, bool accumulate, bool debug,
                                cudaStream_t stream) {
    if (a.P <= 0 || a.p_end <= a.p_begin) return GSB_OK;
    const char *name = "preprocess_bwd";
    const int grid = (int)ceil_div(a.p_end - a.p_begin, PRE_THREADS);
    const bool tma = use_tma_rows(a.shs, a.g.dL_dshs, cb.cam[0].sh_coeffs);
    if (a.peer.world > 0) {
        if (!tma || 3 * cb.cam[0].sh_coeffs < 11) {
            set_error("peer gradients need the TMA row path (option pre_tma, SH rows of 16-byte multiples, at least 4 coefficients)");
            return GSB_ERR_ARGUMENT;
        }
        if (a.peer.world > GSB_MAX_PEERS || a.peer.rows_per_rank <= 0 || a.peer.rows_per_rank % PRE_THREADS) {
            set_error("peer gradients: rows_per_rank must be a positive multiple of %d, world <= %d", PRE_THREADS, GSB_MAX_PEERS);
            return GSB_ERR_ARGUMENT;
        }
    }
    const size_t smem = a.shs ? sh_smem_bytes(tma, cb.cam[0].sh_coeffs, 2) : 0;
    if (a.cam_part) {
        if (a.peer.world > 0) {
            set_error("camera gradients are not available with peer gradients: their sum would have to span the ranks");
            return GSB_ERR_ARGUMENT;
        }
        if (accumulate) {
            if (tma) GSB_PRE_LAUNCH((preprocess_bwd_batch_kernel<true, true, true>), grid, smem, cb, a, st);
            else GSB_PRE_LAUNCH((preprocess_bwd_batch_kernel<true, false, true>), grid, smem, cb, a, st);
        } else {
            if (tma) GSB_PRE_LAUNCH((preprocess_bwd_batch_kernel<false, true, true>), grid, smem, cb, a, st);
            else GSB_PRE_LAUNCH((preprocess_bwd_batch_kernel<false, false, true>), grid, smem, cb, a, st);
        }
    } else if (accumulate) {
        if (tma) GSB_PRE_LAUNCH((preprocess_bwd_batch_kernel<true, true>), grid, smem, cb, a, st);
        else GSB_PRE_LAUNCH((preprocess_bwd_batch_kernel<true, false>), grid, smem, cb, a, st);
    } else {
        if (tma) GSB_PRE_LAUNCH((preprocess_bwd_batch_kernel<false, true>), grid, smem, cb, a, st);
        else GSB_PRE_LAUNCH((preprocess_bwd_batch_kernel<false, false>), grid, smem, cb, a, st);
    }
    return GSB_OK;
}

// ---- camera gradient: the per-view sums ------------------------------------------------------------------------------------
// One block per (output entry, view): the block sums its term's warp partials (or, for bg, final_T * dL/dcolor over the
// pixels) with a strided per-thread loop and a shared-memory tree -- a fixed order, so the result is reproducible bit for bit.
constexpr int CAM_RED_THREADS = 256;

// output entry j (0..15 viewmatrix, 16..31 projmatrix, 32..34 campos) -> term of CamGrad, or -1 for a column the forward never reads
__device__ __forceinline__ int cam_term_of(const int j) {
    if (j < 16) return (j & 3) == 3 ? -1 : 3 * (j >> 2) + (j & 3);
    if (j < 32) {
        const int r = (j - 16) >> 2, c = (j - 16) & 3;
        return c == 2 ? -1 : 12 + 3 * r + (c == 3 ? 2 : c);
    }
    return 24 + (j - 32);
}

// block-wide sum of s (shared-memory tree, fixed order); thread 0 writes it to *out (ACC: adds)
__device__ __forceinline__ void block_sum_to(const float s, float *red, float *out, const bool acc) {
    const int t = threadIdx.x;
    red[t] = s;
    __syncthreads();
    for (int h = CAM_RED_THREADS / 2; h > 0; h >>= 1) {
        if (t < h) red[t] += red[t + h];
        __syncthreads();
    }
    if (t == 0) *out = acc ? *out + red[0] : red[0];
    __syncthreads();   // red is reused by the caller's next sum
}

template <bool ACC>
__global__ void __launch_bounds__(CAM_RED_THREADS)
camera_grad_reduce_kernel(const CamReduceArgs r) {
    __shared__ float red[CAM_RED_THREADS];
    const int j = blockIdx.x, v = blockIdx.y, t = threadIdx.x;
    float *out;
    if (j < 16) out = r.dview ? r.dview + 16 * v + j : nullptr;
    else if (j < 32) out = r.dproj ? r.dproj + 16 * v + (j - 16) : nullptr;
    else if (j < 35) out = r.dcampos ? r.dcampos + 3 * v + (j - 32) : nullptr;
    else out = r.dbg ? r.dbg + 3 * v + (j - 35) : nullptr;
    if (!out) return;                      // uniform per block
    float s = 0.f;
    const float *p;
    int n;
    if (j < 35) {
        const int term = cam_term_of(j);
        if (term < 0) {
            if (t == 0 && !ACC) *out = 0.f;
            return;
        }
        p = r.part + ((size_t)v * CAM_TERMS + term) * r.nslots;
        n = r.nslots;
    } else {
        p = r.bg_part + ((size_t)v * 3 + (j - 35)) * CAM_BG_BLOCKS;
        n = CAM_BG_BLOCKS;
    }
    for (int k = t; k < n; k += CAM_RED_THREADS) s += p[k];
    block_sum_to(s, red, out, ACC);
}

// dL/dbg partials: block b of view v sums final_T * dL/dcolor[c] over its contiguous pixel range, c = 0..2
__global__ void __launch_bounds__(CAM_RED_THREADS)
camera_bg_partial_kernel(const CamReduceArgs r) {
    __shared__ float red[CAM_RED_THREADS];
    const int b = blockIdx.x, v = blockIdx.y, t = threadIdx.x;
    const size_t chunk = (r.npix + CAM_BG_BLOCKS - 1) / CAM_BG_BLOCKS;
    const size_t p0 = b * chunk, p1 = min(r.npix, p0 + chunk);
    const float *T = r.final_T + (size_t)v * r.sv_image;
    for (int c = 0; c < 3; ++c) {
        const float *g = r.dL_dcolor + ((size_t)v * 3 + c) * r.npix;
        float s = 0.f;
        for (size_t k = p0 + t; k < p1; k += CAM_RED_THREADS) s += T[k] * g[k];
        block_sum_to(s, red, r.bg_part + ((size_t)v * 3 + c) * CAM_BG_BLOCKS + b, false);
    }
}

size_t cam_slots(int n_gauss) { return (size_t)ceil_div(n_gauss > 0 ? n_gauss : 0, PRE_THREADS) * (PRE_THREADS / 32); }

int launch_camera_grad_reduce(const CamReduceArgs &r, bool accumulate, bool debug, cudaStream_t stream) {
    if (!r.dview && !r.dproj && !r.dcampos && !r.dbg) return GSB_OK;
    if (r.dbg) {
        const char *name = "camera_bg_partial";
        GSB_LAUNCH(name, debug, stream, camera_bg_partial_kernel, dim3(CAM_BG_BLOCKS, r.V), CAM_RED_THREADS, 0, r);
    }
    const char *name = "camera_grad_reduce";
    const dim3 grid(CAM_OUTPUTS, r.V);
    if (accumulate) GSB_LAUNCH(name, debug, stream, camera_grad_reduce_kernel<true>, grid, CAM_RED_THREADS, 0, r);
    else GSB_LAUNCH(name, debug, stream, camera_grad_reduce_kernel<false>, grid, CAM_RED_THREADS, 0, r);
    return GSB_OK;
}

int launch_mark_visible(int P, const float *means, const float *view, uint8_t *present, cudaStream_t stream) {
    if (P <= 0) return GSB_OK;
    GSB_LAUNCH("mark_visible", false, stream, mark_visible_kernel, (int)ceil_div(P, PRE_THREADS), PRE_THREADS, 0, P, means, view, present);
    return GSB_OK;
}

}  // namespace gsb
