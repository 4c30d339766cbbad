// optim.cu -- the optimizer step that follows the path (SURVEY.md section 8(f) #3): torch.optim.Adam over the reference's six
// parameter groups (scene/gaussian_model.py:176-199, train.py:178-186) as ONE launch over the flat store, with the
// activation backward (exp / sigmoid / normalize, gaussian_model.py:33-46 -- autograd's job in the reference) in front of
// it and the re-activation behind it.  HBM bound: 4 loads + 3 stores of 4 bytes per stored float (28 B/float, 1.65 GB at
// 1 M gaussians and SH degree 3).
#include "common.cuh"
#include "kernels.cuh"

namespace gsb {

constexpr int AD_THREADS = 256, AD_UNROLL = 4;

struct AdamK {
    uint32_t P, F;                     // gaussians, floats per features row (3 * sh_coeffs)
    uint32_t e_feat, e_op, e_sc, E;    // first element of features / opacity / scaling, and of rotation (= elementwise count)
    uint32_t elem_blocks;
    float *p;
    const float *g;
    float *m, *v, *act;
    const uint8_t *vis;
    float ss[6], bc2s[6];              // per group: lr / (1 - beta1^t), sqrt(1 - beta2^t) -- every group has its own step count t
    uint32_t skip;                     // bit g: group g is left untouched (its parameter was just replaced: grad None in the reference)
    float b1, b2, eps;
};

struct AdamCoef {
    float omb1, b2, omb2, eps;
};

__device__ __forceinline__ void adam_update(float &p, float &m, float &v, const float g, const float ss, const float bc2s, const AdamCoef &c) {
    m = m + c.omb1 * (g - m);                       // exp_avg.lerp_(grad, 1 - beta1)
    v = v * c.b2;                                   // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value = 1 - beta2)
    v = v + (c.omb2 * g) * g;
    const float denom = sqrtf(v) / bc2s + c.eps;  // (exp_avg_sq.sqrt() / sqrt(bias_correction2)).add_(eps)
    p = p + (-ss) * (m / denom);                    // param.addcdiv_(exp_avg, denom, value = -lr / bias_correction1)
}

__device__ __forceinline__ float sigmoidf_(const float x) { return 1.0f / (1.0f + expf(-x)); }

__global__ void __launch_bounds__(AD_THREADS)
adam_step_kernel(const AdamK a) {
    const AdamCoef c{1.0f - a.b1, a.b2, 1.0f - a.b2, a.eps};
    if (blockIdx.x < a.elem_blocks) {
        // ---- xyz, features, opacity, scaling: one stored float per item; element index == item index ----
        const uint32_t base = blockIdx.x * (AD_THREADS * AD_UNROLL) + threadIdx.x;
        float p[AD_UNROLL], g[AD_UNROLL], m[AD_UNROLL], v[AD_UNROLL], ss[AD_UNROLL], bc[AD_UNROLL];
        int kind[AD_UNROLL];   // -1 skip, 0 identity, 1 sigmoid, 2 exp
#pragma unroll
        for (int u = 0; u < AD_UNROLL; ++u) {
            const uint32_t e = base + u * AD_THREADS;
            kind[u] = -1;
            if (e >= a.E) continue;
            uint32_t gi, skip;     // (static indices only: a dynamic index into the kernel parameters would copy them to local memory)
            if (e < a.e_feat) { gi = e / 3u; kind[u] = 0; ss[u] = a.ss[0]; bc[u] = a.bc2s[0]; skip = a.skip & 1u; }
            else if (e < a.e_op) {
                const uint32_t j = e - a.e_feat;
                gi = j / a.F; kind[u] = 0;
                const bool dc = (j - gi * a.F) < 3u;
                ss[u] = dc ? a.ss[1] : a.ss[2]; bc[u] = dc ? a.bc2s[1] : a.bc2s[2]; skip = dc ? (a.skip & 2u) : (a.skip & 4u);
            }
            else if (e < a.e_sc) { gi = e - a.e_op; kind[u] = 1; ss[u] = a.ss[3]; bc[u] = a.bc2s[3]; skip = a.skip & 8u; }
            else { gi = (e - a.e_sc) / 3u; kind[u] = 2; ss[u] = a.ss[4]; bc[u] = a.bc2s[4]; skip = a.skip & 16u; }
            if (skip || (a.vis && !a.vis[gi])) { kind[u] = -1; continue; }
            p[u] = a.p[e]; g[u] = a.g[e]; m[u] = a.m[e]; v[u] = a.v[e];
        }
#pragma unroll
        for (int u = 0; u < AD_UNROLL; ++u) {
            if (kind[u] < 0) continue;
            const uint32_t e = base + u * AD_THREADS;
            float gr = g[u];
            if (kind[u] == 1) { const float y = sigmoidf_(p[u]); gr = (gr * (1.0f - y)) * y; }      // sigmoid_backward
            else if (kind[u] == 2) gr = gr * expf(p[u]);                                              // exp backward
            adam_update(p[u], m[u], v[u], gr, ss[u], bc[u], c);
            a.p[e] = p[u]; a.m[e] = m[u]; a.v[e] = v[u];
            if (a.act) {
                if (kind[u] == 1) a.act[e - a.e_op] = sigmoidf_(p[u]);
                else if (kind[u] == 2) a.act[a.P + (e - a.e_sc)] = expf(p[u]);
            }
        }
        return;
    }
    // ---- rotation: one quaternion per item (normalize couples its four components) ----
    const uint32_t i = (blockIdx.x - a.elem_blocks) * AD_THREADS + threadIdx.x;
    if (i >= a.P || ((a.skip >> 5) & 1u) || (a.vis && !a.vis[i])) return;
    const size_t o = (size_t)a.E + 4u * (size_t)i;
    float q[4], g[4], m[4], v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { q[k] = a.p[o + k]; g[k] = a.g[o + k]; m[k] = a.m[o + k]; v[k] = a.v[o + k]; }
    // y = q / max(|q|, 1e-12) (torch.nn.functional.normalize); dq = (g - y (y.g)) / |q| above the clamp, g / 1e-12 below it
    const float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    float gr[4];
    if (n > 1e-12f) {
        const float y0 = q[0] / n, y1 = q[1] / n, y2 = q[2] / n, y3 = q[3] / n;
        const float d = y0 * g[0] + y1 * g[1] + y2 * g[2] + y3 * g[3];
        gr[0] = (g[0] - y0 * d) / n; gr[1] = (g[1] - y1 * d) / n; gr[2] = (g[2] - y2 * d) / n; gr[3] = (g[3] - y3 * d) / n;
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) gr[k] = g[k] / 1e-12f;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        adam_update(q[k], m[k], v[k], gr[k], a.ss[5], a.bc2s[5], c);
        a.p[o + k] = q[k]; a.m[o + k] = m[k]; a.v[o + k] = v[k];
    }
    if (a.act) {
        const float nn = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
#pragma unroll
        for (int k = 0; k < 4; ++k) a.act[4u * (size_t)a.P + 4u * (size_t)i + k] = q[k] / nn;
    }
}

__global__ void __launch_bounds__(AD_THREADS)
activate_kernel(const uint32_t P, const float *__restrict__ opacity, const float *__restrict__ scaling,
                const float *__restrict__ rotation, float *__restrict__ act) {
    const uint32_t i = blockIdx.x * AD_THREADS + threadIdx.x;
    if (i >= P) return;
    act[i] = sigmoidf_(opacity[i]);
#pragma unroll
    for (int k = 0; k < 3; ++k) act[P + 3u * (size_t)i + k] = expf(scaling[3u * (size_t)i + k]);
    float q[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] = rotation[4u * (size_t)i + k];
    const float nn = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
#pragma unroll
    for (int k = 0; k < 4; ++k) act[4u * (size_t)P + 4u * (size_t)i + k] = q[k] / nn;
}

int launch_adam_step(int64_t P, int sh_coeffs, float *params, const float *grads, float *m, float *v, float *act,
                     const uint8_t *visible, const float step_size[6], float beta1, float beta2, float eps, const float bias2_sqrt[6],
                     uint32_t skip_groups, cudaStream_t stream) {
    if (P == 0) return GSB_OK;
    AdamK a;
    a.P = (uint32_t)P; a.F = 3u * (uint32_t)sh_coeffs;
    a.e_feat = 3u * a.P; a.e_op = a.e_feat + a.F * a.P; a.e_sc = a.e_op + a.P; a.E = a.e_sc + 3u * a.P;
    a.elem_blocks = (uint32_t)ceil_div((int64_t)a.E, AD_THREADS * AD_UNROLL);
    a.p = params; a.g = grads; a.m = m; a.v = v; a.act = act; a.vis = visible;
    for (int k = 0; k < 6; ++k) { a.ss[k] = step_size[k]; a.bc2s[k] = bias2_sqrt[k]; }
    a.skip = skip_groups;
    a.b1 = beta1; a.b2 = beta2; a.eps = eps;
    const uint32_t blocks = a.elem_blocks + (uint32_t)ceil_div(P, AD_THREADS);
    GSB_LAUNCH("adam_step", false, stream, adam_step_kernel, blocks, AD_THREADS, 0, a);
    return GSB_OK;
}

// ---- SparseGaussianAdam (train.py --optimizer_type sparse_adam): separate [N, width] tensors per group, one launch ----------
// The blocks of all groups form one grid, group after group (block0[k] = first block of group k).  A visible row costs
// 4 loads + 3 stores of 4 bytes per float; an invisible row costs its mask byte only.
struct SparseAdamK {
    GsbSparseAdamGroup grp[GSB_MAX_SPARSE_GROUPS];
    uint32_t block0[GSB_MAX_SPARSE_GROUPS];
    int n_groups;
    uint32_t N;
    const uint8_t *vis;
    float b1, b2;
};

__global__ void __launch_bounds__(AD_THREADS)
sparse_adam_kernel(const SparseAdamK a) {
    // the block's group, selected with static indices only (a dynamic index into the kernel parameters would copy them to
    // local memory)
    GsbSparseAdamGroup G = a.grp[0];
    uint32_t b0 = 0;
#pragma unroll
    for (int k = 1; k < GSB_MAX_SPARSE_GROUPS; ++k)
        if (k < a.n_groups && blockIdx.x >= a.block0[k]) { G = a.grp[k]; b0 = a.block0[k]; }
    const AdamCoef c{1.0f - a.b1, a.b2, 1.0f - a.b2, G.eps};
    const uint32_t w = (uint32_t)G.width, E = a.N * w;
    const uint32_t base = (blockIdx.x - b0) * (AD_THREADS * AD_UNROLL) + threadIdx.x;
    float p[AD_UNROLL], g[AD_UNROLL], m[AD_UNROLL], v[AD_UNROLL];
    bool on[AD_UNROLL];
#pragma unroll
    for (int u = 0; u < AD_UNROLL; ++u) {
        const uint32_t e = base + u * AD_THREADS;
        on[u] = e < E && a.vis[e / w] != 0;
        if (on[u]) { p[u] = G.param[e]; g[u] = G.grad[e]; m[u] = G.exp_avg[e]; v[u] = G.exp_avg_sq[e]; }
    }
#pragma unroll
    for (int u = 0; u < AD_UNROLL; ++u) {
        if (!on[u]) continue;
        const uint32_t e = base + u * AD_THREADS;
        adam_update(p[u], m[u], v[u], g[u], G.lr, 1.0f, c);     // step_size = lr, bias2_sqrt = 1: no bias correction
        G.param[e] = p[u]; G.exp_avg[e] = m[u]; G.exp_avg_sq[e] = v[u];
    }
}

int launch_sparse_adam_step(const GsbSparseAdamGroup *groups, int n_groups, const uint8_t *visible, int64_t N, float beta1, float beta2,
                            cudaStream_t stream) {
    if (N == 0) return GSB_OK;
    SparseAdamK a{};
    uint32_t blocks = 0;
    for (int k = 0; k < n_groups; ++k) {
        a.grp[k] = groups[k];
        a.block0[k] = blocks;
        blocks += (uint32_t)ceil_div(N * groups[k].width, AD_THREADS * AD_UNROLL);
    }
    a.n_groups = n_groups; a.N = (uint32_t)N; a.vis = visible; a.b1 = beta1; a.b2 = beta2;
    GSB_LAUNCH("sparse_adam", false, stream, sparse_adam_kernel, blocks, AD_THREADS, 0, a);
    return GSB_OK;
}

int launch_activate(int64_t P, int sh_coeffs, const float *params, float *act, cudaStream_t stream) {
    if (P == 0) return GSB_OK;
    const size_t e_op = (size_t)(3 + 3 * sh_coeffs) * P;
    GSB_LAUNCH("activate", false, stream, activate_kernel, (uint32_t)ceil_div(P, AD_THREADS), AD_THREADS, 0, (uint32_t)P,
               params + e_op, params + e_op + P, params + e_op + 4 * (size_t)P, act);
    return GSB_OK;
}

}  // namespace gsb
