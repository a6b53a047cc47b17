// param_row.cuh -- the row-local pieces of a flat GaussianModel's parameter step, shared by train_coarse's
// (coarse_param.cu) and train_single's (single_param.cu): the activations' backward from the rasterizer's activated
// gradients to the six stored tensors, OurAdam on one row (adam.cuh), the big-Gaussian rescale and the activations the
// next forward reads.  train_post's (post_param.cu) takes the quaternion norm and F.normalize's backward from here.
// Every product, quotient and sum is rounded on its own (no FMA contraction); expf and logf are the CUDA math library's
// accurate ones, as torch's exp / log / sigmoid use them.
#pragma once
#include "adam.cuh"

namespace h3dgs {

struct CoarseScratch { float step_size[6], bc2_sqrt[6]; int any; };

struct CoarseConst { float beta1[6], beta2[6], omb1[6], omb2[6], eps[6]; double lr[6], beta1d[6], beta2d[6]; };

__device__ __forceinline__ float sigmoid_f(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// |q| as the forward and the backward take it, and the clamp_min(1e-12) divisor (NaN propagates as torch.clamp_min)
__device__ __forceinline__ void quat_norm(const float q[4], float& n, float& d)
{
    n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q[0], q[0]), __fmul_rn(q[1], q[1])), __fmul_rn(q[2], q[2])),
                             __fmul_rn(q[3], q[3])));
    d = (n != n || n > 1e-12f) ? n : 1e-12f;
}

// F.normalize's backward: x / clamp_min(norm(x), 1e-12).  div: g / d to x, -g * ((x / d) / d) summed to d;
// clamp_min passes where norm >= 1e-12; norm: x * (grad / norm), 0 where norm == 0.  g (the gradient of the normalized
// quaternion) becomes the gradient of the stored one q
__device__ __forceinline__ void normalize_backward(const float q[4], float g[4])
{
    float n, d;
    quat_norm(q, n, d);
    float gd = 0.f;
#pragma unroll
    for (int c = 0; c < 4; c++) gd = __fadd_rn(gd, __fmul_rn(-g[c], __fdiv_rn(__fdiv_rn(q[c], d), d)));
    if (!(n >= 1e-12f)) gd = 0.f;
    const float t = n == 0.f ? 0.f : __fdiv_rn(gd, n);
#pragma unroll
    for (int c = 0; c < 4; c++) g[c] = __fadd_rn(__fdiv_rn(g[c], d), __fmul_rn(q[c], t));
}

// with_rest = false leaves the f_rest part of shs to an element-parallel pass (its copy is the identity)
__device__ __forceinline__ void write_activated(const h3dgs_coarse_args& a, int i, const float s[3], const float e[3], const float q[4],
                                                bool with_rest = true)
{
    const size_t M3 = (size_t)a.sh_coeffs * 3;
#pragma unroll
    for (int c = 0; c < 3; c++) a.means3D[3 * (size_t)i + c] = a.params[0][3 * (size_t)i + c];
#pragma unroll
    for (int c = 0; c < 3; c++) a.shs[M3 * i + c] = a.params[1][3 * (size_t)i + c];
    if (with_rest)
        for (int j = 0; j < (int)M3 - 3; j++) a.shs[M3 * i + 3 + j] = a.params[2][(M3 - 3) * i + j];
    a.opacities[i] = sigmoid_f(a.params[3][i]);
#pragma unroll
    for (int c = 0; c < 3; c++) a.scales[3 * (size_t)i + c] = e[c];
    float n, d;
    quat_norm(q, n, d);
#pragma unroll
    for (int c = 0; c < 4; c++) a.rotations[4 * (size_t)i + c] = __fdiv_rn(q[c], d);
}

// the row's scaling after the step and the rescale (rows >= rescale_from whose largest exp(s) exceeds
// a.rescale_threshold, NaN propagating as torch.max), exp of it, and the activations when anything changed
__device__ __forceinline__ void rescale_and_activate(const h3dgs_coarse_args& a, int i, bool changed, int rescale_from,
                                                     bool with_rest = true)
{
    float s[3], e[3], q[4];
#pragma unroll
    for (int c = 0; c < 3; c++) { s[c] = a.params[4][3 * (size_t)i + c]; e[c] = expf(s[c]); }
    if (i >= rescale_from) {
        float mx = e[0];
#pragma unroll
        for (int c = 1; c < 3; c++) mx = (mx != mx) ? mx : ((e[c] != e[c] || e[c] > mx) ? e[c] : mx);
        if (mx > a.rescale_threshold) {
#pragma unroll
            for (int c = 0; c < 3; c++) {
                s[c] = logf(__fmul_rn(e[c], 0.8f));
                a.params[4][3 * (size_t)i + c] = s[c];
                e[c] = expf(s[c]);
            }
            changed = true;
        }
    }
    if (!changed) return;
#pragma unroll
    for (int c = 0; c < 4; c++) q[c] = a.params[5][4 * (size_t)i + c];
    write_activated(a, i, s, e, q, with_rest);
}

__device__ __forceinline__ void adam_at(const h3dgs_coarse_args& a, const CoarseConst& k, const CoarseScratch& sc, int grp,
                                        size_t o, float g)
{
    float p = a.params[grp][o], m = a.exp_avg[grp][o], v = a.exp_avg_sq[grp][o];
    adam_element(p, g, m, v, k.beta1[grp], k.beta2[grp], k.omb1[grp], k.omb2[grp], sc.step_size[grp], sc.bc2_sqrt[grp], k.eps[grp]);
    a.params[grp][o] = p;
    a.exp_avg[grp][o] = m;
    a.exp_avg_sq[grp][o] = v;
}

// Adam on every stored element of row i, with the stored opacity gradient go already formed.  lock_scaling: the
// scaling gradient is 0 (train_coarse's skybox lock); lock_all: all six stored gradients are 0 (train_single's);
// with_rest = false leaves the f_rest group to an element-parallel pass
__device__ __forceinline__ void adam_row(const h3dgs_coarse_args& a, const CoarseConst& k, const CoarseScratch& sc, int i, float go,
                                         bool lock_scaling, bool lock_all = false, bool with_rest = true)
{
    const size_t M3 = (size_t)a.sh_coeffs * 3;
#pragma unroll
    for (int c = 0; c < 3; c++) adam_at(a, k, sc, 0, 3 * (size_t)i + c, lock_all ? 0.f : a.grad_means3D[3 * (size_t)i + c]);
#pragma unroll
    for (int c = 0; c < 3; c++) adam_at(a, k, sc, 1, 3 * (size_t)i + c, lock_all ? 0.f : a.grad_shs[M3 * i + c]);
    if (with_rest)
        for (int j = 0; j < (int)M3 - 3; j++) adam_at(a, k, sc, 2, (M3 - 3) * i + j, lock_all ? 0.f : a.grad_shs[M3 * i + 3 + j]);
    adam_at(a, k, sc, 3, (size_t)i, go);
    const bool locked = lock_scaling || lock_all;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const size_t o = 3 * (size_t)i + c;
        adam_at(a, k, sc, 4, o, locked ? 0.f : __fmul_rn(a.grad_scales[o], a.scales[o]));
    }
    float q[4], g[4];
#pragma unroll
    for (int c = 0; c < 4; c++) { q[c] = a.params[5][4 * (size_t)i + c]; g[c] = a.grad_rotations[4 * (size_t)i + c]; }
    normalize_backward(q, g);
#pragma unroll
    for (int c = 0; c < 4; c++) adam_at(a, k, sc, 5, 4 * (size_t)i + c, lock_all ? 0.f : g[c]);
}

__device__ __forceinline__ float stored_opacity_grad(const h3dgs_coarse_args& a, int i)
{
    const float y = a.opacities[i];
    return __fmul_rn(__fmul_rn(a.grad_opacities[i], __fsub_rn(1.f, y)), y);        // sigmoid_backward: g * (1 - y) * y
}

// OurAdam's bias corrections of step count `step` (Python floats in the reference), rounded to fp32 once
__device__ __forceinline__ void bias_corrections(double lr, double beta1, double beta2, double step, float& step_size, float& bc2_sqrt)
{
    const double bc1 = 1.0 - pow(beta1, step), bc2 = 1.0 - pow(beta2, step);
    step_size = (float)(lr / bc1);
    bc2_sqrt = (float)sqrt(bc2);
}

}  // namespace h3dgs
