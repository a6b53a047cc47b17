// adam.cuh -- one element of the reference's non-capturable Adam step (scene/OurAdam.py:249-337; amsgrad off,
// weight_decay 0), shared by the sparse Adam (optim.cu) and train_coarse's parameter step (coarse_param.cu):
//   m = b1 m + (1-b1) g ;  v = b2 v + (1-b2) g^2 ;  p -= step_size * m / (sqrt(v)/bc2_sqrt + eps)
// every product, quotient, root and sum rounded on its own (no FMA contraction), step_size = lr / bc1 and bc2_sqrt =
// sqrt(bc2) formed in double and rounded to fp32 once, as the reference's Python floats meet its fp32 tensors.
#pragma once

namespace h3dgs {

__device__ __forceinline__ void adam_element(float& param, float g, float& exp_avg, float& exp_avg_sq, float beta1,
                                             float beta2, float one_minus_b1, float one_minus_b2, float step_size,
                                             float bc2_sqrt, float eps)
{
    // exp_avg.mul_(beta1).add_(grad, alpha=1-beta1) ; exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1-beta2)
    const float m = __fadd_rn(__fmul_rn(exp_avg, beta1), __fmul_rn(one_minus_b1, g));
    const float v = __fadd_rn(__fmul_rn(exp_avg_sq, beta2), __fmul_rn(one_minus_b2, __fmul_rn(g, g)));
    // denom = (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps) ; param.addcdiv_(exp_avg, denom, value=-step_size)
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
    param = __fadd_rn(param, __fmul_rn(-step_size, __fdiv_rn(m, denom)));
    exp_avg = m;
    exp_avg_sq = v;
}

// one element of torch.optim.Adam's default CUDA path (_multi_tensor_adam, non-capturable; amsgrad off, weight_decay
// 0), shared by train_single's exposure step (single_param.cu) and train_post's dense step (post_param.cu).  Its
// foreach kernels compute in fp32 with FMA contraction:
//   m = lerp(m, g, w) with w = (float)(1 - beta1): |w| < 0.5 ? fma(w, g - m, m) : fma(m - g, 1 - w, g)
//   v = v * beta2;  v = fma((float)(1 - beta2), g * g, v)
//   p = fma(step_size, m / (sqrt(v) / bc2_sqrt + eps), p)
// with step_size = (float)(-(lr / (1 - beta1^t))) and bc2_sqrt = (float)sqrt(1 - beta2^t) formed in double (torch's
// Python floats of the host step count t)
__device__ __forceinline__ void torch_adam_element(float& param, float g, float& exp_avg, float& exp_avg_sq, float w,
                                                   float beta2, float one_minus_b2, float step_size, float bc2_sqrt,
                                                   float eps)
{
    const float m0 = exp_avg;
    // at::native::lerp with opmath float, contracted
    const float m = fabsf(w) < 0.5f ? __fmaf_rn(w, __fsub_rn(g, m0), m0) : __fmaf_rn(__fsub_rn(m0, g), __fsub_rn(1.f, w), g);
    const float v = __fmaf_rn(one_minus_b2, __fmul_rn(g, g), __fmul_rn(exp_avg_sq, beta2));
    const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
    param = __fmaf_rn(step_size, __fdiv_rn(m, den), param);
    exp_avg = m;
    exp_avg_sq = v;
}

}  // namespace h3dgs
