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

}  // namespace h3dgs
