// optim.cu -- sparse Adam (SURVEY.md 8f-4): Adam that touches only the rows listed in `relevant`
// (replaces scene/OurAdam.py:249-337, driven by train_single.py:170-178 with relevant = rows whose
// opacity gradient is non-zero).  The reference gathers the rows of param / grad / exp_avg / exp_avg_sq
// with fancy indexing, runs ~10 elementwise kernels on the copies and scatters three tensors back, per
// parameter group; here one kernel per parameter tensor updates the rows in place, with the arithmetic of adam.cuh
// (bc1 = 1 - b1^step, bc2 = 1 - b2^step computed by the caller in host doubles, as the reference does with Python
// floats).  A negative entry of `relevant` is skipped; relevant == NULL is every row of [0, num_relevant).  HBM-bound: 4 reads + 3 writes of 4 B per touched element.
#include "common.cuh"
#include "adam.cuh"

namespace h3dgs {

__global__ void __launch_bounds__(256)
sparse_adam_kernel(int64_t R, int width, const int64_t* __restrict__ relevant, float* __restrict__ param,
                   const float* __restrict__ grad, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                   float beta1, float beta2, float one_minus_b1, float one_minus_b2, float step_size,
                   float bc2_sqrt, float eps)
{
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= R * width) return;
    const int64_t r = t / width;
    const int c = (int)(t - r * width);
    const int64_t row = relevant ? relevant[r] : r;
    if (row < 0) return;                                    // a skipped entry (h3dgs.optim.Adam's [R,2] row sets)
    const size_t o = (size_t)row * width + c;
    float p = param[o], m = exp_avg[o], v = exp_avg_sq[o];
    adam_element(p, grad[o], m, v, beta1, beta2, one_minus_b1, one_minus_b2, step_size, bc2_sqrt, eps);
    param[o] = p;
    exp_avg[o] = m;
    exp_avg_sq[o] = v;
}

}  // namespace h3dgs

extern "C" int h3dgs_sparse_adam(int64_t num_relevant, int32_t width, const int64_t* relevant, float* param,
                                 const float* grad, float* exp_avg, float* exp_avg_sq, double lr, double beta1,
                                 double beta2, double eps, int64_t step, void* stream)
{
    using namespace h3dgs;
    if (num_relevant < 0 || width <= 0 || step <= 0 || (num_relevant > 0 && (!param || !grad || !exp_avg || !exp_avg_sq))) {
        set_error("sparse_adam: bad arguments"); return H3DGS_EINVAL;
    }
    if (num_relevant == 0) return H3DGS_OK;
    // hyper-parameters arrive as doubles and every derived constant is formed in double and rounded to
    // fp32 once, exactly where the reference's Python floats meet its fp32 tensors
    const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
    const float step_size = (float)(lr / bc1), bc2_sqrt = (float)sqrt(bc2);
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t total = num_relevant * width;
    sparse_adam_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(num_relevant, width, relevant, param, grad, exp_avg,
                                                                       exp_avg_sq, (float)beta1, (float)beta2, (float)(1.0 - beta1),
                                                                       (float)(1.0 - beta2), step_size, bc2_sqrt, (float)eps);
    H3_LAUNCHED("sparse_adam", 0, s);
    return H3DGS_OK;
}
