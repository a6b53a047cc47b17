// coarse_param.cu -- train_coarse's parameter side (train_coarse.py:127-145) as one row-local pass on the device: the
// activations' backward from the rasterizer's activated gradients to GaussianModel's six stored tensors, the skybox
// scaling lock, the relevance rule of (grad != 0).nonzero(), OurAdam on the relevant rows, the big-Gaussian rescale and
// the activations the next forward reads.  Nothing returns to the host, so the pass can sit inside a CUDA graph.
//
// Per row i, in the reference's order (every product, quotient and sum rounded on its own, no FMA contraction; expf and
// logf are the CUDA math library's accurate ones, as torch's exp / log / sigmoid use them):
//   stored gradients  xyz: g_means;  f_dc / f_rest: g_shs[:, 0] / g_shs[:, 1:];  opacity: (g * (1 - y)) * y
//                     (sigmoid_backward on the activated opacity y);  scaling: g * exp(s) (exp's backward on the
//                     activated scale);  rotation: F.normalize's backward (div, clamp_min, norm);
//   lock              scaling gradient = 0 for i < skybox_points;
//   relevance         opacity gradient != 0 (NaN counts).  (grad != 0).nonzero() of the [N,1] gradient is [R,2] and its
//                     zero column indexes row 0, so OurAdam updates the relevant rows and row 0 whenever R > 0; with
//                     R == 0 it takes a dense step on every row (scene/OurAdam.py:214-228, _single_tensor_adam2);
//   Adam              adam.cuh on that row set, per group lr / betas / eps, the bias corrections of the new step count;
//   rescale           i >= skybox_points with max_k exp(s_k) > threshold (NaN propagating as torch.max):
//                     s_k = log(exp(s_k) * 0.8f);
//   activations       means3D = xyz, shs = [f_dc, f_rest], opacities = 1 / (1 + exp(-o)), scales = exp(s),
//                     rotations = q / max(|q|, 1e-12) with |q| = sqrt(((q0^2 + q1^2) + q2^2) + q3^2).
// Three launches: a one-thread prologue (step += 1, its bias corrections, the any-relevant word cleared), a relevance
// pass that raises the any-relevant word (8 bytes per row), and the update pass over every row, whose row set the word
// selects.  An overflowed capacity-mode frame (scan_info[2]) changes nothing.
#include "common.cuh"
#include "param_row.cuh"

namespace h3dgs {

static_assert(sizeof(CoarseScratch) <= H3DGS_COARSE_SCRATCH_BYTES, "scratch");

__device__ __forceinline__ bool overflowed(const h3dgs_coarse_args& a) { return a.scan_info && a.scan_info[2]; }

// count = 1 (H3DGS_COARSE_STEP): the step is taken, step += 1 first (OurAdam's step_t += 1 of every call, whatever the
// rows, scene/OurAdam.py:277, 359); the bias corrections are those of the new count
__global__ void coarse_prologue_kernel(h3dgs_coarse_args a, CoarseConst k, int count)
{
    if (overflowed(a)) return;
    CoarseScratch* sc = (CoarseScratch*)a.scratch;
    const double step = (double)(*a.step + 1);
    if (count) *a.step += 1;
    for (int g = 0; g < 6; g++) bias_corrections(k.lr[g], k.beta1d[g], k.beta2d[g], step, sc->step_size[g], sc->bc2_sqrt[g]);
    sc->any = 0;
}

// relevance of every row: raises the any-relevant word that selects the update pass's row set
__global__ void __launch_bounds__(256) coarse_relevance_kernel(h3dgs_coarse_args a)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= a.N || overflowed(a)) return;
    if (stored_opacity_grad(a, i) != 0.f) ((CoarseScratch*)a.scratch)->any = 1;
}

// Adam on OurAdam's row set, then the rescale and the activations.  With a relevant row somewhere the set is the
// relevant rows and row 0 (the zero column of the unflattened index, scene/OurAdam.py:216-228 -> _single_tensor_adam);
// with none, OurAdam takes its dense step on every row (relevant.size(0) == 0 -> _single_tensor_adam2, :339-426)
__global__ void __launch_bounds__(256) coarse_update_kernel(h3dgs_coarse_args a, CoarseConst k)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= a.N || overflowed(a)) return;
    const CoarseScratch& sc = *(const CoarseScratch*)a.scratch;
    const float go = stored_opacity_grad(a, i);
    const bool update = sc.any ? (go != 0.f || i == 0) : true;
    if (update) adam_row(a, k, sc, i, go, i < a.skybox_points);
    rescale_and_activate(a, i, update, a.skybox_points);
}

__global__ void __launch_bounds__(256) coarse_activate_kernel(h3dgs_coarse_args a)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= a.N) return;
    float s[3], e[3], q[4];
#pragma unroll
    for (int c = 0; c < 3; c++) { s[c] = a.params[4][3 * (size_t)i + c]; e[c] = expf(s[c]); }
#pragma unroll
    for (int c = 0; c < 4; c++) q[c] = a.params[5][4 * (size_t)i + c];
    write_activated(a, i, s, e, q);
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" int h3dgs_coarse_param_step(const h3dgs_coarse_args* args, int32_t mode, void* stream)
{
    if (!args || args->N <= 0 || args->sh_coeffs < 1 || args->skybox_points < 0 ||
        (mode != H3DGS_COARSE_STEP && mode != H3DGS_COARSE_ACTIVATE && mode != H3DGS_COARSE_BIAS)) {
        set_error("coarse_param_step: bad arguments"); return H3DGS_EINVAL;
    }
    const h3dgs_coarse_args& a = *args;
    bool null = !a.means3D || !a.shs || !a.opacities || !a.scales || !a.rotations;
    for (int g = 0; g < 6; g++) null = null || (g != 2 && !a.params[g]);
    if (mode != H3DGS_COARSE_ACTIVATE) {
        null = null || !a.step || !a.scratch;
        if (mode == H3DGS_COARSE_STEP) {
            null = null || !a.grad_means3D || !a.grad_shs || !a.grad_opacities || !a.grad_scales || !a.grad_rotations;
            for (int g = 0; g < 6; g++) null = null || (a.params[g] && (!a.exp_avg[g] || !a.exp_avg_sq[g]));
        }
    }
    if (null || (a.sh_coeffs > 1 && !a.params[2])) { set_error("coarse_param_step: NULL pointer"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((a.N + 255) / 256);
    if (mode == H3DGS_COARSE_ACTIVATE) {
        coarse_activate_kernel<<<blocks, 256, 0, s>>>(a);
        H3_LAUNCHED("coarse_activate", 0, s);
        return H3DGS_OK;
    }
    CoarseConst k;
    for (int g = 0; g < 6; g++) {
        if (!(a.lr[g] >= 0.0) || !(a.beta1[g] >= 0.0 && a.beta1[g] < 1.0) || !(a.beta2[g] >= 0.0 && a.beta2[g] < 1.0) || !(a.eps[g] >= 0.0)) {
            set_error("coarse_param_step: bad hyper-parameter of group %d", g); return H3DGS_EINVAL;
        }
        k.beta1[g] = (float)a.beta1[g]; k.beta2[g] = (float)a.beta2[g];
        k.omb1[g] = (float)(1.0 - a.beta1[g]); k.omb2[g] = (float)(1.0 - a.beta2[g]);
        k.eps[g] = (float)a.eps[g];
        k.lr[g] = a.lr[g]; k.beta1d[g] = a.beta1[g]; k.beta2d[g] = a.beta2[g];
    }
    coarse_prologue_kernel<<<1, 1, 0, s>>>(a, k, mode == H3DGS_COARSE_STEP ? 1 : 0);
    H3_LAUNCHED("coarse_prologue", 0, s);
    if (mode == H3DGS_COARSE_BIAS) return H3DGS_OK;
    coarse_relevance_kernel<<<blocks, 256, 0, s>>>(a);
    H3_LAUNCHED("coarse_relevance", 0, s);
    coarse_update_kernel<<<blocks, 256, 0, s>>>(a, k);
    H3_LAUNCHED("coarse_update", 0, s);
    return H3DGS_OK;
}
