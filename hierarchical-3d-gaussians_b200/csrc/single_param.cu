// single_param.cu -- train_single's parameter side (train_single.py:85-88, 157-186) on the device: the exposure's
// torch.optim.Adam step, the skybox lock of all six stored gradients, the relevance rule of the flattened
// (_opacity.grad.flatten() != 0).nonzero(), OurAdam on the relevant rows with the xyz lr of this iteration, the
// big-Gaussian rescale past the scaffold and the activations the next forward reads.  Nothing returns to the host, and
// the learning rates are device words the host fills, so the pass can sit inside a CUDA graph that is never recaptured.
//
// The row-local arithmetic is train_coarse's (param_row.cuh).  Where train_single differs:
//   lock        skybox_locked: every stored gradient of rows < skybox_points is 0 (train_single.py:162-168), the
//               opacity's included, so a locked row is never relevant;
//   relevance   the flattened index lists exactly the rows whose stored opacity gradient is != 0 (NaN counts): no row
//               0 of an unflattened index.  With none, OurAdam takes its dense step on every row (_single_tensor_adam2);
//   lr          xyz: lrs[0], xyz_scheduler_args(iteration), set every iteration (update_learning_rate, :88);
//   rescale     rows >= scaffold_points, threshold float32(extent * 0.02) (:180-186);
//   exposure    torch.optim.Adam([_exposure]) over the whole [n_images,3,4] tensor (:159-160): the frame's image row
//               has its gradient, every other row a zero gradient, and all of them move as their moments decay.  Its
//               arithmetic is that of torch's default CUDA path (adam.cuh's torch_adam_element), with the bias
//               corrections formed in double from the step count (torch's Python floats of the host step count;
//               torch.optim.Adam(capturable=True) would form them from a device fp32 step with fp32 pow instead).
// Launches: a one-thread prologue (step counts, bias corrections of both optimizers, the any-relevant word cleared),
// the exposure Adam, for a full step the relevance pass, an element-parallel pass over f_rest and the row-local update
// pass (train_coarse's, without f_rest); without the Gaussian step the update pass only rescales.
// An overflowed capacity-mode frame (scan_info[2]) changes nothing.
#include "common.cuh"
#include "param_row.cuh"

namespace h3dgs {

struct SingleScratch { CoarseScratch g; float exp_step_size, exp_bc2_sqrt; };
static_assert(sizeof(SingleScratch) <= H3DGS_SINGLE_SCRATCH_BYTES, "scratch");

struct ExposureConst { float w, beta2, omb2, eps; double beta1d, beta2d; };

__device__ __forceinline__ bool overflowed(const h3dgs_single_args& a) { return a.gauss.scan_info && a.gauss.scan_info[2]; }

// mode H3DGS_SINGLE_STEP / _BIAS: the Gaussian step's count and bias corrections (xyz lr from the device word);
// every mode but _EXPOSURE_ROW: the exposure's.  _BIAS counts nothing
__global__ void single_prologue_kernel(h3dgs_single_args a, CoarseConst k, ExposureConst x, int mode)
{
    if (overflowed(a)) return;
    SingleScratch* sc = (SingleScratch*)a.gauss.scratch;
    const bool count = mode != H3DGS_SINGLE_BIAS;
    if (mode != H3DGS_SINGLE_NO_GAUSSIAN_STEP) {
        const double step = (double)(*a.gauss.step + 1);
        if (count) *a.gauss.step += 1;
        for (int g = 0; g < 6; g++)
            bias_corrections(g == 0 ? a.lrs[0] : k.lr[g], k.beta1d[g], k.beta2d[g], step, sc->g.step_size[g], sc->g.bc2_sqrt[g]);
        sc->g.any = 0;
    }
    const double t = (double)(*a.exposure_step + 1);
    if (count) *a.exposure_step += 1;
    const double bc1 = 1.0 - pow(x.beta1d, t), bc2 = 1.0 - pow(x.beta2d, t);
    sc->exp_step_size = (float)(-(a.lrs[1] / bc1));
    sc->exp_bc2_sqrt = (float)sqrt(bc2);
}

__global__ void __launch_bounds__(256) single_exposure_adam_kernel(h3dgs_single_args a, ExposureConst x)
{
    const int e = blockIdx.x * 256 + threadIdx.x;
    if (e >= a.n_images * 12 || overflowed(a)) return;
    const SingleScratch& sc = *(const SingleScratch*)a.gauss.scratch;
    const float g = (e / 12 == *a.image_index) ? a.exposure_grad[e % 12] : 0.f;
    float p = a.exposure[e], m = a.exposure_exp_avg[e], v = a.exposure_exp_avg_sq[e];
    torch_adam_element(p, g, m, v, x.w, x.beta2, x.omb2, sc.exp_step_size, sc.exp_bc2_sqrt, x.eps);
    a.exposure[e] = p;
    a.exposure_exp_avg[e] = m;
    a.exposure_exp_avg_sq[e] = v;
}

__device__ __forceinline__ float locked_opacity_grad(const h3dgs_single_args& a, int i, bool& locked)
{
    locked = a.skybox_locked && i < a.gauss.skybox_points;
    return locked ? 0.f : stored_opacity_grad(a.gauss, i);
}

__global__ void __launch_bounds__(256) single_relevance_kernel(h3dgs_single_args a)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= a.gauss.N || overflowed(a)) return;
    bool locked;
    if (locked_opacity_grad(a, i, locked) != 0.f) ((SingleScratch*)a.gauss.scratch)->g.any = 1;
}

// step: Adam on OurAdam's row set (the relevant rows; every row when there is none), then the rescale and the
// activations.  !step: the rescale and the activations of the rescaled rows only
__global__ void __launch_bounds__(256) single_update_kernel(h3dgs_single_args a, CoarseConst k, int step)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= a.gauss.N || overflowed(a)) return;
    bool update = false;
    if (step) {
        const SingleScratch& sc = *(const SingleScratch*)a.gauss.scratch;
        bool locked;
        const float go = locked_opacity_grad(a, i, locked);
        update = sc.g.any ? go != 0.f : true;
        if (update) adam_row(a.gauss, k, sc.g, i, go, false, locked, false);
    }
    rescale_and_activate(a.gauss, i, update, a.scaffold_points, false);
}

// the f_rest group (45 of a degree-3 row's 59 stored floats) one element per thread, so that a warp's accesses are
// contiguous: Adam on OurAdam's row set, and its activated copy in shs.  Its values are the row pass's: the element
// order does not enter the arithmetic
__global__ void __launch_bounds__(256) single_rest_kernel(h3dgs_single_args a, CoarseConst k)
{
    const size_t R = (size_t)a.gauss.sh_coeffs * 3 - 3, e = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= (size_t)a.gauss.N * R || overflowed(a)) return;
    const SingleScratch& sc = *(const SingleScratch*)a.gauss.scratch;
    const int i = (int)(e / R);
    bool locked;
    const float go = locked_opacity_grad(a, i, locked);
    if (!(sc.g.any ? go != 0.f : true)) return;
    const size_t o = (R + 3) * i + 3 + (e - R * i);
    adam_at(a.gauss, k, sc.g, 2, e, locked ? 0.f : a.gauss.grad_shs[o]);
    a.gauss.shs[o] = a.gauss.params[2][e];
}

__global__ void single_exposure_row_kernel(h3dgs_single_args a)
{
    const int c = threadIdx.x, r = *a.image_index;
    if (c < 12 && r >= 0 && r < a.n_images) a.exposure_row[c] = a.exposure[12 * (size_t)r + c];
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" int h3dgs_single_param_step(const h3dgs_single_args* args, int32_t mode, void* stream)
{
    if (!args || mode < H3DGS_SINGLE_STEP || mode > H3DGS_SINGLE_BIAS) { set_error("single_param_step: bad arguments"); return H3DGS_EINVAL; }
    const h3dgs_single_args& a = *args;
    const h3dgs_coarse_args& b = a.gauss;
    cudaStream_t s = (cudaStream_t)stream;
    if (a.n_images <= 0 || !a.exposure || !a.image_index) { set_error("single_param_step: no exposures"); return H3DGS_EINVAL; }
    if (mode == H3DGS_SINGLE_EXPOSURE_ROW) {
        if (!a.exposure_row) { set_error("single_param_step: NULL exposure_row"); return H3DGS_EINVAL; }
        single_exposure_row_kernel<<<1, 32, 0, s>>>(a);
        H3_LAUNCHED("single_exposure_row", 0, s);
        return H3DGS_OK;
    }
    if (b.N <= 0 || b.sh_coeffs < 1 || b.skybox_points < 0 || a.scaffold_points < 0) {
        set_error("single_param_step: bad sizes"); return H3DGS_EINVAL;
    }
    bool null = !a.lrs || !a.exposure_exp_avg || !a.exposure_exp_avg_sq || !a.exposure_step || !a.exposure_grad || !b.scratch;
    null = null || !b.means3D || !b.shs || !b.opacities || !b.scales || !b.rotations;
    for (int g = 0; g < 6; g++) null = null || (g != 2 && !b.params[g]);
    if (mode != H3DGS_SINGLE_NO_GAUSSIAN_STEP) {
        null = null || !b.step;
        if (mode == H3DGS_SINGLE_STEP) {
            null = null || !b.grad_means3D || !b.grad_shs || !b.grad_opacities || !b.grad_scales || !b.grad_rotations;
            for (int g = 0; g < 6; g++) null = null || (b.params[g] && (!b.exp_avg[g] || !b.exp_avg_sq[g]));
        }
    }
    if (null || (b.sh_coeffs > 1 && !b.params[2])) { set_error("single_param_step: NULL pointer"); return H3DGS_EINVAL; }
    CoarseConst k;
    for (int g = 0; g < 6; g++) {
        if ((g > 0 && !(b.lr[g] >= 0.0)) || !(b.beta1[g] >= 0.0 && b.beta1[g] < 1.0) || !(b.beta2[g] >= 0.0 && b.beta2[g] < 1.0) ||
            !(b.eps[g] >= 0.0)) {
            set_error("single_param_step: bad hyper-parameter of group %d", g); return H3DGS_EINVAL;
        }
        k.beta1[g] = (float)b.beta1[g]; k.beta2[g] = (float)b.beta2[g];
        k.omb1[g] = (float)(1.0 - b.beta1[g]); k.omb2[g] = (float)(1.0 - b.beta2[g]);
        k.eps[g] = (float)b.eps[g];
        k.lr[g] = b.lr[g]; k.beta1d[g] = b.beta1[g]; k.beta2d[g] = b.beta2[g];
    }
    if (!(a.exposure_beta1 >= 0.0 && a.exposure_beta1 < 1.0) || !(a.exposure_beta2 >= 0.0 && a.exposure_beta2 < 1.0) ||
        !(a.exposure_eps >= 0.0)) {
        set_error("single_param_step: bad exposure hyper-parameter"); return H3DGS_EINVAL;
    }
    ExposureConst x;
    x.w = (float)(1.0 - a.exposure_beta1); x.beta2 = (float)a.exposure_beta2; x.omb2 = (float)(1.0 - a.exposure_beta2);
    x.eps = (float)a.exposure_eps; x.beta1d = a.exposure_beta1; x.beta2d = a.exposure_beta2;
    single_prologue_kernel<<<1, 1, 0, s>>>(a, k, x, mode);
    H3_LAUNCHED("single_prologue", 0, s);
    if (mode == H3DGS_SINGLE_BIAS) return H3DGS_OK;
    single_exposure_adam_kernel<<<(unsigned)((a.n_images * 12 + 255) / 256), 256, 0, s>>>(a, x);
    H3_LAUNCHED("single_exposure_adam", 0, s);
    const unsigned blocks = (unsigned)((b.N + 255) / 256);
    const int step = mode == H3DGS_SINGLE_STEP;
    if (step) {
        single_relevance_kernel<<<blocks, 256, 0, s>>>(a);
        H3_LAUNCHED("single_relevance", 0, s);
    }
    if (step && b.sh_coeffs > 1) {           // before the update pass, which rewrites the activated opacities it reads
        single_rest_kernel<<<(unsigned)(((size_t)b.N * (b.sh_coeffs * 3 - 3) + 255) / 256), 256, 0, s>>>(a, k);
        H3_LAUNCHED("single_rest", 0, s);
    }
    single_update_kernel<<<blocks, 256, 0, s>>>(a, k, step);
    H3_LAUNCHED("single_update", 0, s);
    return H3DGS_OK;
}
