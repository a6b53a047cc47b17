// post_param.cu -- train_post's parameter side (train_post.py:85, 165-192) on the device: the activations' backward of
// a create_from_hier model, the skybox and anchor locks, torch.optim.Adam's dense step over every element of every row
// with this iteration's xyz lr, and the activations the next forward reads.  Nothing returns to the host and the xyz lr
// is a device word, so the pass sits at the end of a CUDA graph that is captured once for the whole run.
//
// Where train_post differs from train_coarse and train_single (coarse_param.cu, single_param.cu):
//   opacity     get_opacity = torch.abs (create_from_hier, scene/gaussian_model.py:393), whose backward is
//               g * sign(o) with sign(+-0) = sign(NaN) = 0 ((0 < o) - (o < 0), as torch's CUDA sign), the product
//               rounded as torch's mul; the activated value is fabsf(o);
//   lock        all six stored gradients are 0 on the rows of `locked` (the anchors, and the skybox tail when
//               skybox_locked, train_post.py:167-181); a locked row is still stepped, with g = 0;
//   optimizer   torch.optim.Adam (training_setup(our_adam=False)), DENSE: every element moves, the rows outside this
//               frame's cut with a zero gradient as their moments decay.  Its arithmetic is adam.cuh's
//               torch_adam_element, the bias corrections formed in double from the device step count;
//   no rescale, no relevance rule, no densification.
// Launches: a one-thread prologue, which alone decides whether the frame overflowed (scan_info[2], or the cut plus the
// skybox rows past row_capacity: a row overflow is seen by no other kernel, and the frame still has gradients) and
// stores that decision in scratch, counts the step and forms the six groups' step sizes and sqrt(bc2); then one
// element-parallel pass over the stored floats of xyz, f_dc, f_rest, opacity and scaling (consecutive threads,
// consecutive elements of one group) followed by the rotation rows, one row per thread (its normalize backward needs
// the whole quaternion).  Every thread reads the prologue's decision: an overflowed frame changes no byte of state.
#include "common.cuh"
#include "param_row.cuh"

namespace h3dgs {

struct PostScratch { float step_size[6], bc2_sqrt[6]; int skip; };
static_assert(sizeof(PostScratch) <= H3DGS_POST_SCRATCH_BYTES, "scratch");

struct PostConst { float w[6], beta2[6], omb2[6], eps[6]; double lr[6], beta1d[6], beta2d[6]; };

__global__ void post_prologue_kernel(h3dgs_post_args a, PostConst k, int count)
{
    PostScratch* sc = (PostScratch*)a.gauss.scratch;
    const bool skip = (a.gauss.scan_info && a.gauss.scan_info[2]) ||
                      (a.count && (int64_t)*a.count + a.extra_rows > (int64_t)a.row_capacity);
    sc->skip = skip ? 1 : 0;
    if (skip) return;
    const double t = (double)(*a.gauss.step + 1);
    if (count) *a.gauss.step += 1;
    for (int g = 0; g < 6; g++) {
        const double bc1 = 1.0 - pow(k.beta1d[g], t), bc2 = 1.0 - pow(k.beta2d[g], t);
        sc->step_size[g] = (float)(-((g == 0 ? *a.lrs : k.lr[g]) / bc1));
        sc->bc2_sqrt[g] = (float)sqrt(bc2);
    }
}

__device__ __forceinline__ float sign_f(float x) { return (float)((0.f < x) - (x < 0.f)); }

// one stored element: the stored gradient g (already locked), Adam, and the element's new value
__device__ __forceinline__ float post_adam(const h3dgs_post_args& a, const PostConst& k, const PostScratch* sc, int grp,
                                           size_t o, float g)
{
    float p = a.gauss.params[grp][o], m = a.gauss.exp_avg[grp][o], v = a.gauss.exp_avg_sq[grp][o];
    torch_adam_element(p, g, m, v, k.w[grp], k.beta2[grp], k.omb2[grp], sc->step_size[grp], sc->bc2_sqrt[grp],
                       k.eps[grp]);
    a.gauss.params[grp][o] = p;
    a.gauss.exp_avg[grp][o] = m;
    a.gauss.exp_avg_sq[grp][o] = v;
    return p;
}

// index space: [0, 3N) xyz, [3N, 6N) f_dc, then R N f_rest (R = 3 (sh_coeffs - 1)), N opacity, 3N scaling, then N
// rotation rows.  step = 0 (H3DGS_POST_ACTIVATE): the activations only
__global__ void __launch_bounds__(256) post_param_kernel(h3dgs_post_args a, PostConst k, int step)
{
    const h3dgs_coarse_args& b = a.gauss;
    const size_t N = (size_t)b.N, M3 = (size_t)b.sh_coeffs * 3, R = M3 - 3;
    size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= (11 + R) * N) return;                                  // (10 + R) N elements, N rotation rows
    const PostScratch* sc = (const PostScratch*)b.scratch;         // read only when step
    if (step && sc->skip) return;
    if (e < 6 * N) {                                                // xyz, f_dc
        const int grp = e < 3 * N ? 0 : 1;
        if (grp) e -= 3 * N;
        const size_t i = e / 3, c = e - 3 * i, o = grp ? M3 * i + c : e;
        float p = b.params[grp][e];
        if (step)
            p = post_adam(a, k, sc, grp, e, (a.locked && a.locked[i]) ? 0.f : (grp ? b.grad_shs[o] : b.grad_means3D[o]));
        (grp ? b.shs : b.means3D)[o] = p;
        return;
    }
    e -= 6 * N;
    if (e < R * N) {                                                // f_rest
        const size_t i = e / R, o = M3 * i + 3 + (e - R * i);
        float p = b.params[2][e];
        if (step) p = post_adam(a, k, sc, 2, e, (a.locked && a.locked[i]) ? 0.f : b.grad_shs[o]);
        b.shs[o] = p;
        return;
    }
    e -= R * N;
    if (e < N) {                                                    // opacity: abs
        float p = b.params[3][e];
        if (step) p = post_adam(a, k, sc, 3, e, (a.locked && a.locked[e]) ? 0.f : __fmul_rn(b.grad_opacities[e], sign_f(p)));
        b.opacities[e] = fabsf(p);
        return;
    }
    e -= N;
    if (e < 3 * N) {                                                // scaling: exp, backward g * exp(s) on the activated row
        float p = b.params[4][e];
        if (step) p = post_adam(a, k, sc, 4, e, (a.locked && a.locked[e / 3]) ? 0.f : __fmul_rn(b.grad_scales[e], b.scales[e]));
        b.scales[e] = expf(p);
        return;
    }
    const size_t i = e - 3 * N;                                     // rotation row i: F.normalize
    float q[4];
#pragma unroll
    for (int c = 0; c < 4; c++) q[c] = b.params[5][4 * i + c];
    if (step) {
        float g[4];
        const bool locked = a.locked && a.locked[i];
#pragma unroll
        for (int c = 0; c < 4; c++) g[c] = b.grad_rotations[4 * i + c];
        normalize_backward(q, g);
#pragma unroll
        for (int c = 0; c < 4; c++) q[c] = post_adam(a, k, sc, 5, 4 * i + c, locked ? 0.f : g[c]);
    }
    float n, d;
    quat_norm(q, n, d);
#pragma unroll
    for (int c = 0; c < 4; c++) b.rotations[4 * i + c] = __fdiv_rn(q[c], d);
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" int h3dgs_post_param_step(const h3dgs_post_args* args, int32_t mode, void* stream)
{
    if (!args || (mode != H3DGS_POST_STEP && mode != H3DGS_POST_ACTIVATE && mode != H3DGS_POST_BIAS)) {
        set_error("post_param_step: bad arguments"); return H3DGS_EINVAL;
    }
    const h3dgs_post_args& a = *args;
    const h3dgs_coarse_args& b = a.gauss;
    if (b.N <= 0 || b.sh_coeffs < 1 || (a.count && (a.extra_rows < 0 || a.row_capacity <= 0))) {
        set_error("post_param_step: bad sizes"); return H3DGS_EINVAL;
    }
    bool null = !b.means3D || !b.shs || !b.opacities || !b.scales || !b.rotations;
    for (int g = 0; g < 6; g++) null = null || (g != 2 && !b.params[g]);
    if (mode != H3DGS_POST_ACTIVATE) {
        null = null || !b.step || !b.scratch || !a.lrs;
        if (mode == H3DGS_POST_STEP) {
            null = null || !b.grad_means3D || !b.grad_shs || !b.grad_opacities || !b.grad_scales || !b.grad_rotations;
            for (int g = 0; g < 6; g++) null = null || (b.params[g] && (!b.exp_avg[g] || !b.exp_avg_sq[g]));
        }
    }
    if (null || (b.sh_coeffs > 1 && !b.params[2])) { set_error("post_param_step: NULL pointer"); return H3DGS_EINVAL; }
    PostConst k;
    for (int g = 0; g < 6; g++) {
        if ((g > 0 && !(b.lr[g] >= 0.0)) || !(b.beta1[g] >= 0.0 && b.beta1[g] < 1.0) || !(b.beta2[g] >= 0.0 && b.beta2[g] < 1.0) ||
            !(b.eps[g] >= 0.0)) {
            set_error("post_param_step: bad hyper-parameter of group %d", g); return H3DGS_EINVAL;
        }
        k.w[g] = (float)(1.0 - b.beta1[g]); k.beta2[g] = (float)b.beta2[g]; k.omb2[g] = (float)(1.0 - b.beta2[g]);
        k.eps[g] = (float)b.eps[g];
        k.lr[g] = b.lr[g]; k.beta1d[g] = b.beta1[g]; k.beta2d[g] = b.beta2[g];
    }
    cudaStream_t s = (cudaStream_t)stream;
    if (mode != H3DGS_POST_ACTIVATE) {
        post_prologue_kernel<<<1, 1, 0, s>>>(a, k, mode == H3DGS_POST_STEP ? 1 : 0);
        H3_LAUNCHED("post_prologue", 0, s);
        if (mode == H3DGS_POST_BIAS) return H3DGS_OK;
    }
    const size_t work = (size_t)b.N * (11 + 3 * (size_t)(b.sh_coeffs - 1));
    post_param_kernel<<<(unsigned)((work + 255) / 256), 256, 0, s>>>(a, k, mode == H3DGS_POST_STEP ? 1 : 0);
    H3_LAUNCHED("post_param", 0, s);
    return H3DGS_OK;
}
