// densify.cu -- train_single's densify_and_prune and reset_opacity (scene/gaussian_model.py:510-514, 543-685) on the
// device state: the six stored tensors and their OurAdam moments, read from the old buffers and written once into new
// ones in the reference's final row order
//   [kept originals, in index order | clones | first split copy of each split row | second split copy].
// That is the order of its two appends (clone, split) and two prunes (the split originals, then opacity < min_opacity):
// clones and split copies both need sigmoid(o) > 0.15, and min_opacity <= 0.15 is the caller's promise, so the second
// prune only ever removes originals.
//
// COUNT: one thread per original row decides keep / clone / split into flags[i]; one inclusive scan over
//        [keep flags | clone flags | split flags] (3N int32) numbers the output rows directly: a kept row lands at
//        scan[i] - 1, a clone at scan[N + i] - 1 (K kept rows precede it), a split row's first copy at
//        scan[2N + i] - 1 and its second S rows later; a one-thread tail stores {K, C, S, N'}.
// WRITE: a row pass (xyz, f_dc, opacity, scaling, rotation and their moments) and an element-parallel pass over
//        f_rest (45 of a degree-3 row's 59 floats), so that a warp's accesses are contiguous.
// RESET: opacity rows >= skybox_points in place, both opacity moments zeroed on every row.
// Every product, quotient and sum is rounded on its own (no FMA), left to right as torch evaluates the Python lines;
// expf / logf / powf are the CUDA math library's accurate ones, as torch's exp / log / pow.
#include <cub/cub.cuh>
#include "common.cuh"
#include "param_row.cuh"

namespace h3dgs {
namespace {

constexpr uint8_t kKeep = 1, kClone = 2, kSplit = 4;

struct DensifyLayout { size_t counts, scan, temp, temp_bytes, total; };

DensifyLayout densify_layout(int N)
{
    DensifyLayout l;
    size_t o = 0, t = 0;
    cub::DeviceScan::InclusiveSum(nullptr, t, (const int32_t*)nullptr, (int32_t*)nullptr, 3 * N > 0 ? 3 * N : 1);
    l.temp_bytes = t;
    l.counts = o; o += align_up(4 * sizeof(int32_t));
    l.scan = o;   o += align_up((size_t)3 * N * sizeof(int32_t));
    l.temp = o;   o += align_up(t);
    l.total = o;
    return l;
}

__device__ __forceinline__ float max3_nan(const float e[3])
{
    float mx = e[0];                                  // torch.max(dim=1): NaN propagates
#pragma unroll
    for (int c = 1; c < 3; c++) mx = (mx != mx) ? mx : ((e[c] != e[c] || e[c] > mx) ? e[c] : mx);
    return mx;
}

__global__ void __launch_bounds__(256) densify_decide_kernel(h3dgs_densify_args a, int32_t* scan)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    const int N = a.N;
    if (i >= N) return;
    uint8_t f = kKeep;
    if (i >= a.scaffold_points) {
        float g = a.xyz_gradient_accum[i];
        if (g != g) g = 0.f;                          // grads[grads.isnan()] = 0.0
        const float r = a.max_radii2D[i];
        const float o = sigmoid_f(a.params[3][i]);
        const float p = powf(o, 0.2f);
        float e[3];
#pragma unroll
        for (int c = 0; c < 3; c++) e[c] = expf(a.params[4][3 * (size_t)i + c]);
        const float mx = max3_nan(e);
        const bool bright = o > 0.15f;
        // densify_and_clone: torch.norm over a dimension of size 1 is sqrt(g * g), which under- and overflows
        const float gn = __fsqrt_rn(__fmul_rn(g, g));
        const bool clone = __fmul_rn(__fmul_rn(gn, r), p) >= a.max_grad && bright && mx <= a.size_threshold;
        const bool split = __fmul_rn(__fmul_rn(g, r), p) >= a.max_grad && bright && mx > a.size_threshold;
        f = (split ? 0 : ((o < a.min_opacity) ? 0 : kKeep)) | (clone ? kClone : 0) | (split ? kSplit : 0);
    }
    a.flags[i] = f;
    scan[i] = f & kKeep;
    scan[(size_t)N + i] = (f & kClone) ? 1 : 0;
    scan[2 * (size_t)N + i] = (f & kSplit) ? 1 : 0;
}

__global__ void densify_counts_kernel(int N, const int32_t* scan, int32_t* counts)
{
    const int32_t K = N ? scan[N - 1] : 0, KC = N ? scan[2 * (size_t)N - 1] : 0, KCS = N ? scan[3 * (size_t)N - 1] : 0;
    const int64_t n_out = (int64_t)KCS + (KCS - KC);
    counts[0] = K;
    counts[1] = KC - K;
    counts[2] = KCS - KC;
    counts[3] = n_out > 0x7fffffff ? -1 : (int32_t)n_out;
}

// build_rotation (utils/general_utils.py:82-103) of the stored quaternion, element by element as torch evaluates it
__device__ __forceinline__ void build_rotation(const float r[4], float R[9])
{
    const float n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], r[0]), __fmul_rn(r[1], r[1])),
                                                   __fmul_rn(r[2], r[2])), __fmul_rn(r[3], r[3])));
    const float w = __fdiv_rn(r[0], n), x = __fdiv_rn(r[1], n), y = __fdiv_rn(r[2], n), z = __fdiv_rn(r[3], n);
    const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
    const float xy = __fmul_rn(x, y), xz = __fmul_rn(x, z), yz = __fmul_rn(y, z);
    const float wx = __fmul_rn(w, x), wy = __fmul_rn(w, y), wz = __fmul_rn(w, z);
    R[0] = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(yy, zz)));
    R[1] = __fmul_rn(2.f, __fsub_rn(xy, wz));
    R[2] = __fmul_rn(2.f, __fadd_rn(xz, wy));
    R[3] = __fmul_rn(2.f, __fadd_rn(xy, wz));
    R[4] = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(xx, zz)));
    R[5] = __fmul_rn(2.f, __fsub_rn(yz, wx));
    R[6] = __fmul_rn(2.f, __fsub_rn(xz, wy));
    R[7] = __fmul_rn(2.f, __fadd_rn(yz, wx));
    R[8] = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(xx, yy)));
}

// the row groups other than f_rest: 0 xyz (3), 1 f_dc (3), 3 opacity (1), 4 scaling (3), 5 rotation (4)
__device__ __forceinline__ int group_width(int g) { return g == 3 ? 1 : (g == 5 ? 4 : 3); }

__device__ __forceinline__ void copy_row(const h3dgs_densify_args& a, int g, int src, int64_t dst, bool moments)
{
    const int w = group_width(g);
    for (int c = 0; c < w; c++) {
        a.out_params[g][w * dst + c] = a.params[g][(size_t)w * src + c];
        a.out_exp_avg[g][w * dst + c] = moments ? a.exp_avg[g][(size_t)w * src + c] : 0.f;
        a.out_exp_avg_sq[g][w * dst + c] = moments ? a.exp_avg_sq[g][(size_t)w * src + c] : 0.f;
    }
}

__device__ __forceinline__ void zero_moments(const h3dgs_densify_args& a, int g, int64_t dst)
{
    const int w = group_width(g);
    for (int c = 0; c < w; c++) a.out_exp_avg[g][w * dst + c] = a.out_exp_avg_sq[g][w * dst + c] = 0.f;
}

// densify_and_split's copy k of row i (copy 0 at dst, normals row j): xyz + bmm(R, z * exp(s) + 0), the 3x3 product
// summed in the order of its columns; scaling log(exp(s) * (1 / 1.6f)) (torch's CUDA division by the Python scalar 0.8 * 2
// multiplies by the fp32 reciprocal); rotation, both feature groups and opacity copied; moments zero
__device__ __forceinline__ void split_row(const h3dgs_densify_args& a, int i, int64_t dst, int64_t j, const float R[9],
                                          const float e[3])
{
    float smp[3];
#pragma unroll
    for (int c = 0; c < 3; c++) smp[c] = __fadd_rn(__fmul_rn(a.normals[3 * j + c], e[c]), 0.f);
    const float inv = __fdiv_rn(1.f, 1.6f);
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float d = __fadd_rn(__fadd_rn(__fmul_rn(R[3 * c], smp[0]), __fmul_rn(R[3 * c + 1], smp[1])),
                                  __fmul_rn(R[3 * c + 2], smp[2]));
        a.out_params[0][3 * dst + c] = __fadd_rn(d, a.params[0][3 * (size_t)i + c]);
        a.out_params[4][3 * dst + c] = logf(__fmul_rn(e[c], inv));
    }
    zero_moments(a, 0, dst);
    zero_moments(a, 4, dst);
    copy_row(a, 1, i, dst, false);
    copy_row(a, 3, i, dst, false);
    copy_row(a, 5, i, dst, false);
}

__global__ void __launch_bounds__(256) densify_row_kernel(h3dgs_densify_args a, const int32_t* scan, const int32_t* counts)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    const int N = a.N;
    if (i >= N) return;
    const uint8_t f = a.flags[i];
    if (f & kKeep) {
        const int64_t d = scan[i] - 1;
        for (int g = 0; g < 6; g++)
            if (g != 2) copy_row(a, g, i, d, true);
    }
    if (f & kClone) {
        const int64_t d = scan[(size_t)N + i] - 1;
        for (int g = 0; g < 6; g++)
            if (g != 2) copy_row(a, g, i, d, false);
    }
    if (f & kSplit) {
        const int32_t KC = counts[0] + counts[1], S = counts[2];
        const int64_t d = scan[2 * (size_t)N + i] - 1, k = d - KC;
        float q[4], R[9], e[3];
#pragma unroll
        for (int c = 0; c < 4; c++) q[c] = a.params[5][4 * (size_t)i + c];
        build_rotation(q, R);
#pragma unroll
        for (int c = 0; c < 3; c++) e[c] = expf(a.params[4][3 * (size_t)i + c]);
        split_row(a, i, d, k, R, e);
        split_row(a, i, d + S, S + k, R, e);
    }
}

// f_rest one element per thread: kept rows with their moments, clones and both split copies with zero moments
__global__ void __launch_bounds__(256) densify_rest_kernel(h3dgs_densify_args a, const int32_t* scan, const int32_t* counts)
{
    const size_t R = (size_t)a.sh_coeffs * 3 - 3, e = (size_t)blockIdx.x * 256 + threadIdx.x;
    const int N = a.N;
    if (e >= (size_t)N * R) return;
    const int i = (int)(e / R);
    const size_t j = e - R * i;
    const uint8_t f = a.flags[i];
    const float p = a.params[2][e];
    if (f & kKeep) {
        const size_t o = R * (size_t)(scan[i] - 1) + j;
        a.out_params[2][o] = p;
        a.out_exp_avg[2][o] = a.exp_avg[2][e];
        a.out_exp_avg_sq[2][o] = a.exp_avg_sq[2][e];
    }
    int64_t d[2];
    int n = 0;
    if (f & kClone) d[n++] = scan[(size_t)N + i] - 1;
    if (f & kSplit) {
        d[0] = scan[2 * (size_t)N + i] - 1;
        d[1] = d[0] + counts[2];
        n = 2;
    }
    for (int k = 0; k < n; k++) {
        const size_t o = R * (size_t)d[k] + j;
        a.out_params[2][o] = p;
        a.out_exp_avg[2][o] = a.out_exp_avg_sq[2][o] = 0.f;
    }
}

// reset_opacity: inverse_sigmoid(min(sigmoid(o), 0.01)) = log(x / (1 - x)) past the skybox (torch.min propagates NaN);
// replace_tensor_to_optimizer zeroes both opacity moments of every row
__global__ void __launch_bounds__(256) reset_opacity_kernel(h3dgs_densify_args a)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= a.N) return;
    if (i >= a.skybox_points) {
        float x = sigmoid_f(a.params[3][i]);
        x = (x != x || x < 0.01f) ? x : 0.01f;
        a.params[3][i] = logf(__fdiv_rn(x, __fsub_rn(1.f, x)));
    }
    a.exp_avg[3][i] = 0.f;
    a.exp_avg_sq[3][i] = 0.f;
}

}  // namespace
}  // namespace h3dgs

using namespace h3dgs;

extern "C" size_t h3dgs_densify_scratch_bytes(int32_t N)
{
    if (N < 0 || (int64_t)N * 3 > 0x7fffffff) return 0;
    return densify_layout(N).total;
}

extern "C" int h3dgs_densify(const h3dgs_densify_args* args, int32_t mode, void* stream)
{
    if (!args || mode < H3DGS_DENSIFY_COUNT || mode > H3DGS_DENSIFY_RESET_OPACITY) {
        set_error("densify: bad arguments"); return H3DGS_EINVAL;
    }
    const h3dgs_densify_args& a = *args;
    cudaStream_t s = (cudaStream_t)stream;
    if (a.N < 0 || (int64_t)a.N * 3 > 0x7fffffff || a.sh_coeffs < 1 || a.scaffold_points < 0 || a.skybox_points < 0) {
        set_error("densify: bad sizes"); return H3DGS_EINVAL;
    }
    bool null = false;
    for (int g = 0; g < 6; g++) null = null || (g != 2 && (!a.params[g] || !a.exp_avg[g] || !a.exp_avg_sq[g]));
    if (mode == H3DGS_DENSIFY_RESET_OPACITY) {
        if (null) { set_error("densify: NULL pointer"); return H3DGS_EINVAL; }
        if (a.N == 0) return H3DGS_OK;
        reset_opacity_kernel<<<(unsigned)((a.N + 255) / 256), 256, 0, s>>>(a);
        H3_LAUNCHED("reset_opacity", 0, s);
        return H3DGS_OK;
    }
    null = null || !a.flags || !a.scratch || (a.sh_coeffs > 1 && (!a.params[2] || !a.exp_avg[2] || !a.exp_avg_sq[2]));
    if (((uintptr_t)a.scratch & 255) != 0) { set_error("densify: scratch is not 256-byte aligned"); return H3DGS_EINVAL; }
    const DensifyLayout l = densify_layout(a.N);
    char* sc = (char*)a.scratch;
    int32_t* counts = (int32_t*)(sc + l.counts);
    int32_t* scan = (int32_t*)(sc + l.scan);
    if (mode == H3DGS_DENSIFY_COUNT) {
        null = null || !a.xyz_gradient_accum || !a.max_radii2D;
        if (null) { set_error("densify: NULL pointer"); return H3DGS_EINVAL; }
        if (!(a.max_grad > 0.f) || !(a.min_opacity <= 0.15f)) {
            set_error("densify: need max_grad > 0 and min_opacity <= 0.15 (so that no clone or split copy is pruned)");
            return H3DGS_EINVAL;
        }
        if (a.N > 0) {
            densify_decide_kernel<<<(unsigned)((a.N + 255) / 256), 256, 0, s>>>(a, scan);
            H3_LAUNCHED("densify_decide", 0, s);
            size_t tb = l.temp_bytes;
            H3_CUDA(cub::DeviceScan::InclusiveSum(sc + l.temp, tb, scan, scan, 3 * a.N, s));
        }
        densify_counts_kernel<<<1, 1, 0, s>>>(a.N, scan, counts);
        H3_LAUNCHED("densify_counts", 0, s);
        return H3DGS_OK;
    }
    // H3DGS_DENSIFY_WRITE
    for (int g = 0; g < 6; g++)
        null = null || (g != 2 && (!a.out_params[g] || !a.out_exp_avg[g] || !a.out_exp_avg_sq[g]));
    null = null || (a.sh_coeffs > 1 && (!a.out_params[2] || !a.out_exp_avg[2] || !a.out_exp_avg_sq[2]));
    if (null || (a.split_rows > 0 && !a.normals)) { set_error("densify: NULL pointer"); return H3DGS_EINVAL; }
    if (a.out_rows < 0 || a.out_rows > 0x7fffffffLL || a.split_rows < 0 || 2 * (int64_t)a.split_rows > a.out_rows) {
        set_error("densify: %lld output rows (%d split) do not fit int32", (long long)a.out_rows, a.split_rows);
        return H3DGS_EINVAL;
    }
    if (a.N == 0) return H3DGS_OK;
    densify_row_kernel<<<(unsigned)((a.N + 255) / 256), 256, 0, s>>>(a, scan, counts);
    H3_LAUNCHED("densify_rows", 0, s);
    if (a.sh_coeffs > 1) {
        densify_rest_kernel<<<(unsigned)(((size_t)a.N * (a.sh_coeffs * 3 - 3) + 255) / 256), 256, 0, s>>>(a, scan, counts);
        H3_LAUNCHED("densify_rest", 0, s);
    }
    return H3DGS_OK;
}
