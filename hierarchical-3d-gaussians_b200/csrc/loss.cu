// loss.cu -- fused L1 + SSIM loss, forward and backward (SURVEY.md 8f-2: the step either side of the
// rasterizer in train_post.py:134-142 / train_single.py:101-117).  Semantics = the reference's
// utils/loss_utils.py:17-63 (11x11 Gaussian window, sigma 1.5, zero padding, groups = channels,
// C1 = 0.01^2, C2 = 0.03^2), pinned by golden fixtures generated from that file (tests/golden/loss_*.npz).
//
// The reference runs 5 grouped conv2d (121 taps) + ~20 elementwise kernels forward and their autograd
// backward.  Here: ONE kernel forward (separable 11+11 taps in shared memory, 16x16 output tiles with a
// 5-pixel halo, all five moments at once, SSIM + L1 partial sums, and the three derivative maps the
// backward needs) and ONE kernel backward (the three maps convolved with the same window and combined
// with img / gt per pixel).  The 11 window weights travel as a by-value kernel argument, as in metrics.cu: no
// __constant__ upload, so the first call needs no host synchronisation and may happen inside a CUDA graph capture.
// With mu = G*x etc.:
//   s = A1 A2 / (B1 B2),  A1 = 2 mu1 mu2 + C1, A2 = 2 s12 + C2, B1 = mu1^2 + mu2^2 + C1, B2 = s1 + s2 + C2
//   d(sum s)/d img1 = G*(ds/dmu1) + 2 img1 (G*(ds/dE11)) + img2 (G*(ds/dE12))
//   ds/dmu1 = 2 mu2 (A2 - A1)/(B1 B2) - s (2 mu1/B1 - 2 mu1/B2),  ds/dE11 = -s/B2,  ds/dE12 = 2 A1/(B1 B2)
#include "common.cuh"

namespace h3dgs {

constexpr int kR = 5, kTS = 16, kHalo = kTS + 2 * kR;      // 26
struct LossWindow { float w[11]; };

__device__ __forceinline__ float block_sum_256(float v, float* s_red) {
    v += __shfl_down_sync(0xffffffffu, v, 16); v += __shfl_down_sync(0xffffffffu, v, 8);
    v += __shfl_down_sync(0xffffffffu, v, 4);  v += __shfl_down_sync(0xffffffffu, v, 2);
    v += __shfl_down_sync(0xffffffffu, v, 1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < 8) t = s_red[threadIdx.x];
    if (warp == 0) { t += __shfl_down_sync(0xffffffffu, t, 4); t += __shfl_down_sync(0xffffffffu, t, 2); t += __shfl_down_sync(0xffffffffu, t, 1); }
    __syncthreads();
    return t;      // valid in thread 0
}

// train_post's image before the loss (render_post, gaussian_renderer/__init__.py:279-285): the exposure applied from the
// right, y_c = sum_k img_k E[k][c] + E[c][3].  The fp32 order is pinned, ((img0 E[0][c] + img1 E[1][c]) + img2 E[2][c])
// + E[c][3] with every product and sum rounded (no FMA contraction): the forward's clamp decision and the backward's are
// taken on the same y, and a restatement outside the kernel reproduces it bit for bit.
__device__ __forceinline__ float exposed(const float* __restrict__ img, size_t plane, size_t p, const float* __restrict__ E, int c) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(img[p], E[c]), __fmul_rn(img[plane + p], E[4 + c])),
                               __fmul_rn(img[2 * plane + p], E[8 + c])), E[4 * c + 3]);
}

// kPost = false: the loss of img against gt (h3dgs_l1_ssim_forward).  kPost = true: the loss of a = clamp(y, 0, 1) * mask
// against gt as it is, y = exposed(img) or img[c] (h3dgs_post_loss_forward; C = 3); exposure and mask may be NULL.
// kClamp = false (train_coarse's objective, h3dgs_coarse_loss_forward): a = y * mask, unclamped.
template <bool kPost, bool kClamp = true>
__global__ void __launch_bounds__(256)
l1_ssim_forward_kernel(int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                       double* __restrict__ sums, float* __restrict__ maps, size_t map_stride, const LossWindow win,
                       const float* __restrict__ exposure, const float* __restrict__ mask)
{
    __shared__ float sa[kHalo][kHalo + 1], sb[kHalo][kHalo + 1];
    __shared__ float hz[5][kHalo][kTS];
    __shared__ float s_red[8];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int bx = blockIdx.x * kTS, by = blockIdx.y * kTS, c = blockIdx.z;
    const size_t plane = (size_t)H * W;
    const float* ia = img + (size_t)c * plane;
    const float* ib = gt + (size_t)c * plane;
    for (int i = tid; i < kHalo * kHalo; i += 256) {
        const int ly = i / kHalo, lx = i - ly * kHalo;
        const int gy = by + ly - kR, gx = bx + lx - kR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        if (kPost) {
            float a = 0.f, b = 0.f;                             // zero padding (conv2d padding=5)
            if (in) {
                const size_t p = (size_t)gy * W + gx;
                const float y = exposure ? exposed(img, plane, p, exposure, c) : ia[p];
                a = kClamp ? fminf(fmaxf(y, 0.f), 1.f) : y;
                if (mask) a *= mask[p];
                b = ib[p];                                      // the loader clamped and masked the target already
            }
            sa[ly][lx] = a;
            sb[ly][lx] = b;
        } else {
            sa[ly][lx] = in ? ia[(size_t)gy * W + gx] : 0.f;    // zero padding (conv2d padding=5)
            sb[ly][lx] = in ? ib[(size_t)gy * W + gx] : 0.f;
        }
    }
    __syncthreads();
    for (int i = tid; i < kHalo * kTS; i += 256) {
        const int r = i / kTS, x = i - r * kTS;
        float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; k++) {
            const float w = win.w[k], a = sa[r][x + k], b = sb[r][x + k];
            m1 += w * a; m2 += w * b; e11 += w * a * a; e22 += w * b * b; e12 += w * a * b;
        }
        hz[0][r][x] = m1; hz[1][r][x] = m2; hz[2][r][x] = e11; hz[3][r][x] = e22; hz[4][r][x] = e12;
    }
    __syncthreads();
    float mu1 = 0.f, mu2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
    for (int k = 0; k < 11; k++) {
        const float w = win.w[k];
        mu1 += w * hz[0][ty + k][tx]; mu2 += w * hz[1][ty + k][tx];
        e11 += w * hz[2][ty + k][tx]; e22 += w * hz[3][ty + k][tx]; e12 += w * hz[4][ty + k][tx];
    }
    const int px = bx + tx, py = by + ty;
    float ssim_v = 0.f, l1_v = 0.f;
    if (px < W && py < H) {
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        const float s1 = e11 - mu1 * mu1, s2 = e22 - mu2 * mu2, s12 = e12 - mu1 * mu2;
        const float A1 = 2.f * mu1 * mu2 + C1, A2 = 2.f * s12 + C2;
        const float B1 = mu1 * mu1 + mu2 * mu2 + C1, B2 = s1 + s2 + C2;
        const float iB1 = 1.f / B1, iB2 = 1.f / B2;
        const float s = A1 * A2 * iB1 * iB2;
        ssim_v = s;
        l1_v = fabsf(sa[ty + kR][tx + kR] - sb[ty + kR][tx + kR]);
        if (maps) {
            const size_t o = (size_t)c * plane + (size_t)py * W + px;
            maps[o] = 2.f * mu2 * (A2 - A1) * iB1 * iB2 - s * (2.f * mu1 * iB1 - 2.f * mu1 * iB2);   // ds/dmu1
            maps[map_stride + o] = -s * iB2;                                                       // ds/dE11
            maps[2 * map_stride + o] = 2.f * A1 * iB1 * iB2;                                       // ds/dE12
        }
    }
    const float l1_sum = block_sum_256(l1_v, s_red);
    const float ss_sum = block_sum_256(ssim_v, s_red);
    if (tid == 0) { atomicAdd(sums, (double)l1_sum); atomicAdd(sums + 1, (double)ss_sum); }
}

// The three derivative maps of channel c convolved with the window at this thread's pixel: a horizontal and a vertical
// 11-tap pass through shared memory over the 26x26 halo of the tile at (bx, by), zero outside the frame.
__device__ __forceinline__ void conv_maps(int H, int W, int bx, int by, int c, const float* __restrict__ maps,
                                          size_t map_stride, const LossWindow& win, float (&sm)[3][kHalo][kHalo + 1],
                                          float (&hz)[3][kHalo][kTS], float& c0, float& c1, float& c2)
{
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const size_t plane = (size_t)H * W;
    for (int i = tid; i < kHalo * kHalo; i += 256) {
        const int ly = i / kHalo, lx = i - ly * kHalo;
        const int gy = by + ly - kR, gx = bx + lx - kR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        const size_t o = (size_t)c * plane + (size_t)gy * W + gx;
        sm[0][ly][lx] = in ? maps[o] : 0.f;
        sm[1][ly][lx] = in ? maps[map_stride + o] : 0.f;
        sm[2][ly][lx] = in ? maps[2 * map_stride + o] : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < kHalo * kTS; i += 256) {
        const int r = i / kTS, x = i - r * kTS;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; k++) {
            const float w = win.w[k];
            a0 += w * sm[0][r][x + k]; a1 += w * sm[1][r][x + k]; a2 += w * sm[2][r][x + k];
        }
        hz[0][r][x] = a0; hz[1][r][x] = a1; hz[2][r][x] = a2;
    }
    __syncthreads();
    c0 = 0.f; c1 = 0.f; c2 = 0.f;
#pragma unroll
    for (int k = 0; k < 11; k++) {
        const float w = win.w[k];
        c0 += w * hz[0][ty + k][tx]; c1 += w * hz[1][ty + k][tx]; c2 += w * hz[2][ty + k][tx];
    }
}

__global__ void __launch_bounds__(256)
l1_ssim_backward_kernel(int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                        const float* __restrict__ maps, size_t map_stride, const float* __restrict__ coeffs,
                        float* __restrict__ dL_dimg, const LossWindow win)
{
    __shared__ float sm[3][kHalo][kHalo + 1];
    __shared__ float hz[3][kHalo][kTS];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int bx = blockIdx.x * kTS, by = blockIdx.y * kTS, c = blockIdx.z;
    const size_t plane = (size_t)H * W;
    float c0, c1, c2;
    conv_maps(H, W, bx, by, c, maps, map_stride, win, sm, hz, c0, c1, c2);
    const int px = bx + tx, py = by + ty;
    if (px < W && py < H) {
        const size_t o = (size_t)c * plane + (size_t)py * W + px;
        const float a = img[o], b = gt[o];
        const float sgn = (a > b) ? 1.f : ((a < b) ? -1.f : 0.f);
        dL_dimg[o] = coeffs[0] * sgn + coeffs[1] * (c0 + 2.f * a * c1 + b * c2);
    }
}

// Backward of the post loss: one CTA per 16x16 tile, looping over the three channels, because the exposure's transpose
// needs all three dL/dy_c of a pixel.  Per channel, with a = clamp(y_c, 0, 1) * m recomputed as the forward stages it:
//   dL/dy_c = [0 <= y_c <= 1] * (m * (k0 sign(a - b) + k1 (c0 + 2 a c1 + b c2)))      (torch's clamp passes both ends)
// kept in registers; then dL/dimg_k = (E[k][0] g_0 + E[k][1] g_1) + E[k][2] g_2 (rounded in that order), or g_k
// without an exposure.  dL/dimg is written once; no dL/da buffer.
// kGradE (train_single.py, where the exposure is a trained parameter): the same pass also leaves dL/dE [3][4] -- the
// twelve per-pixel terms img_k * g_c (k, c < 3; one rounded product each) and g_c are summed over the CTA in fp32 (xor
// butterfly over the warp, offsets 16 .. 1), the eight warp sums are added in fp64 in warp order and one fp64 atomic
// per CTA and entry adds them to dL_dE.  dL/dimg does not depend on the flag.
// kClamp = false (train_coarse, h3dgs_coarse_loss_backward): a = y * m and dL/dy_c = m * (...) without the clamp
// indicator -- the rasterizer clamps colours only below, so y > 1 occurs and its gradient passes.
template <bool kGradE, bool kClamp = true>
__global__ void __launch_bounds__(256)
post_loss_backward_kernel(int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                          const float* __restrict__ exposure, const float* __restrict__ mask,
                          const float* __restrict__ maps, size_t map_stride, const float* __restrict__ coeffs,
                          float* __restrict__ dL_dimg, double* __restrict__ dL_dE, const LossWindow win)
{
    __shared__ float sm[3][kHalo][kHalo + 1];
    __shared__ float hz[3][kHalo][kTS];
    __shared__ float s_e[kGradE ? 8 : 1][12];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int bx = blockIdx.x * kTS, by = blockIdx.y * kTS;
    const size_t plane = (size_t)H * W;
    const int px = bx + tx, py = by + ty;
    const bool own = px < W && py < H;
    const size_t p = own ? (size_t)py * W + px : 0;
    const float k0 = coeffs[0], k1 = coeffs[1];
    const float m = (own && mask) ? mask[p] : 1.f;
    float g[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        if (c) __syncthreads();                             // the previous channel's passes are done with sm and hz
        float c0, c1, c2;
        conv_maps(H, W, bx, by, c, maps, map_stride, win, sm, hz, c0, c1, c2);
        g[c] = 0.f;
        if (own) {
            const float y = exposure ? exposed(img, plane, p, exposure, c) : img[(size_t)c * plane + p];
            float a = kClamp ? fminf(fmaxf(y, 0.f), 1.f) : y;
            if (mask) a *= m;
            const float b = gt[(size_t)c * plane + p];
            const float sgn = (a > b) ? 1.f : ((a < b) ? -1.f : 0.f);
            float d = k0 * sgn + k1 * (c0 + 2.f * a * c1 + b * c2);
            if (mask) d = __fmul_rn(m, d);
            g[c] = (!kClamp || (y >= 0.f && y <= 1.f)) ? d : 0.f;
        }
    }
    if (kGradE) {
        float v[12];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float ik = own ? img[(size_t)k * plane + p] : 0.f;
#pragma unroll
            for (int c = 0; c < 3; c++) v[4 * k + c] = __fmul_rn(ik, g[c]);         // dL/dE[k][c]
            v[4 * k + 3] = g[k];                                                     // dL/dE[k][3]
        }
#pragma unroll
        for (int j = 0; j < 12; j++) {
            float t = v[j];
            t += __shfl_xor_sync(0xffffffffu, t, 16); t += __shfl_xor_sync(0xffffffffu, t, 8);
            t += __shfl_xor_sync(0xffffffffu, t, 4);  t += __shfl_xor_sync(0xffffffffu, t, 2);
            t += __shfl_xor_sync(0xffffffffu, t, 1);
            if ((tid & 31) == 0) s_e[tid >> 5][j] = t;
        }
        __syncthreads();
        if (tid < 12) {
            double t = 0.0;
#pragma unroll
            for (int w = 0; w < 8; w++) t += (double)s_e[w][tid];
            if (t != 0.0) atomicAdd(dL_dE + tid, t);
        }
    }
    if (!own) return;
    if (exposure) {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float* Ek = exposure + 4 * k;
            dL_dimg[(size_t)k * plane + p] =
                __fadd_rn(__fadd_rn(__fmul_rn(Ek[0], g[0]), __fmul_rn(Ek[1], g[1])), __fmul_rn(Ek[2], g[2]));
        }
    } else {
#pragma unroll
        for (int k = 0; k < 3; k++) dL_dimg[(size_t)k * plane + p] = g[k];
    }
}

// One thread: the eight status words of train_single's step (h3dgs/singlestep.py) -- loss, photometric loss, L1, SSIM,
// pure inverse-depth L1, D, longest tile list, binning overflow -- and the exposure gradient in fp32 for the caller's
// optimizer, zero for an overflowed frame (which contributes no gradient anywhere else either).
__global__ void single_step_status_kernel(const double* __restrict__ sums, const double* __restrict__ depth_sum,
                                          const float* __restrict__ depth_weight, double inv_numel, double inv_pixels,
                                          double lambda_dssim, const uint32_t* __restrict__ scan_info,
                                          const double* __restrict__ dL_dE, float* __restrict__ exposure_grad, double* __restrict__ out)
{
    if (exposure_grad)
        for (int j = 0; j < 12; j++) exposure_grad[j] = scan_info[2] ? 0.f : (float)dL_dE[j];
    const double l1 = sums[0] * inv_numel, ssim = sums[1] * inv_numel;
    const double photo = (1.0 - lambda_dssim) * l1 + lambda_dssim * (1.0 - ssim);
    // weight 0: the term is absent, as train_single.py:111 skips it
    const double w = depth_sum ? (double)*depth_weight : 0.0, depth = w != 0.0 ? *depth_sum * inv_pixels : 0.0;
    out[0] = photo + w * depth;
    out[1] = photo; out[2] = l1; out[3] = ssim; out[4] = depth;
    out[5] = (double)scan_info[0]; out[6] = (double)scan_info[1]; out[7] = (double)scan_info[2];
}

// One thread: the eight status words of the post-loss step (h3dgs/poststep.py) -- loss, L1, SSIM, rows the cut needs, D,
// longest tile list, binning overflow, row overflow.
__global__ void post_step_status_kernel(const double* __restrict__ sums, double inv_numel, double lambda_dssim,
                                        const int* __restrict__ count, int extra_rows, int row_capacity,
                                        const uint32_t* __restrict__ scan_info, double* __restrict__ out)
{
    const double l1 = sums[0] * inv_numel, ssim = sums[1] * inv_numel;
    const double rows = (double)(*count + extra_rows);
    out[0] = (1.0 - lambda_dssim) * l1 + lambda_dssim * (1.0 - ssim);
    out[1] = l1; out[2] = ssim;
    out[3] = rows;
    out[4] = (double)scan_info[0]; out[5] = (double)scan_info[1]; out[6] = (double)scan_info[2];
    out[7] = rows > (double)row_capacity ? 1.0 : 0.0;
}

static LossWindow make_loss_window() {
    // utils/loss_utils.py:23-25: exp(-(x - 5)^2 / (2 * 1.5^2)), normalised in fp32 (the weights of metrics.cu)
    LossWindow w; float sum = 0.f;
    for (int x = 0; x < 11; x++) { w.w[x] = (float)exp(-(double)((x - 5) * (x - 5)) / (2.0 * 1.5 * 1.5)); sum += w.w[x]; }
    for (int x = 0; x < 11; x++) w.w[x] /= sum;
    return w;
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" int h3dgs_l1_ssim_forward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, double* sums,
                                     float* maps, void* stream)
{
    if (C <= 0 || H <= 0 || W <= 0 || !img || !gt || !sums) { set_error("l1_ssim_forward: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    H3_CUDA(cudaMemsetAsync(sums, 0, 2 * sizeof(double), s));
    const dim3 grid((W + kTS - 1) / kTS, (H + kTS - 1) / kTS, C);
    l1_ssim_forward_kernel<false><<<grid, 256, 0, s>>>(H, W, img, gt, sums, maps, (size_t)C * H * W, make_loss_window(), nullptr, nullptr);
    H3_LAUNCHED("l1_ssim_forward", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_l1_ssim_backward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                      const float* maps, const float* coeffs, float* dL_dimg, void* stream)
{
    if (C <= 0 || H <= 0 || W <= 0 || !img || !gt || !maps || !coeffs || !dL_dimg) { set_error("l1_ssim_backward: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    const dim3 grid((W + kTS - 1) / kTS, (H + kTS - 1) / kTS, C);
    l1_ssim_backward_kernel<<<grid, 256, 0, s>>>(H, W, img, gt, maps, (size_t)C * H * W, coeffs, dL_dimg, make_loss_window());
    H3_LAUNCHED("l1_ssim_backward", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_post_loss_forward(int32_t H, int32_t W, const float* img, const float* gt, const float* exposure,
                                       const float* mask, double* sums, float* maps, void* stream)
{
    if (H <= 0 || W <= 0 || !img || !gt || !sums) { set_error("post_loss_forward: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    H3_CUDA(cudaMemsetAsync(sums, 0, 2 * sizeof(double), s));
    const dim3 grid((W + kTS - 1) / kTS, (H + kTS - 1) / kTS, 3);
    l1_ssim_forward_kernel<true><<<grid, 256, 0, s>>>(H, W, img, gt, sums, maps, (size_t)3 * H * W, make_loss_window(), exposure, mask);
    H3_LAUNCHED("post_loss_forward", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_post_loss_backward(int32_t H, int32_t W, const float* img, const float* gt, const float* exposure,
                                        const float* mask, const float* maps, const float* coeffs, float* dL_dimg, void* stream)
{
    if (H <= 0 || W <= 0 || !img || !gt || !maps || !coeffs || !dL_dimg) { set_error("post_loss_backward: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    const dim3 grid((W + kTS - 1) / kTS, (H + kTS - 1) / kTS, 1);
    post_loss_backward_kernel<false><<<grid, 256, 0, s>>>(H, W, img, gt, exposure, mask, maps, (size_t)3 * H * W, coeffs, dL_dimg, nullptr, make_loss_window());
    H3_LAUNCHED("post_loss_backward", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_post_loss_backward_exposure(int32_t H, int32_t W, const float* img, const float* gt, const float* exposure,
                                                 const float* mask, const float* maps, const float* coeffs, float* dL_dimg,
                                                 double* dL_dexposure, void* stream)
{
    if (H <= 0 || W <= 0 || !img || !gt || !maps || !coeffs || !dL_dimg || !dL_dexposure) { set_error("post_loss_backward_exposure: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    H3_CUDA(cudaMemsetAsync(dL_dexposure, 0, 12 * sizeof(double), s));
    const dim3 grid((W + kTS - 1) / kTS, (H + kTS - 1) / kTS, 1);
    ProfScope prof(H3DGS_STAGE_LOSS_BACKWARD_EXPOSURE, s);
    post_loss_backward_kernel<true><<<grid, 256, 0, s>>>(H, W, img, gt, exposure, mask, maps, (size_t)3 * H * W, coeffs, dL_dimg, dL_dexposure, make_loss_window());
    H3_LAUNCHED("post_loss_backward_exposure", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_coarse_loss_forward(int32_t H, int32_t W, const float* img, const float* gt, const float* mask,
                                         double* sums, float* maps, void* stream)
{
    if (H <= 0 || W <= 0 || !img || !gt || !sums) { set_error("coarse_loss_forward: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    H3_CUDA(cudaMemsetAsync(sums, 0, 2 * sizeof(double), s));
    const dim3 grid((W + kTS - 1) / kTS, (H + kTS - 1) / kTS, 3);
    l1_ssim_forward_kernel<true, false><<<grid, 256, 0, s>>>(H, W, img, gt, sums, maps, (size_t)3 * H * W, make_loss_window(), nullptr, mask);
    H3_LAUNCHED("coarse_loss_forward", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_coarse_loss_backward(int32_t H, int32_t W, const float* img, const float* gt, const float* mask,
                                          const float* maps, const float* coeffs, float* dL_dimg, void* stream)
{
    if (H <= 0 || W <= 0 || !img || !gt || !maps || !coeffs || !dL_dimg) { set_error("coarse_loss_backward: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    const dim3 grid((W + kTS - 1) / kTS, (H + kTS - 1) / kTS, 1);
    post_loss_backward_kernel<false, false><<<grid, 256, 0, s>>>(H, W, img, gt, nullptr, mask, maps, (size_t)3 * H * W, coeffs, dL_dimg, nullptr, make_loss_window());
    H3_LAUNCHED("coarse_loss_backward", 0, s);
    return H3DGS_OK;
}

// One thread: the six status words of train_coarse's step (h3dgs/coarsestep.py) -- loss, L1, SSIM, D, longest tile list,
// binning overflow.
__global__ void coarse_step_status_kernel(const double* __restrict__ sums, double inv_numel, double lambda_dssim,
                                          const uint32_t* __restrict__ scan_info, double* __restrict__ out)
{
    const double l1 = sums[0] * inv_numel, ssim = sums[1] * inv_numel;
    out[0] = (1.0 - lambda_dssim) * l1 + lambda_dssim * (1.0 - ssim);
    out[1] = l1; out[2] = ssim;
    out[3] = (double)scan_info[0]; out[4] = (double)scan_info[1]; out[5] = (double)scan_info[2];
}

extern "C" int h3dgs_coarse_step_status(const double* sums, double inv_numel, double lambda_dssim, const uint32_t* scan_info,
                                        double* out, void* stream)
{
    if (!sums || !scan_info || !out) { set_error("coarse_step_status: NULL argument"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    coarse_step_status_kernel<<<1, 1, 0, s>>>(sums, inv_numel, lambda_dssim, scan_info, out);
    H3_LAUNCHED("coarse_step_status", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_single_step_status(const double* sums, const double* depth_sum, const float* depth_weight, double inv_numel,
                                        double inv_pixels, double lambda_dssim, const uint32_t* scan_info,
                                        const double* dL_dexposure, float* exposure_grad, double* out, void* stream)
{
    if (!sums || !scan_info || !out || (depth_sum && !depth_weight) || (exposure_grad && !dL_dexposure)) { set_error("single_step_status: NULL argument"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    single_step_status_kernel<<<1, 1, 0, s>>>(sums, depth_sum, depth_weight, inv_numel, inv_pixels, lambda_dssim, scan_info, dL_dexposure, exposure_grad, out);
    H3_LAUNCHED("single_step_status", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_post_step_status(const double* sums, double inv_numel, double lambda_dssim, const int32_t* count,
                                      int32_t extra_rows, int32_t row_capacity, const uint32_t* scan_info, double* out, void* stream)
{
    if (!sums || !count || !scan_info || !out) { set_error("post_step_status: NULL argument"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    post_step_status_kernel<<<1, 1, 0, s>>>(sums, inv_numel, lambda_dssim, count, extra_rows, row_capacity, scan_info, out);
    H3_LAUNCHED("post_step_status", 0, s);
    return H3DGS_OK;
}
