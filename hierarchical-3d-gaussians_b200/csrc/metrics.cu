// metrics.cu -- image-quality metrics of one rendered frame in one pass: what render_hierarchy.py:82-113 evaluates on
// top of render_post (gaussian_renderer/__init__.py:279-285) -- exposure, clamp, the train_test_exp half-width crop, the
// alpha mask, PSNR (utils/image_utils.py:17-19, then .mean()) and SSIM (utils/loss_utils.py:33-63: 11x11 Gaussian
// window, sigma 1.5, zero padding at the border of the CROPPED image, C1 = 0.01^2, C2 = 0.03^2).
//
// The reference runs ~40 PyTorch kernels per frame for this and syncs twice (.double() of psnr and ssim).  Here: ONE
// tile kernel (the separable 11+11-tap scheme of loss.cu, 16x16 output tiles with a 5-pixel halo; the per-channel
// squared error and the SSIM map sum go into device doubles) and ONE single-thread finisher that turns the sums into a
// result row and stores it at a slot taken from a device counter.  Nothing returns to the host, so a whole sweep of
// frames can be enqueued -- or replayed from a CUDA graph -- and read back once.
//
// The window weights travel as a kernel argument (no __constant__ upload, which would need a host synchronisation).
#include <math.h>
#include "common.cuh"

namespace h3dgs {
namespace {

constexpr int kMR = 5, kMTS = 16, kMHalo = kMTS + 2 * kMR;      // 26
struct Window { float w[11]; };

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

__device__ __forceinline__ double block_sum_256_d(double v, double* s_red) {
    v += __shfl_xor_sync(0xffffffffu, v, 16); v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);  v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x < 8) t = s_red[threadIdx.x];
    if (warp == 0) { t += __shfl_xor_sync(0xffffffffu, t, 4); t += __shfl_xor_sync(0xffffffffu, t, 2); t += __shfl_xor_sync(0xffffffffu, t, 1); }
    __syncthreads();
    return t;      // valid in thread 0
}

// grid (tiles x, tiles y, channel) over the cropped frame [H, W - x0]; img / gt / mask are the full [3,H,W] / [H,W]
// frames.  sums[c] += sum of squared errors of channel c, sums[3] += SSIM map sum (both after the mask).
__global__ void __launch_bounds__(256)
metrics_kernel(int H, int W, int x0, const float* __restrict__ img, const float* __restrict__ gt,
               const float* __restrict__ exposure, const float* __restrict__ mask, float* __restrict__ out_img,
               double* __restrict__ sums, const Window win)
{
    __shared__ float sa[kMHalo][kMHalo + 1], sb[kMHalo][kMHalo + 1];
    __shared__ float hz[5][kMHalo][kMTS];
    __shared__ double s_red[8];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int bx = blockIdx.x * kMTS, by = blockIdx.y * kMTS, c = blockIdx.z;
    const int Wc = W - x0;
    const size_t plane = (size_t)H * W;
    for (int i = tid; i < kMHalo * kMHalo; i += 256) {
        const int ly = i / kMHalo, lx = i - ly * kMHalo;
        const int gy = by + ly - kMR, gx = bx + lx - kMR;           // cropped coordinates
        float a = 0.f, b = 0.f;                                     // zero padding at the crop border (conv2d padding=5)
        if (gy >= 0 && gy < H && gx >= 0 && gx < Wc) {
            const size_t p = (size_t)gy * W + x0 + gx;
            if (exposure) {
                // image.permute(1,2,0) @ E[:3,:3] + E[:3,3]: the matrix acts from the right, out[c] = sum_k img[k] E[k][c] + E[c][3]
                a = img[p] * exposure[c] + img[plane + p] * exposure[4 + c] + img[2 * plane + p] * exposure[8 + c] + exposure[4 * c + 3];
            } else {
                a = img[(size_t)c * plane + p];
            }
            a = clamp01(a);
            b = clamp01(gt[(size_t)c * plane + p]);
            if (out_img && ly >= kMR && ly < kMR + kMTS && lx >= kMR && lx < kMR + kMTS)
                out_img[((size_t)c * H + gy) * Wc + gx] = a;        // exposed, clamped, cropped; before the mask
            if (mask) { const float m = mask[p]; a *= m; b *= m; }
        }
        sa[ly][lx] = a;
        sb[ly][lx] = b;
    }
    __syncthreads();
    for (int i = tid; i < kMHalo * kMTS; i += 256) {
        const int r = i / kMTS, x = i - r * kMTS;
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
    double ssim_v = 0.0, se_v = 0.0;
    if (px < Wc && py < H) {
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        const float s1 = e11 - mu1 * mu1, s2 = e22 - mu2 * mu2, s12 = e12 - mu1 * mu2;
        const float A1 = 2.f * mu1 * mu2 + C1, A2 = 2.f * s12 + C2;
        const float B1 = mu1 * mu1 + mu2 * mu2 + C1, B2 = s1 + s2 + C2;
        ssim_v = (double)((A1 * A2) / (B1 * B2));
        const float d = sa[ty + kMR][tx + kMR] - sb[ty + kMR][tx + kMR];
        se_v = (double)d * (double)d;
    }
    const double se_sum = block_sum_256_d(se_v, s_red);
    const double ss_sum = block_sum_256_d(ssim_v, s_red);
    if (tid == 0) { atomicAdd(sums + c, se_sum); atomicAdd(sums + 3, ss_sum); }
}

// One thread: the sums of metrics_kernel -> one result row at slot (*counter)++ (see h3dgs.h).
__global__ void metrics_finish_kernel(int H, int Wc, const double* __restrict__ sums, const int* __restrict__ count, int extra_rows,
                                      int row_capacity, const uint32_t* __restrict__ scan_info, int* __restrict__ counter,
                                      double* __restrict__ results, int max_rows)
{
    const double n = (double)H * (double)Wc;
    double psnr = 0.0;
    for (int c = 0; c < 3; c++) psnr += 20.0 * log10(1.0 / sqrt(sums[c] / n));       // +inf where a channel is exact
    const double rows = (double)((count ? *count : 0) + extra_rows);
    const bool bin_overflow = scan_info && scan_info[2] != 0u;
    const int slot = *counter;
    *counter = slot + 1;
    if (slot >= max_rows) return;
    double* row = results + (size_t)slot * H3DGS_EVAL_ROW;
    row[0] = psnr / 3.0;
    row[1] = sums[3] / (3.0 * n);
    row[2] = (bin_overflow || (row_capacity > 0 && rows > (double)row_capacity)) ? 1.0 : 0.0;
    row[3] = rows;
    row[4] = scan_info ? (double)scan_info[0] : 0.0;
    row[5] = scan_info ? (double)scan_info[1] : 0.0;
}

Window make_window() {
    // utils/loss_utils.py:23-25: exp(-(x - 5)^2 / (2 * 1.5^2)), normalised in fp32 (the weights of loss.cu)
    Window w; float sum = 0.f;
    for (int x = 0; x < 11; x++) { w.w[x] = (float)exp(-(double)((x - 5) * (x - 5)) / (2.0 * 1.5 * 1.5)); sum += w.w[x]; }
    for (int x = 0; x < 11; x++) w.w[x] /= sum;
    return w;
}

}  // namespace
}  // namespace h3dgs

using namespace h3dgs;

extern "C" int h3dgs_eval_metrics(int32_t H, int32_t W, const float* img, const float* gt, const float* exposure,
                                  const float* mask, int32_t x0, float* out_img, double* sums, const int32_t* count,
                                  int32_t extra_rows, int32_t row_capacity, const uint32_t* scan_info, int32_t* counter,
                                  double* results, int32_t max_rows, void* stream)
{
    if (H <= 0 || W <= 0 || x0 < 0 || x0 >= W || !img || !gt || !sums || !counter || !results || max_rows <= 0) {
        set_error("eval_metrics: bad arguments"); return H3DGS_EINVAL;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int Wc = W - x0;
    H3_CUDA(cudaMemsetAsync(sums, 0, 4 * sizeof(double), s));
    const dim3 grid((Wc + kMTS - 1) / kMTS, (H + kMTS - 1) / kMTS, 3);
    metrics_kernel<<<grid, 256, 0, s>>>(H, W, x0, img, gt, exposure, mask, out_img, sums, make_window());
    H3_LAUNCHED("eval_metrics", 0, s);
    metrics_finish_kernel<<<1, 1, 0, s>>>(H, Wc, sums, count, extra_rows, row_capacity, scan_info, counter, results, max_rows);
    H3_LAUNCHED("eval_metrics_finish", 0, s);
    return H3DGS_OK;
}
