// l1_loss.cu -- L1 loss and its gradient in one pass (the loss of the step bench.py and h3dgs.graphstep time:
// train_post.py:134-142 with lambda_dssim = 0; the SSIM term lives in loss.cu).
// Also the two per-step kernels of train_single.py beside its photometric loss: the inverse-depth L1 with its gradient
// (:111-117) and the densification statistics (:147-148).
#include <algorithm>
#include "common.cuh"

namespace h3dgs {

__device__ __forceinline__ float warp_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 16); v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);  v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// L1 loss and its gradient in ONE pass (the step of bench.py / h3dgs.graphstep: loss = mean |img - gt|,
// dL/dimg = sign(img - gt) * scale), optionally only over the 16-pixel tile rows one rank of a tile-sharded frame
// owns (y_tile % shard_count == shard_index): L1 is per pixel, so a rank needs no pixel it did not render.
// float4 streams; sum |d| goes to a device double with one atomic per CTA.
template <int VEC>
__global__ void __launch_bounds__(256)
l1_grad_kernel(int C, int H, int W, int shard_count, int shard_index, const float* __restrict__ img,
               const float* __restrict__ gt, float scale, float* __restrict__ dL_dimg, double* __restrict__ loss_sum,
               const PeerPtrs peers, const PeerPtrs images)
{
    __shared__ float s_red[8];
    const int W4 = W / VEC;                                  // VEC = 4 needs W % 4 == 0 (launcher)
    const size_t total4 = (size_t)C * H * W4;
    float acc = 0.f;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total4; i += (size_t)gridDim.x * 256) {
        const int y = (int)((i / W4) % H);
        if (shard_count > 1 && ((y >> 4) % shard_count) != shard_index) continue;
        if (VEC == 1) {
            const float d = img[i] - gt[i];
            acc += fabsf(d);
            dL_dimg[i] = d > 0.f ? scale : (d < 0.f ? -scale : 0.f);
            continue;
        }
        const float4 a = reinterpret_cast<const float4*>(img)[i], b = reinterpret_cast<const float4*>(gt)[i];
        if (images.n > 1) {
            // peer mode: this rank's pixels travel to the other ranks' images from HERE -- one coalesced 128-bit store per
            // lane and rank (512 contiguous bytes per warp), posted over NVLink -- instead of pixel by pixel out of the
            // blend kernel, whose stores would otherwise be scattered pixel by pixel
#pragma unroll
            for (int r = 0; r < H3DGS_MAX_PEERS; r++)
                if (r < images.n && r != shard_index && images.p[r]) reinterpret_cast<float4*>(images.p[r])[i] = a;
        }
        const float d0 = a.x - b.x, d1 = a.y - b.y, d2 = a.z - b.z, d3 = a.w - b.w;
        acc += (fabsf(d0) + fabsf(d1)) + (fabsf(d2) + fabsf(d3));
        float4 g;
        g.x = d0 > 0.f ? scale : (d0 < 0.f ? -scale : 0.f); g.y = d1 > 0.f ? scale : (d1 < 0.f ? -scale : 0.f);
        g.z = d2 > 0.f ? scale : (d2 < 0.f ? -scale : 0.f); g.w = d3 > 0.f ? scale : (d3 < 0.f ? -scale : 0.f);
        reinterpret_cast<float4*>(dL_dimg)[i] = g;
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        const float t = warp_sum(threadIdx.x < 8 ? s_red[threadIdx.x] : 0.f);
        if (threadIdx.x == 0 && t != 0.f) {
            if (peers.n > 1) {
#pragma unroll
                for (int r = 0; r < H3DGS_MAX_PEERS; r++) if (r < peers.n) atomicAdd_system(static_cast<double*>(peers.p[r]), (double)t);
            }
            else atomicAdd(loss_sum, (double)t);
        }
    }
}

// One thread: the six status words of a sync-free step (h3dgs/graphstep.py) -- loss, rows the cut needs, D, longest
// tile list, binning overflow, row overflow -- and, optionally, the reset of the loss accumulator for the next step.
// Replaces nine tiny framework kernels at the end of the step's critical path.
__global__ void step_status_kernel(double* __restrict__ loss_sum, double inv_numel, const int* __restrict__ count, int extra_rows,
                                   int row_capacity, const uint32_t* __restrict__ scan_info, int reset_loss, double* __restrict__ out)
{
    const double rows = (double)(*count + extra_rows);
    out[0] = *loss_sum * inv_numel;
    out[1] = rows;
    out[2] = (double)scan_info[0]; out[3] = (double)scan_info[1]; out[4] = (double)scan_info[2];
    out[5] = rows > (double)row_capacity ? 1.0 : 0.0;
    if (reset_loss) *loss_sum = 0.0;
}

// train_single's inverse-depth term (train_single.py:111-117) and its gradient in ONE pass:
//   t = (invdepth - mono) * depth_mask (difference and product rounded), *sum += |t| (unweighted: Ll1depth_pure before
//   the mean), dL/dinvdepth = ((w / (H W)) * sign(t)) * depth_mask with sign(0) = 0 as torch.abs; w is read on the device.
__device__ __forceinline__ float invdepth_term(float d, float m, float k, float scale, float& acc) {
    const float t = __fmul_rn(__fadd_rn(d, -m), k);
    acc += fabsf(t);
    return __fmul_rn(t > 0.f ? scale : (t < 0.f ? -scale : 0.f), k);
}

template <int VEC>
__global__ void __launch_bounds__(256)
invdepth_l1_grad_kernel(size_t total, float pixels, const float* __restrict__ invdepth, const float* __restrict__ mono,
                        const float* __restrict__ depth_mask, const float* __restrict__ weight,
                        float* __restrict__ dL_dinvdepth, double* __restrict__ sum)
{
    __shared__ float s_red[8];
    const float scale = *weight / pixels;                   // IEEE division, rounded once
    float acc = 0.f;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total / VEC; i += (size_t)gridDim.x * 256) {
        if (VEC == 1) { dL_dinvdepth[i] = invdepth_term(invdepth[i], mono[i], depth_mask[i], scale, acc); continue; }
        const float4 d = reinterpret_cast<const float4*>(invdepth)[i], m = reinterpret_cast<const float4*>(mono)[i];
        const float4 k = reinterpret_cast<const float4*>(depth_mask)[i];
        float4 g;
        g.x = invdepth_term(d.x, m.x, k.x, scale, acc); g.y = invdepth_term(d.y, m.y, k.y, scale, acc);
        g.z = invdepth_term(d.z, m.z, k.z, scale, acc); g.w = invdepth_term(d.w, m.w, k.w, scale, acc);
        reinterpret_cast<float4*>(dL_dinvdepth)[i] = g;
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        const float t = warp_sum(threadIdx.x < 8 ? s_red[threadIdx.x] : 0.f);
        if (threadIdx.x == 0 && t != 0.f) atomicAdd(sum, (double)t);
    }
}

// The densification statistics of one training step (train_single.py:147, scene/gaussian_model.py:687-689), one thread
// per row; rows with radii <= 0 are untouched.  The norm is sqrt(x*x + y*y) with both products, the sum and the root
// rounded to fp32 (no FMA); the maxima propagate a NaN as torch.max does.  An overflowed capacity-mode frame
// (scan_info[2] != 0) changes nothing: its radii are those of the real frame (the preprocess runs before the overflow
// is known) but its gradients are zero, and the caller re-runs it.
__global__ void __launch_bounds__(256)
densify_stats_kernel(int P, const int* __restrict__ radii, const float* __restrict__ dL_dmeans2D, float* __restrict__ max_radii2D,
                     float* __restrict__ xyz_gradient_accum, float* __restrict__ denom, const uint32_t* __restrict__ scan_info)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P || (scan_info && scan_info[2])) return;
    const int r = radii[i];
    if (r <= 0) return;
    const float rf = (float)r, mr = max_radii2D[i];
    max_radii2D[i] = (mr != mr || mr > rf) ? mr : rf;
    if (!denom) return;                                     // max_radii2D only (train_coarse.py:125)
    const float x = dL_dmeans2D[3 * (size_t)i], y = dL_dmeans2D[3 * (size_t)i + 1];
    const float n = sqrtf(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))), a = xyz_gradient_accum[i];
    xyz_gradient_accum[i] = (n != n || n > a) ? n : a;
    denom[i] += 1.f;
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" int h3dgs_invdepth_l1_grad(int32_t H, int32_t W, const float* invdepth, const float* mono, const float* depth_mask,
                                      const float* weight, float* dL_dinvdepth, double* sum, void* stream)
{
    if (H <= 0 || W <= 0 || !invdepth || !mono || !depth_mask || !weight || !dL_dinvdepth || !sum) { set_error("invdepth_l1_grad: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    H3_CUDA(cudaMemsetAsync(sum, 0, sizeof(double), s));
    const size_t total = (size_t)H * W;
    const bool vec = (total & 3) == 0 && (((uintptr_t)invdepth | (uintptr_t)mono | (uintptr_t)depth_mask | (uintptr_t)dL_dinvdepth) & 15) == 0;
    const int blocks = (int)std::min<size_t>(((vec ? total >> 2 : total) + 255) / 256, 132 * 16);
    ProfScope prof(H3DGS_STAGE_INVDEPTH_L1, s);
    if (vec) invdepth_l1_grad_kernel<4><<<blocks, 256, 0, s>>>(total, (float)total, invdepth, mono, depth_mask, weight, dL_dinvdepth, sum);
    else invdepth_l1_grad_kernel<1><<<blocks, 256, 0, s>>>(total, (float)total, invdepth, mono, depth_mask, weight, dL_dinvdepth, sum);
    H3_LAUNCHED("invdepth_l1_grad", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_densify_stats(int32_t P, const int32_t* radii, const float* dL_dmeans2D, float* max_radii2D,
                                   float* xyz_gradient_accum, float* denom, const uint32_t* scan_info, void* stream)
{
    if (P < 0 || (P > 0 && (!radii || !max_radii2D || !xyz_gradient_accum != !denom || (denom && !dL_dmeans2D)))) { set_error("densify_stats: bad arguments"); return H3DGS_EINVAL; }
    if (P == 0) return H3DGS_OK;
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope prof(H3DGS_STAGE_DENSIFY_STATS, s);
    densify_stats_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, radii, dL_dmeans2D, max_radii2D, xyz_gradient_accum, denom, scan_info);
    H3_LAUNCHED("densify_stats", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_step_status(double* loss_sum, double inv_numel, const int32_t* count, int32_t extra_rows, int32_t row_capacity,
                                 const uint32_t* scan_info, int32_t reset_loss, double* out, void* stream)
{
    if (!loss_sum || !count || !scan_info || !out) { set_error("step_status: NULL argument"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    step_status_kernel<<<1, 1, 0, s>>>(loss_sum, inv_numel, count, extra_rows, row_capacity, scan_info, reset_loss, out);
    H3_LAUNCHED("step_status", 0, s);
    return H3DGS_OK;
}

static int l1_launch(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, float scale, int32_t shard_count,
                     int32_t shard_index, float* dL_dimg, double* loss_sum, const PeerPtrs& peers, const PeerPtrs& images, cudaStream_t s)
{
    const bool vec = (W & 3) == 0;
    const size_t total = (size_t)C * H * (vec ? (W >> 2) : W);
    const int blocks = (int)std::min<size_t>((total + 255) / 256, 132 * 16);      // 16 CTAs per SM of an H100
    const int sc = shard_count > 1 ? shard_count : 1, si = shard_count > 1 ? shard_index : 0;
    if (vec) l1_grad_kernel<4><<<blocks, 256, 0, s>>>(C, H, W, sc, si, img, gt, scale, dL_dimg, loss_sum, peers, images);
    else l1_grad_kernel<1><<<blocks, 256, 0, s>>>(C, H, W, sc, si, img, gt, scale, dL_dimg, loss_sum, peers, images);
    H3_LAUNCHED("l1_loss_grad", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_l1_loss_grad(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, float scale,
                                  int32_t shard_count, int32_t shard_index, float* dL_dimg, double* loss_sum, void* stream)
{
    if (C <= 0 || H <= 0 || W <= 0 || !img || !gt || !dL_dimg || !loss_sum) { set_error("l1_loss_grad: bad arguments"); return H3DGS_EINVAL; }
    if (shard_count > 1 && (shard_index < 0 || shard_index >= shard_count)) { set_error("l1_loss_grad: bad shard"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    H3_CUDA(cudaMemsetAsync(loss_sum, 0, sizeof(double), s));
    PeerPtrs none; none.n = 0;
    for (int k = 0; k < H3DGS_MAX_PEERS; k++) none.p[k] = nullptr;
    return l1_launch(C, H, W, img, gt, scale, shard_count, shard_index, dL_dimg, loss_sum, none, none, s);
}

extern "C" int h3dgs_l1_loss_grad_peer(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, float scale,
                                       int32_t shard_count, int32_t shard_index, float* dL_dimg, int32_t peer_count,
                                       double* const* loss_sums, float* const* peer_images, void* stream)
{
    if (C <= 0 || H <= 0 || W <= 0 || !img || !gt || !dL_dimg || !loss_sums || peer_count < 2 || peer_count > H3DGS_MAX_PEERS) {
        set_error("l1_loss_grad_peer: bad arguments"); return H3DGS_EINVAL;
    }
    if (shard_count > 1 && (shard_index < 0 || shard_index >= shard_count)) { set_error("l1_loss_grad_peer: bad shard"); return H3DGS_EINVAL; }
    PeerPtrs images; images.n = 0;
    for (int k = 0; k < H3DGS_MAX_PEERS; k++) images.p[k] = nullptr;
    if (peer_images) {
        if (shard_count != peer_count || (W & 3)) { set_error("l1_loss_grad_peer: the image exchange needs shard_count == peer_count and W %% 4 == 0"); return H3DGS_EINVAL; }
        images = peer_ptrs(reinterpret_cast<void* const*>(peer_images), peer_count);
    }
    return l1_launch(C, H, W, img, gt, scale, shard_count, shard_index, dL_dimg, nullptr,
                     peer_ptrs(reinterpret_cast<void* const*>(loss_sums), peer_count), images, (cudaStream_t)stream);
}
