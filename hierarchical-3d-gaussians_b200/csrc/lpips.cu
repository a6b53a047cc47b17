// lpips.cu -- LPIPS of one frame pair with the VGG16 network (lpipsPyTorch, v0.1), the third number render_hierarchy.py
// reports per tau.  In the reference's order:
//   x -> (x - mean) / std       mean (-.030, -.088, -.188), std (.458, .448, .450), on the [0,1] input as it is
//   torchvision vgg16().features[0..29]: 13 conv3x3 (pad 1, bias, ReLU), max-pool 2x2/2 (floor) before conv 3, 5, 8, 11;
//   taps = the ReLU outputs of conv 2, 4, 7, 10, 13 (64, 128, 256, 512, 512 channels);
//   per tap: n = f / (sqrt(sum_c f^2) + 1e-10), d = sum_c lin_c (n_x - n_y)^2, mean over the tap's pixels;
//   value = the sum of the five means.
//
// Kernels (all NHWC fp32):
//   lpips_input_kernel  [3,H,W] -> [H][W-x0][8] z-scored (channels 3..7 zero, so that layer 1 is a K = 72 GEMM like the
//                       others); the evaluator form first applies exposure, clamp, crop and mask as metrics.cu does.
//   lpips_conv_kernel   implicit GEMM on TF32 tensor cores (mma.m16n8k8, fp32 accumulate): M = 8x16 output pixels, N =
//                       64 or 128 output channels, K = 9 taps x C_in, in stages of 8 input channels.  A stage is the
//                       10x18-pixel halo tile of those 8 channels plus the 9x8xN weight slice, double-buffered in shared
//                       memory by cp.async; out-of-image pixels are zero-filled, which is the padding.  The nine shifted
//                       windows of the halo tile are the A operands.  Bias and ReLU in the epilogue.
//   lpips_pool_kernel   2x2/2 max-pool, floor.
//   lpips_head_kernel   one warp per pixel: both norms, the weighted squared difference, summed per block in double into
//                       a partials array; lpips_finish_kernel (one thread) sums the partials in a fixed order.
// No floating-point atomics: the same inputs give the same bits, eagerly, graphed and on re-run.  Nothing synchronises
// the host, so every pass can be captured in a CUDA graph.
#include <math.h>
#include <string.h>
#include "common.cuh"
#include "eval_pixel.cuh"
#include "mma.cuh"

namespace h3dgs {
namespace {

constexpr int kLayers = 13, kTaps = 5, kLevels = 5;
constexpr int kCin[kLayers] = {8, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};     // layer 1: 3 padded to 8
constexpr int kCinReal[kLayers] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
constexpr int kCout[kLayers] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
constexpr int kLevel[kLayers] = {0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4};        // resolution level: pools before 2, 4, 7, 10
constexpr int kTapLayer[kTaps] = {1, 3, 6, 9, 12};
constexpr int kTapC[kTaps] = {64, 128, 256, 512, 512};
constexpr int kInC = 8;                                                          // channels of the network input

// ---- packed weights: per layer [9 taps][C_in][C_out] (TF32-rounded) then bias [C_out]; then lin 0..4 ----
size_t conv_offset(int l) {
    size_t o = 0;
    for (int i = 0; i < l; i++) o += (size_t)9 * kCin[i] * kCout[i] + kCout[i];
    return o;
}
size_t lin_offset(int k) {
    size_t o = conv_offset(kLayers);
    for (int i = 0; i < k; i++) o += kTapC[i];
    return o;
}

// cvt.rna.tf32.f32 on the host: round to 10 mantissa bits, ties away from zero
float tf32_rna(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) != 0x7f800000u) { u += 0x1000u; u &= 0xffffe000u; }
    memcpy(&x, &u, 4);
    return x;
}

// ---- input ----
__global__ void lpips_input_kernel(int H, int W, int x0, const float* __restrict__ frame, const float* __restrict__ exposure,
                                   const float* __restrict__ mask, int clamp, float* __restrict__ out)
{
    const int Wc = W - x0;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * Wc) return;
    const int y = i / Wc, x = i - y * Wc;
    const size_t plane = (size_t)H * W, p = (size_t)y * W + x0 + x;
    const float mean[3] = {-.030f, -.088f, -.188f}, stdv[3] = {.458f, .448f, .450f};
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float a = clamp ? eval_value(frame, exposure, plane, p, c) : frame[(size_t)c * plane + p];
        if (mask) a *= mask[p];
        v[c] = (a - mean[c]) / stdv[c];
    }
    float4* o = reinterpret_cast<float4*>(out + (size_t)i * kInC);
    o[0] = make_float4(v[0], v[1], v[2], 0.f);
    o[1] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// ---- conv3x3 + bias + ReLU ----
constexpr int kTH = 8, kTW = 16, kHH = kTH + 2, kHW = kTW + 2;      // output tile, halo tile
constexpr int kCK = 8;                                               // input channels per stage: one k8 step per tap
constexpr int kAP = 12;              // halo pixel stride in floats: 8 + 4 makes the A fragment loads conflict-free
constexpr int kConvThreads = 256;    // 8 warps: 4 along M (two tile rows each) x 2 along N
constexpr int kAStage = kHH * kHW * kAP;
template <int BN> constexpr int b_stride() { return BN + 8; }        // + 8: conflict-free B fragment loads
template <int BN> constexpr int b_stage() { return 9 * kCK * b_stride<BN>(); }
template <int BN> constexpr size_t conv_smem() { return 2 * (size_t)(kAStage + b_stage<BN>()) * sizeof(float); }

template <int BN>
__global__ void __launch_bounds__(kConvThreads)
lpips_conv_kernel(int H, int W, int Cin, int Cout, const float* __restrict__ in, const float* __restrict__ wt,
                  const float* __restrict__ bias, float* __restrict__ out)
{
    extern __shared__ float4 lp_smem[];
    constexpr int kBS = b_stride<BN>(), kBStage = b_stage<BN>(), NT = BN / 16;
    float* sA = reinterpret_cast<float*>(lp_smem);
    float* sB = sA + 2 * kAStage;
    const int tiles_x = (W + kTW - 1) / kTW;
    const int ty0 = (blockIdx.x / tiles_x) * kTH, tx0 = (blockIdx.x % tiles_x) * kTW;
    const int n0 = blockIdx.y * BN;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3, wm = warp & 3, wn = warp >> 2;
    float acc[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
        for (int nt = 0; nt < NT; nt++)
#pragma unroll
            for (int e = 0; e < 4; e++) acc[mt][nt][e] = 0.f;

    const int nchunks = Cin / kCK;
    auto load = [&](int stage, int c0) {
        float* a = sA + stage * kAStage;
        for (int i = tid; i < kHH * kHW * 2; i += kConvThreads) {
            const int pix = i >> 1, half = i & 1;
            const int hy = pix / kHW, hx = pix - hy * kHW;
            const int gy = ty0 + hy - 1, gx = tx0 + hx - 1;
            const bool ok = gy >= 0 && gy < H && gx >= 0 && gx < W;
            cp_async16(a + pix * kAP + 4 * half, ok ? in + ((size_t)gy * W + gx) * Cin + c0 + 4 * half : in, ok);
        }
        float* b = sB + stage * kBStage;
        constexpr int kVec = BN / 4;
        for (int i = tid; i < 9 * kCK * kVec; i += kConvThreads) {
            const int r = i / kVec, v = i - r * kVec;              // r = tap * kCK + k
            const int tap = r / kCK, k = r - tap * kCK;
            cp_async16(b + r * kBS + 4 * v, wt + (size_t)(tap * Cin + c0 + k) * Cout + n0 + 4 * v, true);
        }
        cp_async_commit();
    };

    load(0, 0);
    for (int ch = 0; ch < nchunks; ch++) {
        if (ch + 1 < nchunks) {
            load((ch + 1) & 1, (ch + 1) * kCK);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float* a = sA + (ch & 1) * kAStage;
        const float* b = sB + (ch & 1) * kBStage;
#pragma unroll
        for (int tap = 0; tap < 9; tap++) {
            const int dy = tap / 3, dx = tap % 3;
            uint32_t af[2][4];
#pragma unroll
            for (int mt = 0; mt < 2; mt++) {
                const float* p = a + ((2 * wm + mt + dy) * kHW + g + dx) * kAP + t;
                af[mt][0] = to_tf32(p[0]);
                af[mt][1] = to_tf32(p[8 * kAP]);
                af[mt][2] = to_tf32(p[4]);
                af[mt][3] = to_tf32(p[8 * kAP + 4]);
            }
#pragma unroll
            for (int nt = 0; nt < NT; nt++) {
                const float* q = b + (tap * kCK + t) * kBS + wn * (BN / 2) + nt * 8 + g;
                const uint32_t bf[2] = {__float_as_uint(q[0]), __float_as_uint(q[4 * kBS])};     // packed already TF32
                mma_tf32_16x8x8(acc[0][nt], af[0], bf);
                mma_tf32_16x8x8(acc[1][nt], af[1], bf);
            }
        }
        __syncthreads();
    }

#pragma unroll
    for (int mt = 0; mt < 2; mt++) {
        const int y = ty0 + 2 * wm + mt;
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
            const int x = tx0 + g + 8 * hf;
            if (y >= H || x >= W) continue;
            float* o = out + ((size_t)y * W + x) * Cout + n0 + wn * (BN / 2) + 2 * t;
#pragma unroll
            for (int nt = 0; nt < NT; nt++) {
                const int n = n0 + wn * (BN / 2) + nt * 8 + 2 * t;
                *reinterpret_cast<float2*>(o + nt * 8) = make_float2(fmaxf(acc[mt][nt][2 * hf] + bias[n], 0.f),
                                                                     fmaxf(acc[mt][nt][2 * hf + 1] + bias[n + 1], 0.f));
            }
        }
    }
}

// ---- 2x2/2 max-pool: in [H][W][C] -> out [H/2][W/2][C] ----
__global__ void lpips_pool_kernel(int H, int W, int C, const float* __restrict__ in, float* __restrict__ out)
{
    const int C4 = C / 4, Ho = H / 2, Wo = W / 2;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)Ho * Wo * C4) return;
    const int c4 = (int)(i % C4);
    const size_t px = i / C4;
    const int yo = (int)(px / Wo), xo = (int)(px - (size_t)yo * Wo);
    const float4* p = reinterpret_cast<const float4*>(in) + ((size_t)(2 * yo) * W + 2 * xo) * C4 + c4;
    const float4 a = p[0], b = p[C4], c = p[(size_t)W * C4], d = p[(size_t)W * C4 + C4];
    reinterpret_cast<float4*>(out)[i] = make_float4(fmaxf(fmaxf(a.x, b.x), fmaxf(c.x, d.x)), fmaxf(fmaxf(a.y, b.y), fmaxf(c.y, d.y)),
                                                    fmaxf(fmaxf(a.z, b.z), fmaxf(c.z, d.z)), fmaxf(fmaxf(a.w, b.w), fmaxf(c.w, d.w)));
}

// ---- head ----
constexpr int kHeadWarps = 8, kHeadPix = 64;         // pixels per warp; a block covers 512 pixels

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// fx, fy: [npix][C] taps; partials[blockIdx.x] = sum over the block's pixels of sum_c lin_c (n_x - n_y)^2
template <int C>
__global__ void __launch_bounds__(kHeadWarps * 32)
lpips_head_kernel(int npix, const float* __restrict__ fx, const float* __restrict__ fy, const float* __restrict__ lin,
                  double* __restrict__ partials)
{
    __shared__ double s_warp[kHeadWarps];
    constexpr int V = C / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float w[V];
#pragma unroll
    for (int j = 0; j < V; j++) w[j] = lin[j * 32 + lane];
    double acc = 0.0;
    const int p0 = (blockIdx.x * kHeadWarps + warp) * kHeadPix;
    for (int k = 0; k < kHeadPix && p0 + k < npix; k++) {
        const float* a = fx + (size_t)(p0 + k) * C;
        const float* b = fy + (size_t)(p0 + k) * C;
        float xa[V], xb[V], sa = 0.f, sb = 0.f;
#pragma unroll
        for (int j = 0; j < V; j++) {
            xa[j] = a[j * 32 + lane]; xb[j] = b[j * 32 + lane];
            sa += xa[j] * xa[j]; sb += xb[j] * xb[j];
        }
        const float na = sqrtf(warp_sum(sa)) + 1e-10f, nb = sqrtf(warp_sum(sb)) + 1e-10f;
        float d = 0.f;
#pragma unroll
        for (int j = 0; j < V; j++) {
            const float e = xa[j] / na - xb[j] / nb;
            d += w[j] * (e * e);
        }
        acc += (double)warp_sum(d);
    }
    if (lane == 0) s_warp[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < kHeadWarps; i++) s += s_warp[i];
        partials[blockIdx.x] = s;
    }
}

struct HeadPlan { int blocks[kTaps]; double pixels[kTaps]; };

// one thread: the five taps' partials, each in order, / pixels, summed in tap order -> out[slot]
__global__ void lpips_finish_kernel(const double* __restrict__ partials, HeadPlan plan, const int* __restrict__ counter,
                                    double* __restrict__ out, int max_rows)
{
    double v = 0.0;
    for (int k = 0; k < kTaps; k++) {
        double s = 0.0;
        for (int b = 0; b < plan.blocks[k]; b++) s += partials[b];
        partials += plan.blocks[k];
        v += s / plan.pixels[k];
    }
    const int slot = counter ? *counter - 1 : 0;
    if (slot >= 0 && slot < max_rows) out[slot] = v;
}

// ---- host driver ----
struct Levels { int h[kLevels], w[kLevels]; };
Levels levels(int H, int Wc) {
    Levels L;
    L.h[0] = H; L.w[0] = Wc;
    for (int i = 1; i < kLevels; i++) { L.h[i] = L.h[i - 1] / 2; L.w[i] = L.w[i - 1] / 2; }
    return L;
}
int head_blocks(int npix) { return (npix + kHeadWarps * kHeadPix - 1) / (kHeadWarps * kHeadPix); }

template <int BN>
int launch_conv_bn(int H, int W, int Cin, int Cout, const float* in, const float* wt, const float* b, float* out, cudaStream_t s) {
    static bool attr = false;
    if (!attr) {
        H3_CUDA(cudaFuncSetAttribute(lpips_conv_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)conv_smem<BN>()));
        attr = true;
    }
    const dim3 grid(((W + kTW - 1) / kTW) * ((H + kTH - 1) / kTH), Cout / BN);
    lpips_conv_kernel<BN><<<grid, kConvThreads, conv_smem<BN>(), s>>>(H, W, Cin, Cout, in, wt, b, out);
    H3_LAUNCHED("lpips_conv", 0, s);
    return H3DGS_OK;
}

int launch_conv(int l, int H, int W, const float* in, const float* weights, float* out, cudaStream_t s) {
    const float* wt = weights + conv_offset(l);
    const float* b = wt + (size_t)9 * kCin[l] * kCout[l];
    return kCout[l] == 64 ? launch_conv_bn<64>(H, W, kCin[l], kCout[l], in, wt, b, out, s)
                          : launch_conv_bn<128>(H, W, kCin[l], kCout[l], in, wt, b, out, s);
}

int launch_head(int k, int npix, const float* fx, const float* fy, const float* lin, double* partials, cudaStream_t s) {
    const int nb = head_blocks(npix), nt = kHeadWarps * 32;
    switch (kTapC[k]) {
    case 64: lpips_head_kernel<64><<<nb, nt, 0, s>>>(npix, fx, fy, lin, partials); break;
    case 128: lpips_head_kernel<128><<<nb, nt, 0, s>>>(npix, fx, fy, lin, partials); break;
    case 256: lpips_head_kernel<256><<<nb, nt, 0, s>>>(npix, fx, fy, lin, partials); break;
    default: lpips_head_kernel<512><<<nb, nt, 0, s>>>(npix, fx, fy, lin, partials); break;
    }
    H3_LAUNCHED("lpips_head", 0, s);
    return H3DGS_OK;
}

bool lpips_size_ok(int H, int W, int x0) {
    if (H < H3DGS_LPIPS_MIN_SIZE || W - x0 < H3DGS_LPIPS_MIN_SIZE) {
        set_error("lpips: a %d x %d frame leaves a zero-size pooling level (both sides need >= %d pixels)", H, W - x0,
                  H3DGS_LPIPS_MIN_SIZE);
        return false;
    }
    return true;
}

// The network on one frame.  taps_out: store the taps there (the target side); taps_ref: compare each tap against the
// stored one, head partials into `partials` (the image side).
int run_net(int H, int W, int x0, const float* frame, const float* exposure, const float* mask, int clamp,
            const float* weights, float* act, float* taps_out, const float* taps_ref, double* partials, cudaStream_t s)
{
    const int Wc = W - x0;
    const Levels lv = levels(H, Wc);
    float* P = act;
    float* Q = act + (size_t)H * Wc * 64;
    const int npix = H * Wc;
    lpips_input_kernel<<<(npix + 255) / 256, 256, 0, s>>>(H, W, x0, frame, exposure, mask, clamp, P);
    H3_LAUNCHED("lpips_input", 0, s);
    float* cur = P;
    size_t tap_off = 0;
    int tap = 0;
    for (int l = 0; l < kLayers; l++) {
        const int lvl = kLevel[l];
        if (l > 0 && lvl != kLevel[l - 1]) {
            float* dst = cur == P ? Q : P;
            const int n4 = lv.h[lvl] * lv.w[lvl] * (kCout[l - 1] / 4);
            lpips_pool_kernel<<<(n4 + 255) / 256, 256, 0, s>>>(lv.h[lvl - 1], lv.w[lvl - 1], kCout[l - 1], cur, dst);
            H3_LAUNCHED("lpips_pool", 0, s);
            cur = dst;
        }
        const bool is_tap = l == kTapLayer[tap];
        float* dst = (is_tap && taps_out) ? taps_out + tap_off : (cur == P ? Q : P);
        if (int rc = launch_conv(l, lv.h[lvl], lv.w[lvl], cur, weights, dst, s)) return rc;
        cur = dst;
        if (is_tap) {
            const int np = lv.h[lvl] * lv.w[lvl];
            if (taps_ref) {
                if (int rc = launch_head(tap, np, cur, taps_ref + tap_off, weights + lin_offset(tap), partials, s)) return rc;
                partials += head_blocks(np);
            }
            tap_off += (size_t)np * kTapC[tap];
            tap++;
        }
    }
    return H3DGS_OK;
}

}  // namespace
}  // namespace h3dgs

using namespace h3dgs;

extern "C" int64_t h3dgs_lpips_weight_floats(void) { return (int64_t)lin_offset(kTaps); }

extern "C" int h3dgs_lpips_pack_weights(const float* const* conv_weight, const float* const* conv_bias,
                                        const float* const* lin_weight, float* packed)
{
    if (!conv_weight || !conv_bias || !lin_weight || !packed) { set_error("lpips_pack_weights: bad arguments"); return H3DGS_EINVAL; }
    for (int l = 0; l < kLayers; l++) {
        const int ci = kCin[l], cr = kCinReal[l], co = kCout[l];
        if (!conv_weight[l] || !conv_bias[l]) { set_error("lpips_pack_weights: layer %d missing", l); return H3DGS_EINVAL; }
        float* w = packed + conv_offset(l);
        for (int tap = 0; tap < 9; tap++)
            for (int i = 0; i < ci; i++)
                for (int o = 0; o < co; o++)
                    w[((size_t)tap * ci + i) * co + o] = i < cr ? tf32_rna(conv_weight[l][((size_t)o * cr + i) * 9 + tap]) : 0.f;
        memcpy(w + (size_t)9 * ci * co, conv_bias[l], co * sizeof(float));
    }
    for (int k = 0; k < kTaps; k++) {
        if (!lin_weight[k]) { set_error("lpips_pack_weights: lin %d missing", k); return H3DGS_EINVAL; }
        memcpy(packed + lin_offset(k), lin_weight[k], kTapC[k] * sizeof(float));
    }
    return H3DGS_OK;
}

extern "C" int h3dgs_lpips_scratch_floats(int32_t H, int32_t Wc, int64_t* act_floats, int64_t* tap_floats,
                                          int64_t* partial_doubles)
{
    if (!lpips_size_ok(H, Wc, 0)) return H3DGS_EINVAL;
    const Levels lv = levels(H, Wc);
    int64_t taps = 0, parts = 0;
    for (int k = 0; k < kTaps; k++) {
        const int np = lv.h[kLevel[kTapLayer[k]]] * lv.w[kLevel[kTapLayer[k]]];
        taps += (int64_t)np * kTapC[k];
        parts += head_blocks(np);
    }
    if (act_floats) *act_floats = 2 * (int64_t)H * Wc * 64;
    if (tap_floats) *tap_floats = taps;
    if (partial_doubles) *partial_doubles = parts;
    return H3DGS_OK;
}

extern "C" int h3dgs_lpips_features(int32_t H, int32_t W, int32_t x0, const float* frame, const float* exposure,
                                    const float* mask, int32_t clamp, const float* weights, float* act, float* taps,
                                    void* stream)
{
    if (H <= 0 || W <= 0 || x0 < 0 || x0 >= W || !frame || !weights || !act || !taps) {
        set_error("lpips_features: bad arguments"); return H3DGS_EINVAL;
    }
    if (!lpips_size_ok(H, W, x0)) return H3DGS_EINVAL;
    return run_net(H, W, x0, frame, exposure, mask, clamp, weights, act, taps, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" int h3dgs_lpips_distance(int32_t H, int32_t W, int32_t x0, const float* frame, const float* exposure,
                                    const float* mask, int32_t clamp, const float* weights, float* act, const float* taps,
                                    double* partials, const int32_t* counter, double* out, int32_t max_rows, void* stream)
{
    if (H <= 0 || W <= 0 || x0 < 0 || x0 >= W || !frame || !weights || !act || !taps || !partials || !out || max_rows <= 0) {
        set_error("lpips_distance: bad arguments"); return H3DGS_EINVAL;
    }
    if (!lpips_size_ok(H, W, x0)) return H3DGS_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    if (int rc = run_net(H, W, x0, frame, exposure, mask, clamp, weights, act, nullptr, taps, partials, s)) return rc;
    const Levels lv = levels(H, W - x0);
    HeadPlan plan;
    for (int k = 0; k < kTaps; k++) {
        const int lvl = kLevel[kTapLayer[k]];
        plan.blocks[k] = head_blocks(lv.h[lvl] * lv.w[lvl]);
        plan.pixels[k] = (double)lv.h[lvl] * (double)lv.w[lvl];
    }
    lpips_finish_kernel<<<1, 1, 0, s>>>(partials, plan, counter, out, max_rows);
    H3_LAUNCHED("lpips_finish", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_lpips_conv(int32_t layer, int32_t H, int32_t W, const float* in, const float* weights, float* out,
                                void* stream)
{
    if (layer < 0 || layer >= kLayers || H <= 0 || W <= 0 || !in || !weights || !out) {
        set_error("lpips_conv: bad arguments"); return H3DGS_EINVAL;
    }
    return launch_conv(layer, H, W, in, weights, out, (cudaStream_t)stream);
}
