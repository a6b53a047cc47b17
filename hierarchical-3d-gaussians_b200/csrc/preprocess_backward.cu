// preprocess_backward.cu -- K8 + K9 fused: per-Gaussian chain rule from the 2D-space
// accumulators (dmean2D, dconic, dopacity, dcolor, dinvdepth) back to the inputs
// (replaces BACKWARD::computeCov2DCUDA + BACKWARD::preprocessCUDA).  Semantics per
// oracle/oracle.c::oracle_preprocess_backward.  The covariance chain (K8, K9c) lives in
// cov_grad.cuh: fp32 except the 2x2 screen covariance and the gradient of its inverse (~50 fp64
// operations), which is where the published formulas cancel.  One thread per Gaussian; a pure HBM
// stream: reads 40 B accum + 44 B params + 192 B SH, writes 248 B of gradients.
// Every output row is written (zeros for culled Gaussians) so the caller never
// pays a separate memset pass over the gradient tensors.  Two launches -- the fp64 covariance
// chain (preprocess_backward_kernel) and the SH part (sh_backward_kernel) -- because fused they
// needed 189 registers (11 % warp occupancy, latency-bound at a third of the DRAM roofline).
#include "common.cuh"
#include "cov_grad.cuh"

namespace h3dgs {

__device__ __constant__ float bSH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                           -1.0925484305920792f, 0.5462742152960396f};
__device__ __constant__ float bSH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                           0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                           -0.5900435899266435f};
constexpr float bSH_C0 = 0.28209479177387814f;
constexpr float bSH_C1 = 0.4886025119029199f;

__device__ __forceinline__ void store_zero(float* p, int n) {
    for (int k = 0; k < n; k++) p[k] = 0.f;
}

__global__ void __launch_bounds__(128)
preprocess_backward_kernel(int row0, int P, const RowCycle cyc, int deg, int M, const float* __restrict__ means3D, const float* __restrict__ scales,
                           float scale_mod, const float* __restrict__ rots, const float* __restrict__ shs,
                           const float* __restrict__ cov3D_precomp, const float* __restrict__ colors_precomp,
                           const float* __restrict__ ts, const int* __restrict__ ridx, const int* __restrict__ pidx,
                           const float* __restrict__ view, const float* __restrict__ proj,
                           const float* __restrict__ campos, int W, int H, float tanx, float tany, float fx, float fy,
                           int use_depth, const int* __restrict__ radii, const uint8_t* __restrict__ rank_mask, const StagePtrs peers,
                           const Record* __restrict__ records,
                           const float* __restrict__ accum, float* __restrict__ dL_dmeans3D,
                           float* __restrict__ dL_dmeans2D, float* __restrict__ dL_dsh, float* __restrict__ dL_dcolors,
                           float* __restrict__ dL_dopacities, float* __restrict__ dL_dscales,
                           float* __restrict__ dL_drots, float* __restrict__ dL_dcov3D)
{
    __shared__ float s_view[16], s_proj[16];
    if (threadIdx.x < 16) { s_view[threadIdx.x] = view[threadIdx.x]; s_proj[threadIdx.x] = proj[threadIdx.x]; }
    __syncthreads();
    const int local = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = cyc.world > 1 ? cyclic_row(cyc, local) : row0 + local;      // rows [row0, P), or the blocks this rank owns
    if (i >= P) return;

    if (radii[i] <= 0) {
        store_zero(dL_dmeans2D + 3 * i, 3);
        if (ridx) return;                    // scatter mode: full-size gradients are pre-zeroed
        store_zero(dL_dmeans3D + 3 * i, 3);
        dL_dopacities[i] = 0.f;
        if (dL_dcolors) store_zero(dL_dcolors + 3 * i, 3);
        if (dL_dscales) store_zero(dL_dscales + 3 * i, 3);
        if (dL_drots) store_zero(dL_drots + 4 * i, 4);
        if (dL_dcov3D) store_zero(dL_dcov3D + 6 * i, 6);
        return;
    }

    const float* v = s_view;
    float ac[kAccum];
    if (peers.n > 1) gather_accum_pairs<5>(peers, rank_mask[i], i, 0, ac);    // the partial sums of the ranks that touch row i
    else {
        const float2* row = reinterpret_cast<const float2*>(accum + (size_t)i * kAccum);
#pragma unroll
        for (int k = 0; k < 5; k++) { const float2 v = row[k]; ac[2 * k] = v.x; ac[2 * k + 1] = v.y; }
    }
    // the per-tile replay leaves its constant factors to us: d(pixel)/d(ndc) = 0.5 W, 0.5 H and the
    // -1/2 of the quadratic form
    const float g_mx = ac[0] * (0.5f * W), g_my = ac[1] * (0.5f * H);
    const float dcx = -0.5f * ac[2], dcy = -0.5f * ac[3], dcz = -0.5f * ac[4], g_op = ac[5];
    const float g_r = ac[6], g_g = ac[7], g_b = ac[8], g_iv = ac[9];
    // gather + parent lerp exactly as the forward did (preprocess.cu)
    int c = i, p = i;
    float t = 1.0f, u = 0.0f;
    if (ridx) {
        c = ridx[i]; p = pidx[i]; if (p < 0) p = c;
        t = ts[i]; u = 1.0f - t;
    }
    const bool lerp = ridx != nullptr && u != 0.0f;
#define LERP(a, b) (lerp ? __fadd_rn(__fmul_rn(t, (a)), __fmul_rn(u, (b))) : (a))
    const float mx = LERP(means3D[3 * c], means3D[3 * p]);
    const float my = LERP(means3D[3 * c + 1], means3D[3 * p + 1]);
    const float mz = LERP(means3D[3 * c + 2], means3D[3 * p + 2]);
    float qsign = 1.0f;

    // cov3D (recomputed in fp32 exactly as the forward does: cheaper than a 24-B round trip through HBM)
    float cov6[6], R[3][3], Mm[3][3], sc[3], qv[4] = {1.f, 0.f, 0.f, 0.f};
    const bool have_sr = cov3D_precomp == nullptr;
    if (!have_sr) {
#pragma unroll
        for (int k = 0; k < 6; k++) cov6[k] = cov3D_precomp[6 * c + k];
    } else {
        float4 qq = *reinterpret_cast<const float4*>(rots + 4 * c);
        if (lerp) {
            float4 qp = *reinterpret_cast<const float4*>(rots + 4 * p);
            const float dot = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(qq.x, qp.x), __fmul_rn(qq.y, qp.y)), __fmul_rn(qq.z, qp.z)), __fmul_rn(qq.w, qp.w));
            if (dot < 0.f) qsign = -1.0f;
            qq.x = LERP(qq.x, qsign * qp.x); qq.y = LERP(qq.y, qsign * qp.y);
            qq.z = LERP(qq.z, qsign * qp.z); qq.w = LERP(qq.w, qsign * qp.w);
        }
        qv[0] = qq.x; qv[1] = qq.y; qv[2] = qq.z; qv[3] = qq.w;
#pragma unroll
        for (int k = 0; k < 3; k++) sc[k] = scale_mod * LERP(scales[3 * c + k], scales[3 * p + k]);
        cov3d_from_scale_quat(sc, qv, R, Mm, cov6);
    }

    // ---- K8 + K9c: conic -> cov2D -> cov3D -> scale / rotation, and the mean through the Jacobian
    // (cov_grad.cuh: fp32 with the 2x2 screen covariance and the gradient of its inverse in fp64) ----
    CovGradOut cg;
    cov_chain_backward(v, mx, my, mz, fx, fy, tanx, tany, kFovClamp, kDilation, cov6, dcx, dcy, dcz, g_iv, use_depth != 0,
                       have_sr, sc, qv, R, Mm, scale_mod, cg);
    float dmean[3] = {cg.dmean[0], cg.dmean[1], cg.dmean[2]};
    // ---- K9a: screen-space mean -> 3D mean ----
    {
        const float* q = s_proj;
        const float hw = q[3] * mx + q[7] * my + q[11] * mz + q[15];
        const float m_w = 1.0f / (hw + kWEps);
        const float mul1 = (q[0] * mx + q[4] * my + q[8] * mz + q[12]) * m_w * m_w;
        const float mul2 = (q[1] * mx + q[5] * my + q[9] * mz + q[13]) * m_w * m_w;
        dmean[0] += (q[0] * m_w - q[3] * mul1) * g_mx + (q[1] * m_w - q[3] * mul2) * g_my;
        dmean[1] += (q[4] * m_w - q[7] * mul1) * g_mx + (q[5] * m_w - q[7] * mul2) * g_my;
        dmean[2] += (q[8] * m_w - q[11] * mul1) * g_mx + (q[9] * m_w - q[11] * mul2) * g_my;
    }
    dL_dmeans2D[3 * i] = g_mx; dL_dmeans2D[3 * i + 1] = g_my; dL_dmeans2D[3 * i + 2] = 0.f;
    // EMIT: direct store (flat / pre-gathered inputs) or t / (1-t) scatter into the full-size
    // gradients (red.global.add; a parent row is shared by its k children)
#define EMIT(ptr, width, k, val)                                                           \
    do {                                                                                   \
        const float v__ = (val);                                                           \
        if (!ridx) (ptr)[(size_t)i * (width) + (k)] = v__;                                 \
        else {                                                                             \
            atomicAdd((ptr) + (size_t)c * (width) + (k), t * v__);                         \
            if (lerp) atomicAdd((ptr) + (size_t)p * (width) + (k), u * v__);               \
        }                                                                                  \
    } while (0)
    EMIT(dL_dopacities, 1, 0, g_op);

    // ---- K9b (SH -> coefficients and view direction) lives in sh_backward_kernel ----
    if (colors_precomp && dL_dcolors) { dL_dcolors[3 * c] = g_r; dL_dcolors[3 * c + 1] = g_g; dL_dcolors[3 * c + 2] = g_b; }
    EMIT(dL_dmeans3D, 3, 0, dmean[0]); EMIT(dL_dmeans3D, 3, 1, dmean[1]); EMIT(dL_dmeans3D, 3, 2, dmean[2]);

    // ---- K9c outputs ----
    if (!have_sr) {
        if (dL_dcov3D) {
#pragma unroll
            for (int k = 0; k < 6; k++) dL_dcov3D[6 * c + k] = cg.g6[k];
        }
    } else {
#pragma unroll
        for (int k = 0; k < 3; k++) EMIT(dL_dscales, 3, k, cg.dscale[k]);
        const float4 dq = make_float4(cg.dq[0], cg.dq[1], cg.dq[2], cg.dq[3]);
        if (!ridx) *reinterpret_cast<float4*>(dL_drots + 4 * i) = dq;
        else {
            atomicAdd(reinterpret_cast<float4*>(dL_drots) + c, make_float4(t * dq.x, t * dq.y, t * dq.z, t * dq.w));
            if (lerp) {
                const float us = u * qsign;
                atomicAdd(reinterpret_cast<float4*>(dL_drots) + p, make_float4(us * dq.x, us * dq.y, us * dq.z, us * dq.w));
            }
        }
    }
#undef EMIT
#undef LERP
}

// SH basis and its derivatives w.r.t. the unit direction (coefficient-major rows [k][3]); zero past degree deg
__device__ __forceinline__ void sh_basis(int deg, float x, float y, float z, float (&B)[16], float (&Bx)[16], float (&By)[16],
                                         float (&Bz)[16])
{
#pragma unroll
    for (int k = 0; k < 16; k++) { B[k] = 0.f; Bx[k] = 0.f; By[k] = 0.f; Bz[k] = 0.f; }
    B[0] = bSH_C0;
    if (deg > 0) {
        B[1] = -bSH_C1 * y; B[2] = bSH_C1 * z; B[3] = -bSH_C1 * x;
        By[1] = -bSH_C1; Bz[2] = bSH_C1; Bx[3] = -bSH_C1;
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            B[4] = bSH_C2[0] * xy; B[5] = bSH_C2[1] * yz; B[6] = bSH_C2[2] * (2.f * zz - xx - yy);
            B[7] = bSH_C2[3] * xz; B[8] = bSH_C2[4] * (xx - yy);
            Bx[4] = bSH_C2[0] * y; By[4] = bSH_C2[0] * x;
            By[5] = bSH_C2[1] * z; Bz[5] = bSH_C2[1] * y;
            Bx[6] = bSH_C2[2] * 2.f * -x; By[6] = bSH_C2[2] * 2.f * -y; Bz[6] = bSH_C2[2] * 2.f * 2.f * z;
            Bx[7] = bSH_C2[3] * z; Bz[7] = bSH_C2[3] * x;
            Bx[8] = bSH_C2[4] * 2.f * x; By[8] = bSH_C2[4] * 2.f * -y;
            if (deg > 2) {
                B[9] = bSH_C3[0] * y * (3.f * xx - yy); B[10] = bSH_C3[1] * xy * z;
                B[11] = bSH_C3[2] * y * (4.f * zz - xx - yy); B[12] = bSH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
                B[13] = bSH_C3[4] * x * (4.f * zz - xx - yy); B[14] = bSH_C3[5] * z * (xx - yy);
                B[15] = bSH_C3[6] * x * (xx - 3.f * yy);
                Bx[9] = bSH_C3[0] * 3.f * 2.f * xy;   By[9] = bSH_C3[0] * 3.f * (xx - yy);
                Bx[10] = bSH_C3[1] * yz;              By[10] = bSH_C3[1] * xz;               Bz[10] = bSH_C3[1] * xy;
                Bx[11] = bSH_C3[2] * -2.f * xy;       By[11] = bSH_C3[2] * (-3.f * yy + 4.f * zz - xx); Bz[11] = bSH_C3[2] * 4.f * 2.f * yz;
                Bx[12] = bSH_C3[3] * -3.f * 2.f * xz; By[12] = bSH_C3[3] * -3.f * 2.f * yz;  Bz[12] = bSH_C3[3] * 3.f * (2.f * zz - xx - yy);
                Bx[13] = bSH_C3[4] * (-3.f * xx + 4.f * zz - yy); By[13] = bSH_C3[4] * -2.f * xy; Bz[13] = bSH_C3[4] * 4.f * 2.f * xz;
                Bx[14] = bSH_C3[5] * 2.f * xz;        By[14] = bSH_C3[5] * -2.f * yz;        Bz[14] = bSH_C3[5] * (xx - yy);
                Bx[15] = bSH_C3[6] * 3.f * (xx - yy); By[15] = bSH_C3[6] * -3.f * 2.f * xy;
            }
        }
    }
}

// dL/d(unit direction) -> dL/dmean through the normalisation of d0 = mean - campos
__device__ __forceinline__ void dir_grad_to_mean(float d0x, float d0y, float d0z, float ddx, float ddy, float ddz,
                                                 float& dm0, float& dm1, float& dm2)
{
    const float sum2 = d0x * d0x + d0y * d0y + d0z * d0z;
    const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
    dm0 = ((sum2 - d0x * d0x) * ddx - d0y * d0x * ddy - d0z * d0x * ddz) * invsum32;
    dm1 = (-d0x * d0y * ddx + (sum2 - d0y * d0y) * ddy - d0z * d0y * ddz) * invsum32;
    dm2 = (-d0x * d0z * ddx - d0y * d0z * ddy + (sum2 - d0z * d0z) * ddz) * invsum32;
}

// K9b: dL/dcolour -> dL/dSH (basis x dL/dRGB, no intermediate array) and, through the view
// direction, an ADDITIVE term of dL/dmean (runs after preprocess_backward_kernel on the stream).
// One thread per Gaussian.  Flat mode, and scatter mode when 3 M is not a multiple of 4; scatter mode with float4 rows
// takes sh_backward_rows_kernel.
__global__ void __launch_bounds__(128)
sh_backward_kernel(int row0, int P, const RowCycle cyc, int deg, int M, const float* __restrict__ means3D, const float* __restrict__ shs,
                   const float* __restrict__ ts, const int* __restrict__ ridx, const int* __restrict__ pidx,
                   const float* __restrict__ campos, const int* __restrict__ radii, const uint8_t* __restrict__ rank_mask,
                   const StagePtrs peers, const Record* __restrict__ records,
                   const float* __restrict__ accum, float* __restrict__ dL_dmeans3D, float* __restrict__ dL_dsh)
{
    const int local = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = cyc.world > 1 ? cyclic_row(cyc, local) : row0 + local;      // rows [row0, P), or the blocks this rank owns
    if (i >= P) return;
    const int SH3 = M * 3;
    if (radii[i] <= 0) {
        if (!ridx) {                                   // scatter mode: full-size gradients are pre-zeroed
            float* o = dL_dsh + (size_t)i * SH3;
            if ((SH3 & 3) == 0) { for (int k = 0; k < SH3 / 4; k++) reinterpret_cast<float4*>(o)[k] = make_float4(0, 0, 0, 0); }
            else store_zero(o, SH3);
        }
        return;
    }
    int c = i, p = i;
    float t = 1.0f, u = 0.0f;
    if (ridx) {
        c = ridx[i]; p = pidx[i]; if (p < 0) p = c;
        t = ts[i]; u = 1.0f - t;
    }
    const bool lerp = ridx != nullptr && u != 0.0f;
#define LERP(a, b) (lerp ? __fadd_rn(__fmul_rn(t, (a)), __fmul_rn(u, (b))) : (a))
    const float mx = LERP(means3D[3 * c], means3D[3 * p]);
    const float my = LERP(means3D[3 * c + 1], means3D[3 * p + 1]);
    const float mz = LERP(means3D[3 * c + 2], means3D[3 * p + 2]);
    float col[4];                                          // accum columns 6..9: dL/dRGB (and dL/dinvdepth, unused here)
    if (peers.n > 1) gather_accum_pairs<2>(peers, rank_mask[i], i, 3, col);
    else { const float* ac = accum + (size_t)i * kAccum; col[0] = ac[6]; col[1] = ac[7]; col[2] = ac[8]; }
    const uint32_t kb = __float_as_uint(records[i].b.w);
    const float dRGB[3] = {(kb >> kClampShift) & 1u ? 0.f : col[0], (kb >> (kClampShift + 1)) & 1u ? 0.f : col[1],
                           (kb >> (kClampShift + 2)) & 1u ? 0.f : col[2]};
    const float d0x = mx - campos[0], d0y = my - campos[1], d0z = mz - campos[2];
    const float len = sqrtf(d0x * d0x + d0y * d0y + d0z * d0z);
    const float x = d0x / len, y = d0y / len, z = d0z / len;
    const int ncoef = (deg + 1) * (deg + 1);
    float B[16], Bx[16], By[16], Bz[16];
    sh_basis(deg, x, y, z, B, Bx, By, Bz);
    // one pass over the row in 128-bit pieces: float e = 3k + ch.  dL/d(dir) needs the (lerped) coefficients,
    // dL/dSH[k][ch] = B[k] * dRGB[ch] is emitted straight away
    float ddx = 0.f, ddy = 0.f, ddz = 0.f;
    const float* shc = shs + (size_t)c * SH3;
    const float* shp = shs + (size_t)p * SH3;
    float* dshi = dL_dsh + (size_t)i * SH3;
    if ((SH3 & 3) == 0) {
#pragma unroll
        for (int q = 0; q < 12; q++) {
            if (4 * q < SH3) {
                float o4[4] = {0.f, 0.f, 0.f, 0.f};
                if (4 * q < 3 * ncoef) {
                    float4 v = __ldg(reinterpret_cast<const float4*>(shc) + q);
                    if (lerp) {
                        const float4 w = __ldg(reinterpret_cast<const float4*>(shp) + q);
                        v.x = LERP(v.x, w.x); v.y = LERP(v.y, w.y); v.z = LERP(v.z, w.z); v.w = LERP(v.w, w.w);
                    }
                    const float sv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int r = 0; r < 4; r++) {
                        const int e = 4 * q + r, k = e / 3, ch = e - 3 * k;      // compile-time after unrolling
                        const float g = dRGB[ch];
                        o4[r] = B[k] * g;
                        ddx += Bx[k] * sv[r] * g; ddy += By[k] * sv[r] * g; ddz += Bz[k] * sv[r] * g;
                    }
                }
                reinterpret_cast<float4*>(dshi)[q] = make_float4(o4[0], o4[1], o4[2], o4[3]);     // flat mode only
            }
        }
    } else {
#pragma unroll
        for (int e = 0; e < 48; e++) {
            if (e < SH3) {
                const int k = e / 3, ch = e - 3 * k;
                float o = 0.f;
                if (e < 3 * ncoef) {
                    const float sv = LERP(__ldg(shc + e), __ldg(shp + e));
                    const float g = dRGB[ch];
                    o = B[k] * g;
                    ddx += Bx[k] * sv * g; ddy += By[k] * sv * g; ddz += Bz[k] * sv * g;
                }
                if (!ridx) dshi[e] = o;
                else if (e < 3 * ncoef) {
                    atomicAdd(dL_dsh + (size_t)c * SH3 + e, t * o);
                    if (lerp) atomicAdd(dL_dsh + (size_t)p * SH3 + e, u * o);
                }
            }
        }
    }
    float dm0, dm1, dm2;
    dir_grad_to_mean(d0x, d0y, d0z, ddx, ddy, ddz, dm0, dm1, dm2);
    if (!ridx) {       // row i belongs to this thread; preprocess_backward_kernel already stored its part
        dL_dmeans3D[3 * i] += dm0; dL_dmeans3D[3 * i + 1] += dm1; dL_dmeans3D[3 * i + 2] += dm2;
    } else {
        atomicAdd(dL_dmeans3D + 3 * (size_t)c + 0, t * dm0); atomicAdd(dL_dmeans3D + 3 * (size_t)c + 1, t * dm1);
        atomicAdd(dL_dmeans3D + 3 * (size_t)c + 2, t * dm2);
        if (lerp) {
            atomicAdd(dL_dmeans3D + 3 * (size_t)p + 0, u * dm0); atomicAdd(dL_dmeans3D + 3 * (size_t)p + 1, u * dm1);
            atomicAdd(dL_dmeans3D + 3 * (size_t)p + 2, u * dm2);
        }
    }
#undef LERP
}

// K9b in scatter mode with float4 rows (3 M a multiple of 4).  A warp takes 32 consecutive rendered rows in three
// phases, through a per-warp staging area of 32 rows x 13 float4 (one float4 of padding: the row-per-lane reads of
// phase 2 are free of bank conflicts):
//   1. lanes read consecutive 16-B pieces of the rows' own and parent coefficients (every load instruction covers whole
//      32-B sectors) and stage the lerped row;
//   2. one lane per row computes the basis, the view-direction term of dL/dmean (as sh_backward_kernel, in the same
//      order) and overwrites its staged row with dL/dSH = B[k] dRGB[ch];
//   3. lanes write consecutive pieces again.  The own row (t x the piece) is STORED when row_count says that this
//      rendered row is the only writer of that full-size row -- the row was zero-filled, so a store gives what the
//      reduction gives, and a store covering whole sectors needs no read of the evicted zero line -- and reduced
//      otherwise (row_count NULL: always).  A run of consecutive rows with the same parent (siblings are emitted next to
//      each other) sums its (1 - t) x pieces in registers and reduces each parent piece once.
constexpr int kShStage = 13;                 // float4 per staged row: up to 12 pieces + 1 of padding

__global__ void __launch_bounds__(128, 4)
sh_backward_rows_kernel(int row0, int P, const RowCycle cyc, int deg, int M, const float* __restrict__ means3D,
                        const float* __restrict__ shs, const float* __restrict__ ts, const int* __restrict__ ridx,
                        const int* __restrict__ pidx, const float* __restrict__ campos, const int* __restrict__ radii,
                        const uint8_t* __restrict__ rank_mask, const StagePtrs peers, const Record* __restrict__ records,
                        const float* __restrict__ accum, const int* __restrict__ row_count, float* __restrict__ dL_dmeans3D,
                        float* __restrict__ dL_dsh)
{
    __shared__ float4 s_row[4][32][kShStage];
    __shared__ int s_c[4][32], s_p[4][32], s_store[4][32];
    __shared__ float s_t[4][32], s_u[4][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int local = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = cyc.world > 1 ? cyclic_row(cyc, local) : row0 + local;      // rows [row0, P), or the blocks this rank owns
    const int SH3 = M * 3, NQ = SH3 / 4;
    const int ncoef = (deg + 1) * (deg + 1);
    const int nq = min(NQ, (3 * ncoef + 3) / 4);                             // pieces that hold coefficients
    const bool valid = i < P && radii[i] > 0;
    int c = -1, p = -1;
    float t = 1.0f, u = 0.0f;
    if (valid) {
        c = ridx[i]; p = pidx[i]; if (p < 0) p = c;
        t = ts[i]; u = 1.0f - t;
    }
    const bool lerp = valid && u != 0.0f;
    s_c[w][lane] = c; s_p[w][lane] = lerp ? p : -1; s_t[w][lane] = t; s_u[w][lane] = u;
    s_store[w][lane] = valid && row_count != nullptr && row_count[c] == 1;
    __syncwarp();
#define LERP(a, b, tt, uu) __fadd_rn(__fmul_rn((tt), (a)), __fmul_rn((uu), (b)))
    // ---- 1. stage the lerped rows: piece q of row r is item r * NQ + q, item lane + 32 m goes to lane `lane`; six
    // items per lane in flight at a time ----
#pragma unroll
    for (int h = 0; h < 12; h += 6) {
        float4 v[6], pv[6];
#pragma unroll
        for (int j = 0; j < 6; j++) {
            const int m = h + j, it = lane + 32 * m, r = it / NQ, q = it - r * NQ;
            if (m < NQ && q < nq && s_c[w][r] >= 0) {
                v[j] = __ldg(reinterpret_cast<const float4*>(shs + (size_t)s_c[w][r] * SH3) + q);
                if (s_p[w][r] >= 0) pv[j] = __ldg(reinterpret_cast<const float4*>(shs + (size_t)s_p[w][r] * SH3) + q);
            }
        }
#pragma unroll
        for (int j = 0; j < 6; j++) {
            const int m = h + j, it = lane + 32 * m, r = it / NQ, q = it - r * NQ;
            if (m < NQ && q < nq && s_c[w][r] >= 0) {
                float4 a = v[j];
                if (s_p[w][r] >= 0) {
                    const float tt = s_t[w][r], uu = s_u[w][r];
                    const float4 b = pv[j];
                    a.x = LERP(a.x, b.x, tt, uu); a.y = LERP(a.y, b.y, tt, uu);
                    a.z = LERP(a.z, b.z, tt, uu); a.w = LERP(a.w, b.w, tt, uu);
                }
                s_row[w][r][q] = a;
            }
        }
    }
    __syncwarp();
    // ---- 2. one lane per row: dL/dSH into the staged row, the direction term of dL/dmean ----
    if (valid) {
        const float mx = lerp ? LERP(means3D[3 * c], means3D[3 * p], t, u) : means3D[3 * c];
        const float my = lerp ? LERP(means3D[3 * c + 1], means3D[3 * p + 1], t, u) : means3D[3 * c + 1];
        const float mz = lerp ? LERP(means3D[3 * c + 2], means3D[3 * p + 2], t, u) : means3D[3 * c + 2];
        float col[4];                                      // accum columns 6..9: dL/dRGB (and dL/dinvdepth, unused here)
        if (peers.n > 1) gather_accum_pairs<2>(peers, rank_mask[i], i, 3, col);
        else { const float* ac = accum + (size_t)i * kAccum; col[0] = ac[6]; col[1] = ac[7]; col[2] = ac[8]; }
        const uint32_t kb = __float_as_uint(records[i].b.w);
        const float dRGB[3] = {(kb >> kClampShift) & 1u ? 0.f : col[0], (kb >> (kClampShift + 1)) & 1u ? 0.f : col[1],
                               (kb >> (kClampShift + 2)) & 1u ? 0.f : col[2]};
        const float d0x = mx - campos[0], d0y = my - campos[1], d0z = mz - campos[2];
        const float len = sqrtf(d0x * d0x + d0y * d0y + d0z * d0z);
        float B[16], Bx[16], By[16], Bz[16];
        sh_basis(deg, d0x / len, d0y / len, d0z / len, B, Bx, By, Bz);
        float ddx = 0.f, ddy = 0.f, ddz = 0.f;
#pragma unroll
        for (int q = 0; q < 12; q++) {
            if (q < nq) {
                const float4 v = s_row[w][lane][q];
                const float sv[4] = {v.x, v.y, v.z, v.w};
                float o4[4];
#pragma unroll
                for (int r = 0; r < 4; r++) {
                    const int e = 4 * q + r, k = e / 3, ch = e - 3 * k;      // compile-time after unrolling
                    const float g = dRGB[ch];
                    o4[r] = B[k] * g;
                    ddx += Bx[k] * sv[r] * g; ddy += By[k] * sv[r] * g; ddz += Bz[k] * sv[r] * g;
                }
                s_row[w][lane][q] = make_float4(o4[0], o4[1], o4[2], o4[3]);
            }
        }
        float dm0, dm1, dm2;
        dir_grad_to_mean(d0x, d0y, d0z, ddx, ddy, ddz, dm0, dm1, dm2);
        atomicAdd(dL_dmeans3D + 3 * (size_t)c + 0, t * dm0); atomicAdd(dL_dmeans3D + 3 * (size_t)c + 1, t * dm1);
        atomicAdd(dL_dmeans3D + 3 * (size_t)c + 2, t * dm2);
        if (lerp) {
            atomicAdd(dL_dmeans3D + 3 * (size_t)p + 0, u * dm0); atomicAdd(dL_dmeans3D + 3 * (size_t)p + 1, u * dm1);
            atomicAdd(dL_dmeans3D + 3 * (size_t)p + 2, u * dm2);
        }
    }
    __syncwarp();
    // ---- 3. write the rows back piece by piece: own rows stored or reduced, parent pieces once per run of siblings ----
#pragma unroll
    for (int m = 0; m < 12; m++) {
        const int it = lane + 32 * m, r = it / NQ, q = it - r * NQ;
        if (m < NQ && q < nq && s_c[w][r] >= 0) {
            const int cr = s_c[w][r];
            const float4 o = s_row[w][r][q];
            const float tt = s_t[w][r];
            const float4 own = make_float4(tt * o.x, tt * o.y, tt * o.z, tt * o.w);
            float4* dst = reinterpret_cast<float4*>(dL_dsh + (size_t)cr * SH3) + q;
            if (s_store[w][r])             // what a reduction into the zero line gives, -0 included: 0 + (-0) = +0
                *dst = make_float4(__fadd_rn(0.f, own.x), __fadd_rn(0.f, own.y), __fadd_rn(0.f, own.z), __fadd_rn(0.f, own.w));
            else atomicAdd(dst, own);      // red.global.add.v4.f32
            const int pr = s_p[w][r];
            if (pr >= 0 && (r == 0 || s_p[w][r - 1] != pr)) {
                const float uu = s_u[w][r];
                float4 acc = make_float4(uu * o.x, uu * o.y, uu * o.z, uu * o.w);
                for (int r2 = r + 1; r2 < 32 && s_p[w][r2] == pr; r2++) {
                    const float u2 = s_u[w][r2];
                    const float4 o2 = s_row[w][r2][q];
                    acc.x += u2 * o2.x; acc.y += u2 * o2.y; acc.z += u2 * o2.z; acc.w += u2 * o2.w;
                }
                atomicAdd(reinterpret_cast<float4*>(dL_dsh + (size_t)pr * SH3) + q, acc);
            }
        }
    }
#undef LERP
}

// How many rendered rows write each full-size row of dL/dSH in sh_backward_rows_kernel: +1 as its own row, +2 as a
// parent it is lerped with (u != 0; a missing parent is the own row).  `count` is zeroed; a count of 1 means one writer.
// Rows with a negative render index are skipped, as every kernel skips them.
__global__ void __launch_bounds__(256)
sh_row_count_kernel(int P, const int* __restrict__ ridx, const int* __restrict__ pidx, const float* __restrict__ ts,
                    int* __restrict__ count)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int c = ridx[i];
    if (c < 0) return;                       // the tail a device-side cut leaves when P is the capacity of its arrays
    const int p = pidx[i];
    atomicAdd(count + c, 1);
    if (1.0f - ts[i] != 0.0f) atomicAdd(count + (p < 0 ? c : p), 2);
}

int launch_sh_row_count(const h3dgs_raster_args& a, int* count, cudaStream_t s)
{
    H3_CUDA(cudaMemsetAsync(count, 0, (size_t)a.num_source * sizeof(int), s));
    if (a.P == 0) return H3DGS_OK;
    sh_row_count_kernel<<<(a.P + 255) / 256, 256, 0, s>>>(a.P, a.render_indices, a.parent_indices, a.interpolation_weights,
                                                          count);
    H3_LAUNCHED("sh_row_count", a.debug, s);
    return H3DGS_OK;
}

// Peer mode, end of backward phase 1: this rank's partial [P][10] sums are complete.  Rows another rank owns travel
// now: 40 bytes per row this rank touched (its bit in the rank mask), stored into slot [rank] of the owner's staging
// area.  One thread per row, five 8-byte stores: a warp writes 32 consecutive rows = 1280 contiguous bytes, and
// consecutive rows have the same owner (blocks of 2^shift rows), so the stores leave as full lines -- posted writes
// over NVLink, nothing waits for them until the barrier kernel that follows.
__global__ void __launch_bounds__(256)
peer_push_kernel(int P, const RowCycle cyc, const uint8_t* __restrict__ rank_mask, const float* __restrict__ accum,
                 const PeerPtrs stages)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    if (!((rank_mask[i] >> cyc.rank) & 1u)) return;                   // no tile of ours holds this Gaussian: nothing to report
    const int owner = (i >> cyc.shift) % cyc.world;
    if (owner == cyc.rank) return;                                    // our own rows stay in `accum`
    float* dst = nullptr;
#pragma unroll
    for (int r = 0; r < H3DGS_MAX_PEERS; r++) if (r == owner) dst = static_cast<float*>(stages.p[r]);    // parameter-bank indexing
    float2* d2 = reinterpret_cast<float2*>(dst + ((size_t)cyc.rank * P + i) * kAccum);
    const float2* s2 = reinterpret_cast<const float2*>(accum + (size_t)i * kAccum);
#pragma unroll
    for (int k = 0; k < kAccum / 2; k++) d2[k] = s2[k];
}

int launch_peer_push(const h3dgs_raster_args& a, const uint8_t* rank_mask, const float* accum, cudaStream_t s)
{
    if (a.P == 0 || a.peer_count <= 1) return H3DGS_OK;
    const RowCycle cyc = row_cycle(a);
    peer_push_kernel<<<(a.P + 255) / 256, 256, 0, s>>>(a.P, cyc, rank_mask, accum, peer_ptrs(a.peer_stage, a.peer_count));
    H3_LAUNCHED("peer_push", a.debug, s);
    return H3DGS_OK;
}

int launch_preprocess_backward(const h3dgs_raster_args& a, const int32_t* radii, const uint8_t* rank_mask, const Record* records,
                               const float* accum, float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh,
                               float* dL_dcolors, float* dL_dopacities, float* dL_dscales, float* dL_drots,
                               float* dL_dcov3D, cudaStream_t s)
{
    if (a.P == 0) return H3DGS_OK;
    const float fx = a.image_width / (2.0f * a.tanfovx), fy = a.image_height / (2.0f * a.tanfovy);
    const RowCycle cyc = row_cycle(a);
    const int r0 = (cyc.world > 1 || a.grad_row_end <= a.grad_row_begin) ? 0 : a.grad_row_begin;
    const int r1 = (cyc.world > 1 || a.grad_row_end <= a.grad_row_begin) ? a.P : min(a.grad_row_end, a.P);
    const int rows = cyc.world > 1 ? cyclic_local_rows(cyc, a.P) : r1 - r0;
    if (rows <= 0) return H3DGS_OK;
    ProfScope prof(H3DGS_STAGE_PREPROCESS_BWD, s);
    preprocess_backward_kernel<<<(rows + 127) / 128, 128, 0, s>>>(
        r0, r1, cyc, a.sh_degree, a.sh_coeffs, a.means3D, a.scales, a.scale_modifier, a.rotations, a.shs, a.cov3D_precomp,
        a.colors_precomp, a.interpolation_weights, a.render_indices, a.parent_indices, a.viewmatrix, a.projmatrix, a.campos, a.image_width, a.image_height, a.tanfovx, a.tanfovy,
        fx, fy, a.do_depth, radii, rank_mask, stage_ptrs(a, accum), records, accum, dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacities,
        dL_dscales, dL_drots, dL_dcov3D);
    H3_LAUNCHED("preprocess_backward", a.debug, s);
    return H3DGS_OK;
}

int launch_sh_backward(const h3dgs_raster_args& a, const int32_t* radii, const uint8_t* rank_mask, const Record* records,
                       const float* accum, const int* row_count, float* dL_dmeans3D, float* dL_dsh, cudaStream_t s)
{
    if (a.P == 0 || a.colors_precomp) return H3DGS_OK;
    const RowCycle cyc = row_cycle(a);
    const int r0 = (cyc.world > 1 || a.grad_row_end <= a.grad_row_begin) ? 0 : a.grad_row_begin;
    const int r1 = (cyc.world > 1 || a.grad_row_end <= a.grad_row_begin) ? a.P : min(a.grad_row_end, a.P);
    const int rows = cyc.world > 1 ? cyclic_local_rows(cyc, a.P) : r1 - r0;
    if (rows <= 0) return H3DGS_OK;
    ProfScope prof(H3DGS_STAGE_SH_BACKWARD, s);
    if (a.render_indices && ((a.sh_coeffs * 3) & 3) == 0)
        sh_backward_rows_kernel<<<(rows + 127) / 128, 128, 0, s>>>(r0, r1, cyc, a.sh_degree, a.sh_coeffs, a.means3D, a.shs,
                                                                  a.interpolation_weights, a.render_indices, a.parent_indices,
                                                                  a.campos, radii, rank_mask, stage_ptrs(a, accum), records,
                                                                  accum, row_count, dL_dmeans3D, dL_dsh);
    else sh_backward_kernel<<<(rows + 127) / 128, 128, 0, s>>>(r0, r1, cyc, a.sh_degree, a.sh_coeffs, a.means3D, a.shs,
                                                         a.interpolation_weights, a.render_indices, a.parent_indices,
                                                         a.campos, radii, rank_mask, stage_ptrs(a, accum), records, accum,
                                                         dL_dmeans3D, dL_dsh);
    H3_LAUNCHED("sh_backward", a.debug, s);
    return H3DGS_OK;
}

}  // namespace h3dgs
