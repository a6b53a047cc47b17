// preprocess.cu -- K1: per-Gaussian projection (replaces FORWARD::preprocess of the
// absent hierarchy-rasterizer; semantics per oracle/oracle.c::oracle_preprocess).
//
// COMPILED WITH -fmad=false: every value that feeds an integer artefact (depth key
// bits, pixel centre -> tile rect, radius) is evaluated as individually rounded
// fp32 mul/add in a fixed order, so radii / rects / keys / sort order are
// bit-identical to the CPU oracle (gcc -ffp-contract=off).  The kernel is a pure
// HBM stream (44 B in + 192 B SH for visible Gaussians, 56 B out), so the lost FMA
// contraction costs nothing.
#include "common.cuh"

namespace h3dgs {

__device__ __constant__ float kSH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                           -1.0925484305920792f, 0.5462742152960396f};
__device__ __constant__ float kSH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                           0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                           -0.5900435899266435f};
constexpr float kSH_C0 = 0.28209479177387814f;
constexpr float kSH_C1 = 0.4886025119029199f;

// Load the first n3 floats (multiple of 3) of one Gaussian's [K][3] SH block.
// 128-bit loads when the row stride keeps 16-B alignment (K = 4, 16).
template <int MAXF>
__device__ __forceinline__ void load_sh(const float* __restrict__ p, int row_floats, int need_floats, float* c) {
    if ((row_floats & 3) == 0) {
        const float4* p4 = reinterpret_cast<const float4*>(p);
#pragma unroll
        for (int i = 0; i < MAXF / 4; i++) {
            if (i * 4 < need_floats) {
                float4 v = __ldg(p4 + i);
                c[4 * i] = v.x; c[4 * i + 1] = v.y; c[4 * i + 2] = v.z; c[4 * i + 3] = v.w;
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < MAXF; i++)
            if (i < need_floats) c[i] = __ldg(p + i);
    }
}

__global__ void __launch_bounds__(256)
preprocess_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ scales,
                  float scale_mod, const float* __restrict__ rots, const float* __restrict__ opacities,
                  const float* __restrict__ cov3D_precomp,
                  const float* __restrict__ colors_precomp, const float* __restrict__ ts,
                  const int* __restrict__ kids, const int* __restrict__ ridx, const int* __restrict__ pidx,
                  const float* __restrict__ view, const float* __restrict__ proj,
                  int W, int H, float tanx, float tany, float fx, float fy,
                  int shard_count, int shard_index, int prefiltered, ScanInfo* __restrict__ info,
                  int* __restrict__ radii, float* __restrict__ depths, uint32_t* __restrict__ tiles_touched,
                  uint8_t* __restrict__ rank_mask /* peer mode, else NULL */, Record* __restrict__ records,
                  uint32_t* __restrict__ tile_count)
{
    __shared__ float s_view[16], s_proj[16];
    if (threadIdx.x < 16) { s_view[threadIdx.x] = view[threadIdx.x]; s_proj[threadIdx.x] = proj[threadIdx.x]; }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;

    int out_radius = 0; uint32_t out_tiles = 0, out_mask = 0;
    // in-kernel cut gather + parent lerp: x = t*x[c] + (1-t)*x[p], evaluated as two rounded
    // products and one rounded sum (bit-identical to the PyTorch expression of render_post)
    int c = i, p = i;
    float t = 1.0f, u = 0.0f;
    if (ridx) {
        c = ridx[i];
        if (c < 0) { radii[i] = 0; tiles_touched[i] = 0; if (rank_mask) rank_mask[i] = 0; return; }   // tail after a device-side LOD cut (h3dgs_lod_cut)
        p = pidx[i]; if (p < 0) p = c;
        t = ts[i]; u = 1.0f - t;
    }
    const bool lerp = ridx != nullptr && u != 0.0f;
#define LERP(a, b) (lerp ? (t * (a) + u * (b)) : (a))
    const float px_ = LERP(means3D[3 * c], means3D[3 * p]);
    const float py_ = LERP(means3D[3 * c + 1], means3D[3 * p + 1]);
    const float pz_ = LERP(means3D[3 * c + 2], means3D[3 * p + 2]);
    const float* m = s_view;
    // Keep in step with cov_grad.cuh::cov_chain_backward (H3_VIEW): the backward re-evaluates this view transform with
    // the same rounded operations in the same order, so that it takes the same frustum-clamp decision as here.
    const float vx = m[0] * px_ + m[4] * py_ + m[8] * pz_ + m[12];
    const float vy = m[1] * px_ + m[5] * py_ + m[9] * pz_ + m[13];
    const float vz = m[2] * px_ + m[6] * py_ + m[10] * pz_ + m[14];
    if (vz > kNearPlane) {
        const float* q = s_proj;
        const float hx = q[0] * px_ + q[4] * py_ + q[8] * pz_ + q[12];
        const float hy = q[1] * px_ + q[5] * py_ + q[9] * pz_ + q[13];
        const float hw = q[3] * px_ + q[7] * py_ + q[11] * pz_ + q[15];
        const float pw = 1.0f / (hw + kWEps);
        const float ndcx = hx * pw, ndcy = hy * pw;

        float cov6[6];
        if (cov3D_precomp) {
#pragma unroll
            for (int k = 0; k < 6; k++) cov6[k] = cov3D_precomp[6 * c + k];
        } else {
            float4 qq = *reinterpret_cast<const float4*>(rots + 4 * c);
            if (lerp) {
                float4 qp = *reinterpret_cast<const float4*>(rots + 4 * p);
                const float dot = qq.x * qp.x + qq.y * qp.y + qq.z * qp.z + qq.w * qp.w;
                if (dot < 0.f) { qp.x = -qp.x; qp.y = -qp.y; qp.z = -qp.z; qp.w = -qp.w; }
                qq.x = t * qq.x + u * qp.x; qq.y = t * qq.y + u * qp.y;
                qq.z = t * qq.z + u * qp.z; qq.w = t * qq.w + u * qp.w;
            }
            const float r = qq.x, x = qq.y, y = qq.z, z = qq.w;
            float R[3][3];
            R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z); R[0][2] = 2.f * (x * z + r * y);
            R[1][0] = 2.f * (x * y + r * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
            R[2][0] = 2.f * (x * z - r * y); R[2][1] = 2.f * (y * z + r * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
            float Mm[3][3];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const float s = scale_mod * LERP(scales[3 * c + k], scales[3 * p + k]);
#pragma unroll
                for (int j = 0; j < 3; j++) Mm[k][j] = s * R[j][k];
            }
            int o = 0;
#pragma unroll
            for (int a = 0; a < 3; a++)
#pragma unroll
                for (int b = a; b < 3; b++)
                    cov6[o++] = Mm[0][a] * Mm[0][b] + Mm[1][a] * Mm[1][b] + Mm[2][a] * Mm[2][b];
        }

        // EWA: cov2D = (J Rwv) Sigma (J Rwv)^T + 0.3 I
        const float limx = kFovClamp * tanx, limy = kFovClamp * tany;
        const float txtz = vx / vz, tytz = vy / vz;
        const float tx = fminf(limx, fmaxf(-limx, txtz)) * vz;
        const float ty = fminf(limy, fmaxf(-limy, tytz)) * vz;
        const float J00 = fx / vz, J02 = -(fx * tx) / (vz * vz);
        const float J11 = fy / vz, J12 = -(fy * ty) / (vz * vz);
        float A[2][3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            A[0][c] = J00 * m[4 * c + 0] + J02 * m[4 * c + 2];
            A[1][c] = J11 * m[4 * c + 1] + J12 * m[4 * c + 2];
        }
        const float V[3][3] = {{cov6[0], cov6[1], cov6[2]}, {cov6[1], cov6[3], cov6[4]}, {cov6[2], cov6[4], cov6[5]}};
        float AV[2][3];
#pragma unroll
        for (int r2 = 0; r2 < 2; r2++)
#pragma unroll
            for (int c = 0; c < 3; c++)
                AV[r2][c] = A[r2][0] * V[0][c] + A[r2][1] * V[1][c] + A[r2][2] * V[2][c];
        const float ca = (AV[0][0] * A[0][0] + AV[0][1] * A[0][1] + AV[0][2] * A[0][2]) + kDilation;
        const float cb = AV[0][0] * A[1][0] + AV[0][1] * A[1][1] + AV[0][2] * A[1][2];
        const float cc = (AV[1][0] * A[1][0] + AV[1][1] * A[1][1] + AV[1][2] * A[1][2]) + kDilation;
        const float det = ca * cc - cb * cb;
        if (det != 0.0f) {
            const float det_inv = 1.f / det;
            const float conx = cc * det_inv, cony = -cb * det_inv, conz = ca * det_inv;
            const float mid = 0.5f * (ca + cc);
            const float sq = sqrtf(fmaxf(kLambdaFloor, mid * mid - det));
            const float l1 = mid + sq, l2 = mid - sq;
            const float my_radius = ceilf(3.f * sqrtf(fmaxf(l1, l2)));
            const float ix = ((ndcx + 1.0f) * W - 1.0f) * 0.5f;
            const float iy = ((ndcy + 1.0f) * H - 1.0f) * 0.5f;
            const int rad = f2i_sat(my_radius);
            const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
            const TileRect rect = tile_rect(ix, iy, rad, gx, gy);
            const int rminx = rect.x, rminy = rect.y, rmaxx = rect.z, rmaxy = rect.w;
            // A row that does not project to finite values (a NaN or overflowing parameter) or whose radius is not
            // positive is invisible, like an empty rect: the binning kernels skip radii <= 0, so a row that counted
            // tiles here with such a radius would leave histogram slots that nobody fills.
            const bool projects = rad > 0 && is_finite(my_radius) && is_finite(vz) && is_finite(ix) && is_finite(iy)
                               && is_finite(conx) && is_finite(cony) && is_finite(conz);
            const int area = projects ? (rmaxx - rminx) * (rmaxy - rminy) : 0;
            if (area != 0) {
                // colour: precomputed colours are copied here; SH colours are filled in by
                // preprocess_color_kernel (separate launch: keeps this kernel at high occupancy)
                float rgb[3] = {0.f, 0.f, 0.f};
                const uint32_t clampbits = 0;
                if (colors_precomp) {
                    rgb[0] = colors_precomp[3 * c]; rgb[1] = colors_precomp[3 * c + 1]; rgb[2] = colors_precomp[3 * c + 2];
                }
                Record rec;
                rec.a = make_float4(ix, iy, conx, cony);
                const float tt = ts ? ts[i] : 1.0f;
                // k <= 1 (negative included) is the identity; larger counts saturate instead of wrapping in the 20-bit field
                const int32_t kin = kids ? kids[i] : 1;
                const uint32_t k = kin <= 1 ? 1u : min((uint32_t)kin, kKidsMask);
                rec.b = make_float4(conz, LERP(opacities[c], opacities[p]), tt, __uint_as_float(k | clampbits));
                rec.c = make_float4(rgb[0], rgb[1], rgb[2], 1.0f / vz);
                records[i] = rec;
                depths[i] = vz;
                out_radius = rad;
                // tile rows owned by this shard: y % shard_count == shard_index
                const int rows = (rmaxy + shard_count - 1 - shard_index) / shard_count
                               - (rminy + shard_count - 1 - shard_index) / shard_count;
                out_tiles = (uint32_t)(rows * (rmaxx - rminx));
                // peer mode: which ranks' tile rows the rect covers, i.e. whose accumulators will hold sums for this row
                if (rank_mask) {
                    if (rmaxy - rminy >= shard_count) out_mask = (1u << shard_count) - 1u;
                    else for (int y = rminy; y < rmaxy; y++) out_mask |= 1u << (y % shard_count);
                }
                // per-tile histogram for the per-tile sort (binning.cu): replaces the scan over P
                for (int y = rminy; y < rmaxy; y++) {
                    if (shard_count > 1 && (y % shard_count) != shard_index) continue;
                    for (int x = rminx; x < rmaxx; x++) atomicAdd(tile_count + (y * gx + x), 1u);
                }
            }
        }
    }
    else if (prefiltered) info->prefilter_bad = 1u;    // the caller promised that nothing is behind the near plane
#undef LERP
    radii[i] = out_radius;
    tiles_touched[i] = out_tiles;
    if (rank_mask) rank_mask[i] = (uint8_t)out_mask;
}

// K1b: SH -> RGB for the visible Gaussians only (192 B/row, x2 on lerped rows): reads the same
// (lerped) mean as K1a, writes record.c.xyz and the three SH clamp flags.  One thread per Gaussian: a four-threads-per-
// Gaussian form needs fewer registers and keeps more warps resident, but issues several times the instructions for the
// same DRAM traffic.
__global__ void __launch_bounds__(256)
preprocess_color_kernel(int P, int deg, int M, const float* __restrict__ means3D, const float* __restrict__ shs,
                        const float* __restrict__ ts, const int* __restrict__ ridx, const int* __restrict__ pidx,
                        const float* __restrict__ campos, const int* __restrict__ radii,
                        const uint32_t* __restrict__ own_tiles, int row_begin, int row_end, const RowCycle cyc,
                        Record* __restrict__ records)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    if (radii[i] <= 0) return;
    // tile-sharded frame: the colour (and its clamp flags) of a Gaussian is read by the ranks whose tile rows
    // it touches (forward gather) and by the rank that owns its gradient row (SH backward); nobody else needs it
    if (own_tiles && own_tiles[i] == 0u && (cyc.world > 1 ? !cyclic_owned(cyc, i) : (i < row_begin || i >= row_end))) return;
    int c = i, p = i;
    float t = 1.0f, u = 0.0f;
    if (ridx) {
        c = ridx[i]; p = pidx[i]; if (p < 0) p = c;
        t = ts[i]; u = 1.0f - t;
    }
    const bool lerp = ridx != nullptr && u != 0.0f;
#define LERP(a, b) (lerp ? (t * (a) + u * (b)) : (a))
    const int need = 3 * (deg + 1) * (deg + 1);
    float c_[48];
    {
        const float* pc = shs + (size_t)c * M * 3;
        const float* pp = shs + (size_t)p * M * 3;
        if (((M * 3) & 3) == 0) {
#pragma unroll
            for (int k = 0; k < 12; k++)
                if (4 * k < need) {
                    float4 v = __ldg(reinterpret_cast<const float4*>(pc) + k);
                    if (lerp) {
                        const float4 w = __ldg(reinterpret_cast<const float4*>(pp) + k);
                        v.x = t * v.x + u * w.x; v.y = t * v.y + u * w.y; v.z = t * v.z + u * w.z; v.w = t * v.w + u * w.w;
                    }
                    c_[4 * k] = v.x; c_[4 * k + 1] = v.y; c_[4 * k + 2] = v.z; c_[4 * k + 3] = v.w;
                }
        } else {
#pragma unroll
            for (int k = 0; k < 48; k++)
                if (k < need) c_[k] = lerp ? t * __ldg(pc + k) + u * __ldg(pp + k) : __ldg(pc + k);
        }
    }
    const float px_ = LERP(means3D[3 * c], means3D[3 * p]);
    const float py_ = LERP(means3D[3 * c + 1], means3D[3 * p + 1]);
    const float pz_ = LERP(means3D[3 * c + 2], means3D[3 * p + 2]);
#undef LERP
    float dx = px_ - campos[0], dy = py_ - campos[1], dz = pz_ - campos[2];
    const float len = sqrtf(dx * dx + dy * dy + dz * dz);
    dx /= len; dy /= len; dz /= len;
    const float x = dx, y = dy, z = dz;
    float rgb[3];
    uint32_t clampbits = 0;
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
#define S(k) c_[(k) * 3 + ch]
        float r = kSH_C0 * S(0);
        if (deg > 0) {
            r = r - kSH_C1 * y * S(1) + kSH_C1 * z * S(2) - kSH_C1 * x * S(3);
            if (deg > 1) {
                const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                r = r + kSH_C2[0] * xy * S(4) + kSH_C2[1] * yz * S(5) + kSH_C2[2] * (2.0f * zz - xx - yy) * S(6)
                      + kSH_C2[3] * xz * S(7) + kSH_C2[4] * (xx - yy) * S(8);
                if (deg > 2) {
                    r = r + kSH_C3[0] * y * (3.0f * xx - yy) * S(9) + kSH_C3[1] * xy * z * S(10)
                          + kSH_C3[2] * y * (4.0f * zz - xx - yy) * S(11)
                          + kSH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * S(12)
                          + kSH_C3[4] * x * (4.0f * zz - xx - yy) * S(13)
                          + kSH_C3[5] * z * (xx - yy) * S(14) + kSH_C3[6] * x * (xx - 3.0f * yy) * S(15);
                }
            }
        }
#undef S
        r += 0.5f;
        if (r < 0.f) clampbits |= (1u << (kClampShift + ch));
        rgb[ch] = fmaxf(r, 0.f);
    }
    float* rc = reinterpret_cast<float*>(&records[i].c);
    rc[0] = rgb[0]; rc[1] = rgb[1]; rc[2] = rgb[2];
    if (clampbits) {
        uint32_t* kb = reinterpret_cast<uint32_t*>(&records[i].b) + 3;
        *kb = *kb | clampbits;
    }
}

int launch_preprocess(const h3dgs_raster_args& a, int32_t* radii, float* depths, uint32_t* tiles_touched,
                      uint8_t* rank_mask, Record* records, uint32_t* tile_count, ScanInfo* info, cudaStream_t s)
{
    if (a.P == 0) return H3DGS_OK;
    const float fx = a.image_width / (2.0f * a.tanfovx), fy = a.image_height / (2.0f * a.tanfovy);
    const int threads = 256, blocks = (a.P + threads - 1) / threads;
    ProfScope prof(H3DGS_STAGE_PREPROCESS, s);
    preprocess_kernel<<<blocks, threads, 0, s>>>(a.P, a.means3D, a.scales, a.scale_modifier, a.rotations, a.opacities,
                                                 a.cov3D_precomp, a.colors_precomp, a.interpolation_weights,
                                                 a.num_node_kids, a.render_indices, a.parent_indices, a.viewmatrix,
                                                 a.projmatrix, a.image_width, a.image_height, a.tanfovx, a.tanfovy, fx, fy,
                                                 a.shard_count > 0 ? a.shard_count : 1, a.shard_count > 0 ? a.shard_index : 0,
                                                 a.prefiltered, info, radii, depths, tiles_touched, a.peer_count > 1 ? rank_mask : nullptr, records, tile_count);
    H3_LAUNCHED("preprocess", a.debug, s);
    return H3DGS_OK;
}

int launch_preprocess_color(const h3dgs_raster_args& a, const int32_t* radii, const uint32_t* tiles_touched,
                            Record* records, cudaStream_t s)
{
    if (a.P == 0 || a.colors_precomp) return H3DGS_OK;
    const int threads = 256, blocks = (a.P + threads - 1) / threads;
    // only when the caller told the forward which gradient rows this rank will finish (otherwise every visible row may be needed)
    const RowCycle cyc = row_cycle(a);
    const bool skip_foreign = a.shard_count > 1 && (a.grad_row_end > a.grad_row_begin || cyc.world > 1);
    ProfScope prof(H3DGS_STAGE_PREPROCESS_COLOR, s);
    preprocess_color_kernel<<<blocks, threads, 0, s>>>(a.P, a.sh_degree, a.sh_coeffs, a.means3D, a.shs,
                                                       a.interpolation_weights, a.render_indices, a.parent_indices,
                                                       a.campos, radii, skip_foreign ? tiles_touched : nullptr,
                                                       a.grad_row_begin, a.grad_row_end, cyc, records);
    H3_LAUNCHED("preprocess_color", a.debug, s);
    return H3DGS_OK;
}
__global__ void mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ view,
                                    uint8_t* __restrict__ present)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float x = means3D[3 * i], y = means3D[3 * i + 1], z = means3D[3 * i + 2];
    const float vz = view[2] * x + view[6] * y + view[10] * z + view[14];
    present[i] = vz > kNearPlane;
}

}  // namespace h3dgs

extern "C" int h3dgs_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                                  uint8_t* present, void* stream)
{
    (void)projmatrix;
    if (P <= 0) return H3DGS_OK;
    cudaStream_t s = (cudaStream_t)stream;
    h3dgs::mark_visible_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, means3D, viewmatrix, present);
    H3_LAUNCHED("mark_visible", 0, s);
    return H3DGS_OK;
}
