// lod_cull.cu -- the view cull of the LOD cut: a per-row mask of the hierarchy rows that can reach the image.
//
// The cut (hierarchy.cu) pairs every row of a node with one partner row -- the parent node's start row, or the row itself
// for a root -- and K1 (preprocess.cu) draws x(t) = t x_row + (1 - t) x_partner for the cut's t in [0, 1].  A row is KEPT
// (mask 1) unless no t in [0, 1] can give it a positive radius and a non-empty tile rect in K1.  The test does not depend
// on t, so one mask serves the cut at every threshold and the budget's search over all of them.  The bound and its
// margins are derived in DESIGN.md §3.9; in short, for the segment between the two endpoints:
//   depth       drop when both endpoints' view z + dz <= the near plane, dz = 2^-16 S_z (S_z: the view-z row applied to
//               the endpoints' largest |coordinates|, bounds K1's lerp and dot-product rounding, ~13 ulp of S_z);
//   clipping    otherwise clip the segment at near - dz; z_lo = max(near, smallest clipped z - dz) bounds K1's vz;
//   covariance  lambda_max(Sigma) <= (|s|max scale_modifier)^2 ||R(q)||^2, ||R(q)||_2 <= max(1, 2|q|^2 - 1), |q| <= the
//               endpoints' largest norm;
//   projection  ||J||_F^2 <= (fx^2 (1 + lim_x^2) + fy^2 (1 + lim_y^2)) / z_lo^2, ||J W||_2 <= ||J||_F ||W||_F;
//   radius      lambda_1 <= ||J W||^2 lambda_max(Sigma) + 0.3 + sqrt(0.1), radius <= 3 sqrt(lambda_1) + 1;
//   screen      K1's pixel centre over the clipped segment lies between its values at the clipped endpoints (the
//               homogeneous w is affine and positive there, so x / w is monotone); grow that box by the radius and the
//               rounding pads; drop when it misses the tile grid.
// Rows whose endpoints, scales or rotations are not finite are kept (K1 decides them).  Everything is evaluated in
// float64 from the float32 inputs, operation by operation (this file is compiled with -fmad=false), so that
// tests/lod_cull_ref.py restates it bit for bit.  One thread per node: its rows and the partner row (an L2 hit in
// BFS order) in, one byte per row out.
#include "common.cuh"

namespace h3dgs {

constexpr double kCullRel = 1.0 / 65536.0;          // 2^-16: K1's float32 rounding is below ~2^-20 of each scale
constexpr double kCullCov = 1.0 / 4096.0;           // 2^-12: relative slack on the covariance and radius chain
constexpr double kCullEig = 1.0 / 512.0;            // 2^-9: the cancellation of mid^2 - det in K1's eigenvalue
constexpr double kCullCam = 1.0 / 1048576.0;        // 2^-20: fx, fy and the frustum clamp rounded in float32
constexpr double kCullFloorRoot = 0.3163;           // >= sqrt(0.1f) rounded up: the lambda floor's contribution

struct CullCam {
    double m[16], q[16];
    double near_, fx, fy, limx, limy, wf2, smod, W, H, ex, ey, eps;
};

__device__ __forceinline__ bool finite3(const float* p) { return is_finite(p[0]) && is_finite(p[1]) && is_finite(p[2]); }
__device__ __forceinline__ double row_dot(const double* m, int r, double x, double y, double z) {
    return ((m[r] * x + m[r + 4] * y) + m[r + 8] * z) + m[r + 12];
}
__device__ __forceinline__ double row_abs(const double* m, int r, double x, double y, double z) {
    return ((fabs(m[r]) * x + fabs(m[r + 4]) * y) + fabs(m[r + 8]) * z) + fabs(m[r + 12]);
}
__device__ __forceinline__ double qnorm2(const float* q) {
    const double a = q[0], b = q[1], c = q[2], d = q[3];
    return ((a * a + b * b) + c * c) + d * d;
}

// 1: K1 could draw the row (mean a, scales sa, rotation qa) lerped with its partner (b, sb, qb) for some t in [0, 1]
__device__ bool cull_keep(const float* a, const float* sa, const float* qa, const float* b, const float* sb,
                          const float* qb, const CullCam& c)
{
    if (!(finite3(a) && finite3(b) && finite3(sa) && finite3(sb) && finite3(qa) && finite3(qb) && is_finite(qa[3]) &&
          is_finite(qb[3])))
        return true;
    const double ax = a[0], ay = a[1], az = a[2], bx = b[0], by = b[1], bz = b[2];
    const double Ax = fmax(fabs(ax), fabs(bx)), Ay = fmax(fabs(ay), fabs(by)), Az = fmax(fabs(az), fabs(bz));
    // ---- depth ----
    const double za = row_dot(c.m, 2, ax, ay, az), zb = row_dot(c.m, 2, bx, by, bz);
    const double dz = kCullRel * row_abs(c.m, 2, Ax, Ay, Az);
    if (fmax(za, zb) + dz <= c.near_) return false;
    // ---- clip at near - dz (one endpoint at most is behind it) ----
    const double zc = c.near_ - dz;
    double e0x = ax, e0y = ay, e0z = az, e1x = bx, e1y = by, e1z = bz, z0 = za, z1 = zb;
    if (za < zc) {
        const double t = (zc - zb) / (za - zb);
        e0x = bx + t * (ax - bx); e0y = by + t * (ay - by); e0z = bz + t * (az - bz); z0 = zc;
    } else if (zb < zc) {
        const double t = (zc - za) / (zb - za);
        e1x = ax + t * (bx - ax); e1y = ay + t * (by - ay); e1z = az + t * (bz - az); z1 = zc;
    }
    const double z_lo = fmax(c.near_, fmin(z0, z1) - dz);
    // ---- pixel centres of the clipped endpoints ----
    const double Sx = row_abs(c.q, 0, Ax, Ay, Az), Sy = row_abs(c.q, 1, Ax, Ay, Az), Sw = row_abs(c.q, 3, Ax, Ay, Az);
    const double d0 = row_dot(c.q, 3, e0x, e0y, e0z) + c.eps, d1 = row_dot(c.q, 3, e1x, e1y, e1z) + c.eps;
    const double d_lo = fmin(d0, d1) - kCullRel * Sw;
    if (!(d_lo > 0.0)) return true;                                  // w not bounded away from 0: no bound, keep
    const double nx0 = row_dot(c.q, 0, e0x, e0y, e0z) / d0, nx1 = row_dot(c.q, 0, e1x, e1y, e1z) / d1;
    const double ny0 = row_dot(c.q, 1, e0x, e0y, e0z) / d0, ny1 = row_dot(c.q, 1, e1x, e1y, e1z) / d1;
    const double nxm = fmax(fabs(nx0), fabs(nx1)), nym = fmax(fabs(ny0), fabs(ny1));
    const double px = kCullRel * (((Sx + nxm * Sw) / d_lo + nxm) + 1.0);
    const double py = kCullRel * (((Sy + nym * Sw) / d_lo + nym) + 1.0);
    const double ix_lo = ((fmin(nx0, nx1) - px + 1.0) * c.W - 1.0) * 0.5, ix_hi = ((fmax(nx0, nx1) + px + 1.0) * c.W - 1.0) * 0.5;
    const double iy_lo = ((fmin(ny0, ny1) - py + 1.0) * c.H - 1.0) * 0.5, iy_hi = ((fmax(ny0, ny1) + py + 1.0) * c.H - 1.0) * 0.5;
    // ---- radius ----
    double smax = fmax(fmax(fabs((double)sa[0]), fabs((double)sa[1])), fabs((double)sa[2]));
    smax = fmax(smax, fmax(fmax(fabs((double)sb[0]), fabs((double)sb[1])), fabs((double)sb[2])));
    smax = c.smod * smax;
    const double Q2 = fmax(qnorm2(qa), qnorm2(qb));
    const double Rn = fmax(1.0, 2.0 * Q2 - 1.0) + kCullCov * (1.0 + Q2);
    const double lam_v = ((smax * smax) * (Rn * Rn)) * (1.0 + kCullCov);
    const double J2 = ((c.fx * c.fx) * (1.0 + c.limx * c.limx) + (c.fy * c.fy) * (1.0 + c.limy * c.limy)) / (z_lo * z_lo);
    const double lam = (J2 * c.wf2) * lam_v;
    const double L = (lam * (1.0 + kCullCov) + (double)kDilation) * (1.0 + kCullEig) + kCullFloorRoot;
    const double rad = 3.0 * sqrt(L) * (1.0 + kCullCov) + 1.0;
    // ---- the tile grid: K1's rect is empty unless ix + rad >= 1 and ix - rad < 16 gx (likewise y) ----
    const double gxp = 1.0 + kCullRel * (fmax(fabs(ix_lo), fabs(ix_hi)) + rad + c.W);
    const double gyp = 1.0 + kCullRel * (fmax(fabs(iy_lo), fabs(iy_hi)) + rad + c.H);
    if (ix_hi + rad + gxp < 1.0 || iy_hi + rad + gyp < 1.0) return false;
    if (ix_lo - rad - gxp >= c.ex || iy_lo - rad - gyp >= c.ey) return false;
    return true;
}

__global__ void __launch_bounds__(256)
lod_cull_mask_kernel(int N, const int* __restrict__ nodes, const float* __restrict__ means3D, const float* __restrict__ scales,
                     const float* __restrict__ rots, float scale_mod, const float* __restrict__ view,
                     const float* __restrict__ proj, int W, int H, float tanx, float tany, uint8_t* __restrict__ mask)
{
    __shared__ CullCam s_cam;
    if (threadIdx.x < 16) { s_cam.m[threadIdx.x] = view[threadIdx.x]; s_cam.q[threadIdx.x] = proj[threadIdx.x]; }
    if (threadIdx.x == 0) {
        CullCam& c = s_cam;
        c.near_ = (double)kNearPlane;
        c.fx = (double)W / (2.0 * (double)tanx) * (1.0 + kCullCam);
        c.fy = (double)H / (2.0 * (double)tany) * (1.0 + kCullCam);
        c.limx = (double)kFovClamp * (double)tanx * (1.0 + kCullCam);
        c.limy = (double)kFovClamp * (double)tany * (1.0 + kCullCam);
        c.smod = fabs((double)scale_mod);
        c.W = W; c.H = H;
        c.ex = (double)(kTile * ((W + kTile - 1) / kTile)); c.ey = (double)(kTile * ((H + kTile - 1) / kTile));
        c.eps = (double)kWEps;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double f = 0.0;
        for (int k = 0; k < 3; k++)
            for (int j = 0; j < 3; j++) f = f + s_cam.m[4 * k + j] * s_cam.m[4 * k + j];
        s_cam.wf2 = f;
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int* nd = nodes + 7 * (size_t)i;
    const int parent = nd[1], start = nd[2], n = nd[3] + nd[4];
    if (n <= 0) return;
    const int partner = parent == -1 ? -1 : __ldg(nodes + 7 * (size_t)parent + 2);
    float b[3], sb[3], qb[4];
    if (partner >= 0) {
        for (int k = 0; k < 3; k++) { b[k] = __ldg(means3D + 3 * (size_t)partner + k); sb[k] = __ldg(scales + 3 * (size_t)partner + k); }
        for (int k = 0; k < 4; k++) qb[k] = __ldg(rots + 4 * (size_t)partner + k);
    }
    for (int r = start; r < start + n; r++) {
        float a[3], sa[3], qa[4];
        for (int k = 0; k < 3; k++) { a[k] = __ldg(means3D + 3 * (size_t)r + k); sa[k] = __ldg(scales + 3 * (size_t)r + k); }
        for (int k = 0; k < 4; k++) qa[k] = __ldg(rots + 4 * (size_t)r + k);
        mask[r] = partner >= 0 ? (uint8_t)cull_keep(a, sa, qa, b, sb, qb, s_cam) : (uint8_t)cull_keep(a, sa, qa, a, sa, qa, s_cam);
    }
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" int h3dgs_lod_cull_mask(int32_t N, const int32_t* nodes, const float* means3D, const float* scales,
                                   const float* rotations, float scale_modifier, const float* viewmatrix,
                                   const float* projmatrix, int32_t W, int32_t H, float tanfovx, float tanfovy,
                                   uint8_t* mask, void* stream)
{
    if (N <= 0) { set_error("lod_cull_mask: empty hierarchy"); return H3DGS_EINVAL; }
    if (!nodes || !means3D || !scales || !rotations || !viewmatrix || !projmatrix || !mask) {
        set_error("lod_cull_mask: NULL argument");
        return H3DGS_EINVAL;
    }
    if (W <= 0 || H <= 0 || !(tanfovx > 0.0f) || !(tanfovy > 0.0f)) {
        set_error("lod_cull_mask: bad image size or field of view (%d x %d, tan %g %g)", W, H, tanfovx, tanfovy);
        return H3DGS_EINVAL;
    }
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope prof(H3DGS_STAGE_LOD_CULL, s);
    lod_cull_mask_kernel<<<(N + 255) / 256, 256, 0, s>>>(N, nodes, means3D, scales, rotations, scale_modifier, viewmatrix,
                                                         projmatrix, W, H, tanfovx, tanfovy, mask);
    H3_LAUNCHED("lod_cull_mask", 0, s);
    return H3DGS_OK;
}
