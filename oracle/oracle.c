/*
 * oracle.c -- CPU restatement of the hierarchical-Gaussian rasterizer hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is product code: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library.  The product path (libh3dgs.so) never calls it.
 *
 * PARITY UNPINNED.  The reference's implementation of this path lives in two
 * third-party submodules that are EMPTY in the reference checkout:
 *   diff_gaussian_rasterization  <- graphdeco-inria/hierarchy-rasterizer @ 63fa2476
 *   gaussian_hierarchy           <- graphdeco-inria/gaussian-hierarchy   @ 677c8553
 * (.gitmodules:5-13).  The reference ships no tests or golden vectors (SURVEY.md
 * section 4).  This file therefore restates the PUBLISHED algorithm (3D Gaussian
 * Splatting tile rasterizer + the SIGGRAPH'24 hierarchy extensions) and is pinned
 * only where the reference's present Python can pin it:
 *   - SH basis / sign conventions / +0.5 / clamp : utils/sh_utils.py:26-112,
 *     gaussian_renderer/__init__.py:85-89          (tests/golden/sh_*.npz)
 *   - quaternion -> R, Sigma = R S S^T R^T, 6-float packing :
 *     utils/general_utils.py:68-114                (tests/golden/cov3d_*.npz)
 *   - matrix storage (transposed, row-vector convention) : scene/cameras.py:95-98,
 *     utils/graphics_utils.py:38-77                (tests/golden/camera_*.npz)
 *   - argument meaning / shapes at the call sites : gaussian_renderer/__init__.py:44-113,
 *     247-277; train_post.py:91-113; render_hierarchy.py:55-80.
 * The constants below that are NOT derivable from present files are listed in
 * DESIGN.md ("recalled constants") and each is a named #define here.
 *
 * Forward arithmetic is fp32 with contraction disabled (-ffp-contract=off) so that the
 * integer artefacts (radii, tile rects, depth-key bits, sort order, tile ranges)
 * are reproducible bit-for-bit by the CUDA path, which evaluates the same
 * expressions without FMA contraction.  The BACKWARD evaluates the published formulas in
 * double on the fp32 inputs (decisions such as the alpha skip stay fp32): the reference uses
 * fp32 atomics in arbitrary order, so its own result is only defined up to fp32 rounding;
 * the exact-arithmetic value is the order-free target every fp32 implementation approximates.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ---- recalled constants of the published algorithm (see DESIGN.md) ---- */
#define NEAR_PLANE        0.2f        /* cull when view-space z <= 0.2            */
#define FOV_CLAMP         1.3f        /* clamp tx/tz, ty/tz to +-1.3*tanfov       */
#define DILATION          0.3f        /* low-pass: +0.3 px^2 on cov2D diagonal    */
#define LAMBDA_FLOOR      0.1f        /* max(0.1, mid^2 - det) under the sqrt     */
#define TILE              16          /* 16x16 pixel tiles                        */
#define ALPHA_CAP         0.99f
#define ALPHA_SKIP        (1.0f / 255.0f)
#define T_STOP            0.0001f
#define W_EPS             0.0000001f  /* 1/(w + 1e-7) in the projection           */

static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = { 1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                -1.0925484305920792f, 0.5462742152960396f };
static const float SH_C3[7] = { -0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                -0.5900435899266435f };

typedef struct { float x, y, z; } f3;

/* p (row vector, w=1) times the stored 4x4: view = p . M ; storage is the
 * transposed matrix of scene/cameras.py:95, flat index m[4*k + j]. */
static inline f3 xform4x3(const float* m, f3 p) {
    f3 r;
    r.x = m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12];
    r.y = m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13];
    r.z = m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14];
    return r;
}
static inline void xform4x4(const float* m, f3 p, float out[4]) {
    out[0] = m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12];
    out[1] = m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13];
    out[2] = m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14];
    out[3] = m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15];
}

/* quaternion (r,x,y,z) -> rotation rows, exactly utils/general_utils.py:89-98 */
static inline void quat_to_R(const float* q, float R[3][3]) {
    float r = q[0], x = q[1], y = q[2], z = q[3];
    R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z); R[0][2] = 2.f * (x * z + r * y);
    R[1][0] = 2.f * (x * y + r * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
    R[2][0] = 2.f * (x * z - r * y); R[2][1] = 2.f * (y * z + r * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
}

/* Sigma = R S S^T R^T, packed xx,xy,xz,yy,yz,zz (utils/general_utils.py:68-77,
 * scene/gaussian_model.py:30-34).  M[k][i] = s_k * R[i][k]; Sigma_ij = sum_k M[k][i] M[k][j]. */
static void cov3d_from_scale_rot(const float* scale, float mod, const float* rot, float* cov6) {
    float R[3][3], M[3][3];
    quat_to_R(rot, R);
    for (int k = 0; k < 3; k++) {
        float s = mod * scale[k];
        for (int i = 0; i < 3; i++) M[k][i] = s * R[i][k];
    }
    int o = 0;
    for (int i = 0; i < 3; i++)
        for (int j = i; j < 3; j++)
            cov6[o++] = M[0][i] * M[0][j] + M[1][i] * M[1][j] + M[2][i] * M[2][j];
}

/* EWA projection: cov2D = (J Rwv) Sigma (J Rwv)^T + 0.3 I ; returns a,b,c. */
static void cov2d_project(f3 mean, float fx, float fy, float tanx, float tany,
                          const float* cov6, const float* view, float out3[3]) {
    f3 t = xform4x3(view, mean);
    const float limx = FOV_CLAMP * tanx, limy = FOV_CLAMP * tany;
    const float txtz = t.x / t.z, tytz = t.y / t.z;
    t.x = fminf(limx, fmaxf(-limx, txtz)) * t.z;
    t.y = fminf(limy, fmaxf(-limy, tytz)) * t.z;
    /* J rows */
    float J00 = fx / t.z, J02 = -(fx * t.x) / (t.z * t.z);
    float J11 = fy / t.z, J12 = -(fy * t.y) / (t.z * t.z);
    /* Rwv[j][k] = view[4k + j] */
    float A[2][3];
    for (int c = 0; c < 3; c++) {
        A[0][c] = J00 * view[4 * c + 0] + J02 * view[4 * c + 2];
        A[1][c] = J11 * view[4 * c + 1] + J12 * view[4 * c + 2];
    }
    float V[3][3] = { { cov6[0], cov6[1], cov6[2] }, { cov6[1], cov6[3], cov6[4] }, { cov6[2], cov6[4], cov6[5] } };
    float AV[2][3];
    for (int r = 0; r < 2; r++)
        for (int c = 0; c < 3; c++)
            AV[r][c] = A[r][0] * V[0][c] + A[r][1] * V[1][c] + A[r][2] * V[2][c];
    out3[0] = (AV[0][0] * A[0][0] + AV[0][1] * A[0][1] + AV[0][2] * A[0][2]) + DILATION;
    out3[1] = AV[0][0] * A[1][0] + AV[0][1] * A[1][1] + AV[0][2] * A[1][2];
    out3[2] = (AV[1][0] * A[1][0] + AV[1][1] * A[1][1] + AV[1][2] * A[1][2]) + DILATION;
}

/* colour = SH(dir) + 0.5, clamped at 0 with per-channel flag.
 * utils/sh_utils.py:57-112 ; gaussian_renderer/__init__.py:85-89.
 * sh layout [M][3] (coefficient-major), scene/gaussian_model.py:121-124. */
static void sh_to_rgb(int deg, int M, f3 pos, const float* campos, const float* sh, float* rgb, uint8_t* clamped) {
    (void)M;
    f3 d = { pos.x - campos[0], pos.y - campos[1], pos.z - campos[2] };
    float len = sqrtf(d.x * d.x + d.y * d.y + d.z * d.z);
    d.x /= len; d.y /= len; d.z /= len;
    float x = d.x, y = d.y, z = d.z;
    for (int c = 0; c < 3; c++) {
#define S(k) sh[(k) * 3 + c]
        float r = SH_C0 * S(0);
        if (deg > 0) {
            r = r - SH_C1 * y * S(1) + SH_C1 * z * S(2) - SH_C1 * x * S(3);
            if (deg > 1) {
                float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                r = r + SH_C2[0] * xy * S(4) + SH_C2[1] * yz * S(5) + SH_C2[2] * (2.0f * zz - xx - yy) * S(6)
                      + SH_C2[3] * xz * S(7) + SH_C2[4] * (xx - yy) * S(8);
                if (deg > 2) {
                    r = r + SH_C3[0] * y * (3.0f * xx - yy) * S(9) + SH_C3[1] * xy * z * S(10)
                          + SH_C3[2] * y * (4.0f * zz - xx - yy) * S(11)
                          + SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * S(12)
                          + SH_C3[4] * x * (4.0f * zz - xx - yy) * S(13)
                          + SH_C3[5] * z * (xx - yy) * S(14) + SH_C3[6] * x * (xx - 3.0f * yy) * S(15);
                }
            }
        }
#undef S
        r += 0.5f;
        clamped[c] = (r < 0.f);
        rgb[c] = fmaxf(r, 0.f);
    }
}

/* float -> int toward zero, saturating, NaN -> 0: the device's conversion, which the C cast leaves undefined
 * out of range (DESIGN.md 7) */
static int f2i_sat(float x) {
    if (!(x == x)) return 0;
    if (x >= 2147483648.0f) return 2147483647;
    if (x <= -2147483648.0f) return -2147483647 - 1;
    return (int)x;
}
static int is_finite(float x) { return (x - x) == 0.0f; }

/* ------------------------------------------------------------------ */
/* K1: per-Gaussian preprocess                                         */
/* ------------------------------------------------------------------ */
void oracle_preprocess(int P, int deg, int M,
                       const float* means3D, const float* scales, float scale_mod, const float* rots,
                       const float* opacities, const float* shs, const float* cov3D_precomp,
                       const float* colors_precomp, const float* view, const float* proj, const float* campos,
                       int W, int H, float tanx, float tany,
                       /* out */ int* radii, float* xy, float* depths, float* cov3Ds, float* rgb,
                       float* conic_opacity, uint32_t* tiles_touched, uint8_t* clamped, int* rects)
{
    const float fx = W / (2.0f * tanx), fy = H / (2.0f * tany);
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) {
        radii[i] = 0; tiles_touched[i] = 0;
        xy[2 * i] = xy[2 * i + 1] = 0.f; depths[i] = 0.f;
        for (int k = 0; k < 6; k++) cov3Ds[6 * i + k] = 0.f;
        for (int k = 0; k < 3; k++) { rgb[3 * i + k] = 0.f; clamped[3 * i + k] = 0; }
        for (int k = 0; k < 4; k++) { conic_opacity[4 * i + k] = 0.f; rects[4 * i + k] = 0; }

        f3 p = { means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2] };
        f3 pv = xform4x3(view, p);
        if (pv.z <= NEAR_PLANE) continue;
        float ph[4]; xform4x4(proj, p, ph);
        float pw = 1.0f / (ph[3] + W_EPS);
        float px = ph[0] * pw, py = ph[1] * pw;

        const float* cov6;
        if (cov3D_precomp) cov6 = cov3D_precomp + 6 * i;
        else { cov3d_from_scale_rot(scales + 3 * i, scale_mod, rots + 4 * i, cov3Ds + 6 * i); cov6 = cov3Ds + 6 * i; }

        float cov[3]; cov2d_project(p, fx, fy, tanx, tany, cov6, view, cov);
        float det = cov[0] * cov[2] - cov[1] * cov[1];
        if (det == 0.0f) continue;
        float det_inv = 1.f / det;
        float conic[3] = { cov[2] * det_inv, -cov[1] * det_inv, cov[0] * det_inv };
        float mid = 0.5f * (cov[0] + cov[2]);
        float sq = sqrtf(fmaxf(LAMBDA_FLOOR, mid * mid - det));
        float l1 = mid + sq, l2 = mid - sq;
        float my_radius = ceilf(3.f * sqrtf(fmaxf(l1, l2)));
        float ix = ((px + 1.0f) * W - 1.0f) * 0.5f;
        float iy = ((py + 1.0f) * H - 1.0f) * 0.5f;
        int r = f2i_sat(my_radius);
        int rminx = f2i_sat((ix - r) / TILE), rminy = f2i_sat((iy - r) / TILE);
        int rmaxx = f2i_sat((ix + r + TILE - 1) / TILE), rmaxy = f2i_sat((iy + r + TILE - 1) / TILE);
        rminx = rminx < 0 ? 0 : (rminx > gx ? gx : rminx); rminy = rminy < 0 ? 0 : (rminy > gy ? gy : rminy);
        rmaxx = rmaxx < 0 ? 0 : (rmaxx > gx ? gx : rmaxx); rmaxy = rmaxy < 0 ? 0 : (rmaxy > gy ? gy : rmaxy);
        if ((rmaxx - rminx) * (rmaxy - rminy) == 0) continue;
        /* a row that does not project to finite values, or whose radius is not positive, is invisible */
        if (!(r > 0 && is_finite(my_radius) && is_finite(pv.z) && is_finite(ix) && is_finite(iy)
              && is_finite(conic[0]) && is_finite(conic[1]) && is_finite(conic[2]))) continue;

        if (colors_precomp) { for (int k = 0; k < 3; k++) rgb[3 * i + k] = colors_precomp[3 * i + k]; }
        else sh_to_rgb(deg, M, p, campos, shs + (size_t)i * M * 3, rgb + 3 * i, clamped + 3 * i);

        depths[i] = pv.z; radii[i] = r; xy[2 * i] = ix; xy[2 * i + 1] = iy;
        conic_opacity[4 * i] = conic[0]; conic_opacity[4 * i + 1] = conic[1]; conic_opacity[4 * i + 2] = conic[2];
        conic_opacity[4 * i + 3] = opacities[i];
        tiles_touched[i] = (uint32_t)((rmaxx - rminx) * (rmaxy - rminy));
        rects[4 * i] = rminx; rects[4 * i + 1] = rminy; rects[4 * i + 2] = rmaxx; rects[4 * i + 3] = rmaxy;
    }
}

/* ------------------------------------------------------------------ */
/* K2-K5: duplicate with keys, stable sort by (tile, depth bits), tile ranges */
/* ------------------------------------------------------------------ */
static void radix_sort_pairs(uint64_t* keys, uint32_t* vals, uint64_t* tk, uint32_t* tv, size_t n, int bits) {
    /* stable LSD radix, 16-bit digits: same order as any stable sort on the low `bits` bits */
    for (int shift = 0; shift < bits; shift += 16) {
        size_t* cnt = (size_t*)calloc(65537, sizeof(size_t));
        for (size_t i = 0; i < n; i++) cnt[((keys[i] >> shift) & 0xFFFF) + 1]++;
        for (int d = 0; d < 65536; d++) cnt[d + 1] += cnt[d];
        for (size_t i = 0; i < n; i++) { size_t p = cnt[(keys[i] >> shift) & 0xFFFF]++; tk[p] = keys[i]; tv[p] = vals[i]; }
        memcpy(keys, tk, n * sizeof(uint64_t)); memcpy(vals, tv, n * sizeof(uint32_t));
        free(cnt);
    }
}

/* returns D (= num_rendered). keys/vals must hold sum(tiles_touched) entries;
 * call once with keys==NULL to get the count. ranges is uint32 [T][2]. */
long oracle_bin(int P, int W, int H, const float* depths, const int* radii, const int* rects,
                uint64_t* keys, uint32_t* vals, uint32_t* ranges)
{
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    size_t D = 0;
    for (int i = 0; i < P; i++)
        if (radii[i] > 0) D += (size_t)(rects[4 * i + 2] - rects[4 * i]) * (rects[4 * i + 3] - rects[4 * i + 1]);
    if (!keys) return (long)D;
    size_t off = 0;
    for (int i = 0; i < P; i++) {
        if (radii[i] <= 0) continue;
        uint32_t dbits; memcpy(&dbits, &depths[i], 4);
        for (int y = rects[4 * i + 1]; y < rects[4 * i + 3]; y++)
            for (int x = rects[4 * i]; x < rects[4 * i + 2]; x++) {
                uint64_t key = (uint64_t)(y * gx + x);
                key = (key << 32) | dbits;
                keys[off] = key; vals[off] = (uint32_t)i; off++;
            }
    }
    uint64_t* tk = (uint64_t*)malloc(D * sizeof(uint64_t) + 8);
    uint32_t* tv = (uint32_t*)malloc(D * sizeof(uint32_t) + 8);
    radix_sort_pairs(keys, vals, tk, tv, D, 64);
    free(tk); free(tv);
    memset(ranges, 0, (size_t)gx * gy * 2 * sizeof(uint32_t));
    for (size_t i = 0; i < D; i++) {
        uint32_t tile = (uint32_t)(keys[i] >> 32);
        if (i == 0) ranges[2 * tile] = 0;
        else {
            uint32_t prev = (uint32_t)(keys[i - 1] >> 32);
            if (prev != tile) { ranges[2 * prev + 1] = (uint32_t)i; ranges[2 * tile] = (uint32_t)i; }
        }
        if (i == D - 1) ranges[2 * tile + 1] = (uint32_t)D;
    }
    return (long)D;
}

/* Hierarchy transition weight on the per-pixel blending weight (UNPINNED; see
 * DESIGN.md "hierarchy alpha").  k siblings interpolate toward one parent; at
 * t=0 the k coincident copies must composite to the parent's alpha:
 *   a' = t*a + (1-t) * (1 - (1-a)^(1/k)).  t=1 or k=1 is the identity (the skybox
 * rows of gaussian_renderer/__init__.py:232-234 rely on that). */
static inline float hier_alpha(float a, float t, int k) {
    if (k <= 1 || t >= 1.0f) return a;
    /* 1 - (1-a)^(1/k) evaluated as -expm1(log1p(-a)/k): the direct form cancels for the small a
     * that sit at the 1/255 skip threshold and would make the skip decision itself noisy */
    return t * a + (1.0f - t) * (-expm1f(log1pf(-a) / (float)k));
}
static inline float hier_dalpha(float a, float t, int k) {
    if (k <= 1 || t >= 1.0f) return 1.0f;
    float ik = 1.0f / (float)k;
    return t + (1.0f - t) * ik * powf(1.0f - a, ik - 1.0f);
}

/* ------------------------------------------------------------------ */
/* K6: per-tile front-to-back blend                                    */
/* ------------------------------------------------------------------ */
void oracle_render_forward(int W, int H, const uint32_t* ranges, const uint32_t* point_list,
                           const float* xy, const float* rgb, const float* conic_opacity, const float* depths,
                           const float* ts, const int* kids, const float* bg, int do_depth,
                           /* out */ float* out_color, float* final_T, uint32_t* n_contrib, float* out_invdepth)
{
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
#pragma omp parallel for schedule(dynamic, 4)
    for (int tile = 0; tile < gx * gy; tile++) {
        int tx = tile % gx, ty = tile / gx;
        uint32_t s = ranges[2 * tile], e = ranges[2 * tile + 1];
        for (int py = ty * TILE; py < (ty + 1) * TILE && py < H; py++)
            for (int px = tx * TILE; px < (tx + 1) * TILE && px < W; px++) {
                float T = 1.0f, C[3] = { 0, 0, 0 }, invd = 0.f;
                uint32_t contributor = 0, last = 0;
                for (uint32_t j = s; j < e; j++) {
                    contributor++;
                    uint32_t g = point_list[j];
                    float dx = xy[2 * g] - (float)px, dy = xy[2 * g + 1] - (float)py;
                    const float* co = conic_opacity + 4 * g;
                    float power = -0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                    if (power > 0.0f) continue;
                    float alpha = fminf(ALPHA_CAP, co[3] * expf(power));
                    if (ts) alpha = hier_alpha(alpha, ts[g], kids[g]);
                    if (alpha < ALPHA_SKIP) continue;
                    float test_T = T * (1 - alpha);
                    if (test_T < T_STOP) break;
                    for (int c = 0; c < 3; c++) C[c] += rgb[3 * g + c] * alpha * T;
                    if (do_depth) invd += (1.0f / depths[g]) * alpha * T;
                    T = test_T;
                    last = contributor;
                }
                size_t pix = (size_t)py * W + px;
                final_T[pix] = T; n_contrib[pix] = last;
                for (int c = 0; c < 3; c++) out_color[(size_t)c * H * W + pix] = C[c] + T * bg[c];
                if (do_depth) out_invdepth[pix] = invd;
            }
    }
}

/* ------------------------------------------------------------------ */
/* K7: per-tile back-to-front gradient replay                          */
/* accumulators are double [P][k]; caller converts.                    */
/* ------------------------------------------------------------------ */
void oracle_render_backward(int W, int H, const uint32_t* ranges, const uint32_t* point_list,
                            const float* xy, const float* rgb, const float* conic_opacity, const float* depths,
                            const float* ts, const int* kids, const float* bg,
                            const float* final_T, const uint32_t* n_contrib,
                            const float* dL_dpix, const float* dL_dinvdepth_pix,
                            /* out (double, zero-initialised by caller) */
                            double* dL_dmean2D /*[P][2]*/, double* dL_dconic /*[P][3]*/, double* dL_dopacity /*[P]*/,
                            double* dL_dcolor /*[P][3]*/, double* dL_dinvdepth /*[P]*/)
{
    /* DECISIONS (power > 0, alpha < 1/255, which entries contributed) are taken in fp32
     * exactly as the forward took them; VALUES are then evaluated in double, so the result
     * is the exact-arithmetic value of the published backward formulas for the fp32 inputs.
     * Any fp32 implementation (the reference's atomics in arbitrary order included) can
     * only differ from it by its own rounding. */
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    const double ddelx_dx = 0.5 * W, ddely_dy = 0.5 * H;
#pragma omp parallel for schedule(dynamic, 4)
    for (int tile = 0; tile < gx * gy; tile++) {
        int tx = tile % gx, ty = tile / gx;
        uint32_t s = ranges[2 * tile];
        for (int py = ty * TILE; py < (ty + 1) * TILE && py < H; py++)
            for (int px = tx * TILE; px < (tx + 1) * TILE && px < W; px++) {
                size_t pix = (size_t)py * W + px;
                const double T_final = final_T[pix];
                double T = T_final;
                uint32_t last = n_contrib[pix];
                double accum_rec[3] = { 0, 0, 0 }, last_color[3] = { 0, 0, 0 }, last_alpha = 0.;
                double accum_invd = 0., last_invd = 0.;
                double dpix[3];
                for (int c = 0; c < 3; c++) dpix[c] = dL_dpix[(size_t)c * H * W + pix];
                double dinv = dL_dinvdepth_pix ? dL_dinvdepth_pix[pix] : 0.;
                double bg_dot = 0.;
                for (int c = 0; c < 3; c++) bg_dot += (double)bg[c] * dpix[c];
                for (uint32_t jj = last; jj-- > 0;) {
                    uint32_t g = point_list[s + jj];
                    const float* co = conic_opacity + 4 * g;
                    /* fp32 decision path (identical to oracle_render_forward) */
                    float dxf = xy[2 * g] - (float)px, dyf = xy[2 * g + 1] - (float)py;
                    float powerf = -0.5f * (co[0] * dxf * dxf + co[2] * dyf * dyf) - co[1] * dxf * dyf;
                    if (powerf > 0.0f) continue;
                    float alphaf = fminf(ALPHA_CAP, co[3] * expf(powerf));
                    if (ts) alphaf = hier_alpha(alphaf, ts[g], kids[g]);
                    if (alphaf < ALPHA_SKIP) continue;
                    /* double value path */
                    double dx = (double)xy[2 * g] - px, dy = (double)xy[2 * g + 1] - py;
                    double power = -0.5 * ((double)co[0] * dx * dx + (double)co[2] * dy * dy) - (double)co[1] * dx * dy;
                    double G = exp(power);
                    double abase = fmin((double)ALPHA_CAP, (double)co[3] * G);
                    double alpha = abase, dadb = 1.0;
                    if (ts && kids[g] > 1 && ts[g] < 1.0f) {
                        double t = ts[g], ik = 1.0 / kids[g];
                        alpha = t * abase + (1.0 - t) * (1.0 - pow(1.0 - abase, ik));
                        dadb = t + (1.0 - t) * ik * pow(1.0 - abase, ik - 1.0);
                    }
                    T = T / (1. - alpha);
                    const double dchannel_dcolor = alpha * T;
                    double dL_dalpha = 0.;
                    for (int c = 0; c < 3; c++) {
                        double col = rgb[3 * g + c];
                        accum_rec[c] = last_alpha * last_color[c] + (1. - last_alpha) * accum_rec[c];
                        last_color[c] = col;
                        dL_dalpha += (col - accum_rec[c]) * dpix[c];
#pragma omp atomic
                        dL_dcolor[3 * (size_t)g + c] += dchannel_dcolor * dpix[c];
                    }
                    if (dL_dinvdepth_pix) {
                        double invd = 1. / (double)depths[g];
                        accum_invd = last_alpha * last_invd + (1. - last_alpha) * accum_invd;
                        last_invd = invd;
                        dL_dalpha += (invd - accum_invd) * dinv;
#pragma omp atomic
                        dL_dinvdepth[g] += dchannel_dcolor * dinv;
                    }
                    dL_dalpha *= T;
                    last_alpha = alpha;
                    dL_dalpha += (-T_final / (1. - alpha)) * bg_dot;
                    /* chain through the hierarchy weight; the 0.99 cap is NOT differentiated
                     * (published backward treats alpha = o*G). */
                    const double dL_dab = dL_dalpha * dadb;
                    const double dL_dG = (double)co[3] * dL_dab;
                    const double gdx = G * dx, gdy = G * dy;
                    const double dG_ddelx = -gdx * co[0] - gdy * co[1];
                    const double dG_ddely = -gdy * co[2] - gdx * co[1];
#pragma omp atomic
                    dL_dmean2D[2 * (size_t)g] += dL_dG * dG_ddelx * ddelx_dx;
#pragma omp atomic
                    dL_dmean2D[2 * (size_t)g + 1] += dL_dG * dG_ddely * ddely_dy;
#pragma omp atomic
                    dL_dconic[3 * (size_t)g] += -0.5 * gdx * dx * dL_dG;
#pragma omp atomic
                    dL_dconic[3 * (size_t)g + 1] += -0.5 * gdx * dy * dL_dG;
#pragma omp atomic
                    dL_dconic[3 * (size_t)g + 2] += -0.5 * gdy * dy * dL_dG;
#pragma omp atomic
                    dL_dopacity[g] += G * dL_dab;
                }
            }
    }
}

/* ------------------------------------------------------------------ */
/* K8 + K9: per-Gaussian chain rule back to the inputs                 */
/* ------------------------------------------------------------------ */
typedef struct { double x, y, z; } d3;
static inline d3 xform4x3d(const float* m, d3 p) {
    d3 r;
    r.x = (double)m[0] * p.x + (double)m[4] * p.y + (double)m[8] * p.z + m[12];
    r.y = (double)m[1] * p.x + (double)m[5] * p.y + (double)m[9] * p.z + m[13];
    r.z = (double)m[2] * p.x + (double)m[6] * p.y + (double)m[10] * p.z + m[14];
    return r;
}
static inline void xform4x4d(const float* m, d3 p, double out[4]) {
    for (int j = 0; j < 4; j++) out[j] = (double)m[j] * p.x + (double)m[4 + j] * p.y + (double)m[8 + j] * p.z + m[12 + j];
}
static inline void quat_to_Rd(const float* q, double R[3][3]) {
    double r = q[0], x = q[1], y = q[2], z = q[3];
    R[0][0] = 1. - 2. * (y * y + z * z); R[0][1] = 2. * (x * y - r * z); R[0][2] = 2. * (x * z + r * y);
    R[1][0] = 2. * (x * y + r * z); R[1][1] = 1. - 2. * (x * x + z * z); R[1][2] = 2. * (y * z - r * x);
    R[2][0] = 2. * (x * z - r * y); R[2][1] = 2. * (y * z + r * x); R[2][2] = 1. - 2. * (x * x + y * y);
}
/* K8 + K9 evaluate the published chain-rule formulas in DOUBLE on the fp32 inputs
 * (see the note in oracle_render_backward); outputs are rounded to fp32 once. */
void oracle_preprocess_backward(int P, int deg, int M,
                                const float* means3D, const float* scales, float scale_mod, const float* rots,
                                const float* shs, const float* cov3D_precomp, const float* colors_precomp,
                                const float* view, const float* proj, const float* campos,
                                int W, int H, float tanx, float tany,
                                const int* radii, const float* cov3Ds, const uint8_t* clamped,
                                const double* dL_dmean2D /*[P][2]*/, const double* dL_dconic /*[P][3]*/,
                                const double* dL_dcolor /*[P][3]*/, const double* dL_dinvdepth /*[P] or NULL*/,
                                /* out, zero-initialised by caller */
                                float* dL_dmeans3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot)
{
    const double fx = W / (2.0 * tanx), fy = H / (2.0 * tany);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) {
        if (radii[i] <= 0) continue;
        d3 mean = { means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2] };
        const float* cov6 = cov3D_precomp ? cov3D_precomp + 6 * i : cov3Ds + 6 * i;
        double dmean[3] = { 0, 0, 0 };
        double g6d[6] = { 0, 0, 0, 0, 0, 0 };

        /* ---- K8: conic -> cov2D -> cov3D and mean (through J) ---- */
        {
            d3 t = xform4x3d(view, mean);
            const double limx = FOV_CLAMP * tanx, limy = FOV_CLAMP * tany;
            const double txtz = t.x / t.z, tytz = t.y / t.z;
            t.x = fmin(limx, fmax(-limx, txtz)) * t.z;
            t.y = fmin(limy, fmax(-limy, tytz)) * t.z;
            /* the gradient mask is the FORWARD's fp32 clamp decision (cov2d_project), not a double one: the backward
             * differentiates what the forward computed */
            const f3 tf = xform4x3(view, (f3){ means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2] });
            const float limxf = FOV_CLAMP * tanx, limyf = FOV_CLAMP * tany;
            const float txtzf = tf.x / tf.z, tytzf = tf.y / tf.z;
            const double x_grad_mul = (txtzf < -limxf || txtzf > limxf) ? 0. : 1.;
            const double y_grad_mul = (tytzf < -limyf || tytzf > limyf) ? 0. : 1.;
            double J00 = fx / t.z, J02 = -(fx * t.x) / (t.z * t.z);
            double J11 = fy / t.z, J12 = -(fy * t.y) / (t.z * t.z);
            double A[2][3];
            for (int c = 0; c < 3; c++) {
                A[0][c] = J00 * view[4 * c + 0] + J02 * view[4 * c + 2];
                A[1][c] = J11 * view[4 * c + 1] + J12 * view[4 * c + 2];
            }
            double V[3][3] = { { cov6[0], cov6[1], cov6[2] }, { cov6[1], cov6[3], cov6[4] }, { cov6[2], cov6[4], cov6[5] } };
            double AV[2][3];
            for (int r = 0; r < 2; r++)
                for (int c = 0; c < 3; c++)
                    AV[r][c] = A[r][0] * V[0][c] + A[r][1] * V[1][c] + A[r][2] * V[2][c];
            double a = (AV[0][0] * A[0][0] + AV[0][1] * A[0][1] + AV[0][2] * A[0][2]) + DILATION;
            double b = AV[0][0] * A[1][0] + AV[0][1] * A[1][1] + AV[0][2] * A[1][2];
            double c_ = (AV[1][0] * A[1][0] + AV[1][1] * A[1][1] + AV[1][2] * A[1][2]) + DILATION;
            double denom = a * c_ - b * b;
            double dL_da = 0, dL_db = 0, dL_dc = 0;
            double denom2inv = 1.0 / ((denom * denom) + 0.0000001);
            const double dcx = dL_dconic[3 * i], dcy = dL_dconic[3 * i + 1], dcz = dL_dconic[3 * i + 2];
            if (denom2inv != 0) {
                /* conic = (c, -b, a)/denom ; dL_dconic.y holds the gradient of the
                 * single stored off-diagonal (used twice in the quadratic form). */
                dL_da = denom2inv * (-c_ * c_ * dcx + 2 * b * c_ * dcy + (denom - a * c_) * dcz);
                dL_dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * c_) * dcx);
                dL_db = denom2inv * 2 * (b * c_ * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
                /* cov2D = A V A^T : d/dV */
                double* o = g6d;
                o[0] = A[0][0] * A[0][0] * dL_da + A[0][0] * A[1][0] * dL_db + A[1][0] * A[1][0] * dL_dc;
                o[3] = A[0][1] * A[0][1] * dL_da + A[0][1] * A[1][1] * dL_db + A[1][1] * A[1][1] * dL_dc;
                o[5] = A[0][2] * A[0][2] * dL_da + A[0][2] * A[1][2] * dL_db + A[1][2] * A[1][2] * dL_dc;
                /* off-diagonals appear twice in the symmetric V */
                o[1] = 2 * A[0][0] * A[0][1] * dL_da + (A[0][0] * A[1][1] + A[0][1] * A[1][0]) * dL_db + 2 * A[1][0] * A[1][1] * dL_dc;
                o[2] = 2 * A[0][0] * A[0][2] * dL_da + (A[0][0] * A[1][2] + A[0][2] * A[1][0]) * dL_db + 2 * A[1][0] * A[1][2] * dL_dc;
                o[4] = 2 * A[0][2] * A[0][1] * dL_da + (A[0][1] * A[1][2] + A[0][2] * A[1][1]) * dL_db + 2 * A[1][1] * A[1][2] * dL_dc;
            }
            for (int k6 = 0; k6 < 6; k6++) dL_dcov3D[6 * i + k6] = (float)g6d[k6];
            /* d/dA[r][c] = 2*(AV)[r][c]*dL_d{a,c} + (AV)[other][c]*dL_db */
            double dA[2][3];
            for (int c = 0; c < 3; c++) {
                dA[0][c] = 2 * AV[0][c] * dL_da + AV[1][c] * dL_db;
                dA[1][c] = 2 * AV[1][c] * dL_dc + AV[0][c] * dL_db;
            }
            /* A = J Rwv, Rwv[k][c] = view[4c+k] : dJ[r][k] = sum_c dA[r][c] Rwv[k][c] */
            double dJ00 = dA[0][0] * view[0] + dA[0][1] * view[4] + dA[0][2] * view[8];
            double dJ02 = dA[0][0] * view[2] + dA[0][1] * view[6] + dA[0][2] * view[10];
            double dJ11 = dA[1][0] * view[1] + dA[1][1] * view[5] + dA[1][2] * view[9];
            double dJ12 = dA[1][0] * view[2] + dA[1][1] * view[6] + dA[1][2] * view[10];
            double tz = 1. / t.z, tz2 = tz * tz, tz3 = tz2 * tz;
            double dL_dtx = x_grad_mul * -fx * tz2 * dJ02;
            double dL_dty = y_grad_mul * -fy * tz2 * dJ12;
            double dL_dtz = -fx * tz2 * dJ00 - fy * tz2 * dJ11 + (2 * fx * t.x) * tz3 * dJ02 + (2 * fy * t.y) * tz3 * dJ12;
            /* inverse-depth output: invdepth = 1/t.z */
            if (dL_dinvdepth) dL_dtz -= dL_dinvdepth[i] / (t.z * t.z);
            /* t = p . view(4x3): dmean_k = sum_j view[4k + j] dt_j */
            dmean[0] += view[0] * dL_dtx + view[1] * dL_dty + view[2] * dL_dtz;
            dmean[1] += view[4] * dL_dtx + view[5] * dL_dty + view[6] * dL_dtz;
            dmean[2] += view[8] * dL_dtx + view[9] * dL_dty + view[10] * dL_dtz;
        }

        /* ---- K9a: screen-space mean -> 3D mean through the projection ---- */
        {
            double mh[4]; xform4x4d(proj, mean, mh);
            double m_w = 1.0 / (mh[3] + W_EPS);
            double mul1 = (proj[0] * mean.x + proj[4] * mean.y + proj[8] * mean.z + proj[12]) * m_w * m_w;
            double mul2 = (proj[1] * mean.x + proj[5] * mean.y + proj[9] * mean.z + proj[13]) * m_w * m_w;
            double gx_ = dL_dmean2D[2 * i], gy_ = dL_dmean2D[2 * i + 1];
            dmean[0] += (proj[0] * m_w - proj[3] * mul1) * gx_ + (proj[1] * m_w - proj[3] * mul2) * gy_;
            dmean[1] += (proj[4] * m_w - proj[7] * mul1) * gx_ + (proj[5] * m_w - proj[7] * mul2) * gy_;
            dmean[2] += (proj[8] * m_w - proj[11] * mul1) * gx_ + (proj[9] * m_w - proj[11] * mul2) * gy_;
        }

        /* ---- K9b: colour -> SH coefficients and view direction -> mean ---- */
        if (!colors_precomp) {
            const float* sh = shs + (size_t)i * M * 3;
            float* dsh = dL_dsh + (size_t)i * M * 3;
            d3 d0 = { mean.x - campos[0], mean.y - campos[1], mean.z - campos[2] };
            double len = sqrt(d0.x * d0.x + d0.y * d0.y + d0.z * d0.z);
            double x = d0.x / len, y = d0.y / len, z = d0.z / len;
            double dRGB[3];
            for (int c = 0; c < 3; c++) dRGB[c] = clamped[3 * i + c] ? 0. : dL_dcolor[3 * i + c];
            double ddx = 0, ddy = 0, ddz = 0; /* dL/d(dir) */
#define S(k, c) sh[(k) * 3 + (c)]
#define DS(k, c) dsh[(k) * 3 + (c)]
            for (int c = 0; c < 3; c++) {
                double g = dRGB[c];
                double dx_ = 0, dy_ = 0, dz_ = 0;
                DS(0, c) = SH_C0 * g;
                if (deg > 0) {
                    DS(1, c) = -SH_C1 * y * g; DS(2, c) = SH_C1 * z * g; DS(3, c) = -SH_C1 * x * g;
                    dx_ = -SH_C1 * S(3, c); dy_ = -SH_C1 * S(1, c); dz_ = SH_C1 * S(2, c);
                    if (deg > 1) {
                        double xx = x * x, yy = y * y, zz = z * z, xy_ = x * y, yz = y * z, xz = x * z;
                        DS(4, c) = SH_C2[0] * xy_ * g; DS(5, c) = SH_C2[1] * yz * g;
                        DS(6, c) = SH_C2[2] * (2. * zz - xx - yy) * g;
                        DS(7, c) = SH_C2[3] * xz * g; DS(8, c) = SH_C2[4] * (xx - yy) * g;
                        dx_ += SH_C2[0] * y * S(4, c) + SH_C2[2] * 2. * -x * S(6, c) + SH_C2[3] * z * S(7, c) + SH_C2[4] * 2. * x * S(8, c);
                        dy_ += SH_C2[0] * x * S(4, c) + SH_C2[1] * z * S(5, c) + SH_C2[2] * 2. * -y * S(6, c) + SH_C2[4] * 2. * -y * S(8, c);
                        dz_ += SH_C2[1] * y * S(5, c) + SH_C2[2] * 2. * 2. * z * S(6, c) + SH_C2[3] * x * S(7, c);
                        if (deg > 2) {
                            DS(9, c) = SH_C3[0] * y * (3. * xx - yy) * g;
                            DS(10, c) = SH_C3[1] * xy_ * z * g;
                            DS(11, c) = SH_C3[2] * y * (4. * zz - xx - yy) * g;
                            DS(12, c) = SH_C3[3] * z * (2. * zz - 3. * xx - 3. * yy) * g;
                            DS(13, c) = SH_C3[4] * x * (4. * zz - xx - yy) * g;
                            DS(14, c) = SH_C3[5] * z * (xx - yy) * g;
                            DS(15, c) = SH_C3[6] * x * (xx - 3. * yy) * g;
                            dx_ += SH_C3[0] * S(9, c) * 3. * 2. * xy_ + SH_C3[1] * S(10, c) * yz + SH_C3[2] * S(11, c) * -2. * xy_
                                 + SH_C3[3] * S(12, c) * -3. * 2. * xz + SH_C3[4] * S(13, c) * (-3. * xx + 4. * zz - yy)
                                 + SH_C3[5] * S(14, c) * 2. * xz + SH_C3[6] * S(15, c) * 3. * (xx - yy);
                            dy_ += SH_C3[0] * S(9, c) * 3. * (xx - yy) + SH_C3[1] * S(10, c) * xz + SH_C3[2] * S(11, c) * (-3. * yy + 4. * zz - xx)
                                 + SH_C3[3] * S(12, c) * -3. * 2. * yz + SH_C3[4] * S(13, c) * -2. * xy_
                                 + SH_C3[5] * S(14, c) * -2. * yz + SH_C3[6] * S(15, c) * -3. * 2. * xy_;
                            dz_ += SH_C3[1] * S(10, c) * xy_ + SH_C3[2] * S(11, c) * 4. * 2. * yz + SH_C3[3] * S(12, c) * 3. * (2. * zz - xx - yy)
                                 + SH_C3[4] * S(13, c) * 4. * 2. * xz + SH_C3[5] * S(14, c) * (xx - yy);
                        }
                    }
                }
                ddx += dx_ * g; ddy += dy_ * g; ddz += dz_ * g;
            }
#undef S
#undef DS
            /* through dir = d0/|d0| */
            double sum2 = d0.x * d0.x + d0.y * d0.y + d0.z * d0.z;
            double invsum32 = 1.0 / sqrt(sum2 * sum2 * sum2);
            dmean[0] += ((+sum2 - d0.x * d0.x) * ddx - d0.y * d0.x * ddy - d0.z * d0.x * ddz) * invsum32;
            dmean[1] += (-d0.x * d0.y * ddx + (sum2 - d0.y * d0.y) * ddy - d0.z * d0.y * ddz) * invsum32;
            dmean[2] += (-d0.x * d0.z * ddx - d0.y * d0.z * ddy + (sum2 - d0.z * d0.z) * ddz) * invsum32;
        }
        dL_dmeans3D[3 * i] = dmean[0]; dL_dmeans3D[3 * i + 1] = dmean[1]; dL_dmeans3D[3 * i + 2] = dmean[2];

        /* ---- K9c: cov3D -> scale, rotation ---- */
        if (!cov3D_precomp) {
            const float* q = rots + 4 * i;
            double r = q[0], x = q[1], y = q[2], z = q[3];
            double R[3][3]; quat_to_Rd(q, R);
            double s[3] = { scale_mod * scales[3 * i], scale_mod * scales[3 * i + 1], scale_mod * scales[3 * i + 2] };
            /* M[k][i] = s_k R[i][k] ; Sigma = M^T M */
            double Mm[3][3];
            for (int k = 0; k < 3; k++) for (int j = 0; j < 3; j++) Mm[k][j] = s[k] * R[j][k];
            const double* g6 = g6d;
            /* symmetric dL/dSigma with off-diagonals halved (they were accumulated for both uses) */
            double dS[3][3] = { { g6[0], 0.5 * g6[1], 0.5 * g6[2] }, { 0.5 * g6[1], g6[3], 0.5 * g6[4] }, { 0.5 * g6[2], 0.5 * g6[4], g6[5] } };
            /* dL/dM = 2 M dSigma */
            double dM[3][3];
            for (int k = 0; k < 3; k++) for (int j = 0; j < 3; j++)
                dM[k][j] = 2.0 * (Mm[k][0] * dS[0][j] + Mm[k][1] * dS[1][j] + Mm[k][2] * dS[2][j]);
            /* M[k][j] = s_k R[j][k] : dscale_k = sum_j R[j][k] dM[k][j] (times scale_mod) */
            for (int k = 0; k < 3; k++)
                dL_dscale[3 * i + k] = scale_mod * (R[0][k] * dM[k][0] + R[1][k] * dM[k][1] + R[2][k] * dM[k][2]);
            /* dR[j][k] = s_k dM[k][j] */
            double dR[3][3];
            for (int j = 0; j < 3; j++) for (int k = 0; k < 3; k++) dR[j][k] = s[k] * dM[k][j];
            /* R entries as functions of (r,x,y,z) */
            double dq_r = 2 * z * (dR[1][0] - dR[0][1]) + 2 * y * (dR[0][2] - dR[2][0]) + 2 * x * (dR[2][1] - dR[1][2]);
            double dq_x = 2 * y * (dR[0][1] + dR[1][0]) + 2 * z * (dR[0][2] + dR[2][0]) + 2 * r * (dR[2][1] - dR[1][2]) - 4 * x * (dR[1][1] + dR[2][2]);
            double dq_y = 2 * x * (dR[0][1] + dR[1][0]) + 2 * r * (dR[0][2] - dR[2][0]) + 2 * z * (dR[1][2] + dR[2][1]) - 4 * y * (dR[0][0] + dR[2][2]);
            double dq_z = 2 * r * (dR[1][0] - dR[0][1]) + 2 * x * (dR[0][2] + dR[2][0]) + 2 * y * (dR[1][2] + dR[2][1]) - 4 * z * (dR[0][0] + dR[1][1]);
            dL_drot[4 * i] = dq_r; dL_drot[4 * i + 1] = dq_x; dL_drot[4 * i + 2] = dq_y; dL_drot[4 * i + 3] = dq_z;
        }
    }
}

/* ------------------------------------------------------------------ */
/* Hierarchy LOD cut (gaussian_hierarchy._C.expand_to_size /           */
/* get_interpolation_weights; call sites train_post.py:91-113).        */
/* Node = 7 x int32 {depth,parent,start,count_leafs,count_merged,      */
/*        start_children,count_children}; Box = 2 x float4 {min,max},  */
/* min.w carries the node's size numerator (UNPINNED layout).          */
/* ------------------------------------------------------------------ */
static inline float node_size(const float* box, const float* vp) {
    const float* mn = box; const float* mx = box + 4;
    int inside = vp[0] >= mn[0] && vp[0] <= mx[0] && vp[1] >= mn[1] && vp[1] <= mx[1] && vp[2] >= mn[2] && vp[2] <= mx[2];
    if (inside) return FLT_MAX;
    float cx = fmaxf(mn[0], fminf(mx[0], vp[0])) - vp[0];
    float cy = fmaxf(mn[1], fminf(mx[1], vp[1])) - vp[1];
    float cz = fmaxf(mn[2], fminf(mx[2], vp[2])) - vp[2];
    float dist = sqrtf(cx * cx + cy * cy + cz * cz);
    return mn[3] / dist;
}

int oracle_expand_to_size(int N, const int* nodes, const float* boxes, float target, const float* viewpoint,
                          int* render_indices, int* parent_indices, int* nodes_for_render)
{
    int out = 0;
    for (int n = 0; n < N; n++) {
        const int* nd = nodes + 7 * n;
        int parent = nd[1];
        float size = node_size(boxes + 8 * n, viewpoint);
        int count = 0;
        if (size >= target) count = nd[3];                       /* too coarse: only its leaf Gaussians */
        else if (parent != -1) {
            float psize = node_size(boxes + 8 * parent, viewpoint);
            if (psize >= target) { count = nd[3]; if (nd[0] != 0) count += nd[4]; }  /* on the cut */
        }
        int pg = parent != -1 ? nodes[7 * parent + 2] : -1;
        for (int k = 0; k < count; k++) {
            render_indices[out] = nd[2] + k; parent_indices[out] = pg; nodes_for_render[out] = n; out++;
        }
    }
    return out;
}

void oracle_interpolation_weights(int n, const int* node_indices, float target, const int* nodes, const float* boxes,
                                  const float* viewpoint, float* ts, int* kids)
{
    for (int i = 0; i < n; i++) {
        int id = node_indices[i];
        const int* nd = nodes + 7 * id;
        int parent = nd[1];
        float t;
        if (parent == -1) t = 1.0f;
        else {
            float psize = node_size(boxes + 8 * parent, viewpoint);
            if (psize > 2.0f * target) t = 1.0f;
            else {
                float size = node_size(boxes + 8 * id, viewpoint);
                float start = fmaxf(0.5f * psize, size);
                float diff = psize - start;
                if (diff <= 0) t = 1.0f;
                else { float tdiff = fmaxf(0.0f, target - start); t = fmaxf(1.0f - (tdiff / diff), 0.0f); }
            }
        }
        ts[i] = t;
        kids[i] = parent == -1 ? 1 : nodes[7 * parent + 6];
    }
}

/* torchrun exports OMP_NUM_THREADS=1; the CPU legs of bench.py ask for all host cores explicitly */
void oracle_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int oracle_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
