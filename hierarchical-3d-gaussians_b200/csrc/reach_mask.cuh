// reach_mask.cuh -- which 4x4-pixel blocks of a tile an entry can reach (used by the record gather of
// binning.cu; the blend kernels skip everything else).  Also compiled for the host by tests/emul/reach_mask_test.cpp,
// which checks it against a brute-force per-pixel evaluation.
#pragma once
#ifdef H3_REACH_HOST_TEST
#include <math.h>
#include <stdint.h>
#include <algorithm>
#define __device__
#define __forceinline__ inline
struct float4 { float x, y, z, w; };
#define H3_FAST_LOGF(x) logf(x)
#define H3_FMAF(a, b, c) fmaf(a, b, c)
using std::max; using std::min;
namespace h3dgs { constexpr int kTile = 16; }
#else
#define H3_FAST_LOGF(x) __logf(x)
#define H3_FMAF(a, b, c) __fmaf_rn(a, b, c)
#endif

namespace h3dgs {

// Which of the sixteen 4x4-pixel blocks of tile (tile_x, tile_y) can entry (a, b) reach at all?
// Bit 4 q + g: quadrant q = (qx, qy) of the tile (the warp of the blend CTAs), block g = (bx, by) inside it
// (an 8-lane group of that warp); the quadrant is reached iff any of its four bits is set.
// alpha >= 1/255  <=>  q(e) = A ex^2 + 2 B ex ey + C ey^2 <= 2 ln(255 o) =: bound, e = pixel - mean.
// Scanline form: inside a band of rows [y0, y0+3] the ellipse {q <= bound} projects onto the x interval
// [lo, hi]; hi is attained at the band's row nearest to the ellipse's rightmost point (ey = -B sqrt(bound/(det C))),
// lo at the row nearest to the leftmost point (-ey): two square roots per band.  The ellipse cut by the band is
// convex, so a block column [4 bx, 4 bx + 3] is reached iff it overlaps [lo, hi] -- the same (exact, over the
// rectangle of pixel centres) criterion as a per-block minimisation of q, at a fraction of the instructions.
// Margins (U = 2^-24, the fp32 unit roundoff), so that skipping a block never changes a result:
//  - The blend takes a pixel iff fp32 alpha >= fp32(1/255), equality included, and its alpha is o G with G <= 1.
//    fp32(1/255) = 0.0039215689 lies just above the real 1/255: its exact product with 255, 1 + 5.9e-8, rounds down to
//    1.0, so a test o255 > 1 would reject an opacity the blend takes (alpha = o at G = 1, on a pixel centre).  The next
//    opacity below gives 0.99999994 and an alpha below fp32(1/255) for every G, so o255 >= 1 keeps exactly the
//    opacities the blend can take; o255 = 1 leaves bound = the 1e-3 floor, which covers the means within ~1 ulp of a
//    pixel centre there.
//  - One exception to "never changes a result": a NaN opacity gives mask 0, while the blend's own arithmetic would take
//    the entry (fminf(0.99, NaN) = 0.99) wherever power <= 0.  It is the mask that keeps NaN-opacity rows invisible.
//  - A conic that is not positive definite (K1 lists indefinite ones: it only rejects det = 0), a non-finite mean or
//    conic, or a band bound the scanline form cannot use gives 0xFFFF: the blend then decides every pixel itself.
//  - The blend's own alpha is fp32: its power, a sum of terms of total magnitude mag(e) = |A| ex^2 + 2 |B ex ey| + |C| ey^2
//    (q units), and ex2.approx carry a relative alpha error of at most eps = 2 U mag + 2^-22 + 3 U (2 U mag: the
//    4 U-per-power-magnitude bound of tests/blend_ref.py; + 4e-6 for the hierarchy weight), so a pixel with exact q up
//    to bound + 8 eps = bound + 16 U mag + 4e-5 may be taken (ln alpha moves by at most 4 eps: the same fourfold safety
//    factor blend_ref puts on its decision margin).  mag exceeds q only through the cross term: mag = q + 4 |B ex ey|
//    when B ex ey < 0.  Over a band of rows |ey| <= Y (its farthest row) and over the tile's columns |ex| <= X, so the
//    band's bound is bound + 64 U |B| X Y (the 16 U q part and the constants sit under the factor 1.002 and the 1e-3
//    floor).  For a round Gaussian the term is ~1e-5 of bound.  Along a Gaussian seen edge-on (sigma_long of hundreds
//    of px at the 0.3 px^2 dilation floor) q grows as |e|^2 / sigma_long^2, no faster than the fp32 error of its terms
//    (~U |B| |e|^2), so the blend's fp32 power cannot resolve where the tip ends: the term widens it there.
//  - det = A C - B^2 cancels on such needles (A C / det ~1e5..1e6), so A*C - B*B rounded in fp32 would carry a relative
//    error of 2 U A C / det, up to several percent, and move the tips (er, det e^2 against A bound in d) by pixels.
//    Kahan's form -- w = B*B, det = fma(A, C, -w) - fma(B, B, -w) (the second term is w's rounding error, exact) -- is
//    within 2 U of the exact det for any conditioning.
//  - With det, A, B, C exact to a few U, d carries an error of a few U A bound, which the factor 1.002 on the bound
//    (a 2e-3 A bound increase of d) covers with room; hi / lo carry a few U relative on the half width (factor 1.001)
//    and on the offsets of the mean (rx, B/A e: 2e-3 px absolute); __logf's absolute error (~2^-21) sits under the floor.
// Host and device compute the same sequence (binning.cu is compiled with -fmad=false; the fma's are explicit).
__device__ __forceinline__ uint32_t block_mask16(const float4& a, const float4& b, int tile_x, int tile_y)
{
    const float A = a.z, B = a.w, C = b.x;
    const float bb = B * B;
    const float det = H3_FMAF(A, C, -bb) - H3_FMAF(B, B, -bb);
    const float o255 = b.y * 255.0f;
    if (!(o255 >= 1.0f)) return 0u;                    // can never reach alpha >= 1/255 (NaN opacity: hidden here)
    const float bound = 2.0f * H3_FAST_LOGF(o255) * 1.002f + 1e-3f;
    const float rx = a.x - (float)(tile_x * kTile), ry = a.y - (float)(tile_y * kTile);
    // (det <= FLT_MAX: an infinite A or C makes det infinite, and the scanline form would meet inf * 0)
    if (!(det > 0.0f && det <= 3.40282347e38f && A > 0.0f && C > 0.0f) || !(bound == bound && rx == rx && ry == ry))
        return 0xFFFFu;
    const float invA = 1.0f / A, BoA = B * invA;
    const float wBX = 3.8146973e-6f * fabsf(B) * fmaxf(fabsf(rx), fabsf(rx - 15.0f));   // 64 U |B| X
    uint32_t rows = 0u;                                  // row-major: bit 4 by + bx
#pragma unroll
    for (int by = 0; by < 4; by++) {
        const float y0 = (float)(4 * by) - ry, y1 = y0 + 3.0f;          // the band's rows relative to the mean
        const float bnd = bound + wBX * fmaxf(fabsf(y0), fabsf(y1)), Ab = A * bnd;
        const float er = -B * sqrtf(bnd / (det * C));  // row offset (from the mean) of the rightmost point; leftmost: -er
        if (!(er == er) || fabsf(er) > 1e6f || !(Ab < 3.0e37f)) return 0xFFFFu;
        const float e_hi = fminf(y1, fmaxf(y0, er)), e_lo = fminf(y1, fmaxf(y0, -er));
        const float d_hi = Ab - det * e_hi * e_hi, d_lo = Ab - det * e_lo * e_lo;
        if (fmaxf(d_hi, d_lo) < -1e-3f * Ab) continue;                  // the band misses the ellipse
        const float hi = rx - BoA * e_hi + (sqrtf(fmaxf(d_hi, 0.0f)) * invA * 1.001f + 2e-3f);
        const float lo = rx - BoA * e_lo - (sqrtf(fmaxf(d_lo, 0.0f)) * invA * 1.001f + 2e-3f);
        // block bx covers pixel centres 4 bx .. 4 bx + 3 in tile coordinates
        const int b0 = max(0, (int)ceilf((fmaxf(lo, -8.0f) - 3.0f) * 0.25f)), b1 = min(3, (int)floorf(fminf(hi, 24.0f) * 0.25f));
        if (b0 <= b1) rows |= ((2u << b1) - (1u << b0)) << (4 * by);
    }
    // row-major -> quadrant-major: per byte (two block rows) the bit pairs {0,1},{4,5} | {2,3},{6,7} form the nibbles
    const uint32_t m = (rows & 0x0303u) | ((rows >> 2) & 0x0C0Cu) | ((rows << 2) & 0x3030u) | (rows & 0xC0C0u);
    return m;
}

}  // namespace h3dgs
