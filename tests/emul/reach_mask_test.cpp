// CPU check of csrc/reach_mask.cuh::block_mask16 (test infrastructure only): for projected Gaussians and tile positions,
// every pixel of the tile whose alpha = min(0.99, o exp(-q/2)) reaches 1/255 (the blend's fp32 test, equality taken)
// must lie in a block the mask marks (skipping an unmarked block must never change a result), and the mask must be
// tight: marked blocks that the ellipse {q <= 2 ln(255 o)} does not touch at all (exact minimum of q over the block's
// rectangle of pixel centres, in double) and that hold no pixel within the blend's fp32 margin (exact q <= 2 ln(255 o)
// + 16 U mag: tests/blend_ref.py's decision margin on alpha, in q) stay below 2 % of the marked blocks.
// Three families, each judged on its own:
//   random  -- sigma 0.3 .. 12 px at any angle, opacities 10^-2.6 .. 1 and up to 1.6, means up to 22 px off the tile;
//   needle  -- Gaussians seen edge-on: sigma_long 50 .. 600 px at any angle, sigma_short at the 0.3 px^2 dilation floor
//              (condition numbers up to ~1e6), every tile of the ellipse's bounding box;
//   1/255   -- opacity prev / fp32 / next of 1/255 with the mean on a pixel centre, on a tile corner and on tile edges,
//              exactly and 1 ulp off, checked on the tile of the mean and its eight neighbours;
//   degenerate -- conics that are not positive definite (indefinite, negative, det exactly 0) and NaN / inf in the mean
//              or the conic must give the fallback 0xFFFF whenever the opacity can be taken (o >= fp32(1/255)), 0 below
//              it; a NaN opacity gives 0 (the mask hides the row).  No pixel may be missed; tightness is not asked.
#define H3_REACH_HOST_TEST
#include "../../hierarchical-3d-gaussians_b200/csrc/reach_mask.cuh"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
using namespace h3dgs;

static double urand() { return (double)rand() / RAND_MAX; }
static int bit_of(int bx, int by) { return 4 * ((bx >> 1) | ((by >> 1) << 1)) + ((bx & 1) | ((by & 1) << 1)); }

struct Family {
    const char* name;
    long entries = 0, missed = 0, missed_px = 0, marked = 0, marked_untouched = 0, needed = 0, wrong = 0;
    bool tight = true;
};

// exact minimum over [x0, x1] x [y0, y1] of q(e) = A ex^2 + 2 B ex ey + C ey^2, e = p - m (A, C > 0, AC > B^2):
// 0 if the mean is inside, else attained on an edge, where q is a 1-D convex quadratic
static double rect_min_q(double A, double B, double C, double mx, double my, double x0, double x1, double y0, double y1) {
    if (mx >= x0 && mx <= x1 && my >= y0 && my <= y1) return 0.0;
    double best = INFINITY;
    for (int k = 0; k < 2; k++) {
        const double ey = (k ? y1 : y0) - my;                  // horizontal edge: min over ex of A ex^2 + 2 B ex ey
        const double ex = fmin(x1 - mx, fmax(x0 - mx, -B * ey / A));
        best = fmin(best, A * ex * ex + 2 * B * ex * ey + C * ey * ey);
        const double fx = (k ? x1 : x0) - mx;                  // vertical edge
        const double fy = fmin(y1 - my, fmax(y0 - my, -B * fx / C));
        best = fmin(best, A * fx * fx + 2 * B * fx * fy + C * fy * fy);
    }
    return best;
}

static void check(Family& f, const float4& a, const float4& b, int tx, int ty) {
    const uint32_t m = block_mask16(a, b, tx, ty);
    const double A = a.z, B = a.w, C = b.x, bound = 2.0 * log(255.0 * (double)b.y);
    uint32_t need = 0, touch = 0, near = 0;
    int miss_px = 0;
    for (int py = 0; py < 16; py++)
        for (int px = 0; px < 16; px++) {
            const float dx = a.x - (float)(tx * 16 + px), dy = a.y - (float)(ty * 16 + py);
            const float power = -0.5f * (a.z * dx * dx + b.x * dy * dy) - a.w * dx * dy;
            if (power <= 0.0f && fminf(0.99f, b.y * expf(power)) >= 1.0f / 255.0f) {
                need |= 1u << bit_of(px >> 2, py >> 2);
                if (!(m >> bit_of(px >> 2, py >> 2) & 1u)) miss_px++;
            }
            const double ex = tx * 16 + px - (double)a.x, ey = ty * 16 + py - (double)a.y;
            const double q = A * ex * ex + 2 * B * ex * ey + C * ey * ey, mag = fabs(A) * ex * ex + 2 * fabs(B * ex * ey) + fabs(C) * ey * ey;
            if (q <= bound + 16.0 * ldexp(mag, -24) + 3e-5) near |= 1u << bit_of(px >> 2, py >> 2);
        }
    if (bound >= 0 && A * C - B * B > 0 && A > 0)
        for (int by = 0; by < 4; by++)
            for (int bx = 0; bx < 4; bx++) {
                const double x0 = tx * 16 + 4 * bx, y0 = ty * 16 + 4 * by;
                if (rect_min_q(A, B, C, a.x, a.y, x0, x0 + 3, y0, y0 + 3) <= bound) touch |= 1u << bit_of(bx, by);
            }
    f.entries++;
    if (need & ~m) {
        if (f.missed < 5)
            printf("MISSED [%s] mean (%.9g, %.9g) conic (%.9g, %.9g, %.9g) o %.9g tile (%d, %d) need %04x mask %04x\n", f.name,
                   a.x, a.y, a.z, a.w, b.x, b.y, tx, ty, need, m);
        f.missed++;
        f.missed_px += miss_px;
    }
    f.marked += __builtin_popcount(m); f.needed += __builtin_popcount(need);
    f.marked_untouched += __builtin_popcount(m & ~touch & ~need & ~near);
}

// conic of the covariance R diag(s1^2, s2^2) R^T + 0.3 I (the dilation of K1), R the rotation by th
static void conic(double s1, double s2, double th, float4& a, float4& b) {
    const double c = cos(th), s = sin(th);
    const double cxx = c * c * s1 * s1 + s * s * s2 * s2 + 0.3, cxy = c * s * (s1 * s1 - s2 * s2), cyy = s * s * s1 * s1 + c * c * s2 * s2 + 0.3;
    const double det = cxx * cyy - cxy * cxy;
    a.z = (float)(cyy / det); a.w = (float)(-cxy / det); b.x = (float)(cxx / det);
    b.z = 1.0f; b.w = 0.0f;
}

int main() {
    Family fam[4];
    fam[0].name = "random"; fam[1].name = "needle"; fam[2].name = "1/255"; fam[3].name = "degenerate"; fam[3].tight = false;
    srand(7);
    for (int it = 0; it < 200000; it++) {
        float4 a, b;
        conic(0.3 * pow(40.0, urand()), 0.3 * pow(40.0, urand()), urand() * 3.14159265, a, b);
        b.y = (float)(it % 7 == 0 ? 1.6 * urand() : pow(10.0, -2.6 * urand()));        // opacity (may exceed 1 in hierarchy mode)
        const int tx = rand() % 120, ty = rand() % 68;
        a.x = (float)(tx * 16 + (urand() * 60.0 - 22.0)); a.y = (float)(ty * 16 + (urand() * 60.0 - 22.0));
        check(fam[0], a, b, tx, ty);
    }
    for (int it = 0; it < 100; it++) {
        float4 a, b;
        const double L = 50.0 + 550.0 * urand(), th = urand() * 3.14159265;
        conic(L, 0.0, th, a, b);
        b.y = (float)(0.02 + 0.98 * urand());
        a.x = (float)(960.0 + 2000.0 * urand()); a.y = (float)(540.0 + 2000.0 * urand());
        // the ellipse's bounding box: |ex| <= sqrt(bound cxx), |ey| <= sqrt(bound cyy)
        const double det = (double)a.z * b.x - (double)a.w * a.w, bound = 2.0 * log(255.0 * b.y) * 1.01 + 0.01;
        const double hx = sqrt(bound * b.x / det), hy = sqrt(bound * a.z / det);
        for (int ty = (int)floor((a.y - hy) / 16) - 1; ty <= (int)floor((a.y + hy) / 16) + 1; ty++)
            for (int tx = (int)floor((a.x - hx) / 16) - 1; tx <= (int)floor((a.x + hx) / 16) + 1; tx++) {
                if (tx < 0 || ty < 0) continue;
                check(fam[1], a, b, tx, ty);
            }
    }
    const float o0 = 1.0f / 255.0f, ops[3] = {nextafterf(o0, 0.0f), o0, nextafterf(o0, 1.0f)};
    for (int it = 0; it < 3000; it++) {
        float4 a, b;
        conic(0.3 * pow(40.0, urand()), 0.3 * pow(40.0, urand()), urand() * 3.14159265, a, b);
        b.y = ops[it % 3];
        const int tx = 1 + rand() % 118, ty = 1 + rand() % 66, kind = (it / 3) % 4;
        // pixel centre inside the tile, the tile's corner, a point of its left edge, a point of its top edge
        float x = (float)(tx * 16 + (kind == 1 || kind == 2 ? 0 : rand() % 16));
        float y = (float)(ty * 16 + (kind == 1 || kind == 3 ? 0 : rand() % 16));
        const int ulps = (it / 12) % 3;                  // exact, 1 ulp below, 1 ulp above
        if (ulps) { x = nextafterf(x, ulps == 1 ? 0.0f : 1e9f); y = nextafterf(y, (it / 36) % 2 ? 0.0f : 1e9f); }
        a.x = x; a.y = y;
        for (int dy = -1; dy <= 1; dy++)
            for (int dx = -1; dx <= 1; dx++) check(fam[2], a, b, tx + dx, ty + dy);
    }
    const float inf = INFINITY, nan = NAN;
    for (int it = 0; it < 4000; it++) {
        float4 a, b;
        conic(0.3 * pow(40.0, urand()), 0.3 * pow(40.0, urand()), urand() * 3.14159265, a, b);
        const int kind = it % 8, tx = rand() % 120, ty = rand() % 68;
        a.x = (float)(tx * 16 + (urand() * 40.0 - 12.0)); a.y = (float)(ty * 16 + (urand() * 40.0 - 12.0));
        b.y = (float)(it % 3 == 0 ? o0 : 0.01 + urand());
        if (kind == 0) a.w = copysignf(sqrtf(a.z * b.x) * (float)(1.0 + 3.0 * urand()), urand() < 0.5f ? -1.0f : 1.0f);  // indefinite
        if (kind == 1) { a.z = -a.z; b.x = -b.x; }                                   // negative definite
        if (kind == 2) { a.z = 0.25f; a.w = 0.5f; b.x = 1.0f; }                     // det exactly 0
        if (kind == 3) (urand() < 0.5 ? a.x : a.y) = (it / 8) % 2 ? nan : -inf;      // non-finite mean
        if (kind == 4) (it % 3 == 1 ? a.z : it % 3 == 2 ? a.w : b.x) = (it / 8) % 2 ? nan : inf;   // non-finite conic
        if (kind == 5) b.y = nextafterf(o0, 0.0f);                                   // indefinite, opacity never taken
        if (kind == 5) a.w = 2.0f * sqrtf(a.z * b.x);
        if (kind == 6) b.y = nan;                                                     // NaN opacity, regular conic
        if (kind == 7) { b.y = nan; a.w = 2.0f * sqrtf(a.z * b.x); }                 // NaN opacity, indefinite conic
        const uint32_t m = block_mask16(a, b, tx, ty);
        const uint32_t want = (kind >= 5) ? 0u : 0xFFFFu;
        if (m != want) {
            if (fam[3].wrong < 5) printf("WRONG [degenerate] kind %d mean (%.9g, %.9g) conic (%.9g, %.9g, %.9g) o %.9g mask %04x\n",
                                         kind, a.x, a.y, a.z, a.w, b.x, b.y, m);
            fam[3].wrong++;
        }
        if (kind < 6) check(fam[3], a, b, tx, ty);      // a NaN opacity the blend's fminf would take: the mask hides it
    }
    int rc = 0;
    for (const Family& f : fam) {
        printf("[%s] entries %ld missed %ld (%ld pixels) marked %ld needed %ld marked_untouched %ld wrong %ld\n", f.name,
               f.entries, f.missed, f.missed_px, f.marked, f.needed, f.marked_untouched, f.wrong);
        if (f.missed || f.wrong) rc = 1;
        else if (f.tight && (double)f.marked_untouched > 0.02 * (double)f.marked) { printf("[%s] mask not tight\n", f.name); rc = rc ? rc : 2; }
    }
    return rc;
}
