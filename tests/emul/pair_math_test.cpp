// CPU check of the blend kernels' per-entry arithmetic (csrc/pair_math.cuh compiled for the host with
// -DH3_PAIR_HOST_EMU) against a straightforward double-precision restatement of the published per-pixel
// recurrences: front-to-back blend, classic deferred back-to-front gradient.  Test infrastructure only.
#define H3_PAIR_HOST_EMU
#include "../../hierarchical-3d-gaussians_b200/csrc/pair_math.cuh"
#include <stdio.h>
#include <stdlib.h>
#include <vector>
using namespace h3dgs;

struct Entry { float4 a, b, c; };

static int g_flips = 0;
static double urand() { return (double)rand() / RAND_MAX; }

// ---- reference: one pixel, double precision ---------------------------------------------------------
struct RefOut { double C[4], T; int last; std::vector<double> v; };   // v: [n][10]
static void ref_alpha(const Entry& e, double px, double py, bool hier, double& power, double& G, double& alpha, double& dadb) {
    const double dx = e.a.x - px, dy = e.a.y - py;
    power = -0.5 * (e.a.z * dx * dx + e.b.x * dy * dy) - e.a.w * dx * dy;
    G = exp(power);
    double a = fmin(0.99, e.b.y * G);
    alpha = a; dadb = 1.0;
    union { float f; uint32_t u; } kb; kb.f = e.b.w;
    const uint32_t k = kb.u & 0xFFFFu;              // the sorted copy's 16-bit field
    const double t = e.b.z;
    if (hier && k > 1 && t < 1.0) {
        alpha = t * a + (1 - t) * (1 - pow(1 - a, 1.0 / k));
        dadb = t + (1 - t) * (1.0 / k) * pow(1 - a, 1.0 / k - 1);
    }
}
static RefOut ref_pixel(const std::vector<Entry>& es, double px, double py, bool hier, const double g[4], const double bg[3]) {
    RefOut o; o.T = 1; o.last = 0; for (double& c : o.C) c = 0;
    const int n = (int)es.size();
    for (int i = 0; i < n; i++) {
        double pw, G, al, dd; ref_alpha(es[i], px, py, hier, pw, G, al, dd);
        if (pw > 0 || al < 1.0 / 255) continue;
        const double tT = o.T * (1 - al);
        if (tT < 1e-4) break;
        const double w = al * o.T;
        o.C[0] += es[i].c.x * w; o.C[1] += es[i].c.y * w; o.C[2] += es[i].c.z * w; o.C[3] += es[i].c.w * w;
        o.T = tT; o.last = i + 1;
    }
    o.v.assign((size_t)n * 10, 0.0);
    double T = o.T, acc[4] = {0, 0, 0, 0}, la = 0, lc[4] = {0, 0, 0, 0};
    const double bgd = bg[0] * g[0] + bg[1] * g[1] + bg[2] * g[2];
    for (int i = o.last - 1; i >= 0; i--) {
        double pw, G, al, dd; ref_alpha(es[i], px, py, hier, pw, G, al, dd);
        if (pw > 0 || al < 1.0 / 255) continue;
        T = T / (1 - al);
        const double c[4] = {es[i].c.x, es[i].c.y, es[i].c.z, es[i].c.w};
        double dL_dalpha = 0;
        double* v = &o.v[(size_t)i * 10];
        for (int ch = 0; ch < 4; ch++) {
            acc[ch] = la * lc[ch] + (1 - la) * acc[ch];
            lc[ch] = c[ch];
            dL_dalpha += (c[ch] - acc[ch]) * g[ch];
            v[6 + ch] = al * T * g[ch];
        }
        dL_dalpha *= T;
        la = al;
        dL_dalpha += (-o.T / (1 - al)) * bgd;
        const double dL_dab = dL_dalpha * dd;              // the 0.99 cap is not differentiated
        const double dL_dG = es[i].b.y * dL_dab;
        const double dx = es[i].a.x - px, dy = es[i].a.y - py;
        const double gdx = G * dx, gdy = G * dy;
        v[0] = dL_dG * (-gdx * es[i].a.z - gdy * es[i].a.w);
        v[1] = dL_dG * (-gdy * es[i].b.x - gdx * es[i].a.w);
        v[2] = gdx * dx * dL_dG; v[3] = gdx * dy * dL_dG; v[4] = gdy * dy * dL_dG;
        v[5] = G * dL_dab;
    }
    return o;
}

// ---- the kernels' arithmetic on the pair (pair_math.cuh), sequenced as the kernels do ----------------
template <bool HIER>
static int run(int trial, bool verbose) {
    srand(1234 + trial);
    const int n = 40 + rand() % 300;
    const int px = rand() % 64, py0 = 2 * (rand() % 32);
    std::vector<Entry> es(n);
    for (auto& e : es) {
        const double sx = 1.5 + 6 * urand(), sy = 1.5 + 6 * urand(), rho = 1.6 * urand() - 0.8;
        const double det = sx * sx * sy * sy * (1 - rho * rho);
        e.a.x = (float)(px + 14 * (urand() - 0.5)); e.a.y = (float)(py0 + 0.5 + 14 * (urand() - 0.5));
        e.a.z = (float)(sy * sy / det); e.a.w = (float)(-rho * sx * sy / det); e.b.x = (float)(sx * sx / det);
        e.b.y = (float)(urand() < 0.15 ? 1.2 * urand() : 0.05 + 0.5 * urand());     // opacity may exceed 1 (hierarchy)
        e.b.z = (float)(urand() < 0.3 ? 1.0 : urand());
        union { float f; uint32_t u; } kb;
        // k: mostly small families, also the wide counts up to the field's 65535 (1 - (1-a)^(1/k) then sits at the 1/255 cut
        // for a >= 1/16); the reach mask in bits 16..31 must not leak into the count
        const int kd = rand() % 8;
        const uint32_t kk = kd < 5 ? 1 + rand() % 4 : kd == 5 ? 5 + rand() % 60 : kd == 6 ? 60 + rand() % 4000 : 4000 + rand() % 61536;
        kb.u = kk | ((uint32_t)(rand() & 0xFFFF) << 16);
        e.b.w = kb.f;
        e.c.x = (float)urand(); e.c.y = (float)urand(); e.c.z = (float)urand(); e.c.w = (float)(0.05 + urand());
    }
    double g[2][4], bg[3] = {0.3, 0.5, 0.2};
    for (int p = 0; p < 2; p++) for (int ch = 0; ch < 4; ch++) g[p][ch] = urand() - 0.5;
    const RefOut r0 = ref_pixel(es, px, py0, HIER, g[0], bg), r1 = ref_pixel(es, px, py0 + 1, HIER, g[1], bg);

    // forward, as render_forward.cu
    const float fpx = (float)px;
    const f2 nfpy = pk(-(float)py0, -(float)(py0 + 1));
    f2 T = bc(1.0f);
    float Ca[4] = {0, 0, 0, 0}, Cb[4] = {0, 0, 0, 0};
    bool done0 = false, done1 = false;
    int last0 = 0, last1 = 0;
    for (int j = 0; j < n; j++) {
        const Entry& e = es[j];
        union { float f; uint32_t u; } kb; kb.f = e.b.w;
        f2 d, G, al, unused;
        const f2 pw = pair_power(e.a, e.b, e.a.x - fpx, nfpy, d);
        pair_gauss(pw, e.b.y, G, al);
        pair_hier_alpha<HIER, false>(al, e.b.z, kb.u & kSortedKidsMask, al, unused);
        bool v0, v1;
        const f2 w = pair_blend(pw, al, T, done0, done1, v0, v1);
        const float cc[4] = {e.c.x, e.c.y, e.c.z, e.c.w};
        for (int ch = 0; ch < 4; ch++) upk(fma2(bc(cc[ch]), w, pk(Ca[ch], Cb[ch])), Ca[ch], Cb[ch]);
        if (v0) last0 = j + 1;
        if (v1) last1 = j + 1;
    }
    int bad = 0;
    auto close = [&](double x, double y, double scale, double tol, const char* what, int idx) {
        if (fabs(x - y) > tol * scale) { if (verbose || bad < 5) printf("  trial %d %s[%d]: %g vs %g\n", trial, what, idx, x, y); bad++; }
    };
    // a decision that sits within fp32 rounding of its threshold (alpha = 1/255, T = 1e-4) may flip
    // against double precision: counted separately, the trial is then not comparable
    if (last0 != r0.last || last1 != r1.last) { g_flips++; return 0; }
    close(lo(T), r0.T, 1, 2e-6, "T0", 0); close(hi(T), r1.T, 1, 2e-6, "T1", 0);
    for (int ch = 0; ch < 4; ch++) { close(Ca[ch], r0.C[ch], 1, 5e-6, "C0", ch); close(Cb[ch], r1.C[ch], 1, 5e-6, "C1", ch); }

    // backward, as render_backward.cu (final T and last contributor come from the forward)
    const f2 Tf = T;
    PairState ps = {Tf, bc(0.f)};
    const f2 g0 = pk((float)g[0][0], (float)g[1][0]), g1 = pk((float)g[0][1], (float)g[1][1]),
             g2 = pk((float)g[0][2], (float)g[1][2]), gd = pk((float)g[0][3], (float)g[1][3]);
    const f2 neg_bgd = pk(-(float)(bg[0] * g[0][0] + bg[1] * g[0][1] + bg[2] * g[0][2]),
                          -(float)(bg[0] * g[1][0] + bg[1] * g[1][1] + bg[2] * g[1][2]));
    double scale[10] = {0};
    for (int i = 0; i < n; i++) for (int k = 0; k < 10; k++) scale[k] = fmax(scale[k], fabs(r0.v[(size_t)i * 10 + k] + r1.v[(size_t)i * 10 + k]));
    for (int e = n - 1; e >= 0; e--) {
        const Entry& en = es[e];
        union { float f; uint32_t u; } kb; kb.f = en.b.w;
        const float dx = en.a.x - fpx;
        f2 d, G, al, dadb;
        const f2 pw = pair_power(en.a, en.b, dx, nfpy, d);
        pair_gauss(pw, en.b.y, G, al);
        pair_hier_alpha<HIER, true>(al, en.b.z, kb.u & kSortedKidsMask, al, dadb);
        const bool v0 = e < last0 && lo(pw) <= 0.0f && lo(al) >= kAlphaSkip;
        const bool v1 = e < last1 && hi(pw) <= 0.0f && hi(al) >= kAlphaSkip;
        float v[10] = {0};
        if (v0 || v1) {
            G = sel2(v0, v1, G, bc(0.f));
            al = sel2(v0, v1, al, bc(0.f));
            f2 cg = fma2(bc(en.c.z), g2, fma2(bc(en.c.y), g1, mul2(bc(en.c.x), g0)));
            cg = fma2(bc(en.c.w), gd, cg);
            pair_grad<HIER, true>(en.a, en.b, dx, d, G, al, dadb, cg, Tf, neg_bgd, g0, g1, g2, gd, ps, v);
        }
        for (int k = 0; k < 10; k++)
            // fp32 recovers T by repeated division (up to ~300 steps here): ~n eps of drift is inherent
            close(v[k], r0.v[(size_t)e * 10 + k] + r1.v[(size_t)e * 10 + k], scale[k] + 1e-30, 1e-4, "v", e * 10 + k);
    }
    return bad;
}

int main(int argc, char** argv) {
    const int trials = argc > 1 ? atoi(argv[1]) : 200;
    int bad = 0;
    for (int t = 0; t < trials; t++) { bad += run<false>(t, false); bad += run<true>(t, false); }
    const bool fail = bad != 0 || g_flips > trials / 50;
    printf("%s: %d mismatches, %d threshold flips in %d trials x 2 variants\n", fail ? "FAIL" : "ok", bad, g_flips, trials);
    return fail ? 1 : 0;
}
