// pair_math.cuh -- the per-entry arithmetic of the blend kernels for the TWO pixels a thread owns,
// on FP32 pairs {lo = pixel 0, hi = pixel 1}.
//
// Device build (included from common.cuh): sm_90 has no packed FP32 instructions, so a pair is two
// registers and every operation is two FFMA / FMUL / FADD.  The entry's record, its dx terms and the
// survivor loop are still shared by the two pixels.  Each lane is an IEEE fma/mul/add.rn; only the gradient
// terms of pair_grad, which decide nothing, are plain float expressions that nvcc may contract.
//
// Host build (-DH3_PAIR_HOST_EMU, plain g++): the same functions over a two-float struct, so that the
// formulas -- exponent, capped alpha, hierarchy weight, the back-to-front gradient recurrence -- can be
// checked on a CPU against a straightforward double-precision restatement (tests/emul/).
#pragma once

#ifdef H3_PAIR_HOST_EMU
#include <math.h>
#include <stdint.h>
#define H3_PM_FN static inline
namespace h3dgs {
#ifndef H3_SIMT_EMU               /* stand-alone host build (tests/emul/pair_math_test.cpp); the SIMT emulator has common.cuh */
struct float4 { float x, y, z, w; };
constexpr float kAlphaCap = 0.99f;
constexpr float kAlphaSkip = 1.0f / 255.0f;
constexpr float kTStop = 0.0001f;
constexpr uint32_t kSortedKidsMask = 0xFFFFu;
#endif
struct f2 { float lo, hi; };
H3_PM_FN f2 pk(float lo, float hi) { return f2{lo, hi}; }
H3_PM_FN void upk(f2 v, float& lo, float& hi) { lo = v.lo; hi = v.hi; }
H3_PM_FN f2 fma2(f2 a, f2 b, f2 c) { return f2{fmaf(a.lo, b.lo, c.lo), fmaf(a.hi, b.hi, c.hi)}; }
H3_PM_FN f2 mul2(f2 a, f2 b) { return f2{a.lo * b.lo, a.hi * b.hi}; }
H3_PM_FN f2 add2(f2 a, f2 b) { return f2{a.lo + b.lo, a.hi + b.hi}; }
H3_PM_FN f2 sub2(f2 a, f2 b) { return f2{a.lo - b.lo, a.hi - b.hi}; }
H3_PM_FN float fast_exp2(float x) { return exp2f(x); }
H3_PM_FN float fast_log2(float x) { return log2f(x); }
H3_PM_FN float rcp_approx(float x) { return 1.0f / x; }
H3_PM_FN float rsq_approx(float x) { return 1.0f / sqrtf(x); }
#else
#define H3_PM_FN __device__ __forceinline__
namespace h3dgs {
// Two scalar registers per pair; the explicit _rn intrinsics keep nvcc from contracting or reassociating
// across the lanes, so each lane is exactly the fma/mul/add/sub.rn the formulas are written in.
struct f2 { float lo, hi; };
H3_PM_FN f2 pk(float lo, float hi) { return f2{lo, hi}; }
H3_PM_FN void upk(f2 v, float& lo, float& hi) { lo = v.lo; hi = v.hi; }
H3_PM_FN f2 fma2(f2 a, f2 b, f2 c) { return f2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)}; }
H3_PM_FN f2 mul2(f2 a, f2 b) { return f2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
H3_PM_FN f2 add2(f2 a, f2 b) { return f2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
H3_PM_FN f2 sub2(f2 a, f2 b) { return f2{__fsub_rn(a.lo, b.lo), __fsub_rn(a.hi, b.hi)}; }
// 2^x as MUFU.EX2 (ftz: results below 2^-126 flush to 0, far below the 1/255 alpha cut)
H3_PM_FN float fast_exp2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// log2(x) for normal x: MUFU.LG2 without the denormal pre-scaling of __log2f
H3_PM_FN float fast_log2(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
H3_PM_FN float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
H3_PM_FN float rsq_approx(float x) { float y; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
#endif

H3_PM_FN f2 bc(float x) { return pk(x, x); }
H3_PM_FN float lo(f2 v) { float a, b; upk(v, a, b); return a; }
H3_PM_FN float hi(f2 v) { float a, b; upk(v, a, b); return b; }
H3_PM_FN float hsum(f2 v) { float a, b; upk(v, a, b); return a + b; }
H3_PM_FN f2 sel2(bool p0, bool p1, f2 x, f2 y) {      // per-lane p ? x : y
    float x0, x1, y0, y1; upk(x, x0, x1); upk(y, y0, y1);
    return pk(p0 ? x0 : y0, p1 ? x1 : y1);
}
H3_PM_FN f2 ex2_2(f2 v) { float a, b; upk(v, a, b); return pk(fast_exp2(a), fast_exp2(b)); }
// 1/x for x in [0.01, 2^20]: MUFU.RCP + one Newton step (~1 ulp; exactly 1 for x = 1)
H3_PM_FN float fast_rcp(float x) { const float r = rcp_approx(x); return r * (2.0f - x * r); }
H3_PM_FN f2 rcp2(f2 x) {
    float x0, x1; upk(x, x0, x1);
    const f2 r = pk(rcp_approx(x0), rcp_approx(x1));
    return mul2(r, fma2(pk(-x0, -x1), r, bc(2.0f)));
}

// Gaussian exponent of one entry at the thread's two pixels, shared by forward and backward so that
// both take identical decisions:  power_i = -1/2 (cx dx^2 + cz dy_i^2) - cy dx dy_i, evaluated as
// (C d_i + B) d_i + A with A = (cx dx)(-dx/2), B = -cy dx, C = -cz/2.
// a = {x, y, cx, cy}, bb.x = cz;  nfpy = {-py0, -py1};  d = {a.y - py0, a.y - py1} is returned for the gradients.
H3_PM_FN f2 pair_power(const float4& a, const float4& bb, float dx, f2 nfpy, f2& d) {
    d = add2(bc(a.y), nfpy);
    const float A = (a.z * dx) * (dx * -0.5f), B = -a.w * dx, C = -0.5f * bb.x;
    return fma2(fma2(bc(C), d, bc(B)), d, bc(A));
}
// G = exp(power) and the capped base alpha min(0.99, opacity G) of the pair
H3_PM_FN void pair_gauss(f2 power, float opacity, f2& G, f2& abase) {
    G = ex2_2(mul2(power, bc(1.4426950408889634f)));
    float a0, a1; upk(mul2(bc(opacity), G), a0, a1);
    abase = pk(fminf(kAlphaCap, a0), fminf(kAlphaCap, a1));
}
// Hierarchy transition weight on the per-pixel blending weight (UNPINNED semantics, DESIGN.md
// "hierarchy alpha"): a' = t a + (1-t)(1 - (1-a)^(1/k)); identity for k <= 1 or t >= 1.  k and t are
// per-entry, so the early out is warp-uniform.  GRAD = false drops the derivative da'/da.
// 1 - (1-a)^(1/k) = -expm1(log1p(-a)/k).  Near the 1/255 skip threshold a is small and the direct form
// cancels catastrophically (abs error ~2e-7 on a value ~4e-3 moves the skip decision for 100x more
// pixels than in flat mode), so a small result uses the series of expm1 (relative error < 2e-7 from the series, plus
// MUFU.LG2's ~2^-22 absolute error on log2(1-a) for a >= 1/16); a large one goes through MUFU.EX2.
template <bool HIER, bool GRAD>
H3_PM_FN void pair_hier_alpha(f2 a, float t, uint32_t k /* num_node_kids */, f2& alpha, f2& dadb) {
    alpha = a; dadb = bc(1.0f);
    if (!HIER) return;
    if (k <= 1u || t >= 1.0f) return;
    const float u = 1.0f - t;
    float a0, a1; upk(a, a0, a1);
    float o0, o1; upk(sub2(bc(1.0f), a), o0, o1);             // 1 - a is in [0.01, 1]
    if (k == 2u) {
        // Two siblings -- every interior node of a binary hierarchy (the reference's BVH builder, our synthetic trees):
        // 1 - sqrt(1-a) in closed form.  Small a (the ones that sit at the 1/255 threshold) use the series
        // a/2 + a^2/8 + a^3/16 + 5a^4/128 + 7a^5/256 (relative error < 5e-8 below 1/16), larger a the direct
        // difference; one MUFU.RSQ per pixel serves the value (sqrt = x rsqrt x) and the derivative
        // da'/da = t + (1-t) / (2 sqrt(1-a)).
        const f2 r = pk(rsq_approx(o0), rsq_approx(o1));
        const f2 s = mul2(pk(o0, o1), r);
        f2 S = fma2(a, bc(0.02734375f), bc(0.0390625f));
        S = fma2(a, S, bc(0.0625f));
        S = fma2(a, S, bc(0.125f));
        S = fma2(a, S, bc(0.5f));
        const f2 omr = sel2(a0 < 0.0625f, a1 < 0.0625f, mul2(a, S), sub2(bc(1.0f), s));
        alpha = fma2(bc(u), omr, mul2(bc(t), a));
        if (GRAD) dadb = fma2(bc(0.5f * u), r, bc(t));
        return;
    }
    const float ik = fast_rcp((float)k);
    const f2 l2 = pk(fast_log2(o0), fast_log2(o1));
    // yn = -log1p(-a)/k >= 0: for small a the series -log1p(-a) = a (1 + a/2 + a^2/3 + a^3/4 + a^4/5), else -ln2 lg2(1-a)
    f2 L = fma2(a, bc(0.2f), bc(0.25f));
    L = fma2(a, L, bc(0.33333334f));
    L = fma2(a, L, bc(0.5f));
    L = fma2(a, L, bc(1.0f));
    const f2 yn = sel2(a0 < 0.0625f, a1 < 0.0625f, mul2(mul2(a, L), bc(ik)), mul2(l2, bc(-0.6931472f * ik)));
    // -expm1(-yn) = yn (1 - yn/2 + yn^2/6 - yn^3/24).  The switch is on yn, not on a: for large k a moderate a gives a
    // small 1 - (1-a)^(1/k), where 1 - MUFU.EX2 would cancel (abs error ~2^-22 on a value near the 1/255 cut)
    f2 S = fma2(yn, bc(-0.041666668f), bc(0.16666667f));
    S = fma2(yn, S, bc(-0.5f));
    S = fma2(yn, S, bc(1.0f));
    const f2 omr_series = mul2(yn, S);
    const f2 omr_mufu = sub2(bc(1.0f), ex2_2(mul2(l2, bc(ik))));
    float y0, y1; upk(yn, y0, y1);
    const f2 omr = sel2(y0 < 0.0625f, y1 < 0.0625f, omr_series, omr_mufu);
    alpha = fma2(bc(u), omr, mul2(bc(t), a));
    if (GRAD) dadb = fma2(bc(u * ik), ex2_2(mul2(l2, bc(ik - 1.0f))), bc(t));
}

// ---- forward: one entry at the pair -------------------------------------------------------------
// T: transmittance in front of the entry.  Returns the blend weights w = alpha T (0 for a pixel that
// does not take the entry), updates T, and reports per pixel whether it took the entry (v) and
// whether it terminated on it (done: T (1 - alpha) < 1e-4; the entry is then NOT blended).
H3_PM_FN f2 pair_blend(f2 pw, f2 al, f2& T, bool& done0, bool& done1, bool& v0, bool& v1) {
    const f2 tT = mul2(T, sub2(bc(1.0f), al));
    float pw0, pw1, al0, al1, tT0, tT1;
    upk(pw, pw0, pw1); upk(al, al0, al1); upk(tT, tT0, tT1);
    v0 = !done0 && pw0 <= 0.0f && al0 >= kAlphaSkip;
    v1 = !done1 && pw1 <= 0.0f && al1 >= kAlphaSkip;
    if (v0 && tT0 < kTStop) { done0 = true; v0 = false; }
    if (v1 && tT1 < kTStop) { done1 = true; v1 = false; }
    const f2 w = sel2(v0, v1, mul2(al, T), bc(0.f));
    T = sel2(v0, v1, tT, T);
    return w;
}

// ---- backward: replay state and the gradient of one entry at the pair ------------------------------
// T = transmittance in front of the current entry, acc = (colour accumulated behind it) . dL/dC.
// The classic formulation defers the update of acc by one contributor (last_alpha, last_color); the
// equivalent immediate form  acc <- acc + alpha (c.g - acc),  T <- T / (1 - alpha)  is the identity for
// alpha = 0, so a pixel that does not take the entry needs no selects to keep its state.
struct PairState { f2 T, acc; };

// Contribution of entry (a, bb) at the thread's two pixels to the 10 per-Gaussian sums
// (accum row layout: 0,1 dmean2D | 2,3,4 dconic | 5 dopacity | 6,7,8 dcolor | 9 dinvdepth; the constant
// factors 0.5 W, 0.5 H, -0.5 are applied once per Gaussian in preprocess_backward).  G and alpha must be
// zero for a pixel that does not take the entry: every term below then is an exact zero (each carries
// a factor G or alpha, the other factors are finite) and its state is unchanged.
// cg = colour . dL/dC of the pair, neg_bg_dot = -(background . dL/dC), g0..gd = dL/dC channels.
// The gradient terms decide nothing, so they are free to contract (FFMA where a product feeds a sum).  dx is shared by the pair, so the five terms of the exponent's gradient need only the three moments
// S_k = sum_i d_i^k G_i dL/dab_i (k = 0, 1, 2) of the pair, with dL/dG = opacity dL/dab:
//   v0 = o (-cy S1 - cx dx S0), v1 = o (-cy dx S0 - cz S1), v2 = o dx^2 S0, v3 = o dx S1, v4 = o S2, v5 = S0.
// v[9] is written only with DEPTH.
template <bool HIER, bool DEPTH>
H3_PM_FN void pair_grad(const float4& a, const float4& bb, float dx, f2 d, f2 G, f2 alpha, f2 dadb, f2 cg, f2 T_final,
                        f2 neg_bg_dot, f2 g0, f2 g1, f2 g2, f2 gd, PairState& st, float (&v)[10])
{
    const f2 rcp = rcp2(sub2(bc(1.0f), alpha));            // one reciprocal serves T and the background term
    const f2 diff = sub2(cg, st.acc);
    // dL/dalpha = (T_final neg_bg_dot + T diff) / (1 - alpha); T_final neg_bg_dot is loop-invariant in the kernels
    const f2 dL_dalpha = mul2(fma2(st.T, diff, mul2(T_final, neg_bg_dot)), rcp);
    const f2 dL_dab = HIER ? mul2(dL_dalpha, dadb) : dL_dalpha;
    st.T = mul2(st.T, rcp);
    const f2 w = mul2(alpha, st.T);                        // d(pixel colour)/d(entry colour)
    st.acc = fma2(alpha, diff, st.acc);
    float p0, p1, d0, d1;
    upk(mul2(G, dL_dab), p0, p1);
    upk(d, d0, d1);
    const float dp0 = d0 * p0, dp1 = d1 * p1;
    const float S0 = p0 + p1, S1 = dp0 + dp1, S2 = fmaf(d0, dp0, d1 * dp1);
    const float oS0 = bb.y * S0, oS1 = bb.y * S1, dxoS0 = dx * oS0;
    v[0] = fmaf(-a.w, oS1, -a.z * dxoS0);
    v[1] = fmaf(-a.w, dxoS0, -bb.x * oS1);
    v[2] = dx * dxoS0;
    v[3] = dx * oS1;
    v[4] = bb.y * S2;
    v[5] = S0;
    float w0, w1;
    upk(w, w0, w1);
    v[6] = fmaf(w0, lo(g0), w1 * hi(g0)); v[7] = fmaf(w0, lo(g1), w1 * hi(g1)); v[8] = fmaf(w0, lo(g2), w1 * hi(g2));
    if (DEPTH) v[9] = fmaf(w0, lo(gd), w1 * hi(gd));
}

}  // namespace h3dgs
#undef H3_PM_FN
