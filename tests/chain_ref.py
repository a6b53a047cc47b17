"""Float64 restatement of the preprocess backward (K8 + K9a + K9b + K9c): the per-Gaussian chain rule that turns the
blend's [P][10] sums into every returned gradient, with a per-element error budget for the kernels' precision scheme.

Written from the published algorithm (the 3D Gaussian Splatting backward: computeCov2D / computeCov3D / SH backward),
include/h3dgs.h and DESIGN.md §7.  Inputs are the fp32 parameters, the camera, the cut (scatter mode), the [P][10] sums
and the forward's decisions: radii > 0, the SH clamp flags (record kbits 20-22) and the frustum clamp, which
`frustum_clamp_fp32` recomputes here in numpy float32 exactly as K1 evaluates it.  The reference takes those
decisions as given and never re-derives them in double.  Everything else is float64 on the fp32 inputs.

The published quirks, stated explicitly:
  - the gradient of the conic uses 1 / (denom^2 + 1e-7) in place of 1 / denom^2 (`eps`);
  - cov2D = J W Sigma W^T J^T + 0.3 I (the dilation); the conic is (c, -b, a) / denom;
  - tx/tz, ty/tz clamped to +-1.3 tan(fov); where K1 clamped, tx (ty) is a constant: no gradient to the view-space x
    (y), and none to z through the bound;
  - dL/dmeans2D = (S0 0.5 W, S1 0.5 H, 0) (the sums are per pixel, means2D is in NDC);
  - dL/dconic = (-S2 / 2, -S3, -S4 / 2): S3 is the sum for HALF the off-diagonal of the quadratic form;
  - the fused gather: x = t x[c] + (1 - t) x[p], with the parent's quaternion negated when the fp32 dot with the
    child's is negative; the gradients scatter t g to c and (1 - t) g (x the quaternion sign for rotations) to p, a parent
    accumulating over all of its children.

ERROR BUDGET.  Each value carries a running bound e of the error an fp32 evaluation of the same formula has, in units
of U = 2^-24 (class `E`), derived operation by operation:
  - inputs: the fp32 parameters, the camera matrices and the sums are exact (e = 0); constants that the kernels hold
    in fp32 (1.3, 0.3, 1e-7, the SH constants, fx = W / (2 tan)) carry one rounding of their value;
  - a + b: e_a + e_b + m, with m = m_a + m_b the sum of |terms| of the flat sum the addition belongs to: every partial
    sum, in whatever order the kernel associates the terms, is at most m, so each of its roundings is at most U m;
  - a b: e_a |b| + |a| e_b + U e_a e_b + |a b|;
  - a / b: (e_a + |a / b| e_b) / |b| + |a / b|, first order in U e_b / |b| (the denominators here are tz >= 0.2, |d| and
    denom^2 + 1e-7, far from their error);
  - sqrt(a): e_a / (2 sqrt a) + sqrt(a).
  So the budget of an output is kappa U m: m the magnitude of the terms of each operation on its paths and kappa the
  number of roundings, counted term by term by the operations themselves; no factor is fitted.  The kernels contract
  some pairs into FMAs (one rounding instead of two), which only lowers their error.  The magnitude chain a (the same
  formula on absolute values) is also carried; it is the scale of the float64 comparisons.  It is not the budget's m:
  with the camera 1000 units from the origin, tz = 10 carries |view . mean| ~ 1000 in its chain, and every product
  downstream would multiply that up instead of rounding relative to its own value.
The kernels evaluate the 2x2 screen covariance and the gradient of its inverse in fp64 (A V A^T + 0.3 I through
dL/d(a, b, c), csrc/cov_grad.cuh), from the fp32 A and Sigma.  That block adds no rounding of its own that matters; what
it passes on is the error of its fp32 inputs, which is bounded here by the block's exact sensitivity,
sum_x |d out / d x| e_x over the entries x of A and Sigma (computed by complex-step differentiation), plus one rounding
of each output to fp32.  Bounding it by magnitude chains instead would multiply the input errors by the condition
factor (|a c| + b^2) / |denom| even where the true sensitivity is small (a needle's screen covariance is nearly rank one
whatever the rounding of A), and would hide an fp32 evaluation of the block.
Scattered rows add (n - 1) U sum |contributions| for an n-term fp32 atomic sum in any order (scatter_terms, scatter_tol).
"""
import numpy as np

U = 2.0 ** -24
FOV_CLAMP, DILATION, W_EPS = 1.3, 0.3, 1e-7
C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435]


class E:
    """value v (float64); a: the magnitude chain (the formula on absolute values); m: the magnitude that bounds the
    partial sums of the flat sum v is the result of (|v| for any other operation); e: the error bound in units of U"""
    __slots__ = ("v", "a", "m", "e")

    def __init__(self, v, a=None, m=None, e=0.0):
        self.v = np.asarray(v, np.float64)
        self.a = np.abs(self.v) if a is None else a
        self.m = np.abs(self.v) if m is None else m
        self.e = e

    @staticmethod
    def const(v):
        """a constant the kernels hold in fp32: one rounding"""
        return E(v, e=abs(v))

    @staticmethod
    def _w(x):
        return x if isinstance(x, E) else E(x)

    def __add__(self, o):
        o = E._w(o)
        m = self.m + o.m
        return E(self.v + o.v, self.a + o.a, m, self.e + o.e + m)
    __radd__ = __add__

    def __sub__(self, o):
        return self + (-E._w(o))

    def __rsub__(self, o):
        return E._w(o) + (-self)

    def __neg__(self):
        return E(-self.v, self.a, self.m, self.e)

    def __mul__(self, o):
        o = E._w(o)
        v = self.v * o.v
        e = self.e * np.abs(o.v) + np.abs(self.v) * o.e + U * self.e * o.e + np.abs(v)
        return E(v, self.a * o.a, None, e)
    __rmul__ = __mul__

    def __truediv__(self, o):
        o = E._w(o)
        ab = np.abs(o.v)
        v = self.v / o.v
        return E(v, self.a / ab, None, (self.e + np.abs(v) * o.e) / ab + np.abs(v))

    def __rtruediv__(self, o):
        return E._w(o) / self

    def sqrt(self):
        r = np.sqrt(self.v)
        return E(r, np.sqrt(self.a), None, self.e / (2 * r) + r)

    def mask(self, keep):
        """multiplication by an exact 0 / 1"""
        k = np.asarray(keep, np.float64)
        return E(self.v * k, self.a * k, self.m * k, self.e * k)


def _sum(terms):
    out = terms[0]
    for t in terms[1:]:
        out = out + t
    return out


# ---- the forward's decisions, as K1 takes them ------------------------------------------------------------------------
def view_xyz_fp32(view, means):
    """K1's view-space mean: individually rounded fp32 products and sums, in the order (m0 x + m4 y) + m8 z + m12"""
    v = np.asarray(view, np.float32).reshape(16)
    p = np.asarray(means, np.float32)
    out = []
    for r in range(3):
        acc = v[r] * p[:, 0]
        acc = acc + v[4 + r] * p[:, 1]
        acc = acc + v[8 + r] * p[:, 2]
        out.append(acc + v[12 + r])
    return out


def frustum_clamp_fp32(view, means, tanx, tany):
    """K1's frustum-clamp decision per row: [P][2] bool (x, y clamped), and the fp32 ratios tx/tz, ty/tz"""
    with np.errstate(divide="ignore", invalid="ignore"):
        vx, vy, vz = view_xyz_fp32(view, means)
        rx, ry = vx / vz, vy / vz
        lx, ly = np.float32(1.3) * np.float32(tanx), np.float32(1.3) * np.float32(tany)
        return np.stack([(rx < -lx) | (rx > lx), (ry < -ly) | (ry > ly)], 1), rx, ry


def fma_ratio_fp32(view, means):
    """tx/tz, ty/tz as an FMA-contracted evaluation rounds them (the backward's, before it evaluated K1's order
    explicitly): each of tx, ty, tz a rounded product, two fused multiply-adds and a rounded add.  The fma is
    emulated in float64 (exact product; the sum then rounds once, rarely twice)."""
    v = np.asarray(view, np.float32).reshape(16).astype(np.float64)
    p = np.asarray(means, np.float32).astype(np.float64)
    f = lambda a: np.asarray(a, np.float64).astype(np.float32).astype(np.float64)
    out = []
    for r in range(3):
        acc = f(v[r] * p[:, 0])
        acc = f(v[4 + r] * p[:, 1] + acc)
        acc = f(v[8 + r] * p[:, 2] + acc)
        out.append(f(acc + v[12 + r]))
    with np.errstate(divide="ignore", invalid="ignore"):
        return f(out[0] / out[2]), f(out[1] / out[2])


def gather_fp32(means3D, scales, rotations, shs, ridx, pidx, ts):
    """the fused gather + parent lerp exactly as K1 evaluates it (fp32, t a + u b with u = 1 - t, each operation
    rounded; the parent quaternion negated when the fp32 dot ((qc.qp_0 + ...) left to right) is negative).
    -> dict of per-rendered-row fp32 arrays, plus c, p, t, u, lerp, qsign and the quaternion dot."""
    f32 = np.float32
    c = np.asarray(ridx, np.int64)
    p = np.asarray(pidx, np.int64)
    p = np.where(p < 0, c, p)
    t = np.asarray(ts, f32)[: c.size]
    u = f32(1.0) - t
    lerp = u != 0

    def lp(a):
        a = np.asarray(a, f32)
        ac, ap = a[c], a[p]
        sh = (-1,) + (1,) * (a.ndim - 1)
        tt, uu = t.reshape(sh), u.reshape(sh)
        return np.where(lerp.reshape(sh), tt * ac + uu * ap, ac)
    out = dict(c=c, p=p, t=t, u=u, lerp=lerp, means3D=lp(means3D))
    out["scales"] = lp(scales) if scales is not None else None
    out["shs"] = lp(shs) if shs is not None else None
    qsign = np.ones(c.size, f32)
    dot = None
    if rotations is not None:
        q = np.asarray(rotations, f32)
        qc, qp = q[c], q[p]
        dot = qc[:, 0] * qp[:, 0]
        for k in (1, 2, 3):
            dot = dot + qc[:, k] * qp[:, k]
        qsign = np.where(lerp & (dot < 0), f32(-1), f32(1))
        qps = qp * qsign[:, None]
        out["rotations"] = np.where(lerp[:, None], t[:, None] * qc + u[:, None] * qps, qc)
    else:
        out["rotations"] = None
    out["qsign"] = qsign
    out["dot"] = dot
    return out


# ---- the fp64 block ----------------------------------------------------------------------------------------------------
def _block(A, V6, dc, eps):
    """(AV [2][3], dL/da, dL/db, dL/dc) from A [2][3], Sigma (6 unique) and dL/dconic as the published formulas write
    them (`dc` holds dL/dconic with the off-diagonal entry halved, as the published backward takes it)"""
    V = [[V6[0], V6[1], V6[2]], [V6[1], V6[3], V6[4]], [V6[2], V6[4], V6[5]]]
    AV = [[A[r][0] * V[0][c] + A[r][1] * V[1][c] + A[r][2] * V[2][c] for c in range(3)] for r in range(2)]
    a = AV[0][0] * A[0][0] + AV[0][1] * A[0][1] + AV[0][2] * A[0][2] + DILATION
    b = AV[0][0] * A[1][0] + AV[0][1] * A[1][1] + AV[0][2] * A[1][2]
    c = AV[1][0] * A[1][0] + AV[1][1] * A[1][1] + AV[1][2] * A[1][2] + DILATION
    den = a * c - b * b
    inv2 = 1.0 / (den * den + eps)
    x, y, z = dc
    da = inv2 * (-c * c * x + 2 * b * c * y + (den - a * c) * z)
    dcc = inv2 * (-a * a * z + 2 * a * b * y + (den - a * c) * x)
    db = inv2 * 2 * (b * c * x - (den + 2 * b * b) * y + a * b * z)
    return [AV[0][0], AV[0][1], AV[0][2], AV[1][0], AV[1][1], AV[1][2], da, db, dcc]


def _block_e(A, V6, dc, eps):
    """the block on E values: exact float64 results; error = exact sensitivity to the fp32 inputs' errors + one rounding"""
    ins = [A[0][0], A[0][1], A[0][2], A[1][0], A[1][1], A[1][2]] + list(V6)
    vals = [x.v for x in ins]
    dcv = [d.v for d in dc]
    unpack = lambda xs: ([xs[0:3], xs[3:6]], xs[6:12])
    outs = _block(*unpack(vals), dcv, eps)
    err = [np.zeros_like(o) for o in outs]
    h = 1e-60
    for j, x in enumerate(ins):
        cv = [v.astype(np.complex128) for v in vals]
        cv[j] = cv[j] + 1j * h
        d = _block(*unpack(cv), [v.astype(np.complex128) for v in dcv], eps)
        for k in range(len(outs)):
            err[k] = err[k] + np.abs(d[k].imag / h) * x.e
    return [E(o, None, None, er + np.abs(o)) for o, er in zip(outs, err)]


# ---- SH basis and its derivatives by the (unnormalised) direction -------------------------------------------------------
def _sh_basis(deg, x, y, z):
    """-> list of (B, dB/dx, dB/dy, dB/dz) per coefficient (None for an identically zero derivative), E values"""
    k = E.const
    out = [(E(np.full(x.v.shape, C0), e=C0), None, None, None)]
    if deg > 0:
        out += [(-k(C1) * y, None, -k(C1), None), (k(C1) * z, None, None, k(C1)), (-k(C1) * x, -k(C1), None, None)]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        c = [k(v) for v in C2]
        out += [(c[0] * xy, c[0] * y, c[0] * x, None),
                (c[1] * yz, None, c[1] * z, c[1] * y),
                (c[2] * (2 * zz - xx - yy), c[2] * -2 * x, c[2] * -2 * y, c[2] * 4 * z),
                (c[3] * xz, c[3] * z, None, c[3] * x),
                (c[4] * (xx - yy), c[4] * 2 * x, c[4] * -2 * y, None)]
        if deg > 2:
            d = [k(v) for v in C3]
            out += [(d[0] * y * (3 * xx - yy), d[0] * 6 * xy, d[0] * (3 * xx - 3 * yy), None),
                    (d[1] * xy * z, d[1] * yz, d[1] * xz, d[1] * xy),
                    (d[2] * y * (4 * zz - xx - yy), d[2] * -2 * xy, d[2] * (4 * zz - xx - 3 * yy), d[2] * 8 * yz),
                    (d[3] * z * (2 * zz - 3 * xx - 3 * yy), d[3] * -6 * xz, d[3] * -6 * yz, d[3] * (6 * zz - 3 * xx - 3 * yy)),
                    (d[4] * x * (4 * zz - xx - yy), d[4] * (4 * zz - 3 * xx - yy), d[4] * -2 * xy, d[4] * 8 * xz),
                    (d[5] * z * (xx - yy), d[5] * 2 * xz, d[5] * -2 * yz, d[5] * (xx - yy)),
                    (d[6] * x * (xx - 3 * yy), d[6] * (3 * xx - 3 * yy), d[6] * -6 * xy, None)]
    return out


# dR[j][k] / dq (q = r, x, y, z) of R(q) (R[0][0] = 1 - 2 (y^2 + z^2), R[0][1] = 2 (x y - r z), ...): the nonzero
# entries as (j, k, [(coefficient, quaternion index of the factor)]) per quaternion component
_DR_DQ = {
    0: [(0, 1, [(-2, 3)]), (0, 2, [(2, 2)]), (1, 0, [(2, 3)]), (1, 2, [(-2, 1)]), (2, 0, [(-2, 2)]), (2, 1, [(2, 1)])],
    1: [(0, 1, [(2, 2)]), (0, 2, [(2, 3)]), (1, 0, [(2, 2)]), (1, 1, [(-4, 1)]), (1, 2, [(-2, 0)]), (2, 0, [(2, 3)]),
        (2, 1, [(2, 0)]), (2, 2, [(-4, 1)])],
    2: [(0, 0, [(-4, 2)]), (0, 1, [(2, 1)]), (0, 2, [(2, 0)]), (1, 0, [(2, 1)]), (1, 2, [(2, 3)]), (2, 0, [(-2, 0)]),
        (2, 1, [(2, 3)]), (2, 2, [(-4, 2)])],
    3: [(0, 0, [(-4, 3)]), (0, 1, [(-2, 0)]), (0, 2, [(2, 1)]), (1, 0, [(2, 0)]), (1, 1, [(-4, 3)]), (1, 2, [(2, 2)]),
        (2, 0, [(2, 1)]), (2, 1, [(2, 2)])],
}


def scatter_terms(g, rows, v, e, a, acc, sign=None):
    """The float64 statement of the scatter, one column: every full-size row r receives
        sum_{i: c_i = r} t_i g_i  +  sum_{i: p_i = r, u_i != 0} u_i s_i g_i
    over the rendered rows i in `rows` (the visible ones), with g_i = v (its error bound e and magnitude chain a, in
    units of U, from chain_reference), u_i = fp32(1 - t_i) and the lerp taken only where u_i != 0 exactly (gather_fp32's
    `lerp`, the kernels' decision), s_i the quaternion sign (rotations only, else None).  Accumulates into acc = (value,
    error, magnitude, sum of |terms|, term count) [N] float64 arrays: each term carries its own error scaled by the
    weight plus one rounding of the product w g."""
    ref, err, mag, sm, cnt = acc
    tw = g["t"][rows].astype(np.float64)
    uw = g["u"][rows].astype(np.float64) * (sign if sign is not None else 1.0)
    for idx, w, on in ((g["c"][rows], tw, np.ones(rows.size, bool)), (g["p"][rows], uw, g["lerp"][rows])):
        idx, w, aw = idx[on], w[on], np.abs(w[on])
        np.add.at(ref, idx, w * v[on])
        np.add.at(err, idx, aw * e[on] + aw * np.abs(v[on]))
        np.add.at(mag, idx, aw * a[on])
        np.add.at(sm, idx, aw * np.abs(v[on]))
        np.add.at(cnt, idx, 1)


def scatter_tol(err, sm, cnt):
    """budget of a full-size row from scatter_terms' sums: the terms' own errors and roundings, plus (n - 1) U sum |terms|
    for the n-term fp32 atomic sum into the zero-filled row in an unspecified order (the first addition onto 0 is exact).
    A row no visible row reaches, or reached by exact zeros only, has budget 0: it must hold exactly +0.0."""
    return U * (err + np.maximum(cnt - 1, 0) * sm)


def chain_reference(means3D, opacities, scales, rotations, shs, colors_precomp, cov3D_precomp, scale_modifier, view, proj,
                    campos, W, H, tanx, tany, sh_degree, radii, accum, sh_clamp, fclamp, fsign, do_depth,
                    ridx=None, pidx=None, ts=None, eps=1e-7):
    """All parameters as the renderer takes them (fp32; shs [N][M][3]); view / proj [16] (transposed storage); radii [P];
    accum [P][10] (the blend's sums); sh_clamp [P][3] bool (kbits 20-22); fclamp [P][2] bool and fsign [P][2] (+-1: the
    side) of K1's frustum clamp (frustum_clamp_fp32); ridx / pidx / ts: scatter mode (P rendered rows over N source rows), else None.
    eps: the published 1e-7 of the inverse's gradient (0: the exact derivative).
    -> dict name -> (ref, tol, mag) float64 arrays in the layout of the returned gradients (tol: the budget,
    mag: the magnitude chain) for means2D [P][3], means3D, opacities, shs, colors, scales, rotations, cov3D [N][..]."""
    f32 = np.float32
    means3D = np.asarray(means3D, f32)
    N = means3D.shape[0]
    P = np.asarray(radii).shape[0]
    scatter = ridx is not None
    if scatter:
        g = gather_fp32(means3D, scales, rotations, shs, ridx, pidx, ts)
    else:
        ar = np.arange(P)
        g = dict(c=ar, p=ar, t=np.ones(P, f32), u=np.zeros(P, f32), lerp=np.zeros(P, bool), means3D=means3D,
                 scales=None if scales is None else np.asarray(scales, f32),
                 rotations=None if rotations is None else np.asarray(rotations, f32),
                 shs=None if shs is None else np.asarray(shs, f32), qsign=np.ones(P, f32))
    vis = np.asarray(radii) > 0
    rows = np.nonzero(vis)[0]
    ac = np.asarray(accum, f32)[rows].astype(np.float64)
    ex = lambda a: E(np.asarray(a, np.float64))
    v = [ex(np.float32(x)) for x in np.asarray(view, f32).reshape(16)]
    q = [ex(np.float32(x)) for x in np.asarray(proj, f32).reshape(16)]
    tanx, tany = float(f32(tanx)), float(f32(tany))
    m = [ex(g["means3D"][rows, k]) for k in range(3)]

    # ---- K8: view-space mean, clamp, Jacobian ----
    t = [v[r] * m[0] + v[4 + r] * m[1] + v[8 + r] * m[2] + v[12 + r] for r in range(3)]
    tz = t[2]
    fx = ex(W) / (2 * ex(tanx))
    fy = ex(H) / (2 * ex(tany))
    fcl = np.asarray(fclamp, bool)[rows]
    fsg = np.asarray(fsign, np.float64)[rows]

    def clamp(tv, lim_tan, k):
        lim = E.const(FOV_CLAMP) * ex(lim_tan)
        free = (tv / tz) * tz
        bound = E(fsg[:, k]) * lim * tz
        c = fcl[:, k]
        return E(np.where(c, bound.v, free.v), np.where(c, bound.a, free.a), np.where(c, bound.m, free.m),
                 np.where(c, bound.e, free.e))
    tx, ty = clamp(t[0], tanx, 0), clamp(t[1], tany, 1)
    J00, J02 = fx / tz, -(fx * tx) / (tz * tz)
    J11, J12 = fy / tz, -(fy * ty) / (tz * tz)
    A = [[J00 * v[4 * c] + J02 * v[4 * c + 2] for c in range(3)], [J11 * v[4 * c + 1] + J12 * v[4 * c + 2] for c in range(3)]]

    # ---- Sigma ----
    have_sr = cov3D_precomp is None
    if have_sr:
        mod = ex(f32(scale_modifier))
        s = [mod * ex(g["scales"][rows, k]) for k in range(3)]
        qq = [ex(g["rotations"][rows, k]) for k in range(4)]
        r_, x_, y_, z_ = qq
        R = [[1 - 2 * (y_ * y_ + z_ * z_), 2 * (x_ * y_ - r_ * z_), 2 * (x_ * z_ + r_ * y_)],
             [2 * (x_ * y_ + r_ * z_), 1 - 2 * (x_ * x_ + z_ * z_), 2 * (y_ * z_ - r_ * x_)],
             [2 * (x_ * z_ - r_ * y_), 2 * (y_ * z_ + r_ * x_), 1 - 2 * (x_ * x_ + y_ * y_)]]
        Mm = [[s[k] * R[j][k] for j in range(3)] for k in range(3)]
        V6 = [_sum([Mm[k][a] * Mm[k][b] for k in range(3)]) for a, b in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))]
    else:
        cv = np.asarray(cov3D_precomp, f32)[g["c"][rows]]
        V6 = [ex(cv[:, k]) for k in range(6)]

    # ---- the fp64 block: conic -> (a, b, c) ----
    dc = [ex(-0.5 * ac[:, 2]), ex(-0.5 * ac[:, 3]), ex(-0.5 * ac[:, 4])]
    blk = _block_e(A, V6, dc, eps)
    AV = [blk[0:3], blk[3:6]]
    dLa, dLb, dLc = blk[6], blk[7], blk[8]

    # ---- cov2D = A Sigma A^T: d/dSigma (off-diagonals counted for both uses), d/dA, d/dJ, d/dt ----
    g6 = []
    for a_, b_ in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)):
        if a_ == b_:
            g6.append(A[0][a_] * A[0][a_] * dLa + A[0][a_] * A[1][a_] * dLb + A[1][a_] * A[1][a_] * dLc)
        else:
            g6.append(2 * A[0][a_] * A[0][b_] * dLa + (A[0][a_] * A[1][b_] + A[0][b_] * A[1][a_]) * dLb
                      + 2 * A[1][a_] * A[1][b_] * dLc)
    dA = [[2 * AV[0][c] * dLa + AV[1][c] * dLb for c in range(3)], [2 * AV[1][c] * dLc + AV[0][c] * dLb for c in range(3)]]
    dJ00 = _sum([dA[0][c] * v[4 * c] for c in range(3)])
    dJ02 = _sum([dA[0][c] * v[4 * c + 2] for c in range(3)])
    dJ11 = _sum([dA[1][c] * v[4 * c + 1] for c in range(3)])
    dJ12 = _sum([dA[1][c] * v[4 * c + 2] for c in range(3)])
    itz = 1 / tz
    tz2 = itz * itz
    tz3 = tz2 * itz
    dtx = (-fx * tz2 * dJ02).mask(~fcl[:, 0])
    dty = (-fy * tz2 * dJ12).mask(~fcl[:, 1])
    dtz = -fx * tz2 * dJ00 - fy * tz2 * dJ11 + (2 * fx * tx) * tz3 * dJ02 + (2 * fy * ty) * tz3 * dJ12
    if do_depth:
        dtz = dtz - ex(ac[:, 9]) / (tz * tz)
    dmean = [v[4 * k] * dtx + v[4 * k + 1] * dty + v[4 * k + 2] * dtz for k in range(3)]

    # ---- K9a: NDC mean -> mean ----
    gmx, gmy = ex(ac[:, 0]) * ex(0.5 * W), ex(ac[:, 1]) * ex(0.5 * H)
    hw = q[3] * m[0] + q[7] * m[1] + q[11] * m[2] + q[15]
    mw = 1 / (hw + E.const(W_EPS))
    mul1 = (q[0] * m[0] + q[4] * m[1] + q[8] * m[2] + q[12]) * mw * mw
    mul2 = (q[1] * m[0] + q[5] * m[1] + q[9] * m[2] + q[13]) * mw * mw
    for k in range(3):
        dmean[k] = dmean[k] + (q[4 * k] * mw - q[4 * k + 3] * mul1) * gmx + (q[4 * k + 1] * mw - q[4 * k + 3] * mul2) * gmy

    # ---- K9b: SH -> coefficients and view direction ----
    dsh = dmean_sh = None
    if colors_precomp is None:
        M = g["shs"].shape[1]
        sh = g["shs"][rows]
        cp = [ex(np.float32(x)) for x in np.asarray(campos, f32)]
        d0 = [m[k] - cp[k] for k in range(3)]
        ln = (d0[0] * d0[0] + d0[1] * d0[1] + d0[2] * d0[2]).sqrt()
        x, y, z = d0[0] / ln, d0[1] / ln, d0[2] / ln
        shc = np.asarray(sh_clamp, bool)[rows]
        gr = [ex(np.where(shc[:, ch], 0.0, ac[:, 6 + ch])) for ch in range(3)]
        basis = _sh_basis(sh_degree, x, y, z)
        dsh = [[None] * 3 for _ in range(M)]
        dd = [None, None, None]
        for k, (B, *dB) in enumerate(basis):
            for ch in range(3):
                dsh[k][ch] = B * gr[ch]
                for a_ in range(3):
                    if dB[a_] is not None:
                        term = dB[a_] * ex(sh[:, k, ch]) * gr[ch]
                        dd[a_] = term if dd[a_] is None else dd[a_] + term
        zero = ex(np.zeros(rows.size))
        dd = [zero if d is None else d for d in dd]
        sum2 = d0[0] * d0[0] + d0[1] * d0[1] + d0[2] * d0[2]
        inv32 = 1 / (sum2 * sum2 * sum2).sqrt()
        dmean_sh = [_sum([(sum2 - d0[a_] * d0[a_]) * dd[a_] if a_ == b_ else -(d0[b_] * d0[a_]) * dd[b_] for b_ in range(3)])
                    * inv32 for a_ in range(3)]

    # ---- K9c: Sigma -> scale, rotation ----
    dscale = dq = None
    if have_sr:
        dS = [[g6[0], 0.5 * g6[1], 0.5 * g6[2]], [0.5 * g6[1], g6[3], 0.5 * g6[4]], [0.5 * g6[2], 0.5 * g6[4], g6[5]]]
        dM = [[2 * _sum([Mm[k][i] * dS[i][j] for i in range(3)]) for j in range(3)] for k in range(3)]
        dscale = [mod * _sum([R[j][k] * dM[k][j] for j in range(3)]) for k in range(3)]
        dR = [[s[k] * dM[k][j] for k in range(3)] for j in range(3)]
        dq = [_sum([dR[j][k] * (co * qq[f]) for j, k, ((co, f),) in _DR_DQ[w]]) for w in range(4)]

    # ---- emit: direct rows, or the t / (1 - t) scatter ----
    out = {}

    def emit(name, width, vals, weight_u=None):
        """vals: per column, an E over the visible rows or a list of E (parts the kernels add separately)"""
        ref = np.zeros((N if scatter else P, width))
        err, mag, sm, cnt = (np.zeros_like(ref) for _ in range(4))
        for col, val in enumerate(vals):
            for pc in (val if isinstance(val, list) else [val]):
                v, e, a = (np.broadcast_to(x, (rows.size,)) for x in (pc.v, pc.e, pc.a))
                if not scatter:
                    for arr, x in ((ref, v), (err, e), (mag, a), (sm, np.abs(v)), (cnt, 1)):
                        arr[rows, col] += x
                    continue
                scatter_terms(g, rows, v, e, a, (ref[:, col], err[:, col], mag[:, col], sm[:, col], cnt[:, col]),
                              None if weight_u is None else weight_u[rows])
        # direct rows: a second part is one more fp32 add (dL/dmean3D of K8 + K9a, then += the SH term);
        # scattered rows: an n-term fp32 atomic sum in any order (scatter_tol)
        tol = U * (err + (cnt > 1) * sm) if not scatter else scatter_tol(err, sm, cnt)
        out[name] = (ref, tol, mag)

    # dL/dmeans2D: one fp32 multiply of the sum by 0.5 W (0.5 H), so bit-exact; rows per rendered row
    m2 = np.zeros((P, 3))
    acc32 = np.asarray(accum, f32)
    m2[rows, 0] = acc32[rows, 0] * f32(0.5 * W)
    m2[rows, 1] = acc32[rows, 1] * f32(0.5 * H)
    out["means2D"] = (m2, np.zeros_like(m2), np.abs(m2))
    mparts = [[dmean[k]] + ([dmean_sh[k]] if dmean_sh is not None else []) for k in range(3)]
    emit("means3D", 3, mparts)
    emit("opacities", 1, [ex(ac[:, 5])])
    if dsh is not None:
        Mfull = g["shs"].shape[1]
        cols = []
        for k in range(Mfull):
            for ch in range(3):
                cols.append(dsh[k][ch] if k < len(dsh) and dsh[k][ch] is not None else ex(np.zeros(rows.size)))
        emit("shs", 3 * Mfull, cols)
        r_, t_, mg = out["shs"]
        out["shs"] = (r_.reshape(-1, Mfull, 3), t_.reshape(-1, Mfull, 3), mg.reshape(-1, Mfull, 3))
    if colors_precomp is not None:
        emit("colors", 3, [ex(ac[:, 6 + ch]) for ch in range(3)])
    if have_sr:
        emit("scales", 3, dscale)
        emit("rotations", 4, dq, weight_u=g["qsign"].astype(np.float64))
    else:
        emit("cov3D", 6, g6)
    return out


# ---- scenes under general cameras (shared by the CPU and GPU tests) -----------------------------------------------------
def general_camera(W, H, trans, axis=(1.0, 2.0, -0.7), angle_deg=37.0, **kw):
    """a camera rotated about a non-axis direction and translated: view = R^T world + trans (|trans| from the origin)"""
    import math
    from h3dgs import synth
    a = np.asarray(axis, np.float64)
    a /= np.linalg.norm(a)
    th = math.radians(angle_deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    R = np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K
    return synth.make_camera(W, H, R=R, T=np.asarray(trans, np.float64), **kw)


def world_from_view(cam, pv):
    """float64 world positions whose (float64) view-space position is pv [n][3]"""
    V = np.asarray(cam.world_view_transform, np.float64)       # row-vector convention: view = [p, 1] V
    return (np.asarray(pv, np.float64) - V[3, :3]) @ np.linalg.inv(V[:3, :3])


def random_rows(rng, n, deg_M=16, sh_scale=0.3):
    """scales, unit quaternions, opacities, SH for n Gaussians"""
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    sh = (sh_scale * rng.standard_normal((n, deg_M, 3))).astype(np.float32)
    sh[:, 0] = rng.uniform(-3.0, 3.0, (n, 3))                  # colour C0 sh0 + 0.5 below 0 for about a fifth
    return (np.exp(rng.uniform(-4.5, -1.5, (n, 3))).astype(np.float32), q.astype(np.float32),
            rng.uniform(0.05, 0.95, (n, 1)).astype(np.float32), sh)


ACCUM_SCALE = np.array([1e-3, 1e-3, 1e-2, 1e-2, 1e-2, 1e-2, 1e-2, 1e-2, 1e-2, 1e-3])


def random_accum(rng, P, single=None):
    """seeded normal [P][10] sums at realistic per-column scales; single: only that column non-zero"""
    a = rng.standard_normal((P, 10)) * ACCUM_SCALE
    if single is not None:
        keep = np.zeros(10, bool)
        keep[single] = True
        a[:, ~keep] = 0
    return a.astype(np.float32)


def compare(got, ref, tol, mask=None):
    """max |got - ref| / tol over the unmasked elements (an element with tol 0 must be exact), and the element count.
    A non-finite element of `got` counts as infinitely far (a NaN would otherwise compare false against any bar)."""
    got = np.asarray(got, np.float64).reshape(ref.shape)
    d = np.abs(got - ref)
    d = np.where(np.isfinite(got), d, np.inf)
    keep = np.ones(ref.shape, bool) if mask is None else np.broadcast_to(np.asarray(mask).reshape(
        mask.shape + (1,) * (ref.ndim - np.ndim(mask))), ref.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / tol)
    r = r[keep]
    return (float(r.max()) if r.size else 0.0), int(keep.sum())
