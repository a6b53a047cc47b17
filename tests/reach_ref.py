"""Float64 judge of which 4x4-pixel blocks of a tile an entry can reach (csrc/reach_mask.cuh::block_mask16).

Input: the entries' fp32 records (x, y, conic A B C, opacity; `_C.state_view(...)["records"]` rows) and their tiles.
Per (entry, pixel centre of the tile) the base alpha a = min(0.99, o exp(power)) is compared with 1/255 in the log
domain, against blend_ref's decision margin m = max(MARGIN, 4 eps_a), eps_a = 4 U mag + 2^-22 + 3 U (+ EPS_HIER in
hierarchy mode), mag the magnitude of the power's terms -- the blend's own fp32 power and ex2.approx error:
  taken  : ln a >= ln(1/255) + m;     near : |ln a - ln(1/255)| < m;     otherwise not taken.
(For m << 1 this is blend_ref's |a - 1/255| <= m / 255; the log form keeps its meaning where an ill-conditioned conic
makes m exceed 1.)  The hierarchy weight only lowers alpha, so the base alpha is the conservative one to judge.  One
decision is exact rather than near: the blend's fp32 alpha is o G with G = ex2.approx(power) <= 1, so an opacity below
fp32(1/255) is never taken, however close.
Two block sets per entry (bit 4 q + g, the quadrant-major layout of the mask):
  needed  : blocks holding a taken or a near pixel -- the mask must mark every one;
  touched : blocks whose rectangle of pixel centres meets the float64 ellipse {q <= 2 ln(255 o)}, by the exact minimum
            of q over the rectangle (0 with the mean inside, else on an edge) -- a marked block that is neither touched
            nor needed is work the blend does for nothing.
"""
import numpy as np

from blend_ref import ALPHA_CAP, ALPHA_SKIP, EPS_EX2, EPS_HIER, MARGIN, TILE, U

CHUNK = 4096


def block_bit(bx, by):
    return 4 * ((bx >> 1) | ((by >> 1) << 1)) + ((bx & 1) | ((by & 1) << 1))


_PX = np.arange(TILE * TILE) % TILE
_PY = np.arange(TILE * TILE) // TILE
_PBIT = (1 << block_bit(_PX >> 2, _PY >> 2)).astype(np.int64)          # [256] the block bit of each pixel of a tile
_BX, _BY = np.meshgrid(np.arange(4), np.arange(4))
_BBIT = (1 << block_bit(_BX.ravel(), _BY.ravel())).astype(np.int64)    # [16]


def _or_bits(flags, bits):
    """[n][k] bool, [k] bit values -> [n] OR of the bits set"""
    return np.bitwise_or.reduce(np.where(flags, bits[None], 0), axis=1)


def _rect_min_q(A, B, C, ex0, ex1, ey0, ey1):
    """exact min of q = A ex^2 + 2 B ex ey + C ey^2 over [ex0, ex1] x [ey0, ey1] (arrays, positive definite q)"""
    inside = (ex0 <= 0) & (0 <= ex1) & (ey0 <= 0) & (0 <= ey1)
    best = np.full(np.broadcast(A, ex0).shape, np.inf)
    for ey in (ey0, ey1):
        ex = np.clip(-B * ey / A, ex0, ex1)
        best = np.minimum(best, A * ex * ex + 2 * B * ex * ey + C * ey * ey)
    for ex in (ex0, ex1):
        ey = np.clip(-B * ex / C, ey0, ey1)
        best = np.minimum(best, A * ex * ex + 2 * B * ex * ey + C * ey * ey)
    return np.where(inside, 0.0, best)


def judge(rec, tiles, gx, hier=False):
    """rec [n][>=6] fp32 records, tiles [n] tile ids of a grid gx tiles wide ->
    dict(needed [n], touched [n] (uint16 block masks), taken [n][256], near [n][256] (bool, pixel p = 16 py + px))"""
    rec = np.asarray(rec, np.float32)
    tiles = np.asarray(tiles, np.int64)
    n = rec.shape[0]
    out = dict(needed=np.zeros(n, np.int64), touched=np.zeros(n, np.int64), taken=np.zeros((n, 256), bool),
               near=np.zeros((n, 256), bool))
    ln_skip = np.log(ALPHA_SKIP)
    for s in range(0, n, CHUNK):
        r = rec[s:s + CHUNK].astype(np.float64)
        x, y, A, B, C, o = (r[:, c:c + 1] for c in range(6))
        tx, ty = (tiles[s:s + CHUNK] % gx)[:, None], (tiles[s:s + CHUNK] // gx)[:, None]
        dx = x - (TILE * tx + _PX[None])                     # mean - pixel, as the blend forms it
        dy = y - (TILE * ty + _PY[None])
        with np.errstate(all="ignore"):
            power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
            mag = 0.5 * (np.abs(A) * dx * dx + np.abs(C) * dy * dy) + np.abs(B * dx * dy)
            eps_a = 4 * U * mag + EPS_EX2 + 3 * U + (EPS_HIER if hier else 0.0)
            m = np.maximum(MARGIN, 4 * eps_a)
            la = np.minimum(np.log(ALPHA_CAP), np.log(np.where(o > 0, o, np.nan)) + power)
            ok = (power <= 0) & (o >= ALPHA_SKIP)
            taken = ok & (la >= ln_skip + m)
            near = ok & ~taken & (la > ln_skip - m)
        out["taken"][s:s + CHUNK], out["near"][s:s + CHUNK] = taken, near
        out["needed"][s:s + CHUNK] = _or_bits(taken | near, _PBIT)
        # touched: exact minimum of q over each block's rectangle of pixel centres
        with np.errstate(all="ignore"):
            bound = 2 * np.log(255.0 * o)
            pd = (A > 0) & (A * C - B * B > 0) & (bound >= 0) & np.isfinite(x) & np.isfinite(y)
            ex0 = TILE * tx + 4 * _BX.ravel()[None] - x
            ey0 = TILE * ty + 4 * _BY.ravel()[None] - y
            q = _rect_min_q(A, B, C, ex0, ex0 + 3, ey0, ey0 + 3)
        out["touched"][s:s + CHUNK] = _or_bits(pd & (q <= bound), _BBIT)
    return out


def degenerate(rec):
    """[n] bool: records for which the mask is documented to be 0xFFFF (conic not positive definite, or not finite)"""
    r = np.asarray(rec, np.float32).astype(np.float64)
    x, y, A, B, C = r[:, 0], r[:, 1], r[:, 2], r[:, 3], r[:, 4]
    with np.errstate(all="ignore"):
        return ~((A > 0) & (C > 0) & (A * C - B * B > 0) & np.isfinite(x) & np.isfinite(y))
