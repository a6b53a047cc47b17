"""TEST INFRASTRUCTURE ONLY.  A restatement of simple_knn._C.distCUDA2 (include/h3dgs.h h3dgs_dist_knn3) written from
its contract, not from the kernel: candidate neighbours from scipy's cKDTree in float64, the point's own index dropped
(not necessarily the first candidate when there are duplicates), the candidates' distances recomputed in the pinned
float32 order, the three smallest kept, FLT_MAX for each missing neighbour; rows with a non-finite coordinate are left
out of everything (their own output is NaN here: unspecified)."""
import numpy as np
from scipy.spatial import cKDTree

FLT_MAX = np.float32(np.finfo(np.float32).max)


def _fp32_dist2(F, rows, nb):
    """(dx*dx + dy*dy) + dz*dz, dx = q.x - p.x, every operation rounded to float32"""
    p, q = F[rows][:, None, :], F[nb]
    dx, dy, dz = q[..., 0] - p[..., 0], q[..., 1] - p[..., 1], q[..., 2] - p[..., 2]
    d = (dx * dx + dy * dy) + dz * dz
    return np.where(np.isfinite(d), d, FLT_MAX)      # an overflowing distance never beats a missing neighbour


def dist_knn3(points, k=16, chunk=1 << 20):
    pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    out = np.full(pts.shape[0], np.nan, np.float32)
    idx = np.nonzero(np.isfinite(pts).all(axis=1))[0]
    F, n = pts[idx], len(idx)
    if n == 0:
        return out
    tree = cKDTree(F.astype(np.float64))
    res = np.empty(n, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for c0 in range(0, n, chunk):
            rows = np.arange(c0, min(c0 + chunk, n))
            kk = min(k, n)
            while len(rows):
                dist, nb = tree.query(F[rows].astype(np.float64), k=kk, workers=-1)
                nb = nb.reshape(len(rows), kk)
                d = _fp32_dist2(F, rows, nb)
                d[nb == rows[:, None]] = np.inf                      # the point itself, by index
                d = np.sort(d, axis=1)
                best = np.full((len(rows), 3), FLT_MAX, np.float32)
                m = min(3, kk)
                best[:, :m] = np.minimum(d[:, :m], FLT_MAX)
                # exact as long as no point left unfetched could round below the third-best: every point was
                # fetched, the third-best is 0, or the farthest candidate is clearly beyond it (float64 vs float32)
                far = np.asarray(dist, np.float64).reshape(len(rows), kk)[:, -1] ** 2
                ok = (kk >= n) | (best[:, 2] == 0) | (far > best[:, 2].astype(np.float64) * (1 + 1e-5))
                res[rows[ok]] = ((best[ok, 0] + best[ok, 1]) + best[ok, 2]) / np.float32(3.0)
                rows, kk = rows[~ok], min(2 * kk, n)
    out[idx] = res
    return out


SIZES = [0, 1, 2, 3, 4, 5, 31, 32, 33, 1023, 1024, 1025, 4097]


def cases():
    """name -> seeded float32 [P, 3] cloud: the shapes that stress an exact search (ties, degenerate extents, far-apart
    groups, large offsets, a scene inside a skybox shell)"""
    rs = np.random.default_rng(7)
    c = {f"cube{n}": rs.uniform(-1, 1, (n, 3)) for n in SIZES}
    c["cube65536"] = rs.uniform(-1, 1, (65536, 3))
    c["plane"] = np.concatenate([rs.uniform(-5, 5, (3000, 2)), np.full((3000, 1), 0.25)], axis=1)
    t = rs.uniform(-10, 10, (2000, 1))
    c["collinear"] = np.concatenate([t, 2 * t + 1, -0.5 * t], axis=1)
    c["identical"] = np.tile([[0.1, -2.0, 3.5]], (1100, 1))
    base = rs.uniform(-1, 1, (700, 3))
    c["duplicates"] = np.concatenate([base, base[:400], base[:150]])[rs.permutation(1250)]
    g = np.arange(16, dtype=np.float64)
    c["lattice"] = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)
    c["two_clusters"] = np.concatenate([rs.normal(0, 1, (1500, 3)), rs.normal(0, 1, (1500, 3)) + [1e6, -1e6, 1e6]])
    c["offset"] = 1e4 + 1e-3 * rs.integers(0, 40, (3000, 3)) + 1e-4 * rs.uniform(0, 1, (3000, 3))
    scene = rs.normal(0, 1, (6000, 3)) * [4, 4, 1]
    lo, hi = scene.min(0), scene.max(0)
    mean, r = 0.5 * (lo + hi), 10 * np.linalg.norm(hi - 0.5 * (lo + hi))
    th, ph = 2 * np.pi * rs.uniform(0, 1, 400), np.arccos(1 - 1.4 * rs.uniform(0, 1, 400))
    sky = mean + r * np.stack([np.cos(th) * np.sin(ph), np.sin(th) * np.sin(ph), np.cos(ph)], axis=1)
    c["scene_skybox"] = np.concatenate([sky, scene])
    return {k: np.ascontiguousarray(v, np.float32).reshape(-1, 3) for k, v in c.items()}


def with_non_finite(pts, seed=11):
    """pts with NaN / +-inf rows (whole and partial) inserted at random places -> (cloud, mask of the finite rows)"""
    rs = np.random.default_rng(seed)
    bad = np.array([[np.nan, 0, 0], [np.inf, 1, 1], [-np.inf, -np.inf, -np.inf], [0.5, np.nan, 0.5], [0, 0, -np.inf],
                    [np.nan, np.nan, np.nan], [np.inf, -np.inf, np.nan]], np.float32)
    bad = np.concatenate([bad] * 5)
    allp = np.concatenate([pts, bad])
    order = rs.permutation(len(allp))
    finite = np.arange(len(allp)) < len(pts)
    return allp[order], finite[order]
