"""GPU: the SH backward's own-row stores (sh_backward_rows_kernel).  A full-size dL/dSH row that exactly one rendered row
writes -- as its own row, never as a lerped parent -- is stored instead of reduced into the zero-filled line.  On one cut
with every kind of row (tests/test_gpu_scatter_edges.py::cut_scene: fan-in groups, parents that are other rendered rows'
own rows, chains, parent_indices = -1 with t < 1, rows behind the camera), the one-call backward (row counts, stores)
and the serial debug backward (no counts, reductions only) are each checked per full-size row against chain_ref's
float64 scatter, and every single-writer row must be bit-identical between the two.  `case_*` also runs on the
emulation build (test_sh_backward_rows_cpu.py)."""
import numpy as np
import pytest

from chain_ref import gather_fp32, random_accum
import test_gpu_scatter_edges as se

pytestmark = pytest.mark.gpu


def writers(sc, radii):
    """per full-size row: how many visible rendered rows write it (own row +1, lerped parent +1), and the own rows that
    are also some visible row's lerped parent"""
    g = gather_fp32(sc["means3D"], None, None, None, sc["ridx"], sc["pidx"], sc["ts"])
    vis = np.asarray(radii) > 0
    n = np.zeros(len(sc["means3D"]), np.int64)
    np.add.at(n, g["c"][vis], 1)
    np.add.at(n, g["p"][vis & g["lerp"]], 1)
    both = np.intersect1d(g["c"][vis], g["p"][vis & g["lerp"]])
    return n, both


def case_store_equals_reduce(deg, M, seed=5):
    name = f"own-row stores deg={deg} M={M}"
    cam, sc, info = se.cut_scene(deg, M, seed)
    accum = random_accum(np.random.default_rng(seed), len(sc["ridx"]))
    stored, ref, radii, _ = se.check_full(name + " (one call)", cam, sc, deg, accum)
    reduced = se.check_full(name + " (debug: reductions only)", cam, sc, deg, accum, debug=True)[0]
    n, both = writers(sc, radii)
    one = np.flatnonzero(n == 1)
    assert one.size > 50 and both.size > 5 and (n > 2).any(), (name, one.size, both.size)
    a = stored["shs"].reshape(n.size, -1)
    b = reduced["shs"].reshape(n.size, -1)
    assert np.array_equal(a[one].view(np.uint32), b[one].view(np.uint32)), name
    assert a[one].any(), name


@pytest.mark.parametrize("deg,M", [(3, 16), (2, 16), (1, 4), (0, 4), (2, 12)])
def test_store_equals_reduce(deg, M):
    case_store_equals_reduce(deg, M)
