"""CPU: the LOD budget.  The numpy restatement (tests/lod_budget_ref.py) against the oracle's cut count at every
candidate threshold and against its own step-weight derivation; then csrc/lod_budget.cu, built against the SIMT emulator
(tests/emul/), against the restatement bit for bit -- threshold, rows, unmet flag and counts -- over every budget around
every candidate's row count, on creator-built, general, single-node and odd-size (NaN, +-inf, negative, zero,
duplicated) hierarchies, from every viewpoint and floor of the shared cases."""
import os
import sys
from unittest import mock

import numpy as np
import pytest

import lod_budget_ref as ref
from h3dgs import synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emul"))

CAM = synth.make_camera(480, 270)
SCENES = dict(ref.scenes(CAM))


def bits(x):
    return int(np.asarray(x, np.float32).view(np.uint32))


@pytest.mark.parametrize("name", list(SCENES))
def test_restatement_counts_what_the_cut_emits(name):
    from oracle import oracle
    h = SCENES[name]
    nodes, boxes = h["nodes"], h["boxes"]
    seen_nan = False
    for vp in ref.views(h, CAM).values():
        size = ref.hg.node_sizes(boxes, vp)
        seen_nan |= bool(np.isnan(size).any())
        for floor in ref.floors(h, vp, CAM):
            ts = ref.candidates(size, floor) + [ref.t_max(size, floor)]
            ts += [np.float32(s) for s in np.unique(size[np.isfinite(size)])[:50]]
            for t in ts:
                n = oracle.expand_to_size(nodes, boxes, t, vp)[0]
                assert ref.rows(nodes, size, t) == n == ref.rows_by_keys(nodes, size, t), (name, floor, t)
    assert seen_nan == name.startswith("odd")


@pytest.mark.parametrize("name", list(SCENES))
def test_restatement_picks_the_smallest_feasible_candidate(name):
    h = SCENES[name]
    for vp in ref.views(h, CAM).values():
        for floor in ref.floors(h, vp, CAM):
            tab = ref.table(h["nodes"], h["boxes"], vp, floor)
            cands, r, size = tab
            assert all(a < b for a, b in zip(cands, cands[1:]))
            prev = None
            for B in ref.budgets(h["nodes"], tab, floor):
                got = ref.select(h["nodes"], h["boxes"], vp, floor, B, tab)
                t = got["threshold"]
                assert got["rows"] == ref.rows(h["nodes"], size, t)
                assert np.float32(floor) <= t <= ref.t_max(size, floor)
                if got["unmet"]:
                    assert (r > B).all() and t == ref.t_max(size, floor)
                else:
                    assert got["rows"] <= B and all(x > B for x in r[:cands.index(t)])
                    if B >= r[0]:
                        assert bits(t) == bits(floor)
                if prev is not None:
                    assert t <= prev                    # non-increasing in the budget
                prev = t


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """the emulation build of the library's sources plus lod_budget.cu"""
    import build_emu
    from emu_api import Emu
    with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["lod_budget.cu"]):
        return Emu(build_emu.build(str(tmp_path_factory.mktemp("h3dgs_emu_lod_budget"))))


def emu_budget(emu, nodes, boxes, vp, floor, budget, device_words=False):
    from emu_api import aligned, f32, i32, ptr
    L = emu.L
    N = nodes.shape[0]
    nd, bx, v = i32(nodes), f32(boxes), f32(vp)
    thr = aligned(4, np.float32, (1,))
    info = aligned(16, np.int32, (4,))
    thr[:] = np.nan
    info[:] = -7
    scratch = aligned(L.h3dgs_lod_budget_scratch_bytes(N))
    scratch[:] = 0xAB                                    # the call must not rely on zeroed scratch
    fdev, bdev = f32([floor]), i32([budget])
    emu.check(L.h3dgs_lod_budget(N, ptr(nd), ptr(bx), ptr(v), -1.0 if device_words else float(floor),
                                 ptr(fdev) if device_words else None, -1 if device_words else int(budget),
                                 ptr(bdev) if device_words else None, ptr(thr), ptr(info), ptr(scratch), None))
    return dict(threshold=thr[0], rows=int(info[0]), unmet=int(info[1]), kept=int(info[2]), total=int(info[3]))


@pytest.mark.parametrize("name", list(SCENES))
def test_kernel_equals_the_restatement(emu, name):
    h = SCENES[name]
    nodes, boxes = h["nodes"], h["boxes"]
    outcomes = set()
    for vi, vp in enumerate(ref.views(h, CAM).values()):
        for fi, floor in enumerate(ref.floors(h, vp, CAM)):
            tab = ref.table(nodes, boxes, vp, floor)
            for k, B in enumerate(ref.budgets(nodes, tab, floor, limit=24)):
                want = ref.select(nodes, boxes, vp, floor, B, tab)
                got = emu_budget(emu, nodes, boxes, vp, floor, B, device_words=(vi + fi + k) % 2 == 1)
                assert bits(got["threshold"]) == bits(want["threshold"]), (name, vi, floor, B, got, want)
                assert {k: got[k] for k in ("rows", "unmet", "kept", "total")} == \
                    {k: want[k] for k in ("rows", "unmet", "kept", "total")}, (name, vi, floor, B)
                outcomes.add("floor" if bits(want["threshold"]) == bits(floor) else "unmet" if want["unmet"] else "inner")
    if nodes.shape[0] > 5:
        assert outcomes == {"floor", "unmet", "inner"}


def test_argument_checks(emu):
    from emu_api import aligned, f32, i32, ptr
    L = emu.L
    h = SCENES["general5"]
    nd, bx, v = i32(h["nodes"]), f32(h["boxes"]), f32(CAM.camera_center)
    thr, info = aligned(4, np.float32, (1,)), aligned(16, np.int32, (4,))
    scratch = aligned(L.h3dgs_lod_budget_scratch_bytes(5) + 256)
    args = [5, ptr(nd), ptr(bx), ptr(v), 0.0, None, 3, None, ptr(thr), ptr(info), ptr(scratch), None]

    def call(**kw):
        a = list(args)
        for i, val in kw.items():
            a[int(i[1:])] = val
        return L.h3dgs_lod_budget(*a)
    assert call() == 0
    assert call(a0=0) < 0 and b"empty" in L.h3dgs_last_error()
    for i in (1, 2, 3, 8, 9, 10):
        assert call(**{f"a{i}": None}) < 0 and b"NULL" in L.h3dgs_last_error()
    assert call(a2=ptr(bx) + 4) < 0 and b"16-byte" in L.h3dgs_last_error()
    assert call(a10=ptr(scratch) + 16) < 0 and b"256-byte" in L.h3dgs_last_error()
    assert call(a6=-1) < 0 and b"negative" in L.h3dgs_last_error()
