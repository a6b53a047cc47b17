"""CPU: a `merged.hier` written by the command-line merger (emulation build of csrc/hier_merge.cu) is what the
reference's own `GaussianModel.create_from_hier`, given a scaffold as render_hierarchy.py passes it, assigned in
tests/golden/merger_hier.npz, produced by tests/golden/make_golden_merger.py from the same stored inputs: the merged
rows, nodes and boxes pass through the reference's loader unchanged, and the skybox rows it appends from the scaffold
follow them."""
import contextlib

import numpy as np
import pytest
import torch

from test_hier_merge_cpu import _emu_patches, bits, check_against_ref, emu, write_chunk_dirs  # noqa: F401  (emu: fixture)

KEYS = ("xyz", "shs", "opacities", "log_scales", "rotations", "nodes", "boxes")
NAMES = ["0_0", "1_0"]


@pytest.fixture(scope="module")
def golden(golden_dir):
    import os
    return dict(np.load(os.path.join(golden_dir, "merger_hier.npz")))


def _chunks(z):
    return [{k: z[f"chunk{c}_{k}"] for k in KEYS} for c in range(len(NAMES))]


def _merged_file(emu, z, tmp_path):
    from gaussian_hierarchy import merger
    from gaussian_hierarchy._C import load_hierarchy
    write_chunk_dirs(tmp_path, _chunks(z), z["cells"], NAMES)
    out = tmp_path / "output" / "merged.hier"
    with contextlib.ExitStack() as st:
        for p in _emu_patches(emu):
            st.enter_context(p)
        assert merger.main([str(tmp_path / "trained_chunks"), "0", str(tmp_path / "chunks"), str(out)] + NAMES) == 0
    return [t.numpy() for t in load_hierarchy(str(out))]


def test_the_reference_loader_assigns_the_merger_output(emu, golden, tmp_path):
    z = golden
    xyz, shs, opac, ls, rots, nodes, boxes = _merged_file(emu, z, tmp_path)
    S, N = int(z["S"]), xyz.shape[0]
    assert int(z["ref_skybox_points"]) == S and z["ref_xyz"].shape[0] == N + S
    assert np.array_equal(z["ref_nodes"], nodes) and np.array_equal(bits(z["ref_boxes"]), bits(boxes))
    for key, mine in (("ref_xyz", xyz), ("ref_features_dc", shs[:, :1]), ("ref_features_rest", shs[:, 1:]),
                      ("ref_opacity", opac), ("ref_scaling", ls), ("ref_rotation", rots)):
        assert np.array_equal(bits(z[key][:N]), bits(mine)), key


def test_the_stored_merge_follows_the_rule(golden):
    """what the reference loaded is the merge h3dgs.h specifies for the stored chunks (restated in numpy)"""
    z = golden
    N = z["ref_nodes"].shape[0]
    got = dict(xyz=z["ref_xyz"][:N], shs=np.concatenate([z["ref_features_dc"], z["ref_features_rest"]], 1)[:N],
               opacities=z["ref_opacity"][:N, 0], log_scales=z["ref_scaling"][:N], rotations=z["ref_rotation"][:N],
               nodes=z["ref_nodes"], boxes=z["ref_boxes"])
    r = check_against_ref(_with_sources(got, z), _chunks(z), z["cells"])
    assert r["xyz"].shape[0] == N


def _with_sources(got, z):
    """the loaded file carries no sources: take them from the restatement and check the rows against them"""
    import hier_merge_ref as ref
    r = ref.merge(_chunks(z), z["cells"])
    return dict(got, R=r["R"], source_chunk=r["source_chunk"], source_row=r["source_row"])


def test_the_skybox_rows_follow_the_hierarchy(golden):
    """what create_from_hier appends from the scaffold (:355-383): sigmoid opacity, degree-1 SH padded with zeros"""
    z = golden
    S, N = int(z["S"]), z["ref_nodes"].shape[0]
    sc = {k: z[f"scaffold_{k}"][:S] for k in ("xyz", "shs", "log_scales", "rotations")}
    assert np.array_equal(bits(z["ref_xyz"][N:]), bits(sc["xyz"]))
    assert np.array_equal(bits(z["ref_opacity"][N:, 0]), bits(torch.sigmoid(torch.from_numpy(z["scaffold_logit"][:S])).numpy()))
    assert np.array_equal(bits(z["ref_features_dc"][N:, 0]), bits(sc["shs"][:, 0]))
    assert np.array_equal(bits(z["ref_features_rest"][N:, :3]), bits(sc["shs"][:, 1:4])) and not z["ref_features_rest"][N:, 3:].any()
    assert np.array_equal(bits(z["ref_scaling"][N:]), bits(sc["log_scales"]))
    assert np.array_equal(bits(z["ref_rotation"][N:]), bits(sc["rotations"]))
