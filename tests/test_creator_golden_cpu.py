"""CPU: a `hierarchy.hier` written by the command-line creator (emulation build of csrc/hier_build.cu) is what the
reference's own `GaussianModel.create_from_hier` assigned in tests/golden/creator_hier.npz, produced by
tests/golden/make_golden_creator.py from the same stored inputs: the hierarchy rows, nodes and boxes pass through the
reference's loader unchanged, and the skybox rows it appends from the scaffold follow them (N hierarchy rows of N + S)."""
import contextlib
import os

import numpy as np
import pytest
import torch

from test_hier_build_cpu import _emu_patches, bits, emu, write_ply  # noqa: F401  (emu: the module's fixture)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "creator_hier.npz")))


def _creator_file(emu, z, tmp_path):
    from gaussian_hierarchy import creator
    from gaussian_hierarchy._C import load_hierarchy
    part = lambda pre: {k: z[f"{pre}_{k}"] for k in ("xyz", "shs", "opacities", "log_scales", "rotations")}
    chunk, scaffold = part("chunk"), part("scaffold")
    ply = tmp_path / "chunk" / "point_cloud.ply"
    sdir = tmp_path / "scaffold"
    ply.parent.mkdir()
    sdir.mkdir()
    write_ply(ply, chunk["xyz"], chunk["shs"], z["chunk_logit"], chunk["log_scales"], chunk["rotations"])
    write_ply(sdir / "point_cloud.ply", scaffold["xyz"], scaffold["shs"], z["scaffold_logit"], scaffold["log_scales"],
              scaffold["rotations"])
    (sdir / "pc_info.txt").write_text(f"{int(z['S'])}\n")
    with contextlib.ExitStack() as st:
        for p in _emu_patches(emu):
            st.enter_context(p)
        assert creator.main([str(ply), str(tmp_path / "source_chunk"), str(tmp_path / "out"), str(sdir)]) == 0
    return [t.numpy() for t in load_hierarchy(str(tmp_path / "out" / "hierarchy.hier"))], scaffold


def test_the_reference_loader_assigns_the_creator_output(emu, golden, tmp_path):
    z = golden
    (xyz, shs, opac, ls, rots, nodes, boxes), scaffold = _creator_file(emu, z, tmp_path)
    S, N = int(z["S"]), xyz.shape[0]
    assert int(z["ref_skybox_points"]) == S and N == 2 * (z["chunk_xyz"].shape[0] - S) - 1
    assert z["ref_xyz"].shape[0] == N + S and nodes.shape[0] <= z["ref_xyz"].shape[0]
    assert np.array_equal(z["ref_nodes"], nodes) and np.array_equal(bits(z["ref_boxes"]), bits(boxes))
    for key, mine in (("ref_xyz", xyz), ("ref_features_dc", shs[:, :1]), ("ref_features_rest", shs[:, 1:]),
                      ("ref_opacity", opac), ("ref_scaling", ls), ("ref_rotation", rots)):
        assert np.array_equal(bits(z[key][:N]), bits(mine)), key


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
