"""Generates tests/golden/merger_hier.npz by EXECUTING the reference's own `GaussianModel.create_from_hier`
(scene/gaussian_model.py:326-399), with a scaffold as render_hierarchy.py loads it, on a `merged.hier` written by this
repository's merger (gaussian_hierarchy.merger, full_train.py's argv: two chunks whose `hierarchy.hier_opt` carry
skybox rows after the hierarchy's, and `center.txt` / `extent.txt` as make_chunk.py writes them), and storing the
parameters it assigns: _xyz, _features_dc, _features_rest, _opacity, _scaling, _rotation, nodes, boxes, skybox_points.
The chunk hierarchies are built by the creator and the merge runs, both on the emulation build of the kernels
(tests/emul/), so no GPU is needed; the reference's `.cuda()` calls land on the CPU (tests/emul/fake_device.py).  Needs
a checkout of the reference, named by H3DGS_REFERENCE.  The inputs (the chunk hierarchies, the cells and the scaffold's
arrays) are stored beside the result; tests/test_merger_golden_cpu.py rebuilds the merged file from them and checks it
against what the reference assigned."""
import contextlib
import os
import sys
import tempfile
import types
from pathlib import Path
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "emul")):
    sys.path.insert(0, p)

import refharness                                    # noqa: E402
import hier_build_ref as hb                          # noqa: E402
import hier_merge_ref as ref                         # noqa: E402
from fake_device import cuda_names_mean_cpu          # noqa: E402
from make_golden_creator import _PlyData             # noqa: E402

S, SCAFFOLD_EXTRA, P = 12, 40, 120
NAMES = ["0_0", "1_0"]
KEYS = ("xyz", "shs", "opacities", "log_scales", "rotations", "nodes", "boxes")


def main():
    assert refharness.have_reference()
    import build_emu
    from emu_api import Emu
    from test_hier_build_cpu import run as build_run, write_ply
    from test_hier_merge_cpu import _emu_patches, creator_chunk, write_chunk_dirs
    from gaussian_hierarchy import merger
    cells = ref.grid_cells(2, 1)
    scaffold = hb.cloud(S + SCAFFOLD_EXTRA, seed=42, sh_coeffs=4)
    scaffold["xyz"][:S] *= 80.0
    slogit = np.random.default_rng(43).standard_normal(S + SCAFFOLD_EXTRA).astype(np.float32)
    with tempfile.TemporaryDirectory() as d:
        with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["hier_build.cu", "hier_merge.cu"]):
            emu = Emu(build_emu.build(os.path.join(d, "emu")))
        chunks = [creator_chunk(lambda c: build_run(emu, c), cells[k], P + 31 * k, 40 + k) for k in range(2)]
        root = Path(d)
        write_chunk_dirs(root, chunks, cells, NAMES)
        sdir = root / "scaffold"
        sdir.mkdir()
        write_ply(sdir / "point_cloud.ply", scaffold["xyz"], scaffold["shs"], slogit, scaffold["log_scales"],
                  scaffold["rotations"])
        (sdir / "pc_info.txt").write_text(f"{S}\n")
        out = root / "output" / "merged.hier"
        with contextlib.ExitStack() as st:
            for p in _emu_patches(emu):
                st.enter_context(p)
            assert merger.main([str(root / "trained_chunks"), "0", str(root / "chunks"), str(out)] + NAMES) == 0
        # the reference's own loader, as render_hierarchy.py calls it (--hierarchy, --scaffold_file)
        refharness.import_reference_renderer()
        sys.modules["plyfile"] = types.SimpleNamespace(PlyData=_PlyData, PlyElement=object)
        sys.modules.pop("scene.gaussian_model", None)
        with cuda_names_mean_cpu():
            from scene.gaussian_model import GaussianModel
            assert GaussianModel.__module__ == "scene.gaussian_model"
            m = GaussianModel(3)
            m.create_from_hier(str(out), 1.0, str(sdir))
        got = {k: getattr(m, k).detach().numpy() for k in ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")}
        got.update(nodes=m.nodes.numpy(), boxes=m.boxes.numpy(), skybox_points=np.int32(m.skybox_points))
    np.savez_compressed(os.path.join(HERE, "merger_hier.npz"), S=S, cells=cells,
                        **{f"chunk{c}_{k}": ch[k] for c, ch in enumerate(chunks) for k in KEYS},
                        **{f"scaffold_{k}": v for k, v in scaffold.items()}, scaffold_logit=slogit,
                        **{f"ref{k}" if k.startswith("_") else f"ref_{k}": v for k, v in got.items()})
    print({k: v.shape for k, v in got.items()})


if __name__ == "__main__":
    main()
