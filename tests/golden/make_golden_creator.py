"""Generates tests/golden/creator_hier.npz by EXECUTING the reference's own `GaussianModel.create_from_hier`
(scene/gaussian_model.py:326-399, the loader train_post.py and render_hierarchy.py use) on a `hierarchy.hier` written by
this repository's creator (gaussian_hierarchy.creator, full_train.py's argv, a chunk whose skybox rows come first and a
scaffold whose pc_info.txt counts them), and storing the parameters it assigns: _xyz, _features_dc, _features_rest,
_opacity, _scaling, _rotation, nodes, boxes, skybox_points.  The creator runs on the emulation build of the kernels
(tests/emul/), so no GPU is needed; the reference's `.cuda()` calls land on the CPU (tests/emul/fake_device.py).  Needs a
checkout of the reference, named by H3DGS_REFERENCE.  The inputs (both PLY files' arrays) are stored beside the result;
tests/test_creator_golden_cpu.py rebuilds the file from them and checks it against what the reference assigned.

plyfile (which the reference's load_ply_file reads the scaffold with) is not installed: a minimal stand-in below
exposes the two things that function reads, `elements[0][name]` and `elements[0].properties[i].name`."""
import contextlib
import os
import sys
import tempfile
import types
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "emul")):
    sys.path.insert(0, p)

import refharness                                    # noqa: E402
import hier_build_ref as ref                         # noqa: E402
from fake_device import cuda_names_mean_cpu          # noqa: E402

S, P, SCAFFOLD_EXTRA = 24, 300, 50


class _Element:
    def __init__(self, data):
        self.data = data
        self.properties = [types.SimpleNamespace(name=n) for n in data.dtype.names]

    def __getitem__(self, name):
        return self.data[name]


class _PlyData:
    """binary little-endian, float properties only: what GaussianModel.save_ply writes"""

    def __init__(self, elements):
        self.elements = elements

    @staticmethod
    def read(path):
        with open(path, "rb") as f:
            names, n = [], 0
            while True:
                w = f.readline().decode().split()
                if w[0] == "end_header":
                    break
                if w[0] == "element":
                    n = int(w[2])
                elif w[0] == "property":
                    assert w[1] == "float", w
                    names.append(w[2])
            data = np.fromfile(f, dtype=[(x, "<f4") for x in names], count=n)
        return _PlyData([_Element(data)])


def inputs():
    """-> (chunk arrays with the skybox rows first, their logit opacities, scaffold arrays (degree-1 SH), logits)"""
    chunk = ref.cloud(S + P, seed=31)
    chunk["xyz"][:S] *= 60.0
    scaffold = ref.cloud(S + SCAFFOLD_EXTRA, seed=32, sh_coeffs=4)
    scaffold["xyz"][:S] = chunk["xyz"][:S]
    g = np.random.default_rng(33)
    return chunk, g.standard_normal(S + P).astype(np.float32), scaffold, g.standard_normal(S + SCAFFOLD_EXTRA).astype(np.float32)


def main():
    assert refharness.have_reference()
    import torch
    import build_emu
    from emu_api import Emu
    from test_hier_build_cpu import _emu_patches, write_ply
    from gaussian_hierarchy import creator
    chunk, logit, scaffold, slogit = inputs()
    with tempfile.TemporaryDirectory() as d:
        with mock.patch.object(build_emu, "SOURCES", build_emu.SOURCES + ["hier_build.cu"]):
            emu = Emu(build_emu.build(os.path.join(d, "emu")))
        ply = os.path.join(d, "chunk", "point_cloud.ply")
        sdir = os.path.join(d, "scaffold")
        os.makedirs(os.path.dirname(ply)); os.makedirs(sdir)
        write_ply(ply, chunk["xyz"], chunk["shs"], logit, chunk["log_scales"], chunk["rotations"])
        write_ply(os.path.join(sdir, "point_cloud.ply"), scaffold["xyz"], scaffold["shs"], slogit, scaffold["log_scales"],
                  scaffold["rotations"])
        with open(os.path.join(sdir, "pc_info.txt"), "w") as f:
            f.write(f"{S}\n")
        out = os.path.join(d, "trained_chunk")
        with contextlib.ExitStack() as st:
            for p in _emu_patches(emu):
                st.enter_context(p)
            assert creator.main([ply, os.path.join(d, "source_chunk"), out, sdir]) == 0
        # the reference's own loader
        refharness.import_reference_renderer()           # puts the reference on sys.path with simple_knn stubbed
        sys.modules["plyfile"] = types.SimpleNamespace(PlyData=_PlyData, PlyElement=object)
        sys.modules.pop("scene.gaussian_model", None)
        with cuda_names_mean_cpu():
            from scene.gaussian_model import GaussianModel
            assert GaussianModel.__module__ == "scene.gaussian_model"
            m = GaussianModel(3)
            m.create_from_hier(os.path.join(out, "hierarchy.hier"), 1.0, sdir)
        got = {k: getattr(m, k).detach().numpy() for k in ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")}
        got.update(nodes=m.nodes.numpy(), boxes=m.boxes.numpy(), skybox_points=np.int32(m.skybox_points))
    np.savez_compressed(os.path.join(HERE, "creator_hier.npz"), S=S,
                        **{f"chunk_{k}": v for k, v in chunk.items()}, chunk_logit=logit,
                        **{f"scaffold_{k}": v for k, v in scaffold.items()}, scaffold_logit=slogit,
                        **{f"ref{k}" if k.startswith("_") else f"ref_{k}": v for k, v in got.items()})
    print({k: v.shape for k, v in got.items()})


if __name__ == "__main__":
    main()
