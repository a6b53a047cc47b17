"""Generates tests/golden/post_train.npz by EXECUTING the reference's own code on the CPU: GaussianModel(3) built by
create_from_hier (scene/gaussian_model.py:326-399) from a small .hier written by this repo's hier_io, with anchors.bin,
exposure.json and a scaffold (point_cloud.ply + pc_info.txt) beside it; training_setup(our_adam=False) (torch.optim.Adam
with six groups); render_post() (gaussian_renderer/__init__.py:138-292, use_trained_exp=True, the Python gather and
parent lerp) with a CAPTURING fake rasterizer; the reference's utils/loss_utils l1_loss and ssim; and train_post.py:85-192
restated verbatim (train_post.py itself needs a dataset, a GPU and a DataLoader) over four consecutive iterations 1..4.

  - the skybox (the scaffold's first SKY points, appended by create_from_hier after the hierarchy rows) locked in
    iterations 1, 2 and 4, unlocked in 3;
  - anchors.bin lists a duplicate row and a skybox row;
  - stored opacities negative and exactly +0 / -0 (create_from_hier stores the .hier's opacities as they are and
    activates them with abs);
  - each iteration a different synthetic cut (rows, parents, weights strictly inside (0, 1) as well as 0 and 1):
    parents receive lerp gradients, and rows outside the cut move on their moments alone (a dense step);
  - image "img2" has no entry in exposure.json (render_post then applies none), the others their own 4x4;
  - an alpha mask in iterations 2 and 4, none in 1 and 3;
  - the xyz lr of xyz_scheduler_args changing every iteration (position_lr_max_steps = 10).

The full-size activated rows and their gradients (what the rasterizer backward hands the device step) are recorded by
retaining the gradients of the tensors GaussianModel's own get_* properties return.  plyfile is not installed: a
minimal ASCII PLY reader stands in for PlyData.read.  Needs a checkout of the reference, named by H3DGS_REFERENCE.

  tests/test_post_train_cpu.py    tests/post_train_ref.py and the kernel (emulation build) == this fixture
  tests/test_gpu_post_train.py    the kernel on the device == this fixture
"""
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "hierarchical-3d-gaussians_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "emul")):
    sys.path.insert(0, p)

import refharness                                    # noqa: E402
from fake_device import cuda_names_mean_cpu          # noqa: E402
from h3dgs import synth                              # noqa: E402

H, W, LEAVES, SCAFFOLD_PTS, SKY, NIMG = 19, 23, 40, 8, 5, 3
LAMBDA = 0.2
# iteration -> (skybox_locked, image, alpha mask)
PLAN = {1: (True, 0, False), 2: (True, 2, True), 3: (False, 1, False), 4: (True, 2, True)}
NAMES = ("means3D", "shs", "opacities", "scales", "rotations")
PROPS = {"means3D": "get_xyz", "shs": "get_features", "opacities": "get_opacity", "scales": "get_scaling",
         "rotations": "get_rotation"}
ATTRS = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")


class Capture(torch.nn.Module):
    """Stands in for diff_gaussian_rasterization.GaussianRasterizer."""
    raw = pattern = K = None

    def __init__(self, raster_settings):
        super().__init__()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        xs = dict(means3D=means3D, shs=shs, opacities=opacities, scales=scales, rotations=rotations)
        s = sum((x * Capture.K[k]).sum() for k, x in xs.items()) + (means2D * Capture.K["means2D"]).sum()
        radii = torch.ones(means3D.shape[0], dtype=torch.int32)
        return Capture.raw + s * Capture.pattern, radii, torch.zeros((1, H, W))


class _Ply:
    """PlyData.read of an ASCII PLY with one vertex element: elements[0][name] and elements[0].properties[i].name"""

    class _Element:
        def __init__(self, names, data):
            self.properties = [types.SimpleNamespace(name=n) for n in names]
            self._d = {n: data[:, i] for i, n in enumerate(names)}

        def __getitem__(self, name):
            return self._d[name]

    @classmethod
    def read(cls, path):
        with open(path) as f:
            lines = f.read().splitlines()
        end = lines.index("end_header")
        names = [ln.split()[-1] for ln in lines[:end] if ln.startswith("property")]
        data = np.array([[float(x) for x in ln.split()] for ln in lines[end + 1:] if ln.strip()], np.float32)
        return types.SimpleNamespace(elements=[cls._Element(names, data)])


def _write_ply(path, cols):
    names = list(cols)
    n = len(cols[names[0]])
    with open(path, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\n" % n)
        for k in names:
            f.write(f"property float {k}\n")
        f.write("end_header\n")
        for i in range(n):
            f.write(" ".join(repr(float(cols[k][i])) for k in names) + "\n")


def _scene_files(d, rng):
    """the .hier, anchors.bin, exposure.json and the scaffold directory; -> (hier path, scaffold dir, anchors)"""
    from gaussian_hierarchy.hier_io import write_hierarchy
    f32 = lambda a: np.asarray(a, np.float32)
    cam = synth.make_camera(W, H)
    h = synth.build_hierarchy(synth.cloud_v1(LEAVES, cam, zmin=2.0, zmax=20.0, seed=31, scale_k=1.0))
    P = h["means3D"].shape[0]
    op = f32(h["opacities"]).reshape(P).copy()
    op[::5] *= -1                                   # negative stored opacities: abs folds them
    op[3], op[7] = 0.0, -0.0                        # exactly +0 and -0: abs's backward is 0 there
    rot = f32(rng.normal(0, 1, (P, 4)))             # unnormalised stored quaternions
    write_hierarchy(os.path.join(d, "scene.hier"), h["means3D"], h["shs"], op, np.log(f32(h["scales"])), rot,
                    h["nodes"], h["boxes"])
    N = P + SKY
    anchors = np.array([2, 9, 9, P + 1, P - 1], np.int32)        # a duplicate and a skybox row
    with open(os.path.join(d, "anchors.bin"), "wb") as f:
        np.array([anchors.shape[0]], np.int32).tofile(f)
        anchors.tofile(f)
    ex = {}
    for i in range(NIMG):
        if i == 2:
            continue                                # img2 has no exposure
        E = np.eye(4, dtype=np.float32)
        E[:3, :4] += f32(rng.normal(0, 0.05, (3, 4)))
        ex[f"img{i}"] = E.tolist()
    with open(os.path.join(d, "exposure.json"), "w") as f:
        json.dump(ex, f)
    sd = os.path.join(d, "scaffold")
    os.makedirs(os.path.join(sd, "point_cloud"))
    n = SCAFFOLD_PTS
    cols = {"x": rng.normal(0, 50, n), "y": rng.normal(0, 50, n), "z": rng.uniform(60, 90, n)}
    for i in range(3):
        cols[f"f_dc_{i}"] = rng.normal(0, 0.5, n)
    for i in range(9):
        cols[f"f_rest_{i}"] = rng.normal(0, 0.05, n)
    cols["opacity"] = rng.normal(0, 1, n)
    for i in range(3):
        cols[f"scale_{i}"] = rng.normal(0, 0.3, n)
    for i in range(4):
        cols[f"rot_{i}"] = rng.normal(0, 1, n)
    _write_ply(os.path.join(sd, "point_cloud.ply"), cols)
    with open(os.path.join(sd, "pc_info.txt"), "w") as f:
        f.write(f"{SKY}\n")
    return os.path.join(d, "scene.hier"), sd, anchors, N, P, cam


def main():
    assert refharness.have_reference()
    with cuda_names_mean_cpu(), tempfile.TemporaryDirectory() as d:
        gr = refharness.import_reference_renderer()
        gr.GaussianRasterizer = Capture                  # the module-level name render_post() looks up
        import scene.gaussian_model as gm
        from utils.loss_utils import l1_loss, ssim
        gm.PlyData = _Ply

        class Recording(gm.GaussianModel):
            """GaussianModel whose get_* results keep their gradients: the full-size activated rows and gradients"""
            rec = None

        def recorded(name):
            base = getattr(gm.GaussianModel, name)

            def get(self):
                t = base.fget(self)
                if self.rec is not None:
                    if t.requires_grad and not t.is_leaf:
                        t.retain_grad()
                    self.rec[name].append(t)
                return t
            return property(get)
        for prop in PROPS.values():
            setattr(Recording, prop, recorded(prop))

        rng = np.random.default_rng(41)
        f32 = lambda a: np.asarray(a, np.float32)
        q = lambda a: (np.round(a * 256.0) / 256.0).astype(np.float32)
        path, scaffold, anchors, N, P, cam = _scene_files(d, rng)
        gaussians = Recording(3)
        gaussians.active_sh_degree = 3                   # train_post.py:32
        gaussians.create_from_hier(path, 2.0, scaffold)
        assert gaussians._xyz.shape[0] == N and gaussians.skybox_points == SKY
        assert torch.equal(gaussians.anchors, torch.tensor(anchors).long())
        opt = types.SimpleNamespace(percent_dense=0.01, position_lr_init=0.00016, position_lr_final=0.0000016,
                                    position_lr_delay_mult=0.01, position_lr_max_steps=10, feature_lr=0.0025,
                                    opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001, exposure_lr_init=0.01,
                                    exposure_lr_final=0.001, exposure_lr_delay_steps=0, exposure_lr_delay_mult=0.0,
                                    iterations=30_000, lambda_dssim=LAMBDA)
        gaussians.training_setup(opt, our_adam=False)
        assert type(gaussians.optimizer) is torch.optim.Adam
        out = {f"init_{a}": getattr(gaussians, a).detach().numpy().copy() for a in ATTRS}
        vcam = refharness.StubCamera(cam, device="cpu")
        pipe = refharness.Pipe()
        background = torch.zeros(3)
        # train_post.py:59-63's full-size scratch
        render_indices = torch.zeros(N).int()
        parent_indices = torch.zeros(N).int()
        interpolation_weights = torch.zeros(N).float()
        num_siblings = torch.zeros(N).int()
        for c, iteration in enumerate(sorted(PLAN)):
            locked, image, with_mask = PLAN[iteration]
            gaussians.skybox_locked = locked
            # a synthetic cut of the hierarchy rows: n rows, each with a parent, weights in [0, 1]
            n = 24
            ri = rng.choice(P, n, replace=False).astype(np.int32)
            pi = rng.integers(0, P, n).astype(np.int32)
            t = f32(rng.uniform(0.05, 0.95, n))
            t[:3], t[3:5] = 1.0, 0.0
            render_indices[:n] = torch.tensor(ri)
            parent_indices[:n] = torch.tensor(pi)
            interpolation_weights[:n] = torch.tensor(t)
            num_siblings[:] = torch.tensor(rng.integers(1, 4, N).astype(np.int32))
            Pr = n + SKY
            Capture.K = {k: torch.tensor(f32(rng.normal(0, 1, shp)))
                         for k, shp in (("means3D", (Pr, 3)), ("shs", (Pr, 16, 3)), ("opacities", (Pr, 1)),
                                        ("scales", (Pr, 3)), ("rotations", (Pr, 4)), ("means2D", (Pr, 3)))}
            Capture.raw = torch.tensor(q(rng.uniform(0.1, 0.8, (3, H, W))), requires_grad=True)
            Capture.pattern = torch.tensor(f32(rng.normal(0, 1e-3, (3, H, W))))
            gt_image = torch.tensor(q(rng.uniform(0, 1, (3, H, W))))
            vcam.image_name = f"img{image}"
            vcam.alpha_mask = torch.tensor((rng.uniform(size=(1, H, W)) > 0.3).astype(np.float32)) if with_mask else None
            viewpoint_cam = vcam
            gaussians.rec = {p: [] for p in PROPS.values()}
            # ---- train_post.py:85-192 ----
            gaussians.update_learning_rate(iteration)
            if iteration % 1000 == 0:
                gaussians.oneupSHdegree()
            to_render = n
            indices = render_indices[:to_render].int()
            render_pkg = gr.render_post(viewpoint_cam, gaussians, pipe, background, render_indices=indices,
                                        parent_indices=parent_indices, interpolation_weights=interpolation_weights,
                                        num_node_kids=num_siblings, use_trained_exp=True)
            image_t = render_pkg["render"]
            if viewpoint_cam.alpha_mask is not None:
                Ll1 = l1_loss(image_t * viewpoint_cam.alpha_mask.cuda(), gt_image)
                loss = (1.0 - opt.lambda_dssim) * Ll1 + opt.lambda_dssim * (1.0 - ssim(image_t * viewpoint_cam.alpha_mask.cuda(), gt_image))
            else:
                Ll1 = l1_loss(image_t, gt_image)
                loss = (1.0 - opt.lambda_dssim) * Ll1 + opt.lambda_dssim * (1.0 - ssim(image_t, gt_image))
            loss.backward()
            with torch.no_grad():
                # the full-size activated rows the step reads and their gradients (before the lock lines)
                act, act_grad = {}, {}
                for k, prop in PROPS.items():
                    ts = list({id(x): x for x in gaussians.rec[prop]}.values())     # get_xyz: the one leaf, twice
                    act[k] = ts[-1].detach().numpy().copy()
                    gs = [(x.grad if x.grad is not None else torch.zeros_like(x)) for x in ts]
                    act_grad[k] = sum(gs).numpy().copy()
                gaussians.rec = None
                xyz_lr = [g["lr"] for g in gaussians.optimizer.param_groups if g["name"] == "xyz"][0]
                if iteration < opt.iterations:
                    if gaussians._xyz.grad != None:  # noqa: E711  (verbatim)
                        if gaussians.skybox_points != 0 and gaussians.skybox_locked:
                            gaussians._xyz.grad[-gaussians.skybox_points:, :] = 0
                            gaussians._rotation.grad[-gaussians.skybox_points:, :] = 0
                            gaussians._features_dc.grad[-gaussians.skybox_points:, :, :] = 0
                            gaussians._features_rest.grad[-gaussians.skybox_points:, :, :] = 0
                            gaussians._opacity.grad[-gaussians.skybox_points:, :] = 0
                            gaussians._scaling.grad[-gaussians.skybox_points:, :] = 0

                        gaussians._xyz.grad[gaussians.anchors, :] = 0
                        gaussians._rotation.grad[gaussians.anchors, :] = 0
                        gaussians._features_dc.grad[gaussians.anchors, :, :] = 0
                        gaussians._features_rest.grad[gaussians.anchors, :, :] = 0
                        gaussians._opacity.grad[gaussians.anchors, :] = 0
                        gaussians._scaling.grad[gaussians.anchors, :] = 0
                    stored_grad = {a: getattr(gaussians, a).grad.numpy().copy() for a in ATTRS}
                    gaussians.optimizer.step()
                    gaussians.optimizer.zero_grad(set_to_none=True)
            g = lambda a: gaussians.optimizer.state[getattr(gaussians, a)]
            out.update({f"c{c}_iteration": np.int32(iteration), f"c{c}_locked": np.int32(locked),
                        f"c{c}_image": np.int32(image), f"c{c}_mask": np.int32(with_mask), f"c{c}_xyz_lr": np.float64(xyz_lr),
                        f"c{c}_render_indices": ri, f"c{c}_parent_indices": pi, f"c{c}_t": t,
                        f"c{c}_loss": np.float64(loss.item())})
            out.update({f"c{c}_act_{k}": v for k, v in act.items()})
            out.update({f"c{c}_actgrad_{k}": v for k, v in act_grad.items()})
            out.update({f"c{c}_grad{a}": v for a, v in stored_grad.items()})
            out.update({f"c{c}_after{a}": getattr(gaussians, a).detach().numpy().copy() for a in ATTRS})
            out.update({f"c{c}_adam{a}": out[f"c{c}_after{a}"] for a in ATTRS})         # train_post has no rescale
            out.update({f"c{c}_m{a}": g(a)["exp_avg"].numpy().copy() for a in ATTRS})
            out.update({f"c{c}_v{a}": g(a)["exp_avg_sq"].numpy().copy() for a in ATTRS})
            out[f"c{c}_step"] = np.int64(float(g("_xyz")["step"]))
            print(f"iteration {iteration}: locked={locked} image={image} mask={with_mask} N={N} cut={n} "
                  f"xyz_lr={xyz_lr:.4e} loss={loss.item():.5f} step={int(out[f'c{c}_step'])}")
        lrs = [g_["lr"] for g_ in gaussians.optimizer.param_groups]
        np.savez_compressed(os.path.join(HERE, "post_train.npz"), iterations=np.int32(len(PLAN)), lam=np.float64(LAMBDA),
                            skybox=np.int32(SKY), hier_rows=np.int32(P), anchors=anchors, lrs=np.float64(lrs), **out)


if __name__ == "__main__":
    main()
