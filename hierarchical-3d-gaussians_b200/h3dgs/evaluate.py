"""Sync-free evaluation of a hierarchy over a tau sweep: the numbers render_hierarchy.py reports (PSNR and SSIM over every
test camera at tau in {0, 3, 6, 15}), with every frame replayed from one CUDA graph and one read-back at the end.

The drop-in flow of render_hierarchy.py pays, per frame, two host round trips (the int of expand_to_size; num_rendered
sizing the binning buffer), a .cpu() of the camera centre, ~25 PyTorch kernels of gather and lerp, the exposure matmul,
clamps, crop, mask and the metric reductions with a syncing .double() each.  Here one graph per camera size holds

  * h3dgs_lod_cut with the threshold read on the device, and the skybox rows after the cut (GraphedStep._part_a);
  * the capacity-mode forward with the cut gather and lerp fused into K1;
  * h3dgs_eval_metrics (csrc/metrics.cu): exposure, clamp, train_test_exp crop, alpha mask, per-channel squared error
    and the SSIM map sum in one pass, and a one-thread finisher that stores [psnr, ssim, status words] at a slot taken
    from a device counter.

Camera, target, mask, exposure and threshold are device-resident inputs copied in between replays.  A frame that does not
fit the capacities (cut > row capacity, D > bin capacity, a tile list > sort capacity) is flagged in its row and re-run
through the exact path (pipeline.render_hier_fused + the same metrics kernel) after the read-back.  LPIPS (VGG weights)
and writing PNGs (torchvision) are not part of this module: keep_images returns the images instead.
"""
import numpy as np
import torch

from . import _lib, pipeline
from .graphstep import GraphedStep, _check_index_sizing, _ptr


def _metrics(L, H, W, image, gt, exposure, mask, x0, out_image, sums, counter, results, stream, count=None, extra_rows=0,
             row_capacity=0, scan_info=None):
    _lib.check(L.h3dgs_eval_metrics(H, W, image.data_ptr(), gt.data_ptr(), _ptr(exposure), _ptr(mask), x0, _ptr(out_image),
                                    sums.data_ptr(), _ptr(count), extra_rows, row_capacity, _ptr(scan_info),
                                    counter.data_ptr(), results.data_ptr(), results.shape[0], stream))


class GraphedRender(GraphedStep):
    """Forward-only counterpart of GraphedStep for hierarchy scenes on one GPU: ONE graph = LOD cut (device threshold) +
    skybox rows + capacity-mode forward + metrics pass.  It reuses GraphedStep's plumbing (state buffers, raster
    arguments, _part_a, set_camera, set_threshold, scan_info) and allocates no gradient buffers.

    W, H, tanfovx, tanfovy are fixed per instance, and so are whether an exposure and a mask are applied and the
    train_test_exp crop.  Inputs that change between replays: set_camera, set_threshold, and the static buffers
    `gt` [3,H,W], `exposure` [3,4], `mask` [H,W] (set_inputs copies into them).  Outputs: `image` (the raw rasterizer
    output, equal to pipeline.render_hier_fused's image whenever the frame fits), `out_image` [3,H,W-x0] when
    keep_image (exposed, clamped, cropped), and one row per frame in `results` at slot `counter`++."""

    def __init__(self, scene, W, H, tanfovx, tanfovy, bg, threshold, sh_degree=3, row_capacity=None, bin_capacity=1 << 22,
                 sort_capacity=4096, exposure=False, mask=False, train_test_exp=False, keep_image=False, results=None,
                 counter=None, max_frames=1024, capture=True):
        if not scene.hier:
            raise ValueError("GraphedRender drives the hierarchy path (LOD cut + fused gather/lerp)")
        self.L = _lib.lib()
        self.scene, self.W, self.H = scene, int(W), int(H)
        self.threshold, self.sh_degree = float(threshold), int(sh_degree)
        self.world, self.rank, self.group, self.peer, self.arena = 1, 0, None, False, None
        dev = scene.means3D.device
        self.dev = dev
        self.N = scene.means3D.shape[0]
        self.N_nodes = scene.nodes.shape[0]
        _check_index_sizing(self.N_nodes, self.N)
        self.S = scene.skybox_points
        self.P = int(row_capacity) if row_capacity else self.N
        if not (0 < self.P <= self.N):
            raise ValueError(f"row_capacity must be in (0, {self.N}]")
        self.bin_capacity, self.sort_capacity = int(bin_capacity), int(sort_capacity)
        f = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)
        self.view, self.proj, self.campos = f(16), f(16), f(3)
        self.bg = bg.to(dev).float().contiguous()
        self.threshold_dev = torch.full((1,), self.threshold, dtype=torch.float32, device=dev)
        self.count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.radii = torch.zeros(self.P, dtype=torch.int32, device=dev)
        self.image = f(3, H, W)
        self.gt = f(3, H, W)
        self.exposure = torch.eye(3, 4, device=dev) if exposure else None
        self.mask = torch.ones((H, W), device=dev) if mask else None
        self.x0 = self.W // 2 if train_test_exp else 0
        self.out_image = f(3, H, self.W - self.x0) if keep_image else None
        self.sums = torch.zeros(4, dtype=torch.float64, device=dev)
        self.results = results if results is not None else torch.zeros((max_frames, _lib.EVAL_ROW), dtype=torch.float64, device=dev)
        self.counter = counter if counter is not None else torch.zeros(1, dtype=torch.int32, device=dev)
        self._warm_counter = torch.zeros(1, dtype=torch.int32, device=dev)          # the eager frame before capture
        self._warm_results = torch.zeros((1, _lib.EVAL_ROW), dtype=torch.float64, device=dev)
        self.lod_scratch = torch.empty(int(self.L.h3dgs_expand_scratch_bytes(self.N_nodes)), dtype=torch.uint8, device=dev)
        self.sky_arange = torch.arange(self.S, dtype=torch.int64, device=dev)
        self._bufs = [None, None, None]
        self._alloc_cb = _lib.ALLOC_FN(self._alloc)
        self.args = self._make_args(tanfovx, tanfovy)
        self._scan_info = None
        self.graph = None
        self.launches_per_frame = 0
        if capture:
            self.capture()

    def _part_eval(self, counter, results):
        _metrics(self.L, self.H, self.W, self.image, self.gt, self.exposure, self.mask, self.x0, self.out_image, self.sums,
                 counter, results, self._stream(), count=self.count, extra_rows=self.S, row_capacity=self.P,
                 scan_info=self.scan_info())

    def capture(self):
        """One eager frame (sizes the state buffers; its row goes to a private slot), then capture of the single graph."""
        s = torch.cuda.Stream(self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            self._part_a()
            self._part_eval(self._warm_counter, self._warm_results)
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        l0 = _lib.launch_count()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._part_a()
            self._part_eval(self.counter, self.results)
        self.launches_per_frame = _lib.launch_count() - l0

    def set_inputs(self, gt=None, mask=None, exposure=None):
        """Copy a frame's target [3,H,W], mask ([1,H,W] or [H,W]) and exposure [3,4] (or larger: the top 3x4 block; None =
        identity) into the static buffers.  Device or pinned host tensors: nothing here waits for the host."""
        if gt is not None:
            self.gt.copy_(gt, non_blocking=True)
        if mask is not None and self.mask is not None:
            self.mask.copy_(mask.reshape(self.H, self.W), non_blocking=True)
        if self.exposure is not None:
            if exposure is None:
                self.exposure.copy_(torch.eye(3, 4, device=self.dev))
            else:
                self.exposure.copy_(exposure[:3, :4], non_blocking=True)

    def frame(self):
        """Render and evaluate one frame with the current inputs: a graph replay (eager when not captured)."""
        if self.graph is None:
            self._part_a()
            self._part_eval(self.counter, self.results)
        else:
            self.graph.replay()


def _stage(t):
    """A per-camera input for copies that never wait for the host: device tensors as they are, host tensors pinned."""
    if t is None or t.is_cuda:
        return t
    return t.float().contiguous().pin_memory()


class HierarchyEvaluator:
    """evaluate_hierarchy in three steps: __init__ learns the capacities and captures one GraphedRender per camera size
    (host synchronisations happen here), enqueue() runs the whole sweep without synchronising the host, finish() reads
    the rows back once, re-runs the flagged frames through the exact path and averages."""

    def __init__(self, scene, cameras, targets, taus, masks=None, exposures=None, train_test_exp=False, keep_images=False,
                 bg=None, sh_degree=3, capacities=None):
        if not scene.hier:
            raise ValueError("evaluate_hierarchy needs a hierarchy scene")
        if len(targets) != len(cameras) or (masks is not None and len(masks) != len(cameras)) or \
                (exposures is not None and len(exposures) != len(cameras)):
            raise ValueError("targets, masks and exposures need one entry per camera")
        self.scene, self.cameras, self.taus = scene, list(cameras), [float(t) for t in taus]
        self.sh_degree, self.train_test_exp, self.keep_images = int(sh_degree), bool(train_test_exp), bool(keep_images)
        dev = scene.means3D.device
        self.dev = dev
        self.bg = torch.zeros(3, device=dev) if bg is None else bg.to(dev).float()
        self.targets = [_stage(t) for t in targets]
        self.masks = None if masks is None else [_stage(m) for m in masks]
        self.exposures = None if exposures is None else [None if e is None else e.to(dev).float() for e in exposures]
        self.n_frames = len(self.cameras) * len(self.taus)
        self.results = torch.zeros((max(self.n_frames, 1), _lib.EVAL_ROW), dtype=torch.float64, device=dev)
        self.counter = torch.zeros(1, dtype=torch.int32, device=dev)
        self.images = [[None] * len(self.cameras) for _ in self.taus] if keep_images else None
        groups = {}
        for ci, cam in enumerate(self.cameras):
            groups.setdefault((cam.W, cam.H, float(cam.tanfovx), float(cam.tanfovy)), []).append(ci)
        self.order = []                                  # (tau index, camera index) in slot order
        self.renders = {}
        for key, cis in groups.items():
            caps = capacities or self._learn_capacities(self.cameras[cis[0]])
            self.renders[key] = self._make(self.cameras[cis[0]], capture=True, **caps)
            for ci in cis:
                self.order += [(ti, ci) for ti in range(len(self.taus))]
        self.frame_of = {k: i for i, k in enumerate(self.order)}

    def _make(self, cam, **kw):
        return GraphedRender(self.scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, self.bg,
                             pipeline.fov_threshold(min(self.taus), cam), sh_degree=self.sh_degree,
                             exposure=self.exposures is not None, mask=self.masks is not None,
                             train_test_exp=self.train_test_exp, keep_image=self.keep_images, results=self.results,
                             counter=self.counter, **kw)

    def _learn_capacities(self, cam):
        """Eager capacity-mode frames of the first view at the smallest and at the largest tau, with every row and a
        modest binning buffer: rows, D and the longest tile list come back in the frame's row even when the binning did
        not fit (then once more with room for D).  Both ends are needed: the finest cut has the most rows, but the
        coarsest has the largest Gaussians and so the most (tile, Gaussian) entries.  Other views may need more than the
        first: capacities = rows x 1.25, D x 1.5 and the next power of two above twice the longest list; a frame that
        still does not fit is re-run exactly."""
        N = self.scene.means3D.shape[0]
        rows = D = longest = 0
        for tau in sorted({min(self.taus), max(self.taus)}):
            bins = 1 << 20
            for _ in range(2):
                probe = GraphedRender(self.scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, self.bg,
                                      pipeline.fov_threshold(tau, cam), sh_degree=self.sh_degree,
                                      bin_capacity=bins, sort_capacity=8192, max_frames=1, capture=False)
                probe.set_camera(cam)
                probe.frame()
                row = probe.results[0].cpu().numpy()
                del probe
                if not row[2]:
                    break
                bins = int(row[4])
            rows, D, longest = max(rows, int(row[3])), max(D, int(row[4])), max(longest, int(row[5]))
        sort_cap = 32
        while sort_cap < min(2 * longest, 8192):
            sort_cap *= 2
        return dict(row_capacity=min(int(rows * 1.25) + 1, N), bin_capacity=int(D * 1.5) + 1, sort_capacity=sort_cap)

    def _render_of(self, cam):
        return self.renders[(cam.W, cam.H, float(cam.tanfovx), float(cam.tanfovy))]

    def enqueue(self):
        """The sweep: per camera, its inputs are copied in once, then one replay per tau.  No host synchronisation."""
        self.counter.zero_()
        last = None
        for ti, ci in self.order:
            cam = self.cameras[ci]
            r = self._render_of(cam)
            if ci != last:
                r.set_camera(cam)
                r.set_inputs(self.targets[ci], None if self.masks is None else self.masks[ci],
                             None if self.exposures is None else self.exposures[ci])
                last = ci
            r.set_threshold(pipeline.fov_threshold(self.taus[ti], cam))
            r.frame()
            if self.keep_images:
                self.images[ti][ci] = r.out_image.clone()

    def _exact(self, ti, ci):
        """One frame through the exact path (host-synchronising LOD cut and num_rendered sizing) and the same metrics
        kernel -> its row (numpy)."""
        from diff_gaussian_rasterization import _C
        cam, r = self.cameras[ci], self._render_of(self.cameras[ci])
        thr = pipeline.fov_threshold(self.taus[ti], cam)
        with torch.no_grad():
            img, _, n = pipeline.render_hier_fused(self.scene, cam, self.bg, thr, self.sh_degree)
        counter = torch.zeros(1, dtype=torch.int32, device=self.dev)
        results = torch.zeros((1, _lib.EVAL_ROW), dtype=torch.float64, device=self.dev)
        out = torch.zeros((3, cam.H, cam.W - r.x0), device=self.dev) if self.keep_images else None
        gt = self.targets[ci].to(self.dev)
        mask = None if self.masks is None else self.masks[ci].to(self.dev).reshape(cam.H, cam.W).contiguous()
        E = None
        if self.exposures is not None:
            E = torch.eye(3, 4, device=self.dev) if self.exposures[ci] is None else self.exposures[ci][:3, :4].contiguous()
        _metrics(r.L, cam.H, cam.W, img.contiguous(), gt.float().contiguous(), E, mask, r.x0, out, r.sums, counter, results,
                 torch.cuda.current_stream(self.dev).cuda_stream, extra_rows=n + self.scene.skybox_points)
        row = results[0].cpu().numpy()
        row[4] = _C.last_num_rendered()
        if self.keep_images:
            self.images[ti][ci] = out
        return row

    def finish(self):
        """-> dict(psnr={tau: mean}, ssim={tau: mean}, rows [n_taus, n_cameras, EVAL_ROW] (numpy; columns psnr, ssim,
        overflow, rows, D, longest tile list), rerun = frames re-run through the exact path, flagged = their
        (tau index, camera index, capacity-mode row) -- what they needed --, images [tau][camera] when keep_images).
        The means are over the cameras, as render_hierarchy.py:111-119 averages them."""
        flat = self.results[:self.n_frames].cpu().numpy()          # the one read-back of the sweep
        rows = np.zeros((len(self.taus), len(self.cameras), _lib.EVAL_ROW))
        for k, (ti, ci) in enumerate(self.order):
            rows[ti, ci] = flat[k]
        flagged = []
        for ti in range(len(self.taus)):
            for ci in range(len(self.cameras)):
                if rows[ti, ci, 2] != 0.0:
                    flagged.append((ti, ci, rows[ti, ci].copy()))
                    rows[ti, ci] = self._exact(ti, ci)
        psnr = {t: float(rows[ti, :, 0].mean()) for ti, t in enumerate(self.taus)}
        ssim = {t: float(rows[ti, :, 1].mean()) for ti, t in enumerate(self.taus)}
        return dict(psnr=psnr, ssim=ssim, rows=rows, rerun=len(flagged), flagged=flagged, images=self.images)


def evaluate_hierarchy(scene, cameras, targets, taus, masks=None, exposures=None, train_test_exp=False, keep_images=False,
                       bg=None, sh_degree=3, capacities=None):
    """The evaluation of render_hierarchy.py (render_set for every tau), sync-free.

    scene: pipeline.Scene with a hierarchy; cameras: pipeline.DeviceCamera per test view; targets: [3,H,W] per camera
    (device, or host: pinned here); masks: [1,H,W] alpha masks per camera or None; exposures: [3,4] per camera (None
    entries = no exposure for that camera, as render_post does for a missing one) or None; train_test_exp: evaluate the
    right half only; capacities: dict(row_capacity, bin_capacity, sort_capacity) instead of the learned ones.
    Per camera and tau the LOD threshold is pipeline.fov_threshold(tau, camera) (render_hierarchy.py:55-56).
    -> see HierarchyEvaluator.finish."""
    ev = HierarchyEvaluator(scene, cameras, targets, taus, masks, exposures, train_test_exp, keep_images, bg, sh_degree,
                            capacities)
    ev.enqueue()
    return ev.finish()
