"""Sync-free evaluation of a hierarchy over a tau sweep: the numbers render_hierarchy.py reports (PSNR, SSIM and, given a net, LPIPS over every
test camera at tau in {0, 3, 6, 15}), with every frame replayed from one CUDA graph and one read-back at the end.

The drop-in flow of render_hierarchy.py pays, per frame, two host round trips (the int of expand_to_size; num_rendered
sizing the binning buffer), a .cpu() of the camera centre, ~25 PyTorch kernels of gather and lerp, the exposure matmul,
clamps, crop, mask and the metric reductions with a syncing .double() each.  Here one graph per camera size holds

  * h3dgs_lod_cut with the threshold read on the device, and the skybox rows after the cut (graphstep.GraphedLodCut);
  * the capacity-mode forward with the cut gather and lerp fused into K1;
  * h3dgs_eval_metrics (csrc/metrics.cu): exposure, clamp, train_test_exp crop, alpha mask, per-channel squared error
    and the SSIM map sum in one pass, and a one-thread finisher that stores [psnr, ssim, status words] at a slot taken
    from a device counter.

and, when an LpipsVGG net is given (lpips=),
  * the image side of LPIPS (csrc/lpips.cu): the same exposed, clamped, cropped and masked image through VGG16 on TF32
    tensor cores, compared with the target's taps; the value goes to the frame's slot of a device array.
A second graph per camera size computes the target's taps; it is replayed once per camera, before that camera's taus,
so a sweep of T taus runs T + 1 feature passes per camera where the reference runs 2T.

Camera, target, mask, exposure and threshold are device-resident inputs copied in between replays.  A frame that does not
fit the capacities (cut > row capacity, D > bin capacity, a tile list > sort capacity) is flagged in its row and re-run
through the exact path (pipeline.render_hier_fused + the same metrics and LPIPS kernels) after the read-back.  Writing
PNGs (torchvision) is not part of this module: keep_images returns the images instead.
"""
import numpy as np
import torch

from . import _lib, pipeline
from ._lib import ptr
from .graphstep import GraphedLodCut


def _metrics(L, H, W, image, gt, exposure, mask, x0, out_image, sums, counter, results, stream, count=None, extra_rows=0,
             row_capacity=0, scan_info=None):
    _lib.check(L.h3dgs_eval_metrics(H, W, image.data_ptr(), gt.data_ptr(), ptr(exposure), ptr(mask), x0, ptr(out_image),
                                    sums.data_ptr(), ptr(count), extra_rows, row_capacity, ptr(scan_info),
                                    counter.data_ptr(), results.data_ptr(), results.shape[0], stream))


class GraphedRender(GraphedLodCut):
    """Forward-only counterpart of GraphedStep for hierarchy scenes on one GPU: ONE graph = LOD cut (device threshold) +
    skybox rows + capacity-mode forward + metrics pass.  It shares GraphedStep's plumbing (state buffers, raster
    arguments, the LOD cut, set_camera, set_threshold, scan_info, capture) and allocates no gradient buffers.

    W, H, tanfovx, tanfovy are fixed per instance, and so are whether an exposure and a mask are applied and the
    train_test_exp crop.  Inputs that change between replays: set_camera, set_threshold, and the static buffers
    `gt` [3,H,W], `exposure` [3,4], `mask` [H,W] (set_inputs copies into them).  Outputs: `image` (the raw rasterizer
    output, equal to pipeline.render_hier_fused's image whenever the frame fits), `out_image` [3,H,W-x0] when
    keep_image (exposed, clamped, cropped), and one row per frame in `results` at slot `counter`++.

    lpips: an LpipsVGG net, or None.  With one, target_features() computes the target's taps (a second graph, replayed
    after set_inputs), and each frame also stores its LPIPS at the same slot of `lpips_values`.

    budget: a Gaussian budget (GraphedLodCut): the cut's threshold is then chosen on the device, no finer than the
    threshold (the floor; set_threshold), and each frame also stores [threshold, rows, unmet] at its slot of
    `budget_values`.

    cull: the view-culled cut (GraphedLodCut): the same image, with only the rows that can reach it; the frame's rows
    (and a budget's) are the visible rows."""

    def __init__(self, scene, W, H, tanfovx, tanfovy, bg, threshold, sh_degree=3, row_capacity=None, bin_capacity=1 << 22,
                 sort_capacity=4096, exposure=False, mask=False, train_test_exp=False, keep_image=False, results=None,
                 counter=None, max_frames=1024, capture=True, lpips=None, lpips_values=None, budget=None,
                 budget_values=None, cull=False):
        super().__init__(scene, W, H, bg, threshold, sh_degree, row_capacity, bin_capacity, sort_capacity, budget, cull)
        dev, H, W = self.dev, self.H, self.W
        self.image = self._zeros(3, H, W)
        self._init_inputs(exposure, mask)
        self.x0 = W // 2 if train_test_exp else 0
        self.out_image = self._zeros(3, H, W - self.x0) if keep_image else None
        self.sums = torch.zeros(4, dtype=torch.float64, device=dev)
        self.results = results if results is not None else torch.zeros((max_frames, _lib.EVAL_ROW), dtype=torch.float64, device=dev)
        self.counter = counter if counter is not None else torch.zeros(1, dtype=torch.int32, device=dev)
        self._warm_counter = torch.zeros(1, dtype=torch.int32, device=dev)          # the eager frame before capture
        self._warm_results = torch.zeros((1, _lib.EVAL_ROW), dtype=torch.float64, device=dev)
        self.args = self._raster_args(tanfovx, tanfovy)
        self.lpips, self.graph_t = lpips, None
        if lpips is not None:
            lpips.scratch(H, W - self.x0)
            self.lpips_values = lpips_values if lpips_values is not None else \
                torch.zeros(self.results.shape[0], dtype=torch.float64, device=dev)
            self._warm_lpips = torch.zeros(1, dtype=torch.float64, device=dev)
        if budget is not None:
            self.budget_values = budget_values if budget_values is not None else \
                torch.zeros((self.results.shape[0], 3), dtype=torch.float64, device=dev)
            self._warm_budget = torch.zeros((1, 3), dtype=torch.float64, device=dev)
        if capture:
            self.capture()

    graph = property(lambda self: self.graph_a)                         # the frame's one graph
    launches_per_frame = property(lambda self: self.launches_per_step)

    def _part_a(self, counter=None, results=None):
        """LOD cut -> forward -> metrics pass, whose row goes to slot counter++ of results"""
        self._cut()
        if self.budget_dev is not None:
            rec = torch.cat((self.threshold_dev.double(), self.budget_info[:2].double())).unsqueeze(0)
            (self.budget_values if results is None else self._warm_budget).index_copy_(
                0, (self.counter if counter is None else counter).long(), rec)
        self._forward(self.image)
        _metrics(self.L, self.H, self.W, self.image, self.gt, self.exposure, self.mask, self.x0, self.out_image, self.sums,
                 self.counter if counter is None else counter, self.results if results is None else results, self._stream(),
                 count=self.count, extra_rows=self.S, row_capacity=self.P, scan_info=self.scan_info())
        if self.lpips is not None:
            self.lpips.distance(self.image, self.lpips_values if results is None else self._warm_lpips, self.x0,
                                self.exposure, self.mask, clamp=True, counter=self.counter if counter is None else counter,
                                stream=self._stream())

    def _target(self):
        """the target's LPIPS taps (clamped, cropped, masked)"""
        self.lpips.features(self.gt, self.x0, None, self.mask, clamp=True, stream=self._stream())

    def _warm_up(self):
        """capture()'s eager frame (sizes the state buffers): its row goes to a private slot"""
        if self.lpips is not None:
            self._target()
        self._part_a(self._warm_counter, self._warm_results)

    def capture(self):
        super().capture()
        if self.lpips is not None:
            self.graph_t = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph_t, pool=self.graph_a.pool()):
                self._target()

    def target_features(self):
        """The target's taps from the current inputs, for the frames that follow: a graph replay (eager when not
        captured).  Once per camera, after set_inputs."""
        if self.graph_t is None:
            self._target()
        else:
            self.graph_t.replay()

    def set_inputs(self, gt=None, mask=None, exposure=None):
        """Copy a frame's target [3,H,W], mask ([1,H,W] or [H,W]; None = ones) and exposure [3,4] (or larger: the top 3x4
        block; None = identity) into the static buffers.  Device or pinned host tensors: nothing here waits for the host."""
        if gt is not None:
            self.gt.copy_(gt, non_blocking=True)
        self._set_mask(0, mask)
        self._set_exposure(exposure)

    def frame(self):
        """Render and evaluate one frame with the current inputs: a graph replay (eager when not captured)."""
        if self.graph_a is None:
            self._part_a()
        else:
            self.graph_a.replay()


def _stage(t):
    """A per-camera input for copies that never wait for the host: device tensors as they are, host tensors pinned."""
    if t is None or t.is_cuda:
        return t
    return t.float().contiguous().pin_memory()


class HierarchyEvaluator:
    """evaluate_hierarchy in three steps: __init__ learns the capacities and captures one GraphedRender per camera size
    (host synchronisations happen here), enqueue() runs the whole sweep without synchronising the host, finish() reads
    the rows back once, re-runs the flagged frames through the exact path and averages.

    With budgets (and taus None) the sweep runs over Gaussian budgets instead of taus: each frame's threshold is the finest
    one, no finer than fov_threshold(tau_floor, camera), whose cut holds at most the budget's rows (GraphedRender's
    budget=), and the frame's [threshold, rows, unmet] travel in the same read-back.

    cull: every frame takes the view-culled cut (GraphedRender's cull=): the same images and metrics, and a budget counts
    the visible rows only."""

    def __init__(self, scene, cameras, targets, taus, masks=None, exposures=None, train_test_exp=False, keep_images=False,
                 bg=None, sh_degree=3, capacities=None, lpips=None, budgets=None, tau_floor=0.0, cull=False):
        if not scene.hier:
            raise ValueError("evaluate_hierarchy needs a hierarchy scene")
        if (taus is None) == (budgets is None):
            raise ValueError("give taus or budgets (with tau_floor), not both")
        if budgets is not None and min(budgets, default=0) < 0:
            raise ValueError("budgets must be >= 0")
        if len(targets) != len(cameras) or (masks is not None and len(masks) != len(cameras)) or \
                (exposures is not None and len(exposures) != len(cameras)):
            raise ValueError("targets, masks and exposures need one entry per camera")
        self.scene, self.cameras = scene, list(cameras)
        self.taus = None if taus is None else [float(t) for t in taus]
        self.budgets = None if budgets is None else [int(b) for b in budgets]
        self.tau_floor = float(tau_floor)
        self.cull = bool(cull)
        self.sweep = self.taus if budgets is None else self.budgets       # what a frame's first index runs over
        self.sh_degree, self.train_test_exp, self.keep_images = int(sh_degree), bool(train_test_exp), bool(keep_images)
        dev = scene.means3D.device
        self.dev = dev
        self.bg = torch.zeros(3, device=dev) if bg is None else bg.to(dev).float()
        self.targets = [_stage(t) for t in targets]
        self.masks = None if masks is None else [_stage(m) for m in masks]
        self.exposures = None if exposures is None else [None if e is None else e.to(dev).float() for e in exposures]
        self.n_frames = len(self.cameras) * len(self.sweep)
        self.lpips = lpips
        n = max(self.n_frames, 1)
        # the rows, then one LPIPS value per frame, then [threshold, rows, unmet] per frame of a budget sweep: one
        # read-back for the sweep
        widths = [_lib.EVAL_ROW, 1 if lpips is not None else 0, 3 if budgets is not None else 0]
        self._readback = torch.zeros(n * sum(widths), dtype=torch.float64, device=dev)
        self.results = self._readback[:n * widths[0]].view(n, widths[0])
        self.lpips_values = self._readback[n * widths[0]:n * (widths[0] + widths[1])] if lpips is not None else None
        self.budget_values = self._readback[n * (widths[0] + widths[1]):].view(n, 3) if budgets is not None else None
        self.counter = torch.zeros(1, dtype=torch.int32, device=dev)
        self.images = [[None] * len(self.cameras) for _ in self.sweep] if keep_images else None
        groups = {}
        for ci, cam in enumerate(self.cameras):
            groups.setdefault((cam.W, cam.H, float(cam.tanfovx), float(cam.tanfovy)), []).append(ci)
        self.order = []                                  # (tau or budget index, camera index) in slot order
        self.renders = {}
        for key, cis in groups.items():
            caps = capacities or self._learn_capacities(self.cameras[cis[0]])
            self.renders[key] = self._make(self.cameras[cis[0]], capture=True, **caps)
            for ci in cis:
                self.order += [(ti, ci) for ti in range(len(self.sweep))]
        self.frame_of = {k: i for i, k in enumerate(self.order)}

    def _floor(self, cam):
        """the finest threshold of the sweep: the smallest tau's, or the floor of a budget sweep"""
        return pipeline.fov_threshold(self.tau_floor if self.taus is None else min(self.taus), cam)

    def _make(self, cam, **kw):
        budget = None if self.budgets is None else max(self.budgets)
        return GraphedRender(self.scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, self.bg, self._floor(cam),
                             sh_degree=self.sh_degree, exposure=self.exposures is not None, mask=self.masks is not None,
                             train_test_exp=self.train_test_exp, keep_image=self.keep_images, results=self.results,
                             counter=self.counter, lpips=self.lpips, lpips_values=self.lpips_values, budget=budget,
                             budget_values=self.budget_values, cull=self.cull, **kw)

    def _learn_capacities(self, cam):
        """Eager capacity-mode frames of the first view at the smallest and at the largest tau, with every row and a
        modest binning buffer: rows, D and the longest tile list come back in the frame's row even when the binning did
        not fit (then once more with room for D).  Both ends are needed: the finest cut has the most rows, but the
        coarsest has the largest Gaussians and so the most (tile, Gaussian) entries.  Other views may need more than the
        first: capacities = rows x 1.25, D x 1.5 and the next power of two above twice the longest list; a frame that
        still does not fit is re-run exactly.  A budget sweep probes its smallest and largest budget at the floor; its
        rows are bounded by the largest budget (plus the skybox rows) instead."""
        N = self.scene.means3D.shape[0]
        rows = D = longest = 0
        if self.taus is None:
            ends = [(self._floor(cam), b) for b in sorted({min(self.budgets), max(self.budgets)})]
        else:
            ends = [(pipeline.fov_threshold(tau, cam), None) for tau in sorted({min(self.taus), max(self.taus)})]
        for thr, budget in ends:
            bins = 1 << 20
            for _ in range(2):
                probe = GraphedRender(self.scene, cam.W, cam.H, cam.tanfovx, cam.tanfovy, self.bg, thr,
                                      sh_degree=self.sh_degree, row_capacity=N if budget is not None else None,
                                      bin_capacity=bins, sort_capacity=8192, max_frames=1, capture=False, budget=budget,
                                      cull=self.cull)
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
        row_capacity = min(int(rows * 1.25) + 1, N) if self.taus is not None else \
            max(1, min(N, max(self.budgets) + self.scene.skybox_points))
        return dict(row_capacity=row_capacity, bin_capacity=int(D * 1.5) + 1, sort_capacity=sort_cap)

    def _render_of(self, cam):
        return self.renders[(cam.W, cam.H, float(cam.tanfovx), float(cam.tanfovy))]

    def enqueue(self):
        """The sweep: per camera, its inputs are copied in once, then one replay per tau (or budget).  No host
        synchronisation."""
        self.counter.zero_()
        last = None
        for ti, ci in self.order:
            cam = self.cameras[ci]
            r = self._render_of(cam)
            if ci != last:
                r.set_camera(cam)
                r.set_inputs(self.targets[ci], None if self.masks is None else self.masks[ci],
                             None if self.exposures is None else self.exposures[ci])
                if self.lpips is not None:
                    r.target_features()
                if self.budgets is not None:
                    r.set_threshold(self._floor(cam))
                last = ci
            if self.budgets is None:
                r.set_threshold(pipeline.fov_threshold(self.taus[ti], cam))
            else:
                r.set_budget(self.budgets[ti])
            r.frame()
            if self.keep_images:
                self.images[ti][ci] = r.out_image.clone()

    def _exact(self, ti, ci, thr=None):
        """One frame through the exact path (host-synchronising LOD cut and num_rendered sizing) and the same metrics
        kernel -> its row (numpy), and its LPIPS from the same kernels (None without a net).  thr: the frame's threshold
        (a budget frame's own, as it was chosen on the device), else its tau's."""
        from diff_gaussian_rasterization import _C
        cam, r = self.cameras[ci], self._render_of(self.cameras[ci])
        thr = pipeline.fov_threshold(self.taus[ti], cam) if thr is None else thr
        with torch.no_grad():
            img, _, n = pipeline.render_hier_fused(self.scene, cam, self.bg, thr, self.sh_degree, self.cull)
        counter = torch.zeros(1, dtype=torch.int32, device=self.dev)
        results = torch.zeros((1, _lib.EVAL_ROW), dtype=torch.float64, device=self.dev)
        out = torch.zeros((3, cam.H, cam.W - r.x0), device=self.dev) if self.keep_images else None
        gt = self.targets[ci].to(self.dev)
        mask = None if self.masks is None else self.masks[ci]      # None: no mask, the same as ones
        mask = None if mask is None else mask.to(self.dev).reshape(cam.H, cam.W).contiguous()
        E = None
        if self.exposures is not None:
            E = torch.eye(3, 4, device=self.dev) if self.exposures[ci] is None else self.exposures[ci][:3, :4].contiguous()
        _metrics(r.L, cam.H, cam.W, img.contiguous(), gt.float().contiguous(), E, mask, r.x0, out, r.sums, counter, results,
                 torch.cuda.current_stream(self.dev).cuda_stream, extra_rows=n + self.scene.skybox_points)
        lp = None
        if self.lpips is not None:
            value = torch.zeros(1, dtype=torch.float64, device=self.dev)
            self.lpips.features(gt.float().contiguous(), r.x0, None, mask, clamp=True)
            self.lpips.distance(img.contiguous(), value, r.x0, E, mask, clamp=True, counter=counter)
            lp = float(value.cpu()[0])
        row = results[0].cpu().numpy()
        row[4] = _C.last_num_rendered()
        if self.keep_images:
            self.images[ti][ci] = out
        return row, lp

    def finish(self):
        """-> dict(psnr={tau: mean}, ssim={tau: mean}, rows [n_taus, n_cameras, EVAL_ROW] (numpy; columns psnr, ssim,
        overflow, rows, D, longest tile list), rerun = frames re-run through the exact path, flagged = their
        (tau index, camera index, capacity-mode row) -- what they needed --, images [tau][camera] when keep_images;
        with an LPIPS net also lpips={tau: mean} and lpips_rows [n_taus, n_cameras]).
        The means are over the cameras, as render_hierarchy.py:111-119 averages them.
        A budget sweep keys the means by budget and adds budget_rows [n_budgets, n_cameras, 4]: the threshold chosen,
        its tau (the inverse of fov_threshold), the cut's rows and the unmet flag."""
        n = max(self.n_frames, 1)
        both = self._readback.cpu().numpy()                             # the one read-back of the sweep
        flat = both[:n * _lib.EVAL_ROW].reshape(n, _lib.EVAL_ROW)
        rest = both[n * _lib.EVAL_ROW:]
        K, Cn = len(self.sweep), len(self.cameras)
        if self.lpips is not None:
            lp_flat, rest = rest[:n], rest[n:]
            lp_rows = np.zeros((K, Cn))
        if self.budgets is not None:
            b_flat = rest.reshape(n, 3)
            budget_rows = np.zeros((K, Cn, 4))
        rows = np.zeros((K, Cn, _lib.EVAL_ROW))
        for k, (ti, ci) in enumerate(self.order):
            rows[ti, ci] = flat[k]
            if self.lpips is not None:
                lp_rows[ti, ci] = lp_flat[k]
            if self.budgets is not None:
                cam = self.cameras[ci]
                t = float(np.float32(b_flat[k, 0]))
                budget_rows[ti, ci] = (t, t * (0.5 * cam.W) / (2 * cam.tanfovx) - 0.5, b_flat[k, 1], b_flat[k, 2])
        flagged = []
        for ti in range(K):
            for ci in range(Cn):
                if rows[ti, ci, 2] != 0.0:
                    flagged.append((ti, ci, rows[ti, ci].copy()))
                    thr = None if self.budgets is None else budget_rows[ti, ci, 0]
                    rows[ti, ci], lp = self._exact(ti, ci, thr)
                    if self.lpips is not None:
                        lp_rows[ti, ci] = lp
        psnr = {t: float(rows[ti, :, 0].mean()) for ti, t in enumerate(self.sweep)}
        ssim = {t: float(rows[ti, :, 1].mean()) for ti, t in enumerate(self.sweep)}
        out = dict(psnr=psnr, ssim=ssim, rows=rows, rerun=len(flagged), flagged=flagged, images=self.images)
        if self.lpips is not None:
            out["lpips"] = {t: float(lp_rows[ti].mean()) for ti, t in enumerate(self.sweep)}
            out["lpips_rows"] = lp_rows
        if self.budgets is not None:
            out["budget_rows"] = budget_rows
        return out


def evaluate_hierarchy(scene, cameras, targets, taus=None, masks=None, exposures=None, train_test_exp=False, keep_images=False,
                       bg=None, sh_degree=3, capacities=None, lpips=None, budgets=None, tau_floor=0.0, cull=False):
    """The evaluation of render_hierarchy.py (render_set for every tau), sync-free.

    scene: pipeline.Scene with a hierarchy; cameras: pipeline.DeviceCamera per test view; targets: [3,H,W] per camera
    (device, or host: pinned here); masks: [1,H,W] alpha masks per camera (None entries = ones, the reference loader's
    fallback) or None; exposures: [3,4] per camera (None entries = no exposure for that camera, as render_post does for
    a missing one) or None; train_test_exp: evaluate the right half only; capacities: dict(row_capacity, bin_capacity,
    sort_capacity) instead of the learned ones; lpips: an h3dgs.lpips.LpipsVGG net, to also report LPIPS.  Per camera and tau the LOD threshold is pipeline.fov_threshold(tau, camera) (render_hierarchy.py:55-56).
    budgets (instead of taus): Gaussian budgets of the cut; per camera and budget the threshold is the finest one, no
    finer than fov_threshold(tau_floor, camera), whose cut holds at most that many rows.
    cull: cut only the rows that can reach each camera's image (the same images and metrics; a budget then counts the
    visible rows).
    -> see HierarchyEvaluator.finish."""
    ev = HierarchyEvaluator(scene, cameras, targets, taus, masks, exposures, train_test_exp, keep_images, bg, sh_degree,
                            capacities, lpips, budgets, tau_floor, cull)
    ev.enqueue()
    return ev.finish()
