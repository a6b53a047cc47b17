"""Sync-free training-style step (hierarchy scenes), replayed from two CUDA graphs.

The step of h3dgs.pipeline.l1_step has two host round trips that the reference API forces --
the Python int returned by expand_to_size (train_post.py:91-99) and num_rendered, which sizes
the binning buffer -- plus ~20 kernel launches issued from Python.  On one GPU they hide behind
3 ms of kernels; with the frame sharded over 8 GPUs the kernels take 0.8 ms and the host becomes
the critical path.  Here nothing returns to the host inside the step:

  * h3dgs_lod_cut leaves the cut size on the device and marks the rows after the cut with index -1;
    the rasterizer is handed P = row_capacity rows and skips the marked ones;
  * capacity mode (h3dgs_raster_args.bin_capacity / sort_capacity) sizes the binning state from a
    capacity learned on the first frames instead of from num_rendered;
  * a frame that does not fit (cut > row_capacity, D > bin_capacity, a tile list > sort_capacity)
    raises a device flag, renders the background only and contributes zero gradients; status()
    reports it and the caller re-runs that frame through the exact path (pipeline.l1_step).

Sharded over G > 1 ranks the step has two forms.  peer=False: the image slabs travel in one NCCL all-gather, the
[P,10] gradient sums in one NCCL reduce-scatter (h3dgs.dist).  peer=True (G in {2,4,8} on one NVLink box): the
collectives are fused into the kernels through peer memory (h3dgs.peer, csrc/peer.cu) -- the L1 kernel, which reads a rank's freshly rendered
tile rows anyway, forwards them into the image of every other rank with coalesced 128-bit stores; the backward replay leaves each rank's partial (tile, Gaussian) sums in its
own accumulator, a push kernel stores the partial rows that other ranks own (block-cyclic row ownership) into the owners'
staging areas (coalesced posted stores over NVLink), and the owner's per-Gaussian chain rule (K9) adds the staged rows of
the ranks that touch the Gaussian; the L1 kernel evaluates only the rank's
own tile rows and adds its partial loss into every rank's sum.  What remains are two device-side barrier kernels per
step (start: every rank is done reading its staging area and its image buffer is free; middle of backward:
every rank's replay and push have finished, all pixels and partial rows are in place).

With every size static the step is captured once: graph A = LOD cut + forward (+ the all-gather of
the image slabs when sharded), graph B = L1 loss + its gradient + backward (+ the reduce-scatter of
the [P,10] sums).  The split lets the 25 MB target upload of the end-to-end loop overlap graph A.

The arithmetic is the one of the exact path: same kernels, same order, so images and gradients are
bit-identical to pipeline.l1_step(fused=True) whenever the frame fits.
"""
import ctypes as C
import weakref

import torch
import torch.distributed as dist

from . import _lib
from . import dist as hdist
from ._lib import ptr
from .loss import _coefficients


def _check_index_sizing(n_nodes, rows):
    """h3dgs_lod_cut marks all n_nodes entries of render_indices with -1, and Scene sizes that array by Gaussian rows: a
    hierarchy with more nodes than rows (nodes that hold no Gaussian) would be written past its end."""
    if n_nodes > rows:
        raise ValueError(f"the hierarchy has {n_nodes} nodes but only {rows} Gaussian rows: the device LOD cut needs "
                         "index arrays of one entry per node")


class GraphedBase:
    """What every sync-free form shares whatever it renders: the library handle, the sizes and capacities, the camera
    buffers, the state-buffer callback of the C-ABI, the scan_info view, the flat raster arguments, the two target slots
    with what travels with a target, the forward and backward launches, train_post's objective, capture and replay.

    A subclass provides _part_a() and, when the form has a second graph, _part_b(slot); it sets `args` (_raster_args) and
    status_dev, and allocates what it renders into (image; _init_grads, _init_inputs, _init_post_loss)."""
    exposure, mask_bufs, dinvdepth = None, (None, None), None       # forms without an exposure, a mask, a depth term
    _part_b = None                                                  # forms without a part B: one graph

    def __init__(self, scene, W, H, sh_degree, row_capacity, bin_capacity, sort_capacity):
        self.L = _lib.lib()
        self.scene, self.W, self.H, self.sh_degree = scene, int(W), int(H), int(sh_degree)
        dev = self.dev = scene.means3D.device
        N = self.N = scene.means3D.shape[0]                 # rows of the parameter arrays (hierarchy + skybox)
        self.P = int(row_capacity) if row_capacity else N
        if not (0 < self.P <= N):
            raise ValueError(f"row_capacity must be in (0, {N}]")
        self.bin_capacity, self.sort_capacity = int(bin_capacity), int(sort_capacity)
        f = self._zeros
        self.view, self.proj, self.campos = f(16), f(16), f(3)
        # two target buffers: the upload of the next step's target (25 MB over PCIe, ~1 ms) then overlaps the WHOLE current
        # step instead of only its graph A; graph B is captured once per buffer.  self.gt is buffer 0 (gs.gt.copy_ / step(gt=))
        self.gt_bufs = [f(3, self.H, self.W), f(3, self.H, self.W)]
        self.gt = self.gt_bufs[0]
        self.radii = torch.zeros(self.P, dtype=torch.int32, device=dev)
        self._bufs = [None, None, None]
        # the C-ABI callback reaches this instance through a weak reference: a bound method would make a reference
        # cycle, and an instance in a cycle is freed only by Python's cycle collector -- whenever it happens to run,
        # possibly in the middle of another instance's capture
        me = weakref.ref(self)
        self._alloc_cb = _lib.ALLOC_FN(lambda user, which, nbytes: me()._alloc(user, which, nbytes))
        self._scan_info = None
        self.graph_a = self.graph_b = None
        self.launches_per_step = 0
        self._upload_slot, self._pending = 0, None      # slot the next upload_target() writes; (slot, event) of an upload not yet consumed
        self._done = torch.cuda.Event()                 # recorded after part B of every step
        self._done.record(torch.cuda.current_stream(dev))
        self._slot_done = [torch.cuda.Event(), torch.cuda.Event()]      # recorded after the part B that read slot k: it may be overwritten
        for e in self._slot_done:
            e.record(torch.cuda.current_stream(dev))

    def _zeros(self, *shape):
        return torch.zeros(shape, dtype=torch.float32, device=self.dev)

    def _init_inputs(self, exposure, mask):
        """the exposure (a device [3,4], identity until set) and one alpha-mask plane per target slot (all ones until set),
        for a form built to apply them"""
        self._identity = torch.eye(3, 4, device=self.dev)
        self.exposure = self._identity.clone() if exposure else None
        self.mask_bufs = [torch.ones((self.H, self.W), device=self.dev) for _ in range(2)] if mask else [None, None]
        self.mask = self.mask_bufs[0]

    def _init_grads(self, accum_rows):
        """what the backward reads and writes: dL/dimage (dcolor), the full-size Gaussian gradients, d_means2D and the
        [accum_rows, 10] accumulator of the per-tile replay"""
        f, N = self._zeros, self.N
        self.dcolor = f(3, self.H, self.W)
        self.grads = dict(means3D=f(N, 3), shs=f(N, self.scene.shs.shape[1], 3), opacities=f(N, 1), scales=f(N, 3),
                          rotations=f(N, 4))
        self.d_means2D = f(self.P, 3)
        self.accum = torch.zeros(max(accum_rows, 1) * 10, dtype=torch.float32, device=self.dev)

    def _init_post_loss(self, lambda_dssim, exposure, mask):
        """train_post's objective (csrc/loss.cu's post-loss kernels): the exposure, the mask slots, the sums and derivative
        maps, and the weights of sign(a - gt) and of the SSIM-sum gradient for loss.backward(), formed as the exact path's
        backward (loss.post_loss / single_loss) forms them, so that the graphed dL/dimage equals the eager one bit for bit"""
        self._init_inputs(exposure, mask)
        self.lambda_dssim = float(lambda_dssim)
        self.sums = torch.zeros(2, dtype=torch.float64, device=self.dev)
        self.maps = self._zeros(3, 3, self.H, self.W)
        one, zero = torch.ones((), device=self.dev), torch.zeros((), device=self.dev)
        self.coeffs = _coefficients(one, zero, zero, self.lambda_dssim, float(3 * self.H * self.W))

    # ---- C-ABI plumbing -------------------------------------------------------------------
    def _alloc(self, _user, which, nbytes):
        t = self._bufs[which]
        if t is None or t.numel() < nbytes:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("state buffer grew during capture: run one eager step first")
            t = torch.empty((max(int(nbytes), 1),), dtype=torch.uint8, device=self.dev)
            self._bufs[which] = t
        return t.data_ptr()

    def _stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def scan_info(self):
        """int32 view [D, longest tile list, overflow] inside the image state."""
        if self._scan_info is None:
            v = _lib.StateView()
            b = self._bufs
            _lib.check(self.L.h3dgs_state_layout(self.P, self.W, self.H, self.bin_capacity, b[0].data_ptr(),
                                                 b[1].data_ptr(), b[2].data_ptr(), C.byref(v)))
            off = v.scan_info - b[2].data_ptr()
            self._scan_info = b[2][off:off + 12].view(torch.int32)
        return self._scan_info

    def n_contrib_view(self):
        """int32 view [H*W] of the per-pixel last-contributor index inside the image state (bench bookkeeping:
        its sum is the number of list positions the classic per-pixel formulation walks)."""
        v = _lib.StateView()
        b = self._bufs
        _lib.check(self.L.h3dgs_state_layout(self.P, self.W, self.H, self.bin_capacity, b[0].data_ptr(),
                                             b[1].data_ptr(), b[2].data_ptr(), C.byref(v)))
        off = v.n_contrib - b[2].data_ptr()
        return b[2][off:off + 4 * self.W * self.H].view(torch.int32)

    def _raster_args(self, tanfovx, tanfovy, do_depth=0):
        """h3dgs_raster_args of the whole frame on one GPU, flat: P rows of the scene's arrays, capacity mode"""
        sc = self.scene
        a = _lib.RasterArgs()
        a.P, a.sh_degree, a.sh_coeffs = self.P, self.sh_degree, int(sc.shs.shape[1])
        a.image_width, a.image_height = self.W, self.H
        a.tanfovx, a.tanfovy, a.scale_modifier = float(tanfovx), float(tanfovy), 1.0
        a.prefiltered, a.debug, a.do_depth = 0, 0, int(do_depth)
        a.bg, a.viewmatrix, a.projmatrix, a.campos = ptr(self.bg), ptr(self.view), ptr(self.proj), ptr(self.campos)
        a.means3D, a.shs, a.colors_precomp, a.opacities = ptr(sc.means3D), ptr(sc.shs), None, ptr(sc.opacities)
        a.scales, a.rotations, a.cov3D_precomp = ptr(sc.scales), ptr(sc.rotations), None
        a.shard_count, a.shard_index = 1, 0
        a.bin_capacity, a.sort_capacity = self.bin_capacity, self.sort_capacity
        return a

    # ---- launches shared by the forms (eager or under capture) ----------------------------
    def _forward(self, out, invdepth=None):
        """capacity-mode forward into `out` (None: the peer form's image, see GraphedStep) and `invdepth`"""
        n = C.c_int64(0)
        _lib.check(self.L.h3dgs_rasterize_forward(C.byref(self.args), self._alloc_cb, None, ptr(out), self.radii.data_ptr(),
                                                  ptr(invdepth), C.byref(n), self._stream()))

    def _post_loss(self, slot, exposure_grad=None):
        """train_post's objective against target slot `slot` and its mask: sums, derivative maps and dL/dimage (dcolor);
        with exposure_grad (a device fp64 [3,4]), also dL/dE from the same pass"""
        L, st = self.L, self._stream()
        args = (self.H, self.W, self.image.data_ptr(), self.gt_bufs[slot].data_ptr(), ptr(self.exposure),
                ptr(self.mask_bufs[slot]))
        _lib.check(L.h3dgs_post_loss_forward(*args, self.sums.data_ptr(), self.maps.data_ptr(), st))
        args += (self.maps.data_ptr(), self.coeffs.data_ptr(), self.dcolor.data_ptr())
        if exposure_grad is None:
            _lib.check(L.h3dgs_post_loss_backward(*args, st))
        else:
            _lib.check(L.h3dgs_post_loss_backward_exposure(*args, exposure_grad.data_ptr(), st))

    def _backward(self, phases):
        """h3dgs_rasterize_backward from dcolor (and dinvdepth when the form has it) into grads, d_means2D and accum;
        phases as include/h3dgs.h defines them (3 = the whole backward)"""
        g, b = self.grads, self._bufs
        _lib.check(self.L.h3dgs_rasterize_backward(
            C.byref(self.args), self.radii.data_ptr(), b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), self.bin_capacity,
            self.dcolor.data_ptr(), ptr(self.dinvdepth), g["means3D"].data_ptr(), self.d_means2D.data_ptr(),
            g["shs"].data_ptr(), None, g["opacities"].data_ptr(), g["scales"].data_ptr(), g["rotations"].data_ptr(), None,
            self.accum.data_ptr(), phases, self._stream()))

    # ---- driving --------------------------------------------------------------------------
    def set_camera(self, cam):
        """cam: pipeline.DeviceCamera (device tensors) -- three small device copies."""
        self.view.copy_(cam.viewmatrix.reshape(16), non_blocking=True)
        self.proj.copy_(cam.projmatrix.reshape(16), non_blocking=True)
        self.campos.copy_(cam.campos.reshape(3), non_blocking=True)

    def _set_mask(self, slot, mask):
        """the alpha mask of target slot `slot` ([1,H,W] or [H,W]; None = ones, as the reference's loader falls back to)"""
        if self.mask_bufs[slot] is None:
            if mask is not None:
                raise ValueError("this step was built without a mask (mask=False)")
        elif mask is None:
            self.mask_bufs[slot].fill_(1.0)
        else:
            self.mask_bufs[slot].copy_(mask.reshape(self.H, self.W), non_blocking=True)

    def _set_exposure(self, exposure):
        """this step's [3,4] (or larger: its top 3x4 block) exposure; None = identity, as the renderers do for an image
        without one"""
        if self.exposure is not None:
            self.exposure.copy_(self._identity if exposure is None else exposure.detach()[:3, :4], non_blocking=True)
        elif exposure is not None:
            raise ValueError("this step was built without an exposure (exposure=False)")

    def _fill_slot(self, slot, src, mask=None):
        """what travels with a target into its slot: its alpha mask (subclasses add depth maps, ...)"""
        self.gt_bufs[slot].copy_(src, non_blocking=True)
        self._set_mask(slot, mask)

    def upload_target(self, src, stream, *with_target, **kw):
        """Copy the NEXT step's target (device tensor or pinned host tensor) into one of the two static target slots on
        `stream`, after the last step that read that slot has finished; returns the event to hand to step() as gt_ready
        (step() also picks the slot up by itself).  With two slots the copy overlaps the whole step that is still running
        (and this step's graph A).  with_target: what a subclass keeps beside the target in the slot."""
        slot = self._upload_slot
        self._upload_slot ^= 1
        with torch.cuda.stream(stream):
            stream.wait_event(self._slot_done[slot])
            self._fill_slot(slot, src, *with_target, **kw)
            ready = torch.cuda.Event()
            ready.record(stream)
        self._pending = (slot, ready)
        return ready

    def _warm_up(self):
        """the eager step before the capture, on whatever the input buffers hold.  Its outputs are overwritten by the
        first real step; a subclass whose step accumulates into state that outlives a step keeps that state out of it"""
        self._part_a(); self._part_b(0)

    def capture(self):
        """One eager step (sizes the state buffers, creates the library's side stream), then capture: graph A, and graph B
        once per target buffer."""
        s = torch.cuda.Stream(self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            self._warm_up()
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        l0 = _lib.launch_count()
        self.graph_a = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph_a):
            self._part_a()
        if self._part_b is None:
            self.launches_per_step = _lib.launch_count() - l0
            return
        self.graph_b = [torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()]
        with torch.cuda.graph(self.graph_b[0], pool=self.graph_a.pool()):
            self._part_b(0)
        self.launches_per_step = _lib.launch_count() - l0      # library kernels inside one replay of A + B
        with torch.cuda.graph(self.graph_b[1], pool=self.graph_a.pool()):
            self._part_b(1)

    def step(self, cam=None, gt=None, gt_ready=None):
        """cam/gt: optional new inputs (copied into the static buffers; gt goes into buffer 0).  gt_ready: the event
        upload_target() returned, when the caller uploads the target on another stream: this step then reads the buffer
        that upload wrote."""
        if cam is not None:
            self.set_camera(cam)
        slot = 0
        if gt is not None:
            self.gt_bufs[0].copy_(gt, non_blocking=True)
            self._pending = None
        elif self._pending is not None:
            slot, ev = self._pending
            self._pending = None
            gt_ready = ev if gt_ready is None else gt_ready
        cur = torch.cuda.current_stream(self.dev)
        if self.graph_a is None:
            self._part_a()
            if gt_ready is not None:
                cur.wait_event(gt_ready)
            self._part_b(slot)
        else:
            self.graph_a.replay()
            if gt_ready is not None:
                cur.wait_event(gt_ready)
            self.graph_b[slot].replay()
        self._done.record(cur)
        self._slot_done[slot].record(cur)
        return self.status_dev


class GraphedLodCut(GraphedBase):
    """What the hierarchy forms add: the device LOD cut.  h3dgs_lod_cut reads the threshold from threshold_dev (set_threshold
    changes it between replays), leaves the cut size in `count` on the device and marks the rows after the cut -1; the
    skybox rows follow the cut; the raster arguments carry the fields of the gather and lerp fused into K1.

    budget (opt-in): a Gaussian budget for the cut.  Each cut is then preceded by h3dgs_lod_budget, which writes
    threshold_dev: the finest threshold, no finer than the one set_threshold gives (the floor), whose cut holds at most
    the budget's rows (set_budget changes it between replays); budget_info holds {rows, unmet, nodes at or above the
    floor, rows at the floor}.  The row capacity then defaults to budget + skybox rows.

    cull (opt-in): the view cull.  Each frame then starts with h3dgs_lod_cull_mask, the row mask of the hierarchy rows
    that can reach the camera's image, and the budget (if any) and the cut take only those rows: `count` and
    budget_info's rows are the visible rows, the image is the unculled one bit for bit.  Skybox rows are not culled."""

    def __init__(self, scene, W, H, bg, threshold, sh_degree, row_capacity, bin_capacity, sort_capacity, budget=None,
                 cull=False):
        if not scene.hier:
            raise ValueError(f"{type(self).__name__} drives the hierarchy path (LOD cut + fused gather/lerp)")
        self.N_nodes = scene.nodes.shape[0]
        _check_index_sizing(self.N_nodes, scene.means3D.shape[0])
        if budget is not None and int(budget) < 0:
            raise ValueError("budget must be >= 0")
        if budget is not None and not row_capacity:
            row_capacity = max(1, min(scene.means3D.shape[0], int(budget) + scene.skybox_points))
        super().__init__(scene, W, H, sh_degree, row_capacity, bin_capacity, sort_capacity)
        dev = self.dev
        self.S = scene.skybox_points
        self.bg = bg.to(dev).float().contiguous()
        self.threshold = float(threshold)
        self.threshold_dev = torch.full((1,), self.threshold, dtype=torch.float32, device=dev)   # read by the cut kernels
        self.count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.lod_scratch = torch.empty(int(self.L.h3dgs_expand_scratch_bytes(self.N_nodes)), dtype=torch.uint8, device=dev)
        self.sky_arange = torch.arange(self.S, dtype=torch.int64, device=dev)
        self.budget_dev = None
        if budget is not None:
            self.budget_dev = torch.full((1,), int(budget), dtype=torch.int32, device=dev)
            self.floor_dev = torch.full((1,), self.threshold, dtype=torch.float32, device=dev)
            self.budget_info = torch.zeros(4, dtype=torch.int32, device=dev)
            self.budget_scratch = torch.empty(int(self.L.h3dgs_lod_budget_scratch_bytes(self.N_nodes)), dtype=torch.uint8,
                                              device=dev)
        self.cull_mask = torch.zeros(self.N, dtype=torch.uint8, device=dev) if cull else None

    def _raster_args(self, tanfovx, tanfovy):
        sc = self.scene
        a = super()._raster_args(tanfovx, tanfovy)
        a.interpolation_weights, a.num_node_kids = ptr(sc.interpolation_weights), ptr(sc.num_siblings)
        a.render_indices, a.parent_indices, a.num_source = ptr(sc.render_indices), ptr(sc.parent_indices), self.N
        return a

    def _cut(self):
        sc, m = self.scene, self.cull_mask
        if m is not None:
            a = self.args                               # the rows, camera and sizes K1 draws with
            _lib.check(self.L.h3dgs_lod_cull_mask(self.N_nodes, sc.nodes.data_ptr(), a.means3D, a.scales, a.rotations,
                                                  a.scale_modifier, self.view.data_ptr(), self.proj.data_ptr(),
                                                  a.image_width, a.image_height, a.tanfovx, a.tanfovy, m.data_ptr(),
                                                  self._stream()))
        if self.budget_dev is not None:
            if m is None:
                _lib.check(self.L.h3dgs_lod_budget(self.N_nodes, sc.nodes.data_ptr(), sc.boxes.data_ptr(),
                                                   self.campos.data_ptr(), self.threshold, self.floor_dev.data_ptr(), 0,
                                                   self.budget_dev.data_ptr(), self.threshold_dev.data_ptr(),
                                                   self.budget_info.data_ptr(), self.budget_scratch.data_ptr(), self._stream()))
            else:
                _lib.check(self.L.h3dgs_lod_budget_masked(self.N_nodes, sc.nodes.data_ptr(), sc.boxes.data_ptr(),
                                                          self.campos.data_ptr(), m.data_ptr(), self.threshold,
                                                          self.floor_dev.data_ptr(), 0, self.budget_dev.data_ptr(),
                                                          self.threshold_dev.data_ptr(), self.budget_info.data_ptr(),
                                                          self.budget_scratch.data_ptr(), self._stream()))
        if self.N > self.N_nodes:
            sc.render_indices[self.N_nodes:].fill_(-1)  # the library marks [n, N_nodes); these are the skybox slots beyond
        cut_args = (sc.render_indices.data_ptr(), sc.parent_indices.data_ptr(), sc.nodes_for_render.data_ptr(),
                    sc.interpolation_weights.data_ptr(), sc.num_siblings.data_ptr(), self.count.data_ptr(),
                    self.lod_scratch.data_ptr(), self._stream())
        if m is None:
            _lib.check(self.L.h3dgs_lod_cut(self.N_nodes, sc.nodes.data_ptr(), sc.boxes.data_ptr(), self.threshold,
                                            self.threshold_dev.data_ptr(), self.campos.data_ptr(), *cut_args))
        else:
            _lib.check(self.L.h3dgs_lod_cut_masked(self.N_nodes, sc.nodes.data_ptr(), sc.boxes.data_ptr(), self.threshold,
                                                   self.threshold_dev.data_ptr(), self.campos.data_ptr(), m.data_ptr(),
                                                   *cut_args))
        if self.S:
            # skybox rows follow the cut as their own parents with t = 1, kids = 1 (render_post :220-234);
            # a cut so large that they would not fit is reported as a row overflow by status()
            idx = (self.count.long() + self.sky_arange).clamp_(max=self.N - 1)
            sc.render_indices.index_copy_(0, idx, sc.skybox_inds)
            sc.parent_indices.index_copy_(0, idx, sc.skybox_inds)
            sc.interpolation_weights.index_fill_(0, idx, 1.0)
            sc.num_siblings.index_fill_(0, idx, 1)

    def set_threshold(self, threshold):
        """A new LOD threshold for the next step (train_post.py:66-74 draws one per step); with a budget, the floor."""
        self.threshold = float(threshold)
        (self.threshold_dev if self.budget_dev is None else self.floor_dev).fill_(self.threshold)

    def set_budget(self, budget):
        """A new Gaussian budget for the next cut (a form built with budget=)."""
        if self.budget_dev is None:
            raise ValueError("set_budget needs a form built with budget=")
        if int(budget) < 0:
            raise ValueError("budget must be >= 0")
        self.budget_dev.fill_(int(budget))


class GraphedStep(GraphedLodCut):
    """scene: pipeline.Scene with a hierarchy.  The camera-independent sizes (W, H, tanfov) are fixed per
    instance (launch constants inside the graphs); camera, target and LOD threshold are device-resident
    inputs that change between replays (set_camera, upload_target / step(gt=), set_threshold)."""

    def __init__(self, scene, W, H, tanfovx, tanfovy, bg, threshold, sh_degree=3, row_capacity=None,
                 bin_capacity=1 << 22, sort_capacity=4096, world=1, rank=0, group=None, capture=True, peer=False,
                 cyclic_log2=12, cull=False):
        if cull and int(world) > 1:
            raise ValueError("cull=True runs on one GPU: the multi-GPU forms take the unculled cut")
        super().__init__(scene, W, H, bg, threshold, sh_degree, row_capacity, bin_capacity, sort_capacity, cull=cull)
        self.world, self.rank, self.group = int(world), int(rank), group
        self.peer = bool(peer) and self.world > 1
        if self.peer and (self.world & (self.world - 1) or self.world > _lib.MAX_PEERS):
            raise ValueError("peer mode needs 2, 4 or 8 ranks")
        self.cyclic_log2 = int(cyclic_log2)
        dev, H, W, f = self.dev, self.H, self.W, self._zeros
        self.arena = None
        if self.peer:
            from .peer import PeerArena
            self.arena = PeerArena({"loss": 8, "image": 3 * H * W * 4, "stage": world * max(self.P, 1) * 10 * 4}, world, rank, dev, group)
            self.image = self.arena.tensor("image", torch.float32, (3, H, W))
            self.loss_sum = self.arena.tensor("loss", torch.float64, (1,))
            self._loss_ptrs = (C.c_void_p * world)(*self.arena.ptrs("loss"))
            self._image_ptrs = (C.c_void_p * world)(*self.arena.ptrs("image"))
        elif world > 1:
            rows = hdist.owned_rows(H, world, rank)
            self.rpr = hdist.rows_per_rank(H, world)
            self.slab = f(self.rpr, 3, 16, W)           # own packed slab (padded to the common slab height)
            self.slabs = f(world * self.rpr, 3, 16, W)
            self.rows = rows
        else:
            self.image = f(3, H, W)
        if not self.peer:
            self.loss_sum = torch.zeros(1, dtype=torch.float64, device=dev)
        self.status_dev = torch.zeros(6, dtype=torch.float64, device=dev)
        # peer: local, the partial rows travel through "stage"; NCCL: whole row blocks of the reduce-scatter
        self._init_grads(self.P if self.peer else world * ((self.P + world - 1) // world))
        self.args = self._raster_args(tanfovx, tanfovy)
        if capture:
            self.capture()

    def _raster_args(self, tanfovx, tanfovy):
        a = super()._raster_args(tanfovx, tanfovy)
        a.shard_count, a.shard_index = self.world, self.rank
        a.grad_row_begin, a.grad_row_end = hdist.row_block(self.P, self.world, self.rank) if (self.world > 1 and not self.peer) else (0, 0)
        if self.peer:
            a.peer_count, a.grad_cyclic_log2 = self.world, self.cyclic_log2
            for r in range(self.world):
                # the forward stores only into this rank's own image: the L1 kernel forwards the rows to the peers (coalesced)
                a.peer_image[r] = self.arena.ptr("image", r) if r == self.rank else None
                a.peer_stage[r] = self.arena.ptr("stage", r)
        return a

    # ---- the two halves of the step (eager or under capture) ------------------------------
    def _part_a(self):
        """LOD cut -> forward (-> image all-gather)."""
        if self.peer:
            # every rank has finished its previous step: it no longer reads its staging area (our phase 1 stores into it) or
            # its image buffer (our forward stores into it), and its loss sum is zero again
            self.arena.barrier()
        self._cut()
        self._forward(None if self.peer else (self.slab if self.world > 1 else self.image))
        if self.world > 1 and not self.peer:
            dist.all_gather_into_tensor(self.slabs, self.slab, group=self.group)
            self.image = hdist.unpack(self.slabs.view(self.world, self.rpr, 3, 16, self.W), self.H, self.W, self.world)

    def _part_b(self, slot=0):
        """L1 loss against target buffer `slot`, its gradient, backward (-> exchange of the [P,10] sums between the phases)."""
        L = self.L
        gt = self.gt_bufs[slot]
        # loss = mean |image - gt| and dL/dimage in one pass (csrc/l1_loss.cu); every rank evaluates the full image,
        # so the loss value needs no further exchange
        numel = self.image.numel()
        if self.peer:
            # own tile rows only (they were written locally); the partial sum goes into every rank's loss accumulator
            _lib.check(L.h3dgs_l1_loss_grad_peer(3, self.H, self.W, self.image.data_ptr(), gt.data_ptr(), 1.0 / numel,
                                                 self.world, self.rank, self.dcolor.data_ptr(), self.world, self._loss_ptrs,
                                                 self._image_ptrs, self._stream()))
        else:
            _lib.check(L.h3dgs_l1_loss_grad(3, self.H, self.W, self.image.data_ptr(), gt.data_ptr(), 1.0 / numel, 1, 0,
                                            self.dcolor.data_ptr(), self.loss_sum.data_ptr(), self._stream()))
        if self.world == 1:
            self._backward(3)
        elif self.peer:
            # phase 1 fills this rank's partial sums and pushes the rows other ranks own into their staging areas; after the
            # barrier phase 2 adds, for the rows it owns, what the ranks that touched them have staged: the whole "reduce-scatter"
            # (1 | 4: the zero-fill of the full-size gradients runs beside the replay; 2 | 8: ... and is not repeated)
            self._backward(1 | 4)
            self.arena.barrier()
            self._backward(2 | 8)
        else:
            # rows [P, world*chunk) of accum are zero since construction and never written: the blocks reduce cleanly
            self._backward(1 | 4)
            hdist.reduce_accum(self.accum.view(torch.uint8), self.P, self.world, self.rank, self.group)
            # phase 2 rewrites exactly the own row block of d_means2D; the other rows stay zero since construction
            self._backward(2 | 8)
        # status words (loss, rows needed, D, longest list, overflow flags) by one device thread; peer mode: the loss sum is
        # complete since the mid-backward barrier and is reset here for the next step (ordered before anybody's next L1
        # kernel by the start barrier)
        _lib.check(L.h3dgs_step_status(self.loss_sum.data_ptr(), 1.0 / numel, self.count.data_ptr(), self.S, self.P,
                                       self.scan_info().data_ptr(), 1 if self.peer else 0, self.status_dev.data_ptr(), self._stream()))

    def status(self):
        """One 48-byte read-back: loss, rows needed, D, longest tile list, overflow flags."""
        s = self.status_dev.cpu()
        return dict(loss=float(s[0]), rows=int(s[1]), D=int(s[2]), longest_list=int(s[3]),
                    overflow=bool(s[4] != 0 or s[5] != 0))
