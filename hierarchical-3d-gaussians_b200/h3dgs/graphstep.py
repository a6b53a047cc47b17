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

import torch
import torch.distributed as dist

from . import _lib
from . import dist as hdist


def _ptr(t):
    return None if (t is None or t.numel() == 0) else t.data_ptr()


def _check_index_sizing(n_nodes, rows):
    """h3dgs_lod_cut marks all n_nodes entries of render_indices with -1, and Scene sizes that array by Gaussian rows: a
    hierarchy with more nodes than rows (nodes that hold no Gaussian) would be written past its end."""
    if n_nodes > rows:
        raise ValueError(f"the hierarchy has {n_nodes} nodes but only {rows} Gaussian rows: the device LOD cut needs "
                         "index arrays of one entry per node")


class GraphedStep:
    """scene: pipeline.Scene with a hierarchy.  The camera-independent sizes (W, H, tanfov) are fixed per
    instance (launch constants inside the graphs); camera, target and LOD threshold are device-resident
    inputs that change between replays (set_camera, upload_target / step(gt=), set_threshold)."""

    def __init__(self, scene, W, H, tanfovx, tanfovy, bg, threshold, sh_degree=3, row_capacity=None,
                 bin_capacity=1 << 22, sort_capacity=4096, world=1, rank=0, group=None, capture=True, peer=False,
                 cyclic_log2=12):
        if not scene.hier:
            raise ValueError("GraphedStep drives the hierarchy path (LOD cut + fused gather/lerp)")
        self.L = _lib.lib()
        self.scene, self.W, self.H = scene, int(W), int(H)
        self.threshold, self.sh_degree = float(threshold), int(sh_degree)
        self.world, self.rank, self.group = int(world), int(rank), group
        self.peer = bool(peer) and self.world > 1
        if self.peer and (self.world & (self.world - 1) or self.world > _lib.MAX_PEERS):
            raise ValueError("peer mode needs 2, 4 or 8 ranks")
        self.cyclic_log2 = int(cyclic_log2)
        dev = scene.means3D.device
        self.dev = dev
        N = scene.means3D.shape[0]                     # rows of the parameter arrays (hierarchy + skybox)
        self.N = N
        self.N_nodes = scene.nodes.shape[0]
        _check_index_sizing(self.N_nodes, N)
        self.S = scene.skybox_points
        self.P = int(row_capacity) if row_capacity else N
        if not (0 < self.P <= N):
            raise ValueError(f"row_capacity must be in (0, {N}]")
        self.bin_capacity, self.sort_capacity = int(bin_capacity), int(sort_capacity)
        f = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)
        # static inputs
        self.view, self.proj, self.campos = f(16), f(16), f(3)
        self.bg = bg.to(dev).float().contiguous()
        # two target buffers: the upload of the next step's target (25 MB over PCIe, ~1 ms) then overlaps the WHOLE current
        # step instead of only its graph A; graph B is captured once per buffer.  self.gt is buffer 0 (gs.gt.copy_ / step(gt=))
        self.gt_bufs = [f(3, H, W), f(3, H, W)]
        self.gt = self.gt_bufs[0]
        self._upload_slot, self._pending = 0, None          # buffer the next upload_target() writes; (slot, event) of an upload not yet consumed
        self.threshold_dev = torch.full((1,), self.threshold, dtype=torch.float32, device=dev)   # read by the cut kernels
        # static outputs
        self.count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.radii = torch.zeros(self.P, dtype=torch.int32, device=dev)
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
        self.dcolor = f(3, H, W)
        if not self.peer:
            self.loss_sum = torch.zeros(1, dtype=torch.float64, device=dev)
        self.status_dev = torch.zeros(6, dtype=torch.float64, device=dev)
        M = scene.shs.shape[1]
        self.grads = dict(means3D=f(N, 3), shs=f(N, M, 3), opacities=f(N, 1), scales=f(N, 3), rotations=f(N, 4))
        self.d_means2D = f(self.P, 3)
        chunk = (self.P + world - 1) // world
        if self.peer:
            self.accum = torch.zeros(max(self.P, 1) * 10, dtype=torch.float32, device=dev)      # local; partial rows travel through "stage"
        else:
            self.accum = torch.zeros(max(world * chunk, 1) * 10, dtype=torch.float32, device=dev)
        self.lod_scratch = torch.empty(int(self.L.h3dgs_expand_scratch_bytes(self.N_nodes)), dtype=torch.uint8, device=dev)
        self.sky_arange = torch.arange(self.S, dtype=torch.int64, device=dev)
        self._bufs = [None, None, None]
        self._alloc_cb = _lib.ALLOC_FN(self._alloc)     # keep the callback object alive
        self.args = self._make_args(tanfovx, tanfovy)
        self._scan_info = None
        self.graph_a = self.graph_b = None
        self.launches_per_step = 0
        self._done = torch.cuda.Event()                 # recorded after part B of every step
        self._done.record(torch.cuda.current_stream(dev))
        self._slot_done = [torch.cuda.Event(), torch.cuda.Event()]      # recorded after the part B that read buffer k: it may be overwritten
        for e in self._slot_done:
            e.record(torch.cuda.current_stream(dev))
        if capture:
            self.capture()

    # ---- C-ABI plumbing -------------------------------------------------------------------
    def _alloc(self, _user, which, nbytes):
        t = self._bufs[which]
        if t is None or t.numel() < nbytes:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("state buffer grew during capture: run one eager step first")
            t = torch.empty((max(int(nbytes), 1),), dtype=torch.uint8, device=self.dev)
            self._bufs[which] = t
        return t.data_ptr()

    def _make_args(self, tanfovx, tanfovy):
        sc = self.scene
        a = _lib.RasterArgs()
        a.P, a.sh_degree, a.sh_coeffs = self.P, self.sh_degree, int(sc.shs.shape[1])
        a.image_width, a.image_height = self.W, self.H
        a.tanfovx, a.tanfovy, a.scale_modifier = float(tanfovx), float(tanfovy), 1.0
        a.prefiltered, a.debug, a.do_depth = 0, 0, 0
        a.bg, a.viewmatrix, a.projmatrix, a.campos = _ptr(self.bg), _ptr(self.view), _ptr(self.proj), _ptr(self.campos)
        a.means3D, a.shs, a.colors_precomp, a.opacities = _ptr(sc.means3D), _ptr(sc.shs), None, _ptr(sc.opacities)
        a.scales, a.rotations, a.cov3D_precomp = _ptr(sc.scales), _ptr(sc.rotations), None
        a.interpolation_weights, a.num_node_kids = _ptr(sc.interpolation_weights), _ptr(sc.num_siblings)
        a.render_indices, a.parent_indices, a.num_source = _ptr(sc.render_indices), _ptr(sc.parent_indices), self.N
        a.shard_count, a.shard_index = self.world, self.rank
        a.grad_row_begin, a.grad_row_end = hdist.row_block(self.P, self.world, self.rank) if (self.world > 1 and not self.peer) else (0, 0)
        a.bin_capacity, a.sort_capacity = self.bin_capacity, self.sort_capacity
        if self.peer:
            a.peer_count, a.grad_cyclic_log2 = self.world, self.cyclic_log2
            for r in range(self.world):
                # the forward stores only into this rank's own image: the L1 kernel forwards the rows to the peers (coalesced)
                a.peer_image[r] = self.arena.ptr("image", r) if r == self.rank else None
                a.peer_stage[r] = self.arena.ptr("stage", r)
        return a

    def _stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    # ---- the two halves of the step (eager or under capture) ------------------------------
    def _part_a(self):
        """LOD cut -> forward (-> image all-gather)."""
        sc, L = self.scene, self.L
        if self.peer:
            # every rank has finished its previous step: it no longer reads its staging area (our phase 1 stores into it) or
            # its image buffer (our forward stores into it), and its loss sum is zero again
            self.arena.barrier()
        if self.N > self.N_nodes:
            sc.render_indices[self.N_nodes:].fill_(-1)  # the library marks [n, N_nodes); these are the skybox slots beyond
        _lib.check(L.h3dgs_lod_cut(self.N_nodes, sc.nodes.data_ptr(), sc.boxes.data_ptr(), self.threshold,
                                   self.threshold_dev.data_ptr(), self.campos.data_ptr(), sc.render_indices.data_ptr(), sc.parent_indices.data_ptr(),
                                   sc.nodes_for_render.data_ptr(), sc.interpolation_weights.data_ptr(),
                                   sc.num_siblings.data_ptr(), self.count.data_ptr(), self.lod_scratch.data_ptr(),
                                   self._stream()))
        if self.S:
            # skybox rows follow the cut as their own parents with t = 1, kids = 1 (render_post :220-234);
            # a cut so large that they would not fit is reported as a row overflow by status()
            idx = (self.count.long() + self.sky_arange).clamp_(max=self.N - 1)
            sc.render_indices.index_copy_(0, idx, sc.skybox_inds)
            sc.parent_indices.index_copy_(0, idx, sc.skybox_inds)
            sc.interpolation_weights.index_fill_(0, idx, 1.0)
            sc.num_siblings.index_fill_(0, idx, 1)
        out = None if self.peer else (self.slab if self.world > 1 else self.image)
        n = C.c_int64(0)
        _lib.check(L.h3dgs_rasterize_forward(C.byref(self.args), self._alloc_cb, None, _ptr(out),
                                             self.radii.data_ptr(), None, C.byref(n), self._stream()))
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
        g = self.grads
        outs = (g["means3D"].data_ptr(), self.d_means2D.data_ptr(), g["shs"].data_ptr(), None, g["opacities"].data_ptr(),
                g["scales"].data_ptr(), g["rotations"].data_ptr(), None)
        state = (self.radii.data_ptr(), self._bufs[0].data_ptr(), self._bufs[1].data_ptr(), self._bufs[2].data_ptr(),
                 self.bin_capacity, self.dcolor.data_ptr(), None)
        if self.world == 1:
            _lib.check(L.h3dgs_rasterize_backward(C.byref(self.args), *state, *outs, self.accum.data_ptr(), 3, self._stream()))
        elif self.peer:
            # phase 1 fills this rank's partial sums and pushes the rows other ranks own into their staging areas; after the
            # barrier phase 2 adds, for the rows it owns, what the ranks that touched them have staged: the whole "reduce-scatter"
            # (1 | 4: the zero-fill of the full-size gradients runs beside the replay; 2 | 8: ... and is not repeated)
            _lib.check(L.h3dgs_rasterize_backward(C.byref(self.args), *state, *outs, self.accum.data_ptr(), 1 | 4, self._stream()))
            self.arena.barrier()
            _lib.check(L.h3dgs_rasterize_backward(C.byref(self.args), *state, *outs, self.accum.data_ptr(), 2 | 8, self._stream()))
        else:
            # rows [P, world*chunk) of accum are zero since construction and never written: the blocks reduce cleanly
            _lib.check(L.h3dgs_rasterize_backward(C.byref(self.args), *state, *outs, self.accum.data_ptr(), 1 | 4, self._stream()))
            hdist.reduce_accum(self.accum.view(torch.uint8), self.P, self.world, self.rank, self.group)
            # phase 2 rewrites exactly the own row block of d_means2D; the other rows stay zero since construction
            _lib.check(L.h3dgs_rasterize_backward(C.byref(self.args), *state, *outs, self.accum.data_ptr(), 2 | 8, self._stream()))
        # status words (loss, rows needed, D, longest list, overflow flags) by one device thread; peer mode: the loss sum is
        # complete since the mid-backward barrier and is reset here for the next step (ordered before anybody's next L1
        # kernel by the start barrier)
        _lib.check(L.h3dgs_step_status(self.loss_sum.data_ptr(), 1.0 / numel, self.count.data_ptr(), self.S, self.P,
                                       self.scan_info().data_ptr(), 1 if self.peer else 0, self.status_dev.data_ptr(), self._stream()))

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

    # ---- driving --------------------------------------------------------------------------
    def set_camera(self, cam):
        """cam: pipeline.DeviceCamera (device tensors) -- three small device copies."""
        self.view.copy_(cam.viewmatrix.reshape(16), non_blocking=True)
        self.proj.copy_(cam.projmatrix.reshape(16), non_blocking=True)
        self.campos.copy_(cam.campos.reshape(3), non_blocking=True)

    def set_threshold(self, threshold):
        """A new LOD threshold for the next step (train_post.py:66-74 draws one per step)."""
        self.threshold = float(threshold)
        self.threshold_dev.fill_(self.threshold)

    def upload_target(self, src, stream):
        """Copy the NEXT step's target (device tensor or pinned host tensor) into one of the two static target buffers on
        `stream`, after the last step that read that buffer has finished; returns the event to hand to step() as gt_ready.
        With two buffers the copy overlaps the whole step that is still running (and this step's graph A)."""
        slot = self._upload_slot
        self._upload_slot ^= 1
        with torch.cuda.stream(stream):
            stream.wait_event(self._slot_done[slot])
            self.gt_bufs[slot].copy_(src, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(stream)
        self._pending = (slot, ready)
        return ready

    def capture(self):
        """One eager step (sizes the state buffers, creates the library's side stream), then capture: graph A, and graph B
        once per target buffer."""
        s = torch.cuda.Stream(self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            self._part_a(); self._part_b(0)
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        l0 = _lib.launch_count()
        self.graph_a = torch.cuda.CUDAGraph()
        self.graph_b = [torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()]
        with torch.cuda.graph(self.graph_a):
            self._part_a()
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

    def status(self):
        """One 48-byte read-back: loss, rows needed, D, longest tile list, overflow flags."""
        s = self.status_dev.cpu()
        return dict(loss=float(s[0]), rows=int(s[1]), D=int(s[2]), longest_list=int(s[3]),
                    overflow=bool(s[4] != 0 or s[5] != 0))
