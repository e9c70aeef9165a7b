"""Host side of the device-driven frame pipeline shared by both colour back-ends (gauss_render.GaussPythonRenderer,
g2pc.rasterizer.GaussianRasterizer).

A "frame" is one camera.  All kernels of a frame are enqueued without waiting; the sizes later kernels need live in a
device-side header (include/g2pc.h, G2PC_HDR_*).  Frames alternate between two slots (scratch buffers + a CUDA stream
each): the front-end of frame f + 1 (projection, depth sort, tile table, multisplit) overlaps the blend of frame f, whose
tail would otherwise idle most SMs; the blend of frame f + 1 waits (event) for the accumulator update of frame f, so
the per-Gaussian accumulators see the cameras in exactly the reference's order (gauss_to_pc.py:437-454).

In async mode the projection (preprocess) of up to `preprocess_cameras` consecutive cameras of one resolution is one
launch, which reads the scene once for the whole batch (csrc/s3_preprocess.cu).  Only what it writes is per camera:
`proj`, `depth_key`, `val` and the node counters, in one of num_slots "batch sets" used in turn (batch b uses set
b % num_slots).  The preprocess runs on a stream of its own, so that it overlaps the blends of the previous batch instead
of queueing behind them; it waits (event) for the end of the last frame of batch b - num_slots, the last reader of its
set.  Sort, tree, multisplit and blend still run one camera at a time in the frame slots.  With preprocess_cameras = 1
the preprocess runs on the frame's own stream, as the first kernel of its front half.

A frame that does not fit the host's buffers lowers the shared failure word on the device: every kernel of that and of
all later frames is a no-op, earlier frames still complete.  The host copies the 64-byte header of every frame to pinned
memory asynchronously and looks at it when the frame's end event has fired (or when a getter calls flush()): on failure it
grows what was too small, resets the word and replays the skipped frames in order.  No call ever waits for a count; the
reference synchronises the device several times per camera (rasterizer_impl.cu:289 blocking D2H, auxiliary.h:178-185
CHECK_CUDA after every stage).
"""
import torch

from . import capi, config


_HDR_POOLS = {}  # device -> free pinned frame headers (cudaHostAlloc is slow: never once per renderer)


def _resolution(camera):
    return int(camera.image_width), int(camera.image_height)


def total_instances(h):
    """(Gaussian, tile) instances of a frame, from its header."""
    return h[capi.HDR_TOTAL_INST] + (h[capi.HDR_TOTAL_INST_HI] << 32)


class FrameQueue:
    """Mixin.  The owner sets self.device, self.lib and self._n (Gaussians), calls _init_frames() and provides:
    self._ensure_buffers(camera, slot) (allocate / grow the slot's scratch on the current stream, the lists through
    _grow_lists), self._enqueue_front(camera, frame, slot, pre) -> device header tensor (pre = (batch set, camera of the
    batch): where _enqueue_preprocess put the camera's projection),
    self._enqueue_back(camera, frame, camera_index, slot), self._fix(header_list) and self._confirm(header_list); and, when
    it projects a batch of cameras in one launch, self._enqueue_preprocess(cameras, batch_set).
    Per-resolution table sets go in self._tables; each holds per-slot tile counters t["slots"][slot]["node_cnt"] (and
    t["pre_cnt"][batch_set][camera] when the owner batches: [0] is the slot's)."""

    def _init_frames(self, preprocess_cameras=1):
        self._frame = 0
        self._pending = []   # (frame, camera, camera_index, pinned header, end-of-frame event)
        self._deferred = []  # (frame, camera, camera_index) submitted in async mode, not yet enqueued
        self._batch = 0
        self.preprocess_cameras = preprocess_cameras
        self._hdr_pool = _HDR_POOLS.setdefault(str(self.device), [])  # pinned headers are shared by all renderers
        self.replays = 0
        self.async_mode = False
        self.num_slots = max(1, int(config.FRAME_SLOTS))
        self._streams = [torch.cuda.Stream(device=self.device) for _ in range(self.num_slots)]
        self._fail = torch.full((1,), -1, dtype=torch.int32, device=self.device)  # 0xFFFFFFFF: no frame has failed
        self._prev_done = None
        # per-frame scratch: one set per slot (frames alternate between the slots); the lists and the multisplit matrix
        # are sized per resolution (_grow_lists)
        dev, m = self.device, max(self._n, 1)
        nbytes = int(self.lib.g2pc_depth_sort_workspace_bytes(m))
        self._slots = [dict(proj=torch.empty((m, 12), dtype=torch.float32, device=dev),
                            depth_key=torch.empty((m,), dtype=torch.int32, device=dev),
                            val=torch.empty((m,), dtype=torch.int64, device=dev),
                            val_sorted=torch.empty((m,), dtype=torch.int64, device=dev),
                            depth_ws=torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=dev),
                            hdr=torch.zeros((capi.HDR_WORDS,), dtype=torch.int32, device=dev),
                            work=torch.zeros((capi.WORK_COUNTERS,), dtype=torch.int32, device=dev),
                            inst_gid=None, matrix=None, ms_ws=None) for _ in range(self.num_slots)]
        # per-camera projection outputs of the batch sets; camera 0 of set s is slot s's own (allocated when first used)
        self._pre_sets = [[sl] + [None] * (preprocess_cameras - 1) for sl in self._slots]
        self._set_free = [None] * self.num_slots  # end event of the last frame that read each batch set
        self._pre_stream = torch.cuda.Stream(device=self.device) if preprocess_cameras > 1 else None
        self._cam_best = torch.zeros((m,), dtype=torch.int64, device=dev)
        self._stats = torch.zeros((capi.STAT_WORDS,), dtype=torch.int64, device=dev)
        # (Gaussian, tile) instances the lists hold, grown when a frame does not fit
        self._inst_cap = max(8 * self._n, 1 << 16)
        # entries of the multisplit's row lists (one per Gaussian and base-level row it covers), grown the same way
        self._row_cap = max(4 * self._n, 1 << 16)
        self._tables = {}
        self._last_slot = 0
        self.last_stats = {}

    def _grow_lists(self, sl, leaf_cap, rows, grid):
        """Grow the slot's depth-ordered lists, multisplit matrix (rows x leaf_cap; 0 rows: none) and the multisplit
        workspace of the base-level grid (grid_w, grid_h) to the current capacities."""
        need = self._inst_cap + 4 * leaf_cap + 64  # lists are padded to 16 bytes; slack for the last TMA unit
        if sl["inst_gid"] is None or sl["inst_gid"].numel() < need:
            sl["inst_gid"] = torch.empty((need,), dtype=torch.int32, device=self.device)
        mneed = rows * leaf_cap
        if mneed > 0 and (sl["matrix"] is None or sl["matrix"].numel() < mneed):
            sl["matrix"] = torch.empty((mneed,), dtype=torch.int32, device=self.device)
        wneed = int(self.lib.g2pc_multisplit_workspace_bytes(max(self._n, 1), self._row_cap, *grid))
        if sl["ms_ws"] is None or sl["ms_ws"].numel() < wneed:
            sl["ms_ws"] = capi.workspace(wneed, self.device)

    def _depth_sort(self, sl, stream, pre=None):
        """Enqueue the depth sort, into the slot's val_sorted, of the (depth key, value) pairs the preprocess wrote into
        `pre` (default: the slot's own)."""
        pre = sl if pre is None else pre
        capi.call("g2pc_depth_sort", capi.ptr(pre["depth_key"]), capi.ptr(pre["val"]), self._n, capi.ptr(sl["val_sorted"]),
                  capi.ptr(sl["depth_ws"]), sl["depth_ws"].numel(), stream)

    def _grow_inst_cap(self, h):
        """A frame's (Gaussian, tile) instances did not fit the lists: raise their capacity (the next _launch_batch grows
        the buffers)."""
        total = total_instances(h)
        if total > 0x7FFFFFFF:
            raise capi.G2pcError(f"{total} (Gaussian, tile) instances in one camera: more than 2^31 - 1")
        self._inst_cap = max(self._inst_cap, int(1.25 * total) + 1024)

    def _grow_row_cap(self, h):
        """A frame's row lists did not fit the multisplit workspace: raise its capacity (the next _launch_batch grows
        the buffers)."""
        need = h[capi.HDR_ROW_INST]
        if need >= 0x7FFFFFFF:
            raise capi.G2pcError("2^31 - 1 or more row-list entries in one camera")
        self._row_cap = max(self._row_cap, min(int(1.25 * need) + 1024, 0x7FFFFFFF))

    def _reset_counts(self):
        """Zero the per-slot tile counters of every table set (a failed frame left its counts behind)."""
        for t in self._tables.values():
            for ts in t["slots"]:
                ts["node_cnt"].zero_()
            for cnts in t.get("pre_cnt", []):
                for c in cnts:
                    c.zero_()

    def executed_pairs(self):
        """(pixel, Gaussian) pairs the blend evaluated since construction: the device counts warp iterations, and a warp
        blends 32 x 4 pixels."""
        self.flush()
        return int(self._stats[capi.STAT_WARP_GAUSSIANS].item()) * 128

    def get_gaussian_colours(self):
        self.flush()
        return self.gaussian_colours * 255

    def _pre_set(self, bset, j):
        """Projection outputs of camera j of batch set bset (allocated on the caller's stream the first time)."""
        sets = self._pre_sets[bset]
        if sets[j] is None:
            m = max(self._n, 1)
            sets[j] = dict(proj=torch.empty((m, 12), dtype=torch.float32, device=self.device),
                           depth_key=torch.empty((m,), dtype=torch.int32, device=self.device),
                           val=torch.empty((m,), dtype=torch.int64, device=self.device))
        return sets[j]

    def _enqueue_preprocess(self, cameras, bset):
        """Owners whose front half projects each camera itself (the CUDA back-end) have nothing to do here."""

    def _launch_batch(self, batch):
        """Enqueue frames [(frame, camera, camera_index)] of one resolution: one preprocess of all their cameras, then
        each frame's front and back halves on its own slot's stream."""
        bset = self._batch % self.num_slots
        self._batch += 1
        # every buffer is allocated on the CALLER's stream (never inside the side-stream context): torch's caching
        # allocator keeps per-stream pools, and a block allocated under a pooled side stream cannot be reused by the next
        # renderer (different stream objects) — the allocator then falls back to cudaMalloc / cudaFree every step
        for j, (frame, camera, _) in enumerate(batch):
            self._ensure_buffers(camera, frame % self.num_slots)
            self._pre_set(bset, j)
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(self.device))  # inputs prepared on the caller's stream
        st0 = self._pre_stream if self._pre_stream is not None else self._streams[batch[0][0] % self.num_slots]
        st0.wait_event(ready)
        if self._set_free[bset] is not None:
            st0.wait_event(self._set_free[bset])
        with torch.cuda.stream(st0):
            self._enqueue_preprocess([camera for _, camera, _ in batch], bset)
        projected = torch.cuda.Event()
        projected.record(st0)
        for j, (frame, camera, camera_index) in enumerate(batch):
            slot = frame % self.num_slots
            st = self._streams[slot]
            if st is not st0:
                st.wait_event(projected)
            with torch.cuda.stream(st):
                dev_hdr = self._enqueue_front(camera, frame, slot, (bset, j))
                hdr = self._hdr_pool.pop() if self._hdr_pool else torch.zeros((capi.HDR_WORDS,), dtype=torch.int32).pin_memory()
                hdr.copy_(dev_hdr, non_blocking=True)
                if self._prev_done is not None:
                    st.wait_event(self._prev_done)  # the accumulators must have seen the previous camera
                self._enqueue_back(camera, frame, camera_index, slot)
                done = torch.cuda.Event()
                done.record(st)
            self._prev_done = done
            self._pending.append((frame, camera, camera_index, hdr, done))
        self._set_free[bset] = self._prev_done

    def _launch_frames(self, frames):
        """Enqueue frames [(frame, camera, camera_index)] in order, in batches of up to preprocess_cameras consecutive
        cameras of one resolution."""
        batch = []
        for item in frames:
            if batch and (len(batch) == self.preprocess_cameras or _resolution(batch[0][1]) != _resolution(item[1])):
                self._launch_batch(batch)
                batch = []
            batch.append(item)
        if batch:
            self._launch_batch(batch)

    def _submit(self, camera, camera_index=None):
        frame = self._frame
        self._frame += 1
        camera_index = frame if camera_index is None else camera_index
        self._deferred.append((frame, camera, camera_index))
        if not self.async_mode:
            self.flush()
        else:
            if len(self._deferred) >= self.preprocess_cameras:
                self._launch_deferred()
            self._poll(block_if_more_than=8)

    def _launch_deferred(self):
        frames, self._deferred = self._deferred, []
        self._launch_frames(frames)

    def _poll(self, block_if_more_than=None):
        while self._pending:
            frame, camera, cidx, hdr, ev = self._pending[0]
            if not ev.query():
                if block_if_more_than is None or len(self._pending) <= block_if_more_than:
                    return
                ev.synchronize()
            h = hdr.tolist()
            if h[capi.HDR_POISON] and h[capi.HDR_POISON] - 1 <= frame:
                self._recover(h)
                continue
            self._confirm(h)
            self._hdr_pool.append(hdr)
            self._pending.pop(0)

    def flush(self):
        """Enqueue the cameras still deferred, wait for every enqueued frame and replay the ones a failed frame skipped."""
        self._launch_deferred()
        while self._pending:
            self._pending[-1][4].synchronize()
            self._poll(block_if_more_than=0)
        if self._prev_done is not None:
            torch.cuda.current_stream(self.device).wait_event(self._prev_done)

    def _all_streams(self):
        return self._streams + ([self._pre_stream] if self._pre_stream is not None else [])

    def _recover(self, h):
        for st in self._all_streams():
            st.synchronize()
        failed = h[capi.HDR_POISON] - 1
        todo = [p for p in self._pending if p[0] >= failed]
        self._pending = [p for p in self._pending if p[0] < failed]
        self._fix(h)  # capacities only; the buffers are re-allocated by the next _launch_batch, on the caller's stream
        self._fail.fill_(-1)
        self._reset_counts()
        torch.cuda.current_stream(self.device).synchronize()
        self.replays += 1
        for (frame, camera, cidx, hdr, ev) in todo:
            self._hdr_pool.append(hdr)
        # the counters were reset: the replayed frames are projected again, batched as on their first launch
        self._launch_frames([(frame, camera, cidx) for (frame, camera, cidx, hdr, ev) in todo])

    def __del__(self):
        try:
            for st in self._all_streams():
                st.synchronize()
        except Exception:
            pass
