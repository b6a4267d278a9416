"""End-to-end detection pipeline from HOST images: the loop of detect.py:104-122 and
val.py:183-207 (pre-process, inference, NMS), software-pipelined:

* `slots` batches are in flight at once, each on its own CUDA stream with its own plan (activation / record buffers, captured
  forward graph) and its own post-process graph.  The conv kernels are persistent one-CTA-per-SM launches whose ramps and tails
  leave SMs idle, and the NMS stage is a chain of small latency-bound kernels: a second batch on another stream fills both
  (tools/time_streams.py compares slot counts).  Results are bit-identical to the blocking calls: the same kernels run on the same data, only
  their interleaving changes.
* the host->device copy of batch i+1 runs on a copy stream while batch i computes (max(2, slots) device input buffers,
  event-ordered), and the device->host copy of batch i's detections is asynchronous, so the host turns batch i-slots into
  per-image tensors while the GPU works on the batches after it (no stream is drained inside the loop).

`run_images` is the same pipeline for decoded images of any size (detect.py's `LoadImages`, val.py's rect loader): the upload
is the raw packed batch, csrc/letterbox.cu writes the plan's stem input, and the detections come back as polygons in source
pixels (letterbox.py)."""
from typing import Iterable, Iterator, List, NamedTuple, Optional

import torch

from . import letterbox as lb
from .general import DetectRecords, non_max_suppression_obb


class ImageDetections(NamedTuple):
    """What detect.py:129-147 has in hand for one image, as host tensors: `polys` [k, 8] in source-image pixels
    (rbox2poly + scale_polys), `conf` [k], `cls` [k], and `rows` [k, 7] (cx, cy, l, s, theta, conf, cls) in network-input
    pixels; `shapes` is the loader's ((h0, w0), ((h / h0, w / w0), pad)) entry."""
    polys: torch.Tensor
    conf: torch.Tensor
    cls: torch.Tensor
    rows: torch.Tensor
    shapes: tuple


def schedule(i: int, slots: int, n_in: int):
    """Which resources batch i uses: (compute slot, device input buffer, input buffer of batch i+1, pinned result slot).
    The loop below queues batch i AFTER uploading batch i+1 and hands batch i - slots to the caller after queueing batch i, so
    * an input buffer is re-filled only when its previous user (batch i + 1 - n_in <= i - 1) has been queued: n_in >= 2;
    * a pinned result slot is re-filled only when its previous user (batch i - (slots + 1)) has been handed over.
    (tests/test_pipeline_host_cpu.py replays these rules without a GPU.)"""
    return i % slots, i % n_in, (i + 1) % n_in, i % (slots + 1)


class DetectPipeline:
    def __init__(self, model, conf_thres: float = 0.25, iou_thres: float = 0.45, max_det: int = 1500,
                 multi_label: bool = True, classes=None, agnostic: bool = False, device=None, fused_detect: bool = True,
                 slots: int = 2):
        self.model = model
        # fused_detect: Model.detect_records + the post-process on the compact records (the [B, A, no] prediction tensor never
        # crosses HBM); False: Model.forward + non_max_suppression_obb on the tensor, as the two separate reference calls
        self.fused = bool(fused_detect) and hasattr(model, "detect_records")
        self.kw = dict(conf_thres=conf_thres, iou_thres=iou_thres, classes=classes, agnostic=agnostic,
                       multi_label=multi_label, max_det=max_det)
        self.device = torch.device(device) if device is not None else next(model.parameters()).device
        if self.device.type != "cuda":
            raise RuntimeError("DetectPipeline needs a CUDA device; there is no CPU path")
        if int(slots) < 1 or int(slots) > 4:
            raise ValueError("slots must be 1..4")
        # Model.forward (the reference API) has ONE plan per input shape: only the fused entry point takes a slot
        self.slots = int(slots) if self.fused else 1
        # slot 0 with a single slot = the caller's current stream (the behaviour of a plain loop of blocking-free calls)
        self.streams = [torch.cuda.Stream(self.device) for _ in range(self.slots)] if self.slots > 1 else [None]
        self.copy_stream = torch.cuda.Stream(self.device)
        # device input buffers: batch i+1 is uploaded while batch i is being queued, so there are at least two
        self.n_in = max(2, self.slots)
        self._bufs = [None] * self.n_in
        self._copied = [torch.cuda.Event() for _ in range(self.n_in)]
        self._consumed = [torch.cuda.Event() for _ in range(self.n_in)]
        self._reader = [0] * self.n_in          # the slot whose stream read the buffer last
        self._hslots = None
        self._raw_dev = [None] * self.n_in      # run_images: grow-only device / pinned host buffers of the packed batches
        self._raw_host = [None] * self.n_in
        self._raw_hslots = None
        self._next = 0
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    # ------------------------------------------------------------------ device-resident form
    def _stream(self, slot: int):
        return self.streams[slot] if self.streams[slot] is not None else torch.cuda.current_stream(self.device)

    def fork(self) -> None:
        """Order every slot stream after the work queued so far on the caller's current stream."""
        if self.slots == 1:
            return
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        for st in self.streams:
            st.wait_event(ev)

    def join(self) -> None:
        """Order the caller's current stream after everything submitted so far on the slot streams."""
        if self.slots == 1:
            return
        cur = torch.cuda.current_stream(self.device)
        for st in self.streams:
            ev = torch.cuda.Event()
            ev.record(st)
            cur.wait_event(ev)

    def submit(self, x_dev: torch.Tensor, slot: Optional[int] = None):
        """One batch that is already on the device -> (packed [B, max_det, 7], counts int64 [B + 1], cap), device tensors
        (no host read; non_max_suppression_obb's `return_packed="async"` form).  Runs on the slot's stream - round-robin
        when `slot` is None - and the returned tensors stay valid until that slot's next submit.  Bracket a sequence of
        submits with fork() / join() to order it against the caller's stream; x_dev must not be written in between."""
        if slot is None:
            slot = self._next
            self._next = (self._next + 1) % self.slots
        with torch.cuda.stream(self._stream(slot)):
            pred = self.model.detect_records(x_dev, slot=slot) if self.fused else self.model(x_dev)[0]
            return non_max_suppression_obb(pred, return_packed="async", **self.kw)

    # ------------------------------------------------------------------ host-to-host form
    def _host_slot(self, j, B, max_det):
        hs = self._hslots
        if hs is None or hs[0][0].shape[0] != B or hs[0][0].shape[1] != max_det:
            self._hslots = hs = [(torch.empty((B, max_det, 7), dtype=torch.float32).pin_memory(),
                                  torch.empty(B + 1, dtype=torch.int64).pin_memory(), torch.cuda.Event())
                                 for _ in range(self.slots + 1)]
        return hs[j]

    def _upload(self, j: int, x_host: torch.Tensor, first_use: bool) -> None:
        if self._bufs[j] is None or self._bufs[j].shape != x_host.shape or self._bufs[j].dtype != x_host.dtype:
            if not first_use:
                self._stream(self._reader[j]).synchronize()   # (shape change mid-stream: the old buffer may still be read)
            self._bufs[j] = torch.empty(x_host.shape, dtype=x_host.dtype, device=self.device)
            first_use = True
        with torch.cuda.stream(self.copy_stream):
            if not first_use:
                self.copy_stream.wait_event(self._consumed[j])  # the engine finished reading this buffer
            self._bufs[j].copy_(x_host, non_blocking=True)
            self._copied[j].record(self.copy_stream)
        self.h2d_bytes += x_host.numel() * x_host.element_size()

    def __call__(self, host_batches: Iterable[torch.Tensor]) -> Iterator[List[torch.Tensor]]:
        """host_batches: pinned uint8 (0..255) or float (0..1) tensors [B,3,H,W].  Yields, per batch and in order, the list
        of per-image detections [n,7] (cx, cy, l, s, theta, conf, cls) as HOST tensors."""
        it = iter(host_batches)
        cur = next(it, None)
        if cur is None:
            return
        N, NB = self.slots, self.n_in
        used = [False] * NB
        self.fork()
        self._upload(0, cur, True)
        used[0] = True
        i = 0
        pending = []
        while cur is not None:
            slot, j, jn, hs = schedule(i, N, NB)
            nxt = next(it, None)
            if nxt is not None:   # (its previous user, batch i + 1 - NB <= i - 1, has been queued: _consumed[jn] is its event)
                self._upload(jn, nxt, not used[jn])
                used[jn] = True
            compute = self._stream(slot)
            with torch.cuda.stream(compute):
                compute.wait_event(self._copied[j])
                pred = self.model.detect_records(self._bufs[j], slot=slot) if self.fused else self.model(self._bufs[j])[0]
                self._consumed[j].record(compute)  # the layout pass has consumed the input by now (stream order)
                self._reader[j] = slot
                packed, counts, cap = non_max_suppression_obb(pred, return_packed="async", **self.kw)
                # batch i - (N + 1), the previous user of this pinned slot, was handed to the caller before this point
                hout, hcnt, ev = self._host_slot(hs, packed.shape[0], packed.shape[1])
                hout.copy_(packed, non_blocking=True)   # D2H of this batch's result, one copy; nobody waits for it here
                hcnt.copy_(counts, non_blocking=True)
                ev.record(compute)
            self.d2h_bytes += packed.numel() * 4 + counts.numel() * 8
            pending.append((hout, hcnt, ev, cap, cur))
            if len(pending) > N:       # N batches stay queued behind the one the host waits for
                yield self._finish(pending.pop(0))
            cur = nxt
            i += 1
        while pending:
            yield self._finish(pending.pop(0))
        self.join()

    def _finish(self, pending):
        hout, hcnt, ev, cap, x_host = pending
        ev.synchronize()
        c = hcnt.tolist()
        B = len(c) - 1
        if c[B] > cap or c[B] < 0 or any(k < 0 for k in c[:B]):  # rare: more candidates than the optimistic capacity -> re-run, blocking
            torch.cuda.synchronize(self.device)   # the slots' plans are shared with batches in flight: drain them first
            xd = x_host.to(self.device)
            pred = self.model.detect_records(xd) if self.fused else self.model(xd)[0]
            packed, counts = non_max_suppression_obb(pred, return_packed=True, **self.kw)
            host = packed.cpu()
            return [host[b, :k].clone() for b, k in enumerate(counts)]
        return [hout[b, :k].clone() for b, k in enumerate(c[:B])]

    # ------------------------------------------------------------------ decoded images of any size
    def run_images(self, images, img_size: int = 1024, stride: Optional[int] = None, auto: bool = True, batch_size: int = 1,
                   pad: float = 0.0) -> Iterator[ImageDetections]:
        """images: uint8 [H, W, 3] BGR arrays (numpy or CPU tensors, as cv2.imread returns them) of any sizes.  Yields one
        ImageDetections per image, in input order.  Two modes, both the reference's:
        * auto=True, detect.py: each image is letterboxed on its own to the minimum rectangle (INTER_LINEAR, scale-up
          allowed, 114 border up to a multiple of `stride`, by default the model's largest stride as in detect.py:81-82),
          one image per forward (batch_size must be 1), polygons scaled back from the two shapes (detect.py:147).
          `images` may be any iterable.
        * auto=False, val.py's rect loader: `images` is a sequence; the images are sorted by aspect ratio and grouped
          (rect_batch_shapes with `pad`), each resized so that its longer side is img_size (INTER_AREA when shrinking) and
          letterboxed without scale-up into its batch's shape, polygons scaled back with the loader's `shapes` (val.py:232).
        A plan (activations, captured graph) is kept per input shape and slot: a folder of many aspect ratios costs up to
        img_size / stride distinct auto=True shapes (32 at 1024), each planned on first use."""
        if not self.fused:
            raise RuntimeError("run_images runs the fused records plan (fused_detect=True)")
        smax = int(max(self.model.stride))
        img_size, stride, batch_size = int(img_size), smax if stride is None else int(stride), int(batch_size)
        if stride < 1 or stride % smax or img_size < stride or img_size % stride:
            raise RuntimeError(f"img_size ({img_size}) must be a multiple of stride ({stride}), and stride a multiple of the "
                               f"model's largest stride ({smax})")
        if batch_size < 1:
            raise RuntimeError("batch_size must be >= 1")
        if auto:
            if batch_size != 1:
                raise RuntimeError("auto=True letterboxes every image to its own minimum rectangle: batch_size must be 1")

            def batches():
                for k, im in enumerate(images):
                    im = lb.as_image(im)
                    p, (Hp, Wp) = lb.place_detect(im.shape[0], im.shape[1], img_size, stride, True)
                    yield [k], [im], [p], Hp, Wp
        else:
            ims = [lb.as_image(im) for im in images]
            if not ims:
                return
            order, shapes = lb.rect_batch_shapes([(im.shape[1], im.shape[0]) for im in ims], batch_size, img_size, stride, pad)

            def batches():
                for i in range(len(shapes)):
                    idx = [int(k) for k in order[i * batch_size:(i + 1) * batch_size]]
                    Hp, Wp = int(shapes[i][0]), int(shapes[i][1])
                    yield idx, [ims[k] for k in idx], [lb.place_rect(ims[k].shape[0], ims[k].shape[1], img_size, (Hp, Wp))
                                                       for k in idx], Hp, Wp
        ready, nxt_out = {}, 0
        for idx, dets in self._run_raw(batches()):
            ready.update(zip(idx, dets))
            while nxt_out in ready:
                yield ready.pop(nxt_out)
                nxt_out += 1

    def _pack(self, j: int, used: bool, raw):
        idx, ims, places, Hp, Wp = raw
        if used:
            self._copied[j].synchronize()   # the previous upload from this pinned buffer (n_in batches ago) has completed
        batch = lb.pack_batch(ims, places, Hp, Wp, self._raw_host[j])
        self._raw_host[j] = batch.host
        return batch

    def _upload_raw(self, j: int, batch, first_use: bool) -> None:
        buf = self._raw_dev[j]
        if buf is None or buf.numel() < batch.nbytes:
            if buf is not None and not first_use:
                self._stream(self._reader[j]).synchronize()   # (the smaller buffer may still be read)
            buf = self._raw_dev[j] = torch.empty(int(batch.nbytes * 1.25) + 4096, dtype=torch.uint8, device=self.device)
            first_use = True
        with torch.cuda.stream(self.copy_stream):
            if not first_use:
                self.copy_stream.wait_event(self._consumed[j])
            buf[:batch.nbytes].copy_(batch.host[:batch.nbytes], non_blocking=True)
            self._copied[j].record(self.copy_stream)
        self.h2d_bytes += batch.nbytes

    def _raw_host_slot(self, j: int, B: int, max_det: int):
        hs = self._raw_hslots
        if hs is None or hs[0][0].shape[0] < B or hs[0][0].shape[1] != max_det:
            self._raw_hslots = hs = [(torch.empty((B, max_det, 7), dtype=torch.float32).pin_memory(),
                                      torch.empty((B, max_det, 8), dtype=torch.float32).pin_memory(),
                                      torch.empty(B + 1, dtype=torch.int64).pin_memory(), torch.cuda.Event())
                                     for _ in range(self.slots + 1)]
        return hs[j]

    def _detect_raw(self, buf, batch, slot: int):
        """letterbox kernel -> records plan -> (records, per-image (pad_x, pad_y, gain) on the device)."""
        eng = self.model.records_plan((batch.B, 3, batch.Hp, batch.Wp), self.device, slot)
        lb.letterbox_s2d(buf, batch, eng.x_s2d, 1)
        pad_gain = buf[batch.pad_gain_off:batch.pad_gain_off + 12 * batch.B].view(torch.float32)
        return DetectRecords(eng.forward_s2d(), eng.nc), pad_gain

    def _run_raw(self, raw_batches):
        """The loop of __call__ for packed raw batches: yields (input indices, [ImageDetections]) per batch, in batch order."""
        it = iter(raw_batches)
        cur = next(it, None)
        if cur is None:
            return
        N, NB = self.slots, self.n_in
        used = [False] * NB
        self.fork()
        cur_b = self._pack(0, False, cur)
        self._upload_raw(0, cur_b, True)
        used[0] = True
        i = 0
        pending = []
        while cur is not None:
            slot, j, jn, hs = schedule(i, N, NB)
            nxt = next(it, None)
            nxt_b = None
            if nxt is not None:
                nxt_b = self._pack(jn, used[jn], nxt)
                self._upload_raw(jn, nxt_b, not used[jn])
                used[jn] = True
            compute = self._stream(slot)
            B = cur_b.B
            with torch.cuda.stream(compute):
                compute.wait_event(self._copied[j])
                rec, pad_gain = self._detect_raw(self._raw_dev[j], cur_b, slot)
                packed, counts, cap = non_max_suppression_obb(rec, return_packed="async", **self.kw)
                polys = lb.scale_polys_batched(packed, counts, pad_gain)
                self._consumed[j].record(compute)   # (the polygon kernel read the batch's pad / gain table)
                self._reader[j] = slot
                hout, hpoly, hcnt, ev = self._raw_host_slot(hs, B, packed.shape[1])
                hout[:B].copy_(packed, non_blocking=True)
                hpoly[:B].copy_(polys, non_blocking=True)
                hcnt[:B + 1].copy_(counts, non_blocking=True)
                ev.record(compute)
            self.d2h_bytes += packed.numel() * 4 + polys.numel() * 4 + counts.numel() * 8
            pending.append((hout, hpoly, hcnt, ev, cap, cur))
            if len(pending) > N:
                yield self._finish_raw(pending.pop(0))
            cur, cur_b = nxt, nxt_b
            i += 1
        while pending:
            yield self._finish_raw(pending.pop(0))
        self.join()

    def _finish_raw(self, pending):
        hout, hpoly, hcnt, ev, cap, (idx, ims, places, Hp, Wp) = pending
        ev.synchronize()
        B = len(idx)
        c = hcnt[:B + 1].tolist()
        if c[B] > cap or c[B] < 0 or any(k < 0 for k in c[:B]):  # rare: NMS capacity overflow -> re-run, blocking
            torch.cuda.synchronize(self.device)
            batch = lb.pack_batch(ims, places, Hp, Wp)
            buf = batch.host[:batch.nbytes].to(self.device)
            rec, pad_gain = self._detect_raw(buf, batch, 0)
            packed, counts = non_max_suppression_obb(rec, return_packed=True, **self.kw)
            cdev = torch.tensor(counts, dtype=torch.int64).to(self.device)
            hout, hpoly, c = packed.cpu(), lb.scale_polys_batched(packed, cdev, pad_gain).cpu(), counts
        out = []
        for b, k in enumerate(c[:B]):
            rows = hout[b, :k].clone()
            out.append(ImageDetections(hpoly[b, :k].clone(), rows[:, 5], rows[:, 6], rows, places[b].shapes))
        return idx, out
