"""End-to-end detection pipeline from HOST images: the loop of detect.py:104-122 and
val.py:183-207 (pre-process, inference, NMS), software-pipelined:

* `slots` batches are in flight at once, each on its own CUDA stream with its own plan (activation / record buffers, captured
  forward graph) and its own post-process graph.  The conv kernels are persistent one-CTA-per-SM launches whose ramps and tails
  leave SMs idle, and the NMS stage is a chain of small latency-bound kernels: a second batch on another stream fills both
  (tools/time_streams.py compares slot counts).  Results are bit-identical to the blocking calls: the same kernels run on the same data, only
  their interleaving changes.
* the host->device copy of batch i+1 runs on a copy stream while batch i computes (max(2, slots) device input buffers,
  event-ordered), and the device->host copy of batch i's detections is asynchronous, so the host turns batch i-slots into
  per-image tensors while the GPU works on the batches after it (no stream is drained inside the loop)."""
from typing import Iterable, Iterator, List, Optional

import torch

from .general import non_max_suppression_obb


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
