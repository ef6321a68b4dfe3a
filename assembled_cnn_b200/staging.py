"""Host -> device staging of the input loops (training, classification, retrieval and robustness evaluation).

  grow(buf, nbytes, ...)       a growable uint8 buffer (pinned host or device)
  pack_u8(hbuf, dbuf, ...)     uint8 arrays packed at 16-byte aligned offsets (aligned_offsets) into
                               pinned memory (pack_host), copied to the device
  StagingRing                  pinned host sets and device slots fed on a copy stream, overlapped with the
                               previous batch's device work
  read_ahead(pool, ...)        a thread pool working a fixed number of batches ahead of the consumer
"""
from __future__ import annotations

from collections import deque

import numpy as np
import torch


def grow(buf, nbytes, device=None, pin=False):
    """`buf` when it holds nbytes, else a new uint8 buffer with a quarter to spare (pinned host memory with
    `pin`, else on `device`); None: allocate."""
    if buf is not None and buf.numel() >= nbytes:
        return buf
    n = max(nbytes + nbytes // 4, 4096)
    if pin:
        return torch.empty(n, dtype=torch.uint8, pin_memory=True)
    return torch.empty(n, dtype=torch.uint8, device=device)


def aligned_offsets(arrays):
    """The byte offset of each array packed back to back at 16-byte aligned offsets, then the total."""
    return [int(o) for o in np.cumsum([0] + [(a.nbytes + 15) // 16 * 16 for a in arrays])]


def pack_host(hbuf, arrays):
    """Packs uint8 arrays at aligned_offsets into the pinned host buffer `hbuf` (grown when too small).
    Returns (hbuf, offsets)."""
    offs = aligned_offsets(arrays)
    hbuf = grow(hbuf, offs[-1], pin=True)
    hnp = hbuf.numpy()
    for a, o in zip(arrays, offs):
        hnp[o:o + a.nbytes] = a.reshape(-1)
    return hbuf, offs


def pack_u8(hbuf, dbuf, arrays, device):
    """Packs uint8 arrays at 16-byte aligned offsets into the pinned host buffer `hbuf` and enqueues its copy
    to the device buffer `dbuf` on the current stream; either buffer is replaced by a larger one when it is
    too small (None: allocate).  Returns (hbuf, dbuf, the device address of each array)."""
    hbuf, offs = pack_host(hbuf, arrays)
    dbuf = grow(dbuf, offs[-1], device)
    dbuf[:offs[-1]].copy_(hbuf[:offs[-1]], non_blocking=True)
    return hbuf, dbuf, [dbuf.data_ptr() + o for o in offs[:-1]]


class StagingRing:
    """A ring of RING pinned host sets feeding two device slots on a copy stream, so that a batch's copy
    overlaps the previous batch's device work.  `host` and `slots` are the caller's buffers (any per-set
    tensors); the ring owns the copy stream, the channel-mean tensor, one jpeg.JpegDecoder per slot (made
    on first use) and the events that order the reuse of both:

      push(fill)     waits until host set h's previous copy has run, makes the copy stream wait until the
                     slot's previous batch has been read, runs fill(h, slot) on the copy stream (it fills
                     host set h and enqueues the copies into the slot) and records the slot's `copied` event
      take()         makes the current stream wait for the oldest pushed slot's copies; returns the slot
      release(slot)  once the reads of the slot are enqueued on the current stream: the slot may be refilled
    """

    RING = 3        # pinned host sets

    def __init__(self, dev, host, slots):
        from .imagenet_c import CHANNEL_MEANS
        self.dev, self.host, self.slots = dev, host, slots
        self.mean = torch.tensor(CHANNEL_MEANS, dtype=torch.float32, device=dev)
        self.copy_stream = torch.cuda.Stream(dev)
        self.host_free = [None] * len(host)
        self.slot_free = [None] * len(slots)
        self.copied = [None] * len(slots)
        self.decoders = [None] * len(slots)
        self.pushed = self.taken = 0

    def decoder(self, slot):
        if self.decoders[slot] is None:
            from .jpeg import JpegDecoder
            self.decoders[slot] = JpegDecoder(self.dev)
        return self.decoders[slot]

    def push(self, fill):
        h, slot = self.pushed % len(self.host), self.pushed % len(self.slots)
        self.pushed += 1
        if self.host_free[h] is not None:
            self.host_free[h].synchronize()          # its previous host -> device copy has run
        cs = self.copy_stream
        if self.slot_free[slot] is not None:
            cs.wait_event(self.slot_free[slot])       # the batch before the previous one has read it
        with torch.cuda.stream(cs):
            fill(h, slot)
            ev = torch.cuda.Event()
            ev.record(cs)
        self.host_free[h] = self.copied[slot] = ev

    def take(self):
        slot = self.taken % len(self.slots)
        self.taken += 1
        torch.cuda.current_stream(self.dev).wait_event(self.copied[slot])
        return slot

    def release(self, slot):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.dev))
        self.slot_free[slot] = ev


def read_ahead(pool, batches, submit, ahead=4):
    """Yields (batch, [submit(item) for item in batch]) for each batch (a list of items) of `batches`, in
    order, the items run on `pool`.  While batch j is yielded, batches j+1 .. j+ahead are already submitted;
    `batches` is read only as far as that.  A worker's exception is raised when its batch is reached."""
    batches, end = iter(batches), object()
    pending = deque()

    def queue_next():
        b = next(batches, end)
        if b is not end:
            pending.append((b, [pool.submit(submit, x) for x in b]))

    for _ in range(ahead):
        queue_next()
    while pending:
        b, futs = pending.popleft()
        queue_next()
        yield b, [f.result() for f in futs]
