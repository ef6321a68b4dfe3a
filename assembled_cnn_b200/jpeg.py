"""JPEG decoding on the GPU (acnn_jpeg_parse / acnn_jpeg_plan / acnn_jpeg_decode, include/acnn.h), bit for bit
equal to PIL's `Image.open(b).convert("RGB")`, with PIL as the fallback.

  parse(buffers)             host: one descriptor per encoded image (DESC_DTYPE); `supported` says whether the
                             device decoder handles it, `reason` why not (reason_text)
  jpeg_shape(buf)            (height, width) from the header (tf.image.extract_jpeg_shape)
  JpegDecoder                device buffers reused from batch to batch; decode(buffers, windows) returns one
                             device uint8 [h, w, 3] tensor per image (its window when windows are given)
  decode_jpegs(...)          one-shot JpegDecoder(device).decode(...)

Images the device decoder does not handle (progressive, arithmetic-coded, 12-bit, CMYK, Adobe RGB, other
sampling factors, not JPEG) and images whose scan fails the device's checks (status != 0: an invalid code,
too few bits, a wrong MCU count) are decoded by imagenet_c.decode_rgb (PIL) instead, so their pixels, or
their error, are PIL's.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .imagenet_c import decode_rgb
from .staging import grow, pack_host, pack_u8

DESC_BYTES = 6368
# the head of include/acnn.h acnn_jpeg_desc (the tables follow)
DESC_DTYPE = np.dtype({"names": ["supported", "reason", "height", "width", "ncomp", "hmax", "vmax", "bpm",
                                 "mcus_x", "mcus_y", "restart_interval", "n_intervals", "ecs_offset",
                                 "ecs_length"],
                       "formats": ["<i4"] * 12 + ["<i8"] * 2,
                       "offsets": [4 * k for k in range(12)] + [48, 56],
                       "itemsize": DESC_BYTES})
# include/acnn.h acnn_jpeg_job
JOB_DTYPE = np.dtype([("src", "<i8"), ("out", "<i8"), ("win_y", "<i4"), ("win_x", "<i4"), ("win_h", "<i4"),
                      ("win_w", "<i4"), ("active", "<i4"), ("max_sub", "<i4"), ("mcu_r0", "<i4"),
                      ("mcu_r1", "<i4"), ("mcu_c0", "<i4"), ("mcu_c1", "<i4"), ("stored_blocks", "<i4"),
                      ("idct_blocks", "<i4"), ("offsets", "<i8", (10,))])
assert JOB_DTYPE.itemsize == 144

ST_UNSUPPORTED, ST_BAD_CODE, ST_OUT_OF_BITS, ST_MCU_COUNT = 1, 2, 4, 8


class Batch(C.Structure):
    """struct acnn_jpeg_batch (include/acnn.h)."""
    _fields_ = [("work_bytes", C.c_int64), ("out_bytes", C.c_int64), ("coef_begin", C.c_int64),
                ("coef_end", C.c_int64), ("n", C.c_int32), ("max_sub", C.c_int32),
                ("max_idct_blocks", C.c_int32), ("max_pixels", C.c_int32)]


def reason_text(code):
    return _lib.load().acnn_jpeg_reason(int(code)).decode()


def pack(buffers, out=None):
    """(uint8 array of the buffers back to back, int64 offsets, int64 lengths); `out` (a uint8 array or
    pinned tensor's numpy view) is used when it is large enough."""
    lengths = np.array([len(b) for b in buffers], dtype=np.int64)
    offsets = np.zeros(len(buffers), dtype=np.int64)
    if len(buffers) > 1:
        offsets[1:] = np.cumsum(lengths)[:-1]
    total = int(lengths.sum())
    data = out[:total] if out is not None and len(out) >= total else np.empty(total, dtype=np.uint8)
    for b, o, n in zip(buffers, offsets, lengths):
        data[o:o + n] = np.frombuffer(b, dtype=np.uint8)
    return data, offsets, lengths


def parse_packed(data, offsets, lengths, desc=None):
    """Descriptors (DESC_DTYPE records) of the images packed in `data` (host)."""
    n = len(offsets)
    if desc is None:
        desc = np.zeros(n, dtype=DESC_DTYPE)
    data = np.ascontiguousarray(data)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    lengths = np.ascontiguousarray(lengths, dtype=np.int64)
    _lib.check(_lib.load().acnn_jpeg_parse(data.ctypes.data, offsets.ctypes.data, lengths.ctypes.data, n,
                                           desc.ctypes.data), "acnn_jpeg_parse")
    return desc


def parse(buffers):
    data, offsets, lengths = pack(buffers)
    return parse_packed(data, offsets, lengths)


def jpeg_shape(buf):
    """(height, width) of an encoded image from its frame header (tf.image.extract_jpeg_shape); images the
    parser does not accept fall back to PIL's lazy open, which reads the same header."""
    d = parse([buf])[0]
    if d["supported"]:
        return int(d["height"]), int(d["width"])
    import io
    from PIL import Image
    with Image.open(io.BytesIO(buf)) as im:
        return im.size[1], im.size[0]


def plan(desc, offsets, windows=None):
    """(jobs, Batch) of acnn_jpeg_plan; windows int32 [n, 4] (y, x, h, w) or None for whole images."""
    n = len(desc)
    jobs = np.zeros(n, dtype=JOB_DTYPE)
    batch = Batch()
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    win = None if windows is None else np.ascontiguousarray(windows, dtype=np.int32).reshape(n, 4)
    _lib.check(_lib.load().acnn_jpeg_plan(desc.ctypes.data, offsets.ctypes.data,
                                          None if win is None else win.ctypes.data, n, jobs.ctypes.data,
                                          C.addressof(batch)), "acnn_jpeg_plan")
    return jobs, batch


def _window(a, w):
    if w is None:
        return a
    y, x, h, ww = (int(v) for v in w)
    if not (y >= 0 and x >= 0 and h >= 1 and ww >= 1 and y + h <= a.shape[0] and x + ww <= a.shape[1]):
        raise ValueError("window (%d, %d, %d, %d) outside the %dx%d image" % (y, x, h, ww, a.shape[0], a.shape[1]))
    return np.ascontiguousarray(a[y:y + h, x:x + ww])


class JpegDecoder:
    """Device decoder of batches of encoded images; the host staging and the device buffers grow to the
    largest batch seen and are reused.  One decoder serves one batch at a time: every call synchronises with
    its stream once (to read the per-image status) before it returns, so its pinned host buffers are free
    again, but the device outputs of a call are overwritten by the next call on the same decoder.  A pipeline
    that keeps several batches in flight uses one decoder per batch slot, and makes the stream of a slot's
    next decode wait for the work that reads the slot's previous output."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)
        self._h = {}
        self._d = {}

    def _buf(self, key, nbytes, pin=False):
        store = self._h if pin else self._d
        store[key] = grow(store.get(key), nbytes, self.device, pin)
        return store[key]

    def _enqueue(self, buffers, windows, stream, out=None, out_offsets=None):
        """Pack, parse, plan and enqueue the device decode on `stream` (device buffers are allocated on it, so
        the caching allocator orders their reuse after it).  Returns (desc, jobs, out, status)."""
        n = len(buffers)
        total = sum(len(b) for b in buffers)
        hdata = self._buf("data", total, pin=True)
        data, offsets, lengths = pack(buffers, hdata.numpy())
        hdesc = self._buf("desc", n * DESC_BYTES, pin=True)
        desc = parse_packed(data, offsets, lengths, hdesc[:n * DESC_BYTES].numpy().view(DESC_DTYPE))
        jobs, batch = plan(desc, offsets, windows)
        if out is not None:
            jobs["out"] = out_offsets
            need = out_offsets + jobs["win_h"].astype(np.int64) * jobs["win_w"] * 3 * jobs["active"]
            if int(need.max()) > out.numel() or (out_offsets < 0).any():
                raise ValueError("decode: the outputs do not fit in the given buffer")
        hjobs = self._buf("jobs", n * JOB_DTYPE.itemsize, pin=True)
        hjobs[:n * JOB_DTYPE.itemsize].numpy()[:] = jobs.view(np.uint8)
        with torch.cuda.stream(stream):
            ddata = self._buf("data", max(total, 1))
            ddesc = self._buf("desc", n * DESC_BYTES)
            djobs = self._buf("jobs", n * JOB_DTYPE.itemsize)
            work = self._buf("work", batch.work_bytes)
            if out is None:
                out = self._buf("out", batch.out_bytes)
            status = self._buf("status", 4 * n)[:4 * n].view(torch.int32)
            ddata[:total].copy_(hdata[:total], non_blocking=True)
            ddesc[:n * DESC_BYTES].copy_(hdesc[:n * DESC_BYTES], non_blocking=True)
            djobs[:n * JOB_DTYPE.itemsize].copy_(hjobs[:n * JOB_DTYPE.itemsize], non_blocking=True)
            _lib.check(_lib.load().acnn_jpeg_decode(ddesc.data_ptr(), djobs.data_ptr(), C.addressof(batch),
                                                    ddata.data_ptr(), out.data_ptr(), work.data_ptr(),
                                                    work.numel(), status.data_ptr(), stream.cuda_stream),
                       "acnn_jpeg_decode")
        return desc, jobs, out, status

    def stage(self, buffers, windows=None, stream=None, fallback=None, out=None, out_offsets=None):
        """Decode on `stream`, wait for it, and put every image the device did not decode in device memory
        too.  Returns [(device address, h, w)] of each image's uint8 [h, w, 3] window (of the whole image
        without windows).  fallback(i) gives the uint8 array of image i for the PIL path (default: decode_rgb
        and the window); its errors propagate.  With `out` (a device uint8 tensor) and out_offsets (int64 [n]), the device-decoded images are written there and the others copied there."""
        import io
        stream = stream or torch.cuda.current_stream(self.device)
        desc, jobs, dout, status = self._enqueue(buffers, windows, stream, out, out_offsets)
        with torch.cuda.stream(stream):
            st = status.cpu().numpy()   # synchronises with the stream
        if fallback is None:
            def fallback(i):
                return _window(decode_rgb(io.BytesIO(buffers[i])), None if windows is None else windows[i])
        res, slow = [], {}
        for i in range(len(buffers)):
            if st[i] == 0:
                res.append((dout.data_ptr() + int(jobs[i]["out"]), int(jobs[i]["win_h"]), int(jobs[i]["win_w"])))
            else:
                a = np.ascontiguousarray(fallback(i), dtype=np.uint8)
                slow[i] = a
                res.append((None, a.shape[0], a.shape[1]))
        if slow:
            arrs = list(slow.values())
            with torch.cuda.stream(stream):
                if out is None:
                    self._h["fallback"], self._d["fallback"], base = pack_u8(self._h.get("fallback"),
                                                                             self._d.get("fallback"), arrs, self.device)
                else:
                    self._h["fallback"], offs = pack_host(self._h.get("fallback"), arrs)
                    base = []
                    for i, a, o in zip(slow, arrs, offs):
                        oo = int(out_offsets[i])
                        out[oo:oo + a.nbytes].copy_(self._h["fallback"][o:o + a.nbytes], non_blocking=True)
                        base.append(out.data_ptr() + oo)
                done = torch.cuda.Event()
                done.record(stream)
            done.synchronize()          # the pinned fallback bytes are copied before the next call reuses them
            for (i, a), addr in zip(slow.items(), base):
                res[i] = (addr, a.shape[0], a.shape[1])
        return res

    def enqueue(self, buffers, windows=None, stream=None):
        """Pack, parse, plan and enqueue the device decode without waiting.  Returns (desc, jobs, out, status),
        out and status being device tensors `stream` fills.  Call it again on this decoder only after the
        stream has finished with them (the next call reuses the pinned staging and the device buffers)."""
        return self._enqueue(buffers, windows, stream or torch.cuda.current_stream(self.device))

    def decode(self, buffers, windows=None, stream=None):
        """One device uint8 [h, w, 3] tensor per image: its window when windows (int [n, 4] of (y, x, h, w))
        are given.  Images the device does not decode come from decode_rgb (PIL), which also raises their
        errors."""
        stream = stream or torch.cuda.current_stream(self.device)
        placed = self.stage(buffers, windows, stream)
        flat = self._d.get("out"), self._d.get("fallback")
        res = []
        with torch.cuda.stream(stream):
            for addr, h, w in placed:
                src = next(b for b in flat if b is not None and b.data_ptr() <= addr < b.data_ptr() + b.numel())
                o = addr - src.data_ptr()
                res.append(src[o:o + h * w * 3].view(h, w, 3).clone())
        torch.cuda.current_stream(self.device).wait_stream(stream)
        return res


def decode_jpegs(buffers, windows=None, device="cuda"):
    """Decode encoded images (bytes) into device uint8 [h, w, 3] tensors, on the GPU where the device
    decoder handles them, with PIL otherwise: the same bytes as np.array(Image.open(b).convert("RGB")),
    sliced to windows[i] = (y, x, h, w) when windows are given."""
    return JpegDecoder(device).decode(buffers, windows)
