#!/usr/bin/env python
"""The device JPEG decoder (acnn_jpeg_decode) on synthetic JPEGs encoded by PIL.

    python tools/bench_jpeg.py [--iters 20] [--warmup 5]

  decode       CUDA-event time of acnn_jpeg_decode alone (data, descriptors and plans already on the device)
               at B = 256 and 512, on 500 x 375 quality-90 4:2:0 sources and on a size mix (160..2000 px
               sides, 4:4:4 / 4:2:2 / 4:2:0 / grayscale, quality 75..95); images/s and compressed MB/s, and
               the host clock of the whole JpegDecoder.decode call (pack, parse, plan, copies, decode, status)
  overlap      the c3 training step (Assemble-ResNet-50, bf16, 224 px, batch 256, mixup type 1) alone, and
               with a B = 512 decode of the next batch enqueued on a second stream just before it: the step's
               time and the time until both are done, alternated in one run
  torchvision  torchvision.io.decode_jpeg(device="cuda") on the same 500 x 375 batch, if importable
Prints the card name, power limit and max SM clock read in the same run, and one JSON line per measurement.
The pipelined training and classification-evaluation loops from encoded records are not measured here."""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200 import _lib, jpeg  # noqa: E402

FLAGS = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
             anti_alias_filter_size=3)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not readable"


def photo(h, w, rng, gray=False):
    """Smooth content with texture: about the entropy of a natural photograph at quality 90."""
    from PIL import Image
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    f = rng.uniform(5, 40, 6)
    a = np.stack([127 + 90 * np.sin(x / f[c] + c) * np.cos(y / f[c + 3] - c) for c in range(3)], -1)
    a = np.clip(a + rng.normal(0, 14, a.shape), 0, 255).astype(np.uint8)
    im = Image.fromarray(a)
    return im.convert("L") if gray else im


def encode(im, **kw):
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def fixed_set(n, rng):
    base = [encode(photo(375, 500, rng), quality=90, subsampling=2) for _ in range(16)]
    return [base[i % 16] for i in range(n)]


def mixed_set(n, rng):
    out = []
    for i in range(n):
        h, w = (int(v) for v in rng.integers(160, 2001, 2))
        mode = i % 4
        im = photo(h, w, rng, gray=mode == 3)
        kw = dict(quality=int(rng.integers(75, 96)))
        if mode < 3:
            kw["subsampling"] = mode
        out.append(encode(im, **kw))
    return out


def event_ms(fn, stream=None):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    fn()
    b.record(stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b)


class Prepared:
    """A batch with its data, descriptors and plans on the device: acnn_jpeg_decode alone can be replayed."""

    def __init__(self, bufs):
        data, offsets, lengths = jpeg.pack(bufs)
        self.desc = jpeg.parse_packed(data, offsets, lengths)
        assert self.desc["supported"].all()
        self.jobs, self.batch = jpeg.plan(self.desc, offsets)
        self.d_data = torch.from_numpy(data).cuda()
        self.d_desc = torch.from_numpy(self.desc.view(np.uint8).copy()).cuda()
        self.d_jobs = torch.from_numpy(self.jobs.view(np.uint8).copy()).cuda()
        self.work = torch.empty(self.batch.work_bytes, dtype=torch.uint8, device="cuda")
        self.out = torch.empty(self.batch.out_bytes, dtype=torch.uint8, device="cuda")
        self.status = torch.empty(len(bufs), dtype=torch.int32, device="cuda")
        self.nbytes = int(lengths.sum())

    def launch(self, stream=None):
        s = stream or torch.cuda.current_stream()
        _lib.check(_lib.load().acnn_jpeg_decode(self.d_desc.data_ptr(), self.d_jobs.data_ptr(),
                                                jpeg.C.addressof(self.batch), self.d_data.data_ptr(),
                                                self.out.data_ptr(), self.work.data_ptr(), self.work.numel(),
                                                self.status.data_ptr(), s.cuda_stream), "acnn_jpeg_decode")


def bench_decode(name, bufs, a):
    p = Prepared(bufs)
    for _ in range(a.warmup):
        p.launch()
    torch.cuda.synchronize()
    assert int(p.status.abs().sum()) == 0
    ms = statistics.median(event_ms(p.launch) for _ in range(a.iters))
    dec = jpeg.JpegDecoder("cuda")
    dec.decode(bufs)
    torch.cuda.synchronize()
    host = []
    for _ in range(max(3, a.iters // 4)):
        t0 = time.perf_counter()
        dec.decode(bufs)
        torch.cuda.synchronize()
        host.append(time.perf_counter() - t0)
    n = len(bufs)
    return {"set": name, "batch": n, "decode_ms": round(ms, 3), "img_s": round(1000.0 * n / ms, 1),
            "MB_s": round(p.nbytes / ms / 1e3, 1), "mean_KB": round(p.nbytes / n / 1e3, 1),
            "wrapper_ms": round(1000 * statistics.median(host), 2),
            "wrapper_img_s": round(n / statistics.median(host), 1), "work_MB": round(p.batch.work_bytes / 1e6, 1)}


def bench_overlap(bufs, a):
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Trainer, build_model
    from assembled_cnn_b200 import imagenet_train as it
    model = build_model(dtype="bf16", **FLAGS)
    p = params_from_flags(batch_size=256, mixup_type=1, label_smoothing=0.1, dtype="bf16", **FLAGS)
    tr = Trainer(model, p, 224, 224)
    n = tr.input_batch
    x = torch.randn(n, 224, 224, 3, device="cuda") * 50
    lab = torch.randint(0, 1001, (n,), dtype=torch.int32, device="cuda")
    lam = it.mixup_lambdas(0, 0, 0, n // 2)
    tr.train_step(x, lab, lam1=lam)
    prep = Prepared(bufs)
    side = torch.cuda.Stream()
    prep.launch(side)
    torch.cuda.synchronize()
    alone, with_dec, both = [], [], []
    for i in range(a.warmup + a.iters):
        s = event_ms(lambda: tr.train_step(x, lab, lam1=lam))
        t0 = time.perf_counter()
        start = torch.cuda.Event(enable_timing=True)
        end = torch.cuda.Event(enable_timing=True)
        start.record()
        side.wait_event(start)
        prep.launch(side)
        tr.train_step(x, lab, lam1=lam)
        end.record()
        torch.cuda.synchronize()
        w = start.elapsed_time(end)
        b = 1000 * (time.perf_counter() - t0)
        if i >= a.warmup:
            alone.append(s)
            with_dec.append(w)
            both.append(b)
    return {"step_alone_ms": round(statistics.median(alone), 3),
            "step_with_decode_ms": round(statistics.median(with_dec), 3),
            "step_and_decode_done_ms": round(statistics.median(both), 3), "decode_batch": len(bufs),
            "decodes_per_s_next_to_step": round(len(bufs) / (statistics.median(both) / 1000), 1)}


def bench_torchvision(bufs, a):
    try:
        import torchvision
        from torchvision.io import decode_jpeg
    except Exception as e:   # noqa: BLE001
        return {"torchvision": "not importable: %s" % type(e).__name__}
    ts = [torch.frombuffer(bytearray(b), dtype=torch.uint8) for b in bufs]
    for _ in range(a.warmup):
        decode_jpeg(ts, device="cuda")
    torch.cuda.synchronize()
    ms = statistics.median(event_ms(lambda: decode_jpeg(ts, device="cuda")) for _ in range(a.iters))
    return {"torchvision": torchvision.__version__, "batch": len(bufs), "decode_ms": round(ms, 3),
            "img_s": round(1000.0 * len(bufs) / ms, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-step", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_jpeg: no CUDA device")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    rng = np.random.default_rng(0)
    fixed = fixed_set(512, rng)
    mixed = mixed_set(512, rng)
    for B in (256, 512):
        print(json.dumps(bench_decode("500x375_q90_420", fixed[:B], a)), flush=True)
        print(json.dumps(bench_decode("size_mix", mixed[:B], a)), flush=True)
    if not a.no_step:
        print(json.dumps(bench_overlap(fixed, a)), flush=True)
    print(json.dumps(bench_torchvision(fixed[:256], a)), flush=True)


if __name__ == "__main__":
    main()
