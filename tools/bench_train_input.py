#!/usr/bin/env python
"""The training input's device path on synthetic data: Assemble-ResNet-50 (the c3 flags: mixup type 1,
label smoothing 0.1, bf16, 224 px, batch 256, so 512 examples per step), crop windows drawn by the training
sampler from 500 x 375 sources.

    python tools/bench_train_input.py [--iters 20] [--warmup 5] [--decode-images 1024]

CUDA-event times (median of --iters after --warmup):
  crop         acnn_crop_resize_u8 alone at B = 256 and 512 (flip + resize + mean; bytes moved = the windows
               read once + the fp32 output written)
  staged step  the training step fed from device-staged windows (acnn_set_images_cropped + graph replay)
               against the same step fed a device-resident fp32 batch (device copy + graph replay),
               alternated in one run
  pipeline     steps/s and images/s of the staging ring (host packing, copy stream, step) over pre-decoded
               windows, host clock around the loop and a device synchronise
and, separately, the PIL decode rate of the CPU thread pool for full-size 500 x 375 JPEGs with random crops
(imagenet_train.decode_window), with the core count.  Prints the card name and power limit read in the same
run and one JSON line per measurement."""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200 import _lib  # noqa: E402
from assembled_cnn_b200 import imagenet_train as it  # noqa: E402
from assembled_cnn_b200.hparams import params_from_flags  # noqa: E402
from assembled_cnn_b200.model_fns import Trainer, _TrainFeed, build_model  # noqa: E402

FLAGS = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
             anti_alias_filter_size=3)
SIZE, SRC, BATCH = 224, (375, 500), 256


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not readable"


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def windows(n, seed):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, 256, SRC + (3,), dtype=np.uint8)
    out = []
    for p in range(n):
        y, x, ch, cw, flip = it.crop_window(SRC[0], SRC[1], it.example_rng(seed, 0, p))
        out.append((np.ascontiguousarray(src[y:y + ch, x:x + cw]), flip))
    return out


def bench_crop(B, a):
    from assembled_cnn_b200.staging import pack_u8
    wins = windows(B, B)
    hbuf, dbuf, addrs = pack_u8(None, None, [w for w, _ in wins], torch.device("cuda"))   # dbuf: the pixels
    desc = np.zeros(B, it.CROP_DESC_DTYPE)
    for i, (w, f) in enumerate(wins):
        desc[i] = (addrs[i], w.shape[0], w.shape[1], int(f), (0, 0, 0))
    ddesc = torch.from_numpy(desc.view(np.uint8).copy()).cuda()
    out = torch.empty(B, SIZE, SIZE, 3, device="cuda")
    mean = torch.tensor(it.CHANNEL_MEANS, device="cuda")
    lib = _lib.load()
    fn = lambda: _lib.check(lib.acnn_crop_resize_u8(ddesc.data_ptr(), B, B, SIZE, mean.data_ptr(), out.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream), "crop")
    for _ in range(a.warmup):
        fn()
    ms = statistics.median(event_ms(fn) for _ in range(a.iters))
    moved = sum(w.nbytes for w, _ in wins) + B * SIZE * SIZE * 3 * 4
    return {"batch": B, "crop_ms": round(ms, 4), "crop_GB_s": round(moved / ms / 1e6, 1)}


def bench_step(a):
    model = build_model(dtype="bf16", **FLAGS)
    p = params_from_flags(batch_size=BATCH, mixup_type=1, label_smoothing=0.1, dtype="bf16", **FLAGS)
    tr = Trainer(model, p, SIZE, SIZE)
    feed = _TrainFeed(tr, False)
    n = tr.input_batch
    batches = [windows(n, s) for s in range(3)]
    labels = np.random.default_rng(0).integers(0, 1001, n).tolist()
    lam = it.mixup_lambdas(0, 0, 0, n // 2)
    x = torch.randn(n, SIZE, SIZE, 3, device="cuda") * 50
    lab = torch.tensor(labels, dtype=torch.int32, device="cuda")
    tr.train_step(x, lab, lam1=lam)                 # capture
    feed.stage(batches[0], labels)
    feed.step(lam)
    torch.cuda.synchronize()
    staged, resident = [], []
    for i in range(a.warmup + a.iters):
        feed.stage(batches[i % 3], labels)
        torch.cuda.synchronize()                    # time the step only, not the copy
        s = event_ms(lambda: feed.step(lam))
        r = event_ms(lambda: tr.train_step(x, lab, lam1=lam))
        if i >= a.warmup:
            staged.append(s)
            resident.append(r)
    out = {"input_batch": n, "staged_step_ms": round(statistics.median(staged), 3),
           "resident_step_ms": round(statistics.median(resident), 3)}
    out["staged_img_s"] = round(1000.0 * BATCH / out["staged_step_ms"], 1)
    out["resident_img_s"] = round(1000.0 * BATCH / out["resident_step_ms"], 1)
    # the pipelined loop: stage step t + 1 while step t runs
    feed.stage(batches[0], labels)
    for i in range(a.warmup):
        feed.step(lam)
        feed.stage(batches[(i + 1) % 3], labels)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(a.iters):
        feed.step(lam)
        feed.stage(batches[(i + 1) % 3], labels)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    out["pipeline_img_s"] = round(a.iters * BATCH / dt, 1)
    return out


def bench_decode(n, workers, tmp):
    from PIL import Image
    rng = np.random.default_rng(0)
    path = os.path.join(tmp, "jpegs.bin")
    spans, blob = [], b""
    for _ in range(16):
        img = np.clip(rng.integers(0, 256, 3) + rng.normal(0, 30, SRC + (3,)), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="JPEG", quality=90)
        spans.append((len(blob), len(buf.getvalue())))
        blob += buf.getvalue()
    with open(path, "wb") as f:
        f.write(blob)
    job = lambda i: it.decode_window(path, *spans[i % 16], 0, 0, i)
    with ThreadPoolExecutor(max_workers=workers) as pool:
        list(pool.map(job, range(32)))
        t0 = time.perf_counter()
        list(pool.map(job, range(n)))
        return n / (time.perf_counter() - t0)


def main():
    import tempfile
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--decode-images", type=int, default=1024)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_train_input: no CUDA device")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    for B in (256, 512):
        print(json.dumps(bench_crop(B, a)), flush=True)
    print(json.dumps(bench_step(a)), flush=True)
    cores = len(os.sched_getaffinity(0))
    with tempfile.TemporaryDirectory() as tmp:
        rate = bench_decode(a.decode_images, min(32, cores), tmp)
    print(json.dumps(dict(jpeg_decode_crop_img_s=round(rate, 1), cpu_cores=cores, threads=min(32, cores),
                          image="%dx%d" % (SRC[1], SRC[0]))), flush=True)


if __name__ == "__main__":
    main()
