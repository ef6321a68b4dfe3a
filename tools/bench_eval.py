#!/usr/bin/env python
"""The classification evaluation's device path on synthetic data: Assemble-ResNet-50 (the c3 flags), eval,
bf16, 224 px ('imagenet' preprocessing), 500 x 375 sources (the most common ImageNet validation size), at
B = 128 and 256.

    python tools/bench_eval.py [--batches 128,256] [--iters 20] [--warmup 5] [--decode-images 1024]

Per batch size, CUDA-event times of one batch (median of --iters after --warmup):
  resize       acnn_set_images_resized alone (resize + crop + mean; bytes moved = the source images read
               once + the fp32 output written)
  graph        resize + eval forward + acnn_classify_rows, one CUDA graph replay (what
               model_fns.evaluate_classification replays)
  pipeline     images/s of the pipelined loop of evaluate_classification (pinned ring, copy stream, graph
               replays) over pre-decoded batches, host clock around the loop and a device synchronise
and, separately, the PIL decode rate (images/s) of the CPU thread pool on full-size synthetic 500 x 375
JPEGs, with the core count.  Prints the card name and power limit read in the same run and one JSON line
per measurement."""
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
from assembled_cnn_b200.imagenet_eval import decode_rgb, eval_geometry  # noqa: E402
from assembled_cnn_b200.model_fns import _ClassifyEvalDevice, build_model  # noqa: E402

FLAGS = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
             anti_alias_filter_size=3)
SIZE, SRC = 224, (375, 500)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not readable"


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def bench_batch(model, B, a):
    rng = np.random.default_rng(B)
    geom = eval_geometry(SRC[0], SRC[1], "imagenet", SIZE)
    images = [(rng.integers(0, 256, SRC + (3,), dtype=np.uint8), geom) for _ in range(B)]
    labels = rng.integers(1, 1001, B).tolist()
    ev = _ClassifyEvalDevice(model, B, SIZE, False, True, 0.1, B * (a.warmup + a.iters + 1))
    ev.run_batch(images, labels)                   # eager: loads every kernel, fills slot 0
    torch.cuda.synchronize()
    desc = ev.slots[0][2]
    out = {"resize_ms": timed(lambda: ev.rt.set_images_resized(desc, B, ev.mean), a.warmup, a.iters)}
    graph = ev._graph(0, B)
    out["graph_ms"] = timed(graph.replay, a.warmup, a.iters)
    for _ in range(a.warmup):
        ev.run_batch(images, labels)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.iters):
        ev.run_batch(images, labels)
    torch.cuda.synchronize()
    out["pipeline_img_s"] = a.iters * B / (time.perf_counter() - t0)
    out["graph_img_s"] = 1000.0 * B / out["graph_ms"]
    moved = B * (SRC[0] * SRC[1] * 3 + SIZE * SIZE * 3 * 4)
    out["resize_GB_s"] = moved / out["resize_ms"] / 1e6
    return out


def bench_decode(n, workers):
    from PIL import Image
    rng = np.random.default_rng(0)
    blobs = []
    for _ in range(16):
        img = np.clip(rng.integers(0, 256, 3) + rng.normal(0, 30, SRC + (3,)), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="JPEG", quality=90)
        blobs.append(buf.getvalue())
    with ThreadPoolExecutor(max_workers=workers) as pool:
        list(pool.map(lambda b: decode_rgb(io.BytesIO(b)), blobs))
        t0 = time.perf_counter()
        list(pool.map(lambda i: decode_rgb(io.BytesIO(blobs[i % len(blobs)])), range(n)))
        return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="128,256")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--decode-images", type=int, default=1024)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_eval: no CUDA device")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    model = build_model(**FLAGS)
    for B in (int(b) for b in a.batches.split(",")):
        r = bench_batch(model, B, a)
        print(json.dumps(dict(batch=B, **{k: round(v, 3) for k, v in r.items()})), flush=True)
    cores = len(os.sched_getaffinity(0))
    rate = bench_decode(a.decode_images, min(32, cores))
    print(json.dumps(dict(jpeg_decode_img_s=round(rate, 1), cpu_cores=cores, threads=min(32, cores),
                          image="%dx%d" % (SRC[1], SRC[0]))), flush=True)


if __name__ == "__main__":
    main()
