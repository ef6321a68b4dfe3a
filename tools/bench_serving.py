#!/usr/bin/env python
"""The exported servable's binary input (model_fns.Servable.predict) on synthetic 500 x 375 JPEGs, bf16, 224 px
('imagenet' preprocessing), max_batch 256, for Assemble-ResNet-50 (the c3 flags) and vanilla ResNet-50 (c1):

    python tools/bench_serving.py [--repeats 10] [--warmup 3] [--iters 20]

Per model:
  predict   one whole predict(list of n encoded images) call at n = 1, 8, 64, 256: the host's JPEG parse,
            device decode, resize + crop + mean, the eval forward and acnn_predict_rows (one CUDA graph per
            (slot, valid rows)), the copy of the valid rows to the host and the numpy outputs; host clock,
            median of --repeats calls after --warmup calls of the same n
  graph     the graph replay alone at 256 rows (resize -> forward -> acnn_predict_rows), CUDA-event median of
            --iters after --warmup
and acnn_predict_rows alone at B = 256, NC = 1001 (rows 1024 floats apart, as a model's logits view):
CUDA-event median over --iters replays of a graph of 100 launches, divided by 100.  Prints the card name, power limit and max SM clock
read in the same run and one JSON line per measurement."""
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
from assembled_cnn_b200.metrics import predict_rows  # noqa: E402
from assembled_cnn_b200.model_fns import Servable, build_model  # noqa: E402

MODELS = {"assemble_r50_c3": dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                                  anti_alias_filter_size=3),
          "resnet50_c1": dict(resnet_size=50)}
SRC = (375, 500)
SIZES = (1, 8, 64, 256)
MAX_BATCH = 256


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not readable"


def event_ms(fn, warmup, iters):
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


def jpegs(n, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    blobs = []
    for _ in range(16):
        img = np.clip(rng.integers(0, 256, 3) + rng.normal(0, 30, SRC + (3,)), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="JPEG", quality=90)
        blobs.append(buf.getvalue())
    return [blobs[i % len(blobs)] for i in range(n)]


def bench_predict(sv, images, n, a):
    req = images[:n]
    for _ in range(a.warmup):
        sv.predict(req)
    times = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        sv.predict(req)
        times.append(time.perf_counter() - t0)
    return statistics.median(times) * 1e3


def bench_kernel(a):
    """100 launches captured in one CUDA graph, so the host's per-call binding overhead is not timed."""
    logits = (torch.randn(256, 1024, device="cuda") * 4)[:, :1001]
    out = predict_rows(logits)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for _ in range(100):
                predict_rows(logits, 256, out)
    torch.cuda.current_stream().wait_stream(s)
    return event_ms(g.replay, a.warmup, a.iters) * 1e3 / 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_serving: no CUDA device")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    us = bench_kernel(a)
    # read: logits; written: two fp32 [256, 1001] arrays and the classes
    nbytes = 256 * 1001 * 4 * 3 + 256 * 4
    print(json.dumps(dict(kernel="acnn_predict_rows", B=256, NC=1001, us=round(us, 2),
                          gb_s=round(nbytes / us / 1e3, 1))), flush=True)
    images = jpegs(max(SIZES))
    for name, flags in MODELS.items():
        sv = Servable(build_model(dtype="bf16", **flags), preprocessing_type="imagenet", image_size=224,
                      max_batch=MAX_BATCH)
        for n in SIZES:
            ms = bench_predict(sv, images, n, a)
            print(json.dumps(dict(model=name, n=n, predict_ms=round(ms, 3), img_s=round(1000.0 * n / ms, 1))),
                  flush=True)
        ms = event_ms(sv._pipe._graph(0, MAX_BATCH).replay, a.warmup, a.iters)
        print(json.dumps(dict(model=name, graph_rows=MAX_BATCH, graph_ms=round(ms, 3),
                              graph_img_s=round(1000.0 * MAX_BATCH / ms, 1))), flush=True)
        del sv
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
