#!/usr/bin/env python
"""The retrieval evaluation's device path (model_fns.evaluate_retrieval) on synthetic data: Assemble-ResNet-50
(the c3 flags), eval, bf16, 224 px ('imagenet' preprocessing), 500 x 375 sources, return_embedding (the 2048
pooled features), at B = 128 and 256; and the final search at Stanford Online Products size.

    python tools/bench_retrieval_eval.py [--batches 128,256] [--iters 20] [--warmup 5] [--loop-batches 8]

Per batch size:
  graph        resize + crop + mean and the eval forward, one CUDA graph replay (what evaluate_retrieval
               replays per batch), CUDA-event median of --iters after --warmup
  pipeline     images/s of the pipelined loop from encoded JPEGs (device decode on the copy stream, host
               descriptors, graph replay, the rows appended to the device index), --loop-batches batches,
               host clock around the loop and a device synchronise, after one untimed pass
and, for d = 512 and 2048, the final search over a 60 502-row index (every row a query, 11 318 classes):
metrics.recall_of_index with Recall@1/5 (acnn_knn_topk with k = 6, cosine, bf16, plus the finiteness check
and the recall bookkeeping), CUDA-event median.  Prints the card name and power limit read in the same run
and one JSON line per measurement."""
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
from assembled_cnn_b200.imagenet_eval import eval_geometry  # noqa: E402
from assembled_cnn_b200.metrics import recall_of_index  # noqa: E402
from assembled_cnn_b200.model_fns import _RetrievalEvalDevice, build_model  # noqa: E402

FLAGS = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
             anti_alias_filter_size=3)
SIZE, SRC = 224, (375, 500)
SOP_ROWS, SOP_CLASSES = 60502, 11318


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


def jpegs(n):
    from PIL import Image
    rng = np.random.default_rng(0)
    blobs = []
    for _ in range(16):
        img = np.clip(rng.integers(0, 256, 3) + rng.normal(0, 30, SRC + (3,)), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="JPEG", quality=90)
        blobs.append(buf.getvalue())
    return [blobs[i % len(blobs)] for i in range(n)]


def bench_batch(model, B, a):
    blobs = jpegs(B)
    labels = list(range(B))
    geometry = lambda h, w: eval_geometry(h, w, "imagenet", SIZE)
    ev = _RetrievalEvalDevice(model, B, SIZE, False, True, True, B * (2 * a.loop_batches + 2))
    ev.run_batch_encoded(blobs, labels, geometry)            # eager: loads every kernel, fills slot 0
    torch.cuda.synchronize()
    out = {"graph_ms": timed(ev._graph(0, B).replay, a.warmup, a.iters)}
    for _ in range(a.loop_batches):
        ev.run_batch_encoded(blobs, labels, geometry)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.loop_batches):
        ev.run_batch_encoded(blobs, labels, geometry)
    torch.cuda.synchronize()
    out["pipeline_img_s"] = a.loop_batches * B / (time.perf_counter() - t0)
    out["graph_img_s"] = 1000.0 * B / out["graph_ms"]
    return out


def bench_search(d, a):
    g = torch.Generator(device="cuda").manual_seed(d)
    feats = torch.randn(SOP_ROWS, d, device="cuda", generator=g)
    labels = torch.randint(0, SOP_CLASSES, (SOP_ROWS,), device="cuda", generator=g)
    return timed(lambda: recall_of_index(feats, labels, (1, 5), "cosine", "bf16"), 2, a.search_iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="128,256")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--loop-batches", type=int, default=8)
    ap.add_argument("--search-iters", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_retrieval_eval: no CUDA device")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    model = build_model(**FLAGS)
    for B in (int(b) for b in a.batches.split(",")):
        r = bench_batch(model, B, a)
        print(json.dumps(dict(batch=B, **{k: round(v, 3) for k, v in r.items()})), flush=True)
    for d in (512, 2048):
        print(json.dumps(dict(search_rows=SOP_ROWS, d=d, k=6, search_ms=round(bench_search(d, a), 3))), flush=True)


if __name__ == "__main__":
    main()
