#!/usr/bin/env python
"""Image search latency on a Stanford Online Products-size gallery (60 502 rows, d = 512 and 2048, bf16,
cosine), k = 6 and 101, for requests of n = 1, 8, 64 and 256:

  * the search alone: acnn_knn_search on an index prepared once (KnnIndex.search) against acnn_knn_topk
    (which prepares the whole gallery on every call), each with its work buffer allocated once, CUDA-event
    median of --iters calls after --warmup, the two alternating per (d, k, n);
  * the whole call: Servable.search against Servable.predict of n JPEGs (bf16 vanilla ResNet-50, 224 px,
    the ladder (1, 8, 64, 256); d = 2048, the pooled features as the embedding), host clock around the
    call, which ends in a synchronise, median of --repeats calls after --warmup, predict and search
    alternating call by call.

    python tools/bench_gallery_search.py [--iters 50] [--warmup 5] [--repeats 10]

Prints the card name, power limit and max SM clock, the SM clock read after the timed calls, and one JSON
line per measurement."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_serving import jpegs  # noqa: E402
from bench_serving_ladder import smi  # noqa: E402
from assembled_cnn_b200 import _lib  # noqa: E402
from assembled_cnn_b200.metrics import KnnIndex  # noqa: E402
from assembled_cnn_b200.model_fns import Servable, build_model  # noqa: E402

NX = 60502
DIMS = (512, 2048)
KS = (6, 101)
SIZES = (1, 8, 64, 256)
LADDER = (1, 8, 64, 256)


def event_median(fns, warmup, iters):
    """{name: median ms} of each fn in fns, the fns alternating call by call."""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    times = {name: [] for name in fns}
    for _ in range(iters):
        for name, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    return {name: statistics.median(t) for name, t in times.items()}


def bench_kernels(a):
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(0)
    for d in DIMS:
        gallery = torch.randn(NX, d, device="cuda", generator=g)
        index = KnnIndex(gallery, "cosine", "bf16")
        for k in KS:
            for n in SIZES:
                q = torch.randn(n, d, device="cuda", generator=g)
                out = (torch.empty(n, k, dtype=torch.int32, device="cuda"), torch.empty(n, k, device="cuda"))
                sw = torch.empty(index.work_bytes(n, k), dtype=torch.uint8, device="cuda")
                tb = lib.acnn_knn_work_bytes(n, NX, d, k, 0)
                tw = torch.empty(tb, dtype=torch.uint8, device="cuda")

                def topk():
                    _lib.check(lib.acnn_knn_topk(q.data_ptr(), gallery.data_ptr(), n, NX, d, k, 0, 0,
                                                 out[0].data_ptr(), out[1].data_ptr(), tw.data_ptr(), tb, stream),
                               "acnn_knn_topk")

                ms = event_median({"search": lambda: index.search(q, k, out, sw), "topk": topk}, a.warmup, a.iters)
                print(json.dumps(dict(part="kernel", d=d, k=k, n=n, search_ms=round(ms["search"], 4),
                                      topk_ms=round(ms["topk"], 4), speedup=round(ms["topk"] / ms["search"], 2))),
                      flush=True)
        del index, gallery
        torch.cuda.empty_cache()


def call_ms(fns, a):
    """{name: median ms} of each whole call in fns, host clock, the calls alternating one by one: a search
    always follows a predict, as on a servable that answers both."""
    for _ in range(a.warmup):
        for fn in fns.values():
            fn()
    times = {name: [] for name in fns}
    for _ in range(a.repeats):
        for name, fn in fns.items():
            t0 = time.perf_counter()
            fn()
            times[name].append(1000.0 * (time.perf_counter() - t0))
    return {name: statistics.median(t) for name, t in times.items()}


def bench_servable(a):
    model = build_model(resnet_size=50, dtype="bf16")
    sv = Servable(model, max_batch=256, batch_sizes=LADDER, return_embedding=True)
    sv.set_gallery(torch.randn(NX, sv.embedding_width, generator=torch.Generator().manual_seed(1)))
    images = jpegs(max(SIZES))
    for n in SIZES:
        req = images[:n]
        for k in KS:
            ms = call_ms({"predict": lambda: sv.predict(req), "search": lambda: sv.search(req, k)}, a)
            print(json.dumps(dict(part="servable", d=sv.embedding_width, k=k, n=n, predict_ms=round(ms["predict"], 3),
                                  search_ms=round(ms["search"], 3), added_ms=round(ms["search"] - ms["predict"], 3))),
                  flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gallery_search: no CUDA device")
    print("card (name, power limit, max SM clock):", smi("name,power.limit,clocks.max.sm"), flush=True)
    bench_kernels(a)
    print("SM clock after the kernel timings:", smi("clocks.sm"), flush=True)
    bench_servable(a)
    print("SM clock after the servable timings:", smi("clocks.sm"), flush=True)


if __name__ == "__main__":
    main()
