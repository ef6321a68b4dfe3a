#!/usr/bin/env python
"""The robustness evaluation's device path on synthetic data: Assemble-ResNet-50 (the c3 flags), eval,
bf16, 224 px, at B = 128 and 256.

    python tools/bench_mce.py [--batches 128,256] [--iters 20] [--warmup 5] [--decode-images 2048]

Per batch size, CUDA-event times of one batch (median of --iters after --warmup):
  u8_convert   acnn_set_images_u8 alone (the extra uint8 -> fp32 pass: B*H*W*3 bytes read, 4x written)
  u8_device    acnn_set_images_u8 + eval forward + softmax top-1 count, one CUDA graph replay, from a
               device uint8 batch (what model_fns.corruption_error replays)
  f32_host     acnn_set_inputs from a pinned host fp32 batch (today's input path: 4x the bytes over PCIe)
               + the same forward + count, eager
  pipeline     images/s of the pipelined loop of corruption_error (pinned uint8 ring, copy stream, graph
               replays) over pre-decoded batches, host clock around the loop and a device synchronise
and, separately, the JPEG-decode rate (images/s) of the CPU thread pool on synthetic 224 x 224 JPEGs,
with the core count.  Prints the card name and power limit read in the same run and one JSON line per
measurement."""
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
from assembled_cnn_b200.imagenet_c import CHANNEL_MEANS, decode_image  # noqa: E402
from assembled_cnn_b200.metrics import softmax_top1_count  # noqa: E402
from assembled_cnn_b200.model_fns import _CorruptionEvalDevice, build_model  # noqa: E402

FLAGS = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
             anti_alias_filter_size=3)
SIZE = 224


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
    g = torch.Generator().manual_seed(B)
    u8 = torch.randint(0, 256, (B, SIZE, SIZE, 3), generator=g, dtype=torch.uint8)
    labels = torch.randint(1, 1001, (B,), generator=g, dtype=torch.int32)
    ev = _CorruptionEvalDevice(model, B, SIZE, False, True)
    rt = ev.rt
    ev.slots[0][0].copy_(u8)
    ev.slots[0][1].copy_(labels)
    ev._body(0, B)                                     # loads every kernel before the capture
    graph = ev._graph(0, B)
    out = {}
    out["u8_convert_ms"] = timed(lambda: rt.set_images_u8(ev.slots[0][0], ev.mean), a.warmup, a.iters)
    out["u8_device_ms"] = timed(graph.replay, a.warmup, a.iters)

    host_f32 = (u8.float() - torch.tensor(CHANNEL_MEANS)).pin_memory()
    host_lab = labels.pin_memory()
    logits = rt.t[rt.plan.meta["logits"]][:, :1001]

    def f32_host():
        _lib.check(rt.lib.acnn_set_inputs(rt.model.handle, host_f32.data_ptr(), None, None, None, None,
                                          rt.stream), "acnn_set_inputs")
        ev.slots[1][1].copy_(host_lab, non_blocking=True)
        rt.run_forward()
        softmax_top1_count(logits, ev.slots[1][1], ev.acc, B, ev.pred)
    out["f32_host_ms"] = timed(f32_host, a.warmup, a.iters)

    # the two paths compute the same logits
    graph.replay()
    want = logits.clone()
    f32_host()
    out["same_logits"] = bool(torch.equal(logits, want))

    images = [a_.numpy() for a_ in u8]
    lab = labels.tolist()
    for _ in range(a.warmup):
        ev.run_batch(images, lab)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.iters):
        ev.run_batch(images, lab)
    torch.cuda.synchronize()
    out["pipeline_img_s"] = a.iters * B / (time.perf_counter() - t0)
    out["u8_device_img_s"] = 1000.0 * B / out["u8_device_ms"]
    out["f32_host_img_s"] = 1000.0 * B / out["f32_host_ms"]
    out["u8_convert_GB_s"] = B * SIZE * SIZE * 3 * 5 / out["u8_convert_ms"] / 1e6
    return out


def bench_decode(n, workers, tmp):
    from PIL import Image
    rng = np.random.default_rng(0)
    paths = []
    for i in range(32):       # distinct files, read round-robin
        img = np.clip(rng.integers(0, 256, 3) + rng.normal(0, 30, (SIZE, SIZE, 3)), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="JPEG", quality=85)
        p = os.path.join(tmp, "%d.JPEG" % i)
        with open(p, "wb") as f:
            f.write(buf.getvalue())
        paths.append(p)
    with ThreadPoolExecutor(max_workers=workers) as pool:
        list(pool.map(lambda p: decode_image(p, SIZE), paths))
        t0 = time.perf_counter()
        list(pool.map(lambda i: decode_image(paths[i % len(paths)], SIZE), range(n)))
        return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="128,256")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--decode-images", type=int, default=2048)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mce: no CUDA device")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    model = build_model(**FLAGS)
    for B in (int(b) for b in a.batches.split(",")):
        r = bench_batch(model, B, a)
        print(json.dumps(dict(batch=B, **{k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()})),
              flush=True)
    import tempfile
    cores = len(os.sched_getaffinity(0))
    with tempfile.TemporaryDirectory() as tmp:
        rate = bench_decode(a.decode_images, min(32, cores), tmp)
    print(json.dumps(dict(jpeg_decode_img_s=round(rate, 1), cpu_cores=cores, threads=min(32, cores),
                          image=SIZE)), flush=True)


if __name__ == "__main__":
    main()
