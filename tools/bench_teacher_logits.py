#!/usr/bin/env python
"""Teacher-logit extraction (model_fns.extract_teacher_logits) on synthetic data, bf16, for the two teachers
of the README: Assemble-ResNet-152 BigLittle (the c5 flags) at 256 px ('imagenet_224_256a', as an R152
teacher is evaluated) and Assemble-ResNet-50 (the c3 flags) at 224 px ('imagenet').

    python tools/bench_teacher_logits.py [--batch 256] [--images 8192] [--iters 20] [--warmup 5]

Per teacher:
  graph     resize + crop + mean, the eval forward and the logits copy: one CUDA graph replay (what the
            extraction replays per batch), CUDA-event median of --iters after --warmup
  loop      images/s of a whole extract_teacher_logits call over --images synthetic 500 x 375 JPEGs (16
            seeded images repeated) in four train shards and one validation shard: shard checks, device
            decode, graph replays, logits to pinned memory, the CRC checks and the writes of every record;
            host clock, after one untimed call
and acnn_crc32c alone over a 256 MiB host buffer, GB/s (median of 5).  Prints the card name and power limit
read in the same run and one JSON line per measurement.  The shards and outputs go to a temporary
directory that is removed at the end."""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200 import imagenet_eval as ie, native  # noqa: E402
from assembled_cnn_b200.model_fns import _TeacherLogitsDevice, build_model, extract_teacher_logits  # noqa: E402

ASSEMBLE = dict(resnet_version=2, use_sk_block=True, anti_alias_type="sconv", anti_alias_filter_size=3)
TEACHERS = {"assemble_r152_biglittle": (dict(resnet_size=152, bl_alpha=1, bl_beta=2, **ASSEMBLE),
                                        "imagenet_224_256a", 224),
            "assemble_r50": (dict(resnet_size=50, **ASSEMBLE), "imagenet", 224)}
SRC = (375, 500)


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


def jpegs(seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    blobs = []
    for _ in range(16):
        img = np.clip(rng.integers(0, 256, 3) + rng.normal(0, 30, SRC + (3,)), 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="JPEG", quality=90)
        blobs.append(buf.getvalue())
    return blobs


def example(jpeg, label):
    """A serialised tf.train.Example with image/encoded and image/class/label."""
    lf = ie._len_field

    def entry(key, feature):
        body = lf(1, len(key)) + key + lf(2, len(feature)) + feature
        return lf(1, len(body)) + body
    blist = lf(1, len(jpeg)) + jpeg
    ilist = b"\x08" + ie._encode_varint(label)
    feats = entry(b"image/encoded", lf(1, len(blist)) + blist) + entry(b"image/class/label", lf(3, len(ilist)) + ilist)
    return lf(1, len(feats)) + feats


def write_shards(root, n):
    blobs = jpegs()
    names = ["train-%05d-of-00004" % i for i in range(4)] + ["validation-00000-of-00001"]
    for k, name in enumerate(names):
        with open(os.path.join(root, name), "wb") as f:
            for i in range(k, n, len(names)):
                ie.write_record(f, [example(blobs[i % len(blobs)], i % 1000)])


def bench_graph(model, ptype, image_size, a):
    S, _ = ie.eval_size(ptype, image_size)
    ev = _TeacherLogitsDevice(model, a.batch, S, False, True, lambda rows: None)
    blobs = jpegs()
    ev.run_batch_encoded([blobs[i % 16] for i in range(a.batch)], [0] * a.batch,
                         lambda h, w: ie.eval_geometry(h, w, ptype, image_size))     # eager: loads every kernel
    ev.finish()
    torch.cuda.synchronize()
    return timed(ev._graph(0, a.batch).replay, a.warmup, a.iters)


def bench_loop(model, ptype, image_size, root, a):
    kw = dict(preprocessing_type=ptype, image_size=image_size, batch_size=a.batch)
    extract_teacher_logits(model, root, os.path.join(root, "warm", ptype), **kw)
    t0 = time.perf_counter()
    extract_teacher_logits(model, root, os.path.join(root, "timed", ptype), **kw)
    return a.images / (time.perf_counter() - t0)


def bench_crc():
    buf = np.random.default_rng(0).integers(0, 256, 256 << 20, dtype=np.uint8).tobytes()
    native.crc32c(buf)
    times = []
    for _ in range(5):
        t0 = time.perf_counter()
        native.crc32c(buf)
        times.append(time.perf_counter() - t0)
    return len(buf) / statistics.median(times) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--images", type=int, default=8192)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_teacher_logits: no CUDA device")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    print(json.dumps(dict(crc32c_gb_s=round(bench_crc(), 2))), flush=True)
    with tempfile.TemporaryDirectory() as root:
        write_shards(root, a.images)
        for name, (flags, ptype, image_size) in TEACHERS.items():
            model = build_model(dtype="bf16", **flags)
            ms = bench_graph(model, ptype, image_size, a)
            rate = bench_loop(model, ptype, image_size, root, a)
            print(json.dumps(dict(teacher=name, preprocessing_type=ptype, size=ie.eval_size(ptype, image_size)[0],
                                  batch=a.batch, graph_ms=round(ms, 3), graph_img_s=round(1000.0 * a.batch / ms, 1),
                                  loop_img_s=round(rate, 1), images=a.images)), flush=True)
            del model
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
