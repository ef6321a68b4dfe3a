#!/usr/bin/env python
"""Rate of the ImageNet dataset builder (build_data.build('imagenet', ...)) on a synthetic tree, with the
device check and with the PIL-only check, alternated in one run.

    python tools/bench_build_data.py [--images 4096] [--reps 3] [--num_workers N]

The tree is --images seeded 500 x 375 baseline JPEGs (quality 90, 4:2:0) over 16 synset directories in the
ImageNet layout; each build writes its train split in 16 shards (num_threads 8) from that tree: listing,
reads, the check of every scan, the Example serialisation, CRC-32C and the writes.  One untimed build per
mode first (the page cache, the CUDA context, the decoder's buffers), then --reps timed builds per mode,
alternating device / pil, host clock around the whole call.  Prints the card name and power limit and the
host core count read in the same run, and one JSON line per mode (median images/s and every rep).  The tree
and the shards go to a temporary directory that is removed at the end."""
import argparse
import io
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200 import build_data  # noqa: E402

SRC = (375, 500)
SYNSETS = ["n%08d" % (1440764 + 17 * k) for k in range(16)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        import torch
        return torch.cuda.get_device_name() + ", power limit not readable"


def make_tree(root, n, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    for s in SYNSETS:
        os.makedirs(os.path.join(root, "train", s))
    with open(os.path.join(root, "synsets.txt"), "w") as f:
        f.write("\n".join(SYNSETS) + "\n")
    with open(os.path.join(root, "metadata.txt"), "w") as f:
        f.write("".join("%s\tclass %d\n" % (s, k) for k, s in enumerate(SYNSETS)))
    total = 0
    for i in range(n):
        base = rng.integers(0, 256, size=(12, 16, 3), dtype=np.uint8)
        a = np.array(Image.fromarray(base).resize((SRC[1], SRC[0]), Image.BICUBIC), dtype=np.int16)
        a = np.clip(a + rng.integers(-12, 13, size=a.shape), 0, 255).astype(np.uint8)
        b = io.BytesIO()
        Image.fromarray(a).save(b, "JPEG", quality=90)
        s = SYNSETS[i % len(SYNSETS)]
        with open(os.path.join(root, "train", s, "%s_%d.JPEG" % (s, i)), "wb") as f:
            f.write(b.getvalue())
        total += len(b.getvalue())
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--num_workers", type=int, default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_build_data: needs a CUDA device")
    print("card:", card(), "| host cores:", os.cpu_count(), flush=True)
    work = tempfile.mkdtemp(prefix="bench_build_data_")
    try:
        nbytes = make_tree(work, args.images)
        flags = dict(train_shards=16, num_threads=8, make_val=False, labels_file=work + "/synsets.txt",
                     imagenet_metadata_file=work + "/metadata.txt")
        times = {"device": [], "pil": []}

        def run(check):
            out = os.path.join(work, "out")
            t0 = time.perf_counter()
            n = build_data.build("imagenet", out, work + "/train", work + "/validation", check=check,
                                 num_workers=args.num_workers, **flags)
            dt = time.perf_counter() - t0
            assert n == {"train": args.images}
            shutil.rmtree(out)
            return dt

        for check in times:
            run(check)
        for _ in range(args.reps):
            for check in times:
                times[check].append(run(check))
        for check, ts in times.items():
            rates = [args.images / t for t in ts]
            print(json.dumps({"bench": "build_data_imagenet", "check": check, "images": args.images,
                              "jpeg_mb": round(nbytes / 1e6, 1), "src": "%dx%d" % (SRC[1], SRC[0]),
                              "num_workers": args.num_workers or min(32, os.cpu_count() or 1),
                              "images_per_s_median": round(statistics.median(rates), 1),
                              "images_per_s": [round(r, 1) for r in rates], "card": card(),
                              "host_cores": os.cpu_count()}), flush=True)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
