#!/usr/bin/env python
"""Servable.predict latency with one rung (max_batch 256) against the batch ladder (1, 8, 64, 256), on the
synthetic 500 x 375 JPEGs and with the timing protocol of tools/bench_serving.py (one whole predict call,
host clock, median of --repeats calls after --warmup calls of the same n), bf16, 224 px, for vanilla
ResNet-50 (the c1 flags) and Assemble-ResNet-50 (c3):

    python tools/bench_serving_ladder.py [--repeats 10] [--warmup 3]

The two servables of a model share its weights and run alternately, n by n.  After the timed calls it
reports the device memory each servable holds (torch.cuda.memory_allocated while only that servable's
rungs, workspaces, buffers and graphs exist beside the model's weights; the weights are counted once, as
`weights_mib`, with the model's batch-1 runtime that owns them).  Prints the card name, power limit, max
SM clock and the SM clock read right after the timed calls, and one JSON line per measurement."""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_serving import MODELS, SIZES, bench_predict, jpegs  # noqa: E402
from assembled_cnn_b200.model_fns import Servable, build_model  # noqa: E402

MAX_BATCH = 256
LADDER = (1, 8, 64, 256)


def smi(fields):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "not readable"


def mib(b):
    return round(b / 2 ** 20, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_serving_ladder: no CUDA device")
    print("card (name, power limit, max SM clock):", smi("name,power.limit,clocks.max.sm"), flush=True)
    images = jpegs(max(SIZES))
    for name, flags in MODELS.items():
        model = build_model(dtype="bf16", **flags)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        model.runtime(1, 224, 224, training=False)        # the weights: owned by the model's first runtime
        torch.cuda.synchronize()
        weights = torch.cuda.memory_allocated() - base
        servables = {"single": Servable(model, max_batch=MAX_BATCH),
                     "ladder": Servable(model, max_batch=MAX_BATCH, batch_sizes=LADDER)}
        for n in SIZES:
            for kind, sv in servables.items():
                ms = bench_predict(sv, images, n, a)
                print(json.dumps(dict(model=name, servable=kind, n=n, predict_ms=round(ms, 3),
                                      img_s=round(1000.0 * n / ms, 1))), flush=True)
        print("SM clock after the timed calls:", smi("clocks.sm"), flush=True)
        # memory: drop every runtime but the weights' owner, then build each servable alone
        keep = model._primary[False]
        del sv
        servables.clear()
        model._runtimes = {k: v for k, v in model._runtimes.items() if v is keep}
        gc.collect()
        for kind, sizes in (("single", None), ("ladder", LADDER)):
            before = torch.cuda.memory_allocated()
            sv = Servable(model, max_batch=MAX_BATCH, batch_sizes=sizes)
            for n in SIZES:
                sv.predict(images[:n])
            torch.cuda.synchronize()
            held = torch.cuda.memory_allocated() - before
            print(json.dumps(dict(model=name, servable=kind, device_mib=mib(held), weights_mib=mib(weights))),
                  flush=True)
            del sv
            model._runtimes = {k: v for k, v in model._runtimes.items() if v is keep}
            gc.collect()
        del model, keep
        gc.collect()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
