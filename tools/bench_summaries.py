#!/usr/bin/env python
"""The cost of the training summaries (Trainer(train_metrics=True), summary.TrainSummaries): Assemble-ResNet-50
(the c3 flags) with mixup_type = 0 so that the accuracy path runs, bf16, 224 px, batch 256, synthetic device
inputs:

    python tools/bench_summaries.py [--steps 20] [--warmup 3] [--rounds 3] [--iters 20]

  step      the Trainer's step, host clock around --steps steps ending in a device synchronise, for the variants
            off (train_metrics=False), on (train_metrics=True), on + the summary readback every step (N = 1) and
            every 100 steps (N = 100); the variants alternate in one process over --rounds rounds, the median of
            the rounds is reported
  kernels   acnn_classify_rows + acnn_train_metrics_accumulate alone on the step's logits: CUDA events around
            the replay of a graph of 100 launch pairs / 100, median of --iters
  write     the host time of one summary group (decode the ring slot, write and flush the events, log the line)
The card's name, power limit and max SM clock are read in the same run.  One JSON line."""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200.hparams import params_from_flags  # noqa: E402
from assembled_cnn_b200.model_fns import Model, Trainer  # noqa: E402
from assembled_cnn_b200.summary import TrainSummaries  # noqa: E402

C3 = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv", anti_alias_filter_size=3)
BATCH = 256


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_summaries needs a CUDA device")
    print("card:", card(), flush=True)
    p = params_from_flags(batch_size=BATCH, mixup_type=0, label_smoothing=0.1, weight_decay=1e-4,
                          base_learning_rate=0.1, dtype="bf16", **C3)
    trainers = {m: Trainer(Model(num_classes=1001, dtype="bf16", seed=1, **C3), p, 224, 224, use_cuda_graph=True,
                           train_metrics=m) for m in (False, True)}
    g = torch.Generator(device="cuda").manual_seed(0)
    n = trainers[False].input_batch
    x = (torch.randn(n, 224, 224, 3, device="cuda", generator=g) * 64).clamp_(-124, 152)
    lab = torch.randint(1, 1001, (n,), device="cuda", generator=g, dtype=torch.int32)
    tmp = tempfile.mkdtemp(prefix="bench_summaries_")
    summaries = TrainSummaries(tmp, trainers[True])

    def steps(variant):
        tr = trainers[variant != "off"]
        every = {"readback_n1": 1, "readback_n100": 100}.get(variant)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            step = tr.global_step
            loss = tr.train_step(x, lab)
            if every is not None:
                if step % every == 0:
                    summaries.record(loss, step, tr.last_lr, tr.last_keep_prob)
                summaries.poll()
        torch.cuda.synchronize()
        summaries.drain()
        return (time.perf_counter() - t0) * 1e3 / args.steps

    variants = ("off", "on", "readback_n1", "readback_n100")
    for v in variants:
        for _ in range(args.warmup):
            trainers[v != "off"].train_step(x, lab)
    times = {v: [] for v in variants}
    for _ in range(args.rounds):
        for v in variants:
            times[v].append(steps(v))
    step_ms = {v: round(statistics.median(t), 3) for v, t in times.items()}

    # the two launches alone, on the step's logits and labels (they only write the Trainer's own scratch)
    tr = trainers[True]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            for _ in range(100):
                tr._accumulate_metrics(0)
    torch.cuda.current_stream().wait_stream(s)
    kernels_us = event_ms(graph.replay, 2, args.iters) / 100 * 1e3

    # one summary group's host work, from a completed ring slot
    summaries.record(tr._loss_slot, tr.global_step, tr.last_lr, tr.last_keep_prob)
    torch.cuda.synchronize()
    entry = summaries._pending.popleft()
    t0 = time.perf_counter()
    for _ in range(100):
        summaries._write(entry)
    write_us = (time.perf_counter() - t0) * 1e6 / 100
    summaries.close()
    size = os.path.getsize(summaries.writer.path)
    shutil.rmtree(tmp)

    out = dict(batch_size=BATCH, image_size=224, dtype="bf16", mixup_type=0, steps=args.steps, rounds=args.rounds,
               step_ms=step_ms, rounds_ms={v: [round(t, 3) for t in ts] for v, ts in times.items()},
               on_over_off=round(step_ms["on"] / step_ms["off"], 4),
               readback_n1_over_off=round(step_ms["readback_n1"] / step_ms["off"], 4),
               readback_n100_over_off=round(step_ms["readback_n100"] / step_ms["off"], 4),
               kernels_us=round(kernels_us, 2), kernels_share_of_step=round(kernels_us / 1e3 / step_ms["off"], 5),
               write_group_us=round(write_us, 1), summary_file_bytes=size)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
