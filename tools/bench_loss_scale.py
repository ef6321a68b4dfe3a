#!/usr/bin/env python
"""The cost of dynamic loss scaling: Assemble-ResNet-50 (the c3 flags: mixup 1, label smoothing 0.1) in fp16, 224 px,
batch 256, synthetic device inputs, the static scale 128 against dynamic scaling held at 128 (a growth interval
longer than the run), alternating in one process:

    python tools/bench_loss_scale.py [--iters 20] [--warmup 5] [--rounds 3] [--check-iters 200]

  step_ms     the training step (forward + backward + update phase) as one CUDA-graph replay, CUDA events, median
              of --iters after --warmup replays; the median over --rounds alternating rounds.  The dynamic step
              adds the finiteness check, the skip-aware SGD and the scale update
  check_us    acnn_grads_nonfinite alone over the c3 gradient buffer (param_elems fp32), CUDA events around
              --check-iters launches; check_gbps = 4 * param_elems bytes over that time
The card's name, power limit and max SM clock are read in the same run.  One JSON line."""
import argparse
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_fp16 import card, event_ms, init_weights, runtime  # noqa: E402


def check_us(rt, iters):
    flag = torch.zeros(1, dtype=torch.int32, device=rt.dev)
    n, stream = rt.plan.param_elems, torch.cuda.current_stream().cuda_stream
    lib = rt.lib

    def launch():
        for _ in range(iters):
            lib.acnn_grads_nonfinite(rt.grads.data_ptr(), n, flag.data_ptr(), stream)
    launch()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    launch()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000.0 / iters, int(flag.item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--check-iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_loss_scale needs a CUDA device")
    print("card:", card(), flush=True)
    modes = ("static", "dynamic")
    rts, graphs = {}, {}
    for mode in modes:
        rt = runtime("fp16", True)
        init_weights(rt)
        if mode == "static":
            rt.set_hparams(lr=0.01, momentum=0.9, weight_decay=1e-4, grad_scale=1.0 / 128.0)
            rt.loss_scale = 128.0
        else:
            rt.set_hparams(lr=0.01, momentum=0.9, weight_decay=1e-4, grad_scale=0.0)
            rt.enable_dynamic_loss_scale(128.0, 10 ** 9, 1)
        rts[mode], graphs[mode] = rt, rt.capture(train=True)
    step = {m: [] for m in modes}
    for _ in range(args.rounds):
        for m in modes:
            step[m].append(event_ms(graphs[m].replay, args.warmup, args.iters))
    chk, flag = check_us(rts["dynamic"], args.check_iters)
    n = rts["dynamic"].plan.param_elems
    med = lambda v: round(statistics.median(v), 3)  # noqa: E731
    out = dict(card=card(), batch_size=256, image_size=224, flags="c3 (mixup 1, label smoothing 0.1), fp16",
               step_ms={m: med(step[m]) for m in modes},
               rounds_step_ms={m: [round(t, 3) for t in step[m]] for m in modes},
               dynamic_over_static=round(med(step["dynamic"]) / med(step["static"]), 4),
               check_elems=n, check_us=round(chk, 2), check_gbps=round(4.0 * n / (chk * 1e-6) / 1e9, 1),
               check_flag=flag, dynamic_state=rts["dynamic"].loss_scale_state(),
               params_finite={m: bool(torch.isfinite(rts[m].params).all()) for m in modes})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
