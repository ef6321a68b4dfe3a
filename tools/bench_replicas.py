#!/usr/bin/env python
"""Several data-parallel replicas on one GPU (Trainer(replicas_per_device=R)): Assemble-ResNet-50 (the c3 flags),
bf16, 224 px, mixup type 1 + label smoothing, synthetic device inputs:

    python tools/bench_replicas.py [--steps 10] [--warmup 3] [--iters 20]

Per (batch_size, R) in (1024, 8) (the from-scratch recipe: 128 per replica, 256 examples per micro-step with
mixup) and (256, 4) (the fine-tuning recipe's 64 per replica):
  step        one global step (R micro-steps: input copy, forward + backward graph, accumulate graph; then the
              SGD graph), host clock around --steps steps ending in a device synchronise, after --warmup
  micro       the forward + backward graph of one micro-step alone, CUDA-event median of --iters
  ratio       step / (R x micro)
  accumulate  each acnn_replica_accumulate phase alone (its captured graph), CUDA-event median of --iters
              replays of a graph of 20 launches / 20, in GB/s of the bytes the phase must move (computed below
              from param_elems / state_elems), and the sum over one global step as a share of the step
  memory      torch's peak allocation and the device's used memory (total - free) after the run
The card's name, power limit and max SM clock are read in the same run.  One JSON line per configuration."""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200.hparams import params_from_flags  # noqa: E402
from assembled_cnn_b200.model_fns import Model, Trainer  # noqa: E402

C3 = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv", anti_alias_filter_size=3)
CONFIGS = ((1024, 8), (256, 4))
SAVE, FIRST, MIDDLE, LAST = 0, 1, 2, 3


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


def phase_bytes(phase, P, S):
    """Bytes a phase reads and writes: P gradient floats, S state floats (+ the 4 loss floats, negligible)."""
    return 4 * {SAVE: 2 * S, FIRST: 2 * P + 4 * S, MIDDLE: 3 * P + 5 * S, LAST: 3 * P + 3 * S}[phase]


def run(batch, R, args):
    b = batch // R
    model = Model(num_classes=1001, dtype="bf16", seed=1, **C3)
    p = params_from_flags(batch_size=batch, mixup_type=1, label_smoothing=0.1, weight_decay=1e-4,
                          base_learning_rate=0.1, dtype="bf16", **C3)
    tr = Trainer(model, p, 224, 224, use_cuda_graph=True, replicas_per_device=R)
    n = tr.input_batch
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn(R * n, 224, 224, 3, device="cuda", generator=g) * 64).clamp_(-124, 152)
    lab = torch.randint(1, 1001, (R * n,), device="cuda", generator=g, dtype=torch.int32)
    lam = torch.rand(R, n // 2, device="cuda", generator=g)
    for _ in range(args.warmup):
        tr.train_step(x, lab, lam1=lam)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        loss = tr.train_step(x, lab, lam1=lam)
    torch.cuda.synchronize()
    step_ms = (time.perf_counter() - t0) * 1e3 / args.steps
    losses = loss.tolist()
    # the micro-step graph and the accumulate phases alone (they only rewrite the step's own buffers)
    micro_ms = event_ms(tr._graphs[0].replay, args.warmup, args.iters)
    P, S = tr.rt.plan.param_elems, tr.rt.plan.state_elems
    acc = {}
    s = torch.cuda.Stream()
    for ph in (SAVE, FIRST, MIDDLE, LAST):
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(graph, stream=s):
                for _ in range(20):
                    tr.rt.replica_accumulate(ph, tr._acc_bufs, 0, P, R)
        torch.cuda.current_stream().wait_stream(s)
        ms = event_ms(graph.replay, 2, args.iters) / 20
        acc[ph] = dict(us=round(ms * 1e3, 2), gbps=round(phase_bytes(ph, P, S) / (ms * 1e-3) / 1e9, 1))
    per_step_ms = sum(acc[ph]["us"] for ph in (SAVE, FIRST, LAST)) / 1e3 + (R - 2) * acc[MIDDLE]["us"] / 1e3
    free, total = torch.cuda.mem_get_info()
    out = dict(batch_size=batch, replicas_per_device=R, per_replica=b, examples_per_micro_step=n,
               step_ms=round(step_ms, 2), img_per_s=round(batch / step_ms * 1e3, 1), micro_ms=round(micro_ms, 3),
               ratio_to_R_micro=round(step_ms / (R * micro_ms), 3),
               accumulate={k: acc[v] for k, v in (("save", SAVE), ("first", FIRST), ("middle", MIDDLE),
                                                   ("last", LAST))},
               accumulate_share_of_step=round(per_step_ms / step_ms, 4),
               param_elems=P, state_elems=S,
               peak_torch_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2),
               device_used_gb=round((total - free) / 1e9, 2), loss=[round(v, 4) for v in losses],
               finite=all(v == v and abs(v) != float("inf") for v in losses))
    del tr, model, x
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_replicas needs a CUDA device")
    print("card:", card(), flush=True)
    for batch, R in CONFIGS:
        print(json.dumps(run(batch, R, args)), flush=True)


if __name__ == "__main__":
    main()
