#!/usr/bin/env python
"""fp16 against bf16 on the same code: Assemble-ResNet-50 (the c3 flags: mixup 1, label smoothing 0.1), 224 px,
batch 256, synthetic device inputs, the two storage types alternating in one process:

    python tools/bench_fp16.py [--iters 20] [--warmup 5] [--rounds 3]

  step_ms     the training step (forward + backward + SGD) as one CUDA-graph replay, CUDA events, median of
              --iters after --warmup replays; the median over --rounds alternating rounds
  eval_ms     the eval forward (moving statistics) at the same batch, likewise
  gemm_share  the conv GEMM kernels' (fprop / dgrad / wgrad and the wgrad split-K sum) share of the kernel
              time of one eager step, from torch.profiler
The card's name, power limit and max SM clock are read in the same run.  One JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200 import native  # noqa: E402
from assembled_cnn_b200.plan import ModelConfig  # noqa: E402

C3 = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv", anti_alias_filter_size=3)
BATCH, HW = 256, 224
GEMM_KERNELS = ("conv_gemm_kernel", "conv_halo_kernel", "wgrad_gemm_kernel", "wgrad_reduce_kernel")


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


def runtime(dtype, training, share=None):
    kw = dict(training=True, mixup_type=1, label_smoothing=0.1) if training else \
        dict(training=False, with_loss=False)
    rt = native.NativeRuntime(native.NativeModel(ModelConfig(**C3), BATCH, HW, HW, dtype=dtype, **kw), share=share)
    m = rt.plan.meta
    g = torch.Generator(device="cuda").manual_seed(0)
    n = m["input_batch"]
    rt.t[m["images"]].copy_((torch.randn(n, HW, HW, 3, device="cuda", generator=g) * 64).clamp_(-124, 152))
    if "labels" in m:
        rt.t[m["labels"]].copy_(torch.randint(1, 1001, (n,), device="cuda", generator=g, dtype=torch.int32))
    if "lam1" in m:
        rt.t[m["lam1"]].copy_(torch.rand(n // 2, device="cuda", generator=g))
    return rt


def init_weights(rt):
    g = torch.Generator(device="cuda").manual_seed(1)
    for p in rt.plan.params.values():
        fan_in = 1
        for d in p.store_shape[1:]:
            fan_in *= d
        rt.params[p.offset:p.offset + p.size].normal_(0.0, (2.0 / max(fan_in, 1)) ** 0.5, generator=g)
        if p.kind == "gamma":
            rt.params[p.offset:p.offset + p.size].fill_(1.0)
        elif p.kind in ("beta", "dense_bias"):
            rt.params[p.offset:p.offset + p.size].zero_()


def gemm_share(rt):
    from torch.profiler import ProfilerActivity, profile
    rt.run_step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rt.run_step()
        torch.cuda.synchronize()
    tot = gemm = 0.0
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None)
        if t is None:
            t = getattr(e, "self_cuda_time_total", 0.0)
        tot += t
        if any(k in e.key for k in GEMM_KERNELS):
            gemm += t
    return gemm / tot if tot > 0 else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp16 needs a CUDA device")
    print("card:", card(), flush=True)
    dtypes = ("bf16", "fp16")
    train, evals, graphs = {}, {}, {}
    for dt in dtypes:
        train[dt] = runtime(dt, True)
        init_weights(train[dt])
        train[dt].set_hparams(lr=0.01, momentum=0.9, weight_decay=1e-4, grad_scale=1.0 / (128.0 if dt == "fp16" else 1.0))
        train[dt].loss_scale = 128.0 if dt == "fp16" else 1.0
        evals[dt] = runtime(dt, False, share=train[dt])
        graphs[dt] = (train[dt].capture(train=True), evals[dt].capture(train=False))
    step = {dt: [] for dt in dtypes}
    ev = {dt: [] for dt in dtypes}
    for _ in range(args.rounds):
        for dt in dtypes:
            step[dt].append(event_ms(graphs[dt][0].replay, args.warmup, args.iters))
            ev[dt].append(event_ms(graphs[dt][1].replay, args.warmup, args.iters))
    share = {dt: gemm_share(train[dt]) for dt in dtypes}
    finite = {dt: bool(torch.isfinite(train[dt].params).all()) for dt in dtypes}
    loss = {dt: [round(float(v), 4) for v in train[dt].slot_view(train[dt].plan.meta["loss"])[:2]] for dt in dtypes}
    med = lambda v: round(statistics.median(v), 3)  # noqa: E731
    out = dict(card=card(), batch_size=BATCH, image_size=HW, flags="c3 (mixup 1, label smoothing 0.1)",
               step_ms={dt: med(step[dt]) for dt in dtypes}, eval_ms={dt: med(ev[dt]) for dt in dtypes},
               rounds_step_ms={dt: [round(t, 3) for t in step[dt]] for dt in dtypes},
               rounds_eval_ms={dt: [round(t, 3) for t in ev[dt]] for dt in dtypes},
               fp16_over_bf16_step=round(med(step["fp16"]) / med(step["bf16"]), 4),
               fp16_over_bf16_eval=round(med(ev["fp16"]) / med(ev["bf16"]), 4),
               gemm_share={dt: round(share[dt], 4) for dt in dtypes}, params_finite=finite, last_loss=loss)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
