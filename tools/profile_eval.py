#!/usr/bin/env python
"""Per-op CUDA-event times of one eager eval forward (bf16, 224 px) at small batches, for vanilla
ResNet-50 (the c1 flags) and Assemble-ResNet-50 (c3): every plan op runs as its own acnn_run_ops range
between two events, after --warmup forwards, and each op's time is the median over --iters forwards.

    python tools/profile_eval.py [--batches 1 8] [--iters 20] [--warmup 3] [--top 12]

Per (model, batch) it prints the forward's total, the time by op kind, and the conv GEMM launches split
by output tiles (128-row M tiles x 128-column N tiles) against the SM count: the launches with fewer
tiles than SMs are the ones a split-K fprop could spread over more of the GPU.  Then the --top slowest
conv launches.  Each op's time includes its launch gap, as an eager forward pays it; the whole forward
is also timed as one CUDA graph replay (the servable's form), median over --iters replays.  Also prints the
card name, power limit and max SM clock read in the same run, and one JSON line per (model, batch)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200.model_fns import build_model  # noqa: E402

MODELS = {"resnet50_c1": dict(resnet_size=50),
          "assemble_r50_c3": dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                                  anti_alias_filter_size=3)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not readable"


def profile(model, B, a):
    rt = model.runtime(B, 224, 224, training=False)
    rt.t[rt.plan.meta["images"]].copy_(torch.randn(B, 224, 224, 3) * 60)
    ops = rt.plan.forward
    for _ in range(a.warmup):
        rt.run_forward()
    times = [[] for _ in ops]
    for _ in range(a.iters):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(ops) + 1)]
        ev[0].record()
        for i, op in enumerate(ops):
            rt.run([op])
            ev[i + 1].record()
        torch.cuda.synchronize()
        for i in range(len(ops)):
            times[i].append(ev[i].elapsed_time(ev[i + 1]))
    ms = [statistics.median(t) for t in times]
    # the same forward as one CUDA graph, as the servable replays it
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            rt.run_forward()
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(a.warmup):
        g.replay()
    graph = []
    for _ in range(a.iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        graph.append(e0.elapsed_time(e1))
    del g
    by_kind = defaultdict(float)
    convs = []
    for op, t in zip(ops, ms):
        by_kind[op.kind] += t
        if op.kind == "conv":
            g, macs, _ = rt.plan.conv_info(op)
            Ho, Wo = g.out_hw()
            M = g.B * Ho * Wo
            tiles = -(-M // 128) * -(-g.Cout // 128)
            convs.append((t, tiles, "%dx%d %d->%d k%d s%d K=%d M=%d" % (g.H, g.W, g.Cin, g.Cout, g.kh, g.stride,
                                                                        g.kh * g.kw * g.Cin, M)))
    return sum(ms), len(ops), by_kind, convs, statistics.median(graph)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--top", type=int, default=12)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_eval: no CUDA device")
    print("card (name, power limit, max SM clock, SM clock):", card(), flush=True)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for name, flags in MODELS.items():
        model = build_model(dtype="bf16", **flags)
        for B in a.batches:
            total, n_ops, by_kind, convs, graph_ms = profile(model, B, a)
            conv_ms = sum(t for t, _, _ in convs)
            few = [c for c in convs if c[1] < sms]
            few_ms = sum(t for t, _, _ in few)
            print("\n== %s B=%d: forward %.3f ms over %d ops (eager, per-op ranges); %.3f ms as one CUDA graph"
                  % (name, B, total, n_ops, graph_ms))
            for k, t in sorted(by_kind.items(), key=lambda kv: -kv[1]):
                print("  %-16s %8.3f ms %5.1f%%" % (k, t, 100 * t / total))
            print("  conv launches: %d, %.3f ms; with fewer output tiles than the %d SMs: %d, %.3f ms (%.1f%% of "
                  "the forward)" % (len(convs), conv_ms, sms, len(few), few_ms, 100 * few_ms / total))
            for t, tiles, shape in sorted(convs, reverse=True)[:a.top]:
                print("  %7.3f ms  tiles %4d  %s" % (t, tiles, shape))
            print(json.dumps(dict(model=name, B=B, forward_ms=round(total, 3), graph_ms=round(graph_ms, 3),
                                  conv_ms=round(conv_ms, 3),
                                  conv_launches=len(convs), few_tile_launches=len(few),
                                  few_tile_ms=round(few_ms, 3),
                                  kinds={k: round(v, 3) for k, v in by_kind.items()})), flush=True)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
