#!/usr/bin/env python
"""Zero-shot retrieval top-k: the fused wgmma similarity + top-k (acnn_knn_topk, cosine, bf16) against
the reference's own procedure on the same GPU in the same run -- bf16 torch.mm over 10 000-query
chunks (metric/recall_metric.py:182-205 get_sorted_idx) followed by torch.topk, the l2 normalisation
included in both.

    python tools/bench_knn.py [--warmup 2] [--iters 5] [--sizes sop512,sop2048,cub512]

Times are CUDA-event times of whole calls (fused: prep + fused GEMM/top-k + merge kernels), median
of --iters after --warmup.  TFLOP/s = 2 nq nx d / time.  Prints the card name and power limit read in
the same run, one JSON line per case and a summary table."""
import argparse
import json
import statistics
import subprocess
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200.metrics import knn_topk  # noqa: E402

SIZES = {   # name -> (nq = nx, d, k values)
    "sop512": (60502, 512, (6, 101)),
    "sop2048": (60502, 2048, (6, 101)),
    "cub512": (5924, 512, (6,)),
}
CHUNK = 10000


def baseline(feats, k):
    f = torch.nn.functional.normalize(feats, dim=1).to(torch.bfloat16)
    out = [torch.topk(f[i:i + CHUNK] @ f.T, k, dim=1) for i in range(0, f.shape[0], CHUNK)]
    return torch.cat([o.indices for o in out])


def fused(feats, k):
    return knn_topk(feats, feats, k, "cosine", "bf16")[0]


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
    return statistics.median(times), min(times), max(times)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not readable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--sizes", default=",".join(SIZES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_knn: no CUDA device")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    rows = []
    for name in a.sizes.split(","):
        n, d, ks = SIZES[name]
        feats = torch.randn(n, d, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
        for k in ks:
            tf = timed(lambda: fused(feats, k), a.warmup, a.iters)
            tb = timed(lambda: baseline(feats, k), a.warmup, a.iters)
            agree = float((fused(feats, k).long() == baseline(feats, k)).float().mean())
            flop = 2.0 * n * n * d
            r = {"case": name, "nq": n, "nx": n, "d": d, "k": k,
                 "fused_ms": round(tf[0], 3), "fused_min_max_ms": [round(tf[1], 3), round(tf[2], 3)],
                 "baseline_ms": round(tb[0], 3), "baseline_min_max_ms": [round(tb[1], 3), round(tb[2], 3)],
                 "fused_tflops": round(flop / tf[0] / 1e9, 1), "baseline_tflops": round(flop / tb[0] / 1e9, 1),
                 "speedup": round(tb[0] / tf[0], 2), "index_agreement": round(agree, 4)}
            rows.append(r)
            print(json.dumps(r), flush=True)
            del r
        del feats
        torch.cuda.empty_cache()
    print("\n| case | k | fused ms | TFLOP/s | baseline ms | TFLOP/s | speedup |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s (%d x %d, d=%d) | %d | %.2f | %.0f | %.2f | %.0f | %.2fx |" % (
            r["case"], r["nq"], r["nx"], r["d"], r["k"], r["fused_ms"], r["fused_tflops"],
            r["baseline_ms"], r["baseline_tflops"], r["speedup"]))


if __name__ == "__main__":
    main()
