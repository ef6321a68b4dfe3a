#!/usr/bin/env python
"""Per-op timing of one eager training step on the library's executor (CUDA events around every
plan op, each run as its own acnn_run_ops range), grouped by op kind and by conv layer.  Also the
entry used under ncu (`--ncu` runs exactly one un-timed step after warm-up so `-s/-c` can select it).

    python tools/profile_step.py [--batch 256] [--ncu]
"""
import argparse
import os
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from assembled_cnn_b200.hparams import params_from_flags
from assembled_cnn_b200.model_fns import Model, Trainer
from bench import MODEL_FLAGS, TRAIN_FLAGS, synth_batch

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--ncu", action="store_true")
ap.add_argument("--top", type=int, default=40)
ap.add_argument("--conv-mtiles", type=int, default=-1,
                help="acnn_set_conv_mtiles mode: -1 auto, 1 one M tile per CTA tile, 2 two where legal")
ap.add_argument("--csv", default="", help="write every conv GEMM launch (ms, ideal, shape) here")
args = ap.parse_args()

B = args.batch
if args.conv_mtiles != -1:
    from assembled_cnn_b200 import _lib as _l
    _l.load().acnn_set_conv_mtiles(args.conv_mtiles)
params = params_from_flags(batch_size=B, **MODEL_FLAGS, **TRAIN_FLAGS)
model = Model(50, num_classes=1001, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
              anti_alias_filter_size=3)
tr = Trainer(model, params, 224, 224, use_cuda_graph=False)
x, y = synth_batch(tr.input_batch, 224, 1234)
x, y = x.cuda(), y.cuda()
for _ in range(2):
    tr.train_step(x, y)
torch.cuda.synchronize()
if args.ncu:
    from assembled_cnn_b200 import _lib
    c0 = _lib.load().acnn_launch_count()
    torch.cuda.profiler.start()          # ncu --profile-from-start off
    tr.train_step(x, y)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    print("launches in profiled step:", _lib.load().acnn_launch_count() - c0)
    sys.exit(0)

rt = tr.rt
records = []
orig_run = rt.run


def timed_run(ops):
    for op in ops:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        orig_run([op])
        b.record()
        records.append((op, a, b))


def timed_forward():
    rt.zero_step_buffers()
    timed_run(rt.plan.forward)


rt.run, rt.run_forward = timed_run, timed_forward
tr.train_step(x, y)
torch.cuda.synchronize()
del rt.run, rt.run_forward
by_kind = defaultdict(lambda: [0.0, 0])
rows = []
for op, a, b in records:
    ms = a.elapsed_time(b)
    by_kind[op.kind][0] += ms
    by_kind[op.kind][1] += 1
    if op.kind in ("conv", "conv_dgrad", "conv_wgrad"):
        g, _, aux = rt.plan.conv_info(op)       # the geometry the library launches (acnn_op_conv_info)
        Ho, Wo = g.out_hw()
        fl = 2.0 * g.B * Ho * Wo * g.Cout * g.kh * g.kw * g.Cin
        nin, nout = g.B * g.H * g.W * g.Cin, g.B * Ho * Wo * g.Cout
        byt = 2.0 * (nin + nout)
        if op.kind == "conv_dgrad":
            byt += 2.0 * nin * aux
        ideal = max(fl / 989e9, byt / 3350e6)   # ms: tensor vs HBM roofline (H100 SXM data sheet)
        rows.append((ms, op.kind, "%dx%d %d->%d k%d s%d" % (g.H, g.W, g.Cin, g.Cout, g.kh, g.stride),
                     fl / ms / 1e9, ideal))
total = sum(v[0] for v in by_kind.values())
print("total %.2f ms over %d ops" % (total, len(records)))
for k, (ms, n) in sorted(by_kind.items(), key=lambda kv: -kv[1][0]):
    print("%-20s %4d launches-ops %8.3f ms %5.1f%%" % (k, n, ms, 100 * ms / total))
print("conv GEMMs: measured %.2f ms, roofline (max of tensor / HBM per launch) %.2f ms"
      % (sum(r[0] for r in rows), sum(r[4] for r in rows)))
print("--- conv GEMM launches by gap to their roofline (ms, ideal ms, kind, shape, TFLOP/s)")
for ms, kind, shape, tf, ideal in sorted(rows, key=lambda r: r[4] - r[0])[:args.top]:
    print("%7.3f %7.3f %-11s %-28s %7.1f" % (ms, ideal, kind, shape, tf))
if args.csv:
    with open(args.csv, "w") as fh:
        fh.write("ms,ideal_ms,kind,shape,tflops\n")
        for ms, kind, shape, tf, ideal in rows:
            fh.write("%.4f,%.4f,%s,%s,%.1f\n" % (ms, ideal, kind, shape, tf))
