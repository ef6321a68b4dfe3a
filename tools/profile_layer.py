#!/usr/bin/env python
"""Run one conv layer's fprop / dgrad / wgrad a few times (for `ncu --set full -k regex:...`).

    python tools/profile_layer.py --B 256 --H 14 --Cin 512 --Cout 1024 --k 3 [--reps 3]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from assembled_cnn_b200 import _lib

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=256)
ap.add_argument("--H", type=int, default=14)
ap.add_argument("--Cin", type=int, default=512)
ap.add_argument("--Cout", type=int, default=1024)
ap.add_argument("--k", type=int, default=3)
ap.add_argument("--stride", type=int, default=1)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--which", default="fprop,dgrad,wgrad")
a = ap.parse_args()

lib = _lib.load()
lo = (a.k - 1) // 2
hi = a.k - 1 - lo
g = _lib.ConvGeom(a.B, a.H, a.H, a.Cin, a.Cout, a.k, a.k, a.stride, lo, hi, lo, hi)
Ho, Wo = g.out_hw()
dev = "cuda"
x = torch.randn(a.B, a.H, a.H, a.Cin, device=dev).bfloat16()
w = (torch.randn(a.Cout, a.k, a.k, a.Cin, device=dev) * 0.05).bfloat16()
wd = (torch.randn(a.Cin, a.k, a.k, a.Cout, device=dev) * 0.05).bfloat16()
y = torch.empty(a.B, Ho, Wo, a.Cout, device=dev, dtype=torch.bfloat16)
dy = torch.randn(a.B, Ho, Wo, a.Cout, device=dev).bfloat16()
dx = torch.empty_like(x)
dw = torch.zeros(a.Cout, a.k, a.k, a.Cin, device=dev)
s1 = torch.zeros(a.Cout, device=dev)
s2 = torch.zeros(a.Cout, device=dev)
sp = torch.zeros(lib.acnn_conv_stats_parts(g), 2, a.Cout, device=dev)     # partial BN statistics rows
st = torch.cuda.current_stream().cuda_stream
flops = 2.0 * a.B * Ho * Wo * a.Cout * a.k * a.k * a.Cin


def timed(name, fn):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.reps
    print("%-6s %8.3f ms  %7.1f TFLOP/s" % (name, ms, flops / ms / 1e9))


if "fprop" in a.which:
    timed("fprop", lambda: _lib.check(lib.acnn_conv_fprop(
        g, x.data_ptr(), w.data_ptr(), y.data_ptr(), sp.data_ptr(), None, None, None, 0, 0, 0, st)))
if "dgrad" in a.which and a.stride == 1:
    timed("dgrad", lambda: _lib.check(lib.acnn_conv_dgrad(
        g, dy.data_ptr(), wd.data_ptr(), dx.data_ptr(), None, x.data_ptr(), 0, 0, st)))
if "wgrad" in a.which:
    timed("wgrad", lambda: _lib.check(lib.acnn_conv_wgrad(g, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), 0, 0, st)))
