#!/usr/bin/env python
"""Time acnn_conv_wgrad at every distinct conv_wgrad geometry of the c3 training plan (Assemble-
ResNet-50, B = 256, 224 px), at the default split layout and over a sweep of forced split counts
(acnn_set_wgrad_splits).  Each figure is the median of --reps CUDA-event timings of one call after
--warmup calls, with the 10th-90th percentile spread beside it.  Prints the card and its power
limit, then one row per geometry and the per-step total (each geometry weighted by its number of
launches in the plan).

    python tools/profile_wgrad.py [--reps 25] [--warmup 5] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from assembled_cnn_b200 import _lib
from assembled_cnn_b200._lib import ConvGeom
from assembled_cnn_b200.plan import ModelConfig, build_plan

# the sweep: requested split counts (each re-normalised by the plan to a partition of the stages)
SWEEP = (1, 2, 3, 4, 6, 8, 11, 16, 22, 32, 44, 66, 88, 131, 176, 264)


def production_geoms():
    """{geometry key: (ConvGeom, launches per step)} of the c3 plan's conv_wgrad ops, as the library
    launches them: the stem's input is the W-padded space-to-depth image (model_exec.cu's launch
    geometry; acnn_op_conv_info reports the plan's, without that form)."""
    cfg = ModelConfig(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                      anti_alias_filter_size=3)
    plan = build_plan(cfg, 256, 224, 224, training=True, mixup_type=1, label_smoothing=0.1)
    out = {}
    for op in plan.backward:
        if op.kind != "conv_wgrad":
            continue
        g, wpad = op.geom, op.a.get("x_wpad")
        if wpad is None:
            cg = ConvGeom(*g.astuple())
        else:
            lo, hi = wpad
            row = (g.W + lo + hi) * g.Cin
            cg = ConvGeom(g.B, g.H, g.W, g.Cin * g.kw, g.Cout, g.kh, 1, 1, g.pad_h_lo, g.pad_h_hi,
                          0, 0, g.Cin, row, g.H * row, 0)
        key = tuple(getattr(cg, n) for n, _ in ConvGeom._fields_)
        n = out.get(key, (cg, 0))[1]
        out[key] = (cg, n + 1)
    return out


def plan_of(lib, g):
    pix, splits, sps = C.c_int(), C.c_int(), C.c_int()
    _lib.check(lib.acnn_conv_wgrad_plan(g, 0, 0, C.byref(pix), C.byref(splits), C.byref(sps)),
               "acnn_conv_wgrad_plan")
    return pix.value, splits.value, sps.value


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip() or name
    except (OSError, subprocess.SubprocessError):
        return name + " (power limit: nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-sweep", action="store_true", help="time the default layout only")
    ap.add_argument("--json", default="", help="write every timing here")
    a = ap.parse_args()
    assert a.reps >= 20, "at least 20 timed calls per figure"
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    print("card:", card())
    gen = torch.Generator(device="cuda").manual_seed(0)

    def time_call(g, x, dy, dw):
        def call():
            _lib.check(lib.acnn_conv_wgrad(g, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), 0, 0, st),
                       "acnn_conv_wgrad")
        for _ in range(a.warmup):
            call()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
               for _ in range(a.reps)]
        for e0, e1 in evs:
            e0.record()
            call()
            e1.record()
        torch.cuda.synchronize()
        t = sorted(e0.elapsed_time(e1) for e0, e1 in evs)
        return t[len(t) // 2], t[len(t) // 10], t[(9 * len(t)) // 10]

    rows, tot_default, tot_best = [], 0.0, 0.0
    print("%-34s %3s %6s %3s | %-24s | %-24s" % ("geometry (B HxW Cin->Cout k s)", "n", "pix",
                                                 "spl", "default ms (p10-p90)", "best swept"))
    for cg, nlaunch in production_geoms().values():
        Ho, Wo = cg.out_hw()
        P = cg.B * Ho * Wo
        xn = cg.B * cg.x_img_pitch if cg.x_img_pitch > 0 else cg.B * cg.H * cg.W * cg.Cin
        x = torch.randn(xn, device="cuda", generator=gen).bfloat16()
        dy = torch.randn(P * cg.Cout, device="cuda", generator=gen).bfloat16()
        dw = torch.zeros(cg.Cout * cg.kh * cg.kw * cg.Cin, device="cuda")
        pix, splits, sps = plan_of(lib, cg)
        default = time_call(cg, x, dy, dw)
        sweep = {}
        if not a.no_sweep:
            prev = lib.acnn_set_wgrad_splits(0)
            try:
                for s in SWEEP:
                    lib.acnn_set_wgrad_splits(s)
                    eff = plan_of(lib, cg)[1]
                    if eff not in sweep:
                        sweep[eff] = time_call(cg, x, dy, dw)
            finally:
                lib.acnn_set_wgrad_splits(prev)
        best = min(sweep.items(), key=lambda kv: kv[1][0]) if sweep else (splits, default)
        shape = "B%d %dx%d %d->%d k%dx%d s%d" % (cg.B, cg.H, cg.W, cg.Cin, cg.Cout, cg.kh, cg.kw,
                                                 cg.stride)
        print("%-34s %3d %6d %3d | %7.4f (%7.4f-%7.4f) | %3d: %7.4f (%7.4f-%7.4f)" % (
            shape, nlaunch, pix, splits, *default, best[0], *best[1]), flush=True)
        tot_default += nlaunch * default[0]
        tot_best += nlaunch * best[1][0]
        rows.append(dict(shape=shape, launches=nlaunch, P=P, pix=pix, splits=splits,
                         stages_per_split=sps, default_ms=default,
                         sweep_ms={str(k): v for k, v in sorted(sweep.items())}))
        del x, dy, dw
    print("conv_wgrad per step (medians x launches): default layout %.3f ms, best swept %.3f ms"
          % (tot_default, tot_best))
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(dict(card=card(), rows=rows, total_default_ms=tot_default,
                           total_best_ms=tot_best), fh, indent=1)


if __name__ == "__main__":
    main()
