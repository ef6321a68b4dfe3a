#!/usr/bin/env python
"""Static figures of the layer plans the library builds (acnn_create: host logic, no GPU needed) for the
BASELINE configurations: variables, ops per phase, GEMM ops, algorithmic / executed GFLOP per image
(acnn_op_conv_info), device memory of one replica (flat buffers + workspace) and the largest per-GPU batch
that fits 76 GB of the H100's 80 GB of HBM3 (the rest left to the CUDA context and allocator).

    python tools/plan_stats.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from assembled_cnn_b200 import native
from assembled_cnn_b200.plan import ModelConfig

ASSEMBLE = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)
CASES = [
    ("C1 vanilla R50 eval, B=1", dict(resnet_size=50), 1, dict(training=False, with_loss=False)),
    ("C2 Assemble-R50 training-mode forward + loss, B=256 (forward ops of the training plan)", ASSEMBLE, 256,
     dict(training=True, label_smoothing=0.1)),
    ("C3 Assemble-R50 train step (mixup 1), B=256", ASSEMBLE, 256,
     dict(training=True, mixup_type=1, label_smoothing=0.1)),
    ("C3 in the fp32 parity mode, B=64", ASSEMBLE, 64,
     dict(training=True, mixup_type=1, label_smoothing=0.1, dtype="fp32")),
    ("C5 Assemble-R152 (alpha 1, beta 2) train step, B=128", dict(ASSEMBLE, resnet_size=152, bl_alpha=1, bl_beta=2),
     128, dict(training=True, mixup_type=1, label_smoothing=0.1)),
]


def device_bytes(nm):
    s = nm.sizes
    flat = 4 * (s.param_elems + s.state_elems) + 2 * s.w_fprop_elems
    if nm.config.training:
        flat += 4 * 2 * s.param_elems + 2 * s.w_dgrad_elems          # grads, momentum, dgrad-layout weights
    return flat, s.workspace_bytes


print("# Layer plans of the BASELINE configurations (built by acnn_create; `tools/plan_stats.py`)\n")
print("| configuration | variables (trainable elems) | ops fwd / bwd / update | GEMM ops | algorithmic / executed "
      "GFLOP per image | flat buffers | workspace | largest batch in 76 GB |")
print("|---|---:|---:|---:|---:|---:|---:|---:|")
for label, flags, B, kw in CASES:
    nm = native.NativeModel(ModelConfig(**flags), B, 224, 224, **kw)
    s = nm.sizes
    alg = ex = n = 0
    fwd_only = label.startswith("C2")
    for op in nm.forward + ([] if fwd_only else nm.backward):
        if op.kind in ("conv", "conv_dgrad", "conv_wgrad"):
            g, macs, _ = nm.conv_info(op)
            ho, wo = g.out_hw()
            alg += macs
            ex += g.B * ho * wo * g.Cout * g.kh * g.kw * g.Cin
            n += 1
    flat, ws = device_bytes(nm)
    # the workspace grows linearly with the batch (activations / gradients); the flat buffers do not
    per_img = ws / B
    fit = int((76e9 - flat) / per_img)
    print("| %s | %d (%.2f M) | %d / %d / %d | %d | %.2f / %.2f | %.2f GB | %.2f GB | %d |" % (
        label, s.n_variables, s.param_elems / 1e6, s.n_forward, 0 if fwd_only else s.n_backward,
        0 if fwd_only else s.n_update, n,
        2 * alg / B / 1e9, 2 * ex / B / 1e9, flat / 2 ** 30, ws / 2 ** 30, fit))
    nm.close()
print("\nOne statically shaped buffer per tensor of the step (no reuse): the backward recomputes BN / ReLU / SK "
      "from the raw conv outputs instead of storing masks, every forward tensor is live until its backward, and "
      "the gradient tensors are the only transient ones.  GFLOP: 2 x multiply-accumulates of the conv / dense "
      "GEMMs (forward only for C1 / C2; forward + dgrad + wgrad for the training steps).")
