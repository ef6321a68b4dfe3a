#!/usr/bin/env python
"""Launch the HBM-bound pooling kernels of the north star (blur-pool forward / backward, global average
pool forward / backward, the SK block's pooled descriptor, the BigLittle 3x3/2 average pool) once each
at their Assemble-ResNet-50 B=256 shapes, for a kernel profiler, and
print their CUDA-event times with the algorithmic GB/s (tensors read + written, bf16)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from assembled_cnn_b200 import _lib

lib = _lib.load()
dev = "cuda"
st = torch.cuda.current_stream().cuda_stream
B = 256
bf = lambda *s: torch.randn(*s, device=dev).bfloat16()
jobs = []


def add(name, nbytes, fn):
    jobs.append((name, nbytes, fn))


for H, C in ((56, 64), (28, 128)):
    x, out = bf(B, H, H, C), torch.empty(B, H // 2, H // 2, C, device=dev, dtype=torch.bfloat16)
    dout, dx = bf(B, H // 2, H // 2, C), torch.empty(B, H, H, C, device=dev, dtype=torch.bfloat16)
    n_in, n_out = x.numel(), out.numel()
    add("blurpool_fwd %dx%dx%d" % (H, H, C), 2 * (n_in + n_out),
        lambda x=x, out=out, H=H, C=C: lib.acnn_blurpool_fwd(x.data_ptr(), out.data_ptr(), B, H, H, C, 3, 2, 0, st))
    add("blurpool_bwd %dx%dx%d" % (H, H, C), 2 * (n_in + n_out),
        lambda dout=dout, dx=dx, H=H, C=C: lib.acnn_blurpool_bwd(dout.data_ptr(), dx.data_ptr(), None, None, B,
                                                                  H, H, C, 3, 2, 0, st))
for H, C in ((56, 256), (28, 512)):
    Ho = (H + 2 - 3) // 2 + 1
    x, out = bf(B, H, H, C), torch.empty(B, Ho, Ho, C, device=dev, dtype=torch.bfloat16)
    dout, dx, mask = bf(B, Ho, Ho, C), torch.empty(B, H, H, C, device=dev, dtype=torch.bfloat16), bf(B, H, H, C)
    add("avgpool_fwd 3x3/2 %dx%dx%d" % (H, H, C), 2 * (x.numel() + out.numel()),
        lambda x=x, out=out, H=H, C=C, Ho=Ho: lib.acnn_avgpool_fwd(x.data_ptr(), out.data_ptr(), B, H, H, C, 3, 2,
                                                                    1, Ho, Ho, 1, 0, st))
    add("avgpool_bwd 3x3/2 %dx%dx%d (+mask)" % (H, H, C), 2 * (2 * x.numel() + out.numel()),
        lambda dout=dout, dx=dx, mask=mask, H=H, C=C, Ho=Ho: lib.acnn_avgpool_bwd(
            dout.data_ptr(), dx.data_ptr(), None, mask.data_ptr(), B, H, H, C, 3, 2, 1, Ho, Ho, 1, 0, st))
x, pooled = bf(B, 49, 2048), torch.empty(B, 2048, device=dev, dtype=torch.bfloat16)
dpool, dx = bf(B, 2048), torch.empty(B, 49, 2048, device=dev, dtype=torch.bfloat16)
add("gap_fwd 7x7x2048", 2 * (x.numel() + pooled.numel()),
    lambda: lib.acnn_gap_fwd(x.data_ptr(), pooled.data_ptr(), B, 49, 2048, 0, st))
add("gap_bwd 7x7x2048 (+mask)", 2 * (2 * x.numel() + pooled.numel()),
    lambda: lib.acnn_gap_bwd(dpool.data_ptr(), x.data_ptr(), dx.data_ptr(), B, 49, 2048, 0, st))
for HW, f in ((3136, 64), (784, 128), (196, 256)):
    y = bf(B, HW, 2 * f)
    sc, sh = torch.rand(2 * f, device=dev) + 0.5, torch.randn(2 * f, device=dev)
    s = torch.empty(B, f, device=dev)
    add("sk_gap HW=%d f=%d" % (HW, f), 2 * y.numel() + 4 * s.numel(),
        lambda y=y, sc=sc, sh=sh, s=s, HW=HW, f=f: lib.acnn_sk_gap(y.data_ptr(), sc.data_ptr(), sh.data_ptr(),
                                                                  s.data_ptr(), B, HW, f, 0, st))

flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
peak = 3350.0     # GB/s: H100 SXM data sheet (HBM3)
once = os.environ.get("ACNN_PROFILE_ONCE") == "1"     # under ncu: warm-up + ONE profiled launch per job
for name, nbytes, fn in jobs:
    _lib.check(fn(), name)                      # warm-up (first-launch attributes)
    torch.cuda.synchronize()
    if once:
        flush.fill_(1)
        _lib.check(fn(), name)
        torch.cuda.synchronize()
        continue
    ts = []
    for _ in range(3):
        flush.fill_(1)                          # cold L2, as in the step (tensors >> L2 anyway)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.check(fn(), name)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = sorted(ts)[1]
    print("%-36s %7.1f us  %7.0f GB/s algorithmic = %.2f of %.0f" % (name, ms * 1e3, nbytes / ms / 1e6,
                                                                      nbytes / ms / 1e6 / peak, peak))
