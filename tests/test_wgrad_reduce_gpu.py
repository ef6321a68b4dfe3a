"""The wgrad split-K reduction (wgrad_reduce_kernel, csrc/gemm.cu) at a production layer with a single
output tile: Assemble-ResNet-50 at B = 256, the 28x28 1x1 conv 64 -> 256.  Its default layout sums 131
partials per dw element, the longest chain of the c3 step, and not a multiple of the reducer's load
depth, so both its unrolled and its remainder loop run.  The result must equal
dw0 + (((0 + p_0) + p_1) + ... + p_130) in float32, bit for bit, where p_z is a one-split launch over
the pixels of split z."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _plan(lib, g, det=0):
    from assembled_cnn_b200 import _lib
    pix, splits, sps = C.c_int(), C.c_int(), C.c_int()
    _lib.check(lib.acnn_conv_wgrad_plan(g, 0, det, C.byref(pix), C.byref(splits), C.byref(sps)),
               "acnn_conv_wgrad_plan")
    return pix.value, splits.value, sps.value


def _wgrad(lib, g, x, dy, dw, det):
    from assembled_cnn_b200 import _lib
    _lib.check(lib.acnn_conv_wgrad(g, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), 0, det,
                                   torch.cuda.current_stream().cuda_stream), "acnn_conv_wgrad")


def test_one_tile_production_wgrad_equals_its_ordered_decomposition(lib):
    from assembled_cnn_b200._lib import ConvGeom
    B, H, Cin, Cout = 256, 28, 64, 256
    g = ConvGeom(B, H, H, Cin, Cout, 1, 1, 1, 0, 0, 0, 0)
    P = B * H * H
    assert lib.acnn_set_wgrad_splits(0) == 0 and lib.acnn_set_wgrad_pixels(0) == 0
    pix, splits, sps = _plan(lib, g)
    assert (pix, splits, sps) == (64, 131, 24)
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(P, Cin, device="cuda", generator=gen).bfloat16()
    dy = torch.randn(P, Cout, device="cuda", generator=gen).bfloat16()
    dw0 = torch.randn(Cout, Cin, device="cuda", generator=gen)
    dw = dw0.clone()
    _wgrad(lib, g, x, dy, dw, 0)
    # a 1x1 stride-1 conv is a plain GEMM over pixel rows: split z is a one-split launch on rows
    # [z * sps * pix, (z + 1) * sps * pix), which runs the same stages with the same MMAs
    parts = []
    for z in range(splits):
        p0, p1 = z * sps * pix, min((z + 1) * sps * pix, P)
        sg = ConvGeom(1, 1, p1 - p0, Cin, Cout, 1, 1, 1, 0, 0, 0, 0)
        assert _plan(lib, sg, det=1) == (pix, 1, -(-(p1 - p0) // pix))
        part = torch.zeros_like(dw)
        _wgrad(lib, sg, x[p0:p1], dy[p0:p1], part, 1)
        parts.append(part)
    torch.cuda.synchronize()
    t = np.zeros((Cout, Cin), np.float32)
    for p in parts:
        t = (t + p.cpu().numpy()).astype(np.float32)
    want = (dw0.cpu().numpy() + t).astype(np.float32)
    got = dw.cpu().numpy()
    if not np.array_equal(got, want):
        d = np.abs(got.astype(np.float64) - want)
        raise AssertionError("split-K dw differs from its ordered decomposition in %d of %d elements "
                             "(max |d| %.3e)" % (int((d > 0).sum()), d.size, d.max()))
    # and it is the weight gradient
    ref = dy.double().t() @ x.double()
    err = (dw.double() - dw0.double() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-4, err
