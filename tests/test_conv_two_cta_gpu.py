"""The bf16 / fp16 fprop and dgrad conv GEMMs that run two CTAs per SM (one TMA producer warp + one
consumer warpgroup each, 128 x 64 or 128 x 32 tiles): every instantiation fits twice on an SM, and
ragged shapes with the add / mask / statistics epilogues match a float64 reference element by element
(oracle/conv_check.py) and repeat bit for bit.
"""
import itertools
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import conv_check as CC

pytestmark = pytest.mark.gpu

ACNN_BF16, ACNN_F16 = 0, 3
DT = {ACNN_BF16: (torch.bfloat16, "bf16"), ACNN_F16: (torch.float16, "fp16")}


def _geom(B, H, W, Cin, Cout, k, stride):
    from assembled_cnn_b200._lib import ConvGeom
    lo = (k - 1) // 2
    return ConvGeom(B, H, W, Cin, Cout, k, k, stride, lo, k - 1 - lo, lo, k - 1 - lo)


def _check(rc, what):
    from assembled_cnn_b200 import _lib
    _lib.check(rc, what)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rand(shape, seed, dt, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dt).cuda()


def _mask(shape, seed, dt):
    m = _rand(shape, seed, dt)
    m[m.abs() < 0.3] = 0.0                 # the exact zeros of a ReLU output
    return m


def _nan(shape, dt):
    return torch.full(shape, float("nan"), dtype=dt, device="cuda")


def _nhwc_conv(x, w_ohwi, g):
    """float64 NHWC conv of geometry g (and the same conv of |x|, |w|: the accumulation bound)."""
    xp = F.pad(x.double().permute(0, 3, 1, 2), (g.pad_w_lo, g.pad_w_hi, g.pad_h_lo, g.pad_h_hi))
    w = w_ohwi.double().permute(0, 3, 1, 2)
    ref = F.conv2d(xp, w, stride=g.stride).permute(0, 2, 3, 1)
    mag = F.conv2d(xp.abs(), w.abs(), stride=g.stride).permute(0, 2, 3, 1)
    return ref, mag


# B, H, W, Cin, Cout, k, stride.  The two-CTA kernel runs GEMMs with K = kh*kw*(channels in) <= 512
# (fprop: Cin, dgrad: Cout) and >= 2 N tiles; no 3x3 / stride-1 case has >= 56 rows (the halo kernel's)
CASES = [
    (3, 7, 7, 256, 128, 1, 1),       # M = 147: ragged last M tile, 2 M tiles for 264 CTAs
    (2, 14, 14, 32, 64, 3, 1),       # im2col, Cin 32: two taps per stage, partial last k-block
    (2, 12, 12, 32, 96, 3, 1),       # N tile 32, three N tiles
    (2, 10, 10, 16, 64, 3, 1),       # Cin 16: four taps per stage, partial last k-block (one chunk)
    (2, 16, 16, 32, 128, 3, 2),      # strided im2col
    (8, 40, 40, 64, 256, 1, 1),      # 100 M tiles x 4 N tiles: several tiles per CTA
]
# dgrad: N = Cin, K = kh*kw*Cout
DGRAD_CASES = [
    (3, 7, 7, 256, 128, 1, 1),       # K = 128, ragged M
    (2, 14, 14, 96, 32, 3, 1),       # im2col over 32 channels: partial last k-block; N tile 32
    (2, 9, 11, 128, 32, 3, 1),       # odd image shape: tiles cross image borders
    (8, 40, 40, 64, 256, 1, 1),      # K = 256, several tiles per CTA
]
PRECISIONS = [ACNN_BF16, ACNN_F16]


@pytest.mark.parametrize("prec", PRECISIONS, ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_fprop_two_cta(lib, case, prec):
    B, H, W, Cin, Cout, k, stride = case
    dt, fmt = DT[prec]
    g = _geom(*case)
    Ho, Wo = g.out_hw()
    K = k * k * Cin
    x = _rand((B, H, W, Cin), 1, dt)
    w = _rand((Cout, k, k, Cin), 2, dt, 1.0 / math.sqrt(K))
    add = _rand((B, Ho, Wo, Cout), 3, dt)
    mask = _mask((B, Ho, Wo, Cout), 4, dt)
    ref, mag = _nhwc_conv(x, w, g)
    acc = CC.acc_bound(mag, K)
    what = "fprop %s %s" % (case, fmt)

    def launch(with_aux):
        y = _nan((B, Ho, Wo, Cout), dt)
        sp = None if with_aux else _nan((lib.acnn_conv_stats_parts(g), 2, Cout), torch.float32)
        _check(lib.acnn_conv_fprop(g, x.data_ptr(), w.data_ptr(), y.data_ptr(),
                                   None if with_aux else sp.data_ptr(),
                                   add.data_ptr() if with_aux else None,
                                   mask.data_ptr() if with_aux else None, None, 0, prec, 0, _st()),
               "conv_fprop")
        torch.cuda.synchronize()
        return y, sp

    y, sp = launch(False)
    CC.check_16bit(y, ref, acc, what, fmt)
    CC.check_stats(sp, y, what + " statistics")
    y2, sp2 = launch(False)
    assert torch.equal(y.view(torch.int16), y2.view(torch.int16)), what + ": a second launch differs"
    assert torch.equal(sp, sp2), what + ": a second launch's statistics differ"

    ya, _ = launch(True)
    ref_a = ref + add.double()
    CC.check_16bit(torch.where(mask > 0, ya, torch.zeros_like(ya)),
                   torch.where(mask > 0, ref_a, torch.zeros_like(ref_a)),
                   CC.add_epilogue_bound(acc, mag, add), what + " + add, x mask", fmt)
    CC.check_mask(ya, mask, what + " mask")
    ya2, _ = launch(True)
    assert torch.equal(ya.view(torch.int16), ya2.view(torch.int16)), what + ": a second add/mask launch differs"


@pytest.mark.parametrize("prec", PRECISIONS, ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", DGRAD_CASES, ids=[str(c) for c in DGRAD_CASES])
def test_dgrad_two_cta(lib, case, prec):
    B, H, W, Cin, Cout, k, stride = case
    dt, fmt = DT[prec]
    g = _geom(*case)
    K = k * k * Cout
    dy = _rand((B, H, W, Cout), 11, dt)
    w = _rand((Cout, k, k, Cin), 12, dt, 1.0 / math.sqrt(K))
    wd = w.flip(1, 2).permute(3, 1, 2, 0).contiguous()          # [Cin][kh][kw][Cout], taps flipped
    add = _rand((B, H, W, Cin), 13, dt)
    mask = _mask((B, H, W, Cin), 14, dt)
    # dx = the stride-1 conv of dy with the flipped, transposed filter (the padding mirrors)
    from assembled_cnn_b200._lib import ConvGeom
    gt = ConvGeom(B, H, W, Cout, Cin, k, k, 1, k - 1 - g.pad_h_lo, k - 1 - g.pad_h_hi,
                  k - 1 - g.pad_w_lo, k - 1 - g.pad_w_hi)
    ref, mag = _nhwc_conv(dy, wd, gt)
    acc = CC.acc_bound(mag, K)
    what = "dgrad %s %s" % (case, fmt)
    outs = []
    for _ in range(2):
        dx = _nan((B, H, W, Cin), dt)
        _check(lib.acnn_conv_dgrad(g, dy.data_ptr(), wd.data_ptr(), dx.data_ptr(), add.data_ptr(),
                                   mask.data_ptr(), prec, 0, _st()), "conv_dgrad")
        torch.cuda.synchronize()
        outs.append(dx)
    dx = outs[0]
    ref_a = ref + add.double()
    CC.check_16bit(torch.where(mask > 0, dx, torch.zeros_like(dx)),
                   torch.where(mask > 0, ref_a, torch.zeros_like(ref_a)),
                   CC.add_epilogue_bound(acc, mag, add), what, fmt)
    CC.check_mask(dx, mask, what + " mask")
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), what + ": a second launch differs"


# every two-CTA instantiation: N tile 32 / 64 (Cout 64 / 128) x chunk width 16 / 32 / 64 x plain
# (1x1 / stride 1) / im2col (1x1 / stride 2) x bf16 / fp16, with the largest (add + mask) and the
# smallest epilogue staging
OCC = list(itertools.product([64, 128], [16, 32, 64], [1, 2], PRECISIONS, [False, True]))


@pytest.mark.parametrize("Cout,Cin,stride,prec,aux", OCC, ids=["-".join(map(str, c)) for c in OCC])
def test_two_ctas_fit_one_sm(lib, Cout, Cin, stride, prec, aux):
    import ctypes as C
    g = _geom(4, 14, 14, Cin, Cout, 1, stride)
    n = C.c_int(-1)
    _check(lib.acnn_conv_ctas_per_sm(g, prec, int(aux), int(aux), C.byref(n)), "conv_ctas_per_sm")
    assert n.value >= 2, "Cout %d Cin %d stride %d: %d CTA(s) per SM" % (Cout, Cin, stride, n.value)
