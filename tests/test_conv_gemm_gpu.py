"""GPU parity of the wgmma implicit-GEMM convolutions (through the C ABI) against the CPU oracle.

Inputs are bf16-representable, so the only differences are fp32 accumulation order and the final
bf16 rounding of the output: tolerance = 2^-8 relative to the tensor's max magnitude for bf16
outputs, 1e-4 for fp32 outputs (wgrad, logits).
"""
import contextlib

import pytest
import torch

from oracle import tf_ops

pytestmark = pytest.mark.gpu

BF16_TOL = 2.0 ** -8
F32_TOL = 1e-4


def _geom(B, H, W, Cin, Cout, k, stride, pads=None):
    from assembled_cnn_b200._lib import ConvGeom
    kh, kw = (k, k) if isinstance(k, int) else k
    if pads is None:
        if stride == 1:
            pads = ((kh - 1) // 2, kh - 1 - (kh - 1) // 2, (kw - 1) // 2, kw - 1 - (kw - 1) // 2)
        else:  # fixed_padding
            pads = ((kh - 1) // 2, kh - 1 - (kh - 1) // 2, (kw - 1) // 2, kw - 1 - (kw - 1) // 2)
    return ConvGeom(B, H, W, Cin, Cout, kh, kw, stride, *pads)


def _ref_conv(x, w_hwio, g):
    import torch.nn.functional as F
    xp = F.pad(x, (0, 0, g.pad_w_lo, g.pad_w_hi, g.pad_h_lo, g.pad_h_hi))
    return tf_ops.conv2d(xp, w_hwio, g.stride, "VALID")


def _rand_bf16(*shape, seed=0, scale=1.0):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=gen) * scale).bfloat16().float()


def _relerr(a, b):
    return (a.double() - b.double()).abs().max().item() / max(b.abs().max().item(), 1e-30)


@pytest.fixture(autouse=True, params=[0, 2], ids=["epi_joint", "epi_split"])
def conv_split_epilogue(request, lib):
    """Every test of this file under both values of acnn_set_conv_split_epilogue /
    acnn_set_conv_split_mt2.  They select epilogue organisations of earlier kernel generations; the
    sm_90a kernels accept and ignore them, and these runs check that neither setting changes a
    result."""
    prev = lib.acnn_set_conv_split_epilogue(request.param)
    prev2 = lib.acnn_set_conv_split_mt2(request.param)
    yield request.param
    lib.acnn_set_conv_split_epilogue(prev)
    lib.acnn_set_conv_split_mt2(prev2)


@contextlib.contextmanager
def _mtiles(lib, mode):
    """acnn_set_conv_mtiles (M tiles per CTA tile in earlier kernel generations; accepted and ignored
    by the sm_90a kernels, which run one 128-pixel M tile per CTA: both settings must give the same
    results)."""
    prev = lib.acnn_set_conv_mtiles(mode)
    try:
        yield
    finally:
        lib.acnn_set_conv_mtiles(prev)


MT = [1, 2]
MT_IDS = ["mt1", "mt2"]

CASES = [
    # B, H, W, Cin, Cout, k, stride, pads
    (2, 16, 16, 64, 128, 1, 1, None),      # plain 1x1, SW128
    (2, 16, 16, 32, 64, 1, 1, None),       # plain 1x1, Cin 32 (SW64 A and B)
    (3, 7, 7, 256, 64, 1, 1, None),        # M = 147: ragged last tile, K loop 4 stages
    (2, 14, 14, 64, 64, 3, 1, None),       # im2col 3x3, tiles cross image borders
    (2, 12, 12, 32, 32, 3, 1, None),       # Cin 32: two taps per stage, odd tap count
    (2, 16, 16, 64, 64, 3, 2, None),       # strided 3x3 with fixed_padding
    (2, 12, 12, 16, 64, (4, 4), 1, (2, 1, 2, 1)),   # space-to-depth stem: 4x4, asymmetric pad
    (2, 16, 16, 64, 128, 1, 2, (0, 0, 0, 0)),       # strided 1x1 projection (rv=1)
    (2, 7, 7, 128, 256, 3, 1, None),       # 7x7 spatial, two N tiles
    (1, 10, 10, 128, 32, 3, 1, None),      # narrow N = 32
    (8, 40, 40, 64, 256, 3, 1, None),      # 100 M tiles x N = 256: the 128x256 tile, two halves
    (8, 40, 40, 256, 512, 1, 1, None),     # 1x1, two 256-wide N tiles; dgrad runs N = 256 too
]


@pytest.mark.parametrize("mt", MT, ids=MT_IDS)
@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_fprop_matches_oracle(lib, case, mt):
    from assembled_cnn_b200 import _lib
    B, H, W, Cin, Cout, k, stride, pads = case
    g = _geom(B, H, W, Cin, Cout, k, stride, pads)
    x = _rand_bf16(B, H, W, Cin, seed=1)
    w_hwio = _rand_bf16(g.kh, g.kw, Cin, Cout, seed=2, scale=(g.kh * g.kw * Cin) ** -0.5)
    ref = _ref_conv(x, w_hwio, g)
    Ho, Wo = g.out_hw()
    assert ref.shape == (B, Ho, Wo, Cout)
    xd = x.bfloat16().cuda()
    wd = w_hwio.permute(3, 0, 1, 2).contiguous().bfloat16().cuda()      # OHWI
    yd = torch.full((B, Ho, Wo, Cout), float("nan"), dtype=torch.bfloat16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    with _mtiles(lib, mt):
        parts = lib.acnn_conv_stats_parts(g)
        assert 1 <= parts <= 132
        # partial (sum, sumsq) rows: poisoned first -- the kernel must STORE every row it owns
        sp = torch.full((parts, 2, Cout), float("nan"), device="cuda")
        _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), yd.data_ptr(),
                                       sp.data_ptr(), None, None, None, 0, 0, 0, st),
                   "conv_fprop")
        sp2 = torch.full((parts, 2, Cout), float("nan"), device="cuda")
        _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), yd.data_ptr(),
                                       sp2.data_ptr(), None, None, None, 0, 0, 0, st))
    torch.cuda.synchronize()
    y = yd.float().cpu()
    assert _relerr(y, ref) < BF16_TOL
    assert torch.equal(sp, sp2)            # no atomics: bit-reproducible
    s1, s2 = sp[:, 0].double().sum(0).cpu(), sp[:, 1].double().sum(0).cpu()
    # fused batch-norm statistics are those of the stored (rounded) tensor
    assert _relerr(s1, y.sum(dim=(0, 1, 2))) < 1e-3 or (s1 - y.sum(dim=(0, 1, 2))).abs().max() < 1e-2
    assert _relerr(s2, (y * y).sum(dim=(0, 1, 2))) < 1e-3


@pytest.mark.parametrize("mt", MT, ids=MT_IDS)
@pytest.mark.parametrize("cout", [64, 128])
def test_many_tiles_per_cta(lib, mt, cout):
    """392 M tiles: every persistent CTA walks several tiles, the smem ring wraps many times and the
    register accumulators are reused tile after tile; with add + mask epilogue tiles."""
    from assembled_cnn_b200 import _lib
    B, H, W, Cin, Cout = 16, 56, 56, 64, cout
    g = _geom(B, H, W, Cin, Cout, 3, 1)
    x = _rand_bf16(B, H, W, Cin, seed=11)
    w_hwio = _rand_bf16(3, 3, Cin, Cout, seed=12, scale=(9 * Cin) ** -0.5)
    add = _rand_bf16(B, H, W, Cout, seed=13)
    mask = _rand_bf16(B, H, W, Cout, seed=14)
    ref = _ref_conv(x, w_hwio, g)
    st = torch.cuda.current_stream().cuda_stream
    xd, wd = x.bfloat16().cuda(), w_hwio.permute(3, 0, 1, 2).contiguous().bfloat16().cuda()
    addd, maskd = add.bfloat16().cuda(), mask.bfloat16().cuda()
    yd = torch.full((B, H, W, Cout), float("nan"), dtype=torch.bfloat16, device="cuda")
    y2 = torch.full((B, H, W, Cout), float("nan"), dtype=torch.bfloat16, device="cuda")
    with _mtiles(lib, mt):
        sp = torch.full((lib.acnn_conv_stats_parts(g), 2, Cout), float("nan"), device="cuda")
        _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), yd.data_ptr(),
                                       sp.data_ptr(), None, None, None, 0, 0, 0, st))
        _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), y2.data_ptr(), None,
                                       addd.data_ptr(), maskd.data_ptr(), None, 0, 0, 0, st))
    torch.cuda.synchronize()
    y = yd.float().cpu()
    assert _relerr(y, ref) < BF16_TOL
    assert _relerr(sp[:, 1].double().sum(0).cpu(), (y * y).sum(dim=(0, 1, 2))) < 1e-3
    assert _relerr(y2.float().cpu(), (ref + add) * (mask > 0)) < BF16_TOL


def test_fprop_epilogue_add_mask_bias(lib):
    from assembled_cnn_b200 import _lib
    B, H, W, Cin, Cout = 2, 8, 8, 64, 128
    g = _geom(B, H, W, Cin, Cout, 3, 1)
    x = _rand_bf16(B, H, W, Cin, seed=3)
    w_hwio = _rand_bf16(3, 3, Cin, Cout, seed=4, scale=(9 * Cin) ** -0.5)
    add = _rand_bf16(B, H, W, Cout, seed=5)
    mask = _rand_bf16(B, H, W, Cout, seed=6)
    bias = torch.randn(Cout, generator=torch.Generator().manual_seed(7))
    ref = _ref_conv(x, w_hwio, g)
    st = torch.cuda.current_stream().cuda_stream
    xd, wd = x.bfloat16().cuda(), w_hwio.permute(3, 0, 1, 2).contiguous().bfloat16().cuda()
    # add + mask, bf16 out
    yd = torch.empty(B, H, W, Cout, dtype=torch.bfloat16, device="cuda")
    addd, maskd = add.bfloat16().cuda(), mask.bfloat16().cuda()
    _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), yd.data_ptr(), None,
                                   addd.data_ptr(), maskd.data_ptr(), None, 0, 0, 0, st))
    torch.cuda.synchronize()
    want = (ref + add) * (mask > 0)
    assert _relerr(yd.float().cpu(), want) < BF16_TOL
    # bias, fp32 out (dense path)
    yf = torch.empty(B, H, W, Cout, dtype=torch.float32, device="cuda")
    biasd = bias.cuda()
    _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), yf.data_ptr(), None,
                                   None, None, biasd.data_ptr(), 1, 0, 0, st))
    torch.cuda.synchronize()
    assert _relerr(yf.cpu(), ref + bias) < F32_TOL


DGRAD_CASES = [c for c in CASES if c[6] == 1]


@pytest.mark.parametrize("mt", MT, ids=MT_IDS)
@pytest.mark.parametrize("case", DGRAD_CASES, ids=[str(c) for c in DGRAD_CASES])
def test_dgrad_matches_autograd(lib, case, mt):
    from assembled_cnn_b200 import _lib
    B, H, W, Cin, Cout, k, stride, pads = case
    if Cout % 16 or Cin % 32:
        pytest.skip("dgrad needs Cout%16==0 (its K) and Cin%32==0 (its N)")
    g = _geom(B, H, W, Cin, Cout, k, stride, pads)
    x = _rand_bf16(B, H, W, Cin, seed=1).requires_grad_(True)
    w_hwio = _rand_bf16(g.kh, g.kw, Cin, Cout, seed=2, scale=(g.kh * g.kw * Cin) ** -0.5)
    y = _ref_conv(x, w_hwio, g)
    dy = _rand_bf16(*y.shape, seed=8)
    (dx_ref,) = torch.autograd.grad(y, x, dy)
    # dgrad weight layout: [Cin][kh][kw][Cout] with taps flipped
    wdg = w_hwio.flip(0, 1).permute(2, 0, 1, 3).contiguous().bfloat16().cuda()
    dxd = torch.empty(B, H, W, Cin, dtype=torch.bfloat16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    dyd = dy.bfloat16().cuda()
    with _mtiles(lib, mt):
        _lib.check(lib.acnn_conv_dgrad(g, dyd.data_ptr(), wdg.data_ptr(),
                                       dxd.data_ptr(), None, None, 0, 0, st), "conv_dgrad")
    torch.cuda.synchronize()
    assert _relerr(dxd.float().cpu(), dx_ref) < BF16_TOL


@pytest.fixture(params=[64, 128], ids=["pix64", "pix128"])
def wgrad_pix(lib, request):
    """acnn_set_wgrad_pixels: pixels (GEMM K) per wgrad pipeline stage."""
    prev = lib.acnn_set_wgrad_pixels(request.param)
    yield request.param
    lib.acnn_set_wgrad_pixels(prev)


@pytest.mark.parametrize("mt", MT, ids=MT_IDS)
@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_wgrad_matches_autograd(lib, case, mt, wgrad_pix):
    from assembled_cnn_b200 import _lib
    B, H, W, Cin, Cout, k, stride, pads = case
    g = _geom(B, H, W, Cin, Cout, k, stride, pads)
    x = _rand_bf16(B, H, W, Cin, seed=1)
    w_hwio = _rand_bf16(g.kh, g.kw, Cin, Cout, seed=2).requires_grad_(True)
    y = _ref_conv(x, w_hwio, g)
    dy = _rand_bf16(*y.shape, seed=8)
    (dw_ref,) = torch.autograd.grad(y, w_hwio, dy)
    dwd = torch.zeros(Cout, g.kh, g.kw, Cin, dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    xd, dyd = x.bfloat16().cuda(), dy.bfloat16().cuda()
    with _mtiles(lib, mt):
        _lib.check(lib.acnn_conv_wgrad(g, xd.data_ptr(), dyd.data_ptr(), dwd.data_ptr(), 0, 0, st),
                   "conv_wgrad")
    torch.cuda.synchronize()
    got = dwd.cpu().permute(1, 2, 3, 0)      # OHWI -> HWIO
    assert _relerr(got, dw_ref) < F32_TOL


def test_large_shapes_linearity(lib):
    """BASELINE-size layer (stage-4 SK 3x3 512->1024 at 14x14, B=32): conv(a*x1+x2) property and
    a sampled check of output pixels against the oracle."""
    from assembled_cnn_b200 import _lib
    B, H, W, Cin, Cout = 32, 14, 14, 512, 1024
    g = _geom(B, H, W, Cin, Cout, 3, 1)
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=gen).bfloat16()
    w = (torch.randn(Cout, 3, 3, Cin, device="cuda", generator=gen) * (9 * Cin) ** -0.5).bfloat16()
    y = torch.empty(B, H, W, Cout, dtype=torch.bfloat16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.acnn_conv_fprop(g, x.data_ptr(), w.data_ptr(), y.data_ptr(), None, None,
                                   None, None, 0, 0, 0, st))
    torch.cuda.synchronize()
    # sampled pixels vs the oracle (image 0 and the last image)
    for b in (0, B - 1):
        ref = _ref_conv(x[b:b + 1].float().cpu(), w.float().cpu().permute(1, 2, 3, 0), g)
        assert _relerr(y[b:b + 1].float().cpu(), ref) < BF16_TOL


# ---------------------------------------------------------------------------------------------
# fp32 parity mode: operands split into three bf16 planes (acnn_split3), six cross products in the
# fp32 accumulator.  Inputs are full-precision fp32; tolerance 5e-6 relative to the output's
# max magnitude against an fp64 oracle (the tensor core's fp32 accumulation truncates: measured
# 1-3e-6 at K = 2304; fp32 rounding of the result itself is 6e-8).
# ---------------------------------------------------------------------------------------------
F32MODE_TOL = 5e-6


def _planes(lib, t):
    """fp32 CUDA tensor -> bf16 [3, ...] planes through the C ABI."""
    from assembled_cnn_b200 import _lib
    t = t.contiguous()
    out = torch.empty((3,) + tuple(t.shape), dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.acnn_split3(t.data_ptr(), out.data_ptr(), t.numel(),
                               torch.cuda.current_stream().cuda_stream), "split3")
    return out


def test_split3_reconstructs_fp32(lib):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(4096, generator=g) * torch.logspace(-6, 6, 4096)).cuda()
    pl = _planes(lib, x)
    torch.cuda.synchronize()
    rec = pl[0].double() + pl[1].double() + pl[2].double()
    assert ((rec - x.double()).abs() <= x.double().abs() * 2.0 ** -23).all()


@pytest.mark.parametrize("case", CASES[:10], ids=[str(c) for c in CASES[:10]])
def test_fp32_mode_fprop_dgrad_wgrad(lib, case):
    from assembled_cnn_b200 import _lib
    B, H, W, Cin, Cout, k, stride, pads = case
    g = _geom(B, H, W, Cin, Cout, k, stride, pads)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(B, H, W, Cin, generator=gen)
    w_hwio = torch.randn(g.kh, g.kw, Cin, Cout, generator=gen) * (g.kh * g.kw * Cin) ** -0.5
    xr = x.double().requires_grad_(True)
    wr = w_hwio.double().requires_grad_(True)
    ref = _ref_conv(xr, wr, g)
    dy = torch.randn(ref.shape, generator=gen)
    dx_ref, dw_ref = torch.autograd.grad(ref, (xr, wr), dy.double())
    Ho, Wo = g.out_hw()
    st = torch.cuda.current_stream().cuda_stream
    xp = _planes(lib, x.cuda())
    wp = _planes(lib, w_hwio.permute(3, 0, 1, 2).contiguous().cuda())           # OHWI
    y = torch.full((B, Ho, Wo, Cout), float("nan"), device="cuda")
    _lib.check(lib.acnn_conv_fprop(g, xp.data_ptr(), wp.data_ptr(), y.data_ptr(), None, None, None,
                                   None, 1, 1, wp[0].numel(), st), "conv_fprop fp32")
    torch.cuda.synchronize()
    assert _relerr(y.cpu(), ref.detach()) < F32MODE_TOL
    # wgrad (deterministic: no split-K), twice -> bit-identical
    dyp = _planes(lib, dy.cuda())
    dws = []
    for _ in range(2):
        dw = torch.zeros(Cout, g.kh, g.kw, Cin, device="cuda")
        _lib.check(lib.acnn_conv_wgrad(g, xp.data_ptr(), dyp.data_ptr(), dw.data_ptr(), 1, 1, st),
                   "conv_wgrad fp32")
        dws.append(dw)
    torch.cuda.synchronize()
    assert torch.equal(dws[0], dws[1])
    assert _relerr(dws[0].cpu().permute(1, 2, 3, 0), dw_ref) < F32MODE_TOL
    if stride == 1 and Cout % 16 == 0 and Cin % 32 == 0:
        wdg = _planes(lib, w_hwio.flip(0, 1).permute(2, 0, 1, 3).contiguous().cuda())
        dx = torch.full((B, H, W, Cin), float("nan"), device="cuda")
        _lib.check(lib.acnn_conv_dgrad(g, dyp.data_ptr(), wdg.data_ptr(), dx.data_ptr(), None, None,
                                       1, wdg[0].numel(), st), "conv_dgrad fp32")
        torch.cuda.synchronize()
        assert _relerr(dx.cpu(), dx_ref) < F32MODE_TOL


# ---------------------------------------------------------------------------------------------
# CTA pairs (clusters of two sharing the weight stages by TMA multicast): acnn_set_conv_cta_pairs(1)
# ---------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _pairs(lib, on):
    prev = lib.acnn_set_conv_cta_pairs(on)
    try:
        yield
    finally:
        lib.acnn_set_conv_cta_pairs(prev)


PAIR_CASES = [
    # B, H, W, Cin, Cout, k   (64-channel chunks; pairs where K >= 512 and the pair tiles fill the GPU)
    (64, 28, 28, 64, 256, 1),       # 1x1, one k-block, 196 pair tiles
    (16, 28, 28, 256, 512, 1),      # 1x1, K = 256, two N tiles
    (37, 14, 14, 128, 256, 3),      # 3x3 im2col, ragged M (7252 = 28.3 pair tiles x 2 N tiles: single-CTA path)
    (64, 14, 14, 128, 512, 3),      # 3x3 im2col, 49 pair tiles x 2 N tiles
    (50, 20, 20, 64, 256, 3),       # ragged: M = 20000 (78.1 pair tiles), tiles cross image borders
]


@pytest.mark.parametrize("case", PAIR_CASES, ids=[str(c) for c in PAIR_CASES])
def test_cta_pair_fprop_dgrad_match_single_cta_and_oracle(lib, case):
    from assembled_cnn_b200 import _lib
    B, H, W, Cin, Cout, k = case
    g = _geom(B, H, W, Cin, Cout, k, 1)
    x = _rand_bf16(B, H, W, Cin, seed=21)
    w_hwio = _rand_bf16(k, k, Cin, Cout, seed=22, scale=(k * k * Cin) ** -0.5)
    add = _rand_bf16(B, H, W, Cout, seed=23)
    mask = _rand_bf16(B, H, W, Cout, seed=24)
    st = torch.cuda.current_stream().cuda_stream
    xd = x.bfloat16().cuda()
    wd = w_hwio.permute(3, 0, 1, 2).contiguous().bfloat16().cuda()
    addd, maskd = add.bfloat16().cuda(), mask.bfloat16().cuda()
    outs = {}
    for on in (0, 1):
        with _pairs(lib, on):
            parts = lib.acnn_conv_stats_parts(g)
            sp = torch.full((parts, 2, Cout), float("nan"), device="cuda")
            y = torch.full((B, H, W, Cout), float("nan"), dtype=torch.bfloat16, device="cuda")
            y2 = torch.full((B, H, W, Cout), float("nan"), dtype=torch.bfloat16, device="cuda")
            _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), y.data_ptr(),
                                           sp.data_ptr(), None, None, None, 0, 0, 0, st), "fprop")
            _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), y2.data_ptr(), None,
                                           addd.data_ptr(), maskd.data_ptr(), None, 0, 0, 0, st))
            torch.cuda.synchronize()
            outs[on] = (y.float().cpu(), y2.float().cpu(), sp.double().sum(0).cpu(), parts)
    # identical math, identical k order within a tile: the pair path reproduces the single-CTA path
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert _relerr(outs[1][2], outs[0][2]) < 1e-5
    # and a sampled check against the oracle (first and last image)
    for b in (0, B - 1):
        ref = _ref_conv(x[b:b + 1], w_hwio, g)
        assert _relerr(outs[1][0][b:b + 1], ref) < BF16_TOL
        want = (ref + add[b:b + 1]) * (mask[b:b + 1] > 0)
        assert _relerr(outs[1][1][b:b + 1], want) < BF16_TOL


@contextlib.contextmanager
def _halo(lib, mode):
    prev = lib.acnn_set_conv_halo(mode)
    try:
        yield
    finally:
        lib.acnn_set_conv_halo(prev)


HALO_CASES = [
    # B, H, W, Cin, Cout   (3x3, stride 1, pad 1)
    (2, 20, 12, 64, 64),       # ragged patches both ways (20 = 16 + 4, 12 = 8 + 4); weights stationary
    (2, 16, 8, 64, 32),        # exactly one patch per image, N = 32
    (3, 7, 7, 64, 128),        # image smaller than a patch
    (2, 24, 20, 128, 128),     # two 64-channel chunks, weight tiles streamed through the ring
    (2, 18, 18, 256, 64),      # four chunks, N = 64, streamed
    (2, 20, 12, 32, 32),       # 32-channel rows (64-byte swizzle), N = 32
    (2, 20, 12, 32, 64),       # 32-channel rows, N = 64
    (2, 14, 14, 64, 256),      # two N tiles of 128 (mode 2 only)
    (12, 56, 56, 64, 128),     # 336 patches: several per CTA, rings and both accumulators wrap
    (10, 112, 112, 32, 32),    # the stem's shape class: 980 patches, 64-byte rows
]


@pytest.fixture(params=[1, 0], ids=["split_epilogue", "joint_epilogue"])
def halo_split(request, lib):
    """Both settings of acnn_set_conv_halo_split (one epilogue organisation on sm_90a)."""
    prev = lib.acnn_set_conv_halo_split(request.param)
    yield request.param
    lib.acnn_set_conv_halo_split(prev)


@pytest.mark.parametrize("case", HALO_CASES, ids=[str(c) for c in HALO_CASES])
def test_halo_kernel_fprop_dgrad_match_oracle_and_im2col(lib, case, halo_split):
    """The im2col-free 3x3 kernel (acnn_set_conv_halo(2): wherever it applies) against the oracle and
    against the im2col TMA kernel (mode 0): plain + statistics, add + mask epilogue, and the dgrad
    entry point.  The two kernels add the K terms in different orders (chunk-major vs tap-major), so
    they agree to a bf16 ulp, not bit for bit; two halo runs are bit-identical."""
    from assembled_cnn_b200 import _lib
    B, H, W, Cin, Cout = case
    g = _geom(B, H, W, Cin, Cout, 3, 1)
    x = _rand_bf16(B, H, W, Cin, seed=31)
    w_hwio = _rand_bf16(3, 3, Cin, Cout, seed=32, scale=(9 * Cin) ** -0.5)
    add = _rand_bf16(B, H, W, Cout, seed=33)
    mask = _rand_bf16(B, H, W, Cout, seed=34)
    st = torch.cuda.current_stream().cuda_stream
    xd = x.bfloat16().cuda()
    wd = w_hwio.permute(3, 0, 1, 2).contiguous().bfloat16().cuda()
    addd, maskd = add.bfloat16().cuda(), mask.bfloat16().cuda()
    outs = {}
    for mode in (0, 2, 2):
        with _halo(lib, mode):
            parts = lib.acnn_conv_stats_parts(g)
            assert 1 <= parts <= 132
            sp = torch.full((parts, 2, Cout), float("nan"), device="cuda")
            y = torch.full((B, H, W, Cout), float("nan"), dtype=torch.bfloat16, device="cuda")
            y2 = torch.full((B, H, W, Cout), float("nan"), dtype=torch.bfloat16, device="cuda")
            _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), y.data_ptr(),
                                           sp.data_ptr(), None, None, None, 0, 0, 0, st), "fprop")
            _lib.check(lib.acnn_conv_fprop(g, xd.data_ptr(), wd.data_ptr(), y2.data_ptr(), None,
                                           addd.data_ptr(), maskd.data_ptr(), None, 0, 0, 0, st))
            torch.cuda.synchronize()
            prev = outs.get(mode)
            outs[mode] = (y.float().cpu(), y2.float().cpu(), sp.double().sum(0).cpu(), sp.cpu())
            if prev is not None:           # second halo run: bit-identical, statistics rows included
                assert torch.equal(prev[0], outs[mode][0]) and torch.equal(prev[1], outs[mode][1])
                assert torch.equal(prev[3], outs[mode][3])
    ref = _ref_conv(x, w_hwio, g)
    yh, y2h, sh, _ = outs[2]
    assert _relerr(yh, ref) < BF16_TOL
    assert _relerr(y2h, (ref + add) * (mask > 0)) < BF16_TOL
    assert _relerr(yh, outs[0][0]) < BF16_TOL and _relerr(y2h, outs[0][1]) < BF16_TOL
    # statistics of the stored tensor, out-of-image patch pixels excluded
    assert _relerr(sh[1], (yh * yh).sum(dim=(0, 1, 2))) < 1e-3
    s1 = yh.double().sum(dim=(0, 1, 2))
    assert _relerr(sh[0], s1) < 1e-3 or (sh[0] - s1).abs().max() < 1e-2
    # dgrad entry point (its N is Cin, its K channels are Cout)
    xg = x.clone().requires_grad_(True)
    yy = _ref_conv(xg, w_hwio, g)
    dy = _rand_bf16(*yy.shape, seed=35)
    (dx_ref,) = torch.autograd.grad(yy, xg, dy)
    wdg = w_hwio.flip(0, 1).permute(2, 0, 1, 3).contiguous().bfloat16().cuda()
    dxd = torch.full((B, H, W, Cin), float("nan"), dtype=torch.bfloat16, device="cuda")
    if Cout % 64 == 0 or Cout == 32:
        with _halo(lib, 2):
            _lib.check(lib.acnn_conv_dgrad(g, dy.bfloat16().cuda().data_ptr(), wdg.data_ptr(),
                                           dxd.data_ptr(), None, None, 0, 0, st), "conv_dgrad")
        torch.cuda.synchronize()
        assert _relerr(dxd.float().cpu(), dx_ref) < BF16_TOL
