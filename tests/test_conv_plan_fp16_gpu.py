"""Every fp16 conv GEMM launch of the c3 and c5 training plans (B = 256, 224 px; build_plan(...,
dtype="fp16")) against float64, element by element, with the checks of tests/test_conv_plan_bf16_gpu.py
(oracle/conv_check.py at fp16's spacing), and the fp16 range edges at plan geometries:

  * conv (B = 256 and B = 7, statistics rows, the bias + fp32 logits layer, repeats and CTA pairs bit for
    bit), dgrad (exactly the fused epilogue; zero-insert + stride-1 for the stride-2 convs) and wgrad
    (into a nonzero dw, split-K and deterministic, per element and tile by tile): the bf16 file's test
    bodies, run on fp16 operands with the fp16 plans' cases;
  * overflow and subnormal outputs on every kernel the tiling picks for fprop and dgrad -- the one-CTA
    (WG = 2) kernel on a 1x1 and an im2col 3x3 geometry, the two-CTA (WG = 1) kernel, the halo kernel,
    CTA pairs and (fprop) the space-to-depth stem.  The operands are random fp16 values scaled by powers
    of two so that a fraction of the outputs lands beyond 65520 (stored as inf) and some between 65504 and
    65520 (stored as 65504), or between 2^-24 and 2^-14 (subnormal) from subnormal operands; a wgrad on
    subnormal operands must match float64 in its fp32 dw.  Under dynamic loss scaling the data gradients
    reach fp16's overflow (the overflow check needs them stored as inf, not saturated); at scale 1 they
    are often subnormal (a flush to zero loses them).

The range operands carry a per-pixel factor 2^U(-3, 3), so that the outputs of one launch span a wide
range of magnitudes and a power of two can put a part of them across each edge.
"""
import ctypes as C
import math

import pytest
import torch

import test_conv_plan_bf16_gpu as T
from oracle import conv_check as CC
from test_conv_plan_bf16_gpu import _free  # noqa: F401  (autouse: frees the cache after every test)

pytestmark = pytest.mark.gpu

ACNN_F16 = T.ACNN_F16
F16_MAX, F16_INF_AT, F16_MIN_NORMAL, F16_MIN_SUB = 65504.0, 65520.0, 2.0 ** -14, 2.0 ** -24

CASES = CC.plan_cases(T._plans("fp16"))
CONV = [c for c in CASES if c.kind == "conv"]
DGRAD = [c for c in CASES if c.kind == "conv_dgrad"]
WGRAD = [c for c in CASES if c.kind == "conv_wgrad"]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    T.report("fp16")


# ---------------------------------------------------------------------------------------------------
# every launch of the fp16 plans, with the bf16 file's test bodies
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [256, 7])
@pytest.mark.parametrize("case", CONV, ids=[c.id() for c in CONV])
def test_fp16_conv_plan_geometry(lib, case, B):
    T.test_conv_plan_geometry(lib, case, B, "fp16")


@pytest.mark.parametrize("case", DGRAD, ids=[c.id() for c in DGRAD])
def test_fp16_dgrad_plan_geometry(lib, case):
    T.test_dgrad_plan_geometry(lib, case, "fp16")


@pytest.mark.parametrize("case", WGRAD, ids=[c.id() for c in WGRAD])
def test_fp16_wgrad_plan_geometry(lib, case):
    T.test_wgrad_plan_geometry(lib, case, "fp16")


# ---------------------------------------------------------------------------------------------------
# the kernel families of the range tests
# ---------------------------------------------------------------------------------------------------
def _gemm_geom(case):
    """The geometry of the GEMM the library launches for a plan case, as a 12-tuple: fprop's own (the
    stem's space-to-depth launch geometry), dgrad's transposed stride-1 conv of dy (acnn_conv_dgrad)."""
    g = case.geom
    if case.kind == "conv_dgrad":
        B, H, W, Cin, Cout, kh, kw, _, phl, phh, pwl, pwh = g
        return (B, H, W, Cout, Cin, kh, kw, 1, kh - 1 - phl, kh - 1 - phh, kw - 1 - pwl, kw - 1 - pwh)
    if case.x_wpad is not None:
        B, H, W, Cin, Cout, kh, kw, _, phl, phh, _, _ = g
        return (B, H, W, Cin * kw, Cout, kh, 1, 1, phl, phh, 0, 0)
    return tuple(g)


def _halo_slab_fits(Cin, Cout, n_aux):
    """csrc/gemm.cu halo_plan: the N tile's 3x3 weight slab stays in shared memory next to the 18 x 10
    pixel A stages and n_aux staged add / mask tiles (the halo kernel's default mode needs it)."""
    bn = 128 if Cout % 128 == 0 else 64 if Cout % 64 == 0 else 32
    cw = 64 if Cin % 64 == 0 else 32
    a_stage = -(-18 * 10 * cw * 2 // 1024) * 1024
    fixed = 1024 + 128 * bn * 2 * (1 + n_aux)
    slots = Cin // cw * 9
    return slots <= 32 and any((224 * 1024 - fixed - st * a_stage) // (bn * cw * 2) >= slots for st in (3, 2))


def _family(case, n_aux):
    """The conv GEMM kernel csrc/gemm.cu picks for the case with n_aux staged add / mask tiles under its
    default knobs (conv_choice: halo mode 1, tiling), and whether acnn_set_conv_cta_pairs(1) pairs its CTAs."""
    B, H, W, Cin, Cout, kh, kw, stride, phl, phh, pwl, pwh = _gemm_geom(case)
    K = kh * kw * Cin
    M = B * ((H + phl + phh - kh) // stride + 1) * ((W + pwl + pwh - kw) // stride + 1)
    halo = (kh, kw, stride, phl, phh, pwl, pwh) == (3, 3, 1, 1, 1, 1, 1) and H >= 56 and Cin % 64 == 0 \
        and case.x_wpad is None and _halo_slab_fits(Cin, Cout, n_aux)
    pairs = (not halo and Cout % 128 == 0 and Cin % 64 == 0 and K >= 512
             and -(-M // 256) * (Cout // 128) >= T.NUM_SMS // 2)
    bn2 = 64 if Cout % 64 == 0 and Cout >= 128 else 32
    if halo:
        return "halo", pairs
    if K <= 512 and Cout // bn2 >= 2:
        return "wg1", pairs
    return ("wg2-1x1" if kh * kw == 1 else "wg2-im2col"), pairs


def _pick(cases, family, n_aux):
    """The first plan case (smallest geometry first) of the kernel family with the range tests' epilogue
    (n_aux staged tiles: fprop add, dgrad add + mask); "stem": the space-to-depth stem; "pairs": a case
    CTA pairs apply to (run with them on)."""
    for c in cases:
        if c.bias or c.out_f32 or c.src:
            continue
        if family == "stem":
            if c.x_wpad is not None:
                return c
            continue
        if c.x_wpad is not None:
            continue
        f, pairs = _family(c, n_aux)
        if (pairs if family == "pairs" else f == family):
            return c
    raise AssertionError("no plan case of the %s family" % family)


FAMILIES = ["wg2-1x1", "wg2-im2col", "wg1", "halo", "pairs"]
FPROP_RANGE = {f: _pick(CONV, f, 1) for f in FAMILIES + ["stem"]}
DGRAD_RANGE = {f: _pick(DGRAD, f, 2) for f in FAMILIES}
REGIMES = ["overflow", "subnormal"]


def _ctas_per_sm(lib, geom, add, mask):
    """acnn_conv_ctas_per_sm of an fp16 launch: 1 or 2, or "halo" where the halo kernel runs it."""
    from assembled_cnn_b200._lib import ConvGeom
    n = C.c_int(-1)
    if lib.acnn_conv_ctas_per_sm(ConvGeom(*geom), ACNN_F16, int(add), int(mask), C.byref(n)):
        err = lib.acnn_last_error()
        assert b"halo" in err, err
        return "halo"
    return n.value


# resident CTAs per SM of each family
OCCUPANCY = {"wg2-1x1": 1, "wg2-im2col": 1, "wg1": 2, "halo": "halo", "pairs": 1, "stem": 2}


def test_fp16_range_cases_cover_every_kernel(lib):
    """The range cases run on the kernels they are named for, both occupancy classes among them."""
    seen = set()
    for cases in (FPROP_RANGE, DGRAD_RANGE):
        for f, c in cases.items():
            prev = lib.acnn_set_conv_cta_pairs(int(f == "pairs"))
            try:
                n = _ctas_per_sm(lib, _gemm_geom(c), True, c.kind == "conv_dgrad")
            finally:
                lib.acnn_set_conv_cta_pairs(prev)
            assert n == OCCUPANCY[f], (f, c.id(), n)
            seen.add(n)
    assert {1, 2, "halo"} <= seen


# ---------------------------------------------------------------------------------------------------
# range edges: overflow to inf, subnormal outputs
# ---------------------------------------------------------------------------------------------------
def _spread(shape, seed):
    """|randn| (at most 3.5) times a factor 2^U(-3, 3) per pixel, fp32."""
    v = torch.randn(shape, device="cuda", generator=T._gen(seed)).abs().clamp_max(3.5)
    f = torch.rand(shape[:-1] + (1,), device="cuda", generator=T._gen(seed + 1)) * 6 - 3
    return v * torch.exp2(f)


def _f16(t, e):
    """t * 2^e rounded to fp16 (exact where the result is a normal fp16 number)."""
    return (t * 2.0 ** e).half()


def _sample(t, n=1 << 20):
    t = t.flatten()
    return t[::max(1, t.numel() // n)].double()


def _log2_scale(ref_abs, regime):
    """The power of two that puts 30 % of |ref| beyond 65504 (overflow) or the median at 2^-19
    (subnormal: between 2^-24 and 2^-14)."""
    s = _sample(ref_abs)
    if regime == "overflow":
        return round(math.log2(F16_MAX / float(torch.quantile(s, 0.7))))
    return round(-19 - math.log2(float(torch.quantile(s, 0.5))))


def _check_regime(ref, acc, keep, regime, what):
    """The outputs (where keep) reach the edge the test is for."""
    r = ref.abs()[keep]
    a = acc[keep]
    if regime == "overflow":
        over = float((r - a >= F16_INF_AT).double().mean())
        assert 0.01 <= over <= 0.99, "%s: %.4f of the outputs overflow" % (what, over)
        assert bool(((r > F16_MAX) & (r < F16_INF_AT)).any()), what + ": no output between 65504 and 65520"
    else:
        sub = float(((r >= F16_MIN_SUB) & (r < F16_MIN_NORMAL)).double().mean())
        assert sub >= 0.5, "%s: %.4f of the outputs subnormal" % (what, sub)


def _subnormal_fraction(t):
    return float(((t != 0) & (t.abs() < F16_MIN_NORMAL)).double().mean())


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("family", list(FPROP_RANGE))
def test_fp16_fprop_range(lib, family, regime):
    """fprop with the statistics and add epilogues: outputs beyond 65520 are inf (their columns' statistics
    totals too), 65504 < |y| < 65520 rounds to 65504; subnormal outputs from subnormal activations are
    rounded to nearest even, not flushed."""
    case = FPROP_RANGE[family]
    geom = case.geom
    cg = CC.launch_geom(geom, case.x_wpad)
    B, H, W, Cin, Cout, kh, kw = geom[:7]
    K = kh * kw * Cin
    Ho, Wo = cg.out_hw()
    x0 = _spread(T._x_shape(geom, case.x_wpad), 51)
    if case.x_wpad is not None:
        x0[:, :, :case.x_wpad[0]] = 0
        x0[:, :, x0.shape[2] - case.x_wpad[1]:] = 0
    s = T._signs(Cout, 52)
    w0 = (torch.randn((Cout, kh, kw, Cin), device="cuda", generator=T._gen(53)).abs() / math.sqrt(K)
          * s.float()[:, None, None, None])
    # x: activation-like (fp16 normal) for overflow, subnormal for the subnormal outputs; the power of
    # two of w from the outputs of the first 16 images
    ex = 0 if regime == "overflow" else -16
    est, _ = T._fprop_ref(_f16(x0[:16], ex), w0.half(), T._with_batch(geom, 16), case.x_wpad)
    ew = _log2_scale(est.abs(), regime)
    del est
    x, w = _f16(x0, ex), _f16(w0, ew)
    del x0
    add = _f16(torch.randn((B, Ho, Wo, Cout), device="cuda", generator=T._gen(54)), 11 if regime == "overflow" else -20)
    y = T._nan((B, Ho, Wo, Cout), torch.float16)
    prev = lib.acnn_set_conv_cta_pairs(int(family == "pairs"))
    try:
        assert _ctas_per_sm(lib, _gemm_geom(case), True, False) == OCCUPANCY[family]
        sp = CC.stats_poison((lib.acnn_conv_stats_parts(cg), 2, Cout))        # a row per CTA (pair) of the launch
        T._check(lib.acnn_conv_fprop(cg, x.data_ptr(), w.data_ptr(), y.data_ptr(), sp.data_ptr(), add.data_ptr(),
                                     None, None, 0, ACNN_F16, 0, T._st()), "conv_fprop")
        torch.cuda.synchronize()
    finally:
        lib.acnn_set_conv_cta_pairs(prev)
    what = "fprop %s %s %s" % (regime, family, case.id())
    ref, mag = T._fprop_ref(x, w, geom, case.x_wpad)
    acc = CC.add_epilogue_bound(CC.acc_bound(mag, K), mag, add)
    del mag
    ref = ref + add.double()
    _check_regime(ref, acc, torch.ones_like(ref, dtype=torch.bool), regime, what)
    if regime == "subnormal":
        assert _subnormal_fraction(x) >= 0.5, what + ": the activations are not subnormal"
    T.REPORT["fp16"]["decided"][("conv range", what)] = CC.check_16bit(y, ref, acc, what, "fp16")
    del ref, acc
    if regime == "overflow":
        assert bool(torch.isinf(y).any()) and bool((y.abs() == F16_MAX).any()), what
    CC.check_stats(sp, y, what + " statistics")


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("family", list(DGRAD_RANGE))
def test_fp16_dgrad_range(lib, family, regime):
    """dgrad with the add + mask epilogue: dy at a loss-scale magnitude (2^11) with data gradients beyond
    65520 stored as inf, some of them under the mask (stored +-0, not NaN); or subnormal dy (scale 1)
    with subnormal data gradients, rounded to nearest even."""
    case = DGRAD_RANGE[family]
    geom = case.geom
    B, H, W, Cin, Cout, kh, kw = geom[:7]
    K = kh * kw * Cout
    dy0 = _spread((B, H, W, Cout), 61)
    s = T._signs(Cin, 62)
    w0 = torch.randn((Cout, kh, kw, Cin), device="cuda", generator=T._gen(63)).abs() / math.sqrt(K) * s.float()
    ed = 11 if regime == "overflow" else -16              # 2^11 x the spread operand: at most 57344
    est = T._dgrad_ref(w0.half(), _f16(dy0[:16], ed), T._with_batch(geom, 16))
    ew = _log2_scale(est.abs(), regime)
    del est
    dy, w = _f16(dy0, ed), _f16(w0, ew)
    del dy0
    wd = w.flip(1, 2).permute(3, 1, 2, 0).contiguous()
    add = _f16(torch.randn((B, H, W, Cin), device="cuda", generator=T._gen(64)), 11 if regime == "overflow" else -20)
    mask = T._mask((B, H, W, Cin), 65, torch.float16)
    dx = T._nan((B, H, W, Cin), torch.float16)
    prev = lib.acnn_set_conv_cta_pairs(int(family == "pairs"))
    try:
        assert _ctas_per_sm(lib, _gemm_geom(case), True, True) == OCCUPANCY[family]
        T._check(lib.acnn_conv_dgrad(CC.launch_geom(geom), dy.data_ptr(), wd.data_ptr(), dx.data_ptr(), add.data_ptr(), mask.data_ptr(),
                                     ACNN_F16, 0, T._st()), "conv_dgrad")
        torch.cuda.synchronize()
    finally:
        lib.acnn_set_conv_cta_pairs(prev)
    del wd
    what = "dgrad %s %s %s" % (regime, family, case.id())
    ref = T._dgrad_ref(w, dy, geom)
    mag = T._dgrad_ref(w.abs(), dy.abs(), geom)
    acc = CC.add_epilogue_bound(CC.acc_bound(mag, K), mag, add)
    del mag
    ref = ref + add.double()
    keep = mask > 0
    _check_regime(ref, acc, keep, regime, what)
    if regime == "overflow":
        hidden = ~keep & (ref.abs() - acc >= F16_INF_AT)
        assert bool(hidden.any()), what + ": the mask hides no inf"
    else:
        assert _subnormal_fraction(dy) >= 0.5, what + ": dy is not subnormal"
    CC.check_mask(dx, mask, what)
    k = keep.double()
    T.REPORT["fp16"]["decided"][("dgrad range", what)] = CC.check_16bit(dx, ref * k, acc * k, what, "fp16")
    if regime == "overflow":
        assert bool(torch.isinf(dx).any()), what


def _wgrad_range_case():
    """A 3x3 stride-1 wgrad of the fp16 plans on 28 x 28 maps (P = 200704 pixels)."""
    return next(c for c in WGRAD if c.geom[5] == 3 and c.geom[7] == 1 and c.geom[1] == 28 and c.x_wpad is None)


def test_fp16_wgrad_subnormal_operands(lib):
    """wgrad of subnormal x and dy (random signs, |values| mostly below 2^-14) into a nonzero fp32 dw, split-K
    and deterministic: per element and tile by tile against float64 (a flushed operand drops its products)."""
    case = _wgrad_range_case()
    geom = case.geom
    cg = CC.launch_geom(geom)
    B, _, _, Cin, Cout, kh, kw, stride = geom[:8]
    Ho, Wo = cg.out_hw()
    P = B * Ho * Wo
    x = _f16(torch.randn(T._x_shape(geom, None), device="cuda", generator=T._gen(71)), -16)
    dy = _f16(torch.randn((B, Ho, Wo, Cout), device="cuda", generator=T._gen(72)), -16)
    assert _subnormal_fraction(x) >= 0.5 and _subnormal_fraction(dy) >= 0.5
    dw0 = torch.randn((Cout, kh, kw, Cin), device="cuda", generator=T._gen(73)) * 2.0 ** -24
    xp = T._pad_x(x, geom, None)
    wshape = (Cout, Cin, kh, kw)
    ref = T._nhwc(torch.nn.grad.conv2d_weight(xp, wshape, T._nchw(dy), stride=stride)) + dw0.double()
    mag = T._nhwc(torch.nn.grad.conv2d_weight(xp.abs(), wshape, T._nchw(dy).abs(), stride=stride))
    del xp
    worst = []
    for det in (0, 1):
        dw = dw0.clone()
        T._check(lib.acnn_conv_wgrad(cg, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), ACNN_F16, det, T._st()),
                 "conv_wgrad")
        torch.cuda.synchronize()
        what = "wgrad subnormal %s det=%d" % (case.id(), det)
        chain = T._wgrad_chain(lib, cg, ACNN_F16, det)
        worst.append((CC.check_wgrad(dw, ref, mag, dw0, P, what, chain), CC.wgrad_tile_tol(min(P, chain))))
    T.REPORT["fp16"]["wgrad_tile"][("subnormal " + case.id(), P)] = worst
