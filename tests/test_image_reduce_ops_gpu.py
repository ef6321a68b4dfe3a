"""The SE per-image reductions at an SE plan's production shapes, non-finite inputs in the reductions whose
last trip re-reads a clamped row, and fp16's rounding edges in the conv epilogues and bn_act.

  * acnn_se_gap (q = mean_hw(y*s + h)) and acnn_se_bwd_gate (de = sum_hw(g * (y*s + h))), modes 2 and 3 of
    image_reduce_kernel, in bf16, fp16 and fp32: at every (B, HW, C) of the SE ResNet-50 training plan at
    B = 256, 224 px, and at the grid edges (every accepted C, HW in {1, 2, 3, 5, 49}, B = 1), against a
    float64 restatement with oracle/stream_check.py's reduction-per-image tolerance; bit-identical on a
    repeated launch and under CUDA-graph replay.
  * Non-finite propagation: a +inf, a -inf and (separately) a NaN in the last row of a map whose last trip
    is partial, for bn_bwd_reduce, bn_bwd_reduce2, sk_bwd_gate, se_bwd_gate, se_gap and gap_fwd in fp16.
    Every output is +inf, -inf, NaN or finite exactly where the float64 reference is (fp16 training at a
    static loss scale does overflow: an inf gradient is a realistic input).
  * fp16 rounding edges with exact fp32 arithmetic (one nonzero product per output, power-of-two weights or
    scales, add values whose sum with the product is exact): the stored fp16 bits are torch's round-to-
    nearest-even .half() of the exact value, in the subnormal range (halfway cases included) and above
    65504 (inf) -- conv_fprop on the 1x1 GEMM, the im2col and the halo kernel, with and without the add /
    mask epilogue, and its batch-norm statistics rows (inf where the stored output is); conv_dgrad with
    add / mask; bn_act.
"""
import pytest
import torch

import test_stream_ops_gpu as S
from oracle import stream_check as SC

pytestmark = pytest.mark.gpu

ACNN_F16 = 3
DTYPES = {"bf16": (0, torch.bfloat16), "fp16": (ACNN_F16, torch.float16), "fp32": (1, torch.float32)}


def _ulp_f16(x):
    """Spacing of fp16 numbers at |x| (11 significant bits), float64; 2^-24 below 2^-14."""
    x = x.double().abs().clamp_min(2.0 ** -14)
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), (e - 11).to(torch.int64))


def _se_shapes():
    """Every (B, HW, C) of the se_gap / se_bwd_gate ops of the SE ResNet-50 v2 training plan (BigLittle
    branches: SE on 128 .. 2048 channels), B = 256, 224 px."""
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    plan = build_plan(ModelConfig(num_classes=1001, resnet_size=50, resnet_version=2, use_se_block=True),
                      256, 224, 224,
                      mixup_type=1, label_smoothing=0.1)
    return sorted({(op.B, op.HW, op.C) for op in plan.all_ops() if op.kind in ("se_gap", "se_bwd_gate")})


SE_SHAPES = _se_shapes()
SE_EDGES = [(1, hw, C) for C in S.CG_OK_C for hw in (1, 2, 3, 5, 49)]


def _se_rows_per_pass(C):
    """Rows one pass of image_reduce_kernel's CTA covers: one per thread of an 8-channel group."""
    return 256 // min(C // 8, 256)


def _se_inputs(B, HW, C, tdt, seed):
    return dict(y=S._rand((B, HW, C), tdt, seed), g=S._rand((B, HW, C), tdt, seed + 1),
                scale=S._rand((C,), torch.float32, seed + 2, 0.5, 1.0),
                shift=S._rand((C,), torch.float32, seed + 3, 0.5))


def _se_launch(lib, t, code, q, de):
    B, HW, C = t["y"].shape
    st = S._st()
    S._check(lib.acnn_se_gap(S._p(t["y"]), S._p(t["scale"]), S._p(t["shift"]), S._p(q), B, HW, C, code, st),
             "se_gap")
    S._check(lib.acnn_se_bwd_gate(S._p(t["g"]), S._p(t["y"]), S._p(t["scale"]), S._p(t["shift"]), S._p(de),
                                  B, HW, C, code, st), "se_bwd_gate")


def _se_refs(t):
    """float64 q, de and the magnitudes of their terms."""
    y, g = t["y"].double(), t["g"].double()
    ys = y * t["scale"].double()
    tt = ys + t["shift"].double()
    mag = ys.abs() + t["shift"].double().abs()
    HW = y.shape[1]
    return tt.sum(1) / HW, mag.sum(1) / HW, (g * tt).sum(1), (g.abs() * mag).sum(1)


def _se_case(lib, dt, B, HW, C, seed):
    code, tdt = DTYPES[dt]
    t = _se_inputs(B, HW, C, tdt, seed)
    q, de = S._nan((B, C), torch.float32), S._nan((B, C), torch.float32)
    _se_launch(lib, t, code, q, de)
    torch.cuda.synchronize()
    # one thread adds ceil(HW / rpb) rows in a chain, then lane 0 adds the rpb thread sums; each term is
    # an fma (and a product for de), the mean one more multiply by the fp32 1/HW
    rpb = _se_rows_per_pass(C)
    n_eff = -(-HW // rpb) + rpb
    qr, qm, der, dem = _se_refs(t)
    what = "se %s B=%d HW=%d C=%d" % (dt, B, HW, C)
    SC.assert_within(q, qr, SC.reduction_tol(qm, n_eff, extra_ops=4), what + " se_gap")
    SC.assert_within(de, der, SC.reduction_tol(dem, n_eff, extra_ops=4), what + " se_bwd_gate")
    return t, q, de


def test_se_plan_shapes_are_the_se_resnet50_v2_ones():
    assert SE_SHAPES == [(256, 49, 1024), (256, 49, 2048), (256, 196, 512), (256, 196, 1024),
                         (256, 784, 256), (256, 3136, 128)]


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("case", SE_SHAPES, ids=S._ids(SE_SHAPES))
def test_se_reductions_plan_shapes(lib, dt, case):
    """Against float64, then bit-identical on a repeated launch and under CUDA-graph replay."""
    B, HW, C = case
    code, _ = DTYPES[dt]
    t, q, de = _se_case(lib, dt, B, HW, C, seed=HW + C)
    q2, de2 = torch.empty_like(q), torch.empty_like(de)
    _se_launch(lib, t, code, q2, de2)
    qg, deg = torch.empty_like(q), torch.empty_like(de)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            _se_launch(lib, t, code, qg, deg)
    torch.cuda.current_stream().wait_stream(s)
    gr.replay()
    torch.cuda.synchronize()
    for a, b, what in ((q, q2, "se_gap repeat"), (de, de2, "se_bwd_gate repeat"), (q, qg, "se_gap graph"),
                       (de, deg, "se_bwd_gate graph")):
        assert torch.equal(a, b), what


@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_se_reductions_edges(lib, dt):
    """Every accepted channel count (C = 8 .. 2048: 1 .. 256 channel groups, 256 .. 1 rows per pass) at one
    image of 1, 2, 3, 5 and 49 rows: fewer rows than a pass, a partial last trip of 4 passes."""
    for B, HW, C in SE_EDGES:
        _se_case(lib, dt, B, HW, C, seed=C + HW)


# ---------------------------------------------------------------------------------------------------
# non-finite inputs in the last row
# ---------------------------------------------------------------------------------------------------
CH_POS, CH_NEG = 3, 5            # channels of the +inf / -inf (or of the NaN: CH_POS)


def _poison(row, kind):
    """row (a view of the last row) gets +inf / -inf in two channels, or a NaN in one."""
    if kind == "inf":
        row[CH_POS], row[CH_NEG] = float("inf"), float("-inf")
    else:
        row[CH_POS] = float("nan")


def _assert_same_nonfinite(got, ref, tol, what):
    """got is +inf, -inf, NaN exactly where ref is, and within tol of it elsewhere; ref has non-finite
    values (the test reaches what it is about)."""
    got, ref = got.double(), ref.double()
    bad = ~torch.isfinite(ref)
    assert bool(bad.any()), what + ": the reference has no non-finite value"
    for name, f in (("NaN", torch.isnan), ("+inf", torch.isposinf), ("-inf", torch.isneginf)):
        diff = f(got) != f(ref)
        assert not bool(diff.any()), "%s: %d elements differ in being %s (got %s where the reference is %s)" % (
            what, int(diff.sum()), name, got[diff][:4].tolist(), ref[diff][:4].tolist())
    SC.assert_within(got[~bad], ref[~bad], tol.double()[~bad], what + " (finite elements)")


def _trip_is_partial(M, step, rows_per_trip):
    return M % (rows_per_trip * step) != 0


NONFINITE_BN_SHAPES = [(3, 7, 5, 64), (256, 7, 7, 2048)]      # one partial trip; the last stage at B = 256


@pytest.mark.parametrize("kind", ["inf", "nan"])
@pytest.mark.parametrize("where", ["g", "y"])
@pytest.mark.parametrize("shape", NONFINITE_BN_SHAPES, ids=S._ids(NONFINITE_BN_SHAPES))
def test_bn_bwd_reduce_nonfinite_last_row(lib, shape, where, kind):
    """bn_bwd_reduce and bn_bwd_reduce2 in fp16: the non-finite value in row M - 1 of the gradient or of the
    normalised input; the partial rows against the float64 partial sums."""
    B, H, W, C = shape
    HW, M = H * W, B * H * W
    gamma, mean, rstd = S._bn_stats_inputs(C, 7)
    g = S._rand((B, H, W, C), torch.float16, 8)
    ya = (S._rand((B, H, W, C), torch.float32, 9) / rstd + mean).half()
    mb, rb = S._rand((C,), torch.float32, 10, 0.5), S._unif((C,), 11, 0.5, 2.0)
    yb = (S._rand((B, H, W, C), torch.float32, 12) / rb + mb).half()
    _poison((g if where == "g" else ya).view(M, C)[M - 1], kind)
    if where == "y":
        _poison(yb.view(M, C)[M - 1], kind)
    nparts = lib.acnn_bn_bwd_reduce_parts(B, HW, C)
    rpb = 256 // (C // 8)
    assert _trip_is_partial(M, nparts * rpb, 4), "no partial last trip at %s" % (shape,)
    p1 = S._nan((nparts, 2, C), torch.float32)
    pa, pb = S._nan((nparts, 2, C), torch.float32), S._nan((nparts, 2, C), torch.float32)
    st = S._st()
    S._check(lib.acnn_bn_bwd_reduce(S._p(g), S._p(ya), S._p(mean), S._p(rstd), None, None, S._p(p1), B, HW, C,
                                    ACNN_F16, st), "bn_bwd_reduce")
    S._check(lib.acnn_bn_bwd_reduce2(S._p(g), S._p(ya), S._p(yb), S._p(mean), S._p(rstd), S._p(mb), S._p(rb),
                                     S._p(pa), S._p(pb), B, HW, C, ACNN_F16, st), "bn_bwd_reduce2")
    torch.cuda.synchronize()
    n_eff = SC.bn_bwd_reduce_chain(M, C, nparts)
    what = "%s in %s, %s" % (kind, where, (B, H, W, C))
    for parts, y, mu, rs, name in ((p1, ya, mean, rstd, "bn_bwd_reduce"), (pa, ya, mean, rstd, "bn_bwd_reduce2 a"),
                                   (pb, yb, mb, rb, "bn_bwd_reduce2 b")):
        for k, (term, mag) in enumerate(S._bn_bwd_terms(g, y, mu, rs)):
            if where == "y" and k == 0:
                continue                      # sum g does not read y
            ref = S._partials(term, rpb, nparts)
            tol = SC.reduction_tol(S._partials(mag, rpb, nparts), n_eff, extra_ops=5)
            _assert_same_nonfinite(parts[:, k], ref, tol, "%s %s partial %d" % (name, what, k))


@pytest.mark.parametrize("kind", ["inf", "nan"])
def test_image_reductions_nonfinite_last_row(lib, kind):
    """se_gap, se_bwd_gate, gap_fwd and sk_bwd_gate in fp16 with the non-finite value in the last row of the
    last image (the row a partial trip's clamped loads re-read), other images finite."""
    st = S._st()
    f16 = torch.float16
    # se_* / gap: one CTA per image, rpb rows per pass, se_bwd_gate 4 passes per trip
    for B, HW, C in ((2, 49, 256), (3, 49, 2048), (2, 5, 64)):
        rpb = _se_rows_per_pass(C)
        assert _trip_is_partial(HW, rpb, 4)                 # se_bwd_gate's last trip of 4 passes
        for poisoned in ("y", "g"):
            t = _se_inputs(B, HW, C, f16, seed=HW + C)
            _poison(t[poisoned][B - 1, HW - 1], kind)
            q, de = S._nan((B, C), torch.float32), S._nan((B, C), torch.float32)
            _se_launch(lib, t, ACNN_F16, q, de)
            pooled = S._nan((B, C), f16)
            S._check(lib.acnn_gap_fwd(S._p(t[poisoned]), S._p(pooled), B, HW, C, ACNN_F16, st), "gap_fwd")
            torch.cuda.synchronize()
            n_eff = -(-HW // rpb) + rpb
            qr, qm, der, dem = _se_refs(t)
            what = "%s in %s, B=%d HW=%d C=%d" % (kind, poisoned, B, HW, C)
            if poisoned == "y":
                _assert_same_nonfinite(q, qr, SC.reduction_tol(qm, n_eff, extra_ops=4), "se_gap " + what)
            _assert_same_nonfinite(de, der, SC.reduction_tol(dem, n_eff, extra_ops=4), "se_bwd_gate " + what)
            x = t[poisoned].double()
            pr = x.sum(1) / HW
            tol = SC.reduction_tol(x.abs().sum(1) / HW, n_eff, extra_ops=2)
            _assert_same_nonfinite(pooled, pr, tol + _ulp_f16(pr.abs() + tol), "gap_fwd " + what)
    # sk_bwd_gate: one CTA per image, trips of 2 * rpb rows; the gradient dv carries the value (y passes
    # through a ReLU, whose fmaxf maps NaN to 0)
    for B, HW, f in ((2, 49, 512), (4, 49, 64)):
        rpb = 256 // (f // 8)
        assert _trip_is_partial(HW, rpb, 2)
        for poisoned in ("dv",):
            t = S._sk_inputs(B, HW, f, f16, seed=HW + f)
            _poison(t[poisoned][B - 1, HW - 1], kind)
            dA = S._nan((B, f), torch.float32)
            S._check(lib.acnn_sk_bwd_gate(S._p(t["dv"]), S._p(t["y"]), S._p(t["scale"]), S._p(t["shift"]),
                                          S._p(dA), B, HW, f, ACNN_F16, st), "sk_bwd_gate")
            torch.cuda.synchronize()
            _, u0, u1 = S._sk_u(t)
            dv = t["dv"].double()
            ref = (dv * (u0 - u1)).sum(1)
            n_eff = 2 * -(-HW // (2 * rpb)) + rpb
            tol = SC.reduction_tol((dv.abs() * (u0 + u1)).sum(1), n_eff, extra_ops=4)
            _assert_same_nonfinite(dA, ref, tol, "sk_bwd_gate %s in %s, B=%d HW=%d f=%d" % (kind, poisoned, B, HW, f))


# ---------------------------------------------------------------------------------------------------
# fp16 rounding edges: exact fp32 values, stored with one round-to-nearest-even
# ---------------------------------------------------------------------------------------------------
def _rne16(v32):
    """torch's RNE fp16 of fp32 values (exact fp32: the only rounding is this one)."""
    assert v32.dtype == torch.float32
    return v32.half()


def _assert_rne_bits(got, v32, what):
    """The stored fp16 bits equal .half() of the exact fp32 value; a zero may have either sign."""
    want = _rne16(v32)
    same = got.view(torch.int16) == want.view(torch.int16)
    zero = (want == 0) & (got == 0)
    bad = ~(same | zero)
    assert not bool(bad.any()), "%s: %d of %d stored values are not the RNE fp16 value; first: got %s want %s (exact %s)" % (
        what, int(bad.sum()), bad.numel(), got[bad][:4].tolist(), want[bad][:4].tolist(), v32[bad][:4].tolist())


def _exact_operands(shape, case, seed):
    """(x, add, k): fp16 x and add, and the exponent k of the weight 2^k, such that x * 2^k and x * 2^k + add
    are exact in fp32 -- 'sub': results m * 2^-25, |m| < 2^12 (fp16 subnormals and their halfway points, up to
    the smallest normals); 'ovf': x * 16 up to 2^20 and adds in 1/16 steps (|v| across 65504 / 65520: inf)."""
    g = S._gen(seed)
    if case == "sub":
        m = torch.randint(-2047, 2048, shape, generator=g, device="cuda")
        x = (m.float() * 2.0 ** -5).half()                              # exact: |m| < 2^11
        a = torch.randint(-1023, 1024, shape, generator=g, device="cuda")
        add = (a.float() * 2.0 ** -24).half()                           # fp16 subnormals
        return x, add, -20
    x = (torch.rand(shape, generator=g, device="cuda") * 8192 - 4096).half()     # |x * 16| < 65536 ...
    big = torch.rand(shape, generator=g, device="cuda") < 0.3
    x = torch.where(big, (torch.rand(shape, generator=g, device="cuda") * 2 - 1).sign().half() *
                    (torch.rand(shape, generator=g, device="cuda") * 61408 + 4096).half(), x)  # ... or beyond
    x.view(-1)[:4] = torch.tensor([4094.0, 4094.0, -4094.0, 4092.0], dtype=torch.float16)  # 65504, ...
    add = (torch.randint(-1024, 1025, shape, generator=g, device="cuda").float() / 16).half()
    add.view(-1)[:4] = torch.tensor([15.0, 16.0, -16.0, 0.0], dtype=torch.float16)  # 65519 -> 65504, 65520 -> inf
    return x, add, 4


def _geom(B, H, W, C, k):
    from assembled_cnn_b200._lib import ConvGeom
    p = k // 2
    return ConvGeom(B, H, W, C, C, k, k, 1, p, p, p, p)


def _pow2_identity(C, k, e, dgrad=False):
    """A k x k weight whose centre tap is 2^e * I ([Cout][kh][kw][Cin]; the dgrad layout is the same)."""
    w = torch.zeros(C, k, k, C, dtype=torch.float16, device="cuda")
    idx = torch.arange(C, device="cuda")
    w[idx, k // 2, k // 2, idx] = 2.0 ** e
    return w


@pytest.mark.parametrize("case", ["sub", "ovf"])
@pytest.mark.parametrize("path", ["gemm_1x1", "im2col_3x3", "halo_3x3"])
def test_fp16_conv_fprop_rounding_edges(lib, path, case):
    from assembled_cnn_b200 import _lib
    B, H, W, C = 2, 8, 8, 64
    k = 1 if path == "gemm_1x1" else 3
    g = _geom(B, H, W, C, k)
    x, add, e = _exact_operands((B, H, W, C), case, seed=len(path))
    if case == "ovf":                       # one sign of overflow per column for the statistics check
        sign = torch.where(torch.arange(C, device="cuda") % 2 == 0, 1.0, -1.0).half()
        x = x.abs() * sign
        add = add.abs() * sign
    mask = S._rand((B, H, W, C), torch.float16, 5)
    w = _pow2_identity(C, k, e)
    prod = x.float() * 2.0 ** e                                          # exact
    halo_mode = {"gemm_1x1": None, "im2col_3x3": 0, "halo_3x3": 2}[path]
    prev = lib.acnn_set_conv_halo(halo_mode) if halo_mode is not None else None
    try:
        parts = lib.acnn_conv_stats_parts(g)
        if path == "halo_3x3":
            lib.acnn_set_conv_halo(0)
            assert lib.acnn_conv_stats_parts(g) != parts, "the halo kernel does not take this geometry"
            lib.acnn_set_conv_halo(2)
        st = S._st()
        outs = {}
        for epi in ("plain", "add", "add_mask"):
            y = S._nan((B, H, W, C), torch.float16)
            sp = S._nan((parts, 2, C), torch.float32) if epi == "plain" else None
            _lib.check(lib.acnn_conv_fprop(g, x.data_ptr(), w.data_ptr(), y.data_ptr(), S._p(sp),
                                           S._p(add) if epi != "plain" else None,
                                           S._p(mask) if epi == "add_mask" else None, None, 0, ACNN_F16, 0, st),
                       "conv_fprop")
            outs[epi] = (y, sp)
        torch.cuda.synchronize()
    finally:
        if prev is not None:
            lib.acnn_set_conv_halo(prev)
    v = {"plain": prod, "add": prod + add.float()}
    v["add_mask"] = torch.where(mask > 0, v["add"], torch.zeros_like(prod))
    for epi, (y, _) in outs.items():
        _assert_rne_bits(y, v[epi], "conv_fprop %s %s %s" % (path, case, epi))
    want = _rne16(v["plain"])
    if case == "sub":
        sub = (want != 0) & (want.abs() < 2.0 ** -14)
        assert int(sub.sum()) > 1000 and bool(((v["plain"] * 2 ** 25).remainder(2) == 1).any())
    else:
        assert bool(want.isinf().any()) and bool((want.abs() == 65504).any())
        assert bool((_rne16(v["add"]).isinf() & ~want.isinf()).any())      # 65520 = 65504 + 16 -> inf
    # statistics rows of the stored output: inf in the columns where it is, finite elsewhere
    y, sp = outs["plain"]
    yd = y.double().reshape(-1, C)
    tot = sp.double().sum(0)
    n = yd.shape[0]
    for j, (ref, what) in enumerate(((yd.sum(0), "sum"), ((yd * yd).sum(0), "sum of squares"))):
        if case == "ovf":
            _assert_same_nonfinite(tot[j], ref, 2 * n * S.U * (yd.abs() ** (j + 1)).sum(0) + 1e-30,
                                   "conv_fprop %s statistics %s" % (path, what))
        else:
            SC.assert_within(tot[j], ref, 2 * n * S.U * (yd.abs() ** (j + 1)).sum(0) + 1e-45,
                             "conv_fprop %s statistics %s" % (path, what))
    if case == "ovf":
        rows_inf = ~torch.isfinite(sp[:, 1, :])
        col_inf = y.reshape(-1, C).isinf().any(0)
        assert torch.equal(rows_inf.any(0), col_inf)


@pytest.mark.parametrize("case", ["sub", "ovf"])
def test_fp16_conv_dgrad_add_mask_rounding_edges(lib, case):
    """conv_dgrad of a 1x1 conv with w = 2^k * I: dx = dy * 2^k (+ add) (* (mask > 0)), one RNE rounding."""
    from assembled_cnn_b200 import _lib
    B, H, W, C = 2, 8, 8, 64
    g = _geom(B, H, W, C, 1)
    dy, add, e = _exact_operands((B, H, W, C), case, seed=17)
    mask = S._rand((B, H, W, C), torch.float16, 18)
    wd = _pow2_identity(C, 1, e)
    prod = dy.float() * 2.0 ** e
    st = S._st()
    for epi in ("plain", "add", "add_mask"):
        dx = S._nan((B, H, W, C), torch.float16)
        _lib.check(lib.acnn_conv_dgrad(g, dy.data_ptr(), wd.data_ptr(), dx.data_ptr(),
                                       S._p(add) if epi != "plain" else None,
                                       S._p(mask) if epi == "add_mask" else None, ACNN_F16, 0, st), "conv_dgrad")
        torch.cuda.synchronize()
        v = prod if epi == "plain" else prod + add.float()
        if epi == "add_mask":
            v = torch.where(mask > 0, v, torch.zeros_like(v))
        _assert_rne_bits(dx, v, "conv_dgrad %s %s" % (case, epi))


@pytest.mark.parametrize("case", ["sub", "ovf"])
@pytest.mark.parametrize("relu", [False, True])
def test_fp16_bn_act_rounding_edges(lib, case, relu):
    """bn_act with scale 2^k and shift 0: out = a * 2^k (ReLU), one RNE rounding."""
    B, H, W, C = 2, 8, 8, 64
    a, _, e = _exact_operands((B, H, W, C), case, seed=23)
    scale = torch.full((C,), 2.0 ** e, device="cuda")
    shift = torch.zeros(C, device="cuda")
    out = S._nan((B, H, W, C), torch.float16)
    S._check(lib.acnn_bn_act(S._p(a), S._p(scale), S._p(shift), None, None, None, 0, None, int(relu), S._p(out),
                             B, H, W, C, ACNN_F16, S._st()), "bn_act")
    torch.cuda.synchronize()
    v = a.float() * 2.0 ** e
    if relu:
        v = v.clamp_min(0)
    _assert_rne_bits(out, v, "bn_act %s relu=%d" % (case, relu))
