"""oracle/conv_check.py on synthetic CPU data: the checks accept what a correct kernel can return and
reject the errors they exist for, in bf16 and across fp16's overflow and subnormal range; and the case
lists of tests/test_conv_plan_bf16_gpu.py and tests/test_conv_plan_fp16_gpu.py are every distinct conv GEMM
launch of the c3 and c5 training plans in their format."""
import math

import torch

from oracle import conv_check as CC

U = CC.U32


def _bf(t):
    return t.bfloat16().double()


def _gemm(seed, M=4096, K=1152, N=64, one_sign=True):
    """A synthetic bf16 GEMM: (ref, mag, K) in float64, rows of one sign if one_sign (as the GPU tests'
    operands)."""
    g = torch.Generator().manual_seed(seed)
    a = _bf(torch.randn(M, K, generator=g).abs())
    b = _bf(torch.randn(K, N, generator=g) / K ** 0.5)
    if one_sign:
        b = b.abs() * (torch.randint(0, 2, (N,), generator=g) * 2 - 1).double()
    return a @ b, a.abs() @ b.abs(), K


def _perturbed(ref, acc, seed):
    """A value anywhere inside [ref - acc, ref + acc] (what an fp32 accumulation within the bound can give)."""
    g = torch.Generator().manual_seed(seed)
    return ref + (torch.rand(ref.shape, generator=g, dtype=torch.float64) * 2 - 1) * acc


def test_round16_is_nearest_even():
    x = torch.tensor([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8), 1 + 2.0 ** -8 + 2.0 ** -30,
                      2.0 - 2.0 ** -9, 3e-40, 0.0], dtype=torch.float64)
    want = torch.tensor([1.0, 1 + 2.0 ** -6, -1.0, 1 + 2.0 ** -7, 2.0, float(torch.tensor(3e-40).bfloat16()), 0.0],
                        dtype=torch.float64)
    assert torch.equal(CC.round16(x), want)
    # agrees with torch's fp32 -> bf16 conversion (round to nearest even) on fp32 inputs
    v = torch.randn(100000, generator=torch.Generator().manual_seed(0)) * 1e3
    assert torch.equal(CC.round16(v.double()), v.bfloat16().double())
    h = torch.randn(100000, generator=torch.Generator().manual_seed(1)) * 1e-3
    assert torch.equal(CC.round16(h.double(), "fp16"), h.half().double())


def test_exact_rounding_accepts_any_value_within_acc():
    ref, mag, K = _gemm(0)
    acc = CC.acc_bound(mag, K)
    for seed in range(3):
        got = CC.round16(_perturbed(ref, acc, seed)).bfloat16()
        frac = CC.check_16bit(got, ref, acc, "within acc")
        assert frac > 0.9, frac
    # and at the interval's ends
    CC.check_16bit(CC.round16(ref + acc).bfloat16(), ref, acc, "upper end")
    CC.check_16bit(CC.round16(ref - acc).bfloat16(), ref, acc, "lower end")


def _rejects(got, ref, acc, needle="decided"):
    try:
        CC.check_16bit(got, ref, acc, "mutant")
    except AssertionError as e:
        assert needle in str(e), str(e)
        return
    raise AssertionError("the check accepted the mutant")


def test_exact_rounding_rejects_truncation():
    ref, mag, K = _gemm(1)
    acc = CC.acc_bound(mag, K)
    v = _perturbed(ref, acc, 1).float()
    trunc = (v.view(torch.int32) & ~0xFFFF).view(torch.float32)        # toward zero
    # inside the per-element bound everywhere: only the exact-rounding check sees it
    assert bool(((trunc.double() - ref).abs() <= acc + CC.ulp16(ref.abs() + acc)).all())
    _rejects(trunc.bfloat16(), ref, acc)


def test_exact_rounding_rejects_one_ulp_on_one_element():
    ref, mag, K = _gemm(2)
    acc = CC.acc_bound(mag, K)
    got = CC.round16(ref)
    i = int(torch.nonzero(CC.decided(ref, acc).flatten())[1234])
    f = got.flatten()
    f[i] += CC.ulp16(f[i:i + 1])[0]
    _rejects(got.bfloat16(), ref, acc)


def test_exact_rounding_rejects_double_rounded_add_epilogue():
    """(acc + add) with the accumulator rounded to bf16 before the fp32 add, then rounded again."""
    ref, mag, K = _gemm(3)
    g = torch.Generator().manual_seed(3)
    add = _bf(torch.randn(ref.shape, generator=g).abs() * ref.sign() * 0.5)
    acc = CC.add_epilogue_bound(CC.acc_bound(mag, K), mag, add)
    v = _perturbed(ref, CC.acc_bound(mag, K), 3)
    twice = (v.float().bfloat16().float() + add.float()).bfloat16()
    _rejects(twice, ref + add, acc)
    # the kernel's order (fp32 add, one rounding) passes
    CC.check_16bit((v.float() + add.float()).bfloat16(), ref + add, acc, "fp32 add")


def test_exact_rounding_rejects_add_done_in_bf16():
    ref, mag, K = _gemm(4)
    g = torch.Generator().manual_seed(4)
    add = _bf(torch.randn(ref.shape, generator=g).abs() * ref.sign() * 0.5)
    acc = CC.add_epilogue_bound(CC.acc_bound(mag, K), mag, add)
    v = _perturbed(ref, CC.acc_bound(mag, K), 4)
    in_bf16 = v.bfloat16() + add.bfloat16()              # bf16 + bf16 -> bf16
    _rejects(in_bf16, ref + add, acc)


def test_mask_check_rejects_one_nonzero():
    g = torch.Generator().manual_seed(5)
    mask = torch.randn(64, 512, generator=g).bfloat16()
    mask[0, :8] = 0.0
    mask[1, :8] = -0.0
    got = torch.randn(64, 512, generator=g).bfloat16() * (mask > 0)
    CC.check_mask(got, mask, "masked")
    for r in (0, 1, 2):          # +0, -0 and a negative mask value
        c = int(torch.nonzero(~(mask[r] > 0))[0])
        bad = got.clone()
        bad[r, c] = 2.0 ** -20
        try:
            CC.check_mask(bad, mask, "mutant")
        except AssertionError:
            continue
        raise AssertionError("the mask check accepted a nonzero value at mask %r" % float(mask[r, c]))


def test_stats_check_rejects_a_missing_row_and_a_wrong_column():
    g = torch.Generator().manual_seed(6)
    y = torch.randn(1000, 64, generator=g).bfloat16()
    rows = torch.stack([y[i::4].float().sum(0) for i in range(4)]), torch.stack(
        [(y[i::4].float() ** 2).sum(0) for i in range(4)])
    rows = torch.stack(rows, 1)                     # [parts][2][C]
    CC.check_stats(rows, y, "rows")
    missing = rows.clone()
    missing[2] = float("nan")
    for bad in (missing, rows * torch.tensor([1.0, 1.0 + 2.0 ** -10]).view(1, 2, 1)):
        try:
            CC.check_stats(bad, y, "mutant")
        except AssertionError:
            continue
        raise AssertionError("the statistics check accepted a mutant")


def test_wgrad_tile_check_rejects_one_missing_pixel_in_one_tile():
    """P = 200k pixels, dw [Cout 64][8 x 128 rows]: one 128 x 64 tile without one pixel's contribution
    fails the tile-local bound, while the whole-tensor norm-relative error stays below it."""
    P, R, Cout = 200_000, 1024, 64
    g = torch.Generator().manual_seed(7)
    x = _bf(torch.randn(P, R, generator=g))
    dy = _bf(torch.randn(P, Cout, generator=g))
    ref = dy.T @ x                                   # [Cout][rows]
    mag = dy.abs().T @ x.abs()
    dw0 = torch.zeros_like(ref)
    # a correct fp32 result (rounding well inside the bound) passes
    ok = ref.float()
    worst = CC.check_wgrad(ok, ref, mag, dw0, P, "fp32-rounded")
    assert worst < 1e-6
    bad = ref.clone()
    p = 123_456
    bad[:, 256:384] -= torch.outer(dy[p], x[p, 256:384])
    whole = float((bad - ref).norm() / ref.norm())
    assert whole < CC.WGRAD_TILE_TOL, whole
    e = CC.wgrad_tile_errors(bad, ref)
    assert e.shape == (1, 8) and int(torch.argmax(e.flatten())) == 2
    try:
        CC.check_wgrad(bad.float(), ref, mag, dw0, P, "mutant")
    except AssertionError as err:
        assert "tile (0, 2)" in str(err), str(err)
    else:
        raise AssertionError("the tile check accepted a tile without one pixel")


def test_wgrad_tiles_follow_the_gemm_tiles():
    assert [CC.wgrad_bn(c) for c in (32, 64, 96, 128, 192, 256, 512, 2048)] == [32, 64, 64, 128, 128, 256, 256, 256]
    ref = torch.ones(96, 300, dtype=torch.float64)
    e = CC.wgrad_tile_errors(ref * (1 + 1e-3), ref)           # ragged both ways: 2 x 3 blocks
    assert e.shape == (2, 3) and torch.allclose(e, torch.full_like(e, 1e-3))


def _derive_cases(dtype):
    """The distinct conv GEMM launches of the c3 and c5 training plans, derived here on their own."""
    import bench
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    out = set()
    for name in ("c3", "c5"):
        cfg = ModelConfig(num_classes=1001, **bench.CONFIGS[name]["model"])
        plan = build_plan(cfg, 256, 224, 224, training=True, mixup_type=1, label_smoothing=0.1, dtype=dtype)
        ops = plan.all_ops()
        for i, op in enumerate(ops):
            if op.kind not in ("conv", "conv_dgrad", "conv_wgrad"):
                continue
            src = None
            if op.kind == "conv_dgrad":
                zi = [z for z in ops if z.kind == "zero_insert" and z.out == op.dy]
                if zi:
                    src = next(tuple(w.geom.astuple()) for w in ops if w.kind == "conv_wgrad" and w.dy == zi[0].dy)
            a = op.a
            out.add((op.kind, tuple(op.geom.astuple()), a.get("stats") is not None, a.get("add_src") is not None,
                     a.get("mask_src") is not None, a.get("bias") is not None, bool(a.get("out_f32")),
                     tuple(a["x_wpad"]) if a.get("x_wpad") is not None else None, src))
    return out


def test_gpu_case_list_is_every_plan_launch():
    for dtype in ("bf16", "fp16"):
        _check_case_list(dtype)


def _check_case_list(dtype):
    import importlib
    T = importlib.import_module("test_conv_plan_%s_gpu" % dtype)
    want = _derive_cases(dtype)
    got = [tuple(c) for c in T.CASES]
    assert len(got) == len(set(got)) and set(got) == want
    assert len(T.CONV) + len(T.DGRAD) + len(T.WGRAD) == len(want)
    kinds = [c[0] for c in want]
    assert (kinds.count("conv"), kinds.count("conv_dgrad"), kinds.count("conv_wgrad")) == (48, 55, 48)
    # the stem's space-to-depth conv and its wgrad
    stem = [c for c in want if c[7] is not None]
    assert sorted(c[0] for c in stem) == ["conv", "conv_wgrad"] and all(c[1][5] == 4 and c[1][3] == 16 for c in stem)
    # the stride-2 convs' data gradients, composed from zero-insert + stride-1 dgrad: both geometries
    zi = [c for c in want if c[8] is not None]
    assert len({c[8] for c in zi}) == 2 and all(c[8][7] == 2 and c[1][7] == 1 for c in zi)
    # the dense logits layer: bias + fp32 output
    dense = [c for c in want if c[5]]
    assert len(dense) == 1 and dense[0][6] and dense[0][1][3:5] == (2048, 1024)
    # every epilogue of the dgrad: none, add, mask, add + mask
    assert {(c[3], c[4]) for c in want if c[0] == "conv_dgrad"} == {(False, False), (True, False), (False, True),
                                                                      (True, True)}
    # the halo kernel's default mode (3x3 stride 1, H >= 56, Cin % 64 == 0) is reached at B = 256
    assert any(c[1][5] == 3 and c[1][7] == 1 and c[1][1] >= 56 and c[1][3] % 64 == 0 for c in want if c[0] == "conv")


# ---------------------------------------------------------------------------------------------------
# fp16: overflow to inf, subnormals
# ---------------------------------------------------------------------------------------------------
F16_MAX, F16_INF_AT = 65504.0, 65520.0


def test_round16_fp16_overflow_and_subnormals():
    x = torch.tensor([65504.0, 65510.0, 65519.99, 65520.0, 65536.0, 1e6, -65519.0, -65520.0, float("inf"),
                      2.0 ** -24, 1.5 * 2.0 ** -24, 2.0 ** -25, 2.0 ** -25 + 2.0 ** -40, 3 * 2.0 ** -15],
                     dtype=torch.float64)
    inf = float("inf")
    want = [65504.0, 65504.0, 65504.0, inf, inf, inf, -65504.0, -inf, inf,
            2.0 ** -24, 2 * 2.0 ** -24, 0.0, 2.0 ** -24, 3 * 2.0 ** -15]
    assert CC.round16(x, "fp16").tolist() == want
    # torch's fp32 -> fp16 conversion (round to nearest even, overflow to inf) agrees on fp32 inputs,
    # across the overflow threshold and through the subnormals
    g = torch.Generator().manual_seed(11)
    for v in (60000 + torch.rand(100000, generator=g) * 10000, torch.randn(100000, generator=g) * 1e-5):
        s =torch.where(torch.rand(v.shape, generator=g) < 0.5, -v, v)
        assert torch.equal(CC.round16(s.double(), "fp16"), s.half().double())
    # the spacing: 2^-24 through the subnormals, 32 in the top binade and at inf; bf16 unchanged
    u = CC.ulp16(torch.tensor([0.0, 2.0 ** -30, 2.0 ** -14, 1.0, 65504.0, 1e9, inf]), "fp16")
    assert u.tolist() == [2.0 ** -24, 2.0 ** -24, 2.0 ** -24, 2.0 ** -10, 32.0, 32.0, 32.0]
    assert CC.ulp16(torch.tensor([1.0, 3e38, inf])).tolist() == [2.0 ** -7, 2.0 ** 120, 2.0 ** 120]


def _gemm16(seed, scale_to, M=4096, K=576, N=64):
    """A synthetic fp16 GEMM with one sign per output column and a row factor 2^U(-3, 3), scaled by a
    power of two so that 30 % of |ref| lies beyond 65504 ("overflow") or its median at 2^-19
    ("subnormal", from subnormal a): (ref, mag, K, a, b) in float64."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).abs().clamp_max(3.5) * torch.exp2(torch.rand(M, 1, generator=g) * 6 - 3)
    b = torch.randn(K, N, generator=g).abs() / K ** 0.5 * (torch.randint(0, 2, (N,), generator=g) * 2 - 1)
    ea = 0 if scale_to == "overflow" else -16
    a16 = (a * 2.0 ** ea).half().double()
    r = (a16 @ b.half().double()).abs()
    if scale_to == "overflow":
        eb = round(math.log2(F16_MAX / float(torch.quantile(r.flatten()[::7], 0.7))))
    else:
        eb = round(-19 - math.log2(float(r.median())))
    b16 = (b * 2.0 ** eb).half().double()
    return a16 @ b16, a16.abs() @ b16.abs(), K, a16, b16


def _rejects16(got, ref, acc, needle):
    try:
        CC.check_16bit(got, ref, acc, "mutant", "fp16")
    except AssertionError as e:
        assert needle in str(e), str(e)
        return
    raise AssertionError("the check accepted the mutant")


def test_fp16_accepts_any_value_within_acc_across_overflow():
    ref, mag, K, _, _ = _gemm16(20, "overflow")
    acc = CC.acc_bound(mag, K)
    lo, hi = CC.round16(ref - acc, "fp16"), CC.round16(ref + acc, "fp16")
    straddle = (lo != hi) & (torch.isinf(lo) | torch.isinf(hi))
    assert float((lo.abs() == float("inf")).double().mean()) > 0.1 and int(straddle.sum()) > 0
    assert bool(((ref.abs() > F16_MAX) & (ref.abs() < F16_INF_AT)).any())
    for seed in range(3):
        got = CC.round16(_perturbed(ref, acc, seed), "fp16").half()
        assert bool(torch.isinf(got).any()) and bool((got.abs() == F16_MAX).any())
        CC.check_16bit(got, ref, acc, "within acc", "fp16")
    CC.check_16bit(CC.round16(ref + acc, "fp16").half(), ref, acc, "upper end", "fp16")
    CC.check_16bit(CC.round16(ref - acc, "fp16").half(), ref, acc, "lower end", "fp16")
    # the straddling elements may be 65504 or the inf, of the right sign -- not the other sign's inf
    got = CC.round16(ref, "fp16")
    for v in (F16_MAX, float("inf")):
        g2 = torch.where(straddle, torch.full_like(got, v).copysign(ref), got)
        CC.check_16bit(g2.half(), ref, acc, "straddle %g" % v, "fp16")
    _rejects16(torch.where(straddle, torch.full_like(got, float("inf")).copysign(-ref), got).half(), ref, acc,
               "outside")


def test_fp16_rejects_a_saturating_store():
    ref, mag, K, _, _ = _gemm16(21, "overflow")
    acc = CC.acc_bound(mag, K)
    v = _perturbed(ref, acc, 21).float()                    # the fp32 accumulator
    sat = v.clamp(-F16_MAX, F16_MAX).half()                 # cvt.rn.satfinite
    CC.check_16bit(v.half(), ref, acc, "rn", "fp16")
    _rejects16(sat, ref, acc, "overflow")


def test_fp16_rejects_truncation_and_one_ulp():
    ref, mag, K, _, _ = _gemm16(22, "overflow")
    keep = ref.abs() < 60000                                # the finite, normal range of the same data
    ref = torch.where(keep, ref, torch.zeros_like(ref))
    mag = torch.where(keep, mag, torch.zeros_like(mag))
    acc = CC.acc_bound(mag, K)
    v = _perturbed(ref, acc, 22)
    q = CC.ulp16(v, "fp16")
    trunc = torch.trunc(v.float().double() / q) * q          # fp32 -> fp16 toward zero
    assert bool(((trunc - ref).abs() <= acc + CC.ulp16(ref.abs() + acc, "fp16")).all())
    _rejects16(trunc.half(), ref, acc, "decided")
    got = CC.round16(ref, "fp16")
    i = int(torch.nonzero((CC.decided(ref, acc, "fp16") & (ref != 0)).flatten())[777])
    f = got.flatten()
    f[i] += CC.ulp16(f[i:i + 1], "fp16")[0]
    _rejects16(got.half(), ref, acc, "decided")


def test_fp16_rejects_double_rounding_through_bf16():
    ref, mag, K, _, _ = _gemm16(23, "overflow")
    acc = CC.acc_bound(mag, K)
    v = _perturbed(ref, acc, 23).float()
    _rejects16(v.bfloat16().half(), ref, acc, "outside")        # 8 significant bits: beyond the bound


def test_fp16_subnormal_outputs_and_flush_to_zero():
    ref, mag, K, a, _ = _gemm16(24, "subnormal")
    assert float(((a != 0) & (a.abs() < 2.0 ** -14)).double().mean()) > 0.5          # subnormal operands
    sub = (ref.abs() >= 2.0 ** -24) & (ref.abs() < 2.0 ** -14)
    assert float(sub.double().mean()) > 0.5
    acc = CC.acc_bound(mag, K)
    v = _perturbed(ref, acc, 24).float()
    frac = CC.check_16bit(v.half(), ref, acc, "subnormal", "fp16")
    assert frac > 0.99, frac                 # a subnormal ulp (2^-24) dwarfs the accumulation bound
    ftz = torch.where(v.abs() < 2.0 ** -14, torch.zeros_like(v), v).half()
    _rejects16(ftz, ref, acc, "outside")


def test_fp16_mask_of_an_inf_is_zero_not_nan():
    g = torch.Generator().manual_seed(25)
    y = (torch.randn(64, 512, generator=g) * 60000).half()
    assert bool(torch.isinf(y).any())
    mask = torch.randn(64, 512, generator=g).half()
    mask[0, :8] = 0.0
    mask[1, :8] = -0.0
    assert bool((torch.isinf(y) & ~(mask > 0)).any())
    CC.check_mask(torch.where(mask > 0, y, torch.zeros_like(y)), mask, "and")
    CC.check_mask(torch.where(mask > 0, y, -torch.zeros_like(y)), mask, "-0")
    try:
        CC.check_mask(y * (mask > 0).half(), mask, "multiply")          # inf * 0 = NaN
    except AssertionError as e:
        assert "nan" in str(e), str(e)
    else:
        raise AssertionError("the mask check accepted NaN for a masked inf")


def _rows(y, parts=4):
    yf = y.float()
    return torch.stack([torch.stack([yf[i::parts].sum(0), (yf[i::parts] ** 2).sum(0)]) for i in range(parts)])


def test_fp16_stats_with_inf_columns():
    g = torch.Generator().manual_seed(26)
    y = (torch.randn(1000, 64, generator=g).abs() * 20000).half()
    y[:, 1::2] = -y[:, 1::2]                              # one sign per column
    y[:, :8] = (y[:, :8].float() * 4).half()              # overflow in columns 0 .. 7
    inf_cols = torch.isinf(y).any(0)
    assert 0 < int(inf_cols.sum()) < 64
    rows = _rows(y)
    CC.check_stats(rows, y, "inf columns")
    # a finite statistics row where the stored output holds an inf (e.g. the sums of the saturated values)
    sat = _rows(y.float().clamp(-F16_MAX, F16_MAX).half())
    for bad, needle in ((sat, "inf"), (torch.where(torch.arange(4).view(4, 1, 1) == 2, CC.stats_poison(
            rows.shape, "cpu"), rows), "poison"), (rows * torch.tensor([1.0, 1.0 + 2.0 ** -10]).view(1, 2, 1), "bound")):
        try:
            CC.check_stats(bad, y, "mutant")
        except AssertionError as e:
            assert needle in str(e), str(e)
            continue
        raise AssertionError("the statistics check accepted a mutant (%s)" % needle)
