"""Every bf16 conv GEMM launch of the c3 and c5 training plans (B = 256, 224 px, mixup type 1, label
smoothing 0.1) at its own geometry against float64, element by element (oracle/conv_check.py):

  * conv: the output under the per-element bound and the exact-rounding check, the fused batch-norm
    statistics rows, the bias + fp32 logits layer, a repeated launch bit for bit, CTA pairs bit for bit
    where the tiling would pair CTAs; and every conv again at B = 7 (ragged last M tiles, as eval and
    serving batches have);
  * dgrad: with exactly the epilogue the plan fuses (none, add, mask, add + mask); the stride-2 convs'
    data gradient as the plan composes it (acnn_zero_insert2x, then a stride-1 dgrad) against the true
    gradient of the strided conv;
  * wgrad: accumulated into a nonzero dw, split-K (the default) and deterministic, per element and tile
    by tile, repeats bit for bit;
  * the space-to-depth stem end to end in bf16 and fp16 (acnn_pack_input, acnn_s2d_weight_pack, the
    overlapped-pixel conv, its wgrad and acnn_s2d_wgrad_unpack) against the raw 7x7 stride-2 conv;
  * acnn_prep_weights: the bf16 and 3-plane operand copies of every weight, bit for bit.

tests/test_conv_plan_fp16_gpu.py reruns the conv, dgrad and wgrad tests on fp16 storage with the fp16
plans' cases (the `fmt` fixture selects the format of their operands, launches and checks).

The library runs with its default knobs (halo kernel mode 1, the default wgrad split), as training does.
Inputs are generated on the device as 16-bit values; references are float64 on the device.  The conv
operands have one sign per output element (non-negative activations, weights of one sign per output
channel), so mag = |ref| and most elements are decided by the exact-rounding check; the wgrad operands
have random signs, so one missing pixel is visible in the tile norms.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import conv_check as CC

pytestmark = pytest.mark.gpu

ACNN_BF16, ACNN_F16 = 0, 3
NUM_SMS = 132


# storage format -> (acnn precision code, torch dtype)
FMT = {"bf16": (ACNN_BF16, torch.bfloat16), "fp16": (ACNN_F16, torch.float16)}


def _plans(dtype="bf16"):
    import bench
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    for name in ("c3", "c5"):
        cfg = ModelConfig(num_classes=1001, **bench.CONFIGS[name]["model"])
        yield build_plan(cfg, 256, 224, 224, training=True, mixup_type=1, label_smoothing=0.1, dtype=dtype)


CASES = CC.plan_cases(_plans())
CONV = [c for c in CASES if c.kind == "conv"]
DGRAD = [c for c in CASES if c.kind == "conv_dgrad"]
WGRAD = [c for c in CASES if c.kind == "conv_wgrad"]

REPORT = {f: {"decided": {}, "wgrad_tile": {}} for f in FMT}


@pytest.fixture
def fmt():
    return "bf16"


def report(fmt):
    """Print the minimum decided fraction per kind and the worst wgrad tiles of the tests run on fmt."""
    dec = REPORT[fmt]["decided"]
    if dec:
        k = min(dec, key=dec.get)
        print("\nminimum decided fraction: %.4f (%s)" % (dec[k], k[1]))
        for kind in ("conv", "conv_dgrad", "stem", "conv range", "dgrad range"):
            v = [f for (kd, _), f in dec.items() if kd == kind]
            if v:
                print("  %-10s %3d outputs, decided fraction min %.4f" % (kind, len(v), min(v)))
    for (n, P), e in sorted(REPORT[fmt]["wgrad_tile"].items(), key=lambda kv: (kv[0][1], kv[0][0])):
        print("worst wgrad tile norm-relative error P=%d %s: split-K %.3e (tolerance %.3e), deterministic %.3e "
              "(tolerance %.3e)" % (P, n, e[0][0], e[0][1], e[1][0], e[1][1]))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    report("bf16")


@pytest.fixture(autouse=True)
def _free():
    yield
    torch.cuda.empty_cache()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _check(rc, what):
    from assembled_cnn_b200 import _lib
    _lib.check(rc, what)


def _randn(shape, seed, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(shape, device="cuda", generator=_gen(seed)) * scale).to(dtype)


def _pos(shape, seed, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(shape, device="cuda", generator=_gen(seed)).abs() * scale).to(dtype)


def _signs(n, seed):
    return torch.randint(0, 2, (n,), device="cuda", generator=_gen(seed)).double() * 2 - 1


def _mask(shape, seed, dtype=torch.bfloat16):
    """A ReLU mask as the kernels see it: positives, +0 (the ReLU's zeros), -0 and negatives."""
    m = torch.randn(shape, device="cuda", generator=_gen(seed))
    r = torch.rand(shape, device="cuda", generator=_gen(seed + 1))
    m = torch.where(r < 0.3, torch.zeros((), device="cuda"), m)
    m = torch.where((r >= 0.3) & (r < 0.35), torch.full((), -0.0, device="cuda"), m)
    return m.to(dtype)


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _pad_x(x, geom, x_wpad):
    """float64 NCHW input with the geometry's zero padding (the stem's W padding is in its buffer)."""
    _, _, _, _, _, _, _, _, phl, phh, pwl, pwh = geom
    if x_wpad is not None:
        pwl = pwh = 0
    return F.pad(_nchw(x), (pwl, pwh, phl, phh))


def _with_batch(geom, B):
    return (B,) + tuple(geom[1:])


def _x_shape(geom, x_wpad):
    B, H, W, Cin = geom[:4]
    if x_wpad is not None:
        return (B, H, W + x_wpad[0] + x_wpad[1], Cin)
    return (B, H, W, Cin)


def _x_input(geom, x_wpad, seed, signed, dtype=torch.bfloat16):
    """x as the kernel reads it; the stem's space-to-depth buffer has zero W-padding columns (as
    acnn_pack_input writes them)."""
    shape = _x_shape(geom, x_wpad)
    x = _randn(shape, seed, dtype=dtype) if signed else _pos(shape, seed, dtype=dtype)
    if x_wpad is not None:
        x[:, :, :x_wpad[0]] = 0
        x[:, :, x.shape[2] - x_wpad[1]:] = 0
    return x


def _fprop_ref(x, w, geom, x_wpad):
    """float64 NHWC conv of a plan geometry and the same conv of |x|, |w| (ref, mag)."""
    xp = _pad_x(x, geom, x_wpad)
    w64 = w.double().permute(0, 3, 1, 2)
    ref = _nhwc(F.conv2d(xp, w64, stride=geom[7]))
    mag = _nhwc(F.conv2d(xp.abs(), w64.abs(), stride=geom[7]))
    return ref, mag


def _dgrad_ref(w, dy, fwd):
    """float64 NHWC data gradient of the forward conv geometry fwd, [B][H][W][Cin]."""
    B, H, W, Cin = fwd[:4]
    _, _, _, _, _, _, _, st, phl, phh, pwl, pwh = fwd
    full = torch.nn.grad.conv2d_input((B, Cin, H + phl + phh, W + pwl + pwh), w.double().permute(0, 3, 1, 2),
                                      _nchw(dy), stride=st)
    return _nhwc(full[:, :, phl:phl + H, pwl:pwl + W])


def _wgrad_chain(lib, cg, precision, det):
    """Pixels one split of acnn_conv_wgrad sums in one chain (its split layout, acnn_conv_wgrad_plan)."""
    import ctypes as C
    pix, splits, sps = C.c_int(), C.c_int(), C.c_int()
    _check(lib.acnn_conv_wgrad_plan(cg, precision, det, C.byref(pix), C.byref(splits), C.byref(sps)),
           "conv_wgrad_plan")
    return pix.value * sps.value


def _pairs_apply(cg, M, out_f32):
    """conv_tiling (csrc/gemm.cu) pairs CTAs here under acnn_set_conv_cta_pairs(1)."""
    K = cg.kh * cg.kw * cg.Cin
    return (cg.Cout % 128 == 0 and cg.Cin % 64 == 0 and K >= 512 and not out_f32
            and -(-M // 256) * (cg.Cout // 128) >= NUM_SMS // 2)


# ---------------------------------------------------------------------------------------------------
# conv (fprop)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [256, 7])
@pytest.mark.parametrize("case", CONV, ids=[c.id() for c in CONV])
def test_conv_plan_geometry(lib, case, B, fmt):
    code, tdt = FMT[fmt]
    geom = _with_batch(case.geom, B)
    cg = CC.launch_geom(geom, case.x_wpad)
    Ho, Wo = cg.out_hw()
    Cout, kh, kw, Cin = geom[4], geom[5], geom[6], geom[3]
    K = kh * kw * Cin
    M = B * Ho * Wo
    x = _x_input(geom, case.x_wpad, 1, signed=False, dtype=tdt)
    s = _signs(Cout, 2)
    w = (_pos((Cout, kh, kw, Cin), 3, 1.0 / math.sqrt(K)).double() * s[:, None, None, None]).to(tdt)
    bias = torch.randn(Cout, device="cuda", generator=_gen(4)) if case.bias else None
    out_dt = torch.float32 if case.out_f32 else tdt

    def launch(stats):
        y = _nan((B, Ho, Wo, Cout), out_dt)
        sp = CC.stats_poison((lib.acnn_conv_stats_parts(cg), 2, Cout)) if stats else None
        _check(lib.acnn_conv_fprop(cg, x.data_ptr(), w.data_ptr(), y.data_ptr(),
                                   sp.data_ptr() if stats else None, None, None,
                                   bias.data_ptr() if bias is not None else None, int(case.out_f32),
                                   code, 0, _st()), "conv_fprop")
        torch.cuda.synchronize()
        return y, sp

    y, sp = launch(case.stats)
    ref, mag = _fprop_ref(x, w, geom, case.x_wpad)
    acc = CC.acc_bound(mag, K)
    what = "%s B=%d %s" % (case.id(), B, fmt)
    if case.out_f32:
        ref = ref + bias.double()
        tol = acc + CC.U32 * (ref.abs() + acc)
        bad = ~((y.double() - ref).abs() <= tol)
        assert not bool(bad.any()), "%s: %d of %d logits outside acc + u |ref|" % (what, int(bad.sum()), bad.numel())
    else:
        REPORT[fmt]["decided"][("conv", what)] = CC.check_16bit(y, ref, acc, what, fmt)
    del ref, mag, acc
    if case.stats:
        CC.check_stats(sp, y, what + " statistics")
    y2, sp2 = launch(case.stats)
    assert torch.equal(y, y2), what + ": a second launch differs"
    if case.stats:
        assert torch.equal(sp, sp2), what + ": a second launch's statistics differ"
    if _pairs_apply(cg, M, case.out_f32):
        prev = lib.acnn_set_conv_cta_pairs(1)
        try:
            y3, sp3 = launch(case.stats)
        finally:
            lib.acnn_set_conv_cta_pairs(prev)
        assert torch.equal(y.view(torch.int16), y3.view(torch.int16)), what + ": CTA pairs differ from single CTAs"
        if case.stats:
            CC.check_stats(sp3, y3, what + " statistics (CTA pairs)")


# ---------------------------------------------------------------------------------------------------
# dgrad
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", DGRAD, ids=[c.id() for c in DGRAD])
def test_dgrad_plan_geometry(lib, case, fmt):
    code, tdt = FMT[fmt]
    from assembled_cnn_b200._lib import ConvGeom
    geom = case.geom
    g = ConvGeom(*geom)
    B, H, W, Cin, Cout, kh, kw = geom[:7]
    assert g.stride == 1
    fwd = case.src or geom                       # the forward conv whose data gradient this is
    gf = ConvGeom(*fwd)
    Hf, Wf = gf.out_hw()
    dy = _pos((B, Hf, Wf, Cout), 11, dtype=tdt)
    s = _signs(Cin, 12)
    K = kh * kw * Cout
    w = (_pos((Cout, kh, kw, Cin), 13, 1.0 / math.sqrt(K)).double() * s).to(tdt)
    wd = w.flip(1, 2).permute(3, 1, 2, 0).contiguous()
    if case.src:
        # the plan's composition: zero-insert dy to (B, H, W, Cout), then the stride-1 dgrad on g1
        assert gf.stride == 2 and geom[9] == kh - 1 - geom[8] and geom[11] == kw - 1 - geom[10]
        dyz = _nan((B, H, W, Cout), tdt)
        _check(lib.acnn_zero_insert2x(dy.data_ptr(), dyz.data_ptr(), B, Hf, Wf, H, W, Cout, code, _st()),
               "zero_insert2x")
    else:
        dyz = dy
    add = (_pos((B, H, W, Cin), 14, 0.5).double() * s).to(tdt) if case.add else None
    mask = _mask((B, H, W, Cin), 15, tdt) if case.mask else None
    dx = _nan((B, H, W, Cin), tdt)
    _check(lib.acnn_conv_dgrad(g, dyz.data_ptr(), wd.data_ptr(), dx.data_ptr(),
                               add.data_ptr() if add is not None else None,
                               mask.data_ptr() if mask is not None else None, code, 0, _st()), "conv_dgrad")
    torch.cuda.synchronize()
    del dyz, wd
    ref = _dgrad_ref(w, dy, fwd)
    mag = _dgrad_ref(w.abs(), dy.abs(), fwd)
    acc = CC.acc_bound(mag, K)
    if add is not None:
        acc = CC.add_epilogue_bound(acc, mag, add)
        ref = ref + add.double()
    del mag
    what = "%s %s" % (case.id(), fmt)
    if mask is not None:
        keep = (mask > 0).double()
        ref, acc = ref * keep, acc * keep
        CC.check_mask(dx, mask, what)
    REPORT[fmt]["decided"][("conv_dgrad", what)] = CC.check_16bit(dx, ref, acc, what, fmt)


# ---------------------------------------------------------------------------------------------------
# wgrad
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", WGRAD, ids=[c.id() for c in WGRAD])
def test_wgrad_plan_geometry(lib, case, fmt):
    code, tdt = FMT[fmt]
    geom = case.geom
    cg = CC.launch_geom(geom, case.x_wpad)
    B, _, _, Cin, Cout, kh, kw, stride = geom[:8]
    Ho, Wo = cg.out_hw()
    P = B * Ho * Wo
    x = _x_input(geom, case.x_wpad, 21, signed=True, dtype=tdt)
    dy = _randn((B, Ho, Wo, Cout), 22, dtype=tdt)
    dw0 = torch.randn((Cout, kh, kw, Cin), device="cuda", generator=_gen(23))
    xp = _pad_x(x, geom, case.x_wpad)
    wshape = (Cout, Cin, kh, kw)
    ref = _nhwc(torch.nn.grad.conv2d_weight(xp, wshape, _nchw(dy), stride=stride)) + dw0.double()
    mag = _nhwc(torch.nn.grad.conv2d_weight(xp.abs(), wshape, _nchw(dy).abs(), stride=stride))
    del xp
    worst = []
    for det in (0, 1):
        dws = []
        for _ in range(2):
            dw = dw0.clone()
            _check(lib.acnn_conv_wgrad(cg, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), code, det, _st()),
                   "conv_wgrad")
            dws.append(dw)
        torch.cuda.synchronize()
        what = "%s det=%d %s" % (case.id(), det, fmt)
        assert torch.equal(dws[0], dws[1]), what + ": a repeated launch differs"
        chain = _wgrad_chain(lib, cg, code, det)
        worst.append((CC.check_wgrad(dws[0], ref, mag, dw0, P, what, chain), CC.wgrad_tile_tol(min(P, chain))))
    REPORT[fmt]["wgrad_tile"][(case.id(), P)] = worst


# ---------------------------------------------------------------------------------------------------
# the space-to-depth stem, end to end
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["bf16", "fp16"])
def test_stem_space_to_depth_end_to_end(lib, fmt):
    """acnn_pack_input (mode 0) of a B = 256 fp32 224 x 224 x 3 batch, acnn_s2d_weight_pack of the fp32
    7 x 7 x 3 x 64 master, the stem conv as the plan launches it (k2 x 1 taps over overlapping k2*16-channel
    pixels) with its statistics, its wgrad into the packed layout and acnn_s2d_wgrad_unpack -- against the
    raw 7 x 7 stride-2 fixed_padding conv of the 16-bit-rounded images and weights and its weight gradient."""
    from assembled_cnn_b200.plan import PlanBuilder
    code, tdt = FMT[fmt]
    B, HW, k, Cout = 256, 224, 7, 64
    pad, k2, lo, hi = PlanBuilder.stem_s2d_taps(k)
    H2 = HW // 2
    geom = (B, H2, H2, 16, Cout, k2, k2, 1, lo, hi, lo, hi)
    cg = CC.launch_geom(geom, (lo, hi))
    # images: fp32 values that need rounding to 16 bits, non-negative (one sign per output element)
    images = torch.rand((B, HW, HW, 3), device="cuda", generator=_gen(31)) * 2.0
    xs = _nan((B, H2, H2 + lo + hi, 16), tdt)
    _check(lib.acnn_pack_input(images.data_ptr(), None, None, 0, xs.data_ptr(), B, HW, HW, lo, hi, code, _st()),
           "pack_input")
    s = _signs(Cout, 32)
    w = torch.randn((Cout, k, k, 3), device="cuda", generator=_gen(33)).abs() * s[:, None, None, None].float() / 12
    w2 = _nan((Cout, k2, k2, 16), tdt)
    _check(lib.acnn_s2d_weight_pack(w.data_ptr(), w2.data_ptr(), Cout, k, pad, k2, lo, code, _st()), "s2d_weight_pack")
    y = _nan((B, H2, H2, Cout), tdt)
    sp = CC.stats_poison((lib.acnn_conv_stats_parts(cg), 2, Cout))
    _check(lib.acnn_conv_fprop(cg, xs.data_ptr(), w2.data_ptr(), y.data_ptr(), sp.data_ptr(), None, None, None, 0,
                               code, 0, _st()), "stem conv_fprop")
    torch.cuda.synchronize()
    xr = F.pad(_nchw(images.to(tdt)), (pad, pad, pad, pad))
    wr = w.to(tdt).double().permute(0, 3, 1, 2)
    ref = _nhwc(F.conv2d(xr, wr, stride=2))
    mag = _nhwc(F.conv2d(xr.abs(), wr.abs(), stride=2))
    acc = CC.acc_bound(mag, k2 * k2 * 16)      # the launched K (its zero taps add exactly)
    del mag
    what = "stem %s" % fmt
    REPORT["bf16"]["decided"][("stem", what)] = CC.check_16bit(y, ref, acc, what, fmt)
    del ref, acc
    CC.check_stats(sp, y, what + " statistics")
    # weight gradient: into the packed layout (the plan's zeroed slot), then unpacked into dw
    dy = _randn((B, H2, H2, Cout), 34, dtype=tdt)
    dw2 = torch.zeros((Cout, k2, k2, 16), device="cuda")
    _check(lib.acnn_conv_wgrad(cg, xs.data_ptr(), dy.data_ptr(), dw2.data_ptr(), code, 0, _st()), "stem conv_wgrad")
    dw = _nan((Cout, k, k, 3), torch.float32)
    _check(lib.acnn_s2d_wgrad_unpack(dw2.data_ptr(), dw.data_ptr(), Cout, k, pad, k2, lo, _st()), "s2d_wgrad_unpack")
    torch.cuda.synchronize()
    wshape = (Cout, 3, k, k)
    ref_w = _nhwc(torch.nn.grad.conv2d_weight(xr, wshape, _nchw(dy), stride=2))
    mag_w = _nhwc(torch.nn.grad.conv2d_weight(xr.abs(), wshape, _nchw(dy).abs(), stride=2))
    P = B * H2 * H2
    chain = _wgrad_chain(lib, cg, code, 0)
    e = CC.check_wgrad(dw, ref_w, mag_w, torch.zeros_like(dw), P, what + " wgrad", chain)
    REPORT["bf16"]["wgrad_tile"][(what, P)] = ((e, CC.wgrad_tile_tol(min(P, chain))), (float("nan"), float("nan")))


# ---------------------------------------------------------------------------------------------------
# acnn_prep_weights
# ---------------------------------------------------------------------------------------------------
def test_prep_weights_bit_exact(lib):
    """acnn_prep_weights: every conv and dense weight of the c3 plan, plus one whose Cout and Cin are not
    multiples of 32 (the kernel's 32 x 32 tile guards): planes = 1 writes master.bfloat16() (round to
    nearest even) in the fprop layout [Cout][taps][Cin] and the dgrad layout [Cin][taps flipped][Cout];
    planes = 3 writes acnn_split3's three planes of the master, bit for bit, in both layouts at the
    plane strides passed in."""
    import bench
    from assembled_cnn_b200 import _lib
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    cfg = ModelConfig(num_classes=1001, **bench.CONFIGS["c3"]["model"])
    plan = build_plan(cfg, 2, 64, 64, training=True)
    ws = [(p.name, p.offset, p.dgrad_off, p.store_shape) for p in plan.params.values()
          if p.kind in ("conv_kernel", "dense_kernel") and len(p.store_shape) == 4
          and p.store_shape[3] % 16 == 0 and p.store_shape[0] % 32 == 0]
    # a ragged weight after the plan's: Cout 40, 3x3 taps, Cin 24 (dgrad copy after the plan's too)
    odd = (40, 3, 3, 24)
    n_odd = math.prod(odd)
    ws.append(("ragged", plan.param_elems, plan.dgrad_elems, odd))
    n_master = plan.param_elems + n_odd + (-(plan.param_elems + n_odd) % 8)
    fs, ds = n_master, plan.dgrad_elems + n_odd
    descs = [_lib.WeightDesc(off, off, doff, sh[0], sh[1] * sh[2], sh[3], 0) for _, off, doff, sh in ws]
    table = torch.frombuffer(bytearray(bytes((_lib.WeightDesc * len(descs))(*descs))), dtype=torch.uint8).cuda()
    master = torch.zeros(n_master, device="cuda").normal_(0.0, 0.3, generator=_gen(41))
    # values whose rounding is a tie (the even neighbour wins) and values just beyond it
    t = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 1.0 + 2.0 ** -8 + 2.0 ** -20],
                     device="cuda")
    master[ws[0][1]:ws[0][1] + 4] = t
    master[plan.param_elems:plan.param_elems + 4] = t
    split = _nan((3, n_master), torch.bfloat16)
    _check(lib.acnn_split3(master.data_ptr(), split.data_ptr(), n_master, _st()), "split3")
    for planes in (1, 3):
        wf = _nan((planes, fs), torch.bfloat16)
        wd = _nan((planes, ds), torch.bfloat16)
        _check(lib.acnn_prep_weights(master.data_ptr(), table.data_ptr(), len(descs), wf.data_ptr(), wd.data_ptr(),
                                     planes, fs, ds, _st()), "prep_weights")
        torch.cuda.synchronize()
        for name, off, doff, (co, kh, kw, ci) in ws:
            n = co * kh * kw * ci
            m = master[off:off + n]
            for p in range(planes):
                want = m.bfloat16() if planes == 1 else split[p, off:off + n]
                got = wf[p, off:off + n]
                assert torch.equal(got.view(torch.int16), want.view(torch.int16)), "%s planes=%d p=%d fprop" % (
                    name, planes, p)
                if doff >= 0:
                    want_d = want.view(co, kh, kw, ci).flip(1, 2).permute(3, 1, 2, 0).reshape(-1)
                    got_d = wd[p, doff:doff + n]
                    assert torch.equal(got_d.view(torch.int16), want_d.view(torch.int16)), \
                        "%s planes=%d p=%d dgrad" % (name, planes, p)
    assert len(ws) > 50
    # the ties went to the even neighbour: 1 + 2^-8 -> 1, 1 + 3 * 2^-8 -> 1 + 2^-6, and just above a tie up
    got = wf[0, ws[0][1]:ws[0][1] + 4].float().cpu().tolist()
    assert got == [1.0, 1.0 + 2.0 ** -6, -1.0, 1.0 + 2.0 ** -7]
