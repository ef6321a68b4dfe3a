"""The ordered split-K reductions: the conv weight gradient (wgrad_gemm_kernel, csrc/gemm.cu) and the
small fp32 GEMM of the SK / SE attention layers (sgemm + sgemm_reduce_kernel, csrc/small_fc.cu).

Each split stores a partial tile and the partials are added in split order, so the result is a fixed
function of the split layout.  For a known layout it is known exactly: the partial of split z is the
same computation as a one-split (deterministic) launch on the pixel (or batch) sub-range of that split,
so the split-K result must equal  acc0 + (((0 + p_0) + p_1) + ... + p_{s-1})  summed in float32 in
split order, bit for bit.  A reduction that depends on arrival order, drops or doubles a stage, or
keeps state across launches, graph replays or streams fails these comparisons even where its error
is far below any tolerance.  Every repeat here runs a fixed two or three times."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

F32_TOL = 1e-4          # fp64 autograd check of a whole wgrad (as tests/test_conv_gemm_gpu.py)
U = 2.0 ** -24          # fp32 unit roundoff


def _geom(B, H, W, Cin, Cout, k=1, stride=1, pads=(0, 0, 0, 0)):
    from assembled_cnn_b200._lib import ConvGeom
    return ConvGeom(B, H, W, Cin, Cout, k, k, stride, *pads)


def _rows(P, Cin, Cout):
    """A plain wgrad (1x1, stride 1, no padding) over P pixel rows."""
    return _geom(1, 1, P, Cin, Cout)


def _plan(lib, g, precision=0, det=0):
    from assembled_cnn_b200 import _lib
    pix, splits, sps = C.c_int(), C.c_int(), C.c_int()
    _lib.check(lib.acnn_conv_wgrad_plan(g, precision, det, C.byref(pix), C.byref(splits),
                                        C.byref(sps)), "acnn_conv_wgrad_plan")
    return pix.value, splits.value, sps.value


@contextlib.contextmanager
def _wgrad_knobs(lib, splits=0, pix=0):
    prev_s = lib.acnn_set_wgrad_splits(splits)
    prev_p = lib.acnn_set_wgrad_pixels(pix)
    try:
        yield
    finally:
        lib.acnn_set_wgrad_splits(prev_s)
        lib.acnn_set_wgrad_pixels(prev_p)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _wgrad(lib, g, x, dy, dw, precision=0, det=0, stream=None):
    from assembled_cnn_b200 import _lib
    _lib.check(lib.acnn_conv_wgrad(g, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), precision, det,
                                   _stream() if stream is None else stream), "acnn_conv_wgrad")


def _planes(lib, t):
    """fp32 CUDA tensor -> bf16 [3, ...] hi / mid / lo planes (acnn_split3)."""
    from assembled_cnn_b200 import _lib
    out = torch.empty((3,) + tuple(t.shape), dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.acnn_split3(t.contiguous().data_ptr(), out.data_ptr(), t.numel(), _stream()),
               "split3")
    return out


def _dw_ref64(g, x, dy):
    """fp64 weight gradient [Cout, kh, kw, Cin] of the correlation of geometry g (CPU autograd)."""
    xd = x.double().cpu().permute(0, 3, 1, 2)
    xd = F.pad(xd, (g.pad_w_lo, g.pad_w_hi, g.pad_h_lo, g.pad_h_hi))
    w = torch.zeros(g.Cout, g.Cin, g.kh, g.kw, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(xd, w, stride=g.stride)
    (dw,) = torch.autograd.grad(y, w, dy.double().cpu().permute(0, 3, 1, 2))
    return dw.permute(0, 2, 3, 1)


def _relerr(a, b):
    return (a.double() - b.double()).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _ordered_sum(acc0, parts):
    """acc0 + (((0 + p_0) + p_1) + ...) in float32, in split order: what the ordered reduction
    computes from the partials."""
    t = np.zeros_like(parts[0])
    for p in parts:
        t = (t + p).astype(np.float32)
    return (acc0 + t).astype(np.float32)


# ---------------------------------------------------------------------------------------------
# a. wgrad split-K == its split decomposition, bit for bit
# ---------------------------------------------------------------------------------------------
# name: (geometry, precision, acnn_set_wgrad_splits, acnn_set_wgrad_pixels, splits, stages_per_split)
# The expected (splits, stages_per_split) are the layouts these cases are built to produce; the plan
# query must confirm them.
DECOMP = {
    # plain: N tile 128, 64-channel chunks, 10 stages in 4 splits = 3 + 3 + 3 + 1
    "plain_n128_cw64_short_last": (_rows(640, 64, 128), 0, 4, 64, 4, 3),
    # plain: N tile 256, 32-channel chunks, ragged last stage (593 = 9 * 64 + 17), 2 splits
    "plain_n256_cw32_ragged": (_rows(593, 32, 256), 0, 2, 64, 2, 5),
    # plain: N tile 32, 16-channel chunks, 7 stages in 3 splits = 3 + 3 + 1
    "plain_n32_cw16_3splits": (_rows(448, 16, 32), 0, 3, 64, 3, 3),
    # plain: N tile 64, ragged (773 = 12 * 64 + 5), the maximum: one stage per split
    "plain_n64_max_splits": (_rows(773, 64, 64), 0, 1000, 64, 13, 1),
    # 128-pixel stages (default pixel choice) with every split >= 4096 pixels, ragged last stage:
    # 12622 pixels = 99 stages in 3 splits of 33 (4224 + 4224 + 4174 pixels)
    "plain_pix128_3splits": (_rows(12622, 64, 128), 0, 3, 0, 3, 33),
    # im2col 3x3 stride 1 at 8x8 (one 64-pixel stage per image), 10 images in 3 + 3 + 3 + 1
    "im2col_3x3_s1_8x8": (_geom(10, 8, 8, 32, 64, 3, 1, (1, 1, 1, 1)), 0, 4, 64, 4, 3),
    # im2col 3x3 stride 2 from 16x16 (fixed padding) to 8x8, N tile 128, 2 splits
    "im2col_3x3_s2_16x16": (_geom(6, 16, 16, 64, 128, 3, 2, (1, 1, 1, 1)), 0, 2, 64, 2, 3),
    # 1x1 stride 2 projection from 16x16 (8x8 outputs), N tile 256: 7 stages in 3 + 3 + 1
    "im2col_1x1_s2_n256": (_geom(7, 16, 16, 128, 256, 1, 2), 0, 3, 64, 3, 3),
    # 3x3 at 8x8, Cin = Cout = 512: 72 tiles of 128 x 256 floats, so the 64 MiB partial scratch
    # holds 7 splits; 100 requested -> 7 -> 10 stages re-normalised to 5 splits of 2
    "im2col_scratch_capped": (_geom(10, 8, 8, 512, 512, 3, 1, (1, 1, 1, 1)), 0, 100, 64, 5, 2),
    # three-plane fp32 mode (64-pixel stages, N tile <= 128), deterministic = 0
    "fp32_plain_ragged": (_rows(393, 64, 128), 1, 2, 0, 2, 4),
    "fp32_im2col_3x3_max": (_geom(5, 8, 8, 16, 32, 3, 1, (1, 1, 1, 1)), 1, 1000, 0, 5, 1),
}


def _sub_problem(g, x, dy, p0, p1):
    """The wgrad restricted to output pixels [p0, p1): (geometry, x, dy)."""
    plain = g.kh == 1 and g.kw == 1 and g.stride == 1 and g.H == 1 and g.B == 1
    if plain:
        return _rows(p1 - p0, g.Cin, g.Cout), x[..., p0:p1, :], dy[..., p0:p1, :]
    Ho, Wo = g.out_hw()
    assert p0 % (Ho * Wo) == 0 and p1 % (Ho * Wo) == 0, "split boundary inside an image"
    b0, b1 = p0 // (Ho * Wo), p1 // (Ho * Wo)
    sub = _geom(b1 - b0, g.H, g.W, g.Cin, g.Cout, g.kh, g.stride,
                (g.pad_h_lo, g.pad_h_hi, g.pad_w_lo, g.pad_w_hi))
    if x.dim() == 5:          # planes [3, B, H, W, C]
        return sub, x[:, b0:b1], dy[:, b0:b1]
    return sub, x[b0:b1], dy[b0:b1]


@pytest.mark.parametrize("case", sorted(DECOMP))
def test_wgrad_split_k_equals_its_decomposition(lib, case):
    g, precision, force, pix_knob, want_splits, want_sps = DECOMP[case]
    Ho, Wo = g.out_hw()
    P = g.B * Ho * Wo
    gen = torch.Generator().manual_seed(sorted(DECOMP).index(case))
    x32 = torch.randn(g.B, g.H, g.W, g.Cin, generator=gen)
    dy32 = torch.randn(g.B, Ho, Wo, g.Cout, generator=gen)
    if precision == 0:
        x32, dy32 = x32.bfloat16().float(), dy32.bfloat16().float()
        xd, dyd = x32.bfloat16().cuda(), dy32.bfloat16().cuda()
    else:
        xd, dyd = _planes(lib, x32.cuda()), _planes(lib, dy32.cuda())
    # dw accumulates: a random, non-zero running sum
    dw0 = torch.randn(g.Cout, g.kh, g.kw, g.Cin, generator=gen)
    with _wgrad_knobs(lib, force, pix_knob):
        pix, splits, sps = _plan(lib, g, precision, 0)
        assert (splits, sps) == (want_splits, want_sps), (pix, splits, sps)
        assert pix == (128 if pix_knob == 0 and precision == 0 and g.Cout < 256 else 64)
        stages = -(-P // pix)
        assert splits == -(-stages // sps) and (splits - 1) * sps < stages
        assert _plan(lib, g, precision, 1)[1:] == (1, stages)
        dw = dw0.cuda()
        _wgrad(lib, g, xd, dyd, dw, precision, 0)
        parts = []
        for z in range(splits):
            p0, p1 = z * sps * pix, min((z + 1) * sps * pix, P)
            sg, sx, sdy = _sub_problem(g, xd, dyd, p0, p1)
            # the sub-run must use the same stages: same pixels per stage, one split
            assert _plan(lib, sg, precision, 1) == (pix, 1, -(-(p1 - p0) // pix))
            part = torch.zeros_like(dw)
            _wgrad(lib, sg, sx.contiguous(), sdy.contiguous(), part, precision, 1)
            parts.append(part)
        torch.cuda.synchronize()
    got = dw.cpu().numpy()
    want = _ordered_sum(dw0.numpy(), [p.cpu().numpy() for p in parts])
    if not np.array_equal(got, want):
        d = np.abs(got.astype(np.float64) - want)
        raise AssertionError("%s: split-K dw differs from its decomposition in %d of %d elements "
                             "(max |d| %.3e)" % (case, int((d > 0).sum()), d.size, d.max()))
    # and the decomposition itself is the weight gradient (fp64 autograd)
    ref = _dw_ref64(g, x32, dy32)
    assert _relerr(dw.cpu() - dw0, ref) < F32_TOL


# ---------------------------------------------------------------------------------------------
# b. wgrad at the production shapes (Assemble-ResNet-50, B = 256, 224 px), default heuristic
# ---------------------------------------------------------------------------------------------
# Of the C3 plan's 43 distinct conv_wgrad geometries, 42 run split-K under the default cost model on an
# H100 80GB HBM3 (132 SMs; measured, the same answer as the host-only query): all but the final dense
# layer (2048 -> 1024 at 1x1, 4 stages)
PRODUCTION_SPLIT_MIN = 42


def _production_wgrad_geoms():
    """Distinct conv_wgrad geometries of the C3 plan as the library launches them (model_exec.cu's launch
    geometry: acnn_op_conv_info reports the plan's, without the W-padded stem form)."""
    from assembled_cnn_b200._lib import ConvGeom
    from assembled_cnn_b200.plan import ModelConfig, build_plan
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
        else:                     # the W-padded space-to-depth stem input
            lo, hi = wpad
            row = (g.W + lo + hi) * g.Cin
            cg = ConvGeom(g.B, g.H, g.W, g.Cin * g.kw, g.Cout, g.kh, 1, 1, g.pad_h_lo, g.pad_h_hi,
                          0, 0, g.Cin, row, g.H * row, 0)
        key = tuple(getattr(cg, n) for n, _ in ConvGeom._fields_)
        out.setdefault(key, (cg, wpad))
    return list(out.values())


def _x_elems(cg):
    if cg.x_img_pitch > 0:
        return cg.B * cg.x_img_pitch
    return cg.B * cg.H * cg.W * cg.Cin


def test_wgrad_production_shapes_reproducible(lib):
    geoms = _production_wgrad_geoms()
    gen = torch.Generator(device="cuda").manual_seed(3)
    n_split, rows, cost = 0, [], []
    for cg, wpad in geoms:
        pix, splits, sps = _plan(lib, cg)
        n_split += splits > 1
        Ho, Wo = cg.out_hw()
        P = cg.B * Ho * Wo
        rows.append("B%d %dx%d %d->%d k%dx%d s%d: P %d pix %d splits %d x %d stages" % (
            cg.B, cg.H, cg.W, cg.Cin, cg.Cout, cg.kh, cg.kw, cg.stride, P, pix, splits, sps))
        x = torch.randn(_x_elems(cg), device="cuda", generator=gen).bfloat16()
        dy = torch.randn(P * cg.Cout, device="cuda", generator=gen).bfloat16()
        dws = []
        for _ in range(2):
            dw = torch.zeros(cg.Cout * cg.kh * cg.kw * cg.Cin, device="cuda")
            _wgrad(lib, cg, x, dy, dw)
            dws.append(dw)
        torch.cuda.synchronize()
        assert torch.equal(dws[0], dws[1]), rows[-1]
        if wpad is None:
            cost.append((P * cg.kh * cg.kw * cg.Cin * cg.Cout, len(cost), cg, x, dy, dws[0]))
        else:
            del x, dy, dws
    print("\n".join(rows))
    print("production wgrad geometries: %d distinct, %d split" % (len(geoms), n_split))
    assert n_split >= PRODUCTION_SPLIT_MIN
    # the cheapest few (that split or not) against fp64 on the device
    for _, _, cg, x, dy, dw in sorted(cost, key=lambda c: c[:2])[:3]:
        Ho, Wo = cg.out_hw()
        xd = x.view(cg.B, cg.H, cg.W, cg.Cin).double().permute(0, 3, 1, 2)
        xd = F.pad(xd, (cg.pad_w_lo, cg.pad_w_hi, cg.pad_h_lo, cg.pad_h_hi))
        w = torch.zeros(cg.Cout, cg.Cin, cg.kh, cg.kw, dtype=torch.float64, device="cuda",
                        requires_grad=True)
        (ref,) = torch.autograd.grad(F.conv2d(xd, w, stride=cg.stride), w,
                                     dy.view(cg.B, Ho, Wo, cg.Cout).double().permute(0, 3, 1, 2))
        assert _relerr(dw.view(cg.Cout, cg.kh, cg.kw, cg.Cin), ref.permute(0, 2, 3, 1)) < F32_TOL


# ---------------------------------------------------------------------------------------------
# c. the small fp32 GEMM's split-K through the SE / SK ops
# ---------------------------------------------------------------------------------------------
# Bound: every output element of C (+)= A*B is a float32 sum of K products, each split an fma chain and
# the partials added in a chain, then one add into C.  Whatever the order, the rounding error of such a
# sum is at most gamma_n * sum_k |a_k b_k| with gamma_n = n u / (1 - n u), n = number of roundings in
# the chain (<= K + splits + 1), plus u |result| for the final add (Higham, Accuracy and Stability of
# Numerical Algorithms, 3.1).  The check uses n = K + 64 (covers any split count here) element by
# element: tight enough that a dropped or doubled split -- an error of the size of a partial sum, not
# of its rounding -- fails it, and rigorous, so it cannot fail on a correct kernel.  Each GEMM stage is
# checked from the inputs that stage actually received (the previous stage's device output).
def _gamma(n):
    return n * U / (1 - n * U)


def _chk(got, ref, bound, what):
    got = got.double().cpu()
    d = (got - ref).abs()
    bad = d > bound
    if bad.any():
        i = int(torch.argmax((d / bound.clamp_min(1e-300)).flatten()))
        raise AssertionError("%s: %d of %d elements outside the fp32 bound (worst: |d| %.3e, bound "
                             "%.3e)" % (what, int(bad.sum()), d.numel(), d.flatten()[i],
                                        bound.flatten()[i]))


def _gemm_bound(A, B_, K, acc=None):
    """Rounding bound of A @ B_ (+ acc) in float32 (fp64 operands)."""
    b = _gamma(K + 64) * (A.abs() @ B_.abs())
    ref = A @ B_ + (acc if acc is not None else 0)
    return ref, b + U * ref.abs()


def _launches(lib, fn):
    n0 = lib.acnn_launch_count()
    fn()
    return lib.acnn_launch_count() - n0


SE_SHAPES = [(B, C) for B in (33, 64, 200, 256) for C in (256, 512, 1024, 2048)]


def _se_inputs(B, Cc, seed):
    r = Cc // 16
    g = torch.Generator().manual_seed(seed)
    t = dict(q=torch.randn(B, Cc, generator=g), w1=torch.randn(r, Cc, generator=g) / Cc ** 0.5,
             w2=torch.randn(Cc, r, generator=g) / r ** 0.5, de=torch.randn(B, Cc, generator=g),
             e=torch.rand(B, Cc, generator=g),
             h=torch.relu(torch.randn(B, r, generator=g)),           # relu output: exact zeros
             dw1=torch.randn(r, Cc, generator=g), dw2=torch.randn(Cc, r, generator=g))
    return r, {k: v.cuda() for k, v in t.items()}


def _se_bwd(lib, t, B, Cc, r, det, HW=49, stream=None, B_rows=None):
    """acnn_se_fc_bwd on fresh copies of the accumulators; returns (dw1, dw2, dq, scratch)."""
    from assembled_cnn_b200 import _lib
    out = dict(dw1=t["dw1"].clone(), dw2=t["dw2"].clone(), dq=torch.empty(B, Cc, device="cuda"),
               scratch=torch.empty(B * (Cc + r), device="cuda"))
    _lib.check(lib.acnn_se_fc_bwd(t["de"].data_ptr(), t["e"].data_ptr(), t["h"].data_ptr(),
                                  t["q"].data_ptr(), t["w1"].data_ptr(), t["w2"].data_ptr(),
                                  out["dw1"].data_ptr(), out["dw2"].data_ptr(), out["dq"].data_ptr(),
                                  out["scratch"].data_ptr(), B, Cc, r, HW, det,
                                  _stream() if stream is None else stream), "se_fc_bwd")
    return out


@pytest.mark.parametrize("B,Cc", SE_SHAPES, ids=["B%d_C%d" % s for s in SE_SHAPES])
def test_se_fc_split_k_against_fp64(lib, B, Cc):
    from assembled_cnn_b200 import _lib
    r, t = _se_inputs(B, Cc, seed=B * 7 + Cc)
    st = _stream()

    def fwd(det):
        h = torch.empty(B, r, device="cuda")
        e = torch.empty(B, Cc, device="cuda")
        _lib.check(lib.acnn_se_fc_fwd(t["q"].data_ptr(), t["w1"].data_ptr(), t["w2"].data_ptr(),
                                      h.data_ptr(), e.data_ptr(), B, Cc, r, det, st), "se_fc_fwd")
        return h, e

    res = {}
    launches = {}
    for det in (0, 0, 1):
        out = {}
        launches[det] = _launches(lib, lambda: out.update(zip(("h", "e"), fwd(det))))
        launches[det] += _launches(lib, lambda: out.update(_se_bwd(lib, t, B, Cc, r, det)))
        torch.cuda.synchronize()
        if det in res:         # the second det = 0 run: bit-identical
            for k in ("h", "e", "dw1", "dw2", "dq"):
                assert torch.equal(res[det][k], out[k]), k
        res[det] = out
    # the split path really ran: one reduction launch more per split GEMM
    assert launches[0] > launches[1], launches
    d = {k: v.double().cpu() for k, v in t.items()}
    HW = 49
    for det in (0, 1):
        o = res[det]
        # forward: h = relu(q W1^T), e = sigmoid(h W2^T) (sigmoid: 1/4-Lipschitz, + its own rounding)
        ref, b = _gemm_bound(d["q"], d["w1"].t(), Cc)
        _chk(o["h"], torch.relu(ref), b, "se h det=%d" % det)
        h = o["h"].double().cpu()
        ref, b = _gemm_bound(h, d["w2"].t(), r)
        e_ref = torch.sigmoid(ref)
        _chk(o["e"], e_ref, 0.25 * b + 8 * U * e_ref, "se e det=%d" % det)
        # backward from the given (de, e, h): da2 = de e (1 - e) (scratch), dW2 += da2^T h,
        # dh = (da2 W2) [h > 0] (scratch), dW1 += dh^T q, dq = dh W1 / HW
        sc = o["scratch"].double().cpu()
        da2 = sc[:B * Cc].view(B, Cc)
        da2_ref = d["de"] * d["e"] * (1 - d["e"])
        _chk(da2, da2_ref, 4 * U * da2_ref.abs(), "se da2 det=%d" % det)
        ref, b = _gemm_bound(da2.t(), d["h"], B, d["dw2"])
        _chk(o["dw2"], ref, b, "se dw2 det=%d" % det)
        dh = sc[B * Cc:B * (Cc + r)].view(B, r)
        ref, b = _gemm_bound(da2, d["w2"], Cc)
        _chk(dh, ref * (d["h"] > 0), b, "se dh det=%d" % det)
        ref, b = _gemm_bound(dh.t(), d["q"], B, d["dw1"])
        _chk(o["dw1"], ref, b, "se dw1 det=%d" % det)
        ref, b = _gemm_bound(dh, d["w1"], r)
        _chk(o["dq"], ref / HW, b / HW + 3 * U * (ref / HW).abs(), "se dq det=%d" % det)
    # det = 0 and det = 1 agree to fp32 rounding (relative to the tensor's largest element: the
    # accumulated outputs cancel, so element-relative differences are not meaningful)
    for k in ("h", "e", "dw1", "dw2", "dq"):
        assert _relerr(res[0][k], res[1][k]) < 1e-5, k


def _sgemm_layout(M, N, K):
    """Split layout of sgemm() in csrc/small_fc.cu: (splits, k per split).  Restated here because
    the exact expectation below needs it; if the library's choice changes, the sub-runs no longer
    line up with the splits and the bit-exact comparison reports it."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-M // 64) * -(-N // 64)
    splits = min(-(-2 * sms // tiles), -(-K // 32))
    kps = -(-(-(-K // max(splits, 1))) // 16) * 16
    return -(-K // kps), kps


@pytest.mark.parametrize("B,Cc", [(33, 256), (200, 512), (256, 1024), (256, 2048)])
def test_se_dw2_split_k_equals_its_decomposition(lib, B, Cc):
    """dW2 += da2^T h has K = batch: the partial of each split is a deterministic se_fc_bwd on that
    split's sub-batch (da2 is elementwise, so its rows do not depend on the batch)."""
    r, t = _se_inputs(B, Cc, seed=B + Cc)
    splits, kps = _sgemm_layout(Cc, r, B)
    assert splits > 1
    full = _se_bwd(lib, t, B, Cc, r, 0)
    parts = []
    for z in range(splits):
        b0, b1 = z * kps, min((z + 1) * kps, B)
        sub = {k: (v[b0:b1].contiguous() if k in ("q", "de", "e", "h") else v) for k, v in t.items()}
        sub["dw1"], sub["dw2"] = torch.zeros_like(t["dw1"]), torch.zeros_like(t["dw2"])
        parts.append(_se_bwd(lib, sub, b1 - b0, Cc, r, 1)["dw2"])
    torch.cuda.synchronize()
    want = _ordered_sum(t["dw2"].cpu().numpy(), [p.cpu().numpy() for p in parts])
    assert np.array_equal(full["dw2"].cpu().numpy(), want)


SK_SHAPES = [(B, f) for B in (33, 64, 200, 256) for f in (64, 128, 256, 512)]


@pytest.fixture
def sk_multi_launch(lib):
    prev = lib.acnn_set_sk_fc_fused(0)
    yield
    lib.acnn_set_sk_fc_fused(prev)


@pytest.mark.parametrize("B,f", SK_SHAPES, ids=["B%d_f%d" % s for s in SK_SHAPES])
def test_sk_fc_multi_launch_split_k_against_fp64(lib, sk_multi_launch, B, f):
    from assembled_cnn_b200 import _lib
    d_ = max(f // 2, 32)
    g = torch.Generator().manual_seed(B * 13 + f)
    t = dict(s=torch.randn(B, f, generator=g), w1=torch.randn(d_, f, generator=g) / f ** 0.5,
             w2=torch.randn(2 * f, d_, generator=g) / d_ ** 0.5,
             gamma=0.5 + torch.rand(d_, generator=g), beta=0.1 * torch.randn(d_, generator=g),
             dA=torch.randn(B, f, generator=g), dw1=torch.randn(d_, f, generator=g),
             dw2=torch.randn(2 * f, d_, generator=g), dgamma=torch.randn(d_, generator=g),
             dbeta=torch.randn(d_, generator=g))
    t = {k: v.cuda() for k, v in t.items()}
    nscratch = lib.acnn_sk_fc_scratch_floats(B, f, d_)
    st = _stream()

    def run(det):
        o = dict(mm=torch.zeros(d_, device="cuda"), mv=torch.ones(d_, device="cuda"),
                 zpre=torch.empty(B, d_, device="cuda"), bnstat=torch.empty(2 * d_, device="cuda"),
                 z=torch.empty(B, d_, device="cuda"), att=torch.empty(B, f, device="cuda"),
                 scratch=torch.empty(nscratch, device="cuda"), ds=torch.empty(B, f, device="cuda"),
                 dw1=t["dw1"].clone(), dw2=t["dw2"].clone(), dgamma=t["dgamma"].clone(),
                 dbeta=t["dbeta"].clone())
        P = lambda k: o[k].data_ptr()
        T = lambda k: t[k].data_ptr()
        _lib.check(lib.acnn_sk_fc_fwd(T("s"), T("w1"), T("gamma"), T("beta"), P("mm"), P("mv"), 0.997,
                                      1e-5, 1, T("w2"), P("zpre"), P("bnstat"), P("z"), P("att"),
                                      P("scratch"), B, f, d_, det, st), "sk_fc_fwd")
        o["fwd_scratch"] = o["scratch"][:B * 2 * f].clone()          # a = z W2^T
        _lib.check(lib.acnn_sk_fc_bwd(T("dA"), P("att"), P("z"), P("zpre"), P("bnstat"), T("gamma"),
                                      T("s"), T("w1"), T("w2"), P("dw1"), P("dw2"), P("dgamma"),
                                      P("dbeta"), P("ds"), P("scratch"), B, f, d_, det, st),
                   "sk_fc_bwd")
        return o

    res, launches = {}, {}
    for det in (0, 0, 1):
        box = {}
        launches[det] = _launches(lib, lambda: box.update(run(det)))
        torch.cuda.synchronize()
        if det in res:
            for k in ("zpre", "z", "att", "ds", "dw1", "dw2", "dgamma", "dbeta", "mm", "mv"):
                assert torch.equal(res[det][k], box[k]), k
        res[det] = box
    assert launches[0] > launches[1], launches
    d = {k: v.double().cpu() for k, v in t.items()}
    for det in (0, 1):
        o = {k: v.double().cpu() for k, v in res[det].items()}
        ref, b = _gemm_bound(d["s"], d["w1"].t(), f)
        _chk(o["zpre"], ref, b, "sk zpre det=%d" % det)
        # batch norm over the batch from the device's zpre (no split-K here: 1e-5 of the scale)
        zp = o["zpre"]
        mean, var = zp.mean(0), zp.var(0, unbiased=False)
        z_ref = torch.relu((zp - mean) * torch.rsqrt(var + 1e-5) * d["gamma"] + d["beta"])
        assert _relerr(o["z"], z_ref) < 1e-5
        ref, b = _gemm_bound(o["z"], d["w2"].t(), d_)
        _chk(o["fwd_scratch"].view(B, 2 * f), ref, b, "sk a det=%d" % det)
        # backward: da = [t, -t], t = att (1 - att) dA; dW2 += da^T z; dW1 += dzpre^T s; ds = dzpre W1
        tt = o["att"] * (1 - o["att"]) * d["dA"]
        da = o["scratch"][:B * 2 * f].view(B, 2 * f)
        _chk(da, torch.cat([tt, -tt], 1), 4 * U * torch.cat([tt, tt], 1).abs(), "sk da det=%d" % det)
        ref, b = _gemm_bound(da.t(), o["z"], B, d["dw2"])
        _chk(o["dw2"], ref, b, "sk dw2 det=%d" % det)
        dzp = o["scratch"][B * 2 * f:B * (2 * f + d_)].view(B, d_)
        ref, b = _gemm_bound(dzp.t(), d["s"], B, d["dw1"])
        _chk(o["dw1"], ref, b, "sk dw1 det=%d" % det)
        ref, b = _gemm_bound(dzp, d["w1"], d_)
        _chk(o["ds"], ref, b, "sk ds det=%d" % det)
        # dzpre: batch-norm backward of (da W2) [z > 0] (fp64 restatement, 1e-5 of its scale)
        dz = (da @ d["w2"]) * (o["z"] > 0)
        bs = o["bnstat"]
        xh = (o["zpre"] - bs[:d_]) * bs[d_:]
        s1, s2 = dz.sum(0), (dz * xh).sum(0)
        assert _relerr(dzp, d["gamma"] * bs[d_:] * (dz - s1 / B - xh * s2 / B)) < 1e-5
        assert _relerr(o["dgamma"] - d["dgamma"], s2) < 1e-5
        assert _relerr(o["dbeta"] - d["dbeta"], s1) < 1e-5
    for k in ("zpre", "z", "att", "ds", "dw1", "dw2"):
        a, b_ = res[0][k].double(), res[1][k].double()
        assert _relerr(a, b_) < 1e-5, k


# ---------------------------------------------------------------------------------------------
# d. CUDA-graph capture: memory nodes and arrival counters behave the same on every replay
# ---------------------------------------------------------------------------------------------
GRAPH_WGRADS = [
    _geom(32, 28, 28, 128, 128, 3, 1, (1, 1, 1, 1)),    # im2col, 128-pixel stages
    _geom(64, 14, 14, 256, 1024, 1, 1),                 # plain, N tile 256
]


def _wgrad_inputs(g, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    Ho, Wo = g.out_hw()
    return (torch.randn(g.B, g.H, g.W, g.Cin, device="cuda", generator=gen).bfloat16(),
            torch.randn(g.B, Ho, Wo, g.Cout, device="cuda", generator=gen).bfloat16(),
            torch.empty(g.Cout, g.kh, g.kw, g.Cin, device="cuda"))


def test_graph_replay_of_split_k_is_bit_identical_to_eager(lib):
    for g in GRAPH_WGRADS:
        assert _plan(lib, g)[1] > 1, "must run split-K under the default heuristic"
    wg = [_wgrad_inputs(g, i) for i, g in enumerate(GRAPH_WGRADS)]
    B, Cc = 256, 1024
    r, t = _se_inputs(B, Cc, seed=5)
    se = dict(dw1=torch.empty_like(t["dw1"]), dw2=torch.empty_like(t["dw2"]),
              dq=torch.empty(B, Cc, device="cuda"), scratch=torch.empty(B * (Cc + r), device="cuda"))
    outs = [w[2] for w in wg] + [se["dw1"], se["dw2"], se["dq"]]

    def seq():
        st = _stream()
        for o in outs[:4]:
            o.zero_()
        for g, (x, dy, dw) in zip(GRAPH_WGRADS, wg):
            _wgrad(lib, g, x, dy, dw, stream=st)
        from assembled_cnn_b200 import _lib
        _lib.check(lib.acnn_se_fc_bwd(t["de"].data_ptr(), t["e"].data_ptr(), t["h"].data_ptr(),
                                      t["q"].data_ptr(), t["w1"].data_ptr(), t["w2"].data_ptr(),
                                      se["dw1"].data_ptr(), se["dw2"].data_ptr(), se["dq"].data_ptr(),
                                      se["scratch"].data_ptr(), B, Cc, r, 49, 0, st), "se_fc_bwd")

    seq()
    torch.cuda.synchronize()
    eager = [o.clone() for o in outs]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            seq()
    torch.cuda.current_stream().wait_stream(side)
    for o in outs:
        o.fill_(float("nan"))
    for rep in range(3):
        graph.replay()
        torch.cuda.synchronize()
        for i, (a, b) in enumerate(zip(eager, outs)):
            assert torch.equal(a, b), "replay %d output %d" % (rep, i)


# ---------------------------------------------------------------------------------------------
# e. two streams at once: every launch has its own scratch
# ---------------------------------------------------------------------------------------------
def test_two_streams_concurrently_match_sequential(lib):
    specs = [(GRAPH_WGRADS[0], 256, 1024), (GRAPH_WGRADS[1], 200, 512)]
    for g, _, _ in specs:
        assert _plan(lib, g)[1] > 1
    data = []
    for i, (g, B, Cc) in enumerate(specs):
        x, dy, _ = _wgrad_inputs(g, 10 + i)
        r, t = _se_inputs(B, Cc, seed=20 + i)
        data.append((g, x, dy, B, Cc, r, t))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]

    def launch(i):
        g = data[i][0]
        dw = torch.zeros(g.Cout, g.kh, g.kw, g.Cin, device="cuda")
        torch.cuda.synchronize()        # buffers ready before the other stream's work
        return dw

    def run(i, dw, st):
        g, x, dy, B, Cc, r, t = data[i]
        _wgrad(lib, g, x, dy, dw, stream=st)
        return _se_bwd(lib, t, B, Cc, r, 0, stream=st)

    def collect(dw, se):
        return [dw.clone(), se["dw1"].clone(), se["dw2"].clone(), se["dq"].clone()]

    # one after the other
    seq = []
    for i in range(2):
        dw = launch(i)
        se = run(i, dw, streams[i].cuda_stream)
        torch.cuda.synchronize()
        seq.append(collect(dw, se))
    # both in flight, no synchronisation between the streams
    dws = [launch(0), launch(1)]
    ses = [run(i, dws[i], streams[i].cuda_stream) for i in range(2)]
    torch.cuda.synchronize()
    for i in range(2):
        for j, (a, b) in enumerate(zip(seq[i], collect(dws[i], ses[i]))):
            assert torch.equal(a, b), "stream %d output %d" % (i, j)
