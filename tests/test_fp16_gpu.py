"""GPU tests of the fp16 mode (dtype='fp16', ACNN_F16: fp16 activation storage, wgmma .f16.f16 conv GEMMs with
fp32 accumulation, fp32 logits and loss, a static loss scale).

  * the fp16 conv GEMMs (fprop with the statistics / add / mask epilogues, dgrad, wgrad) against float64 with
    per-element bounds derived from their arithmetic, and bit-identical on a repeated launch and under
    CUDA-graph replay;
  * the configurations of test_native_model_gpu.py in fp16 (every fp16 kernel instantiation of the step runs
    there): op by op against the float64 interpreter that rounds at fp16's storage points, and the whole
    step bit for bit against the same ops run one at a time;
  * one training step in fp16 and in bf16 on the same inputs against the float64 plan interpreter;
  * the loss scale: the Trainer's default of 128, and the exactness of a power-of-two scale;
  * the fp16 retrieval search against a float64 restatement on fp16-rounded operands.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_native_model_gpu as nmg

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
ACNN_F16 = 3


def _ulp_f16(x):
    """Spacing of fp16 numbers at |x| (11 significant bits), float64; the subnormal spacing below 2^-14."""
    x = x.double().abs().clamp_min(2.0 ** -14)
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), (e - 11).to(torch.int64))


def _nrel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def _check(got, ref, tol, what):
    d = (got.double() - ref.double()).abs()
    bad = ~(d <= tol)
    assert not bool(bad.any()), "%s: %d of %d outside; max |d| / tol %.3g" % (
        what, int(bad.sum()), bad.numel(), float((d / tol).max()))


def _rand_f16(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).half().cuda()


def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _fwd64(x, w, g):
    """float64 conv of NHWC x with OHWI w under geometry g (explicit padding), NHWC result."""
    xp = F.pad(_nchw(x), (g.pad_w_lo, g.pad_w_hi, g.pad_h_lo, g.pad_h_hi))
    return F.conv2d(xp, w.double().permute(0, 3, 1, 2), stride=g.stride).permute(0, 2, 3, 1)


# (B, H, W, Cin, Cout, k, stride, pads): 1x1 plain, 3x3 on the halo kernel (H >= 56, Cin % 64 == 0), 3x3 on
# im2col (small images, Cin = 32), the stride-2 convs, the narrow N tiles and a 16-channel chunk
GEOMS = [
    (32, 56, 56, 64, 256, 1, 1, (0, 0, 0, 0)),
    (32, 28, 28, 512, 128, 1, 1, (0, 0, 0, 0)),
    (32, 56, 56, 64, 64, 3, 1, (1, 1, 1, 1)),
    (32, 14, 14, 256, 256, 3, 1, (1, 1, 1, 1)),
    (32, 28, 28, 32, 64, 3, 1, (1, 1, 1, 1)),
    (32, 56, 56, 128, 128, 3, 2, (0, 1, 0, 1)),
    (16, 7, 7, 64, 32, 3, 1, (1, 1, 1, 1)),
    (8, 30, 30, 16, 64, 3, 1, (1, 1, 1, 1)),
]


def _geom(B, H, W, Cin, Cout, k, s, pads):
    from assembled_cnn_b200._lib import ConvGeom
    return ConvGeom(B, H, W, Cin, Cout, k, k, s, *pads)


@pytest.mark.parametrize("gi", range(len(GEOMS)))
def test_conv_gemms_fp16_against_float64(gi):
    from assembled_cnn_b200 import _lib
    lib = _lib.load()
    g = _geom(*GEOMS[gi])
    Ho, Wo = g.out_hw()
    K = g.kh * g.kw * g.Cin
    st = torch.cuda.current_stream().cuda_stream
    x = _rand_f16((g.B, g.H, g.W, g.Cin), 1)
    w = _rand_f16((g.Cout, g.kh, g.kw, g.Cin), 2, 1.0 / math.sqrt(K))
    add = _rand_f16((g.B, Ho, Wo, g.Cout), 3, 0.5)
    mask = _rand_f16((g.B, Ho, Wo, g.Cout), 4)
    ref = _fwd64(x, w, g)
    mag = _fwd64(x.abs(), w.abs(), g)
    # fp32 accumulation of K products (each chain of wgmma / register adds rounds at most 2u per add),
    # then one fp16 rounding of the stored value
    acc_tol = 2 * K * U32 * mag

    def fprop(add_src=None, mask_src=None, stats=False):
        y = torch.full((g.B, Ho, Wo, g.Cout), float("nan"), dtype=torch.float16, device="cuda")
        parts = lib.acnn_conv_stats_parts(g)
        sp = torch.full((parts, 2, g.Cout), float("nan"), device="cuda") if stats else None
        _lib.check(lib.acnn_conv_fprop(g, x.data_ptr(), w.data_ptr(), y.data_ptr(),
                                       sp.data_ptr() if stats else None,
                                       add_src.data_ptr() if add_src is not None else None,
                                       mask_src.data_ptr() if mask_src is not None else None, None, 0,
                                       ACNN_F16, 0, st), "conv_fprop")
        return y, sp

    y, sp = fprop(stats=True)
    torch.cuda.synchronize()
    _check(y, ref, acc_tol + _ulp_f16(ref.abs() + acc_tol), "fprop")
    assert _nrel(y, ref) < 2.0 ** -11                 # one fp16 rounding, on average well below its bound
    # statistics = column sums / sums of squares of the STORED fp16 output, summed per CTA row in fp32
    yd = y.double().reshape(-1, g.Cout)
    s, q = sp.double().sum(0)
    n = yd.shape[0]
    _check(s, yd.sum(0), n * U32 * yd.abs().sum(0) + 1e-30, "fprop column sums")
    _check(q, (yd * yd).sum(0), 2 * n * U32 * (yd * yd).sum(0) + 1e-30, "fprop column sums of squares")
    # the same launch again and under graph replay: the same bits
    y2, sp2 = fprop(stats=True)
    gr = torch.cuda.CUDAGraph()
    yg = torch.empty_like(y)
    with torch.cuda.graph(gr):
        _lib.check(lib.acnn_conv_fprop(g, x.data_ptr(), w.data_ptr(), yg.data_ptr(), None, None, None, None, 0,
                                       ACNN_F16, 0, torch.cuda.current_stream().cuda_stream), "conv_fprop")
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, y2) and torch.equal(sp, sp2) and torch.equal(y, yg)
    # fused epilogue: (y + add) * (mask > 0), one fp16 rounding of the fp32 sum
    ya, _ = fprop(add, mask)
    refa = (ref + add.double()) * (mask.double() > 0)
    tola = acc_tol + U32 * (mag + add.double().abs())
    _check(ya, refa, tola + _ulp_f16(refa.abs() + tola), "fprop add / mask")
    assert torch.isfinite(ya).all()

    # weight gradient: dw[Cout][kh][kw][Cin] (fp32) += sum over pixels x (*) dy
    dy = _rand_f16((g.B, Ho, Wo, g.Cout), 5, 0.1)
    P = g.B * Ho * Wo
    for det in (0, 1):
        dw = torch.zeros(g.Cout, g.kh, g.kw, g.Cin, device="cuda")
        _lib.check(lib.acnn_conv_wgrad(g, x.data_ptr(), dy.data_ptr(), dw.data_ptr(), ACNN_F16, det, st),
                   "conv_wgrad")
        torch.cuda.synchronize()
        xp = F.pad(_nchw(x), (g.pad_w_lo, g.pad_w_hi, g.pad_h_lo, g.pad_h_hi))
        ref_w = torch.nn.grad.conv2d_weight(xp, (g.Cout, g.Cin, g.kh, g.kw), _nchw(dy),
                                            stride=g.stride).permute(0, 2, 3, 1)
        mag_w = torch.nn.grad.conv2d_weight(xp.abs(), (g.Cout, g.Cin, g.kh, g.kw), _nchw(dy).abs(),
                                            stride=g.stride).permute(0, 2, 3, 1)
        _check(dw, ref_w, 2 * P * U32 * mag_w + 1e-30, "wgrad det=%d" % det)
        # the per-element bound is a worst case (it grows with P^2 where the rounding error grows with
        # sqrt(P)); as a whole the result must be close: 1e-3 norm-relative (measured 1.2e-4 at P = 100352,
        # the tensor cores' truncating fp32 accumulation), so a wrong or missing sum cannot pass
        assert _nrel(dw, ref_w) < 1e-3, _nrel(dw, ref_w)
        dw2 = torch.zeros_like(dw)
        _lib.check(lib.acnn_conv_wgrad(g, x.data_ptr(), dy.data_ptr(), dw2.data_ptr(), ACNN_F16, det, st),
                   "conv_wgrad")
        torch.cuda.synchronize()
        assert torch.equal(dw, dw2)

    # data gradient of the stride-1 convs: w_dgrad [Cin][kh][kw flipped][Cout] (Cin is its GEMM N: % 32)
    if g.stride == 1 and g.Cin % 32 == 0:
        wd = w.flip(1, 2).permute(3, 1, 2, 0).contiguous()
        dx = torch.full((g.B, g.H, g.W, g.Cin), float("nan"), dtype=torch.float16, device="cuda")
        _lib.check(lib.acnn_conv_dgrad(g, dy.data_ptr(), wd.data_ptr(), dx.data_ptr(), None, None, ACNN_F16, 0,
                                       st), "conv_dgrad")
        torch.cuda.synchronize()
        shape = (g.B, g.Cin, g.H + g.pad_h_lo + g.pad_h_hi, g.W + g.pad_w_lo + g.pad_w_hi)
        full = torch.nn.grad.conv2d_input(shape, w.double().permute(0, 3, 1, 2), _nchw(dy))
        ref_x = full[:, :, g.pad_h_lo:g.pad_h_lo + g.H, g.pad_w_lo:g.pad_w_lo + g.W].permute(0, 2, 3, 1)
        fullm = torch.nn.grad.conv2d_input(shape, w.double().abs().permute(0, 3, 1, 2), _nchw(dy).abs())
        mag_x = fullm[:, :, g.pad_h_lo:g.pad_h_lo + g.H, g.pad_w_lo:g.pad_w_lo + g.W].permute(0, 2, 3, 1)
        tol = 2 * g.kh * g.kw * g.Cout * U32 * mag_x
        _check(dx, ref_x, tol + _ulp_f16(ref_x.abs() + tol), "dgrad")
        assert _nrel(dx, ref_x) < 2.0 ** -11


FP16_CASES = dict(nmg.CASES)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _assert_same_bits(a, b, what):
    """Bit equality (an inf or NaN that both executors produce is the same value here)."""
    assert a.shape == b.shape and a.dtype == b.dtype, what
    ne = _bits(a) != _bits(b)
    assert not bool(ne.any()), "%s differs: %d of %d elements" % (what, int(ne.sum()), ne.numel())


@pytest.mark.parametrize("case", sorted(FP16_CASES))
def test_fp16_step_bit_identical_to_op_by_op(case):
    """The library's whole fp16 step gives the bits of the same ops run one acnn_run_ops call at a time
    (deterministic mode) over two steps: every activation, gradient and input buffer, the loss, the moving
    statistics, weights, gradients and momentum.  The first step's loss is finite.  (With these random weights
    the second step of the 152-layer configuration overflows fp16 -- values above 65504 become inf, as the
    reference's fp16 casts do -- and both runs produce the same infinities and NaNs.)"""
    plan, rt, loss = nmg.step_equals_op_by_op(case, True, dtype="fp16", same=_assert_same_bits)
    assert rt.adt == ACNN_F16
    assert torch.isfinite(loss).all() and float(loss[0]) > 0


@pytest.mark.parametrize("case", sorted(FP16_CASES))
def test_fp16_lockstep_against_interpreter(case):
    """test_fp16_lockstep_gpu's lock-step (fp16 tolerances) on the configurations of test_native_model_gpu.CASES
    in fp16, deterministic mode, on the oracle's weights, unscaled (test_fp16_lockstep_gpu runs scale 128; at
    that scale the 152-layer configuration's backward overflows fp16 here, in the interpreter as on the GPU)."""
    failures, worst = nmg.lockstep_case(case, True, dtype="fp16")
    print("fp16 lock-step %s: worst rel err per op kind:output" % case)
    for k, v in sorted(worst.items()):
        print("  %-28s %.3e" % (k, v))
    assert not failures, "\n".join(failures[:20])


def _oracle_step(plan, w, feeds, hp):
    """float64 plan interpreter: the same plan, op for op, without any rounding of the storage."""
    from oracle import plan_interp as PI
    it = PI.PlanInterpreter(plan, dtype=torch.float64)
    it.set_weights({k: v.double() for k, v in w.items()})
    it.hp.update(hp)
    m = plan.meta
    x = feeds[m["images"]].double()
    lab = feeds[m["labels"]]
    lam1 = feeds.get(m.get("lam1"))
    logits, ce, l2 = it.train_step(x, lab, None if lam1 is None else lam1.double())
    return it, logits, ce


def test_fp16_training_step_error_vs_bf16_against_float64():
    """One Assemble-ResNet-50 training step (mixup 1, label smoothing) in fp16 and in bf16 on the same weights
    and inputs, both against the float64 interpreter of the same plan: the fp16 errors in the logits, the
    loss, the moving statistics and the gradients are no larger than the bf16 ones."""
    from assembled_cnn_b200 import native
    from assembled_cnn_b200.plan import ModelConfig
    flags, B, hw = nmg.ASSEMBLE, 16, 128
    kw = dict(training=True, mixup_type=1, label_smoothing=0.1)
    cfg = ModelConfig(**flags)
    hp = dict(lr=0.05, momentum=0.9, weight_decay=1e-4)
    errs, ref = {}, None
    for dtype in ("bf16", "fp16"):
        nm = native.NativeModel(cfg, B, hw, hw, dtype=dtype, **kw)
        plan = nm.python_mirror()
        w = nmg._weights(plan)
        feeds = nmg._feeds(plan)
        rt = native.NativeRuntime(nm)
        rt.set_weights(w)
        rt.set_hparams(**hp)
        ls = 128.0 if dtype == "fp16" else 1.0
        rt.loss_scale = ls
        rt.set_hparams(grad_scale=1.0 / ls)
        for name, v in feeds.items():
            rt.t[name].copy_(v)
        rt.run_step()
        torch.cuda.synchronize()
        if ref is None:
            ref = _oracle_step(plan, w, feeds, dict(hp))
        it, logits64, ce64 = ref
        m = plan.meta
        nc = m["num_classes"]
        e = {}
        lg = rt.t[m["logits"]][:, :nc].double().cpu()
        e["logits"] = ((lg - logits64[:, :nc]).norm() / logits64[:, :nc].norm()).item()
        e["cross_entropy"] = abs(float(rt.slot_view(m["loss"])[0]) - ce64) / abs(ce64)
        st = rt.state.double().cpu()
        e["moving_statistics"] = ((st - it.state).norm() / it.state.norm()).item()
        gr = rt.grads.double().cpu() / ls
        per = {}
        for name, p in plan.params.items():
            a, b = gr[p.offset:p.offset + p.size], it.grads[p.offset:p.offset + p.size]
            if float(b.norm()) > 0:
                per[name] = ((a - b).norm() / b.norm()).item()
        e["grads"] = per
        errs[dtype] = e
        assert torch.isfinite(rt.grads).all() and torch.isfinite(rt.params).all()
        del rt, nm
    for k in ("logits", "cross_entropy", "moving_statistics"):
        print("fp16 step %s error %.3e (bf16 %.3e)" % (k, errs["fp16"][k], errs["bf16"][k]))
    g16, gbf = np.array(list(errs["fp16"]["grads"].values())), np.array(list(errs["bf16"]["grads"].values()))
    print("gradient tensors' norm-relative errors: fp16 median %.3e max %.3e; bf16 median %.3e max %.3e"
          % (np.median(g16), g16.max(), np.median(gbf), gbf.max()))
    print("gradient tensors where fp16 > bf16: %d of %d" % (int((g16 > gbf).sum()), len(g16)))
    for k in ("logits", "cross_entropy", "moving_statistics"):
        assert errs["fp16"][k] <= errs["bf16"][k], k
    assert (g16 <= gbf).all()


def test_fp16_loss_scale():
    """Trainer: loss_scale 128 by default in fp16 (1 in bf16); an explicit value wins.

    A power-of-two scale is exact wherever no fp16 value it passes through is subnormal or overflows.  A
    whole ResNet-50 backward has no such scale: its fp16 gradients span more than fp16's 2^30 normal range
    (measured on this configuration: subnormal values remain up to scale 2^14 while values overflow from
    2^16 on), so the exactness is asserted on the part of the step built to satisfy the condition -- the
    loss and the dense head with 10 classes, whose fp16 logit gradients are all normal at scales 1 and 128
    (asserted): the bias gradient (fp32, from the fp32 logit gradients) and the dense kernel's gradient (an
    fp16 GEMM on them) at scale 128 are 128 times those at scale 1, bit for bit.  The rest of the step at
    scale 128 stays finite and within 1e-2 of the unscaled one."""
    from assembled_cnn_b200 import model_fns as Fm, native
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.plan import ModelConfig
    for dtype, want in (("fp16", 128.0), ("bf16", 1.0)):
        p = params_from_flags(resnet_size=50, batch_size=4, dtype=dtype)
        tr = Fm.Trainer(Fm.build_model(**{k: p[k] for k in ("resnet_size", "dtype")}), p, 64, 64,
                        use_cuda_graph=False, num_images=1000)
        assert tr.loss_scale == want and tr.rt.loss_scale == want
        p2 = params_from_flags(resnet_size=50, batch_size=4, dtype=dtype, loss_scale=8)
        tr2 = Fm.Trainer(Fm.build_model(**{k: p2[k] for k in ("resnet_size", "dtype")}), p2, 64, 64,
                         use_cuda_graph=False, num_images=1000)
        assert tr2.loss_scale == 8.0
        del tr, tr2
    cfg = ModelConfig(resnet_size=50, num_classes=10)
    B, hw = 4, 64
    out = {}
    for ls in (1.0, 128.0):
        nm = native.NativeModel(cfg, B, hw, hw, dtype="fp16", training=True, deterministic=True)
        plan = nm.python_mirror()
        rt = native.NativeRuntime(nm)
        rt.set_weights(nmg._weights(plan))
        rt.set_hparams(lr=0.05, momentum=0.9, weight_decay=1e-4, grad_scale=1.0 / ls)
        rt.loss_scale = ls
        for name, v in nmg._feeds(plan).items():
            rt.t[name].copy_(v)
        rt.run_step()
        torch.cuda.synchronize()
        ce = next(op for op in plan.forward if op.kind == "softmax_ce")
        dl = rt.t[ce.a["dlogits"]][:, :10].float()
        head = {n: rt.grads[q.offset:q.offset + q.size].clone() for n, q in plan.params.items()
                if n.startswith("resnet_model/dense/")}
        out[ls] = dict(dl=dl, head=head, grads=rt.grads.clone(),
                       finite=all(bool(torch.isfinite(t).all()) for t in rt.t.values() if t.is_floating_point()))
        del rt, nm
    for ls in (1.0, 128.0):
        dl = out[ls]["dl"]
        assert bool(((dl == 0) | (dl.abs() >= 2.0 ** -14)).all()) and bool(torch.isfinite(dl).all())
    assert len(out[1.0]["head"]) == 2
    for n, g1 in out[1.0]["head"].items():
        assert float(g1.abs().sum()) > 0 and torch.equal(out[128.0]["head"][n], 128.0 * g1), n
    assert out[128.0]["finite"]
    rel = ((out[128.0]["grads"] / 128.0 - out[1.0]["grads"]).norm() / out[1.0]["grads"].norm()).item()
    assert rel < 1e-2, rel


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_fp16_retrieval_search_against_restatement(metric):
    """knn_topk(dtype='fp16'): the similarities of fp16-rounded operands with fp32 accumulation, ranked by
    (similarity desc, index asc).  Restated in float64 on the same fp16 operands: every returned similarity
    is that of its index within the accumulation bound, the lists are sorted, and no row is missed that beats
    the k-th by more than the bound."""
    from assembled_cnn_b200.metrics import knn_topk
    g = torch.Generator().manual_seed(3)
    nq, nx, d, k = 300, 1000, 96, 6
    q = torch.randn(nq, d, generator=g)
    x = torch.randn(nx, d, generator=g)
    x[5] = x[7]                                       # an exact tie: the lower index first
    idx, sim = knn_topk(q.cuda(), x.cuda(), k, similarity=metric, dtype="fp16")
    idx, sim = idx.cpu().long(), sim.cpu().double()

    def rows(a):
        a32 = a.float()
        if metric == "cosine":
            a32 = a32 * torch.rsqrt(torch.clamp((a32 * a32).sum(1, keepdim=True), min=1e-12))
        return a32.half().double()
    qh, xh = rows(q), rows(x)
    dots = qh @ xh.T
    if metric == "cosine":
        s64 = dots
    else:
        s64 = -((qh * qh).sum(1)[:, None] + (xh * xh).sum(1)[None, :] - 2 * dots)
    mag = qh.abs() @ xh.abs().T
    if metric == "euclidean":
        mag = mag * 2 + (qh * qh).sum(1)[:, None] + (xh * xh).sum(1)[None, :]
    tol = 4 * d * U32 * mag + 1e-6
    got_ref = s64.gather(1, idx)
    assert ((sim - got_ref).abs() <= tol.gather(1, idx)).all()
    assert (sim[:, :-1] >= sim[:, 1:]).all()
    kth = sim[:, -1:]
    missed = (s64 > kth + 2 * tol) & ~torch.zeros_like(s64, dtype=torch.bool).scatter(1, idx, True)
    assert not bool(missed.any())
    both = (idx == 5).any(1) & (idx == 7).any(1)
    for r in torch.nonzero(both).flatten().tolist():
        l = idx[r].tolist()
        assert l.index(5) < l.index(7)
