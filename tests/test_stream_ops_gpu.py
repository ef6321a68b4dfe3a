"""Op-level tests of the HBM-bound kernels (csrc/bn_ops.cu, pool_ops.cu, head_ops.cu, optim_ops.cu)
through the C ABI, against float64 references, at the production shapes of the c3 / c5 training plans
(B = 256, 224 px: every distinct (op, shape) of plan.build_plan(...).all_ops()) and at the grid edges.

References are float64 and computed from the kernel's own inputs (bf16- or fp32-representable).  The
ops oracle/tf_ops.py defines (blur-pool, avg / max pool, upsample, global pooling, GeM, DropBlock,
softmax CE, KD, mixup, momentum step) use it, on the CPU, over a fixed sample of images (the first, the
last and four seeded ones) and through its autograd for the backward kernels.  The formulas it does not
define (BN backward coefficients, the SK combine / gate / BN backward, bn_act, partial rows) are restated
here in float64 on the device and compared in full.  Tolerances: oracle/stream_check.py (derivations
there); each one is shown sharp enough by tests/test_stream_ops_cpu.py.

  entry point                      production-shape test           edge test                        reference          tolerance
  acnn_bn_act                      test_bn_act_plan_shapes         test_bn_act_edges                restated            elementwise, 4 ops
  acnn_bn_bwd_reduce / _finalize   test_bn_bwd_plan_shapes         test_bn_bwd_edges                restated            reduction per partial row
    / _apply                                                        test_bn_bwd_finalize_nparts                         / coefficient chain / 6 ops
  acnn_bn_bwd_reduce2 / _apply2    test_bn_bwd2_plan_shapes        test_bn_bwd_edges                restated            as above
  acnn_bn_finalize                 test_bn_finalize_plan_channels  test_bn_finalize_nparts          restated            1 ulp of the double result
  acnn_bn_stats                    test_bn_stats_production        test_bn_stats_production (C 8)   exactly summable    exact mean, 1 ulp var
  acnn_sk_gap / _bwd_gate          test_sk_plan_shapes             test_sk_edges                    restated            reduction per image
  acnn_sk_combine                  test_sk_plan_shapes             test_sk_edges                    restated (sk_attention) elementwise, 5 ops
  acnn_sk_bn_bwd_reduce / _apply   test_sk_plan_shapes             test_sk_edges                    restated            reduction per slab / 6 ops
  acnn_se_gap                      test_se_reductions_plan_shapes  test_se_reductions_edges         restated            reduction per image
  acnn_se_bwd_gate                 (both in tests/test_image_reduce_ops_gpu.py, bf16 / fp16 / fp32)  restated            reduction per image
  acnn_blurpool_fwd / _bwd         test_blurpool_plan_shapes       test_blurpool_edges              anti_aliased_downsample  filt^2 chain
  acnn_avgpool_fwd / _bwd          test_avgpool_plan_shapes        test_avgpool_edges               restated, = avg_pool_bl / _resnet_d  k^2 chain
  acnn_maxpool_fwd / _bwd          test_maxpool_production         test_maxpool_edges               restated, = max_pool_same  exact / k^2 chain
  acnn_upsample2x_bwd              test_resample_plan_shapes       test_resample_edges              upsample2x autograd 5-term chain
  acnn_zero_insert2x               test_resample_plan_shapes       test_resample_edges              restated            exact
  acnn_grad_combine                test_grid_cap_bit_identical     test_resample_edges              restated            1 op
  acnn_gap_fwd / _gap_bwd          test_gap_plan_shapes            test_gap_edges                   global_avg_pool     reduction / 2 ops
  acnn_gem_fwd / _bwd              test_gem_production             test_gem_edges                   generalized_mean_pooling  reduction / 10 ops
  acnn_dropblock_apply             test_dropblock_plan_shapes      test_dropblock_edges             dropblock_keep_mask 2 ops
  acnn_softmax_ce                  test_softmax_ce (B 256, 512)    test_softmax_ce (B 1, 33)        softmax_cross_entropy, kd_loss  derived below
  acnn_pack_input / _mix_labels    test_pack_input_plan            test_pack_input_plan (mode 2)    mixup               4 / 3 ops
  acnn_sgd_momentum                test_sgd_c3_parameters          test_sgd_edges                   momentum_step       3 ops / reduction
  grid-stride launches             test_grid_cap_bit_identical (caps 132, 264, default, 65535)
  reductions                       test_reductions_repeat_and_graph_replay_bit_identical
  acnn_set_pdl                     test_pdl_training_step_bit_identical
  cg_ok rejection                  test_channel_groups_rejected_before_launch
"""
import contextlib
import functools
import random

import pytest
import torch
import torch.nn.functional as F

from oracle import stream_check as SC
from oracle import tf_ops

pytestmark = pytest.mark.gpu

U = SC.U32
DTYPES = {"bf16": (0, torch.bfloat16), "f32": (1, torch.float32)}
CG_OK_C = [8, 16, 32, 64, 128, 256, 512, 1024, 2048]     # C / 8 divides 256


def _L():
    from assembled_cnn_b200 import _lib
    return _lib


def _st():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _check(rc, what):
    _L().check(rc, what)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rand(shape, tdt, seed, scale=1.0, shift=0.0):
    return (torch.randn(shape, generator=_gen(seed), device="cuda") * scale + shift).to(tdt)


def _unif(shape, seed, lo=0.0, hi=1.0):
    return torch.rand(shape, generator=_gen(seed), device="cuda") * (hi - lo) + lo


def _nan(shape, tdt):
    return torch.full(shape, float("nan"), dtype=tdt, device="cuda")


def _sample(B):
    """The first, the last and four seeded images."""
    if B <= 6:
        return list(range(B))
    return sorted({0, B - 1, *random.Random(7 * B + 1).sample(range(1, B - 1), 4)})


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


# ---------------------------------------------------------------------------------------------------
# production shapes: every distinct (op, shape) of the c3 / c5 training plans at B = 256, 224 px
# ---------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _plan(name, **extra):
    import bench
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    cfg = ModelConfig(num_classes=1001, **bench.CONFIGS[name]["model"])
    return build_plan(cfg, 256, 224, 224, mixup_type=1, label_smoothing=0.1, **extra)


def _plan_cases(kind, key, plans=(("c3", ()), ("c5", ()))):
    seen = set()
    for name, extra in plans:
        for op in _plan(name, **dict(extra)).all_ops():
            if op.kind == kind:
                seen.add(key(op))
    return sorted(seen)


def _ids(cases):
    return ["-".join(str(v) for v in (c if isinstance(c, tuple) else (c,))).replace(" ", "")
            for c in cases]


@pytest.fixture(params=sorted(DTYPES))
def dt(request):
    return request.param


@contextlib.contextmanager
def _grid_cap(lib, cap):
    prev = lib.acnn_set_stream_grid_cap(cap)
    try:
        yield
    finally:
        lib.acnn_set_stream_grid_cap(prev)


# ---------------------------------------------------------------------------------------------------
# bn_act
# ---------------------------------------------------------------------------------------------------
def _bn_act_inputs(B, H, W, C, b_mode, gate, tdt, seed):
    t = dict(a=_rand((B, H, W, C), tdt, seed), sa=_rand((C,), torch.float32, seed + 1, 0.5, 1.0),
             ha=_rand((C,), torch.float32, seed + 2, 0.5), b=None, sb=None, hb=None, gate=None)
    if b_mode in (1, 2):
        t["b"] = _rand((B, H, W, C), tdt, seed + 3)
    elif b_mode == 3:
        t["b"] = _rand((B, H // 2, W // 2, C), tdt, seed + 3)
    if b_mode == 1:
        t["sb"] = _rand((C,), torch.float32, seed + 4, 0.5, 1.0)
        t["hb"] = _rand((C,), torch.float32, seed + 5, 0.5)
    if gate:
        t["gate"] = _unif((B, C), seed + 6)
    return t


def _bn_act_call(lib, t, b_mode, relu, code, shape):
    B, H, W, C = shape
    out = _nan(shape, t["a"].dtype)
    _check(lib.acnn_bn_act(_p(t["a"]), _p(t["sa"]), _p(t["ha"]), _p(t["b"]), _p(t["sb"]), _p(t["hb"]),
                           b_mode, _p(t["gate"]), int(relu), _p(out), B, H, W, C, code, _st()), "bn_act")
    return out


def _bn_act_check(t, out, idx, b_mode, relu, bf16, what):
    a = t["a"][idx].double()
    v = a * t["sa"].double() + t["ha"].double()
    mag = (a * t["sa"].double()).abs() + t["ha"].double().abs()
    if t["gate"] is not None:
        g = t["gate"][idx].double()[:, None, None, :]
        v, mag = v * g, mag * g
    if b_mode == 1:
        b = t["b"][idx].double()
        v = v + b * t["sb"].double() + t["hb"].double()
        mag = mag + (b * t["sb"].double()).abs() + t["hb"].double().abs()
    elif b_mode == 2:
        v, mag = v + t["b"][idx].double(), mag + t["b"][idx].double().abs()
    elif b_mode == 3:
        r = tf_ops.upsample2x(t["b"][idx].double())
        v, mag = v + r, mag + r.abs()
    if relu:
        v = v.clamp_min(0)
    SC.assert_within(out[idx], v, SC.elementwise_tol(v, mag, bf16, ops=4), what)


BN_ACT_CASES = _plan_cases("bn_act", lambda op: (tuple(op.shape), op.b_mode, op.gate is not None,
                                                 bool(op.relu)))


@pytest.mark.parametrize("case", BN_ACT_CASES, ids=_ids(BN_ACT_CASES))
def test_bn_act_plan_shapes(lib, dt, case):
    shape, b_mode, gate, relu = case
    code, tdt = DTYPES[dt]
    t = _bn_act_inputs(*shape, b_mode, gate, tdt, seed=11)
    out = _bn_act_call(lib, t, b_mode, relu, code, shape)
    torch.cuda.synchronize()
    _bn_act_check(t, out, _sample(shape[0]), b_mode, relu, dt == "bf16", "bn_act %s" % (case,))


@pytest.mark.parametrize("C", CG_OK_C)
def test_bn_act_edges(lib, dt, C):
    """Every accepted channel count, all four b_modes with and without the gate, ReLU on and off, on
    odd maps (modes 0-2) and on 2 x 2 / 6 x 10 maps (mode 3 needs even sizes), at the smallest grid cap
    so that the threads make several trips."""
    code, tdt = DTYPES[dt]
    with _grid_cap(lib, 132):
        for b_mode in range(4):
            for (B, H, W) in ([(3, 7, 5), (1, 1, 1), (64, 9, 13)] if b_mode < 3 else
                              [(3, 2, 2), (64, 6, 10)]):
                for gate in (False, True):
                    for relu in (False, True):
                        t = _bn_act_inputs(B, H, W, C, b_mode, gate, tdt, seed=C + b_mode)
                        out = _bn_act_call(lib, t, b_mode, relu, code, (B, H, W, C))
                        torch.cuda.synchronize()
                        _bn_act_check(t, out, list(range(B)), b_mode, relu, dt == "bf16",
                                      "bn_act C=%d mode=%d B,H,W=%s gate=%d relu=%d"
                                      % (C, b_mode, (B, H, W), gate, relu))


# ---------------------------------------------------------------------------------------------------
# batch-norm backward: reduce (partial rows), finalize (coefficients), apply
# ---------------------------------------------------------------------------------------------------
def _bn_bwd_terms(g, y, mean, rstd, gate=None, addbc=None, HW=1):
    """float64 [M, C] terms of the two partial sums, ge and ge * xhat, each with its magnitude (ge =
    g * gate + addbc is rounded twice in fp32 before it is added: its error scales with |g*gate| +
    |addbc|, not with |ge|)."""
    C = g.shape[-1]
    M = g.numel() // C
    ge = g.reshape(M, C).double()
    mag = ge.abs()
    if gate is not None or addbc is not None:
        B = M // HW
        ge, mag = ge.view(B, HW, C), mag.view(B, HW, C)
        if gate is not None:
            ge, mag = ge * gate.double()[:, None, :], mag * gate.double().abs()[:, None, :]
        if addbc is not None:
            ge, mag = ge + addbc.double()[:, None, :], mag + addbc.double().abs()[:, None, :]
        ge, mag = ge.reshape(M, C), mag.reshape(M, C)
    xhat = (y.reshape(M, C).double() - mean.double()) * rstd.double()
    return (ge, mag), (ge * xhat, mag * xhat.abs())


def _partials(terms, owner_rpb, nparts):
    """Sum [M, C] terms into the partial rows of acnn_bn_bwd_reduce: row r -> (r // RPB) % nparts."""
    M, C = terms.shape
    blk = nparts * owner_rpb
    pad = (-M) % blk
    t = torch.cat([terms, terms.new_zeros(pad, C)]) if pad else terms
    return t.view(-1, nparts, owner_rpb, C).sum(dim=(0, 2))


def _check_bn_bwd_parts(parts, terms_list, M, C, nparts, what):
    rpb = 256 // (C // 8)
    n_eff = SC.bn_bwd_reduce_chain(M, C, nparts)
    for k, (t, mag) in enumerate(terms_list):
        ref = _partials(t, rpb, nparts)
        tol = SC.reduction_tol(_partials(mag, rpb, nparts), n_eff, extra_ops=5)
        SC.assert_within(parts[:, k, :], ref, tol, "%s partial %s" % (what, ("sum ge", "sum ge*xhat")[k]))


def _bn_bwd_coef_ref(parts, gamma, mean, rstd, count):
    """float64 k1, k2, k3, dgamma, dbeta from the kernel's partial rows, and their tolerances: the
    partial rows are summed over chains of ceil(nparts / 32) rows + 32 lanes; k1 = gamma*rstd (1
    rounding), k2 = -k1*rstd*s2/count (3 + the error of s2), k3 = -k1*s1/count - k2*mean (4 + the
    errors of s1 and k2)."""
    nparts = parts.shape[0]
    P = parts.double()
    s1, s2 = P[:, 0].sum(0), P[:, 1].sum(0)
    n_eff = -(-nparts // 32) + 32
    t1, t2 = SC.reduction_tol(P[:, 0].abs().sum(0), n_eff), SC.reduction_tol(P[:, 1].abs().sum(0), n_eff)
    g, m, r = gamma.double(), mean.double(), rstd.double()
    k1 = g * r
    k2 = -k1 * r * s2 / count
    k3 = -k1 * s1 / count - k2 * m
    tk1 = 2 * U * k1.abs()
    tk2 = 5 * U * k2.abs() + (k1 * r / count).abs() * t2
    tk3 = 5 * U * ((k1 * s1 / count).abs() + (k2 * m).abs()) + (k1 / count).abs() * t1 + m.abs() * tk2
    return (k1, k2, k3, s2, s1), (tk1, tk2, tk3, t2, t1)


def _bn_bwd_finalize(lib, parts, gamma, mean, rstd, count, C, what):
    nparts = parts.shape[0]
    coef, dgamma, dbeta = _nan((3, C), torch.float32), _nan((C,), torch.float32), _nan((C,), torch.float32)
    _check(lib.acnn_bn_bwd_finalize(_p(parts), nparts, _p(gamma), _p(mean), _p(rstd), count, _p(coef),
                                    _p(dgamma), _p(dbeta), C, _st()), "bn_bwd_finalize")
    torch.cuda.synchronize()
    refs, tols = _bn_bwd_coef_ref(parts, gamma, mean, rstd, count)
    for name, got, ref, tol in zip(("k1", "k2", "k3", "dgamma", "dbeta"),
                                   (coef[0], coef[1], coef[2], dgamma, dbeta), refs, tols):
        SC.assert_within(got, ref, tol, "%s %s" % (what, name))
    return coef


def _bn_apply_check(dy, g, y, coef, idx, bf16, what, gate=None, addbc=None):
    k1, k2, k3 = (coef[i].double() for i in range(3))
    ge = g[idx].double()
    mag_ge = ge.abs()
    if gate is not None:
        gt = gate[idx].double()[:, None, None, :]
        ge, mag_ge = ge * gt, mag_ge * gt.abs()
    if addbc is not None:
        ab = addbc[idx].double()[:, None, None, :]
        ge, mag_ge = ge + ab, mag_ge + ab.abs()
    yy = y[idx].double()
    ref = k1 * ge + k2 * yy + k3
    mag = (k1 * mag_ge).abs() + (k2 * yy).abs() + k3.abs()
    SC.assert_within(dy[idx], ref, SC.elementwise_tol(ref, mag, bf16, ops=6), what)


def _bn_stats_inputs(C, seed):
    gamma = _rand((C,), torch.float32, seed, 0.3, 1.0)
    mean = _rand((C,), torch.float32, seed + 1, 0.5)
    rstd = _unif((C,), seed + 2, 0.5, 2.0)
    return gamma, mean, rstd


def _bn_bwd_case(lib, dt, B, H, W, C, gate=False, addbc=False, seed=21, idx=None):
    code, tdt = DTYPES[dt]
    HW, M = H * W, B * H * W
    gamma, mean, rstd = _bn_stats_inputs(C, seed)
    g = _rand((B, H, W, C), tdt, seed + 3)
    y = (_rand((B, H, W, C), torch.float32, seed + 4) / rstd + mean).to(tdt)
    gt = _unif((B, C), seed + 5) if gate else None
    ab = _rand((B, C), torch.float32, seed + 6, 0.1) if addbc else None
    nparts = lib.acnn_bn_bwd_reduce_parts(B, HW, C)
    assert 1 <= nparts <= 264
    parts = _nan((nparts, 2, C), torch.float32)
    _check(lib.acnn_bn_bwd_reduce(_p(g), _p(y), _p(mean), _p(rstd), _p(gt), _p(ab), _p(parts), B, HW, C,
                                  code, _st()), "bn_bwd_reduce")
    torch.cuda.synchronize()
    what = "bn_bwd %s %s gate=%d addbc=%d" % (dt, (B, H, W, C), gate, addbc)
    _check_bn_bwd_parts(parts, _bn_bwd_terms(g, y, mean, rstd, gt, ab, HW), M, C, nparts, what)
    coef = _bn_bwd_finalize(lib, parts, gamma, mean, rstd, M, C, what)
    dy = _nan((B, H, W, C), tdt)
    _check(lib.acnn_bn_bwd_apply(_p(g), _p(y), _p(coef), _p(gt), _p(ab), _p(dy), B, HW, C, code, _st()),
           "bn_bwd_apply")
    torch.cuda.synchronize()
    _bn_apply_check(dy, g, y, coef, idx if idx is not None else list(range(B)), dt == "bf16",
                    what + " apply", gt, ab)


BN_BWD_CASES = _plan_cases("bn_bwd_reduce", lambda op: (tuple(op.shape), op.gate is not None,
                                                        op.addbc is not None))


@pytest.mark.parametrize("case", BN_BWD_CASES, ids=_ids(BN_BWD_CASES))
def test_bn_bwd_plan_shapes(lib, dt, case):
    shape, gate, addbc = case
    _bn_bwd_case(lib, dt, *shape, gate=gate, addbc=addbc, idx=_sample(shape[0]))


def _bn_bwd2_case(lib, dt, B, H, W, C, seed=31, idx=None):
    code, tdt = DTYPES[dt]
    HW, M = H * W, B * H * W
    ga, ma, ra = _bn_stats_inputs(C, seed)
    gb, mb, rb = _bn_stats_inputs(C, seed + 10)
    g = _rand((B, H, W, C), tdt, seed + 3)
    ya = (_rand((B, H, W, C), torch.float32, seed + 4) / ra + ma).to(tdt)
    yb = (_rand((B, H, W, C), torch.float32, seed + 5) / rb + mb).to(tdt)
    nparts = lib.acnn_bn_bwd_reduce_parts(B, HW, C)
    pa, pb = _nan((nparts, 2, C), torch.float32), _nan((nparts, 2, C), torch.float32)
    _check(lib.acnn_bn_bwd_reduce2(_p(g), _p(ya), _p(yb), _p(ma), _p(ra), _p(mb), _p(rb), _p(pa), _p(pb),
                                   B, HW, C, code, _st()), "bn_bwd_reduce2")
    # bit-identical to the single-BN kernel (include/acnn.h)
    p1 = _nan((nparts, 2, C), torch.float32)
    _check(lib.acnn_bn_bwd_reduce(_p(g), _p(yb), _p(mb), _p(rb), None, None, _p(p1), B, HW, C, code,
                                  _st()), "bn_bwd_reduce")
    torch.cuda.synchronize()
    assert torch.equal(pb, p1)
    what = "bn_bwd2 %s %s" % (dt, (B, H, W, C))
    _check_bn_bwd_parts(pa, _bn_bwd_terms(g, ya, ma, ra), M, C, nparts, what + " a")
    _check_bn_bwd_parts(pb, _bn_bwd_terms(g, yb, mb, rb), M, C, nparts, what + " b")
    ca = _bn_bwd_finalize(lib, pa, ga, ma, ra, M, C, what + " a")
    cb = _bn_bwd_finalize(lib, pb, gb, mb, rb, M, C, what + " b")
    dya, dyb = _nan((B, H, W, C), tdt), _nan((B, H, W, C), tdt)
    _check(lib.acnn_bn_bwd_apply2(_p(g), _p(ya), _p(yb), _p(ca), _p(cb), _p(dya), _p(dyb), B, HW, C, code,
                                  _st()), "bn_bwd_apply2")
    torch.cuda.synchronize()
    idx = idx if idx is not None else list(range(B))
    _bn_apply_check(dya, g, ya, ca, idx, dt == "bf16", what + " apply2 a")
    _bn_apply_check(dyb, g, yb, cb, idx, dt == "bf16", what + " apply2 b")


BN_BWD2_CASES = _plan_cases("bn_bwd_reduce2", lambda op: tuple(op.shape))


@pytest.mark.parametrize("shape", BN_BWD2_CASES, ids=_ids(BN_BWD2_CASES))
def test_bn_bwd2_plan_shapes(lib, dt, shape):
    _bn_bwd2_case(lib, dt, *shape, idx=_sample(shape[0]))


@pytest.mark.parametrize("C", CG_OK_C)
def test_bn_bwd_edges(lib, dt, C):
    """Every accepted channel count, with the SE gate / pooled-descriptor term, tiny and odd maps (one
    row; fewer rows than one CTA pass) and a map whose last pass is partial."""
    for (B, H, W) in ((1, 1, 1), (3, 7, 5), (5, 13, 9)):
        for gate, addbc in ((False, False), (True, True), (True, False)):
            _bn_bwd_case(lib, dt, B, H, W, C, gate, addbc, seed=C)
        _bn_bwd2_case(lib, dt, B, H, W, C, seed=C)


@pytest.mark.parametrize("nparts", [1, 31, 32, 33, 132, 264])
@pytest.mark.parametrize("C", [8, 100, 2048])
def test_bn_bwd_finalize_nparts(lib, nparts, C):
    """Lane l of the finalize adds rows l, l+32, ...: 1 row (31 idle lanes), 31 / 32 / 33 rows (one lane
    with a second row), 132 and 264 (the reduce grids); C = 100 is not a multiple of 8."""
    parts = _rand((nparts, 2, C), torch.float32, nparts + C, 3.0, 0.5)
    gamma, mean, rstd = _bn_stats_inputs(C, C)
    _bn_bwd_finalize(lib, parts, gamma, mean, rstd, 12345, C, "bn_bwd_finalize nparts=%d C=%d" % (nparts, C))


# ---------------------------------------------------------------------------------------------------
# bn_finalize, bn_stats
# ---------------------------------------------------------------------------------------------------
def _f32(v):
    """The fp32 value the kernel receives for the Python float v."""
    return float(torch.tensor(v, dtype=torch.float32))


def _bn_finalize_case(lib, C, nparts, count, training, stats_mode, seed, what):
    mom, eps = _f32(0.997), _f32(1e-5)
    x_mean = _rand((C,), torch.float32, seed, 0.5)
    x_var = _unif((C,), seed + 1, 0.05, 3.0)
    if stats_mode == 0:
        # partial (sum, sumsq) rows consistent with the statistics above, split unevenly over the rows
        w = _unif((nparts, 1), seed + 2, 0.5, 1.5)
        w = w / w.sum()
        s = (x_mean * count)[None] * w
        q = ((x_var + x_mean ** 2) * count)[None] * w
        stats = torch.stack([s, q], 1).float().contiguous()
    else:
        stats = torch.cat([x_mean, x_var]).contiguous()
    gamma, beta = _rand((C,), torch.float32, seed + 3, 0.3, 1.0), _rand((C,), torch.float32, seed + 4, 0.3)
    mm0, mv0 = _rand((C,), torch.float32, seed + 5, 0.2), _unif((C,), seed + 6, 0.5, 2.0)
    mm, mv = mm0.clone(), mv0.clone()
    outs = [_nan((C,), torch.float32) for _ in range(4)]
    _check(lib.acnn_bn_finalize(_p(stats), nparts, stats_mode, count, _p(gamma), _p(beta), _p(mm), _p(mv),
                                mom, eps, int(training), *(_p(o) for o in outs), C, _st()), "bn_finalize")
    torch.cuda.synchronize()
    scale, shift, mean, rstd = outs
    if training:
        if stats_mode == 0:
            S = stats.double()
            m = S[:, 0].sum(0) / count
            v = (S[:, 1].sum(0) / count - m * m).clamp_min(0)
            # the kernel adds the rows in double: its only fp32 roundings are the two final stores
            tm = SC.ulp_f32(m) + 2.0 ** -45 * m.abs()
            tv = SC.ulp_f32(v) + 2.0 ** -45 * (S[:, 1].sum(0) / count).abs()
        else:
            m, v = x_mean.double(), x_var.double()
            tm, tv = torch.zeros_like(m), torch.zeros_like(v)
        SC.assert_within(mean, m, tm, what + " mean")
        unb = v * (count / max(count - 1, 1))
        tunb = 3 * U * unb + tv * (count / max(count - 1, 1))
        ref_mm = mm0.double() * mom + m * (1 - mom)
        ref_mv = mv0.double() * mom + unb * (1 - mom)
        SC.assert_within(mm, ref_mm, 4 * U * ((mm0.double() * mom).abs() + (m * (1 - mom)).abs()) +
                         tm * (1 - mom), what + " moving_mean")
        SC.assert_within(mv, ref_mv, 4 * U * ((mv0.double() * mom).abs() + (unb * (1 - mom)).abs()) +
                         tunb * (1 - mom), what + " moving_var")
    else:
        m, v, tm, tv = mm0.double(), mv0.double(), torch.zeros(C, dtype=torch.float64, device="cuda"), \
            torch.zeros(C, dtype=torch.float64, device="cuda")
        assert torch.equal(mm, mm0) and torch.equal(mv, mv0), what + ": inference updated the moving stats"
        SC.assert_within(mean, m, tm, what + " mean")
    r = 1.0 / torch.sqrt(v + eps)
    tr = 4 * U * r + 0.5 * r * (tv + U * (v + eps)) / (v + eps)      # rsqrtf: 2 ulp; var error
    SC.assert_within(rstd, r, tr, what + " rstd")
    sc = gamma.double() * r
    tsc = 2 * U * sc.abs() + gamma.double().abs() * tr
    SC.assert_within(scale, sc, tsc, what + " scale")
    sh = beta.double() - m * sc
    SC.assert_within(shift, sh, 3 * U * (beta.double().abs() + (m * sc).abs()) + m.abs() * tsc +
                     sc.abs() * tm, what + " shift")


@pytest.mark.parametrize("nparts", [1, 31, 32, 33, 132, 264])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_bn_finalize_nparts(lib, nparts, training):
    for C in (8, 100, 2048):
        _bn_finalize_case(lib, C, nparts, 256 * 56 * 56, training, 0, nparts + C,
                          "bn_finalize nparts=%d C=%d training=%d" % (nparts, C, training))
    if training:
        _bn_finalize_case(lib, 64, nparts, 5, True, 1, 3, "bn_finalize stats_mode 1")
        _bn_finalize_case(lib, 64, nparts, 1, True, 0, 4, "bn_finalize count 1 (unbiased divisor 1)")


BN_FIN_CASES = _plan_cases("bn_finalize", lambda op: (op.bn.C, op.bn.count))


@pytest.mark.parametrize("case", BN_FIN_CASES, ids=_ids(BN_FIN_CASES))
def test_bn_finalize_plan_channels(lib, case):
    C, count = case
    _bn_finalize_case(lib, C, 132, count, True, 0, C, "bn_finalize plan C=%d count=%d" % case)


@pytest.mark.parametrize("C", [8, 64])
def test_bn_stats_production(lib, dt, C):
    """acnn_bn_stats (fp32 parity mode) at M = 256 * 112^2 on exactly summable data: values offset_c
    + k/8, k in {-1, 0, 1} with sum_k = 0 per channel (the second half of the rows negates the first),
    offset_c in {0, 1/4}.  Every partial sum of either pass is a multiple of 1/64 below 2^18, so fp32
    adds it exactly in any order: the mean must be offset_c exactly and the variance the correctly
    rounded sum_k k^2 / 64 / M (one rounding: the division).  A dropped or doubled row changes either."""
    code, tdt = DTYPES[dt]
    M = 256 * 112 * 112
    k = torch.randint(-1, 2, (M // 2, C), generator=_gen(C), device="cuda").float()
    k = torch.cat([k, -k.flip(0)])
    off = (torch.arange(C, device="cuda") % 2).float() * 0.25
    x = (off + k / 8).to(tdt)
    out = _nan((2 * C,), torch.float32)
    _check(lib.acnn_bn_stats(_p(x), _p(out), M, C, code, _st()), "bn_stats")
    torch.cuda.synchronize()
    assert torch.equal(out[:C], off), "bn_stats mean"
    var = (k.double() ** 2).sum(0) / 64 / M
    SC.assert_within(out[C:], var, 0.5 * SC.ulp_f32(var), "bn_stats variance")


# ---------------------------------------------------------------------------------------------------
# selective-kernel block
# ---------------------------------------------------------------------------------------------------
def _sk_inputs(B, HW, f, tdt, seed):
    C2 = 2 * f
    t = dict(y=_rand((B, HW, C2), tdt, seed), scale=_rand((C2,), torch.float32, seed + 1, 0.5, 1.0),
             shift=_rand((C2,), torch.float32, seed + 2, 0.5), att=_unif((B, f), seed + 3),
             dv=_rand((B, HW, f), tdt, seed + 4), ds=_rand((B, f), torch.float32, seed + 5),
             mean=_rand((C2,), torch.float32, seed + 6, 0.5), rstd=_unif((C2,), seed + 7, 0.5, 2.0),
             coef=torch.cat([_rand((C2,), torch.float32, seed + 8, 0.5, 1.0),
                             _rand((C2,), torch.float32, seed + 9, 0.01),
                             _rand((C2,), torch.float32, seed + 10, 0.01)]).contiguous())
    return t


def _sk_u(t, sl=slice(None)):
    f = t["att"].shape[1]
    tt = t["y"][sl].double() * t["scale"].double() + t["shift"].double()
    return tt, tt.clamp_min(0)[..., :f], tt.clamp_min(0)[..., f:]


def _sk_grad(t, tt, sl=slice(None)):
    """g = [tt > 0] (a_h dv + ds / HW) over the 2f channels, and its magnitude."""
    HW = t["y"].shape[1]
    att = t["att"][sl].double()[:, None, :]
    a = torch.cat([att, 1 - att], -1)
    dv = t["dv"][sl].double()
    dv2 = torch.cat([dv, dv], -1)
    ds = t["ds"][sl].double()[:, None, :] / HW
    ds2 = torch.cat([ds, ds], -1)
    on = (tt > 0).double()
    return on * (a * dv2 + ds2), on * ((a * dv2).abs() + ds2.abs())


def _sk_run(lib, dt, B, HW, f, seed, idx):
    code, tdt = DTYPES[dt]
    t = _sk_inputs(B, HW, f, tdt, seed)
    bf16 = dt == "bf16"
    what = "sk %s B=%d HW=%d f=%d" % (dt, B, HW, f)
    s, dA = _nan((B, f), torch.float32), _nan((B, f), torch.float32)
    v, dy = _nan((B, HW, f), tdt), _nan((B, HW, 2 * f), tdt)
    nparts = lib.acnn_sk_bn_bwd_reduce_parts(B, HW, f)
    slabs, rows_per, rt = SC.sk_slabs(B, HW, f, 2)
    assert nparts == B * slabs
    parts = _nan((nparts, 2, 2 * f), torch.float32)
    st = _st()
    _check(lib.acnn_sk_gap(_p(t["y"]), _p(t["scale"]), _p(t["shift"]), _p(s), B, HW, f, code, st), "sk_gap")
    _check(lib.acnn_sk_combine(_p(t["y"]), _p(t["scale"]), _p(t["shift"]), _p(t["att"]), _p(v), B, HW, f,
                               code, st), "sk_combine")
    _check(lib.acnn_sk_bwd_gate(_p(t["dv"]), _p(t["y"]), _p(t["scale"]), _p(t["shift"]), _p(dA), B, HW, f,
                                code, st), "sk_bwd_gate")
    _check(lib.acnn_sk_bn_bwd_reduce(_p(t["dv"]), _p(t["y"]), _p(t["scale"]), _p(t["shift"]), _p(t["mean"]),
                                     _p(t["rstd"]), _p(t["att"]), _p(t["ds"]), _p(parts), B, HW, f, code,
                                     st), "sk_bn_bwd_reduce")
    _check(lib.acnn_sk_bn_bwd_apply(_p(t["dv"]), _p(t["y"]), _p(t["scale"]), _p(t["shift"]), _p(t["att"]),
                                    _p(t["ds"]), _p(t["coef"]), _p(dy), B, HW, f, code, st),
           "sk_bn_bwd_apply")
    torch.cuda.synchronize()
    # per-image reductions: one CTA per image, 2 rows per thread per trip of 2 * 256 / (f / 8) rows
    rpb = 256 // (f // 8)
    n_eff = 2 * -(-HW // (2 * rpb)) + rpb
    tt, u0, u1 = _sk_u(t)
    SC.assert_within(s, (u0 + u1).sum(1) / HW,
                     SC.reduction_tol((u0 + u1).sum(1) / HW, n_eff, extra_ops=4), what + " sk_gap")
    dvd = t["dv"].double()
    SC.assert_within(dA, (dvd * (u0 - u1)).sum(1),
                     SC.reduction_tol((dvd.abs() * (u0 + u1)).sum(1), n_eff, extra_ops=4),
                     what + " sk_bwd_gate")
    # partial rows: one per (image, slab) of rows_per rows; chains of 4 rows per trip + the RPB lanes
    g, gmag = _sk_grad(t, tt)
    xhat = (t["y"].double() - t["mean"].double()) * t["rstd"].double()
    pad = slabs * rows_per - HW

    def slab_sum(z):
        z = torch.cat([z, z.new_zeros(B, pad, z.shape[-1])], 1) if pad else z
        return z.view(B, slabs, rows_per, -1).sum(2).reshape(B * slabs, -1)

    n_eff = 4 * -(-rows_per // rt) + 1024 // f
    for k, (term, mag) in enumerate(((g, gmag), (g * xhat, gmag * xhat.abs()))):
        SC.assert_within(parts[:, k], slab_sum(term), SC.reduction_tol(slab_sum(mag), n_eff, extra_ops=6),
                         what + " sk_bn_bwd_reduce partial %d" % k)
    # elementwise, on the sampled images
    a = t["att"][idx].double()[:, None, :]
    _, u0s, u1s = _sk_u(t, idx)
    ref = a * u0s + (1 - a) * u1s
    SC.assert_within(v[idx], ref, SC.elementwise_tol(ref, (a * u0s).abs() + ((1 - a) * u1s).abs(), bf16, 5),
                     what + " sk_combine")
    tts, _, _ = _sk_u(t, idx)
    gs, gsmag = _sk_grad(t, tts, idx)
    k1, k2, k3 = (t["coef"].view(3, -1)[i].double() for i in range(3))
    yy = t["y"][idx].double()
    ref = k1 * gs + k2 * yy + k3
    mag = k1.abs() * gsmag + (k2 * yy).abs() + k3.abs()
    SC.assert_within(dy[idx], ref, SC.elementwise_tol(ref, mag, bf16, 6), what + " sk_bn_bwd_apply")


SK_CASES = _plan_cases("sk_gap", lambda op: (op.B, op.HW, op.f))


@pytest.mark.parametrize("case", SK_CASES, ids=_ids(SK_CASES))
def test_sk_plan_shapes(lib, dt, case):
    B, HW, f = case
    _sk_run(lib, dt, B, HW, f, seed=HW + f, idx=_sample(B))


@pytest.mark.parametrize("case", SC.SK_EDGE_SHAPES, ids=_ids(SC.SK_EDGE_SHAPES))
def test_sk_edges(lib, dt, case):
    """For each slab layout (combine / apply: ~8 CTAs per SM, reduce: 2) a shape with an empty slab,
    one whose slab runs more trips than the 3-stage ring, one whose last trip is partial."""
    B, HW, f = case
    _sk_run(lib, dt, B, HW, f, seed=B + HW + f, idx=_sample(B))


# ---------------------------------------------------------------------------------------------------
# pooling / resampling (oracle on the CPU, sampled images)
# ---------------------------------------------------------------------------------------------------
def _cpu64(t, idx):
    return t[idx].double().cpu()


def _grad_ref(fn, x64, dout64):
    """(x.grad, |.| propagated) of fn at x for the cotangent dout -- the weights of these pools are >= 0,
    so the magnitude of the adjoint sum is the adjoint of |dout|."""
    x = x64.clone().requires_grad_(True)
    y = fn(x)
    (gx,) = torch.autograd.grad(y, x, dout64)
    x2 = x64.clone().requires_grad_(True)
    (gm,) = torch.autograd.grad(fn(x2), x2, dout64.abs())
    return gx, gm


def _epilogue_ref(ref, mag, add, mask):
    if add is not None:
        ref, mag = ref + add, mag + add.abs()
    if mask is not None:
        keep = (mask > 0).double()
        ref, mag = ref * keep, mag * keep
    return ref, mag


def _blur_case(lib, dt, B, H, W, C, filt, stride, add_mask, seed, idx):
    code, tdt = DTYPES[dt]
    bf16 = dt == "bf16"
    pad = (filt - 1) // 2
    Ho, Wo = (H + 2 * pad - filt) // stride + 1, (W + 2 * pad - filt) // stride + 1
    x = _rand((B, H, W, C), tdt, seed)
    out = _nan((B, Ho, Wo, C), tdt)
    _check(lib.acnn_blurpool_fwd(_p(x), _p(out), B, H, W, C, filt, stride, code, _st()), "blurpool_fwd")
    dout = _rand((B, Ho, Wo, C), tdt, seed + 1)
    add = _rand((B, H, W, C), tdt, seed + 2) if add_mask else None
    mask = _rand((B, H, W, C), tdt, seed + 3) if add_mask else None
    dx = _nan((B, H, W, C), tdt)
    _check(lib.acnn_blurpool_bwd(_p(dout), _p(dx), _p(add), _p(mask), B, H, W, C, filt, stride, code, _st()),
           "blurpool_bwd")
    torch.cuda.synchronize()
    what = "blurpool %s %s filt=%d stride=%d" % (dt, (B, H, W, C), filt, stride)
    fn = functools.partial(tf_ops.anti_aliased_downsample, filt_size=filt, stride=stride)
    x64 = _cpu64(x, idx)
    ref = fn(x64)
    mag = fn(x64.abs())
    # the binomial weights are powers of two over integers: exact in fp32; filt^2 FMAs per output
    SC.assert_within(out[idx].cpu(), ref, SC.elementwise_tol(ref, mag, bf16, ops=filt * filt), what + " fwd")
    gx, gm = _grad_ref(fn, x64, _cpu64(dout, idx))
    gx, gm = _epilogue_ref(gx, gm, None if add is None else _cpu64(add, idx),
                           None if mask is None else _cpu64(mask, idx))
    # at most (filt + 2 * pad) ^ 2 adjoint taps per input pixel (reflection folds), then the add
    SC.assert_within(dx[idx].cpu(), gx, SC.elementwise_tol(gx, gm, bf16, ops=(2 * filt) ** 2 + 1),
                     what + " bwd")


BLUR_CASES = _plan_cases("blurpool", lambda op: (op.B, op.H, op.W, op.C, op.filt, op.stride))
BLUR_BWD = {k: v for k, v in (((op.B, op.H, op.W, op.C, op.filt, op.stride), op.add_src is not None)
                              for name in ("c3", "c5") for op in _plan(name).all_ops()
                              if op.kind == "blurpool_bwd")}


@pytest.mark.parametrize("case", BLUR_CASES, ids=_ids(BLUR_CASES))
def test_blurpool_plan_shapes(lib, dt, case):
    B, H, W, C, filt, stride = case
    _blur_case(lib, dt, B, H, W, C, filt, stride, BLUR_BWD.get(case, False), seed=H + C, idx=_sample(B))


TINY = [(1, 1), (2, 2), (3, 3), (2, 3), (7, 7), (9, 13), (13, 9), (1, 7)]


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("filt", range(1, 8))
def test_blurpool_edges(lib, dt, filt, stride):
    """filt 1-7 (filt 3 / stride 2 is the compile-time path, the rest the generic one), reflection on
    maps down to pad + 1 wide, heights that are not multiples of kBlurRows = 4, C not a multiple of 16."""
    pad = (filt - 1) // 2
    for (H, W) in TINY:
        if pad < H and pad < W and min(H, W) + 2 * pad >= filt:     # reflection defined, output not empty
            for C in (8, 24):
                _blur_case(lib, dt, 2, H, W, C, filt, stride, (H + W + C) % 2 == 0, seed=H * W + C,
                           idx=[0, 1])


def _avgpool_case(lib, dt, B, H, W, C, k, s, pad_lo, Ho, Wo, count_pad, add_mask, seed, idx):
    code, tdt = DTYPES[dt]
    bf16 = dt == "bf16"
    x = _rand((B, H, W, C), tdt, seed)
    out = _nan((B, Ho, Wo, C), tdt)
    _check(lib.acnn_avgpool_fwd(_p(x), _p(out), B, H, W, C, k, s, pad_lo, Ho, Wo, count_pad, code, _st()),
           "avgpool_fwd")
    dout = _rand((B, Ho, Wo, C), tdt, seed + 1)
    add = _rand((B, H, W, C), tdt, seed + 2) if add_mask else None
    mask = _rand((B, H, W, C), tdt, seed + 3) if add_mask else None
    dx = _nan((B, H, W, C), tdt)
    _check(lib.acnn_avgpool_bwd(_p(dout), _p(dx), _p(add), _p(mask), B, H, W, C, k, s, pad_lo, Ho, Wo,
                                count_pad, code, _st()), "avgpool_bwd")
    torch.cuda.synchronize()
    what = "avgpool %s %s k=%d s=%d pad=%d out=%s count_pad=%d" % (dt, (B, H, W, C), k, s, pad_lo, (Ho, Wo),
                                                                    count_pad)
    fn = functools.partial(SC.avgpool_ref, k=k, s=s, pad_lo=pad_lo, Ho=Ho, Wo=Wo, count_pad=count_pad)
    x64 = _cpu64(x, idx)
    ref, mag = fn(x64), fn(x64.abs())
    SC.assert_within(out[idx].cpu(), ref, SC.elementwise_tol(ref, mag, bf16, ops=k * k + 2), what + " fwd")
    gx, gm = _grad_ref(fn, x64, _cpu64(dout, idx))
    gx, gm = _epilogue_ref(gx, gm, None if add is None else _cpu64(add, idx),
                           None if mask is None else _cpu64(mask, idx))
    SC.assert_within(dx[idx].cpu(), gx, SC.elementwise_tol(gx, gm, bf16, ops=k * k + 4), what + " bwd")


AVG_CASES = _plan_cases("avgpool", lambda op: (op.B, op.H, op.W, op.C, op.k, op.stride, op.pad_lo, op.Ho,
                                               op.Wo, op.count_pad))
AVG_BWD = {k: v for k, v in (((op.B, op.H, op.W, op.C, op.k, op.stride, op.pad_lo, op.Ho, op.Wo,
                               op.count_pad), op.add_src is not None or op.mask_src is not None)
                             for name in ("c3", "c5") for op in _plan(name).all_ops()
                             if op.kind == "avgpool_bwd")}


@pytest.mark.parametrize("case", AVG_CASES, ids=_ids(AVG_CASES))
def test_avgpool_plan_shapes(lib, dt, case):
    _avgpool_case(lib, dt, *case, AVG_BWD.get(case, False), seed=case[1] + case[3], idx=_sample(case[0]))


@pytest.mark.parametrize("k,s", [(1, 1), (2, 1), (2, 2), (3, 1), (3, 2)])
def test_avgpool_edges(lib, dt, k, s):
    """Tiny and odd maps, both divisors: SAME geometry (pad after) and the 'fixed padding' one (pad_lo
    = (k - 1) // 2 before), heights that are not multiples of kPoolRows = 4."""
    for (H, W) in TINY:
        for count_pad in (0, 1):
            Ho, Wo = -(-H // s), -(-W // s)
            lo = max((Ho - 1) * s + k - H, 0) // 2
            _avgpool_case(lib, dt, 2, H, W, 8, k, s, lo, Ho, Wo, count_pad, True, seed=H + W, idx=[0, 1])
            lo = (k - 1) // 2
            Ho, Wo = (H + k - 1 - k) // s + 1, (W + k - 1 - k) // s + 1
            _avgpool_case(lib, dt, 2, H, W, 24, k, s, lo, Ho, Wo, count_pad, False, seed=H * W, idx=[0, 1])


def _maxpool_case(lib, dt, B, H, W, C, k, s, pad_lo, Ho, Wo, add_mask, seed, idx, coarse=False):
    code, tdt = DTYPES[dt]
    bf16 = dt == "bf16"
    x = _rand((B, H, W, C), tdt, seed)
    if coarse:     # many ties: the first-maximum rule decides
        x = (x * 2).round().to(tdt)
    out = _nan((B, Ho, Wo, C), tdt)
    _check(lib.acnn_maxpool_fwd(_p(x), _p(out), B, H, W, C, k, s, pad_lo, Ho, Wo, code, _st()), "maxpool_fwd")
    dout = _rand((B, Ho, Wo, C), tdt, seed + 1)
    add = _rand((B, H, W, C), tdt, seed + 2) if add_mask else None
    mask = _rand((B, H, W, C), tdt, seed + 3) if add_mask else None
    dx = _nan((B, H, W, C), tdt)
    _check(lib.acnn_maxpool_bwd(_p(dout), _p(x), _p(dx), _p(add), _p(mask), B, H, W, C, k, s, pad_lo, Ho, Wo,
                                code, _st()), "maxpool_bwd")
    torch.cuda.synchronize()
    what = "maxpool %s %s k=%d s=%d pad=%d out=%s" % (dt, (B, H, W, C), k, s, pad_lo, (Ho, Wo))
    x64 = _cpu64(x, idx)
    ref, gx = SC.maxpool_ref(x64, k, s, pad_lo, Ho, Wo, _cpu64(dout, idx))
    assert torch.equal(out[idx].cpu().double(), ref), what + " fwd (a max is exact)"
    _, gm = SC.maxpool_ref(x64, k, s, pad_lo, Ho, Wo, _cpu64(dout, idx).abs())
    gx, gm = _epilogue_ref(gx, gm, None if add is None else _cpu64(add, idx),
                           None if mask is None else _cpu64(mask, idx))
    SC.assert_within(dx[idx].cpu(), gx, SC.elementwise_tol(gx, gm, bf16, ops=k * k + 2), what + " bwd")


def test_maxpool_production(lib, dt):
    """The resnet_version=1 stem pool (TF SAME 3x3 / 2 on 112^2: pad 0 before, 1 after) at B = 256,
    taken from that plan."""
    ops = [op for op in _plan("c1").all_ops() if op.kind == "maxpool"]
    assert ops
    op = ops[0]
    _maxpool_case(lib, dt, op.B, op.H, op.W, op.C, op.k, op.stride, op.pad_lo, op.Ho, op.Wo, False, 5,
                  _sample(op.B))


@pytest.mark.parametrize("k,s", [(1, 1), (2, 2), (3, 1), (3, 2)])
def test_maxpool_edges(lib, dt, k, s):
    for (H, W) in TINY:
        Ho, Wo = -(-H // s), -(-W // s)
        lo = max((Ho - 1) * s + k - H, 0) // 2
        _maxpool_case(lib, dt, 2, H, W, 8, k, s, lo, Ho, Wo, True, seed=H + W, idx=[0, 1], coarse=True)
        _maxpool_case(lib, dt, 2, H, W, 24, k, s, 0, Ho, Wo, False, seed=H * W, idx=[0, 1])


def _resample_case(lib, dt, B, H, W, C, add_mask, seed, idx):
    """upsample2x_bwd (dx [B,H,W,C] from dout [B,2H,2W,C]) and zero_insert2x into [B,2H+1,2W+1,C] (and
    into [B,2H,2W,C]) from dy [B,H,W,C]."""
    code, tdt = DTYPES[dt]
    bf16 = dt == "bf16"
    dout = _rand((B, 2 * H, 2 * W, C), tdt, seed)
    add = _rand((B, H, W, C), tdt, seed + 1) if add_mask else None
    mask = _rand((B, H, W, C), tdt, seed + 2) if add_mask else None
    dx = _nan((B, H, W, C), tdt)
    _check(lib.acnn_upsample2x_bwd(_p(dout), _p(dx), _p(add), _p(mask), B, H, W, C, code, _st()),
           "upsample2x_bwd")
    outs = []
    for (Hz, Wz) in ((2 * H, 2 * W), (2 * H + 1, 2 * W + 1)):
        z = _nan((B, Hz, Wz, C), tdt)
        _check(lib.acnn_zero_insert2x(_p(dout[:, :H, :W].contiguous()), _p(z), B, H, W, Hz, Wz, C, code,
                                      _st()), "zero_insert2x")
        outs.append(z)
    comb = _nan((B, H, W, C), tdt)
    _check(lib.acnn_grad_combine(_p(dx), _p(add), _p(mask), _p(comb), B * H * W * C, code, _st()),
           "grad_combine")
    torch.cuda.synchronize()
    what = "resample %s %s" % (dt, (B, H, W, C))
    gx, gm = _grad_ref(tf_ops.upsample2x, torch.zeros(len(idx), H, W, C, dtype=torch.float64),
                       _cpu64(dout, idx))
    gx, gm = _epilogue_ref(gx, gm, None if add is None else _cpu64(add, idx),
                           None if mask is None else _cpu64(mask, idx))
    SC.assert_within(dx[idx].cpu(), gx, SC.elementwise_tol(gx, gm, bf16, ops=5), what + " upsample2x_bwd")
    dy = dout[:, :H, :W]
    for z in outs:
        ref = torch.zeros_like(z)
        ref[:, 0:2 * H:2, 0:2 * W:2] = dy
        assert torch.equal(z, ref), what + " zero_insert2x %s" % (tuple(z.shape),)
    c, cm = _epilogue_ref(dx.double(), dx.double().abs(), None if add is None else add.double(),
                          None if mask is None else mask.double())
    SC.assert_within(comb, c, SC.elementwise_tol(c, cm, bf16, ops=1), what + " grad_combine")


RS_CASES = _plan_cases("upsample2x_bwd", lambda op: (op.B, op.H, op.W, op.C, op.add_src is not None))
ZI_CASES = _plan_cases("zero_insert", lambda op: (op.B, op.Ho, op.Wo, op.H, op.W, op.C))


@pytest.mark.parametrize("case", RS_CASES, ids=_ids(RS_CASES))
def test_resample_plan_shapes(lib, dt, case):
    B, H, W, C, am = case
    _resample_case(lib, dt, B, H, W, C, am, seed=H + C, idx=_sample(B))
    # the stride-2 dgrad inputs of the plan: zero_insert2x at its own (Ho, Wo) -> (H, W)
    code, tdt = DTYPES[dt]
    for (Bz, Ho, Wo, Hz, Wz, Cz) in ZI_CASES:
        dy = _rand((Bz, Ho, Wo, Cz), tdt, 3)
        z = _nan((Bz, Hz, Wz, Cz), tdt)
        _check(lib.acnn_zero_insert2x(_p(dy), _p(z), Bz, Ho, Wo, Hz, Wz, Cz, code, _st()), "zero_insert2x")
        torch.cuda.synchronize()
        ref = torch.zeros_like(z)
        ref[:, 0:2 * Ho:2, 0:2 * Wo:2] = dy[:, :(Hz + 1) // 2, :(Wz + 1) // 2]
        assert torch.equal(z, ref), "zero_insert2x plan %s" % ((Bz, Ho, Wo, Hz, Wz, Cz),)


def test_resample_edges(lib, dt):
    with _grid_cap(lib, 132):
        for (H, W) in TINY:
            for C in (8, 24):
                _resample_case(lib, dt, 3, H, W, C, (H + C) % 2 == 0, seed=H + W + C, idx=[0, 1, 2])


# ---------------------------------------------------------------------------------------------------
# global pools
# ---------------------------------------------------------------------------------------------------
def _gap_case(lib, dt, B, HW, C, seed, idx):
    code, tdt = DTYPES[dt]
    bf16 = dt == "bf16"
    x = _rand((B, HW, C), tdt, seed, 1.0, 0.5)
    pooled = _nan((B, C), tdt)
    _check(lib.acnn_gap_fwd(_p(x), _p(pooled), B, HW, C, code, _st()), "gap_fwd")
    dp = _rand((B, C), tdt, seed + 1)
    mask = _rand((B, HW, C), tdt, seed + 2)
    dx = _nan((B, HW, C), tdt)
    _check(lib.acnn_gap_bwd(_p(dp), _p(mask), _p(dx), B, HW, C, code, _st()), "gap_bwd")
    torch.cuda.synchronize()
    what = "gap %s B=%d HW=%d C=%d" % (dt, B, HW, C)
    x64 = x.double()
    ref = tf_ops.global_avg_pool(x64[:, :, None, :])
    # gap_fwd: C >= 1024 splits the channels over gridDim.y in blocks of 512
    fl = C // (C // 512) if (C >= 1024 and C % 512 == 0) else C
    cgs = min(fl // 8, 256)
    rpb = 256 // cgs
    n_eff = -(-HW // rpb) + rpb
    tol = SC.reduction_tol(x64.abs().mean(1), n_eff, extra_ops=2)
    if bf16:
        tol = tol + SC.ulp_bf16(ref)
    SC.assert_within(pooled, ref, tol, what + " fwd")
    r = dp[idx].double()[:, None, :] / HW * (mask[idx] > 0).double()
    SC.assert_within(dx[idx], r, SC.elementwise_tol(r, r.abs(), bf16, ops=2), what + " bwd")


GAP_CASES = _plan_cases("gap", lambda op: (op.B, op.HW, op.C))


@pytest.mark.parametrize("case", GAP_CASES, ids=_ids(GAP_CASES))
def test_gap_plan_shapes(lib, dt, case):
    _gap_case(lib, dt, *case, seed=7, idx=_sample(case[0]))


@pytest.mark.parametrize("C", CG_OK_C)
def test_gap_edges(lib, dt, C):
    for HW in (1, 2, 7, 49, 197):
        _gap_case(lib, dt, 3, HW, C, seed=HW + C, idx=[0, 1, 2])


# ---------------------------------------------------------------------------------------------------
# head: GeM, DropBlock, softmax cross-entropy (+ KD), input packing / mixup
# ---------------------------------------------------------------------------------------------------
def _gem_case(lib, dt, B, HW, C, seed, idx):
    code, tdt = DTYPES[dt]
    bf16 = dt == "bf16"
    x = _rand((B, HW, C), tdt, seed).clamp_min(0).to(tdt)       # a ReLU output: zeros are clipped
    pooled, ssum = _nan((B, C), tdt), _nan((B, C), torch.float32)
    _check(lib.acnn_gem_fwd(_p(x), _p(pooled), _p(ssum), B, HW, C, code, _st()), "gem_fwd")
    dp = _rand((B, C), tdt, seed + 1)
    dx = _nan((B, HW, C), tdt)
    _check(lib.acnn_gem_bwd(_p(dp), _p(ssum), _p(x), _p(dx), B, HW, C, code, _st()), "gem_bwd")
    torch.cuda.synchronize()
    what = "gem %s B=%d HW=%d C=%d" % (dt, B, HW, C)
    x64 = x.double()
    t3 = x64.clamp(1e-6, 1e12) ** 3
    S = t3.sum(1)
    cgs = min(C // 8, 256)
    rpb = 256 // cgs
    tS = SC.reduction_tol(S, -(-HW // rpb) + rpb, extra_ops=2)
    SC.assert_within(ssum, S, tS, what + " S")
    ref = tf_ops.generalized_mean_pooling(x64[:, :, None, :])
    relS = tS / S
    tol = (8 * U + relS / 3) * ref.abs() + (SC.ulp_bf16(ref) if bf16 else 0)
    SC.assert_within(pooled, ref, tol, what + " pooled")
    xs = _cpu64(x, idx)[:, :, None, :]
    gx, _ = _grad_ref(tf_ops.generalized_mean_pooling, xs, _cpu64(dp, idx))
    gx = gx[:, :, 0, :]
    # dp * N^(-1/3) * x^2 / cbrt(S)^2: ~10 roundings (powf, cbrtf), and the fp32 S the kernel is given
    tol = (10 * U + 2 * relS[idx].cpu()[:, None, :] / 3) * gx.abs()
    tol = tol + (SC.ulp_bf16(gx) if bf16 else 0)
    SC.assert_within(dx[idx].cpu(), gx, tol, what + " bwd")


def test_gem_production(lib, dt):
    """GeM at the final feature map of the c3 plan (B = 256, 7 x 7 x 2048)."""
    (B, HW, C), = GAP_CASES[:1]
    _gem_case(lib, dt, B, HW, C, seed=3, idx=_sample(B))


@pytest.mark.parametrize("C", CG_OK_C + [4096])
def test_gem_edges(lib, dt, C):
    with _grid_cap(lib, 132):
        for HW in (1, 7, 50):
            _gem_case(lib, dt, 3, HW, C, seed=HW + C, idx=[0, 1, 2])


def _dropblock_case(lib, dt, B, HW, C, relu, seed, idx):
    code, tdt = DTYPES[dt]
    H = W = int(round(HW ** 0.5))
    assert H * W == HW
    bs = min(7, H - (1 - H % 2))
    u = torch.rand(1, H - bs + 1, W - bs + 1, C, generator=torch.Generator().manual_seed(seed),
                   dtype=torch.float64)
    keep64, factor = tf_ops.dropblock_keep_mask(u, 0.8, bs, 1.0, H, W)
    keep = keep64.float().cuda().contiguous()
    scale = torch.tensor([float(factor)], dtype=torch.float32, device="cuda")
    x = _rand((B, H, W, C), tdt, seed)
    out = _nan((B, H, W, C), tdt)
    _check(lib.acnn_dropblock_apply(_p(x), _p(keep), _p(scale), int(relu), _p(out), B, HW, C, code, _st()),
           "dropblock_apply")
    torch.cuda.synchronize()
    ref = x[idx].double() * keep.double() * scale.double()
    if relu:
        ref = ref.clamp_min(0)
    SC.assert_within(out[idx], ref, SC.elementwise_tol(ref, ref.abs(), dt == "bf16", ops=2),
                     "dropblock_apply %s %s relu=%d" % (dt, (B, HW, C), relu))


DB_CASES = _plan_cases("dropblock_apply", lambda op: (op.B, op.HW, op.C, bool(op.relu)),
                       plans=(("c3", (("use_dropblock", True),)),))


@pytest.mark.parametrize("case", DB_CASES, ids=_ids(DB_CASES))
def test_dropblock_plan_shapes(lib, dt, case):
    _dropblock_case(lib, dt, *case, seed=case[2], idx=_sample(case[0]))


def test_dropblock_edges(lib, dt):
    with _grid_cap(lib, 132):
        for (HW, C) in ((1, 8), (9, 24), (49, 8), (169, 2048)):
            for relu in (False, True):
                _dropblock_case(lib, dt, 5, HW, C, relu, seed=HW + C, idx=list(range(5)))


def _softmax_case(lib, dt, B, NC, ld, kd, seed):
    code, tdt = DTYPES[dt]
    bf16 = dt == "bf16"
    ls, gs, T = _f32(0.1), 0.75, 2.0
    logits = torch.full((B, ld), float("nan"), device="cuda")        # columns >= NC must not be read
    logits[:, :NC] = _rand((B, NC), torch.float32, seed, 3.0)
    lab1 = torch.randint(0, NC, (B,), generator=_gen(seed + 1), device="cuda")
    lab2 = torch.randint(0, NC, (B,), generator=_gen(seed + 2), device="cuda")
    lam = _unif((B, 1), seed + 3)
    y = (lam * F.one_hot(lab1, NC) + (1 - lam) * F.one_hot(lab2, NC)).float()
    teacher = torch.softmax(_rand((B, NC), torch.float32, seed + 4, 3.0) / T, 1).contiguous() if kd else None
    loss = torch.zeros(3, device="cuda")
    dl = _nan((B, ld), tdt)
    dbias0 = _rand((NC,), torch.float32, seed + 5, 0.1)
    dbias = dbias0.clone()
    work = _nan((2 * ((B + 31) // 32 * 32) + B * ld,), torch.float32)
    _check(lib.acnn_softmax_ce(_p(logits), _p(y), _p(teacher), T, B, NC, ld, ls, gs, _p(loss), _p(dl),
                               _p(dbias), _p(work), code, _st()), "softmax_ce")
    torch.cuda.synchronize()
    what = "softmax_ce %s B=%d NC=%d ld=%d kd=%d" % (dt, B, NC, ld, kd)
    l64 = logits[:, :NC].double().cpu().requires_grad_(True)
    y64 = y.double().cpu()
    ce = tf_ops.softmax_cross_entropy(l64, y64, ls)
    total = ce
    # error model (all float64, per row b): lse = mx + log(sum exp) from chains of <= 4 + 5 + 8 terms
    # plus 2-ulp exp / log: |err lse| <= 20u (1 + |lse|); the row loss (lse*sy - syl)/B adds 25u of its
    # terms; the rows are then added in order (B adds)
    yp = y64 * (1 - ls) + ls / NC
    lse = torch.logsumexp(l64.detach(), 1)
    e_lse = 20 * U * (1 + lse.abs())
    rows = (lse * yp.sum(1) - (yp * l64.detach()).sum(1)) / B
    t_rows = (e_lse * yp.sum(1) + 25 * U * (lse.abs() * yp.sum(1) + (yp * l64.detach()).abs().sum(1))) / B
    tl = t_rows.sum() + (B + 1) * U * rows.abs().sum()
    SC.assert_within(loss[0:1].cpu(), ce.detach().view(1), tl.view(1), what + " loss")
    p = torch.softmax(l64.detach(), 1)
    # g = (exp(l - lse) * sy - y') * (gs / B): the error of lse and of the exp argument, relative to
    # p * sy, plus ~6 roundings of y' = y * (1 - ls) + ls / NC, of the difference and of the scale
    tg = gs / B * (p * yp.sum(1, keepdim=True) * (e_lse[:, None] + U * (l64.detach() - lse[:, None]).abs()
                                                   + 26 * U) + 6 * U * yp)
    if kd:
        t64 = teacher.double().cpu()
        kl = tf_ops.kd_loss(l64, t64, T)
        total = total + kl
        lse_t = torch.logsumexp(l64.detach() / T, 1)
        e_t = 20 * U * (1 + lse_t.abs())
        rows_t = T * T * (lse_t * t64.sum(1) - (t64 * l64.detach() / T).sum(1)) / B
        t_rows_t = T * T * (e_t * t64.sum(1) + 25 * U * (lse_t.abs() * t64.sum(1) +
                                                         (t64 * l64.detach() / T).abs().sum(1))) / B
        SC.assert_within(loss[2:3].cpu(), kl.detach().view(1),
                         (t_rows_t.sum() + (B + 1) * U * rows_t.abs().sum()).view(1), what + " kd loss")
        pt = torch.softmax(l64.detach() / T, 1)
        tg = tg + T * gs / B * (pt * t64.sum(1, keepdim=True) *
                                (e_t[:, None] + U * (l64.detach() / T - lse_t[:, None]).abs() + 26 * U) +
                                6 * U * t64)
    (g,) = torch.autograd.grad(total * gs, l64)
    tol = tg + (SC.ulp_bf16(g) if bf16 else 0)
    got = dl.cpu()
    SC.assert_within(got[:, :NC], g, tol, what + " dlogits")
    assert bool((got[:, NC:] == 0).all()), what + ": padding columns of dlogits not zeroed"
    ref_b = dbias0.double().cpu() + g.sum(0)
    tb = tg.sum(0) + (B + 1) * U * (g.abs().sum(0) + dbias0.double().cpu().abs())
    SC.assert_within(dbias.cpu(), ref_b, tb, what + " dbias")


SM_CASES = _plan_cases("softmax_ce", lambda op: (op.B, op.NC, op.ld))


@pytest.mark.parametrize("kd", [False, True], ids=["ce", "ce_kd"])
@pytest.mark.parametrize("case", SM_CASES + [(512, 1001, 1024), (1, 1001, 1024), (33, 10, 17)],
                         ids=_ids(SM_CASES + [(512, 1001, 1024), (1, 1001, 1024), (33, 10, 17)]))
def test_softmax_ce(lib, dt, case, kd):
    _softmax_case(lib, dt, *case, kd, seed=case[0] + case[1])


def _space_to_depth_ref(x, wlo, whi):
    B, H, W, _ = x.shape
    t = x.reshape(B, H // 2, 2, W // 2, 2, 3).permute(0, 1, 3, 2, 4, 5)
    t = F.pad(t, (0, 1)).reshape(B, H // 2, W // 2, 16)
    return F.pad(t, (0, 0, wlo, whi))


PACK_CASES = _plan_cases("pack_input", lambda op: (op.Bin, op.H, op.W, tuple(op.wpad)))


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("case", PACK_CASES, ids=_ids(PACK_CASES))
def test_pack_input_plan(lib, dt, case, mode):
    """acnn_pack_input / acnn_mix_labels at the plan's input (512 images of 224^2 before mixup type 1;
    type 2 keeps the 512)."""
    code, tdt = DTYPES[dt]
    Bin, H, W, (wlo, whi) = case
    half = Bin // 2
    B = half if mode == 1 else Bin
    imgs = (_rand((Bin, H, W, 3), torch.float32, 1, 64.0)).clamp(-124, 152)
    lam1, lam2 = _unif((half,), 2), _unif((half,), 3)
    labels = torch.randint(0, 1001, (Bin,), generator=_gen(4), device="cuda", dtype=torch.int32)
    out = _nan((B, H // 2, W // 2 + wlo + whi, 16), tdt)
    _check(lib.acnn_pack_input(_p(imgs), _p(lam1), _p(lam2), mode, _p(out), Bin, H, W, wlo, whi, code, _st()),
           "pack_input")
    ys = _nan((B, 1001), torch.float32)
    _check(lib.acnn_mix_labels(_p(labels), _p(lam1), _p(lam2), mode, _p(ys), Bin, 1001, _st()), "mix_labels")
    torch.cuda.synchronize()
    onehot = F.one_hot(labels.long(), 1001).double()
    mx, my = tf_ops.mixup(imgs.double(), onehot, lam1.double(), lam2.double(), keep_batch_size=mode == 2)
    ma, _ = tf_ops.mixup(imgs.double().abs(), onehot, lam1.double(), lam2.double(), keep_batch_size=mode == 2)
    idx = _sample(B)
    ref = _space_to_depth_ref(mx[idx], wlo, whi)
    mag = _space_to_depth_ref(ma[idx], wlo, whi)
    what = "pack_input %s mode %d %s" % (dt, mode, case)
    SC.assert_within(out[idx], ref, SC.elementwise_tol(ref, mag, dt == "bf16", ops=4), what)
    SC.assert_within(ys, my, SC.elementwise_tol(my, torch.ones_like(my), False, ops=3), what + " labels")


# ---------------------------------------------------------------------------------------------------
# optimizer
# ---------------------------------------------------------------------------------------------------
def _sgd_ref(w, grad, acc, flags, hp):
    """float64 step (tf_ops.momentum_step on g = grad*gs + wd*w where decayed) and its tolerances:
    acc' = fma(m, acc, fma(wd, w, grad*gs)) (3 roundings); w' = fma(-lr, acc', w) (1 rounding + lr times
    the error of acc').  L2: 0.5 * wd * sum of w^2 over the decayed elements (tf.nn.l2_loss restated in
    float64: tf_ops.l2_loss rounds to fp32)."""
    lr, mom, wd, gs = (float(v) for v in hp.cpu())
    dec = flags.repeat_interleave(256)[:w.numel()].bool()
    w64, a64 = w.double(), acc.double()
    g = grad.double() * gs + torch.where(dec, wd * w64, torch.zeros_like(w64))
    w1, a1 = tf_ops.momentum_step(w64, a64, g, lr, mom)
    ta = 3 * U * ((mom * a64).abs() + (grad.double() * gs).abs() + torch.where(dec, (wd * w64).abs(), 0))
    tw = 2 * U * (w64.abs() + (lr * a1).abs()) + lr * ta
    l2 = 0.5 * wd * (w64[dec] ** 2).sum()
    return w1, a1, tw, ta, l2


def _sgd_l2_tol(n, l2):
    """Chain of the L2 sum: 4 elements per float4 per trip of a <= 1056-CTA grid of 256 threads, the 5
    warp shuffles, the 8 warp sums, the thread sums of the last CTA (ceil(grid / 256)) and its 256
    thread sums in order; then 0.5 * wd * tot and the add (3 roundings)."""
    grid = min(max(-(-(n // 4) // 256), 1), 132 * 8)
    trips = -(-(n // 4) // (grid * 256))
    return (4 * trips + 5 + 8 + -(-grid // 256) + 256 + 3) * U * abs(l2)


def _sgd_call(lib, w, grad, acc, flags, hp, l2acc, scratch):
    _check(lib.acnn_sgd_momentum(_p(w), _p(grad), _p(acc), w.numel(), _p(flags), _p(hp), _p(l2acc),
                                 _p(scratch), _st()), "sgd_momentum")


def _sgd_check(lib, n, flags, seed, scratch, what, steps=2):
    w = _rand((n,), torch.float32, seed, 0.05)
    grad = _rand((n,), torch.float32, seed + 1, 0.01)
    acc = _rand((n,), torch.float32, seed + 2, 0.01)
    hp = torch.tensor([0.1, 0.9, 1e-4, 0.5], device="cuda")
    for step in range(steps):            # consecutive calls: the arrival counter reset itself
        w1, a1, tw, ta, l2 = _sgd_ref(w, grad, acc, flags, hp)
        l2acc = torch.zeros(1, device="cuda")
        _sgd_call(lib, w, grad, acc, flags, hp, l2acc, scratch)
        torch.cuda.synchronize()
        SC.assert_within(acc, a1, ta, "%s step %d momentum" % (what, step))
        SC.assert_within(w, w1, tw, "%s step %d weights" % (what, step))
        SC.assert_within(l2acc.double(), l2.view(1), torch.tensor([_sgd_l2_tol(n, float(l2))], device="cuda"),
                         "%s step %d l2" % (what, step))
    return w, grad, acc, hp


def _plan_decay_flags(plan):
    flags = torch.zeros(max(plan.param_elems // 256, 1), dtype=torch.uint8)
    for p in plan.params.values():
        if p.decay:
            flags[p.offset // 256:(p.offset + p.size + 255) // 256] = 1
    return flags.cuda()


def test_sgd_c3_parameters(lib):
    """The c3 parameter buffer (every trainable, 256-aligned) with its weight-decay flags: two
    consecutive steps, then the same step captured in a CUDA graph and replayed (bit-identical to the
    eager call, L2 term included: the arrival counter of the last-CTA sum is back to zero each time)."""
    plan = _plan("c3")
    n = plan.param_elems
    flags = _plan_decay_flags(plan)
    assert 0 < int(flags.sum()) < flags.numel()
    scratch = torch.zeros(lib.acnn_sgd_scratch_floats(), device="cuda")
    w, grad, acc, hp = _sgd_check(lib, n, flags, 5, scratch, "sgd c3")
    w0, a0 = w.clone(), acc.clone()
    l2e = torch.zeros(1, device="cuda")
    _sgd_call(lib, w, grad, acc, flags, hp, l2e, scratch)
    we, ae = w.clone(), acc.clone()
    l2g = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            w.copy_(w0)
            acc.copy_(a0)
            l2g.zero_()
            _sgd_call(lib, w, grad, acc, flags, hp, l2g, scratch)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(w, we) and torch.equal(acc, ae) and torch.equal(l2g, l2e), "graph replay"


def test_sgd_edges(lib):
    """n = 256 (one CTA, one float4 per thread of a quarter of it); flags alternating at the 256-float
    granularity; and a small call after a large one with the SAME scratch (the counter must not sit
    where the large call left a partial sum)."""
    scratch = torch.zeros(lib.acnn_sgd_scratch_floats(), device="cuda")
    _sgd_check(lib, 256, torch.ones(1, dtype=torch.uint8, device="cuda"), 1, scratch, "sgd n=256")
    n = 256 * 37
    alt = (torch.arange(37, device="cuda") % 2).to(torch.uint8)
    _sgd_check(lib, n, alt, 2, scratch, "sgd alternating flags")
    _sgd_check(lib, 256 * 132 * 40, torch.ones(132 * 40, dtype=torch.uint8, device="cuda"), 3, scratch,
               "sgd large grid")
    _sgd_check(lib, 256 * 3, torch.ones(3, dtype=torch.uint8, device="cuda"), 4, scratch,
               "sgd small grid after a large one")
    _sgd_check(lib, 256 * 37, alt, 6, scratch, "sgd alternating flags again")


# ---------------------------------------------------------------------------------------------------
# launch independence: grid cap, repeats / graph replay, PDL
# ---------------------------------------------------------------------------------------------------
def _grid_stride_calls(lib, tdt, code, seed=0):
    """Every grid-stride kernel on inputs big enough for several trips at a cap of 132 CTAs (and one
    trip at the default cap): returns a function that runs them all and returns their outputs."""
    B, H, W, C = 16, 56, 56, 64
    sh = (B, H, W, C)
    HW = H * W
    t = _bn_act_inputs(B, H, W, C, 1, True, tdt, seed)
    b2 = _rand(sh, tdt, seed + 10)
    b3 = _rand((B, H // 2, W // 2, C), tdt, seed + 11)
    coef = _rand((3, C), torch.float32, seed + 12, 0.5)
    gate = _unif((B, C), seed + 13)
    addbc = _rand((B, C), torch.float32, seed + 14, 0.1)
    add, mask = _rand(sh, tdt, seed + 15), _rand(sh, tdt, seed + 16)
    half = _rand((B, H // 2, W // 2, C), tdt, seed + 17)
    dp = _rand((B, C), tdt, seed + 18)
    keep = (_unif((HW, C), seed + 19) > 0.2).float()
    scale = torch.tensor([1.25], device="cuda")
    ssum = _unif((B, C), seed + 20, 1.0, 100.0)
    xpos = t["a"].clamp_min(0).to(tdt)
    f32 = _rand((B * HW * C,), torch.float32, seed + 21)
    imgs = _rand((8, 112, 112, 3), torch.float32, seed + 22, 50.0)
    lam = _unif((4,), seed + 23)

    def run():
        outs = []

        def o(shape, dtype=tdt):
            outs.append(_nan(shape, dtype))
            return _p(outs[-1])

        st = _st()
        for b_mode, b in ((0, None), (1, t["b"]), (2, b2), (3, b3)):
            for gate_ in (None, t["gate"]):
                _check(lib.acnn_bn_act(_p(t["a"]), _p(t["sa"]), _p(t["ha"]), _p(b), _p(t["sb"]), _p(t["hb"]),
                                       b_mode, _p(gate_), 1, o(sh), B, H, W, C, code, st), "bn_act")
        _check(lib.acnn_bn_bwd_apply(_p(t["a"]), _p(b2), _p(coef), _p(gate), _p(addbc), o(sh), B, HW, C, code,
                                     st), "bn_bwd_apply")
        _check(lib.acnn_bn_bwd_apply2(_p(t["a"]), _p(b2), _p(add), _p(coef), _p(coef), o(sh), o(sh), B, HW, C,
                                      code, st), "bn_bwd_apply2")
        _check(lib.acnn_maxpool_fwd(_p(t["a"]), o((B, H // 2, W // 2, C)), B, H, W, C, 3, 2, 0, H // 2, W // 2,
                                    code, st), "maxpool_fwd")
        _check(lib.acnn_maxpool_bwd(_p(half), _p(t["a"]), o(sh), _p(add), _p(mask), B, H, W, C, 3, 2, 0, H // 2,
                                    W // 2, code, st), "maxpool_bwd")
        _check(lib.acnn_gap_bwd(_p(dp), _p(mask), o(sh), B, HW, C, code, st), "gap_bwd")
        _check(lib.acnn_grad_combine(_p(t["a"]), _p(add), _p(mask), o(sh), B * HW * C, code, st), "grad_combine")
        _check(lib.acnn_zero_insert2x(_p(half), o(sh), B, H // 2, W // 2, H, W, C, code, st), "zero_insert2x")
        _check(lib.acnn_upsample2x_bwd(_p(t["a"]), o((B, H // 2, W // 2, C)), _p(half), _p(half), B, H // 2,
                                       W // 2, C, code, st), "upsample2x_bwd")
        _check(lib.acnn_dropblock_apply(_p(t["a"]), _p(keep), _p(scale), 1, o(sh), B, HW, C, code, st),
               "dropblock_apply")
        _check(lib.acnn_gem_bwd(_p(dp), _p(ssum), _p(xpos), o(sh), B, HW, C, code, st), "gem_bwd")
        _check(lib.acnn_split3(_p(f32), o((3 * f32.numel(),), torch.bfloat16), f32.numel(), st), "split3")
        _check(lib.acnn_pack_input(_p(imgs), _p(lam), _p(lam), 2, o((8, 56, 59, 16)), 8, 112, 112, 2, 1, code,
                                   st), "pack_input")
        return outs
    return run


def test_grid_cap_bit_identical(lib, dt):
    code, tdt = DTYPES[dt]
    run = _grid_stride_calls(lib, tdt, code)
    results = {}
    for cap in (132, 264, 0, 65535):
        with _grid_cap(lib, cap):
            results[cap] = run()
        torch.cuda.synchronize()
    names = ["bn_act %d/%d" % (m, g) for m in range(4) for g in range(2)] + [
        "bn_bwd_apply", "bn_bwd_apply2 a", "bn_bwd_apply2 b", "maxpool_fwd", "maxpool_bwd", "gap_bwd",
        "grad_combine", "zero_insert2x", "upsample2x_bwd", "dropblock_apply", "gem_bwd", "split3",
        "pack_input"]
    assert len(names) == len(results[0])
    for cap in (132, 264, 65535):
        for name, a, b in zip(names, results[0], results[cap]):
            assert not torch.isnan(a.float()).any(), "%s: element not written" % name
            assert torch.equal(a, b), "%s differs at grid cap %d" % (name, cap)


def test_reductions_repeat_and_graph_replay_bit_identical(lib, dt):
    """Every reduction kernel (partial rows, finalizes, per-image sums, the loss and the SGD L2 sum) gives
    the same bits on repeated eager calls and on replays of a captured CUDA graph."""
    code, tdt = DTYPES[dt]
    B, H, W, C = 32, 28, 28, 128
    HW, f = H * W, 64
    g, ya, yb = (_rand((B, H, W, C), tdt, s) for s in (1, 2, 3))
    gamma, mean, rstd = _bn_stats_inputs(C, 4)
    gate, addbc = _unif((B, C), 12), _rand((B, C), torch.float32, 13, 0.1)
    nparts = lib.acnn_bn_bwd_reduce_parts(B, HW, C)
    sk = _sk_inputs(B, HW, f, tdt, 5)
    skp = lib.acnn_sk_bn_bwd_reduce_parts(B, HW, f)
    logits = _rand((B, 1024), torch.float32, 6, 3.0)
    ys = torch.softmax(_rand((B, 1001), torch.float32, 7), 1).contiguous()
    n = 256 * 1000
    w0, grad, a0 = (_rand((n,), torch.float32, s, 0.05) for s in (8, 9, 10))
    flags = (torch.arange(1000, device="cuda") % 3 != 0).to(torch.uint8)
    hp = torch.tensor([0.1, 0.9, 1e-4, 0.5], device="cuda")
    sgd_scratch = torch.zeros(lib.acnn_sgd_scratch_floats(), device="cuda")
    work = torch.zeros(2 * B + B * 1024, device="cuda")
    w, acc = w0.clone(), a0.clone()
    outs = dict(pa=torch.zeros(nparts, 2, C), pb=torch.zeros(nparts, 2, C), pc=torch.zeros(nparts, 2, C),
                coef=torch.zeros(3, C), dgam=torch.zeros(C), dbet=torch.zeros(C), stats=torch.zeros(2, 2 * C),
                scale=torch.zeros(C), shift=torch.zeros(C), mu=torch.zeros(C), rs=torch.zeros(C),
                mm=torch.zeros(C), mv=torch.zeros(C), s=torch.zeros(B, f), dA=torch.zeros(B, f),
                skparts=torch.zeros(skp, 2, 2 * f), gap=torch.zeros(B, C), gem=torch.zeros(B, C),
                ssum=torch.zeros(B, C), loss=torch.zeros(3), dl=torch.zeros(B, 1024), dbias=torch.zeros(1001),
                l2=torch.zeros(1), mean_var=torch.zeros(2 * C))
    outs = {k: v.cuda() for k, v in outs.items()}
    outs["gap"] = outs["gap"].to(tdt)
    outs["gem"] = outs["gem"].to(tdt)
    outs["dl"] = outs["dl"].to(tdt)
    teacher = torch.softmax(_rand((B, 1001), torch.float32, 11), 1).contiguous()

    def run():
        o, st = outs, _st()
        for k in ("loss", "dbias", "l2", "mm", "mv"):
            o[k].zero_()
        w.copy_(w0)
        acc.copy_(a0)
        _check(lib.acnn_bn_bwd_reduce(_p(g), _p(ya), _p(mean), _p(rstd), _p(gate), _p(addbc), _p(o["pa"]), B,
                                      HW, C, code, st), "bn_bwd_reduce")
        _check(lib.acnn_bn_bwd_reduce2(_p(g), _p(ya), _p(yb), _p(mean), _p(rstd), _p(mean), _p(rstd), _p(o["pb"]),
                                       _p(o["pc"]), B, HW, C, code, st), "bn_bwd_reduce2")
        _check(lib.acnn_bn_bwd_finalize(_p(o["pa"]), nparts, _p(gamma), _p(mean), _p(rstd), B * HW, _p(o["coef"]),
                                        _p(o["dgam"]), _p(o["dbet"]), C, st), "bn_bwd_finalize")
        _check(lib.acnn_bn_stats(_p(g), _p(o["mean_var"]), B * HW, C, code, st), "bn_stats")
        _check(lib.acnn_bn_finalize(_p(o["pa"]), nparts, 0, B * HW, _p(gamma), _p(gamma), _p(o["mm"]), _p(o["mv"]),
                                    0.9, 1e-5, 1, _p(o["scale"]), _p(o["shift"]), _p(o["mu"]), _p(o["rs"]), C,
                                    st), "bn_finalize")
        _check(lib.acnn_sk_gap(_p(sk["y"]), _p(sk["scale"]), _p(sk["shift"]), _p(o["s"]), B, HW, f, code, st),
               "sk_gap")
        _check(lib.acnn_sk_bwd_gate(_p(sk["dv"]), _p(sk["y"]), _p(sk["scale"]), _p(sk["shift"]), _p(o["dA"]), B,
                                    HW, f, code, st), "sk_bwd_gate")
        _check(lib.acnn_sk_bn_bwd_reduce(_p(sk["dv"]), _p(sk["y"]), _p(sk["scale"]), _p(sk["shift"]),
                                         _p(sk["mean"]), _p(sk["rstd"]), _p(sk["att"]), _p(sk["ds"]),
                                         _p(o["skparts"]), B, HW, f, code, st), "sk_bn_bwd_reduce")
        _check(lib.acnn_gap_fwd(_p(g), _p(o["gap"]), B, HW, C, code, st), "gap_fwd")
        _check(lib.acnn_gem_fwd(_p(g), _p(o["gem"]), _p(o["ssum"]), B, HW, C, code, st), "gem_fwd")
        _check(lib.acnn_softmax_ce(_p(logits), _p(ys), _p(teacher), 2.0, B, 1001, 1024, 0.1, 1.0, _p(o["loss"]),
                                   _p(o["dl"]), _p(o["dbias"]), _p(work), code, st), "softmax_ce")
        _sgd_call(lib, w, grad, acc, flags, hp, o["l2"], sgd_scratch)

    def snap():
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in outs.items()} | dict(w=w.clone(), acc=acc.clone())

    run()
    first = snap()
    run()
    second = snap()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            run()
    reps = []
    for _ in range(2):
        graph.replay()
        reps.append(snap())
    for label, other in (("repeat", second), ("replay 1", reps[0]), ("replay 2", reps[1])):
        for k in first:
            assert torch.equal(first[k], other[k]), "%s: %s differs" % (label, k)
    assert float(first["l2"]) > 0 and float(first["loss"][0]) > 0


def test_pdl_training_step_bit_identical(lib):
    """One bf16 Assemble-ResNet-50 training step (B = 16, 224 px, mixup type 1) through NativeModel with
    programmatic dependent launch off, on every launch and on light launches only: the same loss,
    gradients, updated weights, momentum and moving statistics, bit for bit."""
    import bench
    from assembled_cnn_b200 import native
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    flags = dict(bench.CONFIGS["c3"]["model"])
    kw = dict(training=True, mixup_type=1, label_smoothing=0.1)
    B, hw = 16, 224
    cfg = ModelConfig(num_classes=1001, **flags)
    plan = build_plan(cfg, B, hw, hw, **kw)
    gen = torch.Generator().manual_seed(5)
    weights = {}
    for n, p in list(plan.params.items()) + list(plan.state.items()):
        if p.kind in ("conv_kernel", "dense_kernel"):
            fan_in = 1
            for d in p.tf_shape[:-1]:
                fan_in *= d
            weights[n] = torch.randn(p.tf_shape, generator=gen) / fan_in ** 0.5
        elif p.kind in ("gamma", "moving_variance"):
            weights[n] = 0.5 + torch.rand(p.tf_shape, generator=gen)
        else:
            weights[n] = 0.1 * torch.randn(p.tf_shape, generator=gen)
    m = plan.meta
    feeds = {m["images"]: (torch.randn(m["input_batch"], hw, hw, 3, generator=gen) * 64).clamp(-124, 152),
             m["labels"]: torch.randint(1, 1001, (m["input_batch"],), generator=gen).int(),
             m["lam1"]: torch.rand(m["input_batch"] // 2, generator=gen)}
    results = {}
    prev = lib.acnn_set_pdl(0)
    try:
        for mode in (0, 1, 2):
            lib.acnn_set_pdl(mode)
            rt = native.NativeRuntime(native.NativeModel(cfg, B, hw, hw, **kw))
            rt.set_weights(weights)
            rt.set_hparams(lr=0.05, momentum=0.9, weight_decay=1e-4, keep_prob=0.9, step=3)
            for name, v in feeds.items():
                rt.t[name].copy_(v)
            rt.run_step()
            torch.cuda.synchronize()
            results[mode] = dict(loss=rt.slot_view(m["loss"]).clone(), grads=rt.grads.clone(),
                                 params=rt.params.clone(), momentum=rt.momentum.clone(), state=rt.state.clone())
            del rt
            torch.cuda.empty_cache()
    finally:
        lib.acnn_set_pdl(prev)
    assert float(results[0]["loss"][0]) > 0 and float(results[0]["grads"].abs().sum()) > 0
    for mode in (1, 2):
        for k, v in results[0].items():
            assert torch.equal(v, results[mode][k]), "PDL mode %d: %s differs" % (mode, k)


# ---------------------------------------------------------------------------------------------------
# channel groups the grid-stride / partial-row kernels reject
# ---------------------------------------------------------------------------------------------------
def test_channel_groups_rejected_before_launch(lib):
    """C = 24 (C / 8 = 3 does not divide 256): the entry points that need cg_ok return ACNN_ERR_INVALID
    with a message, and launch nothing."""
    B, H, W, C = 2, 4, 4, 24
    x = torch.zeros(B, H, W, 2 * C, dtype=torch.bfloat16, device="cuda")
    v = torch.zeros(4 * C, device="cuda")
    st = _st()
    calls = {
        "bn_act": lambda: lib.acnn_bn_act(_p(x), _p(v), _p(v), None, None, None, 0, None, 1, _p(x), B, H, W, C, 0,
                                          st),
        "bn_bwd_reduce": lambda: lib.acnn_bn_bwd_reduce(_p(x), _p(x), _p(v), _p(v), None, None, _p(v), B, H * W, C,
                                                        0, st),
        "bn_bwd_reduce2": lambda: lib.acnn_bn_bwd_reduce2(_p(x), _p(x), _p(x), _p(v), _p(v), _p(v), _p(v), _p(v),
                                                          _p(v), B, H * W, C, 0, st),
        "bn_bwd_apply": lambda: lib.acnn_bn_bwd_apply(_p(x), _p(x), _p(v), None, None, _p(x), B, H * W, C, 0, st),
        "bn_bwd_apply2": lambda: lib.acnn_bn_bwd_apply2(_p(x), _p(x), _p(x), _p(v), _p(v), _p(x), _p(x), B, H * W,
                                                        C, 0, st),
        "sk_gap": lambda: lib.acnn_sk_gap(_p(x), _p(v), _p(v), _p(v), B, H * W, C, 0, st),
        "sk_combine": lambda: lib.acnn_sk_combine(_p(x), _p(v), _p(v), _p(v), _p(x), B, H * W, C, 0, st),
        "sk_bwd_gate": lambda: lib.acnn_sk_bwd_gate(_p(x), _p(x), _p(v), _p(v), _p(v), B, H * W, C, 0, st),
        "se_gap": lambda: lib.acnn_se_gap(_p(x), _p(v), _p(v), _p(v), B, H * W, C, 0, st),
        "gap_fwd": lambda: lib.acnn_gap_fwd(_p(x), _p(x), B, H * W, C, 0, st),
        "gem_fwd": lambda: lib.acnn_gem_fwd(_p(x), _p(x), _p(v), B, H * W, C, 0, st),
        "sk_bn_bwd_reduce": lambda: lib.acnn_sk_bn_bwd_reduce(_p(x), _p(x), _p(v), _p(v), _p(v), _p(v), _p(v), _p(v),
                                                              _p(v), B, H * W, 12, 0, st),
        "sk_bn_bwd_apply": lambda: lib.acnn_sk_bn_bwd_apply(_p(x), _p(x), _p(v), _p(v), _p(v), _p(v), _p(v), _p(x),
                                                            B, H * W, 12, 0, st),
    }
    torch.cuda.synchronize()
    for name, call in calls.items():
        before = lib.acnn_launch_count()
        rc = call()
        assert rc == 1, "%s accepted C=24 (rc %d)" % (name, rc)
        assert lib.acnn_launch_count() == before, "%s launched" % name
        assert lib.acnn_last_error().decode(), name
    assert lib.acnn_bn_bwd_reduce_parts(B, H * W, C) == 0 and lib.acnn_sk_bn_bwd_reduce_parts(B, H * W, 12) == 0
    torch.cuda.synchronize()
