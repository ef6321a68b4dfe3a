"""Host-side checks of tests/test_stream_ops_gpu.py, no kernel involved: every comparator of
oracle/stream_check.py rejects the errors the GPU tests are there to catch -- one row dropped from one
channel's (or one image's) sum, one border pixel's weight changed by one tap, one element moved by two
bf16 ulps -- at the shapes the GPU tests use; the float64 pool restatements agree with oracle/tf_ops.py;
the SK edge shapes reach the pipeline edges they are meant for; and the launch switches."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import stream_check as SC
from oracle import tf_ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _plan(name):
    sys.path.insert(0, ROOT)
    import bench
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    cfg = ModelConfig(num_classes=1001, **bench.CONFIGS[name]["model"])
    return build_plan(cfg, 256, 224, 224, mixup_type=1, label_smoothing=0.1)


def _plan_ops(kind):
    return [op for name in ("c3", "c5") for op in _plan(name).all_ops() if op.kind == kind]


def _bf16_exact(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) * scale).to(torch.bfloat16).double()


def _rejects_dropped_row(terms, n_eff, extra_ops, what):
    """terms [n] of one output: the exact sum passes as its own reference, the sum without its median-
    magnitude term does not."""
    ref = terms.sum()
    tol = SC.reduction_tol(terms.abs().sum(), n_eff, extra_ops)
    assert not SC.violations(ref, ref, tol).any()
    k = int(terms.abs().argsort()[terms.numel() // 2])
    wrong = ref - terms[k]
    assert SC.violations(wrong, ref, tol).all(), "%s: a dropped row (|term| %.3g) is within tol %.3g" % (
        what, float(terms[k].abs()), float(tol))


# ---------------------------------------------------------------------------------------------------
# elementwise: 2 bf16 ulps, at every operation count the GPU tests use
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ops", [1, 2, 3, 4, 5, 6, 10, 11, 13, 27, 197])
def test_elementwise_rejects_two_bf16_ulps(ops):
    ref = _bf16_exact((4, 112, 112, 8), ops) + _bf16_exact((4, 112, 112, 8), ops + 1) * 2.0 ** -12
    mag = ref.abs() * 1.5                      # terms of mixed sign: some cancellation
    got = ref.to(torch.bfloat16).double()      # a correct kernel: one bf16 rounding
    tol = SC.elementwise_tol(ref, mag, True, ops)
    assert not SC.violations(got, ref, tol).any()
    for i in (0, 12345, ref.numel() - 1):
        bad = got.clone().flatten()
        bad[i] = ref.flatten()[i] + 2 * SC.ulp_bf16(ref.flatten()[i])
        assert SC.violations(bad.view_as(ref), ref, tol).flatten()[i]


def test_elementwise_fp32_rejects_small_errors():
    ref = _bf16_exact((1000,), 3) * _bf16_exact((1000,), 4)
    got = ref.float().double()
    tol = SC.elementwise_tol(ref, ref.abs(), False, 6)
    assert not SC.violations(got, ref, tol).any()
    assert SC.violations(got + ref.abs() * 2.0 ** -16, ref, tol).all()


# ---------------------------------------------------------------------------------------------------
# reductions: one dropped row at the production shapes
# ---------------------------------------------------------------------------------------------------
def test_bn_bwd_partials_reject_dropped_row(lib):
    """One partial row of acnn_bn_bwd_reduce (the rows its CTA owns, summed by chains of rows per thread
    + RPB lanes) at every (M, C) of the plans and at the edge shapes."""
    shapes = {tuple(op.shape) for op in _plan_ops("bn_bwd_reduce") + _plan_ops("bn_bwd_reduce2")}
    shapes |= {(B, H, W, C) for C in (8, 64, 2048) for (B, H, W) in ((1, 1, 1), (3, 7, 5), (5, 13, 9))}
    for (B, H, W, C) in sorted(shapes):
        M = B * H * W
        nparts = lib.acnn_bn_bwd_reduce_parts(B, H * W, C)
        owner = SC.bn_bwd_reduce_owner(M, C, nparts)
        rows = int((owner == 0).sum())
        if rows < 2:
            continue
        g = _bf16_exact((rows,), C)
        xhat = _bf16_exact((rows,), C + 1)
        for terms in (g, g * xhat):
            _rejects_dropped_row(terms, SC.bn_bwd_reduce_chain(M, C, nparts), 5, "bn_bwd %s" % ((B, H, W, C),))


def test_sk_partials_reject_dropped_row(lib):
    """One (image, slab) partial row of acnn_sk_bn_bwd_reduce and one image of sk_gap / sk_bwd_gate at
    every SK shape of the plans and the edge shapes."""
    shapes = {(op.B, op.HW, op.f) for op in _plan_ops("sk_gap")} | set(SC.SK_EDGE_SHAPES)
    for (B, HW, f) in sorted(shapes):
        s, rows_per, rt = SC.sk_slabs(B, HW, f, 2)
        assert lib.acnn_sk_bn_bwd_reduce_parts(B, HW, f) == B * s
        n = min(rows_per, HW)
        if n >= 2:
            t = _bf16_exact((n,), HW).clamp_min(0) + 0.01
            _rejects_dropped_row(t * _bf16_exact((n,), f), 4 * -(-rows_per // rt) + 1024 // f, 6,
                                 "sk_bn_bwd_reduce %s" % ((B, HW, f),))
        if HW >= 2:
            rpb = 256 // (f // 8)
            u = _bf16_exact((HW,), f).abs()
            _rejects_dropped_row(u, 2 * -(-HW // (2 * rpb)) + rpb, 4, "sk_gap %s" % ((B, HW, f),))


@pytest.mark.parametrize("C", [8, 64, 512, 1024, 2048, 4096])
def test_image_reductions_reject_dropped_row(C):
    """gap_fwd / gem_fwd per (image, channel) over the HW rows the GPU tests use (the plans' 7 x 7 map,
    the edge maps): chains of ceil(HW / RPB) + RPB."""
    for HW in (2, 7, 49, 50, 197):
        fl = C // (C // 512) if (C >= 1024 and C % 512 == 0) else C
        rpb = 256 // min(fl // 8, 256)
        x = _bf16_exact((HW,), HW + C, 1.0).abs() + 0.5
        _rejects_dropped_row(x, -(-HW // rpb) + rpb, 2, "gap HW=%d C=%d" % (HW, C))
        rpb = 256 // min(C // 8, 256)
        _rejects_dropped_row(x.abs().clamp_min(1e-6) ** 3, -(-HW // rpb) + rpb, 2, "gem HW=%d C=%d" % (HW, C))


@pytest.mark.parametrize("nparts", [1, 31, 32, 33, 132, 264])
def test_finalize_rejects_dropped_partial_row(nparts):
    if nparts >= 2:
        _rejects_dropped_row(_bf16_exact((nparts,), nparts), -(-nparts // 32) + 32, 0, "finalize")


def test_loss_and_optimizer_sums_reject_dropped_row():
    """softmax_ce: dbias over the B rows (B + 1 adds); sgd L2: one CTA partial of the 1056 of the c3
    step (one element of 42 M parameters is below any fp32 bound -- what a wrong last-CTA sum loses
    is whole partials)."""
    for B in (2, 33, 256, 512):
        _rejects_dropped_row(_bf16_exact((B,), B, 1e-3), B + 1, 0, "dbias B=%d" % B)
    n = 41908992
    grid = 132 * 8
    parts = _bf16_exact((grid,), 1).abs() * 1e-3 + 1e-3
    trips = -(-(n // 4) // (grid * 256))
    _rejects_dropped_row(parts, 4 * trips + 5 + 8 + 5 + 256 + 3, 0, "sgd l2")


def test_bn_stats_exact_design_detects_a_dropped_row():
    """The exactly summable bn_stats data (test_bn_stats_production): dropping a row with k != 0 moves
    the variance by 1/64/M, more than half an fp32 ulp at the variance (the whole tolerance)."""
    M = 256 * 112 * 112
    for nz in (M // 3, 2 * M // 3):
        var = torch.tensor([nz / 64 / M], dtype=torch.float64)
        wrong = torch.tensor([(nz - 1) / 64 / M], dtype=torch.float32).double()
        assert SC.violations(wrong, var, 0.5 * SC.ulp_f32(var)).all()


# ---------------------------------------------------------------------------------------------------
# pools: one border pixel's weight changed by one tap
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("filt,stride,H", [(3, 2, 56), (3, 2, 14), (3, 2, 7), (5, 1, 9), (7, 2, 13),
                                           (6, 1, 7), (4, 2, 7)])
def test_blurpool_tolerance_rejects_one_tap(filt, stride, H):
    """The reference with the weight of one tap of a border output pixel replaced by its neighbour's
    (what a wrong reflection or a shifted window does) is rejected at that pixel, forward and backward."""
    C = 8
    x = _bf16_exact((1, H, H, C), H) + 2.0
    fn = lambda t: tf_ops.anti_aliased_downsample(t, filt, stride)   # noqa: E731
    ref, mag = fn(x), fn(x.abs())
    tol = SC.elementwise_tol(ref, mag, True, filt * filt)
    assert not SC.violations(ref.to(torch.bfloat16).double(), ref, tol).any()
    a = torch.tensor(tf_ops._BINOMIAL[filt], dtype=torch.float64)
    a = a / a.sum()
    # output (0, 0) reads rows reflect(t - pad); swapping the weights of taps 0 and 1 on row 0
    pad = (filt - 1) // 2
    r0, r1 = abs(0 - pad), abs(1 - pad)
    wrong = ref.clone()
    cols = [abs(s - pad) for s in range(filt)]
    row_diff = sum(a[s] * (x[0, r1, cols[s]] - x[0, r0, cols[s]]) for s in range(filt))
    wrong[0, 0, 0] += (a[0] - a[1]) * row_diff
    assert SC.violations(wrong, ref, tol)[0, 0, 0].any()
    # backward: the adjoint at border input pixel (0, 0) with one tap's weight swapped likewise
    dout = _bf16_exact(ref.shape, H + 1) + 2.0
    xg = x.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad(fn(xg), xg, dout)
    xg2 = x.clone().requires_grad_(True)
    (gm,) = torch.autograd.grad(fn(xg2), xg2, dout.abs())
    tol = SC.elementwise_tol(gx, gm, True, (2 * filt) ** 2 + 1)
    assert not SC.violations(gx.to(torch.bfloat16).double(), gx, tol).any()
    wrong = gx.clone()
    wrong[0, 0, 0] += (a[0] - a[1]) * a[pad] * dout[0, 0, 0]
    assert SC.violations(wrong, gx, tol)[0, 0, 0].any()


def test_pool_restatements_match_tf_ops():
    x = _bf16_exact((2, 14, 14, 8), 1)
    for H in (14, 7, 9, 2, 1):
        xs = x[:, :H, :H]
        # bl shortcut: fixed_padding(3) + 3x3 / 2 VALID, zeros counted
        Ho = (H + 2 - 3) // 2 + 1
        assert torch.allclose(SC.avgpool_ref(xs, 3, 2, 1, Ho, Ho, 1), tf_ops.avg_pool_bl(xs, 2), atol=1e-12)
        # resnet-d: 2x2 / 2 after fixed_padding(2) (0 before); 2x2 / 1 SAME, padded cells not counted
        Ho = (H + 1 - 2) // 2 + 1
        assert torch.allclose(SC.avgpool_ref(xs, 2, 2, 0, Ho, Ho, 1), tf_ops.avg_pool_resnet_d(xs, 2),
                              atol=1e-12)
        assert torch.allclose(SC.avgpool_ref(xs, 2, 1, 0, H, H, 0), tf_ops.avg_pool_resnet_d(xs, 1), atol=1e-12)
        # TF SAME 3x3 / 2 max pool (the odd pad cell after)
        Ho = -(-H // 2)
        lo = max((Ho - 1) * 2 + 3 - H, 0) // 2
        assert torch.equal(SC.maxpool_ref(xs, 3, 2, lo, Ho, Ho), tf_ops.max_pool_same(xs, 3, 2))


def test_maxpool_restatement_routes_to_first_maximum():
    x = torch.zeros(1, 2, 2, 1, dtype=torch.float64)          # four tied cells in one window
    _, dx = SC.maxpool_ref(x, 2, 2, 0, 1, 1, torch.ones(1, 1, 1, 1, dtype=torch.float64))
    assert dx.flatten().tolist() == [1.0, 0.0, 0.0, 0.0]


def test_ulps():
    v = torch.tensor([1.0, 1.5, 2.0 ** -10, 3.0, 0.0], dtype=torch.float64)
    assert SC.ulp_bf16(v)[:4].tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -17, 2.0 ** -6]
    assert SC.ulp_f32(v)[:4].tolist() == [2.0 ** -23, 2.0 ** -23, 2.0 ** -33, 2.0 ** -22]


# ---------------------------------------------------------------------------------------------------
# shapes and switches
# ---------------------------------------------------------------------------------------------------
def test_sk_edge_shapes_reach_every_edge():
    for cps in (8, 2):
        seen = set()
        for c in SC.SK_EDGE_SHAPES:
            seen |= SC.sk_slab_edges(*c, cps)
        assert seen == {"empty", "wrap", "partial"}, (cps, seen)
    # the one-CTA-per-image reductions at HW 49, f 512: 7 trips of 8 rows, the last one 1 row
    assert -(-49 // 8) > 3 and 49 % 8


def test_grid_cap_setter(lib):
    """acnn_set_stream_grid_cap (host state only): values below 132 CTAs restore the default 16 x 132."""
    prev = lib.acnn_set_stream_grid_cap(500)
    try:
        assert lib.acnn_set_stream_grid_cap(7) == 500
        assert lib.acnn_set_stream_grid_cap(132) == 132 * 16
        assert lib.acnn_set_stream_grid_cap(0) == 132
    finally:
        lib.acnn_set_stream_grid_cap(prev)


@pytest.mark.parametrize("env,mode", [("1", 1), ("2", 2), ("0", 0), ("3", 0), (None, 0)])
def test_pdl_environment_switch(env, mode):
    """ACNN_PDL=1|2 selects programmatic dependent launch at load time (anything else: off);
    acnn_set_pdl returns the previous setting."""
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from assembled_cnn_b200 import _lib\n"
            "lib = _lib.load()\n"
            "print(lib.acnn_set_pdl(2), lib.acnn_set_pdl(5), lib.acnn_set_pdl(1))\n" % ROOT)
    envv = {k: v for k, v in os.environ.items() if k != "ACNN_PDL"}
    if env is not None:
        envv["ACNN_PDL"] = env
    out = subprocess.run([sys.executable, "-s", "-c", code], env=envv, capture_output=True, text=True,
                         timeout=120)
    assert out.returncode == 0, out.stderr
    assert out.stdout.split() == [str(mode), "2", "0"]
