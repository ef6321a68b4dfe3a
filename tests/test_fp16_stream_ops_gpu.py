"""Op-level tests of the fp16 (ACNN_F16) instantiations of the HBM-bound kernels: batch norm forward and
backward, the SK / SE reductions and combine, blur / average / max pooling, upsample and zero-insert, GAP,
GeM, DropBlock, the softmax cross-entropy (its fp16 dlogits), the input packing, the grid-stride launches
under every grid cap, the reductions under repeat and CUDA-graph replay, and the training step under
programmatic dependent launch -- plus the fp16 weight copies (acnn_prep_weights_f16, the stem's
acnn_s2d_weight_pack).

The element-generic tests of tests/test_stream_ops_gpu.py run here on fp16 storage: the same production
shapes (every distinct (op, shape) of the c3 / c5 training plans at B = 256, 224 px), the same grid edges,
the same float64 references computed from the kernel's own (here fp16-representable) inputs.  Their
tolerances are oracle/stream_check.py's with the storage rounding of the 16-bit outputs taken at fp16's
spacing (11 significant bits: unit roundoff 2^-11) instead of bf16's: the `dt` fixture below selects the
16-bit storage path of those tests with ACNN_F16 / torch.float16 and stream_check's 16-bit ulp function
with the fp16 one."""
import functools

import pytest
import torch

import test_stream_ops_gpu as S
from oracle import stream_check as SC

pytestmark = pytest.mark.gpu

ACNN_F16 = 3


def ulp_f16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 numbers at |x| (11 significant bits), float64; the subnormal spacing 2^-24 below
    2^-14."""
    x = x.double().abs().clamp_min(2.0 ** -14)
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), (e - 11).to(torch.int64))


@pytest.fixture
def dt(monkeypatch):
    # the 16-bit storage path of the shared tests ("bf16" there: code, torch dtype, storage ulp) on fp16
    monkeypatch.setitem(S.DTYPES, "bf16", (ACNN_F16, torch.float16))
    monkeypatch.setattr(SC, "ulp_bf16", ulp_f16)
    return "bf16"


def _on_fp16(fn):
    """The shared test `fn` collected here, with this module's `dt` fixture."""
    @functools.wraps(fn)
    def run(*args, **kwargs):
        return fn(*args, **kwargs)
    return run


for _name in ("test_bn_act_plan_shapes", "test_bn_act_edges", "test_bn_bwd_plan_shapes", "test_bn_bwd2_plan_shapes",
              "test_bn_bwd_edges", "test_bn_stats_production", "test_sk_plan_shapes", "test_sk_edges",
              "test_blurpool_plan_shapes", "test_blurpool_edges", "test_avgpool_plan_shapes", "test_avgpool_edges",
              "test_maxpool_production", "test_maxpool_edges", "test_resample_plan_shapes", "test_resample_edges",
              "test_gap_plan_shapes", "test_gap_edges", "test_gem_production", "test_gem_edges",
              "test_dropblock_plan_shapes", "test_dropblock_edges", "test_softmax_ce", "test_pack_input_plan",
              "test_grid_cap_bit_identical", "test_reductions_repeat_and_graph_replay_bit_identical"):
    globals()[_name.replace("test_", "test_fp16_", 1)] = _on_fp16(getattr(S, _name))


def test_fp16_storage_is_selected(lib, dt):
    """The fixture really runs the fp16 instantiations: an fp16-only value survives bn_act unchanged."""
    code, tdt = S.DTYPES[dt]
    assert (code, tdt) == (ACNN_F16, torch.float16)
    a = torch.full((1, 1, 1, 8), 1.0 + 2.0 ** -10, dtype=tdt, device="cuda")   # not a bf16 value
    one = torch.ones(8, device="cuda")
    zero = torch.zeros(8, device="cuda")
    out = torch.empty_like(a)
    S._check(lib.acnn_bn_act(S._p(a), S._p(one), S._p(zero), None, None, None, 0, None, 0, S._p(out), 1, 1, 1, 8,
                             code, S._st()), "bn_act")
    torch.cuda.synchronize()
    assert torch.equal(out, a)


def test_fp16_pdl_training_step_bit_identical(lib, monkeypatch):
    """The fp16 training step (c3 flags, B = 16, 224 px, mixup 1) with programmatic dependent launch off, on
    every launch and on light launches only: the same loss, gradients, weights, momentum and statistics."""
    from assembled_cnn_b200 import native
    monkeypatch.setattr(native, "NativeModel", functools.partial(native.NativeModel, dtype="fp16"))
    S.test_pdl_training_step_bit_identical(lib)


def test_fp16_weight_copies(lib):
    """acnn_prep_weights_f16: every conv weight of the c3 plan in both layouts is the fp32 master rounded to
    nearest even (torch's float16 conversion), bit for bit, with the copies of an out-of-range weight inf;
    acnn_s2d_weight_pack in fp16 is the fp32 pack rounded likewise."""
    import bench
    from assembled_cnn_b200 import _lib
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    cfg = ModelConfig(num_classes=1001, **bench.CONFIGS["c3"]["model"])
    plan = build_plan(cfg, 2, 64, 64, dtype="fp16", training=True)
    # the weights with GEMM operand copies (Cin % 16 == 0, Cout % 32 == 0), one acnn_weight_desc each: the
    # master at its offset in params and in w_fprop, the dgrad layout at dgrad_off in w_dgrad
    conv = [p for p in plan.params.values() if p.kind in ("conv_kernel", "dense_kernel")
            and len(p.store_shape) == 4 and p.store_shape[3] % 16 == 0 and p.store_shape[0] % 32 == 0]
    descs = [_lib.WeightDesc(p.offset, p.offset, p.dgrad_off, p.store_shape[0], p.store_shape[1] * p.store_shape[2],
                             p.store_shape[3], 0) for p in conv]
    n_descs = len(descs)
    table = torch.frombuffer(bytearray(bytes((_lib.WeightDesc * n_descs)(*descs))), dtype=torch.uint8).cuda()
    g = torch.Generator(device="cuda").manual_seed(3)
    params = torch.zeros(plan.param_elems, device="cuda").normal_(0.0, 0.3, generator=g)
    o = conv[0].offset
    params[o] = 1e6                                             # beyond fp16: inf
    params[o + 1] = 3e-6                                        # an fp16 subnormal
    w_fprop = torch.full((plan.param_elems,), float("nan"), dtype=torch.float16, device="cuda")
    w_dgrad = torch.full((max(plan.dgrad_elems, 1),), float("nan"), dtype=torch.float16, device="cuda")
    S._check(lib.acnn_prep_weights_f16(params.data_ptr(), table.data_ptr(), n_descs, w_fprop.data_ptr(),
                                       w_dgrad.data_ptr(), S._st()), "prep_weights_f16")
    torch.cuda.synchronize()
    n = 0
    for p in conv:
        co, kh, kw, ci = p.store_shape
        master = params[p.offset:p.offset + p.size].view(co, kh, kw, ci)
        want = master.half()
        got = w_fprop[p.offset:p.offset + p.size].view(co, kh, kw, ci)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), p.name
        if p.dgrad_off >= 0:
            wd = want.flip(1, 2).permute(3, 1, 2, 0).contiguous()
            got_d = w_dgrad[p.dgrad_off:p.dgrad_off + p.size].view(ci, kh, kw, co)
            assert torch.equal(got_d.view(torch.int16), wd.view(torch.int16)), p.name
        n += 1
    assert n == n_descs > 50 and torch.isinf(w_fprop[o]) and w_fprop[o + 1] != 0
    # the stem's space-to-depth pack
    Cout, k, pad, k2, pad2 = 64, 7, 3, 4, 2
    w = torch.randn(Cout, k, k, 3, generator=g, device="cuda")
    out = {}
    for code, tdt in ((1, torch.float32), (ACNN_F16, torch.float16)):
        o = torch.full((Cout, k2, k2, 16), float("nan"), dtype=tdt, device="cuda")
        S._check(lib.acnn_s2d_weight_pack(w.data_ptr(), o.data_ptr(), Cout, k, pad, k2, pad2, code, S._st()),
                 "s2d_weight_pack")
        out[code] = o
    torch.cuda.synchronize()
    assert torch.equal(out[ACNN_F16].view(torch.int16), out[1].half().view(torch.int16))

