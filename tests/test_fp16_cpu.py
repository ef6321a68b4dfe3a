"""The fp16 mode (dtype='fp16', the reference's --dtype=fp16) on the host side, no GPU:

  * the C++ and the Python plan builders give the same plan text in fp16 on the plan cases of
    test_native_plan_cpu.py and on a sample of the flag space, and every op resolves (acnn_validate);
  * the fp16 plan is the bf16 plan op for op: only the activation storage type differs;
  * the argument checks of the C ABI and of the Python surface accept fp16 and still refuse what they
    refused (acnn_create dtype 7, acnn_knn_topk dtype 2);
  * the loss scale is resolved as the reference's get_loss_scale: explicit wins, else 128 for fp16 and 1
    for bf16 / fp32.
"""
import ctypes as C

import pytest
from hypothesis import HealthCheck, given, settings

import test_native_plan_cpu as base
from assembled_cnn_b200 import _lib, native
from assembled_cnn_b200.plan import ModelConfig, build_plan, dump


def _fp16(kw):
    return dict(kw, dtype="fp16")


@pytest.mark.parametrize("case", range(len(base.CASES)))
def test_fp16_native_plan_equals_python_plan(case):
    flags, B, H, W, kw = base.CASES[case]
    cfg = ModelConfig(**flags)
    py = dump(build_plan(cfg, B, H, W, **_fp16(kw)))
    nm = native.NativeModel(cfg, B, H, W, **_fp16(kw))
    cc = nm.dump()
    assert py == cc, base._diff(py, cc)
    assert "dtype=f16" in py and "dtype=bf16" not in py
    nm.validate()
    nm.close()


@pytest.mark.parametrize("case", range(len(base.CASES)))
def test_fp16_plan_is_the_bf16_plan_with_fp16_storage(case):
    """Same ops, arguments, buffers and offsets as the bf16 plan; every bf16 tensor becomes fp16."""
    flags, B, H, W, kw = base.CASES[case]
    cfg = ModelConfig(**flags)
    f16 = native.NativeModel(cfg, B, H, W, **_fp16(kw)).dump()
    bf16 = native.NativeModel(cfg, B, H, W, **dict(kw, dtype="bf16")).dump()
    assert f16.replace("dtype=f16", "dtype=bf16").replace("meta dtype=fp16", "meta dtype=bf16") == bf16


@pytest.mark.parametrize("name,case", [("c1", 1), ("c3", 2), ("c5", 4)])
def test_baseline_configurations_resolve_in_fp16(name, case):
    flags, B, H, W, kw = base.CASES[case]
    nm = native.NativeModel(ModelConfig(**flags), B, H, W, **_fp16(kw))
    nm.validate()
    assert nm.meta["dtype"] == "fp16"
    assert all(t.dtype in ("f16", "f32", "i32") for t in nm.tensors.values())
    s = nm.sizes
    assert s.w_fprop_elems == s.param_elems          # one fp16 copy, not three planes
    nm.close()


@settings(max_examples=25, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
@given(base._flag_sets())
def test_fp16_native_and_python_plans_agree_over_the_flag_space(case):
    flags, B, hw, kw = case
    case = (flags, B, hw, _fp16(kw))
    py, cc = base._both(case)
    assert py is not None and cc is not None, case
    assert py == cc, (case, base._diff(py, cc))
    nm = native.NativeModel(ModelConfig(**flags), B, hw[0], hw[1], **_fp16(kw))
    nm.validate()
    nm.close()


def _create_rc(dtype):
    l = native.lib()
    c = native.Config()
    l.acnn_model_config_init(C.byref(c))
    c.dtype = dtype
    h = C.c_void_p()
    r = l.acnn_create(C.byref(c), C.byref(h))
    if r == 0:
        l.acnn_destroy(h)
    return r, l.acnn_last_error().decode()


def test_create_accepts_fp16_and_still_refuses_other_values():
    assert _create_rc(3)[0] == 0                     # ACNN_F16
    for bad in (2, 7, -1):                           # 2 is ACNN_I32, not a storage type
        r, msg = _create_rc(bad)
        assert r == 1 and "fp16" in msg, (bad, r, msg)


def test_python_surface_accepts_fp16():
    from assembled_cnn_b200 import metrics, model_fns as F
    assert "fp16" in F.ALLOWED_TYPES
    m = F.Model(50, dtype="fp16")                    # no GPU work at construction
    assert m.dtype == "fp16"
    with pytest.raises(ValueError):
        F.Model(50, dtype="fp8")
    with pytest.raises(ValueError):
        native.make_config(ModelConfig(resnet_size=50), 1, 64, 64, dtype="fp8")
    with pytest.raises(ValueError):
        build_plan(ModelConfig(resnet_size=50), 1, 64, 64, dtype="fp8")
    assert metrics.RecallAtK(dtype="fp16").dtype == "fp16"


def test_loss_scale_resolution_follows_get_loss_scale():
    from assembled_cnn_b200.hparams import DEFAULTS, get_loss_scale, params_from_flags
    assert DEFAULTS["loss_scale"] is None and DEFAULTS["dtype"] == "bf16"
    assert get_loss_scale(None, "fp16") == 128.0
    assert get_loss_scale(None, "bf16") == 1.0 and get_loss_scale(None, "fp32") == 1.0
    for dt in ("fp16", "bf16", "fp32"):
        assert get_loss_scale(5, dt) == 5.0 and get_loss_scale(1, dt) == 1.0
        assert get_loss_scale(0, dt) == 1.0
    p = params_from_flags(dtype="fp16")
    assert get_loss_scale(p["loss_scale"], p["dtype"]) == 128.0
    with pytest.raises(ValueError):
        get_loss_scale(None, "fp8")


def test_knn_dtype_enum():
    """acnn_knn_topk / acnn_knn_work_bytes: 3 (ACNN_F16) is accepted with the bf16 layout (one operand plane),
    2 is still refused, before any CUDA call."""
    l = _lib.load()
    nq, nx, d, k = 100, 300, 70, 5
    assert l.acnn_knn_work_bytes(nq, nx, d, k, 3) == l.acnn_knn_work_bytes(nq, nx, d, k, 0) > 0
    assert l.acnn_knn_work_bytes(nq, nx, d, k, 1) > l.acnn_knn_work_bytes(nq, nx, d, k, 0)
    assert l.acnn_knn_work_bytes(nq, nx, d, k, 2) == -1
    rc = l.acnn_knn_topk(None, None, nq, nx, d, k, 0, 2, None, None, None, 0, None)
    assert rc == 1 and b"dtype" in l.acnn_last_error()


def test_conv_precision_enum():
    """The conv GEMMs take precision ACNN_F16 (3) with the bf16 path's wgrad split layout; 2 is refused
    before any CUDA call."""
    l = _lib.load()
    g = _lib.ConvGeom(32, 56, 56, 64, 64, 3, 3, 1, 1, 1, 1, 1)
    for det in (0, 1):
        out = {}
        for prec in (0, 3):
            pix, splits, per = C.c_int(), C.c_int(), C.c_int()
            assert l.acnn_conv_wgrad_plan(C.byref(g), prec, det, C.byref(pix), C.byref(splits),
                                          C.byref(per)) == 0
            out[prec] = (pix.value, splits.value, per.value)
        assert out[3] == out[0]
    assert l.acnn_conv_wgrad_plan(C.byref(g), 2, 0, None, None, None) == 1
    dummy = C.c_void_p(256)
    assert l.acnn_conv_fprop(C.byref(g), dummy, dummy, dummy, None, None, None, None, 0, 2, 0, None) == 1
    assert b"precision" in l.acnn_last_error()
    assert l.acnn_conv_wgrad(C.byref(g), dummy, dummy, dummy, 2, 0, None) == 1
