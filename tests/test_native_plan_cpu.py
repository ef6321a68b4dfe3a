"""The model-level C ABI (include/acnn_model.h) builds its layer plan in C++ (csrc/model_plan.cu); the
oracle's interpreter walks the Python plan (assembled_cnn_b200/plan.py) in lockstep with the library's
executor in the op-by-op parity tests.  These CPU tests pin the two to the SAME plan -- variables (TF
names, creation order, layouts, offsets), buffers, and every op with every argument -- by comparing
their canonical texts, so the interpreter runs, op for op, what the library runs.  No GPU: acnn_create
is host logic."""
import ctypes as C
import difflib
import os
import re

import pytest

from assembled_cnn_b200 import _lib, native
from assembled_cnn_b200.plan import ModelConfig, build_plan, dump

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ASSEMBLE = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)

CASES = [
    # (constructor flags, batch, H, W, step flags)
    (dict(resnet_size=50), 4, 64, 64, dict(training=True)),
    (dict(resnet_size=50), 1, 224, 224, dict(training=False, with_loss=False)),            # BASELINE C1
    (ASSEMBLE, 256, 224, 224, dict(training=True, mixup_type=1, label_smoothing=0.1)),     # BASELINE C3
    (ASSEMBLE, 256, 224, 224, dict(training=False, with_loss=True, label_smoothing=0.1)),  # C2 eval
    (dict(ASSEMBLE, resnet_size=152, bl_alpha=1, bl_beta=2), 128, 224, 224,
     dict(training=True, mixup_type=1, label_smoothing=0.1)),                               # BASELINE C5
    (ASSEMBLE, 8, 128, 128, dict(training=True, mixup_type=2, dtype="fp32")),
    (ASSEMBLE, 8, 128, 128, dict(training=False, with_loss=True, dtype="fp32")),
    (dict(ASSEMBLE, use_resnet_d=True), 4, 64, 64, dict(training=True)),
    (dict(resnet_size=50, use_resnet_d=True), 4, 64, 64, dict(training=True, mixup_type=1)),
    (dict(resnet_size=50, resnet_version=2, use_se_block=True, anti_alias_type="proj",
          anti_alias_filter_size=5), 4, 64, 64, dict(training=True)),
    (dict(resnet_size=50, use_se_block=True, zero_gamma=True), 4, 64, 64,
     dict(training=True, dtype="fp32")),
    (dict(resnet_size=101, resnet_version=2, use_sk_block=True, anti_alias_type="sconv,proj",
          anti_alias_filter_size=3, no_downsample=True), 2, 96, 64, dict(training=True)),
    (dict(resnet_size=200), 2, 64, 64, dict(training=True)),
    (dict(resnet_size=101, no_downsample=True), 3, 64, 96, dict(training=False, with_loss=True)),
    (dict(ASSEMBLE, pool_type="gem", embedding_size=256), 4, 64, 64, dict(training=True)),
    (dict(ASSEMBLE, pool_type="gem", embedding_size=256), 4, 64, 64, dict(training=False)),
    (dict(resnet_size=50, pool_type="flatten", num_classes=10), 4, 64, 64, dict(training=True)),
    (dict(resnet_size=50, pool_type="flatten", embedding_size=64), 4, 64, 64,
     dict(training=True, dtype="fp32")),
    (ASSEMBLE, 4, 224, 224, dict(training=True, use_dropblock=True, mixup_type=1)),
    (dict(resnet_size=50), 4, 224, 224, dict(training=True, use_dropblock=True)),
    (dict(resnet_size=50, use_resnet_d=True), 4, 224, 224,
     dict(training=True, use_dropblock=True, dtype="fp32")),
    (ASSEMBLE, 4, 64, 64, dict(training=True, kd_temp=2.0, mixup_type=2)),
    (ASSEMBLE, 4, 64, 64, dict(training=True, kd_temp=4.0, mixup_type=1, label_smoothing=0.1)),
    (dict(ASSEMBLE, bl_alpha=1, bl_beta=4, bn_momentum=0.9), 4, 64, 64, dict(training=True)),
]


def _diff(a, b):
    d = list(difflib.unified_diff(a.splitlines(), b.splitlines(), "python", "native", lineterm="", n=0))
    return "%d differing lines\n%s" % (len(d), "\n".join(d[:40]))


@pytest.mark.parametrize("case", range(len(CASES)))
def test_native_plan_equals_python_plan(case):
    flags, B, H, W, kw = CASES[case]
    cfg = ModelConfig(**flags)
    py = dump(build_plan(cfg, B, H, W, **kw))
    nm = native.NativeModel(cfg, B, H, W, **kw)
    cc = nm.dump()
    assert py == cc, _diff(py, cc)
    assert len(py.splitlines()) > 500
    # every op of the plan resolves into a launch record (acnn_validate: the host side of acnn_bind on
    # synthetic addresses -- partial-row buffers and scratch slots fit what the op level asks for)
    nm.validate()
    nm.close()


def test_native_plan_honours_fuse_bn_pairs(monkeypatch):
    monkeypatch.setenv("ACNN_FUSE_BN_PAIRS", "0")
    cfg = ModelConfig(**ASSEMBLE)
    py = dump(build_plan(cfg, 4, 64, 64, training=True))
    cc = native.NativeModel(cfg, 4, 64, 64, training=True).dump()
    assert "bn_bwd_reduce2" not in py and py == cc, _diff(py, cc)


def test_model_abi_symbols_and_struct_layouts():
    """Every function include/acnn_model.h declares is exported and bound; the ctypes mirrors of the
    ABI structs have the C sizes (checked through struct_size and a compiled probe-free identity:
    acnn_create rejects a config whose struct_size differs)."""
    l = native.lib()
    header = re.sub(r"/\*.*?\*/", " ", open(native.MODEL_HEADER).read(), flags=re.S)
    declared = set(re.findall(r"\b(acnn_[a-z0-9_]+)\s*\(", header))
    assert declared == set(native.PROTOTYPES), declared ^ set(native.PROTOTYPES)
    for name in declared:
        assert hasattr(l, name), name
    c = native.Config()
    l.acnn_model_config_init(C.byref(c))
    assert c.struct_size == C.sizeof(native.Config)          # layout agrees with the library's
    assert (c.resnet_size, c.resnet_version, c.num_classes, c.bl_alpha, c.bl_beta) == (50, 1, 1001, 2, 4)
    assert c.pool_type == b"gap" and c.bn_momentum == 0.997 and c.deterministic == -1
    c.struct_size -= 4
    h = C.c_void_p()
    assert l.acnn_create(C.byref(c), C.byref(h)) != 0
    assert b"struct_size" in l.acnn_last_error()


def test_create_errors_match_reference_messages():
    """nets/resnet_model.py:201-215 / functions/model_fns.py:131-135 argument errors, as status codes."""
    l = native.lib()

    def rc(**over):
        c = native.Config()
        l.acnn_model_config_init(C.byref(c))
        for k, v in over.items():
            setattr(c, k, v)
        h = C.c_void_p()
        r = l.acnn_create(C.byref(c), C.byref(h))
        if r == 0:
            l.acnn_destroy(h)
        return r, l.acnn_last_error().decode()

    assert rc()[0] == 0
    r, msg = rc(resnet_version=3)
    assert r == 1 and "Resnet version should be 1 or 2" in msg
    r, msg = rc(resnet_size=18)
    assert r == 3 and "non-bottleneck" in msg
    r, msg = rc(resnet_size=51)
    assert r == 1 and "Could not find layers" in msg
    assert rc(height=100)[0] == 1 and rc(mixup_type=3)[0] == 1 and rc(dtype=7)[0] == 1
    assert rc(pool_type=b"max")[0] == 3 and rc(loss_type=b"sigmoid")[0] == 3
    r, msg = rc(use_dropblock=1, height=64, width=64)
    assert r == 1 and "dropblock" in msg


def test_variable_inventory_in_tf_creation_order():
    """acnn_variable_info_get lists trainables and moving statistics interleaved in the reference's
    creation order (kernel, gamma, beta, moving_mean, moving_variance per conv), TF names."""
    nm = native.NativeModel(ModelConfig(**ASSEMBLE), 2, 64, 64, training=True)
    l, vi = nm.lib, native.VariableInfo()
    names = []
    for i in range(nm.sizes.n_variables):
        assert l.acnn_variable_info_get(nm.handle, i, C.byref(vi)) == 0
        names.append(vi.name.decode())
    assert names[:5] == ["resnet_model/stage0/conv2d/kernel",
                         "resnet_model/stage0_1/batch_normalization/gamma",
                         "resnet_model/stage0_1/batch_normalization/beta",
                         "resnet_model/stage0_1/batch_normalization/moving_mean",
                         "resnet_model/stage0_1/batch_normalization/moving_variance"]
    assert names[-2:] == ["resnet_model/dense/kernel", "resnet_model/dense/bias"]
    py = build_plan(ModelConfig(**ASSEMBLE), 2, 64, 64, training=True)
    assert [n for n in names if n in py.params] == list(py.params)
    assert [n for n in names if n in py.state] == list(py.state)
    assert len(names) == len(py.params) + len(py.state)
    # gradient readiness: every trainable except dense/bias (written by the loss op in the forward
    # list) gets its gradient from a backward op; later layers are ready earlier
    done = nm.grad_done_at()
    assert set(py.params) - set(done) == {"resnet_model/dense/bias"}
    assert done["resnet_model/dense/kernel"] == 0
    assert done["resnet_model/stage0/conv2d/kernel"] == max(done.values())
    from assembled_cnn_b200 import dp
    assert dp.grad_buckets(py) == dp.grad_buckets(nm)


def test_workspace_layout_is_disjoint_and_aligned():
    nm = native.NativeModel(ModelConfig(**ASSEMBLE), 8, 128, 128, training=True, mixup_type=1)
    s = nm.sizes
    spans = [(s.hp_offset, 32), (s.decay_flags_offset, max(s.param_elems // 256, 1)),
             (s.zero_offset, s.zero_bytes), (s.work_offset, s.work_bytes)]
    esz = {"bf16": 2, "f32": 4, "i32": 4}
    for name, t in nm.tensors.items():
        n = esz[t.dtype]
        for d in t.shape:
            n *= d
        spans.append((nm.tensor_offset[name], n))
    spans.sort()
    for (o, n), (o2, _) in zip(spans, spans[1:]):
        assert o % 1024 == 0 and o + n <= o2
    assert spans[-1][0] + spans[-1][1] <= s.workspace_bytes
    assert s.loss_offset == s.zero_offset + 4 * nm.meta["loss"].offset
    assert nm.meta["input_batch"] == 16 and s.n_loss_first == len(nm.forward) - 2
    assert [op.kind for op in nm.forward[s.n_loss_first:]] == ["mix_labels", "softmax_ce"]


@pytest.mark.skipif(__import__("torch").cuda.is_available(), reason="checks the no-GPU failure mode")
def test_native_runtime_has_no_cpu_path():
    with pytest.raises(_lib.AcnnError):
        native.NativeRuntime(native.NativeModel(ModelConfig(resnet_size=50), 1, 64, 64, training=False))


def build_c_host(tmp_path):
    """gcc (no nvcc, no torch) builds tests/c_host/acnn_host.c against include/acnn_model.h."""
    import shutil
    import subprocess
    if not shutil.which("gcc") or not os.path.exists("/usr/local/cuda/include/cuda_runtime_api.h"):
        pytest.skip("gcc / CUDA headers not available")
    native.lib()
    libdir = os.path.join(ROOT, "assembled_cnn_b200")
    exe = str(tmp_path / "acnn_host")
    cmd = ["gcc", "-std=c99", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
           "-I", "/usr/local/cuda/include", os.path.join(ROOT, "tests", "c_host", "acnn_host.c"),
           "-o", exe, "-L", libdir, "-l:libacnn.so", "-L", "/usr/local/cuda/lib64", "-lcudart", "-lm",
           "-Wl,-rpath," + libdir, "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_plain_c_host_builds_the_plan(tmp_path):
    """The header is C (not C++), and a C program gets the same plan without Python or a GPU."""
    import subprocess
    exe = build_c_host(tmp_path)
    r = subprocess.run([exe, "plan"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    nm = native.NativeModel(ModelConfig(**ASSEMBLE), 8, 64, 64, training=True, mixup_type=1,
                            label_smoothing=0.1)
    s = nm.sizes
    assert "plan: %d variables (first resnet_model/stage0/conv2d/kernel), %d parameters" % (
        s.n_variables, s.param_elems) in r.stdout, r.stdout
    assert "%d+%d+%d ops" % (s.n_forward, s.n_backward, s.n_update) in r.stdout


def test_variable_pack_unpack_match_runtime_layouts():
    """acnn_variable_pack / _unpack (TF checkpoint layout <-> flat-buffer layout, host arrays) against
    the layout code of the Python side (oracle.plan_interp set_weights / get_tf share it with
    native.NativeRuntime.set_tf): HWIO -> OHWI kernels, [in,out] -> padded [ld][in] dense, padded bias."""
    import numpy as np
    import torch
    from oracle import plan_interp as PI
    flags = dict(ASSEMBLE, pool_type="gem", embedding_size=64, num_classes=10)
    nm = native.NativeModel(ModelConfig(**flags), 2, 64, 64, training=True)
    py = nm.python_mirror()
    it = PI.PlanInterpreter(py, dtype=torch.float32)
    g = torch.Generator().manual_seed(0)
    vals = {n: torch.randn(p.tf_shape, generator=g)
            for n, p in list(py.params.items()) + list(py.state.items())}
    it.set_weights(vals)
    l, vi = nm.lib, native.VariableInfo()
    kinds = set()
    for i in range(nm.sizes.n_variables):
        assert l.acnn_variable_info_get(nm.handle, i, C.byref(vi)) == 0
        name = vi.name.decode()
        tf = np.ascontiguousarray(vals[name].numpy())
        stored = np.full(vi.size, np.nan, dtype=np.float32)
        assert l.acnn_variable_pack(nm.handle, i, tf.ctypes.data_as(C.c_void_p),
                                    stored.ctypes.data_as(C.c_void_p)) == 0
        flat = (it.params if vi.buffer == 0 else it.state)[vi.offset:vi.offset + vi.size].numpy()
        assert np.array_equal(stored, flat), name
        back = np.empty_like(tf)
        assert l.acnn_variable_unpack(nm.handle, i, stored.ctypes.data_as(C.c_void_p),
                                      back.ctypes.data_as(C.c_void_p)) == 0
        assert np.array_equal(back, tf), name
        kinds.add(vi.kind.decode())
    assert kinds == {"conv_kernel", "dense_kernel", "dense_bias", "gamma", "beta", "moving_mean",
                     "moving_variance"}


# --------------------------------------------------------------------------------------------------
# Property test over the flag space: for ANY flag combination the two plan builders either both refuse
# or produce the same plan (hypothesis, derandomised: the same examples on every run).
# --------------------------------------------------------------------------------------------------
from hypothesis import given, settings, strategies as st, HealthCheck


@st.composite
def _flag_sets(draw, poisoned=False):
    # poisoned: exactly one value that one of the argument checks refuses
    poison = draw(st.sampled_from(["size", "filter", "pool", "embedding", "width", "db_se", "alpha",
                                   "reflect"])) \
        if poisoned else None
    version = 2 if poison == "alpha" else draw(st.sampled_from([1, 2]))
    size = draw(st.sampled_from([50, 50, 50, 101, 152] + ([200] if version == 1 else [])))
    aa = draw(st.sampled_from(["sconv", "proj"] if poison == "filter" else
                              ["", "sconv", "sconv", "proj", "sconv,proj"]))
    flags = dict(
        resnet_size=draw(st.sampled_from([18, 51] + ([200] if version == 2 else [34]))) if poison == "size"
        else size,
        resnet_version=version,
        use_sk_block=draw(st.booleans()), use_se_block=draw(st.booleans()),
        use_resnet_d=draw(st.booleans()), zero_gamma=draw(st.booleans()),
        no_downsample=draw(st.booleans()), anti_alias_type=aa,
        anti_alias_filter_size=(draw(st.sampled_from([0, 9])) if poison == "filter"
                                else draw(st.sampled_from([1, 2, 3, 3, 4, 5, 7]))),
        pool_type="max" if poison == "pool" else draw(st.sampled_from(["gap", "gap", "gem", "flatten"])),
        # multiples of 32 that are not powers of two fail the batch-norm kernels' channel grouping
        embedding_size=(draw(st.sampled_from([48, 96, 4096])) if poison == "embedding"
                        else draw(st.sampled_from([0, 0, 32, 64, 512]))),
        # bl_alpha = 4 gives the little branches 16 channels: below the tensor-core tile (refused, version 2)
        bl_alpha=4 if poison == "alpha" else draw(st.sampled_from([1, 2])),
        bl_beta=draw(st.sampled_from([1, 2, 4, 8])),
        num_classes=draw(st.sampled_from([1001, 10, 128])),
        bn_momentum=draw(st.sampled_from([0.997, 0.9])))
    training = draw(st.booleans())
    dropblock = poison == "db_se" or (poison != "width" and draw(st.booleans()) and draw(st.booleans()))
    if poison == "db_se":
        flags["use_se_block"], training = True, True
    elif dropblock:
        flags["use_se_block"] = False
    hw = (224, 224) if dropblock else (draw(st.sampled_from([32, 64, 96])),
                                      100 if poison == "width" else draw(st.sampled_from([32, 64])))
    if poison == "reflect":         # 32 px: the last stride-2 blur-pool sees a 2x2 map, REFLECT pad 2 fails
        flags.update(anti_alias_type="sconv", anti_alias_filter_size=5, no_downsample=False)
        hw, dropblock = (32, 32), False
    elif min(hw) == 32 and flags["anti_alias_type"] and flags["anti_alias_filter_size"] > 4 \
            and poison != "filter":
        flags["anti_alias_filter_size"] = 3
    kw = dict(training=training, mixup_type=draw(st.sampled_from([0, 0, 1, 2])),
              label_smoothing=draw(st.sampled_from([0.0, 0.1])), with_loss=draw(st.booleans()),
              dtype=draw(st.sampled_from(["bf16", "bf16", "fp32"])), use_dropblock=dropblock,
              kd_temp=draw(st.sampled_from([0.0, 0.0, 2.0])))
    return flags, draw(st.integers(1, 5)), hw, kw


def _both(case):
    flags, B, (H, W), kw = case
    try:
        py = dump(build_plan(ModelConfig(**flags), B, H, W, **kw))
    except (ValueError, NotImplementedError, KeyError, AssertionError, ZeroDivisionError):
        py = None
    try:
        nm = native.NativeModel(ModelConfig(**flags), B, H, W, **kw)
        cc = nm.dump()
        nm.close()
    except (_lib.AcnnError, ValueError):
        cc = None
    return py, cc


@settings(max_examples=60, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
@given(_flag_sets())
def test_native_and_python_plans_agree_over_the_flag_space(case):
    py, cc = _both(case)
    assert py is not None, ("the Python builder refused a valid flag set", case)
    assert cc is not None, ("acnn_create refused: " + native.lib().acnn_last_error().decode(), case)
    assert py == cc, (case, _diff(py, cc))
    flags, B, (H, W), kw = case
    nm = native.NativeModel(ModelConfig(**flags), B, H, W, **kw)
    nm.validate()                       # ... and every op of it resolves (host side of acnn_bind)
    nm.close()


@settings(max_examples=30, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
@given(_flag_sets(poisoned=True))
def test_native_and_python_plans_refuse_the_same_flag_sets(case):
    py, cc = _both(case)
    assert py is None and cc is None, (case, py is None, cc is None)


def test_op_conv_info_gives_the_algorithmic_flops_of_the_survey():
    """acnn_op_conv_info (what bench.py's roofline reads): geometry of every GEMM op of the library's C3
    plan equals the Python plan's, and the ALGORITHMIC multiply-accumulates add up to the
    34.12 GFLOP per image for the Assemble-ResNet-50 training step (11.45 forward), while the executed
    ones are higher (space-to-depth stem, zero-inserted stride-2 dgrads)."""
    B = 8
    kw = dict(training=True, mixup_type=1, label_smoothing=0.1)
    nm = native.NativeModel(ModelConfig(**ASSEMBLE), B, 224, 224, **kw)
    py = build_plan(ModelConfig(**ASSEMBLE), B, 224, 224, **kw)
    alg = executed = fwd = 0
    n = 0
    for nops, pops in ((nm.forward, py.forward), (nm.backward, py.backward)):
        for nop, pop in zip(nops, pops):
            if nop.kind not in ("conv", "conv_dgrad", "conv_wgrad"):
                continue
            g, macs, aux = nm.conv_info(nop)
            pg = pop.geom
            assert (g.B, g.H, g.W, g.Cin, g.Cout, g.kh, g.kw, g.stride, g.pad_h_lo, g.pad_h_hi, g.pad_w_lo,
                    g.pad_w_hi) == pg.astuple()
            ex = pg.B * pg.Ho * pg.Wo * pg.Cout * pg.kh * pg.kw * pg.Cin
            assert macs == (pop.a.get("alg_macs") or ex)
            assert aux == (pop.a.get("add_src") is not None) + (pop.a.get("mask_src") is not None)
            alg += macs
            executed += ex
            fwd += macs if nop.phase == 0 else 0
            n += 1
    assert n == 230                                           # conv GEMM launches of a step
    gflop = 2.0 * alg / B / 1e9
    assert abs(gflop - 34.12) < 0.15 and abs(2.0 * fwd / B / 1e9 - 11.45) < 0.1, (gflop, fwd)
    assert executed > alg
    # a non-GEMM op is refused with a status code
    import ctypes as C
    g, m, a = _lib.ConvGeom(), C.c_int64(), C.c_int()
    bn = next(op for op in nm.forward if op.kind == "bn_act")
    assert nm.lib.acnn_op_conv_info(nm.handle, 0, bn.index, C.byref(g), C.byref(m), C.byref(a)) == 1
