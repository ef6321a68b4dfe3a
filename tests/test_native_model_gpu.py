"""GPU tests of the model-level C ABI (include/acnn_model.h, csrc/model_plan.cu + model_exec.cu).

The library's executor runs each configuration of CASES op by op in lock-step with the oracle's plan
interpreter (test_plan_gpu.lockstep: after every op its outputs are compared and then overwritten with the
interpreter's) in deterministic mode and, for the bf16 configurations of DEFAULT_MODE_CASES, in the default
mode too, where wgrad and the small SK / SE GEMMs run split-K with ordered reductions.  The whole step
(acnn_step / acnn_forward + acnn_loss) must then be BIT-IDENTICAL to the same ops run one acnn_run_ops call
at a time -- every buffer of the step: logits, loss, every gradient, the updated weights, momentum and
moving statistics.  Plus: the pure C-ABI call sequence with host arrays (acnn_set_inputs ... acnn_get_loss)
against the oracle, piecewise == acnn_step, CUDA-graph capture of acnn_step in both modes, and the Model /
Trainer facade eager == CUDA graph."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ASSEMBLE = dict(resnet_size=50, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                anti_alias_filter_size=3)

CASES = {
    "c3_assemble_mixup1": (ASSEMBLE, 8, 128, dict(training=True, mixup_type=1, label_smoothing=0.1)),
    "c1_vanilla_eval": (dict(resnet_size=50), 2, 224, dict(training=False, with_loss=True)),
    "assemble_fp32_mixup2": (ASSEMBLE, 4, 64, dict(training=True, mixup_type=2, dtype="fp32")),
    "se_proj_resnet_d": (dict(resnet_size=50, resnet_version=2, use_se_block=True, use_resnet_d=True,
                              anti_alias_type="proj", anti_alias_filter_size=5), 4, 64,
                         dict(training=True)),
    "dropblock_kd": (ASSEMBLE, 4, 224, dict(training=True, use_dropblock=True, kd_temp=2.0,
                                            mixup_type=1)),
    "gem_embedding_r1": (dict(resnet_size=50, pool_type="gem", embedding_size=256, zero_gamma=True),
                         4, 64, dict(training=True, label_smoothing=0.1)),
    "c5_r152_topology": (dict(ASSEMBLE, resnet_size=152, bl_alpha=1, bl_beta=2), 4, 64,
                         dict(training=True, mixup_type=1)),
    # B = 64 > 32: the weight-gradient GEMMs of the SK and SE layers (K = batch) split
    "sk_se_b64": (dict(ASSEMBLE, use_se_block=True), 64, 64, dict(training=True, mixup_type=1)),
}
# bf16 configurations also run in the default mode (deterministic=None: split-K on)
DEFAULT_MODE_CASES = ("c3_assemble_mixup1", "se_proj_resnet_d", "c5_r152_topology", "sk_se_b64")


def _weights(plan, seed=5):
    """Random variables in TF layouts (non-trivial BN parameters and statistics)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for n, p in list(plan.params.items()) + list(plan.state.items()):
        if p.kind in ("conv_kernel", "dense_kernel"):
            fan_in = 1
            for d in p.tf_shape[:-1]:
                fan_in *= d
            out[n] = torch.randn(p.tf_shape, generator=g) / fan_in ** 0.5
        elif p.kind in ("gamma", "moving_variance"):
            out[n] = 0.5 + torch.rand(p.tf_shape, generator=g)
        else:
            out[n] = 0.1 * torch.randn(p.tf_shape, generator=g)
    return out


def _feeds(plan, seed=9):
    g = torch.Generator().manual_seed(seed)
    m = plan.meta
    Bin, H, W = m["input_batch"], m["height"], m["width"]
    f = {m["images"]: (torch.randn(Bin, H, W, 3, generator=g) * 64).clamp(-124, 152)}
    if "labels" in m:
        f[m["labels"]] = torch.randint(1, m["num_classes"], (Bin,), generator=g).int()
    for k in ("lam1", "lam2"):
        if k in m:
            f[m[k]] = torch.rand(Bin // 2, generator=g)
    for name in m.get("dropblock_u", []):
        f[name] = torch.rand(plan.tensors[name].shape, generator=g)
    if "teacher_logits" in m:
        f[m["teacher_logits"]] = 3.0 * torch.randn(Bin, m["num_classes"], generator=g)
    return f


def _pair(flags, B, hw, kw, deterministic=True):
    """Two NativeRuntimes of one configuration, each on its own NativeModel, with the same weights,
    hyper-parameters and inputs.  Returns (model of the first, first, second)."""
    from assembled_cnn_b200 import native
    from assembled_cnn_b200.plan import ModelConfig
    cfg = ModelConfig(**flags)
    rts = []
    for _ in range(2):
        nm = native.NativeModel(cfg, B, hw, hw, deterministic=deterministic, **kw)
        rt = native.NativeRuntime(nm)
        rt.set_weights(_weights(nm))
        rt.set_hparams(lr=0.05, momentum=0.9, weight_decay=1e-4, keep_prob=0.9, step=3)
        rt.dropblock_feed = True
        for name, v in _feeds(nm).items():
            rt.t[name].copy_(v)
        rts.append(rt)
    return rts[0].plan, rts[0], rts[1]


def _assert_same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    if not torch.equal(a, b):
        d = (a.double() - b.double()).abs()
        raise AssertionError("%s differs: %d of %d elements, max |d| %.3e" % (
            what, int((d > 0).sum()), d.numel(), float(d.max())))


def lockstep_case(case, deterministic, dtype=None, loss_scale=1.0):
    """test_plan_gpu.lockstep on the configuration CASES[case] (its batch, size and flags; dtype overrides
    its dtype, loss_scale applies to training).  Returns (failures, worst error per op kind:output)."""
    import test_plan_gpu as P
    flags, B, hw, kw = CASES[case]
    flags, kw = dict(flags), dict(kw)
    use_resnet_d = flags.pop("use_resnet_d", False)
    training = kw.pop("training", True)
    case_dtype = kw.pop("dtype", "bf16")
    assert kw.pop("with_loss", True), "lockstep runs the loss"
    args = dict(B=B, HW=hw, training=training, mix=kw.pop("mixup_type", 0),
                label_smoothing=kw.pop("label_smoothing", 0.0), dtype=dtype or case_dtype,
                use_dropblock=kw.pop("use_dropblock", False), kd_temp=kw.pop("kd_temp", 0.0),
                loss_scale=loss_scale if training else 1.0, deterministic=deterministic)
    assert not kw, kw
    return P.lockstep(flags, use_resnet_d, **args)


@pytest.mark.parametrize("case", sorted(CASES))
def test_lockstep_against_interpreter(case):
    failures, _ = lockstep_case(case, deterministic=True)
    assert not failures, "\n".join(failures[:20])


@pytest.mark.parametrize("case", DEFAULT_MODE_CASES)
def test_lockstep_against_interpreter_default_mode(case):
    """The bf16 configurations with deterministic=None: wgrad and the SK / SE GEMMs run split-K."""
    failures, _ = lockstep_case(case, deterministic=None)
    assert not failures, "\n".join(failures[:20])


def step_equals_op_by_op(case, deterministic, dtype=None, same=_assert_same):
    """Two steps of CASES[case] (dtype overriding its dtype): run_step / run_forward on one runtime, the
    same ops one rt.run([op]) at a time after zero_step_buffers on another; every tensor, the zero buffer,
    the moving statistics, weights, gradients and momentum compared with `same` after each step.
    Returns (plan, the runtime that ran whole steps, the loss after the first step)."""
    flags, B, hw, kw = CASES[case]
    if dtype is not None:
        kw = dict(kw, dtype=dtype)
    plan, rt_step, rt_ops = _pair(flags, B, hw, kw, deterministic)
    assert rt_step.det == (1 if deterministic else int(kw.get("dtype") == "fp32"))
    training = kw.get("training", True)
    ops = plan.all_ops() if training else plan.forward
    loss0 = None
    for step in range(2):
        if training:
            rt_step.run_step()
        else:
            rt_step.run_forward()
        rt_ops.zero_step_buffers()
        for op in ops:
            rt_ops.run([op])
        torch.cuda.synchronize()
        if step == 0:
            loss0 = rt_step.slot_view(plan.meta["loss"]).clone()
        for name in plan.tensors:      # every activation, gradient and input buffer of the step
            same(rt_step.t[name], rt_ops.t[name], "%s step %d tensor %s" % (case, step, name))
        same(rt_step.zero, rt_ops.zero, "zero buffer (loss, stem dW)")
        same(rt_step.state, rt_ops.state, "moving statistics")
        same(rt_step.params, rt_ops.params, "weights")
        if training:
            same(rt_step.grads, rt_ops.grads, "gradients")
            same(rt_step.momentum, rt_ops.momentum, "momentum")
    return plan, rt_step, loss0


@pytest.mark.parametrize("case", sorted(CASES))
def test_step_bit_identical_to_op_by_op(case):
    _step_bit_identical(case, deterministic=True)


@pytest.mark.parametrize("case", DEFAULT_MODE_CASES)
def test_step_bit_identical_to_op_by_op_default_mode(case):
    """The bf16 configurations with deterministic=None: wgrad and the SK / SE GEMMs run split-K."""
    _step_bit_identical(case, deterministic=None)


def _step_bit_identical(case, deterministic):
    plan, rt, _ = step_equals_op_by_op(case, deterministic)
    loss = rt.slot_view(plan.meta["loss"])
    assert torch.isfinite(loss).all() and float(loss[0]) > 0
    if CASES[case][3].get("training", True):
        assert float(rt.grads.abs().sum()) > 0 and float(loss[1]) > 0


def test_c_abi_call_sequence_with_host_arrays_against_oracle():
    """The sequence a C host runs -- create, sizes, bind, set_inputs / set_hparams from HOST arrays,
    step, get_logits / get_loss into HOST arrays -- with nothing but pointers crossing the boundary,
    checked against the CPU oracle (same-rounding plan interpreter): loss within 2 %, L2 1e-4."""
    from assembled_cnn_b200 import _lib, native
    from assembled_cnn_b200.plan import ModelConfig
    from oracle import plan_interp as PI
    B, hw = 8, 64
    cfg = ModelConfig(**ASSEMBLE)
    nm = native.NativeModel(cfg, B, hw, hw, training=True, mixup_type=1, label_smoothing=0.1)
    l, h, s = nm.lib, nm.handle, nm.sizes
    dev = torch.device("cuda:0")
    f32 = dict(dtype=torch.float32, device=dev)
    params, grads, mom = (torch.zeros(s.param_elems, **f32) for _ in range(3))
    state = torch.zeros(s.state_elems, **f32)
    wf = torch.zeros(s.w_fprop_elems, dtype=torch.bfloat16, device=dev)
    wd = torch.zeros(s.w_dgrad_elems, dtype=torch.bfloat16, device=dev)
    ws = torch.empty(s.workspace_bytes, dtype=torch.uint8, device=dev).fill_(0xAB)   # bind clears it
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(l.acnn_bind(h, params.data_ptr(), grads.data_ptr(), mom.data_ptr(), state.data_ptr(),
                           wf.data_ptr(), wd.data_ptr(), ws.data_ptr(), st), "acnn_bind")
    # variables: through the Python mirror's layout helpers (a C host would fill OHWI itself)
    pyplan = nm.python_mirror()
    it = PI.PlanInterpreter(pyplan, dtype=torch.float32, emulate_bf16=True)
    w = _weights(pyplan)
    it.set_weights(w)
    params.copy_(it.params.float())
    state.copy_(it.state.float())
    params0 = params.clone()
    feeds = _feeds(pyplan)
    m = pyplan.meta
    x = feeds[m["images"]].numpy()
    lab = feeds[m["labels"]].numpy()
    lam = feeds[m["lam1"]].numpy()
    hp = np.array([0.05, 0.9, 1e-4, 1.0, 1.0, 0, 0, 0], dtype=np.float32)
    as_p = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(l.acnn_set_inputs(h, as_p(x), as_p(lab), as_p(lam), None, None, st), "acnn_set_inputs")
    _lib.check(l.acnn_set_hparams(h, as_p(hp), st), "acnn_set_hparams")
    _lib.check(l.acnn_step(h, st), "acnn_step")
    logits = np.empty((B, 1001), dtype=np.float32)
    loss = np.empty(4, dtype=np.float32)
    _lib.check(l.acnn_get_logits(h, as_p(logits), st), "acnn_get_logits")
    _lib.check(l.acnn_get_loss(h, as_p(loss), st), "acnn_get_loss")
    torch.cuda.synchronize()
    it.hp.update(lr=0.05, momentum=0.9, weight_decay=1e-4)
    lg, ce, l2 = it.train_step(feeds[m["images"]], feeds[m["labels"]], feeds[m["lam1"]])
    print("C-ABI step: CE %.5f (oracle %.5f), L2 %.6f (oracle %.6f)" % (loss[0], ce, loss[1], l2))
    assert np.isfinite(logits).all() and np.isfinite(loss).all()
    assert abs(loss[0] - ce) < 2e-2 * abs(ce)
    assert abs(loss[1] - l2) < 1e-4 * abs(l2)
    assert float(grads.abs().sum()) > 0 and not torch.equal(params, params0)
    # errors come back as status codes + text, never exceptions / aborts
    assert l.acnn_run_ops(h, 1, 0, 10 ** 6, st) == 1 and b"range" in l.acnn_last_error()
    assert l.acnn_set_inputs(h, None, None, None, as_p(lam), None, st) == 1      # no lam2 input here
    nm2 = native.NativeModel(cfg, 2, 64, 64, training=False)
    assert l.acnn_forward(nm2.handle, st) == 1 and b"not bound" in l.acnn_last_error()


def test_piecewise_equals_step_and_graph_replay():
    """acnn_forward + acnn_loss + acnn_backward_range (3 segments) + acnn_sgd_step == acnn_step, eager
    == CUDA-graph replay of acnn_step; all bit-identical (deterministic mode)."""
    _piecewise_step_graph(deterministic=True)


def test_piecewise_equals_step_and_graph_replay_default_mode():
    """The same in the default mode (deterministic=None: split-K wgrad and SK / SE GEMMs)."""
    _piecewise_step_graph(deterministic=None)


def _piecewise_step_graph(deterministic):
    from assembled_cnn_b200 import _lib, native
    from assembled_cnn_b200.plan import ModelConfig
    cfg = ModelConfig(**ASSEMBLE)
    kw = dict(training=True, mixup_type=1, label_smoothing=0.1, deterministic=deterministic)
    outs = []
    for mode in ("step", "piecewise", "graph"):
        nm = native.NativeModel(cfg, 4, 64, 64, **kw)
        rt = native.NativeRuntime(nm)
        rt.set_weights(_weights(nm))
        rt.set_hparams(lr=0.05, momentum=0.9, weight_decay=1e-4)
        for name, v in _feeds(nm).items():
            rt.t[name].copy_(v)
        l, h = nm.lib, nm.handle
        if mode == "graph":
            rt.capture(train=True)       # warm-up free: bind resolved every launch record
        for _ in range(2):
            st = rt.stream
            if mode == "step":
                _lib.check(l.acnn_step(h, st), "step")
            elif mode == "graph":
                rt.graph.replay()
            else:
                n = nm.sizes.n_backward
                _lib.check(l.acnn_forward(h, st), "forward")
                _lib.check(l.acnn_loss(h, st), "loss")
                for a, b in ((0, n // 3), (n // 3, n // 2), (n // 2, n)):
                    _lib.check(l.acnn_backward_range(h, a, b, st), "backward_range")
                _lib.check(l.acnn_sgd_step(h, st), "sgd_step")
        torch.cuda.synchronize()
        outs.append((rt.params.clone(), rt.grads.clone(), rt.state.clone(), rt.momentum.clone(),
                     rt.slot_view(nm.meta["loss"]).clone()))
    for other in outs[1:]:
        for a, b, what in zip(outs[0], other, ("weights", "gradients", "moving statistics",
                                               "momentum", "loss")):
            _assert_same(a, b, what)


def test_model_facade_runs_on_the_native_path():
    """Model / Trainer run on the library's executor, and a Trainer that replays its step as a CUDA graph
    gives the eager Trainer's losses, weights, moving statistics and eval logits bit for bit."""
    from assembled_cnn_b200.hparams import params_from_flags
    from assembled_cnn_b200.model_fns import Model, Trainer
    from assembled_cnn_b200.native import NativeRuntime
    B, hw = 8, 64
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(2 * B, hw, hw, 3, generator=g) * 64).clamp(-124, 152)
    lab = torch.randint(1, 1001, (2 * B,), generator=g).int()
    lam = torch.rand(B, generator=g)
    res = []
    for use_graph in (False, True):
        model = Model(50, num_classes=1001, resnet_version=2, use_sk_block=True, anti_alias_type="sconv",
                      anti_alias_filter_size=3, seed=42, deterministic=True)
        p = params_from_flags(batch_size=B, mixup_type=1, label_smoothing=0.1, weight_decay=1e-4,
                              base_learning_rate=0.05, learning_rate_decay_type="fixed", **ASSEMBLE)
        tr = Trainer(model, p, hw, hw, use_cuda_graph=use_graph)
        assert isinstance(tr.rt, NativeRuntime) and tr.use_graph == use_graph
        losses = [tr.train_step(x, lab, lam1=lam).clone() for _ in range(2)]
        ev = model(x[:B], training=False).clone()
        torch.cuda.synchronize()
        res.append((losses[0], losses[1], tr.rt.params.clone(), tr.rt.state.clone(), ev))
    for a, b, what in zip(res[0], res[1], ("loss 1", "loss 2", "weights", "moving statistics",
                                            "eval logits")):
        _assert_same(a, b, what)


def test_plain_c_host_trains(tmp_path):
    """tests/c_host/acnn_host.c: cudaMalloc'd buffers, host-drawn initializers, host input arrays, three
    acnn_step calls -- finite, plausible losses and weights that move (the numbers of this call sequence
    are checked against the oracle in test_c_abi_call_sequence_with_host_arrays_against_oracle)."""
    import subprocess
    from test_native_plan_cpu import build_c_host
    exe = build_c_host(tmp_path)
    r = subprocess.run([exe, "step"], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), (r.returncode, r.stdout, r.stderr)
