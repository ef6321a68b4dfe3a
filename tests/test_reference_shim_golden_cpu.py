"""The oracle against golden vectors produced by RUNNING THE REFERENCE'S OWN MODEL CODE
(nets/resnet_model.py + nets/blocks.py + nets/model_helper.py) through a TF-1.14 API stand-in
(tests/golden/tf1_shim, generator tests/golden/make_reference_shim_golden.py, run against a checkout
of the original project -- this test only reads the committed json).

Pinned: variable names / shapes / initializer kinds / creation order of 9 model configurations
(including the Assemble-ResNet-50 of the north star, ResNet-D, SE, proj anti-alias, zero-gamma, R101,
R152; the product plan is checked against the same inventories), which of them enter the weight-decay term (nets/run_loop_classification.py:163-176), the
logits + updated BN moving statistics for seeded inputs and seeded variable values in inference and
in training mode, the loss and its gradients (torch autograd through the reference's graph,
inference-mode BN), mixup types 1 / 2 (utils/data_util.py:97-158), the softmax cross entropy with label
smoothing (losses/cls_losses.py) and the five learning-rate schedules (functions/model_fns.py:36-95).

The stand-in's kernels are not the oracle's: it does not import oracle/ ('SAME' padding by Hugging Face's
port of the TF BiT checkpoints, batch norm / convolution / pooling by ATen) and computes in float64, so a
golden number is "the reference's Python on independent kernels without rounding noise"; the fp32 oracle
is held to the tolerances of the individual tests and the float64 oracle to 1e-6 on everything
(test_float64_oracle_matches_reference_code_to_1e6)."""
import hashlib
import importlib.util
import json
import os

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location(
    "make_reference_shim_golden", os.path.join(HERE, "golden", "make_reference_shim_golden.py"))
mg = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mg)
GOLD = json.load(open(os.path.join(HERE, "golden", "reference_shim_golden.json")))
PIECES = GOLD["train_pieces"]

KIND = {"conv_kernel": "variance_scaling", "dense_kernel": "glorot_uniform", "dense_bias": "zeros",
        "beta": "zeros", "moving_mean": "zeros", "moving_variance": "ones"}


def _oracle(flags, use_resnet_d, size):
    from oracle import model as M
    model, vs = M.build(seed=1, input_hw=size, use_resnet_d=use_resnet_d, **flags)
    return M, model, vs


def _close(a, b, rel, abs_=1e-6):
    return abs(a - b) <= max(rel * max(abs(a), abs(b)), abs_)


@pytest.mark.parametrize("name", sorted(mg.CONFIGS))
def test_variable_inventory_matches_reference_code(name):
    flags, d, batch, size = mg.CONFIGS[name]
    gold = GOLD[name]
    _, _, vs = _oracle(flags, d, size)
    names = list(vs.vars)
    assert len(names) == gold["num_variables"]
    assert names[:3] == gold["first_names"] and names[-2:] == gold["last_names"]
    h = hashlib.sha256()
    zero_gammas = 0
    for n in names:
        kind = vs.kind[n]
        init = KIND.get(kind)
        if kind == "gamma":
            init = "zeros" if float(vs.vars[n].abs().sum()) == 0.0 else "ones"
            zero_gammas += init == "zeros"
        h.update(("%s|%s|%s|%d\n" % (n, ",".join(map(str, vs.vars[n].shape)), init,
                                     bool(vs.trainable[n]))).encode())
    assert zero_gammas == gold["zero_init_gammas"]
    assert h.hexdigest() == gold["names_sha256"]
    # the variables that enter the weight-decay term (run_loop_classification.py:163-176)
    from oracle import model as M
    decayed = [n for n in names if vs.trainable[n] and M.decayed(n)]
    assert len(decayed) == gold["num_decayed"]
    assert hashlib.sha256("\n".join(decayed).encode()).hexdigest() == gold["decayed_sha256"]


@pytest.mark.parametrize("name", [n for n in sorted(mg.CONFIGS) if "152" not in n and "101" not in n])
def test_forward_matches_reference_code(name):
    flags, d, batch, size = mg.CONFIGS[name]
    gold = GOLD[name]
    M, model, vs = _oracle(flags, d, size)
    for i, n in enumerate(list(vs.vars)):
        vs.vars[n] = mg.seeded_value(i, n, tuple(vs.vars[n].shape))
    x = mg.seeded_input(batch, size)
    with torch.no_grad():
        y = M.forward(model, vs, x, training=False, use_resnet_d=d)
    got = mg.digest(y)
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(got[k], gold["eval_logits"][k], 2e-4, 1e-4), (k, got[k], gold["eval_logits"][k])
    for a, b in zip(y[0, :8].tolist(), gold["eval_logits_row0_head"]):
        assert _close(a, b, 2e-4, 1e-4)
    # gradients of loss = smoothed CE + 1e-4 * L2 (inference-mode BN) through the reference's graph
    for n in vs.vars:
        vs.vars[n].requires_grad_(bool(vs.trainable[n]))
    lab = torch.nn.functional.one_hot(torch.arange(batch) * 37 % 1001, 1001).float()
    loss, _, _, _ = M.loss_fn(model, vs, x, lab, training=False, use_resnet_d=d, label_smoothing=0.1,
                              weight_decay=1e-4)
    loss.backward()
    assert _close(float(loss.detach()), gold["loss_eval_mode"], 1e-5)
    for n, want in gold["grads_eval_mode"].items():
        got = mg.digest(vs.vars[n].grad)
        assert _close(got["abs_sum"], want["abs_sum"], 2e-3, 1e-7), (n, got, want)
        assert _close(got["sum"], want["sum"], 2e-3, 1e-3 * want["abs_sum"] + 1e-7), (n, got, want)
    for n in vs.vars:
        vs.vars[n] = vs.vars[n].detach()
    # training mode: batch statistics + moving-average updates (UPDATE_OPS)
    with torch.no_grad():
        y = M.forward(model, vs, x, training=True, use_resnet_d=d)
    got = mg.digest(y)
    assert _close(got["abs_sum"], gold["train_logits"]["abs_sum"], 5e-3), (got, gold["train_logits"])
    after = dict(vs.vars)
    after.update(model.bn_updates)          # the UPDATE_OPS of this step
    mm = torch.cat([after[n].flatten() for n in vs.vars if n.endswith("moving_mean")])
    mv = torch.cat([after[n].flatten() for n in vs.vars if n.endswith("moving_variance")])
    for k in ("sum", "abs_sum"):
        assert _close(mg.digest(mm)[k], gold["moving_mean_after"][k], 1e-4)
        assert _close(mg.digest(mv)[k], gold["moving_variance_after"][k], 1e-4)


@pytest.mark.parametrize("name", sorted(mg.CONFIGS))
def test_float64_oracle_matches_reference_code_to_1e6(name):
    """The golden numbers are float64 results of the reference's model code run on kernels that are not
    the oracle's (Hugging Face's TF-'SAME' padding port, ATen's batch norm / convolution / pooling).  In
    float64 nothing is left of the summation-order noise that training-mode statistics over a batch of 2
    amplify, so the oracle must agree to 1e-6 on EVERYTHING, all 11 configurations up to ResNet-152:
    inference- and training-mode logits (sum, |sum|, first, last, head of row 0), the moving statistics
    after the step, the loss and the gradient digests.  A different padding side, variance estimator,
    epsilon placement, pooling divisor or block order shows up here at 1e-2 .. 1."""
    flags, d, batch, size = mg.CONFIGS[name]
    gold = GOLD[name]
    M, model, vs = _oracle(flags, d, size)
    for i, n in enumerate(list(vs.vars)):
        vs.vars[n] = mg.seeded_value(i, n, tuple(vs.vars[n].shape)).double()
    vs.dtype = torch.float64
    x = mg.seeded_input(batch, size).double()
    tight = lambda a, b: _close(a, b, 1e-6, 1e-9)
    with torch.no_grad():
        y = M.forward(model, vs, x, training=False, use_resnet_d=d)
    assert y.dtype == torch.float64
    got = mg.digest(y)
    for k in ("sum", "abs_sum", "first", "last"):
        assert tight(got[k], gold["eval_logits"][k]), (k, got[k], gold["eval_logits"][k])
    for a, b in zip(y[0, :8].tolist(), gold["eval_logits_row0_head"]):
        assert tight(a, b)
    if "grads_eval_mode" in gold:
        for n in vs.vars:
            vs.vars[n].requires_grad_(bool(vs.trainable[n]))
        lab = torch.nn.functional.one_hot(torch.arange(batch) * 37 % 1001, 1001).double()
        loss, _, _, _ = M.loss_fn(model, vs, x, lab, training=False, use_resnet_d=d, label_smoothing=0.1,
                                  weight_decay=1e-4)
        loss.backward()
        # the loss function of the oracle computes the cross-entropy in fp32 (as TF does): 1e-6 there
        assert _close(float(loss.detach()), gold["loss_eval_mode"], 2e-6)
        for n, want in gold["grads_eval_mode"].items():
            g = mg.digest(vs.vars[n].grad)
            assert _close(g["abs_sum"], want["abs_sum"], 1e-5, 1e-10), (n, g, want)
            assert _close(g["sum"], want["sum"], 1e-5, 1e-5 * want["abs_sum"] + 1e-10), (n, g, want)
        for n in vs.vars:
            vs.vars[n] = vs.vars[n].detach()
    with torch.no_grad():
        y = M.forward(model, vs, x, training=True, use_resnet_d=d)
    got = mg.digest(y)
    for k in ("sum", "abs_sum", "first", "last"):
        assert tight(got[k], gold["train_logits"][k]), (k, got[k], gold["train_logits"][k])
    after = dict(vs.vars)
    after.update(model.bn_updates)
    mm = torch.cat([after[n].flatten() for n in vs.vars if n.endswith("moving_mean")])
    mv = torch.cat([after[n].flatten() for n in vs.vars if n.endswith("moving_variance")])
    for k in ("sum", "abs_sum", "first", "last"):
        assert tight(mg.digest(mm)[k], gold["moving_mean_after"][k]), k
        assert tight(mg.digest(mv)[k], gold["moving_variance_after"][k]), k


# (one of the two 152-layer configurations -- BASELINE config 5 -- is enough for the interpreter tests: the
# float64 interpretation of a 152-layer plan takes ~25 s)
_INTERP_CONFIGS = [n for n in sorted(mg.CONFIGS) if n != "assemble_r152_rv2_sk_sconv"]


@pytest.mark.parametrize("name", _INTERP_CONFIGS)
def test_product_plan_interpreted_in_float64_matches_reference_code(name):
    """One hop fewer: the PRODUCT'S layer plan (assembled_cnn_b200/plan.py -- text-for-text the plan the
    library builds, tests/test_native_plan_cpu.py), executed op by op by the float64 interpreter the GPU
    lockstep tests compare every CUDA op with (oracle/plan_interp.py), against the float64 results of the
    reference's own model code on third-party kernels: inference-mode logits, training-mode logits and the
    moving statistics after the step to 1e-6, 10 configurations up to ResNet-152 (fp32-mode plan: fp32 tensors, two-pass
    statistics, operand planes)."""
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    from oracle import plan_interp as PI
    flags, d, batch, size = mg.CONFIGS[name]
    gold = GOLD[name]
    cfg = ModelConfig(use_resnet_d=d, **flags)
    x = mg.seeded_input(batch, size).double()
    values = None
    for training in (False, True):
        plan = build_plan(cfg, batch, size, size, training=training, with_loss=False, dtype="fp32")
        if values is None:
            names = list(plan.params) + list(plan.state)
            # the seeded values are indexed by the reference's creation order (trainables and moving
            # statistics interleaved): recover it from the oracle's variable store
            _, _, vs = _oracle(flags, d, size)
            values = {n: mg.seeded_value(i, n, tuple(vs.vars[n].shape)).double()
                      for i, n in enumerate(list(vs.vars))}
            assert sorted(values) == sorted(names)
        it = PI.PlanInterpreter(plan, dtype=torch.float64)
        it.set_weights(values)
        labels = torch.zeros(batch, dtype=torch.int32) if training else None
        y = it.forward(x, labels)
        got = mg.digest(y)
        want = gold["train_logits" if training else "eval_logits"]
        for k in ("sum", "abs_sum", "first", "last"):
            assert _close(got[k], want[k], 1e-6, 1e-9), (training, k, got[k], want[k])
        if training:
            mm = torch.cat([it.get_tf(n).flatten() for n in values if n.endswith("moving_mean")])
            mv = torch.cat([it.get_tf(n).flatten() for n in values if n.endswith("moving_variance")])
            for k in ("sum", "abs_sum", "first", "last"):
                assert _close(mg.digest(mm)[k], gold["moving_mean_after"][k], 1e-6, 1e-9), k
                assert _close(mg.digest(mv)[k], gold["moving_variance_after"][k], 1e-6, 1e-9), k
        else:
            for a, b in zip(y[0, :8].tolist(), gold["eval_logits_row0_head"]):
                assert _close(a, b, 1e-6, 1e-9)


@pytest.mark.parametrize("name", _INTERP_CONFIGS)
def test_product_plan_backward_in_float64_matches_autograd_through_reference_code(name):
    """The plan's EXPLICIT backward (the reference relies on tf.gradients; the product emits hand-derived
    batch-norm / SK / SE / blur-pool / pooling / merge backward passes and accumulates gradients through
    fused epilogues) executed by the float64 interpreter, against torch autograd through the reference's
    own training-mode graph on third-party kernels: the smoothed cross-entropy to 1e-6 and the gradient
    digests of 10-23 variables spread over the net (stem, BL module, SK / SE fc kernels, BN gammas / betas,
    dense kernel and bias) to 1e-5."""
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    from oracle import plan_interp as PI
    flags, d, batch, size = mg.CONFIGS[name]
    gold = GOLD[name]
    plan = build_plan(ModelConfig(use_resnet_d=d, **flags), batch, size, size, training=True,
                      label_smoothing=0.1, dtype="fp32")
    _, _, vs = _oracle(flags, d, size)
    values = {n: mg.seeded_value(i, n, tuple(vs.vars[n].shape)).double() for i, n in enumerate(list(vs.vars))}
    it = PI.PlanInterpreter(plan, dtype=torch.float64)
    it.set_weights(values)
    it.hp.update(grad_scale=1.0)
    labels = (torch.arange(batch) * 37 % 1001).int()
    it.forward(mg.seeded_input(batch, size).double(), labels)
    it.run(plan.backward)
    ce = float(it.slot(plan.meta["loss"])[0])
    assert _close(ce, gold["ce_train_mode"], 2e-6), (ce, gold["ce_train_mode"])
    worst = 0.0
    for n, want in gold["grads_train_mode"].items():
        g = mg.digest(it.get_tf(n, it.grads))
        assert _close(g["abs_sum"], want["abs_sum"], 1e-5, 1e-12), (n, g, want)
        assert _close(g["sum"], want["sum"], 1e-5, 1e-5 * want["abs_sum"] + 1e-12), (n, g, want)
        assert _close(g["first"], want["first"], 1e-5, 1e-6 * want["abs_sum"] + 1e-12), (n, g, want)
        worst = max(worst, abs(g["abs_sum"] - want["abs_sum"]) / max(want["abs_sum"], 1e-30))
    print("%s: %d gradient tensors, worst |sum| rel diff %.2e" % (name, len(gold["grads_train_mode"]), worst))


@pytest.mark.parametrize("name", sorted(mg.DROPBLOCK_CONFIGS))
def test_product_dropblock_plan_in_float64_matches_reference_code(name):
    """The product's DropBlock plan (mask ops at the reference's 34 / 29 call sites, `cbr_db` /
    `residual_tail_db` tails, SK-output DropBlock) interpreted in float64 with the SAME uniform draws in
    call order, against the reference's Model.__call__(training=True, keep_prob) on third-party kernels:
    training-mode logits at 224 px to 1e-5."""
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    from oracle import model as M, plan_interp as PI
    flags, batch, size, kp = mg.DROPBLOCK_CONFIGS[name]
    gold = GOLD[name]
    plan = build_plan(ModelConfig(**flags), batch, size, size, training=True, use_dropblock=True,
                      dtype="fp32")
    _, vs = M.build(seed=1, input_hw=64, **flags)
    values = {n: mg.seeded_value(i, n, tuple(vs.vars[n].shape)).double() for i, n in enumerate(list(vs.vars))}
    it = PI.PlanInterpreter(plan, dtype=torch.float64)
    it.set_weights(values)
    it.hp.update(keep_prob=kp)
    g = torch.Generator().manual_seed(mg.DROPBLOCK_SEED)
    assert len(plan.meta["dropblock_u"]) == gold["num_dropblock_calls"]
    for u_name in plan.meta["dropblock_u"]:          # the reference draws [1, hs, ws, C] per call, in order
        shape = plan.tensors[u_name].shape
        it.t[u_name] = torch.rand((1,) + tuple(shape), generator=g)[0].double()
    y = it.forward(mg.seeded_input(batch, size).double(), torch.zeros(batch, dtype=torch.int32))
    got = mg.digest(y)
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(got[k], gold["train_logits"][k], 1e-5, 1e-8), (k, got[k], gold["train_logits"][k])
    for a, b in zip(y[0, :8].tolist(), gold["train_logits_row0_head"]):
        assert _close(a, b, 1e-5, 1e-8)


def test_c3_composition_matches_reference_code():
    """BASELINE config 3 end to end as the reference composes it -- utils/data_util.mixup (type 1) ->
    Assemble-ResNet-50 in training mode -> get_sup_loss(label_smoothing 0.1) -> gradients -- executed from
    the reference's sources on third-party kernels in float64, against (a) the float64 oracle and (b) the
    PRODUCT'S plan (mixup fused into pack_input / mix_labels, explicit backward) in the float64
    interpreter: training-mode logits and the loss to 1e-6, 14 gradient digests to 1e-5."""
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    from oracle import model as M, plan_interp as PI, tf_ops as T
    gold = GOLD["c3_composition"]
    flags, d, _, _ = mg.CONFIGS["assemble_r50_rv2_sk_sconv"]
    B, size = gold["batch"], gold["size"]
    x, labels, lam = mg.c3_inputs()
    model, vs = M.build(seed=1, input_hw=size, **flags)
    values = {n: mg.seeded_value(i, n, tuple(vs.vars[n].shape)).double() for i, n in enumerate(list(vs.vars))}
    # (a) oracle
    for n in vs.vars:
        vs.vars[n] = values[n].clone().requires_grad_(bool(vs.trainable[n]))
    vs.dtype = torch.float64
    onehot = torch.nn.functional.one_hot(labels, 1001).double()
    mx, my = T.mixup(x.double(), onehot, lam.double(), keep_batch_size=False)
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(mg.digest(mx)[k], gold["mixed_images"][k], 1e-9)
        assert _close(mg.digest(my)[k], gold["mixed_labels"][k], 1e-9)
    loss, ce, _, y = M.loss_fn(model, vs, mx, my, training=True, label_smoothing=0.1, weight_decay=0.0)
    ce.backward()
    assert _close(float(ce.detach()), gold["cross_entropy"], 2e-6)
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(mg.digest(y)[k], gold["train_logits"][k], 1e-6, 1e-9), k
    for n, want in gold["grads"].items():
        g = mg.digest(vs.vars[n].grad)
        assert _close(g["abs_sum"], want["abs_sum"], 1e-5, 1e-12), ("oracle", n, g, want)
    # (b) the product's plan
    plan = build_plan(ModelConfig(**flags), B, size, size, training=True, mixup_type=1, label_smoothing=0.1,
                      dtype="fp32")
    it = PI.PlanInterpreter(plan, dtype=torch.float64)
    it.set_weights(values)
    it.hp.update(grad_scale=1.0)
    logits = it.forward(x.double(), labels.int(), lam.double())
    it.run(plan.backward)
    assert _close(float(it.slot(plan.meta["loss"])[0]), gold["cross_entropy"], 2e-6)
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(mg.digest(logits)[k], gold["train_logits"][k], 1e-6, 1e-9), k
    for n, want in gold["grads"].items():
        g = mg.digest(it.get_tf(n, it.grads))
        assert _close(g["abs_sum"], want["abs_sum"], 1e-5, 1e-12), ("plan", n, g, want)
        assert _close(g["sum"], want["sum"], 1e-5, 1e-5 * want["abs_sum"] + 1e-12), ("plan", n, g, want)


@pytest.mark.parametrize("keep", [False, True], ids=["mixup_type_1", "mixup_type_2"])
def test_mixup_matches_reference_code(keep):
    """utils/data_util.py:97-158 executed through the stand-in with the same lambdas."""
    from oracle import tf_ops as T
    x, y, lam1, lam2 = mg.mixup_inputs()
    mx, my = T.mixup(x, y, lam1, lam2 if keep else None, keep_batch_size=keep)
    gold = PIECES["mixup_keep_%d" % keep]
    assert list(mx.shape) == gold["x_shape"]
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(mg.digest(mx)[k], gold["x"][k], 1e-6)
        assert _close(mg.digest(my)[k], gold["y"][k], 1e-6)
    assert torch.allclose(my, torch.tensor(gold["y_rows"]), atol=1e-6)


@pytest.mark.parametrize("ls", [0.0, 0.1])
def test_softmax_ce_matches_reference_code(ls):
    """losses/cls_losses.py:23-41 (soft labels, label smoothing over the given number of classes)."""
    from oracle import tf_ops as T
    logits, y = mg.loss_inputs()
    got = float(T.softmax_cross_entropy(logits, y, ls))
    assert _close(got, PIECES["softmax_ce_ls_%g" % ls], 1e-6)


@pytest.mark.parametrize("case", sorted(mg.LR_CASES))
def test_learning_rate_schedule_matches_reference_code(case):
    """functions/model_fns.py:36-95 learning_rate_with_decay executed through the stand-in."""
    from oracle import tf_ops as T
    kw = mg.LR_CASES[case]
    for step, want in zip(mg.LR_STEPS, PIECES["lr_" + case]):
        got = T.learning_rate(step, decay_type=kw["learning_rate_decay_type"], batch_size=kw["batch_size"],
                              num_images=kw["num_images"], base_lr=kw["base_lr"],
                              warmup_epochs=kw["warmup_epochs"], train_epochs=kw["train_epochs"],
                              num_epochs_per_decay=kw["num_epochs_per_decay"],
                              decay_factor=kw["learning_rate_decay_factor"],
                              end_learning_rate=kw["end_learning_rate"],
                              boundary_epochs=tuple(kw["piecewise_lr_boundary_epochs"]),
                              decay_rates=tuple(kw["piecewise_lr_decay_rates"]))
        assert _close(got, want, 1e-5, 1e-9), (case, step, got, want)


def test_flag_names_and_defaults_match_reference_code():
    """nets/hparams_config.py: every flag the product exposes under the reference's name has the
    reference's default (read from the AST of the DEFINE_* calls)."""
    from assembled_cnn_b200.hparams import DEFAULTS
    ref = PIECES["flag_defaults"]
    assert len(ref) >= 50
    common = [k for k in DEFAULTS if k in ref]
    assert len(common) >= 30
    for k in common:
        want = ref[k]["default"]
        got = DEFAULTS[k]
        if ref[k]["kind"] == "enum" and not isinstance(got, str):
            got = str(got)                     # e.g. resnet_version: enum of '1' / '2'
        if isinstance(want, (list, tuple)):
            assert [float(v) for v in got] == [float(v) for v in want], k
        else:
            assert got == want, (k, got, want)
    # flags of the official.utils.flags core set / the run loop, not defined in hparams_config.py
    assert set(DEFAULTS) - set(ref) <= {"resnet_size", "batch_size", "train_epochs", "dtype",
                                        "loss_scale", "data_format", "num_gpus"}


@pytest.mark.parametrize("mtype", [1, 2])
def test_mixup_dispatch_matches_reference_call_site(mtype):
    """nets/run_loop_classification.py:101-109 executed from the source with the reference's own mixup
    behind it: mixup_type 1 -> mixup(keep_batch_size=False) (2B examples in, B out), mixup_type 2 ->
    keep_batch_size=True, teacher labels passed through `y_t`, nothing in EVAL mode.  The oracle's
    convention `keep_batch_size = (mixup_type == 2)` -- what the plan's pack_input / mix_labels /
    kd_teacher ops are tested against -- reproduces images, labels and teacher labels."""
    from oracle import tf_ops as T
    x, y, lam1, lam2 = mg.mixup_inputs()
    yt = mg.teacher_labels()
    gold = PIECES["mixup_dispatch_type%d_train" % mtype]
    mx, my, myt = T.mixup(x.double(), y.double(), lam1.double(), lam2.double() if mtype == 2 else None,
                          keep_batch_size=(mtype == 2), y_t=yt.double())
    assert list(mx.shape) == gold["x_shape"] and mx.shape[0] == (mg.MIXUP_B // 2 if mtype == 1 else mg.MIXUP_B)
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(mg.digest(mx)[k], gold["x"][k], 1e-9)
        assert _close(mg.digest(my)[k], gold["y"][k], 1e-9)
        assert _close(mg.digest(myt)[k], gold["yt"][k], 1e-9)
    ev = PIECES["mixup_dispatch_type%d_eval" % mtype]            # EVAL: inputs untouched
    assert ev["x_shape"] == list(x.shape) and _close(ev["x"]["sum"], mg.digest(x)["sum"], 1e-9)
    assert _close(ev["y"]["sum"], mg.digest(y)["sum"], 1e-12)


def test_kd_loss_matches_reference_code():
    """nets/run_loop_classification.py:89-96,156-162 -- the two `if p['kd_temp'] > 0:` branches of
    resnet_model_fn executed from the reference's source (label tensor = one-hot ++ teacher logits is split,
    teacher labels = softmax(teacher logits / T), loss term = T^2 * CE(logits / T, teacher labels)): the
    oracle's kd_loss and teacher labels (what the CUDA loss kernel and acnn_kd_teacher_labels are tested
    against on the GPU, tests/test_features_gpu.py)."""
    from oracle import tf_ops as T
    gold = PIECES["kd"]
    logits, kd_labels = mg.kd_inputs()
    onehot, teacher_logits = kd_labels.split(mg.KD_NC, dim=1)        # as model_fn_cls splits it
    teacher = torch.softmax(teacher_logits.double() / gold["temp"], dim=1)
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(mg.digest(teacher)[k], gold["teacher_labels"][k], 1e-9)
        assert _close(mg.digest(onehot)[k], gold["onehot"][k], 1e-12)
    for a, b in zip(teacher[0].tolist(), gold["teacher_row0"]):
        assert _close(a, b, 1e-9)
    got = T.kd_loss(logits, teacher, gold["temp"])
    assert _close(float(got), gold["cross_entropy_kd"], 2e-6), (float(got), gold["cross_entropy_kd"])


def test_predictions_dict_matches_reference_code():
    """nets/run_loop_classification.py:126-130 executed from the source: keys and values of the
    EstimatorSpec's `predictions` (what model_fn_cls returns in every mode)."""
    from assembled_cnn_b200.model_fns import predictions_of
    gold = PIECES["predictions"]
    logits, _ = mg.loss_inputs()
    got = predictions_of(logits.double())
    assert set(got) == set(gold) - {"classes_list"}
    assert got["classes"].tolist() == gold["classes_list"]
    for key in ("probabilities", "probabilities_sigmoid"):
        for k in ("sum", "abs_sum", "first", "last"):
            assert _close(mg.digest(got[key])[k], gold[key][k], 1e-9), (key, k)


def test_input_batch_matches_reference_code():
    """functions/input_fns.py:98-102 executed from the source: how many examples the input pipeline delivers
    per step (2 x batch for mixup type 1 in training, batch otherwise) == the plan's input_batch."""
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    for mtype, is_training, want in PIECES["input_batch"]:
        plan = build_plan(ModelConfig(resnet_size=50), 256, 32, 32, training=is_training, mixup_type=mtype)
        assert plan.meta["input_batch"] == want, (mtype, is_training)
        assert plan.tensors[plan.meta["images"]].shape[0] == want


def test_per_device_batch_size_matches_reference_code():
    """official/utils/misc/distribution_utils.py:48-76 executed from the reference's source: per-replica
    batch and the ValueError text of an indivisible global batch (Trainer raises it)."""
    from assembled_cnn_b200.model_fns import per_device_batch_size
    gold = PIECES["per_device_batch"]
    for b, n, want in gold["cases"]:
        assert per_device_batch_size(b, n) == want
    with pytest.raises(ValueError) as e:
        per_device_batch_size(2050, 8)
    assert str(e.value) == gold["error_2050_8"]


@pytest.mark.parametrize("case", sorted(mg.KEEP_PROB_CASES))
def test_keep_prob_schedule_matches_reference_code(case):
    """functions/model_fns.py:26-33 keep_prob_decay (tf.train.polynomial_decay, power 1, no cycle) executed
    from the reference's source: the product's host-side schedule (Trainer feeds hp[4] from it)."""
    from assembled_cnn_b200.model_fns import keep_prob_decay
    fn = keep_prob_decay(*mg.KEEP_PROB_CASES[case])
    for step, want in zip(mg.LR_STEPS, PIECES["keep_prob_" + case]):
        assert abs(fn(step) - want) < 1e-6, (case, step, fn(step), want)


@pytest.mark.parametrize("name", sorted(mg.CONFIGS))
def test_product_plan_inventory_matches_reference_code(name):
    """The product's own layer plan (assembled_cnn_b200/plan.py): trainable variables in the reference's
    creation order with the reference's (TF-layout) shapes, and the BN moving statistics."""
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    flags, d, batch, size = mg.CONFIGS[name]
    gold = GOLD[name]
    plan = build_plan(ModelConfig(use_resnet_d=d, **flags), 2, 64, 64, training=True)
    assert len(plan.params) == gold["num_trainable"]
    tr = "\n".join("%s|%s" % (n, ",".join(map(str, p.tf_shape))) for n, p in plan.params.items())
    assert hashlib.sha256(tr.encode()).hexdigest() == gold["trainable_sha256"]
    st = "\n".join("%s|%s" % (n, ",".join(map(str, p.tf_shape))) for n, p in plan.state.items())
    assert hashlib.sha256(st.encode()).hexdigest() == gold["state_sha256"]


@pytest.mark.parametrize("name", sorted(mg.CONFIGS))
def test_warm_start_filter_matches_reference_code(name):
    """utils/hook_utils.py:36-47 WarmStartHook.begin executed from the reference's source on the variable
    inventory of each configuration (SE blocks keep their dense layers, the classifier and the embedding
    head are left out): checkpoint.warm_start_variables must select the same variables, in order."""
    from assembled_cnn_b200 import checkpoint as C
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    flags, d, batch, size = mg.CONFIGS[name]
    gold = GOLD[name]
    plan = build_plan(ModelConfig(use_resnet_d=d, **flags), 2, 64, 64, training=True)
    ws = C.warm_start_variables(list(plan.params))
    assert len(ws) == gold["num_warm_start"] < len(plan.params)
    assert hashlib.sha256("\n".join(ws).encode()).hexdigest() == gold["warm_start_sha256"]


@pytest.mark.parametrize("name", sorted(mg.CONFIGS))
def test_native_plan_inventory_matches_reference_code(name):
    """The same for the plan the product executes -- built in C++ behind acnn_create
    (csrc/model_plan.cu, include/acnn_model.h): acnn_variable_info_get lists the reference's variables
    in the reference's creation order with the reference's names and TF-layout shapes."""
    import ctypes as C
    from assembled_cnn_b200 import native
    from assembled_cnn_b200.plan import ModelConfig
    flags, d, batch, size = mg.CONFIGS[name]
    gold = GOLD[name]
    nm = native.NativeModel(ModelConfig(use_resnet_d=d, **flags), 2, 64, 64, training=True)
    vi, rows = native.VariableInfo(), {0: [], 1: []}
    for i in range(nm.sizes.n_variables):
        assert nm.lib.acnn_variable_info_get(nm.handle, i, C.byref(vi)) == 0
        rows[vi.buffer].append("%s|%s" % (vi.name.decode(), ",".join(map(str, vi.tf_shape[:vi.tf_rank]))))
    assert len(rows[0]) == gold["num_trainable"]
    assert hashlib.sha256("\n".join(rows[0]).encode()).hexdigest() == gold["trainable_sha256"]
    assert hashlib.sha256("\n".join(rows[1]).encode()).hexdigest() == gold["state_sha256"]


# ---------------------------------------------------------------------------------------------
# The feature rows against the reference's own code: DropBlock, GeM pooling, KD teacher mixup
# (the GeM / embedding / flatten model configurations are part of mg.CONFIGS above)
# ---------------------------------------------------------------------------------------------
def test_gem_pooling_matches_reference_code():
    """nets/blocks.py:22-42 generalized_mean_pooling executed through the stand-in."""
    from oracle import tf_ops as T
    got = T.generalized_mean_pooling(mg.feature_map())
    assert torch.allclose(got, torch.tensor(PIECES["gem"]["rows"]), rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("kp,gs", [(0.9, 1.0), (0.7, 0.25)])
def test_dropblock_function_matches_reference_code(kp, gs):
    """nets/blocks.py:187-251 dropblock (+ _bernoulli) executed through the stand-in with the same
    uniform draws."""
    from oracle import tf_ops as T
    x, u = mg.dropblock_inputs()
    y = T.dropblock(x, kp, 7, gs, u)
    gold = PIECES["dropblock_kp%g_gs%g" % (kp, gs)]
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(mg.digest(y)[k], gold["out"][k], 1e-5)
    assert abs(float((y == 0).float().mean()) - gold["zero_fraction"]) < 1e-9
    assert torch.allclose(y[1, 5, :, 2], torch.tensor(gold["row"]), rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("keep", [False, True], ids=["mixup_type_1", "mixup_type_2"])
def test_teacher_label_mixup_matches_reference_code(keep):
    """utils/data_util.py:128-156: the y_t path, including the type-2 second half that mixes the
    SUPERVISED labels (`lam2_y * y1`, :154)."""
    from oracle import tf_ops as T
    x, y, lam1, lam2 = mg.mixup_inputs()
    _, _, myt = T.mixup(x, y, lam1, lam2 if keep else None, keep_batch_size=keep,
                        y_t=mg.teacher_labels())
    assert torch.allclose(myt, torch.tensor(PIECES["mixup_teacher_keep_%d" % keep]["yt_rows"]),
                          atol=1e-6)


@pytest.mark.parametrize("name", sorted(mg.DROPBLOCK_CONFIGS))
def test_dropblock_through_the_whole_reference_model(name):
    """The reference's Model.__call__(training=True, keep_prob=...) at 224 px with the uniform draws
    replayed from the same seeded generator IN CALL ORDER: pins where the reference calls dropblock
    (34 calls for Assemble-ResNet-50, 29 for the vanilla net), their mask shapes and the logits."""
    from oracle import model as M
    flags, batch, size, kp = mg.DROPBLOCK_CONFIGS[name]
    gold = GOLD[name]
    model, vs = M.build(seed=1, input_hw=64, **flags)
    for i, n in enumerate(list(vs.vars)):
        vs.vars[n] = mg.seeded_value(i, n, tuple(vs.vars[n].shape))
    x = mg.seeded_input(batch, size)
    g = torch.Generator().manual_seed(mg.DROPBLOCK_SEED)
    shapes = []

    def uniform(shape):
        shapes.append(list(shape))
        return torch.rand(shape, generator=g)
    with torch.no_grad():
        y = M.forward(model, vs, x, training=True, keep_prob=kp, dropblock_u=uniform)
    assert len(shapes) == gold["num_dropblock_calls"]
    assert shapes[:5] == gold["first_shapes"] and shapes[-1] == gold["last_shape"]
    got = mg.digest(y)
    assert _close(got["abs_sum"], gold["train_logits"]["abs_sum"], 5e-3), (got, gold["train_logits"])
    for a, b in zip(y[0, :8].tolist(), gold["train_logits_row0_head"]):
        assert _close(a, b, 5e-3, 1e-3)
    # float64 oracle against the float64 golden (kernels that are not the oracle's): 1e-5 on the logits
    # (the mask renormalisation count / sum is fp32 arithmetic on both sides, as in the reference)
    for n in vs.vars:
        vs.vars[n] = vs.vars[n].double()
    vs.dtype = torch.float64
    g = torch.Generator().manual_seed(mg.DROPBLOCK_SEED)
    with torch.no_grad():
        y64 = M.forward(model, vs, x.double(), training=True, keep_prob=kp,
                        dropblock_u=lambda shape: torch.rand(shape, generator=g).double())
    got = mg.digest(y64)
    for k in ("sum", "abs_sum", "first", "last"):
        assert _close(got[k], gold["train_logits"][k], 1e-5, 1e-8), (k, got[k], gold["train_logits"][k])
    for a, b in zip(y64[0, :8].tolist(), gold["train_logits_row0_head"]):
        assert _close(a, b, 1e-5, 1e-8)
    # the product's plan draws its masks at the same sites, in the same order, with the same shapes
    from assembled_cnn_b200.plan import ModelConfig, build_plan
    plan = build_plan(ModelConfig(**flags), batch, size, size, training=True, use_dropblock=True)
    plan_shapes = [[1] + list(plan.tensors[n].shape) for n in plan.meta["dropblock_u"]]
    assert plan_shapes == shapes
    # ... and so does the plan the library builds (acnn_find_tensor("dropblock_u", k))
    from assembled_cnn_b200 import native
    nm = native.NativeModel(ModelConfig(**flags), batch, size, size, training=True, use_dropblock=True)
    assert [[1] + list(nm.tensors[n].shape) for n in nm.meta["dropblock_u"]] == shapes
