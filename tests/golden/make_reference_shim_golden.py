#!/usr/bin/env python
"""Golden vectors produced by EXECUTING the reference's own model code (nets/resnet_model.py,
nets/blocks.py, nets/model_helper.py of a checkout of the original project) through the TF-1.14 API
stand-in in tests/golden/tf1_shim/ (TensorFlow 1.14 has no Python 3.12 build):

    python tests/golden/make_reference_shim_golden.py REFERENCE_DIR   # rewrites reference_shim_golden.json

What a golden entry holds, per model configuration: the variable names / shapes / initializer kinds in
the reference's creation order (a digest + the count), and for seeded inputs and seeded variable
values the logits in training and in inference mode plus digests of the updated BN moving statistics.
tests/test_reference_shim_golden_cpu.py replays the oracle on the same seeds against this file; it
does not need the original project.

The stand-in computes in float64 (TF_SHIM_FLOAT64=1, set below) with kernels that are not the oracle's
(Hugging Face's TF-'SAME' padding port, ATen batch norm: see the stand-in's docstring): the golden
numbers are therefore independent of any fp32 summation order, and the test can hold the float64 oracle to
1e-6 even on the ill-conditioned quantities (training-mode logits of a 152-layer net on a batch of 2).

The wrapper arguments below restate functions/model_fns.py:141-203 (class Model: num_filters=64,
kernel_size=7, conv_stride=2, first_pool 3/2, block sizes by depth, block strides by version);
importing that module itself would pull in the Estimator run loop.
"""
import hashlib
import json
import os
import sys

os.environ["TF_SHIM_FLOAT64"] = "1"      # before the stand-in is imported

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "reference_shim_golden.json")
# checkout of the original project whose code is executed (first argument)
REF_ROOT = None     # set from the command line (the module is also imported by the tests)

# configuration name -> (constructor flags of functions/model_fns.py:Model, use_resnet_d, batch, size)
CONFIGS = {
    "assemble_r50_rv2_sk_sconv": (dict(resnet_size=50, resnet_version=2, use_sk_block=True,
                                       anti_alias_type="sconv", anti_alias_filter_size=3), False, 4, 64),
    "assemble_r50_rv2_sk_sconv_resnet_d": (dict(resnet_size=50, resnet_version=2, use_sk_block=True,
                                                anti_alias_type="sconv", anti_alias_filter_size=3), True, 2, 64),
    "vanilla_r50_rv1": (dict(resnet_size=50, resnet_version=1), False, 2, 64),
    "r50_rv1_resnet_d_sk_aa_zero_gamma": (dict(resnet_size=50, resnet_version=1, use_sk_block=True,
                                               anti_alias_type="sconv", anti_alias_filter_size=3,
                                               zero_gamma=True), True, 2, 64),
    "r50_rv1_se_proj_aa5": (dict(resnet_size=50, resnet_version=1, use_se_block=True,
                                 anti_alias_type="proj_sconv", anti_alias_filter_size=5), False, 2, 64),
    "r50_rv2_se_no_downsample": (dict(resnet_size=50, resnet_version=2, use_se_block=True,
                                      no_downsample=True), False, 2, 64),
    "assemble_r152_rv2_sk_sconv": (dict(resnet_size=152, resnet_version=2, use_sk_block=True,
                                        anti_alias_type="sconv", anti_alias_filter_size=3), False, 4, 64),
    "r101_rv1_resnet_d": (dict(resnet_size=101, resnet_version=1), True, 2, 64),
    "baseline_c5_assemble_r152_alpha1_beta2": (dict(resnet_size=152, resnet_version=2, use_sk_block=True,
                                                    anti_alias_type="sconv", anti_alias_filter_size=3,
                                                    bl_alpha=1, bl_beta=2), False, 4, 64),
    # (batch 4 for the 152-layer nets: on a batch of 2 the SK-attention batch norms see two samples and
    # the training-mode logits are chaotic even in float64 -- a 1e-14 input perturbation moves them 8 %)
    # GeM pooling + embedding head, flatten pooling (nets/resnet_model.py:552-599)
    "assemble_r50_gem_embedding256": (dict(resnet_size=50, resnet_version=2, use_sk_block=True,
                                           anti_alias_type="sconv", anti_alias_filter_size=3,
                                           pool_type="gem", embedding_size=256), False, 4, 64),
    "r50_rv1_flatten": (dict(resnet_size=50, resnet_version=1, pool_type="flatten"), False, 2, 64),
}
# DropBlock through the whole reference model (training mode, keep_prob 0.9, 224 px: the stage-4 map
# must hold the 7x7 block): the uniform draws come from a seeded generator in CALL ORDER, so the
# golden logits also pin the order and shapes of the reference's dropblock calls
DROPBLOCK_CONFIGS = {
    "assemble_r50_dropblock_kp0.9": (dict(resnet_size=50, resnet_version=2, use_sk_block=True,
                                          anti_alias_type="sconv", anti_alias_filter_size=3), 2, 224, 0.9),
    "vanilla_r50_dropblock_kp0.8": (dict(resnet_size=50, resnet_version=1), 2, 224, 0.8),
}
DROPBLOCK_SEED = 4242
BLOCK_SIZES = {1: {50: [3, 4, 6, 3], 101: [3, 4, 23, 3], 152: [3, 8, 36, 3], 200: [3, 24, 36, 3]}}


def block_sizes(resnet_size, resnet_version):
    """functions/model_fns.py:96-135 get_block_sizes (version 2 = BigLittle table)."""
    if resnet_version == 2:
        return {50: [3, 4, 6, 3], 101: [4, 8, 18, 3], 152: [5, 12, 30, 3]}[resnet_size]
    return BLOCK_SIZES[1][resnet_size]


def seeded_value(index, name, shape):
    """Deterministic value of the index-th variable (shared with the test): well-conditioned
    statistics so that training- and inference-mode outputs are both O(1)."""
    g = torch.Generator().manual_seed(1000003 * (index + 1) + len(name))
    leaf = name.rsplit("/", 1)[1]
    if leaf == "moving_variance":
        return 0.5 + torch.rand(shape, generator=g)
    if leaf == "gamma":
        return 1.0 + 0.1 * torch.randn(shape, generator=g)
    if leaf in ("beta", "moving_mean", "bias"):
        return 0.1 * torch.randn(shape, generator=g)
    fan_in = 1
    for d in shape[:-1]:
        fan_in *= d
    return torch.randn(shape, generator=g) * (1.0 / fan_in) ** 0.5


def seeded_input(batch, size):
    return torch.randn(batch, size, size, 3, generator=torch.Generator().manual_seed(20240923))


def digest(t):
    t = t.detach().double().flatten()
    return {"sum": float(t.sum()), "abs_sum": float(t.abs().sum()), "first": float(t[0]), "last": float(t[-1])}


def names_digest(order):
    h = hashlib.sha256()
    for name, shape, kind, trainable in order:
        h.update(("%s|%s|%s|%d\n" % (name, ",".join(map(str, shape)), kind, trainable)).encode())
    return h.hexdigest()


def reference_function(rel_path, name):
    """Compile ONE function of a reference module (by its AST) against the shim: the module's other
    top-level imports (Estimator run loop, preprocessing, absl flags) are not needed for it."""
    import ast
    sys.path.insert(0, os.path.join(HERE, "tf1_shim"))
    import tensorflow as tf
    src = open(os.path.join(REF_ROOT, rel_path)).read()
    # (ast.walk: also finds functions nested inside other functions, e.g. exclude_batch_norm)
    node = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == name)
    ns = {"tf": tf}
    exec(compile(ast.Module(body=[node], type_ignores=[]), rel_path, "exec"), ns)
    return ns[name], tf


def reference_warm_start_list(trainable_names):
    """utils/hook_utils.py:36-47 WarmStartHook.begin executed from the reference's source on a list of
    trainable variable names (TF appends ':0' to a variable's name): which variables a fine-tuning run
    restores.  The TF services the method touches are stubbed with recorders."""
    import types
    begin, tf = reference_function("utils/hook_utils.py", "begin")
    var = lambda n: types.SimpleNamespace(name=n + ":0")
    saved = {}
    tf.contrib.framework = types.SimpleNamespace(get_trainable_variables=lambda: [var(n) for n in trainable_names])
    tf.gfile = types.SimpleNamespace(IsDirectory=lambda path: False)
    old_saver = getattr(tf.train, "Saver", None)
    tf.train.Saver = lambda var_list: saved.setdefault("vars", list(var_list))
    try:
        hook = types.SimpleNamespace(checkpoint_path="ckpt", var_list_warm_start=[], saver=None)
        begin(hook)
    finally:
        tf.train.Saver = old_saver
    assert [v.name for v in saved["vars"]] == [v.name for v in hook.var_list_warm_start]
    return [v.name[:-2] for v in hook.var_list_warm_start]


def reference_if_blocks(rel_path, func_name, test_src):
    """The `if <test_src>:` statements inside one function of a reference module, each compiled on its
    own (for code the reference writes inline in a long function, e.g. the knowledge-distillation
    branches of resnet_model_fn), to be exec'd in a namespace holding the names they read."""
    import ast
    sys.path.insert(0, os.path.join(HERE, "tf1_shim"))
    import tensorflow as tf
    src = open(os.path.join(REF_ROOT, rel_path)).read()
    fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == func_name)
    blocks = sorted((n for n in ast.walk(fn) if isinstance(n, ast.If) and ast.unparse(n.test) == test_src),
                    key=lambda n: n.lineno)            # source order (ast.walk is breadth-first)
    return [compile(ast.fix_missing_locations(ast.Module(body=[b], type_ignores=[])), rel_path, "exec")
            for b in blocks], tf


def run_reference(flags, use_resnet_d, batch, size):
    sys.path.insert(0, os.path.join(HERE, "tf1_shim"))
    sys.path.insert(0, REF_ROOT)
    import tensorflow as tf          # the shim
    from nets import resnet_model   # the REAL reference code
    f = dict(flags)
    rv = f.get("resnet_version", 1)
    strides = [2, 2, 1, 2] if rv == 2 else [1, 2, 2, 2]
    if f.pop("no_downsample", False):
        strides[-1] = 1
    size_ = f.pop("resnet_size")

    def make():
        return resnet_model.Model(resnet_size=size_, bottleneck=True, num_classes=1001, num_filters=64,
                                  kernel_size=7, conv_stride=2, first_pool_size=3, first_pool_stride=2,
                                  block_sizes=block_sizes(size_, rv), block_strides=strides, **f)

    # pass 1: discover the variables (names, shapes, initializers, order)
    tf.reset()
    make()(tf.Tensor(seeded_input(batch, size)), training=False, use_resnet_d=use_resnet_d)
    order = list(tf.variables.order)
    values = {n: seeded_value(i, n, s) for i, (n, s, _, _) in enumerate(order)}
    out = {"num_variables": len(order), "names_sha256": names_digest(order),
           "first_names": [o[0] for o in order[:3]], "last_names": [o[0] for o in order[-2:]],
           "zero_init_gammas": sum(1 for o in order if o[2] == "zeros" and o[0].endswith("/gamma")),
           # separate digests of the trainable variables (creation order, with TF shapes) and of the
           # non-trainable BN statistics: what the product's plan (params / state) is checked against
           "trainable_sha256": hashlib.sha256("\n".join(
               "%s|%s" % (o[0], ",".join(map(str, o[1]))) for o in order if o[3]).encode()).hexdigest(),
           "num_trainable": sum(1 for o in order if o[3]),
           "state_sha256": hashlib.sha256("\n".join(
               "%s|%s" % (o[0], ",".join(map(str, o[1]))) for o in order if not o[3]).encode()).hexdigest(),
           "batch": batch, "size": size, "use_resnet_d": use_resnet_d}
    x = seeded_input(batch, size)
    # pass 2: inference mode with the seeded values
    tf.reset(values)
    y = make()(tf.Tensor(x), training=False, use_resnet_d=use_resnet_d)
    out["eval_logits"] = digest(y.t)
    out["eval_logits_row0_head"] = [float(v) for v in y.t[0, :8]]
    # pass 3: training mode (batch statistics + moving-average updates)
    tf.reset(values)
    y = make()(tf.Tensor(x), training=True, use_resnet_d=use_resnet_d)
    out["train_logits"] = digest(y.t)
    mm = torch.cat([tf.variables.vars[o[0]].t.flatten() for o in order if o[0].endswith("moving_mean")])
    mv = torch.cat([tf.variables.vars[o[0]].t.flatten() for o in order if o[0].endswith("moving_variance")])
    out["moving_mean_after"] = digest(mm)
    out["moving_variance_after"] = digest(mv)
    # gradients of the reference's graph (torch autograd through the stand-in) of
    # loss = get_sup_loss(label_smoothing 0.1) + 1e-4 * sum l2_loss(decayed variables), inference-mode
    # BN (well conditioned) -- what the product's explicit backward is tested against via the oracle
    if out["num_variables"] < 600:
        get_sup_loss, _ = reference_function("losses/cls_losses.py", "get_sup_loss")
        exclude_bn, _ = reference_function("nets/run_loop_classification.py", "exclude_batch_norm")
        tf.reset(values, requires_grad=True)
        y = make()(tf.Tensor(x), training=False, use_resnet_d=use_resnet_d)
        lab = torch.nn.functional.one_hot(torch.arange(batch) * 37 % 1001, 1001).float()
        ce = get_sup_loss(y, tf.Tensor(lab), None, 1001, {"cls_loss_type": "softmax", "label_smoothing": 0.1})
        l2 = sum((tf.variables.vars[o[0]].t ** 2).sum() / 2 for o in order if o[3] and exclude_bn(o[0] + ":0"))
        loss = ce.t + 1e-4 * l2
        loss.backward()
        out["loss_eval_mode"] = float(loss)
        tr = [o[0] for o in order if o[3]]
        picks = [tr[0], tr[len(tr) // 3], tr[len(tr) // 2], tr[-2], tr[-1]]
        out["grads_eval_mode"] = {n: digest(tf.variables.vars[n].t.grad) for n in picks}
    # the same loss with TRAINING-mode batch norm (batch statistics): its value and gradient digests of a
    # spread of variables -- what the product's explicit backward (hand-derived BN / SK / SE / pooling
    # backward passes of the plan) is compared with in float64
    get_sup_loss, _ = reference_function("losses/cls_losses.py", "get_sup_loss")
    tf.reset(values, requires_grad=True)
    y = make()(tf.Tensor(x), training=True, use_resnet_d=use_resnet_d)
    lab = torch.nn.functional.one_hot(torch.arange(batch) * 37 % 1001, 1001).float()
    ce = get_sup_loss(y, tf.Tensor(lab), None, 1001, {"cls_loss_type": "softmax", "label_smoothing": 0.1})
    ce.t.backward()
    out["ce_train_mode"] = float(ce.t)
    tr = [o[0] for o in order if o[3]]
    picks = sorted(set([tr[0], tr[1], tr[2], tr[len(tr) // 3], tr[len(tr) // 2], tr[-2], tr[-1]] + tr[5::61]),
                   key=tr.index)
    out["grads_train_mode"] = {n: digest(tf.variables.vars[n].t.grad) for n in picks}
    # nets/run_loop_classification.py:163-176: which trainable variables enter the L2 term
    exclude_batch_norm, _ = reference_function("nets/run_loop_classification.py", "exclude_batch_norm")
    decayed = [o[0] for o in order if o[3] and exclude_batch_norm(o[0] + ":0")]
    out["num_decayed"] = len(decayed)
    out["decayed_sha256"] = hashlib.sha256("\n".join(decayed).encode()).hexdigest()
    return out, order


C3_BATCH, C3_SIZE = 4, 64


def c3_inputs():
    """2B images, 2B class labels, B mixing coefficients (mixup type 1 halves the batch)."""
    g = torch.Generator().manual_seed(4321)
    x = torch.randn(2 * C3_BATCH, C3_SIZE, C3_SIZE, 3, generator=g)
    labels = torch.randint(1, 1001, (2 * C3_BATCH,), generator=g)
    lam = torch.rand(C3_BATCH, generator=g)
    return x, labels, lam


def run_reference_c3_composition():
    """BASELINE config 3 as the reference composes it (nets/run_loop_classification.py:101-109,141-149):
    utils/data_util.mixup(keep_batch_size=False) on images and one-hot labels -> Assemble-ResNet-50 in
    training mode -> losses/cls_losses.get_sup_loss with label smoothing 0.1; gradients by autograd."""
    sys.path.insert(0, os.path.join(HERE, "tf1_shim"))
    sys.path.insert(0, REF_ROOT)
    import tensorflow as tf
    from nets import resnet_model
    flags, d, _, _ = CONFIGS["assemble_r50_rv2_sk_sconv"]
    f = dict(flags)
    size_ = f.pop("resnet_size")
    mixup, _ = reference_function("utils/data_util.py", "mixup")
    get_sup_loss, _ = reference_function("losses/cls_losses.py", "get_sup_loss")

    def make():
        return resnet_model.Model(resnet_size=size_, bottleneck=True, num_classes=1001, num_filters=64,
                                  kernel_size=7, conv_stride=2, first_pool_size=3, first_pool_stride=2,
                                  block_sizes=block_sizes(size_, 2), block_strides=[2, 2, 1, 2], **f)
    x, labels, lam = c3_inputs()
    tf.reset()
    make()(tf.Tensor(x[:C3_BATCH]), training=False)
    order = list(tf.variables.order)
    values = {n: seeded_value(i, n, s) for i, (n, s, _, _) in enumerate(order)}
    tf.reset(values, requires_grad=True)
    tf.beta_samples.clear()
    tf.beta_samples.append(lam)
    onehot = torch.nn.functional.one_hot(labels, 1001).float()
    mx, my = mixup(tf.Tensor(x), tf.Tensor(onehot), keep_batch_size=False)[:2]
    y = make()(mx, training=True)
    ce = get_sup_loss(y, my, None, 1001, {"cls_loss_type": "softmax", "label_smoothing": 0.1})
    ce.t.backward()
    tr = [o[0] for o in order if o[3]]
    picks = sorted(set([tr[0], tr[1], tr[2], tr[len(tr) // 3], tr[len(tr) // 2], tr[-2], tr[-1]] + tr[7::43]),
                   key=tr.index)
    return {"batch": C3_BATCH, "size": C3_SIZE, "mixed_images": digest(tf._raw(mx)),
            "mixed_labels": digest(tf._raw(my)), "train_logits": digest(y.t), "cross_entropy": float(ce.t),
            "grads": {n: digest(tf.variables.vars[n].t.grad) for n in picks}}


def run_reference_dropblock(flags, batch, size, keep_prob):
    sys.path.insert(0, os.path.join(HERE, "tf1_shim"))
    sys.path.insert(0, REF_ROOT)
    import tensorflow as tf
    from nets import resnet_model
    f = dict(flags)
    rv = f.get("resnet_version", 1)
    strides = [2, 2, 1, 2] if rv == 2 else [1, 2, 2, 2]
    size_ = f.pop("resnet_size")

    def make():
        return resnet_model.Model(resnet_size=size_, bottleneck=True, num_classes=1001, num_filters=64,
                                  kernel_size=7, conv_stride=2, first_pool_size=3, first_pool_stride=2,
                                  block_sizes=block_sizes(size_, rv), block_strides=strides, **f)
    tf.reset()
    make()(tf.Tensor(seeded_input(batch, 64)), training=False)
    order = list(tf.variables.order)
    values = {n: seeded_value(i, n, s) for i, (n, s, _, _) in enumerate(order)}
    x = seeded_input(batch, size)
    g = torch.Generator().manual_seed(DROPBLOCK_SEED)
    shapes = []

    def uniform(shape):
        shapes.append(list(shape))
        return torch.rand(shape, generator=g)
    tf.uniform_fn = uniform
    try:
        tf.reset(values)
        y = make()(tf.Tensor(x), training=True, keep_prob=keep_prob)
    finally:
        tf.uniform_fn = None
    return {"batch": batch, "size": size, "keep_prob": keep_prob, "num_dropblock_calls": len(shapes),
            "first_shapes": shapes[:5], "last_shape": shapes[-1], "train_logits": digest(y.t),
            "train_logits_row0_head": [float(v) for v in y.t[0, :8]]}


MIXUP_B, MIXUP_HW, MIXUP_NC = 8, 4, 5
LR_CASES = {   # name -> kwargs of functions/model_fns.py learning_rate_with_decay (+ probe steps)
    "cosine_warmup5_b1024": dict(learning_rate_decay_type="cosine", batch_size=1024, batch_denom=1024,
                                 num_images=1281167, num_epochs_per_decay=2.0, learning_rate_decay_factor=0.94,
                                 end_learning_rate=0.0001, piecewise_lr_boundary_epochs=[30, 60, 80, 90],
                                 piecewise_lr_decay_rates=[1, 0.1, 0.01, 0.001, 1e-4], base_lr=0.4,
                                 warmup_epochs=5, train_epochs=600),
    "piecewise_b256": dict(learning_rate_decay_type="piecewise", batch_size=256, batch_denom=256,
                           num_images=1281167, num_epochs_per_decay=2.0, learning_rate_decay_factor=0.94,
                           end_learning_rate=0.0001, piecewise_lr_boundary_epochs=[30, 60, 80, 90],
                           piecewise_lr_decay_rates=[1, 0.1, 0.01, 0.001, 1e-4], base_lr=0.1,
                           warmup_epochs=0, train_epochs=100),
    "exponential_warmup1": dict(learning_rate_decay_type="exponential", batch_size=512, batch_denom=512,
                                num_images=1281167, num_epochs_per_decay=2.0, learning_rate_decay_factor=0.94,
                                end_learning_rate=0.0001, piecewise_lr_boundary_epochs=[30],
                                piecewise_lr_decay_rates=[1, 0.1], base_lr=0.2, warmup_epochs=1,
                                train_epochs=100),
    "polynomial": dict(learning_rate_decay_type="polynomial", batch_size=256, batch_denom=256,
                       num_images=50000, num_epochs_per_decay=30.0, learning_rate_decay_factor=0.94,
                       end_learning_rate=0.0001, piecewise_lr_boundary_epochs=[30],
                       piecewise_lr_decay_rates=[1, 0.1], base_lr=0.1, warmup_epochs=0, train_epochs=100),
    "fixed": dict(learning_rate_decay_type="fixed", batch_size=256, batch_denom=256, num_images=50000,
                  num_epochs_per_decay=30.0, learning_rate_decay_factor=0.94, end_learning_rate=0.0001,
                  piecewise_lr_boundary_epochs=[30], piecewise_lr_decay_rates=[1, 0.1], base_lr=0.05,
                  warmup_epochs=0, train_epochs=100),
}
PER_DEVICE_CASES = [(256, 1), (256, 0), (2048, 8), (1024, 8), (512, 2), (96, 4)]
KEEP_PROB_CASES = {"assemble_600_epochs_b1024": (1.0, 0.9, int(600 * 1281167 / 1024)),
                   "short": (1.0, 0.7, 10000)}
LR_STEPS = [0, 1, 100, 1250, 2501, 6254, 6256, 10000, 150134, 150136, 300000, 450408, 700000]


def mixup_inputs():
    g = torch.Generator().manual_seed(77)
    x = torch.randn(MIXUP_B, MIXUP_HW, MIXUP_HW, 3, generator=g)
    y = torch.nn.functional.one_hot(torch.randint(0, MIXUP_NC, (MIXUP_B,), generator=g), MIXUP_NC).float()
    lam1 = torch.rand(MIXUP_B // 2, generator=g)
    lam2 = torch.rand(MIXUP_B // 2, generator=g)
    return x, y, lam1, lam2


def teacher_labels():
    g = torch.Generator().manual_seed(79)
    return torch.softmax(2 * torch.randn(MIXUP_B, MIXUP_NC, generator=g), dim=1)


def feature_map():
    g = torch.Generator().manual_seed(80)
    return torch.relu(torch.randn(3, 5, 5, 6, generator=g)) * 2      # post-ReLU: exact zeros get clipped


def dropblock_inputs():
    g = torch.Generator().manual_seed(81)
    return torch.randn(2, 12, 12, 4, generator=g), torch.rand(1, 6, 6, 4, generator=g)


KD_TEMP, KD_B, KD_NC = 2.0, 6, 11


def kd_inputs():
    """(logits, kd label tensor = one-hot labels ++ teacher logits, as the reference's input pipeline
    delivers it: nets/run_loop_classification.py:86-93)."""
    g = torch.Generator().manual_seed(77)
    logits = 2.0 * torch.randn(KD_B, KD_NC, generator=g)
    onehot = torch.nn.functional.one_hot(torch.randint(0, KD_NC, (KD_B,), generator=g), KD_NC).float()
    teacher_logits = 3.0 * torch.randn(KD_B, KD_NC, generator=g)
    return logits, torch.cat([onehot, teacher_logits], 1)


def loss_inputs():
    g = torch.Generator().manual_seed(78)
    logits = torch.randn(6, 11, generator=g) * 3
    y = torch.softmax(torch.randn(6, 11, generator=g), dim=1)      # soft (mixed) labels
    return logits, y


def reference_flag_defaults():
    """nets/hparams_config.py: every flags.DEFINE_*(name=..., default=...) call, read from the AST
    (literal defaults only)."""
    import ast
    out = {}
    tree = ast.parse(open(os.path.join(REF_ROOT, "nets", "hparams_config.py")).read())
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and \
                node.func.attr.startswith("DEFINE_"):
            kw = {k.arg: k.value for k in node.keywords}
            if "name" in kw and "default" in kw:
                try:
                    out[ast.literal_eval(kw["name"])] = {"kind": node.func.attr[len("DEFINE_"):],
                                                         "default": ast.literal_eval(kw["default"])}
                except ValueError:
                    pass
    return out


def run_train_pieces():
    out = {"flag_defaults": reference_flag_defaults()}
    # utils/data_util.py:97-158 mixup (types 1 and 2)
    mixup, tf = reference_function("utils/data_util.py", "mixup")
    x, y, lam1, lam2 = mixup_inputs()
    for keep in (False, True):
        tf.beta_samples[:] = [lam1, lam2] if keep else [lam1]
        mx, my, _ = mixup(tf.Tensor(x), tf.Tensor(y), alpha=0.2, keep_batch_size=keep)
        out["mixup_keep_%d" % keep] = {"x": digest(mx.t), "y": digest(my.t), "x_shape": list(mx.t.shape),
                                        "y_rows": my.t.tolist()}
        # with knowledge-distillation teacher labels (y_t): the third return value
        tf.beta_samples[:] = [lam1, lam2] if keep else [lam1]
        yt = teacher_labels()
        _, _, myt = mixup(tf.Tensor(x), tf.Tensor(y), alpha=0.2, keep_batch_size=keep, y_t=tf.Tensor(yt))
        out["mixup_teacher_keep_%d" % keep] = {"yt_rows": myt.t.tolist()}
    # nets/blocks.py:22-42 generalized_mean_pooling and :187-251 dropblock, from the reference source
    gem, tf = reference_function("nets/blocks.py", "generalized_mean_pooling")
    xg = feature_map()
    out["gem"] = {"rows": gem(tf.Tensor(xg), data_format="channels_last").t.reshape(xg.shape[0], -1).tolist()}
    bern, tf = reference_function("nets/blocks.py", "_bernoulli")
    dropblock, tf = reference_function("nets/blocks.py", "dropblock")
    dropblock.__globals__["_bernoulli"] = bern
    xd, ud = dropblock_inputs()
    tf.uniform_fn = lambda shape: ud.reshape(shape)
    try:
        for kp, gs in ((0.9, 1.0), (0.7, 0.25)):
            y = dropblock(tf.Tensor(xd), kp, 7, gamma_scale=gs, data_format="channels_last")
            out["dropblock_kp%g_gs%g" % (kp, gs)] = {
                "out": digest(y.t), "zero_fraction": float((y.t == 0).float().mean()),
                "row": y.t[1, 5, :, 2].tolist()}
    finally:
        tf.uniform_fn = None
    # losses/cls_losses.py:23-41 get_sup_loss (softmax + label smoothing)
    get_sup_loss, tf = reference_function("losses/cls_losses.py", "get_sup_loss")
    logits, yy = loss_inputs()
    for ls in (0.0, 0.1):
        ce = get_sup_loss(tf.Tensor(logits), tf.Tensor(yy), None, 11,
                          {"cls_loss_type": "softmax", "label_smoothing": ls})
        out["softmax_ce_ls_%g" % ls] = float(ce.t)
    # functions/model_fns.py:36-95 learning_rate_with_decay
    lr_with_decay, tf = reference_function("functions/model_fns.py", "learning_rate_with_decay")
    for name, kw in LR_CASES.items():
        fn = lr_with_decay(**kw)
        out["lr_" + name] = [float(tf._raw(fn(tf.Tensor(torch.tensor(s))))) for s in LR_STEPS]
    # nets/run_loop_classification.py:89-96 and :156-162: the two `if p['kd_temp'] > 0:` branches of
    # resnet_model_fn (label split + temperatured teacher softmax; T^2 * CE(logits / T, teacher))
    blocks, tf = reference_if_blocks("nets/run_loop_classification.py", "resnet_model_fn", "p['kd_temp'] > 0")
    assert len(blocks) == 2, len(blocks)
    logits, kd_labels = kd_inputs()
    env = {"tf": tf, "p": {"kd_temp": KD_TEMP}, "labels": tf.Tensor(kd_labels), "logits": tf.Tensor(logits)}
    for b in blocks:
        exec(b, env)
    out["kd"] = {"temp": KD_TEMP, "cross_entropy_kd": float(tf._raw(env["cross_entropy_kd"])),
                 "teacher_labels": digest(tf._raw(env["teacher_labels"])),
                 "teacher_row0": [float(v) for v in tf._raw(env["teacher_labels"])[0]],
                 "onehot": digest(tf._raw(env["onehot_labels"]))}
    # nets/run_loop_classification.py:101-109: the call site that maps mixup_type 1 / 2 onto
    # data_util.mixup(keep_batch_size=False / True, y_t=teacher_labels), executed from the source with the
    # reference's own mixup function behind `data_util`
    import types
    blocks, tf = reference_if_blocks("nets/run_loop_classification.py", "resnet_model_fn",
                                     "p['mixup_type'] == 1 and mode == tf.estimator.ModeKeys.TRAIN")
    assert len(blocks) == 1
    ref_mixup, _ = reference_function("utils/data_util.py", "mixup")
    tf.estimator = types.SimpleNamespace(ModeKeys=types.SimpleNamespace(TRAIN="train", EVAL="eval", PREDICT="infer"))
    saved_logging, tf.logging = getattr(tf, "logging", None), tf.summary      # any tf.logging.* is a no-op
    x, y, lam1, lam2 = mixup_inputs()
    yt = teacher_labels()
    for mtype in (1, 2):
        for mode in ("train", "eval"):
            tf.beta_samples.clear()
            tf.beta_samples.extend([lam1, lam2][:mtype])
            env = {"tf": tf, "p": {"mixup_type": mtype}, "mode": mode,
                   "data_util": types.SimpleNamespace(mixup=ref_mixup),
                   "features_sup_may_mixuped": tf.Tensor(x), "onehot_labels": tf.Tensor(y),
                   "teacher_labels": tf.Tensor(yt)}
            exec(blocks[0], env)
            out["mixup_dispatch_type%d_%s" % (mtype, mode)] = {
                "x_shape": list(tf._raw(env["features_sup_may_mixuped"]).shape),
                "x": digest(tf._raw(env["features_sup_may_mixuped"])),
                "y": digest(tf._raw(env["onehot_labels"])),
                "yt": digest(tf._raw(env["teacher_labels"]))}
    tf.logging = saved_logging
    # nets/run_loop_classification.py:126-130: the `predictions` dict (classes / probabilities /
    # probabilities_sigmoid), the assignment statement executed from the source
    import ast
    src = open(os.path.join(REF_ROOT, "nets", "run_loop_classification.py")).read()
    fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == "resnet_model_fn")
    node = next(n for n in ast.walk(fn) if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", "") == "predictions")
    logits, _ = loss_inputs()
    env = {"tf": tf, "logits": tf.Tensor(logits)}
    exec(compile(ast.fix_missing_locations(ast.Module(body=[node], type_ignores=[])), "run_loop", "exec"), env)
    out["predictions"] = {k: digest(tf._raw(v).double()) for k, v in env["predictions"].items()}
    out["predictions"]["classes_list"] = [int(v) for v in tf._raw(env["predictions"]["classes"])]
    # functions/input_fns.py:98-102: the input pipeline delivers 2 x batch_size examples per step for mixup
    # type 1 in training (and only then)
    blocks, _ = reference_if_blocks("functions/input_fns.py", "input_fn_cls",
                                    "flags_obj.mixup_type == 1 and is_training")
    assert len(blocks) == 1
    out["input_batch"] = []
    for mtype in (0, 1, 2):
        for is_training in (True, False):
            env = {"flags_obj": types.SimpleNamespace(mixup_type=mtype, batch_size=256),
                   "is_training": is_training, "num_epochs": 3}
            exec(blocks[0], env)
            out["input_batch"].append([mtype, is_training, env["batch_size"]])
    # official/utils/misc/distribution_utils.py:48-76 per_device_batch_size (values and the error text)
    pdb, _ = reference_function("official/utils/misc/distribution_utils.py", "per_device_batch_size")
    out["per_device_batch"] = {"cases": [[b, n, pdb(b, n)] for b, n in PER_DEVICE_CASES]}
    try:
        pdb(2050, 8)
    except ValueError as e:
        out["per_device_batch"]["error_2050_8"] = str(e)
    # functions/model_fns.py:26-33 keep_prob_decay (the DropBlock schedule, :221-228)
    kp_decay, tf = reference_function("functions/model_fns.py", "keep_prob_decay")
    for name, (kp0, kp1, steps) in KEEP_PROB_CASES.items():
        fn = kp_decay(kp0, kp1, steps)
        out["keep_prob_" + name] = [float(tf._raw(fn(tf.Tensor(torch.tensor(s))))) for s in LR_STEPS]
    return out


if __name__ == "__main__":
    if len(sys.argv) != 2 or not os.path.isdir(os.path.join(sys.argv[1], "nets")):
        sys.exit("usage: python tests/golden/make_reference_shim_golden.py REFERENCE_DIR\n"
                 "  REFERENCE_DIR: a checkout of clovaai/assembled-cnn (the directory holding nets/)")
    REF_ROOT = os.path.abspath(sys.argv[1])
    gold = {"train_pieces": run_train_pieces()}
    print("train pieces:", sorted(gold["train_pieces"]))
    for name, (flags, d, b, s) in CONFIGS.items():
        gold[name], order = run_reference(flags, d, b, s)
        ws = reference_warm_start_list([o[0] for o in order if o[3]])
        gold[name]["num_warm_start"] = len(ws)
        gold[name]["warm_start_sha256"] = hashlib.sha256("\n".join(ws).encode()).hexdigest()
        print(name, gold[name]["num_variables"], gold[name]["eval_logits"]["abs_sum"])
    gold["c3_composition"] = run_reference_c3_composition()
    print("c3 composition", gold["c3_composition"]["cross_entropy"], len(gold["c3_composition"]["grads"]))
    for name, (flags, b, s, kp) in DROPBLOCK_CONFIGS.items():
        gold[name] = run_reference_dropblock(flags, b, s, kp)
        print(name, gold[name]["num_dropblock_calls"], gold[name]["train_logits"]["abs_sum"])
    json.dump(gold, open(OUT, "w"), indent=1, sort_keys=True)
    print("wrote", OUT)
