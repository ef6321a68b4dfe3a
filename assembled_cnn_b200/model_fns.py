"""The reference's operator surface for the hot path, executing on H100 through libacnn.so.

Mirrors (same names, argument meaning and error behaviour):
  * functions/model_fns.py:138-198   Model(resnet_size, data_format, num_classes, ...)
  * nets/resnet_model.py:305-310     model(inputs, training, reuse, use_resnet_d, keep_prob, return_embedding)
  * functions/model_fns.py:201-239   model_fn_cls(features, labels, mode, params)
  * nets/run_loop_classification.py:60-234  resnet_model_fn (loss assembly, train op)
  * functions/model_fns.py:36-95     learning_rate_with_decay ; :26-33 keep_prob_decay
  * metric/recall_metric.py:13-180   recall_at_k (the zero-shot retrieval evaluation)
  * mce/eval_robustness.py:161-326   show_corruption_error (the ImageNet-C robustness evaluation) as
                                     corruption_error
  * nets/run_loop_classification.py:397-402,446-448  classifier.evaluate(input_fn_eval) (the ImageNet
                                     classification evaluation) as evaluate_classification
  * metric/recall_metric.py:13-180 fed by functions/input_fns.py:148-165 (recall_at_k on the validation
                                     shards, run by --zeroshot_eval) as evaluate_retrieval
  * kd/extract_embeddings.py + datasets/build_imagenet_data.py --logits_file_path (the knowledge-
                                     distillation shards) as extract_teacher_logits
  * utils/export_utils.py:36-154     export_pb (the binary_input / preprocessed_input servables) and
                                     export_test as export_model, load_servable / Servable, export_test
plus `build_model(**flags)` (the name BASELINE.json uses; the reference has no such function).

The reference builds a TF graph and lets the Estimator run it; here a call executes on the GPU:
`Model.__call__` runs one forward, `Trainer.train_step` one full step (mixup -> forward -> loss ->
backward -> all-reduce -> SGD).  torch tensors are the device-memory container only.
"""
from __future__ import annotations

import os
import math
from collections import OrderedDict, deque, namedtuple

import numpy as np
import torch

from . import _lib, dp
from .hparams import DATASETS, DEFAULTS, get_loss_scale, params_from_flags
from .plan import BLOCK_SIZES, ModelConfig, build_plan
from .metrics import EvalMetrics, RecallAtK
from .native import NativeModel, NativeRuntime, check_dynamic_loss_scale
from .staging import StagingRing, pack_u8, read_ahead

DEFAULT_VERSION = 1
# dtype: 'bf16' = production path (bf16 storage, fp32 accumulation; the default); 'fp32' = the reference's
# default (nets/resnet_model.py:30-33, official/utils/flags/_performance.py:29-32): fp32 storage, 3-way
# bf16-split wgmma GEMMs, bit-reproducible reductions -- the mode the 1e-3 parity tests run in; 'fp16' =
# the reference's --dtype=fp16 (nets/resnet_model.py:251-303): fp32 variables read as fp16, fp16
# activation / gradient storage, wgmma .f16.f16 GEMMs with fp32 accumulation, fp32 logits and loss, and a
# static loss scale of 128 unless loss_scale is given (hparams.get_loss_scale).  fp16 keeps 10 mantissa
# bits where bf16 keeps 7, at the same tensor-core rate, but only 5 exponent bits: values above 65504
# become inf (as TF's cast does; nothing skips the step).
ALLOWED_TYPES = ("bf16", "fp32", "fp16")

# tf.estimator.ModeKeys values
TRAIN, EVAL, PREDICT = "train", "eval", "infer"

EstimatorSpec = namedtuple("EstimatorSpec", "mode predictions loss train_op eval_metric_ops")


def get_block_sizes(resnet_size, resnet_version=1):
    """functions/model_fns.py:98-135."""
    choices = BLOCK_SIZES[2 if resnet_version == 2 else 1]
    try:
        return choices[resnet_size]
    except KeyError:
        raise ValueError("Could not find layers for selected Resnet size.\n"
                         "Size received: {}; sizes allowed: {}.".format(resnet_size, choices.keys()))


def per_device_batch_size(batch_size, num_gpus):
    """official/utils/misc/distribution_utils.py:48-76: the global batch must divide over the replicas
    (same ValueError text)."""
    if num_gpus <= 1:
        return batch_size
    remainder = batch_size % num_gpus
    if remainder:
        raise ValueError("When running with multiple GPUs, batch size must be a multiple of the number of "
                         "available GPUs. Found {} GPUs with a batch size of {}; try --batch_size={} instead."
                         .format(num_gpus, batch_size, batch_size - remainder))
    return int(batch_size / num_gpus)


def keep_prob_decay(starter_kp, end_kp, decay_steps):
    """functions/model_fns.py:26-33 (linear polynomial decay, no cycle) as a host function."""
    def fn(global_step):
        s = min(global_step, decay_steps)
        return (starter_kp - end_kp) * (1 - s / decay_steps) + end_kp
    return fn


def learning_rate_with_decay(learning_rate_decay_type, batch_size, batch_denom, num_images,
                             num_epochs_per_decay, learning_rate_decay_factor, end_learning_rate,
                             piecewise_lr_boundary_epochs, piecewise_lr_decay_rates, base_lr,
                             warmup_epochs=0, train_epochs=None):
    """functions/model_fns.py:36-95; returns learning_rate_fn(global_step) -> python float."""
    initial = base_lr * batch_size / batch_denom
    bpe = num_images / batch_size
    decay_steps = int(bpe * num_epochs_per_decay)

    def learning_rate_fn(global_step):
        warmup_steps = int(bpe * warmup_epochs)
        g = global_step - warmup_steps
        if learning_rate_decay_type == "exponential":
            lr = initial * learning_rate_decay_factor ** math.floor(g / decay_steps)
        elif learning_rate_decay_type == "fixed":
            lr = base_lr
        elif learning_rate_decay_type == "polynomial":
            gg = min(g, decay_steps)
            lr = (initial - end_learning_rate) * (1 - gg / decay_steps) + end_learning_rate
        elif learning_rate_decay_type == "piecewise":
            bounds = [int(bpe * e) for e in piecewise_lr_boundary_epochs]
            vals = [initial * float(d) for d in piecewise_lr_decay_rates]
            lr = vals[sum(1 for b in bounds if global_step > b)]
        elif learning_rate_decay_type == "cosine":
            total = int(bpe * train_epochs) - warmup_steps
            gg = min(max(g, 0), total)
            lr = initial * 0.5 * (1 + math.cos(math.pi * gg / total))
        else:
            raise NotImplementedError
        if warmup_steps > 0 and global_step < warmup_steps:
            return initial * global_step / warmup_steps
        return lr
    return learning_rate_fn


def _truncated_normal(shape, std, gen):
    w = torch.empty(shape)
    torch.nn.init.trunc_normal_(w, 0.0, std, -2 * std, 2 * std, generator=gen)
    return w


class Model:
    """functions/model_fns.py:138-198 `Model` with ImageNet defaults (64 filters, 7x7/2 stem,
    3x3/2 pool, bottleneck blocks) + nets/resnet_model.py:166-249 argument checks."""

    def __init__(self, resnet_size, data_format=None, num_classes=None,
                 resnet_version=DEFAULT_VERSION, dtype="bf16", no_downsample=False,
                 zero_gamma=False, use_se_block=False, use_sk_block=False, bn_momentum=0.997,
                 embedding_size=0, anti_alias_filter_size=0, anti_alias_type="", pool_type="gap",
                 loss_type="softmax", bl_alpha=2, bl_beta=4, *, seed=42, device="cuda:0",
                 deterministic=None):
        if data_format not in (None, "channels_last"):
            raise ValueError("this implementation is NHWC only (data_format='channels_last')")
        if dtype not in ALLOWED_TYPES:
            raise ValueError("dtype must be one of: {}".format(ALLOWED_TYPES))
        self.resnet_size = int(resnet_size)
        self.num_classes = num_classes if num_classes is not None else 1001
        self.cfg_kwargs = dict(
            resnet_size=self.resnet_size, num_classes=self.num_classes,
            resnet_version=int(resnet_version), no_downsample=no_downsample, zero_gamma=zero_gamma,
            use_se_block=use_se_block, use_sk_block=use_sk_block, bn_momentum=bn_momentum,
            embedding_size=embedding_size, anti_alias_filter_size=anti_alias_filter_size,
            anti_alias_type=anti_alias_type, pool_type=pool_type, loss_type=loss_type,
            bl_alpha=bl_alpha, bl_beta=bl_beta)
        ModelConfig(**self.cfg_kwargs).validate()         # ValueError / NotImplementedError
        self.block_sizes = get_block_sizes(self.resnet_size, int(resnet_version))
        self.dtype = dtype
        self.data_format = "channels_last"
        self.device = device
        self.seed = seed
        # None: bit-reproducible steps in the fp32 mode only; True: also in bf16 (wgrad and the SE
        # fc GEMMs run without split-K -- slower); every other reduction is ordered in both modes
        self.deterministic = deterministic
        self._runtimes = {}          # (B, H, W, training, use_resnet_d, mixup, ls) -> NativeRuntime
        self._primary = {}           # use_resnet_d -> NativeRuntime owning the parameters
        self._pending_weights = None

    # ---------------------------------------------------------------- runtimes / parameters
    def runtime(self, batch, height, width, *, training, use_resnet_d=False, mixup_type=0,
                label_smoothing=0.0, with_loss=False, use_dropblock=False, kd_temp=0.0,
                fc_split_rows=0) -> NativeRuntime:
        """The runtime of one batch shape and mode, built on first use over this model's variables.
        fc_split_rows > batch (eval only): the SK / SE attention GEMMs split K as a batch of that many rows
        would (acnn_set_fc_split_rows), so each row gets the bits it gets in such a batch."""
        rows = int(fc_split_rows) if not training and int(fc_split_rows) > batch else 0
        key = (batch, height, width, bool(training), bool(use_resnet_d), mixup_type,
               float(label_smoothing), bool(with_loss or training), bool(use_dropblock and training),
               float(kd_temp) if training else 0.0, rows)
        rt = self._runtimes.get(key)
        if rt is None:
            cfg = ModelConfig(use_resnet_d=bool(use_resnet_d), **self.cfg_kwargs)
            step = dict(training=training, mixup_type=mixup_type, label_smoothing=label_smoothing,
                        with_loss=with_loss, dtype=self.dtype, use_dropblock=use_dropblock,
                        kd_temp=kd_temp)
            prim = self._primary.get(bool(use_resnet_d))
            # the layer plan is built and executed inside libacnn.so (include/acnn_model.h)
            nm = NativeModel(cfg, batch, height, width, deterministic=self.deterministic, **step)
            if rows:
                prev = nm.lib.acnn_set_fc_split_rows(rows)       # read by acnn_bind
                try:
                    rt = NativeRuntime(nm, self.device, share=prim)
                finally:
                    nm.lib.acnn_set_fc_split_rows(prev)
            else:
                rt = NativeRuntime(nm, self.device, share=prim)
            if prim is None:
                self._primary[bool(use_resnet_d)] = rt
                if self._pending_weights is not None:
                    rt.set_weights(self._pending_weights)
                else:
                    self.init_weights(rt)
            self._runtimes[key] = rt
        return rt

    def init_weights(self, rt: NativeRuntime):
        """The reference's initializers: variance_scaling (truncated normal, fan-in) for conv /
        SK / SE kernels (nets/model_helper.py:77), glorot-uniform dense kernel, zero bias
        (nets/resnet_model.py:595-597), gamma 1 (0 with zero_gamma on block-final BNs), beta 0."""
        gen = torch.Generator().manual_seed(self.seed)
        vals = {}
        for name, p in rt.plan.params.items():
            if p.kind == "conv_kernel":
                kh, kw, cin, cout = p.tf_shape
                std = math.sqrt(1.0 / (kh * kw * cin)) / 0.87962566103423978
                vals[name] = _truncated_normal(p.tf_shape, std, gen)
            elif p.kind == "dense_kernel":
                cin, cout = p.tf_shape
                lim = math.sqrt(6.0 / (cin + cout))
                vals[name] = (torch.rand(cin, cout, generator=gen) * 2 - 1) * lim
            elif p.kind == "gamma":
                vals[name] = torch.zeros(p.tf_shape) if p.zero_init else torch.ones(p.tf_shape)
            else:
                vals[name] = torch.zeros(p.tf_shape)
        for name, p in rt.plan.state.items():
            vals[name] = torch.ones(p.tf_shape) if p.kind == "moving_variance" \
                else torch.zeros(p.tf_shape)
        rt.set_weights(vals)

    def set_weights(self, tf_vars):
        """Load variables given in the reference's names and layouts (HWIO kernels, [in,out]
        dense kernel); applies to every runtime of this model."""
        self._pending_weights = tf_vars
        for rt in self._primary.values():
            rt.set_weights(tf_vars)

    def get_weights(self, use_resnet_d=None):
        if use_resnet_d is None:
            use_resnet_d = getattr(self, "use_resnet_d", False)
        rt = self._primary[bool(use_resnet_d)]
        names = list(rt.plan.params) + list(rt.plan.state)
        return {n: rt.get_tf(n).detach().float().cpu().clone() for n in names}

    # ---------------------------------------------------------------- forward
    def __call__(self, inputs, training, reuse=False, use_resnet_d=None, keep_prob=1.0,
                 return_embedding=False):
        """nets/resnet_model.py:305-599.  inputs: float32 [N,H,W,3] NHWC (CPU or CUDA tensor).
        Returns logits [N, num_classes] fp32 on the GPU (or the pooled embedding [N, C])."""
        # keep_prob == 1.0 (a Python float) is the reference's "DropBlock off" (nets/blocks.py:209);
        # anything else runs the DropBlock plan in training mode (inference ignores it, :205)
        use_db = bool(training) and not (isinstance(keep_prob, float) and keep_prob == 1.0)
        if use_resnet_d is None:
            # the reference's call-time default is False (nets/resnet_model.py:308); build_model()
            # records the flag it was given as the default of this model's calls
            use_resnet_d = getattr(self, "use_resnet_d", False)
        inputs = torch.as_tensor(inputs)
        if inputs.dim() != 4 or inputs.shape[-1] != 3:
            raise ValueError("inputs must be [N, H, W, 3] (NHWC)")
        n, h, w, _ = inputs.shape
        rt = self.runtime(n, h, w, training=False, use_resnet_d=use_resnet_d) if not training \
            else self.runtime(n, h, w, training=True, use_resnet_d=use_resnet_d,
                              use_dropblock=use_db)
        m = rt.plan.meta
        rt.t[m["images"]].copy_(inputs.to(torch.float32), non_blocking=True)
        if training:
            if use_db:
                self._fwd_calls = getattr(self, "_fwd_calls", 0) + 1
                rt.set_hparams(keep_prob=float(keep_prob), step=self._fwd_calls)
            rt.zero_step_buffers()
            fwd = [op for op in rt.plan.forward
                   if op.kind not in ("mix_labels", "softmax_ce", "kd_teacher")]
            rt.run(fwd)
        else:
            rt.run_forward()
        if return_embedding:
            # nets/resnet_model.py:586-590: the (BN-normalised) embedding when embedding_size > 0,
            # else the pooled features
            feat = rt.t[m["embedding"]] if "embedding" in m else rt.t[m["pooled"]]
            return feat.reshape(n, -1).float()
        return rt.t[m["logits"]][:, :self.num_classes]


def build_model(**flags) -> Model:
    """`build_model()` of BASELINE.json's north_star: the Model for a flag set
    (resnet_size, resnet_version, use_sk_block, use_se_block, anti_alias_type, ...).
    `use_resnet_d` is a call-time argument in the reference (nets/resnet_model.py:308); it is
    remembered here as the default of the returned model's calls via `model.use_resnet_d`."""
    use_resnet_d = flags.pop("use_resnet_d", False)
    ctor = {k: flags.pop(k) for k in list(flags) if k in (
        "resnet_size", "data_format", "num_classes", "resnet_version", "dtype", "no_downsample",
        "zero_gamma", "use_se_block", "use_sk_block", "bn_momentum", "embedding_size",
        "anti_alias_filter_size", "anti_alias_type", "pool_type", "loss_type", "bl_alpha",
        "bl_beta", "seed", "device", "deterministic")}
    if flags:
        raise TypeError("build_model: unknown flag(s) %s" % sorted(flags))
    ctor.setdefault("resnet_size", DEFAULTS["resnet_size"])
    model = Model(**ctor)
    model.use_resnet_d = bool(use_resnet_d)
    return model


def check_replicas_per_device(replicas_per_device):
    """replicas_per_device must be an integer >= 1 (ValueError otherwise); returns it as an int."""
    r = replicas_per_device
    if isinstance(r, bool) or not isinstance(r, (int, np.integer)) or r < 1:
        raise ValueError("replicas_per_device must be an integer >= 1 (got %r)" % (r,))
    return int(r)


class Trainer:
    """The data-parallel replicas of the training step this process runs (resnet_model_fn's TRAIN branch +
    get_train_op): owns the step's static buffers, the LR schedule and the CUDA graphs.

    replicas_per_device = R > 1 runs R replicas one after another on this device (micro-steps), each a full
    forward + backward of batch_size / (world * R) examples from the same moving statistics, as R GPUs of a
    MirroredStrategy run would: the gradients are summed in replica order, the updated moving statistics and
    the reported loss averaged (acnn_replica_accumulate), then one SGD step with grad_scale 1 / (world * R *
    loss_scale).  The reference's --num_gpus=N is world * replicas_per_device = N.

    params["loss_scale"] = "dynamic" turns on dynamic loss scaling, for every dtype (the rules at
    acnn_loss_scale_state in include/acnn.h, TF 2 Keras' LossScaleOptimizer): the scale starts at
    initial_loss_scale, a step whose summed (and all-reduced) gradients are not all finite leaves the weights
    and momentum as they were and halves the scale (not below 1), and loss_scale_growth_interval finite steps
    in a row double it.  The decision and the scale live on the device, inside the update graph: no host read.
    The moving statistics, the reported losses and the global step (so the LR and keep-prob schedules) advance
    on every step, skipped or not.  loss_scale_state() reads the state.

    train_metrics=True accumulates the training summaries' metrics on the device (acnn_classify_rows and
    acnn_train_metrics_accumulate after every micro-step's backward, on the current stream; no host read):
    the top-1 / top-5 hits and the ECE bins since reset_train_metrics(), and the step's rows and confidence
    sum (`train_metrics`, a TRAIN_METRICS_DTYPE record).  Only rank 0 accumulates, over the rows of all its
    micro-steps -- the whole global batch with one process.  Other ranks launch nothing and nothing is
    all-reduced, so summaries never add a collective to the step.  With mixup the labels are mixed and only
    the step's confidence is meaningful."""

    def __init__(self, model: Model, params: dict, height=224, width=224, *, use_cuda_graph=True,
                 lam_seed=7, num_images=None, replicas_per_device=1, train_metrics=False,
                 initial_loss_scale=2.0 ** 15, loss_scale_growth_interval=2000):
        """num_images: training images per epoch for the LR and keep-prob schedules (default: the
        dataset's data_config count).  initial_loss_scale and loss_scale_growth_interval apply with
        params["loss_scale"] = "dynamic" only."""
        p = params
        if p.get("cls_loss_type", "softmax") != "softmax":
            raise NotImplementedError("only cls_loss_type='softmax' is on the hot path")
        self.model = model
        self.p = p
        self.replicas = check_replicas_per_device(replicas_per_device)
        self.world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1
        self.local_batch = per_device_batch_size(p["batch_size"], self.world * self.replicas)
        # the reference's get_loss_scale: an explicit loss_scale wins, else 128 for fp16 and 1 otherwise
        loss_scale = get_loss_scale(p.get("loss_scale"), model.dtype)
        self.dynamic = loss_scale == "dynamic"
        if self.dynamic:
            check_dynamic_loss_scale(initial_loss_scale, loss_scale_growth_interval)
        self.mixup_type = int(p.get("mixup_type", 0))
        self.kd_temp = float(p.get("kd_temp", 0) or 0)
        self.use_dropblock = bool(p.get("use_dropblock", False))
        self.rt = model.runtime(self.local_batch, height, width, training=True,
                                use_resnet_d=p.get("use_resnet_d", False),
                                mixup_type=self.mixup_type,
                                label_smoothing=float(p.get("label_smoothing", 0.0)),
                                use_dropblock=self.use_dropblock, kd_temp=self.kd_temp)
        ds = DATASETS[p.get("dataset_name") or "imagenet"]
        if num_images is None:
            num_images = ds["num_images"]["train"]
        # functions/model_fns.py:221-228: keep_prob decays linearly over the whole run
        self.keep_prob_fn = None
        if self.use_dropblock:
            kp0, kp1 = p["dropblock_kp"]
            bpe = num_images / p["batch_size"]
            self.keep_prob_fn = keep_prob_decay(kp0, kp1, int(p["train_epochs"] * bpe))
        self.learning_rate_fn = learning_rate_with_decay(
            learning_rate_decay_type=p["learning_rate_decay_type"], batch_size=p["batch_size"],
            batch_denom=p["batch_size"], num_images=num_images,
            num_epochs_per_decay=p["num_epochs_per_decay"],
            learning_rate_decay_factor=p["learning_rate_decay_factor"],
            end_learning_rate=p["end_learning_rate"],
            piecewise_lr_boundary_epochs=p["piecewise_lr_boundary_epochs"],
            piecewise_lr_decay_rates=p["piecewise_lr_decay_rates"],
            base_lr=p["base_learning_rate"], train_epochs=p["train_epochs"],
            warmup_epochs=p["lr_warmup_epochs"])
        self.global_step = 0
        self.rng = np.random.default_rng(lam_seed)
        self.loss_scale = loss_scale
        if self.dynamic:
            self.rt.enable_dynamic_loss_scale(initial_loss_scale, loss_scale_growth_interval,
                                              self.world * self.replicas)
        else:
            self.rt.loss_scale = self.loss_scale
        self.use_graph = use_cuda_graph
        self._graphs = None
        m = self.rt.plan.meta
        self.images_buf = self.rt.t[m["images"]]
        self.labels_buf = self.rt.t[m["labels"]]
        self.lam1_buf = self.rt.t[m["lam1"]] if "lam1" in m else None
        self.lam2_buf = self.rt.t[m["lam2"]] if "lam2" in m else None
        self.teacher_buf = self.rt.t[m["teacher_logits"]] if "teacher_logits" in m else None
        # hyper-parameters reach the device through a RING of pinned host buffers (one per step in
        # flight, guarded by an event): the host may run several steps ahead of the GPU, and a
        # single buffer would be overwritten before its asynchronous copy has executed
        self._hp_ring = [torch.zeros(8, dtype=torch.float32).pin_memory() for _ in range(4)]
        self._hp_events = [None] * len(self._hp_ring)
        self._loss_slot = self.rt.slot_view(m["loss"])[:3 if self.kd_temp > 0 else 2]
        self._buckets = self._segments = None
        if self.world > 1:
            self._buckets = dp.grad_buckets(self.rt.plan)
            self._segments = dp.backward_segments(self.rt.plan, self._buckets)
        # several replicas: the accumulators (empty between global steps) and one graph per (phase, range)
        self._acc_bufs = self.rt.replica_buffers() if self.replicas > 1 else None
        self._acc_graphs = {}
        # input double-buffering: prefetch() copies the NEXT batch host->device on a side stream
        # while the current step computes; train_step() then takes it with a device-side copy
        self._copy_stream = torch.cuda.Stream(self.rt.dev)
        self._staged = None
        self._consumed = None
        self._stage_imgs = None
        self._stage_labs = None
        self._aug_work = None
        self._metrics = self._metric_rows = None
        rank = torch.distributed.get_rank() if torch.distributed.is_initialized() else 0
        if train_metrics and rank == 0:
            from .metrics import train_metrics_buffer
            self._metrics = train_metrics_buffer(self.rt.dev)
            self._metric_rows = tuple(torch.empty(self.local_batch, dtype=dt, device=self.rt.dev)
                                      for dt in (torch.int32, torch.float32, torch.int32, torch.float32))

    def loss_scale_state(self):
        """{scale, good_steps, skipped_steps} of dynamic loss scaling, with one device read (for tests and
        logging; the step never reads it); None with a static scale."""
        st = self.rt.loss_scale_state()
        return None if st is None else {k: st[k] for k in ("scale", "good_steps", "skipped_steps")}

    def set_loss_scale_state(self, scale, good_steps=0, skipped_steps=0):
        """Overwrite the dynamic state (a resumed run), on the current stream."""
        self.rt.set_loss_scale_state(scale, good_steps, skipped_steps)

    @property
    def train_metrics(self):
        """The device accumulator of the training metrics (uint8 [280], metrics.TRAIN_METRICS_DTYPE), or None
        when this Trainer does not accumulate them."""
        return self._metrics

    def reset_train_metrics(self):
        """Zero the accumulator, on the current stream."""
        if self._metrics is not None:
            self._metrics.zero_()

    def _accumulate_metrics(self, r):
        """classify_rows (k = 5) and acnn_train_metrics_accumulate on micro-step r's logits and labels, which
        the next micro-step overwrites."""
        from .metrics import classify_rows, train_metrics_accumulate
        B = self.local_batch
        logits = self.rt.t[self.rt.plan.meta["logits"]][:B, :self.model.num_classes]
        classify_rows(logits, self.labels_buf, k=5, out=self._metric_rows)
        train_metrics_accumulate(self._metric_rows, self.labels_buf, self._metrics, B, step_begin=r == 0)

    @property
    def input_batch(self):
        """Examples the input pipeline must deliver per replica and step (2x for mixup type 1,
        functions/input_fns.py:98-100)."""
        return self.rt.plan.meta["input_batch"]

    def _capture(self):
        rt = self.rt
        # warm-up launch outside capture (cudaFuncSetAttribute, driver entry points, ...); it is
        # a real forward/backward, so the BN moving statistics it updated are put back
        state_backup = rt.state.clone()
        self._fwd_bwd()
        if self.replicas > 1:     # SAVE only writes the (empty) state_base
            rt.replica_accumulate(rt.REPLICA_SAVE, self._acc_bufs, 0, rt.plan.param_elems, self.replicas)
        torch.cuda.synchronize()
        rt.state.copy_(state_backup)
        s = torch.cuda.Stream(rt.dev)
        s.wait_stream(torch.cuda.current_stream(rt.dev))
        # one graph for forward + backward on a single GPU; with data parallelism the backward is cut
        # at the gradient-bucket boundaries (the all-reduces are issued between the graph replays)
        fns = [self._fwd_bwd]
        if self.world > 1:
            bwd = rt.plan.backward
            fns = []
            for k, (a, b) in enumerate(self._segments):
                if k == 0:
                    fns.append(lambda ops=bwd[a:b]: (rt.run_forward(), rt.run(ops)))
                else:
                    fns.append(lambda ops=bwd[a:b]: rt.run(ops))
        graphs = []
        with torch.cuda.stream(s):
            for fn in fns + [rt.run_update]:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    fn()
                graphs.append(g)
            for key in self._accumulate_variants():
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    rt.replica_accumulate(key[0], self._acc_bufs, key[1], key[2], self.replicas)
                self._acc_graphs[key] = g
        torch.cuda.current_stream(rt.dev).wait_stream(s)
        self._graphs = graphs

    def _accumulate_variants(self):
        """(phase, lo, hi) of every accumulate call of a global step: none with one replica; SAVE, FIRST and
        MIDDLE over the whole gradient buffer; LAST over it, or per gradient bucket with data parallelism."""
        if self.replicas == 1:
            return []
        n, rt = self.rt.plan.param_elems, self.rt
        last = [(0, n)] if self.world == 1 else [(lo, hi) for lo, hi, _ in self._buckets]
        return [(rt.REPLICA_SAVE, 0, n), (rt.REPLICA_FIRST, 0, n), (rt.REPLICA_MIDDLE, 0, n)] + \
            [(rt.REPLICA_LAST, lo, hi) for lo, hi in last]

    def _accumulate(self, phase, lo, hi):
        if self.use_graph:
            self._acc_graphs[(phase, lo, hi)].replay()
        else:
            self.rt.replica_accumulate(phase, self._acc_bufs, lo, hi, self.replicas)

    def _phase(self, r):
        """The accumulate phase after micro-step r (None with one replica)."""
        rt = self.rt
        if self.replicas == 1:
            return None
        return rt.REPLICA_FIRST if r == 0 else (rt.REPLICA_LAST if r == self.replicas - 1 else rt.REPLICA_MIDDLE)

    def _fwd_bwd(self):
        rt = self.rt
        rt.run_forward()
        rt.run(rt.plan.backward)

    def prefetch(self, images, labels):
        """Start the host->device copy of the next step's inputs (pinned host tensors) on a side
        stream; the following train_step(None, None) consumes them.  Lets the PCIe transfer of
        step i+1 overlap the compute of step i."""
        if self._stage_imgs is None:
            n = self.replicas * self.input_batch
            self._stage_imgs = self.images_buf.new_empty((n,) + tuple(self.images_buf.shape[1:]))
            self._stage_labs = self.labels_buf.new_empty((n,))
        cs = self._copy_stream
        # the staging buffers may still be read by the previous step's device-side copy (and only
        # by that: waiting for the whole main stream would serialise the transfer behind the step)
        if self._consumed is not None:
            cs.wait_event(self._consumed)
        with torch.cuda.stream(cs):
            self._stage_imgs.copy_(images, non_blocking=True)
            self._stage_labs.copy_(labels, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(cs)
        self._staged = ev

    def train_step(self, images=None, labels=None, lam1=None, lam2=None, teacher_logits=None,
                   keep_prob=None):
        """images fp32 [input_batch,H,W,3] and int32 labels [input_batch] (pinned host or device),
        or None to consume the batch given to prefetch().  teacher_logits fp32 [input_batch, classes]
        when kd_temp > 0 (the second half of the reference's KD label tensor).  keep_prob overrides
        the DropBlock schedule for this step.  With R = replicas_per_device > 1, images, labels and
        teacher_logits hold R * input_batch rows, replica-major, and lam1 / lam2 are [R, input_batch / 2].
        Returns the device tensor [cross_entropy, l2_loss(, kd_loss)] of this process (the mean over its
        replicas; read it with .tolist() -- that read is the only host sync of the step)."""
        rt = self.rt
        if images is None:
            if self._staged is None:
                raise ValueError("train_step() without inputs needs a preceding prefetch()")
            torch.cuda.current_stream(rt.dev).wait_event(self._staged)
            self._staged = None
            images, labels = self._stage_imgs, self._stage_labs
        n = self.input_batch
        if self.replicas > 1 and (images.shape[0] != self.replicas * n or labels.shape[0] != self.replicas * n):
            raise ValueError("train_step: images and labels need %d x %d rows, got %d and %d"
                             % (self.replicas, n, images.shape[0], labels.shape[0]))

        def load(r):
            rows = slice(r * n, (r + 1) * n)
            self.images_buf.copy_(images[rows] if self.replicas > 1 else images, non_blocking=True)
            self.labels_buf.copy_(labels[rows] if self.replicas > 1 else labels, non_blocking=True)
            if images is self._stage_imgs and r == self.replicas - 1:
                self._consumed = torch.cuda.Event()
                self._consumed.record(torch.cuda.current_stream(rt.dev))
        return self._step(load, lam1, lam2, teacher_logits, keep_prob)

    def train_step_cropped(self, desc, labels, mean, lam1=None, lam2=None, teacher_logits=None, keep_prob=None,
                           augment=None):
        """train_step with the images made on the device from training crop windows: one
        acnn_set_images_cropped launch (flip, resize to H x W, - mean) on the current stream, then the step.
        desc: a CUDA uint8 tensor of input_batch 32-byte acnn_crop_desc (imagenet_train.CROP_DESC_DTYPE,
        checked by the caller); labels int32 [input_batch]; the rest as train_step.
        augment: None, or a CUDA uint8 tensor of input_batch 88-byte AutoAugment descriptors
        (autoaugment.AUTOAUG_DESC_DTYPE, checked by the caller with check_autoaugment_descriptors); then the
        images come from acnn_set_images_augmented instead, through a work buffer allocated on first use.
        With R = replicas_per_device > 1, desc, labels, augment and teacher_logits hold R * input_batch rows,
        replica-major, and lam1 / lam2 are [R, input_batch / 2]."""
        n, R = self.input_batch, self.replicas
        if R > 1 and (desc.numel() != 32 * R * n or labels.shape[0] != R * n
                      or (augment is not None and augment.numel() != 88 * R * n)):
            raise ValueError("train_step_cropped: desc, labels (and augment) need %d x %d rows" % (R, n))
        if augment is not None and self._aug_work is None:
            b, s = self.images_buf.shape[0], self.images_buf.shape[1]
            self._aug_work = torch.empty(self.rt.lib.acnn_autoaugment_work_bytes(b, s), dtype=torch.uint8,
                                         device=self.rt.dev)

        def rows(t, width, r):
            return t[r * n * width:(r + 1) * n * width] if R > 1 else t

        def load(r):
            if augment is None:
                self.rt.set_images_cropped(rows(desc, 32, r), mean)
            else:
                self.rt.set_images_augmented(rows(desc, 32, r), rows(augment, 88, r), self._aug_work, mean)
            self.labels_buf.copy_(rows(labels, 1, r), non_blocking=True)
        return self._step(load, lam1, lam2, teacher_logits, keep_prob)

    def _micro_inputs(self, r, lam1, lam2, teacher_logits):
        """The mixup lambdas and teacher logits of micro-step r (drawn from self.rng when not given)."""
        R, n = self.replicas, self.input_batch

        def lam(given, buf):
            v = self.rng.beta(0.2, 0.2, n // 2).astype(np.float32) if given is None \
                else torch.as_tensor(given).reshape(R, n // 2)[r]
            buf.copy_(torch.as_tensor(v, dtype=torch.float32), non_blocking=True)
        if self.mixup_type:
            lam(lam1, self.lam1_buf)
            if self.mixup_type == 2:
                lam(lam2, self.lam2_buf)
        if self.kd_temp > 0:
            t = torch.as_tensor(teacher_logits, dtype=torch.float32)
            self.teacher_buf.copy_(t[r * n:(r + 1) * n] if R > 1 else t, non_blocking=True)

    def _step(self, load, lam1, lam2, teacher_logits, keep_prob):
        rt = self.rt
        if self.kd_temp > 0 and teacher_logits is None:
            raise ValueError("kd_temp > 0: train_step needs teacher_logits")
        if self.kd_temp > 0 and self.replicas > 1 and teacher_logits.shape[0] != self.replicas * self.input_batch:
            raise ValueError("train_step: teacher_logits need %d x %d rows" % (self.replicas, self.input_batch))
        lr = self.learning_rate_fn(self.global_step)
        slot = self.global_step % len(self._hp_ring)
        if self._hp_events[slot] is not None:
            self._hp_events[slot].synchronize()          # its copy of 4 steps ago has executed
        hp = self._hp_ring[slot]
        hp[0] = lr
        hp[1] = self.p["momentum"]
        hp[2] = self.p["weight_decay"]
        # dynamic loss scaling takes the gradient scale from its device state
        hp[3] = 0.0 if self.dynamic else 1.0 / (self.world * self.replicas * self.loss_scale)
        if keep_prob is None:
            keep_prob = self.keep_prob_fn(self.global_step) if self.keep_prob_fn else 1.0
        hp[4] = keep_prob
        hp.view(torch.int32)[5] = self.global_step & 0x7fffffff      # Philox counter of the masks
        rt.hp.copy_(hp, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(rt.dev))
        self._hp_events[slot] = ev
        for r in range(self.replicas):
            load(r)
            self._micro_inputs(r, lam1, lam2, teacher_logits)
            if r == 0:
                if self.use_graph and self._graphs is None:
                    self._capture()
                if self.replicas > 1:
                    self._accumulate(rt.REPLICA_SAVE, 0, rt.plan.param_elems)
            phase = self._phase(r)
            if self.world == 1:
                if self.use_graph:
                    self._graphs[0].replay()
                else:
                    self._fwd_bwd()
                if phase is not None:
                    self._accumulate(phase, 0, rt.plan.param_elems)
            else:
                self._fwd_bwd_allreduce(phase)
            if self._metrics is not None:
                self._accumulate_metrics(r)
        if self.use_graph:
            self._graphs[-1].replay()
        else:
            rt.run_update()
        if self.world > 1:
            self.sync_moving_statistics()
        self.global_step += 1
        self.last_lr = lr
        self.last_keep_prob = keep_prob
        return self._loss_slot

    # ---------------------------------------------------------------- data parallelism
    def sync_moving_statistics(self):
        """MirroredStrategy keeps the BN moving statistics as mirrored variables whose per-replica
        updates are MEAN-aggregated (official/utils/misc/distribution_utils.py:24-45)."""
        dp.average_moving_statistics(self.rt.state, self.world)

    def _fwd_bwd_allreduce(self, phase=None):
        """forward + backward with the gradient all-reduce overlapped: the backward is cut into
        segments (each its own CUDA graph), and as soon as a segment has produced the last gradient
        of a bucket that bucket is all-reduced asynchronously on NCCL's stream while the next
        segment computes (assembled_cnn_b200/dp.py).  With several replicas per device (phase = the
        accumulate phase of this micro-step) only the last micro-step all-reduces, each bucket right
        after its LAST accumulation; the earlier ones accumulate the whole buffer after the backward."""
        rt = self.rt
        reduce = phase is None or phase == rt.REPLICA_LAST
        works, k = [], 0
        for ev in dp.schedule(self._buckets, self._segments):
            if ev[0] == "run":
                if self.use_graph:
                    self._graphs[k].replay()
                else:
                    if k == 0:
                        rt.run_forward()
                    rt.run(rt.plan.backward[ev[1]:ev[2]])
                k += 1
            elif reduce:
                if phase is not None:
                    self._accumulate(phase, ev[1], ev[2])
                works.append(dp.all_reduce_bucket(rt.grads, ev[1], ev[2], async_op=True))
        for w in works:
            w.wait()            # stream-level wait: the update runs after every bucket
        if not reduce:
            self._accumulate(phase, 0, rt.plan.param_elems)


_TRAINERS = {}


def l2_loss(rt: NativeRuntime, weight_decay: float):
    """weight_decay * sum over the decayed variables of |v|^2 / 2 (run_loop_classification.py:
    166-177), from the flat master buffer and its per-256-element decay flags.  TRAIN gets the same
    number from the SGD kernel; this is the EVAL-mode path (a reduction over 42 M floats, once per
    evaluation batch)."""
    w = rt.params.view(-1, 256)
    return 0.5 * weight_decay * (w[rt.decay_flags.bool()[:w.shape[0]]].double() ** 2).sum().float()


def predictions_of(logits):
    """nets/run_loop_classification.py:126-130: the `predictions` dict of the EstimatorSpec."""
    return {"classes": logits.argmax(dim=1), "probabilities": torch.softmax(logits, dim=1),
            "probabilities_sigmoid": torch.sigmoid(logits)}


def model_fn_cls(features, labels, mode, params):
    """functions/model_fns.py:201-239 -> nets/run_loop_classification.py:60-234.

    features: {'image': float32 [N,H,W,3]} (or the tensor itself in PREDICT mode), labels: int32 [N]
    -- or, with kd_temp > 0, the reference's float KD label tensor [N, 2*num_classes] = one-hot
    labels ++ teacher logits (nets/run_loop_classification.py:86-93).
    TRAIN executes one training step and returns the spec with its loss; EVAL returns loss
    (cross-entropy + L2, as the reference) and predictions of a forward pass with moving statistics
    plus the accuracy / top-5 / ECE metrics; PREDICT only predictions.
    """
    if int(params["resnet_size"]) < 50:
        assert not params.get("use_dropblock")
        assert not params.get("use_se_block")
        assert not params.get("use_sk_block")
        assert not params.get("use_resnet_d")
    p = params_from_flags(**{k: v for k, v in params.items() if k in DEFAULTS})
    ds = DATASETS[p.get("dataset_name") or "imagenet"]
    images = features["image"] if isinstance(features, dict) else features
    images = torch.as_tensor(images)
    key = tuple(sorted((k, str(v)) for k, v in p.items())) + (tuple(images.shape[1:3]),)
    entry = _TRAINERS.get(key)
    if entry is None:
        model = Model(p["resnet_size"], p["data_format"], num_classes=ds["num_classes"],
                      resnet_version=p["resnet_version"], zero_gamma=p["zero_gamma"],
                      use_se_block=p["use_se_block"], use_sk_block=p["use_sk_block"],
                      no_downsample=p["no_downsample"],
                      anti_alias_filter_size=p["anti_alias_filter_size"],
                      anti_alias_type=p["anti_alias_type"], bn_momentum=p["bn_momentum"],
                      embedding_size=p["embedding_size"], pool_type=p["pool_type"],
                      bl_alpha=p["bl_alpha"], bl_beta=p["bl_beta"], dtype=p["dtype"],
                      loss_type=p["cls_loss_type"])
        entry = _TRAINERS[key] = {"model": model, "trainer": None}
    model = entry["model"]

    if mode == PREDICT:
        logits = model(images, False, False, use_resnet_d=p["use_resnet_d"])
        return EstimatorSpec(mode, predictions_of(logits), None, None, None)
    teacher_logits = None
    if mode != PREDICT and p.get("kd_temp", 0) > 0:
        kd_labels = torch.as_tensor(labels, dtype=torch.float32)
        if kd_labels.dim() != 2 or kd_labels.shape[1] != 2 * ds["num_classes"]:
            raise ValueError("kd_temp > 0: labels must be [N, 2*num_classes] (one-hot ++ teacher "
                             "logits, nets/run_loop_classification.py:86-93)")
        onehot, teacher_logits = kd_labels.split(ds["num_classes"], dim=1)
        labels = onehot.argmax(dim=1).to(torch.int32)
    if mode == TRAIN:
        if entry["trainer"] is None:
            entry["trainer"] = Trainer(model, p, images.shape[1], images.shape[2])
        tr = entry["trainer"]
        loss = tr.train_step(images, torch.as_tensor(labels, dtype=torch.int32),
                             teacher_logits=teacher_logits)
        m = tr.rt.plan.meta
        logits = tr.rt.t[m["logits"]][:, :model.num_classes]
        return EstimatorSpec(mode, predictions_of(logits), loss.sum(), tr, None)
    if mode == EVAL:
        n, h, w, _ = images.shape
        rt = model.runtime(n, h, w, training=False, use_resnet_d=p["use_resnet_d"],
                           label_smoothing=p["label_smoothing"], with_loss=True)
        m = rt.plan.meta
        rt.t[m["images"]].copy_(images.to(torch.float32), non_blocking=True)
        rt.t[m["labels"]].copy_(torch.as_tensor(labels, dtype=torch.int32), non_blocking=True)
        rt.run_forward()
        logits = rt.t[m["logits"]][:, :model.num_classes]
        lab = rt.t[m["labels"]].long()
        pred = predictions_of(logits)
        # eval_metric_ops are streaming in the reference (tf.metrics.*): they accumulate over the
        # batches of one evaluation; reset with model_fn_cls.reset_metrics(params)
        em = entry.setdefault("metrics", EvalMetrics(device=logits.device))
        metrics = em.update(logits, lab)
        # loss = cross_entropy + l2_loss in EVAL too (nets/run_loop_classification.py:166-179)
        loss = rt.slot_view(m["loss"])[0] + l2_loss(rt, p["weight_decay"])
        if teacher_logits is not None:
            t = torch.softmax(teacher_logits.to(logits.device) / p["kd_temp"], dim=1)
            loss = loss + p["kd_temp"] ** 2 * -(t * torch.log_softmax(logits / p["kd_temp"], 1)
                                                ).sum(1).mean()
        return EstimatorSpec(mode, pred, loss, None, metrics)
    raise ValueError("unknown mode %r" % (mode,))


def reset_metrics(params=None):
    """Start a new evaluation: drop the streaming accuracy / ECE accumulators."""
    for entry in _TRAINERS.values():
        entry.pop("metrics", None)


model_fn_cls.reset_metrics = reset_metrics


def recall_at_k(model, batches, num_val_images, recall_at_k=(1, 5), eval_similarity="cosine",
                use_resnet_d=False, return_embedding=True, global_step=None):
    """metric/recall_metric.py:13-180, the evaluation of `--zeroshot_eval`: embeds every batch of
    `batches` (an iterable of (images [N,H,W,3], labels [N]); label -1 marks a distractor) with
    `model(images, False, use_resnet_d=..., return_embedding=...)`, then Recall@K of every k in
    `recall_at_k` over queries = non-distractor rows against the index = all rows (RecallAtK).
    The similarity search runs in the model's dtype ('fp32': three bf16 planes per operand), as the
    reference feeds fp32 or fp16 placeholders by `flags_obj.dtype`.
    Returns {'recall_at_<k>': ..., 'global_step': global_step}."""
    dev = torch.device(model.device)
    metric = RecallAtK(recall_at_k, similarity=eval_similarity, dtype=model.dtype, device=dev)
    for images, labels in batches:
        emb = model(images, False, use_resnet_d=use_resnet_d, return_embedding=return_embedding)
        metric.update(emb, labels)
    assert metric.count == num_val_images, (metric.count, num_val_images)
    out = {"recall_at_%d" % k: v for k, v in metric.result().items()}
    out["global_step"] = global_step
    return out


def _replica(model, device, use_resnet_d, batch, size):
    """`model` itself on its device, else a Model of the same flags on `device` with its weights."""
    if torch.device(device) == torch.device(model.device):
        return model
    src = model.runtime(batch, size, size, training=False, use_resnet_d=use_resnet_d)
    names = list(src.plan.params) + list(src.plan.state)
    rep = Model(dtype=model.dtype, seed=model.seed, device=device, deterministic=model.deterministic,
                **model.cfg_kwargs)
    rep.set_weights({n: src.get_tf(n).detach().float().cpu().clone() for n in names})
    return rep


class _EvalPipeline(StagingRing):
    """The evaluation loop of one device: each batch is staged from a ring of pinned host sets into one of two
    device slots on the copy stream, overlapped with the previous batch's forward; the device work of a batch
    (`_body`: input preparation, eval forward, metric kernel) runs as one CUDA graph per (slot, valid rows).
    A subclass gives the host sets and slots, stages a batch's labels beside its images (`_fill`) and defines
    `_body`."""

    def __init__(self, model, batch, size, use_resnet_d, use_cuda_graph, host, slots, fc_split_rows=0):
        torch.cuda.set_device(model.device)
        super().__init__(torch.device(model.device), host, slots)
        self.rt = model.runtime(batch, size, size, training=False, use_resnet_d=use_resnet_d,
                                fc_split_rows=fc_split_rows)
        self.batch, self.use_graph = batch, use_cuda_graph
        self.logits = self.rt.t[self.rt.plan.meta["logits"]][:, :model.num_classes]
        self.graphs = {}
        self.warm = False

    def _graph(self, slot, n_valid):
        g = self.graphs.get((slot, n_valid))
        if g is None:
            main = torch.cuda.current_stream(self.dev)
            s = torch.cuda.Stream(self.dev)
            s.wait_stream(main)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s):
                # thread_local: the other devices' threads keep allocating and launching meanwhile
                with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
                    self._body(slot, n_valid)
            main.wait_stream(s)
            self.graphs[(slot, n_valid)] = g
        return g

    def _run(self, place, labels):
        """Evaluate one batch of len(labels) <= batch rows, whose images place(h, slot) stages."""
        n = len(labels)
        self.push(lambda h, slot: self._fill(h, slot, place, labels))
        slot = self.take()
        if self.use_graph and self.warm:
            self._graph(slot, n).replay()
        else:
            self._body(slot, n)        # the first batch also loads every kernel before any capture
            self.warm = True
        self.release(slot)


class _CorruptionEvalDevice(_EvalPipeline):
    """The robustness evaluation's loop: fixed-size uint8 batches; the u8 -> f32 input conversion, the
    eval forward and the top-1 count run as one CUDA graph per (slot, valid rows)."""

    def __init__(self, model, batch, size, use_resnet_d, use_cuda_graph):
        dev, u8 = torch.device(model.device), dict(dtype=torch.uint8)
        host = [(torch.zeros(batch, size, size, 3, **u8).pin_memory(),
                 torch.zeros(batch, dtype=torch.int32).pin_memory()) for _ in range(self.RING)]
        slots = [(torch.zeros(batch, size, size, 3, **u8, device=dev),
                  torch.zeros(batch, dtype=torch.int32, device=dev)) for _ in range(2)]
        super().__init__(model, batch, size, use_resnet_d, use_cuda_graph, host, slots)
        self.acc = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.pred = torch.zeros(batch, dtype=torch.int32, device=self.dev)

    def run_batch(self, images, labels):
        """Evaluate uint8 [H, W, 3] arrays `images` with int `labels`."""
        def place(h, slot):
            hu8, du8 = self.host[h][0], self.slots[slot][0]
            for i, a in enumerate(images):
                hu8[i].copy_(torch.from_numpy(a))
            du8.copy_(hu8, non_blocking=True)
        self._run(place, labels)

    def run_batch_encoded(self, buffers, labels, files):
        """run_batch from the encoded bytes of `files`, decoded on the copy stream straight into the slot
        (jpeg.JpegDecoder; PIL, through imagenet_c.decode_image, for the images the device does not decode)."""
        from . import imagenet_c, jpeg

        def place(h, slot):
            du8 = self.slots[slot][0]
            S = du8.shape[1]
            for i, d in enumerate(jpeg.parse(buffers)):   # a wrong size raises decode_image's error, as PIL's does
                if d["supported"] and (int(d["height"]), int(d["width"])) != (S, S):
                    imagenet_c.decode_image(files[i], S)
            self.decoder(slot).stage(buffers, None, self.copy_stream,
                                     fallback=lambda i: imagenet_c.decode_image(files[i], S),
                                     out=du8.view(-1), out_offsets=np.arange(len(buffers), dtype=np.int64) * S * S * 3)
        self._run(place, labels)

    def _fill(self, h, slot, place, labels):
        place(h, slot)
        hlab, dlab = self.host[h][1], self.slots[slot][1]
        hlab[:len(labels)].copy_(torch.as_tensor(labels, dtype=torch.int32))
        dlab.copy_(hlab, non_blocking=True)

    def _body(self, slot, n_valid):
        from .metrics import softmax_top1_count
        images, labels = self.slots[slot]
        self.rt.set_images_u8(images, self.mean)
        self.rt.run_forward()
        softmax_top1_count(self.logits, labels, self.acc, n_valid, self.pred)

    def take_count(self):
        """The device count of correct predictions since the last call (a device tensor; no sync)."""
        c = self.acc.clone()
        self.acc.zero_()
        return c


class _ResizedEvalPipeline(_EvalPipeline):
    """The input side of the evaluations over TFRecord shards: decoded images of any sizes are packed into a
    growable pinned uint8 buffer with one acnn_resize_desc per image, or decoded on the device
    (run_batch_encoded), and the batch's labels (`label_dtype`) go to the device slot with them; a subclass's
    `_body` starts with rt.set_images_resized (resize + crop + mean)."""

    def __init__(self, model, batch, size, use_resnet_d, use_cuda_graph, label_dtype=torch.int32,
                 fc_split_rows=0):
        dev, lab = torch.device(model.device), dict(dtype=label_dtype)
        # pinned image bytes (grown on demand), labels, descriptors
        host = [[None, torch.zeros(batch, **lab).pin_memory(), torch.zeros(32 * batch, dtype=torch.uint8).pin_memory()]
                for _ in range(self.RING)]
        # device image bytes (allocated on the copy stream, grown on demand), labels, descriptors: a graph
        # holds the descriptor table's address only, so the image bytes may move
        slots = [[None, torch.zeros(batch, **lab, device=dev), torch.zeros(32 * batch, dtype=torch.uint8, device=dev)]
                 for _ in range(2)]
        super().__init__(model, batch, size, use_resnet_d, use_cuda_graph, host, slots, fc_split_rows)
        self.size = size

    def run_batch(self, images, labels):
        """Evaluate (uint8 [H, W, 3] array, imagenet_eval.eval_geometry) pairs `images` with int `labels`."""
        def place(h, slot):
            self.host[h][0], self.slots[slot][0], addrs = pack_u8(self.host[h][0], self.slots[slot][0],
                                                                 [a for a, _ in images], self.dev)
            return [((addr, a.shape[0], a.shape[1]), g) for addr, (a, g) in zip(addrs, images)]
        self._run(place, labels)

    def run_batch_encoded(self, buffers, labels, geometry):
        """run_batch from encoded images (jpeg.JpegDecoder on the copy stream; PIL for the images the device
        does not decode); geometry(h, w) gives an image's imagenet_eval.eval_geometry."""
        def place(h, slot):
            return [(p, geometry(p[1], p[2])) for p in self.decoder(slot).stage(buffers, None, self.copy_stream)]
        self._run(place, labels)

    def _fill(self, h, slot, place, labels):
        from .imagenet_eval import DESC_DTYPE, check_descriptors
        _, hlab, hdesc = self.host[h]
        desc = hdesc.numpy().view(DESC_DTYPE)
        for i, ((addr, ih, iw), (s, rh, rw, cy, cx)) in enumerate(place(h, slot)):
            desc[i] = (addr, ih, iw, rh, rw, cy, cx)
        check_descriptors(desc, len(labels), self.size)
        hlab[:len(labels)].copy_(torch.as_tensor(labels, dtype=hlab.dtype))
        _, dlab, ddesc = self.slots[slot]
        ddesc.copy_(hdesc, non_blocking=True)
        dlab.copy_(hlab, non_blocking=True)


class _ClassifyEvalDevice(_ResizedEvalPipeline):
    """The classification evaluation's loop: resize + crop + mean, the eval forward and the per-row metrics
    (acnn_classify_rows) run as one CUDA graph per (slot, valid rows).  The per-row results of every batch
    are appended to device arrays of `total` rows (`rows`), read once at the end."""

    def __init__(self, model, batch, size, use_resnet_d, use_cuda_graph, label_smoothing, total):
        super().__init__(model, batch, size, use_resnet_d, use_cuda_graph)
        self.label_smoothing = float(label_smoothing)
        kinds = (torch.int32, torch.float32, torch.int32, torch.float32)       # pred, conf, hit_5, ce
        self.out = tuple(torch.zeros(batch, dtype=dt, device=self.dev) for dt in kinds)
        self.rows = tuple(torch.zeros(total, dtype=dt, device=self.dev) for dt in kinds)
        self.done = 0

    def _body(self, slot, n_valid):
        from .metrics import classify_rows
        _, labels, desc = self.slots[slot]
        self.rt.set_images_resized(desc, n_valid, self.mean)
        self.rt.run_forward()
        classify_rows(self.logits, labels, n_valid, 5, self.label_smoothing, out=self.out)

    def _run(self, place, labels):
        super()._run(place, labels)
        n = len(labels)
        for dst, src in zip(self.rows, self.out):
            dst[self.done:self.done + n].copy_(src[:n])
        self.done += n


class _RetrievalEvalDevice(_ResizedEvalPipeline):
    """The retrieval evaluation's loop: resize + crop + mean and the eval forward run as one CUDA graph per
    (slot, valid rows), which also copies the slot's int64 labels beside the model's outputs.  After each
    batch its valid rows are appended to the device index: `index` fp32 [total, d] (the embedding, else the
    pooled features, with return_embedding; the logits without, as Model.__call__ returns) and `labels`
    int64 [total]."""

    def __init__(self, model, batch, size, use_resnet_d, use_cuda_graph, return_embedding, total):
        super().__init__(model, batch, size, use_resnet_d, use_cuda_graph, label_dtype=torch.int64)
        m = self.rt.plan.meta
        if return_embedding:
            self.feat = self.rt.t[m["embedding"] if "embedding" in m else m["pooled"]].reshape(batch, -1)
        else:
            self.feat = self.logits
        self.batch_labels = torch.zeros(batch, dtype=torch.int64, device=self.dev)
        self.index = torch.zeros(total, self.feat.shape[1], dtype=torch.float32, device=self.dev)
        self.labels = torch.zeros(total, dtype=torch.int64, device=self.dev)
        self.done = 0

    def _body(self, slot, n_valid):
        _, labels, desc = self.slots[slot]
        self.rt.set_images_resized(desc, n_valid, self.mean)
        self.rt.run_forward()
        # the slot is refilled two batches later: its labels are read here, before the batch's event
        self.batch_labels.copy_(labels)

    def _run(self, place, labels):
        super()._run(place, labels)
        n = len(labels)
        self.index[self.done:self.done + n].copy_(self.feat[:n])
        self.labels[self.done:self.done + n].copy_(self.batch_labels[:n])
        self.done += n


def _read_file(path):
    with open(path, "rb") as f:
        return f.read()


def corruption_error(model, data_dir, label_file, *, batch_size=128, image_size=224, label_offset=1,
                     robustness_type="ce", devices=None, use_resnet_d=None, global_step=None,
                     use_cuda_graph=True, num_workers=None, summary_dir=None):
    """mce/eval_robustness.py (show_corruption_error, --robustness_type ce): the top-1 error of `model`
    on every distortion of ALEXNET_CE, pooled over data_dir/<distortion>/<severity 1..5>/<synset>/*,
    its AlexNet-normalised CE and their means.  Labels are synsets2idx[synset dir] + label_offset from
    `label_file`; images must decode to image_size x image_size (RGB), fed as uint8 minus CHANNEL_MEANS.

    Decoding runs on a pool of `num_workers` CPU threads (PIL); the device work of a batch (uint8 ->
    fp32, eval forward in the model's dtype, softmax top-1 count) is one CUDA graph replay
    (use_cuda_graph=False: the same launches, eager).  The last batch of a distortion is padded to
    batch_size and its padding rows are masked.  `devices` (default: the model's device) split the
    distortions as the reference's process() does; every device gets a replica with the model's weights.
    With summary_dir, the mCE is written there as a scalar at global_step (0 when it is None), as
    mce/eval_robustness.py:305-315 does; the directory is made (or refused with ValueError) before any work.
    Returns {'<distortion>': {'error', 'ce'}, ..., 'mCE', 'mCE_unnormalized'} (+ 'global_step')."""
    import threading
    from concurrent.futures import ThreadPoolExecutor
    from . import imagenet_c
    from .metrics import DISTORTIONS, CorruptionError
    from .summary import SummaryWriter, check_summary_dir
    if robustness_type == "fr":
        raise ValueError("not yet supported ({}".format(robustness_type))
    if robustness_type != "ce":
        raise ValueError("invalid type ({})".format(robustness_type))
    summary_dir = check_summary_dir(summary_dir)
    if use_resnet_d is None:
        use_resnet_d = getattr(model, "use_resnet_d", False)
    synsets2idx = imagenet_c.get_synsets2idx(label_file)
    # the whole tree is walked first: a missing directory or an unknown synset fails before any GPU work
    work = {d: imagenet_c.distortion_images(data_dir, d, synsets2idx, label_offset) for d in DISTORTIONS}
    empty = [d for d in DISTORTIONS if not work[d][0]]
    if empty:
        raise ValueError("robustness evaluation: no images for distortion(s) %s" % empty)
    devices = [torch.device(d) for d in (devices or [model.device])]
    quota = imagenet_c.distortion_quota(len(devices))
    metric = CorruptionError(device=devices[0])
    replicas = [_replica(model, d, use_resnet_d, batch_size, image_size) for d in devices]
    pool = ThreadPoolExecutor(max_workers=num_workers or min(32, os.cpu_count() or 1))
    results, errors = [None] * len(devices), []

    def run(i):
        try:
            ev = _CorruptionEvalDevice(replicas[i], batch_size, image_size, use_resnet_d, use_cuda_graph)
            batches = [(d, work[d][0][a:a + batch_size], work[d][1][a:a + batch_size])
                       for d in quota[i] for a in range(0, len(work[d][0]), batch_size)]
            counts = {}
            read = read_ahead(pool, [files for _, files, _ in batches], _read_file)
            for j, ((d, files, labels), (_, buffers)) in enumerate(zip(batches, read)):
                ev.run_batch_encoded(buffers, labels, files)
                if j + 1 == len(batches) or batches[j + 1][0] != d:
                    counts[d] = ev.take_count()
            torch.cuda.current_stream(ev.dev).synchronize()
            results[i] = {d: int(c.item()) for d, c in counts.items()}
        except BaseException as e:        # re-raised in the calling thread
            errors.append(e)

    try:
        if len(devices) == 1:
            run(0)
        else:
            threads = [threading.Thread(target=run, args=(i,)) for i in range(len(devices))]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
    finally:
        pool.shutdown(wait=True, cancel_futures=True)
    if errors:
        raise errors[0]
    for counts in results:
        for d, c in counts.items():
            metric.add_counts(d, c, len(work[d][0]))
    out = metric.result()
    if summary_dir is not None:
        w = SummaryWriter(summary_dir)
        try:
            w.add_scalars(global_step or 0, [("mCE", out["mCE"])])
        finally:
            w.close()
    if global_step is not None:
        out["global_step"] = global_step
    return out


def evaluate_classification(model, data_dir, *, val_regex="validation-*", preprocessing_type="imagenet",
                            image_size=224, batch_size=256, label_smoothing=0.0, weight_decay=4e-5,
                            use_resnet_d=None, global_step=None, use_cuda_graph=True, num_workers=None):
    """classifier.evaluate(input_fn_eval) (nets/run_loop_classification.py:397-402,446-448): top-1 and
    top-5 accuracy, ECE and loss of `model` on the TFRecord shards data_dir/val_regex
    (image/encoded, image/class/label), each image given the reference's eval preprocessing for
    `preprocessing_type` (imagenet_eval.eval_geometry: aspect-preserving TF bilinear resize, central
    crop, - CHANNEL_MEANS).

    Every shard is read and checked first: an empty glob, a corrupt record or a label outside
    [0, num_classes) fails before any GPU work.  Decoding runs on a pool of `num_workers` CPU threads
    (PIL); the device work of a batch (resize + crop from uint8, eval forward in the model's dtype,
    acnn_classify_rows) is one CUDA graph replay (use_cuda_graph=False: the same launches, eager).  The
    last batch is padded to batch_size and its padding rows are masked; the per-row results stay on the
    device until the end.  loss = the mean over batches of the batch-mean label-smoothed cross-entropy
    (a short last batch counts as one batch, as tf.metrics.mean of the per-batch loss does) +
    l2_loss(weight_decay).  Returns {'accuracy', 'accuracy_top_5', 'ece', 'loss', 'global_step'}."""
    from . import imagenet_eval
    from .metrics import classification_result
    size, _ = imagenet_eval.eval_size(preprocessing_type, image_size)
    if use_resnet_d is None:
        use_resnet_d = getattr(model, "use_resnet_d", False)
    records = []
    for path in imagenet_eval.validation_files(data_dir, val_regex):
        for label, offset, length in imagenet_eval.read_records(path):
            if not 0 <= label < model.num_classes:
                raise ValueError("classification evaluation: %s: label %d (image at byte offset %d) outside "
                                 "[0, %d)" % (path, label, offset, model.num_classes))
            records.append((path, offset, length, label))
    if not records:
        raise ValueError("classification evaluation: the shards under %s hold no record" % data_dir)
    labels = np.array([r[3] for r in records], dtype=np.int64)
    ev = _ClassifyEvalDevice(model, batch_size, size, use_resnet_d, use_cuda_graph, label_smoothing,
                             len(records))
    sizes = _feed_records(ev, records, batch_size, preprocessing_type, image_size, num_workers)
    pred, conf, hit, ce = (t.cpu().numpy() for t in ev.rows)
    r = classification_result(pred, conf, hit, ce, labels, sizes)
    l2 = float(l2_loss(ev.rt, weight_decay))
    return {"accuracy": r["accuracy"], "accuracy_top_5": r["accuracy_top_5"], "ece": r["ece"],
            "loss": r["cross_entropy"] + l2, "global_step": global_step}


def _check_recall_args(recall_at_k, eval_similarity):
    """The k list and similarity of the retrieval evaluation, checked before any GPU work."""
    from .metrics import KNN_MAX_K, SIMILARITIES
    if eval_similarity not in SIMILARITIES:
        raise NotImplementedError("eval_similarity must be one of %s" % sorted(SIMILARITIES))
    k_list = tuple(int(k) for k in recall_at_k)
    if not k_list or min(k_list) < 1:
        raise ValueError("recall_at_k must be a non-empty list of positive k (got %r)" % (recall_at_k,))
    if max(k_list) + 1 > KNN_MAX_K:
        raise ValueError("recall_at_k: max(recall_at_k) + 1 = %d exceeds %d, the largest k of the fused top-k "
                         "search (acnn_knn_topk)" % (max(k_list) + 1, KNN_MAX_K))
    return k_list


def _feed_records(ev, records, batch_size, preprocessing_type, image_size, num_workers):
    """Runs the records [(path, offset, length, label)] through `ev` (a _ResizedEvalPipeline) in batches of
    batch_size, in order: a pool of `num_workers` CPU threads reads the encoded images four batches ahead of
    the GPU, ev.run_batch_encoded decodes and evaluates them.  Returns the batch sizes once the device is
    done."""
    from concurrent.futures import ThreadPoolExecutor
    from . import imagenet_eval
    batches = [records[a:a + batch_size] for a in range(0, len(records), batch_size)]
    pool = ThreadPoolExecutor(max_workers=num_workers or min(32, os.cpu_count() or 1))
    geometry = lambda h, w: imagenet_eval.eval_geometry(h, w, preprocessing_type, image_size)
    try:
        for recs, buffers in read_ahead(pool, batches, lambda r: imagenet_eval.read_encoded(*r[:3])):
            ev.run_batch_encoded(buffers, [r[3] for r in recs], geometry)
        torch.cuda.current_stream(ev.dev).synchronize()
    finally:
        pool.shutdown(wait=True, cancel_futures=True)
    return [len(b) for b in batches]


def _retrieval_index(model, records, size, batch_size, preprocessing_type, image_size, return_embedding,
                     use_resnet_d, use_cuda_graph, num_workers):
    """The device index of evaluate_retrieval: (fp32 [N, d] outputs, int64 [N] labels) of the records
    [(path, offset, length, label)], in order."""
    ev = _RetrievalEvalDevice(model, batch_size, size, use_resnet_d, use_cuda_graph, return_embedding,
                              len(records))
    _feed_records(ev, records, batch_size, preprocessing_type, image_size, num_workers)
    return ev.index, ev.labels


def evaluate_retrieval(model, data_dir, *, val_regex="validation-*", preprocessing_type="imagenet",
                       image_size=224, batch_size=256, recall_at_k=(1, 5), eval_similarity="cosine",
                       return_embedding=True, use_resnet_d=None, global_step=None, use_cuda_graph=True,
                       num_workers=None):
    """The zero-shot retrieval evaluation of `--zeroshot_eval` (metric/recall_metric.py:13-180 fed by
    input_fn_ir_eval, functions/input_fns.py:148-165): Recall@K of `model` on the TFRecord shards
    data_dir/val_regex, each image given the eval preprocessing of `preprocessing_type` (as
    evaluate_classification).  A record without image/class/label is a distractor (label -1, the
    reference's default_value): it is in the index, never a query; any other int64 label is kept, so the
    test classes of a zero-shot split need not lie in [0, num_classes).

    Every shard is read and checked first, and so are the arguments: an empty glob, a corrupt record, an
    unknown eval_similarity (NotImplementedError), an empty recall_at_k or max(recall_at_k) + 1 above the
    fused search's 128 fail before any GPU work.  Decoding runs as in evaluate_classification; the device
    work of a batch (resize + crop from uint8, eval forward in the model's dtype) is one CUDA graph replay
    (use_cuda_graph=False: the same launches, eager), and its valid rows are copied into a device index
    of every record: the embedding (return_embedding=True; the pooled features without an embedding layer)
    or the logits, as Model.__call__(..., return_embedding) returns them.  Then one acnn_knn_topk in the
    model's dtype, k = max(recall_at_k) + 1, queries = the rows whose label != -1 against every row, and
    get_recall's rules (metrics.recall_of_index).  Returns {'recall_at_<k>': ..., 'global_step': ...}, as
    recall_at_k does."""
    from . import imagenet_eval
    from .metrics import recall_of_index
    k_list = _check_recall_args(recall_at_k, eval_similarity)
    size, _ = imagenet_eval.eval_size(preprocessing_type, image_size)
    if use_resnet_d is None:
        use_resnet_d = getattr(model, "use_resnet_d", False)
    records = [(path, offset, length, label)
               for path in imagenet_eval.validation_files(data_dir, val_regex)
               for label, offset, length in imagenet_eval.read_records(path, missing_label=-1)]
    n_query = sum(r[3] != -1 for r in records)
    if n_query == 0 or len(records) < max(k_list) + 1:
        raise ValueError("retrieval evaluation: the shards under %s hold %d records, %d of them queries; it "
                         "needs a query and at least max(recall_at_k) + 1 = %d records"
                         % (data_dir, len(records), n_query, max(k_list) + 1))
    index, labels = _retrieval_index(model, records, size, batch_size, preprocessing_type, image_size,
                                     return_embedding, use_resnet_d, use_cuda_graph, num_workers)
    out = {"recall_at_%d" % k: v for k, v in recall_of_index(index, labels, k_list, eval_similarity,
                                                             model.dtype).items()}
    out["global_step"] = global_step
    return out


class _TeacherLogitsDevice(_ResizedEvalPipeline):
    """The teacher-logits loop: resize + crop + mean, the eval forward and a copy of the logits into the slot's
    output buffer run as one CUDA graph per (slot, valid rows).  The valid rows of each batch then go to a ring
    of OUT_RING pinned host buffers on the copy stream, one batch late: after the next batch's input has been
    enqueued there, so the copy never holds up that batch's decode.  `sink(rows)` gets each batch's float32
    [n, num_classes] rows in order, only after their copy's event has completed; `finish` delivers the rest."""

    OUT_RING = 3

    def __init__(self, model, batch, size, use_resnet_d, use_cuda_graph, sink):
        super().__init__(model, batch, size, use_resnet_d, use_cuda_graph)
        nc = model.num_classes
        self.out = [torch.zeros(batch, nc, dtype=torch.float32, device=self.dev) for _ in self.slots]
        self.host_out = [torch.zeros(batch, nc, dtype=torch.float32).pin_memory() for _ in range(self.OUT_RING)]
        self.sink = sink
        self.last = None             # (slot, valid rows) of the batch whose copy is not enqueued yet
        self.copies = 0
        self.ready = deque()         # (event, pinned rows) of the enqueued copies not yet delivered

    def _body(self, slot, n_valid):
        _, _, desc = self.slots[slot]
        self.rt.set_images_resized(desc, n_valid, self.mean)
        self.rt.run_forward()
        self.out[slot].copy_(self.logits)

    def _run(self, place, labels):
        super()._run(place, labels)
        if self.last is not None:
            self._copy_out(*self.last)
        self.last = ((self.taken - 1) % len(self.slots), len(labels))

    def _copy_out(self, slot, n):
        # the slot's output is rewritten two batches later, after the copy stream reaches that batch's input
        while len(self.ready) >= self.OUT_RING - 1:
            self._deliver()
        rows = self.host_out[self.copies % self.OUT_RING][:n]
        self.copies += 1
        cs = self.copy_stream
        cs.wait_event(self.slot_free[slot])          # the batch's graph has run
        with torch.cuda.stream(cs):
            rows.copy_(self.out[slot][:n], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(cs)
        self.ready.append((ev, rows))

    def _deliver(self):
        ev, rows = self.ready.popleft()
        ev.synchronize()
        self.sink(rows.numpy())

    def finish(self):
        if self.last is not None:
            self._copy_out(*self.last)
            self.last = None
        while self.ready:
            self._deliver()


def extract_teacher_logits(teacher, data_dir, out_dir, *, train_regex="train-*", val_regex="validation-*",
                           preprocessing_type="imagenet", image_size=224, batch_size=256, shard_index=0,
                           num_shards=1, dataset_name="imagenet", use_resnet_d=None, use_cuda_graph=True,
                           num_workers=None):
    """Knowledge-distillation shards from a trained teacher: the reference's kd/extract_embeddings.py followed
    by datasets/build_imagenet_data.py --logits_file_path.  Every file of data_dir matching train_regex or
    val_regex is copied to out_dir under its own name, its records in order, each record's Example keeping
    its bytes and gaining 'image/logit', a float32 list of the teacher.num_classes fp32 logits that
    teacher(x, training=False) returns for the record's image x after the eval preprocessing of
    `preprocessing_type` / `image_size` (the teacher's, as evaluate_classification).  out_dir is then a data_dir
    for train_and_evaluate(kd_temp > 0): the validation files get logits too, as the reference's evaluation
    input asks for them whenever kd_temp > 0.

    The sorted files are split round-robin over num_shards processes (the reference's --no_shard /
    --total_num_shard, e.g. one process per GPU); this call writes those of shard_index.  Every shard is read
    and checked first: an empty glob (FileNotFoundError), a corrupt record frame, a record that already
    holds image/logit or is not one features message, a teacher whose num_classes is not that of
    DATASETS[dataset_name], out_dir equal to data_dir and an output file that already exists raise
    ValueError before any GPU work and before any output exists.  The device work is the classification
    evaluation's (device JPEG decode with PIL as the fallback, resize + crop + mean, the eval forward in the
    teacher's dtype, one CUDA graph replay per batch; use_cuda_graph=False: the same launches, eager), in
    batches that run across file boundaries, padded only in the last one.  The host writes a record once its
    batch's logits have reached pinned memory, verifying the input record's data CRC
    (imagenet_eval.FloatFeatureWriter); each output appears complete, by rename, or not at all.  Host memory
    holds a few batches and one input file.  Returns the paths written, in order."""
    from . import imagenet_eval as ie
    from .imagenet_train import train_files
    if dataset_name not in DATASETS:
        raise ValueError("extract_teacher_logits: unknown dataset_name %r" % (dataset_name,))
    nc = DATASETS[dataset_name]["num_classes"]
    if teacher.num_classes != nc:
        raise ValueError("extract_teacher_logits: the teacher has %d classes; %s has %d"
                         % (teacher.num_classes, dataset_name, nc))
    if not 0 <= shard_index < num_shards:
        raise ValueError("extract_teacher_logits: shard_index %d outside [0, num_shards = %d)"
                         % (shard_index, num_shards))
    if os.path.realpath(out_dir) == os.path.realpath(data_dir):
        raise ValueError("extract_teacher_logits: out_dir is data_dir (%s); the inputs would be overwritten"
                         % data_dir)
    size, _ = ie.eval_size(preprocessing_type, image_size)
    if use_resnet_d is None:
        use_resnet_d = getattr(teacher, "use_resnet_d", False)
    files = sorted(set(train_files(data_dir, train_regex)) | set(ie.validation_files(data_dir, val_regex)))
    jobs, records = [], []
    for path in files[shard_index::num_shards]:
        dst = os.path.join(out_dir, os.path.basename(path))
        if os.path.exists(dst):
            raise ValueError("extract_teacher_logits: %s already exists" % dst)
        records += [(path, offset, length, 0) for offset, length in ie.appendable_records(path, ie.LOGIT_KEY)]
        jobs.append((path, dst))
    os.makedirs(out_dir, exist_ok=True)
    writer = ie.FloatFeatureWriter(jobs, ie.LOGIT_KEY)
    ev = None
    try:
        if records:
            ev = _TeacherLogitsDevice(teacher, batch_size, size, use_resnet_d, use_cuda_graph, writer.add)
            _feed_records(ev, records, batch_size, preprocessing_type, image_size, num_workers)
            ev.finish()
        writer.close()
    except BaseException:
        if ev is not None:
            torch.cuda.synchronize(ev.dev)      # no copy into the pinned ring outlives the call
        writer.abort()
        raise
    return [dst for _, dst in jobs]


# ------------------------------------------------------------------------------------------------ export
# utils/export_utils.py: the servables export_pb writes under <export_dir>/<data_format>/
SIGNATURES = ("binary_input", "preprocessed_input")
SERVABLE_FORMAT = "assembled_cnn_b200.servable/1"
EXPORT_DECODERS = ("jpeg", "webp")           # --export_decoder_type (hparams_config.py:262-264)
PREDICT_OUTPUTS = ("classes", "probabilities", "probabilities_sigmoid")


class _PredictDevice(_ResizedEvalPipeline):
    """The servable's loop: resize + crop + mean, the eval forward, acnn_predict_rows and (with an embedding
    output) a copy of the embedding run as one CUDA graph per (slot, valid rows), into one set of output
    buffers.  After each batch, its valid rows go to a ring of OUT_RING pinned host sets on the current stream,
    one copy per output, so the next batch's graph runs after them; `sink(arrays)` gets each batch's rows in
    order, once their copy's event has completed.  run_images runs a batch of preprocessed images instead."""

    OUT_RING = 3

    def __init__(self, model, batch, size, use_resnet_d, embedding, fc_split_rows=0):
        super().__init__(model, batch, size, use_resnet_d, True, fc_split_rows=fc_split_rows)
        nc, m = model.num_classes, self.rt.plan.meta
        self.out = [torch.zeros(batch, dtype=torch.int32, device=self.dev),
                    torch.zeros(batch, nc, dtype=torch.float32, device=self.dev),
                    torch.zeros(batch, nc, dtype=torch.float32, device=self.dev)]
        self.feat = None
        if embedding:
            # Model.__call__(return_embedding=True): the embedding, else the pooled features
            self.feat = self.rt.t[m["embedding"] if "embedding" in m else m["pooled"]].reshape(batch, -1)
            self.out.append(torch.zeros(batch, self.feat.shape[1], dtype=torch.float32, device=self.dev))
        self.images = self.rt.t[m["images"]]
        self.host_out = [[torch.zeros(t.shape, dtype=t.dtype).pin_memory() for t in self.out]
                         for _ in range(self.OUT_RING)]
        self.copies = 0
        self.pending = deque()       # (event, pinned set, rows) of the enqueued copies not yet delivered
        self.sink = None
        # gallery search (Servable.search): the index and k of the current call, one set of buffers sized
        # for the largest k seen (work, device outputs, pinned host ring), and the graphs of each k apart
        # (self.graphs is the current k's set) for the SEARCH_KS most recently used k
        self.knn, self.k, self.k_cap = None, 0, 0
        self.search_bufs = None
        self.graph_sets = OrderedDict({0: self.graphs})

    SEARCH_KS = 4

    def use_search(self, knn, k):
        """Run the gallery search of k neighbours (a metrics.KnnIndex; None, 0: none) after each forward.  A
        call without a search leaves the search's buffers and graphs in place for the next one."""
        if knn is not None and knn is not self.knn:      # a new gallery: the old one's buffers and graphs go
            self._drop_search()
            self.knn, self.k_cap = knn, 0
        if k > self.k_cap:                               # larger buffers: the graphs holding the old ones go
            self._drop_search()
            work = torch.empty(knn.work_bytes(self.batch, k), dtype=torch.uint8, device=self.dev)
            dev_out = (torch.zeros(self.batch * k, dtype=torch.int32, device=self.dev),
                       torch.zeros(self.batch * k, dtype=torch.float32, device=self.dev))
            host = [[torch.zeros(t.shape, dtype=t.dtype).pin_memory() for t in dev_out] for _ in range(self.OUT_RING)]
            self.search_bufs, self.k_cap = (work, dev_out, host), k
        self.k = k
        if k not in self.graph_sets:
            if len(self.graph_sets) > self.SEARCH_KS:    # the least recently used k's graphs go
                del self.graph_sets[next(kk for kk in self.graph_sets if kk)]
            self.graph_sets[k] = {}
            self.warm = False            # its first batch runs eagerly, before any capture
        self.graph_sets.move_to_end(k)
        self.graphs = self.graph_sets[k]

    def _drop_search(self):
        self.graph_sets = OrderedDict({0: self.graph_sets[0]})
        self.search_bufs = None

    def _search_out(self):
        """The device outputs (int32, fp32 [batch, k]) and pinned host ring of the current k."""
        _, dev_out, host = self.search_bufs
        n = self.batch * self.k
        return ([t[:n].view(self.batch, self.k) for t in dev_out],
                [[t[:n].view(self.batch, self.k) for t in h] for h in host])

    def _outputs(self, n_valid):
        from .metrics import predict_rows
        predict_rows(self.logits, n_valid, self.out[:3])
        if self.feat is not None:
            self.out[3].copy_(self.feat)
        if self.k:
            self.knn.search(self.out[3][:n_valid], self.k, out=self._search_out()[0], work=self.search_bufs[0])

    def _body(self, slot, n_valid):
        _, _, desc = self.slots[slot]
        self.rt.set_images_resized(desc, n_valid, self.mean)
        self.rt.run_forward()
        self._outputs(n_valid)

    def _run(self, place, labels):
        super()._run(place, labels)
        self._copy_out(len(labels))

    def run_images(self, images):
        """The outputs of the float32 [n <= batch, S, S, 3] preprocessed `images` (eager launches)."""
        n = images.shape[0]
        self.images[:n].copy_(images)
        self.rt.run_forward()
        self._outputs(n)
        self._copy_out(n)

    def _copy_out(self, n):
        while len(self.pending) >= self.OUT_RING:
            self._deliver()
        host, dev = self.host_out[self.copies % self.OUT_RING], self.out
        if self.k:
            dev_out, ring = self._search_out()
            host, dev = host + ring[self.copies % self.OUT_RING], dev + dev_out
        self.copies += 1
        for h, d in zip(host, dev):
            h[:n].copy_(d[:n], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.dev))
        self.pending.append((ev, host, n))

    def _deliver(self):
        ev, host, n = self.pending.popleft()
        ev.synchronize()
        self.sink([h[:n].numpy() for h in host])

    def finish(self):
        while self.pending:
            self._deliver()


def check_batch_sizes(batch_sizes, max_batch):
    """The rungs of a servable's batch ladder: (max_batch,) for None, else batch_sizes as a tuple of
    positive, strictly increasing ints whose largest is max_batch (ValueError otherwise)."""
    if int(max_batch) < 1:
        raise ValueError("max_batch must be >= 1 (got %r)" % (max_batch,))
    max_batch = int(max_batch)
    if batch_sizes is None:
        return (max_batch,)
    sizes = tuple(batch_sizes)
    if not sizes or any(isinstance(b, bool) or not isinstance(b, (int, np.integer)) or b < 1 for b in sizes):
        raise ValueError("batch_sizes must be positive ints (got %r)" % (batch_sizes,))
    if any(a >= b for a, b in zip(sizes, sizes[1:])):
        raise ValueError("batch_sizes must be strictly increasing (got %r)" % (batch_sizes,))
    if sizes[-1] != max_batch:
        raise ValueError("the largest of batch_sizes must be max_batch = %d (got %r)" % (max_batch, batch_sizes))
    return tuple(int(b) for b in sizes)


def ladder_chunks(n, batch_sizes):
    """The (rung, start, stop) chunks of a request of n rows on the rungs batch_sizes (check_batch_sizes):
    chunks of max(batch_sizes) rows, then the rest on the smallest rung that holds it."""
    top = batch_sizes[-1]
    out = [(top, a, a + top) for a in range(0, n - n % top, top)]
    if n % top:
        out.append((next(b for b in batch_sizes if b >= n % top), n - n % top, n))
    return out


class Servable:
    """An exported model (export_model / load_servable) or an in-memory `model` serving the PREDICT dict of
    nets/run_loop_classification.py:126-130 for encoded images (predict, the reference's binary_input
    SavedModel) or for preprocessed ones (predict_images, preprocessed_input).  Both methods return numpy
    {'classes': int64 [n], 'probabilities': float32 [n, num_classes], 'probabilities_sigmoid': float32
    [n, num_classes]} plus 'embedding' float32 [n, d] when the model has an embedding layer or was exported
    with return_embedding (without an embedding layer, the pooled features, as Model.__call__ returns them).

    The device work runs in chunks of max_batch images on the model's device; the first call builds it.
    batch_sizes, e.g. (1, 8, 64, 256), is a ladder of eval runtimes over the model's one copy of the
    weights, each with its own workspace and CUDA graphs, built on its first use: a request's chunks of
    max_batch = max(batch_sizes) rows run on the largest rung and its remainder on the smallest rung that
    holds it (ladder_chunks), so a small request costs a small forward.  Every rung gives each image the
    bits the largest gives it (the SK / SE attention GEMMs of the smaller rungs split K as max_batch rows
    would: acnn_set_fc_split_rows).  None: the one rung max_batch.

    Image search: set_gallery(embedding, labels) gives a servable with an embedding output a gallery, and
    search / search_images return the PREDICT dict plus each image's k nearest gallery rows.  The search
    runs on the device in the same CUDA graph as the forward of each chunk (metrics.KnnIndex, prepared
    once in the model's dtype), and only the valid rows' neighbours are copied back."""

    def __init__(self, model, *, preprocessing_type="imagenet", image_size=224, use_resnet_d=None,
                 return_embedding=False, max_batch=256, signature="binary_input", decoder_type="jpeg",
                 batch_sizes=None):
        from .imagenet_eval import eval_size
        self.size, _ = eval_size(preprocessing_type, image_size)
        self.batch_sizes = check_batch_sizes(batch_sizes, max_batch)
        self.model, self.max_batch = model, int(max_batch)
        self.preprocessing_type, self.image_size = preprocessing_type, int(image_size)
        self.use_resnet_d = bool(getattr(model, "use_resnet_d", False) if use_resnet_d is None else use_resnet_d)
        self.embedding = bool(return_embedding) or model.cfg_kwargs["embedding_size"] > 0
        self.signature, self.decoder_type = signature, decoder_type
        self.outputs = PREDICT_OUTPUTS + (("embedding",) if self.embedding else ())
        self._pipes = {}             # rung -> _PredictDevice
        self._width = None
        self._gallery = None         # (fp32 [nx, d] tensor, similarity) until the first search prepares it
        self._index = None           # metrics.KnnIndex
        self.gallery_labels = None

    @property
    def embedding_width(self):
        """The width of the embedding output, from the host plan (no GPU work)."""
        if self._width is None:
            cfg = ModelConfig(use_resnet_d=self.use_resnet_d, **self.model.cfg_kwargs)
            plan = build_plan(cfg, 1, self.size, self.size, training=False)
            t = plan.tensors[plan.meta["embedding"] if "embedding" in plan.meta else plan.meta["pooled"]]
            self._width = int(np.prod(t.shape[1:]))
        return self._width

    @property
    def gallery_rows(self):
        """The rows of the gallery (0 without one)."""
        return 0 if self._gallery is None and self._index is None else \
            (self._index.nx if self._index is not None else int(self._gallery[0].shape[0]))

    def set_gallery(self, embedding, labels=None, similarity="cosine"):
        """Replaces the gallery that search ranks: `embedding` [nx, d] (numpy or torch; d = the embedding's
        width), optional int `labels` [nx] returned as neighbor_labels, similarity 'cosine' or 'euclidean'
        (metrics.knn_topk).  A servable without an embedding output, a width that is not the embedding's,
        labels of another length and non-finite rows raise here; the gallery is prepared on the device (in
        the model's dtype) by the first search."""
        from .metrics import SIMILARITIES
        if not self.embedding:
            raise ValueError("set_gallery: the servable has no embedding output; export with return_embedding=True")
        if similarity not in SIMILARITIES:
            raise NotImplementedError("similarity must be one of %s" % sorted(SIMILARITIES))
        emb = torch.as_tensor(embedding).detach().to(torch.float32)
        if emb.dim() != 2 or emb.shape[0] < 1 or emb.shape[1] != self.embedding_width:
            raise ValueError("set_gallery: the gallery must be [nx >= 1, %d] like the embedding (got %s)"
                             % (self.embedding_width, tuple(emb.shape)))
        if labels is not None:
            labels = np.asarray(torch.as_tensor(labels).cpu(), np.int64).reshape(-1)
            if len(labels) != emb.shape[0]:
                raise ValueError("set_gallery: %d labels for %d gallery rows" % (len(labels), emb.shape[0]))
        if not bool(torch.isfinite(emb).all()):
            raise ValueError("set_gallery: the gallery contains NaN or infinite values")
        self._gallery, self._index, self.gallery_labels = (emb, similarity), None, labels

    def _check_k(self, k):
        from .metrics import KNN_MAX_K
        if self._gallery is None and self._index is None:
            raise ValueError("search: no gallery; call set_gallery first")
        top = min(KNN_MAX_K, self.gallery_rows)
        if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= top:
            raise ValueError("search: k must be an int in [1, %d] (got %r)" % (top, k))
        return int(k)

    def _knn_index(self):
        from .metrics import KnnIndex
        if self._index is None:
            emb, similarity = self._gallery
            with torch.cuda.device(self.model.device):
                self._index = KnnIndex(emb.to(self.model.device), similarity, self.model.dtype)
            self._gallery = None
        return self._index

    def _neighbors(self, res, k):
        idx = res.pop("neighbors_i32", None)
        res["neighbors"] = np.zeros((0, k), np.int64) if idx is None else idx.astype(np.int64)
        if res["neighbor_similarities"] is None:
            res["neighbor_similarities"] = np.zeros((0, k), np.float32)
        if self.gallery_labels is not None:
            nb = res["neighbors"]
            ok = nb < len(self.gallery_labels)      # the padding of a query with fewer than k finite similarities
            res["neighbor_labels"] = np.where(ok, self.gallery_labels[np.where(ok, nb, 0)], -1)
        return res

    def search(self, images, k):
        """predict(images) plus each image's k nearest gallery rows, nearest first (ties: lower row first):
        'neighbors' int64 [n, k], 'neighbor_similarities' float32 [n, k] and, with gallery labels,
        'neighbor_labels' int64 [n, k] -- equal to metrics.knn_topk(embedding, gallery, k) in the model's
        dtype.  A query with fewer than k finite similarities gets neighbours 2147483647 (label -1) at
        similarity -inf.  k outside [1, min(128, gallery rows)] and a missing gallery raise first."""
        k = self._check_k(k)
        return self._neighbors(self._predict(images, k), k)

    def search_images(self, images, k):
        """search for float32 [n, S, S, 3] images already preprocessed (predict_images)."""
        k = self._check_k(k)
        return self._neighbors(self._predict_images(images, k), k)

    @property
    def _pipe(self):
        """The pipeline of the max_batch rung (None before its first use)."""
        return self._pipes.get(self.max_batch)

    def _rung(self, batch):
        pipe = self._pipes.get(batch)
        if pipe is None:
            pipe = _PredictDevice(self.model, batch, self.size, self.use_resnet_d, self.embedding,
                                  fc_split_rows=self.max_batch)
            self._pipes[batch] = pipe
        return pipe

    def _empty(self, n, names):
        nc = self.model.num_classes
        res = {"classes": np.zeros(n, np.int64), "probabilities": np.zeros((n, nc), np.float32),
               "probabilities_sigmoid": np.zeros((n, nc), np.float32)}
        for name in names[3:]:
            res[name] = None                 # its width is the runtime's: set by the first delivery
        return res

    def _collect(self, n, run, k=0):
        """Runs run(pipeline, start, stop) for every chunk of the n rows on its rung (ladder_chunks) and
        returns the outputs of the n rows, delivered in order; with k, the gallery search's too."""
        names = self.outputs + (("neighbors_i32", "neighbor_similarities") if k else ())
        knn = self._knn_index() if k and n else None
        res, pos = self._empty(n, names), 0
        if n == 0:
            if self.embedding:
                res["embedding"] = np.zeros((0, 0), np.float32)
            return res

        def sink(arrays):
            nonlocal pos
            rows = len(arrays[0])
            for name, a in zip(names, arrays):
                if res[name] is None:
                    res[name] = np.zeros((n,) + a.shape[1:], a.dtype)
                res[name][pos:pos + rows] = a
            pos += rows

        pipe = None
        try:
            for rung, a, b in ladder_chunks(n, self.batch_sizes):
                if pipe is not None and pipe.batch != rung:
                    pipe.finish()            # the rows of the previous rung are delivered first
                pipe = self._rung(rung)
                pipe.sink = sink
                pipe.use_search(knn, k)
                run(pipe, a, b)
            pipe.finish()
        except BaseException:
            # a batch may be staged and not run: the next call starts new pipelines
            if pipe is not None:
                torch.cuda.synchronize(pipe.dev)
            self._pipes.clear()
            raise
        assert pos == n, (pos, n)
        return res

    def predict(self, images):
        """The PREDICT dict of a list of encoded images (bytes; any number).  Each is decoded on the device
        where the device decoder handles it, by PIL otherwise, and given the eval preprocessing of the
        servable's preprocessing_type (imagenet_eval.eval_geometry); a chunk's decode runs on the copy stream
        while the previous chunk computes."""
        return self._predict(images, 0)

    def _predict(self, images, k):
        from .imagenet_eval import eval_geometry
        images = list(images)
        for i, b in enumerate(images):
            if not isinstance(b, (bytes, bytearray, memoryview)):
                raise TypeError("predict: image %d is a %s, not encoded bytes" % (i, type(b).__name__))
        images = [b if isinstance(b, bytes) else bytes(b) for b in images]

        def geometry(h, w):
            return eval_geometry(h, w, self.preprocessing_type, self.image_size)

        def run(pipe, a, b):
            pipe.run_batch_encoded(images[a:b], [0] * (b - a), geometry)
        return self._collect(len(images), run, k)

    def predict_images(self, images):
        """The PREDICT dict of float32 [n, S, S, 3] images already preprocessed (S: the eval size of the
        servable's preprocessing_type), numpy or torch."""
        return self._predict_images(images, 0)

    def _predict_images(self, images, k):
        x = torch.as_tensor(images)
        S = self.size
        if x.dim() != 4 or tuple(x.shape[1:]) != (S, S, 3):
            raise ValueError("predict_images: images must be [n, %d, %d, 3] (got %s)" % (S, S, tuple(x.shape)))
        x = x.to(torch.float32)
        return self._collect(x.shape[0], lambda pipe, a, b: pipe.run_images(x[a:b]), k)


def _variable_names(cfg_kwargs, use_resnet_d, size):
    """The variables (trainables, then BN moving statistics) of a model's plan, from the host plan."""
    plan = build_plan(ModelConfig(use_resnet_d=bool(use_resnet_d), **cfg_kwargs), 1, size, size, training=False)
    return list(plan.params) + list(plan.state)


def _host_weights(model, use_resnet_d, size):
    """float32 numpy arrays of every variable of `model`: its runtime's, or, before any runtime exists, the
    ones given to set_weights (no GPU work); a model with neither gets its seed's initial weights."""
    if bool(use_resnet_d) not in model._primary and model._pending_weights is not None:
        pending = model._pending_weights
        names = _variable_names(model.cfg_kwargs, use_resnet_d, size)
        missing = [n for n in names if n not in pending]
        if missing:
            raise KeyError("export: the weights lack %d variable(s), e.g. %s" % (len(missing), missing[:3]))
        return {n: torch.as_tensor(pending[n]).detach().float().cpu().numpy() for n in names}
    if bool(use_resnet_d) not in model._primary:
        model.runtime(1, size, size, training=False, use_resnet_d=use_resnet_d)
    return {n: v.numpy() for n, v in model.get_weights(use_resnet_d).items()}


def _partial(path):
    return os.path.join(os.path.dirname(path), ".%s.partial" % os.path.basename(path))


def export_model(model, export_dir, *, preprocessing_type, image_size, use_resnet_d=None, return_embedding=False,
                 decoder_type="jpeg"):
    """utils/export_utils.export_pb: writes the two servables of `model` as Estimator.export_savedmodel
    lays them out, <export_dir>/channels_last/binary_input/<timestamp>/ (encoded images in, the eval
    preprocessing of preprocessing_type / image_size) and <export_dir>/channels_last/preprocessed_input/
    <timestamp>/ (float images in), and returns the two paths.  Each holds config.json (the model's
    constructor flags, use_resnet_d, dtype, preprocessing_type, image_size, decoder_type, the signature's
    input and outputs) and variables.npz (every variable in the checkpoint module's TF naming, without the
    momentum slots or global_step).  load_servable reads them; TF SavedModels are not written (they cannot
    be without TensorFlow).

    An unknown preprocessing_type (NotImplementedError), an image_size that is not a positive int or gives
    an eval size that is not a multiple of 32, an unknown decoder_type and an existing target (FileExistsError)
    raise before anything is written and before any GPU work.  The weights are read from the model's runtime
    (those given to set_weights when it has none yet: then no GPU work at all).  Each directory is written
    under a hidden name beside its target and renamed when complete."""
    import json
    import time
    from .imagenet_eval import eval_size
    if isinstance(image_size, bool) or not isinstance(image_size, (int, np.integer)) or image_size < 1:
        raise ValueError("export: image_size must be a positive int (got %r)" % (image_size,))
    size, _ = eval_size(preprocessing_type, int(image_size))
    if decoder_type not in EXPORT_DECODERS:
        raise ValueError("export: decoder_type must be one of %s (got %r)" % (EXPORT_DECODERS, decoder_type))
    if use_resnet_d is None:
        use_resnet_d = getattr(model, "use_resnet_d", False)
    stamp = str(int(time.time()))
    targets = [os.path.join(export_dir, model.data_format, sig, stamp) for sig in SIGNATURES]
    for t in targets:
        if os.path.lexists(t) or os.path.lexists(_partial(t)):
            raise FileExistsError("export: %s already exists" % t)
    weights = _host_weights(model, use_resnet_d, size)
    nc = model.num_classes
    outputs = {"classes": "int64 [n]", "probabilities": "float32 [n, %d]" % nc,
               "probabilities_sigmoid": "float32 [n, %d]" % nc}
    if return_embedding or model.cfg_kwargs["embedding_size"] > 0:
        outputs["embedding"] = "float32 [n, d]"
    inputs = {"binary_input": "encoded images: bytes [n]",
              "preprocessed_input": "float32 [n, %d, %d, 3], eval-preprocessed" % (size, size)}
    written = []
    try:
        for sig, t in zip(SIGNATURES, targets):
            tmp = _partial(t)
            os.makedirs(tmp)
            written.append(tmp)
            config = {"format": SERVABLE_FORMAT, "signature": sig, "inputs": inputs[sig], "outputs": outputs,
                      "model": dict(model.cfg_kwargs), "dtype": model.dtype, "use_resnet_d": bool(use_resnet_d),
                      "data_format": model.data_format, "preprocessing_type": preprocessing_type,
                      "image_size": int(image_size), "eval_size": size, "decoder_type": decoder_type,
                      "return_embedding": bool(return_embedding), "variables": "variables.npz"}
            with open(os.path.join(tmp, "variables.npz"), "wb") as f:
                np.savez(f, **weights)
                f.flush()
                os.fsync(f.fileno())
            with open(os.path.join(tmp, "config.json"), "w") as f:
                json.dump(config, f, indent=1, sort_keys=True)
        for tmp, t in zip(list(written), targets):
            os.rename(tmp, t)
            written.remove(tmp)
    except BaseException:
        import shutil
        for tmp in written:
            shutil.rmtree(tmp, ignore_errors=True)
        raise
    return targets[0], targets[1]


def read_servable_config(path):
    """The config.json of an exported servable directory, checked (ValueError) before anything is built."""
    import json
    fname = os.path.join(path, "config.json")
    if not os.path.isfile(fname) or not os.path.isfile(os.path.join(path, "variables.npz")):
        raise ValueError("%s is not an exported servable (config.json and variables.npz expected)" % path)
    with open(fname) as f:
        cfg = json.load(f)
    keys = {"format", "signature", "model", "dtype", "use_resnet_d", "preprocessing_type", "image_size",
            "decoder_type", "return_embedding"}
    if not isinstance(cfg, dict) or cfg.get("format") != SERVABLE_FORMAT or not keys <= set(cfg) \
            or cfg["signature"] not in SIGNATURES:
        raise ValueError("%s: not a config.json of format %s" % (fname, SERVABLE_FORMAT))
    return cfg


def load_servable(path, *, device=None, max_batch=256, batch_sizes=None):
    """The Servable of a directory export_model wrote: a new Model of the directory's flags and dtype with
    its variables (on `device`, default the current CUDA device), on the rungs batch_sizes (Servable).
    Host work only: the device work starts with the first predict.  The directory's gallery.npz
    (export_gallery), when present, becomes the servable's cosine gallery (Servable.set_gallery)."""
    from .checkpoint import load_checkpoint
    from .imagenet_eval import eval_size
    check_batch_sizes(batch_sizes, max_batch)
    cfg = read_servable_config(path)
    size, _ = eval_size(cfg["preprocessing_type"], cfg["image_size"])
    model = Model(dtype=cfg["dtype"], device=device or "cuda:%d" % torch.cuda.current_device(), **cfg["model"])
    model.use_resnet_d = bool(cfg["use_resnet_d"])
    weights = load_checkpoint(os.path.join(path, "variables.npz"))
    names = _variable_names(model.cfg_kwargs, model.use_resnet_d, size)
    missing = [n for n in names if n not in weights]
    if missing:
        raise ValueError("%s: variables.npz lacks %d variable(s), e.g. %s" % (path, len(missing), missing[:3]))
    model.set_weights({n: torch.as_tensor(weights[n]) for n in names})
    sv = Servable(model, preprocessing_type=cfg["preprocessing_type"], image_size=cfg["image_size"],
                  use_resnet_d=model.use_resnet_d, return_embedding=cfg["return_embedding"], max_batch=max_batch,
                  signature=cfg["signature"], decoder_type=cfg["decoder_type"], batch_sizes=batch_sizes)
    gallery = os.path.join(path, GALLERY_FILE)
    if os.path.isfile(gallery):
        with np.load(gallery) as g:
            sv.set_gallery(g["embedding"], g["label"])
    return sv


GALLERY_FILE = "gallery.npz"


def export_gallery(binary_dir, data_dir, *, val_regex="validation-*", batch_size=256, num_workers=None):
    """The image-search gallery of the exported binary_input servable at binary_dir: every record of the
    validation shards data_dir/val_regex (read as export_test reads them) embedded by the servable's own
    model, preprocessing and image size (the retrieval evaluation's loop, in batches of batch_size).  Writes
    binary_dir/gallery.npz, which load_servable loads, and returns its path: 'embedding' float32 [N, d],
    'label' int64 [N] (-1 for a record without one), 'shard' int32 [N] (the record's shard, an index into
    'shard_names', the sorted shard file names) and 'record' int64 [N] (its position in that shard), so that
    a neighbour maps back to its record.  A servable without an embedding output, an existing gallery.npz,
    an empty glob and a corrupt record raise before any GPU work.  The file is written under a hidden name
    and renamed when complete."""
    from . import imagenet_eval as ie
    target = os.path.join(binary_dir, GALLERY_FILE)
    if os.path.lexists(target) or os.path.lexists(_partial(target)):
        raise FileExistsError("export_gallery: %s already exists" % target)
    sv = load_servable(binary_dir, max_batch=batch_size)
    if not sv.embedding:
        raise ValueError("export_gallery: the servable has no embedding output; export with return_embedding=True")
    files = ie.validation_files(data_dir, val_regex)
    records, shard, record = [], [], []
    for i, path in enumerate(files):
        for j, (label, offset, length) in enumerate(ie.read_records(path, missing_label=-1)):
            records.append((path, offset, length, label))
            shard.append(i)
            record.append(j)
    if not records:
        raise ValueError("export_gallery: the shards under %s hold no record" % data_dir)
    index, labels = _retrieval_index(sv.model, records, sv.size, sv.max_batch, sv.preprocessing_type,
                                     sv.image_size, True, sv.use_resnet_d, True, num_workers)
    tmp = _partial(target)
    try:
        with open(tmp, "wb") as f:
            np.savez(f, embedding=index.cpu().numpy(), label=labels.cpu().numpy(),
                     shard=np.asarray(shard, np.int32), record=np.asarray(record, np.int64),
                     shard_names=np.asarray([os.path.basename(p) for p in files]))
            f.flush()
            os.fsync(f.fileno())
        os.rename(tmp, target)
    except BaseException:
        if os.path.lexists(tmp):
            os.remove(tmp)
        raise
    return target


def export_recall_at_1(embedding, labels, device=None):
    """Recall@1 of export_test's zero-shot branch (utils/export_utils.py:75-86): every row is a query
    (distractors, label -1, included, and two distractors match), the index is every row but the query
    itself (fill_diagonal(-10)), similarity the cosine of l2-normalised rows, and the nearest row is the
    lowest index among equal similarities (np.argmax).  The search is one acnn_knn_topk with k = 2 in fp32
    (three bf16 planes per operand); the query's own index is skipped."""
    from .metrics import knn_topk
    x = torch.as_tensor(np.asarray(embedding, np.float32)).to(device or "cuda")
    labels = np.asarray(labels, np.int64)
    n = x.shape[0]
    if n < 2 or len(labels) != n:
        raise ValueError("export_test: Recall@1 needs at least two rows with one label each (got %d rows, %d labels)"
                         % (n, len(labels)))
    if not bool(torch.isfinite(x).all()):
        raise ValueError("export_test: the embeddings contain NaN or infinite values")
    idx, _ = knn_topk(x, x, 2, "cosine", "fp32")
    idx = idx.long().cpu().numpy()
    if (idx >= n).any():
        raise ValueError("export_test: similarities are not finite; cannot rank the index")
    nearest = np.where(idx[:, 0] == np.arange(n), idx[:, 1], idx[:, 0])
    return int((labels[nearest] == labels).sum()) / n


def export_test(binary_dir, data_dir, *, val_regex="validation-*", batch_size=256, zeroshot=False):
    """utils/export_utils.export_test: the exported binary_input servable at binary_dir re-reads the
    validation shards data_dir/val_regex (a record without image/class/label has label -1) and scores
    itself: the accuracy of `classes` against the labels, or with zeroshot Recall@1 of its `embedding`
    (export_recall_at_1).  Writes binary_dir/model_performance.txt with the reference's message and returns
    the metric.  A bad directory, an empty glob, a corrupt record and zeroshot on a servable without an
    embedding output raise before any GPU work."""
    from . import imagenet_eval as ie
    sv = load_servable(binary_dir, max_batch=batch_size)
    if zeroshot and not sv.embedding:
        raise ValueError("export_test: zeroshot needs an embedding output; export with return_embedding=True")
    per_file = [(path, ie.read_records(path, missing_label=-1)) for path in ie.validation_files(data_dir, val_regex)]
    labels = np.array([r[0] for _, recs in per_file for r in recs], np.int64)
    if len(labels) == 0:
        raise ValueError("export_test: the shards under %s hold no record" % data_dir)
    group = 8 * sv.max_batch
    classes, emb = [], []
    for path, recs in per_file:
        data = ie._read_file(path)
        for a in range(0, len(recs), group):
            out = sv.predict([data[off:off + n] for _, off, n in recs[a:a + group]])
            classes.append(out["classes"])
            if zeroshot:
                emb.append(out["embedding"])
    if zeroshot:
        metric = export_recall_at_1(np.concatenate(emb), labels, sv.model.device)
    else:
        metric = int((np.concatenate(classes) == labels).sum()) / len(labels)
    msg = "IMPOTANT! Evaluation metric of exported saved_model.pb is {}".format(metric)
    with open(os.path.join(binary_dir, "model_performance.txt"), "w") as fp:
        fp.write(msg)
    return metric


class _TrainFeed(StagingRing):
    """The training input's staging ring: per step, the crop windows packed into a growable pinned uint8
    buffer with one acnn_crop_desc each, the labels and (KD) the teacher logits, copied to one of two
    device slots on the copy stream while the previous step computes; `step` makes the images on the device
    (Trainer.train_step_cropped) and runs the training step.  With several replicas per device a staged batch
    holds the replicas' micro-batches one after another (replicas_per_device x input_batch examples)."""

    def __init__(self, trainer, kd):
        self.tr, dev = trainer, trainer.rt.dev
        n, nc = trainer.replicas * trainer.input_batch, trainer.model.num_classes
        i32, f32 = dict(dtype=torch.int32), dict(dtype=torch.float32)
        host = [[None, torch.zeros(n, **i32).pin_memory(), torch.zeros(32 * n, dtype=torch.uint8).pin_memory(),
                 torch.zeros(n, nc, **f32).pin_memory() if kd else None] for _ in range(self.RING)]
        # a step's graph holds no address of these: the image bytes may move when the buffer grows
        slots = [[None, torch.zeros(n, **i32, device=dev), torch.zeros(32 * n, dtype=torch.uint8, device=dev),
                  torch.zeros(n, nc, **f32, device=dev) if kd else None] for _ in range(2)]
        super().__init__(dev, host, slots)

    def stage(self, windows, labels, teacher_logits=None):
        """`windows` replicas x input_batch (uint8 [h, w, 3] array, flip) pairs, `labels` ints, `teacher_logits`
        float32 [replicas x input_batch, num_classes] with KD."""
        def place(h, slot):
            self.host[h][0], self.slots[slot][0], addrs = pack_u8(self.host[h][0], self.slots[slot][0],
                                                                 [a for a, _ in windows], self.dev)
            return [(ad, a.shape[0], a.shape[1], flip) for ad, (a, flip) in zip(addrs, windows)]
        self._stage(place, labels, teacher_logits)

    def stage_encoded(self, items, labels, teacher_logits=None):
        """As stage, from replicas x input_batch (encoded JPEG bytes, (y, x, h, w) window, flip) triples: the windows are
        decoded on the copy stream (jpeg.JpegDecoder, one per slot; PIL's decode_rgb for the images the
        device does not decode)."""
        def place(h, slot):
            got = self.decoder(slot).stage([b for b, _, _ in items], np.array([w for _, w, _ in items], np.int32),
                                           self.copy_stream)
            return [(ad, hh, ww, flip) for (ad, hh, ww), (_, _, flip) in zip(got, items)]
        self._stage(place, labels, teacher_logits)

    def _stage(self, place, labels, teacher_logits):
        from .imagenet_train import CROP_DESC_DTYPE, check_crop_descriptors

        def fill(h, slot):
            placed = place(h, slot)
            _, hlab, hdesc, hteach = self.host[h]
            desc = hdesc.numpy().view(CROP_DESC_DTYPE)
            for i, (addr, wh, ww, flip) in enumerate(placed):
                desc[i] = (addr, wh, ww, int(flip), (0, 0, 0))
            check_crop_descriptors(desc)
            hlab.copy_(torch.as_tensor(labels, dtype=torch.int32))
            _, dlab, ddesc, dteach = self.slots[slot]
            ddesc.copy_(hdesc, non_blocking=True)
            dlab.copy_(hlab, non_blocking=True)
            if dteach is not None:
                hteach.copy_(torch.as_tensor(teacher_logits, dtype=torch.float32))
                dteach.copy_(hteach, non_blocking=True)
        self.push(fill)

    def step(self, lam1=None, lam2=None):
        """The training step of the oldest staged batch; returns Trainer.train_step's loss tensor."""
        slot = self.take()
        _, dlab, ddesc, dteach = self.slots[slot]
        loss = self.tr.train_step_cropped(ddesc, dlab, self.mean, lam1=lam1, lam2=lam2, teacher_logits=dteach)
        self.release(slot)
        return loss


def _prune_checkpoints(model_dir, keep):
    """RunConfig(keep_checkpoint_max): only the `keep` newest model.ckpt-<step>.npz stay in model_dir."""
    import glob
    found = []
    for f in glob.glob(os.path.join(model_dir, "model.ckpt-*.npz")):
        try:
            found.append((int(os.path.basename(f)[len("model.ckpt-"):-4]), f))
        except ValueError:
            continue
    for _, f in sorted(found)[:max(len(found) - keep, 0)]:
        os.remove(f)


def cycle_schedule(p, epochs_between_evals, cur_epoch):
    """(the training epochs of each train-and-evaluate cycle, the index of the first one) of resnet_main
    (nets/run_loop_classification.py:457-468) for the params p, resumed at epoch cur_epoch: one evaluation with
    eval_only or train_epochs = 0, no cycle with export_only, else imagenet_train.epoch_schedule from
    cur_epoch.  The cycle index keys the cycle's randomness."""
    from . import imagenet_train as it
    if p["eval_only"] or not p["train_epochs"]:
        return [0], 0
    if p["export_only"]:
        return [], 0
    args = (p["train_epochs"], epochs_between_evals, p["ratio_fine_eval"])
    full = it.epoch_schedule(*args)
    schedule = it.epoch_schedule(*args, cur_epoch=cur_epoch)
    return schedule, len(full) - len(schedule)


def train_and_evaluate(data_dir, model_dir, *, epochs_between_evals=1, stop_threshold=None, max_train_steps=None,
                       image_size=224, seed=0, use_cuda_graph=True, num_workers=None, export_dir=None,
                       replicas_per_device=1, save_summary_steps=None, **flags):
    """resnet_main's train-and-evaluate loop (nets/run_loop_classification.py:389-489) over the TFRecord
    shards data_dir/train_regex (training) and data_dir/val_regex (evaluation).  `flags` are hparams
    names (params_from_flags); epochs_between_evals, stop_threshold and max_train_steps are the run loop's
    flags of official/utils/flags (_base.py:51-63, _performance.py:96-97) with their defaults; image_size is
    the `imagenet` preprocessing type's size.

    Every training record is read and checked first (imagenet_train.read_train_records).  The latest
    model.ckpt-<step> in model_dir is restored (weights, momentum slots, global_step), else
    pretrained_model_checkpoint_path warm-starts the run (checkpoint.warm_start).  Cycles follow
    imagenet_train.epoch_schedule from the restored step (one evaluation with eval_only or train_epochs = 0).
    A cycle trains on imagenet_train.CycleStream (at most max_train_steps steps): PIL decoding of the crop
    windows on a pool of `num_workers` CPU threads, _TrainFeed staging, acnn_set_images_cropped and the
    Trainer's step (use_cuda_graph: one graph replay).  It saves model.ckpt-<global step> every
    save_checkpoints_epochs epochs and at its end, keeping keep_checkpoint_max of them, then runs
    evaluate_classification, CheckpointKeeper.save(accuracy) and stops at stop_threshold or once the global
    step reaches train_epochs * int(num_images / batch_size).  With zeroshot_eval the evaluation is
    evaluate_retrieval instead (batch val_batch_size, the recall_at_k, eval_similarity, preprocessing_type
    and val_regex flags, return_embedding=True as the reference's loop passes it), and accuracy is replaced
    by recall_at_1 for the keeper and stop_threshold (nets/run_loop_classification.py:439-448,476-480);
    recall_at_k and eval_similarity are checked before any GPU work.  The seed gives the initial weights, the
    record order, the crop windows, the flips and the mixup lambdas (imagenet_train's counter-based
    generators).  num_images is the number of records in the shards (the reference's data_config count).
    Under torch.distributed every rank trains its slice of each global batch; rank 0 writes the
    checkpoints and evaluates.

    With export_dir (official/utils/flags/_base.py's --export_dir), rank 0 exports the model after the last
    cycle (export_model with the preprocessing_type, image_size and use_resnet_d flags; return_embedding with
    return_embedding or zeroshot_eval) and, when export_decoder_type is 'jpeg', runs export_test on the binary
    servable (batch val_batch_size, val_regex, zeroshot_eval), as nets/run_loop_classification.py:494-495.
    export_only runs no cycle (unless eval_only or train_epochs = 0 ask for an evaluation, as the reference's
    order has it) and exports the latest checkpoint of model_dir; it needs export_dir and a checkpoint, both
    checked before any GPU work.

    replicas_per_device = R runs R data-parallel replicas on each device (Trainer's micro-steps): the reference's
    --num_gpus=N is world * R = N.  Replica q = rank * R + r reads what rank q of a world * R run reads
    (imagenet_train.replica_streams, replica_mixup_lambdas); each global step stages the R micro-batches together.
    R >= 1 and batch_size divisible by world * R are checked before any GPU work.  The evaluation runs at the
    per-replica batch.

    save_summary_steps = N (RunConfig's save_summary_steps; None, the default, writes nothing) makes rank 0
    write the training summaries to model_dir/events.out.tfevents.* on the first step of each cycle and every
    N-th step after it, at the global step the step ran with, log one line per summary to the
    "assembled_cnn_b200" logger at INFO, and write every numeric entry of each evaluation result to
    model_dir/eval/ (summary.TrainSummaries: the metrics are accumulated on the device and read back without a
    per-step host synchronisation).  Anything but None or an integer >= 1 raises before any GPU work.

    Returns the list of the cycles' evaluation results (the recall dicts with zeroshot_eval)."""
    from concurrent.futures import ThreadPoolExecutor
    from . import imagenet_train as it
    from .checkpoint import CheckpointKeeper, latest_checkpoint, restore, save_checkpoint, warm_start
    from .imagenet_eval import eval_size
    from .summary import SummaryWriter, TrainSummaries, check_save_summary_steps, is_summary_step, numeric_scalars
    summary_every = check_save_summary_steps(save_summary_steps)
    p = params_from_flags(**flags)
    if p["autoaugment_type"] is not None:
        raise NotImplementedError("autoaugment_type=%r: AutoAugment is not implemented; train with "
                                  "autoaugment_type=None" % (p["autoaugment_type"],))
    ds_name = p["dataset_name"] or "imagenet"
    ds = DATASETS[ds_name]
    size = it.train_size(p["preprocessing_type"], image_size)
    eval_size(p["preprocessing_type"], image_size)
    zeroshot = bool(p["zeroshot_eval"])
    if zeroshot and 1 not in _check_recall_args(p["recall_at_k"], p["eval_similarity"]):
        raise ValueError("zeroshot_eval ranks the checkpoints by recall_at_1: recall_at_k must hold 1 (got %r)"
                         % (p["recall_at_k"],))
    key = "recall_at_1" if zeroshot else "accuracy"
    if export_dir is not None and p["export_decoder_type"] not in EXPORT_DECODERS:
        raise ValueError("export_decoder_type must be one of %s (got %r)" % (EXPORT_DECODERS, p["export_decoder_type"]))
    if p["export_only"]:
        if export_dir is None:
            raise ValueError("export_only exports the latest checkpoint: give export_dir")
        if not os.path.isdir(model_dir) or latest_checkpoint(model_dir) is None:
            raise ValueError("export_only: no checkpoint in %s" % model_dir)
    dist = torch.distributed.is_initialized()
    world = torch.distributed.get_world_size() if dist else 1
    rank = torch.distributed.get_rank() if dist else 0
    R = check_replicas_per_device(replicas_per_device)
    per_device_batch_size(p["batch_size"], world * R)
    kd = float(p["kd_temp"] or 0) > 0
    records, counts = it.read_train_records(it.train_files(data_dir, p["train_regex"]), ds["num_classes"], kd)
    num_images = len(records)
    steps_per_epoch = int(num_images / p["batch_size"])
    if steps_per_epoch < 1:
        raise ValueError("training: %d records hold no batch of %d" % (num_images, p["batch_size"]))
    dev = torch.device("cuda", torch.cuda.current_device())
    model = Model(p["resnet_size"], p["data_format"], num_classes=ds["num_classes"],
                  resnet_version=p["resnet_version"], zero_gamma=p["zero_gamma"],
                  use_se_block=p["use_se_block"], use_sk_block=p["use_sk_block"],
                  no_downsample=p["no_downsample"], anti_alias_filter_size=p["anti_alias_filter_size"],
                  anti_alias_type=p["anti_alias_type"], bn_momentum=p["bn_momentum"],
                  embedding_size=p["embedding_size"], pool_type=p["pool_type"], bl_alpha=p["bl_alpha"],
                  bl_beta=p["bl_beta"], dtype=p["dtype"], loss_type=p["cls_loss_type"], seed=seed,
                  device=str(dev))
    model.use_resnet_d = bool(p["use_resnet_d"])
    summarize = summary_every is not None and rank == 0
    trainer = Trainer(model, p, size, size, use_cuda_graph=use_cuda_graph, num_images=num_images,
                      replicas_per_device=R, train_metrics=summarize)
    ckpt = latest_checkpoint(model_dir) if os.path.isdir(model_dir) else None
    if ckpt:
        restore(model, ckpt, trainer)
    elif p["pretrained_model_checkpoint_path"]:
        warm_start(model, p["pretrained_model_checkpoint_path"], trainer.global_step)
    schedule, first = cycle_schedule(p, epochs_between_evals, trainer.global_step // steps_per_epoch)
    total_train_steps = p["train_epochs"] * steps_per_epoch
    save_steps = int(p["save_checkpoints_epochs"] * steps_per_epoch)
    shuffle_buffer = it.SHUFFLE_BUFFER.get(ds_name, it.DEFAULT_SHUFFLE_BUFFER)
    keeper = CheckpointKeeper(model_dir, p["num_best_ckpt_to_keep"], p["keep_ckpt_every_eval"], maximize=True) \
        if rank == 0 else None

    summaries = TrainSummaries(model_dir, trainer) if summarize else None
    eval_writer = None

    def save():
        if rank == 0:
            save_checkpoint(os.path.join(model_dir, "model.ckpt-%d" % trainer.global_step), model, trainer)
            _prune_checkpoints(model_dir, p["keep_checkpoint_max"])
            if summaries is not None:       # the checkpoint has read the weights: the ring has completed
                summaries.drain()

    feed = _TrainFeed(trainer, kd)
    n_lam = trainer.input_batch // 2
    pool = ThreadPoolExecutor(max_workers=num_workers or min(32, os.cpu_count() or 1))
    results = []
    try:
        for ci, epochs in enumerate(schedule):
            c = first + ci
            if epochs:
                streams = it.replica_streams(counts, seed, c, epochs * (2 if trainer.mixup_type == 1 else 1),
                                             shuffle_buffer, trainer.input_batch, world, rank, R)
                n_steps = streams[0].steps
                steps = n_steps if max_train_steps is None else min(n_steps, max_train_steps)

                def window(pos_r, c=c):
                    pos, r = pos_r
                    return it.encoded_window(*records[r][:3], seed, c, pos, p["training_random_crop"])

                def step_records(t):
                    return [pr for s in streams for pr in s.records(t)]
                read = read_ahead(pool, map(step_records, range(steps)), window)

                def stage():
                    recs, items = next(read)
                    teacher = np.stack([records[r][4] for _, r in recs]) if kd else None
                    feed.stage_encoded(items, [records[r][3] for _, r in recs], teacher)

                if steps:
                    stage()
                if summaries is not None:
                    summaries.begin_cycle()
                cycle_first = trainer.global_step
                for t in range(steps):
                    lam1 = lam2 = None
                    if trainer.mixup_type:
                        lam = it.replica_mixup_lambdas(seed, trainer.global_step, rank, R, 2 * n_lam).reshape(R, 2, n_lam)
                        lam1, lam2 = lam[:, 0], (lam[:, 1] if trainer.mixup_type == 2 else None)
                    step = trainer.global_step
                    loss = feed.step(lam1, lam2)
                    if summaries is not None:
                        if is_summary_step(step, cycle_first, summary_every):
                            summaries.record(loss, step, trainer.last_lr, trainer.last_keep_prob)
                        summaries.poll()
                    if t + 1 < steps:
                        stage()
                        if save_steps > 0 and trainer.global_step % save_steps == 0:
                            save()
                save()
            if rank == 0:
                if latest_checkpoint(model_dir) is None:
                    raise ValueError("evaluation: no checkpoint in %s" % model_dir)
                if zeroshot:
                    # the reference's loop embeds with return_embedding=True whatever the flag says
                    res = evaluate_retrieval(
                        model, data_dir, val_regex=p["val_regex"], preprocessing_type=p["preprocessing_type"],
                        image_size=image_size, batch_size=p["val_batch_size"], recall_at_k=p["recall_at_k"],
                        eval_similarity=p["eval_similarity"], return_embedding=True,
                        global_step=trainer.global_step, use_cuda_graph=use_cuda_graph, num_workers=num_workers)
                else:
                    res = evaluate_classification(
                        model, data_dir, val_regex=p["val_regex"], preprocessing_type=p["preprocessing_type"],
                        image_size=image_size, batch_size=trainer.local_batch, label_smoothing=p["label_smoothing"],
                        weight_decay=p["weight_decay"], global_step=trainer.global_step,
                        use_cuda_graph=use_cuda_graph, num_workers=num_workers)
                keeper.save(res[key], model_dir)
                if summarize:
                    if eval_writer is None:
                        eval_writer = SummaryWriter(os.path.join(model_dir, "eval"))
                    eval_writer.add_scalars(res["global_step"], numeric_scalars(res))
            else:
                res = None
            if dist:
                box = [res]
                torch.distributed.broadcast_object_list(box, src=0)
                res = box[0]
            results.append(res)
            if stop_threshold is not None and res[key] >= stop_threshold:
                break
            if res["global_step"] >= total_train_steps:
                break
    finally:
        pool.shutdown(wait=True, cancel_futures=True)
    torch.cuda.current_stream(dev).synchronize()
    if summaries is not None:
        summaries.close()
    if eval_writer is not None:
        eval_writer.close()
    if export_dir is not None and rank == 0:
        binary_dir, _ = export_model(model, export_dir, preprocessing_type=p["preprocessing_type"],
                                     image_size=image_size, use_resnet_d=p["use_resnet_d"],
                                     return_embedding=bool(p["return_embedding"] or zeroshot),
                                     decoder_type=p["export_decoder_type"])
        if p["export_decoder_type"] == "jpeg":
            export_test(binary_dir, data_dir, val_regex=p["val_regex"], batch_size=p["val_batch_size"],
                        zeroshot=zeroshot)
    return results
