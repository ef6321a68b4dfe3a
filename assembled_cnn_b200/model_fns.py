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
plus `build_model(**flags)` (the name BASELINE.json uses; the reference has no such function).

The reference builds a TF graph and lets the Estimator run it; here a call executes on the GPU:
`Model.__call__` runs one forward, `Trainer.train_step` one full step (mixup -> forward -> loss ->
backward -> all-reduce -> SGD).  torch tensors are the device-memory container only.
"""
from __future__ import annotations

import os
import math
from collections import namedtuple

import numpy as np
import torch

from . import _lib, dp
from .hparams import DATASETS, DEFAULTS, params_from_flags
from .plan import BLOCK_SIZES, ModelConfig, build_plan
from .metrics import EvalMetrics, RecallAtK
from .runtime import Runtime
from .native import NativeModel, NativeRuntime

DEFAULT_VERSION = 1
# dtype: 'bf16' = production path (bf16 storage, fp32 accumulation -- the analogue of the reference's
# fp16 mode); 'fp32' = the reference's default (nets/resnet_model.py:30-33,
# official/utils/flags/_performance.py:29-32): fp32 storage, 3-way bf16-split wgmma GEMMs,
# bit-reproducible reductions -- the mode the 1e-3 parity tests run in.  'fp16' has no H100
# counterpart here (bf16 replaces it) and is rejected.
ALLOWED_TYPES = ("bf16", "fp32")

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
                 deterministic=None, native=None):
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
        # True (default): the layer plan is built and executed inside libacnn.so through the model-level
        # C ABI (include/acnn_model.h, native.NativeRuntime); False (ACNN_NATIVE_PLAN=0): the Python plan
        # + per-op ctypes executor the lockstep parity tests drive (same plan, text-for-text)
        self.native = (os.environ.get("ACNN_NATIVE_PLAN", "1") != "0") if native is None else bool(native)
        self._runtimes = {}          # (B, H, W, training, use_resnet_d, mixup, ls) -> Runtime
        self._primary = {}           # use_resnet_d -> Runtime owning the parameters
        self._pending_weights = None

    # ---------------------------------------------------------------- runtimes / parameters
    def runtime(self, batch, height, width, *, training, use_resnet_d=False, mixup_type=0,
                label_smoothing=0.0, with_loss=False, use_dropblock=False, kd_temp=0.0) -> Runtime:
        key = (batch, height, width, bool(training), bool(use_resnet_d), mixup_type,
               float(label_smoothing), bool(with_loss or training), bool(use_dropblock and training),
               float(kd_temp) if training else 0.0)
        rt = self._runtimes.get(key)
        if rt is None:
            cfg = ModelConfig(use_resnet_d=bool(use_resnet_d), **self.cfg_kwargs)
            step = dict(training=training, mixup_type=mixup_type, label_smoothing=label_smoothing,
                        with_loss=with_loss, dtype=self.dtype, use_dropblock=use_dropblock,
                        kd_temp=kd_temp)
            prim = self._primary.get(bool(use_resnet_d))
            if self.native:
                rt = NativeRuntime(NativeModel(cfg, batch, height, width,
                                               deterministic=self.deterministic, **step),
                                   self.device, share=prim)
            else:
                rt = Runtime(build_plan(cfg, batch, height, width, **step), self.device, share=prim,
                             deterministic=self.deterministic)
            if prim is None:
                self._primary[bool(use_resnet_d)] = rt
                if self._pending_weights is not None:
                    rt.set_weights(self._pending_weights)
                else:
                    self.init_weights(rt)
            self._runtimes[key] = rt
        return rt

    def init_weights(self, rt: Runtime):
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
        "bl_beta", "seed", "device", "deterministic", "native")}
    if flags:
        raise TypeError("build_model: unknown flag(s) %s" % sorted(flags))
    ctor.setdefault("resnet_size", DEFAULTS["resnet_size"])
    model = Model(**ctor)
    model.use_resnet_d = bool(use_resnet_d)
    return model


class Trainer:
    """One data-parallel replica of the training step (resnet_model_fn's TRAIN branch +
    get_train_op): owns the step's static buffers, the LR schedule and the CUDA graphs."""

    def __init__(self, model: Model, params: dict, height=224, width=224, *, use_cuda_graph=True,
                 lam_seed=7, num_images=None):
        """num_images: training images per epoch for the LR and keep-prob schedules (default: the
        dataset's data_config count)."""
        p = params
        if p.get("cls_loss_type", "softmax") != "softmax":
            raise NotImplementedError("only cls_loss_type='softmax' is on the hot path")
        self.model = model
        self.p = p
        self.world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1
        self.local_batch = per_device_batch_size(p["batch_size"], self.world)
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
        self.loss_scale = float(p.get("loss_scale", 1) or 1)
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
        # input double-buffering: prefetch() copies the NEXT batch host->device on a side stream
        # while the current step computes; train_step() then takes it with a device-side copy
        self._copy_stream = torch.cuda.Stream(self.rt.dev)
        self._staged = None
        self._consumed = None
        self._stage_imgs = None
        self._stage_labs = None

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
            for fn in fns + [lambda: rt.run(rt.plan.update)]:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    fn()
                graphs.append(g)
        torch.cuda.current_stream(rt.dev).wait_stream(s)
        self._graphs = graphs

    def _fwd_bwd(self):
        rt = self.rt
        rt.run_forward()
        # (a second stream for the wgrad GEMMs: Runtime.run(..., overlap_wgrad=True); off by default,
        # every kernel already spans the GPU)
        rt.run(rt.plan.backward, overlap_wgrad=os.environ.get("ACNN_OVERLAP_WGRAD", "0") == "1")

    def prefetch(self, images, labels):
        """Start the host->device copy of the next step's inputs (pinned host tensors) on a side
        stream; the following train_step(None, None) consumes them.  Lets the PCIe transfer of
        step i+1 overlap the compute of step i."""
        if self._stage_imgs is None:
            self._stage_imgs = torch.empty_like(self.images_buf)
            self._stage_labs = torch.empty_like(self.labels_buf)
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
        the DropBlock schedule for this step.
        Returns the device tensor [cross_entropy, l2_loss(, kd_loss)] of this replica (read it with
        .tolist() -- that read is the only host sync of the step)."""
        rt = self.rt
        if images is None:
            if self._staged is None:
                raise ValueError("train_step() without inputs needs a preceding prefetch()")
            torch.cuda.current_stream(rt.dev).wait_event(self._staged)
            self._staged = None
            images, labels = self._stage_imgs, self._stage_labs
        self.images_buf.copy_(images, non_blocking=True)
        self.labels_buf.copy_(labels, non_blocking=True)
        if images is self._stage_imgs:
            self._consumed = torch.cuda.Event()
            self._consumed.record(torch.cuda.current_stream(rt.dev))
        return self._step(lam1, lam2, teacher_logits, keep_prob)

    def train_step_cropped(self, desc, labels, mean, lam1=None, lam2=None, teacher_logits=None, keep_prob=None):
        """train_step with the images made on the device from training crop windows: one
        acnn_set_images_cropped launch (flip, resize to H x W, - mean) on the current stream, then the step.
        desc: a CUDA uint8 tensor of input_batch 32-byte acnn_crop_desc (imagenet_train.CROP_DESC_DTYPE,
        checked by the caller); labels int32 [input_batch]; the rest as train_step."""
        self.rt.set_images_cropped(desc, mean)
        self.labels_buf.copy_(labels, non_blocking=True)
        return self._step(lam1, lam2, teacher_logits, keep_prob)

    def _step(self, lam1, lam2, teacher_logits, keep_prob):
        rt = self.rt
        if self.mixup_type:
            n = self.input_batch // 2
            if lam1 is None:
                lam1 = torch.from_numpy(self.rng.beta(0.2, 0.2, n).astype(np.float32))
            self.lam1_buf.copy_(torch.as_tensor(lam1, dtype=torch.float32), non_blocking=True)
            if self.mixup_type == 2:
                if lam2 is None:
                    lam2 = torch.from_numpy(self.rng.beta(0.2, 0.2, n).astype(np.float32))
                self.lam2_buf.copy_(torch.as_tensor(lam2, dtype=torch.float32), non_blocking=True)
        if self.kd_temp > 0:
            if teacher_logits is None:
                raise ValueError("kd_temp > 0: train_step needs teacher_logits")
            self.teacher_buf.copy_(torch.as_tensor(teacher_logits, dtype=torch.float32),
                                   non_blocking=True)
        lr = self.learning_rate_fn(self.global_step)
        slot = self.global_step % len(self._hp_ring)
        if self._hp_events[slot] is not None:
            self._hp_events[slot].synchronize()          # its copy of 4 steps ago has executed
        hp = self._hp_ring[slot]
        hp[0] = lr
        hp[1] = self.p["momentum"]
        hp[2] = self.p["weight_decay"]
        hp[3] = 1.0 / (self.world * self.loss_scale)
        if keep_prob is None:
            keep_prob = self.keep_prob_fn(self.global_step) if self.keep_prob_fn else 1.0
        hp[4] = keep_prob
        hp.view(torch.int32)[5] = self.global_step & 0x7fffffff      # Philox counter of the masks
        rt.hp.copy_(hp, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(rt.dev))
        self._hp_events[slot] = ev
        if self.use_graph and self._graphs is None:
            self._capture()
        if self.world == 1:
            if self.use_graph:
                self._graphs[0].replay()
            else:
                self._fwd_bwd()
        else:
            self._fwd_bwd_allreduce()
        if self.use_graph:
            self._graphs[-1].replay()
        else:
            rt.run(rt.plan.update)
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

    def _fwd_bwd_allreduce(self):
        """forward + backward with the gradient all-reduce overlapped: the backward is cut into
        segments (each its own CUDA graph), and as soon as a segment has produced the last gradient
        of a bucket that bucket is all-reduced asynchronously on NCCL's stream while the next
        segment computes (assembled_cnn_b200/dp.py)."""
        rt = self.rt
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
            else:
                works.append(dp.all_reduce_bucket(rt.grads, ev[1], ev[2], async_op=True))
        for w in works:
            w.wait()            # stream-level wait: the update runs after every bucket


_TRAINERS = {}


def l2_loss(rt: Runtime, weight_decay: float):
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
                native=model.native, **model.cfg_kwargs)
    rep.set_weights({n: src.get_tf(n).detach().float().cpu().clone() for n in names})
    return rep


def _grown(buf, nbytes, **kw):
    if buf is not None and buf.numel() >= nbytes:
        return buf
    return torch.empty(max(nbytes + nbytes // 4, 1), dtype=torch.uint8, **kw)


def _pack_u8(hbuf, dbuf, arrays, device):
    """Packs uint8 arrays at 16-byte aligned offsets into the pinned host buffer `hbuf` and enqueues its copy
    to the device buffer `dbuf` on the current stream; either buffer is replaced by a larger one when it is
    too small (None: allocate).  Returns (hbuf, dbuf, the device address of each array)."""
    offs = np.cumsum([0] + [(a.nbytes + 15) // 16 * 16 for a in arrays])
    total = int(offs[-1])
    hbuf = _grown(hbuf, total, pin_memory=True)
    dbuf = _grown(dbuf, total, device=device)
    hnp, base = hbuf.numpy(), dbuf.data_ptr()
    for a, o in zip(arrays, offs):
        hnp[o:o + a.nbytes] = a.reshape(-1)
    dbuf[:total].copy_(hbuf[:total], non_blocking=True)
    return hbuf, dbuf, [base + int(o) for o in offs[:-1]]


class _EvalPipeline:
    """The evaluation loop of one device: decoded batches go from a ring of pinned host buffers to one of
    two device slots on a copy stream, overlapped with the previous batch's forward; the device work of
    a batch (`_body`: input preparation, eval forward, metric kernel) runs as one CUDA graph per (slot,
    valid rows).  A subclass fills a host buffer and enqueues its copy (`_stage`) and defines `_body`."""

    RING = 3        # pinned host batches

    def __init__(self, model, batch, size, use_resnet_d, use_cuda_graph):
        from .imagenet_c import CHANNEL_MEANS
        self.dev = torch.device(model.device)
        torch.cuda.set_device(self.dev)
        self.rt = model.runtime(batch, size, size, training=False, use_resnet_d=use_resnet_d)
        self.batch, self.use_graph = batch, use_cuda_graph
        self.logits = self.rt.t[self.rt.plan.meta["logits"]][:, :model.num_classes]
        self.host_free = [None] * self.RING
        self.slot_free = [None, None]
        self.mean = torch.tensor(CHANNEL_MEANS, dtype=torch.float32, device=self.dev)
        self.copy_stream = torch.cuda.Stream(self.dev)
        self.graphs = {}
        self.warm = False
        self.k = 0

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

    def run_batch(self, images, labels):
        """Evaluate one batch of len(images) <= batch rows."""
        n, h, slot = len(images), self.k % self.RING, self.k % 2
        self.k += 1
        if self.host_free[h] is not None:
            self.host_free[h].synchronize()          # its previous host -> device copy has run
        main, cs = torch.cuda.current_stream(self.dev), self.copy_stream
        if self.slot_free[slot] is not None:
            cs.wait_event(self.slot_free[slot])       # the batch before the previous one has read it
        with torch.cuda.stream(cs):
            self._stage(h, slot, images, labels)
            copied = torch.cuda.Event()
            copied.record(cs)
        self.host_free[h] = copied
        main.wait_event(copied)
        if self.use_graph and self.warm:
            self._graph(slot, n).replay()
        else:
            self._body(slot, n)        # the first batch also loads every kernel before any capture
            self.warm = True
        ev = torch.cuda.Event()
        ev.record(main)
        self.slot_free[slot] = ev


class _CorruptionEvalDevice(_EvalPipeline):
    """The robustness evaluation's loop: fixed-size uint8 batches; the u8 -> f32 input conversion, the
    eval forward and the top-1 count run as one CUDA graph per (slot, valid rows)."""

    def __init__(self, model, batch, size, use_resnet_d, use_cuda_graph):
        super().__init__(model, batch, size, use_resnet_d, use_cuda_graph)
        u8 = dict(dtype=torch.uint8)
        self.host = [(torch.zeros(batch, size, size, 3, **u8).pin_memory(),
                      torch.zeros(batch, dtype=torch.int32).pin_memory()) for _ in range(self.RING)]
        self.slots = [(torch.zeros(batch, size, size, 3, **u8, device=self.dev),
                       torch.zeros(batch, dtype=torch.int32, device=self.dev)) for _ in range(2)]
        self.acc = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self.pred = torch.zeros(batch, dtype=torch.int32, device=self.dev)
        self.decoders, self._files = [None, None], None

    def _stage(self, h, slot, images, labels):
        """`images` a list of uint8 [H, W, 3] arrays, `labels` ints; or, from run_batch_encoded, the files'
        encoded bytes, decoded on the copy stream straight into the slot."""
        hu8, hlab = self.host[h]
        du8, dlab = self.slots[slot]
        if self._files is None:
            for i, a in enumerate(images):
                hu8[i].copy_(torch.from_numpy(a))
            du8.copy_(hu8, non_blocking=True)
        else:
            from . import imagenet_c, jpeg
            files, S = self._files, du8.shape[1]
            desc = jpeg.parse(images)
            for i, d in enumerate(desc):      # a wrong size raises decode_image's error, as the PIL path does
                if d["supported"] and (int(d["height"]), int(d["width"])) != (S, S):
                    imagenet_c.decode_image(files[i], S)
            if self.decoders[slot] is None:
                self.decoders[slot] = jpeg.JpegDecoder(self.dev)
            row = S * S * 3
            self.decoders[slot].stage(images, None, torch.cuda.current_stream(self.dev),
                                      fallback=lambda i: imagenet_c.decode_image(files[i], S),
                                      out=du8.view(-1), out_offsets=np.arange(len(images), dtype=np.int64) * row)
        hlab[:len(images)].copy_(torch.as_tensor(labels, dtype=torch.int32))
        dlab.copy_(hlab, non_blocking=True)

    def run_batch_encoded(self, buffers, labels, files):
        """run_batch from the encoded bytes of `files` (jpeg.JpegDecoder on the copy stream; PIL, through
        imagenet_c.decode_image, for the images the device does not decode)."""
        self._files = files
        try:
            self.run_batch(buffers, labels)
        finally:
            self._files = None

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

    def __init__(self, model, batch, size, use_resnet_d, use_cuda_graph, label_dtype=torch.int32):
        super().__init__(model, batch, size, use_resnet_d, use_cuda_graph)
        lab = dict(dtype=label_dtype)
        self.size = size
        # pinned image bytes (grown on demand), labels, descriptors
        self.host = [[torch.empty(0, dtype=torch.uint8), torch.zeros(batch, **lab).pin_memory(),
                      torch.zeros(32 * batch, dtype=torch.uint8).pin_memory()] for _ in range(self.RING)]
        # device image bytes (allocated on the copy stream, grown on demand), labels, descriptors: a graph
        # holds the descriptor table's address only, so the image bytes may move
        self.slots = [[None, torch.zeros(batch, **lab, device=self.dev),
                       torch.zeros(32 * batch, dtype=torch.uint8, device=self.dev)] for _ in range(2)]
        self.decoders, self._geometry = [None, None], None

    def _stage(self, h, slot, images, labels):
        """`images` a list of (uint8 [H, W, 3] array, eval_geometry) pairs, `labels` ints; or, from
        run_batch_encoded, encoded images, decoded on the copy stream."""
        from .imagenet_eval import DESC_DTYPE, check_descriptors
        n = len(images)
        hbuf, hlab, hdesc = self.host[h]
        desc = hdesc.numpy().view(DESC_DTYPE)
        if self._geometry is None:
            self.host[h][0], self.slots[slot][0], addrs = _pack_u8(hbuf, self.slots[slot][0],
                                                                  [a for a, _ in images], self.dev)
            for i, (a, (s, rh, rw, cy, cx)) in enumerate(images):
                desc[i] = (addrs[i], a.shape[0], a.shape[1], rh, rw, cy, cx)
        else:
            from . import jpeg
            if self.decoders[slot] is None:
                self.decoders[slot] = jpeg.JpegDecoder(self.dev)
            placed = self.decoders[slot].stage(images, None, torch.cuda.current_stream(self.dev))
            for i, (addr, ih, iw) in enumerate(placed):
                s, rh, rw, cy, cx = self._geometry(ih, iw)
                desc[i] = (addr, ih, iw, rh, rw, cy, cx)
        check_descriptors(desc, n, self.size)
        hlab[:n].copy_(torch.as_tensor(labels, dtype=hlab.dtype))
        _, dlab, ddesc = self.slots[slot]
        ddesc.copy_(hdesc, non_blocking=True)
        dlab.copy_(hlab, non_blocking=True)

    def run_batch_encoded(self, buffers, labels, geometry):
        """run_batch from encoded images (jpeg.JpegDecoder on the copy stream; PIL for the images the device
        does not decode); geometry(h, w) gives an image's imagenet_eval.eval_geometry."""
        self._geometry = geometry
        try:
            self.run_batch(buffers, labels)
        finally:
            self._geometry = None


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

    def run_batch(self, images, labels):
        super().run_batch(images, labels)
        n = len(images)
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

    def run_batch(self, images, labels):
        super().run_batch(images, labels)
        n = len(images)
        self.index[self.done:self.done + n].copy_(self.feat[:n])
        self.labels[self.done:self.done + n].copy_(self.batch_labels[:n])
        self.done += n


def _read_file(path):
    with open(path, "rb") as f:
        return f.read()


def corruption_error(model, data_dir, label_file, *, batch_size=128, image_size=224, label_offset=1,
                     robustness_type="ce", devices=None, use_resnet_d=None, global_step=None,
                     use_cuda_graph=True, num_workers=None):
    """mce/eval_robustness.py (show_corruption_error, --robustness_type ce): the top-1 error of `model`
    on every distortion of ALEXNET_CE, pooled over data_dir/<distortion>/<severity 1..5>/<synset>/*,
    its AlexNet-normalised CE and their means.  Labels are synsets2idx[synset dir] + label_offset from
    `label_file`; images must decode to image_size x image_size (RGB), fed as uint8 minus CHANNEL_MEANS.

    Decoding runs on a pool of `num_workers` CPU threads (PIL); the device work of a batch (uint8 ->
    fp32, eval forward in the model's dtype, softmax top-1 count) is one CUDA graph replay
    (use_cuda_graph=False: the same launches, eager).  The last batch of a distortion is padded to
    batch_size and its padding rows are masked.  `devices` (default: the model's device) split the
    distortions as the reference's process() does; every device gets a replica with the model's weights.
    Returns {'<distortion>': {'error', 'ce'}, ..., 'mCE', 'mCE_unnormalized'} (+ 'global_step')."""
    import threading
    from concurrent.futures import ThreadPoolExecutor
    from . import imagenet_c
    from .metrics import DISTORTIONS, CorruptionError
    if robustness_type == "fr":
        raise ValueError("not yet supported ({}".format(robustness_type))
    if robustness_type != "ce":
        raise ValueError("invalid type ({})".format(robustness_type))
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
            decode = lambda files: [pool.submit(_read_file, f) for f in files]
            ahead = 4                                   # batches decoding ahead of the GPU
            pending = [decode(b[1]) for b in batches[:ahead]]
            counts = {}
            for j, (d, files, labels) in enumerate(batches):
                futs = pending.pop(0)
                if j + ahead < len(batches):
                    pending.append(decode(batches[j + ahead][1]))
                ev.run_batch_encoded([f.result() for f in futs], labels, files)
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
    decode = lambda recs: [pool.submit(imagenet_eval.read_encoded, r[0], r[1], r[2]) for r in recs]
    geometry = lambda h, w: imagenet_eval.eval_geometry(h, w, preprocessing_type, image_size)
    try:
        ahead = 4                                   # batches decoding ahead of the GPU
        pending = [decode(b) for b in batches[:ahead]]
        for j, recs in enumerate(batches):
            futs = pending.pop(0)
            if j + ahead < len(batches):
                pending.append(decode(batches[j + ahead]))
            ev.run_batch_encoded([f.result() for f in futs], [r[3] for r in recs], geometry)
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


class _TrainFeed:
    """The training input's staging ring: per step, the crop windows packed into a growable pinned uint8
    buffer with one acnn_crop_desc each, the labels and (KD) the teacher logits, copied to one of two
    device slots on a copy stream while the previous step computes; `step` makes the images on the device
    (Trainer.train_step_cropped) and runs the training step."""

    RING = 3        # pinned host batches

    def __init__(self, trainer, kd):
        from .imagenet_c import CHANNEL_MEANS
        self.tr, self.dev = trainer, trainer.rt.dev
        n, nc = trainer.input_batch, trainer.model.num_classes
        i32, f32 = dict(dtype=torch.int32), dict(dtype=torch.float32)
        self.host = [[None, torch.zeros(n, **i32).pin_memory(), torch.zeros(32 * n, dtype=torch.uint8).pin_memory(),
                      torch.zeros(n, nc, **f32).pin_memory() if kd else None] for _ in range(self.RING)]
        # a step's graph holds no address of these: the image bytes may move when the buffer grows
        self.slots = [[None, torch.zeros(n, **i32, device=self.dev),
                       torch.zeros(32 * n, dtype=torch.uint8, device=self.dev),
                       torch.zeros(n, nc, **f32, device=self.dev) if kd else None] for _ in range(2)]
        self.mean = torch.tensor(CHANNEL_MEANS, dtype=torch.float32, device=self.dev)
        self.copy_stream = torch.cuda.Stream(self.dev)
        self.host_free = [None] * self.RING
        self.slot_free = [None, None]
        self.copied = [None, None]
        self.decoders = [None, None]
        self.staged = self.consumed = 0

    def stage(self, windows, labels, teacher_logits=None):
        """`windows` input_batch (uint8 [h, w, 3] array, flip) pairs, `labels` ints, `teacher_logits` float32
        [input_batch, num_classes] with KD."""
        def place(h, slot):
            self.host[h][0], self.slots[slot][0], addrs = _pack_u8(self.host[h][0], self.slots[slot][0],
                                                                  [a for a, _ in windows], self.dev)
            return [(ad, a.shape[0], a.shape[1], flip) for ad, (a, flip) in zip(addrs, windows)]
        self._stage(place, labels, teacher_logits)

    def stage_encoded(self, items, labels, teacher_logits=None):
        """As stage, from input_batch (encoded JPEG bytes, (y, x, h, w) window, flip) triples: the windows are
        decoded on the copy stream (jpeg.JpegDecoder, one per slot; PIL's decode_rgb for the images the
        device does not decode)."""
        def place(h, slot):
            from . import jpeg
            if self.decoders[slot] is None:
                self.decoders[slot] = jpeg.JpegDecoder(self.dev)
            got = self.decoders[slot].stage([b for b, _, _ in items], np.array([w for _, w, _ in items], np.int32),
                                            self.copy_stream)
            return [(ad, hh, ww, flip) for (ad, hh, ww), (_, _, flip) in zip(got, items)]
        self._stage(place, labels, teacher_logits)

    def _stage(self, place, labels, teacher_logits):
        from .imagenet_train import CROP_DESC_DTYPE, check_crop_descriptors
        h, slot = self.staged % self.RING, self.staged % 2
        self.staged += 1
        if self.host_free[h] is not None:
            self.host_free[h].synchronize()          # its previous host -> device copy has run
        cs = self.copy_stream
        if self.slot_free[slot] is not None:
            cs.wait_event(self.slot_free[slot])       # the step before the previous one has read it
        with torch.cuda.stream(cs):
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
            ev = torch.cuda.Event()
            ev.record(cs)
        self.host_free[h] = self.copied[slot] = ev

    def step(self, lam1=None, lam2=None):
        """The training step of the oldest staged batch; returns Trainer.train_step's loss tensor."""
        slot = self.consumed % 2
        self.consumed += 1
        main = torch.cuda.current_stream(self.dev)
        main.wait_event(self.copied[slot])
        _, dlab, ddesc, dteach = self.slots[slot]
        loss = self.tr.train_step_cropped(ddesc, dlab, self.mean, lam1=lam1, lam2=lam2, teacher_logits=dteach)
        ev = torch.cuda.Event()
        ev.record(main)
        self.slot_free[slot] = ev
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


def train_and_evaluate(data_dir, model_dir, *, epochs_between_evals=1, stop_threshold=None, max_train_steps=None,
                       image_size=224, seed=0, use_cuda_graph=True, num_workers=None, **flags):
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
    checkpoints and evaluates.  Returns the list of the cycles' evaluation results (the recall dicts with
    zeroshot_eval)."""
    from concurrent.futures import ThreadPoolExecutor
    from . import imagenet_train as it
    from .checkpoint import CheckpointKeeper, latest_checkpoint, restore, save_checkpoint, warm_start
    from .imagenet_eval import eval_size
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
    dist = torch.distributed.is_initialized()
    world = torch.distributed.get_world_size() if dist else 1
    rank = torch.distributed.get_rank() if dist else 0
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
    trainer = Trainer(model, p, size, size, use_cuda_graph=use_cuda_graph, num_images=num_images)
    ckpt = latest_checkpoint(model_dir) if os.path.isdir(model_dir) else None
    if ckpt:
        restore(model, ckpt, trainer)
    elif p["pretrained_model_checkpoint_path"]:
        warm_start(model, p["pretrained_model_checkpoint_path"], trainer.global_step)
    if p["eval_only"] or not p["train_epochs"]:
        schedule, first = [0], 0
    else:
        args = (p["train_epochs"], epochs_between_evals, p["ratio_fine_eval"])
        full = it.epoch_schedule(*args)
        schedule = it.epoch_schedule(*args, cur_epoch=trainer.global_step // steps_per_epoch)
        first = len(full) - len(schedule)          # the cycle index keys the cycle's randomness
    total_train_steps = p["train_epochs"] * steps_per_epoch
    save_steps = int(p["save_checkpoints_epochs"] * steps_per_epoch)
    shuffle_buffer = it.SHUFFLE_BUFFER.get(ds_name, it.DEFAULT_SHUFFLE_BUFFER)
    keeper = CheckpointKeeper(model_dir, p["num_best_ckpt_to_keep"], p["keep_ckpt_every_eval"], maximize=True) \
        if rank == 0 else None

    def save():
        if rank == 0:
            save_checkpoint(os.path.join(model_dir, "model.ckpt-%d" % trainer.global_step), model, trainer)
            _prune_checkpoints(model_dir, p["keep_checkpoint_max"])

    feed = _TrainFeed(trainer, kd)
    n_lam = trainer.input_batch // 2
    pool = ThreadPoolExecutor(max_workers=num_workers or min(32, os.cpu_count() or 1))
    results = []
    try:
        for ci, epochs in enumerate(schedule):
            c = first + ci
            if epochs:
                stream = it.CycleStream(counts, seed, c, epochs * (2 if trainer.mixup_type == 1 else 1),
                                        shuffle_buffer, trainer.input_batch, world, rank)
                steps = stream.steps if max_train_steps is None else min(stream.steps, max_train_steps)

                def decode(t, c=c, stream=stream):
                    return [(pool.submit(it.encoded_window, *records[r][:3], seed, c, pos,
                                         p["training_random_crop"]), r) for pos, r in stream.records(t)]
                ahead = 4                               # steps decoding ahead of the GPU
                pending = [decode(t) for t in range(min(ahead, steps))]

                def stage(t):
                    futs = pending.pop(0)
                    if t + ahead < steps:
                        pending.append(decode(t + ahead))
                    teacher = np.stack([records[r][4] for _, r in futs]) if kd else None
                    feed.stage_encoded([f.result() for f, _ in futs], [records[r][3] for _, r in futs], teacher)

                if steps:
                    stage(0)
                for t in range(steps):
                    lam1 = lam2 = None
                    if trainer.mixup_type:
                        lam = it.mixup_lambdas(seed, trainer.global_step, rank, 2 * n_lam).reshape(2, n_lam)
                        lam1, lam2 = lam[0], (lam[1] if trainer.mixup_type == 2 else None)
                    feed.step(lam1, lam2)
                    if t + 1 < steps:
                        stage(t + 1)
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
    return results
