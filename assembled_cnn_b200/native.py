"""Python facade of the MODEL-LEVEL C ABI (include/acnn_model.h): the layer plan is built and executed
by libacnn.so (csrc/model_plan.cu, csrc/model_exec.cu); this module only

  * fills `acnn_model_config` from the reference's constructor flags (functions/model_fns.py:141-157),
  * allocates the caller-owned device buffers as torch tensors and hands their pointers to acnn_bind,
  * exposes the variables (TF names / layouts) and the static input / output buffers as torch views,
  * and wraps the host CRC-32C of include/acnn.h (crc32c) for the TFRecord reader and writer.

`NativeModel` (plan + introspection) needs no GPU; `NativeRuntime` (execution) has no CPU path.
The parity tests run NativeRuntime op by op in lockstep with the oracle's plan interpreter, which walks
plan.py's Python plan of the same configuration (NativeModel.python_mirror); tests/test_native_plan_cpu.py
pins the two plans to the same text.
"""
from __future__ import annotations

import ctypes as C
import os
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from .plan import ModelConfig, Param, Slot, Tensor

_DT = {0: "bf16", 1: "f32", 2: "i32", 3: "f16"}
# model dtype <-> acnn_model_config.dtype (ACNN_BF16 / ACNN_F32 / ACNN_F16)
_CFG_DTYPE = {"bf16": 0, "fp32": 1, "fp16": 3}


class Config(C.Structure):
    """struct acnn_model_config."""
    _fields_ = [("struct_size", C.c_int32), ("resnet_size", C.c_int32), ("num_classes", C.c_int32),
                ("resnet_version", C.c_int32), ("no_downsample", C.c_int32), ("zero_gamma", C.c_int32),
                ("use_se_block", C.c_int32), ("use_sk_block", C.c_int32), ("embedding_size", C.c_int32),
                ("anti_alias_filter_size", C.c_int32), ("bl_alpha", C.c_int32), ("bl_beta", C.c_int32),
                ("use_resnet_d", C.c_int32), ("anti_alias_type", C.c_char * 32),
                ("pool_type", C.c_char * 16), ("loss_type", C.c_char * 16), ("bn_momentum", C.c_double),
                ("bn_epsilon", C.c_double), ("batch", C.c_int32), ("height", C.c_int32),
                ("width", C.c_int32), ("training", C.c_int32), ("mixup_type", C.c_int32),
                ("with_loss", C.c_int32), ("dtype", C.c_int32), ("use_dropblock", C.c_int32),
                ("deterministic", C.c_int32), ("fuse_bn_pairs", C.c_int32),
                ("label_smoothing", C.c_double), ("kd_temp", C.c_double), ("loss_scale", C.c_double)]


class Sizes(C.Structure):
    """struct acnn_model_sizes."""
    _fields_ = [(n, C.c_int64) for n in (
        "param_elems", "state_elems", "dgrad_elems", "w_fprop_elems", "w_dgrad_elems",
        "workspace_bytes", "hp_offset", "loss_offset", "decay_flags_offset", "zero_offset",
        "zero_bytes", "work_offset", "work_bytes")] + [(n, C.c_int32) for n in (
            "n_variables", "n_tensors", "n_forward", "n_loss_first", "n_backward", "n_update",
            "input_batch", "ld_logits")]


class VariableInfo(C.Structure):
    """struct acnn_variable_info."""
    _fields_ = [("name", C.c_char * 160), ("kind", C.c_char * 24), ("buffer", C.c_int32),
                ("tf_rank", C.c_int32), ("store_rank", C.c_int32), ("tf_shape", C.c_int64 * 4),
                ("store_shape", C.c_int64 * 4), ("offset", C.c_int64), ("size", C.c_int64),
                ("dgrad_off", C.c_int64), ("decay", C.c_int32), ("zero_init", C.c_int32),
                ("grad_ready_op", C.c_int32), ("reserved_", C.c_int32)]


class TensorInfo(C.Structure):
    """struct acnn_tensor_info."""
    _fields_ = [("name", C.c_char * 64), ("dtype", C.c_int32), ("rank", C.c_int32),
                ("shape", C.c_int64 * 5), ("offset", C.c_int64)]


MODEL_HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include",
                            "acnn_model.h")
_vp, _i, _i64 = C.c_void_p, C.c_int, C.c_int64
PROTOTYPES = {
    "acnn_model_config_init": (None, [C.POINTER(Config)]),
    "acnn_create": (_i, [C.POINTER(Config), C.POINTER(_vp)]),
    "acnn_destroy": (None, [_vp]),
    "acnn_model_get_sizes": (_i, [_vp, C.POINTER(Sizes)]),
    "acnn_variable_count": (_i, [_vp]),
    "acnn_variable_info_get": (_i, [_vp, _i, C.POINTER(VariableInfo)]),
    "acnn_variable_pack": (_i, [_vp, _i, _vp, _vp]),
    "acnn_variable_unpack": (_i, [_vp, _i, _vp, _vp]),
    "acnn_tensor_count": (_i, [_vp]),
    "acnn_tensor_info_get": (_i, [_vp, _i, C.POINTER(TensorInfo)]),
    "acnn_find_tensor": (_i, [_vp, C.c_char_p, _i]),
    "acnn_bind": (_i, [_vp] * 9),
    "acnn_validate": (_i, [_vp]),
    "acnn_set_loss_scale": (_i, [_vp, C.c_double]),
    "acnn_set_dynamic_loss_scale": (_i, [_vp, _vp, C.c_double, _i, _i, _vp]),
    "acnn_get_loss_scale_state": (_i, [_vp, _vp, _vp]),
    "acnn_set_dropblock": (_i, [_vp, C.c_uint64, _i]),
    "acnn_set_inputs": (_i, [_vp] * 7),
    "acnn_set_images_u8": (_i, [_vp] * 4),
    "acnn_set_images_resized": (_i, [_vp, _vp, _i, _vp, _vp]),
    "acnn_set_images_cropped": (_i, [_vp] * 4),
    "acnn_set_images_augmented": (_i, [_vp] * 6),
    "acnn_set_hparams": (_i, [_vp, _vp, _vp]),
    "acnn_get_logits": (_i, [_vp, _vp, _vp]),
    "acnn_get_loss": (_i, [_vp, _vp, _vp]),
    "acnn_forward": (_i, [_vp, _vp]),
    "acnn_loss": (_i, [_vp, _vp]),
    "acnn_backward": (_i, [_vp, _vp]),
    "acnn_backward_range": (_i, [_vp, _i, _i, _vp]),
    "acnn_sgd_step": (_i, [_vp, _vp]),
    "acnn_step": (_i, [_vp, _vp]),
    "acnn_replica_accumulate_model": (_i, [_vp, _i, _vp, _vp, _vp, _i64, _i64, _i, _vp]),
    "acnn_run_ops": (_i, [_vp, _i, _i, _i, _vp]),
    "acnn_clear_step_buffers": (_i, [_vp, _vp]),
    "acnn_op_kind": (C.c_char_p, [_vp, _i, _i]),
    "acnn_op_conv_info": (_i, [_vp, _i, _i, C.POINTER(_lib.ConvGeom), C.POINTER(C.c_int64), C.POINTER(_i)]),
    "acnn_plan_dump": (_i64, [_vp, _vp, _i64]),
}

_bound = None


def lib():
    """libacnn.so with the model-level prototypes bound (raises AcnnError if it is not built)."""
    global _bound
    if _bound is None:
        l = _lib.load()
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(l, name)
            fn.restype, fn.argtypes = res, args
        _bound = l
    return _bound


def crc32c(data, crc=0):
    """acnn_crc32c: the CRC-32C of the bytes-like `data` (bytes, bytearray, memoryview; not copied),
    continued from `crc`, a value this function returned (0 starts a new one)."""
    buf = np.frombuffer(data, dtype=np.uint8)
    return _lib.load().acnn_crc32c(buf.ctypes.data, buf.size, crc)


def make_config(cfg: ModelConfig, batch, height, width, *, training=True, mixup_type=0,
                label_smoothing=0.0, with_loss=True, dtype="bf16", use_dropblock=False, kd_temp=0.0,
                deterministic=None, loss_scale=1.0, eps=1e-5) -> Config:
    if dtype not in _CFG_DTYPE:
        raise ValueError("dtype must be one of: ('bf16', 'fp32', 'fp16')")
    c = Config()
    lib().acnn_model_config_init(C.byref(c))
    for k in ("resnet_size", "num_classes", "resnet_version", "embedding_size",
              "anti_alias_filter_size", "bl_alpha", "bl_beta"):
        setattr(c, k, int(getattr(cfg, k)))
    for k in ("no_downsample", "zero_gamma", "use_se_block", "use_sk_block", "use_resnet_d"):
        setattr(c, k, int(bool(getattr(cfg, k))))
    for k in ("anti_alias_type", "pool_type", "loss_type"):
        raw = str(getattr(cfg, k)).encode()
        if len(raw) >= getattr(Config, k).size:
            raise ValueError("%s=%r is too long for the C ABI" % (k, getattr(cfg, k)))
        setattr(c, k, raw)
    c.bn_momentum, c.bn_epsilon = float(cfg.bn_momentum), float(eps)
    c.batch, c.height, c.width = int(batch), int(height), int(width)
    c.training, c.mixup_type, c.with_loss = int(bool(training)), int(mixup_type), int(bool(with_loss))
    c.dtype = _CFG_DTYPE[dtype]
    c.use_dropblock = int(bool(use_dropblock))
    c.deterministic = -1 if deterministic is None else int(bool(deterministic))
    c.fuse_bn_pairs = int(os.environ.get("ACNN_FUSE_BN_PAIRS", "1") == "1")
    c.label_smoothing, c.kd_temp, c.loss_scale = float(label_smoothing), float(kd_temp), float(loss_scale)
    return c


class NativeOp:
    """One op of the native plan: kind + position (the arguments live in the library)."""
    __slots__ = ("kind", "phase", "index", "a")

    def __init__(self, kind, phase, index):
        self.kind, self.phase, self.index, self.a = kind, phase, index, {}

    def __repr__(self):
        return "NativeOp(%s, %s[%d])" % (self.kind, "FBU"[self.phase], self.index)


class NativeModel:
    """acnn_create() + introspection.  Quacks like plan.Plan where model_fns / dp / checkpoint read
    it: .params / .state (name -> Param), .tensors, .meta, .param_elems ..., .forward / .backward /
    .update (NativeOp lists whose slices NativeRuntime.run() turns into acnn_run_ops ranges)."""

    def __init__(self, cfg: ModelConfig, batch, height=224, width=224, **kw):
        self.lib = lib()
        self.cfg, self.shape, self.step_kwargs = cfg, (batch, height, width), dict(kw)
        self.config = make_config(cfg, batch, height, width, **kw)
        h = _vp()
        _lib.check(self.lib.acnn_create(C.byref(self.config), C.byref(h)), "acnn_create")
        self.handle = h
        s = Sizes()
        _lib.check(self.lib.acnn_model_get_sizes(h, C.byref(s)), "acnn_model_get_sizes")
        self.sizes = s
        self.param_elems, self.state_elems, self.dgrad_elems = s.param_elems, s.state_elems, s.dgrad_elems
        self.zero_elems, self.work_elems = s.zero_bytes // 4, s.work_bytes // 4
        self.params, self.state = OrderedDict(), OrderedDict()
        self.grad_ready = {}
        vi = VariableInfo()
        for i in range(s.n_variables):
            _lib.check(self.lib.acnn_variable_info_get(h, i, C.byref(vi)), "acnn_variable_info_get")
            name = vi.name.decode()
            p = Param(name, tuple(vi.tf_shape[:vi.tf_rank]), vi.kind.decode(), vi.offset, vi.size,
                      tuple(vi.store_shape[:vi.store_rank]), vi.buffer == 0, bool(vi.decay),
                      bool(vi.zero_init), vi.dgrad_off)
            (self.params if vi.buffer == 0 else self.state)[name] = p
            if vi.buffer == 0:
                self.grad_ready[name] = vi.grad_ready_op
        self.tensors, self.tensor_offset, self._tensor_names = OrderedDict(), {}, []
        ti = TensorInfo()
        for i in range(s.n_tensors):
            _lib.check(self.lib.acnn_tensor_info_get(h, i, C.byref(ti)), "acnn_tensor_info_get")
            name = ti.name.decode()
            self.tensors[name] = Tensor(name, tuple(ti.shape[:ti.rank]), _DT[ti.dtype])
            self.tensor_offset[name] = ti.offset
            self._tensor_names.append(name)
        self.forward = [NativeOp(self.lib.acnn_op_kind(h, 0, i).decode(), 0, i) for i in range(s.n_forward)]
        self.backward = [NativeOp(self.lib.acnn_op_kind(h, 1, i).decode(), 1, i) for i in range(s.n_backward)]
        self.update = [NativeOp(self.lib.acnn_op_kind(h, 2, i).decode(), 2, i) for i in range(s.n_update)]
        c = self.config
        self.meta = dict(batch=c.batch, height=c.height, width=c.width, training=bool(c.training),
                         mixup_type=c.mixup_type if c.training else 0,
                         label_smoothing=c.label_smoothing, num_classes=c.num_classes,
                         ld_logits=s.ld_logits, bn_momentum=c.bn_momentum,
                         dtype={v: k for k, v in _CFG_DTYPE.items()}[c.dtype],
                         use_dropblock=bool(c.use_dropblock and c.training),
                         kd_temp=c.kd_temp if c.training else 0.0, input_batch=s.input_batch,
                         dropblock_u=[])
        for role in ("images", "labels", "lam1", "lam2", "teacher_logits", "logits", "pooled",
                     "embedding", "ysoft"):
            t = self.lib.acnn_find_tensor(h, role.encode(), 0)
            if t >= 0:
                self.meta[role] = self._tensor_names[t]
        k = 0
        while True:
            t = self.lib.acnn_find_tensor(h, b"dropblock_u", k)
            if t < 0:
                break
            self.meta["dropblock_u"].append(self._tensor_names[t])
            k += 1
        if s.loss_offset >= 0:
            self.meta["loss"] = Slot("zero", (s.loss_offset - s.zero_offset) // 4, 4)

    def grad_done_at(self):
        """name -> index of the backward op after which that variable's gradient is final."""
        return {n: i for n, i in self.grad_ready.items() if i >= 0}

    def all_ops(self):
        return self.forward + self.backward + self.update

    def python_mirror(self):
        """The plan.py plan of the same configuration -- op for op the same plan (pinned text-for-text by
        tests/test_native_plan_cpu.py).  For the parity tests only: the oracle's interpreter
        (oracle/plan_interp.py) walks Python op objects.  Nothing on the product path calls this."""
        from .plan import build_plan
        kw = {k: v for k, v in self.step_kwargs.items() if k not in ("deterministic", "loss_scale", "eps")}
        return build_plan(self.cfg, *self.shape, **kw)

    def conv_info(self, op):
        """(acnn_conv_geom of the plan, algorithmic MACs, aux tiles of the epilogue) of a GEMM op."""
        g, macs, aux = _lib.ConvGeom(), C.c_int64(), C.c_int()
        _lib.check(self.lib.acnn_op_conv_info(self.handle, op.phase, op.index, C.byref(g), C.byref(macs),
                                              C.byref(aux)), "acnn_op_conv_info")
        return g, macs.value, aux.value

    def validate(self):
        """acnn_validate: every op resolves into a launch record (host-only; raises AcnnError otherwise)."""
        _lib.check(self.lib.acnn_validate(self.handle), "acnn_validate")

    def dump(self) -> str:
        n = self.lib.acnn_plan_dump(self.handle, None, 0)
        buf = C.create_string_buffer(n)
        self.lib.acnn_plan_dump(self.handle, buf, n)
        return buf.value.decode()

    def close(self):
        if getattr(self, "handle", None):
            self.lib.acnn_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def check_dynamic_loss_scale(initial_scale, growth_interval):
    """The initial scale of dynamic loss scaling must be > 0 and finite in fp32, the growth interval an integer
    >= 1 (ValueError otherwise)."""
    s = float(initial_scale)
    with np.errstate(over="ignore"):
        ok = s > 0 and np.isfinite(np.float32(s))
    if not ok:
        raise ValueError("initial loss scale must be > 0 and finite in fp32 (got %r)" % (initial_scale,))
    g = growth_interval
    if isinstance(g, bool) or not isinstance(g, (int, np.integer)) or g < 1:
        raise ValueError("loss scale growth interval must be an integer >= 1 (got %r)" % (g,))


def decode_loss_scale_state(words):
    """struct acnn_loss_scale_state from its 8 int32 words (a CPU tensor or array)."""
    v = np.asarray(words, dtype=np.int32)
    f = v.view(np.float32)
    return {"scale": float(f[0]), "good_steps": int(v[1]), "skipped_steps": int(v[2]), "last_scale": float(f[4])}


def _check_u8_images(images_u8, images, mean):
    """Arguments of set_images_u8: uint8 NHWC of the input buffer's shape on its device, float32 mean[3]."""
    if images_u8.dtype != torch.uint8 or tuple(images_u8.shape) != tuple(images.shape) \
            or images_u8.device != images.device or not images_u8.is_contiguous():
        raise ValueError("images_u8 must be a contiguous uint8 tensor %s on %s, got %s %s on %s"
                         % (tuple(images.shape), images.device, images_u8.dtype, tuple(images_u8.shape),
                            images_u8.device))
    if mean.dtype != torch.float32 or mean.numel() != 3 or not mean.is_contiguous():
        raise ValueError("mean must be a contiguous float32 tensor of 3 values")


def _check_desc_args(method, desc, images, mean, n_valid=None):
    """Arguments of set_images_resized / set_images_cropped (`method`): a square input buffer, B descriptors
    of 32 bytes on its device, n_valid (when given) in [0, B], float32 mean[3].  Returns (B, S)."""
    b, h, w, _ = images.shape
    if h != w:
        raise ValueError("%s needs a square input buffer, got %dx%d" % (method, h, w))
    if desc.dtype != torch.uint8 or desc.numel() != 32 * b or desc.device != images.device \
            or not desc.is_contiguous():
        raise ValueError("desc must be a contiguous uint8 tensor of %d descriptors (%d bytes) on %s"
                         % (b, 32 * b, images.device))
    if n_valid is not None and not 0 <= int(n_valid) <= b:
        raise ValueError("n_valid=%d outside [0, %d]" % (int(n_valid), b))
    if mean.dtype != torch.float32 or mean.numel() != 3 or not mean.is_contiguous():
        raise ValueError("mean must be a contiguous float32 tensor of 3 values")
    return b, h


def _check_augment_args(desc, aug, work, images, mean):
    """Arguments of set_images_augmented: those of set_images_cropped, B descriptors of 88 bytes and a work
    buffer of acnn_autoaugment_work_bytes(B, S) bytes, both uint8 on the input buffer's device.
    Returns (B, S)."""
    b, s = _check_desc_args("set_images_cropped", desc, images, mean)
    if aug.dtype != torch.uint8 or aug.numel() != 88 * b or aug.device != images.device or not aug.is_contiguous():
        raise ValueError("aug must be a contiguous uint8 tensor of %d AutoAugment descriptors (%d bytes) on %s"
                         % (b, 88 * b, images.device))
    need = _lib.load().acnn_autoaugment_work_bytes(b, s)
    if work.dtype != torch.uint8 or work.numel() < need or work.device != images.device \
            or not work.is_contiguous():
        raise ValueError("work must be a contiguous uint8 tensor of at least %d bytes on %s" % (need, images.device))
    return b, s


class NativeRuntime:
    """Executes a NativeModel on one H100 through acnn_bind / acnn_run_ops: params / state / grads /
    momentum / hp / t[name] / run(ops) / capture ..., what Model, Trainer, checkpoint and the
    data-parallel schedule drive.  Every buffer of the step but the variables is a view into ONE
    workspace tensor laid out by the library, and run() is a loop inside libacnn.so over launch
    records resolved at bind time.  torch is the device-memory container only, for streams and for
    CUDA-graph capture; there is no CPU path."""

    REPLICA_SAVE, REPLICA_FIRST, REPLICA_MIDDLE, REPLICA_LAST = 0, 1, 2, 3     # acnn.h ACNN_REPLICA_*
    REPLICA_LOSS_FLOATS = 4                                                    # acnn_model.h

    def __init__(self, model: NativeModel, device="cuda:0", share: "NativeRuntime | None" = None):
        if not torch.cuda.is_available():
            raise _lib.AcnnError("assembled_cnn_b200.NativeRuntime needs a CUDA device (sm_90a); "
                                 "there is no CPU fallback")
        self.lib = model.lib
        self.plan = self.model = model
        self.dev = torch.device(device)
        torch.cuda.set_device(self.dev)
        c, s = model.config, model.sizes
        self.training = bool(c.training)
        self.adt = c.dtype                   # ACNN_BF16 / ACNN_F32 / ACNN_F16
        wdt = torch.float16 if self.adt == 3 else torch.bfloat16
        # deterministic: also the split-K of wgrad and of the small SK / SE GEMMs is disabled (one add
        # per output element).  Every reduction is ordered in both modes (split-K partials are summed
        # in split order), so two runs are bit-identical either way.
        self.det = int(c.dtype == 1 if c.deterministic < 0 else bool(c.deterministic))
        f32 = dict(dtype=torch.float32, device=self.dev)
        if share is not None:
            # same model, another batch shape / mode: the variables are shared, not copied
            if share.plan.param_elems != s.param_elems or share.plan.state_elems != s.state_elems \
                    or share.adt != self.adt:
                raise ValueError("NativeRuntime(share=...): parameter layouts differ")
            self.params, self.state, self.w_fprop = share.params, share.state, share.w_fprop
        else:
            self.params = torch.zeros(s.param_elems, **f32)
            self.state = torch.zeros(max(s.state_elems, 1), **f32)
            self.w_fprop = torch.zeros(s.w_fprop_elems, dtype=wdt, device=self.dev)
            for p in model.state.values():
                if p.kind == "moving_variance":
                    self.state[p.offset:p.offset + p.size] = 1.0
        if self.training:
            self.grads = torch.zeros(s.param_elems, **f32)
            self.momentum = share.momentum if (share is not None and share.momentum is not None) \
                else torch.zeros(s.param_elems, **f32)
            self.w_dgrad = torch.zeros(s.w_dgrad_elems, dtype=wdt, device=self.dev)
        else:
            self.grads = self.momentum = self.w_dgrad = None
        self.workspace = torch.zeros(s.workspace_bytes, dtype=torch.uint8, device=self.dev)
        ws = self.workspace

        def view(off, nbytes, dtype):
            return ws[off:off + nbytes].view(dtype)
        # device hyper-parameters: lr, momentum, wd, grad_scale, dropblock keep_prob, global step
        # (uint32 bits, the Philox counter of the DropBlock masks), 2 spare
        self.hp = view(s.hp_offset, 32, torch.float32)
        self.zero = view(s.zero_offset, max(s.zero_bytes, 4), torch.float32)
        self.work = view(s.work_offset, max(s.work_bytes, 4), torch.float32)
        self.decay_flags = view(s.decay_flags_offset, max(s.param_elems // 256, 1), torch.uint8)
        tdt = {"bf16": (torch.bfloat16, 2), "f32": (torch.float32, 4), "f16": (torch.float16, 2),
               "i32": (torch.int32, 4)}
        self.t = {}
        for name, t in model.tensors.items():
            dt, esz = tdt[t.dtype]
            n = esz
            for d in t.shape:
                n *= d
            self.t[name] = view(model.tensor_offset[name], n, dt).view(t.shape)
        ptr = lambda x: None if x is None else x.data_ptr()
        _lib.check(self.lib.acnn_bind(model.handle, ptr(self.params), ptr(self.grads), ptr(self.momentum),
                                      ptr(self.state), ptr(self.w_fprop), ptr(self.w_dgrad), ptr(ws),
                                      self.stream), "acnn_bind")
        self._loss_scale = c.loss_scale
        self.loss_scale_state_buf = None     # int32 [8], struct acnn_loss_scale_state, with dynamic scaling
        self._db_seed, self._db_feed = 0x5EED5EED, False
        self.graph = None

    @property
    def stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    # ---------------------------------------------------------------- views
    def slot_view(self, slot: Slot):
        buf = self.zero if slot.buf == "zero" else self.work
        return buf[slot.offset:slot.offset + slot.size]

    def pview(self, name, buf=None):
        p = self.plan.params.get(name) or self.plan.state[name]
        base = buf if buf is not None else (self.params if p.trainable else self.state)
        return base[p.offset:p.offset + p.size].view(p.store_shape)

    # ---------------------------------------------------------------- weights (TF layout)
    def set_weights(self, tf_vars):
        """tf_vars: name -> array-like in the reference's layout (HWIO kernels, [in,out] dense)."""
        for name, p in list(self.plan.params.items()) + list(self.plan.state.items()):
            v = torch.as_tensor(tf_vars[name]).to(torch.float32)
            if tuple(v.shape) != tuple(p.tf_shape):
                raise ValueError("shape of %s: got %s, expected %s" % (name, tuple(v.shape), p.tf_shape))
            self.set_tf(name, v)

    def set_tf(self, name, value, buf=None):
        """Inverse of get_tf for one variable (or its momentum slot with buf=self.momentum)."""
        p = self.plan.params.get(name) or self.plan.state[name]
        v = torch.as_tensor(value).to(torch.float32)
        dst = self.pview(name, buf)
        if p.kind == "conv_kernel":
            dst.copy_(v.permute(3, 0, 1, 2))
        elif p.kind == "dense_kernel":
            dst.zero_()
            dst[:v.shape[1], 0, 0, :] = v.t()
        elif p.kind == "dense_bias":
            dst.zero_()
            dst[:v.shape[0]] = v
        else:
            dst.copy_(v)

    def get_tf(self, name, buf=None):
        p = self.plan.params.get(name) or self.plan.state[name]
        v = self.pview(name, buf)
        if p.kind == "conv_kernel":
            return v.permute(1, 2, 3, 0)
        if p.kind == "dense_kernel":
            return v[:p.tf_shape[1], 0, 0, :].t()
        if p.kind == "dense_bias":
            return v[:p.tf_shape[0]]
        return v

    def set_hparams(self, lr=None, momentum=None, weight_decay=None, grad_scale=None,
                    keep_prob=None, step=None):
        cur = self.hp.cpu()
        for i, v in enumerate((lr, momentum, weight_decay, grad_scale, keep_prob)):
            if v is not None:
                cur[i] = float(v)
        if step is not None:
            cur.view(torch.int32)[5] = int(step) & 0x7fffffff
        self.hp.copy_(cur, non_blocking=True)

    # settings the launch records read at enqueue time
    @property
    def loss_scale(self):
        return self._loss_scale

    @loss_scale.setter
    def loss_scale(self, v):
        """A number: the static scale (and dynamic scaling off); "dynamic": enable_dynamic_loss_scale() with
        its defaults."""
        if isinstance(v, str):
            if v != "dynamic":
                raise ValueError('loss_scale must be a number or "dynamic" (got %r)' % (v,))
            self.enable_dynamic_loss_scale()
            return
        if self.loss_scale_state_buf is not None:
            _lib.check(self.lib.acnn_set_dynamic_loss_scale(self.model.handle, None, 0.0, 1, 1, self.stream),
                       "acnn_set_dynamic_loss_scale")
            self.loss_scale_state_buf = None
        self._loss_scale = float(v)
        _lib.check(self.lib.acnn_set_loss_scale(self.model.handle, float(v)), "acnn_set_loss_scale")

    def enable_dynamic_loss_scale(self, initial_scale=2.0 ** 15, growth_interval=2000, grad_divisor=1):
        """acnn_set_dynamic_loss_scale: the loss seed, the skip and the gradient scale of every later step come
        from a device state this runtime owns (`loss_scale_state_buf`, initialised on the current stream).
        grad_divisor: world * replicas per device, the replicas the gradient buffer sums."""
        check_dynamic_loss_scale(initial_scale, growth_interval)
        if self.grads is None:
            raise ValueError("dynamic loss scaling needs a training runtime")
        buf = torch.zeros(8, dtype=torch.int32, device=self.dev)
        _lib.check(self.lib.acnn_set_dynamic_loss_scale(self.model.handle, buf.data_ptr(), float(initial_scale),
                                                        int(growth_interval), int(grad_divisor), self.stream),
                   "acnn_set_dynamic_loss_scale")
        self.loss_scale_state_buf = buf
        self._loss_scale = "dynamic"

    def loss_scale_state(self):
        """{scale, good_steps, skipped_steps, last_scale} of the dynamic state: one device read (it waits for
        the work enqueued so far).  None with a static scale."""
        if self.loss_scale_state_buf is None:
            return None
        return decode_loss_scale_state(self.loss_scale_state_buf.cpu())

    def set_loss_scale_state(self, scale, good_steps=0, skipped_steps=0):
        """Overwrite the dynamic state (a resumed run), on the current stream."""
        if self.loss_scale_state_buf is None:
            raise ValueError("set_loss_scale_state: dynamic loss scaling is not enabled")
        scale = float(np.float32(scale))
        check_dynamic_loss_scale(scale, 1)
        v = np.zeros(8, np.int32)
        v[[0, 4]] = np.array([scale, scale], np.float32).view(np.int32)
        v[1], v[2] = int(good_steps), int(skipped_steps)
        self.loss_scale_state_buf.copy_(torch.from_numpy(v))

    def _push_dropblock(self):
        _lib.check(self.lib.acnn_set_dropblock(self.model.handle, self._db_seed & 0xFFFFFFFFFFFFFFFF,
                                               int(self._db_feed)), "acnn_set_dropblock")

    @property
    def dropblock_seed(self):
        return self._db_seed

    @dropblock_seed.setter
    def dropblock_seed(self, v):
        self._db_seed = int(v)
        self._push_dropblock()

    @property
    def dropblock_feed(self):
        """True: the DropBlock masks come from the uniforms in the plan's dropblock_u tensors."""
        return self._db_feed

    @dropblock_feed.setter
    def dropblock_feed(self, v):
        self._db_feed = bool(v)
        self._push_dropblock()

    # ---------------------------------------------------------------- execution
    def run(self, ops):
        """Enqueue ops (any list or slice of the model's NativeOps) in order: consecutive ops of one
        phase become one acnn_run_ops range."""
        h, st, i, n = self.model.handle, self.stream, 0, len(ops)
        while i < n:
            j = i
            while j + 1 < n and ops[j + 1].phase == ops[i].phase and ops[j + 1].index == ops[j].index + 1:
                j += 1
            _lib.check(self.lib.acnn_run_ops(h, ops[i].phase, ops[i].index, ops[j].index + 1, st),
                       "acnn_run_ops(%s)" % ops[i].kind)
            i = j + 1

    def set_images_u8(self, images_u8, mean):
        """acnn_set_images_u8: the "images" buffer = (float)images_u8 - mean[c], images_u8 a CUDA uint8
        tensor [input_batch, H, W, 3] on this device, mean a float32 tensor of 3 (host or device)."""
        _check_u8_images(images_u8, self.t[self.plan.meta["images"]], mean)
        _lib.check(self.lib.acnn_set_images_u8(self.model.handle, images_u8.data_ptr(), mean.data_ptr(),
                                               self.stream), "acnn_set_images_u8")

    def set_images_resized(self, desc, n_valid, mean):
        """acnn_set_images_resized: the "images" buffer from decoded uint8 images of any sizes (resize,
        central crop, - mean[c]); desc a CUDA uint8 tensor of input_batch 32-byte acnn_resize_desc on
        this device, validated by the caller; mean a float32 tensor of 3 (host or device)."""
        _check_desc_args("set_images_resized", desc, self.t[self.plan.meta["images"]], mean, n_valid)
        _lib.check(self.lib.acnn_set_images_resized(self.model.handle, desc.data_ptr(), int(n_valid),
                                                    mean.data_ptr(), self.stream), "acnn_set_images_resized")

    def set_images_cropped(self, desc, mean):
        """acnn_set_images_cropped: every row of the "images" buffer from training crop windows (flip,
        resize to S x S, - mean[c]); desc a CUDA uint8 tensor of input_batch 32-byte acnn_crop_desc on this
        device, validated by the caller; mean a float32 tensor of 3 (host or device)."""
        _check_desc_args("set_images_cropped", desc, self.t[self.plan.meta["images"]], mean)
        _lib.check(self.lib.acnn_set_images_cropped(self.model.handle, desc.data_ptr(), mean.data_ptr(),
                                                    self.stream), "acnn_set_images_cropped")

    def set_images_augmented(self, desc, aug, work, mean):
        """acnn_set_images_augmented: set_images_cropped with AutoAugment (the resized image truncated to
        uint8, aug's two operations, - mean[c]); aug a CUDA uint8 tensor of input_batch 88-byte
        acnn_autoaugment_desc (autoaugment.AUTOAUG_DESC_DTYPE), validated by the caller; work a CUDA uint8
        tensor of acnn_autoaugment_work_bytes(input_batch, S) bytes."""
        _check_augment_args(desc, aug, work, self.t[self.plan.meta["images"]], mean)
        _lib.check(self.lib.acnn_set_images_augmented(self.model.handle, desc.data_ptr(), aug.data_ptr(),
                                                      work.data_ptr(), mean.data_ptr(), self.stream),
                   "acnn_set_images_augmented")

    def zero_step_buffers(self):
        _lib.check(self.lib.acnn_clear_step_buffers(self.model.handle, self.stream),
                   "acnn_clear_step_buffers")

    def run_forward(self):
        h, st = self.model.handle, self.stream
        _lib.check(self.lib.acnn_forward(h, st), "acnn_forward")
        if self.model.sizes.n_loss_first < self.model.sizes.n_forward:
            _lib.check(self.lib.acnn_loss(h, st), "acnn_loss")

    def run_update(self):
        """acnn_sgd_step: the update phase (with dynamic loss scaling also its check and scale update)."""
        _lib.check(self.lib.acnn_sgd_step(self.model.handle, self.stream), "acnn_sgd_step")

    def run_step(self):
        """zero -> forward -> backward -> SGD, all enqueued on the current stream."""
        _lib.check(self.lib.acnn_step(self.model.handle, self.stream), "acnn_step")

    def capture(self, train=True):
        """Capture one full step (or forward) into a CUDA graph; inputs are read from the static
        input buffers (plan.meta['images'] ...), hyper-parameters from the device `hp` vector."""
        fn = self.run_step if train else self.run_forward
        s = torch.cuda.Stream(self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=s):
                fn()
        torch.cuda.current_stream(self.dev).wait_stream(s)
        return self.graph

    # ---------------------------------------------------------------- several replicas per device
    def replica_buffers(self):
        """The device accumulators of several replicas per device: (acc_grads [param_elems], state_base
        [state_elems], acc_state [state_elems + REPLICA_LOSS_FLOATS], the tail summing the loss)."""
        f32 = dict(dtype=torch.float32, device=self.dev)
        ns = self.plan.state_elems
        return (torch.zeros(self.plan.param_elems, **f32), torch.zeros(max(ns, 1), **f32),
                torch.zeros(ns + self.REPLICA_LOSS_FLOATS, **f32))

    def replica_accumulate(self, phase, bufs, lo, hi, replicas):
        """acnn_replica_accumulate_model over this handle's grads [lo, hi), state and loss."""
        acc_g, base, acc_s = bufs
        _lib.check(self.lib.acnn_replica_accumulate_model(self.model.handle, phase, acc_g.data_ptr(), base.data_ptr(),
                                                          acc_s.data_ptr(), lo, hi, replicas, self.stream),
                   "acnn_replica_accumulate_model")
