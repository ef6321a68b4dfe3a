"""Executes a layer plan on one H100 through the C ABI (libacnn.so).

PyTorch is used only as the device-memory container (`torch.empty(..., device='cuda')`,
`data_ptr()`), for streams and for CUDA-graph capture; every kernel on the path is ours.  There is
no CPU path: constructing a Runtime without a CUDA device or without the built library raises.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .plan import Plan, Geom, Slot

_TORCH_DTYPE = {"bf16": torch.bfloat16, "f32": torch.float32, "i32": torch.int32}


def _check_u8_images(images_u8, images, mean):
    """Arguments of set_images_u8: uint8 NHWC of the input buffer's shape on its device, float32 mean[3]."""
    if images_u8.dtype != torch.uint8 or tuple(images_u8.shape) != tuple(images.shape) \
            or images_u8.device != images.device or not images_u8.is_contiguous():
        raise ValueError("images_u8 must be a contiguous uint8 tensor %s on %s, got %s %s on %s"
                         % (tuple(images.shape), images.device, images_u8.dtype, tuple(images_u8.shape),
                            images_u8.device))
    if mean.dtype != torch.float32 or mean.numel() != 3 or not mean.is_contiguous():
        raise ValueError("mean must be a contiguous float32 tensor of 3 values")


def _check_resize_args(desc, images, n_valid, mean):
    """Arguments of set_images_resized: a square input buffer, B descriptors of 32 bytes on its device,
    n_valid in [0, B], float32 mean[3].  Returns (B, S)."""
    b, h, w, _ = images.shape
    if h != w:
        raise ValueError("set_images_resized needs a square input buffer, got %dx%d" % (h, w))
    if desc.dtype != torch.uint8 or desc.numel() != 32 * b or desc.device != images.device \
            or not desc.is_contiguous():
        raise ValueError("desc must be a contiguous uint8 tensor of %d descriptors (%d bytes) on %s"
                         % (b, 32 * b, images.device))
    if not 0 <= int(n_valid) <= b:
        raise ValueError("n_valid=%d outside [0, %d]" % (int(n_valid), b))
    if mean.dtype != torch.float32 or mean.numel() != 3 or not mean.is_contiguous():
        raise ValueError("mean must be a contiguous float32 tensor of 3 values")
    return b, h


def _check_crop_args(desc, images, mean):
    """Arguments of set_images_cropped: a square input buffer, B descriptors of 32 bytes on its device,
    float32 mean[3].  Returns (B, S)."""
    b, h, w, _ = images.shape
    if h != w:
        raise ValueError("set_images_cropped needs a square input buffer, got %dx%d" % (h, w))
    if desc.dtype != torch.uint8 or desc.numel() != 32 * b or desc.device != images.device \
            or not desc.is_contiguous():
        raise ValueError("desc must be a contiguous uint8 tensor of %d descriptors (%d bytes) on %s"
                         % (b, 32 * b, images.device))
    if mean.dtype != torch.float32 or mean.numel() != 3 or not mean.is_contiguous():
        raise ValueError("mean must be a contiguous float32 tensor of 3 values")
    return b, h


class Runtime:
    def __init__(self, plan: Plan, device="cuda:0", eps: float = 1e-5, share: "Runtime | None" = None,
                 deterministic: "bool | None" = None):
        if not torch.cuda.is_available():
            raise _lib.AcnnError("assembled_cnn_b200.Runtime needs a CUDA device (sm_90a); "
                                 "there is no CPU fallback")
        self.lib = _lib.load()
        self.plan = plan
        self.dev = torch.device(device)
        torch.cuda.set_device(self.dev)
        self.eps = eps
        self.bn_momentum = plan.meta.get("bn_momentum", 0.997)
        self.training = plan.meta["training"]
        # fp32 plan = parity mode: fp32 activations, 3-plane GEMM operands, deterministic reductions
        self.fp32 = plan.meta.get("dtype", "bf16") == "fp32"
        self.adt = 1 if self.fp32 else 0               # ACNN_F32 / ACNN_BF16
        self.planes = 3 if self.fp32 else 1
        # deterministic: also the split-K of wgrad and of the small SK / SE GEMMs is disabled (one add
        # per output element).  Every reduction is ordered in both modes (split-K partials are summed
        # in split order), so two runs are bit-identical either way.
        self.det = int(self.fp32 if deterministic is None else bool(deterministic))
        f32 = dict(dtype=torch.float32, device=self.dev)
        if share is not None:
            # same model, another batch shape / mode: the variables are shared, not copied
            if share.plan.param_elems != plan.param_elems or share.plan.state_elems != plan.state_elems \
                    or share.fp32 != self.fp32:
                raise ValueError("Runtime(share=...): parameter layouts differ")
            self.params, self.state, self.w_fprop = share.params, share.state, share.w_fprop
        else:
            self.params = torch.zeros(plan.param_elems, **f32)
            self.state = torch.zeros(max(plan.state_elems, 1), **f32)
            self.w_fprop = torch.zeros(self.planes * plan.param_elems, dtype=torch.bfloat16,
                                       device=self.dev)
        self.zero = torch.zeros(max(plan.zero_elems, 1), **f32)
        self.work = torch.zeros(max(plan.work_elems, 1), **f32)
        if self.training:
            self.grads = torch.zeros(plan.param_elems, **f32)
            if share is not None and share.momentum is not None:
                self.momentum = share.momentum
            else:
                self.momentum = torch.zeros(plan.param_elems, **f32)
            self.w_dgrad = torch.zeros(self.planes * max(plan.dgrad_elems, 1), dtype=torch.bfloat16,
                                       device=self.dev)
        else:
            self.grads = self.momentum = self.w_dgrad = None
        # device hyper-parameters: lr, momentum, wd, grad_scale, dropblock keep_prob, global step
        # (uint32 bits, the Philox counter of the DropBlock masks), 2 spare
        self.hp = torch.tensor([0.1, 0.9, 0.0, 1.0, 1.0, 0.0, 0.0, 0.0], **f32)
        self.loss_scale = 1.0
        self.dropblock_seed = 0x5EED5EED
        self.dropblock_feed = False     # True: masks from the uniforms in plan.meta['dropblock_u']
        if share is None:
            for p in plan.state.values():
                if p.kind == "moving_variance":
                    self.state[p.offset:p.offset + p.size] = 1.0
        for off, C_ in plan.meta.get("ones", []):        # identity-BN scale vectors (DropBlock tails)
            self.work[off:off + C_] = 1.0
        # activation / gradient buffers (statically shaped, allocated once)
        self.t = {}
        for name, t in plan.tensors.items():
            self.t[name] = torch.zeros(t.shape, dtype=_TORCH_DTYPE[t.dtype], device=self.dev)
        # conv weight descriptor table + weight-decay flags
        descs = []
        flags = torch.zeros(max(plan.param_elems // 256, 1), dtype=torch.uint8)
        for p in plan.params.values():
            if p.decay:
                flags[p.offset // 256:(p.offset + p.size + 255) // 256] = 1
            if p.kind in ("conv_kernel", "dense_kernel") and len(p.store_shape) == 4 \
                    and p.store_shape[3] % 16 == 0 and p.store_shape[0] % 32 == 0:
                co, kh, kw, ci = p.store_shape
                descs.append(_lib.WeightDesc(p.offset, p.offset, p.dgrad_off, co, kh * kw, ci, 0))
        self.decay_flags = flags.to(self.dev)
        self.n_descs = len(descs)
        raw = bytes((_lib.WeightDesc * len(descs))(*descs)) if descs else b"\0" * 40
        self.descs = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.dev)
        self.graph = None
        self._side_stream = None
        self._geom_cache = {}
        self._parts_cache = {}

    # ---------------------------------------------------------------- pointers
    @property
    def stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def P(self, name, buf=None):
        p = self.plan.params.get(name) or self.plan.state[name]
        base = buf if buf is not None else (self.params if p.trainable else self.state)
        return base.data_ptr() + 4 * p.offset

    def G(self, name):
        return self.grads.data_ptr() + 4 * self.plan.params[name].offset

    def WF(self, name):
        return self.w_fprop.data_ptr() + 2 * self.plan.params[name].offset

    def WD(self, name):
        p = self.plan.params[name]
        assert p.dgrad_off >= 0, name
        return self.w_dgrad.data_ptr() + 2 * p.dgrad_off

    def S(self, slot: Slot | None, extra=0):
        if slot is None:
            return None
        buf = self.zero if slot.buf == "zero" else self.work
        return buf.data_ptr() + 4 * (slot.offset + extra)

    def T(self, name):
        return None if name is None else self.t[name].data_ptr()

    def geom(self, g: Geom, x_wpad=None):
        """ConvGeom for the C ABI.  With x_wpad=(lo, hi) the input is the W-padded space-to-depth
        image: the k2 horizontal taps become channels of one wide pixel (x_pix_stride < Cin)."""
        key = g.astuple() + (x_wpad,)
        cg = self._geom_cache.get(key)
        if cg is None:
            if x_wpad is None:
                cg = _lib.ConvGeom(*g.astuple())
            else:
                lo, hi = x_wpad
                assert g.stride == 1 and g.pad_w_lo == lo and g.pad_w_hi == hi
                row = (g.W + lo + hi) * g.Cin
                cg = _lib.ConvGeom(g.B, g.H, g.W, g.Cin * g.kw, g.Cout, g.kh, 1, 1,
                                   g.pad_h_lo, g.pad_h_hi, 0, 0, g.Cin, row, g.H * row, 0)
            self._geom_cache[key] = cg
        return cg

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
            dst = self.pview(name)
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

    # ---------------------------------------------------------------- execution
    def _chk(self, rc, op):
        if rc != 0:
            _lib.check(rc, "op %s" % op.kind)

    _SIDE_KINDS = ("conv_wgrad", "s2d_wgrad_unpack")

    def run(self, ops, overlap_wgrad=False):
        """Enqueue ops in order.  With overlap_wgrad the weight-gradient GEMMs (needed only by
        the SGD step) go to a second stream: they depend on dy alone, so the tensor-core-bound
        wgrads run concurrently with the HBM-bound batch-norm / pooling kernels of the dgrad
        chain.  Works identically under CUDA-graph capture (fork / join through events)."""
        if not overlap_wgrad:
            for op in ops:
                getattr(self, "op_" + op.kind)(op)
            return
        main = torch.cuda.current_stream(self.dev)
        if self._side_stream is None:
            self._side_stream = torch.cuda.Stream(self.dev)
        side = self._side_stream
        forked = False
        for op in ops:
            if op.kind in self._SIDE_KINDS:
                ev = torch.cuda.Event()
                ev.record(main)                      # dy (and everything before it) is ready
                side.wait_event(ev)
                forked = True
                with torch.cuda.stream(side):
                    getattr(self, "op_" + op.kind)(op)
            else:
                getattr(self, "op_" + op.kind)(op)
        if forked:
            main.wait_stream(side)                   # join before the optimizer

    def set_images_u8(self, images_u8, mean):
        """The "images" buffer = (float)images_u8 - mean[c] (acnn_images_from_u8), images_u8 a CUDA uint8
        tensor [input_batch, H, W, 3] on this device, mean a float32 tensor of 3 (host or device)."""
        images = self.t[self.plan.meta["images"]]
        _check_u8_images(images_u8, images, mean)
        b, h, w, _ = images.shape
        _lib.check(self.lib.acnn_images_from_u8(images_u8.data_ptr(), mean.data_ptr(), images.data_ptr(), b, h, w,
                                                self.stream), "acnn_images_from_u8")

    def set_images_resized(self, desc, n_valid, mean):
        """The "images" buffer [B, S, S, 3] from decoded uint8 images of any sizes (acnn_resize_crop_u8:
        resize, central crop, - mean[c]).  desc: a CUDA uint8 tensor of B 32-byte acnn_resize_desc
        (imagenet_eval.DESC_DTYPE) on this device, validated by the caller; rows >= n_valid are not
        written; mean a float32 tensor of 3 (host or device)."""
        images = self.t[self.plan.meta["images"]]
        b, s = _check_resize_args(desc, images, n_valid, mean)
        _lib.check(self.lib.acnn_resize_crop_u8(desc.data_ptr(), b, int(n_valid), s, mean.data_ptr(),
                                                images.data_ptr(), self.stream), "acnn_resize_crop_u8")

    def set_images_cropped(self, desc, mean):
        """Every row of the "images" buffer [B, S, S, 3] from training crop windows (acnn_crop_resize_u8:
        flip, resize to S x S, - mean[c]).  desc: a CUDA uint8 tensor of B 32-byte acnn_crop_desc
        (imagenet_train.CROP_DESC_DTYPE) on this device, validated by the caller; mean a float32 tensor
        of 3 (host or device)."""
        images = self.t[self.plan.meta["images"]]
        b, s = _check_crop_args(desc, images, mean)
        _lib.check(self.lib.acnn_crop_resize_u8(desc.data_ptr(), b, b, s, mean.data_ptr(), images.data_ptr(),
                                                self.stream), "acnn_crop_resize_u8")

    def zero_step_buffers(self):
        st = self.stream
        self.lib.acnn_fill_zero(self.zero.data_ptr(), self.zero.numel() * 4, st)
        if self.grads is not None:
            self.lib.acnn_fill_zero(self.grads.data_ptr(), self.grads.numel() * 4, st)

    def run_forward(self):
        self.zero_step_buffers()
        self.run(self.plan.forward)

    def run_step(self):
        """zero -> forward -> backward -> SGD, all enqueued on the current stream."""
        self.run_forward()
        self.run(self.plan.backward)
        self.run(self.plan.update)

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

    # ---------------------------------------------------------------- forward ops
    def op_prep_weights(self, op):
        if self.n_descs:
            self._chk(self.lib.acnn_prep_weights(
                self.params.data_ptr(), self.descs.data_ptr(), self.n_descs,
                self.w_fprop.data_ptr(),
                self.w_dgrad.data_ptr() if self.w_dgrad is not None else None, self.planes,
                self.plan.param_elems, max(self.plan.dgrad_elems, 1), self.stream), op)

    def op_split3(self, op):
        self._chk(self.lib.acnn_split3(self.T(op.src), self.T(op.dst), op.n, self.stream), op)

    def op_pack_input(self, op):
        self._chk(self.lib.acnn_pack_input(self.T(op.images), self.T(op.lam1), self.T(op.lam2),
                                           op.mode, self.T(op.out), op.Bin, op.H, op.W,
                                           op.wpad[0], op.wpad[1], self.adt, self.stream), op)

    def op_mix_labels(self, op):
        self._chk(self.lib.acnn_mix_labels(self.T(op.labels), self.T(op.lam1), self.T(op.lam2),
                                           op.mode, self.T(op.y), op.Bin, op.NC, self.stream), op)

    def op_s2d_weight_pack(self, op):
        self._chk(self.lib.acnn_s2d_weight_pack(self.P(op.w), self.T(op.w2), op.cout, op.k, op.pad,
                                                op.k2, op.pad2, self.adt, self.stream), op)

    def stats_parts(self, geom, x_wpad=None):
        """Rows of the partial-statistics buffer the conv of this geometry writes."""
        key = ("conv", geom.astuple(), x_wpad)
        n = self._parts_cache.get(key)
        if n is None:
            n = self.lib.acnn_conv_stats_parts(self.geom(geom, x_wpad))
            if n < 1:
                raise _lib.AcnnError("acnn_conv_stats_parts failed for %r" % (geom,))
            self._parts_cache[key] = n
        return n

    def op_conv(self, op):
        is_t = op.a.get("w_is_tensor")
        if self.fp32:
            x = self.T(op.xp)
            w = self.T(op.wp) if is_t else self.WF(op.w)
            wstride = self.t[op.wp].numel() // 3 if is_t else self.plan.param_elems
        else:
            x = self.T(op.x)
            w = self.T(op.w) if is_t else self.WF(op.w)
            wstride = 0
        st = op.stats
        if st is not None:
            n = self.stats_parts(op.geom, op.a.get("x_wpad"))
            assert n * 2 * op.geom.Cout <= st.size, (n, st.size)
        self._chk(self.lib.acnn_conv_fprop(
            self.geom(op.geom, op.a.get("x_wpad")), x, w, self.T(op.y), self.S(st),
            None, None, self.P(op.bias) if op.bias else None,
            1 if (op.out_f32 or self.fp32) else 0, self.adt, wstride, self.stream), op)

    def op_bn_stats(self, op):
        bn = op.bn
        self._chk(self.lib.acnn_bn_stats(self.T(op.x), self.S(bn.stats), op.M, op.C, self.adt,
                                         self.stream), op)

    def op_bn_finalize(self, op):
        bn = op.bn
        C_ = bn.C
        mode = op.a.get("stats_mode", 0)
        nparts = 1
        if self.training and mode == 0:
            nparts = self.stats_parts(op.geom, op.a.get("x_wpad"))
        self._chk(self.lib.acnn_bn_finalize(
            self.S(bn.stats), nparts, mode, bn.count, self.P(bn.gamma),
            self.P(bn.beta), self.P(bn.mm), self.P(bn.mv), self.bn_momentum, self.eps,
            1 if self.training else 0, self.S(bn.work), self.S(bn.work, C_), self.S(bn.work, 2 * C_),
            self.S(bn.work, 3 * C_), C_, self.stream), op)

    def op_bn_act(self, op):
        B, H, W, C_ = op.shape
        bna, bnb = op.bn_a, op.bn_b
        self._chk(self.lib.acnn_bn_act(
            self.T(op.a["a"]), self.S(bna.work), self.S(bna.work, C_), self.T(op.b),
            self.S(bnb.work) if bnb else None, self.S(bnb.work, C_) if bnb else None, op.b_mode,
            self.S(op.gate), 1 if op.relu else 0, self.T(op.out), B, H, W, C_, self.adt,
            self.stream), op)

    def op_sk_gap(self, op):
        bn = op.bn
        self._chk(self.lib.acnn_sk_gap(self.T(op.y), self.S(bn.work), self.S(bn.work, bn.C),
                                       self.S(op.s), op.B, op.HW, op.f, self.adt, self.stream), op)

    def op_sk_fc(self, op):
        bn = op.bn
        assert op.scratch.size >= self.lib.acnn_sk_fc_scratch_floats(op.B, op.f, op.d)
        self._chk(self.lib.acnn_sk_fc_fwd(
            self.S(op.s), self.P(op.w1), self.P(bn.gamma), self.P(bn.beta), self.P(bn.mm),
            self.P(bn.mv), self.bn_momentum, self.eps, 1 if self.training else 0, self.P(op.w2),
            self.S(op.zpre), self.S(bn.work), self.S(op.z), self.S(op.att), self.S(op.scratch),
            op.B, op.f, op.d, self.det, self.stream), op)

    def op_sk_combine(self, op):
        bn = op.bn
        self._chk(self.lib.acnn_sk_combine(self.T(op.y), self.S(bn.work), self.S(bn.work, bn.C),
                                           self.S(op.att), self.T(op.v), op.B, op.HW, op.f,
                                           self.adt, self.stream), op)

    def op_se_gap(self, op):
        bn = op.bn
        self._chk(self.lib.acnn_se_gap(self.T(op.y), self.S(bn.work), self.S(bn.work, bn.C),
                                       self.S(op.q), op.B, op.HW, op.C, self.adt, self.stream), op)

    def op_se_fc(self, op):
        self._chk(self.lib.acnn_se_fc_fwd(self.S(op.q), self.P(op.w1), self.P(op.w2), self.S(op.h),
                                          self.S(op.e), op.B, op.C, op.r, self.det, self.stream), op)

    def op_blurpool(self, op):
        self._chk(self.lib.acnn_blurpool_fwd(self.T(op.x), self.T(op.out), op.B, op.H, op.W, op.C,
                                             op.filt, op.stride, self.adt, self.stream), op)

    def op_avgpool(self, op):
        self._chk(self.lib.acnn_avgpool_fwd(self.T(op.x), self.T(op.out), op.B, op.H, op.W, op.C,
                                            op.k, op.stride, op.pad_lo, op.Ho, op.Wo, op.count_pad,
                                            self.adt, self.stream), op)

    def op_maxpool(self, op):
        self._chk(self.lib.acnn_maxpool_fwd(self.T(op.x), self.T(op.out), op.B, op.H, op.W, op.C,
                                            op.k, op.stride, op.pad_lo, op.Ho, op.Wo, self.adt,
                                            self.stream), op)

    def op_gem(self, op):
        self._chk(self.lib.acnn_gem_fwd(self.T(op.x), self.T(op.out), self.S(op.ssum), op.B, op.HW,
                                        op.C, self.adt, self.stream), op)

    def op_gem_bwd(self, op):
        self._chk(self.lib.acnn_gem_bwd(self.T(op.dpooled), self.S(op.ssum), self.T(op.x),
                                        self.T(op.dx), op.B, op.HW, op.C, self.adt, self.stream), op)

    def op_dropblock_mask(self, op):
        need = self.lib.acnn_dropblock_scratch_floats(op.H, op.W, op.C, op.block_size)
        assert 0 < need <= op.scratch.size, (need, op.scratch.size)
        u = self.T(op.u) if self.dropblock_feed else None
        # one Philox key per call site: the masks of different layers are independent
        seed = (self.dropblock_seed + 0x9E3779B97F4A7C15 * (op.index + 1)) & 0xFFFFFFFFFFFFFFFF
        self._chk(self.lib.acnn_dropblock_mask(
            u, self.hp.data_ptr() + 16, self.hp.data_ptr() + 20, seed, op.gamma_scale,
            op.block_size, self.S(op.keep), self.S(op.scale), self.S(op.scratch), op.H, op.W, op.C,
            self.stream), op)

    def op_dropblock_apply(self, op):
        self._chk(self.lib.acnn_dropblock_apply(self.T(op.x), self.S(op.keep), self.S(op.scale),
                                                1 if op.relu else 0, self.T(op.out), op.B, op.HW,
                                                op.C, self.adt, self.stream), op)

    def op_kd_teacher(self, op):
        self._chk(self.lib.acnn_kd_teacher_labels(
            self.T(op.teacher_logits), self.T(op.labels), self.T(op.lam1), self.T(op.lam2), op.mode,
            op.kd_temp, self.T(op.yt), op.Bin, op.NC, self.stream), op)

    def op_gap(self, op):
        self._chk(self.lib.acnn_gap_fwd(self.T(op.x), self.T(op.out), op.B, op.HW, op.C,
                                        self.adt, self.stream), op)

    def op_softmax_ce(self, op):
        self._chk(self.lib.acnn_softmax_ce(
            self.T(op.logits), self.T(op.y), self.T(op.a.get("yt")), float(op.a.get("kd_temp", 0.0)),
            op.B, op.NC, op.ld, op.label_smoothing,
            self.loss_scale, self.S(op.loss), self.T(op.dlogits),
            self.G(op.dbias) if (op.dbias and self.grads is not None) else None, self.S(op.work),
            self.adt, self.stream), op)

    # ---------------------------------------------------------------- backward ops
    def op_conv_wgrad(self, op):
        slot = op.a.get("dw_slot")
        dw = self.S(slot) if slot is not None else self.G(op.w)
        x, dy = (self.T(op.xp), self.T(op.dyp)) if self.fp32 else (self.T(op.x), self.T(op.dy))
        self._chk(self.lib.acnn_conv_wgrad(self.geom(op.geom, op.a.get("x_wpad")), x, dy, dw,
                                           self.adt, self.det, self.stream), op)

    def op_conv_dgrad(self, op):
        dy = self.T(op.dyp) if self.fp32 else self.T(op.dy)
        self._chk(self.lib.acnn_conv_dgrad(self.geom(op.geom), dy, self.WD(op.w),
                                           self.T(op.dx), self.T(op.add_src), self.T(op.mask_src),
                                           self.adt, max(self.plan.dgrad_elems, 1), self.stream), op)

    def op_zero_insert(self, op):
        self._chk(self.lib.acnn_zero_insert2x(self.T(op.dy), self.T(op.out), op.B, op.Ho, op.Wo,
                                              op.H, op.W, op.C, self.adt, self.stream), op)

    def op_s2d_wgrad_unpack(self, op):
        self._chk(self.lib.acnn_s2d_wgrad_unpack(self.S(op.dw2), self.G(op.w), op.cout, op.k,
                                                 op.pad, op.k2, op.pad2, self.stream), op)

    def op_bn_bwd_reduce(self, op):
        B, H, W, C_ = op.shape
        bn = op.bn
        n = self.lib.acnn_bn_bwd_reduce_parts(B, H * W, C_)
        assert 1 <= n and n * 2 * C_ <= op.sums.size, (n, C_, op.sums.size)
        self._parts_cache[("bwd", op.sums.buf, op.sums.offset)] = n
        self._chk(self.lib.acnn_bn_bwd_reduce(
            self.T(op.g), self.T(op.y), self.S(bn.work, 2 * C_), self.S(bn.work, 3 * C_),
            self.S(op.gate), self.S(op.addbc), self.S(op.sums), B, H * W, C_, self.adt,
            self.stream), op)

    def op_bn_bwd_finalize(self, op):
        bn = op.bn
        C_ = bn.C
        n = self._parts_cache[("bwd", op.sums.buf, op.sums.offset)]
        self._chk(self.lib.acnn_bn_bwd_finalize(
            self.S(op.sums), n, self.P(bn.gamma), self.S(bn.work, 2 * C_), self.S(bn.work, 3 * C_),
            bn.count, self.S(op.coef), self.G(bn.gamma), self.G(bn.beta), C_, self.stream), op)

    def op_bn_bwd_apply(self, op):
        B, H, W, C_ = op.shape
        self._chk(self.lib.acnn_bn_bwd_apply(self.T(op.g), self.T(op.y), self.S(op.coef),
                                             self.S(op.gate), self.S(op.addbc), self.T(op.dy), B,
                                             H * W, C_, self.adt, self.stream), op)

    def op_bn_bwd_reduce2(self, op):
        B, H, W, C_ = op.shape
        bn, bn2 = op.bn, op.bn2
        n = self.lib.acnn_bn_bwd_reduce_parts(B, H * W, C_)
        assert 1 <= n and n * 2 * C_ <= op.sums.size and n * 2 * C_ <= op.sums2.size
        self._parts_cache[("bwd", op.sums.buf, op.sums.offset)] = n
        self._parts_cache[("bwd", op.sums2.buf, op.sums2.offset)] = n
        self._chk(self.lib.acnn_bn_bwd_reduce2(
            self.T(op.g), self.T(op.y), self.T(op.y2), self.S(bn.work, 2 * C_),
            self.S(bn.work, 3 * C_), self.S(bn2.work, 2 * C_), self.S(bn2.work, 3 * C_),
            self.S(op.sums), self.S(op.sums2), B, H * W, C_, self.adt, self.stream), op)

    def op_bn_bwd_apply2(self, op):
        B, H, W, C_ = op.shape
        self._chk(self.lib.acnn_bn_bwd_apply2(
            self.T(op.g), self.T(op.y), self.T(op.y2), self.S(op.coef), self.S(op.coef2),
            self.T(op.dy), self.T(op.dy2), B, H * W, C_, self.adt, self.stream), op)

    def op_sk_bwd_gate(self, op):
        bn = op.bn
        self._chk(self.lib.acnn_sk_bwd_gate(self.T(op.dv), self.T(op.y), self.S(bn.work),
                                            self.S(bn.work, bn.C), self.S(op.dA), op.B, op.HW,
                                            op.f, self.adt, self.stream), op)

    def op_sk_fc_bwd(self, op):
        bn = op.bn
        self._chk(self.lib.acnn_sk_fc_bwd(
            self.S(op.dA), self.S(op.att), self.S(op.z), self.S(op.zpre), self.S(bn.work),
            self.P(bn.gamma), self.S(op.s), self.P(op.w1), self.P(op.w2), self.G(op.w1),
            self.G(op.w2), self.G(bn.gamma), self.G(bn.beta), self.S(op.ds), self.S(op.scratch),
            op.B, op.f, op.d, self.det, self.stream), op)

    def op_sk_bn_bwd_reduce(self, op):
        bn = op.bn
        C_ = bn.C
        n = self.lib.acnn_sk_bn_bwd_reduce_parts(op.B, op.HW, op.f)
        assert 1 <= n and n * 2 * C_ <= op.sums.size, (n, C_, op.sums.size)
        self._parts_cache[("bwd", op.sums.buf, op.sums.offset)] = n
        self._chk(self.lib.acnn_sk_bn_bwd_reduce(
            self.T(op.dv), self.T(op.y), self.S(bn.work), self.S(bn.work, C_),
            self.S(bn.work, 2 * C_), self.S(bn.work, 3 * C_), self.S(op.att), self.S(op.ds),
            self.S(op.sums), op.B, op.HW, op.f, self.adt, self.stream), op)

    def op_sk_bn_bwd_apply(self, op):
        bn = op.bn
        self._chk(self.lib.acnn_sk_bn_bwd_apply(
            self.T(op.dv), self.T(op.y), self.S(bn.work), self.S(bn.work, bn.C), self.S(op.att),
            self.S(op.ds), self.S(op.coef), self.T(op.dy), op.B, op.HW, op.f, self.adt,
            self.stream), op)

    def op_se_bwd_gate(self, op):
        bn = op.bn
        self._chk(self.lib.acnn_se_bwd_gate(self.T(op.g), self.T(op.y), self.S(bn.work),
                                            self.S(bn.work, bn.C), self.S(op.de), op.B, op.HW,
                                            op.C, self.adt, self.stream), op)

    def op_se_fc_bwd(self, op):
        self._chk(self.lib.acnn_se_fc_bwd(
            self.S(op.de), self.S(op.e), self.S(op.h), self.S(op.q), self.P(op.w1), self.P(op.w2),
            self.G(op.w1), self.G(op.w2), self.S(op.dq), self.S(op.scratch), op.B, op.C, op.r,
            op.HW, self.det, self.stream), op)

    def op_blurpool_bwd(self, op):
        self._chk(self.lib.acnn_blurpool_bwd(self.T(op.dout), self.T(op.dx), self.T(op.add_src),
                                             self.T(op.mask_src), op.B, op.H, op.W, op.C, op.filt,
                                             op.stride, self.adt, self.stream), op)

    def op_avgpool_bwd(self, op):
        self._chk(self.lib.acnn_avgpool_bwd(self.T(op.dout), self.T(op.dx), self.T(op.add_src),
                                            self.T(op.mask_src), op.B, op.H, op.W, op.C, op.k,
                                            op.stride, op.pad_lo, op.Ho, op.Wo, op.count_pad,
                                            self.adt, self.stream), op)

    def op_maxpool_bwd(self, op):
        self._chk(self.lib.acnn_maxpool_bwd(self.T(op.dout), self.T(op.x), self.T(op.dx),
                                            self.T(op.add_src), self.T(op.mask_src), op.B, op.H,
                                            op.W, op.C, op.k, op.stride, op.pad_lo, op.Ho, op.Wo,
                                            self.adt, self.stream), op)

    def op_upsample2x_bwd(self, op):
        self._chk(self.lib.acnn_upsample2x_bwd(self.T(op.dout), self.T(op.dx), self.T(op.add_src),
                                               self.T(op.mask_src), op.B, op.H, op.W, op.C,
                                               self.adt, self.stream), op)

    def op_gap_bwd(self, op):
        self._chk(self.lib.acnn_gap_bwd(self.T(op.dpooled), self.T(op.mask_src), self.T(op.dx),
                                        op.B, op.HW, op.C, self.adt, self.stream), op)

    def op_grad_combine(self, op):
        n = 1
        for s in op.shape:
            n *= s
        self._chk(self.lib.acnn_grad_combine(self.T(op.a["a"]), self.T(op.add_src),
                                             self.T(op.mask_src), self.T(op.out), n, self.adt,
                                             self.stream), op)

    def op_sgd(self, op):
        self._chk(self.lib.acnn_sgd_momentum(
            self.params.data_ptr(), self.grads.data_ptr(), self.momentum.data_ptr(),
            self.plan.param_elems, self.decay_flags.data_ptr(), self.hp.data_ptr(),
            self.S(op.loss, 1), self.S(op.scratch), self.stream), op)
