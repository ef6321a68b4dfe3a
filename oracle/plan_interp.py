"""CPU interpreter of the product's layer plan (assembled_cnn_b200/plan.py) in plain torch.

TEST INFRASTRUCTURE ONLY (see oracle/tf_ops.py header).  It gives every op kind of the plan an
independent reference meaning (explicit backward formulas, written with torch ops,
adjoints taken by autograd where that is the definition), so that

  * on CPU, the whole plan -- topology, gradient accumulation, parameter order -- is checked
    against the autograd oracle (oracle/model.py) without a GPU, and
  * on the GPU box, each CUDA kernel and the whole step are checked against it, optionally with the
    same storage rounding points as the CUDA path (`emulate_storage=True`).

Storage emulation: every stored 16-bit tensor is rounded to its own declared type -- "bf16" to
bfloat16, "f16" to float16 -- and the conv weights (GEMM operands, `wq`) to the plan's element type
(plan.meta["dtype"]), each with round to nearest even and overflow to inf, as torch's .bfloat16() /
.half() do.  fp32 tensors and fp32 plans are never rounded.  `emulate_bf16` is the older name of
`emulate_storage` and means the same (on a bf16 plan every 16-bit tensor is "bf16").
`emulate_storage` may also name one 16-bit type ("bf16" or "f16") that every 16-bit tensor and weight
is rounded to instead of its own: a deliberately wrong emulation, for tests that show the choice of
type is visible.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from . import tf_ops as T


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


_ROUND = {"bf16": torch.bfloat16, "f16": torch.float16}
_ELEMENT_TYPE = {"bf16": "bf16", "fp16": "f16", "fp32": "f32"}


class PlanInterpreter:
    def __init__(self, plan, dtype=torch.float32, emulate_storage=False, eps=1e-5, emulate_bf16=None):
        self.plan = plan
        self.dtype = dtype
        if emulate_bf16 is not None:
            emulate_storage = emulate_storage or emulate_bf16
        if emulate_storage not in (False, True, "bf16", "f16"):
            raise ValueError("emulate_storage must be a bool, 'bf16' or 'f16'")
        self.emu = bool(emulate_storage)
        self.emu_as = emulate_storage if isinstance(emulate_storage, str) else None
        self.adt = _ELEMENT_TYPE[plan.meta.get("dtype", "bf16")]
        self.eps = eps
        self.t = {}                                   # activation tensors by name
        self.params = torch.zeros(plan.param_elems, dtype=dtype)
        self.grads = torch.zeros(plan.param_elems, dtype=dtype)
        self.momentum = torch.zeros(plan.param_elems, dtype=dtype)
        self.state = torch.zeros(plan.state_elems, dtype=dtype)
        self.zero = torch.zeros(max(plan.zero_elems, 1), dtype=dtype)
        self.work = torch.zeros(max(plan.work_elems, 1), dtype=dtype)
        self.hp = dict(lr=0.1, momentum=0.9, weight_decay=0.0, grad_scale=1.0, keep_prob=1.0)
        for p in plan.state.values():
            if p.kind == "moving_variance":
                self.state[p.offset:p.offset + p.size] = 1.0
        for off, C in plan.meta.get("ones", []):          # identity-BN scale vectors
            self.work[off:off + C] = 1.0

    # ---------------------------------------------------------------- parameter access
    def pview(self, name, buf=None):
        p = self.plan.params.get(name) or self.plan.state[name]
        base = buf if buf is not None else (self.params if p.trainable else self.state)
        return base[p.offset:p.offset + p.size].view(p.store_shape)

    def set_weights(self, tf_vars):
        """tf_vars: name -> tensor in TF layout (HWIO kernels, [in,out] dense)."""
        for name, p in list(self.plan.params.items()) + list(self.plan.state.items()):
            v = tf_vars[name].to(self.dtype)
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

    def get_tf(self, name, buf=None):
        """Parameter (or its gradient / momentum with buf=...) back in TF layout."""
        p = self.plan.params.get(name) or self.plan.state[name]
        v = self.pview(name, buf)
        if p.kind == "conv_kernel":
            return v.permute(1, 2, 3, 0)
        if p.kind == "dense_kernel":
            return v[:p.tf_shape[1], 0, 0, :].t()
        if p.kind == "dense_bias":
            return v[:p.tf_shape[0]]
        return v

    def slot(self, s):
        buf = self.zero if s.buf == "zero" else self.work
        return buf[s.offset:s.offset + s.size]

    # ---------------------------------------------------------------- helpers
    def round_to(self, value, tdt):
        """value rounded to the 16-bit storage type tdt ("bf16" / "f16"; anything else: unchanged)."""
        if not self.emu or tdt not in _ROUND:
            return value
        return value.to(_ROUND[self.emu_as or tdt]).to(self.dtype)

    def store(self, name, value):
        t = self.plan.tensors[name]
        value = self.round_to(value.to(self.dtype), t.dtype)
        assert tuple(value.shape) == tuple(t.shape), (name, value.shape, t.shape)
        self.t[name] = value

    def wq(self, w):
        """A conv / dense weight as the GEMM reads it: rounded to the plan's element type."""
        return self.round_to(w, self.adt)

    def _conv(self, x, w_ohwi, g):
        xp = F.pad(_nchw(x), (g.pad_w_lo, g.pad_w_hi, g.pad_h_lo, g.pad_h_hi))
        return _nhwc(F.conv2d(xp, w_ohwi.permute(0, 3, 1, 2), stride=g.stride))

    def bn_scale_shift(self, bn):
        w = self.slot(bn.work)
        C = bn.C
        return w[:C], w[C:2 * C], w[2 * C:3 * C], w[3 * C:4 * C]

    def grad_epilogue(self, v, add_src, mask_src):
        if add_src is not None:
            v = v + self.t[add_src]
        if mask_src is not None:
            v = v * (self.t[mask_src] > 0)
        return v

    # ---------------------------------------------------------------- execution
    def run(self, ops):
        for op in ops:
            getattr(self, "op_" + op.kind)(op)

    def zero_step_buffers(self):
        self.zero.zero_()
        self.grads.zero_()

    def forward(self, images, labels=None, lam1=None, lam2=None):
        m = self.plan.meta
        self.zero_step_buffers()
        self.t[m["images"]] = images.to(self.dtype)
        if labels is not None and "labels" in m:
            self.t[m["labels"]] = labels
        if lam1 is not None:
            self.t[m["lam1"]] = lam1.to(self.dtype)
        if lam2 is not None:
            self.t[m["lam2"]] = lam2.to(self.dtype)
        self.run(self.plan.forward)
        return self.t[m["logits"]][:, :m["num_classes"]]

    def train_step(self, images, labels, lam1=None, lam2=None):
        logits = self.forward(images, labels, lam1, lam2)
        self.run(self.plan.backward)
        self.run(self.plan.update)
        loss = self.slot(self.plan.meta["loss"])
        return logits, loss[0].item(), loss[1].item()

    # ---------------------------------------------------------------- forward ops
    def op_prep_weights(self, op):
        pass                                            # bf16 operand copies: layout only

    def op_split3(self, op):
        pass                                            # fp32 mode operand planes: representation only

    def op_bn_stats(self, op):
        """fp32 mode: two-pass batch statistics [mean | biased variance]."""
        x = self.t[op.x]
        s = self.slot(op.bn.stats)
        C = op.C
        s[:C] = x.mean(dim=(0, 1, 2))
        s[C:2 * C] = x.var(dim=(0, 1, 2), unbiased=False)

    def op_pack_input(self, op):
        x = self.t[op.images]
        if op.mode:
            lam1 = self.t[op.lam1]
            lam2 = self.t[op.lam2] if op.lam2 else None
            x, _ = T.mixup(x, torch.zeros(x.shape[0], 1, dtype=x.dtype), lam1, lam2,
                           keep_batch_size=(op.mode == 2))
        B, H, W, _ = x.shape
        x4 = F.pad(x, (0, 1))                                            # c: 3 -> 4
        x4 = x4.view(B, H // 2, 2, W // 2, 2, 4).permute(0, 1, 3, 2, 4, 5)   # b,i,j,dy,dx,c
        x4 = x4.reshape(B, H // 2, W // 2, 16)
        lo, hi = op.wpad
        self.store(op.out, F.pad(x4, (0, 0, lo, hi)))                    # physical W padding

    def op_mix_labels(self, op):
        lab = self.t[op.labels].long()
        y = F.one_hot(lab, op.NC).to(self.dtype)
        if op.mode:
            lam1 = self.t[op.lam1]
            lam2 = self.t[op.lam2] if op.lam2 else None
            _, y = T.mixup(torch.zeros(y.shape[0], 1, 1, 1, dtype=self.dtype), y, lam1, lam2,
                           keep_batch_size=(op.mode == 2))
        self.store(op.y, y)

    def op_s2d_weight_pack(self, op):
        w = self.pview(op.w)                                             # [Cout][k][k][3]
        k, pad, k2, pad2 = op.k, op.pad, op.k2, op.pad2
        w2 = torch.zeros(op.cout, k2, k2, 16, dtype=self.dtype)
        for r2 in range(k2):
            for a in range(2):
                u = 2 * (r2 - pad2) + a + pad
                if not 0 <= u < k:
                    continue
                for s2 in range(k2):
                    for b in range(2):
                        v = 2 * (s2 - pad2) + b + pad
                        if 0 <= v < k:
                            w2[:, r2, s2, (a * 2 + b) * 4:(a * 2 + b) * 4 + 3] = w[:, u, v, :]
        self.store(op.w2, w2)

    def op_conv(self, op):
        g = op.geom
        x = self.t[op.x]
        w = self.t[op.w] if op.a.get("w_is_tensor") else self.wq(self.pview(op.w))
        if x.dim() == 2:
            x = x[:, None, None, :]
        if op.a.get("x_wpad"):
            lo, hi = op.x_wpad
            x = x[:, :, lo:x.shape[2] - hi, :]
        y = self._conv(x, w, g)
        if op.bias:
            y = y + self.pview(op.bias)
        t = self.plan.tensors[op.y]
        if len(t.shape) == 2:
            y = y[:, 0, 0, :]
        self.store(op.y, y)
        if op.stats is not None:
            ys = self.t[op.y]
            s = self.slot(op.stats)         # row 0 of the [parts][2][C] partial buffer = the total
            C = ys.shape[-1]
            s.zero_()
            s[:C] = ys.sum(dim=(0, 1, 2))
            s[C:2 * C] = (ys * ys).sum(dim=(0, 1, 2))

    def op_bn_finalize(self, op):
        bn = op.bn
        scale, shift, mean_o, rstd_o = self.bn_scale_shift(bn)
        gamma, beta = self.pview(bn.gamma), self.pview(bn.beta)
        mm, mv = self.pview(bn.mm), self.pview(bn.mv)
        if self.plan.meta["training"]:
            s = self.slot(bn.stats)
            n = bn.count
            if op.a.get("stats_mode", 0) == 1:
                mean, var = s[:bn.C].clone(), s[bn.C:2 * bn.C].clone()
            else:
                mean = s[:bn.C] / n
                var = (s[bn.C:2 * bn.C] / n - mean * mean).clamp_min(0)
            mom = self.plan.meta.get("bn_momentum", 0.997)
            mm.copy_(mm * mom + mean * (1 - mom))
            mv.copy_(mv * mom + var * (n / max(n - 1, 1)) * (1 - mom))
        else:
            mean, var = mm.clone(), mv.clone()
        rstd = torch.rsqrt(var + self.eps)
        scale.copy_(gamma * rstd)
        shift.copy_(beta - mean * gamma * rstd)
        mean_o.copy_(mean)
        rstd_o.copy_(rstd)

    def _gate(self, gate_slot, B, C):
        return self.slot(gate_slot).view(B, 1, 1, C)

    def op_bn_act(self, op):
        a = self.t[op.a["a"]]
        sa, ha, _, _ = self.bn_scale_shift(op.bn_a)
        v = a * sa + ha
        B, H, W, C = a.shape
        if op.gate is not None:
            v = v * self._gate(op.gate, B, C)
        if op.b_mode == 1:
            sb, hb, _, _ = self.bn_scale_shift(op.bn_b)
            v = v + self.t[op.b] * sb + hb
        elif op.b_mode == 2:
            v = v + self.t[op.b]
        elif op.b_mode == 3:
            v = v + T.upsample2x(self.t[op.b])
        if op.relu:
            v = torch.relu(v)
        self.store(op.out, v)

    def _sk_u(self, op):
        y = self.t[op.y]
        sc, sh, _, _ = self.bn_scale_shift(op.bn)
        u = torch.relu(y * sc + sh)
        return y, u[..., :op.f], u[..., op.f:]

    def op_sk_gap(self, op):
        _, u0, u1 = self._sk_u(op)
        self.slot(op.s).copy_((u0 + u1).mean(dim=(1, 2)).reshape(-1))

    def op_sk_fc(self, op):
        B, f, d = op.B, op.f, op.d
        s = self.slot(op.s).view(B, f)
        w1 = self.pview(op.w1).view(d, f)
        w2 = self.pview(op.w2).view(2 * f, d)
        bn = op.bn
        zpre = s @ w1.t()
        gamma, beta = self.pview(bn.gamma), self.pview(bn.beta)
        mm, mv = self.pview(bn.mm), self.pview(bn.mv)
        if self.plan.meta["training"]:
            mean = zpre.mean(0)
            var = zpre.var(0, unbiased=False)
            mom = self.plan.meta.get("bn_momentum", 0.997)
            mm.copy_(mm * mom + mean * (1 - mom))
            mv.copy_(mv * mom + var * (B / max(B - 1, 1)) * (1 - mom))
        else:
            mean, var = mm.clone(), mv.clone()
        rstd = torch.rsqrt(var + self.eps)
        z = torch.relu((zpre - mean) * rstd * gamma + beta)
        a = z @ w2.t()
        att = torch.sigmoid(a[:, :f] - a[:, f:])
        self.slot(op.zpre).copy_(zpre.reshape(-1))
        self.slot(op.z).copy_(z.reshape(-1))
        self.slot(op.att).copy_(att.reshape(-1))
        bs = self.slot(bn.work)
        bs[:d] = mean
        bs[d:2 * d] = rstd

    def op_sk_combine(self, op):
        _, u0, u1 = self._sk_u(op)
        att = self.slot(op.att).view(op.B, 1, 1, op.f)
        self.store(op.v, att * u0 + (1 - att) * u1)

    def op_se_gap(self, op):
        y = self.t[op.y]
        sc, sh, _, _ = self.bn_scale_shift(op.bn)
        self.slot(op.q).copy_((y * sc + sh).mean(dim=(1, 2)).reshape(-1))

    def op_se_fc(self, op):
        B, C, r = op.B, op.C, op.r
        q = self.slot(op.q).view(B, C)
        w1 = self.pview(op.w1).view(r, C)
        w2 = self.pview(op.w2).view(C, r)
        h = torch.relu(q @ w1.t())
        e = torch.sigmoid(h @ w2.t())
        self.slot(op.h).copy_(h.reshape(-1))
        self.slot(op.e).copy_(e.reshape(-1))

    def op_blurpool(self, op):
        self.store(op.out, T.anti_aliased_downsample(self.t[op.x], op.filt, op.stride))

    def _avgpool(self, x, op):
        k, s, lo = op.k, op.stride, op.pad_lo
        H, W = x.shape[1:3]
        hi_h = (op.Ho - 1) * s + k - H - lo
        hi_w = (op.Wo - 1) * s + k - W - lo
        xp = F.pad(_nchw(x), (lo, max(hi_w, 0), lo, max(hi_h, 0)))
        ssum = F.avg_pool2d(xp, k, s) * (k * k)
        ssum = ssum[:, :, :op.Ho, :op.Wo]
        if op.count_pad:
            return _nhwc(ssum / (k * k))
        ones = F.pad(torch.ones(1, 1, H, W, dtype=x.dtype), (lo, max(hi_w, 0), lo, max(hi_h, 0)))
        cnt = (F.avg_pool2d(ones, k, s) * (k * k))[:, :, :op.Ho, :op.Wo]
        return _nhwc(ssum / cnt)

    def op_avgpool(self, op):
        self.store(op.out, self._avgpool(self.t[op.x], op))

    def _maxpool(self, x, op):
        k, s, lo = op.k, op.stride, op.pad_lo
        H, W = x.shape[1:3]
        hi_h = max((op.Ho - 1) * s + k - H - lo, 0)
        hi_w = max((op.Wo - 1) * s + k - W - lo, 0)
        xp = F.pad(_nchw(x), (lo, hi_w, lo, hi_h), value=float("-inf"))
        return _nhwc(F.max_pool2d(xp, k, s))

    def op_maxpool(self, op):
        self.store(op.out, self._maxpool(self.t[op.x], op))

    def op_gap(self, op):
        self.store(op.out, self.t[op.x].mean(dim=(1, 2)))

    def op_gem(self, op):
        """nets/blocks.py:22-42, p = 3; the clipped cube sum is kept for the backward."""
        x = self.t[op.x]
        s = (x.clamp(1e-6, 1e12) ** 3).sum(dim=(1, 2))
        self.slot(op.ssum).copy_(s.reshape(-1))
        self.store(op.out, float(op.HW) ** (-1.0 / 3) * s.clamp_min(1e-6) ** (1.0 / 3))

    def op_gem_bwd(self, op):
        x = self.t[op.x].clone().requires_grad_(True)
        y = T.generalized_mean_pooling(x)
        (dx,) = torch.autograd.grad(y, x, self.t[op.dpooled].reshape(y.shape))
        self.store(op.dx, dx)

    def op_dropblock_mask(self, op):
        """nets/blocks.py:209-246 with the uniform draws fed through plan.meta['dropblock_u']."""
        u = self.t[op.u].to(self.dtype)[None]
        keep, factor = T.dropblock_keep_mask(u, self.hp["keep_prob"], op.block_size, op.gamma_scale,
                                             op.H, op.W)
        self.slot(op.keep).copy_(keep.reshape(-1))
        self.slot(op.scale)[0] = factor

    def op_dropblock_apply(self, op):
        x = self.t[op.x]
        keep = self.slot(op.keep).view(1, *x.shape[1:])
        v = x * keep * self.slot(op.scale)[0]
        self.store(op.out, torch.relu(v) if op.relu else v)

    def op_kd_teacher(self, op):
        """softmax(teacher_logits / T), mixed with the batch's mixup pairing (data_util.py:128-156)."""
        p = torch.softmax(self.t[op.teacher_logits].to(self.dtype) / op.kd_temp, dim=1)
        if op.mode:
            lab = self.t[op.labels].long()
            y = F.one_hot(lab, op.NC).to(self.dtype)
            lam1 = self.t[op.lam1]
            lam2 = self.t[op.lam2] if op.lam2 else None
            _, _, p = T.mixup(torch.zeros(p.shape[0], 1, 1, 1, dtype=self.dtype), y, lam1, lam2,
                              keep_batch_size=(op.mode == 2), y_t=p)
        self.store(op.yt, p)

    def op_softmax_ce(self, op):
        logits = self.t[op.logits][:, :op.NC]
        y = self.t[op.y]
        ls = op.label_smoothing
        yp = y * (1 - ls) + ls / op.NC
        lsm = F.log_softmax(logits, dim=1)
        self.slot(op.loss)[0] += -(yp * lsm).sum(1).mean()
        gs = self.hp["grad_scale"]
        d = (torch.softmax(logits, 1) * yp.sum(1, keepdim=True) - yp) / op.B * gs
        if op.a.get("yt"):
            tt, Tk = self.t[op.yt], op.kd_temp
            self.slot(op.loss)[2] += Tk * Tk * -(tt * F.log_softmax(logits / Tk, dim=1)).sum(1).mean()
            d = d + Tk * (torch.softmax(logits / Tk, 1) * tt.sum(1, keepdim=True) - tt) / op.B * gs
        if op.dbias:
            self.pview(op.dbias, self.grads)[:op.NC] += d.sum(0)
        self.store(op.dlogits, F.pad(d, (0, op.ld - op.NC)))

    # ---------------------------------------------------------------- backward ops
    def _adjoint(self, fn, x_shape, dout):
        x = torch.zeros(x_shape, dtype=self.dtype, requires_grad=True)
        (dx,) = torch.autograd.grad(fn(x), x, dout)
        return dx

    def op_conv_wgrad(self, op):
        g = op.geom
        x, dy = self.t[op.x], self.t[op.dy]
        if x.dim() == 2:
            x = x[:, None, None, :]
        if dy.dim() == 2:
            dy = dy[:, None, None, :]
        if op.a.get("x_wpad"):
            lo, hi = op.x_wpad
            x = x[:, :, lo:x.shape[2] - hi, :]
        w = torch.zeros(g.Cout, g.kh, g.kw, g.Cin, dtype=self.dtype, requires_grad=True)
        (dw,) = torch.autograd.grad(self._conv(x, w, g), w, dy)
        if op.a.get("dw_slot") is not None:
            self.slot(op.dw_slot).add_(dw.reshape(-1))
        else:
            self.pview(op.w, self.grads).add_(dw)

    def op_conv_dgrad(self, op):
        g = op.geom
        dy = self.t[op.dy]
        two_d = dy.dim() == 2
        if two_d:
            dy = dy[:, None, None, :]
        w = self.wq(self.pview(op.w))
        dx = self._adjoint(lambda x: self._conv(x, w, g), (g.B, g.H, g.W, g.Cin), dy)
        dx = dx.reshape(self.plan.tensors[op.dx].shape)
        self.store(op.dx, self.grad_epilogue(dx, op.add_src, op.mask_src))

    def op_zero_insert(self, op):
        dy = self.t[op.dy]
        out = torch.zeros(op.B, op.H, op.W, op.C, dtype=self.dtype)
        out[:, 0:2 * op.Ho:2, 0:2 * op.Wo:2, :] = dy
        self.store(op.out, out)

    def op_s2d_wgrad_unpack(self, op):
        dw2 = self.slot(op.dw2).view(op.cout, op.k2, op.k2, 16)
        dw = self.pview(op.w, self.grads)
        k, pad, k2, pad2 = op.k, op.pad, op.k2, op.pad2
        for u in range(k):
            r, a = divmod(u - pad, 2)
            for v in range(k):
                s, b = divmod(v - pad, 2)
                dw[:, u, v, :] = dw2[:, r + pad2, s + pad2, (a * 2 + b) * 4:(a * 2 + b) * 4 + 3]

    def _eff_grad(self, g, op, B, C):
        if op.gate is not None:
            g = g * self._gate(op.gate, B, C)
        if op.addbc is not None:
            g = g + self.slot(op.addbc).view(B, 1, 1, C)
        return g

    def op_bn_bwd_reduce(self, op):
        g, y = self.t[op.g], self.t[op.y]
        B, _, _, C = y.shape
        _, _, mean, rstd = self.bn_scale_shift(op.bn)
        ge = self._eff_grad(g, op, B, C)
        s = self.slot(op.sums)              # row 0 of the partial buffer = the total
        s.zero_()
        s[:C] = ge.sum(dim=(0, 1, 2))
        s[C:2 * C] = (ge * (y - mean) * rstd).sum(dim=(0, 1, 2))

    def op_bn_bwd_finalize(self, op):
        bn = op.bn
        C = bn.C
        s = self.slot(op.sums)[:2 * C]
        w = self.slot(bn.work)
        mean, rstd = w[2 * C:3 * C], w[3 * C:4 * C]
        gamma = self.pview(bn.gamma)
        n = bn.count
        k1 = gamma * rstd
        k2 = -k1 * rstd * s[C:] / n
        k3 = -k1 * s[:C] / n - k2 * mean
        self.slot(op.coef).copy_(torch.cat([k1, k2, k3]))
        self.pview(bn.gamma, self.grads).copy_(s[C:])
        self.pview(bn.beta, self.grads).copy_(s[:C])

    def op_bn_bwd_apply(self, op):
        g, y = self.t[op.g], self.t[op.y]
        B, _, _, C = y.shape
        c = self.slot(op.coef)
        ge = self._eff_grad(g, op, B, C)
        self.store(op.dy, c[:C] * ge + c[C:2 * C] * y + c[2 * C:])

    def op_bn_bwd_reduce2(self, op):
        """Two batch norms fed by one gradient (plan.bn_backward2): two bn_bwd_reduce in one op."""
        g = self.t[op.g]
        for yname, bn, sums in ((op.y, op.bn, op.sums), (op.y2, op.bn2, op.sums2)):
            y = self.t[yname]
            C = y.shape[-1]
            _, _, mean, rstd = self.bn_scale_shift(bn)
            s = self.slot(sums)
            s.zero_()
            s[:C] = g.sum(dim=(0, 1, 2))
            s[C:2 * C] = (g * (y - mean) * rstd).sum(dim=(0, 1, 2))

    def op_bn_bwd_apply2(self, op):
        g = self.t[op.g]
        for yname, coef, dy in ((op.y, op.coef, op.dy), (op.y2, op.coef2, op.dy2)):
            y = self.t[yname]
            C = y.shape[-1]
            c = self.slot(coef)
            self.store(dy, c[:C] * g + c[C:2 * C] * y + c[2 * C:])

    def op_sk_bwd_gate(self, op):
        _, u0, u1 = self._sk_u(op)
        dv = self.t[op.dv]
        self.slot(op.dA).copy_((dv * (u0 - u1)).sum(dim=(1, 2)).reshape(-1))

    def op_sk_fc_bwd(self, op):
        B, f, d = op.B, op.f, op.d
        dA = self.slot(op.dA).view(B, f)
        att = self.slot(op.att).view(B, f)
        z = self.slot(op.z).view(B, d)
        zpre = self.slot(op.zpre).view(B, d)
        s = self.slot(op.s).view(B, f)
        w1 = self.pview(op.w1).view(d, f)
        w2 = self.pview(op.w2).view(2 * f, d)
        bn = op.bn
        bs = self.slot(bn.work)
        mean, rstd = bs[:d], bs[d:2 * d]
        gamma = self.pview(bn.gamma)
        da0 = att * (1 - att) * dA
        da = torch.cat([da0, -da0], 1)
        self.pview(op.w2, self.grads).view(2 * f, d).add_(da.t() @ z)
        dz = (da @ w2) * (z > 0)
        xh = (zpre - mean) * rstd
        s1, s2 = dz.sum(0), (dz * xh).sum(0)
        dzpre = gamma * rstd * (dz - s1 / B - xh * s2 / B)
        self.pview(bn.gamma, self.grads).add_(s2)
        self.pview(bn.beta, self.grads).add_(s1)
        self.pview(op.w1, self.grads).view(d, f).add_(dzpre.t() @ s)
        self.slot(op.ds).copy_((dzpre @ w1).reshape(-1))

    def _sk_g(self, op):
        y, u0, u1 = self._sk_u(op)
        dv = self.t[op.dv]
        att = self.slot(op.att).view(op.B, 1, 1, op.f)
        ds = self.slot(op.ds).view(op.B, 1, 1, op.f) / op.HW
        g0 = (att * dv + ds) * (u0 > 0)
        g1 = ((1 - att) * dv + ds) * (u1 > 0)
        return y, torch.cat([g0, g1], -1)

    def op_sk_bn_bwd_reduce(self, op):
        y, g = self._sk_g(op)
        _, _, mean, rstd = self.bn_scale_shift(op.bn)
        C = 2 * op.f
        s = self.slot(op.sums)
        s.zero_()
        s[:C] = g.sum(dim=(0, 1, 2))
        s[C:2 * C] = (g * (y - mean) * rstd).sum(dim=(0, 1, 2))

    def op_sk_bn_bwd_apply(self, op):
        y, g = self._sk_g(op)
        C = 2 * op.f
        c = self.slot(op.coef)
        self.store(op.dy, c[:C] * g + c[C:2 * C] * y + c[2 * C:])

    def op_se_bwd_gate(self, op):
        y = self.t[op.y]
        sc, sh, _, _ = self.bn_scale_shift(op.bn)
        self.slot(op.de).copy_((self.t[op.g] * (y * sc + sh)).sum(dim=(1, 2)).reshape(-1))

    def op_se_fc_bwd(self, op):
        B, C, r = op.B, op.C, op.r
        de = self.slot(op.de).view(B, C)
        e = self.slot(op.e).view(B, C)
        h = self.slot(op.h).view(B, r)
        q = self.slot(op.q).view(B, C)
        w1 = self.pview(op.w1).view(r, C)
        w2 = self.pview(op.w2).view(C, r)
        da2 = de * e * (1 - e)
        self.pview(op.w2, self.grads).view(C, r).add_(da2.t() @ h)
        da1 = (da2 @ w2) * (h > 0)
        self.pview(op.w1, self.grads).view(r, C).add_(da1.t() @ q)
        self.slot(op.dq).copy_(((da1 @ w1) / op.HW).reshape(-1))

    def op_blurpool_bwd(self, op):
        dx = self._adjoint(lambda x: T.anti_aliased_downsample(x, op.filt, op.stride),
                           (op.B, op.H, op.W, op.C), self.t[op.dout])
        self.store(op.dx, self.grad_epilogue(dx, op.add_src, op.mask_src))

    def op_avgpool_bwd(self, op):
        dx = self._adjoint(lambda x: self._avgpool(x, op), (op.B, op.H, op.W, op.C),
                           self.t[op.dout])
        self.store(op.dx, self.grad_epilogue(dx, op.add_src, op.mask_src))

    def op_maxpool_bwd(self, op):
        x = self.t[op.x].clone().requires_grad_(True)
        (dx,) = torch.autograd.grad(self._maxpool(x, op), x, self.t[op.dout])
        self.store(op.dx, self.grad_epilogue(dx, op.add_src, op.mask_src))

    def op_upsample2x_bwd(self, op):
        d = self.t[op.dout]
        dx = d.view(op.B, op.H, 2, op.W, 2, op.C).sum(dim=(2, 4))
        self.store(op.dx, self.grad_epilogue(dx, op.add_src, op.mask_src))

    def op_gap_bwd(self, op):
        dp = self.t[op.dpooled]
        dx = (dp / op.HW)[:, None, :].expand(op.B, op.HW, op.C)
        shape = self.plan.tensors[op.dx].shape
        self.store(op.dx, self.grad_epilogue(dx.reshape(shape), None, op.mask_src))

    def op_grad_combine(self, op):
        a = self.t[op.a["a"]].reshape(self.plan.tensors[op.out].shape)   # flatten head: a view
        self.store(op.out, self.grad_epilogue(a, op.add_src, op.mask_src))

    def op_sgd(self, op):
        hp = self.hp
        l2 = 0.0
        for name, p in self.plan.params.items():
            w = self.params[p.offset:p.offset + p.size]
            g = self.grads[p.offset:p.offset + p.size] * hp.get("sgd_grad_scale", 1.0)
            acc = self.momentum[p.offset:p.offset + p.size]
            if p.decay:
                l2 = l2 + 0.5 * hp["weight_decay"] * (w * w).sum()
                g = g + hp["weight_decay"] * w
            acc.copy_(hp["momentum"] * acc + g)
            w.sub_(hp["lr"] * acc)
        self.slot(op.loss)[1] += l2
